"""Timing of the Interp and Crop kernels (fcuda_interp_forward, fcuda_crop_forward) on segmentation-head shapes, against
a device-to-device cudaMemcpyAsync of the same output bytes, and modelgen.fcn8s_tiny through feather::Net with and
without the Crop folded into its last deconvolution.

    python scripts/seg_layer_bench.py --out DIR [--reps 9] [--iters 20]

Per case, CUDA-event times: after a warm-up, --reps windows of --iters launches each, the case and its copy alternating
window by window; the median window.  GB/s counts the input read once plus the output written once (the bytes the
library's profiling kind 8 reports), against the H100 SXM data sheet's 3.35 TB/s; the copy moves the output's bytes
once in and once out.  "x copy" is the kernel's time over the copy's.  Writes DIR/seg_layer_bench.json and
DIR/seg_layer_bench.md with the card's name and power limit.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import ctypes
import json
import statistics
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

HBM_DATASHEET = 3.35e12  # H100 SXM data sheet (not a measured figure)
BATCH, CLASSES = 16, 21

# (name, kind, (H, W), (OH, OW) or crop (coff, hoff, woff, oc, oh, ow), mode, align)
CASES = [(f"{mode} {'align ' if align else ''}x{f} {512 // f}->512", "interp", (512 // f, 512 // f), (512, 512), mode, align)
         for mode, align in (("nearest", 0), ("bilinear", 0), ("bilinear", 1)) for f in (2, 4, 8)]
CASES += [
    ("bilinear x0.5 512->256", "interp", (512, 512), (256, 256), "bilinear", 0),
    ("nearest x0.5 512->256", "interp", (512, 512), (256, 256), "nearest", 0),
    ("crop FCN-8s score 568->500 off 31", "crop", (568, 568), (0, 31, 31, CLASSES, 500, 500), None, 0),
    ("crop 568->500 off 32 (float4)", "crop", (568, 568), (0, 32, 32, CLASSES, 500, 500), None, 0),
    ("crop FCN score_pool4c 44->34 off 5", "crop", (44, 44), (0, 5, 5, CLASSES, 34, 34), None, 0),
]


def alternated(fns, reps: int, iters: int) -> list[float]:
    """Median ms per launch of each fn, the fns' windows alternating."""
    import torch
    for fn in fns:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(reps):
        for k, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / iters)
    return [statistics.median(t) for t in times]


def _cudart():
    from feathercnn_b200._lib import fcuda
    fcuda()  # libfcuda.so links the CUDA runtime; dlopen by soname returns that already-loaded copy
    for name in ("libcudart.so.12", "libcudart.so"):
        try:
            rt = ctypes.CDLL(name)
            rt.cudaMemcpyAsync.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
            rt.cudaMemcpyAsync.restype = ctypes.c_int
            return rt
        except OSError:
            continue
    raise SystemExit("the CUDA runtime library is not loadable")


def bench_case(case, reps, iters, rt) -> dict:
    import torch
    from feathercnn_b200 import booster
    name, kind, (h, w), geo, mode, align = case
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand((BATCH, CLASSES, h, w), device="cuda", generator=g) * 2 - 1
    if kind == "interp":
        oh, ow = geo
        p = booster.interp_param(h, w, oh, ow, mode, bool(align))
        out = torch.empty((BATCH, CLASSES, oh, ow), device="cuda")
        args = (ctypes.byref(p), booster._ptr(out), booster._ptr(x), CLASSES, BATCH, booster._stream())
        lib = booster.fcuda()
        fn = lambda: booster._check("fcuda_interp_forward", lib.fcuda_interp_forward(*args))  # noqa: E731
        in_bytes = x.numel() * 4
    else:
        co, ho, wo, oc, oh, ow = geo
        out = torch.empty((BATCH, oc, oh, ow), device="cuda")
        lib = booster.fcuda()
        args = (booster._ptr(out), booster._ptr(x), CLASSES, h, w, co, ho, wo, oc, oh, ow, BATCH, booster._stream())
        fn = lambda: booster._check("fcuda_crop_forward", lib.fcuda_crop_forward(*args))  # noqa: E731
        in_bytes = out.numel() * 4  # the window is read once
    out_bytes = out.numel() * 4
    src = torch.empty_like(out)
    dst = torch.empty_like(out)
    stream = booster._stream()

    def copy():
        rc = rt.cudaMemcpyAsync(ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(src.data_ptr()), out_bytes, 3, stream)
        if rc:
            raise RuntimeError(f"cudaMemcpyAsync returned {rc}")

    ms, copy_ms = alternated([fn, copy], reps, iters)
    algo_bytes = in_bytes + out_bytes
    return {"case": name, "batch": BATCH, "channels": CLASSES, "in": [h, w], "out": [oh, ow], "ms": ms, "copy_ms": copy_ms,
            "algo_bytes": algo_bytes, "gbps": algo_bytes / ms / 1e6, "share_of_hbm": algo_bytes / ms * 1e3 / HBM_DATASHEET,
            "copy_gbps": 2 * out_bytes / copy_ms / 1e6, "x_copy": ms / copy_ms}


def bench_fcn(reps, iters, size=500, batch=8) -> dict:
    import numpy as np
    import torch
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    mw = modelgen.fcn8s_tiny(size=size, classes=CLASSES)
    x = np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(batch)])
    nets = {}
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / "fcn8s_tiny")
        for fusion in (False, True):
            net = Net(fusion=fusion, cuda_graph=True)
            net.SetStream(torch.cuda.current_stream().cuda_stream)  # the stream the timing events are recorded on
            net.LoadParam(param)
            net.LoadWeights(binf)
            net.FeedInputBatch(x)
            nets[fusion] = net
    unfused_ms, fused_ms = alternated([nets[False].Forward, nets[True].Forward], reps, iters)
    same = np.array_equal(nets[False].Extract("score").view(np.int32), nets[True].Extract("score").view(np.int32))
    return {"model": "fcn8s_tiny", "size": size, "batch": batch, "classes": CLASSES, "upscore8": list(mw.shape["upscore8"]),
            "unfused_ms": unfused_ms, "fused_ms": fused_ms, "score_bit_identical": bool(same),
            "crop_folded": nets[True].LayerFusedAway("score") == 1}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--iters", type=int, default=20, help="launches per timed window")
    args = ap.parse_args()
    import torch
    from igemm_layer_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    rt = _cudart()
    rows = [bench_case(c, args.reps, args.iters, rt) for c in CASES]
    fcn = bench_fcn(args.reps, max(args.iters // 4, 3))
    info = card()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "seg_layer_bench.json").write_text(json.dumps({"card": info, "rows": rows, "fcn8s_tiny": fcn}, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; batch {BATCH}, {CLASSES} channels", "",
          "| case | kernel ms | GB/s (share of 3.35 TB/s) | copy ms | copy GB/s | x copy |", "|---|---|---|---|---|---|"]
    for r in rows:
        md.append(f"| {r['case']} | {r['ms']:.3f} | {r['gbps']:.0f} ({r['share_of_hbm']:.0%}) | {r['copy_ms']:.3f} | "
                  f"{r['copy_gbps']:.0f} | {r['x_copy']:.2f} |")
    md += ["", f"fcn8s_tiny {fcn['size']}x{fcn['size']}, batch {fcn['batch']}, CUDA graph: fusion off {fcn['unfused_ms']:.3f} ms, "
           f"fusion on (ReLUs fused, final Crop folded: {fcn['crop_folded']}) {fcn['fused_ms']:.3f} ms per forward; "
           f"score bit-identical: {fcn['score_bit_identical']}"]
    (out / "seg_layer_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
