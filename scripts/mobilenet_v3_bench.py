"""What ncnn's activation layers cost: MobileNet-v3 Large / Small, EfficientNet-B0 and ESPCN through feather::Net, and the
activation kernel alone against a device-to-device copy of the same bytes.

    python scripts/mobilenet_v3_bench.py --out DIR [--reps 7] [--iters 5]

Whole nets: MobileNet-v3 Large and Small at 224 x 224, batch 256 and 1; EfficientNet-B0 at 224 x 224, batch 128 and 1;
ESPCN x 3 on a 360 x 640 Y plane, batch 1; and MobileNet-v2 at batch 256 as the point of comparison.  Fp32-split mode,
fusion on, device-resident input, CUDA graphs on.  After a warm-up, --reps windows of --iters forwards each, the nets
alternating window by window, timed with CUDA events on the nets' stream; the median window.  Then, in a run of its own
(the events bracket every launch), each kernel class's device time over two eager forwards
(fcuda_profile_collect_kind): kind 14 is the activation share, kind 4 the pooling share (the SE squeezes run on the
global pooling kernel), kind 6 the element-wise share (in these nets, with fusion on, the SE BinaryOp multiplies).

The kernel alone: each type, out of place and in place, at MobileNet-v3's stem activation (256 x 16 x 112 x 112 floats,
205 MB) and at an L2-resident 2 M floats, against torch's device-to-device copy of the same bytes, alternated.

Writes DIR/mobilenet_v3_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA
device."""
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

KINDS = ["TensorGEMM", "implicit-GEMM conv", "Winograd input", "Winograd output", "pooling", "depthwise",
         "element-wise", "deconvolution", "resize / crop", "detection", "routing", "two-stage detection",
         "instance norm / padding", "pixel shuffle", "activation"]
NETS = [("mobilenet_v3_large", 256), ("mobilenet_v3_large", 1), ("mobilenet_v3_small", 256), ("mobilenet_v3_small", 1),
        ("efficientnet_b0", 128), ("efficientnet_b0", 1), ("espcn", 1), ("mobilenet_v2", 256)]
ACT_TYPES = ["Sigmoid", "TanH", "Swish", "HardSigmoid", "HardSwish"]


def kind_shares(net) -> list[dict]:
    """Device time per kernel class over two eager forwards (the CUDA graph off for the profile)."""
    from feathercnn_b200 import booster
    lib = booster.fcuda()
    net._lib.fnet_set_cuda_graph(net._h, 0)
    net.Forward()
    net.Synchronize()
    lib.fcuda_profile_tensor_gemm(1)
    try:
        for _ in range(2):
            net.Forward()
        net.Synchronize()
        rows = []
        for kind, name in enumerate(KINDS):
            ms, af, mf, ab, n = (ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_double(),
                                 ctypes.c_longlong())
            lib.fcuda_profile_collect_kind(kind, ctypes.byref(ms), ctypes.byref(af), ctypes.byref(mf), ctypes.byref(ab),
                                           ctypes.byref(n))
            if n.value:
                rows.append({"kind": kind, "name": name, "ms_per_forward": ms.value / 2, "launches_per_forward": n.value / 2,
                             "bytes_per_forward": ab.value / 2})
    finally:
        lib.fcuda_profile_tensor_gemm(0)
        net._lib.fnet_set_cuda_graph(net._h, 1)
    total = sum(r["ms_per_forward"] for r in rows)
    for r in rows:
        r["share"] = r["ms_per_forward"] / total if total else 0.0
    return rows


def time_nets(cases, reps: int, iters: int) -> list[float]:
    from mobilenet_v2_bench import alternated
    return alternated([c["net"] for c in cases], reps, iters)


def time_calls(fns, reps: int, iters: int) -> list[float]:
    """Median ms per call of each function, their windows alternating."""
    import torch
    for f in fns:
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(reps):
        for k, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / iters)
    return [statistics.median(t) for t in times]


def kernel_alone(n: int, reps: int, iters: int) -> list[dict]:
    import torch
    from feathercnn_b200 import booster
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.rand(n, device="cuda", generator=gen) - 0.5) * 16
    y = torch.empty_like(x)
    z = x.clone()
    fns = [lambda: y.copy_(x)]
    for t in ACT_TYPES:
        fns.append(lambda t=t: booster.activation(x, t, 1.0 / 6.0, 0.5, out=y))
        fns.append(lambda t=t: booster.activation(z, t, 1.0 / 6.0, 0.5, out=z))  # in place: values drift, bytes do not
    ms = time_calls(fns, reps, iters)
    rows = [{"type": "copy", "mode": "d2d", "ms": ms[0], "vs_copy": 1.0, "GB_per_s": 8.0 * n / (ms[0] * 1e6)}]
    for i, t in enumerate(ACT_TYPES):
        for j, mode in enumerate(("out of place", "in place")):
            m = ms[1 + 2 * i + j]
            rows.append({"type": t, "mode": mode, "ms": m, "vs_copy": m / ms[0], "GB_per_s": 8.0 * n / (m * 1e6)})
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5, help="forwards per timed window")
    args = ap.parse_args()
    import numpy as np
    import torch
    from igemm_layer_bench import card
    from mobilenet_v2_bench import load
    from feathercnn_b200 import booster
    from feathercnn_b200.tools import modelgen
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    booster.set_precision(booster.PRECISION_FP32_SPLIT)
    stream = torch.cuda.current_stream().cuda_stream  # the stream the timing events are recorded on
    cases = []
    with tempfile.TemporaryDirectory() as d:
        for model, batch in NETS:
            mw = modelgen.ZOO[model]()
            shape = mw.shape["data"]
            base = np.stack([modelgen.synthetic_input(shape, i) for i in range(min(batch, 8))])
            x = torch.from_numpy(np.resize(base, (batch,) + tuple(shape))).cuda()
            param, binf = mw.save(Path(d) / model)
            cases.append({"model": model, "batch": batch, "shape": shape, "x": x, "net": load(param, binf, True, x, stream)})
    ms = time_nets(cases, args.reps, args.iters)
    nets = []
    for c, t in zip(cases, ms):
        shares = kind_shares(c["net"])
        share = {r["kind"]: r["share"] for r in shares}
        nets.append({"model": c["model"], "batch": c["batch"], "input": list(c["shape"]), "ms": t,
                     "images_per_s": c["batch"] / (t * 1e-3), "launches_per_forward": c["net"].launches_per_forward,
                     "activation_share": share.get(14, 0.0), "pooling_share": share.get(4, 0.0),
                     "elementwise_share": share.get(6, 0.0), "kind_shares_eager": shares})
        del c["net"], c["x"]
        torch.cuda.empty_cache()
    big = kernel_alone(256 * 16 * 112 * 112, args.reps, args.iters)
    small = kernel_alone(2 * 1024 * 1024, args.reps, 50 * args.iters)
    info = card()
    res = {"card": info, "precision": "fp32split", "fusion": True, "cuda_graph": True, "nets": nets,
           "kernel_alone": {"mobilenet_v3_stem_256x16x112x112": big, "l2_resident_2M": small}}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "mobilenet_v3_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; fp32-split, fusion on, device-resident input, CUDA graph, "
          f"median of {args.reps} alternated windows", "",
          "| net | batch | ms / forward | images/s | launches / forward | activation (14) | pooling (4) | "
          "element-wise (6) |", "|---|---|---|---|---|---|---|---|"]
    md += [f"| {r['model']} | {r['batch']} | {r['ms']:.3f} | {r['images_per_s']:.0f} | {r['launches_per_forward']} | "
           f"{r['activation_share']:.1%} | {r['pooling_share']:.1%} | {r['elementwise_share']:.1%} |" for r in nets]
    for title, rows in (("256 x 16 x 112 x 112 floats (205 MB)", big), ("2 M floats (8 MB, L2-resident)", small)):
        md += ["", f"Activation kernel alone, {title}:", "", "| type | mode | ms | x copy | GB/s (read + write) |",
               "|---|---|---|---|---|"]
        md += [f"| {r['type']} | {r['mode']} | {r['ms']:.4f} | {r['vs_copy']:.3f} | {r['GB_per_s']:.0f} |" for r in rows]
    (out / "mobilenet_v3_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
