"""MobileNet-v2 (modelgen.mobilenet_v2, 224 x 224) through feather::Net at batch 256, the batch the benchmark runs
MobileNet-v1 at: images/s with the Clips (ReLU6) fused into the convolution epilogues and with fusion off, and the
share of each kernel class in one eager forward.

    python scripts/mobilenet_v2_bench.py --out DIR [--batch 256] [--reps 7] [--iters 5]

Device-resident input, CUDA graphs on.  After a warm-up, --reps windows of --iters forwards each, the fused and the
unfused net alternating window by window, timed with CUDA events on the nets' stream; the median window.  The
per-kind shares come from fcuda_profile_collect_kind over two eager forwards of the fused net (a run of its own: the
events bracket every launch).  Writes DIR/mobilenet_v2_bench.json and .md with the card's name and power limit, read
in the same run.  Needs a CUDA device."""
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
         "element-wise (BN/Scale/Eltwise/Clip/PReLU)", "deconvolution", "resize / crop"]


def load(param: str, binf: str, fusion: bool, x, stream: int):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=True)
    net.SetStream(stream)
    net.LoadParam(param)
    net.LoadWeights(binf)
    net.FeedInputDevice(x.data_ptr(), tuple(x.shape))
    return net


def alternated(nets, reps: int, iters: int) -> list[float]:
    """Median ms per forward of each net, their windows alternating."""
    import torch
    for net in nets:
        for _ in range(3):
            net.Forward()
    torch.cuda.synchronize()
    times = [[] for _ in nets]
    for _ in range(reps):
        for k, net in enumerate(nets):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                net.Forward()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / iters)
    return [statistics.median(t) for t in times]


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
                rows.append({"kind": kind, "name": name, "ms_per_forward": ms.value / 2, "launches_per_forward": n.value / 2})
    finally:
        lib.fcuda_profile_tensor_gemm(0)
        net._lib.fnet_set_cuda_graph(net._h, 1)
    total = sum(r["ms_per_forward"] for r in rows)
    for r in rows:
        r["share"] = r["ms_per_forward"] / total if total else 0.0
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5, help="forwards per timed window")
    args = ap.parse_args()
    import numpy as np
    import torch
    from igemm_layer_bench import card
    from feathercnn_b200.tools import modelgen
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    mw = modelgen.mobilenet_v2()
    shape = mw.shape["data"]
    base = np.stack([modelgen.synthetic_input(shape, i) for i in range(min(args.batch, 8))])
    x = torch.from_numpy(np.resize(base, (args.batch,) + tuple(shape))).cuda()
    stream = torch.cuda.current_stream().cuda_stream  # the stream the timing events are recorded on
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / "mobilenet_v2")
        fused, unfused = load(param, binf, True, x, stream), load(param, binf, False, x, stream)
    fused_ms, unfused_ms = alternated([fused, unfused], args.reps, args.iters)
    clips_fused = sum(fused.LayerFusedAway(n) == 1 for n in (line.split()[1] for line in mw.lines if line.startswith("Clip ")))
    shares = kind_shares(fused)
    info = card()
    res = {"card": info, "model": "mobilenet_v2", "size": shape[1], "batch": args.batch, "cuda_graph": True,
           "fused_ms": fused_ms, "unfused_ms": unfused_ms,
           "fused_images_per_s": args.batch / (fused_ms * 1e-3), "unfused_images_per_s": args.batch / (unfused_ms * 1e-3),
           "clips_fused": int(clips_fused), "clips": sum(line.startswith("Clip ") for line in mw.lines),
           "launches_per_forward": {"fused": fused.launches_per_forward, "unfused": unfused.launches_per_forward},
           "kind_shares_fused_eager": shares}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "mobilenet_v2_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; MobileNet-v2 {shape[1]}x{shape[2]}, batch {args.batch}, "
          f"device-resident input, CUDA graph", "",
          "| fusion | ms / forward | images/s | launches / forward |", "|---|---|---|---|",
          f"| on ({res['clips_fused']} of {res['clips']} Clips in conv epilogues) | {fused_ms:.3f} | "
          f"{res['fused_images_per_s']:.0f} | {res['launches_per_forward']['fused']} |",
          f"| off | {unfused_ms:.3f} | {res['unfused_images_per_s']:.0f} | {res['launches_per_forward']['unfused']} |", "",
          "Kernel classes, fusion on, eager forward (CUDA events around every launch):", "",
          "| kind | ms / forward | share | launches / forward |", "|---|---|---|---|"]
    md += [f"| {r['name']} | {r['ms_per_forward']:.3f} | {r['share']:.1%} | {r['launches_per_forward']:.0f} |" for r in shares]
    (out / "mobilenet_v2_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
