"""GoogLeNet and AlexNet (modelgen.googlenet / modelgen.alexnet) through feather::Net with fusion and CUDA graphs on:
images/s at batch 128, latency at batch 1, launches per forward, the share of each kernel class in an eager forward (the
profiling hook) and the share of GoogLeNet's Concat copies (torch.profiler, a run of its own), and the across-channel LRN
alone at norm1's shape (128 x 64 x 56 x 56) and norm2's (128 x 192 x 56 x 56) against a device-to-device copy of the same
bytes.

    python scripts/googlenet_bench.py --out DIR [--batch 128] [--reps 7] [--iters 10]

Device-resident input.  After a warm-up, --reps windows of --iters forwards (or kernel calls), timed with CUDA events;
the median window.  The LRN and the copy are timed alternately, window by window.  Writes DIR/googlenet_bench.json and
.md with the card's name and power limit, read in the same run.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

import mobilenet_v2_bench  # noqa: E402
from mobilenet_v2_bench import load  # noqa: E402
from ssd_bench import kind_shares, timed  # noqa: E402

LRN_TARGET = 1.25  # LRN / copy time, the yardstick of the channel-routing kernel
KINDS = mobilenet_v2_bench.KINDS[:6] + ["element-wise (BN/Scale/Eltwise/Clip/PReLU/Normalize/LRN)"] + \
    mobilenet_v2_bench.KINDS[7:] + ["detection head"]


def lrn_vs_copy(shape, reps: int, iters: int) -> dict:
    """Median ms of the across-channel LRN (local_size 5, the zoo's parameters) and of a device-to-device copy of the
    same blob."""
    import torch
    from feathercnn_b200 import booster
    x = torch.randn(shape, device="cuda")
    y = torch.empty_like(x)
    calls = {"lrn": lambda: booster.lrn(x, 0, 5, 1e-4, 0.75, 1.0, out=y), "copy": lambda: y.copy_(x)}
    for f in calls.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    for _ in range(reps):
        for k, f in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / iters)
    ms = {k: statistics.median(v) for k, v in times.items()}
    moved = 2 * x.numel() * 4  # read once + written once
    return {"shape": list(shape), "lrn_ms": ms["lrn"], "copy_ms": ms["copy"], "ratio": ms["lrn"] / ms["copy"],
            "target_ratio": LRN_TARGET, "lrn_GBps": moved / (ms["lrn"] * 1e-3) / 1e9,
            "copy_GBps": moved / (ms["copy"] * 1e-3) / 1e9}


def concat_share(net) -> dict:
    """Device time of the Concat copies (copy_channels_kernel) over all device time (kernels and copies) in two eager
    forwards."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    net._lib.fnet_set_cuda_graph(net._h, 0)
    try:
        net.Forward()
        net.Synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(2):
                net.Forward()
            net.Synchronize()
    finally:
        net._lib.fnet_set_cuda_graph(net._h, 1)
    total = copy = 0.0
    launches = 0
    for e in prof.events():
        if e.device_type != DeviceType.CUDA:
            continue
        t = e.time_range.elapsed_us()
        total += t
        if "copy_channels" in e.name:
            copy += t
            launches += 1
    return {"concat_ms_per_forward": copy / 2e3, "kernel_ms_per_forward": total / 2e3,
            "concat_share": copy / total if total else 0.0, "concat_launches_per_forward": launches / 2}


def run_model(name: str, batch: int, reps: int, iters: int) -> tuple[dict, object]:
    import numpy as np
    import torch
    from feathercnn_b200.tools import modelgen
    mw = modelgen.ZOO[name]()
    shape = mw.shape["data"]
    base = np.stack([modelgen.synthetic_input(shape, i) for i in range(min(batch, 8))])
    xb = torch.from_numpy(np.resize(base, (batch,) + tuple(shape))).cuda()
    x1 = xb[:1].contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / name)
        net_b = load(param, binf, True, xb, stream)
        net_1 = load(param, binf, True, x1, stream)
    ms_b = timed(net_b, reps, iters)
    ms_1 = timed(net_1, reps, iters)
    res = {"model": name, "size": shape[1], "batch": batch, "ms_per_forward": ms_b, "images_per_s": batch / (ms_b * 1e-3),
           "batch1_latency_ms": ms_1, "launches_per_forward": net_b.launches_per_forward,
           "kind_shares_eager": kind_shares(net_b)}
    del net_1
    return res, net_b


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forwards per timed window")
    args = ap.parse_args()
    import torch
    from igemm_layer_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    models = {}
    for name in ("googlenet", "alexnet"):
        res, net = run_model(name, args.batch, args.reps, args.iters)
        if name == "googlenet":
            res["concat"] = concat_share(net)
        models[name] = res
        del net
        torch.cuda.empty_cache()
    lrn = [lrn_vs_copy((args.batch, c, 56, 56), args.reps, 2 * args.iters) for c in (64, 192)]
    info = card()
    res = {"card": info, "fusion": True, "cuda_graph": True, "models": models, "lrn_alone": lrn}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "googlenet_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; fusion + CUDA graph, device-resident input", ""]
    for name, r in models.items():
        md += [f"- {name} {r['size']}x{r['size']}, batch {r['batch']}: {r['ms_per_forward']:.3f} ms / forward, "
               f"{r['images_per_s']:.0f} images/s, {r['launches_per_forward']} launches / forward; batch 1 latency "
               f"{r['batch1_latency_ms']:.3f} ms"]
    c = models["googlenet"]["concat"]
    md += [f"- googlenet Concat copies (torch.profiler, eager): {c['concat_ms_per_forward']:.3f} ms of "
           f"{c['kernel_ms_per_forward']:.3f} ms kernel time per forward, {c['concat_share']:.1%}, "
           f"{c['concat_launches_per_forward']:.0f} launches"]
    for r in lrn:
        md += [f"- LRN alone, {' x '.join(map(str, r['shape']))}: {r['lrn_ms']:.4f} ms ({r['lrn_GBps']:.0f} GB/s) against "
               f"a device-to-device copy of the same bytes {r['copy_ms']:.4f} ms ({r['copy_GBps']:.0f} GB/s): "
               f"{r['ratio']:.3f}x (target <= {LRN_TARGET}x)"]
    for name, r in models.items():
        md += ["", f"{name}, kernel classes, eager forward (CUDA events around every launch):", "",
               "| kind | ms / forward | share | launches / forward |", "|---|---|---|---|"]
        md += [f"| {KINDS[k['kind']]} | {k['ms_per_forward']:.3f} | {k['share']:.1%} | {k['launches_per_forward']:.0f} |"
               for k in r["kind_shares_eager"]]
    (out / "googlenet_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
