"""DeepLab-v3 on MobileNet-v2 (modelgen.deeplabv3_mobilenet_v2, 513 x 513) at output stride 16 and 8 through feather::Net
with fusion and CUDA graphs on: images/s at batch 16, latency at batch 1, launches per forward, the share of each kernel
class in an eager forward (the profiling hook) and the dilated depthwise layers' share of an eager forward (torch.profiler,
a run of its own); and the dilated 3x3 depthwise kernel alone at the output-stride-8 shapes (16 x 576 x 65 x 65 at
dilation 2, 16 x 960 x 65 x 65 at dilation 4) against a device-to-device copy of the same bytes and the undilated depthwise
kernel at the same shape.

    python scripts/deeplab_bench.py --out DIR [--batch 16] [--reps 7] [--iters 10]

Device-resident input.  After a warm-up, --reps windows of --iters forwards (or kernel calls), timed with CUDA events;
the median window.  The dilated kernel, the copy and the undilated kernel are timed alternately, window by window.  Writes
DIR/deeplab_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA device."""
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

COPY_TARGET = 1.3        # dilated kernel / copy time
UNDILATED_TARGET = 1.10  # dilated / undilated depthwise kernel time
KINDS = mobilenet_v2_bench.KINDS[:6] + ["element-wise (BN/Scale/Eltwise/Clip/PReLU)"] + mobilenet_v2_bench.KINDS[7:] + \
    ["detection head"]


def dilated_share(net) -> dict:
    """Device time of the dilated depthwise kernels over all device time (kernels and copies) in two eager forwards."""
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
    total = dil = 0.0
    launches = 0
    for e in prof.events():
        if e.device_type != DeviceType.CUDA:
            continue
        t = e.time_range.elapsed_us()
        total += t
        if "dw3x3_dilated" in e.name:
            dil += t
            launches += 1
    return {"dilated_ms_per_forward": dil / 2e3, "kernel_ms_per_forward": total / 2e3,
            "dilated_share": dil / total if total else 0.0, "dilated_launches_per_forward": launches / 2}


def _depthwise(x, d: int):
    """A callable running the 3x3 / stride-1 / pad-d depthwise layer of dilation d on x (ConvBooster, DEPTHWISE)."""
    import torch
    from feathercnn_b200 import booster
    n, c, h, w = x.shape
    p = booster.ConvParam.make(c, c, h, w, 3, pad=d, group=c, bias=True)
    p.output_h, p.output_w = h, w
    cb = booster.ConvBooster()
    cb.ForceSelectAlgo(3)  # FCUDA_DEPTHWISE
    _, packed_n = cb.GetBufferSize(p, n)
    packed = torch.empty(packed_n, device="cuda")
    cb.Init(p, packed, torch.randn((c, 1, 3, 3), device="cuda") / 3)
    b = torch.rand(c, device="cuda") - 0.5
    y = torch.empty_like(x)
    scratch = torch.empty(1, device="cuda")
    return lambda: cb.ForwardOpts(p, y, x, packed, scratch, b, dilation=d, batch=n), y


def kernel_alone(shape, d: int, reps: int, iters: int) -> dict:
    """Median ms of the dilated kernel, a device-to-device copy of the input blob and the undilated kernel, alternated."""
    import torch
    x = torch.rand(shape, device="cuda") * 2 - 1
    dil, _ = _depthwise(x, d)
    und, _ = _depthwise(x, 1)
    y = torch.empty_like(x)
    calls = {"dilated": dil, "copy": lambda: y.copy_(x), "undilated": und}
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
    return {"shape": list(shape), "dilation": d, "dilated_ms": ms["dilated"], "copy_ms": ms["copy"],
            "undilated_ms": ms["undilated"], "vs_copy": ms["dilated"] / ms["copy"],
            "vs_undilated": ms["dilated"] / ms["undilated"], "target_vs_copy": COPY_TARGET,
            "target_vs_undilated": UNDILATED_TARGET, "dilated_GBps": moved / (ms["dilated"] * 1e-3) / 1e9,
            "copy_GBps": moved / (ms["copy"] * 1e-3) / 1e9}


def run_model(output_stride: int, batch: int, reps: int, iters: int) -> dict:
    import numpy as np
    import torch
    from feathercnn_b200.tools import modelgen
    mw = modelgen.deeplabv3_mobilenet_v2(output_stride=output_stride)
    shape = mw.shape["data"]
    base = np.stack([modelgen.synthetic_input(shape, i) for i in range(min(batch, 8))])
    xb = torch.from_numpy(np.resize(base, (batch,) + tuple(shape))).cuda()
    x1 = xb[:1].contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / f"deeplabv3_os{output_stride}")
        net_b = load(param, binf, True, xb, stream)
        net_1 = load(param, binf, True, x1, stream)
    ms_b = timed(net_b, reps, iters)
    ms_1 = timed(net_1, reps, iters)
    res = {"model": "deeplabv3_mobilenet_v2", "output_stride": output_stride, "size": shape[1], "batch": batch,
           "ms_per_forward": ms_b, "images_per_s": batch / (ms_b * 1e-3), "batch1_latency_ms": ms_1,
           "launches_per_forward": net_b.launches_per_forward, "kind_shares_eager": kind_shares(net_b),
           "dilated": dilated_share(net_b)}
    del net_1, net_b
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forwards per timed window")
    args = ap.parse_args()
    import torch
    from igemm_layer_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    models = {f"os{os_}": run_model(os_, args.batch, args.reps, args.iters) for os_ in (16, 8)}
    alone = [kernel_alone((args.batch, c, 65, 65), d, args.reps, 5 * args.iters) for c, d in ((576, 2), (960, 4))]
    info = card()
    res = {"card": info, "fusion": True, "cuda_graph": True, "models": models, "kernel_alone": alone}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "deeplab_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; fusion + CUDA graph, device-resident input", ""]
    for r in models.values():
        dl = r["dilated"]
        md += [f"- DeepLab-v3 MobileNet-v2 {r['size']}x{r['size']}, output stride {r['output_stride']}, batch {r['batch']}: "
               f"{r['ms_per_forward']:.3f} ms / forward, {r['images_per_s']:.1f} images/s, {r['launches_per_forward']} "
               f"launches / forward; batch 1 latency {r['batch1_latency_ms']:.3f} ms; dilated depthwise kernels "
               f"(torch.profiler, eager) {dl['dilated_ms_per_forward']:.3f} ms of {dl['kernel_ms_per_forward']:.3f} ms, "
               f"{dl['dilated_share']:.1%}, {dl['dilated_launches_per_forward']:.0f} launches"]
    for r in alone:
        md += [f"- dilated 3x3 depthwise alone, {' x '.join(map(str, r['shape']))}, dilation {r['dilation']}: "
               f"{r['dilated_ms']:.4f} ms ({r['dilated_GBps']:.0f} GB/s); device-to-device copy of the input "
               f"{r['copy_ms']:.4f} ms ({r['copy_GBps']:.0f} GB/s): {r['vs_copy']:.3f}x (target <= {COPY_TARGET}x); "
               f"undilated depthwise {r['undilated_ms']:.4f} ms: {r['vs_undilated']:.3f}x (target <= {UNDILATED_TARGET}x)"]
    for name, r in models.items():
        md += ["", f"{name}, kernel classes, eager forward (CUDA events around every launch):", "",
               "| kind | ms / forward | share | launches / forward |", "|---|---|---|---|"]
        md += [f"| {KINDS[k['kind']]} | {k['ms_per_forward']:.3f} | {k['share']:.1%} | {k['launches_per_forward']:.0f} |"
               for k in r["kind_shares_eager"]]
    (out / "deeplab_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
