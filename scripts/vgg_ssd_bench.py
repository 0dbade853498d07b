"""VGG-SSD 300 (modelgen.vgg_ssd) through feather::Net with fusion and CUDA graphs on: images/s at batch 64, latency at
batch 1, launches per forward, the share of each kernel class in an eager forward, the head's share by difference (the
net against the same net cut before its head: Permute .. DetectionOutput), and the per-pixel Normalize alone at
conv4_3's shape (64 x 512 x 38 x 38) against a device-to-device copy of the same bytes.

    python scripts/vgg_ssd_bench.py --out DIR [--batch 64] [--reps 7] [--iters 10]

Device-resident input.  After a warm-up, --reps windows of --iters forwards (or kernel calls), timed with CUDA events;
the median window.  The Normalize and the copy are timed alternately, window by window.  Writes DIR/vgg_ssd_bench.json
and .md with the card's name and power limit, read in the same run.  Needs a CUDA device."""
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
from ssd_bench import headless, kind_shares, timed  # noqa: E402

NORM_TARGET = 1.25  # Normalize / copy time, the yardstick of the channel-routing kernel


def normalize_vs_copy(shape, reps: int, iters: int) -> dict:
    """Median ms of the per-pixel Normalize (out of place) and of a device-to-device copy of the same blob."""
    import torch
    from feathercnn_b200 import booster
    x = torch.randn(shape, device="cuda")
    y = torch.empty_like(x)
    s = torch.full((shape[1],), 20.0, device="cuda")
    calls = {"normalize": lambda: booster.normalize(x, s, 0, 1, 1e-10, 0, out=y), "copy": lambda: y.copy_(x)}
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
    return {"shape": list(shape), "normalize_ms": ms["normalize"], "copy_ms": ms["copy"],
            "ratio": ms["normalize"] / ms["copy"], "target_ratio": NORM_TARGET,
            "normalize_GBps": moved / (ms["normalize"] * 1e-3) / 1e9, "copy_GBps": moved / (ms["copy"] * 1e-3) / 1e9}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forwards per timed window")
    args = ap.parse_args()
    import numpy as np
    import torch
    from igemm_layer_bench import card
    from feathercnn_b200.tools import modelgen
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    mw = modelgen.vgg_ssd()
    shape = mw.shape["data"]
    base = np.stack([modelgen.synthetic_input(shape, i) for i in range(min(args.batch, 8))])
    xb = torch.from_numpy(np.resize(base, (args.batch,) + tuple(shape))).cuda()
    x1 = xb[:1].contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / "vgg_ssd")
        hparam, hbinf = headless(mw).save(Path(d) / "vgg_ssd_headless")
        net_b = load(param, binf, True, xb, stream)
        net_1 = load(param, binf, True, x1, stream)
        head_b = load(hparam, hbinf, True, xb, stream)
    ms_b = timed(net_b, args.reps, args.iters)
    ms_1 = timed(net_1, args.reps, args.iters)
    ms_headless = timed(head_b, args.reps, args.iters)
    shares = kind_shares(net_b)
    norm = normalize_vs_copy((args.batch,) + mw.shape["conv4_3_norm"], args.reps, 2 * args.iters)
    info = card()
    res = {"card": info, "model": "vgg_ssd", "size": shape[1], "fusion": True, "cuda_graph": True,
           "batch": args.batch, "ms_per_forward": ms_b, "images_per_s": args.batch / (ms_b * 1e-3),
           "batch1_latency_ms": ms_1, "launches_per_forward": net_b.launches_per_forward,
           "headless_ms_per_forward": ms_headless, "head_share_by_difference": (ms_b - ms_headless) / ms_b,
           "kind_shares_eager": shares, "normalize_alone": norm}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "vgg_ssd_bench.json").write_text(json.dumps(res, indent=1))
    names = mobilenet_v2_bench.KINDS + ["detection head"]
    md = [f"{info['name']}, power limit {info['power_limit']}; VGG-SSD {shape[1]}x{shape[2]}, fusion + CUDA graph, "
          "device-resident input", "",
          f"- batch {args.batch}: {ms_b:.3f} ms / forward, {res['images_per_s']:.0f} images/s, "
          f"{res['launches_per_forward']} launches / forward",
          f"- batch 1 latency: {ms_1:.3f} ms",
          f"- without the head (Permute .. DetectionOutput): {ms_headless:.3f} ms; head share "
          f"{res['head_share_by_difference']:.1%}",
          f"- Normalize alone, {' x '.join(map(str, norm['shape']))}: {norm['normalize_ms']:.4f} ms "
          f"({norm['normalize_GBps']:.0f} GB/s) against a device-to-device copy of the same bytes {norm['copy_ms']:.4f} ms "
          f"({norm['copy_GBps']:.0f} GB/s): {norm['ratio']:.3f}x (target <= {NORM_TARGET}x)", "",
          "Kernel classes, eager forward (CUDA events around every launch):", "",
          "| kind | ms / forward | share | launches / forward |", "|---|---|---|---|"]
    md += [f"| {names[r['kind']]} | {r['ms_per_forward']:.3f} | {r['share']:.1%} | {r['launches_per_forward']:.0f} |"
           for r in shares]
    (out / "vgg_ssd_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
