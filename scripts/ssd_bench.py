"""MobileNet-SSD (modelgen.mobilenet_ssd, 300 x 300) through feather::Net with fusion and CUDA graphs on: images/s at batch
64, latency at batch 1, launches per forward, the share of each kernel class (kind 9 is the detection head: Permute, axis
Softmax, PriorBox, decode, NMS, merge), and DetectionOutput alone at MobileNet-SSD's size (P = 1917, C = 21, nms_top_k
100, keep_top_k 100) and at VGG-SSD / COCO's (P = 8732, C = 81, nms_top_k 400, keep_top_k 200).

    python scripts/ssd_bench.py --out DIR [--batch 64] [--reps 7] [--iters 10]

Device-resident input.  After a warm-up, --reps windows of --iters forwards, timed with CUDA events on the net's stream;
the median window.  The per-kind shares come from fcuda_profile_collect_kind over two eager forwards (a run of its own).
The whole-blob concatenations of the head (fcuda_copy_channels) are not profiled; the head's share is also given as the
difference between the net and the same net cut before its head.  Writes DIR/ssd_bench.json and .md with the card's name
and power limit, read in the same run.  Needs a CUDA device."""
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

HEAD_TYPES = ("Permute", "Flatten", "Reshape", "Softmax", "Concat", "PriorBox", "DetectionOutput")


def kind_shares(net) -> list[dict]:
    """mobilenet_v2_bench.kind_shares over kinds 0-9 (9: the detection head)."""
    kinds = mobilenet_v2_bench.KINDS
    mobilenet_v2_bench.KINDS = kinds + ["detection head"]
    try:
        return mobilenet_v2_bench.kind_shares(net)
    finally:
        mobilenet_v2_bench.KINDS = kinds


def timed(net, reps: int, iters: int) -> float:
    import torch
    for _ in range(3):
        net.Forward()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            net.Forward()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return statistics.median(times)


def headless(mw):
    """The same model without its detection head and without the loc / conf head convolutions' consumers: the backbone,
    extras and head convolutions only (their outputs unread)."""
    import copy
    m = copy.copy(mw)
    m.lines = [L for L in mw.lines if L.split()[0] not in HEAD_TYPES]
    m.blobs = {L.split()[4 + int(L.split()[2])] for L in m.lines}
    return m


def detection_alone(P, C, top, keep, batch, reps, iters) -> float:
    import numpy as np
    import torch
    from feathercnn_b200 import booster
    rng = np.random.default_rng(0)
    c = rng.uniform(0.05, 0.95, (P, 2))
    wh = rng.uniform(0.02, 0.5, (P, 2))
    pri = np.stack([np.concatenate([c - wh / 2, c + wh / 2], 1).reshape(-1), np.tile([0.1, 0.1, 0.2, 0.2], P)])
    pri = torch.from_numpy(pri.astype(np.float32)).cuda()
    loc = torch.randn((batch, 4 * P), device="cuda")
    conf = torch.softmax(torch.randn((batch, P, C), device="cuda") * 3, -1).reshape(batch, -1).contiguous()
    for _ in range(3):
        booster.detection_output(loc, conf, pri, C, 0.01, 0.45, top, keep)
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            booster.detection_output(loc, conf, pri, C, 0.01, 0.45, top, keep)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return statistics.median(times)


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
    mw = modelgen.mobilenet_ssd()
    shape = mw.shape["data"]
    base = np.stack([modelgen.synthetic_input(shape, i) for i in range(min(args.batch, 8))])
    xb = torch.from_numpy(np.resize(base, (args.batch,) + tuple(shape))).cuda()
    x1 = xb[:1].contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / "mobilenet_ssd")
        hparam, hbinf = headless(mw).save(Path(d) / "mobilenet_ssd_headless")
        net_b = load(param, binf, True, xb, stream)
        net_1 = load(param, binf, True, x1, stream)
        head_b = load(hparam, hbinf, True, xb, stream)
    ms_b = timed(net_b, args.reps, args.iters)
    ms_1 = timed(net_1, args.reps, args.iters)
    ms_headless = timed(head_b, args.reps, args.iters)
    shares = kind_shares(net_b)
    det = {"mobilenet_ssd_P1917_C21": {}, "vgg_ssd_coco_P8732_C81": {}}
    for key, (P, C, top, keep) in (("mobilenet_ssd_P1917_C21", (1917, 21, 100, 100)),
                                   ("vgg_ssd_coco_P8732_C81", (8732, 81, 400, 200))):
        for b in (1, args.batch):
            det[key][f"batch{b}_ms"] = detection_alone(P, C, top, keep, b, args.reps, args.iters)
    info = card()
    det_share = next((r["share"] for r in shares if r["kind"] == 9), 0.0)
    res = {"card": info, "model": "mobilenet_ssd", "size": shape[1], "fusion": True, "cuda_graph": True,
           "batch": args.batch, "ms_per_forward": ms_b, "images_per_s": args.batch / (ms_b * 1e-3),
           "batch1_latency_ms": ms_1, "launches_per_forward": net_b.launches_per_forward,
           "headless_ms_per_forward": ms_headless, "head_share_by_difference": (ms_b - ms_headless) / ms_b,
           "detection_kind_share_eager": det_share, "kind_shares_eager": shares, "detection_output_alone": det}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "ssd_bench.json").write_text(json.dumps(res, indent=1))
    names = mobilenet_v2_bench.KINDS + ["detection head"]
    md = [f"{info['name']}, power limit {info['power_limit']}; MobileNet-SSD {shape[1]}x{shape[2]}, fusion + CUDA graph, "
          "device-resident input", "",
          f"- batch {args.batch}: {ms_b:.3f} ms / forward, {res['images_per_s']:.0f} images/s, "
          f"{res['launches_per_forward']} launches / forward",
          f"- batch 1 latency: {ms_1:.3f} ms",
          f"- without the head (Permute .. DetectionOutput): {ms_headless:.3f} ms; head share "
          f"{res['head_share_by_difference']:.1%}", "",
          "Kernel classes, eager forward (CUDA events around every launch):", "",
          "| kind | ms / forward | share | launches / forward |", "|---|---|---|---|"]
    md += [f"| {names[r['kind']]} | {r['ms_per_forward']:.3f} | {r['share']:.1%} | {r['launches_per_forward']:.0f} |"
           for r in shares]
    md += ["", "DetectionOutput alone (decode + NMS + merge):", "", "| problem | batch 1 ms | batch "
           f"{args.batch} ms |", "|---|---|---|"]
    md += [f"| {k} | {v['batch1_ms']:.3f} | {v[f'batch{args.batch}_ms']:.3f} |" for k, v in det.items()]
    (out / "ssd_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
