"""ResNet-50 R-FCN through feather::Net, and its PSROIPooling layer alone.

    python scripts/rfcn_bench.py --out DIR [--reps 7] [--iters 10] [--layer-iters 200]

Model (modelgen.rfcn_resnet50 at 600 x 800, 6000 / 300 proposals, fusion and CUDA graphs on, device-resident inputs):
images/s and latency per forward at batch 1 and 4 (CUDA events, --reps windows of --iters forwards, the median);
launches per forward; the share of each kernel class in an eager forward (fcuda_profile_collect_kind, kind 11 is
Proposal, ROIPooling and PSROIPooling); Proposal's and PSROIPooling's shares from a torch.profiler run of two eager
forwards of their own; and the share of the three dilated res5 3x3 convolutions: a net of those three layers alone (512
channels, 38 x 50, dilation 2, ReLU; the same convolution shapes) over the forward's time.
PSROIPooling alone (rfcn_cls's 1029 x 38 x 50 maps, 300 RoIs, 7 x 7 x 21 at 1/16) against a device-to-device copy of its
output bytes and against ROIPooling of a 21-channel 38 x 50 map over the same RoIs (the same output shape).
Writes DIR/rfcn_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

import mobilenet_v2_bench  # noqa: E402
from faster_rcnn_bench import HEIGHT, POST, WIDTH, kernel_ms, load  # noqa: E402
from shufflenet_v2_bench import KINDS as ROUTE_KINDS  # noqa: E402
from ssd_bench import timed  # noqa: E402
from yolo_bench import time_calls  # noqa: E402

KINDS = ROUTE_KINDS + ["two-stage detection (Proposal, ROIPooling, PSROIPooling)"]
CLASSES, POOLED = 21, 7
FEAT_H, FEAT_W = 38, 50  # res4f / res5c at 1 / 16 of 600 x 800


def res5_dilated_alone(batch: int, stream: int, reps: int, iters: int) -> float:
    """ms per forward of res5a/b/c_branch2b's shapes alone: three 512 -> 512 3x3 convolutions at dilation 2 and pad 2 on
    batch x 38 x 50, each with a ReLU, fused and graph-captured."""
    import numpy as np
    import torch
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter(0)
    x = m.input("x", 512, FEAT_H, FEAT_W)
    for blk in ("5a", "5b", "5c"):
        x = m.relu(f"relu{blk}", m.conv(f"res{blk}_branch2b", x, 512, 3, 1, 2, False, dilation=2))
    c, h, w = m.shape["x"]
    xs = torch.from_numpy(np.random.default_rng(0).uniform(0, 1, (batch, c, h, w)).astype(np.float32)).cuda()
    with tempfile.TemporaryDirectory() as d:
        param, binf = m.save(Path(d) / "res5")
        net = Net(fusion=True, cuda_graph=True)
        net.SetStream(stream)
        net.LoadParam(param)
        net.LoadWeights(binf)
    net.FeedInputDevice(xs.data_ptr(), tuple(xs.shape))
    return timed(net, reps, iters)


def psroi_pooling_alone(reps: int, iters: int) -> dict:
    import numpy as np
    import torch
    from feathercnn_b200 import booster
    rng = np.random.default_rng(1)
    h, w = FEAT_H, FEAT_W
    x = torch.from_numpy(rng.standard_normal((1, CLASSES * POOLED * POOLED, h, w)).astype(np.float32)).cuda()
    xy = rng.uniform(0, [WIDTH - 64, HEIGHT - 64], (POST, 2))
    wh = rng.uniform(32, 400, (POST, 2))
    rois = torch.from_numpy(np.concatenate([xy, np.minimum(xy + wh, [WIDTH - 1, HEIGHT - 1])], 1)
                            .astype(np.float32)[None]).cuda()
    out = booster.psroi_pooling(x, rois, POOLED, POOLED, CLASSES)
    dst = torch.empty_like(out)
    ms = time_calls(lambda: booster.psroi_pooling(x, rois, POOLED, POOLED, CLASSES), reps, iters)
    copy = time_calls(lambda: dst.copy_(out), reps, iters)
    x21 = x[:, :CLASSES].contiguous()
    roi = time_calls(lambda: booster.roi_pooling(x21, rois, POOLED, POOLED), reps, iters)
    return {"maps": [CLASSES * POOLED * POOLED, h, w], "rois": POST, "pooled": [POOLED, POOLED], "output_dim": CLASSES,
            "out_bytes": out.numel() * 4, "ms": ms, "d2d_copy_ms": copy, "vs_copy": ms / copy,
            "roi_pooling_21ch_ms": roi, "vs_roi_pooling": ms / roi}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forwards per timed window")
    ap.add_argument("--layer-iters", type=int, default=200, help="layer-alone calls per timed window")
    args = ap.parse_args()
    import torch
    from igemm_layer_bench import card
    from feathercnn_b200.tools import modelgen
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    mw = modelgen.rfcn_resnet50(height=HEIGHT, width=WIDTH)
    models = []
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / "rfcn_resnet50")
        for batch in (1, 4):
            net = load(param, binf, batch, stream)
            ms = timed(net, args.reps, args.iters)
            launches = net.launches_per_forward
            mobilenet_v2_bench.KINDS = KINDS  # kind_shares reads the module's list
            shares = mobilenet_v2_bench.kind_shares(net)  # leaves the graph off: the profile below is eager too
            k = kernel_ms(lambda: net.Forward(), ["proposal_", "psroi_pool_kernel"], 2)
            res5 = res5_dilated_alone(batch, stream, args.reps, args.iters)
            models.append({"batch": batch, "ms_per_forward": ms, "images_per_s": batch / (ms * 1e-3),
                           "launches_per_forward": launches, "kind_shares_eager": shares,
                           "proposal_share_eager": k["proposal_"] / k["total"],
                           "psroi_pooling_share_eager": k["psroi_pool_kernel"] / k["total"],
                           "res5_dilated_alone_ms": res5, "res5_dilated_share": res5 / ms})
            del net
    pool = psroi_pooling_alone(args.reps, args.layer_iters)
    info = card()
    res = {"card": info, "size": [HEIGHT, WIDTH], "fusion": True, "cuda_graph": True, "models": models,
           "psroi_pooling_alone": pool}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "rfcn_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; ResNet-50 R-FCN {HEIGHT} x {WIDTH}, 6000 / 300 "
          "proposals, fusion + CUDA graph, device-resident input", ""]
    for r in models:
        md.append(f"- batch {r['batch']}: {r['ms_per_forward']:.2f} ms / forward, {r['images_per_s']:.1f} images/s, "
                  f"{r['launches_per_forward']} launches / forward; eager shares: Proposal {r['proposal_share_eager']:.2%}, "
                  f"PSROIPooling {r['psroi_pooling_share_eager']:.2%}; dilated res5 3x3 alone "
                  f"{r['res5_dilated_alone_ms']:.2f} ms ({r['res5_dilated_share']:.1%} of the forward)")
    md += ["", "| kind | batch 1 ms / forward | share | batch 4 ms / forward | share |", "|---|---|---|---|---|"]
    for a, b in zip(models[0]["kind_shares_eager"], models[1]["kind_shares_eager"]):
        md.append(f"| {KINDS[a['kind']]} | {a['ms_per_forward']:.3f} | {a['share']:.1%} | {b['ms_per_forward']:.3f} | "
                  f"{b['share']:.1%} |")
    md += ["", f"PSROIPooling alone ({pool['maps'][0]} x {pool['maps'][1]} x {pool['maps'][2]}, {POST} RoIs, 7 x 7 x 21): "
           f"{pool['ms']:.4f} ms; a device-to-device copy of its {pool['out_bytes'] / 1e6:.2f} MB output "
           f"{pool['d2d_copy_ms']:.4f} ms ({pool['vs_copy']:.2f}x); ROIPooling of 21 channels over the same RoIs "
           f"{pool['roi_pooling_21ch_ms']:.4f} ms ({pool['vs_roi_pooling']:.2f}x)"]
    (out / "rfcn_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
