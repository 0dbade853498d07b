"""VGG-16 Faster R-CNN through feather::Net, and its Proposal and ROIPooling layers alone.

    python scripts/faster_rcnn_bench.py --out DIR [--reps 7] [--iters 10] [--layer-iters 200]

Model (modelgen.faster_rcnn_vgg16 at 600 x 800, 6000 / 300 proposals, fusion and CUDA graphs on, device-resident
inputs): images/s and latency per forward at batch 1 and 4 (CUDA events, --reps windows of --iters forwards, the
median); launches per forward; the share of each kernel class in an eager forward (fcuda_profile_collect_kind, kind 11
is Proposal and ROIPooling); Proposal's and ROIPooling's shares from a torch.profiler run of two eager forwards of their
own; and the fc6 / fc7 share, the time of a net of fc6 -> ReLU -> fc7 -> ReLU alone over batch x 300 RoIs (the same
InnerProduct layers and shapes) over the forward's time.
Proposal alone (17,100 anchors: a 38 x 50 map, 6000 / 300, nms 0.7) at batch 1 and 4: the layer timed with CUDA events
and each of its four kernels from a torch.profiler run.  ROIPooling alone (512 x 38 x 50, 300 RoIs, 7 x 7 at 1/16)
against a device-to-device copy of its output bytes.
Writes DIR/faster_rcnn_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA
device."""
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
from shufflenet_v2_bench import KINDS as ROUTE_KINDS  # noqa: E402
from ssd_bench import timed  # noqa: E402
from yolo_bench import time_calls  # noqa: E402

KINDS = ROUTE_KINDS + ["two-stage detection (Proposal, ROIPooling)"]
PROPOSAL_KERNELS = ["proposal_decode_kernel", "proposal_select_kernel", "proposal_mask_kernel", "proposal_sweep_kernel"]
HEIGHT, WIDTH, POST = 600, 800, 300


def load(param, binf, batch, stream):
    """A fused, graph-captured Net fed device-resident data and im_info of `batch` images."""
    import numpy as np
    import torch
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    base = np.stack([modelgen.synthetic_input((3, HEIGHT, WIDTH), i) for i in range(batch)])
    x = torch.from_numpy(base).cuda()
    info = torch.tensor([[[[HEIGHT, WIDTH, 1.0]]]] * batch, dtype=torch.float32).cuda()
    net = Net(fusion=True, cuda_graph=True)
    net.SetStream(stream)
    net.LoadParam(param)
    net.LoadWeights(binf)
    net.FeedInputDevice(x.data_ptr(), tuple(x.shape))
    net.FeedInputDevice(info.data_ptr(), tuple(info.shape), "im_info")
    net._keep = (x, info)
    return net


def kernel_ms(fn, names, iters: int) -> dict:
    """Mean device ms per call of the kernels whose names contain each of `names`, and of all kernels ("total")."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in names}
    out["total"] = 0.0
    for ev in prof.key_averages():
        if ev.device_time_total <= 0:
            continue
        out["total"] += ev.device_time_total / 1000.0 / iters
        for k in names:
            if k in ev.key:
                out[k] += ev.device_time_total / 1000.0 / iters
    return out


def fc_alone(batch: int, stream: int, reps: int, iters: int) -> float:
    """ms per forward of fc6 -> ReLU -> fc7 -> ReLU over batch x 300 pooled RoIs, fused and graph-captured."""
    import numpy as np
    import torch
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter(0)
    x = m.input("pool5", 512, 7, 7)
    m.relu("relu7", m.fc("fc7", m.relu("relu6", m.fc("fc6", x, 4096)), 4096))
    xs = torch.from_numpy(np.random.default_rng(0).standard_normal((batch * POST, 512, 7, 7)).astype(np.float32)).cuda()
    with tempfile.TemporaryDirectory() as d:
        param, binf = m.save(Path(d) / "fc")
        net = Net(fusion=True, cuda_graph=True)
        net.SetStream(stream)
        net.LoadParam(param)
        net.LoadWeights(binf)
    net.FeedInputDevice(xs.data_ptr(), tuple(xs.shape))
    return timed(net, reps, iters)


def proposal_alone(batch: int, reps: int, iters: int) -> dict:
    import ctypes

    import numpy as np
    import torch
    from feathercnn_b200 import booster
    rng = np.random.default_rng(batch)
    h, w = 38, 50
    score = torch.from_numpy(rng.random((batch, 18, h, w), np.float32)).cuda()
    bbox = torch.from_numpy((rng.standard_normal((batch, 36, h, w)) * 0.1).astype(np.float32)).cuda()
    info = torch.tensor([[HEIGHT, WIDTH, 1.0]] * batch, dtype=torch.float32).cuda()
    p = booster.proposal_param()
    lib = booster.fcuda()
    ws = ctypes.c_size_t()
    booster._check("ws", lib.fcuda_proposal_workspace_size(ctypes.byref(p), h, w, batch, ctypes.byref(ws)))
    workspace = torch.empty(ws.value, device="cuda")
    rois = torch.empty((batch, POST, 4), device="cuda")
    scores = torch.empty((batch, POST), device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = [ctypes.c_void_p(t.data_ptr()) for t in (rois, scores, score, bbox, info)]

    def call():
        rc = lib.fcuda_proposal_forward(*args, ctypes.byref(p), h, w, ctypes.c_void_p(workspace.data_ptr()), batch,
                                        stream)
        assert rc == 0, rc
    call()
    torch.cuda.synchronize()
    kept = int((scores >= 0).sum().item()) / batch
    row = {"batch": batch, "anchors": 9 * h * w, "kept_per_image": kept, "ms": time_calls(call, reps, iters)}
    row.update({k: v for k, v in kernel_ms(call, PROPOSAL_KERNELS, iters).items() if k != "total"})
    return row


def roi_pooling_alone(reps: int, iters: int) -> dict:
    import numpy as np
    import torch
    from feathercnn_b200 import booster
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.standard_normal((1, 512, 38, 50)).astype(np.float32)).cuda()
    xy = rng.uniform(0, [WIDTH - 64, HEIGHT - 64], (POST, 2))
    wh = rng.uniform(32, 400, (POST, 2))
    rois = torch.from_numpy(np.concatenate([xy, np.minimum(xy + wh, [WIDTH - 1, HEIGHT - 1])], 1)
                            .astype(np.float32)[None]).cuda()
    out = booster.roi_pooling(x, rois)
    dst = torch.empty_like(out)
    ms = time_calls(lambda: booster.roi_pooling(x, rois), reps, iters)
    copy = time_calls(lambda: dst.copy_(out), reps, iters)
    return {"feature": [512, 38, 50], "rois": POST, "pooled": [7, 7], "out_bytes": out.numel() * 4, "ms": ms,
            "d2d_copy_ms": copy, "vs_copy": ms / copy}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forwards per timed window")
    ap.add_argument("--layer-iters", type=int, default=200, help="layer-alone calls per timed window and per profile")
    args = ap.parse_args()
    import torch
    from igemm_layer_bench import card
    from feathercnn_b200.tools import modelgen
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    mw = modelgen.faster_rcnn_vgg16(height=HEIGHT, width=WIDTH)
    models = []
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / "faster_rcnn_vgg16")
        for batch in (1, 4):
            net = load(param, binf, batch, stream)
            ms = timed(net, args.reps, args.iters)
            launches = net.launches_per_forward
            mobilenet_v2_bench.KINDS = KINDS  # kind_shares reads the module's list
            shares = mobilenet_v2_bench.kind_shares(net)  # leaves the graph off: the profile below is eager too
            k = kernel_ms(lambda: net.Forward(), ["proposal_", "roi_pool_kernel"], 2)
            fc = fc_alone(batch, stream, args.reps, args.iters)
            models.append({"batch": batch, "ms_per_forward": ms, "images_per_s": batch / (ms * 1e-3),
                           "launches_per_forward": launches, "kind_shares_eager": shares,
                           "proposal_share_eager": k["proposal_"] / k["total"],
                           "roi_pooling_share_eager": k["roi_pool_kernel"] / k["total"],
                           "fc6_fc7_alone_ms": fc, "fc6_fc7_share": fc / ms})
            del net
    heads = [proposal_alone(b, args.reps, args.layer_iters) for b in (1, 4)]
    pool = roi_pooling_alone(args.reps, args.layer_iters)
    info = card()
    res = {"card": info, "size": [HEIGHT, WIDTH], "fusion": True, "cuda_graph": True, "models": models,
           "proposal_alone": heads, "roi_pooling_alone": pool}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "faster_rcnn_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; VGG-16 Faster R-CNN {HEIGHT} x {WIDTH}, 6000 / 300 "
          "proposals, fusion + CUDA graph, device-resident input", ""]
    for r in models:
        md.append(f"- batch {r['batch']}: {r['ms_per_forward']:.2f} ms / forward, {r['images_per_s']:.1f} images/s, "
                  f"{r['launches_per_forward']} launches / forward; eager shares: Proposal {r['proposal_share_eager']:.2%}, "
                  f"ROIPooling {r['roi_pooling_share_eager']:.2%}; fc6 + fc7 alone {r['fc6_fc7_alone_ms']:.2f} ms "
                  f"({r['fc6_fc7_share']:.1%} of the forward)")
    md += ["", "| kind | batch 1 ms / forward | share | batch 4 ms / forward | share |", "|---|---|---|---|---|"]
    for a, b in zip(models[0]["kind_shares_eager"], models[1]["kind_shares_eager"]):
        md.append(f"| {KINDS[a['kind']]} | {a['ms_per_forward']:.3f} | {a['share']:.1%} | {b['ms_per_forward']:.3f} | "
                  f"{b['share']:.1%} |")
    md += ["", "Proposal alone (17,100 anchors, 6000 / 300), ms per call; kernels from torch.profiler:", "",
           "| batch | kept / image | layer | decode | select | mask | sweep |", "|---|---|---|---|---|---|---|"]
    md += [f"| {r['batch']} | {r['kept_per_image']:.0f} | {r['ms']:.4f} | " + " | ".join(f"{r[k]:.4f}" for k in PROPOSAL_KERNELS)
           + " |" for r in heads]
    md += ["", f"ROIPooling alone (512 x 38 x 50, 300 RoIs, 7 x 7): {pool['ms']:.4f} ms; a device-to-device copy of its "
           f"{pool['out_bytes'] / 1e6:.1f} MB output {pool['d2d_copy_ms']:.4f} ms ({pool['vs_copy']:.2f}x)"]
    (out / "faster_rcnn_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
