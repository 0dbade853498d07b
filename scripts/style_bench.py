"""Fast neural style transfer (TransformerNet) through feather::Net, and its InstanceNorm and Padding layers alone.

    python scripts/style_bench.py --out DIR [--reps 7] [--iters 10] [--layer-iters 100]

Model (modelgen.fast_neural_style, device-resident input, CUDA graphs on): at 512 x 512 batch 1 and 8 and at 1080 x 1920
batch 1, images/s and latency per forward with fusion on and off (CUDA events, --reps windows of --iters forwards, the
median); launches per forward; each kernel class's device time in an eager forward (fcuda_profile_collect_kind, kind 12
is InstanceNorm and Padding) as a share of the forward and of the instrumented launches; and the two 9 x 9 convolutions (conv1 3 -> 32, conv6 32 -> 3, both on im2col: 81 taps are
past the implicit GEMM's 63) each timed alone as a one-layer net of the same shape, with their share of the forward.
InstanceNorm alone at (32, 512, 512), (128, 128, 128) and (32, 1080, 1920), without and with a fused reflect pad of 1,
each against a device-to-device copy of the same bytes (the input blob; with the pad, the padded output); Padding alone
(reflect 1 and 4) against a copy of its output.
Writes DIR/style_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA device."""
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
from rfcn_bench import KINDS as RCNN_KINDS  # noqa: E402
from ssd_bench import timed  # noqa: E402
from yolo_bench import time_calls  # noqa: E402

KINDS = RCNN_KINDS + ["instance normalisation / padding (InstanceNorm, Padding)"]
CASES = [(512, 512, 1), (512, 512, 8), (1080, 1920, 1)]
IN_SHAPES = [(32, 512, 512), (128, 128, 128), (32, 1080, 1920)]


def load(param, binf, x, stream, fusion):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=True)
    net.SetStream(stream)
    net.LoadParam(param)
    net.LoadWeights(binf)
    net.FeedInputDevice(x.data_ptr(), tuple(x.shape))
    return net


def conv9_alone(name, ic, oc, h, w, batch, stream, reps, iters) -> float:
    """ms per forward of one 9 x 9 convolution (pad 0, bias) on a batch x ic x (h + 8) x (w + 8) input, graph-captured:
    the shape of `name` in fast_neural_style."""
    import numpy as np
    import torch
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter(0)
    m.conv(name, m.input("x", ic, h + 8, w + 8), oc, 9, 1, 0, True)
    xs = torch.from_numpy(np.random.default_rng(0).uniform(0, 1, (batch, ic, h + 8, w + 8)).astype(np.float32)).cuda()
    with tempfile.TemporaryDirectory() as d:
        param, binf = m.save(Path(d) / name)
        net = load(param, binf, xs, stream, True)
    ms = timed(net, reps, iters)
    del net
    return ms


def model_case(h, w, batch, stream, reps, iters) -> dict:
    import numpy as np
    import torch
    from feathercnn_b200.tools import modelgen
    m = modelgen.fast_neural_style(height=h, width=w)
    x = torch.from_numpy(np.stack([modelgen.synthetic_input((3, h, w), i) for i in range(batch)])).cuda()
    res = {"size": [h, w], "batch": batch, "gflop_per_image": m.flops / 1e9}
    with tempfile.TemporaryDirectory() as d:
        param, binf = m.save(Path(d) / "style")
        for fusion in (True, False):
            net = load(param, binf, x, stream, fusion)
            ms = timed(net, reps, iters)
            key = "fused" if fusion else "unfused"
            res[f"ms_{key}"] = ms
            res[f"images_per_s_{key}"] = batch / (ms * 1e-3)
            res[f"launches_{key}"] = net.launches_per_forward
            if fusion:
                mobilenet_v2_bench.KINDS = KINDS  # kind_shares reads the module's list
                res["kind_shares_eager"] = mobilenet_v2_bench.kind_shares(net)
                # `share` is over the instrumented launches only (im2col's gather is not one of them); this is the
                # class's eager device time over the whole graph-replayed forward
                for k in res["kind_shares_eager"]:
                    k["share_of_forward"] = k["ms_per_forward"] / ms
            del net
    res["conv1_9x9_ms"] = conv9_alone("conv1", 3, 32, h, w, batch, stream, reps, iters)
    res["conv6_9x9_ms"] = conv9_alone("conv6", 32, 3, h, w, batch, stream, reps, iters)
    res["conv9x9_share"] = (res["conv1_9x9_ms"] + res["conv6_9x9_ms"]) / res["ms_fused"]
    return res


def layers_alone(reps, iters) -> dict:
    import torch
    from feathercnn_b200 import booster
    rows = []
    for c, h, w in IN_SHAPES:
        x = torch.randn(1, c, h, w, device="cuda") * 2 + 0.5
        g, b = torch.rand(c, device="cuda") + 0.5, torch.rand(c, device="cuda") - 0.5
        for pad in (None, (1, 1, 1, 1, 2, 0.0)):
            out = booster.instance_norm(x, g, b, 1e-5, True, pad)
            src = out if pad else x
            dst = torch.empty_like(src)
            ms = time_calls(lambda: booster.instance_norm(x, g, b, 1e-5, True, pad, out), reps, iters)
            copy = time_calls(lambda: dst.copy_(src), reps, iters)
            rows.append({"layer": "InstanceNorm+ReLU" + ("+reflect pad 1" if pad else ""), "shape": [c, h, w],
                         "in_mb": x.numel() * 4e-6, "out_mb": out.numel() * 4e-6, "ms": ms, "d2d_copy_ms": copy,
                         "vs_copy": ms / copy})
        for p in (1, 4):
            out = booster.padding(x, p, p, p, p, 2)
            dst = torch.empty_like(out)
            ms = time_calls(lambda: booster.padding(x, p, p, p, p, 2, 0.0, out), reps, iters)
            copy = time_calls(lambda: dst.copy_(out), reps, iters)
            rows.append({"layer": f"Padding reflect {p}", "shape": [c, h, w], "in_mb": x.numel() * 4e-6,
                         "out_mb": out.numel() * 4e-6, "ms": ms, "d2d_copy_ms": copy, "vs_copy": ms / copy})
        del x
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forwards per timed window")
    ap.add_argument("--layer-iters", type=int, default=100, help="layer-alone calls per timed window")
    args = ap.parse_args()
    import torch
    from igemm_layer_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    models = [model_case(h, w, b, stream, args.reps, args.iters) for h, w, b in CASES]
    alone = layers_alone(args.reps, args.layer_iters)
    info = card()
    res = {"card": info, "cuda_graph": True, "models": models, "layers_alone": alone}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "style_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; fast_neural_style, CUDA graph, device-resident input", ""]
    for r in models:
        md.append(f"- {r['size'][0]} x {r['size'][1]} batch {r['batch']}: fused {r['ms_fused']:.2f} ms / forward "
                  f"({r['images_per_s_fused']:.1f} images/s, {r['launches_fused']} launches), unfused "
                  f"{r['ms_unfused']:.2f} ms ({r['launches_unfused']} launches); 9 x 9 alone: conv1 "
                  f"{r['conv1_9x9_ms']:.2f} ms, conv6 {r['conv6_9x9_ms']:.2f} ms ({r['conv9x9_share']:.1%} of the "
                  "fused forward)")
        for k in r["kind_shares_eager"]:
            md.append(f"  - {KINDS[k['kind']]}: {k['ms_per_forward']:.3f} ms ({k['share_of_forward']:.1%} of the "
                      f"forward, {k['share']:.1%} of the instrumented time), {k['launches_per_forward']:.0f} launches")
    md += ["", "| layer | C x H x W | in MB | out MB | ms | copy ms | vs copy |", "|---|---|---|---|---|---|---|"]
    for r in alone:
        md.append(f"| {r['layer']} | {' x '.join(map(str, r['shape']))} | {r['in_mb']:.1f} | {r['out_mb']:.1f} | "
                  f"{r['ms']:.4f} | {r['d2d_copy_ms']:.4f} | {r['vs_copy']:.2f} |")
    (out / "style_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
