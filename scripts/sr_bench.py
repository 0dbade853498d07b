"""Super-resolution (SRVGGNetCompact and EDSR baseline) through feather::Net, and PixelShuffle and its fused tail alone.

    python scripts/sr_bench.py --out DIR [--reps 7] [--iters 10] [--layer-iters 100]

Models (device-resident input, CUDA graphs on): modelgen.srvgg_compact x 4 (realesr-animevideov3's layout) at 270 x 480
(1080p output) and 540 x 960 (4K output), batch 1 and 4; modelgen.edsr_baseline x 2 and x 4 at 270 x 480, batch 1.  For
each, images/s and latency per forward with fusion on and off (CUDA events, --reps windows of --iters forwards, the
median) and launches per forward; each kernel class's device time in an eager forward (fcuda_profile_collect_kind,
kind 13 is PixelShuffle) as a share of the forward.  In SRVGGNetCompact the element-wise class (kind 6) is PReLU alone
(the tail's Eltwise is fused away, and the script checks that its launches are the PReLU layers'), so its share is
reported as the PReLU share.
PixelShuffle alone (r = 4, mode 0, the SRVGGNetCompact tail's shapes) against a device-to-device copy of its input,
which moves the same bytes; the fused tail alone (with the nearest x 4 addend) against a copy of its input and addend,
and against PixelShuffle, Interp and Eltwise run as three calls into preallocated outputs.
Writes DIR/sr_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA device."""
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
from ssd_bench import timed  # noqa: E402
from style_bench import KINDS as STYLE_KINDS  # noqa: E402
from style_bench import load  # noqa: E402
from yolo_bench import time_calls  # noqa: E402

KINDS = STYLE_KINDS + ["pixel shuffle (PixelShuffle, alone or with its fused tail)"]
ELEMENTWISE = 6
CASES = [("srvgg_compact", dict(scale=4, height=270, width=480), 1), ("srvgg_compact", dict(scale=4, height=270, width=480), 4),
         ("srvgg_compact", dict(scale=4, height=540, width=960), 1), ("srvgg_compact", dict(scale=4, height=540, width=960), 4),
         ("edsr_baseline", dict(scale=2, height=270, width=480), 1), ("edsr_baseline", dict(scale=4, height=270, width=480), 1)]
TAIL_SHAPES = [(1, 270, 480), (4, 270, 480), (1, 540, 960), (4, 540, 960)]   # (batch, H, W) of conv_last, r = 4


def model_case(name, kw, batch, stream, reps, iters) -> dict:
    import numpy as np
    import torch
    from feathercnn_b200.tools import modelgen
    m = modelgen.ZOO[name](**kw)
    x = torch.from_numpy(np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])).cuda()
    res = {"model": name, **kw, "batch": batch, "gflop_per_image": m.flops / 1e9}
    n_prelu = sum(L.startswith("PReLU ") for L in m.lines)
    with tempfile.TemporaryDirectory() as d:
        param, binf = m.save(Path(d) / name)
        for fusion in (True, False):
            net = load(param, binf, x, stream, fusion)
            ms = timed(net, reps, iters)
            key = "fused" if fusion else "unfused"
            res[f"ms_{key}"] = ms
            res[f"images_per_s_{key}"] = batch / (ms * 1e-3)
            res[f"launches_{key}"] = net.launches_per_forward
            if fusion:
                mobilenet_v2_bench.KINDS = KINDS  # kind_shares reads the module's list
                shares = mobilenet_v2_bench.kind_shares(net)
                for k in shares:
                    k["share_of_forward"] = k["ms_per_forward"] / ms
                res["kind_shares_eager"] = shares
                if n_prelu:
                    ew = [k for k in shares if k["kind"] == ELEMENTWISE]
                    assert len(ew) == 1 and ew[0]["launches_per_forward"] == n_prelu, ew
                    res["prelu_share_of_forward"] = ew[0]["share_of_forward"]
            del net
    return res


def three_calls(x, base, shuffled, up, total):
    """PixelShuffle, nearest Interp x 4 and Eltwise SUM as three launches into preallocated outputs, as the unfused
    layers run them: the same allocation-free work as the fused tail apart from the two extra blobs."""
    import ctypes

    from feathercnn_b200 import booster
    lib = booster.fcuda()
    booster.pixel_shuffle(x, 4, 0, None, None, shuffled)
    n, c, h, w = base.shape
    p = booster.interp_param(h, w, 0, 0, "nearest", scale=4.0)
    booster._check("fcuda_interp_forward", lib.fcuda_interp_forward(ctypes.byref(p), booster._ptr(up), booster._ptr(base),
                                                                    c, n, booster._stream()))
    booster._check("fcuda_eltwise_add_forward",
                   lib.fcuda_eltwise_add_forward(booster._ptr(total), booster._ptr(shuffled), booster._ptr(up),
                                                 total.numel(), 0, booster._stream()))


def layers_alone(reps, iters) -> list[dict]:
    import torch
    from feathercnn_b200 import booster
    rows = []
    for n, h, w in TAIL_SHAPES:
        x = torch.randn(n, 48, h, w, device="cuda")
        base = torch.randn(n, 3, h, w, device="cuda")
        out = booster.pixel_shuffle(x, 4)
        up, total = torch.empty_like(out), torch.empty_like(out)
        src = torch.empty_like(x)
        src_tail = torch.empty(x.numel() + base.numel(), device="cuda")
        dst_tail = torch.empty_like(src_tail)
        ps = time_calls(lambda: booster.pixel_shuffle(x, 4, 0, None, None, out), reps, iters)
        copy = time_calls(lambda: src.copy_(x), reps, iters)
        tail = time_calls(lambda: booster.pixel_shuffle(x, 4, 0, base, 4.0, out), reps, iters)
        copy_tail = time_calls(lambda: dst_tail.copy_(src_tail), reps, iters)
        three = time_calls(lambda: three_calls(x, base, out, up, total), reps, iters)
        mb = x.numel() * 4e-6
        rows.append({"shape": [n, 48, h, w], "in_mb": mb, "addend_mb": base.numel() * 4e-6, "pixel_shuffle_ms": ps,
                     "d2d_copy_ms": copy, "pixel_shuffle_vs_copy": ps / copy, "tail_ms": tail,
                     "tail_d2d_copy_ms": copy_tail, "tail_vs_copy": tail / copy_tail, "three_calls_ms": three,
                     "three_calls_vs_tail": three / tail})
        del x, base, out, up, total, src, src_tail, dst_tail
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
    models = [model_case(name, kw, b, stream, args.reps, args.iters) for name, kw, b in CASES]
    alone = layers_alone(args.reps, args.layer_iters)
    info = card()
    res = {"card": info, "cuda_graph": True, "models": models, "layers_alone": alone}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "sr_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; CUDA graph, device-resident input", ""]
    for r in models:
        md.append(f"- {r['model']} x{r['scale']} {r['height']} x {r['width']} batch {r['batch']}: fused "
                  f"{r['ms_fused']:.2f} ms / forward ({r['images_per_s_fused']:.1f} images/s, {r['launches_fused']} "
                  f"launches), unfused {r['ms_unfused']:.2f} ms ({r['images_per_s_unfused']:.1f} images/s, "
                  f"{r['launches_unfused']} launches)"
                  + (f"; PReLU {r['prelu_share_of_forward']:.1%} of the forward" if "prelu_share_of_forward" in r else ""))
        for k in r["kind_shares_eager"]:
            md.append(f"  - {KINDS[k['kind']]}: {k['ms_per_forward']:.3f} ms ({k['share_of_forward']:.1%} of the "
                      f"forward, {k['share']:.1%} of the instrumented time), {k['launches_per_forward']:.0f} launches")
    md += ["", "| N x C x H x W (r = 4) | in MB | PixelShuffle ms | copy ms | vs copy | tail ms | copy (in + addend) ms | "
           "vs copy | three calls ms | three calls / tail |", "|---|---|---|---|---|---|---|---|---|---|"]
    for r in alone:
        md.append(f"| {' x '.join(map(str, r['shape']))} | {r['in_mb']:.1f} | {r['pixel_shuffle_ms']:.4f} | "
                  f"{r['d2d_copy_ms']:.4f} | {r['pixel_shuffle_vs_copy']:.2f} | {r['tail_ms']:.4f} | "
                  f"{r['tail_d2d_copy_ms']:.4f} | {r['tail_vs_copy']:.2f} | {r['three_calls_ms']:.4f} | "
                  f"{r['three_calls_vs_tail']:.2f} |")
    (out / "sr_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
