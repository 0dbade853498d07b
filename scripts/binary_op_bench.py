"""ncnn's BinaryOp alone, and ResNet-50 and SRVGGNetCompact with their adds written as Eltwise SUM or as BinaryOp ADD.

    python scripts/binary_op_bench.py --out DIR [--reps 7] [--iters 10] [--layer-iters 100]

BinaryOp alone at ResNet-50's res2 size at batch 128 (128 x 256 x 56 x 56), each against a device-to-device copy that
moves the same bytes (CUDA events, --reps windows of --layer-iters calls, the median): the same-shape ADD (two inputs,
one output: a copy of 1.5 blobs), a per-channel MUL ([N, C, H, W] x [N, C, 1, 1]), a scalar MUL, and a row broadcast
ADD ([N, C, H, W] + [N, 1, 1, W]); the last three read one full blob and write one, as a copy of it does.
Whole nets (device-resident input, CUDA graphs and fusion on): modelgen.resnet50 at 224 x 224 batch 128 and
modelgen.srvgg_compact x 4 at 270 x 480 (1080p output) batch 1, each in the "eltwise" and "binaryop" layouts, measured
alternately in the same run: images/s per layout (the median of the windows) and launches per forward.
Writes DIR/binary_op_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA
device."""
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

from ssd_bench import timed  # noqa: E402
from style_bench import load  # noqa: E402
from yolo_bench import time_calls  # noqa: E402

RES2 = (128, 256, 56, 56)
NETS = [("resnet50", dict(size=224), 128), ("srvgg_compact", dict(scale=4, height=270, width=480), 1)]
ROUNDS = 3   # eltwise / binaryop alternations per net


def layers_alone(reps, iters) -> list[dict]:
    import torch
    from feathercnn_b200 import booster
    n, c, h, w = RES2
    a = torch.randn(RES2, device="cuda")
    cases = [("same-shape ADD", torch.randn(RES2, device="cuda"), 0, 3),
             ("per-channel MUL", torch.randn(n, c, 1, 1, device="cuda"), 2, 2),
             ("scalar MUL", 0.5, 2, 2),
             ("row-broadcast ADD", torch.randn(n, 1, 1, w, device="cuda"), 0, 2)]
    out = torch.empty_like(a)
    rows = []
    for name, b, op, blobs in cases:
        src = torch.empty(a.numel() * blobs // 2, device="cuda")   # a copy reads and writes it: `blobs` blobs moved
        dst = torch.empty_like(src)
        t = time_calls(lambda: booster.binary_op(a, b, op, False, out), reps, iters)
        copy = time_calls(lambda: dst.copy_(src), reps, iters)
        mb = a.numel() * 4e-6 * blobs
        rows.append({"case": name, "shape": list(RES2), "b_shape": list(b.shape) if torch.is_tensor(b) else "scalar",
                     "op": op, "mb_moved": mb, "binary_op_ms": t, "d2d_copy_ms": copy, "vs_copy": t / copy,
                     "gb_per_s": mb * 1e-3 / (t * 1e-3)})
        del src, dst
    return rows


def nets(stream, reps, iters) -> list[dict]:
    import numpy as np
    import torch
    from feathercnn_b200.tools import modelgen
    rows = []
    for name, kw, batch in NETS:
        m = modelgen.ZOO[name](**kw)
        x = torch.from_numpy(np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])).cuda()
        with tempfile.TemporaryDirectory() as d:
            loaded = {}
            for adds in ("eltwise", "binaryop"):
                param, binf = modelgen.ZOO[name](adds=adds, **kw).save(Path(d) / adds)
                loaded[adds] = load(param, binf, x, stream, True)
        times = {adds: [] for adds in loaded}
        for _ in range(ROUNDS):
            for adds, net in loaded.items():
                times[adds].append(timed(net, reps, iters))
        row = {"model": name, **kw, "batch": batch}
        for adds, net in loaded.items():
            ms = statistics.median(times[adds])
            row[adds] = {"ms": ms, "ms_rounds": times[adds], "images_per_s": batch / (ms * 1e-3),
                         "launches_per_forward": net.launches_per_forward}
        rows.append(row)
        del loaded, x
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
    alone = layers_alone(args.reps, args.layer_iters)
    whole = nets(stream, args.reps, args.iters)
    info = card()
    res = {"card": info, "layers_alone": alone, "nets": whole}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "binary_op_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}", "",
          f"BinaryOp alone, a = {' x '.join(map(str, RES2))} (ResNet-50 res2, batch 128):", "",
          "| case | b | MB moved | BinaryOp ms | copy ms | vs copy | GB/s |", "|---|---|---|---|---|---|---|"]
    for r in alone:
        b = r["b_shape"] if r["b_shape"] == "scalar" else " x ".join(map(str, r["b_shape"]))
        md.append(f"| {r['case']} | {b} | {r['mb_moved']:.0f} | {r['binary_op_ms']:.4f} | {r['d2d_copy_ms']:.4f} | "
                  f"{r['vs_copy']:.2f} | {r['gb_per_s']:.0f} |")
    md += ["", "Whole nets, fusion and CUDA graphs on, device-resident input, layouts alternated in one run:", "",
           "| model | batch | Eltwise images/s | BinaryOp images/s | launches (Eltwise / BinaryOp) |", "|---|---|---|---|---|"]
    for r in whole:
        e, b = r["eltwise"], r["binaryop"]
        md.append(f"| {r['model']} | {r['batch']} | {e['images_per_s']:.1f} | {b['images_per_s']:.1f} | "
                  f"{e['launches_per_forward']} / {b['launches_per_forward']} |")
    (out / "binary_op_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
