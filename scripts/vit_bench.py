"""What a Vision Transformer costs: ViT-B/16, ViT-S/16 and ViT-Ti/16 through feather::Net, the attention kernel alone
at ViT-B's shapes, and LayerNorm / GELU alone against a device-to-device copy of the same bytes.

    python scripts/vit_bench.py --out DIR [--reps 7] [--iters 5]

Whole nets at 224 x 224: ViT-B/16 at batch 64, ViT-S/16 and ViT-Ti/16 at batch 256.  Fp32-split mode, fusion on,
device-resident input, CUDA graphs on; after a warm-up, --reps windows of --iters forwards each, the nets alternating
window by window, timed with CUDA events; the median window.  Then, in a run of its own, torch.profiler's CUDA kernel
times over two eager forwards, grouped by kernel name: TensorGEMM (the InnerProduct and projection GEMMs, and the patch
convolution's GEMM), fc_reduce, attention, LayerNorm, GELU (the activation kernel), BinaryOp (element-wise adds) and
the rest.  The patch convolution (16 x 16 taps, im2col) is also timed alone as a one-layer net, as a share of the
forward.

The attention kernel alone: ViT-B's 12 heads of 64 at L = 197 (batch 64) and L = 577 (384 x 384 input, batch 16), its
achieved rate (4 L^2 d per head, the FLOPs of S and P V) against the BF16x3 bound of 989 / 3 TFLOP/s (the data sheet's
dense BF16 rate over the three products of the split).

Writes DIR/vit_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA device."""
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

NETS = [("vit_b_16", 64), ("vit_s_16", 256), ("vit_ti_16", 256)]
GROUPS = [("TensorGEMM", "tensor_gemm"), ("fc_reduce", "fc_reduce"), ("attention", "attention_kernel"),
          ("LayerNorm", "layer_norm_kernel"), ("GELU", "activation_kernel"), ("BinaryOp", "add_relu"),
          ("BinaryOp", "binary"), ("patch conv im2col", "im2col")]
BF16X3_TFLOPS = 989.0 / 3


def group_of(name: str) -> str:
    for g, key in GROUPS:
        if key in name:
            return g
    return "other"


def profile_shares(net) -> list[dict]:
    import torch
    net._lib.fnet_set_cuda_graph(net._h, 0)
    net.Forward()
    net.Synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            net.Forward()
        net.Synchronize()
    net._lib.fnet_set_cuda_graph(net._h, 1)
    per: dict[str, float] = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if us > 0:
            g = group_of(e.key)
            per[g] = per.get(g, 0.0) + us / 2e3
    total = sum(per.values())
    return [{"group": g, "ms_per_forward": ms, "share": ms / total if total else 0.0}
            for g, ms in sorted(per.items(), key=lambda kv: -kv[1])]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5, help="forwards per timed window")
    args = ap.parse_args()
    import numpy as np
    import torch
    from igemm_layer_bench import card
    from mobilenet_v2_bench import alternated, load
    from mobilenet_v3_bench import time_calls
    from feathercnn_b200 import booster
    from feathercnn_b200.tools import modelgen
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    booster.set_precision(booster.PRECISION_FP32_SPLIT)
    stream = torch.cuda.current_stream().cuda_stream
    cases = []
    with tempfile.TemporaryDirectory() as d:
        for model, batch in NETS:
            mw = modelgen.ZOO[model]()
            shape = mw.shape["data"]
            base = np.stack([modelgen.synthetic_input(shape, i) for i in range(8)])
            x = torch.from_numpy(np.resize(base, (batch,) + tuple(shape))).cuda()
            param, binf = mw.save(Path(d) / model)
            dim = mw.shape["conv_proj"][0]
            pc = modelgen.single_conv(3, dim, 224, 224, 16, 16, 0)
            pparam, pbinf = pc.save(Path(d) / f"{model}_patch")
            cases.append({"model": model, "batch": batch, "x": x, "net": load(param, binf, True, x, stream),
                          "patch": load(pparam, pbinf, True, x, stream)})
    ms = alternated([c["net"] for c in cases] + [c["patch"] for c in cases], args.reps, args.iters)
    nets = []
    for i, c in enumerate(cases):
        t, tp = ms[i], ms[len(cases) + i]
        nets.append({"model": c["model"], "batch": c["batch"], "ms": t, "images_per_s": c["batch"] / (t * 1e-3),
                     "launches_per_forward": c["net"].launches_per_forward, "patch_conv_ms": tp,
                     "patch_conv_share": tp / t, "kernel_groups_eager": profile_shares(c["net"])})
        del c["net"], c["patch"], c["x"]
        torch.cuda.empty_cache()

    attn = []
    for n, l in ((64, 197), (16, 577)):
        qkv = torch.randn((n, l, 3 * 768), device="cuda")
        q, k, v = qkv[:, :, :768], qkv[:, :, 768:1536], qkv[:, :, 1536:]
        out = torch.empty((n, l, 768), device="cuda")
        t = time_calls([lambda: booster.attention(q, k, v, 12, out=out)], args.reps, 10 * args.iters)[0]
        flops = 4.0 * n * 12 * l * l * 64
        attn.append({"batch": n, "L": l, "heads": 12, "head_dim": 64, "ms": t, "tflops": flops / (t * 1e9),
                     "share_of_bf16x3_bound": flops / (t * 1e9) / BF16X3_TFLOPS})
        del qkv, out

    norm = []
    n_rows = 256 * 197
    x = torch.randn((n_rows, 768), device="cuda")
    y = torch.empty_like(x)
    g, b = torch.rand(768, device="cuda") + 0.5, torch.rand(768, device="cuda") - 0.5
    fns = [lambda: y.copy_(x), lambda: booster.layer_norm(x, 768, g, b, 1e-6, out=y),
           lambda: booster.activation(x, "GELU", out=y), lambda: booster.activation(x, "GELU_TANH", out=y)]
    t = time_calls(fns, args.reps, 10 * args.iters)
    for name, m in zip(("copy", "LayerNorm (rows of 768)", "GELU", "GELU tanh"), t):
        norm.append({"kernel": name, "ms": m, "vs_copy": m / t[0], "GB_per_s": 8.0 * x.numel() / (m * 1e6)})

    info = card()
    res = {"card": info, "precision": "fp32split", "fusion": True, "cuda_graph": True, "nets": nets,
           "attention_alone": attn, "memory_bound_alone": {"floats": x.numel(), "rows": norm}}
    out_dir = Path(args.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    (out_dir / "vit_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; fp32-split, fusion on, device-resident input, CUDA graph, "
          f"median of {args.reps} alternated windows", "",
          "| net | batch | ms / forward | images/s | launches / forward | patch conv alone |", "|---|---|---|---|---|---|"]
    md += [f"| {r['model']} | {r['batch']} | {r['ms']:.2f} | {r['images_per_s']:.0f} | {r['launches_per_forward']} | "
           f"{r['patch_conv_share']:.1%} |" for r in nets]
    for r in nets:
        md += ["", f"{r['model']} b{r['batch']}, kernel time by group (torch.profiler, eager):", "",
               "| group | ms / forward | share |", "|---|---|---|"]
        md += [f"| {k['group']} | {k['ms_per_forward']:.3f} | {k['share']:.1%} |" for k in r["kernel_groups_eager"]]
    md += ["", "Attention kernel alone (ViT-B: 12 heads of 64):", "",
           "| batch | L | ms | TFLOP/s | of the BF16x3 bound (329.7) |", "|---|---|---|---|---|"]
    md += [f"| {r['batch']} | {r['L']} | {r['ms']:.3f} | {r['tflops']:.1f} | {r['share_of_bf16x3_bound']:.1%} |"
           for r in attn]
    md += ["", f"LayerNorm and GELU alone on {x.numel()} floats ({4 * x.numel() / 1e6:.0f} MB):", "",
           "| kernel | ms | x copy | GB/s (read + write) |", "|---|---|---|---|"]
    md += [f"| {r['kernel']} | {r['ms']:.4f} | {r['vs_copy']:.3f} | {r['GB_per_s']:.0f} |" for r in norm]
    (out_dir / "vit_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
