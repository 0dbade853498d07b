"""Per-layer timing of Deconvolution / DeconvolutionDepthWise (fcuda_deconv_forward) on DCGAN, U-Net and FCN shapes.

    python scripts/deconv_layer_bench.py --out DIR [--reps 7] [--iters 20]

Per layer, CUDA-event times (median over --reps windows of --iters launches each, after a warm-up):
  - layer ms: the whole fcuda_deconv_forward;
  - contraction ms: the equivalent stride-1 convolution alone (fcuda_conv_forward_ext into the same scratch);
  - scatter / direct ms: the scatter or depthwise gather kernel, from the library's per-launch profiling events;
  - the algorithmic GFLOP of the deconvolution (2*N*IC*OC/group*H*W*KH*KW) and the GFLOP the equivalent convolution issues
    (its output channels include the empty sub-pixel phases when the stride does not divide the kernel);
  - algorithmic TFLOP/s over the layer time, and the scatter / gather kernel's algorithmic bytes (output written plus
    phase planes or input read) per second against the H100 SXM data sheet's 3.35 TB/s;
  - for context only: torch.nn.functional.conv_transpose2d in fp32 with TF32 disabled, same shapes.
Writes DIR/deconv_layer_bench.json and DIR/deconv_layer_bench.md with the card's name and power limit.  Needs a CUDA
device."""
from __future__ import annotations

import argparse
import ctypes
import json
import statistics
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

HBM_DATASHEET = 3.35e12  # H100 SXM data sheet (not a measured figure)
PROF_DECONV = 7

# (name, batch, oc, ic, hw, k, stride, pad, output_pad, group)
CASES = [
    ("dcgan 512->256 k4s2p1 8->16", 64, 256, 512, 8, 4, 2, 1, 0, 1),
    ("dcgan 256->128 k4s2p1 16->32", 64, 128, 256, 16, 4, 2, 1, 0, 1),
    ("dcgan 128->64 k4s2p1 32->64", 64, 64, 128, 32, 4, 2, 1, 0, 1),
    ("dcgan 64->3 k4s2p1 64->128", 64, 3, 64, 64, 4, 2, 1, 0, 1),
    ("unet 512->256 k2s2 28->56", 32, 256, 512, 28, 2, 2, 0, 0, 1),
    ("unet 256->128 k2s2 56->112", 32, 128, 256, 56, 2, 2, 0, 0, 1),
    ("128->64 k3s2p1 op1 56->112", 32, 64, 128, 56, 3, 2, 1, 1, 1),
    ("256->256 k3s1p1 28 (direct)", 64, 256, 256, 28, 3, 1, 1, 0, 1),
    ("fcn bilinear C21 k4s2p1 16->32", 64, 21, 21, 16, 4, 2, 1, 0, 21),
    ("fcn bilinear C21 k16s8p4 32->256", 64, 21, 21, 32, 16, 8, 4, 0, 21),
]


def timed(fn, reps: int, iters: int) -> float:
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return statistics.median(times)


def bench_case(case, reps: int, iters: int) -> dict:
    import torch
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    name, n, oc, ic, hw, k, s, pad, op, group = case
    p = booster.deconv_param(oc, ic, hw, hw, k, k, s, pad, op, 1, group, True, False)
    eq, algo = booster.deconv_plan(p)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand((n, ic, hw, hw), device="cuda", generator=g) * 2 - 1
    w = torch.randn((oc, ic // group, k, k), device="cuda", generator=g) * (2.0 * s * s / (ic // group * k * k)) ** 0.5
    b = torch.rand(oc, device="cuda", generator=g) - 0.5
    sc, pk = ctypes.c_size_t(), ctypes.c_size_t()
    booster._check("fcuda_deconv_get_buffer_size", lib.fcuda_deconv_get_buffer_size(ctypes.byref(p), n, ctypes.byref(sc), ctypes.byref(pk)))
    packed = torch.empty(max(pk.value, 1), device="cuda")
    scratch = torch.empty(max(sc.value, 1), device="cuda")
    out = torch.empty((n, oc, p.output_h, p.output_w), device="cuda")
    booster._check("fcuda_deconv_init", lib.fcuda_deconv_init(ctypes.byref(p), booster._ptr(packed), ctypes.c_void_p(w.data_ptr()), booster._stream()))
    args = (ctypes.byref(p), booster._ptr(out), booster._ptr(x), booster._ptr(packed), booster._ptr(scratch), booster._ptr(b), n,
            booster._stream())

    def layer():
        booster._check("fcuda_deconv_forward", lib.fcuda_deconv_forward(*args))

    layer_ms = timed(layer, reps, iters)
    depthwise = algo == booster.DEPTHWISE
    subpixel = not depthwise and eq.output_channels != oc
    contraction_ms = None
    if not depthwise:
        cs, ck = ctypes.c_size_t(), ctypes.c_size_t()
        lib.fcuda_conv_get_buffer_size(ctypes.byref(eq), algo, n, ctypes.byref(cs), ctypes.byref(ck))
        dst = scratch[-(-cs.value // 64) * 64:] if subpixel else out
        dil = 1

        def contraction():
            booster._check("fcuda_conv_forward_ext",
                           lib.fcuda_conv_forward_ext(ctypes.byref(eq), algo, booster._ptr(dst), booster._ptr(x),
                                                      booster._ptr(packed), booster._ptr(scratch),
                                                      None if subpixel else booster._ptr(b), None, 0, dil, dil, n,
                                                      booster._stream()))
        contraction_ms = timed(contraction, reps, iters)
    kernel_ms = kernel_bytes = None
    if subpixel or depthwise:
        lib.fcuda_profile_tensor_gemm(1)
        for _ in range(iters):
            layer()
        ms, af, mf, ab, cnt = (ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong())
        lib.fcuda_profile_collect_kind(PROF_DECONV, ctypes.byref(ms), ctypes.byref(af), ctypes.byref(mf), ctypes.byref(ab),
                                       ctypes.byref(cnt))
        lib.fcuda_profile_tensor_gemm(0)
        kernel_ms, kernel_bytes = ms.value / cnt.value, ab.value / cnt.value
    algo_flops = 2.0 * n * ic * (oc // group) * hw * hw * k * k
    issued = algo_flops if depthwise else 2.0 * n * eq.output_channels * (ic // group) * eq.output_h * eq.output_w * eq.kernel_h * eq.kernel_w
    # torch, for context: fp32 without TF32; its weight layout is (IC, OC/group, kh, kw), crop = pad, output_padding = op
    wt = w.view(group, oc // group, ic // group, k, k).transpose(1, 2).reshape(ic, oc // group, k, k).contiguous()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch_ms = timed(lambda: torch.nn.functional.conv_transpose2d(x, wt, b, s, pad, op, group), reps, iters)
    ref = torch.nn.functional.conv_transpose2d(x, wt, b, s, pad, op, group)
    layer()
    torch.cuda.synchronize()
    rel = float((out - ref).abs().max() / ref.abs().max())
    return {
        "case": name, "batch": n, "conv_algo": booster.ALGO_NAMES[algo], "equivalent_oc": eq.output_channels,
        "algo_gflop": algo_flops / 1e9, "issued_gflop": issued / 1e9,
        "contraction_ms": contraction_ms, "scatter_or_direct_ms": kernel_ms, "layer_ms": layer_ms,
        "algo_tflops": algo_flops / layer_ms / 1e9,
        "kernel_gbps": None if kernel_ms is None else kernel_bytes / kernel_ms / 1e6,
        "kernel_share_of_hbm": None if kernel_ms is None else kernel_bytes / kernel_ms * 1e3 / HBM_DATASHEET,
        "torch_fp32_ms": torch_ms, "max_rel_diff_vs_torch": rel,
    }


def _fmt(v, f):
    return "-" if v is None else format(v, f)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20, help="launches per timed window")
    args = ap.parse_args()
    import torch
    from igemm_layer_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    rows = [bench_case(c, args.reps, args.iters) for c in CASES]
    info = card()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "deconv_layer_bench.json").write_text(json.dumps({"card": info, "rows": rows}, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}", "",
          "| case | N | conv algo | algo GFLOP | issued GFLOP | contraction ms | scatter/direct ms | layer ms | algo TFLOP/s |"
          " scatter/direct GB/s (share of 3.35 TB/s) | torch fp32 ms |",
          "|---|---|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        share = "-" if r["kernel_gbps"] is None else f"{r['kernel_gbps']:.0f} ({r['kernel_share_of_hbm']:.0%})"
        md.append(f"| {r['case']} | {r['batch']} | {r['conv_algo']} | {r['algo_gflop']:.2f} | {r['issued_gflop']:.2f} | "
                  f"{_fmt(r['contraction_ms'], '.3f')} | {_fmt(r['scatter_or_direct_ms'], '.3f')} | {r['layer_ms']:.3f} | "
                  f"{r['algo_tflops']:.1f} | {share} | {r['torch_fp32_ms']:.3f} |")
    (out / "deconv_layer_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
