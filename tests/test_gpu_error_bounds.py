"""Per-element error bounds of every convolution and GEMM path against a float64 reference.

The other parity tests hold a whole blob to max|got - ref| / max|ref| < 2e-4.  That is too coarse to tell the arithmetic
modes apart (plain TF32 is ~2.5e-4 per layer) and it forgives errors confined to small outputs.  Here every output
element is checked on its own:

    |got_i - ref_i| <= (eps_mode + K * 2^-23) * S_i + 2^-23 * |ref_i|,      S_i = |b_i| + sum_k |x_k w_k| (+ |residual_i|)

ref is torch's float64 convolution / matmul (CPU, or cuDNN's float64 path on the GPU: no TF32 there), S the same
operation applied to |x| and |w|: the condition scale of the dot product, independent of cancellation and of the blob's
largest output.  K is the number of products per output.  Every partial sum is bounded by S, and each of the K
accumulations may lose up to 2^-23 of it (a full ulp: the tensor-core adder need not round to nearest), hence K * 2^-23.

eps_mode bounds the relative error of one product under the operand split (include/fcuda.h, DESIGN.md §2):
  - 3xTF32 (the TensorGEMM in FP32_SPLIT and TF32X3 modes, the implicit GEMM in TF32X3): x = hi + lo, hi = RN_tf32(x),
    lo = x - hi with |lo| <= 2^-11 |x|; the MMA reads lo with 10 mantissa bits, so lo loses <= 2^-10 |lo| <= 2^-21 |x|.
    hi*hi + hi*lo + lo*hi then misses <= 2^-21 (a's lo) + 2^-21 (b's lo) + 2^-22 (the dropped lo*lo) of |ab|
    < 3 * 2^-20.
  - BF16x3 (the implicit GEMM in FP32_SPLIT mode): x = p1 + p2 + r, p1 = RN_bf16(x), p2 = RN_bf16(x - p1), |p2| <= 2^-8 |x|,
    |r| <= 2^-16 |x|.  p1*q1 + p1*q2 + p2*q1 misses p2*q2 (<= 2^-16), p1*rq, rp*q1 and the smaller terms:
    < 3 * 2^-16 of |ab|.
  - TF32: both operands cut to 10 mantissa bits (truncation in the worst case, 2^-10 each): 2^-9.
  - fp32 FMA paths (NAIVE, depthwise, the SIMT InnerProduct): 0; only the accumulation term remains.
These are worst-case bounds: they do not fail on a correct kernel whatever the data.

Winograd F(6,3) / F(2,3) transform the operands before the contraction, and the transforms amplify rounding, so the
convolution-domain bound above does not apply.  Their ceiling comes from `wino_model`, a float64 model of the same
pipeline with the kernel's own transform matrices (winograd.cu): input / filter / output transforms in fp32, the
contraction with operands rounded as the mode rounds them and an fp32 accumulator rounded every 8 channels (one MMA
k-step).  On the same inputs the model's worst |d|/S is rho; the kernel is held to WINO_MARGIN * rho * S_i (+ 2^-23 |ref_i|).
The margin (8) covers what the model leaves out: the kernel's operation order inside the transforms and the
accumulator's truncating adds, each of which can at most double the modelled error; the worst element of a large
output is a maximum over many roughly independent errors, so its run-to-run spread is well under 2x.

The mode probes show the check resolves the modes: on small-K layers (accumulation error negligible) plain TF32
exceeds the 3xTF32 bound while 3xTF32 and BF16x3 meet theirs.  The CPU tests at the end feed the checker simulated
defects (TF32 operands where 3xTF32 was due, a dropped BF16x3 term, a dropped tap or k-block, a shifted bias, swapped
images) computed in float64 on the sweep's shapes, and require it to reject each.

Run with -s to print the worst |d|/S and the share of the bound used per (path, mode).
"""
from __future__ import annotations

import dataclasses
import functools
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu

U = 2.0 ** -23
EPS_3XTF32 = 3 * 2.0 ** -20
EPS_BF16X3 = 3 * 2.0 ** -16
EPS_TF32 = 2.0 ** -9
WINO_MARGIN = 8.0

# include/fcuda.h FcudaPrecision / FcudaConvAlgo (kept literal so the CPU tests need no native library)
TF32X3, TF32, FP32_SPLIT = 0, 1, 2
MODES = {"fp32split": FP32_SPLIT, "tf32x3": TF32X3, "tf32": TF32}
MODE_NAME = {v: k for k, v in MODES.items()}
NAIVE, IM2COL, SGECONV, DEPTHWISE, WINOGRADF63, WINOGRADF63FUSED, WINOGRADF23 = range(7)
PATH = {NAIVE: "naive", IM2COL: "im2col", SGECONV: "sgeconv", DEPTHWISE: "depthwise", WINOGRADF63: "f63",
        WINOGRADF23: "f23"}


def eps_for(path: str, mode: int) -> float:
    if path in ("naive", "depthwise", "simt"):
        return 0.0
    if mode == TF32:
        return EPS_TF32
    if path == "sgeconv" and mode == FP32_SPLIT:
        return EPS_BF16X3
    return EPS_3XTF32


# ---- report ---------------------------------------------------------------------------------------
REPORT: dict[tuple[str, str], list[float]] = {}


def _record(path: str, mode: int, worst_rel: float, used: float) -> None:
    r = REPORT.setdefault((path, MODE_NAME[mode]), [0.0, 0.0])
    r[0] = max(r[0], worst_rel)
    r[1] = max(r[1], used)


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\nworst |d|/S and the largest share of the per-element bound used, per (path, mode):")
        for (path, mode), (rel, used) in sorted(REPORT.items()):
            print(f"  {path:10s} {mode:10s} |d|/S {rel:.3e}   bound used {used:.3f}")


# ---- the checker ----------------------------------------------------------------------------------
def excess(got, ref, scale, coef, ref_coef=U) -> tuple[float, float]:
    """(max_i |got_i - ref_i| / bound_i, max_i |got_i - ref_i| / S_i) with bound_i = coef * S_i + ref_coef * |ref_i|.
    `coef` is a number or a tensor broadcast against S.  The first value is <= 1 when every element is inside its bound."""
    got = torch.as_tensor(got).to(torch.float64)
    ref = torch.as_tensor(ref).to(device=got.device, dtype=torch.float64)
    scale = torch.as_tensor(scale).to(device=got.device, dtype=torch.float64)
    assert got.shape == ref.shape == scale.shape, (got.shape, ref.shape, scale.shape)
    d = (got - ref).abs()
    bound = coef * scale + ref_coef * ref.abs()
    # a zero bound (all-zero receptive field, no bias) admits only an exact zero
    ratio = torch.where(d == 0, torch.zeros_like(d), d / bound.clamp_min(1e-300))
    rel = torch.where(d == 0, torch.zeros_like(d), d / scale.clamp_min(1e-300))
    return float(ratio.max()), float(rel.max())


# ---- rounding of operands (float32 tensors) -------------------------------------------------------
def tf32(x: torch.Tensor, trunc: bool = False) -> torch.Tensor:
    u = x.to(torch.float32).contiguous().view(torch.int32)
    if not trunc:
        u = u + 0x1000  # round half away from zero on the magnitude
    return (u & -0x2000).view(torch.float32)


def bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).to(torch.bfloat16).to(torch.float32)


# ---- problem description ---------------------------------------------------------------------------
@dataclasses.dataclass
class Conv:
    name: str
    oc: int
    ic: int
    h: int
    w: int
    kh: int = 3
    kw: int | None = None
    sh: int = 1
    sw: int | None = None
    pad: tuple[int, int, int, int] | int = 1   # int, or (left, bottom, right, top) like ConvParam.make(pad_lbrt=)
    group: int = 1
    dil: int = 1
    bias: bool = True
    relu: bool = False
    res: bool = False
    relu_after_add: bool = False
    pool: bool = False
    batch: int = 2
    algo: int | None = None      # None: the tuned policy (what feather::Net uses)
    chunk: int | None = None     # L2 chunk bytes for the Winograd / im2col intermediates
    clip: tuple[float, float] | None = None   # (lo, hi): the Clip epilogue of fcuda_conv_forward_clip, after any ReLU

    def __post_init__(self):
        self.kw = self.kh if self.kw is None else self.kw
        self.sw = self.sh if self.sw is None else self.sw
        if isinstance(self.pad, int):
            self.pad = (self.pad,) * 4

    @property
    def out_hw(self):
        pl, pb, pr, pt = self.pad
        oh = (self.h + pt + pb - self.dil * (self.kh - 1) - 1) // self.sh + 1
        ow = (self.w + pl + pr - self.dil * (self.kw - 1) - 1) // self.sw + 1
        return oh, ow

    @property
    def depthwise(self):
        return self.group > 1 and self.group == self.ic and self.oc == self.ic

    @property
    def K(self):
        return self.ic // self.group * self.kh * self.kw

    def seed(self):
        return zlib.crc32(self.name.encode())


def make_data(c: Conv, device="cpu", images=None):
    """Distinct images; per-output-channel weight scales spread over two decades so small-weight channels are checked
    on their own scale."""
    g = torch.Generator(device=device).manual_seed(c.seed())
    n = c.batch
    x = torch.rand((n, c.ic, c.h, c.w), generator=g, device=device) * 2 - 1
    icg = c.ic // c.group
    w = torch.randn((c.oc, icg, c.kh, c.kw), generator=g, device=device) * math.sqrt(2.0 / (icg * c.kh * c.kw))
    w = w * torch.pow(10.0, -2 * torch.rand((c.oc, 1, 1, 1), generator=g, device=device))
    b = (torch.rand(c.oc, generator=g, device=device) - 0.5) if c.bias else None
    oh, ow = c.out_hw
    r = (torch.rand((n, c.oc, oh, ow), generator=g, device=device) * 2 - 1) if c.res else None
    return x, w, b, r


def conv_ref(c: Conv, x, w, b, r, absolute=False):
    """float64 conv (absolute=True: the same op on |x|, |w|, |b|, |r|, i.e. S) before the pooling."""
    pl, pb, pr, pt = c.pad
    x, w = x.to(torch.float64), w.to(torch.float64)
    b = b.to(torch.float64) if b is not None else None
    if absolute:
        x, w = x.abs(), w.abs()
        b = b.abs() if b is not None else None
    y = F.conv2d(F.pad(x, (pl, pr, pt, pb)), w, b, stride=(c.sh, c.sw), dilation=c.dil, groups=c.group)
    if not absolute and c.relu:
        y = y.clamp_min(0)
    if not absolute and c.clip is not None:
        y = y.clamp(*c.clip)
    if r is not None:
        y = y + (r.to(torch.float64).abs() if absolute else r.to(torch.float64))
        if not absolute and c.relu_after_add:
            y = y.clamp_min(0)
    return y


def pool2(t):
    return F.max_pool2d(t, 2, 2, ceil_mode=True)


# ---- Winograd model -------------------------------------------------------------------------------
_BT63 = [[1, 0, -5.25, 0, 5.25, 0, -1, 0], [0, 1, 1, -4.25, -4.25, 1, 1, 0], [0, -1, 1, 4.25, -4.25, -1, 1, 0],
         [0, .5, .25, -2.5, -1.25, 2, 1, 0], [0, -.5, .25, 2.5, -1.25, -2, 1, 0], [0, 2, 4, -2.5, -5, .5, 1, 0],
         [0, -2, 4, 2.5, -5, -.5, 1, 0], [0, -1, 0, 5.25, 0, -5.25, 0, 1]]
_G63 = [[1, 0, 0], [-2 / 9, -2 / 9, -2 / 9], [-2 / 9, 2 / 9, -2 / 9], [1 / 90, 1 / 45, 2 / 45], [1 / 90, -1 / 45, 2 / 45],
        [1 / 45, 1 / 90, 1 / 180], [1 / 45, -1 / 90, 1 / 180], [0, 0, 1]]
_AT63 = [[1, 1, 1, 1, 1, 32, 32, 0], [0, 1, -1, 2, -2, 16, -16, 0], [0, 1, 1, 4, 4, 8, 8, 0], [0, 1, -1, 8, -8, 4, -4, 0],
         [0, 1, 1, 16, 16, 2, 2, 0], [0, 1, -1, 32, -32, 1, -1, 1]]
_BT23 = [[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]]
_G23 = [[1, 0, 0], [.5, .5, .5], [.5, -.5, .5], [0, 0, 1]]
_AT23 = [[1, 1, 1, 0], [0, 1, -1, -1]]


def wino_model(c: Conv, x, w, b, tile: int, mode: int | None):
    """F(tile-2, 3) as the kernels compute it, before ReLU / residual / pooling.  mode None: every step in float64
    (must reproduce the convolution)."""
    dev = x.device
    dt = torch.float64 if mode is None else torch.float32
    BT, G, AT = (torch.tensor(m, dtype=torch.float64, device=dev).to(dt) for m in
                 ((_BT63, _G63, _AT63) if tile == 8 else (_BT23, _G23, _AT23)))
    m = tile - 2
    pl, pb, pr, pt = c.pad
    oh, ow = c.out_hw
    ty, tx = -(-oh // m), -(-ow // m)
    xp = F.pad(x.to(dt), (pl, tx * m + 2 - c.w - pl, pt, ty * m + 2 - c.h - pt))
    tiles = xp.unfold(2, tile, m).unfold(3, tile, m)                       # (N, C, ty, tx, t, t)
    V = torch.einsum("ai,ncyxij,bj->ncyxab", BT, tiles, BT)
    Uw = torch.einsum("ai,ocij,bj->ocab", G, w.to(dt), G)
    if mode is None:
        M = torch.einsum("ncyxab,ocab->noyxab", V, Uw)
    else:
        if mode == TF32:
            pairs = [(tf32(V), tf32(Uw))]
        else:
            vh, uh = tf32(V), tf32(Uw)
            vl, ul = tf32(V - vh, trunc=True), tf32(Uw - uh, trunc=True)
            pairs = [(vh, uh), (vh, ul), (vl, uh)]
        M = None
        for c0 in range(0, c.ic, 8):  # one MMA k-step per 8 channels, fp32 accumulator
            part = sum(torch.einsum("ncyxab,ocab->noyxab", a[:, c0:c0 + 8].double(), u[:, c0:c0 + 8].double())
                       for a, u in pairs)
            M = part.float() if M is None else (M.double() + part).float()
    Y = torch.einsum("ia,noyxab,jb->noyixj", AT, M.to(dt), AT)
    Y = Y.reshape(Y.shape[0], Y.shape[1], ty * m, tx * m)[:, :, :oh, :ow]
    if b is not None:
        Y = Y + b.to(dt).view(1, -1, 1, 1)
    return Y.to(torch.float64)


def wino_finish(c: Conv, y, r):
    if c.relu:
        y = y.clamp_min(0)
    if c.clip is not None:
        y = y.clamp(*c.clip)
    if r is not None:
        y = y + r.to(torch.float64)
        if c.relu_after_add:
            y = y.clamp_min(0)
    return y


# ---- running a convolution through the C ABI ------------------------------------------------------
def _ref_chunk(c: Conv, per_image_floats: int) -> int:
    return max(1, min(c.batch, int(4e8 // (8 * 4 * max(per_image_floats, 1)))))


def run_conv(c: Conv, mode: int, expect_algo: int | None = None, tuned: bool = False):
    """Runs `c` on the GPU in `mode`; returns (share of the per-element bound used, worst |d|/S, algo)."""
    from feathercnn_b200 import booster
    booster.set_precision(mode)
    x, w, b, r = make_data(c, "cuda")
    pl, pb, pr, pt = c.pad
    p = booster.ConvParam.make(c.oc, c.ic, c.h, c.w, c.kh, c.kw, stride=c.sh, stride_w=c.sw, pad_lbrt=c.pad,
                               group=c.group, bias=c.bias, relu=c.relu)
    if c.clip is not None:
        p.activation = booster.ACT_CLIP
    oh, ow = c.out_hw
    p.output_h, p.output_w = oh, ow  # (what AssignOutputDim gives without dilation)
    default_chunk = booster.fcuda().fcuda_get_l2_chunk_bytes() if c.chunk else None
    if c.chunk:
        booster.set_l2_chunk_bytes(c.chunk)
    try:
        got, algo = booster.conv_forward(p, x, w, b, algo=c.algo, residual=r, relu_after_add=c.relu_after_add,
                                         dilation=c.dil, tuned=tuned, pool=c.pool, clip=c.clip)
        torch.cuda.synchronize()
    finally:
        if c.chunk:
            booster.set_l2_chunk_bytes(default_chunk)
    if expect_algo is not None:
        assert algo == expect_algo, (c.name, booster.ALGO_NAMES[algo])
    path = PATH[algo]
    wino = algo in (WINOGRADF63, WINOGRADF23)
    rho = None
    if wino:  # the model's worst |d|/S on the first images (a statistic of many outputs: stable across images)
        n0 = min(c.batch, 2)
        ym = wino_model(c, x[:n0], w, b, 8 if algo == WINOGRADF63 else 4, mode)
        want = conv_ref(c, x[:n0], w, b, None)
        s = conv_ref(c, x[:n0], w, b, None, absolute=True)
        _, rho = excess(wino_finish(dataclasses.replace(c, res=False), ym, None), want, s, 1.0)
    coef = WINO_MARGIN * rho if wino else eps_for(path, mode) + c.K * U
    worst_used = worst_rel = 0.0
    step = _ref_chunk(c, c.ic * c.h * c.w + 3 * c.oc * oh * ow)
    for i0 in range(0, c.batch, step):
        sl = slice(i0, i0 + step)
        ref = conv_ref(c, x[sl], w, b, r[sl] if r is not None else None)
        s = conv_ref(c, x[sl], w, b, r[sl] if r is not None else None, absolute=True)
        # a clamp is 1-Lipschitz: the bound of the unclamped result holds for the clamped one
        free = ref if c.clip is None else conv_ref(dataclasses.replace(c, clip=None), x[sl], w, b, r[sl] if r is not None else None)
        bound = coef * s + U * free.abs()
        if c.pool:
            ref, s, bound = pool2(ref), pool2(s), pool2(bound)
        used, _ = excess(got[sl], ref, bound, 1.0, 0.0)
        _, rel = excess(got[sl], ref, s, 1.0, 0.0)
        worst_used, worst_rel = max(worst_used, used), max(worst_rel, rel)
        del ref, s, bound, free
    _record(path, mode, worst_rel, worst_used)
    return worst_used, worst_rel, algo


MODE_PARAMS = pytest.mark.parametrize("mode", list(MODES.values()), ids=list(MODES))


# ---- 1. mode probes ---------------------------------------------------------------------------------
PROBES = [
    Conv("probe_1x1_ic32", 48, 32, 12, 12, 1, pad=0, batch=2),
    Conv("probe_1x1_ic64", 40, 64, 9, 14, 1, pad=0, batch=2),
    Conv("probe_3x3_ic4", 36, 4, 16, 15, batch=2),
    Conv("probe_3x3_ic5", 33, 5, 13, 16, batch=2),
    Conv("probe_3x3_ic7", 64, 7, 12, 12, batch=2),
]


@gpu
@pytest.mark.parametrize("algo", [SGECONV, IM2COL], ids=["sgeconv", "im2col"])
@pytest.mark.parametrize("c", PROBES, ids=[p.name for p in PROBES])
def test_mode_probe_resolves_modes(cuda, c, algo):
    """On small-K layers plain TF32 must exceed the 3xTF32 bound while 3xTF32 (and BF16x3) meet theirs: the check can
    see a path that lost its lo plane."""
    c = dataclasses.replace(c, algo=algo)
    coef3 = EPS_3XTF32 + c.K * U
    used3, _, _ = run_conv(c, TF32X3, expect_algo=algo)
    assert used3 <= 1.0
    used_split, _, _ = run_conv(c, FP32_SPLIT, expect_algo=algo)
    assert used_split <= 1.0
    used1, rel1, _ = run_conv(c, TF32, expect_algo=algo)
    assert used1 <= 1.0                 # within its own (TF32) bound ...
    assert rel1 > coef3 + U, (rel1, coef3)  # ... and visibly outside the 3xTF32 one


# ---- 2. edge-geometry sweep -------------------------------------------------------------------------
SGECONV_SWEEP = (
    # output channels around the N tiles (BN 32 / 64 / 128) and the padded rows of the pre-tiled BF16x3 planes
    [Conv(f"sg_oc{oc}", oc, 32, 7, 9) for oc in (31, 32, 33, 64, 65, 128, 129, 257)]
    # pixels per image 127 / 128 / 129, batch 3: 128-pixel tiles straddle images
    + [Conv("sg_pix127", 40, 32, 1, 127, 1, pad=0, batch=3), Conv("sg_pix128", 40, 32, 8, 16, 1, pad=0, batch=3),
       Conv("sg_pix129", 40, 32, 3, 43, 1, pad=0, batch=3)]
    # k-block counts 1, 3, 4, 5, 8, 9 around the 4-deep ring: IC % 32 == 0 (arithmetic offsets) ...
    + [Conv(f"sg_kb{ic // 32}_fast", 48, ic, 6, 7, 1, pad=0) for ic in (32, 96, 128, 160, 256, 288)]
    # ... and the k-table (IC % 32 != 0): ceil(9 * IC / 32) = 3, 4, 5, 8, 9
    + [Conv(f"sg_kb_table_ic{ic}", 40, ic, 7, 6) for ic in (10, 14, 17, 28, 31)]
    + [Conv("sg_fast_3x3_3blocks", 72, 96, 9, 10),                          # 3 channel blocks x 9 taps
       Conv("sg_table_max", 40, 682, 6, 6),                                # K = 6138 <= kMaxTableK = 6144
       Conv("sg_taps63", 24, 3, 20, 23, 7, 9, pad=(4, 3, 4, 3)),            # 63 taps (7 x 9)
       Conv("sg_1x7", 40, 32, 9, 17, 1, 7, pad=(3, 0, 3, 0)),
       Conv("sg_7x1", 40, 20, 17, 9, 7, 1, pad=(0, 3, 0, 3)),
       Conv("sg_3x1_s2", 36, 24, 15, 11, 3, 1, sh=2, pad=(0, 1, 0, 1)),
       Conv("sg_stride_1x2", 40, 32, 13, 17, sh=1, sw=2),
       Conv("sg_stride_2x1", 40, 12, 13, 17, sh=2, sw=1),
       Conv("sg_pad_top2_left0", 40, 32, 11, 12, pad=(0, 1, 2, 2)),
       Conv("sg_pad_asym_br", 36, 20, 10, 13, pad=(1, 0, 2, 1)),            # bottom 0, right 2
       # a 1x1 / stride 1 layer padded only at the bottom and right is not the pointwise H * W-row layout (OH > H)
       Conv("psweep854", 62, 514, 40, 40, kh=1, kw=1, pad=(0, 2, 2, 0), group=2),
       Conv("sg_1x1_pad_br_table", 31, 33, 9, 10, 1, pad=(0, 1, 2, 0), batch=3),
       # a halo patch whose TF32 box and filter ring fill the 227 KB but for the kernel's static mbarriers
       Conv("psweep981", 96, 32, 7, 32, kh=7, kw=1, pad=(2, 0, 2, 0), bias=False, batch=1, clip=(-0.125, 0.25)),
       Conv("sg_dil2", 40, 32, 14, 13, dil=2, pad=2),
       Conv("sg_dil3_table", 24, 12, 15, 16, dil=3, pad=(3, 1, 2, 3)),
       Conv("sg_group4_table", 96, 64, 9, 10, group=4),                    # 16 channels per group: channel slices
       Conv("sg_group2_fast", 64, 128, 8, 9, group=2, relu=True),
       Conv("sg_res", 65, 32, 9, 11, res=True),
       Conv("sg_res_relu", 65, 32, 9, 11, res=True, relu_after_add=True),
       Conv("sg_res_1x1_relu", 129, 64, 7, 7, 1, pad=0, bias=False, res=True, relu_after_add=True),
       Conv("sg_pool_odd", 48, 32, 13, 68, pad=(1, 1, 0, 1), pool=True, relu=True),   # OW = 67, OH = 13
       Conv("sg_pool_wide", 40, 64, 9, 132, pad=2, pool=True),                        # OW = 134: three 64-column patches
       ])


@gpu
@MODE_PARAMS
@pytest.mark.parametrize("c", SGECONV_SWEEP, ids=[c.name for c in SGECONV_SWEEP])
def test_sgeconv_sweep(cuda, c, mode):
    used, _, _ = run_conv(dataclasses.replace(c, algo=SGECONV), mode, expect_algo=SGECONV)
    assert used <= 1.0


# non-square kernels, unequal strides and asymmetric pads (group 1, dense): IM2COL and NAIVE take any of them
GENERIC_SWEEP = [
    Conv("g_1x7", 40, 32, 9, 17, 1, 7, pad=(3, 0, 3, 0)),
    Conv("g_7x1_oc_tail", 33, 20, 17, 9, 7, 1, pad=(0, 3, 0, 3)),
    Conv("g_3x1_s2", 36, 24, 15, 11, 3, 1, sh=2, pad=(0, 1, 0, 1)),
    Conv("g_stride_1x2", 40, 32, 13, 17, sh=1, sw=2, relu=True),
    Conv("g_stride_2x1", 40, 12, 13, 17, sh=2, sw=1),
    Conv("g_pad_top2_left0", 40, 32, 11, 12, pad=(0, 1, 2, 2)),
    Conv("g_pad_asym_br", 36, 20, 10, 13, pad=(1, 0, 2, 1)),
    Conv("g_7x9_ic3", 24, 3, 20, 23, 7, 9, pad=(4, 3, 4, 3)),
    Conv("g_res_relu", 65, 32, 9, 11, res=True, relu_after_add=True),
]
# the L2 chunk (pixels of 128-pixel multiples) ends inside an image: NCHW epilogue with m_offset
IM2COL_CHUNKED = Conv("im2col_chunk_in_image", 72, 16, 20, 21, batch=3, chunk=128 * 144 * 4)


@gpu
@MODE_PARAMS
@pytest.mark.parametrize("c", GENERIC_SWEEP + [IM2COL_CHUNKED], ids=[c.name for c in GENERIC_SWEEP + [IM2COL_CHUNKED]])
def test_im2col_sweep(cuda, c, mode):
    used, _, _ = run_conv(dataclasses.replace(c, algo=IM2COL), mode, expect_algo=IM2COL)
    assert used <= 1.0


@gpu
@pytest.mark.parametrize("c", GENERIC_SWEEP, ids=[c.name for c in GENERIC_SWEEP])
def test_naive_sweep(cuda, c):
    used, _, _ = run_conv(dataclasses.replace(c, algo=NAIVE), FP32_SPLIT, expect_algo=NAIVE)
    assert used <= 1.0


WINO_SWEEP = [
    Conv("w_oc160", 160, 32, 14, 14),                              # several N tiles
    Conv("w_tails", 36, 20, 13, 17, relu=True),                    # IC and OC not multiples of 32
    Conv("w_odd", 40, 24, 15, 13),                                 # odd output: partial tiles
    Conv("w_pad0", 32, 16, 17, 15, pad=0),
    Conv("w_pool", 40, 16, 15, 13, pool=True, relu=True),
    Conv("w_chunked", 32, 32, 60, 120, batch=2, chunk=1),          # one chunk holds a few tile rows of an image
    Conv("w_res_relu", 48, 32, 12, 14, res=True, relu_after_add=True),
    Conv("w_oc40_ic48", 40, 48, 26, 22, batch=3, relu=True),       # OC 40: a partial BN 64 tile; IC 48: K % 32 = 16
]


@gpu
@MODE_PARAMS
@pytest.mark.parametrize("algo", [WINOGRADF63, WINOGRADF23], ids=["f63", "f23"])
@pytest.mark.parametrize("c", WINO_SWEEP, ids=[c.name for c in WINO_SWEEP])
def test_winograd_sweep(cuda, c, algo, mode):
    used, _, _ = run_conv(dataclasses.replace(c, algo=algo), mode, expect_algo=algo)
    assert used <= 1.0


# depthwise.cu depthwise_forward picks the kernel from the geometry; each case names the branch its geometry takes
# (k3 = 3x3, pad_top == pad_left == 1, stride_h == stride_w in {1, 2}, OW >= 24).
DW_CASES = [
    Conv("dw_vec4", 8, 8, 10, 128, group=8),                       # k3, s1, OW == W, W % 4 == 0, OW >= 96
    Conv("dw_vec2_s1", 8, 8, 9, 50, group=8, relu=True),           # k3, s1, OW == W, W % 4 != 0, OW >= 48
    Conv("dw_vec2_s2", 8, 8, 19, 96, sh=2, group=8),               # k3, s2, W == 2 OW, W % 4 == 0, OW = 48
    Conv("dw_shuffle_s1", 6, 6, 21, 45, group=6),                  # k3, s1, OW = 45 < 48
    Conv("dw_shuffle_s2", 6, 6, 21, 62, sh=2, group=6),            # k3, s2, OW = 31 < 48
    Conv("dw_shuffle_s1_pad_br0", 6, 6, 17, 64, pad=(1, 0, 0, 1), group=6),   # OW = 63 != W: shuffle, right pad 0
    Conv("dw_cols8", 12, 12, 12, 7, group=12),                     # not k3 (OW < 24), s1, H, W <= 16, W <= 8
    Conv("dw_cols16", 12, 12, 16, 13, group=12, relu=True),        # same with 8 < W <= 16
    Conv("dw_plane_s1", 10, 10, 20, 22, group=10),                 # H, W <= 34, not <= 16
    Conv("dw_plane_s1_pad0", 10, 10, 20, 22, pad=0, group=10),
    Conv("dw_plane_s2", 10, 10, 28, 27, sh=2, group=10),           # OW = 14
    Conv("dw_generic_5x5", 8, 8, 19, 21, 5, pad=2, group=8),
    Conv("dw_generic_3x1", 8, 8, 19, 21, 3, 1, pad=(0, 1, 0, 1), group=8),
    Conv("dw_generic_pad_top2", 8, 8, 19, 40, pad=(1, 1, 1, 2), group=8),
    Conv("dw_generic_big", 8, 8, 40, 20, sh=2, group=8),           # H > 34, OW = 10 < 24
    # stride_h != stride_w: the geometric definition (the reference swaps the two strides in its index,
    # depthwise.cu:9-10, which only agrees when they are equal)
    Conv("dw_generic_stride_1x2", 8, 8, 19, 40, sh=1, sw=2, group=8),
    Conv("dw_generic_stride_2x1", 8, 8, 19, 40, sh=2, sw=1, group=8),
]


@gpu
@pytest.mark.parametrize("c", DW_CASES, ids=[c.name for c in DW_CASES])
def test_depthwise_branches(cuda, c):
    used, _, _ = run_conv(dataclasses.replace(c, algo=DEPTHWISE, bias=True), FP32_SPLIT, expect_algo=DEPTHWISE)
    assert used <= 1.0


# ---- TensorGEMM and InnerProduct through the C ABI ------------------------------------------------
GEMM_CASES = (
    [(2, 129, n, 44) for n in (32, 33, 64, 65, 128, 129, 300)]     # N tiles; K % 32 = 12
    + [(3, m, 65, 60) for m in (127, 128, 129)]                    # M tiles; K % 32 = 28
    + [(64, 127, 33, 36), (64, 64, 64, 100), (1, 128, 300, 228)]   # G up to 64; K % 32 = 4
    + [(64, 1024, 256, 128),                                       # 1024 tiles: several per persistent CTA
       (7, 127, 65, 1000)]                                         # 32 k-blocks (K % 32 = 8) per tile, odd G
)


@gpu
@pytest.mark.parametrize("x3", [True, False], ids=["3xtf32", "tf32"])
@pytest.mark.parametrize("g,m,n,k", GEMM_CASES)
def test_tensor_gemm_bounds(cuda, g, m, n, k, x3):
    from feathercnn_b200 import booster
    gen = torch.Generator(device="cuda").manual_seed(g * 1000003 + m * 1009 + n * 31 + k)
    a = torch.rand((g, m, k), generator=gen, device="cuda") * 2 - 1
    b = torch.randn((g, n, k), generator=gen, device="cuda") * torch.pow(10.0, -2 * torch.rand((g, n, 1), generator=gen, device="cuda"))
    got = booster.tensor_gemm(a, b, x3=x3)
    torch.cuda.synchronize()
    ref = torch.einsum("gmk,gnk->gmn", a.double(), b.double())
    s = torch.einsum("gmk,gnk->gmn", a.double().abs(), b.double().abs())
    mode = TF32X3 if x3 else TF32
    used, rel = excess(got, ref, s, eps_for("gemm", mode) + k * U)
    _record("gemm", mode, rel, used)
    assert used <= 1.0


def _fc_split(in_size, out_size, batch, mode) -> int:
    """The InnerProduct's k-split count, read back from its scratch size (fcuda_api.cu fc_split)."""
    import ctypes
    from feathercnn_b200._lib import fcuda
    s, k = ctypes.c_size_t(), ctypes.c_size_t()
    assert fcuda().fcuda_inner_product_get_buffer_size(in_size, out_size, batch, ctypes.byref(s), ctypes.byref(k)) == 0
    planes = 2 if in_size % 4 == 0 and mode != TF32 else 1
    rest = s.value - (2 * batch * in_size if planes == 2 else 0)
    assert rest % (batch * out_size) == 0
    return rest // (batch * out_size)


def ip_rule(in_size: int, mode: int) -> tuple[str, float]:
    """(path, coef) of an InnerProduct with `in_size` inputs: the TensorGEMM when in_size % 4 == 0 (operands split per
    mode), else the fp32 SIMT kernel; coef multiplies S = |b| + sum |x w|."""
    path = "ip" if in_size % 4 == 0 else "simt"
    return path, eps_for(path, mode) + in_size * U


def run_inner_product(in_size, out_size, batch, relu, mode, seed=0):
    from feathercnn_b200 import booster
    booster.set_precision(mode)
    gen = torch.Generator(device="cuda").manual_seed(seed + in_size * 7 + out_size * 13 + batch)
    x = torch.rand((batch, in_size), generator=gen, device="cuda") * 2 - 1
    w = torch.randn((out_size, in_size), generator=gen, device="cuda") * math.sqrt(2.0 / in_size)
    w = w * torch.pow(10.0, -2 * torch.rand((out_size, 1), generator=gen, device="cuda"))
    b = torch.rand(out_size, generator=gen, device="cuda") - 0.5
    got = booster.inner_product(x, w, b, relu)
    torch.cuda.synchronize()
    ref = x.double() @ w.double().T + b.double()
    if relu:
        ref = ref.clamp_min(0)
    s = x.double().abs() @ w.double().abs().T + b.double().abs()
    path, coef = ip_rule(in_size, mode)
    used, rel = excess(got, ref, s, coef)
    _record(path, mode, rel, used)
    return used


IP_CASES = [
    (512, 300, 129, False),     # batch 129: two N tiles of the k-split partial-plane epilogue
    (1024, 1000, 256, True),    # batch 256: images 128-255 in the second N tile
    (4096, 1000, 256, False),   # several k-splits, two N tiles
    (36, 65, 129, False),       # K % 32 = 4
    (998, 40, 7, True),         # input_size % 4 != 0: SIMT fallback
    (25088, 4096, 64, True),    # VGG-16 fc6: 784 k-blocks in 9 splits of 88; the last owns 80
    (1316, 200, 129, True),     # 42 k-blocks in 5 splits of 9; the last owns 6
    (4096, 1000, 1, True),      # batch 1: one partial N tile
]


@gpu
@MODE_PARAMS
@pytest.mark.parametrize("in_size,out_size,batch,relu", IP_CASES)
def test_inner_product_bounds(cuda, in_size, out_size, batch, relu, mode):
    assert run_inner_product(in_size, out_size, batch, relu, mode) <= 1.0


# ---- 3. benchmark-size layers and batches ------------------------------------------------------------
BENCH = [("vgg16", 64), ("resnet50", 128), ("mobilenet_v1", 256)]


def _parse(mw):
    layers = []
    for line in mw.lines:
        f = line.split()
        type_, name, nb, nt = f[0], f[1], int(f[2]), int(f[3])
        bottoms, tops = f[4:4 + nb], f[4 + nb:4 + nb + nt]
        params = dict(kv.split("=") for kv in f[4 + nb + nt:])
        layers.append((type_, name, bottoms, tops, {int(k): v for k, v in params.items()}))
    return layers


@functools.lru_cache(maxsize=None)
def bench_layers(model: str, batch: int):
    """Every distinct Convolution / ConvolutionDepthWise / InnerProduct of a zoo model as feather::Net runs it with
    fusion on: BN / Scale folded into the filters (a bias), a following ReLU in the epilogue, a following 2x2 / s2 max
    pooling fused, the Eltwise SUM of a ResNet shortcut fused into the expand 1x1 (bottom 1) with the ReLU after it."""
    from feathercnn_b200.tools import modelgen
    mw = modelgen.ZOO[model]()
    layers = _parse(mw)
    readers = {}
    for L in layers:
        for bname in L[2]:
            readers.setdefault(bname, []).append(L)
    convs, fcs = {}, {}
    for type_, name, bottoms, tops, p in layers:
        if type_ == "InnerProduct":
            n_in = int(np.prod(mw.shape[bottoms[0]]))
            nxt = readers.get(tops[0], [])
            relu = len(nxt) == 1 and nxt[0][0] == "ReLU"
            fcs.setdefault((n_in, int(p[0]), relu), name)
            continue
        if type_ not in ("Convolution", "ConvolutionDepthWise"):
            continue
        ic, h, w = mw.shape[bottoms[0]]
        k, s, pad, group = int(p[1]), int(p.get(3, 1)), int(p.get(4, 0)), int(p.get(7, 1))
        c = Conv(name, int(p[0]), ic, h, w, k, sh=s, pad=pad, group=group, bias=p.get(5) == "1", batch=batch)
        cur = tops[0]
        while True:
            nxt = readers.get(cur, [])
            if len(nxt) != 1:
                break
            t2, _, b2, tops2, p2 = nxt[0]
            if t2 in ("BatchNorm", "Scale") and not c.relu:
                c.bias = True
            elif t2 == "ReLU" and not c.relu:
                c.relu = True
            elif t2 == "Pooling" and p2.get(0) == "0" and p2.get(1) == "2" and p2.get(2) == "2" and \
                    p2.get(3, "0") == "0" and p2.get(4, "0") == "0":
                c.pool = True
                break
            elif t2 == "Eltwise" and not c.relu and b2.index(cur) == 1:
                c.res = True
                after = readers.get(tops2[0], [])
                c.relu_after_add = len(after) == 1 and after[0][0] == "ReLU"
                break
            else:
                break
            cur = tops2[0]
        key = dataclasses.astuple(dataclasses.replace(c, name=""))
        convs.setdefault(key, c)
    return list(convs.values()), [(n_in, out, relu) for (n_in, out, relu) in fcs]


def _bench_params():
    out = []
    for model, batch in BENCH:
        try:
            convs, fcs = bench_layers(model, batch)
        except Exception:  # pragma: no cover - collection must not fail on a broken zoo; the test below reports it
            convs, fcs = [], []
        out += [pytest.param(model, c, id=f"{model}-b{batch}-{c.name}") for c in convs]
        out += [pytest.param(model, f, id=f"{model}-b{batch}-fc{f[0]}x{f[1]}") for f in fcs]
    return out


def test_bench_layer_inventory():
    """The geometries the benchmark runs, as bench_layers finds them (CPU only)."""
    convs, fcs = bench_layers("vgg16", 64)
    assert len(convs) == 12 and sorted(f[:2] for f in fcs) == [(4096, 1000), (4096, 4096), (25088, 4096)]
    assert sum(c.pool for c in convs) == 5 and all(c.relu for c in convs)
    convs, fcs = bench_layers("resnet50", 128)
    assert fcs == [(2048, 1000, False)]
    assert len(convs) == 21 and sum(c.res for c in convs) == 4 and all(c.relu_after_add for c in convs if c.res)
    convs, fcs = bench_layers("mobilenet_v1", 256)
    assert fcs == [] and sum(c.depthwise for c in convs) == 9
    assert any(c.name == "fc7" and (c.h, c.w, c.oc, c.batch) == (1, 1, 1000, 256) for c in convs)


@gpu
@pytest.mark.parametrize("model,layer", _bench_params())
def test_bench_layer_every_image(cuda, model, layer):
    """One distinct layer at the benchmark batch, default mode, tuned policy, every image against float64."""
    if isinstance(layer, tuple):
        n_in, out, relu = layer
        batch = dict(BENCH)[model]
        assert run_inner_product(n_in, out, batch, relu, FP32_SPLIT) <= 1.0
        return
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    import ctypes
    c = layer
    a = ctypes.c_int()
    p = booster.ConvParam.make(c.oc, c.ic, c.h, c.w, c.kh, stride=c.sh, pad=c.pad[0], group=c.group, bias=c.bias)
    assert fcuda().fcuda_conv_select_algo_tuned(ctypes.byref(p), ctypes.byref(a)) == 0
    if c.pool and not fcuda().fcuda_conv_can_pool(ctypes.byref(p), a.value):
        c = dataclasses.replace(c, pool=False)  # Net runs the pooling kernel after the convolution
    used, _, _ = run_conv(c, FP32_SPLIT, expect_algo=a.value, tuned=True)
    assert used <= 1.0


def _net_blobs(mw, net):
    """Blobs of the layers that survive fusion."""
    names = set(net.BlobNames())
    keep = []
    for type_, name, bottoms, tops, _ in _parse(mw):
        if type_ == "Input" or net.LayerFusedAway(name) == 1:
            continue
        keep += [t for t in tops if t in names]
    return keep


@gpu
@pytest.mark.parametrize("model,batch", BENCH, ids=[f"{m}-b{b}" for m, b in BENCH])
def test_benchmark_batch_images_equal_batch1(cuda, model_dir, model, batch):
    """With fusion and the CUDA graph on, images {0, 1, 127, 128, B-2, B-1} of a benchmark batch equal the same images
    forwarded alone, bit for bit, on every surviving blob: no image depends on its position in the batch."""
    from feathercnn_b200 import booster
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    booster.set_precision(FP32_SPLIT)
    mw = modelgen.ZOO[model]()
    param, binf = mw.save(model_dir / f"{model}_bits")
    # bit identity holds while every InnerProduct splits K the same way at both batch sizes
    for (n_in, out, _) in bench_layers(model, batch)[1]:
        assert _fc_split(n_in, out, batch, FP32_SPLIT) == _fc_split(n_in, out, 1, FP32_SPLIT), (n_in, out)
    gen = torch.Generator().manual_seed(batch)
    x = (torch.rand((batch,) + tuple(mw.shape["data"]), generator=gen) - 0.5).numpy()
    idx = sorted({i for i in (0, 1, 127, 128, batch - 2, batch - 1) if 0 <= i < batch})
    big = Net(fusion=True, cuda_graph=True)
    big.LoadParam(param)
    big.LoadWeights(binf)
    for _ in range(2):  # eager warm-up, then the captured graph
        big.Forward(x)
    blobs = _net_blobs(mw, big)
    assert blobs
    want = {}
    for bname in blobs:
        full = big.Extract(bname)
        assert full.shape[0] == batch
        want[bname] = full[idx].copy()
        del full
    del big
    one = Net(fusion=True, cuda_graph=True)
    one.LoadParam(param)
    one.LoadWeights(binf)
    for j, i in enumerate(idx):
        one.Forward(x[i:i + 1])
        for bname in blobs:
            got = one.Extract(bname)
            assert np.array_equal(got[0], want[bname][j]), (model, i, bname)


# ---- 4. the checker bites (CPU) -----------------------------------------------------------------------
def _cpu_case(c: Conv):
    x, w, b, r = make_data(c, "cpu")
    return x, w, b, r, conv_ref(c, x, w, b, r), conv_ref(c, x, w, b, r, absolute=True)


SENS_SHAPES = [c for c in SGECONV_SWEEP if c.name in ("sg_oc65", "sg_pix129", "sg_kb_table_ic17", "sg_1x7", "sg_pad_asym_br",
                                                     "sg_stride_1x2", "sg_group4_table", "sg_res_relu")]


@pytest.mark.parametrize("c", PROBES, ids=[p.name for p in PROBES])
def test_checker_rejects_tf32_operands_in_3xtf32_case(c):
    x, w, b, r, ref, s = _cpu_case(c)
    bad = conv_ref(c, tf32(x), tf32(w), b, r)
    used, _ = excess(bad, ref, s, EPS_3XTF32 + c.K * U)
    assert used > 1.0


@pytest.mark.parametrize("c", PROBES, ids=[p.name for p in PROBES])
def test_checker_rejects_dropped_bf16x3_term(c):
    x, w, b, r, ref, s = _cpu_case(c)
    p1x, p1w = bf16(x), bf16(w)
    p2x, p2w = bf16(x - p1x), bf16(w - p1w)
    nob = dataclasses.replace(c, bias=False, relu=False)
    good = conv_ref(nob, p1x, p1w, None, None) + conv_ref(nob, p1x, p2w, None, None) + conv_ref(nob, p2x, p1w, None, None)
    bad = good - conv_ref(nob, p2x, p1w, None, None)  # p2 * q1 dropped
    if b is not None:
        good, bad = good + b.double().view(1, -1, 1, 1), bad + b.double().view(1, -1, 1, 1)
    assert c.relu is False and r is None
    assert excess(good, ref, s, EPS_BF16X3 + c.K * U)[0] <= 1.0  # the modelled BF16x3 result itself passes
    assert excess(bad, ref, s, EPS_BF16X3 + c.K * U)[0] > 1.0


@pytest.mark.parametrize("c", SENS_SHAPES, ids=[c.name for c in SENS_SHAPES])
def test_checker_rejects_structural_defects(c):
    """Against the loosest (TF32) bound of the shape, each defect must still be caught."""
    x, w, b, r, ref, s = _cpu_case(c)
    coef = EPS_TF32 + c.K * U
    assert excess(ref, ref, s, coef)[0] == 0.0
    defects = {}
    # one border tap dropped: the middle-row, leftmost tap of the last output column (it reads image data there)
    wt = torch.zeros_like(w)
    wt[:, :, c.kh // 2, 0] = w[:, :, c.kh // 2, 0]
    tap = conv_ref(dataclasses.replace(c, bias=False, relu=False, res=False), x, wt, None, None)
    pre = conv_ref(dataclasses.replace(c, relu=False, res=False), x, w, b, None)
    pre_bad = pre.clone()
    pre_bad[..., -1] -= tap[..., -1]
    post = lambda y: wino_finish(c, y, r)
    defects["border tap"] = post(pre_bad)
    # the last k-block dropped (k = tap * ICg + ic, the implicit GEMM's order)
    icg = c.ic // c.group
    K = c.K
    kb_last = (K - 1) // 32 * 32
    if kb_last > 0:
        kidx = torch.arange(K).view(c.kh, c.kw, icg).permute(2, 0, 1)   # (ICg, KH, KW) -> k
        wk = w * (kidx < kb_last).to(w.dtype)
        defects["last k-block"] = conv_ref(c, x, wk, b, r)
    # bias shifted by one channel
    if b is not None:
        defects["bias shift"] = conv_ref(c, x, w, torch.roll(b, 1), r)
    # one image's outputs swapped with its neighbour's
    defects["image swap"] = ref[[1, 0] + list(range(2, ref.shape[0]))]
    for what, bad in defects.items():
        assert excess(bad, ref, s, coef)[0] > 1.0, what


@pytest.mark.parametrize("tile", [8, 4])
@pytest.mark.parametrize("c", WINO_SWEEP[:5], ids=[c.name for c in WINO_SWEEP[:5]])
def test_winograd_model(c, tile):
    """The float64 model with the kernels' transform matrices reproduces the convolution; in each mode its error is
    larger than rounding noise and below the TF32 convolution-domain scale by the amplification the margin allows."""
    c = dataclasses.replace(c, batch=1, res=False, pool=False)
    x, w, b, r = make_data(c, "cpu")
    want = conv_ref(dataclasses.replace(c, relu=False), x, w, b, None)
    s = conv_ref(c, x, w, b, None, absolute=True)
    assert excess(wino_model(c, x, w, b, tile, None), want, s, 1e-12)[0] <= 1.0
    rhos = {m: excess(wino_model(c, x, w, b, tile, m), want, s, 1.0)[1] for m in (TF32X3, TF32)}
    assert 2.0 ** -26 < rhos[TF32X3] < rhos[TF32] < 2.0 ** -4, rhos
    # a 3xTF32 kernel that lost its lo plane must fall outside the ceiling
    assert rhos[TF32] > WINO_MARGIN * rhos[TF32X3], rhos
