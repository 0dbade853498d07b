"""Every layer of the benchmarked nets, as feather::Net runs them, against a float64 restatement with per-element bounds.

tests/test_gpu_error_bounds.py holds each convolution / GEMM kernel to a per-element bound on inputs it draws itself.
This file checks what feather::Net computes around those kernels: the BatchNorm / Scale statistics folded into the
filters on the host (ConvLayer::Fuse / Init), the BN formula (BatchNormLayer::LoadWeights), the shortcut fusion
(Net::ApplyFusion), the pooling after a convolution that cannot pool in its epilogue, and the memory-bound kernels
(layers.cu) at the shapes the benchmark runs.

Chains.  With fusion on, a surviving layer stands for a chain of reference layers: a fused-away single-input layer
extends the chain that produced its bottom; a fused-away two-input Eltwise belongs to the convolution whose top was
not materialised, and the other addend is that convolution's residual.  `rebuild_chains` derives the chains from
LayerFusedAway, BlobNames and the param file only, and asserts that exactly the blobs it says are materialised exist
and that every surviving layer's bottoms do.

Restatement.  Each chain is evaluated in float64 (torch, on the GPU) from the Net's own bottom blobs of the checked
images, read zero-copy through ExtractDevice.  Errors therefore do not add up over depth: every bound is a one-layer
bound.  Semantics are the reference's: BN alpha / beta from slope / mean / var / bias with sqrt(var + eps); Scale with
or without bias; pooling in ceil mode, the window start subtracting both pads of an axis, average pooling dividing by
the number of in-bounds elements; softmax over one image's whole blob; Dropout multiplies by its scale.

Bounds (U = 2^-23, u = 2^-24 the unit roundoff; a folded chain is y = m * (conv(x, W) + b) + a per channel):
  - Convolution chains: the existing bound of test_gpu_error_bounds on
        S' = sum |x w m| + |b m| + A  (+ |residual|),
    where A is the sum of the absolute values of the terms that make up the offset a (|beta mean s| + |bn_bias s| + |t|
    for BN then Scale): a may cancel, its rounding error does not.  Plus the fold term FOLD * S', FOLD = 4 U, for the
    float32 rounding on the host (batchnorm_layer.h, conv_layer.h Fuse / Init):
      sqrt_var = fl(sqrt(fl(var + eps)))          rel. error <= 1.5 u
      beta     = fl(slope / sqrt_var)             <= 2.5 u
      alpha    = fl(bias - fl(fl(slope mean) / sqrt_var))   abs. error <= 3.5 u |beta mean| + u |alpha|
      fold_mul = fl(beta * s)                      <= 3.5 u;   W' = fl(W * fold_mul): <= 4.5 u per product |x w m|
      fold_add = fl(fl(alpha * s) + t)             <= (3.5 u |beta mean| + u |alpha|) |s| + u |alpha s| + u |fold_add|
      b'       = fl(fl(b * fold_mul) + fold_add)   <= 5.5 u |b m| + u |b'| + error(fold_add)
    With |alpha| <= |bn_bias| + |beta mean| and |b'| <= |b m| + A, the total is <= 4.5 u sum|x w m| + 6.5 u |b m|
    + 7.5 u A <= 7.5 u S' < FOLD S'.  A chain folds at most one BatchNorm and one Scale (asserted).
  - Winograd layers: WINO_MARGIN * rho * S', rho measured by wino_model on the folded filters rebuilt in numpy float32
    with the host's operations in the host's order, plus the same fold term.
  - A fused ReLU is 1-Lipschitz: the bound carries through.  Max pooling, fused or not: the max of the window's bounds.
  - Max pooling, ReLU, Split, Concat and Dropout with scale 1 on the Net's own input are exact.
  - Unfused BN / Scale (channel_affine_kernel: fmaf(mul, x, add), * mul2, + add2): AFFINE * S + U |ref| with
    S = |x m| + A, AFFINE = 4 U (alpha / beta as above, three roundings of partial results bounded by S).
  - Unfused Eltwise SUM of n bottoms: (n - 1) U S, S = sum |bottom|: one rounding per addition.
  - Average pooling: (cnt + 5) U S + U |ref|, S = sum |x| / cnt: the generic kernel adds cnt values in sequence, the
    global kernel ceil(HW / 32) per lane then five shuffle levels; the division by cnt rounds once.
  - InnerProduct: `ip_rule` of test_gpu_error_bounds.  Dropout with scale != 1: one rounding, U |ref|.
  - Softmax, per element relative to itself.  got_i / got_max against e_i = exp(x_i - max): that ratio does not depend
    on the sum, so its bound has no n 2^-23 term.  fl(x_i - max) errs by |x_i - max| u in the exponent, expf by 2 ulp,
    the two divisions by u each: e_i (|x_i - max| + 4) U.  Where e_i or p_i is below 2^-125 (fp32 subnormals or zero)
    an absolute floor (n + 4) 2^-149 covers the subnormal spacing.  Then the normalisation: |sum got - 1| <=
    (ceil(n / 256) + 15) U: each thread adds ceil(n / 256) terms, then five warp levels and eight warp partials.

The CPU tests feed the checker simulated Net outputs with one defect each and require it to reject every one.
Run with -s to print the worst |d|/S and the share of the bound used per (layer type, path, mode).
"""
from __future__ import annotations

import ctypes
import dataclasses
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_error_bounds import (FP32_SPLIT, MODE_NAME, NAIVE, PATH, TF32, TF32X3, U, WINO_MARGIN, WINOGRADF23,
                                   WINOGRADF63, Conv, conv_ref, eps_for, excess, ip_rule, wino_model)

gpu = pytest.mark.gpu

FOLD = 4 * U
AFFINE = 4 * U
CONV_TYPES = ("Convolution", "ConvolutionDepthWise")


# ---- report ---------------------------------------------------------------------------------------
REPORT: dict[tuple[str, str, str], list[float]] = {}


def _record(kind: str, path: str, mode: int, worst_rel: float, used: float) -> None:
    r = REPORT.setdefault((kind, path, MODE_NAME[mode]), [0.0, 0.0])
    r[0] = max(r[0], worst_rel)
    r[1] = max(r[1], used)


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\nworst |d|/S and the largest share of the per-element bound used, per (layer type, path, mode):")
        for (kind, path, mode), (rel, used) in sorted(REPORT.items()):
            print(f"  {kind:22s} {path:10s} {mode:10s} |d|/S {rel:.3e}   bound used {used:.3f}")


# ---- model: param file + weights ------------------------------------------------------------------
def load_model(param, binf) -> list[dict]:
    """oracle.parse_param plus every layer's weights in file order (ModelBin semantics of oracle._BinReader)."""
    from oracle import oracle as O
    layers = O.parse_param(param)
    mb = O._BinReader(binf)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))
    for L in layers:
        pd, typ = L["params"], L["type"]
        if typ in CONV_TYPES:
            kw = pd.get(1, 0)
            kh = pd.get(11, kw)
            num, size = pd.get(0, 0), pd.get(6, 0)
            L["w"] = t(mb.load(size, 0).reshape(num, size // (num * kh * kw), kh, kw))
            L["b"] = t(mb.load(num, 1)) if pd.get(5, 0) else None
        elif typ == "InnerProduct":
            out, size = pd.get(0, 0), pd.get(2, 0)
            L["w"] = t(mb.load(size, 0).reshape(out, size // out))
            L["b"] = t(mb.load(out, 1)) if pd.get(1, 0) else None
        elif typ == "BatchNorm":
            L["bn"] = [t(mb.load(pd.get(0, 0), 1)) for _ in range(4)]  # slope, mean, var, bias
        elif typ == "Scale":
            c = pd.get(0, 0)
            L["s"] = t(mb.load(c, 1))
            L["t"] = t(mb.load(c, 1)) if pd.get(1, 0) else None
    return layers


# ---- chains ---------------------------------------------------------------------------------------
@dataclasses.dataclass
class Chain:
    head: dict
    tops: list
    ops: list = dataclasses.field(default_factory=list)   # fused-away layers after the head, in order
    residual: str | None = None                            # the other addend of a fused Eltwise

    @property
    def bottoms(self):
        return list(self.head["bottoms"]) + ([self.residual] if self.residual else [])


def rebuild_chains(layers, fused_away, blob_names) -> tuple[list[Chain], set]:
    """Chains of the layers that survive fusion, from LayerFusedAway (`fused_away(name)`), BlobNames and the param file.
    Returns (chains, materialised blobs)."""
    chains, producer, materialised = [], {}, set()
    for L in layers:
        f = fused_away(L["name"])
        assert f in (0, 1), (L["name"], f)
        if L["type"] == "Input":
            assert f == 0
            materialised |= set(L["tops"])
            continue
        if not f:
            ch = Chain(L, list(L["tops"]))
            chains.append(ch)
            for t in ch.tops:
                producer[t] = ch
            materialised |= set(ch.tops)
            continue
        if len(L["bottoms"]) == 1:
            ch = producer[L["bottoms"][0]]
            assert ch.tops == L["bottoms"], (L["name"], ch.tops)
        else:
            assert L["type"] == "Eltwise" and len(L["bottoms"]) == 2, L["name"]
            mine = [b for b in L["bottoms"] if b not in blob_names and producer[b].head["type"] in CONV_TYPES
                    and producer[b].tops == [b]]
            assert len(mine) == 1, (L["name"], mine)
            ch = producer[mine[0]]
            ch.residual = [b for b in L["bottoms"] if b != mine[0]][0]
            assert ch.residual in materialised, (L["name"], ch.residual)
        ch.ops.append(L)
        materialised -= set(ch.tops)
        ch.tops = list(L["tops"])
        materialised |= set(ch.tops)
        for t in ch.tops:
            producer[t] = ch
    for ch in chains:
        missing = [b for b in ch.bottoms if b not in materialised]
        assert not missing, (ch.head["name"], missing)
    return chains, materialised


# ---- float64 restatement --------------------------------------------------------------------------
def _ch(v, like):
    return v.to(device=like.device, dtype=torch.float64).view(1, -1, 1, 1)


def affine_of(L):
    """float64 (m, a, A) of a BatchNorm / Scale layer: y = m x + a; A = sum of the absolute terms of a."""
    if L["type"] == "BatchNorm":
        slope, mean, var, bias = (v.double() for v in L["bn"])
        eps = float(np.float32(L["params"].get(1, 0.0)))
        sv = torch.sqrt(var + eps)
        return slope / sv, bias - slope * mean / sv, bias.abs() + (slope * mean / sv).abs()
    s = L["s"].double()
    t = L["t"].double() if L["t"] is not None else torch.zeros_like(s)
    return s, t, t.abs()


def host_affine32(L):
    """(mul, add) in float32 as BatchNormLayer::LoadWeights / ScaleLayer hold them (batchnorm_layer.h:37-41)."""
    if L["type"] == "BatchNorm":
        slope, mean, var, bias = (v.numpy() for v in L["bn"])
        eps = np.float32(L["params"].get(1, 0.0))
        sv = np.sqrt(var + eps).astype(np.float32)
        return (slope / sv).astype(np.float32), (bias - slope * mean / sv).astype(np.float32)
    s = L["s"].numpy()
    return s, (L["t"].numpy() if L["t"] is not None else np.zeros_like(s))


def folded_filters32(head, folds):
    """W' and b' as ConvLayer::Fuse / Init compute them on the host: fold_add = fold_add * m + a, fold_mul *= m in
    float32, then W' = W * fold_mul, b' = b * fold_mul + fold_add."""
    w, b = head["w"].numpy(), head["b"]
    mul = np.ones(w.shape[0], np.float32)
    add = np.zeros(w.shape[0], np.float32)
    for L in folds:
        m, a = host_affine32(L)
        add = (add * m + a).astype(np.float32)
        mul = (mul * m).astype(np.float32)
    w2 = (w * mul[:, None, None, None]).astype(np.float32)
    b2 = ((b.numpy() * mul).astype(np.float32) + add).astype(np.float32) if b is not None else add
    return torch.from_numpy(w2), torch.from_numpy(b2)


def pool_params(L, h, w):
    """(type, kh, kw, sh, sw, window row offset, window column offset, oh, ow) of PoolingLayer L on an h x w plane."""
    pd = L["params"]
    kw = pd.get(1, 0)
    kh = pd.get(11, kw)
    sw = pd.get(2, 1)
    sh = pd.get(12, sw)
    pl = pd.get(3, 0)
    pr, pt = pd.get(14, pl), pd.get(13, pl)
    pb = pd.get(15, pt)
    if pd.get(4, 0):
        return pd.get(0, 0), h, w, 1, 1, 0, 0, 1, 1
    oh = math.ceil((h + pt + pb - kh) / sh) + 1
    ow = math.ceil((w + pl + pr - kw) / sw) + 1
    return pd.get(0, 0), kh, kw, sh, sw, pt + pb, pl + pr, oh, ow


def pool_windows(t, L, fill):
    """(N, C, OH, OW, KH * KW) windows of pooling layer L over t (window start = o * stride - both pads), `fill` outside
    the image, and the in-bounds count per window (1, 1, OH, OW)."""
    h, w = t.shape[2:]
    _, kh, kw, sh, sw, oy, ox, oh, ow = pool_params(L, h, w)
    pad_b = max(0, (oh - 1) * sh - oy + kh - h)
    pad_r = max(0, (ow - 1) * sw - ox + kw - w)
    grid = lambda z, v: F.pad(z, (ox, pad_r, oy, pad_b), value=v).unfold(2, kh, sh).unfold(3, kw, sw)[:, :, :oh, :ow]
    win = grid(t, fill).reshape(t.shape[0], t.shape[1], oh, ow, kh * kw)
    cnt = grid(torch.ones((1, 1, h, w), dtype=t.dtype, device=t.device), 0.0).sum((-1, -2))
    return win, cnt


def pool_max(t, L):
    return pool_windows(t, L, -math.inf)[0].amax(-1)


def pool_avg(t, L):
    win, cnt = pool_windows(t, L, 0.0)
    return win.sum(-1) / cnt, cnt


@dataclasses.dataclass
class Result:
    top: str
    ref: torch.Tensor
    bound: torch.Tensor      # absolute, per element
    scale: torch.Tensor      # S, for the |d|/S report
    kind: str
    path: str


def conv_geometry(L, x) -> Conv:
    pd = L["params"]
    assert pd.get(2, 1) == 1 and pd.get(12, 1) == 1, "dilated convolutions are not in the checked nets"
    kw = pd.get(1, 0)
    kh = pd.get(11, kw)
    sw = pd.get(3, 1)
    pl = pd.get(4, 0)
    pt = pd.get(14, pl)
    return Conv(L["name"], pd.get(0, 0), x.shape[1], x.shape[2], x.shape[3], kh, kw, sh=pd.get(13, sw), sw=sw,
                pad=(pl, pt, pl, pt), group=pd.get(7, 1), bias=L["b"] is not None, batch=x.shape[0])


def restate_conv_chain(ch: Chain, ins: dict, mode: int, algo: int) -> list[Result]:
    head = ch.head
    x = ins[head["bottoms"][0]]
    c = conv_geometry(head, x)
    dev = x.device
    w, b = head["w"].to(dev), (head["b"].to(dev) if head["b"] is not None else None)
    ref = conv_ref(c, x, w, b, None)
    s = conv_ref(c, x, w, b, None, absolute=True)
    folds, pool, relu_seen = [], None, False
    for L in ch.ops:
        assert pool is None, (head["name"], "pooling must end the chain")
        if L["type"] in ("BatchNorm", "Scale"):
            assert not relu_seen and L["type"] not in [f["type"] for f in folds], (head["name"], L["name"])
            m, a, A = affine_of(L)
            ref = ref * _ch(m, ref) + _ch(a, ref)
            s = s * _ch(m.abs(), s) + _ch(A, s)
            folds.append(L)
        elif L["type"] == "ReLU":
            ref = ref.clamp_min(0)
            relu_seen = True
        elif L["type"] == "Eltwise":
            r = ins[ch.residual]
            ref, s = ref + r, s + r.abs()
        elif L["type"] == "Pooling":
            pool = L
        else:
            raise AssertionError((head["name"], L["type"]))
    path = PATH[algo]
    if algo in (WINOGRADF63, WINOGRADF23):
        # rho of the kernel's pipeline on the folded float32 filters, measured on the first checked image
        w2, b2 = (v.to(dev) for v in folded_filters32(head, folds))
        c2 = dataclasses.replace(c, bias=True)
        ym = wino_model(c2, x[:1], w2, b2, 8 if algo == WINOGRADF63 else 4, mode)
        _, rho = excess(ym, conv_ref(c2, x[:1], w2, b2, None), conv_ref(c2, x[:1], w2, b2, None, absolute=True), 1.0)
        coef = WINO_MARGIN * rho
    else:
        coef = eps_for(path, mode) + c.K * U
    if folds:
        coef = coef + FOLD
    bound = coef * s + U * ref.abs()
    if pool is not None:
        assert pool["params"].get(0, 0) == 0, "a convolution absorbs max pooling only"
        ref, bound, s = pool_max(ref, pool), pool_max(bound, pool), pool_max(s, pool)
    return [Result(ch.tops[0], ref, bound, s, head["type"] + ("+" + "+".join(L["type"] for L in ch.ops) if ch.ops else ""),
                   path)]


def restate_chain(ch: Chain, ins: dict, mode: int, algo: int = -1) -> list[Result]:
    """float64 reference, per-element bound and S of every top of a chain, from its bottoms `ins` (float64)."""
    head, typ = ch.head, ch.head["type"]
    if typ in CONV_TYPES:
        return restate_conv_chain(ch, ins, mode, algo)
    x = ins[head["bottoms"][0]]
    zero = lambda t: torch.zeros_like(t)
    if typ in ("BatchNorm", "Scale"):
        ref, s = x, x.abs()
        for L in [head] + ch.ops:
            if L["type"] == "ReLU":
                ref = ref.clamp_min(0)
                continue
            m, a, A = affine_of(L)
            ref, s = ref * _ch(m, ref) + _ch(a, ref), s * _ch(m.abs(), s) + _ch(A, s)
        return [Result(ch.tops[0], ref, AFFINE * s + U * ref.abs(), s, "+".join([typ] + [L["type"] for L in ch.ops]), "affine")]
    if typ == "Eltwise":
        assert head["params"].get(0, 1) == 1 and 1 not in head["params"], "Eltwise SUM without coefficients only"
        xs = [ins[b] for b in head["bottoms"]]
        ref, s = sum(xs), sum(v.abs() for v in xs)
        for L in ch.ops:
            assert L["type"] == "ReLU"
            ref = ref.clamp_min(0)
        return [Result(ch.tops[0], ref, (len(xs) - 1) * U * s, s, "+".join([typ] + [L["type"] for L in ch.ops]), "add")]
    if typ == "InnerProduct":
        xf = x.reshape(x.shape[0], -1)
        w = head["w"].to(x.device).double()
        b = head["b"].to(x.device).double() if head["b"] is not None else torch.zeros(w.shape[0], dtype=torch.float64,
                                                                                       device=x.device)
        ref, s = xf @ w.T + b, xf.abs() @ w.abs().T + b.abs()
        for L in ch.ops:
            assert L["type"] == "ReLU"
            ref = ref.clamp_min(0)
        path, coef = ip_rule(xf.shape[1], mode)
        return [Result(ch.tops[0], ref, coef * s + U * ref.abs(), s, "+".join([typ] + [L["type"] for L in ch.ops]), path)]
    assert not ch.ops, (head["name"], "not fusible")
    if typ == "Pooling":
        if head["params"].get(0, 0) == 0:
            ref = pool_max(x, head)
            return [Result(ch.tops[0], ref, zero(ref), ref.abs(), "Pooling max", "exact")]
        ref, cnt = pool_avg(x, head)
        s = pool_avg(x.abs(), head)[0]
        return [Result(ch.tops[0], ref, (cnt + 5) * U * s + U * ref.abs(), s, "Pooling avg", "sum")]
    if typ == "ReLU":
        ref = x.clamp_min(0)
        return [Result(ch.tops[0], ref, zero(ref), ref.abs(), typ, "exact")]
    if typ == "Split":
        return [Result(t, x, zero(x), x.abs(), typ, "exact") for t in ch.tops]
    if typ == "Concat":
        axis = head["params"].get(0, 0)
        ref = torch.cat([ins[b] for b in head["bottoms"]], dim=1 + axis)
        return [Result(ch.tops[0], ref, zero(ref), ref.abs(), typ, "exact")]
    if typ == "Dropout":
        scale = float(np.float32(head["params"].get(0, 1.0)))
        ref = x * scale
        return [Result(ch.tops[0], ref, U * ref.abs(), ref.abs(), typ, "exact" if scale == 1.0 else "scale")]
    raise AssertionError(f"no restatement for {typ}")


def softmax_excess(x, got) -> tuple[float, float, float]:
    """Softmax over each row of x (float64 logits, (N, n)) against `got`: (share of the ratio bound used, share of the
    normalisation bound used, worst relative error of the ratio)."""
    x, got = x.double().reshape(x.shape[0], -1), got.double().reshape(got.shape[0], -1)
    n = x.shape[1]
    arg = x - x.max(1, keepdim=True).values
    e = torch.exp(arg)
    p = e / e.sum(1, keepdim=True)
    tiny = 2.0 ** -125
    floor = torch.where((e < tiny) | (p < tiny), torch.full_like(e, (n + 4) * 2.0 ** -149), torch.zeros_like(e))
    ratio = got / got.max(1, keepdim=True).values
    used_ratio, _ = excess(ratio, e, e * (arg.abs() + 4) * U + floor, 1.0, 0.0)
    _, rel = excess(torch.where(floor > 0, e, ratio), e, e, 1.0, 0.0)   # relative error where fp32 is normal
    used_sum = float(((got.sum(1) - 1).abs() / ((math.ceil(n / 256) + 15) * U)).max())
    return used_ratio, used_sum, rel


def check_chain(ch: Chain, ins: dict, got: dict, mode: int, algo: int = -1) -> list[tuple[str, float, float, str, str]]:
    """[(top, share of the bound used, worst |d|/S, kind, path)] of every top of `ch`; `got` maps tops to the Net's
    values (float64) of the same images as `ins`."""
    if ch.head["type"] == "Softmax":
        assert not ch.ops
        x, g = ins[ch.head["bottoms"][0]], got[ch.tops[0]]
        used_ratio, used_sum, rel = softmax_excess(x, g)
        return [(ch.tops[0], max(used_ratio, used_sum), rel, "Softmax", "ratio+sum")]
    out = []
    for r in restate_chain(ch, ins, mode, algo):
        g = got[r.top]
        assert g.numel() == r.ref.numel(), (r.top, g.shape, r.ref.shape)
        shape = g.shape
        used, _ = excess(g, r.ref.reshape(shape), r.bound.reshape(shape), 1.0, 0.0)
        _, rel = excess(g, r.ref.reshape(shape), r.scale.reshape(shape), 1.0, 0.0)
        out.append((r.top, used, rel, r.kind, r.path))
    return out


# ---- CPU: chain rebuild, restatement, the checker rejects defects ----------------------------------
def _cpu_net(fusion: bool):
    from feathercnn_b200.net import Net
    return Net(fusion=fusion)


@pytest.mark.parametrize("fusion", [True, False], ids=["fused", "plain"])
@pytest.mark.parametrize("model", ["mini", "vgg16", "resnet50", "mobilenet_v1"])
def test_chain_rebuild_on_host(tmp_path, model, fusion):
    """The rebuild agrees with the Net's own fusion rewrite on the host (no weights there, so BN / Scale are not folded
    into convolutions; BN absorbs its Scale and ReLU instead)."""
    from oracle import oracle as O
    from feathercnn_b200.tools import modelgen
    mw = modelgen.ZOO[model]()
    param, _ = mw.save(tmp_path / model)
    net = _cpu_net(fusion)
    net.LoadParamFromText(open(param).read())
    absorbed = net.FuseNow()
    layers = O.parse_param(param)
    names = set(net.BlobNames())
    chains, mat = rebuild_chains(layers, net.LayerFusedAway, names)
    assert mat == names
    assert len(chains) + absorbed + 1 == len(layers)
    assert sum(len(ch.ops) for ch in chains) == absorbed
    if not fusion:
        assert absorbed == 0 and all(not ch.ops for ch in chains)
    elif model == "resnet50":  # shortcut adds stay unfused: their addends come from BatchNorm layers here
        bns = [ch for ch in chains if ch.head["type"] == "BatchNorm"]
        assert len(bns) == 53 and all(ch.ops[0]["type"] == "Scale" for ch in bns)
    elif model == "vgg16":
        assert sum(any(L["type"] == "Pooling" for L in ch.ops) for ch in chains) == 5
    for ch in chains:
        assert net.LayerConvAlgo(ch.head["name"]) == -1  # before any Reshape the booster holds no algorithm
    assert net.LayerConvAlgo("no_such_layer") == -1


def _small_model(tmp_path):
    """conv -> BN -> Scale -> ReLU -> Split -> (1x1 conv -> BN -> Scale) + shortcut -> ReLU -> 3x3/s2 average pooling
    with clipped ceil-mode windows -> InnerProduct -> Softmax, wide statistics."""
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter(seed=5, wide_stats=True)
    x = m.input("data", 5, 10, 12)
    x = m.conv("conv1", x, 40, 3, 1, 1, True)
    x = m.batchnorm("bn1", x); x = m.scale("scale1", x, True); x = m.relu("relu1", x)
    a, b = m.split("split1", x, ["s1a", "s1b"])
    y = m.conv("conv2", b, 40, 1, 1, 0, False)
    y = m.batchnorm("bn2", y); y = m.scale("scale2", y, True)
    x = m.eltwise("sum1", [a, y]); x = m.relu("relu2", x)
    x = m.pool("pool1", x, 1, 3, 2, 0)
    x = m.fc("fc1", x, 30, True)
    m.softmax("prob", x)
    param, binf = m.save(tmp_path / "small")
    return load_model(param, binf)


# what feather::Net's fusion does to the small model on the GPU (BN / Scale folded into the convolutions)
SMALL_FUSED = {"bn1", "scale1", "relu1", "bn2", "scale2", "sum1", "relu2"}


def _forward_all(chains, x, mode=FP32_SPLIT):
    """float64 'Net outputs' of every materialised blob: each chain's restatement on the previous outputs."""
    blobs = {"data": x}
    for ch in chains:
        if ch.head["type"] == "Softmax":
            v = blobs[ch.head["bottoms"][0]]
            blobs[ch.tops[0]] = torch.softmax(v.reshape(v.shape[0], -1), 1).reshape(v.shape)
            continue
        for r in restate_chain(ch, blobs, mode, NAIVE):
            blobs[r.top] = r.ref
    return blobs


@pytest.fixture(scope="module")
def small(tmp_path_factory):
    layers = _small_model(tmp_path_factory.mktemp("small"))
    names = {t for L in layers for t in L["tops"]} - {"conv1", "bn1", "scale1", "conv2", "bn2", "scale2", "sum1"}
    chains, mat = rebuild_chains(layers, lambda n: int(n in SMALL_FUSED), names)
    assert mat == names
    byname = {ch.head["name"]: ch for ch in chains}
    assert [L["name"] for L in byname["conv1"].ops] == ["bn1", "scale1", "relu1"]
    assert [L["name"] for L in byname["conv2"].ops] == ["bn2", "scale2", "sum1", "relu2"]
    assert byname["conv2"].residual == "s1a"
    x = torch.rand((3, 5, 10, 12), generator=torch.Generator().manual_seed(0), dtype=torch.float64) - 0.5
    return layers, chains, byname, _forward_all(chains, x)


def _used(ch, blobs, outs):
    return max(u for _, u, *_ in check_chain(ch, blobs, outs, FP32_SPLIT, NAIVE))


def test_small_model_statistics_are_wide(small):
    """The wide statistics do what they are for: a negative multiplier, a dead channel, var <= eps channels whose
    multiplier moves by >= sqrt(2) without eps, and offsets that are not small."""
    layers, _, _, blobs = small
    bn = {L["name"]: L for L in layers}["bn1"]
    slope, mean, var, bias = (v.double() for v in bn["bn"])
    eps = float(np.float32(bn["params"][1]))
    assert abs(eps - 1e-3) < 1e-9 and (var <= eps).float().mean() >= 0.25
    m = slope / torch.sqrt(var + eps)
    assert (m < 0).any() and (m == 0).sum() == 1
    assert 1e4 <= m.abs().max() / m.abs()[m != 0].min() and abs(float(m.pow(2).mean().sqrt()) - 1) < 1e-3
    small_var = var <= eps
    assert (slope[small_var] / var[small_var].sqrt() / m[small_var]).abs().min() >= math.sqrt(2) * (1 - 1e-6)
    alpha = bias - m * mean
    assert alpha.abs().mean() > 0.3
    for name, v in blobs.items():
        assert float(v.abs().max()) < 1e4 and bool(v.abs().max() > 0), name


def test_checker_accepts_the_restatement(small):
    _, chains, _, blobs = small
    for ch in chains:
        assert _used(ch, blobs, blobs) < 1e-6, ch.head["name"]


def _copy(L, **kw):
    L = dict(L)
    L.update(kw)
    return L


def _redo(ch, blobs, **chain_kw):
    bad = dataclasses.replace(ch, **chain_kw)
    return {r.top: r.ref for r in restate_chain(bad, blobs, FP32_SPLIT, NAIVE)}


def test_checker_rejects_bn_without_eps(small):
    _, _, byname, blobs = small
    ch = byname["conv1"]
    bn = ch.ops[0]
    bad = _redo(ch, blobs, ops=[_copy(bn, params={**bn["params"], 1: 0.0})] + ch.ops[1:])
    assert _used(ch, blobs, bad) > 1.0


def test_checker_rejects_dropped_scale_bias_of_one_channel(small):
    _, _, byname, blobs = small
    ch = byname["conv2"]
    sc = ch.ops[1]
    t = sc["t"].clone()
    t[int(t.argmax())] = 0.0   # the largest positive bias: the ReLU after the add cannot hide all of it
    bad = _redo(ch, blobs, ops=[ch.ops[0], _copy(sc, t=t)] + ch.ops[2:])
    assert _used(ch, blobs, bad) > 1.0


def test_checker_rejects_residual_added_after_relu(small):
    _, _, byname, blobs = small
    ch = byname["conv2"]
    bn, sc, add, relu = ch.ops
    bad = _redo(ch, blobs, ops=[bn, sc, relu, add])
    assert _used(ch, blobs, bad) > 1.0


def test_checker_rejects_relu_before_negative_multiplier(small):
    _, _, byname, blobs = small
    ch = byname["conv1"]
    bn, sc, relu = ch.ops
    assert (affine_of(bn)[0] * affine_of(sc)[0] < 0).any()
    # ReLU on the raw convolution, then the affine: wrong exactly on the channels with a negative multiplier
    conv_only = _redo(ch, blobs, ops=[relu])[ch.tops[0]]
    m, a, _ = affine_of(bn)
    s, t, _ = affine_of(sc)
    bad = {ch.tops[0]: (conv_only * _ch(m, conv_only) + _ch(a, conv_only)) * _ch(s, conv_only) + _ch(t, conv_only)}
    assert _used(ch, blobs, bad) > 1.0


def test_checker_rejects_neighbouring_image(small):
    _, chains, _, blobs = small
    for ch in chains:
        shifted = {t: torch.roll(blobs[t], -1, 0) for t in ch.tops}
        assert _used(ch, blobs, shifted) > 1.0, ch.head["name"]


def test_checker_rejects_average_over_full_window_area(small):
    _, _, byname, blobs = small
    ch = byname["pool1"]
    x = blobs[ch.head["bottoms"][0]]
    ref, cnt = pool_avg(x, ch.head)
    assert (cnt < 9).any()                      # the ceil-mode windows at the right and bottom edges are clipped
    bad = {ch.tops[0]: ref * cnt / 9.0}
    assert _used(ch, blobs, bad) > 1.0


def _spread_logits(n_img, n, seed):
    """Logits whose softmax spans normal, subnormal and underflowing probabilities (x - max down to -120)."""
    g = torch.Generator().manual_seed(seed)
    return -120.0 * torch.rand((n_img, n), generator=g, dtype=torch.float64).float().double()


def test_checker_softmax_defects():
    x = _spread_logits(3, 1000, 1)
    p = torch.softmax(x, 1).float().double()                   # float32 rounding of the true probabilities passes
    assert softmax_excess(x, p)[:2] <= (1.0, 1.0)
    assert ((p > 0) & (p < 2.0 ** -100)).sum() > 10
    flushed = torch.where(p < 2.0 ** -100, torch.zeros_like(p), p)
    assert softmax_excess(x, flushed)[0] > 1.0
    e = torch.exp(x - x.max(1, keepdim=True).values)
    other = e / e.sum(1, keepdim=True).roll(1, 0)              # normalised by another image's sum
    assert softmax_excess(x, other)[1] > 1.0


def test_checker_softmax_rejects_neighbouring_image():
    x = _spread_logits(3, 257, 2)
    p = torch.softmax(x, 1)
    assert softmax_excess(x, p.roll(1, 0))[0] > 1.0


# ---- GPU: every layer of the benchmarked nets ------------------------------------------------------
class _DeviceBuffer:
    def __init__(self, ptr: int, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (ptr, False), "version": 3}


def fetch(net, name, idx) -> torch.Tensor:
    """Images `idx` of blob `name`, float64, read in place through ExtractDevice."""
    ptr, shape = net.ExtractDevice(name)
    return torch.as_tensor(_DeviceBuffer(ptr, shape), device="cuda")[idx].double()


@dataclasses.dataclass(frozen=True)
class NetCase:
    model: str
    batch: int
    fusion: bool
    mode: int = FP32_SPLIT
    wide: bool = False

    @property
    def id(self):
        return (f"{self.model}{'-wide' if self.wide else ''}-b{self.batch}-{'fused' if self.fusion else 'plain'}"
                f"-{MODE_NAME[self.mode]}")


NET_CASES = (
    [NetCase(m, b, f) for m in ("vgg16", "resnet50", "mobilenet_v1") for b in (64, 128, 256) for f in (True, False)]
    + [NetCase("resnet50", 128, True, TF32X3), NetCase("resnet50", 128, True, TF32)]
    + [NetCase("mini", 3, f) for f in (True, False)]
    + [NetCase(m, b, f, wide=True) for m, b in (("resnet50", 128), ("mobilenet_v1", 256), ("mini", 3))
       for f in (True, False)]
)

_MODELS: dict = {}


def _model(model_dir, model, wide):
    key = (model, wide)
    if key not in _MODELS:
        from feathercnn_b200.tools import modelgen
        mw = modelgen.ZOO[model](wide_stats=True) if wide else modelgen.ZOO[model]()
        param, binf = mw.save(model_dir / f"bounds_{model}{'_wide' if wide else ''}")
        _MODELS.clear()  # one model's weights in host memory at a time (cases are grouped by model)
        _MODELS[key] = (param, binf, mw.shape["data"], load_model(param, binf))
    return _MODELS[key]


def _images(batch, model):
    if model == "mini":
        return list(range(batch))
    pick = int(np.random.default_rng(batch).integers(batch))
    return sorted({i for i in (0, 127, 128, batch - 1, pick) if 0 <= i < batch})


@gpu
@pytest.mark.parametrize("case", NET_CASES, ids=[c.id for c in NET_CASES])
def test_net_layers_within_bounds(cuda, model_dir, case):
    """Run the Net as bench.py does (fusion + graph: eager, capture, then check the replay), then check every surviving
    layer's chain on the sampled images against its float64 restatement fed the Net's own bottoms."""
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    from feathercnn_b200.net import Net
    booster.set_precision(case.mode)
    param, binf, shape, layers = _model(model_dir, case.model, case.wide)
    net = Net(fusion=case.fusion, cuda_graph=case.fusion)
    net.LoadParam(param)
    net.LoadWeights(binf)
    gen = torch.Generator().manual_seed(case.batch)
    x = (torch.rand((case.batch,) + tuple(shape), generator=gen) - 0.5).numpy()
    for _ in range(3 if case.fusion else 1):
        net.Forward(x)
    net.Synchronize()
    names = set(net.BlobNames())
    chains, mat = rebuild_chains(layers, net.LayerFusedAway, names)
    assert mat == names
    idx = _images(case.batch, case.model)
    failures = []
    for ch in chains:
        algo = -1
        if ch.head["type"] in CONV_TYPES:
            algo = net.LayerConvAlgo(ch.head["name"])
            n, c, h, w = net.BlobShape(ch.head["bottoms"][0])
            g = conv_geometry(ch.head, torch.empty((1, c, h, w), device="meta"))
            # the ConvParam the layer selected with: BN / Scale folds set bias_term, a ReLU before any shortcut add
            # (not the one after it) sets the activation
            types = [L["type"] for L in ch.ops]
            folded = "BatchNorm" in types or "Scale" in types
            relu = "ReLU" in types and ("Eltwise" not in types or types.index("ReLU") < types.index("Eltwise"))
            p = booster.ConvParam.make(g.oc, g.ic, g.h, g.w, g.kh, g.kw, stride=g.sh, stride_w=g.sw, pad_lbrt=g.pad,
                                       group=g.group, bias=g.bias or folded, relu=relu)
            want = ctypes.c_int()
            assert fcuda().fcuda_conv_select_algo_tuned(ctypes.byref(p), ctypes.byref(want)) == 0
            if algo != want.value:
                failures.append(f"{ch.head['name']}: Net runs algo {algo}, select_algo_tuned gives {want.value}")
                continue
        ins = {b: fetch(net, b, idx) for b in dict.fromkeys(ch.bottoms)}
        got = {t: fetch(net, t, idx) for t in ch.tops}
        for top, used, rel, kind, path in check_chain(ch, ins, got, case.mode, algo):
            _record(kind, path, case.mode, rel, used)
            if used > 1.0:
                failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}, |d|/S {rel:.3g}")
        if case.wide:
            for t, v in got.items():
                if not (float(v.abs().max()) < 1e4 and bool((v != 0).any())):
                    failures.append(f"{t}: wide-statistics blob out of range (max |v| {float(v.abs().max()):.3g})")
        del ins, got
    del net
    torch.cuda.empty_cache()
    assert not failures, f"{case.id}: {len(failures)} failures\n" + "\n".join(failures[:40])


# ---- GPU: edge cases of the memory-bound kernels -----------------------------------------------------
def _pool_layer(type_, k, s, pads=(0, 0, 0, 0), glob=False):
    pl, pr, pt, pb = pads
    return {"type": "Pooling", "name": "p", "params": {0: type_, 1: k, 2: s, 3: pl, 14: pr, 13: pt, 15: pb, 4: int(glob)}}


GLOBAL_POOL_CASES = [(6, 3, 5), (6, 4, 7), (64, 7, 7), (8, 56, 56)]   # (C, H, W): HW 15, 28, 49, 3136


@gpu
@pytest.mark.parametrize("type_", [0, 1], ids=["max", "avg"])
@pytest.mark.parametrize("chw", GLOBAL_POOL_CASES, ids=[f"hw{h * w}" for _, h, w in GLOBAL_POOL_CASES])
def test_global_pooling_within_bounds(cuda, chw, type_):
    from feathercnn_b200 import booster
    c, h, w = chw
    x = torch.rand((3, c, h, w), generator=torch.Generator(device="cuda").manual_seed(h * w), device="cuda") * 2 - 1
    got = booster.pooling(x, type_, h, w, 1, 1, 0, 0, 0, 0, True).double()
    ch = Chain(_pool_layer(type_, h, 1, glob=True), ["out"])
    ch.head["bottoms"] = ["x"]
    [(_, used, rel, kind, path)] = check_chain(ch, {"x": x.double()}, {"out": got}, FP32_SPLIT)
    _record(kind + " global", path, FP32_SPLIT, rel, used)
    assert used <= 1.0


SOFTMAX_N = [1, 255, 256, 257, 1000, 100352]


@gpu
@pytest.mark.parametrize("n", SOFTMAX_N)
def test_softmax_within_bounds(cuda, n):
    """Batch 256; logits spread to x - max = -120, so small probabilities are subnormal or underflow; image 1 has a
    tied maximum."""
    from feathercnn_b200 import booster
    x = _spread_logits(256, n, n).float().cuda()
    if n > 1:
        x[1, n // 2] = x[1].max()
    got = booster.softmax(x.view(256, n, 1, 1)).view(256, n)
    used_ratio, used_sum, rel = softmax_excess(x.double(), got)
    _record("Softmax", "ratio+sum", FP32_SPLIT, rel, max(used_ratio, used_sum))
    assert used_ratio <= 1.0 and used_sum <= 1.0


AFFINE_CASES = [(mul2, add2, relu) for mul2 in (False, True) for add2 in (False, True) for relu in (False, True)]


@gpu
@pytest.mark.parametrize("hw", [1, 13])
@pytest.mark.parametrize("mul2,add2,relu", AFFINE_CASES, ids=[f"mul2{int(a)}-add2{int(b)}-relu{int(c)}" for a, b, c in AFFINE_CASES])
def test_batchnorm_affine_variants(cuda, hw, mul2, add2, relu):
    """channel_affine_kernel at batch 3 through fcuda_batchnorm_forward with every combination of the fused Scale
    multiplier (mul2), Scale bias (add2) and ReLU, and through fcuda_scale_forward with and without bias, against the
    float64 affine of the stored statistics.  Both entry points require mul and add (fcuda_scale_forward: mul), so the
    kernel's add-only branch has no caller and is not reached."""
    from feathercnn_b200 import booster
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter(seed=hw + 2 * mul2 + 4 * add2 + 8 * relu, wide_stats=True)
    m.input("data", 37, 1, hw)
    m.batchnorm("bn", "data")
    m.scale("sc", "bn", bias=True)
    import tempfile
    from pathlib import Path
    with tempfile.TemporaryDirectory() as d:
        layers = load_model(*m.save(Path(d) / "bn"))
    bn, sc = layers[1], layers[2]
    x = (torch.rand((3, 37, 1, hw), generator=torch.Generator(device="cuda").manual_seed(hw), device="cuda") * 4 - 2)
    beta, alpha = (torch.from_numpy(v).cuda() for v in host_affine32(bn))
    s = sc["s"].cuda() if mul2 else None
    t = sc["t"].cuda() if add2 else None
    got = booster.batchnorm(x, alpha, beta, s, t, relu=relu).double()
    ops = []
    if mul2 or add2:
        ops.append(_copy(sc, s=sc["s"] if mul2 else torch.ones_like(sc["s"]), t=sc["t"] if add2 else None))
    if relu:
        ops.append({"type": "ReLU", "name": "r"})
    ch = Chain(_copy(bn, bottoms=["x"]), ["out"], ops)
    [(_, used, rel, kind, path)] = check_chain(ch, {"x": x.double()}, {"out": got}, FP32_SPLIT)
    _record(kind, path, FP32_SPLIT, rel, used)
    assert used <= 1.0
    if not mul2 and not relu:  # fcuda_scale_forward, with add2 as its bias or without bias
        got = booster.scale(x, sc["s"].cuda(), t).double()
        ch = Chain(_copy(sc, bottoms=["x"], t=sc["t"] if add2 else None), ["out"])
        [(_, used, rel, kind, path)] = check_chain(ch, {"x": x.double()}, {"out": got}, FP32_SPLIT)
        _record(kind, path, FP32_SPLIT, rel, used)
        assert used <= 1.0


# float offsets of (a, b, out) from 256-byte-aligned allocations: the float4 path needs all three 16-byte aligned
OFFSETS = {"aligned": (0, 0, 0), "all_off4B": (1, 1, 1), "b_off12B": (0, 3, 0), "all_off12B": (3, 3, 3)}


@gpu
@pytest.mark.parametrize("n", [1003, 4096, 4099])
@pytest.mark.parametrize("offsets", list(OFFSETS.values()), ids=list(OFFSETS))
def test_add_relu_and_scale_misaligned(cuda, n, offsets):
    """Eltwise add (+ReLU), ReLU and Dropout scaling with the float4 path plus an n % 4 != 0 tail (aligned) and on
    pointers misaligned to 16 bytes (the scalar path): each output is one fp32 rounding of the float64 result."""
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    g = torch.Generator(device="cuda").manual_seed(n + 7 * sum(offsets))
    oa, ob, oo = offsets
    a = torch.randn(n + 8, generator=g, device="cuda")[oa:oa + n]
    b = torch.randn(n + 8, generator=g, device="cuda")[ob:ob + n]
    out = torch.zeros(n + 8, device="cuda")[oo:oo + n]
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    torch.cuda.synchronize()
    for relu in (False, True):
        assert lib.fcuda_eltwise_add_forward(ptr(out), ptr(a), ptr(b), n, int(relu), None) == 0
        torch.cuda.synchronize()
        want = (a.double() + b.double()).float()
        assert torch.equal(out, want.clamp_min(0) if relu else want), relu
    out2 = torch.zeros(n + 8, device="cuda")[ob:ob + n]  # the scale / ReLU kernel checks in and out only
    for o in (out, out2):
        assert lib.fcuda_relu_forward(ptr(o), ptr(a), n, None) == 0
        torch.cuda.synchronize()
        assert torch.equal(o, a.clamp_min(0))
        scale = np.float32(0.3)
        assert lib.fcuda_dropout_forward(ptr(o), ptr(a), n, float(scale), None) == 0
        torch.cuda.synchronize()
        assert torch.equal(o, (a.double() * float(scale)).float())


@gpu
@pytest.mark.parametrize("axis", [0, 1, 2], ids=["channels", "height", "width"])
def test_concat_three_odd_bottoms(cuda, axis):
    """ConcatLayer::Forward's copies (fcuda_copy_channels, [outer][mid][inner]) for three bottoms of 3, 5 and 7 along
    the axis at batch 3: the destination offset of each bottom must be the sum of the earlier ones.  Exact."""
    from feathercnn_b200._lib import fcuda
    g = torch.Generator(device="cuda").manual_seed(axis)
    n, c, h, w = 3, 4, 5, 6
    sizes = [3, 5, 7]
    shapes = [[n, c, h, w] for _ in sizes]
    for sh, k in zip(shapes, sizes):
        sh[1 + axis] = k
    bottoms = [torch.randn(sh, generator=g, device="cuda") for sh in shapes]
    want = torch.cat(bottoms, 1 + axis)
    out = torch.full_like(want, float("nan"))
    offset = 0
    torch.cuda.synchronize()
    for bt in bottoms:
        outer = int(np.prod(bt.shape[:1 + axis]))
        inner = int(np.prod(want.shape[2 + axis:]))
        mid = bt.shape[1 + axis]
        assert fcuda().fcuda_copy_channels(ctypes.c_void_p(out.data_ptr()), want.shape[1 + axis], offset,
                                           ctypes.c_void_p(bt.data_ptr()), mid, inner, outer, None) == 0
        offset += mid
    torch.cuda.synchronize()
    assert torch.equal(out, want)
