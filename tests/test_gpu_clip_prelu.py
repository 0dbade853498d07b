"""Clip (ReLU6) and PReLU on the GPU.

  - The standalone kernels bit for bit against NumPy's float32 definitions (np.minimum(np.maximum(x, lo), hi), NaN -> lo;
    np.where(x < 0, x * s, x)).
  - The clamp in every convolution epilogue: fcuda_conv_forward_clip equals min(max(fcuda_conv_forward with
    FCUDA_ACT_NONE, lo), hi) bit for bit, on every algorithm and kernel (the arithmetic before the epilogue is the same),
    with the implicit-GEMM tile queries asserting that each geometry lands on the kernel it is meant for.
  - MobileNet-v2 and a PReLU model through feather::Net, every surviving layer against a float64 restatement of its chain
    (from the Net's own bottom blobs, so errors do not add up over depth) within a per-element bound, with fusion and CUDA
    graphs on and off; and an image's output is the same alone and in a batch.

The per-element bound of a convolution chain is CONV_REL * S, S = conv(|x|, |w m|) + |b m| + A (+ |residual|), with m, A
the folded BatchNorm / Scale multipliers and the absolute terms of their offsets (test_gpu_net_bounds.affine_of).
CONV_REL = 2^-13 covers the fp32-split BF16x3 contraction (dropped terms <= 3 * 2^-16 of each product) and the host's
float32 folding; a clamp is 1-Lipschitz, so the bound carries through it.  Element-wise layers are one rounding
(U |ref|) or exact.
"""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_net_bounds import affine_of, fetch, rebuild_chains

gpu = pytest.mark.gpu
U = 2.0 ** -23
CONV_REL = 2.0 ** -13


def _bits_equal(a: np.ndarray, b: np.ndarray) -> bool:
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a, np.float32).view(np.int32),
                                                 np.ascontiguousarray(b, np.float32).view(np.int32))


def _clamp_np(x, lo, hi):
    """fminf(fmaxf(x, lo), hi): np.fmax / np.fmin, which (unlike np.maximum) return the non-NaN operand, so NaN -> lo."""
    return np.fmin(np.fmax(x, np.float32(lo)), np.float32(hi)).astype(np.float32)


def _same_clamped(a: np.ndarray, b: np.ndarray) -> bool:
    """Bit-identical, except that a zero may carry either sign (fmaxf(-0, +0) may return either zero)."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.int32) == b.view(np.int32)) | ((a == 0) & (b == 0))))


def _prelu_np(x, s):
    s = np.asarray(s, np.float32)
    s = s.reshape(1, -1, *([1] * (x.ndim - 2))) if s.size > 1 else s.reshape(())
    return np.where(x < 0, x * s, x).astype(np.float32)


# ---- standalone kernels -----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 4096, 65536 + 7])
@pytest.mark.parametrize("offset", [0, 1])  # offset 1: not 16-byte aligned (scalar path)
@pytest.mark.parametrize("inplace", [False, True])
def test_clip_kernel_bit_exact(cuda, n, offset, inplace):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(n + offset)
    x = rng.uniform(-10, 10, n + offset).astype(np.float32)
    specials = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 6.0, -1.0, 6.5], np.float32)
    x[offset:offset + min(len(specials), n)] = specials[:n]
    for lo, hi in ((0.0, 6.0), (-1.5, 2.25), (3.0, 3.0), (-np.float32(3.4e38), np.float32(3.4e38))):
        d = torch.from_numpy(x).cuda()
        src = d[offset:]
        out = src if inplace else torch.empty_like(src)
        booster.clip(src, lo, hi, out=out)
        torch.cuda.synchronize()
        want = _clamp_np(x[offset:], lo, hi)
        assert _same_clamped(out.cpu().numpy(), want), (n, offset, lo, hi)
        if n >= 1:  # NaN maps to min
            assert out.cpu().numpy()[0] == np.float32(lo)


@gpu
@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (2, 3, 5, 7), (3, 16, 8, 8), (1, 32, 15, 15), (4, 8, 28, 28), (2, 5, 1, 4)])
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("inplace", [False, True])
def test_prelu_kernel_bit_exact(cuda, shape, shared, inplace):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(sum(shape))
    x = rng.standard_normal(shape).astype(np.float32)
    x.flat[0] = -0.0
    s = rng.uniform(-0.5, 0.5, 1 if shared else shape[1]).astype(np.float32)
    d = torch.from_numpy(x).cuda()
    out = d if inplace else torch.empty_like(d)
    booster.prelu(d, torch.from_numpy(s).cuda(), out=out)
    torch.cuda.synchronize()
    assert _bits_equal(out.cpu().numpy(), _prelu_np(x, s)), (shape, shared, inplace)


@gpu
def test_prelu_rejects_slope_count(cuda):
    from feathercnn_b200 import booster
    x = torch.zeros((1, 4, 2, 2), device="cuda")
    with pytest.raises(booster.FcudaError) as e:
        booster.prelu(x, torch.zeros(3, device="cuda"))
    assert e.value.code == -200


# ---- the clamp in every convolution path ------------------------------------------------------------------------------
# (name, (oc, ic, h, w, k, stride, pad, group), algo, precision, dw_vec, expected tile kernel)
P = dict(fp32split=2, tf32x3=0, tf32=1)
CONV_CASES = [
    ("naive", (16, 16, 12, 12, 3, 1, 1, 1), "NAIVE", "fp32split", 1, None),
    ("im2col", (24, 16, 12, 12, 3, 2, 1, 1), "IM2COL", "fp32split", 1, None),
    ("im2col-tf32", (24, 16, 12, 12, 3, 1, 1, 1), "IM2COL", "tf32", 1, None),
    ("winograd63", (32, 32, 20, 20, 3, 1, 1, 1), "WINOGRADF63", "fp32split", 1, None),
    ("winograd23", (32, 32, 20, 20, 3, 1, 1, 1), "WINOGRADF23", "fp32split", 1, None),
    ("winograd63-tf32x3", (32, 32, 20, 20, 3, 1, 1, 1), "WINOGRADF63", "tf32x3", 1, None),
    ("sgeconv-arith-s2", (40, 64, 14, 14, 3, 2, 1, 1), "SGECONV", "fp32split", 1, "gather"),
    ("sgeconv-ktable", (24, 3, 17, 17, 3, 1, 1, 1), "SGECONV", "fp32split", 1, "gather"),
    ("sgeconv-1x1", (48, 32, 9, 9, 1, 1, 0, 1), "SGECONV", "fp32split", 1, None),
    ("sgeconv-grouped", (32, 64, 10, 10, 3, 1, 1, 2), "SGECONV", "fp32split", 1, None),
    ("halo-tf32x3", (40, 64, 16, 16, 3, 1, 1, 1), "SGECONV", "tf32x3", 1, "halo"),
    ("halo-tf32", (64, 32, 16, 16, 3, 1, 1, 1), "SGECONV", "tf32", 1, "halo"),
    ("presplit", (32, 64, 16, 16, 3, 1, 1, 1), "SGECONV", "fp32split", 1, "presplit"),
    ("presplit-ragged", (24, 32, 12, 20, 3, 1, 1, 1), "SGECONV", "fp32split", 1, "presplit"),
    ("wide-64", (64, 64, 56, 56, 3, 1, 1, 1), "SGECONV", "fp32split", 1, "wide"),
    ("wide-128", (128, 64, 28, 28, 3, 1, 1, 1), "SGECONV", "fp32split", 1, "wide"),
    ("dw-vec4", (32, 32, 112, 112, 3, 1, 1, 32), "DEPTHWISE", "fp32split", 1, None),
    ("dw-vec2", (32, 32, 56, 56, 3, 1, 1, 32), "DEPTHWISE", "fp32split", 1, None),
    ("dw-vec2-s2", (32, 32, 112, 112, 3, 2, 1, 32), "DEPTHWISE", "fp32split", 1, None),
    ("dw-shuffle", (32, 32, 56, 56, 3, 1, 1, 32), "DEPTHWISE", "fp32split", 0, None),
    ("dw-shuffle-s2", (32, 32, 112, 112, 3, 2, 1, 32), "DEPTHWISE", "fp32split", 0, None),
    ("dw-cols8", (32, 32, 7, 7, 3, 1, 1, 32), "DEPTHWISE", "fp32split", 1, None),
    ("dw-cols16", (32, 32, 14, 14, 3, 1, 1, 32), "DEPTHWISE", "fp32split", 1, None),
    ("dw-plane", (32, 32, 14, 14, 3, 1, 1, 32), "DEPTHWISE", "fp32split", 0, None),
    ("dw-plane-s2", (32, 32, 14, 14, 3, 2, 1, 32), "DEPTHWISE", "fp32split", 1, None),
    ("dw-generic", (16, 16, 20, 20, 5, 1, 2, 16), "DEPTHWISE", "fp32split", 1, None),
]


def _tiles(p):
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    g = (ctypes.c_int * 4)()
    return {"halo": lib.fcuda_igemm_halo_tile(ctypes.byref(p), g), "presplit": lib.fcuda_igemm_presplit_tile(ctypes.byref(p), g),
            "wide": lib.fcuda_igemm_wide_tile(ctypes.byref(p), g)}


@gpu
@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_clip_equals_clamped_plain_conv(cuda, case):
    from feathercnn_b200 import booster
    name, (oc, ic, h, w, k, s, pad, group), algo_name, prec, dw_vec, tile = case
    algo = getattr(booster, algo_name)
    booster.set_precision(P[prec])
    lib = booster.fcuda()
    old_vec = lib.fcuda_get_tuning(b"dw_vec")
    assert lib.fcuda_set_tuning(b"dw_vec", dw_vec) == 0
    try:
        pn = booster.ConvParam.make(oc, ic, h, w, k, stride=s, pad=pad, group=group, bias=True)
        pc = booster.ConvParam.make(oc, ic, h, w, k, stride=s, pad=pad, group=group, bias=True)
        pc.activation = booster.ACT_CLIP
        if tile is not None:
            t = _tiles(pn)
            if tile == "gather":
                assert t == {"halo": 0, "presplit": 0, "wide": 0}, (name, t)
            elif tile == "halo":
                assert t["halo"] == 1 and t["presplit"] == 0, (name, t)
            elif tile == "presplit":
                assert t["presplit"] == 1 and t["wide"] == 0, (name, t)
            else:
                assert t["wide"] == 1, (name, t)
        rng = np.random.default_rng(oc * 131 + ic)
        x = torch.from_numpy(rng.uniform(-1, 1, (2, ic, h, w)).astype(np.float32)).cuda()
        wshape = (ic, 1, k, k) if group == ic and group > 1 and oc == ic else (oc, ic // group, k, k)
        wt = torch.from_numpy((rng.standard_normal(wshape) / np.sqrt(np.prod(wshape[1:]))).astype(np.float32)).cuda()
        b = torch.from_numpy(rng.uniform(-0.2, 0.2, oc).astype(np.float32)).cuda()
        plain, a0 = booster.conv_forward(pn, x, wt, b, algo=algo)
        for lo, hi in ((0.0, 6.0), (-0.3, 0.25), (0.1, 0.1)):
            clipped, a1 = booster.conv_forward(pc, x, wt, b, algo=algo, clip=(lo, hi))
            torch.cuda.synchronize()
            assert a0 == a1 == algo
            assert _bits_equal(clipped.cpu().numpy(), _clamp_np(plain.cpu().numpy(), lo, hi)), (name, lo, hi)
        # the ReLU epilogue is the clamp with [0, +inf]: bit-identical to max(plain, 0)
        pr = booster.ConvParam.make(oc, ic, h, w, k, stride=s, pad=pad, group=group, bias=True, relu=True)
        relu, _ = booster.conv_forward(pr, x, wt, b, algo=algo)
        torch.cuda.synchronize()
        assert _bits_equal(relu.cpu().numpy(), np.maximum(plain.cpu().numpy(), np.float32(0))), name
    finally:
        lib.fcuda_set_tuning(b"dw_vec", old_vec)


@gpu
def test_conv_clip_rejections(cuda):
    from feathercnn_b200 import booster
    p = booster.ConvParam.make(8, 8, 8, 8, 3, pad=1)
    x = torch.zeros((1, 8, 8, 8), device="cuda")
    w = torch.zeros((8, 8, 3, 3), device="cuda")
    with pytest.raises(booster.FcudaError) as e:  # activation is not Clip
        booster.conv_forward(p, x, w, None, algo=booster.SGECONV, clip=(0.0, 6.0))
    assert e.value.code == -200
    p.activation = booster.ACT_CLIP
    with pytest.raises(booster.FcudaError) as e:  # min > max
        booster.conv_forward(p, x, w, None, algo=booster.SGECONV, clip=(1.0, 0.0))
    assert e.value.code == -200
    for kw in (dict(), dict(pool=True)):  # the entry points without bounds
        with pytest.raises(booster.FcudaError) as e:
            booster.conv_forward(p, x, w, None, algo=booster.WINOGRADF63, **kw)
        assert e.value.code == -200


# ---- feather::Net ----------------------------------------------------------------------------------------------------
def load_model_ext(param, binf) -> list[dict]:
    """test_gpu_net_bounds.load_model plus PReLU slopes (raw fp32 in file order)."""
    from oracle import oracle as O
    layers = O.parse_param(param)
    mb = O._BinReader(binf)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))  # noqa: E731
    for L in layers:
        pd, typ = L["params"], L["type"]
        if typ in ("Convolution", "ConvolutionDepthWise"):
            kw = pd.get(1, 0)
            kh = pd.get(11, kw)
            num, size = pd.get(0, 0), pd.get(6, 0)
            L["w"] = t(mb.load(size, 0).reshape(num, size // (num * kh * kw), kh, kw))
            L["b"] = t(mb.load(num, 1)) if pd.get(5, 0) else None
        elif typ == "BatchNorm":
            L["bn"] = [t(mb.load(pd.get(0, 0), 1)) for _ in range(4)]
        elif typ == "Scale":
            c = pd.get(0, 0)
            L["s"] = t(mb.load(c, 1))
            L["t"] = t(mb.load(c, 1)) if pd.get(1, 0) else None
        elif typ == "PReLU":
            L["slope"] = t(mb.load(pd.get(0, 0), 1))
        else:
            assert typ in ("Input", "Split", "Eltwise", "Clip", "Pooling", "Softmax"), typ
    return layers


def _apply(L, y, S):
    """One single-input layer on (value, bound scale) in float64."""
    typ = L["type"]
    if typ in ("BatchNorm", "Scale"):
        m, a, A = (v.to(y.device).view(1, -1, 1, 1) for v in affine_of(L))
        return m * y + a, m.abs() * S + A, 0
    if typ == "Clip":
        lo, hi = float(L["params"].get(0, -3.4e38)), float(L["params"].get(1, 3.4e38))
        return y.clamp(np.float32(lo), np.float32(hi)), S, 0
    if typ == "PReLU":
        s = L["slope"].double().to(y.device)
        s = s.view(1, -1, 1, 1) if s.numel() > 1 else s.view(())
        return torch.where(y < 0, y * s, y), S * s.abs().clamp(min=1.0), 1
    raise AssertionError(typ)


def restate(ch, ins):
    """(value, per-element bound) of a chain in float64 from its bottoms `ins`."""
    L = ch.head
    typ = L["type"]
    if typ in ("Convolution", "ConvolutionDepthWise"):
        pd = L["params"]
        k = pd.get(1, 0)
        s, pad, group = pd.get(3, 1), pd.get(4, 0), pd.get(7, 1)
        x = ins[L["bottoms"][0]]
        w = L["w"].double().to(x.device)
        b = L["b"].double().to(x.device) if L["b"] is not None else None
        y = F.conv2d(x, w, b, stride=s, padding=pad, groups=group)
        S = F.conv2d(x.abs(), w.abs(), b.abs() if b is not None else None, stride=s, padding=pad, groups=group)
        roundings = 0
        for op in ch.ops:
            if op["type"] == "Eltwise":
                r = ins[ch.residual]
                y, S = y + r, S + r.abs()
            else:
                y, S, _ = _apply(op, y, S)
        assert k > 0
        return y, CONV_REL * S + 4 * U * y.abs()
    if typ in ("BatchNorm", "Scale", "Clip", "PReLU"):
        y, S, r = _apply(L, ins[L["bottoms"][0]], ins[L["bottoms"][0]].abs())
        for op in ch.ops:
            y, S, r2 = _apply(op, y, S)
            r += r2
        return y, (4 * U) * S + U * y.abs()
    if typ == "Eltwise":
        a, b = (ins[n] for n in L["bottoms"])
        return a + b, U * (a.abs() + b.abs())
    if typ == "Pooling":
        x = ins[L["bottoms"][0]]
        assert L["params"].get(4, 0) == 1 and L["params"].get(0, 0) == 1  # global average
        y = x.mean(dim=(2, 3), keepdim=True)
        return y, (x.shape[2] * x.shape[3] + 8) * U * x.abs().mean(dim=(2, 3), keepdim=True)
    if typ == "Softmax":
        x = ins[L["bottoms"][0]]
        y = torch.softmax(x.flatten(1), dim=1).view_as(x)
        return y, 64 * U * (1 + x.abs().amax(dim=(1, 2, 3), keepdim=True)) * y + 2.0 ** -126
    if typ == "Split":
        x = ins[L["bottoms"][0]]
        return x, torch.zeros_like(x)
    raise AssertionError(typ)


def _net(param, binf, fusion, graph):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    return net


def check_net(net, layers, idx, fusion):
    names = set(net.BlobNames())
    chains, _ = rebuild_chains(layers, net.LayerFusedAway, names)
    worst = 0.0
    for ch in chains:
        if ch.head["type"] == "Split":
            continue
        ins = {b: fetch(net, b, idx) for b in ch.bottoms}
        want, bound = restate(ch, ins)
        for t in ch.tops:
            got = fetch(net, t, idx)
            ex = ((got - want).abs() / bound.clamp(min=1e-300)).max().item() if bound.numel() else 0.0
            if not torch.isfinite(got).all():
                ex = float("inf")
            worst = max(worst, ex)
            assert ex <= 1.0, (ch.head["name"], [o["name"] for o in ch.ops], fusion, ex)
    return chains, worst


MOBILENET_V2_CASES = [(32, 3, True, True), (32, 3, False, False), (32, 3, True, False), (224, 2, True, True),
                      (224, 2, False, True)]


@gpu
@pytest.mark.parametrize("size, batch, fusion, graph", MOBILENET_V2_CASES,
                         ids=[f"s{c[0]}-b{c[1]}-{'fused' if c[2] else 'plain'}-{'graph' if c[3] else 'eager'}"
                              for c in MOBILENET_V2_CASES])
def test_mobilenet_v2_layers_within_bounds(cuda, model_dir, size, batch, fusion, graph):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.mobilenet_v2(size=size)
    param, binf = mw.save(model_dir / f"mnv2_{size}")
    layers = load_model_ext(param, binf)
    net = _net(param, binf, fusion, graph)
    x = np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(batch)])
    net.Forward(x)
    net.Synchronize()
    chains, worst = check_net(net, layers, list(range(batch)), fusion)
    n_clip = sum(L["type"] == "Clip" for L in layers)
    fused_clips = sum(net.LayerFusedAway(L["name"]) for L in layers if L["type"] == "Clip")
    if fusion:
        # every Clip follows conv -> BN -> Scale: all 35 fold into a convolution epilogue, the 10 shortcuts too
        assert n_clip == 35 and fused_clips == 35
        assert sum(net.LayerFusedAway(L["name"]) for L in layers if L["type"] == "Eltwise") == 10
        assert net.FuseNow() == 52 * 2 + 35 + 10
    else:
        assert fused_clips == 0
    print(f"\nmobilenet_v2 {size} b{batch} fusion={fusion} graph={graph}: {len(chains)} chains, worst bound share {worst:.3f}")


@gpu
def test_mobilenet_v2_image_is_batch_independent(cuda, model_dir):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.mobilenet_v2(size=64)
    param, binf = mw.save(model_dir / "mnv2_64")
    xs = np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(5)])
    net = _net(param, binf, True, True)
    net.Forward(xs)
    batched = net.Extract("prob")
    alone = _net(param, binf, True, True)
    for i in (0, 3):
        alone.Forward(xs[i:i + 1])
        assert _bits_equal(alone.Extract("prob")[0], batched[i]), i


@gpu
@pytest.mark.parametrize("fusion, graph", [(True, True), (False, False)])
def test_prelu_model_within_bounds(cuda, model_dir, fusion, graph):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.prelu_tiny()
    param, binf = mw.save(model_dir / "prelu_tiny")
    layers = load_model_ext(param, binf)
    net = _net(param, binf, fusion, graph)
    x = np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(3)])
    net.Forward(x)
    net.Synchronize()
    check_net(net, layers, [0, 1, 2], fusion)
    # PReLU is never fused; with fusion the BN / Scale before it fold into the convolution
    assert all(net.LayerFusedAway(n) == 0 for n in ("prelu1", "prelu2"))
    assert [net.LayerFusedAway(n) for n in ("bn1", "scale1")] == ([1, 1] if fusion else [0, 0])


@gpu
def test_prelu_slope_count_checked_at_reshape(cuda):
    """PReLULayer::Reshape rejects 3 slopes for 4 channels (FEATHER_ERR_TOPOLOGY); Net::Reshape reports every layer's
    shape failure as FEATHER_ERR_WEIGHTS (-100), like the reference's net.cpp."""
    from feathercnn_b200.net import FeatherError, Net
    net = Net()
    net.LoadParamFromText("7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=4\nPReLU p 1 1 data out 0=3\n")
    net.LoadWeights(_slopes_bin(3))
    with pytest.raises(FeatherError) as e:
        net.Forward(np.zeros((1, 4, 4, 4), np.float32))
    assert e.value.code == -100


def _slopes_bin(n):
    import tempfile
    f = tempfile.NamedTemporaryFile(suffix=".bin", delete=False)
    f.write(np.full(n, 0.25, np.float32).tobytes())
    f.close()
    return f.name
