"""Fast neural style's InstanceNorm and Padding on the host (no kernel is launched): the NumPy definitions the GPU tests
hold the kernels to, checked by hand; a float32 restatement of InstanceNorm's stated summation order against float64
within the per-element bound include/fcuda.h states, and the naive E[x^2] - mean^2 variance breaking that bound on an
offset plane; the C ABI's rejections and workspace size (every call here fails its checks before a launch); the loader's
ids, defaults and rejections; and the blob shapes of modelgen's style models.

pad_ref, instance_norm64 and instance_norm_bound are what tests/test_gpu_style.py holds the kernels to;
tests/test_gpu_memory_bound_sweep.py also holds InstanceNorm to instance_norm32 bit for bit."""
from __future__ import annotations

import ctypes
import math

import numpy as np
import pytest

from test_faster_rcnn_host import FAKE

F = np.float32
U = 2.0 ** -24
CHUNK = 8192


# ---- the definitions ------------------------------------------------------------------------------------------------
def pad_ref(x, top, bottom, left, right, type_, value=0.0, dtype=np.float32):
    """ncnn Padding of the last two axes: type 0 constant, 1 replicate, 2 reflect (edge excluded).  `dtype` float64
    pads a float64 reference without rounding it (the constant `value` is still the float32 the kernel writes)."""
    x = np.asarray(x, dtype)
    width = [(0, 0)] * (x.ndim - 2) + [(top, bottom), (left, right)]
    if type_ == 0:
        return np.pad(x, width, mode="constant", constant_values=dtype(F(value)))
    return np.pad(x, width, mode="edge" if type_ == 1 else "reflect")


def instance_norm64(x, gamma=None, beta=None, eps=1e-5):
    """float64 InstanceNorm of (N, C, H, W) float32 x: (y64, mean, biased variance, a, b) with the plane statistics of
    shape (N, C, 1, 1)."""
    xd = np.asarray(x, np.float64)
    mu = xd.mean(axis=(2, 3), keepdims=True)
    s2 = ((xd - mu) ** 2).mean(axis=(2, 3), keepdims=True)
    c = xd.shape[1]
    g = np.ones((1, c, 1, 1)) if gamma is None else np.asarray(gamma, np.float64).reshape(1, c, 1, 1)
    bt = np.zeros((1, c, 1, 1)) if beta is None else np.asarray(beta, np.float64).reshape(1, c, 1, 1)
    a = g / np.sqrt(s2 + eps)
    return a * (xd - mu) + bt, mu, s2, a, bt


def instance_norm_bound(x, gamma=None, beta=None, eps=1e-5):
    """(y64, per-element bound) of include/fcuda.h's InstanceNorm error bound, before any ReLU or padding."""
    xd = np.asarray(x, np.float64)
    y64, mu, s2, a, bt = instance_norm64(x, gamma, beta, eps)
    S = xd.shape[2] * xd.shape[3]
    K = math.ceil(S / CHUNK)
    D = 64 + math.ceil(K / 32)
    X = np.abs(xd).max(axis=(2, 3), keepdims=True)
    A = np.abs(a)
    dmu = D * U * X
    V = (D + 8) * U * s2 + 4 * D * U * X * np.sqrt(s2) + 6 * D * D * U * U * X * X
    rho = V / (s2 + eps) + 6 * U
    bound = A * (rho * np.abs(xd - mu) + (1 + 2 * rho) * dmu) + U * (np.abs(bt) + (1 + rho) * A * (np.abs(mu) + dmu)
                                                                      + np.abs(y64))
    return y64, bound


def _fmaf(a, b, c):
    """fmaf of float32 operands, correctly rounded: the product is exact in float64 and s = p + c rounds once there, with
    e = (p + c) - s exact (TwoSum).  Rounding s to float32 is right unless s sits exactly halfway between two floats while
    e != 0; then the exact sum lies on e's side of the midpoint.  Bit for bit what the GPU's fmaf gives."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    s = p + c
    t = s - p
    e = (p - (s - t)) + (c - t)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    other = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf))).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        tie = (s != r64) & ((r64 + other.astype(np.float64)) / 2 == s) & (e != 0)
        toward = np.where((e > 0) == (other.astype(np.float64) > r64), other, r)
    return np.where(tie, toward, r).astype(np.float32)


def _block_sum(v):
    """fcuda's fixed-order block sum of 256 thread values: 32-lane xor-shuffle trees, then the warp partials in order."""
    w = v.reshape(8, 32).copy()
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, lanes ^ o]
    r = w[0, 0]
    for k in range(1, 8):
        r = F(r + w[k, 0])
    return F(r)


def _warp_sum(v):
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[lanes ^ o]
    return F(v[0])


def _thread_view(c):
    """A chunk padded to 8192 as (256 threads, 32 elements in each thread's order: j outer, q inner) and its mask."""
    n = len(c)
    buf = np.zeros(CHUNK, np.float32)
    buf[:n] = c
    mask = np.zeros(CHUNK, bool)
    mask[:n] = True
    tv = lambda a: a.reshape(8, 256, 4).transpose(1, 0, 2).reshape(256, 32)
    return tv(buf), tv(mask)


def plane_stats32(x, naive=False):
    """float32 (mean, var) of one plane in the stated order (naive: var = E[x^2] - mean^2 with x^2 summed in the same
    order, the formula the kernel must not use)."""
    x = np.asarray(x, np.float32).ravel()
    S = len(x)
    sums, m2s, ns, sqs = [], [], [], []
    for k in range(0, S, CHUNK):
        c = x[k:k + CHUNK]
        v, mask = _thread_view(c)
        acc = np.zeros(256, np.float32)
        sq = np.zeros(256, np.float32)
        for i in range(32):
            acc = np.where(mask[:, i], acc + v[:, i], acc)
            sq = np.where(mask[:, i], _fmaf(v[:, i], v[:, i], sq), sq)
        s = _block_sum(acc)
        m = F(s / F(len(c)))
        m2 = np.zeros(256, np.float32)
        for i in range(32):
            d = F(1) * (v[:, i] - m)
            m2 = np.where(mask[:, i], _fmaf(d, d, m2), m2)
        sums.append(s), m2s.append(_block_sum(m2)), ns.append(F(len(c))), sqs.append(_block_sum(sq))
    K = len(sums)
    lane = lambda vals: np.array([F(sum_seq(vals[l::32])) for l in range(32)], np.float32)
    mean = F(_warp_sum(lane(sums)) / F(S))
    if naive:
        return mean, F(F(_warp_sum(lane(sqs)) / F(S)) - F(mean * mean))
    terms = [F(_fmaf(F(ns[k] * (d := F(F(sums[k] / ns[k]) - mean))), d, m2s[k])) for k in range(K)]
    return mean, F(_warp_sum(lane(terms)) / F(S))


def sum_seq(vals):
    r = F(0)
    for v in vals:
        r = F(r + v)
    return r


def instance_norm32(x, gamma=None, beta=None, eps=1e-5, naive=False):
    """The float32 restatement of one image batch (N, C, H, W), plane by plane."""
    x = np.asarray(x, np.float32)
    y = np.empty_like(x)
    for n in range(x.shape[0]):
        for c in range(x.shape[1]):
            mean, var = plane_stats32(x[n, c], naive)
            with np.errstate(invalid="ignore"):
                r = np.sqrt(F(var + F(eps)), dtype=np.float32)
            a = F(F(gamma[c]) / r) if gamma is not None else F(F(1) / r)
            b = _fmaf(-mean, a, F(beta[c]) if beta is not None else F(0))
            y[n, c] = _fmaf(x[n, c], a, b)
    return y


def _used(y, y64, bound):
    with np.errstate(invalid="ignore"):
        r = np.abs(np.float64(y) - y64) / bound
    return float(np.nanmax(np.where(np.isnan(r), np.inf, r)))


# ---- the definitions, by hand ---------------------------------------------------------------------------------------
ROW = np.array([[[[1, 2, 3, 4]]]], np.float32)


def test_pad_ref_by_hand():
    assert pad_ref(ROW, 0, 0, 2, 3, 2).ravel().tolist() == [3, 2, 1, 2, 3, 4, 3, 2, 1]
    assert pad_ref(ROW, 0, 0, 2, 3, 1).ravel().tolist() == [1, 1, 1, 2, 3, 4, 4, 4, 4]
    assert pad_ref(ROW, 0, 0, 2, 3, 0, 7.0).ravel().tolist() == [7, 7, 1, 2, 3, 4, 7, 7, 7]
    col = pad_ref(ROW.reshape(1, 1, 4, 1), 3, 1, 0, 0, 2).ravel().tolist()
    assert col == [4, 3, 2, 1, 2, 3, 4, 3]


def test_instance_norm64_by_hand():
    x = np.array([[[[1, 3], [5, 7]]]], np.float32)        # mean 4, biased variance 5
    y, mu, s2, a, b = instance_norm64(x, [2.0], [0.5], eps=0.0)
    assert mu.item() == 4 and s2.item() == 5
    assert np.allclose(y.ravel(), 2 * (np.array([1, 3, 5, 7]) - 4) / math.sqrt(5) + 0.5)


@pytest.mark.parametrize("shape", [(1, 1), (1, 7), (3, 2731), (1, 8192), (1, 3 * 8192 + 1)])
@pytest.mark.parametrize("affine", [False, True])
def test_restatement_within_bound(shape, affine):
    rng = np.random.default_rng(shape[1])
    x = (rng.standard_normal((1, 2) + shape) * 3 + 0.5).astype(np.float32)
    g, b = (rng.uniform(0.5, 1.5, 2), rng.uniform(-1, 1, 2)) if affine else (None, None)
    y64, bound = instance_norm_bound(x, g, b, 1e-5)
    assert _used(instance_norm32(x, g, b, 1e-5), y64, bound) <= 1.0


def test_offset_plane_breaks_the_naive_variance():
    """mean 1e4, std 1: E[x^2] - mean^2 in float32 cancels (x^2 ~ 1e8, its rounding ~ 8), so the naive variance is
    off by far more than the bound allows (or negative); the stated order meets the bound."""
    rng = np.random.default_rng(3)
    x = (1e4 + rng.standard_normal((1, 1, 64, 200))).astype(np.float32)
    y64, bound = instance_norm_bound(x, eps=1e-5)
    assert _used(instance_norm32(x, eps=1e-5), y64, bound) <= 1.0
    assert _used(instance_norm32(x, eps=1e-5, naive=True), y64, bound) > 1.0


def test_constant_plane_within_bound():
    x = np.full((1, 1, 37, 41), 0.1, np.float32)
    y64, bound = instance_norm_bound(x, [2.0], [0.25], 1e-5)
    assert np.all(y64 == 0.25)
    assert _used(instance_norm32(x, [2.0], [0.25], 1e-5), y64, bound) <= 1.0


# ---- C ABI ----------------------------------------------------------------------------------------------------------
def _pad(top=0, bottom=0, left=0, right=0, type_=2, value=0.0):
    from feathercnn_b200._lib import FcudaPad
    return FcudaPad(top, bottom, left, right, type_, value)


OTHER = ctypes.c_void_p(512)
IN_REJECTS = [
    (dict(out=None), -100), (dict(x=None), -100), (dict(ws=None), -100), (dict(gamma=None), -100),
    (dict(beta=None), -100), (dict(c=0), -100), (dict(h=0), -100), (dict(w=0), -100), (dict(n=0), -100),
    (dict(eps=-1e-5), -200), (dict(eps=float("nan")), -200),
    (dict(pad=_pad(top=-1)), -200), (dict(pad=_pad(right=-2)), -200), (dict(pad=_pad(1, 1, 1, 1, 3)), -200),
    (dict(pad=_pad(1, 1, 1, 1, -1)), -200), (dict(pad=_pad(top=8)), -200), (dict(pad=_pad(left=6)), -200),
    (dict(pad=_pad(bottom=8)), -200), (dict(pad=_pad(right=6)), -200), (dict(pad=_pad(1, 1, 1, 1), out=FAKE), -200),
    (dict(h=65536, w=32768), -200), (dict(h=46341, w=46340, pad=_pad(1, 1, 1, 1, 0)), -200),
    (dict(h=4096, w=4097), -200), (dict(h=4096, w=4096, pad=_pad(0, 1, 0, 0, 0)), -200),   # planes over 2^24 floats
]


def _in_call(**kw):
    from feathercnn_b200._lib import fcuda
    a = dict(out=OTHER, x=FAKE, c=4, h=8, w=6, gamma=FAKE, beta=FAKE, eps=1e-5, relu=1, pad=None, ws=FAKE, n=2)
    a.update(kw)
    pad = ctypes.byref(a["pad"]) if a["pad"] is not None else None
    return fcuda().fcuda_instance_norm_forward(a["out"], a["x"], a["c"], a["h"], a["w"], a["gamma"], a["beta"], a["eps"],
                                               a["relu"], pad, a["ws"], a["n"], None)


@pytest.mark.parametrize("kw, code", IN_REJECTS, ids=[str(i) for i in range(len(IN_REJECTS))])
def test_instance_norm_abi_rejects(kw, code):
    assert _in_call(**kw) == code


PAD_REJECTS = [(dict(out=None), -100), (dict(x=None), -100), (dict(pad=None), -100), (dict(c=0), -100),
               (dict(h=0), -100), (dict(w=0), -100), (dict(n=0), -100), (dict(pad=_pad(-1, 0, 0, 0)), -200),
               (dict(pad=_pad(0, 0, 0, 0, 3)), -200), (dict(pad=_pad(8, 0, 0, 0)), -200),
               (dict(pad=_pad(0, 0, 0, 6)), -200), (dict(pad=_pad(1, 0, 0, 0, 0), out=FAKE), -200)]


@pytest.mark.parametrize("kw, code", PAD_REJECTS, ids=[str(i) for i in range(len(PAD_REJECTS))])
def test_padding_abi_rejects(kw, code):
    from feathercnn_b200._lib import fcuda
    a = dict(out=OTHER, x=FAKE, c=4, h=8, w=6, pad=_pad(1, 1, 1, 1), n=2)
    a.update(kw)
    pad = ctypes.byref(a["pad"]) if a["pad"] is not None else None
    assert fcuda().fcuda_padding_forward(a["out"], a["x"], a["c"], a["h"], a["w"], pad, a["n"], None) == code


@pytest.mark.parametrize("c, plane, n", [(1, 1, 1), (3, 8192, 2), (3, 8193, 2), (32, 512 * 512, 8),
                                         (32, 1080 * 1920, 1)])
def test_workspace_size(c, plane, n):
    from feathercnn_b200._lib import fcuda
    floats = ctypes.c_size_t(0)
    assert fcuda().fcuda_instance_norm_workspace_size(c, plane, n, ctypes.byref(floats)) == 0
    assert floats.value == 2 * c * n * math.ceil(plane / 8192)
    for args in ((0, plane, n), (c, 0, n), (c, plane, 0)):
        assert fcuda().fcuda_instance_norm_workspace_size(*args, ctypes.byref(floats)) == -100
    assert fcuda().fcuda_instance_norm_workspace_size(c, plane, n, None) == -100


# ---- loader ---------------------------------------------------------------------------------------------------------
HEAD = "Input d 0 1 d 0=6 1=5 2=4\n"


def _load(line, fusion=False):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion)
    net.LoadParamFromText(f"7767517\n2 2\n{HEAD}{line}\n")
    return net


@pytest.mark.parametrize("line", [
    "Padding p 1 1 d p 0=-1", "Padding p 1 1 d p 3=-1", "Padding p 1 1 d p 4=3", "Padding p 1 1 d p 4=-1",
    "Padding p 1 1 d p 0=1 6=4", "Padding p 1 1 d p 0=1 7=1", "Padding p 1 1 d p 0=1 8=1",
    "InstanceNorm i 1 1 d i", "InstanceNorm i 1 1 d i 0=0", "InstanceNorm i 1 1 d i 0=4 1=-1.0",
])
def test_loader_rejects(line):
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError) as e:
        _load(line)
    assert e.value.code == -200, line


@pytest.mark.parametrize("line", [
    "Padding p 1 1 d p", "Padding p 1 1 d p 0=4 1=4 2=5 3=5 4=2", "Padding p 1 1 d p 0=1 1=2 2=3 3=4 4=0 5=2.5",
    "Padding p 1 1 d p 0=9 4=1 6=0 7=0 8=0", "InstanceNorm i 1 1 d i 0=4", "InstanceNorm i 1 1 d i 0=4 1=1e-5 2=0",
])
def test_loader_accepts(line):
    _load(line)


def test_padding_never_fuses_on_its_own():
    from feathercnn_b200.net import Net
    net = Net(fusion=True)
    net.LoadParamFromText(f"7767517\n3 3\n{HEAD}Padding p 1 1 d p 0=1 4=2\nReLU r 1 1 p r\n")
    assert net.FuseNow() == 0


def test_instance_norm_fuses_relu_then_padding_only():
    """IN absorbs one ReLU, then one Padding, which ends the chain; a Padding first also ends it, and a second ReLU
    after the Padding stays."""
    from feathercnn_b200.net import Net
    for body, fused in (("ReLU r 1 1 i r\nPadding p 1 1 r p 0=1 4=2\nReLU r2 1 1 p r2\n", {"r", "p"}),
                        ("Padding p 1 1 i p 0=1 4=2\nReLU r 1 1 p r\nReLU r2 1 1 r r2\n", {"p"}),
                        ("ReLU r 1 1 i r\nReLU r2 1 1 r r2\nPadding p 1 1 r2 p 0=1\n", {"r"})):
        net = Net(fusion=True)
        net.LoadParamFromText(f"7767517\n5 5\n{HEAD}InstanceNorm i 1 1 d i 0=4\n{body}")
        net.FuseNow()
        names = [L.split()[1] for L in body.strip().split("\n")]
        assert {n for n in names if net.LayerFusedAway(n)} == fused, body


# ---- models ---------------------------------------------------------------------------------------------------------
def _style_layers(m):
    """(type, name, bottoms, params) of every layer line."""
    out = []
    for L in m.lines:
        t = L.split()
        nb, nt = int(t[2]), int(t[3])
        out.append((t[0], t[1], t[4:4 + nb], dict(kv.split("=") for kv in t[4 + nb + nt:])))
    return out


@pytest.mark.parametrize("h, w", [(512, 512), (1080, 1920)])
def test_fast_neural_style_shapes(h, w):
    from feathercnn_b200.tools import modelgen
    m = modelgen.fast_neural_style(height=h, width=w)
    assert m.shape["conv6"] == (3, h, w) and m.shape["conv1_pad"] == (3, h + 8, w + 8)
    assert m.shape["relu3"] == (128, h // 4, w // 4) and m.shape["res5"] == (128, h // 4, w // 4)
    assert m.shape["up4"] == (128, h // 2, w // 2) and m.shape["relu4"] == (64, h // 2, w // 2)
    assert m.shape["relu5"] == (32, h, w) and m.shape["conv6_pad"] == (32, h + 8, w + 8)
    layers = _style_layers(m)
    types = [L[0] for L in layers]
    assert types.count("InstanceNorm") == 15 and types.count("Padding") == 16 and types.count("ReLU") == 10
    assert types.count("Eltwise") == 5 and types.count("Interp") == 2 and types.count("Convolution") == 16
    for L in layers:
        p = L[3]
        if L[0] == "Convolution":
            assert p["4"] == "0" and L[2][0].endswith("_pad"), L
        if L[0] == "Padding":
            assert p["4"] == "2" and len({p["0"], p["1"], p["2"], p["3"]}) == 1, L
        if L[0] == "InstanceNorm":
            assert p["2"] == "1", L
    assert "Interp up4 1 1 res5 up4 0=1 1=2.000000e+00 2=2.000000e+00" in m.lines
    assert "Convolution conv1 1 1 conv1_pad conv1 0=32 1=9 3=1 4=0 5=1 6=7776" in m.lines
    assert "Convolution conv6 1 1 conv6_pad conv6 0=3 1=9 3=1 4=0 5=1 6=7776" in m.lines
    assert "Eltwise res3 2 1 res3_in_a res3_in2 res3 0=1" in m.lines
    assert abs(m.flops / 1e9 - 80.6) < 0.1 if (h, w) == (512, 512) else True
    assert modelgen.ZOO["fast_neural_style"] is modelgen.fast_neural_style
    with pytest.raises(AssertionError):
        modelgen.fast_neural_style(height=514)


def test_style_tiny_shapes_and_weights():
    """style_tiny keeps the layout at 8 / 16 / 16 channels with two residual blocks; every InstanceNorm writes gamma and
    beta (2 x channels raw floats) after its convolution's weights and bias."""
    from feathercnn_b200.tools import modelgen
    m = modelgen.style_tiny()
    assert m.shape["conv6"] == (3, 32, 32) and m.shape["relu3"] == (16, 8, 8) and m.shape["res2"] == (16, 8, 8)
    assert m.shape["relu5"] == (8, 32, 32)
    types = [L[0] for L in _style_layers(m)]
    assert types.count("InstanceNorm") == 9 and types.count("Eltwise") == 2 and types.count("Interp") == 2
    floats = 0
    for L in _style_layers(m):
        p = L[3]
        if L[0] == "Convolution":
            floats += 1 + int(p["6"]) + int(p["0"])           # flag word, weights, bias
        elif L[0] == "InstanceNorm":
            floats += 2 * int(p["0"])
    assert len(m.bin) == 4 * floats
    assert modelgen.ZOO["style_tiny"] is modelgen.style_tiny
