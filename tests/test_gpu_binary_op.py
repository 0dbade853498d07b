"""ncnn's BinaryOp on the GPU.

  - Ops 0-5, 7 and 8 (ADD, SUB, MUL, DIV, MAX, MIN, RSUB, RDIV) bit for bit against NumPy float32, with and without the
    ReLU, in every operand form: same shape, the layer's scalar, a one-element operand, per channel, a row, a column and
    both sides broadcast, with the broadcast operand on either side.  Inputs carry -0.0, +-Inf and NaN on both sides;
    odd and float4 widths, unaligned pointers, in place, and more than 65535 (n, c) planes.
  - Ops 6 and 9-11 (POW, RPOW, ATAN2, RATAN2) within the CUDA C Programming Guide's ulp bounds for powf (4) and atan2f
    (3) against float64.
  - The same bits eager and in a CUDA graph.
  - modelgen's "binaryop" layout of each model against its Eltwise twin through feather::Net at batch 2, with fusion and
    CUDA graphs on and off: the same launches per forward and every surviving blob bit-identical.
  - A convolution whose only-read output is added to a per-channel (C, 1, 1) blob from a global pooling (+ReLU): fusion
    on equals fusion off bit for bit, with the broadcast add after the convolution; fed a 1 x 1 image the shapes
    coincide and the epilogue takes the addend; then a larger image again.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_gpu_faster_rcnn import SETTINGS, _all

gpu = pytest.mark.gpu
F = np.float32
EXACT_OPS = [0, 1, 2, 3, 4, 5, 7, 8]


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _same_or_nan(a, b):
    """Bit-identical where a number; NaN in the same places (NumPy keeps payloads the GPU replaces)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int32), b[~nb].view(np.int32))


def _max0(a, b, take_max):
    """fmaxf / fminf: a NaN operand yields the other; -0.0 < +0.0."""
    r = np.fmax(a, b) if take_max else np.fmin(a, b)
    zeros = (a == 0) & (b == 0)
    pos = ~np.signbit(a) | ~np.signbit(b) if take_max else ~np.signbit(a) & ~np.signbit(b)
    return np.where(zeros, np.where(pos, F(0.0), F(-0.0)), r).astype(F)


def binary_ref(a, b, op, relu=False):
    """include/fcuda.h FcudaBinaryOp in NumPy float32 (ops 0-5, 7, 8)."""
    a, b = np.asarray(a, F), np.asarray(b, F)
    with np.errstate(all="ignore"):
        r = {0: lambda: a + b, 1: lambda: a - b, 2: lambda: a * b, 3: lambda: a / b, 4: lambda: _max0(a, b, True),
             5: lambda: _max0(a, b, False), 7: lambda: b - a, 8: lambda: b / a}[op]()
    r = np.asarray(r, F)
    if relu:
        r = np.where(r > 0, r, F(0)).astype(F)  # the Eltwise ReLU: fmaxf(r, 0), NaN becomes 0
    return r


SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, 3e-39], np.float32)


def _operand(rng, shape):
    x = rng.standard_normal(shape).astype(F)
    flat = x.reshape(-1)
    k = min(flat.size, 2 * len(SPECIALS))
    idx = rng.choice(flat.size, k, replace=False)
    flat[idx] = np.resize(SPECIALS, k)
    return x


# (a shape, b shape) per image: b broadcasts, then the same pair with a broadcasting
FORMS = {"same": ((3, 5, 7), (3, 5, 7)), "one-element": ((3, 5, 7), (1, 1, 1)), "channel": ((3, 5, 7), (3, 1, 1)),
         "row": ((3, 5, 7), (1, 1, 7)), "column": ((3, 5, 7), (1, 5, 1)), "both": ((3, 1, 8), (1, 5, 1)),
         "plane": ((3, 5, 8), (1, 5, 8)), "channel-w8": ((4, 3, 8), (4, 1, 1))}


def _run(a, b, op, relu=False, out=None):
    from feathercnn_b200 import booster
    return booster.binary_op(a, b, op, relu, out)


@gpu
@pytest.mark.parametrize("op", EXACT_OPS)
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("swap", [False, True], ids=["b-broadcast", "a-broadcast"])
def test_ops_bit_exact(cuda, op, form, swap):
    rng = np.random.default_rng(op * 100 + len(form) + swap)
    sa, sb = FORMS[form]
    if swap:
        sa, sb = sb, sa
    a, b = _operand(rng, (2,) + sa), _operand(rng, (2,) + sb)
    for relu in (False, True):
        got = _run(_t(a), _t(b), op, relu).cpu().numpy()
        assert _same_or_nan(got, binary_ref(a, b, op, relu)), (op, form, swap, relu)


@gpu
@pytest.mark.parametrize("op", EXACT_OPS)
@pytest.mark.parametrize("w", [7, 8])
def test_scalar_bit_exact(cuda, op, w):
    rng = np.random.default_rng(op + w)
    a = _operand(rng, (2, 3, 5, w))
    for s in (0.5, -0.0, float("inf"), float("nan"), -3.25):
        for relu in (False, True):
            got = _run(_t(a), s, op, relu).cpu().numpy()
            assert _same_or_nan(got, binary_ref(a, np.full_like(a, s), op, relu)), (op, s, relu)


@gpu
@pytest.mark.parametrize("op", [0, 3, 4, 8])
@pytest.mark.parametrize("form", ["same", "channel", "row", "both"])
def test_unaligned_pointers(cuda, op, form):
    """Each tensor one float past a 16-byte boundary: the scalar paths."""
    rng = np.random.default_rng(7)
    sa, sb = FORMS[form]
    a, b = _operand(rng, (2,) + sa), _operand(rng, (2,) + sb)
    want = binary_ref(a, b, op)
    ga, gb = torch.empty(a.size + 1, device="cuda"), torch.empty(b.size + 1, device="cuda")
    ga[1:].copy_(_t(a).reshape(-1))
    gb[1:].copy_(_t(b).reshape(-1))
    out = torch.empty(want.size + 1, device="cuda")
    got = _run(ga[1:].view(a.shape), gb[1:].view(b.shape), op, out=out[1:].view(want.shape))
    assert _same_or_nan(got.cpu().numpy(), want)


@gpu
@pytest.mark.parametrize("op", [0, 1, 8])
@pytest.mark.parametrize("form", ["same", "channel", "row", "one-element"])
def test_in_place(cuda, op, form):
    rng = np.random.default_rng(11)
    sa, sb = FORMS[form]
    a, b = _operand(rng, (2,) + sa), _operand(rng, (2,) + sb)
    ga = _t(a)
    got = _run(ga, _t(b), op, out=ga)
    assert got.data_ptr() == ga.data_ptr() and _same_or_nan(ga.cpu().numpy(), binary_ref(a, b, op))


@gpu
@pytest.mark.parametrize("b_shape", [(1, 70001, 1, 1), (1, 1, 1, 3), (1, 70001, 1, 3)], ids=["channel", "row", "same"])
def test_more_planes_than_grid_rows(cuda, b_shape):
    rng = np.random.default_rng(3)
    a, b = _operand(rng, (1, 70001, 1, 3)), _operand(rng, b_shape)
    for op in (2, 7):
        assert _same_or_nan(_run(_t(a), _t(b), op).cpu().numpy(), binary_ref(a, b, op))


def _ulps(got, ref64):
    """|got - the correctly rounded float32 of ref64| in units of the last place (float32 bit patterns as ordered ints)."""
    def ordered(x):
        i = np.ascontiguousarray(x, F).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(got) - ordered(ref64.astype(F)))


@gpu
@pytest.mark.parametrize("op, bound", [(6, 4), (9, 4), (10, 3), (11, 3)], ids=["POW", "RPOW", "ATAN2", "RATAN2"])
@pytest.mark.parametrize("form", ["same", "channel", "row"])
def test_transcendental_ulp_bounds(cuda, op, bound, form):
    rng = np.random.default_rng(op)
    sa, sb = FORMS[form]
    if op in (6, 9):  # base and exponent
        base, expo = rng.uniform(0.05, 4.0, (2,) + sa).astype(F), rng.uniform(-4, 4, (2,) + sb).astype(F)
        a, b = (base, expo) if op == 6 else (expo, base)   # RPOW: powf(b, a)
        ref = np.power(base.astype(np.float64), expo.astype(np.float64))
    else:
        a, b = rng.standard_normal((2,) + sa).astype(F), rng.standard_normal((2,) + sb).astype(F)
        y, x = (a, b) if op == 10 else (b, a)
        ref = np.arctan2(y.astype(np.float64), x.astype(np.float64))
    got = _run(_t(a), _t(b), op).cpu().numpy()
    ref = np.broadcast_to(ref, got.shape)
    assert np.isfinite(got).all()
    assert _ulps(got, ref).max() <= bound, (op, form, _ulps(got, ref).max())


@gpu
def test_pow_specials_follow_c99(cuda):
    """powf's special cases (C99 Annex F): x^0 = 1 for any x, 1^y = 1 for any y, a negative base with an integral
    exponent, and a NaN from a negative base with a fractional one."""
    a = np.array([np.nan, 2.0, -2.0, -2.0, 1.0, 0.0, -8.0], F).reshape(1, 1, 1, 7)
    b = np.array([0.0, 0.5, 3.0, 0.5, np.nan, 2.0, 2.0], F).reshape(1, 1, 1, 7)
    got = _run(_t(a), _t(b), 6).cpu().numpy().reshape(-1)
    assert got[0] == 1 and got[2] == -8 and np.isnan(got[3]) and got[4] == 1 and got[5] == 0 and got[6] == 64
    assert abs(got[1] - np.sqrt(2.0)) <= 4 * np.spacing(F(np.sqrt(2.0)))


@gpu
@pytest.mark.parametrize("form", ["same", "channel", "both"])
def test_graph_equals_eager(cuda, form):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(5)
    sa, sb = FORMS[form]
    a, b = _t(_operand(rng, (2,) + sa)), _t(_operand(rng, (2,) + sb))
    ref = _run(a, b, 3, True).cpu().numpy()
    out = torch.empty(ref.shape, device="cuda")
    booster.binary_op(a, b, 3, True, out)                     # warm up outside the capture
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    out.zero_()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        booster.binary_op(a, b, 3, True, out)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.int32), ref.view(np.int32))


# ---- models: the "binaryop" layout against its Eltwise twin -----------------------------------------------------------
MODELS = {"style_tiny": ("style_tiny", {}), "sr_tiny": ("sr_tiny", {}),
          "srvgg_small": ("srvgg_compact", dict(num_conv=3, num_feat=16, height=20, width=28)),
          "edsr_x3_small": ("edsr_baseline", dict(scale=3, n_resblocks=2, n_feats=16, height=12, width=10)),
          "resnet50": ("resnet50", {}), "mobilenet_v2": ("mobilenet_v2", {})}


def _net(param, binf, x, fusion, graph):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    for _ in range(3 if graph else 1):
        net.Forward(x)
    net.Synchronize()
    return net


@gpu
@pytest.mark.parametrize("key", list(MODELS))
def test_model_twins(cuda, tmp_path, key):
    from feathercnn_b200.tools import modelgen
    name, kw = MODELS[key]
    files = {adds: modelgen.ZOO[name](adds=adds, **kw).save(tmp_path / adds) for adds in ("eltwise", "binaryop")}
    m = modelgen.ZOO[name](**kw)
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(2)])
    for fusion, graph in SETTINGS:
        nets = {adds: _net(*files[adds], x, fusion, graph) for adds in files}
        e, b = nets["eltwise"], nets["binaryop"]
        assert e.launches_per_forward == b.launches_per_forward > 0, (fusion, graph)
        names = e.BlobNames()
        assert names == b.BlobNames()
        for n in names:
            ge, gb = _all(e, n).float().cpu().numpy(), _all(b, n).float().cpu().numpy()
            assert np.array_equal(ge.view(np.int32), gb.view(np.int32)), (key, fusion, graph, n)
        del nets, e, b


# ---- a residual that broadcasts -------------------------------------------------------------------------------------
def _pool_residual_net(tmp_path, relu):
    """conv1 -> split; global average pooling of one branch to (16, 1, 1); conv2 of the other, its only reader the
    BinaryOp ADD of the pooled blob (+ReLU).  The pooling runs before conv2, so fusion gives conv2 the addend."""
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter(3)
    x = m.conv("conv1", m.input("data", 8, 12, 10), 16, 3, 1, 1)
    x1, x2 = m.split("split", x, ["x1", "x2"])
    p = m.pool("gap", x2, 1, global_pooling=True)
    y = m.conv("conv2", x1, 16, 3, 1, 1)
    s = m.binary_op("sum", [y, p], 0)
    if relu:
        m.relu("relu", s)
    return m.save(tmp_path / ("pool_residual_relu" if relu else "pool_residual")), "relu" if relu else "sum"


@gpu
@pytest.mark.parametrize("relu", [False, True])
def test_broadcast_residual_fusion_on_equals_off(cuda, tmp_path, relu):
    (param, binf), out = _pool_residual_net(tmp_path, relu)
    rng = np.random.default_rng(9)
    nets = {f: _net(param, binf, rng.standard_normal((2, 8, 12, 10)).astype(F), f, False) for f in (True, False)}
    assert nets[True].LayerFusedAway("sum") == 1 and nets[False].LayerFusedAway("sum") == 0
    for h, w in ((12, 10), (1, 1), (7, 9)):   # broadcast add, then equal shapes (the epilogue), then broadcast again
        x = np.random.default_rng(h * w).standard_normal((2, 8, h, w)).astype(F)
        got = {}
        for f, net in nets.items():
            net.Forward(x)
            net.Synchronize()
            assert net.BlobShape(out) == (2, 16, h, w)
            got[f] = net.Extract(out)
        assert np.array_equal(got[True].view(np.int32), got[False].view(np.int32)), (h, w)
        conv2 = _all(nets[False], "conv2").float().cpu().numpy()
        gap = _all(nets[False], "gap").float().cpu().numpy()
        want = binary_ref(conv2, gap, 0, relu)
        assert np.array_equal(got[False].view(np.int32), want.view(np.int32))


@gpu
def test_broadcast_residual_on_the_convolution_side_is_a_topology_error(cuda, tmp_path):
    """With fusion the addend may not be the larger side: conv2's output (16, 1, 1) plus a (16, h, w) blob would need
    a new output, which the convolution does not own.  Reshape fails; without fusion the BinaryOp serves it."""
    from feathercnn_b200.net import FeatherError
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter(4)
    x = m.conv("conv1", m.input("data", 8, 6, 6), 16, 3, 1, 1)
    x1, x2 = m.split("split", x, ["x1", "x2"])
    y = m.conv("conv2", m.pool("gap", x1, 1, global_pooling=True), 16, 1, 1, 0)
    m.binary_op("sum", [y, x2], 0)
    param, binf = m.save(tmp_path / "conv_side")
    x = np.random.default_rng(1).standard_normal((2, 8, 6, 6)).astype(F)
    plain = _net(param, binf, x, False, False)
    assert plain.BlobShape("sum") == (2, 16, 6, 6)
    with pytest.raises(FeatherError):
        _net(param, binf, x, True, False)
