"""Fast neural style's InstanceNorm and Padding on the GPU.

  - InstanceNorm against float64 within include/fcuda.h's per-element bound (test_style_host.instance_norm_bound):
    planes of 1, 7, 8191, 8192, 8193, 3 x 8192 + 1, 270 x 480 and 1080 x 1920 floats, affine 0 and 1, eps 1e-5 and
    1e-3; offset planes (mean 1e4, std 1); a constant plane (variance 0); a NaN that poisons only its own plane.
  - The same bits across batch splits, a one-float pointer offset, in and out of place (unpadded), eager and graph.
  - Padding bit for bit against NumPy for every type, every reflect pad from 0 to dim - 1, odd and unaligned widths.
  - IN + ReLU + Padding in one call equals the three separate calls bit for bit.
  - Reshape rejections: a channel count other than the blob's, a reflect pad >= the plane's dimension.
  - modelgen's style_tiny and fast_neural_style (at 256 x 256), batch 2, with fusion and CUDA graphs on and off: every
    convolution within test_gpu_net_bounds' float64 bounds (the 9 x 9 layers included), InstanceNorm recomputed from the
    net's own blobs within its bound, Padding, ReLU, Interp and Eltwise bit for bit; 8 Paddings and all 10 ReLUs fused away
    in fast_neural_style; the output bit-identical with graphs on and off and with fusion on and off.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_gpu_faster_rcnn import SETTINGS, _all, _bits_equal
from test_gpu_net_bounds import CONV_TYPES, check_chain, rebuild_chains
from test_style_host import instance_norm_bound, pad_ref

gpu = pytest.mark.gpu


def _in(x, gamma=None, beta=None, eps=1e-5, relu=False, pad=None, out=None):
    from feathercnn_b200 import booster
    t = lambda a: a if a is None or torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    xs = x if torch.is_tensor(x) else t(x)
    return booster.instance_norm(xs, t(gamma), t(beta), eps, relu, pad, out)


def _used(got, y64, bound):
    d = np.abs(np.asarray(got, np.float64) - y64)
    return float(np.max(np.where(d == 0, 0.0, d / bound)))


# ---- InstanceNorm against float64 -----------------------------------------------------------------------------------
PLANES = [(1, 1), (1, 7), (1, 8191), (64, 128), (1, 8193), (1, 3 * 8192 + 1), (270, 480), (1080, 1920)]


@gpu
@pytest.mark.parametrize("hw", PLANES, ids=[f"{h}x{w}" for h, w in PLANES])
@pytest.mark.parametrize("affine", [0, 1])
@pytest.mark.parametrize("eps", [1e-5, 1e-3])
def test_instance_norm_within_bound(cuda, hw, affine, eps):
    h, w = hw
    n, c = (1, 2) if h * w > 100000 else (2, 3)
    rng = np.random.default_rng(h * 7 + w)
    x = (rng.standard_normal((n, c, h, w)) * rng.uniform(0.1, 10, (1, c, 1, 1)) + rng.uniform(-3, 3, (1, c, 1, 1)))
    x = x.astype(np.float32)
    g, b = (rng.uniform(0.5, 1.5, c), rng.uniform(-1, 1, c)) if affine else (None, None)
    got = _in(x, g, b, eps).cpu().numpy()
    y64, bound = instance_norm_bound(x, g, b, eps)
    assert _used(got, y64, bound) <= 1.0


@gpu
@pytest.mark.parametrize("hw", [(64, 128), (270, 480)])
def test_offset_planes_within_bound(cuda, hw):
    rng = np.random.default_rng(11)
    x = (np.array([1e4, -1e4, 3e3])[None, :, None, None] + rng.standard_normal((2, 3) + hw)).astype(np.float32)
    got = _in(x, eps=1e-5).cpu().numpy()
    y64, bound = instance_norm_bound(x, eps=1e-5)
    assert _used(got, y64, bound) <= 1.0
    assert np.abs(got).max() < 10                           # still normalised


@gpu
def test_constant_plane(cuda):
    x = np.full((1, 2, 37, 41), 0.1, np.float32)
    x[0, 1] = 3.0
    got = _in(x, [2.0, 1.0], [0.25, -0.5], 1e-5).cpu().numpy()
    y64, bound = instance_norm_bound(x, [2.0, 1.0], [0.25, -0.5], 1e-5)
    assert _used(got, y64, bound) <= 1.0
    assert np.all(got[0, 1] == -0.5)                        # 3.0 sums exactly: x - mean is 0


@gpu
def test_nan_poisons_only_its_plane(cuda):
    rng = np.random.default_rng(2)
    x = rng.standard_normal((2, 3, 40, 300)).astype(np.float32)
    x[1, 2, 17, 123] = np.nan
    got = _in(x).cpu().numpy()
    assert np.all(np.isnan(got[1, 2]))
    ok = np.ones((2, 3), bool)
    ok[1, 2] = False
    y64, bound = instance_norm_bound(np.where(np.isnan(x), 0, x))
    assert _used(got[ok], y64[ok], bound[ok]) <= 1.0
    relu = _in(x, relu=True).cpu().numpy()
    assert np.all(relu[1, 2] == 0)                          # fmaxf(NaN, 0) = 0, as the ReLU kernel


# ---- identical bits -------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("hw", [(270, 480), (7, 9), (64, 128)])
def test_bits_independent_of_split_offset_place_and_graph(cuda, hw):
    rng = np.random.default_rng(4)
    x = (rng.standard_normal((4, 3) + hw) * 2 + 1).astype(np.float32)
    g, b = rng.uniform(0.5, 1.5, 3), rng.uniform(-1, 1, 3)
    ref = _in(x, g, b, relu=True).cpu().numpy()
    for i in range(4):
        assert _bits_equal(_in(x[i:i + 1], g, b, relu=True).cpu().numpy(), ref[i:i + 1])
    flat = torch.zeros(x.size + 1, device="cuda")
    flat[1:] = torch.from_numpy(x.ravel()).cuda()
    shifted = flat[1:].view(x.shape)                        # 4 bytes off 16-byte alignment
    assert _bits_equal(_in(shifted, g, b, relu=True).cpu().numpy(), ref)
    inplace = torch.from_numpy(x).cuda()
    _in(inplace, g, b, relu=True, out=inplace)
    assert _bits_equal(inplace.cpu().numpy(), ref)
    xs, gs, bs = (torch.from_numpy(np.asarray(v, np.float32)).cuda() for v in (x, g, b))
    _in(xs, gs, bs, relu=True)                               # warm up outside the capture
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        out = _in(xs, gs, bs, relu=True)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert _bits_equal(out.cpu().numpy(), ref)


# ---- Padding --------------------------------------------------------------------------------------------------------
def _pad(x, top, bottom, left, right, type_, value=0.0):
    from feathercnn_b200 import booster
    xs = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return booster.padding(xs, top, bottom, left, right, type_, value).cpu().numpy()


@gpu
@pytest.mark.parametrize("hw", [(5, 7), (6, 8), (1, 1), (3, 1), (9, 33)])
def test_padding_every_reflect_pad(cuda, hw):
    h, w = hw
    x = np.random.default_rng(h * w).standard_normal((2, 3, h, w)).astype(np.float32)
    for p in range(max(h, w)):
        for pads in ((min(p, h - 1), 0, 0, min(p, w - 1)), (0, min(p, h - 1), min(p, w - 1), 0)):
            assert _bits_equal(_pad(x, *pads, 2), pad_ref(x, *pads, 2)), (hw, pads)


@gpu
@pytest.mark.parametrize("type_", [0, 1, 2])
@pytest.mark.parametrize("hw, pads", [((16, 16), (4, 4, 4, 4)), ((17, 23), (1, 2, 3, 4)), ((64, 61), (0, 0, 1, 0)),
                                      ((128, 128), (1, 1, 1, 1)), ((7, 13), (0, 0, 0, 0))])
def test_padding_bit_exact(cuda, type_, hw, pads):
    rng = np.random.default_rng(sum(hw))
    x = rng.standard_normal((2, 5) + hw).astype(np.float32)
    x[0, 0, 0, 0] = -0.0
    x[1, 1, -1, -1] = np.nan
    want = pad_ref(x, *pads, type_, -1.5)
    assert _bits_equal(_pad(x, *pads, type_, -1.5), want)
    flat = torch.zeros(x.size + 1, device="cuda")
    flat[1:] = torch.from_numpy(x.ravel()).cuda()
    assert _bits_equal(_pad(flat[1:].view(x.shape), *pads, type_, -1.5), want)     # unaligned input


# ---- fused against unfused ------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("type_", [0, 1, 2])
@pytest.mark.parametrize("hw, pads", [((64, 64), (1, 1, 1, 1)), ((33, 45), (4, 4, 4, 4)), ((270, 480), (1, 2, 0, 3))])
def test_fused_equals_separate_calls(cuda, type_, hw, pads):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((2, 4) + hw) * 2 + 0.3).astype(np.float32)
    g, b = rng.uniform(0.5, 1.5, 4), rng.uniform(-1, 1, 4)
    fused = _in(x, g, b, relu=True, pad=pads + (type_, 0.75)).cpu().numpy()
    y = booster.relu(_in(x, g, b))
    sep = _pad(y.contiguous(), *pads, type_, 0.75)
    assert _bits_equal(fused, sep)
    assert _bits_equal(fused, pad_ref(_in(x, g, b, relu=True).cpu().numpy(), *pads, type_, 0.75))


@gpu
@pytest.mark.parametrize("kw", [dict(pad=(7, 7, 5, 5, 2, 0.0)), dict(pad=(9, 9, 9, 9, 0, -2.0)),
                                dict(pad=(9, 9, 9, 9, 1, 0.0)), dict(pad=(0, 0, 0, 0, 2, 0.0), inplace=True),
                                dict(affine=False, pad=(1, 2, 3, 4, 1, 0.0))])
def test_accepted_arguments(cuda, kw):
    """The edges of what the C ABI accepts, on real allocations: reflect pads one below the dimension, constant and
    replicate pads wider than the plane, an all-zero pad in place, affine 0; each equals IN, ReLU and Padding apart."""
    from feathercnn_b200 import booster
    rng = np.random.default_rng(6)
    x = rng.standard_normal((2, 3, 8, 6)).astype(np.float32)
    g, b = (rng.uniform(0.5, 1.5, 3), rng.uniform(-1, 1, 3)) if kw.get("affine", True) else (None, None)
    pad = kw["pad"]
    want = pad_ref(booster.relu(_in(x, g, b)).cpu().numpy(), *pad[:5], pad[5])
    if kw.get("inplace"):
        xs = torch.from_numpy(x).cuda()
        got = _in(xs, g, b, relu=True, pad=pad, out=xs)
    else:
        got = _in(x, g, b, relu=True, pad=pad)
    assert _bits_equal(got.cpu().numpy(), want)


# ---- Reshape rejections ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("body", ["InstanceNorm i 1 1 d i 0=3 2=0", "Padding p 1 1 d p 0=5 4=2",
                                  "Padding p 1 1 d p 2=6 4=2", "InstanceNorm i 1 1 d i 0=4 2=0\nPadding p 1 1 i p 3=6 4=2"])
@pytest.mark.parametrize("fusion", [False, True])
def test_reshape_rejections(cuda, tmp_path, body, fusion):
    """A channel count other than the blob's, or a reflect pad >= the plane's dimension, fails at Reshape
    (FEATHER_ERR_TOPOLOGY), which Net reports as -100 like every shape failure."""
    from feathercnn_b200.net import FeatherError, Net
    net = Net(fusion=fusion)
    n = 2 + body.count("\n")
    net.LoadParamFromText(f"7767517\n{n} {n}\nInput d 0 1 d 0=6 1=5 2=4\n{body}\n")
    empty = tmp_path / "empty.bin"
    empty.write_bytes(b"")
    net.LoadWeights(str(empty))
    with pytest.raises(FeatherError) as e:
        net.Forward(np.zeros((1, 4, 5, 6), np.float32))
    assert e.value.code == -100


@gpu
def test_affine_weight_counts(cuda, tmp_path):
    """affine 1 reads gamma and beta (2 x channels floats); a shorter bin fails to load; affine 0 reads none."""
    from feathercnn_b200.net import FeatherError, Net
    text = "7767517\n2 2\nInput d 0 1 d 0=6 1=5 2=4\nInstanceNorm i 1 1 d i 0=4 1=1e-5 2={}\n"
    binf = tmp_path / "w.bin"
    for affine, floats, ok in ((1, 8, True), (1, 7, False), (0, 0, True)):
        binf.write_bytes(np.arange(floats, dtype=np.float32).tobytes())
        net = Net()
        net.LoadParamFromText(text.format(affine))
        if not ok:
            with pytest.raises(FeatherError):
                net.LoadWeights(str(binf))
            continue
        net.LoadWeights(str(binf))
        x = np.random.default_rng(0).standard_normal((1, 4, 5, 6)).astype(np.float32)
        net.Forward(x)
        g, b = (np.arange(4, dtype=np.float32), np.arange(4, 8, dtype=np.float32)) if affine else (None, None)
        assert _bits_equal(net.Extract("i"), _in(x, g, b).cpu().numpy())


# ---- models end to end ----------------------------------------------------------------------------------------------
MODELS = {"style_tiny": {}, "fast_neural_style": dict(height=256, width=256)}


@pytest.fixture(scope="module")
def style_models(tmp_path_factory):
    from feathercnn_b200.tools import modelgen
    d = tmp_path_factory.mktemp("style")
    out = {}
    for name, kw in MODELS.items():
        m = modelgen.ZOO[name](**kw)
        param, binf = m.save(d / name)
        out[name] = (m, param, binf, _load_layers(param, binf))
    return out


def _load_layers(param, binf):
    """test_gpu_net_bounds.load_model for these nets: the convolutions' weights and biases, and InstanceNorm's gamma and
    beta (which load_model does not read), walked through the bin in file order."""
    from oracle import oracle as O
    layers = O.parse_param(param)
    mb = O._BinReader(binf)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))
    for L in layers:
        pd = L["params"]
        if L["type"] in CONV_TYPES:
            k, num, size = pd.get(1, 0), pd.get(0, 0), pd.get(6, 0)
            L["w"] = t(mb.load(size, 0).reshape(num, size // (num * k * k), k, k))
            L["b"] = t(mb.load(num, 1)) if pd.get(5, 0) else None
        elif L["type"] == "InstanceNorm" and pd.get(2, 1):
            L["gamma"], L["beta"] = (np.asarray(mb.load(pd[0], 1), np.float32) for _ in range(2))
    return layers


def _run(param, binf, x, fusion, graph):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    for _ in range(3 if graph else 1):
        net.Forward(x)
    net.Synchronize()
    return net


def _check_layers(net, layers):
    """Convolutions within their float64 bounds; InstanceNorm (+ReLU, +Padding) within its bound from the net's own
    bottom blob; Padding, an unfused ReLU, Interp (nearest x 2) and Eltwise SUM bit for bit.  Returns the count of each
    kind checked."""
    chains, _ = rebuild_chains(layers, net.LayerFusedAway, set(net.BlobNames()))
    failures, seen = [], {}
    for ch in chains:
        typ, pd = ch.head["type"], ch.head["params"]
        seen[typ] = seen.get(typ, 0) + 1
        if typ in ("Input", "Split"):
            continue
        got = _all(net, ch.tops[0]).cpu().numpy()
        x = _all(net, ch.head["bottoms"][0]).float().cpu().numpy()
        if typ == "InstanceNorm":
            g, b, eps = ch.head.get("gamma"), ch.head.get("beta"), float(pd.get(1, 0.001))
            y64, bound = instance_norm_bound(x, g, b, eps)
            pad = None
            for L in ch.ops:
                if L["type"] == "ReLU":
                    y64, bound = np.maximum(y64, 0), bound     # fmaxf is non-expansive
                else:
                    assert L["type"] == "Padding", L["name"]
                    pad = tuple(L["params"].get(k, 0) for k in range(5)) + (float(L["params"].get(5, 0.0)),)
            if pad is not None:
                y64 = pad_ref(y64, *pad[:4], pad[4], pad[5], dtype=np.float64)
                bound = pad_ref(bound, *pad[:4], pad[4], 0.0, dtype=np.float64)
            d = np.abs(got - y64)
            used = float(np.max(np.where(d == 0, 0.0, d / bound)))
            if used > 1.0:
                failures.append(f"{ch.head['name']}: bound used {used:.3g}")
            continue
        if typ == "Padding":
            pads = tuple(pd.get(k, 0) for k in range(5))
            assert _bits_equal(got, pad_ref(x, *pads[:4], pads[4], float(pd.get(5, 0.0)))), ch.head["name"]
            continue
        if typ == "Interp":
            assert _bits_equal(got, x.repeat(2, axis=2).repeat(2, axis=3)), ch.head["name"]
            continue
        if typ == "ReLU":                                    # unfused: the ReLU kernel, fmaxf(x, 0.f)
            assert _bits_equal(got, np.maximum(x, np.float32(0))), ch.head["name"]
            continue
        if typ == "Eltwise":
            a, b = (_all(net, t).float().cpu().numpy() for t in ch.head["bottoms"])
            assert _bits_equal(got, a + b), ch.head["name"]
            continue
        assert typ in CONV_TYPES and not ch.ops, (typ, ch.head["name"])
        algo = net.LayerConvAlgo(ch.head["name"])
        ins = {b: _all(net, b) for b in dict.fromkeys(ch.bottoms)}
        tops = {t: _all(net, t) for t in ch.tops}
        for top, used, _, kind, path in check_chain(ch, ins, tops, 2, algo):
            if used > 1.0:
                failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
    assert not failures, "\n".join(failures[:20])
    return seen


@gpu
@pytest.mark.parametrize("name", list(MODELS))
def test_model_end_to_end(cuda, style_models, name):
    from feathercnn_b200.tools import modelgen
    m, param, binf, layers = style_models[name]
    batch = 2
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])
    outs = []
    for fusion, graph in SETTINGS:
        net = _run(param, binf, x, fusion, graph)
        assert net.BlobShape("conv6") == (batch,) + m.shape["data"]
        if fusion and name == "fast_neural_style":
            fused = {L["name"] for L in layers if net.LayerFusedAway(L["name"])}
            pads = {n for n in fused if n.endswith("_pad")}
            relus = {n for n in fused if "relu" in n}
            assert pads == {"conv2_pad", "conv3_pad", "conv6_pad"} | {f"res{b}_conv2_pad" for b in range(1, 6)}
            assert len(relus) == 10 and fused == pads | relus
        seen = _check_layers(net, layers)
        assert seen["InstanceNorm"] == sum(L["type"] == "InstanceNorm" for L in layers)
        outs.append(net.Extract("conv6"))
        del net
    assert all(_bits_equal(outs[0], o) for o in outs[1:])
