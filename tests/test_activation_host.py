"""Sigmoid, TanH, Swish, HardSigmoid and HardSwish on the host (no kernel is launched): a NumPy float32 restatement of the
hard types, the C ABI's rejections, the loader's defaults and rejections, which layers fusion takes (none of these), the
Caffe converter's Sigmoid / TanH, the new models' shapes, and their topology against torchvision.

Topology check.  modelgen's weights are loaded into torchvision's module (BatchNorm + Scale become one BatchNorm2d:
weight = slope * s, bias = bias * s + t), and both are evaluated in float64 on the same image: the module's eval forward
and `run_net64`, a float64 evaluation of the written .param / .bin by ncnn's layer definitions.  The file writes PyTorch's
alpha 1/6 as 1.666667e-01 (pnnx's six digits), so the two nets differ by design.  The tolerance is derived from that:
`run_net64` is run with the file's alpha and with alpha = 1/6 exactly.  With 1/6 it must equal the module to float64
rounding (TOPO_REL of the output's scale); with the file's alpha it must stay within the measured alpha effect (the two
`run_net64` results' difference) plus the same rounding term.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_clip_prelu_host import _fused_away, _net_param, _strip_bn_scale
from test_tools import layer as caffe_layer

ACTS = ("Sigmoid", "TanH", "Swish", "HardSigmoid", "HardSwish")
HEAD = "7767517\n2 2\nInput data 0 1 data 0=4 1=8 2=8\n"
TOPO_REL = 1e-10


# ---- NumPy float32 restatement of the hard types --------------------------------------------------------------------
def hard_bounds(alpha, beta):
    """(lower, upper) as ncnn's load_param computes them in fp32: lower = -beta / alpha, upper = 1 / alpha + lower."""
    alpha, beta = np.float32(alpha), np.float32(beta)
    lower = np.float32(-beta / alpha)
    return lower, np.float32(np.float32(np.float32(1) / alpha) + lower)


def hard_np(x, kind, alpha=0.2, beta=0.5):
    """HardSigmoid / HardSwish in float32, one rounding per operation (no FMA), as include/fcuda.h defines them."""
    x = np.asarray(x, np.float32)
    a, b = np.float32(alpha), np.float32(beta)
    lower, upper = hard_bounds(a, b)
    with np.errstate(over="ignore", invalid="ignore"):
        lin = (x * a).astype(np.float32) + b
        if kind == "HardSigmoid":
            return np.where(x < lower, np.float32(0), np.where(x > upper, np.float32(1), lin)).astype(np.float32)
        return np.where(x < lower, np.float32(0), np.where(x > upper, x, (x * lin).astype(np.float32))).astype(np.float32)


def test_hard_bounds_at_ncnn_defaults_and_pnnx_alpha():
    assert hard_bounds(0.2, 0.5) == (np.float32(-2.5), np.float32(2.5))
    lo, hi = hard_bounds(np.float32(1.666667e-01), 0.5)
    # fp32 of 1.666667e-01 is 0.16666670143..., so the branch points sit just inside +-3
    assert lo == np.float32(-0.5) / np.float32(1.666667e-01) and -3 < lo < -2.9999
    assert hi == np.float32(np.float32(1) / np.float32(1.666667e-01)) + lo and 2.9999 < hi < 3


@pytest.mark.parametrize("kind", ["HardSigmoid", "HardSwish"])
def test_hard_restatement_by_hand(kind):
    lo, hi = hard_bounds(0.2, 0.5)
    x = np.array([-np.inf, -3.0, np.nextafter(lo, -np.inf), lo, 0.0, -0.0, 1.0, hi, np.nextafter(hi, np.inf), 4.0, np.inf,
                  np.nan], np.float32)
    y = hard_np(x, kind)
    if kind == "HardSigmoid":
        want = [0, 0, 0, 0, 0.5, 0.5, 0.7, 1, 1, 1, 1]
    else:
        want = [0, 0, 0, 0, 0, 0, 0.7, 2.5, np.nextafter(hi, np.inf), 4, np.inf]
    # at lower the linear branch runs: -2.5 * 0.2 + 0.5 rounds to 0 exactly
    assert np.array_equal(y[:-1], np.asarray(want, np.float32)), y
    assert np.isnan(y[-1])  # NaN fails both comparisons and propagates


@pytest.mark.parametrize("kind", ["HardSigmoid", "HardSwish"])
def test_hard_restatement_against_torch(kind):
    """PyTorch's hardsigmoid / hardswish are alpha = 1/6 exactly; with pnnx's 1.666667e-01 the difference is at most
    |x| * |alpha - 1/6| (HardSigmoid) or x^2 * |alpha - 1/6| (HardSwish) inside the branch points, plus what the branch
    points' shift by the same amount allows, and float32 rounding of the result."""
    x = np.linspace(-8, 8, 200001, dtype=np.float32)
    a = np.float32(1.666667e-01)
    da = abs(float(a) - 1 / 6)
    got = hard_np(x, kind, a, 0.5).astype(np.float64)
    tx = torch.from_numpy(x.astype(np.float64))
    want = (F.hardsigmoid(tx) if kind == "HardSigmoid" else F.hardswish(tx)).numpy()
    xx = np.abs(x.astype(np.float64))
    slack = (xx if kind == "HardSigmoid" else xx * xx) * da + 3 * xx * da + 2.0 ** -22 * (np.abs(want) + xx)
    assert np.all(np.abs(got - want) <= slack)


# ---- C ABI -----------------------------------------------------------------------------------------------------------
def test_abi_rejects_before_any_launch():
    """A fake device pointer is never touched: every rejection is decided first."""
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    d = ctypes.c_void_p(16)
    f = lib.fcuda_activation_forward
    assert f(None, d, 4, 0, 0.2, 0.5, None) == -100
    assert f(d, None, 4, 0, 0.2, 0.5, None) == -100
    assert f(d, d, 0, 0, 0.2, 0.5, None) == -100
    for t in (-1, 5, 14):
        assert f(d, d, 4, t, 0.2, 0.5, None) == -200
    for t in (3, 4):
        for alpha, beta in ((0.0, 0.5), (-0.0, 0.5), (math.inf, 0.5), (-math.inf, 0.5), (math.nan, 0.5), (0.2, math.inf),
                            (0.2, math.nan)):
            assert f(d, d, 4, t, alpha, beta, None) == -200, (t, alpha, beta)


def test_wrapper_maps_names():
    from feathercnn_b200 import booster
    assert booster.ACTIVATIONS == list(ACTS)


# ---- loader ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("line", [
    "Sigmoid s 1 1 data out",
    "TanH t 1 1 data out",
    "Swish w 1 1 data out",
    "HardSigmoid h 1 1 data out",                               # defaults 0.2 / 0.5
    "HardSwish h 1 1 data out 0=1.666667e-01 1=5.000000e-01",   # pnnx
    "HardSwish h 1 1 data out 0=-0.25 1=-1.0",                  # negative alpha is a valid line
    "Sigmoid s 1 1 data out 0=0.0",                             # parameters of other types are ignored
])
def test_load_param_accepts(line):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(HEAD + line + "\n")
    assert "out" in net.BlobNames()


@pytest.mark.parametrize("line", [
    "HardSigmoid h 1 1 data out 0=0.0",
    "HardSwish h 1 1 data out 0=0.0 1=0.5",
    "HardSwish h 1 1 data out 0=1e39",        # overflows fp32 to inf
    "HardSigmoid h 1 1 data out 0=0.2 1=-1e39",
    "HardSwish h 1 1 data out 0=1e-46",       # underflows fp32 to 0
])
def test_load_param_rejects_bad_alpha_beta(line):
    from feathercnn_b200.net import FeatherError, Net
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(HEAD + line + "\n")
    assert e.value.code == -200


@pytest.mark.parametrize("act", ACTS)
def test_load_param_rejects_blob_counts(act):
    from feathercnn_b200.net import FeatherError, Net
    text = "7767517\n3 3\nInput data 0 1 data 0=4 1=8 2=8\nSplit sp 1 2 data a b\n" + f"{act} x 2 1 a b out\n"
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(text)
    assert e.value.code == -200
    text = "7767517\n2 3\nInput data 0 1 data 0=4 1=8 2=8\n" + f"{act} x 1 2 data o1 o2\n"
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(text)
    assert e.value.code == -200


# ---- fusion: none ----------------------------------------------------------------------------------------------------
INP = "Input data 0 1 data 0=8 1=8 2=16"
CONV = "Convolution {n} 1 1 {b} {t} 0=16 1=3 4=1 5=1 6=2304"


@pytest.mark.parametrize("act", ACTS)
def test_conv_takes_no_activation(act):
    lines = [INP, CONV.format(n="conv", b="data", t="c"), f"{act} act 1 1 c out"]
    assert _fused_away(lines, ["act"]) == (0, {"act": 0})


@pytest.mark.parametrize("act", ACTS)
def test_relu_and_clip_still_fold_ahead_of_an_activation(act):
    for prev in ("ReLU relu 1 1 c r", "Clip relu 1 1 c r 0=0.0 1=6.0"):
        lines = [INP, CONV.format(n="conv", b="data", t="c"), prev, f"{act} act 1 1 r out"]
        assert _fused_away(lines, ["relu", "act"]) == (1, {"relu": 1, "act": 0})


def test_se_tiny_activations_never_fuse():
    """With BatchNorm / Scale stripped (their folding needs the weights on the device; test_gpu_activation checks it):
    the SE ReLU folds into its convolution and no activation layer is fused away."""
    from feathercnn_b200.tools import modelgen
    m = modelgen.se_tiny()
    lines = _strip_bn_scale(m.lines)
    acts = [l.split()[1] for l in lines if l.split()[0] in ACTS]
    assert sorted(l.split()[0] for l in lines if l.split()[0] in ACTS) == sorted(ACTS)
    n, f = _fused_away(lines, acts + ["se_relu"])
    assert all(f[a] == 0 for a in acts), f
    assert f["se_relu"] == 1


def test_every_type_is_registered():
    from feathercnn_b200.net import Net
    for act in ACTS:
        Net().LoadParamFromText(HEAD + f"{act} x 1 1 data out\n")
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError):
        Net().LoadParamFromText(HEAD + "Mish x 1 1 data out\n")


# ---- Caffe converter -------------------------------------------------------------------------------------------------
def test_caffe_sigmoid_tanh_convert():
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import caffe2feather
    model = _net_param([caffe_layer("sig", "Sigmoid", ["data"], ["a"]), caffe_layer("th", "TanH", ["a"], ["b"])])
    text, binary = caffe2feather.convert(model)
    lines = text.splitlines()
    assert "Sigmoid sig 1 1 data a" in lines and "TanH th 1 1 a b" in lines
    assert binary == b""
    Net().LoadParamFromText(text)


# ---- models ----------------------------------------------------------------------------------------------------------
def _types(m):
    return [l.split()[0] for l in m.lines]


def test_model_shapes_and_layer_counts():
    from feathercnn_b200.tools import modelgen
    large, small, eff = modelgen.mobilenet_v3_large(), modelgen.mobilenet_v3_small(), modelgen.efficientnet_b0()
    assert large.shape["conv_last"] == (960, 7, 7) and large.shape["fc1"] == (1280, 1, 1)
    assert small.shape["conv_last"] == (576, 7, 7) and small.shape["fc1"] == (1024, 1, 1)
    assert eff.shape["conv_last"] == (1280, 7, 7)
    for m in (large, small, eff):
        assert m.shape["prob"] == (1000, 1, 1)
    t = _types(large)
    assert (t.count("HardSigmoid"), t.count("BinaryOp")) == (8, 8 + 10)  # 8 SE gates; 8 SE multiplies, 10 shortcuts
    t = _types(small)
    assert (t.count("HardSigmoid"), t.count("BinaryOp")) == (9, 9 + 6)
    t = _types(eff)
    assert (t.count("Sigmoid"), t.count("BinaryOp"), t.count("Swish")) == (16, 16 + 9, 1 + 15 + 16 + 16 + 1)
    # torchvision's multiply-add counts: 0.22, 0.06 and 0.39 G
    assert 0.21e9 < large.flops / 2 < 0.23e9 and 0.05e9 < small.flops / 2 < 0.065e9 and 0.38e9 < eff.flops / 2 < 0.40e9
    e = modelgen.espcn()
    assert e.shape["output"] == (1, 1080, 1920) and _types(e).count("TanH") == 2
    assert modelgen.espcn(scale=2, height=8, width=5).shape["output"] == (1, 16, 10)
    s = modelgen.se_tiny()
    assert set(ACTS) <= set(_types(s)) and s.shape["dw"] == (16, 8, 8) and s.shape["prob"] == (10, 1, 1)
    assert "ConvolutionDepthWise dw 1 1 " in "\n".join(s.lines) and " 1=5 3=2 4=2 " in [l for l in s.lines
                                                                                       if l.startswith("ConvolutionDepthWise")][0]


def test_hard_layers_written_as_pnnx_does():
    from feathercnn_b200.tools import modelgen
    for l in modelgen.mobilenet_v3_small().lines:
        if l.split()[0] in ("HardSigmoid", "HardSwish"):
            assert l.endswith(" 0=1.666667e-01 1=5.000000e-01"), l


# ---- float64 evaluation of a written net ------------------------------------------------------------------------------
def act64(kind, x, alpha=0.2, beta=0.5, exact_alpha=None):
    """float64 value of an activation; the hard types' branch points are the fp32 ones (hard_bounds), or those of
    `exact_alpha` computed in float64 when given."""
    if kind == "Sigmoid":
        return torch.sigmoid(x)
    if kind == "TanH":
        return torch.tanh(x)
    if kind == "Swish":
        return x * torch.sigmoid(x)
    if exact_alpha is not None:
        a, b = exact_alpha, float(np.float32(beta))
        lo, hi = -b / a, 1 / a - b / a
    else:
        a, b = float(np.float32(alpha)), float(np.float32(beta))
        lo, hi = (float(v) for v in hard_bounds(alpha, beta))
    lin = x * a + b
    top = torch.ones_like(x) if kind == "HardSigmoid" else x
    mid = lin if kind == "HardSigmoid" else x * lin
    return torch.where(x < lo, torch.zeros_like(x), torch.where(x > hi, top, mid))


def layer64(L, ins, exact_alpha=None):
    """{top: float64 value} of one layer from its bottoms' values (N, C, H, W)."""
    typ, pd = L["type"], L["params"]
    x = ins[0] if ins else None
    if typ in ("Convolution", "ConvolutionDepthWise"):
        w = L["w"].to(x.device).double()
        b = L["b"].to(x.device).double() if L["b"] is not None else None
        y = F.conv2d(x, w, b, stride=pd.get(3, 1), padding=pd.get(4, 0), groups=pd.get(7, 1))
    elif typ in ("BatchNorm", "Scale"):
        from test_gpu_net_bounds import affine_of
        m, a, _ = (v.to(x.device).view(1, -1, 1, 1) for v in affine_of(L))
        y = x * m + a
    elif typ == "ReLU":
        y = x.clamp_min(0)
    elif typ == "Split":
        return {t: x for t in L["tops"]}
    elif typ == "Pooling":
        assert pd.get(4, 0) == 1 and pd.get(0, 0) == 1, L["name"]
        y = x.mean(dim=(2, 3), keepdim=True)
    elif typ == "BinaryOp":
        op = pd.get(0, 0)
        assert op in (0, 2) and len(ins) == 2, L["name"]
        y = ins[0] + ins[1] if op == 0 else ins[0] * ins[1]
    elif typ == "InnerProduct":
        w = L["w"].to(x.device).double()
        y = x.reshape(x.shape[0], -1) @ w.T
        if L["b"] is not None:
            y = y + L["b"].to(x.device).double()
        y = y.reshape(x.shape[0], -1, 1, 1)
    elif typ == "Softmax":
        y = torch.softmax(x.reshape(x.shape[0], -1), dim=1).reshape(x.shape)
    elif typ == "Dropout":
        y = x
    elif typ == "PixelShuffle":
        assert pd.get(1, 0) == 0
        y = F.pixel_shuffle(x, pd.get(0, 1))
    elif typ in ACTS:
        y = act64(typ, x, pd.get(0, 0.2), pd.get(1, 0.5), exact_alpha)
    else:
        raise AssertionError(typ)
    return {L["tops"][0]: y}


def run_net64(layers, x, exact_alpha=None):
    blobs = {}
    for L in layers:
        if L["type"] == "Input":
            blobs[L["tops"][0]] = x
            continue
        blobs.update(layer64(L, [blobs[b] for b in L["bottoms"]], exact_alpha))
    return blobs


# ---- topology against torchvision ------------------------------------------------------------------------------------
def _load_into_torchvision(layers, module):
    """modelgen's weights, in file order, into the module's Conv2d / BatchNorm2d / Linear, in definition order."""
    targets = [mod for mod in module.modules() if isinstance(mod, (torch.nn.Conv2d, torch.nn.BatchNorm2d, torch.nn.Linear))]
    k = 0
    with torch.no_grad():
        for i, L in enumerate(layers):
            typ = L["type"]
            if typ in ("Convolution", "ConvolutionDepthWise", "InnerProduct"):
                t = targets[k]
                assert isinstance(t, torch.nn.Linear if typ == "InnerProduct" else torch.nn.Conv2d), (L["name"], t)
                assert tuple(t.weight.shape) == tuple(L["w"].shape), (L["name"], t.weight.shape, L["w"].shape)
                t.weight.copy_(L["w"].double())
                assert (t.bias is None) == (L["b"] is None), L["name"]
                if t.bias is not None:
                    t.bias.copy_(L["b"].double())
                k += 1
            elif typ == "BatchNorm":
                t = targets[k]
                S = layers[i + 1]
                assert isinstance(t, torch.nn.BatchNorm2d) and S["type"] == "Scale", L["name"]
                slope, mean, var, bias = (v.double() for v in L["bn"])
                s, sb = S["s"].double(), S["t"].double()
                assert t.eps == pytest.approx(L["params"][1], rel=1e-6), (L["name"], t.eps)
                t.eps = float(np.float32(L["params"][1]))
                t.weight.copy_(slope * s)
                t.bias.copy_(bias * s + sb)
                t.running_mean.copy_(mean)
                t.running_var.copy_(var)
                k += 1
    assert k == len(targets), (k, len(targets))


TOPOLOGY = ["mobilenet_v3_large", "mobilenet_v3_small", "efficientnet_b0"]


@pytest.mark.parametrize("name", TOPOLOGY)
def test_topology_matches_torchvision(tmp_path, name):
    import torchvision
    from feathercnn_b200.tools import modelgen
    from test_gpu_net_bounds import load_model
    size = 96
    mw = modelgen.ZOO[name](size=size)
    layers = load_model(*mw.save(tmp_path / name))
    module = getattr(torchvision.models, name)(weights=None).double().eval()
    _load_into_torchvision(layers, module)
    x = torch.from_numpy(np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(2)])).double()
    with torch.no_grad():
        logits = module(x)
    fc = [L for L in layers if L["type"] == "InnerProduct"][-1]["tops"][0]
    file_alpha = run_net64(layers, x)[fc].reshape(2, -1)
    exact = run_net64(layers, x, exact_alpha=1 / 6)[fc].reshape(2, -1)
    scale = float(logits.abs().max())
    assert scale > 0
    rounding = TOPO_REL * scale
    assert float((exact - logits).abs().max()) <= rounding, name
    alpha_effect = (file_alpha - exact).abs()
    assert bool(((file_alpha - logits).abs() <= alpha_effect + rounding).all()), name
    # and the alpha effect is the size the 2e-7 relative change of alpha predicts, not a topology difference in disguise
    if name != "efficientnet_b0":
        assert 0 < float(alpha_effect.max()) < 1e-4 * scale, (name, float(alpha_effect.max()), scale)
    else:
        assert float(alpha_effect.max()) == 0.0  # no hard activation
