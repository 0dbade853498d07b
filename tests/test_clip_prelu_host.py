"""Clip and PReLU on the host (no kernel is launched): the loaders' parameters, defaults and rejections, the C ABI's
rejection of FCUDA_ACT_CLIP outside fcuda_conv_forward_clip, which layers Net::ApplyFusion folds a Clip into, and the
Caffe converter's ReLU6 / Clip / PReLU."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

from test_tools import ffloat, fbytes, fint, layer as caffe_layer

HEAD = "7767517\n2 2\nInput data 0 1 data 0=4 1=8 2=8\n"


def _text(lines):
    blobs = {t for l in lines for t in l.split()[4 + int(l.split()[2]):4 + int(l.split()[2]) + int(l.split()[3])]}
    return "7767517\n" + f"{len(lines)} {len(blobs)}\n" + "\n".join(lines) + "\n"


# ---- loaders ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("line", [
    "Clip c 1 1 data out",                       # defaults: -FLT_MAX .. FLT_MAX
    "Clip c 1 1 data out 0=0.000000e+00 1=6.000000e+00",
    "Clip c 1 1 data out 0=2.5 1=2.5",           # min == max
    "Clip c 1 1 data out 1=-1.0",                # max only
    "PReLU p 1 1 data out 0=1",
    "PReLU p 1 1 data out 0=4",
])
def test_load_param_accepts(line):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(HEAD + line + "\n")
    assert "out" in net.BlobNames()


@pytest.mark.parametrize("line, code", [
    ("Clip c 1 1 data out 0=1.0 1=0.5", -200),      # min > max
    ("PReLU p 1 1 data out", -100),                 # num_slope missing (0)
    ("PReLU p 1 1 data out 0=-2", -100),
])
def test_load_param_rejections(line, code):
    from feathercnn_b200.net import FeatherError, Net
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(HEAD + line + "\n")
    assert e.value.code == code


def test_clip_one_bound_keeps_the_other_default():
    from feathercnn_b200.net import FeatherError, Net
    Net().LoadParamFromText(HEAD + "Clip c 1 1 data out 0=7.0\n")     # max defaults to FLT_MAX
    Net().LoadParamFromText(HEAD + "Clip c 1 1 data out 1=-7.0\n")    # min defaults to -FLT_MAX
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(HEAD + "Clip c 1 1 data out 0=1.0 1=-1.0\n")
    assert e.value.code == -200


# ---- C ABI -----------------------------------------------------------------------------------------------------------
def test_clip_activation_value():
    from feathercnn_b200 import booster
    assert (booster.ACT_NONE, booster.ACT_RELU, booster.ACT_CLIP) == (0, 1, 2)


@pytest.mark.parametrize("algo", [0, 1, 2, 3, 4, 6])
def test_entry_points_without_bounds_reject_clip(algo):
    """fcuda_conv_forward / _residual / _ext / _pool return -200 for FCUDA_ACT_CLIP before touching any pointer."""
    from feathercnn_b200._lib import FcudaConvParam, fcuda
    lib = fcuda()
    group = 16 if algo == 3 else 1
    p = FcudaConvParam(16, 16, 12, 12, 3, 3, 0, 0, 1, 1, 1, 1, 1, 1, group, 1, 2)
    assert lib.fcuda_conv_assign_output_dim(ctypes.byref(p)) == 0
    dummy = ctypes.c_void_p(16)
    args = (ctypes.byref(p), algo, dummy, dummy, dummy, dummy, dummy)
    assert lib.fcuda_conv_forward(*args, 1, None) == -200
    assert lib.fcuda_conv_forward_residual(*args, dummy, 0, 1, None) == -200
    assert lib.fcuda_conv_forward_ext(*args, None, 0, 1, 1, 1, None) == -200
    if lib.fcuda_conv_can_pool(ctypes.byref(p), algo):
        assert lib.fcuda_conv_forward_pool(*args, 1, None) == -200
    # and the clip entry point wants FCUDA_ACT_CLIP and ordered bounds
    assert lib.fcuda_conv_forward_clip(*args, 1.0, 0.0, 1, None) == -200
    assert lib.fcuda_conv_forward_clip(*args, float("nan"), 6.0, 1, None) == -200
    p.activation = 1
    assert lib.fcuda_conv_forward_clip(*args, 0.0, 6.0, 1, None) == -200


def test_elementwise_entry_points_reject_bad_arguments():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    d = ctypes.c_void_p(16)
    assert lib.fcuda_clip_forward(d, d, 4, 1.0, 0.0, None) == -200
    assert lib.fcuda_clip_forward(None, d, 4, 0.0, 1.0, None) == -100
    assert lib.fcuda_prelu_forward(d, d, 4, 16, d, 3, 1, None) == -200
    assert lib.fcuda_prelu_forward(d, d, 4, 16, None, 4, 1, None) == -100


# ---- fusion ----------------------------------------------------------------------------------------------------------
def _fused_away(lines, layers):
    from feathercnn_b200.net import Net
    net = Net(fusion=True)
    net.LoadParamFromText(_text(lines))
    n = net.FuseNow()
    return n, {name: net.LayerFusedAway(name) for name in layers}


INP = "Input data 0 1 data 0=8 1=8 2=16"
CONV = "Convolution {n} 1 1 {b} {t} 0=16 1=3 4=1 5=1 6=2304"


def test_conv_absorbs_clip():
    n, f = _fused_away([INP, CONV.format(n="conv", b="data", t="c"), "Clip clip 1 1 c out 0=0.0 1=6.0"], ["clip"])
    assert (n, f) == (1, {"clip": 1})


def test_depthwise_conv_absorbs_clip():
    dw = "ConvolutionDepthWise dw 1 1 data c 0=16 1=3 4=1 5=0 6=144 7=16"
    n, f = _fused_away([INP, dw, "Clip clip 1 1 c out 0=0.0 1=6.0"], ["clip"])
    assert (n, f) == (1, {"clip": 1})


def test_clip_after_relu_stays():
    lines = [INP, CONV.format(n="conv", b="data", t="c"), "ReLU relu 1 1 c r", "Clip clip 1 1 r out 0=0.0 1=6.0"]
    assert _fused_away(lines, ["relu", "clip"]) == (1, {"relu": 1, "clip": 0})


def test_clipped_conv_takes_no_pooling_and_no_relu():
    lines = [INP, CONV.format(n="conv", b="data", t="c"), "Clip clip 1 1 c r 0=0.0 1=6.0",
             "Pooling pool 1 1 r p 0=0 1=2 2=2 3=0", "ReLU relu 1 1 p out"]
    assert _fused_away(lines, ["clip", "pool", "relu"]) == (1, {"clip": 1, "pool": 0, "relu": 0})
    lines = [INP, CONV.format(n="conv", b="data", t="c"), "Clip clip 1 1 c r 0=0.0 1=6.0", "ReLU relu 1 1 r out"]
    assert _fused_away(lines, ["clip", "relu"]) == (1, {"clip": 1, "relu": 0})


def test_dilated_conv_keeps_its_clip():
    dil = "Convolution conv 1 1 data c 0=16 1=3 2=2 4=2 5=1 6=2304"
    assert _fused_away([INP, dil, "Clip clip 1 1 c out 0=0.0 1=6.0"], ["clip"]) == (0, {"clip": 0})


def test_shared_conv_top_keeps_its_clip():
    lines = [INP, CONV.format(n="conv", b="data", t="c"), "Split sp 1 2 c c1 c2", "Clip clip 1 1 c1 r 0=0.0 1=6.0",
             "Eltwise sum 2 1 r c2 out 0=1"]
    assert _fused_away(lines, ["clip"])[1] == {"clip": 0}


def test_clip_without_conv_producer_and_prelu_stay():
    lines = [INP, "Pooling pool 1 1 data p 0=1 1=2 2=2 3=0", "Clip clip 1 1 p q 0=0.0 1=6.0",
             CONV.format(n="conv", b="q", t="c"), "PReLU prelu 1 1 c out 0=16"]
    assert _fused_away(lines, ["clip", "prelu"]) == (0, {"clip": 0, "prelu": 0})


def _strip_bn_scale(lines):
    """mobilenet_v2's text without BatchNorm / Scale (their folding needs the weights on the device)."""
    out, rename = [], {}
    for l in lines:
        tok = l.split()
        nb, nt = int(tok[2]), int(tok[3])
        bottoms = [rename.get(b, b) for b in tok[4:4 + nb]]
        if tok[0] in ("BatchNorm", "Scale"):
            rename[tok[4 + nb]] = bottoms[0]
            continue
        out.append(" ".join(tok[:4] + bottoms + tok[4 + nb:]))
    return out


def test_mobilenet_v2_clips_and_shortcuts_fuse():
    from feathercnn_b200.tools import modelgen
    m = modelgen.mobilenet_v2(size=64)
    lines = _strip_bn_scale(m.lines)
    clips = [l.split()[1] for l in lines if l.startswith("Clip ")]
    sums = [l.split()[1] for l in lines if l.startswith("Eltwise ")]
    assert (len(clips), len(sums)) == (35, 10)
    n, f = _fused_away(lines, clips + sums)
    assert n == 45 and all(f[c] == 1 for c in clips + sums), f


def test_mobilenet_v2_topology():
    from feathercnn_b200.tools import modelgen
    m = modelgen.mobilenet_v2()
    types = [l.split()[0] for l in m.lines]
    convs = types.count("Convolution") + types.count("ConvolutionDepthWise")
    assert (convs, types.count("ConvolutionDepthWise"), types.count("BatchNorm"), types.count("Scale")) == (53, 17, 52, 52)
    assert m.shape["conv_last"] == (1280, 7, 7) and m.shape["prob"] == (1000, 1, 1)
    assert 0.55e9 < m.flops < 0.65e9  # ~300 M multiply-adds
    # projections are linear: no Clip reads a *_linear Scale
    for l in m.lines:
        if l.startswith("Clip "):
            assert "_linear" not in l.split()[4], l


def test_prelu_model_writer():
    from feathercnn_b200.tools import modelgen
    m = modelgen.prelu_tiny()
    lines = [l for l in m.lines if l.startswith("PReLU ")]
    assert [l.split()[-1] for l in lines] == ["0=16", "0=1"]


# ---- converter -------------------------------------------------------------------------------------------------------
def _net_param(layers: list[bytes]) -> bytes:
    """NetParameter with input "data" (1, 4, 6, 6) and the given layers (test_tools.layer messages)."""
    return fbytes(3, b"data") + b"".join(fint(4, v) for v in (1, 4, 6, 6)) + b"".join(layers)


def test_caffe_relu6_clip_prelu_convert():
    from feathercnn_b200.tools import caffe2feather
    slopes = np.array([0.1, -0.2, 0.3, 0.4], np.float32)
    shared = np.array([0.125], np.float32)
    clip_param = ffloat(1, -1.5) + ffloat(2, 0.123456789)
    model = _net_param([
        caffe_layer("r6", "ReLU6", ["data"], ["a"]),
        caffe_layer("cl", "Clip", ["a"], ["b"], f148=clip_param),
        caffe_layer("pr", "PReLU", ["b"], ["c"], blobs=[slopes]),
        caffe_layer("prs", "PReLU", ["c"], ["d"], blobs=[shared], f131=fint(2, 1)),
    ])
    text, binary = caffe2feather.convert(model)
    lines = text.splitlines()
    assert "Clip r6 1 1 data a 0=0.000000e+00 1=6.000000e+00" in lines
    cl = [l for l in lines if l.startswith("Clip cl ")][0].split()
    assert float(np.float32(cl[-2].split("=")[1])) == np.float32(-1.5)
    assert np.float32(cl[-1].split("=")[1]) == np.float32(0.123456789)  # nine significant digits survive
    assert "PReLU pr 1 1 b c 0=4" in lines and "PReLU prs 1 1 c d 0=1" in lines
    assert binary == slopes.tobytes() + shared.tobytes()  # raw fp32, no flag
    # and the loader takes what the converter wrote
    from feathercnn_b200.net import Net
    Net().LoadParamFromText(text)


def test_caffe_clip_without_bounds_is_rejected():
    from feathercnn_b200.tools import caffe2feather
    model = _net_param([caffe_layer("cl", "Clip", ["data"], ["b"])])
    with pytest.raises(ValueError):
        caffe2feather.convert(model)
