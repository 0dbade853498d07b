"""Dilated depthwise convolution and DeepLab-v3 on the host (no kernel is launched): the loader and the fusion of a Clip into
a dilated depthwise layer, the C ABI's return codes for dilated depthwise calls, the DeepLab-v3 MobileNet-v2 blob shapes,
the Caffe converter on a hand-encoded dilated depthwise layer, and the new kernels' SASS."""
from __future__ import annotations

import collections
import ctypes
import re

import numpy as np
import pytest

from test_igemm_presplit_sass import _functions, _kernels
from test_tools import fbytes, fint, layer as caffe_layer

NAIVE, IM2COL, SGECONV, DEPTHWISE, WINOGRADF63 = range(5)
NONE, RELU, CLIP = 0, 1, 2
D = 16  # a non-NULL pointer no rejected call may touch

INP = "Input data 0 1 data 0=33 1=33 2=16"
DW_DIL = "ConvolutionDepthWise dw 1 1 data c 0=16 1=3 2=2 4=2 5=0 6=144 7=16"
CONV_DIL = "Convolution conv 1 1 data c 0=16 1=3 2=2 4=2 5=1 6=2304"


def _text(lines):
    blobs = {t for l in lines for t in l.split()[4 + int(l.split()[2]):4 + int(l.split()[2]) + int(l.split()[3])]}
    return "7767517\n" + f"{len(lines)} {len(blobs)}\n" + "\n".join(lines) + "\n"


def _fused_away(lines, layers):
    from feathercnn_b200.net import Net
    net = Net(fusion=True)
    net.LoadParamFromText(_text(lines))
    n = net.FuseNow()
    return n, {name: net.LayerFusedAway(name) for name in layers}


# ---- loader and fusion -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("line", [DW_DIL, DW_DIL.replace(" 2=2 ", " 2=4 12=2 "), DW_DIL.replace("1=3 2=2 4=2 5=0 6=144", "1=5 2=2 4=4 5=0 6=400")])
def test_load_param_accepts_dilated_depthwise(line):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(_text([INP, line]))
    assert "c" in net.BlobNames()


def test_dilated_depthwise_absorbs_its_clip():
    assert _fused_away([INP, DW_DIL, "Clip clip 1 1 c out 0=0.0 1=6.0"], ["clip"]) == (1, {"clip": 1})


def test_dilated_ordinary_conv_keeps_its_clip():
    assert _fused_away([INP, CONV_DIL, "Clip clip 1 1 c out 0=0.0 1=6.0"], ["clip"]) == (0, {"clip": 0})


def test_dilated_depthwise_takes_no_residual():
    """A residual sum after a dilated depthwise layer stays an Eltwise: the depthwise epilogue cannot add it."""
    lines = [INP, "Split sp 1 2 data d1 d2", DW_DIL.replace(" data c ", " d1 c "), "Eltwise sum 2 1 c d2 out 0=1"]
    assert _fused_away(lines, ["sum"])[1] == {"sum": 0}


# ---- C ABI -----------------------------------------------------------------------------------------------------------
def _param(activation=NONE, ch=16, group=16, dil=2):
    from feathercnn_b200._lib import FcudaConvParam, fcuda
    p = FcudaConvParam(ch, ch, 33, 33, 3, 3, dil, dil, dil, dil, 1, 1, 1, 1, group, 1, activation)
    assert fcuda().fcuda_conv_assign_output_dim(ctypes.byref(p)) == 0
    p.output_h = p.output_w = 33  # pad = dilation keeps the plane
    return p


def _opts(**kw):
    from feathercnn_b200._lib import FcudaConvOptions
    return FcudaConvOptions(**kw)


def _opts_call(p, algo, o, ptrs=(D, D, D, D, D)):
    from feathercnn_b200._lib import fcuda
    return fcuda().fcuda_conv_forward_opts(ctypes.byref(p), algo, *ptrs, ctypes.byref(o), 1, None)


def test_depthwise_algorithm_is_selected_for_dilated_depthwise():
    from feathercnn_b200._lib import fcuda
    algo = ctypes.c_int(-1)
    assert fcuda().fcuda_conv_select_algo_tuned(ctypes.byref(_param()), ctypes.byref(algo)) == 0
    assert algo.value == DEPTHWISE


@pytest.mark.parametrize("dil", [(2, 2), (4, 1), (1, 18)])
def test_dilated_depthwise_passes_the_dilation_gate(dil):
    """A NULL output gives -100: the call got past every -200 of the dilation, with and without a Clip."""
    from feathercnn_b200._lib import fcuda
    no_out = (None, D, D, D, D)
    o = _opts(dilation_h=dil[0], dilation_w=dil[1])
    assert _opts_call(_param(), DEPTHWISE, o, no_out) == -100
    p = _param()
    assert fcuda().fcuda_conv_forward_ext(ctypes.byref(p), DEPTHWISE, *no_out, None, 0, dil[0], dil[1], 1, None) == -100
    assert _opts_call(_param(CLIP), DEPTHWISE, _opts(clip_min=0, clip_max=6, dilation_h=dil[0], dilation_w=dil[1]),
                      no_out) == -100


def test_dilated_codes_outside_depthwise_are_unchanged():
    clip_dil = _opts(clip_min=0, clip_max=6, dilation_h=2, dilation_w=2)
    assert _opts_call(_param(CLIP, group=1), SGECONV, clip_dil) == -200
    for algo in (NAIVE, IM2COL, WINOGRADF63):
        assert _opts_call(_param(group=1), algo, _opts(dilation_h=2, dilation_w=2)) == -200, algo
    # a residual, which the depthwise kernels never add in their epilogue, and the pooling
    assert _opts_call(_param(), DEPTHWISE, _opts(residual=D, dilation_h=2, dilation_w=2)) == -200
    assert _opts_call(_param(CLIP), DEPTHWISE, _opts(residual=D, clip_min=0, clip_max=6, dilation_h=2, dilation_w=2)) == -200
    assert _opts_call(_param(), DEPTHWISE, _opts(pool=1, dilation_h=2, dilation_w=2)) == -200
    assert _opts_call(_param(), DEPTHWISE, _opts(dilation_h=-1, dilation_w=2)) == -100


def test_dilated_depthwise_needs_no_scratch():
    from feathercnn_b200._lib import fcuda
    s, k = ctypes.c_size_t(7), ctypes.c_size_t(0)
    assert fcuda().fcuda_conv_get_buffer_size(ctypes.byref(_param()), DEPTHWISE, 16, ctypes.byref(s), ctypes.byref(k)) == 0
    assert (s.value, k.value) == (0, 16 * 9)


# ---- models ----------------------------------------------------------------------------------------------------------
def _dilations(m):
    out = {}
    for line in m.lines:
        tok = line.split()
        if tok[0] == "ConvolutionDepthWise":
            kv = dict(t.split("=") for t in tok[6:])
            out[tok[1]] = (int(kv.get("2", 1)), int(kv.get("3", 1)), int(kv["1"]), int(kv["4"]))
    return out


@pytest.mark.parametrize("os_, feat", [(16, 33), (8, 65)])
def test_deeplabv3_mobilenet_v2_shapes(os_, feat):
    from feathercnn_b200.tools import modelgen
    m = modelgen.deeplabv3_mobilenet_v2(output_stride=os_)
    assert m.shape["data"] == (3, 513, 513)
    assert m.shape["aspp_in_a"] == (320, feat, feat)
    assert m.shape["image_pool"] == (320, 1, 1)
    assert m.shape["image_pool_up"] == (256, feat, feat)
    assert m.shape["aspp_concat"] == (512, feat, feat)
    assert m.shape["logits"] == (21, feat, feat)
    assert m.shape["logits_up"] == (21, 513, 513)
    d = _dilations(m)
    assert all(pad == dil for dil, _, _, pad in d.values())
    if os_ == 16:  # the 160 block's first depthwise at rate 1 and stride 1, the rest at 2
        assert d["conv7_1_dw"] == (1, 1, 3, 1) and m.shape["conv7_1_dw"] == (576, 33, 33)
        assert [d[n][0] for n in ("conv7_2_dw", "conv7_3_dw", "conv8_1_dw")] == [2, 2, 2]
        assert sum(v[0] > 1 for v in d.values()) == 3
    else:          # the 64 block at 1 then 2, the 160 block at 2 then 4
        assert d["conv5_1_dw"] == (1, 1, 3, 1) and [d[f"conv5_{i}_dw"][0] for i in (2, 3, 4)] == [2, 2, 2]
        assert [d[f"conv6_{i}_dw"][0] for i in (1, 2, 3)] == [2, 2, 2]
        assert d["conv7_1_dw"] == (2, 1, 3, 2) and [d[n][0] for n in ("conv7_2_dw", "conv7_3_dw", "conv8_1_dw")] == [4, 4, 4]
    assert all(stride == 1 for dil, stride, _, _ in d.values() if dil > 1)


def test_deeplabv3_tiny_takes_both_dilated_kernels():
    from feathercnn_b200.tools import modelgen
    m = modelgen.deeplabv3_tiny()
    assert m.shape["logits_up"] == (5, 65, 65)
    assert max(c for c, _, _ in m.shape.values()) <= 64
    d = _dilations(m)
    fast = {dil for dil, stride, k, _ in d.values() if dil > 1 and k == 3 and stride == 1}
    generic = [n for n, (dil, stride, k, _) in d.items() if dil > 1 and (k != 3 or stride != 1)]
    assert fast == {2, 4} and generic == ["conv6_1_dw"]


def test_deeplabv3_loads():
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    for m in (modelgen.deeplabv3_tiny(), modelgen.deeplabv3_mobilenet_v2(output_stride=8)):
        net = Net()
        net.LoadParamFromText("7767517\n" + f"{len(m.lines)} {len(m.blobs)}\n" + "\n".join(m.lines) + "\n")
        assert "logits_up" in net.BlobNames()


# ---- converter -------------------------------------------------------------------------------------------------------
def test_caffe_dilated_depthwise_converts_and_loads():
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import caffe2feather
    w = np.random.default_rng(0).standard_normal((4, 1, 3, 3)).astype(np.float32)
    conv_p = fint(1, 4) + fint(2, 0) + fint(3, 2) + fint(4, 3) + fint(5, 4) + fint(18, 2)  # pad 2, group 4, dilation 2
    model = (fbytes(3, b"data") + b"".join(fint(4, v) for v in (1, 4, 9, 9))
             + caffe_layer("dw", "DepthwiseConvolution", ["data"], ["dw"], [w], f106=conv_p)
             + caffe_layer("dwg", "Convolution", ["dw"], ["dwg"], [w], f106=conv_p))
    text, binary = caffe2feather.convert(model)
    for name, bottom in (("dw", "data"), ("dwg", "dw")):
        line = [l for l in text.splitlines() if l.split()[:2] == ["ConvolutionDepthWise", name]][0]
        kv = dict(t.split("=") for t in line.split()[6:])
        assert line.split()[4:6] == [bottom, name]
        assert (kv["0"], kv["1"], kv["2"], kv["4"], kv["7"], kv["6"]) == ("4", "3", "2", "2", "4", "36"), line
    assert binary == 2 * (b"\0\0\0\0" + w.tobytes())
    Net().LoadParamFromText(text)


# ---- SASS ------------------------------------------------------------------------------------------------------------
def test_dilated_kernels_have_no_local_memory():
    funcs = _functions()
    fast = _kernels(funcs, r"dw3x3_dilated_kernelILi[14]ELb[01]EE")
    assert len(fast) == 4, fast  # VEC 1 / 4 x ReLU / Clip
    for k in fast + _kernels(funcs, r"dw_generic_kernelILb[01]EE"):
        ops = collections.Counter(op for _, op, _ in funcs[k])
        assert ops["LDL"] == 0 and ops["STL"] == 0, (k, ops["LDL"], ops["STL"])
        assert not any(re.match(r"LDL|STL", op) for _, op, _ in funcs[k]), k
