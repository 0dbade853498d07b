"""Deconvolution / DeconvolutionDepthWise on the host (no kernel is launched): the geometry and plan of the C ABI against
a NumPy restatement of the layer's definition (include/fcuda.h), the loader's rejections, workspace sizes, the sub-pixel
decomposition in float64, the Caffe converter and the SASS of the two new kernels.

The helpers at the top (deconv_ref, equivalent_filter, scatter, plan_ref) are the definition the GPU tests hold the
kernels to."""
from __future__ import annotations

import ctypes
import re
import shutil
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_tools import blob as caffe_blob
from test_tools import fbytes, fint, layer as caffe_layer

ROOT = Path(__file__).resolve().parents[1]
NAIVE, IM2COL, SGECONV, DEPTHWISE = 0, 1, 2, 3


# ---- the definition ------------------------------------------------------------------------------------------------
def out_dim(h, k, s, d, pa, pb, op):
    return (h - 1) * s + d * (k - 1) + 1 + op - pa - pb


def deconv_ref(x, w, b, stride=(1, 1), pad=(0, 0, 0, 0), output_pad=(0, 0), dil=(1, 1), group=1, relu=False,
               absolute=False):
    """float64 ncnn Deconvolution through torch's conv_transpose2d.  w is (OC, IC/group, KH, KW) as ncnn stores it; pad is
    (top, bottom, left, right), output_pad (bottom, right).  absolute=True: the same on |x|, |w|, |b| (the scale S)."""
    x, w = torch.as_tensor(x).double(), torch.as_tensor(w).double()
    b = None if b is None else torch.as_tensor(b).double()
    if absolute:
        x, w, b = x.abs(), w.abs(), None if b is None else b.abs()
    oc, icg, kh, kw = w.shape
    ocg = oc // group
    wt = w.view(group, ocg, icg, kh, kw).transpose(1, 2).reshape(group * icg, ocg, kh, kw)
    y = F.conv_transpose2d(x, wt, None, stride=stride, dilation=dil, groups=group)
    y = F.pad(y, (0, output_pad[1], 0, output_pad[0]))
    if b is not None:
        y = y + b.view(1, -1, 1, 1)
    pt, pb, pl, pr = pad
    y = y[:, :, pt:y.shape[2] - pb, pl:y.shape[3] - pr]
    return y.clamp_min(0) if relu and not absolute else y


def deconv_scatter_form(x, w, b, stride, pad, output_pad, dil, group):
    """The definition written out literally: every product x[i][j] * w[ky][kx] lands on (i*s + ky*d, j*s + kx*d)."""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    n, ic, h, wd = x.shape
    oc, icg, kh, kw = w.shape
    ocg = oc // group
    (sh, sw), (dh, dw) = stride, dil
    hf, wf = (h - 1) * sh + dh * (kh - 1) + 1 + output_pad[0], (wd - 1) * sw + dw * (kw - 1) + 1 + output_pad[1]
    full = np.zeros((n, oc, hf, wf))
    for g in range(group):
        xs = x[:, g * icg:(g + 1) * icg]
        for ky in range(kh):
            for kx in range(kw):
                contrib = np.einsum("nihw,oi->nohw", xs, w[g * ocg:(g + 1) * ocg, :, ky, kx])
                full[:, g * ocg:(g + 1) * ocg, ky * dh:ky * dh + (h - 1) * sh + 1:sh, kx * dw:kx * dw + (wd - 1) * sw + 1:sw] += contrib
    if b is not None:
        full += np.asarray(b, np.float64).reshape(1, -1, 1, 1)
    pt, pb, pl, pr = pad
    return full[:, :, pt:hf - pb, pl:wf - pr]


def plan_ref(oc, ic, h, w, kh, kw, stride, pad, output_pad, dil, group):
    """(path, equivalent convolution as a dict) of include/fcuda.h's rule; path 'dw', 'direct' or 'subpixel'."""
    (sh, sw), (dh, dw) = stride, dil
    pt, pb, pl, pr = pad
    oph, opw = output_pad
    if group > 1 and group == ic and oc == ic:
        return "dw", None
    eh, ew = dh * (kh - 1), dw * (kw - 1)
    if sh == sw == 1 and max(pt, pb) <= eh and max(pl, pr) <= ew and oph <= pb and opw <= pr:
        return "direct", dict(output_channels=oc, kernel_h=kh, kernel_w=kw, pad_top=eh - pt, pad_bottom=eh - pb + oph,
                              pad_left=ew - pl, pad_right=ew - pr + opw, dil=(dh, dw),
                              output_h=out_dim(h, kh, sh, dh, pt, pb, oph), output_w=out_dim(w, kw, sw, dw, pl, pr, opw))
    th, tw = -(-kh // sh), -(-kw // sw)
    edh, edw = (dh if sh == 1 else 1), (dw if sw == 1 else 1)
    return "subpixel", dict(output_channels=oc * sh * sw, kernel_h=th, kernel_w=tw, pad_top=edh * (th - 1),
                            pad_bottom=edh * (th - 1), pad_left=edw * (tw - 1), pad_right=edw * (tw - 1), dil=(edh, edw),
                            output_h=h + edh * (th - 1), output_w=w + edw * (tw - 1))


def equivalent_filter(w, stride, group, path):
    """The filter of the equivalent convolution: flipped (direct path) or the sub-pixel phase filters
    W'[(g, ry, rx, oc)][ic][u][v] = w[g*OCg + oc][ic][ry + sh*(Th-1-u)][rx + sw*(Tw-1-v)], 0 past the kernel."""
    w = np.asarray(w, np.float32)
    if path == "direct":
        return np.ascontiguousarray(w[:, :, ::-1, ::-1])
    oc, icg, kh, kw = w.shape
    sh, sw = stride
    ocg = oc // group
    th, tw = -(-kh // sh), -(-kw // sw)
    wp = np.zeros((group, sh, sw, ocg, icg, th, tw), np.float32)
    wg = w.reshape(group, ocg, icg, kh, kw)
    for ry in range(sh):
        for rx in range(sw):
            for u in range(th):
                ky = ry + sh * (th - 1 - u)
                if ky >= kh:
                    continue
                for v in range(tw):
                    kx = rx + sw * (tw - 1 - v)
                    if kx < kw:
                        wp[:, ry, rx, :, :, u, v] = wg[:, :, :, ky, kx]
    return wp.reshape(group * sh * sw * ocg, icg, th, tw)


def scatter(P, oc, group, stride, pad, out_hw):
    """Phase planes P (N, OC', Hc, Wc) -> the cropped output (N, OC, OH, OW) before bias; zero where Y / s >= Hc."""
    P = torch.as_tensor(P)
    n, _, hc, wc = P.shape
    sh, sw = stride
    ocg = oc // group
    oh, ow = out_hw
    Y = torch.arange(oh, device=P.device) + pad[0]
    X = torch.arange(ow, device=P.device) + pad[2]
    ty, ry, tx, rx = Y // sh, Y % sh, X // sw, X % sw
    Pz = F.pad(P.view(n, group, sh, sw, ocg, hc, wc), (0, int(tx.max()) + 1, 0, int(ty.max()) + 1))  # zero rows past Hc
    Pz = Pz.permute(0, 1, 4, 2, 3, 5, 6)  # (n, g, oc, sh, sw, hc+, wc+)
    out = Pz[:, :, :, ry.view(-1, 1), rx.view(1, -1), ty.view(-1, 1), tx.view(1, -1)]
    return out.reshape(n, oc, oh, ow)


def equivalent_conv_ref(x, w, b, stride, pad, output_pad, dil, group):
    """float64: the equivalent convolution of plan_ref, then the scatter / bias of the plan's path."""
    oc, _, kh, kw = w.shape
    n, ic, h, wd = x.shape
    path, e = plan_ref(oc, ic, h, wd, kh, kw, stride, pad, output_pad, dil, group)
    wp = torch.from_numpy(equivalent_filter(w, stride, group, path)).double()
    xp = F.pad(torch.as_tensor(x).double(), (e["pad_left"], e["pad_right"], e["pad_top"], e["pad_bottom"]))
    y = F.conv2d(xp, wp, None, dilation=e["dil"], groups=group)
    if path == "subpixel":
        y = scatter(y, oc, group, stride, pad, (out_dim(h, kh, stride[0], dil[0], pad[0], pad[1], output_pad[0]),
                                                out_dim(wd, kw, stride[1], dil[1], pad[2], pad[3], output_pad[1])))
    return y if b is None else y + torch.as_tensor(b).double().view(1, -1, 1, 1)


# ---- geometry and plan against the library -------------------------------------------------------------------------
def _param(oc, ic, h, w, kh, kw, stride, pad, output_pad, dil, group, bias=True, relu=False):
    from feathercnn_b200._lib import FcudaDeconvParam
    return FcudaDeconvParam(output_channels=oc, input_channels=ic, input_h=h, input_w=w, kernel_h=kh, kernel_w=kw,
                            stride_h=stride[0], stride_w=stride[1], dilation_h=dil[0], dilation_w=dil[1], pad_left=pad[2],
                            pad_right=pad[3], pad_top=pad[0], pad_bottom=pad[1], output_pad_right=output_pad[1],
                            output_pad_bottom=output_pad[0], group=group, bias_term=int(bias), activation=int(relu))


def _random_geometry(rng):
    group = int(rng.choice([1, 1, 1, 2, 4]))
    dw = rng.random() < 0.2
    if dw:
        group = int(rng.choice([2, 8, 21]))
        ic = oc = group
    else:
        ic = group * int(rng.choice([1, 3, 8, 17, 32]))
        oc = group * int(rng.choice([1, 4, 13, 32]))
    h, w = (int(v) for v in rng.integers(1, 20, 2))
    kh, kw = (int(v) for v in rng.integers(1, 8, 2))
    stride = tuple(int(v) for v in rng.integers(1, 5, 2))
    dil = tuple(1 if s > 1 or rng.random() < 0.6 else int(rng.integers(2, 4)) for s in stride)
    pad = tuple(int(v) for v in rng.integers(0, 5, 4))
    output_pad = tuple(int(v) for v in rng.integers(0, 3, 2))
    return oc, ic, h, w, kh, kw, stride, pad, output_pad, dil, group


def test_output_dim_and_plan_follow_the_definition():
    from feathercnn_b200._lib import FcudaConvParam, fcuda
    lib = fcuda()
    rng = np.random.default_rng(7)
    paths = set()
    for _ in range(300):
        oc, ic, h, w, kh, kw, stride, pad, output_pad, dil, group = g = _random_geometry(rng)
        p = _param(*g)
        oh = out_dim(h, kh, stride[0], dil[0], pad[0], pad[1], output_pad[0])
        ow = out_dim(w, kw, stride[1], dil[1], pad[2], pad[3], output_pad[1])
        rc = lib.fcuda_deconv_output_dim(ctypes.byref(p))
        if oh <= 0 or ow <= 0:
            assert rc == -100, g
            continue
        assert rc == 0 and (p.output_h, p.output_w) == (oh, ow), g
        eq, algo = FcudaConvParam(), ctypes.c_int(-7)
        rc = lib.fcuda_deconv_plan(ctypes.byref(p), ctypes.byref(eq), ctypes.byref(algo))
        path, e = plan_ref(*g)
        paths.add(path)
        if path == "dw":
            assert rc == 0 and algo.value == DEPTHWISE, g
            continue
        assert rc == 0, (g, rc)
        for k in ("output_channels", "kernel_h", "kernel_w", "pad_top", "pad_bottom", "pad_left", "pad_right",
                  "output_h", "output_w"):
            assert getattr(eq, k) == e[k], (g, k, getattr(eq, k), e[k])
        assert (eq.input_channels, eq.input_h, eq.input_w, eq.stride_h, eq.stride_w, eq.group) == (ic, h, w, 1, 1, group)
        assert eq.bias_term == (1 if path == "direct" else 0) and eq.activation == 0
        if e["dil"] != (1, 1) or group > 1:
            assert algo.value == SGECONV, g
        else:
            tuned = ctypes.c_int(-1)
            assert lib.fcuda_conv_select_algo_tuned(ctypes.byref(eq), ctypes.byref(tuned)) == 0
            assert algo.value == tuned.value, g
    assert paths == {"dw", "direct", "subpixel"}


@pytest.mark.parametrize("fields, code", [
    (dict(pad=(-1, 0, 0, 0)), -200),
    (dict(output_pad=(0, -1)), -200),
    (dict(stride=(2, 1), dil=(2, 1)), -200),
    (dict(group=3), -200),                          # 8 channels in 3 groups
    (dict(relu=2), -200),
    (dict(h=1, pad=(1, 1, 0, 0), kh=1), -100),      # empty output
    (dict(h=0), -100),
])
def test_abi_rejections(fields, code):
    from feathercnn_b200._lib import fcuda
    a = dict(oc=8, ic=8, h=4, w=4, kh=3, kw=3, stride=(2, 2), pad=(1, 1, 1, 1), output_pad=(0, 0), dil=(1, 1), group=1)
    relu = fields.pop("relu", 0)
    a.update(fields)
    p = _param(**a)
    p.activation = relu
    assert fcuda().fcuda_deconv_output_dim(ctypes.byref(p)) == code


HEAD = "7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=8\n"


@pytest.mark.parametrize("params", [
    "0=8 1=3 3=2 6=576 20=9",            # output_w
    "0=8 1=3 3=2 6=576 21=9",            # output_h
    "0=8 1=3 3=2 4=-233 6=576",          # ncnn "same" padding
    "0=8 1=3 3=2 14=-234 6=576",
    "0=8 1=3 3=2 9=2 6=576",             # leaky ReLU
    "0=8 1=3 3=2 2=2 6=576",             # stride and dilation in one direction
    "0=8 1=3 3=2 8=1 6=576",             # int8
    "0=6 1=3 3=2 7=4 6=108",             # 6 outputs in 4 groups
])
def test_load_param_rejections(params):
    from feathercnn_b200.net import FeatherError, Net
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(HEAD + f"Deconvolution d 1 1 data out {params}\n")
    assert e.value.code == -200


@pytest.mark.parametrize("line", [
    "Deconvolution d 1 1 data out 0=8 1=4 3=2 4=1 5=1 6=1024 9=1",
    "Deconvolution d 1 1 data out 0=8 1=3 11=5 3=2 13=1 4=0 15=1 14=2 16=0 18=1 6=960",
    "DeconvolutionDepthWise d 1 1 data out 0=8 1=4 3=2 4=1 5=0 6=128 7=8",
    "DeconvolutionDepthWise d 1 1 data out 0=16 1=4 3=2 4=1 5=0 6=256 7=8",   # channel multiplier 2
    "Deconvolution d 1 1 data out 0=8 1=3 2=2 6=576",                        # stride 1, dilation 2
])
def test_load_param_accepts(line):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(HEAD + line + "\n")
    assert "out" in net.BlobNames()


@pytest.mark.parametrize("g", [
    (64, 32, 8, 8, 4, 4, (2, 2), (1, 1, 1, 1), (0, 0), (1, 1), 1),
    (16, 32, 9, 7, 3, 3, (2, 2), (1, 1, 1, 1), (1, 1), (1, 1), 1),
    (64, 64, 28, 28, 3, 3, (1, 1), (1, 1, 1, 1), (0, 0), (1, 1), 1),      # direct, Winograd
    (8, 8, 6, 6, 3, 3, (1, 1), (0, 0, 0, 0), (0, 0), (2, 2), 1),          # direct, dilated
    (16, 16, 6, 6, 4, 4, (2, 2), (1, 1, 1, 1), (0, 0), (1, 1), 4),        # grouped
    (21, 21, 16, 16, 16, 16, (8, 8), (4, 4, 4, 4), (0, 0), (1, 1), 21),   # depthwise
])
@pytest.mark.parametrize("batch", [1, 5])
def test_buffer_sizes(g, batch):
    from feathercnn_b200._lib import FcudaConvParam, fcuda
    lib = fcuda()
    p = _param(*g)
    assert lib.fcuda_deconv_output_dim(ctypes.byref(p)) == 0
    eq, algo = FcudaConvParam(), ctypes.c_int()
    assert lib.fcuda_deconv_plan(ctypes.byref(p), ctypes.byref(eq), ctypes.byref(algo)) == 0
    s, k = ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.fcuda_deconv_get_buffer_size(ctypes.byref(p), batch, ctypes.byref(s), ctypes.byref(k)) == 0
    path, _ = plan_ref(*g)
    if path == "dw":
        assert (s.value, k.value) == (0, g[1] * g[4] * g[5])
        return
    cs, ck, cs1 = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.fcuda_conv_get_buffer_size(ctypes.byref(eq), algo.value, batch, ctypes.byref(cs), ctypes.byref(ck)) == 0
    assert lib.fcuda_conv_get_buffer_size(ctypes.byref(eq), algo.value, 1, ctypes.byref(cs1), ctypes.byref(ck)) == 0
    phases = batch * eq.output_channels * eq.output_h * eq.output_w if path == "subpixel" else 0
    assert s.value == -(-cs.value // 64) * 64 + phases
    assert k.value == ck.value
    assert lib.fcuda_deconv_get_buffer_size(ctypes.byref(p), 0, ctypes.byref(s), ctypes.byref(k)) == -100


# ---- the decomposition in float64 -----------------------------------------------------------------------------------
DEF_CASES = [
    # (oc, ic, h, w, kh, kw, stride, pad, output_pad, dil, group)
    (5, 3, 4, 5, 4, 4, (2, 2), (1, 1, 1, 1), (0, 0), (1, 1), 1),
    (4, 6, 3, 4, 3, 3, (2, 2), (1, 1, 1, 1), (1, 1), (1, 1), 2),       # output_pad
    (3, 2, 4, 3, 5, 5, (3, 3), (0, 2, 1, 3), (0, 0), (1, 1), 1),       # four different pads
    (3, 2, 3, 3, 1, 1, (2, 2), (0, 0, 0, 0), (1, 1), (1, 1), 1),       # k < s: phases without taps
    (2, 2, 4, 4, 2, 3, (3, 2), (0, 1, 2, 0), (2, 1), (1, 1), 1),       # k < s on one axis, asymmetric crop
    (4, 3, 5, 5, 3, 3, (1, 1), (1, 1, 1, 1), (0, 0), (2, 2), 1),       # stride 1, dilated: direct
    (4, 3, 5, 5, 3, 3, (1, 1), (3, 0, 0, 1), (0, 0), (1, 1), 1),       # stride 1, pad > k-1: sub-pixel path
    (4, 4, 5, 5, 4, 4, (2, 2), (1, 1, 1, 1), (0, 0), (1, 1), 4),       # depthwise
    (8, 4, 5, 5, 3, 3, (2, 1), (1, 1, 1, 1), (0, 0), (1, 1), 4),       # channel multiplier
]


@pytest.mark.parametrize("g", DEF_CASES)
def test_definition_torch_scatter_form_and_decomposition_agree(g):
    oc, ic, h, w, kh, kw, stride, pad, output_pad, dil, group = g
    rng = np.random.default_rng(1)
    x = rng.uniform(-1, 1, (2, ic, h, w))
    wt = rng.standard_normal((oc, ic // group, kh, kw)).astype(np.float32)
    b = rng.uniform(-1, 1, oc)
    ref = deconv_ref(x, wt, b, stride, pad, output_pad, dil, group)
    assert ref.shape[2:] == (out_dim(h, kh, stride[0], dil[0], pad[0], pad[1], output_pad[0]),
                             out_dim(w, kw, stride[1], dil[1], pad[2], pad[3], output_pad[1]))
    np.testing.assert_allclose(deconv_scatter_form(x, wt, b, stride, pad, output_pad, dil, group), ref.numpy(),
                               rtol=1e-12, atol=1e-12)
    if plan_ref(oc, ic, h, w, kh, kw, stride, pad, output_pad, dil, group)[0] != "dw":
        np.testing.assert_allclose(equivalent_conv_ref(x, wt, b, stride, pad, output_pad, dil, group).numpy(), ref.numpy(),
                                   rtol=1e-12, atol=1e-12)
    if output_pad != (0, 0):  # output_pad rows hold the bias alone
        full = deconv_ref(x, wt, b, stride, (0, 0, 0, 0), output_pad, dil, group)
        np.testing.assert_array_equal(full[:, :, -1, :].numpy(), np.broadcast_to(b.reshape(1, -1, 1), full[:, :, -1, :].shape))


# ---- converter ----------------------------------------------------------------------------------------------------
def fcn_caffemodel(w1, b1, w2, group2, ic=8, hw=6):
    """Input -> Deconvolution k4 s2 p1 (group 1, bias) -> Deconvolution k4 s2 p1 (group2, no bias), Caffe layout."""
    p1 = fint(1, w1.shape[1]) + fint(2, 1) + fint(3, 1) + fint(4, 4) + fint(6, 2)
    p2 = fint(1, w2.shape[1] * group2) + fint(2, 0) + fint(3, 1) + fint(4, 4) + fint(6, 2) + fint(5, group2)
    return (fbytes(1, "fcn") + fbytes(3, "data") + b"".join(fint(4, d) for d in (1, ic, hw, hw))
            + caffe_layer("up1", "Deconvolution", ["data"], ["up1"], [w1, b1], f106=p1)
            + caffe_layer("up2", "Deconvolution", ["up1"], ["up2"], [w2], f106=p2))


def caffe_to_ncnn(w, group):
    """Caffe's (IC, OC/group, kh, kw) -> ncnn's [group][OC/group][IC/group][kh][kw]."""
    ic, ocg, kh, kw = w.shape
    return w.reshape(group, ic // group, ocg, kh, kw).transpose(0, 2, 1, 3, 4)


def test_caffe_deconvolution_converts():
    from feathercnn_b200.tools import caffe2feather
    rng = np.random.default_rng(3)
    w1 = rng.standard_normal((8, 12, 4, 4)).astype(np.float32)     # IC 8 -> OC 12
    b1 = rng.uniform(-1, 1, 12).astype(np.float32)
    w2 = rng.standard_normal((12, 2, 4, 4)).astype(np.float32)     # IC 12 -> OC 8 in 4 groups
    text, blob_bytes = caffe2feather.convert(fcn_caffemodel(w1, b1, w2, 4))
    lines = text.splitlines()
    assert lines[3] == "Deconvolution up1 1 1 data up1 0=12 1=4 11=4 2=1 12=1 3=2 13=2 4=1 14=1 5=1 6=1536"
    assert lines[4] == "DeconvolutionDepthWise up2 1 1 up1 up2 0=8 1=4 11=4 2=1 12=1 3=2 13=2 4=1 14=1 5=0 6=384 7=4"
    flag = struct.pack("<I", 0)
    want = flag + caffe_to_ncnn(w1, 1).tobytes() + b1.tobytes() + flag + caffe_to_ncnn(w2, 4).tobytes()
    assert blob_bytes == want
    # the reordering is the one the definition needs: ncnn weights through deconv_ref == torch on Caffe's weights as-is
    x = rng.uniform(-1, 1, (1, 12, 3, 3))
    ours = deconv_ref(x, caffe_to_ncnn(w2, 4).reshape(8, 3, 4, 4), None, (2, 2), (1, 1, 1, 1), group=4)
    theirs = F.conv_transpose2d(torch.from_numpy(x), torch.from_numpy(w2).double(), None, 2, 1, groups=4)
    np.testing.assert_allclose(ours.numpy(), theirs.numpy(), rtol=1e-12, atol=1e-12)
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(text)
    assert {"up1", "up2"} <= set(net.BlobNames())


def test_decoder_tiny_loads():
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.decoder_tiny()
    text = "7767517\n" + f"{len(m.lines)} {len(m.blobs)}\n" + "\n".join(m.lines) + "\n"
    assert sum(l.startswith("Deconvolution ") for l in m.lines) == 2
    assert sum(l.startswith("DeconvolutionDepthWise ") for l in m.lines) == 1
    assert m.shape["upscore"] == (4, 64, 64)
    net = Net()
    net.LoadParamFromText(text)
    assert sorted(net.BlobNames()) == sorted(m.blobs)


# ---- SASS -----------------------------------------------------------------------------------------------------------
EXISTING_PATTERNS = [r"conv_igemm_kernelILi(32|64|128)ELi[123]E", r"tensor_gemm_(pipe_)?kernel", r"wino_(in|out)put_kernel"]


def test_new_kernels_are_cuda_core_and_match_no_existing_pattern():
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    so = ROOT / "feathercnn_b200" / "lib" / "libfcuda.so"
    sass = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True, check=True).stdout
    ops: dict[str, dict[str, int]] = {}
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            ops[cur] = {}
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
        if m and cur:
            ops[cur][m.group(1)] = ops[cur].get(m.group(1), 0) + 1
    new = [k for k in ops if "deconv_" in k]
    assert any("deconv_scatter_kernel" in k for k in new) and any("deconv_dw_gather_kernel" in k for k in new), new
    for k in new:
        assert not any(re.search(p, k) for p in EXISTING_PATTERNS), k
        assert ops[k].get("HGMMA", 0) == 0 and ops[k].get("HMMA", 0) == 0, k
    gather = next(k for k in new if "deconv_dw_gather_kernel" in k)
    assert ops[gather].get("FFMA", 0) >= 1
