"""Interp and Crop on the host (no kernel is launched): the C ABI's output sizes against a restatement of ncnn's fp32
rules over random shapes, every rejection of the ABI and the loader, the Caffe converter on an FCN-8s-style model, the
pad arithmetic that folds a Crop into a deconvolution, and which crops Net::ApplyFusion folds.

The helpers at the top (nearest_scale, nearest_index, interp_out_dim, fold_pads, crop_caffemodel) are the definitions
the GPU tests hold the kernels and the Net to."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from test_deconv_host import _param as deconv_param
from test_deconv_host import deconv_ref
from test_tools import fbytes, fint, layer as caffe_layer


# ---- the definitions -----------------------------------------------------------------------------------------------
def interp_out_dim(h, w, out_height, out_width, hs, ws):
    """ncnn: the explicit size when both are set, else (int)(h * height_scale) with an fp32 product."""
    if out_height > 0 and out_width > 0:
        return out_height, out_width
    return int(np.float32(h) * np.float32(hs)), int(np.float32(w) * np.float32(ws))


def nearest_scale(n_in, out, explicit_out, scale):
    """hs = output_height ? in / (float)out : 1.f / height_scale, in fp32."""
    return np.float32(n_in) / np.float32(out) if explicit_out else np.float32(1) / np.float32(scale)


def nearest_index(out, n_in, scale):
    """min((int)(d * hs), in - 1) with the fp32 product."""
    return np.minimum((np.arange(out, dtype=np.float32) * np.float32(scale)).astype(np.int64), n_in - 1)


def fold_pads(pads, full_hw, hoff, woff, out_hw):
    """(top, bottom, left, right) of a deconvolution whose (full_h, full_w) output is cropped to out_hw at (hoff, woff)."""
    pt, pb, pl, pr = pads
    return (pt + hoff, pb + full_hw[0] - hoff - out_hw[0], pl + woff, pr + full_hw[1] - woff - out_hw[1])


def _interp_param(rt=2, align=0, hs=1.0, ws=1.0, oh=0, ow=0, h=8, w=8):
    from feathercnn_b200._lib import FcudaInterpParam
    return FcudaInterpParam(resize_type=rt, align_corner=align, height_scale=hs, width_scale=ws, output_height=oh,
                            output_width=ow, input_h=h, input_w=w)


# ---- C ABI ----------------------------------------------------------------------------------------------------------
def test_interp_output_dim_follows_the_fp32_rule():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    rng = np.random.default_rng(17)
    truncated = 0
    for _ in range(400):
        h, w = (int(v) for v in rng.integers(1, 300, 2))
        rt = int(rng.choice([1, 2]))
        hs, ws = (float(np.float32(v)) for v in rng.choice([0.3, 0.5, 1 / 3, 2.0, 2.5, 8.0, 1.7, 0.1], 2))
        oh, ow = (int(v) if rng.random() < 0.4 else 0 for v in rng.integers(1, 600, 2))
        p = _interp_param(rt, int(rng.integers(0, 2)), hs, ws, oh, ow, h, w)
        want = interp_out_dim(h, w, oh, ow, hs, ws)
        rc = lib.fcuda_interp_output_dim(ctypes.byref(p))
        if min(want) <= 0:
            assert rc == -100, (h, w, hs, ws, oh, ow)
            continue
        assert rc == 0 and (p.output_h, p.output_w) == want, (h, w, hs, ws, oh, ow)
        truncated += int(not (oh and ow) and want[0] != int(round(h * hs)))
    assert truncated > 0  # some products were truncated, not rounded
    # the fp32 product, not the double one: 10 * fl32(0.7) is 6.99999988 in double, which fp32 rounds to 7
    p = _interp_param(2, 0, float(np.float32(0.7)), 1.0, 0, 0, 10, 10)
    assert int(10 * float(np.float32(0.7))) == 6
    assert lib.fcuda_interp_output_dim(ctypes.byref(p)) == 0 and p.output_h == 7


@pytest.mark.parametrize("fields, code", [
    (dict(rt=0), -200),
    (dict(rt=3), -200),
    (dict(hs=0.0), -100),
    (dict(ws=-2.0), -100),
    (dict(hs=0.05), -100),                          # (int)(8 * 0.05) == 0: empty output
    (dict(h=0), -100),
    (dict(oh=-1, ow=4), -100),
    (dict(rt=1, hs=0.0, oh=0, ow=16), -100),        # nearest reads 1 / height_scale without output_height
])
def test_interp_abi_rejections(fields, code):
    from feathercnn_b200._lib import fcuda
    p = _interp_param(**fields)
    assert fcuda().fcuda_interp_output_dim(ctypes.byref(p)) == code
    assert fcuda().fcuda_interp_forward(ctypes.byref(p), None, None, 1, 1, None) == code


def test_bilinear_with_explicit_size_ignores_the_scales():
    from feathercnn_b200._lib import fcuda
    p = _interp_param(2, 0, 0.0, -1.0, 24, 40)
    assert fcuda().fcuda_interp_output_dim(ctypes.byref(p)) == 0 and (p.output_h, p.output_w) == (24, 40)


@pytest.mark.parametrize("args", [
    (3, 8, 8, 0, 0, 1, 3, 8, 8),   # woff + out_w > in_w
    (3, 8, 8, 0, 5, 0, 3, 4, 8),
    (3, 8, 8, 1, 0, 0, 3, 8, 8),   # coff + out_c > channels
    (3, 8, 8, -1, 0, 0, 1, 8, 8),
    (3, 8, 8, 0, 0, 0, 3, 0, 8),   # empty
])
def test_crop_abi_rejects_windows_outside_the_input(args):
    from feathercnn_b200._lib import fcuda
    c, h, w, co, ho, wo, oc, oh, ow = args
    assert fcuda().fcuda_crop_forward(None, None, c, h, w, co, ho, wo, oc, oh, ow, 1, None) == -100


def test_nearest_rule_matches_torch_for_integer_scales():
    for n_in, out in ((4, 8), (3, 24), (5, 15), (7, 7)):
        got = nearest_index(out, n_in, nearest_scale(n_in, out, out, 1.0))
        src = torch.nn.functional.interpolate(torch.arange(n_in, dtype=torch.float32).view(1, 1, 1, -1), size=(1, out),
                                              mode="nearest").view(-1).long().numpy()
        assert np.array_equal(got, src), (n_in, out)


# ---- loader ---------------------------------------------------------------------------------------------------------
HEAD = "7767517\n{n} {b}\nInput data 0 1 data 0=8 1=8 2=3\n"


@pytest.mark.parametrize("line", [
    "Interp i 1 1 data out 0=2 5=1",                    # dynamic_target_size
    "Interp i 1 1 data out",                            # resize_type 0 (ncnn's default)
    "Interp i 1 1 data out 0=0 1=2.0 2=2.0",
    "Interp i 1 1 data out 0=3 1=2.0 2=2.0",            # bicubic
    "Interp i 2 1 data data out 0=2 3=4 4=4",           # a second bottom
    "Crop c 1 1 data out 6=1",                          # end offsets
    "Crop c 1 1 data out 7=1",
    "Crop c 1 1 data out 8=1",
    "Crop c 1 1 data out -23309=1,2",                   # starts / ends / axes
    "Crop c 1 1 data out -23310=1,4",
    "Crop c 1 1 data out -23311=1,0",
    "Crop c 1 1 data out 0=-1",
])
def test_load_param_rejections(line):
    from feathercnn_b200.net import FeatherError, Net
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(HEAD.format(n=2, b=2) + line + "\n")
    assert e.value.code == -200


@pytest.mark.parametrize("line", [
    "Interp i 1 1 data out 0=1 1=2.000000e+00 2=3.0",
    "Interp i 1 1 data out 0=2 3=16 4=24 6=1",
    "Crop c 1 1 data out 0=1 1=2",
    "Crop c 1 1 data out 0=1 1=2 2=1 3=4 4=5 5=2",
    "Crop c 2 1 data data out 0=3 1=3",
])
def test_load_param_accepts(line):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(HEAD.format(n=2, b=2) + line + "\n")
    assert "out" in net.BlobNames()


# ---- the fold -------------------------------------------------------------------------------------------------------
FOLD_CASES = [
    # (ic, oc, h, w, k, stride, pads (t, b, l, r), group, hoff, woff, out_hw)
    (4, 3, 5, 6, 4, (2, 2), (1, 1, 1, 1), 1, 1, 2, (6, 7)),
    (3, 3, 4, 4, 16, (8, 8), (0, 0, 0, 0), 3, 9, 5, (20, 31)),
    (2, 5, 3, 7, 3, (2, 3), (0, 2, 1, 0), 1, 0, 4, (4, 10)),
    (6, 6, 5, 5, 3, (1, 1), (0, 0, 0, 0), 6, 1, 1, (5, 5)),        # stride 1, depthwise
]


@pytest.mark.parametrize("g", FOLD_CASES)
def test_fold_pads_are_the_crop(g):
    from feathercnn_b200._lib import fcuda
    ic, oc, h, w, k, stride, pads, group, hoff, woff, out_hw = g
    rng = np.random.default_rng(2)
    x = rng.uniform(-1, 1, (2, ic, h, w))
    wt = rng.standard_normal((oc, ic // group, k, k))
    b = rng.uniform(-1, 1, oc)
    full = deconv_ref(x, wt, b, stride, pads, group=group)
    folded = fold_pads(pads, full.shape[2:], hoff, woff, out_hw)
    want = full[:, :, hoff:hoff + out_hw[0], woff:woff + out_hw[1]]
    assert want.shape[2:] == out_hw
    assert torch.equal(deconv_ref(x, wt, b, stride, folded, group=group), want)
    p = deconv_param(oc, ic, h, w, k, k, stride, folded, (0, 0), (1, 1), group)
    assert fcuda().fcuda_deconv_output_dim(ctypes.byref(p)) == 0 and (p.output_h, p.output_w) == out_hw


def _fused_away(lines, layers):
    from feathercnn_b200.net import Net
    blobs = {t for l in lines for t in l.split()[4 + int(l.split()[2]):4 + int(l.split()[2]) + int(l.split()[3])]}
    net = Net(fusion=True)
    net.LoadParamFromText("7767517\n" + f"{len(lines)} {len(blobs)}\n" + "\n".join(lines) + "\n")
    net.FuseNow()
    return {n: net.LayerFusedAway(n) for n in layers}


def test_fusion_folds_only_crops_of_unshared_deconvolution_tops():
    from feathercnn_b200.tools import modelgen
    m = modelgen.fcn8s_tiny()
    assert _fused_away(m.lines, ["score", "score_pool4c", "score_pool3c", "upscore8"]) == \
        {"score": 1, "score_pool4c": 0, "score_pool3c": 0, "upscore8": 0}
    inp = "Input data 0 1 data 0=8 1=8 2=4"
    dec = "Deconvolution up 1 1 {b} up 0=4 1=4 3=2 4=1 6=256"
    cases = {
        # one bottom, whole channels: folded
        "one_bottom": ([inp, dec.format(b="data"), "Crop c 1 1 up out 0=1 1=1 3=8 4=8"], 1),
        # a channel crop stays a layer
        "channels": ([inp, dec.format(b="data"), "Crop c 1 1 up out 2=1"], 0),
        # stride 1 (not depthwise) keeps its Crop: the folded pads could leave the direct path
        "stride1": ([inp, "Deconvolution up 1 1 data up 0=4 1=3 6=144", "Crop c 1 1 up out 0=1 1=1"], 0),
        # the reference is produced after the deconvolution
        "late_reference": ([inp, "Split s 1 2 data d0 d1", dec.format(b="d0"),
                            "Convolution r 1 1 d1 ref 0=4 1=1 6=16", "Crop c 2 1 up ref out 0=1 1=1"], 0),
        # the deconvolution's top has a second reader
        "shared": ([inp, dec.format(b="data"), "Split s 1 2 up u0 u1", "Crop c 1 1 u0 out 0=1 1=1"], 0),
        # a ReLU fused first, then the Crop
        "after_relu": ([inp, dec.format(b="data"), "ReLU r 1 1 up upr", "Crop c 2 1 upr data out 0=2 1=2"], 1),
    }
    for name, (lines, want) in cases.items():
        assert _fused_away(lines, ["c"])["c"] == want, name


def test_zoo_entries():
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.fcn8s_tiny()
    assert m.shape["score"] == (5, 64, 64) and m.shape["upscore8"] == (5, 120, 120)
    assert sum(l.startswith("Crop ") for l in m.lines) == 3
    assert [l for l in m.lines if l.startswith("Crop score ")] == ["Crop score 2 1 upscore8 data score 0=27 1=27"]
    assert modelgen.fcn8s_tiny(size=500, classes=21).shape["score"] == (21, 500, 500)
    d = modelgen.deeplab_head_tiny()
    assert d.shape["upsample"] == (5, 32, 32)
    assert "Interp upsample 1 1 classifier upsample 0=2 1=8.000000e+00 2=8.000000e+00" in d.lines
    assert any(" 2=2" in l and l.startswith("Convolution aspp ") for l in d.lines)
    for mw in (m, d):
        net = Net()
        net.LoadParamFromText("7767517\n" + f"{len(mw.lines)} {len(mw.blobs)}\n" + "\n".join(mw.lines) + "\n")
        assert sorted(net.BlobNames()) == sorted(mw.blobs)


# ---- converter ------------------------------------------------------------------------------------------------------
def _conv_param(num_output, k, stride=1, pad=0, bias=True, group=1):
    p = fint(1, num_output) + fint(2, int(bias)) + fint(3, pad) + fint(4, k) + fint(6, stride)
    return p + (fint(5, group) if group > 1 else b"")


def crop_caffemodel(rng):
    """An FCN-8s-style Caffe model on a (4, 16, 16) input: two strided convolutions (the first padded by 10), a score
    convolution, a k4 s2 deconvolution, a skip score cropped to it (offset 1) and summed, a k4 s2 depthwise
    deconvolution and a crop back to the input (offset 9).  Returns (caffemodel bytes, weights)."""
    ws = {
        "c1": (rng.standard_normal((8, 4, 3, 3)) * 0.3).astype(np.float32), "c1_b": rng.uniform(-.1, .1, 8).astype(np.float32),
        "c2": (rng.standard_normal((8, 8, 5, 5)) * 0.1).astype(np.float32), "c2_b": rng.uniform(-.1, .1, 8).astype(np.float32),
        "score_fr": (rng.standard_normal((3, 8, 1, 1)) * 0.5).astype(np.float32),
        "score_fr_b": rng.uniform(-.1, .1, 3).astype(np.float32),
        "upscore2": (rng.standard_normal((3, 3, 4, 4)) * 0.3).astype(np.float32),     # Caffe (IC, OC, k, k)
        "score_c1": (rng.standard_normal((3, 8, 1, 1)) * 0.2).astype(np.float32),
        "score_c1_b": rng.uniform(-.1, .1, 3).astype(np.float32),
        "upscore": (rng.standard_normal((3, 1, 4, 4)) * 0.3).astype(np.float32),      # 3 groups
    }
    crop = lambda off: fint(1, 2) + fint(2, off)  # noqa: E731  CropParameter: axis 2, one offset
    model = (fbytes(1, "fcn8s") + fbytes(3, "data") + b"".join(fint(4, d) for d in (1, 4, 16, 16))
             + caffe_layer("c1", "Convolution", ["data"], ["c1"], [ws["c1"], ws["c1_b"]], f106=_conv_param(8, 3, 2, 10))
             + caffe_layer("c2", "Convolution", ["c1"], ["c2"], [ws["c2"], ws["c2_b"]], f106=_conv_param(8, 5, 2))
             + caffe_layer("score_fr", "Convolution", ["c2"], ["score_fr"], [ws["score_fr"], ws["score_fr_b"]],
                           f106=_conv_param(3, 1))
             + caffe_layer("upscore2", "Deconvolution", ["score_fr"], ["upscore2"], [ws["upscore2"]],
                           f106=_conv_param(3, 4, 2, bias=False))
             + caffe_layer("score_c1", "Convolution", ["c1"], ["score_c1"], [ws["score_c1"], ws["score_c1_b"]],
                           f106=_conv_param(3, 1))
             + caffe_layer("score_c1c", "Crop", ["score_c1", "upscore2"], ["score_c1c"], f144=crop(1))
             + caffe_layer("fuse", "Eltwise", ["upscore2", "score_c1c"], ["fuse"])
             + caffe_layer("upscore", "Deconvolution", ["fuse"], ["upscore"], [ws["upscore"]],
                           f106=_conv_param(3, 4, 2, bias=False, group=3))
             + caffe_layer("score", "Crop", ["upscore", "data"], ["score"], f144=crop(9)))
    return model, ws


def test_caffe_crop_converts():
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import caffe2feather
    text, _ = caffe2feather.convert(crop_caffemodel(np.random.default_rng(0))[0])
    crops = [l for l in text.splitlines() if l.startswith("Crop ")]
    assert crops == ["Crop score_c1c 2 1 score_c1 upscore2_splitncnn_0 score_c1c 0=1 1=1",
                     "Crop score 2 1 upscore data_splitncnn_1 score 0=9 1=9"]
    net = Net(fusion=True)
    net.LoadParamFromText(text)
    assert {"score_c1c", "score"} <= set(net.BlobNames())
    net.FuseNow()
    assert (net.LayerFusedAway("score"), net.LayerFusedAway("score_c1c")) == (1, 0)


def _one_crop(crop_param):
    w = np.ones((2, 3, 1, 1), np.float32)
    return (fbytes(1, "n") + fbytes(3, "data") + b"".join(fint(4, d) for d in (1, 3, 8, 8))
            + caffe_layer("conv", "Convolution", ["data"], ["conv"], [w], f106=_conv_param(2, 1, bias=False))
            + caffe_layer("crop", "Crop", ["conv", "data"], ["crop"], f144=crop_param))


@pytest.mark.parametrize("param, want", [
    (b"", "0=0 1=0"),                                         # axis 2, offset 0
    (fint(2, 3), "0=3 1=3"),                                  # one offset for both axes
    (fint(2, 1) + fint(2, 5), "0=5 1=1"),                     # (h, w)
    (fint(1, 3) + fint(2, 7), "0=7 1=0"),                     # axis 3: width only
    (fint(1, (1 << 64) - 2) + fint(2, 4), "0=4 1=4"),         # axis -2 == 2
])
def test_caffe_crop_axes_and_offsets(param, want):
    from feathercnn_b200.tools import caffe2feather
    text, _ = caffe2feather.convert(_one_crop(param))
    assert text.splitlines()[-1] == f"Crop crop 2 1 conv data_splitncnn_1 crop {want}"


@pytest.mark.parametrize("param", [fint(1, 1), fint(1, 0), fint(2, 1) + fint(2, 2) + fint(2, 3)])
def test_caffe_crop_rejects_channel_and_batch_axes(param):
    from feathercnn_b200.tools import caffe2feather
    with pytest.raises(ValueError):
        caffe2feather.convert(_one_crop(param))
