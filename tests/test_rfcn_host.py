"""R-FCN's PSROIPooling on the host (no kernel is launched): the NumPy definition the GPU tests hold the kernel to, checked
by hand; the loader's and the C ABI's rejections (every call here fails its checks before a launch); the blob shapes and
written parameters of modelgen's R-FCN models; and the models the shared ResNet-50 trunk and RPN builders also write,
byte for byte as before those builders were shared.

psroi_pooling_ref is the definition tests/test_gpu_rfcn.py holds the kernel to (include/fcuda.h states it)."""
from __future__ import annotations

import ctypes
import hashlib
import math

import numpy as np
import pytest

from test_faster_rcnn_host import FAKE, HEAD, _load

F = np.float32


# ---- the definition -------------------------------------------------------------------------------------------------
def _roundf(v):
    """roundf, half away from zero, of a float32: exact in float64 and representable in float32."""
    v = np.float64(v)
    return F(np.sign(v) * np.floor(np.abs(v) + 0.5))


def _edge(v, hi):
    """(int) of a float32 floor / ceil, converted saturating with NaN -> 0, then clamped to [0, hi]."""
    v = float(v)
    return 0 if math.isnan(v) else int(min(max(v, 0.0), hi))


def psroi_bins(roi, pooled_h, pooled_w, spatial_scale, h, w):
    """Bin edges of one RoI: (hs, he, ws, we) int arrays of shape (pooled_h, pooled_w), float32 operation by operation."""
    s = F(spatial_scale)
    x1, y1 = _roundf(F(roi[0])) * s, _roundf(F(roi[1])) * s
    x2, y2 = _roundf(F(roi[2]) + F(1)) * s, _roundf(F(roi[3]) + F(1)) * s
    with np.errstate(invalid="ignore", over="ignore"):
        bin_w = np.fmax(x2 - x1, F(0.1)) / F(pooled_w)
        bin_h = np.fmax(y2 - y1, F(0.1)) / F(pooled_h)
        hs = [_edge(np.floor(y1 + F(p) * bin_h), h) for p in range(pooled_h)]
        he = [_edge(np.ceil(y1 + F(p + 1) * bin_h), h) for p in range(pooled_h)]
        ws = [_edge(np.floor(x1 + F(p) * bin_w), w) for p in range(pooled_w)]
        we = [_edge(np.ceil(x1 + F(p + 1) * bin_w), w) for p in range(pooled_w)]
    return hs, he, ws, we


def psroi_pooling_ref(x, rois, pooled_h, pooled_w, output_dim, spatial_scale):
    """x (N, output_dim * pooled_h * pooled_w, H, W) float32, rois (N, R, 4) -> (N * R, output_dim, pooled_h, pooled_w).
    Each bin is summed in row-major order from 0.f, one float32 addition at a time (np.add.accumulate is sequential;
    np.sum would add pairwise), then divided by its area."""
    x = np.asarray(x, np.float32)
    n, c, h, w = x.shape
    assert c == output_dim * pooled_h * pooled_w, (c, output_dim, pooled_h, pooled_w)
    rois = np.asarray(rois, np.float32).reshape(n, -1, 4)
    r_ = rois.shape[1]
    maps = x.reshape(n, output_dim, pooled_h, pooled_w, h, w)
    out = np.zeros((n * r_, output_dim, pooled_h, pooled_w), np.float32)
    zero = np.zeros((output_dim, 1), np.float32)
    for i in range(n):
        for r in range(r_):
            hs, he, ws, we = psroi_bins(rois[i, r], pooled_h, pooled_w, spatial_scale, h, w)
            for ph in range(pooled_h):
                for pw in range(pooled_w):
                    if he[ph] <= hs[ph] or we[pw] <= ws[pw]:
                        continue
                    block = maps[i, :, ph, pw, hs[ph]:he[ph], ws[pw]:we[pw]].reshape(output_dim, -1)
                    total = np.add.accumulate(np.concatenate([zero, block], 1), axis=1, dtype=np.float32)[:, -1]
                    out[i * r_ + r, :, ph, pw] = total / F((he[ph] - hs[ph]) * (we[pw] - ws[pw]))
    return out


# ---- the definition, by hand ----------------------------------------------------------------------------------------
def _planes(c, h, w):
    """Plane k of a (1, c, h, w) map holds 100 k + its row-major pixel index."""
    return (np.arange(h * w, dtype=np.float32).reshape(1, 1, h, w) + 100 * np.arange(c, dtype=np.float32)[None, :, None,
                                                                                                           None])


def test_known_bins():
    """A 4 x 4 map, RoI (0, 0, 3, 3) at scale 1: x2 = y2 = round(3 + 1) = 4, roi 4 x 4, 2 x 2 bins of 2 x 2 pixels; bin
    (ph, pw) reads plane 2 ph + pw.  Means: plane 0 {0, 1, 4, 5}, plane 1 100 + {2, 3, 6, 7}, plane 2 200 + {8, 9, 12,
    13}, plane 3 300 + {10, 11, 14, 15}."""
    out = psroi_pooling_ref(_planes(4, 4, 4), [[[0, 0, 3, 3]]], 2, 2, 1, 1.0)
    assert out.tolist() == [[[[2.5, 104.5], [210.5, 312.5]]]]
    # .5 corners round half away from zero: (0.5, 0.5, 2.49, 2.5) -> x1 = y1 = 1, x2 = round(3.49) = 3, y2 = round(3.5) = 4
    hs, he, ws, we = psroi_bins([0.5, 0.5, 2.49, 2.5], 1, 1, 1.0, 8, 8)
    assert (hs, he, ws, we) == ([1], [4], [1], [3])


def test_empty_bin_and_roi_partly_outside():
    """RoI (-8, 0, 3, 3) on a 4 x 4 map, 1 x 2 bins: x1 = -8, x2 = 4, bin_w = 6.  Bin 0 spans [-8, -2): clamped to [0, 0),
    empty, 0.  Bin 1 spans [-2, 4), clamped to columns 0-3: the whole map, mean 7.5 of plane 1 (+ 100)."""
    out = psroi_pooling_ref(_planes(2, 4, 4), [[[-8, 0, 3, 3]]], 1, 2, 1, 1.0)
    assert out.tolist() == [[[[0.0, 107.5]]]]
    # wholly outside: every bin is empty
    assert np.all(psroi_pooling_ref(_planes(4, 4, 4), [[[-10, 0, -5, 3], [9, 9, 20, 20]]], 2, 2, 1, 1.0) == 0)


def test_width_floor():
    """RoI (5, 0, 2, 3): x2 = 3 < x1 = 5, so roi_w = 0.1 and the one bin spans [5, 5.1): column 5 of rows 0-3 of an 8 x 8
    map, {5, 13, 21, 29}, mean 17."""
    hs, he, ws, we = psroi_bins([5, 0, 2, 3], 1, 1, 1.0, 8, 8)
    assert (hs, he, ws, we) == ([0], [4], [5], [6])
    assert psroi_pooling_ref(_planes(1, 8, 8), [[[5, 0, 2, 3]]], 1, 1, 1, 1.0).ravel().tolist() == [17.0]
    # at 1/16 a 0-wide RoI is 1 / 16 wide before the floor: (5, 5, 5, 5) -> x1 = 0.3125, x2 = 0.375
    s = F(1 / 16)
    assert np.fmax(_roundf(F(6)) * s - _roundf(F(5)) * s, F(0.1)) == F(0.1)


def test_padding_row():
    """Proposal's [0, 0, 0, 0] padding row at 1/16: x1 = 0, x2 = 1/16, roi 0.1 x 0.1, every 7 x 7 bin is pixel (0, 0) of
    its own plane."""
    x = np.random.default_rng(0).standard_normal((1, 2 * 49, 5, 6)).astype(np.float32)
    out = psroi_pooling_ref(x, [[[0, 0, 0, 0]]], 7, 7, 2, 1 / 16)
    assert np.array_equal(out[0], x[0, :, 0, 0].reshape(2, 7, 7))


def test_non_square_channel_order():
    """pooled 2 x 3, output_dim 2 on a 4 x 6 map whose plane c is the constant c: RoI (0, 0, 5, 3) gives 2 x 2 bins, and
    output (q, ph, pw) is channel (q * 2 + ph) * 3 + pw."""
    x = np.broadcast_to(np.arange(12, dtype=np.float32)[None, :, None, None], (1, 12, 4, 6))
    out = psroi_pooling_ref(x, [[[0, 0, 5, 3]]], 2, 3, 2, 1.0)
    assert out[0].tolist() == [[[0, 1, 2], [3, 4, 5]], [[6, 7, 8], [9, 10, 11]]]


def test_sum_is_sequential():
    """A 2 x 2 bin of (2^24, 1, 1, 1): each + 1 after 2^24 rounds back to 2^24 (a tie, to even), so the sequential sum is
    2^24 and the mean 2^22; adding the ones first would give 2^24 + 4."""
    x = np.array([[[[2 ** 24, 1], [1, 1]]]], np.float32)
    assert psroi_pooling_ref(x, [[[0, 0, 1, 1]]], 1, 1, 1, 1.0).ravel().tolist() == [2.0 ** 22]
    assert F(2 ** 24) + (F(1) + F(1) + F(1)) != F(2 ** 24)


def test_nan_corner_reads_as_zero():
    """A NaN corner makes x1 NaN; floorf / ceilf keep it NaN and the saturating conversion makes it 0."""
    assert _edge(np.floor(F(np.nan)), 10) == 0 and _edge(F(np.inf), 10) == 10 and _edge(F(-np.inf), 10) == 0


# ---- layer ----------------------------------------------------------------------------------------------------------
PS = "PSROIPooling p 2 1 f s out"


@pytest.mark.parametrize("line", [
    PS, f"{PS} 3=0", f"{PS} 3=-1", f"{PS} 0=0 3=2", f"{PS} 1=0 3=2", f"{PS} 2=0 3=2", f"{PS} 2=-0.0625 3=2",
    "PSROIPooling p 1 1 f out 3=2", "PSROIPooling p 3 1 f s b out 3=2",
])
def test_loader_rejects(line):
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError) as e:
        _load(f"5 6\n{HEAD}{line}\n")
    assert e.value.code == -200, line


@pytest.mark.parametrize("line", [f"{PS} 3=1", f"{PS} 0=7 1=7 2=6.250000e-02 3=21", f"{PS} 0=2 1=3 2=0.25 3=8"])
def test_loader_accepts(line):
    _load(f"5 6\n{HEAD}{line}\n")


def test_layer_registered_and_never_fused(tmp_path):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    param, _ = modelgen.rfcn_tiny().save(tmp_path / "rfcn")
    net = Net(fusion=True)
    net.LoadParam(param)
    net.FuseNow()
    for name in ("psroipooled_cls_rois", "psroipooled_loc_rois", "ave_cls_score_rois", "ave_bbox_pred_rois", "proposal"):
        assert net.LayerFusedAway(name) == 0, name


# ---- C ABI ----------------------------------------------------------------------------------------------------------
PSROI_REJECTS = [(dict(ph=0), -200), (dict(pw=0), -200), (dict(d=0), -200), (dict(d=-21), -200), (dict(scale=0.0), -200),
                 (dict(scale=-1.0), -200), (dict(scale=float("nan")), -200), (dict(scale=float("inf")), -200),
                 (dict(c=1028), -200), (dict(c=0), -200), (dict(ph=6), -200), (dict(d=20), -200),
                 (dict(d=2 ** 30, c=0), -200),                           # no overflow in output_dim * pooled_h * pooled_w
                 (dict(h=0), -100), (dict(w=0), -100), (dict(r=0), -100), (dict(n=0), -100), (dict(out=None), -100),
                 (dict(x=None), -100), (dict(rois=None), -100)]


@pytest.mark.parametrize("kw, code", PSROI_REJECTS, ids=[str(i) for i in range(len(PSROI_REJECTS))])
def test_psroi_pooling_abi_rejects(kw, code):
    from feathercnn_b200._lib import fcuda
    a = dict(out=FAKE, x=FAKE, rois=FAKE, c=1029, h=38, w=50, r=300, ph=7, pw=7, d=21, scale=0.0625, n=1)
    a.update(kw)
    assert fcuda().fcuda_psroi_pooling_forward(a["out"], a["x"], a["rois"], a["c"], a["h"], a["w"], a["r"], a["ph"],
                                               a["pw"], a["d"], a["scale"], a["n"], None) == code


def test_wrapper_checks_inputs():
    """booster.psroi_pooling refuses, before any call, what the C side would read out of bounds: rois of another batch,
    rows that are not 4 values, host or non-float32 tensors; a channel count that is not output_dim x pooled^2 comes back
    from the library as -200."""
    import torch
    from feathercnn_b200 import booster
    for x, r in ((torch.zeros(2, 18, 4, 4), torch.zeros(1, 5, 4)), (torch.zeros(2, 18, 4, 4), torch.zeros(2, 5, 3)),
                 (torch.zeros(2, 18, 4, 4), torch.zeros(2, 5, 4)), (torch.zeros(2, 18, 4, 4).double(),
                                                                    torch.zeros(2, 5, 4))):
        with pytest.raises(AssertionError):
            booster.psroi_pooling(x, r, 3, 3, 2, 0.25)


# ---- models ---------------------------------------------------------------------------------------------------------
def test_rfcn_resnet50_shapes():
    from feathercnn_b200.tools import modelgen
    m = modelgen.rfcn_resnet50()
    want = {"data": (3, 600, 800), "im_info": (1, 1, 3), "res4f": (1024, 38, 50), "res4f_relu": (1024, 38, 50),
            "res5c": (2048, 38, 50), "res5c_relu": (2048, 38, 50), "rpn_cls_score": (18, 38, 50),
            "rpn_bbox_pred": (36, 38, 50), "rois": (300, 1, 4), "conv_new_1": (1024, 38, 50), "rfcn_cls": (1029, 38, 50),
            "rfcn_bbox": (392, 38, 50), "psroipooled_cls_rois": (21, 7, 7), "psroipooled_loc_rois": (8, 7, 7),
            "cls_score": (21, 1, 1), "cls_prob": (21, 1, 1), "bbox_pred": (8, 1, 1)}
    for blob, shape in want.items():
        assert m.shape[blob] == shape, blob
    text = "\n".join(m.lines)
    assert "Convolution rpn_conv/3x3 1 1 res4f_relu rpn_conv/3x3 0=512 1=3 3=1 4=1 5=1 6=4718592" in text
    assert ("Proposal proposal 3 1 rpn_cls_prob_reshape rpn_bbox_pred im_info rois 0=16 1=16 2=6000 3=300 "
            "4=7.000000e-01 5=16") in text
    assert "Convolution conv_new_1 1 1 res5c_relu conv_new_1 0=1024 1=1 3=1 4=0 5=1 6=2097152" in text
    assert "PSROIPooling psroipooled_cls_rois 2 1 rfcn_cls rois psroipooled_cls_rois 0=7 1=7 2=6.250000e-02 3=21" in text
    assert "PSROIPooling psroipooled_loc_rois 2 1 rfcn_bbox rois psroipooled_loc_rois 0=7 1=7 2=6.250000e-02 3=8" in text
    assert "Pooling ave_cls_score_rois 1 1 psroipooled_cls_rois cls_score 0=1 1=7 2=7 3=0 4=0" in text
    assert "Pooling ave_bbox_pred_rois 1 1 psroipooled_loc_rois bbox_pred 0=1 1=7 2=7 3=0 4=0" in text
    assert "Softmax cls_prob 1 1 cls_score cls_prob" in text
    assert modelgen.ZOO["rfcn_resnet50"] is modelgen.rfcn_resnet50


def test_rfcn_resnet50_res5_dilated():
    """res5 runs at stride 1: res5a_branch1 and res5a_branch2a at stride 1 (3=1), every res5 3x3 at dilation 2 (2=2) and
    pad 2 (4=2); res2 .. res4 keep ResNet-50's strides and no dilation."""
    from feathercnn_b200.tools import modelgen
    lines = {L.split()[1]: L for L in modelgen.rfcn_resnet50().lines}
    for blk in ("5a", "5b", "5c"):
        p = lines[f"res{blk}_branch2b"].split()[6:]
        assert "1=3" in p and "2=2" in p and "3=1" in p and "4=2" in p, p
    for name in ("res5a_branch1", "res5a_branch2a"):
        p = lines[name].split()[6:]
        assert "3=1" in p and not any(k.startswith("2=") for k in p), p
    assert "3=2" in lines["res4a_branch1"].split()[6:] and "3=2" in lines["res3a_branch2a"].split()[6:]
    for blk in ("2a", "3b", "4f"):
        assert not any(k.startswith("2=") for k in lines[f"res{blk}_branch2b"].split()[6:]), blk


def test_rfcn_tiny_shapes():
    from feathercnn_b200.tools import modelgen
    m = modelgen.rfcn_tiny()
    assert m.shape["relu3"] == (32, 24, 32) and m.shape["rois"] == (64, 1, 4)
    assert m.shape["rfcn_cls"] == (45, 24, 32) and m.shape["rfcn_bbox"] == (72, 24, 32)
    assert m.shape["psroipooled_cls_rois"] == (5, 3, 3) and m.shape["psroipooled_loc_rois"] == (8, 3, 3)
    assert m.shape["cls_prob"] == (5, 1, 1) and m.shape["bbox_pred"] == (8, 1, 1)
    text = "\n".join(m.lines)
    assert "Convolution conv3 1 1 relu2 conv3 0=32 1=3 3=1 4=2 5=1 6=9216 2=2" in text
    line = next(L for L in m.lines if L.startswith("Proposal"))
    assert line.endswith("0=4 1=2 2=2000 3=64 4=7.000000e-01 5=4")   # 6,912 anchors: both limits bind
    assert "PSROIPooling psroipooled_cls_rois 2 1 rfcn_cls rois psroipooled_cls_rois 0=3 1=3 2=2.500000e-01 3=5" in text
    assert modelgen.ZOO["rfcn_tiny"] is modelgen.rfcn_tiny


# sha256 of (.param, .bin) as each model was written before the trunk and RPN builders were shared
UNCHANGED = {
    "resnet50": ("94b4f56354eaa7dd5f604e7a280517811795ada35d3621828370121b2e26733e",
                 "b2384943b512aa7a97d5affa31de3a01b6c4ab63d423f153a379d943d7d0e623"),
    "faster_rcnn_vgg16": ("ca9114880ac89aa2b42d70cfabe5cdddeb25379a6a07105a546cfc7e85c3425e",
                          "a06610631082bddaf880b33d86d474723cc2c3afe33c715ae25bdac80ef2c7eb"),
    "faster_rcnn_tiny": ("4d71d59d32bd97fd173b4cf722ca8035976fa19e83fd4e27da2563f0c09cda86",
                         "e5282a2883c296c5e9e55d76f25e2e78b222f0673cf383f42f39be4942ac6b49"),
}


@pytest.mark.parametrize("name", list(UNCHANGED))
def test_shared_builders_write_the_same_bytes(tmp_path, name):
    from feathercnn_b200.tools import modelgen
    param, binf = modelgen.ZOO[name]().save(tmp_path / name)
    got = tuple(hashlib.sha256(open(p, "rb").read()).hexdigest() for p in (param, binf))
    assert got == UNCHANGED[name]
