"""Faster R-CNN's Proposal and ROIPooling on the host (no kernel is launched): the NumPy definitions the GPU tests hold the
kernels to, checked by hand; the anchor table; the loader's and the C ABI's rejections at every limit (every call here
fails its checks before a launch); the workspace formula; the blob shapes of modelgen's Faster R-CNN models.

proposal_decode_ref, proposal_ref and roi_pooling_ref are the definitions tests/test_gpu_faster_rcnn.py holds the kernels
to (include/fcuda.h states them)."""
from __future__ import annotations

import ctypes
import math

import numpy as np
import pytest

A = 9
F = np.float32


# ---- the definitions -----------------------------------------------------------------------------------------------
def anchors_ref(base_size=16):
    """(9, 4) float32 rows (ax1, ay1, aw, ah), anchor q = ratio * 3 + scale; roundf is half away from zero."""
    out = np.zeros((A, 4), np.float32)
    base = F(base_size)
    for r, ratio in enumerate((F(0.5), F(1.0), F(2.0))):
        v = base / np.sqrt(ratio)
        rw = F(np.sign(v) * np.floor(np.abs(np.float64(v)) + 0.5))
        v = rw * ratio
        rh = F(np.sign(v) * np.floor(np.abs(np.float64(v)) + 0.5))
        for k, scale in enumerate((F(8), F(16), F(32))):
            aw, ah = rw * scale, rh * scale
            out[r * 3 + k] = [base * F(0.5) - aw * F(0.5), base * F(0.5) - ah * F(0.5), aw, ah]
    return out


def proposal_decode_ref(bbox, im_info, feat_stride=16, base_size=16):
    """Decode and clip in float64: bbox (N, 36, H, W), im_info (N, 3) -> boxes (N, 9 * H * W, 4), index q * H * W +
    y * W + x; also the unclipped boxes and the anchor widths (aw, ah) per index, for the error bounds."""
    bbox = np.asarray(bbox, np.float64)
    n, _, h, w = bbox.shape
    an = anchors_ref(base_size).astype(np.float64)
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    d = bbox.reshape(n, A, 4, h, w)
    raw = np.zeros((n, A, h, w, 4))
    awh = np.zeros((A, h, w, 2))
    with np.errstate(over="ignore", invalid="ignore"):
        for q in range(A):
            ax1, ay1, aw, ah = an[q]
            ax, ay = ax1 + xx * feat_stride, ay1 + yy * feat_stride
            pcx = ax + aw * 0.5 + aw * d[:, q, 0]
            pcy = ay + ah * 0.5 + ah * d[:, q, 1]
            pw, ph = aw * np.exp(d[:, q, 2]), ah * np.exp(d[:, q, 3])
            raw[:, q] = np.stack([pcx - pw * 0.5, pcy - ph * 0.5, pcx + pw * 0.5, pcy + ph * 0.5], -1)
            awh[q] = [aw, ah]
    raw = raw.reshape(n, -1, 4)
    info = np.asarray(im_info, np.float64).reshape(n, 3)
    hi = np.stack([info[:, 1] - 1, info[:, 0] - 1, info[:, 1] - 1, info[:, 0] - 1], -1)[:, None, :]
    boxes = np.maximum(np.minimum(raw, hi), 0.0)
    return boxes, raw, awh.reshape(-1, 2)


def iou_plus1(a, b):
    """The + 1 IoU of box a against rows b, float32 operation by operation (include/fcuda.h)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32).reshape(-1, 4)
    one = F(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        iw = np.maximum((np.minimum(a[2], b[:, 2]) - np.maximum(a[0], b[:, 0])) + one, F(0))
        ih = np.maximum((np.minimum(a[3], b[:, 3]) - np.maximum(a[1], b[:, 1])) + one, F(0))
        inter = iw * ih
        area_a = ((a[2] - a[0]) + one) * ((a[3] - a[1]) + one)
        area_b = ((b[:, 2] - b[:, 0]) + one) * ((b[:, 3] - b[:, 1]) + one)
        return inter / ((area_a + area_b) - inter)


def proposal_ref(boxes, score, im_info, pre_nms_top_n, post_nms_top_n, nms_thresh, min_size):
    """Candidates, order, NMS and rows decision by decision from float32 boxes (N, 9 * H * W, 4) (fcuda_proposal_decode's
    bits) and score (N, 18, H, W).  Returns (rois (N, post, 4), scores (N, post), stats): stats per image
    (candidates, kept, suppressed)."""
    boxes = np.asarray(boxes, np.float32)
    n = boxes.shape[0]
    fg = np.asarray(score, np.float32)[:, A:].reshape(n, -1)
    info = np.asarray(im_info, np.float32).reshape(n, 3)
    rois = np.zeros((n, post_nms_top_n, 4), np.float32)
    scores = np.full((n, post_nms_top_n), -1, np.float32)
    stats = []
    thr_nms = F(nms_thresh)
    for i in range(n):
        b = boxes[i]
        thr = F(min_size) * info[i, 2]
        ok = (((b[:, 2] - b[:, 0]) + F(1)) >= thr) & (((b[:, 3] - b[:, 1]) + F(1)) >= thr) & ~np.isnan(fg[i])
        idx = np.nonzero(ok)[0]
        idx = idx[np.lexsort((idx, -fg[i, idx].astype(np.float64)))][:pre_nms_top_n]
        sup = np.zeros(len(idx), bool)
        kept = []
        for j in range(len(idx)):
            if sup[j]:
                continue
            kept.append(idx[j])
            if len(kept) == post_nms_top_n:
                break
            sup[j + 1:] |= iou_plus1(b[idx[j]], b[idx[j + 1:]]) > thr_nms
        for r, k in enumerate(kept):
            rois[i, r] = b[k]
            scores[i, r] = fg[i, k]
        stats.append((int(ok.sum()), len(kept), int(sup.sum())))
    return rois, scores, stats


def _roundf(v):
    v = np.float64(v)
    return int(np.sign(v) * np.floor(np.abs(v) + 0.5))


def roi_pooling_ref(x, rois, pooled_h, pooled_w, spatial_scale):
    """x (N, C, H, W) float32, rois (N, R, 4) -> (N * R, C, pooled_h, pooled_w), Caffe's / ncnn's arithmetic in float32."""
    x = np.asarray(x, np.float32)
    rois = np.asarray(rois, np.float32).reshape(x.shape[0], -1, 4)
    n, c, h, w = x.shape
    r_ = rois.shape[1]
    out = np.zeros((n * r_, c, pooled_h, pooled_w), np.float32)
    s = F(spatial_scale)
    for i in range(n):
        for r in range(r_):
            x1, y1, x2, y2 = (_roundf(v * s) for v in rois[i, r])
            bw = F(max(x2 - x1 + 1, 1)) / F(pooled_w)
            bh = F(max(y2 - y1 + 1, 1)) / F(pooled_h)
            for ph in range(pooled_h):
                hs = min(max(int(np.floor(F(ph) * bh)) + y1, 0), h)
                he = min(max(int(np.ceil(F(ph + 1) * bh)) + y1, 0), h)
                for pw in range(pooled_w):
                    ws = min(max(int(np.floor(F(pw) * bw)) + x1, 0), w)
                    we = min(max(int(np.ceil(F(pw + 1) * bw)) + x1, 0), w)
                    if he > hs and we > ws:
                        out[i * r_ + r, :, ph, pw] = np.maximum(x[i, :, hs:he, ws:we].reshape(c, -1).max(1),
                                                                F(-3.4028234663852886e38))
    return out


# ---- the definitions, by hand ---------------------------------------------------------------------------------------
PY_FASTER_RCNN_ANCHORS = [[-84, -40, 99, 55], [-176, -88, 191, 103], [-360, -184, 375, 199], [-56, -56, 71, 71],
                          [-120, -120, 135, 135], [-248, -248, 263, 263], [-36, -80, 51, 95], [-80, -168, 95, 183],
                          [-168, -344, 183, 359]]


def test_anchor_table():
    """py-faster-rcnn's generate_anchors() table, as (ax1, ay1, ax1 + aw - 1, ay1 + ah - 1), from both the NumPy
    definition and the library."""
    from feathercnn_b200 import booster
    ref = anchors_ref(16)
    lib = np.array(booster.proposal_anchors(booster.proposal_param()), np.float32)
    assert np.array_equal(lib, ref)
    corners = np.stack([ref[:, 0], ref[:, 1], ref[:, 0] + ref[:, 2] - 1, ref[:, 1] + ref[:, 3] - 1], 1)
    assert corners.tolist() == PY_FASTER_RCNN_ANCHORS
    # another base size: 16 / sqrt(0.5) = 22.6 -> 23 but 2 / sqrt(0.5) = 2.83 -> 3 and 3 * 0.5 = 1.5 -> 2 (half away)
    lib2 = np.array(booster.proposal_anchors(booster.proposal_param(base_size=2)), np.float32)
    assert np.array_equal(lib2, anchors_ref(2)) and lib2[0].tolist() == [1 - 12, 1 - 8, 24, 16]


def test_decode_clip_filter_by_hand():
    """Anchor q = 4 (ratio 1, scale 16: 256 x 256 at ax1 = ay1 = -120) at cell (y, x) = (1, 2), stride 16:
    ax = -88, ay = -104, centre (40, 24).  dx = 0.25, dy = 0, dw = ln 0.5, dh = 0: pcx = 104, pcy = 24, pw = 128,
    ph = 256 -> (40, -104, 168, 152), clipped to a 100 x 120 (h x w) image: (40, 0, 119, 99)."""
    h, w = 3, 4
    bbox = np.zeros((1, 36, h, w))
    bbox[0, 4 * 4:4 * 4 + 4, 1, 2] = [0.25, 0.0, math.log(0.5), 0.0]
    boxes, raw, _ = proposal_decode_ref(bbox, [[100, 120, 1.0]])
    i = 4 * h * w + 1 * w + 2
    assert np.allclose(raw[0, i], [40, -104, 168, 152], rtol=0, atol=1e-12)
    assert boxes[0, i].tolist() == [40, 0, 119, 99]
    # filter: width 119 - 40 + 1 = 80, height 100; min_size 16 at scale 5 needs 80: kept; at scale 5.0625 dropped
    score = np.zeros((1, 18, h, w), np.float32)
    score[0, A + 4, 1, 2] = 0.9
    b32 = boxes.astype(np.float32)
    for scale, want in ((5.0, 1), (5.0625, 0)):
        _, _, stats = proposal_ref(b32[:, i:i + 1].repeat(A * h * w, 1) * 0 + b32[:, i:i + 1], score,
                                   [[100, 120, scale]], 10, 10, 0.7, 16)
        assert stats[0][0] == want * A * h * w
    # a NaN score is never a candidate
    score[0, A + 4, 1, 2] = np.nan
    _, _, stats = proposal_ref(b32, score, [[100, 120, 1.0]], 10, 10, 0.7, 16)
    assert stats[0][0] == int((((b32[0, :, 2] - b32[0, :, 0]) + 1 >= 16) & ((b32[0, :, 3] - b32[0, :, 1]) + 1 >= 16)).sum()) - 1


def test_iou_plus_one_by_hand():
    """(0, 0, 9, 9) and (5, 0, 14, 9): 10 x 10 boxes overlapping 5 x 10 pixels: 50 / 150 = 1/3 (DetectionOutput's
    convention would give 45 / 135, also 1/3, so take a case where they differ: (0, 0, 9, 9) and (9, 9, 18, 18) touch
    in one pixel, 1 / 199, where the + 0 convention gives 0."""
    assert iou_plus1([0, 0, 9, 9], [[5, 0, 14, 9]])[0] == F(50) / F(150)
    assert iou_plus1([0, 0, 9, 9], [[9, 9, 18, 18]])[0] == F(1) / F(199)
    assert iou_plus1([0, 0, 9, 9], [[0, 0, 9, 9]])[0] == 1
    assert iou_plus1([0, 0, 9, 9], [[20, 20, 29, 29]])[0] == 0


def test_proposal_ref_tie_rule_and_stop():
    """Equal scores go by index ascending; -0 and +0 are equal; the NMS stops at post_nms_top_n kept boxes; rows past the
    count are zero with score -1; pre_nms_top_n drops the lowest-ranked candidates before NMS."""
    h, w = 1, 1
    boxes = np.array([[[0, 0, 99, 99], [0, 0, 99, 99], [200, 200, 299, 299], [0, 0, 99, 98], [400, 400, 499, 499],
                       [600, 600, 699, 699], [800, 800, 899, 899], [1000, 1000, 1099, 1099], [5, 5, 30, 30]]], np.float32)
    score = np.zeros((1, 18, h, w), np.float32)
    score[0, A:, 0, 0] = [0.5, 0.5, 0.5, 0.9, -0.0, 0.0, 0.25, 0.25, 0.1]
    info = [[2000, 2000, 1.0]]
    rois, sc, stats = proposal_ref(boxes, score, info, 100, 20, 0.7, 16)
    # order: 3 (0.9), 0, 1, 2 (0.5 by index), 6, 7 (0.25), 8 (0.1), 4, 5 (-0 == +0, by index)
    # 0 and 1 overlap 3 almost entirely: suppressed
    assert stats[0] == (9, 7, 2)
    assert rois[0, :7, 0].tolist() == [0, 200, 800, 1000, 5, 400, 600]
    assert sc[0, :7].tolist() == [F(0.9), 0.5, 0.25, 0.25, F(0.1), 0, 0] and np.signbit(sc[0, 5])
    assert np.all(rois[0, 7:] == 0) and np.all(sc[0, 7:] == -1)
    rois, sc, stats = proposal_ref(boxes, score, info, 100, 3, 0.7, 16)   # the stop
    assert stats[0][1] == 3 and rois[0, :3, 0].tolist() == [0, 200, 800]
    rois, sc, stats = proposal_ref(boxes, score, info, 2, 20, 0.7, 16)    # pre_nms_top_n: 3 and 0 only
    assert stats[0][1] == 1 and rois[0, 0, 0] == 0 and rois[0, 0, 3] == 98


def test_roi_pooling_ref_by_hand():
    """One 4 x 4 map, RoI (0.5, 0.5, 2.49, 3.5) at scale 1: corners round half away to (1, 1, 2, 4) -> roi 2 wide, 4 high;
    2 x 2 bins of 1 x 2: rows 1-2 / 3 (4 is clamped to H), columns 1 / 2.  An RoI left of the map pools empty bins to 0."""
    x = np.arange(16, dtype=np.float32).reshape(1, 1, 4, 4)
    out = roi_pooling_ref(x, [[[0.5, 0.5, 2.49, 3.5]]], 2, 2, 1.0)
    assert out[0, 0].tolist() == [[9, 10], [13, 14]]
    out = roi_pooling_ref(x, [[[-10, 0, -5, 3]]], 2, 2, 1.0)
    assert np.all(out == 0)
    out = roi_pooling_ref(-x - 1, [[[0, 0, 0, 0]]], 1, 1, 1.0)   # a zero-area RoI is one pixel
    assert out.ravel().tolist() == [-1]


# ---- layers ---------------------------------------------------------------------------------------------------------
def _load(text):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText("7767517\n" + text)
    return net


HEAD = "Input s 0 1 s 0=4 1=4 2=18\nInput b 0 1 b 0=4 1=4 2=36\nInput i 0 1 i 0=3\nInput f 0 1 f 0=4 1=4 2=8\n"
PROP = "Proposal p 3 1 s b i rois"


@pytest.mark.parametrize("line", [
    f"{PROP} 0=0", f"{PROP} 1=0", f"{PROP} 2=0", f"{PROP} 2=8193", f"{PROP} 3=0", f"{PROP} 3=8193",
    "Proposal p 2 1 s b rois", "Proposal p 3 3 s b i r1 r2 r3",
    "ROIPooling r 2 1 f s out 0=0", "ROIPooling r 2 1 f s out 1=0", "ROIPooling r 2 1 f s out 2=0",
    "ROIPooling r 2 1 f s out 2=-0.0625", "ROIPooling r 1 1 f out",
])
def test_loader_rejects(line):
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError) as e:
        _load(f"5 6\n{HEAD}{line}\n")
    assert e.value.code == -200, line


@pytest.mark.parametrize("line", [
    PROP, f"{PROP} 0=16 1=16 2=6000 3=300 4=7.000000e-01 5=16", f"{PROP} 2=8192 3=8192 4=0 5=0",
    "Proposal p 3 2 s b i rois scores 3=1", "ROIPooling r 2 1 f s out", "ROIPooling r 2 1 f s out 0=3 1=5 2=0.125",
])
def test_loader_accepts(line):
    _load(f"5 6\n{HEAD}{line}\n")


def test_layers_registered_and_never_fused(tmp_path):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.faster_rcnn_tiny()
    param, _ = m.save(tmp_path / "frcnn")
    net = Net(fusion=True)
    net.LoadParam(param)
    net.FuseNow()
    for name in ("proposal", "roi_pool5", "rpn_cls_prob", "rpn_cls_score_reshape", "rpn_cls_prob_reshape"):
        assert net.LayerFusedAway(name) == 0, name


# ---- C ABI ----------------------------------------------------------------------------------------------------------
FAKE = ctypes.c_void_p(256)  # never dereferenced: every call below fails its argument checks first


def _p(**kw):
    from feathercnn_b200 import booster
    return booster.proposal_param(**kw)


PROPOSAL_REJECTS = [
    (dict(feat_stride=0), {}, -200), (dict(feat_stride=-16), {}, -200), (dict(base_size=0), {}, -200),
    (dict(pre_nms_topN=0), {}, -200), (dict(pre_nms_topN=8193), {}, -200), (dict(after_nms_topN=0), {}, -200),
    (dict(after_nms_topN=8193), {}, -200), (dict(nms_thresh=float("nan")), {}, -200),
    ({}, dict(h=1, w=1864136), -200),                      # 9 * H * W = 16,777,224 >= 2^24
    ({}, dict(h=2 ** 31 - 1, w=2 ** 31 - 1), -200),        # no overflow in 9 * H * W
    ({}, dict(h=65536, w=65536), -200), ({}, dict(batch=65536), -200),
    ({}, dict(h=0), -100), ({}, dict(w=0), -100), ({}, dict(batch=0), -100),
]


@pytest.mark.parametrize("kw, geo, code", PROPOSAL_REJECTS, ids=[str(i) for i in range(len(PROPOSAL_REJECTS))])
def test_proposal_abi_rejects(kw, geo, code):
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    p = _p(**kw)
    h, w, n = geo.get("h", 38), geo.get("w", 50), geo.get("batch", 1)
    sz = ctypes.c_size_t()
    assert lib.fcuda_proposal_workspace_size(ctypes.byref(p), h, w, n, ctypes.byref(sz)) == code
    assert lib.fcuda_proposal_forward(FAKE, FAKE, FAKE, FAKE, FAKE, ctypes.byref(p), h, w, FAKE, n, None) == code
    assert lib.fcuda_proposal_decode(FAKE, FAKE, FAKE, FAKE, ctypes.byref(p), h, w, n, None) == code


def test_proposal_abi_accepts_the_limits_and_checks_pointers():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    sz = ctypes.c_size_t()
    p = _p(pre_nms_topN=8192, after_nms_topN=8192)
    assert lib.fcuda_proposal_workspace_size(ctypes.byref(p), 1, 1864135, 1, ctypes.byref(sz)) == 0  # 9 H W = 2^24 - 1
    assert lib.fcuda_proposal_workspace_size(ctypes.byref(p), 38, 50, 65535, ctypes.byref(sz)) == 0
    p = _p()
    args = [FAKE, FAKE, FAKE, FAKE, FAKE]
    for k in (0, 2, 3, 4):  # rois, score, bbox, im_info; scores (1) may be NULL
        a = list(args)
        a[k] = None
        assert lib.fcuda_proposal_forward(*a, ctypes.byref(p), 38, 50, FAKE, 1, None) == -100
    assert lib.fcuda_proposal_forward(*args, ctypes.byref(p), 38, 50, None, 1, None) == -100
    assert lib.fcuda_proposal_forward(*args, ctypes.byref(p), 38, 50, ctypes.c_void_p(264), 1, None) == -100  # 16-byte
    assert lib.fcuda_proposal_forward(*args, None, 38, 50, FAKE, 1, None) == -100
    assert lib.fcuda_proposal_decode(None, FAKE, FAKE, FAKE, ctypes.byref(p), 38, 50, 1, None) == -100
    assert lib.fcuda_proposal_workspace_size(ctypes.byref(p), 38, 50, 1, None) == -100
    assert lib.fcuda_proposal_anchors(ctypes.byref(p), None) == -100
    assert lib.fcuda_proposal_anchors(ctypes.byref(_p(base_size=0)), (ctypes.c_float * 36)()) == -200


ROI_REJECTS = [(dict(ph=0), -200), (dict(pw=0), -200), (dict(scale=0.0), -200), (dict(scale=-1.0), -200),
               (dict(scale=float("nan")), -200), (dict(scale=float("inf")), -200), (dict(c=0), -100), (dict(h=0), -100),
               (dict(w=0), -100), (dict(r=0), -100), (dict(n=0), -100), (dict(out=None), -100), (dict(x=None), -100),
               (dict(rois=None), -100)]


@pytest.mark.parametrize("kw, code", ROI_REJECTS, ids=[str(i) for i in range(len(ROI_REJECTS))])
def test_roi_pooling_abi_rejects(kw, code):
    from feathercnn_b200._lib import fcuda
    a = dict(out=FAKE, x=FAKE, rois=FAKE, c=512, h=38, w=50, r=300, ph=7, pw=7, scale=0.0625, n=1)
    a.update(kw)
    assert fcuda().fcuda_roi_pooling_forward(a["out"], a["x"], a["rois"], a["c"], a["h"], a["w"], a["r"], a["ph"],
                                             a["pw"], a["scale"], a["n"], None) == code


def test_wrappers_check_inputs():
    """booster.proposal / proposal_decode / roi_pooling refuse, before any call, what the C side would read out of
    bounds: wrong channel counts, mismatched maps or batches, im_info without 3 values per image, non-float32 or host
    tensors."""
    import torch
    from feathercnn_b200 import booster
    p = booster.proposal_param()
    s, b, i = torch.zeros(2, 18, 3, 4), torch.zeros(2, 36, 3, 4), torch.zeros(2, 3)
    bad = [(torch.zeros(2, 16, 3, 4), b, i), (s, torch.zeros(2, 36, 3, 5), i), (s, torch.zeros(1, 36, 3, 4), i),
           (s, b, torch.zeros(2, 4)), (s, b, torch.zeros(1, 3)), (s.double(), b, i), (s, b, i)]  # last: host memory
    for args in bad:
        for fn in (booster.proposal, booster.proposal_decode):
            with pytest.raises(AssertionError):
                fn(*args, p)
    for x, r in ((torch.zeros(2, 8, 4, 4), torch.zeros(1, 5, 4)), (torch.zeros(2, 8, 4, 4), torch.zeros(2, 5, 3)),
                 (torch.zeros(2, 8, 4, 4), torch.zeros(2, 5, 4))):
        with pytest.raises(AssertionError):
            booster.roi_pooling(x, r)


def test_proposal_workspace_size():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    sz = ctypes.c_size_t()
    assert lib.fcuda_proposal_workspace_size(ctypes.byref(_p()), 38, 50, 2, ctypes.byref(sz)) == 0
    P, K = 9 * 38 * 50, 6000
    assert P == 17100
    per_image = 4 * P + P + 4 * K + 2 * K + K * 188  # boxes, keys, selected boxes, areas and indices, mask
    assert sz.value == 2 * per_image + 4
    assert lib.fcuda_proposal_workspace_size(ctypes.byref(_p(pre_nms_topN=33)), 1, 1, 5, ctypes.byref(sz)) == 0
    assert sz.value == 5 * (36 + 12 + 4 * 33 + 2 * 36 + 33 * 2) + 8


# ---- models ---------------------------------------------------------------------------------------------------------
def test_faster_rcnn_vgg16_shapes():
    from feathercnn_b200.tools import modelgen
    m = modelgen.faster_rcnn_vgg16()
    want = {"data": (3, 600, 800), "im_info": (1, 1, 3), "relu5_3": (512, 38, 50), "rpn_cls_score": (18, 38, 50),
            "rpn_bbox_pred": (36, 38, 50), "rpn_cls_score_reshape": (2, 342, 50), "rpn_cls_prob": (2, 342, 50),
            "rpn_cls_prob_reshape": (18, 38, 50), "rois": (300, 1, 4), "pool5": (512, 7, 7), "fc6": (4096, 1, 1),
            "fc7": (4096, 1, 1), "cls_prob": (21, 1, 1), "bbox_pred": (84, 1, 1)}
    for blob, shape in want.items():
        assert m.shape[blob] == shape, blob
    assert 9 * 38 * 50 == 17100
    assert m.lines[0].startswith("Input data") and m.lines[1] == "Input im_info 0 1 im_info 0=3 1=1 2=1"
    text = "\n".join(m.lines)
    assert ("Proposal proposal 3 1 rpn_cls_prob_reshape rpn_bbox_pred im_info rois 0=16 1=16 2=6000 3=300 "
            "4=7.000000e-01 5=16") in text
    assert "ROIPooling roi_pool5 2 1 relu5_3 rois pool5 0=7 1=7 2=6.250000e-02" in text
    assert "InnerProduct fc6 1 1 pool5 fc6 0=4096 1=1 2=102760448" in text
    # fc6 runs over 300 RoIs per image: 2 x 300 x 25088 x 4096 FLOP
    assert 2 * 300 * 25088 * 4096 / 1e9 == pytest.approx(61.65, abs=0.01)
    assert modelgen.ZOO["faster_rcnn_vgg16"] is modelgen.faster_rcnn_vgg16


def test_faster_rcnn_tiny_shapes():
    from feathercnn_b200.tools import modelgen
    m = modelgen.faster_rcnn_tiny()
    assert m.shape["relu2"] == (32, 24, 32) and m.shape["rois"] == (64, 1, 4) and m.shape["pool5"] == (32, 4, 4)
    assert m.shape["cls_prob"] == (5, 1, 1) and m.shape["bbox_pred"] == (20, 1, 1)
    line = next(L for L in m.lines if L.startswith("Proposal"))
    assert line.endswith("0=4 1=2 2=2000 3=64 4=7.000000e-01 5=4")
    assert modelgen.ZOO["faster_rcnn_tiny"] is modelgen.faster_rcnn_tiny
