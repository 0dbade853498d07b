"""The YOLO detection head on the host (no kernel is launched): parameter parsing and rejections of YoloDetectionOutput
and Yolov3DetectionOutput; the -100 / -200 rejections of their C ABI entry points (every call here fails its checks
before a launch); the workspace-size formula; the blob shapes and ranks of modelgen's YOLO models; hand-computed decodes of
one cell for each version; and the tie rule of the NumPy restatement of selection, NMS and output.

yolo_decode_ref and yolo_ref are the definitions tests/test_gpu_yolo.py holds the kernels to."""
from __future__ import annotations

import ctypes
import math

import numpy as np
import pytest

from test_ssd_host import iou32


# ---- the definitions -----------------------------------------------------------------------------------------------
def _sigmoid(t):
    return 1.0 / (1.0 + np.exp(-t))


def yolo_decode_ref(inputs, version, num_class, num_box, biases, mask=(), anchors_scale=()):
    """Decode in float64 (include/fcuda.h): inputs one (N, num_box * (5 + C), h, w) array per scale.  Returns
    (scores (N, S), classes (N, S), boxes (N, S, 4), second (N, S)), slots in (scale, box, row, column) order; `second` is the
    runner-up of the quantity the class is the argmax of (raw logits for v3, probabilities for v2), for near-tie checks."""
    scores, classes, boxes, second = [], [], [], []
    with np.errstate(over="ignore"):
        for b, x in enumerate(inputs):
            x = np.asarray(x, np.float64)
            n, _, h, w = x.shape
            x = x.reshape(n, num_box, 5 + num_class, h, w)
            jj, ii = np.meshgrid(np.arange(w), np.arange(h))
            for pp in range(num_box):
                t = x[:, pp]
                logit = t[:, 5:]
                if version == 3:
                    k = int(mask[b * num_box + pp])
                    bw_, bh_ = biases[2 * k], biases[2 * k + 1]
                    nw = float(int(np.float32(anchors_scale[b]) * np.float32(w)))
                    nh = float(int(np.float32(anchors_scale[b]) * np.float32(h)))
                    cls = logit.argmax(1)
                    top = logit.max(1)
                    srt = np.sort(logit, 1)
                    sec = srt[:, -2] if num_class > 1 else np.full_like(top, -np.inf)
                    conf = 1.0 / (1.0 + np.exp(-t[:, 4]) * (1.0 + np.exp(-top)))
                else:
                    bw_, bh_ = biases[2 * pp], biases[2 * pp + 1]
                    nw, nh = float(w), float(h)
                    e = np.exp(logit - logit.max(1, keepdims=True))
                    p = e / e.sum(1, keepdims=True)
                    cls = p.argmax(1)
                    srt = np.sort(p, 1)
                    sec = srt[:, -2] if num_class > 1 else np.zeros_like(srt[:, -1])
                    conf = _sigmoid(t[:, 4]) * p.max(1)
                cx = (jj + _sigmoid(t[:, 0])) / w
                cy = (ii + _sigmoid(t[:, 1])) / h
                bw = np.exp(t[:, 2]) * bw_ / nw
                bh = np.exp(t[:, 3]) * bh_ / nh
                box = np.stack([cx - bw * 0.5, cy - bh * 0.5, cx + bw * 0.5, cy + bh * 0.5], -1)
                scores.append(conf.reshape(n, -1))
                classes.append(cls.reshape(n, -1))
                boxes.append(box.reshape(n, -1, 4))
                second.append(sec.reshape(n, -1))
    return (np.concatenate(scores, 1), np.concatenate(classes, 1), np.concatenate(boxes, 1), np.concatenate(second, 1))


def yolo_ref(scores, classes, boxes, conf_thr, nms_thr, nms_top_k, keep_top_k):
    """Selection, class-agnostic NMS and output decision by decision: scores (N, S) float32, classes (N, S), boxes
    (N, S, 4) float32 (fcuda_yolo_decode's bits).  Returns (out (N, keep_top_k, 6) float32, number of candidates
    suppressed, number of candidates)."""
    n_img = scores.shape[0]
    out = np.zeros((n_img, keep_top_k, 6), np.float32)
    out[:, :, 0] = -1
    suppressed = candidates = 0
    nms_thr = np.float32(nms_thr)
    for n in range(n_img):
        s = scores[n]
        idx = np.nonzero(s >= np.float32(conf_thr))[0]
        candidates += len(idx)
        idx = idx[np.lexsort((idx, -s[idx].astype(np.float64)))][:nms_top_k]
        b = boxes[n, idx]
        area = ((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])).astype(np.float32)
        sup = np.zeros(len(idx), bool)
        kept = []
        for i in range(len(idx)):
            if sup[i]:
                continue
            r = iou32(b[i], area[i], b[i + 1:], area[i + 1:])
            sup[i + 1:] |= r > nms_thr
            kept.append(idx[i])
        suppressed += int(sup.sum())
        for r, slot in enumerate(kept[:keep_top_k]):
            out[n, r] = [classes[n, slot] + 1, s[slot], *boxes[n, slot]]
    return out, suppressed, candidates


# ---- layers ---------------------------------------------------------------------------------------------------------
def _load(text):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText("7767517\n" + text)
    return net


HEAD = "Input a 0 1 a 0=4 1=4 2=30\nInput b 0 1 b 0=8 1=8 2=30\nInput c 0 1 c 0=8 1=8 2=30\n"
B6 = "-23304=12,1.0,2.0,3.0,4.0,5.0,6.0,7.0,8.0,9.0,10.0,11.0,12.0"
V3 = f"Yolov3DetectionOutput d 2 1 a b out 0=5 1=3 {B6}"


@pytest.mark.parametrize("line", [
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0 0=0",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0 0=1025",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0 1=0",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0 1=17",
    f"{V3} -23305=5,3.0,4.0,5.0,0.0,1.0 -23306=2,8.0,4.0",                  # mask shorter than num_box x bottoms
    f"{V3} -23305=9,3.0,4.0,5.0,0.0,1.0,2.0,0.0,1.0,2.0 -23306=2,8.0,4.0",  # longer
    f"{V3} -23305=6,3.0,4.0,6.0,0.0,1.0,2.0 -23306=2,8.0,4.0",              # anchor 6 needs 14 biases
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,-1.0,2.0 -23306=2,8.0,4.0",
    f"{V3} -23305=6,3.0,4.0,5.5,0.0,1.0,2.0 -23306=2,8.0,4.0",              # not an index
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,0.0",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=1,8.0",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0 20=0",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0 20=1025",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0 21=0",
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0 21=1025",
    "Yolov3DetectionOutput d 5 1 a b c a b out 0=5 1=1 -23304=2,1.0,1.0 -23305=5,0,0,0,0,0 -23306=5,1.0,1.0,1.0,1.0,1.0",
    "Yolov3DetectionOutput d 1 1 a out 0=5 1=1 -23304=130," + ",".join(["1.0"] * 130) + " -23305=1,0 -23306=1,8.0",
    "YoloDetectionOutput d 2 1 b c out 0=5 1=3 " + B6,                          # one bottom only
    "YoloDetectionOutput d 1 1 b out 0=5 1=3 -23304=4,1.0,2.0,3.0,4.0",         # 2 * num_box biases
])
def test_loader_rejects(line):
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError) as e:
        _load(f"4 4\n{HEAD}{line}\n")
    assert e.value.code == -200, line


@pytest.mark.parametrize("line", [
    f"{V3} -23305=6,3.0,4.0,5.0,0.0,1.0,2.0 -23306=2,8.0,4.0",
    f"{V3} -23305=6,3,4,5,0,1,2 -23306=2,8.0,4.0 2=0.25 3=0.5 20=1 21=1024",  # integer mask entries
    "Yolov3DetectionOutput d 1 1 a out 0=5 1=3 -23304=6,1.0,2.0,3.0,4.0,5.0,6.0 -23305=3,2.0,1.0,0.0 -23306=1,8.0",
    "YoloDetectionOutput d 1 1 b out 0=5 1=6 " + B6,
    "YoloDetectionOutput d 1 1 b out 0=1 1=3 2=0.5 3=0.3 20=7 21=3 " + B6,
])
def test_loader_accepts(line):
    _load(f"4 4\n{HEAD}{line}\n")


# ---- C ABI ----------------------------------------------------------------------------------------------------------
FAKE = ctypes.c_void_p(256)  # never dereferenced: every call below fails its argument checks first


def _param(**kw):
    from feathercnn_b200 import booster
    a = dict(version=3, num_class=80, num_box=3, grids=[(13, 13), (26, 26), (52, 52)],
             biases=[10, 13, 16, 30, 33, 23, 30, 61, 62, 45, 59, 119, 116, 90, 156, 198, 373, 326],
             mask=[6, 7, 8, 3, 4, 5, 0, 1, 2], anchors_scale=[32.0, 16.0, 8.0])
    a.update(kw)
    return booster.yolo_param(**a)


REJECTS = [
    (dict(version=4), -200), (dict(num_class=0), -200), (dict(num_class=1025), -200), (dict(num_box=17), -200),
    (dict(num_box=0), -200), (dict(grids=[(4, 4)] * 5), -200), (dict(grids=[]), -200),
    (dict(mask=[6, 7, 9, 3, 4, 5, 0, 1, 2]), -200), (dict(mask=[6, 7, 8, 3, -1, 5, 0, 1, 2]), -200),
    (dict(anchors_scale=[32.0, 0.0, 8.0]), -200), (dict(anchors_scale=[32.0, float("nan"), 8.0]), -200),
    (dict(nms_threshold=float("nan")), -200), (dict(nms_top_k=0), -200), (dict(nms_top_k=1025), -200),
    (dict(keep_top_k=0), -200), (dict(keep_top_k=1025), -200), (dict(grids=[(4096, 4096)], mask=[0, 1, 2],
                                                                       anchors_scale=[8.0]), -200),
    (dict(version=2, grids=[(13, 13)] * 2, biases=[1.0] * 6), -200), (dict(version=2, grids=[(13, 13)], biases=[1.0] * 4),
                                                                       -200),
    (dict(grids=[(13, 13), (0, 26), (52, 52)]), -100),
    (dict(mask=[6, 7, 8, 3, 4, 5, 0, 1, 2 ** 31 - 1]), -200),                 # no overflow in the bias-pair test
    (dict(anchors_scale=[32.0, 1e30, 8.0]), -200),                            # (int)(anchors_scale * side) must exist
    (dict(anchors_scale=[32.0, float("inf"), 8.0]), -200),
    (dict(anchors_scale=[32.0, 16.0, 2.0 ** 31 / 52]), -200),
]


@pytest.mark.parametrize("kw, code", REJECTS, ids=[str(i) for i in range(len(REJECTS))])
def test_yolo_abi_rejects(kw, code):
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    p = _param(**kw)
    if len(kw.get("grids", [0, 0, 0])) > 4:
        p.num_scales = 5
    ins = (ctypes.c_void_p * 4)(256, 256, 256, 256)
    n = ctypes.c_size_t()
    assert lib.fcuda_yolo_detection_workspace_size(ctypes.byref(p), 1, ctypes.byref(n)) == code
    assert lib.fcuda_yolo_detection_forward(FAKE, ins, ctypes.byref(p), FAKE, 1, None) == code
    assert lib.fcuda_yolo_decode(FAKE, FAKE, FAKE, ins, ctypes.byref(p), 1, None) == code


def test_yolo_abi_pointers_and_batch():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    p = _param()
    ins = (ctypes.c_void_p * 4)(256, 256, 256, 256)
    n = ctypes.c_size_t()
    assert lib.fcuda_yolo_detection_forward(FAKE, ins, ctypes.byref(p), FAKE, 65536, None) == -200
    assert lib.fcuda_yolo_detection_forward(FAKE, ins, ctypes.byref(p), FAKE, 0, None) == -100
    assert lib.fcuda_yolo_detection_forward(None, ins, ctypes.byref(p), FAKE, 1, None) == -100
    assert lib.fcuda_yolo_detection_forward(FAKE, ins, ctypes.byref(p), None, 1, None) == -100
    assert lib.fcuda_yolo_detection_forward(FAKE, ins, ctypes.byref(p), ctypes.c_void_p(260), 1, None) == -100
    # the sweep stages the mask with 16-byte loads: a workspace 8 mod 16 is refused before any launch
    assert lib.fcuda_yolo_detection_forward(FAKE, ins, ctypes.byref(p), ctypes.c_void_p(264), 1, None) == -100
    assert lib.fcuda_yolo_detection_forward(FAKE, None, ctypes.byref(p), FAKE, 1, None) == -100
    assert lib.fcuda_yolo_detection_forward(FAKE, (ctypes.c_void_p * 4)(256, 256, None, 256), ctypes.byref(p), FAKE, 1,
                                            None) == -100
    assert lib.fcuda_yolo_detection_forward(FAKE, ins, None, FAKE, 1, None) == -100
    assert lib.fcuda_yolo_decode(FAKE, None, FAKE, ins, ctypes.byref(p), 1, None) == -100
    assert lib.fcuda_yolo_detection_workspace_size(ctypes.byref(p), 1, None) == -100
    assert lib.fcuda_yolo_detection_workspace_size(None, 1, ctypes.byref(n)) == -100


def test_yolo_wrappers_check_inputs_against_the_param():
    """booster.yolo_decode / yolo_detection refuse, before any call, inputs the C side would read out of bounds: a scale
    count other than num_scales, a grid or channel count other than the param's, mixed batches, non-float32 or host
    tensors."""
    import torch
    from feathercnn_b200 import booster
    p = _param(grids=[(2, 3), (4, 6)], mask=[3, 4, 5, 0, 1, 2], anchors_scale=[16.0, 8.0], num_class=2)
    ok = [torch.zeros(1, 21, 2, 3), torch.zeros(1, 21, 4, 6)]
    bad = [ok[:1], ok + [ok[0]], [ok[0], torch.zeros(1, 21, 4, 5)], [ok[0], torch.zeros(1, 24, 4, 6)],
           [ok[0], torch.zeros(2, 21, 4, 6)], [ok[0], ok[1].double()], ok]  # the last: right shapes, host memory
    for xs in bad:
        for fn in (booster.yolo_decode, booster.yolo_detection):
            with pytest.raises(AssertionError):
                fn(xs, p)


def test_yolo_workspace_size():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    n = ctypes.c_size_t()
    assert lib.fcuda_yolo_detection_workspace_size(ctypes.byref(_param()), 2, ctypes.byref(n)) == 0
    S = 3 * (13 * 13 + 26 * 26 + 52 * 52)
    assert S == 10647
    per_image = 2 * 1024 + 1024 * 32 + 1024 * 4 + 1024 + 1  # keys, mask, selected boxes, areas, count
    assert n.value == 2 * (6 * S + per_image) and per_image == 39937
    assert lib.fcuda_yolo_detection_workspace_size(ctypes.byref(_param(grids=[(19, 19), (38, 38), (76, 76)])), 1,
                                                   ctypes.byref(n)) == 0
    assert n.value == 6 * 22743 + 39937


# ---- models ---------------------------------------------------------------------------------------------------------
def test_mobilenetv2_yolov3_shapes_and_ranks(tmp_path):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.mobilenetv2_yolov3()
    want = {"conv_last_relu6": ((1280, 13, 13), 3), "block4_3": ((32, 52, 52), 3), "block6_3": ((96, 26, 26), 3),
            "up26": ((128, 26, 26), 3), "cat26": ((224, 26, 26), 3), "up52": ((64, 52, 52), 3), "cat52": ((96, 52, 52), 3),
            "yolo13_out": ((255, 13, 13), 3), "yolo26_out": ((255, 26, 26), 3), "yolo52_out": ((255, 52, 52), 3),
            "detection_out": ((1, 1024, 6), 2)}
    for blob, (shape, rank) in want.items():
        assert (m.shape[blob], m.rank.get(blob, 3)) == (shape, rank), blob
    assert 3 * (13 * 13 + 26 * 26 + 52 * 52) == 10647
    text = "\n".join(m.lines)
    assert ("Yolov3DetectionOutput detection_out 3 1 yolo13_out yolo26_out yolo52_out detection_out 0=80 1=3 "
            "2=1.000000e-02 3=4.500000e-01 -23304=18,1.000000e+01,1.300000e+01") in text
    assert "-23305=9,6.000000e+00,7.000000e+00,8.000000e+00,3.000000e+00" in text
    assert "-23306=3,3.200000e+01,1.600000e+01,8.000000e+00" in text
    assert "Interp up26 1 1 up26_reduce_relu6 up26 0=1 1=2.000000e+00 2=2.000000e+00" in text
    param, _ = m.save(tmp_path / "yolov3")
    net = Net(fusion=True)
    net.LoadParam(param)
    net.FuseNow()
    for L in m.lines:  # the head convolutions keep their outputs; the YOLO layer fuses nothing
        typ, name = L.split()[:2]
        if typ in ("Yolov3DetectionOutput", "Interp", "Concat") or name.endswith("_out"):
            assert net.LayerFusedAway(name) == 0, name


def test_mobilenet_yolov2_and_tiny_shapes():
    from feathercnn_b200.tools import modelgen
    m = modelgen.mobilenet_yolov2()
    assert m.shape["yolo_out"] == (125, 13, 13) and m.shape["detection_out"] == (1, 1024, 6)
    assert m.rank["detection_out"] == 2
    line = next(L for L in m.lines if L.startswith("YoloDetectionOutput"))
    assert line.startswith("YoloDetectionOutput detection_out 1 1 yolo_out detection_out 0=20 1=5 2=1.000000e-02 "
                           "3=4.500000e-01 -23304=10,1.080000e+00")
    t = modelgen.yolo_tiny()
    assert t.shape["yolo8_out"] == (30, 8, 8) and t.shape["yolo16_out"] == (30, 16, 16)
    for name in ("mobilenet_yolov2", "mobilenetv2_yolov3", "yolo_tiny"):
        assert modelgen.ZOO[name] is getattr(modelgen, name)


def test_yolo_head_bias():
    """The output convolutions' bias is obj_bias on every objectness channel and 0 elsewhere, as written to the bin."""
    from feathercnn_b200.tools import modelgen
    m = modelgen.yolo_tiny(obj_bias=-2.5)
    line = next(L for L in m.lines if L.split()[1] == "yolo8_out")
    assert " 5=1 " in line + " "
    n = 30 * 64  # weights of yolo8_out: 30 x 64 x 1 x 1, flagged
    # the bin is walked by modelgen itself: conv1 (16x3x3x3 + bias), conv2 (32x16x9 + bias), conv3 (64x32x9 + bias)
    off = sum(4 + 4 * w + 4 * b for w, b in ((16 * 27, 16), (32 * 144, 32), (64 * 288, 64)))
    bias = np.frombuffer(bytes(m.bin[off + 4 + 4 * n: off + 4 + 4 * n + 4 * 30]), np.float32).reshape(3, 10)
    assert np.all(bias[:, 4] == np.float32(-2.5)) and np.all(np.delete(bias, 4, 1) == 0)


# ---- the definitions, by hand ---------------------------------------------------------------------------------------
def test_decode_v3_one_cell_by_hand():
    """Scale 13 x 13 (anchors_scale 32: net 416), box 1 with anchor mask[1] = 7 = (156, 198), cell row 2, column 1:
    x = y = 0 (s = 0.5), tw = 0, th = ln 2, obj = 0, logits (1, 3, 3): class 1 (the first maximum),
    conf = 1 / (1 + 1 * (1 + e^-3))."""
    C, B = 3, 2
    x = np.zeros((1, B * (5 + C), 13, 13))
    x[0, 1 * (5 + C) + 3, 2, 1] = math.log(2.0)
    x[0, 1 * (5 + C) + 5:1 * (5 + C) + 8, 2, 1] = [1.0, 3.0, 3.0]
    biases = [0] * 12 + [116, 90, 156, 198]
    s, c, b, _ = yolo_decode_ref([x], 3, C, B, biases, mask=[6, 7], anchors_scale=[32.0])
    slot = 1 * 169 + 2 * 13 + 1
    assert c[0, slot] == 1
    assert s[0, slot] == pytest.approx(1 / (2 + 0.049787068367863944), rel=1e-12)
    cx, cy, bw, bh = 1.5 / 13, 2.5 / 13, 156 / 416, 2 * 198 / 416
    assert np.allclose(b[0, slot], [cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], rtol=0, atol=1e-15)
    # the expression is not s(obj) * s(logit): at obj = 0, logit 3 that would be 0.5 * 0.9526 = 0.4763
    assert abs(s[0, slot] - 0.5 * _sigmoid(3.0)) > 0.01


def test_decode_v2_one_cell_by_hand():
    """Grid 5 x 7 (h x w), box 0 with anchor (1.08, 1.19) cells, cell row 4, column 6: x = 2 (s = 0.880797), y = -1
    (0.268941), tw = th = 0, obj = ln 3 (s = 0.75), logits (0, ln 2, ln 2): p = (0.2, 0.4, 0.4), class 1, conf = 0.3."""
    C, B = 3, 1
    x = np.zeros((1, B * (5 + C), 5, 7))
    x[0, :, 4, 6] = [2.0, -1.0, 0.0, 0.0, math.log(3.0), 0.0, math.log(2.0), math.log(2.0)]
    s, c, b, _ = yolo_decode_ref([x], 2, C, B, [1.08, 1.19])
    slot = 4 * 7 + 6
    assert c[0, slot] == 1 and s[0, slot] == pytest.approx(0.3, rel=1e-12)
    cx, cy = (6 + 0.8807970779778823) / 7, (4 + 0.2689414213699951) / 5
    bw, bh = 1.08 / 7, 1.19 / 5
    assert np.allclose(b[0, slot], [cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], rtol=0, atol=1e-12)


def test_yolo_ref_tie_rule():
    """Equal confidences are ordered by slot ascending; NMS is class-agnostic; the label is class + 1; a candidate at
    exactly the threshold is one (>=)."""
    boxes = np.array([[[0, 0, 1, 1], [0, 0, 1, 1], [4, 4, 5, 5], [4, 4, 5, 5.1], [8, 8, 9, 9]]], np.float32)
    scores = np.float32([[0.5, 0.5, 0.5, 0.7, 0.25]])
    classes = np.array([[3, 0, 1, 2, 0]])
    out, sup, cand = yolo_ref(scores, classes, boxes, 0.25, 0.5, 10, 4)
    # order: slot 3 (0.7), then the 0.5 ties by slot: 0, 1, 2; then 4 (0.25 >= 0.25)
    # slot 1 duplicates slot 0 (another class: still suppressed); slot 2 overlaps slot 3
    assert cand == 5 and sup == 2
    assert out[0, :, 0].tolist() == [3, 4, 1, -1]
    assert out[0, 0, 1] == np.float32(0.7) and out[0, 1, 2:].tolist() == [0, 0, 1, 1]
    assert out[0, 3].tolist() == [-1, 0, 0, 0, 0, 0]
    # truncation: nms_top_k = 2 keeps slots 3 and 0 only
    out2, _, _ = yolo_ref(scores, classes, boxes, 0.25, 0.5, 2, 4)
    assert out2[0, :, 0].tolist() == [3, 4, -1, -1]
