"""The SSD detection head on the host (no kernel is launched): parameter parsing, defaults and rejections of Permute,
Flatten, Reshape, axis Softmax, PriorBox and DetectionOutput; the -100 / -200 rejections of their C ABI entry points (every
call here fails its checks before a launch); the blob shapes and ranks of modelgen's MobileNet-SSD; and a NumPy PriorBox
restatement against hand-computed Caffe values.

priorbox_ref and detection_ref are the definitions tests/test_gpu_ssd.py holds the kernels to."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest


# ---- the definitions -----------------------------------------------------------------------------------------------
def priorbox_ref(fw, fh, iw, ih, min_sizes, max_sizes=(), ars=(), flip=True, clip=False, step=(0.0, 0.0), offset=0.5):
    """Caffe / ncnn PriorBox in float64: (4 * P,) boxes in location-major, Caffe prior order."""
    sw = step[0] if step[0] > 0 else iw / fw
    sh = step[1] if step[1] > 0 else ih / fh
    out = []
    for y in range(fh):
        for x in range(fw):
            cx, cy = (x + offset) * sw, (y + offset) * sh
            for k, mn in enumerate(min_sizes):
                sizes = [(mn, mn)]
                if max_sizes:
                    s = np.sqrt(mn * max_sizes[k])
                    sizes.append((s, s))
                for a in ars:
                    if abs(a - 1.0) < 1e-6:
                        continue
                    r = np.sqrt(a)
                    sizes.append((mn * r, mn / r))
                    if flip:
                        sizes.append((mn / r, mn * r))
                for bw, bh in sizes:
                    out += [(cx - bw / 2) / iw, (cy - bh / 2) / ih, (cx + bw / 2) / iw, (cy + bh / 2) / ih]
    out = np.array(out, np.float64)
    return np.clip(out, 0, 1) if clip else out


def iou32(a, area_a, b, area_b):
    """IoU of box a (the kept one) with boxes b, in float32, operation by operation as include/fcuda.h states it."""
    f = np.float32
    iw = np.maximum(np.minimum(a[2], b[:, 2]) - np.maximum(a[0], b[:, 0]), f(0))
    ih = np.maximum(np.minimum(a[3], b[:, 3]) - np.maximum(a[1], b[:, 1]), f(0))
    inter = (iw * ih).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (inter / ((area_b + area_a).astype(np.float32) - inter)).astype(np.float32)


def detection_ref(boxes, conf, num_classes, conf_thr, nms_thr, nms_top_k, keep_top_k):
    """DetectionOutput decision by decision: boxes (N, P, 4) float32 (fcuda_ssd_decode's bits), conf (N, P * C).
    Returns (out (N, keep_top_k, 6) float32, number of candidates suppressed by NMS)."""
    n_img, P = boxes.shape[:2]
    C = num_classes
    conf = conf.reshape(n_img, P, C)
    out = np.zeros((n_img, keep_top_k, 6), np.float32)
    out[:, :, 0] = -1
    suppressed = 0
    nms_thr = np.float32(nms_thr)
    for n in range(n_img):
        kept = []  # (score, class, prior)
        for c in range(1, C):
            s = conf[n, :, c]
            idx = np.nonzero(s > np.float32(conf_thr))[0]
            idx = idx[np.lexsort((idx, -s[idx].astype(np.float64)))][:nms_top_k]
            b = boxes[n, idx]
            area = ((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])).astype(np.float32)
            sup = np.zeros(len(idx), bool)
            for i in range(len(idx)):
                if sup[i]:
                    continue
                r = iou32(b[i], area[i], b[i + 1:], area[i + 1:])
                sup[i + 1:] |= r > nms_thr
                kept.append((s[idx[i]], c, idx[i]))
            suppressed += int(sup.sum())
        kept.sort(key=lambda t: (-float(t[0]), t[1], t[2]))
        for r, (sc, c, p) in enumerate(kept[:keep_top_k]):
            out[n, r] = [c, sc, *boxes[n, p]]
    return out, suppressed


# ---- layers ---------------------------------------------------------------------------------------------------------
def _load(text):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText("7767517\n" + text)
    return net


HEAD = "Input data 0 1 data 0=8 1=8 2=3\nInput feat 0 1 feat 0=4 1=4 2=12\n"


@pytest.mark.parametrize("line", [
    "Permute p 1 1 feat out 0=6",
    "Permute p 1 1 feat out 0=-1",
    "Reshape r 1 1 feat out 0=4 1=-1 3=1",
    "Reshape r 1 1 feat out 0=-1 1=-1",
    "Reshape r 1 1 feat out 1=4",
    "Reshape r 1 1 feat out 0=-5",
    "PriorBox pb 2 1 feat data out 7=1",
    "PriorBox pb 2 1 feat data out -23300=17," + ",".join(["1.0"] * 17),
    "PriorBox pb 2 1 feat data out -23300=2,2.0,3.0 -23301=1,4.0",
    "PriorBox pb 2 1 feat data out -23300=1,4.0 -23301=1,4.0",
    "PriorBox pb 2 1 feat data out -23300=1,-4.0",
    "PriorBox pb 2 1 feat data out -23300=1,4.0 -23302=1,-2.0",
    "PriorBox pb 1 1 feat out -23300=1,4.0",
    "PriorBox pb 2 1 feat data out -23300=1,4.0 11=-8.0",
    "DetectionOutput d 3 1 feat feat data out 0=0",
    "DetectionOutput d 3 1 feat feat data out 0=1025",
    "DetectionOutput d 3 1 feat feat data out 0=21 2=1025",
    "DetectionOutput d 3 1 feat feat data out 0=21 3=0",
    "DetectionOutput d 2 1 feat data out 0=21",
])
def test_loader_rejects(line):
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError) as e:
        _load(f"3 3\n{HEAD}{line}\n")
    assert e.value.code == -200, line


@pytest.mark.parametrize("line", [
    "Permute p 1 1 feat out 0=3",
    "Flatten f 1 1 feat out",
    "Reshape r 1 1 feat out 0=12 1=-1",
    "Reshape r 1 1 feat out 0=0 1=0 2=-1",
    "Softmax s 1 1 feat out 0=1 1=1",
    "Softmax s 1 1 feat out 0=-1",
    "PriorBox pb 2 1 feat data out -23300=1,4.0 -23301=1,6.0 -23302=2,2.0,3.0 8=1 11=2.0 12=2.0 13=0.25",
    "PriorBox pb 1 1 feat out -23300=1,4.0 9=8 10=8",
    "DetectionOutput d 3 1 feat feat data out 0=21",
])
def test_loader_accepts(line):
    _load(f"3 3\n{HEAD}{line}\n")


# ---- C ABI ----------------------------------------------------------------------------------------------------------
FAKE = ctypes.c_void_p(256)  # never dereferenced: every call below fails its argument checks first


def _pb(**kw):
    from feathercnn_b200 import booster
    args = dict(min_sizes=[60.0], max_sizes=[], aspect_ratios=[2.0])
    args.update(kw)
    return booster.priorbox_param(**args)


def test_priorbox_per_location():
    from feathercnn_b200 import booster
    assert booster.priorbox_per_location(_pb()) == 3
    assert booster.priorbox_per_location(_pb(min_sizes=[105.0], max_sizes=[150.0], aspect_ratios=[2.0, 3.0])) == 6
    assert booster.priorbox_per_location(_pb(aspect_ratios=[1.0, 2.0], flip=False)) == 2  # ar 1 is skipped
    assert booster.priorbox_per_location(_pb(min_sizes=[30.0, 60.0], max_sizes=[60.0, 90.0], aspect_ratios=[])) == 4


@pytest.mark.parametrize("kw", [dict(min_sizes=[]), dict(min_sizes=[1.0] * 17), dict(min_sizes=[0.0]),
                                dict(max_sizes=[50.0]), dict(min_sizes=[1.0, 2.0], max_sizes=[3.0]),
                                dict(aspect_ratios=[0.0]), dict(aspect_ratios=[float("nan")])])
def test_priorbox_abi_rejects(kw):
    from feathercnn_b200._lib import fcuda
    p = _pb(**kw)
    if len(kw.get("min_sizes", [1])) > 16:
        p.num_min_sizes = 17
    n = ctypes.c_int()
    assert fcuda().fcuda_priorbox_per_location(ctypes.byref(p), ctypes.byref(n)) == -200
    assert fcuda().fcuda_priorbox_forward(FAKE, ctypes.byref(p), 4, 4, 8, 8, None) == -200


def test_priorbox_abi_sizes():
    from feathercnn_b200._lib import fcuda
    p = _pb()
    lib = fcuda()
    assert lib.fcuda_priorbox_forward(None, ctypes.byref(p), 4, 4, 8, 8, None) == -100
    assert lib.fcuda_priorbox_forward(FAKE, ctypes.byref(p), 0, 4, 8, 8, None) == -100
    assert lib.fcuda_priorbox_forward(FAKE, ctypes.byref(p), 4, 4, 8, -1, None) == -100
    assert lib.fcuda_priorbox_forward(FAKE, ctypes.byref(p), 4096, 4096, 8, 8, None) == -200  # 2^24 * 3 / 4 priors


def test_permute_softmax_decode_abi_rejects():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    for order in (-1, 6):
        assert lib.fcuda_permute_forward(FAKE, FAKE, 2, 3, 4, order, 1, None) == -200
    assert lib.fcuda_permute_forward(FAKE, None, 2, 3, 4, 3, 1, None) == -100
    assert lib.fcuda_permute_forward(FAKE, FAKE, 0, 3, 4, 3, 1, None) == -100
    assert lib.fcuda_permute_forward(FAKE, FAKE, 2, 3, 4, 3, 0, None) == -100
    assert lib.fcuda_softmax_axis_forward(FAKE, FAKE, 1, 0, 1, 1, None) == -100
    assert lib.fcuda_softmax_axis_forward(FAKE, None, 1, 21, 1, 1, None) == -100
    assert lib.fcuda_ssd_decode(FAKE, FAKE, FAKE, 1 << 24, 1, None) == -200
    assert lib.fcuda_ssd_decode(FAKE, FAKE, None, 10, 1, None) == -100
    assert lib.fcuda_ssd_decode(FAKE, FAKE, FAKE, 10, 0, None) == -100


@pytest.mark.parametrize("args, code", [
    (dict(P=1 << 24), -200), (dict(C=1025), -200), (dict(top=0), -200), (dict(top=1025), -200), (dict(keep=0), -200),
    (dict(keep=1025), -200), (dict(nms=float("nan")), -200), (dict(batch=65536), -200), (dict(P=0), -100),
    (dict(batch=0), -100), (dict(ws=ctypes.c_void_p(260)), -100), (dict(ws=None), -100),
])
def test_detection_output_abi_rejects(args, code):
    from feathercnn_b200._lib import fcuda
    a = dict(P=100, C=21, top=100, keep=100, nms=0.45, batch=1, ws=FAKE)
    a.update(args)
    rc = fcuda().fcuda_detection_output_forward(FAKE, FAKE, FAKE, FAKE, a["P"], a["C"], 0.5, a["nms"], a["top"], a["keep"],
                                                a["ws"], a["batch"], None)
    assert rc == code


def test_detection_output_workspace_size():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    n = ctypes.c_size_t()
    assert lib.fcuda_detection_output_workspace_size(1917, 21, 100, 2, ctypes.byref(n)) == 0
    assert n.value == 2 * 1917 * 4 + 2 * 21 * 100 * 2 + 2 * 21
    assert lib.fcuda_detection_output_workspace_size(1917, 21, 2000, 2, ctypes.byref(n)) == -200
    assert lib.fcuda_detection_output_workspace_size(1917, 0, 100, 2, ctypes.byref(n)) == -100


# ---- models ---------------------------------------------------------------------------------------------------------
def test_mobilenet_ssd_shapes_and_ranks(tmp_path):
    from feathercnn_b200.tools import modelgen
    m = modelgen.mobilenet_ssd()
    assert m.shape["conv11_relu"] == (512, 19, 19) and m.shape["conv13_relu"] == (1024, 10, 10)
    assert [m.shape[f"conv{i}_2_relu"][1:] for i in range(14, 18)] == [(5, 5), (3, 3), (2, 2), (1, 1)]
    P = 1917
    assert 19 * 19 * 3 + (100 + 25 + 9 + 4 + 1) * 6 == P
    want = {"mbox_loc": ((1, 1, 4 * P), 1), "mbox_conf": ((1, 1, 21 * P), 1), "mbox_priorbox": ((1, 2, 4 * P), 2),
            "mbox_conf_reshape": ((1, P, 21), 2), "mbox_conf_softmax": ((1, P, 21), 2),
            "mbox_conf_flatten": ((1, 1, 21 * P), 1), "detection_out": ((1, 100, 6), 2),
            "conv11_relu_mbox_loc_perm": ((19, 19, 12), 3), "conv13_relu_mbox_conf_perm": ((10, 10, 126), 3)}
    for blob, (shape, rank) in want.items():
        assert (m.shape[blob], m.rank.get(blob, 3)) == (shape, rank), blob
    text = "\n".join(m.lines)
    assert "Softmax mbox_conf_softmax 1 1 mbox_conf_reshape mbox_conf_softmax 0=1 1=1" in text
    assert "DetectionOutput detection_out 3 1 mbox_loc mbox_conf_flatten mbox_priorbox detection_out 0=21 1=4.500000e-01 " \
           "2=100 3=100" in text
    param, _ = m.save(tmp_path / "ssd")
    from feathercnn_b200.net import Net
    net = Net(fusion=True)
    net.LoadParam(param)
    net.FuseNow()
    # the head takes part in no fusion
    for L in m.lines:
        typ, name = L.split()[:2]
        if typ in ("Permute", "Flatten", "Reshape", "Softmax", "Concat", "PriorBox", "DetectionOutput"):
            assert net.LayerFusedAway(name) == 0, name
        if name.endswith("_mbox_loc") or name.endswith("_mbox_conf"):
            assert net.LayerFusedAway(name) == 0, name


def test_softmax_without_axis_emits_no_axis():
    """Every existing zoo model's Softmax line carries no 0=, so SoftmaxLayer keeps its whole-blob kernel for them."""
    from feathercnn_b200.tools import modelgen
    for name in ("vgg16", "resnet50", "mobilenet_v1", "mobilenet_v2", "mini"):
        lines = [L for L in modelgen.ZOO[name]().lines if L.startswith("Softmax")]
        assert lines and all("=" not in L for L in lines), name


def test_priorbox_ref_matches_hand_computed_caffe_values():
    """conv13 of MobileNet-SSD (10 x 10 of 300 x 300, min 105, max 150, aspect ratios 2 and 3, flip, clip), location (0, 0):
    step 30, centre (15, 15); sizes 105, sqrt(105 * 150) = 125.4990..., 105 * sqrt(2) = 148.4924..., 105 / sqrt(2) =
    74.2462..., 105 * sqrt(3) = 181.8653..., 105 / sqrt(3) = 60.6218..."""
    got = priorbox_ref(10, 10, 300, 300, [105.0], [150.0], [2.0, 3.0], flip=True, clip=True)[:24].reshape(6, 4)
    want = np.array([
        [0.0, 0.0, 67.5 / 300, 67.5 / 300],
        [0.0, 0.0, (15 + 62.74950199) / 300, (15 + 62.74950199) / 300],
        [0.0, 0.0, (15 + 74.24621202) / 300, (15 + 37.12310601) / 300],
        [0.0, 0.0, (15 + 37.12310601) / 300, (15 + 74.24621202) / 300],
        [0.0, 0.0, (15 + 90.93266739) / 300, (15 + 30.31088913) / 300],
        [0.0, 0.0, (15 + 30.31088913) / 300, (15 + 90.93266739) / 300],
    ])
    assert np.allclose(got, want, rtol=0, atol=1e-9)
    # unclipped, the first box runs off the image: (15 - 52.5) / 300
    raw = priorbox_ref(10, 10, 300, 300, [105.0], [150.0], [2.0, 3.0], flip=True, clip=False)
    assert raw[0] == pytest.approx(-0.125) and raw.size == 4 * 600
    # the last location's centre: (9.5 * 30) / 300 = 0.95
    last = raw[-24:].reshape(6, 4)
    assert np.allclose((last[:, 0] + last[:, 2]) / 2, 0.95)


def test_detection_ref_tie_rule():
    """Equal scores: lower prior first within a class, lower class first across classes."""
    boxes = np.array([[[0, 0, 1, 1], [2, 2, 3, 3], [4, 4, 5, 5]]], np.float32)
    conf = np.zeros((1, 3, 3), np.float32)
    conf[0, :, 1] = [0.5, 0.7, 0.7]
    conf[0, :, 2] = [0.7, 0.1, 0.0]
    out, sup = detection_ref(boxes, conf, 3, 0.2, 0.5, 10, 4)
    assert out[0, :, 0].tolist() == [1, 1, 2, 1] and sup == 0
    assert out[0, 0, 2:].tolist() == [2, 2, 3, 3]
