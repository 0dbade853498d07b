"""The SSD detection head on the GPU.

  - Permute: all six orders bit-exact against np.transpose, odd shapes, batch > 1.  Flatten and Reshape are views: their
    device pointer is their bottom's.
  - Softmax over an axis, against float64, per element.  With x the row, m = max x, the kernel computes
    d = fl(x - m) (relative error <= U, so |d - (x - m)| <= U |x - m|), e = expf(d) (<= 2 ulp, and the argument error
    moves e by a factor exp(U |x - m|)), a sum of `len` positive terms (relative error <= (len - 1) U), and one division
    (U).  So |y - y*| <= y* ((len + 4) U + 2 U max|x - m|) to first order; the test allows twice that plus 2^-140 for
    results below the normal range.  Without an axis the layer's output is bit-identical to fcuda_softmax_forward.
  - PriorBox: the coordinates (c +- b / 2) / img with c = (x + offset) * step and b = min * sqrt(ar): four roundings on c,
    three on b, one subtraction and one division; each <= U of its operand.  The bound is 8 U (|c| + |b|) / img plus U of
    the result; variances are the fp32 parameters exactly.
  - Decode: cx = var0 l0 pw + pcx rounds 5 times on terms bounded by |var0 l0 pw| + |pcx|, plus the rounding of pw itself
    (U |p2| + U |p0| times |var0 l0|); w = expf(var2 l2) pw carries (4 + |var2 l2|) U relative.  The test allows
    8 U (|pcx| + |pw| (1 + |var0 l0|) + |p0| + |p2|) + (6 + |var2 l2|) U w / 2 + U |box| per coordinate.
  - DetectionOutput decision by decision against test_ssd_host.detection_ref fed the boxes of fcuda_ssd_decode, bit for
    bit, over: no candidates, every score above the threshold at P = 8732 and C = 81, nms_top_k / keep_top_k truncation,
    exact score ties, zero-area boxes, one survivor per class and -0 / +0 scores under a negative threshold.  Each case (but the first) asserts suppression happened.
  - Batch independence, and modelgen's MobileNet-SSD end to end with fusion and CUDA graphs on and off: the backbone per
    layer within test_gpu_net_bounds's bounds, every head blob against the checks above from the net's own blobs, and the
    detections bit-identical with CUDA graphs on and off.  Fusion folds BatchNorm / Scale into the convolution weights,
    which rounds the backbone differently, so fused and unfused nets are each checked against their own blobs rather
    than against each other.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_gpu_net_bounds import CONV_TYPES, check_chain, fetch, load_model, rebuild_chains
from test_ssd_host import detection_ref, priorbox_ref

gpu = pytest.mark.gpu
U = 2.0 ** -23
AXES = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


def _bits_equal(a, b) -> bool:
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


# ---- Permute, Flatten, Reshape ------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("order", range(6))
@pytest.mark.parametrize("shape", [(3, 5, 7, 9), (2, 33, 17, 9), (1, 64, 19, 19), (2, 1, 1, 13), (4, 126, 10, 10)])
def test_permute_bit_exact(cuda, order, shape):
    from feathercnn_b200 import booster
    x = torch.randn(shape, device="cuda")
    got = booster.permute(x, order).cpu().numpy()
    want = np.transpose(x.cpu().numpy(), (0,) + tuple(a + 1 for a in AXES[order]))
    assert _bits_equal(got, want)


def _empty_bin(tmp_path):
    p = tmp_path / "empty.bin"
    p.write_bytes(b"")
    return str(p)


@gpu
def test_flatten_and_reshape_are_views(cuda, tmp_path):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText("7767517\n5 5\nInput data 0 1 data 0=6 1=5 2=4\nFlatten f 1 1 data flat\n"
                          "Reshape r 1 1 flat r2 0=10 1=-1\nReshape r3 1 1 r2 r3 0=0 1=3 2=-1\nSoftmax s 1 1 r2 sm 0=0\n")
    net.LoadWeights(_empty_bin(tmp_path))
    x = np.random.default_rng(0).standard_normal((2, 4, 5, 6)).astype(np.float32)
    net.Forward(x)
    p0, _ = net.ExtractDevice("data")
    for blob, shape, rank in (("flat", (2, 1, 1, 120), 1), ("r2", (2, 1, 12, 10), 2), ("r3", (2, 4, 3, 10), 3)):
        p, s = net.ExtractDevice(blob)
        assert p == p0 and s == shape and net.BlobDims(blob) == rank, blob
    # rank-2 axis 0 is h: the softmax runs down each of the 10 columns of 12
    sm = net.Extract("sm").reshape(2, 12, 10)
    assert np.allclose(sm.sum(axis=1), 1, atol=1e-5)


# ---- Softmax ------------------------------------------------------------------------------------------------------
def _softmax_check(x64, got, axis):
    m = x64.max(axis=axis, keepdims=True)
    e = np.exp(x64 - m)
    y = e / e.sum(axis=axis, keepdims=True)
    n = x64.shape[axis]
    spread = np.abs(x64 - m).max(axis=axis, keepdims=True)
    bound = 2 * y * ((n + 4) * U + 2 * U * spread) + 2.0 ** -140
    used = float((np.abs(got - y) / bound).max())
    assert used <= 1.0, used
    return used


@gpu
@pytest.mark.parametrize("outer, length, inner", [(1917, 21, 1), (7, 1, 1), (3, 100, 1), (5, 33, 7), (1, 64, 300),
                                                  (2, 8732, 1), (300, 5, 2)])
def test_softmax_axis_within_bound(cuda, outer, length, inner):
    from feathercnn_b200 import booster
    x = (torch.randn((3, outer, length, inner), device="cuda") * 6).contiguous()
    got = booster.softmax_axis(x, outer, length, inner).cpu().numpy().astype(np.float64)
    _softmax_check(x.cpu().numpy().astype(np.float64), got, 2)


@gpu
@pytest.mark.parametrize("rank_line, axis, np_axis", [
    ("Reshape r 1 1 data v 0=20 1=-1", "0=1", 2), ("Reshape r 1 1 data v 0=20 1=-1", "0=0", 1),
    ("Reshape r 1 1 data v 0=20 1=-1", "0=-1", 2), ("Flatten r 1 1 data v", "0=0", 2),
    ("Reshape r 1 1 data v 0=0 1=0 2=0", "0=0", 0), ("Reshape r 1 1 data v 0=0 1=0 2=0", "0=1", 1),
    ("Reshape r 1 1 data v 0=0 1=0 2=0", "0=2 1=1", 2), ("Reshape r 1 1 data v 0=0 1=0 2=0", "0=-3", 0)])
def test_softmax_layer_axes(cuda, tmp_path, rank_line, axis, np_axis):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(f"7767517\n3 3\nInput data 0 1 data 0=20 1=6 2=5\n{rank_line}\nSoftmax s 1 1 v out {axis}\n")
    net.LoadWeights(_empty_bin(tmp_path))
    x = (np.random.default_rng(1).standard_normal((2, 5, 6, 20)) * 4).astype(np.float32)
    net.Forward(x)
    _, s = net.ExtractDevice("v")
    got = net.Extract("out").reshape(2, *s[1:]).astype(np.float64)
    _softmax_check(x.reshape(2, *s[1:]).astype(np.float64), got, np_axis + 1 if np_axis < 3 else np_axis)


@gpu
def test_softmax_without_axis_is_the_whole_blob_kernel(cuda, tmp_path):
    from feathercnn_b200 import booster
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText("7767517\n2 2\nInput data 0 1 data 0=9 1=7 2=5\nSoftmax s 1 1 data out\n")
    net.LoadWeights(_empty_bin(tmp_path))
    x = (np.random.default_rng(2).standard_normal((3, 5, 7, 9)) * 3).astype(np.float32)
    net.Forward(x)
    want = booster.softmax(torch.from_numpy(x).cuda()).cpu().numpy()
    assert _bits_equal(net.Extract("out"), want)


# ---- PriorBox and decode ------------------------------------------------------------------------------------------
PRIOR_CASES = [
    dict(fw=10, fh=10, iw=300, ih=300, min_sizes=[105.0], max_sizes=[150.0], ars=[2.0, 3.0], flip=True, clip=True),
    dict(fw=19, fh=19, iw=300, ih=300, min_sizes=[60.0], max_sizes=[], ars=[2.0], flip=True, clip=False),
    dict(fw=7, fh=5, iw=320, ih=200, min_sizes=[30.0, 50.0], max_sizes=[45.0, 70.0], ars=[2.0, 1.0, 0.5], flip=False,
         clip=False, step=(48.0, 41.0), offset=0.25),
    dict(fw=3, fh=9, iw=97, ih=301, min_sizes=[21.5], max_sizes=[], ars=[], flip=True, clip=True, offset=0.0),
]


def _priors(case):
    from feathercnn_b200 import booster
    p = booster.priorbox_param(case["min_sizes"], case["max_sizes"], case["ars"], flip=case["flip"], clip=case["clip"],
                               step=case.get("step", (0.0, 0.0)), offset=case.get("offset", 0.5))
    return booster.priorbox(p, case["fw"], case["fh"], case["iw"], case["ih"])


@gpu
@pytest.mark.parametrize("case", PRIOR_CASES, ids=[f"prior{i}" for i in range(len(PRIOR_CASES))])
def test_priorbox_within_bound(cuda, case):
    got = _priors(case).cpu().numpy()
    want = priorbox_ref(case["fw"], case["fh"], case["iw"], case["ih"], case["min_sizes"], case["max_sizes"], case["ars"],
                        case["flip"], case["clip"], case.get("step", (0.0, 0.0)), case.get("offset", 0.5))
    assert got.shape == (2, want.size)
    img = np.tile([case["iw"], case["ih"]], want.size // 2).astype(np.float64)
    # magnitudes of the centre and the half size in pixels: |c| + |b| <= (|v| + 2 |b/2|) img, b/2 <= max size
    half = max(case["min_sizes"] + case["max_sizes"]) * 2.0
    bound = 8 * U * (np.abs(want) * img + 2 * half) / img + U * np.abs(want) + 2.0 ** -149
    assert float((np.abs(got[0] - want) / bound).max()) <= 1.0
    var = np.tile(np.float32([0.1, 0.1, 0.2, 0.2]), want.size // 4)
    assert _bits_equal(got[1], var)


def _random_priors(rng, P):
    c = rng.uniform(0.05, 0.95, (P, 2))
    wh = rng.uniform(0.02, 0.6, (P, 2))
    boxes = np.concatenate([c - wh / 2, c + wh / 2], 1).astype(np.float32).reshape(-1)
    var = np.tile(np.float32([0.1, 0.1, 0.2, 0.2]), P)
    return np.stack([boxes, var])


def _decode_ref(loc, priors):
    P = priors.shape[1] // 4
    pb = priors[0].reshape(P, 4).astype(np.float64)
    v = priors[1].reshape(P, 4).astype(np.float64)
    l = loc.reshape(loc.shape[0], P, 4).astype(np.float64)
    pw, ph = pb[:, 2] - pb[:, 0], pb[:, 3] - pb[:, 1]
    pcx, pcy = (pb[:, 0] + pb[:, 2]) / 2, (pb[:, 1] + pb[:, 3]) / 2
    cx, cy = v[:, 0] * l[..., 0] * pw + pcx, v[:, 1] * l[..., 1] * ph + pcy
    w, h = np.exp(v[:, 2] * l[..., 2]) * pw, np.exp(v[:, 3] * l[..., 3]) * ph
    want = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], -1)
    sx = 8 * U * (np.abs(pcx) + pw * (1 + np.abs(v[:, 0] * l[..., 0])) + np.abs(pb[:, 0]) + np.abs(pb[:, 2]))
    sy = 8 * U * (np.abs(pcy) + ph * (1 + np.abs(v[:, 1] * l[..., 1])) + np.abs(pb[:, 1]) + np.abs(pb[:, 3]))
    bw = (6 + np.abs(v[:, 2] * l[..., 2])) * U * w / 2
    bh = (6 + np.abs(v[:, 3] * l[..., 3])) * U * h / 2
    bound = np.stack([sx + bw, sy + bh, sx + bw, sy + bh], -1) + U * np.abs(want) + 2.0 ** -149
    return want, bound


@gpu
@pytest.mark.parametrize("P, batch", [(1917, 2), (8732, 1), (7, 5)])
def test_decode_within_bound(cuda, P, batch):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(P)
    priors = _random_priors(rng, P)
    loc = rng.standard_normal((batch, 4 * P)).astype(np.float32) * 2
    got = booster.ssd_decode(torch.from_numpy(loc).cuda(), torch.from_numpy(priors).cuda()).cpu().numpy()
    want, bound = _decode_ref(loc, priors)
    assert float((np.abs(got - want) / bound).max()) <= 1.0
    # the real priors of a PriorBox as well
    pri = _priors(PRIOR_CASES[0]).cpu().numpy()
    loc2 = rng.standard_normal((1, pri.shape[1])).astype(np.float32)
    got2 = booster.ssd_decode(torch.from_numpy(loc2).cuda(), torch.from_numpy(pri).cuda()).cpu().numpy()
    want2, bound2 = _decode_ref(loc2, pri)
    assert float((np.abs(got2 - want2) / bound2).max()) <= 1.0


# ---- DetectionOutput ----------------------------------------------------------------------------------------------
def _run_detection(loc, conf, priors, C, thr, nms, top, keep):
    from feathercnn_b200 import booster
    dl, dc, dp = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (loc, conf, priors))
    boxes = booster.ssd_decode(dl, dp).cpu().numpy()
    got = booster.detection_output(dl, dc, dp, C, thr, nms, top, keep).cpu().numpy()
    want, suppressed = detection_ref(boxes, conf, C, thr, nms, top, keep)
    return got, want, suppressed


def _softmax_scores(rng, n, P, C, gain):
    z = rng.standard_normal((n, P, C)) * gain
    e = np.exp(z - z.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32).reshape(n, P * C)


def _case(name, rng):
    """(loc, conf, priors, C, conf_threshold, nms_threshold, nms_top_k, keep_top_k)"""
    if name == "no_candidates":
        P, C = 500, 21
        return (rng.standard_normal((2, 4 * P)).astype(np.float32), _softmax_scores(rng, 2, P, C, 0.1),
                _random_priors(rng, P), C, 0.9, 0.45, 100, 50)
    if name == "all_above_8732x81":
        P, C = 8732, 81
        conf = rng.uniform(0.01, 1.0, (1, P * C)).astype(np.float32)
        return (rng.standard_normal((1, 4 * P)).astype(np.float32), conf, _random_priors(rng, P), C, 0.0, 0.45, 400, 200)
    if name == "truncation":
        P, C = 300, 6
        return (rng.standard_normal((2, 4 * P)).astype(np.float32) * 0.5, _softmax_scores(rng, 2, P, C, 3.0),
                _random_priors(rng, P), C, 0.05, 0.3, 7, 9)
    if name == "ties":
        P, C = 400, 5
        conf = (rng.integers(1, 5, (2, P * C)) / 8).astype(np.float32)
        pri = _random_priors(rng, 40)
        pri = np.tile(pri.reshape(2, 40, 4), (1, 10, 1)).reshape(2, -1)  # repeated priors: many overlapping boxes
        return (rng.standard_normal((2, 4 * P)).astype(np.float32) * 0.3, conf, pri, C, 0.2, 0.5, 150, 300)
    if name == "zero_area":
        P, C = 600, 4
        loc = rng.standard_normal((1, P, 4)).astype(np.float32) * 0.3
        loc[0, ::3, 2] = -1000.0  # expf underflows: width 0
        loc[0, ::5, 3] = -1000.0
        return (loc.reshape(1, -1), _softmax_scores(rng, 1, P, C, 2.0), _random_priors(rng, P), C, 0.1, 0.4, 300, 200)
    if name == "one_survivor":
        P, C = 256, 3
        pri = np.tile(_random_priors(rng, 1).reshape(2, 1, 4), (1, P, 1)).reshape(2, -1)
        return (np.zeros((2, 4 * P), np.float32), rng.uniform(0.3, 1.0, (2, P * C)).astype(np.float32), pri, C, 0.2,
                0.5, 200, 100)
    if name == "signed_zero":
        # -0 and +0 scores above a negative threshold are equal: ordered by prior within a class and by class in the
        # merge, and each row keeps its score's sign; duplicated priors give suppression
        P, C = 64, 3
        conf = np.float32([-0.0, 0.0, -0.25])[rng.integers(0, 3, (2, P * C))]
        pri = np.tile(_random_priors(rng, 16).reshape(2, 16, 4), (1, 4, 1)).reshape(2, -1)
        return (np.zeros((2, 4 * P), np.float32), conf, pri, C, -0.5, 0.45, 40, 60)
    raise AssertionError(name)


DET_CASES = ["no_candidates", "all_above_8732x81", "truncation", "ties", "zero_area", "one_survivor", "signed_zero"]


@gpu
@pytest.mark.parametrize("name", DET_CASES)
def test_detection_output_decisions(cuda, name):
    rng = np.random.default_rng(DET_CASES.index(name) + 11)
    loc, conf, priors, C, thr, nms, top, keep = _case(name, rng)
    got, want, suppressed = _run_detection(loc, conf, priors, C, thr, nms, top, keep)
    assert _bits_equal(got, want), (name, np.argwhere(got != want)[:5])
    n_det = int((want[..., 0] >= 0).sum())
    if name == "no_candidates":
        assert n_det == 0 and np.all(want[..., 0] == -1) and np.all(want[..., 1:] == 0)
        return
    assert suppressed > 0 and n_det > 0, (name, suppressed, n_det)
    if name == "one_survivor":
        assert np.all(want[:, :C - 1, 0] >= 1) and np.all(want[:, C - 1:, 0] == -1)
    if name == "truncation":
        assert np.all(want[..., 0] >= 0)  # keep_top_k rows all filled, each class cut at nms_top_k
    if name == "zero_area":
        assert np.any((want[..., 4] == want[..., 2]) & (want[..., 0] >= 0))


@gpu
def test_detection_output_batch_independent(cuda):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(5)
    P, C = 1917, 21
    loc = rng.standard_normal((4, 4 * P)).astype(np.float32)
    conf = _softmax_scores(rng, 4, P, C, 3.0)
    pri = torch.from_numpy(_random_priors(rng, P)).cuda()
    batched = booster.detection_output(torch.from_numpy(loc).cuda(), torch.from_numpy(conf).cuda(), pri, C, 0.05, 0.45,
                                       100, 100).cpu().numpy()
    for i in range(4):
        alone = booster.detection_output(torch.from_numpy(loc[i:i + 1]).cuda(), torch.from_numpy(conf[i:i + 1]).cuda(), pri,
                                         C, 0.05, 0.45, 100, 100).cpu().numpy()
        assert _bits_equal(alone[0], batched[i]), i


# ---- MobileNet-SSD end to end -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ssd_model(tmp_path_factory):
    from feathercnn_b200.tools import modelgen
    m = modelgen.mobilenet_ssd(conf_threshold=0.02, conf_gain=3.0)
    param, binf = m.save(tmp_path_factory.mktemp("ssd") / "mobilenet_ssd")
    return m, param, binf, load_model(param, binf)


def _check_head(net, m, idx):
    """The head's blobs from the net's own inputs: Permute bit-exact, Flatten / Reshape views, Concat bit-exact,
    Softmax within its bound, PriorBox bit-equal to the kernel alone, DetectionOutput decision by decision."""
    from feathercnn_b200 import booster
    def host(b):  # PriorBox blobs hold one image, read by every image of the batch
        return fetch(net, b, idx if net.BlobShape(b)[0] > 1 else [0]).float().cpu().numpy()
    lines = [L.split() for L in m.lines]
    candidates = 0
    for L in lines:
        typ, name, nb, nt = L[0], L[1], int(L[2]), int(L[3])
        bottoms, tops = L[4:4 + nb], L[4 + nb:4 + nb + nt]
        if typ == "Permute":
            x = host(bottoms[0])
            assert _bits_equal(host(tops[0]), np.transpose(x, (0, 2, 3, 1))), name
        elif typ in ("Flatten", "Reshape"):
            assert net.ExtractDevice(tops[0])[0] == net.ExtractDevice(bottoms[0])[0], name
        elif typ == "Concat":
            axis = 3  # rank 1: w; rank 2, axis 1: w
            want = np.concatenate([host(b) for b in bottoms], axis=axis)
            assert _bits_equal(host(tops[0]), want), name
        elif typ == "Softmax":
            _softmax_check(host(bottoms[0]).astype(np.float64), host(tops[0]).astype(np.float64), 3)
        elif typ == "PriorBox":
            _, c, fh, fw = net.BlobShape(bottoms[0])
            kv = dict(t.split("=", 1) for t in L[4 + nb + nt:])
            arr = lambda k: [float(v) for v in kv[k].split(",")[1:]] if k in kv else []  # noqa: E731
            p = booster.priorbox_param(arr("-23300"), arr("-23301"), arr("-23302"), flip=int(kv["7"]), clip=int(kv["8"]),
                                       offset=float(kv["13"]))
            _, _, ih, iw = net.BlobShape("data")
            want = booster.priorbox(p, fw, fh, iw, ih).cpu().numpy()
            got = fetch(net, tops[0], [0]).float().cpu().numpy().reshape(want.shape)
            assert _bits_equal(got, want), name
        elif typ == "DetectionOutput":
            kv = dict(t.split("=", 1) for t in L[4 + nb + nt:])
            C, nms, top, keep, thr = int(kv["0"]), float(kv["1"]), int(kv["2"]), int(kv["3"]), float(kv["4"])
            loc = fetch(net, bottoms[0], idx).float().reshape(len(idx), -1).contiguous()  # noqa: F841
            conf = host(bottoms[1]).reshape(len(idx), -1)
            pri = fetch(net, bottoms[2], [0]).float().reshape(2, -1).contiguous()
            boxes = booster.ssd_decode(loc, pri).cpu().numpy()
            want, suppressed = detection_ref(boxes, conf, C, np.float32(thr), np.float32(nms), top, keep)
            got = host(tops[0]).reshape(want.shape)
            assert _bits_equal(got, want), name
            candidates = int((conf.reshape(len(idx), -1, C)[..., 1:] > np.float32(thr)).sum())
            assert suppressed > 0, suppressed
    return candidates


SSD_SETTINGS = [(True, True), (True, False), (False, True), (False, False)]


@gpu
def test_mobilenet_ssd_end_to_end(cuda, ssd_model):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m, param, binf, layers = ssd_model
    batch = 2
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])
    idx = list(range(batch))
    dets = []
    for fusion, graph in SSD_SETTINGS:
        net = Net(fusion=fusion, cuda_graph=graph)
        net.LoadParam(param)
        net.LoadWeights(binf)
        for _ in range(3 if graph else 1):
            net.Forward(x)
        net.Synchronize()
        names = set(net.BlobNames())
        for blob, (c, h, w) in m.shape.items():
            if blob in names:
                n, bc, bh, bw = net.BlobShape(blob)
                assert (bc, bh, bw) == (c, h, w) and net.BlobDims(blob) == m.rank.get(blob, 3), blob
        assert net.BlobShape("mbox_priorbox") == (1, 1, 2, 4 * 1917)
        chains, _ = rebuild_chains(layers, net.LayerFusedAway, names)
        failures = []
        for ch in chains:
            if ch.head["type"] not in CONV_TYPES + ("BatchNorm", "Scale", "ReLU"):
                continue
            algo = net.LayerConvAlgo(ch.head["name"]) if ch.head["type"] in CONV_TYPES else -1
            ins = {b: fetch(net, b, idx) for b in dict.fromkeys(ch.bottoms)}
            got = {t: fetch(net, t, idx) for t in ch.tops}
            for top, used, rel, kind, path in check_chain(ch, ins, got, 2, algo):
                if used > 1.0:
                    failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
        assert not failures, "\n".join(failures[:20])
        candidates = _check_head(net, m, idx)
        assert candidates >= 200, candidates
        dets.append(net.Extract("detection_out"))
        assert int((dets[-1][..., 0] >= 0).sum()) > 0
        del net
    assert _bits_equal(dets[0], dets[1]) and _bits_equal(dets[2], dets[3])


@gpu
def test_mobilenet_ssd_batch_independent(cuda, ssd_model):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m, param, binf, _ = ssd_model
    xs = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(3)])
    net = Net(fusion=True, cuda_graph=True)
    net.LoadParam(param)
    net.LoadWeights(binf)
    net.Forward(xs)
    batched = net.Extract("detection_out")
    alone = Net(fusion=True, cuda_graph=True)
    alone.LoadParam(param)
    alone.LoadWeights(binf)
    for i in (0, 2):
        alone.Forward(xs[i:i + 1])
        assert _bits_equal(alone.Extract("detection_out")[0], batched[i]), i


@gpu
def test_ssd_tiny_runs_in_a_graph(cuda, tmp_path):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.ssd_tiny()
    param, binf = m.save(tmp_path / "ssd_tiny")
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(4)])
    outs = []
    for graph in (False, True):
        net = Net(fusion=True, cuda_graph=graph)
        net.LoadParam(param)
        net.LoadWeights(binf)
        for _ in range(3):
            net.Forward(x)
        outs.append(net.Extract("detection_out"))
    assert _bits_equal(outs[0], outs[1]) and outs[0].shape == (4, 1, 100, 6)
    assert int((outs[0][..., 0] >= 0).sum()) > 0
