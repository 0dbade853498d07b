"""The YOLO detection head on the GPU.

  - Decode against float64 (test_yolo_host.yolo_decode_ref), per element.  U = 2^-23; each fp32 operation rounds by at most
    U relative and CUDA's expf errs by at most 2 ulp (2 U relative).  Doubling every bound below gives the test's margin.
      s(t) = 1 / (1 + e), e = expf(-t): 1 + e carries 2 U e + U (1 + e) <= 3 U (1 + e), the division one more U, so
        s has relative error <= 4 U.
      c = (j + s) / w: 4 U s + U (j + s) on the sum, then U on the quotient: <= 6 U c.
      bw = expf(tw) * bias / norm: 2 U + U + U = 4 U relative.  bw * 0.5 is exact.
      a coordinate c -+ bw * 0.5 adds U of itself: |err| <= 6 U c + 2 U bw + U |coord|.
      v3 confidence 1 / (1 + a (1 + b)) with a = expf(-obj), b = expf(-logit_max): (1 + b) <= 3 U, a (1 + b) <= 6 U,
        1 + a (1 + b) <= 7 U of itself, the quotient <= 8 U relative.  The logits are read exactly, so the class is the
        same argmax bit for bit.
      v2 confidence s(obj) * p: with r = max |l - max|, each exponential carries U r + 2 U, the class-order sum of C of
        them (C - 1) U more, the quotient U: p <= (C + 4) U + 2 U r relative (twice the exponential's error, once for the
        numerator and once inside the sum); with s(obj) (4 U) and the product (U): <= (C + 9) U + 2 U r.  The class is
        compared where the float64 runner-up probability is below (1 - 8 x that bound) times the maximum.
    Cover: odd grids, 1 to 4 scales, C = 1 / 20 / 80, batch > 1, and (v2) the bottom left unmodified.
  - Selection, NMS and output decision by decision, bit for bit, against test_yolo_host.yolo_ref fed the kernel's own
    decoded candidates (fcuda_yolo_decode): no candidates; exactly 32 / 33 / 1023 / 1024 / 1025; nms_top_k / keep_top_k
    truncation; exact confidence ties; zero-area boxes; one survivor; all 10647 slots of the 416 x 416 YOLOv3 geometry
    above the threshold.  Every case but the first asserts that NMS suppressed something.
  - A seeded sweep of random geometries across the decode (scale boundaries, grid sides, C, num_box), select (candidate
    counts around 32 and 1024, nms_top_k), mask (row blocks of 32) and sweep (keep_top_k) boundaries.
  - Batch independence of the layer and of the nets; a channel-count mismatch fails at Reshape.
  - modelgen's mobilenetv2_yolov3 and mobilenet_yolov2 end to end with fusion and CUDA graphs on and off: the backbone per
    layer within the float64 bounds of test_gpu_net_bounds / test_gpu_clip_prelu, nearest Interp and Concat bit-exact,
    the head from the net's own blobs, and the detections bit-identical with CUDA graphs on and off.  YOLOv3 has more
    than 1024 candidates.  yolo_tiny runs inside a CUDA graph.
"""
from __future__ import annotations

import zlib

import numpy as np
import pytest
import torch

from test_gpu_net_bounds import CONV_TYPES, check_chain, fetch, load_model, rebuild_chains
from test_yolo_host import yolo_decode_ref, yolo_ref

gpu = pytest.mark.gpu
U = 2.0 ** -23
COCO = [10, 13, 16, 30, 33, 23, 30, 61, 62, 45, 59, 119, 116, 90, 156, 198, 373, 326]
VOC = [1.08, 1.19, 3.42, 4.41, 6.63, 11.38, 9.42, 5.11, 16.62, 10.52]


def _bits_equal(a, b) -> bool:
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _param(version, C, B, grids, biases, mask=(), scales=(), thr=0.01, nms=0.45, top=1024, keep=1024):
    from feathercnn_b200 import booster
    return booster.yolo_param(version, C, B, grids, biases, mask, scales, thr, nms, top, keep)


def _cuda(xs):
    return [torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda() for x in xs]


# ---- decode -------------------------------------------------------------------------------------------------------
def check_decode(xs, p, got):
    """got = (scores, classes, boxes) of fcuda_yolo_decode for inputs xs (float32 arrays); asserts the bounds above and
    returns the largest share of a bound used."""
    C, B = p.num_class, p.num_box
    mask = list(p.mask)[:p.num_scales * B]
    scales = list(p.anchors_scale)[:p.num_scales]
    biases = list(p.biases)[:p.num_biases]
    s_ref, c_ref, b_ref, second = yolo_decode_ref(xs, p.version, C, B, biases, mask, scales)
    s, c, b = (t.cpu().numpy() for t in got)
    # coordinates
    cxy = (b_ref[..., 0:2] + b_ref[..., 2:4]) / 2
    wh = b_ref[..., 2:4] - b_ref[..., 0:2]
    c4 = np.concatenate([cxy, cxy], -1)
    h4 = np.concatenate([wh, wh], -1)
    bound = 2 * (6 * U * np.abs(c4) + 2 * U * h4 + U * np.abs(b_ref)) + 2.0 ** -140
    used = float((np.abs(b - b_ref) / bound).max())
    assert used <= 1.0, ("box", used)
    # confidence and class
    if p.version == 3:
        rel = np.full_like(s_ref, 8 * U)
        assert np.array_equal(c, c_ref)
    else:
        spread = []
        for x in xs:
            x = np.asarray(x, np.float64).reshape(x.shape[0], B, 5 + C, -1)[:, :, 5:]
            spread.append((x.max(2) - x.min(2)).reshape(x.shape[0], -1))
        r = np.concatenate(spread, 1)
        rel = (C + 9) * U + 2 * U * r
        pmax = s_ref / (1 / (1 + np.exp(-np.concatenate([np.asarray(x, np.float64).reshape(
            x.shape[0], B, 5 + C, -1)[:, :, 4].reshape(x.shape[0], -1) for x in xs], 1))))
        clear = second < (1 - 8 * rel) * pmax
        assert np.array_equal(c[clear], c_ref[clear])
    sb = 2 * rel * s_ref + 2.0 ** -140
    used_s = float((np.abs(s - s_ref) / sb).max())
    assert used_s <= 1.0, ("confidence", used_s)
    return max(used, used_s)


DECODE_CASES = [
    dict(version=3, C=80, B=3, grids=[(13, 13), (26, 26), (52, 52)], batch=2, biases=COCO, mask=[6, 7, 8, 3, 4, 5, 0, 1, 2],
         scales=[32.0, 16.0, 8.0]),
    dict(version=3, C=1, B=3, grids=[(7, 5), (3, 11)], batch=3, biases=COCO[:12], mask=[3, 4, 5, 0, 1, 2],
         scales=[9.0, 13.5]),
    dict(version=3, C=20, B=2, grids=[(1, 1), (5, 3), (9, 17), (2, 33)], batch=2, biases=COCO[:16],
         mask=[7, 6, 5, 4, 3, 2, 1, 0], scales=[64.0, 30.5, 7.0, 3.3]),
    dict(version=2, C=20, B=5, grids=[(13, 13)], batch=2, biases=VOC),
    dict(version=2, C=1, B=5, grids=[(9, 7)], batch=1, biases=VOC),
    dict(version=2, C=80, B=3, grids=[(5, 17)], batch=3, biases=VOC[:6]),
]


@gpu
@pytest.mark.parametrize("case", DECODE_CASES, ids=[f"v{c['version']}-C{c['C']}-s{len(c['grids'])}" for c in DECODE_CASES])
def test_decode_within_bound(cuda, case):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(len(case["grids"]) * 100 + case["C"])
    xs = [(rng.standard_normal((case["batch"], case["B"] * (5 + case["C"]), h, w)) * 2).astype(np.float32)
          for h, w in case["grids"]]
    p = _param(case["version"], case["C"], case["B"], case["grids"], case["biases"], case.get("mask", ()),
               case.get("scales", ()))
    dev = _cuda(xs)
    before = [t.clone() for t in dev]
    got = booster.yolo_decode(dev, p)
    torch.cuda.synchronize()
    check_decode(xs, p, got)
    assert all(torch.equal(a, b) for a, b in zip(dev, before))  # v2's softmax does not write its bottom
    # the layer's output boxes and confidences are the decode's bits
    out = booster.yolo_detection(dev, p).cpu().numpy()
    s, c, b = (t.cpu().numpy() for t in got)
    want, _, _ = yolo_ref(s, c, b, p.confidence_threshold, p.nms_threshold, p.nms_top_k, p.keep_top_k)
    assert _bits_equal(out, want)


# ---- selection, NMS, output ---------------------------------------------------------------------------------------
def _candidates_input(rng, batch, C, B, grid, k, big=1.0):
    """v3 input with exactly k candidates per image at threshold 0.5: objectness 4 + U(0, 1) there, -30 elsewhere."""
    h, w = grid
    x = (rng.standard_normal((batch, B, 5 + C, h, w)) * 0.5).astype(np.float32)
    x[:, :, 4] = -30.0
    for n in range(batch):
        slots = rng.choice(B * h * w, size=k, replace=False)
        pp, cell = slots // (h * w), slots % (h * w)
        x[n, pp, 4, cell // w, cell % w] = 4.0 + rng.uniform(0, 1, k)
    return [x.reshape(batch, B * (5 + C), h, w)]


def _sel_case(name, rng):
    """(inputs, param) per case."""
    anchors = [200, 200, 256, 192, 160, 240, 220, 180]  # most of the 256 x 256 network: boxes overlap
    if name == "no_candidates":
        x = _candidates_input(rng, 2, 4, 2, (32, 32), 0)
        return x, _param(3, 4, 2, [(32, 32)], anchors, [0, 1], [8.0], thr=0.5)
    if name.startswith("k"):
        k = int(name[1:])
        x = _candidates_input(rng, 2, 4, 2, (32, 32), k)
        return x, _param(3, 4, 2, [(32, 32)], anchors, [0, 1], [8.0], thr=0.5)
    if name == "truncation":
        x = _candidates_input(rng, 2, 4, 2, (32, 32), 600)
        return x, _param(3, 4, 2, [(32, 32)], anchors, [2, 3], [8.0], thr=0.5, top=100, keep=20)
    if name == "ties":
        # three objectness values and one class pattern: confidences tie exactly across hundreds of slots
        x = np.zeros((2, 2, 9, 24, 24), np.float32)
        x[:, :, :4] = rng.standard_normal((2, 2, 4, 24, 24)) * 0.3
        x[:, :, 4] = np.float32([1.0, 2.0, 3.0])[rng.integers(0, 3, (2, 2, 24, 24))]
        x[:, :, 5] = 2.0
        return [x.reshape(2, 18, 24, 24)], _param(3, 4, 2, [(24, 24)], anchors, [0, 1], [8.0], thr=0.5, top=1024,
                                                  keep=700)
    if name == "zero_area":
        x = _candidates_input(rng, 1, 4, 2, (32, 32), 900)[0].reshape(1, 2, 9, 32, 32)
        x[:, 0, 2, ::3] = -200.0  # expf underflows: width 0
        x[:, 1, 3, :, ::5] = -200.0
        return [x.reshape(1, 18, 32, 32)], _param(3, 4, 2, [(32, 32)], anchors, [0, 1], [8.0], thr=0.5)
    if name == "one_survivor":
        # anchors 1000 x the network: every box covers the others almost exactly
        x = _candidates_input(rng, 2, 3, 2, (8, 8), 128)[0].reshape(2, 2, 8, 8, 8)
        x[:, :, 2:4] = 0.0
        return [x.reshape(2, 16, 8, 8)], _param(3, 3, 2, [(8, 8)], [64000, 64000, 64000, 64000], [0, 1], [8.0], thr=0.5)
    if name == "all_10647":
        xs = [(rng.standard_normal((1, 255, g, g)) * 2).astype(np.float32) for g in (13, 26, 52)]
        return xs, _param(3, 80, 3, [(13, 13), (26, 26), (52, 52)], COCO, [6, 7, 8, 3, 4, 5, 0, 1, 2], [32.0, 16.0, 8.0],
                          thr=0.0)
    raise AssertionError(name)


SEL_CASES = ["no_candidates", "k32", "k33", "k1023", "k1024", "k1025", "truncation", "ties", "zero_area", "one_survivor",
             "all_10647"]


def run_and_check(xs, p):
    """The layer against yolo_ref fed the kernel's decode, bit for bit; returns (want, suppressed, candidates)."""
    from feathercnn_b200 import booster
    dev = _cuda(xs)
    s, c, b = (t.cpu().numpy() for t in booster.yolo_decode(dev, p))
    got = booster.yolo_detection(dev, p).cpu().numpy()
    want, suppressed, candidates = yolo_ref(s, c, b, p.confidence_threshold, p.nms_threshold, p.nms_top_k,
                                            p.keep_top_k)
    assert _bits_equal(got, want), np.argwhere(got.view(np.int32) != want.view(np.int32))[:5]
    return want, suppressed, candidates, s


@gpu
@pytest.mark.parametrize("name", SEL_CASES)
def test_selection_nms_decisions(cuda, name):
    rng = np.random.default_rng(SEL_CASES.index(name) + 31)
    xs, p = _sel_case(name, rng)
    want, suppressed, candidates, s = run_and_check(xs, p)
    n_img = want.shape[0]
    n_det = int((want[..., 0] >= 0).sum())
    if name == "no_candidates":
        assert candidates == 0 and n_det == 0 and np.all(want[..., 1:] == 0)
        return
    assert suppressed > 0 and n_det > 0, (name, suppressed, n_det)
    if name.startswith("k"):
        assert candidates == n_img * int(name[1:])
    if name == "truncation":
        assert np.all(want[..., 0] >= 1)  # 20 rows filled from the first 100 candidates
    if name == "ties":
        kept = want[0][want[0, :, 0] >= 0]
        assert len(np.unique(kept[:, 1])) <= 3 and candidates > 2 * 1024
    if name == "zero_area":
        assert np.any((want[..., 4] == want[..., 2]) & (want[..., 0] >= 0))
    if name == "one_survivor":
        assert np.all(want[:, 0, 0] >= 1) and np.all(want[:, 1:, 0] == -1)
    if name == "all_10647":
        assert candidates == 10647


# ---- random geometries --------------------------------------------------------------------------------------------
SWEEP_N = 48


def _sweep_case(i):
    rng = np.random.default_rng(zlib.crc32(f"yolo{i}".encode()))
    version = 2 if i % 4 == 0 else 3
    scales = 1 if version == 2 else int(rng.integers(1, 5))
    B = int(rng.integers(1, 17))
    C = int(rng.choice([1, 2, 7, 20, 33, 80, 129]))
    grids = []
    for _ in range(scales):
        grids.append((int(rng.integers(1, 25)), int(rng.integers(1, 25))))
    batch = int(rng.integers(1, 4))
    n_anchor = B * scales if version == 3 else B
    biases = [float(v) for v in rng.uniform(0.5, 12.0, 2 * n_anchor) * (1 if version == 2 else 16)]
    mask = [int(v) for v in rng.permutation(n_anchor)] if version == 3 else []
    anchors_scale = [float(v) for v in rng.uniform(4.0, 40.0, scales)] if version == 3 else []
    top = int(rng.choice([1, 31, 32, 33, 64, 500, 1023, 1024]))
    keep = int(rng.choice([1, 20, 32, 33, 1000, 1024]))
    thr = float(rng.choice([0.0, 0.05, 0.3, 0.6]))
    nms = float(rng.choice([0.0, 0.3, 0.45, 0.7, 1.0]))
    obj = float(rng.uniform(-4, 3))
    xs = []
    for h, w in grids:
        x = rng.standard_normal((batch, B, 5 + C, h, w)) * 1.5
        x[:, :, 4] += obj
        xs.append(x.reshape(batch, B * (5 + C), h, w).astype(np.float32))
    p = _param(version, C, B, grids, biases, mask, anchors_scale, thr, nms, top, keep)
    return xs, p


def test_sweep_cases_cover_the_boundaries():
    """The sweep spans 1 to 4 scales, both versions, C of 1 and > 32, candidate counts on both sides of 32 and 1024 is
    left to the GPU run; here: the shapes are valid and the top-k choices reach the boundaries."""
    from feathercnn_b200._lib import fcuda
    import ctypes
    tops, keeps, scales, versions = set(), set(), set(), set()
    for i in range(SWEEP_N):
        xs, p = _sweep_case(i)
        n = ctypes.c_size_t()
        assert fcuda().fcuda_yolo_detection_workspace_size(ctypes.byref(p), xs[0].shape[0], ctypes.byref(n)) == 0, i
        tops.add(p.nms_top_k)
        keeps.add(p.keep_top_k)
        scales.add(p.num_scales)
        versions.add(p.version)
    assert {32, 33, 1024} <= tops and {32, 33, 1024} <= keeps and scales == {1, 2, 3, 4} and versions == {2, 3}


@gpu
@pytest.mark.parametrize("i", range(SWEEP_N))
def test_random_geometry_matches_reference(cuda, i):
    from feathercnn_b200 import booster
    xs, p = _sweep_case(i)
    dev = _cuda(xs)
    check_decode(xs, p, booster.yolo_decode(dev, p))
    run_and_check(xs, p)


# ---- batch independence, Reshape --------------------------------------------------------------------------------
@gpu
def test_layer_batch_independent(cuda):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(7)
    xs = []
    for g in (13, 26, 52):
        x = rng.standard_normal((4, 3, 85, g, g)) * 2
        x[:, :, 4] -= 3.0  # fewer candidates, but still many
        xs.append(x.reshape(4, 255, g, g).astype(np.float32))
    p = _param(3, 80, 3, [(13, 13), (26, 26), (52, 52)], COCO, [6, 7, 8, 3, 4, 5, 0, 1, 2], [32.0, 16.0, 8.0], thr=0.05)
    batched = booster.yolo_detection(_cuda(xs), p).cpu().numpy()
    for i in range(4):
        alone = booster.yolo_detection(_cuda([x[i:i + 1] for x in xs]), p).cpu().numpy()
        assert _bits_equal(alone[0], batched[i]), i
    assert int((batched[..., 0] >= 0).sum()) > 0


@gpu
def test_channel_count_checked_at_reshape(cuda, tmp_path):
    """29 channels are not num_box * (5 + num_class) = 30: Yolov3DetectionOutput's Reshape fails (FEATHER_ERR_TOPOLOGY),
    which Net reports as FEATHER_ERR_WEIGHTS (-100) like every shape failure."""
    from feathercnn_b200.net import FeatherError, Net
    net = Net()
    net.LoadParamFromText("7767517\n2 2\nInput a 0 1 a 0=4 1=4 2=29\nYolov3DetectionOutput d 1 1 a out 0=5 1=5 "
                          "-23304=10,1.0,1.0,2.0,2.0,3.0,3.0,4.0,4.0,5.0,5.0 -23305=5,0,1,2,3,4 -23306=1,8.0\n")
    empty = tmp_path / "empty.bin"
    empty.write_bytes(b"")
    net.LoadWeights(str(empty))
    with pytest.raises(FeatherError) as e:
        net.Forward(np.zeros((1, 29, 4, 4), np.float32))
    assert e.value.code == -100


# ---- models end to end --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def yolo_models(tmp_path_factory):
    from feathercnn_b200.tools import modelgen
    d = tmp_path_factory.mktemp("yolo")
    out = {}
    for name in ("mobilenetv2_yolov3", "mobilenet_yolov2"):
        m = modelgen.ZOO[name]()
        param, binf = m.save(d / name)
        out[name] = (m, param, binf, load_model(param, binf))
    return out


def _check_backbone(net, layers, idx):
    """Every chain but the head's own layers within its float64 bound: ReLU nets through test_gpu_net_bounds.check_chain,
    Clip nets through test_gpu_clip_prelu.restate; nearest Interp x2 and Concat bit-exact."""
    from test_gpu_clip_prelu import restate
    names = set(net.BlobNames())
    chains, _ = rebuild_chains(layers, net.LayerFusedAway, names)
    clip_net = any(L["type"] == "Clip" for L in layers)
    failures = []
    for ch in chains:
        typ = ch.head["type"]
        if typ == "Interp":
            x = fetch(net, ch.head["bottoms"][0], idx)
            want = x.repeat_interleave(2, 2).repeat_interleave(2, 3)
            assert torch.equal(fetch(net, ch.tops[0], idx), want), ch.head["name"]
            continue
        if typ == "Concat":
            want = torch.cat([fetch(net, b, idx) for b in ch.head["bottoms"]], 1)
            assert torch.equal(fetch(net, ch.tops[0], idx), want), ch.head["name"]
            continue
        if typ in ("Split", "Input", "YoloDetectionOutput", "Yolov3DetectionOutput"):
            continue
        ins = {b: fetch(net, b, idx) for b in dict.fromkeys(ch.bottoms)}
        if clip_net:
            want, bound = restate(ch, ins)
            for t in ch.tops:
                ex = ((fetch(net, t, idx) - want).abs() / bound.clamp(min=1e-300)).max().item()
                if ex > 1.0:
                    failures.append(f"{ch.head['name']} -> {t}: bound used {ex:.3g}")
        else:
            algo = net.LayerConvAlgo(ch.head["name"]) if typ in CONV_TYPES else -1
            got = {t: fetch(net, t, idx) for t in ch.tops}
            for top, used, _, kind, path in check_chain(ch, ins, got, 2, algo):
                if used > 1.0:
                    failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
    assert not failures, "\n".join(failures[:20])


def _check_head(net, m, idx):
    """The YOLO layer from the net's own bottoms: fcuda_yolo_decode on them, then yolo_ref, bit for bit."""
    from feathercnn_b200 import booster
    L = next(L.split() for L in m.lines if "DetectionOutput" in L.split()[0])
    nb = int(L[2])
    bottoms = L[4:4 + nb]
    kv = dict(t.split("=", 1) for t in L[4 + nb + 1:])
    arr = lambda k: [float(v) for v in kv[k].split(",")[1:]] if k in kv else []  # noqa: E731
    version = 3 if L[0] == "Yolov3DetectionOutput" else 2
    xs = [fetch(net, b, idx).float().contiguous() for b in bottoms]
    p = _param(version, int(kv["0"]), int(kv["1"]), [tuple(x.shape[2:]) for x in xs], arr("-23304"),
               [int(v) for v in arr("-23305")], arr("-23306"), float(kv["2"]), float(kv["3"]))
    s, c, b = (t.cpu().numpy() for t in booster.yolo_decode(xs, p))
    want, suppressed, candidates = yolo_ref(s, c, b, p.confidence_threshold, p.nms_threshold, p.nms_top_k, p.keep_top_k)
    got = fetch(net, L[4 + nb], idx).float().cpu().numpy().reshape(want.shape)
    assert _bits_equal(got, want)
    assert suppressed > 0
    return candidates // len(idx)


SETTINGS = [(True, True), (True, False), (False, True), (False, False)]


@gpu
@pytest.mark.parametrize("name, min_candidates", [("mobilenetv2_yolov3", 1025), ("mobilenet_yolov2", 200)])
def test_model_end_to_end(cuda, yolo_models, name, min_candidates):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m, param, binf, layers = yolo_models[name]
    batch = 2
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])
    idx = list(range(batch))
    dets = []
    for fusion, graph in SETTINGS:
        net = Net(fusion=fusion, cuda_graph=graph)
        net.LoadParam(param)
        net.LoadWeights(binf)
        for _ in range(3 if graph else 1):
            net.Forward(x)
        net.Synchronize()
        assert net.BlobShape("detection_out") == (batch, 1, 1024, 6) and net.BlobDims("detection_out") == 2
        _check_backbone(net, layers, idx)
        candidates = _check_head(net, m, idx)
        assert candidates >= min_candidates, candidates
        dets.append(net.Extract("detection_out"))
        del net
    assert _bits_equal(dets[0], dets[1]) and _bits_equal(dets[2], dets[3])


@gpu
@pytest.mark.parametrize("name", ["mobilenetv2_yolov3", "mobilenet_yolov2"])
def test_model_batch_independent(cuda, yolo_models, name):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m, param, binf, _ = yolo_models[name]
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
def test_yolo_tiny_runs_in_a_graph(cuda, tmp_path):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.yolo_tiny()
    param, binf = m.save(tmp_path / "yolo_tiny")
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(4)])
    outs = []
    for graph in (False, True):
        net = Net(fusion=True, cuda_graph=graph)
        net.LoadParam(param)
        net.LoadWeights(binf)
        for _ in range(3):
            net.Forward(x)
        outs.append(net.Extract("detection_out"))
    assert _bits_equal(outs[0], outs[1]) and outs[0].shape == (4, 1, 1024, 6)
    assert int((outs[0][..., 0] >= 0).sum()) > 0
