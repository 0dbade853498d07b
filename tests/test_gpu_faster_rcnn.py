"""Faster R-CNN's Proposal and ROIPooling on the GPU.

  - Decode against float64 (test_faster_rcnn_host.proposal_decode_ref), per element.  U = 2^-23; each fp32 operation
    rounds by at most U relative and CUDA's expf errs by at most 2 ulp (2 U relative).  The anchor terms ax1 + x * stride
    and ax + aw * 0.5 are exact (integers and halves far below 2^24), so for x1 = pcx - pw * 0.5:
      aw * dx carries U |aw dx|; pcx = c + aw dx adds U |pcx|; pw = aw * expf(dw) carries 3 U pw, of which half reaches
      x1; x1 itself adds U |x1|.  |err x1| <= U (|aw dx| + |pcx| + 1.5 pw + |x1|), y alike.  Clipping to [0, side - 1]
      is 1-Lipschitz and side - 1 is exact, so the clipped box keeps the bound.  The test doubles it.
  - Selection, NMS and rows decision by decision, bit for bit, against test_faster_rcnn_host.proposal_ref fed the
    kernel's own boxes (fcuda_proposal_decode): no candidates; fewer than after_nms_topN; exactly pre_nms_topN and one
    more; 1024 / 1025 candidates at pre_nms_topN 1024 and 8192 candidates at 6000 and at 8192 (past the old 1024 cap);
    exact score ties; identical boxes (one survivor); the stop at after_nms_topN; boxes wholly outside the image; a
    different im_info per image of one batch.  Every case with candidates asserts that NMS suppressed something.
  - ROIPooling bit for bit against roi_pooling_ref: RoIs partly and wholly outside the map, .5 rounding ties, empty bins,
    7 x 7 and non-square grids, scales 1/16 and 1/8, R = 1, the zero padding rows.
  - A seeded sweep of random geometries across both layers; batch independence of both.
  - modelgen's faster_rcnn_tiny (96 x 128) and faster_rcnn_vgg16 (at 320 x 480) end to end with fusion and CUDA graphs
    on and off: the backbone and the fc layers per layer within the float64 bounds of test_gpu_net_bounds, the RPN
    Reshapes bit-exact views, its channel Softmax within 16 U, Proposal and ROIPooling recomputed bit for bit from the
    net's own blobs, the outputs bit-identical with graphs on and off.  The tiny model has 6,912 candidates per image
    (pre_nms_topN 2,000 binds, after_nms_topN 64 binds); VGG-16 at 320 x 480 has 5,400 (after_nms_topN 300 binds).
    faster_rcnn_tiny replays inside a CUDA graph.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_faster_rcnn_host import A, proposal_decode_ref, proposal_ref, roi_pooling_ref
from test_gpu_net_bounds import CONV_TYPES, check_chain, load_model, rebuild_chains

gpu = pytest.mark.gpu
U = 2.0 ** -23


def _bits_equal(a, b) -> bool:
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _cuda(*xs):
    return [torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda() for x in xs]


def _param(**kw):
    from feathercnn_b200 import booster
    return booster.proposal_param(**kw)


# ---- decode ---------------------------------------------------------------------------------------------------------
DECODE_CASES = [dict(n=1, h=38, w=50, stride=16, base=16, delta=0.3, info=[(600, 800, 1.0)]),
                dict(n=3, h=7, w=11, stride=16, base=16, delta=2.0, info=[(100, 180, 1.0), (60, 30, 0.5), (112, 176, 2.0)]),
                dict(n=2, h=24, w=32, stride=4, base=2, delta=1.0, info=[(96, 128, 1.0), (90, 100, 1.5)]),
                dict(n=1, h=1, w=1, stride=1, base=1, delta=5.0, info=[(5, 5, 1.0)])]


@gpu
@pytest.mark.parametrize("case", DECODE_CASES, ids=[f"{c['h']}x{c['w']}-n{c['n']}-s{c['stride']}" for c in DECODE_CASES])
def test_decode_within_bound(cuda, case):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(case["h"] * 1000 + case["w"])
    n, h, w = case["n"], case["h"], case["w"]
    score = rng.random((n, 2 * A, h, w), np.float32)
    bbox = (rng.standard_normal((n, 4 * A, h, w)) * case["delta"]).astype(np.float32)
    info = np.array(case["info"], np.float32)
    p = _param(feat_stride=case["stride"], base_size=case["base"])
    got = booster.proposal_decode(*_cuda(score, bbox, info), p).cpu().numpy().astype(np.float64)
    ref, raw, awh = proposal_decode_ref(bbox, info, case["stride"], case["base"])
    d = bbox.astype(np.float64).reshape(n, A, 4, h * w).transpose(0, 1, 3, 2).reshape(n, -1, 4)
    aw, ah = awh[None, :, 0], awh[None, :, 1]
    pcx, pcy = (raw[..., 0] + raw[..., 2]) / 2, (raw[..., 1] + raw[..., 3]) / 2
    pw, ph = raw[..., 2] - raw[..., 0], raw[..., 3] - raw[..., 1]
    bx = np.abs(aw * d[..., 0]) + np.abs(pcx) + 1.5 * pw
    by = np.abs(ah * d[..., 1]) + np.abs(pcy) + 1.5 * ph
    bound = 2 * U * (np.stack([bx, by, bx, by], -1) + np.abs(raw)) + 2.0 ** -140
    used = float((np.abs(got - ref) / bound).max())
    assert used <= 1.0, used
    assert np.all(got >= 0) and np.all(got[..., 2] <= info[:, None, 1] - 1) and np.all(got[..., 3] <= info[:, None, 0] - 1)


# ---- selection, NMS, rows -------------------------------------------------------------------------------------------
def run_and_check(score, bbox, info, p):
    """Proposal on the GPU against proposal_ref over the GPU's own boxes, bit for bit; returns the per-image stats."""
    from feathercnn_b200 import booster
    s, b, i = _cuda(score, bbox, info)
    boxes = booster.proposal_decode(s, b, i, p).cpu().numpy()
    rois, sc = (t.cpu().numpy() for t in booster.proposal(s, b, i, p))
    want_r, want_s, stats = proposal_ref(boxes, score, info, p.pre_nms_topN, p.after_nms_topN, p.nms_thresh, p.min_size)
    assert _bits_equal(rois, want_r) and _bits_equal(sc, want_s)
    return stats


def _inputs(rng, n, h, w, delta=0.1, candidates=None):
    """Random scores and deltas; with `candidates`, exactly that many non-NaN foreground scores per image."""
    score = rng.random((n, 2 * A, h, w), np.float32)
    bbox = (rng.standard_normal((n, 4 * A, h, w)) * delta).astype(np.float32)
    if candidates is not None:
        fg = score[:, A:].reshape(n, -1)
        for i in range(n):
            fg[i, rng.permutation(fg.shape[1])[candidates:]] = np.nan
        score[:, A:] = fg.reshape(n, A, h, w)
    return score, bbox


def _sel_case(name, rng):
    info1 = np.array([[600, 800, 1.0]], np.float32)
    if name == "no_candidates":
        s, b = _inputs(rng, 1, 8, 8)
        return s, b, info1, _param(min_size=100000), 0
    if name == "fewer_than_post":
        s, b = _inputs(rng, 1, 2, 2)
        return s, b, info1, _param(), 1
    if name in ("pre_exact", "pre_plus_one"):
        s, b = _inputs(rng, 1, 12, 12, candidates=500 + (name == "pre_plus_one"))
        return s, b, info1, _param(pre_nms_topN=500, after_nms_topN=8192, min_size=0), 500
    if name in ("1024", "1025"):
        s, b = _inputs(rng, 1, 12, 12, candidates=int(name))
        return s, b, info1, _param(pre_nms_topN=1024, after_nms_topN=2000, min_size=0), 1024
    if name in ("8192_at_6000", "8192_at_8192"):
        s, b = _inputs(rng, 1, 32, 32, candidates=8192)
        pre = int(name.split("_")[-1])
        return s, b, np.array([[2000, 2000, 1.0]], np.float32), _param(pre_nms_topN=pre, after_nms_topN=8192,
                                                                       min_size=0), pre
    if name == "ties":
        s, b = _inputs(rng, 2, 9, 9)
        s[:, A:] = np.float32(0.25) * rng.integers(1, 4, s[:, A:].shape)
        s[0, A, 0, :3] = [0.0, -0.0, 0.0]
        return s, b, np.repeat(info1, 2, 0), _param(min_size=0), 1
    if name == "identical_boxes":
        s, b = _inputs(rng, 1, 6, 6)
        b.reshape(1, A, 4, 36)[:, :, 2:] = 20.0  # every box covers the whole image
        return s, b, np.array([[100, 120, 1.0]], np.float32), _param(), 1
    if name == "stop_at_post":
        s, b = _inputs(rng, 1, 20, 20)
        return s, b, info1, _param(after_nms_topN=7), 7
    if name == "outside_image":
        s, b = _inputs(rng, 1, 10, 10)
        b.reshape(1, A, 4, 100)[:, :4, 0] = 60.0  # anchors 0-3 pushed right of the image
        return s, b, np.array([[160, 160, 1.0]], np.float32), _param(min_size=0), 1
    if name == "im_info_per_image":
        s, b = _inputs(rng, 3, 14, 18, delta=0.3)
        info = np.array([[224, 288, 1.0], [150, 100, 0.5], [200, 240, 2.0]], np.float32)
        return s, b, info, _param(pre_nms_topN=1500, after_nms_topN=200), 1
    raise KeyError(name)


SEL_CASES = ["no_candidates", "fewer_than_post", "pre_exact", "pre_plus_one", "1024", "1025", "8192_at_6000",
             "8192_at_8192", "ties", "identical_boxes", "stop_at_post", "outside_image", "im_info_per_image"]


@gpu
@pytest.mark.parametrize("name", SEL_CASES)
def test_selection_nms_decisions(cuda, name):
    rng = np.random.default_rng(SEL_CASES.index(name))
    score, bbox, info, p, min_kept = _sel_case(name, rng)
    stats = run_and_check(score, bbox, info, p)
    for cand, kept, sup in stats:
        if name == "no_candidates":
            assert cand == 0 and kept == 0
            continue
        assert kept >= 1 and sup > 0, (name, stats)
        if name == "fewer_than_post":
            assert kept < p.after_nms_topN
        if name == "identical_boxes":
            assert kept == 1
        if name == "stop_at_post":
            assert kept == p.after_nms_topN
        if name in ("pre_exact", "pre_plus_one", "1024", "1025"):
            assert cand == int({"pre_exact": 500, "pre_plus_one": 501}.get(name, name))
        if name.startswith("8192"):
            assert cand == 8192


# ---- ROIPooling -----------------------------------------------------------------------------------------------------
def _rois_cases():
    """(name, x shape, rois (N, R, 4), pooled_h, pooled_w, scale)."""
    cases = []
    edge = [[-40, -40, 100, 60], [150, 150, 400, 300], [-300, -300, -100, -50], [1000, 0, 2000, 50],  # partly / wholly out
            [8, 8, 24, 24], [-8, -8, 7.9, 40], [24, 40, 56, 72.0], [0, 0, 0, 0],                        # .5 ties, padding
            [3, 5, 260, 200], [16, 16, 17, 17]]
    cases.append(("edges_7x7_s16", (2, 5, 13, 17), np.array([edge, edge[::-1]], np.float32), 7, 7, 1 / 16))
    cases.append(("edges_3x5_s8", (1, 3, 26, 34), np.array([edge], np.float32), 3, 5, 1 / 8))
    cases.append(("r1", (1, 8, 9, 9), np.array([[[10, 20, 90, 100]]], np.float32), 7, 7, 1 / 16))
    cases.append(("empty_bins", (1, 2, 4, 4), np.array([[[0, 0, 160, 160], [-100, 0, -20, 200]]], np.float32), 7, 7,
                  1 / 16))
    return cases


ROI_CASES = _rois_cases()


@gpu
@pytest.mark.parametrize("i", range(len(ROI_CASES)), ids=[c[0] for c in ROI_CASES])
def test_roi_pooling_bit_exact(cuda, i):
    from feathercnn_b200 import booster
    name, shape, rois, ph, pw, scale = ROI_CASES[i]
    x = np.random.default_rng(i).standard_normal(shape).astype(np.float32)
    got = booster.roi_pooling(*_cuda(x, rois), ph, pw, scale).cpu().numpy()
    want = roi_pooling_ref(x, rois, ph, pw, scale)
    assert _bits_equal(got, want)
    if name.startswith("edges"):
        assert np.any(want == 0) and np.any(want != 0)


# ---- seeded sweep ---------------------------------------------------------------------------------------------------
SWEEP_N = 24


def _sweep_case(i):
    rng = np.random.default_rng(9000 + i)
    n = int(rng.integers(1, 4))
    h, w = int(rng.integers(1, 41)), int(rng.integers(1, 41))
    stride = int(rng.choice([4, 8, 16]))
    base = int(rng.choice([2, 8, 16]))
    pre = int(rng.choice([1, 31, 32, 33, 1023, 1024, 1025, int(rng.integers(1, 8193))]))
    post = int(rng.integers(1, pre + 1)) if rng.random() < 0.7 else int(rng.integers(1, 8193))
    thresh = float(rng.choice([0.3, 0.5, 0.7, 0.9]))
    min_size = int(rng.choice([0, 4, 16]))
    info = np.stack([rng.integers(max(h * stride // 2, 1), h * stride + 64, n), rng.integers(max(w * stride // 2, 1),
                                                                                               w * stride + 64, n),
                     rng.choice([0.5, 1.0, 1.6], n)], 1).astype(np.float32)
    return dict(seed=9000 + i, n=n, h=h, w=w, p=dict(feat_stride=stride, base_size=base, pre_nms_topN=pre,
                                                     after_nms_topN=post, nms_thresh=thresh, min_size=min_size),
                info=info, delta=float(rng.choice([0.05, 0.3, 1.0])))


@gpu
@pytest.mark.parametrize("i", range(SWEEP_N))
def test_random_geometry_matches_reference(cuda, i):
    from feathercnn_b200 import booster
    c = _sweep_case(i)
    rng = np.random.default_rng(c["seed"])
    score, bbox = _inputs(rng, c["n"], c["h"], c["w"], c["delta"])
    stats = run_and_check(score, bbox, c["info"], _param(**c["p"]))
    assert all(k <= c["p"]["after_nms_topN"] for _, k, _ in stats)
    # ROIPooling over the proposals of the same images, on a random map at 1 / stride
    s, b, inf = _cuda(score, bbox, c["info"])
    rois = booster.proposal(s, b, inf, _param(**c["p"]))[0][:, :64].contiguous()
    x = rng.standard_normal((c["n"], 3, c["h"], c["w"])).astype(np.float32)
    ph, pw = int(rng.integers(1, 8)), int(rng.integers(1, 8))
    scale = 1.0 / c["p"]["feat_stride"]
    got = booster.roi_pooling(_cuda(x)[0], rois, ph, pw, scale).cpu().numpy()
    assert _bits_equal(got, roi_pooling_ref(x, rois.cpu().numpy(), ph, pw, scale))


def test_sweep_cases_cover_the_boundaries():
    cases = [_sweep_case(i) for i in range(SWEEP_N)]
    pres = {c["p"]["pre_nms_topN"] for c in cases}
    assert pres & {31, 32, 33} and pres & {1023, 1024, 1025} and any(p > 1025 for p in pres)
    assert any(c["n"] > 1 for c in cases) and any(c["h"] * c["w"] * 9 > 1024 for c in cases)


# ---- batch independence ---------------------------------------------------------------------------------------------
@gpu
def test_layers_batch_independent(cuda):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(5)
    score, bbox = _inputs(rng, 4, 19, 23, 0.3)
    info = np.array([[300, 360, 1.0], [200, 300, 0.8], [304, 368, 1.0], [150, 150, 1.2]], np.float32)
    p = _param(pre_nms_topN=3000, after_nms_topN=100)
    s, b, inf = _cuda(score, bbox, info)
    rois, sc = booster.proposal(s, b, inf, p)
    x = _cuda(rng.standard_normal((4, 6, 19, 23)))[0]
    pooled = booster.roi_pooling(x, rois, 7, 7, 1 / 16).cpu().numpy()
    for i in range(4):
        r1, s1 = booster.proposal(s[i:i + 1], b[i:i + 1], inf[i:i + 1], p)
        assert _bits_equal(r1.cpu().numpy()[0], rois.cpu().numpy()[i]) and _bits_equal(s1.cpu().numpy()[0], sc.cpu().numpy()[i])
        alone = booster.roi_pooling(x[i:i + 1], r1, 7, 7, 1 / 16).cpu().numpy()
        assert _bits_equal(alone, pooled[i * 100:(i + 1) * 100])


@gpu
def test_channel_counts_checked_at_reshape(cuda, tmp_path):
    """A score blob of 16 channels is not 2 x 9: Proposal's Reshape fails (FEATHER_ERR_TOPOLOGY), which Net reports as
    -100 like every shape failure."""
    from feathercnn_b200.net import FeatherError, Net
    net = Net()
    net.LoadParamFromText("7767517\n4 4\nInput s 0 1 s 0=4 1=4 2=16\nInput b 0 1 b 0=4 1=4 2=36\nInput i 0 1 i 0=3\n"
                          "Proposal p 3 1 s b i rois\n")
    empty = tmp_path / "empty.bin"
    empty.write_bytes(b"")
    net.LoadWeights(str(empty))
    net.FeedInputBatch(np.zeros((1, 36, 4, 4), np.float32), "b")
    net.FeedInputBatch(np.array([[[[64, 64, 1]]]], np.float32), "i")
    with pytest.raises(FeatherError) as e:
        net.Forward(np.zeros((1, 16, 4, 4), np.float32))
    assert e.value.code == -100


# ---- models end to end ----------------------------------------------------------------------------------------------
MODELS = {"faster_rcnn_tiny": {}, "faster_rcnn_vgg16": dict(height=320, width=480)}


@pytest.fixture(scope="module")
def rcnn_models(tmp_path_factory):
    from feathercnn_b200.tools import modelgen
    d = tmp_path_factory.mktemp("rcnn")
    out = {}
    for name, kw in MODELS.items():
        m = modelgen.ZOO[name](**kw)
        param, binf = m.save(d / name)
        out[name] = (m, param, binf, load_model(param, binf))
    return out


def _all(net, name) -> torch.Tensor:
    from test_gpu_net_bounds import fetch
    return fetch(net, name, slice(None))


def _run(m, param, binf, x, info, fusion, graph):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    for _ in range(3 if graph else 1):
        net.FeedInputBatch(info, "im_info")
        net.Forward(x)
    net.Synchronize()
    return net


def _check_layers(net, m, layers):
    """Backbone and fc chains within their float64 bounds; the RPN Reshapes bit-exact views, its Softmax within 16 U;
    Proposal and ROIPooling bit for bit from the net's own blobs.  Returns Proposal's per-image stats."""
    from feathercnn_b200 import booster
    names = set(net.BlobNames())
    chains, _ = rebuild_chains(layers, net.LayerFusedAway, names)
    failures = []
    stats = None
    for ch in chains:
        typ = ch.head["type"]
        if typ in ("Input", "Split", "Dropout"):
            continue
        if typ == "Reshape":
            assert torch.equal(_all(net, ch.tops[0]).flatten(), _all(net, ch.head["bottoms"][0]).flatten())
            continue
        if typ == "Softmax" and 0 in ch.head["params"]:
            x = _all(net, ch.head["bottoms"][0])
            assert (_all(net, ch.tops[0]) - torch.softmax(x, 1)).abs().max().item() <= 16 * U, ch.head["name"]
            continue
        if typ == "Proposal":
            pd = ch.head["params"]
            p = _param(feat_stride=pd[0], base_size=pd[1], pre_nms_topN=pd[2], after_nms_topN=pd[3], nms_thresh=pd[4],
                       min_size=pd[5])
            s, b, inf = (_all(net, t).float().contiguous() for t in ch.head["bottoms"])
            boxes = booster.proposal_decode(s, b, inf, p).cpu().numpy()
            want, _, stats = proposal_ref(boxes, s.cpu().numpy(), inf.cpu().numpy(), p.pre_nms_topN, p.after_nms_topN,
                                          p.nms_thresh, p.min_size)
            assert _bits_equal(_all(net, ch.tops[0]).float().cpu().numpy().reshape(want.shape), want)
            continue
        if typ == "ROIPooling":
            pd = ch.head["params"]
            x, rois = (_all(net, t).float().cpu().numpy() for t in ch.head["bottoms"])
            want = roi_pooling_ref(x, rois, pd[1], pd[0], pd[2])
            assert _bits_equal(_all(net, ch.tops[0]).float().cpu().numpy(), want)
            continue
        algo = net.LayerConvAlgo(ch.head["name"]) if typ in CONV_TYPES else -1
        ins = {b: _all(net, b) for b in dict.fromkeys(ch.bottoms)}
        got = {t: _all(net, t) for t in ch.tops}
        for top, used, _, kind, path in check_chain(ch, ins, got, 2, algo):
            if used > 1.0:
                failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
    assert not failures, "\n".join(failures[:20])
    assert stats is not None
    return stats


SETTINGS = [(True, True), (True, False), (False, True), (False, False)]


@gpu
@pytest.mark.parametrize("name", list(MODELS))
def test_model_end_to_end(cuda, rcnn_models, name):
    from feathercnn_b200.tools import modelgen
    m, param, binf, layers = rcnn_models[name]
    batch = 2
    c, h, w = m.shape["data"]
    x = np.stack([modelgen.synthetic_input((c, h, w), i) for i in range(batch)])
    info = np.array([[[[h, w, 1.0]]], [[[h - 16, w - 40, 1.0]]]], np.float32)
    post = m.shape["rois"][0]
    outs = []
    for fusion, graph in SETTINGS:
        net = _run(m, param, binf, x, info, fusion, graph)
        assert net.BlobShape("rois") == (batch, post, 1, 4)
        assert net.BlobShape("pool5")[0] == batch * post and net.BlobShape("cls_prob")[0] == batch * post
        stats = _check_layers(net, m, layers)
        for cand, kept, sup in stats:
            assert kept == post and sup > 0, stats          # after_nms_topN binds
            assert cand > 1024, stats
        if name == "faster_rcnn_tiny":
            assert all(cand > 2000 for cand, _, _ in stats)  # pre_nms_topN binds
        outs.append([net.Extract(b) for b in ("rois", "cls_prob", "bbox_pred")])
        del net
    for a, b in ((0, 1), (2, 3)):
        assert all(_bits_equal(u, v) for u, v in zip(outs[a], outs[b]))


@gpu
def test_model_batch_independent(cuda, rcnn_models):
    """Proposal's rows and ROIPooling's items of each image do not depend on the other images of the batch (the fc layers
    after them may pick another split of K for another number of rows, so they are checked per layer instead)."""
    from feathercnn_b200.tools import modelgen
    m, param, binf, _ = rcnn_models["faster_rcnn_tiny"]
    c, h, w = m.shape["data"]
    x = np.stack([modelgen.synthetic_input((c, h, w), i) for i in range(3)])
    info = np.array([[[[h, w, 1.0]]], [[[h - 8, w, 0.8]]], [[[h, w - 24, 1.25]]]], np.float32)
    net = _run(m, param, binf, x, info, True, True)
    rois, pool5 = net.Extract("rois"), net.Extract("pool5")
    post = rois.shape[1]
    for i in range(3):
        one = _run(m, param, binf, x[i:i + 1], info[i:i + 1], True, True)
        assert _bits_equal(one.Extract("rois")[0], rois[i])
        assert _bits_equal(one.Extract("pool5"), pool5[i * post:(i + 1) * post])


@gpu
def test_faster_rcnn_tiny_runs_in_a_graph(cuda, rcnn_models):
    from feathercnn_b200.tools import modelgen
    m, param, binf, _ = rcnn_models["faster_rcnn_tiny"]
    c, h, w = m.shape["data"]
    x = modelgen.synthetic_input((c, h, w), 0)[None]
    info = np.array([[[[h, w, 1.0]]]], np.float32)
    eager = _run(m, param, binf, x, info, True, False)
    graph = _run(m, param, binf, x, info, True, True)
    assert graph.launches_per_forward > 0
    for blob in ("rois", "pool5", "cls_prob", "bbox_pred"):
        assert _bits_equal(graph.Extract(blob), eager.Extract(blob)), blob
