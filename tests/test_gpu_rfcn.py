"""R-FCN's PSROIPooling on the GPU.

  - PSROIPooling bit for bit against test_rfcn_host.psroi_pooling_ref (the same float32 operations, each bin summed in
    row-major order): the hand cases of the host tests (known bins, .5 ties, an empty bin, RoIs partly and wholly outside
    the map, the 0.1 width floor, the [0, 0, 0, 0] padding row, a non-square grid, the sequential sum, a NaN corner), and a
    seeded sweep of 1-3 images, up to 300 RoIs, pooled 1-9 on each side, output_dim 1-21 and RoIs tiny, huge, off the
    map or padding.
  - Batch independence: each image's items equal a batch-1 run.  A channel count that is not output_dim x pooled^2 fails
    at Reshape.
  - modelgen's rfcn_tiny (96 x 128) and rfcn_resnet50 (at 320 x 480), batch 2, with fusion and CUDA graphs on and off:
    every convolution, pooling, element-wise and Softmax chain within the float64 bounds of test_gpu_net_bounds (the
    dilated 3x3 layers by the same rule with the dilation), the RPN Reshapes bit-exact views and its channel Softmax within
    16 U, Proposal and PSROIPooling recomputed bit for bit from the net's own blobs, the outputs bit-identical with graphs
    on and off.  Proposal keeps after_nms_topN boxes per image in both models (rfcn_tiny: 6,912 anchors, pre_nms_topN
    2,000 binds too; rfcn_resnet50 at 320 x 480: 5,400 anchors).
"""
from __future__ import annotations

import dataclasses

import numpy as np
import pytest
import torch

import test_gpu_net_bounds
from test_faster_rcnn_host import proposal_ref
from test_gpu_faster_rcnn import SETTINGS, U, _all, _bits_equal, _cuda, _param, _run
from test_gpu_net_bounds import CONV_TYPES, check_chain, load_model, rebuild_chains
from test_rfcn_host import _planes, psroi_pooling_ref

gpu = pytest.mark.gpu


def _pool(x, rois, ph, pw, d, scale):
    from feathercnn_b200 import booster
    return booster.psroi_pooling(*_cuda(x, rois), ph, pw, d, scale).cpu().numpy()


# ---- the hand cases -------------------------------------------------------------------------------------------------
def _hand_cases():
    """(name, x, rois (N, R, 4), pooled_h, pooled_w, output_dim, scale)."""
    rng = np.random.default_rng(0)
    return [
        ("known_bins", _planes(4, 4, 4), [[[0, 0, 3, 3], [0.5, 0.5, 2.49, 2.5]]], 2, 2, 1, 1.0),
        ("empty_bin_partly_outside", _planes(2, 4, 4), [[[-8, 0, 3, 3]]], 1, 2, 1, 1.0),
        ("wholly_outside", _planes(4, 4, 4), [[[-10, 0, -5, 3], [9, 9, 20, 20]]], 2, 2, 1, 1.0),
        ("width_floor", _planes(1, 8, 8), [[[5, 0, 2, 3]]], 1, 1, 1, 1.0),
        ("padding_row", rng.standard_normal((1, 98, 5, 6)).astype(np.float32), [[[0, 0, 0, 0]] * 3], 7, 7, 2, 1 / 16),
        ("non_square", np.ascontiguousarray(np.broadcast_to(np.arange(12, dtype=np.float32)[None, :, None, None],
                                                            (1, 12, 4, 6))), [[[0, 0, 5, 3]]], 2, 3, 2, 1.0),
        ("sequential_sum", np.array([[[[2 ** 24, 1], [1, 1]]]], np.float32), [[[0, 0, 1, 1]]], 1, 1, 1, 1.0),
        ("nan_and_inf_corners", rng.standard_normal((1, 9, 6, 6)).astype(np.float32),
         [[[np.nan, 0, 3, 3], [0, 0, np.inf, 3], [-np.inf, -np.inf, 2, 2], [1e30, 0, 2e30, 4]]], 3, 3, 1, 0.5),
    ]


HAND = _hand_cases()


@gpu
@pytest.mark.parametrize("i", range(len(HAND)), ids=[c[0] for c in HAND])
def test_hand_cases_bit_exact(cuda, i):
    name, x, rois, ph, pw, d, scale = HAND[i]
    rois = np.array(rois, np.float32)
    got = _pool(x, rois, ph, pw, d, scale)
    assert _bits_equal(got, psroi_pooling_ref(x, rois, ph, pw, d, scale)), name
    if name == "known_bins":
        assert got[0].tolist() == [[[2.5, 104.5], [210.5, 312.5]]]
    if name == "sequential_sum":
        assert got.ravel().tolist() == [2.0 ** 22]
    if name == "padding_row":
        assert all(np.array_equal(g, x[0, :, 0, 0].reshape(2, 7, 7)) for g in got)


# ---- seeded sweep ---------------------------------------------------------------------------------------------------
SWEEP_N = 16


def _sweep_case(i):
    rng = np.random.default_rng(7000 + i)
    n = int(rng.integers(1, 4))
    r = int(rng.choice([1, int(rng.integers(2, 64)), int(rng.integers(64, 301)), 300]))
    ph, pw = int(rng.integers(1, 10)), int(rng.integers(1, 10))
    d = int(rng.choice([1, 2, 8, 21, int(rng.integers(1, 22))]))
    h, w = int(rng.integers(1, 41)), int(rng.integers(1, 41))
    scale = float(rng.choice([1.0, 0.5, 0.25, 0.125, 0.0625]))
    img_w, img_h = w / scale, h / scale
    kind = rng.integers(0, 5, (n, r))
    xy = rng.uniform([-0.2 * img_w, -0.2 * img_h], [img_w, img_h], (n, r, 2))
    wh = np.where((kind == 0)[..., None], rng.uniform(-3, 3, (n, r, 2)),                     # tiny (or inverted)
                  np.where((kind == 1)[..., None], rng.uniform(4, 20, (n, r, 2)) * [img_w, img_h],   # huge
                           rng.uniform(0.05, 0.8, (n, r, 2)) * [img_w, img_h]))
    rois = np.concatenate([xy, xy + wh], -1)
    rois[kind == 2] += [[3 * img_w, -2 * img_h, 3 * img_w, -2 * img_h]]                     # off the map
    rois[kind == 3] = 0                                                                      # Proposal's padding
    return dict(seed=7000 + i, n=n, r=r, ph=ph, pw=pw, d=d, h=h, w=w, scale=scale, rois=rois.astype(np.float32))


@gpu
@pytest.mark.parametrize("i", range(SWEEP_N))
def test_random_geometry_matches_reference(cuda, i):
    c = _sweep_case(i)
    x = np.random.default_rng(c["seed"]).standard_normal((c["n"], c["d"] * c["ph"] * c["pw"], c["h"], c["w"]))
    x = x.astype(np.float32)
    got = _pool(x, c["rois"], c["ph"], c["pw"], c["d"], c["scale"])
    want = psroi_pooling_ref(x, c["rois"], c["ph"], c["pw"], c["d"], c["scale"])
    assert _bits_equal(got, want)
    if c["r"] >= 64:
        assert np.any(want == 0) and np.any(want != 0)


def test_sweep_cases_cover_the_boundaries():
    cases = [_sweep_case(i) for i in range(SWEEP_N)]
    assert any(c["n"] > 1 for c in cases) and any(c["r"] == 300 for c in cases) and any(c["r"] == 1 for c in cases)
    assert any(c["ph"] != c["pw"] for c in cases) and {1, 21} <= {c["d"] for c in cases}
    assert any(c["ph"] == 9 or c["pw"] == 9 for c in cases) and any(c["ph"] == 1 or c["pw"] == 1 for c in cases)
    assert all(np.any(np.all(c["rois"] == 0, -1)) for c in cases if c["r"] >= 64)


# ---- batch independence and shape checks ----------------------------------------------------------------------------
@gpu
def test_batch_independent(cuda):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((3, 21 * 49, 19, 23)).astype(np.float32)
    xy = rng.uniform(0, 300, (3, 100, 2))
    rois = np.concatenate([xy, xy + rng.uniform(8, 200, (3, 100, 2))], -1).astype(np.float32)
    rois[:, 90:] = 0
    pooled = _pool(x, rois, 7, 7, 21, 1 / 16)
    for i in range(3):
        assert _bits_equal(_pool(x[i:i + 1], rois[i:i + 1], 7, 7, 21, 1 / 16), pooled[i * 100:(i + 1) * 100])


@gpu
def test_channel_count_checked_at_reshape(cuda, tmp_path):
    """10 channels are not output_dim 1 x 3 x 3: PSROIPooling's Reshape fails (FEATHER_ERR_TOPOLOGY), which Net reports
    as -100 like every shape failure."""
    from feathercnn_b200.net import FeatherError, Net
    net = Net()
    net.LoadParamFromText("7767517\n3 3\nInput f 0 1 f 0=4 1=4 2=10\nInput r 0 1 r 0=4 1=1 2=5\n"
                          "PSROIPooling p 2 1 f r out 0=3 1=3 2=0.25 3=1\n")
    empty = tmp_path / "empty.bin"
    empty.write_bytes(b"")
    net.LoadWeights(str(empty))
    net.FeedInputBatch(np.zeros((1, 5, 1, 4), np.float32), "r")
    with pytest.raises(FeatherError) as e:
        net.Forward(np.zeros((1, 10, 4, 4), np.float32))
    assert e.value.code == -100


# ---- models end to end ----------------------------------------------------------------------------------------------
MODELS = {"rfcn_tiny": {}, "rfcn_resnet50": dict(height=320, width=480)}


@pytest.fixture(scope="module")
def rfcn_models(tmp_path_factory):
    from feathercnn_b200.tools import modelgen
    d = tmp_path_factory.mktemp("rfcn")
    out = {}
    for name, kw in MODELS.items():
        m = modelgen.ZOO[name](**kw)
        param, binf = m.save(d / name)
        out[name] = (m, param, binf, load_model(param, binf))
    return out


_plain_geometry = test_gpu_net_bounds.conv_geometry


def _geometry_with_dilation(L, x):
    """test_gpu_net_bounds.conv_geometry for a convolution that may be dilated (2=, the same on both axes)."""
    d = L["params"].get(2, 1)
    assert L["params"].get(12, d) == d, L["name"]
    plain = dict(L, params={k: v for k, v in L["params"].items() if k not in (2, 12)})
    return dataclasses.replace(_plain_geometry(plain, x), dil=d)


def _check_layers(net, layers):
    """test_gpu_faster_rcnn._check_layers for R-FCN: every chain within its float64 bound (dilated convolutions
    included); the RPN Reshapes bit-exact views, its Softmax within 16 U; Proposal and PSROIPooling bit for bit from the
    net's own blobs.  Returns Proposal's per-image stats and the number of PSROIPooling layers checked."""
    from feathercnn_b200 import booster
    chains, _ = rebuild_chains(layers, net.LayerFusedAway, set(net.BlobNames()))
    failures, stats, psroi = [], None, 0
    for ch in chains:
        typ, pd = ch.head["type"], ch.head["params"]
        if typ in ("Input", "Split", "Dropout"):
            continue
        if typ == "Reshape":
            assert torch.equal(_all(net, ch.tops[0]).flatten(), _all(net, ch.head["bottoms"][0]).flatten())
            continue
        if typ == "Softmax" and 0 in pd:
            x = _all(net, ch.head["bottoms"][0])
            assert (_all(net, ch.tops[0]) - torch.softmax(x, 1)).abs().max().item() <= 16 * U, ch.head["name"]
            continue
        if typ == "Proposal":
            p = _param(feat_stride=pd[0], base_size=pd[1], pre_nms_topN=pd[2], after_nms_topN=pd[3], nms_thresh=pd[4],
                       min_size=pd[5])
            s, b, inf = (_all(net, t).float().contiguous() for t in ch.head["bottoms"])
            boxes = booster.proposal_decode(s, b, inf, p).cpu().numpy()
            want, _, stats = proposal_ref(boxes, s.cpu().numpy(), inf.cpu().numpy(), p.pre_nms_topN, p.after_nms_topN,
                                          p.nms_thresh, p.min_size)
            assert _bits_equal(_all(net, ch.tops[0]).float().cpu().numpy().reshape(want.shape), want)
            continue
        if typ == "PSROIPooling":
            x, rois = (_all(net, t).float().cpu().numpy() for t in ch.head["bottoms"])
            want = psroi_pooling_ref(x, rois, pd[1], pd[0], pd[3], pd[2])
            assert _bits_equal(_all(net, ch.tops[0]).float().cpu().numpy(), want), ch.head["name"]
            psroi += 1
            continue
        algo = net.LayerConvAlgo(ch.head["name"]) if typ in CONV_TYPES else -1
        ins = {b: _all(net, b) for b in dict.fromkeys(ch.bottoms)}
        got = {t: _all(net, t) for t in ch.tops}
        for top, used, _, kind, path in check_chain(ch, ins, got, 2, algo):
            if used > 1.0:
                failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
    assert not failures, "\n".join(failures[:20])
    assert stats is not None
    return stats, psroi


@gpu
@pytest.mark.parametrize("name", list(MODELS))
def test_model_end_to_end(cuda, rfcn_models, name, monkeypatch):
    from feathercnn_b200.tools import modelgen
    monkeypatch.setattr(test_gpu_net_bounds, "conv_geometry", _geometry_with_dilation)
    m, param, binf, layers = rfcn_models[name]
    assert any(L["type"] == "Convolution" and L["params"].get(2, 1) == 2 for L in layers)
    batch = 2
    c, h, w = m.shape["data"]
    x = np.stack([modelgen.synthetic_input((c, h, w), i) for i in range(batch)])
    info = np.array([[[[h, w, 1.0]]], [[[h - 16, w - 40, 1.0]]]], np.float32)
    post = m.shape["rois"][0]
    outs = []
    for fusion, graph in SETTINGS:
        net = _run(m, param, binf, x, info, fusion, graph)
        assert net.BlobShape("rois") == (batch, post, 1, 4)
        for blob in ("psroipooled_cls_rois", "psroipooled_loc_rois", "cls_prob", "bbox_pred"):
            assert net.BlobShape(blob) == (batch * post,) + m.shape[blob], blob
        stats, psroi = _check_layers(net, layers)
        assert psroi == 2
        for cand, kept, sup in stats:
            assert kept == post and sup > 0, stats          # after_nms_topN binds
        if name == "rfcn_tiny":
            assert all(cand > 2000 for cand, _, _ in stats)  # pre_nms_topN binds
        outs.append([net.Extract(b) for b in ("rois", "cls_prob", "bbox_pred")])
        del net
    for a, b in ((0, 1), (2, 3)):
        assert all(_bits_equal(u, v) for u, v in zip(outs[a], outs[b]))
