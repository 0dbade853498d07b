"""Normalize on the GPU, and modelgen's VGG-SSD 300 end to end.

Kernels against float64 (test_normalize_host.normalize_ref), per element.  U = 2^-23, u = U / 2.  The kernel's documented
summation order (include/fcuda.h) adds nonnegative terms, and each term passes through at most m roundings on its way into
ssum:
    per pixel      m = ceil(C / 8) fmaf steps of its warp's chain + 7 additions of the warp partials;
    across_spatial m = ceil(min(n, 8192) / 256) fmaf steps of its thread + 5 shuffle levels + 7 warp partials
                       + ceil(K / 32) lane-strided additions of the chunk sums + 5 shuffle levels (n floats per set,
                       K = ceil(n / 8192) chunks).
A sum of nonnegative terms with at most m roundings per term errs by at most ((1 + u)^m - 1) ssum ~ m u ssum.  Then eps
mode 0 adds eps (one rounding, relative to ssum + eps); max() is exact; sqrt halves the relative error and rounds once;
the division rounds once: |a - a*| <= ((m + 1) / 2 + 2) u a*.  The two products fl(fl(x a) s) round twice more, so
    |y - y*| <= ((m + 1) / 2 + 4) u |y*| = ((m + 1) / 4 + 2) U |y*|
to first order.  The test allows twice that, ((m + 1) / 2 + 4) U |y*|, plus 2^-140 for results below the normal range.

Cases where the result is known in advance: an eps-dominated input on which the three eps_modes give visibly different
factors (about 10, 100 and 10), each within the bound of its own formula, and an all-zero pixel with eps > 0, which gives
exactly 0.  Bit-exact: one image of a batch against the same image alone, in place against out of place, and a launch
captured in a CUDA graph against the eager one.

VGG-SSD end to end at batch 2 with fusion and CUDA graphs each on and off, from the Net's own blobs: every convolution
chain within test_gpu_net_bounds.check_chain's bound (fc6, dilated, which check_chain does not take, with the same rule:
conv_ref with dilation 6 and eps_for(path) + K U), the poolings (pool3 ceil mode 75 -> 38, pool5 3x3 / 1 / 1) exact,
conv4_3_norm within the bound above, the head as test_gpu_ssd._check_head checks it with PriorBox compared with its
explicit steps (keys 11 / 12), enough candidates, suppression, and detections bit-identical with graphs on and off.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from test_gpu_error_bounds import FP32_SPLIT, PATH, U, Conv, conv_ref, eps_for, excess
from test_gpu_net_bounds import CONV_TYPES, check_chain, fetch, rebuild_chains
from test_gpu_ssd import _bits_equal, _check_head
from test_normalize_host import normalize_ref

gpu = pytest.mark.gpu
MODES = [(0, 1), (1, 1), (1, 0)]  # (across_spatial, across_channel)
MODE_IDS = ["pixel", "image", "plane"]


def _roundings(c, plane, across_spatial, across_channel):
    if not across_spatial:
        return math.ceil(c / 8) + 7
    n = c * plane if across_channel else plane
    k = math.ceil(n / 8192)
    return math.ceil(min(n, 8192) / 256) + 5 + 7 + math.ceil(k / 32) + 5


def _check(x, scale, y, sp, ch, eps, mode) -> float:
    """Share of the per-element bound used by y = normalize(x); x, y (N, C, ...) torch tensors."""
    n, c = x.shape[:2]
    plane = x[0, 0].numel()
    want, _ = normalize_ref(x.cpu().numpy(), scale.cpu().numpy(), sp, ch, eps, mode)
    m = _roundings(c, plane, sp, ch)
    bound = ((m + 1) / 2 + 4) * U * np.abs(want) + 2.0 ** -140
    got = y.cpu().numpy().astype(np.float64)
    assert np.isfinite(got).all()
    return float((np.abs(got - want) / bound).max())


def _data(shape, seed, offset=0):
    """Values in +-[0.25, 2] (no near-zeros: the bound is relative), optionally starting `offset` floats into a buffer."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = math.prod(shape)
    buf = torch.rand(n + offset, generator=g, device="cuda") * 1.75 + 0.25
    buf = buf * torch.where(torch.rand(n + offset, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    return buf[offset:].view(shape)


SHAPES = [(1, 512, 38, 38), (4, 512, 38, 38), (2, 1024, 19, 19), (3, 1, 13, 17), (2, 3, 20, 20), (2, 2048, 5, 7),
          (5, 64, 1, 1), (2, 512, 38, 38, 1)]  # the last: input offset by one float (unaligned, 4-byte path)
SHAPE_IDS = ["512x38-b1-wide", "512x38-b4-wide", "1024x19-narrow", "c1", "c3", "c2048-l2", "plane1", "512x38-unaligned"]


# ---- kernels against float64 ----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("sp, ch", MODES, ids=MODE_IDS)
def test_normalize_within_bound(cuda, shape, sp, ch):
    from feathercnn_b200 import booster
    shape, offset = (shape[:4], shape[4]) if len(shape) == 5 else (shape, 0)
    c = shape[1]
    x = _data(shape, 7 + c, offset)
    if offset:
        assert x.data_ptr() % 16 != 0
    worst = 0.0
    for mode in range(3):
        for shared in (False, True):
            s = torch.rand(1 if shared else c, device="cuda") * 30 + 1
            eps = (1e-4, 1e-10, 1e-12)[mode]
            y = booster.normalize(x, s, sp, ch, eps, mode)
            used = _check(x, s, y, sp, ch, eps, mode)
            assert used <= 1.0, (mode, shared, used)
            worst = max(worst, used)
    print(f"\nnormalize {shape} offset {offset} mode ({sp}, {ch}): worst bound share {worst:.3f}")


@gpu
@pytest.mark.parametrize("sp, ch", MODES, ids=MODE_IDS)
def test_eps_modes_differ_on_eps_dominated_input(cuda, sp, ch):
    """|x| in [1.75e-4, 1.4e-3] on 4 channels of 3 x 3 against eps = 1e-2: every reduction set has ssum <= 36 * 1.96e-6
    < 1e-4 = eps^2, so PyTorch's factor is 1 / eps = 100, TensorFlow's 1 / sqrt(eps) = 10, and Caffe's 1 / sqrt(eps + ssum)
    lies in (9.96, 10)."""
    from feathercnn_b200 import booster
    x = _data((2, 4, 3, 3), 3) * 7e-4
    s = torch.ones(4, device="cuda")
    ys = []
    for mode in range(3):
        y = booster.normalize(x, s, sp, ch, 1e-2, mode)
        assert _check(x, s, y, sp, ch, 1e-2, mode) <= 1.0, mode
        ys.append((y / x).cpu().numpy())
    assert np.allclose(ys[1], 100.0, rtol=1e-6) and np.allclose(ys[2], 10.0, rtol=1e-6)
    assert (ys[0] < ys[2]).all() and (ys[0] > 9.96).all()


@gpu
@pytest.mark.parametrize("sp, ch", MODES, ids=MODE_IDS)
def test_zero_input_with_positive_eps_gives_zero(cuda, sp, ch):
    from feathercnn_b200 import booster
    x = _data((2, 6, 4, 4), 5)
    x[1] = 0.0
    if not sp:
        x[0, :, 1, 2] = 0.0  # one zero pixel in an otherwise nonzero image
    s = torch.rand(6, device="cuda") + 1
    for mode in range(3):
        y = booster.normalize(x, s, sp, ch, 1e-10, mode)
        assert (y[1] == 0).all() and torch.isfinite(y).all(), mode
        if not sp:
            assert (y[0, :, 1, 2] == 0).all(), mode


# ---- bit-exact properties ------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("shape", [(4, 512, 38, 38), (3, 2048, 3, 5), (4, 3, 10, 10)], ids=["wide", "l2", "c3"])
@pytest.mark.parametrize("sp, ch", MODES, ids=MODE_IDS)
def test_batch_independent_and_in_place(cuda, shape, sp, ch):
    from feathercnn_b200 import booster
    x = _data(shape, 11)
    s = torch.rand(shape[1], device="cuda") * 20
    batched = booster.normalize(x, s, sp, ch, 1e-10, 0)
    for i in (0, shape[0] - 1):
        alone = booster.normalize(x[i:i + 1].clone(), s, sp, ch, 1e-10, 0)
        assert _bits_equal(alone[0].cpu().numpy(), batched[i].cpu().numpy()), i
    inplace = x.clone()
    booster.normalize(inplace, s, sp, ch, 1e-10, 0, out=inplace)
    assert _bits_equal(inplace.cpu().numpy(), batched.cpu().numpy())
    # the same values one float into a buffer (the 4-byte path): the same summation order, the same bits
    buf = torch.empty(x.numel() + 1, device="cuda")
    buf[1:].copy_(x.flatten())
    shifted = booster.normalize(buf[1:].view(shape), s, sp, ch, 1e-10, 0)
    assert _bits_equal(shifted.cpu().numpy(), batched.cpu().numpy())


@gpu
@pytest.mark.parametrize("sp, ch", MODES, ids=MODE_IDS)
def test_graph_replay_is_bit_identical(cuda, sp, ch):
    from feathercnn_b200 import booster
    x = _data((2, 512, 38, 38), 13)
    s = torch.rand(512, device="cuda") * 20
    eager = booster.normalize(x, s, sp, ch, 1e-10, 0)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        booster.normalize(x, s, sp, ch, 1e-10, 0)  # warm up outside the capture
    torch.cuda.current_stream().wait_stream(stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = booster.normalize(x, s, sp, ch, 1e-10, 0)
    g.replay()
    torch.cuda.synchronize()
    assert _bits_equal(out.cpu().numpy(), eager.cpu().numpy())


# ---- the layer ---------------------------------------------------------------------------------------------------------
def _raw_bin(tmp_path, *arrays):
    p = tmp_path / "w.bin"
    p.write_bytes(b"".join(np.ascontiguousarray(a, np.float32).tobytes() for a in arrays))
    return str(p)


@gpu
def test_layer_modes_through_the_net(cuda, tmp_path):
    """Three Normalize layers on one bottom (per pixel, per image with a shared scale, per plane with eps_mode 2) and a
    channel_shared layer with three scales (scale[0] is used), against the definition; the workspace comes from the
    Net's scratch pool."""
    from feathercnn_b200.net import Net
    text = ("7767517\n5 5\nInput data 0 1 data 0=10 1=6 2=4\n"
            "Normalize a 1 1 data ya 0=0 1=0 2=1.0e-10 3=4\n"
            "Normalize b 1 1 data yb 0=1 1=1 2=1.0e-05 3=1 9=1\n"
            "Normalize c 1 1 data yc 0=1 1=0 2=1.0e-06 3=4 4=0 9=2\n"
            "Normalize d 1 1 data yd 1=1 3=3\n")
    sa, sb, sc, sd = np.arange(1, 5, dtype=np.float32), np.float32([3]), np.float32([2, 4, 6, 8]), np.float32([5, 7, 9])
    x = np.random.default_rng(0).uniform(0.25, 2, (3, 4, 6, 10)).astype(np.float32)
    for graph in (False, True):
        net = Net(cuda_graph=graph)
        net.LoadParamFromText(text)
        net.LoadWeights(_raw_bin(tmp_path, sa, sb, sc, sd))
        for _ in range(2):
            net.Forward(x)
        for blob, args in (("ya", (sa, 0, 1, 1e-10, 0)), ("yb", (sb, 1, 1, 1e-5, 1)), ("yc", (sc, 1, 0, 1e-6, 2)),
                           ("yd", (sd[:1], 0, 1, 1e-4, 0))):
            got = torch.from_numpy(net.Extract(blob).reshape(x.shape))
            assert net.BlobDims(blob) == 3 and net.LayerFusedAway(blob[1]) == 0
            assert _check(torch.from_numpy(x), torch.from_numpy(args[0]), got, *args[1:]) <= 1.0, blob


@gpu
def test_scale_count_checked_at_reshape(cuda, tmp_path):
    """NormalizeLayer::Reshape rejects 3 scales for 4 channels (FEATHER_ERR_TOPOLOGY); Net::Reshape reports every layer's
    shape failure as FEATHER_ERR_WEIGHTS (-100)."""
    from feathercnn_b200.net import FeatherError, Net
    net = Net()
    net.LoadParamFromText("7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=4\nNormalize n 1 1 data out 3=3\n")
    net.LoadWeights(_raw_bin(tmp_path, np.ones(3)))
    with pytest.raises(FeatherError) as e:
        net.Forward(np.ones((1, 4, 4, 4), np.float32))
    assert e.value.code == -100


# ---- VGG-SSD end to end ----------------------------------------------------------------------------------------------
def load_model_vgg(param, binf) -> list[dict]:
    """test_gpu_net_bounds.load_model plus Normalize scales (raw fp32 in file order)."""
    from oracle import oracle as O
    layers = O.parse_param(param)
    mb = O._BinReader(binf)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))  # noqa: E731
    for L in layers:
        pd, typ = L["params"], L["type"]
        if typ in CONV_TYPES:
            kw = pd.get(1, 0)
            kh = pd.get(11, kw)
            num, size = pd.get(0, 0), pd.get(6, 0)
            L["w"] = t(mb.load(size, 0).reshape(num, size // (num * kh * kw), kh, kw))
            L["b"] = t(mb.load(num, 1)) if pd.get(5, 0) else None
        elif typ == "Normalize":
            L["scale"] = t(mb.load(pd.get(3, 0), 1))
        else:
            assert typ in ("Input", "ReLU", "Pooling", "Permute", "Flatten", "Concat", "Reshape", "Softmax", "PriorBox",
                           "DetectionOutput"), typ
    assert mb.off == len(mb.buf)
    return layers


@pytest.fixture(scope="module")
def vgg_ssd_model(tmp_path_factory):
    from feathercnn_b200.tools import modelgen
    m = modelgen.vgg_ssd(conf_threshold=0.02, conf_gain=3.0)
    param, binf = m.save(tmp_path_factory.mktemp("vgg_ssd") / "vgg_ssd")
    return m, param, binf, load_model_vgg(param, binf)


def _check_dilated_chain(ch, ins, got, algo):
    """check_chain's convolution rule for a dilated convolution (+ ReLU): conv_ref with the dilation, eps_for(path)
    + K U on S, plus U |ref|."""
    pd, x = ch.head["params"], ins[ch.head["bottoms"][0]]
    k, pad, dil = pd.get(1, 0), pd.get(4, 0), pd.get(2, 1)
    c = Conv(ch.head["name"], pd.get(0, 0), x.shape[1], x.shape[2], x.shape[3], k, pad=pad, dil=dil,
             bias=ch.head["b"] is not None, batch=x.shape[0])
    w, b = ch.head["w"].to(x.device), ch.head["b"].to(x.device)
    ref, s = conv_ref(c, x, w, b, None), conv_ref(c, x, w, b, None, absolute=True)
    for L in ch.ops:
        assert L["type"] == "ReLU", L["type"]
        ref = ref.clamp_min(0)
    used, _ = excess(got[ch.tops[0]], ref, s, eps_for(PATH[algo], FP32_SPLIT) + c.K * U)
    return used


def _check_priorboxes(net, m):
    """Every PriorBox blob bit-equal to fcuda_priorbox_forward with the layer's explicit steps (keys 11 / 12)."""
    from feathercnn_b200 import booster
    n = 0
    for L in (L.split() for L in m.lines if L.startswith("PriorBox ")):
        kv = dict(t.split("=", 1) for t in L[7:])
        arr = lambda k: [float(v) for v in kv[k].split(",")[1:]] if k in kv else []  # noqa: E731
        p = booster.priorbox_param(arr("-23300"), arr("-23301"), arr("-23302"), flip=int(kv["7"]), clip=int(kv["8"]),
                                   step=(float(kv["11"]), float(kv["12"])), offset=float(kv["13"]))
        _, _, fh, fw = net.BlobShape(L[4])
        _, _, ih, iw = net.BlobShape("data")
        want = booster.priorbox(p, fw, fh, iw, ih).cpu().numpy()
        got = fetch(net, L[6], [0]).float().cpu().numpy().reshape(want.shape)
        assert _bits_equal(got, want), L[1]
        n += 1
    return n


class _HeadWithoutPriorBoxes:
    """modelgen's lines without the PriorBox layers, for _check_head (which builds its PriorBox reference without steps)."""

    def __init__(self, m):
        self.lines = [L for L in m.lines if not L.startswith("PriorBox ")]


SETTINGS = [(True, True), (True, False), (False, True), (False, False)]


@gpu
def test_vgg_ssd_end_to_end(cuda, vgg_ssd_model):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m, param, binf, layers = vgg_ssd_model
    batch = 2
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])
    idx = list(range(batch))
    norm = next(L for L in layers if L["type"] == "Normalize")
    dets = []
    for fusion, graph in SETTINGS:
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
        assert net.BlobShape("mbox_priorbox") == (1, 1, 2, 4 * 8732)
        chains, _ = rebuild_chains(layers, net.LayerFusedAway, names)
        failures, checked = [], 0
        for ch in chains:
            if ch.head["type"] not in CONV_TYPES + ("ReLU", "Pooling"):
                continue
            algo = net.LayerConvAlgo(ch.head["name"]) if ch.head["type"] in CONV_TYPES else -1
            ins = {b: fetch(net, b, idx) for b in dict.fromkeys(ch.bottoms)}
            got = {t: fetch(net, t, idx) for t in ch.tops}
            if ch.head["type"] in CONV_TYPES and ch.head["params"].get(2, 1) > 1:
                results = [(ch.tops[0], _check_dilated_chain(ch, ins, got, algo), 0.0, "dilated", PATH[algo])]
            else:
                results = check_chain(ch, ins, got, FP32_SPLIT, algo)
            for top, used, rel, kind, path in results:
                checked += 1
                if used > 1.0:
                    failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
        assert not failures, "\n".join(failures[:20])
        assert checked >= 35, checked
        assert net.LayerFusedAway("conv4_3_norm") == 0
        xin, yout = fetch(net, norm["bottoms"][0], idx), fetch(net, norm["tops"][0], idx)
        assert _check(xin, norm["scale"], yout, 0, 1, 1e-10, 0) <= 1.0
        assert _check_priorboxes(net, m) == 6
        candidates = _check_head(net, _HeadWithoutPriorBoxes(m), idx)
        assert candidates >= 200, candidates
        dets.append(net.Extract("detection_out"))
        assert int((dets[-1][..., 0] >= 0).sum()) > 0
        del net
    assert _bits_equal(dets[0], dets[1]) and _bits_equal(dets[2], dets[3])
