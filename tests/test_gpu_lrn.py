"""LRN on the GPU, and modelgen's GoogLeNet and AlexNet end to end.

Kernels against two references (test_lrn_host), per element:
  * the float32 restatement lrn_restated gives s = fl(bias + fl(a * ss)) in fcuda.h's order and y64 = x * s^-beta in
    float64.  powf's maximum error is 4 ulp over its full range (CUDA C++ Programming Guide, "Mathematical Functions",
    single-precision table); an ulp of powf's result is at most 2^-23 of it, and the product with x rounds once more, so
        |y - y64| <= 4 * 2^-23 * |y64| + ulp_fp32(y64).
  * the float64 LRN lrn_ref.  With u = 2^-24 and n terms in the window (local_size, or local_size^2 within a channel),
    each square rounds once, the sum of n nonnegative terms errs by at most (n - 1) u ss, a = fl(alpha / n) once and
    fl(a * ss) once: |dt| <= (n + 2) u t.  Then s = fl(bias + t) errs by u s + |dt|, s^-beta by beta times that relative
    error plus powf's 4 * 2^-23, and the product by u:
        |y - y*| <= (beta (u + (n + 2) u |t| / s) + 4 * 2^-23 + u) |y*|   (first order; the test allows twice that).
Cases: both regions; local_size 1, 3, 5, 7 and 9 (9: the generic kernel across channels); C below the window, C = 1 and
C = 1024; planes 1x1, 2x3, 7x7, 56x56 (16-byte path) and 57x61 (4-byte path; within a channel it crosses the 32 x 16
tile seams in both directions); the zoo's alpha 1e-4 and alpha near 1, where the factor varies widely.  Bit-exact: the
same values one float into a buffer (the 4-byte path) against the aligned 16-byte path, each image of a batch of 5 alone,
and a launch replayed from a CUDA graph against the eager one.  The -100 / -200 returns on real device buffers.

GoogLeNet and AlexNet end to end at batch 2, with lrn_alpha 1e-4 and 0.9, fusion and CUDA graphs each on and off, from the
Net's own blobs: every convolution, pooling, ReLU, InnerProduct and Softmax chain within test_gpu_net_bounds.check_chain's
bound, every LRN within both bounds above against its actual input, every Concat bit-equal to its bottoms, and the
Softmax output bit-identical with graphs on and off at the same fusion setting.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import pytest
import torch

from test_gpu_error_bounds import FP32_SPLIT
from test_gpu_net_bounds import CONV_TYPES, check_chain, fetch, load_model, rebuild_chains
from test_gpu_ssd import _bits_equal
from test_lrn_host import lrn_ref, lrn_restated

gpu = pytest.mark.gpu
POWF_ULP = 4          # CUDA C++ Programming Guide: powf(x, y), 4 ulp (full range)
U23 = 2.0 ** -23
u = 2.0 ** -24


def check_lrn(x, y, region, size, alpha, beta, bias) -> tuple[float, float]:
    """Shares of the two bounds used by y = lrn(x): (restated, float64).  x, y (N, C, H, W) tensors."""
    x32 = x.float().cpu().numpy()
    got = y.double().cpu().numpy()
    assert np.isfinite(got).all()
    _, y64 = lrn_restated(x32, region, size, alpha, beta, bias)
    bound = POWF_ULP * U23 * np.abs(y64) + np.spacing(np.abs(y64).astype(np.float32)).astype(np.float64) + 2.0 ** -140
    used_restated = float((np.abs(got - y64) / bound).max())
    want, t, s = lrn_ref(x32, region, size, alpha, beta, bias)
    n = size if region == 0 else size * size
    be = float(np.float32(beta))
    rel = be * (u + (n + 2) * u * np.abs(t) / s) + POWF_ULP * U23 + u
    used_ref = float((np.abs(got - want) / (2 * rel * np.abs(want) + 2.0 ** -140)).max())
    return used_restated, used_ref


def _data(shape, seed, offset=0):
    """Values in +-[0.25, 2] (no near-zeros: the bounds are relative), optionally `offset` floats into a buffer."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = math.prod(shape)
    buf = torch.rand(n + offset, generator=g, device="cuda") * 1.75 + 0.25
    buf = buf * torch.where(torch.rand(n + offset, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    return buf[offset:].view(shape)


PARAMS = [(1e-4, 0.75, 1.0), (2.0, 0.75, 1.0), (0.9, 0.5, 2.0)]  # (alpha, beta, bias): the zoo's, then strong
ACROSS_SHAPES = [(2, 64, 56, 56), (3, 3, 7, 7), (2, 1, 2, 3), (1, 1024, 7, 7), (2, 16, 57, 61), (5, 12, 1, 1)]
ACROSS_IDS = ["64x56-wide", "c3", "c1", "c1024", "57x61-narrow", "plane1"]
WITHIN_SHAPES = [(2, 3, 1, 1), (2, 4, 2, 3), (3, 2, 7, 7), (2, 3, 56, 56), (2, 2, 57, 61)]
WITHIN_IDS = ["1x1", "2x3", "7x7", "56x56", "57x61"]


def _run_cases(shape, region, size, offset=0):
    from feathercnn_b200 import booster
    x = _data(shape, 7 + size + shape[1], offset)
    if offset:
        assert x.data_ptr() % 16 != 0
    worst = (0.0, 0.0)
    for alpha, beta, bias in PARAMS:
        y = booster.lrn(x, region, size, alpha, beta, bias)
        used = check_lrn(x, y, region, size, alpha, beta, bias)
        assert max(used) <= 1.0, (alpha, beta, bias, used)
        worst = tuple(max(a, b) for a, b in zip(worst, used))
    print(f"\nlrn {shape} region {region} size {size} offset {offset}: bound shares {worst[0]:.3f} / {worst[1]:.3f}")


# ---- kernels against the references ----------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("size", [1, 3, 5, 7, 9])
@pytest.mark.parametrize("shape", ACROSS_SHAPES, ids=ACROSS_IDS)
def test_across_within_bounds(cuda, shape, size):
    _run_cases(shape, 0, size)


@gpu
@pytest.mark.parametrize("size", [1, 3, 5, 7, 9])
@pytest.mark.parametrize("shape", WITHIN_SHAPES, ids=WITHIN_IDS)
def test_within_channel_within_bounds(cuda, shape, size):
    _run_cases(shape, 1, size)


@gpu
@pytest.mark.parametrize("region, size", [(0, 5), (0, 3), (0, 9), (1, 3)])
def test_misaligned_pointer(cuda, region, size):
    _run_cases((2, 24, 28, 28), region, size, offset=1)


@gpu
def test_large_window_within_channel(cuda):
    """local_size 91 on a 120 x 130 plane: the clipped halo tile, 106 x 122 floats, exceeds the 48 KB shared-memory budget,
    so the squares come from global memory."""
    _run_cases((1, 2, 120, 130), 1, 91)


# ---- bit-exact properties ------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("region, size", [(0, 5), (0, 7), (0, 9), (1, 5)])
@pytest.mark.parametrize("shape", [(5, 64, 56, 56), (5, 7, 9, 11)], ids=["wide", "narrow"])
def test_batch_split_and_alignment_give_the_same_bits(cuda, shape, region, size):
    from feathercnn_b200 import booster
    x = _data(shape, 11)
    batched = booster.lrn(x, region, size, 0.9, 0.75, 1.0)
    for i in range(shape[0]):
        alone = booster.lrn(x[i:i + 1].clone(), region, size, 0.9, 0.75, 1.0)
        assert _bits_equal(alone[0].cpu().numpy(), batched[i].cpu().numpy()), i
    buf = torch.empty(x.numel() + 1, device="cuda")
    buf[1:].copy_(x.flatten())
    out = torch.empty(x.numel() + 1, device="cuda")
    shifted = booster.lrn(buf[1:].view(shape), region, size, 0.9, 0.75, 1.0, out=out[1:].view(shape))
    assert _bits_equal(shifted.cpu().numpy(), batched.cpu().numpy())


@gpu
@pytest.mark.parametrize("region, size", [(0, 5), (0, 9), (1, 5)])
def test_graph_replay_is_bit_identical(cuda, region, size):
    from feathercnn_b200 import booster
    x = _data((2, 192, 56, 56), 13)
    eager = booster.lrn(x, region, size, 0.9, 0.75, 1.0)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        booster.lrn(x, region, size, 0.9, 0.75, 1.0)  # warm up outside the capture
    torch.cuda.current_stream().wait_stream(stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = booster.lrn(x, region, size, 0.9, 0.75, 1.0)
    g.replay()
    torch.cuda.synchronize()
    assert _bits_equal(out.cpu().numpy(), eager.cpu().numpy())


@gpu
def test_return_codes_on_device_buffers(cuda):
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    x = _data((2, 8, 5, 5), 3)
    y = torch.full_like(x, 7.0)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = lambda out, inp, c=8, h=5, w=5, reg=0, size=5, n=2: lib.fcuda_lrn_forward(  # noqa: E731
        out, inp, c, h, w, reg, size, 1.0, 0.75, 1.0, n, s)
    assert call(p(y), p(x), reg=2) == -200
    assert call(p(y), p(x), size=4) == -200
    assert call(p(y), p(x), size=0) == -200
    assert call(p(x), p(x)) == -200                 # in place: the kernels run out of place
    assert call(None, p(x)) == -100 and call(p(y), None) == -100
    assert call(p(y), p(x), c=0) == -100 and call(p(y), p(x), h=0) == -100 and call(p(y), p(x), n=0) == -100
    torch.cuda.synchronize()
    assert (y == 7.0).all()                         # nothing ran
    assert call(p(y), p(x)) == 0


# ---- GoogLeNet and AlexNet end to end --------------------------------------------------------------------------------
SETTINGS = [(True, True), (True, False), (False, True), (False, False)]
NETS = [("googlenet", 1e-4), ("googlenet", 0.9), ("alexnet", 1e-4), ("alexnet", 0.9)]


def _lrn_args(L):
    pd = L["params"]
    return pd.get(0, 0), pd.get(1, 5), pd.get(2, 1.0), pd.get(3, 0.75), pd.get(4, 1.0)


@gpu
@pytest.mark.parametrize("model, lrn_alpha", NETS, ids=[f"{m}-alpha{a:g}" for m, a in NETS])
def test_net_end_to_end(cuda, tmp_path, model, lrn_alpha):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.ZOO[model](lrn_alpha=lrn_alpha)
    param, binf = m.save(tmp_path / model)
    layers = load_model(param, binf)
    batch = 2
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])
    idx = list(range(batch))
    lrns = [L for L in layers if L["type"] == "LRN"]
    concats = [L for L in layers if L["type"] == "Concat"]
    assert len(lrns) == 2 and len(concats) == (9 if model == "googlenet" else 0)
    probs = {}
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
                assert net.BlobShape(blob)[1:] == (c, h, w), blob
        chains, _ = rebuild_chains(layers, net.LayerFusedAway, names)
        failures, checked = [], 0
        for ch in chains:
            if ch.head["type"] == "LRN":
                continue
            algo = net.LayerConvAlgo(ch.head["name"]) if ch.head["type"] in CONV_TYPES else -1
            ins = {b: fetch(net, b, idx) for b in dict.fromkeys(ch.bottoms)}
            got = {t: fetch(net, t, idx) for t in ch.tops}
            for top, used, rel, kind, path in check_chain(ch, ins, got, FP32_SPLIT, algo):
                checked += 1
                if used > 1.0:
                    failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
        assert not failures, f"fusion {fusion} graph {graph}\n" + "\n".join(failures[:20])
        assert checked >= (60 if model == "googlenet" else 10), checked
        for L in lrns:
            assert net.LayerFusedAway(L["name"]) == 0
            xin, yout = fetch(net, L["bottoms"][0], idx), fetch(net, L["tops"][0], idx)
            used = check_lrn(xin, yout, *_lrn_args(L))
            assert max(used) <= 1.0, (L["name"], used)
            if lrn_alpha > 0.5:  # the factor must vary visibly for the check to see a wrong window
                nz = xin != 0  # ReLU zeros stay zero
                ratio = (yout[nz] / xin[nz]).cpu().numpy()
                assert ratio.max() - ratio.min() > 0.1, (L["name"], ratio.min(), ratio.max())
        for L in concats:
            want = torch.cat([fetch(net, b, idx) for b in L["bottoms"]], dim=1)
            assert _bits_equal(fetch(net, L["tops"][0], idx).cpu().numpy(), want.cpu().numpy()), L["name"]
        probs[(fusion, graph)] = net.Extract("prob")
        del net
        torch.cuda.empty_cache()
    for fusion in (True, False):
        assert _bits_equal(probs[(fusion, True)], probs[(fusion, False)]), fusion
