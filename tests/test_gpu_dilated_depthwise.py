"""Dilated depthwise convolution on the GPU: the shared-memory 3x3 / stride-1 kernel and the generic kernel against float64
per element (test_gpu_error_bounds' depthwise rule: |d| <= K U S + U |ref|), on DeepLab's shapes and a seeded random sweep
across the kernel-selection and strip boundaries; the Clip / ReLU epilogues against the clamp of the plain output; the bits
across batch splits, alignment paths and CUDA-graph replay; and DeepLab-v3 through feather::Net, chain by chain."""
from __future__ import annotations

import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_error_bounds import FP32_SPLIT, PATH, U, eps_for, excess
from test_gpu_interp_crop import bilinear_check
from test_gpu_net_bounds import CONV_TYPES, FOLD, Result, affine_of, load_model, rebuild_chains, restate_chain

pytestmark = pytest.mark.gpu
DEPTHWISE = 3


# ---- one layer through the C ABI -------------------------------------------------------------------------------------
def _geom(case):
    c, h, w, k, s, dh, dw, pt, pl = (case[k_] for k_ in ("c", "h", "w", "k", "s", "dh", "dw", "pt", "pl"))
    oh = (h + 2 * pt - dh * (k - 1) - 1) // s + 1
    ow = (w + 2 * pl - dw * (k - 1) - 1) // s + 1
    return oh, ow


def _data(case, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand((case["n"], case["c"], case["h"], case["w"]), generator=g, device="cuda") * 2 - 1
    w = torch.randn((case["c"], 1, case["k"], case["k"]), generator=g, device="cuda") / case["k"]
    b = torch.rand(case["c"], generator=g, device="cuda") - 0.5
    return x, w, b


def _ref(case, x, w, b, absolute=False):
    x, w, b = x.double(), w.double(), b.double()
    if absolute:
        x, w, b = x.abs(), w.abs(), b.abs()
    pt, pl = case["pt"], case["pl"]
    return F.conv2d(F.pad(x, (pl, pl, pt, pt)), w, b, stride=case["s"], dilation=(case["dh"], case["dw"]), groups=case["c"])


def _run(case, x, w, b, clip=None, relu=False, in_off=0, out_off=0, graph=False):
    from feathercnn_b200 import booster
    n, c, h, wd = x.shape
    k, s, pt, pl = case["k"], case["s"], case["pt"], case["pl"]
    p = booster.ConvParam.make(c, c, h, wd, k, k, stride=s, pad_lbrt=(pl, pt, pl, pt), group=c, bias=True, relu=relu)
    if clip is not None:
        p.activation = booster.ACT_CLIP
    oh, ow = _geom(case)
    p.output_h, p.output_w = oh, ow
    cb = booster.ConvBooster()
    cb.ForceSelectAlgo(DEPTHWISE)
    scratch_n, packed_n = cb.GetBufferSize(p, n)
    assert scratch_n == 0
    packed = torch.empty(packed_n, device="cuda")
    cb.Init(p, packed, w.contiguous())
    xin = torch.empty(x.numel() + in_off, device="cuda")[in_off:].view_as(x)
    xin.copy_(x)
    out = torch.full((n * c * oh * ow + out_off,), float("nan"), device="cuda")[out_off:].view(n, c, oh, ow)
    scratch = torch.empty(1, device="cuda")
    fwd = lambda: cb.ForwardOpts(p, out, xin, packed, scratch, b, clip=clip, dilation=(case["dh"], case["dw"]), batch=n)
    if graph:
        fwd()
        torch.cuda.synchronize()
        out.fill_(float("nan"))
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            fwd()
        gr.replay()
    else:
        fwd()
    torch.cuda.synchronize()
    return out.clone()


def _check(case, seed=0, **kw):
    x, w, b = _data(case, seed)
    got = _run(case, x, w, b, **kw)
    ref, s = _ref(case, x, w, b), _ref(case, x, w, b, absolute=True)
    used, _ = excess(got, ref, s, eps_for("depthwise", FP32_SPLIT) + case["k"] * case["k"] * U)
    assert used <= 1.0, (case, used)
    return x, w, b, got


def _case(c, h, w, d, n=2, k=3, s=1, dw=None, pad=None):
    """pad None: pad = dilation * (k - 1) / 2 on each axis, the plane-keeping pad of DeepLab's layers."""
    dw = d if dw is None else dw
    pt = d * (k - 1) // 2 if pad is None else pad
    pl = dw * (k - 1) // 2 if pad is None else pad
    return dict(c=c, h=h, w=w, k=k, s=s, dh=d, dw=dw, pt=pt, pl=pl, n=n)


DEEPLAB = [_case(960, 33, 33, 2), _case(576, 65, 65, 2, n=1), _case(960, 65, 65, 4, n=1), _case(384, 65, 65, 2, n=1),
           _case(320, 33, 33, 6), _case(320, 33, 33, 12), _case(256, 33, 33, 18), _case(64, 129, 129, 2, n=1)]


@pytest.mark.parametrize("case", DEEPLAB, ids=[f"c{c['c']}-{c['h']}x{c['w']}-d{c['dh']}" for c in DEEPLAB])
def test_deeplab_shapes_within_bounds(cuda, case):
    _check(case)


def _sweep(n_cases=100, seed=2024):
    """n_cases seeded geometries with a non-empty output (draws without one are skipped)."""
    rng = random.Random(seed)
    out, i = [], 0
    while len(out) < n_cases:
        i += 1
        k = rng.choice([3, 3, 3, 5])
        s = 1 if rng.random() < 0.75 else 2
        dh, dw = rng.randint(1, 18), rng.randint(1, 18)
        if dh == dw == 1:
            dh = 2
        h = rng.choice([1, 2, 3, rng.randint(4, 20), rng.randint(20, 70), rng.randint(60, 140)])
        w = rng.choice([2, 3, 5, rng.randint(4, 20), rng.randint(20, 70), rng.randint(60, 300)])
        pt, pl = rng.randint(0, dh + 1), rng.randint(0, dw + 1)
        case = dict(c=rng.choice([1, 3, 8, 17]), h=h, w=w, k=k, s=s, dh=dh, dw=dw, pt=pt, pl=pl, n=rng.randint(1, 3))
        oh, ow = _geom(case)
        if oh >= 1 and ow >= 1:
            out.append((i, case, rng.randint(0, 3), rng.randint(0, 3)))
    return out


SWEEP = _sweep()


@pytest.mark.parametrize("i, case, in_off, out_off", SWEEP, ids=[f"s{c[0]}" for c in SWEEP])
def test_random_geometries_within_bounds(cuda, i, case, in_off, out_off):
    _check(case, seed=i, in_off=in_off, out_off=out_off)


def test_sweep_reaches_both_kernels():
    fast = [c for _, c, _, _ in SWEEP if c["k"] == 3 and c["s"] == 1 and c["w"] >= 2]
    assert len(fast) >= 40 and len(SWEEP) - len(fast) >= 15
    assert any(c["h"] < c["dh"] for c in fast) and any(c["w"] < c["dw"] for c in fast)
    assert any(c["w"] % 4 for c in fast) and any(_geom(c)[1] % 4 == 0 for c in fast)
    assert any(_geom(c)[0] > 64 for c in fast)  # more than one strip
    assert any(c["c"] == 1 for _, c, _, _ in SWEEP) and any(c["n"] == 3 for _, c, _, _ in SWEEP)


EPI = [_case(16, 65, 65, 2), _case(8, 33, 36, 4), _case(5, 19, 23, 2, k=5, s=2)]


@pytest.mark.parametrize("case", EPI, ids=["d2-65", "d4-36wide", "generic"])
def test_clip_and_relu_are_the_clamp_of_the_plain_output(cuda, case):
    x, w, b, plain = _check(case)
    for lo, hi in ((0.0, 6.0), (-0.25, 0.3)):
        got = _run(case, x, w, b, clip=(lo, hi))
        assert torch.equal(got.view(torch.int32), plain.clamp(lo, hi).view(torch.int32))
    got = _run(case, x, w, b, relu=True)
    assert torch.equal(got.view(torch.int32), plain.clamp_min(0).view(torch.int32))


BITS = [_case(24, 65, 64, 2, n=3), _case(24, 33, 33, 6, n=3), _case(7, 40, 52, 3, n=3, dw=5), _case(6, 21, 17, 2, n=3, k=5)]


@pytest.mark.parametrize("case", BITS, ids=["d2-w64", "d6-33", "d3x5", "generic"])
def test_bits_across_batch_split_alignment_and_graph(cuda, case):
    x, w, b, whole = _check(case)
    bits = lambda t: t.view(torch.int32)
    for i in range(case["n"]):
        assert torch.equal(bits(_run(case, x[i:i + 1], w, b)[0]), bits(whole[i])), i
    for in_off, out_off in ((1, 0), (0, 1), (3, 2)):
        assert torch.equal(bits(_run(case, x, w, b, in_off=in_off, out_off=out_off)), bits(whole)), (in_off, out_off)
    assert torch.equal(bits(_run(case, x, w, b, graph=True)), bits(whole))


# ---- DeepLab-v3 through feather::Net ---------------------------------------------------------------------------------
def _restate_conv(ch, ins, mode, algo):
    """float64 reference, bound and S of a (possibly dilated) convolution chain: conv, folded BatchNorm / Scale, ReLU, Clip."""
    head, pd = ch.head, ch.head["params"]
    x = ins[head["bottoms"][0]]
    kw, dil = pd.get(1, 0), pd.get(2, 1)
    kh, dil_h = pd.get(11, kw), pd.get(12, dil)
    sw, pl = pd.get(3, 1), pd.get(4, 0)
    sh, pt = pd.get(13, sw), pd.get(14, pl)
    group = pd.get(7, 1)
    w = head["w"].to(x.device).double()
    b = head["b"].to(x.device).double() if head["b"] is not None else None
    conv = lambda t, ww, bb: F.conv2d(F.pad(t, (pl, pl, pt, pt)), ww, bb, stride=(sh, sw), dilation=(dil_h, dil), groups=group)
    ref, s = conv(x, w, b), conv(x.abs(), w.abs(), b.abs() if b is not None else None)
    folds = []
    for L in ch.ops:
        if L["type"] in ("BatchNorm", "Scale"):
            m, a, A = affine_of(L)
            ref = ref * m.to(ref).view(1, -1, 1, 1) + a.to(ref).view(1, -1, 1, 1)
            s = s * m.abs().to(s).view(1, -1, 1, 1) + A.to(s).view(1, -1, 1, 1)
            folds.append(L)
        elif L["type"] == "ReLU":
            ref = ref.clamp_min(0)
        elif L["type"] == "Clip":
            ref = ref.clamp(float(np.float32(L["params"].get(0, 0.0))), float(np.float32(L["params"].get(1, 0.0))))
        elif L["type"] == "Eltwise":  # a shortcut added in the implicit GEMM's epilogue
            r = ins[ch.residual]
            ref, s = ref + r, s + r.abs()
        else:
            raise AssertionError((head["name"], L["type"]))
    assert algo in PATH and "f" not in PATH[algo], (head["name"], algo)  # no Winograd layer in these nets
    coef = eps_for(PATH[algo], mode) + w.shape[1] * kh * kw * U + (FOLD if folds else 0.0)
    kind = head["type"] + "".join("+" + L["type"] for L in ch.ops)
    return Result(ch.tops[0], ref, coef * s + U * ref.abs(), s, kind, PATH[algo])


def _clip_chain(ch, ins):
    x = ins[ch.head["bottoms"][0]]
    pd = ch.head["params"]
    ref = x.clamp(float(np.float32(pd.get(0, 0.0))), float(np.float32(pd.get(1, 0.0))))
    return Result(ch.tops[0], ref, torch.zeros_like(ref), ref.abs(), "Clip", "exact")


def check_deeplab(net, layers, x):
    """Every surviving blob against the float64 restatement of its chain from the Net's own inputs of that chain.  Returns
    the chains checked and the dilated depthwise layers seen, with their algorithms."""
    names = set(net.BlobNames())
    chains, _ = rebuild_chains(layers, net.LayerFusedAway, names)
    got = {n: torch.from_numpy(net.Extract(n)).cuda().double() for n in names}
    got["data"] = torch.from_numpy(x).cuda().double()
    dilated = {}
    for ch in chains:
        head, typ = ch.head, ch.head["type"]
        if typ == "Interp":
            assert not ch.ops
            used, _, _ = bilinear_check(got[ch.tops[0]].cpu(), got[head["bottoms"][0]].cpu(), head["params"].get(6, 0))
            assert used <= 1.0, (head["name"], used)
            continue
        ins = {b: got[b] for b in ch.bottoms}
        if typ in CONV_TYPES:
            algo = net.LayerConvAlgo(head["name"])
            if head["params"].get(2, 1) > 1:
                dilated[head["name"]] = algo
            results = [_restate_conv(ch, ins, FP32_SPLIT, algo)]
        elif typ == "Clip":
            results = [_clip_chain(ch, ins)]
        else:
            results = restate_chain(ch, ins, FP32_SPLIT)
        for r in results:
            g = got[r.top].reshape(r.ref.shape)
            used, _ = excess(g, r.ref, r.bound, 1.0, 0.0)
            assert used <= 1.0, (r.top, r.kind, used)
    return len(chains), dilated


@pytest.mark.parametrize("model", ["deeplabv3_tiny", "deeplabv3_mobilenet_v2"])
def test_deeplab_net_within_bounds(cuda, tmp_path, model):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    mw = getattr(modelgen, model)()
    param, binf = mw.save(tmp_path / model)
    layers = load_model(param, binf)
    x = np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(2)])
    dw_clips = {L["name"]: L["tops"][0] for L in layers if L["type"] == "Clip"}
    dilated_dw = [L["name"] for L in layers if L["type"] == "ConvolutionDepthWise" and L["params"].get(2, 1) > 1]
    assert dilated_dw
    outs = {}
    for fusion in (False, True):
        for graph in (False, True):
            net = Net(fusion=fusion, cuda_graph=graph)
            net.LoadParam(param)
            net.LoadWeights(binf)
            for _ in range(3 if graph else 1):  # graph: eager warm-up, capture, replay
                net.Forward(x)
            n, dilated = check_deeplab(net, layers, x)
            assert dilated == {name: DEPTHWISE for name in dilated_dw}, dilated
            for name in dilated_dw:
                clip = name + "_relu6"
                assert clip in dw_clips and net.LayerFusedAway(clip) == int(fusion), clip
            outs[fusion, graph] = net.Extract("logits_up")
            assert outs[fusion, graph].shape == (2,) + mw.shape["logits_up"]
    for fusion in (False, True):
        assert np.array_equal(outs[fusion, True].view(np.int32), outs[fusion, False].view(np.int32))
