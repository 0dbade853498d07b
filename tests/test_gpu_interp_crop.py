"""Interp and Crop on the GPU: nearest and crops bit-exact, bilinear within a per-element bound of float64 torch, batch
independence, feather::Net end to end on modelgen.fcn8s_tiny() / deeplab_head_tiny() (fusion and CUDA graphs on and
off, folded crops bit-identical to unfused ones) and a converted Caffe FCN-8s-style model.

Bilinear bound.  With u = 2^-24 (fp32 rounding to nearest), the kernel computes for each output
    a = f - i0 (exact), a0 = fl(1 - a) (|error| <= u), h = fl(a * p1 + fl(a0 * p0)) on two input rows, then
    v = fl(b * h1 + fl(b0 * h0)).
Each two-term lerp carries at most 3u relative to |w0 * p0| + |w1 * p1| (weight, product, FMA), so the value error is
at most 6u * S + O(u^2), S = the same interpolation of |x| (torch float64 on |x|); the bound uses 8u * S.  The fp32
source coordinate f differs from the exact one by at most 4u * max(in, 1) (the rounded scale, product and
subtraction, each <= u * in), which moves the output along its piecewise-linear profile by at most that times the local
slope L: the largest |x[j + 1] - x[j]| over the neighbouring intervals j in {i0 - 1, i0, i0 + 1} of the rows (columns)
involved.  So |got - ref| <= 8u * S + 4u * W * Lx + 4u * H * Ly + 2^-23 * |ref| (the last term as in
test_gpu_error_bounds.excess), element by element; no global tolerance."""
from __future__ import annotations

import types
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_deconv import _load_layers
from test_gpu_deconv import _restate as deconv_restate
from test_gpu_error_bounds import FP32_SPLIT, PATH, U, WINO_MARGIN, WINOGRADF23, WINOGRADF63, Conv, conv_ref, eps_for, \
    wino_model
from test_interp_crop_host import crop_caffemodel, nearest_index, nearest_scale

pytestmark = pytest.mark.gpu

UR = 2.0 ** -24


# ---- the bilinear checker ------------------------------------------------------------------------------------------
def _coords64(out, n_in, align):
    d = np.arange(out, dtype=np.float64)
    if align:
        f = d * ((n_in - 1) / (out - 1)) if out > 1 else np.zeros(out)
    else:
        f = np.maximum((d + 0.5) * n_in / out - 0.5, 0.0)
    i0 = np.minimum(np.floor(f).astype(np.int64), n_in - 1)
    return i0, np.minimum(i0 + 1, n_in - 1)


def _neighbour_slopes(diffs, i0):
    """max of |diff| over intervals i0 - 1, i0, i0 + 1 along the last axis (0 past the ends)."""
    n = diffs.shape[-1]
    pad = np.concatenate([diffs, np.zeros(diffs.shape[:-1] + (1,))], -1) if n else np.zeros(diffs.shape[:-1] + (1,))
    last = pad.shape[-1] - 1
    idx = [np.clip(i0 + k, 0, last) for k in (-1, 0, 1)]
    return np.maximum(np.maximum(pad[..., idx[0]], pad[..., idx[1]]), pad[..., idx[2]])


def bilinear_check(got, x, align, coef_in=0.0, s_in=None):
    """(largest share of the per-element bound used, reference) for a bilinear Interp of x (N, C, H, W) -> got."""
    x64 = torch.as_tensor(x).double()
    n, c, h, w = x64.shape
    oh, ow = got.shape[2:]
    ref = F.interpolate(x64, size=(oh, ow), mode="bilinear", align_corners=bool(align))
    s = F.interpolate(x64.abs() if s_in is None else torch.as_tensor(s_in).double(), size=(oh, ow), mode="bilinear",
                      align_corners=bool(align))
    xa = x64.numpy()
    y0, y1 = _coords64(oh, h, align)
    x0, x1 = _coords64(ow, w, align)
    mx = _neighbour_slopes(np.abs(np.diff(xa, axis=3)), x0)                   # (N, C, H, OW)
    lx = np.maximum(mx[:, :, y0, :], mx[:, :, y1, :])                         # (N, C, OH, OW)
    my = _neighbour_slopes(np.abs(np.diff(xa, axis=2)).transpose(0, 1, 3, 2), y0).transpose(0, 1, 3, 2)  # (N, C, OH, W)
    ly = np.maximum(my[:, :, :, x0], my[:, :, :, x1])
    bound = (coef_in + 8 * UR) * s.numpy() + 4 * UR * max(w, 1) * lx + 4 * UR * max(h, 1) * ly + U * np.abs(ref.numpy())
    d = np.abs(torch.as_tensor(got).double().cpu().numpy() - ref.numpy())
    used = np.where(d == 0, 0.0, d / np.maximum(bound, 1e-300))
    return float(used.max()), ref, s


def nearest_ref(x, oh, ow, hs, ws):
    """The fp32 gather rule of include/fcuda.h in NumPy."""
    x = np.asarray(x)
    sy = nearest_index(oh, x.shape[2], hs)
    sx = nearest_index(ow, x.shape[3], ws)
    return x[:, :, sy][:, :, :, sx]


# ---- Interp ---------------------------------------------------------------------------------------------------------
# (name, N, C, H, W, out_h, out_w, scale)
INTERP_CASES = [
    ("x2", 2, 3, 16, 16, 32, 32, None),
    ("x8_b16", 16, 21, 16, 16, 128, 128, None),
    ("ow_not_mult4", 2, 3, 7, 9, 13, 18, None),
    ("ow_lt4", 2, 2, 5, 5, 6, 3, None),
    ("h1", 2, 2, 1, 8, 4, 16, None),
    ("w1", 2, 2, 8, 1, 16, 5, None),
    ("oh1", 2, 2, 8, 8, 1, 12, None),
    ("ow1", 2, 2, 8, 8, 12, 1, None),
    ("odd", 3, 5, 11, 13, 37, 29, None),
    ("equal", 2, 3, 9, 12, 9, 12, None),
    ("tiles", 1, 2, 4, 300, 3, 1100, None),
    ("down_half", 2, 3, 20, 30, 0, 0, 0.5),
    ("down_0p3", 2, 3, 23, 31, 0, 0, 0.3),
    ("up_2p5", 2, 3, 7, 9, 0, 0, 2.5),
]


def _data(name, shape):
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    return torch.rand(shape, generator=g) * 2 - 1


@pytest.mark.parametrize("case", INTERP_CASES, ids=[c[0] for c in INTERP_CASES])
def test_nearest_is_the_fp32_gather(cuda, case):
    from feathercnn_b200 import booster
    name, n, c, h, w, oh, ow, scale = case
    x = _data(name, (n, c, h, w))
    got = booster.interp(x.cuda(), oh, ow, "nearest", scale=scale).cpu()
    p = booster.interp_param(h, w, oh, ow, "nearest", scale=scale)
    hs = nearest_scale(h, p.output_h, oh, 1.0 if scale is None else scale)
    ws = nearest_scale(w, p.output_w, ow, 1.0 if scale is None else scale)
    want = nearest_ref(x.numpy(), p.output_h, p.output_w, hs, ws)
    assert np.array_equal(got.numpy().view(np.int32), want.view(np.int32)), name
    if oh and ow and oh % h == 0 and ow % w == 0:  # integer scales: torch's nearest is the same gather
        assert torch.equal(got, F.interpolate(x, size=(oh, ow), mode="nearest"))


@pytest.mark.parametrize("align", [0, 1], ids=["half_pixel", "align_corners"])
@pytest.mark.parametrize("case", INTERP_CASES, ids=[c[0] for c in INTERP_CASES])
def test_bilinear_within_bounds(cuda, case, align):
    from feathercnn_b200 import booster
    name, n, c, h, w, oh, ow, scale = case
    x = _data(name, (n, c, h, w))
    got = booster.interp(x.cuda(), oh, ow, "bilinear", bool(align), scale=scale).cpu()
    used, ref, _ = bilinear_check(got, x, align)
    assert used <= 1.0, (name, used)
    if (oh, ow) == (h, w):
        assert torch.equal(got, x)


# ---- Crop -----------------------------------------------------------------------------------------------------------
# (name, N, C, H, W, coff, hoff, woff, oc, oh, ow)
CROP_CASES = [
    ("fcn_odd", 2, 5, 40, 43, 0, 19, 19, 5, 20, 21),
    ("odd_channels", 2, 7, 20, 23, 1, 5, 9, 3, 11, 13),
    ("vec", 2, 4, 16, 32, 0, 3, 8, 4, 10, 16),
    ("vec_channels", 3, 6, 9, 64, 2, 0, 4, 3, 9, 56),
    ("whole", 2, 3, 5, 7, 0, 0, 0, 3, 5, 7),
    ("one_column", 2, 3, 6, 7, 0, 1, 6, 3, 4, 1),
    ("wide_row", 1, 2, 3, 1000, 1, 1, 3, 1, 2, 997),
]


@pytest.mark.parametrize("case", CROP_CASES, ids=[c[0] for c in CROP_CASES])
def test_crop_is_exact(cuda, case):
    from feathercnn_b200 import booster
    name, n, c, h, w, co, ho, wo, oc, oh, ow = case
    x = _data(name, (n, c, h, w))
    got = booster.crop(x.cuda(), co, ho, wo, oc, oh, ow).cpu()
    assert torch.equal(got, x[:, co:co + oc, ho:ho + oh, wo:wo + ow]), name


def test_crop_window_outside_the_input_is_rejected(cuda):
    from feathercnn_b200 import booster
    x = torch.zeros((1, 3, 8, 8), device="cuda")
    for args in ((0, 0, 1, 3, 8, 8), (1, 0, 0, 3, 8, 8), (0, 5, 0, 3, 4, 8)):
        with pytest.raises(booster.FcudaError) as e:
            booster.crop(x, *args)
        assert e.value.code == -100


def test_batch_images_equal_single_images(cuda):
    from feathercnn_b200 import booster
    x = _data("batch5", (5, 3, 13, 17)).cuda()
    runs = [lambda t: booster.interp(t, 50, 36, "bilinear"), lambda t: booster.interp(t, 50, 37, "bilinear", True),
            lambda t: booster.interp(t, 0, 0, "nearest", scale=3.0), lambda t: booster.crop(t, 1, 3, 5, 2, 9, 11)]
    for run in runs:
        full = run(x)
        for i in range(5):
            assert torch.equal(run(x[i:i + 1].contiguous())[0].view(torch.int32), full[i].view(torch.int32))


def test_interp_and_crop_are_capturable(cuda):
    from feathercnn_b200 import booster
    x = _data("graph", (2, 3, 10, 12)).cuda()
    eager = [booster.interp(x, 40, 48, "bilinear"), booster.crop(x, 1, 2, 3, 2, 5, 7)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        booster.interp(x, 40, 48, "bilinear")  # warm-up on the capture stream
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            outs = [booster.interp(x, 40, 48, "bilinear"), booster.crop(x, 1, 2, 3, 2, 5, 7)]
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(outs, eager):
        assert torch.equal(a, b)


# ---- feather::Net end to end ----------------------------------------------------------------------------------------
def _conv_restate(layer, ins, mode, net):
    t, name, bottoms, tops, prm, wts = layer
    x, sx, cx = ins[0][:3]
    oc, kw, st, pw = int(prm[0]), int(prm[1]), int(prm.get(3, 1)), int(prm.get(4, 0))
    kh, ph, dil = int(prm.get(11, kw)), int(prm.get(14, pw)), int(prm.get(2, 1))
    w = wts[0].view(oc, -1, kh, kw)
    b = wts[1] if len(wts) > 1 else None
    c = Conv(name, oc, x.shape[1], x.shape[2], x.shape[3], kh, kw, st, st, (pw, ph, pw, ph), dil=dil, bias=b is not None,
             batch=x.shape[0])
    y = conv_ref(c, x, w, b, None)
    s = conv_ref(c, sx, w, b, None, absolute=True)
    algo = net.LayerConvAlgo(name)
    if algo in (WINOGRADF63, WINOGRADF23):  # the Winograd model's worst |d| / S on the first image, times the margin
        ym = wino_model(c, x[:1].float(), w, b, 8 if algo == WINOGRADF63 else 4, mode)
        rho = float(((ym - y[:1]).abs() / s[:1].clamp_min(1e-300)).max())
        return y, s, cx + WINO_MARGIN * rho + c.K * U
    assert algo in (0, 1, 2, 3), (name, algo)
    return y, s, cx + eps_for(PATH[algo], mode) + c.K * U


def _restate(layer, ins, mode, net):
    """float64 (ref, S, coef, extra) of one layer: |got - ref| <= coef * S + U * |ref| + extra."""
    t, name, bottoms, tops, prm, wts = layer
    x, sx, cx = ins[0][:3]
    if t == "Convolution":
        return _conv_restate(layer, ins, mode, net) + (0.0,)
    if t == "Pooling":
        assert int(prm.get(0, 0)) == 0 and int(prm[1]) == 2 and int(prm.get(2, 1)) == 2
        return F.max_pool2d(x, 2, 2, ceil_mode=True), F.max_pool2d(sx, 2, 2, ceil_mode=True), cx, 0.0
    if t == "Eltwise":
        (a, sa, ca), (b, sb, cb) = (i[:3] for i in ins)
        return a + b, sa + sb, max(ca, cb) + U, 0.0
    if t == "Crop":
        wo, ho = int(prm.get(0, 0)), int(prm.get(1, 0))
        if len(ins) > 1:
            oh, ow = ins[1][0].shape[2:]
        else:
            oh, ow = int(prm.get(4, 0)) or x.shape[2] - ho, int(prm.get(3, 0)) or x.shape[3] - wo
        sl = (slice(None), slice(None), slice(ho, ho + oh), slice(wo, wo + ow))
        return x[sl], sx[sl], cx, 0.0
    if t == "Interp":
        assert int(prm[0]) == 2 and float(prm[1]) == 8.0
        got = torch.from_numpy(net.Extract(tops[0])).double()
        used, ref, s = bilinear_check(got, x, int(prm.get(6, 0)), cx, sx)
        assert used <= 1.0, (name, used)
        return ref, s, cx + 8 * UR, float("inf")  # checked here: the coordinate term needs the input's slopes
    return deconv_restate(layer, [i[:3] for i in ins], mode, net) + (0.0,)


def check_net(mw, net, x, mode=FP32_SPLIT):
    """Every surviving blob against the float64 restatement of the chain of (possibly fused) layers that produced it,
    starting from the Net's own values of the blobs that chain reads (test_gpu_deconv.check_net with the new layers)."""
    names = set(net.BlobNames())
    have = {}
    for layer in _load_layers(mw):
        t, name, bottoms, tops = layer[:4]
        if t == "Input":
            have[tops[0]] = (torch.from_numpy(x).double(), torch.from_numpy(x).double().abs(), 0.0, 0.0)
            continue
        ins = []
        for bn in bottoms:
            if bn in names and bn != "data":
                v = torch.from_numpy(net.Extract(bn)).double().reshape(have[bn][0].shape)
                ins.append((v, v.abs(), 0.0, 0.0))
            else:
                ins.append(have[bn])
        if t == "Split":
            for tn in tops:
                have[tn] = ins[0]
            continue
        have[tops[0]] = _restate(layer, ins, mode, net)
    checked = 0
    for bn, (ref, s, coef, extra) in have.items():
        if bn not in names or bn == "data" or extra == float("inf"):
            continue
        got = torch.from_numpy(net.Extract(bn)).double().reshape(ref.shape)
        d = (got - ref).abs()
        bound = coef * s + U * ref.abs() + extra
        used = float(torch.where(d == 0, torch.zeros_like(d), d / bound.clamp_min(1e-300)).max())
        assert used <= 1.0, (bn, used)
        checked += 1
    return checked


def _net(mw, tmp_path, fusion, graph, stem="model"):
    from feathercnn_b200.net import Net
    param, binf = mw.save(tmp_path / stem)
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    return net


def _images(n, shape, scale=2.0):
    from feathercnn_b200.tools import modelgen
    return np.stack([modelgen.synthetic_input(shape, i) * scale for i in range(n)])


def _forward(net, x, graph):
    for _ in range(3 if graph else 1):  # graph: eager warm-up, capture, replay
        net.Forward(x)


@pytest.mark.parametrize("model", ["fcn8s_tiny", "deeplab_head_tiny"])
def test_segmentation_nets(cuda, tmp_path, model):
    from feathercnn_b200.tools import modelgen
    mw = getattr(modelgen, model)()
    x = _images(5, mw.shape["data"])
    outs = {}
    for fusion in (False, True):
        for graph in (False, True):
            net = _net(mw, tmp_path, fusion, graph)
            _forward(net, x, graph)
            outs[fusion, graph] = {n: net.Extract(n) for n in net.BlobNames()}
            assert check_net(mw, net, x) >= (8 if model == "fcn8s_tiny" else 5)
            if model == "fcn8s_tiny":
                assert net.LayerFusedAway("score") == int(fusion)
                assert net.LayerFusedAway("score_pool4c") == 0 and net.LayerFusedAway("score_pool3c") == 0
                assert ("upscore8" in outs[fusion, graph]) == (not fusion)
            single = _net(mw, tmp_path, fusion, graph)
            for i in (0, 4):
                _forward(single, x[i:i + 1], graph)
                for n in single.BlobNames():
                    if n != "data":
                        assert np.array_equal(single.Extract(n)[0].view(np.int32),
                                              outs[fusion, graph][n][i].view(np.int32)), (n, i)
    ref = outs[False, False]
    for key, o in outs.items():
        for n in o:  # the fused nets have fewer blobs; every one they have is bit-identical to the unfused net's
            assert np.array_equal(o[n].view(np.int32), ref[n].view(np.int32)), (key, n)
    final = "score" if model == "fcn8s_tiny" else "upsample"
    assert outs[True, True][final].shape == (5,) + mw.shape[final]


def test_folded_crop_of_a_depthwise_deconvolution(cuda, tmp_path):
    """The gather kernel's path: a bilinear DeconvolutionDepthWise cropped to the input (one-bottom and two-bottom)."""
    from feathercnn_b200.tools import modelgen
    for two_bottoms in (False, True):
        mw = modelgen.ModelWriter(3)
        data = mw.input("data", 4, 12, 12)
        x = mw.conv("conv", data, 4, 3, 2, 1, True)
        x = mw.deconv("up", x, 4, 8, 4, 0, False, group=4, weights=modelgen.bilinear_kernel(4, 8))
        if two_bottoms:
            mw.crop("crop", x, 3, 5, reference=data)
        else:
            mw.crop("crop", x, 3, 5, outh=12, outw=11)
        xs = _images(3, mw.shape["data"])
        got = {}
        for fusion in (False, True):
            net = _net(mw, tmp_path, fusion, False, f"dw{int(two_bottoms)}")
            net.Forward(xs)
            assert net.LayerFusedAway("crop") == int(fusion)
            assert check_net(mw, net, xs) >= 2
            got[fusion] = net.Extract("crop")
        assert np.array_equal(got[False].view(np.int32), got[True].view(np.int32))


def test_stride1_deconvolution_keeps_its_crop(cuda, tmp_path):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.ModelWriter(4)
    data = mw.input("data", 8, 10, 10)
    x = mw.deconv("up", data, 8, 2, 1, 0, True)   # direct path; 2x2 keeps the equivalent convolution off Winograd
    mw.crop("crop", x, 1, 1, reference=data)
    net = _net(mw, tmp_path, True, False)
    net.Forward(_images(2, mw.shape["data"]))
    assert net.LayerFusedAway("crop") == 0
    assert check_net(mw, net, _images(2, mw.shape["data"])) >= 2


def test_crop_window_outside_fails_forward(cuda, tmp_path):
    from feathercnn_b200.net import FeatherError, Net
    net = Net()
    net.LoadParamFromText("7767517\n2 2\nInput data 0 1 data 0=8 1=8 2=3\nCrop c 1 1 data out 0=2 1=2 3=7 4=7\n")
    with pytest.raises(FeatherError):
        net.Forward(np.zeros((1, 3, 8, 8), np.float32))


# ---- a converted Caffe model ----------------------------------------------------------------------------------------
def test_caffe_fcn8s_style_model(cuda, tmp_path):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import caffe2feather
    rng = np.random.default_rng(5)
    model, _ = crop_caffemodel(rng)
    path = tmp_path / "fcn8s.caffemodel"
    path.write_bytes(model)
    param, binf = caffe2feather.convert_file(path, tmp_path / "fcn8s")
    text = open(param).read()
    mw = types.SimpleNamespace(lines=text.splitlines()[2:], bin=open(binf, "rb").read())
    x = rng.uniform(-1, 1, (3, 4, 16, 16)).astype(np.float32)
    outs = {}
    for fusion in (False, True):
        net = Net(fusion=fusion)
        net.LoadParam(param)
        net.LoadWeights(binf)
        net.Forward(x)
        assert net.LayerFusedAway("score") == int(fusion)
        assert check_net(mw, net, x) >= 5
        outs[fusion] = net.Extract("score")
    assert outs[True].shape == (3, 3, 16, 16)
    assert np.array_equal(outs[False].view(np.int32), outs[True].view(np.int32))
