"""Deconvolution on the GPU: per-element bounds against float64, bit-exactness against the equivalent convolution run on
its own, feather::Net end to end on modelgen.decoder_tiny(), and a converted Caffe FCN-style model.

The bound is the one of test_gpu_error_bounds.py:  |got - ref| <= (eps(path, mode) + K * 2^-23) * S + 2^-23 * |ref|, with
S the deconvolution on |x|, |w| plus |b|, K the products per output, eps of the path the plan reports (0 for the CUDA-core
gather) and, on a Winograd equivalent convolution, the Winograd model's ceiling instead."""
from __future__ import annotations

import ctypes
import dataclasses
import zlib

import numpy as np
import pytest
import torch

from test_deconv_host import (caffe_to_ncnn, deconv_ref, equivalent_filter, fcn_caffemodel, plan_ref, scatter)
from test_gpu_error_bounds import (FP32_SPLIT, MODES, PATH, TF32, U, WINO_MARGIN, WINOGRADF23, WINOGRADF63, Conv, conv_ref,
                                   eps_for, excess, wino_model)

pytestmark = pytest.mark.gpu


@dataclasses.dataclass
class Case:
    name: str
    oc: int
    ic: int
    h: int
    w: int
    k: int | tuple[int, int] = 4
    stride: tuple[int, int] = (2, 2)
    pad: tuple[int, int, int, int] = (1, 1, 1, 1)   # top, bottom, left, right
    output_pad: tuple[int, int] = (0, 0)             # bottom, right
    dil: tuple[int, int] = (1, 1)
    group: int = 1
    bias: bool = True
    relu: bool = False
    batch: int = 2

    @property
    def kh(self):
        return self.k if isinstance(self.k, int) else self.k[0]

    @property
    def kw(self):
        return self.k if isinstance(self.k, int) else self.k[1]

    @property
    def geometry(self):
        return (self.oc, self.ic, self.h, self.w, self.kh, self.kw, self.stride, self.pad, self.output_pad, self.dil,
                self.group)

    def data(self):
        g = torch.Generator().manual_seed(zlib.crc32(self.name.encode()))
        icg = self.ic // self.group
        x = torch.rand((self.batch, self.ic, self.h, self.w), generator=g) * 2 - 1
        fan = icg * self.kh * self.kw / (self.stride[0] * self.stride[1])
        w = torch.randn((self.oc, icg, self.kh, self.kw), generator=g) * (2.0 / fan) ** 0.5
        w = w * torch.pow(10.0, -2 * torch.rand((self.oc, 1, 1, 1), generator=g))
        b = (torch.rand(self.oc, generator=g) - 0.5) if self.bias else None
        return x, w, b


CASES = [
    Case("k4s2p1", 32, 64, 9, 11, relu=True),
    Case("k2s2", 48, 32, 8, 8, k=2, pad=(0, 0, 0, 0)),
    Case("k3s2p1_op1", 24, 32, 7, 9, k=3, output_pad=(1, 1)),
    Case("k1s2_empty_phases", 16, 32, 6, 6, k=1, pad=(0, 0, 0, 0), output_pad=(1, 1)),
    Case("k5s3_four_pads", 16, 32, 5, 6, k=5, stride=(3, 3), pad=(0, 2, 1, 3)),
    Case("s21_k43", 16, 32, 6, 7, k=(4, 3), stride=(2, 1), pad=(1, 2, 1, 0)),
    Case("k3s1d2_direct", 32, 32, 12, 12, k=3, stride=(1, 1), dil=(2, 2), pad=(2, 2, 2, 2), relu=True),
    Case("k3s1p1_direct", 64, 64, 20, 20, k=3, stride=(1, 1), relu=True),   # equivalent convolution on Winograd F(6,3)
    Case("s1_pad_gt_k", 16, 32, 8, 8, k=3, stride=(1, 1), pad=(3, 0, 1, 4)),
    Case("ic3", 16, 3, 8, 8),
    Case("ic17_ktable", 16, 17, 8, 8),
    Case("oc1", 1, 32, 8, 8),
    Case("oc65", 65, 32, 8, 8, k=3, output_pad=(1, 0)),
    Case("group4", 32, 64, 8, 8, group=4, relu=True),
    Case("dw_k4s2p1", 21, 21, 16, 16, group=21, bias=False),
    Case("dw_k16s8p4", 21, 21, 8, 8, k=16, stride=(8, 8), pad=(4, 4, 4, 4), group=21, bias=False),
    Case("dw_k3s1d2_relu", 8, 8, 9, 9, k=3, stride=(1, 1), dil=(2, 2), pad=(1, 2, 0, 3), group=8, relu=True),
    Case("dw_multiplier2", 32, 16, 8, 8, group=16),
    Case("dcgan_b1", 128, 256, 16, 16, batch=1),
    Case("dcgan_b3", 128, 256, 16, 16, batch=3),
    Case("dcgan_b64", 128, 256, 16, 16, batch=64),
]
MODE_SUBSET = {"k4s2p1", "k3s2p1_op1", "k3s1p1_direct", "group4", "dw_k4s2p1"}


def _params():
    for c in CASES:
        for mname, mode in MODES.items():
            if mode == FP32_SPLIT or c.name in MODE_SUBSET:
                yield pytest.param(c, mode, id=f"{c.name}-{mname}")


def _eq_conv(eq, w) -> Conv:
    return Conv("eq", eq.output_channels, eq.input_channels, eq.input_h, eq.input_w, eq.kernel_h, eq.kernel_w,
                pad=(eq.pad_left, eq.pad_bottom, eq.pad_right, eq.pad_top), bias=False, batch=1)


def run_case(c: Case, mode: int):
    from feathercnn_b200 import booster
    booster.set_precision(mode)
    x, w, b = c.data()
    got, algo = booster.deconv_forward(x.cuda(), w.cuda(), None if b is None else b.cuda(), c.stride, c.pad, c.output_pad,
                                       c.dil, c.group, c.relu)
    torch.cuda.synchronize()
    return x, w, b, got, algo


def bound_coef(c: Case, mode: int, algo: int, x, w) -> float:
    path, e = plan_ref(*c.geometry)
    K = c.ic // c.group * -(-c.kh // c.stride[0]) * -(-c.kw // c.stride[1])
    if algo not in (WINOGRADF63, WINOGRADF23):
        return (0.0 if path == "dw" else eps_for(PATH[algo], mode)) + K * U
    # Winograd equivalent convolution: the model's worst |d|/S on the first image, times the margin
    from feathercnn_b200 import booster
    eq, _ = booster.deconv_plan(booster.deconv_param(*c.geometry[:6], c.stride, c.pad, c.output_pad, c.dil, c.group))
    cc = _eq_conv(eq, w)
    wp = torch.from_numpy(equivalent_filter(w.numpy(), c.stride, c.group, path))
    ym = wino_model(cc, x[:1], wp, None, 8 if algo == WINOGRADF63 else 4, mode)
    _, rho = excess(ym, conv_ref(cc, x[:1], wp, None, None), conv_ref(cc, x[:1], wp, None, None, absolute=True), 1.0)
    return WINO_MARGIN * rho


@pytest.mark.parametrize("c, mode", list(_params()))
def test_deconv_within_bounds(cuda, c, mode):
    x, w, b, got, algo = run_case(c, mode)
    path, _ = plan_ref(*c.geometry)
    assert (algo == 3) == (path == "dw"), (c.name, algo)
    coef = bound_coef(c, mode, algo, x, w)
    step = 8
    for i0 in range(0, c.batch, step):
        sl = slice(i0, i0 + step)
        ref = deconv_ref(x[sl], w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, c.relu)
        s = deconv_ref(x[sl], w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, absolute=True)
        used, _ = excess(got[sl].cpu(), ref, s, coef)
        assert used <= 1.0, (c.name, used)


@pytest.mark.parametrize("c, mode", [p for p in _params() if plan_ref(*p.values[0].geometry)[0] != "dw"])
def test_deconv_equals_its_equivalent_convolution(cuda, c, mode):
    """Bit for bit: the equivalent convolution with the NumPy-built filter (no bias), scattered, + bias, then ReLU; the
    stride-1 direct path is that convolution with the bias and ReLU in it."""
    from feathercnn_b200 import booster
    x, w, b, got, algo = run_case(c, mode)
    path, e = plan_ref(*c.geometry)
    eq, algo2 = booster.deconv_plan(booster.deconv_param(*c.geometry[:6], c.stride, c.pad, c.output_pad, c.dil, c.group,
                                                         c.bias, c.relu))
    assert algo2 == algo
    wp = torch.from_numpy(equivalent_filter(w.numpy(), c.stride, c.group, path)).cuda()
    xc = x.cuda()
    bc = None if b is None else b.cuda()
    if path == "direct":
        want, a = booster.conv_forward(eq, xc, wp, bc if c.bias else None, algo=algo, dilation=e["dil"][0])
    else:
        P, a = booster.conv_forward(eq, xc, wp, None, algo=algo, dilation=e["dil"][0])
        want = scatter(P, c.oc, c.group, c.stride, c.pad, tuple(got.shape[2:]))
        if bc is not None:
            want = want + bc.view(1, -1, 1, 1)
        if c.relu:
            want = torch.where(want > 0, want, torch.zeros_like(want))
    torch.cuda.synchronize()
    assert a == algo
    assert torch.equal(got.view(torch.int32), want.contiguous().view(torch.int32)), c.name


# ---- feather::Net end to end ----------------------------------------------------------------------------------------
def _load_layers(mw):
    """(type, name, bottoms, tops, params, weights) of a ModelWriter's layers, weights read back from its .bin bytes."""
    buf = bytes(mw.bin)
    off = 0

    def take(n, flagged):
        nonlocal off
        off += 4 if flagged else 0
        a = np.frombuffer(buf, "<f4", n, off).copy()
        off += 4 * n
        return torch.from_numpy(a)

    layers = []
    for line in mw.lines:
        tok = line.split()
        t, name, nb, nt = tok[0], tok[1], int(tok[2]), int(tok[3])
        bottoms, tops = tok[4:4 + nb], tok[4 + nb:4 + nb + nt]
        prm = {int(k): v for k, v in (kv.split("=") for kv in tok[4 + nb + nt:])}
        wts = []
        if t in ("Convolution", "Deconvolution", "DeconvolutionDepthWise"):
            wts.append(take(int(prm[6]), True))
            if int(prm.get(5, 0)):
                wts.append(take(int(prm[0]), False))
        elif t == "BatchNorm":
            wts = [take(int(prm[0]), False) for _ in range(4)]
        elif t == "Scale":
            wts = [take(int(prm[0]), False) for _ in range(1 + int(prm.get(1, 0)))]
        layers.append((t, name, bottoms, tops, prm, wts))
    assert off == len(buf)
    return layers


def _restate(layer, ins, mode, net):
    """float64 (ref, S, coef) of one layer from (ref, S, coef) of its bottoms."""
    from feathercnn_b200 import booster
    t, name, bottoms, tops, prm, wts = layer
    (x, sx, cx) = ins[0]
    if t == "Convolution":
        k, st, pd, oc = int(prm[1]), int(prm.get(3, 1)), int(prm.get(4, 0)), int(prm[0])
        w = wts[0].double().view(oc, -1, k, k)
        b = wts[1].double() if len(wts) > 1 else None
        y = torch.nn.functional.conv2d(x, w, b, st, pd)
        s = torch.nn.functional.conv2d(sx, w.abs(), None if b is None else b.abs(), st, pd)
        algo = net.LayerConvAlgo(name)
        assert algo in (0, 1, 2, 3), (name, algo)  # no Winograd in this net: one product bound per path
        return y, s, cx + eps_for(PATH[algo], mode) + w.shape[1] * k * k * U
    if t.startswith("Deconvolution"):
        k, st, pd, oc, g = int(prm[1]), int(prm.get(3, 1)), int(prm.get(4, 0)), int(prm[0]), int(prm.get(7, 1))
        w = wts[0].view(oc, -1, k, k)
        b = wts[1] if len(wts) > 1 else None
        y = deconv_ref(x, w, b, (st, st), (pd,) * 4, group=g)
        s = deconv_ref(sx, w, b, (st, st), (pd,) * 4, group=g, absolute=True)
        _, algo = booster.deconv_plan(booster.deconv_param(oc, x.shape[1], x.shape[2], x.shape[3], k, k, st, pd, group=g))
        K = w.shape[1] * (-(-k // st)) ** 2
        return y, s, cx + (0.0 if algo == 3 else eps_for(PATH[algo], mode)) + K * U
    if t == "ReLU":
        return x.clamp_min(0), sx, cx
    if t == "BatchNorm":
        slope, mean, var, bias = (v.double().view(1, -1, 1, 1) for v in wts)
        eps = float(prm[1])
        m = slope / torch.sqrt(var + eps)
        return (x - mean) * m + bias, (sx + mean.abs()) * m.abs() + bias.abs(), cx + 8 * U
    if t == "Scale":
        m = wts[0].double().view(1, -1, 1, 1)
        a = wts[1].double().view(1, -1, 1, 1) if len(wts) > 1 else torch.zeros_like(m)
        return x * m + a, sx * m.abs() + a.abs(), cx + 4 * U
    if t == "Concat":
        return (torch.cat([i[0] for i in ins], 1), torch.cat([i[1] for i in ins], 1),
                torch.cat([torch.full_like(i[0], i[2]) for i in ins], 1))
    if t == "Split":
        return x, sx, cx
    raise AssertionError(t)


def _net(mw, tmp_path, fusion, graph):
    from feathercnn_b200.net import Net
    param, binf = mw.save(tmp_path / "decoder_tiny")
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    return net


def _images(n, shape):
    from feathercnn_b200.tools import modelgen
    return np.stack([modelgen.synthetic_input(shape, i) * 2 for i in range(n)])


def check_net(mw, net, x, mode):
    """Every surviving blob against the float64 restatement of the chain of (possibly fused) layers that produced it,
    starting from the Net's own values of the blobs that chain reads."""
    names = set(net.BlobNames())
    have = {}
    for layer in _load_layers(mw):
        t, name, bottoms, tops = layer[:4]
        if t == "Input":
            have[tops[0]] = (torch.from_numpy(x).double(), torch.from_numpy(x).double().abs(), 0.0)
            continue
        ins = []
        for bn in bottoms:
            if bn in names:
                v = torch.from_numpy(net.Extract(bn)).double().reshape(have[bn][0].shape)
                ins.append((v, v.abs(), 0.0))
            else:
                ins.append(have[bn])
        if t == "Split":
            for tn in tops:
                have[tn] = ins[0]
            continue
        have[tops[0]] = _restate(layer, ins, mode, net)
    checked = 0
    for bn, (ref, s, coef) in have.items():
        if bn not in names or bn == "data":
            continue
        got = torch.from_numpy(net.Extract(bn)).double().reshape(ref.shape)
        used, _ = excess(got, ref, s, coef)
        assert used <= 1.0, (bn, used)
        checked += 1
    return checked


@pytest.mark.parametrize("fusion", [False, True], ids=["unfused", "fused"])
def test_decoder_net(cuda, tmp_path, fusion):
    from feathercnn_b200 import booster
    from feathercnn_b200.tools import modelgen
    mw = modelgen.decoder_tiny()
    x = _images(5, mw.shape["data"])
    outs = {}
    for graph in (False, True):
        net = _net(mw, tmp_path, fusion, graph)
        for _ in range(3 if graph else 1):  # graph: eager warm-up, capture, replay
            net.Forward(x)
        outs[graph] = {n: net.Extract(n) for n in net.BlobNames()}
        assert check_net(mw, net, x, FP32_SPLIT) >= 8
        if not graph:
            # the deconvolutions, against the C ABI on the Net's own bottoms: a fused ReLU is the ReLU layer's max
            for dname, bottom, top, k, s, p, relu in (("up1", "enc2_relu", "up1", 4, 2, 1, False),
                                                      ("up2", "cat1", "up2_relu" if fusion else "up2", 2, 2, 0, fusion)):
                xb = torch.from_numpy(net.Extract(bottom)).cuda().reshape(5, *mw.shape[bottom]).contiguous()
                lay = next(l for l in _load_layers(mw) if l[1] == dname)
                w = lay[5][0].view(16, -1, k, k).cuda()
                b = lay[5][1].cuda()
                plain, _ = booster.deconv_forward(xb, w, b, s, p)
                fused, _ = booster.deconv_forward(xb, w, b, s, p, relu=True)
                assert torch.equal(booster.relu(plain).view(torch.int32), fused.view(torch.int32))
                want = fused if relu else plain
                assert np.array_equal(net.Extract(top).reshape(-1).view(np.int32),
                                      want.cpu().numpy().reshape(-1).view(np.int32)), dname
        # each image of the batch equals the same image forwarded alone
        single = _net(mw, tmp_path, fusion, graph)
        for i in (0, 4):
            for _ in range(3 if graph else 1):
                single.Forward(x[i:i + 1])
            for n in single.BlobNames():
                if n != "data":
                    assert np.array_equal(single.Extract(n)[0].view(np.int32), outs[graph][n][i].view(np.int32)), (n, i)
    for n in outs[False]:
        assert np.array_equal(outs[False][n].view(np.int32), outs[True][n].view(np.int32)), n
    # switching the precision mode re-packs every filter and meets that mode's bound
    net = _net(mw, tmp_path, fusion, False)
    net.Forward(x)
    booster.set_precision(TF32)
    net.Forward(x)
    assert check_net(mw, net, x, TF32) >= 8


# ---- a converted Caffe model ----------------------------------------------------------------------------------------
def test_caffe_fcn_round_trip(cuda, tmp_path):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import caffe2feather, modelgen
    rng = np.random.default_rng(11)
    w1 = (rng.standard_normal((8, 12, 4, 4)) * 0.25).astype(np.float32)
    b1 = rng.uniform(-0.5, 0.5, 12).astype(np.float32)
    w2 = (rng.standard_normal((12, 3, 4, 4)) * 0.3).astype(np.float32)   # 4 groups, 12 outputs
    path = tmp_path / "fcn.caffemodel"
    path.write_bytes(fcn_caffemodel(w1, b1, w2, 4, ic=8, hw=6))
    param, binf = caffe2feather.convert_file(path, tmp_path / "fcn")
    net = Net()
    net.LoadParam(param)
    net.LoadWeights(binf)
    x = rng.uniform(-1, 1, (3, 8, 6, 6)).astype(np.float32)
    net.Forward(x)
    xt = torch.from_numpy(x).double()
    mid = torch.nn.functional.conv_transpose2d(xt, torch.from_numpy(w1).double(), torch.from_numpy(b1).double(), 2, 1)
    got1 = torch.from_numpy(net.Extract("up1")).double().reshape(mid.shape)
    s1 = torch.nn.functional.conv_transpose2d(xt.abs(), torch.from_numpy(w1).double().abs(), torch.from_numpy(b1).double().abs(), 2, 1)
    used, _ = excess(got1, mid, s1, eps_for("sgeconv", FP32_SPLIT) + 8 * 4 * U)
    assert used <= 1.0
    ref = torch.nn.functional.conv_transpose2d(got1, torch.from_numpy(w2).double(), None, 2, 1, groups=4)
    s2 = torch.nn.functional.conv_transpose2d(got1.abs(), torch.from_numpy(w2).double().abs(), None, 2, 1, groups=4)
    got2 = torch.from_numpy(net.Extract("up2")).double().reshape(ref.shape)
    used, _ = excess(got2, ref, s2, eps_for("sgeconv", FP32_SPLIT) + 3 * 4 * U)
    assert used <= 1.0
