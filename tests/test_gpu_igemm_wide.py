"""The wide pre-split kernel (switch igemm_wide = 1) against the pre-split kernel (igemm_wide = 0).

Both issue the same bf16 products (q1*p2, q2*p1, q1*p1 per k-step of 16) on the same operand bits in the same k order
with the same N tile; only the roles of the wgmma M and N sides are swapped.  So every output must be BIT-identical: per
layer, and on every surviving blob of the benchmark nets as feather::Net runs them (fusion and CUDA graphs on,
benchmark batch)."""
import ctypes
import zlib

import numpy as np
import pytest

from test_gpu_igemm_presplit import CASES as PRESPLIT_CASES
from test_gpu_igemm_presplit import _param

pytestmark = pytest.mark.gpu

# (name, oc, ic, h, w, kh, kw, pad or pad_lbrt, n, group, extra), every one taken by the wide kernel
WIDE_CASES = [
    ("wide_oh27_ow20_oc257", 257, 64, 27, 20, 3, 3, 1, 2, 1, ""),
    ("wide_bn64_oh55_ow52_oc40", 40, 32, 55, 52, 3, 3, 1, 2, 1, ""),
    ("wide_pool_bn128_oh55", 128, 32, 55, 56, 3, 3, 1, 2, 1, "pool"),
    ("wide_pool_bn64_oh27", 64, 64, 27, 28, 3, 3, 1, 3, 1, "pool"),
    ("wide_residual_relu_bn128", 128, 64, 28, 28, 3, 3, 1, 3, 1, "res_relu"),
    ("wide_residual_bn64", 64, 64, 28, 28, 3, 3, 1, 3, 1, "res"),
    ("wide_grouped_bn128", 256, 64, 28, 28, 3, 3, 1, 2, 2, ""),
    ("wide_pad2_bn128", 128, 32, 26, 24, 3, 3, 2, 2, 1, ""),
    ("wide_pad0_bn64", 64, 32, 30, 32, 3, 3, 0, 2, 1, ""),
    ("wide_k5x5_pad2_bn128", 128, 64, 28, 28, 5, 5, 2, 2, 1, ""),
    ("wide_many_tiles_per_cta", 128, 64, 56, 56, 3, 3, 1, 40, 1, ""),
]


def _tile(fn, p):
    from feathercnn_b200._lib import fcuda
    geom = (ctypes.c_int * 4)()
    ok = getattr(fcuda(), fn)(ctypes.byref(p), geom)
    return tuple(geom) if ok else None


@pytest.fixture
def wide_switch():
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    names = (b"igemm_wide", b"igemm_presplit", b"igemm_halo")
    saved = [lib.fcuda_get_tuning(n) for n in names], booster.get_precision()
    booster.set_precision(booster.PRECISION_FP32_SPLIT)
    assert lib.fcuda_set_tuning(b"igemm_halo", 1) == 0
    assert lib.fcuda_set_tuning(b"igemm_presplit", 1) == 0

    def setter(v):
        assert lib.fcuda_set_tuning(b"igemm_wide", v) == 0
    yield setter
    for n, v in zip(names, saved[0]):
        lib.fcuda_set_tuning(n, v)
    booster.set_precision(saved[1])


def _params(case):
    name, oc, ic, h, w, kh, kw, pad, n, group, extra = case
    lbrt = pad if isinstance(pad, tuple) else None
    return _param(oc, ic, h, w, kh, kw, 0 if lbrt else pad, group=group, pad_lbrt=lbrt)


@pytest.mark.parametrize("case", PRESPLIT_CASES + WIDE_CASES, ids=[c[0] for c in PRESPLIT_CASES + WIDE_CASES])
def test_wide_is_bit_identical_to_presplit_kernel(cuda, wide_switch, case):
    from feathercnn_b200 import booster
    name, oc, ic, h, w, kh, kw, pad, n, group, extra = case
    p = _params(case)
    t = _tile("fcuda_igemm_wide_tile", p)
    if case in WIDE_CASES:
        assert t is not None, name
        bn = 64 if oc // group <= 64 else 128
        assert t == (28, 16 if bn == 64 else 8, 28 + kh - 1, t[3]) and t[3] % 4 == 0 and t[3] >= t[1] + kw - 1, (name, t)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = cuda.from_numpy(rng.uniform(-1.0, 1.0, (n, ic, h, w)).astype(np.float32)).cuda()
    wt = cuda.from_numpy((rng.standard_normal((oc, ic // group, kh, kw)) * np.sqrt(2.0 / (ic // group * kh * kw))).astype(np.float32)).cuda()
    b = cuda.from_numpy(rng.uniform(-0.1, 0.1, oc).astype(np.float32)).cuda()
    res = None
    if extra.startswith("res"):
        res = cuda.from_numpy(rng.uniform(-1.0, 1.0, (n, oc, p.output_h, p.output_w)).astype(np.float32)).cuda()

    def run():
        out, algo = booster.conv_forward(p, x, wt, b, algo=booster.SGECONV, residual=res, relu_after_add=extra == "res_relu",
                                         pool=extra == "pool")
        cuda.cuda.synchronize()
        return out

    wide_switch(0)
    old = run()
    wide_switch(1)
    new = run()
    assert old.shape == new.shape
    if not cuda.equal(old, new):
        diff = (old != new)
        np.testing.assert_array_equal(new.cpu().numpy(), old.cpu().numpy(),
                                      err_msg=f"{name}: {int(diff.sum())} of {diff.numel()} outputs differ")
    assert float(old.abs().max()) > 0  # the comparison saw real data


def test_wide_geometry():
    from feathercnn_b200 import booster
    saved = booster.get_precision()
    try:
        booster.set_precision(booster.PRECISION_FP32_SPLIT)
        assert _tile("fcuda_igemm_wide_tile", _param(64, 64, 224, 224, 3, 3, 1)) == (28, 16, 30, 24)     # VGG conv1_2
        assert _tile("fcuda_igemm_wide_tile", _param(128, 64, 112, 112, 3, 3, 1)) == (28, 8, 30, 16)     # VGG conv2_1
        assert _tile("fcuda_igemm_wide_tile", _param(128, 128, 112, 112, 3, 3, 1)) == (28, 8, 30, 16)    # VGG conv2_2
        assert _tile("fcuda_igemm_wide_tile", _param(32, 64, 224, 224, 3, 3, 1)) is None                 # N tile 32
        assert _tile("fcuda_igemm_wide_tile", _param(64, 64, 20, 24, 2, 2, 0)) is None                   # 4 taps
        assert _tile("fcuda_igemm_wide_tile", _param(64, 64, 30, 20, 3, 3, 1)) is None                   # pads more
        booster.set_precision(booster.PRECISION_TF32X3)                                                  # no pre-split
        assert _tile("fcuda_igemm_wide_tile", _param(64, 64, 224, 224, 3, 3, 1)) is None
    finally:
        booster.set_precision(saved)


@pytest.mark.parametrize("name, batch", [("vgg16", 64), ("resnet50", 128)])
def test_benchmark_nets_are_byte_identical(cuda, wide_switch, tmp_path, name, batch):
    """What bench.py times (SetFusion + SetCudaGraph, graph replay, benchmark batch): every surviving blob is the same
    bytes with the pre-split and with the wide kernel."""
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.ZOO[name]()
    param, binf = m.save(tmp_path / name)
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i % 4) for i in range(batch)])
    nets = {}
    for v in (0, 1):
        wide_switch(v)
        net = Net(fusion=True, cuda_graph=True)
        net.LoadParam(param)
        net.LoadWeights(binf)
        for _ in range(3):  # eager, capture, replay
            net.Forward(x)
        net.Synchronize()
        nets[v] = net
    names = [b for b in nets[0].BlobNames() if b in m.blobs]
    assert len(names) >= 10
    compared = 0
    for b in names:
        try:
            a = nets[0].Extract(b)
        except Exception:
            continue  # a view that fusion left without storage
        np.testing.assert_array_equal(nets[1].Extract(b), a, err_msg=f"{name} blob {b}")
        compared += 1
    assert compared >= 10, compared
