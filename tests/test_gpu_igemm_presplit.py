"""The pre-split halo kernel (switch igemm_presplit = 1) against the per-tap split of the halo kernel (igemm_presplit = 0).

Both issue the same wgmma sequence on the same bf16 operand bits in the same k order with the same N tile, so every
output must be BIT-identical: per layer on the halo kernel's cases, and on every surviving blob of the benchmark nets
as feather::Net runs them (fusion and CUDA graphs on, benchmark batch)."""
import ctypes
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (name, oc, ic, h, w, kh, kw, pad or pad_lbrt, n, group, extra): extra = "pool" | "res" | "res_relu" | ""
CASES = [
    ("vgg16_conv1_2_pool_b64", 64, 64, 224, 224, 3, 3, 1, 64, 1, "pool"),
    ("vgg16_conv1_2_b8", 64, 64, 224, 224, 3, 3, 1, 8, 1, ""),
    ("vgg16_conv2_1_b64", 128, 64, 112, 112, 3, 3, 1, 64, 1, ""),
    ("vgg16_conv2_2_pool_b64", 128, 128, 112, 112, 3, 3, 1, 64, 1, "pool"),
    ("resnet50_3x3_56_b128", 64, 64, 56, 56, 3, 3, 1, 128, 1, ""),
    ("resnet50_3x3_28_b128", 128, 128, 28, 28, 3, 3, 1, 128, 1, ""),
    ("ragged_oh30_ow20", 40, 64, 30, 20, 3, 3, 1, 2, 1, ""),
    ("pad0", 64, 32, 36, 28, 3, 3, 0, 2, 1, ""),
    ("pad2", 64, 32, 28, 24, 3, 3, 2, 2, 1, ""),
    ("k1x3", 48, 32, 20, 36, 1, 3, (1, 0, 1, 0), 2, 1, ""),
    ("k3x1", 48, 32, 20, 36, 3, 1, (0, 1, 0, 1), 2, 1, ""),
    ("k5x5_pad2", 72, 64, 40, 44, 5, 5, 2, 2, 1, ""),
    ("k2x2_even_taps", 64, 64, 20, 24, 2, 2, 0, 2, 1, ""),
    ("oc31_bn32", 31, 32, 24, 24, 3, 3, 1, 3, 1, ""),
    ("oc33_bn64", 33, 32, 24, 24, 3, 3, 1, 3, 1, ""),
    ("oc100_bn128", 100, 32, 24, 24, 3, 3, 1, 3, 1, ""),
    ("oc257_bn128", 257, 64, 24, 24, 3, 3, 1, 8, 1, ""),
    ("pool_odd_oh27", 64, 64, 27, 28, 3, 3, 1, 3, 1, "pool"),
    ("pool_pad0_oh27", 96, 32, 29, 36, 3, 3, 0, 2, 1, "pool"),
    ("pool_pad2", 64, 32, 21, 20, 3, 3, 2, 2, 1, "pool"),
    ("residual", 64, 64, 28, 28, 3, 3, 1, 3, 1, "res"),
    ("residual_relu", 64, 64, 28, 28, 3, 3, 1, 3, 1, "res_relu"),
    ("grouped_icg32", 128, 64, 20, 20, 3, 3, 1, 2, 2, ""),
    ("batch1", 64, 64, 56, 56, 3, 3, 1, 1, 1, ""),
    ("tiny_fewer_tiles_than_sms", 32, 32, 8, 8, 3, 3, 1, 1, 1, ""),
    ("tile_straddles_edge_oh13_ow20", 64, 96, 13, 20, 3, 3, 1, 3, 1, ""),
]


def _param(oc, ic, h, w, kh, kw, pad, group=1, pad_lbrt=None):
    from feathercnn_b200 import booster
    return booster.ConvParam.make(oc, ic, h, w, kh, kw, stride=1, pad=pad, group=group, relu=True, pad_lbrt=pad_lbrt)


def _presplit_tile(p):
    from feathercnn_b200._lib import fcuda
    geom = (ctypes.c_int * 4)()
    ok = fcuda().fcuda_igemm_presplit_tile(ctypes.byref(p), geom)
    return tuple(geom) if ok else None


@pytest.fixture
def presplit_switch():
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    saved = lib.fcuda_get_tuning(b"igemm_presplit"), lib.fcuda_get_tuning(b"igemm_halo"), booster.get_precision()
    booster.set_precision(booster.PRECISION_FP32_SPLIT)
    assert lib.fcuda_set_tuning(b"igemm_halo", 1) == 0

    def setter(v):
        assert lib.fcuda_set_tuning(b"igemm_presplit", v) == 0
    yield setter
    lib.fcuda_set_tuning(b"igemm_presplit", saved[0])
    lib.fcuda_set_tuning(b"igemm_halo", saved[1])
    booster.set_precision(saved[2])


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_presplit_is_bit_identical_to_halo_kernel(cuda, presplit_switch, case):
    from feathercnn_b200 import booster
    name, oc, ic, h, w, kh, kw, pad, n, group, extra = case
    lbrt = pad if isinstance(pad, tuple) else None
    p = _param(oc, ic, h, w, kh, kw, 0 if lbrt else pad, group=group, pad_lbrt=lbrt)
    t = _presplit_tile(p)
    assert t is not None, name
    r, c, rb, cb = t
    assert r * c == 128 and rb == r + kh - 1 and cb >= c + kw - 1 and cb % 4 == 0, (name, t)
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

    presplit_switch(0)
    old = run()
    presplit_switch(1)
    new = run()
    assert old.shape == new.shape
    if not cuda.equal(old, new):
        diff = (old != new)
        np.testing.assert_array_equal(new.cpu().numpy(), old.cpu().numpy(),
                                      err_msg=f"{name}: {int(diff.sum())} of {diff.numel()} outputs differ")
    assert float(old.abs().max()) > 0  # the comparison saw real data


def test_presplit_geometry_follows_halo_eligibility():
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    saved = booster.get_precision()
    try:
        booster.set_precision(booster.PRECISION_FP32_SPLIT)
        assert _presplit_tile(_param(64, 64, 224, 224, 3, 3, 1)) == (8, 16, 10, 24)
        assert _presplit_tile(_param(64, 3, 224, 224, 3, 3, 1)) is None       # IC = 3: gathering kernel
        assert _presplit_tile(_param(64, 64, 30, 30, 3, 3, 1)) is None        # W % 4 != 0
        geom = (ctypes.c_int * 4)()
        for mode in (booster.PRECISION_TF32X3, booster.PRECISION_TF32):      # the TF32 modes keep the halo kernel
            booster.set_precision(mode)
            p = _param(64, 64, 224, 224, 3, 3, 1)
            assert _presplit_tile(p) is None and lib.fcuda_igemm_halo_tile(ctypes.byref(p), geom) == 1
    finally:
        booster.set_precision(saved)


@pytest.mark.parametrize("name, batch", [("vgg16", 64), ("resnet50", 128)])
def test_benchmark_nets_are_byte_identical(cuda, presplit_switch, tmp_path, name, batch):
    """What bench.py times (SetFusion + SetCudaGraph, graph replay, benchmark batch): every surviving blob is the same
    bytes with the per-tap split and with the pre-split kernel."""
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.ZOO[name]()
    param, binf = m.save(tmp_path / name)
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i % 4) for i in range(batch)])
    nets = {}
    for v in (0, 1):
        presplit_switch(v)
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
