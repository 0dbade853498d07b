"""LRN on the host (no kernel is launched): the loader's parameters, defaults and rejections; the -100 / -200 returns of
fcuda_lrn_forward (every call here fails its checks before a launch); the two references tests/test_gpu_lrn.py holds the
kernels to, on hand-computed cases; the Caffe converter on hand-encoded caffemodels; and modelgen's GoogLeNet and AlexNet
blob shapes.

lrn_restated is the float32 restatement of fcuda.h's documented order up to s (NumPy float32 operations round each product
and sum on its own); lrn_ref is an independent float64 LRN."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

from test_tools import fbytes, ffloat, fint, layer


# ---- the references ------------------------------------------------------------------------------------------------
def lrn_restated(x, region=0, local_size=5, alpha=1.0, beta=0.75, bias=1.0):
    """(s, y64): s = fl(bias + fl(a * ss)) in float32 in the documented order, and y64 = x * s^-beta in float64 from that s."""
    x = np.asarray(x, np.float32)
    n, c, h, w = x.shape
    r = local_size // 2
    sq = x * x
    ss = np.zeros_like(x)
    if region == 0:
        a = np.float32(alpha) / np.float32(local_size)
        for q in range(c):
            for p in range(max(0, q - r), min(c - 1, q + r) + 1):
                ss[:, q] = ss[:, q] + sq[:, p]
    else:
        a = np.float32(alpha) / np.float32(local_size * local_size)
        pad = np.zeros((n, c, h + 2 * r, w + 2 * r), np.float32)
        pad[:, :, r:r + h, r:r + w] = sq
        for di in range(-r, r + 1):
            for dj in range(-r, r + 1):
                ss = ss + pad[:, :, r + di:r + di + h, r + dj:r + dj + w]
    s = np.float32(bias) + a * ss
    assert s.dtype == np.float32
    with np.errstate(divide="ignore", invalid="ignore"):
        y64 = x.astype(np.float64) * np.power(s.astype(np.float64), -float(np.float32(beta)))
    return s, y64


def lrn_ref(x, region=0, local_size=5, alpha=1.0, beta=0.75, bias=1.0):
    """float64 LRN with the fp32 parameters: (y, t, s) with t = a * ss and s = bias + t, a = alpha / n."""
    x = np.asarray(x, np.float64)
    n, c, h, w = x.shape
    r = local_size // 2
    al, be, bi = (float(np.float32(v)) for v in (alpha, beta, bias))
    sq = x * x
    if region == 0:
        pad = np.concatenate([np.zeros((n, r, h, w)), sq, np.zeros((n, r, h, w))], axis=1)
        ss = sum(pad[:, d:d + c] for d in range(local_size))
        t = al / local_size * ss
    else:
        pad = np.pad(sq, ((0, 0), (0, 0), (r, r), (r, r)))
        ss = sum(pad[:, :, di:di + h, dj:dj + w] for di in range(local_size) for dj in range(local_size))
        t = al / (local_size * local_size) * ss
    s = bi + t
    with np.errstate(divide="ignore", invalid="ignore"):
        return x * np.power(s, -be), t, s


def test_references_hand_computed():
    # across, size 3, alpha 3 (a = 1), beta 1, bias 1: s = 1 + ss over channels q-1..q+1
    x = np.array([1.0, 2.0, 3.0], np.float32).reshape(1, 3, 1, 1)
    want_s = np.array([1 + 1 + 4, 1 + 1 + 4 + 9, 1 + 4 + 9])
    y, _, s = lrn_ref(x, 0, 3, 3.0, 1.0, 1.0)
    assert np.allclose(s.ravel(), want_s) and np.allclose(y.ravel(), [1 / 6, 2 / 15, 3 / 14])
    s32, y64 = lrn_restated(x, 0, 3, 3.0, 1.0, 1.0)
    assert np.array_equal(s32.ravel(), want_s.astype(np.float32)) and np.allclose(y64.ravel(), y.ravel())
    # within, size 3 on a 2 x 2 plane (window larger than the plane), alpha 9 (a = 1), beta 0.5, bias 0: every pixel's
    # window covers the whole plane, s = 1 + 4 + 9 + 16 = 30
    x = np.array([1.0, 2.0, 3.0, 4.0], np.float32).reshape(1, 1, 2, 2)
    y, _, s = lrn_ref(x, 1, 3, 9.0, 0.5, 0.0)
    assert np.allclose(s, 30.0) and np.allclose(y, x / np.sqrt(30.0))
    s32, y64 = lrn_restated(x, 1, 3, 9.0, 0.5, 0.0)
    assert np.array_equal(s32, np.full_like(x, 30.0)) and np.allclose(y64, y)
    # local_size 1: each value on its own; the zoo defaults (5, 1e-4, 0.75, 1) barely change a value of order 1
    x = np.random.default_rng(0).uniform(-2, 2, (2, 7, 3, 4)).astype(np.float32)
    y, _, _ = lrn_ref(x, 0, 1, 2.0, 0.75, 1.0)
    assert np.allclose(y, x * (1 + 2 * x.astype(np.float64) ** 2) ** -0.75)
    y, _, _ = lrn_ref(x, 0, 5, 1e-4, 0.75, 1.0)
    assert np.abs(y / x - 1).max() < 1e-3


def test_restatement_adds_in_ascending_order():
    """The float32 restatement rounds after every term: 2^24 + 1 + 1 in ascending order stays 2^24 (each +1 is lost),
    where the exact sum is 2^24 + 2."""
    x = np.array([4096.0, 1.0, 1.0], np.float32).reshape(1, 3, 1, 1)   # squares 2^24, 1, 1
    s32, _ = lrn_restated(x, 0, 5, 5.0, 1.0, 0.0)                      # a = 1, bias 0
    assert s32.ravel()[0] == np.float32(2.0 ** 24)
    _, _, s = lrn_ref(x, 0, 5, 5.0, 1.0, 0.0)
    assert s.ravel()[0] == 2.0 ** 24 + 2


# ---- loader --------------------------------------------------------------------------------------------------------
HEAD = "7767517\n2 2\nInput data 0 1 data 0=8 1=8 2=16\n"


@pytest.mark.parametrize("line", [
    "LRN n 1 1 data out",                                                            # defaults: 0 5 1 0.75 1
    "LRN n 1 1 data out 0=0 1=5 2=1.000000e-04 3=7.500000e-01 4=1.000000e+00",       # BVLC AlexNet / GoogLeNet
    "LRN n 1 1 data out 0=1 1=3 2=5.000000e-05 3=7.500000e-01 4=1.000000e+00",       # CIFAR-10 full, WITHIN_CHANNEL
    "LRN n 1 1 data out 1=1",
    "LRN n 1 1 data out 1=9 4=2.0",                                                  # generic size, k = 2
])
def test_load_param_accepts(line):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(HEAD + line + "\n")
    assert "out" in net.BlobNames()


@pytest.mark.parametrize("line", [
    "LRN n 1 1 data out 0=2",            # region_type outside 0..1
    "LRN n 1 1 data out 0=-1",
    "LRN n 1 1 data out 1=4",            # even local_size
    "LRN n 1 1 data out 0=1 1=2",
    "LRN n 1 1 data out 1=0",            # local_size < 1
    "LRN n 1 1 data out 1=-3",
])
def test_load_param_rejections(line):
    from feathercnn_b200.net import FeatherError, Net
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(HEAD + line + "\n")
    assert e.value.code == -200, line


def test_lrn_is_registered_and_never_fused():
    from feathercnn_b200.net import Net
    text = ("7767517\n4 4\nInput data 0 1 data 0=8 1=8 2=16\nConvolution conv 1 1 data c 0=16 1=3 4=1 5=1 6=2304\n"
            "LRN n 1 1 c m\nReLU relu 1 1 m out\n")
    net = Net(fusion=True)
    net.LoadParamFromText(text)
    net.FuseNow()
    assert net.LayerFusedAway("n") == 0 and net.LayerFusedAway("relu") == 0


# ---- C ABI ---------------------------------------------------------------------------------------------------------
FAKE_OUT, FAKE_IN = ctypes.c_void_p(256), ctypes.c_void_p(512)  # never dereferenced: every call below fails its checks


def _fwd(**kw):
    from feathercnn_b200._lib import fcuda
    a = dict(out=FAKE_OUT, inp=FAKE_IN, C=16, h=8, w=8, region=0, size=5, alpha=1e-4, beta=0.75, bias=1.0, batch=2)
    a.update(kw)
    return fcuda().fcuda_lrn_forward(a["out"], a["inp"], a["C"], a["h"], a["w"], a["region"], a["size"], a["alpha"],
                                     a["beta"], a["bias"], a["batch"], None)


@pytest.mark.parametrize("kw", [dict(out=None), dict(inp=None), dict(C=0), dict(h=0), dict(w=0), dict(batch=0),
                                dict(C=-1), dict(h=-5), dict(batch=-2), dict(out=None, region=3)])
def test_forward_rejects_null_and_empty(kw):
    assert _fwd(**kw) == -100


@pytest.mark.parametrize("kw", [dict(region=2), dict(region=-1), dict(size=0), dict(size=-1), dict(size=4), dict(size=2),
                                dict(region=1, size=6), dict(out=FAKE_IN)])
def test_forward_rejects_parameters(kw):
    assert _fwd(**kw) == -200


# ---- converter -----------------------------------------------------------------------------------------------------
def _net(*layers) -> bytes:
    return (fbytes(1, "lrn") + fbytes(3, "data") + b"".join(fint(4, d) for d in (1, 8, 6, 6)) + b"".join(layers))


def _lrn_layer(name, bottom, top, **fields):
    """lrn_param = 118 with the given fields: local_size 1, alpha 2, beta 3, norm_region 4, k 5."""
    ids = {"local_size": 1, "alpha": 2, "beta": 3, "norm_region": 4, "k": 5}
    p = b"".join(fint(ids[k], v) if k in ("local_size", "norm_region") else ffloat(ids[k], v) for k, v in fields.items())
    return layer(name, "LRN", [bottom], [top], f118=p)


def test_converter_lrn_regions():
    from feathercnn_b200.tools import caffe2feather
    text, blob = caffe2feather.convert(_net(
        _lrn_layer("norm1", "data", "norm1", local_size=5, alpha=1e-4, beta=0.75),            # AlexNet's
        _lrn_layer("norm2", "norm1", "norm2"),                                                # every default
        _lrn_layer("norm3", "norm2", "norm3", local_size=3, alpha=5e-5, beta=0.75, norm_region=1, k=2.0),
        _lrn_layer("norm4", "norm3", "norm3", local_size=7, alpha=0.5, beta=0.5, k=2.5)))   # in place, k honoured
    f = lambda v: f"{np.float32(v):.8e}"  # noqa: E731
    assert text.splitlines()[3:] == [
        f"LRN norm1 1 1 data norm1 0=0 1=5 2={f(1e-4)} 3={f(0.75)} 4={f(1.0)}",
        f"LRN norm2 1 1 norm1 norm2 0=0 1=5 2={f(1.0)} 3={f(0.75)} 4={f(1.0)}",
        f"LRN norm3 1 1 norm2 norm3 0=1 1=3 2={f(5e-5)} 3={f(0.75)} 4={f(1.0)}",   # WITHIN_CHANNEL: k ignored, 4=1
        f"LRN norm4 1 1 norm3 norm3_norm4 0=0 1=7 2={f(0.5)} 3={f(0.5)} 4={f(2.5)}",
    ]
    assert blob == b""
    # the alpha written reads back as the same fp32
    assert np.float32(float(text.splitlines()[3].split()[8][2:])) == np.float32(1e-4)
    from feathercnn_b200.net import Net
    Net().LoadParamFromText(text)


@pytest.mark.parametrize("size", [2, 4, 0])
def test_converter_rejects_even_local_size(size):
    from feathercnn_b200.tools import caffe2feather
    with pytest.raises(ValueError, match="even"):
        caffe2feather.convert(_net(_lrn_layer("norm1", "data", "norm1", local_size=size)))


# ---- models --------------------------------------------------------------------------------------------------------
def test_googlenet_shapes():
    from feathercnn_b200.tools import modelgen
    m = modelgen.googlenet()
    assert m.shape["conv1/relu_7x7"] == (64, 112, 112) and m.shape["pool1/3x3_s2"] == (64, 56, 56)
    assert m.shape["pool1/norm1"] == (64, 56, 56) and m.shape["conv2/norm2"] == (192, 56, 56)
    assert m.shape["pool2/3x3_s2"] == (192, 28, 28)
    outs = {t: m.shape[f"inception_{t}/output"] for t, *_ in modelgen.GOOGLENET_INCEPTIONS}
    assert outs == {"3a": (256, 28, 28), "3b": (480, 28, 28), "4a": (512, 14, 14), "4b": (512, 14, 14),
                    "4c": (512, 14, 14), "4d": (528, 14, 14), "4e": (832, 14, 14), "5a": (832, 7, 7),
                    "5b": (1024, 7, 7)}
    assert m.shape["pool3/3x3_s2"] == (480, 14, 14) and m.shape["pool4/3x3_s2"] == (832, 7, 7)
    assert m.shape["pool5/7x7_s1"] == (1024, 1, 1) and m.shape["prob"] == (1000, 1, 1)
    fc = [L for L in m.lines if L.startswith("InnerProduct ")]
    assert fc == ["InnerProduct loss3/classifier 1 1 pool5/drop_7x7_s1 loss3/classifier 0=1000 1=1 2=1024000"]
    types = [L.split()[0] for L in m.lines]
    assert types.count("LRN") == 2 and types.count("Split") == 9 and types.count("Concat") == 9
    assert all(L.split()[3] == "4" for L in m.lines if L.startswith("Split "))
    assert all(L.split()[2] == "4" for L in m.lines if L.startswith("Concat "))
    assert "LRN pool1/norm1 1 1 pool1/3x3_s2 pool1/norm1 0=0 1=5 2=1.000000e-04 3=7.500000e-01 4=1.000000e+00" in m.lines
    # the convolution shapes this net brings: 5x5 on 16, 24, 32 and 48 channels, 1x1 on 528 and 832, a 7x7 / 2 stem
    five = sorted({m.shape[L.split()[4]][0] for L in m.lines if L.startswith("Convolution ") and "/5x5 " in L})
    assert five == [16, 24, 32, 48]
    assert "Convolution conv1/7x7_s2 1 1 data conv1/7x7_s2 0=64 1=7 3=2 4=3 5=1 6=9408" in m.lines
    m2 = modelgen.googlenet(lrn_alpha=0.9)
    assert [L for L in m2.lines if L.startswith("LRN ")][0].split()[8] == "2=9.000000e-01"
    assert bytes(m2.bin) == bytes(m.bin)  # lrn_alpha changes the LRN lines only


def test_alexnet_shapes():
    from feathercnn_b200.tools import modelgen
    m = modelgen.alexnet()
    want = {"relu1": (96, 55, 55), "norm1": (96, 55, 55), "pool1": (96, 27, 27), "relu2": (256, 27, 27),
            "norm2": (256, 27, 27), "pool2": (256, 13, 13), "relu3": (384, 13, 13), "relu4": (384, 13, 13),
            "relu5": (256, 13, 13), "pool5": (256, 6, 6), "fc6": (4096, 1, 1), "fc8": (1000, 1, 1), "prob": (1000, 1, 1)}
    assert {k: m.shape[k] for k in want} == want
    assert "InnerProduct fc6 1 1 pool5 fc6 0=4096 1=1 2=37748736" in m.lines   # 9216 inputs
    grouped = [L.split()[1] for L in m.lines if L.startswith("ConvolutionDepthWise ") and " 7=2" in L]
    assert grouped == ["conv2", "conv4", "conv5"]
    assert [L.split()[1] for L in m.lines if L.startswith("LRN ")] == ["norm1", "norm2"]
    from feathercnn_b200.net import Net
    for mw in (m, modelgen.googlenet()):
        net = Net(fusion=True)
        net.LoadParamFromText("7767517\n" + f"{len(mw.lines)} {len(mw.blobs)}\n" + "\n".join(mw.lines) + "\n")
        net.FuseNow()
        assert all(net.LayerFusedAway(L.split()[1]) == 0 for L in mw.lines if L.startswith("LRN "))
