"""GPU parity of the dense / pooling / element-wise layers (SURVEY.md §8 rows a12-a15) and of the raw
TensorGEMM (row a8) through the C ABI, against the oracle restatement."""
import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu


def _t(cuda, a):
    return cuda.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


@pytest.mark.parametrize("shape", [(1, 128, 64, 32), (2, 300, 72, 100), (64, 100, 64, 64), (16, 1000, 24, 36)])
@pytest.mark.parametrize("x3", [True, False])
def test_tensor_gemm(cuda, shape, x3):
    """a8: for each tile element g, M_g = V_g U_g^T  (avx/winograd_kernels_F63.cpp:518-757)."""
    from feathercnn_b200 import booster
    g, m, n, k = shape
    rng = np.random.default_rng(0)
    a = rng.uniform(-1, 1, (g, m, k)).astype(np.float32)
    b = rng.uniform(-1, 1, (g, n, k)).astype(np.float32)
    got = booster.tensor_gemm(_t(cuda, a), _t(cuda, b), x3=x3).cpu().numpy()
    want = np.einsum("gmk,gnk->gmn", a.astype(np.float64), b.astype(np.float64))
    assert rel_err(got, want) < (1e-5 if x3 else 1e-3)


@pytest.mark.parametrize("in_size,out_size,batch", [(512, 256, 1), (25088, 128, 4), (1000, 10, 3), (2048, 1000, 64),
                                                    (30, 7, 2)])
@pytest.mark.parametrize("relu", [False, True])
def test_inner_product(cuda, restatement, in_size, out_size, batch, relu):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(1)
    x = rng.uniform(-0.5, 0.5, (batch, in_size)).astype(np.float32)
    w = (rng.standard_normal((out_size, in_size)) * np.sqrt(2.0 / in_size)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, out_size).astype(np.float32)
    got = booster.inner_product(_t(cuda, x), _t(cuda, w), _t(cuda, b), relu).cpu().numpy()
    for n in range(batch):
        want = restatement.inner_product(x[n], w, b, relu)
        assert rel_err(got[n], want) < 1e-4


POOL_CASES = [
    # type, k, s, pad(l, r, t, b), global, (c, h, w)
    (0, 2, 2, (0, 0, 0, 0), False, (8, 28, 28)),      # VGG max 2x2 s2
    (0, 3, 2, (0, 0, 0, 0), False, (16, 112, 112)),   # ResNet pool1: ceil mode -> 56
    (0, 3, 2, (0, 0, 0, 0), False, (4, 13, 17)),      # ragged windows at the border
    (1, 3, 1, (0, 0, 0, 0), False, (4, 9, 9)),
    (1, 7, 1, (0, 0, 0, 0), True, (64, 7, 7)),        # global average
    (0, 7, 1, (0, 0, 0, 0), True, (5, 6, 9)),         # global max
    (0, 3, 2, (1, 1, 1, 1), False, (4, 16, 16)),      # padded: window start subtracts both pads (pooling_layer.h:56,67)
    (1, 3, 2, (1, 0, 1, 0), False, (3, 15, 15)),
    (1, 2, 2, (0, 0, 0, 0), False, (8, 28, 28)),      # average through the 2x2 fast path
    (0, 2, 2, (0, 0, 0, 0), False, (3, 10, 4)),       # fast path, one output pair per row
    (0, 2, 2, (0, 0, 0, 0), False, (3, 10, 14)),      # W % 4 != 0 -> generic kernel
    (0, 2, 2, (0, 0, 0, 0), False, (4, 9, 12)),       # odd H (ceil mode) -> generic kernel
    (1, 3, 2, (0, 0, 0, 0), False, (8, 57, 64)),      # 3x3 s2 strip kernel, average, several strips
    (0, 3, 2, (0, 0, 0, 0), False, (4, 50, 50)),      # 3x3 s2 strip kernel, last window clipped in x and y (ceil mode)
    (1, 3, 2, (0, 0, 0, 0), False, (4, 50, 50)),      # same, average divides by the in-bounds count (pooling_layer.h:84)
    (0, 3, 2, (0, 0, 0, 0), False, (3, 20, 46)),      # OW = 23: one below the strip kernel's dispatch boundary
    (1, 3, 2, (0, 0, 0, 0), False, (3, 20, 46)),
    (0, 3, 2, (0, 0, 0, 0), False, (3, 20, 48)),      # OW = 24: the smallest strip-kernel output
    (1, 3, 2, (0, 0, 0, 0), False, (3, 20, 48)),
    (1, 3, 2, (0, 0, 0, 0), False, (3, 21, 47)),      # odd H and W: generic kernel, windows end on the last row / column
    (0, 3, 2, (0, 0, 0, 0), False, (3, 34, 64)),      # strip kernel, last row and column clipped in both axes
    (1, 3, 2, (0, 0, 0, 0), False, (3, 34, 64)),
    (1, 2, 2, (0, 0, 0, 0), False, (3, 10, 4)),       # 2x2 fast path, average, one output pair per row
    (0, 2, 2, (0, 0, 0, 0), False, (2, 6, 256)),      # 2x2 fast path, 64 output pairs per row
    (1, 2, 2, (0, 0, 0, 0), False, (2, 6, 256)),
]


@pytest.mark.parametrize("case", POOL_CASES)
def test_pooling(cuda, restatement, case):
    from feathercnn_b200 import booster
    type_, k, s, (pl, pr, pt, pb), glob, (c, h, w) = case
    rng = np.random.default_rng(2)
    x = rng.uniform(-1, 1, (2, c, h, w)).astype(np.float32)
    got = booster.pooling(_t(cuda, x), type_, k, k, s, s, pl, pr, pt, pb, glob).cpu().numpy()
    for n in range(2):
        want = restatement.pooling(x[n], type_, k, k, s, s, pl, pr, pt, pb, glob)
        assert got[n].shape == want.shape
        np.testing.assert_allclose(got[n], want, rtol=1e-6, atol=1e-6)


def test_batchnorm_scale_eltwise_relu_softmax_dropout(cuda, restatement):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(3)
    n, c, h, w = 3, 37, 9, 11
    x = rng.uniform(-2, 2, (n, c, h, w)).astype(np.float32)
    slope, mean = rng.uniform(0.9, 1.1, c).astype(np.float32), rng.uniform(-0.1, 0.1, c).astype(np.float32)
    var, bias = rng.uniform(0.5, 1.5, c).astype(np.float32), rng.uniform(-0.1, 0.1, c).astype(np.float32)
    eps = 1e-5
    sqrt_var = np.sqrt(var + np.float32(eps)).astype(np.float32)
    alpha = (bias - slope * mean / sqrt_var).astype(np.float32)   # batchnorm_layer.h:70-75
    beta = (slope / sqrt_var).astype(np.float32)
    sc, sb = rng.uniform(0.9, 1.1, c).astype(np.float32), rng.uniform(-0.1, 0.1, c).astype(np.float32)
    xd = _t(cuda, x)
    bn = booster.batchnorm(xd, _t(cuda, alpha), _t(cuda, beta)).cpu().numpy()
    scl = booster.scale(xd, _t(cuda, sc), _t(cuda, sb)).cpu().numpy()
    scl_nb = booster.scale(xd, _t(cuda, sc), None).cpu().numpy()
    fused = booster.batchnorm(xd, _t(cuda, alpha), _t(cuda, beta), _t(cuda, sc), _t(cuda, sb), relu=True).cpu().numpy()
    add = booster.eltwise_add(xd, _t(cuda, x[::-1].copy()), relu=True).cpu().numpy()
    rl = booster.relu(xd).cpu().numpy()
    sm = booster.softmax(xd).cpu().numpy()
    dr = booster.dropout(xd, 0.5).cpu().numpy()
    for i in range(n):
        want_bn = restatement.batchnorm(x[i], slope, mean, var, bias, eps)
        np.testing.assert_allclose(bn[i], want_bn, rtol=2e-6, atol=2e-6)
        np.testing.assert_allclose(scl[i], restatement.scale(x[i], sc, sb), rtol=2e-6, atol=2e-6)
        np.testing.assert_allclose(scl_nb[i], restatement.scale(x[i], sc, None), rtol=2e-6, atol=2e-6)
        want_fused = restatement.relu(restatement.scale(want_bn, sc, sb))
        np.testing.assert_allclose(fused[i], want_fused, rtol=4e-6, atol=4e-6)
        np.testing.assert_array_equal(add[i], restatement.eltwise_add(x[i], x[n - 1 - i], relu=True))
        np.testing.assert_array_equal(rl[i], restatement.relu(x[i]))
        assert rel_err(sm[i], restatement.softmax(x[i])) < 1e-5
        assert abs(float(sm[i].sum()) - 1.0) < 1e-4
        np.testing.assert_array_equal(dr[i], restatement.dropout(x[i], 0.5))


def test_softmax_large_and_relu_unaligned(cuda, restatement):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(4)
    x = (rng.standard_normal((2, 1000, 1, 1)) * 5).astype(np.float32)
    sm = booster.softmax(_t(cuda, x)).cpu().numpy()
    for i in range(2):
        assert rel_err(sm[i], restatement.softmax(x[i])) < 1e-5
    y = rng.standard_normal(1003).astype(np.float32)  # odd length: scalar tail path
    yd = _t(cuda, y)
    np.testing.assert_array_equal(booster.relu(yd).cpu().numpy(), np.maximum(y, 0))
    np.testing.assert_array_equal(booster.relu(yd[1:].clone()).cpu().numpy(), np.maximum(y[1:], 0))


def test_from_pixels_resize_mean_normalize(cuda, oracle):
    """fcuda_from_pixels: every ncnn pixel type, with and without the fixed-point bilinear resize, bit-exact against the
    reference's from_pixels[_resize] (or its pinned NumPy restatement when oracle/_ref is absent); mean / norm variants of
    Mat::substract_mean_normalize (mat.cpp:30-107) to fp32 rounding."""
    from feathercnn_b200 import booster
    from test_oracle import PIXEL_TYPES
    ref = oracle.Reference() if oracle.reference_available() else None
    rng = np.random.default_rng(1)
    for (h, w, tw, th) in [(32, 48, 0, 0), (37, 53, 224, 224), (240, 320, 224, 224), (17, 9, 40, 31), (2, 2, 5, 7)]:
        for t, c in PIXEL_TYPES:
            imgs = rng.integers(0, 256, (3, h, w, c), dtype=np.uint8)
            got = booster.from_pixels(cuda.from_numpy(imgs).cuda(), t, tw, th).cpu().numpy()
            for n in range(3):
                want = ref.from_pixels(imgs[n], t, tw, th) if ref else oracle.from_pixels(imgs[n], t, tw, th)
                np.testing.assert_array_equal(got[n], want, err_msg=f"type {t:#x} {w}x{h}->{tw}x{th} image {n}")
    imgs = rng.integers(0, 256, (2, 60, 80, 3), dtype=np.uint8)
    mean, norm = [104.0, 117.0, 123.0], [0.017, 0.0175, 0.0171]
    for m, s in ((mean, None), (None, norm), (mean, norm)):
        got = booster.from_pixels(cuda.from_numpy(imgs).cuda(), 1 | (2 << 16), 32, 24, mean=m, norm=s).cpu().numpy()
        for n in range(2):
            want = oracle.from_pixels(imgs[n], 1 | (2 << 16), 32, 24, mean=m, norm=s)
            np.testing.assert_allclose(got[n], want, rtol=2e-6, atol=1e-6)
    with pytest.raises(booster.FcudaError) as e:
        booster.from_pixels(cuda.from_numpy(imgs).cuda(), 3)
    assert e.value.code == -200


def test_net_feed_input_pixels(cuda, oracle, model_dir):
    """Net::FeedInputPixels == from_pixels_resize + substract_mean_normalize + FeedInput, then Forward, against the
    reference chain on the CPU."""
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.mini()
    param, binf = m.save(model_dir / "mini_px")
    c, h, w = m.shape["data"]
    rng = np.random.default_rng(2)
    n_src_c = 4 if c == 3 else c
    if c not in (1, 3, 4):
        pytest.skip("mini net input is not an image")
    t = {1: 4, 3: 8 | (2 << 16), 4: 8}[c]   # GRAY, RGBA->BGR, RGBA
    imgs = rng.integers(0, 256, (2, 50, 70, {1: 1, 3: 4, 4: 4}[c]), dtype=np.uint8)
    mean, norm = [120.0] * c, [1.0 / 128] * c
    net = Net()
    net.LoadParam(param)
    net.LoadWeights(binf)
    net.FeedInputPixels(imgs, t, w, h, mean, norm)
    net.Forward()
    got = net.Extract("prob")
    cpu = oracle.ReferenceNet(param, binf) if oracle.reference_available() else oracle.OracleNet(param, binf)
    for n in range(2):
        x = oracle.from_pixels(imgs[n], t, w, h, mean=mean, norm=norm)
        cpu.forward(x)
        want = cpu.extract("prob")
        assert np.abs(got[n].reshape(want.shape) - want).max() / np.abs(want).max() < 2e-4
