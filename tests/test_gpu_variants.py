"""Every kernel variant behind fcuda_set_tuning computes the same convolution (the vectorised depthwise kernel must be
BIT-identical to the plain one), and the implicit-GEMM / TensorGEMM arithmetic modes agree with the CUDA-core direct
convolution and with each other."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture
def tuning():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    names = ["dw_vec"]
    saved = {n: lib.fcuda_get_tuning(n.encode()) for n in names}

    def setter(**kw):
        for k, v in kw.items():
            assert lib.fcuda_set_tuning(k.encode(), v) == 0, (k, v)
    yield setter
    for n, v in saved.items():
        lib.fcuda_set_tuning(n.encode(), v)


def _conv(cuda, booster, geom, algo, seed=0, group=1):
    oc, ic, h, w, k, stride, pad, n = geom
    rng = np.random.default_rng(seed)
    x = cuda.from_numpy(rng.uniform(-0.5, 0.5, (n, ic, h, w)).astype(np.float32)).cuda()
    wt = cuda.from_numpy((rng.standard_normal((oc, ic // group, k, k)) * np.sqrt(2.0 / (ic // group * k * k))).astype(np.float32)).cuda()
    b = cuda.from_numpy(rng.uniform(-0.1, 0.1, oc).astype(np.float32)).cuda()
    p = booster.ConvParam.make(oc, ic, h, w, k, stride=stride, pad=pad, relu=True, group=group)
    out, _ = booster.conv_forward(p, x, wt, b, algo=algo)
    cuda.cuda.synchronize()
    return out.cpu().numpy()


IGEMM_GEOMS = [(64, 64, 96, 96, 3, 1, 1, 3), (128, 64, 56, 56, 3, 1, 1, 4), (256, 64, 28, 28, 1, 1, 0, 8),
               (64, 256, 28, 28, 1, 1, 0, 8), (128, 96, 29, 31, 3, 2, 1, 3), (64, 3, 64, 64, 3, 1, 1, 2),
               (96, 128, 14, 14, 1, 1, 0, 5),     # pointwise, 196-pixel images: boxes end inside a tile, tiles straddle images
               (512, 2048, 7, 7, 1, 1, 0, 3),     # 49-pixel images (H*W % 4 != 0): the pointwise slab does not apply
               (40, 32, 10, 6, 1, 1, 0, 1)]       # one partial tile (60 pixels): two of the four boxes are out of range


@pytest.mark.parametrize("geom", IGEMM_GEOMS)
def test_implicit_gemm_variants_are_bit_identical(cuda, geom):
    """3xTF32 implicit GEMM: within 2e-4 of the CUDA-core direct convolution and bit-identical from run to run."""
    from feathercnn_b200 import booster
    booster.set_precision(booster.PRECISION_TF32X3)
    base = _conv(cuda, booster, geom, booster.SGECONV)
    naive = _conv(cuda, booster, geom, booster.NAIVE)
    assert np.abs(base - naive).max() / np.abs(naive).max() < 2e-4
    np.testing.assert_array_equal(_conv(cuda, booster, geom, booster.SGECONV), base)


@pytest.mark.parametrize("geom", IGEMM_GEOMS)
def test_bf16x3_implicit_gemm_variants(cuda, geom):
    """The default split mode (BF16x3 operands in the implicit GEMM): within 5e-5 of the 3xTF32 result (dropped terms
    <= 3 * 2^-16 per product, random sign) and bit-identical from run to run."""
    from feathercnn_b200 import booster
    booster.set_precision(booster.PRECISION_TF32X3)
    ref = _conv(cuda, booster, geom, booster.SGECONV)
    booster.set_precision(booster.PRECISION_FP32_SPLIT)
    base = _conv(cuda, booster, geom, booster.SGECONV)
    assert np.abs(base - ref).max() / np.abs(ref).max() < 5e-5
    np.testing.assert_array_equal(_conv(cuda, booster, geom, booster.SGECONV), base)   # run to run


@pytest.mark.parametrize("geom", [(64, 64, 56, 56, 3, 1, 1, 4), (256, 128, 28, 28, 3, 1, 1, 8), (512, 256, 14, 14, 3, 1, 1, 16)])
def test_winograd_tensor_gemm_matches_direct_conv(cuda, geom):
    """Winograd F(6,3) through the 3xTF32 TensorGEMM: within 2e-4 of the direct convolution and bit-identical from run
    to run."""
    from feathercnn_b200 import booster
    booster.set_precision(booster.PRECISION_TF32X3)
    base = _conv(cuda, booster, geom, booster.WINOGRADF63)
    naive = _conv(cuda, booster, geom, booster.NAIVE)
    assert np.abs(base - naive).max() / np.abs(naive).max() < 2e-4
    np.testing.assert_array_equal(_conv(cuda, booster, geom, booster.WINOGRADF63), base)   # run to run


@pytest.mark.parametrize("geom", [(32, 32, 112, 112, 3, 1, 1, 3), (64, 64, 112, 112, 3, 2, 1, 3), (128, 128, 56, 56, 3, 1, 1, 2),
                                  (128, 128, 56, 56, 3, 2, 1, 2), (512, 512, 14, 14, 3, 1, 1, 2), (1024, 1024, 7, 7, 3, 1, 1, 3)])
def test_vectorised_depthwise_is_bit_identical(cuda, tuning, geom):
    from feathercnn_b200 import booster
    tuning(dw_vec=0)
    base = _conv(cuda, booster, geom, booster.DEPTHWISE, group=geom[1])
    tuning(dw_vec=1)
    np.testing.assert_array_equal(_conv(cuda, booster, geom, booster.DEPTHWISE, group=geom[1]), base)
