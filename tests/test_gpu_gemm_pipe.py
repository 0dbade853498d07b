"""The persistent, pipelined TensorGEMM (switch gemm_pipe = 1) against the one-tile-per-CTA kernel (gemm_pipe = 0).

Both run the same tiles, the same k-blocks in the same order and the same wgmma sequence per accumulator, with the same
epilogue, so every output must be BIT-identical: Winograd F(6,3) / F(2,3) (batched, row-major), im2col (NCHW + bias +
ReLU, a chunk ending inside an image), InnerProduct (k-split partial planes) and the raw TensorGEMM."""
import zlib

import numpy as np
import pytest
import torch

MODES = ["fp32split", "tf32x3", "tf32"]
NAIVE, IM2COL, SGECONV, DEPTHWISE, WINOGRADF63, WINOGRADF63FUSED, WINOGRADF23 = range(7)


def _set_mode(mode):
    from feathercnn_b200 import booster
    booster.set_precision({"fp32split": booster.PRECISION_FP32_SPLIT, "tf32x3": booster.PRECISION_TF32X3,
                           "tf32": booster.PRECISION_TF32}[mode])


@pytest.fixture
def pipe_switch():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    saved = lib.fcuda_get_tuning(b"gemm_pipe")

    def setter(v):
        assert lib.fcuda_set_tuning(b"gemm_pipe", v) == 0
    yield setter
    lib.fcuda_set_tuning(b"gemm_pipe", saved)


def _same(name, old, new):
    assert old.shape == new.shape, name
    if not torch.equal(old, new):
        diff = old != new
        np.testing.assert_array_equal(new.cpu().numpy(), old.cpu().numpy(),
                                      err_msg=f"{name}: {int(diff.sum())} of {diff.numel()} outputs differ")
    assert float(old.abs().max()) > 0  # the comparison saw real data


def _both(pipe_switch, run):
    pipe_switch(0)
    old = run()
    torch.cuda.synchronize()
    pipe_switch(1)
    new = run()
    torch.cuda.synchronize()
    return old, new


# ------------------------------------------------------------------------------------------------- convolutions
# (name, oc, ic, h, w, batch, algo): every distinct layer of VGG-16 (b64) and ResNet-50 (b128) the tuned policy sends to
# Winograd F(6,3) (a 64-way batched TensorGEMM), and an F(2,3) layer (16-way)
WINO = [
    ("vgg16_conv3_1_b64", 256, 128, 56, 56, 64, WINOGRADF63),
    ("vgg16_conv3_2_b64", 256, 256, 56, 56, 64, WINOGRADF63),
    ("vgg16_conv4_1_b64", 512, 256, 28, 28, 64, WINOGRADF63),
    ("vgg16_conv4_2_b64", 512, 512, 28, 28, 64, WINOGRADF63),
    ("vgg16_conv5_1_b64", 512, 512, 14, 14, 64, WINOGRADF63),
    ("resnet50_3x3_14_b128", 256, 256, 14, 14, 128, WINOGRADF63),
    ("f23_oc40_ic48", 40, 48, 26, 22, 3, WINOGRADF23),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", WINO, ids=[c[0] for c in WINO])
def test_winograd_gemm_pipe_is_bit_identical(cuda, pipe_switch, mode, case):
    from feathercnn_b200 import booster
    name, oc, ic, h, w, n, algo = case
    _set_mode(mode)
    p = booster.ConvParam.make(oc, ic, h, w, 3, pad=1, relu=True)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = torch.from_numpy(rng.uniform(-1.0, 1.0, (n, ic, h, w)).astype(np.float32)).cuda()
    wt = torch.from_numpy((rng.standard_normal((oc, ic, 3, 3)) * np.sqrt(2.0 / (ic * 9))).astype(np.float32)).cuda()
    b = torch.from_numpy(rng.uniform(-0.1, 0.1, oc).astype(np.float32)).cuda()

    def run():
        out, got = booster.conv_forward(p, x, wt, b, algo=algo)
        assert got == algo
        return out
    _same(f"{name} {mode}", *_both(pipe_switch, run))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_im2col_gemm_pipe_is_bit_identical(cuda, pipe_switch, mode):
    """NCHW epilogue with bias and ReLU; the L2 chunk (a multiple of 128 pixels) ends inside an image (m_offset)."""
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    _set_mode(mode)
    oc, ic, h, w, n = 72, 16, 20, 21, 3
    p = booster.ConvParam.make(oc, ic, h, w, 3, pad=1, relu=True)
    rng = np.random.default_rng(7)
    x = torch.from_numpy(rng.uniform(-1.0, 1.0, (n, ic, h, w)).astype(np.float32)).cuda()
    wt = torch.from_numpy(rng.standard_normal((oc, ic, 3, 3)).astype(np.float32) * 0.1).cuda()
    b = torch.from_numpy(rng.uniform(-0.5, 0.5, oc).astype(np.float32)).cuda()
    saved = fcuda().fcuda_get_l2_chunk_bytes()
    booster.set_l2_chunk_bytes(128 * 144 * 4)
    try:
        old, new = _both(pipe_switch, lambda: booster.conv_forward(p, x, wt, b, algo=IM2COL)[0])
    finally:
        booster.set_l2_chunk_bytes(saved)
    _same(f"im2col {mode}", old, new)
    assert float((old == 0).float().mean()) > 0.05  # the ReLU clipped something


# ------------------------------------------------------------------------------------------------- InnerProduct
# (in, out, batch): VGG-16's classifier, ResNet-50's, and K % 32 = 4 with a last k-split that owns fewer k-blocks
IP = [
    (25088, 4096, 64),   # 784 k-blocks in 9 splits of 88; the last owns 80
    (4096, 4096, 64),
    (4096, 1000, 1),
    (4096, 1000, 256),   # two N tiles of the partial-plane epilogue
    (2048, 1000, 128),
    (1316, 200, 129),    # 42 k-blocks in 5 splits of 9; the last owns 6
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("in_size,out_size,batch", IP)
def test_inner_product_gemm_pipe_is_bit_identical(cuda, pipe_switch, mode, in_size, out_size, batch):
    from feathercnn_b200 import booster
    _set_mode(mode)
    gen = torch.Generator(device="cuda").manual_seed(in_size * 7 + out_size * 13 + batch)
    x = torch.rand((batch, in_size), generator=gen, device="cuda") * 2 - 1
    w = torch.randn((out_size, in_size), generator=gen, device="cuda") * (2.0 / in_size) ** 0.5
    b = torch.rand(out_size, generator=gen, device="cuda") - 0.5
    old, new = _both(pipe_switch, lambda: booster.inner_product(x, w, b, relu=True))
    _same(f"ip {in_size}x{out_size} b{batch} {mode}", old, new)


# ------------------------------------------------------------------------------------------------- raw TensorGEMM
# (g, m, n, k): K % 32 in {4, 12, 28}, K = 32 / 64 (fewer k-blocks than ring stages), odd k-block counts, M 127-129,
# N 32-300 (BN 32 / 64 / 128 and tails), G up to 64, a single tile, and >= 3 tiles per CTA
RAW = [
    (1, 128, 32, 32),
    (1, 64, 16, 64),
    (3, 127, 64, 36),
    (2, 129, 300, 44),
    (4, 128, 33, 60),
    (64, 129, 100, 96),
    (64, 36, 256, 160),
    (7, 127, 65, 1000),
    (64, 1024, 256, 128),  # 1024 tiles: several per persistent CTA
]


@pytest.mark.gpu
@pytest.mark.parametrize("x3", [True, False], ids=["3xtf32", "tf32"])
@pytest.mark.parametrize("g,m,n,k", RAW)
def test_raw_tensor_gemm_pipe_is_bit_identical(cuda, pipe_switch, x3, g, m, n, k):
    from feathercnn_b200 import booster
    gen = torch.Generator(device="cuda").manual_seed(g * 1000003 + m * 1009 + n * 31 + k)
    a = torch.rand((g, m, k), generator=gen, device="cuda") * 2 - 1
    b = torch.randn((g, n, k), generator=gen, device="cuda")
    old, new = _both(pipe_switch, lambda: booster.tensor_gemm(a, b, x3=x3))
    _same(f"gemm g{g} m{m} n{n} k{k} x3={x3}", old, new)
    if g * ((m + 127) // 128) * ((n + 127) // 128) >= 3 * torch.cuda.get_device_properties(0).multi_processor_count:
        again = booster.tensor_gemm(a, b, x3=x3)  # the static tile walk gives the same result on every run
        torch.cuda.synchronize()
        assert torch.equal(again, new)
    ref = torch.einsum("gmk,gnk->gmn", a.double(), b.double())
    rel = float((new.double() - ref).abs().max() / ref.abs().max())
    assert rel < (1e-5 if x3 else 5e-3), rel
