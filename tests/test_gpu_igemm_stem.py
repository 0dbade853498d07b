"""The persistent stem kernel (switch igemm_stem = 1) against the gathering kernel (igemm_stem = 0).

Both gather the same operand values in the same k order (k = tap * IC + ic), split them the same way and issue the same
wgmma sequence (p2*q1, p1*q2, p1*q1 per k-step) against the same filter planes, and apply the same fp32 epilogue; only
the tiling over the CTAs and the way the outputs reach global memory differ.  So every output must be BIT-identical, and
both must lie inside the BF16x3 per-element bound against float64."""
import ctypes
import dataclasses

import numpy as np
import pytest
import torch

from test_gpu_error_bounds import FP32_SPLIT, SGECONV, TF32, TF32X3, U, Conv, conv_ref, eps_for, excess, make_data

pytestmark = pytest.mark.gpu

CASES = [
    Conv("vgg16_conv1_1_b64", 64, 3, 224, 224, 3, pad=1, relu=True, batch=64),
    Conv("resnet50_conv1_7x7s2_b128", 64, 3, 224, 224, 7, sh=2, pad=3, relu=True, batch=128),
    Conv("mobilenet_v1_conv1_s2_oc32_b256", 32, 3, 224, 224, 3, sh=2, pad=1, relu=True, batch=256),
    Conv("pointwise_16_to_96_clip", 96, 16, 56, 56, 1, pad=0, clip=(0.0, 6.0), batch=4),
    Conv("ic1_oc32", 32, 1, 40, 36, 3, pad=1, relu=True, batch=3),
    Conv("ic4_5x5_four_kblocks", 48, 4, 30, 30, 5, pad=2, relu=True, batch=3),
    Conv("no_activation", 64, 3, 48, 40, 3, pad=1, batch=3),
    Conv("no_bias", 64, 3, 48, 40, 3, pad=1, relu=True, bias=False, batch=3),
    Conv("clip", 64, 3, 48, 40, 3, pad=1, clip=(-0.25, 0.5), batch=3),
    Conv("ohow400_partial_tiles", 40, 3, 20, 20, 3, pad=1, relu=True, batch=5),
    Conv("ohow225_scalar_stores", 64, 3, 15, 15, 3, pad=1, relu=True, batch=5),
    Conv("k256_oc128_one_staging_buffer", 128, 16, 24, 24, 4, pad=(1, 2, 2, 1), relu=True, batch=3),
    Conv("oc20_bn32", 20, 3, 33, 31, 3, sh=2, pad=1, relu=True, batch=4),
    Conv("batch1", 64, 3, 224, 224, 3, pad=1, relu=True, batch=1),
    # every group writes a channel slice of the output (and reads one of the input): out_img_c > OC
    Conv("channel_slices_aligned", 128, 6, 32, 32, 3, pad=1, group=2, relu=True, batch=3),
    Conv("channel_slices_unaligned", 128, 6, 17, 17, 3, pad=1, group=2, relu=True, batch=3),
]


def _param(c: Conv):
    from feathercnn_b200 import booster
    p = booster.ConvParam.make(c.oc, c.ic, c.h, c.w, c.kh, c.kw, stride=c.sh, stride_w=c.sw, pad_lbrt=c.pad, group=c.group,
                               bias=c.bias, relu=c.relu)
    if c.clip is not None:
        p.activation = booster.ACT_CLIP
    # AssignOutputDim keeps the reference's rule that group == input_channels is depthwise, which with IC = 1 would
    # make this a one-output-channel layer
    p.output_channels = c.oc
    p.output_h, p.output_w = c.out_hw
    return p


def _supported(p, **opts):
    from feathercnn_b200._lib import FcudaConvOptions, fcuda
    o = FcudaConvOptions(**opts)
    return fcuda().fcuda_igemm_stem_supported(ctypes.byref(p), ctypes.byref(o)) == 1


@pytest.fixture
def stem(cuda):
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    saved = lib.fcuda_get_tuning(b"igemm_stem"), booster.get_precision()
    booster.set_precision(FP32_SPLIT)

    def setter(v):
        assert lib.fcuda_set_tuning(b"igemm_stem", v) == 0
    yield setter
    lib.fcuda_set_tuning(b"igemm_stem", saved[0])
    booster.set_precision(saved[1])


@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_stem_is_bit_identical_to_gathering_kernel(stem, c):
    from feathercnn_b200 import booster
    p = _param(c)
    assert _supported(p), c.name
    x, w, b, _ = make_data(c, "cuda")

    def run():
        out, algo = booster.conv_forward(p, x, w, b, algo=SGECONV, clip=c.clip)
        torch.cuda.synchronize()
        assert algo == SGECONV
        return out

    stem(0)
    old = run()
    stem(1)
    new = run()
    assert old.shape == new.shape
    if not torch.equal(old, new):
        diff = old.view(torch.int32) != new.view(torch.int32)
        np.testing.assert_array_equal(new.cpu().numpy(), old.cpu().numpy(),
                                      err_msg=f"{c.name}: {int(diff.sum())} of {diff.numel()} outputs differ")
    assert torch.equal(old.view(torch.int32), new.view(torch.int32)), c.name  # -0.0 / +0.0 and NaN payloads too
    del old
    assert float(new.abs().max()) > 0  # the comparison saw real data

    # the float64 bound of every BF16x3 implicit-GEMM output (tests/test_gpu_error_bounds.py)
    coef = eps_for("sgeconv", FP32_SPLIT) + c.K * U
    step = max(1, min(c.batch, int(4e8 // (8 * 4 * (c.ic * c.h * c.w + 3 * c.oc * c.out_hw[0] * c.out_hw[1])))))
    for i0 in range(0, c.batch, step):
        sl = slice(i0, i0 + step)
        ref = conv_ref(c, x[sl], w, b, None)
        s = conv_ref(c, x[sl], w, b, None, absolute=True)
        free = ref if c.clip is None else conv_ref(dataclasses.replace(c, clip=None), x[sl], w, b, None)
        used, _ = excess(new[sl], ref, coef * s + U * free.abs(), 1.0, 0.0)
        assert used <= 1.0, (c.name, i0, used)
        del ref, s, free


def test_stem_supported_query(cuda):
    from feathercnn_b200 import booster
    saved = booster.get_precision()
    try:
        booster.set_precision(FP32_SPLIT)
        vgg = _param(CASES[0])
        assert _supported(vgg)
        assert not _supported(vgg, residual=16)  # only tested for NULL, never read
        assert not _supported(vgg, pool=1)
        assert not _supported(vgg, dilation_h=2, dilation_w=2)
        assert _supported(vgg, dilation_h=1, dilation_w=1)
        assert not _supported(_param(Conv("oc129", 129, 3, 32, 32, 3)))                 # two N tiles
        assert _supported(_param(Conv("oc128", 128, 3, 32, 32, 3)))
        assert not _supported(_param(Conv("k294", 64, 6, 32, 32, 7, pad=3)))           # K = 294
        assert _supported(_param(Conv("k256", 64, 16, 32, 32, 4, pad=0)))
        assert not _supported(_param(Conv("ic32", 64, 32, 32, 32, 3)))                 # k-blocks of one tap
        booster.set_precision(TF32X3)
        assert not _supported(vgg)
        booster.set_precision(TF32)
        assert not _supported(vgg)
    finally:
        booster.set_precision(saved)
