"""The implicit-GEMM halo kernel (switch igemm_halo = 1) against the gathering kernel (igemm_halo = 0).

Both issue the same wgmma sequence on the same operand values in the same k order with the same N tile, so every output
must be BIT-identical, in all three arithmetic modes.  The host tests pin which layers take the halo kernel and that the
shared-memory box it picks is free of bank conflicts."""
import ctypes
import zlib

import numpy as np
import pytest

MODES = ["fp32split", "tf32x3", "tf32"]


def _param(oc, ic, h, w, kh, kw, pad, group=1, pad_lbrt=None, stride=1):
    from feathercnn_b200 import booster
    return booster.ConvParam.make(oc, ic, h, w, kh, kw, stride=stride, pad=pad, group=group, relu=True, pad_lbrt=pad_lbrt)


def _halo_tile(p):
    from feathercnn_b200._lib import fcuda
    geom = (ctypes.c_int * 4)()
    ok = fcuda().fcuda_igemm_halo_tile(ctypes.byref(p), geom)
    return tuple(geom) if ok else None


def _set_mode(mode):
    from feathercnn_b200 import booster
    booster.set_precision({"fp32split": booster.PRECISION_FP32_SPLIT, "tf32x3": booster.PRECISION_TF32X3,
                           "tf32": booster.PRECISION_TF32}[mode])


def _conflict_free(cstride, mode):
    """Bank model of one ld.shared of the A gather: lane l reads column l // 4 of channel plane (l % 4) * (2 for the bf16
    pairs of fp32split, 1 for tf32) of the box; conflict-free when the 32 words hit 32 different banks."""
    m = 2 if mode == "fp32split" else 1
    return len({((l >> 2) + m * (l & 3) * cstride) % 32 for l in range(32)}) == 32


# ---------------------------------------------------------------------------------------------------------------- host
# (oc, ic, h, w, kh, kw, pad, group): the SGECONV layers of the benchmark nets and the edge cases below
ELIGIBLE = {
    "vgg16_conv1_2": (64, 64, 224, 224, 3, 3, 1, 1),
    "vgg16_conv2_1": (128, 64, 112, 112, 3, 3, 1, 1),
    "vgg16_conv2_2": (128, 128, 112, 112, 3, 3, 1, 1),
    "resnet50_3x3_56": (64, 64, 56, 56, 3, 3, 1, 1),
    "resnet50_3x3_28": (128, 128, 28, 28, 3, 3, 1, 1),
    "k5x5_pad2": (72, 64, 40, 44, 5, 5, 2, 1),
    "grouped_icg32": (128, 64, 20, 20, 3, 3, 1, 2),
}
INELIGIBLE = {
    "vgg16_conv1_1_ic3": (64, 3, 224, 224, 3, 3, 1, 1),
    "pointwise": (256, 64, 56, 56, 1, 1, 0, 1),
    "w7": (512, 512, 7, 7, 3, 3, 1, 1),
    "ic48_k_table": (64, 48, 32, 32, 3, 3, 1, 1),
    "w_not_multiple_of_4": (64, 64, 30, 30, 3, 3, 1, 1),
    "grouped_icg16": (64, 32, 20, 20, 3, 3, 1, 2),
}


@pytest.mark.parametrize("mode", MODES)
def test_halo_eligibility_and_bank_free_boxes(mode):
    _set_mode(mode)
    for name, (oc, ic, h, w, kh, kw, pad, g) in ELIGIBLE.items():
        t = _halo_tile(_param(oc, ic, h, w, kh, kw, pad, group=g))
        assert t is not None, name
        r, c, rb, cb = t
        assert r * c == 128 and c in (8, 16, 32, 64), (name, t)
        assert rb >= r + kh - 1 and cb >= c + kw - 1 and cb % 4 == 0 and rb <= 256 and cb <= 256, (name, t)
        assert _conflict_free(rb * cb, mode), (name, t)
    for name, (oc, ic, h, w, kh, kw, pad, g) in INELIGIBLE.items():
        assert _halo_tile(_param(oc, ic, h, w, kh, kw, pad, group=g)) is None, name
    assert _halo_tile(_param(64, 64, 56, 56, 3, 3, 1, stride=2)) is None
    # patches that waste no columns / rows where one exists: 224 and 112 = 16-column patches, 28 = 32 x 4
    assert _halo_tile(_param(64, 64, 224, 224, 3, 3, 1))[:2] == (8, 16)
    assert _halo_tile(_param(128, 64, 112, 112, 3, 3, 1))[:2] == (8, 16)
    assert _halo_tile(_param(128, 128, 28, 28, 3, 3, 1))[:2] == (4, 32)


def test_halo_switch_is_registered():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    assert lib.fcuda_get_tuning(b"igemm_halo") == 1
    assert lib.fcuda_set_tuning(b"igemm_halo", 2) == -200


# ----------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture
def halo_switch():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    saved = lib.fcuda_get_tuning(b"igemm_halo")

    def setter(v):
        assert lib.fcuda_set_tuning(b"igemm_halo", v) == 0
    yield setter
    lib.fcuda_set_tuning(b"igemm_halo", saved)


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
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_halo_kernel_is_bit_identical_to_gathering_kernel(cuda, halo_switch, mode, case):
    from feathercnn_b200 import booster
    name, oc, ic, h, w, kh, kw, pad, n, group, extra = case
    _set_mode(mode)
    lbrt = pad if isinstance(pad, tuple) else None
    p = _param(oc, ic, h, w, kh, kw, 0 if lbrt else pad, group=group, pad_lbrt=lbrt)
    assert _halo_tile(p) is not None, name
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

    halo_switch(0)
    old = run()
    halo_switch(1)
    new = run()
    assert old.shape == new.shape
    if not cuda.equal(old, new):
        diff = (old != new)
        np.testing.assert_array_equal(new.cpu().numpy(), old.cpu().numpy(),
                                      err_msg=f"{name} {mode}: {int(diff.sum())} of {diff.numel()} outputs differ")
    assert float(old.abs().max()) > 0  # the comparison saw real data
