"""Super-resolution's PixelShuffle on the host (no kernel is launched): NumPy definitions of both channel orders, checked
by hand and against PyTorch's pixel_shuffle; the deconvolution scatter's index map, with the geometry
fcuda_pixel_shuffle_forward gives it, restated in NumPy and equal to those definitions; the nearest map of the fused
tail, where fp32 1/3 and Y // 3 part; the C ABI's rejections (every call here fails its checks before a launch); the
loader's ids, defaults and rejections; Net's tail fusion decisions; and the blob shapes of modelgen's SR models.

pixel_shuffle_ref and upsample_ref are what tests/test_gpu_sr.py holds the kernels to."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from test_faster_rcnn_host import FAKE

F = np.float32


# ---- the definitions ------------------------------------------------------------------------------------------------
def pixel_shuffle_ref(x, r, mode=0):
    """(N, C, H, W) -> (N, C / r^2, H r, W r).  Output (p, h' r + i, w' r + j) reads channel p r^2 + i r + j (mode 0) or
    (i r + j) OC + p (mode 1) at (h', w')."""
    n, c, h, w = x.shape
    oc = c // (r * r)
    if mode == 0:
        y = x.reshape(n, oc, r, r, h, w).transpose(0, 1, 4, 2, 5, 3)
    else:
        y = x.reshape(n, r, r, oc, h, w).transpose(0, 3, 4, 1, 5, 2)
    return np.ascontiguousarray(y.reshape(n, oc, h * r, w * r))


def nearest_index(out, inp, scale):
    """ncnn's nearest source index of every output index: min((int)(d * scale), in - 1) with the fp32 product."""
    d = np.arange(out, dtype=np.float64).astype(np.float32)
    return np.minimum((d * F(scale)).astype(np.int64), inp - 1)


def upsample_ref(base, oh, ow, hs, ws):
    """ncnn's nearest Interp of (N, C, H, W) base to (oh, ow) with the fp32 scales hs, ws."""
    h, w = base.shape[2:]
    return np.ascontiguousarray(base[:, :, nearest_index(oh, h, hs)][:, :, :, nearest_index(ow, w, ws)])


def scatter_ref(P, OC, group, s, OH, OW):
    """deconv_scatter_kernel's index map (no pads, bias or ReLU), element by element in NumPy: out[n][oc][oy][ox] =
    P[n][((grp s + ry) s + rx) OCg + ocg][oy / s][ox / s], grp = oc / OCg, ry = oy % s, rx = ox % s."""
    n = P.shape[0]
    ocg_n = OC // group
    oc = np.arange(OC)[:, None, None]
    oy = np.arange(OH)[None, :, None]
    ox = np.arange(OW)[None, None, :]
    grp, ocg = oc // ocg_n, oc % ocg_n
    ch = ((grp * s + oy % s) * s + ox % s) * ocg_n + ocg
    return np.stack([P[i][ch, oy // s, ox // s] for i in range(n)])


# ---- the definitions, by hand ---------------------------------------------------------------------------------------
def test_pixel_shuffle_ref_by_hand():
    x = np.arange(8, dtype=np.float32).reshape(1, 8, 1, 1)          # C = 8, r = 2: OC = 2, one 2 x 2 block each
    assert pixel_shuffle_ref(x, 2, 0)[0].tolist() == [[[0, 1], [2, 3]], [[4, 5], [6, 7]]]
    assert pixel_shuffle_ref(x, 2, 1)[0].tolist() == [[[0, 2], [4, 6]], [[1, 3], [5, 7]]]
    x = np.arange(8, dtype=np.float32).reshape(1, 4, 1, 2)          # OC = 1, two input columns
    assert pixel_shuffle_ref(x, 2, 0)[0, 0].tolist() == [[0, 2, 1, 3], [4, 6, 5, 7]]
    assert np.array_equal(pixel_shuffle_ref(x, 1, 1), x)


@pytest.mark.parametrize("shape, r", [((2, 12, 3, 5), 2), ((1, 27, 4, 3), 3), ((3, 32, 2, 7), 4), ((1, 5, 3, 3), 1)])
def test_mode0_is_torch_pixel_shuffle(shape, r):
    x = np.random.default_rng(sum(shape)).standard_normal(shape).astype(np.float32)
    assert np.array_equal(pixel_shuffle_ref(x, r, 0), torch.nn.functional.pixel_shuffle(torch.from_numpy(x), r).numpy())


@pytest.mark.parametrize("shape, r", [((2, 12, 3, 5), 2), ((1, 18, 4, 3), 3), ((3, 32, 2, 7), 4)])
def test_mode1_is_depth_to_space_dcr(shape, r):
    """DCR: the depth axis splits as (i, j, p), which is mode 0 after moving p to the front of the channels."""
    x = np.random.default_rng(sum(shape)).standard_normal(shape).astype(np.float32)
    n, c, h, w = shape
    oc = c // (r * r)
    crd = x.reshape(n, r * r, oc, h, w).transpose(0, 2, 1, 3, 4).reshape(shape)
    assert np.array_equal(pixel_shuffle_ref(x, r, 1), pixel_shuffle_ref(crd, r, 0))


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("shape, r", [((2, 12, 3, 5), 2), ((1, 27, 4, 3), 3), ((2, 32, 2, 7), 4), ((1, 3, 2, 2), 1)])
def test_scatter_geometry_is_pixel_shuffle(mode, shape, r):
    """group = OC gives mode 0 and group = 1 mode 1 (fcuda_pixel_shuffle_forward's geometry)."""
    x = np.random.default_rng(r).standard_normal(shape).astype(np.float32)
    n, c, h, w = shape
    oc = c // (r * r)
    got = scatter_ref(x, oc, oc if mode == 0 else 1, r, h * r, w * r)
    assert np.array_equal(got, pixel_shuffle_ref(x, r, mode))


def test_upsample_ref_by_hand():
    base = np.arange(6, dtype=np.float32).reshape(1, 1, 2, 3)
    up = upsample_ref(base, 4, 6, 0.5, 0.5)
    assert up[0, 0].tolist() == [[0, 0, 1, 1, 2, 2], [0, 0, 1, 1, 2, 2], [3, 3, 4, 4, 5, 5], [3, 3, 4, 4, 5, 5]]


# An input width at which the nearest map of x 3 (scale 1 / 3.0f, as ncnn's Interp with scale 3 computes it) reads
# another column than X // 3 for some output columns X < 3 W: from X = 3 * 2^22 + 2 on, the fp32 product X * fp32(1/3)
# can round up to the next integer.
WIDE_X3 = 2 ** 22 + 128


def test_fp32_third_parts_from_integer_division():
    third = F(1) / F(3.0)
    idx = nearest_index(3 * WIDE_X3, WIDE_X3, third)
    x = np.arange(3 * WIDE_X3)
    differ = np.nonzero(idx != x // 3)[0]
    assert differ.size > 100 and differ[0] >= 3 * 2 ** 22
    small = nearest_index(3 * 4096, 4096, third)
    assert np.array_equal(small, np.arange(3 * 4096) // 3)       # at small widths the two agree


# ---- C ABI ----------------------------------------------------------------------------------------------------------
OTHER = ctypes.c_void_p(512)
BASE = ctypes.c_void_p(768)


def _map(h=8, w=6, out_h=0, out_w=0, scale=2.0, resize_type=1):
    from feathercnn_b200._lib import FcudaInterpParam
    return FcudaInterpParam(resize_type=resize_type, align_corner=0, height_scale=scale, width_scale=scale,
                            output_height=out_h, output_width=out_w, input_h=h, input_w=w)


PS_REJECTS = [
    (dict(out=None), -100), (dict(x=None), -100), (dict(amap=None), -100), (dict(c=0), -100), (dict(h=0), -100),
    (dict(w=0), -100), (dict(n=0), -100), (dict(amap=_map(h=0)), -100), (dict(amap=_map(scale=0.0)), -100),
    (dict(r=0), -200), (dict(r=-2), -200), (dict(r=65536), -200), (dict(mode=2), -200), (dict(mode=-1), -200),
    (dict(c=18), -200), (dict(c=2), -200), (dict(r=3), -200), (dict(out=FAKE), -200), (dict(out=BASE), -200),
    (dict(amap=_map(resize_type=2)), -200), (dict(amap=_map(scale=3.0)), -200), (dict(amap=_map(h=9)), -200),
    (dict(amap=_map(out_h=16, out_w=13)), -200), (dict(h=46341, w=46341, r=1, c=4, base=None, amap=None), -200),
    (dict(h=32768, w=32768, r=2, base=None, amap=None), -200),
]


def _ps_call(**kw):
    from feathercnn_b200._lib import fcuda
    a = dict(out=OTHER, x=FAKE, c=8, h=8, w=6, r=2, mode=0, base=BASE, amap=_map(), n=2)
    a.update(kw)
    amap = ctypes.byref(a["amap"]) if a["amap"] is not None else None
    return fcuda().fcuda_pixel_shuffle_forward(a["out"], a["x"], a["c"], a["h"], a["w"], a["r"], a["mode"], a["base"],
                                               amap, a["n"], None)


@pytest.mark.parametrize("kw, code", PS_REJECTS, ids=[str(i) for i in range(len(PS_REJECTS))])
def test_pixel_shuffle_abi_rejects(kw, code):
    assert _ps_call(**kw) == code


# ---- loader ---------------------------------------------------------------------------------------------------------
HEAD = "Input d 0 1 d 0=6 1=5 2=12\n"


def _load(body, fusion=False):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion)
    n = 1 + body.strip().count("\n") + 1
    net.LoadParamFromText(f"7767517\n{n} {n + 2}\n{HEAD}{body.strip()}\n")
    return net


@pytest.mark.parametrize("line", ["PixelShuffle p 1 1 d p 0=0", "PixelShuffle p 1 1 d p 0=-2",
                                  "PixelShuffle p 1 1 d p 0=2 1=2", "PixelShuffle p 1 1 d p 0=2 1=-1"])
def test_loader_rejects(line):
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError) as e:
        _load(line)
    assert e.value.code == -200, line


@pytest.mark.parametrize("line", ["PixelShuffle p 1 1 d p", "PixelShuffle p 1 1 d p 0=2", "PixelShuffle p 1 1 d p 0=2 1=1",
                                  "PixelShuffle p 1 1 d p 0=3 1=0"])
def test_loader_accepts(line):
    _load(line)


# ---- fusion decisions -----------------------------------------------------------------------------------------------
CONV = "Convolution c 1 1 d c 0=12 1=1 5=0 6=144"
FUSES = [
    f"{CONV}\nPixelShuffle ps 1 1 c ps 0=2\nInterp up 1 1 d3 up 0=1 1=2.0 2=2.0\nEltwise e 2 1 ps up e 0=1",
    f"{CONV}\nPixelShuffle ps 1 1 c ps 0=2 1=1\nInterp up 1 1 d3 up 0=1 3=10 4=12\nEltwise e 2 1 up ps e 0=1",
]
TAIL = ["ps", "up", "e"]


def _fused(net, names):
    return {n for n in names if net.LayerFusedAway(n)}


def _with_d3(body):
    """The three-channel blob the Interp reads, computed before the PixelShuffle."""
    return "Convolution c3 1 1 d d3 0=3 1=1 5=0 6=36\n" + body


@pytest.mark.parametrize("body", FUSES, ids=["shuffle-first", "interp-first"])
def test_tail_fuses(body):
    net = _load(_with_d3(body), fusion=True)
    assert net.FuseNow() == 2
    assert _fused(net, TAIL) == {"up", "e"}
    assert "e" in net.BlobNames() and "ps" not in net.BlobNames() and "up" not in net.BlobNames()


NO_FUSE = {
    "bilinear": FUSES[0].replace("0=1 1=2.0", "0=2 1=2.0"),
    "shuffle-read-twice": FUSES[0] + "\nReLU r 1 1 ps r",
    "interp-read-twice": FUSES[0] + "\nReLU r 1 1 up r",
    "eltwise-relu": FUSES[0] + "\nReLU r 1 1 e r",
    "eltwise-coeffs": FUSES[0].replace("e 0=1", "e 0=1 -23301=2,1.0,1.0"),
    "eltwise-max": FUSES[0].replace("e 0=1", "e 0=2"),
    "not-interp": FUSES[0].replace("Interp up 1 1 d3 up 0=1 1=2.0 2=2.0", "Deconvolution up 1 1 d3 up 0=3 1=2 3=2 6=36"),
}


@pytest.mark.parametrize("case", list(NO_FUSE))
def test_tail_left_in_place(case):
    net = _load(_with_d3(NO_FUSE[case]), fusion=True)
    net.FuseNow()
    assert _fused(net, TAIL) == set(), case
    if case == "eltwise-relu":
        assert net.LayerFusedAway("r") == 1        # the ReLU still joins the Eltwise, which then keeps both addends


def test_tail_left_when_interp_input_comes_after_shuffle():
    body = (f"{CONV}\nPixelShuffle ps 1 1 c ps 0=2\nConvolution c3 1 1 d d3 0=3 1=1 5=0 6=36\n"
            "Interp up 1 1 d3 up 0=1 1=2.0 2=2.0\nEltwise e 2 1 ps up e 0=1")
    net = _load(body, fusion=True)
    assert net.FuseNow() == 0


def test_tail_not_fused_without_fusion():
    net = _load(_with_d3(FUSES[0]), fusion=False)
    assert net.FuseNow() == 0


# ---- models ---------------------------------------------------------------------------------------------------------
def _types(m):
    return [L.split()[0] for L in m.lines]


@pytest.mark.parametrize("num_conv", [16, 32])
def test_srvgg_compact_shapes(num_conv):
    from feathercnn_b200.tools import modelgen
    m = modelgen.srvgg_compact(num_conv=num_conv)
    assert m.shape["output"] == (3, 1080, 1920) and m.shape["conv_last"] == (48, 270, 480)
    assert m.shape["upsample"] == (3, 1080, 1920) and m.shape["base"] == (3, 1080, 1920)
    t = _types(m)
    assert t.count("Convolution") == num_conv + 2 and t.count("PReLU") == num_conv + 1
    assert t.count("PixelShuffle") == 1 and t.count("Interp") == 1 and t.count("Eltwise") == 1
    assert "PixelShuffle upsample 1 1 conv_last upsample 0=4" in m.lines
    assert "Interp base 1 1 data_skip base 0=1 1=4.000000e+00 2=4.000000e+00" in m.lines
    assert "Eltwise output 2 1 upsample base output 0=1" in m.lines
    big = modelgen.srvgg_compact(height=540, width=960)
    assert big.shape["output"] == (3, 2160, 3840)
    assert modelgen.ZOO["srvgg_compact"] is modelgen.srvgg_compact


@pytest.mark.parametrize("scale, shuffles", [(2, [2]), (3, [3]), (4, [2, 2])])
def test_edsr_baseline_shapes(scale, shuffles):
    from feathercnn_b200.tools import modelgen
    m = modelgen.edsr_baseline(scale=scale, height=48, width=40)
    assert m.shape["add_mean"] == (3, 48 * scale, 40 * scale) and m.shape["body"] == (64, 48, 40)
    t = _types(m)
    assert t.count("Eltwise") == 17 and t.count("ReLU") == 16 and t.count("Convolution") == 2 + 1 + 32 + 1 + len(shuffles) + 1
    ps = [L for L in m.lines if L.startswith("PixelShuffle")]
    assert [int(L.split()[-1].split("=")[1]) for L in ps] == shuffles
    # every PixelShuffle feeds a convolution (the next upsampling stage or the tail)
    for L in ps:
        top = L.split()[5]
        assert any(x.startswith("Convolution") and x.split()[4] == top for x in m.lines), L
    assert "Convolution sub_mean 1 1 data sub_mean 0=3 1=1 3=1 4=0 5=1 6=9" in m.lines
    assert modelgen.ZOO["edsr_baseline"] is modelgen.edsr_baseline


def test_sr_tiny_contents():
    from feathercnn_b200.tools import modelgen
    m = modelgen.sr_tiny()
    assert m.shape["output"] == (3, 54, 66) and m.shape["shuffle1"] == (8, 18, 22)
    assert "PixelShuffle shuffle1 1 1 conv1 shuffle1 0=2 1=1" in m.lines
    assert "PixelShuffle shuffle2 1 1 conv2 shuffle2 0=3" in m.lines
    assert "Convolution conv2 1 1 shuffle1 conv2 0=27 1=3 3=1 4=1 5=1 6=1944" in m.lines
    from feathercnn_b200.net import Net
    net = Net(fusion=True)
    net.LoadParamFromText("7767517\n%d %d\n" % (len(m.lines), len(m.blobs)) + "\n".join(m.lines) + "\n")
    assert net.FuseNow() == 2 and net.LayerFusedAway("base") == 1 and net.LayerFusedAway("output") == 1
    assert net.LayerFusedAway("shuffle1") == 0 and net.LayerFusedAway("shuffle2") == 0
    assert modelgen.ZOO["sr_tiny"] is modelgen.sr_tiny
