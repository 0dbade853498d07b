"""Normalize on the host (no kernel is launched): the loader's parameters, defaults and rejections; the -100 / -200 returns
of fcuda_normalize_workspace_size and fcuda_normalize_forward (every call here fails its checks before a launch) and the
workspace size arithmetic; the float64 definition normalize_ref on hand-computed cases of every mode and eps_mode; and
modelgen's VGG-SSD 300 (source shapes, 8732 priors, the Normalize line and its scales in the bin), with the MobileNet-SSD
and tiny-SSD files pinned to what modelgen wrote before the per-source PriorBox step existed.

NormalizeLayer::Reshape's scale-count check needs device blobs; tests/test_gpu_normalize.py runs it.  normalize_ref is the
definition tests/test_gpu_normalize.py holds the kernels to."""
from __future__ import annotations

import ctypes
import hashlib
import math

import numpy as np
import pytest


# ---- the definition ------------------------------------------------------------------------------------------------
def normalize_ref(x, scale, across_spatial=0, across_channel=1, eps=1e-4, eps_mode=0):
    """ncnn Normalize in float64 on (N, C, ...) with the fp32 eps: y = x * a * s_c (include/fcuda.h).  Returns (y, ssum)
    with ssum broadcastable to x viewed as (N, C, plane)."""
    x = np.asarray(x, np.float64)
    n, c = x.shape[:2]
    v = x.reshape(n, c, -1)
    sq = v * v
    if not across_spatial:
        ssum = sq.sum(axis=1, keepdims=True)
    elif across_channel:
        ssum = sq.sum(axis=(1, 2), keepdims=True)
    else:
        ssum = sq.sum(axis=2, keepdims=True)
    e = float(np.float32(eps))
    with np.errstate(divide="ignore", invalid="ignore"):
        if eps_mode == 0:
            a = 1.0 / np.sqrt(ssum + e)
        elif eps_mode == 1:
            a = 1.0 / np.maximum(np.sqrt(ssum), e)
        else:
            a = 1.0 / np.sqrt(np.maximum(ssum, e))
        s = np.asarray(scale, np.float64).reshape(-1)
        s = s[0] if s.size == 1 else s.reshape(1, c, 1)
        y = v * a * s
    return y.reshape(x.shape), ssum


def test_ref_per_pixel_hand_computed():
    x = np.array([[[3.0, 0.0, 1.0], [4.0, 0.0, 1.0]]])          # (1, 2, 3): pixels (3, 4), (0, 0), (1, 1)
    y, _ = normalize_ref(x, [1.0, 2.0], eps=0.0)
    assert np.allclose(y[0, :, 0], [0.6, 1.6])
    assert np.isnan(y[0, :, 1]).all()                            # an all-zero pixel with eps == 0: 0 * inf
    assert np.allclose(y[0, :, 2], [1 / math.sqrt(2), 2 / math.sqrt(2)])
    y, _ = normalize_ref(x, [1.0, 2.0], eps=1e-4)
    assert (y[0, :, 1] == 0).all()                               # eps > 0: a zero pixel stays 0
    y, _ = normalize_ref(x, [3.0], eps=0.0)                      # one shared scale
    assert np.allclose(y[0, :, 0], [1.8, 2.4])


@pytest.mark.parametrize("mode, want", [(0, 1 / math.sqrt(125.0)), (1, 1 / 100.0), (2, 1 / math.sqrt(100.0))])
def test_ref_eps_modes_hand_computed(mode, want):
    """ssum = 25, eps = 100: Caffe 1 / sqrt(25 + 100), PyTorch 1 / max(5, 100), TensorFlow 1 / sqrt(max(25, 100))."""
    x = np.array([[[3.0], [4.0]]])
    y, _ = normalize_ref(x, [1.0, 1.0], eps=100.0, eps_mode=mode)
    assert np.allclose(y[0, :, 0], [3 * want, 4 * want], rtol=1e-6)
    # ssum 2500 above eps: mode 0 adds eps, mode 1 compares it with sqrt(ssum) = 50 and keeps it, mode 2 ignores it
    x = np.array([[[30.0], [40.0]]])
    y, _ = normalize_ref(x, [1.0, 1.0], eps=100.0, eps_mode=mode)
    a = (1 / math.sqrt(2600.0), 1 / 100.0, 1 / 50.0)[mode]
    assert np.allclose(y[0, :, 0], [30 * a, 40 * a], rtol=1e-6)


def test_ref_across_spatial_hand_computed():
    x = np.array([[[1.0, 1.0], [1.0, 1.0]], [[3.0, 4.0], [0.0, 2.0]]])   # (2, 2, 2)
    y, _ = normalize_ref(x, [1.0, 2.0], across_spatial=1, across_channel=1, eps=0.0)
    assert np.allclose(y[0], [[0.5, 0.5], [1.0, 1.0]])                   # the image: ssum 4
    assert np.allclose(y[1], np.array([[3.0, 4.0], [0.0, 4.0]]) / math.sqrt(29.0))
    y, _ = normalize_ref(x, [1.0, 2.0], across_spatial=1, across_channel=0, eps=0.0)
    assert np.allclose(y[1], [[0.6, 0.8], [0.0, 2.0]])                   # per channel: ssum 25, then 4
    assert np.allclose(y[0], [[1 / math.sqrt(2)] * 2, [2 / math.sqrt(2)] * 2])


# ---- loader --------------------------------------------------------------------------------------------------------
HEAD = "7767517\n2 2\nInput data 0 1 data 0=8 1=8 2=4\n"


@pytest.mark.parametrize("line", [
    "Normalize n 1 1 data out 3=4",                                        # defaults: per pixel, eps 1e-4, mode 0
    "Normalize n 1 1 data out 0=0 1=0 2=1.000000e-10 3=4",                 # VGG-SSD's conv4_3_norm
    "Normalize n 1 1 data out 0=1 1=1 2=1.000000e-05 3=1",                 # whole image, shared scale
    "Normalize n 1 1 data out 0=1 3=4 4=0",                                # per channel plane
    "Normalize n 1 1 data out 1=1 3=3 9=1",                                # shared with 3 scales: scale[0] is used
    "Normalize n 1 1 data out 2=0 3=4 9=2",                                # eps 0 is allowed
])
def test_load_param_accepts(line):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText(HEAD + line + "\n")
    assert "out" in net.BlobNames()


@pytest.mark.parametrize("line, code", [
    ("Normalize n 1 1 data out", -100),                      # scale_data_size missing (0)
    ("Normalize n 1 1 data out 3=0", -100),
    ("Normalize n 1 1 data out 3=-4", -100),
    ("Normalize n 1 1 data out 3=4 9=3", -200),              # eps_mode outside 0..2
    ("Normalize n 1 1 data out 3=4 9=-1", -200),
    ("Normalize n 1 1 data out 0=0 3=4 4=0", -200),          # neither across_spatial nor across_channel
    ("Normalize n 1 1 data out 2=-1.0e-4 3=4", -200),        # negative eps
    ("Normalize n 1 1 data out 2=nan.0 3=4", -200),          # NaN eps
])
def test_load_param_rejections(line, code):
    from feathercnn_b200.net import FeatherError, Net
    with pytest.raises(FeatherError) as e:
        Net().LoadParamFromText(HEAD + line + "\n")
    assert e.value.code == code, line


def test_normalize_is_registered_and_never_fused():
    from feathercnn_b200.net import Net
    text = ("7767517\n4 4\nInput data 0 1 data 0=8 1=8 2=16\nConvolution conv 1 1 data c 0=16 1=3 4=1 5=1 6=2304\n"
            "Normalize n 1 1 c m 3=16\nReLU relu 1 1 m out\n")
    net = Net(fusion=True)
    net.LoadParamFromText(text)
    net.FuseNow()
    assert net.LayerFusedAway("n") == 0 and net.LayerFusedAway("relu") == 0


# ---- C ABI ---------------------------------------------------------------------------------------------------------
FAKE = ctypes.c_void_p(256)  # never dereferenced: every call below fails its argument checks first


def _fwd(**kw):
    from feathercnn_b200._lib import fcuda
    a = dict(out=FAKE, inp=FAKE, C=16, plane=64, scale=FAKE, ns=16, sp=0, ch=1, eps=1e-4, mode=0, ws=FAKE, batch=2)
    a.update(kw)
    return fcuda().fcuda_normalize_forward(a["out"], a["inp"], a["C"], a["plane"], a["scale"], a["ns"], a["sp"], a["ch"],
                                           a["eps"], a["mode"], a["ws"], a["batch"], None)


@pytest.mark.parametrize("kw", [dict(out=None), dict(inp=None), dict(scale=None), dict(C=0), dict(plane=0),
                                dict(batch=0), dict(sp=1, ws=None), dict(sp=1, ch=0, ws=None)])
def test_forward_rejects_null_and_empty(kw):
    assert _fwd(**kw) == -100


@pytest.mark.parametrize("kw", [dict(ns=0), dict(ns=2), dict(ns=17), dict(mode=3), dict(mode=-1), dict(sp=0, ch=0),
                                dict(eps=-1e-6), dict(eps=float("nan")), dict(eps=float("-inf"))])
def test_forward_rejects_parameters(kw):
    assert _fwd(**kw) == -200


def test_workspace_size():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    n = ctypes.c_size_t(7)
    assert lib.fcuda_normalize_workspace_size(0, 1, 512, 38 * 38, 64, ctypes.byref(n)) == 0 and n.value == 0
    assert lib.fcuda_normalize_workspace_size(1, 1, 512, 38 * 38, 4, ctypes.byref(n)) == 0
    assert n.value == 4 * math.ceil(512 * 1444 / 8192)                 # one partial per 8192-float chunk of an image
    assert lib.fcuda_normalize_workspace_size(1, 0, 512, 38 * 38, 4, ctypes.byref(n)) == 0
    assert n.value == 4 * 512 * 1                                      # one chunk per 1444-float plane
    assert lib.fcuda_normalize_workspace_size(1, 0, 3, 100 * 100, 2, ctypes.byref(n)) == 0
    assert n.value == 2 * 3 * 2                                        # 10000 floats: two chunks per plane
    assert lib.fcuda_normalize_workspace_size(1, 1, 1, 1, 1, ctypes.byref(n)) == 0 and n.value == 1
    assert lib.fcuda_normalize_workspace_size(0, 0, 16, 64, 2, ctypes.byref(n)) == -200
    assert lib.fcuda_normalize_workspace_size(0, 1, 0, 64, 2, ctypes.byref(n)) == -100
    assert lib.fcuda_normalize_workspace_size(0, 1, 16, 0, 2, ctypes.byref(n)) == -100
    assert lib.fcuda_normalize_workspace_size(0, 1, 16, 64, 0, ctypes.byref(n)) == -100
    assert lib.fcuda_normalize_workspace_size(0, 1, 16, 64, 2, None) == -100


# ---- models --------------------------------------------------------------------------------------------------------
def _weight_bytes(line: str) -> int:
    """Bytes a layer reads from the model bin, for the layer types modelgen's SSD models use."""
    tok = line.split()
    kv = dict(t.split("=", 1) for t in tok[4 + int(tok[2]) + int(tok[3]):])
    if tok[0] in ("Convolution", "ConvolutionDepthWise"):
        return 4 + 4 * int(kv["6"]) + (4 * int(kv["0"]) if kv.get("5", "0") != "0" else 0)
    if tok[0] == "Normalize":
        return 4 * int(kv["3"])
    return 0


def test_vgg_ssd_shapes_priors_and_normalize_scales(tmp_path):
    from feathercnn_b200.tools import modelgen
    m = modelgen.vgg_ssd()
    sources = ["conv4_3_norm", "relu7", "conv6_2_relu", "conv7_2_relu", "conv8_2_relu", "conv9_2_relu"]
    assert [m.shape[s] for s in sources] == [(512, 38, 38), (1024, 19, 19), (512, 10, 10), (256, 5, 5), (256, 3, 3),
                                             (256, 1, 1)]
    assert m.shape["pool3"] == (256, 38, 38) and m.shape["pool5"] == (512, 19, 19) and m.shape["relu6"] == (1024, 19, 19)
    P = 38 * 38 * 4 + 19 * 19 * 6 + 10 * 10 * 6 + 5 * 5 * 6 + 3 * 3 * 4 + 1 * 1 * 4
    assert P == 8732 and m.shape["mbox_priorbox"] == (1, 2, 4 * P)
    assert m.shape["mbox_conf_reshape"] == (1, P, 21) and m.shape["detection_out"] == (1, 200, 6)
    norm = [L for L in m.lines if L.startswith("Normalize ")]
    assert norm == ["Normalize conv4_3_norm 1 1 relu4_3 conv4_3_norm 0=0 1=0 2=1.000000e-10 3=512"]
    text = "\n".join(m.lines)
    assert "DetectionOutput detection_out 3 1 mbox_loc mbox_conf_flatten mbox_priorbox detection_out 0=21 " \
           "1=4.500000e-01 2=400 3=200" in text
    assert "Convolution fc6 1 1 pool5 fc6 0=1024 1=3 3=1 4=6 5=1 6=4718592 2=6" in text
    for src, step in zip(sources, (8, 16, 32, 64, 100, 300)):
        pb = [L for L in m.lines if L.startswith(f"PriorBox {src}_mbox_priorbox ")][0]
        assert f" 11={float(step):e} 12={float(step):e} " in pb, pb
    # the bin: every layer's weights in file order, the 512 scales of 20 raw (no flag) where the walk puts them
    param, binf = m.save(tmp_path / "vgg_ssd")
    data = open(binf, "rb").read()
    off = 0
    for L in m.lines:
        if L.startswith("Normalize "):
            assert np.array_equal(np.frombuffer(data[off:off + 2048], np.float32), np.full(512, 20.0, np.float32))
            assert data[off + 2048:off + 2052] == b"\0\0\0\0"  # the next layer (a convolution) starts with its flag
        off += _weight_bytes(L)
    assert off == len(data)
    from feathercnn_b200.net import Net
    net = Net(fusion=True)
    net.LoadParam(param)
    net.FuseNow()
    assert net.LayerFusedAway("conv4_3_norm") == 0


def test_normalize_writer_keys():
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter()
    m.input("data", 6, 4, 4)
    m.normalize("a", "data")
    m.normalize("b", "data", across_spatial=1, channel_shared=1, eps=1e-5, scale=[2.5], across_channel=0, eps_mode=2)
    assert m.lines[1:] == ["Normalize a 1 1 data a 0=0 1=0 2=1.000000e-10 3=6",
                           "Normalize b 1 1 data b 0=1 1=1 2=1.000000e-05 3=1 4=0 9=2"]
    assert bytes(m.bin) == np.full(6, 20.0, np.float32).tobytes() + np.float32(2.5).tobytes()


# sha256 of (.param, .bin) as modelgen wrote them before _ssd_heads took a per-source step
SSD_FILES = {
    "mobilenet_ssd": ("4a9a0d438827e1f966e0d6ce5fa94f0b930698ddc6b96721307c17605286d2a0",
                      "5f711877219de30f64088e4cab199268336cf587cafff1986f73a7fae039c70a"),
    "ssd_tiny": ("b8a307c361ec184a3a7b518add88b4e063a5d6f3e1ffea2e78e9dd49173c4ede",
                 "443ba6ccdb297fe6b8ec3bf5f4a37419b2ede158e2888f620763f153e2edb34b"),
}


@pytest.mark.parametrize("name", sorted(SSD_FILES))
def test_existing_ssd_models_are_byte_identical(tmp_path, name):
    from feathercnn_b200.tools import modelgen
    param, binf = modelgen.ZOO[name]().save(tmp_path / name)
    got = tuple(hashlib.sha256(open(f, "rb").read()).hexdigest() for f in (param, binf))
    assert got == SSD_FILES[name]
