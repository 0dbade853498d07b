"""Channel routing on the host (no kernel is launched): ShuffleChannel and Slice parsing and rejections, ncnn's Slice
rule (fcuda_slice_plan) against a Python restatement, the -100 / -200 rejections of fcuda_route_forward (every call here
fails its checks before a launch), the routing fusion pass on modelgen's nets, and the Caffe converter's Slice.

slice_ref is the definition tests/test_gpu_route.py holds the layers to."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

from test_tools import fbytes, fint, layer


# ---- the definitions -----------------------------------------------------------------------------------------------
def slice_ref(shape, axis, slices):
    """ncnn's Slice of one image of shape `shape` (rank = len(shape)): (dimension index into shape, sizes), or None when
    the layer must refuse (axis out of range, a size below 1, sizes past the extent)."""
    rank = len(shape)
    a = axis + rank if axis < 0 else axis
    if not 0 <= a < rank:
        return None
    extent, taken, sizes = shape[a], 0, []
    for i, s in enumerate(slices):
        n = (extent - taken) // (len(slices) - i) if s == -233 else s
        if n < 1 or taken + n > extent:
            return None
        sizes.append(n)
        taken += n
    return a, sizes


def shuffle_ref(x, group, reverse=0):
    """ncnn ShuffleChannel of x (N, C, ...): top channel k * j + i = bottom channel cpg * i + j."""
    c = x.shape[1]
    k = c // group if reverse else group
    return x.reshape((x.shape[0], k, c // k) + x.shape[2:]).swapaxes(1, 2).reshape(x.shape)


def test_shuffle_ref_hand_example():
    x = np.arange(6).reshape(1, 6)
    assert shuffle_ref(x, 2).tolist() == [[0, 3, 1, 4, 2, 5]]
    assert shuffle_ref(x, 3).tolist() == [[0, 2, 4, 1, 3, 5]]
    assert shuffle_ref(x, 3, reverse=1).tolist() == shuffle_ref(x, 2).tolist()  # k = 6 / 3 = 2
    assert shuffle_ref(shuffle_ref(x, 3), 3, reverse=1).tolist() == x.tolist()  # reverse undoes the shuffle


# ---- layers ---------------------------------------------------------------------------------------------------------
def _load(text):
    from feathercnn_b200.net import Net
    net = Net()
    net.LoadParamFromText("7767517\n" + text)
    return net


HEAD = "Input data 0 1 data 0=5 1=6 2=12\n"


@pytest.mark.parametrize("line", [
    "Slice s 1 2 data a b -23300=2,-233,-233",
    "Slice s 1 2 data a b -23300=2,5,-233 1=0",
    "Slice s 1 3 data a b c -23300=3,1,2,3 1=-1",
    "Slice s 1 1 data a -23300=1,4 1=2",
    "Slice s 1 2 data a b -23300=2,-233,-233 1=-3",
    "ShuffleChannel sc 1 1 data a",
    "ShuffleChannel sc 1 1 data a 0=3 1=1",
])
def test_loader_accepts(line):
    n_blobs = 1 + int(line.split()[3])
    _load(f"2 {n_blobs}\n{HEAD}{line}\n")


@pytest.mark.parametrize("line", [
    "Slice s 1 2 data a b -23300=3,1,1,1",           # more sizes than tops
    "Slice s 1 2 data a b -23300=1,4",               # fewer
    "Slice s 1 2 data a b 0=2",                      # not an array
    "Slice s 1 2 data a b",                          # no sizes at all
    "Slice s 1 2 data a b -23300=2,0,-233",          # a size below 1
    "Slice s 1 2 data a b -23300=2,-1,-233",
    "Slice s 1 2 data a b -23300=2,-233,-233 1=3",   # axis out of range for every rank
    "Slice s 1 2 data a b -23300=2,-233,-233 1=-4",
    "Slice s 1 2 data a b -23300=2,-233,-233 -23302=1,4",  # ncnn's 2=indices form
    "Slice s 1 2 data a b 2=4",
    "ShuffleChannel sc 1 1 data a 0=0",
    "ShuffleChannel sc 1 1 data a 0=-2",
])
def test_loader_rejects(line):
    from feathercnn_b200.net import FeatherError
    n_blobs = 1 + int(line.split()[3])
    with pytest.raises(FeatherError) as e:
        _load(f"2 {n_blobs}\n{HEAD}{line}\n")
    assert e.value.code == -200, line


def _random_case(rng):
    rank = int(rng.integers(1, 4))
    shape = tuple(int(v) for v in rng.integers(1, 20, rank))
    axis = int(rng.integers(-rank - 1, rank + 1))          # one out-of-range value on each side
    tops = int(rng.integers(1, 6))
    slices = [int(rng.choice([-233, int(rng.integers(0, 6))])) for _ in range(tops)]
    return shape, axis, slices


def test_slice_plan_matches_the_rule():
    """fcuda_slice_plan, which SliceLayer::Reshape and booster.slice use, on 300 seeded random (rank, axis, sizes)."""
    from feathercnn_b200 import booster
    rng = np.random.default_rng(7)
    accepted = refused = 0
    for _ in range(300):
        shape, axis, slices = _random_case(rng)
        want = slice_ref(shape, axis, slices)
        if want is None:
            with pytest.raises(booster.FcudaError) as e:
                booster.slice_plan(shape, axis, slices)
            assert e.value.code == -200, (shape, axis, slices)
            refused += 1
            continue
        sa, sizes = booster.slice_plan(shape, axis, slices)
        assert sizes == want[1], (shape, axis, slices)
        assert sa == want[0] + 3 - len(shape), (shape, axis, slices)
        accepted += 1
    assert accepted > 80 and refused > 80, (accepted, refused)


def test_slice_plan_rejects_bad_arguments():
    from feathercnn_b200._lib import fcuda
    i3 = (ctypes.c_int * 3)
    sa, sizes = ctypes.c_int(), i3()
    f = fcuda().fcuda_slice_plan
    assert f(3, 0, i3(4, 1, 1), i3(-233, 0, 0), 1, ctypes.byref(sa), sizes) == 0 and sizes[0] == 4
    assert f(3, 0, None, i3(-233, 0, 0), 1, ctypes.byref(sa), sizes) == -100
    assert f(3, 0, i3(4, 1, 1), None, 1, ctypes.byref(sa), sizes) == -100
    assert f(3, 0, i3(4, 1, 1), i3(-233, 0, 0), 0, ctypes.byref(sa), sizes) == -100
    assert f(4, 0, i3(4, 1, 1), i3(-233, 0, 0), 1, ctypes.byref(sa), sizes) == -100
    assert f(0, 0, i3(4, 1, 1), i3(-233, 0, 0), 1, ctypes.byref(sa), sizes) == -100
    assert f(3, 0, i3(0, 1, 1), i3(-233, 0, 0), 1, ctypes.byref(sa), sizes) == -100
    assert f(3, 0, i3(4, 1, 1), i3(5, 0, 0), 1, ctypes.byref(sa), sizes) == -200       # overrun
    assert f(3, 0, i3(4, 1, 1), i3(-233, -233, -233), 3, ctypes.byref(sa), sizes) == 0 and list(sizes) == [1, 1, 2]
    assert f(3, 0, i3(2, 1, 1), i3(-233, -233, -233), 3, ctypes.byref(sa), sizes) == -200  # 2 // 3 = 0


# ---- C ABI ----------------------------------------------------------------------------------------------------------
FAKE = 256  # never dereferenced: every call below fails its argument checks first


def _route(**kw):
    from feathercnn_b200._lib import FcudaRoute
    r = FcudaRoute()
    r.outer, r.inner, r.num_src, r.num_dst, r.group = 1, 49, 2, 2, 2
    r.src[0], r.src[1], r.dst[0], r.dst[1] = FAKE, FAKE, FAKE, FAKE
    r.src_extent[0], r.src_extent[1], r.dst_extent[0], r.dst_extent[1] = 58, 58, 58, 58
    for k, v in kw.items():
        if k in ("src", "dst", "src_extent", "dst_extent"):
            for i, x in v.items():
                getattr(r, k)[i] = x
        else:
            setattr(r, k, v)
    return r


@pytest.mark.parametrize("kw, batch, code", [
    (dict(src={0: None}), 1, -100), (dict(dst={1: None}), 1, -100), (dict(src_extent={1: 0}), 1, -100),
    (dict(dst_extent={0: 0}), 1, -100), (dict(outer=0), 1, -100), (dict(inner=0), 1, -100), ({}, 0, -100),
    (dict(dst_begin=-1), 1, -100), (dict(dst_begin=1), 1, -100), (dict(dst_extent={1: 59}), 1, -100),
    (dict(num_src=9), 1, -200), (dict(num_dst=9), 1, -200), (dict(num_src=0), 1, -200), (dict(num_dst=0), 1, -200),
    (dict(group=0), 1, -200), (dict(group=3), 1, -200), (dict(group=5, reverse=1), 1, -200),
    (dict(outer=1 << 16, inner=1 << 16), 1, -200),
])
def test_route_abi_rejects(kw, batch, code):
    from feathercnn_b200._lib import fcuda
    r = _route(**kw)
    assert fcuda().fcuda_route_forward(ctypes.byref(r), batch, None) == code, kw


def test_route_abi_rejects_null_route():
    from feathercnn_b200._lib import fcuda
    assert fcuda().fcuda_route_forward(None, 1, None) == -100


# ---- fusion ---------------------------------------------------------------------------------------------------------
def _net(tmp_path, name, fusion=True, **kw):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.ZOO[name](**kw)
    param, _ = m.save(tmp_path / name)
    net = Net(fusion=fusion)
    net.LoadParam(param)
    return m, net


ROUTE_TYPES = ("Concat", "ShuffleChannel", "Slice")


def _route_layers(m):
    return [(ln.split()[0], ln.split()[1]) for ln in m.lines if ln.split()[0] in ROUTE_TYPES]


@pytest.mark.parametrize("width", [0.5, 1.0])
def test_shufflenet_v2_fusion(tmp_path, width):
    """Every Concat is absorbed, every ShuffleChannel but the last of a stage (its top goes to a Split or conv5), no
    Slice: 13 Concat -> ShuffleChannel -> Slice chains and 3 Concat -> ShuffleChannel pairs."""
    m, net = _net(tmp_path, "shufflenet_v2", width=width, size=64)
    plain = _net(tmp_path, "shufflenet_v2", fusion=False, width=width, size=64)[1].FuseNow()
    assert plain == 0
    n = net.FuseNow()
    fused = {name for typ, name in _route_layers(m) if net.LayerFusedAway(name) == 1}
    last = {f"stage{s}_{u}_shuffle" for s, u in ((2, 4), (3, 8), (4, 4))}
    want = ({name for typ, name in _route_layers(m) if typ == "Concat"} |
            {name for typ, name in _route_layers(m) if typ == "ShuffleChannel"} - last)
    assert fused == want and len(fused) == 29
    # the other passes as on every net: each BatchNorm absorbs its Scale and ReLU
    absorbed = sum(ln.split()[0] in ("Scale", "ReLU") for ln in m.lines)
    assert n == 29 + absorbed
    names = set(net.BlobNames())
    for typ, name in _route_layers(m):
        line = next(ln.split() for ln in m.lines if ln.split()[1] == name)
        tops = line[4 + int(line[2]):4 + int(line[2]) + int(line[3])]
        assert all((t in names) == (name not in fused) for t in tops), name


def test_route_fuse_switch_turns_only_the_routing_pass_off(tmp_path):
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    assert lib.fcuda_set_tuning(b"route_fuse", 0) == 0
    try:
        m, net = _net(tmp_path, "shufflenet_v2", width=0.5, size=64)
        n = net.FuseNow()
    finally:
        lib.fcuda_set_tuning(b"route_fuse", 1)
    assert all(net.LayerFusedAway(name) == 0 for _, name in _route_layers(m))
    assert n == sum(ln.split()[0] in ("Scale", "ReLU") for ln in m.lines)


def test_shuffle_tiny_fusion(tmp_path):
    m, net = _net(tmp_path, "shuffle_tiny")
    net.FuseNow()
    fused = {name for typ, name in _route_layers(m) if net.LayerFusedAway(name) == 1}
    # shuffle_g3 -> slice_uneven, cat1 -> shuffle_rev -> slice_even, cat2 -> slice_cat; slice_h reads a Split and
    # slice_w an unshuffled Slice top; cat3 feeds a pooling layer
    assert fused == {"shuffle_g3", "cat1", "shuffle_rev", "cat2"}


EXISTING_FUSED = {"single_conv": 0, "vgg16": 20, "resnet50": 102, "mobilenet_v1": 54, "mini": 7, "decoder_tiny": 5,
                  "fcn8s_tiny": 13, "deeplab_head_tiny": 4, "mobilenet_v2": 52, "prelu_tiny": 2, "mobilenet_ssd": 70,
                  "ssd_tiny": 3, "mobilenet_yolov2": 58, "mobilenetv2_yolov3": 60, "yolo_tiny": 5}


@pytest.mark.parametrize("name", sorted(EXISTING_FUSED))
def test_existing_models_fuse_as_before(tmp_path, name):
    m, net = _net(tmp_path, name)
    assert net.FuseNow() == EXISTING_FUSED[name]
    assert all(net.LayerFusedAway(n) == 0 for t, n in _route_layers(m))


def test_shufflenet_v2_shapes():
    from feathercnn_b200.tools import modelgen
    for width, stages in modelgen.SHUFFLENET_V2_STAGES.items():
        m = modelgen.shufflenet_v2(width=width)
        assert m.shape["pool1"] == (24, 56, 56)
        for s, (c, hw) in zip((2, 3, 4), zip(stages, (28, 14, 7))):
            last = {2: 4, 3: 8, 4: 4}[s]
            assert m.shape[f"stage{s}_{last}_shuffle"] == (c, hw, hw)
            assert m.shape[f"stage{s}_2_slice_0"] == (c // 2, hw, hw)
        assert m.shape["conv5"][0] == (2048 if width == 2.0 else 1024)
        assert m.shape["prob"] == (1000, 1, 1)


# ---- Caffe converter ------------------------------------------------------------------------------------------------
def _caffe(slice_param: bytes, tops) -> str:
    from feathercnn_b200.tools import caffe2feather
    net = fbytes(3, "data") + b"".join(fint(4, d) for d in (1, 12, 6, 5))
    net += layer("sl", "Slice", ["data"], list(tops), p126=slice_param)
    text, _ = caffe2feather.convert(net)
    return next(ln for ln in text.splitlines() if ln.startswith("Slice"))


@pytest.mark.parametrize("param, tops, want", [
    (b"", ["a", "b"], "-23300=2,-233,-233"),                                  # no points: even split on channels
    (fint(2, 5), ["a", "b"], "-23300=2,5,-233"),
    (fint(2, 2) + fint(2, 7), ["a", "b", "c"], "-23300=3,2,5,-233"),
    (fint(3, 2) + fint(2, 4), ["a", "b"], "-23300=2,4,-233 1=1"),              # axis = 2: h
    (fint(1, 3) + fint(2, 1), ["a", "b"], "-23300=2,1,-233 1=2"),              # slice_dim = 3: w
    (fint(3, (1 << 64) - 1), ["a", "b", "c"], "-23300=3,-233,-233,-233 1=2"),  # axis = -1
])
def test_converter_maps_slice(param, tops, want):
    line = _caffe(param, tops)
    assert line == f"Slice sl 1 {len(tops)} data {' '.join(tops)} {want}"
    _load(f"2 {1 + len(tops)}\n{HEAD}{line}\n")


@pytest.mark.parametrize("param, tops", [
    (fint(3, 0), ["a", "b"]),                    # the batch axis
    (fint(2, 4), ["a", "b", "c"]),               # too few cut points
    (fint(2, 4) + fint(2, 4), ["a", "b", "c"]),  # not increasing
])
def test_converter_rejects_slice(param, tops):
    with pytest.raises(ValueError):
        _caffe(param, tops)


def test_converter_has_no_shuffle_channel():
    from feathercnn_b200.tools import caffe2feather
    net = fbytes(3, "data") + b"".join(fint(4, d) for d in (1, 12, 6, 5))
    net += layer("sc", "ShuffleChannel", ["data"], ["out"])
    with pytest.raises(ValueError, match="no FeatherCNN counterpart"):
        caffe2feather.convert(net)
