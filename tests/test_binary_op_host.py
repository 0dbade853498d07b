"""ncnn's BinaryOp on the host (no kernel is launched): fcuda_binary_op_shape against a NumPy restatement of the operand
rule over seeded random rank and shape pairs, the per-channel rule where numpy alignment disagrees, the C ABI's
rejections (every call here fails its checks before a launch), the loader's accepts and rejects, and modelgen's
"binaryop" layouts: the same layers fused away as their Eltwise twins (so the residual and super-resolution tail passes
take a BinaryOp ADD), the same .bin, and default files unchanged.

binary_shape_ref is what tests/test_gpu_binary_op.py holds the layer's shapes to."""
from __future__ import annotations

import ctypes
import hashlib

import numpy as np
import pytest

from test_faster_rcnn_host import FAKE


# ---- the operand rule -----------------------------------------------------------------------------------------------
def binary_shape_ref(a_rank, a, b_rank, b):
    """include/fcuda.h fcuda_binary_op_shape restated: (rank, out, a aligned, b aligned) or None outside the rule."""
    a, b = list(a), list(b)
    size = lambda s: int(np.prod(s))  # noqa: E731
    rank = max(a_rank, b_rank)
    if a == b:
        pass
    elif size(a) == 1:
        rank = b_rank
    elif size(b) == 1:
        rank = a_rank
    elif a_rank == 3 and b_rank == 1 and b[2] == a[0]:
        b = [b[2], 1, 1]
    elif b_rank == 3 and a_rank == 1 and a[2] == b[0]:
        a = [a[2], 1, 1]
    try:
        out = np.broadcast_shapes(tuple(a), tuple(b))
    except ValueError:
        return None
    return rank, tuple(out), tuple(a), tuple(b)


def _shape_call(a_rank, a, b_rank, b):
    from feathercnn_b200._lib import fcuda
    i3 = ctypes.c_int * 3
    rank, out, aa, ba = ctypes.c_int(), i3(), i3(), i3()
    rc = fcuda().fcuda_binary_op_shape(a_rank, i3(*a), b_rank, i3(*b), ctypes.byref(rank), out, aa, ba)
    return rc, (rank.value, tuple(out), tuple(aa), tuple(ba))


def _random_operand(rng, rank, like=None):
    """A (c, h, w) of ncnn rank `rank`; with `like`, each axis often equal to like's or 1."""
    dims = []
    for k in range(3):
        if k < 3 - rank:
            dims.append(1)
        elif like is not None and rng.random() < 0.7:
            dims.append(like[k] if rng.random() < 0.6 else 1)
        else:
            dims.append(int(rng.integers(1, 6)))
    return dims


def test_shape_rule_matches_restatement():
    rng = np.random.default_rng(2024)
    outcomes = {"ok": 0, "reject": 0}
    for _ in range(400):
        ar, br = int(rng.integers(1, 4)), int(rng.integers(1, 4))
        a = _random_operand(rng, ar)
        b = _random_operand(rng, br, like=a if rng.random() < 0.8 else None)
        if rng.random() < 0.5:
            a, b, ar, br = b, a, br, ar
        want = binary_shape_ref(ar, a, br, b)
        rc, got = _shape_call(ar, a, br, b)
        if want is None:
            assert rc == -200, (ar, a, br, b, got)
            outcomes["reject"] += 1
        else:
            assert rc == 0 and got == want, (ar, a, br, b, got, want)
            outcomes["ok"] += 1
    assert outcomes["ok"] > 150 and outcomes["reject"] > 30, outcomes


@pytest.mark.parametrize("swap", [False, True])
def test_per_channel_wins_over_numpy(swap):
    """(4, 5, 4) with a rank-1 operand of 4: numpy would broadcast it along w; ncnn's per-channel rule takes c."""
    args = (3, (4, 5, 4), 1, (1, 1, 4))
    if swap:
        args = args[2:] + args[:2]
    rc, (rank, out, aa, ba) = _shape_call(*args)
    assert rc == 0 and rank == 3 and out == (4, 5, 4)
    assert (ba if not swap else aa) == (4, 1, 1)
    assert np.broadcast_shapes((4, 5, 4), (1, 1, 4)) == (4, 5, 4)  # numpy agrees on the shape, not on the axis


def test_shape_rule_cases():
    assert _shape_call(3, (8, 6, 7), 3, (8, 1, 1))[1] == (3, (8, 6, 7), (8, 6, 7), (8, 1, 1))
    assert _shape_call(3, (1, 6, 7), 3, (8, 1, 1))[1] == (3, (8, 6, 7), (1, 6, 7), (8, 1, 1))   # both broadcast
    assert _shape_call(2, (1, 6, 7), 1, (1, 1, 7))[1] == (2, (1, 6, 7), (1, 6, 7), (1, 1, 7))   # row
    assert _shape_call(3, (8, 6, 7), 1, (1, 1, 8))[1] == (3, (8, 6, 7), (8, 6, 7), (8, 1, 1))   # per channel
    assert _shape_call(1, (1, 1, 1), 3, (8, 6, 7))[1] == (3, (8, 6, 7), (1, 1, 1), (8, 6, 7))   # scalar
    assert _shape_call(3, (1, 1, 1), 1, (1, 1, 5))[1][0] == 1                                    # scalar: other rank
    assert _shape_call(3, (8, 6, 7), 3, (8, 6, 3))[0] == -200
    assert _shape_call(3, (8, 6, 7), 1, (1, 1, 6))[0] == -200


@pytest.mark.parametrize("args", [
    (0, (1, 1, 4), 1, (1, 1, 4)), (4, (1, 1, 4), 1, (1, 1, 4)), (1, (1, 1, 4), 3, (0, 2, 2)),
    (1, (2, 1, 4), 1, (1, 1, 4)), (1, (1, 2, 4), 1, (1, 1, 4)), (2, (2, 2, 4), 2, (1, 2, 4))])
def test_shape_rule_rejects_malformed(args):
    assert _shape_call(*args)[0] == -100


def test_shape_rule_null_pointers():
    from feathercnn_b200._lib import fcuda
    i3 = ctypes.c_int * 3
    rank, out, aa, ba = ctypes.c_int(), i3(), i3(), i3()
    lib = fcuda()
    assert lib.fcuda_binary_op_shape(3, None, 3, i3(1, 2, 3), ctypes.byref(rank), out, aa, ba) == -100
    assert lib.fcuda_binary_op_shape(3, i3(1, 2, 3), 3, i3(1, 2, 3), None, out, aa, ba) == -100
    assert lib.fcuda_binary_op_shape(3, i3(1, 2, 3), 3, i3(1, 2, 3), ctypes.byref(rank), out, None, ba) == -100


# ---- ABI rejections, before any launch ------------------------------------------------------------------------------
def _fwd(out=FAKE, a=FAKE, a_shape=(2, 3, 4, 5), b=FAKE, b_shape=(2, 3, 4, 5), op=0):
    from feathercnn_b200._lib import fcuda
    i4 = ctypes.c_int * 4
    return fcuda().fcuda_binary_op_forward(out, a, i4(*a_shape) if a_shape else None, b,
                                           i4(*b_shape) if b_shape else None, 1.0, op, 0, None)


OTHER = ctypes.c_void_p(4096)
REJECTS = {
    "null-out": (dict(out=None), -100), "null-a": (dict(a=None), -100), "null-a-shape": (dict(a_shape=None), -100),
    "b-without-shape": (dict(b_shape=None), -100), "empty-a": (dict(a_shape=(2, 0, 4, 5)), -100),
    "empty-b": (dict(b_shape=(2, 3, 4, 0)), -100), "zero-batch": (dict(a_shape=(0, 3, 4, 5)), -100),
    "op-negative": (dict(op=-1), -200), "op-12": (dict(op=12), -200), "batch-differs": (dict(b_shape=(1, 3, 4, 5)), -200),
    "no-broadcast": (dict(b_shape=(2, 3, 4, 2)), -200), "no-broadcast-c": (dict(b_shape=(2, 2, 1, 1)), -200),
    "plane-too-big": (dict(a_shape=(1, 1, 65536, 32768), b_shape=(1, 1, 1, 1)), -200),
    "out-is-broadcast-b": (dict(out=OTHER, b=OTHER, b_shape=(2, 3, 1, 5)), -200),
    "out-is-broadcast-a": (dict(out=OTHER, a=OTHER, a_shape=(2, 1, 4, 5)), -200),
    "out-is-broadcast-a-b-bigger": (dict(out=OTHER, a=OTHER, a_shape=(2, 3, 4, 1), b_shape=(2, 3, 1, 5)), -200),
}


@pytest.mark.parametrize("case", list(REJECTS))
def test_abi_rejects(case):
    kw, code = REJECTS[case]
    assert _fwd(**kw) == code


def test_abi_scalar_ignores_b_shape():
    """b NULL: the scalar form, where b_shape may be NULL; its checks still run first."""
    assert _fwd(b=None, b_shape=None, op=12) == -200
    assert _fwd(b=None, b_shape=None, a_shape=(1, 0, 1, 1)) == -100


# ---- loader ---------------------------------------------------------------------------------------------------------
HEAD = "Input d 0 1 d 0=6 1=5 2=4\nSplit s 1 2 d d1 d2\n"


def _load(body, fusion=False):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion)
    n = 2 + body.strip().count("\n") + 1
    net.LoadParamFromText(f"7767517\n{n} {n + 3}\n{HEAD}{body.strip()}\n")
    return net


@pytest.mark.parametrize("line", ["BinaryOp b 2 1 d1 d2 b", "BinaryOp b 2 1 d1 d2 b 0=11",
                                  "BinaryOp b 1 1 d1 b 0=2 1=1 2=5.000000e-01", "BinaryOp b 1 1 d1 b 0=6 1=1",
                                  "BinaryOp b 2 1 d1 d2 b 0=3 1=0"])
def test_loader_accepts(line):
    _load(line)


@pytest.mark.parametrize("line", ["BinaryOp b 2 1 d1 d2 b 0=12", "BinaryOp b 2 1 d1 d2 b 0=-1",
                                  "BinaryOp b 1 1 d1 b 0=0", "BinaryOp b 2 1 d1 d2 b 0=0 1=1",
                                  "BinaryOp b 2 1 d1 d2 b 1=2", "BinaryOp b 2 2 d1 d2 b c"])
def test_loader_rejects(line):
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError) as e:
        _load(line)
    assert e.value.code == -200, line


# ---- fusion decisions -----------------------------------------------------------------------------------------------
CONV = "Convolution c 1 1 d1 c 0=6 1=1 5=0 6=36"


@pytest.mark.parametrize("order", ["c d2", "d2 c"])
def test_residual_fuses(order):
    net = _load(f"{CONV}\nBinaryOp b 2 1 {order} b 0=0\nReLU r 1 1 b r", fusion=True)
    assert net.FuseNow() == 2 and (net.LayerFusedAway("b"), net.LayerFusedAway("r")) == (1, 1)


@pytest.mark.parametrize("line", ["BinaryOp b 2 1 c d2 b 0=1", "BinaryOp b 2 1 c d2 b 0=2", "BinaryOp b 2 1 c c b 0=0"])
def test_residual_left_in_place(line):
    """SUB and MUL are no sums; an ADD of one blob to itself has no second addend."""
    net = _load(f"{CONV}\n{line}", fusion=True)
    net.FuseNow()
    assert net.LayerFusedAway("b") == 0


def test_scalar_add_left_in_place():
    net = _load(f"{CONV}\nBinaryOp b 1 1 c b 0=0 1=1 2=1.000000e+00", fusion=True)
    net.FuseNow()
    assert net.LayerFusedAway("b") == 0 and net.LayerFusedAway("c") == 0


# ---- models ---------------------------------------------------------------------------------------------------------
MODELS = {"resnet50": {}, "mobilenet_v2": {}, "fast_neural_style": {}, "style_tiny": {}, "srvgg_compact": {},
          "sr_tiny": {}, "edsr_baseline": dict(n_resblocks=4, scale=3)}

# every sum fuses at load: a residual read straight from a convolution (EDSR) or an SR tail (SRVGGNetCompact)
SUMS_FUSE = {"srvgg_compact", "sr_tiny", "edsr_baseline"}

# sha256 of the default (.param text, .bin) at the parent commit: adds="eltwise" writes the same bytes
PINNED = {
    "resnet50": ("94b4f56354eaa7dd5f604e7a280517811795ada35d3621828370121b2e26733e",
                 "b2384943b512aa7a97d5affa31de3a01b6c4ab63d423f153a379d943d7d0e623"),
    "mobilenet_v2": ("bd0b5682be1188b73ce487e97a5e3373b306ecea9e0bd7db18597a09d63d56b4",
                     "82abbaba576a61e9f5e078a645fb64dbba12685c579675ea37fc05e4c4a1c3f3"),
    "fast_neural_style": ("986c96e982291ad0f9742a0ae14d4c87a9f00eb20445ce4cf3cf6b47dbdcb314",
                          "20e2fee8a080b6f9fdc73c1eef03cec3a81b1f2727b1beaa6daed589cac02dfa"),
    "style_tiny": ("814ec92af25be7919c491e2e5b8a603e7fb70da1a64a4f4a1052762e6b1d5ea9",
                   "857712655f74ceef8b6559706f82c59d749ba1cedbd70667de2a384fefe1afa0"),
    "srvgg_compact": ("807270e2b17addcf2bc06ef01d3d56e774c34183211d7be22dfb42ab4d68b126",
                      "9affe074759e683944d915ac9fd4bbc35574aa6589ec382f24ed31536124c49d"),
    "sr_tiny": ("3a476baa0d45fe5cb6fb150cdafc79e53e68e41c15dbee606ba8cf73032845aa",
                "80d01fca4b5f437da9136f5f14352a2719a7064a5e6a4cb4f69f9bcf435cac94"),
    "edsr_baseline": ("7bc085736623bc6d311ab001877bd0f57443f2076241d51cf138bac664cdf051",
                      "300c1627e6f155798bd518f2c28d6c1809885b4359ae304195b60b8705a36dc6"),
}


def _text(m):
    return "7767517\n" + f"{len(m.lines)} {len(m.blobs)}\n" + "\n".join(m.lines) + "\n"


def _sha(b):
    return hashlib.sha256(b).hexdigest()


@pytest.mark.parametrize("name", list(PINNED))
def test_default_layout_unchanged(name):
    from feathercnn_b200.tools import modelgen
    m = modelgen.ZOO[name]()
    assert (_sha(_text(m).encode()), _sha(bytes(m.bin))) == PINNED[name]
    assert not any(L.startswith("BinaryOp ") for L in m.lines)


def _fused(m, fusion=True):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion)
    net.LoadParamFromText(_text(m))
    count = net.FuseNow()
    return count, {L.split()[1] for L in m.lines if net.LayerFusedAway(L.split()[1])}


@pytest.mark.parametrize("name", list(MODELS))
def test_binaryop_twin(name):
    from feathercnn_b200.tools import modelgen
    e = modelgen.ZOO[name](**MODELS[name])
    b = modelgen.ZOO[name](adds="binaryop", **MODELS[name])
    assert bytes(b.bin) == bytes(e.bin)
    el = [L for L in e.lines if L.startswith("Eltwise ")]
    bl = [L for L in b.lines if L.startswith("BinaryOp ")]
    assert len(el) == len(bl) > 0 and not any(L.startswith("Eltwise ") for L in b.lines)
    assert all(L.endswith(" 0=0") for L in bl)
    # the same layers, names and blobs, with each Eltwise SUM written as BinaryOp ADD
    assert [L.replace("Eltwise ", "BinaryOp ", 1).replace(" 0=1", " 0=0") if L.startswith("Eltwise ") else L
            for L in e.lines] == b.lines
    assert b.shape == e.shape
    fe, fb = _fused(e), _fused(b)
    assert fe == fb and fe[0] > 0
    if name in SUMS_FUSE:  # without weights loaded only sums read straight from a convolution or a PixelShuffle fuse
        assert {L.split()[1] for L in el} <= fe[1]
    assert _fused(b, fusion=False) == (0, set())


def test_binary_op_writer():
    from feathercnn_b200.tools import modelgen
    m = modelgen.ModelWriter()
    x = m.input("data", 4, 5, 6)
    p = m.pool("gp", x, 1, global_pooling=True)
    y = m.binary_op("mul", [x, p], 2)
    z = m.binary_op("half", [y], 2, scalar=0.5)
    assert m.shape[y] == (4, 5, 6) and m.shape[z] == (4, 5, 6)
    assert m.lines[-2] == "BinaryOp mul 2 1 data gp mul 0=2"
    assert m.lines[-1] == "BinaryOp half 1 1 mul half 0=2 1=1 2=5.000000e-01"
    with pytest.raises(AssertionError):
        modelgen.ModelWriter(adds="sum")
