"""fcuda_conv_forward_opts against the five entry points it stands behind: the same return code for every malformed call
an older entry point can express (including which code wins when a call is wrong in two ways), -200 for the combinations
none of them could express, and bit-identical outputs on every algorithm."""
import ctypes

import numpy as np
import pytest

gpu = pytest.mark.gpu
NAIVE, IM2COL, SGECONV, DEPTHWISE, WINOGRADF63, FUSED, WINOGRADF23 = range(7)
NONE, RELU, CLIP = 0, 1, 2
D = 16  # a non-NULL pointer no rejected call may touch
NAN = float("nan")


def _param(activation=NONE, ch=16, group=1):
    from feathercnn_b200._lib import FcudaConvParam, fcuda
    p = FcudaConvParam(ch, ch, 12, 12, 3, 3, 0, 0, 1, 1, 1, 1, 1, 1, group, 1, activation)
    assert fcuda().fcuda_conv_assign_output_dim(ctypes.byref(p)) == 0
    return p


def _call(entry, p, algo, o, batch=1, ptrs=(D, D, D, D, D), stream=None):
    """`entry` with the arguments its signature has, taken from the options `o`."""
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    head = (None if p is None else ctypes.byref(p), algo) + tuple(ptrs)
    if entry == "opts":
        return lib.fcuda_conv_forward_opts(*head, None if o is None else ctypes.byref(o), batch, stream)
    if entry == "forward":
        return lib.fcuda_conv_forward(*head, batch, stream)
    if entry == "clip":
        return lib.fcuda_conv_forward_clip(*head, o.clip_min, o.clip_max, batch, stream)
    if entry == "residual":
        return lib.fcuda_conv_forward_residual(*head, o.residual, o.relu_after_add, batch, stream)
    if entry == "pool":
        return lib.fcuda_conv_forward_pool(*head, batch, stream)
    assert entry == "ext"
    return lib.fcuda_conv_forward_ext(*head, o.residual, o.relu_after_add, o.dilation_h, o.dilation_w, batch, stream)


def _opts(**kw):
    from feathercnn_b200._lib import FcudaConvOptions
    return FcudaConvOptions(**kw)


NO_OUT = (None, D, D, D, D)
NO_IN = (D, None, D, D, D)
# (id, entry, activation, algo, options, call keywords, code).  "null" in the id: the parameter pointer is NULL.
MALFORMED = [
    ("forward-null", "forward", NONE, IM2COL, {}, {}, -100),
    ("forward-batch0", "forward", NONE, IM2COL, {}, dict(batch=0), -100),
    ("forward-no-input", "forward", RELU, WINOGRADF63, {}, dict(ptrs=NO_IN), -100),
    ("forward-fused-winograd", "forward", NONE, FUSED, {}, {}, -1),
    ("clip-null", "clip", CLIP, SGECONV, dict(clip_min=0, clip_max=6), {}, -100),
    ("clip-not-clip", "clip", RELU, SGECONV, dict(clip_min=0, clip_max=6), {}, -200),
    ("clip-min-above-max", "clip", CLIP, SGECONV, dict(clip_min=1, clip_max=0), {}, -200),
    ("clip-nan", "clip", CLIP, NAIVE, dict(clip_min=NAN, clip_max=6), {}, -200),
    ("clip-min-above-max+batch0", "clip", CLIP, SGECONV, dict(clip_min=1, clip_max=0), dict(batch=0), -200),
    ("clip-not-clip+unknown-algo", "clip", NONE, FUSED, dict(clip_min=0, clip_max=6), {}, -200),
    ("clip-batch0", "clip", CLIP, SGECONV, dict(clip_min=0, clip_max=6), dict(batch=0), -100),
    ("clip-unknown-algo", "clip", CLIP, FUSED, dict(clip_min=0, clip_max=6), {}, -1),
    ("clip-no-output", "clip", CLIP, IM2COL, dict(clip_min=0, clip_max=6), dict(ptrs=NO_OUT), -100),
    ("ext-null", "ext", NONE, SGECONV, dict(dilation_h=2, dilation_w=2), {}, -100),
    ("ext-negative-dilation", "ext", NONE, SGECONV, dict(dilation_h=-1, dilation_w=1), {}, -100),
    ("ext-negative-dilation+im2col", "ext", NONE, IM2COL, dict(dilation_h=2, dilation_w=-2), {}, -100),
    ("ext-dilated-im2col", "ext", NONE, IM2COL, dict(dilation_h=2, dilation_w=2), {}, -200),
    ("ext-dilated-im2col+batch0", "ext", NONE, IM2COL, dict(dilation_h=1, dilation_w=2), dict(batch=0), -200),
    ("ext-dilated-winograd+unfused-residual", "ext", NONE, WINOGRADF63, dict(residual=D, dilation_h=2, dilation_w=2), {}, -200),
    ("ext-dilated+unfused-residual", "ext", RELU, SGECONV, dict(residual=D, relu_after_add=1, dilation_h=2, dilation_w=2), {},
     -200),
    ("ext-dilated+unfused-residual+batch0", "ext", RELU, SGECONV, dict(residual=D, dilation_h=2, dilation_w=2), dict(batch=0),
     -200),
    ("ext-dilated-batch0", "ext", NONE, SGECONV, dict(dilation_h=2, dilation_w=2), dict(batch=0), -100),
    ("ext-dilated-residual-no-output", "ext", NONE, SGECONV, dict(residual=D, dilation_h=2, dilation_w=2), dict(ptrs=NO_OUT),
     -100),
    ("residual-null", "residual", NONE, SGECONV, dict(residual=D), {}, -100),
    ("residual-batch0", "residual", NONE, SGECONV, dict(residual=D, relu_after_add=1), dict(batch=0), -100),
    ("residual-unfused-no-output", "residual", RELU, WINOGRADF23, dict(residual=D), dict(ptrs=NO_OUT), -100),
    ("residual-unknown-algo", "residual", NONE, FUSED, dict(residual=D), {}, -1),
    ("pool-null", "pool", NONE, WINOGRADF63, dict(pool=1), {}, -100),
    ("pool-im2col", "pool", NONE, IM2COL, dict(pool=1), {}, -200),
    ("pool-naive", "pool", RELU, NAIVE, dict(pool=1), {}, -200),
    ("pool-depthwise", "pool", NONE, DEPTHWISE, dict(pool=1), {}, -200),
    ("pool-sgeconv-16-channels", "pool", NONE, SGECONV, dict(pool=1), {}, -200),
    ("pool-im2col+batch0", "pool", NONE, IM2COL, dict(pool=1), dict(batch=0), -200),
    ("pool-batch0", "pool", NONE, WINOGRADF63, dict(pool=1), dict(batch=0), -100),
    ("pool-no-input", "pool", RELU, WINOGRADF23, dict(pool=1), dict(ptrs=NO_IN), -100),
]


@pytest.mark.parametrize("case", MALFORMED, ids=[c[0] for c in MALFORMED])
def test_opts_returns_the_code_of_the_older_entry_point(case):
    name, entry, activation, algo, okw, ckw, code = case
    p = None if "null" in name else _param(activation, group=16 if algo == DEPTHWISE else 1)
    o = _opts(**okw)
    assert _call(entry, p, algo, o, **ckw) == code
    assert _call("opts", p, algo, o, **ckw) == code


def test_older_entry_points_keep_the_checks_the_options_cannot_express():
    d2 = _opts(dilation_h=2, dilation_w=2)
    assert _call("residual", _param(), SGECONV, _opts(residual=None)) == -100
    assert _call("ext", _param(), SGECONV, _opts(dilation_h=0, dilation_w=1)) == -100
    assert _call("opts", _param(), IM2COL, _opts(dilation_h=0, dilation_w=0), batch=0) == -100  # 0 means 1: reaches the plan
    # a Clip through an entry point without bounds: -200 after the plan's own error, before the tensor checks
    for entry, o in (("forward", _opts()), ("residual", _opts(residual=D)), ("ext", d2), ("pool", _opts(pool=1))):
        algo = WINOGRADF63 if entry == "pool" else SGECONV
        assert _call(entry, _param(CLIP), algo, o) == -200, entry
        assert _call(entry, _param(CLIP), algo, o, ptrs=NO_OUT) == -200, entry
        assert _call(entry, _param(CLIP), algo, o, batch=0) == -100, entry
        # (the pooling and the dilation are refused on an unknown algorithm before it is planned)
        assert _call(entry, _param(CLIP), FUSED, o) == (-200 if entry in ("pool", "ext") else -1), entry


NOT_BUILT = [
    ("clip+pool", CLIP, WINOGRADF63, 16, dict(clip_min=0, clip_max=6, pool=1)),
    ("clip+residual", CLIP, SGECONV, 16, dict(clip_min=0, clip_max=6, residual=D)),
    ("clip+dilation", CLIP, SGECONV, 16, dict(clip_min=0, clip_max=6, dilation_h=2, dilation_w=2)),
    ("pool+residual", NONE, WINOGRADF63, 16, dict(pool=1, residual=D, relu_after_add=1)),
    ("pool+dilation", NONE, SGECONV, 32, dict(pool=1, dilation_h=2, dilation_w=2)),
    ("pool+fused-residual", NONE, SGECONV, 32, dict(pool=1, residual=D)),
    ("bounds-without-clip", RELU, SGECONV, 16, dict(clip_min=0, clip_max=6)),
    ("nan-bound-without-clip", NONE, IM2COL, 16, dict(clip_min=NAN)),
]


@pytest.mark.parametrize("case", NOT_BUILT, ids=[c[0] for c in NOT_BUILT])
def test_opts_rejects_what_no_older_entry_point_could_express(case):
    from feathercnn_b200._lib import fcuda
    _, activation, algo, ch, okw = case
    p = _param(activation, ch)
    if okw.get("pool"):
        assert fcuda().fcuda_conv_can_pool(ctypes.byref(p), algo) == 1
    assert _call("opts", p, algo, _opts(**okw)) == -200
    assert _call("opts", p, algo, _opts(**okw), batch=0) == -200  # before the plan


# ---- the same bits through both doors --------------------------------------------------------------------------------
# (name, (oc, ic, h, w, k, stride, pad, group), algo, precision, the implicit-GEMM tile kernel the layer takes)
LAYERS = [
    ("winograd63", (32, 32, 20, 20, 3, 1, 1, 1), WINOGRADF63, 2, None),
    ("winograd23", (32, 32, 20, 20, 3, 1, 1, 1), WINOGRADF23, 2, None),
    ("im2col", (24, 16, 12, 12, 3, 2, 1, 1), IM2COL, 2, None),
    ("gather", (40, 64, 14, 14, 3, 2, 1, 1), SGECONV, 2, "gather"),
    ("halo", (40, 64, 16, 16, 3, 1, 1, 1), SGECONV, 0, "halo"),
    ("presplit", (32, 64, 16, 16, 3, 1, 1, 1), SGECONV, 2, "presplit"),
    ("wide", (64, 64, 56, 56, 3, 1, 1, 1), SGECONV, 2, "wide"),
    ("grouped", (32, 64, 10, 10, 3, 1, 1, 2), SGECONV, 2, None),
    ("depthwise", (32, 32, 56, 56, 3, 1, 1, 32), DEPTHWISE, 2, None),
    ("naive", (16, 16, 12, 12, 3, 1, 1, 1), NAIVE, 2, None),
]
# (name, entry, activation, options); the residual pointer is filled in by the test
VARIANTS = [
    ("plain", "forward", NONE, {}),
    ("relu", "forward", RELU, {}),
    ("clip", "clip", CLIP, dict(clip_min=-0.3, clip_max=0.25)),
    ("residual", "residual", NONE, dict(residual=True)),
    ("residual-relu", "residual", NONE, dict(residual=True, relu_after_add=1)),
    ("relu-residual-relu", "ext", RELU, dict(residual=True, relu_after_add=1, dilation_h=1, dilation_w=1)),
    ("pool", "pool", RELU, dict(pool=1)),
    ("dilation", "ext", RELU, dict(dilation_h=2, dilation_w=2)),
    ("dilation-residual", "ext", NONE, dict(residual=True, relu_after_add=1, dilation_h=2, dilation_w=2)),
]


@gpu
@pytest.mark.parametrize("layer", LAYERS, ids=[c[0] for c in LAYERS])
def test_opts_output_equals_the_older_entry_point(cuda, layer):
    torch = cuda
    from feathercnn_b200 import booster
    name, (oc, ic, h, w, k, s, pad, group), algo, precision, tile = layer
    booster.set_precision(precision)
    lib = booster.fcuda()
    rng = np.random.default_rng(oc * 131 + ic)
    x = torch.from_numpy(rng.uniform(-1, 1, (2, ic, h, w)).astype(np.float32)).cuda()
    wshape = (ic, 1, k, k) if algo == DEPTHWISE else (oc, ic // group, k, k)
    wt = torch.from_numpy((rng.standard_normal(wshape) / np.sqrt(np.prod(wshape[1:]))).astype(np.float32)).cuda()
    b = torch.from_numpy(rng.uniform(-0.2, 0.2, oc).astype(np.float32)).cuda()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ran = []
    for vname, entry, activation, okw in VARIANTS:
        p = booster.ConvParam.make(oc, ic, h, w, k, stride=s, pad=pad, group=group, bias=True)
        p.activation = activation
        dil = okw.get("dilation_h", 1)
        if dil > 1:
            if algo != SGECONV:
                continue
            p.output_h = (h + 2 * pad - dil * (k - 1) - 1) // s + 1
            p.output_w = (w + 2 * pad - dil * (k - 1) - 1) // s + 1
        elif tile is not None and vname == "plain":
            g = (ctypes.c_int * 4)()
            got = [n for n, f in (("halo", lib.fcuda_igemm_halo_tile), ("presplit", lib.fcuda_igemm_presplit_tile),
                                  ("wide", lib.fcuda_igemm_wide_tile)) if f(ctypes.byref(p), g)]
            assert (got[-1] if got else "gather") == tile, (name, got)
        if okw.get("pool") and not lib.fcuda_conv_can_pool(ctypes.byref(p), algo):
            continue
        cb = booster.ConvBooster()
        cb.ForceSelectAlgo(algo)
        scratch_n, packed_n = cb.GetBufferSize(p, 2)
        packed = torch.empty(max(packed_n, 1), device="cuda")
        scratch = torch.empty(max(scratch_n, 1), device="cuda")
        cb.Init(p, packed, wt)
        oh, ow = ((p.output_h + 1) // 2, (p.output_w + 1) // 2) if okw.get("pool") else (p.output_h, p.output_w)
        res = torch.from_numpy(rng.uniform(-1, 1, (2, oc, oh, ow)).astype(np.float32)).cuda()
        o = _opts(**dict(okw, residual=res.data_ptr() if okw.get("residual") else None))
        outs = []
        for e in (entry, "opts"):
            out = torch.full((2, oc, oh, ow), NAN, device="cuda")
            ptrs = tuple(ctypes.c_void_p(t.data_ptr()) for t in (out, x, packed, scratch, b))
            assert _call(e, p, algo, o, batch=2, ptrs=ptrs, stream=stream) == 0, (name, vname, e)
            outs.append(out)
        torch.cuda.synchronize()
        assert not torch.isnan(outs[0]).any(), (name, vname)
        assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), (name, vname)
        if vname == "plain":  # a NULL options pointer is the all-zero struct
            out = torch.full((2, oc, oh, ow), NAN, device="cuda")
            ptrs = tuple(ctypes.c_void_p(t.data_ptr()) for t in (out, x, packed, scratch, b))
            assert _call("opts", p, algo, None, batch=2, ptrs=ptrs, stream=stream) == 0
            torch.cuda.synchronize()
            assert torch.equal(outs[0].view(torch.int32), out.view(torch.int32)), name
        ran.append(vname)
    expect = [v[0] for v in VARIANTS if (algo == SGECONV or not v[0].startswith("dilation"))
              and (v[0] != "pool" or algo in (WINOGRADF63, WINOGRADF23) or tile in ("halo", "presplit", "wide"))]
    assert ran == expect, (name, ran)
