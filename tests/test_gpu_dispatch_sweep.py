"""Seeded random geometries across every convolution, depthwise and pooling kernel boundary, against float64.

The hand-written lists of test_gpu_error_bounds.py and test_gpu_layers.py sit where their authors expected trouble.  The
dispatch, though, picks a kernel from a dozen geometry predicates (conv_igemm.cu launch_conv and its *_geometry,
depthwise.cu dw_launch, layers.cu pooling_forward, the Winograd chunking of fcuda_api.cu), and a geometry one pixel, one
channel or one pad away from a listed case can take another kernel.  This sweep draws geometries biased to both sides of
every such predicate: one deterministic generator, each case seeded from the crc32 of its index.

Each convolution case runs the tuned choice plus every algorithm fcuda_conv_get_buffer_size accepts for it (those the
case's entry point allows: dilation is the implicit GEMM's, the fused pooling fcuda_conv_can_pool's), and is checked per
element with the bound of test_gpu_error_bounds.py:

    |got - ref| <= coef * S + 2^-23 |ref|,     coef = eps(path, mode) + K 2^-23   (Winograd: WINO_MARGIN * rho)

  - Clip: the clamp is 1-Lipschitz, so |clamp(got) - clamp(ref)| <= |got - ref|: the bound of the unclamped result
    (with its |ref| term) holds for the clamped one.
  - Fused 2x2 max pooling: the max of the window's bounds (as run_conv does).
  - Winograd: rho is the model's worst |d| / S_tile and the bound WINO_MARGIN * rho * S_tile, S_tile the maximum of S
    over the output tile.  The transforms mix a tile's outputs, so an output whose window lies wholly in a padding of 2
    or more (S = 0) still carries its neighbours' rounding; with S per element such an output would fail on a correct
    kernel.
  - Pooling layers against the float64 restatement of test_gpu_net_bounds.py (ceil mode, the window start subtracting
    both pads, average over the in-bounds elements): max pooling exactly, average pooling within one fp32 rounding of
    the running sum per add plus one for the division, n_adds 2^-23 sum|x| / cnt + 2^-23 |ref|.

Depthwise and pooling cases also run on views that start 0..3 floats past an aligned allocation (input and output
separately), through the C ABI: the vector kernels must then give way to the scalar ones.  The output view sits in a
NaN-filled buffer and the floats around it must stay NaN.

Every case is labelled with the kernel it reaches (the implicit-GEMM stem and tile queries for stem / gather / halo /
presplit / wide, a
restatement of dw_launch and of pooling_forward, the Winograd chunk plan); the CPU tests below check that the generated
list hits every reachable (kernel, epilogue, mode) cell and both sides of every predicate boundary, and that the checker
rejects simulated defects on the sweep's own shapes.  A failing case prints a ready-to-paste Conv(...) literal, to be
pinned into the matching hand-written list.

FCUDA_SWEEP_SCALE (a float, default 1) scales the case count.  Run with -s to print, per cell, the case count and the
largest share of the bound used.
"""
from __future__ import annotations

import ctypes
import dataclasses
import math
import os
import random
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_error_bounds import (DEPTHWISE, FP32_SPLIT, IM2COL, MODE_NAME, NAIVE, PATH, SGECONV, TF32, TF32X3, U,
                                   WINO_MARGIN, WINOGRADF23, WINOGRADF63, Conv, conv_ref, eps_for, excess, make_data, pool2,
                                   wino_model)
from test_gpu_net_bounds import pool_avg, pool_max

gpu = pytest.mark.gpu

N_CASES = 1200          # about 3200 kernel runs: 35 s on an H100 (80 GB)
SCALE = float(os.environ.get("FCUDA_SWEEP_SCALE", "1"))
CASES_RUN = max(1, int(round(N_CASES * SCALE)))

ALGOS = (NAIVE, IM2COL, SGECONV, DEPTHWISE, WINOGRADF63, WINOGRADF23)
MODES3 = (FP32_SPLIT, TF32X3, TF32)
EPILOGUES = ("none", "relu", "clip", "res", "res_relu", "pool")
OC_EDGES = (31, 32, 33, 63, 64, 65, 127, 128, 129)
HW_EDGES = (8, 9, 16, 17, 34, 35)
TAP_SHAPES = {1: [(1, 1)], 2: [(1, 2), (2, 1)], 4: [(2, 2), (1, 4)], 5: [(1, 5), (5, 1)], 9: [(3, 3)], 49: [(7, 7)],
              63: [(7, 9), (9, 7)]}


# ---- the generator ----------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    idx: int
    family: str
    mode: int
    conv: Conv | None = None
    pool: tuple | None = None        # (type, kh, kw, sh, sw, (pl, pr, pt, pb), global, (n, c, h, w))
    in_off: int = 0                  # float offsets of the input / output views (memory-bound kernels only)
    out_off: int = 0

    @property
    def name(self):
        return f"{self.idx:04d}-{self.family}"


def _pads(r, hi=3):
    return tuple(r.randint(0, hi) for _ in range(4))   # (left, bottom, right, top)


def _apply_epilogue(c: Conv, epi: str, r) -> Conv:
    if epi == "relu":
        c.relu = True
    elif epi == "clip":
        f32 = lambda v: float(np.float32(v))  # noqa: E731  (the kernels clamp to float32 bounds)
        c.clip = (v := f32(round(r.uniform(-0.2, 0.2), 3)), v) if r.random() < 0.25 else \
            (f32(-round(r.uniform(0.02, 0.3), 3)), f32(round(r.uniform(0.02, 0.3), 3)))
    elif epi in ("res", "res_relu"):
        c.res, c.relu_after_add = True, epi == "res_relu"
        # the convolution's own ReLU before the sum (unfused path; forward_ext takes none with dilation)
        c.relu = epi == "res" and c.dil == 1 and r.random() < 0.2
    elif epi == "pool":
        c.pool, c.relu = True, r.random() < 0.5
    return c


def _gen_igemm_halo(r, k, mode):
    """Stride 1, no dilation, more than one tap: the halo family.  In fp32split mode blocks of 18 cases alternate between
    geometries near the wide tile (28 rows, N tiles of 64 / 128), 49 / 63 taps with N tile 128 (the pre-split box does
    not fit shared memory: the halo kernel runs) and the general draw, which in the other modes also pushes W % 4 and
    IC % 32 off."""
    style = (k // 18) % 3 if mode == FP32_SPLIT else 2
    pool = EPILOGUES[k % len(EPILOGUES)] == "pool"     # the fused pooling takes 3x3 layers only
    ic = r.choice([32, 32, 64, 96])
    if style == 0:
        kh, kw = (3, 3) if pool else r.choice([(1, 5), (5, 1), (3, 3), (5, 5)])
        oc, h, w = r.choice(OC_EDGES[4:] + OC_EDGES[6:]), r.choice([27, 28, 28, 56]), r.choice([16, 28, 32, 56])
    elif style == 1:
        kh, kw = r.choice(TAP_SHAPES[49] + TAP_SHAPES[63])
        oc, h, w = r.choice(OC_EDGES[5:]), r.choice([9, 16, 17, 28]), r.choice([12, 16, 20])
    else:
        split = mode == FP32_SPLIT    # (aimed at the pre-split kernel)
        kh, kw = (3, 3) if pool else r.choice(TAP_SHAPES[r.choice([2, 4, 5, 9, 9, 9] + ([] if split else [49, 63]))])
        oc, h, w = r.choice(OC_EDGES), r.choice([8, 9, 16, 17, 27, 28, 29, 34, 35, 56]), r.choice([8, 12, 16, 20, 24, 32, 36])
        if not pool and not split and r.random() < 0.3:
            if r.random() < 0.5:
                w += r.randint(1, 3)
            else:
                ic = r.choice([31, 33, 65])
    pad = _pads(r, 2 if pool else 3) if r.random() < (0.2 if style == 0 else 0.5) else (kw // 2, kh // 2, kw // 2, kh // 2)
    return Conv("", oc, ic, max(h, kh), max(w, kw), kh, kw, pad=pad, batch=r.choice([1, 2, 3]))


def _gen_igemm_gather(r, k, mode):
    """Anything the implicit GEMM takes: strides, dilation, groups, IC % 32 in {0, 1, 31}, 1..63 taps, big pads."""
    taps = r.choice(list(TAP_SHAPES))
    kh, kw = r.choice(TAP_SHAPES[taps])
    group = r.choice([1, 1, 1, 2, 3, 4])
    # (IC per group 1 makes group == IC, which AssignOutputDim turns into a depthwise layer)
    icg = r.choice([2, 3, 5, 31, 32, 33, 64]) if taps * 33 <= 6144 else 32
    ocg = r.choice([1, 5, 16, 31, 32, 33]) if group > 1 else r.choice(OC_EDGES)
    sh, sw = r.choice([(1, 1), (2, 2), (1, 2), (2, 1), (2, 2)])
    dil = r.choice([1, 1, 1, 2, 3]) if taps > 1 else 1
    pad = _pads(r, 3) if r.random() < 0.7 else (0, 0, 0, 0)
    if kh * kw == 1 and r.random() < 0.5:
        pad = tuple(r.randint(2, 3) for _ in range(4))       # pad larger than the kernel
    h = max(r.choice(HW_EDGES + (5, 11)), dil * (kh - 1) + 1)
    w = max(r.choice(HW_EDGES + (5, 13)), dil * (kw - 1) + 1)
    return Conv("", ocg * group, icg * group, h, w, kh, kw, sh=sh, sw=sw, pad=pad, group=group, dil=dil,
                batch=r.choice([1, 2, 3, 5]))


def _gen_wino(r, k, mode):
    """3x3 / stride 1 / group 1 with IC % 4 == 0: both Winograd tiles, every other block of 18 cases with the smallest L2
    chunk on few channels and several tile rows (both tiles then run in several chunks)."""
    pad = r.choice([(1, 1, 1, 1), (0, 0, 0, 0), (1, 0, 1, 1), (1, 1, 0, 1)])
    if (k // 18) % 2:
        ic, oc = r.choice([4, 8, 12]), r.choice([4, 8, 12])
        return Conv("", oc, ic, r.choice([24, 25, 30]), r.choice([17, 24, 26]), 3, pad=pad, batch=r.choice([2, 3]), chunk=1)
    ic, oc = r.choice([4, 8, 12, 32, 36]), r.choice([8, 31, 32, 33, 64])
    return Conv("", oc, ic, r.choice([9, 12, 13, 17, 24, 25]), r.choice([9, 12, 13, 17, 24, 26]), 3, pad=pad,
                batch=r.choice([1, 2, 3]))


DW_K3_TARGETS = ("vec4", "vec2-s1", "vec2-s2", "shuffle-s1", "shuffle-s2")


def _gen_dw_k3(r, k, mode):
    """3x3 / pad 1 depthwise strips, aimed in turn at each strip kernel; every fourth block of 25 cases is pushed across
    the edges (OW at 23/24/25, 47/48/49, 95/96/97, odd W, pads right / bottom 0, pad top 0 / 2, offset views)."""
    target = DW_K3_TARGETS[(k // 5) % len(DW_K3_TARGETS)]
    edge = _dw_edge_block(k)
    s = 2 if target.endswith("s2") else 1
    ow = {"vec4": r.choice([96, 100, 128]), "vec2-s1": r.choice([48, 50, 64, 94]), "vec2-s2": r.choice([48, 50, 64]),
          "shuffle-s1": r.choice([24, 25, 33, 47, 95]), "shuffle-s2": r.choice([24, 25, 31, 47])}[target]
    pr, pb, pt = 1, 1, 1
    w = ow if s == 1 else 2 * ow
    if edge:
        ow += r.choice([-1, 0, 1])
        pr, pb = r.randint(0, 1), r.randint(0, 1)
        w = ow + (1 - pr) if s == 1 else 2 * ow - r.randint(0, 1)
        pt = 1 if r.random() < 0.7 else r.choice([0, 2])
    h = r.choice([3, 15, 16, 17, 33]) * s
    c = r.choice([2, 3, 5])
    return Conv("", c, c, h, w, 3, sh=s, pad=(1, pb, pr, pt), group=c, batch=r.choice([1, 2, 3, 5]))


def _dw_edge_block(k):
    return (k // 25) % 4 == 3


DW_SMALL_TARGETS = ("cols8", "cols16", "plane-s1", "plane-s2", "generic")


def _gen_dw_small(r, k, mode):
    """Small depthwise planes, aimed in turn at the column, plane and generic kernels: H, W at 8/9, 16/17, 34/35, pads
    0 / 1 / 2, equal and unequal strides, other kernel sizes."""
    target = DW_SMALL_TARGETS[(k // 5) % len(DW_SMALL_TARGETS)]
    c = r.choice([2, 3, 4, 7])
    kh, kw, sh, sw, pad = 3, 3, 1, 1, (1, 1, 1, 1)
    if target == "cols8":
        h, w = r.choice([1, 8, 9, 16]), r.choice([3, 7, 8])
    elif target == "cols16":
        h, w = r.choice([8, 9, 16]), r.choice([9, 15, 16])
    elif target == "plane-s1":
        h, w = r.choice([8, 17, 33, 34]), r.choice([17, 23, 34])
        pad = (1, 1, 1, 1) if r.random() < 0.5 else (r.randint(0, 1), r.randint(0, 1), r.randint(0, 1), r.randint(0, 1))
    elif target == "plane-s2":
        sh = sw = 2
        h, w = r.choice([8, 9, 16, 17, 34]), r.choice([8, 9, 17, 34])
        pad = (r.randint(0, 1), r.randint(0, 1), r.randint(0, 1), r.randint(0, 1))
    else:
        h, w = r.choice(HW_EDGES + (7, 15)), r.choice(HW_EDGES + (7, 15))
        how = r.randrange(4)
        if how == 0:
            kh, kw = r.choice([(5, 5), (3, 1), (1, 3), (2, 2)])
            pad = _pads(r, 2)
        elif how == 1:
            sh, sw = r.choice([(1, 2), (2, 1)])
        elif how == 2:
            pad = (2, 2, 2, 2) if r.random() < 0.5 else (1, 1, 1, 2)
        else:
            h, w = r.choice([(35, 20), (20, 35), (35, 35)])
    return Conv("", c, c, max(h, kh), max(w, kw), kh, kw, sh=sh, sw=sw, pad=pad, group=c, batch=r.choice([1, 2, 3, 5]))


POOL_KINDS = ("global", "2x2", "3x3s2", "generic")


def _gen_pool(r, k, mode):
    """Aimed in turn at each pooling kernel (max and average), then pushed across its edges."""
    n, c = r.choice([1, 2, 3]), r.choice([1, 3, 4])
    t, kind = k % 2, POOL_KINDS[(k // 2) % len(POOL_KINDS)]
    if kind == "global":
        return (t, 0, 0, 1, 1, (0, 0, 0, 0), True, (n, c, r.choice([1, 3, 7, 9]), r.choice([1, 5, 7, 33])))
    if kind == "2x2":
        return (t, 2, 2, 2, 2, (0, 0, 0, 0), False,
                (n, c, r.choice([2, 6, 10, 10, 7]), r.choice([4, 8, 12, 64, 64, 66]) + (0 if r.random() < 0.8 else 1)))
    if kind == "3x3s2":
        ow = r.choice([24, 25, 33, 23])
        return (t, 3, 3, 2, 2, (0, 0, 0, 0), False, (n, c, r.choice([5, 20, 33, 34]), 2 * ow + r.choice([0, 0, 1, -1])))
    kh, kw = r.randint(1, 4), r.randint(1, 4)
    sh, sw = r.randint(1, kh), r.randint(1, kw)
    pl, pr = (r.randint(0, kw - 1), 0) if r.random() < 0.5 else (0, r.randint(0, kw - 1))
    pt, pb = (r.randint(0, kh - 1), 0) if r.random() < 0.5 else (0, r.randint(0, kh - 1))
    # pads of an axis sum below the kernel and stride <= kernel: no window lies wholly outside the image
    return (t, kh, kw, sh, sw, (pl, pr, pt, pb), False, (n, c, r.randint(kh, 20), r.randint(kw, 40)))


GENERATORS = {"halo": _gen_igemm_halo, "gather": _gen_igemm_gather, "wino": _gen_wino, "dw_k3": _gen_dw_k3,
              "dw_small": _gen_dw_small, "pool": _gen_pool}
SLOTS = ["halo", "wino", "dw_k3", "halo", "dw_small", "pool", "wino", "halo", "dw_k3", "gather", "halo", "wino", "dw_k3",
         "dw_small", "pool"]


def _offsets(r, p):
    """(input, output) float offsets of the views: nonzero with probability p."""
    return (r.randint(0, 3), r.randint(0, 3)) if r.random() < p else (0, 0)


def gen_case(i: int) -> Case:
    """Case i.  k counts the cases of its family: the epilogue cycles with k, the mode with k // 6 (every combination
    in 18 cases), and the depthwise and pooling families aim at their kernels in turn."""
    r = random.Random(zlib.crc32(f"dispatch-sweep-{i}".encode()))
    fam = SLOTS[i % len(SLOTS)]
    k = i // len(SLOTS) * SLOTS.count(fam) + SLOTS[:i % len(SLOTS)].count(fam)
    mode = MODES3[(k // len(EPILOGUES)) % 3]
    if fam == "pool":
        return Case(i, fam, FP32_SPLIT, pool=_gen_pool(r, k, mode), **dict(zip(("in_off", "out_off"), _offsets(r, 0.3))))
    c = GENERATORS[fam](r, k, mode)
    c.bias = r.random() < 0.8
    c.name = f"sweep{i}"
    allowed = [e for e in EPILOGUES if epilogue_possible(c, e)]
    c = _apply_epilogue(c, allowed[k % len(allowed)] if r.random() < 0.85 else r.choice(allowed), r)
    case = Case(i, fam, mode, conv=c)
    if c.depthwise:
        case.in_off, case.out_off = _offsets(r, (0.8 if _dw_edge_block(k) else 0.0) if fam == "dw_k3" else 0.25)
    return case


# ---- what runs where ---------------------------------------------------------------------------------------------------
def _lib():
    from feathercnn_b200._lib import fcuda
    return fcuda()


def conv_param(c: Conv):
    from feathercnn_b200 import booster
    p = booster.ConvParam.make(c.oc, c.ic, c.h, c.w, c.kh, c.kw, stride=c.sh, stride_w=c.sw, pad_lbrt=c.pad, group=c.group,
                               bias=c.bias, relu=c.relu)
    p.output_h, p.output_w = c.out_hw
    return p


def _accepts(c: Conv, algo: int) -> bool:
    s, k = ctypes.c_size_t(), ctypes.c_size_t()
    return _lib().fcuda_conv_get_buffer_size(ctypes.byref(conv_param(c)), algo, c.batch, ctypes.byref(s), ctypes.byref(k)) == 0


def tuned_algo(c: Conv) -> int:
    a = ctypes.c_int(-1)
    _lib().fcuda_conv_select_algo_tuned(ctypes.byref(conv_param(c)), ctypes.byref(a))
    return a.value


def algos_for(c: Conv, in_off=0, out_off=0) -> list[int]:
    """The algorithms a case runs: every one the buffer-size query accepts and the case's entry point allows."""
    if in_off or out_off:     # offset views are for the memory-bound depthwise kernels only
        return [DEPTHWISE] if _accepts(c, DEPTHWISE) else []
    out = []
    for a in ALGOS:
        if not _accepts(c, a):
            continue
        if c.dil > 1 and a != SGECONV:
            continue                                      # fcuda_conv_forward_ext: the implicit GEMM spaces its taps
        if c.pool and not _lib().fcuda_conv_can_pool(ctypes.byref(conv_param(c)), a):
            continue
        out.append(a)
    return out


def epilogue_possible(c: Conv, epi: str) -> bool:
    if c.dil > 1:
        return epi in ("none", "relu", "res", "res_relu")  # forward_ext: no clamp bounds, no pooling
    if epi == "pool":
        return bool(algos_for(dataclasses.replace(c, pool=True)))
    return True


def epilogue_of(c: Conv) -> str:
    if c.pool:
        return "pool"
    if c.clip is not None:
        return "clip"
    if c.res:
        return "res_relu" if c.relu_after_add else "res"
    return "relu" if c.relu else "none"


def _set_mode(mode):
    _lib().fcuda_set_precision(mode)


def igemm_kernel(c: Conv, mode: int) -> str:
    """stem / gather / halo / presplit / wide from the queries of the per-group problem in `mode`, in launch_conv's
    order: the stem query (with the case's residual, pooling and dilation), then the tile queries."""
    from feathercnn_b200._lib import FcudaConvOptions
    lib, p, g = _lib(), conv_param(c), (ctypes.c_int * 4)()
    old = lib.fcuda_get_precision()
    _set_mode(mode)
    try:
        o = FcudaConvOptions(residual=1 if c.res else None, pool=int(c.pool), dilation_h=c.dil, dilation_w=c.dil)
        if lib.fcuda_igemm_stem_supported(ctypes.byref(p), ctypes.byref(o)):
            return "stem"
        if c.dil > 1:
            return "gather"      # the tile queries do not see dilation; halo_geometry rejects it
        if lib.fcuda_igemm_wide_tile(ctypes.byref(p), g):
            return "wide"
        if lib.fcuda_igemm_presplit_tile(ctypes.byref(p), g):
            return "presplit"
        return "halo" if lib.fcuda_igemm_halo_tile(ctypes.byref(p), g) else "gather"
    finally:
        _set_mode(old)


def dw_kernel(c: Conv, in_off=0, out_off=0) -> str:
    """depthwise.cu dw_launch (switch dw_vec on), including the alignment of the input / output views."""
    oh, ow = c.out_hw
    pl, pb, pr, pt = c.pad
    ia, oa = 4 * in_off, 4 * out_off    # bytes past a 256-byte-aligned allocation
    k3 = c.kh == 3 and c.kw == 3 and pt == 1 and pl == 1 and c.sh == c.sw and c.sh in (1, 2) and ow >= 24
    if k3:
        if c.sh == 1 and ow == c.w:
            if c.w % 4 == 0 and ow >= 96 and (ia | oa) % 16 == 0:
                return "vec4"
            if c.w % 2 == 0 and ow >= 48 and (ia | oa) % 8 == 0:
                return "vec2-s1"
        elif c.sh == 2 and c.w == 2 * ow and c.w % 4 == 0 and ow >= 48 and ia % 16 == 0 and oa % 8 == 0:
            return "vec2-s2"
        return f"shuffle-s{c.sh}"
    if c.kh == 3 and c.kw == 3 and pt == 1 and pl == 1 and c.sh == 1 and c.sw == 1 and c.h <= 16 and c.w <= 16 and \
            oh == c.h and ow == c.w:
        return "cols8" if c.w <= 8 else "cols16"
    if c.kh == 3 and c.kw == 3 and pt in (0, 1) and pl in (0, 1) and c.sh == c.sw and c.sh in (1, 2) and c.h <= 34 and \
            c.w <= 34 and (oh - 1) * c.sh - pt + 2 <= c.h and (ow - 1) * c.sw - pl + 2 <= c.w:
        return f"plane-s{c.sh}"
    return "generic"


def wino_chunked(c: Conv, algo: int, mode: int) -> bool:
    """fcuda_api.cu make_plan: more than one chunk of tile rows."""
    t = 8 if algo == WINOGRADF63 else 4
    oh, ow = c.out_hw
    tiles_x, tiles_y = -(-ow // (t - 2)), -(-oh // (t - 2))
    total = c.batch * tiles_y
    np_ = 1 if mode == TF32 else 2
    per_row = tiles_x * t * t * (c.ic + c.oc) * 4
    budget = c.chunk if c.chunk else 8 << 30
    budget = max(budget, 2 * np_ * t * t * c.ic * c.oc * 4)
    return max(1, budget // per_row) < total


def kernel_label(case: Case, algo: int) -> str:
    c = case.conv
    if algo == SGECONV:
        return igemm_kernel(c, case.mode)
    if algo == DEPTHWISE:
        return "dw-" + dw_kernel(c, case.in_off, case.out_off)
    if algo in (WINOGRADF63, WINOGRADF23):
        return PATH[algo] + ("-chunked" if wino_chunked(c, algo, case.mode) else "")
    return PATH[algo]


def pool_geometry(pc):
    t, kh, kw, sh, sw, (pl, pr, pt, pb), glob, (n, ch, h, w) = pc
    if glob:
        return h, w, 1, 1, 1, 1
    lib = _lib()
    return kh, kw, lib.fcuda_pooling_out_dim(h, pt, pb, kh, sh), lib.fcuda_pooling_out_dim(w, pl, pr, kw, sw), sh, sw


def pool_kernel(pc, in_off=0, out_off=0) -> str:
    """layers.cu pooling_forward, including the alignment of the views."""
    t, _, _, _, _, (pl, pr, pt, pb), glob, (n, ch, h, w) = pc
    kh, kw, oh, ow, sh, sw = pool_geometry(pc)
    ia, oa = 4 * in_off, 4 * out_off
    nopad = pl + pr == 0 and pt + pb == 0
    if oh == 1 and ow == 1 and kh >= h and kw >= w and nopad:
        return "global"
    if kh == kw == 2 and sh == sw == 2 and nopad and w % 4 == 0 and h % 2 == 0 and ow == w // 2 and oh == h // 2 and \
            ia % 16 == 0 and oa % 8 == 0:
        return "2x2"
    if kh == kw == 3 and sh == sw == 2 and nopad and w % 2 == 0 and ow >= 24 and 2 * (ow - 1) < w and 2 * (oh - 1) < h \
            and ia % 8 == 0:
        return "3x3s2"
    return "generic"


# mode does not change these kernels' arithmetic (fp32 FMA / compare / add); their cells are mode-independent
MODE_FREE = ("naive", "dw-", "pool-")


def runs_of(case: Case) -> list[tuple[int, str, str, str]]:
    """(algo, kernel, epilogue, mode) of every run of a case; algo -1 for a pooling layer."""
    if case.pool is not None:
        return [(-1, "pool-" + pool_kernel(case.pool, case.in_off, case.out_off), "max" if case.pool[0] == 0 else "avg",
                 "any")]
    c = case.conv
    out = []
    for a in algos_for(c, case.in_off, case.out_off):
        k = kernel_label(case, a)
        out.append((a, k, epilogue_of(c), "any" if k.startswith(MODE_FREE) else MODE_NAME[case.mode]))
    return out


@dataclasses.dataclass
class Sweep:
    cases: list
    runs: list        # (case, algo, kernel, epilogue, mode)


_SWEEP = None


def sweep() -> Sweep:
    global _SWEEP
    if _SWEEP is None:
        cases = [gen_case(i) for i in range(CASES_RUN)]
        _SWEEP = Sweep(cases, [(cs, *r) for cs in cases for r in runs_of(cs)])
    return _SWEEP


def literal(c: Conv) -> str:
    """A ready-to-paste Conv(...) for a hand-written list."""
    d = Conv("x", 1, 1, 1, 1)
    kw = [f"{f.name}={getattr(c, f.name)!r}" for f in dataclasses.fields(Conv)[5:]
          if getattr(c, f.name) != getattr(d, f.name) and f.name not in ("algo",)]
    return f"Conv({c.name!r}, {c.oc}, {c.ic}, {c.h}, {c.w}" + "".join(", " + k for k in kw) + ")"


# ---- the checker -------------------------------------------------------------------------------------------------------
def wino_tile(algo: int) -> int:
    """Output tile edge of a Winograd algorithm, 0 for the others."""
    return {WINOGRADF63: 6, WINOGRADF23: 2}.get(algo, 0)


def tile_max(s, m: int):
    """S replaced by its maximum over each m x m output tile (tiles start at the origin): the Winograd transforms mix
    the outputs of a tile, so an output's rounding error scales with the tile's S, not its own (an output whose window
    lies wholly in the padding, S = 0, still receives its neighbours' rounding)."""
    if not m:
        return s
    oh, ow = s.shape[-2:]
    t = F.max_pool2d(s, m, m, ceil_mode=True)
    return t.repeat_interleave(m, -2).repeat_interleave(m, -1)[..., :oh, :ow]


def conv_coef(c: Conv, algo: int, mode: int, x, w, b) -> float:
    if algo not in (WINOGRADF63, WINOGRADF23):
        return eps_for(PATH[algo], mode) + c.K * U
    # the Winograd model's worst |d| / tile_max(S) on the first images, before any epilogue
    n0 = min(c.batch, 2)
    plain = dataclasses.replace(c, relu=False, clip=None, res=False, pool=False)
    ym = wino_model(plain, x[:n0], w, b, 8 if algo == WINOGRADF63 else 4, mode)
    want = conv_ref(plain, x[:n0], w, b, None)
    s = tile_max(conv_ref(plain, x[:n0], w, b, None, absolute=True), wino_tile(algo))
    _, rho = excess(ym, want, s, 1.0)
    return WINO_MARGIN * rho


def conv_expect(c: Conv, x, w, b, r, coef: float, tile: int = 0):
    """(ref, per-element bound, S) of case c in float64.  The bound is that of the result before the clamp; `tile` > 0
    (Winograd) takes S per output tile (tile_max)."""
    free = conv_ref(dataclasses.replace(c, clip=None), x, w, b, r)
    s = conv_ref(c, x, w, b, r, absolute=True)
    if tile:
        s = tile_max(conv_ref(dataclasses.replace(c, res=False), x, w, b, None, absolute=True), tile) + \
            (r.double().abs() if r is not None else 0.0)
    bound = coef * s + U * free.abs()
    ref = free.clamp(*c.clip) if c.clip is not None else free
    if c.pool:
        ref, s, bound = pool2(ref), pool2(s), pool2(bound)
    return ref, bound, s


def check_conv(got, ref, bound, s) -> tuple[float, float]:
    """(share of the bound used, worst |d|/S)."""
    used, _ = excess(got, ref, bound, 1.0, 0.0)
    _, rel = excess(got, ref, s, 1.0, 0.0)
    return used, rel


def _pool_layer(pc):
    t, kh, kw, sh, sw, (pl, pr, pt, pb), glob, _ = pc
    return {"type": "Pooling", "name": "p",
            "params": {0: t, 1: kw, 11: kh, 2: sw, 12: sh, 3: pl, 14: pr, 13: pt, 15: pb, 4: int(glob)}}


def pool_expect(pc, x, kernel: str):
    """(ref, bound) of a pooling case: max exact; average one rounding per add of the kernel's summation plus the
    division."""
    L = _pool_layer(pc)
    if pc[0] == 0:
        ref = pool_max(x, L)
        return ref, torch.zeros_like(ref)
    ref, cnt = pool_avg(x, L)
    s = pool_avg(x.abs(), L)[0]
    if kernel == "pool-global":
        adds = -(-x.shape[2] * x.shape[3] // 32) + 4          # per-lane running sum, then five shuffle levels
    else:
        adds = cnt - 1
    return ref, adds * U * s + U * ref.abs()


def check_pool(got, ref, bound) -> float:
    d = (got - ref).abs()
    if not torch.isfinite(got).all():
        return math.inf
    return float(torch.where(d == 0, torch.zeros_like(d), d / bound.clamp_min(1e-300)).max())


# ---- report ------------------------------------------------------------------------------------------------------------
REPORT: dict[tuple[str, str, str], list] = {}


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\ncases and the largest share of the per-element bound used, per (kernel, epilogue, mode):")
        for (k, e, m), (n, used) in sorted(REPORT.items()):
            print(f"  {k:18s} {e:9s} {m:9s} {n:4d} cases   bound used {used:.3f}")


def _record(kernel, epi, mode, used):
    r = REPORT.setdefault((kernel, epi, mode), [0, 0.0])
    r[0] += 1
    r[1] = max(r[1], used)


# ---- running a case on the GPU -----------------------------------------------------------------------------------------
def _view(n: int, off: int, fill=None, src=None):
    """n floats starting `off` floats into a larger allocation (and that allocation)."""
    buf = torch.full((n + 8,), math.nan, device="cuda") if fill is None else torch.zeros(n + 8, device="cuda")
    v = buf[off:off + n]
    if src is not None:
        v.copy_(src.reshape(-1))
    return v, buf


def _guard_ok(buf, off, n) -> bool:
    return bool(torch.isnan(buf[:off]).all() and torch.isnan(buf[off + n:]).all())


def forward_conv_case(case: Case, algo: int):
    """Runs case on `algo` through its entry point; returns (x, w, b, r, the output (N, OC, OH, OW), guard ok)."""
    from feathercnn_b200 import booster
    c, mode = case.conv, case.mode
    booster.set_precision(mode)
    x, w, b, r = make_data(c, "cuda")
    p = conv_param(c)
    if c.clip is not None:
        p.activation = booster.ACT_CLIP
    cb = booster.ConvBooster()
    cb.ForceSelectAlgo(algo)
    n = c.batch
    lib = booster.fcuda()
    default_chunk = lib.fcuda_get_l2_chunk_bytes()
    if c.chunk:
        booster.set_l2_chunk_bytes(c.chunk)
    try:
        scratch_n, packed_n = cb.GetBufferSize(p, n)
        packed = torch.empty(max(packed_n, 1), device="cuda")
        scratch = torch.empty(max(scratch_n, 1), device="cuda")
        cb.Init(p, packed, w.contiguous())
        oh, ow = c.out_hw
        if c.pool:
            oh, ow = (oh + 1) // 2, (ow + 1) // 2
        n_out = n * c.oc * oh * ow
        xin, _ = _view(x.numel(), case.in_off, fill=0.0, src=x)
        out, obuf = _view(n_out, case.out_off)
        P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        args = (ctypes.byref(p), algo, P(out), P(xin), P(packed), P(scratch), P(b))
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if c.pool:
            rc = lib.fcuda_conv_forward_pool(*args, n, st)
        elif c.dil > 1:
            rc = lib.fcuda_conv_forward_ext(*args, P(r), int(c.relu_after_add), c.dil, c.dil, n, st)
        elif c.clip is not None:
            rc = lib.fcuda_conv_forward_clip(*args, float(c.clip[0]), float(c.clip[1]), n, st)
        elif c.res:
            rc = lib.fcuda_conv_forward_residual(*args, P(r), int(c.relu_after_add), n, st)
        else:
            rc = lib.fcuda_conv_forward(*args, n, st)
        torch.cuda.synchronize()
    finally:
        booster.set_l2_chunk_bytes(default_chunk)
    assert rc == 0, (booster.ALGO_NAMES[algo], rc)
    return x, w, b, r, out.view(n, c.oc, oh, ow), _guard_ok(obuf, case.out_off, n_out)


def run_conv_case(case: Case, algo: int):
    c, mode = case.conv, case.mode
    x, w, b, r, got, guard = forward_conv_case(case, algo)
    coef = conv_coef(c, algo, mode, x, w, b)
    ref, bound, s = conv_expect(c, x, w, b, r, coef, wino_tile(algo))
    used, rel = check_conv(got, ref, bound, s)
    if not torch.isfinite(got).all():
        used = math.inf
    return used, guard


def run_pool_case(case: Case):
    from feathercnn_b200._lib import fcuda
    t, kh, kw, sh, sw, (pl, pr, pt, pb), glob, (n, ch, h, w) = case.pool
    _, _, oh, ow, _, _ = pool_geometry(case.pool)
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(case.name.encode()))
    x = torch.rand((n, ch, h, w), generator=g, device="cuda") * 2 - 1
    if case.idx % 3 == 0:
        x = x - 1.5            # every value negative: a window that counted a padding 0 would show
    xin, _ = _view(x.numel(), case.in_off, fill=0.0, src=x)
    n_out = n * ch * oh * ow
    out, obuf = _view(n_out, case.out_off)
    rc = fcuda().fcuda_pooling_forward(ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(xin.data_ptr()), ch, h, w, t, kh, kw,
                                       sh, sw, pl, pr, pt, pb, int(glob), n, None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    kernel = pool_kernel(case.pool, case.in_off, case.out_off)
    ref, bound = pool_expect(case.pool, x.double(), "pool-" + kernel)
    return check_pool(out.view(n, ch, oh, ow).double(), ref, bound), _guard_ok(obuf, case.out_off, n_out)


def _ids():
    return [cs.name for cs in (gen_case(i) for i in range(CASES_RUN))]


@gpu
@pytest.mark.parametrize("i", range(CASES_RUN), ids=_ids())
def test_dispatch_sweep(cuda, i):
    case = sweep().cases[i]
    if case.pool is not None:
        (algo, kernel, epi, mode), = runs_of(case)
        used, guard = run_pool_case(case)
        _record(kernel, epi, mode, used)
        assert used <= 1.0 and guard, (case.name, kernel, case.pool, case.in_off, case.out_off, used, guard)
        return
    failures = []
    for algo, kernel, epi, mode in runs_of(case):
        used, guard = run_conv_case(case, algo)
        _record(kernel, epi, mode, used)
        if not (used <= 1.0 and guard):
            failures.append(f"{PATH[algo]} ({kernel}, {MODE_NAME[case.mode]}): bound used {used:.3g}, guard {guard}")
    assert not failures, (f"{literal(case.conv)}  # offsets in / out {case.in_off} / {case.out_off}\n  " +
                          "\n  ".join(failures))


# ---- coverage of the generated list (CPU) ------------------------------------------------------------------------------
# cells that cannot occur:
#   - the gathering implicit GEMM with a fused pool: fcuda_conv_can_pool's layers (3x3, stride 1, IC % 32 == 0, W % 4 == 0)
#     all fit the halo kernel, which takes them;
#   - presplit / wide outside fp32split: both read the BF16x3 split planes (wide with Clip in TF32 is one of these);
#     halo in fp32split only where the pre-split box does not fit shared memory (49 / 63 taps, N tile 128), so never with
#     the fused pool, which needs 3x3 taps;
#   - im2col / naive / depthwise with a fused pool (fcuda_conv_forward_pool rejects them);
#   - naive and depthwise in a given mode: fp32 FMA kernels, mode-independent ("any").
#   - stem outside fp32split (it reads the BF16x3 split planes), and with a residual or pool: fcuda_igemm_stem_supported
#     rejects both (the kernel fuses neither), and res / res_relu carry a residual;
EXPECTED_CELLS = (
    [("gather", e, m) for e in EPILOGUES if e != "pool" for m in MODE_NAME.values()]
    + [("stem", e, "fp32split") for e in ("none", "relu", "clip")]
    + [("halo", e, m) for e in EPILOGUES for m in MODE_NAME.values() if (e, m) != ("pool", "fp32split")]
    + [(k, e, "fp32split") for k in ("presplit", "wide") for e in EPILOGUES]
    + [(k, e, m) for k in ("f63", "f63-chunked", "f23", "f23-chunked") for e in EPILOGUES for m in MODE_NAME.values()]
    + [("im2col", e, m) for e in EPILOGUES if e != "pool" for m in MODE_NAME.values()]
    + [("naive", e, "any") for e in EPILOGUES if e != "pool"]
    + [("dw-" + k, e, "any") for k in ("vec4", "vec2-s1", "vec2-s2", "shuffle-s1", "shuffle-s2", "cols8", "cols16",
                                       "plane-s1", "plane-s2", "generic") for e in EPILOGUES if e != "pool"]
    + [("pool-" + k, t, "any") for k in ("global", "2x2", "3x3s2", "generic") for t in ("max", "avg")]
)


def test_sweep_hits_every_cell():
    pytest.importorskip("feathercnn_b200._lib")
    cells: dict = {}
    for cs, algo, kernel, epi, mode in sweep().runs:
        cells[(kernel, epi, mode)] = cells.get((kernel, epi, mode), 0) + 1
    idle = [cs.name for cs in sweep().cases if not runs_of(cs)]
    assert not idle, f"cases no algorithm runs: {idle}"
    # the tuned choice (what feather::Net runs) is among the algorithms of every case whose entry point it serves
    untuned = [cs.name for cs in sweep().cases if cs.conv is not None and cs.conv.dil == 1 and not cs.conv.pool and
               not cs.in_off and not cs.out_off and tuned_algo(cs.conv) not in algos_for(cs.conv)]
    assert not untuned, untuned
    unexpected = sorted(set(cells) - set(EXPECTED_CELLS))
    assert not unexpected, f"cells the coverage table says cannot occur: {unexpected}"
    if SCALE < 1:
        pytest.skip("a scaled-down sweep need not cover every cell")
    thin = sorted((cell, cells.get(cell, 0)) for cell in EXPECTED_CELLS if cells.get(cell, 0) < 3)
    assert not thin, f"cells hit fewer than 3 times: {thin}"


def _both(values, pred) -> bool:
    vs = list(values)
    return any(pred(v) for v in vs) and any(not pred(v) for v in vs)


def test_sweep_covers_both_sides_of_every_boundary():
    pytest.importorskip("feathercnn_b200._lib")
    if SCALE < 1:
        pytest.skip("a scaled-down sweep need not cover every boundary")
    S = sweep()
    convs = [cs.conv for cs in S.cases if cs.conv is not None]
    igemm = [cs.conv for cs, algo, *_ in S.runs if algo == SGECONV]
    dw = [(cs.conv, cs.in_off, cs.out_off) for cs, algo, *_ in S.runs if algo == DEPTHWISE]
    pools = [cs for cs in S.cases if cs.pool is not None]
    have = lambda vals, want: set(want) <= set(vals)  # noqa: E731
    assert have((c.w % 4 for c in igemm), range(4))
    assert have((c.ic // c.group % 32 for c in igemm), (0, 1, 31))
    assert have((c.kh * c.kw for c in igemm), (1, 2, 4, 5, 9, 49, 63))
    assert have((c.oc // c.group for c in igemm), OC_EDGES)
    assert have((c.out_hw[1] for c, *_ in dw), (23, 24, 25, 47, 48, 95, 96))
    assert have((c.w for c, *_ in dw), (8, 9, 16, 17, 34, 35)) and have((c.h for c, *_ in dw), (8, 9, 16, 17, 34, 35))
    assert have((c.w % 4 for c, *_ in dw), range(4))
    assert have((p for c in convs for p in c.pad), range(4))
    assert any(max(c.pad) > max(c.kh, c.kw) for c in convs)                            # pad larger than the kernel
    assert any(c.pad[0] != c.pad[2] or c.pad[1] != c.pad[3] for c in convs)             # asymmetric
    assert have(((c.sh, c.sw) for c in convs), ((1, 1), (2, 2), (1, 2), (2, 1)))
    assert have((c.dil for c in igemm), (1, 2, 3))
    assert _both(convs, lambda c: c.group > 1 and not c.depthwise)
    assert have((c.batch for c in convs), (1, 2, 3, 5))
    assert _both(convs, lambda c: c.bias)
    assert _both((c for c in convs if c.clip), lambda c: c.clip[0] == c.clip[1])
    assert all(c.clip[0] <= 0 <= c.clip[1] or c.clip[0] == c.clip[1] for c in convs if c.clip)
    assert _both((c for c in convs if c.res), lambda c: c.relu_after_add)
    assert have((cs.mode for cs in S.cases if cs.conv is not None), MODES3)
    # the views: offsets 0..3 on input and output, and the vector kernels' geometry on misaligned views
    assert have((i for _, i, _ in dw), range(4)) and have((o for _, _, o in dw), range(4))
    assert have((cs.in_off for cs in pools), range(4)) and have((cs.out_off for cs in pools), range(4))
    vec_geom = [(c, i, o) for c, i, o in dw if dw_kernel(c).startswith("vec")]
    assert any(dw_kernel(c, i, o).startswith("shuffle") for c, i, o in vec_geom)       # misaligned: the scalar strip kernel
    for k in ("2x2", "3x3s2"):
        geom = [cs for cs in pools if pool_kernel(cs.pool) == k]
        assert any(pool_kernel(cs.pool, cs.in_off, cs.out_off) == "generic" for cs in geom), k
    assert _both((cs for cs in S.cases if cs.family == "wino"), lambda cs: cs.conv.chunk is not None)


# ---- the checker bites (CPU) -------------------------------------------------------------------------------------------
def _sweep_convs(pred, n=4):
    out = [cs.conv for cs in (gen_case(i) for i in range(N_CASES)) if cs.conv is not None and pred(cs.conv)]
    assert len(out) >= n, len(out)
    return [dataclasses.replace(c, batch=min(c.batch, 2)) for c in out[:n]]


def _tf32_coef(c):
    return eps_for("sgeconv", TF32) + c.K * U        # the loosest convolution bound of the shape


CLIP_SHAPES = _sweep_convs(lambda c: c.clip is not None and c.clip[0] < c.clip[1] and c.bias and not c.pool and
                           c.oc * c.out_hw[0] * c.out_hw[1] < 40000)
RES_SHAPES = _sweep_convs(lambda c: c.res and c.relu_after_add and not c.relu and c.oc * c.out_hw[0] * c.out_hw[1] < 40000)
SEAM_SHAPES = _sweep_convs(lambda c: c.depthwise and not c.relu and c.clip is None and not c.relu_after_add and
                          dw_kernel(c).startswith(("vec", "shuffle")) and c.out_hw[1] > 32 * (
    4 if dw_kernel(c) == "vec4" else 2 if dw_kernel(c).startswith("vec2") else 1))


def _accepts_good(c, ref, bound, s):
    assert check_conv(ref, ref, bound, s)[0] == 0.0


@pytest.mark.parametrize("c", CLIP_SHAPES, ids=[c.name for c in CLIP_SHAPES])
def test_checker_rejects_clamp_before_bias(c):
    x, w, b, r = make_data(c, "cpu")
    ref, bound, s = conv_expect(c, x, w, b, r, _tf32_coef(c))
    _accepts_good(c, ref, bound, s)
    nob = dataclasses.replace(c, bias=False)
    bad = conv_ref(nob, x, w, None, r) + b.double().view(1, -1, 1, 1)   # clamp(conv) + bias
    assert check_conv(bad, ref, bound, s)[0] > 1.0


@pytest.mark.parametrize("c", RES_SHAPES, ids=[c.name for c in RES_SHAPES])
def test_checker_rejects_residual_added_after_the_clamp(c):
    x, w, b, r = make_data(c, "cpu")
    ref, bound, s = conv_expect(c, x, w, b, r, _tf32_coef(c))
    _accepts_good(c, ref, bound, s)
    bad = conv_ref(dataclasses.replace(c, res=False, relu=True), x, w, b, None) + r.double()   # relu(conv) + residual
    if c.pool:
        bad = pool2(bad)
    assert check_conv(bad, ref, bound, s)[0] > 1.0


@pytest.mark.parametrize("c", SEAM_SHAPES, ids=[c.name for c in SEAM_SHAPES])
def test_checker_rejects_depthwise_column_shift_at_a_strip_seam(c):
    x, w, b, r = make_data(c, "cpu")
    ref, bound, s = conv_expect(c, x, w, b, r, eps_for("depthwise", FP32_SPLIT) + c.K * U)
    _accepts_good(c, ref, bound, s)
    k = dw_kernel(c)
    seam = 32 * (4 if k == "vec4" else 2 if k.startswith("vec2") else 1)
    bad = ref.clone()
    bad[..., seam:] = ref[..., seam - 1:-1]       # the strip from the seam on reads one column to the left
    assert check_conv(bad, ref, bound, s)[0] > 1.0


def _clipped_window(pc) -> bool:
    """Some window of the pooling reaches past the image (padding, or ceil mode's last window)."""
    t, kh, kw, *_ = pc
    if pc[6]:
        return False
    n, ch, h, w = pc[7]
    cnt = pool_avg(torch.ones((1, 1, h, w), dtype=torch.float64), _pool_layer(pc))[1]
    return bool(cnt.min() < kh * kw)


POOL_SHAPES = [cs for cs in (gen_case(i) for i in range(N_CASES)) if cs.pool is not None and _clipped_window(cs.pool)][:8]


@pytest.mark.parametrize("cs", POOL_SHAPES, ids=[cs.name for cs in POOL_SHAPES])
def test_checker_rejects_pool_window_counting_outside_pixels(cs):
    """A window that takes an out-of-image pixel as 0 (max over a zero, average over the full window area) is rejected."""
    import torch.nn.functional as F
    pc = cs.pool
    t, kh, kw, sh, sw, (pl, pr, pt, pb), _, (n, ch, h, w) = pc
    g = torch.Generator().manual_seed(cs.idx)
    x = (torch.rand((n, ch, h, w), generator=g) * 2 - 1 - (1.5 if t == 0 else 0.0)).double()
    kernel = "pool-" + pool_kernel(pc)
    ref, bound = pool_expect(pc, x, kernel)
    assert check_pool(ref, ref, bound) == 0.0
    _, _, oh, ow, _, _ = pool_geometry(pc)
    oy, ox = pt + pb, pl + pr
    pad_b = max(0, (oh - 1) * sh - oy + kh - h)
    pad_r = max(0, (ow - 1) * sw - ox + kw - w)
    win = F.pad(x, (ox, pad_r, oy, pad_b), value=0.0).unfold(2, kh, sh).unfold(3, kw, sw)[:, :, :oh, :ow]
    bad = win.amax((-1, -2)) if t == 0 else win.sum((-1, -2)) / (kh * kw)
    assert check_pool(bad, ref, bound) > 1.0
