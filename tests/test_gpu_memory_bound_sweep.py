"""Seeded random geometries across the memory-bound kernels' instantiation boundaries, against float64 and bit-exact
references.

test_gpu_dispatch_sweep.py, test_gpu_layer_sweep.py and test_gpu_persistent_sweep.py sweep the convolution, deconvolution,
resize and SSD-head kernels.  The kernels below pick an instantiation from the shape and from pointer alignment, and were
otherwise tested only on short hand-picked lists:

  - InstanceNorm (instance_norm.cu): the stats kernel is VEC iff S % 4 == 0 and `in` is 16-byte aligned; the apply
    kernel is PAD x VEC, VEC iff So % 4 == 0, `out` aligned and (padded or the stats kernel VEC).  K = ceil(S / 8192)
    chunks around 1 / 2 and above 32 (a lane combines more than one chunk), a pad that takes the output plane across a
    chunk boundary (K2 != K), short last chunks, So % 4 != S % 4, reflect pads at n - 1, replicate, a constant border
    with the ReLU, affine on and off, several eps, in place.  Padding alone on the same four instantiations.
  - Normalize (normalize.cu): the per-pixel tile tp from 32 to 256, staged (C * 4 * tp <= 128 KB) or the L2 fallback,
    16-byte staging (plane % 4 == 0 and both pointers aligned) or 4-byte, partial tiles and planes below 32; the
    across_spatial segments around multiples of 8192 and past 32 chunks; shared and per-channel scales, every eps_mode.
  - LRN (lrn.cu): across channels local_size 1 / 3 / 5 / 7 (the specialisations) at V = 4 and V = 1, and >= 9 (the
    generic kernel), C below the window and below the 8-stage cp.async ring, thread groups straddling images; within a
    channel the staged halo tile or the recomputed squares (a halo over 48 KB), planes below the 32 x 16 tile, r >= H, W.
  - Routing (route.cu): V = 4 iff inner % 4 == 0 and every source and destination is aligned (one misaligned pointer
    among up to 8 flips the launch); Concat of 1 - 8 unequal bottoms, ShuffleChannel, Slice with a begin offset, chains.
  - PixelShuffle (deconv.cu's scatter): r 1 - 4, both modes, VEC iff OW % 4 == 0 and `out` aligned, more than 65535
    planes (the grid-y loop), the ADD tail sized by scale factor and by size.
  - BinaryOp (binary_op.cu): the same-shape kernel (vec iff a, b and out aligned; a scalar b; tails; past the grid cap of
    sm_count * 32 CTAs), the broadcast kernel (row4 iff W % 4 == 0 and `out` aligned) on every axis and side, ncnn's
    rank-1 per-channel rule, in place, all 12 ops with and without the ReLU.
  - Activations (activation.cu): vec and tail, the grid cap, in place, all five types, ncnn's and PyTorch's alpha.

Oracles are the existing ones: bit for bit test_style_host.pad_ref, test_route_host.shuffle_ref / slice_ref and
np.concatenate, test_sr_host.pixel_shuffle_ref (+ upsample_ref in one fp32 add for the tail), test_gpu_binary_op.binary_ref,
test_activation_host.hard_np, and InstanceNorm against test_style_host.instance_norm32 (fcuda.h's stated summation order,
restated in float32; on large cases a sample of planes: the first, the last and a seeded one) with fmaxf and pad_ref
applied; within bounds test_style_host.instance_norm_bound, test_gpu_normalize._check, test_gpu_lrn.check_lrn (both
shares), test_gpu_activation's act_bound and test_gpu_binary_op's ulp bounds for POW / ATAN2.  InstanceNorm, Normalize and
LRN are run a second time with the alignment flipped, in place where allowed and the batch split in two: the bits must
not change.  Every call goes through the C ABI on views 0 - 3 floats past a 16-byte boundary, each view inside a
NaN-filled buffer whose other floats must stay NaN.

One deterministic generator; each case seeded from the crc32 of its index and labelled with the instantiation a Python
restatement of the launcher's predicate says it reaches.  The CPU tests check that the list hits every reachable cell and
both sides of every predicate, and that the checkers reject simulated defects on the sweep's own shapes.  A failing case
prints a ready-to-paste literal for the family's hand-written list.

At the net level, seeded small nets of these layers' fusion patterns (InstanceNorm -> ReLU -> Padding, Concat ->
ShuffleChannel -> Slice, PixelShuffle + nearest Interp -> sum), some with a second reader of an intermediate blob, run
with fusion, CUDA graphs and route_fuse each on and off: the layers fused away must be those a restatement of
Net::ApplyFusion predicts, and every blob materialised in two runs must have the same bits in both.

FCUDA_SWEEP_SCALE (a float, default 1) scales the case and net counts.  Run with -s to print, per cell, the case count and the
largest share of the bound used.
"""
from __future__ import annotations

import dataclasses
import math
import os
import random
import zlib

import numpy as np
import pytest
import torch

from test_activation_host import hard_np
from test_gpu_activation import PNNX_ALPHA, _within
from test_gpu_binary_op import SPECIALS, _same_or_nan, _ulps, binary_ref
from test_gpu_lrn import PARAMS as LRN_PARAMS
from test_gpu_lrn import check_lrn
from test_gpu_normalize import _check as normalize_check
from test_normalize_host import normalize_ref
from test_route_host import shuffle_ref
from test_sr_host import pixel_shuffle_ref, upsample_ref
from test_style_host import instance_norm32, instance_norm_bound, pad_ref

gpu = pytest.mark.gpu
F = np.float32

N_CASES = 480
SCALE = float(os.environ.get("FCUDA_SWEEP_SCALE", "1"))
CASES_RUN = max(1, int(round(N_CASES * SCALE)))

CHUNK = 8192                      # instance_norm.cu kChunk, normalize.cu kSpatialChunk
GRID_CAP = 132 * 32 * 256 * 4     # floats the same-shape BinaryOp / activation grid covers in one pass on 132 SMs
PLANES_Y = 65535                  # grid-y limit of the scatter's plane loop
WITHIN_SMEM = 48 * 1024           # lrn.cu kWithinSmemBudget
STAGE_BUDGET = 128 * 1024         # normalize.cu kStageBudget
PAYLOAD_NAN = np.array([0x7FC12345, 0xFFA00001], np.uint32).view(np.float32)


# ---- the generator ----------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    idx: int
    family: str
    p: dict = dataclasses.field(default_factory=dict)

    @property
    def name(self):
        return f"{self.idx:04d}-{self.family}"


def _off(r, aligned=None):
    """A view offset in floats: 0 (16-byte aligned), 1..3 (not), or either."""
    if aligned is None:
        return r.choice([0, 0, 1, 2, 3])
    return 0 if aligned else r.randint(1, 3)


def _pads(r, h, w, type_, So4=None):
    """(top, bottom, left, right) of a pad of `type_` (reflect pads < the dimension, biased to n - 1)."""
    def one(n):
        if type_ == 2:
            return min(n - 1, r.choice([0, 1, n - 1, n - 1, r.randint(0, 3)])) if n > 1 else 0
        return r.choice([0, 1, 2, 4, 9])
    pads = [one(h), one(h), one(w), one(w)]
    if not any(pads):
        if w > 1 or type_ != 2:
            pads[3] = 1
        elif h > 1:
            pads[1] = 1
    return tuple(pads)


def _pad_to(r, h, w, type_, want4):
    """A pad whose output plane is (want4) or is not a multiple of 4 floats; None when none is found."""
    for _ in range(40):
        t = _pads(r, h, w, type_)
        if any(t) and (((h + t[0] + t[1]) * (w + t[2] + t[3])) % 4 == 0) == want4:
            return t
    return None


IN_TARGETS = ("small", "vec", "scalar", "k12", "cross", "short", "big", "pad-vec", "pad-scalar", "misaligned")
K12_PLANES = [(1, 8191), (1, 8192), (1, 8193), (64, 128), (128, 128), (127, 129), (2, 8191), (3, 5461), (1, 16385),
              (91, 90), (16, 1024)]


def _gen_in(r, k) -> dict:
    target = IN_TARGETS[k % len(IN_TARGETS)]
    n, c = r.choice([1, 2, 3]), r.choice([1, 2, 3, 5])
    h, w = r.randint(1, 40), r.randint(1, 40)
    in_off, out_off = _off(r), _off(r)
    pad = None
    if target == "vec":
        w = 4 * r.randint(1, 12)
        in_off = out_off = 0
    elif target == "scalar":
        w = 4 * r.randint(1, 12) + r.randint(1, 3)
        h = r.choice([1, 3, 5, 7])
    elif target == "k12":
        h, w = r.choice(K12_PLANES)
        n, c = r.choice([1, 2]), r.choice([1, 2])
    elif target == "cross":      # S <= 8192, the padded plane past it: K = 1, K2 = 2
        w = r.choice([64, 90, 91, 100, 127])
        h = 8192 // w - r.randint(0, 1)
        n, c = 1, r.choice([1, 2])
        type_ = r.choice([0, 1, 2])
        pad = (r.randint(1, 2), 0, r.randint(0, 1), 1, type_, r.uniform(-2, 2))
    elif target == "short":      # K = 2..4 with a short last chunk
        w = r.choice([1, 3, 64, 97])
        h = (CHUNK * r.randint(1, 3)) // w + r.randint(1, 3)
        n, c = 1, r.choice([1, 2])
    elif target == "big":        # K > 32: a lane of the combination adds more than one chunk
        h, w = r.choice([(1, 262145), (512, 513), (300, 1000), (640, 512), (1, 40 * CHUNK + 5)])
        n, c = 1, r.choice([1, 2])
    elif target in ("pad-vec", "pad-scalar"):
        type_ = r.choice([0, 1, 2])
        if type_ == 2:
            h, w = max(h, 2), max(w, 2)
        t = _pad_to(r, h, w, type_, target == "pad-vec")
        if t is None:
            w += 1
            t = _pad_to(r, h, w, type_, target == "pad-vec") or _pads(r, h, w, type_)
        pad = t + (type_, r.choice([0.0, -1.5, 2.25, -0.5]))
        if target == "pad-vec":
            out_off = 0
            if k % 20 < 10:          # a VEC stats kernel too
                in_off = 0
                if (h * w) % 4:
                    h = 4 * (h // 4 + 1)
    elif target == "misaligned":
        w = 4 * r.randint(1, 10)
        in_off, out_off = r.choice([(r.randint(1, 3), 0), (0, r.randint(1, 3)), (0, r.randint(1, 3)),
                                    (r.randint(1, 3), r.randint(1, 3))])
    if pad is None and target not in ("vec", "scalar", "big") and r.random() < 0.35:
        type_ = r.choice([0, 1, 2])
        if type_ == 2 and (h == 1 and w == 1):
            type_ = 1
        pad = _pads(r, h, w, type_) + (type_, r.choice([0.0, 0.5, -3.0]))
    affine = r.random() < 0.6
    inplace = pad is None and r.random() < 0.25
    if inplace:
        out_off = in_off
    return dict(target=target, n=n, c=c, h=h, w=w, pad=pad, affine=affine, eps=r.choice([1e-5, 1e-3, 0.1, 0.0]),
                relu=r.random() < 0.5, in_off=in_off, out_off=out_off, inplace=inplace,
                gain=r.choice([0.1, 1.0, 10.0]), shift=r.choice([0.0, 3.0, -50.0]))


PAD_TARGETS = ("pad-vec", "pad-scalar", "nopad", "pad-vec", "misaligned")


def _gen_pad(r, k) -> dict:
    target = PAD_TARGETS[k % len(PAD_TARGETS)]
    n, c, h, w = r.choice([1, 2, 3]), r.choice([1, 2, 4]), r.randint(1, 30), r.randint(1, 30)
    type_ = r.choice([0, 1, 2])
    if type_ == 2:
        h, w = max(h, 2), max(w, 2)
    in_off, out_off = _off(r), _off(r)
    if target == "nopad":
        pad = (0, 0, 0, 0)
        if k % 10 < 5:
            w, in_off, out_off = 4 * r.randint(1, 8), 0, 0
    else:
        pad = _pad_to(r, h, w, type_, target != "pad-scalar") or _pads(r, h, w, type_)
        if target == "pad-vec":
            out_off = 0
        elif target == "misaligned":
            out_off = r.randint(1, 3)
    return dict(target=target, n=n, c=c, h=h, w=w, pad=pad + (type_, r.choice([0.0, -1.5, 7.0])), in_off=in_off,
                out_off=out_off)


NORM_TARGETS = ("tp", "stage", "fallback", "partial", "tiny", "image", "plane", "stage", "stage", "tp", "image", "plane")
STAGE_C = (16, 33, 65, 200)      # tp 256, 128, 64 and 32 on planes past 256 pixels
IMAGE_SEGS = (CHUNK - 1, 33 * CHUNK + 17, CHUNK + 1, 2000, CHUNK, 40 * CHUNK + 1, 5 * CHUNK + 3)
PLANE_SEGS = (CHUNK, 33 * CHUNK + 5, CHUNK + 1, 700, 3 * CHUNK, CHUNK - 1, 36 * CHUNK)
TP_C = (1, 3, 16, 32, 33, 64, 65, 128, 129, 256, 512, 1024)


def _gen_norm(r, k) -> dict:
    target = NORM_TARGETS[k % len(NORM_TARGETS)]
    j = k // len(NORM_TARGETS) * NORM_TARGETS.count(target) + NORM_TARGETS[:k % len(NORM_TARGETS)].count(target)
    in_off, out_off = _off(r), _off(r)
    sp, ch = 0, 1
    n = r.choice([1, 2, 3])
    c = r.choice(TP_C)
    plane = r.randint(1, 600) if c <= 128 else r.randint(1, 80)
    if target == "stage":        # each tp with the 16-byte staging, then with one side of its predicate broken
        c = STAGE_C[j % 4]
        plane = 4 * (r.randint(70, 150) if c <= 128 else r.randint(8, 50))
        if j // 4 % 2:
            if r.random() < 0.5:
                plane += r.randint(1, 3)
            else:
                in_off, out_off = r.choice([(r.randint(1, 3), 0), (0, r.randint(1, 3))])
        else:
            in_off = out_off = 0
    elif target == "fallback":
        c, plane = r.choice([1025, 1100, 2048, 1024]), r.choice([1, 7, 31, 32, 33, 40, 64])
        n = r.choice([1, 2])
    elif target == "partial":
        tp = 1 << pixel_tile_shift(c, 10 ** 6)
        plane = tp * r.randint(1, 3) + r.randint(1, tp - 1)
    elif target == "tiny":
        plane = r.randint(1, 31)
    elif target == "image":
        sp, ch = 1, 1
        seg = IMAGE_SEGS[j % len(IMAGE_SEGS)]
        c = 1 if seg % CHUNK in (0, 1, CHUNK - 1) else r.choice([1, 3, 8])
        plane = max(1, seg // c)
        n = 1 if seg > 4 * CHUNK else r.choice([1, 2, 3])
    elif target == "plane":
        sp, ch = 1, 0
        plane = PLANE_SEGS[j % len(PLANE_SEGS)]
        c = r.choice([1, 2]) if plane > 4 * CHUNK else r.choice([1, 3, 5])
        n = 1 if plane > 4 * CHUNK else r.choice([1, 2, 3])
    if c > 128 and plane > 200:
        plane = r.randint(1, 200)
    mode = r.randint(0, 2)
    return dict(target=target, n=n, c=c, plane=plane, sp=sp, ch=ch, eps_mode=mode, eps=(1e-4, 1e-10, 1e-12)[mode],
                shared=r.random() < 0.3, in_off=in_off, out_off=out_off, inplace=r.random() < 0.25)


LRN_TARGETS = ("across-v4", "across", "generic", "smallc", "straddle", "within", "within-big", "within-tiny", "across-v4",
               "across", "within")
BIG_WINDOWS = ((89, 104, 120), (91, 110, 125), (45, 60, 60), (89, 110, 130), (89, 40, 200))   # (local_size, h, w)


def _gen_lrn(r, k) -> dict:
    target = LRN_TARGETS[k % len(LRN_TARGETS)]
    j = k // len(LRN_TARGETS) * LRN_TARGETS.count(target) + LRN_TARGETS[:k % len(LRN_TARGETS)].count(target)
    in_off, out_off = _off(r), _off(r)
    n, c = r.choice([1, 2, 3]), r.choice([3, 8, 16, 17, 33])
    h, w = r.randint(1, 20), r.randint(1, 20)
    region, size = 0, r.choice([1, 3, 5, 7])
    if target == "across-v4":    # each specialisation on the 16-byte path
        size, w, in_off, out_off = (1, 3, 5, 7)[j % 4], 4 * r.randint(1, 6), 0, 0
    elif target == "across":     # each specialisation on the 4-byte path: an odd plane or a misaligned pointer
        size = (1, 3, 5, 7)[j % 4]
        if r.random() < 0.5:
            h, w = 2 * r.randint(1, 10) - 1, 2 * r.randint(1, 10) - 1
        elif _al(in_off) and _al(out_off):
            in_off = r.randint(1, 3)
    elif target == "generic":
        size = r.choice([9, 11, 15])
    elif target == "smallc":
        c = r.choice([1, 2, 3, 4, 6, 7, 9])
        size = r.choice([3, 5, 7, 9])
    elif target == "straddle":    # batch * plane / V not a multiple of 128, thread groups across images
        n = r.choice([2, 3, 5])
        h, w = r.choice([(7, 12), (5, 20), (13, 4), (9, 9), (30, 30)])
    elif target == "within":
        region, size = 1, r.choice([1, 3, 5, 7, 9])
        h, w = r.randint(1, 70), r.randint(1, 70)
        c = r.choice([1, 2, 3])
    elif target == "within-big":
        region, c, n = 1, r.choice([1, 2]), 1
        size, h, w = BIG_WINDOWS[j % len(BIG_WINDOWS)]
    elif target == "within-tiny":
        region, c = 1, r.choice([1, 2, 4])
        h, w = r.randint(1, 15), r.randint(1, 31)
        size = r.choice([3, 5, 2 * max(h, w) + 1, 2 * max(h, w) + 3])
    alpha, beta, bias = r.choice(LRN_PARAMS)
    return dict(target=target, n=n, c=c, h=h, w=w, region=region, size=size, alpha=alpha, beta=beta, bias=bias,
                in_off=in_off, out_off=out_off)


ROUTE_TARGETS = ("concat", "shuffle", "slice", "chain", "chain", "concat", "slice")
INNERS = (1, 2, 3, 4, 7, 8, 12, 16, 49, 64, 196)


def _gen_route(r, k) -> dict:
    kind = ROUTE_TARGETS[k % len(ROUTE_TARGETS)]
    j = k // len(ROUTE_TARGETS) * ROUTE_TARGETS.count(kind) + ROUTE_TARGETS[:k % len(ROUTE_TARGETS)].count(kind)
    n = r.choice([1, 2, 3, 7])
    inner = r.choice(INNERS)
    axis = 1
    count = {"concat": (1, 8, 3, 5, 2)[j % 5], "chain": r.randint(2, 8)}.get(kind, 1)
    srcs = [r.randint(1, 12) for _ in range(count)]
    if kind == "shuffle":
        srcs = [r.choice([6, 8, 12, 24, 30, 9])]
    mid = sum(srcs)
    group, reverse, begin = 1, 0, 0
    if kind in ("shuffle", "chain"):
        divs = [g for g in range(1, mid) if mid % g == 0 and g * g != mid]
        group = r.choice(divs[1:] if len(divs) > 1 else divs)
        reverse = r.randint(0, 1)
    if kind in ("concat", "shuffle"):
        dsts = [mid]
    else:
        begin = r.randint(0, mid - 1)
        left = mid - begin
        dsts = []
        while left > 0 and len(dsts) < 8:
            s = r.randint(1, min(left, 5))
            dsts.append(s)
            left -= s
            if r.random() < 0.15:
                break
    offs = {"src": [0] * len(srcs), "dst": [0] * len(dsts)}
    mis = r.random()
    if j % 2 == 0 and kind in ("shuffle", "slice", "concat"):   # the 16-byte path
        inner, mis = r.choice([4, 8, 16, 64]), 1.0
    if mis < 0.35:     # one pointer misaligned among up to 16
        side = r.choice(["src", "dst"])
        offs[side][r.randrange(len(offs[side]))] = r.randint(1, 3)
    elif mis < 0.5:
        offs = {s: [_off(r) for _ in v] for s, v in offs.items()}
    if kind == "slice" and r.random() < 0.3:
        axis = 2      # slicing rows: outer = channels
    return dict(target=kind, n=n, inner=inner, srcs=srcs, group=group, reverse=reverse, begin=begin, dsts=dsts,
                offs=offs, axis=axis, outer_c=r.choice([1, 3]) if axis == 2 else 1)


PS_TARGETS = ("copy", "copy", "tail-scale", "tail-size", "planes", "vec", "tail-scale", "copy")


def _gen_ps(r, k) -> dict:
    target = PS_TARGETS[k % len(PS_TARGETS)]
    rr, mode = r.randint(1, 4), r.randint(0, 1)
    n, oc, h, w = r.choice([1, 2, 3]), r.choice([1, 2, 3, 5]), r.randint(1, 20), r.randint(1, 20)
    out_off = _off(r)
    add = None
    if target == "vec":
        w = r.choice([1, 2, 3, 4, 5, 8]) * (4 // math.gcd(4, rr))
        out_off = 0
    elif target == "planes":     # 2049 * 33 planes: the grid-y loop carries (n, oc)
        n, oc, h, w, rr = 2049, 33, 1, r.choice([1, 2, 3]), r.choice([1, 2])
    elif target == "tail-scale":
        if r.random() < 0.5:
            w, out_off = 4 * r.randint(1, 4), 0
        add = ("scale", h, w)
    elif target == "tail-size":
        add = ("size", r.randint(1, 2 * h + 3), r.randint(1, 2 * w + 3))
    return dict(target=target, n=n, oc=oc, h=h, w=w, r=rr, mode=mode, add=add, out_off=out_off)


BIN_TARGETS = ("same", "same-vec", "scalar", "bcast", "bcast-row4", "both", "rank1", "inplace", "gridcap", "bcast")
TRANSCENDENTAL = (6, 9, 10, 11)


def _bshape(r, c, h, w, force=True):
    """(a, b) per-image shapes: on each axis neither, a or b is 1 (at least one broadcast when `force`)."""
    while True:
        sides = [r.choice([0, 0, 1, 2]) for _ in range(3)]
        if any(sides) or not force:
            break
    full = (c, h, w)
    a = tuple(1 if s == 1 else e for s, e in zip(sides, full))
    b = tuple(1 if s == 2 else e for s, e in zip(sides, full))
    return a, b


def _gen_binop(r, k) -> dict:
    target = BIN_TARGETS[k % len(BIN_TARGETS)]
    op = (5 * k + k // 24) % 12          # every op in each run of 12 cases, the ReLU on every other run
    relu = (k // 12) % 2 == 1
    n = r.choice([1, 2, 3])
    c, h, w = r.choice([1, 2, 3, 5]), r.randint(1, 9), r.randint(1, 13)
    offs = [_off(r), _off(r), _off(r)]        # a, b, out
    a_s = b_s = (c, h, w)
    scalar, inplace, rank1 = None, None, False
    if target == "same" and k // len(BIN_TARGETS) % 3 == 0:
        op, relu = 0, k % 2 == 1   # the same-shape ADD: the Eltwise SUM kernel
    if target == "same-vec":
        offs = [0, 0, 0]
        w = 4 * r.randint(1, 4) + r.choice([0, 1, 2, 3])
        a_s = b_s = (c, h, w)
    elif target == "scalar":
        b_s, scalar = None, r.choice([0.5, -0.0, -3.25, 2.0, float("inf")])
    elif target in ("bcast", "both", "bcast-row4"):
        if target == "bcast-row4":
            w = 4 * r.randint(1, 5)
            offs[2] = 0
        a_s, b_s = _bshape(r, c, h, w)
        if target == "both":
            a_s, b_s = r.choice([((c, 1, w), (1, h, 1)), ((1, h, w), (c, 1, 1)), ((c, h, 1), (1, 1, w))])
            if r.random() < 0.5:
                a_s, b_s = b_s, a_s
    elif target == "rank1":      # ncnn's per-channel rule: b a rank-1 blob of c values, possibly with w == c or h == c
        c = r.choice([2, 3, 4, 5])
        h, w = r.choice([(c, 7), (5, c), (c, c), (3, 6)])
        a_s, b_s, rank1 = (c, h, w), (c, 1, 1), True
    elif target == "inplace":
        inplace = r.choice(["a", "b"])
        other = r.choice([(c, h, w), (c, 1, 1), (1, h, w), (1, 1, w), (c, h, 1)])
        a_s, b_s = ((c, h, w), other) if inplace == "a" else (other, (c, h, w))
    elif target == "gridcap":    # past sm_count * 32 CTAs of 1024 floats: the grid-stride loop runs twice
        op = {6: 2, 9: 7, 10: 3, 11: 8}.get(op, op)     # exact ops only: POW -> MUL, RPOW -> RSUB, ATAN2 / RATAN2 -> DIV / RDIV
        n, c, h, w = 1, 3, r.choice([1000, 1001]), 1500
        a_s = b_s = (c, h, w)
        if r.random() < 0.5:
            b_s, scalar = None, 0.75
        offs = r.choice([[0, 0, 0], [1, 1, 1], [0, 0, 2]])
    if scalar is not None:
        offs[1] = 0
    if inplace == "a":
        offs[2] = offs[0]
    elif inplace == "b":
        offs[2] = offs[1]
    return dict(target=target, op=op, relu=relu, n=n, a=a_s, b=b_s, scalar=scalar, offs=offs, inplace=inplace,
                rank1=rank1)


ACT_KINDS = ("Sigmoid", "TanH", "Swish", "HardSigmoid", "HardSwish")
ACT_TARGETS = ("tail", "vec", "medium", "misaligned", "inplace", "vec", "tail9", "gridcap")


def _gen_act(r, k) -> dict:
    kind = ACT_KINDS[k % 5]
    target = ACT_TARGETS[(k // 5) % len(ACT_TARGETS)]
    n = {"tail": r.randint(1, 3), "tail9": r.randint(5, 9), "vec": 4 * r.randint(1, 300) + r.randint(0, 3), "medium": r.randint(1000, 70000),
         "misaligned": r.randint(1, 5000), "inplace": r.randint(1, 5000),
         "gridcap": GRID_CAP + r.choice([1, 3, 4096, 200001])}[target]
    in_off, out_off = _off(r), _off(r)
    if target in ("vec", "medium"):
        in_off = out_off = 0
    elif target == "misaligned":
        in_off, out_off = r.choice([(0, r.randint(1, 3)), (r.randint(1, 3), 0)])
    inplace = target == "inplace" or r.random() < 0.15
    if inplace:
        out_off = in_off
    alpha = r.choice([0.2, PNNX_ALPHA]) if kind.startswith("Hard") else 0.2
    return dict(target=target, kind=kind, n=n, alpha=alpha, beta=0.5, in_off=in_off, out_off=out_off, inplace=inplace)


SLOTS = ["in", "pad", "norm", "lrn", "in", "route", "ps", "binop", "norm", "lrn", "binop", "act"]
GENS = {"in": _gen_in, "pad": _gen_pad, "norm": _gen_norm, "lrn": _gen_lrn, "route": _gen_route, "ps": _gen_ps,
        "binop": _gen_binop, "act": _gen_act}


def gen_case(i: int) -> Case:
    """Case i.  k counts the cases of its family; each family cycles its targets with k."""
    r = random.Random(zlib.crc32(f"memory-bound-sweep-{i}".encode()))
    fam = SLOTS[i % len(SLOTS)]
    k = i // len(SLOTS) * SLOTS.count(fam) + SLOTS[:i % len(SLOTS)].count(fam)
    return Case(i, fam, GENS[fam](r, k))


_CASES = None


def cases() -> list[Case]:
    global _CASES
    if _CASES is None:
        _CASES = [gen_case(i) for i in range(CASES_RUN)]
    return _CASES


# ---- restatements of the launchers' predicates ------------------------------------------------------------------------
def _al(off) -> bool:
    """A view `off` floats into a fresh allocation is 16-byte aligned."""
    return off % 4 == 0


def in_geometry(p):
    pad = p["pad"] or (0, 0, 0, 0, 0, 0.0)
    S = p["h"] * p["w"]
    Ho, Wo = p["h"] + pad[0] + pad[1], p["w"] + pad[2] + pad[3]
    return S, Ho, Wo, Ho * Wo, math.ceil(S / CHUNK), math.ceil(Ho * Wo / CHUNK)


def in_kernels(p, in_off=None, out_off=None, padded=None) -> tuple[str, str]:
    """instance_norm.cu instance_norm_forward / padding_forward: (stats, apply) instantiations."""
    in_off = p["in_off"] if in_off is None else in_off
    out_off = p["out_off"] if out_off is None else out_off
    S, _, _, So, _, _ = in_geometry(p)
    padded = any(p["pad"][:4]) if p["pad"] else False
    vin = S % 4 == 0 and _al(in_off)
    vout = So % 4 == 0 and _al(out_off) and (padded or vin)
    return ("vec" if vin else "scalar"), f"{'pad' if padded else 'nopad'}-{'vec' if vout else 'scalar'}"


def pixel_tile_shift(C, plane) -> int:
    """normalize.cu pixel_tile_shift."""
    shift = 5
    while (1 << shift) < 256 and C << (shift + 1) <= 8192 and (1 << shift) < plane:
        shift += 1
    return shift


def norm_kernel(p, in_off=None, out_off=None) -> tuple[str, str]:
    in_off = p["in_off"] if in_off is None else in_off
    out_off = p["out_off"] if out_off is None else out_off
    c, plane = p["c"], p["plane"]
    if p["sp"]:
        K = math.ceil((c * plane if p["ch"] else plane) / CHUNK)
        return ("norm-image" if p["ch"] else "norm-plane"), ("k1" if K == 1 else "k2-32" if K <= 32 else "k33+")
    tp = 1 << pixel_tile_shift(c, plane)
    staged = c * 4 * tp <= STAGE_BUDGET
    wide = staged and plane % 4 == 0 and _al(in_off) and _al(out_off)
    return "norm-pixel", f"tp{tp}-" + ("stage16" if wide else "stage4" if staged else "l2")


def lrn_kernel(p, in_off=None, out_off=None) -> tuple[str, str]:
    in_off = p["in_off"] if in_off is None else in_off
    out_off = p["out_off"] if out_off is None else out_off
    h, w, size = p["h"], p["w"], p["size"]
    if p["region"] == 0:
        if size > 7:
            return "lrn-across", "generic"
        v = 4 if (h * w) % 4 == 0 and _al(in_off) and _al(out_off) else 1
        return "lrn-across", f"L{size}-V{v}"
    r = size // 2
    smem = min(16 + 2 * r, h) * min(32 + 2 * r, w) * 4
    return "lrn-within", "staged" if smem <= WITHIN_SMEM else "recomputed"


def route_kernel(p) -> str:
    ok = p["inner"] % 4 == 0 and all(_al(o) for v in p["offs"].values() for o in v)
    return "v4" if ok else "v1"


def ps_kernel(p, out_off=None) -> tuple[str, str]:
    out_off = p["out_off"] if out_off is None else out_off
    vec = (p["w"] * p["r"]) % 4 == 0 and _al(out_off)
    return ("add" if p["add"] else "copy"), ("vec" if vec else "scalar")


def bin_kernel(p) -> tuple[str, str]:
    a, b = p["a"], p["b"]
    full = tuple(max(x, y) for x, y in zip(a, b)) if b is not None else a
    if a == full and (b is None or b == full):
        if b is not None and p["op"] == 0:
            return "binop-same", "eltwise"
        vec = _al(p["offs"][0]) and _al(p["offs"][2]) and (b is None or _al(p["offs"][1]))
        return "binop-same", "vec" if vec else "scalar"
    return "binop-bcast", "row4" if full[2] % 4 == 0 and _al(p["offs"][2]) else "row"


def act_kernel(p) -> str:
    return "vec" if _al(p["in_off"]) and _al(p["out_off"]) and p["n"] >= 4 else "scalar"


def labels(case: Case) -> tuple[str, str]:
    p = case.p
    if case.family == "in":
        s, a = in_kernels(p)
        return "instance-norm", f"stats-{s}/{a}"
    if case.family == "pad":
        return "padding", in_kernels(p)[1]
    if case.family == "norm":
        return norm_kernel(p)
    if case.family == "lrn":
        return lrn_kernel(p)
    if case.family == "route":
        return f"route-{p['target']}", route_kernel(p)
    if case.family == "ps":
        k, v = ps_kernel(p)
        return f"pixel-shuffle-{k}", v
    if case.family == "binop":
        return bin_kernel(p)
    return f"act-{p['kind']}", act_kernel(p)


def literal(case: Case) -> str:
    """A ready-to-paste entry for the family's hand-written list."""
    p = case.p
    if case.family == "in":
        return (f"PLANES: ({p['h']}, {p['w']})  # batch {p['n']}, channels {p['c']}, pad {p['pad']}, affine "
                f"{int(p['affine'])}, eps {p['eps']}, relu {int(p['relu'])}, offsets in / out {p['in_off']} / "
                f"{p['out_off']}, in place {int(p['inplace'])}")
    if case.family == "pad":
        return (f"test_padding_bit_exact: (({p['h']}, {p['w']}), {p['pad'][:4]})  # type {p['pad'][4]}, value "
                f"{p['pad'][5]}, batch {p['n']}, channels {p['c']}, offsets in / out {p['in_off']} / {p['out_off']}")
    if case.family == "norm":
        return (f"SHAPES: ({p['n']}, {p['c']}, 1, {p['plane']})  # mode (across_spatial {p['sp']}, across_channel "
                f"{p['ch']}), eps_mode {p['eps_mode']}, shared {int(p['shared'])}, offsets in / out {p['in_off']} / "
                f"{p['out_off']}, in place {int(p['inplace'])}")
    if case.family == "lrn":
        lst = "ACROSS_SHAPES" if p["region"] == 0 else "WITHIN_SHAPES"
        return (f"{lst}: ({p['n']}, {p['c']}, {p['h']}, {p['w']})  # local_size {p['size']}, (alpha, beta, bias) "
                f"{(p['alpha'], p['beta'], p['bias'])}, offsets in / out {p['in_off']} / {p['out_off']}")
    if case.family == "route":
        if p["target"] == "slice" and len(p["srcs"]) == 1:
            sizes = p["dsts"] + ([p["srcs"][0] - p["begin"] - sum(p["dsts"])] if p["begin"] + sum(p["dsts"]) <
                                 p["srcs"][0] else [])
            return (f"SLICE_CASES: (({p['outer_c'] if p['axis'] == 2 else p['srcs'][0]}, "
                    f"{p['srcs'][0] if p['axis'] == 2 else 1}, {p['inner']}), {p['axis'] - 1}, {sizes})  # begin "
                    f"{p['begin']}, batch {p['n']}, offsets {p['offs']}")
        return (f"ROUTE_CASES: ({p['srcs']}, {p['dsts']}, {p['group']}, {p['reverse']}, {p['begin']}, {p['inner']}, "
                f"{p['n']})  # offsets {p['offs']}")
    if case.family == "ps":
        if p["add"]:
            scale = float(p["r"]) if p["add"][0] == "scale" else None
            return (f"TAILS: ({p['r']}, {p['mode']}, ({p['n']}, {p['h']}, {p['w']}), {scale})  # channels "
                    f"{p['oc'] * p['r'] ** 2}, addend {p['add']}, output offset {p['out_off']}")
        return (f"SHAPES: ({p['n']}, {p['h']}, {p['w']})  # r {p['r']}, mode {p['mode']}, channels "
                f"{p['oc'] * p['r'] ** 2}, output offset {p['out_off']}")
    if case.family == "binop":
        return (f"FORMS: \"{case.name}\": ({p['a']}, {p['b'] or (1, 1, 1)})  # op {p['op']}, relu {int(p['relu'])}, "
                f"batch {p['n']}, scalar {p['scalar']}, offsets a / b / out {p['offs']}, in place {p['inplace']}")
    return (f"{p['kind']}: n {p['n']}, offsets in / out {p['in_off']} / {p['out_off']}, in place {int(p['inplace'])}, "
            f"alpha {p['alpha']}")


# ---- data ------------------------------------------------------------------------------------------------------------
def _rng(case: Case) -> np.random.Generator:
    return np.random.default_rng(zlib.crc32(case.name.encode()))


def in_data(case: Case):
    """(x, gamma, beta): per-channel scale and offset, so planes are offset from 0 by up to 50 standard deviations."""
    p, rng = case.p, _rng(case)
    shape = (p["n"], p["c"], p["h"], p["w"])
    x = rng.standard_normal(shape) * rng.uniform(0.5, 2, (1, p["c"], 1, 1)) * p["gain"]
    x = (x + p["shift"] * rng.uniform(0.5, 1, (1, p["c"], 1, 1))).astype(F)
    g, b = (rng.uniform(0.5, 1.5, p["c"]).astype(F), rng.uniform(-1, 1, p["c"]).astype(F)) if p["affine"] else (None, None)
    return x, g, b


def signed_data(case: Case, shape):
    """Values in +-[0.25, 2]: no near-zeros, so the relative bounds of Normalize and LRN bite."""
    rng = _rng(case)
    return ((rng.uniform(0.25, 2, shape)) * rng.choice([-1, 1], shape)).astype(F)


def copy_data(case: Case, shape):
    """Normal values with -0.0 and NaN payloads sprinkled in: a copy must keep every bit."""
    rng = _rng(case)
    x = rng.standard_normal(shape).astype(F)
    flat = x.reshape(-1)
    k = min(flat.size, 6)
    idx = rng.choice(flat.size, k, replace=False)
    flat[idx] = np.resize(np.concatenate([PAYLOAD_NAN, np.float32([-0.0, np.inf])]), k)
    return x


# ---- report ----------------------------------------------------------------------------------------------------------
REPORT: dict[tuple[str, str], list] = {}


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\ncases and the largest share of the per-element bound used (0 for bit-exact checks), per cell:")
        for (f, k), (n, used) in sorted(REPORT.items()):
            print(f"  {f:24s} {k:26s} {n:4d} cases   bound used {used:.3f}")


def _record(cell, used):
    r = REPORT.setdefault(cell, [0, 0.0])
    r[0] += 1
    r[1] = max(r[1], used)


# ---- device views ----------------------------------------------------------------------------------------------------
def _buf(n: int, off: int, src=None):
    """(view, buffer): n floats `off` floats into a NaN-filled device buffer of n + 8, `src` copied into the view."""
    buf = torch.full((n + 8,), math.nan, device="cuda")
    v = buf[off:off + n]
    if src is not None:
        v.copy_(torch.from_numpy(np.ascontiguousarray(src, F).reshape(-1)))
    return v, buf


def _guard_ok(buf, off, n) -> bool:
    return bool(torch.isnan(buf[:off]).all() and torch.isnan(buf[off + n:]).all())


def _bits(a) -> np.ndarray:
    return np.ascontiguousarray(a, F).view(np.uint32)


def _bits_eq(a, b) -> bool:
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _flip(off) -> int:
    return 1 if _al(off) else 0


def _halves(n):
    return [(0, n)] if n == 1 else [(0, n // 2), (n // 2, n)]


# ---- InstanceNorm and Padding ----------------------------------------------------------------------------------------
def _in_call(x, g, b, p, in_off, out_off, inplace):
    """One InstanceNorm call on views: (output, guard intact)."""
    from feathercnn_b200 import booster
    n, c, h, w = x.shape
    _, Ho, Wo, _, _, _ = in_geometry(p)
    xin, xbuf = _buf(x.size, in_off, x)
    out, obuf, ooff = (xin, xbuf, in_off) if inplace else (*_buf(n * c * Ho * Wo, out_off), out_off)
    t = lambda a: None if a is None else torch.from_numpy(a).cuda()  # noqa: E731
    booster.instance_norm(xin.view(x.shape), t(g), t(b), p["eps"], p["relu"], p["pad"], out=out.view(n, c, Ho, Wo))
    torch.cuda.synchronize()
    ok = _guard_ok(obuf, ooff, out.numel()) and (inplace or _guard_ok(xbuf, in_off, x.size))
    return out.view(n, c, Ho, Wo).cpu().numpy(), ok


def in_planes(case: Case, n, c) -> list[tuple[int, int]]:
    """The planes restated in float32: all, or on large cases the first, the last and a seeded one."""
    S, _, _, _, K, _ = in_geometry(case.p)
    allp = [(i, j) for i in range(n) for j in range(c)]
    if n * c * K <= 24:
        return allp
    r = random.Random(case.idx)
    return sorted({allp[0], allp[-1], r.choice(allp)})


def in_expected(p, x, g, b, i, j):
    """The stated order's bits of output plane (i, j): instance_norm32, fmaxf with the ReLU, then pad_ref."""
    y = instance_norm32(x[i:i + 1, j:j + 1], None if g is None else g[j:j + 1], None if b is None else b[j:j + 1],
                        p["eps"])
    if p["relu"]:
        y = np.fmax(y, F(0))
    if p["pad"] and any(p["pad"][:4]):
        y = pad_ref(y, *p["pad"][:5], p["pad"][5])
    return y[0, 0]


def in_bound_used(p, x, g, b, got) -> float:
    y64, bound = instance_norm_bound(x, g, b, p["eps"])
    if p["relu"]:
        y64 = np.maximum(y64, 0)
    if p["pad"] and any(p["pad"][:4]):
        y64 = pad_ref(y64, *p["pad"][:5], p["pad"][5], dtype=np.float64)
        bound = pad_ref(bound, *p["pad"][:5], 0.0, dtype=np.float64)
    d = np.abs(got.astype(np.float64) - y64)
    with np.errstate(invalid="ignore", divide="ignore"):
        share = np.where(d == 0, 0.0, d / bound)
    return float(np.nanmax(np.where(np.isnan(share), np.inf, share)))


def run_in(case: Case) -> tuple[float, list[str]]:
    p = case.p
    x, g, b = in_data(case)
    problems = []
    got, ok = _in_call(x, g, b, p, p["in_off"], p["out_off"], p["inplace"])
    if not ok:
        problems.append("wrote outside the output view")
    used = in_bound_used(p, x, g, b, got)
    if used > 1.0:
        problems.append(f"bound used {used:.3g}")
    for i, j in in_planes(case, p["n"], p["c"]):
        if not _bits_eq(got[i, j], in_expected(p, x, g, b, i, j)):
            problems.append(f"plane ({i}, {j}) differs from the stated order (test_style_host.instance_norm32)")
            used = math.inf
            break
    # the same bits with the alignment flipped, the batch split in two and in place where allowed
    padded = bool(p["pad"] and any(p["pad"][:4]))
    for n0, n1 in _halves(p["n"]):
        inplace = not padded and not p["inplace"]
        ioff = _flip(p["in_off"])
        again, ok = _in_call(x[n0:n1], g, b, p, ioff, ioff if inplace else _flip(p["out_off"]), inplace)
        if not ok or not _bits_eq(again, got[n0:n1]):
            problems.append(f"images {n0}..{n1 - 1} differ with alignment flipped / in place {int(inplace)}")
            used = math.inf
    return used, problems


def run_pad(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p = case.p
    n, c, h, w = p["n"], p["c"], p["h"], p["w"]
    x = copy_data(case, (n, c, h, w))
    _, Ho, Wo, _, _, _ = in_geometry(p)
    xin, xbuf = _buf(x.size, p["in_off"], x)
    out, obuf = _buf(n * c * Ho * Wo, p["out_off"])
    booster.padding(xin.view(x.shape), *p["pad"], out=out.view(n, c, Ho, Wo))
    torch.cuda.synchronize()
    problems = [] if _guard_ok(obuf, p["out_off"], out.numel()) else ["wrote outside the output view"]
    if not _bits_eq(out.view(n, c, Ho, Wo).cpu().numpy(), pad_ref(x, *p["pad"][:5], p["pad"][5])):
        problems.append("differs from pad_ref")
    return (0.0 if not problems else math.inf), problems


# ---- Normalize -------------------------------------------------------------------------------------------------------
def _norm_call(x, s, p, in_off, out_off, inplace):
    from feathercnn_b200 import booster
    xin, xbuf = _buf(x.size, in_off, x)
    out, obuf, ooff = (xin, xbuf, in_off) if inplace else (*_buf(x.size, out_off), out_off)
    booster.normalize(xin.view(x.shape), torch.from_numpy(s).cuda(), p["sp"], p["ch"], p["eps"], p["eps_mode"],
                      out=out.view(x.shape))
    torch.cuda.synchronize()
    return out.view(x.shape).cpu().numpy(), _guard_ok(obuf, ooff, out.numel())


def norm_data(case: Case):
    p = case.p
    x = signed_data(case, (p["n"], p["c"], 1, p["plane"]))
    s = (_rng(case).uniform(1, 31, 1 if p["shared"] else p["c"])).astype(F)
    return x, s


def run_norm(case: Case) -> tuple[float, list[str]]:
    p = case.p
    x, s = norm_data(case)
    problems = []
    got, ok = _norm_call(x, s, p, p["in_off"], p["out_off"], p["inplace"])
    if not ok:
        problems.append("wrote outside the output view")
    try:
        used = normalize_check(torch.from_numpy(x), torch.from_numpy(s), torch.from_numpy(got), p["sp"], p["ch"],
                               p["eps"], p["eps_mode"])
    except AssertionError:
        used = math.inf
    if used > 1.0:
        problems.append(f"bound used {used:.3g}")
    for n0, n1 in _halves(p["n"]):
        ioff = _flip(p["in_off"])
        inplace = not p["inplace"]
        again, ok = _norm_call(x[n0:n1], s, p, ioff, ioff if inplace else _flip(p["out_off"]), inplace)
        if not ok or not _bits_eq(again, got[n0:n1]):
            problems.append(f"images {n0}..{n1 - 1} differ with alignment flipped / in place {int(inplace)}")
            used = math.inf
    return used, problems


# ---- LRN -------------------------------------------------------------------------------------------------------------
def _lrn_call(x, p, in_off, out_off):
    from feathercnn_b200 import booster
    xin, xbuf = _buf(x.size, in_off, x)
    out, obuf = _buf(x.size, out_off)
    booster.lrn(xin.view(x.shape), p["region"], p["size"], p["alpha"], p["beta"], p["bias"], out=out.view(x.shape))
    torch.cuda.synchronize()
    return out.view(x.shape).cpu().numpy(), _guard_ok(obuf, out_off, out.numel()) and _guard_ok(xbuf, in_off, x.size)


def run_lrn(case: Case) -> tuple[float, list[str]]:
    p = case.p
    x = signed_data(case, (p["n"], p["c"], p["h"], p["w"]))
    problems = []
    got, ok = _lrn_call(x, p, p["in_off"], p["out_off"])
    if not ok:
        problems.append("wrote outside the output view")
    try:
        used = max(check_lrn(torch.from_numpy(x), torch.from_numpy(got), p["region"], p["size"], p["alpha"], p["beta"],
                             p["bias"]))
    except AssertionError:
        used = math.inf
    if used > 1.0:
        problems.append(f"bound used {used:.3g}")
    for n0, n1 in _halves(p["n"]):
        again, ok = _lrn_call(x[n0:n1], p, _flip(p["in_off"]), _flip(p["out_off"]))
        if not ok or not _bits_eq(again, got[n0:n1]):
            problems.append(f"images {n0}..{n1 - 1} differ with the alignment flipped")
            used = math.inf
    return used, problems


# ---- routing ---------------------------------------------------------------------------------------------------------
def route_shapes(p):
    """(source shapes, destination shapes) as (batch, outer, extent, inner) collapsed to the tensors booster.route sees."""
    if p["axis"] == 2:
        c = p["outer_c"]
        return ([(p["n"], c, e, p["inner"]) for e in p["srcs"]], [(p["n"], c, e, p["inner"]) for e in p["dsts"]])
    return ([(p["n"], e, p["inner"]) for e in p["srcs"]], [(p["n"], e, p["inner"]) for e in p["dsts"]])


def route_ref(p, xs):
    cat = np.concatenate(xs, axis=p["axis"])
    if p["group"] > 1:
        cat = shuffle_ref(cat, p["group"], p["reverse"])
    outs, b = [], p["begin"]
    for e in p["dsts"]:
        outs.append(np.take(cat, range(b, b + e), axis=p["axis"]))
        b += e
    return outs


def run_route(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p = case.p
    sshapes, dshapes = route_shapes(p)
    rng = _rng(case)
    xs = []
    for sh in sshapes:
        x = rng.standard_normal(sh).astype(F)
        x.reshape(-1)[rng.integers(0, x.size)] = PAYLOAD_NAN[0]
        xs.append(x)
    srcs = [_buf(x.size, o, x)[0].view(x.shape) for x, o in zip(xs, p["offs"]["src"])]
    outs = [_buf(math.prod(sh), o) for sh, o in zip(dshapes, p["offs"]["dst"])]
    booster.route(srcs, p["dsts"], p["group"], p["reverse"], p["begin"], axis=p["axis"],
                  outs=[v.view(sh) for (v, _), sh in zip(outs, dshapes)])
    torch.cuda.synchronize()
    problems = []
    for k, ((v, buf), sh, want, o) in enumerate(zip(outs, dshapes, route_ref(p, xs), p["offs"]["dst"])):
        if not _guard_ok(buf, o, v.numel()):
            problems.append(f"destination {k} written outside its view")
        if not _bits_eq(v.view(sh).cpu().numpy(), want):
            problems.append(f"destination {k} differs")
    return (0.0 if not problems else math.inf), problems


# ---- PixelShuffle ----------------------------------------------------------------------------------------------------
def ps_expected(p, x, base):
    r, h, w = p["r"], p["h"], p["w"]
    y = pixel_shuffle_ref(x, r, p["mode"])
    if base is None:
        return y
    ah, aw = base.shape[2:]
    if p["add"][0] == "scale":
        hs = ws = F(1) / F(r)
    else:
        hs, ws = F(ah) / F(h * r), F(aw) / F(w * r)
    return (y + upsample_ref(base, h * r, w * r, hs, ws)).astype(F)


def ps_inputs(case: Case):
    p = case.p
    shape = (p["n"], p["oc"] * p["r"] ** 2, p["h"], p["w"])
    if not p["add"]:
        return copy_data(case, shape), None
    rng = _rng(case)
    x = rng.standard_normal(shape).astype(F)
    ah, aw = p["add"][1:]
    return x, rng.standard_normal((p["n"], p["oc"], ah, aw)).astype(F)


def run_ps(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p = case.p
    x, base = ps_inputs(case)
    r = p["r"]
    oshape = (p["n"], p["oc"], p["h"] * r, p["w"] * r)
    out, obuf = _buf(math.prod(oshape), p["out_off"])
    scale = float(r) if p["add"] and p["add"][0] == "scale" else None
    booster.pixel_shuffle(torch.from_numpy(x).cuda(), r, p["mode"], None if base is None else torch.from_numpy(base).cuda(),
                          scale, out=out.view(oshape))
    torch.cuda.synchronize()
    problems = [] if _guard_ok(obuf, p["out_off"], out.numel()) else ["wrote outside the output view"]
    if not _bits_eq(out.view(oshape).cpu().numpy(), ps_expected(p, x, base)):
        problems.append("differs from pixel_shuffle_ref" + (" + upsample_ref" if base is not None else ""))
    return (0.0 if not problems else math.inf), problems


# ---- BinaryOp --------------------------------------------------------------------------------------------------------
def bin_inputs(case: Case):
    p = case.p
    rng = _rng(case)
    sa = (p["n"],) + p["a"]
    sb = None if p["b"] is None else (p["n"],) + p["b"]
    op = p["op"]
    if op in (6, 9):             # base and exponent
        base_on_a = op == 6
        a = rng.uniform(0.05, 4.0, sa) if base_on_a else rng.uniform(-4, 4, sa)
        b = None if sb is None else (rng.uniform(-4, 4, sb) if base_on_a else rng.uniform(0.05, 4.0, sb))
        return a.astype(F), None if b is None else b.astype(F)
    if op in (10, 11):
        return rng.standard_normal(sa).astype(F), None if sb is None else rng.standard_normal(sb).astype(F)
    a = rng.standard_normal(sa).astype(F)
    b = None if sb is None else rng.standard_normal(sb).astype(F)
    if a.size < 10 ** 6:        # specials on both sides (test_gpu_binary_op)
        for t in (a, b):
            if t is not None:
                flat = t.reshape(-1)
                k = min(flat.size, 2 * len(SPECIALS))
                flat[rng.choice(flat.size, k, replace=False)] = np.resize(SPECIALS, k)
    return a, b


def bin_expected(p, a, b) -> np.ndarray:
    bb = np.full_like(a, F(p["scalar"])) if b is None else b
    return binary_ref(a, bb, p["op"], p["relu"])


def bin_ref64(p, a, b):
    a64 = a.astype(np.float64)
    b64 = np.full_like(a64, float(np.float32(p["scalar"]))) if b is None else b.astype(np.float64)
    ref = {6: lambda: np.power(a64, b64), 9: lambda: np.power(b64, a64), 10: lambda: np.arctan2(a64, b64),
           11: lambda: np.arctan2(b64, a64)}[p["op"]]()
    return np.maximum(ref, 0.0) if p["relu"] else ref


def run_binop(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p = case.p
    a, b = bin_inputs(case)
    if p["rank1"]:               # the shape rule places a rank-1 blob of c values on the channel axis
        _, out_chw, a_al, b_al = booster.binary_op_shape(3, p["a"], 1, (1, 1, p["a"][0]))
        assert tuple(b_al) == p["b"] and tuple(out_chw) == p["a"], (out_chw, b_al)
    oshape = (p["n"],) + (tuple(max(x, y) for x, y in zip(p["a"], p["b"])) if p["b"] is not None else p["a"])
    av, abuf = _buf(a.size, p["offs"][0], a)
    bv, bbuf = (None, None) if b is None else _buf(b.size, p["offs"][1], b)
    if p["inplace"] == "a":
        out, obuf = av, abuf
    elif p["inplace"] == "b":
        out, obuf = bv, bbuf
    else:
        out, obuf = _buf(math.prod(oshape), p["offs"][2])
    booster.binary_op(av.view(a.shape), p["scalar"] if b is None else bv.view(b.shape), p["op"], p["relu"],
                      out=out.view(oshape))
    torch.cuda.synchronize()
    problems = [] if _guard_ok(obuf, p["offs"][2], out.numel()) else ["wrote outside the output view"]
    got = out.view(oshape).cpu().numpy()
    used = 0.0
    if p["op"] in TRANSCENDENTAL:
        bound = 4 if p["op"] in (6, 9) else 3
        ref = np.broadcast_to(bin_ref64(p, a, b), oshape)
        worst = int(_ulps(got, ref).max()) if np.isfinite(got).all() else 1 << 30
        used = worst / bound
        if used > 1.0:
            problems.append(f"{worst} ulp, bound {bound}")
    elif not _same_or_nan(got, bin_expected(p, a, b)):
        problems.append("differs from binary_ref")
        used = math.inf
    return used, problems


# ---- activations -----------------------------------------------------------------------------------------------------
def act_inputs(case: Case) -> np.ndarray:
    from test_gpu_activation import _inputs
    p = case.p
    x = _inputs(case.idx, max(1, p["n"] // 6 + 1), p["alpha"], p["beta"])
    if x.size < p["n"]:
        x = np.resize(x, p["n"])
    perm = _rng(case).permutation(x.size)
    return np.ascontiguousarray(x[perm][:p["n"]])


def run_act(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p = case.p
    x = act_inputs(case)
    xin, xbuf = _buf(x.size, p["in_off"], x)
    out, obuf = (xin, xbuf) if p["inplace"] else _buf(x.size, p["out_off"])
    booster.activation(xin, p["kind"], p["alpha"], p["beta"], out=out)
    torch.cuda.synchronize()
    problems = [] if _guard_ok(obuf, p["out_off"], out.numel()) else ["wrote outside the output view"]
    got = out.cpu()
    try:
        used = _within(got, torch.from_numpy(x), p["kind"], p["alpha"], p["beta"])
    except AssertionError as e:
        used = math.inf
        problems.append(f"outside fcuda.h's bound: {e}")
    if p["kind"].startswith("Hard"):
        g, want = got.numpy(), hard_np(x, p["kind"], p["alpha"], p["beta"])
        nan = np.isnan(want)
        if not (np.array_equal(np.isnan(g), nan) and np.array_equal(_bits(g[~nan]), _bits(want[~nan]))):
            problems.append("differs from hard_np")
            used = math.inf
    return used, problems


RUNNERS = {"in": run_in, "pad": run_pad, "norm": run_norm, "lrn": run_lrn, "route": run_route, "ps": run_ps,
           "binop": run_binop, "act": run_act}


def _ids():
    return [cs.name for cs in (gen_case(i) for i in range(CASES_RUN))]


@gpu
@pytest.mark.parametrize("i", range(CASES_RUN), ids=_ids())
def test_memory_bound_sweep(cuda, i):
    case = cases()[i]
    used, problems = RUNNERS[case.family](case)
    _record(labels(case), used)
    assert not problems, f"{literal(case)}\n  " + "\n  ".join(problems)


# ---- rejections ------------------------------------------------------------------------------------------------------
@gpu
def test_rejections_leave_the_output_untouched(cuda):
    """Arguments the C ABI rejects before any launch, on real device buffers: the documented code, and the output view
    (and, where the output is the input, the input) still as it was."""
    import ctypes

    from feathercnn_b200._lib import FcudaPad, fcuda
    lib = fcuda()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    x, _ = _buf(2 * 3 * 5 * 6, 1, np.arange(180, dtype=F))
    out, obuf = _buf(2 * 3 * 9 * 10, 2)
    ws = torch.zeros(64, device="cuda")
    before = x.clone()
    calls = {
        "instance norm, reflect pad = h": lambda: lib.fcuda_instance_norm_forward(
            P(out), P(x), 3, 5, 6, None, None, 1e-5, 0, ctypes.byref(FcudaPad(5, 0, 0, 0, 2, 0.0)), P(ws), 2, s),
        "instance norm, reflect pad = w + 1": lambda: lib.fcuda_instance_norm_forward(
            P(out), P(x), 3, 5, 6, None, None, 1e-5, 0, ctypes.byref(FcudaPad(0, 0, 0, 7, 2, 0.0)), P(ws), 2, s),
        "padding, reflect pad = w": lambda: lib.fcuda_padding_forward(
            P(out), P(x), 3, 5, 6, ctypes.byref(FcudaPad(0, 0, 6, 0, 2, 0.0)), 2, s),
        "lrn, even local_size": lambda: lib.fcuda_lrn_forward(P(out), P(x), 3, 5, 6, 0, 4, 1.0, 0.75, 1.0, 2, s),
        "lrn within, even local_size": lambda: lib.fcuda_lrn_forward(P(out), P(x), 3, 5, 6, 1, 2, 1.0, 0.75, 1.0, 2, s),
        "lrn, output == input": lambda: lib.fcuda_lrn_forward(P(x), P(x), 3, 5, 6, 0, 5, 1.0, 0.75, 1.0, 2, s),
        "pixel shuffle, C < r^2": lambda: lib.fcuda_pixel_shuffle_forward(P(out), P(x), 3, 5, 6, 2, 0, None, None, 2, s),
        "pixel shuffle, C % r^2": lambda: lib.fcuda_pixel_shuffle_forward(P(out), P(x), 6, 5, 3, 2, 0, None, None, 2, s),
        "pixel shuffle, C % r^2 (mode 1)": lambda: lib.fcuda_pixel_shuffle_forward(P(out), P(x), 6, 5, 3, 2, 1, None,
                                                                                 None, 2, s),
    }
    i4 = ctypes.c_int * 4
    calls["binary op over an operand that broadcasts (a)"] = lambda: lib.fcuda_binary_op_forward(
        P(x), P(x), i4(2, 3, 1, 6), P(out), i4(2, 3, 5, 6), 0.0, 1, 0, s)
    calls["binary op over an operand that broadcasts (b)"] = lambda: lib.fcuda_binary_op_forward(
        P(x), P(out), i4(2, 3, 5, 6), P(x), i4(2, 1, 5, 6), 0.0, 2, 0, s)
    for what, call in calls.items():
        rc = call()
        torch.cuda.synchronize()
        assert rc == -200, (what, rc)
        assert torch.isnan(obuf).all(), what
        assert torch.equal(x.view(torch.int32), before.view(torch.int32)), what


# ---- coverage of the generated list (CPU) ----------------------------------------------------------------------------
# cells that cannot occur:
#   - InstanceNorm stats scalar with an unpadded VEC apply: unpadded, the apply kernel is VEC only when the stats kernel
#     is (its float4 loads read the same input);
#   - Normalize's L2 fallback at tp > 32: tp doubles only while C * 2 tp <= 8192, and the fallback needs C * tp > 32768.
EXPECTED_CELLS = (
    [("instance-norm", f"stats-{s}/{a}") for s in ("vec", "scalar")
     for a in ("pad-vec", "pad-scalar", "nopad-vec", "nopad-scalar") if (s, a) != ("scalar", "nopad-vec")]
    + [("padding", f"{a}-{v}") for a in ("pad", "nopad") for v in ("vec", "scalar")]
    + [("norm-pixel", f"tp{t}-{s}") for t in (32, 64, 128, 256) for s in ("stage4", "stage16")]
    + [("norm-pixel", "tp32-l2")]
    + [(f"norm-{m}", k) for m in ("image", "plane") for k in ("k1", "k2-32", "k33+")]
    + [("lrn-across", f"L{L}-V{v}") for L in (1, 3, 5, 7) for v in (4, 1)] + [("lrn-across", "generic")]
    + [("lrn-within", k) for k in ("staged", "recomputed")]
    + [(f"route-{k}", v) for k in ("concat", "shuffle", "slice", "chain") for v in ("v4", "v1")]
    + [(f"pixel-shuffle-{k}", v) for k in ("copy", "add") for v in ("vec", "scalar")]
    + [("binop-same", k) for k in ("vec", "scalar", "eltwise")] + [("binop-bcast", k) for k in ("row4", "row")]
    + [(f"act-{k}", v) for k in ACT_KINDS for v in ("vec", "scalar")]
)


def test_sweep_hits_every_cell():
    cells: dict = {}
    for cs in cases():
        cell = labels(cs)
        cells[cell] = cells.get(cell, 0) + 1
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
    if SCALE < 1:
        pytest.skip("a scaled-down sweep need not cover every boundary")
    S = cases()
    fam = lambda f: [cs.p for cs in S if cs.family == f]  # noqa: E731
    # InstanceNorm
    ins = fam("in")
    geo = [(p, in_geometry(p)) for p in ins]
    assert _both(ins, lambda p: in_kernels(p)[0] == "vec")
    assert _both([p for p in ins if p["h"] * p["w"] % 4 == 0], lambda p: _al(p["in_off"]))     # alignment flips it
    assert {1, 2} <= {g[4] for _, g in geo} and any(g[4] > 32 for _, g in geo)                # K = 1, 2 and > 32
    assert any(g[0] > 262144 for _, g in geo)
    assert any(g[4] != g[5] for _, g in geo)                                                   # K2 != K
    assert any(g[4] > 1 and g[0] % CHUNK for _, g in geo)                                      # a short last chunk
    padded = [(p, g) for p, g in geo if p["pad"] and any(p["pad"][:4])]
    assert any(g[3] % 4 != g[0] % 4 for _, g in padded)                                        # So % 4 != S % 4
    assert any(p["pad"][4] == 2 and (max(p["pad"][:2]) == p["h"] - 1 or max(p["pad"][2:4]) == p["w"] - 1)
               for p, _ in padded if p["h"] > 1)                                               # reflect at n - 1
    assert {0, 1, 2} <= {p["pad"][4] for p, _ in padded}
    assert any(p["pad"][4] == 0 and p["relu"] and p["pad"][5] < 0 for p, _ in padded)        # a border not ReLU'd
    assert _both(ins, lambda p: p["affine"]) and _both(ins, lambda p: p["relu"]) and _both(ins, lambda p: p["inplace"])
    assert len({p["eps"] for p in ins}) >= 3
    pads = fam("pad")
    assert _both([p for p in pads if any(p["pad"][:4])], lambda p: in_kernels(p)[1].endswith("vec"))
    assert {0, 1, 2} <= {p["pad"][4] for p in pads}
    # Normalize
    nm = fam("norm")
    pix = [p for p in nm if not p["sp"]]
    assert {32, 64, 128, 256} <= {1 << pixel_tile_shift(p["c"], p["plane"]) for p in pix}
    assert {1024, 1025} <= {p["c"] for p in pix}
    assert _both([p for p in pix if p["c"] <= 1024 and p["plane"] % 4 == 0], lambda p: norm_kernel(p)[1].endswith("16"))
    assert _both([p for p in pix if p["c"] <= 1024], lambda p: p["plane"] % 4 == 0)
    assert any(p["plane"] > (1 << pixel_tile_shift(p["c"], p["plane"])) and
               p["plane"] % (1 << pixel_tile_shift(p["c"], p["plane"])) for p in pix)         # a partial last tile
    assert any(p["plane"] < 32 for p in pix)
    for ch in (0, 1):
        segs = [p["plane"] * (p["c"] if ch else 1) for p in nm if p["sp"] and p["ch"] == ch]
        assert any(s % CHUNK == 0 for s in segs) and any(s % CHUNK == 1 for s in segs) and any(s > 32 * CHUNK for s in segs)
    assert _both(nm, lambda p: p["shared"]) and _both(nm, lambda p: p["inplace"])
    assert {p["eps_mode"] for p in nm} == {0, 1, 2}
    # LRN
    lr = fam("lrn")
    across = [p for p in lr if p["region"] == 0]
    assert {1, 3, 5, 7} <= {p["size"] for p in across} and any(p["size"] >= 9 for p in across)
    assert any(p["c"] < p["size"] for p in across) and any(p["c"] < 8 for p in across)
    assert any((p["c"] + p["size"] // 2) % p["size"] for p in across if p["size"] > 1)
    assert any(p["n"] > 1 and (p["h"] * p["w"] // (4 if lrn_kernel(p)[1].endswith("V4") else 1)) % 128
               for p in across if p["size"] <= 7)                                              # groups straddle images
    within = [p for p in lr if p["region"] == 1]
    assert _both(within, lambda p: lrn_kernel(p)[1] == "staged")
    assert any(p["size"] >= 89 for p in within if lrn_kernel(p)[1] == "recomputed")
    assert any(p["h"] < 16 and p["w"] < 32 for p in within)
    assert any(p["size"] // 2 >= max(p["h"], p["w"]) for p in within)
    assert _both(lr, lambda p: p["alpha"] > 0.5)
    # routing
    rt = fam("route")
    assert {len(p["srcs"]) for p in rt if p["target"] == "concat"} >= {1, 8}
    assert any(len(set(p["srcs"])) > 1 for p in rt)
    assert any(p["group"] > 1 and p["group"] ** 2 != sum(p["srcs"]) for p in rt)
    assert _both([p for p in rt if p["group"] > 1], lambda p: p["reverse"])
    assert any(p["begin"] > 0 for p in rt if p["target"] == "slice") and any(len(p["dsts"]) == 8 for p in rt)
    assert any(p["inner"] == 1 for p in rt)
    one_bad = [p for p in rt if p["inner"] % 4 == 0 and sum(not _al(o) for v in p["offs"].values() for o in v) == 1]
    assert any(not _al(o) for p in one_bad for o in p["offs"]["dst"]) and any(len(p["dsts"]) > 1 for p in one_bad)
    # PixelShuffle
    ps = fam("ps")
    assert {1, 2, 3, 4} <= {p["r"] for p in ps} and {0, 1} <= {p["mode"] for p in ps}
    assert _both(ps, lambda p: p["n"] * p["oc"] > PLANES_Y)
    assert {"scale", "size"} <= {p["add"][0] for p in ps if p["add"]}
    assert _both([p for p in ps if (p["w"] * p["r"]) % 4 == 0], lambda p: _al(p["out_off"]))
    # BinaryOp
    bo = fam("binop")
    assert {(p["op"], p["relu"]) for p in bo} == {(o, r) for o in range(12) for r in (False, True)}
    same = [p for p in bo if bin_kernel(p)[0] == "binop-same" and bin_kernel(p)[1] != "eltwise"]
    assert _both(same, lambda p: p["scalar"] is None) and {1, 2, 3} <= {math.prod(p["a"]) * p["n"] % 4 for p in same}
    assert _both(same, lambda p: p["n"] * math.prod(p["a"]) > GRID_CAP)
    bc = [p for p in bo if bin_kernel(p)[0] == "binop-bcast"]
    for ax in range(3):
        assert any(p["a"][ax] == 1 < p["b"][ax] for p in bc) and any(p["b"][ax] == 1 < p["a"][ax] for p in bc), ax
    assert any(any(x == 1 < y for x, y in zip(p["a"], p["b"])) and any(y == 1 < x for x, y in zip(p["a"], p["b"]))
               for p in bc)                                                                     # both sides at once
    assert any(p["rank1"] and p["a"][0] in p["a"][1:] for p in bo)
    assert {"a", "b"} <= {p["inplace"] for p in bo}
    # activations
    ac = fam("act")
    for kind in ACT_KINDS:
        mine = [p for p in ac if p["kind"] == kind]
        assert _both(mine, lambda p: p["n"] > GRID_CAP) and _both(mine, lambda p: p["inplace"]), kind
        assert any(p["n"] < 4 for p in mine), kind
    assert {0.2, PNNX_ALPHA} <= {p["alpha"] for p in ac if p["kind"] == "HardSwish"}
    assert {0.2, PNNX_ALPHA} <= {p["alpha"] for p in ac if p["kind"] == "HardSigmoid"}


# ---- the checkers bite (CPU) -----------------------------------------------------------------------------------------
def _first(pred, n=3, family=None):
    out = [cs for cs in (gen_case(i) for i in range(N_CASES)) if (family is None or cs.family == family) and pred(cs)]
    assert len(out) >= n, len(out)
    return out[:n]


def _in_equal_weights(x, g, b, eps):
    """float64 InstanceNorm whose Chan combination weighs every chunk as a full 8192 (wrong only on a short last chunk)."""
    n, c, h, w = x.shape
    v = x.astype(np.float64).reshape(n, c, -1)
    S = v.shape[2]
    sums, m2s = [], []
    for k0 in range(0, S, CHUNK):
        ck = v[..., k0:k0 + CHUNK]
        sums.append(ck.sum(-1))
        m2s.append(((ck - ck.mean(-1, keepdims=True)) ** 2).sum(-1))
    mean = sum(sums) / S
    var = sum(m2 + CHUNK * (s / CHUNK - mean) ** 2 for s, m2 in zip(sums, m2s)) / S
    gg = np.ones(c) if g is None else g.astype(np.float64)
    bb = np.zeros(c) if b is None else b.astype(np.float64)
    a = gg[None, :] / np.sqrt(var + eps)
    return (a[..., None] * (v - mean[..., None]) + bb[None, :, None]).reshape(x.shape)


SHORT_CHUNK = _first(lambda cs: cs.p["target"] == "short" and cs.p["shift"] != 0, family="in")


@pytest.mark.parametrize("cs", SHORT_CHUNK, ids=[cs.name for cs in SHORT_CHUNK])
def test_checker_rejects_equal_chunk_weights(cs):
    x, g, b = in_data(cs)
    y64, bound = instance_norm_bound(x, g, b, cs.p["eps"])
    good = dataclasses.replace(cs, p=dict(cs.p, relu=False, pad=None))
    assert in_bound_used(good.p, x, g, b, y64.astype(F)) <= 1.0
    assert in_bound_used(good.p, x, g, b, _in_equal_weights(x, g, b, cs.p["eps"])) > 1.0


REFLECT = _first(lambda cs: cs.p["pad"] is not None and cs.p["pad"][4] == 2 and any(cs.p["pad"][:4]), family="pad")


@pytest.mark.parametrize("cs", REFLECT, ids=[cs.name for cs in REFLECT])
def test_checker_rejects_reflect_that_repeats_the_edge(cs):
    p = cs.p
    x = copy_data(cs, (p["n"], p["c"], p["h"], p["w"]))
    t, bo, le, ri = p["pad"][:4]
    bad = np.pad(x, [(0, 0), (0, 0), (t, bo), (le, ri)], mode="symmetric")
    assert not _bits_eq(bad, pad_ref(x, t, bo, le, ri, 2))


SEAMS = _first(lambda cs: not cs.p["sp"] and cs.p["plane"] > (1 << pixel_tile_shift(cs.p["c"], cs.p["plane"])),
               family="norm")


@pytest.mark.parametrize("cs", SEAMS, ids=[cs.name for cs in SEAMS])
def test_checker_rejects_factor_from_the_neighbouring_pixel_at_a_seam(cs):
    p = cs.p
    x, s = norm_data(cs)
    tp = 1 << pixel_tile_shift(p["c"], p["plane"])
    want, ssum = normalize_ref(x, s, 0, 1, p["eps"], p["eps_mode"])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    assert normalize_check(t(x), t(s), t(want.astype(F)), 0, 1, p["eps"], p["eps_mode"]) <= 1.0
    ss = ssum.reshape(p["n"], 1, -1).copy()
    ss[..., tp] = ss[..., tp - 1]                       # the first pixel of tile 1 takes pixel tp - 1's factor
    scale = s.astype(np.float64).reshape(1, -1, 1) if s.size > 1 else float(s[0])
    e = float(F(p["eps"]))
    a = (1 / np.sqrt(ss + e), 1 / np.maximum(np.sqrt(ss), e), 1 / np.sqrt(np.maximum(ss, e)))[p["eps_mode"]]
    bad = (x.astype(np.float64).reshape(p["n"], p["c"], -1) * a * scale).reshape(x.shape)
    assert normalize_check(t(x), t(s), t(bad.astype(F)), 0, 1, p["eps"], p["eps_mode"]) > 1.0


DROP_LAST = _first(lambda cs: cs.p["region"] == 0 and cs.p["alpha"] > 0.5 and cs.p["size"] > 1 and cs.p["c"] > 1 and
                   cs.p["n"] * cs.p["c"] * cs.p["h"] * cs.p["w"] < 40000, family="lrn")


@pytest.mark.parametrize("cs", DROP_LAST, ids=[cs.name for cs in DROP_LAST])
def test_checker_rejects_window_without_the_last_channel(cs):
    p = cs.p
    x = signed_data(cs, (p["n"], p["c"], p["h"], p["w"]))
    c, r = p["c"], p["size"] // 2
    xd = x.astype(np.float64)
    sq = xd * xd
    ss = np.stack([sq[:, max(0, q - r):min(c - 1, q + r) + 1].sum(1) for q in range(c)], 1)
    al, be, bi = (float(F(v)) for v in (p["alpha"], p["beta"], p["bias"]))
    good = xd * (bi + al / p["size"] * ss) ** -be
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    assert max(check_lrn(t(x), t(good.astype(F)), 0, p["size"], p["alpha"], p["beta"], p["bias"])) <= 1.0
    for q in range(max(0, c - 1 - r), c):
        ss[:, q] -= sq[:, c - 1]
    bad = xd * (bi + al / p["size"] * ss) ** -be
    assert max(check_lrn(t(x), t(bad.astype(F)), 0, p["size"], p["alpha"], p["beta"], p["bias"])) > 1.0


SWAPPED_G = _first(lambda cs: cs.p["group"] > 1 and cs.p["group"] ** 2 != sum(cs.p["srcs"]), family="route")


@pytest.mark.parametrize("cs", SWAPPED_G, ids=[cs.name for cs in SWAPPED_G])
def test_checker_rejects_group_and_channels_per_group_swapped(cs):
    p = cs.p
    x = np.arange(p["n"] * sum(p["srcs"]) * p["inner"], dtype=F).reshape(p["n"], sum(p["srcs"]), p["inner"])
    good = shuffle_ref(x, p["group"], p["reverse"])
    assert not _bits_eq(shuffle_ref(x, sum(p["srcs"]) // p["group"], p["reverse"]), good)


MODES = _first(lambda cs: cs.p["r"] > 1 and cs.p["oc"] > 1 and cs.p["n"] < 10, family="ps")


@pytest.mark.parametrize("cs", MODES, ids=[cs.name for cs in MODES])
def test_checker_rejects_modes_swapped(cs):
    p = cs.p
    x, base = ps_inputs(cs)
    want = ps_expected(p, x, base)
    bad = ps_expected(dict(p, mode=1 - p["mode"]), x, base)
    assert not _bits_eq(bad, want)


ROWS = _first(lambda cs: cs.p["b"] is not None and cs.p["op"] not in TRANSCENDENTAL and cs.p["b"][:2] == (1, 1) and
              cs.p["b"][2] > 1, family="binop")


@pytest.mark.parametrize("cs", ROWS, ids=[cs.name for cs in ROWS])
def test_checker_rejects_row_operand_read_at_column_zero(cs):
    p = cs.p
    a, b = bin_inputs(cs)
    want = bin_expected(p, a, b)
    bad = bin_expected(p, a, np.ascontiguousarray(np.broadcast_to(b[..., :1], b.shape)))
    assert not _same_or_nan(bad, want)


# ---- feather::Net: the fusions of these layers -------------------------------------------------------------------------
# Seeded small nets from the three fusion patterns of these layers, each block's layers adjacent:
#   - InstanceNorm (-> ReLU) (-> Padding), the InstanceNorm reading the input;
#   - two or three adjacent layers of Concat (axis 0) -> ShuffleChannel -> Slice (axis 0);
#   - PixelShuffle of one slice of the input plus the nearest Interp of another, joined by Eltwise SUM or BinaryOp ADD (the
#     Interp's input computed before the PixelShuffle, or, in a share of the nets, after it; a bilinear Interp in another).
# In a share of the nets a Dropout at the end of the net reads an intermediate blob a second time, which must block the
# fusion that would have removed it.
N_NETS = max(4, int(round(12 * SCALE)))
NET_SETTINGS = [(f, g, rf) for f in (False, True) for g in (False, True) for rf in (0, 1)]


def _net_blocks(r, m, C, oc, rr, H, W):
    """The three blocks' layer writers, in a seeded order; returns the intermediate blobs a second reader may take."""
    inter = []

    def in_block():
        top = m.instance_norm("inorm", "data", eps=r.choice([1e-5, 1e-3]), affine=r.random() < 0.7)
        if r.random() < 0.7:
            inter.append(top)
            top = m.relu("in_relu", top)
        if r.random() < 0.7:
            inter.append(top)
            type_ = r.choice([0, 1, 2])
            pads = [r.randint(0, 2) for _ in range(4)]
            if type_ == 2:
                pads = [min(p, H - 1) for p in pads[:2]] + [min(p, W - 1) for p in pads[2:]]
            m.padding("in_pad", top, *pads, type_=type_, value=r.choice([0.0, -1.5]))

    def route_block():
        kind = r.choice(["cat-sh-sl", "cat-sh", "sh-sl", "cat-sl"])
        blob = "data"
        if kind.startswith("cat"):
            blob = m.concat("cat", r.choice([["data", "xs_1"], ["xs_0", "data", "xs_1"], ["xs_0", "xs_1"]]))
        mid = m.shape[blob][0]
        if "sh" in kind:
            inter.append(blob)
            groups = [g for g in range(2, mid) if mid % g == 0] or [1]
            blob = m.shuffle_channel("sh", blob, r.choice(groups), r.randint(0, 1))
        if "sl" in kind:
            inter.append(blob)
            first = r.randint(1, max(1, mid // 3))
            sizes = [first, -233] + ([1] if r.random() < 0.5 and mid - first >= 2 else [])
            m.slice("sl", blob, sizes)

    def ps_block():
        late = r.random() < 0.2                      # the Interp's input computed after the PixelShuffle: no tail
        if not late:
            m.slice("ys", "data", [oc * rr * rr, -233], tops=["ys_0", "y"])
        ps = m.pixel_shuffle("ps", "xs_0", rr, r.randint(0, 1))
        if late:
            m.slice("ys", "data", [oc * rr * rr, -233], tops=["ys_0", "y"])
        if r.random() < 0.15:
            up = m.interp("up", "y", 2, out_h=H * rr, out_w=W * rr)
        elif r.random() < 0.5:
            up = m.interp("up", "y", 1, scale=float(rr))
        else:
            up = m.interp("up", "y", 1, out_h=H * rr, out_w=W * rr)
        inter.extend([ps, up])
        pair = [ps, up] if r.random() < 0.5 else [up, ps]
        m.add("sum", pair)

    blocks = [in_block, route_block, ps_block]
    r.shuffle(blocks)
    for b in blocks:
        b()
    return inter


def gen_net(i: int):
    """(ModelWriter, input batch) of net i."""
    from feathercnn_b200.tools import modelgen
    r = random.Random(zlib.crc32(f"memory-bound-net-{i}".encode()))
    m = modelgen.ModelWriter(seed=i, adds=r.choice(["eltwise", "binaryop"]))
    oc, rr = r.choice([1, 2, 3]), r.choice([1, 2, 3])
    C, H, W = oc * rr * rr + oc, r.randint(2, 9), r.randint(2, 9)
    m.input("data", C, H, W)
    m.slice("xs", "data", [oc * rr * rr, -233])     # xs_0 feeds the PixelShuffle; both halves may feed the Concat
    inter = _net_blocks(r, m, C, oc, rr, H, W)
    if r.random() < 0.45:
        for k, b in enumerate(r.sample(inter, min(len(inter), r.choice([1, 1, 2])))):
            m.dropout(f"again{k}", b, top=f"again{k}")
    assert all(min(shape) > 0 for shape in m.shape.values()), m.lines
    x = np.random.default_rng(i).standard_normal((2, C, H, W)).astype(F)
    return m, x


def _layers_of(lines):
    out = []
    for ln in lines:
        t = ln.split()
        nb, nt = int(t[2]), int(t[3])
        params = dict(kv.split("=", 1) for kv in t[4 + nb + nt:])
        out.append(dict(type=t[0], name=t[1], bottoms=t[4:4 + nb], tops=t[4 + nb:4 + nb + nt], params=params,
                        fused=False, relu=False, pad=False))
    return out


def _accepts(a, b) -> bool:
    """Layer::TryFuse of the fusible producers in these nets (InstanceNorm, Eltwise, BinaryOp)."""
    if a["type"] == "InstanceNorm":
        if a["pad"]:
            return False
        if b["type"] == "ReLU" and not a["relu"]:
            a["relu"] = True
            return True
        if b["type"] == "Padding":
            a["pad"] = True
            return True
        return False
    if b["type"] != "ReLU" or (a["type"] == "BinaryOp" and a["relu"]):
        return False
    a["relu"] = True
    return True


def _plain_sum(e) -> bool:
    if e["fused"] or len(e["bottoms"]) != 2 or len(e["tops"]) != 1:
        return False
    if e["type"] == "Eltwise":
        return e["params"].get("0", "1") == "1" and "-23301" not in e["params"]
    return e["type"] == "BinaryOp" and e["params"].get("0", "0") == "0" and e["params"].get("1", "0") == "0"


def fusion_ref(lines, fusion: bool, route_fuse: int) -> set[str]:
    """The layers Net::ApplyFusion removes from these nets: its first pass (a fusible producer absorbs the adjacent
    layers that read its top when that top has no other reader), the super-resolution tail pass and, with route_fuse, the
    routing pass.  The residual and crop passes take convolutions and deconvolutions, which these nets do not have."""
    if not fusion:
        return set()
    L = _layers_of(lines)
    readers: dict[str, int] = {}
    for lay in L:
        for b in lay["bottoms"]:
            readers[b] = readers.get(b, 0) + 1
    for i, a in enumerate(L):
        if a["fused"] or a["type"] not in ("InstanceNorm", "Eltwise", "BinaryOp") or len(a["tops"]) != 1:
            continue
        for b in L[i + 1:]:
            if b["fused"]:
                continue
            if len(b["bottoms"]) != 1 or len(b["tops"]) != 1 or b["bottoms"][0] != a["tops"][0]:
                break
            if readers.get(a["tops"][0], 0) != 1 or not _accepts(a, b):
                break
            a["tops"] = [b["tops"][0]]
            b["tops"], b["bottoms"], b["fused"] = [], [], True
    producer = {t: i for i, lay in enumerate(L) for t in lay["tops"]}
    for j, e in enumerate(L):
        if not _plain_sum(e) or e["relu"]:
            continue
        for k in (0, 1):
            mine, other = e["bottoms"][k], e["bottoms"][1 - k]
            if mine == other or readers.get(mine) != 1 or readers.get(other) != 1 or mine not in producer or \
                    other not in producer:
                continue
            i, n = producer[mine], producer[other]
            ps, up = L[i], L[n]
            if ps["type"] != "PixelShuffle" or up["type"] != "Interp" or i >= j or n >= j or ps["fused"] or \
                    up["fused"] or len(up["bottoms"]) != 1:
                continue
            base = up["bottoms"][0]
            if base in producer and producer[base] >= i:
                continue
            if up["params"].get("0") != "1":               # PixelShuffleLayer::FuseUpsampledAdd: nearest only
                continue
            producer.pop(mine)
            producer.pop(other)
            ps["tops"] = e["tops"]
            producer[e["tops"][0]] = i
            up["tops"], up["bottoms"], up["fused"] = [], [], True
            e["tops"], e["bottoms"], e["fused"] = [], [], True
            break
    if route_fuse == 1:
        made_by = {t: lay for lay in L for t in lay["tops"]}
        for r_ in L:
            if r_["type"] not in ("ShuffleChannel", "Slice") or r_["fused"] or len(r_["bottoms"]) != 1:
                continue
            if r_["type"] == "Slice" and r_["params"].get("1", "0") != "0":
                continue
            mine = r_["bottoms"][0]
            if readers.get(mine) != 1 or mine not in made_by:
                continue
            p = made_by[mine]
            if p["fused"] or len(p["tops"]) != 1:
                continue
            cat = p["type"] == "Concat"
            sh = r_["type"] == "Slice" and p["type"] == "ShuffleChannel"
            if cat and (p["params"].get("0", "0") != "0" or not p["bottoms"] or len(p["bottoms"]) > 8):
                continue
            if not cat and not sh:
                continue
            r_["bottoms"] = p["bottoms"]
            p["tops"], p["bottoms"], p["fused"] = [], [], True
    return {lay["name"] for lay in L if lay["fused"]}


def _set_route_fuse(v):
    from feathercnn_b200._lib import fcuda
    return fcuda().fcuda_set_tuning(b"route_fuse", v)


@pytest.fixture
def route_fuse_restored():
    from feathercnn_b200._lib import fcuda
    saved = fcuda().fcuda_get_tuning(b"route_fuse")
    yield
    fcuda().fcuda_set_tuning(b"route_fuse", saved)


def _fused_names(net, lines) -> set[str]:
    return {ln.split()[1] for ln in lines if net.LayerFusedAway(ln.split()[1])}


def test_fusion_restatement_matches_the_net(route_fuse_restored):
    """On the host (FuseNow runs no kernel): the restatement predicts every net's fused layers, with fusion and
    route_fuse each on and off."""
    from feathercnn_b200.net import Net
    for i in range(N_NETS):
        m, _ = gen_net(i)
        text = "7767517\n" + f"{len(m.lines)} {len(m.blobs)}\n" + "\n".join(m.lines) + "\n"
        for fusion in (False, True):
            for rf in (0, 1):
                assert _set_route_fuse(rf) == 0
                net = Net(fusion=fusion)
                net.LoadParamFromText(text)
                net.FuseNow()
                assert _fused_names(net, m.lines) == fusion_ref(m.lines, fusion, rf), (i, fusion, rf, m.lines)
                del net


def test_nets_cover_every_fusion_and_every_block():
    """Across the nets, each fusion happens, and each is blocked by a second reader (or, for the tail, by an Interp
    input computed too late and by a bilinear Interp)."""
    seen = set()
    for i in range(N_NETS if SCALE >= 1 else 12):
        m, _ = gen_net(i)
        fused = fusion_ref(m.lines, True, 1)
        L = {lay["name"]: lay for lay in _layers_of(m.lines)}
        again = {lay["bottoms"][0] for lay in L.values() if lay["type"] == "Dropout"}
        for name in ("in_relu", "in_pad", "up", "cat", "sh"):
            if name in L:
                seen.add((name, name in fused))
        if "in_relu" in L and "inorm" in again:
            seen.add(("in_relu-read-twice", "in_relu" in fused))
        if "up" in L:
            order = [lay["name"] for lay in L.values()]
            late = order.index("ys") > order.index("ps")
            twice = bool({"ps", "up"} & again)
            bilinear = L["up"]["params"]["0"] == "2"
            if late or twice or bilinear:
                seen.add(("tail-blocked", "up" in fused))
    for name in ("in_relu", "in_pad", "up", "cat", "sh"):
        assert (name, True) in seen and (name, False) in seen, (name, sorted(seen))
    assert ("in_relu-read-twice", False) in seen and ("tail-blocked", True) not in seen


@gpu
@pytest.mark.parametrize("i", range(N_NETS))
def test_net_fusions_keep_the_bits(cuda, tmp_path, route_fuse_restored, i):
    """Net i with fusion, CUDA graphs and route_fuse each on and off: the layers fused away are the restatement's, and
    every blob materialised in two runs has the same bits in both."""
    from feathercnn_b200.net import Net
    m, x = gen_net(i)
    param, binf = m.save(tmp_path / f"net{i}")
    runs = {}
    for fusion, graph, rf in NET_SETTINGS:
        assert _set_route_fuse(rf) == 0
        net = Net(fusion=fusion, cuda_graph=graph)
        net.LoadParam(param)
        net.LoadWeights(binf)
        for _ in range(3 if graph else 1):
            net.Forward(x)
        net.Synchronize()
        assert _fused_names(net, m.lines) == fusion_ref(m.lines, fusion, rf), (fusion, graph, rf)
        runs[fusion, graph, rf] = {b: net.Extract(b) for b in net.BlobNames()}
        del net
    base = runs[False, False, 1]
    for key, blobs in runs.items():
        shared = [b for b in blobs if b in base]
        assert "data" in shared and len(shared) > 1, key
        for b in shared:
            assert _bits_eq(blobs[b], base[b]), (key, b)
