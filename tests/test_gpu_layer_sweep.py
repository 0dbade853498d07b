"""Seeded random geometries across the deconvolution, Interp / Crop and SSD-head kernel boundaries, against float64.

test_gpu_dispatch_sweep.py does this for the convolution, depthwise and pooling dispatch.  The layers below have their
own predicates and index arithmetic, tested otherwise only on hand-picked lists:

  - Deconvolution (deconv.cu make_plan): the depthwise gather (group == IC == OC; a channel multiplier is not depthwise),
    the stride-1 direct convolution (every pad <= dil * (K - 1), output_pad <= pad on its side) or the sub-pixel phases
    (T = ceil(K / s): K < s, K % s == 0, K = s + 1), mixed strides with dilation on the stride-1 axis, the equivalent
    convolution's tuned algorithm (FCUDA_SGECONV with groups or dilation), the scatter's ty < Hc test (output_pad rows
    get the bias only), pads larger than the kernel, more than 65535 planes (the grid-y loop of the scatter and the
    gather), the gather's filter staging past 256 taps and its Y % stride tap starts, and plans fcuda_deconv_plan rejects.
  - Interp (resize.cu interp_forward): the memcpy shortcut, the float4 stores (OW % 4 == 0 and a 16-byte-aligned output),
    512-column tiles, the band of [1, 64] rows, more than 65535 planes, H or W = 1, size and scale-factor sizing.
  - Crop: the float4 path (woff, W, OW % 4 == 0 and both pointers aligned) against the scalar one, OW around 512.
  - Permute: order 3's 32 x 33 tiled transpose while batch <= 65535, the gather otherwise.
  - Softmax over an axis: one warp per row (inner == 1) or one thread per column.
  - DetectionOutput: the radix select and its ordered tie compaction in chunks of 512 threads, the bitonic sort's padding
    to a power of two, the merge over C * nms_top_k entries against keep_top_k, IoU exactly at the threshold (the test is
    strict), negative scores with a negative threshold and signed zeros.

One deterministic generator; each case seeded from the crc32 of its index.  The checks are the existing ones:
deconv_ref with test_gpu_deconv.bound_coef (and, on a seeded subset, bit equality with the equivalent convolution plus
test_deconv_host.scatter), nearest_ref / bilinear_check, _softmax_check, _decode_ref, and detection_ref fed the kernel's own
decoded boxes, bit for bit.  Interp and Crop run on views 0..3 floats past an aligned allocation through the C ABI; the
output view sits in a NaN-filled buffer whose other floats must stay NaN.

Every case is labelled with the kernel it reaches (plan_ref and the equivalent convolution's tuned choice, restatements of
the Interp / Crop / Permute / Softmax predicates); on the GPU the deconvolution label is also checked against the
algorithm fcuda_deconv_plan reports.  The CPU tests check that the list hits every reachable cell and both sides of every
boundary, and that the checkers reject simulated defects on the sweep's own shapes.  A failing case prints a
ready-to-paste literal for the matching hand-written list.

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

from test_deconv_host import deconv_ref, equivalent_filter, out_dim, plan_ref, scatter
from test_gpu_deconv import Case as Deconv
from test_gpu_deconv import _eq_conv, bound_coef
from test_gpu_error_bounds import (FP32_SPLIT, MODE_NAME, PATH, TF32, TF32X3, U, WINO_MARGIN, WINOGRADF23, WINOGRADF63,
                                   conv_ref, eps_for, excess, wino_model)
from test_gpu_interp_crop import bilinear_check, nearest_ref
from test_gpu_ssd import AXES, _bits_equal, _decode_ref, _random_priors, _softmax_check, _softmax_scores
from test_interp_crop_host import interp_out_dim, nearest_scale
from test_ssd_host import detection_ref, iou32

gpu = pytest.mark.gpu

N_CASES = 600
SCALE = float(os.environ.get("FCUDA_SWEEP_SCALE", "1"))
CASES_RUN = max(1, int(round(N_CASES * SCALE)))

MODES3 = (FP32_SPLIT, TF32X3, TF32)
IC_EDGES = (3, 17, 31, 32, 33, 63, 64, 65)
OCP_EDGES = (31, 32, 33, 63, 64, 65, 127, 128, 129)    # OC * s_h * s_w around the implicit GEMM's N tiles
MAX_TABLE_K = 6144                                       # conv_igemm.cu kMaxTableK
PLANES_Y = 65535                                         # grid-y / grid-z limit of the plane loops


# ---- the generator ----------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    idx: int
    family: str
    mode: int = FP32_SPLIT
    deconv: Deconv | None = None
    equiv: bool = False                  # also bit-compare with the equivalent convolution and the scatter
    p: dict = dataclasses.field(default_factory=dict)    # the other families' parameters
    in_off: int = 0                      # float offsets of the input / output views (Interp and Crop)
    out_off: int = 0

    @property
    def name(self):
        return f"{self.idx:04d}-{self.family}"


def _igemm_ok(icg, kh, kw) -> bool:
    """conv_igemm.cu conv_igemm_supported."""
    return kh * kw <= 63 and (icg % 32 == 0 or kh * kw * icg <= MAX_TABLE_K)


def _fit(c: Deconv) -> Deconv:
    """Shrinks the pads until the output is not empty."""
    while True:
        oh = out_dim(c.h, c.kh, c.stride[0], c.dil[0], c.pad[0], c.pad[1], c.output_pad[0])
        ow = out_dim(c.w, c.kw, c.stride[1], c.dil[1], c.pad[2], c.pad[3], c.output_pad[1])
        if oh > 0 and ow > 0:
            return c
        c.pad = tuple(max(0, p - 1) for p in c.pad)


def _oc_for(r, sh, sw, group):
    ocp = r.choice(OCP_EDGES)
    return max(1, round(ocp / (sh * sw) / group)) * group


def _kernel_for(r, s):
    """Kernel extent along an axis of stride s: K < s (phases without taps), K % s == 0, K = s + 1, or any."""
    return max(1, r.choice([s - 1, s, 2 * s, s + 1, r.randint(1, 7)]))


def _direct_pads(r, e, op_side):
    """(pad_a, pad_b, op) on one axis of the direct path: pads <= e, op <= pad_b."""
    pa, pb = r.randint(0, e), r.randint(0, e)
    return pa, pb, r.randint(0, pb) if op_side else 0


DECONV_TARGETS = ("dw", "direct", "subpixel", "direct-f63", "subpixel", "subpixel-f63", "im2col-direct", "multiplier",
                  "subpixel", "direct", "im2col-subpixel", "dw")


def _gen_deconv(r, k, name) -> tuple[Deconv, int]:
    """(geometry, return code fcuda_deconv_plan must give: 0, or -1 for an equivalent convolution no kernel takes)."""
    bias, relu, batch = r.random() < 0.75, r.random() < 0.4, r.choice([1, 1, 2, 3])
    sp = k % 60
    if sp == 0:      # 2049 * 33 planes through the scatter's grid-y loop
        return Deconv(name, 33, 3, 2, 2, 4, (2, 2), (1, 1, 1, 1), (1, 0), bias=bias, relu=relu, batch=2049), 0
    if sp == 1:      # 21846 * 3 planes through the gather's grid-y loop
        return Deconv(name, 3, 3, 2, 3, 3, (2, 2), (1, 0, 0, 1), (1, 1), group=3, bias=bias, relu=relu, batch=21846), 0
    if sp == 2:      # 17 x 16 = 272 taps: the gather stages its filter in two passes of 256 threads
        return Deconv(name, 4, 4, 3, 4, (17, 16), (8, 8), (4, 5, 3, 4), (1, 2), group=4, bias=bias, relu=relu,
                      batch=batch), 0
    if sp == 3:      # dilated direct path with 9 x 8 taps: the implicit GEMM (forced by the dilation) takes at most 63
        return Deconv(name, 8, 8, 6, 6, (9, 8), (1, 1), (8, 8, 7, 7), (0, 0), (2, 2)), -1
    if sp == 4:      # grouped sub-pixel path, 7 x 7 phase taps on 129 channels per group: the k-table does not fit
        return Deconv(name, 4, 258, 3, 3, 14, (2, 2), (0, 0, 0, 0), group=2), -1
    target = DECONV_TARGETS[k % len(DECONV_TARGETS)]
    if target == "dw":
        ch = r.choice([2, 3, 8, 21, 33])
        stride = r.choice([(1, 1), (2, 2), (1, 2), (2, 1), (3, 3), (4, 2)])
        kh, kw = r.choice([(1, 1), (2, 2), (3, 3), (4, 4), (3, 5), (5, 2), (6, 6), (7, 3)])
        dil = tuple(r.choice([1, 1, 2, 3]) if s == 1 else 1 for s in stride)
        pad = tuple(r.randint(0, max(kh, kw) + 1) for _ in range(4))
        op = (r.randint(0, stride[0]), r.randint(0, stride[1]))
        return _fit(Deconv(name, ch, ch, r.randint(1, 12), r.randint(1, 12), (kh, kw), stride, pad, op, dil, ch, bias,
                           relu, batch)), 0
    if target in ("direct", "direct-f63", "im2col-direct"):
        f63 = target == "direct-f63"
        if f63:
            kh = kw = 3
            dil = (1, 1)
        elif target == "im2col-direct":   # past 63 taps the tuned choice stays on im2col
            kh, kw = r.choice([(8, 8), (9, 8), (7, 10)])
            dil = (1, 1)
        else:
            kh, kw = r.randint(1, 5), r.randint(1, 5)
            dil = (r.choice([1, 1, 2, 3]), r.choice([1, 1, 2, 3]))
        pt, pb, oph = _direct_pads(r, dil[0] * (kh - 1), True)
        pl, pr, opw = _direct_pads(r, dil[1] * (kw - 1), True)
        group = 1 if f63 or target == "im2col-direct" else r.choice([1, 1, 1, 2])
        if target == "im2col-direct":
            icg = r.choice([1, 3, 17, 32])
        else:
            icg = r.choice((4, 8, 32, 64)) if f63 else r.choice(IC_EDGES)
        oc = r.choice((4, 8, 32, 64)) if f63 else _oc_for(r, 1, 1, group)
        h, w = (r.randint(9, 20), r.randint(9, 20)) if f63 else (r.randint(1, 16), r.randint(1, 16))
        return _fit(Deconv(name, oc, icg * group, h, w, (kh, kw), (1, 1), (pt, pb, pl, pr), (oph, opw), dil, group, bias,
                           relu, batch)), 0
    if target == "multiplier":   # group == IC, OC = m * IC: the grouped implicit GEMM, not the gather
        ch, m = r.choice([2, 3, 8]), r.choice([2, 3])
        stride = r.choice([(1, 1), (2, 2), (2, 1)])
        kh, kw = _kernel_for(r, stride[0]), _kernel_for(r, stride[1])
        if stride == (1, 1):
            pt, pb, oph = _direct_pads(r, kh - 1, True)
            pl, pr, opw = _direct_pads(r, kw - 1, True)
            pad, op = (pt, pb, pl, pr), (oph, opw)
        else:
            pad, op = tuple(r.randint(0, 2) for _ in range(4)), (r.randint(0, 1), 0)
        return _fit(Deconv(name, ch * m, ch, r.randint(1, 10), r.randint(1, 10), (kh, kw), stride, pad, op, group=ch,
                           bias=bias, relu=relu, batch=batch)), 0
    # sub-pixel
    if target == "subpixel-f63":
        stride, (kh, kw), dil, group = (2, 2), (r.choice([5, 6]), r.choice([5, 6])), (1, 1), 1
        icg, h, w = r.choice((4, 8, 32, 64)), r.randint(9, 16), r.randint(9, 16)
    elif target == "im2col-subpixel":
        # 8 x 8 phase taps (more than 63), or 7 x 7 on 129 channels (a k-table past 6144 entries): im2col
        stride, dil, group = (2, 2), (1, 1), 1
        kh, kw, icg = r.choice([(15, 16, 3), (16, 16, 17), (16, 15, 1), (14, 13, 129)])
        h, w = r.randint(1, 6), r.randint(1, 6)
    else:
        stride = r.choice([(2, 2), (2, 2), (3, 3), (1, 2), (2, 1), (4, 4), (2, 3), (1, 1), (1, 1)])
        kh, kw = _kernel_for(r, stride[0]), _kernel_for(r, stride[1])
        dil = tuple(r.choice([1, 2, 3]) if s == 1 else 1 for s in stride)
        group, icg = r.choice([1, 1, 1, 2, 4]), r.choice(IC_EDGES)
        h, w = r.randint(1, 14), r.randint(1, 14)
    pad = tuple(r.randint(0, k_ + 1) if r.random() < 0.8 else 0 for k_ in (kh, kh, kw, kw))
    op = (r.randint(0, stride[0]), r.randint(0, stride[1]))
    if stride == (1, 1):
        # stride 1 off the direct path: a pad past dil * (K - 1), or an output pad past its pad
        eh = dil[0] * (kh - 1)
        if r.random() < 0.5:
            pad = (eh + r.choice([1, 1, 2]), r.randint(0, eh), 0, 0)
            op = (0, 0)
        else:
            pb = r.randint(0, eh)
            pad, op = (0, pb, 0, 0), (pb + 1, 0)
    oc = r.choice((4, 8, 16, 32)) if target == "subpixel-f63" else _oc_for(r, *stride, group)
    c = _fit(Deconv(name, oc, icg * group, h, w, (kh, kw), stride, pad, op, dil, group, bias, relu, batch))
    path, e = plan_ref(*c.geometry)
    if (group > 1 or e["dil"] != (1, 1)) and not _igemm_ok(icg, e["kernel_h"], e["kernel_w"]):
        c = dataclasses.replace(c, ic=32 * group)     # keep the random draw runnable; the rejections are pinned above
    return c, 0


INTERP_TARGETS = ("equal", "vec", "scalar", "tile512", "band", "hw1", "scale", "vec", "planes", "scalar")
INTERP_MODES = ("nearest", "bilinear-half", "bilinear-align")


def _gen_interp(r, k) -> dict:
    target = INTERP_TARGETS[k % len(INTERP_TARGETS)]
    mode = INTERP_MODES[(k // len(INTERP_TARGETS)) % 3] if target != "equal" else INTERP_MODES[k % 3]
    n, c = r.choice([1, 2, 3]), r.choice([1, 2, 3, 5])
    h, w = r.randint(2, 24), r.randint(2, 24)
    oh, ow, scale = r.randint(1, 40), r.randint(1, 40), None
    if target == "equal":
        oh, ow = h, w
        if mode == "nearest" and r.random() < 0.5:   # equal size from scale factors other than 1: the kernel runs
            oh = ow = 0
            scale = (1.0 + 0.5 / h, 1.0 + 0.5 / w)
    elif target == "vec":
        ow = 4 * r.randint(1, 40)
    elif target == "scalar":
        ow = 4 * r.randint(1, 40) + r.choice([0, 1, 2, 3])
    elif target == "tile512":
        h, w, n, c = r.randint(1, 3), r.choice([3, 40, 200, 511, 700]), 1, r.choice([1, 2])
        oh, ow = r.randint(1, 5), r.choice([511, 512, 513, 1023, 1024, 1025, 1536])
    elif target == "band":
        oh, ow = r.choice([63, 64, 65, 129]), r.choice([1, 3, 4, 8, 31, 33, 64, 128, 132])
    elif target == "hw1":
        h, w = (1, r.randint(1, 20)) if r.random() < 0.5 else (r.randint(1, 20), 1)
    elif target == "scale":
        oh = ow = 0
        sc = r.choice([0.5, 1 / 3, 2.0, 2.5, 0.3, 8.0, 1.7])
        scale = (sc, r.choice([sc, 0.5, 3.0]))
        h, w = max(h, 4), max(w, 4)
    elif target == "planes":      # more than 65535 planes: the grid-z loop
        n, c, h, w = 2, 32769, r.randint(1, 2), r.randint(1, 3)
        oh, ow = r.randint(1, 3), r.randint(1, 4)
    if scale is not None:
        scale = tuple(float(np.float32(v)) for v in scale)
    return dict(mode=mode, n=n, c=c, h=h, w=w, oh=oh, ow=ow, scale=scale, target=target)


CROP_TARGETS = ("vec", "scalar", "wide", "scalar", "wide")


def _gen_crop(r, k) -> dict:
    target = CROP_TARGETS[k % len(CROP_TARGETS)]
    n, c = r.choice([1, 2, 3]), r.randint(1, 5)
    coff = r.randint(0, c - 1)
    oc = r.randint(1, c - coff)
    if target == "wide":
        ow = r.choice([508, 511, 512, 513, 516, 1023, 1025])
        h, oh = r.randint(1, 3), 1
    else:
        ow, h = r.randint(1, 40), r.randint(1, 12)
        oh = r.randint(1, h)
    if target == "scalar" or r.random() < 0.3:
        woff, w = r.randint(0, 5), 0
    else:
        ow, woff = -(-ow // 4) * 4, 4 * r.randint(0, 2)
        w = 0
    w = woff + ow + (r.choice([0, 4, 8]) if target != "scalar" else r.randint(0, 5))
    if target == "vec":
        w = -(-w // 4) * 4
    return dict(n=n, c=c, h=h, w=w, coff=coff, hoff=r.randint(0, h - oh), woff=woff, oc=oc, oh=oh, ow=ow, target=target)


PERMUTE_HW = [(1, 1), (1, 31), (1, 32), (4, 8), (3, 11), (5, 13), (1, 33), (8, 8), (6, 6), (2, 17)]


def _gen_permute(r, k) -> dict:
    order = k % 6
    if k % 60 == 3:       # order 3 past the grid-z limit: the gather takes it
        return dict(order=3, n=65536, c=1, h=1, w=1)
    if k % 60 == 9:
        return dict(order=3, n=65535, c=1, h=1, w=1)
    if k % 60 in (15, 21):
        return dict(order=3, n=65537, c=2, h=1, w=1) if k % 60 == 15 else dict(order=3, n=65600, c=1, h=2, w=1)
    h, w = r.choice(PERMUTE_HW)
    return dict(order=order, n=r.choice([1, 2, 3]), c=r.choice([1, 2, 31, 32, 33, 64, 65]), h=h, w=w)


def _gen_softmax(r, k) -> dict:
    if k % 2 == 0:
        length = r.choice([1, 31, 32, 33, 64, 65, 100, 1000, 8732])
        outer, inner = (r.randint(1, 300) if length <= 100 else r.randint(1, 8)), 1
    else:
        length, inner, outer = r.choice([1, 5, 21, 33]), r.choice([2, 7, 31, 32, 33, 300]), r.randint(1, 20)
    return dict(n=r.choice([1, 2, 3]), outer=outer, len=length, inner=inner, gain=r.choice([1.0, 6.0, 30.0]))


def _gen_decode(r, k) -> dict:
    return dict(P=r.choice([1, 7, 255, 256, 257, 1917]), n=r.choice([1, 2, 3]), gain=r.choice([0.5, 2.0, 4.0]))


DET_TARGETS = ("random", "select", "ties", "bitonic", "merge", "iou_eq", "negative", "select", "merge", "random")
TOP_KS = (1, 1024, 2, 63, 513, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 64, 65, 127, 128, 129, 255, 256, 257, 511,
          512, 1023)   # nms_top_k of the bitonic cases in turn: 1, 2^j and 2^j +- 1 up to 1024


def _gen_detect(r, k) -> dict:
    if k % 25 == 24:      # the large cases: detection_ref is a Python loop
        return dict(target="large", seed=r.getrandbits(32), n=1, P=8732, C=21, top=400, keep=200)
    target = DET_TARGETS[k % len(DET_TARGETS)]
    d = dict(target=target, seed=r.getrandbits(32), n=r.choice([1, 2, 3]))
    if target == "random":
        d.update(P=r.randint(5, 700), C=r.randint(2, 8), top=r.choice([1, 10, 100, 300]), keep=r.choice([1, 20, 100, 500]))
    elif target == "select":
        j = k // len(DET_TARGETS) * 2 + (k % len(DET_TARGETS) > 1)      # counts the select cases
        P = (511, 512, 513, 1024, 1025, 1536)[j % 6]
        top = min(r.choice([100, 200, 511, 512, 513]), P - 1)
        d.update(P=P, C=r.choice([2, 3]), top=top, keep=r.choice([50, 1024]), quantized=r.random() < 0.5,
                 valid=top + (-1, 0, 1)[j % 3])
    elif target == "ties":
        d.update(P=r.randint(300, 1100), C=r.choice([2, 4]), top=r.choice([50, 300, 512, 600]), keep=r.choice([100, 600]))
    elif target == "bitonic":
        top = TOP_KS[k // len(DET_TARGETS) % len(TOP_KS)]
        d.update(P=top + r.randint(0, 40), C=2, top=top, keep=r.choice([1, top, 1024]))
    elif target == "merge":
        d.update(P=r.randint(10, 120), C=r.randint(3, 6), top=r.choice([1, 5, 16, 50]), keep_side=r.choice([-1, 0, 1]))
    elif target == "iou_eq":
        d.update(pairs=r.randint(3, 40), C=r.choice([2, 3]), top=r.choice([16, 100]), keep=100)
    else:
        d.update(P=r.randint(20, 300), C=r.choice([2, 3, 5]), top=r.choice([8, 100, 256]), keep=r.choice([10, 300]),
                 thr=r.choice([-0.5, -1.0]))
    return d


SLOTS = ["deconv", "interp", "deconv", "crop", "permute", "deconv", "softmax", "interp", "deconv", "detect", "decode",
         "deconv"]


def gen_case(i: int) -> Case:
    """Case i.  k counts the cases of its family; the deconvolution cycles its targets with k and the precision mode
    with k // 12 (every target in every mode in 36 cases)."""
    r = random.Random(zlib.crc32(f"layer-sweep-{i}".encode()))
    fam = SLOTS[i % len(SLOTS)]
    k = i // len(SLOTS) * SLOTS.count(fam) + SLOTS[:i % len(SLOTS)].count(fam)
    if fam == "deconv":
        c, rc = _gen_deconv(r, k, f"lsweep{i}")
        case = Case(i, fam, MODES3[(k // len(DECONV_TARGETS)) % 3], deconv=c, p=dict(reject=rc))
        case.equiv = rc == 0 and plan_ref(*c.geometry)[0] != "dw" and c.batch * c.oc <= PLANES_Y and r.random() < 0.3
        return case
    gen = {"interp": _gen_interp, "crop": _gen_crop, "permute": _gen_permute, "softmax": _gen_softmax,
           "decode": _gen_decode, "detect": _gen_detect}[fam]
    case = Case(i, fam, p=gen(r, k))
    if fam in ("interp", "crop") and case.p["target"] not in ("vec",) and r.random() < 0.5:
        case.in_off, case.out_off = r.randint(0, 3), r.randint(0, 3)
    return case


# ---- what runs where -------------------------------------------------------------------------------------------------
def _lib():
    from feathercnn_b200._lib import fcuda
    return fcuda()


def deconv_label(c: Deconv) -> tuple[str, str]:
    """(path, algorithm) from plan_ref and the equivalent convolution's tuned choice (fcuda_conv_select_algo_tuned),
    FCUDA_SGECONV with groups or dilation; ("reject", "-") where that convolution fails conv_igemm_supported."""
    from feathercnn_b200._lib import FcudaConvParam
    path, e = plan_ref(*c.geometry)
    if path == "dw":
        return "dw", "gather"
    if c.group > 1 or e["dil"] != (1, 1):
        return (path, "sgeconv") if _igemm_ok(c.ic // c.group, e["kernel_h"], e["kernel_w"]) else ("reject", "-")
    p = FcudaConvParam(output_channels=e["output_channels"], input_channels=c.ic, input_h=c.h, input_w=c.w,
                       kernel_h=e["kernel_h"], kernel_w=e["kernel_w"], output_h=e["output_h"], output_w=e["output_w"],
                       stride_h=1, stride_w=1, pad_left=e["pad_left"], pad_bottom=e["pad_bottom"],
                       pad_right=e["pad_right"], pad_top=e["pad_top"], group=1)
    a = ctypes.c_int(-1)
    assert _lib().fcuda_conv_select_algo_tuned(ctypes.byref(p), ctypes.byref(a)) == 0, c
    return path, PATH[a.value]


def interp_geometry(p) -> tuple[int, int, float, float]:
    """(OH, OW, hs, ws): the output size and nearest's fp32 scales (test_interp_crop_host)."""
    hs_f, ws_f = p["scale"] if p["scale"] is not None else (1.0, 1.0)
    oh, ow = interp_out_dim(p["h"], p["w"], p["oh"], p["ow"], hs_f, ws_f)
    explicit = p["oh"] > 0 and p["ow"] > 0
    return oh, ow, nearest_scale(p["h"], oh, explicit, hs_f), nearest_scale(p["w"], ow, explicit, ws_f)


def interp_kernel(p, out_off=0) -> str:
    """resize.cu interp_forward: memcpy (equal size, bilinear or unit nearest scales), vec (OW % 4 == 0 and a 16-byte
    aligned output), scalar."""
    oh, ow, hs, ws = interp_geometry(p)
    if (oh, ow) == (p["h"], p["w"]) and (p["mode"] != "nearest" or (hs == 1 and ws == 1)):
        return "memcpy"
    return "vec" if ow % 4 == 0 and (4 * out_off) % 16 == 0 else "scalar"


def interp_band(p, out_off=0) -> int:
    oh, ow, _, _ = interp_geometry(p)
    groups = min(ow, 512) // (4 if interp_kernel(p, out_off) == "vec" else 1)
    return max(1, min(64, 2048 // groups))


def crop_kernel(p, in_off=0, out_off=0) -> str:
    vec = p["woff"] % 4 == 0 and p["w"] % 4 == 0 and p["ow"] % 4 == 0 and in_off % 4 == 0 and out_off % 4 == 0
    return "vec" if vec else "scalar"


def permute_kernel(p) -> str:
    if p["order"] == 0:
        return "memcpy"
    return "transpose" if p["order"] == 3 and p["n"] <= PLANES_Y else "gather"


def labels(case: Case) -> tuple[str, str, str]:
    """(family-path, kernel, mode) cell of a case."""
    p = case.p
    if case.family == "deconv":
        path, algo = deconv_label(case.deconv)
        free = path in ("dw", "reject")
        return f"deconv-{path}", algo, "any" if free else MODE_NAME[case.mode]
    if case.family == "interp":
        return f"interp-{p['mode']}", interp_kernel(p, case.out_off), "any"
    if case.family == "crop":
        return "crop", crop_kernel(p, case.in_off, case.out_off), "any"
    if case.family == "permute":
        return f"permute-{p['order']}", permute_kernel(p), "any"
    if case.family == "softmax":
        return "softmax", "rows" if p["inner"] == 1 else "cols", "any"
    if case.family == "decode":
        return "decode", "-", "any"
    return "detect", p["target"], "any"


_CASES = None


def cases() -> list[Case]:
    global _CASES
    if _CASES is None:
        _CASES = [gen_case(i) for i in range(CASES_RUN)]
    return _CASES


def literal(case: Case) -> str:
    """A ready-to-paste entry for the matching hand-written list."""
    p = case.p
    if case.family == "deconv":
        c = case.deconv
        d = Deconv("x", 1, 1, 1, 1)
        kw = [f"{f.name}={getattr(c, f.name)!r}" for f in dataclasses.fields(Deconv)[5:] if getattr(c, f.name) != getattr(d, f.name)]
        return f"Case({c.name!r}, {c.oc}, {c.ic}, {c.h}, {c.w}" + "".join(", " + s for s in kw) + f")  # {MODE_NAME[case.mode]}"
    if case.family == "interp":
        return (f"({case.name!r}, {p['n']}, {p['c']}, {p['h']}, {p['w']}, {p['oh']}, {p['ow']}, {p['scale']!r})"
                f"  # {p['mode']}, offsets in / out {case.in_off} / {case.out_off}")
    if case.family == "crop":
        return (f"({case.name!r}, {p['n']}, {p['c']}, {p['h']}, {p['w']}, {p['coff']}, {p['hoff']}, {p['woff']}, {p['oc']}, "
                f"{p['oh']}, {p['ow']})  # offsets in / out {case.in_off} / {case.out_off}")
    if case.family == "permute":
        return f"order {p['order']}, shape {(p['n'], p['c'], p['h'], p['w'])}"
    if case.family == "softmax":
        return f"({p['outer']}, {p['len']}, {p['inner']})  # batch {p['n']}, gain {p['gain']}"
    return f"{case.family} {p!r}"


# ---- data ------------------------------------------------------------------------------------------------------------
def _gen(case: Case) -> np.random.Generator:
    return np.random.default_rng(zlib.crc32(case.name.encode()))


def _grid_priors(P, size=0.0625):
    """P dyadic boxes of edge `size` on a grid two edges apart: no two overlap, and decode with loc 0 returns them
    exactly (every sum and product of the decode is exact)."""
    per_row = 16
    j = np.arange(P)
    x0, y0 = (j % per_row) * 2 * size, (j // per_row) * 2 * size
    boxes = np.stack([x0, y0, x0 + size, y0 + size], 1).astype(np.float32).reshape(-1)
    return np.stack([boxes, np.tile(np.float32([0.1, 0.1, 0.2, 0.2]), P)])


def det_data(case: Case):
    """(loc, conf, priors, C, conf_threshold, nms_threshold, nms_top_k, keep_top_k) of a DetectionOutput case."""
    p, rng = case.p, np.random.default_rng(case.p["seed"])
    t, n = p["target"], p["n"]
    if t == "iou_eq":
        # pairs of dyadic boxes: A = [x, y, x + s, y + s] and B shifted by s/2 (IoU 1/3, exactly the threshold: kept), or
        # by s/4 (IoU 3/5 > threshold: suppressed); pairs 2s apart do not overlap
        s = np.float32(0.0625)
        boxes = []
        for j in range(p["pairs"]):
            x, y = np.float32((j % 8) * 3 * s), np.float32((j // 8) * 3 * s)
            dx = s / 2 if j % 3 else s / 4
            boxes += [[x, y, x + s, y + s], [x + dx, y, x + dx + s, y + s]]
        b = np.array(boxes, np.float32)
        P, C = len(b), p["C"]
        priors = np.stack([b.reshape(-1), np.tile(np.float32([0.1, 0.1, 0.2, 0.2]), P)])
        area = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
        nms = float(iou32(b[2], area[2], b[3:4], area[3:4])[0])     # pair 1: B shifted by s / 2
        conf = rng.uniform(0.05, 1.0, (n, P * C)).astype(np.float32)
        return np.zeros((n, 4 * P), np.float32), conf, priors, C, 0.01, nms, p["top"], p["keep"]
    P, C, top = p["P"], p["C"], p["top"]
    loc = (rng.standard_normal((n, 4 * P)) * 0.5).astype(np.float32)
    priors = _random_priors(rng, P)
    thr, nms = 0.05, 0.45
    if t in ("random", "large"):
        conf = _softmax_scores(rng, n, P, C, 3.0)
        thr, nms = (0.01, 0.45) if t == "large" else (float(rng.choice([0.01, 0.05, 0.2])), float(rng.choice([0.3, 0.45, 0.6])))
    elif t == "select":
        # exactly `valid` candidates per class above the threshold, the others below; quantized scores make tie runs
        # that cross the 512-thread chunks of the compaction
        conf = rng.uniform(0.0, 0.1, (n, P, C)).astype(np.float32)
        for i in range(n):
            for c in range(1, C):
                idx = rng.permutation(P)[:p["valid"]]
                v = rng.uniform(0.3, 1.0, len(idx))
                conf[i, idx, c] = (np.ceil(v * 4) / 4 if p["quantized"] else v).astype(np.float32)
        conf, thr = conf.reshape(n, -1), 0.2
    elif t == "ties":
        conf = (rng.integers(1, 5, (n, P * C)) / 8).astype(np.float32)
        base = _random_priors(rng, 40)
        priors = np.tile(base.reshape(2, 40, 4), (1, -(-P // 40), 1))[:, :P].reshape(2, -1)
        loc, thr, nms = loc * 0.3, 0.2, 0.5
    elif t == "bitonic":
        conf, thr = rng.uniform(0.01, 1.0, (n, P * C)).astype(np.float32), 0.0
    elif t == "merge":
        conf = rng.uniform(0.0, 1.0, (n, P * C)).astype(np.float32)
        priors, loc, thr = _grid_priors(P), np.zeros((n, 4 * P), np.float32), 0.5
    else:   # negative scores, signed zeros and duplicate boxes under a negative threshold
        levels = np.float32([-0.0, 0.0, -0.0, 0.0, -0.25, -0.125, 0.5, -2.0])
        conf = levels[rng.integers(0, len(levels), (n, P * C))]
        base = _random_priors(rng, max(1, P // 3))
        priors = np.tile(base.reshape(2, -1, 4), (1, 3, 1))[:, :P].reshape(2, -1)
        if priors.shape[1] < 4 * P:
            priors = np.concatenate([priors, _random_priors(rng, P - priors.shape[1] // 4)], 1)
        loc, thr = np.zeros((n, 4 * P), np.float32), p["thr"]
    keep = p.get("keep")
    if t == "merge":
        kept = merge_kept(conf, P, C, thr, top)
        keep = int(min(1024, max(1, kept.min() + p["keep_side"])))
    return loc, conf, priors, C, thr, nms, top, keep


def merge_kept(conf, P, C, thr, top) -> np.ndarray:
    """Detections per image of a merge case (boxes that never overlap: every candidate of the nms_top_k survives)."""
    valid = (conf.reshape(conf.shape[0], P, C)[..., 1:] > np.float32(thr)).sum(1)
    return np.minimum(valid, top).sum(1)


def class_valid(conf, P, C, thr) -> np.ndarray:
    return (conf.reshape(conf.shape[0], P, C)[..., 1:] > np.float32(thr)).sum(1)


# ---- report ----------------------------------------------------------------------------------------------------------
REPORT: dict[tuple[str, str, str], list] = {}


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\ncases and the largest share of the per-element bound used (0 for bit-exact checks), per cell:")
        for (f, k, m), (n, used) in sorted(REPORT.items()):
            print(f"  {f:18s} {k:12s} {m:9s} {n:4d} cases   bound used {used:.3f}")


def _record(cell, used):
    r = REPORT.setdefault(cell, [0, 0.0])
    r[0] += 1
    r[1] = max(r[1], used)


# ---- running a case on the GPU ---------------------------------------------------------------------------------------
def _view(n: int, off: int, src=None):
    """n floats starting `off` floats into a larger allocation, and that allocation (NaN-filled for outputs)."""
    buf = torch.full((n + 8,), math.nan, device="cuda") if src is None else torch.zeros(n + 8, device="cuda")
    v = buf[off:off + n]
    if src is not None:
        v.copy_(src.reshape(-1))
    return v, buf


def _guard_ok(buf, off, n) -> bool:
    return bool(torch.isnan(buf[:off]).all() and torch.isnan(buf[off + n:]).all())


def _P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _equivalent_conv(eq, algo, x, wp, b, dil):
    """The equivalent convolution on its own through the ConvBooster protocol, with per-axis dilation."""
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import FcudaConvOptions
    cb = booster.ConvBooster()
    cb.ForceSelectAlgo(algo)
    n = x.shape[0]
    s, k = cb.GetBufferSize(eq, n)
    packed = torch.empty(max(k, 1), device="cuda")
    scratch = torch.empty(max(s, 1), device="cuda")
    cb.Init(eq, packed, wp.contiguous())
    out = torch.empty((n, eq.output_channels, eq.output_h, eq.output_w), device="cuda")
    o = FcudaConvOptions(dilation_h=dil[0], dilation_w=dil[1])
    rc = _lib().fcuda_conv_forward_opts(ctypes.byref(eq), algo, _P(out), _P(x.contiguous()), _P(packed), _P(scratch), _P(b),
                                        ctypes.byref(o), n, _stream())
    assert rc == 0, rc
    return out


def deconv_bound(c: Deconv, mode: int, algo: int, x, w, b):
    """(coef, S) of |got - ref| <= coef * S + 2^-23 |ref|: bound_coef and the S of deconv_ref, except on a Winograd
    equivalent convolution.  Its transforms mix the outputs of a tile, so an output whose taps all land in the padding
    (S = 0; the sub-pixel pads T - 1 and pads past the kernel make these) still carries its neighbours' rounding.  There
    S is the equivalent convolution's S maximised over each output tile (test_gpu_dispatch_sweep.tile_max), scattered,
    plus |b|, and the Winograd model's worst |d| / S is taken against that S."""
    s = deconv_ref(x, w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, absolute=True)
    if algo not in (WINOGRADF63, WINOGRADF23):
        return bound_coef(c, mode, algo, x, w), s
    from feathercnn_b200 import booster
    from test_gpu_dispatch_sweep import tile_max
    path, _ = plan_ref(*c.geometry)
    eq, _ = booster.deconv_plan(booster.deconv_param(*c.geometry[:6], c.stride, c.pad, c.output_pad, c.dil, c.group))
    cc = _eq_conv(eq, w)
    wp = torch.from_numpy(equivalent_filter(w.numpy(), c.stride, c.group, path).copy())
    st = tile_max(conv_ref(cc, x, wp, None, None, absolute=True), 6 if algo == WINOGRADF63 else 2)
    ym = wino_model(cc, x[:1], wp, None, 8 if algo == WINOGRADF63 else 4, mode)
    _, rho = excess(ym, conv_ref(cc, x[:1], wp, None, None), st[:1], 1.0)
    if path == "subpixel":
        st = scatter(st, c.oc, c.group, c.stride, c.pad, tuple(s.shape[2:]))
    if b is not None:
        st = st + b.double().abs().view(1, -1, 1, 1)
    return WINO_MARGIN * rho, st


def run_deconv(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    c = case.deconv
    problems = []
    p = booster.deconv_param(*c.geometry[:6], c.stride, c.pad, c.output_pad, c.dil, c.group, c.bias, c.relu)
    path, algo_name = deconv_label(c)
    eq, algo = booster.FcudaConvParam(), ctypes.c_int(-7)
    rc = _lib().fcuda_deconv_plan(ctypes.byref(p), ctypes.byref(eq), ctypes.byref(algo))
    if case.p["reject"]:
        if rc != case.p["reject"] or path != "reject":
            problems.append(f"fcuda_deconv_plan returned {rc}, label {path}; want {case.p['reject']}")
        return 0.0, problems
    want_algo = "depthwise" if path == "dw" else algo_name
    if rc != 0 or PATH.get(algo.value) != want_algo:
        problems.append(f"fcuda_deconv_plan: rc {rc}, algorithm {PATH.get(algo.value)}, label {want_algo}")
        return math.inf, problems
    booster.set_precision(case.mode)
    x, w, b = c.data()
    bc = None if b is None else b.cuda()
    got, a = booster.deconv_forward(x.cuda(), w.cuda(), bc, c.stride, c.pad, c.output_pad, c.dil, c.group, c.relu)
    torch.cuda.synchronize()
    coef, s = deconv_bound(c, case.mode, a, x, w, b)
    ref = deconv_ref(x, w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, c.relu)
    gc = got.cpu()
    used = excess(gc, ref, s, coef)[0] if torch.isfinite(gc).all() else math.inf
    if used > 1.0:
        problems.append(f"bound used {used:.3g}")
    if case.equiv:
        _, e = plan_ref(*c.geometry)
        wp = torch.from_numpy(equivalent_filter(w.numpy(), c.stride, c.group, path).copy()).cuda()
        out = _equivalent_conv(eq, algo.value, x.cuda(), wp, bc if path == "direct" else None, e["dil"])
        if path == "subpixel":
            want = scatter(out, c.oc, c.group, c.stride, c.pad, tuple(got.shape[2:]))
            if bc is not None:
                want = want + bc.view(1, -1, 1, 1)
            if c.relu:
                want = torch.where(want > 0, want, torch.zeros_like(want))
        else:
            want = out
        torch.cuda.synchronize()
        if not torch.equal(got.view(torch.int32), want.contiguous().view(torch.int32)):
            problems.append("differs from the equivalent convolution + scatter")
    return used, problems


def _data(case: Case, shape):
    g = torch.Generator().manual_seed(zlib.crc32(case.name.encode()))
    return torch.rand(shape, generator=g) * 2 - 1


def run_interp(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p = case.p
    n, c, h, w = p["n"], p["c"], p["h"], p["w"]
    mode, align = ("nearest", False) if p["mode"] == "nearest" else ("bilinear", p["mode"] == "bilinear-align")
    prm = booster.interp_param(h, w, p["oh"], p["ow"], mode, align, p["scale"])
    oh, ow, hs, ws = interp_geometry(p)
    problems = []
    if (prm.output_h, prm.output_w) != (oh, ow):
        return math.inf, [f"output {prm.output_h} x {prm.output_w}, want {oh} x {ow}"]
    x = _data(case, (n, c, h, w))
    xin, _ = _view(x.numel(), case.in_off, x.cuda())
    out, obuf = _view(n * c * oh * ow, case.out_off)
    rc = _lib().fcuda_interp_forward(ctypes.byref(prm), _P(out), _P(xin), c, n, _stream())
    torch.cuda.synchronize()
    assert rc == 0, rc
    if not _guard_ok(obuf, case.out_off, out.numel()):
        problems.append("wrote outside the output view")
    got = out.view(n, c, oh, ow).cpu()
    if mode == "nearest":
        used = 0.0
        if not np.array_equal(got.numpy().view(np.int32), nearest_ref(x.numpy(), oh, ow, hs, ws).view(np.int32)):
            used = math.inf
            problems.append("nearest differs from the fp32 gather")
    else:
        used = bilinear_check(got, x, int(align))[0] if torch.isfinite(got).all() else math.inf
        if used > 1.0:
            problems.append(f"bilinear bound used {used:.3g}")
    return used, problems


def run_crop(case: Case) -> tuple[float, list[str]]:
    p = case.p
    n, c, h, w = p["n"], p["c"], p["h"], p["w"]
    x = _data(case, (n, c, h, w))
    xin, _ = _view(x.numel(), case.in_off, x.cuda())
    out, obuf = _view(n * p["oc"] * p["oh"] * p["ow"], case.out_off)
    rc = _lib().fcuda_crop_forward(_P(out), _P(xin), c, h, w, p["coff"], p["hoff"], p["woff"], p["oc"], p["oh"], p["ow"],
                                   n, _stream())
    torch.cuda.synchronize()
    assert rc == 0, rc
    problems = [] if _guard_ok(obuf, case.out_off, out.numel()) else ["wrote outside the output view"]
    want = x[:, p["coff"]:p["coff"] + p["oc"], p["hoff"]:p["hoff"] + p["oh"], p["woff"]:p["woff"] + p["ow"]]
    if not torch.equal(out.view(n, p["oc"], p["oh"], p["ow"]).cpu(), want):
        problems.append("crop differs")
    return 0.0 if not problems else math.inf, problems


def run_permute(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p = case.p
    x = _data(case, (p["n"], p["c"], p["h"], p["w"]))
    got = booster.permute(x.cuda(), p["order"]).cpu().numpy()
    want = np.transpose(x.numpy(), (0,) + tuple(a + 1 for a in AXES[p["order"]]))
    return (0.0, []) if _bits_equal(got, want) else (math.inf, ["permute differs"])


def run_softmax(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p = case.p
    x = _data(case, (p["n"], p["outer"], p["len"], p["inner"])) * p["gain"]
    got = booster.softmax_axis(x.cuda(), p["outer"], p["len"], p["inner"]).cpu().numpy().astype(np.float64)
    try:
        return _softmax_check(x.numpy().astype(np.float64), got, 2), []
    except AssertionError as e:
        return math.inf, [f"softmax bound: {e}"]


def run_decode(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    p, rng = case.p, _gen(case)
    priors = _random_priors(rng, p["P"])
    loc = (rng.standard_normal((p["n"], 4 * p["P"])) * p["gain"]).astype(np.float32)
    got = booster.ssd_decode(torch.from_numpy(loc).cuda(), torch.from_numpy(priors).cuda()).cpu().numpy()
    want, bound = _decode_ref(loc, priors)
    used = float((np.abs(got - want) / bound).max())
    return used, [] if used <= 1.0 else [f"decode bound used {used:.3g}"]


def run_detect(case: Case) -> tuple[float, list[str]]:
    from feathercnn_b200 import booster
    loc, conf, priors, C, thr, nms, top, keep = det_data(case)
    dl, dc, dp = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (loc, conf, priors))
    boxes = booster.ssd_decode(dl, dp).cpu().numpy()
    got = booster.detection_output(dl, dc, dp, C, thr, nms, top, keep).cpu().numpy()
    want, _ = detection_ref(boxes, conf, C, np.float32(thr), np.float32(nms), top, keep)
    if _bits_equal(got, want):
        return 0.0, []
    bad = np.argwhere(got.view(np.int32) != want.view(np.int32))[:4]
    return math.inf, [f"detections differ at {bad.tolist()}: got {[got[tuple(b[:2])].tolist() for b in bad]}, "
                      f"want {[want[tuple(b[:2])].tolist() for b in bad]}"]


RUNNERS = {"deconv": run_deconv, "interp": run_interp, "crop": run_crop, "permute": run_permute, "softmax": run_softmax,
           "decode": run_decode, "detect": run_detect}


def _ids():
    return [cs.name for cs in (gen_case(i) for i in range(CASES_RUN))]


@gpu
@pytest.mark.parametrize("i", range(CASES_RUN), ids=_ids())
def test_layer_sweep(cuda, i):
    case = cases()[i]
    used, problems = RUNNERS[case.family](case)
    _record(labels(case), used)
    assert not problems, f"{literal(case)}\n  " + "\n  ".join(problems)


# ---- feather::Net: every Deconvolution parameter id set, and a folded crop --------------------------------------------
# ncnn ids: 0 OC, 1 / 11 kernel w / h, 2 / 12 dilation w / h, 3 / 13 stride w / h, 4 / 15 / 14 / 16 pad left / right /
# top / bottom, 18 / 19 output pad right / bottom, 5 bias, 6 weight count, 7 group, 9 activation.  Every pair differs,
# so a swapped id changes the output.
NET_LAYERS = [
    # (type, name, top, ncnn params, the same geometry as a test_gpu_deconv Case)
    ("Deconvolution", "dA", "dA", "0=6 1=3 11=4 2=2 12=1 3=1 13=2 4=1 15=3 14=2 16=0 18=1 19=1 5=1 6=144 7=2 9=1",
     Deconv("dA", 6, 4, 7, 6, (4, 3), (2, 1), (2, 0, 1, 3), (1, 1), (1, 2), 2, True, True, 3)),
    ("DeconvolutionDepthWise", "dB", "dB", "0=4 1=4 11=3 2=1 12=2 3=2 13=1 4=0 15=2 14=1 16=3 18=1 19=0 5=1 6=48 7=4 9=1",
     Deconv("dB", 4, 4, 7, 6, (3, 4), (1, 2), (1, 3, 0, 2), (0, 1), (2, 1), 4, True, True, 3)),
    ("DeconvolutionDepthWise", "dC", "dC", "0=8 1=2 11=3 3=2 13=2 4=1 15=0 14=0 16=1 18=1 19=1 5=0 6=48 7=4",
     Deconv("dC", 8, 4, 7, 6, (3, 2), (2, 2), (0, 1, 1, 0), (1, 1), (1, 1), 4, False, False, 3)),
    ("Deconvolution", "dD", "dD", "0=5 1=4 11=3 3=2 13=2 4=1 15=1 14=1 16=1 5=1 6=240",
     Deconv("dD", 5, 4, 7, 6, (3, 4), (2, 2), (1, 1, 1, 1), (0, 0), (1, 1), 1, True, False, 3)),
]
NET_CROP = (2, 1, 7, 9)     # woff, hoff, out w, out h of the Crop after dD (folds into its pads)


def _net_model(tmp_path):
    rng = np.random.default_rng(23)
    lines = ["Input data 0 1 data 0=6 1=7 2=4"]
    binf = bytearray()
    weights = {}
    for typ, name, top, prm, c in NET_LAYERS:
        lines.append(f"{typ} {name} 1 1 data {top} {prm}")
        w = (rng.standard_normal((c.oc, c.ic // c.group, c.kh, c.kw)) * 0.4).astype(np.float32)
        b = rng.uniform(-0.5, 0.5, c.oc).astype(np.float32) if c.bias else None
        binf += np.uint32(0).tobytes() + w.tobytes() + (b.tobytes() if b is not None else b"")
        weights[name] = (torch.from_numpy(w), None if b is None else torch.from_numpy(b))
    lines += ["ReLU rC 1 1 dC dC_relu", "Crop cD 1 1 dD cD 0=%d 1=%d 3=%d 4=%d" % NET_CROP]
    text = f"7767517\n{len(lines)} {len(lines)}\n" + "\n".join(lines) + "\n"     # one top per layer
    (tmp_path / "net.param").write_text(text)
    (tmp_path / "net.bin").write_bytes(bytes(binf))
    return str(tmp_path / "net.param"), str(tmp_path / "net.bin"), weights


@gpu
def test_net_deconvolution_parameter_ids(cuda, tmp_path):
    from feathercnn_b200 import booster
    from feathercnn_b200.net import Net
    param, binf, weights = _net_model(tmp_path)
    x = (np.random.default_rng(5).uniform(-1, 1, (3, 4, 7, 6))).astype(np.float32)
    xt = torch.from_numpy(x)
    outs = {}
    for fusion in (False, True):
        for graph in (False, True):
            net = Net(fusion=fusion, cuda_graph=graph)
            net.LoadParam(param)
            net.LoadWeights(binf)
            for _ in range(3 if graph else 1):
                net.Forward(x)
            assert net.LayerFusedAway("cD") == int(fusion)
            outs[fusion, graph] = {b: net.Extract(b) for b in ("dA", "dB", "dC_relu", "cD")}
            for typ, name, top, prm, c in NET_LAYERS:
                w, b = weights[name]
                _, algo = booster.deconv_plan(booster.deconv_param(*c.geometry[:6], c.stride, c.pad, c.output_pad, c.dil,
                                                                   c.group))
                coef = bound_coef(c, FP32_SPLIT, algo, xt, w)
                ref = deconv_ref(xt, w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, c.relu)
                s = deconv_ref(xt, w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, absolute=True)
                blob = {"dC": "dC_relu", "dD": "cD"}.get(name, name)
                if name == "dC":
                    ref = ref.clamp_min(0)
                if name == "dD":
                    wo, ho, cw, ch = NET_CROP
                    ref, s = ref[..., ho:ho + ch, wo:wo + cw], s[..., ho:ho + ch, wo:wo + cw]
                got = torch.from_numpy(outs[fusion, graph][blob]).double().reshape(ref.shape)
                used, _ = excess(got, ref, s, coef)
                assert used <= 1.0, (name, fusion, graph, used)
            del net
    for key, o in outs.items():   # the folded crop and the fused ReLU are bit-identical to the unfused net
        for b in o:
            assert np.array_equal(o[b].view(np.int32), outs[False, False][b].view(np.int32)), (key, b)


# ---- coverage of the generated list (CPU) ----------------------------------------------------------------------------
# cells that cannot occur:
#   - the gather and the rejections are mode-free ("any"): the gather is fp32 FMA, a rejection runs nothing;
#   - Permute order 0 is one memcpy, orders 1, 2, 4, 5 always the gather, order 3 the transpose or (batch > 65535) the
#     gather.
EXPECTED_CELLS = (
    [("deconv-dw", "gather", "any"), ("deconv-reject", "-", "any")]
    + [(f"deconv-{p}", a, m) for p in ("direct", "subpixel") for a in ("sgeconv", "im2col", "f63")
       for m in MODE_NAME.values()]
    + [(f"interp-{m}", k, "any") for m in INTERP_MODES for k in ("memcpy", "vec", "scalar")]
    + [("crop", k, "any") for k in ("vec", "scalar")]
    + [("permute-0", "memcpy", "any"), ("permute-3", "transpose", "any"), ("permute-3", "gather", "any")]
    + [(f"permute-{o}", "gather", "any") for o in (1, 2, 4, 5)]
    + [("softmax", k, "any") for k in ("rows", "cols")]
    + [("decode", "-", "any")]
    + [("detect", t, "any") for t in set(DET_TARGETS) | {"large"}]
)


def test_sweep_hits_every_cell():
    pytest.importorskip("feathercnn_b200._lib")
    cells: dict = {}
    for cs in cases():
        cell = labels(cs)
        cells[cell] = cells.get(cell, 0) + 1
    unexpected = sorted(set(cells) - set(EXPECTED_CELLS))
    assert not unexpected, f"cells the coverage table says cannot occur: {unexpected}"
    # every rejection the generator pins is one the label restatement predicts, and only those
    for cs in cases():
        if cs.family == "deconv":
            assert (labels(cs)[0] == "deconv-reject") == bool(cs.p["reject"]), literal(cs)
    if SCALE < 1:
        pytest.skip("a scaled-down sweep need not cover every cell")
    least = {("detect", "large", "any"): 2}       # detection_ref is a Python loop: two large cases
    thin = sorted((cell, cells.get(cell, 0)) for cell in EXPECTED_CELLS if cells.get(cell, 0) < least.get(cell, 3))
    assert not thin, f"cells hit fewer than 3 times: {thin}"


def _both(values, pred) -> bool:
    vs = list(values)
    return any(pred(v) for v in vs) and any(not pred(v) for v in vs)


def _scatter_reads_past_hc(c: Deconv) -> bool:
    """Some output row or column of the sub-pixel path has ty >= Hc (or tx >= Wc): the scatter writes the bias alone."""
    path, e = plan_ref(*c.geometry)
    if path != "subpixel":
        return False
    oh = out_dim(c.h, c.kh, c.stride[0], c.dil[0], c.pad[0], c.pad[1], c.output_pad[0])
    ow = out_dim(c.w, c.kw, c.stride[1], c.dil[1], c.pad[2], c.pad[3], c.output_pad[1])
    return (oh - 1 + c.pad[0]) // c.stride[0] >= e["output_h"] or (ow - 1 + c.pad[2]) // c.stride[1] >= e["output_w"]


def test_sweep_covers_both_sides_of_every_boundary():
    pytest.importorskip("feathercnn_b200._lib")
    if SCALE < 1:
        pytest.skip("a scaled-down sweep need not cover every boundary")
    S = cases()
    have = lambda vals, want: set(want) <= set(vals)  # noqa: E731
    dc = [cs.deconv for cs in S if cs.family == "deconv" and not cs.p["reject"]]
    paths = [(c, plan_ref(*c.geometry)[0]) for c in dc]
    sub = [c for c, p in paths if p == "subpixel"]
    dws = [c for c, p in paths if p == "dw"]
    # the path predicates
    assert any(c.group == c.ic and c.oc != c.ic and c.group > 1 for c, p in paths if p != "dw")     # channel multiplier
    s1 = [(c, p) for c, p in paths if c.stride == (1, 1) and p != "dw"]
    assert _both(s1, lambda cp: cp[1] == "direct")
    assert any(max(c.pad[0], c.pad[1]) == c.dil[0] * (c.kh - 1) for c, p in s1 if p == "direct")   # pad at the edge
    assert any(c.pad[0] == c.dil[0] * (c.kh - 1) + 1 for c, p in s1 if p == "subpixel")            # one past it
    assert any(c.output_pad[0] == c.pad[1] > 0 for c, p in s1 if p == "direct")
    assert any(c.output_pad[0] == c.pad[1] + 1 for c, p in s1 if p == "subpixel")
    for rel in (lambda k, s: k < s, lambda k, s: k % s == 0, lambda k, s: k == s + 1):
        assert any(rel(c.kh, c.stride[0]) for c in sub if c.stride[0] > 1)
    assert any(c.stride[0] != c.stride[1] and max(d for d, s in zip(c.dil, c.stride) if s == 1) > 1
               for c in dc if 1 in c.stride)                                                           # mixed stride + dil
    assert _both([c for c, p in paths if p != "dw"], lambda c: c.group > 1 or c.dil != (1, 1))         # forced SGECONV
    assert _both(sub, _scatter_reads_past_hc)
    assert any(max(c.pad) > max(c.kh, c.kw) for c in dc)                                              # pad past the kernel
    assert _both([c for c, p in paths if p == "subpixel"], lambda c: c.batch * c.oc > PLANES_Y)
    assert _both(dws, lambda c: c.batch * c.oc > PLANES_Y)
    assert _both(dws, lambda c: c.kh * c.kw > 256)
    assert any(c.stride[0] > 1 and c.pad[0] % c.stride[0] for c in dws)                              # Y % stride tap starts
    assert have((c.ic // c.group for c in dc if c.group == 1 or c.group != c.ic), IC_EDGES)
    assert have((c.oc * c.stride[0] * c.stride[1] for c, p in paths if p != "dw" and c.group == 1), OCP_EDGES[1::3])
    assert have((c.batch for c in dc), (1, 2, 3)) and _both(dc, lambda c: c.bias) and _both(dc, lambda c: c.relu)
    assert have((cs.mode for cs in S if cs.family == "deconv"), MODES3)
    assert sum(cs.equiv for cs in S) >= 20
    assert {cs.p["reject"] for cs in S if cs.family == "deconv"} == {0, -1}
    # Interp
    ip = [cs for cs in S if cs.family == "interp"]
    assert _both(ip, lambda cs: interp_kernel(cs.p, cs.out_off) == "memcpy")
    eq_n = [cs for cs in ip if cs.p["mode"] == "nearest" and interp_geometry(cs.p)[:2] == (cs.p["h"], cs.p["w"])]
    assert _both(eq_n, lambda cs: interp_kernel(cs.p, cs.out_off) == "memcpy")     # equal size, unit and other scales
    v4 = [cs for cs in ip if interp_geometry(cs.p)[1] % 4 == 0 and interp_kernel(cs.p) == "vec"]
    assert _both(v4, lambda cs: cs.out_off == 0)                                      # OW % 4 == 0 on misaligned views
    assert have((interp_geometry(cs.p)[1] for cs in ip), (511, 512, 513))
    assert _both([cs for cs in ip if interp_kernel(cs.p, cs.out_off) != "memcpy"], lambda cs: interp_band(cs.p, cs.out_off) == 64)
    assert _both(ip, lambda cs: cs.p["n"] * cs.p["c"] > PLANES_Y)
    assert any(cs.p["h"] == 1 for cs in ip) and any(cs.p["w"] == 1 for cs in ip)
    assert _both(ip, lambda cs: cs.p["scale"] is None)
    assert have((cs.in_off for cs in ip), range(4)) and have((cs.out_off for cs in ip), range(4))
    # Crop
    cp = [cs for cs in S if cs.family == "crop"]
    assert have((cs.p["ow"] for cs in cp), (511, 512, 513))
    assert _both([cs for cs in cp if cs.p["ow"] > 500], lambda cs: crop_kernel(cs.p, cs.in_off, cs.out_off) == "vec")
    geom_vec = [cs for cs in cp if crop_kernel(cs.p) == "vec"]
    assert _both(geom_vec, lambda cs: crop_kernel(cs.p, cs.in_off, cs.out_off) == "vec")             # misaligned views
    assert any(cs.p["woff"] % 4 for cs in cp) and any(cs.p["w"] % 4 and cs.p["woff"] % 4 == 0 for cs in cp)
    # Permute and Softmax
    pm = [cs.p for cs in S if cs.family == "permute"]
    assert have((p["order"] for p in pm), range(6))
    assert _both([p for p in pm if p["order"] == 3], lambda p: p["n"] > PLANES_Y)
    assert have((p["c"] for p in pm), (31, 32, 33)) and have((p["h"] * p["w"] for p in pm), (31, 32, 33))
    assert any(p["c"] % 32 and p["c"] > 32 for p in pm if p["order"] == 3)     # a partial tile of the transpose
    sm = [cs.p for cs in S if cs.family == "softmax"]
    assert have((p["len"] for p in sm if p["inner"] == 1), (1, 31, 32, 33)) and any(p["len"] >= 1000 for p in sm)
    assert any(p["inner"] > 1 and p["len"] == 1 for p in sm)
    # DetectionOutput
    det = [cs for cs in S if cs.family == "detect"]
    data = {cs.idx: det_data(cs) for cs in det}
    assert have((cs.p["P"] for cs in det if "P" in cs.p), (511, 512, 513, 1024, 1025))
    sides = set()
    for cs in det:
        if cs.p["target"] == "select":
            loc, conf, pri, C, thr, nms, top, keep = data[cs.idx]
            sides |= {int(v) - top for v in class_valid(conf, cs.p["P"], C, thr).reshape(-1)}
    assert {-1, 0, 1} <= sides                                                       # k - 1, k, k + 1 valid candidates
    assert any(cs.p["target"] == "select" and cs.p["quantized"] and cs.p["valid"] > 512 for cs in det)    # tie runs past 512
    tops = {data[cs.idx][6] for cs in det}
    assert {1, 2, 1024} <= tops and any(t & (t - 1) for t in tops) and any(((t + 1) & t) == 0 for t in tops if t > 2)
    keep_sides = set()
    for cs in det:
        if cs.p["target"] == "merge":
            loc, conf, pri, C, thr, nms, top, keep = data[cs.idx]
            keep_sides |= {int(np.sign(keep - k)) for k in merge_kept(conf, cs.p["P"], C, thr, top)}
    assert {-1, 0, 1} <= keep_sides                                                  # keep_top_k below, at and above
    assert any(cs.p["target"] == "iou_eq" for cs in det)
    neg = [data[cs.idx] for cs in det if cs.p["target"] == "negative"]
    assert any(np.any(np.signbit(d[1]) & (d[1] == 0)) and np.any(~np.signbit(d[1]) & (d[1] == 0)) and d[4] < 0 for d in neg)
    assert _both(det, lambda cs: cs.p["n"] > 1)
    assert sum(cs.p["target"] == "large" for cs in det) >= 2


# ---- the checkers bite (CPU) -----------------------------------------------------------------------------------------
def _first(pred, n=4, family=None):
    out = [cs for cs in (gen_case(i) for i in range(N_CASES)) if (family is None or cs.family == family) and pred(cs)]
    assert len(out) >= n, len(out)
    return out[:n]


def _small(cs):
    c = cs.deconv
    return c is not None and not cs.p["reject"] and c.batch * c.oc <= 200


def _deconv_bits(c: Deconv):
    x, w, b = c.data()
    ref = deconv_ref(x, w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, c.relu)
    s = deconv_ref(x, w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, absolute=True)
    K = c.ic // c.group * -(-c.kh // c.stride[0]) * -(-c.kw // c.stride[1])
    coef = eps_for("sgeconv", TF32) + K * U            # the loosest bound of the shape
    assert excess(ref, ref, s, coef)[0] == 0.0
    return x, w, b, ref, s, coef


PHASE_SHAPES = _first(lambda cs: _small(cs) and plan_ref(*cs.deconv.geometry)[0] == "subpixel" and
                      cs.deconv.stride[0] == cs.deconv.stride[1] > 1 and min(cs.deconv.kh, cs.deconv.kw) > 1 and
                      cs.deconv.oc <= 64, family="deconv")


@pytest.mark.parametrize("cs", PHASE_SHAPES, ids=[cs.name for cs in PHASE_SHAPES])
def test_checker_rejects_swapped_phases(cs):
    c = cs.deconv
    x, w, b, ref, s, coef = _deconv_bits(c)
    path, e = plan_ref(*c.geometry)
    wp = torch.from_numpy(equivalent_filter(w.numpy(), c.stride, c.group, path)).double()
    xp = F.pad(x.double(), (e["pad_left"], e["pad_right"], e["pad_top"], e["pad_bottom"]))
    P = F.conv2d(xp, wp, None, dilation=e["dil"], groups=c.group)
    n, _, hc, wc = P.shape
    Pswap = P.view(n, c.group, c.stride[0], c.stride[1], -1, hc, wc).transpose(2, 3).reshape(P.shape)   # ry <-> rx
    bad = scatter(Pswap, c.oc, c.group, c.stride, c.pad, tuple(ref.shape[2:]))
    if b is not None:
        bad = bad + b.double().view(1, -1, 1, 1)
    if c.relu:
        bad = bad.clamp_min(0)
    assert excess(bad, ref, s, coef)[0] > 1.0


BIAS_SHAPES = _first(lambda cs: _small(cs) and cs.deconv.bias and _scatter_reads_past_hc(cs.deconv), family="deconv")


@pytest.mark.parametrize("cs", BIAS_SHAPES, ids=[cs.name for cs in BIAS_SHAPES])
def test_checker_rejects_output_pad_region_without_bias(cs):
    c = dataclasses.replace(cs.deconv, relu=False)
    x, w, b, ref, s, coef = _deconv_bits(c)
    _, e = plan_ref(*c.geometry)
    Y = torch.arange(ref.shape[2]) + c.pad[0]
    X = torch.arange(ref.shape[3]) + c.pad[2]
    region = (Y // c.stride[0] >= e["output_h"]).view(-1, 1) | (X // c.stride[1] >= e["output_w"]).view(1, -1)
    bad = torch.where(region, ref - b.double().view(1, -1, 1, 1), ref)
    assert excess(bad, ref, s, coef)[0] > 1.0


DW_SHAPES = _first(lambda cs: _small(cs) and plan_ref(*cs.deconv.geometry)[0] == "dw" and cs.deconv.h >= 2 and
                   cs.deconv.stride[0] > 1, family="deconv")


@pytest.mark.parametrize("cs", DW_SHAPES, ids=[cs.name for cs in DW_SHAPES])
def test_checker_rejects_depthwise_tap_off_by_one_stride(cs):
    """The gather reading input row iy + 1 for tap ky (a tap start one stride off)."""
    c = cs.deconv
    x, w, b, ref, s, coef = _deconv_bits(c)
    shifted = F.pad(x[:, :, 1:], (0, 0, 0, 1))
    bad = deconv_ref(shifted, w, b, c.stride, c.pad, c.output_pad, c.dil, c.group, c.relu)
    assert excess(bad, ref, s, coef)[0] > 1.0


def _bilinear_matrix(n_out, n_in, align, swap_from=None):
    """float64 interpolation matrix of one axis (torch's coordinates); weights of the two neighbours swapped from
    output index `swap_from` on."""
    m = torch.zeros((n_out, n_in), dtype=torch.float64)
    for d in range(n_out):
        f = d * (n_in - 1) / (n_out - 1) if align and n_out > 1 else (0.0 if align else max((d + 0.5) * n_in / n_out - 0.5, 0.0))
        i0 = min(int(math.floor(f)), n_in - 1)
        i1, a = min(i0 + 1, n_in - 1), f - i0
        if swap_from is not None and d >= swap_from:
            a = 1 - a
        m[d, i0] += 1 - a
        m[d, i1] += a
    return m


SEAM_SHAPES = _first(lambda cs: cs.p["mode"] != "nearest" and interp_geometry(cs.p)[1] >= 1023 and cs.p["w"] > 1,
                     n=3, family="interp")


@pytest.mark.parametrize("cs", SEAM_SHAPES, ids=[cs.name for cs in SEAM_SHAPES])
def test_checker_rejects_bilinear_weights_swapped_at_the_512_seam(cs):
    p = cs.p
    oh, ow, _, _ = interp_geometry(p)
    align = p["mode"] == "bilinear-align"
    x = _data(cs, (p["n"], p["c"], p["h"], p["w"]))
    ry = _bilinear_matrix(oh, p["h"], align)
    good = ry @ x.double() @ _bilinear_matrix(ow, p["w"], align).T
    assert bilinear_check(good, x, int(align))[0] <= 1.0
    bad = ry @ x.double() @ _bilinear_matrix(ow, p["w"], align, swap_from=512).T
    assert bilinear_check(bad, x, int(align))[0] > 1.0


CROP_SHAPES = _first(lambda cs: cs.p["ow"] > 512 and cs.p["woff"] + cs.p["ow"] < cs.p["w"], n=3, family="crop")


@pytest.mark.parametrize("cs", CROP_SHAPES, ids=[cs.name for cs in CROP_SHAPES])
def test_checker_rejects_crop_off_by_one_column_past_512(cs):
    p = cs.p
    x = _data(cs, (p["n"], p["c"], p["h"], p["w"]))
    y0, x0 = p["hoff"], p["woff"]
    want = x[:, p["coff"]:p["coff"] + p["oc"], y0:y0 + p["oh"], x0:x0 + p["ow"]]
    bad = want.clone()
    bad[..., 512:] = x[:, p["coff"]:p["coff"] + p["oc"], y0:y0 + p["oh"], x0 + 513:x0 + p["ow"] + 1]
    assert not torch.equal(bad, want)


def _det_cpu(cs):
    """(boxes, conf, C, thr, nms, top, keep) with the float64 decode rounded to fp32 in place of the kernel's boxes."""
    loc, conf, priors, C, thr, nms, top, keep = det_data(cs)
    boxes = _decode_ref(loc, priors)[0].astype(np.float32)
    return boxes, conf, C, np.float32(thr), np.float32(nms), top, keep


DET_SMALL = lambda cs: cs.p["target"] != "large" and cs.p.get("P", 0) <= 700  # noqa: E731
TIE_SHAPES = _first(lambda cs: DET_SMALL(cs) and cs.p["target"] in ("ties", "negative"), n=3, family="detect")


@pytest.mark.parametrize("cs", TIE_SHAPES, ids=[cs.name for cs in TIE_SHAPES])
def test_checker_rejects_ties_broken_by_the_higher_prior(cs):
    boxes, conf, C, thr, nms, top, keep = _det_cpu(cs)
    good, _ = detection_ref(boxes, conf, C, thr, nms, top, keep)
    n, P = boxes.shape[:2]
    rev = conf.reshape(n, P, C)[:, ::-1].reshape(n, -1)      # prior order reversed: equal scores take the higher prior
    bad, _ = detection_ref(np.ascontiguousarray(boxes[:, ::-1]), np.ascontiguousarray(rev), C, thr, nms, top, keep)
    assert not _bits_equal(bad, good)


IOU_SHAPES = _first(lambda cs: cs.p["target"] == "iou_eq" and cs.p["pairs"] > 1, n=3, family="detect")


@pytest.mark.parametrize("cs", IOU_SHAPES, ids=[cs.name for cs in IOU_SHAPES])
def test_checker_rejects_nms_with_greater_or_equal(cs):
    boxes, conf, C, thr, nms, top, keep = _det_cpu(cs)
    good, _ = detection_ref(boxes, conf, C, thr, nms, top, keep)
    # IoU > next float below the threshold == IoU >= threshold for fp32 IoUs
    bad, _ = detection_ref(boxes, conf, C, thr, np.nextafter(nms, np.float32(-1)), top, keep)
    assert not _bits_equal(bad, good)


KEEP_SHAPES = _first(lambda cs: DET_SMALL(cs) and cs.p["target"] == "merge" and cs.p["C"] >= 4 and
                     cs.p["keep_side"] < 0, n=3, family="detect")


@pytest.mark.parametrize("cs", KEEP_SHAPES, ids=[cs.name for cs in KEEP_SHAPES])
def test_checker_rejects_keep_top_k_per_class(cs):
    boxes, conf, C, thr, nms, top, keep = _det_cpu(cs)
    good, _ = detection_ref(boxes, conf, C, thr, nms, top, keep)
    n, P = boxes.shape[:2]
    bad = np.zeros_like(good)
    bad[..., 0] = -1
    rows = [[] for _ in range(n)]
    for c in range(1, C):       # each class cut at keep_top_k, the classes one after another
        only = np.full((n, P, C), -np.inf, np.float32)
        only[..., c] = conf.reshape(n, P, C)[..., c]
        out, _ = detection_ref(boxes, only.reshape(n, -1), C, thr, nms, top, keep)
        for i in range(n):
            rows[i] += [r for r in out[i] if r[0] >= 0]
    for i in range(n):
        for j, r in enumerate(rows[i][:keep]):
            bad[i, j] = r
    assert not _bits_equal(bad, good)
