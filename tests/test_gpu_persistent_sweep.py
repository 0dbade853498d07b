"""Seeded random shapes across the persistent tensor-core kernels, with a set number of CTAs, against float64.

Five kernels run on persistent CTAs that walk the tile list with a static stride: the stem kernel, the halo, pre-split
and wide implicit-GEMM kernels (conv_igemm.cu, launch_igemm_kernel(..., persistent=true)) and tensor_gemm_kernel
(Winograd, im2col, InnerProduct, the raw TensorGEMM).  Most of their hardest code runs only when a CTA gets a second
tile: ring slots and mbarrier phases carried over from one tile to the next (the TensorGEMM's running k-block count,
the halo family's 4-deep filter and 2-deep box rings), the next tile's loads or gather issued during the current tile's
epilogue, the stem kernel's staging-buffer swap.  The device gives a layer min(tiles, SMs x occupancy) CTAs, so on an
H100 a CTA gets a second tile only past ~132-264 tiles, and the other sweeps' shapes are smaller than that.

The switch persistent_ctas = n caps the grid at n CTAs.  Every H100 has more than 64 SMs (114 on the PCIe card), so
with n <= 114 the grid is min(n, tiles) whatever the card: the tiles each CTA runs and the uneven tail follow from the
shape alone.  Each case runs at cap 0 (the device's grid) and at caps 1, 2, 3, ceil(tiles / 2), one cap that does not
divide the tile count and tiles - 1.  The checks:

  - the output sits in a NaN-filled buffer, and the floats around it stay NaN;
  - every capped run is bit-identical to the cap-0 run (int32 views: -0.0 and NaN payloads count).  Each tile writes
    only its own outputs with a fixed k order, and the split-K partials have fixed slots, so which CTA runs a tile, and
    after which other tile, must not change a bit;
  - the cap-0 run is inside the float64 per-element bound of test_gpu_error_bounds.py / test_gpu_dispatch_sweep.py
    (convolutions: conv_coef / conv_expect, Winograd through wino_model; InnerProduct: ip_rule; TensorGEMM: eps_for).

Every run is labelled with its kernel (the stem query, then the wide / pre-split / halo tile queries, in launch_conv's
order; the TensorGEMM for Winograd, im2col and InnerProduct), its tile count (stem: N * ceil(OH * OW / 128); halo
family: N * ceil(OH / R) * ceil(OW / C) * ceil(OC / BN); TensorGEMM: ceil(M / 128) * ceil(N / BN) * G * splits) and its
k-blocks per tile.  The CPU tests check that the list hits every (kernel, tiles per CTA in {1, 2, >= 3}, uneven tail,
k-blocks per tile mod 4) cell and both sides of every stem predicate, and that the checker rejects simulated cross-tile
defects on the sweep's own shapes.  A net-level test runs small zoo nets, fused and graph-captured, at caps 1 and 3
against cap 0.  A failing case prints a ready-to-paste literal for the matching hand-written list.

FCUDA_SWEEP_SCALE (a float, default 1) scales the case count.  Run with -s to print the runs per cell.
"""
from __future__ import annotations

import ctypes
import dataclasses
import math
import os
import random
import zlib
from collections import Counter

import numpy as np
import pytest
import torch

from test_gpu_dispatch_sweep import Case as SweepCase
from test_gpu_dispatch_sweep import (_guard_ok, _view, check_conv, conv_coef, conv_expect, conv_param, forward_conv_case,
                                     igemm_kernel, literal, wino_chunked, wino_tile)
from test_gpu_error_bounds import (FP32_SPLIT, IM2COL, MODE_NAME, SGECONV, TF32, TF32X3, U, WINOGRADF23, WINOGRADF63,
                                   Conv, _fc_split, eps_for, excess, ip_rule, make_data)

gpu = pytest.mark.gpu

N_CASES = 420           # about 2200 kernel runs: 45 s for the file on an H100 SXM (80 GB, 700 W)
SCALE = float(os.environ.get("FCUDA_SWEEP_SCALE", "1"))
CASES_RUN = max(1, int(round(N_CASES * SCALE)))
MIN_SLOTS = 114         # SMs of the smallest H100 (PCIe), at one CTA per SM: a grid up to this is min(cap, tiles)
KERNELS = ("stem", "halo", "presplit", "wide", "gemm")
HALO_FAMILY = ("halo", "presplit", "wide")
MODES3 = (FP32_SPLIT, TF32X3, TF32)


# ---- the generator ----------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    idx: int
    family: str
    mode: int
    conv: Conv | None = None
    algo: int = SGECONV
    ip: tuple | None = None      # (in_size, out_size, batch, relu)
    gemm: tuple | None = None    # (g, m, n, k)
    out_off: int = 0             # float offset of the output view (stem: the scalar stores)

    @property
    def name(self):
        return f"{self.idx:04d}-{self.family}"


# (IC per group, KH, KW) of the stem kernel by k-blocks per tile (K = KH * KW * IC <= 256, IC % 32 != 0, IC > 1)
STEM_SHAPES = {1: [(3, 3, 3), (2, 3, 4), (2, 3, 3)], 2: [(4, 3, 3), (7, 3, 3), (3, 3, 5)],
               3: [(3, 5, 5), (10, 3, 3), (5, 3, 5)], 4: [(3, 7, 5), (12, 3, 3), (2, 7, 7)],
               5: [(3, 7, 7), (16, 3, 3), (5, 5, 6)], 6: [(20, 3, 3), (4, 7, 6), (7, 5, 5)],
               7: [(24, 3, 3), (5, 7, 6), (4, 7, 7)], 8: [(28, 3, 3), (16, 4, 4), (5, 7, 7)]}
# just past the stem kernel (the gathering kernel takes them): K = 257, K = 261
STEM_OFF_K = [(257, 1, 1), (29, 3, 3)]
HW = (7, 9, 12, 15, 16, 17, 20, 23, 24, 28, 32, 40, 48)


def _pads(r, kh, kw):
    if r.random() < 0.6:
        return (kw // 2, kh // 2, kw // 2, kh // 2)
    return tuple(r.randint(0, 2) for _ in range(4))


def _epilogue(c: Conv, k: int, r) -> Conv:
    e = k % 3
    c.relu = e == 1
    if e == 2:
        c.clip = (-0.125, 0.25) if r.random() < 0.5 else (0.0, 0.5)
    return c


def _gen_stem(r, k):
    """Both sides of K = 256 / 257 and OC = 128 / 129, nbuf 1 and 2, vector and scalar stores, partial last tiles,
    batches whose CTAs span images, grouped layers writing channel slices."""
    off = k % 8 == 7
    kb = 1 + (k * 3 + k // 8) % 8
    icg, kh, kw = r.choice(STEM_OFF_K if off and k % 16 == 7 else STEM_SHAPES[kb])
    if kb >= 6 and r.random() < 0.6:
        ocg = r.choice([65, 96, 128])                       # N tile 128 with >= 6 k-blocks: one staging buffer
    else:
        ocg = r.choice([8, 16, 31, 32, 33, 48, 64, 65, 100, 128])
    if off and k % 16 == 15:
        ocg = 129                                           # two N tiles
    group = 2 if r.random() < 0.2 and ocg <= 64 else 1
    s = 2 if r.random() < 0.3 else 1
    h, w = max(r.choice(HW), kh), max(r.choice(HW), kw)
    c = Conv("", ocg * group, icg * group, h, w, kh, kw, sh=s, pad=_pads(r, kh, kw), group=group,
             bias=r.random() < 0.8, batch=r.choice([1, 2, 2, 3, 4, 6]))
    return _epilogue(c, k, r), (r.randint(1, 3) if r.random() < 0.3 else 0)


# halo family: (KH, KW) and IC per group; k-blocks per tile = KH * KW * IC / 32
TAPS_SMALL = [(1, 2), (2, 1), (1, 3), (3, 1), (2, 2), (1, 4)]
TAPS_WIDE = [(1, 5), (5, 1), (2, 3), (3, 2), (1, 7), (7, 1), (2, 4), (4, 2), (3, 3)]
TAPS_BIG = [(7, 7), (7, 9), (9, 7)]


def _pick_kb(r, shapes, ics, res):
    """A (KH, KW, IC) from the products of `shapes` and `ics` whose k-block count is `res` mod 4; the fewest k-blocks
    with probability 0.4."""
    kb = lambda o: o[0] * o[1] * o[2] // 32  # noqa: E731
    opts = [(kh, kw, ic) for kh, kw in shapes for ic in ics if (kh * kw * ic // 32) % 4 == res]
    if r.random() < 0.4:
        opts = [o for o in opts if kb(o) == min(map(kb, opts))]
    return r.choice(opts)


def _halo_conv(r, kh, kw, icg, oc, hs, ws, batch):
    h, w = max(r.choice(hs), kh), r.choice(ws)
    return Conv("", oc, icg, h, max(w, (kw + 3) // 4 * 4), kh, kw, pad=_pads(r, kh, kw), bias=r.random() < 0.8,
                batch=batch)


def _gen_halo(r, k):
    """TF32X3 and TF32 on 2..9 taps; every fourth case fp32split at 49 or 63 taps with an N tile of 128 (the pre-split
    box does not fit shared memory)."""
    if k % 4 == 3:
        kh, kw, icg = _pick_kb(r, TAPS_BIG, [32, 64, 96, 128], (k // 4) % 4)
        c = _halo_conv(r, kh, kw, icg, r.choice([65, 96, 128]), (9, 12, 16, 24), (12, 16, 20), r.choice([1, 2, 3]))
        return _epilogue(c, k, r), FP32_SPLIT
    kh, kw, icg = _pick_kb(r, TAPS_SMALL + TAPS_WIDE, [32, 64, 96], (k + k // 4) % 4)
    c = _halo_conv(r, kh, kw, icg, r.choice([16, 32, 33, 64, 65, 96, 128, 129]), (5, 8, 9, 16, 17, 24, 33),
                   (8, 12, 16, 20, 24, 32, 40), r.choice([1, 2, 3, 4, 6]))
    return _epilogue(c, k, r), (TF32X3, TF32)[(k // 4) % 2]


def _gen_presplit(r, k):
    """fp32split: 2..4 taps, or more taps with an N tile of 32 (the wide kernel takes N tiles of 64 and 128 only)."""
    if k % 3 == 2:
        kh, kw, icg = _pick_kb(r, TAPS_WIDE, [32, 64], k % 4)
        oc = r.choice([8, 16, 31, 32])
    else:
        kh, kw, icg = _pick_kb(r, TAPS_SMALL, [32, 64, 96], k % 4)
        oc = r.choice([16, 32, 33, 64, 65, 128, 129])
    c = _halo_conv(r, kh, kw, icg, oc, (5, 8, 9, 16, 17, 24, 33), (8, 12, 16, 20, 24, 32, 40), r.choice([1, 2, 3, 4, 6]))
    return _epilogue(c, k, r), FP32_SPLIT


def _gen_wide(r, k):
    """fp32split, 5..9 taps, N tiles of 64 and 128, planes near the 28-row wide tile."""
    kh, kw, icg = _pick_kb(r, TAPS_WIDE, [32, 64], k % 4)
    c = _halo_conv(r, kh, kw, icg, r.choice([33, 48, 64, 65, 96, 128, 129]), (27, 28, 28, 56), (16, 16, 24, 32),
                   r.choice([1, 2, 3, 4, 5]))
    return _epilogue(c, k, r), FP32_SPLIT


WINO_IC = {1: [4, 8, 28], 2: [36, 64], 3: [68, 96], 0: [100, 128]}


def _gen_wino(r, k):
    """3x3 / stride 1 on both Winograd tiles; k-blocks per tile = ceil(IC / 32)."""
    algo = (WINOGRADF63, WINOGRADF23)[k % 2]
    ic = r.choice(WINO_IC[(k // 2) % 4] + ([160] if (k // 2) % 4 == 1 else []))
    oc = r.choice([8, 32, 33, 64, 65, 128])
    hw = (12, 16, 18, 24, 30, 40) if algo == WINOGRADF63 else (8, 12, 16, 17)
    c = Conv("", oc, ic, r.choice(hw), r.choice(hw), 3, pad=r.choice([1, 1, 0]), bias=r.random() < 0.8,
             batch=r.choice([1, 2, 3]))
    return _epilogue(c, k, r), algo


def _gen_im2col(r, k):
    ic = r.choice([3, 4, 8, 13, 16, 24, 32, 40])
    kh = r.choice([1, 3, 3, 5])
    s = r.choice([1, 1, 2])
    c = Conv("", r.choice([8, 16, 32, 33, 64, 65, 128]), ic, r.choice([8, 12, 16, 17, 24]), r.choice([8, 12, 16, 17, 24]),
             kh, sh=s, pad=kh // 2, bias=r.random() < 0.8, batch=r.choice([1, 2, 3]))
    return _epilogue(c, k, r)


def _gen_ip(r, k):
    """Split-K InnerProduct: 16..40 k-blocks in kb // 8 splits (the SM-count term of fc_split does not bind at these
    sizes), so the last split of a row owns fewer k-blocks than the others."""
    kb = r.choice([16, 17, 18, 19, 20, 21, 24, 25, 26, 27, 33, 35, 40])
    return (32 * kb - r.choice([0, 0, 4, 28]), r.choice([40, 100, 128, 129, 200]), r.choice([1, 7, 32, 33, 64, 65, 100]),
            r.random() < 0.5)


def _gen_gemm(r, k):
    kb = 1 + k % 9
    m, n = r.choice([60, 127, 128, 129, 200]), r.choice([16, 32, 33, 64, 65, 100, 128, 129])
    per_g = -(-m // 128) * -(-n // gemm_bn(n))
    g = r.choice([g for g in (1, 2, 3, 5, 8, 16, 33) if g * per_g <= 200])
    return g, m, n, max(4, 32 * kb - r.choice([0, 4, 20]))


SLOTS = ["stem", "halo", "wino", "presplit", "wide", "stem", "wide", "im2col", "halo", "ip", "stem", "gemm", "presplit",
         "wide"]


def gen_case(i: int) -> Case:
    r = random.Random(zlib.crc32(f"persistent-sweep-{i}".encode()))
    fam = SLOTS[i % len(SLOTS)]
    k = i // len(SLOTS) * SLOTS.count(fam) + SLOTS[:i % len(SLOTS)].count(fam)
    if fam == "stem":
        c, off = _gen_stem(r, k)
        case = Case(i, fam, FP32_SPLIT, conv=c, out_off=off)
    elif fam == "halo":
        c, mode = _gen_halo(r, k)
        case = Case(i, fam, mode, conv=c)
    elif fam in ("presplit", "wide"):
        c, mode = (_gen_presplit if fam == "presplit" else _gen_wide)(r, k)
        case = Case(i, fam, mode, conv=c)
    elif fam == "wino":
        c, algo = _gen_wino(r, k)
        case = Case(i, fam, MODES3[(k // 8) % 3], conv=c, algo=algo)
    elif fam == "im2col":
        case = Case(i, fam, MODES3[k % 3], conv=_gen_im2col(r, k), algo=IM2COL)
    elif fam == "ip":
        case = Case(i, fam, MODES3[k % 3], ip=_gen_ip(r, k))
    else:
        case = Case(i, fam, MODES3[k % 3], gemm=_gen_gemm(r, k))
    if case.conv is not None:
        case.conv.name = f"psweep{i}"
    return case


# ---- labels: kernel, tiles, k-blocks per tile --------------------------------------------------------------------------
def _lib():
    from feathercnn_b200._lib import fcuda
    return fcuda()


def gemm_bn(n: int) -> int:
    """N tile of launch_tile (TensorGEMM) and of igemm_bn_for (implicit GEMM)."""
    return 32 if n <= 32 else 64 if n <= 64 else 128


def _cdiv(a, b):
    return -(-a // b)


def stem_nbuf(bn: int, kb: int) -> int:
    """Staging buffers of the stem kernel (conv_igemm.cu stem_smem_bytes, kStemPitch 132)."""
    two = kb * 2 * bn * 64 + 2 * bn * 132 * 4 + kb * 32 * 8 + 1024
    return 2 if two <= 227 * 1024 else 1


def halo_tile(c: Conv, mode: int, kernel: str) -> tuple[int, int]:
    """(R, C) of the output patch from the tile query of `kernel` in `mode`."""
    lib, g = _lib(), (ctypes.c_int * 4)()
    old = lib.fcuda_get_precision()
    lib.fcuda_set_precision(mode)
    try:
        assert getattr(lib, f"fcuda_igemm_{kernel}_tile")(ctypes.byref(conv_param(c)), g) == 1
    finally:
        lib.fcuda_set_precision(old)
    return g[0], g[1]


@dataclasses.dataclass(frozen=True)
class Launch:
    kernel: str     # stem / halo / presplit / wide / gemm, or gather (not persistent)
    tiles: int      # tiles of one launch (one launch per group)
    kb: int         # k-blocks per tile (split-K: those of every split but the last)


_LAUNCH: dict = {}


def launch_of(case: Case) -> Launch:
    if case.idx not in _LAUNCH:
        _LAUNCH[case.idx] = _launch_of(case)
    return _LAUNCH[case.idx]


def _launch_of(case: Case) -> Launch:
    if case.gemm is not None:
        g, m, n, k = case.gemm
        return Launch("gemm", g * _cdiv(m, 128) * _cdiv(n, gemm_bn(n)), _cdiv(k, 32))
    if case.ip is not None:
        in_size, out_size, batch, _ = case.ip
        lib = _lib()
        old = lib.fcuda_get_precision()
        lib.fcuda_set_precision(case.mode)      # (the scratch size _fc_split reads depends on the mode)
        try:
            split = _fc_split(in_size, out_size, batch, case.mode)
        finally:
            lib.fcuda_set_precision(old)
        return Launch("gemm", _cdiv(out_size, 128) * _cdiv(batch, gemm_bn(batch)) * split,
                      _cdiv(_cdiv(in_size, 32), split))
    c = case.conv
    oh, ow = c.out_hw
    if case.algo in (WINOGRADF63, WINOGRADF23):
        assert not wino_chunked(c, case.algo, case.mode), case.name     # one TensorGEMM over every tile row
        t = 8 if case.algo == WINOGRADF63 else 4
        m = c.batch * _cdiv(oh, t - 2) * _cdiv(ow, t - 2)
        return Launch("gemm", t * t * _cdiv(m, 128) * _cdiv(c.oc, gemm_bn(c.oc)), _cdiv(c.ic, 32))
    if case.algo == IM2COL:
        kp = (c.ic * c.kh * c.kw + 3) // 4 * 4
        return Launch("gemm", _cdiv(c.batch * oh * ow, 128) * _cdiv(c.oc, gemm_bn(c.oc)), _cdiv(kp, 32))
    kernel = igemm_kernel(c, case.mode)
    icg, ocg = c.ic // c.group, c.oc // c.group
    kb = _cdiv(icg * c.kh * c.kw, 32)
    if kernel == "stem":
        return Launch(kernel, c.batch * _cdiv(oh * ow, 128), kb)
    if kernel in HALO_FAMILY:
        R, C = halo_tile(c, case.mode, kernel)
        return Launch(kernel, c.batch * _cdiv(oh, R) * _cdiv(ow, C) * _cdiv(ocg, gemm_bn(ocg)), kb)
    return Launch(kernel, 0, kb)


def caps_for(case: Case) -> list[int]:
    """The caps a case runs at besides 0: 1, 2, 3, ceil(tiles / 2), one cap that does not divide the tile count and
    tiles - 1 (each below the tile count); cap 1 alone for a kernel that is not persistent (the switch leaves it be)."""
    T = launch_of(case).tiles
    if T == 0:
        return [1]
    r = random.Random(zlib.crc32(f"persistent-caps-{case.idx}".encode()))
    uneven = [n for n in range(4, min(T, MIN_SLOTS + 1)) if T % n]
    caps = {1, 2, 3, _cdiv(T, 2), T - 1} | ({r.choice(uneven)} if uneven else set())
    return sorted(n for n in caps if 1 <= n < T)


def grid_of(tiles: int, cap: int) -> int | None:
    """CTAs of a launch at `cap` when the same on every H100, else None."""
    g = min(tiles, cap) if cap else tiles
    return g if g <= MIN_SLOTS else None


def cell_of(case: Case, cap: int):
    """(kernel, tiles per CTA class 1 / 2 / 3 (= 3 or more), uneven tail, k-blocks per tile mod 4) of one run."""
    la = launch_of(case)
    g = grid_of(la.tiles, cap) if la.tiles else None
    if g is None:
        return None
    return la.kernel, min(3, _cdiv(la.tiles, g)), la.tiles % g != 0, la.kb % 4


def _literal(case: Case) -> str:
    if case.conv is not None:
        from feathercnn_b200 import booster
        return (f"{literal(case.conv)}  # {case.family}, {MODE_NAME[case.mode]}, {booster.ALGO_NAMES[case.algo]}, "
                f"output offset {case.out_off}")
    if case.ip is not None:
        return f"({', '.join(map(str, case.ip))})  # InnerProduct (in, out, batch, relu), {MODE_NAME[case.mode]}"
    return f"({', '.join(map(str, case.gemm))})  # TensorGEMM (g, m, n, k), x3={case.mode != TF32}"


_CASES = None


def cases() -> list[Case]:
    global _CASES
    if _CASES is None:
        _CASES = [gen_case(i) for i in range(CASES_RUN)]
    return _CASES


# ---- running a case ----------------------------------------------------------------------------------------------------
@pytest.fixture
def ctas(cuda):
    """Sets persistent_ctas; restores it and the precision mode afterwards."""
    from feathercnn_b200 import booster
    lib = _lib()
    saved = lib.fcuda_get_tuning(b"persistent_ctas"), booster.get_precision()

    def setter(v):
        assert lib.fcuda_set_tuning(b"persistent_ctas", v) == 0
    yield setter
    lib.fcuda_set_tuning(b"persistent_ctas", saved[0])
    booster.set_precision(saved[1])


def _gen(case: Case):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(case.name.encode()))


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ip_data(case: Case):
    in_size, out_size, batch, _ = case.ip
    g = _gen(case)
    x = torch.rand((batch, in_size), generator=g, device="cuda") * 2 - 1
    w = torch.randn((out_size, in_size), generator=g, device="cuda") * math.sqrt(2.0 / in_size)
    w = w * torch.pow(10.0, -2 * torch.rand((out_size, 1), generator=g, device="cuda"))
    return x, w, torch.rand(out_size, generator=g, device="cuda") - 0.5


def gemm_data(case: Case):
    g_, m, n, k = case.gemm
    g = _gen(case)
    a = torch.rand((g_, m, k), generator=g, device="cuda") * 2 - 1
    b = torch.randn((g_, n, k), generator=g, device="cuda") * torch.pow(10.0, -2 * torch.rand((g_, n, 1), generator=g,
                                                                                             device="cuda"))
    return a, b


def forward(case: Case):
    """One run of the case at the current cap: (output, guard ok, the float64 check of the output: share of the bound
    used)."""
    from feathercnn_b200 import booster
    booster.set_precision(case.mode)
    lib = _lib()
    if case.conv is not None:
        sc = SweepCase(case.idx, case.family, case.mode, conv=case.conv, out_off=case.out_off)
        x, w, b, r, got, guard = forward_conv_case(sc, case.algo)

        def check():
            coef = conv_coef(case.conv, case.algo, case.mode, x, w, b)
            ref, bound, s = conv_expect(case.conv, x, w, b, r, coef, wino_tile(case.algo))
            return check_conv(got, ref, bound, s)[0] if torch.isfinite(got).all() else math.inf
        return got, guard, check
    if case.ip is not None:
        in_size, out_size, batch, relu = case.ip
        x, w, b = ip_data(case)
        s, kb = ctypes.c_size_t(), ctypes.c_size_t()
        assert lib.fcuda_inner_product_get_buffer_size(in_size, out_size, batch, ctypes.byref(s), ctypes.byref(kb)) == 0
        packed, scratch = torch.empty(max(kb.value, 1), device="cuda"), torch.empty(max(s.value, 1), device="cuda")
        assert lib.fcuda_inner_product_init(in_size, out_size, _ptr(packed), _ptr(w), _stream()) == 0
        out, obuf = _view(batch * out_size, 0)
        rc = lib.fcuda_inner_product_forward(in_size, out_size, _ptr(out), _ptr(x), _ptr(packed), _ptr(b), _ptr(scratch),
                                             int(relu), batch, _stream())
        torch.cuda.synchronize()
        assert rc == 0, rc
        got = out.view(batch, out_size)

        def check():
            ref = x.double() @ w.double().T + b.double()
            ref = ref.clamp_min(0) if relu else ref
            s = x.double().abs() @ w.double().abs().T + b.double().abs()
            return excess(got, ref, s, ip_rule(in_size, case.mode)[1])[0] if torch.isfinite(got).all() else math.inf
        return got, _guard_ok(obuf, 0, got.numel()), check
    g, m, n, k = case.gemm
    a, bm = gemm_data(case)
    out, obuf = _view(g * m * n, 0)
    if case.mode == TF32:
        rc = lib.fcuda_tensor_gemm(_ptr(out), _ptr(a), _ptr(bm), None, m, n, k, g, _stream())
    else:   # A is split inside the kernel; B carries its hi / lo planes
        bh, bl = torch.empty_like(bm), torch.empty_like(bm)
        assert lib.fcuda_split_tf32(_ptr(bh), _ptr(bl), _ptr(bm), bm.numel(), _stream()) == 0
        rc = lib.fcuda_tensor_gemm(_ptr(out), _ptr(a), _ptr(bh), _ptr(bl), m, n, k, g, _stream())
    torch.cuda.synchronize()
    assert rc == 0, rc
    got = out.view(g, m, n)

    def check():
        ref = torch.einsum("gmk,gnk->gmn", a.double(), bm.double())
        s = torch.einsum("gmk,gnk->gmn", a.double().abs(), bm.double().abs())
        mode = TF32 if case.mode == TF32 else TF32X3
        return excess(got, ref, s, eps_for("gemm", mode) + k * U)[0] if torch.isfinite(got).all() else math.inf
    return got, _guard_ok(obuf, 0, got.numel()), check


def differing(got, base) -> int:
    """Outputs whose bits differ (int32 views: -0.0 against 0.0 and NaN payloads count)."""
    return int((got.contiguous().view(torch.int32) != base.contiguous().view(torch.int32)).sum())


REPORT: Counter = Counter()


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    REPORT.pop(None, None)     # runs whose grid depends on the card, and the gathering kernel's
    if REPORT:
        print("\nruns per (kernel, tiles per CTA, uneven tail, k-blocks per tile mod 4):")
        for cell, n in sorted(REPORT.items()):
            print(f"  {cell[0]:9s} {cell[1]}{'+' if cell[1] == 3 else ' '} {'uneven' if cell[2] else 'even  '} "
                  f"kb%4={cell[3]}  {n:4d} runs")


def _ids():
    return [cs.name for cs in cases()]


@gpu
@pytest.mark.parametrize("i", range(CASES_RUN), ids=_ids())
def test_persistent_sweep(ctas, i):
    case = cases()[i]
    ctas(0)
    base, guard, check = forward(case)
    used = check()
    failures = []
    if not guard:
        failures.append("cap 0: the floats around the output were overwritten")
    if not used <= 1.0:
        failures.append(f"cap 0: bound used {used:.3g}")
    REPORT[cell_of(case, 0)] += 1
    del check
    for cap in caps_for(case):
        ctas(cap)
        got, guard, _ = forward(case)
        REPORT[cell_of(case, cap)] += 1
        if not guard:
            failures.append(f"cap {cap}: the floats around the output were overwritten")
        if (n := differing(got, base)):
            failures.append(f"cap {cap}: {n} of {got.numel()} outputs differ from cap 0")
        del got
    la = launch_of(case)
    assert not failures, (f"{_literal(case)}\n  {la.kernel}, {la.tiles} tiles, {la.kb} k-blocks per tile\n  " +
                          "\n  ".join(failures))


# ---- coverage of the generated list (CPU) ------------------------------------------------------------------------------
# Cells that cannot occur: one tile per CTA with an uneven tail (tiles % grid != 0 needs a CTA with two tiles).  Runs
# whose grid depends on the card (more than 114 CTAs) are not labelled.
EXPECTED_CELLS = [(k, cls, uneven, r) for k in KERNELS for cls in (1, 2, 3) for uneven in (False, True) for r in range(4)
                  if not (cls == 1 and uneven)]


def _cells() -> Counter:
    n = Counter()
    for cs in cases():
        for cap in [0] + caps_for(cs):
            cell = cell_of(cs, cap)
            if cell is not None:
                n[cell] += 1
    return n


def test_sweep_hits_every_cell():
    pytest.importorskip("feathercnn_b200._lib")
    cells = _cells()
    unexpected = sorted(set(cells) - set(EXPECTED_CELLS))
    assert not unexpected, f"cells the coverage table says cannot occur: {unexpected}"
    if SCALE < 1:
        pytest.skip("a scaled-down sweep need not cover every cell")
    thin = sorted((cell, cells.get(cell, 0)) for cell in EXPECTED_CELLS if cells.get(cell, 0) < 3)
    assert not thin, f"cells hit fewer than 3 times: {thin}"
    # every family reaches the kernel it aims at (the labels come from the library's own queries)
    aimed = {"stem": "stem", "halo": "halo", "presplit": "presplit", "wide": "wide"}
    for fam, kernel in aimed.items():
        got = Counter(launch_of(cs).kernel for cs in cases() if cs.family == fam)
        assert got[kernel] >= 0.5 * sum(got.values()), (fam, got)
    # k-blocks per tile: 1..5 where the kernel allows them (the halo family has >= 2 taps of 32 channels, wide >= 5 taps)
    kbs = {k: {launch_of(cs).kb for cs in cases() if launch_of(cs).kernel == k} for k in KERNELS}
    for k, want in (("stem", range(1, 9)), ("gemm", range(1, 6)), ("halo", range(2, 6)), ("presplit", range(2, 6)),
                    ("wide", range(5, 10))):
        assert set(want) <= kbs[k], (k, sorted(kbs[k]))
    # the split-K InnerProduct: tiles of one CTA with different k-block counts
    assert any(_cdiv(cs.ip[0], 32) % launch_of(cs).kb for cs in cases() if cs.ip is not None)


def _both(values, pred) -> bool:
    vs = list(values)
    return any(pred(v) for v in vs) and any(not pred(v) for v in vs)


def test_sweep_covers_both_sides_of_every_stem_predicate():
    pytest.importorskip("feathercnn_b200._lib")
    if SCALE < 1:
        pytest.skip("a scaled-down sweep need not cover every boundary")
    stem_fam = [cs for cs in cases() if cs.family == "stem"]
    label = {cs.idx: launch_of(cs).kernel for cs in stem_fam}
    K = lambda c: c.ic // c.group * c.kh * c.kw  # noqa: E731
    assert any(K(cs.conv) == 256 and label[cs.idx] == "stem" for cs in stem_fam)
    assert any(K(cs.conv) == 257 and label[cs.idx] == "gather" for cs in stem_fam)
    assert any(K(cs.conv) > 256 and cs.conv.oc // cs.conv.group <= 128 and label[cs.idx] == "gather" for cs in stem_fam)
    assert any(cs.conv.oc // cs.conv.group == 128 and label[cs.idx] == "stem" for cs in stem_fam)
    assert any(cs.conv.oc // cs.conv.group == 129 and label[cs.idx] == "gather" for cs in stem_fam)
    stem = [cs for cs in stem_fam if label[cs.idx] == "stem"]
    assert _both(stem, lambda cs: stem_nbuf(gemm_bn(cs.conv.oc // cs.conv.group), launch_of(cs).kb) == 1)
    oplane = lambda cs: cs.conv.out_hw[0] * cs.conv.out_hw[1]  # noqa: E731
    assert _both(stem, lambda cs: cs.out_off == 0 and oplane(cs) % 4 == 0)          # vector / scalar stores
    assert any(cs.out_off and oplane(cs) % 4 == 0 for cs in stem)                    # scalar for the alignment alone
    assert _both(stem, lambda cs: oplane(cs) % 128 != 0)                             # partial last tile per image
    assert _both(stem, lambda cs: cs.conv.group > 1)                                 # channel slices

    def spans(cs, cap):   # some CTA runs tiles of two images
        T, tpi = launch_of(cs).tiles, _cdiv(oplane(cs), 128)
        g = grid_of(T, cap)
        return g is not None and any(t // tpi != (t + g) // tpi for t in range(T - g))
    runs = [(cs, cap) for cs in stem for cap in caps_for(cs)]
    assert _both(runs, lambda rc: spans(*rc))


# ---- the checker bites (CPU) -------------------------------------------------------------------------------------------
def tile_layout(case: Case):
    """(tile, position inside the tile) of every output element of a group-1 stem / halo-family convolution or a raw
    TensorGEMM, as int64 tensors shaped like the output."""
    if case.gemm is not None:
        g_, m, n, _ = case.gemm
        bn = gemm_bn(n)
        G, M, N = torch.meshgrid(torch.arange(g_), torch.arange(m), torch.arange(n), indexing="ij")
        return (G * _cdiv(m, 128) + M // 128) * _cdiv(n, bn) + N // bn, (M % 128) * bn + N % bn
    c = case.conv
    oh, ow = c.out_hw
    I, O, Y, X = torch.meshgrid(torch.arange(c.batch), torch.arange(c.oc), torch.arange(oh), torch.arange(ow),
                                indexing="ij")
    la = launch_of(case)
    if la.kernel == "stem":
        p = Y * ow + X
        return I * _cdiv(oh * ow, 128) + p // 128, O * 128 + p % 128
    R, C = halo_tile(c, case.mode, la.kernel)
    bn = gemm_bn(c.oc)
    tile = ((I * _cdiv(oh, R) + Y // R) * _cdiv(ow, C) + X // C) * _cdiv(c.oc, bn) + O // bn
    return tile, ((O % bn) * R + Y % R) * C + X % C


def simulate(defect: str, good, tile, pos, grid: int):
    """`good` as a kernel with `defect` would leave it on `grid` CTAs (CTA b runs tiles b, b + grid, ...)."""
    bad = good.clone()
    T = int(tile.max()) + 1
    at = lambda t: {int(p): i for i, p in zip(torch.nonzero(tile.flatten() == t).flatten().tolist(),  # noqa: E731
                                              pos.flatten()[tile.flatten() == t].tolist())}
    flat, src = bad.view(-1), good.reshape(-1)
    if defect == "previous_tile_added":        # the accumulators are not cleared between a CTA's tiles
        for t in range(grid, T):
            prev = at(t - grid)
            for p, i in at(t).items():
                if p in prev:
                    flat[i] = flat[i] + src[prev[p]]
    elif defect == "last_tile_unwritten":      # a CTA stops one tile early: the guard NaN stays
        for i in at(T - 1).values():
            flat[i] = math.nan
    else:                                      # the second tile of CTA 0 lands one tile over
        dst = at(grid + 1)
        for p, i in at(grid).items():
            if p in dst:
                flat[dst[p]] = src[i]
    return bad


DEFECTS = ("previous_tile_added", "last_tile_unwritten", "tile_shifted")


def _defect_cases():
    out, seen = [], set()
    for cs in (gen_case(i) for i in range(N_CASES)):
        if cs.conv is not None and (cs.conv.group > 1 or cs.algo != SGECONV or cs.out_off):
            continue
        if cs.ip is not None or (cs.conv is not None and cs.conv.batch * cs.conv.oc * cs.conv.h * cs.conv.w > 400000):
            continue
        la = launch_of(cs)
        if la.kernel in seen or la.tiles < 5 or la.kernel == "gather":
            continue
        seen.add(la.kernel)
        out.append(cs)
    return out


@pytest.mark.parametrize("defect", DEFECTS)
def test_checker_rejects_cross_tile_defects(defect):
    """On one sweep case per kernel: the defect on a capped run differs from the cap-0 run, and the same defect in every
    run (as at cap 0 on a layer of more tiles than CTAs) leaves the float64 bound."""
    pytest.importorskip("feathercnn_b200._lib")
    picked = _defect_cases()
    assert {launch_of(cs).kernel for cs in picked} == set(KERNELS), [launch_of(cs).kernel for cs in picked]
    for cs in picked:
        tile, pos = tile_layout(cs)
        if cs.gemm is not None:
            g_, m, n, k = cs.gemm
            gen = torch.Generator().manual_seed(cs.idx)
            a, b = torch.rand((g_, m, k), generator=gen) * 2 - 1, torch.randn((g_, n, k), generator=gen)
            ref = torch.einsum("gmk,gnk->gmn", a.double(), b.double())
            s = torch.einsum("gmk,gnk->gmn", a.double().abs(), b.double().abs())
            check = lambda got: excess(got, ref, s, eps_for("gemm", TF32) + k * U)[0]  # noqa: E731
        else:
            c = cs.conv
            x, w, b, r = make_data(c, "cpu")
            ref, bound, s = conv_expect(c, x, w, b, r, eps_for("sgeconv", TF32) + c.K * U)
            check = lambda got: check_conv(got, ref, bound, s)[0]  # noqa: E731
        good = ref.float()
        assert check(good) <= 1.0 and differing(good, good) == 0
        for cap in (2, 3):
            bad = simulate(defect, good, tile, pos, cap)
            assert differing(bad, good) > 0, (cs.name, cap)
            used = check(bad)
            assert not used <= 1.0, (cs.name, defect, cap, used)


# ---- nets --------------------------------------------------------------------------------------------------------------
# (model, size, batch, kinds of persistent kernel it launches: 0 TensorGEMM, 1 implicit GEMM).  MobileNet-v2's
# classifier is a 1x1 convolution and at 32 px none of its layers takes Winograd: it runs no TensorGEMM.
NETS = [("mini", {}, 2, (0, 1)), ("mobilenet_v2", dict(size=32), 2, (1,)), ("vgg16", dict(size=32), 2, (0, 1)),
        ("resnet50", dict(size=64), 2, (0, 1)), ("shufflenet_v2", dict(size=96), 2, (0, 1))]


@gpu
@pytest.mark.parametrize("model,kw,batch,kinds", NETS, ids=[n[0] for n in NETS])
def test_net_blobs_do_not_depend_on_the_cta_count(ctas, tmp_path, model, kw, batch, kinds):
    """Fused, graph-captured nets, each in a fresh Net (the graphs capture the grids) at caps 1 and 3: every surviving
    blob bit-identical to cap 0."""
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m = modelgen.ZOO[model](**kw)
    param, binf = m.save(tmp_path / model)
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])
    lib = _lib()
    blobs = {}
    for cap in (0, 1, 3):
        ctas(cap)
        net = Net(fusion=True, cuda_graph=True)
        net.LoadParam(param)
        net.LoadWeights(binf)
        for _ in range(2):
            net.Forward(x)
        net.Synchronize()
        blobs[cap] = {n: net.Extract(n) for n in net.BlobNames()}
        del net
    for cap in (1, 3):
        assert blobs[cap].keys() == blobs[0].keys()
        bad = [n for n in blobs[0] if not np.array_equal(blobs[cap][n].view(np.int32), blobs[0][n].view(np.int32))]
        assert not bad, (cap, bad[:10])
    # the net runs the persistent kernels: the TensorGEMM (kind 0) and the implicit GEMM (kind 1)
    net = Net(fusion=True, cuda_graph=False)
    net.LoadParam(param)
    net.LoadWeights(binf)
    lib.fcuda_profile_tensor_gemm(1)
    try:
        net.Forward(x)
        net.Synchronize()
        launched = []
        for kind in kinds:
            n = ctypes.c_longlong()
            lib.fcuda_profile_collect_kind(kind, None, None, None, None, ctypes.byref(n))
            launched.append(n.value)
    finally:
        lib.fcuda_profile_tensor_gemm(0)
    assert all(launched), (kinds, launched)
    assert np.array_equal(net.Extract("prob").view(np.int32), blobs[0]["prob"].view(np.int32))
