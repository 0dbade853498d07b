"""Super-resolution's PixelShuffle on the GPU.

  - PixelShuffle bit for bit against NumPy (test_sr_host.pixel_shuffle_ref) for r = 1 to 4, both modes, batch > 1, odd
    heights and widths, -0.0 and NaN payloads, an unaligned input, and more than 65535 (n, c) planes.
  - The fused tail (an addend upsampled by a nearest map and added in the same pass) bit-identical to PixelShuffle,
    Interp and Eltwise SUM run as three calls, and to NumPy: scale and explicit-size maps, NaN in either input, and r = 3
    on a row of 3 * (2^22 + 128) outputs, where fp32 1/3 reads other columns than X // 3.
  - The same bits eager and in a CUDA graph.
  - Reshape rejects a channel count that is not a multiple of r^2.
  - modelgen's sr_tiny, a small srvgg_compact and small edsr_baseline nets (x 3 and x 4) through feather::Net, batch 2,
    with fusion and CUDA graphs on and off: every convolution within test_gpu_net_bounds' float64 bounds, PReLU (as
    test_gpu_clip_prelu restates it), PixelShuffle with or without its fused tail, Interp, ReLU and Eltwise bit for bit;
    the tail's Interp and Eltwise fused away where the pattern holds, and the outputs the same bits with graphs on and
    off (and, for the nets without residual convolution epilogues, with fusion on and off).
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_gpu_clip_prelu import _prelu_np
from test_gpu_faster_rcnn import SETTINGS, _all, _bits_equal
from test_gpu_net_bounds import CONV_TYPES, check_chain, rebuild_chains
from test_sr_host import WIDE_X3, pixel_shuffle_ref, upsample_ref

gpu = pytest.mark.gpu
F = np.float32
PAYLOAD_NAN = np.array([0x7FC12345], np.uint32).view(np.float32)[0]


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _ps(x, r, mode=0, addend=None, scale=None):
    from feathercnn_b200 import booster
    return booster.pixel_shuffle(x if torch.is_tensor(x) else _t(x), r, mode,
                                 None if addend is None else (addend if torch.is_tensor(addend) else _t(addend)), scale)


def _same_or_nan(a, b):
    """Bit-identical where either is a number; NaN in the same places (NumPy keeps payloads the GPU add replaces)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int32), b[~nb].view(np.int32))


# ---- PixelShuffle alone ---------------------------------------------------------------------------------------------
SHAPES = [(2, 3, 5), (3, 7, 9), (1, 1, 1), (2, 16, 33)]   # (batch, H, W)


@gpu
@pytest.mark.parametrize("r", [1, 2, 3, 4])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("nhw", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_pixel_shuffle_bit_exact(cuda, r, mode, nhw):
    n, h, w = nhw
    c = 3 * r * r
    x = np.random.default_rng(r * 10 + mode).standard_normal((n, c, h, w)).astype(np.float32)
    x.flat[0] = -0.0
    x.flat[-1] = PAYLOAD_NAN
    want = pixel_shuffle_ref(x, r, mode)
    assert _bits_equal(_ps(x, r, mode).cpu().numpy(), want)
    flat = torch.zeros(x.size + 1, device="cuda")
    flat[1:] = _t(x.ravel())
    assert _bits_equal(_ps(flat[1:].view(x.shape), r, mode).cpu().numpy(), want)     # 4 bytes off alignment


@gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_pixel_shuffle_more_planes_than_grid_rows(cuda, mode):
    """2 x 33000 output planes: more than the 65535 CTA rows, so CTAs loop over planes."""
    x = np.random.default_rng(7).standard_normal((2, 4 * 33000, 1, 3)).astype(np.float32)
    assert _bits_equal(_ps(x, 2, mode).cpu().numpy(), pixel_shuffle_ref(x, 2, mode))


# ---- the fused tail -------------------------------------------------------------------------------------------------
def _three_calls(x, r, mode, base, scale):
    from feathercnn_b200 import booster
    y = _ps(x, r, mode)
    up = booster.interp(_t(base), y.shape[2] if scale is None else 0, y.shape[3] if scale is None else 0, "nearest",
                        scale=scale)
    return booster.eltwise_add(y, up)


TAILS = [(2, 0, (2, 5, 7), 2.0), (3, 0, (2, 9, 11), 3.0), (3, 1, (1, 4, 6), None), (4, 1, (3, 6, 5), 4.0),
         (2, 1, (2, 3, 3), None), (1, 0, (2, 4, 5), 1.0)]


@gpu
@pytest.mark.parametrize("r, mode, nhw, scale", TAILS, ids=[f"r{t[0]}-m{t[1]}-{'s' if t[3] else 'size'}" for t in TAILS])
def test_fused_tail_equals_three_calls(cuda, r, mode, nhw, scale):
    n, h, w = nhw
    rng = np.random.default_rng(r + 3 * mode)
    x = rng.standard_normal((n, 3 * r * r, h, w)).astype(np.float32)
    base = rng.standard_normal((n, 3, h, w)).astype(np.float32)
    x[0, 0, 0, 0] = PAYLOAD_NAN
    base[-1, -1, -1, -1] = np.nan
    base[0, 1, 0, 0] = np.inf
    fused = _ps(x, r, mode, base, scale).cpu().numpy()
    assert _bits_equal(fused, _three_calls(x, r, mode, base, scale).cpu().numpy())
    s = F(1) / F(scale) if scale else F(h) / F(h * r)
    with np.errstate(invalid="ignore"):
        want = pixel_shuffle_ref(x, r, mode) + upsample_ref(base, h * r, w * r, s, s)
    assert _same_or_nan(fused, want)


@gpu
def test_fused_tail_fp32_third_on_a_wide_row(cuda):
    """r = 3 on a 1 x WIDE_X3 plane: the fused tail reads the addend where ncnn's nearest Interp does (fp32 1/3), which
    for some columns is not X // 3."""
    rng = np.random.default_rng(9)
    x = rng.standard_normal((1, 9, 1, WIDE_X3)).astype(np.float32)
    base = rng.standard_normal((1, 1, 1, WIDE_X3)).astype(np.float32)
    fused = _ps(x, 3, 0, base, 3.0).cpu().numpy()
    assert _bits_equal(fused, _three_calls(x, 3, 0, base, 3.0).cpu().numpy())
    third = F(1) / F(3.0)
    want = pixel_shuffle_ref(x, 3, 0) + upsample_ref(base, 3, 3 * WIDE_X3, third, third)
    assert _bits_equal(fused, want)
    by_division = pixel_shuffle_ref(x, 3, 0) + base[:, :, np.zeros(3, int)][:, :, :, np.arange(3 * WIDE_X3) // 3]
    assert not _bits_equal(fused, by_division)


@gpu
@pytest.mark.parametrize("tail", [False, True])
def test_graph_equals_eager(cuda, tail):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(5)
    x = _t(rng.standard_normal((2, 27, 37, 53)))
    base = _t(rng.standard_normal((2, 3, 37, 53))) if tail else None
    ref = _ps(x, 3, 1, base, 3.0 if tail else None).cpu().numpy()
    out = torch.empty((2, 3, 111, 159), device="cuda")
    booster.pixel_shuffle(x, 3, 1, base, 3.0 if tail else None, out)        # warm up outside the capture
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    out.zero_()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        booster.pixel_shuffle(x, 3, 1, base, 3.0 if tail else None, out)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert _bits_equal(out.cpu().numpy(), ref)


@gpu
@pytest.mark.parametrize("body", ["PixelShuffle p 1 1 d p 0=2", "PixelShuffle p 1 1 d p 0=3 1=1"])
def test_reshape_rejects_channels(cuda, tmp_path, body):
    """6 channels are not a multiple of 4 or 9: FEATHER_ERR_TOPOLOGY at Reshape, which Net reports as -100."""
    from feathercnn_b200.net import FeatherError, Net
    net = Net()
    net.LoadParamFromText(f"7767517\n2 2\nInput d 0 1 d 0=6 1=5 2=6\n{body}\n")
    empty = tmp_path / "empty.bin"
    empty.write_bytes(b"")
    net.LoadWeights(str(empty))
    with pytest.raises(FeatherError) as e:
        net.Forward(np.zeros((1, 6, 5, 6), np.float32))
    assert e.value.code == -100


# ---- models end to end ----------------------------------------------------------------------------------------------
MODELS = {"sr_tiny": ("sr_tiny", {}),
          "srvgg_small": ("srvgg_compact", dict(num_conv=3, num_feat=16, height=20, width=28)),
          "edsr_x3_small": ("edsr_baseline", dict(scale=3, n_resblocks=2, n_feats=16, height=12, width=10)),
          "edsr_x4_small": ("edsr_baseline", dict(scale=4, n_resblocks=2, n_feats=16, height=12, width=10))}
TAIL_FUSED = {"sr_tiny": {"base", "output"}, "srvgg_small": {"base", "output"}}
OUTPUT = {"sr_tiny": "output", "srvgg_small": "output", "edsr_x3_small": "add_mean", "edsr_x4_small": "add_mean"}


def _load_layers(param, binf):
    """The param file's layers with the convolutions' weights and biases and the PReLU slopes, in file order."""
    from oracle import oracle as O
    layers = O.parse_param(param)
    mb = O._BinReader(binf)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))  # noqa: E731
    for L in layers:
        pd = L["params"]
        if L["type"] in CONV_TYPES:
            k, num, size = pd.get(1, 0), pd.get(0, 0), pd.get(6, 0)
            L["w"] = t(mb.load(size, 0).reshape(num, size // (num * k * k), k, k))
            L["b"] = t(mb.load(num, 1)) if pd.get(5, 0) else None
        elif L["type"] == "PReLU":
            L["slope"] = np.asarray(mb.load(pd[0], 1), np.float32)
    return layers


@pytest.fixture(scope="module")
def sr_models(tmp_path_factory):
    from feathercnn_b200.tools import modelgen
    d = tmp_path_factory.mktemp("sr")
    out = {}
    for key, (name, kw) in MODELS.items():
        m = modelgen.ZOO[name](**kw)
        param, binf = m.save(d / key)
        out[key] = (m, param, binf, _load_layers(param, binf))
    return out


def _fold_tails(net, layers):
    """The layer list as the Net runs it: a PixelShuffle whose tail fused writes the Eltwise's top and carries the
    Interp (`tail`); the fused Interp and Eltwise leave the list."""
    by_top = {t: L for L in layers for t in L["tops"]}
    tails = {}
    for L in layers:
        if L["type"] == "Eltwise" and net.LayerFusedAway(L["name"]):
            kinds = {by_top[b]["type"]: by_top[b] for b in L["bottoms"]}
            if set(kinds) == {"PixelShuffle", "Interp"}:
                assert net.LayerFusedAway(kinds["Interp"]["name"]) == 1
                tails[kinds["PixelShuffle"]["name"]] = (kinds["Interp"], L)
    drop = {n for up, e in tails.values() for n in (up["name"], e["name"])}
    out = []
    for L in layers:
        if L["name"] in drop:
            continue
        if L["name"] in tails:
            up, e = tails[L["name"]]
            L = dict(L, tops=list(e["tops"]), tail=up)
        out.append(L)
    return out


def _interp_scales(L, h, w, oh, ow):
    pd = L["params"]
    if pd.get(3, 0) and pd.get(4, 0):
        return F(h) / F(oh), F(w) / F(ow)
    return F(1) / F(pd.get(1, 1.0)), F(1) / F(pd.get(2, 1.0))


def _check_layers(net, layers):
    """Convolution chains within their float64 bounds, every other layer bit for bit from the Net's own bottoms.
    Returns the count of each layer type checked."""
    chains, _ = rebuild_chains(_fold_tails(net, layers), net.LayerFusedAway, set(net.BlobNames()))
    failures, seen = [], {}
    arr = lambda name: _all(net, name).float().cpu().numpy()  # noqa: E731
    for ch in chains:
        L = ch.head
        typ = L["type"]
        seen[typ] = seen.get(typ, 0) + 1
        if typ in ("Input", "Split"):
            continue
        if typ in CONV_TYPES:
            ins = {b: _all(net, b) for b in dict.fromkeys(ch.bottoms)}
            tops = {t: _all(net, t) for t in ch.tops}
            for top, used, _, kind, path in check_chain(ch, ins, tops, 2, net.LayerConvAlgo(L["name"])):
                if used > 1.0:
                    failures.append(f"{L['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
            continue
        assert not ch.ops, (L["name"], [o["name"] for o in ch.ops])
        got, x = arr(ch.tops[0]), arr(L["bottoms"][0])
        if typ == "PReLU":
            want = _prelu_np(x, L["slope"])
        elif typ == "ReLU":
            want = np.maximum(x, F(0))
        elif typ == "Eltwise":
            a, b = (arr(n) for n in L["bottoms"])
            want = a + b
        elif typ == "Interp":
            hs, ws = _interp_scales(L, x.shape[2], x.shape[3], got.shape[2], got.shape[3])
            want = upsample_ref(x, got.shape[2], got.shape[3], hs, ws)
        else:
            assert typ == "PixelShuffle", typ
            pd = L["params"]
            want = pixel_shuffle_ref(x, pd.get(0, 1), pd.get(1, 0))
            if "tail" in L:
                base = arr(L["tail"]["bottoms"][0])
                hs, ws = _interp_scales(L["tail"], base.shape[2], base.shape[3], want.shape[2], want.shape[3])
                want = want + upsample_ref(base, want.shape[2], want.shape[3], hs, ws)
                seen["tail"] = seen.get("tail", 0) + 1
        if not _bits_equal(got, want):
            failures.append(f"{L['name']} ({typ}): not bit-identical")
    assert not failures, "\n".join(failures[:20])
    return seen


def _run(param, binf, x, fusion, graph):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    for _ in range(3 if graph else 1):
        net.Forward(x)
    net.Synchronize()
    return net


@gpu
@pytest.mark.parametrize("key", list(MODELS))
def test_model_end_to_end(cuda, sr_models, key):
    from feathercnn_b200.tools import modelgen
    m, param, binf, layers = sr_models[key]
    batch = 2
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])
    outs = {}
    n_shuffles = sum(L["type"] == "PixelShuffle" for L in layers)
    for fusion, graph in SETTINGS:
        net = _run(param, binf, x, fusion, graph)
        out = OUTPUT[key]
        assert net.BlobShape(out) == (batch,) + m.shape[out]
        fused = {L["name"] for L in layers if net.LayerFusedAway(L["name"])}
        if not fusion:
            assert not fused
        elif key in TAIL_FUSED:
            assert fused == TAIL_FUSED[key]
        else:   # EDSR: each PixelShuffle feeds a convolution and stays; ReLUs and residual sums join convolutions
            assert not fused & {L["name"] for L in layers if L["type"] in ("PixelShuffle", "Interp")}
            assert fused == {n for L in layers for n in [L["name"]] if L["type"] in ("ReLU", "Eltwise")}
        seen = _check_layers(net, layers)
        assert seen["PixelShuffle"] == n_shuffles
        assert seen.get("tail", 0) == (1 if fusion and key in TAIL_FUSED else 0)
        outs[(fusion, graph)] = net.Extract(out)
        del net
    for fusion in (True, False):
        assert _bits_equal(outs[(fusion, True)], outs[(fusion, False)])
    if key in TAIL_FUSED:
        assert _bits_equal(outs[(True, True)], outs[(False, False)])
