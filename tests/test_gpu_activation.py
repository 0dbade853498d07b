"""Sigmoid, TanH, Swish, HardSigmoid and HardSwish on the GPU.

  - Each type against float64 within include/fcuda.h's stated bound, on seeded inputs at several scales and on special
    values: +-0, +-inf, NaN, subnormals, +-88 / +-89 / +-1e30 and the nextafter neighbours of the hard types' branch
    points.  HardSigmoid / HardSwish also bit for bit against the NumPy float32 restatement (test_activation_host), NaN payloads aside.
  - Tails of n = 1..9, pointers offset by 1..3 floats, in place, and the same bits eager and in a CUDA graph.
  - se_tiny, MobileNet-v3 Large / Small, EfficientNet-B0 and ESPCN through feather::Net at batch 2, with fusion on and
    off, each run eager and in a CUDA graph: every surviving layer within a per-element bound of its float64 restatement
    from the Net's own bottoms (so errors do not add up over depth), the activation layers within fcuda.h's bound, and
    the same launches per forward and identical bits in every blob with graphs on or off.

Per-element bounds of the other layers (U = 2^-23): a convolution chain CONV_REL * S + 4 U |ref| with S its absolute
sum (test_gpu_clip_prelu's rule: CONV_REL = 2^-13 covers the fp32-split contraction and the host's BatchNorm / Scale
folding); InnerProduct the same with S = |x| |w|^T + |b|; unfused BatchNorm / Scale 4 U S + U |ref|; an add U (|a| + |b|);
the SE multiply U |ref|; global average pooling (HW + 8) U mean |x|; Softmax test_gpu_clip_prelu's rule; ReLU, Split and
PixelShuffle exact.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_activation_host import ACTS, act64, hard_bounds, hard_np, layer64
from test_gpu_net_bounds import fetch, load_model, rebuild_chains

gpu = pytest.mark.gpu
U = 2.0 ** -23
CONV_REL = 2.0 ** -13
PNNX_ALPHA = float(np.float32(1.666667e-01))


def act_bound(kind, x, ref, alpha=0.2, beta=0.5):
    """include/fcuda.h's bound of each type, per element, from the float64 input x and the float64 value ref."""
    r = ref.abs()
    if kind == "Sigmoid":
        return 2.0 ** -21 * r + 2.0 ** -126
    if kind == "Swish":
        return 2.0 ** -21 * r + 2.0 ** -118
    if kind == "TanH":
        return 2.0 ** -22 * r + 2.0 ** -148
    a, b = float(np.float32(alpha)), float(np.float32(beta))
    xa = (x * a).abs()
    if kind == "HardSigmoid":
        return U * (xa + r) + 2.0 ** -149
    return U * (x.abs() * (xa + (x * a + b).abs()) + r) + 2.0 ** -149 * (x.abs() + 1)


def _within(got, x, kind, alpha=0.2, beta=0.5):
    """got (float32 tensor) against float64 at x: NaN exactly where float64 is NaN, infinities equal, else within the
    bound.  Returns the largest share of the bound used."""
    x64 = x.double()
    ref = act64(kind, x64, alpha, beta)
    g = got.double()
    nan = torch.isnan(ref)  # Swish(-inf): -inf / inf in fp32, -inf * 0 in float64; NaN both
    assert torch.equal(torch.isnan(g), nan), (kind, x[torch.isnan(g) != nan][:8])
    inf = torch.isinf(ref) & ~nan
    assert torch.equal(g[inf], ref[inf]), kind
    fin = ~nan & ~inf
    d = (g[fin] - ref[fin]).abs()
    b = act_bound(kind, x64[fin], ref[fin], alpha, beta)
    share = torch.where(d == 0, torch.zeros_like(d), d / b)  # the hard types' bound is 0 where they are exact
    used = share.max().item() if d.numel() else 0.0
    assert used <= 1.0, (kind, used, x64[fin][share.argmax()].item())
    return used


def _specials(alpha, beta):
    lo, hi = hard_bounds(alpha, beta)
    v = [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754944e-38, -1.1754944e-38, 88.0, -88.0,
         89.0, -89.0, 87.3, -87.3, 88.72, -88.72, 1e30, -1e30, 3.4e38, -3.4e38, 1.0, -1.0, 9.0, -9.0, 20.0, -20.0]
    for p in (lo, hi):
        v += [p, np.nextafter(p, np.float32(-np.inf)), np.nextafter(p, np.float32(np.inf))]
    return np.array(v, np.float32)


def _inputs(seed, n, alpha=0.2, beta=0.5):
    rng = np.random.default_rng(seed)
    parts = [_specials(alpha, beta)]
    for scale in (1e-3, 1.0, 4.0, 30.0, 100.0):
        parts.append((rng.standard_normal(n) * scale).astype(np.float32))
    parts.append(np.float32(10.0) ** rng.uniform(-40, 38, n).astype(np.float32) * rng.choice([-1, 1], n).astype(np.float32))
    return np.concatenate(parts).astype(np.float32)


HARD_PARAMS = [(0.2, 0.5), (PNNX_ALPHA, 0.5), (-0.25, 0.75), (3.0, -1.0)]


@gpu
@pytest.mark.parametrize("kind", ACTS)
def test_each_type_within_bound(cuda, kind):
    from feathercnn_b200 import booster
    params = HARD_PARAMS if kind.startswith("Hard") else [(0.2, 0.5)]
    for alpha, beta in params:
        x = _inputs(len(kind) * 7 + int(alpha * 100), 20000, alpha, beta)
        d = torch.from_numpy(x).cuda()
        got = booster.activation(d, kind, alpha, beta).cpu()
        _within(got, torch.from_numpy(x), kind, alpha, beta)
        if kind.startswith("Hard"):  # bit for bit; NaN payloads aside (the GPU returns its canonical NaN)
            g, want = got.numpy(), hard_np(x, kind, alpha, beta)
            nan = np.isnan(want)
            assert np.array_equal(np.isnan(g), nan), (kind, alpha, beta)
            assert np.array_equal(g[~nan].view(np.int32), want[~nan].view(np.int32)), (kind, alpha, beta)


@gpu
def test_sigmoid_and_swish_edges(cuda):
    from feathercnn_b200 import booster
    x = torch.tensor([-np.inf, np.inf, -100.0, 100.0, np.nan], device="cuda")
    s = booster.activation(x, "Sigmoid").cpu().numpy()
    w = booster.activation(x, "Swish").cpu().numpy()
    assert list(s[:4]) == [0.0, 1.0, 0.0, 1.0] and np.isnan(s[4])
    assert np.isnan(w[0]) and w[1] == np.inf and w[2] == 0.0 and np.signbit(w[2]) and w[3] == 100.0 and np.isnan(w[4])


@gpu
@pytest.mark.parametrize("kind", ACTS)
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_tails_offsets_in_place(cuda, kind, offset):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(offset)
    for n in list(range(1, 10)) + [1023, 4099]:
        x = (rng.standard_normal(n + offset) * 4).astype(np.float32)
        base = torch.from_numpy(x).cuda()
        src = base[offset:]
        out = torch.full((n + offset,), 7.0, device="cuda")
        booster.activation(src, kind, PNNX_ALPHA, 0.5, out=out[offset:])
        if offset:
            assert torch.all(out[:offset] == 7.0)
        ref = out[offset:].clone()
        _within(ref.cpu(), torch.from_numpy(x[offset:]), kind, PNNX_ALPHA, 0.5)
        booster.activation(src, kind, PNNX_ALPHA, 0.5, out=src)  # in place
        assert torch.equal(src.view(torch.int32), ref.view(torch.int32)), (kind, n, offset)


@gpu
@pytest.mark.parametrize("kind", ACTS)
def test_graph_replay_is_bit_identical(cuda, kind):
    from feathercnn_b200 import booster
    x = torch.from_numpy(_inputs(5, 50000)).cuda()
    eager = booster.activation(x, kind, PNNX_ALPHA, 0.5)
    out = torch.empty_like(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        booster.activation(x, kind, PNNX_ALPHA, 0.5, out=out)  # warm-up outside the capture
        g = torch.cuda.CUDAGraph()
        out.zero_()
        with torch.cuda.graph(g, stream=s):
            booster.activation(x, kind, PNNX_ALPHA, 0.5, out=out)
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), eager.view(torch.int32))


# ---- feather::Net -----------------------------------------------------------------------------------------------------
def _chain_layers(layers):
    """rebuild_chains takes a fused two-bottom add as an Eltwise: a BinaryOp ADD of two blobs is one (Net::ApplyFusion
    treats it so)."""
    out = []
    for L in layers:
        if L["type"] == "BinaryOp" and L["params"].get(0, 0) == 0 and len(L["bottoms"]) == 2:
            L = dict(L, type="Eltwise", params={0: 1}, binary_op=True)
        out.append(L)
    return out


def restate(ch, ins):
    """(top, float64 value, per-element bound, kind) of a chain from its bottoms `ins` (float64)."""
    L = ch.head
    typ = L["type"]
    xs = [ins[b] for b in L["bottoms"]]
    if typ in ("Convolution", "ConvolutionDepthWise", "InnerProduct"):
        absL = dict(L, w=L["w"].abs(), b=L["b"].abs() if L["b"] is not None else None)
        y = layer64(L, xs)[L["tops"][0]]
        S = layer64(absL, [x.abs() for x in xs])[L["tops"][0]]
        for op in ch.ops:
            if op["type"] == "Eltwise":
                r = ins[ch.residual]
                y, S = y + r, S + r.abs()
            elif op["type"] == "ReLU":
                y = y.clamp_min(0)
            else:
                from test_gpu_net_bounds import affine_of
                m, a, A = (v.to(y.device).view(1, -1, 1, 1) for v in affine_of(op))
                y, S = y * m + a, S * m.abs() + A
        return [(ch.tops[0], y, CONV_REL * S + 4 * U * y.abs(), typ)]
    assert not ch.ops, (L["name"], [o["name"] for o in ch.ops])
    if typ == "Eltwise":
        return [(ch.tops[0], xs[0] + xs[1], U * (xs[0].abs() + xs[1].abs()), "add")]
    res = layer64(L, xs)
    if typ == "Split":
        return [(t, v, torch.zeros_like(v), typ) for t, v in res.items()]
    y = res[L["tops"][0]]
    x = xs[0]
    if typ in ACTS:
        b = act_bound(typ, x, y, L["params"].get(0, 0.2), L["params"].get(1, 0.5))
    elif typ in ("BatchNorm", "Scale"):
        from test_gpu_net_bounds import affine_of
        m, a, A = (v.to(x.device).view(1, -1, 1, 1) for v in affine_of(L))
        b = 4 * U * (x.abs() * m.abs() + A) + U * y.abs()
    elif typ == "BinaryOp":
        b = U * y.abs()
    elif typ == "Pooling":
        b = (x.shape[2] * x.shape[3] + 8) * U * x.abs().mean(dim=(2, 3), keepdim=True)
    elif typ == "Softmax":
        b = 64 * U * (1 + x.abs().amax(dim=(1, 2, 3), keepdim=True)) * y + 2.0 ** -126
    elif typ in ("ReLU", "PixelShuffle", "Dropout"):
        b = torch.zeros_like(y)
    else:
        raise AssertionError(typ)
    return [(L["tops"][0], y, b, typ)]


def _net(param, binf, x, fusion, graph):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    for _ in range(3 if graph else 1):
        net.Forward(x)
    net.Synchronize()
    return net


def _all(net, name):
    return fetch(net, name, slice(None)).float()


MODELS = {"se_tiny": {}, "mobilenet_v3_large": {}, "mobilenet_v3_small": {}, "efficientnet_b0": {},
          "espcn": dict(height=90, width=160)}


@gpu
@pytest.mark.parametrize("fusion", [True, False], ids=["fused", "plain"])
@pytest.mark.parametrize("name", list(MODELS))
def test_model_layers_within_bounds(cuda, model_dir, name, fusion):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.ZOO[name](**MODELS[name])
    param, binf = mw.save(model_dir / f"act_{name}")
    layers = load_model(param, binf)
    x = np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(2)])
    eager = _net(param, binf, x, fusion, False)
    graph = _net(param, binf, x, fusion, True)
    # graphs on or off: the same launches and the same bits in every blob
    assert eager.launches_per_forward == graph.launches_per_forward > 0
    names = graph.BlobNames()
    assert names == eager.BlobNames()
    for n in names:
        assert torch.equal(_all(eager, n).view(torch.int32), _all(graph, n).view(torch.int32)), (name, fusion, n)
    del eager
    acts = [L for L in layers if L["type"] in ACTS]
    assert acts and all(graph.LayerFusedAway(L["name"]) == 0 for L in acts)
    if fusion:  # BatchNorm / Scale fold into the convolution ahead of them, activation or not
        assert all(graph.LayerFusedAway(L["name"]) == 1 for L in layers if L["type"] in ("BatchNorm", "Scale"))
        relus = [L for L in layers if L["type"] == "ReLU"]
        assert all(graph.LayerFusedAway(L["name"]) == 1 for L in relus)
    chains, _ = rebuild_chains(_chain_layers(layers), graph.LayerFusedAway, set(names))
    worst = {}
    for ch in chains:
        ins = {b: fetch(graph, b, slice(None)) for b in dict.fromkeys(ch.bottoms)}
        for top, want, bound, kind in restate(ch, ins):
            got = fetch(graph, top, slice(None)).reshape(want.shape)
            assert torch.isfinite(got).all(), (ch.head["name"], top)
            used = ((got - want).abs() / bound.clamp(min=1e-300)).max().item()
            worst[kind] = max(worst.get(kind, 0.0), used)
            assert used <= 1.0, (name, fusion, ch.head["name"], [o["name"] for o in ch.ops], kind, used)
        del ins
    print(f"\n{name} fusion={fusion}: {len(chains)} chains; worst share of the bound per kind: "
          + ", ".join(f"{k} {v:.3f}" for k, v in sorted(worst.items())))
