"""Vision Transformer kernels and nets on the GPU against float64.

- fcuda_attention_forward over a seeded sweep of Lq, Lk (1 and tails included), head_dim 16..128, heads, scale, both
  operand layouts (one fused [N L][3E] projection read in place, or three buffers) and more than 65535 images x heads,
  per element within the bound fcuda.h states;
- LayerNorm over rows and channel planes, with and without the affine, in place, and GELU in both forms, within their
  stated bounds;
- the same bits across batch splits and between eager runs and CUDA-graph replay;
- vit_tiny and ViT-Ti/S/B through feather::Net layer by layer against float64 (test_vit_host.run64's layers), with
  fusion and graphs on and off, and a MemoryData that is refilled when the batch changes."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from test_gpu_error_bounds import EPS_BF16X3, FP32_SPLIT, ip_rule
from test_gpu_net_bounds import fetch
from test_vit_host import layer64, load_vit

gpu = pytest.mark.gpu
U = 2.0 ** -24


# ---- bounds (include/fcuda.h) -----------------------------------------------------------------------------------------
def attention_bound(q, k, v, scale):
    """The per-element bound of fcuda_attention_forward for float64 q (N, H, Lq, d), k, v (N, H, Lk, d)."""
    d, lk = q.shape[-1], k.shape[-2]
    t = math.ceil(lk / 64)
    s = scale * q @ k.transpose(-1, -2)
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    a = q.abs() @ k.abs().transpose(-1, -2)
    dmax = (abs(scale) * a * (2.0 ** -14 + (d + 1) * 2.0 ** -21) + (t + 1) * U * (s - m).abs()).amax(-1, keepdim=True)
    eta = 2.01 * (dmax + (t + 1) * 2.0 ** -22 + (2 * t + 18) * U)
    w = (p @ v.abs()) / p.sum(-1, keepdim=True)
    ref = (p @ v) / p.sum(-1, keepdim=True)
    return ref, (2.01 * eta + 2.0 ** -14 + (3 * lk + 3 * t + 1) * 2.0 ** -23) * w + 2.0 ** -126, p, w


def layer_norm_bound(x, n, gamma, beta, eps):
    """Reference and bound of LayerNorm over runs of n floats of x (float64)."""
    r = x.reshape(-1, n)
    mu = r.mean(-1, keepdim=True)
    s2 = ((r - mu) ** 2).mean(-1, keepdim=True)
    sigma = torch.sqrt(s2 + eps)
    g = torch.ones(n, dtype=torch.float64, device=x.device) if gamma is None else gamma.double()
    b = torch.zeros(n, dtype=torch.float64, device=x.device) if beta is None else beta.double()
    y = (r - mu) / sigma * g + b
    L = math.ceil(n / 32) + 5
    e = (L + 1) * U * r.abs().mean(-1, keepdim=True)
    rho = (L + 6) * U + (e / sigma) ** 2
    bound = g.abs() * (rho * (r - mu).abs() + (1 + rho) * e) / sigma + 2.0 ** -23 * (
        y.abs() + g.abs() * (r - mu).abs() / sigma) + 2.0 ** -149
    return y.reshape(x.shape), bound.reshape(x.shape)


def gelu64(x, fast):
    if fast:
        return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def gelu_bound(x, ref):
    return 2.0 ** -21 * x.abs() + 2.0 ** -23 * ref.abs() + 2.0 ** -148


def _share(got, ref, bound):
    return ((got.double() - ref).abs() / bound).max().item()


# ---- attention --------------------------------------------------------------------------------------------------------
def _attn_cases():
    rng = np.random.default_rng(7)
    cases = [(1, 1, 16, 1, 1, None, True), (2, 3, 64, 197, 197, None, True), (1, 2, 128, 65, 64, 0.3, False),
             (2, 1, 32, 1, 577, None, False), (1, 4, 48, 130, 1, -0.5, False), (3, 2, 80, 63, 129, None, True),
             (1, 1, 96, 64, 65, 2.0, False), (1, 2, 112, 100, 33, None, True)]
    for _ in range(24):
        d = int(rng.choice(range(16, 129, 16)))
        heads = int(rng.integers(1, 5))
        lq = int(rng.choice([1, 2, 63, 64, 65, int(rng.integers(1, 300))]))
        lk = int(rng.choice([1, 2, 63, 64, 65, int(rng.integers(1, 300))]))
        scale = None if rng.random() < 0.5 else float(rng.uniform(0.05, 1.5) * rng.choice([-1, 1]))
        cases.append((int(rng.integers(1, 4)), heads, d, lq, lk, scale, bool(rng.random() < 0.5)))
    return cases


def _operands(n, heads, d, lq, lk, fused, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    e = heads * d
    if fused:  # one [N L][3E] buffer read in place, as MultiHeadAttention's fused projection writes it
        qkv = torch.randn((n, lq, 3 * e), generator=g, device="cuda")
        return qkv[:, :, :e], qkv[:, :, e:2 * e], qkv[:, :, 2 * e:]
    return (torch.randn((n, lq, e), generator=g, device="cuda"), torch.randn((n, lk, e), generator=g, device="cuda"),
            torch.randn((n, lk, e), generator=g, device="cuda") * 3)


def _heads(t, heads):
    n, l, e = t.shape
    return t.double().reshape(n, l, heads, e // heads).transpose(1, 2)


@gpu
@pytest.mark.parametrize("case", _attn_cases(), ids=lambda c: "n{}h{}d{}q{}k{}s{}{}".format(*c[:5], c[5], "f" if c[6] else ""))
def test_attention_within_bound(cuda, case):
    from feathercnn_b200 import booster
    n, heads, d, lq, lk, scale, fused = case
    if fused:
        lk = lq
    q, k, v = _operands(n, heads, d, lq, lk, fused, 7 * n + 13 * heads + d + 3 * lq + lk)
    sc = 1.0 / math.sqrt(d) if scale is None else scale
    got = booster.attention(q, k, v, heads, sc, out=torch.empty((n, lq, heads * d), device="cuda"))
    torch.cuda.synchronize()
    ref, bound, _, _ = attention_bound(_heads(q, heads), _heads(k, heads), _heads(v, heads), float(np.float32(sc)))
    used = _share(_heads(got, heads), ref, bound)
    assert used <= 1.0, (case, used)


@gpu
def test_attention_past_65535_images_and_batch_split(cuda):
    """33000 images x 2 heads on grid x; the bits of every image equal those of a run of that image's slice."""
    from feathercnn_b200 import booster
    n, heads, d, lq, lk = 33000, 2, 16, 3, 5
    q, k, v = _operands(n, heads, d, lq, lk, False, 3)
    got = booster.attention(q, k, v, heads)
    part = torch.cat([booster.attention(q[i:j], k[i:j], v[i:j], heads) for i, j in ((0, 7), (7, 32999), (32999, n))])
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int32), part.view(torch.int32))
    ref, bound, _, _ = attention_bound(_heads(q, heads), _heads(k, heads), _heads(v, heads), float(np.float32(0.25)))
    assert _share(_heads(got, heads), ref, bound) <= 1.0


@gpu
def test_attention_graph_replay_is_bit_identical(cuda):
    from feathercnn_b200 import booster
    q, k, v = _operands(2, 3, 64, 197, 197, True, 11)
    eager = booster.attention(q, k, v, 3)
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        booster.attention(q, k, v, 3, out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        booster.attention(q, k, v, 3, out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.view(torch.int32), out.view(torch.int32))


# ---- LayerNorm and GELU -----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("shape, n", [((4, 197, 768), 768), ((3, 1, 5), 5), ((2, 8, 7, 9), 63), ((2, 3, 40, 40), 1600),
                                      ((5, 33, 1025), 1025), ((1, 1, 1), 1)])
@pytest.mark.parametrize("affine", [True, False])
def test_layer_norm_within_bound(cuda, shape, n, affine):
    from feathercnn_b200 import booster
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(shape, generator=g, device="cuda") * 3 + 1.5
    gamma = torch.rand(n, generator=g, device="cuda") + 0.5 if affine else None
    beta = torch.rand(n, generator=g, device="cuda") - 0.5 if affine else None
    got = booster.layer_norm(x, n, gamma, beta, 1e-6)
    inplace = x.clone()
    booster.layer_norm(inplace, n, gamma, beta, 1e-6, out=inplace)
    torch.cuda.synchronize()
    ref, bound = layer_norm_bound(x.double(), n, gamma, beta, float(np.float32(1e-6)))
    assert _share(got, ref, bound) <= 1.0
    assert torch.equal(got.view(torch.int32), inplace.view(torch.int32))
    rows = x.numel() // n
    if rows > 1:  # the bits of a row do not depend on the launch that covers it
        half = (rows // 2) * n
        flat = x.reshape(-1)
        parts = torch.cat([booster.layer_norm(flat[:half], n, gamma, beta, 1e-6),
                           booster.layer_norm(flat[half:], n, gamma, beta, 1e-6)])
        torch.cuda.synchronize()
        assert torch.equal(parts.view(torch.int32), got.reshape(-1).view(torch.int32))


@gpu
@pytest.mark.parametrize("kind", ["GELU", "GELU_TANH"])
def test_gelu_within_bound(cuda, kind):
    from feathercnn_b200 import booster
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.cat([torch.randn(1 << 20, generator=g, device="cuda") * 4,
                   torch.tensor([0.0, -0.0, 1e-30, -1e-30, 5.0, -5.0, 10.0, -10.0, 30.0, -30.0, 1e4, -1e4, 3e12],
                                device="cuda")])
    got = booster.activation(x, kind)
    torch.cuda.synchronize()
    ref = gelu64(x.double(), kind == "GELU_TANH")
    assert _share(got, ref, gelu_bound(x.double(), ref)) <= 1.0
    assert torch.isnan(booster.activation(torch.tensor([math.nan], device="cuda"), kind)).all()


# ---- nets -------------------------------------------------------------------------------------------------------------
def mha_bound(L, x, got_shape_like):
    """Reference and bound of a one-bottom MultiHeadAttention layer for its fp32 input x (N, L, E) in float64: the
    projections' InnerProduct bound, the attention bound, the attention's sensitivity to the projection errors, and the
    output projection's bound."""
    e, heads = L["params"][0], L["params"][1]
    d = e // heads
    scale = float(np.float32(L["params"].get(6, 1.0 / math.sqrt(d))))
    coef = ip_rule(e, FP32_SPLIT)[1]
    (wq, bq), (wk, bk), (wv, bv), (wo, bo) = [(w.to(x.device), b.to(x.device)) for w, b in L["mats"]]
    proj, err = [], []
    for w, b in ((wq, bq), (wk, bk), (wv, bv)):
        y = x @ w.T + b
        proj.append(_heads(y, heads))
        err.append(_heads(coef * (x.abs() @ w.abs().T + b.abs()) + U * y.abs(), heads))
    q, k, v = proj
    dq, dk, dv = err
    o, b_att, p, w_abs = attention_bound(q, k, v, scale)
    ds = (abs(scale) * (dq @ k.abs().transpose(-1, -2) + (q.abs() + dq) @ dk.transpose(-1, -2))).amax(-1, keepdim=True)
    do = b_att + 4.02 * ds * w_abs + (p @ dv) / p.sum(-1, keepdim=True)
    n, _, lq, _ = o.shape
    o, do = [t.transpose(1, 2).reshape(n, lq, e) for t in (o, do)]
    ref = o @ wo.T + bo
    bound = do @ wo.abs().T + coef * (o.abs() @ wo.abs().T + bo.abs()) + U * ref.abs()
    return ref, bound


def net_bound(L, ins, ref):
    typ = L["type"]
    x = ins[0] if ins else None
    if typ == "Convolution":
        k = L["w"][0].numel()
        s = torch.nn.functional.conv2d(x.abs(), L["w"].abs().to(x.device), L["b"].abs().to(x.device),
                                       stride=L["params"].get(3, 1))
        return (EPS_BF16X3 + k * 2.0 ** -23) * s + U * ref.abs()
    if typ == "InnerProduct":
        w, b = L["w"].to(x.device), L["b"].to(x.device)
        xs = x if (x.shape[2] > 1 and x.shape[3] == w.shape[1]) else x.reshape(x.shape[0], -1)
        s = xs.abs() @ w.abs().T + b.abs()
        s = s if xs is x else s[:, :, None, None]
        return ip_rule(w.shape[1], FP32_SPLIT)[1] * s + U * ref.abs()
    if typ == "LayerNorm":
        return layer_norm_bound(x, x.shape[3], L["g"].to(x.device), L["b"].to(x.device),
                                float(np.float32(L["params"].get(1, 1e-3))))[1]
    if typ == "GELU":
        return gelu_bound(x, ref)
    if typ == "BinaryOp":
        return U * ref.abs()
    return torch.zeros_like(ref)  # Reshape, Permute, Concat, Crop: copies


def _net(param, binf, x, fusion, graph):
    from feathercnn_b200.net import Net
    net = Net(fusion=fusion, cuda_graph=graph)
    net.LoadParam(param)
    net.LoadWeights(binf)
    for _ in range(3 if graph else 1):
        net.Forward(x)
    net.Synchronize()
    return net


@gpu
@pytest.mark.parametrize("fusion", [True, False], ids=["fused", "plain"])
@pytest.mark.parametrize("name", ["vit_tiny", "vit_ti_16", "vit_s_16", "vit_b_16"])
def test_vit_layers_within_bounds(cuda, model_dir, name, fusion):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.ZOO[name]()
    param, binf = mw.save(model_dir / f"vit_{name}")
    layers = load_vit(param, binf)
    x = np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(2)])
    eager = _net(param, binf, x, fusion, False)
    graph = _net(param, binf, x, fusion, True)
    assert eager.launches_per_forward == graph.launches_per_forward > 0
    names = graph.BlobNames()
    assert names == eager.BlobNames()
    for b in names:
        assert torch.equal(fetch(eager, b, slice(None)).float().view(torch.int32),
                           fetch(graph, b, slice(None)).float().view(torch.int32)), (name, fusion, b)
    del eager
    worst = {}
    for L in layers:
        if L["type"] in ("Input", "Split", "MemoryData"):
            continue
        assert graph.LayerFusedAway(L["name"]) == 0, L["name"]
        ins = [fetch(graph, b, slice(None)).reshape(2, *graph.BlobShape(b)[1:]) for b in L["bottoms"]]
        got = fetch(graph, L["tops"][0], slice(None)).reshape(2, *graph.BlobShape(L["tops"][0])[1:])
        if L["type"] == "MultiHeadAttention":
            ref, bound = mha_bound(L, ins[0][:, 0], None)
            ref, bound = ref[:, None], bound[:, None]
        else:
            ref = layer64(L, ins)
            bound = net_bound(L, ins, ref)
        got = got.reshape(ref.shape)
        assert torch.isfinite(got).all(), L["name"]
        used = ((got - ref).abs() / bound.clamp(min=1e-300)).max().item() if bound.abs().max() > 0 else \
            float(not torch.equal(got, ref))
        worst[L["type"]] = max(worst.get(L["type"], 0.0), used)
        assert used <= 1.0, (name, fusion, L["name"], used)
    print(f"\n{name} fusion={fusion}: worst share of the bound per type: "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


@gpu
def test_memory_data_refilled_when_batch_changes(cuda, model_dir):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.vit_tiny()
    param, binf = mw.save(model_dir / "vit_tiny_batch")
    layers = {L["name"]: L for L in load_vit(param, binf)}
    pos = layers["pos_embedding"]["data"].float().cuda()
    from feathercnn_b200.net import Net
    net = Net(fusion=True, cuda_graph=True)
    net.LoadParam(param)
    net.LoadWeights(binf)
    for batch in (2, 5, 5, 5, 1, 2, 2):
        x = np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(batch)])
        net.Forward(x)
        net.Synchronize()
        got = fetch(net, "pos_embedding", slice(None)).float()
        assert got.shape[0] == batch and torch.equal(got, pos.expand(batch, -1, -1, -1).reshape(got.shape)), batch
        logits = net.Extract("logits").reshape(batch, -1)
        ref = layer64(layers["logits"], [fetch(net, "cls", slice(None)).reshape(batch, 1, 1, -1)]).reshape(batch, -1)
        assert np.allclose(logits, ref.cpu().numpy(), rtol=1e-4, atol=1e-4)


@gpu
def test_three_bottom_attention_layer(cuda, model_dir):
    """MultiHeadAttention with separate q, k, v (kdim, vdim != embed_dim) against torch.nn.MultiheadAttention."""
    from feathercnn_b200.net import Net
    rng = np.random.default_rng(3)
    e, heads, kdim, vdim, lq, lk = 64, 2, 48, 80, 70, 130
    mats = [(rng.standard_normal((e, i)) / math.sqrt(i), rng.uniform(-0.1, 0.1, e)) for i in (e, kdim, vdim, e)]
    blob = b""
    import struct
    for w, b in mats:
        blob += struct.pack("<I", 0) + w.astype(np.float32).tobytes() + b.astype(np.float32).tobytes()
    (model_dir / "mha3.bin").write_bytes(blob)
    (model_dir / "mha3.param").write_text(
        f"7767517\n7 7\nInput q 0 1 q 0={e} 1={lq}\nInput k 0 1 k 0={kdim} 1={lk}\nInput v 0 1 v 0={vdim} 1={lk}\n"
        f"Reshape rq 1 1 q q2 0={e} 1={lq}\nReshape rk 1 1 k k2 0={kdim} 1={lk}\nReshape rv 1 1 v v2 0={vdim} 1={lk}\n"
        f"MultiHeadAttention a 3 1 q2 k2 v2 out 0={e} 1={heads} 2={e * e} 3={kdim} 4={vdim}\n")
    net = Net()
    net.LoadParam(str(model_dir / "mha3.param"))
    net.LoadWeights(str(model_dir / "mha3.bin"))
    xs = [torch.randn((2, 1, l, w), device="cuda") for l, w in ((lq, e), (lk, kdim), (lk, vdim))]
    for name, t in zip("qkv", xs):
        net.FeedInputDevice(t.data_ptr(), t.shape, name)
    net.Forward()
    net.Synchronize()
    got = fetch(net, "out", slice(None)).reshape(2, lq, e)
    m = torch.nn.MultiheadAttention(e, heads, kdim=kdim, vdim=vdim, batch_first=True).double().cuda()
    with torch.no_grad():
        m.q_proj_weight.copy_(torch.from_numpy(np.float32(mats[0][0])).double())
        m.k_proj_weight.copy_(torch.from_numpy(np.float32(mats[1][0])).double())
        m.v_proj_weight.copy_(torch.from_numpy(np.float32(mats[2][0])).double())
        m.in_proj_bias.copy_(torch.from_numpy(np.float32(np.concatenate([b for _, b in mats[:3]]))).double())
        m.out_proj.weight.copy_(torch.from_numpy(np.float32(mats[3][0])).double())
        m.out_proj.bias.copy_(torch.from_numpy(np.float32(mats[3][1])).double())
        ref = m(*[t[:, 0].double() for t in xs], need_weights=False)[0]
    err = ((got - ref).abs().max() / ref.abs().max()).item()
    assert err < 1e-4, err
