"""Vision Transformer layers on the host: LayerNorm, GELU, MemoryData and MultiHeadAttention parameters and rejections,
InnerProduct and Permute on rank-2 token blobs, the ABI return codes of fcuda_layer_norm_forward and
fcuda_attention_forward, fusion, ViT blob shapes, and a float64 restatement of each modelgen ViT's layer list against
torchvision's VisionTransformer with the same weights.  The restatement (`run64`) is also the reference of the GPU tests
(test_gpu_vit.py)."""
from __future__ import annotations

import ctypes
import math
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
HEAD = "7767517\n2 2\nInput data 0 1 data 0=8 1=4 2=1\n"
VIT_TYPES = ("LayerNorm", "GELU", "MemoryData", "MultiHeadAttention")


# ---- float64 restatement ---------------------------------------------------------------------------------------------
def load_vit(param, binf) -> list[dict]:
    """The layer list with every layer's weights in file order (ncnn ModelBin: matrices flagged, vectors raw)."""
    from oracle import oracle as O
    layers = O.parse_param(param)
    mb = O._BinReader(binf)
    t = lambda a: torch.from_numpy(np.array(a, np.float64))
    for L in layers:
        pd, typ = L["params"], L["type"]
        if typ == "Convolution":
            oc, k, size = pd[0], pd[1], pd[6]
            L["w"] = t(mb.load(size, 0)).reshape(oc, size // (oc * k * k), k, k)
            L["b"] = t(mb.load(oc, 1))
        elif typ == "InnerProduct":
            out, size = pd[0], pd[2]
            L["w"] = t(mb.load(size, 0)).reshape(out, size // out)
            L["b"] = t(mb.load(out, 1))
        elif typ == "LayerNorm":
            n = pd[0]
            L["g"], L["b"] = t(mb.load(n, 1)), t(mb.load(n, 1))
        elif typ == "MemoryData":
            w, h, c = pd.get(0, 0), pd.get(1, 0), pd.get(2, 0)
            L["data"] = t(mb.load(w * max(h, 1) * max(c, 1), 1)).reshape(max(c, 1), max(h, 1), w)
        elif typ == "MultiHeadAttention":
            e = pd[0]
            L["mats"] = [(t(mb.load(e * e, 0)).reshape(e, e), t(mb.load(e, 1))) for _ in range(4)]
    return layers


def mha64(L, x):
    """torch.nn.MultiheadAttention(batch_first=True) of x (N, L, E) with q = k = v, no mask, in float64."""
    e, heads = L["params"][0], L["params"].get(1, 1)
    d = e // heads
    scale = L["params"].get(6, 1.0 / math.sqrt(d))
    (wq, bq), (wk, bk), (wv, bv), (wo, bo) = [(w.to(x.device), b.to(x.device)) for w, b in L["mats"]]
    n, l, _ = x.shape
    q, k, v = [(x @ w.T + b).view(n, l, heads, d).transpose(1, 2) for w, b in ((wq, bq), (wk, bk), (wv, bv))]
    p = torch.softmax(scale * q @ k.transpose(-1, -2), dim=-1)
    o = (p @ v).transpose(1, 2).reshape(n, l, e)
    return o @ wo.T + bo


def layer64(L, ins):
    """One layer in float64 on blobs of storage shape (N, c, h, w)."""
    typ, pd = L["type"], L["params"]
    x = ins[0] if ins else None
    if typ == "Convolution":
        return F.conv2d(x, L["w"].to(x.device), L["b"].to(x.device), stride=pd.get(3, 1), padding=pd.get(4, 0))
    if typ == "Reshape":
        w, h = pd[0], pd.get(1, 1)
        return x.reshape(x.shape[0], 1, h, w)
    if typ == "Permute":
        assert pd[0] == 1
        return x.transpose(2, 3)
    if typ == "Concat":
        assert pd.get(0, 0) == 0
        return torch.cat(ins, dim=2)
    if typ == "BinaryOp":
        assert pd.get(0, 0) == 0
        return ins[0] + ins[1]
    if typ == "LayerNorm":
        assert pd[0] == x.shape[3]
        return F.layer_norm(x, (x.shape[3],), L["g"].to(x.device), L["b"].to(x.device), float(pd.get(1, 1e-3)))
    if typ == "MultiHeadAttention":
        return mha64(L, x[:, 0])[:, None]
    if typ == "InnerProduct":
        w, b = L["w"].to(x.device), L["b"].to(x.device)
        if x.shape[2] > 1 and x.shape[3] == w.shape[1]:  # rank-2 rows
            return x @ w.T + b
        return (x.reshape(x.shape[0], -1) @ w.T + b)[:, :, None, None]
    if typ == "GELU":
        if pd.get(0, 0):
            return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
        return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
    if typ == "Crop":
        hoff, outh = pd.get(1, 0), pd.get(4, 0)
        return x[:, :, hoff:hoff + outh]
    raise AssertionError(typ)


def run64(layers, x):
    """Every blob of the net for the input batch x (N, 3, H, W), float64."""
    blobs = {}
    for L in layers:
        if L["type"] == "Input":
            blobs[L["tops"][0]] = x.double()
        elif L["type"] == "MemoryData":
            blobs[L["tops"][0]] = L["data"].to(x.device).expand(x.shape[0], -1, -1, -1)
        elif L["type"] == "Split":
            for t in L["tops"]:
                blobs[t] = blobs[L["bottoms"][0]]
        else:
            blobs[L["tops"][0]] = layer64(L, [blobs[b] for b in L["bottoms"]])
    return blobs


def torchvision_vit(layers, size):
    """torchvision's VisionTransformer with the weights of the layer list (each block's heads as written)."""
    from torchvision.models.vision_transformer import VisionTransformer
    by = {L["name"]: L for L in layers}
    conv = by["conv_proj"]
    dim, patch = conv["w"].shape[0], conv["w"].shape[2]
    blocks = sorted({int(m.group(1)) for m in (re.match(r"layer(\d+)_attn", n) for n in by) if m})
    mlp = by["layer0_fc1"]["w"].shape[0]
    classes = by["logits"]["w"].shape[0]
    vt = VisionTransformer(size, patch, len(blocks), 1, dim, mlp, num_classes=classes).double().eval()
    with torch.no_grad():
        vt.conv_proj.weight.copy_(conv["w"])
        vt.conv_proj.bias.copy_(conv["b"])
        vt.class_token.copy_(by["class_token"]["data"].reshape(1, 1, dim))
        vt.encoder.pos_embedding.copy_(by["pos_embedding"]["data"].reshape(1, -1, dim))
        for i in blocks:
            blk = vt.encoder.layers[i]
            a = by[f"layer{i}_attn"]
            blk.self_attention = torch.nn.MultiheadAttention(dim, a["params"][1], batch_first=True).double().eval()
            mats = a["mats"]
            blk.self_attention.in_proj_weight.copy_(torch.cat([w for w, _ in mats[:3]]))
            blk.self_attention.in_proj_bias.copy_(torch.cat([b for _, b in mats[:3]]))
            blk.self_attention.out_proj.weight.copy_(mats[3][0])
            blk.self_attention.out_proj.bias.copy_(mats[3][1])
            for ln, tag in ((blk.ln_1, "ln1"), (blk.ln_2, "ln2")):
                ln.weight.copy_(by[f"layer{i}_{tag}"]["g"])
                ln.bias.copy_(by[f"layer{i}_{tag}"]["b"])
            for lin, tag in ((blk.mlp[0], "fc1"), (blk.mlp[3], "fc2")):
                lin.weight.copy_(by[f"layer{i}_{tag}"]["w"])
                lin.bias.copy_(by[f"layer{i}_{tag}"]["b"])
        vt.encoder.ln.weight.copy_(by["ln"]["g"])
        vt.encoder.ln.bias.copy_(by["ln"]["b"])
        vt.heads.head.weight.copy_(by["logits"]["w"])
        vt.heads.head.bias.copy_(by["logits"]["b"])
    return vt


@pytest.mark.parametrize("name", ["vit_tiny", "vit_b_16"])
def test_layer_list_matches_torchvision(tmp_path, name):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.ZOO[name]()
    param, binf = mw.save(tmp_path / name)
    layers = load_vit(param, binf)
    size = mw.shape["data"][1]
    x = torch.from_numpy(np.stack([modelgen.synthetic_input(mw.shape["data"], i) for i in range(2)])).double()
    got = run64(layers, x)["logits"].reshape(2, -1)
    with torch.no_grad():
        want = torchvision_vit(layers, size)(x)
    assert got.shape == want.shape
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err < 1e-10, err


# ---- shapes and fusion ------------------------------------------------------------------------------------------------
def _net_from(mw, tmp_path, fusion=False):
    from feathercnn_b200.net import Net
    param, _ = mw.save(tmp_path / "m")
    net = Net(fusion=fusion)
    net.LoadParam(param)
    return net


@pytest.mark.parametrize("name, tokens, dim", [("vit_tiny", 17, 64), ("vit_ti_16", 197, 192), ("vit_s_16", 197, 384),
                                               ("vit_b_16", 197, 768)])
def test_vit_blob_shapes(name, tokens, dim):
    from feathercnn_b200.tools import modelgen
    mw = modelgen.ZOO[name]()
    assert mw.shape["add_pos"] == (1, tokens, dim) and mw.rank["add_pos"] == 2
    assert mw.shape["layer0_attn"] == (1, tokens, dim) and mw.rank["layer0_attn"] == 2
    assert mw.shape["cls"] == (1, 1, dim)
    assert mw.shape["logits"][0] == (10 if name == "vit_tiny" else 1000)
    types = [l.split()[0] for l in mw.lines]
    blocks = 3 if name == "vit_tiny" else 12
    assert types.count("MultiHeadAttention") == blocks and types.count("GELU") == blocks
    assert types.count("LayerNorm") == 2 * blocks + 1 and types.count("MemoryData") == 2
    assert "Crop cls 1 1 ln cls 0=0 1=0 4=1" in mw.lines


def test_vit_tiny_covers_head_dims():
    from feathercnn_b200.tools import modelgen
    mw = modelgen.vit_tiny()
    dims = [int(re.search(r" 0=(\d+)", l).group(1)) // int(re.search(r" 1=(\d+)", l).group(1))
            for l in mw.lines if l.startswith("MultiHeadAttention")]
    assert dims == [16, 32, 64]


def test_no_vit_layer_is_fused(tmp_path):
    from feathercnn_b200.tools import modelgen
    net = _net_from(modelgen.vit_tiny(), tmp_path, fusion=True)
    net.FuseNow()
    for line in modelgen.vit_tiny().lines:
        typ, name = line.split()[:2]
        if typ in VIT_TYPES or typ in ("InnerProduct", "BinaryOp", "Permute", "Concat"):
            assert net.LayerFusedAway(name) == 0, name


def test_every_vit_type_is_registered():
    from feathercnn_b200.net import Net
    Net().LoadParamFromText(HEAD.replace("2 2", "2 2") + "LayerNorm ln 1 1 data out 0=8\n")
    Net().LoadParamFromText(HEAD + "GELU g 1 1 data out\n")
    Net().LoadParamFromText(HEAD + "MultiHeadAttention a 1 1 data out 0=16 1=1 2=256\n")
    Net().LoadParamFromText("7767517\n1 1\nMemoryData m 0 1 out 0=4 1=2\n")


# ---- loader rejections ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("line", [
    "LayerNorm ln 1 1 data out 0=0",                       # affine_size < 1
    "LayerNorm ln 1 1 data out 0=8 1=-1.0",                # negative eps
    "LayerNorm ln 1 1 data out 0=8 2=2",                   # affine neither 0 nor 1
    "GELU g 1 1 data out 0=2",                             # fast_gelu neither 0 nor 1
    "MultiHeadAttention a 1 1 data out 0=48 1=5 2=2304",   # 48 % 5 != 0
    "MultiHeadAttention a 1 1 data out 0=24 1=2 2=576",    # head_dim 12: not a multiple of 16
    "MultiHeadAttention a 1 1 data out 0=288 1=1 2=82944",  # head_dim 288 > 128
    "MultiHeadAttention a 1 1 data out 0=16 1=1 2=255",    # weight_data_size != embed_dim^2
    "MultiHeadAttention a 1 1 data out 0=16 1=1 2=256 5=1",  # attn_mask
    "MultiHeadAttention a 1 1 data out 0=16 1=1 2=256 3=8",  # one bottom with kdim != embed_dim
    "MultiHeadAttention a 1 1 data out 0=16 1=1 2=256 6=0.0",  # scale 0
    "MultiHeadAttention a 2 1 data data out 0=16 1=1 2=256",   # two bottoms
])
def test_load_param_rejects(line):
    from feathercnn_b200.net import FeatherError, Net
    with pytest.raises(FeatherError):
        Net().LoadParamFromText(HEAD + line + "\n")


@pytest.mark.parametrize("line", [
    "MemoryData m 0 1 out 0=4 1=2 2=3 11=2",  # depth
    "MemoryData m 0 1 out",                   # no dims
    "MemoryData m 0 1 out 0=4 1=-2",          # negative h
    "MemoryData m 1 1 data out 0=4",          # a bottom
])
def test_memory_data_rejects(line):
    from feathercnn_b200.net import FeatherError, Net
    text = "7767517\n2 2\nInput data 0 1 data 0=4\n" + line + "\n"
    with pytest.raises(FeatherError):
        Net().LoadParamFromText(text)


def test_multihead_attention_defaults_and_three_bottoms():
    from feathercnn_b200.net import Net
    text = ("7767517\n4 4\nInput q 0 1 q 0=32 1=5\nInput k 0 1 k 0=16 1=7\nInput v 0 1 v 0=8 1=7\n"
            "MultiHeadAttention a 3 1 q k v out 0=32 1=2 2=1024 3=16 4=8\n")
    net = Net()
    net.LoadParamFromText(text)
    assert "out" in net.BlobNames()


# ---- C ABI ------------------------------------------------------------------------------------------------------------
def test_layer_norm_abi_rejects_before_any_launch():
    from feathercnn_b200._lib import fcuda
    f = fcuda().fcuda_layer_norm_forward
    d = ctypes.c_void_p(16)
    assert f(None, d, 8, 2, None, None, 1e-5, None) == -100
    assert f(d, None, 8, 2, None, None, 1e-5, None) == -100
    assert f(d, d, 0, 2, None, None, 1e-5, None) == -100
    assert f(d, d, 8, 0, None, None, 1e-5, None) == -100
    assert f(d, d, 8, 2, d, None, 1e-5, None) == -200
    assert f(d, d, 8, 2, None, d, 1e-5, None) == -200
    for eps in (-1e-5, math.inf, math.nan):
        assert f(d, d, 8, 2, None, None, eps, None) == -200


def test_attention_abi_rejects_before_any_launch():
    from feathercnn_b200._lib import fcuda
    f = fcuda().fcuda_attention_forward
    q, o = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 30)
    ok = dict(ldq=192, ldk=192, ldv=192, batch=2, heads=1, d=64, lq=5, lk=7, scale=0.125)

    def call(o_=o, q_=q, **kw):
        a = dict(ok, **kw)
        return f(o_, q_, a["ldq"], q_, a["ldk"], q_, a["ldv"], a["batch"], a["heads"], a["d"], a["lq"], a["lk"],
                 a["scale"], None)
    assert call(o_=None) == -100 and call(q_=None) == -100
    for k in ("batch", "heads", "lq", "lk"):
        assert call(**{k: 0}) == -100, k
    for d in (0, 8, 24, 144, -16):
        assert call(d=d) == -200, d
    assert call(ldq=63) == -200 and call(ldk=63) == -200 and call(ldv=63) == -200
    assert call(heads=3, ldq=191) == -200                               # ld below heads * d
    assert call(heads=1025, ldq=1 << 17, ldk=1 << 17, ldv=1 << 17, lq=4096) == -200  # heads * query tiles > 65535
    for s in (0.0, math.inf, math.nan):
        assert call(scale=s) == -200
    assert call(o_=q) == -200                                           # output overlaps the operands
    assert call(o_=ctypes.c_void_p((1 << 20) + 4 * 100)) == -200


# ---- SASS -------------------------------------------------------------------------------------------------------------
def test_attention_kernel_issues_hgmma_without_local_memory():
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    so = ROOT / "feathercnn_b200" / "lib" / "libfcuda.so"
    sass = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    attn = {f.split()[0]: f for f in funcs if f.startswith("_ZN5fcuda16attention_kernel")}
    assert len(attn) == 8, sorted(attn)
    for name, body in attn.items():
        d = int(re.search(r"ILi(\d+)E", name).group(1))
        hgmma = len(re.findall(r"\bHGMMA\.", body))
        depbar = len(re.findall(r"WARPGROUP\.DEPBAR", body))
        assert hgmma == 3 * d // 16 + 12, (name, hgmma)     # S: 3 per k-step of 16; P V: 3 x 4 k-steps
        assert 1 <= depbar <= 2, (name, depbar)             # one wait per product, none per HGMMA
        assert not re.search(r"\b(LDL|STL)\b", body), name  # no local memory (spills)
