"""Channel routing on the GPU: ShuffleChannel, Slice and the fused Concat -> ShuffleChannel -> Slice launch bit for bit
against NumPy (tests/test_route_host.py holds the definitions), on the 16-byte and the 4-byte path, and modelgen's
ShuffleNet-v2 and shuffle_tiny through feather::Net with fusion and CUDA graphs on and off: every routing output
bit-identical to NumPy of its bottoms, every other layer within its float64 bound, fused and unfused outputs identical,
batch independence, and the launches the fusion saves.  "Unfused" here is the route_fuse switch at 0: the net's other
fusions stay, so the convolutions run the same kernels on the same inputs and the outputs must be bit-identical."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_gpu_net_bounds import CONV_TYPES, check_chain, fetch, load_model, rebuild_chains
from test_route_host import ROUTE_TYPES, shuffle_ref, slice_ref

gpu = pytest.mark.gpu


def _dev(a: np.ndarray, misalign: bool) -> torch.Tensor:
    """a on the device; `misalign` puts it 4 bytes past a 16-byte boundary (the 4-byte path)."""
    t = torch.from_numpy(np.ascontiguousarray(a, np.float32))
    if not misalign:
        return t.cuda()
    buf = torch.empty(t.numel() + 1, device="cuda")
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 4
    return v


def _bits(t) -> np.ndarray:
    return (t.cpu().numpy() if isinstance(t, torch.Tensor) else t).view(np.uint32)


# ---- the layers alone ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("group", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("hw, misalign", [((8, 8), False), ((8, 8), True), ((7, 7), False), ((1, 3), False)])
@pytest.mark.parametrize("batch", [1, 7])
def test_shuffle_channel_bit_exact(cuda, group, reverse, hw, misalign, batch):
    from feathercnn_b200 import booster
    x = np.random.default_rng(group * 10 + batch).standard_normal((batch, 24) + hw).astype(np.float32)
    got = booster.shuffle_channel(_dev(x, misalign), group, reverse)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(got), shuffle_ref(x, group, reverse).view(np.uint32))


SLICE_CASES = [
    ((29,), 0, [-233, -233]), ((29,), -1, [5, 3, -233]), ((29,), 0, [4, 7]),            # rank 1; dropped remainder
    ((6, 9), 0, [-233, -233, -233]), ((6, 9), 1, [2, -233]), ((6, 9), -1, [1] * 9),      # rank 2
    ((6, 9), -2, [4]),
    ((12, 7, 7), 0, [-233, -233]), ((12, 8, 8), 0, [5, 4]), ((10, 8, 8), 0, [1] * 10),   # rank 3 c; > 8 tops
    ((12, 7, 9), 1, [-233, -233]), ((12, 7, 9), -2, [3, 3]),                              # h
    ((12, 7, 15), 2, [3, -233, 5]), ((4, 8, 16), -1, [4, 8, -233]),                        # w
]


@gpu
@pytest.mark.parametrize("shape, axis, slices", SLICE_CASES)
@pytest.mark.parametrize("misalign", [False, True])
@pytest.mark.parametrize("batch", [1, 7])
def test_slice_bit_exact(cuda, shape, axis, slices, misalign, batch):
    from feathercnn_b200 import booster
    x = np.random.default_rng(len(shape) + batch).standard_normal((batch,) + shape).astype(np.float32)
    got = booster.slice(_dev(x, misalign), slices, axis)
    torch.cuda.synchronize()
    a, sizes = slice_ref(shape, axis, slices)
    starts = np.cumsum([0] + sizes)
    assert len(got) == len(sizes)
    for t, s0, n in zip(got, starts, sizes):
        want = np.take(x, range(s0, s0 + n), axis=1 + a)
        assert np.array_equal(_bits(t), want.view(np.uint32))


@gpu
@pytest.mark.parametrize("hw", [(8, 8), (7, 7)])
@pytest.mark.parametrize("group, reverse", [(2, 0), (3, 1), (1, 0)])
@pytest.mark.parametrize("batch", [1, 7])
def test_fused_chain_equals_layers_one_by_one(cuda, hw, group, reverse, batch):
    """Concat of three sources -> ShuffleChannel -> Slice dropping a remainder, in one launch, against the three
    layers run one by one (the concatenation by torch.cat, a plain copy)."""
    from feathercnn_b200 import booster
    rng = np.random.default_rng(batch)
    xs = [rng.standard_normal((batch, c) + hw).astype(np.float32) for c in (6, 9, 3)]
    srcs = [_dev(x, False) for x in xs]
    fused = booster.route(srcs, [7, 5, 4], group, reverse)             # 16 of 18 channels
    cat = torch.cat(srcs, 1)
    one_by_one = booster.slice(booster.shuffle_channel(cat, group, reverse), [7, 5, 4, -233], 0)[:3]
    torch.cuda.synchronize()
    want = shuffle_ref(np.concatenate(xs, 1), group, reverse)
    for f, o, s0, n in zip(fused, one_by_one, (0, 7, 12), (7, 5, 4)):
        assert np.array_equal(_bits(f), _bits(o))
        assert np.array_equal(_bits(f), want[:, s0:s0 + n].view(np.uint32))
    # begin: the destinations may start inside the shuffled axis
    part = booster.route(srcs, [3, 2], group, reverse, begin=11)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(part[0]), want[:, 11:14].view(np.uint32))
    assert np.array_equal(_bits(part[1]), want[:, 14:16].view(np.uint32))


ROUTE_CASES = [
    # (source channels, destination sizes, group, reverse, begin, inner, batch): one fcuda_route_forward launch
    ([3, 1, 4, 1, 5, 9, 2, 6], [31], 1, 0, 0, 7, 2),          # Concat of eight unequal bottoms
    ([30], [30], 5, 1, 0, 4, 3),                             # ShuffleChannel, group != C / group
    ([5, 7], [3, 4, 2], 4, 0, 3, 1, 7),                      # Concat -> ShuffleChannel -> Slice from position 3, inner 1
]


@gpu
@pytest.mark.parametrize("srcs, sizes, group, reverse, begin, inner, batch", ROUTE_CASES)
@pytest.mark.parametrize("misalign", [False, True])
def test_route_cases_bit_exact(cuda, srcs, sizes, group, reverse, begin, inner, batch, misalign):
    from feathercnn_b200 import booster
    rng = np.random.default_rng(sum(srcs) + inner)
    xs = [rng.standard_normal((batch, c, inner)).astype(np.float32) for c in srcs]
    got = booster.route([_dev(x, misalign and k == 0) for k, x in enumerate(xs)], sizes, group, reverse, begin)
    torch.cuda.synchronize()
    want = np.concatenate(xs, 1)
    want = shuffle_ref(want, group, reverse) if group > 1 else want
    for t, s0, n in zip(got, np.cumsum([begin] + sizes), sizes):
        assert np.array_equal(_bits(t), want[:, s0:s0 + n].view(np.uint32))


HEAD = "Input data 0 1 data 0=6 1=5 2=12\n"


@gpu
@pytest.mark.parametrize("lines, fusion", [
    (["ShuffleChannel sc 1 1 data out 0=5"], False),                      # 12 % 5
    (["ShuffleChannel sc 1 1 data out 0=5 1=1"], False),
    (["Slice s 1 2 data out out2 -23300=2,8,5"], False),                   # sizes past the extent
    (["Slice s 1 2 data out out2 -23300=2,-233,4 1=1"], False),            # 5 / 2 rows, then 4 > 3
    (["Slice s 1 6 data o1 o2 o3 o4 o5 o6 -23300=6,-233,-233,-233,-233,-233,-233 1=1"], False),  # 5 / 6 = 0 rows
    (["Flatten f 1 1 data flat", "Slice s 1 2 flat out out2 -23300=2,-233,-233 1=1"], False),     # rank 1: no axis 1
    (["Split sp 1 2 data d1 d2", "Concat c 2 1 d1 d2 cat", "ShuffleChannel sc 1 1 cat out 0=5"], True),  # 24 % 5, fused
])
def test_reshape_rejects(cuda, tmp_path, lines, fusion):
    from feathercnn_b200.net import FeatherError, Net
    blobs = 1 + sum(int(ln.split()[3]) for ln in lines)
    net = Net(fusion=fusion)
    net.LoadParamFromText(f"7767517\n{1 + len(lines)} {blobs}\n{HEAD}" + "\n".join(lines) + "\n")
    empty = tmp_path / "empty.bin"
    empty.write_bytes(b"")
    net.LoadWeights(str(empty))
    with pytest.raises(FeatherError):
        net.Forward(np.zeros((1, 12, 5, 6), np.float32))
    if fusion:
        assert net.LayerFusedAway("c") == 1


# ---- nets ---------------------------------------------------------------------------------------------------------
NET_CASES = [("shufflenet_v2", dict(width=0.5, size=96)), ("shufflenet_v2", dict(width=1.0, size=96)),
             ("shuffle_tiny", {})]


@pytest.fixture
def route_fuse():
    """Sets the route_fuse switch for the nets created next; restores it afterwards."""
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    saved = lib.fcuda_get_tuning(b"route_fuse")
    yield lambda v: lib.fcuda_set_tuning(b"route_fuse", v)
    lib.fcuda_set_tuning(b"route_fuse", saved)


@pytest.fixture(scope="module")
def route_models(tmp_path_factory):
    from feathercnn_b200.tools import modelgen
    d = tmp_path_factory.mktemp("route")
    out = {}
    for name, kw in NET_CASES:
        key = f"{name}-{kw.get('width', '')}"
        m = modelgen.ZOO[name](**kw)
        param, binf = m.save(d / key.replace(".", "_"))
        out[key] = (m, param, binf, load_model(param, binf))
    return out


def _np_route(layer, xs):
    typ, p = layer["type"], layer["params"]
    if typ == "Concat":
        return [np.concatenate(xs, 1)]
    if typ == "ShuffleChannel":
        return [shuffle_ref(xs[0], p.get(0, 1), p.get(1, 0))]
    x = xs[0]
    slices = [int(v) for v in p[0]]
    a, sizes = slice_ref(x.shape[1:], p.get(1, 0), slices)
    starts = np.cumsum([0] + sizes)
    return [np.take(x, range(s, s + n), axis=1 + a) for s, n in zip(starts, sizes)]


def _route_groups(layers, fused_away):
    """(surviving routing layer, its chain of routing layers in order) for every routing layer that runs."""
    by_top = {t: L for L in layers for t in L["tops"]}
    groups = []
    for L in layers:
        if L["type"] not in ROUTE_TYPES or fused_away(L["name"]):
            continue
        chain = [L]
        while len(chain[0]["bottoms"]) == 1 and chain[0]["bottoms"][0] in by_top:
            p = by_top[chain[0]["bottoms"][0]]
            if not (p["type"] in ROUTE_TYPES and fused_away(p["name"])):
                break
            chain.insert(0, p)
        groups.append((L, chain))
    return groups


def _check_net(net, layers, idx):
    """Routing outputs bit for bit from the net's own bottoms; every other chain within its float64 bound.
    Returns the number of routing groups that absorbed other layers, by length."""
    groups = _route_groups(layers, net.LayerFusedAway)
    for head, chain in groups:
        xs = [fetch(net, b, idx).float().cpu().numpy() for b in chain[0]["bottoms"]]
        for L in chain:
            xs = _np_route(L, xs)
        for t, want in zip(head["tops"], xs):
            got = fetch(net, t, idx).float().cpu().numpy()
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (head["name"], t)
    # the other layers: routing heads stand in as inputs of the chains they feed
    rest = []
    for L in layers:
        if L["type"] in ROUTE_TYPES:
            if not net.LayerFusedAway(L["name"]):
                rest.append({"type": "Input", "name": L["name"], "tops": L["tops"], "bottoms": [], "params": {}})
            continue
        rest.append(L)
    chains, _ = rebuild_chains(rest, net.LayerFusedAway, set(net.BlobNames()))
    failures = []
    for ch in chains:
        if ch.head["type"] in ("Input", "Split"):
            continue
        algo = net.LayerConvAlgo(ch.head["name"]) if ch.head["type"] in CONV_TYPES else -1
        ins = {b: fetch(net, b, idx) for b in dict.fromkeys(ch.bottoms)}
        got = {t: fetch(net, t, idx) for t in ch.tops}
        for top, used, _, kind, path in check_chain(ch, ins, got, 2, algo):
            if used > 1.0:
                failures.append(f"{ch.head['name']} -> {top} ({kind}, {path}): bound used {used:.3g}")
    assert not failures, "\n".join(failures[:20])
    return [len(chain) for _, chain in groups if len(chain) > 1]


def _unfused_launches(layers, chain_names):
    """Launches the layers named would issue unfused: Concat one per bottom, ShuffleChannel one (none as a view, group
    1), Slice one per 8 tops."""
    n = 0
    for L in layers:
        if L["name"] not in chain_names:
            continue
        if L["type"] == "Concat":
            n += len(L["bottoms"])
        elif L["type"] == "ShuffleChannel":
            n += 0 if L["params"].get(0, 1) == 1 and not L["params"].get(1, 0) else 1
        else:
            n += -(-len(L["tops"]) // 8)
    return n


@gpu
@pytest.mark.parametrize("key", [f"{n}-{kw.get('width', '')}" for n, kw in NET_CASES])
def test_net_end_to_end(cuda, route_models, route_fuse, key):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m, param, binf, layers = route_models[key]
    batch = 3
    x = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(batch)])
    idx = list(range(batch))
    probs, launches = {}, {}
    for fusion in (True, False):   # the routing pass on / off (route_fuse), every other fusion on
        for graph in (True, False):
            route_fuse(int(fusion))
            net = Net(fusion=True, cuda_graph=graph)
            net.LoadParam(param)
            net.LoadWeights(binf)
            for _ in range(3 if graph else 1):
                net.Forward(x)
            net.Synchronize()
            lengths = _check_net(net, layers, idx)
            if fusion:
                assert lengths, "nothing fused"
                if key.startswith("shufflenet_v2"):
                    assert sorted(lengths) == [2] * 3 + [3] * 13
            else:
                assert not lengths
            probs[fusion, graph] = net.Extract("prob")
            launches[fusion, graph] = net.launches_per_forward
            if fusion and not graph:
                groups = _route_groups(layers, net.LayerFusedAway)
                saved = sum(_unfused_launches(layers, {L["name"] for L in chain}) - _unfused_launches(layers, {h["name"]})
                            for h, chain in groups if len(chain) > 1)
            del net
    ref = probs[False, False]
    for k, v in probs.items():
        assert np.array_equal(v.view(np.uint32), ref.view(np.uint32)), k
    # Concat launches once per bottom: a fused two-bottom Concat -> ShuffleChannel -> Slice saves 3, a Concat ->
    # ShuffleChannel pair 2
    assert launches[False, False] - launches[True, False] == saved
    if key.startswith("shufflenet_v2"):
        assert saved == 13 * 3 + 3 * 2
    assert launches[True, True] == launches[True, False] and launches[False, True] == launches[False, False]


@gpu
@pytest.mark.parametrize("key", ["shufflenet_v2-1.0", "shuffle_tiny-"])
def test_net_batch_independent(cuda, route_models, key):
    from feathercnn_b200.net import Net
    from feathercnn_b200.tools import modelgen
    m, param, binf, _ = route_models[key]
    xs = np.stack([modelgen.synthetic_input(m.shape["data"], i) for i in range(3)])
    net = Net(fusion=True, cuda_graph=True)
    net.LoadParam(param)
    net.LoadWeights(binf)
    net.Forward(xs)
    batched = net.Extract("prob")
    alone = Net(fusion=True, cuda_graph=True)
    alone.LoadParam(param)
    alone.LoadWeights(binf)
    for i in (0, 2):
        alone.Forward(xs[i:i + 1])
        assert np.array_equal(alone.Extract("prob")[0].view(np.uint32), batched[i].view(np.uint32)), i
