"""ShuffleNet-v2 1.0x (modelgen.shufflenet_v2, 224 x 224) through feather::Net at batch 256: images/s with the
Concat -> ShuffleChannel -> Slice chains fused into one routing launch and with that pass off (the route_fuse switch at
0; every other fusion on in both), launches per forward of
each, the share of each kernel class in one eager forward, and the routing kernel alone on the stage-2 / 3 / 4 unit
shapes against a device-to-device copy of the same bytes.

    python scripts/shufflenet_v2_bench.py --out DIR [--batch 256] [--reps 7] [--iters 5]

Device-resident input, CUDA graphs on.  After a warm-up, --reps windows of --iters forwards each, the fused and the
unfused net alternating window by window, timed with CUDA events on the nets' stream; the median window.  The per-kind
shares come from fcuda_profile_collect_kind over two eager forwards of the fused net.  The routing kernel alone runs a
unit's Concat -> ShuffleChannel(2) -> Slice(-233, -233) on two (batch, C/2, H, W) halves, windows alternating with a
contiguous Tensor.copy_ of the same (batch, C, H, W) bytes (cudaMemcpyAsync device-to-device); both move C * H * W * 8
bytes per image.  Writes DIR/shufflenet_v2_bench.json and .md with the card's name and power limit, read in the same
run.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

import mobilenet_v2_bench  # noqa: E402

KINDS = mobilenet_v2_bench.KINDS + ["detection", "channel routing"]
UNITS = [("stage2", 116, 28), ("stage3", 232, 14), ("stage4", 464, 7)]


def route_vs_copy(batch: int, c: int, hw: int, reps: int, iters: int = 50) -> dict:
    """Median ms of the fused routing launch of one unit and of a D2D copy of the same bytes, windows alternating."""
    import torch
    from feathercnn_b200 import booster
    half = c // 2
    srcs = [torch.rand((batch, half, hw, hw), device="cuda") for _ in range(2)]
    outs = [torch.empty_like(srcs[0]) for _ in range(2)]
    a, b = torch.rand((batch, c, hw, hw), device="cuda"), torch.empty((batch, c, hw, hw), device="cuda")
    runs = [lambda: booster.route(srcs, [half, half], group=2, outs=outs), lambda: b.copy_(a)]
    for r in runs:
        for _ in range(5):
            r()
    torch.cuda.synchronize()
    times = [[], []]
    for _ in range(reps):
        for k, r in enumerate(runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                r()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / iters)
    route_ms, copy_ms = (statistics.median(t) for t in times)
    nbytes = 8.0 * batch * c * hw * hw
    return {"shape": [batch, c, hw, hw], "route_ms": route_ms, "copy_ms": copy_ms, "route_over_copy": route_ms / copy_ms,
            "route_TBps": nbytes / (route_ms * 1e-3) / 1e12, "copy_TBps": nbytes / (copy_ms * 1e-3) / 1e12}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5, help="forwards per timed window")
    args = ap.parse_args()
    import numpy as np
    import torch
    from igemm_layer_bench import card
    from feathercnn_b200 import booster
    from feathercnn_b200.tools import modelgen
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    mw = modelgen.shufflenet_v2()
    shape = mw.shape["data"]
    base = np.stack([modelgen.synthetic_input(shape, i) for i in range(min(args.batch, 8))])
    x = torch.from_numpy(np.resize(base, (args.batch,) + tuple(shape))).cuda()
    stream = torch.cuda.current_stream().cuda_stream  # the stream the timing events are recorded on
    with tempfile.TemporaryDirectory() as d:
        param, binf = mw.save(Path(d) / "shufflenet_v2")
        lib = booster.fcuda()
        nets = []
        for route_fuse in (1, 0):  # the routing pass reads the switch when the net first fuses
            lib.fcuda_set_tuning(b"route_fuse", route_fuse)
            nets.append(mobilenet_v2_bench.load(param, binf, True, x, stream))
            nets[-1].FuseNow()
        lib.fcuda_set_tuning(b"route_fuse", 1)
        fused, unfused = nets
    fused_ms, unfused_ms = mobilenet_v2_bench.alternated([fused, unfused], args.reps, args.iters)
    same = bool(np.array_equal(fused.Extract("prob"), unfused.Extract("prob")))
    routes = [line.split()[1] for line in mw.lines if line.split()[0] in ("Concat", "ShuffleChannel", "Slice")]
    mobilenet_v2_bench.KINDS = KINDS  # kind_shares reads the module's list: add detection and channel routing
    shares = mobilenet_v2_bench.kind_shares(fused)
    units = {name: route_vs_copy(args.batch, c, hw, args.reps) for name, c, hw in UNITS}
    info = card()
    res = {"card": info, "model": "shufflenet_v2", "width": 1.0, "size": shape[1], "batch": args.batch,
           "cuda_graph": True, "fused_ms": fused_ms, "unfused_ms": unfused_ms,
           "fused_images_per_s": args.batch / (fused_ms * 1e-3), "unfused_images_per_s": args.batch / (unfused_ms * 1e-3),
           "outputs_bit_identical": same,
           "routing_layers_fused_away": int(sum(fused.LayerFusedAway(n) == 1 for n in routes)), "routing_layers": len(routes),
           "launches_per_forward": {"fused": fused.launches_per_forward, "unfused": unfused.launches_per_forward},
           "kind_shares_fused_eager": shares, "route_vs_d2d_copy": units}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "shufflenet_v2_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; ShuffleNet-v2 1.0x {shape[1]}x{shape[2]}, batch "
          f"{args.batch}, device-resident input, CUDA graph", "",
          "| fusion | ms / forward | images/s | launches / forward |", "|---|---|---|---|",
          f"| on ({res['routing_layers_fused_away']} of {len(routes)} routing layers absorbed) | {fused_ms:.3f} | "
          f"{res['fused_images_per_s']:.0f} | {res['launches_per_forward']['fused']} |",
          f"| routing pass off | {unfused_ms:.3f} | {res['unfused_images_per_s']:.0f} | {res['launches_per_forward']['unfused']} |", "",
          f"Fused and unfused outputs bit-identical: {same}", "",
          "Kernel classes, fusion on, eager forward (CUDA events around every launch):", "",
          "| kind | ms / forward | share | launches / forward |", "|---|---|---|---|"]
    md += [f"| {r['name']} | {r['ms_per_forward']:.3f} | {r['share']:.1%} | {r['launches_per_forward']:.0f} |" for r in shares]
    md += ["", "Routing kernel alone (Concat -> ShuffleChannel 2 -> Slice of one unit) vs a D2D copy of the same bytes:", "",
           "| unit | (N, C, H, W) | route ms | copy ms | route / copy | route TB/s | copy TB/s |", "|---|---|---|---|---|---|---|"]
    md += [f"| {k} | {tuple(u['shape'])} | {u['route_ms']:.4f} | {u['copy_ms']:.4f} | {u['route_over_copy']:.3f} | "
           f"{u['route_TBps']:.2f} | {u['copy_TBps']:.2f} |" for k, u in units.items()]
    (out / "shufflenet_v2_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))
    print(json.dumps({k: res[k] for k in ("fused_images_per_s", "unfused_images_per_s", "launches_per_forward")}))


if __name__ == "__main__":
    main()
