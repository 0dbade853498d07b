"""MobileNet-YOLO through feather::Net and the YOLO head alone.

    python scripts/yolo_bench.py --out DIR [--batch 64] [--reps 7] [--iters 10]

Models (modelgen.mobilenet_yolov2 and mobilenetv2_yolov3, 416 x 416, fusion and CUDA graphs on, device-resident input):
images/s at --batch, latency at batch 1, launches per forward, and the share of each kernel class in an eager forward
(kind 9 is the detection head: YOLO decode, select, mask, sweep).  The head alone (fcuda_yolo_detection_forward, 80
classes, 3 anchors per scale, nms_top_k = keep_top_k = 1024) at 416 (13 / 26 / 52: 10647 slots) and 608 (19 / 38 / 76:
22743 slots), with hundreds of candidates and with more than 1024, at batch 1 and --batch: the whole head timed with
CUDA events (--reps windows of --head-iters calls, the median), and each kernel from a torch.profiler run of its own over
--head-iters calls.
Writes DIR/yolo_bench.json and .md with the card's name and power limit, read in the same run.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import ctypes
import json
import statistics
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from mobilenet_v2_bench import load  # noqa: E402
from ssd_bench import kind_shares, timed  # noqa: E402

COCO = [10, 13, 16, 30, 33, 23, 30, 61, 62, 45, 59, 119, 116, 90, 156, 198, 373, 326]
KERNELS = ["yolo_decode_kernel", "yolo_select_kernel", "yolo_mask_kernel", "yolo_sweep_kernel"]


class Head:
    """fcuda_yolo_detection_forward on preallocated buffers: one call per __call__, no host work beyond the launch."""

    def __init__(self, size: int, batch: int, obj: float):
        import numpy as np
        import torch
        from feathercnn_b200 import booster
        grids = [(size // s, size // s) for s in (32, 16, 8)]
        self.p = booster.yolo_param(3, 80, 3, grids, COCO, [6, 7, 8, 3, 4, 5, 0, 1, 2], [32.0, 16.0, 8.0], 0.01, 0.45)
        rng = np.random.default_rng(size + batch)
        self.xs = []
        for g, _ in grids:
            x = rng.standard_normal((batch, 3, 85, g, g)).astype(np.float32) * 2
            x[:, :, 4] += obj
            self.xs.append(torch.from_numpy(x.reshape(batch, 255, g, g)).cuda())
        self.arr = (ctypes.c_void_p * 3)(*[x.data_ptr() for x in self.xs])
        lib = booster.fcuda()
        ws = ctypes.c_size_t()
        booster._check("ws", lib.fcuda_yolo_detection_workspace_size(ctypes.byref(self.p), batch, ctypes.byref(ws)))
        self.ws = torch.empty(ws.value, device="cuda")
        self.out = torch.empty((batch, 1024, 6), device="cuda")
        self.batch = batch
        self.slots = sum(3 * g * g for g, _ in grids)
        self.lib = lib
        self.stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        scores = booster.yolo_decode(self.xs, self.p)[0]
        self.candidates = int((scores >= 0.01).sum().item()) / batch

    def __call__(self):
        rc = self.lib.fcuda_yolo_detection_forward(ctypes.c_void_p(self.out.data_ptr()), self.arr, ctypes.byref(self.p),
                                                   ctypes.c_void_p(self.ws.data_ptr()), self.batch, self.stream)
        assert rc == 0, rc


def time_calls(fn, reps: int, iters: int) -> float:
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return statistics.median(times)


def kernel_times(fn, iters: int) -> dict:
    """Mean device ms per call of each head kernel, from torch.profiler (CUDA activities)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                out[k] += ev.device_time_total / 1000.0 / iters
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forwards per timed window")
    ap.add_argument("--head-iters", type=int, default=200, help="head-alone calls per timed window and per profile")
    args = ap.parse_args()
    import numpy as np
    import torch
    from igemm_layer_bench import card
    from feathercnn_b200.tools import modelgen
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    models = {}
    for name in ("mobilenetv2_yolov3", "mobilenet_yolov2"):
        mw = modelgen.ZOO[name]()
        shape = mw.shape["data"]
        base = np.stack([modelgen.synthetic_input(shape, i) for i in range(min(args.batch, 8))])
        xb = torch.from_numpy(np.resize(base, (args.batch,) + tuple(shape))).cuda()
        x1 = xb[:1].contiguous()
        with tempfile.TemporaryDirectory() as d:
            param, binf = mw.save(Path(d) / name)
            net_b = load(param, binf, True, xb, stream)
            net_1 = load(param, binf, True, x1, stream)
        ms_b = timed(net_b, args.reps, args.iters)
        ms_1 = timed(net_1, args.reps, args.iters)
        shares = kind_shares(net_b)
        models[name] = {"size": shape[1], "batch": args.batch, "ms_per_forward": ms_b,
                        "images_per_s": args.batch / (ms_b * 1e-3), "batch1_latency_ms": ms_1,
                        "launches_per_forward": net_b.launches_per_forward,
                        "head_kind9_share_eager": next((r["share"] for r in shares if r["kind"] == 9), 0.0),
                        "kind_shares_eager": shares}
        del net_b, net_1
    heads = []
    for size in (416, 608):
        for label, obj in (("hundreds", -8.0), ("many", 0.0)):
            for b in (1, args.batch):
                h = Head(size, b, obj)
                row = {"size": size, "slots": h.slots, "candidates_per_image": h.candidates, "label": label,
                       "batch": b, "ms": time_calls(h, args.reps, args.head_iters)}
                row.update(kernel_times(h, args.head_iters))
                heads.append(row)
                del h
    info = card()
    res = {"card": info, "fusion": True, "cuda_graph": True, "models": models, "head_alone": heads}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "yolo_bench.json").write_text(json.dumps(res, indent=1))
    md = [f"{info['name']}, power limit {info['power_limit']}; 416 x 416, fusion + CUDA graph, device-resident input", ""]
    for name, r in models.items():
        md.append(f"- {name}: batch {args.batch} {r['ms_per_forward']:.3f} ms / forward, {r['images_per_s']:.0f} images/s, "
                  f"{r['launches_per_forward']} launches / forward; batch 1 latency {r['batch1_latency_ms']:.3f} ms; "
                  f"detection head (kind 9) {r['head_kind9_share_eager']:.1%} of an eager forward")
    md += ["", "Head alone (80 classes, nms_top_k = keep_top_k = 1024), ms per call; kernels from torch.profiler:", "",
           "| slots | candidates / image | batch | head | decode | select | mask | sweep |",
           "|---|---|---|---|---|---|---|---|"]
    md += [f"| {r['slots']} ({r['size']}) | {r['candidates_per_image']:.0f} | {r['batch']} | {r['ms']:.4f} | "
           + " | ".join(f"{r[k]:.4f}" for k in KERNELS) + " |" for r in heads]
    (out / "yolo_bench.md").write_text("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
