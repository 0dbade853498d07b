"""Per-layer timing of the TensorGEMM, for every layer of VGG-16 (b64) and ResNet-50 (b128) that
fcuda_conv_select_algo_tuned sends to Winograd, and for VGG-16's three InnerProduct layers at b64.

    python scripts/gemm_layer_bench.py --out DIR [--reps 5] [--iters 20]

For each layer, over --reps repetitions (median and every value): the CUDA-event time of the whole layer per forward,
the time of its TensorGEMM launches alone (the per-launch profile hooks, a separate pass), the issued tensor-pipe rate of
the GEMM (TF32 MMA FLOPs of the launches: M, N, K as launched, x3 in the split modes) and its fraction of the H100 SXM
data-sheet dense TF32 rate.  Two builds are compared by running the script on each.  Writes DIR/gemm_layer_bench.json
with the card's name and power limit.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import ctypes
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

DATASHEET_TF32_DENSE = 495e12  # H100 SXM data sheet, dense TF32 (not a measured figure)
BATCH = {"vgg16": 64, "resnet50": 128}


def winograd_layers(model: str):
    """(name, ConvParam fields, algo, fused pool) of every Convolution layer the tuned selector sends to Winograd, and
    (name, in, out) of every InnerProduct layer."""
    from feathercnn_b200 import booster
    from feathercnn_b200.tools import modelgen
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    m = getattr(modelgen, model)()
    convs, fcs = [], []
    lines = [ln.split() for ln in m.lines]
    for i, ln in enumerate(lines):
        ltype, name, nb, nt = ln[0], ln[1], int(ln[2]), int(ln[3])
        bottoms, tops = ln[4:4 + nb], ln[4 + nb:4 + nb + nt]
        kv = dict(s.split("=") for s in ln[4 + nb + nt:])
        if ltype == "InnerProduct":
            n_in = 1
            for d in m.shape[bottoms[0]]:
                n_in *= d
            fcs.append((name, n_in, int(kv["0"])))
            continue
        if ltype != "Convolution":
            continue
        oc, k, s, pad = int(kv["0"]), int(kv["1"]), int(kv.get("3", 1)), int(kv.get("4", 0))
        group = int(kv.get("7", 1))
        ic, ih, iw = m.shape[bottoms[0]]
        p = booster.ConvParam.make(oc, ic, ih, iw, k, stride=s, pad=pad, group=group, relu=True)
        a = ctypes.c_int(-1)
        if lib.fcuda_conv_select_algo_tuned(ctypes.byref(p), ctypes.byref(a)) != 0 or \
                a.value not in (booster.WINOGRADF63, booster.WINOGRADF23):
            continue
        pool = False  # a following ReLU + 2x2 / stride-2 max pooling is fused into the conv by feather::Net
        rest = lines[i + 1:i + 3]
        if len(rest) == 2 and rest[0][0] == "ReLU" and rest[1][0] == "Pooling":
            pk = dict(s.split("=") for s in rest[1][6:])
            pool = pk.get("0") == "0" and pk.get("1") == "2" and pk.get("2") == "2" and pk.get("4", "0") == "0"
            pool = pool and lib.fcuda_conv_can_pool(ctypes.byref(p), a.value) == 1
        convs.append((name, (oc, ic, ih, iw, k, s, pad, group), a.value, pool))
    return convs, fcs


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plimit, clk = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": plimit, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001 — the timing stays valid, the label says what is missing
        return {"name": "unknown", "power_limit": "unknown", "error": str(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20, help="forwards per timed repetition")
    ap.add_argument("--models", default="vgg16,resnet50")
    args = ap.parse_args()

    import torch
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    if not torch.cuda.is_available():
        raise SystemExit("gemm_layer_bench needs a CUDA device")
    torch.cuda.set_device(0)
    lib = fcuda()
    stream = booster._stream
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731

    def prepare_conv(pfields, algo, n, pool):
        oc, ic, ih, iw, k, s, pad, group = pfields
        p = booster.ConvParam.make(oc, ic, ih, iw, k, stride=s, pad=pad, group=group, relu=True)
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.empty((n, ic, ih, iw), device="cuda").uniform_(-1, 1, generator=g)
        wt = torch.empty((oc, ic // group, k, k), device="cuda").normal_(0, 0.05, generator=g)
        b = torch.empty(oc, device="cuda").uniform_(-0.1, 0.1, generator=g)
        cb = booster.ConvBooster()
        cb.ForceSelectAlgo(algo)
        scratch_n, packed_n = cb.GetBufferSize(p, n)
        packed = torch.empty(max(packed_n, 1), device="cuda")
        scratch = torch.empty(max(scratch_n, 1), device="cuda")
        cb.Init(p, packed, wt)
        oh, ow = ((p.output_h + 1) // 2, (p.output_w + 1) // 2) if pool else (p.output_h, p.output_w)
        out = torch.empty((n, oc, oh, ow), device="cuda")

        def launch():
            if pool:
                rc = lib.fcuda_conv_forward_pool(ctypes.byref(p), algo, ptr(out), ptr(x), ptr(packed), ptr(scratch), ptr(b), n,
                                                 stream())
            else:
                rc = lib.fcuda_conv_forward(ctypes.byref(p), algo, ptr(out), ptr(x), ptr(packed), ptr(scratch), ptr(b), n,
                                            stream())
            assert rc == 0, rc
        return launch, out

    def prepare_ip(n_in, n_out, n):
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.empty((n, n_in), device="cuda").uniform_(-1, 1, generator=g)
        w = torch.empty((n_out, n_in), device="cuda").normal_(0, (2.0 / n_in) ** 0.5, generator=g)
        b = torch.empty(n_out, device="cuda").uniform_(-0.1, 0.1, generator=g)
        s, k = ctypes.c_size_t(0), ctypes.c_size_t(0)
        assert lib.fcuda_inner_product_get_buffer_size(n_in, n_out, n, ctypes.byref(s), ctypes.byref(k)) == 0
        packed = torch.empty(max(k.value, 1), device="cuda")
        scratch = torch.empty(max(s.value, 1), device="cuda")
        assert lib.fcuda_inner_product_init(n_in, n_out, ptr(packed), ptr(w), stream()) == 0
        out = torch.empty((n, n_out), device="cuda")

        def launch():
            rc = lib.fcuda_inner_product_forward(n_in, n_out, ptr(out), ptr(x), ptr(packed), ptr(b), ptr(scratch), 1, n,
                                                 stream())
            assert rc == 0, rc
        return launch, out

    def time_ms(launch, iters):
        launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    def gemm_ms(launch, iters):
        """TensorGEMM device time and issued MMA FLOPs per forward, from the per-launch profile events"""
        launch()
        torch.cuda.synchronize()
        lib.fcuda_profile_tensor_gemm(1)
        for _ in range(iters):
            launch()
        ms, af, mf, ab = ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_double()
        nl = ctypes.c_longlong()
        assert lib.fcuda_profile_collect_kind(0, ctypes.byref(ms), ctypes.byref(af), ctypes.byref(mf), ctypes.byref(ab),
                                              ctypes.byref(nl)) == 0
        lib.fcuda_profile_tensor_gemm(0)
        assert nl.value > 0, "no TensorGEMM launch in this layer"
        return ms.value / iters, mf.value / iters, nl.value // iters

    result = {"card": card(), "reps": args.reps, "iters": args.iters,
              "datasheet_tf32_dense_tflops": DATASHEET_TF32_DENSE / 1e12,
              "precision": {0: "tf32x3", 1: "tf32", 2: "fp32split"}[lib.fcuda_get_precision()], "layers": []}
    for model in args.models.split(","):
        n = BATCH[model]
        convs, fcs = winograd_layers(model)
        jobs = {}
        for name, pf, algo, pool in convs:  # one measurement per distinct shape
            jobs.setdefault(("conv", pf, algo, pool), []).append(name)
        if model == "vgg16":
            for name, n_in, n_out in fcs:
                jobs.setdefault(("ip", n_in, n_out), []).append(name)
        for key, names in jobs.items():
            if key[0] == "conv":
                launch, out = prepare_conv(key[1], key[2], n, key[3])
                desc = {"kind": booster.ALGO_NAMES[key[2]] if hasattr(booster, "ALGO_NAMES") else key[2],
                        "oc_ic_h_w_k_s_pad_group": list(key[1]), "fused_pool": key[3]}
            else:
                launch, out = prepare_ip(key[1], key[2], n)
                desc = {"kind": "InnerProduct", "in": key[1], "out": key[2]}
            layer_t, gemm_t = [], []
            for _ in range(args.reps):
                layer_t.append(time_ms(launch, args.iters))
                ms, issued, launches = gemm_ms(launch, args.iters)
                gemm_t.append(ms)
            layer_med, gemm_med = statistics.median(layer_t), statistics.median(gemm_t)
            rec = {"model": model, "layer": ",".join(names), "count": len(names), "batch": n, **desc,
                   "gemm_launches_per_forward": launches, "issued_mma_gflop": issued / 1e9,
                   "layer_ms_median": layer_med, "gemm_ms_median": gemm_med, "layer_ms": layer_t, "gemm_ms": gemm_t,
                   "issued_tf32_tflops": issued / gemm_med / 1e9,
                   "issued_fraction_of_datasheet_tf32": issued / gemm_med / 1e-3 / DATASHEET_TF32_DENSE}
            result["layers"].append(rec)
            print(json.dumps({k2: rec[k2] for k2 in ("model", "layer", "layer_ms_median", "gemm_ms_median",
                                                      "issued_tf32_tflops")}), flush=True)
            del launch, out
            torch.cuda.empty_cache()
    for model in BATCH:
        rows = [r for r in result["layers"] if r["model"] == model]
        if rows:
            result[f"{model}_gemm_total_ms"] = sum(r["gemm_ms_median"] * r["count"] for r in rows)
            result[f"{model}_layer_total_ms"] = sum(r["layer_ms_median"] * r["count"] for r in rows)
    out_dir = Path(args.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    (out_dir / "gemm_layer_bench.json").write_text(json.dumps(result, indent=1))
    print(json.dumps({k: v for k, v in result.items() if k != "layers"}))


if __name__ == "__main__":
    main()
