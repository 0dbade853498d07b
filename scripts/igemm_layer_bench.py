"""Per-layer timing of the implicit-GEMM convolution (SGECONV), switch --switch at 0 against 1: igemm_presplit (default:
the pre-split halo kernel against the per-tap split) or igemm_halo (the halo kernel against the gathering kernel), for
every layer of the benchmark nets that fcuda_conv_select_algo_tuned sends to SGECONV, at the nets' benchmark batch sizes.

    python scripts/igemm_layer_bench.py --out DIR [--reps 5] [--iters 20] [--switch igemm_presplit]

For each layer: CUDA-event time per launch of both kernels (alternated over --reps repetitions; median and every value),
the algorithmic rate (direct-convolution FLOPs), the issued tensor-pipe rate (padded patch pixels, N tiles and the three
MMAs per product of the split modes) and that rate's fraction of the H100 SXM data-sheet dense BF16 rate, and for the
halo kernels the bytes one launch moves from L2 to the SMs (filter ring stages + input boxes, from the geometry).  The Winograd
F(6,3) time of the same shape is listed for reference only.  Writes DIR/igemm_layer_bench.json with the card's name and
power limit.  Needs a CUDA device."""
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

DATASHEET_BF16_DENSE = 989e12  # H100 SXM data sheet, dense BF16 (not a measured figure)
BATCH = {"vgg16": 64, "resnet50": 128, "mobilenet_v1": 256}


def sgeconv_layers(model: str):
    """(name, ConvParam fields, fused pool) of every Convolution layer the tuned selector sends to SGECONV."""
    from feathercnn_b200 import booster
    from feathercnn_b200.tools import modelgen
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    m = getattr(modelgen, model)()
    out = []
    lines = [ln.split() for ln in m.lines]
    for i, ln in enumerate(lines):
        ltype, name, nb, nt = ln[0], ln[1], int(ln[2]), int(ln[3])
        bottoms, tops = ln[4:4 + nb], ln[4 + nb:4 + nb + nt]
        if ltype not in ("Convolution", "ConvolutionDepthWise"):
            continue
        kv = dict(s.split("=") for s in ln[4 + nb + nt:])
        oc, k, s, pad = int(kv["0"]), int(kv["1"]), int(kv.get("3", 1)), int(kv.get("4", 0))
        group = int(kv.get("7", 1))
        ic, ih, iw = m.shape[bottoms[0]]
        p = booster.ConvParam.make(oc, ic, ih, iw, k, stride=s, pad=pad, group=group, relu=True)
        a = ctypes.c_int(-1)
        if lib.fcuda_conv_select_algo_tuned(ctypes.byref(p), ctypes.byref(a)) != 0 or a.value != booster.SGECONV:
            continue
        # a following ReLU + 2x2 / stride-2 max pooling is fused into the conv by feather::Net
        pool = False
        rest = [x for x in lines[i + 1:i + 3]]
        if len(rest) == 2 and rest[0][0] == "ReLU" and rest[1][0] == "Pooling":
            pk = dict(s.split("=") for s in rest[1][6:])
            pool = pk.get("0") == "0" and pk.get("1") == "2" and pk.get("2") == "2" and pk.get("4", "0") == "0"
            pool = pool and lib.fcuda_conv_can_pool(ctypes.byref(p), booster.SGECONV) == 1
        out.append((name, (oc, ic, ih, iw, k, s, pad, group), pool))
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plimit = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": plimit}
    except Exception as e:  # noqa: BLE001 — the timing stays valid, the label says what is missing
        return {"name": "unknown", "power_limit": "unknown", "error": str(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20, help="launches per timed repetition")
    ap.add_argument("--models", default="vgg16,resnet50,mobilenet_v1")
    ap.add_argument("--switch", default="igemm_presplit", choices=["igemm_presplit", "igemm_halo"])
    args = ap.parse_args()

    import torch
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    if not torch.cuda.is_available():
        raise SystemExit("igemm_layer_bench needs a CUDA device")
    torch.cuda.set_device(0)
    lib = fcuda()
    switch = args.switch.encode()
    saved = lib.fcuda_get_tuning(switch)
    stream = booster._stream

    def prepare(pfields, algo, n, pool):
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
        oh, ow = (p.output_h + 1) // 2 if pool else p.output_h, (p.output_w + 1) // 2 if pool else p.output_w
        out = torch.empty((n, oc, oh, ow), device="cuda")
        ptr = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731

        def launch():
            if pool:
                rc = lib.fcuda_conv_forward_pool(ctypes.byref(p), algo, ptr(out), ptr(x), ptr(packed), ptr(scratch), ptr(b), n,
                                                 stream())
            else:
                rc = lib.fcuda_conv_forward(ctypes.byref(p), algo, ptr(out), ptr(x), ptr(packed), ptr(scratch), ptr(b), n,
                                            stream())
            assert rc == 0, rc
        return p, launch, out

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

    result = {"card": card(), "switch": args.switch, "reps": args.reps, "iters": args.iters,
              "datasheet_bf16_dense_tflops": DATASHEET_BF16_DENSE / 1e12,
              "precision": {0: "tf32x3", 1: "tf32", 2: "fp32split"}[lib.fcuda_get_precision()], "layers": []}
    try:
        for model in args.models.split(","):
            n = BATCH[model]
            layers = {}
            for name, pf, pool in sgeconv_layers(model):  # one measurement per distinct shape
                layers.setdefault((pf, pool), []).append(name)
            for (pf, pool), names in layers.items():
                name = ",".join(names)
                p, launch, out = prepare(pf, booster.SGECONV, n, pool)
                geom = (ctypes.c_int * 4)()
                halo = lib.fcuda_igemm_halo_tile(ctypes.byref(p), geom) == 1
                pgeom = (ctypes.c_int * 4)()
                presplit = lib.fcuda_igemm_presplit_tile(ctypes.byref(p), pgeom) == 1
                t = {0: [], 1: []}
                outs = {}
                for _ in range(args.reps):
                    for sw in (0, 1):
                        lib.fcuda_set_tuning(switch, sw)
                        t[sw].append(time_ms(launch, args.iters))
                        outs[sw] = out.clone()
                identical = bool(torch.equal(outs[0], outs[1]))
                del outs
                oc, ic, ih, iw, k, s, pad, group = pf
                algo_flops = 2.0 * n * oc * p.output_h * p.output_w * (ic // group) * k * k
                bn = 32 if oc // group <= 32 else 64 if oc // group <= 64 else 128
                ocp = -(-(oc // group) // bn) * bn * group
                kpad = -(-((ic // group) * k * k) // 32) * 32
                if halo:
                    r, c = geom[0], geom[1]
                    pix = n * (-(-p.output_h // r) * r) * (-(-p.output_w // c) * c)
                elif pool:
                    pix = n * (-(-p.output_h // 2) * 2) * (-(-p.output_w // 64) * 64)
                else:
                    pix = -(-(n * p.output_h * p.output_w) // 128) * 128
                mult = 3 if result["precision"] != "tf32" else 1

                def l2_to_sm_bytes(g):
                    """Filter ring stages + input boxes one launch fetches: per tile, every k-block's filter stage and
                    one box of 32 channels x box rows x box columns (fp32) per channel block."""
                    r, c, rb, cb = g[0], g[1], g[2], g[3]
                    tiles = n * -(-p.output_h // r) * -(-p.output_w // c) * (ocp // bn)
                    stage = bn * 32 * (2 if result["precision"] == "fp32split" else 4) * (1 if result["precision"] == "tf32" else 2)
                    return tiles * ((kpad // 32) * stage + (ic // group // 32) * 32 * rb * cb * 4)
                issued_new = 2.0 * pix * ocp * kpad * mult
                old_ms, new_ms = statistics.median(t[0]), statistics.median(t[1])
                wino_ms = None  # Winograd F(6,3) on the same shape (3x3, stride 1), for reference only
                if k == 3 and s == 1 and group == 1:
                    del launch, out
                    try:
                        _, wlaunch, _ = prepare(pf, booster.WINOGRADF63, n, pool)
                        wino_ms = statistics.median([time_ms(wlaunch, args.iters) for _ in range(args.reps)])
                        del wlaunch
                    except booster.FcudaError as e:  # e.g. IC = 3: Winograd does not take the layer
                        wino_ms = f"n/a ({e})"
                rec = {"model": model, "layer": name, "count": len(names), "batch": n, "oc": oc, "ic": ic, "h": ih, "w": iw, "k": k, "stride": s,
                       "pad": pad, "group": group, "fused_pool": pool, "halo_eligible": halo,
                       "halo_patch_rows_cols": [geom[0], geom[1]] if halo else None,
                       "old_ms_median": old_ms, "new_ms_median": new_ms, "old_ms": t[0], "new_ms": t[1],
                       "speedup": old_ms / new_ms, "bit_identical": identical,
                       "algo_tflops_old": algo_flops / old_ms / 1e9, "algo_tflops_new": algo_flops / new_ms / 1e9,
                       "issued_tflops_new": issued_new / new_ms / 1e9,
                       "issued_fraction_of_datasheet_bf16_new": issued_new / new_ms / 1e-3 / DATASHEET_BF16_DENSE,
                       "winograd_f63_ms_reference_only": wino_ms,
                       "presplit_tile_rows_cols_box": list(pgeom) if presplit else None,
                       "l2_to_sm_bytes_halo": l2_to_sm_bytes(geom) if halo else None,
                       "l2_to_sm_bytes_presplit": l2_to_sm_bytes(pgeom) if presplit else None}
                result["layers"].append(rec)
                print(json.dumps({k2: rec[k2] for k2 in ("model", "layer", "old_ms_median", "new_ms_median", "speedup",
                                                          "bit_identical", "algo_tflops_new", "issued_tflops_new",
                                                          "l2_to_sm_bytes_presplit")}),
                      flush=True)
                torch.cuda.empty_cache()
    finally:
        lib.fcuda_set_tuning(switch, saved)
    for model in BATCH:
        rows = [r for r in result["layers"] if r["model"] == model]
        if rows:
            result[f"{model}_sgeconv_total_old_ms"] = sum(r["old_ms_median"] * r["count"] for r in rows)
            result[f"{model}_sgeconv_total_new_ms"] = sum(r["new_ms_median"] * r["count"] for r in rows)
    out_dir = Path(args.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    (out_dir / "igemm_layer_bench.json").write_text(json.dumps(result, indent=1))
    print(json.dumps({k: v for k, v in result.items() if k != "layers"}))


if __name__ == "__main__":
    main()
