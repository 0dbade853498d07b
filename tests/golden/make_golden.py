"""Generates the committed golden fixtures from the UNMODIFIED reference build (oracle/_ref, compiled from
/root/reference by oracle/Makefile).  Run in the authoring container:  python tests/golden/make_golden.py

The reference ships no golden vectors of its own (SURVEY.md §4), so these are outputs of the reference itself:
  conv_cases.npz   ConvBooster::Forward outputs for small layers covering every SelectAlgo branch
  mini_net.npz     every blob of feather::Net::Forward on the "mini" model (all layer types), seed-fixed input
  reference_build_conv.npz   ConvBooster::Forward of the layers of tests/test_gpu_conv.py::REF_CASES (inputs from that
                   test's seeded generator): a fixed sample of 4096 output values per layer plus max|y| of the whole output
                   (python tests/golden/make_golden.py reference_build_conv)
Inputs and weights are stored too, so the fixtures do not depend on NumPy's RNG staying stable.
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from feathercnn_b200.tools import modelgen  # noqa: E402
from oracle import oracle as O  # noqa: E402

# name, oc, ic, h, w, k, stride, pad, group, bias, relu
CONV_CASES = [
    ("wino_16x16_12", 16, 16, 12, 12, 3, 1, 1, 1, True, False),
    ("wino_ragged_relu", 8, 12, 13, 10, 3, 1, 1, 1, True, True),
    ("im2col_1x1", 12, 16, 9, 9, 1, 1, 0, 1, False, False),
    ("im2col_7x7_s2", 8, 3, 20, 20, 7, 2, 3, 1, True, False),
    ("im2col_small_hw", 8, 8, 7, 7, 3, 1, 1, 1, True, True),
    ("im2col_oc_not4", 6, 8, 12, 12, 3, 1, 1, 1, True, False),
    ("dw_s1", 8, 8, 10, 10, 3, 1, 1, 8, False, False),
    ("dw_s2_relu", 8, 8, 11, 11, 3, 2, 1, 8, False, True),
    ("dw_global", 8, 8, 5, 5, 5, 1, 0, 8, False, False),
]


def main():
    out = Path(__file__).resolve().parent
    O.build(ref=True)
    ref = O.Reference()
    rng = np.random.default_rng(20260922)
    conv = {}
    for name, oc, ic, h, w, k, s, pad, group, bias, relu in CONV_CASES:
        p = O.ConvParam.make(oc, ic, h, w, k, stride=s, pad=pad, group=group, bias=bias, relu=relu)
        x = rng.uniform(-0.5, 0.5, (ic, h, w)).astype(np.float32)
        fan_in = (ic if group == 1 else 1) * k * k
        wt = (rng.standard_normal(p.weight_shape) * np.sqrt(2.0 / fan_in)).astype(np.float32)
        b = rng.uniform(-0.1, 0.1, p.output_channels).astype(np.float32)
        y = ref.conv(p, x, wt, b if bias else None)
        conv[name + "/x"], conv[name + "/w"], conv[name + "/b"], conv[name + "/y"] = x, wt, b, y
        conv[name + "/geom"] = np.array([oc, ic, h, w, k, s, pad, group, int(bias), int(relu)], np.int32)
    np.savez_compressed(out / "conv_cases.npz", **conv)

    m = modelgen.mini(seed=0, size=20, ch=8)
    param, binf = m.save(out / "mini")
    x = modelgen.synthetic_input(m.shape["data"], 0)
    net = O.ReferenceNet(param, binf)
    net.forward(x)
    blobs = {"input": x}
    for b in sorted(m.blobs):
        blobs["blob/" + b] = net.extract(b)
    np.savez_compressed(out / "mini_net.npz", **blobs)
    print("wrote", out / "conv_cases.npz", out / "mini_net.npz", out / "mini.param", out / "mini.bin")


def reference_build_conv():
    sys.path.insert(0, str(ROOT / "tests"))
    import test_gpu_conv as T
    out = Path(__file__).resolve().parent
    O.build(ref=True)
    ref = O.Reference()
    gold = {}
    for case in T.REF_CASES:
        p, x, wt, b = T._data(O, case, 1, seed=7)
        y = ref.conv(p, x[0], wt, b).ravel()
        idx = np.sort(np.random.default_rng(1234).choice(y.size, min(4096, y.size), replace=False)).astype(np.int32)
        gold[case[0] + "/idx"], gold[case[0] + "/y"] = idx, y[idx].astype(np.float32)
        gold[case[0] + "/absmax"] = np.float64(np.abs(y).max())
    np.savez_compressed(out / "reference_build_conv.npz", **gold)
    print("wrote", out / "reference_build_conv.npz")


if __name__ == "__main__":
    reference_build_conv() if sys.argv[1:] == ["reference_build_conv"] else main()
