"""The pre-split halo kernel (switch igemm_presplit) as compiled: registered switch, pipelined wgmma, and a main loop that
loads its A fragments with ldmatrix and no longer splits fp32 values (the split runs once per input box, outside it).
Checked on the built library without a GPU.

Run as a script, prints the instruction mix of the main loop of every BF16x3 halo kernel, old and new."""
import collections
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
NEW = r"conv_igemm_presplit_kernelILi(32|64|128)EE"
OLD = r"conv_igemm_halo_kernelILi(32|64|128)ELi3EE"


def _functions():
    """{mangled name: [(address, opcode, branch target or None)]} of libfcuda.so."""
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    so = ROOT / "feathercnn_b200" / "lib" / "libfcuda.so"
    sass = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True, check=True).stdout
    funcs: dict[str, list] = {}
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)?)(.*)", line)
        if m and cur is not None:
            op = m.group(2)
            op = op if op.startswith("WARPGROUP") else op.split(".")[0]
            t = re.match(r"\s+0x([0-9a-f]+)", m.group(3)) if op == "BRA" else None
            cur.append((int(m.group(1), 16), op, int(t.group(1), 16) if t else None))
    return funcs


def main_loop(instrs):
    """Opcode counts of the innermost loop (a backward branch and its target) that issues wgmma."""
    best = None
    for addr, op, tgt in instrs:
        if op == "BRA" and tgt is not None and tgt <= addr:
            body = [o for a, o, _ in instrs if tgt <= a <= addr]
            if "HGMMA" in body and (best is None or len(body) < sum(best.values())):
                best = collections.Counter(body)
    return best


def _kernels(funcs, pattern):
    hit = sorted(k for k in funcs if re.search(pattern, k))
    assert hit, pattern
    return hit


def test_presplit_switch_is_registered():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    assert lib.fcuda_get_tuning(b"igemm_presplit") == 1
    assert lib.fcuda_set_tuning(b"igemm_presplit", 2) == -200
    assert lib.fcuda_set_tuning(b"igemm_presplit", -1) == -200


def test_presplit_wgmma_are_not_serialised():
    funcs = _functions()
    kernels = _kernels(funcs, NEW)
    assert len(kernels) == 3, kernels
    for k in kernels:
        c = collections.Counter(op for _, op, _ in funcs[k])
        hgmma, depbar = c["HGMMA"], c["WARPGROUP.DEPBAR"]
        assert hgmma >= 6 and hgmma % 6 == 0, (k, dict(c))  # 3 MMAs x 2 k-steps per commit group
        assert 1 <= depbar <= hgmma // 6 + 1 and depbar < hgmma, (k, hgmma, depbar)


def test_presplit_main_loop_loads_fragments_and_does_not_split():
    funcs = _functions()
    for k in _kernels(funcs, NEW):
        loop = main_loop(funcs[k])
        assert loop is not None, k
        assert loop["HGMMA"] >= 6 and loop["LDSM"] >= 4, (k, dict(loop))
        assert loop["F2FP"] == 0 and loop["FADD"] == 0, (k, dict(loop))
        # the split still exists, once per box, outside the main loop
        assert sum(op == "F2FP" for _, op, _ in funcs[k]) > 0, k
    for k in _kernels(funcs, OLD):  # the per-tap split of the halo kernel, for contrast
        assert main_loop(funcs[k])["F2FP"] > 0, k


if __name__ == "__main__":
    funcs = _functions()
    keys = ("HGMMA", "LDSM", "LDS", "F2FP", "FADD", "IMAD", "IADD3", "R2UR", "LOP3", "ISETP", "BRA", "SYNCS", "WARPGROUP.DEPBAR")
    print("kernel | main-loop instructions | " + " | ".join(keys))
    for pat in (OLD, NEW):
        for k in _kernels(funcs, pat):
            loop = main_loop(funcs[k])
            short = re.search(r"(conv_igemm_(?:halo|presplit)_kernel)ILi(\d+)E(?:Li(\d)E)?", k)
            name = f"{short.group(1)}<{short.group(2)}{', ' + short.group(3) if short.group(3) else ''}>"
            print(f"{name} | {sum(loop.values())} | " + " | ".join(str(loop.get(x, 0)) for x in keys))
    sys.exit(0)
