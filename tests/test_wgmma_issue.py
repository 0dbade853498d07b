"""The tensor-core kernels keep several wgmma in flight.

ptxas serialises every wgmma of a kernel it cannot pipeline (a function call inside the pipeline, a register operand it
cannot prove untouched, too few registers): each HGMMA is then followed by its own `WARPGROUP.DEPBAR.LE gsb0, 0x0`,
so a warpgroup never has two MMAs running.  A pipelined kernel waits once per commit group instead, so its SASS has far
fewer DEPBARs than HGMMAs.  Checked on the built library without a GPU."""
import collections
import re
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def _sass_ops():
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    so = ROOT / "feathercnn_b200" / "lib" / "libfcuda.so"
    sass = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True, check=True).stdout
    ops: dict[str, collections.Counter] = collections.defaultdict(collections.Counter)
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)?)", line)
        if m and cur:
            op = m.group(1)
            ops[cur][op.split(".")[0] if not op.startswith("WARPGROUP") else op] += 1
    return ops


def _kernels(ops, pattern):
    hit = sorted(k for k in ops if re.search(pattern, k))
    assert hit, pattern
    return hit


@pytest.mark.parametrize("pattern, per_group", [
    (r"tensor_gemm_kernelILi(32|64|128)ELi2E", 12),        # 3xTF32 TensorGEMM: 3 MMAs x 4 k-steps per k-block
    (r"tensor_gemm_kernelILi(32|64|128)ELi1E", 4),         # TF32 TensorGEMM
    (r"conv_igemm_kernelILi(32|64|128)ELi3E", 6),          # BF16x3 gathering implicit GEMM: 3 MMAs x 2 k-steps
    (r"conv_igemm_kernelILi(32|64|128)ELi1E", 4),          # TF32 gathering implicit GEMM
    pytest.param(r"conv_igemm_halo_kernelILi(32|64|128)ELi3ELb0E", 6,  # BF16x3 per-tap halo implicit GEMM
                 id="conv_igemm_halo_kernelILi(32|64|128)ELi3E-6"),
])
def test_wgmma_are_not_serialised(pattern, per_group):
    ops = _sass_ops()
    for k in _kernels(ops, pattern):
        c = ops[k]
        hgmma, depbar = c["HGMMA"], c["WARPGROUP.DEPBAR"]
        assert hgmma >= per_group and hgmma % per_group == 0, (k, dict(c))
        # at most one wait per commit group plus the drain at the end of a tile (serialised code has one per HGMMA)
        assert 1 <= depbar <= hgmma // per_group + 1 and depbar < hgmma, (k, hgmma, depbar)

