"""The wide pre-split kernel (switch igemm_wide) as compiled: registered switch, pipelined SS wgmma, a main loop that
reads both operands by descriptor (no ldmatrix, no split), and no local-memory spills.  Checked on the built library
without a GPU."""
import collections

from test_igemm_presplit_sass import _functions, _kernels, main_loop

NEW = r"conv_igemm_wide_kernelILi(64|128)ELb0EE"


def test_wide_switch_is_registered():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    assert lib.fcuda_get_tuning(b"igemm_wide") == 1
    assert lib.fcuda_set_tuning(b"igemm_wide", 2) == -200
    assert lib.fcuda_set_tuning(b"igemm_wide", -1) == -200


def test_wide_wgmma_are_not_serialised():
    funcs = _functions()
    kernels = _kernels(funcs, NEW)
    assert len(kernels) == 2, kernels
    for k in kernels:
        c = collections.Counter(op for _, op, _ in funcs[k])
        hgmma, depbar = c["HGMMA"], c["WARPGROUP.DEPBAR"]
        assert hgmma >= 6 and hgmma % 6 == 0, (k, dict(c))  # 3 MMAs x 2 k-steps per commit group
        assert 1 <= depbar <= hgmma // 6 + 1 and depbar < hgmma, (k, hgmma, depbar)


def test_wide_main_loop_reads_operands_by_descriptor():
    funcs = _functions()
    for k in _kernels(funcs, NEW):
        loop = main_loop(funcs[k])
        assert loop is not None, k
        assert loop["HGMMA"] == 6, (k, dict(loop))
        assert loop["LDSM"] == 0 and loop["F2FP"] == 0 and loop["FADD"] == 0, (k, dict(loop))
        # the split exists, once per half box, outside the main loop
        assert sum(op == "F2FP" for _, op, _ in funcs[k]) > 0, k


def test_wide_kernel_does_not_spill():
    funcs = _functions()
    for k in _kernels(funcs, NEW):
        ops = collections.Counter(op for _, op, _ in funcs[k])
        assert ops["LDL"] == 0 and ops["STL"] == 0, (k, ops["LDL"], ops["STL"])
