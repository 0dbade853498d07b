"""The persistent stem kernel (switch igemm_stem) as compiled: registered switch, exported query, wgmma not serialised
(one WARPGROUP.DEPBAR for the six HGMMA of a k-block) and no local memory.  Checked on the built library without a GPU."""
import collections

from test_igemm_presplit_sass import _functions, _kernels

NEW = r"conv_igemm_stem_kernelILi(32|64|128)ELb[01]EE"


def test_stem_switch_is_registered():
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    assert lib.fcuda_get_tuning(b"igemm_stem") == 1
    assert lib.fcuda_set_tuning(b"igemm_stem", 2) == -200
    assert lib.fcuda_set_tuning(b"igemm_stem", -1) == -200
    assert lib.fcuda_igemm_stem_supported(None, None) == 0


def test_stem_wgmma_are_not_serialised():
    funcs = _functions()
    kernels = _kernels(funcs, NEW)
    assert len(kernels) == 6, kernels  # N tiles 32, 64, 128 x ReLU / Clip
    for k in kernels:
        c = collections.Counter(op for _, op, _ in funcs[k])
        hgmma, depbar = c["HGMMA"], c["WARPGROUP.DEPBAR"]
        assert hgmma == 6, (k, dict(c))  # 3 MMAs x 2 k-steps, one commit group per k-block
        assert depbar == 1, (k, hgmma, depbar)


def test_stem_kernel_has_no_local_memory():
    funcs = _functions()
    for k in _kernels(funcs, NEW):
        ops = collections.Counter(op for _, op, _ in funcs[k])
        assert ops["LDL"] == 0 and ops["STL"] == 0, (k, ops["LDL"], ops["STL"])
