"""CPU-side checks of the product: the native libraries load and export every symbol the headers declare, the
host-only parts of the C ABI (geometry, SelectAlgo, workspace planning) follow the reference's rules, and
feather::Net's loader parses / rejects model files like the reference.  No kernel is launched here."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def _declared(header: Path) -> list[str]:
    text = re.sub(r"/\*.*?\*/", "", header.read_text(), flags=re.S)
    return sorted(set(re.findall(r"\b(f(?:cuda|net)_[a-z0-9_]+)\s*\(", text)))


def test_libfcuda_exports_every_declared_symbol():
    from feathercnn_b200 import _lib
    lib = _lib.fcuda()
    names = _declared(ROOT / "include" / "fcuda.h")
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"libfcuda.so does not export {n}"


def test_libfeather_exports_every_declared_symbol():
    from feathercnn_b200 import _lib
    lib = _lib.feather()
    names = _declared(ROOT / "include" / "feather_c.h")
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"libfeather_b200.so does not export {n}"


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from feathercnn_b200 import _lib
    monkeypatch.setattr(_lib, "_LIBDIR", tmp_path)
    monkeypatch.setattr(_lib, "_fcuda", None)
    with pytest.raises(_lib.NativeLibraryError):
        _lib.fcuda()


def test_conv_param_layout_matches_booster_struct():
    """booster::ConvParam = 15 ints, bool, enum (booster.h:59-77): 68 bytes, activation at offset 64."""
    from feathercnn_b200._lib import FcudaConvParam
    assert ctypes.sizeof(FcudaConvParam) == 68
    assert FcudaConvParam.bias_term.offset == 60 and FcudaConvParam.activation.offset == 64
    assert FcudaConvParam.group.offset == 56


def test_geometry_and_select_algo_follow_reference_rules(oracle, restatement):
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    rng = np.random.default_rng(0)
    seen = set()
    for _ in range(400):
        ic = int(rng.choice([3, 4, 8, 16, 30, 32, 64]))
        oc = int(rng.choice([4, 6, 16, 62, 64]))
        k = int(rng.choice([1, 3, 5, 7]))
        s = int(rng.choice([1, 2]))
        pad = int(rng.integers(0, k // 2 + 1))
        h, w = int(rng.integers(k, 40)), int(rng.integers(k, 40))
        group = int(rng.choice([1, 1, 1, ic, 2]))
        if group == ic:
            oc = ic
        po = oracle.ConvParam.make(oc, ic, h, w, k, stride=s, pad=pad, group=group)
        pg = booster.ConvParam.make(oc, ic, h, w, k, stride=s, pad=pad, group=group)
        assert (pg.output_h, pg.output_w, pg.output_channels) == (po.output_h, po.output_w, po.output_channels)
        a = ctypes.c_int()
        rc = fcuda().fcuda_conv_select_algo(ctypes.byref(pg), ctypes.byref(a))
        want = restatement.select_algo(po)
        assert a.value == want and (rc == 0) == (want >= 0)
        seen.add(want)
    assert {oracle.ALGO_WINOGRADF63, oracle.ALGO_IM2COL, oracle.ALGO_DEPTHWISE, -1} <= seen


def test_workspace_planning_is_host_only_and_consistent():
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    p = booster.ConvParam.make(64, 64, 56, 56, 3, pad=1)
    cb = booster.ConvBooster()
    assert cb.SelectAlgo(p) == 0 and cb.algo == booster.WINOGRADF63
    booster.set_precision(booster.PRECISION_TF32X3)
    s1, k1 = cb.GetBufferSize(p, 1)
    s64, k64 = cb.GetBufferSize(p, 64)
    assert k1 == k64 == 2 * 64 * 64 * 64          # hi + lo planes of U[64][OC][IC]
    assert s1 == 64 * 100 * (64 + 64)              # V (plain fp32, split on chip) + M for the 10x10 tiles of one image
    assert s64 >= s1
    booster.set_precision(booster.PRECISION_TF32)
    try:
        _, k_tf32 = cb.GetBufferSize(p, 1)
        assert k_tf32 == 64 * 64 * 64              # reference: processed kernel = 64*IC*OC (avx/booster.cpp:196)
    finally:
        booster.set_precision(booster.PRECISION_TF32X3)
    # errors: partial groups / unsupported algorithms are -1 like avx/booster.cpp:304-308,349-353
    s, k = ctypes.c_size_t(), ctypes.c_size_t()
    assert fcuda().fcuda_conv_get_buffer_size(ctypes.byref(p), booster.WINOGRADF63FUSED, 1, ctypes.byref(s), ctypes.byref(k)) == -1
    assert fcuda().fcuda_conv_get_buffer_size(ctypes.byref(p), booster.SGECONV, 1, ctypes.byref(s), ctypes.byref(k)) == 0
    assert s.value == 0 and k.value == 2 * 9 * 64 * 64   # implicit GEMM: no scratch, [tap][OC][IC] hi+lo
    # the same buffer holds the pre-tiled BF16x3 planes of the default mode: 2 planes x k-blocks x OCpad x 64 bytes, where OCpad
    # is OC rounded up to the N tile (32 / 64 / 128) — larger than the fp32 rows for short K or few output channels
    for oc, ic, kk in ((64, 3, 3), (40, 64, 1), (200, 32, 1), (8, 8, 3)):
        q = booster.ConvParam.make(oc, ic, 16, 16, kk, pad=kk // 2)
        assert fcuda().fcuda_conv_get_buffer_size(ctypes.byref(q), booster.SGECONV, 1, ctypes.byref(s), ctypes.byref(k)) == 0
        K = ic * kk * kk
        bn = 32 if oc <= 32 else 64 if oc <= 64 else 128
        ocpad = -(-oc // bn) * bn
        tiled_floats = (2 * -(-K // 32) * ocpad * 64 + 3) // 4
        assert k.value == max(2 * oc * ((K + 3) // 4 * 4), tiled_floats), (oc, ic, kk, k.value)
    assert fcuda().fcuda_conv_get_buffer_size(ctypes.byref(p), booster.WINOGRADF63, 0, ctypes.byref(s), ctypes.byref(k)) == -100
    assert fcuda().fcuda_pooling_out_dim(112, 0, 0, 3, 2) == 56


def test_tuned_select_algo_moves_bandwidth_bound_layers():
    """Tuned cost model: VGG conv1_2/conv2_x and every layer the reference sends to im2col go to the implicit GEMM;
    deep 3x3 layers stay on Winograd F(6,3); depthwise stays depthwise."""
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda

    def tuned(*a, **kw):
        p = booster.ConvParam.make(*a, **kw)
        al = ctypes.c_int()
        assert fcuda().fcuda_conv_select_algo_tuned(ctypes.byref(p), ctypes.byref(al)) == 0
        return al.value

    assert tuned(64, 64, 224, 224, 3, pad=1) == booster.SGECONV
    assert tuned(128, 128, 112, 112, 3, pad=1) == booster.SGECONV
    assert tuned(256, 256, 56, 56, 3, pad=1) == booster.WINOGRADF63
    assert tuned(512, 512, 14, 14, 3, pad=1) == booster.WINOGRADF63
    assert tuned(64, 3, 224, 224, 3, pad=1) == booster.SGECONV         # reference: IM2COL (IC % 4 != 0)
    assert tuned(256, 64, 56, 56, 1) == booster.SGECONV                # ResNet pointwise
    assert tuned(512, 256, 56, 56, 1, stride=2) == booster.SGECONV     # strided downsample
    assert tuned(64, 3, 224, 224, 7, stride=2, pad=3) == booster.SGECONV
    assert tuned(512, 512, 7, 7, 3, pad=1) == booster.SGECONV          # reference: IM2COL (input_h <= 8)
    assert tuned(32, 32, 56, 56, 3, stride=1, pad=1, group=32) == booster.DEPTHWISE


def _net(**kw):
    from feathercnn_b200.net import Net
    return Net(**kw)


def test_load_param_builds_the_blob_graph(tmp_path):
    from feathercnn_b200.tools import modelgen
    m = modelgen.mini()
    param, _ = m.save(tmp_path / "mini")
    net = _net()
    net.LoadParam(param)
    assert sorted(net.BlobNames()) == sorted(m.blobs)
    assert net.input_name == "data" and net.input_shape == (4, 32, 32)
    net2 = _net()
    net2.LoadParamFromText(Path(param).read_text())
    assert sorted(net2.BlobNames()) == sorted(m.blobs)


@pytest.mark.parametrize("text,code", [
    ("7767516\n1 1\nInput data 0 1 data 0=4 1=4 2=1\n", -1),                                   # bad magic, utils.cpp:36-40
    ("7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=1\nReLU r 1 1 nope out\n", -300),            # topology, net.cpp:127-131
    ("7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=1\nFancyOp f 1 1 data out\n", -200),        # unregistered, net.cpp:107-111
    ("7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=1\nConvolution c 1 1 data out 0=4 1=3 8=1 6=36\n", -200),  # int8, conv_layer.h:49-54
    ("7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=1\nEltwise e 1 1 data out 0=7\n", -100),     # unknown Eltwise op
    ("7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=1\nEltwise e 1 1 data out 0=0 -23301=2,0.5,0.5\n", -100),  # coeffs only with SUM
    ("7767517\n-3 2\nInput data 0 1 data 0=4 1=4 2=1\n", -1),                                   # corrupt counts (ADVICE r1)
    ("7767517\n1 1\nInput data 0 -5 data 0=4 1=4 2=1\n", -1),                                   # negative top count
])
def test_load_param_rejects_like_the_reference(text, code):
    from feathercnn_b200.net import FeatherError
    with pytest.raises(FeatherError) as e:
        _net().LoadParamFromText(text)
    assert e.value.code == code


@pytest.mark.parametrize("text", [
    # SURVEY.md §8f rank 4: what the reference rejects (conv_layer.h:43-47, eltwise_layer.h:57-66, avx/booster.cpp:304-308,
    # concat_layer.h:50-54) loads here
    "7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=1\nConvolution c 1 1 data out 0=4 1=3 2=2 6=36\n",        # dilation 2
    "7767517\n2 2\nInput data 0 1 data 0=8 1=8 2=8\nConvolution c 1 1 data out 0=16 1=3 7=4 6=288\n",      # 4 groups of 2 -> 4
    "7767517\n3 3\nInput a 0 1 a 0=4 1=4 2=1\nInput b 0 1 b 0=4 1=4 2=1\nEltwise e 2 1 a b out 0=0\n",      # PROD
    "7767517\n3 3\nInput a 0 1 a 0=4 1=4 2=1\nInput b 0 1 b 0=4 1=4 2=1\nEltwise e 2 1 a b out 0=2\n",      # MAX
    "7767517\n3 3\nInput a 0 1 a 0=4 1=4 2=1\nInput b 0 1 b 0=4 1=4 2=1\nEltwise e 2 1 a b out 0=1 -23301=2,0.5,-2.0\n",
    "7767517\n3 3\nInput a 0 1 a 0=4 1=4 2=1\nInput b 0 1 b 0=4 1=4 2=1\nConcat c 2 1 a b out 0=2\n",       # concat along w
])
def test_load_param_accepts_the_section_8f_extensions(text):
    _net().LoadParamFromText(text)


def test_truncated_or_corrupt_container_is_an_error_not_a_crash(tmp_path):
    """ADVICE r1: InitFromBuffer on a short / corrupt .feathermodel must return an error code (the FILE path already did)."""
    from feathercnn_b200.net import FeatherError
    from feathercnn_b200.tools import feathermodel, modelgen
    m = modelgen.mini()
    param, binf = m.save(tmp_path / "mini")
    blob = Path(feathermodel.pack(param, binf, tmp_path / "mini.feathermodel")).read_bytes()
    for cut in (len(blob) - 1, len(blob) // 2, 24, 17):
        with pytest.raises(FeatherError):
            _net().InitFromBuffer(blob[:cut])
    huge = bytearray(blob)
    huge[8:16] = (2**64 - 8).to_bytes(8, "little")  # param_len that wraps 16 + param_len
    with pytest.raises(FeatherError):
        _net().InitFromBuffer(bytes(huge))


RESNET_BLOCK = """7767517
9 10
Input data 0 1 data 0=8 1=8 2=8
Convolution conv_in 1 1 data conv_in 0=8 1=3 3=1 4=1 5=1 6=576
ReLU relu_in 1 1 conv_in relu_in
Split split 1 2 relu_in sa sb
Convolution branch 1 1 sb branch 0=8 1=1 3=1 4=0 5=1 6=64
Eltwise sum 2 1 sa branch sum 0=1
ReLU relu_out 1 1 sum relu_out
Convolution tail 1 1 relu_out tail 0=8 1=3 3=1 4=1 5=0 6=576
ReLU tail_relu 1 1 tail tail_relu
"""


def test_fusion_pass_rewrites_the_graph_on_the_host():
    """The live TryFuse pass (layer.h:61-68, dead in the reference) + the shortcut pass: conv+ReLU, Eltwise+ReLU, and the
    Eltwise SUM itself absorbed into the convolution that produces its otherwise unread addend.  Host only."""
    net = _net(fusion=True)
    net.LoadParamFromText(RESNET_BLOCK)
    assert net.FuseNow() == 4                      # relu_in, relu_out, sum, tail_relu
    assert net.FuseNow() == 4                      # idempotent
    for name, fused in [("relu_in", 1), ("relu_out", 1), ("sum", 1), ("tail_relu", 1),
                        ("conv_in", 0), ("branch", 0), ("split", 0), ("tail", 0)]:
        assert net.LayerFusedAway(name) == fused, name
    assert net.LayerFusedAway("nope") == -1
    names = set(net.BlobNames())
    # the absorbed layers' intermediate blobs are gone; the surviving producer writes the last name of the chain
    assert {"data", "relu_in", "sa", "sb", "relu_out", "tail_relu"} <= names
    assert not ({"conv_in", "branch", "sum", "tail"} & names)
    plain = _net()
    plain.LoadParamFromText(RESNET_BLOCK)
    assert plain.FuseNow() == 0                    # SetFusion(false): nothing is rewritten


def test_residual_and_profile_entry_points_validate_arguments():
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    p = booster.ConvParam.make(8, 8, 8, 8, 1)
    assert lib.fcuda_conv_forward_residual(ctypes.byref(p), booster.SGECONV, None, None, None, None, None, None, 1, 1, None) == -100
    ms, af, mf, ab = ctypes.c_double(-1), ctypes.c_double(-1), ctypes.c_double(-1), ctypes.c_double(-1)
    n = ctypes.c_longlong(-1)
    # enabling drops the records that a profiled run earlier in this process (a GPU test) left behind
    lib.fcuda_profile_tensor_gemm(1)
    lib.fcuda_profile_tensor_gemm(0)
    for kind in (-1, 0, 1, 6):
        assert lib.fcuda_profile_collect_kind(kind, ctypes.byref(ms), ctypes.byref(af), ctypes.byref(mf), ctypes.byref(ab),
                                              ctypes.byref(n)) == 0
        assert (ms.value, af.value, ab.value, n.value) == (0.0, 0.0, 0.0, 0)


def test_hot_kernels_run_on_wgmma_and_tma_in_sass():
    """wgmma.mma_async -> HGMMA, TMA tensor loads -> UTMALDG, 1-D bulk copies -> UBLKCP.  The two product GEMM-class
    kernels must contain them (and no legacy HMMA / mma.sync path); a kernel that silently fell back to CUDA cores would
    show here without a GPU."""
    import collections
    import shutil
    import subprocess
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
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
        if m and cur:
            ops[cur][m.group(1)] += 1
    assert "arch = sm_90a" in sass

    def only(pattern):
        hit = [k for k in ops if re.search(pattern, k)]
        assert hit, pattern
        return hit

    for k in only(r"conv_igemm_kernelILi(32|64|128)ELi2E"):     # 3xTF32 implicit-GEMM conv
        c = ops[k]
        # three tf32 MMAs per 8-k step, four steps per k-block; hi and lo filter planes by TMA
        assert c["HGMMA"] == 12 and c["UTMALDG"] >= 2, (k, dict(c))
        assert c["HMMA"] == 0 and c["FFMA"] == 0, k              # no tensor-core-less inner product hiding in there
    for k in only(r"conv_igemm_kernelILi(32|64|128)ELi3E"):     # BF16x3 implicit-GEMM conv (the default mode)
        c = ops[k]
        # three bf16 MMAs per 16-k step, two steps per k-block; filters by ONE 1-D bulk copy (UBLKCP) per k-block
        assert c["HGMMA"] == 6 and c["UBLKCP"] >= 1, (k, dict(c))
        assert c["F2FP"] >= 16 and c["HMMA"] == 0 and c["FFMA"] == 0, (k, dict(c))   # on-chip bf16 RN split, no CUDA-core GEMM
    for k in only(r"tensor_gemm_kernelILi(32|64|128)ELi2E"):     # 3xTF32 TensorGEMM, A split on chip
        c = ops[k]
        # 12 MMAs per k-block, issued from the k-block-pair loop body and the odd tail
        assert c["HGMMA"] >= 12 and c["HGMMA"] % 12 == 0 and c["UTMALDG"] >= 3, (k, dict(c))
        assert c["HMMA"] == 0
    for k in only(r"wino_(in|out)put_kernelILi8E"):              # transforms stay on CUDA cores, as designed
        assert ops[k]["HGMMA"] == 0 and ops[k]["FFMA"] + ops[k]["FADD"] > 100


PLUGIN_SRC = r"""
// a user-defined layer written against the public headers only, as it would be against the reference's
#include <feather/layer_factory.h>
namespace feather {
class NegateLayer : public Layer {
public:
    explicit NegateLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) { factor = pd.get(0, -1.f); return 0; }
    int Forward() { return 0; }
    float factor = 0.f;
};
DEFINE_LAYER_CREATOR(Negate)
REGISTER_LAYER_CREATOR(Negate, Negate)
}  // namespace feather
extern "C" int plugin_loaded() { return 1; }
"""


def test_user_layer_registers_through_the_plugin_macros(tmp_path):
    """DEFINE_LAYER_CREATOR / REGISTER_LAYER_CREATOR (layer_factory.h:85-90): a layer compiled outside the library is
    created by Net::LoadParam from its ncnn type name; unknown types are still refused with -200 (net.cpp:101-105)."""
    import subprocess
    from feathercnn_b200 import _lib
    text = "7767517\n2 2\nInput data 0 1 data 0=4 1=4 2=2\nNegate neg 1 1 data neg 0=-2.5\n"
    before = _net()
    with pytest.raises(Exception) as e:
        before.LoadParamFromText(text)
    assert "-200" in str(e.value)
    src = tmp_path / "plugin.cpp"
    src.write_text(PLUGIN_SRC)
    so = tmp_path / "libnegate_plugin.so"
    libdir = ROOT / "feathercnn_b200" / "lib"
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{ROOT / 'include'}", "-I/usr/local/cuda/include",
                    str(src), "-o", str(so), f"-L{libdir}", "-lfeather_b200", f"-Wl,-rpath,{libdir}"], check=True)
    _lib.feather()                      # the host library first: the plugin's static registrar calls into it
    plugin = ctypes.CDLL(str(so), mode=ctypes.RTLD_GLOBAL)
    assert plugin.plugin_loaded() == 1
    net = _net()
    net.LoadParamFromText(text)
    assert sorted(net.BlobNames()) == ["data", "neg"]


def _modelbin_cases():
    rng = np.random.default_rng(11)
    w = 37  # odd on purpose: fp16 and LUT payloads are padded to 4 bytes (modelbin.cpp alignSize)
    vals = rng.standard_normal(w).astype(np.float32)
    half = vals.astype(np.float16)
    table = rng.standard_normal(256).astype(np.float32)
    idx = rng.integers(0, 256, w).astype(np.uint8)
    pad = lambda b: b + b"\0" * (-len(b) % 4)
    tag = lambda t: np.uint32(t).tobytes()
    return [
        ("raw fp32 (tag 0)", 0, tag(0) + vals.tobytes(), vals, 4 + 4 * w),
        ("fp16 (tag 0x01306B47)", 0, tag(0x01306B47) + pad(half.tobytes()), half.astype(np.float32), 4 + len(pad(half.tobytes()))),
        ("256-entry LUT", 0, tag(0x00000101) + table.tobytes() + pad(idx.tobytes()), table[idx], 4 + 1024 + len(pad(idx.tobytes()))),
        ("raw fp32 via the 0x0002C056 tag", 0, tag(0x0002C056) + vals.tobytes(), vals, 4 + 4 * w),
        ("type 1: untagged fp32", 1, vals.tobytes(), vals, 4 * w),
    ]


@pytest.mark.parametrize("case", _modelbin_cases(), ids=[c[0] for c in _modelbin_cases()])
def test_weight_blob_decoder_matches_the_reference_loader(oracle, case):
    """SURVEY §8(f) rank 2: fp16 and LUT-quantised ncnn weight blobs and the from-memory loader
    (src/ncnn/modelbin.cpp:77-160, 204-293) decode exactly like the reference's ModelBinFromMemory."""
    from feathercnn_b200._lib import feather
    name, type_, blob, want, nbytes = case
    w = len(want)
    out = np.zeros(w, np.float32)
    n = feather().fnet_modelbin_load_mem(blob + b"\0" * 64, w, type_, out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
    assert n == nbytes, name
    np.testing.assert_array_equal(out, want)
    if oracle.reference_available():
        ref_vals, ref_n = oracle.Reference().modelbin_load_mem(blob, w, type_)
        assert ref_n == n, name
        np.testing.assert_array_equal(ref_vals, out)


def test_weight_blob_decoder_rejects_int8_like_the_layer_does():
    from feathercnn_b200._lib import feather
    blob = np.uint32(0x000D4B38).tobytes() + bytes(64)  # int8 weights: conv_layer.h:49-54 refuses them
    out = np.zeros(8, np.float32)
    assert feather().fnet_modelbin_load_mem(blob, 8, 0, out.ctypes.data_as(ctypes.POINTER(ctypes.c_float))) == -1
    assert feather().fnet_modelbin_load_mem(blob, 8, 7, out.ctypes.data_as(ctypes.POINTER(ctypes.c_float))) == -1  # unknown type


def test_launch_list_summary_and_traffic_json(tmp_path):
    """scripts/summarize_launches.py: shares of one Forward (between the last two softmax launches) and the per-kernel DRAM
    bytes that bench.py reports as roofline.traffic."""
    import json
    import subprocess
    import sys
    hdr = '"ID","Process ID","Process Name","Host Name","Kernel Name","Context","Stream","Block Size","Grid Size","Device","CC","Section Name","Metric Name","Metric Unit","Metric Value"'
    rows = [hdr]

    def launch(i, name, us, rd_mb, wr_mb):
        base = f'"{i}","1","python","box","{name}","1","7","(128, 1, 1)","(148, 1, 1)","0","10.0","Command line profiler metrics"'
        rows.append(f'{base},"dram__bytes_read.sum","Mbyte","{rd_mb}"')
        rows.append(f'{base},"dram__bytes_write.sum","Mbyte","{wr_mb}"')
        rows.append(f'{base},"gpu__time_duration.sum","us","{us}"')

    i = 0
    for step in range(2):
        launch(i, "void unnamed>::conv_igemm_kernel<64, 2>(CUtensorMap_st, CUtensorMap_st, unnamed>::IgemmArgs)", 300, 50, 750); i += 1
        launch(i, "void unnamed>::conv_igemm_kernel<64, 2>(CUtensorMap_st, CUtensorMap_st, unnamed>::IgemmArgs)", 900, 800, 800); i += 1
        launch(i, "void tensor_gemm_ts_kernel<128, 1>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, GemmKernelArgs)", 200, 400, 0); i += 1
        launch(i, "softmax_kernel(const float *, float *, unsigned long)", 5, 0.1, 0.1); i += 1
    csv_path = tmp_path / "launches.csv"
    csv_path.write_text("==PROF== Connected\n" + "\n".join(rows) + "\n")
    out_json = tmp_path / "traffic.json"
    r = subprocess.run([sys.executable, str(ROOT / "scripts" / "summarize_launches.py"), str(csv_path), str(out_json)],
                       capture_output=True, text=True, check=True)
    assert "one Forward (between the last two softmax launches): 4 launches" in r.stdout
    assert "conv_igemm_kernel" in r.stdout and "85." in r.stdout        # 1200 of 1405 us
    t = json.loads(out_json.read_text())
    assert t["conv_igemm_kernel"] == pytest.approx(1.2e9) and t["tensor_gemm_ts_kernel"] == pytest.approx(4e8)


def test_clock_sampler_uses_only_rows_inside_the_timed_windows(tmp_path, monkeypatch):
    """bench.py's `clocks` object: nvidia-smi is polled from before the warm-up, only rows received inside the marked
    timed regions count, and throttle reasons are collected from them."""
    import importlib.util
    import os
    import stat
    import time
    fake = tmp_path / "nvidia-smi"
    # index, clocks.sm, clocks.max.sm, power, hw_slowdown, hw_thermal, sw_thermal, sw_power_cap — one row every 20 ms;
    # the first 10 rows (idle clocks) fall before the timed window
    fake.write_text("#!/bin/bash\ni=0\nwhile true; do\n  if [ $i -lt 10 ]; then echo '0, 345, 1965, 140.0, Not Active, Not Active, Not Active, Not Active';\n"
                    "  else echo '0, 1755, 1965, 990.0, Not Active, Not Active, Not Active, Active'; fi\n  i=$((i+1)); sleep 0.02\ndone\n")
    fake.chmod(fake.stat().st_mode | stat.S_IEXEC)
    monkeypatch.setenv("PATH", f"{tmp_path}{os.pathsep}{os.environ['PATH']}")
    spec = importlib.util.spec_from_file_location("bench_mod", ROOT / "bench.py")
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    s = bench.ClockSampler(0)
    s.start()
    time.sleep(0.45)   # "warm-up": idle rows arrive, outside any window
    s.begin()
    time.sleep(0.3)
    s.end()
    out = s.stop()
    assert out["samples"] >= 5 and out["sampled"] == "inside the timed regions"
    assert out["sm_mhz"] == 1755.0 and out["sm_max_mhz"] == 1965.0 and out["reasons"] == ["sw_power_cap"]
    assert 0.25 <= out["window_s"] <= 0.6


def test_bench_reference_arm_prints_the_contract_line(oracle):
    """`bench.py --impl reference` (the arm the driver runs next to ours) on BASELINE.json configs[0]: CPU only, same
    metric / unit / config keys, rank != 0 exits silently."""
    import json
    import os
    import subprocess
    import sys
    if not oracle.reference_available():
        pytest.skip("oracle/_ref not built")
    cmd = [sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--model", "single_conv", "--steps", "1", "--warmup", "0"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-500:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "images/sec" and line["unit"] == "images/s"
    assert line["higher_is_better"] is True and line["vs_baseline"] is None and line["value"] > 0
    assert line["config"]["workload"].startswith("single_conv_b64") and line["cpu_baseline"]["kind"] == "reference"
    assert line["e2e"] == {"value": line["value"], "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r1 = subprocess.run(cmd, capture_output=True, text=True, timeout=60, cwd=ROOT, env=env)
    assert r1.returncode == 0 and r1.stdout.strip() == ""


def test_feathermodel_container_round_trip(tmp_path):
    from feathercnn_b200.tools import feathermodel, modelgen
    param, binf = modelgen.single_conv(ic=4, oc=4, h=9, w=9).save(tmp_path / "m")
    fm = feathermodel.pack(param, binf, tmp_path / "m.feathermodel")
    p2, b2 = feathermodel.unpack(fm, tmp_path / "again")
    assert Path(p2).read_bytes() == Path(param).read_bytes() and Path(b2).read_bytes() == Path(binf).read_bytes()


def test_modelgen_flop_counts_match_survey():
    """SURVEY.md §8(d) algorithmic FLOPs per image (booster.h:145-148 convention)."""
    from feathercnn_b200.tools import modelgen
    assert abs(modelgen.single_conv().flops / 1e9 - 0.2312) < 1e-3
    # parse-only instantiation of the big models is slow (random weights); count FLOPs from a shape-only walk
    m = modelgen.resnet50.__wrapped__() if hasattr(modelgen.resnet50, "__wrapped__") else None
    assert m is None or abs(m.flops / 1e9 - 7.716) < 0.05


def test_tuning_switch_names_and_ranges_are_validated():
    """fcuda_set_tuning / fcuda_get_tuning (kernel-variant switches): names and ranges are checked, defaults are the
    measured-best configuration."""
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    assert lib.fcuda_set_tuning(b"nope", 1) == -200
    assert lib.fcuda_set_tuning(b"dw_vec", 2) == -200
    assert lib.fcuda_set_tuning(b"persistent_ctas", 65537) == -200
    assert lib.fcuda_get_tuning(b"nope") == -200
    assert lib.fcuda_get_tuning(b"dw_vec") == 1 and lib.fcuda_get_tuning(b"persistent_ctas") == 0
    assert lib.fcuda_set_tuning(b"dw_vec", 0) == 0 and lib.fcuda_get_tuning(b"dw_vec") == 0
    assert lib.fcuda_set_tuning(b"dw_vec", 1) == 0


def test_retired_tuning_switches_are_unknown_names():
    """include/fcuda.h: the retired switches wino_mlp, gemm_pipe and yolo_nms are unknown names, -200 to get or set."""
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    for name in (b"wino_mlp", b"gemm_pipe", b"yolo_nms"):
        assert lib.fcuda_get_tuning(name) == -200, name
        assert lib.fcuda_set_tuning(name, 0) == -200 and lib.fcuda_set_tuning(name, 1) == -200, name


def test_every_documented_tuning_switch_and_precision_mode_exists():
    """include/fcuda.h documents the kernel-variant switches as `name (range, default)` and the three arithmetic modes; the
    registry in libfcuda.so must know each name, report the documented default and reject out-of-range values."""
    from feathercnn_b200 import booster
    from feathercnn_b200._lib import fcuda
    lib = fcuda()
    text = (ROOT / "include" / "fcuda.h").read_text()
    found = re.findall(r"^ \*   (\w+) \(([0-9|\-]+), (\d+)\)", text, flags=re.M)
    assert len(found) >= 2, found
    for name, rng, default in found:
        assert lib.fcuda_get_tuning(name.encode()) == int(default), (name, default)
        hi = int(re.split(r"[|\-]", rng)[-1])
        assert lib.fcuda_set_tuning(name.encode(), hi + 1) == -200, name
        assert lib.fcuda_set_tuning(name.encode(), int(default)) == 0, name
    saved = booster.get_precision()
    try:
        for mode in (booster.PRECISION_TF32X3, booster.PRECISION_TF32, booster.PRECISION_FP32_SPLIT):
            booster.set_precision(mode)
            assert booster.get_precision() == mode
        assert lib.fcuda_set_precision(3) == -200 and lib.fcuda_set_precision(-1) == -200
    finally:
        booster.set_precision(saved)
