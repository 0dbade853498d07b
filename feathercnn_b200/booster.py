"""Python mirror of ``booster::ConvBooster`` / ``booster::ConvParam`` over the fcuda C ABI.

Same names and call protocol as the reference (/root/reference/src/booster/include/booster/booster.h:42-170,
used as in src/layers/conv_layer.h:92-172): fill a ConvParam -> AssignOutputDim -> SelectAlgo ->
GetBufferSize -> Init (once) -> Forward.  Tensors are torch CUDA tensors used purely as device memory;
every call goes through ``libfcuda.so`` (no torch ops on the data path).
"""
from __future__ import annotations

import ctypes
import math

import torch

from ._lib import FcudaConvOptions, FcudaConvParam, fcuda
from ._lib import FcudaDeconvParam as DeconvParam
from ._lib import FcudaInterpParam as InterpParam
from ._lib import FcudaPad
from ._lib import FcudaPriorBoxParam as PriorBoxParam
from ._lib import FcudaProposalParam as ProposalParam
from ._lib import FcudaYoloParam as YoloParam

NAIVE, IM2COL, SGECONV, DEPTHWISE, WINOGRADF63, WINOGRADF63FUSED, WINOGRADF23 = range(7)
ALGO_NAMES = ["NAIVE", "IM2COL", "SGECONV", "DEPTHWISE", "WINOGRADF63", "WINOGRADF63FUSED", "WINOGRADF23"]
PRECISION_TF32X3, PRECISION_TF32, PRECISION_FP32_SPLIT = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_CLIP = 0, 1, 2  # FcudaActivation


class FcudaError(RuntimeError):
    def __init__(self, fn: str, code: int):
        super().__init__(f"{fn} returned {code}")
        self.code = code


def _check(fn: str, rc: int) -> None:
    if rc != 0:
        raise FcudaError(fn, rc)


def _ptr(t: torch.Tensor | None):
    if t is None:
        return None
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def set_precision(mode: int) -> None:
    _check("fcuda_set_precision", fcuda().fcuda_set_precision(mode))


def get_precision() -> int:
    return fcuda().fcuda_get_precision()


def set_l2_chunk_bytes(n: int) -> None:
    fcuda().fcuda_set_l2_chunk_bytes(n)


class ConvParam(FcudaConvParam):
    @classmethod
    def make(cls, oc, ic, h, w, kh, kw=None, stride=1, pad=0, group=1, bias=True, relu=False, stride_w=None,
             pad_lbrt=None):
        kw = kh if kw is None else kw
        sw = stride if stride_w is None else stride_w
        pl, pb, pr, pt = pad_lbrt if pad_lbrt is not None else (pad, pad, pad, pad)
        p = cls(oc, ic, h, w, kh, kw, 0, 0, stride, sw, pl, pb, pr, pt, group, int(bool(bias)), int(bool(relu)))
        p.AssignOutputDim()
        return p

    def AssignOutputDim(self):
        _check("fcuda_conv_assign_output_dim", fcuda().fcuda_conv_assign_output_dim(ctypes.byref(self)))

    def GetFLOPS(self) -> float:  # booster.h:145-148
        return (2.0 * self.output_channels * self.input_channels * self.output_h * self.output_w * self.kernel_h *
                self.kernel_w / self.group)

    @property
    def weight_shape(self):
        if self.group == self.input_channels and self.group > 1:
            return (self.input_channels, 1, self.kernel_h, self.kernel_w)
        return (self.output_channels, self.input_channels, self.kernel_h, self.kernel_w)


class ConvBooster:
    """ConvBooster doesn't allocate any memory (booster.h:155): the caller passes every buffer."""

    def __init__(self):
        self.algo = -1

    def SelectAlgo(self, param: ConvParam) -> int:
        a = ctypes.c_int(-1)
        rc = fcuda().fcuda_conv_select_algo(ctypes.byref(param), ctypes.byref(a))
        self.algo = a.value
        return rc

    def SelectAlgoTuned(self, param: ConvParam) -> int:
        a = ctypes.c_int(-1)
        rc = fcuda().fcuda_conv_select_algo_tuned(ctypes.byref(param), ctypes.byref(a))
        self.algo = a.value
        return rc

    def ForceSelectAlgo(self, algo: int) -> int:
        self.algo = int(algo)
        return 0

    def GetBufferSize(self, param: ConvParam, batch: int = 1) -> tuple[int, int]:
        s, k = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _check("fcuda_conv_get_buffer_size",
               fcuda().fcuda_conv_get_buffer_size(ctypes.byref(param), self.algo, batch, ctypes.byref(s), ctypes.byref(k)))
        return s.value, k.value

    def Init(self, param: ConvParam, processed_kernel: torch.Tensor, kernel: torch.Tensor) -> None:
        kp = ctypes.c_void_p(kernel.data_ptr())  # host or device pointer
        _check("fcuda_conv_init",
               fcuda().fcuda_conv_init(ctypes.byref(param), self.algo, _ptr(processed_kernel), kp, _stream()))

    def ForwardOpts(self, param: ConvParam, output, input, kernel, buffer, bias_arr, residual=None, relu_after_add=False,
                    clip: tuple[float, float] | None = None, dilation=1, pool: bool = False, batch: int = 1) -> None:
        """Forward with everything the epilogue can fuse (fcuda.h, FcudaConvOptions).  `clip` = (min, max) are the bounds
        of param.activation == ACT_CLIP; a Clip without them is refused (-200), as are bounds without a Clip.  `dilation`
        is an int or an (h, w) pair."""
        if clip is None:
            clip = (math.nan, math.nan) if param.activation == ACT_CLIP else (0.0, 0.0)
        dh, dw = _hw(dilation)
        o = FcudaConvOptions(residual=None if residual is None else _ptr(residual).value, relu_after_add=int(relu_after_add),
                             clip_min=clip[0], clip_max=clip[1], dilation_h=dh, dilation_w=dw, pool=int(pool))
        _check("fcuda_conv_forward_opts",
               fcuda().fcuda_conv_forward_opts(ctypes.byref(param), self.algo, _ptr(output), _ptr(input), _ptr(kernel),
                                               _ptr(buffer), _ptr(bias_arr), ctypes.byref(o), batch, _stream()))

    def ForwardResidual(self, param: ConvParam, output, input, kernel, buffer, bias_arr, residual, relu_after_add,
                        batch: int = 1) -> None:
        _check("fcuda_conv_forward_residual",
               fcuda().fcuda_conv_forward_residual(ctypes.byref(param), self.algo, _ptr(output), _ptr(input), _ptr(kernel),
                                                   _ptr(buffer), _ptr(bias_arr), _ptr(residual), int(relu_after_add), batch,
                                                   _stream()))

    def Forward(self, param: ConvParam, output, input, kernel, buffer, bias_arr, batch: int = 1) -> None:
        _check("fcuda_conv_forward",
               fcuda().fcuda_conv_forward(ctypes.byref(param), self.algo, _ptr(output), _ptr(input), _ptr(kernel),
                                          _ptr(buffer), _ptr(bias_arr), batch, _stream()))

    def ForwardClip(self, param: ConvParam, output, input, kernel, buffer, bias_arr, clip_min: float, clip_max: float,
                    batch: int = 1) -> None:
        """Forward with param.activation == ACT_CLIP: the output clamped to [clip_min, clip_max] in the epilogue."""
        _check("fcuda_conv_forward_clip",
               fcuda().fcuda_conv_forward_clip(ctypes.byref(param), self.algo, _ptr(output), _ptr(input), _ptr(kernel),
                                               _ptr(buffer), _ptr(bias_arr), float(clip_min), float(clip_max), batch,
                                               _stream()))


def conv_forward(param: ConvParam, x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None = None,
                 algo: int | None = None, residual: torch.Tensor | None = None,
                 relu_after_add: bool = False, dilation=1, tuned: bool = False,
                 pool: bool = False, clip: tuple[float, float] | None = None) -> tuple[torch.Tensor, int]:
    """Whole ConvBooster protocol for a batch x (N, IC, H, W) -> (N, OC, OH, OW).  Returns (output, algo).
    `residual` (shaped like the output), `clip` = (min, max) (param.activation must be ACT_CLIP), `dilation` (an int or
    an (h, w) pair; the caller sets param.output_h/w for the dilated extent) and `pool` (the output is the pooled blob)
    are ForwardOpts's."""
    cb = ConvBooster()
    if algo is None:
        rc = cb.SelectAlgoTuned(param) if tuned else cb.SelectAlgo(param)
        if rc != 0:
            raise FcudaError("fcuda_conv_select_algo", rc)
    else:
        cb.ForceSelectAlgo(algo)
    n = x.shape[0]
    scratch_n, packed_n = cb.GetBufferSize(param, n)
    packed = torch.empty(max(packed_n, 1), device=x.device, dtype=torch.float32)
    scratch = torch.empty(max(scratch_n, 1), device=x.device, dtype=torch.float32)
    cb.Init(param, packed, w.contiguous())
    oh, ow = ((param.output_h + 1) // 2, (param.output_w + 1) // 2) if pool else (param.output_h, param.output_w)
    out = torch.empty((n, param.output_channels, oh, ow), device=x.device, dtype=torch.float32)
    cb.ForwardOpts(param, out, x.contiguous(), packed, scratch, b, None if residual is None else residual.contiguous(),
                   relu_after_add, clip, dilation, pool, n)
    return out, cb.algo


# ---- deconvolution ---------------------------------------------------------------------------------
def _hw(v) -> tuple[int, int]:
    return (int(v), int(v)) if isinstance(v, int) else (int(v[0]), int(v[1]))


def deconv_param(oc: int, ic: int, h: int, w: int, kh: int, kw: int | None = None, stride=1, pad=0, output_pad=0,
                 dilation=1, group: int = 1, bias: bool = True, relu: bool = False) -> DeconvParam:
    """FcudaDeconvParam with output_h / output_w filled.  stride, dilation and output_pad are an int or (h, w);
    pad is an int or (top, bottom, left, right)."""
    kw = kh if kw is None else kw
    sh, sw = _hw(stride)
    dh, dw = _hw(dilation)
    oph, opw = _hw(output_pad)
    pt, pb, pl, pr = (pad,) * 4 if isinstance(pad, int) else tuple(pad)
    p = DeconvParam(output_channels=oc, input_channels=ic, input_h=h, input_w=w, kernel_h=kh, kernel_w=kw, stride_h=sh,
                    stride_w=sw, dilation_h=dh, dilation_w=dw, pad_left=pl, pad_right=pr, pad_top=pt, pad_bottom=pb,
                    output_pad_right=opw, output_pad_bottom=oph, group=group, bias_term=int(bool(bias)),
                    activation=int(bool(relu)))
    _check("fcuda_deconv_output_dim", fcuda().fcuda_deconv_output_dim(ctypes.byref(p)))
    return p


def deconv_plan(param: DeconvParam) -> tuple[FcudaConvParam, int]:
    """The equivalent stride-1 convolution and the algorithm it runs with (DEPTHWISE: the direct gather kernel)."""
    eq, algo = FcudaConvParam(), ctypes.c_int(-1)
    _check("fcuda_deconv_plan", fcuda().fcuda_deconv_plan(ctypes.byref(param), ctypes.byref(eq), ctypes.byref(algo)))
    return eq, algo.value


def deconv_forward(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None = None, stride=1, pad=0, output_pad=0,
                   dilation=1, group: int = 1, relu: bool = False) -> tuple[torch.Tensor, int]:
    """ncnn Deconvolution of x (N, IC, H, W) with w (OC, IC/group, KH, KW), not flipped.  Returns (output, conv_algo)."""
    n, ic, h, wd = x.shape
    oc, _, kh, kw = w.shape
    p = deconv_param(oc, ic, h, wd, kh, kw, stride, pad, output_pad, dilation, group, b is not None, relu)
    _, algo = deconv_plan(p)
    lib = fcuda()
    s, k = ctypes.c_size_t(0), ctypes.c_size_t(0)
    _check("fcuda_deconv_get_buffer_size", lib.fcuda_deconv_get_buffer_size(ctypes.byref(p), n, ctypes.byref(s), ctypes.byref(k)))
    packed = torch.empty(max(k.value, 1), device=x.device, dtype=torch.float32)
    scratch = torch.empty(max(s.value, 1), device=x.device, dtype=torch.float32)
    w = w.contiguous()
    _check("fcuda_deconv_init", lib.fcuda_deconv_init(ctypes.byref(p), _ptr(packed), ctypes.c_void_p(w.data_ptr()), _stream()))
    out = torch.empty((n, oc, p.output_h, p.output_w), device=x.device, dtype=torch.float32)
    _check("fcuda_deconv_forward",
           lib.fcuda_deconv_forward(ctypes.byref(p), _ptr(out), _ptr(x.contiguous()), _ptr(packed), _ptr(scratch), _ptr(b), n,
                                    _stream()))
    return out, algo


# ---- resize / crop ---------------------------------------------------------------------------------
INTERP_NEAREST, INTERP_BILINEAR = 1, 2


def interp_param(h: int, w: int, out_h: int, out_w: int, mode: str = "bilinear", align_corners: bool = False,
                 scale=None) -> InterpParam:
    """FcudaInterpParam with output_h / output_w filled.  out_h / out_w are ncnn's output_height / output_width; `scale`
    (a float or (h, w)) sets height_scale / width_scale, which size the output when out_h or out_w is 0."""
    sh, sw = (1.0, 1.0) if scale is None else ((scale, scale) if isinstance(scale, (int, float)) else scale)
    rt = {"nearest": INTERP_NEAREST, "bilinear": INTERP_BILINEAR}.get(mode, mode)
    p = InterpParam(resize_type=rt, align_corner=int(bool(align_corners)), height_scale=sh, width_scale=sw,
                    output_height=out_h, output_width=out_w, input_h=h, input_w=w)
    _check("fcuda_interp_output_dim", fcuda().fcuda_interp_output_dim(ctypes.byref(p)))
    return p


def interp(x: torch.Tensor, out_h: int, out_w: int, mode: str = "bilinear", align_corners: bool = False,
           scale=None) -> torch.Tensor:
    """ncnn Interp of x (N, C, H, W): mode "nearest" (resize_type 1) or "bilinear" (2)."""
    n, c, h, w = x.shape
    p = interp_param(h, w, out_h, out_w, mode, align_corners, scale)
    out = torch.empty((n, c, p.output_h, p.output_w), device=x.device, dtype=torch.float32)
    _check("fcuda_interp_forward",
           fcuda().fcuda_interp_forward(ctypes.byref(p), _ptr(out), _ptr(x.contiguous()), c, n, _stream()))
    return out


def pixel_shuffle(x: torch.Tensor, r: int, mode: int = 0, addend: torch.Tensor | None = None, addend_scale=None,
                  out: torch.Tensor | None = None) -> torch.Tensor:
    """ncnn PixelShuffle of x (N, C, H, W) to (N, C / r^2, H r, W r): mode 0 PyTorch's channel order, 1 ONNX
    DepthToSpace DCR (include/fcuda.h).  With `addend` (N, C / r^2, h, w) its nearest Interp to the output size is added
    in the same pass; `addend_scale` (a float or (h, w), ncnn's Interp scales) maps it, or by default the explicit
    output size."""
    n, c, h, w = x.shape
    amap = None
    if addend is not None:
        ah, aw = addend.shape[2:]
        amap = (interp_param(ah, aw, 0, 0, "nearest", scale=addend_scale) if addend_scale is not None
                else interp_param(ah, aw, h * r, w * r, "nearest"))
        addend = addend.contiguous()
    oc = c // (r * r) if r > 0 else c
    out = torch.empty((n, oc, h * r, w * r), device=x.device, dtype=torch.float32) if out is None else out
    _check("fcuda_pixel_shuffle_forward",
           fcuda().fcuda_pixel_shuffle_forward(_ptr(out), _ptr(x.contiguous()), c, h, w, r, mode,
                                               _ptr(addend) if addend is not None else None,
                                               ctypes.byref(amap) if amap is not None else None, n, _stream()))
    return out


BINARY_OPS = ["ADD", "SUB", "MUL", "DIV", "MAX", "MIN", "POW", "RSUB", "RDIV", "RPOW", "ATAN2", "RATAN2"]  # FcudaBinaryOp


def binary_op_shape(a_rank: int, a_shape, b_rank: int, b_shape):
    """fcuda_binary_op_shape for two images of ncnn ranks a_rank, b_rank stored as (c, h, w): (output rank, output
    (c, h, w), a's and b's extents along the output's axes)."""
    i3 = ctypes.c_int * 3
    rank, out, aa, ba = ctypes.c_int(), i3(), i3(), i3()
    _check("fcuda_binary_op_shape", fcuda().fcuda_binary_op_shape(a_rank, i3(*a_shape), b_rank, i3(*b_shape),
                                                                   ctypes.byref(rank), out, aa, ba))
    return rank.value, tuple(out), tuple(aa), tuple(ba)


def binary_op(a: torch.Tensor, b, op: int, relu: bool = False, out: torch.Tensor | None = None) -> torch.Tensor:
    """ncnn BinaryOp `op` (0..11, BINARY_OPS) of a (N, C, H, W) and b: a tensor of the same rank that broadcasts
    against a on C, H and W (either side may be 1 there; N equal), or a float scalar.  Optional ReLU (include/fcuda.h)."""
    i4 = ctypes.c_int * 4
    if torch.is_tensor(b):
        shape = (a.shape[0],) + tuple(max(x, y) if 1 in (x, y) else x for x, y in zip(a.shape[1:], b.shape[1:]))
        bp, bshape, scalar = _ptr(b.contiguous()), i4(*b.shape), 0.0
    else:
        shape, bp, bshape, scalar = tuple(a.shape), None, None, float(b)
    out = torch.empty(shape, device=a.device, dtype=torch.float32) if out is None else out
    _check("fcuda_binary_op_forward", fcuda().fcuda_binary_op_forward(_ptr(out), _ptr(a.contiguous()), i4(*a.shape), bp,
                                                                      bshape, scalar, op, int(relu), _stream()))
    return out


def crop(x: torch.Tensor, coff: int, hoff: int, woff: int, oc: int, oh: int, ow: int) -> torch.Tensor:
    """out[n][c][y][x] = x[n][c + coff][y + hoff][x + woff], shape (N, oc, oh, ow)."""
    n, c, h, w = x.shape
    out = torch.empty((n, oc, oh, ow), device=x.device, dtype=torch.float32)
    _check("fcuda_crop_forward",
           fcuda().fcuda_crop_forward(_ptr(out), _ptr(x.contiguous()), c, h, w, coff, hoff, woff, oc, oh, ow, n, _stream()))
    return out


# ---- channel routing -------------------------------------------------------------------------------
def route(sources, sizes, group: int = 1, reverse: int = 0, begin: int = 0, axis: int = 1, outs=None) -> list:
    """fcuda_route_forward: `sources` (same shape but along `axis`, a dimension of the (N, ...) tensors) concatenated
    along `axis`, ShuffleChannel(group, reverse) on it, and positions [begin, begin + sum(sizes)) written to one new
    tensor per size (or into `outs`).  At most 8 sources and 8 sizes: one launch."""
    from ._lib import FcudaRoute
    x0 = sources[0]
    shape = list(x0.shape)
    r = FcudaRoute()
    r.outer, r.inner = math.prod(shape[1:axis]), math.prod(shape[axis + 1:])
    r.num_src, r.num_dst = len(sources), len(sizes)
    r.group, r.reverse, r.dst_begin = group, reverse, begin
    if outs is None:
        outs = [torch.empty(shape[:axis] + [s] + shape[axis + 1:], device=x0.device, dtype=torch.float32) for s in sizes]
    for k, x in enumerate(sources[:8]):
        r.src[k], r.src_extent[k] = _ptr(x).value, x.shape[axis]
    for k, (o, s) in enumerate(list(zip(outs, sizes))[:8]):
        r.dst[k], r.dst_extent[k] = _ptr(o).value, s
    _check("fcuda_route_forward", fcuda().fcuda_route_forward(ctypes.byref(r), x0.shape[0], _stream()))
    return outs


def shuffle_channel(x: torch.Tensor, group: int, reverse: int = 0) -> torch.Tensor:
    """ncnn ShuffleChannel of x (N, C, H, W) (include/fcuda.h, fcuda_route_forward)."""
    return route([x.contiguous()], [x.shape[1]], group, reverse)[0]


def slice_plan(shape, axis: int, slices) -> tuple[int, list[int]]:
    """fcuda_slice_plan for one image of ncnn rank len(shape): (storage axis 0..2 of (c, h, w), the tops' sizes)."""
    rank = len(shape)
    chw = (ctypes.c_int * 3)(*([1] * (3 - rank) + list(shape)))
    sl = (ctypes.c_int * len(slices))(*slices)
    sizes = (ctypes.c_int * len(slices))()
    sa = ctypes.c_int()
    _check("fcuda_slice_plan", fcuda().fcuda_slice_plan(rank, axis, chw, sl, len(slices), ctypes.byref(sa), sizes))
    return sa.value, list(sizes)


def slice(x: torch.Tensor, slices, axis: int = 0) -> list:
    """ncnn Slice of x (N, ...), each image of rank x.dim() - 1 (1..3), along ncnn's per-rank `axis`; -233 takes an
    even share of what is left.  One launch per 8 tops."""
    x = x.contiguous()
    sa, sizes = slice_plan(tuple(x.shape[1:]), axis, slices)
    dim = 1 + sa - (4 - x.dim())
    outs, begin = [], 0
    for t0 in range(0, len(sizes), 8):
        outs += route([x], sizes[t0:t0 + 8], begin=begin, axis=dim)
        begin += sum(sizes[t0:t0 + 8])
    return outs


# ---- SSD detection head ----------------------------------------------------------------------------
def permute(x: torch.Tensor, order: int) -> torch.Tensor:
    """ncnn Permute of x (N, C, H, W): order 0 (c,h,w) 1 (c,w,h) 2 (h,c,w) 3 (h,w,c) 4 (w,c,h) 5 (w,h,c)."""
    n, c, h, w = x.shape
    axes = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)][order] if 0 <= order <= 5 else (0, 1, 2)
    d = (c, h, w)
    out = torch.empty((n,) + tuple(d[a] for a in axes), device=x.device, dtype=torch.float32)
    _check("fcuda_permute_forward",
           fcuda().fcuda_permute_forward(_ptr(out), _ptr(x.contiguous()), c, h, w, order, n, _stream()))
    return out


def softmax_axis(x: torch.Tensor, outer: int, length: int, inner: int) -> torch.Tensor:
    """Softmax over the middle axis of each image of x viewed as (N, outer, length, inner)."""
    out = torch.empty_like(x)
    _check("fcuda_softmax_axis_forward",
           fcuda().fcuda_softmax_axis_forward(_ptr(out), _ptr(x.contiguous()), outer, length, inner, x.shape[0], _stream()))
    return out


def priorbox_param(min_sizes, max_sizes=(), aspect_ratios=(), variances=(0.1, 0.1, 0.2, 0.2), flip=True, clip=False,
                   step=(0.0, 0.0), offset=0.5) -> PriorBoxParam:
    """FcudaPriorBoxParam; step (w, h) <= 0 derives the step from the image and feature sizes."""
    p = PriorBoxParam()
    p.num_min_sizes, p.num_max_sizes, p.num_aspect_ratios = len(min_sizes), len(max_sizes), len(aspect_ratios)
    for dst, src in ((p.min_sizes, min_sizes), (p.max_sizes, max_sizes), (p.aspect_ratios, aspect_ratios),
                     (p.variances, variances)):
        for k, v in enumerate(list(src)[:len(dst)]):
            dst[k] = float(v)
    p.flip, p.clip = int(bool(flip)), int(bool(clip))
    p.step_w, p.step_h = float(step[0]), float(step[1])
    p.offset = float(offset)
    return p


def priorbox_per_location(p: PriorBoxParam) -> int:
    n = ctypes.c_int(0)
    _check("fcuda_priorbox_per_location", fcuda().fcuda_priorbox_per_location(ctypes.byref(p), ctypes.byref(n)))
    return n.value


def priorbox(p: PriorBoxParam, feat_w: int, feat_h: int, img_w: int, img_h: int, device="cuda") -> torch.Tensor:
    """(2, 4 * P) priors: row 0 the boxes, row 1 the variances."""
    num = feat_w * feat_h * priorbox_per_location(p)
    out = torch.empty((2, 4 * num), device=device, dtype=torch.float32)
    _check("fcuda_priorbox_forward",
           fcuda().fcuda_priorbox_forward(_ptr(out), ctypes.byref(p), feat_w, feat_h, img_w, img_h, _stream()))
    return out


def ssd_decode(loc: torch.Tensor, priors: torch.Tensor) -> torch.Tensor:
    """loc (N, 4P), priors (2, 4P) -> boxes (N, P, 4) as (xmin, ymin, xmax, ymax)."""
    n = loc.shape[0]
    num = priors.shape[-1] // 4
    out = torch.empty((n, num, 4), device=loc.device, dtype=torch.float32)
    _check("fcuda_ssd_decode", fcuda().fcuda_ssd_decode(_ptr(out), _ptr(loc.contiguous()), _ptr(priors.contiguous()), num, n,
                                                        _stream()))
    return out


def detection_output(loc: torch.Tensor, conf: torch.Tensor, priors: torch.Tensor, num_classes: int,
                     conf_threshold: float = 0.5, nms_threshold: float = 0.05, nms_top_k: int = 300,
                     keep_top_k: int = 100) -> torch.Tensor:
    """loc (N, 4P), conf (N, P * C), priors (2, 4P) -> (N, keep_top_k, 6) rows [label, score, xmin, ymin, xmax, ymax]."""
    lib = fcuda()
    n = loc.shape[0]
    num = priors.shape[-1] // 4
    ws = ctypes.c_size_t(0)
    _check("fcuda_detection_output_workspace_size",
           lib.fcuda_detection_output_workspace_size(num, num_classes, nms_top_k, n, ctypes.byref(ws)))
    workspace = torch.empty(max(ws.value, 1), device=loc.device, dtype=torch.float32)
    out = torch.empty((n, keep_top_k, 6), device=loc.device, dtype=torch.float32)
    _check("fcuda_detection_output_forward",
           lib.fcuda_detection_output_forward(_ptr(out), _ptr(loc.contiguous()), _ptr(conf.contiguous()),
                                              _ptr(priors.contiguous()), num, num_classes, float(conf_threshold),
                                              float(nms_threshold), nms_top_k, keep_top_k, _ptr(workspace), n, _stream()))
    return out


# ---- YOLO detection head ---------------------------------------------------------------------------
def yolo_param(version: int, num_class: int, num_box: int, grids, biases, mask=(), anchors_scale=(),
               confidence_threshold: float = 0.01, nms_threshold: float = 0.45, nms_top_k: int = 1024,
               keep_top_k: int = 1024) -> YoloParam:
    """FcudaYoloParam: version 2 (YoloDetectionOutput) or 3 (Yolov3DetectionOutput); grids = [(h, w)] per scale."""
    p = YoloParam()
    p.version, p.num_class, p.num_box, p.num_scales = version, num_class, num_box, len(grids)
    p.confidence_threshold, p.nms_threshold = float(confidence_threshold), float(nms_threshold)
    p.nms_top_k, p.keep_top_k, p.num_biases = nms_top_k, keep_top_k, len(biases)
    for dst, src in ((p.biases, biases), (p.mask, mask), (p.anchors_scale, anchors_scale),
                     (p.grid_h, [g[0] for g in grids]), (p.grid_w, [g[1] for g in grids])):
        for k, v in enumerate(list(src)[:len(dst)]):
            dst[k] = v
    return p


def _yolo_inputs(inputs, p: YoloParam):
    """The inputs as the C side reads them: p.num_scales float32 CUDA tensors of one batch, scale b shaped
    (N, num_box * (5 + num_class), grid_h[b], grid_w[b])."""
    xs = [x.contiguous() for x in inputs]
    assert len(xs) == p.num_scales >= 1, (len(xs), p.num_scales)
    n = xs[0].shape[0]
    for b, x in enumerate(xs):
        want = (n, p.num_box * (5 + p.num_class), p.grid_h[b], p.grid_w[b])
        assert x.is_cuda and x.dtype == torch.float32 and tuple(x.shape) == want, (b, tuple(x.shape), want)
    arr = (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
    return xs, arr


def yolo_decode(inputs, p: YoloParam):
    """inputs: one (N, num_box * (5 + C), h, w) tensor per scale -> (scores (N, S), classes (N, S) int32,
    boxes (N, S, 4)) for every slot S, candidate or not."""
    xs, arr = _yolo_inputs(inputs, p)
    n = xs[0].shape[0]
    slots = sum(p.num_box * x.shape[2] * x.shape[3] for x in xs)
    scores = torch.empty((n, slots), device=xs[0].device, dtype=torch.float32)
    classes = torch.empty((n, slots), device=xs[0].device, dtype=torch.int32)
    boxes = torch.empty((n, slots, 4), device=xs[0].device, dtype=torch.float32)
    _check("fcuda_yolo_decode", fcuda().fcuda_yolo_decode(_ptr(scores), ctypes.c_void_p(classes.data_ptr()), _ptr(boxes),
                                                          arr, ctypes.byref(p), n, _stream()))
    return scores, classes, boxes


def yolo_detection(inputs, p: YoloParam) -> torch.Tensor:
    """inputs as yolo_decode -> (N, keep_top_k, 6) rows [class + 1, confidence, xmin, ymin, xmax, ymax]."""
    lib = fcuda()
    xs, arr = _yolo_inputs(inputs, p)
    n = xs[0].shape[0]
    ws = ctypes.c_size_t(0)
    _check("fcuda_yolo_detection_workspace_size", lib.fcuda_yolo_detection_workspace_size(ctypes.byref(p), n,
                                                                                          ctypes.byref(ws)))
    workspace = torch.empty(max(ws.value, 1), device=xs[0].device, dtype=torch.float32)
    out = torch.empty((n, p.keep_top_k, 6), device=xs[0].device, dtype=torch.float32)
    _check("fcuda_yolo_detection_forward", lib.fcuda_yolo_detection_forward(_ptr(out), arr, ctypes.byref(p),
                                                                            _ptr(workspace), n, _stream()))
    return out


# ---- other layer entry points (thin wrappers used by the parity tests) ------------------------------
def inner_product(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, relu: bool = False) -> torch.Tensor:
    lib = fcuda()
    n = x.shape[0]
    in_size = x[0].numel()
    out_size = w.shape[0]
    s, k = ctypes.c_size_t(0), ctypes.c_size_t(0)
    _check("fcuda_inner_product_get_buffer_size",
           lib.fcuda_inner_product_get_buffer_size(in_size, out_size, n, ctypes.byref(s), ctypes.byref(k)))
    packed = torch.empty(max(k.value, 1), device=x.device)
    scratch = torch.empty(max(s.value, 1), device=x.device)
    _check("fcuda_inner_product_init", lib.fcuda_inner_product_init(in_size, out_size, _ptr(packed), _ptr(w.contiguous()), _stream()))
    out = torch.empty((n, out_size), device=x.device)
    _check("fcuda_inner_product_forward",
           lib.fcuda_inner_product_forward(in_size, out_size, _ptr(out), _ptr(x.contiguous()), _ptr(packed), _ptr(b),
                                           _ptr(scratch), int(relu), n, _stream()))
    return out


def eltwise(a: torch.Tensor, b: torch.Tensor, op: int, ca: float = 1.0, cb: float = 1.0, relu: bool = False) -> torch.Tensor:
    """op 0 PROD, 1 SUM (with coefficients), 2 MAX — ncnn Eltwise semantics (the reference only has plain SUM)."""
    out = torch.empty_like(a)
    _check("fcuda_eltwise_forward",
           fcuda().fcuda_eltwise_forward(_ptr(out), _ptr(a.contiguous()), _ptr(b.contiguous()), a.numel(), op, ca, cb,
                                         int(relu), _stream()))
    return out


PIXEL_RGB, PIXEL_BGR, PIXEL_GRAY, PIXEL_RGBA = 1, 2, 4, 8  # ncnn pixel types (mat.h:126-129); conversion = from | (to << 16)


def from_pixels(pixels: torch.Tensor, type_: int, target_w: int = 0, target_h: int = 0, mean=None, norm=None) -> torch.Tensor:
    """(N, h, w[, c]) uint8 CUDA tensor -> (N, C, th, tw) fp32: from_pixels[_resize] + substract_mean_normalize on the GPU."""
    import numpy as np
    lib = fcuda()
    assert pixels.is_cuda and pixels.dtype == torch.uint8 and pixels.is_contiguous()
    n, h, w = pixels.shape[:3]
    sc, oc = ctypes.c_int(), ctypes.c_int()
    _check("fcuda_pixel_channels", lib.fcuda_pixel_channels(type_, ctypes.byref(sc), ctypes.byref(oc)))
    assert pixels[0].numel() == h * w * sc.value
    tw, th = target_w or w, target_h or h
    out = torch.empty((n, oc.value, th, tw), device=pixels.device, dtype=torch.float32)
    fp = ctypes.POINTER(ctypes.c_float)
    m = None if mean is None else np.ascontiguousarray(mean, np.float32)
    s = None if norm is None else np.ascontiguousarray(norm, np.float32)
    _check("fcuda_from_pixels",
           lib.fcuda_from_pixels(_ptr(out), ctypes.c_void_p(pixels.data_ptr()), type_, w, h, tw, th,
                                 None if m is None else m.ctypes.data_as(fp), None if s is None else s.ctypes.data_as(fp), n,
                                 _stream()))
    return out


def pooling(x: torch.Tensor, type_: int, kh, kw, sh, sw, pl, pr, pt, pb, global_pooling=False) -> torch.Tensor:
    lib = fcuda()
    n, c, h, w = x.shape
    if global_pooling:
        oh = ow = 1
    else:
        oh = lib.fcuda_pooling_out_dim(h, pt, pb, kh, sh)
        ow = lib.fcuda_pooling_out_dim(w, pl, pr, kw, sw)
    out = torch.empty((n, c, oh, ow), device=x.device)
    _check("fcuda_pooling_forward",
           lib.fcuda_pooling_forward(_ptr(out), _ptr(x.contiguous()), c, h, w, type_, kh, kw, sh, sw, pl, pr, pt, pb,
                                     int(global_pooling), n, _stream()))
    return out


def batchnorm(x, alpha, beta, scale=None, scale_bias=None, relu=False):
    n, c = x.shape[:2]
    out = torch.empty_like(x)
    _check("fcuda_batchnorm_forward",
           fcuda().fcuda_batchnorm_forward(_ptr(out), _ptr(x.contiguous()), c, x[0, 0].numel(), _ptr(alpha), _ptr(beta),
                                           _ptr(scale), _ptr(scale_bias), int(relu), n, _stream()))
    return out


def scale(x, s, b=None):
    n, c = x.shape[:2]
    out = torch.empty_like(x)
    _check("fcuda_scale_forward",
           fcuda().fcuda_scale_forward(_ptr(out), _ptr(x.contiguous()), c, x[0, 0].numel(), _ptr(s), _ptr(b), n, _stream()))
    return out


def eltwise_add(a, b, relu=False):
    out = torch.empty_like(a)
    _check("fcuda_eltwise_add_forward",
           fcuda().fcuda_eltwise_add_forward(_ptr(out), _ptr(a.contiguous()), _ptr(b.contiguous()), a.numel(), int(relu), _stream()))
    return out


def relu(x):
    out = torch.empty_like(x)
    _check("fcuda_relu_forward", fcuda().fcuda_relu_forward(_ptr(out), _ptr(x.contiguous()), x.numel(), _stream()))
    return out


def clip(x, lo, hi, out=None):
    """ncnn Clip: min(max(x, lo), hi), NaN -> lo.  `out` may be `x` (in place)."""
    out = torch.empty_like(x) if out is None else out
    _check("fcuda_clip_forward",
           fcuda().fcuda_clip_forward(_ptr(out), _ptr(x.contiguous()), x.numel(), float(lo), float(hi), _stream()))
    return out


ACTIVATIONS = ["Sigmoid", "TanH", "Swish", "HardSigmoid", "HardSwish"]  # FcudaActivationType, ncnn's layer type names
GELU_TYPES = {"GELU": 6, "GELU_TANH": 7}  # FcudaActivationType of GELU with fast_gelu 0 / 1


def activation(x, kind, alpha: float = 0.2, beta: float = 0.5, out=None):
    """ncnn activation `kind` (an FcudaActivationType, a name of ACTIVATIONS, or "GELU" / "GELU_TANH") over every
    element of x; alpha / beta are read by HardSigmoid / HardSwish only (ncnn's defaults 0.2 / 0.5).  `out` may be `x`
    (in place).  Definitions, roundings and bounds: include/fcuda.h."""
    if isinstance(kind, str):
        kind = GELU_TYPES[kind] if kind in GELU_TYPES else ACTIVATIONS.index(kind)
    kind = int(kind)
    out = torch.empty_like(x) if out is None else out
    _check("fcuda_activation_forward", fcuda().fcuda_activation_forward(_ptr(out), _ptr(x.contiguous()), x.numel(), kind,
                                                                        float(alpha), float(beta), _stream()))
    return out


def prelu(x, slope, out=None):
    """ncnn PReLU over (N, C, ...): x < 0 ? x * slope[c] : x; a one-element `slope` is shared.  `out` may be `x`."""
    n, c = x.shape[:2]
    out = torch.empty_like(x) if out is None else out
    _check("fcuda_prelu_forward",
           fcuda().fcuda_prelu_forward(_ptr(out), _ptr(x.contiguous()), c, x[0, 0].numel(), _ptr(slope), slope.numel(), n,
                                       _stream()))
    return out


def normalize(x, scale, across_spatial=0, across_channel=1, eps=1e-4, eps_mode=0, out=None):
    """ncnn Normalize over (N, C, ...): y = (x * a) * scale[c], a from the sum of squares over each pixel's channels
    (across_spatial 0), the whole image (1, 1) or each channel plane (1, 0); a one-element `scale` is shared
    (include/fcuda.h).  The workspace comes from torch.  `out` may be `x`."""
    lib = fcuda()
    n, c = x.shape[:2]
    plane = x[0, 0].numel()
    ws = ctypes.c_size_t(0)
    _check("fcuda_normalize_workspace_size",
           lib.fcuda_normalize_workspace_size(int(across_spatial), int(across_channel), c, plane, n, ctypes.byref(ws)))
    workspace = torch.empty(ws.value, device=x.device, dtype=torch.float32) if ws.value else None
    out = torch.empty_like(x) if out is None else out
    _check("fcuda_normalize_forward",
           lib.fcuda_normalize_forward(_ptr(out), _ptr(x.contiguous()), c, plane, _ptr(scale.contiguous()), scale.numel(),
                                       int(across_spatial), int(across_channel), float(eps), int(eps_mode),
                                       _ptr(workspace), n, _stream()))
    return out


def _pad(top, bottom, left, right, type_, value) -> FcudaPad:
    return FcudaPad(int(top), int(bottom), int(left), int(right), int(type_), float(value))


def _padded_shape(x, p: FcudaPad | None):
    n, c, h, w = x.shape
    return (n, c, h + p.top + p.bottom, w + p.left + p.right) if p is not None else (n, c, h, w)


def instance_norm(x, gamma, beta, eps, relu=False, pad=None, out=None):
    """ncnn InstanceNorm over (N, C, H, W): y = fmaf(x, a, b) per plane from its mean and biased variance, a ReLU with
    `relu`, and with `pad` = (top, bottom, left, right, type, value) the output plane padded in the same pass
    (include/fcuda.h).  gamma = beta = None: affine 0.  The workspace comes from torch.  `out` may be `x` when unpadded."""
    lib = fcuda()
    assert x.dim() == 4, x.shape
    n, c, h, w = x.shape
    p = _pad(*pad) if pad is not None else None
    ws = ctypes.c_size_t(0)
    _check("fcuda_instance_norm_workspace_size", lib.fcuda_instance_norm_workspace_size(c, h * w, n, ctypes.byref(ws)))
    workspace = torch.empty(ws.value, device=x.device, dtype=torch.float32)
    out = torch.empty(_padded_shape(x, p), device=x.device, dtype=torch.float32) if out is None else out
    assert tuple(out.shape) == _padded_shape(x, p), (out.shape, x.shape)
    _check("fcuda_instance_norm_forward",
           lib.fcuda_instance_norm_forward(_ptr(out), _ptr(x), c, h, w,
                                           _ptr(gamma.contiguous()) if gamma is not None else None,
                                           _ptr(beta.contiguous()) if beta is not None else None, float(eps), int(relu),
                                           ctypes.byref(p) if p is not None else None, _ptr(workspace), n, _stream()))
    return out


def layer_norm(x, n, gamma=None, beta=None, eps=1e-3, out=None):
    """ncnn LayerNorm: every run of n contiguous floats of x (a row, or a channel plane) normalised with its mean and
    biased variance, then * gamma + beta (n floats each, or both None).  `out` may be `x`.  Rounding order and bound:
    include/fcuda.h."""
    assert x.numel() % n == 0, (x.shape, n)
    out = torch.empty_like(x) if out is None else out
    _check("fcuda_layer_norm_forward",
           fcuda().fcuda_layer_norm_forward(_ptr(out), _ptr(x.contiguous()), int(n), x.numel() // n,
                                            _ptr(gamma.contiguous()) if gamma is not None else None,
                                            _ptr(beta.contiguous()) if beta is not None else None, float(eps),
                                            _stream()))
    return out


def attention(q, k, v, heads, scale=None, out=None):
    """Scaled dot-product attention per head of fcuda_attention_forward.  q (N, Lq, >= E), k and v (N, Lk, >= E), each
    with unit stride in its last dimension and any row stride (a slice of a fused [N, L, 3E] projection is read in
    place); E = heads * head_dim is taken from `out`'s width, or q's when `out` is None.  Returns (N, Lq, E).  scale
    defaults to 1 / sqrt(head_dim)."""
    n, lq = q.shape[:2]
    lk = k.shape[1]
    e = out.shape[2] if out is not None else q.shape[2]
    d = e // heads
    scale = 1.0 / math.sqrt(d) if scale is None else scale
    for t in (q, k, v):  # row-strided: a column slice of a contiguous buffer is read in place
        assert t.is_cuda and t.dtype == torch.float32, (t.device, t.dtype)
        assert t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1), t.stride()
    rows = [ctypes.c_void_p(t.data_ptr()) for t in (q, k, v)]
    out = torch.empty((n, lq, e), device=q.device, dtype=torch.float32) if out is None else out
    _check("fcuda_attention_forward",
           fcuda().fcuda_attention_forward(_ptr(out), rows[0], q.stride(1), rows[1], k.stride(1), rows[2], v.stride(1),
                                           n, heads, d, lq, lk, float(scale), _stream()))
    return out


def padding(x, top, bottom, left, right, type=0, value=0.0, out=None):
    """ncnn Padding of every (N, C) plane of x: type 0 constant `value`, 1 replicate, 2 reflect (include/fcuda.h)."""
    p = _pad(top, bottom, left, right, type, value)
    n, c, h, w = x.shape
    out = torch.empty(_padded_shape(x, p), device=x.device, dtype=torch.float32) if out is None else out
    assert tuple(out.shape) == _padded_shape(x, p), (out.shape, x.shape)
    _check("fcuda_padding_forward",
           fcuda().fcuda_padding_forward(_ptr(out), _ptr(x), c, h, w, ctypes.byref(p), n, _stream()))
    return out


def lrn(x, region_type=0, local_size=5, alpha=1.0, beta=0.75, bias=1.0, out=None):
    """ncnn LRN over (N, C, H, W): y = x * (bias + alpha / n * ss)^-beta, ss the sum of squares over `local_size`
    neighbouring channels (region_type 0) or a local_size x local_size window of the plane (1; n = local_size^2)
    (include/fcuda.h).  Out of place: `out` may not be `x`."""
    n, c, h, w = x.shape
    x = x.contiguous()
    out = torch.empty_like(x) if out is None else out
    _check("fcuda_lrn_forward",
           fcuda().fcuda_lrn_forward(_ptr(out), _ptr(x), c, h, w, int(region_type), int(local_size), float(alpha),
                                     float(beta), float(bias), n, _stream()))
    return out


def softmax(x):
    out = torch.empty_like(x)
    _check("fcuda_softmax_forward",
           fcuda().fcuda_softmax_forward(_ptr(out), _ptr(x.contiguous()), x[0].numel(), x.shape[0], _stream()))
    return out


def dropout(x, s):
    out = torch.empty_like(x)
    _check("fcuda_dropout_forward", fcuda().fcuda_dropout_forward(_ptr(out), _ptr(x.contiguous()), x.numel(), float(s), _stream()))
    return out


def tensor_gemm(a: torch.Tensor, b: torch.Tensor, x3: bool = True) -> torch.Tensor:
    """D[g] = A[g] @ B[g]^T with A (G, M, K), B (G, N, K) — the raw TensorGEMM (a8 in SURVEY.md §8)."""
    lib = fcuda()
    g, m, k = a.shape
    n = b.shape[1]
    a = a.contiguous(); b = b.contiguous()
    d = torch.empty((g, m, n), device=a.device)
    if x3:  # A is split inside the kernel (registers); B carries its hi / lo planes
        bh, bl = torch.empty_like(b), torch.empty_like(b)
        _check("fcuda_split_tf32", lib.fcuda_split_tf32(_ptr(bh), _ptr(bl), _ptr(b), b.numel(), _stream()))
        _check("fcuda_tensor_gemm", lib.fcuda_tensor_gemm(_ptr(d), _ptr(a), _ptr(bh), _ptr(bl), m, n, k, g, _stream()))
    else:
        _check("fcuda_tensor_gemm", lib.fcuda_tensor_gemm(_ptr(d), _ptr(a), _ptr(b), None, m, n, k, g, _stream()))
    return d


# ---- Faster R-CNN: Proposal and ROIPooling ------------------------------------------------------------------------
PROPOSAL_ANCHORS = 9


def proposal_param(feat_stride: int = 16, base_size: int = 16, pre_nms_topN: int = 6000, after_nms_topN: int = 300,
                   nms_thresh: float = 0.7, min_size: int = 16) -> ProposalParam:
    """FcudaProposalParam with ncnn's defaults."""
    p = ProposalParam()
    p.feat_stride, p.base_size, p.pre_nms_topN, p.after_nms_topN = feat_stride, base_size, pre_nms_topN, after_nms_topN
    p.nms_thresh, p.min_size = float(nms_thresh), min_size
    return p


def proposal_anchors(p: ProposalParam) -> list[tuple[float, float, float, float]]:
    """The 9 anchors of p as (ax1, ay1, aw, ah), from the library."""
    table = (ctypes.c_float * (4 * PROPOSAL_ANCHORS))()
    _check("fcuda_proposal_anchors", fcuda().fcuda_proposal_anchors(ctypes.byref(p), table))
    return [tuple(table[4 * q:4 * q + 4]) for q in range(PROPOSAL_ANCHORS)]


def _proposal_inputs(score: torch.Tensor, bbox: torch.Tensor, im_info: torch.Tensor):
    """The bottoms as the C side reads them: float32 CUDA tensors of one batch, score (N, 18, H, W), bbox (N, 36, H, W),
    im_info 3 values per image."""
    score, bbox, im_info = score.contiguous(), bbox.contiguous(), im_info.contiguous()
    for t in (score, bbox, im_info):
        assert t.is_cuda and t.dtype == torch.float32, (t.device, t.dtype)
    assert score.dim() == 4 and score.shape[1] == 2 * PROPOSAL_ANCHORS, tuple(score.shape)
    n, _, h, w = score.shape
    assert tuple(bbox.shape) == (n, 4 * PROPOSAL_ANCHORS, h, w), (tuple(bbox.shape), tuple(score.shape))
    assert im_info.shape[0] == n and im_info.numel() == 3 * n, tuple(im_info.shape)
    return score, bbox, im_info, n, h, w


def proposal_decode(score: torch.Tensor, bbox: torch.Tensor, im_info: torch.Tensor, p: ProposalParam) -> torch.Tensor:
    """-> (N, 9 * H * W, 4) clipped boxes of every anchor and cell, index q * H * W + y * W + x, candidate or not."""
    score, bbox, im_info, n, h, w = _proposal_inputs(score, bbox, im_info)
    boxes = torch.empty((n, PROPOSAL_ANCHORS * h * w, 4), device=score.device, dtype=torch.float32)
    _check("fcuda_proposal_decode", fcuda().fcuda_proposal_decode(_ptr(boxes), _ptr(score), _ptr(bbox), _ptr(im_info),
                                                                  ctypes.byref(p), h, w, n, _stream()))
    return boxes


def proposal(score: torch.Tensor, bbox: torch.Tensor, im_info: torch.Tensor, p: ProposalParam):
    """-> (rois (N, after_nms_topN, 4) [x1, y1, x2, y2], zero rows past each image's count; scores (N, after_nms_topN),
    -1 past the count)."""
    lib = fcuda()
    score, bbox, im_info, n, h, w = _proposal_inputs(score, bbox, im_info)
    ws = ctypes.c_size_t(0)
    _check("fcuda_proposal_workspace_size", lib.fcuda_proposal_workspace_size(ctypes.byref(p), h, w, n, ctypes.byref(ws)))
    workspace = torch.empty(max(ws.value, 1), device=score.device, dtype=torch.float32)
    rois = torch.empty((n, p.after_nms_topN, 4), device=score.device, dtype=torch.float32)
    scores = torch.empty((n, p.after_nms_topN), device=score.device, dtype=torch.float32)
    _check("fcuda_proposal_forward", lib.fcuda_proposal_forward(_ptr(rois), _ptr(scores), _ptr(score), _ptr(bbox),
                                                                _ptr(im_info), ctypes.byref(p), h, w, _ptr(workspace), n,
                                                                _stream()))
    return rois, scores


def _roi_inputs(x: torch.Tensor, rois: torch.Tensor):
    """The bottoms as the C side reads them: float32 CUDA tensors, x (N, C, H, W) and rois (N, R, 4) or (N, R, 1, 4)."""
    x, rois = x.contiguous(), rois.contiguous()
    for t in (x, rois):
        assert t.is_cuda and t.dtype == torch.float32, (t.device, t.dtype)
    assert x.dim() == 4 and rois.shape[0] == x.shape[0] and rois.shape[-1] == 4 and rois.dim() in (3, 4), \
        (tuple(x.shape), tuple(rois.shape))
    n, c, h, w = x.shape
    r = rois.shape[1]
    assert rois.numel() == 4 * n * r, tuple(rois.shape)
    return x, rois, n, c, h, w, r


def roi_pooling(x: torch.Tensor, rois: torch.Tensor, pooled_h: int = 7, pooled_w: int = 7,
                spatial_scale: float = 0.0625) -> torch.Tensor:
    """x (N, C, H, W), rois (N, R, 4) or (N, R, 1, 4) -> (N * R, C, pooled_h, pooled_w); RoI r of image n pools image n."""
    x, rois, n, c, h, w, r = _roi_inputs(x, rois)
    out = torch.empty((n * r, c, pooled_h, pooled_w), device=x.device, dtype=torch.float32)
    _check("fcuda_roi_pooling_forward", fcuda().fcuda_roi_pooling_forward(_ptr(out), _ptr(x), _ptr(rois), c, h, w, r,
                                                                          pooled_h, pooled_w, float(spatial_scale), n,
                                                                          _stream()))
    return out


def psroi_pooling(x: torch.Tensor, rois: torch.Tensor, pooled_h: int = 7, pooled_w: int = 7, output_dim: int = 21,
                  spatial_scale: float = 0.0625) -> torch.Tensor:
    """R-FCN's position-sensitive RoI average pooling: x (N, output_dim * pooled_h * pooled_w, H, W), rois (N, R, 4) or
    (N, R, 1, 4) -> (N * R, output_dim, pooled_h, pooled_w); RoI r of image n pools image n."""
    x, rois, n, c, h, w, r = _roi_inputs(x, rois)
    out = torch.empty((n * r, output_dim, pooled_h, pooled_w), device=x.device, dtype=torch.float32)
    _check("fcuda_psroi_pooling_forward", fcuda().fcuda_psroi_pooling_forward(_ptr(out), _ptr(x), _ptr(rois), c, h, w, r,
                                                                              pooled_h, pooled_w, output_dim,
                                                                              float(spatial_scale), n, _stream()))
    return out
