"""Synthetic ncnn-format (.param/.bin) model writer.

The reference snapshot loads ncnn ``.param`` (text, magic 7767517) + ``.bin`` (4-byte flag + fp32 for
weight blobs, raw fp32 for bias/BN/Scale blobs) — /root/reference/src/net.cpp:68-230,
/root/reference/src/ncnn/modelbin.cpp:47-197.  Its own converter (``tools/``) is absent from the
snapshot, and there is no network for pretrained checkpoints, so benchmarks and tests use random-init
models of the architectures BASELINE.json names: a single 3x3 conv, VGG-16, ResNet-50 (Caffe topology:
BN + Scale + ReLU as separate layers, Split/Eltwise residuals), MobileNet-v1, MobileNet-v2 (ReLU6 as Clip), GoogLeNet and
AlexNet (BVLC's deploy nets, with LRN), plus a small "mini" net
that exercises every layer type, single-shot detectors (MobileNet-SSD, VGG-SSD 300, a two-head tiny SSD), YOLO detectors
(MobileNet-YOLOv2, MobileNet-v2 YOLOv3, a two-scale tiny YOLOv3), two-stage detectors (py-faster-rcnn's VGG-16 Faster
R-CNN, py-R-FCN's ResNet-50 R-FCN and a tiny one of each), fast neural style transfer (TransformerNet, with a tiny
one), super-resolution (Real-ESRGAN's SRVGGNetCompact and EDSR baseline, with a tiny PixelShuffle net, and ESPCN), ShuffleNet-v2
with a small routing probe net, and the nets of ncnn's activation layers (MobileNet-v3 Large / Small and EfficientNet-B0
in torchvision's layouts, with a small squeeze-and-excitation net), and Vision Transformers (ViT-B/16, ViT-S/16 and
ViT-Ti/16 in torchvision's layout, with a tiny one).  Weight
statistics follow SURVEY.md §8(d).
"""
from __future__ import annotations

import math
import struct
from pathlib import Path

import numpy as np


class ModelWriter:
    def __init__(self, seed: int = 0, wide_stats: bool = False, adds: str = "eltwise"):
        assert adds in ("eltwise", "binaryop"), adds
        self.rng = np.random.default_rng(seed)
        self.adds = adds  # how add() writes a two-input sum: Caffe's Eltwise SUM, or BinaryOp ADD as onnx2ncnn / pnnx do
        self.wide_stats = wide_stats       # BatchNorm / Scale statistics of _batchnorm_wide (default: mild, near identity)
        self._bn_mul: dict[str, np.ndarray] = {}
        self.lines: list[str] = []
        self.blobs: set[str] = set()
        self.bin = bytearray()
        self.flops = 0.0  # direct-conv FLOPs per image, booster.h:145-148 convention
        self.rank: dict[str, int] = {}  # ncnn rank of a blob (1, 2 or 3; absent = 3); shape stays (c, h, w) storage

    # ---- low level ---------------------------------------------------------------------------
    def _layer(self, type_: str, name: str, bottoms: list[str], tops: list[str], params: dict | None = None):
        kv = " ".join(f"{k}={v}" for k, v in (params or {}).items())
        self.lines.append(f"{type_} {name} {len(bottoms)} {len(tops)} {' '.join(bottoms + tops)} {kv}".rstrip())
        self.blobs.update(tops)

    def _weights(self, a: np.ndarray, flagged: bool):
        if flagged:
            self.bin += struct.pack("<I", 0)  # raw fp32 tag
        self.bin += np.ascontiguousarray(a, np.float32).tobytes()

    # ---- layers ------------------------------------------------------------------------------
    def input(self, name="data", c=3, h=224, w=224):
        self._layer("Input", name, [], [name], {0: w, 1: h, 2: c})
        self.shape = {name: (c, h, w)}
        return name

    def conv(self, name, bottom, oc, k, stride=1, pad=0, bias=True, group=1, top=None, gain=None, dilation=1,
             bias_values=None):
        """bias_values: the bias as given instead of uniform(-0.1, 0.1) draws."""
        top = top or name
        ic, h, w = self.shape[bottom]
        icg = ic // group
        fan_in = icg * k * k
        std = np.sqrt(2.0 / fan_in) if gain is None else gain
        wts = (self.rng.standard_normal((oc, icg, k, k)) * std).astype(np.float32)
        ltype = "ConvolutionDepthWise" if group > 1 else "Convolution"
        params = {0: oc, 1: k, 3: stride, 4: pad, 5: int(bias), 6: wts.size}
        if group > 1:
            params[7] = group
        if dilation > 1:
            params[2] = dilation
        self._layer(ltype, name, [bottom], [top], params)
        self._weights(wts, True)
        if bias and bias_values is not None:
            self._weights(np.asarray(bias_values, np.float32).reshape(oc), False)
        elif bias:
            self._weights(self.rng.uniform(-0.1, 0.1, oc).astype(np.float32), False)
        oh = (h + 2 * pad - dilation * (k - 1) - 1) // stride + 1
        ow = (w + 2 * pad - dilation * (k - 1) - 1) // stride + 1
        self.shape[top] = (oc, oh, ow)
        self.flops += 2.0 * oc * icg * oh * ow * k * k
        return top

    def deconv(self, name, bottom, oc, k, stride=1, pad=0, bias=True, group=1, top=None, weights=None):
        """ncnn Deconvolution (DeconvolutionDepthWise when group > 1): weights [group][oc/group][ic/group][k][k], He init
        over the k*k/stride^2 taps that reach one output, or `weights` as given."""
        top = top or name
        ic, h, w = self.shape[bottom]
        icg = ic // group
        if weights is None:
            std = np.sqrt(2.0 * stride * stride / (icg * k * k))
            weights = self.rng.standard_normal((oc, icg, k, k)) * std
        wts = np.ascontiguousarray(weights, np.float32)
        assert wts.shape == (oc, icg, k, k), wts.shape
        ltype = "DeconvolutionDepthWise" if group > 1 else "Deconvolution"
        params = {0: oc, 1: k, 3: stride, 4: pad, 5: int(bias), 6: wts.size}
        if group > 1:
            params[7] = group
        self._layer(ltype, name, [bottom], [top], params)
        self._weights(wts, True)
        if bias:
            self._weights(self.rng.uniform(-0.1, 0.1, oc).astype(np.float32), False)
        self.shape[top] = (oc, (h - 1) * stride + k - 2 * pad, (w - 1) * stride + k - 2 * pad)
        self.flops += 2.0 * ic * (oc // group) * h * w * k * k
        return top

    def relu(self, name, bottom, top=None):
        top = top or name
        self._layer("ReLU", name, [bottom], [top])
        self.shape[top] = self.shape[bottom]
        return top

    def clip(self, name, bottom, lo=0.0, hi=6.0, top=None):
        """ncnn Clip 0=min 1=max (Caffe's ReLU6 is Clip 0..6)."""
        top = top or name
        self._layer("Clip", name, [bottom], [top], {0: f"{lo:e}", 1: f"{hi:e}"})
        self.shape[top] = self.shape[bottom]
        return top

    def prelu(self, name, bottom, shared=False, top=None, slopes=None):
        """ncnn PReLU 0=num_slope: one slope per channel (or one for all when `shared`), raw fp32 in the bin."""
        top = top or name
        c = self.shape[bottom][0]
        n = 1 if shared else c
        if slopes is None:
            slopes = self.rng.uniform(0.05, 0.3, n)
        slopes = np.ascontiguousarray(slopes, np.float32)
        assert slopes.shape == (n,), slopes.shape
        self._layer("PReLU", name, [bottom], [top], {0: n})
        self._weights(slopes, False)
        self.shape[top] = self.shape[bottom]
        return top

    def normalize(self, name, bottom, across_spatial=0, channel_shared=0, eps=1e-10, scale=20.0, across_channel=1,
                  eps_mode=0, top=None):
        """ncnn Normalize 0=across_spatial 1=channel_shared 2=eps 3=scale_data_size (4=across_channel, 9=eps_mode only
        when not the defaults 1 / 0); the scales, raw fp32 in the bin, are all `scale` (SSD's initial value) or the array
        given."""
        top = top or name
        c = self.shape[bottom][0]
        n = 1 if channel_shared else c
        scales = np.ascontiguousarray(np.broadcast_to(np.asarray(scale, np.float32), (n,)), np.float32)
        params = {0: int(across_spatial), 1: int(channel_shared), 2: f"{eps:e}", 3: n}
        if across_channel != 1:
            params[4] = int(across_channel)
        if eps_mode != 0:
            params[9] = int(eps_mode)
        self._layer("Normalize", name, [bottom], [top], params)
        self._weights(scales, False)
        self.shape[top] = self.shape[bottom]
        return top

    def lrn(self, name, bottom, local_size=5, alpha=1e-4, beta=0.75, bias=1.0, region=0, top=None):
        """ncnn LRN 0=region_type 1=local_size 2=alpha 3=beta 4=bias (every key written); no weights."""
        top = top or name
        self._layer("LRN", name, [bottom], [top],
                    {0: int(region), 1: int(local_size), 2: f"{alpha:e}", 3: f"{beta:e}", 4: f"{bias:e}"})
        self.shape[top] = self.shape[bottom]
        return top

    def pool(self, name, bottom, type_=0, k=2, stride=2, pad=0, global_pooling=False, top=None):
        top = top or name
        c, h, w = self.shape[bottom]
        params = {0: type_, 1: k, 2: stride, 3: pad, 4: int(global_pooling)}
        self._layer("Pooling", name, [bottom], [top], params)
        if global_pooling:
            self.shape[top] = (c, 1, 1)
        else:  # ceil mode, pooling_layer.h:129-130
            oh = int(np.ceil((h + 2 * pad - k) / stride)) + 1
            ow = int(np.ceil((w + 2 * pad - k) / stride)) + 1
            self.shape[top] = (c, oh, ow)
        return top

    def fc(self, name, bottom, out, bias=True, top=None):
        top = top or name
        n_in = int(np.prod(self.shape[bottom]))
        wts = (self.rng.standard_normal((out, n_in)) * np.sqrt(2.0 / n_in)).astype(np.float32)
        self._layer("InnerProduct", name, [bottom], [top], {0: out, 1: int(bias), 2: wts.size})
        self._weights(wts, True)
        if bias:
            self._weights(self.rng.uniform(-0.1, 0.1, out).astype(np.float32), False)
        self.shape[top] = (out, 1, 1)
        self.flops += 2.0 * out * n_in
        return top

    def batchnorm(self, name, bottom, top=None, eps=None):
        top = top or name
        c = self.shape[bottom][0]
        if self.wide_stats:
            return self._batchnorm_wide(name, bottom, top, c, 1e-3 if eps is None else eps)
        eps = 1e-5 if eps is None else eps
        self._layer("BatchNorm", name, [bottom], [top], {0: c, 1: f"{eps:e}"})
        r = self.rng
        self._weights(r.uniform(0.9, 1.1, c).astype(np.float32), False)   # slope
        self._weights(r.uniform(-0.1, 0.1, c).astype(np.float32), False)  # mean
        self._weights(r.uniform(0.5, 1.5, c).astype(np.float32), False)   # var
        self._weights(r.uniform(-0.1, 0.1, c).astype(np.float32), False)  # bias
        self.shape[top] = self.shape[bottom]
        return top

    def _batchnorm_wide(self, name, bottom, top, c, eps):
        """Statistics under which a wrong BN / Scale fold is visible per element (wide_stats=True):
        - the per-channel multiplier slope / sqrt(var + eps) is log-uniform over five decades, rescaled to RMS 1;
        - about 10% of the multipliers are negative and one channel is dead (slope 0);
        - eps defaults to 1e-3 and ceil(30%) of the channels have var <= eps, so dropping eps changes their multiplier by
          >= sqrt(2);
        - |mean| up to 2, so the offset bias - slope * mean / sqrt(var + eps) is O(1), not a small correction."""
        r = self.rng
        self._layer("BatchNorm", name, [bottom], [top], {0: c, 1: f"{eps:e}"})
        var = eps * 10.0 ** r.uniform(1, 4, c)                     # 10 to 1e4 times eps ...
        small = r.permutation(c)[:math.ceil(0.3 * c)]
        var[small] = r.uniform(0.1, 1.0, small.size) * eps       # ... except on these channels
        mul = 10.0 ** r.uniform(-2.5, 2.5, c) * np.where(r.random(c) < 0.1, -1.0, 1.0)
        mul[r.integers(c)] = 0.0
        mul /= np.sqrt(np.mean(mul ** 2))
        var32 = var.astype(np.float32)
        self._weights((mul * np.sqrt(var32.astype(np.float64) + eps)).astype(np.float32), False)  # slope
        self._weights(r.uniform(-2, 2, c).astype(np.float32), False)   # mean
        self._weights(var32, False)                                      # var
        self._weights(r.uniform(-1, 1, c).astype(np.float32), False)   # bias
        self._bn_mul[top] = mul
        self.shape[top] = self.shape[bottom]
        return top

    def scale(self, name, bottom, bias=True, top=None, center=1.0):
        top = top or name
        c = self.shape[bottom][0]
        self._layer("Scale", name, [bottom], [top], {0: c, 1: int(bias)})
        if self.wide_stats:
            # a positive multiplier in [0.5, 2]; its product with the BatchNorm's is rescaled to RMS `center`
            s = self.rng.uniform(0.5, 2.0, c)
            prev = self._bn_mul.get(bottom)
            if prev is not None and np.any(prev * s):
                s *= center / np.sqrt(np.mean((prev * s) ** 2))
            self._weights(s.astype(np.float32), False)
            if bias:
                self._weights(self.rng.uniform(-1, 1, c).astype(np.float32), False)
        else:
            self._weights((center * self.rng.uniform(0.9, 1.1, c)).astype(np.float32), False)
            if bias:
                self._weights(self.rng.uniform(-0.1, 0.1, c).astype(np.float32), False)
        self.shape[top] = self.shape[bottom]
        return top

    def split(self, name, bottom, tops):
        self._layer("Split", name, [bottom], tops)
        for t in tops:
            self.shape[t] = self.shape[bottom]
            self.rank[t] = self.rank.get(bottom, 3)
        return tops

    def eltwise(self, name, bottoms, top=None):
        top = top or name
        self._layer("Eltwise", name, bottoms, [top], {0: 1})
        self.shape[top] = self.shape[bottoms[0]]
        return top

    def binary_op(self, name, bottoms, op, scalar=None, top=None):
        """ncnn BinaryOp 0=op (0 ADD .. 11 RATAN2) of two bottoms, or of one bottom and `scalar` (1=1 2=scalar).  Two
        bottoms broadcast by numpy's rule on their (c, h, w)."""
        top = top or name
        if scalar is None:
            assert len(bottoms) == 2, (name, bottoms)
            self._layer("BinaryOp", name, bottoms, [top], {0: op})
            self.shape[top] = tuple(np.broadcast_shapes(*(self.shape[b] for b in bottoms)))
            self.rank[top] = max(self.rank.get(b, 3) for b in bottoms)
        else:
            assert len(bottoms) == 1, (name, bottoms)
            self._layer("BinaryOp", name, bottoms, [top], {0: op, 1: 1, 2: f"{float(scalar):e}"})
            self.shape[top] = self.shape[bottoms[0]]
        return top

    def add(self, name, bottoms, top=None):
        """A two-input sum in the writer's `adds` layout: Eltwise SUM, or BinaryOp ADD."""
        return self.eltwise(name, bottoms, top) if self.adds == "eltwise" else self.binary_op(name, bottoms, 0, top=top)

    def concat(self, name, bottoms, top=None, axis=0):
        """ncnn Concat over `axis` of the bottoms' rank (rank 1: 0 = w; rank 2: 0 = h, 1 = w; rank 3: 0 = c, 1 = h, 2 = w)."""
        top = top or name
        self._layer("Concat", name, bottoms, [top], {0: axis})
        rank = self.rank.get(bottoms[0], 3)
        a = (axis + rank if axis < 0 else axis) + 3 - rank
        shape = list(self.shape[bottoms[0]])
        shape[a] = sum(self.shape[b][a] for b in bottoms)
        self.shape[top] = tuple(shape)
        self.rank[top] = rank
        return top

    def shuffle_channel(self, name, bottom, group, reverse=0, top=None):
        """ncnn ShuffleChannel 0=group 1=reverse (1= only when set)."""
        top = top or name
        self._layer("ShuffleChannel", name, [bottom], [top], {0: group, 1: 1} if reverse else {0: group})
        self.shape[top] = self.shape[bottom]
        return top

    def slice(self, name, bottom, slices, axis=0, tops=None):
        """ncnn Slice -23300=slices 1=axis (1= only when not 0); -233 takes (extent - taken) / (tops left)."""
        tops = tops or [f"{name}_{i}" for i in range(len(slices))]
        params = {-23300: f"{len(slices)}," + ",".join(str(v) for v in slices)}
        if axis:
            params[1] = axis
        self._layer("Slice", name, [bottom], tops, params)
        rank = self.rank.get(bottom, 3)
        a = (axis + rank if axis < 0 else axis) + 3 - rank
        taken = 0
        for i, (t, v) in enumerate(zip(tops, slices)):
            n = (self.shape[bottom][a] - taken) // (len(slices) - i) if v == -233 else v
            shape = list(self.shape[bottom])
            shape[a] = n
            self.shape[t] = tuple(shape)
            self.rank[t] = rank
            taken += n
        return tops

    def softmax(self, name, bottom, top=None, axis=None):
        """Without `axis` (no 0= emitted): over each image's whole blob; with it, ncnn's softmax over that axis."""
        top = top or name
        self._layer("Softmax", name, [bottom], [top], None if axis is None else {0: axis, 1: 1})
        self.shape[top] = self.shape[bottom]
        self.rank[top] = self.rank.get(bottom, 3)
        return top

    def permute(self, name, bottom, order, top=None):
        """ncnn Permute 0=order_type: (c,h,w) -> 0 (c,h,w) 1 (c,w,h) 2 (h,c,w) 3 (h,w,c) 4 (w,c,h) 5 (w,h,c)."""
        top = top or name
        self._layer("Permute", name, [bottom], [top], {0: order})
        axes = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)][order]
        self.shape[top] = tuple(self.shape[bottom][a] for a in axes)
        self.rank[top] = self.rank.get(bottom, 3)
        return top

    def flatten(self, name, bottom, top=None):
        top = top or name
        self._layer("Flatten", name, [bottom], [top])
        self.shape[top] = (1, 1, int(np.prod(self.shape[bottom])))
        self.rank[top] = 1
        return top

    def reshape(self, name, bottom, w, h=-233, c=-233, top=None):
        """ncnn Reshape 0=w 1=h 2=c (-233 absent: the rank is the number present; 0 keeps the bottom's, -1 infers)."""
        top = top or name
        params = {k: v for k, v in ((0, w), (1, h), (2, c)) if v != -233}
        self._layer("Reshape", name, [bottom], [top], params)
        bc, bh, bw = self.shape[bottom]
        total = bc * bh * bw
        d = [v if v != 0 else keep for v, keep in zip((w, h, c)[:len(params)], (bw, bh, bc))]
        if -1 in d:
            d[d.index(-1)] = total // int(np.prod([v for v in d if v != -1]))
        d += [1] * (3 - len(d))
        assert d[0] * d[1] * d[2] == total, (name, d, total)
        self.shape[top] = (d[2], d[1], d[0])
        self.rank[top] = len(params)
        return top

    @staticmethod
    def _floats(vals) -> str:
        return f"{len(vals)}," + ",".join(f"{float(v):e}" for v in vals)

    def priorbox(self, name, feat, image, min_sizes, max_sizes=(), aspect_ratios=(), flip=True, clip=False,
                 variances=(0.1, 0.1, 0.2, 0.2), step=None, offset=0.5, top=None):
        """ncnn PriorBox on a feature map and the image: a rank-2 (2, 4 * P) blob of one image (boxes, variances)."""
        top = top or name
        params = {-23300: self._floats(min_sizes)}
        if max_sizes:
            params[-23301] = self._floats(max_sizes)
        if aspect_ratios:
            params[-23302] = self._floats(aspect_ratios)
        for k, v in zip((3, 4, 5, 6), variances):
            params[k] = f"{v:e}"
        params[7], params[8] = int(flip), int(clip)
        if step is not None:
            params[11], params[12] = f"{float(step[0]):e}", f"{float(step[1]):e}"
        params[13] = f"{offset:e}"
        self._layer("PriorBox", name, [feat, image], [top], params)
        ars = sum(0 if abs(a - 1) < 1e-6 else (2 if flip else 1) for a in aspect_ratios)
        per_loc = len(min_sizes) * (1 + (1 if max_sizes else 0) + ars)
        _, fh, fw = self.shape[feat]
        self.shape[top] = (1, 2, 4 * fh * fw * per_loc)
        self.rank[top] = 2
        return top

    def detection_output(self, name, loc, conf, priors, num_classes, nms_threshold=0.45, nms_top_k=100, keep_top_k=100,
                         conf_threshold=0.25, top=None):
        top = top or name
        self._layer("DetectionOutput", name, [loc, conf, priors], [top],
                    {0: num_classes, 1: f"{nms_threshold:e}", 2: nms_top_k, 3: keep_top_k, 4: f"{conf_threshold:e}"})
        self.shape[top] = (1, keep_top_k, 6)
        self.rank[top] = 2
        return top

    def yolo_detection_output(self, name, bottom, num_class, num_box, biases, confidence_threshold=0.01,
                              nms_threshold=0.45, nms_top_k=None, keep_top_k=None, top=None):
        """ncnn YoloDetectionOutput (YOLOv2): biases are num_box (w, h) anchor pairs in grid cells; 20= / 21= (nms_top_k /
        keep_top_k, default 1024) only when given.  Rank-2 (keep_top_k, 6) top."""
        return self._yolo("YoloDetectionOutput", name, [bottom], num_class, num_box, biases, None, None,
                          confidence_threshold, nms_threshold, nms_top_k, keep_top_k, top)

    def yolov3_detection_output(self, name, bottoms, num_class, num_box, biases, mask, anchors_scale,
                                confidence_threshold=0.01, nms_threshold=0.45, nms_top_k=None, keep_top_k=None, top=None):
        """ncnn Yolov3DetectionOutput: one bottom per scale; biases are anchor (w, h) pairs in input pixels, mask the anchor
        index of each (scale, box), anchors_scale the stride of each scale."""
        return self._yolo("Yolov3DetectionOutput", name, list(bottoms), num_class, num_box, biases, mask, anchors_scale,
                          confidence_threshold, nms_threshold, nms_top_k, keep_top_k, top)

    def _yolo(self, type_, name, bottoms, num_class, num_box, biases, mask, anchors_scale, confidence_threshold,
              nms_threshold, nms_top_k, keep_top_k, top):
        top = top or name
        for b in bottoms:
            assert self.shape[b][0] == num_box * (5 + num_class), (name, b, self.shape[b])
        params = {0: num_class, 1: num_box, 2: f"{confidence_threshold:e}", 3: f"{nms_threshold:e}",
                  -23304: self._floats(biases)}
        if mask is not None:
            params[-23305] = self._floats(mask)
            params[-23306] = self._floats(anchors_scale)
        if nms_top_k is not None:
            params[20] = nms_top_k
        if keep_top_k is not None:
            params[21] = keep_top_k
        self._layer(type_, name, bottoms, [top], params)
        self.shape[top] = (1, keep_top_k or 1024, 6)
        self.rank[top] = 2
        return top

    def extra_input(self, name, c=1, h=1, w=3):
        """A further Input after the first (input() starts a new net): Faster R-CNN's im_info, 3 values per image."""
        self._layer("Input", name, [], [name], {0: w, 1: h, 2: c})
        self.shape[name] = (c, h, w)
        return name

    def proposal(self, name, score, bbox, im_info, feat_stride=16, base_size=16, pre_nms_top_n=6000, post_nms_top_n=300,
                 nms_thresh=0.7, min_size=16, tops=None):
        """ncnn Proposal, every key written: rois (post_nms_top_n, 1, 4) per image and, with a second top, scores
        (post_nms_top_n, 1, 1).  Returns the rois top."""
        tops = tops or [name]
        self._layer("Proposal", name, [score, bbox, im_info], tops,
                    {0: feat_stride, 1: base_size, 2: pre_nms_top_n, 3: post_nms_top_n, 4: f"{nms_thresh:e}", 5: min_size})
        self.shape[tops[0]] = (post_nms_top_n, 1, 4)
        if len(tops) > 1:
            self.shape[tops[1]] = (post_nms_top_n, 1, 1)
        return tops[0]

    def roi_pooling(self, name, bottom, rois, pooled_w=7, pooled_h=7, spatial_scale=0.0625, top=None):
        """ncnn ROIPooling 0=pooled_w 1=pooled_h 2=spatial_scale.  The top has one item per RoI of every image; its shape
        here is one item's (C, pooled_h, pooled_w)."""
        top = top or name
        self._layer("ROIPooling", name, [bottom, rois], [top], {0: pooled_w, 1: pooled_h, 2: f"{spatial_scale:e}"})
        self.shape[top] = (self.shape[bottom][0], pooled_h, pooled_w)
        return top

    def psroi_pooling(self, name, bottom, rois, output_dim, pooled_w=7, pooled_h=7, spatial_scale=0.0625, top=None):
        """ncnn PSROIPooling 0=pooled_w 1=pooled_h 2=spatial_scale 3=output_dim on output_dim x pooled_h x pooled_w score
        maps.  One item per RoI of every image, as roi_pooling; its shape here is one item's (output_dim, pooled_h,
        pooled_w)."""
        top = top or name
        assert self.shape[bottom][0] == output_dim * pooled_h * pooled_w, (name, self.shape[bottom])
        self._layer("PSROIPooling", name, [bottom, rois], [top],
                    {0: pooled_w, 1: pooled_h, 2: f"{spatial_scale:e}", 3: output_dim})
        self.shape[top] = (output_dim, pooled_h, pooled_w)
        return top

    def instance_norm(self, name, bottom, eps=1e-5, affine=True, top=None):
        """ncnn InstanceNorm 0=channels 1=eps 2=affine; with affine, gamma (uniform(0.8, 1.2)) then beta (uniform(-0.1,
        0.1)), raw fp32 in the bin."""
        top = top or name
        c = self.shape[bottom][0]
        self._layer("InstanceNorm", name, [bottom], [top], {0: c, 1: f"{eps:e}", 2: int(affine)})
        if affine:
            self._weights(self.rng.uniform(0.8, 1.2, c).astype(np.float32), False)
            self._weights(self.rng.uniform(-0.1, 0.1, c).astype(np.float32), False)
        self.shape[top] = self.shape[bottom]
        return top

    def padding(self, name, bottom, top, bottom_, left, right, type_=2, value=0.0):
        """ncnn Padding 0=top 1=bottom 2=left 3=right 4=type (0 constant, 1 replicate, 2 reflect) 5=value (written when
        not 0).  The output blob is `name`."""
        c, h, w = self.shape[bottom]
        assert type_ != 2 or (max(top, bottom_) < h and max(left, right) < w), (name, self.shape[bottom])
        params = {0: top, 1: bottom_, 2: left, 3: right, 4: type_}
        if value:
            params[5] = f"{value:e}"
        self._layer("Padding", name, [bottom], [name], params)
        self.shape[name] = (c, h + top + bottom_, w + left + right)
        return name

    def dropout(self, name, bottom, top=None, scale=None):
        top = top or name
        self._layer("Dropout", name, [bottom], [top], {} if scale is None else {0: f"{scale:e}"})
        self.shape[top] = self.shape[bottom]
        return top

    def interp(self, name, bottom, resize_type=2, out_h=0, out_w=0, scale=None, align_corner=0, top=None):
        """ncnn Interp: resize_type 1 nearest, 2 bilinear; an explicit (out_h, out_w), or `scale` when either is 0."""
        top = top or name
        c, h, w = self.shape[bottom]
        params = {0: resize_type}
        if scale is not None:
            params[1] = params[2] = f"{scale:e}"
        if out_h or out_w:
            params[3], params[4] = out_h, out_w
        if align_corner:
            params[6] = 1
        self._layer("Interp", name, [bottom], [top], params)
        if out_h and out_w:
            self.shape[top] = (c, out_h, out_w)
        else:  # fp32 products, truncated (fcuda_interp_output_dim)
            s = np.float32(1.0 if scale is None else scale)
            self.shape[top] = (c, int(np.float32(h) * s), int(np.float32(w) * s))
        return top

    def activation(self, type_, name, bottom, alpha=None, beta=None, top=None):
        """ncnn Sigmoid / TanH / Swish (no parameters), HardSigmoid / HardSwish 0=alpha 1=beta (each written when given;
        pnnx writes PyTorch's 1/6 and 0.5 as 0=1.666667e-01 1=5.000000e-01)."""
        assert type_ in ("Sigmoid", "TanH", "Swish", "HardSigmoid", "HardSwish"), type_
        top = top or name
        params = {k: f"{v:e}" for k, v in ((0, alpha), (1, beta)) if v is not None}
        self._layer(type_, name, [bottom], [top], params)
        self.shape[top] = self.shape[bottom]
        return top

    def hard(self, type_, name, bottom, top=None):
        """HardSigmoid / HardSwish with PyTorch's alpha 1/6 and beta 0.5, as pnnx writes them."""
        return self.activation(type_, name, bottom, 1.0 / 6.0, 0.5, top)

    def pixel_shuffle(self, name, bottom, r, mode=0, top=None):
        """ncnn PixelShuffle 0=upscale_factor 1=mode (0 PyTorch's channel order, 1 DepthToSpace DCR; written when 1)."""
        top = top or name
        c, h, w = self.shape[bottom]
        assert c % (r * r) == 0, (name, self.shape[bottom], r)
        self._layer("PixelShuffle", name, [bottom], [top], {0: r, 1: mode} if mode else {0: r})
        self.shape[top] = (c // (r * r), h * r, w * r)
        return top

    def fixed_conv1x1(self, name, bottom, weights, bias, top=None):
        """A 1x1 Convolution with the given (oc, ic) weights and oc biases (EDSR's MeanShift)."""
        top = top or name
        wts = np.ascontiguousarray(weights, np.float32)
        oc, ic = wts.shape
        c, h, w = self.shape[bottom]
        assert ic == c, (name, self.shape[bottom])
        self._layer("Convolution", name, [bottom], [top], {0: oc, 1: 1, 3: 1, 4: 0, 5: 1, 6: wts.size})
        self._weights(wts, True)
        self._weights(np.asarray(bias, np.float32).reshape(oc), False)
        self.shape[top] = (oc, h, w)
        self.flops += 2.0 * oc * ic * h * w
        return top

    def crop(self, name, bottom, woff=0, hoff=0, reference=None, coff=0, outc=0, outh=0, outw=0, top=None):
        """ncnn Crop: with `reference` the output height and width are that blob's; a size of 0 runs to the end."""
        top = top or name
        c, h, w = self.shape[bottom]
        params = {k: v for k, v in ((0, woff), (1, hoff), (2, coff), (3, outw), (4, outh), (5, outc)) if v or k < 2}
        self._layer("Crop", name, [bottom] + ([reference] if reference else []), [top], params)
        oc = outc or c - coff
        if reference:
            oh, ow = self.shape[reference][1:]
        else:
            oh, ow = outh or h - hoff, outw or w - woff
        assert coff + oc <= c and hoff + oh <= h and woff + ow <= w, (name, self.shape[bottom], (oc, oh, ow))
        self.shape[top] = (oc, oh, ow)
        return top

    # ---- Vision Transformer layers (token blobs are rank 2: w = features, h = tokens) -----------------------------
    def memory_data(self, name, w, h=0, c=0, data=None, std=0.02):
        """ncnn MemoryData 0=w 1=h 2=c (the rank is the number of leading dims given): `data` (w * h * c raw floats), or
        normal(0, std) draws."""
        shape = (max(c, 1), max(h, 1), w)
        data = self.rng.standard_normal(shape) * std if data is None else data
        params = {k: v for k, v in ((0, w), (1, h), (2, c)) if v}
        self._layer("MemoryData", name, [], [name], params)
        self._weights(np.asarray(data, np.float32).reshape(shape), False)
        self.shape[name] = shape
        self.rank[name] = len(params)
        return name

    def layer_norm(self, name, bottom, eps=1e-6, top=None):
        """ncnn LayerNorm 0=affine_size (the bottom's w) 1=eps 2=1; gamma uniform(0.8, 1.2), beta uniform(-0.1, 0.1)."""
        top = top or name
        n = self.shape[bottom][2]
        self._layer("LayerNorm", name, [bottom], [top], {0: n, 1: f"{eps:e}", 2: 1})
        self._weights(self.rng.uniform(0.8, 1.2, n).astype(np.float32), False)
        self._weights(self.rng.uniform(-0.1, 0.1, n).astype(np.float32), False)
        self.shape[top] = self.shape[bottom]
        self.rank[top] = self.rank.get(bottom, 3)
        return top

    def linear(self, name, bottom, out, top=None):
        """InnerProduct on a rank-2 token blob: each row is one input vector (ncnn's rule), the top is rank 2.  Weights
        normal(0, 1 / sqrt(in)), bias uniform(-0.1, 0.1)."""
        top = top or name
        _, h, n_in = self.shape[bottom]
        assert self.rank.get(bottom, 3) == 2 and h > 1, (name, self.shape[bottom])
        wts = (self.rng.standard_normal((out, n_in)) / np.sqrt(n_in)).astype(np.float32)
        self._layer("InnerProduct", name, [bottom], [top], {0: out, 1: 1, 2: wts.size})
        self._weights(wts, True)
        self._weights(self.rng.uniform(-0.1, 0.1, out).astype(np.float32), False)
        self.shape[top] = (1, h, out)
        self.rank[top] = 2
        self.flops += 2.0 * out * n_in * h
        return top

    def gelu(self, name, bottom, fast=0, top=None):
        """ncnn GELU 0=fast_gelu (written when 1)."""
        top = top or name
        self._layer("GELU", name, [bottom], [top], {0: 1} if fast else None)
        self.shape[top] = self.shape[bottom]
        self.rank[top] = self.rank.get(bottom, 3)
        return top

    def multihead_attention(self, name, bottom, heads, top=None):
        """ncnn MultiHeadAttention of one bottom (q = k = v): 0=embed_dim 1=num_heads 2=embed_dim^2, default scale.
        Weights q_w, q_b, k_w, k_b, v_w, v_b, out_w, out_b (matrices normal(0, 1 / sqrt(E)) flagged, biases
        uniform(-0.1, 0.1) raw)."""
        top = top or name
        _, l, e = self.shape[bottom]
        self._layer("MultiHeadAttention", name, [bottom], [top], {0: e, 1: heads, 2: e * e})
        for _ in range(4):
            self._weights((self.rng.standard_normal((e, e)) / np.sqrt(e)).astype(np.float32), True)
            self._weights(self.rng.uniform(-0.1, 0.1, e).astype(np.float32), False)
        self.shape[top] = (1, l, e)
        self.rank[top] = 2
        self.flops += 8.0 * l * e * e + 4.0 * l * l * e
        return top

    # ---- output ------------------------------------------------------------------------------
    def save(self, prefix) -> tuple[str, str]:
        prefix = str(prefix)
        Path(prefix).parent.mkdir(parents=True, exist_ok=True)
        text = "7767517\n" + f"{len(self.lines)} {len(self.blobs)}\n" + "\n".join(self.lines) + "\n"
        Path(prefix + ".param").write_text(text)
        Path(prefix + ".bin").write_bytes(bytes(self.bin))
        return prefix + ".param", prefix + ".bin"


# --------------------------------------------------------------------------------------------------
# model zoo
# --------------------------------------------------------------------------------------------------
def single_conv(ic=64, oc=64, h=56, w=56, k=3, stride=1, pad=1, bias=True, group=1, seed=0) -> ModelWriter:
    """BASELINE.json configs[0]: one 3x3 conv 64->64 on 56x56."""
    m = ModelWriter(seed)
    m.input("data", ic, h, w)
    m.conv("conv", "data", oc, k, stride, pad, bias, group)
    return m


def vgg16(seed=0, num_classes=1000, size=224) -> ModelWriter:
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    cfg = [(64, 2), (128, 2), (256, 3), (512, 3), (512, 3)]
    for si, (ch, n) in enumerate(cfg, 1):
        for li in range(1, n + 1):
            x = m.conv(f"conv{si}_{li}", x, ch, 3, 1, 1, True)
            x = m.relu(f"relu{si}_{li}", x)
        x = m.pool(f"pool{si}", x, 0, 2, 2)
    x = m.fc("fc6", x, 4096); x = m.relu("relu6", x); x = m.dropout("drop6", x)
    x = m.fc("fc7", x, 4096); x = m.relu("relu7", x); x = m.dropout("drop7", x)
    x = m.fc("fc8", x, num_classes)
    m.softmax("prob", x)
    return m


def _bn_scale_relu(m: ModelWriter, tag: str, x: str, relu=True, center=1.0):
    x = m.batchnorm("bn" + tag, x)
    x = m.scale("scale" + tag, x, True, center=center)
    if relu:
        x = m.relu(tag.lstrip("_") + "_relu", x)
    return x


def _resnet50_trunk(m: ModelWriter, x: str, strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1)) -> str:
    """Caffe ResNet-50 conv1 .. res5c_relu: stride on the first 1x1 of each stage (strides[i] for res2 .. res5), every
    3x3 branch2b of stage i at dilation and pad dilations[i], BN/Scale/ReLU layers, Split/Eltwise."""
    x = m.conv("conv1", x, 64, 7, 2, 3, True)
    x = _bn_scale_relu(m, "_conv1", x)
    x = m.pool("pool1", x, 0, 3, 2, 0)
    stages = [(2, 3, 64), (3, 4, 128), (4, 6, 256), (5, 3, 512)]
    for (sid, nblocks, width), stride, dil in zip(stages, strides, dilations):
        for b in range(nblocks):
            blk = f"{sid}{chr(ord('a') + b)}"
            s = stride if b == 0 else 1
            a, c = m.split(f"res{blk}_split", x, [f"res{blk}_in_a", f"res{blk}_in_b"])
            if b == 0:
                sc = m.conv(f"res{blk}_branch1", a, width * 4, 1, s, 0, False)
                sc = _bn_scale_relu(m, f"{blk}_branch1", sc, relu=False)
            else:
                sc = a
            y = m.conv(f"res{blk}_branch2a", c, width, 1, s, 0, False)
            y = _bn_scale_relu(m, f"{blk}_branch2a", y)
            y = m.conv(f"res{blk}_branch2b", y, width, 3, 1, dil, False, dilation=dil)
            y = _bn_scale_relu(m, f"{blk}_branch2b", y)
            y = m.conv(f"res{blk}_branch2c", y, width * 4, 1, 1, 0, False)
            y = _bn_scale_relu(m, f"{blk}_branch2c", y, relu=False, center=0.3)  # keep residual sums O(1)
            x = m.add(f"res{blk}", [sc, y])
            x = m.relu(f"res{blk}_relu", x)
    return x


def resnet50(seed=0, num_classes=1000, size=224, wide_stats=False, adds="eltwise") -> ModelWriter:
    """Caffe ResNet-50 layout: stride on the first 1x1 of each stage, BN/Scale/ReLU layers, Split/Eltwise.  adds=
    "binaryop" writes each shortcut sum as BinaryOp ADD (onnx2ncnn's and pnnx's layout), the same .bin."""
    m = ModelWriter(seed, wide_stats, adds)
    x = _resnet50_trunk(m, m.input("data", 3, size, size))
    x = m.pool("pool5", x, 1, 7, 1, 0, global_pooling=True)
    x = m.fc("fc1000", x, num_classes)
    m.softmax("prob", x)
    return m


def mobilenet_v1(seed=0, num_classes=1000, size=224, wide_stats=False) -> ModelWriter:
    m = ModelWriter(seed, wide_stats)
    x = m.input("data", 3, size, size)
    x = m.conv("conv1", x, 32, 3, 2, 1, False)
    x = _bn_scale_relu(m, "_conv1", x)
    cfg = [(64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1), (512, 1), (512, 1), (512, 1), (512, 1),
           (1024, 2), (1024, 1)]
    for i, (oc, s) in enumerate(cfg, 2):
        ic = m.shape[x][0]
        x = m.conv(f"conv{i}_dw", x, ic, 3, s, 1, False, group=ic)
        x = _bn_scale_relu(m, f"_conv{i}_dw", x)
        x = m.conv(f"conv{i}_pw", x, oc, 1, 1, 0, False)
        x = _bn_scale_relu(m, f"_conv{i}_pw", x)
    x = m.pool("pool6", x, 1, 7, 1, 0, global_pooling=True)
    x = m.conv("fc7", x, num_classes, 1, 1, 0, True)
    m.softmax("prob", x)
    return m


def _bn_scale_clip(m: ModelWriter, tag: str, x: str, clip=True, center=1.0):
    x = m.batchnorm("bn" + tag, x)
    x = m.scale("scale" + tag, x, True, center=center)
    if clip:
        x = m.clip(tag.lstrip("_") + "_relu6", x, 0.0, 6.0)
    return x


def mobilenet_v2(seed=0, num_classes=1000, size=224, wide_stats=False, adds="eltwise") -> ModelWriter:
    """MobileNet-v2 (Sandler et al. 2018): inverted residual blocks from the (t, c, n, s) table, every convolution followed
    by BatchNorm + Scale, ReLU6 as ncnn's Clip 0..6 after the stem, expansion and depthwise convolutions, linear
    projections, and an Eltwise SUM shortcut (through a Split) where the stride is 1 and the channel count is kept.
    adds="binaryop" writes each shortcut as BinaryOp ADD, the same .bin."""
    m = ModelWriter(seed, wide_stats, adds)
    x = m.input("data", 3, size, size)
    x = m.conv("conv1", x, 32, 3, 2, 1, False)
    x = _bn_scale_clip(m, "_conv1", x)
    table = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]
    for bi, (t, c, n, s) in enumerate(table, 2):
        for i in range(n):
            tag = f"{bi}_{i + 1}"
            stride = s if i == 0 else 1
            ic = m.shape[x][0]
            shortcut = stride == 1 and ic == c
            if shortcut:
                sc, x = m.split(f"block{tag}_split", x, [f"block{tag}_in_a", f"block{tag}_in_b"])
            y = x
            if t != 1:
                y = m.conv(f"conv{tag}_expand", y, ic * t, 1, 1, 0, False)
                y = _bn_scale_clip(m, f"_conv{tag}_expand", y)
            y = m.conv(f"conv{tag}_dw", y, ic * t, 3, stride, 1, False, group=ic * t)
            y = _bn_scale_clip(m, f"_conv{tag}_dw", y)
            y = m.conv(f"conv{tag}_linear", y, c, 1, 1, 0, False)
            y = _bn_scale_clip(m, f"_conv{tag}_linear", y, clip=False, center=0.3 if shortcut else 1.0)
            x = m.add(f"block{tag}", [sc, y]) if shortcut else y
    x = m.conv("conv_last", x, 1280, 1, 1, 0, False)
    x = _bn_scale_clip(m, "_conv_last", x)
    x = m.pool("pool_last", x, 1, 7, 1, 0, global_pooling=True)
    x = m.conv("fc", x, num_classes, 1, 1, 0, True)
    m.softmax("prob", x)
    return m


SHUFFLENET_V2_STAGES = {0.5: (48, 96, 192), 1.0: (116, 232, 464), 1.5: (176, 352, 704), 2.0: (244, 488, 976)}


def shufflenet_v2(seed=0, num_classes=1000, size=224, width=1.0, wide_stats=False) -> ModelWriter:
    """ShuffleNet-v2 (Ma et al. 2018) as ncnn's converted models lay it out: a 3x3 / 2 stem (24 channels) with BatchNorm +
    Scale + ReLU and a 3x3 / 2 max pool, three stages of 4 / 8 / 4 units, conv5 (1024 channels, 2048 at 2.0x), global
    average pool, InnerProduct and Softmax.  A downsampling unit Splits its input into two stride-2 branches (3x3 depthwise
    + 1x1; 1x1 + 3x3 depthwise + 1x1); a stride-1 unit Slices its input into two halves and runs the second through the
    1x1 / depthwise / 1x1 branch.  Both Concat their halves and ShuffleChannel with group 2."""
    m = ModelWriter(seed, wide_stats)
    x = m.input("data", 3, size, size)
    x = m.conv("conv1", x, 24, 3, 2, 1, False)
    x = _bn_scale_relu(m, "_conv1", x)
    x = m.pool("pool1", x, 0, 3, 2, 0)
    for si, (oc, n) in enumerate(zip(SHUFFLENET_V2_STAGES[width], (4, 8, 4)), 2):
        half = oc // 2
        for u in range(1, n + 1):
            tag = f"stage{si}_{u}"
            ic = m.shape[x][0]
            if u == 1:
                a, b = m.split(f"{tag}_split", x, [f"{tag}_in_a", f"{tag}_in_b"])
                a = m.conv(f"{tag}_b1_dw", a, ic, 3, 2, 1, False, group=ic)
                a = _bn_scale_relu(m, f"_{tag}_b1_dw", a, relu=False)
                a = m.conv(f"{tag}_b1_pw", a, half, 1, 1, 0, False)
                a = _bn_scale_relu(m, f"_{tag}_b1_pw", a)
                stride = 2
            else:
                a, b = m.slice(f"{tag}_slice", x, [-233, -233])
                stride = 1
            b = m.conv(f"{tag}_b2_pw1", b, half, 1, 1, 0, False)
            b = _bn_scale_relu(m, f"_{tag}_b2_pw1", b)
            b = m.conv(f"{tag}_b2_dw", b, half, 3, stride, 1, False, group=half)
            b = _bn_scale_relu(m, f"_{tag}_b2_dw", b, relu=False)
            b = m.conv(f"{tag}_b2_pw2", b, half, 1, 1, 0, False)
            b = _bn_scale_relu(m, f"_{tag}_b2_pw2", b)
            x = m.concat(f"{tag}_concat", [a, b])
            x = m.shuffle_channel(f"{tag}_shuffle", x, 2)
    x = m.conv("conv5", x, 2048 if width == 2.0 else 1024, 1, 1, 0, False)
    x = _bn_scale_relu(m, "_conv5", x)
    x = m.pool("pool5", x, 1, 7, 1, 0, global_pooling=True)
    x = m.fc("fc", x, num_classes)
    m.softmax("prob", x)
    return m


def shuffle_tiny(seed=0, size=15, classes=10, wide_stats=False) -> ModelWriter:
    """What ShuffleNet-v2 does not route: ShuffleChannel group 3 after a grouped 1x1 convolution (ShuffleNet-v1's
    pattern) fused into an uneven Slice that drops a remainder, a reverse ShuffleChannel in a Concat -> ShuffleChannel ->
    Slice chain, a Concat -> Slice pair, and Slices on h and w.  The 15 x 15 planes take the 4-byte path."""
    m = ModelWriter(seed, wide_stats)
    x = m.input("data", 3, size, size)
    x = m.relu("relu1", m.conv("conv1", x, 12, 3, 1, 1, True))
    x = m.relu("gconv_relu", m.conv("gconv", x, 12, 1, 1, 0, True, group=3))
    x = m.shuffle_channel("shuffle_g3", x, 3)
    a, b = m.slice("slice_uneven", x, [5, 4])                 # channels 9..11 are dropped
    a = m.relu("conv_a_relu", m.conv("conv_a", a, 6, 1, 1, 0, True))
    b, bs = m.split("split_b", b, ["b_conv", "b_rows"])
    h0, h1 = m.slice("slice_h", bs, [-233, -233], axis=1)      # rows 7 + 8
    m.slice("slice_w", h1, [3, -233, 5], axis=2)               # columns 3 + 6 + 5, one dropped
    b = m.relu("conv_b_relu", m.conv("conv_b", b, 6, 1, 1, 0, True))
    x = m.concat("cat1", [a, b])
    x = m.shuffle_channel("shuffle_rev", x, 4, reverse=1)     # 12 channels: 3 groups of 4
    c, d = m.slice("slice_even", x, [-233, -233])
    c = m.relu("conv_c_relu", m.conv("conv_c", c, 6, 3, 1, 1, True))
    x = m.concat("cat2", [d, c])
    e, f = m.slice("slice_cat", x, [4, -233])
    e = m.relu("conv_e_relu", m.conv("conv_e", e, 4, 1, 1, 0, True))
    x = m.concat("cat3", [e, f])
    x = m.pool("pool", x, 1, 2, 2, 0, global_pooling=True)
    x = m.conv("fc", x, classes, 1, 1, 0, True)
    m.softmax("prob", x)
    return m


def prelu_tiny(seed=0, size=15, classes=10, wide_stats=False) -> ModelWriter:
    """Convolutions followed by BatchNorm + Scale + PReLU, as in face-detection nets (MTCNN, MobileFaceNet): per-channel
    slopes on a 15 x 15 plane (not a multiple of 4: the scalar kernel), one shared slope on the 8 x 8 plane after it."""
    m = ModelWriter(seed, wide_stats)
    x = m.input("data", 3, size, size)
    x = m.conv("conv1", x, 16, 3, 1, 1, True)
    x = m.batchnorm("bn1", x); x = m.scale("scale1", x, True)
    x = m.prelu("prelu1", x)
    x = m.conv("conv2", x, 32, 3, 2, 1, True)
    x = m.batchnorm("bn2", x); x = m.scale("scale2", x, True)
    x = m.prelu("prelu2", x, shared=True)
    x = m.pool("pool2", x, 1, 2, 2, 0, global_pooling=True)
    x = m.conv("fc", x, classes, 1, 1, 0, True)
    m.softmax("prob", x)
    return m


def mini(seed=0, size=32, ch=16, wide_stats=False) -> ModelWriter:
    """Small net touching every layer type (SURVEY.md §8c's 12-layer probe net, plus concat/dropout/depthwise)."""
    m = ModelWriter(seed, wide_stats)
    x = m.input("data", 4, size, size)
    x = m.conv("conv1", x, ch, 3, 1, 1, True)               # Winograd F63 eligible (size > 8, ch % 4 == 0)
    x = m.batchnorm("bn1", x); x = m.scale("scale1", x, True); x = m.relu("relu1", x)
    a, b = m.split("split1", x, ["s1a", "s1b"])
    y = m.conv("conv2", b, ch, 1, 1, 0, False)               # 1x1 -> IM2COL
    y = m.batchnorm("bn2", y); y = m.scale("scale2", y, False)
    x = m.eltwise("sum1", [a, y]); x = m.relu("relu2", x)
    x = m.conv("conv3_dw", x, ch, 3, 2, 1, False, group=ch)  # depthwise s2
    x = m.relu("relu3", x)
    p, q = m.split("split2", x, ["s2a", "s2b"])
    q = m.conv("conv4", q, ch, 3, 2, 1, True)                # 3x3 s2 -> IM2COL
    p = m.pool("pool1", p, 0, 3, 2, 0)                       # max, ceil mode
    x = m.concat("cat1", [p, q])
    x = m.conv("conv5", x, ch * 2, 3, 1, 1, True)            # Winograd if spatial > 8 else IM2COL
    x = m.relu("relu5", x)
    x = m.pool("pool2", x, 1, 2, 2, 0, global_pooling=True)  # global average
    x = m.dropout("drop1", x, scale=0.5)
    x = m.fc("fc1", x, 24, True)
    x = m.relu("relu6", x)
    x = m.fc("fc2", x, 10, True)
    m.softmax("prob", x)
    return m


def bilinear_kernel(channels: int, k: int) -> np.ndarray:
    """(channels, 1, k, k) bilinear upsampling filter, as Caffe's "bilinear" filler makes it (FCN's upsampling layers)."""
    f = math.ceil(k / 2)
    c = (2 * f - 1 - f % 2) / (2.0 * f)
    t = 1 - np.abs(np.arange(k) / f - c)
    return np.broadcast_to(np.outer(t, t), (channels, 1, k, k)).astype(np.float32)


def decoder_tiny(seed=0, size=16, classes=4) -> ModelWriter:
    """Encoder-decoder with a Split/Concat skip connection: learned upsampling by Deconvolution (k4 s2 p1 + BN + Scale +
    ReLU, k2 s2 + ReLU), a 1x1 classifier and FCN's fixed bilinear DeconvolutionDepthWise (k4 s2 p1, no bias)."""
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = m.conv("enc1", x, 16, 3, 1, 1, True)
    x = m.relu("enc1_relu", x)
    skip, x = m.split("enc1_split", x, ["skip", "down_in"])
    x = m.conv("enc2", x, 32, 3, 2, 1, True)
    x = m.relu("enc2_relu", x)
    x = m.deconv("up1", x, 16, 4, 2, 1, True)
    x = _bn_scale_relu(m, "_up1", x)
    x = m.concat("cat1", [skip, x])
    x = m.deconv("up2", x, 16, 2, 2, 0, True)
    x = m.relu("up2_relu", x)
    x = m.conv("score", x, classes, 1, 1, 0, True)
    m.deconv("upscore", x, classes, 4, 2, 1, False, group=classes, weights=bilinear_kernel(classes, 4))
    return m


def fcn8s_tiny(seed=0, size=64, classes=5) -> ModelWriter:
    """FCN-8s topology at small width: five 2x2 poolings behind a first convolution padded by 50 (FCN pads by 100) and
    an unpadded 5x5 "fc6", score convolutions on pool3 / pool4, k4 s2 deconvolutions with two-bottom crops of the skip
    scores before each Eltwise SUM, and a k16 s8 deconvolution cropped to the input.  The crop offsets (5, 7, 27) are
    odd, like FCN's (5, 9, 31); the windows fit sizes 32 to 700 except those = 30 (mod 32)."""
    m = ModelWriter(seed)
    data = m.input("data", 3, size, size)
    x = m.relu("relu1", m.conv("conv1", data, 16, 3, 1, 50, True))
    x = m.pool("pool1", x)
    x = m.relu("relu2", m.conv("conv2", x, 16, 3, 1, 1, True))
    x = m.pool("pool2", x)
    x = m.relu("relu3", m.conv("conv3", x, 32, 3, 1, 1, True))
    pool3 = m.pool("pool3", x)
    p3a, p3b = m.split("pool3_split", pool3, ["pool3_a", "pool3_b"])
    x = m.relu("relu4", m.conv("conv4", p3a, 32, 3, 1, 1, True))
    pool4 = m.pool("pool4", x)
    p4a, p4b = m.split("pool4_split", pool4, ["pool4_a", "pool4_b"])
    x = m.relu("relu5", m.conv("conv5", p4a, 64, 3, 1, 1, True))
    x = m.pool("pool5", x)
    x = m.relu("relu_fc6", m.conv("fc6", x, 64, 5, 1, 0, True))
    x = m.relu("relu_fc7", m.conv("fc7", x, 64, 1, 1, 0, True))
    x = m.conv("score_fr", x, classes, 1, 1, 0, True)
    up2 = m.deconv("upscore2", x, classes, 4, 2, 0, False)
    up2a, up2b = m.split("upscore2_split", up2, ["upscore2_a", "upscore2_b"])
    sp4 = m.conv("score_pool4", p4b, classes, 1, 1, 0, True, gain=0.01)
    sp4c = m.crop("score_pool4c", sp4, 5, 5, reference=up2a)
    x = m.eltwise("fuse_pool4", [up2b, sp4c])
    upp4 = m.deconv("upscore_pool4", x, classes, 4, 2, 0, False)
    upp4a, upp4b = m.split("upscore_pool4_split", upp4, ["upscore_pool4_a", "upscore_pool4_b"])
    sp3 = m.conv("score_pool3", p3b, classes, 1, 1, 0, True, gain=0.001)
    sp3c = m.crop("score_pool3c", sp3, 7, 7, reference=upp4a)
    x = m.eltwise("fuse_pool3", [upp4b, sp3c])
    x = m.deconv("upscore8", x, classes, 16, 8, 0, False)
    m.crop("score", x, 27, 27, reference=data)
    return m


def deeplab_head_tiny(seed=0, size=32, classes=5) -> ModelWriter:
    """DeepLab-style head: a stride-8 encoder, a dilated 3x3 convolution (dilation 2), a 1x1 classifier and a fixed x8
    bilinear Interp (scales, half-pixel) back to the input size."""
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = m.relu("relu1", m.conv("conv1", x, 16, 3, 2, 1, True))
    x = m.relu("relu2", m.conv("conv2", x, 32, 3, 2, 1, True))
    x = m.relu("relu3", m.conv("conv3", x, 32, 3, 2, 1, True))
    x = m.relu("relu_aspp", m.conv("aspp", x, 32, 3, 1, 2, True, dilation=2))
    x = m.conv("classifier", x, classes, 1, 1, 0, True)
    m.interp("upsample", x, 2, scale=8.0)
    return m


def _deeplabv3(m: ModelWriter, x: str, table, output_stride: int, aspp: int, num_classes: int, size: int) -> str:
    """DeepLab-v3's atrous backbone and mobile ASPP head on `x` (after a stride-2 stem).  The MobileNet-v2 blocks of `table`
    ((t, c, n, s, k) rows) follow TF-DeepLab's rule: once the stride so far equals `output_stride`, a block's stride becomes
    1, that layer keeps the current rate, and every later depthwise layer runs at the rate times that stride (pad = rate,
    pad = rate * (k - 1) / 2 for k != 3)."""
    stride_so_far, rate = 2, 1
    for bi, (t, c, n, s, k) in enumerate(table, 2):
        for i in range(n):
            tag = f"{bi}_{i + 1}"
            stride, layer_rate = s if i == 0 else 1, rate
            if stride_so_far == output_stride:
                rate *= stride
                stride = 1
            else:
                stride_so_far *= stride
            ic = m.shape[x][0]
            shortcut = stride == 1 and ic == c
            if shortcut:
                sc, x = m.split(f"block{tag}_split", x, [f"block{tag}_in_a", f"block{tag}_in_b"])
            y = x
            if t != 1:
                y = m.conv(f"conv{tag}_expand", y, ic * t, 1, 1, 0, False)
                y = _bn_scale_clip(m, f"_conv{tag}_expand", y)
            y = m.conv(f"conv{tag}_dw", y, ic * t, k, stride, layer_rate * (k - 1) // 2, False, group=ic * t,
                       dilation=layer_rate)
            y = _bn_scale_clip(m, f"_conv{tag}_dw", y)
            y = m.conv(f"conv{tag}_linear", y, c, 1, 1, 0, False)
            y = _bn_scale_clip(m, f"_conv{tag}_linear", y, clip=False, center=0.3 if shortcut else 1.0)
            x = m.eltwise(f"block{tag}", [sc, y]) if shortcut else y
    _, fh, fw = m.shape[x]
    feat_a, feat_b = m.split("aspp_split", x, ["aspp_in_a", "aspp_in_b"])
    p = m.pool("image_pool", feat_a, 1, 1, 1, 0, global_pooling=True)
    p = _bn_scale_relu(m, "_image_pool_conv", m.conv("image_pool_conv", p, aspp, 1, 1, 0, False))
    p = m.interp("image_pool_up", p, 2, out_h=fh, out_w=fw)
    b = _bn_scale_relu(m, "_aspp0", m.conv("aspp0", feat_b, aspp, 1, 1, 0, False))
    y = m.concat("aspp_concat", [p, b])
    y = _bn_scale_relu(m, "_aspp_proj", m.conv("aspp_proj", y, aspp, 1, 1, 0, False))
    y = m.conv("logits", y, num_classes, 1, 1, 0, True)
    return m.interp("logits_up", y, 2, out_h=size, out_w=size, align_corner=1)


def deeplabv3_mobilenet_v2(seed=0, size=513, num_classes=21, output_stride=16) -> ModelWriter:
    """DeepLab-v3 (Chen et al. 2017) on MobileNet-v2, as TF-DeepLab's mobilenet_v2 variant: `mobilenet_v2`'s stem and
    blocks up to the 320 one, with the last strides turned into depthwise dilations so the features stay at
    `output_stride` 8 (65 x 65 for a 513 input) or 16 (33 x 33), then the mobile ASPP head (image pooling and a 1x1 branch,
    256 channels) and a bilinear Interp (align_corner) of the logits back to `size`."""
    assert output_stride in (8, 16), output_stride
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = _bn_scale_clip(m, "_conv1", m.conv("conv1", x, 32, 3, 2, 1, False))
    table = [(1, 16, 1, 1, 3), (6, 24, 2, 2, 3), (6, 32, 3, 2, 3), (6, 64, 4, 2, 3), (6, 96, 3, 1, 3), (6, 160, 3, 2, 3),
             (6, 320, 1, 1, 3)]
    _deeplabv3(m, x, table, output_stride, 256, num_classes, size)
    return m


def deeplabv3_tiny(seed=0, size=65, num_classes=5) -> ModelWriter:
    """A small DeepLab-v3 for fast tests: 65 x 65 input, at most 48 channels, output stride 8.  Its dilated depthwise
    layers run at dilation 2 and 4 (3x3, the shared-memory kernel) and one 5x5 layer at dilation 2 takes the generic one."""
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = _bn_scale_clip(m, "_conv1", m.conv("conv1", x, 8, 3, 2, 1, False))
    table = [(1, 8, 1, 1, 3), (2, 8, 1, 2, 3), (2, 16, 2, 2, 3), (2, 16, 2, 2, 3), (2, 24, 1, 1, 5), (2, 24, 2, 2, 3)]
    _deeplabv3(m, x, table, 8, 16, num_classes, size)
    return m


def _ssd_heads(m: ModelWriter, data: str, sources, num_classes: int, conf_gain: float, conf_threshold: float,
               nms_top_k: int = 100, keep_top_k: int = 100):
    """3x3 loc / conf heads and PriorBoxes on each (blob, min_sizes, max_sizes, aspect_ratios[, step]) source (a step
    writes PriorBox keys 11 / 12; without one the step is image / feature size); Permute 0=3 -> Flatten -> Concat, the
    conf branch through Reshape (w = classes) -> Softmax over the class axis -> Flatten; and DetectionOutput (nms 0.45)."""
    locs, confs, priors = [], [], []
    for src, mins, maxs, ars, *step in sources:
        per_loc = len(mins) * (1 + (1 if maxs else 0) + 2 * sum(abs(a - 1) >= 1e-6 for a in ars))
        fan_in = m.shape[src][0] * 9
        x = m.conv(f"{src}_mbox_loc", src, per_loc * 4, 3, 1, 1, True)
        locs.append(m.flatten(f"{src}_mbox_loc_flat", m.permute(f"{src}_mbox_loc_perm", x, 3)))
        x = m.conv(f"{src}_mbox_conf", src, per_loc * num_classes, 3, 1, 1, True, gain=conf_gain * np.sqrt(2.0 / fan_in))
        confs.append(m.flatten(f"{src}_mbox_conf_flat", m.permute(f"{src}_mbox_conf_perm", x, 3)))
        priors.append(m.priorbox(f"{src}_mbox_priorbox", src, data, mins, maxs, ars, flip=True, clip=False,
                                 step=(step[0], step[0]) if step else None))
    loc = m.concat("mbox_loc", locs, axis=0)
    conf = m.concat("mbox_conf", confs, axis=0)
    pri = m.concat("mbox_priorbox", priors, axis=1)
    conf = m.reshape("mbox_conf_reshape", conf, num_classes, -1)
    conf = m.softmax("mbox_conf_softmax", conf, axis=1)
    conf = m.flatten("mbox_conf_flatten", conf)
    return m.detection_output("detection_out", loc, conf, pri, num_classes, 0.45, nms_top_k, keep_top_k, conf_threshold)


def mobilenet_ssd(seed=0, size=300, num_classes=21, conf_threshold=0.25, conf_gain=1.0) -> ModelWriter:
    """MobileNet-SSD in chuanqi305's Caffe layout: the MobileNet-v1 body (conv0 .. conv13, BatchNorm + Scale + ReLU after
    every convolution), extras conv14_1/2 .. conv17_1/2 (1x1 then 3x3 stride 2), 3x3 loc and conf heads on conv11 (3 priors
    per location, min 60), conv13 (6, 105 / 150) and the four extras (150 / 195, 195 / 240, 240 / 285, 285 / 300), aspect
    ratios 2 (and 3 from conv13 on), flipped, and DetectionOutput 0=21 1=0.45 2=100 3=100.  1917 priors at 300 x 300.
    conf_gain scales the spread of the conf head's logits (more, sharper candidates above the threshold)."""
    m = ModelWriter(seed)
    data = m.input("data", 3, size, size)
    x = _bn_scale_relu(m, "_conv0", m.conv("conv0", data, 32, 3, 2, 1, False))
    cfg = [(64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1), (512, 1), (512, 1), (512, 1), (512, 1),
           (1024, 2), (1024, 1)]
    for i, (oc, s) in enumerate(cfg, 1):
        ic = m.shape[x][0]
        x = _bn_scale_relu(m, f"_conv{i}_dw", m.conv(f"conv{i}_dw", x, ic, 3, s, 1, False, group=ic))
        x = _bn_scale_relu(m, f"_conv{i}", m.conv(f"conv{i}_pw", x, oc, 1, 1, 0, False))
        if i == 11:
            conv11 = x
    conv13 = x
    extras = []
    for i, (mid, oc) in enumerate([(256, 512), (128, 256), (128, 256), (64, 128)], 14):
        x = _bn_scale_relu(m, f"_conv{i}_1", m.conv(f"conv{i}_1", x, mid, 1, 1, 0, False))
        x = _bn_scale_relu(m, f"_conv{i}_2", m.conv(f"conv{i}_2", x, oc, 3, 2, 1, False))
        extras.append(x)
    sizes = [(150, 195), (195, 240), (240, 285), (285, 300)]
    sources = [(conv11, [60.0], [], [2.0]), (conv13, [105.0], [150.0], [2.0, 3.0])]
    sources += [(e, [float(a)], [float(b)], [2.0, 3.0]) for e, (a, b) in zip(extras, sizes)]
    _ssd_heads(m, data, sources, num_classes, conf_gain, conf_threshold)
    return m


def ssd_tiny(seed=0, size=64, num_classes=5, conf_threshold=0.05, conf_gain=3.0) -> ModelWriter:
    """Two-head SSD at small size: heads on a 16 x 16 map (min 12, aspect ratio 2: 3 priors per location) and an 8 x 8 map
    (min 24, max 40, aspect ratios 2 and 3: 6 per location); 1152 priors at 64 x 64."""
    m = ModelWriter(seed)
    data = m.input("data", 3, size, size)
    x = m.relu("relu1", m.conv("conv1", data, 16, 3, 2, 1, True))
    a = m.relu("relu2", m.conv("conv2", x, 32, 3, 2, 1, True))
    b = m.relu("relu3", m.conv("conv3", a, 32, 3, 2, 1, True))
    _ssd_heads(m, data, [(a, [12.0], [], [2.0]), (b, [24.0], [40.0], [2.0, 3.0])], num_classes, conf_gain, conf_threshold)
    return m


def vgg_ssd(seed=0, size=300, num_classes=21, conf_threshold=0.01, conf_gain=1.0) -> ModelWriter:
    """VGG-SSD 300 in weiliu89's Caffe layout: VGG-16 conv1_1 .. conv5_3 with ReLU, 2x2 / 2 pool1-4 (pool3 75 -> 38 by
    ceil mode) and a 3x3 / 1 / pad 1 pool5; fc6 as a 3x3 convolution of 1024 channels with dilation 6 and pad 6, fc7 as a
    1x1 of 1024; extras conv6_1/2 (1x1 256, 3x3 / 2 / pad 1 512: 10 x 10), conv7_1/2 (128, 256 / 2: 5 x 5), conv8_1/2 and
    conv9_1/2 (128, 256 3x3 unpadded: 3 x 3, then 1 x 1); conv4_3_norm, a per-pixel Normalize of relu4_3 (eps 1e-10,
    scales 20); 3x3 loc and conf heads with PriorBoxes (flip, no clip) on conv4_3_norm (min 30, max 60, aspect ratio 2,
    step 8), fc7 (60 / 111, 2 and 3, 16), conv6_2 (111 / 162, 2 and 3, 32), conv7_2 (162 / 213, 2 and 3, 64), conv8_2
    (213 / 264, 2, 100) and conv9_2 (264 / 315, 2, 300); DetectionOutput 0=21 1=0.45 2=400 3=200.  8732 priors at
    300 x 300.  conf_gain scales the spread of the conf head's logits."""
    m = ModelWriter(seed)
    data = m.input("data", 3, size, size)
    x = data
    for si, (ch, n) in enumerate([(64, 2), (128, 2), (256, 3), (512, 3), (512, 3)], 1):
        for li in range(1, n + 1):
            x = m.relu(f"relu{si}_{li}", m.conv(f"conv{si}_{li}", x, ch, 3, 1, 1, True))
        if si == 4:
            conv4_3 = x
        x = m.pool(f"pool{si}", x, 0, 3, 1, 1) if si == 5 else m.pool(f"pool{si}", x, 0, 2, 2)
    x = m.relu("relu6", m.conv("fc6", x, 1024, 3, 1, 6, True, dilation=6))
    fc7 = x = m.relu("relu7", m.conv("fc7", x, 1024, 1, 1, 0, True))
    extras = []
    for i, (mid, oc, stride, pad) in enumerate([(256, 512, 2, 1), (128, 256, 2, 1), (128, 256, 1, 0), (128, 256, 1, 0)], 6):
        x = m.relu(f"conv{i}_1_relu", m.conv(f"conv{i}_1", x, mid, 1, 1, 0, True))
        x = m.relu(f"conv{i}_2_relu", m.conv(f"conv{i}_2", x, oc, 3, stride, pad, True))
        extras.append(x)
    norm = m.normalize("conv4_3_norm", conv4_3, across_spatial=0, channel_shared=0, eps=1e-10, scale=20.0)
    sources = [(norm, [30.0], [60.0], [2.0], 8.0), (fc7, [60.0], [111.0], [2.0, 3.0], 16.0)]
    sources += [(e, [float(a)], [float(b)], ars, float(st)) for e, (a, b, ars, st) in
                zip(extras, [(111, 162, [2.0, 3.0], 32), (162, 213, [2.0, 3.0], 64), (213, 264, [2.0], 100),
                             (264, 315, [2.0], 300)])]
    _ssd_heads(m, data, sources, num_classes, conf_gain, conf_threshold, nms_top_k=400, keep_top_k=200)
    return m


# BVLC GoogLeNet's inception modules: name, 1x1, 3x3 reduce, 3x3, 5x5 reduce, 5x5, pool projection
GOOGLENET_INCEPTIONS = [("3a", 64, 96, 128, 16, 32, 32), ("3b", 128, 128, 192, 32, 96, 64),
                        ("4a", 192, 96, 208, 16, 48, 64), ("4b", 160, 112, 224, 24, 64, 64),
                        ("4c", 128, 128, 256, 24, 64, 64), ("4d", 112, 144, 288, 32, 64, 64),
                        ("4e", 256, 160, 320, 32, 128, 128), ("5a", 256, 160, 320, 32, 128, 128),
                        ("5b", 384, 192, 384, 48, 128, 128)]


def googlenet(seed=0, num_classes=1000, size=224, lrn_alpha=1e-4) -> ModelWriter:
    """BVLC GoogLeNet (Inception-v1), deploy net without the training-only auxiliary heads: conv1/7x7_s2 (pad 3) -> ReLU ->
    pool1 3x3 / 2 -> norm1 (LRN 5, beta 0.75) -> conv2/3x3_reduce 1x1 64 -> ReLU -> conv2/3x3 192 -> ReLU -> norm2 -> pool2
    3x3 / 2; nine inception modules (GOOGLENET_INCEPTIONS: outputs 256, 480, 512, 512, 512, 528, 832, 832, 1024), each
    reading its input through an explicit 4-top Split (1x1; 3x3 reduce -> 3x3; 5x5 reduce -> 5x5; 3x3 / 1 / pad 1 max
    pool -> 1x1 projection, every convolution with a ReLU) into a 4-bottom Concat; pool3 and pool4 3x3 / 2 after 3b and
    4e; a 7x7 average pool, Dropout, the 1024 -> num_classes classifier and Softmax.  56 / 28 / 14 / 7 planes at 224.
    lrn_alpha is both LRNs' alpha (the zoo's 1e-4 barely changes the activations; near 1 the factor varies widely)."""
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = m.relu("conv1/relu_7x7", m.conv("conv1/7x7_s2", x, 64, 7, 2, 3, True))
    x = m.pool("pool1/3x3_s2", x, 0, 3, 2)
    x = m.lrn("pool1/norm1", x, 5, lrn_alpha, 0.75)
    x = m.relu("conv2/relu_3x3_reduce", m.conv("conv2/3x3_reduce", x, 64, 1, 1, 0, True))
    x = m.relu("conv2/relu_3x3", m.conv("conv2/3x3", x, 192, 3, 1, 1, True))
    x = m.lrn("conv2/norm2", x, 5, lrn_alpha, 0.75)
    x = m.pool("pool2/3x3_s2", x, 0, 3, 2)
    for tag, c1, r3, c3, r5, c5, pp in GOOGLENET_INCEPTIONS:
        if tag in ("4a", "5a"):
            x = m.pool(f"pool{int(tag[0]) - 1}/3x3_s2", x, 0, 3, 2)
        t = f"inception_{tag}"
        a, b, c, d = m.split(f"{t}/split", x, [f"{t}/split_{i}" for i in range(4)])
        a = m.relu(f"{t}/relu_1x1", m.conv(f"{t}/1x1", a, c1, 1, 1, 0, True))
        b = m.relu(f"{t}/relu_3x3_reduce", m.conv(f"{t}/3x3_reduce", b, r3, 1, 1, 0, True))
        b = m.relu(f"{t}/relu_3x3", m.conv(f"{t}/3x3", b, c3, 3, 1, 1, True))
        c = m.relu(f"{t}/relu_5x5_reduce", m.conv(f"{t}/5x5_reduce", c, r5, 1, 1, 0, True))
        c = m.relu(f"{t}/relu_5x5", m.conv(f"{t}/5x5", c, c5, 5, 1, 2, True))
        d = m.pool(f"{t}/pool", d, 0, 3, 1, 1)
        d = m.relu(f"{t}/relu_pool_proj", m.conv(f"{t}/pool_proj", d, pp, 1, 1, 0, True))
        x = m.concat(f"{t}/output", [a, b, c, d])
    x = m.pool("pool5/7x7_s1", x, 1, 7, 1)
    x = m.dropout("pool5/drop_7x7_s1", x)
    x = m.fc("loss3/classifier", x, num_classes)
    m.softmax("prob", x)
    return m


def alexnet(seed=0, num_classes=1000, size=227, lrn_alpha=1e-4) -> ModelWriter:
    """BVLC AlexNet, deploy net: conv1 11x11 / 4 96 -> ReLU -> norm1 (LRN 5, beta 0.75) -> pool1 3x3 / 2; conv2 5x5 pad 2
    256 in 2 groups -> ReLU -> norm2 -> pool2; conv3 3x3 384, conv4 3x3 384 in 2 groups, conv5 3x3 256 in 2 groups (each
    with a ReLU) -> pool5 3x3 / 2; fc6 9216 -> 4096, fc7 4096 (ReLU and Dropout after each), fc8 and Softmax.  55 / 27 /
    13 / 6 planes at 227.  lrn_alpha as in googlenet()."""
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = m.relu("relu1", m.conv("conv1", x, 96, 11, 4, 0, True))
    x = m.pool("pool1", m.lrn("norm1", x, 5, lrn_alpha, 0.75), 0, 3, 2)
    x = m.relu("relu2", m.conv("conv2", x, 256, 5, 1, 2, True, group=2))
    x = m.pool("pool2", m.lrn("norm2", x, 5, lrn_alpha, 0.75), 0, 3, 2)
    x = m.relu("relu3", m.conv("conv3", x, 384, 3, 1, 1, True))
    x = m.relu("relu4", m.conv("conv4", x, 384, 3, 1, 1, True, group=2))
    x = m.relu("relu5", m.conv("conv5", x, 256, 3, 1, 1, True, group=2))
    x = m.pool("pool5", x, 0, 3, 2)
    x = m.dropout("drop6", m.relu("relu6", m.fc("fc6", x, 4096)))
    x = m.dropout("drop7", m.relu("relu7", m.fc("fc7", x, 4096)))
    m.softmax("prob", m.fc("fc8", x, num_classes))
    return m


VOC_ANCHORS = [1.08, 1.19, 3.42, 4.41, 6.63, 11.38, 9.42, 5.11, 16.62, 10.52]  # YOLOv2 VOC, grid cells
COCO_ANCHORS = [10, 13, 16, 30, 33, 23, 30, 61, 62, 45, 59, 119, 116, 90, 156, 198, 373, 326]  # YOLOv3, input pixels


def _yolo_out(m: ModelWriter, name: str, x: str, num_box: int, num_class: int, head_gain: float, obj_bias: float) -> str:
    """The 1x1 output convolution of a YOLO head: num_box * (5 + num_class) channels, weights head_gain times He init, bias
    0 except obj_bias on each box's objectness channel (so the synthetic weights give many candidates)."""
    fan_in = m.shape[x][0]
    bias = np.zeros((num_box, 5 + num_class), np.float32)
    bias[:, 4] = obj_bias
    return m.conv(name, x, num_box * (5 + num_class), 1, 1, 0, True, gain=head_gain * np.sqrt(2.0 / fan_in),
                  bias_values=bias.reshape(-1))


def _dw_pw(m: ModelWriter, tag: str, x: str, oc: int, act) -> str:
    """Depthwise 3x3 + BatchNorm + Scale + activation, then pointwise 1x1 to oc + BatchNorm + Scale + activation."""
    ic = m.shape[x][0]
    x = act(m, f"_{tag}_dw", m.conv(f"{tag}_dw", x, ic, 3, 1, 1, False, group=ic))
    return act(m, f"_{tag}_pw", m.conv(f"{tag}_pw", x, oc, 1, 1, 0, False))


def mobilenet_yolov2(seed=0, size=416, num_classes=20, confidence_threshold=0.01, head_gain=1.0,
                     obj_bias=-3.0) -> ModelWriter:
    """MobileNet-YOLO (YOLOv2 head): the MobileNet-v1 body (conv1 .. conv14, BatchNorm + Scale + ReLU) at 416 x 416, one more
    depthwise / pointwise 1024 block on the 13 x 13 map, a 1x1 convolution to 5 x (5 + 20) channels and
    YoloDetectionOutput with the 5 VOC anchors: 845 slots."""
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = _bn_scale_relu(m, "_conv1", m.conv("conv1", x, 32, 3, 2, 1, False))
    cfg = [(64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1), (512, 1), (512, 1), (512, 1), (512, 1),
           (1024, 2), (1024, 1)]
    for i, (oc, s) in enumerate(cfg, 2):
        ic = m.shape[x][0]
        x = _bn_scale_relu(m, f"_conv{i}_dw", m.conv(f"conv{i}_dw", x, ic, 3, s, 1, False, group=ic))
        x = _bn_scale_relu(m, f"_conv{i}_pw", m.conv(f"conv{i}_pw", x, oc, 1, 1, 0, False))
    x = _dw_pw(m, "yolo_conv", x, 1024, _bn_scale_relu)
    x = _yolo_out(m, "yolo_out", x, 5, num_classes, head_gain, obj_bias)
    m.yolo_detection_output("detection_out", x, num_classes, 5, VOC_ANCHORS, confidence_threshold, 0.45)
    return m


def mobilenetv2_yolov3(seed=0, size=416, num_classes=80, confidence_threshold=0.01, head_gain=1.0,
                       obj_bias=-5.0) -> ModelWriter:
    """MobileNet-v2 YOLOv3: the MobileNet-v2 body (ReLU6 as Clip) at 416 x 416 up to conv_last (1280 x 13 x 13); heads on
    13 x 13 (conv_last), 26 x 26 (a 1x1 reduction of the 13 x 13 branch, nearest Interp x2, channel Concat with the
    96-channel stride-16 block) and 52 x 52 (likewise with the 32-channel stride-8 block), each a depthwise / pointwise
    block and a 1x1 convolution to 3 x (5 + 80); Yolov3DetectionOutput with the 9 COCO anchors, mask 6,7,8 / 3,4,5 / 0,1,2
    and anchors_scale 32, 16, 8: 10647 slots."""
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = _bn_scale_clip(m, "_conv1", m.conv("conv1", x, 32, 3, 2, 1, False))
    table = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]
    taps = {}
    for bi, (t, c, n, s) in enumerate(table, 2):
        for i in range(n):
            tag = f"{bi}_{i + 1}"
            stride = s if i == 0 else 1
            ic = m.shape[x][0]
            shortcut = stride == 1 and ic == c
            if shortcut:
                sc, x = m.split(f"block{tag}_split", x, [f"block{tag}_in_a", f"block{tag}_in_b"])
            y = x
            if t != 1:
                y = _bn_scale_clip(m, f"_conv{tag}_expand", m.conv(f"conv{tag}_expand", y, ic * t, 1, 1, 0, False))
            y = _bn_scale_clip(m, f"_conv{tag}_dw", m.conv(f"conv{tag}_dw", y, ic * t, 3, stride, 1, False, group=ic * t))
            y = m.conv(f"conv{tag}_linear", y, c, 1, 1, 0, False)
            y = _bn_scale_clip(m, f"_conv{tag}_linear", y, clip=False, center=0.3 if shortcut else 1.0)
            x = m.eltwise(f"block{tag}", [sc, y]) if shortcut else y
        taps[bi] = x
    x = _bn_scale_clip(m, "_conv_last", m.conv("conv_last", x, 1280, 1, 1, 0, False))
    anchors_mask = [6, 7, 8, 3, 4, 5, 0, 1, 2]
    outs = []
    h = _dw_pw(m, "yolo13", x, 512, _bn_scale_clip)
    outs.append(_yolo_out(m, "yolo13_out", h, 3, num_classes, head_gain, obj_bias))
    for grid, tap, mid, width in ((26, taps[6], 128, 192), (52, taps[4], 64, 96)):
        u = _bn_scale_clip(m, f"_up{grid}_reduce", m.conv(f"up{grid}_reduce", x, mid, 1, 1, 0, False))
        u = m.interp(f"up{grid}", u, 1, scale=2.0)
        x = m.concat(f"cat{grid}", [u, tap])
        h = _dw_pw(m, f"yolo{grid}", x, width, _bn_scale_clip)
        outs.append(_yolo_out(m, f"yolo{grid}_out", h, 3, num_classes, head_gain, obj_bias))
    m.yolov3_detection_output("detection_out", outs, num_classes, 3, COCO_ANCHORS, anchors_mask, [32.0, 16.0, 8.0],
                              confidence_threshold, 0.45)
    return m


def yolo_tiny(seed=0, size=64, num_classes=5, confidence_threshold=0.05, head_gain=1.0, obj_bias=-2.0) -> ModelWriter:
    """Two-scale YOLOv3 head at small size: 8 x 8 and 16 x 16 maps (the second through nearest Interp x2 and Concat),
    3 anchors each, 5 classes, anchors_scale 8 and 4: 960 slots at 64 x 64."""
    m = ModelWriter(seed)
    x = m.input("data", 3, size, size)
    x = m.relu("relu1", m.conv("conv1", x, 16, 3, 2, 1, True))
    a = m.relu("relu2", m.conv("conv2", x, 32, 3, 2, 1, True))
    b = m.relu("relu3", m.conv("conv3", a, 64, 3, 2, 1, True))
    o8 = _yolo_out(m, "yolo8_out", b, 3, num_classes, head_gain, obj_bias)
    u = m.interp("up16", m.relu("up16_relu", m.conv("up16_reduce", b, 16, 1, 1, 0, True)), 1, scale=2.0)
    x = m.relu("yolo16_relu", m.conv("yolo16_conv", m.concat("cat16", [u, a]), 32, 3, 1, 1, True))
    o16 = _yolo_out(m, "yolo16_out", x, 3, num_classes, head_gain, obj_bias)
    m.yolov3_detection_output("detection_out", [o8, o16], num_classes, 3, [4, 6, 8, 10, 12, 9, 16, 20, 24, 18, 32, 40],
                              [3, 4, 5, 0, 1, 2], [8.0, 4.0], confidence_threshold, 0.45)
    return m


def _rpn(m: ModelWriter, feat: str, rpn_width: int, feat_stride: int, base_size: int, pre_nms_top_n: int,
         post_nms_top_n: int, min_size: int, rpn_cls_gain: float, rpn_bbox_gain: float) -> str:
    """py-faster-rcnn's region proposal network on `feat`: rpn_conv/3x3 + ReLU; rpn_cls_score (2 x 9) and rpn_bbox_pred
    (4 x 9) 1x1 convolutions; Reshape (2, -1, W) -> Softmax over the channel axis -> Reshape (18, -1, W); Proposal (nms
    0.7) on im_info.  The gains multiply He init: rpn_cls_gain spreads the objectness logits, rpn_bbox_gain keeps the box
    deltas small so the boxes stay finite and neighbouring anchors overlap.  Returns the rois blob."""
    fan_in = rpn_width
    x = m.relu("rpn_relu/3x3", m.conv("rpn_conv/3x3", feat, rpn_width, 3, 1, 1, True))
    cls = m.conv("rpn_cls_score", x, 18, 1, 1, 0, True, gain=rpn_cls_gain * np.sqrt(2.0 / fan_in))
    bbox = m.conv("rpn_bbox_pred", x, 36, 1, 1, 0, True, gain=rpn_bbox_gain * np.sqrt(2.0 / fan_in),
                  bias_values=np.zeros(36, np.float32))
    cls = m.reshape("rpn_cls_score_reshape", cls, 0, -1, 2)
    cls = m.softmax("rpn_cls_prob", cls, axis=0)
    cls = m.reshape("rpn_cls_prob_reshape", cls, 0, -1, 18)
    return m.proposal("proposal", cls, bbox, "im_info", feat_stride, base_size, pre_nms_top_n, post_nms_top_n, 0.7,
                      min_size, tops=["rois"])


def _faster_rcnn_head(m: ModelWriter, feat: str, num_classes: int, rpn_width: int, fc_width: int, feat_stride: int,
                      base_size: int, pre_nms_top_n: int, post_nms_top_n: int, min_size: int, pooled: int,
                      rpn_cls_gain: float, rpn_bbox_gain: float):
    """py-faster-rcnn's test net after the backbone: _rpn; ROIPooling pooled x pooled at 1 / feat_stride; fc6 and fc7
    (ReLU, Dropout); cls_score -> Softmax (cls_prob) and bbox_pred."""
    rois = _rpn(m, feat, rpn_width, feat_stride, base_size, pre_nms_top_n, post_nms_top_n, min_size, rpn_cls_gain,
                rpn_bbox_gain)
    x = m.roi_pooling("roi_pool5", feat, rois, pooled, pooled, 1.0 / feat_stride, top="pool5")
    x = m.dropout("drop6", m.relu("relu6", m.fc("fc6", x, fc_width)))
    x = m.dropout("drop7", m.relu("relu7", m.fc("fc7", x, fc_width)))
    m.softmax("cls_prob", m.fc("cls_score", x, num_classes))
    m.fc("bbox_pred", x, 4 * num_classes)


def faster_rcnn_vgg16(seed=0, height=600, width=800, num_classes=21, pre_nms_top_n=6000, post_nms_top_n=300,
                      rpn_cls_gain=1.0, rpn_bbox_gain=0.1) -> ModelWriter:
    """py-faster-rcnn's VGG-16 Faster R-CNN test net: Input data (3, height, width) and Input im_info (3 values per image:
    height, width, scale), VGG-16 conv1_1 .. conv5_3 with ReLU and the four 2x2 / 2 pools (conv5_3 at 1 / 16: 38 x 50 at
    600 x 800, 17,100 anchors), then _faster_rcnn_head: RPN 512 wide, Proposal 16 / 16 / pre_nms_top_n / post_nms_top_n /
    0.7 / 16, ROIPooling 7 x 7, fc6 25088 -> 4096, fc7 4096, cls_score num_classes and bbox_pred 4 x num_classes.  fc6
    to bbox_pred run once over batch x post_nms_top_n RoIs."""
    m = ModelWriter(seed)
    x = m.input("data", 3, height, width)
    m.extra_input("im_info")
    for si, (ch, n) in enumerate([(64, 2), (128, 2), (256, 3), (512, 3), (512, 3)], 1):
        for li in range(1, n + 1):
            x = m.relu(f"relu{si}_{li}", m.conv(f"conv{si}_{li}", x, ch, 3, 1, 1, True))
        if si < 5:
            x = m.pool(f"pool{si}", x, 0, 2, 2)
    _faster_rcnn_head(m, x, num_classes, 512, 4096, 16, 16, pre_nms_top_n, post_nms_top_n, 16, 7, rpn_cls_gain,
                      rpn_bbox_gain)
    return m


def faster_rcnn_tiny(seed=0, height=96, width=128, num_classes=5, pre_nms_top_n=2000, post_nms_top_n=64,
                     rpn_cls_gain=1.0, rpn_bbox_gain=0.1) -> ModelWriter:
    """Faster R-CNN at float64-checkable size: two 3x3 / 2 convolutions (16, 32 channels, ReLU) to a 1 / 4 map (24 x 32 at
    96 x 128: 6,912 anchors), then _faster_rcnn_head with RPN width 32, Proposal feat_stride 4, base_size 2 (anchors 24 to
    96 pixels wide), min_size 4, ROIPooling 4 x 4 at 1 / 4, fc6 / fc7 64 wide."""
    m = ModelWriter(seed)
    x = m.input("data", 3, height, width)
    m.extra_input("im_info")
    x = m.relu("relu1", m.conv("conv1", x, 16, 3, 2, 1, True))
    x = m.relu("relu2", m.conv("conv2", x, 32, 3, 2, 1, True))
    _faster_rcnn_head(m, x, num_classes, 32, 64, 4, 2, pre_nms_top_n, post_nms_top_n, 4, 4, rpn_cls_gain, rpn_bbox_gain)
    return m


def _rfcn_head(m: ModelWriter, feat: str, rois: str, num_classes: int, width: int, pooled: int, feat_stride: int):
    """py-R-FCN's test net after the trunk: conv_new_1 (1x1, width) + ReLU; the position-sensitive score maps rfcn_cls
    (pooled^2 x num_classes) and rfcn_bbox (pooled^2 x 8: class-agnostic boxes) as 1x1 convolutions; PSROIPooling of both
    pooled x pooled at 1 / feat_stride; the vote, a pooled x pooled / pooled average Pooling, to cls_score and bbox_pred;
    cls_score -> Softmax (cls_prob)."""
    x = m.relu("conv_new_1_relu", m.conv("conv_new_1", feat, width, 1, 1, 0, True))
    cls = m.conv("rfcn_cls", x, pooled * pooled * num_classes, 1, 1, 0, True)
    loc = m.conv("rfcn_bbox", x, pooled * pooled * 8, 1, 1, 0, True)
    cls = m.psroi_pooling("psroipooled_cls_rois", cls, rois, num_classes, pooled, pooled, 1.0 / feat_stride)
    loc = m.psroi_pooling("psroipooled_loc_rois", loc, rois, 8, pooled, pooled, 1.0 / feat_stride)
    cls = m.pool("ave_cls_score_rois", cls, 1, pooled, pooled, top="cls_score")
    m.pool("ave_bbox_pred_rois", loc, 1, pooled, pooled, top="bbox_pred")
    m.softmax("cls_prob", cls)


def rfcn_resnet50(seed=0, height=600, width=800, num_classes=21, pre_nms_top_n=6000, post_nms_top_n=300,
                  rpn_cls_gain=1.0, rpn_bbox_gain=0.1) -> ModelWriter:
    """py-R-FCN's ResNet-50 rfcn_end2end test net: Input data (3, height, width) and Input im_info; Caffe ResNet-50 with
    res5 at stride 1 (res5a_branch1 and res5a_branch2a stride 1, every res5 3x3 at dilation 2 and pad 2), so res4f and
    res5c are both at 1 / 16 (38 x 50 at 600 x 800); _rpn on res4f (512 wide, Proposal 16 / 16 / pre_nms_top_n /
    post_nms_top_n / 0.7 / 16); _rfcn_head on res5c: conv_new_1 1024, rfcn_cls 7 x 7 x num_classes, rfcn_bbox 7 x 7 x 8,
    PSROIPooling 7 x 7 at 1 / 16 and the 7 x 7 average vote, over batch x post_nms_top_n RoIs."""
    m = ModelWriter(seed)
    x = m.input("data", 3, height, width)
    m.extra_input("im_info")
    x = _resnet50_trunk(m, x, strides=(1, 2, 2, 1), dilations=(1, 1, 1, 2))
    rois = _rpn(m, "res4f_relu", 512, 16, 16, pre_nms_top_n, post_nms_top_n, 16, rpn_cls_gain, rpn_bbox_gain)
    _rfcn_head(m, x, rois, num_classes, 1024, 7, 16)
    return m


def rfcn_tiny(seed=0, height=96, width=128, num_classes=5, pre_nms_top_n=2000, post_nms_top_n=64, rpn_cls_gain=1.0,
              rpn_bbox_gain=0.1) -> ModelWriter:
    """R-FCN at float64-checkable size: two 3x3 / 2 convolutions (16, 32 channels, ReLU) to a 1 / 4 map (24 x 32 at
    96 x 128: 6,912 anchors) and a 3x3 convolution at dilation 2 (32 channels, ReLU); _rpn on it (32 wide, feat_stride 4,
    base_size 2, min_size 4); _rfcn_head with conv_new_1 64 wide, PSROIPooling 3 x 3 at 1 / 4 (rfcn_cls 9 x num_classes,
    rfcn_bbox 72 channels) and the 3 x 3 vote."""
    m = ModelWriter(seed)
    x = m.input("data", 3, height, width)
    m.extra_input("im_info")
    x = m.relu("relu1", m.conv("conv1", x, 16, 3, 2, 1, True))
    x = m.relu("relu2", m.conv("conv2", x, 32, 3, 2, 1, True))
    x = m.relu("relu3", m.conv("conv3", x, 32, 3, 1, 2, True, dilation=2))
    rois = _rpn(m, x, 32, 4, 2, pre_nms_top_n, post_nms_top_n, 4, rpn_cls_gain, rpn_bbox_gain)
    _rfcn_head(m, x, rois, num_classes, 64, 3, 4)
    return m


def _style_conv(m: ModelWriter, name: str, x: str, oc: int, k: int, stride: int = 1) -> str:
    """TransformerNet's ConvLayer: a reflect Padding of k // 2 on every side, then the convolution with pad 0."""
    return m.conv(name, m.padding(name + "_pad", x, k // 2, k // 2, k // 2, k // 2), oc, k, stride, 0, True)


def _transformer_net(m: ModelWriter, x: str, widths, blocks: int) -> str:
    """The PyTorch examples' fast-neural-style TransformerNet on widths (w1, w2, w3): conv 9x9 3 -> w1, conv 3x3 / 2 to
    w2 and to w3, `blocks` residual blocks (conv, IN, ReLU, conv, IN, then the Eltwise SUM skip), twice nearest x2
    Interp, conv 3x3 and IN (w3 -> w2 -> w1), and a 9x9 w1 -> 3 output convolution.  Every convolution but the last is
    followed by an affine InstanceNorm, and every InstanceNorm by a ReLU except the second of each residual block."""
    w1, w2, w3 = widths
    for i, (oc, k, s) in enumerate(((w1, 9, 1), (w2, 3, 2), (w3, 3, 2)), 1):
        x = m.relu(f"relu{i}", m.instance_norm(f"in{i}", _style_conv(m, f"conv{i}", x, oc, k, s)))
    for b in range(1, blocks + 1):
        a, c = m.split(f"res{b}_split", x, [f"res{b}_in_a", f"res{b}_in_b"])
        y = m.relu(f"res{b}_relu1", m.instance_norm(f"res{b}_in1", _style_conv(m, f"res{b}_conv1", c, w3, 3)))
        y = m.instance_norm(f"res{b}_in2", _style_conv(m, f"res{b}_conv2", y, w3, 3))
        x = m.add(f"res{b}", [a, y])
    for i, oc in ((4, w2), (5, w1)):
        x = m.interp(f"up{i}", x, resize_type=1, scale=2.0)
        x = m.relu(f"relu{i}", m.instance_norm(f"in{i}", _style_conv(m, f"conv{i}", x, oc, 3)))
    return _style_conv(m, "conv6", x, 3, 9)


def fast_neural_style(seed=0, height=512, width=512, adds="eltwise") -> ModelWriter:
    """Johnson et al.'s fast neural style transfer network in the layout of the PyTorch examples' TransformerNet: 32,
    64 and 128 channels, five residual blocks, nearest x2 upsampling.  The output (`conv6`) is shaped like the input.
    adds="binaryop" writes the residual sums as BinaryOp ADD (an ONNX export's layout), the same .bin."""
    assert height % 4 == 0 and width % 4 == 0, (height, width)
    m = ModelWriter(seed, adds=adds)
    _transformer_net(m, m.input("data", 3, height, width), (32, 64, 128), 5)
    return m


def style_tiny(seed=0, height=32, width=32, adds="eltwise") -> ModelWriter:
    """fast_neural_style's layout at float64-checkable size: 8, 16 and 16 channels, two residual blocks (the second
    block's first Padding reads an Eltwise), both upsamples."""
    assert height % 4 == 0 and width % 4 == 0, (height, width)
    m = ModelWriter(seed, adds=adds)
    _transformer_net(m, m.input("data", 3, height, width), (8, 16, 16), 2)
    return m


def srvgg_compact(seed=0, scale=4, num_conv=16, num_feat=64, height=270, width=480, adds="eltwise") -> ModelWriter:
    """Real-ESRGAN's SRVGGNetCompact (basicsr): conv 3 -> num_feat and PReLU, num_conv x (conv num_feat -> num_feat,
    PReLU), conv num_feat -> 3 scale^2 and PixelShuffle(scale), plus the input upsampled by a nearest Interp x scale,
    added by an Eltwise SUM.  The defaults are realesr-animevideov3; num_conv=32 gives realesr-general-x4v3.  The output
    (`output`) is (3, height * scale, width * scale).  adds="binaryop" writes the tail's sum as BinaryOp ADD (a pnnx or
    ONNX export's layout), the same .bin."""
    m = ModelWriter(seed, adds=adds)
    x, skip = m.split("data_split", m.input("data", 3, height, width), ["data_body", "data_skip"])
    x = m.prelu("prelu0", m.conv("conv0", x, num_feat, 3, 1, 1), slopes=np.full(num_feat, 0.25))
    for i in range(1, num_conv + 1):
        x = m.prelu(f"prelu{i}", m.conv(f"conv{i}", x, num_feat, 3, 1, 1), slopes=np.full(num_feat, 0.25))
    x = m.pixel_shuffle("upsample", m.conv("conv_last", x, 3 * scale * scale, 3, 1, 1), scale)
    base = m.interp("base", skip, resize_type=1, scale=float(scale))
    m.add("output", [x, base])
    return m


EDSR_RGB_MEAN = (0.4488, 0.4371, 0.4040)


def _edsr_upsampler(m: ModelWriter, x: str, scale: int, n_feats: int) -> str:
    """EDSR's Upsampler: log2(scale) x (conv n_feats -> 4 n_feats, PixelShuffle 2) for 2, 4, 8; conv to 9 n_feats and
    PixelShuffle 3 for 3."""
    if scale == 3:
        return m.pixel_shuffle("up_shuffle1", m.conv("up_conv1", x, 9 * n_feats, 3, 1, 1), 3)
    assert scale in (2, 4, 8), scale
    for i in range(1, int(math.log2(scale)) + 1):
        x = m.pixel_shuffle(f"up_shuffle{i}", m.conv(f"up_conv{i}", x, 4 * n_feats, 3, 1, 1), 2)
    return x


def edsr_baseline(seed=0, scale=4, n_resblocks=16, n_feats=64, height=270, width=480, rgb_range=255.0,
                  res_gain=0.1, adds="eltwise") -> ModelWriter:
    """EDSR baseline (Lim et al. 2017): MeanShift (sub_mean) as a fixed 1x1 convolution, the head conv 3 -> n_feats,
    n_resblocks x (conv, ReLU, conv, + skip), a conv plus the global skip, the upsampler (_edsr_upsampler), the tail conv
    n_feats -> 3 and add_mean.  Each residual block's second convolution draws its weights at res_gain times He init, so
    the activations stay in range over depth as trained weights keep them.  The output (`add_mean`) is
    (3, height * scale, width * scale).  adds="binaryop" writes the residual sums as BinaryOp ADD, the same .bin."""
    m = ModelWriter(seed, adds=adds)
    mean = rgb_range * np.asarray(EDSR_RGB_MEAN)
    x = m.fixed_conv1x1("sub_mean", m.input("data", 3, height, width), np.eye(3), -mean)
    x, head = m.split("head_split", m.conv("head", x, n_feats, 3, 1, 1), ["body_in", "head_skip"])
    for b in range(1, n_resblocks + 1):
        a, c = m.split(f"res{b}_split", x, [f"res{b}_in", f"res{b}_skip"])
        y = m.relu(f"res{b}_relu", m.conv(f"res{b}_conv1", a, n_feats, 3, 1, 1))
        y = m.conv(f"res{b}_conv2", y, n_feats, 3, 1, 1, gain=res_gain * np.sqrt(2.0 / (9 * n_feats)))
        x = m.add(f"res{b}", [c, y])
    x = m.add("body", [head, m.conv("body_conv", x, n_feats, 3, 1, 1)])
    x = m.conv("tail", _edsr_upsampler(m, x, scale, n_feats), 3, 3, 1, 1)
    m.fixed_conv1x1("add_mean", x, np.eye(3), mean)
    return m


def sr_tiny(seed=0, height=9, width=11, adds="eltwise") -> ModelWriter:
    """PixelShuffle at float64-checkable size, odd height and width: conv 3 -> 8 and PReLU, conv to 32 and PixelShuffle 2
    in mode 1 (DepthToSpace DCR) feeding conv 8 -> 27, PixelShuffle 3 in mode 0, and SRVGGNetCompact's tail: the input
    upsampled x 6 by a nearest Interp and added by an Eltwise SUM, which fuses into the second PixelShuffle.  The output
    (`output`) is (3, 6 height, 6 width)."""
    m = ModelWriter(seed, adds=adds)
    x, skip = m.split("data_split", m.input("data", 3, height, width), ["data_body", "data_skip"])
    x = m.prelu("prelu0", m.conv("conv0", x, 8, 3, 1, 1))
    x = m.pixel_shuffle("shuffle1", m.conv("conv1", x, 32, 3, 1, 1), 2, mode=1)
    x = m.pixel_shuffle("shuffle2", m.conv("conv2", x, 27, 3, 1, 1), 3)
    base = m.interp("base", skip, resize_type=1, scale=6.0)
    m.add("output", [x, base])
    return m


def make_divisible(v: float, divisor: int = 8) -> int:
    """torchvision's _make_divisible: the nearest multiple of divisor, at least divisor and not below 90 % of v."""
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


def _conv_bn(m: ModelWriter, name: str, x: str, oc: int, k: int, stride: int, eps: float, group: int = 1,
             act: str | None = None) -> str:
    """torchvision's Conv2dNormActivation as pnnx exports it: a convolution without bias, BatchNorm + Scale with eps, then
    the activation layer ("ReLU", or an ncnn activation type)."""
    x = m.conv(name, x, oc, k, stride, (k - 1) // 2, False, group=group)
    x = m.scale(name + "_scale", m.batchnorm(name + "_bn", x, eps=eps), True)
    if act == "ReLU":
        x = m.relu(name + "_relu", x)
    elif act in ("HardSwish", "HardSigmoid"):
        x = m.hard(act, name + "_hs", x)
    elif act is not None:
        x = m.activation(act, name + "_" + act.lower(), x)
    return x


def _squeeze_excitation(m: ModelWriter, name: str, x: str, squeeze: int, act: str, gate: str) -> str:
    """SE block: Split, global average Pooling, 1 x 1 Convolution (bias), `act`, 1 x 1 Convolution (bias), `gate`, and
    BinaryOp MUL of the (C, 1, 1) gate and the block's activation, the gate first (torchvision's `scale * input`)."""
    c = m.shape[x][0]
    a, b = m.split(name + "_split", x, [name + "_in", name + "_sq"])
    g = m.pool(name + "_pool", b, 1, 1, 1, 0, global_pooling=True)
    g = m.conv(name + "_fc1", g, squeeze, 1, 1, 0, True)
    g = m.relu(name + "_relu", g) if act == "ReLU" else m.activation(act, name + "_" + act.lower(), g)
    g = m.conv(name + "_fc2", g, c, 1, 1, 0, True)
    g = m.hard(gate, name + "_gate", g) if gate == "HardSigmoid" else m.activation(gate, name + "_gate", g)
    return m.binary_op(name + "_mul", [g, a], 2)


# (input_c, kernel, expanded_c, out_c, use_se, activation, stride) of torchvision's _mobilenet_v3_conf
MOBILENET_V3_LARGE = [(16, 3, 16, 16, False, "RE", 1), (16, 3, 64, 24, False, "RE", 2), (24, 3, 72, 24, False, "RE", 1),
                      (24, 5, 72, 40, True, "RE", 2), (40, 5, 120, 40, True, "RE", 1), (40, 5, 120, 40, True, "RE", 1),
                      (40, 3, 240, 80, False, "HS", 2), (80, 3, 200, 80, False, "HS", 1),
                      (80, 3, 184, 80, False, "HS", 1), (80, 3, 184, 80, False, "HS", 1),
                      (80, 3, 480, 112, True, "HS", 1), (112, 3, 672, 112, True, "HS", 1),
                      (112, 5, 672, 160, True, "HS", 2), (160, 5, 960, 160, True, "HS", 1),
                      (160, 5, 960, 160, True, "HS", 1)]
MOBILENET_V3_SMALL = [(16, 3, 16, 16, True, "RE", 2), (16, 3, 72, 24, False, "RE", 2), (24, 3, 88, 24, False, "RE", 1),
                      (24, 5, 96, 40, True, "HS", 2), (40, 5, 240, 40, True, "HS", 1), (40, 5, 240, 40, True, "HS", 1),
                      (40, 5, 120, 48, True, "HS", 1), (48, 5, 144, 48, True, "HS", 1), (48, 5, 288, 96, True, "HS", 2),
                      (96, 5, 576, 96, True, "HS", 1), (96, 5, 576, 96, True, "HS", 1)]


def _mobilenet_v3(table, last_channel: int, seed: int, num_classes: int, size: int) -> ModelWriter:
    m = ModelWriter(seed)
    x = _conv_bn(m, "conv_stem", m.input("data", 3, size, size), 16, 3, 2, 1e-3, act="HardSwish")
    for i, (ic, k, exp, oc, se, act, stride) in enumerate(table, 1):
        act = "ReLU" if act == "RE" else "HardSwish"
        res = stride == 1 and ic == oc
        if res:
            sc, x = m.split(f"block{i}_split", x, [f"block{i}_skip", f"block{i}_body"])
        y = x
        if exp != ic:
            y = _conv_bn(m, f"block{i}_expand", y, exp, 1, 1, 1e-3, act=act)
        y = _conv_bn(m, f"block{i}_dw", y, exp, k, stride, 1e-3, group=exp, act=act)
        if se:
            y = _squeeze_excitation(m, f"block{i}_se", y, make_divisible(exp / 4), "ReLU", "HardSigmoid")
        y = _conv_bn(m, f"block{i}_project", y, oc, 1, 1, 1e-3)
        x = m.binary_op(f"block{i}_add", [sc, y], 0) if res else y
    x = _conv_bn(m, "conv_last", x, 6 * m.shape[x][0], 1, 1, 1e-3, act="HardSwish")
    x = m.pool("pool", x, 1, 1, 1, 0, global_pooling=True)
    x = m.hard("HardSwish", "fc1_hs", m.fc("fc1", x, last_channel))
    x = m.fc("fc2", x, num_classes)
    m.softmax("prob", x)
    return m


def mobilenet_v3_large(seed=0, num_classes=1000, size=224) -> ModelWriter:
    """MobileNet-v3 Large (Howard et al. 2019) in torchvision's layout as pnnx exports it: every convolution followed by
    BatchNorm + Scale (eps 1e-3), HardSwish / ReLU as the block table says, squeeze-and-excitation with a
    make_divisible(expanded / 4, 8) squeeze, ReLU and a HardSigmoid gate, BinaryOp ADD shortcuts, and the classifier
    InnerProduct 1280, HardSwish, InnerProduct, Softmax."""
    return _mobilenet_v3(MOBILENET_V3_LARGE, 1280, seed, num_classes, size)


def mobilenet_v3_small(seed=0, num_classes=1000, size=224) -> ModelWriter:
    """MobileNet-v3 Small, as mobilenet_v3_large with the small block table and a 1024-wide classifier."""
    return _mobilenet_v3(MOBILENET_V3_SMALL, 1024, seed, num_classes, size)


# (expand_ratio, kernel, stride, input_channels, out_channels, num_layers) of torchvision's efficientnet_b0
EFFICIENTNET_B0 = [(1, 3, 1, 32, 16, 1), (6, 3, 2, 16, 24, 2), (6, 5, 2, 24, 40, 2), (6, 3, 2, 40, 80, 3),
                   (6, 5, 1, 80, 112, 3), (6, 5, 2, 112, 192, 4), (6, 3, 1, 192, 320, 1)]


def efficientnet_b0(seed=0, num_classes=1000, size=224) -> ModelWriter:
    """EfficientNet-B0 (Tan & Le 2019) in torchvision's layout as pnnx exports it: SiLU as Swish, every convolution
    followed by BatchNorm + Scale (eps 1e-5), seven MBConv stages (3 x 3 and 5 x 5 depthwise), squeeze-and-excitation
    with a max(1, input / 4) squeeze of the block input, Swish and a Sigmoid gate, BinaryOp ADD shortcuts, a 1280-channel
    head, global average pooling, InnerProduct and Softmax."""
    m = ModelWriter(seed)
    x = _conv_bn(m, "conv_stem", m.input("data", 3, size, size), 32, 3, 2, 1e-5, act="Swish")
    i = 0
    for t, k, s, ic0, oc, n in EFFICIENTNET_B0:
        for j in range(n):
            i += 1
            ic, stride = (ic0, s) if j == 0 else (oc, 1)
            exp = make_divisible(ic * t)
            res = stride == 1 and ic == oc
            if res:
                sc, x = m.split(f"block{i}_split", x, [f"block{i}_skip", f"block{i}_body"])
            y = x
            if exp != ic:
                y = _conv_bn(m, f"block{i}_expand", y, exp, 1, 1, 1e-5, act="Swish")
            y = _conv_bn(m, f"block{i}_dw", y, exp, k, stride, 1e-5, group=exp, act="Swish")
            y = _squeeze_excitation(m, f"block{i}_se", y, max(1, ic // 4), "Swish", "Sigmoid")
            y = _conv_bn(m, f"block{i}_project", y, oc, 1, 1, 1e-5)
            x = m.binary_op(f"block{i}_add", [sc, y], 0) if res else y
    x = _conv_bn(m, "conv_last", x, 1280, 1, 1, 1e-5, act="Swish")
    x = m.pool("pool", x, 1, 1, 1, 0, global_pooling=True)
    x = m.fc("fc", x, num_classes)
    m.softmax("prob", x)
    return m


def espcn(seed=0, scale=3, height=360, width=640) -> ModelWriter:
    """ESPCN (Shi et al. 2016) on the Y channel: 5 x 5 / 64 + TanH, 3 x 3 / 32 + TanH, 3 x 3 / scale^2, PixelShuffle
    scale.  The output (`output`) is (1, scale height, scale width)."""
    m = ModelWriter(seed)
    x = m.input("data", 1, height, width)
    x = m.activation("TanH", "tanh1", m.conv("conv1", x, 64, 5, 1, 2))
    x = m.activation("TanH", "tanh2", m.conv("conv2", x, 32, 3, 1, 1))
    m.pixel_shuffle("output", m.conv("conv3", x, scale * scale, 3, 1, 1), scale)
    return m


def se_tiny(seed=0, size=16, classes=10) -> ModelWriter:
    """All five activation types at float64-checkable size: a 3 x 3 stem with BatchNorm + Scale + HardSwish, a 5 x 5
    stride-2 depthwise layer + Swish, an SE gate (ReLU, HardSigmoid), a linear projection, a block with a Sigmoid branch
    added back by BinaryOp ADD, TanH, global pooling, InnerProduct and Softmax."""
    m = ModelWriter(seed)
    x = _conv_bn(m, "stem", m.input("data", 3, size, size), 16, 3, 1, 1e-3, act="HardSwish")
    x = _conv_bn(m, "dw", x, 16, 5, 2, 1e-3, group=16, act="Swish")
    x = _squeeze_excitation(m, "se", x, 8, "ReLU", "HardSigmoid")
    x = _conv_bn(m, "project", x, 16, 1, 1, 1e-3)
    sc, x = m.split("block_split", x, ["block_skip", "block_body"])
    x = _conv_bn(m, "branch", x, 16, 1, 1, 1e-3, act="Sigmoid")
    x = m.activation("TanH", "tanh", m.binary_op("add", [sc, x], 0))
    x = m.pool("pool", x, 1, 1, 1, 0, global_pooling=True)
    m.softmax("prob", m.fc("fc", x, classes))
    return m



def vit(patch=16, dim=768, depth=12, heads=12, mlp_dim=3072, size=224, classes=1000, seed=0) -> ModelWriter:
    """torchvision's VisionTransformer as pnnx exports it: the patch convolution, Reshape + Permute 0=1 to tokens, a
    MemoryData class token concatenated in front, a MemoryData position embedding added by BinaryOp; per encoder block
    LayerNorm (eps 1e-6), MultiHeadAttention, BinaryOp ADD, LayerNorm, InnerProduct, GELU, InnerProduct, BinaryOp ADD;
    the final LayerNorm, the class token cut out by Crop 1=0 4=1, and the InnerProduct head (`logits`)."""
    m = ModelWriter(seed)
    g = size // patch
    x = m.input("data", 3, size, size)
    x = m.conv("conv_proj", x, dim, patch, patch, 0, gain=np.sqrt(1.0 / (3 * patch * patch)))
    x = m.permute("tokens", m.reshape("flatten", x, g * g, dim), 1)
    x = m.concat("cat_cls", [m.memory_data("class_token", dim, 1), x], axis=0)
    x = m.binary_op("add_pos", [x, m.memory_data("pos_embedding", dim, g * g + 1)], 0)
    for i in range(depth):
        b = f"layer{i}"
        skip, x = m.split(f"{b}_split1", x, [f"{b}_skip1", f"{b}_in1"])
        x = m.multihead_attention(f"{b}_attn", m.layer_norm(f"{b}_ln1", x), heads)
        x = m.binary_op(f"{b}_add1", [skip, x], 0)
        skip, x = m.split(f"{b}_split2", x, [f"{b}_skip2", f"{b}_in2"])
        x = m.gelu(f"{b}_gelu", m.linear(f"{b}_fc1", m.layer_norm(f"{b}_ln2", x), mlp_dim))
        x = m.binary_op(f"{b}_add2", [skip, m.linear(f"{b}_fc2", x, dim)], 0)
    x = m.crop("cls", m.layer_norm("ln", x), hoff=0, outh=1)
    m.fc("logits", x, classes)
    return m


def vit_b_16(seed=0, size=224, classes=1000) -> ModelWriter:
    """ViT-B/16: 768 wide, 12 blocks of 12 heads (head_dim 64), MLP 3072."""
    return vit(16, 768, 12, 12, 3072, size, classes, seed)


def vit_s_16(seed=0, size=224, classes=1000) -> ModelWriter:
    """ViT-S/16 (DeiT-S's shape): 384 wide, 12 blocks of 6 heads (head_dim 64), MLP 1536."""
    return vit(16, 384, 12, 6, 1536, size, classes, seed)


def vit_ti_16(seed=0, size=224, classes=1000) -> ModelWriter:
    """ViT-Ti/16 (DeiT-Ti's shape): 192 wide, 12 blocks of 3 heads (head_dim 64), MLP 768."""
    return vit(16, 192, 12, 3, 768, size, classes, seed)


def vit_tiny(seed=0, size=32, classes=10) -> ModelWriter:
    """A ViT at float64-checkable size: 8 x 8 patches of a 32 x 32 image (17 tokens), 64 wide, three blocks of 4, 2 and
    1 heads (head_dim 16, 32 and 64), MLP 128."""
    m = ModelWriter(seed)
    patch, dim, g = 8, 64, size // 8
    x = m.input("data", 3, size, size)
    x = m.conv("conv_proj", x, dim, patch, patch, 0, gain=np.sqrt(1.0 / (3 * patch * patch)))
    x = m.permute("tokens", m.reshape("flatten", x, g * g, dim), 1)
    x = m.concat("cat_cls", [m.memory_data("class_token", dim, 1), x], axis=0)
    x = m.binary_op("add_pos", [x, m.memory_data("pos_embedding", dim, g * g + 1)], 0)
    for i, heads in enumerate((4, 2, 1)):
        b = f"layer{i}"
        skip, x = m.split(f"{b}_split1", x, [f"{b}_skip1", f"{b}_in1"])
        x = m.multihead_attention(f"{b}_attn", m.layer_norm(f"{b}_ln1", x), heads)
        x = m.binary_op(f"{b}_add1", [skip, x], 0)
        skip, x = m.split(f"{b}_split2", x, [f"{b}_skip2", f"{b}_in2"])
        x = m.gelu(f"{b}_gelu", m.linear(f"{b}_fc1", m.layer_norm(f"{b}_ln2", x), 128))
        x = m.binary_op(f"{b}_add2", [skip, m.linear(f"{b}_fc2", x, dim)], 0)
    x = m.crop("cls", m.layer_norm("ln", x), hoff=0, outh=1)
    m.fc("logits", x, classes)
    return m

ZOO = {"single_conv": single_conv, "vgg16": vgg16, "resnet50": resnet50, "mobilenet_v1": mobilenet_v1, "mini": mini,
       "decoder_tiny": decoder_tiny, "fcn8s_tiny": fcn8s_tiny, "deeplab_head_tiny": deeplab_head_tiny,
       "mobilenet_v2": mobilenet_v2, "prelu_tiny": prelu_tiny, "mobilenet_ssd": mobilenet_ssd, "ssd_tiny": ssd_tiny,
       "vgg_ssd": vgg_ssd, "googlenet": googlenet, "alexnet": alexnet,
       "mobilenet_yolov2": mobilenet_yolov2, "mobilenetv2_yolov3": mobilenetv2_yolov3, "yolo_tiny": yolo_tiny,
       "shufflenet_v2": shufflenet_v2, "shuffle_tiny": shuffle_tiny, "deeplabv3_mobilenet_v2": deeplabv3_mobilenet_v2,
       "deeplabv3_tiny": deeplabv3_tiny, "faster_rcnn_vgg16": faster_rcnn_vgg16, "faster_rcnn_tiny": faster_rcnn_tiny,
       "rfcn_resnet50": rfcn_resnet50, "rfcn_tiny": rfcn_tiny, "fast_neural_style": fast_neural_style,
       "style_tiny": style_tiny, "srvgg_compact": srvgg_compact, "edsr_baseline": edsr_baseline, "sr_tiny": sr_tiny,
       "mobilenet_v3_large": mobilenet_v3_large, "mobilenet_v3_small": mobilenet_v3_small,
       "efficientnet_b0": efficientnet_b0, "espcn": espcn, "se_tiny": se_tiny, "vit_b_16": vit_b_16,
       "vit_s_16": vit_s_16, "vit_ti_16": vit_ti_16, "vit_tiny": vit_tiny}


def synthetic_input(shape, index: int = 0) -> np.ndarray:
    """uniform(-0.5, 0.5), seed 1234 + image index (SURVEY.md §8d)."""
    return np.random.default_rng(1234 + index).uniform(-0.5, 0.5, shape).astype(np.float32)


if __name__ == "__main__":
    import argparse

    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("model", choices=sorted(ZOO))
    ap.add_argument("prefix")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    mw = ZOO[a.model](seed=a.seed)
    print(mw.save(a.prefix), f"{mw.flops / 1e9:.3f} GFLOP/image")
