"""Caffe -> ncnn ``.param/.bin`` (and ``.feathermodel``) converter.

SURVEY.md §8f rank 2: the reference's own converter lives in ``tools/`` (``/root/reference/CMakeLists.txt:84-89``,
``add_subdirectory(tools)``) and is absent from the snapshot, so real Caffe models could not be brought to the loader
(``/root/reference/src/net.cpp:68-230``).  This tool reads a binary ``.caffemodel`` (a serialized ``caffe.NetParameter``;
models saved by Caffe carry the full layer definitions next to the weights) with a minimal protobuf wire-format reader —
no caffe / protobuf-generated code is needed — and writes the ncnn text ``.param`` + ``.bin`` the loader expects:

* layer grammar and parameter ids as ``ConvLayer::LoadParam`` & co. read them (``src/layers/*.h``; ids follow ncnn's
  caffe2ncnn): Convolution / ConvolutionDepthWise, Deconvolution / DeconvolutionDepthWise, InnerProduct, Pooling, ReLU, BatchNorm, Scale, Eltwise, Concat, Dropout,
  Softmax, Split, Input, Crop, Clip, PReLU, Slice, LRN, Sigmoid, TanH;
* LRN (``lrn_param``: ``local_size``, ``alpha``, ``beta``, ``norm_region``, ``k``) becomes ncnn's LRN
  ``0=region 1=local_size 2=alpha 3=beta 4=bias``.  Caffe's WITHIN_CHANNEL LRN divides by a fixed ``1 + alpha / n * ss``
  and ignores ``k``, so that region is written with ``4=1``; an even ``local_size`` (which Caffe rejects) is an error;
* Slice (``slice_param``: ``axis`` or the older ``slice_dim``, ``slice_point``) becomes ncnn's Slice: the cut points become
  sizes with ``-233`` (the rest) for the last top, and no cut points an even split (``-233`` for every top).  Caffe has no
  ShuffleChannel in its upstream ``caffe.proto``, so that type keeps the "no counterpart" error;
* Sigmoid and TanH keep their names; ``sigmoid_param`` / ``tanh_param`` only choose Caffe's compute engine;
* ReLU6 (the type MobileNet-v2 Caffe ports use) becomes ``Clip 0=0 1=6``, Caffe's Clip (``clip_param.min / max``) Clip with its
  bounds, PReLU ``PReLU 0=num_slope`` with its slopes (one, ``channel_shared``, or one per channel) raw in the ``.bin``;
* Crop (``axis`` 2 or 3, FCN's score crops) becomes ncnn's two-bottom Crop: the output height and width are the reference
  bottom's, the offsets are ``offset``'s; with axis 3 the height offset is 0, and the reference must then have the height
  of the cropped blob, as ncnn's two-bottom Crop takes both sizes from it;
* in-place Caffe layers (top == bottom) get a fresh blob name, and a blob read by several layers gets an explicit
  ``Split`` layer — the reference's Net looks blobs up by name and its layers own their tops (``net.cpp:112-160``);
* weight blobs are written with the 4-byte raw-fp32 tag, bias / BatchNorm / Scale blobs raw (``modelbin.cpp:47-197``);
* BatchNorm: Caffe stores (mean, variance, scale_factor); the file gets slope = 1, mean / sf, var / sf, bias = 0
  (``batchnorm_layer.h:52-75``).

Field numbers are those of BVLC ``caffe.proto`` (NetParameter.layer = 100, LayerParameter.convolution_param = 106, ...).
V1 (``layers = 2``) models are not supported.

    python -m feathercnn_b200.tools.caffe2feather net.caffemodel out_prefix [--feathermodel]
"""
from __future__ import annotations

import struct
from pathlib import Path

import numpy as np


# --------------------------------------------------------------------------------------------------
# protobuf wire format
# --------------------------------------------------------------------------------------------------
def _varint(buf: bytes, i: int) -> tuple[int, int]:
    v = shift = 0
    while True:
        b = buf[i]
        i += 1
        v |= (b & 0x7F) << shift
        if not b & 0x80:
            return v, i
        shift += 7


def parse_message(buf: bytes) -> dict[int, list]:
    """field number -> list of raw values (int for varint / fixed, bytes for length-delimited)."""
    out: dict[int, list] = {}
    i, n = 0, len(buf)
    while i < n:
        key, i = _varint(buf, i)
        field, wt = key >> 3, key & 7
        if wt == 0:
            v, i = _varint(buf, i)
        elif wt == 1:
            v = buf[i:i + 8]; i += 8
        elif wt == 2:
            ln, i = _varint(buf, i)
            v = buf[i:i + ln]; i += ln
        elif wt == 5:
            v = buf[i:i + 4]; i += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt} (field {field})")
        out.setdefault(field, []).append(v)
    return out


def _ints(vals: list) -> list[int]:
    """repeated (possibly packed) varint field."""
    out = []
    for v in vals:
        if isinstance(v, (bytes, bytearray)):
            i = 0
            while i < len(v):
                x, i = _varint(v, i)
                out.append(x)
        else:
            out.append(v)
    return out


def _floats(vals: list) -> np.ndarray:
    """repeated (possibly packed) float field."""
    parts = [np.frombuffer(v, "<f4") for v in vals if isinstance(v, (bytes, bytearray))]
    return np.concatenate(parts) if parts else np.zeros(0, np.float32)


def _first(msg: dict, field: int, default=None):
    return msg[field][0] if field in msg else default


def _f32(raw, default: float) -> float:
    return struct.unpack("<f", raw)[0] if raw is not None else default


def _str(raw) -> str:
    return raw.decode() if raw is not None else ""


def _blob(raw: bytes) -> np.ndarray:
    """caffe.BlobProto -> flat float32 (data = 5, double_data = 8)."""
    m = parse_message(raw)
    if 5 in m:
        return _floats(m[5]).astype(np.float32)
    if 8 in m:
        return np.concatenate([np.frombuffer(v, "<f8") for v in m[8]]).astype(np.float32)
    return np.zeros(0, np.float32)


# --------------------------------------------------------------------------------------------------
# conversion
# --------------------------------------------------------------------------------------------------
class _Out:
    def __init__(self):
        self.lines: list[str] = []
        self.bin = bytearray()
        self.blobs: list[str] = []

    def layer(self, type_: str, name: str, bottoms: list[str], tops: list[str], params: str = ""):
        self.lines.append(f"{type_} {name} {len(bottoms)} {len(tops)} {' '.join(bottoms + tops)} {params}".rstrip())
        self.blobs += tops

    def weights(self, a: np.ndarray, flagged: bool):
        if flagged:
            self.bin += struct.pack("<I", 0)
        self.bin += np.ascontiguousarray(a, "<f4").tobytes()


def _hw(msg: dict, rep: int, fh: int, fw: int, default: int) -> tuple[int, int]:
    """Caffe's (repeated field | _h / _w pair) convention -> (h, w)."""
    if fh in msg or fw in msg:
        return int(_first(msg, fh, default)), int(_first(msg, fw, default))
    r = _ints(msg.get(rep, []))
    if not r:
        return default, default
    return (r[0], r[0]) if len(r) == 1 else (r[0], r[1])


def convert(caffemodel: bytes) -> tuple[str, bytes]:
    """Serialized caffe.NetParameter -> (ncnn .param text, .bin bytes)."""
    net = parse_message(caffemodel)
    if 2 in net and 100 not in net:
        raise ValueError("V1 caffemodel (NetParameter.layers): upgrade it with caffe's upgrade_net_proto_binary first")
    layers = [parse_message(raw) for raw in net.get(100, [])]
    # keep test-phase layers only (LayerParameter.include = 8 -> NetStateRule.phase = 1; TRAIN = 0, TEST = 1)
    kept = []
    for L in layers:
        phases = [parse_message(r) for r in L.get(8, [])]
        if phases and all(_first(p, 1, 1) == 0 for p in phases):
            continue
        kept.append(L)
    layers = kept

    out = _Out()
    # ---- inputs: NetParameter.input (3) + input_dim (4) / input_shape (8), or Input layers ----------------------
    net_inputs = [_str(v) for v in net.get(3, [])]
    if net_inputs:
        dims = _ints(net.get(4, []))
        if not dims and 8 in net:
            dims = _ints(parse_message(net[8][0]).get(1, []))
        for k, nm in enumerate(net_inputs):
            d = dims[4 * k:4 * k + 4] if len(dims) >= 4 * (k + 1) else [1, 3, 224, 224]
            out.layer("Input", nm, [], [nm], f"0={d[3]} 1={d[2]} 2={d[1]}")

    # ---- blob renaming: in-place tops and multi-reader splits ---------------------------------------------------
    current: dict[str, str] = {n: n for n in net_inputs}   # caffe blob name -> name of the blob that currently holds it
    readers: dict[str, int] = {}
    # first pass: resolve the producer-side names so that reader counts refer to final blob names
    resolved = []
    cur = dict(current)
    for L in layers:
        name, type_ = _str(_first(L, 1)), _str(_first(L, 2))
        bottoms = [cur.get(_str(b), _str(b)) for b in L.get(3, [])]
        tops = []
        for t in (_str(t) for t in L.get(4, [])):
            new = t if t not in cur else f"{t}_{name}"  # in-place (or re-defined) blob: fresh name, like caffe2ncnn
            cur[t] = new
            tops.append(new)
        for b in bottoms:
            readers[b] = readers.get(b, 0) + 1
        resolved.append((L, name, type_, bottoms, tops))
    split_next: dict[str, int] = {}

    def take(blob: str) -> str:
        """Name a reader uses for `blob`: the blob itself, or the next output of its Split layer."""
        if readers.get(blob, 0) <= 1:
            return blob
        k = split_next.get(blob, 0)
        split_next[blob] = k + 1
        return f"{blob}_splitncnn_{k}"

    def emit_split(blob: str):
        n = readers.get(blob, 0)
        if n > 1:
            out.layer("Split", f"splitncnn_{blob}", [blob], [f"{blob}_splitncnn_{k}" for k in range(n)])

    for nm in net_inputs:
        emit_split(nm)

    for L, name, type_, bottoms, tops in resolved:
        blobs = [_blob(r) for r in L.get(7, [])]
        bottoms = [take(b) for b in bottoms]
        if type_ == "Input":
            shape = _ints(parse_message(parse_message(_first(L, 143, b"")).get(1, [b""])[0]).get(1, [])) or [1, 3, 224, 224]
            out.layer("Input", name, [], tops, f"0={shape[3]} 1={shape[2]} 2={shape[1]}")
        elif type_ == "Convolution" or type_ == "DepthwiseConvolution":
            p = parse_message(_first(L, 106, b""))
            num_output = int(_first(p, 1, 0))
            bias = int(_first(p, 2, 1))
            kh, kw = _hw(p, 4, 11, 12, 1)
            sh, sw = _hw(p, 6, 13, 14, 1)
            ph, pw = _hw(p, 3, 9, 10, 0)
            dil = _ints(p.get(18, [])) or [1]
            group = int(_first(p, 5, 1))
            w = blobs[0]
            ltype = "ConvolutionDepthWise" if group > 1 else "Convolution"
            ps = f"0={num_output} 1={kw} 11={kh} 2={dil[0]} 3={sw} 13={sh} 4={pw} 14={ph} 5={bias} 6={w.size}"
            if group > 1:
                ps += f" 7={group}"
            out.layer(ltype, name, bottoms, tops, ps)
            out.weights(w, True)
            if bias:
                out.weights(blobs[1], False)
        elif type_ == "Deconvolution":
            # same convolution_param; Caffe's blob is (IC, OC/group, kh, kw), ncnn's [group][OC/group][IC/group][kh][kw]
            p = parse_message(_first(L, 106, b""))
            num_output = int(_first(p, 1, 0))
            bias = int(_first(p, 2, 1))
            kh, kw = _hw(p, 4, 11, 12, 1)
            sh, sw = _hw(p, 6, 13, 14, 1)
            ph, pw = _hw(p, 3, 9, 10, 0)
            dil = _ints(p.get(18, [])) or [1]
            group = int(_first(p, 5, 1))
            ocg = num_output // group
            w = blobs[0].reshape(group, -1, ocg, kh, kw).transpose(0, 2, 1, 3, 4)
            ltype = "DeconvolutionDepthWise" if group > 1 else "Deconvolution"
            ps = f"0={num_output} 1={kw} 11={kh} 2={dil[-1]} 12={dil[0]} 3={sw} 13={sh} 4={pw} 14={ph} 5={bias} 6={w.size}"
            if group > 1:
                ps += f" 7={group}"
            out.layer(ltype, name, bottoms, tops, ps)
            out.weights(w, True)
            if bias:
                out.weights(blobs[1], False)
        elif type_ == "InnerProduct":
            p = parse_message(_first(L, 117, b""))
            num_output, bias = int(_first(p, 1, 0)), int(_first(p, 2, 1))
            out.layer("InnerProduct", name, bottoms, tops, f"0={num_output} 1={bias} 2={blobs[0].size}")
            out.weights(blobs[0], True)
            if bias:
                out.weights(blobs[1], False)
        elif type_ == "Pooling":
            p = parse_message(_first(L, 121, b""))
            pool = int(_first(p, 1, 0))
            kh, kw = _hw(p, 2, 5, 6, 1) if (2 in p or 5 in p) else (1, 1)
            sh, sw = _hw(p, 3, 7, 8, 1)
            ph, pw = _hw(p, 4, 9, 10, 0)
            glob = int(_first(p, 12, 0))
            out.layer("Pooling", name, bottoms, tops, f"0={pool} 1={kw} 11={kh} 2={sw} 12={sh} 3={pw} 13={ph} 4={glob}")
        elif type_ == "ReLU":
            slope = _f32(_first(parse_message(_first(L, 123, b"")), 1), 0.0)
            out.layer("ReLU", name, bottoms, tops, f"0={slope:e}" if slope else "")
        elif type_ in ("Sigmoid", "TanH"):
            out.layer(type_, name, bottoms, tops, "")
        elif type_ == "ReLU6":
            out.layer("Clip", name, bottoms, tops, f"0={0.0:e} 1={6.0:e}")
        elif type_ == "Clip":
            p = parse_message(_first(L, 148, b""))  # clip_param = 148: min = 1, max = 2 (both required)
            if 1 not in p or 2 not in p:
                raise ValueError(f"layer {name}: Clip without clip_param.min / max")
            out.layer("Clip", name, bottoms, tops, f"0={_f32(_first(p, 1), 0.0):.8e} 1={_f32(_first(p, 2), 0.0):.8e}")
        elif type_ == "PReLU":
            # prelu_param = 131 (filler, channel_shared) only shapes the blob: (1,) when shared, (channels,) otherwise
            slope = blobs[0].reshape(-1)
            out.layer("PReLU", name, bottoms, tops, f"0={slope.size}")
            out.weights(slope, False)
        elif type_ == "BatchNorm":
            p = parse_message(_first(L, 139, b""))
            eps = _f32(_first(p, 3), 1e-5)
            c = blobs[0].size
            sf = float(blobs[2][0]) if len(blobs) > 2 and blobs[2].size and blobs[2][0] != 0 else 1.0
            out.layer("BatchNorm", name, bottoms, tops, f"0={c} 1={eps:e}")
            out.weights(np.ones(c, np.float32), False)        # slope
            out.weights(blobs[0] / np.float32(sf), False)     # mean
            out.weights(blobs[1] / np.float32(sf), False)     # var
            out.weights(np.zeros(c, np.float32), False)       # bias
        elif type_ == "Scale":
            p = parse_message(_first(L, 142, b""))
            bias = int(_first(p, 4, 0))
            out.layer("Scale", name, bottoms, tops, f"0={blobs[0].size} 1={bias}")
            out.weights(blobs[0], False)
            if bias:
                out.weights(blobs[1], False)
        elif type_ == "Eltwise":
            p = parse_message(_first(L, 110, b""))
            op = int(_first(p, 1, 1))
            coeff = _floats(p.get(2, []))
            if not coeff.size and 2 in p:  # non-packed repeated float
                coeff = np.array([struct.unpack("<f", v)[0] for v in p[2]], np.float32)
            ps = f"0={op}"
            if coeff.size:
                ps += f" -23301={coeff.size}," + ",".join(f"{c:e}" for c in coeff)
            out.layer("Eltwise", name, bottoms, tops, ps)
        elif type_ == "Concat":
            p = parse_message(_first(L, 104, b""))
            axis = int(_first(p, 2, _first(p, 1, 1)))
            out.layer("Concat", name, bottoms, tops, f"0={axis - 1}")
        elif type_ == "Slice":
            # slice_param = 126: axis = 3 (default 1), slice_point = 2 (repeated), slice_dim = 1 (deprecated axis)
            p = parse_message(_first(L, 126, b""))
            axis = int(_first(p, 3, _first(p, 1, 1)))
            if axis >= 1 << 63:  # a negative int32 on the wire
                axis -= 1 << 64
            axis = axis + 4 if axis < 0 else axis
            points = _ints(p.get(2, []))
            if axis not in (1, 2, 3):
                raise ValueError(f"layer {name}: Slice along axis {axis} (the batch) has no FeatherCNN counterpart")
            if points and (len(points) != len(tops) - 1 or any(b <= a for a, b in zip([0] + points, points))):
                raise ValueError(f"layer {name}: Slice needs {len(tops) - 1} increasing positive slice points, "
                                 f"not {points}")
            # cut points become sizes, the last top takes the rest; none: an even split (every entry -233)
            sizes = [b - a for a, b in zip([0] + points, points)] + [-233] if points else [-233] * len(tops)
            ps = f"-23300={len(sizes)}," + ",".join(str(s) for s in sizes)
            out.layer("Slice", name, bottoms, tops, ps + (f" 1={axis - 1}" if axis != 1 else ""))
        elif type_ == "LRN":
            # lrn_param = 118: local_size = 1 (5), alpha = 2 (1), beta = 3 (0.75), norm_region = 4 (ACROSS_CHANNELS), k = 5 (1)
            p = parse_message(_first(L, 118, b""))
            size = int(_first(p, 1, 5))
            region = int(_first(p, 4, 0))
            if size % 2 == 0:
                raise ValueError(f"layer {name}: LRN local_size {size} is even (Caffe accepts odd sizes only)")
            if region not in (0, 1):
                raise ValueError(f"layer {name}: LRN norm_region {region} has no FeatherCNN counterpart")
            bias = 1.0 if region == 1 else _f32(_first(p, 5), 1.0)  # Caffe's WITHIN_CHANNEL shifts by 1, not k
            out.layer("LRN", name, bottoms, tops, f"0={region} 1={size} 2={_f32(_first(p, 2), 1.0):.8e} "
                                                  f"3={_f32(_first(p, 3), 0.75):.8e} 4={bias:.8e}")
        elif type_ == "Dropout":
            out.layer("Dropout", name, bottoms, tops)   # identity at test time (dropout_layer.h:40-43)
        elif type_ == "Softmax":
            out.layer("Softmax", name, bottoms, tops)
        elif type_ == "Split":
            out.layer("Split", name, bottoms, tops)
        elif type_ == "Crop":
            # crop_param = 144: axis = 1 (default 2), offset = 2 (repeated; one value applies to every cropped axis)
            p = parse_message(_first(L, 144, b""))
            axis = int(_first(p, 1, 2))
            if axis >= 1 << 63:  # a negative int32 on the wire
                axis -= 1 << 64
            axis = axis + 4 if axis < 0 else axis
            if axis not in (2, 3) or len(bottoms) != 2:
                raise ValueError(f"layer {name}: Crop with axis {axis} (channels or batch) or without a reference bottom "
                                 f"has no FeatherCNN counterpart")
            offs = _ints(p.get(2, [])) or [0]
            n_axes = 4 - axis
            if len(offs) not in (1, n_axes):
                raise ValueError(f"layer {name}: Crop has {len(offs)} offsets for {n_axes} cropped axes")
            offs = offs * n_axes if len(offs) == 1 else offs
            hoff, woff = (offs[0], offs[1]) if axis == 2 else (0, offs[0])
            out.layer("Crop", name, bottoms, tops, f"0={woff} 1={hoff}")
        else:
            raise ValueError(f"layer {name}: Caffe type {type_!r} has no FeatherCNN counterpart (layer_factory.cpp:55-67)")
        for t in tops:
            emit_split(t)

    text = "7767517\n" + f"{len(out.lines)} {len(out.blobs)}\n" + "\n".join(out.lines) + "\n"
    return text, bytes(out.bin)


def convert_file(caffemodel_path, prefix, feathermodel: bool = False) -> tuple[str, str]:
    text, blob = convert(Path(caffemodel_path).read_bytes())
    prefix = str(prefix)
    Path(prefix + ".param").write_text(text)
    Path(prefix + ".bin").write_bytes(blob)
    if feathermodel:
        from . import feathermodel as fm
        fm.pack(prefix + ".param", prefix + ".bin", prefix + ".feathermodel")
    return prefix + ".param", prefix + ".bin"


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser(description="Caffe .caffemodel -> ncnn .param/.bin for feather::Net")
    ap.add_argument("caffemodel")
    ap.add_argument("prefix")
    ap.add_argument("--feathermodel", action="store_true", help="also write the single-file FTHRB200 container")
    a = ap.parse_args()
    print(convert_file(a.caffemodel, a.prefix, a.feathermodel))
