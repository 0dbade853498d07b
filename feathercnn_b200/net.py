"""Python face of ``feather::Net`` (include/feather/net.h) — same method names as the C++ class, which keeps the
reference's API (/root/reference/src/net.h:30-70 and README.md:56-75).  All compute happens inside
libfeather_b200.so / libfcuda.so; numpy / torch objects are only buffers."""
from __future__ import annotations

import ctypes

import numpy as np

from ._lib import feather


class FeatherError(RuntimeError):
    def __init__(self, fn: str, code: int):
        super().__init__(f"{fn} returned {code}")
        self.code = code


def _check(fn: str, rc: int) -> None:
    if rc != 0:
        raise FeatherError(fn, rc)


class Net:
    def __init__(self, num_threads: int = 1, fusion: bool = False, cuda_graph: bool = False):
        self._lib = feather()
        self._h = ctypes.c_void_p(self._lib.fnet_create())
        if fusion:
            self._lib.fnet_set_fusion(self._h, 1)
        if cuda_graph:
            self._lib.fnet_set_cuda_graph(self._h, 1)

    def __del__(self):
        try:
            if self._h:
                self._lib.fnet_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- loading ---------------------------------------------------------------------------------
    def LoadParam(self, path) -> None:
        _check("LoadParam", self._lib.fnet_load_param(self._h, str(path).encode()))

    def LoadParamFromText(self, text: str | bytes) -> None:
        if isinstance(text, str):
            text = text.encode()
        _check("LoadParamFromText", self._lib.fnet_load_param_text(self._h, text))

    def LoadWeights(self, path) -> None:
        _check("LoadWeights", self._lib.fnet_load_weights(self._h, str(path).encode()))

    def InitFromPath(self, path) -> None:
        _check("InitFromPath", self._lib.fnet_init_from_path(self._h, str(path).encode()))

    def InitFromBuffer(self, buf: bytes) -> None:
        _check("InitFromBuffer", self._lib.fnet_init_from_buffer(self._h, buf, len(buf)))

    def PrepareWeightArena(self) -> None:
        _check("PrepareWeightArena", self._lib.fnet_prepare_weight_arena(self._h))

    def WeightArena(self) -> tuple[int, int]:
        p, n = ctypes.c_void_p(), ctypes.c_size_t()
        self._lib.fnet_weight_arena(self._h, ctypes.byref(p), ctypes.byref(n))
        return (p.value or 0), n.value

    def AttachWeights(self) -> None:
        _check("AttachWeights", self._lib.fnet_attach_weights(self._h))

    def SetStream(self, cuda_stream: int) -> None:
        self._lib.fnet_set_stream(self._h, ctypes.c_void_p(cuda_stream))

    # ---- inference -------------------------------------------------------------------------------
    @property
    def input_name(self) -> str:
        return self._lib.fnet_input_name(self._h).decode()

    @property
    def input_shape(self) -> tuple[int, int, int]:
        c, h, w = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        self._lib.fnet_input_shape(self._h, ctypes.byref(c), ctypes.byref(h), ctypes.byref(w))
        return c.value, h.value, w.value

    def FeedInputBatch(self, x: np.ndarray, name: str | None = None) -> None:
        x = np.ascontiguousarray(x, np.float32)
        if x.ndim == 3:
            x = x[None]
        n, c, h, w = x.shape
        _check("FeedInputBatch", self._lib.fnet_feed_input_batch(self._h, (name or self.input_name).encode(),
                                                                 x.ctypes.data_as(ctypes.c_void_p), n, c, h, w))
        self._keepalive = x

    def FeedInputPixels(self, pixels: np.ndarray, type_: int, target_w: int = 0, target_h: int = 0, mean=None, norm=None,
                        name: str | None = None) -> None:
        """(N, h, w[, c]) uint8 interleaved images -> resize -> planar fp32 -> (x - mean) * norm, on the device
        (ncnn::Mat::from_pixels_resize + substract_mean_normalize + FeedInput, /root/reference/src/ncnn/mat.h:149-160)."""
        pixels = np.ascontiguousarray(pixels, np.uint8)
        n, h, w = pixels.shape[:3]
        fp = ctypes.POINTER(ctypes.c_float)
        m = None if mean is None else np.ascontiguousarray(mean, np.float32)
        s = None if norm is None else np.ascontiguousarray(norm, np.float32)
        _check("FeedInputPixels", self._lib.fnet_feed_input_pixels(
            self._h, (name or self.input_name).encode(), pixels.ctypes.data_as(ctypes.c_void_p), type_, w, h, target_w,
            target_h, n, None if m is None else m.ctypes.data_as(fp), None if s is None else s.ctypes.data_as(fp)))
        self.Synchronize()  # the pageable host array may be released by the caller

    def FeedInputDevice(self, data_ptr: int, shape, name: str | None = None) -> None:
        n, c, h, w = shape
        _check("FeedInputDevice", self._lib.fnet_feed_input_device(self._h, (name or self.input_name).encode(),
                                                                   ctypes.c_void_p(data_ptr), n, c, h, w))

    def Forward(self, x: np.ndarray | None = None) -> None:
        if x is not None:
            self.FeedInputBatch(x)
        _check("Forward", self._lib.fnet_forward(self._h))

    def ForwardBatchHostPtr(self, host_ptr: int, batch: int) -> None:
        """README-style ``Forward(float*)`` over a (pinned) host buffer holding `batch` images."""
        _check("ForwardBatch", self._lib.fnet_forward_batch(self._h, ctypes.c_void_p(host_ptr), batch))

    def SubmitBatch(self, host_ptr: int, batch: int, blob: str | None = None, host_out_ptr: int = 0) -> int:
        """Pipelined end-to-end step (two in flight): H2D on a copy stream, Forward, D2H of `blob` into `host_out_ptr`.
        Returns a ticket for WaitBatch.  Host buffers should be pinned and stay valid until the wait."""
        t = self._lib.fnet_submit_batch(self._h, ctypes.c_void_p(host_ptr), batch, blob.encode() if blob else None,
                                        ctypes.c_void_p(host_out_ptr))
        if t < 0:
            raise FeatherError("SubmitBatch", t)
        return t

    def WaitBatch(self, ticket: int) -> None:
        _check("WaitBatch", self._lib.fnet_wait_batch(self._h, ticket))

    def Synchronize(self) -> None:
        _check("Synchronize", self._lib.fnet_synchronize(self._h))

    def BlobShape(self, name: str) -> tuple[int, int, int, int]:
        n, c, h, w = (ctypes.c_int() for _ in range(4))
        _check("BlobShape", self._lib.fnet_blob_shape(self._h, name.encode(), ctypes.byref(n), ctypes.byref(c),
                                                      ctypes.byref(h), ctypes.byref(w)))
        return n.value, c.value, h.value, w.value

    def BlobDims(self, name: str) -> int:
        """ncnn rank of one image of the blob: 1 = Mat(w), 2 = Mat(w, h), 3 = Mat(w, h, c).  BlobShape is (n, c, h, w)
        whatever the rank (a rank-1 blob is (n, 1, 1, w), a rank-2 one (n, 1, h, w))."""
        d = int(self._lib.fnet_blob_dims(self._h, name.encode()))
        if d < 0:
            raise FeatherError("BlobDims", d)
        return d

    def Extract(self, name: str) -> np.ndarray:
        shape = self.BlobShape(name)
        out = np.empty(shape, np.float32)
        _check("ExtractBlob", self._lib.fnet_extract_blob(self._h, name.encode(), out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def ExtractInto(self, name: str, host_ptr: int) -> None:
        _check("ExtractBlob", self._lib.fnet_extract_blob(self._h, name.encode(), ctypes.c_void_p(host_ptr)))

    def ExtractDevice(self, name: str) -> tuple[int, tuple[int, int, int, int]]:
        p = ctypes.c_void_p()
        n, c, h, w = (ctypes.c_int() for _ in range(4))
        _check("ExtractDevice", self._lib.fnet_extract_device(self._h, name.encode(), ctypes.byref(p), ctypes.byref(n),
                                                              ctypes.byref(c), ctypes.byref(h), ctypes.byref(w)))
        return p.value, (n.value, c.value, h.value, w.value)

    def FuseNow(self) -> int:
        """Run the SetFusion graph rewrite now (host only); returns the number of layers absorbed."""
        return int(self._lib.fnet_fuse_now(self._h))

    def LayerFusedAway(self, layer_name: str) -> int:
        return int(self._lib.fnet_layer_fused_away(self._h, layer_name.encode()))

    def LayerConvAlgo(self, layer_name: str) -> int:
        """The FcudaConvAlgo a convolution layer runs (valid after a Forward); -1 for an unknown layer, a layer that is
        not a convolution, or one fused away."""
        return int(self._lib.fnet_layer_conv_algo(self._h, layer_name.encode()))

    def BlobNames(self) -> list[str]:
        need = self._lib.fnet_blob_names(self._h, None, 0)
        buf = ctypes.create_string_buffer(need)
        self._lib.fnet_blob_names(self._h, buf, need)
        return [s for s in buf.value.decode().split("\n") if s]

    @property
    def launches_per_forward(self) -> int:
        return int(self._lib.fnet_launches_per_forward(self._h))


class NetGroup:
    """``feather::NetGroup`` (include/feather/net_group.h): one model on several GPUs of one box from ONE process — the file
    is read once, the weight arena reaches the other devices by one ncclBroadcast, every batch is sharded contiguously
    over the devices, no collective in Forward."""

    def __init__(self, fusion: bool = True, cuda_graph: bool = True):
        self._lib = feather()
        self._h = ctypes.c_void_p(self._lib.fgroup_create())
        self._lib.fgroup_set_options(self._h, int(fusion), int(cuda_graph))

    def __del__(self):
        try:
            if self._h:
                self._lib.fgroup_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def InitFromPath(self, path, devices: list[int] | None = None) -> None:
        if devices:
            arr = (ctypes.c_int * len(devices))(*devices)
            rc = self._lib.fgroup_init_from_path(self._h, str(path).encode(), arr, len(devices))
        else:
            rc = self._lib.fgroup_init_from_path(self._h, str(path).encode(), None, 0)
        _check("NetGroup.InitFromPath", rc)

    def Size(self) -> int:
        return int(self._lib.fgroup_size(self._h))

    def Device(self, member: int) -> int:
        return int(self._lib.fgroup_device(self._h, member))

    def BroadcastTransport(self) -> str:
        return self._lib.fgroup_broadcast_transport(self._h).decode()

    def Member(self, member: int) -> Net:
        """A non-owning view of a member Net (Extract / BlobShape / ... on that device)."""
        h = self._lib.fgroup_member(self._h, member)
        if not h:
            raise FeatherError("NetGroup.Member", -1)
        return _BorrowedNet(self._lib, ctypes.c_void_p(h), self)

    def ForwardBatch(self, x: np.ndarray, blob: str, out_shape_per_image: tuple[int, ...]) -> np.ndarray:
        """Shards the host batch `x` (N, C, H, W) over the members; returns `blob` of every image, in input order."""
        x = np.ascontiguousarray(x, np.float32)
        out = np.empty((x.shape[0],) + tuple(out_shape_per_image), np.float32)
        _check("NetGroup.ForwardBatch", self._lib.fgroup_forward_batch(
            self._h, x.ctypes.data_as(ctypes.c_void_p), x.shape[0], blob.encode(), out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def ForwardBatchPtr(self, host_ptr: int, batch: int, blob: str | None, host_out_ptr: int = 0) -> None:
        _check("NetGroup.ForwardBatch", self._lib.fgroup_forward_batch(
            self._h, ctypes.c_void_p(host_ptr), batch, blob.encode() if blob else None, ctypes.c_void_p(host_out_ptr)))

    def ShardRange(self, batch: int, member: int) -> tuple[int, int]:
        lo, hi = ctypes.c_int(), ctypes.c_int()
        _check("NetGroup.ShardRange", self._lib.fgroup_shard_range(batch, self.Size(), member, ctypes.byref(lo), ctypes.byref(hi)))
        return lo.value, hi.value

    def Synchronize(self) -> None:
        _check("NetGroup.Synchronize", self._lib.fgroup_synchronize(self._h))


class _BorrowedNet(Net):
    """Net methods on a handle owned by a NetGroup."""

    def __init__(self, lib, handle, owner):
        self._lib = lib
        self._h = handle
        self._owner = owner

    def __del__(self):
        self._h = None
