"""ctypes binding of libtengine_b200.so (the C ABI in include/tengine_b200.h) for tests and bench.py."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
# TB200_LIB: debug builds of the same library (tools/build_trace_lib.sh); never a different implementation
LIB_PATH = os.environ.get("TB200_LIB") or os.path.join(_HERE, "libtengine_b200.so")
_lib = None


class TB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"tb200 error {code}: {msg}")
        self.code = code


def build(verbose=False):
    """Compile tengine_b200/csrc for sm_90a (nvcc cross-compiles without a GPU)."""
    r = subprocess.run(["make", "-C", os.path.join(_HERE, "csrc")], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building libtengine_b200.so failed:\n" + r.stdout[-3000:] + r.stderr[-3000:])
    if verbose:
        print(r.stdout[-1500:])


def lib():
    """Load the library; fails loudly when it has not been built (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(the H100 backend has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.tb200_last_error.restype = C.c_char_p
        L.tb200_graph_layer_kernel.restype = C.c_char_p
        L.tb200_context_stream.restype = C.c_void_p
        L.tb200_host_alloc.restype = C.c_void_p
        L.tb200_host_alloc.argtypes = [C.c_size_t]
        L.tb200_host_free.argtypes = [C.c_void_p]
        L.tb200_graph_layer_kernel.argtypes = [C.c_void_p, C.c_int]
        for name in ("tb200_graph_run", "tb200_graph_upload", "tb200_graph_launch", "tb200_graph_download",
                     "tb200_graph_sync", "tb200_graph_postrun", "tb200_graph_weight_arena",
                     "tb200_graph_num_launches", "tb200_graph_read_tensor", "tb200_graph_profile",
                     "tb200_graph_work", "tb200_context_destroy", "tb200_graph_set_batch", "tb200_graph_batch"):
            getattr(L, name).restype = C.c_int
        L.tb200_graph_upload.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.tb200_graph_upload_images.restype = C.c_int
        L.tb200_graph_upload_images.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        L.tb200_graph_upload_detect_images.restype = C.c_int
        L.tb200_graph_upload_detect_images.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        L.tb200_detections_to_source.restype = C.c_int
        L.tb200_detections_to_source.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.tb200_graph_download.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.tb200_graph_launch.argtypes = [C.c_void_p]
        L.tb200_graph_sync.argtypes = [C.c_void_p]
        L.tb200_graph_postrun.argtypes = [C.c_void_p]
        L.tb200_graph_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.tb200_graph_read_tensor.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.tb200_graph_profile.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.tb200_graph_work.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.tb200_graph_weight_arena.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.tb200_graph_num_launches.argtypes = [C.c_void_p]
        L.tb200_context_destroy.argtypes = [C.c_void_p]
        L.tb200_context_stream.argtypes = [C.c_void_p]
        L.tb200_context_create_multi.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.tb200_context_num_gpus.argtypes = [C.c_void_p]
        L.tb200_context_gpu.argtypes = [C.c_void_p, C.c_int]
        L.tb200_context_stream_of.argtypes = [C.c_void_p, C.c_int]
        L.tb200_context_stream_of.restype = C.c_void_p
        L.tb200_context_broadcast_kind.argtypes = [C.c_void_p]
        L.tb200_context_broadcast_kind.restype = C.c_char_p
        L.tb200_graph_num_shards.argtypes = [C.c_void_p]
        L.tb200_graph_shard.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.tb200_graph_arena_bytes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.tb200_graph_broadcast_weights.argtypes = [C.c_void_p]
        L.tb200_pack_cache_dir.argtypes = [C.c_char_p]
        L.tb200_graph_pack_cache_state.argtypes = [C.c_void_p]
        L.tb200_graph_set_batch.argtypes = [C.c_void_p, C.c_int]
        L.tb200_graph_batch.argtypes = [C.c_void_p]
        L.tb200_graph_topk.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.tb200k_class_topk.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int32, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise TB200Error(rc, lib().tb200_last_error().decode(errors="replace"))


def set_pack_cache_dir(path):
    """Directory of the packed-weight cache (None disables); see include/tengine_b200.h tb200_pack_cache_dir."""
    lib().tb200_pack_cache_dir(path.encode() if path else None)


def shard_range(n_images, world, rank):
    """(first image, number of images) of shard `rank` of `world` for a batch of n_images: the library's own rule."""
    f, c = C.c_int(), C.c_int()
    _check(lib().tb200_shard_range(int(n_images), int(world), int(rank), C.byref(f), C.byref(c)))
    return f.value, c.value


def detections_to_source(geometry, boxes, letterbox=True):
    """Per image a list of (x, y, w, h, prob, label) in network-input pixels -> the same in source pixels of that image, mapped by
    tb200_detections_to_source with the geometry Graph.upload_detect_images returned (letterbox: its mode)."""
    n, m = len(boxes), max([1] + [len(b) for b in boxes])
    if len(geometry) != n:
        raise ValueError(f"{len(geometry)} geometries for {n} images")
    dets = (abi.Detection * (n * m))()
    counts = (C.c_int32 * n)(*[len(b) for b in boxes])
    for i, img in enumerate(boxes):
        for k, b in enumerate(img):
            d = dets[i * m + k]
            d.x, d.y, d.w, d.h, d.prob, d.label = b
    _check(lib().tb200_detections_to_source(abi.PRE_LETTERBOX if letterbox else abi.PRE_STRETCH, geometry, n, dets, m, counts))
    return [[(d.x, d.y, d.w, d.h, d.prob, d.label) for d in dets[i * m:i * m + counts[i]]] for i in range(n)]


def class_topk(in_ptr, n, c, h, w, is_uint8, scale, zero_point, k, out_ptr, stream=None):
    """tb200k_class_topk on DEVICE pointers: `in_ptr` an [n, h, w, cpad(c)] int8 / uint8 tensor, `out_ptr` room for n * k
    abi.ClassScore records; asynchronous on `stream`."""
    _check(lib().tb200k_class_topk(in_ptr, int(n), int(c), int(h), int(w), int(bool(is_uint8)), float(scale), int(zero_point), int(k), out_ptr, stream))


def device_count():
    return lib().tb200_device_count()


class Context:
    """interface->init / release_device: binds one GPU, or (devices=[...]) a group of GPUs driven by this process over
    which every graph shards its batch (tb200_context_create_multi)."""

    def __init__(self, device=0, devices=None):
        self.h = C.c_void_p()
        if devices is None:
            _check(lib().tb200_context_create(int(device), C.byref(self.h)))
            self.devices = [int(device)]
        else:
            arr = (C.c_int * len(devices))(*[int(d) for d in devices])
            _check(lib().tb200_context_create_multi(arr, len(devices), C.byref(self.h)))
            self.devices = [int(d) for d in devices]
        self.device = self.devices[0]

    @property
    def stream(self):
        return lib().tb200_context_stream(self.h)

    @property
    def num_gpus(self):
        return lib().tb200_context_num_gpus(self.h)

    def stream_of(self, index):
        return lib().tb200_context_stream_of(self.h, int(index))

    def probe_int8_tops(self):
        """Measured peak of the int8 tensor pipe of GPU 0 of this context in TOP/s (tb200_probe_int8_tops)."""
        t = C.c_double()
        lib().tb200_probe_int8_tops.argtypes = [C.c_void_p, C.c_void_p]
        _check(lib().tb200_probe_int8_tops(self.h, C.byref(t)))
        return t.value

    @property
    def broadcast_kind(self):
        return lib().tb200_context_broadcast_kind(self.h).decode()

    def close(self):
        if self.h:
            lib().tb200_context_destroy(self.h)
            self.h = C.c_void_p()


class PinnedBuffer:
    def __init__(self, shape, dtype):
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self.ptr = lib().tb200_host_alloc(self.nbytes)
        if not self.ptr:
            raise MemoryError("tb200_host_alloc failed")
        buf = (C.c_uint8 * self.nbytes).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dtype).reshape(shape)

    def free(self):
        if self.ptr:
            self.array = None
            lib().tb200_host_free(self.ptr)
            self.ptr = None


class Graph:
    """tb200_graph_prerun / run / postrun over a GraphDef (device->interface pre_run/run/post_run)."""

    def __init__(self, ctx, gdef, flags=abi.PRERUN_DEFAULT):
        self.ctx, self.gdef = ctx, gdef
        T, L = gdef.c_tables()
        self.h = C.c_void_p()
        _check(lib().tb200_graph_prerun(ctx.h, T, len(gdef.tensors), L, len(gdef.layers), gdef.id_array(gdef.inputs),
                                        len(gdef.inputs), gdef.id_array(gdef.outputs), len(gdef.outputs), int(flags),
                                        C.byref(self.h)))

    def set_batch(self, n):
        """Make images [0, n) the batch of every later call, 1 <= n <= the batch the graph was prepared for
        (tb200_graph_set_batch): host arrays then hold n images."""
        _check(lib().tb200_graph_set_batch(self.h, int(n)))

    @property
    def batch(self):
        """The active batch: the prepared one until set_batch changes it."""
        n = lib().tb200_graph_batch(self.h)
        if n < 0:
            _check(n)
        return n

    def dims(self, t):
        """Dims of tensor t at the active batch: the GraphDef's own at the prepared batch, else dim 0 is the active batch."""
        d = tuple(self.gdef.dims(t))
        n = self.batch
        return d if n == self.gdef.dims(0)[0] else (n,) + d[1:]  # prerun's batch is dim 0 of tensor 0

    def run(self, inputs, outputs=None):
        g = self.gdef
        ins = [np.ascontiguousarray(x) for x in inputs]
        for x, t in zip(ins, g.inputs):
            assert x.shape == self.dims(t) and x.dtype == g.np_dtype, (x.shape, self.dims(t), x.dtype)
        if outputs is None:
            outputs = [np.empty(self.dims(t), dtype=g.np_dtype) for t in g.outputs]
        assert len(ins) == len(g.inputs) and len(outputs) == len(g.outputs), "one host buffer per graph input / output"
        ip = (C.c_void_p * len(ins))(*[a.ctypes.data for a in ins])
        op = (C.c_void_p * len(outputs))(*[a.ctypes.data for a in outputs])
        _check(lib().tb200_graph_run(self.h, ip, op))
        return outputs

    def upload(self, i, x):
        _check(lib().tb200_graph_upload(self.h, i, x.ctypes.data))

    def _stage_pixels(self, i, images):
        """The images packed into a page-locked buffer kept on the graph (waiting first for the graph's queued work, which may still
        read it) and their descriptors."""
        imgs = [np.ascontiguousarray(a) for a in images]
        if len(imgs) != self.dims(self.gdef.inputs[i])[0]:
            raise ValueError(f"{len(imgs)} images for a batch of {self.dims(self.gdef.inputs[i])[0]}")
        descs = (abi.Image * len(imgs))()
        off = 0
        for d, a in zip(descs, imgs):
            if a.dtype != np.uint8 or a.ndim != 3:
                raise ValueError(f"images must be HxWxC uint8 arrays, not {a.dtype} {a.shape}")
            d.offset, d.h, d.w, d.c = off, a.shape[0], a.shape[1], a.shape[2]
            off += a.nbytes
        self.sync()
        buf = getattr(self, "_pixels", None)
        if buf is None or buf.nbytes < off:
            if buf is not None:
                buf.free()
            buf = self._pixels = PinnedBuffer((off,), np.uint8)
        for d, a in zip(descs, imgs):
            buf.array[d.offset:d.offset + a.nbytes] = a.reshape(-1)
        return buf, descs

    def upload_images(self, i, images, mean, scale):
        """Fill graph input i on the device from decoded images (tb200_graph_upload_images): one HxWxC uint8 array per image of the
        batch, C = 3 (RGB) or 4 (RGBA), sizes may differ; mean and scale index the B, G, R planes.  The pixels are packed into a
        page-locked buffer kept on the graph; since an earlier upload may still be reading it, packing first waits for the graph's
        queued work.  Asynchronous like upload: follow with launch and download."""
        buf, descs = self._stage_pixels(i, images)
        m = (C.c_float * 3)(*[float(v) for v in mean])
        s = (C.c_float * 3)(*[float(v) for v in scale])
        _check(lib().tb200_graph_upload_images(self.h, i, buf.ptr, buf.nbytes, descs, m, s))

    def upload_detect_images(self, i, images, mean, scale, letterbox=True, focus=False):
        """Fill graph input i on the device from decoded images as the YOLO examples prepare them (tb200_graph_upload_detect_images):
        letterboxed as tm_yolov5s.cpp or stretched as tm_yolov3_tiny_uint8.cpp, with the Focus slicing when focus (the input is then
        [N, 12, H/2, W/2]).  Images as for upload_images, but mean and scale index the R, G, B planes.  Returns the per-image geometry
        (a ctypes array of abi.DetectGeometry) that yolo_detect / detections_to_source take to map boxes back to the images."""
        buf, descs = self._stage_pixels(i, images)
        pre = abi.DetectPre()
        pre.mode, pre.focus = (abi.PRE_LETTERBOX if letterbox else abi.PRE_STRETCH), int(bool(focus))
        for k in range(3):
            pre.mean[k], pre.scale[k] = float(mean[k]), float(scale[k])
        geo = (abi.DetectGeometry * len(descs))()
        _check(lib().tb200_graph_upload_detect_images(self.h, i, buf.ptr, buf.nbytes, descs, C.byref(pre), geo))
        return geo

    def launch(self):
        _check(lib().tb200_graph_launch(self.h))

    def download(self, i, out):
        _check(lib().tb200_graph_download(self.h, i, out.ctypes.data))

    def sync(self):
        _check(lib().tb200_graph_sync(self.h))

    def read_tensor(self, t):
        out = np.empty(self.dims(t), dtype=self.gdef.np_dtype)
        _check(lib().tb200_graph_read_tensor(self.h, t, out.ctypes.data))
        return out

    def layer_kernels(self):
        return [lib().tb200_graph_layer_kernel(self.h, i).decode() for i in range(len(self.gdef.layers))]

    def num_launches(self):
        return lib().tb200_graph_num_launches(self.h)

    def profile(self):
        ms = (C.c_float * len(self.gdef.layers))()
        _check(lib().tb200_graph_profile(self.h, ms, len(self.gdef.layers)))
        return list(ms)

    def work(self):
        ops, byts = C.c_double(), C.c_double()
        _check(lib().tb200_graph_work(self.h, C.byref(ops), C.byref(byts)))
        return ops.value, byts.value

    def weight_arena(self):
        p, n = C.c_void_p(), C.c_size_t()
        _check(lib().tb200_graph_weight_arena(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def shards(self):
        """[(cuda device, first image, number of images)] -- how the batch was cut over the context's GPUs."""
        out = []
        for i in range(lib().tb200_graph_num_shards(self.h)):
            d, f, n = C.c_int(), C.c_int(), C.c_int()
            _check(lib().tb200_graph_shard(self.h, i, C.byref(d), C.byref(f), C.byref(n)))
            out.append((d.value, f.value, n.value))
        return out

    def arena_bytes(self):
        """(activation arena, the same without slot reuse, weight arena) in bytes, GPU 0's shard."""
        a, u, w = C.c_size_t(), C.c_size_t(), C.c_size_t()
        _check(lib().tb200_graph_arena_bytes(self.h, C.byref(a), C.byref(u), C.byref(w)))
        return a.value, u.value, w.value

    def yolo_detect(self, heads, num_classes=80, prob_threshold=0.4, nms_threshold=0.25, max_per_image=256, max_candidates=0, version=3,
                    geometry=None, letterbox=True):
        """Region decode + NMS on the device from the graph's output tensors of the last run: tb200_graph_yolo_detect (version=3,
        the box formula of examples/tm_yolov3_tiny_uint8.cpp) or tb200_graph_yolov5_detect (version=5, examples/tm_yolov5s.cpp).
        heads: [(graph output index, stride, six anchor values)] in proposal order.  Returns per image a list of
        (x, y, w, h, prob, label), in network-input pixels, or with `geometry` (from upload_detect_images, made with the same
        `letterbox`) in source pixels of each image (tb200_detections_to_source)."""
        if version not in (3, 5):
            raise ValueError(f"version must be 3 or 5, not {version!r}")
        p = abi.YoloParams()
        p.num_heads = len(heads)
        for i, (oi, stride, anchors) in enumerate(heads):
            p.heads[i].output_index, p.heads[i].stride = int(oi), int(stride)
            for k in range(6):
                p.heads[i].anchors[k] = float(anchors[k])
        p.num_classes, p.prob_threshold, p.nms_threshold, p.max_candidates = int(num_classes), float(prob_threshold), float(nms_threshold), int(max_candidates)
        n = self.dims(self.gdef.outputs[0])[0]
        out = (abi.Detection * (n * max_per_image))()
        counts = (C.c_int32 * n)()
        fn = lib().tb200_graph_yolo_detect if version == 3 else lib().tb200_graph_yolov5_detect
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        _check(fn(self.h, C.byref(p), out, int(max_per_image), counts))
        if geometry is not None:
            if len(geometry) != n:
                raise ValueError(f"{len(geometry)} geometries for {n} images")
            _check(lib().tb200_detections_to_source(abi.PRE_LETTERBOX if letterbox else abi.PRE_STRETCH, geometry, n, out, int(max_per_image), counts))
        res = []
        for i in range(n):
            if counts[i] < 0:
                raise TB200Error(abi.ERR_INVALID, f"image {i}: {-counts[i]} boxes / candidates do not fit")
            res.append([(d.x, d.y, d.w, d.h, d.prob, d.label) for d in out[i * max_per_image:i * max_per_image + counts[i]]])
        return res

    def topk(self, output_index=0, k=5):
        """What the classification examples print for every image of the last run (tb200_graph_topk): graph output `output_index`
        dequantised and ranked on the device in print_topk's order, its tie order included.  Returns (scores [N, k] float32,
        ids [N, k] int32); an id is the class's position among the image's elements in NCHW order."""
        n = self.dims(self.gdef.outputs[output_index])[0]
        out = np.zeros((n, max(int(k), 0)), np.dtype([("score", np.float32), ("id", np.int32)]))
        assert out.dtype.itemsize == C.sizeof(abi.ClassScore)
        _check(lib().tb200_graph_topk(self.h, int(output_index), int(k), out.ctypes.data))
        return np.ascontiguousarray(out["score"]), np.ascontiguousarray(out["id"])

    def pack_cache_state(self):
        """0: no cache directory, 1: packed and written to the cache, 2: arena image read from the cache."""
        return lib().tb200_graph_pack_cache_state(self.h)

    def close(self):
        if self.h:
            lib().tb200_graph_postrun(self.h)
            self.h = C.c_void_p()
        if getattr(self, "_pixels", None) is not None:
            self._pixels.free()
            self._pixels = None
