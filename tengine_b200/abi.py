"""ctypes mirror of include/tengine_b200.h (struct layouts and constants only; no library is loaded here).

Python is not the host language of the backend -- the host side is the C++ Tengine device under
tengine_b200/device/ -- but tests and bench.py drive the same C ABI through these definitions.
"""
import ctypes as C

ABI_VERSION = 2

# TENGINE_DT_* (source/api/c_api.h:58-63)
DT_FP32, DT_INT8, DT_UINT8, DT_INT32 = 0, 2, 3, 4

(OP_CONV, OP_FC, OP_POOL, OP_RELU, OP_ELTWISE, OP_CONCAT, OP_UPSAMPLE, OP_IDENTITY, OP_SOFTMAX, OP_SIGMOID, OP_HARDSWISH,
 OP_RESHAPE) = range(12)
OP_NAMES = ["conv", "fc", "pool", "relu", "eltwise", "concat", "upsample", "identity", "softmax", "sigmoid", "hardswish", "reshape"]

RECIPE_HCL, RECIPE_REF = 0, 1
ELT_PROD, ELT_SUM = 0, 2
POOL_MAX, POOL_AVG = 0, 1

PRERUN_DEFAULT, PRERUN_NO_WEIGHTS, PRERUN_NO_GRAPH, PRERUN_NO_TENSORCORE, PRERUN_POISON_ARENA = 0, 1, 2, 4, 8

ERR_INVALID, ERR_NO_DEVICE, ERR_CUDA, ERR_NOMEM, ERR_UNSUPPORTED = -1, -2, -3, -4, -5


class TensorDesc(C.Structure):
    _fields_ = [("data_type", C.c_int32), ("dims", C.c_int32 * 4), ("scale", C.c_float), ("zero_point", C.c_int32)]


class LayerDesc(C.Structure):
    _fields_ = [
        ("op", C.c_int32), ("num_inputs", C.c_int32), ("inputs", C.c_int32 * 4), ("output", C.c_int32),
        ("kernel_h", C.c_int32), ("kernel_w", C.c_int32), ("stride_h", C.c_int32), ("stride_w", C.c_int32),
        ("pad_h0", C.c_int32), ("pad_h1", C.c_int32), ("pad_w0", C.c_int32), ("pad_w1", C.c_int32),
        ("dilation_h", C.c_int32), ("dilation_w", C.c_int32), ("group", C.c_int32), ("activation", C.c_int32),
        ("recipe", C.c_int32),
        ("pool_method", C.c_int32), ("pool_global", C.c_int32), ("caffe_flavor", C.c_int32),
        ("negative_slope", C.c_float), ("elt_type", C.c_int32), ("axis", C.c_int32), ("up_scale", C.c_int32),
        ("weight", C.c_void_p), ("bias", C.c_void_p), ("weight_scales", C.c_void_p),
        ("weight_zero", C.c_int32), ("bias_scale", C.c_float),
    ]


class KEpilogue(C.Structure):
    _fields_ = [("bias", C.c_void_p), ("w_scale", C.c_void_p), ("in_scale", C.c_float), ("out_scale", C.c_float),
                ("in_zero", C.c_int32), ("w_zero", C.c_int32), ("out_zero", C.c_int32), ("activation", C.c_int32),
                ("recipe", C.c_int32), ("is_uint8", C.c_int32), ("fc_rounding", C.c_int32),
                ("w_scale_tensor", C.c_float)]


class KConvShape(C.Structure):
    _fields_ = [(n, C.c_int32) for n in
                ("n", "h", "w", "c", "oh", "ow", "oc", "kh", "kw", "sh", "sw", "ph0", "pw0", "dh", "dw", "group")]


# every symbol include/tengine_b200.h declares (tests check the library exports exactly these)
EXPORTS = [
    "tb200_abi_version", "tb200_last_error", "tb200_device_count", "tb200_context_create", "tb200_context_destroy",
    "tb200_context_stream", "tb200_context_create_multi", "tb200_context_num_gpus", "tb200_context_gpu", "tb200_context_stream_of",
    "tb200_context_broadcast_kind", "tb200_shard_range", "tb200_graph_broadcast_weights", "tb200_graph_num_shards", "tb200_graph_shard", "tb200_graph_arena_bytes", "tb200_probe_int8_tops", "tb200_pack_cache_dir", "tb200_graph_pack_cache_state", "tb200_graph_yolo_detect", "tb200_graph_yolov5_detect", "tb200_graph_topk", "tb200_graph_set_batch", "tb200_graph_batch", "tb200k_conv_winograd43_f32_workspace", "tb200k_conv_winograd43_f32", "tb200k_conv_dw3x3_f32",
    "tb200_host_alloc", "tb200_host_free", "tb200_graph_prerun", "tb200_graph_run",
    "tb200_graph_upload", "tb200_graph_upload_images", "tb200_graph_upload_detect_images", "tb200_detections_to_source", "tb200_graph_launch", "tb200_graph_download", "tb200_graph_sync", "tb200_graph_postrun",
    "tb200_graph_weight_arena", "tb200_graph_num_launches", "tb200_graph_layer_kernel", "tb200_graph_read_tensor",
    "tb200_graph_profile", "tb200_graph_work", "tb200k_cpad", "tb200k_conv_direct", "tb200k_conv_dw3x3",
    "tb200k_conv_stem_nchw", "tb200k_gemm_i8", "tb200k_nchw_to_nhwc", "tb200k_nhwc_to_nchw", "tb200k_class_topk",
]


class Image(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("w", C.c_int32), ("h", C.c_int32), ("c", C.c_int32)]


PRE_STRETCH, PRE_LETTERBOX = 0, 1


class DetectPre(C.Structure):
    _fields_ = [("mode", C.c_int32), ("focus", C.c_int32), ("mean", C.c_float * 3), ("scale", C.c_float * 3)]


class DetectGeometry(C.Structure):
    _fields_ = [("src_w", C.c_int32), ("src_h", C.c_int32), ("resize_w", C.c_int32), ("resize_h", C.c_int32), ("left", C.c_int32),
                ("top", C.c_int32), ("scale", C.c_float)]


class YoloHead(C.Structure):
    _fields_ = [("output_index", C.c_int32), ("stride", C.c_int32), ("anchors", C.c_float * 6)]


class YoloParams(C.Structure):
    _fields_ = [("num_heads", C.c_int32), ("heads", YoloHead * 3), ("num_classes", C.c_int32), ("prob_threshold", C.c_float),
                ("nms_threshold", C.c_float), ("max_candidates", C.c_int32)]


class Detection(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("w", C.c_float), ("h", C.c_float), ("prob", C.c_float), ("label", C.c_int32)]


TOPK_MAX, TOPK_MAX_CLASSES = 64, 32768


class ClassScore(C.Structure):
    _fields_ = [("score", C.c_float), ("id", C.c_int32)]
