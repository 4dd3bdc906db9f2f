/*
 * tengine_b200.h -- C ABI of the H100 (sm_90a) int8/uint8 convolution + GEMM device backend for Tengine.
 *
 * Plain C, plain pointers and sizes; no CUDA, torch or Tengine types appear in any signature.
 * libtengine_b200.so exports exactly the symbols declared here.  Every entry point names the
 * reference interface (path relative to the Tengine tree, file:line) whose role it takes over.
 *
 * Two layers:
 *   tb200_graph_*   what `struct device` (source/device/device.h:41-108) asks of a device for one
 *                   subgraph: pre_run / run / post_run.  source/device/b200/ (this repo's
 *                   tengine_b200/device/) translates ir_subgraph -> tb200_tensor_desc/tb200_layer_desc and
 *                   forwards to these.
 *   tb200k_*        thin per-kernel launchers on DEVICE pointers (NHWC, channel-padded), the analogue of
 *                   the CPU device's per-op kernels (conv_hcl_run, conv_dw_run_int8, ref_fc_int8 ...).
 *
 * Conventions: every function returns 0 on success and a negative value on failure
 * (Tengine's convention, source/api/c_api.c:463,482,533); tb200_last_error() describes the failure.
 * There is NO CPU fallback anywhere behind this ABI: without a usable CUDA device every compute entry
 * point fails with TB200_ERR_NO_DEVICE.
 */
#ifndef TENGINE_B200_H
#define TENGINE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define TB200_API __attribute__((visibility("default")))
#else
#define TB200_API
#endif

#define TB200_ABI_VERSION 2

/* ---- error codes ------------------------------------------------------------------------------- */
#define TB200_OK 0
#define TB200_ERR_INVALID (-1)     /* bad argument / unsupported parameter combination                 */
#define TB200_ERR_NO_DEVICE (-2)   /* no CUDA device, or not sm_90                                     */
#define TB200_ERR_CUDA (-3)        /* a CUDA runtime/driver call failed                                */
#define TB200_ERR_NOMEM (-4)
#define TB200_ERR_UNSUPPORTED (-5) /* op/dtype not implemented on device (caller must keep it on CPU)  */

/* ---- data types: values equal TENGINE_DT_* (source/api/c_api.h:58-63) --------------------------- */
#define TB200_DT_FP32 0
#define TB200_DT_INT8 2
#define TB200_DT_UINT8 3
#define TB200_DT_INT32 4

/* ---- ops: the subset of source/operator/op.h:38-145 that appears in the five north-star graphs --- */
enum tb200_op
{
    TB200_OP_CONV = 0,     /* OP_CONV     conv_param  (operator/prototype/convolution_param.h:28-45) */
    TB200_OP_FC = 1,       /* OP_FC       fc_param    (operator/prototype/fc_param.h:27)             */
    TB200_OP_POOL = 2,     /* OP_POOL     pool_param  (operator/prototype/pooling_param.h:36-57)     */
    TB200_OP_RELU = 3,     /* OP_RELU     relu_param  (operator/prototype/relu_param.h:27-30)        */
    TB200_OP_ELTWISE = 4,  /* OP_ELTWISE  eltwise_param (operator/prototype/eltwise_param.h:50-57)   */
    TB200_OP_CONCAT = 5,   /* OP_CONCAT   concat_param (axis == 1 only)                              */
    TB200_OP_UPSAMPLE = 6, /* OP_UPSAMPLE upsample_param (nearest, integer scale)                    */
    TB200_OP_IDENTITY = 7, /* OP_DROPOUT at inference                                                */
    TB200_OP_SOFTMAX = 8,  /* OP_SOFTMAX  softmax_param (axis == 1), softmax/softmax_kernel_ref_{int8,uint8}.c */
    TB200_OP_SIGMOID = 9,  /* OP_SIGMOID  sigmoid/sigmoid_ref.c:84 (int8), :129 (uint8)               */
    TB200_OP_HARDSWISH = 10, /* OP_HARDSWISH hardswish/hardswish_kernel_ref_uint8.c:41 (uint8 only, as the reference) */
    TB200_OP_RESHAPE = 11, /* OP_RESHAPE / OP_FLATTEN: the same bytes in NCHW order under the output tensor's dims
                              (flatten/flatten_ref.c:49-83, reshape/reshape_ref.c)                     */
    TB200_OP_COUNT_
};

/* Numeric recipe of the requantising epilogue.  The reference has several float recipes for the
 * "same" op (SURVEY.md section 7 "Hard parts"); the device reproduces whichever the CPU device would have
 * selected so that results are bit-identical, not merely within +-1 LSB.
 *   HCL : conv_kernel_x86.c:1796-1893 / conv_dw_hcl_x86.c:97-269 / conv_direct_hcl_int8_x86.c
 *         f = ((float)(acc+bias) * s_in) * s_w[oc]; act>0 means clip to [0,6]; q = round(f / s_out)
 *   REF : conv_kernel_ref_int8.c:42-177
 *         f = (float)(acc+bias) * (s_in*s_w[oc]); act in {0,1,6}; q = round(f / s_out)
 * For uint8 convs both mean "integer-exact sum of (q_x-zp_x)(q_w-zp_w), then the float epilogue of
 * conv_kernel_x86.c:1703-1794 (HCL) or conv_kernel_ref_uint8.c:42-195 (REF)"; the reference accumulates in
 * fp32, which is where the +-1 LSB tolerance of the north star comes from. */
#define TB200_RECIPE_HCL 0
#define TB200_RECIPE_REF 1

/* eltwise types used: values equal enum EltType (operator/prototype/eltwise_param.h:28-48) */
#define TB200_ELT_PROD 0
#define TB200_ELT_SUM 2

/* pooling methods (operator/prototype/pooling_param.h:30-34) */
#define TB200_POOL_MAX 0
#define TB200_POOL_AVG 1

/* A tensor of the graph as the host sees it: logical layout NCHW (Tengine's internal layout,
 * source/serializer/tmfile/tm2_serializer.c:169-173), per-tensor quantisation
 * (source/graph/tensor.h:52-98: scale, zero_point). */
typedef struct tb200_tensor_desc
{
    int32_t data_type;  /* TB200_DT_INT8 | TB200_DT_UINT8 (activations)                    */
    int32_t dims[4];    /* n, c, h, w (FC outputs: n, c, 1, 1)                             */
    float scale;        /* ir_tensor->scale                                                */
    int32_t zero_point; /* ir_tensor->zero_point (0 for int8)                              */
} tb200_tensor_desc;

/* One node of the subgraph.  Field names follow the reference parameter structs. */
typedef struct tb200_layer_desc
{
    int32_t op;            /* enum tb200_op                                                          */
    int32_t num_inputs;    /* activation inputs (1; 2 for eltwise; up to 4 for concat)               */
    int32_t inputs[4];     /* indices into the tensor table                                          */
    int32_t output;        /* index into the tensor table                                            */
    /* conv_param / pool_param */
    int32_t kernel_h, kernel_w, stride_h, stride_w;
    int32_t pad_h0, pad_h1, pad_w0, pad_w1;
    int32_t dilation_h, dilation_w;
    int32_t group;
    int32_t activation;    /* conv_param.activation: -1 none, 0 ReLU, 1 ReLU1, 6 ReLU6               */
    int32_t recipe;        /* TB200_RECIPE_*                                                         */
    /* pool_param */
    int32_t pool_method, pool_global, caffe_flavor;
    /* relu_param / eltwise_param / concat_param / upsample_param */
    float negative_slope;
    int32_t elt_type;
    int32_t axis;
    int32_t up_scale;
    /* constant operands (HOST pointers, read during tb200_graph_prerun only):
     * weight : [Cout][Cin/group][kh][kw] int8 or uint8 (FC: [Cout][hidden]) -- ir_tensor->data of input 1
     * bias   : [Cout] int32 or NULL                                        -- ir_tensor->data of input 2
     * weight_scales : int8: per-output-channel scale_list[Cout]; uint8: pointer to ONE float (per tensor)
     * weight_zero   : uint8 per-tensor zero point (0 for int8)
     * bias_scale    : bias_tensor->scale (only fc_ref.c:142 uses it; conv recomputes s_in*s_w) */
    const void* weight;
    const int32_t* bias;
    const float* weight_scales;
    int32_t weight_zero;
    float bias_scale;
} tb200_layer_desc;

typedef struct tb200_context tb200_context; /* one GPU -- or a group of GPUs driven by this process -- : streams, NCCL communicators */
typedef struct tb200_graph tb200_graph;     /* one per Tengine subgraph (subgraph->device_graph) */

/* ---- library / device ---------------------------------------------------------------------------- */
TB200_API int tb200_abi_version(void);
TB200_API const char* tb200_last_error(void);
/* number of visible sm_90 devices (0 if none; never fails) */
TB200_API int tb200_device_count(void);

/* interface->init / release_device (source/device/device.h:44,65): bind one GPU. */
TB200_API int tb200_context_create(int cuda_device, tb200_context** out);
TB200_API int tb200_context_destroy(tb200_context* ctx);
/* the CUDA stream (cudaStream_t) all work of this context is ordered on, for callers that time with events */
TB200_API void* tb200_context_stream(tb200_context* ctx);

/* Several GPUs behind ONE device (SURVEY.md 8(e); the option-blob precedent is trt_option,
 * source/device/tensorrt/trt_define.h:36-42).  Every tb200_graph_* call on such a context shards dim 0 of the batch
 * contiguously over the GPUs: prerun plans one shard per GPU, packs the weights once (GPU 0) and moves the arena to
 * the others with ONE grouped ncclBroadcast (communicators from ncclCommInitAll; NCCL is dlopen'ed); run copies each
 * GPU's slice of the caller's NCHW buffers straight to that GPU and joins all streams before it returns.  There is no
 * collective in the steady state.  Listing a device twice (single-GPU test boxes) keeps every mechanism except NCCL
 * itself, which refuses duplicate devices: the arena is then copied with cudaMemcpyPeerAsync. */
TB200_API int tb200_context_create_multi(const int* cuda_devices, int num_devices, tb200_context** out);
TB200_API int tb200_context_num_gpus(tb200_context* ctx);
TB200_API int tb200_context_gpu(tb200_context* ctx, int index);        /* CUDA ordinal of GPU `index` of the group */
TB200_API void* tb200_context_stream_of(tb200_context* ctx, int index); /* its stream (cudaStream_t) */
TB200_API const char* tb200_context_broadcast_kind(tb200_context* ctx); /* "none" | "nccl" | "memcpy_peer" */

/* What set_context_device(ctx, "B200", &opt, sizeof opt) carries (source/api/c_api.c:207-211 memcpy's it; the first field
 * must be the device name because sched_prerun dereferences *(char**)options, scheduler.c:49).  Zero = default. */
typedef struct tb200_device_option
{
    char* dev_name;
    int32_t num_gpus;   /* 0: TG_B200_GPUS or 1 */
    int32_t first_gpu;  /* CUDA ordinal of the first GPU of the group (TG_B200_GPU) */
} tb200_device_option;

/* Page-locked host memory for callers that want it.  tb200_graph_run does not require it: a pageable caller buffer is
 * page-locked in place (cudaHostRegister) the first time it is seen and stays registered until postrun. */
TB200_API void* tb200_host_alloc(size_t bytes);
TB200_API void tb200_host_free(void* p);

/* ---- subgraph life cycle -------------------------------------------------------------------------- */
#define TB200_PRERUN_DEFAULT 0
#define TB200_PRERUN_NO_WEIGHTS 1 /* allocate the packed-weight arena but leave it for a broadcast to fill */
#define TB200_PRERUN_NO_GRAPH 2   /* do not capture a CUDA graph (debug / profiling by kernel)          */
#define TB200_PRERUN_NO_TENSORCORE 4 /* route every conv through the CUDA-core direct kernels (cross-check) */
#define TB200_PRERUN_POISON_ARENA 8  /* fill the activation arena with 0xA5 instead of 0 (tests: producers own their pad lanes) */

/* interface->pre_run (device.h:47; cuda precedent cuda_graph.cc:36-42, cuda_executor.cc:136-180):
 * validate, choose a kernel per layer, pre-pack weights/bias/scales into ONE device arena (the analogue of
 * conv_hcl_prerun, conv_kernel_x86.c:2137-2209), plan the activation arena for `dims[0]` images, record
 * the launch sequence into a CUDA graph.  `input_ids/output_ids` are subgraph->input/output_tensor_list. */
TB200_API int tb200_graph_prerun(tb200_context* ctx, const tb200_tensor_desc* tensors, int num_tensors,
                                 const tb200_layer_desc* layers, int num_layers, const int32_t* input_ids,
                                 int num_inputs, const int32_t* output_ids, int num_outputs, int flags,
                                 tb200_graph** out);

/* interface->run (device.h:50; cuda precedent cuda_executor.cc:182-215): synchronous.  Host NCHW buffers in,
 * host NCHW buffers out (ir_tensor->data of the subgraph's input/output tensors).  Copies H2D, converts
 * NCHW->NHWC on device, launches the graph, converts back, copies D2H, waits. */
TB200_API int tb200_graph_run(tb200_graph* g, const void* const* host_inputs, void* const* host_outputs);

/* The same three stages separately, for callers that keep data resident or time the kernels alone. */
TB200_API int tb200_graph_upload(tb200_graph* g, int input_index, const void* host_nchw);
TB200_API int tb200_graph_launch(tb200_graph* g);                 /* asynchronous on the context stream */
TB200_API int tb200_graph_download(tb200_graph* g, int output_index, void* host_nchw);
TB200_API int tb200_graph_sync(tb200_graph* g);

/* interface->post_run (device.h:53) */
TB200_API int tb200_graph_postrun(tb200_graph* g);

/* Packed-weight arena (device pointer + size): the object of the single NCCL broadcast at prerun when the
 * batch is sharded over several GPUs (SURVEY.md 8(e)); identical layout on every rank for identical graphs. */
TB200_API int tb200_graph_weight_arena(tb200_graph* g, void** device_ptr, size_t* bytes);

/* On-box peak of the int8 tensor pipe in TOP/s: a pure wgmma m64n128k32 s8 loop (two warpgroups per SM), the measured
 * denominator of the tensor roofline that bench.py reports for compute-bound kernel families (SURVEY.md 8(d)). */
TB200_API int tb200_probe_int8_tops(tb200_context* ctx, double* tops);

/* Packed-weight cache (SURVEY.md 8(f)-3; the CPU analogue is conv_hcl_prerun's interleaved weights, conv_kernel_x86.c:2137-2209,
 * rebuilt at every prerun): with a directory set -- here or with TG_B200_PACK_CACHE -- prerun stores the packed arena image under a
 * hash of everything it depends on (descriptors, kernel choices, weights, biases, scales) and later preruns of the same model read
 * it back instead of packing.  NULL or "" disables.  tb200_graph_pack_cache_state: 0 no cache, 1 packed + written, 2 read.
 * (The north star's int4 weights are not offered: Tengine has no int4 tensor type, c_api.h:58-63, so nothing could be checked
 * against the reference; int8 / uint8 weights are what its files carry.) */
TB200_API int tb200_pack_cache_dir(const char* dir);
TB200_API int tb200_graph_pack_cache_state(tb200_graph* g);

/* The sharding rule (pure function, no GPU needed): images [first, first + num) of a batch of n belong to shard `rank` of `world`;
 * contiguous slices of dim 0 of the NCHW buffers, the first n % world shards one image longer. */
TB200_API int tb200_shard_range(int n_images, int world, int rank, int* first_image, int* num_images);

/* multi-GPU contexts: re-send the arena (after a caller filled GPU 0's arena itself, TB200_PRERUN_NO_WEIGHTS) */
TB200_API int tb200_graph_broadcast_weights(tb200_graph* g);
/* how the batch was cut: shard `index` runs images [first_image, first_image + num_images) on CUDA device *cuda_device */
TB200_API int tb200_graph_num_shards(tb200_graph* g);
TB200_API int tb200_graph_shard(tb200_graph* g, int index, int* cuda_device, int* first_image, int* num_images);
/* bytes of the activation arena of GPU 0's shard, what it would be without slot reuse, and of the weight arena */
TB200_API int tb200_graph_arena_bytes(tb200_graph* g, size_t* activation_bytes, size_t* unshared_bytes, size_t* weight_bytes);

/* Introspection for tests / bench / TG_DEBUG_TIME-style reports */
TB200_API int tb200_graph_num_launches(tb200_graph* g);            /* kernels launched per tb200_graph_launch */
TB200_API const char* tb200_graph_layer_kernel(tb200_graph* g, int layer); /* name of the kernel chosen */
/* copy any tensor of the graph back to host NCHW (valid after a launch when prerun had TB200_PRERUN_NO_GRAPH
 * or the tensor is a graph output; intermediates share arena slots otherwise) */
TB200_API int tb200_graph_read_tensor(tb200_graph* g, int tensor_id, void* host_nchw);
/* per-layer device time in ms of the last tb200_graph_profile() run (events around each launch) */
TB200_API int tb200_graph_profile(tb200_graph* g, float* layer_ms, int num_layers);
/* algorithmic work of one launch: 2*MACs of conv+fc, and bytes = conv/fc in+out activations + weights + bias */
TB200_API int tb200_graph_work(tb200_graph* g, double* ops, double* bytes);

/* ---- detection post-processing on the device (SURVEY.md 8(f)-4) ------------------------------------------------------
 * YOLO region decode + score threshold + sort + NMS on the graph's quantised output tensors where they lie in HBM (after
 * tb200_graph_run / tb200_graph_launch); only the kept boxes come back.  Restates the application code of
 * examples/tm_yolov3_tiny_uint8.cpp:57-132,176-250,464-500 (the head tensors are [N, anchors*(5+classes), H, W]; proposals are
 * generated head by head in the order given here, sorted by the example's quicksort, suppressed greedily). */
typedef struct tb200_yolo_head
{
    int32_t output_index; /* which graph output */
    int32_t stride;       /* 32, 16, 8 */
    float anchors[6];     /* (w, h) of the three anchors of this head */
} tb200_yolo_head;
typedef struct tb200_yolo_params
{
    int32_t num_heads;    /* <= 3 */
    tb200_yolo_head heads[3];
    int32_t num_classes;  /* 80 */
    float prob_threshold, nms_threshold;
    int32_t max_candidates; /* per image, before NMS (0: 4096) */
} tb200_yolo_params;
typedef struct tb200_detection
{
    float x, y, w, h; /* box in network-input pixels (cv::Rect_<float> of the example) */
    float prob;
    int32_t label;
} tb200_detection;
/* out: [images][max_per_image]; counts[image] = boxes kept (negative: more than fit -- -needed is returned there) */
TB200_API int tb200_graph_yolo_detect(tb200_graph* g, const tb200_yolo_params* p, tb200_detection* out, int max_per_image, int32_t* counts);

/* ---- kernel launchers (device pointers; NHWC with channels padded to tb200k_cpad(c)) --------------- */
typedef struct tb200k_epilogue
{
    const int32_t* bias;   /* [Cout_pad] device, zeros when the layer has no bias          */
    const float* w_scale;  /* [Cout_pad] device (uint8: every entry = the per-tensor scale) */
    float in_scale, out_scale;
    int32_t in_zero, w_zero, out_zero;
    int32_t activation;    /* conv_param.activation */
    int32_t recipe;        /* TB200_RECIPE_* */
    int32_t is_uint8;      /* 0: int8 clamp +-127; 1: uint8 clamp 0..255 */
    int32_t fc_rounding;   /* 1: fc_ref.c:225 recipe roundf(acc * ((s_in*s_w)/s_out)) */
    float w_scale_tensor;  /* uint8 only: the per-tensor weight scale (host copy of w_scale[0]) */
} tb200k_epilogue;

typedef struct tb200k_conv_shape
{
    int32_t n, h, w, c;         /* input  (c = logical channels) */
    int32_t oh, ow, oc;         /* output */
    int32_t kh, kw, sh, sw, ph0, pw0, dh, dw, group;
} tb200k_conv_shape;

TB200_API int tb200k_cpad(int channels); /* channel padding rule of the device layout (multiple of 16) */

/* generic direct convolution on CUDA cores (any kernel/stride/pad/dilation/group); weights
 * [Cout_pad][kh][kw][Cin_g_pad].  Takes the role of ref_conv_int8/ref_conv_uint8. */
TB200_API int tb200k_conv_direct(const void* in, const void* weight, void* out, const tb200k_conv_shape* s,
                                 const tb200k_epilogue* e, void* stream);
/* depthwise 3x3 (group == c == oc), weights [3][3][C_pad].  Takes the role of convdw3x3s{1,2}_int8_sse. */
TB200_API int tb200k_conv_dw3x3(const void* in, const void* weight, void* out, const tb200k_conv_shape* s,
                                const tb200k_epilogue* e, void* stream);
/* NCHW stem (c <= 4) -> NHWC, weights [Cout_pad][kh][kw][4].  Takes the role of conv3x3s2_int8_sse on the
 * network input; it also performs the NCHW->NHWC conversion of the graph input. */
TB200_API int tb200k_conv_stem_nchw(const void* in_nchw, const void* weight, void* out, const tb200k_conv_shape* s,
                                    const tb200k_epilogue* e, void* stream);
/* 1x1 convolution / FC as a wgmma (s8 / u8) GEMM: out[M][Cout_pad] = in[M][K_pad] . weight[Cout_pad][K_pad]^T,
 * TMA-staged operands, a shared-memory accumulator image, fused requantising epilogue.  Takes the role of
 * im2col + sgemm_i8 + sgemm_int8 epilogue (conv_kernel_x86.c:187,1008,1796) for kernel 1x1. */
TB200_API int tb200k_gemm_i8(const void* in, const void* weight, void* out, int64_t m, int32_t k_pad, int32_t oc,
                             const tb200k_epilogue* e, void* stream);
/* layout conversion host-NCHW <-> device-NHWC(pad) */
TB200_API int tb200k_nchw_to_nhwc(const void* in, void* out, int n, int c, int h, int w, void* stream);
TB200_API int tb200k_nhwc_to_nchw(const void* in, void* out, int n, int c, int h, int w, void* stream);

/* ---- fp32 members of the path (north star: "fp32 paths within 1e-4 rel"); NCHW fp32 DEVICE pointers as Tengine lays them out.
 * Winograd F(4x4, 3x3): 3x3, stride 1, dilation 1, group 1 -- what winograd_support() admits (conv_kernel_x86.c:1896-1915;
 * kernels wino_conv_kernel_x86.c:126,1118,1291,1376).  weight [Cout][Cin][3][3], bias [Cout] or NULL, activation as
 * conv_param.activation (-1 none, 0 ReLU, n > 0 clip to [0, n]).  workspace: tb200k_conv_winograd43_f32_workspace() bytes. */
TB200_API size_t tb200k_conv_winograd43_f32_workspace(const tb200k_conv_shape* s);
TB200_API int tb200k_conv_winograd43_f32(const float* in, const float* weight, const float* bias, float* out, const tb200k_conv_shape* s, int activation,
                                         void* workspace, void* stream);
/* fp32 depthwise 3x3, stride 1 / 2 (conv_dw_kernel_x86.c:2524 conv_dw_run): weight [C][3][3] */
TB200_API int tb200k_conv_dw3x3_f32(const float* in, const float* weight, const float* bias, float* out, const tb200k_conv_shape* s, int activation,
                                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TENGINE_B200_H */
