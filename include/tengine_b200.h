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
 * fp32, which is where the +-1 LSB tolerance comes from.  That tolerance holds while the fp32 sum stays near exact
 * (measured: full-size ResNet-50 / YOLOv3-tiny layers, |acc| <= 0.023 * 2^24; K = 4608 with far-end operands, 16.5 * 2^24);
 * at K = 25088 with far-end operands (|acc| ~ 90 * 2^24) the reference's rounded sum is up to 15 LSB from the exact
 * result, which the device keeps. */
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

typedef struct tb200_context tb200_context; /* one GPU -- or a group of GPUs driven by this process -- : streams */
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
 * the others with one cudaMemcpyPeerAsync per GPU; run copies each GPU's slice of the caller's NCHW buffers straight
 * to that GPU and joins all streams before it returns.  There is no collective in the steady state.  A device may be
 * listed more than once (single-GPU test boxes): every mechanism stays the same. */
TB200_API int tb200_context_create_multi(const int* cuda_devices, int num_devices, tb200_context** out);
TB200_API int tb200_context_num_gpus(tb200_context* ctx);
TB200_API int tb200_context_gpu(tb200_context* ctx, int index);        /* CUDA ordinal of GPU `index` of the group */
TB200_API void* tb200_context_stream_of(tb200_context* ctx, int index); /* its stream (cudaStream_t) */
TB200_API const char* tb200_context_broadcast_kind(tb200_context* ctx); /* "none" (one GPU) | "memcpy_peer" (a group) */

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

/* ---- partial batches --------------------------------------------------------------------------------------------------------
 * Make images [0, n) the batch of every later call on g, 1 <= n <= the batch g was prepared for (dims[0] at prerun), without a
 * new prerun: run, upload, download, launch, upload_images, upload_detect_images (and the geometry they return), topk,
 * yolo_detect, yolov5_detect, read_tensor, profile, work and num_launches then cover n images.  Caller buffers need room for n
 * images only; nothing is read or written beyond them (tb200_graph_run page-locks exactly n images of each buffer).  Images
 * n.. of the device arena keep stale bytes that no output ever reaches.
 * On a multi-GPU context shard r runs tb200_shard_range(n, shards, r), and tb200_graph_shard reports that split; a shard whose
 * share is 0 images (n < shards) issues no copy, kernel or graph launch, and its rows of topk / detect outputs do not exist.
 * Synchronous with respect to queued work: every stream of every shard is drained before any launch sequence or CUDA graph is
 * replaced.  Setting the active batch again does nothing; returning to the prepared batch reuses the CUDA graphs captured at
 * prerun (the state is that of prerun, bit for bit); another n builds the launch sequences for n -- the whole batch and the
 * pipeline chunks of tb200_graph_run, cut by prerun's rule at n: two chunks for an even n >= 32, a quarter and three
 * quarters from 64 -- and captures them once (TB200_PRERUN_NO_GRAPH: builds them only).  Those of the most recent such n are
 * kept, so alternating between the prepared batch and one n costs nothing after the first switch.
 * Unchanged: the weight arena, the pack cache, the fused-node plan, the kernel of each layer (tb200_graph_layer_kernel) and
 * the activation arena.
 * TB200_ERR_INVALID for a null graph, n < 1 or n above the prepared batch; TB200_ERR_UNSUPPORTED for n other than the
 * prepared batch on a graph whose tensors differ in dim 0 (prerun runs such a graph unsharded, as a whole).  A failed call
 * leaves the active batch, and everything that runs, as it was. */
TB200_API int tb200_graph_set_batch(tb200_graph* g, int n);
/* the active batch: the prepared one until tb200_graph_set_batch changes it (TB200_ERR_INVALID for a null graph) */
TB200_API int tb200_graph_batch(tb200_graph* g);

/* The same three stages separately, for callers that keep data resident or time the kernels alone. */
TB200_API int tb200_graph_upload(tb200_graph* g, int input_index, const void* host_nchw);
TB200_API int tb200_graph_launch(tb200_graph* g);                 /* asynchronous on the context stream */
TB200_API int tb200_graph_download(tb200_graph* g, int output_index, void* host_nchw);
TB200_API int tb200_graph_sync(tb200_graph* g);

/* ---- classification preprocessing on the device -----------------------------------------------------------------------------
 * Decoded 8-bit images in, the quantised graph input out.  Restates what examples/tm_classification_int8.c:43-62
 * (get_input_int8_data) and examples/tm_classification_uint8.c:43-62 (get_input_uint8_data) do per image through
 * examples/common/tengine_operations.c: load_image_stb (:51-82; RGBA loses its alpha byte), rgb2bgr_permute (:651-673; output plane k
 * is source channel 2 - k), the fixed-point bilinear resize tengine_resize_f32 (:870-979, non-NEON branch; 11-bit weights from float
 * positions, including its extrapolating first outputs of an upsample and its last output taking source pixel w - 2 with weight 1),
 * imread2caffe (:101-115: (v - mean[k]) * scale[k]), then int8: round(x / scale) clamped to +-127, uint8: round(x / scale +
 * zero_point) clamped to 0..255, with the graph input's own H, W, scale and zero point.  round() takes halfway cases away from zero; a
 * quotient outside int's range (or NaN) converts to INT_MIN as on x86-64 and so clamps to -127 / 0. */
typedef struct tb200_image
{
    uint64_t offset; /* byte offset of pixel (0,0) in the pixel buffer */
    int32_t w, h, c; /* h rows of w pixels of c interleaved bytes, rows unpadded: what stbi_load returns; c = 3 (RGB) or 4 (RGBA) */
} tb200_image;
/* Fills graph input `input_index` ([N, 3, H, W], int8 or uint8) from images[0..N) on the device, byte for byte as the examples'
 * get_input_int8_data / get_input_uint8_data would fill the host tensor for each image.  `mean` and `scale` index the B, G, R planes,
 * as the examples' -w / -s options do.  Images may have different sizes and lie anywhere in the buffer.
 * pixels: HOST memory, page-locked in place like tb200_graph_run's buffers; it must stay unchanged until a tb200_graph_sync has
 * returned after this call.  Asynchronous on the context stream, like tb200_graph_upload; follow with tb200_graph_launch.
 * Checked before anything is copied: TB200_ERR_INVALID for a null argument, an input index out of range, an input whose dims[1] != 3,
 * w or h outside 2..32767 (the resize reads column w - 2 and keeps positions in int16_t), an image not inside pixel_bytes, a
 * non-finite mean or scale.  TB200_ERR_UNSUPPORTED for c other than 3 or 4: for c == 1 the example's gray2bgr (:694-713) writes three
 * interleaved copies into an image it then reads as planar, so there is no meaningful result to reproduce; for c == 2
 * rgb2bgr_permute writes plane 2 - c outside a two-plane image. */
TB200_API int tb200_graph_upload_images(tb200_graph* g, int input_index, const void* pixels, size_t pixel_bytes,
                                        const tb200_image* images, const float mean[3], const float scale[3]);

/* ---- detection preprocessing on the device ----------------------------------------------------------------------------------
 * Decoded 8-bit images in, the quantised input of a YOLO graph out, byte for byte as the examples fill it after cv::imread(file, 1) and
 * cv::cvtColor(BGR2RGB), so the planes are R, G, B and mean / scale index R, G, B (unlike tb200_graph_upload_images):
 *   TB200_PRE_STRETCH    examples/tm_yolov3_tiny_uint8.cpp:136-170 (tm_yolov4_tiny_uint8.cpp:137-170): cv::resize to the input's W x H.
 *   TB200_PRE_LETTERBOX  examples/tm_yolov5s.cpp:263-337 / :339-392: a float scale chosen by a double comparison, resized size
 *                        int(scale * cols) (a float product truncated: it can be one short of the input size), cv::resize to it,
 *                        borders top = (H - resize_h) / 2, left = (W - resize_w) / 2, filled by cv::copyMakeBorder with byte 0
 *                        (its destination takes the 8-bit source type, so the grey float image built before it is unused).
 * cv::resize is INTER_LINEAR on 8-bit images as OpenCV computes it: float positions from double arithmetic, 11-bit weights rounded to
 * nearest, the horizontal position clamped to the image, the vertical one not (rows are clipped instead, so an upscale's first and last
 * rows blend a row with itself), and the two-term fixed-point vertical sum of OpenCV's SIMD path.  Then (v - mean[c]) * scale[c] in
 * float and round(x / s_in + (float)zero_point) clamped to +-127 (int8) or 0..255 (uint8), halfway cases away from zero, a quotient
 * out of int's range (or NaN) -> INT_MIN as on x86-64 (tm_yolox_int8.cpp:336-341, tm_yolov3_tiny_uint8.cpp:164-168).
 * focus = 1: the YOLOv5 (<= v5) Focus slicing of tm_yolov5s.cpp:317-337: the image is laid out at H x W and output channel
 * (i * 2 + g) * 3 + c takes column offset i and row offset g of plane c; the graph input is then [N, 12, H/2, W/2]. */
#define TB200_PRE_STRETCH 0
#define TB200_PRE_LETTERBOX 1
typedef struct tb200_detect_pre
{
    int32_t mode;     /* TB200_PRE_STRETCH | TB200_PRE_LETTERBOX */
    int32_t focus;    /* 1: graph input [N, 12, H/2, W/2] from an H x W image; 0: graph input [N, 3, H, W] */
    float mean[3];    /* R, G, B */
    float scale[3];
} tb200_detect_pre;
/* Where image i landed in the H x W laid-out input, computed on the host with the example's own arithmetic.  Stretch: resize = W x H,
 * left = top = 0, scale = 0.  Letterbox: the resized size, the left / top borders and scale_letterbox. */
typedef struct tb200_detect_geometry
{
    int32_t src_w, src_h;       /* the image's size */
    int32_t resize_w, resize_h; /* the size cv::resize produced */
    int32_t left, top;          /* its position in the laid-out image */
    float scale;
} tb200_detect_geometry;
/* Fills graph input `input_index` from images[0..N) on the device and writes each image's geometry to geometry_out[0..N) (host memory;
 * NULL skips it).  Images, buffer and asynchrony are those of tb200_graph_upload_images; follow with tb200_graph_launch.  Checked before
 * anything is copied: TB200_ERR_INVALID for a null argument, an input index out of range, an input that is not int8 / uint8, a mode
 * other than the two, focus not 0 / 1, an input whose dims[1] is not 3 (12 with focus), w or h outside 2..32767,
 * an image not inside pixel_bytes, a letterbox whose resized width or height would be 0, a non-finite mean or scale;
 * TB200_ERR_UNSUPPORTED for c other than 3 or 4. */
TB200_API int tb200_graph_upload_detect_images(tb200_graph* g, int input_index, const void* pixels, size_t pixel_bytes, const tb200_image* images,
                                               const tb200_detect_pre* pre, tb200_detect_geometry* geometry_out);
/* tb200_detections_to_source (after tb200_detection below) maps the boxes found in such an input back to source pixels. */

/* interface->post_run (device.h:53) */
TB200_API int tb200_graph_postrun(tb200_graph* g);

/* Packed-weight arena (device pointer + size): what prerun copies from GPU 0 to the other GPUs when the
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
/* how the active batch is cut: shard `index` runs images [first_image, first_image + num_images) on CUDA device *cuda_device
 * (num_images may be 0 after tb200_graph_set_batch to fewer images than shards) */
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
/* The same for YOLOv5 heads: restates examples/tm_yolov5s.cpp:140-207,561-576.  Parameters, output layout and the overflow
 * convention are those of tb200_graph_yolo_detect; only the box formula differs:
 *   centre = (sigmoid(tx) * 2 - 0.5 + w) * stride, size = sigmoid(tw) * sigmoid(tw) * 4 * anchor_w  (float, in that order).
 * Quantised heads are dequantised as ((float)q - zero_point) * scale.  Pass the heads in the example's proposal order:
 * stride 32, 16, 8 (:567-572), with anchors {116,90, 156,198, 373,326}, {30,61, 62,45, 59,119}, {10,13, 16,30, 33,23} (:143).
 * Boxes are in network-input pixels; tb200_detections_to_source applies the example's letterbox back-mapping (:580-626). */
TB200_API int tb200_graph_yolov5_detect(tb200_graph* g, const tb200_yolo_params* p, tb200_detection* out, int max_per_image, int32_t* counts);
/* Pure host function (no GPU needed), the step the examples take after NMS: rewrites dets[i * max_per_image + k], k < counts[i], from
 * network-input pixels to source pixels of image i in place, `mode` and geometry[i] as tb200_graph_upload_detect_images used and returned
 * them.  Stretch: tm_yolov3_tiny_uint8.cpp:501-532 (multiply by source size / input size).  Letterbox: tm_yolov5s.cpp:580-625 (subtract
 * left / top, then multiply x by src_h / resize_h and y by src_w / resize_w -- the example's swap, kept).  Both then clamp the corners to
 * [0, src_w - 1] x [0, src_h - 1] and rebuild w / h from them, in float.  Images with a negative (overflow) count are left as they are.
 * TB200_ERR_INVALID for a bad mode, a null pointer, num_images < 0, max_per_image < 1, a count above max_per_image or a geometry size
 * below 1. */
TB200_API int tb200_detections_to_source(int mode, const tb200_detect_geometry* geometry, int num_images, tb200_detection* dets, int max_per_image,
                                         const int32_t* counts);

/* ---- classification post-processing on the device ---------------------------------------------------------------------------
 * The last step of examples/tm_classification_int8.c and examples/tm_classification_uint8.c on the graph's quantised output tensor
 * where it lies in HBM (after tb200_graph_run / tb200_graph_launch): k (score, id) pairs per image come back instead of every class.
 *   classes  The classes of image i are its E = C*H*W elements in NCHW order, id = c*H*W + h*W + w: what the examples read from
 *            get_tensor_buffer at batch 1.  The usual tensor is [N, classes, 1, 1].
 *   score    int8: (float)q * scale (tm_classification_int8.c:163-164; the zero point is not used).  uint8: ((float)q -
 *            (float)zero_point) * scale (tm_classification_uint8.c:169-170).  Float arithmetic, one rounding per operation.  Scale and
 *            zero point are the output tensor's own.
 *   order    print_topk (examples/common/tengine_operations.c:1021-1038) fills an array with (id, score) in buffer order, sorts all of
 *            it with sort_cls_score(array, 0, E - 1) (:991-1019) and prints entries 0..k-1; out holds exactly those entries.  The sort
 *            is an unstable quicksort and a quantised output is mostly equal scores, so which of several equal classes is reported, and
 *            in which order, is the example's choice and is reproduced.  Every comparison is the example's own operator on the
 *            dequantised floats, so the result is the example's for any finite scale: zero, negative, overflowing to infinity.  (A NaN
 *            score fails both comparisons of sort_cls_score and its loop never ends, so a scale that is not finite is refused.)
 * tb200_class_score carries the two fields of cls_score (tengine_operations.h:57-61), score first. */
#define TB200_TOPK_MAX 64            /* largest k */
#define TB200_TOPK_MAX_CLASSES 32768 /* largest E: an image's scores and ids are staged in shared memory (6 bytes per class of the
                                        227 KB a thread block may use on sm_90) */
typedef struct tb200_class_score
{
    float score;
    int32_t id;
} tb200_class_score;
/* out[image * k + r], r < k: entry r of the example's sorted array for that image of graph output `output_index`; HOST memory for
 * N * k entries.  Synchronous, like tb200_graph_yolo_detect; on a multi-GPU context every shard writes its own images' rows.
 * Checked before any work, `out` left untouched: TB200_ERR_INVALID for a null pointer, an output index out of range, k < 1, k > E (the
 * example asserts total_num >= topk), k > TB200_TOPK_MAX, an output that is not int8 / uint8, a scale that is not finite; TB200_ERR_UNSUPPORTED for
 * E > TB200_TOPK_MAX_CLASSES. */
TB200_API int tb200_graph_topk(tb200_graph* g, int output_index, int k, tb200_class_score* out);

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
/* tb200_graph_topk's kernel on a DEVICE tensor in the device layout ([n][h][w][tb200k_cpad(c)] bytes; pad lanes are not read):
 * out is a DEVICE pointer to n * k entries; asynchronous on `stream`.  Same semantics and the same checks. */
TB200_API int tb200k_class_topk(const void* in, int n, int c, int h, int w, int is_uint8, float scale, int32_t zero_point, int k,
                                tb200_class_score* out, void* stream);

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
