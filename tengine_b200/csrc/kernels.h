// kernels.h -- internal launcher interface between the graph executor (engine.cu) and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace tb200 {

struct ConvShape
{
    int n, h, w, c, cp;  // input: logical channels c, padded pitch cp
    int cg, cgp;         // channels per group (logical) and per-group pitch of the weight layout
    int oh, ow, oc, ocp; // output
    int kh, kw, sh, sw, ph0, pw0, dh, dw, group;
};

struct PoolShape
{
    int n, h, w, c, cp, oh, ow;
    int kh, kw, sh, sw, ph0, pw0;
    int method, caffe_flavor;
    float in_scale, out_scale;
    int in_zero, out_zero;
    const uint8_t* lut; // a (leaky) ReLU node folded in front of a same-scale max pooling: applied to the window's maximum (engine.cu)
    int c_real;         // uint8 with lut: channels >= c_real are pad lanes and stay 0
};

struct PointwiseParams
{
    int mode; // 0 relu / leaky relu, 1 sum, 2 prod
    int c, cp;
    float scale0, scale1, out_scale;
    int zero0, zero1, out_zero;
    float negative_slope;
    int post_relu;        // a same-scale ReLU node folded into this eltwise: bytes = max(bytes, zero point)
    uint32_t post_floor4; // uint8: the output zero point replicated x4
};

// One input of a concat: its c channels (pitch cp_in) of npix pixels go to output channels [c_off, c_off + c_write) (pitch cp_out);
// the last input's c_write reaches cp_out, so it also clears the output's pad lanes.
struct ConcatPart
{
    long long npix;
    int c, c_write, cp_in, cp_out, c_off;
    float s_in, s_out; // requantisation from the input's quantisation to the output's
    int z_in, z_out;
    const uint8_t* lut; // the same requantisation as a 256-entry byte table (launch_concat_lut); nullptr = equal quantisation
};

struct SoftmaxShape
{
    long long npix;
    int c, cp;
    float s_in, s_out;
    int z_in, z_out;
};

cudaError_t launch_conv_direct(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st);
cudaError_t launch_conv_dw(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st);
cudaError_t launch_conv_stem(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st);
cudaError_t launch_pool(const void* in, void* out, const PoolShape& p, bool u8, cudaStream_t st);
cudaError_t launch_pointwise(const void* a, const void* b, void* out, long long bytes, const PointwiseParams& p, bool u8, cudaStream_t st);
cudaError_t launch_concat_part(const void* in, void* out, const ConcatPart& p, bool u8, cudaStream_t st);
// unary byte ops (sigmoid, hardswish) as a 256-entry table built at prerun; pad lanes (channel >= c) stay 0
cudaError_t launch_byte_lut(const void* in, void* out, const uint8_t* lut, long long bytes, int c, int cp, cudaStream_t st);
// softmax over the channel axis (softmax_kernel_ref_int8.c / _uint8.c), one thread per pixel
cudaError_t launch_softmax(const void* in, void* out, const SoftmaxShape& p, bool u8, cudaStream_t st);
cudaError_t launch_concat_lut(const void* in, void* out, const ConcatPart& p, cudaStream_t st);
cudaError_t launch_upsample(const void* in, void* out, int n, int h, int w, int cp, int scale, cudaStream_t st);
cudaError_t launch_nchw_to_nhwc(const void* in, void* out, int n, int c, int h, int w, cudaStream_t st);
cudaError_t launch_nhwc_to_nchw(const void* in, void* out, int n, int c, int h, int w, cudaStream_t st);

// ---- TMA-staged depthwise 3x3 (dw_tma.cu) ---------------------------------------------------------------
struct DwPlan
{
    alignas(64) unsigned char tmap_in[128]; // CUtensorMap over the NHWC input (C, W, H, N)
    int valid;
    int tw, gpr, rows_per_cta, tile_cols, tile_rows, smem_bytes;
};
int dw_plan_create(DwPlan* plan, const void* in, const ConvShape& s, const EpiParams& e);
cudaError_t launch_conv_dw_tma(const DwPlan& plan, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st);

// ---- fp32 members of the path (conv_fp32.cu): Winograd F(4x4,3x3) and depthwise 3x3 on NCHW fp32 ---------------
size_t wino43_workspace_bytes(int n, int c, int oc, int oh, int ow);
cudaError_t launch_conv_winograd43_f32(const float* in, const float* w, const float* bias, float* out, int n, int c, int h, int wd, int oc, int oh, int ow, int ph,
                                       int pw, int activation, float* ws, cudaStream_t st);
cudaError_t launch_conv_dw3x3_f32(const float* in, const float* w, const float* bias, float* out, int n, int c, int h, int wd, int oh, int ow, int stride, int ph,
                                  int pw, int activation, cudaStream_t st);

// ---- detection post-processing (yolo_detect.cu) ----------------------------------------------------------------
struct YoloCand
{
    float x, y, w, h, prob;
    int label;
    unsigned key; // position in the reference's proposal list (head order, then h, w, anchor)
};
struct YoloDet
{
    float x, y, w, h, prob;
    int label;
};
// box formula of the region decode: examples/tm_yolov3_tiny_uint8.cpp (V3) or examples/tm_yolov5s.cpp (V5)
enum class YoloBox
{
    V3,
    V5
};
cudaError_t launch_yolo_decode(YoloBox f, const void* tensor, int cp, int h, int w, int n_img, int classes, const float* sig, const double* ex, float stride,
                               const float* anchors6, float thr, YoloCand* cand, int* count, int max_cand, unsigned key_base, bool is_u8, cudaStream_t st);
cudaError_t launch_yolo_nms(const YoloCand* cand, const int* count, int n_img, int max_cand, float nms_thr, YoloCand* sorted, YoloDet* out, int max_out,
                            int* out_count, cudaStream_t st);

// ---- classification post-processing (classify_topk.cu) ---------------------------------------------------------
struct ClassScore // tb200_class_score
{
    float score;
    int32_t id;
};
constexpr int CLASS_TOPK_MAX_K = 64;          // TB200_TOPK_MAX
constexpr int CLASS_TOPK_MAX_CLASSES = 32768; // TB200_TOPK_MAX_CLASSES: one image's scores and ids are staged in shared memory
// in: [n][h][w][cpad(c)] int8 (u8 = false) or uint8 bytes; out[image * k + r]: entry r of the array the classification examples' print_topk
// holds after sorting the image's c*h*w dequantised scores (ids in NCHW order)
cudaError_t launch_class_topk(const void* in, int n, int c, int h, int w, bool u8, float scale, int zero_point, int k, ClassScore* out, cudaStream_t st);

// ---- input preprocessing (image_pre.cu, detect_pre.cu) ------------------------------------------------------------
// One image of a staged batch: h rows of w pixels of c interleaved bytes (c = 3 or 4) at `offset` of the shard's staging buffer; for
// detection also where its resized copy lies in the laid-out image (tb200_detect_geometry; unused by image_pre)
struct ImageDesc
{
    uint64_t offset;
    int32_t w, h, c;
    int32_t resize_w, resize_h, left, top;
};
// out: [n][3][H][W] int8 (u8 = false) or uint8 bytes, as examples/tm_classification_{int8,uint8}.c would fill the input tensor
cudaError_t launch_image_pre(const uint8_t* pixels, const ImageDesc* images, int n, uint8_t* out, int H, int W, const float mean[3], const float scale[3],
                             float s_in, int zp, bool u8, cudaStream_t st);
// out: [n][3][H][W], or with focus [n][12][H/2][W/2], int8 or uint8 bytes as the YOLO examples fill the input tensor (tengine_b200.h)
cudaError_t launch_detect_pre(const uint8_t* pixels, const ImageDesc* images, int n, uint8_t* out, int H, int W, bool focus, const float mean[3],
                              const float scale[3], float s_in, int zp, bool u8, cudaStream_t st);

// ---- small-Cin convolutions with a TMA-staged input window (conv_window.cu) -----------------------------------
struct WindowPlan
{
    alignas(64) unsigned char tmap_in[128]; // CUtensorMap over the input: NCHW (W, H, C, N) or NHWC (Cp, W, H, N)
    int valid;
    int layout; // 0 NCHW 3x3, 1 NCHW 7x7, 2 NHWC 16 B/pixel 3x3, 3 NHWC 32 B/pixel 3x3
    int box_w, box_h, xoff, in_bytes, ks, smem_bytes;
};
int window_plan_create(WindowPlan* plan, const void* in, const ConvShape& s, int nhwc); // < 0: not applicable
bool window_nhwc_fits(int cp, int ocp, int stride); // a 3x3 conv over an NHWC input of cp bytes per pixel fits the kernel's shared memory
cudaError_t launch_conv_window(const WindowPlan& plan, const void* w, void* out, const ConvShape& s, const EpiParams& e, int num_sms, cudaStream_t st);
// the same layers without a window plan: every thread gathers its pixel's taps from global memory (NCHW stems, 16-channel NHWC inputs)
cudaError_t launch_conv_gather_tc(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, int nhwc16, int num_sms,
                                  cudaStream_t st);

// ---- wgmma GEMM (gemm_tcgen05.cu) --------------------------------------------------------------------
// out[M][ldo] (bytes) = requant( A[M][K] (row pitch lda bytes) . B[OCp][K]^T )
struct GemmPlan
{
    alignas(64) unsigned char tmap_a[128]; // CUtensorMap
    alignas(64) unsigned char tmap_b[128];
    alignas(64) unsigned char tmap_out[128];      // (C, rows, outer) over the output, box = 16*cs x 32 rows
    alignas(64) unsigned char tmap_out_tail[128]; // same with rows_valid % 32 rows (last quarter of a short conv patch)
    long long m;
    int k;       // padded K (multiple of 16)
    int oc, ocp; // logical / padded output channels
    int ldo;     // output row pitch in bytes
    int block_n, block_k, stages, k_blocks, n_tiles;
    int mt; // m-tiles per accumulator stage
    // conv mode (implicit GEMM over a 4-D tensor map)
    int conv, cblocks, kw_n, pad_h, pad_w, cstride, cp, bw, bh, bn, tiles_w, tiles_h, oh, ow, nimg;
    unsigned a_tx_bytes;
    int u8, taps, in_h, in_w; // uint8: unsigned A operand
    int b_signed, cplane;     // uint8: B holds w - 128 as int8, the epilogue adds (128 - zw) * sum(x) (gemm_tcgen05.cu)
    long long m_tiles;
    int swizzle; // 32 / 64 / 128
    int cs, ngroups, rows_valid, out_mode; // epilogue store groups, see gemm_tcgen05.cu plan_epilogue
    int b_res;                             // weights of the N tile resident in smem (ring carries A only)
    void* out;
    // deferred rare path (gemm_tcgen05.cu fixq_*): per-context scratch of fixq_cap 16-byte entries per CTA; null = fix inline
    void* fixq;
    int fixq_cap;
};
// Build TMA descriptors for fixed device pointers. Returns 0 or a negative TB200_ERR_*.
// ordinal of the calling thread's current CUDA device (launchers keep per-device state: cudaFuncSetAttribute is per device)
static inline int current_device()
{
    int d = 0;
    cudaGetDevice(&d);
    return d;
}
int gemm_block_n(int ocp); // channels of one N tile = rows of one packed B tile
// TB200_DEBUG_LAUNCH (read once per process): the templated launchers print one stderr line per launch naming the instantiation,
// "tengine_b200: launch <kernel><ARG=value,...>"; diagnostic only, changes nothing else
bool debug_launch();
int gemm_plan_create(GemmPlan* plan, const void* a, long long lda, const void* b, void* out, long long m, int k, int oc, int ocp, int ldo, int u8);
int gemm_plan_create_conv(GemmPlan* plan, const void* in, const void* w, void* out, const ConvShape& s, int u8);
cudaError_t launch_gemm_i8(const GemmPlan& plan, const EpiParams& e, const int32_t* btab, int num_sms, cudaStream_t st);
// measured peak of wgmma m64n128k32 s8 (two warpgroups per SM) on this GPU, in TOP/s: the tensor roofline's denominator
cudaError_t probe_int8_mma_peak(int num_sms, double* tops, cudaStream_t st);

} // namespace tb200
