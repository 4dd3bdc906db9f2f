// kernels.h -- internal launcher interface between the graph executor (engine.cu) and the kernels.
#pragma once
#include <cuda.h> // CUtensorMap
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
cudaError_t launch_concat_lut(const void* in, void* out, const ConcatPart& p, bool u8, cudaStream_t st);
cudaError_t launch_upsample(const void* in, void* out, int n, int h, int w, int cp, int scale, cudaStream_t st);
cudaError_t launch_nchw_to_nhwc(const void* in, void* out, int n, int c, int h, int w, cudaStream_t st);
cudaError_t launch_nhwc_to_nchw(const void* in, void* out, int n, int c, int h, int w, cudaStream_t st);

// ---- TMA-staged depthwise 3x3 (dw_tma.cu) ---------------------------------------------------------------
struct DwPlan
{
    CUtensorMap tmap_in; // over the NHWC input (C, W, H, N)
    const uint8_t* w;
    uint8_t* out;
    ConvShape s;
    EpiParams e;
    int gpr, rows_per_cta, tile_cols, tile_rows, smem_bytes;
    dim3 grid;
    int mode; // the epilogue the kernels take at run time (epi_mode), for TB200_DEBUG_LAUNCH
};
// 0, or < 0 when this layer must use the generic depthwise kernel
int dw_plan_create(DwPlan* plan, const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e);
cudaError_t launch_conv_dw_tma(const DwPlan& plan, cudaStream_t st);

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
struct WindowArgs
{
    const uint8_t* w; // [OCp][ks*32]; NCHW: k = (c*KH + kh)*KW + kw ; NHWC: k = (kh*3 + kw)*CB + c ; zero padded
    uint8_t* out;     // NHWC, OCp bytes per pixel
    int n, c, h, w_in, oh, ow, ocp, oc, stride, ph, pw;
    unsigned ntiles;
    int tiles_w, tiles_h;
    uint32_t tw_magic, th_magic; // floor(2^32 / d) + 1: q = umulhi(x, magic) is x / d for the tile counts that occur (checked by the planner)
    int box_w, box_h, xoff, in_bytes, ks;
    uint32_t fill; // uint8: the input zero point replicated x4 (0 for int8: the TMA zero fill already is the padding)
};
struct WindowPlan
{
    CUtensorMap tmap_in; // over the input: NCHW (W, H, C, N) or NHWC (Cp, W, H, N)
    WindowArgs a;
    EpiParams e;
    int smem_bytes;
    int num_sms; // the grid is as many CTAs as the SMs hold at once, at most one per tile
    // the instantiation conv_window_tc_kernel<MODE, U8 = e.is_uint8, LAYOUT>
    int mode;
    int layout; // 0 NCHW 3x3, 1 NCHW 7x7, 2 NHWC 16 B/pixel 3x3, 3 NHWC 32 B/pixel 3x3
};
// 0; 1 when the window kernel does not apply (the gather kernel takes the layer); < 0 (TB200_ERR_UNSUPPORTED) when it applies but
// the layer has more output pixels or tiles than its 32-bit indices address
int window_plan_create(WindowPlan* plan, const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, int nhwc, int num_sms);
bool window_nhwc_fits(int cp, int ocp, int stride); // a 3x3 conv over an NHWC input of cp bytes per pixel fits the kernel's shared memory
cudaError_t launch_conv_window(const WindowPlan& plan, cudaStream_t st);

// the same layers without a window plan: every thread gathers its pixel's taps from global memory (NCHW stems, 16-channel NHWC inputs)
struct GatherArgs
{
    const uint8_t* in;
    const uint8_t* w; // [OCp][ks*32]; NCHW: k = (c*3 + kh)*3 + kw ; NHWC16: k = (kh*3 + kw)*16 + c ; zero padded
    uint8_t* out;
    int n, c, h, w_in, oh, ow, ocp, oc, stride, ph, pw;
    unsigned npix, ntiles;
    int ks, nhwc16;
    uint32_t fill; // byte for taps outside the image, replicated x4 (uint8: the input zero point; int8: 0)
    uint32_t fill16[4]; // NHWC16: the same for a whole 16-channel tap; pad channels (c >= C) stay 0 like in the tensor itself
};
struct GatherPlan
{
    GatherArgs a;
    EpiParams e;
    int smem_bytes;
    unsigned grid;
    int mode, khw; // the instantiation conv_gather_tc_kernel<MODE, U8 = e.is_uint8, KHW>
};
void gather_plan_create(GatherPlan* plan, const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, int nhwc16, int num_sms);
cudaError_t launch_conv_gather_tc(const GatherPlan& plan, cudaStream_t st);

// ---- wgmma GEMM (gemm_tcgen05.cu) --------------------------------------------------------------------
// out[M][ldo] (bytes) = requant( A[M][K] (row pitch lda bytes) . B[OCp][K]^T )
struct GemmArgs
{
    int m_tiles, num_super; // 32-bit on purpose: 64-bit divisions in the tile decode cost ~100 instructions each
    int k_blocks, n_tiles, block_n, block_k, stages, swizzle;
    int mt;     // m-tiles (128 rows each) per accumulator stage
    uint32_t bw_rcp, bh_rcp; // ceil(65536/d): q = (x * rcp) >> 16 is exact for x < 4096, d <= 256
    int oc, ocp;
    // conv mode (implicit GEMM): an m-tile is a bw x bh x bn patch of output pixels, a k-block is (tap, channel block)
    int conv, cblocks, kw_n, pad_h, pad_w, cstride, cp;
    int bw, bh, bn, tiles_w, tiles_h, oh, ow, nimg;
    uint32_t a_tx_bytes; // bytes one A load delivers (block_k * rows of the patch)
    // uint8 (unsigned A): B holds w - 128 as int8 (plain w when zw == 0), so the accumulator is sum x*(w - 128); what is left of
    // sum x*(w - zw) is cplane * sum(x) with cplane = 128 - zw, and the epilogue adds cplane * sum(x) inside the IADD3 that also
    // adds the per-channel constant.
    // sum(x) comes from two extra warps that add up the rows of every A tile in shared memory (cplane != 0 only).
    int u8, taps, in_h, in_w, b_signed, cplane;
    // epilogue / stores
    int cs, ngroups; // 16-column chunks per store group (1 or 2) and groups per m-tile
    int rows_valid;  // rows of an m-tile that are output pixels (128, or bw*bh*bn of a smaller conv patch)
    int out_mode;    // coordinates of the output map: 0 (c, row, 0)  1 (c, pixel in image, image)  2 (c, x, image row)
    int par_all;     // the constants of every channel are resident (loaded once); else reloaded per N tile
    int b_res;       // the N tile's weights (all k-blocks) are loaded once and stay in smem; the ring carries A only
    // deferred rare path: a guarded element is queued {m-tile, row, channel, accumulator} and recomputed literally by all threads of the
    // CTA after its last tile, instead of holding up its epilogue warp (and with it the accumulator stage); null = inline
    uint4* fixq;
    int fixq_cap; // entries per CTA
    uint8_t* out_base;
    int ldo, m_rows; // output row pitch in bytes; rows of the flat GEMM
    const int32_t* btab; // uint8 convolutions: [border pattern][OCp] summed corrections of the taps a border pixel misses (engine.cu)
    unsigned long long* trace; // debug (TB200_GEMM_TRACE): event timeline of CTA 0, see gemm_trace_report
};
struct GemmPlan
{
    CUtensorMap tmap_a, tmap_b;
    CUtensorMap tmap_out;      // (C, rows, outer) over the output, box = 16*cs x 32 rows
    CUtensorMap tmap_out_tail; // same with rows_valid % 32 rows (last quarter of a short conv patch)
    GemmArgs g;
    EpiParams e;
    int grid, smem_bytes;
    int mode, border; // with g.u8 and g.cs: the instantiation gemm_i8_tcgen05_kernel<U8, MODE, CS, BORDER>
};
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
// Build the TMA descriptors for fixed device pointers and every launch parameter.  Returns 0 or a negative TB200_ERR_*.
// u8: 0 for int8, 1 + the weight zero point for uint8.  fixq: the deferred rare path's scratch of fixq_cap 16-byte entries per CTA
// (gemm_tcgen05.cu fixq_*), null = fix inline.  btab: see GemmArgs.
int gemm_plan_create(GemmPlan* plan, const void* a, long long lda, const void* b, void* out, long long m, int k, int oc, int ocp, int ldo, int u8,
                     const EpiParams& e, const int32_t* btab, void* fixq, int fixq_cap, int num_sms);
int gemm_plan_create_conv(GemmPlan* plan, const void* in, const void* w, void* out, const ConvShape& s, int u8, const EpiParams& e,
                          const int32_t* btab, void* fixq, int fixq_cap, int num_sms);
cudaError_t launch_gemm_i8(const GemmPlan& plan, cudaStream_t st);
// measured peak of wgmma m64n128k32 s8 (two warpgroups per SM) on this GPU, in TOP/s: the tensor roofline's denominator
cudaError_t probe_int8_mma_peak(int num_sms, double* tops, cudaStream_t st);

} // namespace tb200
