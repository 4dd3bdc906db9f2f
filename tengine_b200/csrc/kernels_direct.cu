// kernels_direct.cu -- CUDA-core (dp4a) kernels of the H100 backend: generic direct convolution, depthwise,
// NCHW stem, and the HBM-bound glue ops (pool / relu / eltwise / concat / upsample / layout).
//
// Device layout: activations NHWC, channels padded to a multiple of 16 (pad lanes hold 0), 1 byte/element.
// These kernels are the general path (any kernel/stride/pad/dilation/group) and the on-device cross-check
// for the tensor-core GEMM path; the dense 1x1 / FC contractions run in gemm_tcgen05.cu.
#include "common.cuh"
#include "kernels.h"

#include <cmath>
#include <cstdlib>

namespace tb200 {

// ------------------------------------------------------------------------------------------------------
// Generic direct convolution.  Thread = one output pixel x OCT consecutive output channels.
// Weights [OCp][KH][KW][CGp] (CGp = padded channels per group, multiple of 16 when group == 1,
// multiple of 4 otherwise).  Takes the role of ref_conv_int8 / ref_conv_uint8 (conv_kernel_ref_*.c) and of
// im2col+sgemm for shapes the tensor-core path does not cover.
// ------------------------------------------------------------------------------------------------------
template <bool U8, int OCT>
__global__ void __launch_bounds__(128) conv_direct_kernel(const uint8_t* __restrict__ in, const uint8_t* __restrict__ wgt,
                                                          uint8_t* __restrict__ out, const ConvShape s, const __grid_constant__ EpiParams e)
{
    // 32-bit index math (the launcher guarantees n*oh*ow < 2^31): 64-bit divisions cost ~100 instructions each
    const unsigned pix = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned npix = (unsigned)s.n * s.oh * s.ow;
    if (pix >= npix) return;
    const int oc0 = blockIdx.y * OCT;
    const unsigned prow = pix / (unsigned)s.ow;
    const int ow = (int)(pix - prow * s.ow);
    const int n = (int)(prow / (unsigned)s.oh);
    const int oh = (int)(prow - (unsigned)n * s.oh);
    const int og = s.oc / s.group;              // logical out channels per group
    const int g = (oc0 < s.oc) ? oc0 / og : 0;  // OCT divides og or group == 1 (host guarantees)
    const int cin0 = g * s.cg;                  // first logical input channel of the group
    const int words = s.cgp / 4;

    int acc[OCT];
    int sw_sum[OCT]; // uint8: sum of weights over in-bounds taps
#pragma unroll
    for (int j = 0; j < OCT; j++) acc[j] = 0, sw_sum[j] = 0;
    int sx_sum = 0, taps = 0;

    for (int kh = 0; kh < s.kh; kh++)
    {
        const int iy = oh * s.sh - s.ph0 + kh * s.dh;
        if (iy < 0 || iy >= s.h) continue;
        for (int kw = 0; kw < s.kw; kw++)
        {
            const int ix = ow * s.sw - s.pw0 + kw * s.dw;
            if (ix < 0 || ix >= s.w) continue;
            taps++;
            const int* xp = reinterpret_cast<const int*>(in + (((size_t)n * s.h + iy) * s.w + ix) * s.cp + cin0);
            const int* wp = reinterpret_cast<const int*>(wgt + ((size_t)oc0 * s.kh * s.kw + (size_t)kh * s.kw + kw) * s.cgp);
            const size_t wstride = (size_t)s.kh * s.kw * words; // ints between consecutive output channels
            for (int c = 0; c < words; c++)
            {
                const int xv = __ldg(xp + c);
                if (U8) sx_sum = (int)dp4a_u8((unsigned)xv, 0x01010101u, (unsigned)sx_sum);
#pragma unroll
                for (int j = 0; j < OCT; j++)
                {
                    const int wv = __ldg(wp + j * wstride + c);
                    if (U8)
                    {
                        acc[j] = (int)dp4a_u8((unsigned)xv, (unsigned)wv, (unsigned)acc[j]);
                        sw_sum[j] = (int)dp4a_u8((unsigned)wv, 0x01010101u, (unsigned)sw_sum[j]);
                    }
                    else
                        acc[j] = dp4a_s8(xv, wv, acc[j]);
                }
            }
        }
    }

    uint8_t* op = out + (size_t)pix * s.ocp + oc0;
#pragma unroll
    for (int j = 0; j < OCT; j += 4)
    {
        int32_t a4[4];
#pragma unroll
        for (int t = 0; t < 4; t++)
        {
            a4[t] = acc[j + t];
            if (U8) // sum (x-zx)(w-zw) = Sxw - zw*Sx - zx*Sw + cnt*zx*zw   (cnt counts REAL channels only)
                a4[t] = a4[t] - e.w_zero * sx_sum - e.in_zero * sw_sum[j + t] + taps * s.cg * e.in_zero * e.w_zero;
        }
        *reinterpret_cast<unsigned*>(op + j) = requant_word<U8>(a4, oc0 + j, s.oc, e);
    }
}

// ------------------------------------------------------------------------------------------------------
// Depthwise convolution (group == C == OC), any kernel size.  Thread = one output pixel x 4 channels.
// Weights [KH][KW][Cp].  Takes the role of convdw3x3s{1,2}_int8_sse (conv_dw_hcl_x86.c:97-445) and of
// ref_conv_* for the depthwise cases the reference sends to conv_ref (batch > 1, uint8).
// ------------------------------------------------------------------------------------------------------
template <bool U8>
__global__ void __launch_bounds__(256) conv_dw_kernel(const uint8_t* __restrict__ in, const uint8_t* __restrict__ wgt,
                                                      uint8_t* __restrict__ out, const ConvShape s, const __grid_constant__ EpiParams e)
{
    const int cw = s.cp / 4; // channel words per pixel
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; // launchers guarantee totals < 2^31
    const unsigned total = (unsigned)(s.n * s.oh * s.ow * cw);
    if (idx >= total) return;
    const unsigned pix = idx / (unsigned)cw;
    const int c4 = (int)(idx - pix * cw);
    const unsigned prow = pix / (unsigned)s.ow;
    const int ow = (int)(pix - prow * s.ow);
    const int n = (int)(prow / (unsigned)s.oh);
    const int oh = (int)(prow - (unsigned)n * s.oh);

    int acc[4] = {0, 0, 0, 0};
    for (int kh = 0; kh < s.kh; kh++)
    {
        const int iy = oh * s.sh - s.ph0 + kh * s.dh;
        if (iy < 0 || iy >= s.h) continue;
        for (int kw = 0; kw < s.kw; kw++)
        {
            const int ix = ow * s.sw - s.pw0 + kw * s.dw;
            if (ix < 0 || ix >= s.w) continue;
            const unsigned xv = __ldg(reinterpret_cast<const unsigned*>(in + (((size_t)n * s.h + iy) * s.w + ix) * s.cp) + c4);
            const unsigned wv = __ldg(reinterpret_cast<const unsigned*>(wgt + ((size_t)kh * s.kw + kw) * s.cp) + c4);
#pragma unroll
            for (int t = 0; t < 4; t++)
            {
                int xb, wb;
                if (U8)
                {
                    xb = (int)((xv >> (8 * t)) & 0xff) - e.in_zero;
                    wb = (int)((wv >> (8 * t)) & 0xff) - e.w_zero;
                }
                else
                {
                    xb = (int)(int8_t)(xv >> (8 * t));
                    wb = (int)(int8_t)(wv >> (8 * t));
                }
                acc[t] += xb * wb;
            }
        }
    }
    reinterpret_cast<unsigned*>(out + (size_t)pix * s.ocp)[c4] = requant_word<U8>(acc, c4 * 4, s.oc, e);
}

// ------------------------------------------------------------------------------------------------------
// Depthwise 3x3, int8, stride 1 or 2, dilation 1: the MobileNet hot depthwise path.
// Thread = 4 channels (one 32-bit word) x TW consecutive output pixels of one output row; the 3 x ((TW-1)*S+3) input
// window is loaded once and slides through registers, so each input word is fetched once per thread instead of up to
// 9 times.  A MAC is ONE dp4a: the weight word is split into four one-hot-byte words (w & 0xff<<8j), so
// dp4a(x_word, w_j, acc) = x[byte j] * w[byte j] + acc with no unpacking of the activations.
// Takes the role of convdw3x3s1_int8_sse / convdw3x3s2_int8_sse (conv_dw_hcl_x86.c:97-445).
// ------------------------------------------------------------------------------------------------------
template <int TW, int S>
__global__ void __launch_bounds__(128) conv_dw3x3_i8_kernel(const uint8_t* __restrict__ in, const uint8_t* __restrict__ wgt,
                                                            uint8_t* __restrict__ out, const ConvShape s, const __grid_constant__ EpiParams e)
{
    const int cw = s.cp / 4;
    const int gpr = (s.ow + TW - 1) / TW; // pixel groups per output row
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; // launchers guarantee totals < 2^31
    const unsigned total = (unsigned)(s.n * s.oh * gpr * cw);
    if (idx >= total) return;
    unsigned r = idx / (unsigned)cw;
    const int c4 = (int)(idx - r * cw);
    const unsigned r2 = r / (unsigned)gpr;
    const int pg = (int)(r - r2 * gpr);
    const int n = (int)(r2 / (unsigned)s.oh);
    const int oh = (int)(r2 - (unsigned)n * s.oh);
    const int ow0 = pg * TW;

    int wj[9][4];
#pragma unroll
    for (int t = 0; t < 9; t++)
    {
        const unsigned wv = __ldg(reinterpret_cast<const unsigned*>(wgt + (size_t)t * s.cp) + c4);
#pragma unroll
        for (int j = 0; j < 4; j++) wj[t][j] = (int)(wv & (0xffu << (8 * j)));
    }
    int acc[TW][4];
#pragma unroll
    for (int t = 0; t < TW; t++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[t][j] = 0;

    constexpr int COLS = (TW - 1) * S + 3;
    const int ix0 = ow0 * S - s.pw0;
#pragma unroll
    for (int kh = 0; kh < 3; kh++)
    {
        const int iy = oh * S - s.ph0 + kh;
        if (iy < 0 || iy >= s.h) continue;
        const unsigned* rowp = reinterpret_cast<const unsigned*>(in + ((size_t)n * s.h + iy) * s.w * s.cp) + c4;
        int xv[COLS];
#pragma unroll
        for (int col = 0; col < COLS; col++)
        {
            const int ix = ix0 + col;
            xv[col] = (ix >= 0 && ix < s.w) ? (int)__ldg(rowp + (size_t)ix * cw) : 0;
        }
#pragma unroll
        for (int t = 0; t < TW; t++)
#pragma unroll
            for (int kw = 0; kw < 3; kw++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[t][j] = dp4a_s8(xv[t * S + kw], wj[kh * 3 + kw][j], acc[t][j]);
    }

    uint8_t* orow = out + (((size_t)n * s.oh + oh) * s.ow + ow0) * s.ocp;
#pragma unroll
    for (int t = 0; t < TW; t++)
        if (ow0 + t < s.ow) reinterpret_cast<unsigned*>(orow + (size_t)t * s.ocp)[c4] = requant_word<false>(acc[t], c4 * 4, s.oc, e);
}

// ------------------------------------------------------------------------------------------------------
// Stem: NCHW input with C <= 4 (the network input as the application hands it over) -> NHWC output.
// Thread = one output pixel x OCT output channels.  Weights [OCp][KH][KW][4].
// Fuses the NCHW->NHWC conversion of the graph input into the first convolution.
// ------------------------------------------------------------------------------------------------------
template <bool U8, int OCT>
__global__ void __launch_bounds__(128, (OCT == 32 && !U8) ? 4 : 2)
    conv_stem_kernel(const uint8_t* __restrict__ in, const uint8_t* __restrict__ wgt, uint8_t* __restrict__ out, const ConvShape s,
                     const __grid_constant__ EpiParams e)
{
    // weights of this CTA's OCT output channels, transposed to [tap][oc] so that one LDS.128 feeds four dp4a
    extern __shared__ __align__(16) int stem_w[];
    const int oc0 = blockIdx.y * OCT;
    const int taps_total = s.kh * s.kw;
    for (int i = threadIdx.x; i < taps_total * OCT; i += blockDim.x)
    {
        const int t = i / OCT, j = i - t * OCT;
        stem_w[i] = __ldg(reinterpret_cast<const int*>(wgt) + (size_t)(oc0 + j) * taps_total + t);
    }
    __syncthreads();
    const unsigned pix = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned npix = (unsigned)s.n * s.oh * s.ow;
    if (pix >= npix) return;
    const unsigned prow = pix / (unsigned)s.ow;
    const int ow = (int)(pix - prow * s.ow);
    const int n = (int)(prow / (unsigned)s.oh);
    const int oh = (int)(prow - (unsigned)n * s.oh);
    const size_t plane = (size_t)s.h * s.w;
    const uint8_t* img = in + (size_t)n * s.c * plane;

    int acc[OCT];
    int sw_sum[U8 ? OCT : 1];
#pragma unroll
    for (int j = 0; j < OCT; j++) acc[j] = 0;
    if (U8)
    {
#pragma unroll
        for (int j = 0; j < (U8 ? OCT : 1); j++) sw_sum[j] = 0;
    }
    int sx_sum = 0, taps = 0;

#pragma unroll 1
    for (int kh = 0; kh < s.kh; kh++)
    {
        const int iy = oh * s.sh - s.ph0 + kh * s.dh;
        if (iy < 0 || iy >= s.h) continue;
#pragma unroll 1
        for (int kw = 0; kw < s.kw; kw++)
        {
            const int ix = ow * s.sw - s.pw0 + kw * s.dw;
            if (ix < 0 || ix >= s.w) continue;
            taps++;
            const uint8_t* px = img + (size_t)iy * s.w + ix;
            unsigned xv = __ldg(px);
            if (s.c > 1) xv |= (unsigned)__ldg(px + plane) << 8;
            if (s.c > 2) xv |= (unsigned)__ldg(px + 2 * plane) << 16;
            if (s.c > 3) xv |= (unsigned)__ldg(px + 3 * plane) << 24;
            if (U8) sx_sum = (int)dp4a_u8(xv, 0x01010101u, (unsigned)sx_sum);
            const int4* wrow = reinterpret_cast<const int4*>(stem_w + (kh * s.kw + kw) * OCT);
#pragma unroll
            for (int j = 0; j < OCT; j += 4)
            {
                const int4 wv = wrow[j >> 2];
                const int w4[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                for (int t = 0; t < 4; t++)
                {
                    if (U8)
                    {
                        acc[j + t] = (int)dp4a_u8(xv, (unsigned)w4[t], (unsigned)acc[j + t]);
                        sw_sum[j + t] = (int)dp4a_u8((unsigned)w4[t], 0x01010101u, (unsigned)sw_sum[j + t]);
                    }
                    else
                        acc[j + t] = dp4a_s8((int)xv, w4[t], acc[j + t]);
                }
            }
        }
    }
    uint8_t* op = out + (size_t)pix * s.ocp + oc0;
#pragma unroll
    for (int j = 0; j < OCT; j += 4)
    {
        int32_t a4[4];
#pragma unroll
        for (int t = 0; t < 4; t++)
        {
            a4[t] = acc[j + t];
            if (U8) a4[t] = a4[t] - e.w_zero * sx_sum - e.in_zero * sw_sum[j + t] + taps * s.c * e.in_zero * e.w_zero;
        }
        *reinterpret_cast<unsigned*>(op + j) = requant_word<U8>(a4, oc0 + j, s.oc, e);
    }
}

// ------------------------------------------------------------------------------------------------------
// Glue ops.  All follow the reference's dequant -> fp32 op -> requant arithmetic literally.
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int clamp_i8(int q) { return (q > 127 ? 127 : (q < -127 ? -127 : q)) & 0xff; }
__device__ __forceinline__ int clamp_u8(int q) { return q > 255 ? 255 : (q < 0 ? 0 : q); }

// A ReLU node whose output has its input's quantisation, folded into the eltwise that feeds it (engine.cu planner): on the
// requantised bytes it is max(byte, zero point) / max(byte, 0) -- see relu_same_scale_kernel.  uint8 only without pad lanes.
#define POINTWISE_POST_RELU(wo)                                                                            \
    if (p.post_relu)                                                                                       \
    {                                                                                                      \
        _Pragma("unroll") for (int w_ = 0; w_ < 4; w_++)                                                   \
            (wo)[w_] = U8 ? __vmaxu4((wo)[w_], p.post_floor4) : __vmaxs4((wo)[w_], 0u);                    \
    }

// pooling/pooling_kernel_ref_int8.c:84-189, pooling_kernel_ref_uint8.c:91-204. Thread = pixel x 4 channels.
template <bool U8>
__global__ void __launch_bounds__(256) pool_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, PoolShape p)
{
    const int cw = p.cp / 4;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; // launchers guarantee totals < 2^31
    const unsigned total = (unsigned)(p.n * p.oh * p.ow * cw);
    if (idx >= total) return;
    const unsigned pix = idx / (unsigned)cw;
    const int c4 = (int)(idx - pix * cw);
    const unsigned prow = pix / (unsigned)p.ow;
    const int pw = (int)(pix - prow * p.ow);
    const int n = (int)(prow / (unsigned)p.oh);
    const int ph = (int)(prow - (unsigned)n * p.oh);

    int h_start = ph * p.sh - p.ph0, h_end = h_start + p.kh;
    if (h_end > p.h + p.ph0) h_end = p.h + p.ph0;
    int w_start = pw * p.sw - p.pw0, w_end = w_start + p.kw;
    if (w_end > p.w + p.pw0) w_end = p.w + p.pw0;
    int pool_size = 1;
    if (p.caffe_flavor) pool_size = (h_end - h_start) * (w_end - w_start);
    h_start = h_start > 0 ? h_start : 0;
    w_start = w_start > 0 ? w_start : 0;
    h_end = h_end < p.h ? h_end : p.h;
    w_end = w_end < p.w ? w_end : p.w;
    if (!p.caffe_flavor) pool_size = (h_end - h_start) * (w_end - w_start);

    int isum[4] = {0, 0, 0, 0};
    int imax[4];
    float fsum[4] = {0.f, 0.f, 0.f, 0.f};
    float fmax[4];
    bool first = true;
    for (int i = h_start; i < h_end; i++)
        for (int j = w_start; j < w_end; j++)
        {
            const unsigned xv = __ldg(reinterpret_cast<const unsigned*>(in + (((size_t)n * p.h + i) * p.w + j) * p.cp) + c4);
#pragma unroll
            for (int t = 0; t < 4; t++)
            {
                if (U8)
                {
                    // dequantise first, then max / sum in fp32 (pooling_kernel_ref_uint8.c:131-133)
                    const float f = __fmul_rn((float)((int)((xv >> (8 * t)) & 0xff) - p.in_zero), p.in_scale);
                    fmax[t] = first ? f : (fmax[t] > f ? fmax[t] : f);
                    fsum[t] = __fadd_rn(fsum[t], f);
                }
                else
                {
                    const int v = (int)(int8_t)(xv >> (8 * t));
                    imax[t] = first ? v : (imax[t] > v ? imax[t] : v);
                    isum[t] += v;
                }
            }
            first = false;
        }
    unsigned packed = 0;
#pragma unroll
    for (int t = 0; t < 4; t++)
    {
        int q = 0;
        if (c4 * 4 + t < p.c)
        {
            if (U8)
            {
                const float v = (p.method == TB200_POOL_MAX) ? fmax[t] : __fdiv_rn(fsum[t], (float)pool_size);
                q = (int)roundf(__fdiv_rn(v, p.out_scale)) + p.out_zero;
                q = (q > 255 ? 255 : q) & 0xff; // pooling_kernel_ref_uint8.c:197: upper clamp only
            }
            else if (p.method == TB200_POOL_MAX)
                q = clamp_i8((int)roundf(__fmul_rn((float)imax[t], __fdiv_rn(p.in_scale, p.out_scale))));
            else
            {
                float f = __fmul_rn((float)isum[t], p.in_scale);
                f = __fdiv_rn(f, (float)pool_size);
                q = clamp_i8((int)roundf(__fdiv_rn(f, p.out_scale)));
            }
        }
        packed |= (unsigned)q << (8 * t);
    }
    reinterpret_cast<unsigned*>(out + (size_t)pix * p.cp)[c4] = packed;
}

// relu/relu_kernel_ref_int8.c:41-94, relu_kernel_ref_uint8.c:41-96; eltwise/eltwise_ref.c:311-583,585-845.
// One thread = 16 bytes.  mode 0: relu(a); 1: a+b; 2: a*b.  Pad lanes: int8 0 -> 0; uint8 handled by `c` mask.
template <bool U8>
__global__ void __launch_bounds__(256) pointwise_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b,
                                                        uint4* __restrict__ out, long long nvec, PointwiseParams p)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nvec) return;
    const uint4 va = __ldg(a + i);
    uint4 vb = make_uint4(0, 0, 0, 0);
    if (p.mode != 0) vb = __ldg(b + i);
    const unsigned wa[4] = {va.x, va.y, va.z, va.w};
    const unsigned wb[4] = {vb.x, vb.y, vb.z, vb.w};
    unsigned wo[4];
    const int lane0 = (int)((i * 16) % p.cp); // channel index of byte 0 of this vector
#pragma unroll
    for (int w = 0; w < 4; w++)
    {
        unsigned packed = 0;
#pragma unroll
        for (int t = 0; t < 4; t++)
        {
            const int ch = lane0 + w * 4 + t;
            int q = 0;
            if (ch < p.c)
            {
                float f0, f1 = 0.f;
                if (U8)
                {
                    f0 = __fmul_rn((float)((int)((wa[w] >> (8 * t)) & 0xff) - p.zero0), p.scale0);
                    f1 = __fmul_rn((float)((int)((wb[w] >> (8 * t)) & 0xff) - p.zero1), p.scale1);
                }
                else
                {
                    f0 = __fmul_rn((float)(int)(int8_t)(wa[w] >> (8 * t)), p.scale0);
                    f1 = __fmul_rn((float)(int)(int8_t)(wb[w] >> (8 * t)), p.scale1);
                }
                float f;
                if (p.mode == 0)
                    f = (f0 < 0.f) ? ((p.negative_slope == 0.f) ? 0.f : __fmul_rn(f0, p.negative_slope)) : f0;
                else if (p.mode == 1)
                    f = __fadd_rn(f0, f1);
                else
                    f = __fmul_rn(f0, f1);
                if (U8)
                {
                    if (p.mode == 0) // relu_kernel_ref_uint8.c:85 round(f/s + zp): zero point added INSIDE round
                        q = clamp_u8((int)roundf(__fadd_rn(__fdiv_rn(f, p.out_scale), (float)p.out_zero)));
                    else
                        q = clamp_u8((int)roundf(__fdiv_rn(f, p.out_scale)) + p.out_zero);
                }
                else
                    q = clamp_i8((int)roundf(__fdiv_rn(f, p.out_scale)));
            }
            packed |= (unsigned)q << (8 * t);
        }
        wo[w] = packed;
    }
    POINTWISE_POST_RELU(wo);
    out[i] = make_uint4(wo[0], wo[1], wo[2], wo[3]);
}

// ---- fast exact variant ---------------------------------------------------------------------------------------------
// Same guarantee as the convolution epilogue (common.cuh): f is formed with the reference's own operations and roundings,
// only the final division by s_out is replaced by a multiplication with fl(1/s_out); |t - t_ref| <= 3*2^-24*|t| (+ one more
// rounding when the uint8 zero point is added inside the round), far inside the 2^-13 tie guard for |t| <= 512.  Elements
// inside the guard band, vectors that touch pad lanes of a uint8 tensor and parameter sets outside the proven range
// (launcher) go through the literal code above.  Arithmetic: bytes -> floats without I2FP (PRMT into the mantissa of
// 1.5*2^23, packed FADD), packed FMUL2/FADD2 chain, integer-domain clamp with one DPX instruction per channel pair.
template <bool U8>
__device__ __noinline__ unsigned pointwise_exact_byte(unsigned a, unsigned b, const PointwiseParams& p)
{
    float f0, f1;
    if (U8)
    {
        f0 = __fmul_rn((float)((int)a - p.zero0), p.scale0);
        f1 = __fmul_rn((float)((int)b - p.zero1), p.scale1);
    }
    else
    {
        f0 = __fmul_rn((float)(int)(int8_t)a, p.scale0);
        f1 = __fmul_rn((float)(int)(int8_t)b, p.scale1);
    }
    float f;
    if (p.mode == 0) f = (f0 < 0.f) ? ((p.negative_slope == 0.f) ? 0.f : __fmul_rn(f0, p.negative_slope)) : f0;
    else if (p.mode == 1) f = __fadd_rn(f0, f1);
    else f = __fmul_rn(f0, f1);
    if (U8)
    {
        if (p.mode == 0) return (unsigned)clamp_u8((int)roundf(__fadd_rn(__fdiv_rn(f, p.out_scale), (float)p.out_zero)));
        return (unsigned)clamp_u8((int)roundf(__fdiv_rn(f, p.out_scale)) + p.out_zero);
    }
    return (unsigned)clamp_i8((int)roundf(__fdiv_rn(f, p.out_scale)));
}

struct PointwiseFast
{
    float r_out;          // fl(1 / s_out)
    float off0, off1;     // what to subtract from MAGIC + raw byte to get the signed / zero-point-corrected input value
    uint32_t xor_mask;    // int8: 0x80808080 (bytes become excess-128), uint8: 0
    uint32_t q_add2, q_max2, q_byte_add; // integer clamp, see common.cuh requant_fast4_i8
    float zp_in_round;    // uint8 relu: the zero point is added before rounding
};

template <bool U8, int MODE>
__global__ void __launch_bounds__(256) pointwise_fast_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ out,
                                                             long long nvec, const PointwiseParams p, const PointwiseFast q)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nvec) return;
    const uint4 va = __ldg(a + i);
    uint4 vb = make_uint4(0, 0, 0, 0);
    if (MODE != 0) vb = __ldg(b + i);
    const unsigned wa[4] = {va.x, va.y, va.z, va.w};
    const unsigned wb[4] = {vb.x, vb.y, vb.z, vb.w};
    unsigned wo[4];
    const int lane0 = (int)((i * 16) % p.cp);
    if (lane0 + 16 > p.c)
    {
        // the vector holds pad lanes: literal path (they must come out as 0)
#pragma unroll
        for (int w = 0; w < 4; w++)
        {
            unsigned packed = 0;
            for (int t = 0; t < 4; t++)
                if (lane0 + w * 4 + t < p.c) packed |= pointwise_exact_byte<U8>((wa[w] >> (8 * t)) & 0xff, (wb[w] >> (8 * t)) & 0xff, p) << (8 * t);
            wo[w] = packed;
        }
        POINTWISE_POST_RELU(wo);
    out[i] = make_uint4(wo[0], wo[1], wo[2], wo[3]);
        return;
    }
    const uint64_t mg = f2_pack(TB200_MAGIC, TB200_MAGIC);
    const uint64_t o0 = f2_pack(q.off0, q.off0), o1 = f2_pack(q.off1, q.off1);
    const uint64_t s0 = f2_pack(p.scale0, p.scale0), s1 = f2_pack(p.scale1, p.scale1), rr = f2_pack(q.r_out, q.r_out);
    const uint64_t sl = f2_pack(p.negative_slope, p.negative_slope), zz = f2_pack(q.zp_in_round, q.zp_in_round);
    float gmax[4];
#pragma unroll
    for (int w = 0; w < 4; w++)
    {
        const unsigned xa = wa[w] ^ q.xor_mask, xb = wb[w] ^ q.xor_mask;
        uint32_t rb[4];
        float dm = 0.f;
#pragma unroll
        for (int h = 0; h < 2; h++)
        {
            // two bytes -> (MAGIC + byte) bit patterns -> exact floats
            const uint64_t fa = f2_sub(f2_pack(__uint_as_float(__byte_perm(xa, TB200_MAGIC_BITS, h ? 0x7652 : 0x7650)),
                                               __uint_as_float(__byte_perm(xa, TB200_MAGIC_BITS, h ? 0x7653 : 0x7651))), o0);
            uint64_t f = f2_mul(fa, s0);
            if (MODE != 0)
            {
                const uint64_t fb = f2_sub(f2_pack(__uint_as_float(__byte_perm(xb, TB200_MAGIC_BITS, h ? 0x7652 : 0x7650)),
                                                   __uint_as_float(__byte_perm(xb, TB200_MAGIC_BITS, h ? 0x7653 : 0x7651))), o1);
                const uint64_t g1 = f2_mul(fb, s1);
                f = (MODE == 1) ? f2_add(f, g1) : f2_mul(f, g1);
            }
            else
            {
                // (leaky) relu: max(f0, fl(f0 * slope)) for 0 <= slope < 1 (checked by the launcher)
                const uint64_t fn = f2_mul(f, sl);
                float f_lo, f_hi, n_lo, n_hi;
                f2_unpack(f, f_lo, f_hi);
                f2_unpack(fn, n_lo, n_hi);
                f = f2_pack(fmaxf(f_lo, n_lo), fmaxf(f_hi, n_hi));
            }
            uint64_t t = f2_mul(f, rr);
            if (U8 && MODE == 0) t = f2_add(t, zz);
            const uint64_t r = f2_add(t, mg);
            const uint64_t d = f2_sub(t, f2_sub(r, mg));
            float d_lo, d_hi;
            f2_unpack(d, d_lo, d_hi);
            dm = fmaxf(dm, fmaxf(fabsf(d_lo), fabsf(d_hi)));
            f2_unpack_bits(r, rb[2 * h], rb[2 * h + 1]);
        }
        gmax[w] = dm;
        const uint32_t p01 = __viaddmin_s16x2_relu(__byte_perm(rb[0], rb[1], 0x5410), q.q_add2, q.q_max2);
        const uint32_t p23 = __viaddmin_s16x2_relu(__byte_perm(rb[2], rb[3], 0x5410), q.q_add2, q.q_max2);
        unsigned word = __byte_perm(p01, p23, 0x6420);
        if (q.q_byte_add) word = ((word & 0x7f7f7f7fu) + (q.q_byte_add & 0x7f7f7f7fu)) ^ ((word ^ q.q_byte_add) & 0x80808080u);
        wo[w] = word;
    }
    if (fmaxf(fmaxf(gmax[0], gmax[1]), fmaxf(gmax[2], gmax[3])) > 0.5f - TB200_TIE_EPS)
    {
#pragma unroll
        for (int w = 0; w < 4; w++)
            if (gmax[w] > 0.5f - TB200_TIE_EPS)
            {
                unsigned packed = 0;
                for (int t = 0; t < 4; t++) packed |= pointwise_exact_byte<U8>((wa[w] >> (8 * t)) & 0xff, (wb[w] >> (8 * t)) & 0xff, p) << (8 * t);
                wo[w] = packed;
            }
    }
    POINTWISE_POST_RELU(wo);
    out[i] = make_uint4(wo[0], wo[1], wo[2], wo[3]);
}

// concat along channels with per-input requantisation (concat_kernel_ref_int8.c:70-80 roundf(q*s_in/s_out),
// concat_kernel_ref_uint8.c:82 roundf((q-zp)*s_in/s_out + zp_out)), and nearest upsample (upsample_ref.c:74); one byte per thread
// (channel counts such as 255 / 384 need not be multiples of 4 at the seams).
template <bool U8>
__global__ void __launch_bounds__(256) concat_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                     long long npix, int c, int c_write, int cp_in, int cp_out, int c_off, float s_in,
                                                     int z_in, float s_out, int z_out)
{
    // c_write >= c channels are written from c_off on: the last input of a concat also clears the output's pad lanes
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; // launchers guarantee totals < 2^31
    if (idx >= (unsigned)(npix * c_write)) return;
    const unsigned pix = idx / (unsigned)c_write;
    const int ch = (int)(idx - pix * c_write);
    if (ch >= c)
    {
        out[(size_t)pix * cp_out + c_off + ch] = 0;
        return;
    }
    const uint8_t v = in[(size_t)pix * cp_in + ch];
    int q;
    if (U8)
    {
        // concat_kernel_ref_uint8.c:82: roundf((q - zp_in) * (s_in / s_out) + zp_out), the zero point inside the rounding
        const float f = __fmul_rn((float)((int)v - z_in), __fdiv_rn(s_in, s_out));
        q = clamp_u8((int)roundf(__fadd_rn(f, (float)z_out)));
    }
    else
    {
        q = (int)roundf(__fmul_rn((float)(int)(int8_t)v, __fdiv_rn(s_in, s_out)));
        q = (q > 127 ? 127 : (q < -127 ? 127 : q)) & 0xff; // sic: concat_kernel_ref_int8.c:77-78
    }
    out[(size_t)pix * cp_out + c_off + ch] = (uint8_t)q;
}

__global__ void __launch_bounds__(256) upsample_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int n, int h,
                                                       int w, int cvec, int scale)
{
    const int oh = h * scale, ow = w * scale;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; // launchers guarantee totals < 2^31
    const unsigned total = (unsigned)(n * oh * ow * cvec);
    if (idx >= total) return;
    const unsigned pix = idx / (unsigned)cvec;
    const int cv = (int)(idx - pix * cvec);
    const unsigned prow = pix / (unsigned)ow;
    const int x = (int)(pix - prow * ow), b = (int)(prow / (unsigned)oh), y = (int)(prow - (unsigned)b * oh);
    out[idx] = __ldg(in + (((size_t)b * h + y / scale) * w + x / scale) * cvec + cv);
}

// host NCHW <-> device NHWC(pad).  32x32 byte tile transposes through shared memory: coalesced both ways.
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int c,
                                                           int hw, int cp)
{
    __shared__ uint8_t tile[32][33];
    const int n = blockIdx.z;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5; // 32 x 8
    for (int r = ty; r < 32; r += 8)
    {
        const int ch = c0 + r, p = hw0 + tx;
        tile[r][tx] = (ch < c && p < hw) ? in[((size_t)n * c + ch) * hw + p] : 0;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8)
    {
        const int p = hw0 + r, ch = c0 + tx;
        if (p < hw && ch < cp) out[((size_t)n * hw + p) * cp + ch] = tile[tx][r];
    }
}

__global__ void __launch_bounds__(256) nhwc_to_nchw_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int c,
                                                           int hw, int cp)
{
    __shared__ uint8_t tile[32][33];
    const int n = blockIdx.z;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8)
    {
        const int p = hw0 + r, ch = c0 + tx;
        tile[r][tx] = (p < hw && ch < cp) ? in[((size_t)n * hw + p) * cp + ch] : 0;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8)
    {
        const int ch = c0 + r, p = hw0 + tx;
        if (ch < c && p < hw) out[((size_t)n * c + ch) * hw + p] = tile[tx][r];
    }
}

// ------------------------------------------------------------------------------------------------------
// Launchers
// ------------------------------------------------------------------------------------------------------
static inline unsigned blocks_for(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }
#define TB200_CHECK_32BIT(total) \
    if ((long long)(total) >= 2147483647LL) return cudaErrorInvalidValue // kernels index with 32 bits

cudaError_t launch_conv_direct(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st)
{
    const long long npix = (long long)s.n * s.oh * s.ow;
    TB200_CHECK_32BIT(npix);
    const int og = s.oc / s.group;
    // OCT output channels per thread; with groups every tile must stay inside one group
    int oct = 8;
    if (s.group > 1 && (og % 8) != 0) oct = 4;
    if (s.group > 1 && (og % 4) != 0) return cudaErrorInvalidValue;
    dim3 grid(blocks_for(npix, 128), (s.ocp + oct - 1) / oct);
    const uint8_t* i8 = (const uint8_t*)in;
    const uint8_t* w8 = (const uint8_t*)w;
    uint8_t* o8 = (uint8_t*)out;
    if (e.is_uint8)
    {
        if (oct == 8) conv_direct_kernel<true, 8><<<grid, 128, 0, st>>>(i8, w8, o8, s, e);
        else conv_direct_kernel<true, 4><<<grid, 128, 0, st>>>(i8, w8, o8, s, e);
    }
    else
    {
        if (oct == 8) conv_direct_kernel<false, 8><<<grid, 128, 0, st>>>(i8, w8, o8, s, e);
        else conv_direct_kernel<false, 4><<<grid, 128, 0, st>>>(i8, w8, o8, s, e);
    }
    return cudaGetLastError();
}

cudaError_t launch_conv_dw(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st)
{
    if (!e.is_uint8 && s.kh == 3 && s.kw == 3 && s.dh == 1 && s.dw == 1 && s.sh == s.sw && (s.sh == 1 || s.sh == 2))
    {
        const int cw = s.cp / 4;
        if (s.sh == 1)
        {
            constexpr int TW = 8;
            const long long total = (long long)s.n * s.oh * ((s.ow + TW - 1) / TW) * cw;
            TB200_CHECK_32BIT(total * TW);
            conv_dw3x3_i8_kernel<TW, 1><<<blocks_for(total, 128), 128, 0, st>>>((const uint8_t*)in, (const uint8_t*)w, (uint8_t*)out, s, e);
        }
        else
        {
            constexpr int TW = 4;
            const long long total = (long long)s.n * s.oh * ((s.ow + TW - 1) / TW) * cw;
            TB200_CHECK_32BIT(total * TW);
            conv_dw3x3_i8_kernel<TW, 2><<<blocks_for(total, 128), 128, 0, st>>>((const uint8_t*)in, (const uint8_t*)w, (uint8_t*)out, s, e);
        }
        return cudaGetLastError();
    }
    const long long total = (long long)s.n * s.oh * s.ow * (s.cp / 4);
    TB200_CHECK_32BIT(total * 4);
    if (e.is_uint8) conv_dw_kernel<true><<<blocks_for(total, 256), 256, 0, st>>>((const uint8_t*)in, (const uint8_t*)w, (uint8_t*)out, s, e);
    else conv_dw_kernel<false><<<blocks_for(total, 256), 256, 0, st>>>((const uint8_t*)in, (const uint8_t*)w, (uint8_t*)out, s, e);
    return cudaGetLastError();
}

cudaError_t launch_conv_stem(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st)
{
    const long long npix = (long long)s.n * s.oh * s.ow;
    TB200_CHECK_32BIT(npix);
    if (s.ocp % 32 == 0)
    {
        dim3 grid(blocks_for(npix, 128), s.ocp / 32);
        const size_t sm = (size_t)s.kh * s.kw * 32 * 4;
        if (e.is_uint8) conv_stem_kernel<true, 32><<<grid, 128, sm, st>>>((const uint8_t*)in, (const uint8_t*)w, (uint8_t*)out, s, e);
        else conv_stem_kernel<false, 32><<<grid, 128, sm, st>>>((const uint8_t*)in, (const uint8_t*)w, (uint8_t*)out, s, e);
        return cudaGetLastError();
    }
    dim3 grid(blocks_for(npix, 128), s.ocp / 16);
    const size_t sm16 = (size_t)s.kh * s.kw * 16 * 4;
    if (e.is_uint8) conv_stem_kernel<true, 16><<<grid, 128, sm16, st>>>((const uint8_t*)in, (const uint8_t*)w, (uint8_t*)out, s, e);
    else conv_stem_kernel<false, 16><<<grid, 128, sm16, st>>>((const uint8_t*)in, (const uint8_t*)w, (uint8_t*)out, s, e);
    return cudaGetLastError();
}

// Max pooling whose output has the input's quantisation (the normal case: YOLO, ResNet): the reference's
// dequantise -> max -> requantise is then the identity on the winning byte (|fl(fl(k*s)/s) - k| <= 1.5*2^-23*|k| << 1/2 before
// its round()), so the result is the byte-wise max of the window -- int8: followed by the reference's clamp to -127.
// Thread = one output pixel x 16 channels.
template <bool U8>
__global__ void __launch_bounds__(256) pool_max_same_scale_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, PoolShape p)
{
    // p.lut: a (leaky) ReLU that preceded the pooling in the graph, as a byte table.  relu -> max == max -> relu because the
    // table is non-decreasing in the (signed / unsigned) byte order, so it is applied ONCE per output to the window's maximum
    // instead of to every input byte in a pass of its own (YOLOv3-tiny: conv -> leaky ReLU -> 2x2 max pool, six times).
    __shared__ uint8_t tab[256];
    if (p.lut)
    {
        tab[threadIdx.x] = __ldg(p.lut + threadIdx.x);
        __syncthreads();
    }
    const int cv = p.cp / 16;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned total = (unsigned)(p.n * p.oh * p.ow * cv);
    if (idx >= total) return;
    const unsigned pix = idx / (unsigned)cv;
    const int c16 = (int)(idx - pix * cv);
    const unsigned prow = pix / (unsigned)p.ow;
    const int pw = (int)(pix - prow * p.ow);
    const int n = (int)(prow / (unsigned)p.oh);
    const int ph = (int)(prow - (unsigned)n * p.oh);
    int h0 = ph * p.sh - p.ph0, h1 = h0 + p.kh, w0 = pw * p.sw - p.pw0, w1 = w0 + p.kw;
    h0 = h0 > 0 ? h0 : 0, w0 = w0 > 0 ? w0 : 0, h1 = h1 < p.h ? h1 : p.h, w1 = w1 < p.w ? w1 : p.w;
    uint4 m = U8 ? make_uint4(0, 0, 0, 0) : make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
    for (int i = h0; i < h1; i++)
        for (int j = w0; j < w1; j++)
        {
            const uint4 v = __ldg(in + (((size_t)n * p.h + i) * p.w + j) * cv + c16);
            if (U8) m = make_uint4(__vmaxu4(m.x, v.x), __vmaxu4(m.y, v.y), __vmaxu4(m.z, v.z), __vmaxu4(m.w, v.w));
            else m = make_uint4(__vmaxs4(m.x, v.x), __vmaxs4(m.y, v.y), __vmaxs4(m.z, v.z), __vmaxs4(m.w, v.w));
        }
    if (!U8) m = make_uint4(__vmaxs4(m.x, 0x81818181u), __vmaxs4(m.y, 0x81818181u), __vmaxs4(m.z, 0x81818181u), __vmaxs4(m.w, 0x81818181u));
    if (p.lut)
    {
        uint32_t w[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
        for (int j = 0; j < 4; j++)
        {
            uint32_t r = 0;
#pragma unroll
            for (int t = 0; t < 4; t++)
            {
                const uint32_t y = (c16 * 16 + j * 4 + t < p.c_real) ? (uint32_t)tab[(w[j] >> (8 * t)) & 0xffu] : 0u;
                r |= y << (8 * t);
            }
            w[j] = r;
        }
        m = make_uint4(w[0], w[1], w[2], w[3]);
    }
    out[(size_t)pix * cv + c16] = m;
}

cudaError_t launch_pool(const void* in, void* out, const PoolShape& p, bool u8, cudaStream_t st)
{
    if (p.method == TB200_POOL_MAX && (p.lut || (p.in_scale == p.out_scale && (!u8 || p.in_zero == p.out_zero))))
    {
        const long long tot = (long long)p.n * p.oh * p.ow * (p.cp / 16);
        TB200_CHECK_32BIT(tot * 16);
        TB200_CHECK_32BIT((long long)p.n * p.h * p.w * (p.cp / 16));
        if (u8) pool_max_same_scale_kernel<true><<<blocks_for(tot, 256), 256, 0, st>>>((const uint4*)in, (uint4*)out, p);
        else pool_max_same_scale_kernel<false><<<blocks_for(tot, 256), 256, 0, st>>>((const uint4*)in, (uint4*)out, p);
        return cudaGetLastError();
    }
    const long long total = (long long)p.n * p.oh * p.ow * (p.cp / 4);
    TB200_CHECK_32BIT(total * 4);
    TB200_CHECK_32BIT((long long)p.n * p.h * p.w * p.cp);
    if (u8) pool_kernel<true><<<blocks_for(total, 256), 256, 0, st>>>((const uint8_t*)in, (uint8_t*)out, p);
    else pool_kernel<false><<<blocks_for(total, 256), 256, 0, st>>>((const uint8_t*)in, (uint8_t*)out, p);
    return cudaGetLastError();
}

// ReLU whose output has the input's quantisation (what the reference's quantisation tool writes, quant_save_graph.cpp:136-200):
// dequantise -> max(., 0) -> requantise is then max(byte, zero point) (int8: max(byte, 0), and the clamp to -127 cannot trigger).
template <bool U8>
__global__ void __launch_bounds__(256) relu_same_scale_kernel(const uint4* __restrict__ a, uint4* __restrict__ out, long long nvec, uint32_t floor4)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nvec) return;
    const uint4 v = __ldg(a + i);
    // pad lanes of uint8 tensors hold 0 and must stay 0: max(0, zp) would be zp -> keep bytes that are 0... they are only 0 in
    // pad lanes or where the value really is 0 (< zp), in which case zp is the right answer; the launcher therefore uses this
    // kernel for uint8 only when the tensor has no pad lanes.
    if (U8) out[i] = make_uint4(__vmaxu4(v.x, floor4), __vmaxu4(v.y, floor4), __vmaxu4(v.z, floor4), __vmaxu4(v.w, floor4));
    else out[i] = make_uint4(__vmaxs4(v.x, 0u), __vmaxs4(v.y, 0u), __vmaxs4(v.z, 0u), __vmaxs4(v.w, 0u));
}

cudaError_t launch_pointwise(const void* a, const void* b, void* out, long long bytes, const PointwiseParams& p, bool u8, cudaStream_t st)
{
    const long long nvec = bytes / 16;
    if (p.mode == 0 && p.negative_slope == 0.f && p.scale0 == p.out_scale && (!u8 || (p.zero0 == p.out_zero && p.c == p.cp)))
    {
        const unsigned grid = (unsigned)blocks_for(nvec, 256);
        if (u8) relu_same_scale_kernel<true><<<grid, 256, 0, st>>>((const uint4*)a, (uint4*)out, nvec, (uint32_t)(p.out_zero & 0xff) * 0x01010101u);
        else relu_same_scale_kernel<false><<<grid, 256, 0, st>>>((const uint4*)a, (uint4*)out, nvec, 0u);
        return cudaGetLastError();
    }
    // ---- fast exact path when the value range is provably inside what its integer clamp / magic rounding can hold ----
    {
        const double so = p.out_scale, a0 = fabs((double)p.scale0), a1 = fabs((double)p.scale1);
        const double in0 = u8 ? 255.0 : 128.0;
        double tmax = 0;
        if (p.mode == 0) tmax = in0 * a0 / so;
        else if (p.mode == 1) tmax = in0 * (a0 + a1) / so;
        else tmax = in0 * a0 * in0 * a1 / so;
        const bool slope_ok = p.mode != 0 || (p.negative_slope >= 0.f && p.negative_slope < 1.f);
        if (so > 1e-30 && so < 1e30 && tmax + 256.0 < 32000.0 && slope_ok && p.c >= 16)
        {
            PointwiseFast q;
            q.r_out = 1.0f / p.out_scale;
            q.xor_mask = u8 ? 0u : 0x80808080u;
            // as_float(MAGIC_BITS | byte) = MAGIC + byte ; int8 bytes are excess-128 after the xor
            q.off0 = TB200_MAGIC + (u8 ? (float)p.zero0 : 128.f);
            q.off1 = TB200_MAGIC + (u8 ? (float)p.zero1 : 128.f);
            const int q_lo = u8 ? 0 : -127, q_hi = u8 ? 255 : 127;
            const int zp_after = (u8 && p.mode != 0) ? p.out_zero : 0; // uint8 sum / prod add the zero point after rounding
            // q' = max(min(q + zp_after - q_lo, q_hi - q_lo), 0), bytes = q' + q_lo
            const uint32_t add = (uint32_t)(zp_after - q_lo) & 0xffffu, mx = (uint32_t)(q_hi - q_lo) & 0xffffu;
            q.q_add2 = add | (add << 16), q.q_max2 = mx | (mx << 16);
            q.q_byte_add = ((uint32_t)q_lo & 0xffu) * 0x01010101u;
            q.zp_in_round = (u8 && p.mode == 0) ? (float)p.out_zero : 0.f;
            const unsigned grid = (unsigned)blocks_for(nvec, 256);
#define TB200_PW_CASE(U, MD)                                                                                                       \
    if (u8 == U && p.mode == MD)                                                                                                   \
    {                                                                                                                              \
        pointwise_fast_kernel<U, MD><<<grid, 256, 0, st>>>((const uint4*)a, (const uint4*)b, (uint4*)out, nvec, p, q);             \
        return cudaGetLastError();                                                                                                 \
    }
            TB200_PW_CASE(false, 0) TB200_PW_CASE(false, 1) TB200_PW_CASE(false, 2) TB200_PW_CASE(true, 0) TB200_PW_CASE(true, 1) TB200_PW_CASE(true, 2)
#undef TB200_PW_CASE
        }
    }
    if (u8) pointwise_kernel<true><<<blocks_for(nvec, 256), 256, 0, st>>>((const uint4*)a, (const uint4*)b, (uint4*)out, nvec, p);
    else pointwise_kernel<false><<<blocks_for(nvec, 256), 256, 0, st>>>((const uint4*)a, (const uint4*)b, (uint4*)out, nvec, p);
    return cudaGetLastError();
}

// Vectorised form for 16-channel-aligned inputs: the per-input requantisation of concat_kernel_ref_{int8,uint8}.c is a function of one
// byte, so it is a 256-entry table (built by engine.cu with the reference's arithmetic; nullptr = identity: equal quantisation).
// Thread = 16 channels of one pixel; the last input also clears the output's pad lanes (vectors beyond its channels).
__global__ void __launch_bounds__(256) concat_lut_kernel(const uint4* __restrict__ in, uint8_t* __restrict__ out, const uint8_t* __restrict__ lut, long long npix,
                                                         int cv_in, int cv_write, int cp_in, int cp_out, int c_off)
{
    __shared__ uint8_t tab[256];
    if (lut)
    {
        tab[threadIdx.x] = __ldg(lut + threadIdx.x);
        __syncthreads();
    }
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= npix * cv_write) return;
    const long long pix = idx / cv_write;
    const int v = (int)(idx - pix * cv_write);
    uint4 r = make_uint4(0, 0, 0, 0);
    if (v < cv_in)
    {
        r = __ldg(in + (size_t)pix * (cp_in / 16) + v);
        if (lut)
        {
            uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
            for (int j = 0; j < 4; j++)
                w[j] = (uint32_t)tab[w[j] & 0xffu] | ((uint32_t)tab[(w[j] >> 8) & 0xffu] << 8) | ((uint32_t)tab[(w[j] >> 16) & 0xffu] << 16) |
                       ((uint32_t)tab[w[j] >> 24] << 24);
            r = make_uint4(w[0], w[1], w[2], w[3]);
        }
    }
    *reinterpret_cast<uint4*>(out + (size_t)pix * cp_out + c_off + v * 16) = r;
}

cudaError_t launch_concat_lut(const void* in, void* out, const uint8_t* lut, long long npix, int c, int c_write, int cp_in, int cp_out, int c_off, cudaStream_t st)
{
    if ((c % 16) || (c_off % 16) || (c_write % 16)) return cudaErrorInvalidValue;
    const long long total = npix * (c_write / 16);
    TB200_CHECK_32BIT(total * 16);
    concat_lut_kernel<<<blocks_for(total, 256), 256, 0, st>>>((const uint4*)in, (uint8_t*)out, lut, npix, c / 16, c_write / 16, cp_in, cp_out, c_off);
    return cudaGetLastError();
}

cudaError_t launch_concat_part(const void* in, void* out, long long npix, int c, int c_write, int cp_in, int cp_out, int c_off, float s_in,
                               int z_in, float s_out, int z_out, bool u8, cudaStream_t st)
{
    const long long total = npix * c_write;
    TB200_CHECK_32BIT(total);
    if (u8) concat_kernel<true><<<blocks_for(total, 256), 256, 0, st>>>((const uint8_t*)in, (uint8_t*)out, npix, c, c_write, cp_in, cp_out, c_off, s_in, z_in, s_out, z_out);
    else concat_kernel<false><<<blocks_for(total, 256), 256, 0, st>>>((const uint8_t*)in, (uint8_t*)out, npix, c, c_write, cp_in, cp_out, c_off, s_in, z_in, s_out, z_out);
    return cudaGetLastError();
}

// ---- unary byte ops through a table (sigmoid_ref.c:84-172, hardswish_kernel_ref_uint8.c:41-80) ---------------------------
// Thread = 16 bytes (the 16 channels of one channel block of one pixel).  The table lives in shared memory replicated per
// bank group so that the 16 byte lookups of a thread rarely conflict; pad lanes (channel >= c) are written as 0.
__global__ void __launch_bounds__(256) byte_lut_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, const uint8_t* __restrict__ lut,
                                                       long long nvec, int c, int cvec)
{
    __shared__ uint8_t tab[256];
    tab[threadIdx.x] = __ldg(lut + threadIdx.x);
    __syncthreads();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nvec) return;
    const uint4 v = __ldg(in + i);
    const int c0 = (int)(i % cvec) * 16;
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; j++)
    {
        uint32_t r = 0;
#pragma unroll
        for (int t = 0; t < 4; t++)
        {
            const uint32_t b = (w[j] >> (8 * t)) & 0xffu;
            const uint32_t y = (c0 + j * 4 + t < c) ? (uint32_t)tab[b] : 0u;
            r |= y << (8 * t);
        }
        o[j] = r;
    }
    out[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

cudaError_t launch_byte_lut(const void* in, void* out, const uint8_t* lut, long long bytes, int c, int cp, cudaStream_t st)
{
    const long long nvec = bytes / 16;
    byte_lut_kernel<<<blocks_for(nvec, 256), 256, 0, st>>>((const uint4*)in, (uint4*)out, lut, nvec, c, cp / 16);
    return cudaGetLastError();
}

// ---- softmax over channels (softmax_kernel_ref_int8.c:41-118, softmax_kernel_ref_uint8.c:41-120; helpers
//      softmax_kernel_ref.h:36-82) ---------------------------------------------------------------------------------------------
// The reference dequantises, takes the per-position maximum, exp() in DOUBLE stored to float, a float running sum in channel
// order, a float division and round(f / s_out).  One thread per (image, position) walks the channels in the same order so the
// float sum has the same rounding sequence; CUDA's double exp() differs from glibc's by < 1 ulp of double, i.e. the float it
// rounds to is the same except on a double-rounding tie.
template <bool U8>
__global__ void __launch_bounds__(128) softmax_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, long long npix, int c, int cp,
                                                      float s_in, int z_in, float s_out, int z_out)
{
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= npix) return;
    const uint8_t* ip = in + (size_t)pix * cp;
    uint8_t* op = out + (size_t)pix * cp;
    auto deq = [&](int k) -> float
    {
        const uint8_t b = ip[k];
        return U8 ? __fmul_rn((float)b - (float)z_in, s_in) : __fmul_rn((float)(int)(int8_t)b, s_in);
    };
    float mx = deq(0);
    for (int k = 1; k < c; k++)
    {
        const float v = deq(k);
        if (mx < v) mx = v;
    }
    float sum = 0.f;
    for (int k = 0; k < c; k++) sum = __fadd_rn(sum, (float)exp((double)__fsub_rn(deq(k), mx)));
    for (int k = 0; k < c; k++)
    {
        const float e = (float)exp((double)__fsub_rn(deq(k), mx));
        const float f = __fdiv_rn(e, sum);
        int q = (int)roundf(__fdiv_rn(f, s_out));
        if (U8) q = clamp_u8(q + z_out);
        else q = clamp_i8(q);
        op[k] = (uint8_t)q;
    }
    for (int k = c; k < cp; k++) op[k] = 0;
}

cudaError_t launch_softmax(const void* in, void* out, long long npix, int c, int cp, float s_in, int z_in, float s_out, int z_out, bool u8,
                           cudaStream_t st)
{
    TB200_CHECK_32BIT(npix);
    if (u8) softmax_kernel<true><<<blocks_for(npix, 128), 128, 0, st>>>((const uint8_t*)in, (uint8_t*)out, npix, c, cp, s_in, z_in, s_out, z_out);
    else softmax_kernel<false><<<blocks_for(npix, 128), 128, 0, st>>>((const uint8_t*)in, (uint8_t*)out, npix, c, cp, s_in, z_in, s_out, z_out);
    return cudaGetLastError();
}

cudaError_t launch_upsample(const void* in, void* out, int n, int h, int w, int cp, int scale, cudaStream_t st)
{
    const long long total = (long long)n * h * scale * w * scale * (cp / 16);
    TB200_CHECK_32BIT(total * 16);
    upsample_kernel<<<blocks_for(total, 256), 256, 0, st>>>((const uint4*)in, (uint4*)out, n, h, w, cp / 16, scale);
    return cudaGetLastError();
}

cudaError_t launch_nchw_to_nhwc(const void* in, void* out, int n, int c, int h, int w, cudaStream_t st)
{
    const int hw = h * w, cp = cpad(c);
    dim3 grid((hw + 31) / 32, (cp + 31) / 32, n);
    nchw_to_nhwc_kernel<<<grid, 256, 0, st>>>((const uint8_t*)in, (uint8_t*)out, c, hw, cp);
    return cudaGetLastError();
}

cudaError_t launch_nhwc_to_nchw(const void* in, void* out, int n, int c, int h, int w, cudaStream_t st)
{
    const int hw = h * w, cp = cpad(c);
    dim3 grid((hw + 31) / 32, (cp + 31) / 32, n);
    nhwc_to_nchw_kernel<<<grid, 256, 0, st>>>((const uint8_t*)in, (uint8_t*)out, c, hw, cp);
    return cudaGetLastError();
}

} // namespace tb200
