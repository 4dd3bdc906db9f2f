/*
 * tb200_oracle.c -- CPU restatement of the reference's int8/uint8 hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (tengine_b200/, libtengine_b200.so) may include, link
 * or call this file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg use it, as the
 * checker.  Parity status: PINNED -- tests/test_oracle_vs_reference.py runs every function below against
 * the unmodified reference built by oracle/build_ref.py (oracle/_ref/libtengine-lite.so) on seeded inputs,
 * and tests/test_oracle_golden.py checks it against the known-answer vectors the reference's own op tests
 * embed (tests/golden/).
 *
 * All tensors are host NCHW, as in the reference (tm2_serializer.c:169-173).  Paths in comments are
 * relative to /root/reference/source/device/cpu/op/.
 *
 * Build: gcc -O2 -fopenmp -shared -fPIC -ffp-contract=off tb200_oracle.c -o libtb200_oracle.so -lm
 * (-ffp-contract=off: the reference is compiled -mfma, but its epilogues are written as separate
 *  statements through float arrays, so no contraction can happen there either.)
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/tengine_b200.h"

#define ORACLE_API __attribute__((visibility("default")))

static inline int conv_out_dim(int in, int k, int s, int p0, int p1, int d)
{
    return (in + p0 + p1 - (d * (k - 1) + 1)) / s + 1;
}

/* ---- activation + requant tails ---------------------------------------------------------------- */

/* conv/x86/conv_kernel_x86.c:1841-1889 (HCL): activation==0 -> max(f,0); activation>0 -> clip [0,6];
 * q = (int32)round(f / s_out); clamp +-127.  `round` is the double libm round applied to the float quotient. */
static inline int8_t tail_int8_hcl(float f, int activation, float s_out)
{
    if (activation == 0 && f < 0) f = 0;
    if (activation > 0)
    {
        if (f < 0) f = 0;
        if (f > 6) f = 6;
    }
    int32_t q = (int32_t)(round(f / s_out));
    if (q > 127) q = 127;
    else if (q < -127) q = -127;
    return (int8_t)q;
}

/* conv/conv_kernel_ref_int8.c:142-167 (REF): activation 0 / 1 / 6 distinguished */
static inline float act_ref(float total, int activation)
{
    if (activation >= 0)
    {
        if (total < 0 && activation != 1) total = 0;
        if (total > 1 && activation == 1) total = 1;
        if (total > 6 && activation == 6) total = 6;
        if (total < -1 && activation == 1) total = -1;
    }
    return total;
}

static inline int8_t tail_int8_ref(float total, int activation, float s_out)
{
    total = act_ref(total, activation);
    int out = round(total / s_out);
    if (out > 127) out = 127;
    if (out < -127) out = -127;
    return (int8_t)out;
}

/* ---- convolution, int8 ----------------------------------------------------------------------------
 * Integer accumulation is exact and order-independent, so one loop nest serves every int8 variant:
 *   conv/conv_kernel_ref_int8.c:87-171           (ref_conv_int8, all shapes)
 *   conv/x86/conv_kernel_x86.c:187-242,1008,1796 (im2col_int8 + sgemm_i8 + sgemm_int8)
 *   conv/x86/conv_dw_hcl_x86.c:97-445            (convdw3x3s{1,2}_int8_sse)
 *   conv/x86/conv_direct_hcl_int8_x86.c:95-449   (conv3x3s{1,2}_int8_sse)
 * They differ only in the float epilogue, selected by L->recipe. */
ORACLE_API int tb200_oracle_conv_int8(const tb200_tensor_desc* tin, const int8_t* x, const tb200_tensor_desc* tout,
                                      int8_t* y, const tb200_layer_desc* L)
{
    const int N = tin->dims[0], C = tin->dims[1], H = tin->dims[2], W = tin->dims[3];
    const int OC = tout->dims[1], OH = tout->dims[2], OW = tout->dims[3];
    const int G = L->group, cg = C / G, og = OC / G;
    const int KH = L->kernel_h, KW = L->kernel_w;
    const int8_t* w = (const int8_t*)L->weight;
    const float s_in = tin->scale, s_out = tout->scale;
    if (OH != conv_out_dim(H, KH, L->stride_h, L->pad_h0, L->pad_h1, L->dilation_h)) return -1;
    if (OW != conv_out_dim(W, KW, L->stride_w, L->pad_w0, L->pad_w1, L->dilation_w)) return -1;

#pragma omp parallel for collapse(2) schedule(static)
    for (int n = 0; n < N; n++)
        for (int oc = 0; oc < OC; oc++)
        {
            const int g = oc / og;
            const int8_t* wk = w + (size_t)oc * cg * KH * KW;
            const float s_w = L->weight_scales[oc];
            const float dq = s_in * s_w; /* conv_kernel_ref_int8.c:77 */
            for (int oh = 0; oh < OH; oh++)
                for (int ow = 0; ow < OW; ow++)
                {
                    int32_t acc = 0;
                    for (int c = 0; c < cg; c++)
                        for (int kh = 0; kh < KH; kh++)
                        {
                            const int iy = oh * L->stride_h - L->pad_h0 + kh * L->dilation_h;
                            if (iy < 0 || iy >= H) continue;
                            for (int kw = 0; kw < KW; kw++)
                            {
                                const int ix = ow * L->stride_w - L->pad_w0 + kw * L->dilation_w;
                                if (ix < 0 || ix >= W) continue;
                                acc += (int32_t)x[(((size_t)n * C + g * cg + c) * H + iy) * W + ix]
                                       * (int32_t)wk[(c * KH + kh) * KW + kw];
                            }
                        }
                    if (L->bias) acc += L->bias[oc];
                    int8_t q;
                    if (L->recipe == TB200_RECIPE_HCL)
                    {
                        /* conv_kernel_x86.c:1834: (float)(acc + bias) * input_scale * kernel_scales[i] */
                        float f = (float)acc * s_in * s_w;
                        q = tail_int8_hcl(f, L->activation, s_out);
                    }
                    else
                    {
                        /* conv_kernel_ref_int8.c:140: total_i32 * dequant_scales[] */
                        float f = acc * dq;
                        q = tail_int8_ref(f, L->activation, s_out);
                    }
                    y[(((size_t)n * OC + oc) * OH + oh) * OW + ow] = q;
                }
        }
    return 0;
}

/* ---- convolution, uint8 ---------------------------------------------------------------------------
 * The reference simulates uint8 in fp32: dequantise both operands, accumulate in fp32, requantise
 *   conv/conv_kernel_ref_uint8.c:42-195                 (REF: sequential fp32 accumulation, c,kh,kw order)
 *   conv/x86/conv_kernel_x86.c:68-80,124-185,1703-1794  (HCL: AVX/FMA sgemm_fp accumulation order)
 * mode 0 ("exact"): integer-exact sum of (q_x-zp_x)(q_w-zp_w), then f = (float)acc * (s_x*s_w); this is what
 *                   the device computes and differs from the reference only by fp32 summation rounding.
 * mode 1 ("fp32seq"): the literal ref_conv_uint8 arithmetic (bit-exact with the reference under TG_DEBUG_REF). */
ORACLE_API int tb200_oracle_conv_uint8(const tb200_tensor_desc* tin, const uint8_t* x, const tb200_tensor_desc* tout,
                                       uint8_t* y, const tb200_layer_desc* L, int mode)
{
    const int N = tin->dims[0], C = tin->dims[1], H = tin->dims[2], W = tin->dims[3];
    const int OC = tout->dims[1], OH = tout->dims[2], OW = tout->dims[3];
    const int G = L->group, cg = C / G, og = OC / G;
    const int KH = L->kernel_h, KW = L->kernel_w;
    const uint8_t* w = (const uint8_t*)L->weight;
    const float s_in = tin->scale, s_out = tout->scale, s_w = L->weight_scales[0];
    const int z_in = tin->zero_point, z_out = tout->zero_point, z_w = L->weight_zero;
    if (OH != conv_out_dim(H, KH, L->stride_h, L->pad_h0, L->pad_h1, L->dilation_h)) return -1;
    if (OW != conv_out_dim(W, KW, L->stride_w, L->pad_w0, L->pad_w1, L->dilation_w)) return -1;

#pragma omp parallel for collapse(2) schedule(static)
    for (int n = 0; n < N; n++)
        for (int oc = 0; oc < OC; oc++)
        {
            const int g = oc / og;
            const uint8_t* wk = w + (size_t)oc * cg * KH * KW;
            for (int oh = 0; oh < OH; oh++)
                for (int ow = 0; ow < OW; ow++)
                {
                    int32_t acc = 0;
                    float facc = 0.f;
                    for (int c = 0; c < cg; c++)
                        for (int kh = 0; kh < KH; kh++)
                        {
                            const int iy = oh * L->stride_h - L->pad_h0 + kh * L->dilation_h;
                            if (iy < 0 || iy >= H) continue;
                            for (int kw = 0; kw < KW; kw++)
                            {
                                const int ix = ow * L->stride_w - L->pad_w0 + kw * L->dilation_w;
                                if (ix < 0 || ix >= W) continue; /* padding taps contribute 0.0f (:167-181) */
                                const uint8_t qx = x[(((size_t)n * C + g * cg + c) * H + iy) * W + ix];
                                const uint8_t qw = wk[(c * KH + kh) * KW + kw];
                                if (mode == 0)
                                    acc += ((int32_t)qx - z_in) * ((int32_t)qw - z_w);
                                else
                                {
                                    /* conv_kernel_ref_uint8.c:76,82,152 */
                                    float xf = ((float)qx - z_in) * s_in;
                                    float wf = ((float)qw - z_w) * s_w;
                                    facc += xf * wf;
                                }
                            }
                        }
                    float f;
                    if (mode == 0)
                    {
                        f = (float)acc * (s_in * s_w);
                        if (L->bias) f += (float)L->bias[oc] * (s_in * s_w); /* conv_kernel_x86.c:1723,1740 */
                    }
                    else
                    {
                        f = facc;
                        if (L->bias) f += (float)L->bias[oc] * s_in * s_w; /* conv_kernel_ref_uint8.c:94 */
                    }
                    int q;
                    if (L->recipe == TB200_RECIPE_HCL)
                    {
                        /* conv_kernel_x86.c:1745-1789 */
                        if (L->activation == 0 && f < 0) f = 0;
                        if (L->activation > 0)
                        {
                            if (f < 0) f = 0;
                            if (f > 6) f = 6;
                        }
                        q = (int)(round(f / s_out) + z_out);
                    }
                    else
                    {
                        f = act_ref(f, L->activation);
                        q = round(f / s_out) + z_out; /* conv_kernel_ref_uint8.c:181 */
                    }
                    if (q > 255) q = 255;
                    if (q < 0) q = 0;
                    y[(((size_t)n * OC + oc) * OH + oh) * OW + ow] = (uint8_t)q;
                }
        }
    return 0;
}

/* ---- fully connected: fc/fc_ref.c:121-297 ---------------------------------------------------------- */
ORACLE_API int tb200_oracle_fc_int8(const tb200_tensor_desc* tin, const int8_t* x, const tb200_tensor_desc* tout,
                                    int8_t* y, const tb200_layer_desc* L)
{
    const int N = tin->dims[0], K = tin->dims[1] * tin->dims[2] * tin->dims[3], O = tout->dims[1];
    const int8_t* w = (const int8_t*)L->weight;
#pragma omp parallel for collapse(2)
    for (int n = 0; n < N; n++)
        for (int o = 0; o < O; o++)
        {
            /* fc_ref.c:225: requant_scales[i] = (input_scale * weight_scales[i]) / output_scale */
            const float rq = (tin->scale * L->weight_scales[o]) / tout->scale;
            int32_t acc = L->bias ? L->bias[o] : 0;
            for (int k = 0; k < K; k++) acc += (int32_t)x[(size_t)n * K + k] * (int32_t)w[(size_t)o * K + k];
            int q = roundf(acc * rq); /* fc_ref.c:252 */
            if (q > 127) q = 127;
            else if (q < -127) q = -127;
            y[(size_t)n * O + o] = (int8_t)q;
        }
    return 0;
}

/* mode 0: exact-integer accumulation (device definition); mode 1: literal fc_ref.c:121-207 fp32 simulation */
ORACLE_API int tb200_oracle_fc_uint8(const tb200_tensor_desc* tin, const uint8_t* x, const tb200_tensor_desc* tout,
                                     uint8_t* y, const tb200_layer_desc* L, int mode)
{
    const int N = tin->dims[0], K = tin->dims[1] * tin->dims[2] * tin->dims[3], O = tout->dims[1];
    const uint8_t* w = (const uint8_t*)L->weight;
    const float s_in = tin->scale, s_out = tout->scale, s_w = L->weight_scales[0];
    const int z_in = tin->zero_point, z_out = tout->zero_point, z_w = L->weight_zero;
#pragma omp parallel for collapse(2)
    for (int n = 0; n < N; n++)
        for (int o = 0; o < O; o++)
        {
            float data;
            if (mode == 0)
            {
                int32_t acc = 0;
                for (int k = 0; k < K; k++)
                    acc += ((int32_t)x[(size_t)n * K + k] - z_in) * ((int32_t)w[(size_t)o * K + k] - z_w);
                data = (float)acc * (s_in * s_w);
                if (L->bias) data += L->bias[o] * L->bias_scale;
            }
            else
            {
                data = L->bias ? L->bias[o] * L->bias_scale : 0.f; /* fc_ref.c:146 */
                for (int k = 0; k < K; k++)
                {
                    float xf = ((float)x[(size_t)n * K + k] - (float)z_in) * s_in;
                    float wf = ((float)w[(size_t)o * K + k] - (float)z_w) * s_w;
                    data += xf * wf;
                }
            }
            int q = (L->bias ? roundf(data / s_out) : round(data / s_out)) + z_out; /* fc_ref.c:162,193 */
            if (q > 255) q = 255;
            else if (q < 0) q = 0;
            y[(size_t)n * O + o] = (uint8_t)q;
        }
    return 0;
}

/* ---- pooling: pooling/pooling_kernel_ref_int8.c:84-189, pooling_kernel_ref_uint8.c:91-204 ----------- */
static void pool_window(const tb200_layer_desc* L, int H, int W, int ph, int pw, int* hs, int* he, int* ws, int* we,
                        int* pool_size)
{
    int h_start = ph * L->stride_h - L->pad_h0, h_end = h_start + L->kernel_h;
    if (h_end > H + L->pad_h0) h_end = H + L->pad_h0;
    int w_start = pw * L->stride_w - L->pad_w0, w_end = w_start + L->kernel_w;
    if (w_end > W + L->pad_w0) w_end = W + L->pad_w0;
    if (L->caffe_flavor) *pool_size = (h_end - h_start) * (w_end - w_start);
    h_start = h_start > 0 ? h_start : 0;
    w_start = w_start > 0 ? w_start : 0;
    h_end = h_end < H ? h_end : H;
    w_end = w_end < W ? w_end : W;
    if (!L->caffe_flavor) *pool_size = (h_end - h_start) * (w_end - w_start);
    *hs = h_start, *he = h_end, *ws = w_start, *we = w_end;
}

/* For `global` pooling the reference's infer_shape/prerun has already rewritten kernel=HxW, stride=1, pad=0
 * (operator/prototype/pooling.c); callers of the oracle pass those resolved values. */
ORACLE_API int tb200_oracle_pool_int8(const tb200_tensor_desc* tin, const int8_t* x, const tb200_tensor_desc* tout,
                                      int8_t* y, const tb200_layer_desc* L)
{
    const int N = tin->dims[0], C = tin->dims[1], H = tin->dims[2], W = tin->dims[3];
    const int OH = tout->dims[2], OW = tout->dims[3];
    const float s_in = tin->scale, s_out = tout->scale;
    const float requant = s_in / s_out;
#pragma omp parallel for collapse(2)
    for (int n = 0; n < N; n++)
        for (int c = 0; c < C; c++)
        {
            const int8_t* p = x + ((size_t)n * C + c) * H * W;
            for (int ph = 0; ph < OH; ph++)
                for (int pw = 0; pw < OW; pw++)
                {
                    int hs, he, ws, we, psz = 1;
                    pool_window(L, H, W, ph, pw, &hs, &he, &ws, &we, &psz);
                    int32_t q;
                    if (L->pool_method == TB200_POOL_MAX)
                    {
                        int8_t mx = p[hs * W + ws];
                        for (int i = hs; i < he; i++)
                            for (int j = ws; j < we; j++)
                                if (p[i * W + j] > mx) mx = p[i * W + j];
                        q = round((float)mx * requant);
                    }
                    else
                    {
                        int32_t sum = 0;
                        for (int i = hs; i < he; i++)
                            for (int j = ws; j < we; j++) sum += p[i * W + j];
                        float f = sum * s_in;
                        f = f / (float)psz;
                        q = round((float)f / s_out);
                    }
                    if (q > 127) q = 127;
                    else if (q < -127) q = -127;
                    y[(((size_t)n * C + c) * OH + ph) * OW + pw] = (int8_t)q;
                }
        }
    return 0;
}

ORACLE_API int tb200_oracle_pool_uint8(const tb200_tensor_desc* tin, const uint8_t* x, const tb200_tensor_desc* tout,
                                       uint8_t* y, const tb200_layer_desc* L)
{
    const int N = tin->dims[0], C = tin->dims[1], H = tin->dims[2], W = tin->dims[3];
    const int OH = tout->dims[2], OW = tout->dims[3];
    const float s_in = tin->scale, s_out = tout->scale;
    const int z_in = tin->zero_point, z_out = tout->zero_point;
#pragma omp parallel for collapse(2)
    for (int n = 0; n < N; n++)
        for (int c = 0; c < C; c++)
        {
            const uint8_t* p = x + ((size_t)n * C + c) * H * W;
            for (int ph = 0; ph < OH; ph++)
                for (int pw = 0; pw < OW; pw++)
                {
                    int hs, he, ws, we, psz = 1;
                    pool_window(L, H, W, ph, pw, &hs, &he, &ws, &we, &psz);
                    float v;
                    if (L->pool_method == TB200_POOL_MAX)
                    {
                        v = (p[hs * W + ws] - z_in) * s_in; /* pooling_kernel_ref_uint8.c:131 dequant */
                        for (int i = hs; i < he; i++)
                            for (int j = ws; j < we; j++)
                            {
                                float t = (p[i * W + j] - z_in) * s_in;
                                v = v > t ? v : t;
                            }
                    }
                    else
                    {
                        float sum = 0.f;
                        for (int i = hs; i < he; i++)
                            for (int j = ws; j < we; j++) sum += (p[i * W + j] - z_in) * s_in;
                        v = sum / psz;
                    }
                    int q = round(v / s_out) + z_out;
                    y[(((size_t)n * C + c) * OH + ph) * OW + pw] = q > 255 ? 255 : q; /* :197 no lower clamp */
                }
        }
    return 0;
}

/* ---- relu / leaky relu: relu/relu_kernel_ref_int8.c:41-94, relu_kernel_ref_uint8.c:41-96 ------------ */
ORACLE_API int tb200_oracle_relu_int8(const tb200_tensor_desc* tin, const int8_t* x, const tb200_tensor_desc* tout,
                                      int8_t* y, const tb200_layer_desc* L)
{
    const size_t total = (size_t)tin->dims[0] * tin->dims[1] * tin->dims[2] * tin->dims[3];
#pragma omp parallel for
    for (size_t i = 0; i < total; i++)
    {
        float f = (float)x[i] * tin->scale;
        if (f < 0) f = (L->negative_slope == 0) ? 0 : f * L->negative_slope;
        int q = round(f / tout->scale);
        if (q > 127) q = 127;
        else if (q < -127) q = -127;
        y[i] = (int8_t)q;
    }
    return 0;
}

ORACLE_API int tb200_oracle_relu_uint8(const tb200_tensor_desc* tin, const uint8_t* x, const tb200_tensor_desc* tout,
                                       uint8_t* y, const tb200_layer_desc* L)
{
    const size_t total = (size_t)tin->dims[0] * tin->dims[1] * tin->dims[2] * tin->dims[3];
#pragma omp parallel for
    for (size_t i = 0; i < total; i++)
    {
        float f = ((float)x[i] - (float)tin->zero_point) * tin->scale;
        if (f < 0) f = (L->negative_slope == 0) ? 0 : f * L->negative_slope;
        int q = round(f / tout->scale + tout->zero_point); /* relu_kernel_ref_uint8.c:85: zp inside round */
        if (q > 255) q = 255;
        else if (q < 0) q = 0;
        y[i] = (uint8_t)q;
    }
    return 0;
}

/* ---- eltwise sum / prod of two same-shape tensors: eltwise/eltwise_ref.c:311-583 (uint8), 585-845 (int8) */
ORACLE_API int tb200_oracle_eltwise_int8(const tb200_tensor_desc* t0, const int8_t* a, const tb200_tensor_desc* t1,
                                         const int8_t* b, const tb200_tensor_desc* tout, int8_t* y,
                                         const tb200_layer_desc* L)
{
    const size_t total = (size_t)t0->dims[0] * t0->dims[1] * t0->dims[2] * t0->dims[3];
#pragma omp parallel for
    for (size_t i = 0; i < total; i++)
    {
        float f0 = (float)a[i] * t0->scale, f1 = (float)b[i] * t1->scale;
        float f = (L->elt_type == TB200_ELT_SUM) ? f0 + f1 : f0 * f1;
        int q = round(f / tout->scale);
        if (q > 127) q = 127;
        else if (q < -127) q = -127;
        y[i] = (int8_t)q;
    }
    return 0;
}

ORACLE_API int tb200_oracle_eltwise_uint8(const tb200_tensor_desc* t0, const uint8_t* a, const tb200_tensor_desc* t1,
                                          const uint8_t* b, const tb200_tensor_desc* tout, uint8_t* y,
                                          const tb200_layer_desc* L)
{
    const size_t total = (size_t)t0->dims[0] * t0->dims[1] * t0->dims[2] * t0->dims[3];
#pragma omp parallel for
    for (size_t i = 0; i < total; i++)
    {
        float f0 = (a[i] - t0->zero_point) * t0->scale, f1 = (b[i] - t1->zero_point) * t1->scale;
        float f = (L->elt_type == TB200_ELT_SUM) ? f0 + f1 : f0 * f1;
        int q = round(f / tout->scale) + tout->zero_point;
        if (q > 255) q = 255;
        else if (q < 0) q = 0;
        y[i] = (uint8_t)q;
    }
    return 0;
}

/* ---- channel concat (4-D, axis 1): concat/concat_kernel_ref_int8.c, concat_kernel_ref_uint8.c ------- */
ORACLE_API int tb200_oracle_concat(const tb200_tensor_desc* const* tins, const void* const* xs, int num_inputs,
                                   const tb200_tensor_desc* tout, void* y)
{
    const int N = tout->dims[0], OC = tout->dims[1], HW = tout->dims[2] * tout->dims[3];
    const int is_u8 = tout->data_type == TB200_DT_UINT8;
    int coff = 0;
    for (int k = 0; k < num_inputs; k++)
    {
        const tb200_tensor_desc* t = tins[k];
        const int C = t->dims[1];
        if (num_inputs == 1)
        {
            memcpy(y, xs[0], (size_t)N * C * HW);
            return 0;
        }
        for (int n = 0; n < N; n++)
            for (size_t i = 0; i < (size_t)C * HW; i++)
            {
                const size_t src = (size_t)n * C * HW + i, dst = ((size_t)n * OC + coff) * HW + i;
                if (is_u8)
                {
                    /* concat_kernel_ref_uint8.c:82: roundf((q - zp_in) * (s_in/s_out) + zp_out) -- zp inside the rounding */
                    uint8_t q = ((const uint8_t*)xs[k])[src];
                    float rescale = t->scale / tout->scale;
                    int u = roundf((float)((int)q - t->zero_point) * rescale + (float)tout->zero_point);
                    if (u > 255) u = 255;
                    else if (u < 0) u = 0;
                    ((uint8_t*)y)[dst] = (uint8_t)u;
                }
                else
                {
                    /* concat_kernel_ref_int8.c:70-80: roundf(q * (s_in/s_out)); note the reference clamps
                     * values below -127 to +127 (sic); unreachable because |q| <= 127 and rescale is what it is */
                    float rescale = t->scale / tout->scale;
                    int v = roundf(((const int8_t*)xs[k])[src] * rescale);
                    if (v > 127) v = 127;
                    else if (v < -127) v = 127;
                    ((int8_t*)y)[dst] = (int8_t)v;
                }
            }
        coff += C;
    }
    return 0;
}

/* ---- nearest upsample by an integer factor: upsample/upsample_ref.c:74 (uint8 path: pure byte copy) -- */
ORACLE_API int tb200_oracle_upsample(const tb200_tensor_desc* tin, const void* x, const tb200_tensor_desc* tout,
                                     void* y, const tb200_layer_desc* L)
{
    const int N = tin->dims[0], C = tin->dims[1], H = tin->dims[2], W = tin->dims[3];
    const int OH = tout->dims[2], OW = tout->dims[3], s = L->up_scale;
    const uint8_t* in = (const uint8_t*)x;
    uint8_t* out = (uint8_t*)y;
    for (size_t nc = 0; nc < (size_t)N * C; nc++)
        for (int oh = 0; oh < OH; oh++)
            for (int ow = 0; ow < OW; ow++)
            {
                int ih = oh / s, iw = ow / s;
                if (ih >= H) ih = H - 1;
                if (iw >= W) iw = W - 1;
                out[(nc * OH + oh) * OW + ow] = in[(nc * H + ih) * W + iw];
            }
    return 0;
}

/* ---- sigmoid: sigmoid/sigmoid_ref.c:84-127 (int8), :129-172 (uint8).  The reference's MIN(x, 30) result is overwritten by
 *      its MAX(x, -30) line (:110-111), so only the lower clamp acts; exp() runs in double on the float argument. ------------ */
ORACLE_API int tb200_oracle_sigmoid(const tb200_tensor_desc* tin, const void* x, const tb200_tensor_desc* tout, void* y)
{
    const size_t total = (size_t)tin->dims[0] * tin->dims[1] * tin->dims[2] * tin->dims[3];
    const int u8 = tin->data_type == TB200_DT_UINT8;
    for (size_t i = 0; i < total; i++)
    {
        const float q = u8 ? (float)((const uint8_t*)x)[i] : (float)((const int8_t*)x)[i];
        float in = (q - (float)tin->zero_point) * tin->scale;
        float o = (in > -30.0f) ? in : -30.0f;
        o = 1 / (1 + exp(-o));
        int v = round(o / tout->scale + tout->zero_point);
        if (u8)
        {
            if (v > 255) v = 255;
            else if (v < 0) v = 0;
            ((uint8_t*)y)[i] = (uint8_t)v;
        }
        else
        {
            if (v > 127) v = 127;
            else if (v < -127) v = -127;
            ((int8_t*)y)[i] = (int8_t)v;
        }
    }
    return 0;
}

/* ---- hardswish, uint8 only as in the reference: hardswish/hardswish_kernel_ref_uint8.c:41-80 --------------------------- */
ORACLE_API int tb200_oracle_hardswish_uint8(const tb200_tensor_desc* tin, const uint8_t* x, const tb200_tensor_desc* tout, uint8_t* y)
{
    const size_t total = (size_t)tin->dims[0] * tin->dims[1] * tin->dims[2] * tin->dims[3];
    for (size_t i = 0; i < total; i++)
    {
        float d = ((float)x[i] - (float)tin->zero_point) * tin->scale;
        float tmp = d + 3.f;
        if (tmp < 0.f) tmp = 0.f;
        if (tmp > 6.f) tmp = 6.f;
        d = d * (tmp / 6.f);
        int v = round(d / tout->scale + tout->zero_point);
        if (v > 255) v = 255;
        else if (v < 0) v = 0;
        y[i] = (uint8_t)v;
    }
    return 0;
}

/* ---- softmax over axis 1 of an NCHW tensor: softmax/softmax_kernel_ref_int8.c:41-118, softmax_kernel_ref_uint8.c:41-120,
 *      GetMaxArray / GetOutResult of softmax_kernel_ref.h:36-82 (float max, exp in double stored to float, float running sum in
 *      channel order, float division) ------------------------------------------------------------------------------------------ */
ORACLE_API int tb200_oracle_softmax(const tb200_tensor_desc* tin, const void* x, const tb200_tensor_desc* tout, void* y)
{
    const int N = tin->dims[0], C = tin->dims[1], HW = tin->dims[2] * tin->dims[3];
    const int u8 = tin->data_type == TB200_DT_UINT8;
    float* f = (float*)malloc(sizeof(float) * (size_t)C * HW);
    float* o = (float*)malloc(sizeof(float) * (size_t)C * HW);
    float* mx = (float*)malloc(sizeof(float) * HW);
    float* sum = (float*)malloc(sizeof(float) * HW);
    for (int n = 0; n < N; n++)
    {
        const size_t base = (size_t)n * C * HW;
        for (size_t i = 0; i < (size_t)C * HW; i++)
            f[i] = u8 ? ((float)((const uint8_t*)x)[base + i] - (float)(uint8_t)tin->zero_point) * tin->scale
                      : (float)((const int8_t*)x)[base + i] * tin->scale;
        memcpy(mx, f, sizeof(float) * HW);
        for (int j = 0; j < C; j++)
            for (int l = 0; l < HW; l++)
                if (mx[l] < f[j * HW + l]) mx[l] = f[j * HW + l];
        memset(sum, 0, sizeof(float) * HW);
        for (int j = 0; j < C; j++)
            for (int l = 0; l < HW; l++)
            {
                o[j * HW + l] = exp(f[j * HW + l] - mx[l]);
                sum[l] += o[j * HW + l];
            }
        for (int j = 0; j < C; j++)
            for (int l = 0; l < HW; l++) o[j * HW + l] /= sum[l];
        for (size_t i = 0; i < (size_t)C * HW; i++)
        {
            if (u8)
            {
                int v = (int)(round(o[i] / tout->scale) + (uint8_t)tout->zero_point);
                if (v > 255) v = 255;
                else if (v < 0) v = 0;
                ((uint8_t*)y)[base + i] = (uint8_t)v;
            }
            else
            {
                int v = round(o[i] / tout->scale);
                if (v > 127) v = 127;
                else if (v < -127) v = -127;
                ((int8_t*)y)[base + i] = (int8_t)v;
            }
        }
    }
    free(f), free(o), free(mx), free(sum);
    return 0;
}

/* ---- run a whole layer list on host NCHW buffers (buffers[i] is tensor i; inputs filled by the caller) */
ORACLE_API int tb200_oracle_run(const tb200_tensor_desc* tensors, int num_tensors, const tb200_layer_desc* layers,
                                int num_layers, void* const* buffers, int uint8_mode)
{
    (void)num_tensors;
    for (int i = 0; i < num_layers; i++)
    {
        const tb200_layer_desc* L = &layers[i];
        const tb200_tensor_desc* tin = &tensors[L->inputs[0]];
        const tb200_tensor_desc* tout = &tensors[L->output];
        const void* x = buffers[L->inputs[0]];
        void* y = buffers[L->output];
        const int u8 = tin->data_type == TB200_DT_UINT8;
        int rc = -1;
        switch (L->op)
        {
        case TB200_OP_CONV:
            rc = u8 ? tb200_oracle_conv_uint8(tin, x, tout, y, L, uint8_mode) : tb200_oracle_conv_int8(tin, x, tout, y, L);
            break;
        case TB200_OP_FC:
            rc = u8 ? tb200_oracle_fc_uint8(tin, x, tout, y, L, uint8_mode) : tb200_oracle_fc_int8(tin, x, tout, y, L);
            break;
        case TB200_OP_POOL:
            rc = u8 ? tb200_oracle_pool_uint8(tin, x, tout, y, L) : tb200_oracle_pool_int8(tin, x, tout, y, L);
            break;
        case TB200_OP_RELU:
            rc = u8 ? tb200_oracle_relu_uint8(tin, x, tout, y, L) : tb200_oracle_relu_int8(tin, x, tout, y, L);
            break;
        case TB200_OP_ELTWISE:
            rc = u8 ? tb200_oracle_eltwise_uint8(tin, x, &tensors[L->inputs[1]], buffers[L->inputs[1]], tout, y, L)
                    : tb200_oracle_eltwise_int8(tin, x, &tensors[L->inputs[1]], buffers[L->inputs[1]], tout, y, L);
            break;
        case TB200_OP_CONCAT:
        {
            const tb200_tensor_desc* tt[4];
            const void* xx[4];
            for (int k = 0; k < L->num_inputs; k++) tt[k] = &tensors[L->inputs[k]], xx[k] = buffers[L->inputs[k]];
            rc = tb200_oracle_concat(tt, xx, L->num_inputs, tout, y);
            break;
        }
        case TB200_OP_UPSAMPLE: rc = tb200_oracle_upsample(tin, x, tout, y, L); break;
        case TB200_OP_IDENTITY:
        case TB200_OP_RESHAPE: /* flatten/flatten_ref.c:49-83, reshape: the same bytes in NCHW order */
            memcpy(y, x, (size_t)tin->dims[0] * tin->dims[1] * tin->dims[2] * tin->dims[3]);
            rc = 0;
            break;
        case TB200_OP_SIGMOID: rc = tb200_oracle_sigmoid(tin, x, tout, y); break;
        case TB200_OP_HARDSWISH: rc = u8 ? tb200_oracle_hardswish_uint8(tin, x, tout, y) : -1; break;
        case TB200_OP_SOFTMAX: rc = (L->axis == 1) ? tb200_oracle_softmax(tin, x, tout, y) : -1; break;
        default: rc = -1;
        }
        if (rc != 0) return -(i + 1);
    }
    return 0;
}
