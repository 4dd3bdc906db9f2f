// common.cuh -- device-side numerics shared by every kernel of the H100 backend.
//
// The requantising epilogue reproduces the reference CPU device's float arithmetic operation for
// operation (no FMA contraction, IEEE division, C round() = half away from zero), so that int8 results are
// bit-identical to the reference and uint8 results differ only by the reference's own fp32 summation noise.
// Reference recipes (paths relative to source/device/cpu/op/):
//   HCL int8  : conv/x86/conv_kernel_x86.c:1827-1889, conv/x86/conv_dw_hcl_x86.c:198-262
//   REF int8  : conv/conv_kernel_ref_int8.c:136-171
//   HCL uint8 : conv/x86/conv_kernel_x86.c:1729-1791
//   REF uint8 : conv/conv_kernel_ref_uint8.c:157-186
//   FC int8   : fc/fc_ref.c:225,252      FC uint8 : fc/fc_ref.c:146-166
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tengine_b200.h"

namespace tb200 {

// Scalar epilogue parameters, passed by value to kernels (per-channel arrays stay in global memory).
struct EpiParams
{
    const int32_t* bias;  // [OCp]
    const float* w_scale; // [OCp]
    float in_scale, out_scale;
    float in_w_scale;     // uint8: s_in * s_w (per tensor), computed once on the host in fp32
    float bias_scale;     // uint8 FC: the bias tensor's own scale (fc_ref.c:141-146); == in_w_scale for convolutions
    int32_t in_zero, w_zero, out_zero;
    int32_t activation;
    int32_t recipe;
    int32_t is_uint8;
    int32_t fc_rounding;
    int32_t has_bias;
    // ---- fast path (see requant_fast) ----
    const float2* fast_par; // [OCp] int8: (M[oc] ~ s_in*s_w[oc]/s_out [FC: exactly the reference's requant scale], bias bits);
                            //       uint8: (the bias term in real units, exactly as the reference rounds it, 0)
    float fast_lo, fast_hi;   // clamp of t = f/s_out: activation and the +-127 / 0..255 saturation folded together
    float fast_flo, fast_fhi; // uint8: activation clamp in real units
    float fast_r;             // uint8: fl(1/s_out)
    int32_t fast_ok;          // 0: scales are degenerate, always take the exact path
    int32_t fuse_bias;        // int8 conv: the .y lanes of fast_par hold fl(bias*M) (a float) and t = fma((float)acc, M, .y)
    // int8 fast path: clamp in the integer domain on s16x2 pairs, q' = max(min(q + q_add, q_max), 0)  (one DPX instruction),
    // then bytes += q_byte_add (mod 256) for layers whose lower clamp is not 0.  See requant_fast4_i8.
    uint32_t q_add2, q_max2;  // the two constants replicated into both halfwords
    uint32_t q_byte_add;      // lower clamp (as a byte) replicated x4; 0 for ReLU-type layers
};

// C round(): half away from zero, exact for every float (CUDA's roundf is the exact, slow-path version).
__device__ __forceinline__ float round_half_away(float x) { return roundf(x); }

__device__ __forceinline__ float act_hcl(float f, int activation)
{
    if (activation == 0) f = (f < 0.f) ? 0.f : f;
    if (activation > 0)
    {
        f = (f < 0.f) ? 0.f : f;
        f = (f > 6.f) ? 6.f : f;
    }
    return f;
}

__device__ __forceinline__ float act_ref(float t, int activation)
{
    if (activation >= 0)
    {
        if (t < 0.f && activation != 1) t = 0.f;
        if (t > 1.f && activation == 1) t = 1.f;
        if (t > 6.f && activation == 6) t = 6.f;
        if (t < -1.f && activation == 1) t = -1.f;
    }
    return t;
}

// acc = exact integer dot product (int8: sum x*w; uint8: sum (x-zx)(w-zw) over in-bounds taps), WITHOUT bias.
// Returns the output byte (int8 bit pattern or uint8).
static __device__ __noinline__ int requant(int32_t acc, int oc, const EpiParams& e)
{
    const int32_t b = e.has_bias ? __ldg(e.bias + oc) : 0;
    if (!e.is_uint8)
    {
        const float s_w = __ldg(e.w_scale + oc);
        int q;
        if (e.fc_rounding)
        {
            // fc_ref.c:225 requant = (s_in*s_w)/s_out ; :252 roundf(acc_with_bias * requant)
            const float rq = __fdiv_rn(__fmul_rn(e.in_scale, s_w), e.out_scale);
            q = (int)roundf(__fmul_rn((float)(acc + b), rq));
        }
        else if (e.recipe == TB200_RECIPE_HCL)
        {
            float f = __fmul_rn(__fmul_rn((float)(acc + b), e.in_scale), s_w);
            f = act_hcl(f, e.activation);
            q = (int)round_half_away(__fdiv_rn(f, e.out_scale));
        }
        else
        {
            float f = __fmul_rn((float)(acc + b), __fmul_rn(e.in_scale, s_w));
            f = act_ref(f, e.activation);
            q = (int)round_half_away(__fdiv_rn(f, e.out_scale));
        }
        q = q > 127 ? 127 : q;
        q = q < -127 ? -127 : q;
        return q & 0xff;
    }
    else
    {
        float f = __fmul_rn((float)acc, e.in_w_scale);
        int q;
        if (e.fc_rounding)
        {
            // fc_ref.c:146,162: data = bias*bias_scale + sum ; roundf(data / s_out) + zp  (bias_scale: the bias tensor's scale)
            if (e.has_bias) f = __fadd_rn(f, __fmul_rn((float)b, e.bias_scale));
            q = (int)roundf(__fdiv_rn(f, e.out_scale)) + e.out_zero;
        }
        else
        {
            if (e.has_bias)
            {
                // conv_kernel_x86.c:1723,1740: bias * (s_in*s_w) ; conv_kernel_ref_uint8.c:94: (bias * s_in) * s_w
                const float bt = (e.recipe == TB200_RECIPE_HCL)
                                     ? __fmul_rn((float)b, e.in_w_scale)
                                     : __fmul_rn(__fmul_rn((float)b, e.in_scale), __ldg(e.w_scale + oc));
                f = __fadd_rn(f, bt);
            }
            f = (e.recipe == TB200_RECIPE_HCL) ? act_hcl(f, e.activation) : act_ref(f, e.activation);
            q = (int)round_half_away(__fdiv_rn(f, e.out_scale)) + e.out_zero;
        }
        q = q > 255 ? 255 : q;
        q = q < 0 ? 0 : q;
        return q;
    }
}

// Fast requantisation with an exactness guarantee.
//
// The reference rounds t_ref = fl(fl(fl(x*s_in)*s_w)/s_out) (three roundings) half away from zero.  The fast path forms
// t = fl(x*M) with M = fl(s_in*s_w/s_out computed in double): |t - t_ref| <= 5*2^-24*|t| < 4e-5 for |t| <= 256.
// Rounding t to nearest (magic-number add) therefore gives the reference's integer unless t lies within kTieEps of a
// half-integer; exactly those elements (about 2.4e-4 of them) are recomputed with the literal reference arithmetic
// (requant()).  Clamps commute with the monotone division/rounding, so activation and saturation are applied after the
// rounding, in the integer domain (|t| > 256 rounds to something beyond every clamp bound, so its larger absolute
// error is harmless; prerun proves |t| < 32000 for every reachable accumulator, else the layer takes the exact path).
// For FC the reference itself computes roundf(x*rq) and M = rq exactly, so t == t_ref.
//
// The epilogues are bound by the issue rate of integer / logic instructions, so the arithmetic is arranged to keep work off them:
//   * the float chain runs on the FMA pipe (channel pairs carried in one 64-bit value),
//   * both clamps + the zero point are ONE DPX instruction per channel pair (VIADDMNMX.S16x2.RELU),
//   * the tie guard is a 3-input FMNMX tree and one FSETP per 4 channels.
#define TB200_MAGIC 12582912.0f       // 1.5 * 2^23
#define TB200_MAGIC_BITS 0x4B400000   // its bit pattern: as_float(MAGIC_BITS + i) == MAGIC + i for |i| < 2^22
#ifndef TB200_TIE_EPS // (tools/build_nofix_lib.sh overrides it to measure what the rare path costs; never in the product build)
#define TB200_TIE_EPS 1.220703125e-4f // 2^-13
#endif

// ---- fp32 pairs in one 64-bit value (two lanes, each rounded to nearest like the scalar instruction) ----
__device__ __forceinline__ uint64_t f2_pack(float lo, float hi)
{
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void f2_unpack(uint64_t v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ void f2_unpack_bits(uint64_t v, uint32_t& lo, uint32_t& hi) { asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v)); }
__device__ __forceinline__ uint64_t f2_fma(uint64_t a, uint64_t b, uint64_t c)
{
    float a0, a1, b0, b1, c0, c1;
    f2_unpack(a, a0, a1), f2_unpack(b, b0, b1), f2_unpack(c, c0, c1);
    return f2_pack(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ uint64_t f2_mul(uint64_t a, uint64_t b)
{
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1), f2_unpack(b, b0, b1);
    return f2_pack(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t f2_add(uint64_t a, uint64_t b)
{
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1), f2_unpack(b, b0, b1);
    return f2_pack(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t f2_sub(uint64_t a, uint64_t b)
{
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1), f2_unpack(b, b0, b1);
    return f2_pack(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}

// Per-channel constants of four consecutive channels oc0..oc0+3 (oc0 % 4 == 0) in the arena's int8 layout: channel
// pairs interleaved so that (M0, M1) and (y0, y1) are register pairs after one 16-byte load:
//   fast_par as float4[OCp/2] : { M[2k], M[2k+1], y[2k], y[2k+1] },  y = fl(bias*M) (FUSE) or the bias bits (int32).
struct FastPar4
{
    float4 a, b; // channels (0,1) and (2,3)
};
__device__ __forceinline__ FastPar4 fast_par4_ldg(const EpiParams& e, int oc0)
{
    const float4* p = reinterpret_cast<const float4*>(e.fast_par) + (oc0 >> 1);
    FastPar4 f;
    f.a = __ldg(p), f.b = __ldg(p + 1);
    return f;
}

// Two channels: t (packed), r = t + MAGIC (packed), d = t - (r - MAGIC) (packed).
// MAGIC_ACC: the caller's accumulators were initialised with TB200_MAGIC_BITS (|sum| < 2^22 proven by the kernel's K),
// so the int->float conversion is one packed FADD on the FMA pipe instead of two I2FP on the ALU pipe.
template <bool FUSE, bool MAGIC_ACC>
__device__ __forceinline__ void requant_pair_i8(int32_t a0, int32_t a1, float m0, float m1, float y0, float y1, uint64_t& r, uint64_t& d)
{
    const uint64_t mg = f2_pack(TB200_MAGIC, TB200_MAGIC);
    if (!FUSE) a0 += __float_as_int(y0), a1 += __float_as_int(y1);
    const uint64_t x = MAGIC_ACC ? f2_sub(f2_pack(__int_as_float(a0), __int_as_float(a1)), mg) : f2_pack((float)a0, (float)a1);
    const uint64_t t = FUSE ? f2_fma(x, f2_pack(m0, m1), f2_pack(y0, y1)) : f2_mul(x, f2_pack(m0, m1));
    r = f2_add(t, mg);
    d = f2_sub(t, f2_sub(r, mg));
}

// Four consecutive channels -> one packed 32-bit word; `guard` is set when any of the four lies in the tie guard band
// (the caller then runs requant_fix_word on that word).  The returned bytes still need requant_byte_fix().
template <bool FUSE, bool MAGIC_ACC = false>
__device__ __forceinline__ uint32_t requant_fast4_i8(const int32_t (&acc)[4], const EpiParams& e, const FastPar4& f, bool& guard)
{
    uint64_t r01, d01, r23, d23;
    requant_pair_i8<FUSE, MAGIC_ACC>(acc[0], acc[1], f.a.x, f.a.y, f.a.z, f.a.w, r01, d01);
    requant_pair_i8<FUSE, MAGIC_ACC>(acc[2], acc[3], f.b.x, f.b.y, f.b.z, f.b.w, r23, d23);
    float d0, d1, d2, d3;
    f2_unpack(d01, d0, d1);
    f2_unpack(d23, d2, d3);
    guard = fmaxf(fmaxf(fabsf(d0), fabsf(d1)), fmaxf(fabsf(d2), fabsf(d3))) > (0.5f - TB200_TIE_EPS);
    uint32_t r0, r1, r2, r3;
    f2_unpack_bits(r01, r0, r1);
    f2_unpack_bits(r23, r2, r3);
    // low halfwords of MAGIC_BITS + q are q (|q| < 2^15): pair them, clamp both with one DPX op, pick the low bytes
    const uint32_t p01 = __viaddmin_s16x2_relu(__byte_perm(r0, r1, 0x5410), e.q_add2, e.q_max2);
    const uint32_t p23 = __viaddmin_s16x2_relu(__byte_perm(r2, r3, 0x5410), e.q_add2, e.q_max2);
    return __byte_perm(p01, p23, 0x6420);
}

// Eight consecutive channels, instruction order pinned stage by stage (asm volatile keeps its order): the four channel
// pairs advance through the dependent chain fma -> +MAGIC -> -MAGIC -> t-(..) together, so every instruction has three
// independent neighbours.  ptxas on its own schedules the chains one after the other, and with only four epilogue warps
// per scheduler the fixed-latency stalls then halve the issue rate (ncu: stall_wait 2.2 per issue).
// w0/w1: the two packed words (before requant_byte_fix); g0/g1: max |d| of each word for the tie guard.
template <bool FUSE>
__device__ __forceinline__ void requant_fast8_i8(const int32_t (&a)[8], const float4 (&p)[4], const EpiParams& e, uint32_t& w0, uint32_t& w1,
                                                 float& g0, float& g1)
{
    const uint64_t mg = f2_pack(TB200_MAGIC, TB200_MAGIC);
    uint64_t x[4], t[4], r[4], s[4], d[4];
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        const int32_t a0 = FUSE ? a[2 * k] : a[2 * k] + __float_as_int(p[k].z), a1 = FUSE ? a[2 * k + 1] : a[2 * k + 1] + __float_as_int(p[k].w);
        x[k] = f2_pack((float)a0, (float)a1);
    }
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        if (FUSE) t[k] = f2_fma(x[k], f2_pack(p[k].x, p[k].y), f2_pack(p[k].z, p[k].w));
        else t[k] = f2_mul(x[k], f2_pack(p[k].x, p[k].y));
    }
#pragma unroll
    for (int k = 0; k < 4; k++) r[k] = f2_add(t[k], mg);
#pragma unroll
    for (int k = 0; k < 4; k++) s[k] = f2_sub(r[k], mg);
#pragma unroll
    for (int k = 0; k < 4; k++) d[k] = f2_sub(t[k], s[k]);
    float dl[4], dh[4];
    uint32_t rl[4], rh[4];
#pragma unroll
    for (int k = 0; k < 4; k++) f2_unpack(d[k], dl[k], dh[k]), f2_unpack_bits(r[k], rl[k], rh[k]);
    g0 = fmaxf(fmaxf(fabsf(dl[0]), fabsf(dh[0])), fmaxf(fabsf(dl[1]), fabsf(dh[1])));
    g1 = fmaxf(fmaxf(fabsf(dl[2]), fabsf(dh[2])), fmaxf(fabsf(dl[3]), fabsf(dh[3])));
    uint32_t q[4];
#pragma unroll
    for (int k = 0; k < 4; k++) q[k] = __viaddmin_s16x2_relu(__byte_perm(rl[k], rh[k], 0x5410), e.q_add2, e.q_max2);
    w0 = __byte_perm(q[0], q[1], 0x6420), w1 = __byte_perm(q[2], q[3], 0x6420);
}

// bytes += q_byte_add (mod 256, no carries between bytes): only layers whose lower clamp is not 0 (warp-uniform test)
__device__ __forceinline__ uint32_t requant_byte_fix(uint32_t w, const EpiParams& e)
{
    if (e.q_byte_add)
    {
        const uint32_t c = e.q_byte_add;
        w = ((w & 0x7f7f7f7fu) + (c & 0x7f7f7f7fu)) ^ ((w ^ c) & 0x80808080u);
    }
    return w;
}

// Rare path for a guarded word (final bytes in `word`): re-derive which of the four elements sit in the guard band and
// replace exactly those bytes by the literal reference arithmetic.  `acc` are TRUE accumulators (no magic offset).
template <bool FUSE>
__device__ __noinline__ uint32_t requant_fix_word(uint32_t word, int32_t a0, int32_t a1, int32_t a2, int32_t a3, int oc0, const EpiParams& e)
{
    const FastPar4 f = fast_par4_ldg(e, oc0);
    const int32_t a[4] = {a0, a1, a2, a3};
    const float m[4] = {f.a.x, f.a.y, f.b.x, f.b.y}, y[4] = {f.a.z, f.a.w, f.b.z, f.b.w};
#pragma unroll
    for (int j = 0; j < 4; j++)
    {
        const float t = FUSE ? __fmaf_rn((float)a[j], m[j], y[j]) : __fmul_rn((float)(a[j] + __float_as_int(y[j])), m[j]);
        const float r = __fadd_rn(t, TB200_MAGIC);
        const float d = __fsub_rn(t, __fsub_rn(r, TB200_MAGIC));
        if (fabsf(d) > 0.5f - TB200_TIE_EPS)
        {
            const uint32_t q = (uint32_t)requant(a[j], oc0 + j, e) & 0xffu;
            word = (word & ~(0xffu << (8 * j))) | (q << (8 * j));
        }
    }
    return word;
}

// The same for the uint8 tensor-core layers, whose fast epilogue has the int8 form t = fl((float)a * M) with a = true accumulator +
// y[oc] (y: integer constant of the channel INCLUDING the bias, FastPar4 {M, M, y, y}): `a` are those sums.  Only the elements that
// really sit in the guard band go through the literal arithmetic (which wants the accumulator without the bias).  One call per
// guarded word: the four candidates are examined together, so the rare path costs one parameter load and usually one literal
// requantisation -- an epilogue warp that lingers here holds up its whole accumulator stage.
static __device__ __noinline__ uint32_t requant_fix_word_u8(uint32_t word, int32_t a0, int32_t a1, int32_t a2, int32_t a3, int oc0, int oc_limit, const EpiParams& e)
{
    const FastPar4 f = fast_par4_ldg(e, oc0);
    const int32_t a[4] = {a0, a1, a2, a3};
    const float m[4] = {f.a.x, f.a.y, f.b.x, f.b.y};
#pragma unroll
    for (int j = 0; j < 4; j++)
    {
        const float t = __fmul_rn((float)a[j], m[j]);
        const float r = __fadd_rn(t, TB200_MAGIC);
        const float d = __fsub_rn(t, __fsub_rn(r, TB200_MAGIC));
        if (fabsf(d) > 0.5f - TB200_TIE_EPS && oc0 + j < oc_limit)
        {
            const int32_t b = e.has_bias ? __ldg(e.bias + oc0 + j) : 0;
            const uint32_t q = (uint32_t)requant(a[j] - b, oc0 + j, e) & 0xffu;
            word = (word & ~(0xffu << (8 * j))) | (q << (8 * j));
        }
    }
    return word;
}

// ---- uint8 fast path (scalar; the uint8 chain has a float-domain activation clamp between two multiplies) ----
// One element: returns the bit pattern of r = t + MAGIC (low byte = the rounded, clamped integer) and ORs `bit` into
// `bad` when t is inside the tie guard band.
__device__ __forceinline__ uint32_t requant_fast_bits_u8(int32_t acc, const EpiParams& e, float m, uint32_t& bad, uint32_t bit)
{
    // f is bit-identical to the reference's (same operations); only the division is replaced by * fl(1/s_out)
    float f = __fadd_rn(__fmul_rn((float)acc, e.in_w_scale), m);
    f = fminf(fmaxf(f, e.fast_flo), e.fast_fhi);
    float t = __fmul_rn(f, e.fast_r);
    t = fminf(fmaxf(t, e.fast_lo), e.fast_hi);
    const float r = __fadd_rn(t, TB200_MAGIC);
    const float d = __fsub_rn(t, __fsub_rn(r, TB200_MAGIC));
    // bad |= bit when |d| > 0.5 - eps : one FSETP (|d| folds into the operand modifier) + one predicated LOP3
    asm("{\n\t.reg .pred p;\n\tsetp.gt.f32 p, %1, %2;\n\t@p or.b32 %0, %0, %3;\n\t}" : "+r"(bad) : "f"(fabsf(d)), "f"(0.5f - TB200_TIE_EPS), "r"(bit));
    return (uint32_t)__float_as_int(r) + (uint32_t)e.out_zero;
}

// Four consecutive channels -> one packed 32-bit word (3 PRMT).  `bad` receives bits (bit0 << j) for guarded elements.
__device__ __forceinline__ uint32_t requant_fast4_u8(const int32_t (&acc)[4], const EpiParams& e, const float (&m)[4], uint32_t& bad, uint32_t bit0)
{
    const uint32_t r0 = requant_fast_bits_u8(acc[0], e, m[0], bad, bit0);
    const uint32_t r1 = requant_fast_bits_u8(acc[1], e, m[1], bad, bit0 << 1);
    const uint32_t r2 = requant_fast_bits_u8(acc[2], e, m[2], bad, bit0 << 2);
    const uint32_t r3 = requant_fast_bits_u8(acc[3], e, m[3], bad, bit0 << 3);
    return __byte_perm(__byte_perm(r0, r1, 0x0040), __byte_perm(r2, r3, 0x0040), 0x5410);
}

// Replace byte j of `word` by the exact result (rare path: ~2.4e-4 of the elements).
__device__ __forceinline__ uint32_t requant_fix_byte(uint32_t word, int j, int32_t acc, int oc, const EpiParams& e)
{
    const uint32_t q = (uint32_t)requant(acc, oc, e) & 0xffu;
    return (word & ~(0xffu << (8 * j))) | (q << (8 * j));
}

// uint8 flavour of requant_fast8_i8: the reference's chain is f = fl(fl(acc*S) + bias_term), activation clip, q = round(f / s_out)
// + zero point, saturate.  f is formed with the reference's own two roundings (packed FMUL2 + FADD2); only the division is
// replaced by a multiplication with fl(1/s_out) (|t - t_ref| <= 3*2^-24*|t|); clip, zero point and saturation are one DPX
// instruction per channel pair after the rounding (q_add2 carries the zero point).  `a` are TRUE accumulators
// sum (x-zx)(w-zw); bt = the per-channel bias terms.
__device__ __forceinline__ void requant_fast8_u8(const int32_t (&a)[8], const float (&bt)[8], const EpiParams& e, uint32_t& w0, uint32_t& w1,
                                                 float& g0, float& g1)
{
    const uint64_t mg = f2_pack(TB200_MAGIC, TB200_MAGIC);
    const uint64_t S2 = f2_pack(e.in_w_scale, e.in_w_scale), R2 = f2_pack(e.fast_r, e.fast_r);
    uint64_t f[4], t[4], r[4], s[4], d[4];
#pragma unroll
    for (int k = 0; k < 4; k++) f[k] = f2_mul(f2_pack((float)a[2 * k], (float)a[2 * k + 1]), S2);
#pragma unroll
    for (int k = 0; k < 4; k++) f[k] = f2_add(f[k], f2_pack(bt[2 * k], bt[2 * k + 1]));
#pragma unroll
    for (int k = 0; k < 4; k++) t[k] = f2_mul(f[k], R2);
#pragma unroll
    for (int k = 0; k < 4; k++) r[k] = f2_add(t[k], mg);
#pragma unroll
    for (int k = 0; k < 4; k++) s[k] = f2_sub(r[k], mg);
#pragma unroll
    for (int k = 0; k < 4; k++) d[k] = f2_sub(t[k], s[k]);
    float dl[4], dh[4];
    uint32_t rl[4], rh[4];
#pragma unroll
    for (int k = 0; k < 4; k++) f2_unpack(d[k], dl[k], dh[k]), f2_unpack_bits(r[k], rl[k], rh[k]);
    g0 = fmaxf(fmaxf(fabsf(dl[0]), fabsf(dh[0])), fmaxf(fabsf(dl[1]), fabsf(dh[1])));
    g1 = fmaxf(fmaxf(fabsf(dl[2]), fabsf(dh[2])), fmaxf(fabsf(dl[3]), fabsf(dh[3])));
    uint32_t q[4];
#pragma unroll
    for (int k = 0; k < 4; k++) q[k] = __viaddmin_s16x2_relu(__byte_perm(rl[k], rh[k], 0x5410), e.q_add2, e.q_max2);
    w0 = __byte_perm(q[0], q[1], 0x6420), w1 = __byte_perm(q[2], q[3], 0x6420);
}

// 16 channels of one uint8 output row: acc = TRUE accumulators, par = (bias term, -) per channel as loaded from the arena layout
// float2[OCp].  Returns the four packed words; pad lanes (oc0 + k >= oc_limit) come out 0.
__device__ __forceinline__ void requant_unit16_u8(const int32_t (&acc)[16], const float (&bt)[16], int oc0, int oc_limit, const EpiParams& e,
                                                  uint32_t (&w)[4])
{
    float gw[4];
#pragma unroll
    for (int h = 0; h < 2; h++)
    {
        const int32_t a8[8] = {acc[h * 8], acc[h * 8 + 1], acc[h * 8 + 2], acc[h * 8 + 3], acc[h * 8 + 4], acc[h * 8 + 5], acc[h * 8 + 6], acc[h * 8 + 7]};
        const float b8[8] = {bt[h * 8], bt[h * 8 + 1], bt[h * 8 + 2], bt[h * 8 + 3], bt[h * 8 + 4], bt[h * 8 + 5], bt[h * 8 + 6], bt[h * 8 + 7]};
        requant_fast8_u8(a8, b8, e, w[2 * h], w[2 * h + 1], gw[2 * h], gw[2 * h + 1]);
    }
    if (e.q_byte_add)
    {
#pragma unroll
        for (int j = 0; j < 4; j++) w[j] = requant_byte_fix(w[j], e);
    }
    if (fmaxf(fmaxf(gw[0], gw[1]), fmaxf(gw[2], gw[3])) > 0.5f - TB200_TIE_EPS)
    {
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (gw[j] > 0.5f - TB200_TIE_EPS)
            {
#pragma unroll
                for (int t = 0; t < 4; t++) w[j] = requant_fix_byte(w[j], t, acc[j * 4 + t], oc0 + j * 4 + t, e);
            }
    }
    if (oc0 + 16 > oc_limit)
    {
        // pad lanes of uint8 tensors hold 0, not the zero point
#pragma unroll
        for (int k = 0; k < 16; k++)
            if (oc0 + k >= oc_limit) w[k >> 2] &= ~(0xffu << (8 * (k & 3)));
    }
}

// Generic entry for kernels that handle one word (4 channels oc0..oc0+3) at a time with constants in global memory.
// Pad channels (>= oc_limit) have m = 0, y = 0 in fast_par and therefore produce 0.
template <bool U8>
__device__ __forceinline__ uint32_t requant_word(const int32_t (&acc)[4], int oc0, int oc_limit, const EpiParams& e)
{
    if (!e.fast_ok)
    {
        uint32_t w = 0;
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (oc0 + j < oc_limit) w |= ((uint32_t)requant(acc[j], oc0 + j, e) & 0xffu) << (8 * j);
        return w;
    }
    if (!U8)
    {
        const FastPar4 f = fast_par4_ldg(e, oc0);
        bool guard;
        uint32_t w = e.fuse_bias ? requant_fast4_i8<true>(acc, e, f, guard) : requant_fast4_i8<false>(acc, e, f, guard);
        w = requant_byte_fix(w, e); // pad channels: M = y = 0 -> q = 0 -> byte 0 (0 lies inside every clamp range)
        if (guard) w = e.fuse_bias ? requant_fix_word<true>(w, acc[0], acc[1], acc[2], acc[3], oc0, e) : requant_fix_word<false>(w, acc[0], acc[1], acc[2], acc[3], oc0, e);
        return w;
    }
    float m[4];
#pragma unroll
    for (int j = 0; j < 4; j++) m[j] = __ldg(e.fast_par + oc0 + j).x;
    uint32_t bad = 0;
    uint32_t w = requant_fast4_u8(acc, e, m, bad, 1u);
    // pad lanes of uint8 tensors must hold 0 (not the zero point): mask them
#pragma unroll
    for (int j = 0; j < 4; j++)
        if (oc0 + j >= oc_limit) w &= ~(0xffu << (8 * j)), bad &= ~(1u << j);
    if (bad)
    {
#pragma unroll
        for (int j = 0; j < 4; j++)
            if ((bad >> j) & 1u) w = requant_fix_byte(w, j, acc[j], oc0 + j, e);
    }
    return w;
}

__device__ __forceinline__ int dp4a_s8(int a, int b, int c) { return __dp4a(a, b, c); }
__device__ __forceinline__ unsigned dp4a_u8(unsigned a, unsigned b, unsigned c) { return __dp4a(a, b, c); }

static inline int cpad(int c) { return (c + 15) & ~15; }

} // namespace tb200
