// dw_tma.cu -- depthwise 3x3 int8 (stride 1 / 2), the MobileNet depthwise path, with TMA-staged input tiles.
//
// One CTA = 32 channels x R output rows x up to 128/R... output pixels: ONE elected thread issues ONE 4-D
// cp.async.bulk.tensor load (box = 32 channels x cols x rows x 1 image; out-of-bounds coordinates are zero-filled by
// the TMA unit, which IS the convolution's zero padding), everybody waits on the mbarrier, then each thread computes
// 4 channels x TW consecutive output pixels from shared memory with one dp4a per MAC (one-hot weight bytes) and the
// fused requantising epilogue.  No per-thread global loads, no boundary predicates, every input byte crosses L2->SM
// once per CTA.  Several CTAs per SM overlap one CTA's TMA latency with the others' arithmetic.
// Takes the role of convdw3x3s1_int8_sse / convdw3x3s2_int8_sse (source/device/cpu/op/conv/x86/conv_dw_hcl_x86.c:97-445).
#include "common.cuh"
#include "kernels.h"
#include "ptx.cuh"

#include <cstdio>
#include <cstdlib>

namespace tb200 {

static constexpr int DW_THREADS = 128;
static constexpr int DW_CH = 32; // channels per CTA (8 words)
#ifndef TB200_DW_MIN_CTAS
#define TB200_DW_MIN_CTAS 6
#endif
static constexpr int DW_MIN_CTAS = TB200_DW_MIN_CTAS; // 6 caps the kernels at 80 registers and spills (ptxas: 32-byte stack)

// Fused epilogue of both kernels: TW pixels x 4 channels per thread.  The accumulators were initialised with
// TB200_MAGIC_BITS (|sum of 9 products| < 2^22), so the int->float conversion is a packed FADD on the FMA pipe
// (common.cuh requant_pair_i8<.., MAGIC_ACC>): the ALU pipe, which also carries this kernel's PRMTs, is the busy one.
template <int TW>
__device__ __forceinline__ void dw_epilogue(int (&acc)[TW][4], const FastPar4& f, int c4, int ow0, uint8_t* orow, const ConvShape& s,
                                            const EpiParams& e)
{
    uint32_t w[TW];
    if (!e.fast_ok || !e.fuse_bias)
    {
        // exact path, or a bias too large to fold into the FMA: true accumulators, generic per-word routine
#pragma unroll
        for (int t = 0; t < TW; t++)
        {
#pragma unroll
            for (int j = 0; j < 4; j++) acc[t][j] -= TB200_MAGIC_BITS;
            w[t] = requant_word<false>(acc[t], c4 * 4, s.oc, e);
        }
    }
    else
    {
        bool gd[TW], any = false;
#pragma unroll
        for (int t = 0; t < TW; t++)
        {
            w[t] = requant_fast4_i8<true, true>(acc[t], e, f, gd[t]);
            any |= gd[t];
        }
        if (e.q_byte_add)
        {
#pragma unroll
            for (int t = 0; t < TW; t++) w[t] = requant_byte_fix(w[t], e);
        }
        if (any)
        {
#pragma unroll
            for (int t = 0; t < TW; t++)
                if (gd[t])
                    w[t] = requant_fix_word<true>(w[t], acc[t][0] - TB200_MAGIC_BITS, acc[t][1] - TB200_MAGIC_BITS, acc[t][2] - TB200_MAGIC_BITS,
                                                  acc[t][3] - TB200_MAGIC_BITS, c4 * 4, e);
        }
    }
#pragma unroll
    for (int t = 0; t < TW; t++)
        if (ow0 + t < s.ow) reinterpret_cast<unsigned*>(orow + (size_t)t * s.ocp)[c4] = w[t];
}

template <int TW, int S>
__global__ void __launch_bounds__(DW_THREADS, DW_MIN_CTAS)
    conv_dw3x3_tma_kernel(const __grid_constant__ CUtensorMap tmap_in, const uint8_t* __restrict__ wgt, uint8_t* __restrict__ out,
                          const ConvShape s, const __grid_constant__ EpiParams e, const int rows_per_cta, const int gpr, const int tile_cols,
                          const int tile_rows)
{
    extern __shared__ __align__(128) uint8_t dw_smem[];
    __shared__ __align__(8) uint64_t bar;
    const int chunk = blockIdx.x;           // 32-channel chunk
    const int oh0 = blockIdx.y * rows_per_cta;
    const int n = blockIdx.z;
    const int word = threadIdx.x & 7;       // 4-channel word inside the chunk
    const int pg = threadIdx.x >> 3;        // pixel group 0..15
    const int r = pg / gpr, gi = pg - r * gpr;
    const int oh = oh0 + r, ow0 = gi * TW;
    const int c4 = chunk * 8 + word;        // word index in the full channel dimension

    if (threadIdx.x == 0)
    {
        mbar_init(&bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0)
    {
        mbar_expect_tx(&bar, (uint32_t)(tile_rows * tile_cols * DW_CH));
        tma_load_4d(&tmap_in, &bar, dw_smem, chunk * DW_CH, -s.pw0, oh0 * S - s.ph0, n);
    }
    // weights / epilogue constants while the tile is in flight
    const bool active = (r < rows_per_cta) && (oh < s.oh) && (ow0 < s.ow) && (c4 * 4 < s.cp);
    int wj[9][4];
    FastPar4 fp;
    fp.a = fp.b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (active)
    {
#pragma unroll
        for (int t = 0; t < 9; t++)
        {
            const unsigned wv = __ldg(reinterpret_cast<const unsigned*>(wgt + (size_t)t * s.cp) + c4);
#pragma unroll
            for (int j = 0; j < 4; j++) wj[t][j] = (int)(wv & (0xffu << (8 * j)));
        }
        if (e.fast_ok) fp = fast_par4_ldg(e, c4 * 4);
    }
    mbar_wait(&bar, 0);
    if (!active) return;

    int acc[TW][4];
#pragma unroll
    for (int t = 0; t < TW; t++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[t][j] = TB200_MAGIC_BITS;
    constexpr int COLS = (TW - 1) * S + 3;
    const uint32_t base = smem_u32(dw_smem) + (uint32_t)(((r * S) * tile_cols + ow0 * S) * DW_CH + word * 4);
#pragma unroll
    for (int kh = 0; kh < 3; kh++)
    {
        int xv[COLS];
#pragma unroll
        for (int col = 0; col < COLS; col++)
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(xv[col]) : "r"(base + (uint32_t)((kh * tile_cols + col) * DW_CH)));
#pragma unroll
        for (int t = 0; t < TW; t++)
#pragma unroll
            for (int kw = 0; kw < 3; kw++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[t][j] = dp4a_s8(xv[t * S + kw], wj[kh * 3 + kw][j], acc[t][j]);
    }

    uint8_t* orow = out + (((size_t)n * s.oh + oh) * s.ow + ow0) * s.ocp;
    dw_epilogue<TW>(acc, fp, c4, ow0, orow, s, e);
}

// ---- stride-1 variant with three taps per dp4a ---------------------------------------------------------------
// The dp4a / IMAD pipe is the busiest unit of the kernel above (9 dp4a per output).  Here each row of the window is
// byte-transposed in registers (4 pixels x 4 channels -> 4 channel words, 8 PRMT on the ALU pipe), so that one dp4a
// multiplies THREE horizontally adjacent taps of one channel: 3 dp4a + ~4.5 PRMT per output instead of 9 dp4a.
__device__ __forceinline__ void transpose4x4(unsigned x0, unsigned x1, unsigned x2, unsigned x3, unsigned (&ch)[4])
{
    const unsigned t0 = __byte_perm(x0, x1, 0x5140), t1 = __byte_perm(x2, x3, 0x5140); // [a0 b0 a1 b1] [c0 d0 c1 d1]
    const unsigned t2 = __byte_perm(x0, x1, 0x7362), t3 = __byte_perm(x2, x3, 0x7362); // [a2 b2 a3 b3] [c2 d2 c3 d3]
    ch[0] = __byte_perm(t0, t1, 0x5410), ch[1] = __byte_perm(t0, t1, 0x7632);
    ch[2] = __byte_perm(t2, t3, 0x5410), ch[3] = __byte_perm(t2, t3, 0x7632);
}

__global__ void __launch_bounds__(DW_THREADS, DW_MIN_CTAS)
    conv_dw3x3_tma_pack3_kernel(const __grid_constant__ CUtensorMap tmap_in, const uint8_t* __restrict__ wgt, uint8_t* __restrict__ out,
                                const ConvShape s, const __grid_constant__ EpiParams e, const int rows_per_cta, const int gpr,
                                const int tile_cols, const int tile_rows)
{
    constexpr int TW = 8;
    extern __shared__ __align__(128) uint8_t dw_smem[];
    __shared__ __align__(8) uint64_t bar;
    const int chunk = blockIdx.x;
    const int oh0 = blockIdx.y * rows_per_cta;
    const int n = blockIdx.z;
    const int word = threadIdx.x & 7;
    const int pg = threadIdx.x >> 3;
    const int r = pg / gpr, gi = pg - r * gpr;
    const int oh = oh0 + r, ow0 = gi * TW;
    const int c4 = chunk * 8 + word;

    if (threadIdx.x == 0)
    {
        mbar_init(&bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0)
    {
        mbar_expect_tx(&bar, (uint32_t)(tile_rows * tile_cols * DW_CH));
        tma_load_4d(&tmap_in, &bar, dw_smem, chunk * DW_CH, -s.pw0, oh0 - s.ph0, n);
    }
    const bool active = (r < rows_per_cta) && (oh < s.oh) && (ow0 < s.ow) && (c4 * 4 < s.cp);
    unsigned wr[3][4]; // per filter row and channel: [w(kh,0), w(kh,1), w(kh,2), 0]
    FastPar4 fp;
    fp.a = fp.b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (active)
    {
#pragma unroll
        for (int kh = 0; kh < 3; kh++)
        {
            const unsigned w0 = __ldg(reinterpret_cast<const unsigned*>(wgt + (size_t)(kh * 3 + 0) * s.cp) + c4);
            const unsigned w1 = __ldg(reinterpret_cast<const unsigned*>(wgt + (size_t)(kh * 3 + 1) * s.cp) + c4);
            const unsigned w2 = __ldg(reinterpret_cast<const unsigned*>(wgt + (size_t)(kh * 3 + 2) * s.cp) + c4);
            unsigned tr[4];
            transpose4x4(w0, w1, w2, 0u, tr);
#pragma unroll
            for (int j = 0; j < 4; j++) wr[kh][j] = tr[j];
        }
        if (e.fast_ok) fp = fast_par4_ldg(e, c4 * 4);
    }
    mbar_wait(&bar, 0);
    if (!active) return;

    int acc[TW][4];
#pragma unroll
    for (int t = 0; t < TW; t++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[t][j] = TB200_MAGIC_BITS;
    const uint32_t base = smem_u32(dw_smem) + (uint32_t)((r * tile_cols + ow0) * DW_CH + word * 4);
#pragma unroll
    for (int kh = 0; kh < 3; kh++)
    {
        unsigned xv[10];
#pragma unroll
        for (int col = 0; col < 10; col++)
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(xv[col]) : "r"(base + (uint32_t)((kh * tile_cols + col) * DW_CH)));
        unsigned pa[4], pb[4];
        transpose4x4(xv[0], xv[1], xv[2], xv[3], pa); // channel j: pixels 0..3
        transpose4x4(xv[4], xv[5], xv[6], xv[7], pb); // channel j: pixels 4..7
        const unsigned u0 = __byte_perm(xv[8], xv[9], 0x5140); // [i0 j0 i1 j1] (pixels 8, 9; channels 0, 1)
        const unsigned u1 = __byte_perm(xv[8], xv[9], 0x7362); // [i2 j2 i3 j3]
#pragma unroll
        for (int j = 0; j < 4; j++)
        {
            const unsigned w = wr[kh][j];
            const unsigned uu = (j < 2) ? u0 : u1;
            const unsigned s6 = (j & 1) ? 0x0632u : 0x0432u; // [P1.b2, P1.b3, pix8, -]
            const unsigned s7 = (j & 1) ? 0x0763u : 0x0543u; // [P1.b3, pix8, pix9, -]
            acc[0][j] = dp4a_s8((int)pa[j], (int)w, acc[0][j]);
            acc[1][j] = dp4a_s8((int)__byte_perm(pa[j], pb[j], 0x4321), (int)w, acc[1][j]);
            acc[2][j] = dp4a_s8((int)__byte_perm(pa[j], pb[j], 0x5432), (int)w, acc[2][j]);
            acc[3][j] = dp4a_s8((int)__byte_perm(pa[j], pb[j], 0x6543), (int)w, acc[3][j]);
            acc[4][j] = dp4a_s8((int)pb[j], (int)w, acc[4][j]);
            acc[5][j] = dp4a_s8((int)(pb[j] >> 8), (int)w, acc[5][j]);
            acc[6][j] = dp4a_s8((int)__byte_perm(pb[j], uu, s6), (int)w, acc[6][j]);
            acc[7][j] = dp4a_s8((int)__byte_perm(pb[j], uu, s7), (int)w, acc[7][j]);
        }
    }

    uint8_t* orow = out + (((size_t)n * s.oh + oh) * s.ow + ow0) * s.ocp;
    dw_epilogue<TW>(acc, fp, c4, ow0, orow, s, e);
}

// Plan: tile geometry + the 4-D tensor map (C, W, H, N) of the input.  Returns 0, or <0 when this layer must use the
// generic depthwise kernel (uint8, stride > 2, very wide rows ...).
int dw_plan_create(DwPlan* p, const void* in, const ConvShape& s, const EpiParams& e)
{
    p->valid = 0;
    if (e.is_uint8 || s.kh != 3 || s.kw != 3 || s.dh != 1 || s.dw != 1 || s.sh != s.sw || (s.sh != 1 && s.sh != 2)) return -1;
    const int S = s.sh;
    p->tw = (S == 1) ? 8 : 4;
    p->gpr = (s.ow + p->tw - 1) / p->tw;
    if (p->gpr > 16) return -1; // rows wider than 16 pixel groups: generic kernel
    p->rows_per_cta = 16 / p->gpr;
    if (p->rows_per_cta > s.oh) p->rows_per_cta = s.oh;
    p->tile_cols = (p->gpr * p->tw - 1) * S + 3;
    p->tile_rows = (p->rows_per_cta - 1) * S + 3;
    if (p->tile_cols > 256 || p->tile_rows > 256) return -1;
    p->smem_bytes = p->tile_rows * p->tile_cols * DW_CH;
    if (p->smem_bytes > 48 * 1024) return -1;
    const uint64_t dims[4] = {(uint64_t)s.cp, (uint64_t)s.w, (uint64_t)s.h, (uint64_t)s.n};
    const uint64_t strides[3] = {(uint64_t)s.cp, (uint64_t)s.w * s.cp, (uint64_t)s.h * s.w * s.cp};
    const uint32_t box[4] = {(uint32_t)DW_CH, (uint32_t)p->tile_cols, (uint32_t)p->tile_rows, 1u};
    if (tmap_encode(p->tmap_in, in, 4, dims, strides, box, nullptr, 0) != 0) return -2;
    p->valid = 1;
    return 0;
}

cudaError_t launch_conv_dw_tma(const DwPlan& p, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st)
{
    dim3 grid((s.cp + DW_CH - 1) / DW_CH, (s.oh + p.rows_per_cta - 1) / p.rows_per_cta, s.n);
    CUtensorMap tm;
    memcpy(&tm, p.tmap_in, sizeof tm);
    // not templated on the epilogue: MODE is the run-time choice of the same rule as the other launchers (2 = exact)
    if (debug_launch())
        fprintf(stderr, "tengine_b200: launch %s MODE=%d\n", s.sh == 1 ? "conv_dw3x3_tma_pack3_kernel" : "conv_dw3x3_tma_kernel<4,2>",
                !e.fast_ok ? 2 : (!e.is_uint8 && e.fuse_bias ? 1 : 0));
    if (s.sh == 1)
        conv_dw3x3_tma_pack3_kernel<<<grid, DW_THREADS, p.smem_bytes, st>>>(tm, (const uint8_t*)w, (uint8_t*)out, s, e, p.rows_per_cta, p.gpr,
                                                                           p.tile_cols, p.tile_rows);
    else
        conv_dw3x3_tma_kernel<4, 2><<<grid, DW_THREADS, p.smem_bytes, st>>>(tm, (const uint8_t*)w, (uint8_t*)out, s, e, p.rows_per_cta, p.gpr,
                                                                            p.tile_cols, p.tile_rows);
    return cudaGetLastError();
}

} // namespace tb200
