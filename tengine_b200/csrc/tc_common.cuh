// tc_common.cuh -- device helpers shared by the tensor-core kernels (gemm_tcgen05.cu, conv_window.cu): wgmma shared-memory
// descriptors, the accumulator image, the SW32 tile addressing of the thread-built A tiles, the requantising row unit.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace tb200 {

static constexpr int BLOCK_M = 128;

// K-major operand tile in shared memory, rows of `swizzle` bytes, 8-row groups `8*swizzle` bytes apart: the wgmma matrix
// descriptor (PTX ISA "Matrix Descriptor Format" for sm_90a: start >> 4, leading byte offset >> 4 (unused for swizzled K-major),
// stride byte offset >> 4, base offset 0 (tiles are aligned to the swizzle repeat), layout 1 = 128B, 2 = 64B, 3 = 32B swizzle).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, int swizzle)
{
    const uint64_t layout = (swizzle == 128) ? 1ull : (swizzle == 64) ? 2ull : 3ull;
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(((8 * swizzle) >> 4) & 0x3fff) << 32;
    d |= layout << 62;
    return d;
}

// bytes of one row of an accumulator image of `cols` s32 columns (16 bytes of padding: the epilogue's 16-byte row loads of
// 32 consecutive rows then hit distinct banks)
__host__ __device__ inline uint32_t acc_pitch(int cols) { return (uint32_t)cols * 4u + 16u; }

// The CTA's first warpgroup: D[128 x ncols] = sum over nkb k-blocks of A[128 x swizzle] . B[ncols x swizzle]^T into the
// accumulator image.  Operands are K-major swizzled tiles (A: 128 rows, B: ncols rows; one tile per k-block, a_kb / b_kb bytes
// apart).  The two 64-row halves and column groups of at most 128 run one after the other so that the fragment stays at 64
// registers.  The image is complete for the warpgroup when this returns; other threads need a barrier.
template <bool AU, bool BU>
__device__ __forceinline__ void wg_mma_to_image(uint32_t sA, uint32_t a_kb, uint32_t sB, uint32_t b_kb, int nkb, int swizzle, int ncols,
                                                uint32_t img, uint32_t pitch)
{
    const int nch = ncols >> 4, ksteps = swizzle >> 5;
    for (int mh = 0; mh < 2; mh++)
        for (int c0 = 0; c0 < nch; c0 += 8)
        {
            uint32_t acc[8][8];
#pragma unroll
            for (int j = 0; j < 8; j++)
#pragma unroll
                for (int r = 0; r < 8; r++) acc[j][r] = 0;
            wgmma_fence();
            for (int kb = 0; kb < nkb; kb++)
            {
                const uint64_t da = make_smem_desc(sA + (uint32_t)kb * a_kb + (uint32_t)(mh * 64 * swizzle), swizzle);
                const uint64_t db = make_smem_desc(sB + (uint32_t)kb * b_kb + (uint32_t)(c0 * 16 * swizzle), swizzle);
                for (int k = 0; k < ksteps; k++)
#pragma unroll
                    for (int j = 0; j < 8; j++)
                        // +32 bytes along K inside the swizzled rows: +2 in 16-byte units; +16 rows of B: +16*swizzle bytes
                        if (c0 + j < nch) wgmma_n16<AU, BU>(acc[j], da + (uint64_t)(k * 2), db + (uint64_t)(j * swizzle + k * 2), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < 8; j++)
                if (c0 + j < nch) frag_to_image(acc[j], img, pitch, mh * 64, (c0 + j) * 16);
        }
}

// Requantise accumulator columns oc0..oc0+15 of one row (v) into four output words.  par_addr: the 16 channels' epilogue
// constants in shared memory, 8 bytes each (unused by int8 MODE 2).  oc: real channels; pad channels come out 0.
// MODE: 0 fast, 1 fast + fused bias (int8), 2 exact.  U8: uint8 layers in the int8 form (engine.cu: constants {M, M, y, y} with
// y = corr[oc] + bias[oc]): a' = v + rowc + y, t = fl(a' * M), where rowc = -zw * sum(x) of the row; int8 ignores rowc.
template <int MODE, bool U8>
__device__ __forceinline__ void tc_unit16(const uint32_t (&v)[16], int32_t rowc, uint32_t par_addr, int oc0, int oc, const EpiParams& e,
                                          uint32_t (&w)[4])
{
    if (MODE == 2)
    {
#pragma unroll
        for (int k = 0; k < 16; k++)
        {
            if ((k & 3) == 0) w[k >> 2] = 0;
            if (oc0 + k < oc)
            {
                int32_t acc = (int32_t)v[k];
                if (U8)
                {
                    const float4 pp = lds_f4(par_addr + (k >> 1) * 16);
                    acc += rowc + __float_as_int((k & 1) ? pp.w : pp.z) - (e.has_bias ? __ldg(e.bias + oc0 + k) : 0);
                }
                w[k >> 2] |= ((uint32_t)requant(acc, oc0 + k, e) & 0xffu) << (8 * (k & 3));
            }
        }
        return;
    }
    constexpr bool FUSE = !U8 && MODE == 1;
    float gw[4];
#pragma unroll
    for (int h = 0; h < 2; h++)
    {
        FastPar4 p[2];
#pragma unroll
        for (int k = 0; k < 2; k++) p[k].a = lds_f4(par_addr + h * 64 + k * 32), p[k].b = lds_f4(par_addr + h * 64 + k * 32 + 16);
        int32_t a8[2][4];
#pragma unroll
        for (int k = 0; k < 8; k++) a8[k >> 2][k & 3] = (int32_t)v[h * 8 + k] + (U8 ? rowc : 0);
        uint32_t w2[2];
        float g2[2];
        requant_fast_words_i8<FUSE, 2, 2>(a8, p, e, w2, g2);
        w[2 * h] = w2[0], w[2 * h + 1] = w2[1], gw[2 * h] = g2[0], gw[2 * h + 1] = g2[1];
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
                if (U8)
                {
                    int32_t at[4]; // accumulator + y of the word's four channels (what the fast path multiplied by M)
#pragma unroll
                    for (int t = 0; t < 4; t++)
                    {
                        const float4 pp = lds_f4(par_addr + ((j * 4 + t) >> 1) * 16);
                        at[t] = (int32_t)v[j * 4 + t] + rowc + __float_as_int((t & 1) ? pp.w : pp.z);
                    }
                    w[j] = requant_fix_word_u8(w[j], at[0], at[1], at[2], at[3], oc0 + j * 4, oc, e);
                }
                else
                    w[j] = requant_fix_word<FUSE>(w[j], (int32_t)v[j * 4], (int32_t)v[j * 4 + 1], (int32_t)v[j * 4 + 2], (int32_t)v[j * 4 + 3],
                                                  oc0 + j * 4, e);
            }
    }
    if (U8 && oc0 + 16 > oc)
    {
        // pad lanes of uint8 tensors hold 0, not the zero point
#pragma unroll
        for (int k = 0; k < 16; k++)
            if (oc0 + k >= oc) w[k >> 2] &= ~(0xffu << (8 * (k & 3)));
    }
}

// row r, 16-byte chunk c16 of a SW32 K-major tile (8-row groups of 256 bytes, chunk index ^= bit 2 of the row)
__device__ __forceinline__ uint32_t sw32_offset(int r, int c16) { return (uint32_t)((r >> 3) * 256 + (r & 7) * 32 + ((c16 ^ ((r >> 2) & 1)) << 4)); }


} // namespace tb200
