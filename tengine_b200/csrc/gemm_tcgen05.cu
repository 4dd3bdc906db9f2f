// gemm_tcgen05.cu -- int8 x int8 -> int32 GEMM on the Hopper tensor cores (wgmma.mma_async .s32.s8/.u8, m64nNk32, N = block_n)
// with TMA-staged operands, a shared-memory accumulator image and the fused requantising epilogue.
//
//   out[m][oc] = requant( sum_k A[m][k] * B[oc][k] ),   A = NHWC activations (row = pixel, K = padded Cin),
//                                                        B = pre-packed weights [OCp][K], both K-major.
// This is the device's form of the reference's im2col + sgemm_i8 + sgemm_int8 epilogue for 1x1 convolutions
// (source/device/cpu/op/conv/x86/conv_kernel_x86.c:187-242, 1008-1631, 1796-1893) and of ref_fc_int8
// (fc/fc_ref.c:209-297): with NHWC activations a 1x1 convolution IS this GEMM, no im2col pass exists.
//
// Structure (one persistent CTA per SM, 512 threads = four warpgroups, int8 and uint8 alike):
//   WG0, warp 0   : TMA producer  (cp.async.bulk.tensor.2d -> 128B/64B/32B-swizzled smem ring, mbarrier expect_tx)
//   WG0, warps 1-2: uint8 only: the row sums sum(x) of every A tile (idle for int8); warp 3 idle
//   WG1, warps 4-7: MMA.  One accumulator stage (mt m-tiles x block_n columns) in registers: per m-tile and k-step two
//                   m64n<block_n>k32, rows 0-63 and 64-127; one commit group in flight, a ring stage is released when the
//                   group after it has been committed and the one reading it has completed.  At the end of the stage the
//                   fragments go into the accumulator image ([128 rows][mt * block_n] s32 in shared memory) as soon as the
//                   epilogue has read the previous stage out of it (mbarriers img_empty / img_full).
//   WG2-3, warps 8-15: epilogue.  Two warps per 32-row quarter of the image; a warp owns whole "store groups" = 32 rows x
//                   16/32 channels: image -> registers -> requant_fast4_i8 -> bytes -> its own swizzled smem buffer -> ONE
//                   TMA store per group (cp.async.bulk.tensor, double-buffered).  No address arithmetic for the stores,
//                   rows outside the tensor are clipped by the TMA unit.
// So the tensor cores multiply stage s+1 while the epilogue requantises stage s: the registers are the second accumulator
// buffer.  Registers per thread (setmaxnreg): WG0 40, MMA 200 (at most 128 accumulators), epilogue 136.
// The producer runs ahead through the ring, so the next tile's operands are resident when its MMAs start.  K is small
// (32..1024), so these layers are bound by the epilogue's ALU-pipe issue rate, not by the tensor pipe: see common.cuh
// (requant_fast4_i8) for the instruction budget.
#include <cuda.h>

#include "common.cuh"
#include "kernels.h"
#include "ptx.cuh"
#include "tc_common.cuh"

#include <cstdio>
#include <cstdlib>

namespace tb200 {

#ifdef TB200_GEMM_TIMELINE
#define TLOG_E(tag) do { if (lane == 0 && (warp == EPI_WARP0 || warp == 15)) tlog(warp == EPI_WARP0 ? 2 : 3, tag); } while (0)
#else
#define TLOG_E(tag) do { } while (0)
#endif


// warp roles (four warpgroups, int8 and uint8 alike)
static constexpr int GEMM_THREADS = 512;
static constexpr int PRODUCER_WARP = 0;
static constexpr int SUM_WARP0 = 1, SUM_WARPS = 2; // uint8 kernels only: two warps that add up the rows of every A tile (sum x)
static constexpr int MMA_THREAD0 = 128;            // the MMA warpgroup: threads 128..255
static constexpr int EPI_WARP0 = 8, EPI_WARPS = 8; // two epilogue warpgroups; two warps per 32-row quarter of the accumulator image
static constexpr int EPI_THREAD0 = EPI_WARP0 * 32, EPI_THREADS = EPI_WARPS * 32;
// registers per thread of each role (setmaxnreg): the kernel launches with 128 (512 threads, the 64 K registers of the SM); WG0
// gives registers back, the MMA warpgroup (up to 128 accumulators) and the epilogue warpgroups take them
static constexpr int REG_LAUNCH = 128, REG_WG0 = 40, REG_MMA = 200, REG_EPI = 136;
static_assert(REG_WG0 + REG_MMA + 2 * REG_EPI == 4 * REG_LAUNCH, "the register split must fill the register file");
static constexpr int ACC_COLS_MAX = 128; // columns of the accumulator image (m-tiles per stage x block_n)
// staging warps the planner budgets shared memory for: the ring depth and the resident-B decision were made against a 16-warp
// epilogue, and keeping that budget keeps every plan as it was
static constexpr int PLAN_STG_WARPS = 16;
static constexpr int PAR_MAX = 2048; // channels whose epilogue constants stay resident in smem for the whole kernel
static constexpr int MAX_STAGES = 24;
static constexpr int B_RESIDENT_MAX = 96 * 1024; // weights of the CTA's N tile stay in smem when they fit in this many bytes

// Diagnosis of a failed (or, with TB200_DEBUG_LAUNCH, every) GEMM launch: device, stream's device, limits and what was asked for.
static void gemm_launch_debug(const void* fn, const char* what, cudaError_t err, int grid, size_t smem, cudaStream_t st)
{
    int dev = -1, optin = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncAttributes fa{};
    const cudaError_t e2 = cudaFuncGetAttributes(&fa, fn);
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cap);
    fprintf(stderr, "tengine_b200: gemm %s -> %s | device %d (%d SMs, opt-in smem %d) grid %d dynamic smem %zu | kernel static smem %zu max dynamic %d regs %d (%s) | capturing %d\n",
            what, cudaGetErrorString(err), dev, sms, optin, grid, smem, fa.sharedSizeBytes, fa.maxDynamicSharedSizeBytes, fa.numRegs, cudaGetErrorString(e2), (int)cap);
    cudaGetLastError();
}

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

// m-tile -> first output pixel coordinates (conv mode)
__device__ __forceinline__ void tile_origin(const GemmArgs& g, int mt, int& n0, int& oh0, int& ow0)
{
    const int r = mt / g.tiles_w;
    ow0 = (mt - r * g.tiles_w) * g.bw;
    const int nn = r / g.tiles_h;
    oh0 = (r - nn * g.tiles_h) * g.bh;
    n0 = nn * g.bn;
}

struct __align__(16) GemmSmemCtl
{
    uint64_t full[MAX_STAGES], empty[MAX_STAGES];
    uint64_t b_full; // resident-B mode: all k-blocks of the N tile's weights have landed
    uint64_t sx_full[2], sx_empty[2]; // uint8 row sums of stage s published by the row-sum warps / read by the epilogue
    uint64_t img_full, img_empty;     // the accumulator image holds a complete stage (MMA -> epilogue) / has been read (epilogue -> MMA)
};

// named barrier 1 over the epilogue warps only (the MMA warpgroup never joins it)
__device__ __forceinline__ void epilogue_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory"); }

// ---- the rare path of the fast epilogue, deferred -----------------------------------------------------------------------------
// An element whose t sits inside the tie guard needs the literal reference arithmetic (common.cuh requant(): divisions, per-channel
// loads, every recipe).  Done inline it occupies ONE lane of an epilogue warp for hundreds of cycles while the other fifteen warps
// finish their groups and then wait for it at the stage hand-over.  Instead the lane appends {m-tile, row, channel, accumulator} to the CTA's queue in
// global memory (L2) and carries on with the fast byte; after the CTA's last tile all 256 epilogue threads recompute the queued
// elements in parallel and patch the bytes in the output tensor (the tile's TMA store has completed by then).  A full or absent
// queue falls back to the inline computation, so the result never depends on the queue.
// (queue state in static shared memory, so that the rare-path functions need no extra arguments: passing the kernel arguments and a
//  counter pointer through the epilogue's inner loop cost registers there and made the int8 kernel 12 % slower)
struct FixQueue
{
    uint4* q;       // this CTA's segment, null = fix inline
    uint32_t cap;   // entries in the segment
    uint32_t count; // elements queued so far (may exceed cap: the surplus was fixed inline)
};
__shared__ FixQueue s_fixq;

__device__ __forceinline__ bool fixq_push(uint32_t mtile, int oc, int32_t acc)
{
    if (!s_fixq.q) return false;
    const uint32_t slot = atomicAdd(&s_fixq.count, 1u);
    if (slot >= s_fixq.cap) return false;
    const uint32_t row = ((threadIdx.x >> 5) & 3u) * 32u + (threadIdx.x & 31u); // image row of this thread = row of the m-tile
    s_fixq.q[slot] = make_uint4(mtile, row | ((uint32_t)oc << 8), (uint32_t)acc, 0u);
    return true;
}

// One guarded word (final fast bytes in `word`): find the elements that really sit in the band, queue them (or fix them here).
// a[j]: what the fast path converted to float -- int8: the raw accumulator (y is added inside), uint8: accumulator + sum(x) term + y.
template <bool U8, bool FUSE>
__device__ __noinline__ uint32_t gemm_fix_word(uint32_t word, int32_t a0, int32_t a1, int32_t a2, int32_t a3, int oc0, int oc_limit, uint32_t mtile,
                                               const EpiParams& e)
{
    const FastPar4 f = fast_par4_ldg(e, oc0);
    const int32_t a[4] = {a0, a1, a2, a3};
    const float m[4] = {f.a.x, f.a.y, f.b.x, f.b.y}, y[4] = {f.a.z, f.a.w, f.b.z, f.b.w};
#pragma unroll
    for (int j = 0; j < 4; j++)
    {
        const float t = U8 ? __fmul_rn((float)a[j], m[j]) : (FUSE ? __fmaf_rn((float)a[j], m[j], y[j]) : __fmul_rn((float)(a[j] + __float_as_int(y[j])), m[j]));
        const float r = __fadd_rn(t, TB200_MAGIC);
        const float d = __fsub_rn(t, __fsub_rn(r, TB200_MAGIC));
        if (fabsf(d) > 0.5f - TB200_TIE_EPS && oc0 + j < oc_limit)
        {
            if (!fixq_push(mtile, oc0 + j, a[j]))
            {
                // the literal arithmetic wants the accumulator without the bias (uint8: y holds it)
                const int32_t acc = a[j] - ((U8 && e.has_bias) ? __ldg(e.bias + oc0 + j) : 0);
                const uint32_t q = (uint32_t)requant(acc, oc0 + j, e) & 0xffu;
                word = (word & ~(0xffu << (8 * j))) | (q << (8 * j));
            }
        }
    }
    return word;
}

// After the CTA's last tile (every epilogue warp has waited for its own bulk stores): recompute the queued elements, one per epilogue
// thread.
template <bool U8>
__device__ __forceinline__ void fixq_drain(const GemmArgs& g, const EpiParams& e)
{
    const uint32_t n = s_fixq.count < s_fixq.cap ? s_fixq.count : s_fixq.cap;
    for (uint32_t k = threadIdx.x - EPI_THREAD0; k < n; k += EPI_THREADS)
    {
        const uint4 q = s_fixq.q[k];
        const int mt = (int)q.x, r = (int)(q.y & 127u), oc = (int)(q.y >> 8);
        long long pix;
        bool ok = r < g.rows_valid;
        if (!g.conv)
            pix = (long long)mt * BLOCK_M + r, ok = ok && pix < g.m_rows;
        else
        {
            int cn0, coh0, cow0;
            tile_origin(g, mt, cn0, coh0, cow0);
            if (g.out_mode == 0) pix = (long long)cn0 * g.oh * g.ow + r, ok = ok && pix < (long long)g.nimg * g.oh * g.ow;
            else if (g.out_mode == 1) pix = (long long)cn0 * g.oh * g.ow + coh0 * g.ow + r, ok = ok && coh0 * g.ow + r < g.oh * g.ow;
            else pix = ((long long)cn0 * g.oh + coh0) * g.ow + cow0 + r, ok = ok && cow0 + r < g.ow;
        }
        if (!ok || oc >= g.oc) continue; // a row the TMA store clipped
        const int32_t acc = (int32_t)q.z - ((U8 && e.has_bias) ? __ldg(e.bias + oc) : 0);
        g.out_base[(size_t)pix * g.ldo + oc] = (uint8_t)requant(acc, oc, e);
    }
}

// 16 accumulator columns of one row -> 16 output bytes into the warp's staging buffer (int8, fast path).
template <bool FUSE>
__device__ __forceinline__ void epilogue_unit_fast(const uint32_t (&v)[16], uint32_t par_addr, uint32_t dst_addr, int oc0, uint32_t mtile, const EpiParams& e)
{
    uint32_t w[4];
    float gw[4];
#pragma unroll
    for (int h = 0; h < 2; h++)
    {
        float4 p[4];
#pragma unroll
        for (int k = 0; k < 4; k++) p[k] = lds_f4(par_addr + h * 64 + k * 16);
        const int32_t a8[8] = {(int32_t)v[h * 8], (int32_t)v[h * 8 + 1], (int32_t)v[h * 8 + 2], (int32_t)v[h * 8 + 3],
                               (int32_t)v[h * 8 + 4], (int32_t)v[h * 8 + 5], (int32_t)v[h * 8 + 6], (int32_t)v[h * 8 + 7]};
        requant_fast8_i8<FUSE>(a8, p, e, w[2 * h], w[2 * h + 1], gw[2 * h], gw[2 * h + 1]);
    }
    if (e.q_byte_add)
    {
#pragma unroll
        for (int j = 0; j < 4; j++) w[j] = requant_byte_fix(w[j], e);
    }
    if (fmaxf(fmaxf(gw[0], gw[1]), fmaxf(gw[2], gw[3])) > 0.5f - TB200_TIE_EPS)
    {
        // rare (2.4e-4 of the elements): exact recomputation of the guarded bytes
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (gw[j] > 0.5f - TB200_TIE_EPS)
                w[j] = gemm_fix_word<false, FUSE>(w[j], (int32_t)v[j * 4], (int32_t)v[j * 4 + 1], (int32_t)v[j * 4 + 2], (int32_t)v[j * 4 + 3], oc0 + j * 4, 0x7fffffff /* pad channels have M = y = 0: never guarded */, mtile, e);
    }
    sts_u4(dst_addr, w[0], w[1], w[2], w[3]);
}

// degenerate scales / accumulators that could leave the 16-bit clamp range: literal arithmetic for every element
__device__ __forceinline__ void epilogue_unit_exact(const uint32_t (&v)[16], uint32_t dst_addr, int oc0, int oc_limit, const EpiParams& e)
{
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 16; k++)
    {
        if ((k & 3) == 0) w[k >> 2] = 0;
        if (oc0 + k < oc_limit) w[k >> 2] |= ((uint32_t)requant((int32_t)v[k], oc0 + k, e) & 0xffu) << (8 * (k & 3));
    }
    sts_u4(dst_addr, w[0], w[1], w[2], w[3]);
}

// uint8 flavour: v = sum x*w over in-bounds taps (raw bytes), sx = sum x.  The true accumulator is
//   sum (x-zx)(w-zw) = v - zw*sx + corr[oc] + sum_{padding taps t} btab[t][oc]
// with corr[oc] = -zx*sum_k w + taps*Cin*zx*zw (interior pixels) folded into the per-channel constants.
// uint8 flavour: v = sum x*w over in-bounds taps (raw bytes), sx = sum x.  The true accumulator is
//   sum (x-zx)(w-zw) = v - zw*sx + corr[oc] + sum_{padding taps t} btab[t][oc]
// with corr[oc] = -zx*sum_k w + taps*Cin*zx*zw (interior pixels).  The per-channel constants are in the int8 layout
// { M[2k], M[2k+1], y[2k], y[2k+1] } with y = corr + bias (an integer), so the fast path IS the int8 one on a' = v + rowc + y:
// t = fl((float)a' * M), exact up to the tie guard under the bound engine.cu proves per layer (|bias*M| <= 250).

template <bool EXACT, bool BORDER>
__device__ __forceinline__ void epilogue_unit_u8(const uint32_t (&v)[16], int32_t rowc, uint32_t pad_mask_in, const GemmArgs& g, uint32_t par_addr,
                                                 uint32_t dst_addr, int oc0, uint32_t mtile, const EpiParams& e)
{
    const uint32_t pad_mask = BORDER ? pad_mask_in : 0u; // BORDER == false (1x1 / FC, unpadded convs): the correction code compiles away
    uint32_t w[4];
    if (!EXACT)
    {
        float gw[4];
#pragma unroll
        for (int h = 0; h < 2; h++)
        {
            float4 p[4];
#pragma unroll
            for (int k = 0; k < 4; k++) p[k] = lds_f4(par_addr + h * 64 + k * 16);
            int32_t a8[8];
#pragma unroll
            for (int k = 0; k < 8; k++) a8[k] = (int32_t)v[h * 8 + k] + rowc; // (+ y inside requant_fast8_i8<false>: one IADD3)
            if (pad_mask)
            {
                // border row: the summed corrections of its missing taps, one 16-byte load per four channels
                const int4* pt = reinterpret_cast<const int4*>(g.btab + (size_t)pad_mask * g.ocp + oc0 + h * 8);
                const int4 c0 = __ldg(pt), c1 = __ldg(pt + 1);
                a8[0] += c0.x, a8[1] += c0.y, a8[2] += c0.z, a8[3] += c0.w, a8[4] += c1.x, a8[5] += c1.y, a8[6] += c1.z, a8[7] += c1.w;
            }
            requant_fast8_i8<false>(a8, p, e, w[2 * h], w[2 * h + 1], gw[2 * h], gw[2 * h + 1]);
        }
        if (e.q_byte_add)
        {
#pragma unroll
            for (int j = 0; j < 4; j++) w[j] = requant_byte_fix(w[j], e);
        }
        if (fmaxf(fmaxf(gw[0], gw[1]), fmaxf(gw[2], gw[3])) > 0.5f - TB200_TIE_EPS)
        {
            // rare (2.4e-4 of the elements): the guarded words again -- requant_fix_word_u8 finds the elements inside the band and
            // runs the literal reference arithmetic on exactly those
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (gw[j] > 0.5f - TB200_TIE_EPS)
                {
                    int32_t a[4];
#pragma unroll
                    for (int t = 0; t < 4; t++)
                    {
                        const float4 pp = lds_f4(par_addr + ((j * 4 + t) >> 1) * 16);
                        a[t] = (int32_t)v[j * 4 + t] + rowc + __float_as_int((t & 1) ? pp.w : pp.z);
                    }
                    if (pad_mask && oc0 + j * 4 < g.ocp)
                    {
                        const int4 c = __ldg(reinterpret_cast<const int4*>(g.btab + (size_t)pad_mask * g.ocp + oc0 + j * 4));
                        a[0] += c.x, a[1] += c.y, a[2] += c.z, a[3] += c.w;
                    }
                    w[j] = gemm_fix_word<true, false>(w[j], a[0], a[1], a[2], a[3], oc0 + j * 4, g.oc, mtile, e);
                }
        }
        if (oc0 + 16 > g.oc)
        {
            // pad lanes of uint8 tensors hold 0, not the zero point
#pragma unroll
            for (int k = 0; k < 16; k++)
                if (oc0 + k >= g.oc) w[k >> 2] &= ~(0xffu << (8 * (k & 3)));
        }
    }
    else
    {
#pragma unroll
        for (int k = 0; k < 16; k++)
        {
            if ((k & 3) == 0) w[k >> 2] = 0;
            const int oc = oc0 + k;
            if (oc < g.oc)
            {
                const float4 pp = lds_f4(par_addr + (k >> 1) * 16);
                int32_t a = (int32_t)v[k] + rowc + __float_as_int((k & 1) ? pp.w : pp.z) - (e.has_bias ? __ldg(e.bias + oc) : 0);
                if (pad_mask) a += __ldg(g.btab + (size_t)pad_mask * g.ocp + oc);
                w[k >> 2] |= ((uint32_t)requant(a, oc, e) & 0xffu) << (8 * (k & 3));
            }
        }
    }
    sts_u4(dst_addr, w[0], w[1], w[2], w[3]);
}

// border pattern of output pixel r of m-tile mt (0 = every tap inside the image): how many rows / columns of the filter window are
// cut at the top (a), bottom (b), left (c), right (d); index into the table engine.cu builds
__device__ __forceinline__ uint32_t padding_taps(const GemmArgs& g, int mt, int r)
{
    if (!g.conv) return 0; // (a 1x1 convolution padded at the bottom / right only has border pixels too)
    int n0, oh0, ow0;
    tile_origin(g, mt, n0, oh0, ow0);
    const int t = (int)(((uint32_t)r * g.bw_rcp) >> 16), w = r - t * g.bw;
    const int n = (int)(((uint32_t)t * g.bh_rcp) >> 16), h = t - n * g.bh;
    const int iy0 = (oh0 + h) * g.cstride - g.pad_h, ix0 = (ow0 + w) * g.cstride - g.pad_w;
    const int khn = g.taps / g.kw_n;
    int a = -iy0, b = iy0 + khn - g.in_h, c = -ix0, d = ix0 + g.kw_n - g.in_w;
    a = a < 0 ? 0 : a, b = b < 0 ? 0 : (b > khn ? khn : b), c = c < 0 ? 0 : c, d = d < 0 ? 0 : (d > g.kw_n ? g.kw_n : d);
    // (a <= pad_h and c <= pad_w by construction; rows of the tile beyond the output map are clipped by the store anyway)
    a = a > g.pad_h ? g.pad_h : a, c = c > g.pad_w ? g.pad_w : c;
    return (uint32_t)(((a * (khn + 1) + b) * (g.pad_w + 1) + c) * (g.kw_n + 1) + d);
}

// ---- the MMA warpgroup ---------------------------------------------------------------------------------------------------------
// One accumulator stage (MT m-tiles x BN columns, MT * BN <= ACC_COLS_MAX) is computed in registers: per m-tile and k-step two
// m64nBNk32, rows 0-63 and 64-127, into MT * BN s32 registers per thread.  One commit group per k-block stays in flight: after
// committing k-block kb the warpgroup waits for the group of kb - 1 and releases the ring stage that group read; the pipe is
// drained (wait_group 0) only at the end of the stage.  The registers are the second accumulator buffer: while this stage is
// multiplied the epilogue drains the previous one from the image; the fragments are then written into the image once every
// epilogue warp has read it (img_empty) and published with img_full.  BN, MT and the operand signs are template parameters so
// that the accumulators are indexed statically and no wgmma sits in a branch the compiler cannot prove uniform.
template <bool AU, bool BU, int BN, int MT, typename Log>
__device__ __forceinline__ void gemm_mma(const GemmArgs& g, GemmSmemCtl* ctl, uint8_t* smem, uint32_t stage_bytes, uint32_t b_res_base,
                                         uint32_t img_base, uint32_t img_pitch, Log&& tlog)
{
    constexpr int NR = BN / 2; // registers of one m64nBN fragment
    uint32_t acc[MT][2][NR];
#pragma unroll
    for (int i = 0; i < MT; i++)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int r = 0; r < NR; r++) acc[i][h][r] = 0;
    const bool elected = threadIdx.x == MMA_THREAD0; // arrives on the ring's empty barriers for the warpgroup
    const uint32_t a_bytes = BLOCK_M * g.block_k, b_al = (BN * g.block_k + 1023) & ~1023u;
    const int ks = g.block_k / 32;
    const uint64_t half = (uint64_t)((64 * g.swizzle) >> 4); // A rows 64.. in descriptor units (16 bytes)
    int stage = 0, held = -1; // held: the ring stage the group in flight reads
    uint32_t phase = 0, iphase = 0;
    if (g.b_res) mbar_wait(&ctl->b_full, 0);
    for (int st = blockIdx.x; st < g.num_super; st += gridDim.x)
    {
        const int rem = g.m_tiles - (st / g.n_tiles) * MT;
        const int mtc = rem < MT ? rem : MT;
#pragma unroll
        for (int i = 0; i < MT; i++)
        {
            if (i >= mtc) break;
            for (int kb = 0; kb < g.k_blocks; kb++)
            {
                mbar_wait(&ctl->full[stage], phase); // TMA bytes have landed
                const uint32_t sa = smem_u32(smem + (size_t)stage * stage_bytes);
                const uint32_t sb = g.b_res ? b_res_base + (uint32_t)kb * b_al : sa + a_bytes;
                const uint64_t da = make_smem_desc(sa, g.swizzle), db = make_smem_desc(sb, g.swizzle);
                wgmma_fence();
                for (int k = 0; k < ks; k++)
                {
                    // +32 bytes along K inside the swizzled rows: +2 in 16-byte units; the first k-step of the tile overwrites
                    const uint32_t accumulate = (kb | k) != 0;
                    wgmma_m64<BN, AU, BU>(acc[i][0], da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), accumulate);
                    wgmma_m64<BN, AU, BU>(acc[i][1], da + half + (uint64_t)(k * 2), db + (uint64_t)(k * 2), accumulate);
                }
                wgmma_commit();
                wgmma_wait<1>(); // the previous group has completed: the ring stage it read may be refilled
                if (held >= 0 && elected) mbar_arrive(&ctl->empty[held]);
                held = stage;
                if (++stage == g.stages) stage = 0, phase ^= 1;
            }
        }
        wgmma_wait<0>();
        if (elected) mbar_arrive(&ctl->empty[held]);
        held = -1;
#pragma unroll
        for (int i = 0; i < MT; i++)
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int r = 0; r < NR; r++) reg_fence(acc[i][h][r]);
        tlog(1, 0);
        mbar_wait(&ctl->img_empty, iphase ^ 1); // every epilogue warp has read the previous stage out of the image
        tlog(1, 1);
#pragma unroll
        for (int i = 0; i < MT; i++)
        {
            if (i >= mtc) break;
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int c = 0; c < BN / 16; c++)
                    frag_to_image(*reinterpret_cast<const uint32_t(*)[8]>(&acc[i][h][8 * c]), img_base, img_pitch, h * 64, i * BN + c * 16);
        }
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(&ctl->img_full); // (release) this warp's rows of the stage are in the image
        tlog(1, 2);
        iphase ^= 1;
    }
}

// (block_n, m-tiles per stage) of the launch -> the MMA warpgroup's code for it; uniform across the CTA
template <bool AU, bool BU, typename Log>
__device__ __forceinline__ void gemm_mma_dispatch(const GemmArgs& g, GemmSmemCtl* ctl, uint8_t* smem, uint32_t stage_bytes, uint32_t b_res_base,
                                                  uint32_t img_base, uint32_t img_pitch, Log&& tlog)
{
#define TB200_MMA_CASE(BN, MT)                                                                                                 \
    case BN * 4 + MT - 1: gemm_mma<AU, BU, BN, MT>(g, ctl, smem, stage_bytes, b_res_base, img_base, img_pitch, tlog); break;
    switch (g.block_n * 4 + g.mt - 1)
    {
        TB200_MMA_CASE(16, 1) TB200_MMA_CASE(16, 2) TB200_MMA_CASE(16, 4)
        TB200_MMA_CASE(32, 1) TB200_MMA_CASE(32, 2) TB200_MMA_CASE(32, 4)
        TB200_MMA_CASE(48, 1) TB200_MMA_CASE(48, 2)
        TB200_MMA_CASE(64, 1) TB200_MMA_CASE(64, 2)
        TB200_MMA_CASE(80, 1) TB200_MMA_CASE(96, 1) TB200_MMA_CASE(112, 1) TB200_MMA_CASE(128, 1)
        default: __trap(); // plan_stage never makes another (block_n, mt)
    }
#undef TB200_MMA_CASE
}

// MODE: 0 fast epilogue, 1 fast epilogue with the bias folded into the FMA (int8 only), 2 exact epilogue.
// CS: 16-column chunks per store group (1 or 2).  Compile-time so that each kernel carries exactly one epilogue body.
template <bool U8, int MODE, int CS, bool BORDER>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_i8_tcgen05_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                           const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_out_tail,
                           const GemmArgs g, const __grid_constant__ EpiParams e)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // operand ring first (1024-byte aligned for the 128B swizzle), then the per-warp output staging buffers (1024-byte
    // aligned: their TMA swizzle pattern is a function of the address), the control block and the epilogue constants
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t a_bytes = BLOCK_M * g.block_k, b_bytes = g.block_n * g.block_k;
    const uint32_t b_al = (b_bytes + 1023) & ~1023u;
    const uint32_t stage_bytes = a_bytes + (g.b_res ? 0u : b_al);
    uint8_t* b_region = smem + (size_t)g.stages * stage_bytes; // resident-B mode: [k_blocks][b_al]
    constexpr uint32_t buf_bytes = 512u * CS; // 32 rows x 16*CS bytes
    uint8_t* sxs = b_region + (g.b_res ? (size_t)g.k_blocks * b_al : 0); // uint8: sum(x) of the rows, [2 accumulator stages][4 m-tiles][128] int32
    uint8_t* stg = sxs + (g.cplane ? 4096u : 0u);
    const uint32_t sx_base = smem_u32(sxs);
    const uint32_t stg_base = smem_u32(stg);
    GemmSmemCtl* ctl = reinterpret_cast<GemmSmemCtl*>(stg + (size_t)EPI_WARPS * 2 * buf_bytes);
    const uint32_t par_base = smem_u32(ctl) + (uint32_t)sizeof(GemmSmemCtl); // [par channels] x 8 bytes (see FastPar4)
    const int acc_cols = g.mt * g.block_n; // accumulator image columns of one stage
    const uint32_t img_pitch = acc_pitch(acc_cols);
    const uint32_t img_base = (par_base + (uint32_t)(g.par_all ? g.n_tiles * g.block_n : g.block_n) * 8u + 15u) & ~15u;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // debug timeline: CTA 0 only, 4 logs x 1024 events of (clock << 8 | tag); plain global stores, no atomics
#ifdef TB200_GEMM_TIMELINE
    int tl_n = 0;
    auto tlog = [&](int role, int tag)
    {
        if (g.trace && blockIdx.x == 0 && tl_n < 1024) g.trace[role * 1024 + tl_n++] = ((unsigned long long)clock64() << 8) | (unsigned)tag;
    };
#else
    auto tlog = [](int, int) {}; // the timeline costs instructions in the epilogue's inner loop: debug builds only
#endif

    if (threadIdx.x == 0)
    {
        const uint32_t sumw = (U8 && g.cplane) ? SUM_WARPS : 0; // the row-sum warps read every operand stage and publish with the accumulators
        for (int s = 0; s < g.stages; s++) mbar_init(&ctl->full[s], 1), mbar_init(&ctl->empty[s], 1 + sumw);
        for (int s = 0; s < 2; s++) mbar_init(&ctl->sx_full[s], sumw ? sumw : 1), mbar_init(&ctl->sx_empty[s], EPI_WARPS);
        mbar_init(&ctl->b_full, 1);
        mbar_init(&ctl->img_full, 4), mbar_init(&ctl->img_empty, EPI_WARPS);
        s_fixq.q = g.fixq ? g.fixq + (size_t)blockIdx.x * g.fixq_cap : nullptr, s_fixq.cap = (uint32_t)g.fixq_cap, s_fixq.count = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // the warpgroup index, broadcast from lane 0 so that the compiler sees the role branches as warp-uniform
    const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
    if (wg == 0)
    {
        setmaxnreg_dec<REG_WG0>();
        if (warp == PRODUCER_WARP)
        {
            // ===================== TMA producer =====================
            if (lane == 0)
            {
                asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_a)) : "memory");
                asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_b)) : "memory");
                int stage = 0;
                uint32_t phase = 0;
                if (g.b_res)
                {
                    // the grid is a multiple of n_tiles, so this CTA only ever sees N tile blockIdx.x % n_tiles: load its
                    // weights (every k-block) once
                    const int nb = (blockIdx.x % g.n_tiles) * g.block_n;
                    mbar_expect_tx(&ctl->b_full, (uint32_t)g.k_blocks * b_bytes);
                    for (int kb = 0; kb < g.k_blocks; kb++)
                    {
                        const int kc = g.conv ? (kb / g.cblocks) * g.cp + (kb % g.cblocks) * g.block_k : kb * g.block_k;
                        tma_load_2d(&tmap_b, &ctl->b_full, b_region + (size_t)kb * b_al, kc, nb);
                    }
                }
                for (int st = blockIdx.x; st < g.num_super; st += gridDim.x)
                {
                    const int msup = st / g.n_tiles;
                    const int mt0 = msup * g.mt;
                    const int ntile = st - msup * g.n_tiles;
                    const int n0 = ntile * g.block_n; // row of this N tile in the packed weight matrix
                    for (int i = 0; i < g.mt && mt0 + i < g.m_tiles; i++)
                    {
                        const int m0 = (mt0 + i) * BLOCK_M;
                        int cn0 = 0, coh0 = 0, cow0 = 0;
                        if (g.conv) tile_origin(g, mt0 + i, cn0, coh0, cow0);
                        for (int kb = 0; kb < g.k_blocks; kb++)
                        {
                            mbar_wait(&ctl->empty[stage], phase ^ 1);
                            uint8_t* sa = smem + (size_t)stage * stage_bytes;
                            if (!g.conv)
                            {
                                mbar_expect_tx(&ctl->full[stage], a_bytes + (g.b_res ? 0u : b_bytes));
                                tma_load_2d(&tmap_a, &ctl->full[stage], sa, kb * g.block_k, m0);
                                if (!g.b_res) tma_load_2d(&tmap_b, &ctl->full[stage], sa + a_bytes, kb * g.block_k, n0);
                            }
                            else
                            {
                                // k-block = (filter tap, channel block): the A tile is the output patch shifted by the tap;
                                // coordinates outside the image are zero-filled by the TMA unit = the convolution's padding
                                const int tap = kb / g.cblocks, cb = kb - tap * g.cblocks;
                                const int kh = tap / g.kw_n, kw = tap - kh * g.kw_n;
                                mbar_expect_tx(&ctl->full[stage], g.a_tx_bytes + (g.b_res ? 0u : b_bytes));
                                tma_load_4d(&tmap_a, &ctl->full[stage], sa, cb * g.block_k, cow0 * g.cstride - g.pad_w + kw,
                                            coh0 * g.cstride - g.pad_h + kh, cn0);
                                if (!g.b_res) tma_load_2d(&tmap_b, &ctl->full[stage], sa + a_bytes, tap * g.cp + cb * g.block_k, n0);
                            }
                            tlog(0, kb & 0xff);
                            if (++stage == g.stages) stage = 0, phase ^= 1;
                        }
                    }
                }
            }
        }
        else if (U8 && warp < SUM_WARP0 + SUM_WARPS && g.cplane)
        {
            // ===================== row sums (uint8, warps 1 and 2) =====================
            // sum x*(w - zw) = sum x*(w - 128) [tensor cores, B signed] + (128 - zw) * sum(x).  sum(x) of output row r is the sum of ALL bytes
            // of row r of every A tile of the m-tile (taps outside the image were zero-filled by the TMA unit, K tails too), and a sum
            // does not care about the swizzle that permutes the 16-byte chunks inside a row.  Each of the two warps owns 64 rows (two per
            // lane), reads them with 16-byte loads (chunk order rotated per lane so that a quarter-warp covers all banks), dp4a against
            // 0x01010101, and publishes the sums through shared memory together with the accumulator stage.  This keeps the uint8 tiling
            // identical to the int8 one: no extra B rows, no extra accumulator columns, no second MMA.
            const int sw = warp - SUM_WARP0;
            const int cpr = g.block_k >> 4;                  // 16-byte chunks per row: 2, 4 or 8
            const int rot = (lane * g.block_k) >> 7;         // lanes whose rows start in the same 128-byte window get different chunks
            const uint32_t row0 = (uint32_t)(sw * 64 + lane) * (uint32_t)g.block_k, row1 = row0 + 32u * (uint32_t)g.block_k;
            int stage = 0;
            uint32_t phase = 0;
            int as = 0;
            uint32_t aphase = 0;
            for (int st = blockIdx.x; st < g.num_super; st += gridDim.x)
            {
                const int mt0 = (st / g.n_tiles) * g.mt;
                mbar_wait(&ctl->sx_empty[as], aphase ^ 1); // the epilogue has read this stage's sums
                for (int i = 0; i < g.mt && mt0 + i < g.m_tiles; i++)
                {
                    unsigned s0 = 0, s1 = 0;
                    for (int kb = 0; kb < g.k_blocks; kb++)
                    {
                        mbar_wait(&ctl->full[stage], phase);
                        const uint32_t sa = smem_u32(smem + (size_t)stage * stage_bytes);
                        for (int c = 0; c < cpr; c++)
                        {
                            const uint32_t ch = (uint32_t)((c + rot) & (cpr - 1)) << 4;
                            const uint4 u = lds_u4(sa + row0 + ch), v = lds_u4(sa + row1 + ch);
                            s0 = __dp4a(u.x, 0x01010101u, s0), s1 = __dp4a(v.x, 0x01010101u, s1);
                            s0 = __dp4a(u.y, 0x01010101u, s0), s1 = __dp4a(v.y, 0x01010101u, s1);
                            s0 = __dp4a(u.z, 0x01010101u, s0), s1 = __dp4a(v.z, 0x01010101u, s1);
                            s0 = __dp4a(u.w, 0x01010101u, s0), s1 = __dp4a(v.w, 0x01010101u, s1);
                        }
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&ctl->empty[stage]); // this warp has read the stage
                        if (++stage == g.stages) stage = 0, phase ^= 1;
                    }
                    const uint32_t dst = sx_base + (uint32_t)(((as * 4 + i) * 128 + sw * 64 + lane) * 4);
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst), "r"(s0) : "memory");
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst + 128u), "r"(s1) : "memory");
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&ctl->sx_full[as]); // (release) the sums of this stage are in shared memory
                if (++as == 2) as = 0, aphase ^= 1;
            }
        }
    }
    else if (wg == 1)
    {
        // ===================== MMA (warps 4..7) =====================
        setmaxnreg_inc<REG_MMA>();
        const uint32_t b_res_base = smem_u32(b_region);
        if (U8 && !g.b_signed) gemm_mma_dispatch<U8, true>(g, ctl, smem, stage_bytes, b_res_base, img_base, img_pitch, tlog);
        else gemm_mma_dispatch<U8, false>(g, ctl, smem, stage_bytes, b_res_base, img_base, img_pitch, tlog);
    }
    else
    {
        // ===================== epilogue (warps 8..15) =====================
        // Image quarter q (rows 32q..32q+31) is served by the two warps {8 + q, 12 + q}.  The work of an accumulator stage is cut
        // into store groups (m-tile i, columns [grp*16*cs, (grp+1)*16*cs)) of 32 rows each, dealt round-robin to the quarter's
        // warps.  A warp requantises its group chunk by chunk (16 columns per load, the next chunk's load in flight), writes the
        // bytes to its own swizzled staging buffer and hands the buffer to the TMA unit with one store.  It releases the image to
        // the MMA warpgroup (img_empty) as soon as it has issued its last load of the stage.
        setmaxnreg_inc<REG_EPI>();
        const int ew = warp - EPI_WARP0; // epilogue warp 0..7
        const int q = warp & 3;
        const int sub = ew >> 2;
        const int et = (int)threadIdx.x - EPI_THREAD0;
        const int ngroups = g.ngroups;
        int qrows = g.rows_valid - q * 32; // rows of this quarter that are output pixels
        qrows = qrows < 0 ? 0 : (qrows > 32 ? 32 : qrows);
        const CUtensorMap* tm_out = (qrows == 32) ? &tmap_out : &tmap_out_tail;
        const uint32_t buf0 = stg_base + (uint32_t)ew * 2u * buf_bytes;
        // swizzle of the staging buffer = the output map's swizzle: 16-byte chunk index ^= row bit 2 (Swizzle<1,4,3>, CS 2 only)
        const uint32_t xl = CS == 2 ? (uint32_t)((lane >> 2) & 1) << 4 : 0u;
        const uint32_t row_off = (uint32_t)lane * 16u * CS;
        uint32_t ucount = 0; // groups this warp has stored (buffer parity)
        const int par_ch = g.n_tiles * g.block_n;
        const bool fast = MODE != 2;
        if (g.par_all)
        {
            // per-channel fast-path constants of every N tile, once; pad / overhanging channels get (0, 0)
            for (int c = et; c < par_ch; c += EPI_THREADS)
                sts_f2(par_base + c * 8, (c < g.ocp && (fast || U8)) ? __ldg(e.fast_par + c) : make_float2(0.f, 0.f));
            epilogue_bar_sync();
        }
        if (lane == 0 && qrows > 0) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm_out)) : "memory");
        int as = 0;
        uint32_t aphase = 0, iphase = 0;
        for (int st = blockIdx.x; st < g.num_super; st += gridDim.x)
        {
            const int msup = st / g.n_tiles;
            const int mt0 = msup * g.mt;
            const int n0 = (st - msup * g.n_tiles) * g.block_n;
            const int rem = g.m_tiles - mt0;
            const int mtc = rem < g.mt ? rem : g.mt;
            uint32_t par_s = par_base + (uint32_t)n0 * 8u;
            if (!g.par_all)
            {
                epilogue_bar_sync(); // every epilogue warp is done with the previous tile's constants
                for (int c = et; c < g.block_n; c += EPI_THREADS)
                    sts_f2(par_base + c * 8, (n0 + c < g.ocp && (fast || U8)) ? __ldg(e.fast_par + n0 + c) : make_float2(0.f, 0.f));
                epilogue_bar_sync();
                par_s = par_base;
            }
            mbar_wait(&ctl->img_full, iphase); // the image holds this stage
            iphase ^= 1;
            if (U8 && g.cplane) mbar_wait(&ctl->sx_full[as], aphase); // the row sums of this stage
            TLOG_E(0);
            const uint32_t tbase = img_base + (uint32_t)(q * 32 + lane) * img_pitch;
            bool released = false; // this warp has arrived on img_empty for this stage
            if (qrows > 0)
            {
                // groups of this warp: flattened index u = i * ngroups + grp, u = sub, sub + 2, ...
                uint32_t v0[16], v1[16];
                int i = 0, grp = sub;
                while (grp >= ngroups) grp -= ngroups, i++;
                if (CS > 1 && i < mtc)
                    acc_ld16(tbase + 4u * (i * g.block_n + grp * (CS * 16)), reinterpret_cast<uint32_t(&)[16]>(v0));
                while (i < mtc)
                {
                    int i2 = i, g2 = grp + 2; // the group after this one
                    while (g2 >= ngroups) g2 -= ngroups, i2++;
                    const uint32_t buf = buf0 + (ucount & 1u) * buf_bytes;
                    // the store issued two groups ago has finished reading this buffer
                    if (lane == 0) bulk_wait_read<1>();
                    __syncwarp();
                    uint32_t pad = 0;
                    int32_t rowc = 0;
                    if (U8)
                    {
                        // the pixel's sum(x), once per group
                        if (g.cplane)
                        {
                            int32_t sx;
                            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(sx) : "r"(sx_base + (uint32_t)(((as * 4 + i) * 128 + q * 32 + lane) * 4)));
                            rowc = g.cplane * sx;
                        }
                        if (BORDER) pad = padding_taps(g, mt0 + i, q * 32 + lane);
                    }
                    const uint32_t tg = tbase + 4u * (i * g.block_n + grp * (CS * 16));
                    const int cg0 = grp * (CS * 16); // first column of the group inside the N tile
                    const uint32_t sdst = buf + row_off;
                    auto unit = [&](const uint32_t (&v)[16], int k)
                    {
                        const int c = cg0 + k * 16;
                        const uint32_t dst = sdst + (((uint32_t)k << 4) ^ xl);
                        if (U8) epilogue_unit_u8<MODE == 2, BORDER>(v, rowc, pad, g, par_s + c * 8, dst, n0 + c, (uint32_t)(mt0 + i), e);
                        else if (MODE == 2) epilogue_unit_exact(v, dst, n0 + c, g.oc, e);
                        else epilogue_unit_fast<MODE == 1>(v, par_s + c * 8, dst, n0 + c, (uint32_t)(mt0 + i), e);
                    };
                    // after the last image load of the stage: (release) the MMA warpgroup may overwrite the image
                    auto release = [&]()
                    {
                        if (i2 >= mtc)
                        {
                            __syncwarp();
                            if (lane == 0) mbar_arrive(&ctl->img_empty);
                            released = true;
                        }
                    };
                    if (CS == 1)
                    {
                        acc_ld16(tg, reinterpret_cast<uint32_t(&)[16]>(v0));
                        release();
                        unit(reinterpret_cast<const uint32_t(&)[16]>(v0), 0);
                    }
                    else
                    {
#pragma unroll
                        for (int k = 0; k < CS; k++)
                        {
                            TLOG_E(3);
                            // the next chunk's accumulators are in flight while this one is requantised
                            if (k + 1 < CS) acc_ld16(tg + (k + 1) * 64, reinterpret_cast<uint32_t(&)[16]>(*((k & 1) ? v0 : v1)));
                            else if (i2 < mtc) acc_ld16(tbase + 4u * (i2 * g.block_n + g2 * (CS * 16)), reinterpret_cast<uint32_t(&)[16]>(v0));
                            if (k + 1 == CS) release();
                            unit(reinterpret_cast<const uint32_t(&)[16]>(*((k & 1) ? v1 : v0)), k);
                            TLOG_E(4);
                        }
                    }
                    fence_proxy_async_smem(); // generic-proxy writes -> visible to the TMA unit
                    __syncwarp();
                    if (lane == 0)
                    {
                        int x1, x2 = 0;
                        if (!g.conv)
                            x1 = (mt0 + i) * BLOCK_M;
                        else
                        {
                            int cn0, coh0, cow0;
                            tile_origin(g, mt0 + i, cn0, coh0, cow0);
                            if (g.out_mode == 0) x1 = cn0 * g.oh * g.ow;
                            else if (g.out_mode == 1) x1 = coh0 * g.ow, x2 = cn0;
                            else x1 = cow0, x2 = cn0 * g.oh + coh0;
                        }
                        tma_store_3d(tm_out, buf, n0 + cg0, x1 + q * 32, x2);
                        bulk_commit();
                    }
                    TLOG_E(1);
                    ucount++;
                    i = i2, grp = g2;
                }
            }
            __syncwarp();
            if (lane == 0)
            {
                if (!released) mbar_arrive(&ctl->img_empty); // a warp without a group in this stage
                mbar_arrive(&ctl->sx_empty[as]);             // stage drained: the row-sum warps may overwrite its sums
            }
            TLOG_E(2);
            if (++as == 2) as = 0, aphase ^= 1;
        }
        if (lane == 0) bulk_wait<0>(); // all of this warp's stores have completed
        if (g.fixq && MODE != 2)
        {
            // deferred rare path: every warp's stores are complete (and its queue entries written) once all have passed this barrier
            __threadfence_block();
            epilogue_bar_sync();
            fixq_drain<U8>(g, e);
        }
    }
}

// ---- on-box peak of the int8 tensor pipe (SURVEY.md 8(d): "replace the nominal numbers by on-box microbenchmark peaks") ---------
// One CTA of two warpgroups per SM; each warpgroup issues `iters` x 4 wgmma m64n128k32 s8 on fixed shared-memory tiles (contents
// irrelevant) into its own registers; no loads, no epilogue.  ops = CTAs * 2 * iters * 4 * 2 * 64 * 128 * 32.
__device__ __forceinline__ void wgmma_n128_ss(uint32_t (&d)[64], uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(desc_a), "l"(desc_b)
                 : "memory");
}
__global__ void __launch_bounds__(256) i8_mma_peak_kernel(int iters)
{
    extern __shared__ __align__(1024) uint8_t peak_smem[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(peak_smem) + 1023) & ~(uintptr_t)1023);
    for (int i = threadIdx.x; i < (16384 + 32768) / 16; i += 256) sts_u4(smem_u32(sm) + i * 16, 0x01010101u, 0x01020304u, 0x7f7f0101u, 0u);
    fence_proxy_async_smem();
    __syncthreads();
    uint32_t d[64];
#pragma unroll
    for (int i = 0; i < 64; i++) d[i] = 0;
    const uint64_t da = make_smem_desc(smem_u32(sm) + (uint32_t)(threadIdx.x >> 7) * 8192u, 128), db = make_smem_desc(smem_u32(sm) + 16384u, 128);
    wgmma_fence();
    for (int it = 0; it < iters; it++)
    {
#pragma unroll
        for (int k = 0; k < 4; k++) wgmma_n128_ss(d, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < 64; i++) x ^= d[i];
    if (x == 0x9e3779b9u) sts_u4(smem_u32(sm), x, x, x, x); // keeps the accumulators live
}

cudaError_t probe_int8_mma_peak(int num_sms, double* tops, cudaStream_t st)
{
    cudaError_t err = cudaFuncSetAttribute(i8_mma_peak_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    if (err != cudaSuccess) return err;
    cudaEvent_t a, b;
    cudaEventCreate(&a), cudaEventCreate(&b);
    const int iters = 20000;
    double best = 0;
    for (int rep = 0; rep < 4; rep++)
    {
        cudaEventRecord(a, st);
        i8_mma_peak_kernel<<<num_sms, 256, 16384 + 32768 + 1024, st>>>(iters);
        cudaEventRecord(b, st);
        if ((err = cudaEventSynchronize(b)) != cudaSuccess) break;
        float ms = 0;
        cudaEventElapsedTime(&ms, a, b);
        const double t = (double)num_sms * 2.0 * iters * 4.0 * 2.0 * 64 * 128 * 32 / (ms * 1e-3) / 1e12;
        if (rep > 0 && t > best) best = t; // the first repetition is the warm-up
    }
    cudaEventDestroy(a), cudaEventDestroy(b);
    if (err == cudaSuccess) err = cudaGetLastError();
    *tops = best;
    return err;
}

// ---- host side ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode()
{
    static PFN_encodeTiled fn = nullptr;
    if (!fn)
    {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
            qr == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)p;
    }
    return fn;
}

int tmap_encode(void* tmap, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                const uint32_t* elem_strides, int swizzle_bytes)
{
    PFN_encodeTiled enc = get_encode();
    if (!enc) return TB200_ERR_CUDA;
    cuuint64_t d[5], st[5];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; i++) d[i] = dims[i], bx[i] = box[i], es[i] = elem_strides ? elem_strides[i] : 1;
    for (int i = 0; i + 1 < rank; i++) st[i] = strides_bytes[i];
    CUtensorMapSwizzle sw = swizzle_bytes == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                            : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                            : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                  : CU_TENSOR_MAP_SWIZZLE_NONE;
    CUresult r = enc((CUtensorMap*)tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, (cuuint32_t)rank, const_cast<void*>(base), d, st, bx, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : TB200_ERR_CUDA;
}

static int encode_2d(void* tmap, const void* base, uint64_t inner, uint64_t rows, uint64_t pitch, uint32_t box_inner,
                     uint32_t box_rows, int swizzle)
{
    const uint64_t dims[2] = {inner, rows}, strides[1] = {pitch};
    const uint32_t box[2] = {box_inner, box_rows};
    return tmap_encode(tmap, base, 2, dims, strides, box, nullptr, swizzle);
}

bool debug_launch()
{
    static const bool on = getenv("TB200_DEBUG_LAUNCH") != nullptr;
    return on;
}

int gemm_block_n(int ocp)
{
    // N tiles of at most 128 channels: the accumulator image of a stage shares shared memory with the operand ring; the
    // channels are dealt evenly to the fewest such tiles
    const int nt = (ocp + 127) / 128;
    return ((ocp + nt - 1) / nt + 15) & ~15;
}

// m-tiles per accumulator stage and the store-group width.  Several m-tiles share a stage when the CTA stays on one N tile
// anyway (a single N tile): that amortises the per-stage synchronisation over up to ACC_COLS_MAX image columns of work.  A
// store group is 32 rows x 16*cs channels; cs is 2 when that divides the N tile's chunk count and deals the stage's groups
// evenly to the four warps of a 32-row image quarter, else 1.
static void plan_stage(GemmPlan* p)
{
    p->mt = 1;
    if (p->n_tiles == 1)
        while (p->mt < 4 && (p->mt * 2) * p->block_n <= ACC_COLS_MAX && p->mt * 2 <= p->m_tiles) p->mt *= 2;
    const int nch = p->block_n / 16;
    p->cs = (nch % 2 == 0 && (p->mt * (nch / 2)) % 4 == 0) ? 2 : 1;
    p->ngroups = nch / p->cs;
}

// Output tensor maps: a box of 32 rows x one store group; 32-byte groups are swizzled like the warp's staging buffer.
static int plan_epilogue(GemmPlan* p, const void* out, uint64_t d1, uint64_t d2)
{
    const int cs = p->cs;
    const uint64_t dims[3] = {(uint64_t)p->ocp, d1, d2};
    const uint64_t strides[2] = {(uint64_t)p->ldo, (uint64_t)p->ldo * d1};
    const int swz = cs == 2 ? 32 : 0;
    const uint32_t box[3] = {(uint32_t)(16 * cs), 32u, 1u};
    int rc = tmap_encode(p->tmap_out, out, 3, dims, strides, box, nullptr, swz);
    if (rc) return rc;
    const int tail = p->rows_valid % 32;
    const uint32_t box_t[3] = {(uint32_t)(16 * cs), (uint32_t)(tail ? tail : 32), 1u};
    return tmap_encode(p->tmap_out_tail, out, 3, dims, strides, box_t, nullptr, swz);
}

// shared memory the epilogue needs next to the operand ring
static int epilogue_smem_bytes(const GemmPlan* p)
{
    const int par_ch = p->n_tiles * p->block_n;
    return PLAN_STG_WARPS * 2 * 512 * p->cs + (par_ch <= PAR_MAX ? par_ch : p->block_n) * 8 + (int)sizeof(GemmSmemCtl) + 2048 +
           128 * (int)acc_pitch(p->mt * p->block_n) + 16;
}

// Operand ring depth and the resident-B decision.  With the N tile's weights resident the ring carries A tiles only,
// which for the small-K layers (K = 32..128, one 4-16 KB A tile per m-tile) is the difference between 8 and 24 m-tiles
// of prefetch distance.
static int plan_ring(GemmPlan* p)
{
    const int a_bytes = BLOCK_M * p->block_k, b_al = (p->block_n * p->block_k + 1023) & ~1023;
    const int budget = 224 * 1024 - epilogue_smem_bytes(p) - (p->cplane ? 4096 : 0);
    p->b_res = (long long)p->k_blocks * b_al <= B_RESIDENT_MAX ? 1 : 0;
    int stages = p->b_res ? (budget - p->k_blocks * b_al) / a_bytes : budget / (a_bytes + b_al);
    if (p->b_res && stages < 3) p->b_res = 0, stages = budget / (a_bytes + b_al);
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    if (stages < 2) return TB200_ERR_INVALID;
    p->stages = stages;
    return 0;
}

int gemm_plan_create(GemmPlan* p, const void* a, long long lda, const void* b, void* out, long long m, int k, int oc, int ocp, int ldo, int u8)
{
    if (m <= 0 || k <= 0 || (k & 15) || (ocp & 15) || (lda & 15) || (ldo & 15)) return TB200_ERR_INVALID;
    memset(p, 0, sizeof *p);
    p->m = m, p->k = k, p->oc = oc, p->ocp = ocp, p->ldo = ldo, p->out = out;
    p->block_k = k <= 32 ? 32 : (k <= 64 ? 64 : 128);
    p->swizzle = p->block_k;
    p->k_blocks = (k + p->block_k - 1) / p->block_k;
    p->u8 = u8 != 0; // u8 = 1 + weight zero point for uint8 layers
    p->b_signed = !p->u8 || u8 != 1;
    p->cplane = (p->u8 && u8 != 1 && !getenv("TB200_DEBUG_NO_CPLANE")) ? 128 - (u8 - 1) : 0; // (debug switch: WRONG results, timing experiments only)
    p->block_n = gemm_block_n(ocp);
    p->taps = 1;
    p->n_tiles = (ocp + p->block_n - 1) / p->block_n;
    p->m_tiles = (m + BLOCK_M - 1) / BLOCK_M;
    plan_stage(p);
    int rc = plan_ring(p);
    if (rc) return rc;
    rc = encode_2d(p->tmap_a, a, (uint64_t)k, (uint64_t)m, (uint64_t)lda, p->block_k, BLOCK_M, p->swizzle);
    if (rc) return rc;
    rc = encode_2d(p->tmap_b, b, (uint64_t)k, (uint64_t)p->n_tiles * p->block_n, (uint64_t)k, p->block_k, p->block_n, p->swizzle);
    if (rc) return rc;
    p->rows_valid = BLOCK_M, p->out_mode = 0;
    return plan_epilogue(p, out, (uint64_t)m, 1);
}

// Implicit-GEMM plan for a dense (group 1, dilation 1) convolution with any kernel size and stride 1 or 2:
// A = 4-D tensor map (C, W, H, N) over the NHWC input with traversal strides (1, s, s, 1); B = [OCp][taps*Cp].
int gemm_plan_create_conv(GemmPlan* p, const void* in, const void* w, void* out, const ConvShape& s, int u8)
{
    if (s.group != 1 || s.dh != 1 || s.dw != 1 || s.sh != s.sw || (s.sh != 1 && s.sh != 2)) return TB200_ERR_UNSUPPORTED;
    const int taps = s.kh * s.kw;
    if (taps > 1 && (s.cp % 32)) return TB200_ERR_UNSUPPORTED; // a k-block must not straddle two taps
    memset(p, 0, sizeof *p);
    p->conv = 1;
    p->m = (long long)s.n * s.oh * s.ow, p->oc = s.oc, p->ocp = s.ocp, p->ldo = s.ocp, p->out = out;
    if (taps == 1) p->block_k = s.cp <= 32 ? 32 : (s.cp <= 64 ? 64 : 128);
    else p->block_k = (s.cp % 128 == 0) ? 128 : ((s.cp % 64 == 0) ? 64 : 32);
    p->swizzle = p->block_k;
    p->cblocks = (s.cp + p->block_k - 1) / p->block_k;
    p->k_blocks = taps * p->cblocks;
    p->k = taps * s.cp;
    p->u8 = u8 != 0; // u8 = 1 + weight zero point for uint8 layers
    p->b_signed = !p->u8 || u8 != 1;
    p->cplane = (p->u8 && u8 != 1 && !getenv("TB200_DEBUG_NO_CPLANE")) ? 128 - (u8 - 1) : 0; // (debug switch: WRONG results, timing experiments only)
    p->block_n = gemm_block_n(s.ocp);
    p->taps = taps, p->in_h = s.h, p->in_w = s.w;
    if (taps > 64) return TB200_ERR_UNSUPPORTED;
    p->n_tiles = (s.ocp + p->block_n - 1) / p->block_n;
    // output patch of one m-tile: whole rows when they fit (then the patch is contiguous in the NHWC output)
    if (s.ow <= BLOCK_M)
    {
        p->bw = s.ow;
        p->bh = BLOCK_M / s.ow < s.oh ? BLOCK_M / s.ow : s.oh;
        p->bn = (p->bh == s.oh) ? BLOCK_M / (s.ow * s.oh) : 1;
        if (p->bn > s.n) p->bn = s.n;
        if (p->bn < 1) p->bn = 1;
    }
    else
        p->bw = BLOCK_M, p->bh = 1, p->bn = 1;
    p->tiles_w = (s.ow + p->bw - 1) / p->bw;
    p->tiles_h = (s.oh + p->bh - 1) / p->bh;
    const long long tiles_n = (s.n + p->bn - 1) / p->bn;
    p->m_tiles = (long long)p->tiles_w * p->tiles_h * tiles_n;
    p->kw_n = s.kw, p->pad_h = s.ph0, p->pad_w = s.pw0, p->cstride = s.sh, p->cp = s.cp, p->oh = s.oh, p->ow = s.ow, p->nimg = s.n;
    p->a_tx_bytes = (uint32_t)(p->block_k * p->bw * p->bh * p->bn);
    plan_stage(p);
    int rc = plan_ring(p);
    if (rc) return rc;
    const uint64_t dims[4] = {(uint64_t)s.cp, (uint64_t)s.w, (uint64_t)s.h, (uint64_t)s.n};
    const uint64_t strides[3] = {(uint64_t)s.cp, (uint64_t)s.w * s.cp, (uint64_t)s.h * s.w * s.cp};
    const uint32_t box[4] = {(uint32_t)p->block_k, (uint32_t)((p->bw - 1) * s.sw + 1), (uint32_t)((p->bh - 1) * s.sh + 1), (uint32_t)p->bn};
    const uint32_t estr[4] = {1u, (uint32_t)s.sw, (uint32_t)s.sh, 1u};
    if (box[1] > 256 || box[2] > 256 || box[3] > 256) return TB200_ERR_UNSUPPORTED;
    rc = tmap_encode(p->tmap_a, in, 4, dims, strides, box, estr, p->swizzle);
    if (rc) return rc;
    rc = encode_2d(p->tmap_b, w, (uint64_t)p->k, (uint64_t)p->n_tiles * p->block_n, (uint64_t)p->k, p->block_k, p->block_n, p->swizzle);
    if (rc) return rc;
    // The rows of an m-tile are consecutive output pixels along one axis of the NHWC output (see the patch shapes above):
    //   bn > 1 (whole images)   : rows = pixels of bn consecutive images        -> map (C, N*OH*OW, 1), clipped at the end
    //   bn == 1, bw == OW       : rows = pixels of image n from row oh0 on       -> map (C, OH*OW, N), clipped per image
    //   bw == 128 < OW          : rows = 128 pixels of one image row             -> map (C, OW, N*OH), clipped per row
    p->rows_valid = p->bw * p->bh * p->bn;
    if (p->bw != s.ow)
    {
        p->out_mode = 2;
        return plan_epilogue(p, out, (uint64_t)s.ow, (uint64_t)s.n * s.oh);
    }
    if (p->bn > 1)
    {
        p->out_mode = 0;
        return plan_epilogue(p, out, (uint64_t)s.n * s.oh * s.ow, 1);
    }
    p->out_mode = 1;
    return plan_epilogue(p, out, (uint64_t)s.oh * s.ow, (uint64_t)s.n);
}

// debug: event timeline of CTA 0 of the launch that just went out (needs a stream that is not being captured).
// One line per event, sorted by time: cycles since the first event, role (P producer, M mma, E8/E15 epilogue warps), tag.
static void gemm_trace_report(const GemmPlan& p, const GemmArgs& g, int grid, cudaStream_t st)
{
    static unsigned long long h[4 * 1024];
    if (cudaStreamSynchronize(st) != cudaSuccess) return;
    cudaMemcpy(h, g.trace, sizeof h, cudaMemcpyDeviceToHost);
    fprintf(stderr, "[gemm timeline] m_tiles=%lld k_blocks=%d bn=%d mt=%d stages=%d b_res=%d cs=%d grid=%d\n", (long long)p.m_tiles, p.k_blocks,
            p.block_n, p.mt, p.stages, p.b_res, p.cs, grid);
    unsigned long long t0 = ~0ull;
    for (int i = 0; i < 4 * 1024; i++)
        if (h[i] && (h[i] >> 8) < t0) t0 = h[i] >> 8;
    static const char* role[4] = {"P", "M", "E8", "E15"};
    static const char* tagM[3] = {"stage multiplied", "got img_empty", "arrive img_full"};
    static const char* tagE[5] = {"got img_full", "group stored", "arrive sx_empty", "image ld issued", "unit done"};
    for (int r = 0; r < 4; r++)
        for (int i = 0; i < 1024 && h[r * 1024 + i]; i++)
        {
            const unsigned long long v = h[r * 1024 + i];
            const int tag = (int)(v & 0xff);
            fprintf(stderr, "TL %8llu %-3s %s%s%d\n", (v >> 8) - t0, role[r], r == 0 ? "load issued kb=" : (r == 1 ? tagM[tag % 3] : tagE[tag % 5]),
                    r == 0 ? "" : " #", r == 0 ? tag : i);
        }
}

cudaError_t launch_gemm_i8(const GemmPlan& p, const EpiParams& e, const int32_t* btab, int num_sms, cudaStream_t st)
{
    if (p.block_n <= 0 || p.mt <= 0 || p.stages <= 0 || p.cs <= 0) return cudaErrorInvalidValue; // plan was never created
    GemmArgs g;
    g.m_tiles = (int)p.m_tiles, g.k_blocks = p.k_blocks, g.n_tiles = p.n_tiles, g.block_n = p.block_n;
    g.conv = p.conv, g.cblocks = p.cblocks, g.kw_n = p.kw_n, g.pad_h = p.pad_h, g.pad_w = p.pad_w, g.cstride = p.cstride, g.cp = p.cp;
    g.bw = p.bw, g.bh = p.bh, g.bn = p.bn, g.tiles_w = p.tiles_w, g.tiles_h = p.tiles_h, g.oh = p.oh, g.ow = p.ow, g.nimg = p.nimg;
    g.a_tx_bytes = p.a_tx_bytes;
    g.u8 = p.u8, g.taps = p.taps, g.in_h = p.in_h, g.in_w = p.in_w, g.btab = btab, g.b_signed = p.b_signed, g.cplane = p.cplane;
    g.fixq = (uint4*)p.fixq, g.fixq_cap = p.fixq_cap, g.out_base = (uint8_t*)p.out, g.ldo = p.ldo, g.m_rows = (int)p.m;
    g.mt = p.mt;
    g.num_super = (int)(((p.m_tiles + p.mt - 1) / p.mt) * p.n_tiles);
    g.bw_rcp = p.conv ? (65536u + (uint32_t)p.bw - 1) / (uint32_t)p.bw : 0;
    g.bh_rcp = p.conv ? (65536u + (uint32_t)p.bh - 1) / (uint32_t)p.bh : 0;
    g.block_k = p.block_k, g.stages = p.stages, g.swizzle = p.swizzle, g.oc = p.oc, g.ocp = p.ocp;
    g.cs = p.cs, g.ngroups = p.ngroups, g.rows_valid = p.rows_valid, g.out_mode = p.out_mode;
    const int par_ch = p.n_tiles * p.block_n;
    g.par_all = par_ch <= PAR_MAX ? 1 : 0;
    const int a_bytes = BLOCK_M * p.block_k, b_bytes = (p.block_n * p.block_k + 1023) & ~1023;
    g.b_res = p.b_res;
    const size_t smem = (size_t)p.stages * (a_bytes + (p.b_res ? 0 : b_bytes)) + (p.b_res ? (size_t)p.k_blocks * b_bytes : 0) + (p.cplane ? 4096 : 0) +
                        (size_t)EPI_WARPS * 2 * 512 * p.cs + sizeof(GemmSmemCtl) +
                        (size_t)(g.par_all ? par_ch : p.block_n) * 8 + 16 + 128 * (size_t)acc_pitch(p.mt * p.block_n) + 1024;
    static const bool trace_on = getenv("TB200_GEMM_TRACE") != nullptr;
    const bool launch_dbg = debug_launch();
    static unsigned long long* trace_buf = nullptr;
    g.trace = nullptr;
    if (trace_on)
    {
        if (!trace_buf) cudaMalloc(&trace_buf, 4 * 1024 * sizeof(unsigned long long));
        cudaMemsetAsync(trace_buf, 0, 4 * 1024 * sizeof(unsigned long long), st);
        g.trace = trace_buf;
    }
    int grid = (int)(g.num_super < num_sms ? g.num_super : num_sms);
    if (p.b_res) grid -= grid % p.n_tiles; // a CTA must see one N tile only (num_super is a multiple of n_tiles, so grid >= n_tiles)
    CUtensorMap ta, tb, to, tt;
    memcpy(&ta, p.tmap_a, sizeof ta);
    memcpy(&tb, p.tmap_b, sizeof tb);
    memcpy(&to, p.tmap_out, sizeof to);
    memcpy(&tt, p.tmap_out_tail, sizeof tt);
    const int mode = !e.fast_ok ? 2 : ((!p.u8 && e.fuse_bias) ? 1 : 0);
    cudaError_t err = cudaErrorInvalidValue;
    // uint8 border corrections only exist for convolutions with taps that can fall into the padding: any window larger than one
    // pixel, or a 1x1 window whose last row / column lies past the image (bottom / right padding, e.g. TF-style (0, 1))
    const bool pad_1x1 = p.pad_h || p.pad_w || (p.oh - 1) * p.cstride >= p.in_h || (p.ow - 1) * p.cstride >= p.in_w;
    const bool border = p.u8 && p.conv && (p.taps > 1 || pad_1x1);
#define TB200_GEMM_CASE(U, MD, C, B)                                                                                           \
    if ((p.u8 != 0) == U && mode == MD && p.cs == C && border == B)                                                            \
    {                                                                                                                          \
        /* the opt-in is per device AND per context: set it before every launch (launches happen at graph capture only) */ \
        {                                                                                                                      \
            err = cudaFuncSetAttribute(gemm_i8_tcgen05_kernel<U, MD, C, B>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024); \
            if (launch_dbg) gemm_launch_debug((const void*)gemm_i8_tcgen05_kernel<U, MD, C, B>, "set attribute", err, grid, smem, st);    \
            if (err != cudaSuccess) return err;                                                                                \
        }                                                                                                                      \
        if (launch_dbg)                                                                                                        \
            fprintf(stderr, "tengine_b200: launch gemm_i8_tcgen05_kernel<U8=%d,MODE=%d,CS=%d,BORDER=%d> out_mode=%d conv=%d n_tiles=%d b_res=%d fixq=%d mt=%d par_all=%d\n", \
                    (int)U, MD, C, (int)B, p.out_mode, p.conv, p.n_tiles, p.b_res, p.fixq != nullptr, p.mt, g.par_all);     \
        gemm_i8_tcgen05_kernel<U, MD, C, B><<<grid, GEMM_THREADS, smem, st>>>(ta, tb, to, tt, g, e);                                                \
        if (trace_on) gemm_trace_report(p, g, grid, st);                                                                       \
        err = cudaGetLastError();                                                                                              \
        if (launch_dbg || err != cudaSuccess) gemm_launch_debug((const void*)gemm_i8_tcgen05_kernel<U, MD, C, B>, "launch", err, grid, smem, st); \
        return err;                                                                                                            \
    }
#define TB200_GEMM_CS(U, MD, B) TB200_GEMM_CASE(U, MD, 1, B) TB200_GEMM_CASE(U, MD, 2, B)
    TB200_GEMM_CS(false, 0, false)
    TB200_GEMM_CS(false, 1, false)
    TB200_GEMM_CS(false, 2, false)
    TB200_GEMM_CS(true, 0, false)
    TB200_GEMM_CS(true, 2, false)
    TB200_GEMM_CS(true, 0, true)
    TB200_GEMM_CS(true, 2, true)
#undef TB200_GEMM_CS
#undef TB200_GEMM_CASE
    return err;
}

} // namespace tb200
