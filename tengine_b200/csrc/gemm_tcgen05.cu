// gemm_tcgen05.cu -- int8 x int8 -> int32 GEMM on the Hopper tensor cores (wgmma.mma_async .s32.s8/.u8, m64n16k32)
// with TMA-staged operands, a shared-memory accumulator image and the fused requantising epilogue.
//
//   out[m][oc] = requant( sum_k A[m][k] * B[oc][k] ),   A = NHWC activations (row = pixel, K = padded Cin),
//                                                        B = pre-packed weights [OCp][K], both K-major.
// This is the device's form of the reference's im2col + sgemm_i8 + sgemm_int8 epilogue for 1x1 convolutions
// (source/device/cpu/op/conv/x86/conv_kernel_x86.c:187-242, 1008-1631, 1796-1893) and of ref_fc_int8
// (fc/fc_ref.c:209-297): with NHWC activations a 1x1 convolution IS this GEMM, no im2col pass exists.
//
// Structure (one persistent CTA per SM, 544 threads):
//   warp 16   : TMA producer  (cp.async.bulk.tensor.2d -> 128B/64B/32B-swizzled smem ring, mbarrier expect_tx)
//   warps 0-15: four warpgroups that first multiply, then requantise.  MMA: warpgroup w takes rows 64*(w & 1).. and one
//               half of the N tile's 16-column chunks, issues wgmma per ring stage, releases the stage after
//               wgmma.wait_group and finally writes its s32 fragments into the accumulator image ([128 rows][BN] in
//               shared memory).  Epilogue: four warps per 32-row quarter of the image; a warp owns whole "store groups"
//               = 32 rows x 16/32/64 channels: image -> registers -> requant_fast4_i8 -> bytes -> its own swizzled smem
//               buffer -> ONE TMA store per group (cp.async.bulk.tensor, double-buffered).  No address arithmetic for the
//               stores, rows outside the tensor are clipped by the TMA unit.
// The producer runs ahead through the ring while the epilogue works, so the next tile's operands are resident when its
// MMAs start.  K is small (32..1024), so these layers are bound by the epilogue's ALU-pipe issue rate, not by the tensor
// pipe: see common.cuh (requant_fast4_i8) for the instruction budget.
#include <cuda.h>

#include "common.cuh"
#include "kernels.h"
#include "ptx.cuh"
#include "tc_common.cuh"

#include <cstdio>
#include <cstdlib>

namespace tb200 {

#ifdef TB200_GEMM_TIMELINE
#define TLOG_E(tag) do { if (lane == 0 && (warp == 0 || warp == 15)) tlog(warp == 0 ? 2 : 3, tag); } while (0)
#else
#define TLOG_E(tag) do { } while (0)
#endif


static constexpr int EPI_WARPS = 16; // four warpgroups; four warps per 32-row quarter of the accumulator image
static constexpr int EPI_THREADS = EPI_WARPS * 32;
static constexpr int GEMM_THREADS = 32 + EPI_THREADS;
static constexpr int SUM_WARP0 = EPI_WARPS + 1, SUM_WARPS = 2; // uint8 kernels only: two warps that add up the rows of every A tile (sum x)
static constexpr int GEMM_THREADS_U8 = GEMM_THREADS + 32 * SUM_WARPS;
static constexpr int PRODUCER_WARP = EPI_WARPS;
static constexpr int ACC_COLS_MAX = 144; // columns of the accumulator image (m-tiles per stage x B tile rows)
static constexpr int MMA_CHUNKS = 5;     // 16-column chunks of one warpgroup: half of at most 144 columns
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
    int u8, bnx, taps, in_h, in_w, b_signed, cplane;
    int sx_mode; // where sum(x) comes from when cplane != 0: 3 = two extra warps add up the rows of every A tile in shared memory (default), 0 = 16 rows of ones inside every B tile (TB200_U8_SX=0)
    int tcols; // accumulator image columns per m-tile: bnx (block_n, + 16 when 16 rows of ones in B form sum(x))
    // epilogue / stores
    int cs, ngroups; // 16-column chunks per store group (1, 2 or 4) and groups per m-tile
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
};

__device__ __forceinline__ void epilogue_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory"); }

// ---- the rare path of the fast epilogue, deferred -----------------------------------------------------------------------------
// An element whose t sits inside the tie guard needs the literal reference arithmetic (common.cuh requant(): divisions, per-channel
// loads, every recipe).  Done inline it occupies ONE lane of an epilogue warp for hundreds of cycles while the other fifteen warps
// finish their groups and then wait for it at the stage hand-over.  Instead the lane appends {m-tile, row, channel, accumulator} to the CTA's queue in
// global memory (L2) and carries on with the fast byte; after the CTA's last tile all 512 epilogue threads recompute the queued
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

// After the CTA's last tile (every epilogue warp has waited for its own bulk stores): recompute the queued elements, one per thread.
template <bool U8>
__device__ __forceinline__ void fixq_drain(const GemmArgs& g, const EpiParams& e)
{
    const uint32_t n = s_fixq.count < s_fixq.cap ? s_fixq.count : s_fixq.cap;
    for (uint32_t k = threadIdx.x; k < n; k += EPI_THREADS)
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
    if (!g.conv || g.taps == 1 && g.pad_h == 0 && g.pad_w == 0) return 0;
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

// MODE: 0 fast epilogue, 1 fast epilogue with the bias folded into the FMA (int8 only), 2 exact epilogue.
// CS: 16-column chunks per store group (1, 2, 4 or 8).  Compile-time so that each kernel carries exactly one epilogue body.
// CS == 8: a group is 32 rows x 128 bytes filled by a PAIR of warps (64 bytes each) and stored by one of them: the TMA
// unit's cost is per row (~4 cycles for anything up to 128 bytes), so 128-byte rows halve the store side's share of it.
template <bool U8, int MODE, int CS, bool BORDER>
__global__ void __launch_bounds__(U8 ? GEMM_THREADS_U8 : GEMM_THREADS, 1)
    gemm_i8_tcgen05_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                           const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_out_tail,
                           const GemmArgs g, const __grid_constant__ EpiParams e)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // operand ring first (1024-byte aligned for the 128B swizzle), then the per-warp output staging buffers (1024-byte
    // aligned: their TMA swizzle pattern is a function of the address), the control block and the epilogue constants
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t a_bytes = BLOCK_M * g.block_k, b_bytes = g.bnx * g.block_k;
    const uint32_t b_al = (b_bytes + 1023) & ~1023u;
    const uint32_t stage_bytes = a_bytes + (g.b_res ? 0u : b_al);
    uint8_t* b_region = smem + (size_t)g.stages * stage_bytes; // resident-B mode: [k_blocks][b_al]
    constexpr uint32_t buf_bytes = 512u * CS; // 32 rows x 16*CS bytes
    constexpr int WCH = CS == 8 ? 4 : CS;     // chunks one warp requantises per group
    uint8_t* sxs = b_region + (g.b_res ? (size_t)g.k_blocks * b_al : 0); // uint8: sum(x) of the rows, [2 accumulator stages][4 m-tiles][128] int32
    uint8_t* stg = sxs + (g.cplane ? 4096u : 0u);
    const uint32_t sx_base = smem_u32(sxs);
    const uint32_t stg_base = smem_u32(stg);
    GemmSmemCtl* ctl = reinterpret_cast<GemmSmemCtl*>(stg + (size_t)(CS == 8 ? EPI_WARPS / 2 : EPI_WARPS) * 2 * buf_bytes);
    const uint32_t par_base = smem_u32(ctl) + (uint32_t)sizeof(GemmSmemCtl); // [par channels] x 8 bytes (see FastPar4)
    const int acc_cols = g.mt * g.tcols; // accumulator image columns of one stage
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
        const uint32_t sumw = (U8 && g.sx_mode == 3) ? SUM_WARPS : 0; // the row-sum warps read every operand stage and publish with the accumulators
        for (int s = 0; s < g.stages; s++) mbar_init(&ctl->full[s], 1), mbar_init(&ctl->empty[s], EPI_WARPS + sumw);
        for (int s = 0; s < 2; s++) mbar_init(&ctl->sx_full[s], sumw ? sumw : 1), mbar_init(&ctl->sx_empty[s], EPI_WARPS);
        mbar_init(&ctl->b_full, 1);
        s_fixq.q = g.fixq ? g.fixq + (size_t)blockIdx.x * g.fixq_cap : nullptr, s_fixq.cap = (uint32_t)g.fixq_cap, s_fixq.count = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

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
                const int nb = (blockIdx.x % g.n_tiles) * g.bnx;
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
                const int n0 = ntile * g.bnx; // row of this N tile in the packed weight matrix
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
    else if (U8 && warp >= SUM_WARP0)
    {
        // ===================== row sums (uint8, warps 18 and 19) =====================
        // sum x*(w - zw) = sum x*(w - 128) [tensor cores, B signed] + (128 - zw) * sum(x).  sum(x) of output row r is the sum of ALL bytes
        // of row r of every A tile of the m-tile (taps outside the image were zero-filled by the TMA unit, K tails too), and a sum
        // does not care about the swizzle that permutes the 16-byte chunks inside a row.  Each of the two warps owns 64 rows (two per
        // lane), reads them with 16-byte loads (chunk order rotated per lane so that a quarter-warp covers all banks), dp4a against
        // 0x01010101, and publishes the sums through shared memory together with the accumulator stage.  This keeps the uint8 tiling
        // identical to the int8 one: no extra B rows, no extra accumulator columns, no second MMA.
        if (g.sx_mode == 3)
        {
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
    else
    {
        // ===================== MMA + epilogue (warps 0..15) =====================
        // Image quarter q (rows 32q..32q+31) is served by the four warps {q, q+4, q+8, q+12}.  The work of an accumulator
        // stage is cut into store groups (m-tile i, columns [grp*16*cs, (grp+1)*16*cs)) of 32 rows each, dealt round-robin to
        // the quarter's warps.  A warp requantises its group chunk by chunk (16 columns per load, the next chunk's load in
        // flight), writes the bytes to its own swizzled staging buffer and hands the buffer to the TMA unit with one store.
        const int q = warp & 3;
        const int sub = warp >> 2;
        const int ngroups = g.ngroups;
        // MMA share of this warpgroup (= sub): rows 64*mh.., chunks [c_lo, c_lo + c_n) of every B tile
        const int mh = sub & 1, nch = g.tcols >> 4, chalf = (nch + 1) >> 1;
        const int c_lo = (sub >> 1) ? chalf : 0, c_n = (sub >> 1) ? nch - chalf : chalf;
        const uint32_t a_bytes_mma = BLOCK_M * g.block_k, b_al_mma = (g.bnx * g.block_k + 1023) & ~1023u;
        int stage = 0;
        uint32_t phase = 0;
        if (g.b_res) mbar_wait(&ctl->b_full, 0);
        int qrows = g.rows_valid - q * 32; // rows of this quarter that are output pixels
        qrows = qrows < 0 ? 0 : (qrows > 32 ? 32 : qrows);
        const CUtensorMap* tm_out = (qrows == 32) ? &tmap_out : &tmap_out_tail;
        const int half = CS == 8 ? (sub & 1) : 0;        // which 64-byte half of the pair's 128-byte rows this warp fills
        const int pair = q * 2 + (sub >> 1);             // CS == 8: staging buffers and the named barrier are per pair
        const uint32_t buf0 = stg_base + (uint32_t)(CS == 8 ? pair : warp) * 2u * buf_bytes;
        // swizzle of the staging buffer = the output map's swizzle: 16-byte chunk index ^= row bits (Swizzle<1|2|3,4,3>)
        const uint32_t xl = CS == 8   ? (uint32_t)(lane & 7) << 4
                            : CS == 4 ? (uint32_t)((lane >> 1) & 3) << 4
                                      : (CS == 2 ? (uint32_t)((lane >> 2) & 1) << 4 : 0u);
        const uint32_t row_off = (uint32_t)lane * 16u * CS;
        const int gfirst = CS == 8 ? (sub >> 1) : sub, gstep = CS == 8 ? 2 : 4;
        auto pair_sync = [&]() { asm volatile("bar.sync %0, 64;" ::"r"(2 + pair) : "memory"); };
        uint32_t ucount = 0; // groups this warp has stored (buffer parity)
        const int par_ch = g.n_tiles * g.block_n;
        const bool fast = MODE != 2;
        if (g.par_all)
        {
            // per-channel fast-path constants of every N tile, once; pad / overhanging channels get (0, 0)
            for (int c = threadIdx.x; c < par_ch; c += EPI_THREADS)
                sts_f2(par_base + c * 8, (c < g.ocp && (fast || U8)) ? __ldg(e.fast_par + c) : make_float2(0.f, 0.f));
            epilogue_bar_sync();
        }
        if (lane == 0 && qrows > 0) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm_out)) : "memory");
        int as = 0;
        uint32_t aphase = 0;
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
                epilogue_bar_sync(); // every warp is done with the previous tile's constants
                for (int c = threadIdx.x; c < g.block_n; c += EPI_THREADS)
                    sts_f2(par_base + c * 8, (n0 + c < g.ocp && (fast || U8)) ? __ldg(e.fast_par + n0 + c) : make_float2(0.f, 0.f));
                epilogue_bar_sync();
                par_s = par_base;
            }
            // ---- MMA: every m-tile of the stage into the accumulator image ----
            epilogue_bar_sync(); // every warp has read the previous stage's image
            for (int i = 0; i < mtc; i++)
            {
                uint32_t acc[MMA_CHUNKS][8];
#pragma unroll
                for (int j = 0; j < MMA_CHUNKS; j++)
#pragma unroll
                    for (int r = 0; r < 8; r++) acc[j][r] = 0;
                for (int kb = 0; kb < g.k_blocks; kb++)
                {
                    mbar_wait(&ctl->full[stage], phase); // TMA bytes have landed
                    const uint32_t sa = smem_u32(smem + (size_t)stage * stage_bytes);
                    const uint32_t sb = g.b_res ? smem_u32(b_region) + (uint32_t)kb * b_al_mma : sa + a_bytes_mma;
                    const uint64_t da = make_smem_desc(sa + (uint32_t)(mh * 64 * g.swizzle), g.swizzle);
                    const uint64_t db = make_smem_desc(sb + (uint32_t)(c_lo * 16 * g.swizzle), g.swizzle);
                    wgmma_fence();
                    for (int k = 0; k < g.block_k / 32; k++)
#pragma unroll
                        for (int j = 0; j < MMA_CHUNKS; j++)
                            if (j < c_n)
                            {
                                // +32 bytes along K inside the swizzled rows: +2 in 16-byte units; +16 rows of B: +16*swizzle bytes
                                const uint64_t a_d = da + (uint64_t)(k * 2), b_d = db + (uint64_t)(j * g.swizzle + k * 2);
                                if (U8 && !g.b_signed) wgmma_n16<true, true>(acc[j], a_d, b_d, 1u);
                                else wgmma_n16<U8, false>(acc[j], a_d, b_d, 1u);
                            }
                    wgmma_commit();
                    wgmma_wait<0>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&ctl->empty[stage]); // this warp's MMAs have read the stage
                    if (++stage == g.stages) stage = 0, phase ^= 1;
                }
#pragma unroll
                for (int j = 0; j < MMA_CHUNKS; j++)
                    if (j < c_n) frag_to_image(acc[j], img_base, img_pitch, mh * 64, i * g.tcols + (c_lo + j) * 16);
            }
            epilogue_bar_sync(); // the image is complete
            if (U8 && g.sx_mode == 3) mbar_wait(&ctl->sx_full[as], aphase); // the row sums of this stage
            TLOG_E(0);
            const uint32_t tbase = img_base + (uint32_t)(q * 32 + lane) * img_pitch;
            if (qrows > 0)
            {
                // groups of this warp: flattened index u = i * ngroups + grp, u = sub, sub + 4, ...
                uint32_t v0[16], v1[16];
                int i = 0, grp = gfirst;
                while (grp >= ngroups) grp -= ngroups, i++;
                if (CS > 1 && i < mtc)
                    acc_ld16(tbase + 4u * (i * g.tcols + grp * (CS * 16) + half * 64), reinterpret_cast<uint32_t(&)[16]>(v0));
                while (i < mtc)
                {
                    int i2 = i, g2 = grp + gstep; // the group after this one
                    while (g2 >= ngroups) g2 -= ngroups, i2++;
                    const uint32_t buf = buf0 + (ucount & 1u) * buf_bytes;
                    // the store issued two groups ago has finished reading this buffer
                    if (lane == 0 && half == 0) bulk_wait_read<1>();
                    if (CS == 8) pair_sync();
                    else __syncwarp();
                    uint32_t pad = 0;
                    int32_t rowc = 0;
                    if (U8)
                    {
                        // the pixel's sum(x), once per group
                        if (g.cplane)
                        {
                            if (g.sx_mode == 3)
                            {
                                int32_t sx;
                                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(sx) : "r"(sx_base + (uint32_t)(((as * 4 + i) * 128 + q * 32 + lane) * 4)));
                                rowc = g.cplane * sx;
                            }
                            else
                                rowc = g.cplane * (int32_t)acc_ld1(tbase + 4u * (i * g.tcols + g.block_n)); // the column of the ones rows in B
                        }
                        if (BORDER) pad = padding_taps(g, mt0 + i, q * 32 + lane);
                    }
                    const uint32_t tg = tbase + 4u * (i * g.tcols + grp * (CS * 16) + half * 64);
                    const int cg0 = grp * (CS * 16); // first column of the group inside the N tile
                    const uint32_t sdst = buf + row_off;
                    auto unit = [&](const uint32_t (&v)[16], int k)
                    {
                        const int c = cg0 + half * 64 + k * 16;
                        const uint32_t dst = sdst + (((uint32_t)(half * 4 + k) << 4) ^ xl);
                        if (U8) epilogue_unit_u8<MODE == 2, BORDER>(v, rowc, pad, g, par_s + c * 8, dst, n0 + c, (uint32_t)(mt0 + i), e);
                        else if (MODE == 2) epilogue_unit_exact(v, dst, n0 + c, g.oc, e);
                        else epilogue_unit_fast<MODE == 1>(v, par_s + c * 8, dst, n0 + c, (uint32_t)(mt0 + i), e);
                    };
                    if (CS == 1)
                    {
                        acc_ld16(tg, reinterpret_cast<uint32_t(&)[16]>(v0));
                        unit(reinterpret_cast<const uint32_t(&)[16]>(v0), 0);
                    }
                    else
                    {
#pragma unroll
                        for (int k = 0; k < WCH; k++)
                        {
                            TLOG_E(3);
                            // the next chunk's accumulators are in flight while this one is requantised
                            if (k + 1 < WCH) acc_ld16(tg + (k + 1) * 64, reinterpret_cast<uint32_t(&)[16]>(*((k & 1) ? v0 : v1)));
                            else if (i2 < mtc) acc_ld16(tbase + 4u * (i2 * g.tcols + g2 * (CS * 16) + half * 64), reinterpret_cast<uint32_t(&)[16]>(v0));
                            unit(reinterpret_cast<const uint32_t(&)[16]>(*((k & 1) ? v1 : v0)), k);
                            TLOG_E(4);
                        }
                    }
                    fence_proxy_async_smem(); // generic-proxy writes -> visible to the TMA unit
                    if (CS == 8) pair_sync();
                    else __syncwarp();
                    if (lane == 0 && half == 0)
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
            if (lane == 0) mbar_arrive(&ctl->sx_empty[as]); // stage drained: the row-sum warps may overwrite its sums
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

// ---- stem on the tensor cores ------------------------------------------------------------------------------
// First convolution of a network: NCHW int8 input with C <= 3 channels (as the application hands it over), 3x3 filter,
// any stride / padding -> NHWC output.  K = C*9 <= 27 is padded to ONE 32-byte wgmma k-step: the 128 threads of a CTA
// each gather the 27 input bytes of one output pixel, write them as one row of a SW32 K-major A tile, the warpgroup
// multiplies it (128 x OCp x 32) into the shared-memory accumulator image, and every thread requantises its own row and
// writes OCp contiguous bytes.
// Replaces ~290 dp4a per pixel of the CUDA-core stem kernel (kernels_direct.cu) by one MMA; the work left is the gather
// (~80 instructions) and the epilogue.  Several CTAs per SM overlap each other.
// Takes the role of the first im2col + sgemm of conv_hcl_run (conv_kernel_x86.c:187-242).
struct StemArgs
{
    const uint8_t* in;  // NCHW
    const uint8_t* w;   // [OCp][32]: k = (c*3 + kh)*3 + kw, zero padded
    uint8_t* out;       // NHWC, OCp bytes per pixel
    int n, c, h, w_in, oh, ow, ocp, oc, stride, ph, pw;
    unsigned npix, ntiles;
    int tiles_w, tiles_h, box_w, box_h, in_bytes; // TMA-staged input window (16 x 8 output pixels per tile)
    int xoff; // the window starts xoff bytes left of the first tap: the innermost TMA coordinate must be 16-byte aligned
};

// TMA_IN: the input window of the tile (3 channel planes x box_h rows x box_w bytes, zero-filled outside the image) is
// staged in shared memory by one 4-D TMA load, double-buffered; the gather is then 27 unpredicated LDS.U8 + IMAD per
// pixel.  Without it (image width not a multiple of 16) every thread gathers from global memory with bounds predicates,
// which costs more instructions than the whole epilogue.
template <int MODE, bool TMA_IN> // MODE: 0 fast, 1 fast + fused bias, 2 exact
__global__ void __launch_bounds__(128) stem_tc_kernel(const __grid_constant__ CUtensorMap tmap_in, const StemArgs a, const __grid_constant__ EpiParams e)
{
    extern __shared__ __align__(1024) uint8_t stem_smem[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(stem_smem) + 1023) & ~(uintptr_t)1023);
    const uint32_t sA = smem_u32(sm), sB = sA + 4096, sPar = sB + (uint32_t)a.ocp * 32u;
    const uint32_t in_stride = ((uint32_t)a.in_bytes + 127u) & ~127u;
    const uint32_t sIn = (sPar + (uint32_t)a.ocp * 8u + 127u) & ~127u;
    const uint32_t pitch = acc_pitch(a.ocp), sImg = sIn + 2u * in_stride; // accumulator image [128][pitch]
    __shared__ __align__(8) uint64_t in_full[2];
    const int tid = threadIdx.x;
    const int tw = tid & 15, th = tid >> 4; // TMA_IN: the tile is 16 x 8 output pixels

    if (tid == 0)
    {
        mbar_init(&in_full[0], 1), mbar_init(&in_full[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto tile_coords = [&](unsigned tile, int& n, int& oh0, int& ow0)
    {
        const unsigned r = tile / (unsigned)a.tiles_w;
        ow0 = (int)(tile - r * a.tiles_w) * 16;
        n = (int)(r / (unsigned)a.tiles_h);
        oh0 = (int)(r - (unsigned)n * a.tiles_h) * 8;
    };
    // (kept in the kernel body: the tensor map must be addressed as the kernel parameter itself, which a lambda that is
    //  not inlined does not guarantee -- compute-sanitizer: illegal instruction at the cp.async.bulk.tensor)
#define TB200_STEM_LOAD_TILE(TILE, BUF)                                                                                               \
    do                                                                                                                                \
    {                                                                                                                                 \
        int n_, oh0_, ow0_;                                                                                                           \
        tile_coords((TILE), n_, oh0_, ow0_);                                                                                          \
        mbar_expect_tx(&in_full[(BUF)], (uint32_t)a.in_bytes);                                                                        \
        tma_load_4d(&tmap_in, &in_full[(BUF)], sm + (sIn - sA) + (size_t)(BUF) * in_stride, ow0_ * a.stride - a.pw - a.xoff, oh0_ * a.stride - a.ph, \
                    0, n_);                                                                                                           \
    } while (0)
    if (TMA_IN && tid == 0 && blockIdx.x < a.ntiles) TB200_STEM_LOAD_TILE(blockIdx.x, 0);
    // ---- B tile and the epilogue constants (identical for every CTA; L2 / L1 resident) ----
    for (int i = tid; i < a.ocp * 2; i += 128)
    {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(a.w) + i);
        sts_u4(sB + sw32_offset(i >> 1, i & 1), v.x, v.y, v.z, v.w);
    }
    for (int c = tid; c < a.ocp; c += 128) sts_f2(sPar + c * 8, (MODE != 2) ? __ldg(e.fast_par + c) : make_float2(0.f, 0.f));

    uint32_t it = 0;
    for (unsigned tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x, it++)
    {
        uint32_t row[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        unsigned pix;
        bool valid;
        if (TMA_IN)
        {
            int n, oh0, ow0;
            tile_coords(tile, n, oh0, ow0);
            const int oh = oh0 + th, ow = ow0 + tw;
            valid = oh < a.oh && ow < a.ow;
            pix = ((unsigned)n * a.oh + oh) * a.ow + ow;
            const int buf = it & 1;
            mbar_wait(&in_full[buf], (it >> 1) & 1);
            const uint32_t base = sIn + (uint32_t)buf * in_stride + (uint32_t)((th * a.stride) * a.box_w + tw * a.stride + a.xoff);
#pragma unroll
            for (int c = 0; c < 3; c++)
            {
                if (c < a.c)
                {
#pragma unroll
                    for (int kh = 0; kh < 3; kh++)
#pragma unroll
                        for (int kw = 0; kw < 3; kw++)
                        {
                            uint32_t b;
                            asm volatile("ld.shared.u8 %0, [%1];" : "=r"(b) : "r"(base + (uint32_t)((c * a.box_h + kh) * a.box_w + kw)));
                            const int k = (c * 3 + kh) * 3 + kw; // compile-time after unrolling
                            row[k >> 2] += b << (8 * (k & 3)); // disjoint bytes: add == or (IMAD, off the ALU pipe)
                        }
                }
            }
        }
        else
        {
            // ---- gather the 3x3 x C window from the NCHW planes in global memory ----
            pix = tile * 128u + (unsigned)tid;
            valid = pix < a.npix;
            if (valid)
            {
                const unsigned prow = pix / (unsigned)a.ow;
                const int ow = (int)(pix - prow * a.ow);
                const int n = (int)(prow / (unsigned)a.oh);
                const int oh = (int)(prow - (unsigned)n * a.oh);
                const int iy0 = oh * a.stride - a.ph, ix0 = ow * a.stride - a.pw;
                const size_t plane = (size_t)a.h * a.w_in;
                const uint8_t* img = a.in + (size_t)n * a.c * plane;
#pragma unroll
                for (int c = 0; c < 3; c++)
                {
                    if (c < a.c)
                    {
#pragma unroll
                        for (int kh = 0; kh < 3; kh++)
                        {
                            const int iy = iy0 + kh;
                            const bool rok = iy >= 0 && iy < a.h;
                            const uint8_t* rp = img + (size_t)c * plane + (size_t)(rok ? iy : 0) * a.w_in;
#pragma unroll
                            for (int kw = 0; kw < 3; kw++)
                            {
                                const int ix = ix0 + kw;
                                const uint32_t b = (rok && ix >= 0 && ix < a.w_in) ? (uint32_t)__ldg(rp + ix) : 0u;
                                const int k = (c * 3 + kh) * 3 + kw;
                                row[k >> 2] |= b << (8 * (k & 3));
                            }
                        }
                    }
                }
            }
        }
        sts_u4(sA + sw32_offset(tid, 0), row[0], row[1], row[2], row[3]);
        sts_u4(sA + sw32_offset(tid, 1), row[4], row[5], row[6], row[7]);
        fence_proxy_async_smem(); // the MMA reads these generic-proxy writes through the async proxy
        __syncthreads();          // (first iteration: also publishes the B tile and the constants)
        // everybody has read this tile's window: prefetch the next one into the other buffer
        if (TMA_IN && tid == 0 && tile + gridDim.x < a.ntiles) TB200_STEM_LOAD_TILE(tile + gridDim.x, (it + 1) & 1);
        wg_mma_to_image<false, false>(sA, 0u, sB, 0u, 1, 32, a.ocp, sImg, pitch);
        __syncthreads();

        // ---- epilogue: thread = pixel = accumulator row, 16 channels per load, OCp contiguous output bytes per pixel ----
        uint8_t* op = a.out + (size_t)pix * a.ocp;
        const uint32_t tb = sImg + (uint32_t)tid * pitch;
        for (int c = 0; c < a.ocp; c += 16)
        {
            uint32_t v[16];
            acc_ld16(tb + 4u * c, v);
            uint32_t w[4];
            if (MODE == 2)
            {
#pragma unroll
                for (int k = 0; k < 16; k++)
                {
                    if ((k & 3) == 0) w[k >> 2] = 0;
                    if (c + k < a.oc) w[k >> 2] |= ((uint32_t)requant((int32_t)v[k], c + k, e) & 0xffu) << (8 * (k & 3));
                }
            }
            else
                stem_unit_fast<MODE == 1>(v, sPar + c * 8, c, e, w);
            if (valid) *reinterpret_cast<uint4*>(op + c) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        // the next tile's MMA overwrites the accumulator image and its gather overwrites the A tile
        __syncthreads();
    }
}

#undef TB200_STEM_LOAD_TILE

bool stem_tc_supported(const ConvShape& s, const EpiParams& e)
{
    return !e.is_uint8 && s.kh == 3 && s.kw == 3 && s.c <= 3 && s.group == 1 && s.dh == 1 && s.dw == 1 && s.sh == s.sw && s.ocp <= 256 &&
           (long long)s.n * s.oh * s.ow < (1ll << 31);
}

// Tensor map over the NCHW network input for the TMA-staged variant: dims (W, H, C, N), box (box_w, box_h, C, 1).
int stem_plan_create(DwPlan* p, const void* in, const ConvShape& s)
{
    p->valid = 0;
    if (s.w % 16 || getenv("TB200_STEM_NO_TMA")) return -1; // global strides of a tensor map are multiples of 16 bytes
    // innermost coordinate = ow0*S - pw - xoff must be a multiple of 16 (ow0*S is a multiple of 16*S)
    const int xoff = (16 - (((-s.pw0) % 16) + 16) % 16) % 16 == 0 ? 0 : ((((-s.pw0) % 16) + 16) % 16);
    const int box_w = (xoff + (16 - 1) * s.sw + 3 + 15) & ~15, box_h = (8 - 1) * s.sh + 3;
    if (box_w > 256 || box_h > 256) return -1;
    const uint64_t dims[4] = {(uint64_t)s.w, (uint64_t)s.h, (uint64_t)s.c, (uint64_t)s.n};
    const uint64_t strides[3] = {(uint64_t)s.w, (uint64_t)s.w * s.h, (uint64_t)s.w * s.h * s.c};
    const uint32_t box[4] = {(uint32_t)box_w, (uint32_t)box_h, (uint32_t)s.c, 1u};
    if (tmap_encode(p->tmap_in, in, 4, dims, strides, box, nullptr, 0)) return -1;
    p->tile_cols = box_w, p->tile_rows = box_h, p->gpr = xoff;
    p->valid = 1;
    return 0;
}

cudaError_t launch_stem_tc(const DwPlan& plan, const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, cudaStream_t st)
{
    StemArgs a;
    a.in = (const uint8_t*)in, a.w = (const uint8_t*)w, a.out = (uint8_t*)out;
    a.n = s.n, a.c = s.c, a.h = s.h, a.w_in = s.w, a.oh = s.oh, a.ow = s.ow, a.ocp = s.ocp, a.oc = s.oc, a.stride = s.sh, a.ph = s.ph0, a.pw = s.pw0;
    a.npix = (unsigned)((long long)s.n * s.oh * s.ow);
    const bool tma = plan.valid != 0;
    a.tiles_w = (s.ow + 15) / 16, a.tiles_h = (s.oh + 7) / 8;
    a.box_w = plan.tile_cols, a.box_h = plan.tile_rows, a.in_bytes = tma ? plan.tile_cols * plan.tile_rows * s.c : 0, a.xoff = plan.gpr;
    a.ntiles = tma ? (unsigned)a.tiles_w * a.tiles_h * s.n : (a.npix + 127u) / 128u;
    const size_t smem = 4096 + (size_t)s.ocp * 32 + (size_t)s.ocp * 8 + 128 + 2 * (size_t)((a.in_bytes + 127) & ~127) + 128 * (size_t)acc_pitch(s.ocp) + 1024;
    static int sms = 0;
    if (!sms)
    {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    // several resident CTAs per SM overlap gather / MMA / epilogue of different tiles; each loops over its share
    const unsigned cap = (unsigned)sms * 8u;
    const unsigned grid = a.ntiles < cap ? a.ntiles : cap;
    const int mode = !e.fast_ok ? 2 : (e.fuse_bias ? 1 : 0);
    CUtensorMap tm;
    memcpy(&tm, plan.tmap_in, sizeof tm);
#define TB200_STEM_CASE(MD, T)                                                                                                 \
    if (mode == MD && tma == T)                                                                                                \
    {                                                                                                                          \
        cudaError_t err = cudaFuncSetAttribute(stem_tc_kernel<MD, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
        if (err != cudaSuccess) return err;                                                                                    \
        if (debug_launch()) fprintf(stderr, "tengine_b200: launch stem_tc_kernel<MODE=%d,TMA_IN=%d>\n", MD, (int)T);         \
        stem_tc_kernel<MD, T><<<grid, 128, smem, st>>>(tm, a, e);                                                              \
        return cudaGetLastError();                                                                                             \
    }
    TB200_STEM_CASE(0, true) TB200_STEM_CASE(1, true) TB200_STEM_CASE(2, true)
    TB200_STEM_CASE(0, false) TB200_STEM_CASE(1, false) TB200_STEM_CASE(2, false)
#undef TB200_STEM_CASE
    return cudaErrorInvalidValue;
}

// ---- gather convolution on the tensor cores (uint8 stems, 3x3 convolutions over 16-channel NHWC tensors) ---------------
// Same skeleton as the stem above, for the two YOLOv3-tiny layers the implicit GEMM cannot take: the uint8 NCHW stem
// (3 -> 16 channels at 416x416) and the 3x3 convolution whose input has only 16 channels (a 32-byte wgmma k-step would
// straddle two filter taps of a 4-D TMA box).  Every thread gathers the K bytes of its output pixel itself -- NCHW: 27 byte
// loads; NHWC16: nine 16-byte loads, one per tap -- and writes them as one row of `ks` SW32 K-major k-block tiles; `ks`
// k-steps (K = 32 each) accumulate.  uint8: taps outside the image are filled with the input zero point (they then contribute
// (zx-zx)(w-zw) = 0, exactly like the reference, which skips them), padding K positions hold 0 in A and B, and the thread
// sums its own row (dp4a) so that  sum (x-zx)(w-zw) = acc - zw*sum(x) + corr[oc]  needs no ones-row and no border table.
// Takes the role of im2col + sgemm of conv_hcl_run for these shapes (conv_kernel_x86.c:187-242, 1008-1631).
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

template <int MODE, bool U8, int KHW> // MODE: 0 fast, 1 fast + fused bias (int8), 2 exact; KHW: 3 or 7 (NCHW stems; NHWC16 is 3x3)
__global__ void __launch_bounds__(128) conv_gather_tc_kernel(const GatherArgs a, const __grid_constant__ EpiParams e)
{
    extern __shared__ __align__(1024) uint8_t gat_smem[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(gat_smem) + 1023) & ~(uintptr_t)1023);
    const uint32_t sA = smem_u32(sm), sB = sA + (uint32_t)a.ks * 4096u, b_tile = (uint32_t)a.ocp * 32u, sPar = sB + (uint32_t)a.ks * b_tile;
    const uint32_t pitch = acc_pitch(a.ocp), sImg = (sPar + (uint32_t)a.ocp * 8u + 15u) & ~15u; // accumulator image [128][pitch]
    const int tid = threadIdx.x;
    // B tiles (one per k-step) and the epilogue constants: identical for every CTA, L2 resident
    for (int i = tid; i < a.ks * a.ocp * 2; i += 128)
    {
        const int kb = i / (a.ocp * 2), j = i - kb * (a.ocp * 2), r = j >> 1, c16 = j & 1;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(a.w + ((size_t)r * a.ks + kb) * 32) + c16);
        sts_u4(sB + (uint32_t)kb * b_tile + sw32_offset(r, c16), v.x, v.y, v.z, v.w);
    }
    for (int c = tid; c < a.ocp; c += 128) sts_f2(sPar + c * 8, (MODE != 2 || U8) ? __ldg(e.fast_par + c) : make_float2(0.f, 0.f));

    for (unsigned tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x)
    {
        const unsigned pix = tile * 128u + (unsigned)tid;
        const bool valid = pix < a.npix;
        int32_t sx = 0;
        int n = 0, oh = 0, ow = 0;
        if (valid)
        {
            const unsigned prow = pix / (unsigned)a.ow;
            ow = (int)(pix - prow * a.ow);
            n = (int)(prow / (unsigned)a.oh);
            oh = (int)(prow - (unsigned)n * a.oh);
        }
        const int iy0 = oh * a.stride - a.ph, ix0 = ow * a.stride - a.pw;
        if (a.nhwc16)
        {
            // nine 16-byte taps + one half-row of padding = 160 bytes = five k-steps
            const uint8_t* img = a.in + (size_t)n * a.h * a.w_in * 16;
#pragma unroll
            for (int t = 0; t < 10; t++)
            {
                uint4 v = make_uint4(0, 0, 0, 0);
                if (t < 9)
                {
                    const int iy = iy0 + t / 3, ix = ix0 + t % 3;
                    v = make_uint4(a.fill16[0], a.fill16[1], a.fill16[2], a.fill16[3]);
                    if (valid && iy >= 0 && iy < a.h && ix >= 0 && ix < a.w_in) v = __ldg(reinterpret_cast<const uint4*>(img + ((size_t)iy * a.w_in + ix) * 16));
                    if (U8) sx = (int32_t)__dp4a(v.w, 0x01010101u, __dp4a(v.z, 0x01010101u, __dp4a(v.y, 0x01010101u, __dp4a(v.x, 0x01010101u, (unsigned)sx))));
                }
                sts_u4(sA + (uint32_t)(t >> 1) * 4096u + sw32_offset(tid, t & 1), v.x, v.y, v.z, v.w);
            }
        }
        else
        {
            // NCHW stem: C*KHW*KHW bytes (27 for 3x3, 147 for ResNet's 7x7), k = (c*KHW + kh)*KHW + kw, in NW words = NW/8 k-steps
            constexpr int NW = KHW == 3 ? 8 : 40;
            uint32_t row[NW];
#pragma unroll
            for (int j = 0; j < NW; j++) row[j] = 0;
            const size_t plane = (size_t)a.h * a.w_in;
            const uint8_t* img = a.in + (size_t)n * a.c * plane;
            const uint32_t fb = a.fill & 0xffu;
#pragma unroll
            for (int c = 0; c < 3; c++)
            {
                if (c < a.c)
                {
#pragma unroll
                    for (int kh = 0; kh < KHW; kh++)
                    {
                        const int iy = iy0 + kh;
                        const bool rok = valid && iy >= 0 && iy < a.h;
                        const uint8_t* rp = img + (size_t)c * plane + (size_t)(rok ? iy : 0) * a.w_in;
#pragma unroll
                        for (int kw = 0; kw < KHW; kw++)
                        {
                            const int ix = ix0 + kw;
                            const uint32_t b = (rok && ix >= 0 && ix < a.w_in) ? (uint32_t)__ldg(rp + ix) : fb;
                            const int k = (c * KHW + kh) * KHW + kw; // compile-time after unrolling
                            row[k >> 2] |= b << (8 * (k & 3));
                        }
                    }
                }
            }
            if (U8)
            {
#pragma unroll
                for (int j = 0; j < NW; j++) sx = (int32_t)__dp4a(row[j], 0x01010101u, (unsigned)sx);
            }
#pragma unroll
            for (int j = 0; j < NW / 4; j++)
                sts_u4(sA + (uint32_t)(j >> 1) * 4096u + sw32_offset(tid, j & 1), row[4 * j], row[4 * j + 1], row[4 * j + 2], row[4 * j + 3]);
        }
        fence_proxy_async_smem(); // the MMAs read these generic-proxy writes through the async proxy
        __syncthreads();          // (first iteration: also publishes the B tiles and the constants)
        wg_mma_to_image<U8, U8>(sA, 4096u, sB, b_tile, a.ks, 32, a.ocp, sImg, pitch);
        __syncthreads();

        uint8_t* op = a.out + (size_t)pix * a.ocp;
        const uint32_t tb = sImg + (uint32_t)tid * pitch;
        const int32_t rowc = U8 ? -e.w_zero * sx : 0;
        for (int c = 0; c < a.ocp; c += 16)
        {
            uint32_t v[16];
            acc_ld16(tb + 4u * c, v);
            uint32_t w[4];
            if (U8)
            {
                // the int8 form (engine.cu: constants { M, M, y, y } with y = corr[oc] + bias[oc]): a' = v - zw*sum(x) + y, t = fl(a' * M)
                if (MODE == 2)
                {
#pragma unroll
                    for (int k = 0; k < 16; k++)
                    {
                        if ((k & 3) == 0) w[k >> 2] = 0;
                        if (c + k < a.oc)
                        {
                            const float4 pp = lds_f4(sPar + c * 8 + (k >> 1) * 16);
                            const int32_t acc = (int32_t)v[k] + rowc + __float_as_int((k & 1) ? pp.w : pp.z) - (e.has_bias ? __ldg(e.bias + c + k) : 0);
                            w[k >> 2] |= ((uint32_t)requant(acc, c + k, e) & 0xffu) << (8 * (k & 3));
                        }
                    }
                }
                else
                {
                    float gw[4];
#pragma unroll
                    for (int h = 0; h < 2; h++)
                    {
                        float4 p[4];
#pragma unroll
                        for (int k = 0; k < 4; k++) p[k] = lds_f4(sPar + c * 8 + h * 64 + k * 16);
                        int32_t a8[8];
#pragma unroll
                        for (int k = 0; k < 8; k++) a8[k] = (int32_t)v[h * 8 + k] + rowc;
                        requant_fast8_i8<false>(a8, p, e, w[2 * h], w[2 * h + 1], gw[2 * h], gw[2 * h + 1]);
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
                                int32_t at[4]; // accumulator + y of the word's four channels (what the fast path multiplied by M)
#pragma unroll
                                for (int t = 0; t < 4; t++)
                                {
                                    const float4 pp = lds_f4(sPar + c * 8 + ((j * 4 + t) >> 1) * 16);
                                    at[t] = (int32_t)v[j * 4 + t] + rowc + __float_as_int((t & 1) ? pp.w : pp.z);
                                }
                                w[j] = requant_fix_word_u8(w[j], at[0], at[1], at[2], at[3], c + j * 4, a.oc, e);
                            }
                    }
                    if (c + 16 > a.oc)
                    {
                        // pad lanes of uint8 tensors hold 0, not the zero point
#pragma unroll
                        for (int k = 0; k < 16; k++)
                            if (c + k >= a.oc) w[k >> 2] &= ~(0xffu << (8 * (k & 3)));
                    }
                }
            }
            else if (MODE == 2)
            {
#pragma unroll
                for (int k = 0; k < 16; k++)
                {
                    if ((k & 3) == 0) w[k >> 2] = 0;
                    if (c + k < a.oc) w[k >> 2] |= ((uint32_t)requant((int32_t)v[k], c + k, e) & 0xffu) << (8 * (k & 3));
                }
            }
            else
                stem_unit_fast<MODE == 1>(v, sPar + c * 8, c, e, w);
            if (valid) *reinterpret_cast<uint4*>(op + c) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        __syncthreads(); // the next tile's gather overwrites the A tiles, its MMAs the accumulator image
    }
}

cudaError_t launch_conv_gather_tc(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, int nhwc16, cudaStream_t st)
{
    const int khw = nhwc16 ? 3 : s.kh;
    GatherArgs a;
    a.in = (const uint8_t*)in, a.w = (const uint8_t*)w, a.out = (uint8_t*)out;
    a.n = s.n, a.c = s.c, a.h = s.h, a.w_in = s.w, a.oh = s.oh, a.ow = s.ow, a.ocp = s.ocp, a.oc = s.oc, a.stride = s.sh, a.ph = s.ph0, a.pw = s.pw0;
    a.npix = (unsigned)((long long)s.n * s.oh * s.ow);
    a.ntiles = (a.npix + 127u) / 128u;
    a.ks = nhwc16 ? 5 : (s.c * s.kh * s.kw + 31) / 32, a.nhwc16 = nhwc16;
    a.fill = e.is_uint8 ? ((uint32_t)(e.in_zero & 0xff) * 0x01010101u) : 0u;
    for (int j = 0; j < 4; j++)
    {
        a.fill16[j] = 0;
        for (int t = 0; t < 4; t++)
            if (j * 4 + t < s.c) a.fill16[j] |= (a.fill & 0xffu) << (8 * t);
    }
    const size_t smem = (size_t)a.ks * 4096 + (size_t)a.ks * s.ocp * 32 + (size_t)s.ocp * 8 + 16 + 128 * (size_t)acc_pitch(s.ocp) + 1024;
    static int sms = 0;
    if (!sms)
    {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    const unsigned cap = (unsigned)sms * 6u;
    const unsigned grid = a.ntiles < cap ? a.ntiles : cap;
    const int mode = !e.fast_ok ? 2 : ((!e.is_uint8 && e.fuse_bias) ? 1 : 0);
#define TB200_GAT_CASE(MD, U, K)                                                                                                   \
    if (mode == MD && (e.is_uint8 != 0) == U && khw == K)                                                                          \
    {                                                                                                                              \
        /* the opt-in is per device AND per context: set it before every launch (launches happen at graph capture only) */ \
        {                                                                                                                          \
            cudaError_t err = cudaFuncSetAttribute(conv_gather_tc_kernel<MD, U, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
            if (err != cudaSuccess) return err;                                                                                    \
        }                                                                                                                          \
        if (debug_launch()) fprintf(stderr, "tengine_b200: launch conv_gather_tc_kernel<MODE=%d,U8=%d,KHW=%d>\n", MD, (int)U, K);  \
        conv_gather_tc_kernel<MD, U, K><<<grid, 128, smem, st>>>(a, e);                                                            \
        return cudaGetLastError();                                                                                                 \
    }
    TB200_GAT_CASE(0, false, 3) TB200_GAT_CASE(1, false, 3) TB200_GAT_CASE(2, false, 3) TB200_GAT_CASE(0, true, 3) TB200_GAT_CASE(2, true, 3)
    TB200_GAT_CASE(0, false, 7) TB200_GAT_CASE(1, false, 7) TB200_GAT_CASE(2, false, 7) TB200_GAT_CASE(0, true, 7) TB200_GAT_CASE(2, true, 7)
#undef TB200_GAT_CASE
    return cudaErrorInvalidValue;
}

// ---- small-K pointwise GEMM: many small CTAs instead of one warp-specialised persistent CTA ---------------------------
// For K <= 256 (the first pointwise layers: K = 32..128, one or two k-blocks) the persistent kernel above spends more
// time in hand-overs between its roles than in work (timeline: the epilogue warps idle ~50% of the time).  Here a CTA is
// one warpgroup; it keeps the N tile's weights in shared memory, double-buffers the A tile (TMA), and per m-tile does:
// wait A -> the warpgroup's MMAs into the accumulator image -> everybody requantises its own accumulator row and writes its
// bn contiguous output bytes straight to global memory.  There is no pipelining inside a CTA beyond the A prefetch; several
// CTAs are resident per SM (bounded by shared memory) and overlap each other, the way the tensor-core stem above does.
struct SimpleArgs
{
    uint8_t* out;
    long long m;
    int m_tiles, n_tiles, k_blocks, block_n, block_k, swizzle, ocp, oc, ldo;
};

template <int MODE> // 0 fast, 1 fast + fused bias, 2 exact
__global__ void __launch_bounds__(128) gemm_simple_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                                                           const SimpleArgs g, const __grid_constant__ EpiParams e)
{
    extern __shared__ __align__(1024) uint8_t simple_smem[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(simple_smem) + 1023) & ~(uintptr_t)1023);
    const uint32_t a_bytes = BLOCK_M * g.block_k, b_bytes = g.block_n * g.block_k, b_al = (b_bytes + 1023) & ~1023u;
    uint8_t* sA = sm;                                               // [2][k_blocks][a_bytes]
    uint8_t* sB = sA + 2u * (size_t)g.k_blocks * a_bytes;           // [k_blocks][b_al]
    const uint32_t sPar = smem_u32(sB) + (uint32_t)g.k_blocks * b_al; // [block_n] x 8 bytes
    const uint32_t pitch = acc_pitch(g.block_n), sImg = sPar + (uint32_t)g.block_n * 8u; // accumulator image [128][pitch]
    __shared__ __align__(8) uint64_t a_full[2], b_full;
    const int tid = threadIdx.x;
    const int ntile = blockIdx.x % g.n_tiles, n0 = ntile * g.block_n;
    const int mfirst = blockIdx.x / g.n_tiles, mstep = gridDim.x / g.n_tiles; // the grid is a multiple of n_tiles

    if (tid == 0)
    {
        mbar_init(&a_full[0], 1), mbar_init(&a_full[1], 1), mbar_init(&b_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0)
    {
        mbar_expect_tx(&b_full, (uint32_t)g.k_blocks * b_bytes);
        for (int kb = 0; kb < g.k_blocks; kb++) tma_load_2d(&tmap_b, &b_full, sB + (size_t)kb * b_al, kb * g.block_k, n0);
        if (mfirst < g.m_tiles)
        {
            mbar_expect_tx(&a_full[0], (uint32_t)g.k_blocks * a_bytes);
            for (int kb = 0; kb < g.k_blocks; kb++) tma_load_2d(&tmap_a, &a_full[0], sA + (size_t)kb * a_bytes, kb * g.block_k, mfirst * BLOCK_M);
        }
    }
    for (int c = tid; c < g.block_n; c += 128)
        sts_f2(sPar + c * 8, (MODE != 2 && n0 + c < g.ocp) ? __ldg(e.fast_par + n0 + c) : make_float2(0.f, 0.f));
    __syncthreads();
    const uint32_t tb = sImg + (uint32_t)tid * pitch;

    uint32_t it = 0;
    for (int mt = mfirst; mt < g.m_tiles; mt += mstep, it++)
    {
        const int buf = it & 1;
        // the other buffer was read by the MMAs of the previous tile, which have completed: prefetch the next tile
        if (tid == 0 && mt + mstep < g.m_tiles)
        {
            mbar_expect_tx(&a_full[buf ^ 1], (uint32_t)g.k_blocks * a_bytes);
            for (int kb = 0; kb < g.k_blocks; kb++)
                tma_load_2d(&tmap_a, &a_full[buf ^ 1], sA + ((size_t)(buf ^ 1) * g.k_blocks + kb) * a_bytes, kb * g.block_k, (mt + mstep) * BLOCK_M);
        }
        if (it == 0) mbar_wait(&b_full, 0);
        mbar_wait(&a_full[buf], (it >> 1) & 1);
        wg_mma_to_image<false, false>(smem_u32(sA + (size_t)buf * g.k_blocks * a_bytes), a_bytes, smem_u32(sB), b_al, g.k_blocks, g.swizzle,
                                      g.block_n, sImg, pitch);
        __syncthreads();

        // ---- epilogue: thread = output row, 16 channels per load, straight to global memory ----
        const long long row = (long long)mt * BLOCK_M + tid;
        uint8_t* op = g.out + (size_t)(row < g.m ? row : 0) * g.ldo + n0;
        uint32_t v0[16], v1[16];
        acc_ld16(tb, v0);
        const int nch = g.block_n >> 4;
        for (int c = 0; c < nch; c += 2)
        {
            if (c + 1 < nch) acc_ld16(tb + (c + 1) * 64, v1);
            {
                uint32_t w[4];
                if (MODE == 2)
                {
#pragma unroll
                    for (int k = 0; k < 16; k++)
                    {
                        if ((k & 3) == 0) w[k >> 2] = 0;
                        if (n0 + c * 16 + k < g.oc) w[k >> 2] |= ((uint32_t)requant((int32_t)v0[k], n0 + c * 16 + k, e) & 0xffu) << (8 * (k & 3));
                    }
                }
                else
                    stem_unit_fast<MODE == 1>(v0, sPar + c * 128, n0 + c * 16, e, w);
                if (row < g.m && n0 + c * 16 < g.ocp) *reinterpret_cast<uint4*>(op + c * 16) = make_uint4(w[0], w[1], w[2], w[3]);
            }
            if (c + 1 >= nch) break;
            if (c + 2 < nch) acc_ld16(tb + (c + 2) * 64, v0);
            {
                uint32_t w[4];
                if (MODE == 2)
                {
#pragma unroll
                    for (int k = 0; k < 16; k++)
                    {
                        if ((k & 3) == 0) w[k >> 2] = 0;
                        if (n0 + (c + 1) * 16 + k < g.oc) w[k >> 2] |= ((uint32_t)requant((int32_t)v1[k], n0 + (c + 1) * 16 + k, e) & 0xffu) << (8 * (k & 3));
                    }
                }
                else
                    stem_unit_fast<MODE == 1>(v1, sPar + (c + 1) * 128, n0 + (c + 1) * 16, e, w);
                if (row < g.m && n0 + (c + 1) * 16 < g.ocp) *reinterpret_cast<uint4*>(op + (c + 1) * 16) = make_uint4(w[0], w[1], w[2], w[3]);
            }
        }
        // the next tile's MMAs overwrite the accumulator image
        __syncthreads();
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

// Where the uint8 path's sum(x) comes from (TB200_U8_SX, A/B switch): 3 (default) = two extra warps add up the rows of the A tiles,
// 0 = 16 rows of ones in every B tile (sum(x) is then a 17th..32nd accumulator column; costs image columns and m-tiles per stage).
bool debug_launch()
{
    static const bool on = getenv("TB200_DEBUG_LAUNCH") != nullptr;
    return on;
}

int gemm_sx_mode()
{
    static const int mode = [] { const char* e = getenv("TB200_U8_SX"); return (e && atoi(e) == 0) ? 0 : 3; }();
    return mode;
}

// rows of one packed B tile: block_n, + 16 rows of ones for uint8 layers with a weight zero point (u8 = 1 + zero point) in mode 0
int gemm_tile_rows(int ocp, int u8) { return gemm_block_n(ocp, u8) + ((u8 > 1 && gemm_sx_mode() == 0) ? 16 : 0); }

int gemm_block_n(int ocp, int u8)
{
    // N tiles of at most 128 channels (+ 16 ones rows in mode 0): the accumulator image of a stage shares shared memory with
    // the operand ring; the channels are dealt evenly to the fewest such tiles
    (void)u8;
    const int nt = (ocp + 127) / 128;
    return ((ocp + nt - 1) / nt + 15) & ~15;
}

// Store-group width and output tensor maps.  A group is 32 rows x 16*cs channels; cs is the largest of 4 / 2 / 1 that
// divides the N tile's chunk count and deals the stage's groups evenly to the four warps of a 32-row image quarter.
static void plan_store_groups(GemmPlan* p)
{
    const int nch = p->block_n / 16;
    int cs = 1;
    for (int c = 4; c >= 1; c >>= 1)
        if (nch % c == 0 && ((p->mt * (nch / c)) % 4 == 0 || c == 1))
        {
            cs = c;
            break;
        }
    // 128-byte rows filled by warp pairs when the stage deals an even number of 128-column groups to each quarter
    // (measured on MobileNet-v1, batch 256: the pair hand-over costs more than the halved row count saves -- 0.75 ms vs
    //  0.68 ms for all GEMMs -- so this mode is opt-in)
    if (nch % 8 == 0 && (p->mt * (nch / 8)) % 2 == 0 && getenv("TB200_GEMM_PAIR")) cs = 8;
    if (const char* ev = getenv("TB200_GEMM_STORE_CS"))
    {
        const int f = atoi(ev);
        if ((f == 1 || f == 2 || f == 4) && nch % f == 0) cs = f;
    }
    p->cs = cs, p->ngroups = nch / cs;
}

static int plan_epilogue(GemmPlan* p, const void* out, uint64_t d1, uint64_t d2)
{
    const int cs = p->cs;
    const uint64_t dims[3] = {(uint64_t)p->ocp, d1, d2};
    const uint64_t strides[2] = {(uint64_t)p->ldo, (uint64_t)p->ldo * d1};
    const int swz = cs == 8 ? 128 : (cs == 4 ? 64 : (cs == 2 ? 32 : 0));
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
    return EPI_WARPS * 2 * 512 * (p->cs == 8 ? 4 : p->cs) + (par_ch <= PAR_MAX ? par_ch : p->block_n) * 8 + (int)sizeof(GemmSmemCtl) + 2048 +
           128 * (int)acc_pitch(p->mt * p->bnx) + 16;
}

// Operand ring depth and the resident-B decision.  With the N tile's weights resident the ring carries A tiles only,
// which for the small-K layers (K = 32..128, one 4-16 KB A tile per m-tile) is the difference between 8 and 24 m-tiles
// of prefetch distance.
static int plan_ring(GemmPlan* p)
{
    const int a_bytes = BLOCK_M * p->block_k, b_al = (p->bnx * p->block_k + 1023) & ~1023;
    const int budget = 224 * 1024 - epilogue_smem_bytes(p) - (p->cplane ? 4096 : 0);
    p->b_res = ((long long)p->k_blocks * b_al <= B_RESIDENT_MAX && !getenv("TB200_GEMM_NO_BRES")) ? 1 : 0;
    int stages = p->b_res ? (budget - p->k_blocks * b_al) / a_bytes : budget / (a_bytes + b_al);
    if (p->b_res && stages < 3) p->b_res = 0, stages = budget / (a_bytes + b_al);
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    if (stages < 2) return TB200_ERR_INVALID;
    p->stages = stages;
    return 0;
}

int gemm_plan_create(GemmPlan* p, const void* a, long long lda, const void* b, void* out, long long m, int k, int oc, int ocp, int ldo,
                     int variant, int u8)
{
    if (m <= 0 || k <= 0 || (k & 15) || (ocp & 15) || (lda & 15) || (ldo & 15)) return TB200_ERR_INVALID;
    memset(p, 0, sizeof *p);
    p->m = m, p->k = k, p->oc = oc, p->ocp = ocp, p->ldo = ldo, p->variant = variant, p->out = out;
    p->block_k = k <= 32 ? 32 : (k <= 64 ? 64 : 128);
    p->swizzle = p->block_k;
    p->k_blocks = (k + p->block_k - 1) / p->block_k;
    p->u8 = u8 != 0; // u8 = 1 + weight zero point for uint8 layers
    p->b_signed = !p->u8 || u8 != 1;
    p->cplane = (p->u8 && u8 != 1 && !getenv("TB200_DEBUG_NO_CPLANE")) ? 128 - (u8 - 1) : 0; // (debug switch: WRONG results, timing experiments only)
    p->block_n = gemm_block_n(ocp, u8);
    p->bnx = gemm_tile_rows(ocp, u8);
    p->taps = 1;
    p->n_tiles = (ocp + p->block_n - 1) / p->block_n;
    p->m_tiles = (m + BLOCK_M - 1) / BLOCK_M;
    // m-tiles per accumulator stage: amortise the per-stage synchronisation over up to ACC_COLS_MAX image columns of work
    p->mt = 1;
    {
        // several m-tiles per stage when the CTA stays on one N tile anyway (single tile, or resident weights)
        const bool resident = (long long)p->k_blocks * ((p->bnx * p->block_k + 1023) & ~1023) <= B_RESIDENT_MAX;
        if (p->n_tiles == 1 || (resident && getenv("TB200_GEMM_PAIR")))
            while (p->mt < 4 && (p->mt * 2) * p->bnx <= ACC_COLS_MAX && (long long)(p->mt * 2) * 132 <= p->m_tiles * (p->n_tiles == 1 ? 132 : 1)) p->mt *= 2;
    }
    plan_store_groups(p);
    int rc = plan_ring(p);
    if (rc) return rc;
    rc = encode_2d(p->tmap_a, a, (uint64_t)k, (uint64_t)m, (uint64_t)lda, p->block_k, BLOCK_M, p->swizzle);
    if (rc) return rc;
    rc = encode_2d(p->tmap_b, b, (uint64_t)k, (uint64_t)p->n_tiles * p->bnx, (uint64_t)k, p->block_k, p->bnx, p->swizzle);
    if (rc) return rc;
    p->rows_valid = BLOCK_M, p->out_mode = 0;
    rc = plan_epilogue(p, out, (uint64_t)m, 1);
    if (rc) return rc;
    // small-K layers: the many-small-CTAs kernel (gemm_simple_kernel), N tiles of at most 128 channels
    p->simple = 0;
    static const int maxk = getenv("TB200_GEMM_SIMPLE_MAXK") ? atoi(getenv("TB200_GEMM_SIMPLE_MAXK")) : 256;
    // Opt-in (TB200_GEMM_SIMPLE=1): the cross-check implementation of the same contraction.
    if (!u8 && k <= maxk && getenv("TB200_GEMM_SIMPLE"))
    {
        const int bn = ocp <= 128 ? ocp : 128;
        const int a_bytes = BLOCK_M * p->block_k, b_al = (bn * p->block_k + 1023) & ~1023;
        const int smem = p->k_blocks * (2 * a_bytes + b_al) + bn * 8 + 128 * (int)acc_pitch(bn) + 2048;
        if (smem <= 200 * 1024 &&
            encode_2d(p->tmap_b_s, b, (uint64_t)k, (uint64_t)ocp, (uint64_t)k, p->block_k, bn, p->swizzle) == 0)
            p->simple = 1, p->s_block_n = bn, p->s_n_tiles = (ocp + bn - 1) / bn, p->s_smem = smem, p->out = out;
    }
    return 0;
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
    p->m = (long long)s.n * s.oh * s.ow, p->oc = s.oc, p->ocp = s.ocp, p->ldo = s.ocp, p->variant = 0, p->out = out;
    if (taps == 1) p->block_k = s.cp <= 32 ? 32 : (s.cp <= 64 ? 64 : 128);
    else p->block_k = (s.cp % 128 == 0) ? 128 : ((s.cp % 64 == 0) ? 64 : 32);
    p->swizzle = p->block_k;
    p->cblocks = (s.cp + p->block_k - 1) / p->block_k;
    p->k_blocks = taps * p->cblocks;
    p->k = taps * s.cp;
    p->u8 = u8 != 0; // u8 = 1 + weight zero point for uint8 layers
    p->b_signed = !p->u8 || u8 != 1;
    p->cplane = (p->u8 && u8 != 1 && !getenv("TB200_DEBUG_NO_CPLANE")) ? 128 - (u8 - 1) : 0; // (debug switch: WRONG results, timing experiments only)
    p->block_n = gemm_block_n(s.ocp, u8);
    p->bnx = gemm_tile_rows(s.ocp, u8);
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
    p->mt = 1;
    {
        // several m-tiles per stage when the CTA stays on one N tile anyway (single tile, or resident weights)
        const bool resident = (long long)p->k_blocks * ((p->bnx * p->block_k + 1023) & ~1023) <= B_RESIDENT_MAX;
        if (p->n_tiles == 1 || (resident && getenv("TB200_GEMM_PAIR")))
            while (p->mt < 4 && (p->mt * 2) * p->bnx <= ACC_COLS_MAX && (long long)(p->mt * 2) * 132 <= p->m_tiles * (p->n_tiles == 1 ? 132 : 1)) p->mt *= 2;
    }
    plan_store_groups(p);
    int rc = plan_ring(p);
    if (rc) return rc;
    const uint64_t dims[4] = {(uint64_t)s.cp, (uint64_t)s.w, (uint64_t)s.h, (uint64_t)s.n};
    const uint64_t strides[3] = {(uint64_t)s.cp, (uint64_t)s.w * s.cp, (uint64_t)s.h * s.w * s.cp};
    const uint32_t box[4] = {(uint32_t)p->block_k, (uint32_t)((p->bw - 1) * s.sw + 1), (uint32_t)((p->bh - 1) * s.sh + 1), (uint32_t)p->bn};
    const uint32_t estr[4] = {1u, (uint32_t)s.sw, (uint32_t)s.sh, 1u};
    if (box[1] > 256 || box[2] > 256 || box[3] > 256) return TB200_ERR_UNSUPPORTED;
    rc = tmap_encode(p->tmap_a, in, 4, dims, strides, box, estr, p->swizzle);
    if (rc) return rc;
    rc = encode_2d(p->tmap_b, w, (uint64_t)p->k, (uint64_t)p->n_tiles * p->bnx, (uint64_t)p->k, p->block_k, p->bnx, p->swizzle);
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
// One line per event, sorted by time: cycles since the first event, role (P producer, M mma, E2/E17 epilogue warps), tag.
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
    static const char* role[4] = {"P", "M", "E0", "E15"};
    static const char* tagM[3] = {"kblock mma issued", "got sx_empty", "commit sx_full"};
    static const char* tagE[5] = {"got sx_full", "group stored", "arrive sx_empty", "tmem ld done", "unit done"};
    for (int r = 0; r < 4; r++)
        for (int i = 0; i < 1024 && h[r * 1024 + i]; i++)
        {
            const unsigned long long v = h[r * 1024 + i];
            const int tag = (int)(v & 0xff);
            fprintf(stderr, "TL %8llu %-3s %s%s%d\n", (v >> 8) - t0, role[r], r == 0 ? "load issued kb=" : (r == 1 ? tagM[tag % 3] : tagE[tag % 5]),
                    r == 0 ? "" : " #", r == 0 ? tag : i);
        }
}

static cudaError_t launch_gemm_simple(const GemmPlan& p, const EpiParams& e, int num_sms, cudaStream_t st)
{
    SimpleArgs g;
    g.out = (uint8_t*)p.out, g.m = p.m, g.m_tiles = (int)p.m_tiles, g.n_tiles = p.s_n_tiles, g.k_blocks = p.k_blocks, g.block_n = p.s_block_n;
    g.block_k = p.block_k, g.swizzle = p.swizzle, g.ocp = p.ocp, g.oc = p.oc, g.ldo = p.ldo;
    int per_sm = (220 * 1024) / (p.s_smem + 1024);
    if (per_sm > 16) per_sm = 16;
    if (per_sm < 1) per_sm = 1;
    long long want = p.m_tiles * p.s_n_tiles, cap = (long long)num_sms * per_sm;
    int grid = (int)(want < cap ? want : cap);
    grid -= grid % p.s_n_tiles;
    if (grid < p.s_n_tiles) grid = p.s_n_tiles;
    CUtensorMap ta, tb;
    memcpy(&ta, p.tmap_a, sizeof ta);
    memcpy(&tb, p.tmap_b_s, sizeof tb);
    const int mode = !e.fast_ok ? 2 : (e.fuse_bias ? 1 : 0);
    const size_t smem = (size_t)p.s_smem;
#define TB200_SIMPLE_CASE(MD)                                                                                                  \
    if (mode == MD)                                                                                                            \
    {                                                                                                                          \
        /* the opt-in is per device AND per context: set it before every launch (launches happen at graph capture only) */ \
        {                                                                                                                      \
            cudaError_t err = cudaFuncSetAttribute(gemm_simple_kernel<MD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
            if (err != cudaSuccess) return err;                                                                                \
        }                                                                                                                      \
        if (debug_launch()) fprintf(stderr, "tengine_b200: launch gemm_simple_kernel<MODE=%d>\n", MD);                          \
        gemm_simple_kernel<MD><<<grid, 128, smem, st>>>(ta, tb, g, e);                                                         \
        return cudaGetLastError();                                                                                             \
    }
    TB200_SIMPLE_CASE(0) TB200_SIMPLE_CASE(1) TB200_SIMPLE_CASE(2)
#undef TB200_SIMPLE_CASE
    return cudaErrorInvalidValue;
}

cudaError_t launch_gemm_i8(const GemmPlan& p, const EpiParams& e, const int32_t* btab, int num_sms, cudaStream_t st)
{
    if (p.simple) return launch_gemm_simple(p, e, num_sms, st);
    if (p.block_n <= 0 || p.mt <= 0 || p.stages <= 0 || p.cs <= 0) return cudaErrorInvalidValue; // plan was never created
    GemmArgs g;
    g.m_tiles = (int)p.m_tiles, g.k_blocks = p.k_blocks, g.n_tiles = p.n_tiles, g.block_n = p.block_n;
    g.conv = p.conv, g.cblocks = p.cblocks, g.kw_n = p.kw_n, g.pad_h = p.pad_h, g.pad_w = p.pad_w, g.cstride = p.cstride, g.cp = p.cp;
    g.bw = p.bw, g.bh = p.bh, g.bn = p.bn, g.tiles_w = p.tiles_w, g.tiles_h = p.tiles_h, g.oh = p.oh, g.ow = p.ow, g.nimg = p.nimg;
    g.a_tx_bytes = p.a_tx_bytes;
    g.u8 = p.u8, g.bnx = p.bnx, g.taps = p.taps, g.in_h = p.in_h, g.in_w = p.in_w, g.btab = btab, g.b_signed = p.b_signed, g.cplane = p.cplane;
    g.sx_mode = !p.cplane ? -1 : (p.bnx != p.block_n ? 0 : 3);
    g.fixq = (uint4*)p.fixq, g.fixq_cap = p.fixq_cap, g.out_base = (uint8_t*)p.out, g.ldo = p.ldo, g.m_rows = (int)p.m;
    g.tcols = p.bnx;
    g.mt = p.mt;
    g.num_super = (int)(((p.m_tiles + p.mt - 1) / p.mt) * p.n_tiles);
    g.bw_rcp = p.conv ? (65536u + (uint32_t)p.bw - 1) / (uint32_t)p.bw : 0;
    g.bh_rcp = p.conv ? (65536u + (uint32_t)p.bh - 1) / (uint32_t)p.bh : 0;
    g.block_k = p.block_k, g.stages = p.stages, g.swizzle = p.swizzle, g.oc = p.oc, g.ocp = p.ocp;
    g.cs = p.cs, g.ngroups = p.ngroups, g.rows_valid = p.rows_valid, g.out_mode = p.out_mode;
    const int par_ch = p.n_tiles * p.block_n;
    g.par_all = par_ch <= PAR_MAX ? 1 : 0;
    const int a_bytes = BLOCK_M * p.block_k, b_bytes = (p.bnx * p.block_k + 1023) & ~1023;
    g.b_res = p.b_res;
    const size_t smem = (size_t)p.stages * (a_bytes + (p.b_res ? 0 : b_bytes)) + (p.b_res ? (size_t)p.k_blocks * b_bytes : 0) + (p.cplane ? 4096 : 0) +
                        (size_t)EPI_WARPS * 2 * 512 * (p.cs == 8 ? 4 : p.cs) + sizeof(GemmSmemCtl) +
                        (size_t)(g.par_all ? par_ch : p.block_n) * 8 + 16 + 128 * (size_t)acc_pitch(p.mt * g.tcols) + 1024;
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
    // uint8 border corrections only exist for convolutions with taps that can fall into the padding
    const bool border = p.u8 && p.conv && !(p.taps == 1 && p.pad_h == 0 && p.pad_w == 0);
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
            fprintf(stderr, "tengine_b200: launch gemm_i8_tcgen05_kernel<U8=%d,MODE=%d,CS=%d,BORDER=%d> out_mode=%d conv=%d n_tiles=%d b_res=%d fixq=%d\n", \
                    (int)U, MD, C, (int)B, p.out_mode, p.conv, p.n_tiles, p.b_res, p.fixq != nullptr);                      \
        gemm_i8_tcgen05_kernel<U, MD, C, B><<<grid, U ? GEMM_THREADS_U8 : GEMM_THREADS, smem, st>>>(ta, tb, to, tt, g, e);                           \
        if (trace_on) gemm_trace_report(p, g, grid, st);                                                                       \
        err = cudaGetLastError();                                                                                              \
        if (launch_dbg || err != cudaSuccess) gemm_launch_debug((const void*)gemm_i8_tcgen05_kernel<U, MD, C, B>, "launch", err, grid, smem, st); \
        return err;                                                                                                            \
    }
#define TB200_GEMM_CS(U, MD, B) TB200_GEMM_CASE(U, MD, 1, B) TB200_GEMM_CASE(U, MD, 2, B) TB200_GEMM_CASE(U, MD, 4, B) TB200_GEMM_CASE(U, MD, 8, B)
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
