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
//                   fragments go into the accumulator image ([128 rows][mt * block_n] s32 in shared memory) quarter by quarter:
//                   32-row quarter q is written by two MMA warps as soon as its two epilogue warps have read the previous stage
//                   out of it (mbarriers img_empty[q] / img_full[q]), so no warp waits for the whole CTA at the hand-over.
//   WG2-3, warps 8-15: epilogue.  Two warps per 32-row quarter of the image; a warp owns whole "store groups" = 32 rows x
//                   16 cs channels (cs = 1 or 2): image -> registers -> requant_fast_words_i8 -> bytes -> its own swizzled
//                   smem buffer -> ONE TMA store per group (cp.async.bulk.tensor, double-buffered).  Inside a group each lane
//                   owns one 4-channel word of 4 cs rows: its constants stay in registers, and its 4 cs words are requantised
//                   side by side.  No address arithmetic for the stores, rows outside the tensor are clipped by the TMA unit.
// So the tensor cores multiply stage s+1 while the epilogue requantises stage s: the registers are the second accumulator
// buffer.  Registers per thread (setmaxnreg): WG0 40, MMA 200 (at most 128 accumulators), epilogue 136.
// The producer runs ahead through the ring, so the next tile's operands are resident when its MMAs start.  K is small
// (32..1024), so the epilogue sets the pace of these layers, not the tensor pipe.  With only two epilogue warps per scheduler
// it is bound by latency unless each lane has many independent chains in flight: hence 4 cs words per lane, their image
// loads issued together and their fp32 chains interleaved (common.cuh, requant_fast_words_i8).
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
    // per 32-row quarter q of the accumulator image: its rows of the stage are written (the two MMA warps of q -> epilogue) /
    // have been read (the two epilogue warps of q -> MMA)
    uint64_t img_full[4], img_empty[4];
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

// row: the element's image row = its row of the m-tile (0..127)
__device__ __forceinline__ bool fixq_push(uint32_t mtile, uint32_t row, int oc, int32_t acc)
{
    if (!s_fixq.q) return false;
    const uint32_t slot = atomicAdd(&s_fixq.count, 1u);
    if (slot >= s_fixq.cap) return false;
    s_fixq.q[slot] = make_uint4(mtile, row | ((uint32_t)oc << 8), (uint32_t)acc, 0u);
    return true;
}

// One guarded word (final fast bytes in `word`) of image row `row`: find the elements that really sit in the band, queue them
// (or fix them here).
// a[j]: what the fast path converted to float -- int8: the raw accumulator (y is added inside), uint8: accumulator + sum(x) term + y.
template <bool U8, bool FUSE>
__device__ __noinline__ uint32_t gemm_fix_word(uint32_t word, int32_t a0, int32_t a1, int32_t a2, int32_t a3, int oc0, int oc_limit, uint32_t mtile,
                                               uint32_t row, const EpiParams& e)
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
            if (!fixq_push(mtile, row, oc0 + j, a[j]))
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

// Exact mode, one word: the literal arithmetic for each of its real channels (uint8: y from the constants in shared memory, the
// bias taken off again, the padding taps' corrections added).  Not inlined: the lane's other words then stay in registers across
// the requant() calls instead of spilling.
template <bool U8, bool BORDER>
__device__ __noinline__ uint32_t epilogue_word_exact(uint32_t v0, uint32_t v1, uint32_t v2, uint32_t v3, int32_t rowc, uint32_t pad, uint32_t par_addr,
                                                     int oc0, int oc_limit, int ocp, const int32_t* btab, const EpiParams& e)
{
    const uint32_t v[4] = {v0, v1, v2, v3};
    uint32_t w = 0;
#pragma unroll
    for (int j = 0; j < 4; j++)
    {
        const int oc = oc0 + j;
        if (oc < oc_limit)
        {
            int32_t acc = (int32_t)v[j];
            if (U8)
            {
                const float4 pp = lds_f4(par_addr + (j >> 1) * 16);
                acc += rowc + __float_as_int((j & 1) ? pp.w : pp.z) - (e.has_bias ? __ldg(e.bias + oc) : 0);
                if (BORDER && pad) acc += __ldg(btab + (size_t)pad * ocp + oc);
            }
            w |= ((uint32_t)requant(acc, oc, e) & 0xffu) << (8 * j);
        }
    }
    return w;
}

// One lane's share of a store group: channel word oc0..oc0+3 of the 4*CS rows row0 + k*(8/CS) of the image (row0: the lane's
// first row of the m-tile), v[k] their accumulators -> 4*CS output words, one 32-bit store each into the warp's staging buffer
// (dst[k & 1] + 128 k: the CS == 2 swizzle flips chunk bit 4 on the rows with bit 2 set, i.e. on odd k).  All 4*CS words go
// through the fast requantisation together, so each lane has 4*CS independent chains in flight; f: the word's constants,
// held in registers by the caller (fast modes), par_addr: the same in shared memory (exact mode).
// uint8 flavour: v = sum x*w over in-bounds taps (raw bytes), sx = sum x.  The true accumulator is
//   sum (x-zx)(w-zw) = v - zw*sx + corr[oc] + sum_{padding taps t} btab[t][oc]
// with corr[oc] = -zx*sum_k w + taps*Cin*zx*zw (interior pixels).  The per-channel constants are in the int8 layout
// { M[2k], M[2k+1], y[2k], y[2k+1] } with y = corr + bias (an integer), so the fast path IS the int8 one on
// a' = v + rowc[k] + btab[pad[k]] (BORDER only) + y: t = fl((float)a' * M), exact up to the tie guard under the bound engine.cu
// proves per layer (|bias*M| <= 250).  rowc[k] = cplane * sx of row k.
// MODE: 0 fast, 1 fast with the bias fused into the FMA (int8 only), 2 exact (literal arithmetic for every element: degenerate
// scales, or accumulators that could leave the 16-bit clamp range).
template <bool U8, int MODE, int CS, bool BORDER>
__device__ __forceinline__ void epilogue_words(const uint32_t (&v)[4 * CS][4], const int32_t (&rowc)[4 * CS], const uint32_t (&pad)[4 * CS],
                                               const FastPar4& f, uint32_t par_addr, int oc0, uint32_t row0, const uint32_t (&dst)[2],
                                               uint32_t mtile, const GemmArgs& g, const EpiParams& e)
{
    constexpr int W = 4 * CS, RPI = 8 / CS;
    constexpr bool FUSE = !U8 && MODE == 1;
    uint32_t w[W];
    if (MODE != 2)
    {
        const int32_t y[4] = {__float_as_int(f.a.z), __float_as_int(f.a.w), __float_as_int(f.b.z), __float_as_int(f.b.w)}; // uint8: integers
        int32_t a[W][4];
#pragma unroll
        for (int k = 0; k < W; k++)
#pragma unroll
            for (int j = 0; j < 4; j++) a[k][j] = (int32_t)v[k][j] + (U8 ? rowc[k] : 0); // (+ y inside requant_fast_words_i8<false>)
        if (U8 && BORDER && oc0 < g.ocp) // (channels of an N tile past ocp have no table entries; they come out 0)
        {
#pragma unroll
            for (int k = 0; k < W; k++)
                if (pad[k])
                {
                    // border row: the summed corrections of its missing taps, one 16-byte load per word
                    const int4 c = __ldg(reinterpret_cast<const int4*>(g.btab + (size_t)pad[k] * g.ocp + oc0));
                    a[k][0] += c.x, a[k][1] += c.y, a[k][2] += c.z, a[k][3] += c.w;
                }
        }
        float gw[W];
        const FastPar4 fp[1] = {f};
        requant_fast_words_i8<FUSE, W, 1>(a, fp, e, w, gw);
        if (e.q_byte_add)
        {
#pragma unroll
            for (int k = 0; k < W; k++) w[k] = requant_byte_fix(w[k], e);
        }
        float gmax = gw[0];
#pragma unroll
        for (int k = 1; k < W; k++) gmax = fmaxf(gmax, gw[k]);
        if (gmax > 0.5f - TB200_TIE_EPS)
        {
            // rare (2.4e-4 of the elements): the guarded words again -- gemm_fix_word finds the elements inside the band and queues
            // them for the literal reference arithmetic
#pragma unroll
            for (int k = 0; k < W; k++)
                if (gw[k] > 0.5f - TB200_TIE_EPS)
                {
                    const uint32_t row = row0 + (uint32_t)(k * RPI);
                    if (U8)
                        w[k] = gemm_fix_word<true, false>(w[k], a[k][0] + y[0], a[k][1] + y[1], a[k][2] + y[2], a[k][3] + y[3], oc0, g.oc, mtile, row, e);
                    else
                        w[k] = gemm_fix_word<false, FUSE>(w[k], a[k][0], a[k][1], a[k][2], a[k][3], oc0,
                                                          0x7fffffff /* pad channels have M = y = 0: never guarded */, mtile, row, e);
                }
        }
        if (U8 && oc0 + 4 > g.oc)
        {
            // pad lanes of uint8 tensors hold 0, not the zero point
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (oc0 + j >= g.oc)
#pragma unroll
                    for (int k = 0; k < W; k++) w[k] &= ~(0xffu << (8 * j));
        }
    }
    else
    {
#pragma unroll
        for (int k = 0; k < W; k++)
            w[k] = epilogue_word_exact<U8, BORDER>(v[k][0], v[k][1], v[k][2], v[k][3], rowc[k], pad[k], par_addr, oc0, g.oc, g.ocp, g.btab, e);
    }
#pragma unroll
    for (int k = 0; k < W; k++) sts_b32(dst[k & 1] + 128u * k, w[k]);
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
// multiplied the epilogue drains the previous one from the image; the fragments are then written into each 32-row quarter of the
// image once that quarter's two epilogue warps have read it (img_empty[q]) and published with img_full[q].  BN, MT and the operand
// signs are template parameters so that the accumulators are indexed statically and no wgmma sits in a branch the compiler cannot
// prove uniform.
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
        // Hand the stage over per 32-row image quarter.  Warp w of the warpgroup holds rows 16w..16w+15 of each half h, i.e. half of
        // quarter q = 2h + w/2; warp w ^ 1 holds the other half, and only epilogue warps 8 + q and 12 + q read it.  So each quarter
        // waits for its own two readers only, not for the slowest of all eight.
        const int wq = (threadIdx.x >> 6) & 1; // w / 2
#pragma unroll
        for (int h = 0; h < 2; h++)
        {
            const int q = 2 * h + wq;
            mbar_wait(&ctl->img_empty[q], iphase ^ 1); // both epilogue warps of quarter q have read the previous stage out of it
            if (h == 0) tlog(1, 1);
#pragma unroll
            for (int i = 0; i < MT; i++)
            {
                if (i >= mtc) break;
#pragma unroll
                for (int c = 0; c < BN / 16; c++)
                    frag_to_image(*reinterpret_cast<const uint32_t(*)[8]>(&acc[i][h][8 * c]), img_base, img_pitch, h * 64, i * BN + c * 16);
            }
            __syncwarp();
            if ((threadIdx.x & 31) == 0) mbar_arrive(&ctl->img_full[q]); // (release) this warp's rows of quarter q are in the image
        }
        tlog(1, 2);
        iphase ^= 1;
        // The four warps leave these waits at different times and need no barrier among themselves before the next stage's
        // wgmma_fence: wgmma.fence / mma_async / commit / wait are .sync.aligned warpgroup-collective instructions that the
        // hardware synchronises across the four warps, just as after the ring's full-barrier waits, which each warp leaves on
        // its own too.
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
        for (int q = 0; q < 4; q++) mbar_init(&ctl->img_full[q], 2), mbar_init(&ctl->img_empty[q], 2);
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
        // warps.  Inside a group lane L owns channel word w = L % (4 cs) (channels cg0 + 4w .. +3) of the 4 cs rows
        // L / (4 cs) + k * (8 / cs), k = 0 .. 4 cs - 1: it issues the 4 cs image loads of its rows first, then requantises the
        // 4 cs words together with the word's constants in registers, and writes each word with one 32-bit store into the warp's
        // own swizzled staging buffer, which it hands to the TMA unit with one store.  It releases its quarter of the image to
        // the MMA warpgroup (img_empty[q]) as soon as it has issued its last load of the stage; a warp with no group in the
        // stage, or whose quarter has no valid rows, arrives at the end of the stage, so each warp arrives once per stage.
        // Shared-memory banks (a 16-byte access is served eight lanes at a time, 128 bytes per wavefront):
        //   image loads, cs 2: the eight lanes of a quarter-warp read the 8 words = 128 contiguous bytes of one row: one
        //     wavefront each, 4 per instruction (512 bytes), the minimum.
        //   image loads, cs 1: a quarter-warp reads 64 contiguous bytes of each of two rows, one pitch apart; the pitch
        //     (cols * 4 + 16, cols a multiple of 16) is 16 or 80 modulo 128, so the two 64-byte runs share banks: 2 wavefronts
        //     per quarter-warp.  Only the cs 1 plans (N tiles of an odd number of 16-channel chunks, which MobileNet-v1 has
        //     none of) pay it; a pitch of 64 modulo 128 would cost every plan 6 KB of ring and the MMA warps' conflict-free
        //     fragment stores.
        //   staging stores: instruction k writes rows 4k / 8k .. of the buffer, i.e. bytes [128 k, 128 k + 128) (permuted by
        //     the swizzle inside), 4 bytes per lane: one wavefront.
        //   constants: the lanes of one word read the same 32 bytes (broadcast), 4 cs distinct 16-byte addresses: one wavefront.
        setmaxnreg_inc<REG_EPI>();
        constexpr int WPR = 4 * CS, RPI = 8 / CS; // words per group row, rows per warp-wide load
        const int ew = warp - EPI_WARP0; // epilogue warp 0..7
        const int q = warp & 3;
        const int sub = ew >> 2;
        const int et = (int)threadIdx.x - EPI_THREAD0;
        const int ngroups = g.ngroups;
        int qrows = g.rows_valid - q * 32; // rows of this quarter that are output pixels
        qrows = qrows < 0 ? 0 : (qrows > 32 ? 32 : qrows);
        const CUtensorMap* tm_out = (qrows == 32) ? &tmap_out : &tmap_out_tail;
        const uint32_t buf0 = stg_base + (uint32_t)ew * 2u * buf_bytes;
        const int lw = lane % WPR, lr = lane / WPR; // this lane's word and first row of a group
        const uint32_t img_lane = img_base + (uint32_t)(q * 32 + lr) * img_pitch + 16u * (uint32_t)lw;
        // staging offsets of word lw in rows lr + RPI k: even k, and odd k, whose row has bit 2 set, so that the output map's
        // swizzle (16-byte chunk index ^= row bit 2, Swizzle<1,4,3>, CS 2 only) flips the chunk
        uint32_t st_off[2];
        st_off[0] = (uint32_t)lr * (16u * CS) + 4u * (uint32_t)lw;
        st_off[1] = CS == 2 ? st_off[0] ^ 16u : st_off[0];
        uint32_t ucount = 0; // groups this warp has stored (buffer parity)
        const int par_ch = g.n_tiles * g.block_n;
        const bool fast = MODE != 2;
        FastPar4 f = {};       // fast modes: this lane's word's constants ...
        uint32_t par_at = ~0u; // ... from this shared-memory address (~0: none)
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
                par_at = ~0u; // the registers hold the previous tile's constants
            }
            mbar_wait(&ctl->img_full[q], iphase); // this warp's quarter of the image holds this stage
            iphase ^= 1;
            if (U8 && g.cplane) mbar_wait(&ctl->sx_full[as], aphase); // the row sums of this stage
            TLOG_E(0);
            bool released = false; // this warp has arrived on img_empty for this stage
            if (qrows > 0)
            {
                // groups of this warp: flattened index u = i * ngroups + grp, u = sub, sub + 2, ...
                int i = 0, grp = sub;
                while (grp >= ngroups) grp -= ngroups, i++;
                while (i < mtc)
                {
                    int i2 = i, g2 = grp + 2; // the group after this one
                    while (g2 >= ngroups) g2 -= ngroups, i2++;
                    const uint32_t buf = buf0 + (ucount & 1u) * buf_bytes;
                    // the store issued two groups ago has finished reading this buffer
                    if (lane == 0) bulk_wait_read<1>();
                    __syncwarp();
                    const int cg0 = grp * (CS * 16); // first column of the group inside the N tile
                    const int c = cg0 + 4 * lw;      // first channel of this lane's word inside the N tile
                    // the accumulators of this lane's rows, all loads in flight before the first is used
                    uint32_t v[WPR][4];
                    const uint32_t src = img_lane + 4u * (uint32_t)(i * g.block_n + cg0);
#pragma unroll
                    for (int k = 0; k < WPR; k++)
                    {
                        const uint4 u = lds_u4(src + (uint32_t)(k * RPI) * img_pitch);
                        v[k][0] = u.x, v[k][1] = u.y, v[k][2] = u.z, v[k][3] = u.w;
                    }
                    TLOG_E(3);
                    if (i2 >= mtc)
                    {
                        // the last image loads of the stage are issued: (release) the MMA warpgroup may overwrite the image
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&ctl->img_empty[q]);
                        released = true;
                    }
                    const uint32_t pa = par_s + (uint32_t)c * 8u; // the word's constants in shared memory
                    if (MODE != 2 && pa != par_at) f.a = lds_f4(pa), f.b = lds_f4(pa + 16u), par_at = pa; // (the group's columns changed)
                    int32_t rowc[WPR];
                    uint32_t pad[WPR];
#pragma unroll
                    for (int k = 0; k < WPR; k++) rowc[k] = 0, pad[k] = 0;
                    if (U8)
                    {
                        if (g.cplane)
                        {
                            // the rows' sum(x) terms
                            const uint32_t sx = sx_base + (uint32_t)(((as * 4 + i) * 128 + q * 32 + lr) * 4);
#pragma unroll
                            for (int k = 0; k < WPR; k++)
                            {
                                int32_t s;
                                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(s) : "r"(sx + (uint32_t)(k * RPI * 4)));
                                rowc[k] = g.cplane * s;
                            }
                        }
                        if (BORDER)
                        {
                            // border pattern of row `lane` of the quarter, then each lane fetches those of its own rows
                            const uint32_t pl = padding_taps(g, mt0 + i, q * 32 + lane);
#pragma unroll
                            for (int k = 0; k < WPR; k++) pad[k] = __shfl_sync(0xffffffffu, pl, lr + k * RPI);
                        }
                    }
                    const uint32_t dst[2] = {buf + st_off[0], buf + st_off[1]};
                    epilogue_words<U8, MODE, CS, BORDER>(v, rowc, pad, f, pa, n0 + c, (uint32_t)(q * 32 + lr), dst, (uint32_t)(mt0 + i), g, e);
                    TLOG_E(4);
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
                if (!released) mbar_arrive(&ctl->img_empty[q]); // a warp without a group in this stage (or a quarter without valid rows)
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
static void plan_stage(GemmArgs& g, long long m_tiles)
{
    g.mt = 1;
    if (g.n_tiles == 1)
        while (g.mt < 4 && (g.mt * 2) * g.block_n <= ACC_COLS_MAX && g.mt * 2 <= m_tiles) g.mt *= 2;
    const int nch = g.block_n / 16;
    g.cs = (nch % 2 == 0 && (g.mt * (nch / 2)) % 4 == 0) ? 2 : 1;
    g.ngroups = nch / g.cs;
}

// Output tensor maps: a box of 32 rows x one store group; 32-byte groups are swizzled like the warp's staging buffer.
static int plan_epilogue(GemmPlan* p, const void* out, uint64_t d1, uint64_t d2)
{
    const int cs = p->g.cs;
    const uint64_t dims[3] = {(uint64_t)p->g.ocp, d1, d2};
    const uint64_t strides[2] = {(uint64_t)p->g.ldo, (uint64_t)p->g.ldo * d1};
    const int swz = cs == 2 ? 32 : 0;
    const uint32_t box[3] = {(uint32_t)(16 * cs), 32u, 1u};
    int rc = tmap_encode(&p->tmap_out, out, 3, dims, strides, box, nullptr, swz);
    if (rc) return rc;
    const int tail = p->g.rows_valid % 32;
    const uint32_t box_t[3] = {(uint32_t)(16 * cs), (uint32_t)(tail ? tail : 32), 1u};
    return tmap_encode(&p->tmap_out_tail, out, 3, dims, strides, box_t, nullptr, swz);
}

// shared memory the epilogue needs next to the operand ring, with `warps` output staging warps: their double-buffered store
// groups, the control block, the epilogue constants and the accumulator image
static int epilogue_smem_bytes(const GemmArgs& g, int warps)
{
    return warps * 2 * 512 * g.cs + (int)sizeof(GemmSmemCtl) + (g.par_all ? g.n_tiles * g.block_n : g.block_n) * 8 + 16 +
           128 * (int)acc_pitch(g.mt * g.block_n);
}

// Operand ring depth and the resident-B decision.  With the N tile's weights resident the ring carries A tiles only,
// which for the small-K layers (K = 32..128, one 4-16 KB A tile per m-tile) is the difference between 8 and 24 m-tiles
// of prefetch distance.  Then the launch: one persistent CTA per SM at most, and the dynamic shared memory.
static int plan_ring(GemmPlan* p, long long m_tiles, int num_sms)
{
    GemmArgs& g = p->g;
    g.m_tiles = (int)m_tiles;
    plan_stage(g, m_tiles);
    g.par_all = g.n_tiles * g.block_n <= PAR_MAX ? 1 : 0;
    const int a_bytes = BLOCK_M * g.block_k, b_al = (g.block_n * g.block_k + 1023) & ~1023, sx_bytes = g.cplane ? 4096 : 0;
    const int budget = 224 * 1024 - epilogue_smem_bytes(g, PLAN_STG_WARPS) - 2048 - sx_bytes;
    g.b_res = (long long)g.k_blocks * b_al <= B_RESIDENT_MAX ? 1 : 0;
    int stages = g.b_res ? (budget - g.k_blocks * b_al) / a_bytes : budget / (a_bytes + b_al);
    if (g.b_res && stages < 3) g.b_res = 0, stages = budget / (a_bytes + b_al);
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    if (stages < 2) return TB200_ERR_INVALID;
    g.stages = stages;
    // + 1024: the kernel aligns the ring to 1024 bytes
    p->smem_bytes = stages * (a_bytes + (g.b_res ? 0 : b_al)) + (g.b_res ? g.k_blocks * b_al : 0) + sx_bytes + epilogue_smem_bytes(g, EPI_WARPS) + 1024;
    g.num_super = (int)(((m_tiles + g.mt - 1) / g.mt) * g.n_tiles);
    p->grid = g.num_super < num_sms ? g.num_super : num_sms;
    if (g.b_res) p->grid -= p->grid % g.n_tiles; // a CTA must see one N tile only (num_super is a multiple of n_tiles, so grid >= n_tiles)
    return 0;
}

// What both planners set first: the output, the epilogue, the N tiles and the operands.  u8 = 1 + weight zero point for uint8
// layers: A is unsigned, and unless zw == 0 B holds w - 128 and the epilogue adds cplane * sum(x).
static void plan_begin(GemmPlan* p, void* out, int oc, int ocp, int ldo, int u8, const EpiParams& e, const int32_t* btab, void* fixq, int fixq_cap)
{
    memset(p, 0, sizeof *p);
    GemmArgs& g = p->g;
    g.oc = oc, g.ocp = ocp, g.ldo = ldo, g.out_base = (uint8_t*)out;
    g.block_n = gemm_block_n(ocp);
    g.n_tiles = (ocp + g.block_n - 1) / g.block_n;
    g.u8 = u8 != 0;
    g.b_signed = !g.u8 || u8 != 1;
    g.cplane = (g.u8 && u8 != 1 && !getenv("TB200_DEBUG_NO_CPLANE")) ? 128 - (u8 - 1) : 0; // (debug switch: WRONG results, timing experiments only)
    g.btab = btab, g.fixq = (uint4*)fixq, g.fixq_cap = fixq_cap;
    p->e = e;
    p->mode = epi_mode(e, g.u8);
}

int gemm_plan_create(GemmPlan* p, const void* a, long long lda, const void* b, void* out, long long m, int k, int oc, int ocp, int ldo, int u8,
                     const EpiParams& e, const int32_t* btab, void* fixq, int fixq_cap, int num_sms)
{
    if (m <= 0 || k <= 0 || (k & 15) || (ocp & 15) || (lda & 15) || (ldo & 15)) return TB200_ERR_INVALID;
    plan_begin(p, out, oc, ocp, ldo, u8, e, btab, fixq, fixq_cap);
    GemmArgs& g = p->g;
    g.m_rows = (int)m;
    g.block_k = k <= 32 ? 32 : (k <= 64 ? 64 : 128);
    g.swizzle = g.block_k;
    g.k_blocks = (k + g.block_k - 1) / g.block_k;
    g.taps = 1;
    int rc = plan_ring(p, (m + BLOCK_M - 1) / BLOCK_M, num_sms);
    if (rc) return rc;
    rc = encode_2d(&p->tmap_a, a, (uint64_t)k, (uint64_t)m, (uint64_t)lda, g.block_k, BLOCK_M, g.swizzle);
    if (rc) return rc;
    rc = encode_2d(&p->tmap_b, b, (uint64_t)k, (uint64_t)g.n_tiles * g.block_n, (uint64_t)k, g.block_k, g.block_n, g.swizzle);
    if (rc) return rc;
    g.rows_valid = BLOCK_M, g.out_mode = 0;
    return plan_epilogue(p, out, (uint64_t)m, 1);
}

// Implicit-GEMM plan for a dense (group 1, dilation 1) convolution with any kernel size and stride 1 or 2:
// A = 4-D tensor map (C, W, H, N) over the NHWC input with traversal strides (1, s, s, 1); B = [OCp][taps*Cp].
int gemm_plan_create_conv(GemmPlan* p, const void* in, const void* w, void* out, const ConvShape& s, int u8, const EpiParams& e,
                          const int32_t* btab, void* fixq, int fixq_cap, int num_sms)
{
    if (s.group != 1 || s.dh != 1 || s.dw != 1 || s.sh != s.sw || (s.sh != 1 && s.sh != 2)) return TB200_ERR_UNSUPPORTED;
    const int taps = s.kh * s.kw;
    if (taps > 1 && (s.cp % 32)) return TB200_ERR_UNSUPPORTED; // a k-block must not straddle two taps
    if (taps > 64) return TB200_ERR_UNSUPPORTED;
    plan_begin(p, out, s.oc, s.ocp, s.ocp, u8, e, btab, fixq, fixq_cap);
    GemmArgs& g = p->g;
    g.conv = 1;
    g.m_rows = (int)((long long)s.n * s.oh * s.ow);
    if (taps == 1) g.block_k = s.cp <= 32 ? 32 : (s.cp <= 64 ? 64 : 128);
    else g.block_k = (s.cp % 128 == 0) ? 128 : ((s.cp % 64 == 0) ? 64 : 32);
    g.swizzle = g.block_k;
    g.cblocks = (s.cp + g.block_k - 1) / g.block_k;
    g.k_blocks = taps * g.cblocks;
    const int k = taps * s.cp;
    g.taps = taps, g.in_h = s.h, g.in_w = s.w;
    // output patch of one m-tile: whole rows when they fit (then the patch is contiguous in the NHWC output)
    if (s.ow <= BLOCK_M)
    {
        g.bw = s.ow;
        g.bh = BLOCK_M / s.ow < s.oh ? BLOCK_M / s.ow : s.oh;
        g.bn = (g.bh == s.oh) ? BLOCK_M / (s.ow * s.oh) : 1;
        if (g.bn > s.n) g.bn = s.n;
        if (g.bn < 1) g.bn = 1;
    }
    else
        g.bw = BLOCK_M, g.bh = 1, g.bn = 1;
    g.bw_rcp = (65536u + (uint32_t)g.bw - 1) / (uint32_t)g.bw;
    g.bh_rcp = (65536u + (uint32_t)g.bh - 1) / (uint32_t)g.bh;
    g.tiles_w = (s.ow + g.bw - 1) / g.bw;
    g.tiles_h = (s.oh + g.bh - 1) / g.bh;
    const long long tiles_n = (s.n + g.bn - 1) / g.bn;
    g.kw_n = s.kw, g.pad_h = s.ph0, g.pad_w = s.pw0, g.cstride = s.sh, g.cp = s.cp, g.oh = s.oh, g.ow = s.ow, g.nimg = s.n;
    g.a_tx_bytes = (uint32_t)(g.block_k * g.bw * g.bh * g.bn);
    // uint8 border corrections only exist for convolutions with taps that can fall into the padding: any window larger than one
    // pixel, or a 1x1 window whose last row / column lies past the image (bottom / right padding, e.g. TF-style (0, 1))
    const bool pad_1x1 = s.ph0 || s.pw0 || (s.oh - 1) * s.sh >= s.h || (s.ow - 1) * s.sh >= s.w;
    p->border = g.u8 && (taps > 1 || pad_1x1);
    int rc = plan_ring(p, (long long)g.tiles_w * g.tiles_h * tiles_n, num_sms);
    if (rc) return rc;
    const uint64_t dims[4] = {(uint64_t)s.cp, (uint64_t)s.w, (uint64_t)s.h, (uint64_t)s.n};
    const uint64_t strides[3] = {(uint64_t)s.cp, (uint64_t)s.w * s.cp, (uint64_t)s.h * s.w * s.cp};
    const uint32_t box[4] = {(uint32_t)g.block_k, (uint32_t)((g.bw - 1) * s.sw + 1), (uint32_t)((g.bh - 1) * s.sh + 1), (uint32_t)g.bn};
    const uint32_t estr[4] = {1u, (uint32_t)s.sw, (uint32_t)s.sh, 1u};
    if (box[1] > 256 || box[2] > 256 || box[3] > 256) return TB200_ERR_UNSUPPORTED;
    rc = tmap_encode(&p->tmap_a, in, 4, dims, strides, box, estr, g.swizzle);
    if (rc) return rc;
    rc = encode_2d(&p->tmap_b, w, (uint64_t)k, (uint64_t)g.n_tiles * g.block_n, (uint64_t)k, g.block_k, g.block_n, g.swizzle);
    if (rc) return rc;
    // The rows of an m-tile are consecutive output pixels along one axis of the NHWC output (see the patch shapes above):
    //   bn > 1 (whole images)   : rows = pixels of bn consecutive images        -> map (C, N*OH*OW, 1), clipped at the end
    //   bn == 1, bw == OW       : rows = pixels of image n from row oh0 on       -> map (C, OH*OW, N), clipped per image
    //   bw == 128 < OW          : rows = 128 pixels of one image row             -> map (C, OW, N*OH), clipped per row
    g.rows_valid = g.bw * g.bh * g.bn;
    if (g.bw != s.ow)
    {
        g.out_mode = 2;
        return plan_epilogue(p, out, (uint64_t)s.ow, (uint64_t)s.n * s.oh);
    }
    if (g.bn > 1)
    {
        g.out_mode = 0;
        return plan_epilogue(p, out, (uint64_t)s.n * s.oh * s.ow, 1);
    }
    g.out_mode = 1;
    return plan_epilogue(p, out, (uint64_t)s.oh * s.ow, (uint64_t)s.n);
}

// debug: event timeline of CTA 0 of the launch that just went out (needs a stream that is not being captured).
// One line per event, sorted by time: cycles since the first event, role (P producer, M mma, E8/E15 epilogue warps), tag.
static void gemm_trace_report(const GemmArgs& g, int grid, cudaStream_t st)
{
    static unsigned long long h[4 * 1024];
    if (cudaStreamSynchronize(st) != cudaSuccess) return;
    cudaMemcpy(h, g.trace, sizeof h, cudaMemcpyDeviceToHost);
    fprintf(stderr, "[gemm timeline] m_tiles=%lld k_blocks=%d bn=%d mt=%d stages=%d b_res=%d cs=%d grid=%d\n", (long long)g.m_tiles, g.k_blocks,
            g.block_n, g.mt, g.stages, g.b_res, g.cs, grid);
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

cudaError_t launch_gemm_i8(const GemmPlan& p, cudaStream_t st)
{
    if (p.grid <= 0) return cudaErrorInvalidValue; // plan was never created
    static const bool trace_on = getenv("TB200_GEMM_TRACE") != nullptr;
    const bool launch_dbg = debug_launch();
    static unsigned long long* trace_buf = nullptr;
    GemmArgs g = p.g;
    if (trace_on)
    {
        if (!trace_buf) cudaMalloc(&trace_buf, 4 * 1024 * sizeof(unsigned long long));
        cudaMemsetAsync(trace_buf, 0, 4 * 1024 * sizeof(unsigned long long), st);
        g.trace = trace_buf;
    }
    const int grid = p.grid;
    const size_t smem = (size_t)p.smem_bytes;
    cudaError_t err = cudaErrorInvalidValue;
#define TB200_GEMM_CASE(U, MD, C, B)                                                                                           \
    if ((g.u8 != 0) == U && p.mode == MD && g.cs == C && (p.border != 0) == B)                                                 \
    {                                                                                                                          \
        /* the opt-in is per device AND per context: set it before every launch (launches happen at graph capture only) */ \
        {                                                                                                                      \
            err = cudaFuncSetAttribute(gemm_i8_tcgen05_kernel<U, MD, C, B>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024); \
            if (launch_dbg) gemm_launch_debug((const void*)gemm_i8_tcgen05_kernel<U, MD, C, B>, "set attribute", err, grid, smem, st);    \
            if (err != cudaSuccess) return err;                                                                                \
        }                                                                                                                      \
        if (launch_dbg)                                                                                                        \
            fprintf(stderr, "tengine_b200: launch gemm_i8_tcgen05_kernel<U8=%d,MODE=%d,CS=%d,BORDER=%d> out_mode=%d conv=%d n_tiles=%d b_res=%d fixq=%d mt=%d par_all=%d block_n=%d b_signed=%d cplane=%d\n", \
                    (int)U, MD, C, (int)B, g.out_mode, g.conv, g.n_tiles, g.b_res, g.fixq != nullptr, g.mt, g.par_all, g.block_n,           \
                    (int)g.b_signed, g.cplane);                                                                                        \
        gemm_i8_tcgen05_kernel<U, MD, C, B><<<grid, GEMM_THREADS, smem, st>>>(p.tmap_a, p.tmap_b, p.tmap_out, p.tmap_out_tail, g, p.e); \
        if (trace_on) gemm_trace_report(g, grid, st);                                                                          \
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
