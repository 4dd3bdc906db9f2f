// conv_window.cu -- small-Cin convolutions on the tensor cores: the window kernel (TMA-staged input window) and the gather
// kernel (taps gathered from global memory) it falls back to.
//
// The layers an implicit GEMM over 4-D TMA boxes serves badly: the NCHW network input (C <= 3; 3x3 and 7x7 stems, int8 and
// uint8) and 3x3 convolutions over NHWC tensors with 16 or 32 channels (YOLOv3-tiny's second and third layer).  Their K rows
// are 16-32 bytes per tap, and the TMA unit's cost is per row, not per byte: feeding nine shifted
// 128-row boxes per tile through it left the tensor pipe idle 90% of the time, and gathering every tap from global memory
// with bounds predicates (conv_gather_tc_kernel below) costs more instructions than the whole epilogue.
//
// Here a CTA (128 threads = 16 x 8 output pixels) receives the input window of its tile ONCE -- one 4-D cp.async.bulk.tensor
// load, double-buffered, out-of-image coordinates zero-filled by the TMA unit = the convolution's padding -- and every thread
// builds its pixel's K bytes from shared memory (NHWC: one 16-byte LDS/STS pair per tap and 16 channels; NCHW: byte loads
// packed with IMADs) as one row of `ks` SW32 K-major k-step tiles.  The warpgroup multiplies them with wgmma (64 x 16 x 32
// per instruction) into a shared-memory accumulator image; every thread requantises its own row and stores OCp contiguous bytes.  uint8: border tiles first overwrite the window's
// out-of-image bytes with the input zero point (such taps then contribute (zx-zx)(w-zw) = 0, exactly like the reference,
// which skips them), each thread sums its own row with dp4a, and sum (x-zx)(w-zw) = acc - zw*sum(x) + corr[oc].
// Takes the role of im2col + sgemm of conv_hcl_run (source/device/cpu/op/conv/x86/conv_kernel_x86.c:124-242, 1008-1631) and of
// conv3x3s{1,2}_int8_sse (conv_direct_hcl_int8_x86.c:95,272) for these shapes.
#include <cuda.h>

#include "common.cuh"
#include "kernels.h"
#include "ptx.cuh"
#include "tc_common.cuh"

#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace tb200 {

struct WindowArgs
{
    const uint8_t* w; // [OCp][ks*32]; NCHW: k = (c*KH + kh)*KW + kw ; NHWC: k = (kh*3 + kw)*CB + c ; zero padded
    uint8_t* out;     // NHWC, OCp bytes per pixel
    int n, c, h, w_in, oh, ow, ocp, oc, stride, ph, pw;
    unsigned ntiles;
    int tiles_w, tiles_h;
    uint32_t tw_magic, th_magic; // floor(2^32 / d) + 1: q = umulhi(x, magic) is x / d for the tile counts that occur (checked by the launcher)
    int box_w, box_h, xoff, in_bytes, ks;
    uint32_t fill; // uint8: the input zero point replicated x4 (0 for int8: the TMA zero fill already is the padding)
};

// The B tiles (weights [OCp][ks*32] -> one SW32 K-major tile of OCp rows per k-step) and the epilogue constants into shared
// memory: identical for every CTA, L2 resident.  Int8 MODE 2 reads no constants.
template <int MODE, bool U8>
__device__ __forceinline__ void stage_b_and_constants(const uint8_t* w, int ks, int ocp, uint32_t sB, uint32_t sPar, const EpiParams& e)
{
    const uint32_t b_tile = (uint32_t)ocp * 32u;
    for (int i = threadIdx.x; i < ks * ocp * 2; i += 128)
    {
        const int kb = i / (ocp * 2), j = i - kb * (ocp * 2), r = j >> 1, c16 = j & 1;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(w + ((size_t)r * ks + kb) * 32) + c16);
        sts_u4(sB + (uint32_t)kb * b_tile + sw32_offset(r, c16), v.x, v.y, v.z, v.w);
    }
    for (int c = threadIdx.x; c < ocp; c += 128) sts_f2(sPar + c * 8, (MODE != 2 || U8) ? __ldg(e.fast_par + c) : make_float2(0.f, 0.f));
}

// LAYOUT: 0 NCHW 3x3, 1 NCHW 7x7, 2 NHWC 16 bytes per pixel (3x3), 3 NHWC 32 bytes per pixel (3x3)
template <int MODE, bool U8, int LAYOUT> // MODE: 0 fast, 1 fast + fused bias (int8), 2 exact
__global__ void __launch_bounds__(128) conv_window_tc_kernel(const __grid_constant__ CUtensorMap tmap_in, const WindowArgs a, const __grid_constant__ EpiParams e)
{
    constexpr bool NCHW = LAYOUT < 2;
    constexpr int KHW = LAYOUT == 1 ? 7 : 3;
    constexpr int CB = LAYOUT == 3 ? 32 : 16; // NHWC: bytes per pixel
    extern __shared__ __align__(1024) uint8_t win_smem[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(win_smem) + 1023) & ~(uintptr_t)1023);
    const uint32_t sA = smem_u32(sm), sB = sA + (uint32_t)a.ks * 4096u, b_tile = (uint32_t)a.ocp * 32u, sPar = sB + (uint32_t)a.ks * b_tile;
    const uint32_t in_stride = ((uint32_t)a.in_bytes + 127u) & ~127u;
    const uint32_t sIn = (sPar + (uint32_t)a.ocp * 8u + 127u) & ~127u;
    const uint32_t pitch = acc_pitch(a.ocp), sImg = sIn + 2u * in_stride; // accumulator image [128][pitch]
    __shared__ __align__(8) uint64_t in_full[2];
    const int tid = threadIdx.x;
    const int tw = tid & 15, th = tid >> 4; // the tile is 16 x 8 output pixels

    if (tid == 0)
    {
        mbar_init(&in_full[0], 1), mbar_init(&in_full[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto tile_coords = [&](unsigned tile, int& n, int& oh0, int& ow0)
    {
        // two divisions by launch constants as multiply-high (a 32-bit division costs ~40 instructions and this runs per tile)
        const unsigned r = a.tw_magic ? __umulhi(tile, a.tw_magic) : tile; // magic 0: divisor 1
        ow0 = (int)(tile - r * a.tiles_w) * 16;
        n = (int)(a.th_magic ? __umulhi(r, a.th_magic) : r);
        oh0 = (int)(r - (unsigned)n * a.tiles_h) * 8;
    };
    // (a macro, not a lambda: the tensor map must be addressed as the kernel parameter itself)
#define TB200_WIN_LOAD_TILE(TILE, BUF)                                                                                                  \
    do                                                                                                                                  \
    {                                                                                                                                   \
        int n_, oh0_, ow0_;                                                                                                             \
        tile_coords((TILE), n_, oh0_, ow0_);                                                                                            \
        mbar_expect_tx(&in_full[(BUF)], (uint32_t)a.in_bytes);                                                                          \
        if (NCHW)                                                                                                                       \
            tma_load_4d(&tmap_in, &in_full[(BUF)], sm + (sIn - sA) + (size_t)(BUF) * in_stride, ow0_ * a.stride - a.pw - a.xoff,       \
                        oh0_ * a.stride - a.ph, 0, n_);                                                                                 \
        else                                                                                                                            \
            tma_load_4d(&tmap_in, &in_full[(BUF)], sm + (sIn - sA) + (size_t)(BUF) * in_stride, 0, ow0_ * a.stride - a.pw,              \
                        oh0_ * a.stride - a.ph, n_);                                                                                    \
    } while (0)
    if (tid == 0 && blockIdx.x < a.ntiles) TB200_WIN_LOAD_TILE(blockIdx.x, 0);
    stage_b_and_constants<MODE, U8>(a.w, a.ks, a.ocp, sB, sPar, e);
    if (LAYOUT == 2) sts_u4(sA + 4u * 4096u + sw32_offset(tid, 1), 0u, 0u, 0u, 0u); // K = 144 of 160: the last half k-step stays 0

    uint32_t it = 0;
    for (unsigned tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x, it++)
    {
        int n, oh0, ow0;
        tile_coords(tile, n, oh0, ow0);
        const int oh = oh0 + th, ow = ow0 + tw;
        const bool valid = oh < a.oh && ow < a.ow;
        const unsigned pix = ((unsigned)n * a.oh + oh) * a.ow + ow;
        const int buf = it & 1;
        mbar_wait(&in_full[buf], (it >> 1) & 1);
        const uint32_t win = sIn + (uint32_t)buf * in_stride;
        if (U8 && a.fill)
        {
            // uint8 border tiles: bytes of the window that lie outside the image become the input zero point
            const int iy0 = oh0 * a.stride - a.ph, ix0 = ow0 * a.stride - a.pw - (NCHW ? a.xoff : 0);
            if (iy0 < 0 || ix0 < 0 || iy0 + a.box_h > a.h || ix0 + a.box_w > a.w_in) // uniform over the CTA
            {
                if (NCHW)
                {
                    // one thread per window row (C * box_h of them); only the columns the gather reads: [xoff, xoff + 15*S + K)
                    const int x_lo = a.xoff, x_hi = a.xoff + 15 * a.stride + KHW;
                    for (int row = tid; row < a.c * a.box_h; row += 128)
                    {
                        const int y = row % a.box_h;
                        const bool row_oob = iy0 + y < 0 || iy0 + y >= a.h;
                        const uint32_t rp = win + (uint32_t)(row * a.box_w);
                        for (int x = x_lo; x < x_hi; x++)
                            if (row_oob || ix0 + x < 0 || ix0 + x >= a.w_in) asm volatile("st.shared.u8 [%0], %1;" ::"r"(rp + (uint32_t)x), "r"(a.fill & 0xffu) : "memory");
                    }
                }
                else
                {
                    // real channels only: pad lanes (c >= C) hold 0 in the tensor and must stay 0
                    for (int p = tid; p < a.box_w * a.box_h; p += 128)
                    {
                        const int x = p % a.box_w, y = p / a.box_w;
                        if (iy0 + y < 0 || iy0 + y >= a.h || ix0 + x < 0 || ix0 + x >= a.w_in)
                            for (int c = 0; c < a.c; c++)
                                asm volatile("st.shared.u8 [%0], %1;" ::"r"(win + (uint32_t)(p * CB + c)), "r"(a.fill & 0xffu) : "memory");
                    }
                }
                __syncthreads();
            }
        }
        // ---- gather this pixel's K bytes from the window into one row of the k-step tiles ----
        int32_t sx = 0;
        if (NCHW)
        {
            constexpr int NW = KHW == 3 ? 8 : 40; // 32-bit words per row (K = 27 -> 32 bytes, K = 147 -> 160 bytes)
            uint32_t row[NW];
#pragma unroll
            for (int j = 0; j < NW; j++) row[j] = 0;
            // row bases advance by box_w (and by the rest of the plane between channels): the 27 / 147 byte loads then carry
            // immediate offsets 0..K-1 instead of one IMAD each
            uint32_t rb = win + (uint32_t)((th * a.stride) * a.box_w + tw * a.stride + a.xoff);
            const uint32_t plane_skip = (uint32_t)((a.box_h - KHW) * a.box_w);
#pragma unroll
            for (int c = 0; c < 3; c++)
            {
                if (c < a.c)
                {
#pragma unroll
                    for (int kh = 0; kh < KHW; kh++)
                    {
#pragma unroll
                        for (int kw = 0; kw < KHW; kw++)
                        {
                            uint32_t b;
                            asm volatile("ld.shared.u8 %0, [%1];" : "=r"(b) : "r"(rb + (uint32_t)kw)); // rb + constant: folds into the load's immediate
                            const int k = (c * KHW + kh) * KHW + kw; // compile-time after unrolling
                            row[k >> 2] += b << (8 * (k & 3));       // disjoint bytes: add == or (IMAD, off the ALU pipe)
                        }
                        rb += (uint32_t)a.box_w;
                    }
                    rb += plane_skip;
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
        else
        {
            constexpr int CH = CB / 16; // 16-byte chunks per tap
            const uint32_t base = win + (uint32_t)(((th * a.stride) * a.box_w + tw * a.stride) * CB);
#pragma unroll
            for (int t = 0; t < 9; t++)
            {
#pragma unroll
                for (int h = 0; h < CH; h++)
                {
                    const uint4 v = lds_u4(base + (uint32_t)(((t / 3) * a.box_w + (t % 3)) * CB + h * 16));
                    if (U8) sx = (int32_t)__dp4a(v.w, 0x01010101u, __dp4a(v.z, 0x01010101u, __dp4a(v.y, 0x01010101u, __dp4a(v.x, 0x01010101u, (unsigned)sx))));
                    const int j = t * CH + h; // 16-byte chunk index along K
                    sts_u4(sA + (uint32_t)(j >> 1) * 4096u + sw32_offset(tid, j & 1), v.x, v.y, v.z, v.w);
                }
            }
        }
        fence_proxy_async_smem(); // the MMAs read these generic-proxy writes through the async proxy
        __syncthreads();          // (first iteration: also publishes the B tiles and the constants)
        // everybody has read this tile's window: prefetch the next one into the other buffer
        if (tid == 0 && tile + gridDim.x < a.ntiles) TB200_WIN_LOAD_TILE(tile + gridDim.x, (it + 1) & 1);
        wg_mma_to_image<U8, U8>(sA, 4096u, sB, b_tile, a.ks, 32, a.ocp, sImg, pitch);
        __syncthreads();

        // ---- epilogue: thread = pixel = accumulator row, 16 channels per load, OCp contiguous output bytes per pixel ----
        uint8_t* op = a.out + (size_t)pix * a.ocp;
        const uint32_t tb = sImg + (uint32_t)tid * pitch;
        const int32_t rowc = U8 ? -e.w_zero * sx : 0;
        for (int c = 0; c < a.ocp; c += 16)
        {
            uint32_t v[16], w[4];
            acc_ld16(tb + 4u * c, v);
            tc_unit16<MODE, U8>(v, rowc, sPar + c * 8, c, a.oc, e, w);
            if (valid) *reinterpret_cast<uint4*>(op + c) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        // the next tile's MMAs overwrite the accumulator image and its gather overwrites the A tiles
        __syncthreads();
    }
#undef TB200_WIN_LOAD_TILE
}

// ---- host side ------------------------------------------------------------------------------------------------------------
static constexpr int WINDOW_SMEM_MAX = 200 * 1024;

// shared memory of one CTA: A tiles, B tiles, constants, the double-buffered input window, the accumulator image
static int window_smem_bytes(int ks, int ocp, int in_bytes)
{
    return ks * 4096 + ks * ocp * 32 + ocp * 8 + 128 + 2 * ((in_bytes + 127) & ~127) + 128 * (int)acc_pitch(ocp) + 1024;
}

bool window_nhwc_fits(int cp, int ocp, int stride)
{
    const int box_w = 15 * stride + 3, box_h = 7 * stride + 3;
    return window_smem_bytes((9 * cp + 31) / 32, ocp, box_w * box_h * cp) <= WINDOW_SMEM_MAX;
}
// nhwc == 0: `in` is the NCHW network input (C <= 3); the tensor map is (W, H, C, N) with box (box_w, box_h, C, 1).
// nhwc == 1: `in` is an NHWC tensor with cp = 16 or 32 bytes per pixel; the map is (cp, W, H, N) with box (cp, box_w, box_h, 1).
int window_plan_create(WindowPlan* p, const void* in, const ConvShape& s, int nhwc)
{
    memset(p, 0, sizeof *p);
    if (s.group != 1 || s.dh != 1 || s.dw != 1 || s.sh != s.sw || s.sh < 1 || s.sh > 2 || s.kh != s.kw || s.ocp > 256) return -1;
    if (nhwc)
    {
        if (s.kh != 3 || (s.cp != 16 && s.cp != 32)) return -1;
        p->layout = s.cp == 16 ? 2 : 3;
        p->xoff = 0;
        p->box_w = 15 * s.sw + 3, p->box_h = 7 * s.sh + 3;
        p->in_bytes = p->box_w * p->box_h * s.cp;
        p->ks = (9 * s.cp + 31) / 32;
        const uint64_t dims[4] = {(uint64_t)s.cp, (uint64_t)s.w, (uint64_t)s.h, (uint64_t)s.n};
        const uint64_t strides[3] = {(uint64_t)s.cp, (uint64_t)s.w * s.cp, (uint64_t)s.h * s.w * s.cp};
        const uint32_t box[4] = {(uint32_t)s.cp, (uint32_t)p->box_w, (uint32_t)p->box_h, 1u};
        if (tmap_encode(p->tmap_in, in, 4, dims, strides, box, nullptr, 0)) return -1;
    }
    else
    {
        if ((s.kh != 3 && s.kh != 7) || s.c > 3 || (s.w % 16)) return -1; // global strides of a tensor map are multiples of 16 bytes
        p->layout = s.kh == 3 ? 0 : 1;
        // the innermost coordinate ow0*S - pw - xoff must be a multiple of 16 (ow0*S is one)
        p->xoff = (16 - (s.pw0 % 16)) % 16;
        p->box_w = (p->xoff + 15 * s.sw + s.kw + 15) & ~15, p->box_h = 7 * s.sh + s.kh;
        if (p->box_w > 256 || p->box_h > 256) return -1;
        p->in_bytes = p->box_w * p->box_h * s.c;
        p->ks = (s.c * s.kh * s.kw + 31) / 32;
        const uint64_t dims[4] = {(uint64_t)s.w, (uint64_t)s.h, (uint64_t)s.c, (uint64_t)s.n};
        const uint64_t strides[3] = {(uint64_t)s.w, (uint64_t)s.w * s.h, (uint64_t)s.w * s.h * s.c};
        const uint32_t box[4] = {(uint32_t)p->box_w, (uint32_t)p->box_h, (uint32_t)s.c, 1u};
        if (tmap_encode(p->tmap_in, in, 4, dims, strides, box, nullptr, 0)) return -1;
    }
    p->smem_bytes = window_smem_bytes(p->ks, s.ocp, p->in_bytes);
    if (p->smem_bytes > WINDOW_SMEM_MAX) return -1;
    p->valid = 1;
    return 0;
}

cudaError_t launch_conv_window(const WindowPlan& p, const void* w, void* out, const ConvShape& s, const EpiParams& e, int num_sms, cudaStream_t st)
{
    if (!p.valid) return cudaErrorInvalidValue;
    if ((long long)s.n * s.oh * s.ow >= (1ll << 31)) return cudaErrorInvalidValue; // 32-bit pixel index
    WindowArgs a;
    a.w = (const uint8_t*)w, a.out = (uint8_t*)out;
    a.n = s.n, a.c = s.c, a.h = s.h, a.w_in = s.w, a.oh = s.oh, a.ow = s.ow, a.ocp = s.ocp, a.oc = s.oc, a.stride = s.sh, a.ph = s.ph0, a.pw = s.pw0;
    a.tiles_w = (s.ow + 15) / 16, a.tiles_h = (s.oh + 7) / 8;
    a.ntiles = (unsigned)((long long)a.tiles_w * a.tiles_h * s.n);
    // umulhi(x, floor(2^32/d) + 1) == x / d whenever x * d < 2^32 (error term x * (d - 2^32 mod d) / (d * 2^32) < 1 / d)
    if ((unsigned long long)a.ntiles * (unsigned)a.tiles_w >= (1ull << 32) || (unsigned long long)a.ntiles * (unsigned)a.tiles_h >= (1ull << 32)) return cudaErrorInvalidValue;
    a.tw_magic = a.tiles_w == 1 ? 0u : (uint32_t)((1ull << 32) / (unsigned)a.tiles_w) + 1u;
    a.th_magic = a.tiles_h == 1 ? 0u : (uint32_t)((1ull << 32) / (unsigned)a.tiles_h) + 1u;
    a.box_w = p.box_w, a.box_h = p.box_h, a.xoff = p.xoff, a.in_bytes = p.in_bytes, a.ks = p.ks;
    a.fill = e.is_uint8 ? ((uint32_t)(e.in_zero & 0xff) * 0x01010101u) : 0u;
    const int mode = !e.fast_ok ? 2 : ((!e.is_uint8 && e.fuse_bias) ? 1 : 0);
    CUtensorMap tm;
    memcpy(&tm, p.tmap_in, sizeof tm);
    // Several resident CTAs per SM overlap gather / MMA / epilogue of different tiles; each loops over its share.  The grid is
    // exactly the CTAs that can be resident at once (registers and shared memory): a larger one leaves a tail of late CTAs.
#define TB200_WIN_CASE(MD, U, LY)                                                                                                           \
    if (mode == MD && (e.is_uint8 != 0) == U && p.layout == LY)                                                                             \
    {                                                                                                                                       \
        /* the opt-in is per device AND per context: set it before every launch (launches happen at graph capture only) */ \
        cudaError_t err = cudaFuncSetAttribute(conv_window_tc_kernel<MD, U, LY>, cudaFuncAttributeMaxDynamicSharedMemorySize, WINDOW_SMEM_MAX); \
        if (err != cudaSuccess) return err;                                                                                                 \
        int per_sm = 0;                                                                                                                     \
        err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, conv_window_tc_kernel<MD, U, LY>, 128, (size_t)p.smem_bytes);          \
        if (err != cudaSuccess) return err;                                                                                                 \
        const unsigned cap = (unsigned)num_sms * (unsigned)(per_sm > 1 ? per_sm : 1), grid = a.ntiles < cap ? a.ntiles : cap;             \
        if (debug_launch()) fprintf(stderr, "tengine_b200: launch conv_window_tc_kernel<MODE=%d,U8=%d,LAYOUT=%d>\n", MD, (int)U, LY);     \
        conv_window_tc_kernel<MD, U, LY><<<grid, 128, (size_t)p.smem_bytes, st>>>(tm, a, e);                                                \
        return cudaGetLastError();                                                                                                          \
    }
#define TB200_WIN_LAYOUTS(MD, U) TB200_WIN_CASE(MD, U, 0) TB200_WIN_CASE(MD, U, 1) TB200_WIN_CASE(MD, U, 2) TB200_WIN_CASE(MD, U, 3)
    TB200_WIN_LAYOUTS(0, false) TB200_WIN_LAYOUTS(1, false) TB200_WIN_LAYOUTS(2, false) TB200_WIN_LAYOUTS(0, true) TB200_WIN_LAYOUTS(2, true)
#undef TB200_WIN_LAYOUTS
#undef TB200_WIN_CASE
    return cudaErrorInvalidValue;
}

// ---- gather convolution on the tensor cores (NCHW stems, 3x3 convolutions over 16-channel NHWC tensors) ----------------
// The window kernel's layers when it has no plan: NCHW inputs whose width is not a multiple of 16 (a tensor map's global
// strides must be), windows too large for shared memory.  Same skeleton, without the staged window:
// every thread gathers the K bytes of its output pixel itself -- NCHW: 27 / 147 byte loads; NHWC16: nine 16-byte loads, one
// per tap -- and writes them as one row of `ks` SW32 K-major k-block tiles; `ks`
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
    stage_b_and_constants<MODE, U8>(a.w, a.ks, a.ocp, sB, sPar, e);

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
            uint32_t v[16], w[4];
            acc_ld16(tb + 4u * c, v);
            tc_unit16<MODE, U8>(v, rowc, sPar + c * 8, c, a.oc, e, w);
            if (valid) *reinterpret_cast<uint4*>(op + c) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        __syncthreads(); // the next tile's gather overwrites the A tiles, its MMAs the accumulator image
    }
}

cudaError_t launch_conv_gather_tc(const void* in, const void* w, void* out, const ConvShape& s, const EpiParams& e, int nhwc16, int num_sms, cudaStream_t st)
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
    const unsigned cap = (unsigned)num_sms * 6u;
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

} // namespace tb200
