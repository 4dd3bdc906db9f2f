// ptx.cuh -- inline-PTX wrappers shared by the TMA / wgmma kernels (mbarrier, cp.async.bulk.tensor, wgmma.*).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tb200 {

// ---- PTX wrappers -------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// try_wait with a suspend-time hint: the hardware parks the thread until the phase completes or ~hint ns elapse, so a
// waiting role does not burn issue slots that the epilogue warps of the same SM sub-partition need.
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity, uint32_t hint_ns = 2000)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(hint_ns)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trap (-> CUDA error), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    if (mbar_try_wait(bar, parity)) return;
    int spins = 0;
    while (!mbar_try_wait(bar, parity))
    {
        if (++spins > 2000000) __trap(); // > ~4 s of suspended waiting
    }
}
__device__ __forceinline__ void tma_load_2d(const void* tmap, uint64_t* bar, void* smem, int c0, int c1)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// ---- warpgroup MMA (wgmma, sm_90a): 64 x 16 x 32 int8 / uint8 products accumulated in s32 registers -------------------
// Accumulator fragment of one m64n16 product (PTX ISA "wgmma .m64nNk32 D matrix"): warp w of the warpgroup holds rows
// 16w..16w+15; lane l holds d[0..1] = (row l/4, cols 2(l%4)+{0,1}), d[2..3] = (row l/4+8, same cols), d[4..7] = the same for
// cols 8 + 2(l%4)+{0,1}.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait()
{
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
#define TB200_WGMMA_N16(NAME, AT, BT)                                                                                           \
    __device__ __forceinline__ void NAME(uint32_t (&d)[8], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)              \
    {                                                                                                                          \
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"                                                      \
                     "wgmma.mma_async.sync.aligned.m64n16k32.s32." AT "." BT " {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}"               \
                     : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])            \
                     : "l"(desc_a), "l"(desc_b), "r"(accumulate)                                                               \
                     : "memory");                                                                                              \
    }
TB200_WGMMA_N16(wgmma_n16_ss, "s8", "s8")
TB200_WGMMA_N16(wgmma_n16_us, "u8", "s8")
TB200_WGMMA_N16(wgmma_n16_su, "s8", "u8")
TB200_WGMMA_N16(wgmma_n16_uu, "u8", "u8")
#undef TB200_WGMMA_N16
// AU / BU: A / B operand unsigned
template <bool AU, bool BU>
__device__ __forceinline__ void wgmma_n16(uint32_t (&d)[8], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    if (AU && BU) wgmma_n16_uu(d, desc_a, desc_b, accumulate);
    else if (AU) wgmma_n16_us(d, desc_a, desc_b, accumulate);
    else if (BU) wgmma_n16_su(d, desc_a, desc_b, accumulate);
    else wgmma_n16_ss(d, desc_a, desc_b, accumulate);
}
// m64nNk32 for N = 16, 32, .., 128: one instruction per 64 rows x N columns, so the A slice is read from shared memory once per
// k-step whatever N is.  The s32 fragment is N/2 registers per thread = N/16 consecutive n16 fragments (above), column chunk c in
// d[8c .. 8c+7].  The operand lists are spelled out per N because an asm string cannot be computed.
#define TB200_WG_REGS_16 "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p"
#define TB200_WG_PRED_16 "setp.ne.b32 p, %10, 0;"
#define TB200_WG_OPS_16 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
#define TB200_WG_REGS_32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p"
#define TB200_WG_PRED_32 "setp.ne.b32 p, %18, 0;"
#define TB200_WG_OPS_32 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
#define TB200_WG_REGS_48 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p"
#define TB200_WG_PRED_48 "setp.ne.b32 p, %26, 0;"
#define TB200_WG_OPS_48 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23])
#define TB200_WG_REGS_64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p"
#define TB200_WG_PRED_64 "setp.ne.b32 p, %34, 0;"
#define TB200_WG_OPS_64 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
#define TB200_WG_REGS_80 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p"
#define TB200_WG_PRED_80 "setp.ne.b32 p, %42, 0;"
#define TB200_WG_OPS_80 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39])
#define TB200_WG_REGS_96 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p"
#define TB200_WG_PRED_96 "setp.ne.b32 p, %50, 0;"
#define TB200_WG_OPS_96 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47])
#define TB200_WG_REGS_112 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p"
#define TB200_WG_PRED_112 "setp.ne.b32 p, %58, 0;"
#define TB200_WG_OPS_112 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55])
#define TB200_WG_REGS_128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p"
#define TB200_WG_PRED_128 "setp.ne.b32 p, %66, 0;"
#define TB200_WG_OPS_128 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
#define TB200_WGMMA_N(N, AT, BT)                                                                                                \
    asm volatile("{\n\t.reg .pred p;\n\t" TB200_WG_PRED_##N "\n\t"                                                                    \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k32.s32." AT "." BT " " TB200_WG_REGS_##N ";\n\t}"                         \
                 : TB200_WG_OPS_##N                                                                                             \
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate)                                                                    \
                 : "memory")
#define TB200_WGMMA_AB(N)                                                                                                      \
    if constexpr (AU && BU) TB200_WGMMA_N(N, "u8", "u8");                                                                     \
    else if constexpr (AU) TB200_WGMMA_N(N, "u8", "s8");                                                                      \
    else if constexpr (BU) TB200_WGMMA_N(N, "s8", "u8");                                                                      \
    else TB200_WGMMA_N(N, "s8", "s8")
// AU / BU: A / B operand unsigned; accumulate = 0 overwrites d (the first k-step of a tile)
template <int N, bool AU, bool BU>
__device__ __forceinline__ void wgmma_m64(uint32_t (&d)[N / 2], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    static_assert(N % 16 == 0 && N >= 16 && N <= 128, "m64nNk32: N = 16, 32, .., 128");
    if constexpr (N == 16) { TB200_WGMMA_AB(16); }
    else if constexpr (N == 32) { TB200_WGMMA_AB(32); }
    else if constexpr (N == 48) { TB200_WGMMA_AB(48); }
    else if constexpr (N == 64) { TB200_WGMMA_AB(64); }
    else if constexpr (N == 80) { TB200_WGMMA_AB(80); }
    else if constexpr (N == 96) { TB200_WGMMA_AB(96); }
    else if constexpr (N == 112) { TB200_WGMMA_AB(112); }
    else { TB200_WGMMA_AB(128); }
}
#undef TB200_WGMMA_AB
#undef TB200_WGMMA_N
// Pins a register between asm statements: reads of an accumulator stay after the wgmma.wait_group that completes it, and writes
// before the wgmma.fence that orders them ahead of the next wgmma.
__device__ __forceinline__ void reg_fence(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }
// Register budget of the executing warpgroup (all four warps execute it): a role gives registers back to the SM's pool or takes them
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void sts_u2(uint32_t addr, uint32_t a, uint32_t b)
{
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ float4 lds_f4(uint32_t addr)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ float2 lds_f2(uint32_t addr)
{
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint4 lds_u4(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_u4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d)
{
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void sts_f2(uint32_t addr, float2 v)
{
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}

// ---- accumulator image: the s32 accumulators of a 128-row tile as [row][pitch bytes] in shared memory --------------------
// The MMA warpgroups write their fragments here; the epilogues read one row per thread, 16 consecutive columns at a time.
__device__ __forceinline__ void frag_to_image(const uint32_t (&d)[8], uint32_t img, uint32_t pitch, int row0, int col0)
{
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const uint32_t r = (uint32_t)(row0 + 16 * w + (lane >> 2)), c = (uint32_t)(col0 + 2 * (lane & 3));
    const uint32_t p0 = img + r * pitch + c * 4u, p1 = p0 + 8u * pitch;
    sts_u2(p0, d[0], d[1]);
    sts_u2(p1, d[2], d[3]);
    sts_u2(p0 + 32u, d[4], d[5]);
    sts_u2(p1 + 32u, d[6], d[7]);
}
__device__ __forceinline__ void acc_ld16(uint32_t addr, uint32_t (&v)[16])
{
#pragma unroll
    for (int j = 0; j < 4; j++)
    {
        const uint4 u = lds_u4(addr + 16u * j);
        v[4 * j] = u.x, v[4 * j + 1] = u.y, v[4 * j + 2] = u.z, v[4 * j + 3] = u.w;
    }
}

__device__ __forceinline__ void tma_load_4d(const void* tmap, uint64_t* bar, void* smem, int c0, int c1, int c2, int c3)
{
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
            smem_u32(smem)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---- TMA stores (shared -> global through a tensor map; rows outside the tensor are clipped by the TMA unit) ----
__device__ __forceinline__ void tma_store_3d(const void* tmap, uint32_t smem_addr, int c0, int c1, int c2)
{
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(reinterpret_cast<uint64_t>(tmap)),
                 "r"(smem_addr), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's bulk groups still READ their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read()
{
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait()
{
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (TMA) that reads them next
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// host: cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
int tmap_encode(void* tmap, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                const uint32_t* elem_strides, int swizzle_bytes);

} // namespace tb200
