// classify_topk.cu -- the last step of the classification examples on the device: dequantise the graph's output tensor where it
// lies in HBM and rank its classes, so that k (score, id) pairs per image travel to the host instead of every class byte.
//
// Restates the application code of examples/tm_classification_int8.c:163-166 and examples/tm_classification_uint8.c:169-172
// (dequantisation, then print_topk(output_data, output_size, 5)) and of examples/common/tengine_operations.c: print_topk
// (:1021-1038; id = position in the NCHW buffer) and sort_cls_score (:991-1019), a first-element-pivot quicksort whose scans pass
// over scores equal to the pivot.  It is unstable, and a quantised output is mostly ties, so its tie order is part of the result:
// the sort is replayed, not replaced.  One CTA per image.
//
// Two things make the replay cheap without changing one move of it:
//  - Pruning.  After a partition the two sub-ranges are sorted independently and only positions < k are reported, so a sub-range
//    that starts at or beyond k is never looked at.  The left sub-range is continued with at once; a pending right-hand one starts
//    below k and pending ranges are disjoint, so a stack of k entries holds them.
//  - Parallel scans.  Each inner loop of sort_cls_score walks to the nearest element where a fixed comparison against the pivot's
//    score fails.  One warp tests 32 positions per step and takes the nearest failing lane (__ballot_sync); the moves between the
//    scans are made in the example's order.
// All comparisons are the example's own operators on the dequantised floats, so zero, negative and overflowing scales behave as they do
// there.  A NaN score would stop both scans where they stand, in the example as here, for ever: callers refuse a non-finite scale.
#include "common.cuh"
#include "kernels.h"

namespace tb200 {

// Shared memory of one image: float score[E], uint16_t id[E] (ids fit: E <= CLASS_TOPK_MAX_CLASSES = 32768), then int2 pending[k].
// At the largest E and k that is 197120 of the 232448 bytes a CTA may have on sm_90.
__host__ __device__ static inline size_t class_topk_pending_offset(int e) { return ((size_t)e * 6 + 7) & ~(size_t)7; }
static inline size_t class_topk_smem(int e, int k) { return class_topk_pending_offset(e) + (size_t)k * sizeof(int2); }

template <bool U8>
__global__ void __launch_bounds__(128) class_topk_kernel(const uint8_t* __restrict__ in, int C, int cp, int HW, float scale, float zero, int k,
                                                         ClassScore* __restrict__ out)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int E = C * HW;
    float* s_score = reinterpret_cast<float*>(smem);
    uint16_t* s_id = reinterpret_cast<uint16_t*>(s_score + E);
    int2* s_pending = reinterpret_cast<int2*>(smem + class_topk_pending_offset(E));

    // (1) the image's bytes in device order (pixel-major, cp bytes per pixel: coalesced), each to its NCHW position
    const uint8_t* img = in + (size_t)blockIdx.x * HW * cp;
    for (int e = threadIdx.x; e < HW * cp; e += blockDim.x)
    {
        const int hw = e / cp, c = e - hw * cp;
        if (c >= C) continue; // pad lanes
        const int id = c * HW + hw;
        const uint8_t b = __ldg(img + e);
        const float q = U8 ? (float)b : (float)(int)(int8_t)b;
        s_score[id] = __fmul_rn(U8 ? __fsub_rn(q, zero) : q, scale);
        s_id[id] = (uint16_t)id;
    }
    __syncthreads();

    // (2) sort_cls_score(array, 0, E - 1) by warp 0; every lane holds the same i, j, left, right, key
    if (threadIdx.x < 32)
    {
        const int lane = threadIdx.x;
        int sp = 0, i = 0, j = E - 1;
        for (;;)
        {
            if (i >= j) // `if (left >= right) return;`
            {
                if (sp == 0) break;
                const int2 r = s_pending[--sp];
                i = r.x, j = r.y;
                continue;
            }
            int left = i, right = j;
            const float key = s_score[left];
            const uint16_t key_id = s_id[left];
            while (left < right)
            {
                // while (left < right && key.score >= array[right].score) --right;
                while (left < right)
                {
                    const int p = right - lane;
                    const unsigned stop = __ballot_sync(0xffffffffu, p > left && !(key >= s_score[p]));
                    if (stop)
                    {
                        right -= __ffs(stop) - 1;
                        break;
                    }
                    right = max(left, right - 32);
                }
                if (lane == 0) s_score[left] = s_score[right], s_id[left] = s_id[right];
                __syncwarp();
                // while (left < right && key.score <= array[left].score) ++left;
                while (left < right)
                {
                    const int p = left + lane;
                    const unsigned stop = __ballot_sync(0xffffffffu, p < right && !(key <= s_score[p]));
                    if (stop)
                    {
                        left += __ffs(stop) - 1;
                        break;
                    }
                    left = min(right, left + 32);
                }
                if (lane == 0) s_score[right] = s_score[left], s_id[right] = s_id[left];
                __syncwarp();
            }
            if (lane == 0) s_score[left] = key, s_id[left] = key_id;
            // sort_cls_score(array, left + 1, j) later, if it reaches a reported position; sort_cls_score(array, i, left - 1) now
            if (left + 1 < k && left + 1 < j)
            {
                if (lane == 0) s_pending[sp] = make_int2(left + 1, j);
                sp++;
            }
            __syncwarp();
            j = left - 1;
        }
    }
    __syncthreads();

    // (3) entries 0..k-1 of the sorted array
    for (int r = threadIdx.x; r < k; r += blockDim.x)
    {
        ClassScore o;
        o.score = s_score[r], o.id = (int)s_id[r];
        out[(size_t)blockIdx.x * k + r] = o;
    }
}

cudaError_t launch_class_topk(const void* in, int n, int c, int h, int w, bool u8, float scale, int zero_point, int k, ClassScore* out, cudaStream_t st)
{
    const long long e = (long long)c * h * w;
    if (n < 1 || c < 1 || h < 1 || w < 1 || e > CLASS_TOPK_MAX_CLASSES || k < 1 || k > CLASS_TOPK_MAX_K || k > e) return cudaErrorInvalidValue;
    const size_t smem = class_topk_smem((int)e, k);
    auto kern = u8 ? class_topk_kernel<true> : class_topk_kernel<false>;
    if (smem > 48 * 1024)
    {
        // the opt-in is per device and per context: set it before every such launch
        const cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)class_topk_smem(CLASS_TOPK_MAX_CLASSES, CLASS_TOPK_MAX_K));
        if (err != cudaSuccess) return err;
    }
    kern<<<(unsigned)n, 128, smem, st>>>((const uint8_t*)in, c, cpad(c), h * w, scale, (float)zero_point, k, out);
    return cudaGetLastError();
}

} // namespace tb200
