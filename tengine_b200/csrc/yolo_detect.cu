// yolo_detect.cu -- detection post-processing on the device (SURVEY.md 8(f)-4): YOLO region decode, score threshold, sort by
// score and greedy NMS, straight from the graph's quantised output tensors in HBM.  Only the kept boxes travel to the host
// (YOLOv3-tiny at batch 128: 27.6 MB of raw head tensors stay on the GPU; YOLOv5s at batch 64 and 640x640: 137 MB).
//
// Restates the application code of examples/tm_yolov3_tiny_uint8.cpp: dequantisation (:464-478), generate_proposals (:176-250),
// qsort_descent_inplace (:57-100), nms_sorted_bboxes (:102-132); and of examples/tm_yolov5s.cpp, whose generate_proposals
// (:140-207) differs only in the box formula (the sort and NMS are the same functions).  Every per-element function of a byte
// there -- sigmoid, exp -- is a 256-entry table built on the host with the same float arithmetic (engine.cu build_yolo_tables), so
// the device only looks up and multiplies; sorting and NMS replay the example's algorithms literally (including its quicksort's tie
// order), one CTA per image.
#include "common.cuh"
#include "kernels.h"

namespace tb200 {

// ---- decode: a group of S lanes per cell (S = the power of two >= cp / 16, at most 32) ----------------------------------------------
// The cell's NHWC row of cp bytes is read with 16-byte loads, lane j of the group taking chunks j, j + S, ...; the 32 / S cells of a
// warp are adjacent rows, so a warp's loads are contiguous.  Before that, every lane reads the three objectness bytes of its cell:
// sigmoid(class) <= 1 makes sigmoid(obj) * sigmoid(class) <= sigmoid(obj) in float, so an anchor whose sigmoid(obj) is below the
// threshold cannot produce a proposal and its class bytes are not read at all.  The class arg-max of each live anchor is a lane-local
// maximum of the key (byte << 24 | 0xFFFFFF - class) followed by a shuffle reduction over the group: the larger byte wins and, among
// equal bytes, the lower class index -- the first maximum of the example's strict `score > class_score` scan (dequantisation is
// increasing in the byte).  Lane (anchor mod S) of the group then forms that anchor's box.
template <YoloBox F>
__global__ void __launch_bounds__(256) yolo_decode_kernel(const uint8_t* __restrict__ t, int cp, int H, int W, long long cells, int classes, int S,
                                                          const float* __restrict__ sig,  // [256]: sigmoid(dequantised byte), as a float
                                                          const double* __restrict__ ex,  // [256] (V3): the example's float exp(dequantised byte), as a double
                                                          float stride, float a0w, float a0h, float a1w, float a1h, float a2w, float a2h, float thr,
                                                          YoloCand* __restrict__ cand, int* __restrict__ count, int max_cand, unsigned key_base, bool is_u8)
{
    const int lane = threadIdx.x & 31, j = lane & (S - 1);
    const long long cell = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (32 / S) + lane / S;
    const bool valid = cell < cells;
    const uint8_t* row = t + (size_t)(valid ? cell : 0) * cp;
    const int per = classes + 5;
    bool live[3];
#pragma unroll
    for (int a = 0; a < 3; a++) live[a] = valid && sig[__ldg(row + a * per + 4)] >= thr;
    const unsigned flip = is_u8 ? 0u : 0x80808080u; // int8 bytes compare as unsigned after flipping the sign bit
    unsigned key[3] = {0, 0, 0};
    if (live[0] || live[1] || live[2])
    {
        for (int k = j; k * 16 < cp; k += S)
        {
            int lo[3], hi[3]; // class bytes of anchor a inside this chunk: [lo, hi)
            bool need = false;
#pragma unroll
            for (int a = 0; a < 3; a++)
            {
                lo[a] = max(a * per + 5 - k * 16, 0), hi[a] = min(a * per + per - k * 16, 16);
                need |= live[a] && lo[a] < hi[a];
            }
            if (!need) continue;
            const uint4 q = __ldg(reinterpret_cast<const uint4*>(row) + k);
            const unsigned wd[4] = {q.x ^ flip, q.y ^ flip, q.z ^ flip, q.w ^ flip};
#pragma unroll
            for (int a = 0; a < 3; a++)
            {
                if (!(live[a] && lo[a] < hi[a])) continue;
                const unsigned cb = 0xFFFFFFu - (unsigned)(k * 16 - a * per - 5); // 0xFFFFFF - class of byte i is cb - i
                unsigned m = key[a];
#pragma unroll
                for (int i = 0; i < 16; i++)
                    if (i >= lo[a] && i < hi[a]) m = max(m, ((wd[i >> 2] >> (8 * (i & 3))) << 24) | (cb - i));
                key[a] = m;
            }
        }
    }
#pragma unroll
    for (int a = 0; a < 3; a++)
        for (int off = S >> 1; off > 0; off >>= 1) key[a] = max(key[a], __shfl_xor_sync(0xffffffffu, key[a], off));
    const int hw = (int)(valid ? cell % ((long long)H * W) : 0), n = (int)(valid ? cell / ((long long)H * W) : 0);
    const int h = hw / W, w = hw % W;
#pragma unroll
    for (int a = 0; a < 3; a++)
    {
        if ((a & (S - 1)) != j || !live[a]) continue;
        const int best = 0xFFFFFF - (int)(key[a] & 0xFFFFFFu);
        const uint8_t* p = row + a * per;
        const float final_score = __fmul_rn(sig[__ldg(p + 4)], sig[(key[a] >> 24) ^ (flip & 0xFFu)]);
        if (!(final_score >= thr)) continue;
        const float dx = sig[__ldg(p + 0)], dy = sig[__ldg(p + 1)];
        const float aw = a == 0 ? a0w : (a == 1 ? a1w : a2w), ah = a == 0 ? a0h : (a == 1 ? a1h : a2h);
        float x0, y0, x1, y1;
        if (F == YoloBox::V3)
        {
            // tm_yolov3_tiny_uint8.cpp:226-236.  `float pred_w = exp(dw) * anchor_w;` is a float product (exp resolves to the float
            // overload there): the double product of two float values is exact, so narrowing it rounds once, exactly like the float multiply
            const float pred_x = __fmul_rn(__fadd_rn((float)w, dx), stride), pred_y = __fmul_rn(__fadd_rn((float)h, dy), stride);
            const float pred_w = (float)__dmul_rn(ex[__ldg(p + 2)], (double)aw), pred_h = (float)__dmul_rn(ex[__ldg(p + 3)], (double)ah);
            x0 = __fsub_rn(pred_x, __fmul_rn(pred_w, 0.5f)), y0 = __fsub_rn(pred_y, __fmul_rn(pred_h, 0.5f));
            x1 = __fadd_rn(pred_x, __fmul_rn(pred_w, 0.5f)), y1 = __fadd_rn(pred_y, __fmul_rn(pred_h, 0.5f));
        }
        else
        {
            // tm_yolov5s.cpp:180-193: (dx * 2.0f - 0.5f + w) * stride and dw * dw * 4.0f * anchor_w, left to right in float
            const float dw = sig[__ldg(p + 2)], dh = sig[__ldg(p + 3)];
            const float pred_cx = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(dx, 2.0f), 0.5f), (float)w), stride);
            const float pred_cy = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(dy, 2.0f), 0.5f), (float)h), stride);
            const float pred_w = __fmul_rn(__fmul_rn(__fmul_rn(dw, dw), 4.0f), aw), pred_h = __fmul_rn(__fmul_rn(__fmul_rn(dh, dh), 4.0f), ah);
            x0 = __fsub_rn(pred_cx, __fmul_rn(pred_w, 0.5f)), y0 = __fsub_rn(pred_cy, __fmul_rn(pred_h, 0.5f));
            x1 = __fadd_rn(pred_cx, __fmul_rn(pred_w, 0.5f)), y1 = __fadd_rn(pred_cy, __fmul_rn(pred_h, 0.5f));
        }
        const int slot = atomicAdd(count + n, 1);
        if (slot >= max_cand) continue; // counted, reported as overflow by the host
        YoloCand c;
        c.x = x0, c.y = y0, c.w = __fsub_rn(x1, x0), c.h = __fsub_rn(y1, y0), c.prob = final_score, c.label = best;
        c.key = key_base + (unsigned)(hw * 3 + a); // position in the reference's proposal list
        cand[(size_t)n * max_cand + slot] = c;
    }
}

// ---- per image: restore the proposal order, the example's quicksort, greedy NMS ---------------------------------------------------
__device__ void yolo_qsort(YoloCand* v, int left, int right)
{
    // qsort_descent_inplace (tm_yolov3_tiny_uint8.cpp:57-92) with an explicit stack (the recursion's two halves are independent)
    int stack[64][2];
    int sp = 0;
    stack[sp][0] = left, stack[sp][1] = right, sp++;
    while (sp > 0)
    {
        sp--;
        const int l = stack[sp][0], r = stack[sp][1];
        int i = l, j = r;
        const float p = v[(l + r) / 2].prob;
        while (i <= j)
        {
            while (v[i].prob > p) i++;
            while (v[j].prob < p) j--;
            if (i <= j)
            {
                const YoloCand tmp = v[i];
                v[i] = v[j], v[j] = tmp;
                i++, j--;
            }
        }
        // push the larger part first so that the stack depth stays logarithmic; the parts are disjoint, so the order they are
        // sorted in does not change the result
        const bool left_ok = l < j, right_ok = i < r;
        if (left_ok && right_ok)
        {
            if (j - l > r - i)
                stack[sp][0] = l, stack[sp][1] = j, sp++, stack[sp][0] = i, stack[sp][1] = r, sp++;
            else
                stack[sp][0] = i, stack[sp][1] = r, sp++, stack[sp][0] = l, stack[sp][1] = j, sp++;
        }
        else if (left_ok)
            stack[sp][0] = l, stack[sp][1] = j, sp++;
        else if (right_ok)
            stack[sp][0] = i, stack[sp][1] = r, sp++;
    }
}

__global__ void __launch_bounds__(256) yolo_nms_kernel(const YoloCand* __restrict__ cand, const int* __restrict__ count, int max_cand, float nms_thr,
                                                       YoloCand* __restrict__ sorted, // scratch [n_img][max_cand]
                                                       YoloDet* __restrict__ out, int max_out, int* __restrict__ out_count)
{
    const int n = blockIdx.x;
    int m = count[n];
    __shared__ int s_picked[1024];
    __shared__ int s_np, s_keep;
    if (m > max_cand)
    {
        if (threadIdx.x == 0) out_count[n] = -m; // overflow: the caller must raise max_candidates
        return;
    }
    const YoloCand* src = cand + (size_t)n * max_cand;
    YoloCand* v = sorted + (size_t)n * max_cand;
    // (1) proposal order of the reference = ascending key (keys are unique): rank sort
    for (int i = threadIdx.x; i < m; i += blockDim.x)
    {
        const unsigned k = src[i].key;
        int rank = 0;
        for (int j = 0; j < m; j++) rank += src[j].key < k;
        v[rank] = src[i];
    }
    __syncthreads();
    // (2) the example's quicksort by score, literally (one thread: its tie order is part of the result)
    if (threadIdx.x == 0)
    {
        if (m > 0) yolo_qsort(v, 0, m - 1);
        s_np = 0;
    }
    __syncthreads();
    // (3) nms_sorted_bboxes (:102-132): candidate i is kept unless its IoU with an already kept box exceeds the threshold
    for (int i = 0; i < m; i++)
    {
        if (threadIdx.x == 0) s_keep = 1;
        __syncthreads();
        const YoloCand a = v[i];
        const float area_a = __fmul_rn(a.w, a.h);
        const int np = s_np;
        for (int j = threadIdx.x; j < np; j += blockDim.x)
        {
            const YoloCand b = v[s_picked[j]];
            // cv::Rect_<float> operator& and area()
            const float x1 = fmaxf(a.x, b.x), y1 = fmaxf(a.y, b.y);
            const float iw = __fsub_rn(fminf(__fadd_rn(a.x, a.w), __fadd_rn(b.x, b.w)), x1), ih = __fsub_rn(fminf(__fadd_rn(a.y, a.h), __fadd_rn(b.y, b.h)), y1);
            const float inter = (iw <= 0.f || ih <= 0.f) ? 0.f : __fmul_rn(iw, ih);
            const float uni = __fsub_rn(__fadd_rn(area_a, __fmul_rn(b.w, b.h)), inter);
            if (__fdiv_rn(inter, uni) > nms_thr) s_keep = 0;
        }
        __syncthreads();
        if (threadIdx.x == 0 && s_keep)
        {
            if (s_np < 1024) s_picked[s_np] = i;
            s_np++;
        }
        __syncthreads();
        if (s_np > 1024) break; // more kept boxes than the list holds: reported below
    }
    __syncthreads();
    const int np = s_np;
    if (threadIdx.x == 0) out_count[n] = (np > 1024 || np > max_out) ? -np : np;
    for (int j = threadIdx.x; j < np && j < max_out && j < 1024; j += blockDim.x)
    {
        const YoloCand c = v[s_picked[j]];
        YoloDet d;
        d.x = c.x, d.y = c.y, d.w = c.w, d.h = c.h, d.prob = c.prob, d.label = c.label;
        out[(size_t)n * max_out + j] = d;
    }
}

cudaError_t launch_yolo_decode(YoloBox f, const void* tensor, int cp, int h, int w, int n_img, int classes, const float* sig, const double* ex, float stride,
                               const float* anchors6, float thr, YoloCand* cand, int* count, int max_cand, unsigned key_base, bool is_u8, cudaStream_t st)
{
    const long long cells = (long long)n_img * h * w;
    // cp: a multiple of 16 holding 3 x (5 + classes) channels; the arg-max key holds a class index in 24 bits
    if (cells <= 0 || cp % 16 != 0 || classes < 1 || classes > 0xFFFFFF || 3 * (classes + 5) > cp || (size_t)tensor % 16 != 0) return cudaErrorInvalidValue;
    int S = 1;
    while (S < 32 && S * 16 < cp) S *= 2;
    const long long warps = (cells + 32 / S - 1) / (32 / S), blocks = (warps + 7) / 8;
    if (blocks >= (1ll << 31)) return cudaErrorInvalidValue;
    auto kern = f == YoloBox::V3 ? yolo_decode_kernel<YoloBox::V3> : yolo_decode_kernel<YoloBox::V5>;
    kern<<<(unsigned)blocks, 256, 0, st>>>((const uint8_t*)tensor, cp, h, w, cells, classes, S, sig, ex, stride, anchors6[0], anchors6[1], anchors6[2], anchors6[3],
                                           anchors6[4], anchors6[5], thr, cand, count, max_cand, key_base, is_u8);
    return cudaGetLastError();
}

cudaError_t launch_yolo_nms(const YoloCand* cand, const int* count, int n_img, int max_cand, float nms_thr, YoloCand* sorted, YoloDet* out, int max_out,
                            int* out_count, cudaStream_t st)
{
    yolo_nms_kernel<<<n_img, 256, 0, st>>>(cand, count, max_cand, nms_thr, sorted, out, max_out, out_count);
    return cudaGetLastError();
}

} // namespace tb200
