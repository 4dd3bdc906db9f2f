// detect_pre.cu -- detection preprocessing on the device: decoded 8-bit images (HWC, RGB or RGBA) to the quantised input of a YOLO
// graph, stretched or letterboxed, with or without the Focus slicing, for a whole batch in one launch.
//
// Restates the application code of examples/tm_yolov3_tiny_uint8.cpp:136-170 (stretch) and examples/tm_yolov5s.cpp:263-337 / :339-392
// (letterbox, Focus / no Focus), quantised as tm_yolox_int8.cpp:336-341 / tm_yolov3_tiny_uint8.cpp:164-168, with OpenCV's cv::resize
// (INTER_LINEAR, 8-bit) and cv::copyMakeBorder (constant byte 0) in between; include/tengine_b200.h states the arithmetic.  The host
// computes each image's geometry (resized size, left / top border) with the example's own float arithmetic; every pixel's resize
// positions and weights are computed here, where they are used, with the double arithmetic spelled out in round-to-nearest intrinsics
// so that nothing is contracted into an FMA.
#include "common.cuh"
#include "kernels.h"
#include "preproc.cuh"

namespace tb200 {

// Source index and 11-bit weights of output coordinate d along an axis of `src` pixels resized to `dst` (OpenCV resize.cpp, fixed-point
// INTER_LINEAR): scale = 1. / ((double)dst / src), fx = (float)((d + 0.5) * scale - 0.5), cvFloor, weights saturate_cast<short>(w * 2048)
// (round half to even).  `clamp` (the horizontal axis): a position before the first pixel or at / after the last takes that pixel with
// weight 1.  The vertical axis is not clamped; its caller clips the two row indices instead.
__device__ __forceinline__ void cv_linear_coef(int d, double scale, int src, bool clamp, int& s, int& c0, int& c1)
{
    float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
    s = __float2int_rd(f);
    f = __fsub_rn(f, (float)s);
    if (clamp)
    {
        if (s < 0) s = 0, f = 0.f;
        if (s >= src - 1) s = src - 1, f = 0.f;
    }
    c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
    c1 = __float2int_rn(__fmul_rn(f, 2048.f));
}

__device__ __forceinline__ double cv_inv_scale(int dst, int src) { return __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src)); }

// One CTA per row y of image n's H x W laid-out image.  Threads walk the row; with Focus, thread j takes column 2j (j < W/2) or
// 2(j - W/2) + 1, so a warp writes consecutive bytes of one output plane.
template <bool U8, bool FOCUS>
__global__ void __launch_bounds__(128) detect_pre_kernel(const uint8_t* __restrict__ pixels, const ImageDesc* __restrict__ images, uint8_t* __restrict__ out,
                                                         int H, int W, float m0, float m1, float m2, float s0, float s1, float s2, float s_in, int zp)
{
    const int n = blockIdx.x / H, y = blockIdx.x - n * H;
    const ImageDesc d = images[n];
    const float mean[3] = {m0, m1, m2}, scl[3] = {s0, s1, s2};
    const size_t plane = FOCUS ? (size_t)(H / 2) * (W / 2) : (size_t)H * W;
    uint8_t* o = out + (size_t)n * (FOCUS ? 12 : 3) * plane;
    o += FOCUS ? (size_t)(y & 1) * 3 * plane + (size_t)(y >> 1) * (W / 2) : (size_t)y * W; // Focus: row offset g = y & 1
    // the vertical pass: two clipped source rows and their weights, or a border row
    const int ry = y - d.top;
    const bool row_in = ry >= 0 && ry < d.resize_h;
    const size_t pitch = (size_t)d.w * d.c;
    const uint8_t *r0 = pixels + d.offset, *r1 = r0;
    int cy0 = 0, cy1 = 0;
    if (row_in)
    {
        int sy;
        cv_linear_coef(ry, cv_inv_scale(d.resize_h, d.h), d.h, false, sy, cy0, cy1);
        r0 += (size_t)min(max(sy, 0), d.h - 1) * pitch;
        r1 += (size_t)min(max(sy + 1, 0), d.h - 1) * pitch;
    }
    const double scale_x = cv_inv_scale(d.resize_w, d.w);
    for (int j = threadIdx.x; j < W; j += blockDim.x)
    {
        int x = j, oofs = j;
        if (FOCUS)
        {
            const int i = j >= W / 2, xo = j - i * (W / 2); // column offset i
            x = 2 * xo + i, oofs = i * 6 * (int)plane + xo;
        }
        int v[3] = {0, 0, 0}; // the border: byte 0
        const int rx = x - d.left;
        if (row_in && rx >= 0 && rx < d.resize_w)
        {
            int sx, cx0, cx1;
            cv_linear_coef(rx, scale_x, d.w, true, sx, cx0, cx1);
            const int a = sx * d.c, b = min(sx + 1, d.w - 1) * d.c;
#pragma unroll
            for (int k = 0; k < 3; k++)
            {
                const int h0 = (int)r0[a + k] * cx0 + (int)r0[b + k] * cx1;
                const int h1 = (int)r1[a + k] * cx0 + (int)r1[b + k] * cx1;
                // OpenCV's SIMD vertical pass: mulhi of 16-bit (S >> 4) by the weight, twice, then a rounding shift by 2
                const int t = ((((cy0 * (h0 >> 4)) >> 16) + ((cy1 * (h1 >> 4)) >> 16) + 2) >> 2);
                v[k] = t > 255 ? 255 : t;
            }
        }
#pragma unroll
        for (int k = 0; k < 3; k++)
        {
            const float f = __fmul_rn(__fsub_rn((float)v[k], mean[k]), scl[k]);
            int q = round_to_int_x86(__fadd_rn(__fdiv_rn(f, s_in), (float)zp));
            if (U8)
                q = q > 255 ? 255 : (q < 0 ? 0 : q);
            else
                q = q > 127 ? 127 : (q < -127 ? -127 : q);
            o[k * plane + oofs] = (uint8_t)q;
        }
    }
}

template <bool U8, bool FOCUS>
static void launch(unsigned rows, const uint8_t* pixels, const ImageDesc* images, uint8_t* out, int H, int W, const float* mean, const float* scale, float s_in,
                   int zp, cudaStream_t st)
{
    detect_pre_kernel<U8, FOCUS><<<rows, 128, 0, st>>>(pixels, images, out, H, W, mean[0], mean[1], mean[2], scale[0], scale[1], scale[2], s_in, zp);
}

cudaError_t launch_detect_pre(const uint8_t* pixels, const ImageDesc* images, int n, uint8_t* out, int H, int W, bool focus, const float mean[3],
                              const float scale[3], float s_in, int zp, bool u8, cudaStream_t st)
{
    const unsigned rows = (unsigned)n * (unsigned)H;
    if (u8)
        (focus ? launch<true, true> : launch<true, false>)(rows, pixels, images, out, H, W, mean, scale, s_in, zp, st);
    else
        (focus ? launch<false, true> : launch<false, false>)(rows, pixels, images, out, H, W, mean, scale, s_in, zp, st);
    return cudaGetLastError();
}

} // namespace tb200
