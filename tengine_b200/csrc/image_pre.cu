// image_pre.cu -- classification preprocessing on the device: decoded 8-bit images (HWC, RGB or RGBA, what stbi_load returns) to
// the quantised NCHW bytes of a graph input, for a whole batch in one launch.
//
// Restates the application code of examples/tm_classification_int8.c / _uint8.c (get_input_int8_data / get_input_uint8_data,
// :43-62) and what they call in examples/common/tengine_operations.c: load_image_stb (:51-82, the alpha byte of RGBA is skipped),
// rgb2bgr_permute (:651-673, output plane k is source channel 2 - k), tengine_resize_f32 (:870-979, the non-NEON branch) and
// imread2caffe (:101-115).  Each output pixel's resize coefficients are computed where they are used, with the example's float
// arithmetic spelled out in round-to-nearest intrinsics (the example is compiled without FMA contraction), so images of any size can
// share a batch and no host tables exist.
#include "common.cuh"
#include "kernels.h"
#include "preproc.cuh"

namespace tb200 {

// Position and 11-bit weights of output coordinate i along an axis of `in` source pixels scaled by `scale` (tengine_resize_f32
// :882-900): truncation toward zero leaves s = 0 with a negative f in the first outputs of an upsample (the weights then
// extrapolate), and the last output always takes s = in - 2 with weight 1 on it.  The int16_t stores of the example truncate.
__device__ __forceinline__ void resize_coef(int i, int in, float scale, int& s, int& c0, int& c1)
{
    float f = __fsub_rn(__fmul_rn(__fadd_rn((float)i, 0.5f), scale), 0.5f);
    s = (int)f;
    f = __fsub_rn(f, (float)s);
    if (s < 0) s = 0, f = 0.f;
    if (s >= in - 1) s = in - 2, f = 0.f;
    c1 = (int)(int16_t)(int)__fmul_rn(f, 2048.f);
    c0 = (int)(int16_t)(int)__fmul_rn(__fsub_rn(1.f, f), 2048.f);
}

// One CTA per output row (image n, row y); its threads walk the row's pixels and write the three planes' bytes, coalesced along x.
template <bool U8>
__global__ void __launch_bounds__(128) image_pre_kernel(const uint8_t* __restrict__ pixels, const ImageDesc* __restrict__ images, uint8_t* __restrict__ out,
                                                        int H, int W, float m0, float m1, float m2, float s0, float s1, float s2, float s_in, int zp)
{
    const int n = blockIdx.x / H, y = blockIdx.x - n * H;
    const ImageDesc d = images[n];
    const uint8_t* src = pixels + d.offset;
    int sy, cy0, cy1;
    resize_coef(y, d.h, __fdiv_rn((float)d.h, (float)H), sy, cy0, cy1);
    const float scale_x = __fdiv_rn((float)d.w, (float)W);
    const size_t row = (size_t)d.w * d.c;
    const uint8_t* r0 = src + (size_t)sy * row;
    const uint8_t* r1 = r0 + row;
    const float mean[3] = {m0, m1, m2}, scl[3] = {s0, s1, s2};
    const size_t plane = (size_t)H * W;
    uint8_t* o = out + (size_t)n * 3 * plane + (size_t)y * W;
    for (int x = threadIdx.x; x < W; x += blockDim.x)
    {
        int sx, cx0, cx1;
        resize_coef(x, d.w, scale_x, sx, cx0, cx1);
        const int a = sx * d.c, b = a + d.c;
#pragma unroll
        for (int k = 0; k < 3; k++)
        {
            const int ch = 2 - k; // BGR planes from RGB(A) bytes
            const int u = ((int)r0[a + ch] * cx0 >> 11) + ((int)r0[b + ch] * cx1 >> 11);
            const int dn = ((int)r1[a + ch] * cx0 >> 11) + ((int)r1[b + ch] * cx1 >> 11);
            const int v = (u * cy0 + dn * cy1) >> 11;
            const float f = __fmul_rn(__fsub_rn((float)v, mean[k]), scl[k]);
            int q;
            if (U8)
            {
                q = round_to_int_x86(__fadd_rn(__fdiv_rn(f, s_in), (float)zp));
                q = q > 255 ? 255 : (q < 0 ? 0 : q);
            }
            else
            {
                q = round_to_int_x86(__fdiv_rn(f, s_in));
                q = q > 127 ? 127 : (q < -127 ? -127 : q);
            }
            o[k * plane + x] = (uint8_t)q;
        }
    }
}

cudaError_t launch_image_pre(const uint8_t* pixels, const ImageDesc* images, int n, uint8_t* out, int H, int W, const float mean[3], const float scale[3],
                             float s_in, int zp, bool u8, cudaStream_t st)
{
    const unsigned rows = (unsigned)n * (unsigned)H;
    if (u8)
        image_pre_kernel<true><<<rows, 128, 0, st>>>(pixels, images, out, H, W, mean[0], mean[1], mean[2], scale[0], scale[1], scale[2], s_in, zp);
    else
        image_pre_kernel<false><<<rows, 128, 0, st>>>(pixels, images, out, H, W, mean[0], mean[1], mean[2], scale[0], scale[1], scale[2], s_in, zp);
    return cudaGetLastError();
}

} // namespace tb200
