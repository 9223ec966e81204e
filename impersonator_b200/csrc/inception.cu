// InceptionV3 features of his_evaluators' unpaired metrics (metrics/metrics.py:16-158, 634-781): the input transform
// and the segmented eval-mode BatchNorm + ReLU epilogue behind the conv engine.  The convolutions themselves run on the
// conv engine (lwb_conv_plan_*) and the stem on lwb_conv2d_direct_relu_nhwc; the pools are lwb_maxpool_nhwc(_slice) and
// lwb_global_avgpool_nhwc.  No reduction here depends on scheduling, so the features repeat bit for bit.
#include "common.cuh"
#include "operands.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int SIDE = 299;                                           // InceptionScoreMetric / FIDMetric height, width

// preprocess (metrics.py:645-669, 715-740): x * 2 - 1 in float32, then F.interpolate(size=(299, 299), mode='bilinear',
// align_corners=False) in float32 as torch computes it: scale = in / out, src = max(scale * (dst + 0.5) - 0.5, 0),
// the upper neighbour clamped to the last row / column.  NCHW [n,3,h,w] -> NCHW [n,3,299,299].
__global__ void __launch_bounds__(THREADS) k_inception_input(const float* __restrict__ x, int n, int h, int w,
                                                             float* __restrict__ out)
{
    const long total = (long)n * 3 * SIDE * SIDE;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int ox = (int)(i % SIDE), oy = (int)((i / SIDE) % SIDE);
    const long plane = i / ((long)SIDE * SIDE);
    // written as torch's upsample_bilinear2d kernel writes it, so that nvcc contracts the same products into FMAs
    const float rh = (float)h / SIDE, rw = (float)w / SIDE;
    const float sy = fmaxf(rh * (oy + 0.5f) - 0.5f, 0.f);
    const float sx = fmaxf(rw * (ox + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int yp = y0 < h - 1 ? 1 : 0, xp = x0 < w - 1 ? 1 : 0;
    const float ly1 = sy - y0, ly0 = 1.f - ly1;
    const float lx1 = sx - x0, lx0 = 1.f - lx1;
    const float* p = x + plane * h * w;
    auto at = [&](int yy, int xx) { return __fsub_rn(__fmul_rn(__ldg(p + (size_t)yy * w + xx), 2.f), 1.f); };
    out[i] = ly0 * (lx0 * at(y0, x0) + lx1 * at(y0, x0 + xp)) + ly1 * (lx0 * at(y0 + yp, x0) + lx1 * at(y0 + yp, x0 + xp));
}

// One channel segment of a raw NHWC fp32 conv output (pitch ld_raw, channels [c0, c0 + c)):
//   r = raw, or its 3x3 box mean (zero padded, always / 9) when `box`: avg_pool2d(3, 1, 1, count_include_pad=True)
//       followed by a bias-free 1x1 conv equals the 1x1 conv followed by the same pool, so the Inception pool branches
//       share the block's merged 1x1 GEMM;
//   v = relu?(r * scale[ch] + shift[ch])  (the eval-mode BatchNorm affine; identity when scale is null)
// written to channels [off_y, off_y + c_out) of outputs with pitch ld_y: fp32 and / or fp16 hi / lo operands, zeros in
// the c_out - c pad channels (the conv engine reads multiples of 64 channels).
__global__ void __launch_bounds__(THREADS) k_bn_act_segment(const float* __restrict__ raw, int n, int h, int w, int ld_raw,
                                                            int c0, int c, int c_out, int box,
                                                            const float* __restrict__ scale, const float* __restrict__ shift,
                                                            int relu, float* __restrict__ y_f32, __half* __restrict__ y_hi,
                                                            __half* __restrict__ y_lo, int ld_y, int off_y)
{
    const long total = (long)n * h * w * c_out;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int ch = (int)(i % c_out);
    const long pix = i / c_out;
    float v = 0.f;
    if (ch < c) {
        const float* p = raw + (size_t)pix * ld_raw + c0 + ch;
        float r;
        if (box) {
            const int x = (int)(pix % w), y = (int)((pix / w) % h);
            float s = 0.f;
            for (int dy = -1; dy <= 1; dy++)
                for (int dx = -1; dx <= 1; dx++)
                    if (y + dy >= 0 && y + dy < h && x + dx >= 0 && x + dx < w)
                        s += __ldg(p + ((long)dy * w + dx) * ld_raw);
            r = s / 9.f;
        } else {
            r = __ldg(p);
        }
        v = scale ? fmaf(r, __ldg(scale + ch), __ldg(shift + ch)) : r;
        if (relu) v = fmaxf(v, 0.f);
    }
    lwb::store_operand(v, (size_t)pix * ld_y + off_y + ch, y_f32, y_hi, y_lo);
}

}  // namespace

extern "C" int lwb_inception_input(const float* x, int n, int h, int w, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0, "bad sizes");
    const long total = (long)n * 3 * SIDE * SIDE;
    k_inception_input<<<lwb::ceil_div(total, THREADS), THREADS, 0, (cudaStream_t)stream>>>(x, n, h, w, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_bn_act_segment(const float* raw, int n, int h, int w, int ld_raw, int c0, int c, int c_out, int box,
                                  const float* scale, const float* shift, int relu, float* y_f32, void* y_hi, void* y_lo,
                                  int ld_y, int off_y, lwb_stream_t stream)
{
    LWB_CHECK_ARG(raw && (y_f32 || y_hi), "null pointer");
    LWB_CHECK_ARG((scale == nullptr) == (shift == nullptr), "scale and shift go together");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0 && c > 0 && c_out >= c, "bad sizes");
    LWB_CHECK_ARG(c0 >= 0 && c0 + c <= ld_raw && off_y >= 0 && off_y + c_out <= ld_y, "channel segment outside the pitch");
    const long total = (long)n * h * w * c_out;
    k_bn_act_segment<<<lwb::ceil_div(total, THREADS), THREADS, 0, (cudaStream_t)stream>>>(
        raw, n, h, w, ld_raw, c0, c, c_out, box ? 1 : 0, scale, shift, relu ? 1 : 0, y_f32, (__half*)y_hi, (__half*)y_lo,
        ld_y, off_y);
    LWB_LAUNCH_OK();
    return LWB_OK;
}
