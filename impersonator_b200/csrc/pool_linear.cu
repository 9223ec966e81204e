// Small fp32 kernels around the conv engine for the HMR encoder (networks/hmr.py:119-166, 214-252, 275-300):
// the stem's max-pool, the global average pool behind post_bn + ReLU, and the fully connected layers of the
// iterative theta regressor.  All three are far from any roofline-relevant size (per image: 0.8 M max-pool
// outputs, a 49 x 2048 mean, 3 x 3.3 M multiply-adds); they exist so that no torch operator sits on the path.
#include "common.cuh"

namespace {

// F.max_pool2d(x, kernel_size=k, stride=s, ceil_mode=True), no padding (networks/hmr.py:150):
// out = ceil((in - k) / s) + 1 windows, the last one clipped at the border.  NCHW in -> NHWC out.
__global__ void __launch_bounds__(256) k_maxpool_nchw_to_nhwc(const float* __restrict__ x, int n, int c, int h, int w,
                                                              int k, int s, int ho, int wo, float* __restrict__ out)
{
    const long total = (long)n * ho * wo * c;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    // consecutive threads walk x (coalesced reads of the NCHW plane); the NHWC write is strided by c
    const int ox = (int)(i % wo), oy = (int)((i / wo) % ho), ch = (int)((i / ((long)wo * ho)) % c), b = (int)(i / ((long)wo * ho * c));
    const float* p = x + ((size_t)b * c + ch) * h * w;
    float m = -INFINITY;
    for (int dy = 0; dy < k; dy++) {
        const int y = oy * s + dy;
        if (y >= h) break;
        for (int dx = 0; dx < k; dx++) {
            const int xx = ox * s + dx;
            if (xx >= w) break;
            m = fmaxf(m, __ldg(p + (size_t)y * w + xx));
        }
    }
    out[(((size_t)b * ho + oy) * wo + ox) * c + ch] = m;
}

// F.max_pool2d(x, kernel_size=k, stride=s) with the default ceil_mode=False (torchvision AlexNet's pools): out =
// floor((in - k) / s) + 1 windows, all inside the input.  NHWC fp32 in -> NHWC fp32 and / or the conv engine's fp16 hi / lo
// operands.  Consecutive threads walk the channels: coalesced reads and writes.  Channels [0, c) of an input with
// channel pitch ld_x land in channels [off_y, off_y + c) of outputs with pitch ld_y (InceptionV3's Mixed_6a / 7a pool
// branches write their slice of the block's concat buffer this way).
__global__ void __launch_bounds__(256) k_maxpool_nhwc(const float* __restrict__ x, int n, int h, int w, int c, int ld_x, int k,
                                                      int s, int ho, int wo, float* __restrict__ y_f32, __half* __restrict__ y_hi,
                                                      __half* __restrict__ y_lo, int ld_y, int off_y)
{
    const long total = (long)n * ho * wo * c;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int ch = (int)(i % c);
    const long pix = i / c;
    const int ox = (int)(pix % wo), oy = (int)((pix / wo) % ho), b = (int)(pix / ((long)wo * ho));
    const float* p = x + (((size_t)b * h + oy * s) * w + ox * s) * ld_x + ch;
    float m = -INFINITY;
    for (int dy = 0; dy < k; dy++)
        for (int dx = 0; dx < k; dx++)
            m = fmaxf(m, __ldg(p + ((size_t)dy * w + dx) * ld_x));
    const size_t o = (size_t)pix * ld_y + off_y + ch;
    if (y_f32) y_f32[o] = m;
    if (y_hi) {
        __half hi, lo;
        lwb::split_half(m, hi, lo);
        y_hi[o] = hi;
        if (y_lo) y_lo[o] = lo;
    }
}

// out[b, ch] = mean over hw of relu?(x[b, p, ch] * scale[ch] + shift[ch])   (post_bn + ReLU + avg_pool2d(7), hmr.py:160-163)
__global__ void __launch_bounds__(256) k_global_avgpool_nhwc(const float* __restrict__ x, int n, int hw, int c,
                                                             const float* __restrict__ scale, const float* __restrict__ shift,
                                                             int relu, float* __restrict__ out, int ld_out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * c) return;
    const int ch = i % c, b = i / c;
    const float sc = scale ? scale[ch] : 1.f, sh = shift ? shift[ch] : 0.f;
    const float* p = x + (size_t)b * hw * c + ch;
    float acc = 0.f;
    for (int q = 0; q < hw; q++) {
        float v = fmaf(__ldg(p + (size_t)q * c), sc, sh);
        if (relu) v = fmaxf(v, 0.f);
        acc += v;
    }
    out[(size_t)b * ld_out + ch] = acc / (float)hw;
}

// nn.Linear: out[b, m] (+)= relu?(sum_k x[b, k] * w[m, k] + bias[m]); one warp per (b, m).
__global__ void __launch_bounds__(256) k_linear(const float* __restrict__ x, int ld_x, const float* __restrict__ w,
                                                const float* __restrict__ bias, int n, int k, int m, int relu, int accumulate,
                                                float* __restrict__ out, int ld_out)
{
    const int warp = (int)(((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (warp >= n * m) return;
    const int b = warp / m, j = warp % m;
    const float* xr = x + (size_t)b * ld_x;
    const float* wr = w + (size_t)j * k;
    float acc = 0.f;
    for (int q = lane; q < k; q += 32) acc = fmaf(__ldg(xr + q), __ldg(wr + q), acc);
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) {
        float v = acc + (bias ? bias[j] : 0.f);
        if (relu) v = fmaxf(v, 0.f);
        float* o = out + (size_t)b * ld_out + j;
        *o = accumulate ? *o + v : v;
    }
}

}  // namespace

extern "C" int lwb_maxpool_nchw_to_nhwc(const float* x, int n, int c, int h, int w, int k, int stride, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && c > 0 && h >= k && w >= k && k > 0 && stride > 0, "bad sizes");
    const int ho = lwb::ceil_div(h - k, stride) + 1, wo = lwb::ceil_div(w - k, stride) + 1;
    const long total = (long)n * ho * wo * c;
    k_maxpool_nchw_to_nhwc<<<lwb::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(x, n, c, h, w, k, stride, ho, wo, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_maxpool_nhwc(const float* x, int n, int h, int w, int c, int k, int stride, float* y_f32, void* y_hi, void* y_lo,
                                lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && (y_f32 || y_hi), "null pointer");
    LWB_CHECK_ARG(n > 0 && c > 0 && h >= k && w >= k && k > 0 && stride > 0, "bad sizes");
    const int ho = (h - k) / stride + 1, wo = (w - k) / stride + 1;
    const long total = (long)n * ho * wo * c;
    k_maxpool_nhwc<<<lwb::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(x, n, h, w, c, c, k, stride, ho, wo, y_f32,
                                                                                (__half*)y_hi, (__half*)y_lo, c, 0);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_maxpool_nhwc_slice(const float* x, int n, int h, int w, int c, int ld_x, int k, int stride, float* y_f32,
                                      void* y_hi, void* y_lo, int ld_y, int off_y, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && (y_f32 || y_hi), "null pointer");
    LWB_CHECK_ARG(n > 0 && c > 0 && h >= k && w >= k && k > 0 && stride > 0, "bad sizes");
    LWB_CHECK_ARG(ld_x >= c && off_y >= 0 && off_y + c <= ld_y, "channel slice outside the pitch");
    const int ho = (h - k) / stride + 1, wo = (w - k) / stride + 1;
    const long total = (long)n * ho * wo * c;
    k_maxpool_nhwc<<<lwb::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(x, n, h, w, c, ld_x, k, stride, ho, wo, y_f32,
                                                                                (__half*)y_hi, (__half*)y_lo, ld_y, off_y);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_global_avgpool_nhwc(const float* x, int n, int hw, int c, const float* scale, const float* shift, int relu,
                                       float* out, int ld_out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && hw > 0 && c > 0 && ld_out >= c, "bad sizes");
    LWB_CHECK_ARG((scale == nullptr) == (shift == nullptr), "scale and shift go together");
    k_global_avgpool_nhwc<<<lwb::ceil_div((long)n * c, 256), 256, 0, (cudaStream_t)stream>>>(x, n, hw, c, scale, shift, relu, out, ld_out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_linear(const float* x, int ld_x, const float* w, const float* bias, int n, int k, int m, int relu, int accumulate,
                          float* out, int ld_out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && w && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && k > 0 && m > 0 && ld_x >= k && ld_out >= m, "bad sizes");
    const long threads = (long)n * m * 32;
    k_linear<<<lwb::ceil_div(threads, 256), 256, 0, (cudaStream_t)stream>>>(x, ld_x, w, bias, n, k, m, relu, accumulate, out, ld_out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}
