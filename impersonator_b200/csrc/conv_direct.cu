// CUDA-core convolutions: the generator's 7x7 output heads (64 -> 3+1 channels, far too narrow
// for a 128-wide MMA tile) and a plain direct NCHW convolution for the once-per-source inpaintor
// layers (networks/inpaintor.py:12-47: 5x5, 4x4 stride 2, 3x3 dilated, biased).
#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------
// heads: out[n,y,x,0..3] = sum_{ky,kx,c} x[n,y+ky-3,x+kx-3,c] * w4[ky*7+kx][c][0..3]
//   networks/generator.py:126-134 (img_reg 64->3, attetion_reg 64->1, k7 p3, bias=False)
// Block = 128 threads -> 16 rows x 32 cols of outputs; each thread owns 4 consecutive x.
// Channels are processed 8 at a time: halo tile (22 x 38 px x 8 ch) + weights (49 x 8 x 4) in smem.
// Per (ky, c-chunk): 10 input float4 pairs feed 4 px x 7 kx x 8 c x 4 co = 896 FMAs.
// ------------------------------------------------------------------------------------------
constexpr int HT_H = 16, HT_W = 64, HC = 4, HALO = 3, HPX = 8;       // 8 px per thread along x
constexpr int HP_H = HT_H + 2 * HALO, HP_W = HT_W + 2 * HALO;       // 22 x 70 halo tile
constexpr int HP_WP = 72;                                           // padded row pitch (floats), 16B aligned

__global__ void __launch_bounds__(128) k_heads7x7(const float* __restrict__ x, const float* __restrict__ w4,
                                                  int n, int h, int w, float* __restrict__ out)
{
    // s_in[row][channel][x]: a thread's 16 consecutive x of one channel are 4 aligned float4 loads (14 used for
    // 8 outputs x 7 taps).
    __shared__ __align__(16) float s_in[HP_H][HC][HP_WP];           // 25344 B
    __shared__ __align__(16) float s_w[49][HC][4];                  //  3136 B
    const int b = blockIdx.z;
    const int y0 = blockIdx.y * HT_H, x0 = blockIdx.x * HT_W;
    const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;          // 8 x 16 threads, 8 px each along x
    float2 acc[HPX][2];
#pragma unroll
    for (int p = 0; p < HPX; p++) { acc[p][0] = make_float2(0.f, 0.f); acc[p][1] = make_float2(0.f, 0.f); }

    for (int c0 = 0; c0 < 64; c0 += HC) {
        __syncthreads();
        // fill: consecutive threads take consecutive x of one row -> 16B global reads (stride 256B between pixels)
        // and conflict-free scalar smem stores
        for (int i = threadIdx.x; i < HP_H * HP_WP; i += 128) {
            const int px = i % HP_WP, py = i / HP_WP;
            const int yy = y0 + py - HALO, xx = x0 + px - HALO;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (px < HP_W && yy >= 0 && yy < h && xx >= 0 && xx < w)
                v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)b * h + yy) * w + xx) * 64 + c0));
            const int ps = (((px >> 2) ^ ((px >> 5) & 1)) << 2) | (px & 3);      // float4-slot swizzle, see the loads below
            s_in[py][0][ps] = v.x; s_in[py][1][ps] = v.y; s_in[py][2][ps] = v.z; s_in[py][3][ps] = v.w;
        }
        for (int i = threadIdx.x; i < 49 * HC; i += 128) {
            const int tap = i / HC, c = i % HC;
            *reinterpret_cast<float4*>(&s_w[tap][c][0]) = __ldg(reinterpret_cast<const float4*>(w4 + ((size_t)tap * 64 + c0 + c) * 4));
        }
        __syncthreads();
#pragma unroll 1
        for (int ky = 0; ky < 7; ky++) {
#pragma unroll
            for (int c = 0; c < HC; c++) {
                float in[16];
                // lanes tx and tx+4 of a quarter-warp would hit the same banks (their float4 slots differ by 8):
                // slots 8..15 are stored with their lowest bit flipped, which makes the 8 accesses conflict-free
                const float4* src = reinterpret_cast<const float4*>(&s_in[ty + ky][c][0]);
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int slot = tx * 2 + j;
                    const float4 a = src[slot ^ ((slot >> 3) & 1)];
                    in[4 * j] = a.x; in[4 * j + 1] = a.y; in[4 * j + 2] = a.z; in[4 * j + 3] = a.w;
                }
#pragma unroll
                for (int kx = 0; kx < 7; kx++) {
                    const float4 wv = *reinterpret_cast<const float4*>(&s_w[ky * 7 + kx][c][0]);
                    const float2 w01 = make_float2(wv.x, wv.y), w23 = make_float2(wv.z, wv.w);
#pragma unroll
                    for (int p = 0; p < HPX; p++) {
                        const float vv = in[p + kx];
                        acc[p][0].x = fmaf(vv, w01.x, acc[p][0].x); acc[p][0].y = fmaf(vv, w01.y, acc[p][0].y);
                        acc[p][1].x = fmaf(vv, w23.x, acc[p][1].x); acc[p][1].y = fmaf(vv, w23.y, acc[p][1].y);
                    }
                }
            }
        }
    }
    const int y = y0 + ty;
    if (y < h) {
#pragma unroll
        for (int p = 0; p < HPX; p++) {
            const int xx = x0 + tx * HPX + p;
            if (xx < w)
                *reinterpret_cast<float4*>(out + (((size_t)b * h + y) * w + xx) * 4) =
                    make_float4(acc[p][0].x, acc[p][0].y, acc[p][1].x, acc[p][1].y);
        }
    }
}

__global__ void k_pack_heads(const float* __restrict__ w_img, const float* __restrict__ w_att, float* __restrict__ w4)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;            // over 49*64*4
    if (i >= 49 * 64 * 4) return;
    const int o = i & 3, c = (i >> 2) & 63, tap = i >> 8;
    w4[i] = o < 3 ? w_img[((size_t)o * 64 + c) * 49 + tap] : w_att[(size_t)c * 49 + tap];
}

// ------------------------------------------------------------------------------------------
// generic direct convolution, NCHW fp32 (cold path: once per source image)
// one thread = one output pixel x 4 output channels; weights are warp-uniform (broadcast loads)
// NHWC_RELU: relu(out) written NHWC (LPIPS' AlexNet conv1, 11x11 s4, whose output feeds an NHWC pool and a metric tap)
// ------------------------------------------------------------------------------------------
template <bool NHWC_RELU>
__global__ void __launch_bounds__(256) k_conv_direct(const float* __restrict__ x, const float* __restrict__ w,
                                                     const float* __restrict__ bias,
                                                     int cin, int h, int wd, int cout, int kh, int kw,
                                                     int stride, int pad, int dil, int ho, int wo, float* __restrict__ out)
{
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    const int co0 = blockIdx.y * 4, b = blockIdx.z;
    if (pix >= ho * wo) return;
    const int oy = pix / wo, ox = pix % wo;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const size_t plane = (size_t)h * wd;
    const float* xb = x + (size_t)b * cin * plane;
    const size_t wstride = (size_t)cin * kh * kw;
    for (int ky = 0; ky < kh; ky++) {
        const int iy = oy * stride - pad + ky * dil;
        if (iy < 0 || iy >= h) continue;
        for (int kx = 0; kx < kw; kx++) {
            const int ix = ox * stride - pad + kx * dil;
            if (ix < 0 || ix >= wd) continue;
            const float* xp = xb + (size_t)iy * wd + ix;
            const float* wp = w + (size_t)co0 * wstride + ky * kw + kx;
            for (int c = 0; c < cin; c++) {
                const float v = __ldg(xp + c * plane);
                const float* wc = wp + (size_t)c * kh * kw;
#pragma unroll
                for (int j = 0; j < 4; j++)
                    if (co0 + j < cout) acc[j] = fmaf(v, __ldg(wc + j * wstride), acc[j]);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 4; j++)
        if (co0 + j < cout) {
            const float v = acc[j] + (bias ? __ldg(bias + co0 + j) : 0.f);
            if (NHWC_RELU) out[((size_t)b * ho * wo + pix) * cout + co0 + j] = fmaxf(v, 0.f);
            else           out[((size_t)b * cout + co0 + j) * ho * wo + pix] = v;
        }
}

}  // namespace

extern "C" int lwb_pack_head_weights(const float* w_img, const float* w_att, float* w4, lwb_stream_t stream)
{
    LWB_CHECK_ARG(w_img && w_att && w4, "null pointer");
    k_pack_heads<<<lwb::ceil_div(49 * 64 * 4, 256), 256, 0, (cudaStream_t)stream>>>(w_img, w_att, w4);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_conv7x7_heads_nhwc(const float* x, const float* w4, int n, int h, int w, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && w4 && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0 && n <= 65535, "bad sizes");
    dim3 grid(lwb::ceil_div(w, HT_W), lwb::ceil_div(h, HT_H), n);
    k_heads7x7<<<grid, 128, 0, (cudaStream_t)stream>>>(x, w4, n, h, w, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_conv2d_direct_nchw(const float* x, const float* w, const float* bias,
                                      int n, int cin, int h, int wd, int cout, int kh, int kw,
                                      int stride, int pad, int dil, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && w && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && cin > 0 && h > 0 && wd > 0 && cout > 0 && kh > 0 && kw > 0 && stride > 0 && dil > 0 && pad >= 0, "bad sizes");
    const int ho = (h + 2 * pad - dil * (kh - 1) - 1) / stride + 1;
    const int wo = (wd + 2 * pad - dil * (kw - 1) - 1) / stride + 1;
    LWB_CHECK_ARG(ho > 0 && wo > 0 && n <= 65535, "empty output");
    dim3 grid(lwb::ceil_div((long)ho * wo, 256), lwb::ceil_div(cout, 4), n);
    k_conv_direct<false><<<grid, 256, 0, (cudaStream_t)stream>>>(x, w, bias, cin, h, wd, cout, kh, kw, stride, pad, dil, ho, wo, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_conv2d_direct_relu_nhwc(const float* x, const float* w, const float* bias,
                                           int n, int cin, int h, int wd, int cout, int kh, int kw,
                                           int stride, int pad, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && w && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && cin > 0 && h > 0 && wd > 0 && cout > 0 && kh > 0 && kw > 0 && stride > 0 && pad >= 0, "bad sizes");
    const int ho = (h + 2 * pad - kh) / stride + 1, wo = (wd + 2 * pad - kw) / stride + 1;
    LWB_CHECK_ARG(h + 2 * pad >= kh && wd + 2 * pad >= kw && n <= 65535, "empty output");
    dim3 grid(lwb::ceil_div((long)ho * wo, 256), lwb::ceil_div(cout, 4), n);
    k_conv_direct<true><<<grid, 256, 0, (cudaStream_t)stream>>>(x, w, bias, cin, h, wd, cout, kh, kw, stride, pad, 1, ho, wo, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}
