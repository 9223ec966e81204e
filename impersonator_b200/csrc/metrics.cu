// Paired image-quality metrics (his_evaluators/metrics/metrics.py:450-631):
//   SSIM  = skimage.metrics.structural_similarity(pred, ref, multichannel=True) of skimage 0.16.2 on [-1, 1] float32 HWC
//           images: 7x7 uniform window, sample covariance (49/48), K1 0.01, K2 0.03, data_range 2, the map cropped by 3
//           pixels per side and averaged per channel, then the mean over the channels;
//   PSNR  = skimage.metrics.peak_signal_noise_ratio(image_true=ref, image_test=pred): mean of the float32 (ref - pred)^2
//           accumulated in float64, data_range 1 when min(ref) >= 0 and 2 otherwise;
//   LPIPS = the per-layer tail of PNetLin (lpips/models/networks_basic.py:121-168): unit-normalised channels of both
//           images' AlexNet features, squared difference, the 1x1 `lin` weights, spatial mean, summed over the 5 taps.
// Every reduction runs in a fixed order (no float atomics), so the scores repeat bit for bit.
#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------
// SSIM + PSNR: tiles of 8 rows x 64 columns of one channel of one frame.  The per-pixel statistics are float64 (the
// variance terms are differences of nearly equal moments, which float32 would leave at ~1e-7 and the SSIM map at
// ~1e-5 per pixel).  Only pixels at least 3 from every border enter the SSIM mean, so the 7x7 windows that matter never
// leave the image and the filter's boundary mode never shows.
// ------------------------------------------------------------------------------------------
constexpr int ST_H = 8, ST_W = 64, SR = 3;
constexpr int SP_H = ST_H + 2 * SR, SP_W = ST_W + 2 * SR;       // 14 x 70 input window
constexpr int S_THREADS = 256;

__device__ __forceinline__ float load01(const float* p, int from01)
{
    const float v = __ldg(p);
    return from01 ? __fsub_rn(__fmul_rn(v, 2.f), 1.f) : v;        // metrics.py:471-472: x * 2 - 1 in float32
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* red)
{
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] = red[threadIdx.x] + red[threadIdx.x + s];
        __syncthreads();
    }
    const T r = red[0];
    __syncthreads();
    return r;
}

template <typename T>
__device__ __forceinline__ T block_min(T v, T* red)
{
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] = red[threadIdx.x + s] < red[threadIdx.x] ? red[threadIdx.x + s] : red[threadIdx.x];
        __syncthreads();
    }
    const T r = red[0];
    __syncthreads();
    return r;
}

// part[(img*3 + ch) * tiles + tile] = {sum of the SSIM map over the tile's interior pixels, sum of (ref - pred)^2 over
// the tile's pixels, min(ref) over the tile's pixels}
__global__ void __launch_bounds__(S_THREADS) k_ssim_tiles(const float* __restrict__ pred, const float* __restrict__ ref,
                                                          int h, int w, int from01, double3* __restrict__ part)
{
    __shared__ float s_x[SP_H][SP_W], s_y[SP_H][SP_W];
    __shared__ double s_h[5][SP_H][ST_W];                           // horizontal 7-sums of x, y, xx, yy, xy
    __shared__ double s_red[S_THREADS];
    const int plane = blockIdx.z;                                   // img * 3 + ch
    const int y0 = blockIdx.y * ST_H, x0 = blockIdx.x * ST_W;
    const float* xp = pred + (size_t)plane * h * w;
    const float* yp = ref + (size_t)plane * h * w;
    for (int i = threadIdx.x; i < SP_H * SP_W; i += S_THREADS) {
        const int r = i / SP_W, c = i % SP_W;
        const int yy = y0 + r - SR, xx = x0 + c - SR;
        const bool in = yy >= 0 && yy < h && xx >= 0 && xx < w;
        s_x[r][c] = in ? load01(xp + (size_t)yy * w + xx, from01) : 0.f;
        s_y[r][c] = in ? load01(yp + (size_t)yy * w + xx, from01) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < SP_H * ST_W; i += S_THREADS) {
        const int r = i / ST_W, c = i % ST_W;
        double sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
        for (int k = 0; k < 7; k++) {
            const double a = s_x[r][c + k], b = s_y[r][c + k];
            sx += a; sy += b; sxx += a * a; syy += b * b; sxy += a * b;
        }
        s_h[0][r][c] = sx; s_h[1][r][c] = sy; s_h[2][r][c] = sxx; s_h[3][r][c] = syy; s_h[4][r][c] = sxy;
    }
    __syncthreads();
    const double C1 = (0.01 * 2.0) * (0.01 * 2.0), C2 = (0.03 * 2.0) * (0.03 * 2.0), cov_norm = 49.0 / 48.0;
    double s_sum = 0.0, e_sum = 0.0;
    float r_min = INFINITY;
    for (int i = threadIdx.x; i < ST_H * ST_W; i += S_THREADS) {
        const int r = i / ST_W, c = i % ST_W;
        const int yy = y0 + r, xx = x0 + c;
        if (yy >= h || xx >= w) continue;
        const float xv = s_x[r + SR][c + SR], yv = s_y[r + SR][c + SR];
        const float d = __fsub_rn(yv, xv);                          // float32 (ref - pred) ** 2, summed in float64
        e_sum += (double)__fmul_rn(d, d);
        r_min = fminf(r_min, yv);
        if (yy < SR || yy >= h - SR || xx < SR || xx >= w - SR) continue;
        double m[5];
#pragma unroll
        for (int q = 0; q < 5; q++) {
            double s = 0;
#pragma unroll
            for (int k = 0; k < 7; k++) s += s_h[q][r + k][c];
            m[q] = s / 49.0;
        }
        const double ux = m[0], uy = m[1];
        const double vx = cov_norm * (m[2] - ux * ux), vy = cov_norm * (m[3] - uy * uy), vxy = cov_norm * (m[4] - ux * uy);
        const double A1 = 2 * ux * uy + C1, A2 = 2 * vxy + C2, B1 = ux * ux + uy * uy + C1, B2 = vx + vy + C2;
        s_sum += (A1 * A2) / (B1 * B2);
    }
    s_sum = block_sum(s_sum, s_red);
    e_sum = block_sum(e_sum, s_red);
    r_min = block_min(r_min, reinterpret_cast<float*>(s_red));
    if (threadIdx.x == 0)
        part[(size_t)plane * gridDim.x * gridDim.y + blockIdx.y * gridDim.x + blockIdx.x] = make_double3(s_sum, e_sum, (double)r_min);
}

// one block per frame: fixed-order sums of its 3 x tiles partials
__global__ void __launch_bounds__(S_THREADS) k_ssim_finish(const double3* __restrict__ part, int tiles, int h, int w,
                                                           double* __restrict__ ssim, double* __restrict__ psnr)
{
    __shared__ double s_red[S_THREADS];
    const int img = blockIdx.x;
    double ssim_c[3], err = 0.0, rmin = INFINITY;
    for (int ch = 0; ch < 3; ch++) {
        const double3* p = part + ((size_t)img * 3 + ch) * tiles;
        double s = 0.0, e = 0.0, mn = INFINITY;
        for (int t = threadIdx.x; t < tiles; t += S_THREADS) { s += p[t].x; e += p[t].y; mn = fmin(mn, p[t].z); }
        ssim_c[ch] = block_sum(s, s_red) / ((double)(h - 2 * SR) * (double)(w - 2 * SR));
        err += block_sum(e, s_red);
        rmin = fmin(rmin, block_min(mn, s_red));
    }
    if (threadIdx.x == 0) {
        ssim[img] = (ssim_c[0] + ssim_c[1] + ssim_c[2]) / 3.0;
        const double mse = err / (3.0 * h * w);
        const double range = rmin >= 0.0 ? 1.0 : 2.0;
        psnr[img] = 10.0 * log10((range * range) / mse);             // mse = 0 -> +inf, as numpy's division gives
    }
}

// ------------------------------------------------------------------------------------------
// LPIPS
// ------------------------------------------------------------------------------------------
// PNetLin's input: x (from [0,1]: x * 2 - 1) -> (x - shift) / scale (networks_basic.py:102-103,122-123), float32.
// Rows 0..n-1 of out are pred, n..2n-1 ref.
__global__ void __launch_bounds__(256) k_lpips_input(const float* __restrict__ pred, const float* __restrict__ ref, int n, int hw,
                                                     int from01, float* __restrict__ out)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long per = 3L * hw, total = 2L * n * per;
    if (i >= total) return;
    const long img = i / per, rem = i % per;
    const int ch = (int)(rem / hw);
    const float* src = img < n ? pred + img * per : ref + (img - n) * per;
    const float shift = ch == 0 ? -.030f : ch == 1 ? -.088f : -.188f;
    const float scale = ch == 0 ? .458f : ch == 1 ? .448f : .450f;
    out[i] = __fdiv_rn(__fsub_rn(load01(src + rem, from01), shift), scale);
}

// One block per frame; one warp per pixel at a time, lanes over channels.  feat NHWC [2n, hw, c]: frame i's pred
// features are image i, its ref features image n + i.
constexpr int L_THREADS = 256, L_WARPS = L_THREADS / 32;

__global__ void __launch_bounds__(L_THREADS) k_lpips_layer(const float* __restrict__ feat, int n, int hw, int c,
                                                           const float* __restrict__ lin, int layer, int num_layers,
                                                           float* __restrict__ layers, float* __restrict__ score)
{
    __shared__ double s_red[L_WARPS];
    const int img = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* f1 = feat + (size_t)img * hw * c;                  // pred (in1)
    const float* f0 = feat + (size_t)(n + img) * hw * c;            // ref (in0)
    double acc = 0.0;
    for (int p = warp; p < hw; p += L_WARPS) {
        const float* a = f0 + (size_t)p * c;
        const float* b = f1 + (size_t)p * c;
        float ss0 = 0.f, ss1 = 0.f;
        for (int k = lane; k < c; k += 32) {
            const float u = __ldg(a + k), v = __ldg(b + k);
            ss0 = fmaf(u, u, ss0); ss1 = fmaf(v, v, ss1);
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            ss0 += __shfl_xor_sync(0xffffffffu, ss0, off);
            ss1 += __shfl_xor_sync(0xffffffffu, ss1, off);
        }
        const float d0 = sqrtf(ss0) + 1e-10f, d1 = sqrtf(ss1) + 1e-10f;     // util.normalize_tensor, eps 1e-10
        float t = 0.f;
        for (int k = lane; k < c; k += 32) {
            const float e = __ldg(a + k) / d0 - __ldg(b + k) / d1;
            t = fmaf(__ldg(lin + k), e * e, t);
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
        acc += (double)t;
    }
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int k = 0; k < L_WARPS; k++) s += s_red[k];
        const float v = (float)(s / hw);
        layers[(size_t)img * num_layers + layer] = v;
        score[img] = layer == 0 ? v : score[img] + v;               // the taps run in order on one stream
    }
}

}  // namespace

extern "C" size_t lwb_ssim_psnr_workspace_bytes(int n, int h, int w)
{
    if (n <= 0 || h <= 0 || w <= 0) return 0;
    return (size_t)n * 3 * lwb::ceil_div(h, ST_H) * lwb::ceil_div(w, ST_W) * sizeof(double3);
}

extern "C" int lwb_ssim_psnr(const float* pred, const float* ref, int n, int h, int w, int from01, void* workspace,
                             double* ssim_out, double* psnr_out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(pred && ref && workspace && ssim_out && psnr_out, "null pointer");
    LWB_CHECK_ARG(n > 0 && n <= 65535 / 3 && h >= 7 && w >= 7, "bad sizes (the 7x7 window needs h, w >= 7)");
    dim3 grid(lwb::ceil_div(w, ST_W), lwb::ceil_div(h, ST_H), n * 3);
    LWB_CHECK_ARG(grid.y <= 65535, "image too tall");
    k_ssim_tiles<<<grid, S_THREADS, 0, (cudaStream_t)stream>>>(pred, ref, h, w, from01 ? 1 : 0, (double3*)workspace);
    LWB_LAUNCH_OK();
    k_ssim_finish<<<n, S_THREADS, 0, (cudaStream_t)stream>>>((const double3*)workspace, (int)(grid.x * grid.y), h, w,
                                                            ssim_out, psnr_out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_lpips_input(const float* pred, const float* ref, int n, int h, int w, int from01, float* out,
                               lwb_stream_t stream)
{
    LWB_CHECK_ARG(pred && ref && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0, "bad sizes");
    const long total = 2L * n * 3 * h * w;
    k_lpips_input<<<lwb::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(pred, ref, n, h * w, from01 ? 1 : 0, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_lpips_layer(const float* feat, int n, int hw, int c, const float* lin, int layer, int num_layers,
                               float* layers_out, float* score, lwb_stream_t stream)
{
    LWB_CHECK_ARG(feat && lin && layers_out && score, "null pointer");
    LWB_CHECK_ARG(n > 0 && hw > 0 && c > 0 && num_layers > 0 && layer >= 0 && layer < num_layers, "bad sizes");
    k_lpips_layer<<<n, L_THREADS, 0, (cudaStream_t)stream>>>(feat, n, hw, c, lin, layer, num_layers, layers_out, score);
    LWB_LAUNCH_OK();
    return LWB_OK;
}
