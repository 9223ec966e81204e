// Input path: a batch of uint8 HxWx3 frames -> the resized tensors Imitator._personalize / inference build on the host
// (utils/cv_utils.py:10-47 read_cv2_img + transform_img, models/imitator.py:82-145, 157-189), in one launch.
//
// Each resized byte is what cv2.resize(frame, (S, S)) with its default INTER_LINEAR returns on uint8, which is not the
// textbook bilinear filter but OpenCV's fixed-point one (imgproc resize, the CV_8U path):
//   * coefficients: scale = 1 / (S / src) in double; f = (float)((d + 0.5) * scale - 0.5); s = floor(f); f -= s;
//     w0 = round_half_even((1 - f) * 2048), w1 = round_half_even(f * 2048), each rounded on its own, in float.
//     Columns clamp (s < 0 or s >= src - 1 -> f = 0 and s into range); rows keep f and only clamp the row indices.
//   * horizontal pass, exact in int32: H = p[s0] * a0 + p[s1] * a1.
//   * vertical pass, as OpenCV's vector code computes it for every output byte (16-bit high multiplies):
//     out = (((H0 >> 4) * b0 >> 16) + ((H1 >> 4) * b1 >> 16) + 2) >> 2, saturated to 0..255.
// The float outputs are numpy's float32 x / 255.0 * 2 - 1.0 on those bytes, rounded step by step (no FMA).
#include "common.cuh"

namespace {

struct Axis {
    int s0, s1, a0, a1;
};

// One output coordinate d of a src -> dst resize (dst / src given as scale = 1 / (dst / src) in double, as OpenCV has it).
__device__ __forceinline__ Axis linear_axis(int d, int src, double scale, bool clamp_weights)
{
    float f = __double2float_rn(__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5));
    int s = (int)floorf(f);
    f = __fsub_rn(f, (float)s);
    if (clamp_weights) {
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
    }
    Axis a;
    a.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
    a.a1 = __float2int_rn(__fmul_rn(f, 2048.f));
    a.s0 = min(max(s, 0), src - 1);
    a.s1 = min(max(s + 1, 0), src - 1);
    return a;
}

__device__ __forceinline__ float u8_to_signed(int v)
{
    return __fsub_rn(__fmul_rn(__fdiv_rn((float)v, 255.f), 2.f), 1.f);
}

// grid (pixel blocks, n): the first size*size pixels of a frame belong to the size x size resize (img and / or u8), the
// next hmr_size*hmr_size to the HMR resize.
__global__ void __launch_bounds__(256) k_frames_in(const uint8_t* __restrict__ frames, int h, int w, int bgr,
                                                    int size, double sc_x, double sc_y, float* __restrict__ img,
                                                    uint8_t* __restrict__ u8_bgr, long main_px,
                                                    int hmr_size, double hsc_x, double hsc_y, float* __restrict__ hmr,
                                                    long hmr_px)
{
    long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long b = blockIdx.y;
    const bool to_hmr = p >= main_px;
    if (to_hmr) {
        p -= main_px;
        if (p >= hmr_px) return;
    }
    const int out = to_hmr ? hmr_size : size;
    const int dy = (int)(p / out), dx = (int)(p % out);
    const Axis ax = linear_axis(dx, w, to_hmr ? hsc_x : sc_x, true), ay = linear_axis(dy, h, to_hmr ? hsc_y : sc_y, false);
    const uint8_t* src = frames + (size_t)b * h * w * 3;
    const uint8_t* r0 = src + (size_t)ay.s0 * w * 3;
    const uint8_t* r1 = src + (size_t)ay.s1 * w * 3;
    int v[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int h0 = __ldg(r0 + (size_t)ax.s0 * 3 + k) * ax.a0 + __ldg(r0 + (size_t)ax.s1 * 3 + k) * ax.a1;
        const int h1 = __ldg(r1 + (size_t)ax.s0 * 3 + k) * ax.a0 + __ldg(r1 + (size_t)ax.s1 * 3 + k) * ax.a1;
        const int t = ((((h0 >> 4) * ay.a0) >> 16) + (((h1 >> 4) * ay.a1) >> 16) + 2) >> 2;
        v[k] = min(max(t, 0), 255);
    }
    // v[] is in the frame's channel order; rgb[c] is channel c of the RGB image cv2.cvtColor(BGR2RGB) makes
    const int rgb[3] = {bgr ? v[2] : v[0], v[1], bgr ? v[0] : v[2]};
    const size_t plane = (size_t)out * out;
    float* f32 = to_hmr ? hmr : img;
    if (f32) {
#pragma unroll
        for (int c = 0; c < 3; c++) f32[((size_t)b * 3 + c) * plane + p] = u8_to_signed(rgb[c]);
    }
    if (!to_hmr && u8_bgr) {
        uint8_t* o = u8_bgr + ((size_t)b * plane + p) * 3;
        o[0] = (uint8_t)rgb[2]; o[1] = (uint8_t)rgb[1]; o[2] = (uint8_t)rgb[0];
    }
}

}  // namespace

extern "C" int lwb_frames_in(const uint8_t* frames, int n, int h, int w, int bgr, int size, float* img, int hmr_size,
                             float* hmr, uint8_t* u8_bgr, lwb_stream_t stream)
{
    LWB_CHECK_ARG(frames, "null frames");
    LWB_CHECK_ARG(img || hmr || u8_bgr, "no output requested (img, hmr and u8_bgr are all null)");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0, "non-positive batch or frame size");
    LWB_CHECK_ARG(!(img || u8_bgr) || size > 0, "non-positive size");
    LWB_CHECK_ARG(!hmr || hmr_size > 0, "non-positive hmr_size");
    LWB_CHECK_ARG(n <= 65535, "more than 65535 frames in one call");
    const long main_px = (img || u8_bgr) ? (long)size * size : 0, hmr_px = hmr ? (long)hmr_size * hmr_size : 0;
    // every offset is 64-bit; refuse batches whose byte counts do not fit (a 4096^2 batch of 16 is 805 MB)
    LWB_CHECK_ARG((double)n * h * w * 3 < 9e18 && (double)n * (main_px + hmr_px) * 12 < 9e18, "frame batch overflows 64-bit offsets");
    LWB_CHECK_ARG((main_px + hmr_px + 255) / 256 <= 0x7fffffff, "too many output pixels per frame");
    const double sc_x = 1.0 / ((double)size / w), sc_y = 1.0 / ((double)size / h);      // OpenCV: 1 / inv_scale
    const double hsc_x = 1.0 / ((double)hmr_size / w), hsc_y = 1.0 / ((double)hmr_size / h);
    const dim3 grid((unsigned)((main_px + hmr_px + 255) / 256), (unsigned)n);
    k_frames_in<<<grid, 256, 0, (cudaStream_t)stream>>>(frames, h, w, bgr, size, sc_x, sc_y, img, u8_bgr, main_px,
                                                          hmr_size, hsc_x, hsc_y, hmr, hmr_px);
    LWB_LAUNCH_OK();
    return LWB_OK;
}
