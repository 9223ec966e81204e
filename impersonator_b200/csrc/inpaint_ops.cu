// Glue of the background inpaintor (networks/inpaintor.py, once per source image) around the wgmma conv engine:
//   k_gated_act   the gated-convolution epilogue  y = BN(act(a + bias_a) * sigmoid(b + bias_b))        (:37-47)
//                 on the engine's raw NHWC output [.., a(0..c-1) | b(c..2c-1) | pad], emitting the NEXT layer's operands
//                 (hi / lo, channels padded with zeros to the 64-wide K chunks) -- optionally on the nearest-neighbour
//                 2x grid that GatedDeConv2dWithActivation convolves (:65-68), optionally clamped to [-1, 1] (:187,196)
//   k_self_attention  SelfAttention (:86-107): softmax(Q K^T) V over all N = H*W positions, flash-style (online softmax,
//                 K / V tiles in shared memory), fp32 on the CUDA cores: 2 N^2 (16 + 128) = 4.8 GFLOP per image
#include "common.cuh"
#include "operands.cuh"

namespace {

struct GatedParams {
    const float* raw; int n, h, w, c, c_stride;          // raw [n,h,w,c_stride]: a = [0,c), b = [c,2c)
    const float* bias;                                   // [2c] (conv2d.bias | mask_conv2d.bias), nullable
    int act;                                             // 0 none, 2 LeakyReLU(0.2)
    const float* scale; const float* shift;              // folded eval-mode BatchNorm [c], nullable
    int up;                                              // 1, or 2: every output pixel is written to its 2x2 block of a [2h,2w] grid
    int clamp;                                           // clamp y to [-1, 1] before emitting
    float* y_f32; int f32_stride;                        // [n,h*up,w*up,f32_stride] (first c channels), nullable
    __half* y_hi; __half* y_lo; int c_pad, lo_format;    // operands [n,h*up,w*up,c_pad], channels >= c zero; nullable
    int* range_flag;
};

// one thread = one pixel x 8 output channels of the padded operand row
__global__ void __launch_bounds__(256) k_gated_act(GatedParams P)
{
    lwb::pdl_wait();
    lwb::pdl_trigger();
    const int groups = (P.y_hi ? P.c_pad : ((P.c + 7) & ~7)) >> 3;
    const long total = (long)P.n * P.h * P.w * groups;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int g = (int)(i % groups);
    const long pix = i / groups;
    const int x = (int)(pix % P.w), y = (int)((pix / P.w) % P.h), b = (int)(pix / ((long)P.w * P.h));
    const float* r = P.raw + (size_t)pix * P.c_stride;
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int ch = g * 8 + k;
        float out = 0.f;
        if (ch < P.c) {
            float a = __ldg(r + ch), gt = __ldg(r + P.c + ch);
            if (P.bias) { a += __ldg(P.bias + ch); gt += __ldg(P.bias + P.c + ch); }
            if (P.act == 2) a = a > 0.f ? a : 0.2f * a;
            out = a * (1.f / (1.f + expf(-gt)));
            if (P.scale) out = fmaf(out, __ldg(P.scale + ch), __ldg(P.shift + ch));
            // torch.clamp (networks/inpaintor.py:187,196) keeps a NaN; fminf / fmaxf would return -1 for it
            if (P.clamp) out = out > 1.f ? 1.f : (out < -1.f ? -1.f : out);
        }
        v[k] = out;
    }
    const lwb::Operand8 e = lwb::encode8(v, P.lo_format);
    if (P.range_flag && P.y_hi) { if (const int bits = lwb::range_bits(e.hi)) atomicOr(P.range_flag, bits); }
    const int ho = P.h * P.up, wo = P.w * P.up;
    for (int dy = 0; dy < P.up; dy++) for (int dx = 0; dx < P.up; dx++) {
        const size_t opix = ((size_t)b * ho + (size_t)y * P.up + dy) * wo + (size_t)x * P.up + dx;
        if (P.y_f32) {
#pragma unroll
            for (int k = 0; k < 8; k++) if (g * 8 + k < P.c) P.y_f32[opix * P.f32_stride + g * 8 + k] = v[k];
        }
        if (P.y_hi) lwb::store8(e, nullptr, P.y_hi, P.y_lo, P.lo_format, opix * P.c_pad + g * 8, g * 8);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// out[i, :] = gamma * sum_j softmax_j(q_i . k_j) v_j + x[i, :]
// qkv [n, N, ld] fp32 (q at column 0, k at column dq, v at column 2*dq; + bias[2*dq + dv]); x / out [n, N, dv].
// Block = 256 threads = 64 queries x 4 threads; every thread keeps the full q (DQ = 16) and a quarter of the
// accumulator (32 of the DV = 128 channels, interleaved in float4 slots); keys / values stream through shared memory 64 at a time.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int AT_Q = 64, AT_K = 64, DQ = 16, DV = 128;

__global__ void __launch_bounds__(256) k_self_attention(const float* __restrict__ qkv, int ld, const float* __restrict__ bias,
                                                        int N, const float* __restrict__ x, const float* __restrict__ gamma,
                                                        float* __restrict__ out)
{
    __shared__ float s_k[AT_K][DQ];
    __shared__ __align__(16) float s_v[AT_K][DV];
    const int b = blockIdx.y;
    const int qi = blockIdx.x * AT_Q + (threadIdx.x >> 2), part = threadIdx.x & 3;
    const float* base = qkv + (size_t)b * N * ld;
    float q[DQ];
#pragma unroll
    for (int d = 0; d < DQ; d++) q[d] = qi < N ? base[(size_t)qi * ld + d] + bias[d] : 0.f;
    float acc[DV / 4];
#pragma unroll
    for (int d = 0; d < DV / 4; d++) acc[d] = 0.f;
    float m = -INFINITY, l = 0.f;
    for (int k0 = 0; k0 < N; k0 += AT_K) {
        __syncthreads();
        for (int t = threadIdx.x; t < AT_K * DQ; t += 256) {
            const int j = t / DQ, d = t % DQ;
            s_k[j][d] = (k0 + j < N) ? base[(size_t)(k0 + j) * ld + DQ + d] + bias[DQ + d] : 0.f;
        }
        for (int t = threadIdx.x; t < AT_K * DV; t += 256) {
            const int j = t / DV, d = t % DV;
            s_v[j][d] = (k0 + j < N) ? base[(size_t)(k0 + j) * ld + 2 * DQ + d] + bias[2 * DQ + d] : 0.f;
        }
        __syncthreads();
        const int kn = min(AT_K, N - k0);
        for (int j = 0; j < kn; j++) {
            float s = 0.f;
#pragma unroll
            for (int d = 0; d < DQ; d++) s = fmaf(q[d], s_k[j][d], s);
            if (s > m) {                                   // rescale the running sums to the new maximum
                const float f = expf(m - s);
                l *= f;
#pragma unroll
                for (int d = 0; d < DV / 4; d++) acc[d] *= f;
                m = s;
            }
            const float p = expf(s - m);
            l += p;
            // thread `part` owns the float4 slots part, part + 4, ... of the value row: the four threads of a query read
            // consecutive 16-byte words (conflict-free), the eight queries of a warp read the same words (broadcast)
            const float4* vv = reinterpret_cast<const float4*>(&s_v[j][0]);
#pragma unroll
            for (int d = 0; d < DV / 16; d++) {
                const float4 t = vv[d * 4 + part];
                acc[4 * d] = fmaf(p, t.x, acc[4 * d]); acc[4 * d + 1] = fmaf(p, t.y, acc[4 * d + 1]);
                acc[4 * d + 2] = fmaf(p, t.z, acc[4 * d + 2]); acc[4 * d + 3] = fmaf(p, t.w, acc[4 * d + 3]);
            }
        }
    }
    if (qi >= N) return;
    const float gm = gamma[0], inv = 1.f / l;
    const size_t o = ((size_t)b * N + qi) * DV;
#pragma unroll
    for (int d = 0; d < DV / 16; d++) {
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const size_t ch = o + (size_t)(d * 4 + part) * 4 + e;
            out[ch] = fmaf(gm, acc[4 * d + e] * inv, x[ch]);
        }
    }
}

}  // namespace

extern "C" int lwb_gated_act_nhwc(const float* raw, int n, int h, int w, int c, int c_stride, const float* bias, int act,
                                  const float* scale, const float* shift, int upsample, int clamp,
                                  float* y_f32, int f32_stride, uint16_t* y_hi, uint16_t* y_lo, int c_pad, int lo_format,
                                  int* range_flag, lwb_stream_t stream)
{
    LWB_CHECK_ARG(raw && (y_f32 || y_hi), "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0 && c > 0 && c_stride >= 2 * c, "bad sizes");
    LWB_CHECK_ARG(act == 0 || act == 2, "act must be 0 (none) or 2 (LeakyReLU 0.2)");
    LWB_CHECK_ARG((scale == nullptr) == (shift == nullptr), "scale and shift go together");
    LWB_CHECK_ARG(upsample == 1 || upsample == 2, "upsample must be 1 or 2");
    LWB_CHECK_ARG(!y_hi || (c_pad >= c && c_pad % 8 == 0 && (lo_format == 0 || (lo_format == 1 && c_pad % 64 == 0))), "bad operand padding");
    LWB_CHECK_ARG(!y_f32 || f32_stride >= c, "bad f32 stride");
    GatedParams P;
    P.raw = raw; P.n = n; P.h = h; P.w = w; P.c = c; P.c_stride = c_stride; P.bias = bias; P.act = act;
    P.scale = scale; P.shift = shift; P.up = upsample; P.clamp = clamp; P.y_f32 = y_f32; P.f32_stride = f32_stride;
    P.y_hi = (__half*)y_hi; P.y_lo = (__half*)y_lo; P.c_pad = c_pad; P.lo_format = lo_format; P.range_flag = range_flag;
    const int groups = (y_hi ? c_pad : ((c + 7) & ~7)) / 8;
    const long total = (long)n * h * w * groups;
    LWB_CUDA_OK(lwb::launch_pdl(k_gated_act, dim3(lwb::ceil_div(total, 256)), dim3(256), 0, (cudaStream_t)stream, P));
    return LWB_OK;
}

extern "C" int lwb_self_attention_nhwc(const float* qkv, int ld, const float* bias, int n, int npos, int dq, int dv,
                                       const float* x, const float* gamma, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(qkv && bias && x && gamma && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && npos > 0 && n <= 65535, "bad sizes");
    LWB_CHECK_ARG(dq == DQ && dv == DV && ld >= 2 * DQ + DV, "the kernel is specialised for 16-dim queries / 128-dim values (SelfAttention(128))");
    dim3 grid(lwb::ceil_div(npos, AT_Q), n);
    k_self_attention<<<grid, 256, 0, (cudaStream_t)stream>>>(qkv, ld, bias, npos, x, gamma, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}
