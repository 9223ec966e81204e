// HBM-bound glue kernels of the conv engine (sm_90a): layout conversion, weight packing,
// InstanceNorm + ReLU + residual + Liquid-Warping-Block add, output heads + composite.
//
// networks/generator.py:8-20 (ResidualBlock), :80-95 (Conv+IN+ReLU), :283-295 (tsf + warp),
// :183-184 (tanh / sigmoid heads), models/imitator.py:330-331 (composite).
#include "common.cuh"
#include "operands.cuh"
#include "sample.cuh"

namespace {

using lwb::split_half;

// ---------------------------------------------------------------------------------------------
// weights: OIHW (Conv2d) / IOHW (ConvTranspose2d) fp32 -> [tap][cout_pad][cin_pad] hi = fp16 of w * 2^E and
//   LO_FORMAT 0: lo (nullable) = the fp16 residual of w * 2^E;
//   LO_FORMAT 1: hi = fp16(w_hi) * 2^E, lo = the pair blocks [64 x e4m3(w_lo * 2^(E+4))][64 x e4m3(w * 2^(E-10))]
// (wscale = 2^E, the layer's exponent: max|w| * 2^E in [2^14, 2^15) keeps hi and lo out of the fp16 subnormals)
// ---------------------------------------------------------------------------------------------
template <int LO_FORMAT>
__global__ void k_pack_weight(const float* __restrict__ w, int cout, int cin, int kh, int kw, int transposed,
                              int cout_pad, int cin_pad, float wscale, __half* __restrict__ hi, void* __restrict__ lo)
{
    const long total = (long)kh * kw * cout_pad * cin_pad;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int ci = (int)(i % cin_pad);
        const int co = (int)((i / cin_pad) % cout_pad);
        const int tap = (int)(i / ((long)cin_pad * cout_pad));
        float v = 0.f;
        if (ci < cin && co < cout) {
            const int ky = tap / kw, kx = tap % kw;
            v = transposed ? w[(((size_t)ci * cout + co) * kh + ky) * kw + kx]
                           : w[(((size_t)co * cin + ci) * kh + ky) * kw + kx];
        }
        if (LO_FORMAT == 1) {
            const __half h = __float2half_rn(v);
            hi[i] = __float2half_rn(__half2float(h) * wscale);         // exact: |w| * 2^E < 2^15 (host picks E)
            uint8_t* blk = lwb::pair_block(lo, i, ci);
            blk[0] = lwb::to_e4m3((v - __half2float(h)) * (wscale * lwb::kF8WLoRel));
            blk[64] = lwb::to_e4m3(v * (wscale * lwb::kF8WRel));
        } else {
            __half h, l;
            split_half(v * wscale, h, l);
            hi[i] = h;
            if (lo) static_cast<__half*>(lo)[i] = l;
        }
    }
}

// First-layer packing for the row-contiguous 7x7 trick (see conv_tc.cu): [ky][cout_pad][kxs*cpx]
// with K index = kx*cpx + c  (kx < kw real taps, the rest zero), of w * 2^E like k_pack_weight.
__global__ void k_pack_weight_rowk(const float* __restrict__ w, int cout, int cin, int kh, int kw,
                                   int cout_pad, int cpx, int kxs, float wscale, __half* __restrict__ hi, __half* __restrict__ lo)
{
    const int kk = kxs * cpx;
    const long total = (long)kh * cout_pad * kk;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int k = (int)(i % kk);
        const int co = (int)((i / kk) % cout_pad);
        const int ky = (int)(i / ((long)kk * cout_pad));
        const int kx = k / cpx, c = k % cpx;
        float v = 0.f;
        if (kx < kw && c < cin && co < cout) v = w[(((size_t)co * cin + c) * kh + ky) * kw + kx];
        __half h, l;
        split_half(v * wscale, h, l);
        hi[i] = h;
        if (lo) lo[i] = l;
    }
}

// ---------------------------------------------------------------------------------------------
// NCHW fp32 -> NHWC fp16 hi/lo into a (possibly spatially padded) buffer [n, hp, wp, c_pad]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_nchw_to_nhwc_split(
        const float* __restrict__ x, int n, int c, int h, int w, int c_pad,
        int hp, int wp, int oy, int ox, __half* __restrict__ hi, __half* __restrict__ lo)
{
    const long total = (long)n * hp * wp;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int px = (int)(i % wp), py = (int)((i / wp) % hp), b = (int)(i / ((long)wp * hp));
    const int y = py - oy, xx = px - ox;
    const bool in = y >= 0 && y < h && xx >= 0 && xx < w;
    const size_t plane = (size_t)h * w;
    const float* src = x + (size_t)b * c * plane + (in ? (size_t)y * w + xx : 0);
    for (int ch = 0; ch < c_pad; ch++) {
        const float v = (in && ch < c) ? __ldg(src + ch * plane) : 0.f;
        __half a, l;
        split_half(v, a, l);
        hi[i * c_pad + ch] = a;
        if (lo) lo[i * c_pad + ch] = l;
    }
}

__global__ void __launch_bounds__(256) k_nhwc_to_nchw(
        const float* __restrict__ x, int n, int c, int h, int w, int c_stride, float* __restrict__ out)
{
    // tile transpose through shared memory: 32 pixels x 32 channels
    __shared__ float tile[32][33];
    const long npix = (long)h * w;
    const int b = blockIdx.z;
    const long p0 = (long)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;     // 256 threads: ty 0..7
    for (int j = ty; j < 32; j += 8) {
        const long p = p0 + j;
        const int ch = c0 + tx;
        tile[j][tx] = (p < npix && ch < c) ? x[((size_t)b * npix + p) * c_stride + ch] : 0.f;
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        const int ch = c0 + j;
        const long p = p0 + tx;
        if (p < npix && ch < c) out[((size_t)b * c + ch) * npix + p] = tile[tx][j];
    }
}

// ---------------------------------------------------------------------------------------------
// InstanceNorm statistics (sum, sumsq in f64 from the conv epilogue) -> per-(n,c) scale/shift
//   y = gamma*(x-mean)*rstd + beta = x*scale + shift        (biased variance, eps inside the sqrt)
// ---------------------------------------------------------------------------------------------
__global__ void k_finalize_stats(const double* __restrict__ stats, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, float eps, int n, int c, double inv_hw,
                                 float2* __restrict__ ss)
{
    lwb::pdl_wait();                                     // the statistics come from the conv kernel just before
    lwb::pdl_trigger();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * c) return;
    const int ch = i % c;
    const double mean = stats[2 * i] * inv_hw;
    double var = stats[2 * i + 1] * inv_hw - mean * mean;
    if (var < 0) var = 0;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    const float g = gamma ? gamma[ch] : 1.f, bt = beta ? beta[ch] : 0.f;
    ss[i] = make_float2(g * rstd, bt - (float)mean * g * rstd);
}

// Per-channel affine (eval-mode BatchNorm folded to scale / shift, or a conv bias) broadcast to the [n, c] table.
__global__ void k_fill_ss(const float* __restrict__ scale, const float* __restrict__ shift, int n, int c, float2* __restrict__ ss)
{
    lwb::pdl_wait();
    lwb::pdl_trigger();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * c) return;
    ss[i] = make_float2(scale ? scale[i % c] : 1.f, shift ? shift[i % c] : 0.f);
}

// Plain (two-pass, fp64) statistics for tensors that did not come out of the conv epilogue.
__global__ void __launch_bounds__(256) k_stats_nhwc(const float* __restrict__ x, int hw, int c, double* __restrict__ stats)
{
    // grid: (c/32 rounded up, n, splits); block 256 = 8 pixel lanes x 32 channels
    const int ch = blockIdx.x * 32 + (threadIdx.x & 31);
    const int b = blockIdx.y;
    const int lane_p = threadIdx.x >> 5;
    double s = 0, q = 0;
    if (ch < c) {
        for (long p = (long)blockIdx.z * 8 + lane_p; p < hw; p += (long)gridDim.z * 8) {
            const float v = x[((size_t)b * hw + p) * c + ch];
            s += v; q += (double)v * v;
        }
    }
    __shared__ double sh[2][8][32];
    sh[0][lane_p][threadIdx.x & 31] = s;
    sh[1][lane_p][threadIdx.x & 31] = q;
    __syncthreads();
    if (lane_p == 0 && ch < c) {
        for (int j = 1; j < 8; j++) { s += sh[0][j][threadIdx.x & 31]; q += sh[1][j][threadIdx.x & 31]; }
        atomicAdd(stats + 2 * ((size_t)b * c + ch), s);
        atomicAdd(stats + 2 * ((size_t)b * c + ch) + 1, q);
    }
}

// ---------------------------------------------------------------------------------------------
// y = act(x*scale + shift) + residual + warp(src, T)  ->  fp32 and/or fp16 hi/lo, NHWC
// one thread = one pixel x 8 channels (32B fp32 loads, 16B fp16 stores)
// ---------------------------------------------------------------------------------------------
struct NormActParams {
    const float* raw; const float2* ss; int relu;
    int n, h, w, c;
    const float* residual;
    const float* warp_src; int src_batch; const float* T; int th, tw, align_corners;
    float* y_f32; __half* y_hi; __half* y_lo;
    int lo_format;                                       // 0: y_lo = fp16 residual; 1: fp8 pair blocks (operands.cuh)
    int* range_flag;                                     // |= lwb::range_bits of the emitted operands
    // EXT only (BatchNorm-style nets, networks/hmr.py): the operands are relu?(y * post_scale[c] + post_shift[c]) while
    // y_f32 keeps y; the residual is read at (res_step*y, res_step*x) of a [n, h*res_step, w*res_step, c] tensor
    const float* post_scale; const float* post_shift; int post_relu; int res_step;
};

// Block = 256 threads = (256 / groups) pixels x groups channel-octets, two pixel rounds per thread so
// that four 16B loads per operand are in flight before any math.  The bilinear taps of a pixel are
// computed once (by one thread) and shared through smem instead of once per channel octet.
struct TapRec { int o00, m; float w00, w01, w10, w11; };
constexpr int kNormRounds = 2;                           // pixel rounds per thread

// WARP: the launch's dynamic shared memory holds the ppb * R tap records of the block (768 bytes at 128 channels), so
// that the block fits beside a resident conv CTA (about 17 KB of shared memory left, conv_tc.cu).
template <bool WARP, bool EXT>
__global__ void __launch_bounds__(256, 4) k_norm_act(NormActParams P)
{
    constexpr int R = kNormRounds;
    lwb::pdl_wait();                                     // raw / scale-shift / residual come from the kernels before
    lwb::pdl_trigger();                                  // the next conv may set up while this grid drains
    const int groups = P.c >> 3;
    const int ppb = 256 / groups;                        // pixels per block per round (groups <= 256)
    const int g = threadIdx.x % groups, lp = threadIdx.x / groups;
    const long npix = (long)P.n * P.h * P.w;
    const int hw = P.h * P.w;
    const long pix0 = (long)blockIdx.x * (ppb * R);
    extern __shared__ TapRec s_tap[];                    // WARP: ppb * R records
    if (WARP) {
        for (int i = threadIdx.x; i < ppb * R; i += 256) {
            const long pg = pix0 + i;
            TapRec t = {0, 0, 0.f, 0.f, 0.f, 0.f};
            if (pg < npix) {
                const int b = (int)(pg / hw), pix = (int)(pg % hw);
                float gx, gy;
                lwb::flow_at(P.T + (size_t)b * P.th * P.tw * 2, P.th, P.tw, P.h, P.w, pix / P.w, pix % P.w, gx, gy);
                lwb::Taps tp;
                lwb::make_taps(gx, gy, P.h, P.w, P.align_corners, tp);
                t.o00 = tp.o00; t.m = tp.m; t.w00 = tp.w00; t.w01 = tp.w01; t.w10 = tp.w10; t.w11 = tp.w11;
            }
            s_tap[i] = t;
        }
        __syncthreads();
    }
    if (lp >= ppb) return;                               // (256 % groups != 0 never happens for c = 64..2048)

    float v[R][8];
    bool ok[R];
    size_t off[R];
    int bb[R];
#pragma unroll
    for (int r = 0; r < R; r++) {
        const long pg = pix0 + r * ppb + lp;
        ok[r] = pg < npix;
        bb[r] = ok[r] ? (int)(pg / hw) : 0;
        off[r] = (size_t)(ok[r] ? pg : 0) * P.c + g * 8;
        if (ok[r]) lwb::ldg_f32x8(P.raw + off[r], v[r]);             // one 32-byte sector per lane (LDG.256)
        else {
#pragma unroll
            for (int k = 0; k < 8; k++) v[r][k] = 0.f;
        }
    }
    float res[R][8];
    if (P.residual && !WARP) {                           // WARP loads it per round: the warp taps need the registers
#pragma unroll
        for (int r = 0; r < R; r++) {
            size_t roff = off[r];
            if (EXT && P.res_step > 1 && ok[r]) {
                const int pix = (int)((pix0 + r * ppb + lp) % hw), y = pix / P.w, x = pix % P.w, st = P.res_step;
                roff = (((size_t)bb[r] * (P.h * st) + (size_t)y * st) * (P.w * st) + (size_t)x * st) * P.c + g * 8;
            }
            if (ok[r]) lwb::ldg_f32x8(P.residual + roff, res[r]);
            else {
#pragma unroll
                for (int k = 0; k < 8; k++) res[r][k] = 0.f;
            }
        }
    }
#pragma unroll
    for (int r = 0; r < R; r++) {
        if (P.ss) {
            const float4* ss = reinterpret_cast<const float4*>(P.ss + (size_t)bb[r] * P.c + g * 8);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const float4 s2 = __ldg(ss + k);         // (scale, shift) of channels 2k, 2k+1
                v[r][2 * k] = fmaf(v[r][2 * k], s2.x, s2.y);
                v[r][2 * k + 1] = fmaf(v[r][2 * k + 1], s2.z, s2.w);
            }
        }
        if (P.relu) {
#pragma unroll
            for (int k = 0; k < 8; k++) v[r][k] = fmaxf(v[r][k], 0.f);
        }
        if (P.residual) {
            if (WARP) {
                if (ok[r]) lwb::ldg_f32x8(P.residual + off[r], res[r]);
                else {
#pragma unroll
                    for (int k = 0; k < 8; k++) res[r][k] = 0.f;
                }
            }
#pragma unroll
            for (int k = 0; k < 8; k++) v[r][k] += res[r][k];
        }
        if (WARP) {
            const TapRec tp = s_tap[r * ppb + lp];
            const float* src = P.warp_src + (size_t)(P.src_batch == 1 ? 0 : bb[r]) * hw * P.c + g * 8;
            const int offs[4] = {tp.o00, tp.o00 + 1, tp.o00 + P.w, tp.o00 + P.w + 1};
            const float wt[4] = {tp.w00, tp.w01, tp.w10, tp.w11};
            float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
            for (int t = 0; t < 4; t++) {
                if (tp.m & (1 << t)) {
                    float q[8];
                    lwb::ldg_f32x8(src + (size_t)offs[t] * P.c, q);
#pragma unroll
                    for (int k = 0; k < 8; k++) acc[k] += q[k] * wt[t];
                }
            }
#pragma unroll
            for (int k = 0; k < 8; k++) v[r][k] += acc[k];
        }
        if (!ok[r]) continue;
        if (P.y_f32) lwb::stg_f32x8(P.y_f32 + off[r], v[r]);
        if (P.y_hi) {
            if (EXT && P.post_scale) {
                const float4* ps = reinterpret_cast<const float4*>(P.post_scale + g * 8);
                const float4* pt = reinterpret_cast<const float4*>(P.post_shift + g * 8);
                const float4 s0 = __ldg(ps), s1 = __ldg(ps + 1), t0 = __ldg(pt), t1 = __ldg(pt + 1);
                const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
                const float sh[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    v[r][k] = fmaf(v[r][k], sc[k], sh[k]);
                    if (P.post_relu) v[r][k] = fmaxf(v[r][k], 0.f);
                }
            }
            const lwb::Operand8 e = lwb::encode8(v[r], 0);
            if (P.range_flag) { if (const int bits = lwb::range_bits(e.hi)) atomicOr(P.range_flag, bits); }
            lwb::store8(e, v[r], P.y_hi, P.y_lo, P.lo_format, off[r], g * 8);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// heads: color = tanh(raw[0:3]), mask = sigmoid(raw[3]), pred = mask*bg + (1-mask)*color
// ---------------------------------------------------------------------------------------------
// numpy's ((img + 1) / 2.0 * 255).astype(uint8) of cv_utils.save_cv2_img (utils/cv_utils.py:31-33): fp32, truncation
__device__ __forceinline__ uint8_t to_u8(float x) {
    return (uint8_t)__float2int_rz(__fmul_rn(__fmul_rn(__fadd_rn(x, 1.f), 0.5f), 255.f));
}

// folded_kw > 0: ``raw`` is the output of the 7x7 heads run as a (kh x 1) tensor-core conv whose N dimension holds the
// filter columns -- raw[y, x', kx*4 + co] = sum_{ky,c} in[y+ky-3, x', c] * w[co, c, ky, kx] -- and the filter row is summed here:
//   out[y, x, co] = sum_kx raw[y, x + kx - kw/2, kx*4 + co]        (columns outside the image contribute the zero padding)
__global__ void __launch_bounds__(256) k_heads(const float* __restrict__ raw, int n, int hw, int w, int c_stride, int folded_kw,
                                               const float* __restrict__ bg, int bg_batch,
                                               float* __restrict__ color, float* __restrict__ mask, float* __restrict__ pred,
                                               float* __restrict__ pred_hwc, uint8_t* __restrict__ pred_u8_bgr,
                                               int* __restrict__ range_flag)
{
    lwb::pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n * hw) return;
    const int b = (int)(i / hw), p = (int)(i % hw);
    float4 r;
    if (folded_kw > 0) {
        const int x = p % w;
        r = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int kx = 0; kx < folded_kw; kx++) {
            const int xs = x + kx - folded_kw / 2;
            if (xs < 0 || xs >= w) continue;
            const float4 t = __ldg(reinterpret_cast<const float4*>(raw + (size_t)(i + (xs - x)) * c_stride + kx * 4));
            r.x += t.x; r.y += t.y; r.z += t.z; r.w += t.w;
        }
    } else {
        r = __ldg(reinterpret_cast<const float4*>(raw + (size_t)i * c_stride));
    }
    if (range_flag) {
        // Output-head pre-activations of +-8 and more: the ~1e-4 end-to-end RELATIVE precision of the fp16f8 operand split is
        // then no longer enough for 1e-3 on the (unsaturated) pixels -- report it, the caller switches to fp16x3.
        // (fmaxf would drop a NaN component, so each one is compared on its own)
        const bool big = !(fabsf(r.x) < 8.f && fabsf(r.y) < 8.f && fabsf(r.z) < 8.f && fabsf(r.w) < 8.f);
        if (__any_sync(__activemask(), big) && big && !(*reinterpret_cast<volatile int*>(range_flag) & LWB_RANGE_HEADS))
            atomicOr(range_flag, LWB_RANGE_HEADS);
    }
    const float col[3] = {tanhf(r.x), tanhf(r.y), tanhf(r.z)};
    const float m = 1.f / (1.f + expf(-r.w));
    if (mask) mask[i] = m;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        if (color) color[((size_t)b * 3 + k) * hw + p] = col[k];
        if (bg) {
            const float bgv = __ldg(bg + ((size_t)(bg_batch == 1 ? 0 : b) * 3 + k) * hw + p);
            const float pv = m * bgv + (1.f - m) * col[k];
            if (pred) pred[((size_t)b * 3 + k) * hw + p] = pv;
            if (pred_hwc) pred_hwc[(size_t)i * 3 + k] = pv;                      // preds[0].permute(1, 2, 0)  (imitator.py:178)
            if (pred_u8_bgr) pred_u8_bgr[(size_t)i * 3 + (2 - k)] = to_u8(pv);   // RGB2BGR + normalize (cv_utils.py:24-33)
        }
    }
}

// Output path for frames that did not come straight out of k_heads (e.g. after warp_front): NCHW fp32 -> HWC fp32 / BGR u8
__global__ void __launch_bounds__(256) k_frames_out(const float* __restrict__ x, int n, int hw,
                                                    float* __restrict__ hwc, uint8_t* __restrict__ u8_bgr)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n * hw) return;
    const int b = (int)(i / hw), p = (int)(i % hw);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float v = __ldg(x + ((size_t)b * 3 + k) * hw + p);
        if (hwc) hwc[(size_t)i * 3 + k] = v;
        if (u8_bgr) u8_bgr[(size_t)i * 3 + (2 - k)] = to_u8(v);
    }
}

// ---------------------------------------------------------------------------------------------
// gated conv epilogue of the inpaintor (networks/inpaintor.py:37-47), NCHW fp32:
//   ab = [conv2d(x) ; mask_conv2d(x)] stacked on channels;  y = act(a) * sigmoid(b);  out = y*scale + shift
//   (scale/shift = eval-mode BatchNorm2d folded: gamma/sqrt(var+eps), beta - mean*scale)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_gated_bn(const float* __restrict__ ab, int n, int c, int hw, int act,
                                                  const float* __restrict__ scale, const float* __restrict__ shift,
                                                  float* __restrict__ out)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n * c * hw) return;
    const int p = (int)(i % hw), ch = (int)((i / hw) % c), b = (int)(i / ((long)hw * c));
    float a = ab[((size_t)b * 2 * c + ch) * hw + p];
    const float g = ab[((size_t)b * 2 * c + c + ch) * hw + p];
    if (act == 2) a = a > 0.f ? a : 0.2f * a;
    else if (act == 1) a = fmaxf(a, 0.f);
    float y = a * (1.f / (1.f + expf(-g)));
    if (scale) y = fmaf(y, __ldg(scale + ch), __ldg(shift + ch));
    out[i] = y;
}

}  // namespace

extern "C" int lwb_gated_bn_nchw(const float* ab, int n, int c, int h, int w, int act,
                                 const float* scale, const float* shift, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(ab && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && c > 0 && h > 0 && w > 0, "bad sizes");
    LWB_CHECK_ARG((scale == nullptr) == (shift == nullptr), "scale and shift go together");
    k_gated_bn<<<lwb::ceil_div((long)n * c * h * w, 256), 256, 0, (cudaStream_t)stream>>>(ab, n, c, h * w, act, scale, shift, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_pack_conv_weight(const float* w, int cout, int cin, int kh, int kw, int transposed,
                                    int cout_pad, int cin_pad, int w_exp, uint16_t* w_hi, uint16_t* w_lo, lwb_stream_t stream)
{
    LWB_CHECK_ARG(w && w_hi, "null pointer");
    LWB_CHECK_ARG(cout > 0 && cin > 0 && kh > 0 && kw > 0 && cout_pad >= cout && cin_pad >= cin, "bad sizes");
    LWB_CHECK_ARG(w_exp >= -40 && w_exp <= 60, "w_exp out of range");
    const long total = (long)kh * kw * cout_pad * cin_pad;
    k_pack_weight<0><<<(int)min((total + 255) / 256, 4096l), 256, 0, (cudaStream_t)stream>>>(
        w, cout, cin, kh, kw, transposed, cout_pad, cin_pad, ldexpf(1.f, w_exp), (__half*)w_hi, w_lo);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_pack_conv_weight_f8(const float* w, int cout, int cin, int kh, int kw, int transposed,
                                       int cout_pad, int cin_pad, int w_exp, uint16_t* w_hi, uint8_t* w_lo8, lwb_stream_t stream)
{
    LWB_CHECK_ARG(w && w_hi && w_lo8, "null pointer");
    LWB_CHECK_ARG(cout > 0 && cin > 0 && kh > 0 && kw > 0 && cout_pad >= cout && cin_pad >= cin && (cin_pad % 64) == 0, "bad sizes");
    LWB_CHECK_ARG(w_exp >= -40 && w_exp <= 60, "w_exp out of range");
    const long total = (long)kh * kw * cout_pad * cin_pad;
    k_pack_weight<1><<<(int)min((total + 255) / 256, 4096l), 256, 0, (cudaStream_t)stream>>>(
        w, cout, cin, kh, kw, transposed, cout_pad, cin_pad, ldexpf(1.f, w_exp), (__half*)w_hi, w_lo8);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_pack_conv_weight_rowk(const float* w, int cout, int cin, int kh, int kw,
                                         int cout_pad, int cpx, int kxs, int w_exp, uint16_t* w_hi, uint16_t* w_lo,
                                         lwb_stream_t stream)
{
    LWB_CHECK_ARG(w && w_hi, "null pointer");
    LWB_CHECK_ARG(cout > 0 && cin > 0 && cin <= cpx && kw <= kxs && cout_pad >= cout, "bad sizes");
    LWB_CHECK_ARG(w_exp >= -40 && w_exp <= 60, "w_exp out of range");
    const long total = (long)kh * cout_pad * kxs * cpx;
    k_pack_weight_rowk<<<(int)min((total + 255) / 256, 4096l), 256, 0, (cudaStream_t)stream>>>(
        w, cout, cin, kh, kw, cout_pad, cpx, kxs, ldexpf(1.f, w_exp), (__half*)w_hi, (__half*)w_lo);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_nchw_to_nhwc_split(const float* x, int n, int c, int h, int w, int c_pad,
                                      int hp, int wp, int oy, int ox,
                                      uint16_t* hi, uint16_t* lo, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && hi, "null pointer");
    LWB_CHECK_ARG(n > 0 && c > 0 && h > 0 && w > 0 && c_pad >= c && hp >= h + oy && wp >= w + ox && oy >= 0 && ox >= 0, "bad sizes");
    const long total = (long)n * hp * wp;
    k_nchw_to_nhwc_split<<<lwb::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
        x, n, c, h, w, c_pad, hp, wp, oy, ox, (__half*)hi, (__half*)lo);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_nhwc_to_nchw(const float* x, int n, int c, int h, int w, int c_stride, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && out, "null pointer");
    LWB_CHECK_ARG(n > 0 && c > 0 && h > 0 && w > 0 && c_stride >= c && n <= 65535, "bad sizes");
    dim3 grid(lwb::ceil_div((long)h * w, 32), lwb::ceil_div(c, 32), n);
    k_nhwc_to_nchw<<<grid, 256, 0, (cudaStream_t)stream>>>(x, n, c, h, w, c_stride, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_instance_stats_nhwc(const float* x, int n, int h, int w, int c, double* stats, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && stats, "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0 && c > 0 && n <= 65535, "bad sizes");
    const int hw = h * w;
    const int splits = max(1, min(64, hw / 256));
    dim3 grid(lwb::ceil_div(c, 32), n, splits);
    k_stats_nhwc<<<grid, 256, 0, (cudaStream_t)stream>>>(x, hw, c, stats);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_norm_act_nhwc(const float* raw, const double* stats, const float* gamma, const float* beta,
                                 float eps, int relu, int n, int h, int w, int c,
                                 const float* residual,
                                 const float* warp_src, int src_batch, const float* T, int th, int tw, int align_corners,
                                 float* scale_shift_ws,
                                 float* y_f32, uint16_t* y_hi, uint16_t* y_lo, int lo_format,
                                 const float* post_scale, const float* post_shift, int post_relu, int res_step,
                                 int* range_flag, lwb_stream_t stream)
{
    LWB_CHECK_ARG(lo_format == 0 || (lo_format == 1 && (c % 64) == 0), "lo_format 1 (fp8 pairs) needs channels in blocks of 64");
    LWB_CHECK_ARG(raw, "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0 && c > 0 && (c % 8) == 0, "channels must be a multiple of 8");
    const bool affine = !stats && (gamma || beta);       // no statistics: y = x * gamma[c] + beta[c] (folded BatchNorm / bias)
    LWB_CHECK_ARG(!(stats || affine) || scale_shift_ws, "normalisation needs the scale/shift workspace [n,c,2] f32");
    LWB_CHECK_ARG(!warp_src || (T && th > 0 && tw > 0 && (src_batch == 1 || src_batch == n)), "bad warp arguments");
    LWB_CHECK_ARG(!warp_src || c >= 16, "the warp variant needs at least 16 channels");
    LWB_CHECK_ARG((post_scale == nullptr) == (post_shift == nullptr), "post_scale and post_shift go together");
    LWB_CHECK_ARG(res_step >= 0 && res_step <= 8, "bad residual step");
    if (res_step == 0) res_step = 1;
    const bool ext = post_scale != nullptr || res_step > 1;
    LWB_CHECK_ARG(!(ext && warp_src), "post-affine / strided residual are not combined with the warp");
    cudaStream_t st = (cudaStream_t)stream;
    if (stats) {
        LWB_CUDA_OK(lwb::launch_pdl(k_finalize_stats, dim3(lwb::ceil_div((long)n * c, 256)), dim3(256), 0, st,
                                    stats, gamma, beta, eps, n, c, 1.0 / ((double)h * w), (float2*)scale_shift_ws));
    } else if (affine) {
        LWB_CUDA_OK(lwb::launch_pdl(k_fill_ss, dim3(lwb::ceil_div((long)n * c, 256)), dim3(256), 0, st,
                                    gamma, beta, n, c, (float2*)scale_shift_ws));
    }
    NormActParams P;
    P.raw = raw; P.ss = (stats || affine) ? (const float2*)scale_shift_ws : nullptr; P.relu = relu;
    P.range_flag = range_flag; P.post_scale = post_scale; P.post_shift = post_shift; P.post_relu = post_relu; P.res_step = res_step;
    P.n = n; P.h = h; P.w = w; P.c = c;
    P.residual = residual;
    P.warp_src = warp_src; P.src_batch = src_batch; P.T = T; P.th = th; P.tw = tw; P.align_corners = align_corners;
    P.y_f32 = y_f32; P.y_hi = (__half*)y_hi; P.y_lo = (__half*)y_lo; P.lo_format = lo_format;
    const int groups = c / 8;
    LWB_CHECK_ARG(groups <= 256 && 256 % groups == 0, "channels / 8 must divide 256");
    const int px_per_block = (256 / groups) * kNormRounds;
    const long blocks = lwb::ceil_div((long)n * h * w, px_per_block);
    if (warp_src) LWB_CUDA_OK(lwb::launch_pdl(k_norm_act<true, false>, dim3((unsigned)blocks), dim3(256),
                                              px_per_block * sizeof(TapRec), st, P));
    else if (ext) LWB_CUDA_OK(lwb::launch_pdl(k_norm_act<false, true>, dim3((unsigned)blocks), dim3(256), 0, st, P));
    else          LWB_CUDA_OK(lwb::launch_pdl(k_norm_act<false, false>, dim3((unsigned)blocks), dim3(256), 0, st, P));
    return LWB_OK;
}

extern "C" int lwb_heads_composite(const float* raw, int n, int h, int w, int c_stride, int folded_kw,
                                   const float* bg, int bg_batch,
                                   float* color, float* mask, float* pred,
                                   float* pred_hwc, uint8_t* pred_u8_bgr, int* range_flag, lwb_stream_t stream)
{
    LWB_CHECK_ARG(raw, "null pointer");
    LWB_CHECK_ARG(bg || (!pred && !pred_hwc && !pred_u8_bgr), "the composite outputs need bg");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0 && c_stride >= 4 && (c_stride % 4) == 0, "bad sizes");
    LWB_CHECK_ARG(!bg || bg_batch == 1 || bg_batch == n, "bg_batch must be 1 or n");
    LWB_CHECK_ARG(folded_kw >= 0 && (folded_kw == 0 || ((folded_kw & 1) && folded_kw * 4 <= c_stride)), "bad folded_kw");
    LWB_CUDA_OK(lwb::launch_pdl(k_heads, dim3(lwb::ceil_div((long)n * h * w, 256)), dim3(256), 0, (cudaStream_t)stream,
                                raw, n, h * w, w, c_stride, folded_kw, bg, bg_batch, color, mask, pred, pred_hwc, pred_u8_bgr, range_flag));
    return LWB_OK;
}

extern "C" int lwb_frames_out(const float* frames, int n, int h, int w, float* hwc, uint8_t* u8_bgr, lwb_stream_t stream)
{
    LWB_CHECK_ARG(frames && (hwc || u8_bgr), "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0, "bad sizes");
    k_frames_out<<<lwb::ceil_div((long)n * h * w, 256), 256, 0, (cudaStream_t)stream>>>(frames, n, h * w, hwc, u8_bgr);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

// Resources of the HBM-bound kernels that run beside the convolutions of the other sub-batch stream: which = 0
// k_norm_act (plain), 1 k_norm_act<WARP> at c channels, 2 k_norm_act<EXT>, 3 k_heads, 4 k_nchw_to_nhwc_split.
// out: [registers per thread, static smem, dynamic smem, local bytes per thread, threads per block, blocks per SM alone].
template <typename F>
static int glue_resources(F* fn, int threads, int dyn_smem, int* out)
{
    cudaFuncAttributes a;
    LWB_CUDA_OK(cudaFuncGetAttributes(&a, fn));
    int blocks = 0;
    LWB_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, fn, threads, dyn_smem));
    out[0] = a.numRegs; out[1] = (int)a.sharedSizeBytes; out[2] = dyn_smem; out[3] = (int)a.localSizeBytes;
    out[4] = threads; out[5] = blocks;
    return LWB_OK;
}

extern "C" int lwb_glue_kernel_resources(int which, int c, int* out)
{
    LWB_CHECK_ARG(out, "null pointer");
    LWB_CHECK_ARG(which != 1 || (c >= 16 && c % 8 == 0 && 256 % (c / 8) == 0), "bad channel count");
    switch (which) {
        case 0: return glue_resources(k_norm_act<false, false>, 256, 0, out);
        case 1: return glue_resources(k_norm_act<true, false>, 256, (int)((256 / (c / 8)) * kNormRounds * sizeof(TapRec)), out);
        case 2: return glue_resources(k_norm_act<false, true>, 256, 0, out);
        case 3: return glue_resources(k_heads, 256, 0, out);
        case 4: return glue_resources(k_nchw_to_nhwc_split, 256, 0, out);
    }
    lwb::set_error("unknown kernel %d", which);
    return LWB_E_INVALID;
}
