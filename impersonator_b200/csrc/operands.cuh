// The operand formats of the conv engine (conv_tc.cu), for every kernel that writes its activations or weights:
//   fp16 hi / lo (lo_format 0)   hi = fp16(x), lo = fp16(x - hi), both [.., c_pad] like the fp32 tensor
//   fp8 pair blocks (lo_format 1, the lo of split = 2 plans)   hi as above; lo holds, per element row and 64-channel
//                                block, 64 bytes of the first e4m3 term then 64 bytes of the second (scales below)
//   the operand-range flag       LWB_RANGE_* bits (include/lwb_b200.h)
#pragma once
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>

#include "../../include/lwb_b200.h"

namespace lwb {

// x ~= hi + lo with hi = fp16(x), lo = fp16(x - hi): the 2-term operand split of the conv engine.
__device__ __forceinline__ void split_half(float x, __half& hi, __half& lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}

// fp8 scales of the "fp16 + fp8" operand split (conv_tc.cu, f8 mode).  With hi = fp16(v), lo = v - hi:
//     x * w ~= x_hi * w_hi + x * w_lo + x_lo * w            (the two small products only need ~4 bits)
// and everything is accumulated 2^E too large so that no fp8 operand underflows; E is chosen PER LAYER so that
// max|w| * 2^E lies in [2^14, 2^15) (lwb_conv_desc.w_exp; any weight magnitude packs without overflow):
//     A_hi = x_hi                           B_hi  = fp16(w_hi * 2^E)          (exact: a power of two)
//     A_lo8[0:64]   = e4m3(x * 2^-4)        B_lo8[0:64]   = e4m3(w_lo * 2^(E+4))     |.| <= 2^8
//     A_lo8[64:128] = e4m3(x_lo * 2^10)     B_lo8[64:128] = e4m3(w * 2^(E-10))       |.| <  2^5
// per 64-channel block (one 128 B K row); the epilogue multiplies by 2^-E.  Activation range: e4m3 saturates at 448,
// i.e. x_lo (<= half an fp16 ulp of x) clips for |x| >= 1024 and x itself for |x| >= 7168 -- the split then degrades
// gracefully towards single-pass fp16 for those elements; the activation writers report it through the range flag.
constexpr float kF8XScale = 1.f / 16.f, kF8XLoScale = 1024.f;
constexpr float kF8WLoRel = 16.f, kF8WRel = 1.f / 1024.f;       // relative to the layer's 2^E

__device__ __forceinline__ uint8_t to_e4m3(float v) { return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3); }

// The first term of channel ch of element i (i = row * c_pad + ch, c_pad % 64 == 0) in the pair blocks at lo; the second
// term is 64 bytes further.
__device__ __forceinline__ uint8_t* pair_block(void* lo, size_t i, int ch) {
    return static_cast<uint8_t*>(lo) + (i - ch) * 2 + (size_t)(ch / 64) * 128 + (ch % 64);
}

// The range bits of eight fp16 hi operands: LWB_RANGE_F8 from |hi| >= 1024, with LWB_RANGE_FP16 from |hi| >= 60000 or
// non-finite.  max |hi| is taken on the fp16 bits as integers (monotone in |x|; inf / NaN sort above everything).
__device__ __forceinline__ int range_bits(uint4 hv) {
    unsigned m = __vmaxu2(__vmaxu2(hv.x & 0x7fff7fffu, hv.y & 0x7fff7fffu), __vmaxu2(hv.z & 0x7fff7fffu, hv.w & 0x7fff7fffu));
    m = max(m & 0xffffu, m >> 16);
    return m >= 0x6400u ? (m >= 0x7b53u ? LWB_RANGE_F8 | LWB_RANGE_FP16 : LWB_RANGE_F8) : 0;      // fp16 1024.0 / 60000
}

// One element: y_f32[i] = v and / or the fp16 hi / lo pair at index i (each output nullable).
__device__ __forceinline__ void store_operand(float v, size_t i, float* y_f32, __half* y_hi, __half* y_lo) {
    if (y_f32) y_f32[i] = v;
    if (y_hi) {
        __half h, l;
        split_half(v, h, l);
        y_hi[i] = h;
        if (y_lo) y_lo[i] = l;
    }
}

// Eight consecutive channels of one element, encoded once and stored at one or more NHWC offsets.
struct Operand8 {
    uint4 hi;
    uint4 lo;        // lo_format 0: the fp16 lo; 1: x, y = the first pair-block term of the eight, z, w = the second
};

// The pair-block terms of v (eight channels) with its fp16 hi.
__device__ __forceinline__ uint4 pair8(const float* v, uint4 hi) {
    const __half* hh = reinterpret_cast<const __half*>(&hi);
    __align__(8) uint8_t x8[8];
    __align__(8) uint8_t l8[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        x8[k] = to_e4m3(v[k] * kF8XScale);
        l8[k] = to_e4m3((v[k] - __half2float(hh[k])) * kF8XLoScale);
    }
    const uint2 a = *reinterpret_cast<const uint2*>(x8), b = *reinterpret_cast<const uint2*>(l8);
    return make_uint4(a.x, a.y, b.x, b.y);
}

__device__ __forceinline__ Operand8 encode8(const float* v, int lo_format) {
    __align__(16) __half hh[8];
    __align__(16) __half ll[8];
#pragma unroll
    for (int k = 0; k < 8; k++) split_half(v[k], hh[k], ll[k]);
    Operand8 e;
    e.hi = *reinterpret_cast<const uint4*>(hh);
    e.lo = lo_format == 0 ? *reinterpret_cast<const uint4*>(ll) : pair8(v, e.hi);
    return e;
}

// e at offset off = row * c_pad + ch of y_hi and (nullable) y_lo; ch % 8 == 0.  With v given, e comes from
// encode8(v, 0) and the pair blocks are encoded here, after the hi is stored (fewer registers live in a kernel that
// stores each element once).
__device__ __forceinline__ void store8(const Operand8& e, const float* v, __half* y_hi, __half* y_lo, int lo_format,
                                       size_t off, int ch) {
    *reinterpret_cast<uint4*>(y_hi + off) = e.hi;
    if (y_lo && lo_format == 0) {
        *reinterpret_cast<uint4*>(y_lo + off) = e.lo;
    } else if (y_lo) {
        const uint4 p = v ? pair8(v, e.hi) : e.lo;
        uint8_t* blk = pair_block(y_lo, off, ch);
        *reinterpret_cast<uint2*>(blk) = make_uint2(p.x, p.y);
        *reinterpret_cast<uint2*>(blk + 64) = make_uint2(p.z, p.w);
    }
}

}  // namespace lwb
