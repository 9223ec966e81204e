// Rasterizer + fused correspondence pass (sm_90a).
//
// Replaces, with identical results, the reference's
//   thirdparty/neural_renderer/neural_renderer/cuda/rasterize_cuda_kernel.cu
//     :40-84   forward_face_index_map_cuda_kernel_1  (one thread per face)
//     :86-186  forward_face_index_map_cuda_kernel_2  (one thread per pixel, loops over ALL faces)
// and, in lwb_correspond, the torch glue around them (utils/nmr.py:10-28,263-278,328-341,617-659,
// rasterize.py:334-338, models/imitator.py:259-260).
//
// Design: instead of O(pixels x faces) the work is O(sum of per-face bounding boxes):
//   pass 1  one thread per (frame, face): project / gather the triangle, back-face cull, build
//           the 3x3 inverse, then visit only the pixels of its (conservative) bounding box and
//           z-test them with ONE 64-bit atomicMin per hit on a packed key (depth bits << 32 | face).
//           min over (depth, face index) == the reference's ascending scan with a strict '<'
//           (lowest face index wins ties).  Faces with a large box, or degenerate / sliver faces
//           (whose inside test is not confined to the box, see DESIGN.md), are handled by the
//           whole warp cooperatively, 32 pixels at a time.
//   pass 2  one thread per pixel: decode the winner, recompute its barycentric weights with the
//           same instruction sequence, and emit every per-pixel product in one coalesced sweep
//           (fim, wim, depth | cond, T, warped source image, concatenated generator input),
//           with the vertical flip folded into the store.
//
// Bit-exactness: every fp32 operation of the reference kernels is issued here with explicit
// round-to-nearest intrinsics in the contraction pattern nvcc 12.9 emits for the reference
// (read off its SASS, see DESIGN.md / oracle/raster_ref.c), so face_index_map is identical.
#include "common.cuh"

namespace {

constexpr int   kSmallBox   = 48;       // boxes up to this many pixels are walked by one thread
constexpr int   kBigBox     = 2048;     // boxes beyond this are walked by the whole grid (k_face_whole), not by one warp
constexpr float kSliverTol  = 1e-5f;
constexpr float kBoxMargin  = 0.02f;    // pixels added around the exact bounding box    // |det| / (longest edge)^2 below this -> whole-image scan

struct RasterParams {
    // geometry source: either faces [B,F,3,3] or (cam, verts, face_idx)
    const float*   faces;
    const float*   cam;
    const float*   verts;
    const int32_t* face_idx;
    int B, V, F, is;
    float nearv, farv, eye_z;
    unsigned long long* zbuf;           // [B,is,is] packed (depth bits << 32 | face)
    unsigned* qcount;                   // deferred whole-image faces: counter (0xFFFFFFFF = empty) ...
    unsigned* queue;                    // ... and entries (b * F + face), capacity B * F
    float* f2verts;                     // nullable [B,F,3,3]
    float* faces_inv;                   // nullable [B,F,3,3]
    // resolve outputs (raster API)
    int32_t* fim; float* wim; float* depth; int flip;
    // correspondence extras
    const float* map_fn; int map_c;
    const float* src_p2verts; const float* src_img; int src_batch; int align_corners;
    float* T; float* tsf_inputs;
};

template <bool FROM_VERTS>
__device__ __forceinline__ void load_face(const RasterParams& P, int b, int fn, float* f)
{
    if (FROM_VERTS) {
        // utils/nmr.py:10-28 (s*(X+t)), :271 (y *= -1), look_at.py:57-58 (v - eye; R = I)
        const float s = __ldg(P.cam + b * 3 + 0), tx = __ldg(P.cam + b * 3 + 1), ty = __ldg(P.cam + b * 3 + 2);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int vi = __ldg(P.face_idx + fn * 3 + k);
            const float* v = P.verts + ((size_t)b * P.V + vi) * 3;
            f[3 * k + 0] = __fmul_rn(s, __fadd_rn(__ldg(v + 0), tx));
            f[3 * k + 1] = -__fmul_rn(s, __fadd_rn(__ldg(v + 1), ty));
            f[3 * k + 2] = __fsub_rn(__fadd_rn(__ldg(v + 2), 0.0f), P.eye_z);
        }
    } else {
        const float* src = P.faces + ((size_t)b * P.F + fn) * 9;
#pragma unroll
        for (int k = 0; k < 9; k++) f[k] = __ldg(src + k);
    }
}

// rasterize_cuda_kernel.cu:57 / :128
__device__ __forceinline__ bool back_facing(const float* f)
{
    return __fmul_rn(__fsub_rn(f[7], f[1]), __fsub_rn(f[3], f[0])) <
           __fmul_rn(__fsub_rn(f[4], f[1]), __fsub_rn(f[6], f[0]));
}

// rasterize_cuda_kernel.cu:60-79 in nvcc's contraction pattern.  p[] = pixel-space x,y of the 3 verts.
__device__ __forceinline__ void face_setup(const float* f, int is, float* p, float* inv, float& det)
{
    const float fis = (float)is;
#pragma unroll
    for (int n = 0; n < 3; n++)
#pragma unroll
        for (int d = 0; d < 2; d++)
            p[2 * n + d] = __fmul_rn(__fadd_rn(__fmaf_rn(f[3 * n + d], fis, fis), -1.0f), 0.5f);
    const float p00 = p[0], p01 = p[1], p10 = p[2], p11 = p[3], p20 = p[4], p21 = p[5];
    float a[9];
    a[0] = __fsub_rn(p11, p21);
    a[1] = __fsub_rn(p20, p10);
    a[2] = __fmaf_rn(p10, p21, -__fmul_rn(p20, p11));
    a[3] = __fsub_rn(p21, p01);
    a[4] = __fsub_rn(p00, p20);
    a[5] = __fmaf_rn(p20, p01, -__fmul_rn(p00, p21));
    a[6] = __fsub_rn(p01, p11);
    a[7] = __fsub_rn(p10, p00);
    a[8] = __fmaf_rn(p00, p11, -__fmul_rn(p10, p01));
    det = __fmaf_rn(p10, __fsub_rn(p21, p01),
          __fmaf_rn(p20, __fsub_rn(p01, p11), __fmul_rn(p00, __fsub_rn(p11, p21))));
#pragma unroll
    for (int k = 0; k < 9; k++) inv[k] = __fdiv_rn(a[k], det);
}

// rasterize_cuda_kernel.cu:113-114: (float)((2.*i + 1 - is) / is), a double division rounded to float.
// Numerator and denominator are integers < 2^24, i.e. exact floats, and for such operands a
// correctly rounded double quotient rounded again to float equals the correctly rounded float
// quotient (53 >= 2*24 + 2), so one IEEE fp32 division reproduces it bit for bit -- without the
// two FP64 divisions per pixel test.
__device__ __forceinline__ float ndc_center(int i, int is) { return __fdiv_rn((float)(2 * i + 1 - is), (float)is); }

// rasterize_cuda_kernel.cu:132-134 (strict '<' rejects: a centre exactly on an edge is inside)
__device__ __forceinline__ bool inside(const float* f, float xp, float yp)
{
    if (__fmul_rn(__fsub_rn(yp, f[1]), __fsub_rn(f[3], f[0])) < __fmul_rn(__fsub_rn(xp, f[0]), __fsub_rn(f[4], f[1]))) return false;
    if (__fmul_rn(__fsub_rn(yp, f[4]), __fsub_rn(f[6], f[3])) < __fmul_rn(__fsub_rn(xp, f[3]), __fsub_rn(f[7], f[4]))) return false;
    if (__fmul_rn(__fsub_rn(yp, f[7]), __fsub_rn(f[0], f[6])) < __fmul_rn(__fsub_rn(xp, f[6]), __fsub_rn(f[1], f[7]))) return false;
    return true;
}

// rasterize_cuda_kernel.cu:139-151: w = inv * (xi, yi, 1), clamp to [0,1] (NaN -> 0), renormalise
__device__ __forceinline__ void bary_weights(const float* inv, int xi, int yi, float* w)
{
    const float fx = (float)xi, fy = (float)yi;
    float ws = 0.0f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float t = __fadd_rn(__fmaf_rn(inv[3 * k + 0], fx, __fmul_rn(inv[3 * k + 1], fy)), inv[3 * k + 2]);
        t = fminf(fmaxf(t, 0.0f), 1.0f);
        w[k] = t;
        ws = __fadd_rn(ws, t);
    }
#pragma unroll
    for (int k = 0; k < 3; k++) w[k] = __fdiv_rn(w[k], ws);
}

// rasterize_cuda_kernel.cu:153
__device__ __forceinline__ float persp_depth(const float* f, const float* w)
{
    return __frcp_rn(__fadd_rn(__fadd_rn(__fdiv_rn(w[0], f[2]), __fdiv_rn(w[1], f[5])), __fdiv_rn(w[2], f[8])));
}

__device__ __forceinline__ void test_pixel(const RasterParams& P, const float* f, const float* inv,
                                           int b, int fn, int xi, int yi)
{
    const float xp = ndc_center(xi, P.is), yp = ndc_center(yi, P.is);
    if (!inside(f, xp, yp)) return;
    float w[3];
    bary_weights(inv, xi, yi, w);
    const float zp = persp_depth(f, w);
    // :154-159  (zp <= near || far <= zp) -> skip; NaN fails every '<' and is skipped as well.
    if (zp > P.nearv && zp < P.farv) {
        const unsigned long long key = ((unsigned long long)__float_as_uint(zp) << 32) | (unsigned)fn;
        atomicMin(P.zbuf + ((size_t)b * P.is + yi) * P.is + xi, key);
    }
}

// Conservative pixel box of a non-degenerate face (see k_face_raster), or whole = true when the reference's inside test is not
// confined to the box (degenerate / sliver / non-finite faces).
__device__ __forceinline__ void face_box(const float* p, float det, int is, bool& whole, int& bx0, int& bx1, int& by0, int& by1)
{
    const float xmin = fminf(p[0], fminf(p[2], p[4])), xmax = fmaxf(p[0], fmaxf(p[2], p[4]));
    const float ymin = fminf(p[1], fminf(p[3], p[5])), ymax = fmaxf(p[1], fmaxf(p[3], p[5]));
    const float ex = fmaxf(xmax - xmin, ymax - ymin);
    bool finite = true;
#pragma unroll
    for (int k = 0; k < 6; k++) finite = finite && (fabsf(p[k]) < 1e30f);    // false for NaN / inf
    whole = !finite || !(fabsf(det) > kSliverTol * ex * ex);
    bx0 = by0 = 0; bx1 = by1 = -1;
    if (!whole) {
        bx0 = max(0, (int)ceilf(xmin - kBoxMargin)); bx1 = min(is - 1, (int)floorf(xmax + kBoxMargin));
        by0 = max(0, (int)ceilf(ymin - kBoxMargin)); by1 = min(is - 1, (int)floorf(ymax + kBoxMargin));
    }
}

template <bool FROM_VERTS>
__global__ void __launch_bounds__(256) k_face_raster(RasterParams P)
{
    const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = gid < (long)P.B * P.F;
    const int b = valid ? (int)(gid / P.F) : 0;
    const int fn = valid ? (int)(gid % P.F) : 0;
    const unsigned lane = threadIdx.x & 31;

    float f[9], inv[9];
    int bx0 = 0, bx1 = -1, by0 = 0, by1 = -1;
    int mode = 0;                               // 0 nothing, 1 this thread walks its box, 2 warp walks it
    if (valid) {
        load_face<FROM_VERTS>(P, b, fn, f);
        if (P.f2verts) {
            float* o = P.f2verts + (size_t)gid * 9;
#pragma unroll
            for (int k = 0; k < 9; k++) o[k] = f[k];
        }
        if (!back_facing(f)) {
            float p[6], det;
            face_setup(f, P.is, p, inv, det);
            if (P.faces_inv) {
                float* o = P.faces_inv + (size_t)gid * 9;
#pragma unroll
                for (int k = 0; k < 9; k++) o[k] = inv[k];
            }
            // Degenerate or sliver triangles: the reference's inside test is then not confined to the
            // bounding box (all three edge products can round to equality), so scan the whole image
            // exactly like the reference does.  Conservative box otherwise, in pixel-centre coordinates (pixel i has
            // p-coordinate exactly i): for a non-sliver triangle a rounding-induced false accept of the reference's edge
            // tests lies within ~1e-6 NDC (< 1e-3 px up to 2048^2) of the triangle; kBoxMargin absorbs that.
            bool whole;
            face_box(p, det, P.is, whole, bx0, bx1, by0, by1);
            const int area = whole ? 0 : max(0, bx1 - bx0 + 1) * max(0, by1 - by0 + 1);
            if (whole || area > kBigBox) {
                // deferred to k_face_whole, where the whole grid shares the scan of each such face (one warp walking a full
                // image -- or a face covering thousands of pixels -- would straggle for up to ~1 ms)
                const unsigned slot = atomicAdd(P.qcount, 1u) + 1u;          // counter starts at 0xFFFFFFFF
                P.queue[slot] = (unsigned)gid;
            } else if (area > 0) {
                mode = (area <= kSmallBox) ? 1 : 2;
            }
        }
    }
    if (mode == 1) {
        for (int yi = by0; yi <= by1; yi++)
            for (int xi = bx0; xi <= bx1; xi++)
                test_pixel(P, f, inv, b, fn, xi, yi);
    }
    unsigned pending = __ballot_sync(0xffffffffu, mode == 2);
    while (pending) {
        const int src = __ffs(pending) - 1;
        pending &= pending - 1;
        float g[9], ginv[9];
#pragma unroll
        for (int k = 0; k < 9; k++) { g[k] = __shfl_sync(0xffffffffu, f[k], src); ginv[k] = __shfl_sync(0xffffffffu, inv[k], src); }
        const int gx0 = __shfl_sync(0xffffffffu, bx0, src), gx1 = __shfl_sync(0xffffffffu, bx1, src);
        const int gy0 = __shfl_sync(0xffffffffu, by0, src), gy1 = __shfl_sync(0xffffffffu, by1, src);
        const int gb = __shfl_sync(0xffffffffu, b, src), gfn = __shfl_sync(0xffffffffu, fn, src);
        const int bw = gx1 - gx0 + 1, n = bw * (gy1 - gy0 + 1);
        for (int i = lane; i < n; i += 32)
            test_pixel(P, g, ginv, gb, gfn, gx0 + i % bw, gy0 + i / bw);
    }
}

// Faces whose inside test is not confined to their bounding box (degenerate / sliver / non-finite):
// the reference effectively tests them against every pixel, and so does this kernel -- spread over the
// whole grid: blockIdx.y strides over the queued faces, blockIdx.x over pixel chunks.  Ordinary faces with a box of more
// than kBigBox pixels are queued here too and scanned over their box only.
template <bool FROM_VERTS>
__global__ void __launch_bounds__(256) k_face_whole(RasterParams P)
{
    const unsigned count = *P.qcount + 1u;
    const int npix = P.is * P.is;
    for (unsigned slot = blockIdx.y; slot < count; slot += gridDim.y) {
        const unsigned gid = P.queue[slot];
        const int b = (int)(gid / (unsigned)P.F), fn = (int)(gid % (unsigned)P.F);
        float f[9], p[6], inv[9], det;
        load_face<FROM_VERTS>(P, b, fn, f);
        face_setup(f, P.is, p, inv, det);
        bool whole;
        int bx0, bx1, by0, by1;
        face_box(p, det, P.is, whole, bx0, bx1, by0, by1);
        if (whole) {
            for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += gridDim.x * blockDim.x)
                test_pixel(P, f, inv, b, fn, i % P.is, i / P.is);
        } else {                                             // a big ordinary face: only its box, spread over the x-blocks
            const int bw = bx1 - bx0 + 1, n = bw * (by1 - by0 + 1);
            for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
                test_pixel(P, f, inv, b, fn, bx0 + i % bw, by0 + i / bw);
        }
    }
}

// torch grid_sampler_2d (bilinear, zeros padding) coordinate un-normalisation
// (ATen/native/GridSampler.h:27-36): align_corners=False -> ((x+1)*size-1)/2, True -> (x+1)/2*(size-1)
__device__ __forceinline__ float unnormalize(float x, int size, int align_corners)
{
    return align_corners ? ((x + 1.f) / 2.f) * (float)(size - 1) : ((x + 1.f) * (float)size - 1.f) / 2.f;
}

template <bool FROM_VERTS, bool CORRESPOND>
__global__ void __launch_bounds__(256) k_resolve(RasterParams P)
{
    const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long npix = (long)P.B * P.is * P.is;
    if (gid >= npix) return;
    const int is = P.is;
    const int b = (int)(gid / ((long)is * is));
    const int pn = (int)(gid % ((long)is * is));
    const int r = pn / is, c = pn % is;                 // output coordinates
    const int yi = P.flip ? (is - 1 - r) : r;           // kernel row (row 0 = bottom)
    const unsigned long long key = P.zbuf[((size_t)b * is + yi) * is + c];
    const bool hit = key != ~0ull;
    int fn = -1;
    float w[3] = {0.f, 0.f, 0.f};
    if (hit) {
        fn = (int)(unsigned)(key & 0xffffffffull);
        float f[9], p[6], inv[9], det;
        load_face<FROM_VERTS>(P, b, fn, f);
        face_setup(f, is, p, inv, det);
        bary_weights(inv, c, yi, w);
    }
    if (!CORRESPOND) {
        // rasterize_cuda_kernel.cu:174-185: only covered pixels are written (caller pre-fills)
        if (hit) {
            P.fim[gid] = fn;
            P.wim[3 * gid + 0] = w[0]; P.wim[3 * gid + 1] = w[1]; P.wim[3 * gid + 2] = w[2];
            if (P.depth) P.depth[gid] = __uint_as_float((unsigned)(key >> 32));
        }
        return;
    }
    P.fim[gid] = fn;
    P.wim[3 * gid + 0] = w[0]; P.wim[3 * gid + 1] = w[1]; P.wim[3 * gid + 2] = w[2];
    // cal_bc_transform (utils/nmr.py:617-659): T = sum_k w_k * src_p2verts[fim, k, :], -2 elsewhere
    float tx = -2.f, ty = -2.f;
    const int sb = P.src_batch == 1 ? 0 : b;
    if (hit) {
        const float* q = P.src_p2verts + ((size_t)sb * P.F + fn) * 6;
        tx = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(q + 0), w[0]), __fmul_rn(__ldg(q + 2), w[1])), __fmul_rn(__ldg(q + 4), w[2]));
        ty = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(q + 1), w[0]), __fmul_rn(__ldg(q + 3), w[1])), __fmul_rn(__ldg(q + 5), w[2]));
    }
    reinterpret_cast<float2*>(P.T)[gid] = make_float2(tx, ty);
    if (!P.tsf_inputs) return;
    const size_t plane = (size_t)is * is;
    float* out = P.tsf_inputs + (size_t)b * (3 + P.map_c) * plane + pn;
    // models/imitator.py:259: tsf_img = F.grid_sample(src_img, T) over the whole image, background included: T = -2 there,
    // which still reaches pixel 0 at image sizes 1 and 2 with align_corners (and no pixel from size 3 on)
    float rgb[3] = {0.f, 0.f, 0.f};
    if (P.src_img) {
        const float ix = unnormalize(tx, is, P.align_corners), iy = unnormalize(ty, is, P.align_corners);
        const float x0f = floorf(ix), y0f = floorf(iy);
        const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
        const float wx1 = ix - x0f, wx0 = (x0f + 1.f) - ix, wy1 = iy - y0f, wy0 = (y0f + 1.f) - iy;
        const float* img = P.src_img + (size_t)sb * 3 * plane;
        const bool vx0 = x0 >= 0 && x0 < is, vx1 = x1 >= 0 && x1 < is, vy0 = y0 >= 0 && y0 < is, vy1 = y1 >= 0 && y1 < is;
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
            const float* pl = img + ch * plane;
            float acc = 0.f;
            if (vy0 && vx0) acc += __ldg(pl + y0 * is + x0) * (wx0 * wy0);
            if (vy0 && vx1) acc += __ldg(pl + y0 * is + x1) * (wx1 * wy0);
            if (vy1 && vx0) acc += __ldg(pl + y1 * is + x0) * (wx0 * wy1);
            if (vy1 && vx1) acc += __ldg(pl + y1 * is + x1) * (wx1 * wy1);
            rgb[ch] = acc;
        }
    }
#pragma unroll
    for (int ch = 0; ch < 3; ch++) out[ch * plane] = rgb[ch];
    // encode_fim (utils/nmr.py:336): cond = map_fn[fim]; fim == -1 indexes the last (background) row
    const float* row = P.map_fn + (size_t)(hit ? fn : P.F) * P.map_c;
    for (int k = 0; k < P.map_c; k++) out[(3 + k) * plane] = __ldg(row + k);
}

int run(RasterParams& P, bool from_verts, bool correspond, cudaStream_t st)
{
    const size_t zbytes = (size_t)P.B * P.is * P.is * sizeof(unsigned long long);
    P.qcount = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(P.zbuf) + zbytes);
    P.queue = P.qcount + 4;
    LWB_CUDA_OK(cudaMemsetAsync(P.zbuf, 0xff, zbytes + 16, st));      // z-buffer "empty" + queue counter "empty"
    const long nfaces = (long)P.B * P.F, npix = (long)P.B * P.is * P.is;
    const int t = 256;
    if (from_verts) k_face_raster<true><<<lwb::ceil_div(nfaces, t), t, 0, st>>>(P);
    else            k_face_raster<false><<<lwb::ceil_div(nfaces, t), t, 0, st>>>(P);
    LWB_LAUNCH_OK();
    if (from_verts) k_face_whole<true><<<dim3(64, 64), t, 0, st>>>(P);
    else            k_face_whole<false><<<dim3(64, 64), t, 0, st>>>(P);
    LWB_LAUNCH_OK();
    if (from_verts && correspond) k_resolve<true, true><<<lwb::ceil_div(npix, t), t, 0, st>>>(P);
    else if (!from_verts && !correspond) k_resolve<false, false><<<lwb::ceil_div(npix, t), t, 0, st>>>(P);
    else { lwb::set_error("raster: unsupported mode"); return LWB_E_INVALID; }
    LWB_LAUNCH_OK();
    return LWB_OK;
}

}  // namespace

extern "C" size_t lwb_raster_workspace_bytes(int batch, int image_size, int num_faces)
{
    if (batch <= 0 || image_size <= 0 || num_faces <= 0) return 0;
    // z-buffer + queue counter (16 B) + queue of deferred faces (worst case: every face)
    return (size_t)batch * image_size * image_size * sizeof(unsigned long long) + 16 + (size_t)batch * num_faces * sizeof(unsigned);
}

extern "C" int lwb_raster_forward_face_index_map(
        const float* faces, int batch, int num_faces, int image_size, float near, float far,
        int32_t* face_index_map, float* weight_map, float* depth_map, float* faces_inv,
        int flip_rows, void* workspace, lwb_stream_t stream)
{
    LWB_CHECK_ARG(faces && face_index_map && weight_map && workspace, "null pointer");
    LWB_CHECK_ARG(batch > 0 && num_faces > 0 && image_size > 0, "non-positive size");
    LWB_CHECK_ARG((long)batch * num_faces < (1l << 31) && (long)batch * image_size * image_size < (1l << 31), "too large");
    RasterParams P = {};
    P.faces = faces; P.B = batch; P.F = num_faces; P.is = image_size;
    P.nearv = near; P.farv = far;
    P.zbuf = (unsigned long long*)workspace;
    P.faces_inv = faces_inv;
    P.fim = face_index_map; P.wim = weight_map; P.depth = depth_map; P.flip = flip_rows ? 1 : 0;
    return run(P, false, false, (cudaStream_t)stream);
}

extern "C" int lwb_correspond(
        const float* cam, const float* verts, const int32_t* face_idx,
        int batch, int num_verts, int num_faces, int image_size, float near, float far, float eye_z,
        const float* map_fn, int map_c,
        const float* src_p2verts, const float* src_img, int src_batch, int align_corners,
        int32_t* fim, float* wim, float* T, float* tsf_inputs, float* f2verts,
        void* workspace, lwb_stream_t stream)
{
    LWB_CHECK_ARG(cam && verts && face_idx && fim && wim && T && workspace && src_p2verts, "null pointer");
    LWB_CHECK_ARG(batch > 0 && num_faces > 0 && num_verts > 0 && image_size > 0, "non-positive size");
    LWB_CHECK_ARG(src_batch == 1 || src_batch == batch, "src_batch must be 1 or batch");
    LWB_CHECK_ARG(!tsf_inputs || (map_fn && map_c > 0), "tsf_inputs needs map_fn");
    LWB_CHECK_ARG((long)batch * num_faces < (1l << 31) && (long)batch * image_size * image_size < (1l << 31), "too large");
    RasterParams P = {};
    P.cam = cam; P.verts = verts; P.face_idx = face_idx;
    P.B = batch; P.V = num_verts; P.F = num_faces; P.is = image_size;
    P.nearv = near; P.farv = far;
    P.eye_z = eye_z;   // utils/nmr.py:177 eye = [0, 0, -(1/tan(30 deg) + 1)] as float32 (look_at.py:33)
    P.zbuf = (unsigned long long*)workspace;
    P.f2verts = f2verts;
    P.fim = fim; P.wim = wim; P.flip = 1;
    P.map_fn = map_fn; P.map_c = map_c;
    P.src_p2verts = src_p2verts; P.src_img = src_img; P.src_batch = src_batch; P.align_corners = align_corners;
    P.T = T; P.tsf_inputs = tsf_inputs;
    return run(P, true, true, (cudaStream_t)stream);
}
