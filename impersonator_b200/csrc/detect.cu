// Kernels of the Mask R-CNN person detector (torchvision maskrcnn_resnet50_fpn in eval mode, as utils/detectors.py:25-85
// builds it).  The convolutions and fully connected layers run on the conv engine (conv_tc.cu); what is here is the
// rest: the input transform, the stem's max-pool, the bias / residual / ReLU passes between convs, the RPN's top-k and
// decode, batched NMS, multi-scale RoIAlign, the box and mask post-processing, paste_masks_in_image and the person pick.
//
// Everything works on fixed-size device buffers with device-side counts, so a whole forward pass needs no host sync.
// The discrete decisions (top-k order, NMS keep lists, RoI levels, mask paste) reproduce torchvision's CPU arithmetic
// operation by operation: explicit __f*_rn intrinsics where the CPU code performs separately rounded operations, so
// nvcc cannot contract them into FMAs.
#include <string.h>

#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "operands.cuh"

namespace {

constexpr int kNmsBlock = 64;

__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }

// float -> unsigned key with the same order (larger float, larger key).  -0 maps to +0's key: the CPU's stable sort
// compares them equal and keeps index order between them.
__device__ __forceinline__ unsigned int order_key(float f)
{
    const unsigned int u = __float_as_uint(f == 0.f ? 0.f : f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

using lwb::store_operand;

// ---- GeneralizedRCNNTransform: (x + 1) / 2, normalise, bilinear resize (align_corners=False), zero pad ----------------
__global__ void k_det_transform(const float* __restrict__ img, int h, int w, int ho, int wo, int hp, int wp, float sy, float sx,
                                float* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * hp * wp) return;
    const int x = i % wp, y = (i / wp) % hp, c = i / (wp * hp);
    const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
    float v = 0.f;
    if (y < ho && x < wo) {
        const float ry = fmaxf(sy * ((float)y + 0.5f) - 0.5f, 0.f), rx = fmaxf(sx * ((float)x + 0.5f) - 0.5f, 0.f);
        const int y0 = min((int)floorf(ry), h - 1), x0 = min((int)floorf(rx), w - 1);
        const float ly = fminf(fmaxf(ry - (float)y0, 0.f), 1.f), lx = fminf(fmaxf(rx - (float)x0, 0.f), 1.f);
        const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
        const float* p = img + (size_t)c * h * w;
        auto px = [&](int yy, int xx) { return ((__ldg(p + (size_t)yy * w + xx) + 1.f) / 2.f - mean[c]) / stdv[c]; };
        v = (px(y0, x0) * (1.f - lx) + px(y0, x1) * lx) * (1.f - ly) + (px(y1, x0) * (1.f - lx) + px(y1, x1) * lx) * ly;
    }
    out[i] = v;
}

// ---- stem: max_pool2d(relu(x * scale + shift), 3, 2, padding=1), NCHW fp32 -> NHWC conv operands ----------------------
__global__ void k_det_stem_pool(const float* __restrict__ x, int n, int c, int h, int w, const float* __restrict__ scale,
                                const float* __restrict__ shift, int ho, int wo, __half* __restrict__ y_hi, __half* __restrict__ y_lo)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n * ho * wo * c) return;
    const int ch = (int)(i % c);
    const long pix = i / c;
    const int ox = (int)(pix % wo), oy = (int)((pix / wo) % ho), b = (int)(pix / ((long)wo * ho));
    const float* p = x + ((size_t)b * c + ch) * h * w;
    const float sc = scale[ch], sh = shift[ch];
    float m = -INFINITY;
    for (int dy = -1; dy <= 1; dy++) {
        const int yy = oy * 2 + dy;
        if (yy < 0 || yy >= h) continue;
        for (int dx = -1; dx <= 1; dx++) {
            const int xx = ox * 2 + dx;
            if (xx < 0 || xx >= w) continue;
            m = fmaxf(m, fmaxf(__ldg(p + (size_t)yy * w + xx) * sc + sh, 0.f));
        }
    }
    store_operand(m, (size_t)i, nullptr, y_hi, y_lo);
}

// ---- y = act(raw[step * (y, x)] (+ raw2) (+ bias) (+ res | nearest-2x res)) -> fp32 and / or conv operands --------------
__global__ void k_det_bias_act(const float* __restrict__ raw, int ld_raw, const float* __restrict__ raw2, const float* __restrict__ bias,
                               const float* __restrict__ res, int res_half, int step, int h_in, int w_in, int relu,
                               int n, int h, int w, int c, float* __restrict__ y_f32, __half* __restrict__ y_hi, __half* __restrict__ y_lo)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n * h * w * c) return;
    const int ch = (int)(i % c);
    const long pix = i / c;
    const int x = (int)(pix % w), y = (int)((pix / w) % h), b = (int)(pix / ((long)w * h));
    const size_t src = (((size_t)b * h_in + (size_t)y * step) * w_in + (size_t)x * step) * ld_raw + ch;
    float v = raw[src];
    if (raw2) v = add(v, raw2[src]);
    if (bias) v = add(v, bias[ch]);
    if (res) {
        const size_t r = res_half ? ((((size_t)b * (h / 2) + y / 2) * (w / 2) + x / 2) * c + ch) : (size_t)i;
        v = add(v, res[r]);
    }
    if (relu) v = fmaxf(v, 0.f);
    store_operand(v, (size_t)i, y_f32, y_hi, y_lo);
}

// ---- ConvTranspose2d(k=2, s=2) from its 1x1 form: raw [n,h,w,4c] (column (dy*2+dx)*c + co) -> relu(. + bias) at 2x -----
__global__ void k_det_d2s_bias_relu(const float* __restrict__ raw, const float* __restrict__ bias, int n, int h, int w, int c,
                                    float* __restrict__ y_f32, __half* __restrict__ y_hi, __half* __restrict__ y_lo)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n * 4 * h * w * c) return;
    const int co = (int)(i % c);
    const long pix = i / c;
    const int X = (int)(pix % (2 * w)), Y = (int)((pix / (2 * w)) % (2 * h)), b = (int)(pix / (4L * w * h));
    const int ph = (Y & 1) * 2 + (X & 1);
    const float v = fmaxf(add(raw[(((size_t)b * h + Y / 2) * w + X / 2) * 4 * c + ph * c + co], bias[co]), 0.f);
    store_operand(v, (size_t)i, y_f32, y_hi, y_lo);
}

// ---- BoxCoder.decode_single for one box (torchvision det_utils), separately rounded as on the CPU ---------------------
__device__ __forceinline__ void decode_box(const float* anc, float d0, float d1, float d2, float d3, float wx, float wy,
                                           float ww, float wh, float clip, float* out)
{
    const float widths = sub(anc[2], anc[0]), heights = sub(anc[3], anc[1]);
    const float cx = add(anc[0], mul(0.5f, widths)), cy = add(anc[1], mul(0.5f, heights));
    const float dx = dvd(d0, wx), dy = dvd(d1, wy);
    const float dw = fminf(dvd(d2, ww), clip), dh = fminf(dvd(d3, wh), clip);
    const float pcx = add(mul(dx, widths), cx), pcy = add(mul(dy, heights), cy);
    const float pw = mul(expf(dw), widths), ph = mul(expf(dh), heights);
    const float hw = mul(0.5f, pw), hh = mul(0.5f, ph);
    out[0] = sub(pcx, hw); out[1] = sub(pcy, hh); out[2] = add(pcx, hw); out[3] = add(pcy, hh);
}

__device__ __forceinline__ void clip_box(float* b, float ch, float cw)
{
    b[0] = fminf(fmaxf(b[0], 0.f), cw); b[2] = fminf(fmaxf(b[2], 0.f), cw);
    b[1] = fminf(fmaxf(b[1], 0.f), ch); b[3] = fminf(fmaxf(b[3], 0.f), ch);
}

// ---- RPN, one level per block: top-k of the objectness logits (radix select, ties to the lower index, sorted), then
// decode against the anchors, clip, small-box filter, sigmoid.  head: [gh*gw, 16] raw 1x1-head output, columns 0..2
// logits, 3 + a*4 + k deltas; anchors in (y, x, a) order.
constexpr int kRpnThreads = 1024, kRpnMaxK = 1024;

struct RpnLevel {
    const float* head;
    int gh, gw, stride_h, stride_w, offset;    // offset of the level's candidates in the concatenated arrays
    float cell[12];                            // rounded cell anchors, 3 x (x0, y0, x1, y1)
};
struct RpnArgs {
    RpnLevel lv[5];
    int k;
    float clip_h, clip_w, min_size, xform_clip;
};

__global__ void __launch_bounds__(kRpnThreads) k_det_rpn_level(RpnArgs A, const float* __restrict__ bias, int* __restrict__ top_out,
                                                               float* __restrict__ boxes, float* __restrict__ scores,
                                                               int* __restrict__ groups, int* __restrict__ valid)
{
    const RpnLevel& L = A.lv[blockIdx.x];
    const int n = L.gh * L.gw * 3;
    const int k = min(A.k, n);
    __shared__ unsigned int hist[256];
    __shared__ unsigned int s_prefix, s_need;
    __shared__ int s_nsel;
    __shared__ int sel[kRpnMaxK];
    __shared__ unsigned int selkey[kRpnMaxK];
    __shared__ int sorted[kRpnMaxK];
    typedef cub::BlockScan<int, kRpnThreads> Scan;
    __shared__ typename Scan::TempStorage scan_tmp;
    auto key_of = [&](int i) { return order_key(add(L.head[(size_t)(i / 3) * 16 + i % 3], bias[i % 3])); };

    // radix select of the k-th largest key: prefix / mask narrow from the top byte down
    unsigned int prefix = 0, mask = 0, need = (unsigned int)k;
    if (k < n) {
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int j = threadIdx.x; j < 256; j += blockDim.x) hist[j] = 0;
            __syncthreads();
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const unsigned int key = key_of(i);
                if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                unsigned int acc = 0, d = 255;
                for (int j = 255; j >= 0; j--) {
                    if (acc + hist[j] >= need) { d = (unsigned int)j; break; }
                    acc += hist[j];
                }
                s_prefix = prefix | (d << shift);
                s_need = need - acc;
            }
            __syncthreads();
            prefix = s_prefix; need = s_need; mask |= 255u << shift;
            __syncthreads();
        }
    }
    // gather: every key above the threshold, then the first `need` (lowest index) equal to it
    if (threadIdx.x == 0) s_nsel = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned int key = key_of(i);
        if (k == n || key > prefix) { const int s = atomicAdd(&s_nsel, 1); sel[s] = i; selkey[s] = key; }
    }
    __syncthreads();
    if (k < n) {
        const int base0 = s_nsel;
        int taken = 0;
        for (int start = 0; start < n && taken < (int)need; start += blockDim.x) {
            const int i = start + threadIdx.x;
            const int flag = (i < n && key_of(i) == prefix) ? 1 : 0;
            int pos, total;
            Scan(scan_tmp).ExclusiveSum(flag, pos, total);
            if (flag && taken + pos < (int)need) { sel[base0 + taken + pos] = i; selkey[base0 + taken + pos] = prefix; }
            taken += total;
            __syncthreads();
        }
    }
    __syncthreads();
    // sort the k selected by (key desc, index asc): rank counting
    for (int s = threadIdx.x; s < k; s += blockDim.x) {
        const unsigned int ks = selkey[s];
        const int is = sel[s];
        int r = 0;
        for (int m = 0; m < k; m++) {
            const unsigned int km = selkey[m];
            r += (km > ks || (km == ks && sel[m] < is)) ? 1 : 0;
        }
        sorted[r] = is;
    }
    __syncthreads();
    for (int r = threadIdx.x; r < k; r += blockDim.x) {
        const int i = sorted[r], p = i / 3, a = i % 3;
        const float* hd = L.head + (size_t)p * 16;
        const float sx = (float)((p % L.gw) * L.stride_w), sy = (float)((p / L.gw) * L.stride_h);
        const float anc[4] = {add(sx, L.cell[a * 4 + 0]), add(sy, L.cell[a * 4 + 1]), add(sx, L.cell[a * 4 + 2]), add(sy, L.cell[a * 4 + 3])};
        float b[4];
        decode_box(anc, add(hd[3 + a * 4 + 0], bias[3 + a * 4 + 0]), add(hd[3 + a * 4 + 1], bias[3 + a * 4 + 1]),
                   add(hd[3 + a * 4 + 2], bias[3 + a * 4 + 2]), add(hd[3 + a * 4 + 3], bias[3 + a * 4 + 3]),
                   1.f, 1.f, 1.f, 1.f, A.xform_clip, b);
        clip_box(b, A.clip_h, A.clip_w);
        const float logit = add(hd[a], bias[a]);
        const float sc = 1.f / (1.f + expf(-logit));
        const int o = L.offset + r;
        if (top_out) top_out[o] = i;
        for (int q = 0; q < 4; q++) boxes[(size_t)o * 4 + q] = b[q];
        scores[o] = sc;
        groups[o] = blockIdx.x;
        valid[o] = (sub(b[2], b[0]) >= A.min_size && sub(b[3], b[1]) >= A.min_size && sc >= 0.f) ? 1 : 0;
    }
}

// ---- batched NMS (torchvision's vanilla branch: one greedy NMS per group, kept boxes by descending score) -------------
// 1. compact the valid slots; 2. rank by (score desc, slot asc) and gather sorted boxes; 3. IoU bitmask over same-group
// pairs (j after i); 4. one warp sweeps the sorted list.
__global__ void k_nms_compact(const int* __restrict__ valid, int n, int m_max, int* __restrict__ comp, int* __restrict__ count)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (valid == nullptr || valid[i])) {
        const int s = atomicAdd(count, 1);
        if (s < m_max) comp[s] = i;
    }
}

__global__ void k_nms_rank(const int* __restrict__ comp, const int* __restrict__ count, int m_max, const float* __restrict__ scores,
                           const float* __restrict__ boxes, const int* __restrict__ groups, int* __restrict__ order,
                           float* __restrict__ sboxes, int* __restrict__ sgroups)
{
    const int m = min(*count, m_max);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    __shared__ float ts[256];
    __shared__ int ti[256];
    int slot = -1;
    float s = 0.f;
    if (j < m) { slot = comp[j]; s = scores[slot]; }
    int r = 0;
    for (int t0 = 0; t0 < m; t0 += 256) {
        __syncthreads();
        if (t0 + (int)threadIdx.x < m) { const int q = comp[t0 + threadIdx.x]; ti[threadIdx.x] = q; ts[threadIdx.x] = scores[q]; }
        __syncthreads();
        if (j < m) {
            const int lim = min(256, m - t0);
            for (int u = 0; u < lim; u++) r += (ts[u] > s || (ts[u] == s && ti[u] < slot)) ? 1 : 0;
        }
    }
    if (j < m) {
        order[r] = slot;
        for (int q = 0; q < 4; q++) sboxes[(size_t)r * 4 + q] = boxes[(size_t)slot * 4 + q];
        sgroups[r] = groups ? groups[slot] : 0;
    }
}

__device__ __forceinline__ float box_area(const float* b) { return mul(sub(b[2], b[0]), sub(b[3], b[1])); }

// torchvision nms_kernel.cpp: IoU = inter / (area_i + area_j - inter), suppress when > thresh
__device__ __forceinline__ bool iou_above(const float* a, const float* b, float thresh)
{
    const float w = fmaxf(0.f, sub(fminf(a[2], b[2]), fmaxf(a[0], b[0])));
    const float h = fmaxf(0.f, sub(fminf(a[3], b[3]), fmaxf(a[1], b[1])));
    const float inter = mul(w, h);
    return dvd(inter, sub(add(box_area(a), box_area(b)), inter)) > thresh;
}

__global__ void k_nms_mask(const int* __restrict__ count, int m_max, const float* __restrict__ sboxes, const int* __restrict__ sgroups,
                           float thresh, int col_blocks, unsigned long long* __restrict__ mask)
{
    const int m = min(*count, m_max);
    const int rb = blockIdx.y, cb = blockIdx.x;
    if (rb * kNmsBlock >= m || cb < rb || cb * kNmsBlock >= m) return;
    __shared__ float cbox[kNmsBlock * 4];
    __shared__ int cgrp[kNmsBlock];
    const int ncols = min(kNmsBlock, m - cb * kNmsBlock);
    if ((int)threadIdx.x < ncols) {
        for (int q = 0; q < 4; q++) cbox[threadIdx.x * 4 + q] = sboxes[(size_t)(cb * kNmsBlock + threadIdx.x) * 4 + q];
        cgrp[threadIdx.x] = sgroups[cb * kNmsBlock + threadIdx.x];
    }
    __syncthreads();
    const int i = rb * kNmsBlock + threadIdx.x;
    if (i >= m) return;
    const float* bi = sboxes + (size_t)i * 4;
    const int gi = sgroups[i];
    unsigned long long bits = 0;
    for (int t = (cb == rb ? threadIdx.x + 1 : 0); t < ncols; t++)
        if (cgrp[t] == gi && iou_above(bi, cbox + t * 4, thresh)) bits |= 1ull << t;
    mask[(size_t)i * col_blocks + cb] = bits;
}

__global__ void k_nms_sweep(const int* __restrict__ count, int m_max, const int* __restrict__ order, const float* __restrict__ sboxes,
                            const int* __restrict__ sgroups, const float* __restrict__ scores, const unsigned long long* __restrict__ mask,
                            int col_blocks, int max_keep, int* __restrict__ keep, float* __restrict__ out_boxes,
                            float* __restrict__ out_scores, int* __restrict__ out_groups, int* __restrict__ out_count)
{
    extern __shared__ unsigned long long removed[];
    const int m = min(*count, m_max), lane = threadIdx.x;
    for (int w = lane; w < col_blocks; w += 32) removed[w] = 0;
    __syncwarp();
    int nk = 0;
    for (int i = 0; i < m && nk < max_keep; i++) {
        const bool gone = (removed[i / 64] >> (i % 64)) & 1ull;
        __syncwarp();
        if (gone) continue;
        if (lane == 0) {
            keep[nk] = order[i];
            if (out_boxes) for (int q = 0; q < 4; q++) out_boxes[nk * 4 + q] = sboxes[(size_t)i * 4 + q];
            if (out_scores) out_scores[nk] = scores[order[i]];
            if (out_groups) out_groups[nk] = sgroups[i];
        }
        const unsigned long long* row = mask + (size_t)i * col_blocks;
        for (int w = i / 64 + lane; w < col_blocks && w * 64 < m; w += 32) removed[w] |= row[w];
        __syncwarp();
        nk++;
    }
    for (int r = nk + lane; r < max_keep; r += 32) {
        keep[r] = -1;
        if (out_boxes) for (int q = 0; q < 4; q++) out_boxes[r * 4 + q] = 0.f;
        if (out_scores) out_scores[r] = 0.f;
        if (out_groups) out_groups[r] = 0;
    }
    if (lane == 0) *out_count = nk;
}

// ---- MultiScaleRoIAlign (torchvision roi_align CPU arithmetic, aligned=False) -> RoI-major NHWC --------------------------
struct Pyramid { const float* p[4]; int h[4], w[4]; };

__device__ __forceinline__ int roi_level(const float* b)
{
    const float s = sqrtf(box_area(b));
    const float lv = floorf(add(add(4.f, log2f(dvd(s, 224.f))), 1e-6f));
    return (int)fminf(fmaxf(lv, 2.f), 5.f) - 2;
}

__global__ void k_det_roi_align(Pyramid P, int c, const float* __restrict__ boxes, const int* __restrict__ count, int r_max,
                                int out, int sampling, int* __restrict__ levels, float* __restrict__ y_f32,
                                __half* __restrict__ y_hi, __half* __restrict__ y_lo)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)r_max * out * out * c) return;
    const int ch = (int)(i % c);
    const long bin = i / c;
    const int pw = (int)(bin % out), ph = (int)((bin / out) % out), r = (int)(bin / ((long)out * out));
    float v = 0.f;
    const int n = count ? *count : r_max;
    if (r < n) {
        const float* b = boxes + (size_t)r * 4;
        const int l = roi_level(b);
        if (levels && ph == 0 && pw == 0 && ch == 0) levels[r] = l;
        const float scale = ldexpf(1.f, -(l + 2));
        const int H = P.h[l], W = P.w[l];
        const float* f = P.p[l] + ch;
        const float x1 = mul(b[0], scale), y1 = mul(b[1], scale), x2 = mul(b[2], scale), y2 = mul(b[3], scale);
        const float rw = fmaxf(sub(x2, x1), 1.f), rh = fmaxf(sub(y2, y1), 1.f);
        const float bw = dvd(rw, (float)out), bh = dvd(rh, (float)out);
        const float g = (float)sampling;
        for (int iy = 0; iy < sampling; iy++) {
            float y = add(add(y1, mul((float)ph, bh)), dvd(mul((float)iy + 0.5f, bh), g));
            for (int ix = 0; ix < sampling; ix++) {
                float x = add(add(x1, mul((float)pw, bw)), dvd(mul((float)ix + 0.5f, bw), g));
                float yy = y, xx = x;
                if (yy < -1.f || yy > (float)H || xx < -1.f || xx > (float)W) continue;
                if (yy <= 0.f) yy = 0.f;
                if (xx <= 0.f) xx = 0.f;
                int yl = (int)yy, xl = (int)xx, yh, xh;
                if (yl >= H - 1) { yh = yl = H - 1; yy = (float)yl; } else yh = yl + 1;
                if (xl >= W - 1) { xh = xl = W - 1; xx = (float)xl; } else xh = xl + 1;
                const float ly = sub(yy, (float)yl), lx = sub(xx, (float)xl), hy = sub(1.f, ly), hx = sub(1.f, lx);
                const float t = add(add(add(mul(mul(hy, hx), f[((size_t)yl * W + xl) * c]), mul(mul(hy, lx), f[((size_t)yl * W + xh) * c])),
                                        mul(mul(ly, hx), f[((size_t)yh * W + xl) * c])), mul(mul(ly, lx), f[((size_t)yh * W + xh) * c]));
                v = add(v, t);
            }
        }
        v = dvd(v, (float)(sampling * sampling));
    }
    store_operand(v, (size_t)i, y_f32, y_hi, y_lo);
}

// ---- RoIHeads.postprocess_detections, candidate stage: softmax, per-class decode (10, 10, 5, 5), clip, > score, >= size.
// One warp per RoI; slot r * (nc - 1) + (j - 1) keeps torchvision's (RoI, class) order.
__global__ void k_det_box_candidates(const float* __restrict__ pred, int ld, int nc, const float* __restrict__ props,
                                     const int* __restrict__ count, int r_max, float clip_h, float clip_w, float score_thresh,
                                     float min_size, float xform_clip, float* __restrict__ boxes, float* __restrict__ scores,
                                     int* __restrict__ groups, int* __restrict__ valid)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= r_max) return;
    const int r = warp;
    const bool live = r < *count;
    const float* lg = pred + (size_t)r * ld;
    float mx = -INFINITY;
    for (int j = lane; j < nc; j += 32) mx = fmaxf(mx, lg[j]);
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < nc; j += 32) sum += expf(lg[j] - mx);
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    for (int j = 1 + lane; j < nc; j += 32) {
        const size_t s = (size_t)r * (nc - 1) + (j - 1);
        const float sc = expf(lg[j] - mx) / sum;
        const float* d = lg + nc + j * 4;
        float b[4];
        decode_box(props + (size_t)r * 4, d[0], d[1], d[2], d[3], 10.f, 10.f, 5.f, 5.f, xform_clip, b);
        clip_box(b, clip_h, clip_w);
        for (int q = 0; q < 4; q++) boxes[s * 4 + q] = b[q];
        scores[s] = sc;
        groups[s] = j;
        valid[s] = (live && sc > score_thresh && sub(b[2], b[0]) >= min_size && sub(b[3], b[1]) >= min_size) ? 1 : 0;
    }
}

// ---- maskrcnn_inference: sigmoid of the label's channel ------------------------------------------------------------
__global__ void k_det_mask_probs(const float* __restrict__ raw, int ld, const float* __restrict__ bias, const int* __restrict__ labels,
                                 const int* __restrict__ count, int d_max, int hw, float* __restrict__ logits, float* __restrict__ probs)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d_max * hw) return;
    const int d = i / hw;
    float l = 0.f, p = 0.f;
    if (d < *count) {
        const int lab = labels[d];
        l = add(raw[(size_t)i * ld + lab], bias[lab]);
        p = 1.f / (1.f + expf(-l));
    }
    if (logits) logits[i] = l;
    probs[i] = p;
}

// ---- transform.postprocess: resize_boxes + paste_masks_in_image (padding 1) ------------------------------------------
// F.interpolate(bilinear, align_corners=False) as ATen's CPU kernel computes it (see tests: bit-identical to it).
__device__ __forceinline__ void interp_index(int o, int in, int outn, int& i0, int& i1, float& l0, float& l1)
{
    if (outn == in) { i0 = i1 = o; l0 = 1.f; l1 = 0.f; return; }
    const float scale = dvd((float)in, (float)outn);
    float src = __fmaf_rn(scale, add((float)o, 0.5f), -0.5f);
    if (src < 0.f) src = 0.f;
    i0 = min((int)floorf(src), in - 1);
    l1 = fminf(fmaxf(sub(src, (float)i0), 0.f), 1.f);
    i1 = i0 + (i0 < in - 1 ? 1 : 0);
    l0 = sub(1.f, l1);
}

__global__ void k_det_paste(const float* __restrict__ probs, int M, const float* __restrict__ boxes, const int* __restrict__ count,
                            int d_max, float rh, float rw, int H, int W, float* __restrict__ masks, float* __restrict__ out_boxes)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)d_max * H * W) return;
    const int x = (int)(i % W), y = (int)((i / W) % H), d = (int)(i / ((long)W * H));
    float v = 0.f;
    const bool live = d < *count;
    const float* bb = boxes + (size_t)d * 4;
    const float b[4] = {mul(bb[0], rw), mul(bb[1], rh), mul(bb[2], rw), mul(bb[3], rh)};
    if (x == 0 && y == 0) for (int q = 0; q < 4; q++) out_boxes[d * 4 + q] = live ? b[q] : 0.f;
    if (live) {
        const float scale = (float)((double)(M + 2) / M);
        const float wh = mul(mul(sub(b[2], b[0]), 0.5f), scale), hh = mul(mul(sub(b[3], b[1]), 0.5f), scale);
        const float xc = mul(add(b[2], b[0]), 0.5f), yc = mul(add(b[3], b[1]), 0.5f);
        const long long e0 = (long long)sub(xc, wh), e1 = (long long)sub(yc, hh), e2 = (long long)add(xc, wh), e3 = (long long)add(yc, hh);
        const long long w = max(e2 - e0 + 1, 1LL), h = max(e3 - e1 + 1, 1LL);
        const long long x0 = max(e0, 0LL), x1 = min(e2 + 1, (long long)W), y0 = max(e1, 0LL), y1 = min(e3 + 1, (long long)H);
        if (x >= x0 && x < x1 && y >= y0 && y < y1) {
            const int P = M + 2;
            int a0, a1, c0, c1;
            float la0, la1, lc0, lc1;
            interp_index((int)(y - e1), P, (int)h, a0, a1, la0, la1);
            interp_index((int)(x - e0), P, (int)w, c0, c1, lc0, lc1);
            const float* pm = probs + (size_t)d * M * M;
            auto at = [&](int yy, int xx) { return (yy >= 1 && yy <= M && xx >= 1 && xx <= M) ? pm[(yy - 1) * M + (xx - 1)] : 0.f; };
            const float t0 = __fmaf_rn(at(a0, c1), lc1, mul(at(a0, c0), lc0));
            const float t1 = __fmaf_rn(at(a1, c1), lc1, mul(at(a1, c0), lc0));
            v = __fmaf_rn(t1, la1, mul(t0, la0));
        }
    }
    if (masks) masks[i] = v;
}

// ---- PersonMaskRCNNDetector.get_bbox_max_ids + (mask > threshold) + morph(dilate, ks) ------------------------------
__device__ int person_pick(const float* boxes, const int* labels, int n, int person)
{
    int pid = -1;
    float best = -1.f;
    for (int d = 0; d < n; d++) {
        if (labels[d] != person) continue;
        const float* b = boxes + d * 4;
        const float a = fabsf(mul(sub(b[2], b[0]), sub(b[3], b[1])));
        if (a > best) { best = a; pid = d; }
    }
    return pid < 0 ? n - 1 : pid;                 // the reference's bboxs[-1] when no person was found
}

__global__ void k_det_person_mask(const float* __restrict__ boxes, const int* __restrict__ labels, const int* __restrict__ count,
                                  int person, const float* __restrict__ masks, int H, int W, float thresh, int ks,
                                  int* __restrict__ pid_out, float* __restrict__ box_out, float* __restrict__ out)
{
    __shared__ int s_pid;
    const int n = *count;
    if (threadIdx.x == 0) s_pid = n > 0 ? person_pick(boxes, labels, n, person) : -1;
    __syncthreads();
    const int pid = s_pid;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        *pid_out = pid;
        for (int q = 0; q < 4; q++) box_out[q] = pid >= 0 ? boxes[pid * 4 + q] : 0.f;
    }
    if (i >= H * W) return;
    const int x = i % W, y = i / W;
    float v = 0.f;
    if (pid >= 0) {
        const float* m = masks + (size_t)pid * H * W;
        if (ks > 0) {
            const int pad = ks / 2;
            for (int dy = 0; dy < ks && v == 0.f; dy++) {
                const int yy = y + dy - pad;
                if (yy < 0 || yy >= H) continue;
                for (int dx = 0; dx < ks; dx++) {
                    const int xx = x + dx - pad;
                    if (xx >= 0 && xx < W && m[(size_t)yy * W + xx] > thresh) { v = 1.f; break; }
                }
            }
        } else {
            v = m[i] > thresh ? 1.f : 0.f;
        }
    }
    out[i] = v;
}

}  // namespace

// =====================================================================================================================
extern "C" int lwb_det_transform(const float* img, int h, int w, int ho, int wo, int hp, int wp, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(img && out, "null pointer");
    LWB_CHECK_ARG(h > 0 && w > 0 && ho > 0 && wo > 0 && hp >= ho && wp >= wo, "bad sizes");
    const float sy = (float)h / (float)ho, sx = (float)w / (float)wo;
    k_det_transform<<<lwb::ceil_div(3L * hp * wp, 256), 256, 0, (cudaStream_t)stream>>>(img, h, w, ho, wo, hp, wp, sy, sx, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_stem_pool(const float* x, int n, int c, int h, int w, const float* scale, const float* shift,
                                 void* y_hi, void* y_lo, lwb_stream_t stream)
{
    LWB_CHECK_ARG(x && scale && shift && y_hi && y_lo, "null pointer");
    LWB_CHECK_ARG(n > 0 && c > 0 && h > 1 && w > 1, "bad sizes");
    const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
    k_det_stem_pool<<<lwb::ceil_div((long)n * ho * wo * c, 256), 256, 0, (cudaStream_t)stream>>>(
        x, n, c, h, w, scale, shift, ho, wo, (__half*)y_hi, (__half*)y_lo);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_bias_act(const float* raw, int ld_raw, const float* raw2, const float* bias, const float* res, int res_half,
                                int step, int h_in, int w_in, int relu, int n, int h, int w, int c,
                                float* y_f32, void* y_hi, void* y_lo, lwb_stream_t stream)
{
    LWB_CHECK_ARG(raw && (y_f32 || y_hi), "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0 && c > 0 && ld_raw >= c && step >= 1, "bad sizes");
    LWB_CHECK_ARG((h - 1) * step < h_in && (w - 1) * step < w_in, "output grid outside the input");
    LWB_CHECK_ARG(!res_half || (h % 2 == 0 && w % 2 == 0), "nearest 2x residual needs an even grid");
    k_det_bias_act<<<lwb::ceil_div((long)n * h * w * c, 256), 256, 0, (cudaStream_t)stream>>>(
        raw, ld_raw, raw2, bias, res, res_half, step, h_in, w_in, relu, n, h, w, c, y_f32, (__half*)y_hi, (__half*)y_lo);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_d2s_bias_relu(const float* raw, const float* bias, int n, int h, int w, int c,
                                     float* y_f32, void* y_hi, void* y_lo, lwb_stream_t stream)
{
    LWB_CHECK_ARG(raw && bias && (y_f32 || y_hi), "null pointer");
    LWB_CHECK_ARG(n > 0 && h > 0 && w > 0 && c > 0, "bad sizes");
    k_det_d2s_bias_relu<<<lwb::ceil_div(4L * n * h * w * c, 256), 256, 0, (cudaStream_t)stream>>>(
        raw, bias, n, h, w, c, y_f32, (__half*)y_hi, (__half*)y_lo);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_rpn(int levels, const float* const* heads, const int* gh, const int* gw, const int* stride_h,
                           const int* stride_w, const float* cell_anchors, const int* offsets, const float* bias, int k,
                           float clip_h, float clip_w, float min_size, float xform_clip, int* top_idx, float* boxes,
                           float* scores, int* groups, int* valid, lwb_stream_t stream)
{
    LWB_CHECK_ARG(heads && gh && gw && stride_h && stride_w && cell_anchors && offsets && bias && boxes && scores && groups && valid,
                  "null pointer");
    LWB_CHECK_ARG(levels >= 1 && levels <= 5 && k > 0 && k <= kRpnMaxK, "1..5 levels, k <= 1024");
    RpnArgs A;
    memset(&A, 0, sizeof(A));
    for (int l = 0; l < levels; l++) {
        LWB_CHECK_ARG(heads[l] && gh[l] > 0 && gw[l] > 0, "bad level");
        A.lv[l].head = heads[l];
        A.lv[l].gh = gh[l]; A.lv[l].gw = gw[l]; A.lv[l].stride_h = stride_h[l]; A.lv[l].stride_w = stride_w[l];
        A.lv[l].offset = offsets[l];
        for (int q = 0; q < 12; q++) A.lv[l].cell[q] = cell_anchors[l * 12 + q];
    }
    A.k = k; A.clip_h = clip_h; A.clip_w = clip_w; A.min_size = min_size; A.xform_clip = xform_clip;
    k_det_rpn_level<<<levels, kRpnThreads, 0, (cudaStream_t)stream>>>(A, bias, top_idx, boxes, scores, groups, valid);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// workspace sections: count | compacted slots | order | sorted boxes | sorted groups | IoU bitmask (each 256-B aligned:
// the bitmask is read as 64-bit words)
extern "C" size_t lwb_det_nms_workspace_bytes(int n, int m_max)
{
    (void)n;
    const size_t cb = (size_t)lwb::ceil_div(m_max, kNmsBlock), m = (size_t)m_max;
    return 256 + 3 * align256(m * 4) + align256(m * 16) + align256(m * cb * 8);
}

// n slots (valid[] nullable), of which at most m_max are valid: the keep list holds slot indices in descending score order
extern "C" int lwb_det_nms(const float* boxes, const float* scores, const int* groups, const int* valid, int n, int m_max, float thresh,
                           int max_keep, void* workspace, int* keep, float* out_boxes, float* out_scores, int* out_groups,
                           int* out_count, lwb_stream_t stream)
{
    LWB_CHECK_ARG(boxes && scores && workspace && keep && out_count, "null pointer");
    LWB_CHECK_ARG(n > 0 && m_max > 0 && max_keep > 0, "bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    const int cb = lwb::ceil_div(m_max, kNmsBlock);
    LWB_CHECK_ARG((size_t)cb * 8 <= 48 * 1024, "too many boxes for one sweep");
    LWB_CHECK_ARG(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    char* p = (char*)workspace;
    int* count = (int*)p;                    p += 256;
    int* comp = (int*)p;                     p += align256((size_t)m_max * 4);
    int* order = (int*)p;                    p += align256((size_t)m_max * 4);
    float* sboxes = (float*)p;               p += align256((size_t)m_max * 16);
    int* sgroups = (int*)p;                  p += align256((size_t)m_max * 4);
    unsigned long long* mask = (unsigned long long*)p;
    LWB_CUDA_OK(cudaMemsetAsync(count, 0, sizeof(int), st));
    k_nms_compact<<<lwb::ceil_div(n, 256), 256, 0, st>>>(valid, n, m_max, comp, count);
    k_nms_rank<<<lwb::ceil_div(m_max, 256), 256, 0, st>>>(comp, count, m_max, scores, boxes, groups, order, sboxes, sgroups);
    k_nms_mask<<<dim3(cb, cb), kNmsBlock, 0, st>>>(count, m_max, sboxes, sgroups, thresh, cb, mask);
    k_nms_sweep<<<1, 32, (size_t)cb * 8, st>>>(count, m_max, order, sboxes, sgroups, scores, mask, cb, max_keep, keep, out_boxes,
                                                out_scores, out_groups, out_count);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_roi_align(const float* const* feats, const int* fh, const int* fw, int c, const float* boxes, const int* count,
                                 int r_max, int out, int sampling, int* levels, float* y_f32, void* y_hi, void* y_lo, lwb_stream_t stream)
{
    LWB_CHECK_ARG(feats && fh && fw && boxes && (y_f32 || y_hi), "null pointer");
    LWB_CHECK_ARG(c > 0 && r_max > 0 && out > 0 && sampling > 0, "bad sizes");
    Pyramid P;
    for (int l = 0; l < 4; l++) {
        LWB_CHECK_ARG(feats[l] && fh[l] > 0 && fw[l] > 0, "bad level");
        P.p[l] = feats[l]; P.h[l] = fh[l]; P.w[l] = fw[l];
    }
    k_det_roi_align<<<lwb::ceil_div((long)r_max * out * out * c, 256), 256, 0, (cudaStream_t)stream>>>(
        P, c, boxes, count, r_max, out, sampling, levels, y_f32, (__half*)y_hi, (__half*)y_lo);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_box_candidates(const float* pred, int ld, int nc, const float* proposals, const int* count, int r_max,
                                      float clip_h, float clip_w, float score_thresh, float min_size, float xform_clip,
                                      float* boxes, float* scores, int* groups, int* valid, lwb_stream_t stream)
{
    LWB_CHECK_ARG(pred && proposals && count && boxes && scores && groups && valid, "null pointer");
    LWB_CHECK_ARG(nc > 1 && ld >= nc * 5 && r_max > 0, "bad sizes");
    k_det_box_candidates<<<lwb::ceil_div(32L * r_max, 256), 256, 0, (cudaStream_t)stream>>>(
        pred, ld, nc, proposals, count, r_max, clip_h, clip_w, score_thresh, min_size, xform_clip, boxes, scores, groups, valid);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_mask_probs(const float* raw, int ld, const float* bias, const int* labels, const int* count, int d_max, int hw,
                                  float* logits, float* probs, lwb_stream_t stream)
{
    LWB_CHECK_ARG(raw && bias && labels && count && probs, "null pointer");
    LWB_CHECK_ARG(d_max > 0 && hw > 0 && ld > 0, "bad sizes");
    k_det_mask_probs<<<lwb::ceil_div((long)d_max * hw, 256), 256, 0, (cudaStream_t)stream>>>(raw, ld, bias, labels, count, d_max, hw,
                                                                                             logits, probs);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_paste_masks(const float* probs, int m, const float* boxes, const int* count, int d_max, float rh, float rw,
                                   int h, int w, float* masks, float* out_boxes, lwb_stream_t stream)
{
    LWB_CHECK_ARG(probs && boxes && count && out_boxes, "null pointer");
    LWB_CHECK_ARG(m > 0 && d_max > 0 && h > 0 && w > 0, "bad sizes");
    k_det_paste<<<lwb::ceil_div((long)d_max * h * w, 256), 256, 0, (cudaStream_t)stream>>>(probs, m, boxes, count, d_max, rh, rw, h, w,
                                                                                          masks, out_boxes);
    LWB_LAUNCH_OK();
    return LWB_OK;
}

extern "C" int lwb_det_person_mask(const float* boxes, const int* labels, const int* count, int person, const float* masks, int h, int w,
                                   float thresh, int ks, int* pid, float* box, float* out, lwb_stream_t stream)
{
    LWB_CHECK_ARG(boxes && labels && count && masks && pid && box && out, "null pointer");
    LWB_CHECK_ARG(h > 0 && w > 0 && ks >= 0, "bad sizes");
    // utils/util.py morph pads ks // 2 on every side, so an even ks gives an (h+1) x (w+1) mask that the callers'
    // img * mask cannot broadcast: refuse it here instead of returning a shifted h x w dilation
    LWB_CHECK_ARG(ks == 0 || ks % 2 == 1, "ks must be 0 or odd");
    k_det_person_mask<<<lwb::ceil_div((long)h * w, 256), 256, 0, (cudaStream_t)stream>>>(boxes, labels, count, person, masks, h, w,
                                                                                        thresh, ks, pid, box, out);
    LWB_LAUNCH_OK();
    return LWB_OK;
}
