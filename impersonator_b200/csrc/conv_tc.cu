// Implicit-GEMM convolution on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a only.
//
// Replaces the cuDNN calls behind nn.Conv2d / nn.ConvTranspose2d (all bias=False) of
//   networks/generator.py:8-20 (ResidualBlock 3x3), :80-95 (7x7 stem, 3x3 stride-2 encoders),
//   :107-124 (ConvTranspose 3x3 s2 p1 op1 decoders, 3x3 "skippers" on cat[skip, d]).
//
// GEMM view (no im2col buffer is ever materialised):
//   D[m, n] = sum_{tap, c} A_tap[m, c] * W[tap][n][c]
//   m = one output pixel of a 16 x 8 spatial tile (M = 128),  n = output channel,
//   A_tap = the same NHWC fp16 activation tensor fetched by TMA at the tap's spatial offset
//           (out-of-bounds rows/cols are zero-filled by the TMA unit = the conv padding),
//   W     = weights repacked once to [tap][Cout][Cin] fp16 (K-major rows of 128 bytes).
// Both operands land in shared memory in the canonical K-major SWIZZLE_128B layout.  A CTA is one
// producer warpgroup (one warp issues the TMA loads, see Regs) and two consumer warpgroups that issue, per tap and K = 64
// chunk, 4 x wgmma (K16) into register accumulators.
//
// Y-halo tap groups: one image row of the tile (8 px x 128 B) is exactly one 1024-byte swizzle atom, so
// taps that read the same input view at the same dx with consecutive dy share ONE activation box of
// TILE_H + cnt - 1 rows; tap i of the group starts its activation descriptor i x 1024 B further in (the swizzle
// phase lives in address bits 7-9 and does not change).  The K loop runs (group, chunk, tap in group):
// one activation fetch per (group, chunk) into the A ring, one weight fetch per tap into the B ring.
//
// Channel-major orientation (every plan whose N tile is 64 or 128): the accumulator is D^T[cout, pixel] =
// W[cout, K] . X[pixel, K]^T, with the channels on the wgmma M side.  The [N][128 B] weight tile is the A operand and the
// activation box the B operand (both already K-major SWIZZLE_128B); each consumer warpgroup issues M64 x N128 wgmmas:
//   N tile 128: 16 x 8-pixel tiles, warpgroup g takes weight rows 64 g .. 64 g + 63 and the whole 128-pixel window;
//   N tile 64 : 32 x 8-pixel tiles (the same 16K-output accumulator budget), both warpgroups take all 64 weight rows,
//               warpgroup g box rows 16 g .. 16 g + 15.
// Each thread then holds two whole channels of its warpgroup's pixels.  With N tiles of 128 the two warpgroups hold
// different channels, so a warpgroup's epilogue (stores and InstanceNorm statistics) needs nothing from the other one:
// the warpgroup that finishes its K loop first goes on to the next tile's wgmmas, bounded only by the rings, and the
// other's epilogue runs under them.  N = 64 tiles merge the two warpgroups' statistics (epilogue_channel_major).
// N tiles of 16 / 32 (the folded heads) keep the pixel-major orientation: M = 128 pixels, warpgroup g tile rows
// 8 g .. 8 g + 7, D[pixel, cout] = X . W^T with m64nNk16.
//
// Precision: x ~= x_hi + x_lo, w ~= w_hi + w_lo in fp16; with SPLIT the accumulator receives
// x_hi*w_hi + x_hi*w_lo + x_lo*w_hi (fp32 accumulate), which reproduces the fp32 reference
// convolution to ~1e-5 (single pass fp16 cannot meet the 1e-3 parity bar, SURVEY.md 0.4).
// In f8 mode (MODE_F8, the default of the host side) the two small products are issued as ONE
// e4m3 x e4m3 wgmma (K32) per K16 step on operand pairs stored in the lo buffers (elementwise.cu, kF8*),
// into a second accumulator that the epilogue adds to the fp16 one.
//
// Variants, all through the same kernel:
//   stride 2      : four parity views of the input (plain strided tensor maps), tap -> view
//   transposed    : four sub-pixel output phases, each a 1/2/2/4-tap stride-1 conv
//   merged transp.: one stride-1 pass whose N columns are the four phases (phase_cols)
//   concat input  : K chunks 0..chunks0-1 from tensor 0, the rest from tensor 1 (torch.cat free)
//   7x7 stem      : "row-K" trick -- with 8 channels per pixel, 8 consecutive pixels of a padded
//                   NHWC8 row are 64 contiguous fp16, so one K = 64 stage covers a whole filter
//                   row (overlapping-stride tensor map); 7 stages instead of 49.  With 16 or 24 channels per
//                   pixel (the wide conditioning maps) a filter row is 2 or 3 such K stages.
// Epilogue: accumulator registers -> fp32 NHWC global + per-(n, c) sum / sum of squares for the
// InstanceNorm that follows every conv (f64 atomics).
#include <cuda.h>

#include <stdlib.h>

#include <algorithm>
#include <new>
#include <type_traits>

#include "common.cuh"

namespace {

constexpr int TILE_H = 16, TILE_W = 8;          // output pixels per tile (M = 128)
constexpr int SWAP_N_TILE = 64;                  // plans with this N tile run channel-major ...
constexpr int SWAP_TILE_H = 32;                  // ... on 32 x 8 = 256-pixel tiles (N = 128: channel-major on 16 x 8)
constexpr int KCHUNK = 64;                       // fp16 elements per K stage (128 B swizzle span)
constexpr int ROW_BYTES = TILE_W * 128;          // one image row of an A box = one SWIZZLE_128B atom
constexpr int MAX_TAPS = 49;
constexpr int MAX_GROUP = 8;                     // taps per y-halo group: A boxes of at most tile height + 7 rows
constexpr int RING_BYTES = 200 * 1024;           // A ring + B ring
constexpr int MAX_STAGES = 8;                    // entries per ring
constexpr int NUM_CONSUMERS = 256;               // warps 0..7: two consumer warpgroups
constexpr int NUM_THREADS = NUM_CONSUMERS + 128; // warps 8..11: producer warpgroup (warp 8 issues the TMA loads)
constexpr int MAX_N_TILE = 128;                  // 64 fp32 accumulator registers per consumer thread
static_assert(2 * 2 * (TILE_H + MAX_GROUP - 1) * ROW_BYTES + 2 * 2 * MAX_N_TILE * 128 <= RING_BYTES,
              "every plan needs two A and two B entries in the ring");
static_assert(2 * 2 * (SWAP_TILE_H + MAX_GROUP - 1) * ROW_BYTES + 2 * 2 * SWAP_N_TILE * 128 <= RING_BYTES,
              "every swapped plan needs two A and two B entries in the ring");
static_assert(SWAP_N_TILE * (SWAP_TILE_H * TILE_W) == MAX_N_TILE * (TILE_H * TILE_W), "same accumulator budget");

__host__ __device__ constexpr int tile_rows(int n_tile) { return n_tile == SWAP_N_TILE ? SWAP_TILE_H : TILE_H; }

struct ConvParams {
    CUtensorMap a_hi[4];
    CUtensorMap a_lo[4];
    CUtensorMap w_hi;
    CUtensorMap w_lo;
    int n_img, tiles_y, tiles_x, n_tiles_n;
    int dom_h, dom_w;                 // extent of the tile domain (output grid, or phase grid)
    int ntaps, chunks0, chunks1;
    signed char dy[MAX_TAPS], dx[MAX_TAPS], tmap[MAX_TAPS];
    short wtap[MAX_TAPS];
    int ngroups;                      // y-halo groups: taps g_first .. g_first + g_cnt - 1, dy consecutive (group_taps)
    signed char g_first[MAX_TAPS], g_cnt[MAX_TAPS];
    int a_rows;                       // A box height: tile height + longest group - 1
    int a_stages, b_stages;           // ring depths inside RING_BYTES (pick_rings)
    float* out; int out_h, out_w, cout;
    int oy_mul, oy_add, ox_mul, ox_add;
    double* stats;
    float out_scale;                  // accumulator -> output (2^-w_exp)
    int phase_cols;                   // > 0: merged transposed conv -- column block col / phase_cols = sub-pixel phase (a, b) =
                                      // (ph >> 1, ph & 1) of output pixel (2y + a, 2x + b), channel = col % phase_cols
};

// Shared memory: [A ring: a_stages x (hi | lo) boxes of a_rows rows][B ring: b_stages x (hi | lo) weight tiles] inside
// RING_BYTES, then the barriers and the statistics partials.
template <int N_TILE, bool SPLIT>
struct Cfg {
    static constexpr int B_BYTES = N_TILE * 128;
    static constexpr int B_STAGE_BYTES = B_BYTES * (SPLIT ? 2 : 1);
    static constexpr int BAR_BYTES = 4 * MAX_STAGES * 8;         // A full / empty, B full / empty
    // [PARTS][N_TILE] float2 partial statistics: the 8 consumer warps of a pixel-major tile, the 2 warpgroups of an N = 64
    // tile; N = 128 tiles share nothing
    static constexpr int STATS_PARTS = N_TILE < SWAP_N_TILE ? 8 : N_TILE == SWAP_N_TILE ? 2 : 0;
    static constexpr int STATS_BYTES = STATS_PARTS * N_TILE * 8;
    static constexpr int SMEM_BYTES = 1024 + RING_BYTES + BAR_BYTES + STATS_BYTES;
    static_assert(B_STAGE_BYTES % 1024 == 0, "B entries must keep the 1024-byte swizzle alignment");
    static_assert(SMEM_BYTES <= 227 * 1024, "exceeds the shared memory of a block");
};

// ----------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (kernel error) instead of hanging the GPU.  No printf here: a function call inside
// the consumer's main loop would make ptxas serialise the asynchronous wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000ll) __trap();
    }
}
// One lane of a CONVERGED warp: issuing TMA under `if (elect_one())` (instead of `if (lane == 0)`) keeps the surrounding
// control flow warp-uniform, so descriptors and coordinates stay in uniform registers.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, void* dst, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, void* dst, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// K-major SWIZZLE_128B wgmma operand descriptor: start>>4 | LBO(16 B, unused)>>4 << 16 | SBO(1024 B: one 8-row
// swizzle atom)>>4 << 32 | layout SWIZZLE_128B(1) << 62.  A K step inside the 128-byte row advances the start address.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// Keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma.
__device__ __forceinline__ void acc_fence(float& r) { asm volatile("" : "+f"(r) :: "memory"); }

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp16 operands, both K-major in shared memory
template <int N> __device__ __forceinline__ void wgmma_f16(float* d, uint64_t da, uint64_t db);
// D[64 x N] (+)= A[64 x 32] * B[N x 32]^T, e4m3 operands: the same 32-byte descriptor step at twice the fp16 rate
template <int N> __device__ __forceinline__ void wgmma_e4m3(float* d, uint64_t da, uint64_t db);
template <> __device__ __forceinline__ void wgmma_f16<16>(float* d, uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(da), "l"(db), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_f16<32>(float* d, uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_f16<128>(float* d, uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_e4m3<16>(float* d, uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(da), "l"(db), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_e4m3<32>(float* d, uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_e4m3<128>(float* d, uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(1));
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Persistent tile schedule shared by the producer and the consumer warpgroups: tile = blockIdx.x + k * gridDim.x,
// N tile = tile / m_tiles (consecutive tiles share the weight tile and run through the images in order).
struct TileCoord {
    int n_idx, img, y0, x0;
};
template <int TH>
__device__ __forceinline__ TileCoord decode_tile(const ConvParams& P, int tile, int m_tiles) {
    TileCoord t;
    t.n_idx = tile / m_tiles;
    const int m_idx = tile % m_tiles;
    t.img = m_idx / (P.tiles_y * P.tiles_x);
    const int rem = m_idx % (P.tiles_y * P.tiles_x);
    t.y0 = (rem / P.tiles_x) * TH; t.x0 = (rem % P.tiles_x) * TILE_W;
    return t;
}

// Per-column sum / sum of squares of this warp's 16 rows (accumulator fragment: d[4j + 2h + e] = row lane/4 + 8h,
// column 8j + 2(lane%4) + e of the warp's 16 x N_TILE slice) -> s_stats[warp][col]; rows outside the domain count 0.
template <int N_TILE>
__device__ __forceinline__ void warp_tile_stats(const float* acc, bool v0, bool v1, int warp, unsigned lane, float2* s_stats)
{
#pragma unroll
    for (int j = 0; j < N_TILE / 8; j++) {
        const float a0 = v0 ? acc[4 * j] : 0.f, a1 = v0 ? acc[4 * j + 1] : 0.f;
        const float b0 = v1 ? acc[4 * j + 2] : 0.f, b1 = v1 ? acc[4 * j + 3] : 0.f;
        float s0 = a0 + b0, s1 = a1 + b1, q0 = a0 * a0 + b0 * b0, q1 = a1 * a1 + b1 * b1;
#pragma unroll
        for (int off = 4; off <= 16; off <<= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, off); s1 += __shfl_xor_sync(0xffffffffu, s1, off);
            q0 += __shfl_xor_sync(0xffffffffu, q0, off); q1 += __shfl_xor_sync(0xffffffffu, q1, off);
        }
        if (lane < 4) {
            s_stats[warp * N_TILE + 8 * j + 2 * lane] = make_float2(s0, q0);
            s_stats[warp * N_TILE + 8 * j + 2 * lane + 1] = make_float2(s1, q1);
        }
    }
}

// s_stats of the PARTS partial rows (8 consumer warps, or 2 warpgroups of an N = 64 tile) -> one f64 atomic pair per
// column of the tile (all consumer threads).
template <int N_TILE, int PARTS>
__device__ __forceinline__ void flush_tile_stats(const ConvParams& P, const float2* s_stats, int img, int n_idx)
{
    consumer_sync();
    for (int col = threadIdx.x; col < N_TILE; col += NUM_CONSUMERS) {
        float s = 0.f, q = 0.f;
#pragma unroll
        for (int w = 0; w < PARTS; w++) { const float2 v = s_stats[w * N_TILE + col]; s += v.x; q += v.y; }
        int ch = n_idx * N_TILE + col;
        if (P.phase_cols > 0) ch %= P.phase_cols;      // the four phases of a channel share its statistics
        double* dst = P.stats + 2 * ((size_t)img * P.cout + ch);
        atomicAdd(dst, (double)s);
        atomicAdd(dst + 1, (double)q);
    }
    consumer_sync();
}

// Pixel-major epilogue (N tiles of 16 / 32): accumulators -> fp32 NHWC global + InstanceNorm partial statistics.
template <int N_TILE>
__device__ __forceinline__ void epilogue_plain(const ConvParams& P, float* acc, const TileCoord& t, int warp, unsigned lane,
                                               float2* s_stats)
{
    const int tx = (int)(lane >> 2), x = t.x0 + tx;
    const int y[2] = {t.y0 + 2 * warp, t.y0 + 2 * warp + 1};       // rows 16 warp + lane/4 (+8) = tile rows 2 warp (+1)
    const bool valid[2] = {y[0] < P.dom_h && x < P.dom_w, y[1] < P.dom_h && x < P.dom_w};
    if (P.out_scale != 1.f) {
#pragma unroll
        for (int i = 0; i < N_TILE / 2; i++) acc[i] *= P.out_scale;
    }
    if (P.out) {
        const int out_w_c = P.out_w * P.cout;                       // one output row, in floats (merged transposed conv)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (!valid[h]) continue;
            float* optr = P.out + (((size_t)t.img * P.out_h + (P.oy_mul * y[h] + P.oy_add)) * P.out_w + (P.ox_mul * x + P.ox_add)) * P.cout
                        + (size_t)t.n_idx * N_TILE;
#pragma unroll
            for (int j = 0; j < N_TILE / 8; j++) {
                const int c = 8 * j + 2 * (int)(lane & 3);
                float* o = optr + c;
                if (P.phase_cols > 0) {
                    const int col = t.n_idx * N_TILE + c, ph = col / P.phase_cols;
                    o = P.out + (((size_t)t.img * P.out_h + 2 * y[h]) * P.out_w + 2 * x) * P.cout
                      + (size_t)(ph >> 1) * out_w_c + (ph & 1) * P.cout + (col - ph * P.phase_cols);
                }
                *reinterpret_cast<float2*>(o) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        }
    }
    if (P.stats) {
        warp_tile_stats<N_TILE>(acc, valid[0], valid[1], warp, lane, s_stats);
        flush_tile_stats<N_TILE, 8>(P, s_stats, t.img, t.n_idx);
    }
}

// Epilogue of the channel-major orientation: the accumulator is D^T, d[4j + 2h + e] = channel c0 + 8h of the N tile at
// pixel (tile row row0 + j, column 2(lane%4) + e), c0 = c_base + 16(warp%4) + lane/4, where warpgroup g has c_base =
// 64 g, row0 = 0 for N tiles of 128 and c_base = 0, row0 = 16 g for N tiles of 64.  fp32 NHWC stores: one warp-wide store
// covers 4 pixels x 8 consecutive channels, whole 32-byte sectors.  Each thread's two channels are complete in the warp:
// in-thread sums over the valid pixels, then two quad shuffles.  N = 128: the quad leader issues the f64 atomics, with no
// shared memory and no barrier, so the two warpgroups never wait for each other.  N = 64: both warpgroups hold the same
// channels, and the two halves meet in s_stats before one atomic pair per channel and tile: with an atomic pair per
// warpgroup (twice the same-address f64 atomics on an image's 64 channels) the stem and the 64+64->64 skipper ran
// 4-22 % slower (DESIGN section 5).  In a merged transposed plan N column col is channel col % phase_cols of
// sub-pixel phase ph = col / phase_cols, written to output pixel (2y + (ph >> 1), 2x + (ph & 1)).
template <int N_TILE>
__device__ __forceinline__ void epilogue_channel_major(const ConvParams& P, float* acc, const TileCoord& t, int warp,
                                                       unsigned lane, float2* s_stats)
{
    const int wg = warp >> 2;
    const int c_base = N_TILE == MAX_N_TILE ? 64 * wg : 0, row0 = N_TILE == MAX_N_TILE ? 0 : 16 * wg;
    const int c0 = c_base + 16 * (warp & 3) + (int)(lane >> 2);       // channels c0 and c0 + 8 of the N tile
    const int y0 = t.y0 + row0, x0 = t.x0 + 2 * (int)(lane & 3);
    const int rows = P.dom_h - y0;                                     // row j is in the domain iff j < rows
    const bool vx[2] = {x0 < P.dom_w, x0 + 1 < P.dom_w};
    // output channel of c0 and its offset from the pixel's NHWC address; phase_cols is a multiple of 32, so channel
    // c0 + 8 is in the same phase at ch + 8
    const int col = t.n_idx * N_TILE + c0;
    const int ph = P.phase_cols > 0 ? col / P.phase_cols : 0;
    const int ch = col - ph * P.phase_cols;
    const size_t coff = ((size_t)(ph >> 1) * P.out_w + (ph & 1)) * P.cout + ch;
    if (P.out_scale != 1.f) {
#pragma unroll
        for (int i = 0; i < 64; i++) acc[i] *= P.out_scale;
    }
    if (P.out) {
#pragma unroll
        for (int j = 0; j < 16; j++) {
            if (j >= rows) break;
            const size_t orow = ((size_t)t.img * P.out_h + (P.oy_mul * (y0 + j) + P.oy_add)) * P.out_w;
#pragma unroll
            for (int e = 0; e < 2; e++) {
                if (!vx[e]) continue;
                float* o = P.out + (orow + (P.ox_mul * (x0 + e) + P.ox_add)) * P.cout;
                o[coff] = acc[4 * j + e];
                o[coff + 8] = acc[4 * j + 2 + e];
            }
        }
    }
    if (P.stats) {
        float s[2] = {0.f, 0.f}, q[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 16; j++) {
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const bool v = j < rows && vx[e];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const float a = v ? acc[4 * j + 2 * h + e] : 0.f;
                    s[h] += a; q[h] += a * a;
                }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int off = 1; off <= 2; off <<= 1) {
                s[h] += __shfl_xor_sync(0xffffffffu, s[h], off);
                q[h] += __shfl_xor_sync(0xffffffffu, q[h], off);
            }
        }
        if constexpr (N_TILE == SWAP_N_TILE) {
            if ((lane & 3) == 0) {
                s_stats[wg * N_TILE + c0] = make_float2(s[0], q[0]);
                s_stats[wg * N_TILE + c0 + 8] = make_float2(s[1], q[1]);
            }
            flush_tile_stats<N_TILE, 2>(P, s_stats, t.img, t.n_idx);
        } else if ((lane & 3) == 0) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                double* dst = P.stats + 2 * ((size_t)t.img * P.cout + ch + 8 * h);
                atomicAdd(dst, (double)s[h]);
                atomicAdd(dst + 1, (double)q[h]);
            }
        }
    }
}

// ----------------------------------------------------------------------------------- kernel
// Operand modes (lwb_conv_desc.split): one fp16 product, the three fp16 products of the hi/lo split, or the fp16 hi
// product + one e4m3 wgmma on the lo pair blocks (A entries then hold [A_hi | A_lo8], B entries [B_hi | B_lo8]).
enum { MODE_FP16 = 0, MODE_FP16X3 = 1, MODE_F8 = 2 };

// Register budget per thread (setmaxnreg).  Registers are allocated per SM sub-partition (16 K each), and warp w of a CTA
// lands on sub-partition w % 4.  A CTA of two consumer warpgroups and one producer warp at the consumers' 161 registers
// (fp16f8) put three 168-register warps on sub-partition 0 and left 256 registers there, so no 256-thread block of any
// other kernel (k_norm_act of the other sub-batch stream) could become resident beside a conv CTA.  With a producer
// warpgroup the CTA launches at LAUNCH registers per thread (three warps per sub-partition), the producer warpgroup gives
// all but PRODUCER back and the consumers take CONSUMER: 2 CONSUMER + PRODUCER = 3 LAUNCH, and every sub-partition keeps
// 16 K - 3 x 32 LAUNCH registers for other kernels (4 K, one 64-register warp pair, for the fp16f8 instances).
// CONSUMER is at least what ptxas needs for the consumer path of the instance (no spills, see -Xptxas -v).
template <int N_TILE, int MODE>
struct Regs {
    static constexpr int CONSUMER = N_TILE >= 64 ? (MODE == MODE_F8 ? 168 : 120) : N_TILE == 32 ? 80 : 64;
    static constexpr int LAUNCH = ((2 * CONSUMER + 40 + 2) / 3 + 7) / 8 * 8;
    static constexpr int PRODUCER = 3 * LAUNCH - 2 * CONSUMER;
    static_assert(PRODUCER >= 40 && PRODUCER % 8 == 0 && CONSUMER % 8 == 0, "setmaxnreg takes multiples of 8");
};

// One fp16 wgmma step of the tile: activation rows x weight rows, or (CM) 64 weight rows x activation rows on 128 pixels.
template <int N_TILE, bool CM>
__device__ __forceinline__ void mma_f16(float* d, uint64_t act, uint64_t w) {
    if constexpr (CM) wgmma_f16<128>(d, w, act);
    else              wgmma_f16<N_TILE>(d, act, w);
}
template <int N_TILE, bool CM>
__device__ __forceinline__ void mma_e4m3(float* d, uint64_t act, uint64_t w) {
    if constexpr (CM) wgmma_e4m3<128>(d, w, act);
    else              wgmma_e4m3<N_TILE>(d, act, w);
}

template <int N_TILE, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1) __maxnreg__((Regs<N_TILE, MODE>::LAUNCH))
k_conv_wg(const __grid_constant__ ConvParams P)
{
    // N tiles of 64 and 128 run channel-major (N = 64 on 256-pixel tiles, see the top of the file); plan creation sized
    // its tiles and boxes with tile_rows(n_tile) to match.
    constexpr bool CM = N_TILE >= SWAP_N_TILE;
    constexpr bool SPLIT = MODE != MODE_FP16;
    constexpr int TH = N_TILE == SWAP_N_TILE ? SWAP_TILE_H : TILE_H;  // tile rows
    constexpr int ACC = CM ? 64 : N_TILE / 2;                         // fp32 accumulators per consumer thread
    using C = Cfg<N_TILE, SPLIT>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int a_op_bytes = P.a_rows * ROW_BYTES;                     // one operand (hi or lo) of an A entry
    const int a_stage_bytes = a_op_bytes * (SPLIT ? 2 : 1);
    uint8_t* b_ring = smem + P.a_stages * a_stage_bytes;
    uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + RING_BYTES);
    uint64_t* a_empty = a_full + MAX_STAGES;
    uint64_t* b_full = a_empty + MAX_STAGES;
    uint64_t* b_empty = b_full + MAX_STAGES;
    float2* s_stats = reinterpret_cast<float2*>(smem + RING_BYTES + C::BAR_BYTES);   // [Cfg::STATS_PARTS][N_TILE]

    const int warp = threadIdx.x >> 5;
    const unsigned lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        // empty[s] collects one arrival per consumer warp once its wgmma reads of the entry have retired
        for (int s = 0; s < P.a_stages; s++) { mbar_init(a_full + s, 1); mbar_init(a_empty + s, NUM_CONSUMERS / 32); }
        for (int s = 0; s < P.b_stages; s++) { mbar_init(b_full + s, 1); mbar_init(b_empty + s, NUM_CONSUMERS / 32); }
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    // everything above touched only shared memory; global memory (operands, output, statistics) is produced / still read
    // by the preceding kernel of the stream: wait for it (no-op without a programmatic launch)
    lwb::pdl_wait();
    lwb::pdl_trigger();

    const int nchunks = P.chunks0 + P.chunks1;
    const int m_tiles = P.n_img * P.tiles_y * P.tiles_x;
    const int total = m_tiles * P.n_tiles_n;

    if (warp >= NUM_CONSUMERS / 32) {
        // ================================ TMA producer (warp 8; one elected lane issues) ==============
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(Regs<N_TILE, MODE>::PRODUCER));
        if (warp != NUM_CONSUMERS / 32) return;
        if (elect_one()) {
            asm volatile("prefetch.tensormap [%0];" :: "l"(&P.a_hi[0]) : "memory");
            asm volatile("prefetch.tensormap [%0];" :: "l"(&P.w_hi) : "memory");
            if (SPLIT) {
                asm volatile("prefetch.tensormap [%0];" :: "l"(&P.a_lo[0]) : "memory");
                asm volatile("prefetch.tensormap [%0];" :: "l"(&P.w_lo) : "memory");
            }
        }
        int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
        for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
            const TileCoord t = decode_tile<TH>(P, tile, m_tiles);
            for (int g = 0; g < P.ngroups; g++) {
                const int first = P.g_first[g], cnt = P.g_cnt[g];
                const int xx = t.x0 + P.dx[first], yy = t.y0 + P.dy[first];
                for (int chunk = 0; chunk < nchunks; chunk++) {
                    const bool second = chunk >= P.chunks0;
                    const int mi = second ? 1 : P.tmap[first];
                    const int c0 = (second ? chunk - P.chunks0 : chunk) * KCHUNK;
                    // one box of a_rows image rows serves every tap of the group
                    mbar_wait(a_empty + as, aph ^ 1);
                    uint8_t* sa = smem + as * a_stage_bytes;
                    if (elect_one()) {
                        mbar_expect_tx(a_full + as, (uint32_t)a_stage_bytes);
                        tma_load_4d(&P.a_hi[mi], sa, a_full + as, c0, xx, yy, t.img);
                        if (SPLIT) tma_load_4d(&P.a_lo[mi], sa + a_op_bytes, a_full + as, c0, xx, yy, t.img);
                    }
                    __syncwarp();
                    if (++as == P.a_stages) { as = 0; aph ^= 1; }
                    for (int i = 0; i < cnt; i++) {
                        mbar_wait(b_empty + bs, bph ^ 1);
                        uint8_t* sb = b_ring + bs * C::B_STAGE_BYTES;
                        const int wt = P.wtap[first + i];
                        if (elect_one()) {
                            mbar_expect_tx(b_full + bs, (uint32_t)C::B_STAGE_BYTES);
                            tma_load_3d(&P.w_hi, sb, b_full + bs, chunk * KCHUNK, t.n_idx * N_TILE, wt);
                            if (SPLIT) tma_load_3d(&P.w_lo, sb + C::B_BYTES, b_full + bs, chunk * KCHUNK, t.n_idx * N_TILE, wt);
                        }
                        __syncwarp();
                        if (++bs == P.b_stages) { bs = 0; bph ^= 1; }
                    }
                }
            }
        }
    } else {
        // ================================ consumers (2 warpgroups) =====================================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(Regs<N_TILE, MODE>::CONSUMER));
        // Warpgroup g reads weight rows 64 g .. 64 g + 63 on all 16 tile rows (N tile 128), or all weight rows on tile
        // rows (TH/2) g .. (TH/2)(g + 1) - 1 (N tiles of 16 .. 64).
        constexpr bool CH_SPLIT = N_TILE == MAX_N_TILE;
        const uint32_t wg = (uint32_t)(warp >> 2);
        const uint32_t a_base = smem_u32(smem) + (CH_SPLIT ? 0 : wg * (TH / 2) * ROW_BYTES);
        const uint32_t b_base = smem_u32(b_ring) + (CH_SPLIT ? wg * 64 * 128 : 0);
        // The e4m3 products get their own accumulator: Hopper's fp8 wgmma adds into D with a reduced-precision
        // accumulation, which would truncate the fp16 main product's fp32 sum.  The two are added in the epilogue.
        float acc[ACC];
        float acc8[MODE == MODE_F8 ? ACC : 1];
        int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
        for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
            const TileCoord t = decode_tile<TH>(P, tile, m_tiles);
#pragma unroll
            for (int i = 0; i < ACC; i++) acc[i] = 0.f;
#pragma unroll
            for (int i = 0; i < (MODE == MODE_F8 ? ACC : 1); i++) acc8[i] = 0.f;
            // B entry of the last committed wgmma group, and the A entry whose last tap is in that group: both are
            // released once the group has retired
            int prev_b = -1, prev_a = -1;
            for (int g = 0; g < P.ngroups; g++) {
                const int cnt = P.g_cnt[g];
                for (int chunk = 0; chunk < nchunks; chunk++) {
                    mbar_wait(a_full + as, aph);
                    const uint32_t a_hi = a_base + as * a_stage_bytes;
                    for (int i = 0; i < cnt; i++) {
                        mbar_wait(b_full + bs, bph);
                        const uint32_t ai = a_hi + i * ROW_BYTES, al = ai + a_op_bytes;      // tap i: i box rows further in
                        const uint32_t b_hi = b_base + bs * C::B_STAGE_BYTES, b_lo = b_hi + C::B_BYTES;
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < KCHUNK / 16; k++) {
                            const uint64_t da = make_desc(ai + k * 32), db = make_desc(b_hi + k * 32);
                            mma_f16<N_TILE, CM>(acc, da, db);
                            if constexpr (MODE == MODE_F8) {
                                mma_e4m3<N_TILE, CM>(acc8, make_desc(al + k * 32), make_desc(b_lo + k * 32));
                            } else if constexpr (MODE == MODE_FP16X3) {
                                mma_f16<N_TILE, CM>(acc, da, make_desc(b_lo + k * 32));
                                mma_f16<N_TILE, CM>(acc, make_desc(al + k * 32), db);
                            }
                        }
                        wgmma_commit();
                        // the previous wgmma group has retired: its entries may be refilled
                        if (prev_b >= 0) {
                            wgmma_wait<1>();
                            if (lane == 0) {
                                mbar_arrive(b_empty + prev_b);
                                if (prev_a >= 0) mbar_arrive(a_empty + prev_a);
                            }
                            prev_a = -1;
                        }
                        prev_b = bs;
                        if (++bs == P.b_stages) { bs = 0; bph ^= 1; }
                    }
                    prev_a = as;
                    if (++as == P.a_stages) { as = 0; aph ^= 1; }
                }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < ACC; i++) acc_fence(acc[i]);
            if constexpr (MODE == MODE_F8) {
#pragma unroll
                for (int i = 0; i < ACC; i++) { acc_fence(acc8[i]); acc[i] += acc8[i]; }
            }
            if (lane == 0) { mbar_arrive(b_empty + prev_b); mbar_arrive(a_empty + prev_a); }
            if constexpr (CM) epilogue_channel_major<N_TILE>(P, acc, t, warp, lane, s_stats);
            else              epilogue_plain<N_TILE>(P, acc, t, warp, lane, s_stats);
        }
    }
}

// ------------------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return nullptr;
        fn = (EncodeTiledFn)p;
    }
    return fn;
}

// fp16 tensor map, 128B swizzle, zero OOB fill. dims/strides innermost first; strides in bytes for dims 1..rank-1.
int encode_map(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box)
{
    EncodeTiledFn enc = get_encode();
    if (!enc) { lwb::set_error("cuTensorMapEncodeTiled entry point not available"); return LWB_E_CUDA; }
    cuuint64_t gdim[5]; cuuint64_t gstr[4]; cuuint32_t bx[5]; cuuint32_t es[5];
    for (int i = 0; i < rank; i++) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
    for (int i = 0; i < rank - 1; i++) gstr[i] = strides_bytes[i];
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        lwb::set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,%llu,%llu] strides [%llu,%llu,%llu] box [%u,%u,%u,%u]",
                       (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
                       (unsigned long long)(rank > 3 ? dims[3] : 0), (unsigned long long)strides_bytes[0],
                       (unsigned long long)(rank > 2 ? strides_bytes[1] : 0), (unsigned long long)(rank > 3 ? strides_bytes[2] : 0),
                       box[0], box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
        return LWB_E_CUDA;
    }
    return LWB_OK;
}

struct Launch {
    ConvParams p;
    int n_tile;
    int mode;
    int grid;
};

template <int N_TILE, int MODE>
int launch_wg(const Launch& L, cudaStream_t st)
{
    using C = Cfg<N_TILE, MODE != MODE_FP16>;
    static bool attr_set_dev[lwb::kMaxDevices] = {};          // function attributes are per device
    bool& attr_set = attr_set_dev[lwb::device_slot()];
    if (!attr_set) {
        LWB_CUDA_OK(cudaFuncSetAttribute(k_conv_wg<N_TILE, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
        attr_set = true;
    }
    LWB_CUDA_OK(lwb::launch_pdl(k_conv_wg<N_TILE, MODE>, dim3(L.grid), dim3(NUM_THREADS), C::SMEM_BYTES, st, L.p));
    LWB_LAUNCH_OK();
    return LWB_OK;
}

// The one list of k_conv_wg instances: calls f(N_TILE, MODE), both std::integral_constant, for an N tile of 16, 32, 64
// or 128 and an operand mode.
template <class F>
int with_instance(int n_tile, int mode, F&& f)
{
    auto modes = [&](auto nt) {
        if (mode == MODE_F8) return f(nt, std::integral_constant<int, MODE_F8>());
        if (mode == MODE_FP16X3) return f(nt, std::integral_constant<int, MODE_FP16X3>());
        return f(nt, std::integral_constant<int, MODE_FP16>());
    };
    switch (n_tile) {
        case 16:  return modes(std::integral_constant<int, 16>());
        case 32:  return modes(std::integral_constant<int, 32>());
        case 64:  return modes(std::integral_constant<int, 64>());
        case 128: return modes(std::integral_constant<int, 128>());
    }
    lwb::set_error("conv_tc: unsupported N tile %d", n_tile);
    return LWB_E_UNSUPPORTED;
}

int launch(const Launch& L, cudaStream_t st)
{
    return with_instance(L.n_tile, L.mode,
                         [&](auto nt, auto md) { return launch_wg<decltype(nt)::value, decltype(md)::value>(L, st); });
}

int pick_n_tile(int cout, int forced)
{
    if (forced > 0) return forced > MAX_N_TILE && forced % MAX_N_TILE == 0 ? MAX_N_TILE : forced;
    if (cout % 128 == 0) return 128;
    if (cout % 64 == 0) return 64;
    if (cout % 32 == 0) return 32;
    if (cout % 16 == 0) return 16;
    return -1;
}

// One tensor of a plan as a hi / lo pair of fp16 TMA views with the same shape.  dims innermost first, strides in bytes
// for dims 1..rank-1; activations are rank 4 [C, W, H, N], weights rank 3 [K, N, tap].
struct View {
    const uint16_t* hi;
    const uint16_t* lo;
    uint64_t dims[4], str[3];
};

// What sets one launch of a plan apart; build_launch turns it into a Launch.
struct LaunchSpec {
    int ntaps;
    signed char dy[MAX_TAPS], dx[MAX_TAPS], tmap[MAX_TAPS];
    short wtap[MAX_TAPS];
    int chunks0, chunks1;
    int nviews;
    View a[4];                          // activation views, indexed by tmap
    View w;
    int ncols;                          // GEMM N: cout, or 4 x cout for the merged transposed conv
    int dom_h, dom_w;
    int oy_mul, oy_add, ox_mul, ox_add, phase_cols;
    int n_tile;

    void tap(int y, int x, int view, int wt)
    {
        dy[ntaps] = (signed char)y; dx[ntaps] = (signed char)x; tmap[ntaps] = (signed char)view; wtap[ntaps] = (short)wt;
        ntaps++;
    }
};

}  // namespace

struct lwb_conv_plan {
    int num;
    Launch launches[4];
};

// Padded channels per pixel of a row-K stem input: 8 (one K stage per filter row), 16 or 24 (two or three).
static bool rowk_cin(int cin0) { return cin0 == 8 || cin0 == 16 || cin0 == 24; }

// NHWC activation view of every step-th pixel from (py, px): element (y', x') = input (step y' + py, step x' + px).
// step 1 is the plain view, step 2 the parity views of stride-2 convs.
static View nhwc_view(const uint16_t* hi, const uint16_t* lo, int n, int h, int w, int c, int step = 1, int py = 0, int px = 0)
{
    const size_t off = ((size_t)py * w + px) * c;
    return View{hi + off, lo ? lo + off : lo,
                {(uint64_t)c, (uint64_t)((w - px + step - 1) / step), (uint64_t)((h - py + step - 1) / step), (uint64_t)n},
                {(uint64_t)step * c * 2, (uint64_t)step * w * c * 2, (uint64_t)h * w * c * 2}};
}

// Weights [taps][ncols][k] fp16.
static View weight_view(const uint16_t* hi, const uint16_t* lo, int k, int ncols, int taps)
{
    return View{hi, lo, {(uint64_t)k, (uint64_t)ncols, (uint64_t)taps}, {(uint64_t)k * 2, (uint64_t)ncols * k * 2}};
}

// Encodes the hi map of a view, and in split mode its lo map.
static int encode_pair(CUtensorMap* hi, CUtensorMap* lo, int rank, const View& v, const uint32_t* box, bool split)
{
    const int rc = encode_map(hi, v.hi, rank, v.dims, v.str, box);
    return rc != LWB_OK || !split ? rc : encode_map(lo, v.lo, rank, v.dims, v.str, box);
}

// Orders the taps of p into y-halo groups: taps that read the same input view (tmap) at the same dx with consecutive
// ascending dy share one activation box (at most MAX_GROUP taps per group; a tap that matches nothing is a group of
// one).  wtap keeps addressing the weights, so the order of the taps is free.  Sets the groups and a_rows (boxes of
// tile_h output rows plus the group's halo).
static void group_taps(ConvParams& p, int tile_h)
{
    int order[MAX_TAPS];
    for (int t = 0; t < p.ntaps; t++) order[t] = t;
    std::stable_sort(order, order + p.ntaps, [&](int a, int b) {
        if (p.tmap[a] != p.tmap[b]) return p.tmap[a] < p.tmap[b];
        if (p.dx[a] != p.dx[b]) return p.dx[a] < p.dx[b];
        return p.dy[a] < p.dy[b];
    });
    const ConvParams src = p;
    int longest = 0;
    p.ngroups = 0;
    for (int t = 0; t < p.ntaps; t++) {
        const int o = order[t];
        p.dy[t] = src.dy[o]; p.dx[t] = src.dx[o]; p.tmap[t] = src.tmap[o]; p.wtap[t] = src.wtap[o];
        const bool joins = t > 0 && p.tmap[t] == p.tmap[t - 1] && p.dx[t] == p.dx[t - 1] && p.dy[t] == p.dy[t - 1] + 1 &&
                           p.g_cnt[p.ngroups - 1] < MAX_GROUP;
        if (!joins) { p.g_first[p.ngroups] = (signed char)t; p.g_cnt[p.ngroups] = 0; p.ngroups++; }
        p.g_cnt[p.ngroups - 1]++;
        longest = std::max(longest, (int)p.g_cnt[p.ngroups - 1]);
    }
    p.a_rows = tile_h + longest - 1;
}

// Ring depths inside RING_BYTES: at least two entries per ring (the consumers release an entry one wgmma group late),
// otherwise the split that keeps the most taps in flight, min(A entries x longest group, B entries).  With the 32-row
// tiles of the swapped orientation the activation entry is the large one (fp16f8 3x3: 2 x 68 KB A + 4 x 16 KB B).
static void pick_rings(ConvParams& p, int n_tile, bool split)
{
    const int ops = split ? 2 : 1;
    const int a_bytes = p.a_rows * ROW_BYTES * ops, b_bytes = n_tile * 128 * ops;
    const int longest = p.a_rows - tile_rows(n_tile) + 1;
    int best = 0;
    for (int a = 2; a <= MAX_STAGES; a++) {
        const int b = std::min(MAX_STAGES, (RING_BYTES - a * a_bytes) / b_bytes);
        if (b < 2) break;
        if (std::min(a * longest, b) > best) { best = std::min(a * longest, b); p.a_stages = a; p.b_stages = b; }
    }
}

// The one path from a spec to a launch: y-halo groups, TMA maps, tile grid, ring depths and grid size.
static int build_launch(Launch& L, const LaunchSpec& s, const lwb_conv_desc* d, float* out_raw, double* stats, int sms)
{
    const bool split = d->split != 0;
    ConvParams& p = L.p;
    memset(&p, 0, sizeof(p));
    p.ntaps = s.ntaps; p.chunks0 = s.chunks0; p.chunks1 = s.chunks1;
    for (int t = 0; t < s.ntaps; t++) { p.dy[t] = s.dy[t]; p.dx[t] = s.dx[t]; p.tmap[t] = s.tmap[t]; p.wtap[t] = s.wtap[t]; }
    group_taps(p, tile_rows(s.n_tile));
    int rc;
    const uint32_t a_box[4] = {KCHUNK, TILE_W, (uint32_t)p.a_rows, 1};
    for (int v = 0; v < s.nviews; v++)
        if ((rc = encode_pair(&p.a_hi[v], &p.a_lo[v], 4, s.a[v], a_box, split)) != LWB_OK) return rc;
    const uint32_t w_box[3] = {KCHUNK, (uint32_t)s.n_tile, 1};
    if ((rc = encode_pair(&p.w_hi, &p.w_lo, 3, s.w, w_box, split)) != LWB_OK) return rc;
    p.n_img = d->n;
    p.dom_h = s.dom_h; p.dom_w = s.dom_w;
    p.tiles_y = lwb::ceil_div(s.dom_h, tile_rows(s.n_tile)); p.tiles_x = lwb::ceil_div(s.dom_w, TILE_W);
    p.n_tiles_n = s.ncols / s.n_tile;
    p.out = out_raw; p.out_h = d->h_out; p.out_w = d->w_out; p.cout = d->cout;
    p.oy_mul = s.oy_mul; p.oy_add = s.oy_add; p.ox_mul = s.ox_mul; p.ox_add = s.ox_add; p.phase_cols = s.phase_cols;
    p.stats = stats;
    p.out_scale = ldexpf(1.f, -d->w_exp);      // weights are packed x 2^w_exp in every operand mode (lwb_pack_conv_weight*)
    L.n_tile = s.n_tile; L.mode = d->split;
    pick_rings(p, s.n_tile, split);
    const long total = (long)p.n_img * p.tiles_y * p.tiles_x * p.n_tiles_n;
    L.grid = (int)(total < sms ? total : sms);
    return LWB_OK;
}

extern "C" int lwb_conv_plan_create(const lwb_conv_desc* d,
                                    const uint16_t* x0_hi, const uint16_t* x0_lo,
                                    const uint16_t* x1_hi, const uint16_t* x1_lo,
                                    const uint16_t* w_hi, const uint16_t* w_lo,
                                    float* out_raw, double* stats, lwb_conv_plan** plan_out)
{
    LWB_CHECK_ARG(d && x0_hi && w_hi && out_raw && plan_out, "null pointer");
    const bool split = d->split != 0;
    const bool f8 = d->split == 2;     // lo operands are fp8 pairs (lwb_pack_conv_weight_f8 / lo_format 1 of lwb_norm_act_nhwc)
    LWB_CHECK_ARG(d->split >= 0 && d->split <= 2, "split must be 0, 1 or 2");
    LWB_CHECK_ARG(!split || (x0_lo && w_lo), "split mode needs the lo operands");
    LWB_CHECK_ARG(!f8 || (!d->rowk && !d->halo), "the fp8 lo mode is not available for row-K / halo plans");
    LWB_CHECK_ARG(d->n > 0 && d->h_in > 0 && d->w_in > 0 && d->cout > 0, "non-positive size");
    LWB_CHECK_ARG(d->cout % 16 == 0, "cout must be a multiple of 16");
    LWB_CHECK_ARG(d->w_exp >= -40 && d->w_exp <= 60, "w_exp out of range");
    const int n_tile = pick_n_tile(d->cout, d->n_tile);
    LWB_CHECK_ARG(n_tile > 0 && d->cout % n_tile == 0, "no N tile divides cout");
    if (d->halo) {
        // halo plans ("same"-padded stride-1 k x k convs and the row-K stem) run through the tap-group kernel below
        LWB_CHECK_ARG(d->stride == 1 && !d->transposed && d->dil == 1, "halo mode needs stride 1, dilation 1, not transposed");
        if (d->rowk) LWB_CHECK_ARG(d->kw <= 8 && rowk_cin(d->cin0) && d->cin1 == 0 && d->row_pitch >= d->w_in + 8, "row-K shape");
        else         LWB_CHECK_ARG(d->kw <= 9 && (d->kw & 1) && (d->kh & 1), "halo mode needs an odd kernel, kw <= 9, with 'same' padding (kh/2, kw/2)");
    }

    const int sms = lwb::sm_count();

    // Every variant starts from one stride-1 pass over the output grid with N = cout.
    LaunchSpec s = {};
    s.n_tile = n_tile; s.ncols = d->cout;
    s.dom_h = d->h_out; s.dom_w = d->w_out;
    s.oy_mul = s.ox_mul = 1;
    s.nviews = 1;
    LaunchSpec specs[4];
    int num = 1;
    if (d->rowk) {
        // 7x7 stem through the row-K trick.  Input: padded NHWC buffer [n, h_in + kh - 1, wp, cpx] (cpx = cin0 = 8, 16
        // or 24 channels per pixel) whose pixel (y + pad, x + pad) holds input pixel (y, x); wp >= w_in + 8.  8
        // consecutive pixels of a padded row are 8 cpx contiguous fp16 = one whole filter row (taps kx >= kw weigh 0):
        // K = 8 cpx per filter row, in cpx / 8 stages of 64.  The activation view steps one pixel (cpx elements) per
        // output column and spans 8 cpx elements, so stage c of output pixel x reads pixels x + 8c/cpx ..; the packed
        // weights [ky][cout][kx * cpx + c] (lwb_pack_conv_weight_rowk, cpx) follow the same K order.
        LWB_CHECK_ARG(d->stride == 1 && !d->transposed && d->kw <= 8, "row-K needs stride 1, kw <= 8, 8 channels");
        LWB_CHECK_ARG(rowk_cin(d->cin0) && d->cin1 == 0, "row-K needs 8, 16 or 24 padded input channels in one input");
        LWB_CHECK_ARG(d->h_out == d->h_in && d->w_out == d->w_in && d->row_pitch >= d->w_in + 8, "row-K shape");
        for (int ky = 0; ky < d->kh; ky++) s.tap(ky, 0, 0, ky);
        const int k_row = 8 * d->cin0;                       // K of one filter row
        s.chunks0 = k_row / KCHUNK;
        const uint64_t hp = d->h_in + d->kh - 1, px_bytes = (uint64_t)d->cin0 * 2, row_bytes = (uint64_t)d->row_pitch * px_bytes;
        s.a[0] = View{x0_hi, x0_lo, {(uint64_t)k_row, (uint64_t)d->w_in, hp, (uint64_t)d->n}, {px_bytes, row_bytes, hp * row_bytes}};
        s.w = weight_view(w_hi, w_lo, k_row, d->cout, d->kh);
    } else {
        LWB_CHECK_ARG(d->cin0 % KCHUNK == 0 && d->cin1 % KCHUNK == 0 && d->cin0 > 0, "input channels must be multiples of 64");
        LWB_CHECK_ARG(d->cin1 == 0 || (x1_hi && (!split || x1_lo)), "second input missing");
        const int cin_total = d->cin0 + d->cin1;
        const int ntaps_w = d->kh * d->kw;
        LWB_CHECK_ARG(ntaps_w <= MAX_TAPS, "too many filter taps");
        s.chunks0 = d->cin0 / KCHUNK; s.chunks1 = d->cin1 / KCHUNK;
        s.a[0] = nhwc_view(x0_hi, x0_lo, d->n, d->h_in, d->w_in, d->cin0);
        s.w = weight_view(w_hi, w_lo, cin_total, d->cout, ntaps_w);
        if (d->transposed) {
            // both transposed forms tile the input grid and write output pixel (2y + a, 2x + b)
            LWB_CHECK_ARG(d->kh == 3 && d->kw == 3 && d->stride == 2 && d->pad == 1 && d->cin1 == 0, "transposed conv: only k3 s2 p1 op1");
            LWB_CHECK_ARG(d->h_out == 2 * d->h_in && d->w_out == 2 * d->w_in, "transposed conv output must be 2x input");
            s.dom_h = d->h_in; s.dom_w = d->w_in;
            s.oy_mul = s.ox_mul = 2;
        }
        if (d->transposed == 2) {
            // Merged transposed conv: ONE stride-1 pass over the input grid with the four taps (dy, dx) in {0,1}^2 and
            // N = 4 x cout columns = the four sub-pixel phases (weights from the host in [tap][phase*cout + co][cin] layout,
            // zero where a phase does not use a tap: 9 of 16 blocks are non-zero).  One launch, one read of every input tile.
            s.n_tile = MAX_N_TILE;
            s.ncols = 4 * d->cout;
            LWB_CHECK_ARG(d->cout % 32 == 0 && s.ncols % s.n_tile == 0, "merged transposed conv needs cout in multiples of 32");
            for (int t = 0; t < 4; t++) s.tap(t >> 1, t & 1, 0, t);
            s.w = weight_view(w_hi, w_lo, cin_total, s.ncols, 4);
            s.phase_cols = d->cout;
        } else if (d->transposed) {
            // ConvTranspose2d(k=3, s=2, p=1, output_padding=1): out[2i+a, 2j+b] gathers, per axis,
            //   a = 0: (k=1, d=0)            a = 1: (k=2, d=0), (k=0, d=+1)        (oy = 2*iy - 1 + ky)
            // one launch per sub-pixel phase (a, b)
            const int ky_list[2][2] = {{1, -1}, {2, 0}}, d_list[2][2] = {{0, 0}, {0, 1}}, cnt[2] = {1, 2};
            num = 4;
            for (int a = 0; a < 2; a++) for (int b = 0; b < 2; b++) {
                LaunchSpec& q = specs[a * 2 + b];
                q = s;
                for (int i = 0; i < cnt[a]; i++) for (int j = 0; j < cnt[b]; j++)
                    q.tap(d_list[a][i], d_list[b][j], 0, ky_list[a][i] * 3 + ky_list[b][j]);
                q.oy_add = a; q.ox_add = b;
            }
        } else {
            LWB_CHECK_ARG(d->stride == 1 || d->stride == 2, "stride must be 1 or 2");
            LWB_CHECK_ARG(d->stride == 1 || d->cin1 == 0, "concat input only with stride 1");
            const int st = d->stride;
            for (int ky = 0; ky < d->kh; ky++) for (int kx = 0; kx < d->kw; kx++) {
                const int oy = ky * d->dil - d->pad, ox = kx * d->dil - (d->pad_w >= 0 ? d->pad_w : d->pad);   // input offset relative to stride*y
                if (oy < -127 || oy > 127 || ox < -127 || ox > 127) { lwb::set_error("conv_tc: tap offset out of range"); return LWB_E_UNSUPPORTED; }
                // input coordinate st y + oy = st (y + floor(oy / st)) + (oy mod st): view (py, px) + index shift
                const int py = ((oy % st) + st) % st, px = ((ox % st) + st) % st;
                s.tap((oy - py) / st, (ox - px) / st, py * 2 + px, s.ntaps);
            }
            // stride 2 reads four parity views of the input, a concat input (stride 1 only) a second tensor
            s.nviews = st * st;
            for (int v = 0; v < s.nviews; v++) s.a[v] = nhwc_view(x0_hi, x0_lo, d->n, d->h_in, d->w_in, d->cin0, st, v >> 1, v & 1);
            if (d->cin1) {
                s.nviews = 2;
                s.a[1] = nhwc_view(x1_hi, x1_lo, d->n, d->h_in, d->w_in, d->cin1);
            }
        }
    }
    if (num == 1) specs[0] = s;

    lwb_conv_plan* plan = new (std::nothrow) lwb_conv_plan();
    LWB_CHECK_ARG(plan, "out of host memory");
    for (; plan->num < num; plan->num++) {
        const int rc = build_launch(plan->launches[plan->num], specs[plan->num], d, out_raw, stats, sms);
        if (rc != LWB_OK) { delete plan; return rc; }
    }
    *plan_out = plan;
    return LWB_OK;
}

extern "C" int lwb_conv_plan_run(const lwb_conv_plan* plan, lwb_stream_t stream)
{
    LWB_CHECK_ARG(plan, "null plan");
    for (int i = 0; i < plan->num; i++) {
        const int rc = launch(plan->launches[i], (cudaStream_t)stream);
        if (rc != LWB_OK) return rc;
    }
    return LWB_OK;
}

extern "C" void lwb_conv_plan_destroy(lwb_conv_plan* plan) { delete plan; }

extern "C" int lwb_conv_plan_num_launches(const lwb_conv_plan* plan) { return plan ? plan->num : 0; }

extern "C" int lwb_conv_plan_launch_info(const lwb_conv_plan* plan, int i, int* out)
{
    LWB_CHECK_ARG(plan && out, "null pointer");
    LWB_CHECK_ARG(i >= 0 && i < plan->num, "launch index out of range");
    const Launch& L = plan->launches[i];
    out[0] = L.n_tile; out[1] = L.mode; out[2] = L.p.chunks0 + L.p.chunks1; out[3] = L.p.ntaps;
    return LWB_OK;
}

extern "C" int lwb_conv2d_nhwc(const lwb_conv_desc* d,
                               const uint16_t* x0_hi, const uint16_t* x0_lo,
                               const uint16_t* x1_hi, const uint16_t* x1_lo,
                               const uint16_t* w_hi, const uint16_t* w_lo,
                               float* out_raw, double* stats, lwb_stream_t stream)
{
    lwb_conv_plan* plan = nullptr;
    int rc = lwb_conv_plan_create(d, x0_hi, x0_lo, x1_hi, x1_lo, w_hi, w_lo, out_raw, stats, &plan);
    if (rc != LWB_OK) return rc;
    rc = lwb_conv_plan_run(plan, stream);
    lwb_conv_plan_destroy(plan);
    return rc;
}

// Resources of one k_conv_wg instance as launched: [registers per thread at launch, static smem, dynamic smem, local
// bytes per thread, threads per CTA, CTAs per SM alone (occupancy API), consumer registers after setmaxnreg].
template <int N_TILE, int MODE>
static int conv_resources(int* out)
{
    using C = Cfg<N_TILE, MODE != MODE_FP16>;
    cudaFuncAttributes a;
    LWB_CUDA_OK(cudaFuncSetAttribute(k_conv_wg<N_TILE, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    LWB_CUDA_OK(cudaFuncGetAttributes(&a, k_conv_wg<N_TILE, MODE>));
    int blocks = 0;
    LWB_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, k_conv_wg<N_TILE, MODE>, NUM_THREADS, C::SMEM_BYTES));
    out[0] = a.numRegs; out[1] = (int)a.sharedSizeBytes; out[2] = C::SMEM_BYTES; out[3] = (int)a.localSizeBytes;
    out[4] = NUM_THREADS; out[5] = blocks; out[6] = Regs<N_TILE, MODE>::CONSUMER;
    return LWB_OK;
}

extern "C" int lwb_conv_kernel_resources(int n_tile, int mode, int* out)
{
    LWB_CHECK_ARG(out, "null pointer");
    LWB_CHECK_ARG(mode >= 0 && mode <= 2, "mode must be 0, 1 or 2");
    return with_instance(n_tile, mode,
                         [&](auto nt, auto md) { return conv_resources<decltype(nt)::value, decltype(md)::value>(out); });
}
