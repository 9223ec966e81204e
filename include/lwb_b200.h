/*
 * lwb_b200 -- C ABI of the Liquid-Warping hot path on the H100 (sm_90a).
 *
 * Drop-in boundary for svip-lab/impersonator's per-frame inference path.  Every entry point
 * takes plain device pointers + sizes and a cudaStream_t (passed as void*), returns 0 on
 * success or a negative LWB_E_* code (lwb_last_error() gives the text).  No torch types.
 * All launches are asynchronous on the caller's stream; nothing here synchronises.
 *
 * Each declaration cites the reference interface (file:line under /root/reference) it replaces.
 */
#ifndef LWB_B200_H_
#define LWB_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LWB_OK            0
#define LWB_E_INVALID    -1   /* bad argument (null pointer, unsupported size) */
#define LWB_E_CUDA       -2   /* a CUDA runtime/driver call failed */
#define LWB_E_UNSUPPORTED -3  /* shape outside what the kernels were built for */

/* Bits of the operand-range flag (the range_flag arguments below) */
#define LWB_RANGE_F8      1   /* an emitted operand has |y| >= 1024: its e4m3 correction terms clip */
#define LWB_RANGE_FP16    2   /* an emitted operand has |y| >= 60000 or is not finite: the fp16 hi itself overflows */
#define LWB_RANGE_HEADS   4   /* a head pre-activation reached +-8 */

typedef void* lwb_stream_t;   /* cudaStream_t */

int         lwb_version(void);
const char* lwb_last_error(void);
/* SM count / compute capability of the current device (0 when no device): lets the host fail loudly. */
int         lwb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------------
 * Rasterizer.  Replaces the pybind11 entry point
 *   neural_renderer.cuda.rasterize.forward_face_index_map
 *   thirdparty/neural_renderer/neural_renderer/cuda/rasterize_cuda.cpp:70-95  (launcher
 *   rasterize_cuda_kernel.cu:613-668, kernels :40-186), as called from rasterize.py:164-169.
 * Same contract: the caller allocates and pre-fills face_index_map (-1), weight_map (0),
 * depth_map (far); only covered pixels are written.  faces_inv (nullable) receives kernel_1's
 * per-face inverse matrices (caller zero-fills, culled faces are left untouched).
 * flip_rows = 0 gives the native kernel's row order (row 0 = bottom, +y up); flip_rows = 1 writes
 * row (H-1-y) instead, i.e. folds the torch.flip of rasterize.py:334-338 into the store.
 * workspace: lwb_raster_workspace_bytes(batch, image_size, num_faces) bytes of device scratch
 * (64-bit z-buffer + a queue for degenerate faces that need a whole-image scan).
 * face_index_map is bit-exact with the reference kernels compiled by the same nvcc.
 * ------------------------------------------------------------------------------------------ */
size_t lwb_raster_workspace_bytes(int batch, int image_size, int num_faces);
int lwb_raster_forward_face_index_map(
        const float* faces /* [B,F,3,3] */, int batch, int num_faces, int image_size,
        float near, float far,
        int32_t* face_index_map /* [B,H,W] */, float* weight_map /* [B,H,W,3] */,
        float* depth_map /* [B,H,W], nullable */, float* faces_inv /* [B,F,3,3], nullable */,
        int flip_rows, void* workspace, lwb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused correspondence pass = SMPLRenderer.render_fim_wim + encode_fim + cal_bc_transform +
 * the image-level warp and concat of Imitator.transfer_params_by_smpl:
 *   utils/nmr.py:263-278 (proj :10-28, y-flip :271, look_at look_at.py:48-60 with the constant
 *   eye of utils/nmr.py:177, gather vertices_to_faces.py:17-21), rasterize.py:22-98,334-338,
 *   utils/nmr.py:328-341, utils/nmr.py:617-659, models/imitator.py:259-260.
 * Inputs : cam [B,3] = (s,tx,ty); verts [B,V,3]; face_idx [F,3] (shared by the batch);
 *          map_fn [(F+1), map_c] (row F = background, hit by fim == -1);
 *          src_p2verts [src_batch,F,3,2] with src_batch in {1,B} (models/imitator.py:105-107);
 *          src_img [src_batch,3,H,W] (nullable -> no image warp).
 * Outputs: fim i32 [B,H,W], wim [B,H,W,3] (top row first, i.e. after the flips),
 *          T [B,H,W,2] (-2 where uncovered), tsf_inputs [B,3+map_c,H,W] = cat[tsf_img, cond]
 *          (channels 0..2 = grid_sample(src_img, T), 3.. = cond), f2verts [B,F,3,3] (nullable).
 *          All outputs are fully written (no pre-fill needed).
 * align_corners selects the grid_sample convention (0 = torch>=1.3 default, the oracle;
 * 1 = torch 1.2 behaviour the reference was written against).
 * ------------------------------------------------------------------------------------------ */
int lwb_correspond(
        const float* cam, const float* verts, const int32_t* face_idx,
        int batch, int num_verts, int num_faces, int image_size, float near, float far,
        float eye_z /* z of the look_at eye, utils/nmr.py:177, as float32 */,
        const float* map_fn, int map_c,
        const float* src_p2verts, const float* src_img, int src_batch, int align_corners,
        int32_t* fim, float* wim, float* T, float* tsf_inputs, float* f2verts,
        void* workspace, lwb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Bilinear warp = ImpersonatorGenerator.transform / stn / resize_trans
 *   networks/generator.py:303-320 (F.interpolate(T, (h,w), bilinear, align_corners=True) followed
 *   by F.grid_sample(x, T_scale), zeros padding) and models/imitator.py:259.
 * x [src_batch,C,h,w] NCHW fp32 (src_batch in {1,B}: one source broadcast over the frame batch,
 * which torch's grid_sampler cannot do), T [B,TH,TW,2].  When (TH,TW) != (h,w) the flow is
 * resized on the fly (transform); out [B,C,h,w].  accumulate != 0 adds into out (the "+ warp").
 * ------------------------------------------------------------------------------------------ */
int lwb_warp_nchw(const float* x, int src_batch, int channels, int h, int w,
                  const float* T, int batch, int th, int tw, int align_corners,
                  float* out, int accumulate, lwb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Conv engine (NHWC, wgmma implicit GEMM).  Replaces the cuDNN calls behind nn.Conv2d /
 * nn.ConvTranspose2d / nn.InstanceNorm2d of networks/generator.py:8-20,77-134,163-184.
 * Activations are channels-last pairs (hi = fp16(x), lo = 2 more bytes per element) so that the
 * products hi*hi + x*w_lo + x_lo*w (fp32 accumulate) reproduce fp32 convolution to ~1e-5 per layer
 * (SURVEY.md section 0 fact 4): split = 1 keeps lo in fp16 and issues three fp16 tensor-core passes,
 * split = 2 keeps the two correction operands in e4m3 and issues them as one fp8 pass, split = 0
 * runs the single hi*hi pass ("fast" mode, not parity-gated).
 * ------------------------------------------------------------------------------------------ */

/* Repack an OIHW (Conv2d) or IOHW (ConvTranspose2d, transposed != 0) fp32 weight into the
 * engine's [tap][Cout_pad][Cin_pad] fp16 hi/lo layout (done once at load time): w_hi = fp16(w * 2^w_exp),
 * w_lo = fp16(w * 2^w_exp - w_hi).  w_lo nullable.  The caller picks w_exp as for lwb_pack_conv_weight_f8 (max|w| * 2^w_exp
 * in [2^14, 2^15), so that small weights do not fall into the fp16 subnormals) and passes the same value in
 * lwb_conv_desc.w_exp; w_exp = 0 packs the weights unscaled. */
int lwb_pack_conv_weight(const float* w, int cout, int cin, int kh, int kw, int transposed,
                         int cout_pad, int cin_pad, int w_exp, uint16_t* w_hi, uint16_t* w_lo, lwb_stream_t stream);
/* Weights for the "fp16 + fp8" operand split (lwb_conv_desc.split = 2): w_hi [taps][cout_pad][cin_pad] fp16 holds
 * fp16(w) * 2^w_exp; w_lo8 (same byte size) holds, per 64-input-channel block of 128 bytes,
 * 64 x e4m3((w - fp16(w)) * 2^(w_exp+4)) followed by 64 x e4m3(w * 2^(w_exp-10)).  The caller picks the layer's w_exp
 * with max|w| * 2^w_exp in [2^14, 2^15) (any weight magnitude packs; 15 for |w| in [0.5, 1)) and passes the same
 * value in lwb_conv_desc.w_exp.  cin_pad % 64 == 0.  See DESIGN.md section 4. */
int lwb_pack_conv_weight_f8(const float* w, int cout, int cin, int kh, int kw, int transposed,
                            int cout_pad, int cin_pad, int w_exp, uint16_t* w_hi, uint8_t* w_lo8, lwb_stream_t stream);

/* Row-K packing for the 7x7 stem: [ky][cout_pad][kxs*cpx], K index = kx*cpx + c (zero beyond kw / cin), hi/lo of
 * w * 2^w_exp as in lwb_pack_conv_weight. */
int lwb_pack_conv_weight_rowk(const float* w, int cout, int cin, int kh, int kw,
                              int cout_pad, int cpx, int kxs, int w_exp, uint16_t* w_hi, uint16_t* w_lo, lwb_stream_t stream);

/* NCHW fp32 -> NHWC fp16 hi/lo [n, hp, wp, c_pad]; input pixel (y,x) lands at (y+oy, x+ox), the rest
 * (spatial border, channels >= c) is zero.  hp >= h+oy, wp >= w+ox.  lo nullable. */
int lwb_nchw_to_nhwc_split(const float* x, int n, int c, int h, int w, int c_pad,
                           int hp, int wp, int oy, int ox,
                           uint16_t* hi, uint16_t* lo, lwb_stream_t stream);
/* NHWC fp32 [n,h,w,c_stride] (first c channels) -> NCHW fp32 [n,c,h,w]. */
int lwb_nhwc_to_nchw(const float* x, int n, int c, int h, int w, int c_stride, float* out, lwb_stream_t stream);

typedef struct lwb_conv_desc {
    int n, h_in, w_in;        /* input  [n, h_in, w_in, cin]  (NHWC fp16 hi/lo) */
    int h_out, w_out;         /* output [n, h_out, w_out, cout] (NHWC fp32, raw conv result) */
    int cin0, cin1;           /* channels of input 0 / input 1 (virtual torch.cat, cin1 = 0 if single); x64 */
    int cout;                 /* multiple of 16 */
    int kh, kw, stride, pad, dil;
    int transposed;           /* 1: ConvTranspose2d(k=3, s=2, p=1, output_padding=1) as four sub-pixel phase launches, weights
                                 packed from IOHW (lwb_pack_conv_weight, transposed = 1).  2: the same layer as ONE stride-1
                                 pass over the input grid: weights [4 taps (dy,dx)][4*cout][cin] (phase 2a+b of output pixel
                                 (2y+a, 2x+b) in column block 2a+b; zero blocks where a phase does not use a tap), packed as
                                 an ordinary OIHW [4*cout, cin, 2, 2] filter; cout % 32 == 0, cout <= 128 recommended */
    int split;                /* 1 = 3-pass fp16 split (parity mode), 0 = single pass ("fast"), 2 = fp16 main product +
                                 both small products in fp8 (lo operands from lwb_pack_conv_weight_f8 / lo_format 1) */
    int rowk;                 /* 1 = 7x7-stem row-K mode: input is a padded NHWC buffer of cin0 = 8, 16 or 24 channels
                                 (see conv_tc.cu), weights from lwb_pack_conv_weight_rowk with cpx = cin0, kxs = 8 */
    int row_pitch;            /* rowk: pixels per padded row (>= w_in + 8) */
    int n_tile;               /* 0 = auto; else force the N tile (16/32/64/128, must divide cout; 256 runs as 128) */
    int halo;                 /* 1 = halo plan (stride-1 'same' k x k convs and the row-K stem): checked as such, then run
                                 by the same tap-group kernel as halo = 0 */
    int w_exp;                /* the power of two the weights were packed with (lwb_pack_conv_weight*), every split; the
                                 output is scaled by 2^-w_exp.  In [-40, 60] */
    int pad_w;                /* horizontal padding when it differs from pad (e.g. a 7x1 filter); -1 = same as pad */
} lwb_conv_desc;

/* A plan owns the TMA descriptors of one conv layer bound to fixed device buffers; creating it
 * costs a few driver calls, running it is one launch (four for a transposed conv).
 * out_raw = conv(x) (no bias); stats [n, cout, 2] f64 += per-(n,c) (sum, sum of squares) over
 * H*W (nullable; caller zero-fills) -- the InstanceNorm statistics, accumulated by the conv epilogue. */
typedef struct lwb_conv_plan lwb_conv_plan;
int  lwb_conv_plan_create(const lwb_conv_desc* d,
                          const uint16_t* x0_hi, const uint16_t* x0_lo,
                          const uint16_t* x1_hi, const uint16_t* x1_lo,
                          const uint16_t* w_hi, const uint16_t* w_lo,
                          float* out_raw, double* stats, lwb_conv_plan** plan);
int  lwb_conv_plan_run(const lwb_conv_plan* plan, lwb_stream_t stream);
int  lwb_conv_plan_num_launches(const lwb_conv_plan* plan);
/* The kernel instance and K loop of launch i of a plan: out[4] = {N tile, operand mode, K stages of 64 per filter tap,
 * filter taps}.  A row-K stem over 8 / 16 / 24 padded channels has 1 / 2 / 3 K stages per tap (one tap per filter row). */
int  lwb_conv_plan_launch_info(const lwb_conv_plan* plan, int i, int* out);
void lwb_conv_plan_destroy(lwb_conv_plan* plan);
/* Resources of the conv kernel instance (n_tile 16/32/64/128, mode = lwb_conv_desc.split) as launched:
 * out[7] = {registers per thread at launch, static smem, dynamic smem, local bytes per thread, threads per CTA,
 * CTAs per SM alone, consumer registers per thread after setmaxnreg}.  Needs a device. */
int  lwb_conv_kernel_resources(int n_tile, int mode, int* out);
/* create + run + destroy */
int lwb_conv2d_nhwc(const lwb_conv_desc* d,
                    const uint16_t* x0_hi, const uint16_t* x0_lo,
                    const uint16_t* x1_hi, const uint16_t* x1_lo,
                    const uint16_t* w_hi, const uint16_t* w_lo,
                    float* out_raw, double* stats, lwb_stream_t stream);

/* Per-(n,c) sum / sum-of-squares of an NHWC fp32 tensor into stats [n,c,2] f64 (+=, caller zero-fills):
 * the InstanceNorm statistics for tensors that did not come out of lwb_conv2d_nhwc. */
int lwb_instance_stats_nhwc(const float* x, int n, int h, int w, int c, double* stats, lwb_stream_t stream);

/* InstanceNorm2d(affine, eps) [+ ReLU] [+ residual] [+ LWB warp] applied to a raw conv output,
 * emitting the next layer's operands:  y = act(gamma*(x-mean)*rstd + beta) + res + warp(src, T)
 *   networks/generator.py:13-20 (ResidualBlock), :80-95 (encoders), :283-295 (the "+ warp" of the LWB).
 * raw [n,h,w,c] fp32; stats from the conv epilogue (nullable -> no normalisation); gamma/beta [c];
 * residual (nullable) [n,h,w,c] fp32; warp_src (nullable) [src_batch,h,w,c] fp32 NHWC sampled at
 * T [n,TH,TW,2] resized to (h,w) (generator.py:303-320).  scale_shift_ws: [n,c,2] f32 scratch.
 * Outputs (each nullable): y_f32 [n,h,w,c]; y_hi / y_lo fp16 [n,h,w,c].  c % 8 == 0.
 * lo_format 0: y_lo = fp16(y - y_hi).  lo_format 1 (c % 64 == 0; consumers are split = 2 conv plans): y_lo holds, per
 * pixel and 64-channel block of 128 bytes, 64 x e4m3(y * 2^-4) followed by 64 x e4m3((y - y_hi) * 2^10).
 * stats == NULL with gamma / beta given: plain per-channel affine y = x*gamma[c] + beta[c] (eval-mode BatchNorm folded,
 * or a conv bias: networks/hmr.py:66-103).  post_scale / post_shift [c] (nullable): the OPERANDS (y_hi / y_lo) hold
 * relu?(y*post_scale + post_shift) while y_f32 keeps y (pre-activation ResNets: the next block's bn1+relu).
 * res_step s > 1: residual is [n, h*s, w*s, c] and is read at (s*y, s*x) (the subsampled identity shortcut, hmr.py:21-36).
 * range_flag (nullable, device int, caller zero-fills): |= LWB_RANGE_F8 when an emitted operand has |y| >= 1024 (the e4m3
 * correction terms clip: precision of those elements degrades towards single-pass fp16), |= LWB_RANGE_F8 | LWB_RANGE_FP16
 * when |y| >= 60000 or not finite. */
int lwb_norm_act_nhwc(const float* raw, const double* stats, const float* gamma, const float* beta,
                      float eps, int relu, int n, int h, int w, int c,
                      const float* residual,
                      const float* warp_src, int src_batch, const float* T, int th, int tw, int align_corners,
                      float* scale_shift_ws,
                      float* y_f32, uint16_t* y_hi, uint16_t* y_lo, int lo_format,
                      const float* post_scale, const float* post_shift, int post_relu, int res_step,
                      int* range_flag, lwb_stream_t stream);

/* 7x7 output heads of the generator (networks/generator.py:126-134): img_reg (64->3) and
 * attetion_reg (64->1) as ONE 64->4 convolution, x [n,h,w,64] fp32 NHWC, w4 [49][64][4] fp32
 * (tap-major, output channel innermost: 0..2 = img_reg, 3 = attetion_reg), out [n,h,w,4] fp32. */
int lwb_pack_head_weights(const float* w_img /* [3,64,7,7] */, const float* w_att /* [1,64,7,7] */,
                          float* w4, lwb_stream_t stream);
int lwb_conv7x7_heads_nhwc(const float* x, const float* w4, int n, int h, int w, float* out, lwb_stream_t stream);

/* Resources of the HBM-bound kernels launched beside the convolutions: which = 0 lwb_norm_act_nhwc (plain),
 * 1 its warp variant at c channels, 2 its post-affine / strided-residual variant, 3 lwb_heads_composite,
 * 4 lwb_nchw_to_nhwc_split.  out[6] = the first six entries of lwb_conv_kernel_resources.  Needs a device. */
int lwb_glue_kernel_resources(int which, int c, int* out);

/* Output heads + composite:  color = tanh(raw[...,0:3]), mask = sigmoid(raw[...,3]),
 * pred = mask*bg + (1-mask)*color   (networks/generator.py:183-184, models/imitator.py:330-331).
 * raw [n,h,w,c_stride] fp32 NHWC (channels 0..3 used); bg [bg_batch,3,h,w] NCHW (nullable -> no pred).
 * color [n,3,h,w], mask [n,1,h,w], pred [n,3,h,w] NCHW, each nullable.
 * Output path (SURVEY.md 8f rank 2), each nullable: pred_hwc [n,h,w,3] fp32 = preds.permute(1,2,0) of
 * models/imitator.py:178-180; pred_u8_bgr [n,h,w,3] uint8 = the image cv_utils.save_cv2_img(normalize=True) hands to
 * cv2.imwrite (utils/cv_utils.py:23-36: RGB->BGR, ((x+1)/2*255) in fp32, truncated).
 * folded_kw = 0: raw[...,0:4] are the four head channels.  folded_kw = kw (7): raw is the output of the 7x7 heads run on
 * the tensor cores as a kh x 1 filter whose N dimension carries the filter columns, raw[y,x',kx*4+co] (c_stride >= 4*kw);
 * the row sum  out[y,x,co] = sum_kx raw[y, x+kx-kw/2, kx*4+co]  happens here, before tanh / sigmoid.
 * range_flag (nullable, device int): |= LWB_RANGE_HEADS when a head pre-activation reaches +-8 -- beyond that the ~1e-4 relative
 * end-to-end precision of the split = 2 operand mode no longer guarantees 1e-3 on the pixels (use split = 1). */
int lwb_heads_composite(const float* raw, int n, int h, int w, int c_stride, int folded_kw,
                        const float* bg, int bg_batch,
                        float* color, float* mask, float* pred,
                        float* pred_hwc, uint8_t* pred_u8_bgr, int* range_flag, lwb_stream_t stream);

/* The same output-path conversion for frames [n,3,h,w] NCHW fp32 that did not come straight out of the heads
 * (e.g. after Imitator.warp_front, models/imitator.py:338-342). */
int lwb_frames_out(const float* frames, int n, int h, int w, float* hwc, uint8_t* u8_bgr, lwb_stream_t stream);

/* Input path: n uint8 frames [n,h,w,3] (bgr = 1: B,G,R as cv2.imread returns them; 0: R,G,B), all one size, resized the
 * way cv2.resize(frame, (s, s)) resizes uint8 with INTER_LINEAR -- the same bytes -- and written in one launch to any of
 *   img    [n,3,size,size]         fp32 RGB, x / 255.0 * 2 - 1.0 in fp32 (utils/cv_utils.py:10-47 + models/imitator.py:89),
 *   hmr    [n,3,hmr_size,hmr_size] fp32 RGB, the same formula, resized from the frame itself (the HMR input),
 *   u8_bgr [n,size,size,3]         uint8 BGR, what cv_utils.save_cv2_img(frame, image_size=size) hands to cv2.imwrite.
 * A null output is skipped; at least one must be given. */
int lwb_frames_in(const uint8_t* frames, int n, int h, int w, int bgr, int size, float* img, int hmr_size,
                  float* hmr, uint8_t* u8_bgr, lwb_stream_t stream);

/* Direct (CUDA-core) convolution, NCHW fp32, arbitrary kernel / stride / dilation, optional bias:
 * the once-per-source inpaintor layers (networks/inpaintor.py:12-47) and odd shapes. */
int lwb_conv2d_direct_nchw(const float* x, const float* w, const float* bias,
                           int n, int cin, int h, int wd, int cout, int kh, int kw,
                           int stride, int pad, int dil, float* out, lwb_stream_t stream);
/* The same convolution (dilation 1) with relu(out) written NHWC [n,ho,wo,cout]: LPIPS' AlexNet conv1 (11x11 s4 p2). */
int lwb_conv2d_direct_relu_nhwc(const float* x, const float* w, const float* bias,
                                int n, int cin, int h, int wd, int cout, int kh, int kw,
                                int stride, int pad, float* out, lwb_stream_t stream);

/* Gated-conv epilogue of the inpaintor (networks/inpaintor.py:37-47): ab [n,2c,h,w] = conv2d(x) and
 * mask_conv2d(x) stacked on channels; out [n,c,h,w] = (act(a) * sigmoid(b)) * scale[c] + shift[c]
 * (eval-mode BatchNorm2d folded; scale/shift nullable).  act: 0 none, 1 ReLU, 2 LeakyReLU(0.2). */
int lwb_gated_bn_nchw(const float* ab, int n, int c, int h, int w, int act,
                      const float* scale, const float* shift, float* out, lwb_stream_t stream);

/* ---- background inpaintor glue (networks/inpaintor.py; once per source image) -----------------------------------
 * Every GatedConv2dWithActivation (:12-47) = ONE conv-engine plan over the stacked [conv2d ; mask_conv2d] filters (cout =
 * 2c, padded to x16) + this epilogue:  y = BN_eval(act(a + bias[ch]) * sigmoid(b + bias[c + ch])),  a = raw[..., ch],
 * b = raw[..., c + ch].  act: 0 none, 2 LeakyReLU(0.2).  upsample 2: y is written to the 2x2 block of every pixel of a
 * [2h, 2w] grid = the nearest-neighbour resize GatedDeConv2dWithActivation convolves next (:65-68).  clamp: to [-1, 1]
 * (:187,196).  Outputs (each nullable): y_f32 [n, h*u, w*u, f32_stride] (first c channels); the next layer's operands
 * y_hi / y_lo [n, h*u, w*u, c_pad] with channels >= c zero (the engine's K chunks are 64 wide), lo_format as in
 * lwb_norm_act_nhwc; range_flag as in lwb_norm_act_nhwc. */
int lwb_gated_act_nhwc(const float* raw, int n, int h, int w, int c, int c_stride, const float* bias, int act,
                       const float* scale, const float* shift, int upsample, int clamp,
                       float* y_f32, int f32_stride, uint16_t* y_hi, uint16_t* y_lo, int c_pad, int lo_format,
                       int* range_flag, lwb_stream_t stream);
/* SelfAttention (networks/inpaintor.py:71-107) after the stacked 1x1 query / key / value convolution:
 * qkv [n, npos, ld] fp32 rows = [q (dq) | k (dq) | v (dv) | pad], bias [2*dq + dv];
 * out[i] = gamma[0] * sum_j softmax_j(q_i . k_j) v_j + x[i],  x / out [n, npos, dv] fp32.  dq = 16, dv = 128. */
int lwb_self_attention_nhwc(const float* qkv, int ld, const float* bias, int n, int npos, int dq, int dv,
                            const float* x, const float* gamma, float* out, lwb_stream_t stream);

/* ---- HMR image encoder glue (SURVEY.md 8f rank 3; networks/hmr.py:119-166, 214-252, 275-300) -----------------------
 * The pre-activation ResNet-50's convolutions run on the conv engine above (lwb_conv_plan_*; eval-mode BatchNorm folded
 * into lwb_norm_act_nhwc's per-channel affine); these three cover the rest, fp32:
 *   F.max_pool2d(x, k, stride, ceil_mode=True) (hmr.py:150), x NCHW [n,c,h,w] -> out NHWC [n,ho,wo,c], ho = ceil((h-k)/stride)+1
 *   relu?(x*scale+shift) averaged over the hw pixels (post_bn + ReLU + avg_pool2d(7), hmr.py:160-163), x NHWC [n,hw,c] ->
 *     out[b*ld_out + ch]
 *   nn.Linear (+ReLU) of the theta regressor (hmr.py:223-252): out[b*ld_out + j] (+)= relu?(x[b*ld_x + :k] . w[j,:k] + bias[j]) */
int lwb_maxpool_nchw_to_nhwc(const float* x, int n, int c, int h, int w, int k, int stride, float* out, lwb_stream_t stream);
/* F.max_pool2d(x, k, stride) in floor mode (ceil_mode=False, AlexNet's pools), x NHWC fp32 [n,h,w,c] -> [n,ho,wo,c],
 * ho = (h-k)/stride+1: fp32 (y_f32) and / or the conv engine's fp16 hi / lo operands (y_lo nullable); either may be null. */
int lwb_maxpool_nhwc(const float* x, int n, int h, int w, int c, int k, int stride, float* y_f32, void* y_hi, void* y_lo,
                     lwb_stream_t stream);
int lwb_global_avgpool_nhwc(const float* x, int n, int hw, int c, const float* scale, const float* shift, int relu,
                            float* out, int ld_out, lwb_stream_t stream);
int lwb_linear(const float* x, int ld_x, const float* w, const float* bias, int n, int k, int m, int relu, int accumulate,
               float* out, int ld_out, lwb_stream_t stream);

/* ---- SMPL body model: pose -> vertices (SURVEY.md 8f rank 1) -------------------------------------------------
 * Replaces SMPL.forward (networks/batch_smpl.py:285-375; batch_rodrigues :64-101, batch_global_rigid_transformation
 * :129-218) as called by HumanModelRecovery.get_details (networks/hmr.py:302-330).
 * beta [B,num_betas], theta [B,72] axis-angle (global rotation first).  Model tensors (device, fp32):
 *   v_template [V,3]; shapedirs [num_betas][V*3]; posedirs [207][V*3]   (the registered buffers of batch_smpl.py:254-273)
 *   j_template [24,3] = J_regressor^T v_template and j_shapedirs [24*3][num_betas] = J_regressor^T shapedirs
 *       (the joint regression of :318-321 is linear in beta, so it is folded into the model once at load time);
 *   parents int32[24] (kintree_table[0]); weights [V,24]; joint_regressor_t [num_joints][V] (cocoplus, transposed).
 * Outputs: verts [B,V,3]; joints [B,num_joints,3] (nullable); Rs [B,24,3,3] (nullable); J_transformed [B,24,3]
 * (nullable); j2d [B,num_joints,2] (nullable) = cam_s * (joints_xy + cam_t) with cam [B,3] (batch_orth_proj_idrot,
 * batch_smpl.py:221-233).  workspace: lwb_smpl_workspace_bytes(B) bytes. */
size_t lwb_smpl_workspace_bytes(int batch);
int lwb_smpl_forward(const float* beta, const float* theta, int batch, int num_betas, int num_verts,
                     const float* v_template, const float* shapedirs, const float* posedirs,
                     const float* j_template, const float* j_shapedirs, const int* parents,
                     const float* weights, const float* joint_regressor_t, int num_joints, int rotate_base,
                     float* verts, float* joints, float* Rs, float* J_transformed,
                     const float* cam, float* j2d, void* workspace, lwb_stream_t stream);

/* ---- Mask R-CNN person detector (utils/detectors.py:25-85: torchvision maskrcnn_resnet50_fpn, eval) ------------
 * The convolutions and fully connected layers run through lwb_conv_plan_*; these are the passes between them.
 * Every count lives on the device (int32), so a forward pass needs no host synchronisation.  Operands (y_hi, y_lo)
 * are the conv engine's NHWC fp16 hi / lo pair; either output of a pass may be null when not needed.
 *   transform     img [3,h,w] in [-1,1] -> (img + 1) / 2, normalised, bilinear to [ho,wo], zero padded: out [3,hp,wp]
 *   stem_pool     max_pool2d(relu(x * scale + shift), 3, 2, 1): x NCHW fp32 -> operands [n,(h+1)/2,(w+1)/2,c]
 *   bias_act      y = act(raw[step*(y,x)] + raw2 + bias + res) with res at the same grid or (res_half) nearest 2x from
 *                 [n,h/2,w/2,c]; raw / raw2 have channel pitch ld_raw on an [h_in,w_in] grid
 *   d2s_bias_relu ConvTranspose2d(k=2, s=2) from its 1x1 form: raw [n,h,w,4c], column (dy*2+dx)*c + co -> [n,2h,2w,c]
 *   rpn           per level: top k of the logits (ties to the lower index, sorted), decoded against the anchors,
 *                 clipped, with sigmoid scores and the small-box filter; heads [gh*gw,16] raw (0..2 logits,
 *                 3+a*4+k deltas), bias [16]; candidates at offsets[l] of boxes / scores / groups (= level) / valid
 *   nms           batched NMS over n slots (at most m_max valid): per group greedy, IoU > thresh suppresses; keep
 *                 = slot indices by descending score (first max_keep, -1 after), gathered boxes / scores / groups
 *   roi_align     MultiScaleRoIAlign over 4 NHWC levels (scales 1/4..1/32, sampling_ratio, aligned=False) for the
 *                 first *count of r_max boxes -> RoI-major [r_max,out,out,c] (zeros past *count), levels[r] (nullable)
 *   box_candidates softmax + per-class decode (10,10,5,5) + clip + filters of pred [r_max, ld] (nc logits, nc*4
 *                 deltas): slot r*(nc-1)+j-1 for class j
 *   mask_probs    sigmoid of the label's channel of raw [d_max,hw,ld] + bias
 *   paste_masks   resize_boxes by (rh, rw) + paste_masks_in_image (padding 1) of probs [d_max,m,m] -> masks [d_max,h,w]
 *   person_mask   largest-area person (the last detection if none) -> pid, its box, (mask > thresh) dilated by ks */
int lwb_det_transform(const float* img, int h, int w, int ho, int wo, int hp, int wp, float* out, lwb_stream_t stream);
int lwb_det_stem_pool(const float* x, int n, int c, int h, int w, const float* scale, const float* shift,
                      void* y_hi, void* y_lo, lwb_stream_t stream);
int lwb_det_bias_act(const float* raw, int ld_raw, const float* raw2, const float* bias, const float* res, int res_half,
                     int step, int h_in, int w_in, int relu, int n, int h, int w, int c,
                     float* y_f32, void* y_hi, void* y_lo, lwb_stream_t stream);
int lwb_det_d2s_bias_relu(const float* raw, const float* bias, int n, int h, int w, int c,
                          float* y_f32, void* y_hi, void* y_lo, lwb_stream_t stream);
int lwb_det_rpn(int levels, const float* const* heads, const int* gh, const int* gw, const int* stride_h,
                const int* stride_w, const float* cell_anchors, const int* offsets, const float* bias, int k,
                float clip_h, float clip_w, float min_size, float xform_clip, int* top_idx, float* boxes,
                float* scores, int* groups, int* valid, lwb_stream_t stream);
size_t lwb_det_nms_workspace_bytes(int n, int m_max);
int lwb_det_nms(const float* boxes, const float* scores, const int* groups, const int* valid, int n, int m_max, float thresh,
                int max_keep, void* workspace, int* keep, float* out_boxes, float* out_scores, int* out_groups,
                int* out_count, lwb_stream_t stream);
int lwb_det_roi_align(const float* const* feats, const int* fh, const int* fw, int c, const float* boxes, const int* count,
                      int r_max, int out, int sampling, int* levels, float* y_f32, void* y_hi, void* y_lo, lwb_stream_t stream);
int lwb_det_box_candidates(const float* pred, int ld, int nc, const float* proposals, const int* count, int r_max,
                           float clip_h, float clip_w, float score_thresh, float min_size, float xform_clip,
                           float* boxes, float* scores, int* groups, int* valid, lwb_stream_t stream);
int lwb_det_mask_probs(const float* raw, int ld, const float* bias, const int* labels, const int* count, int d_max, int hw,
                       float* logits, float* probs, lwb_stream_t stream);
int lwb_det_paste_masks(const float* probs, int m, const float* boxes, const int* count, int d_max, float rh, float rw,
                        int h, int w, float* masks, float* out_boxes, lwb_stream_t stream);
int lwb_det_person_mask(const float* boxes, const int* labels, const int* count, int person, const float* masks, int h, int w,
                        float thresh, int ks, int* pid, float* box, float* out, lwb_stream_t stream);

/* ---- Paired image-quality metrics (his_evaluators/metrics/metrics.py:450-631) --------------------------------------
 * pred / ref: [n,3,h,w] fp32 NCHW in [-1,1], or in [0,1] with from01 = 1 (mapped by x * 2 - 1 in fp32, as the metrics'
 * preprocess does).
 *   ssim_psnr     per frame: skimage 0.16.2 structural_similarity(pred, ref, multichannel=True) on the HWC image (7x7
 *                 uniform window, sample covariance, K1 0.01, K2 0.03, data_range 2, map cropped by 3, mean per channel
 *                 then over channels) and peak_signal_noise_ratio(image_true=ref, image_test=pred) (data_range 1 when
 *                 min(ref) >= 0, else 2; +inf for identical frames), both fp64 [n].  h, w >= 7; n has no upper
 *                 limit (batches of more than 21845 frames run their tiles in several launches).  workspace:
 *                 lwb_ssim_psnr_workspace_bytes(n, h, w) bytes.  Fixed-order reductions: results repeat bit for bit.
 *   lpips_input   PNetLin's scaling layer (x - shift) / scale of pred and ref stacked as one batch: out [2n,3,h,w]
 *                 (pred first), the input of the AlexNet features (conv1 via lwb_conv2d_direct_relu_nhwc, the pools via
 *                 lwb_maxpool_nhwc, conv2..5 via lwb_conv_plan_* + lwb_det_bias_act).
 *   lpips_layer   one tap: feat NHWC [2n,hw,c] (pred features = image i, ref = image n+i); per frame the spatial mean of
 *                 sum_c lin[c] * (f0/(|f0|+1e-10) - f1/(|f1|+1e-10))^2 -> layers_out[i*num_layers + layer]; score[i] =
 *                 that value for layer 0, score[i] + it after (run the taps in order on one stream). */
size_t lwb_ssim_psnr_workspace_bytes(int n, int h, int w);
int lwb_ssim_psnr(const float* pred, const float* ref, int n, int h, int w, int from01, void* workspace,
                  double* ssim_out, double* psnr_out, lwb_stream_t stream);
int lwb_lpips_input(const float* pred, const float* ref, int n, int h, int w, int from01, float* out, lwb_stream_t stream);
int lwb_lpips_layer(const float* feat, int n, int hw, int c, const float* lin, int layer, int num_layers,
                    float* layers_out, float* score, lwb_stream_t stream);

/* ---- Unpaired image-quality metrics: InceptionV3 features (his_evaluators/metrics/metrics.py:16-158, 634-781) -------
 *   inception_input   x [n,3,h,w] fp32 in [0,1] -> out [n,3,299,299]: x * 2 - 1, then F.interpolate(size=(299, 299),
 *                     mode='bilinear', align_corners=False) in fp32 (the metric classes' preprocess).  The stem is
 *                     lwb_conv2d_direct_relu_nhwc with BN folded into its weights and bias, the other 93 convolutions
 *                     the conv engine (lwb_conv_plan_*).
 *   bn_act_segment    channels [c0, c0+c) of a raw NHWC fp32 conv output [n,h,w,ld_raw] -> v = relu?(r * scale + shift),
 *                     r = the raw value, or with box = 1 its 3x3 zero-padded box sum / 9 (avg_pool2d(3, 1, 1) commutes
 *                     with the bias-free 1x1 conv of an Inception pool branch); scale / shift [c] or both null
 *                     (identity).  Written to channels [off_y, off_y+c_out) of fp32 y_f32 and / or fp16 hi / lo operands
 *                     y_hi, y_lo (nullable) of pitch ld_y, channels c..c_out-1 zero.
 *   maxpool_nhwc_slice  lwb_maxpool_nhwc of channels [0, c) of x (pitch ld_x) into channels [off_y, off_y+c) of outputs
 *                     with pitch ld_y (the Mixed_6a / 7a pool branches into their concat buffer). */
int lwb_inception_input(const float* x, int n, int h, int w, float* out, lwb_stream_t stream);
int lwb_bn_act_segment(const float* raw, int n, int h, int w, int ld_raw, int c0, int c, int c_out, int box,
                       const float* scale, const float* shift, int relu, float* y_f32, void* y_hi, void* y_lo,
                       int ld_y, int off_y, lwb_stream_t stream);
int lwb_maxpool_nhwc_slice(const float* x, int n, int h, int w, int c, int ld_x, int k, int stride, float* y_f32,
                           void* y_hi, void* y_lo, int ld_y, int off_y, lwb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LWB_B200_H_ */
