/*
 * vtoonify_b200.h — C-ABI of libvtoonify_b200.so (hand-written sm_90a CUDA kernels).
 *
 * This is the drop-in boundary for the VToonify per-frame StyleGAN2 synthesis hot path.
 * Every entry point is `extern "C"`, takes plain device pointers + sizes + a CUDA stream
 * handle (`void*` == cudaStream_t) and returns 0 on success / non-zero on error (message via
 * vt_last_error()).  The library never allocates or frees user-visible memory: outputs and
 * workspaces are caller-allocated.  All pointers are DEVICE pointers unless noted.  There is no
 * CPU fallback anywhere in this library.
 *
 * Reference interfaces replaced (paths relative to the reference repo williamyang1991/VToonify):
 *   vt_upfirdn2d_f32        <- pybind `upfirdn2d(input,kernel,up_x,up_y,down_x,down_y,pad_x0,pad_x1,pad_y0,pad_y1)`
 *                              model/stylegan/op/upfirdn2d.cpp:17-31, upfirdn2d_kernel.cu:209-369
 *   vt_fused_bias_act_f32   <- pybind `fused_bias_act(input,bias,refer,act,grad,alpha,scale)` (act=3, grad=0)
 *                              model/stylegan/op/fused_bias_act.cpp:18-32, fused_bias_act_kernel.cu:18-105
 *   vt_conv2d_*             <- conv2d_gradfix.conv2d / conv_transpose2d (cuDNN via F.conv2d)
 *                              model/stylegan/op/conv2d_gradfix.py:22-75, and nn.Conv2d at model/vtoonify.py:96-97,111-113,162-182,195-198
 *   vt_conv2d_wgrad         <- the weight gradient of conv2d_gradfix's backward (cudnn_convolution_backward_weight),
 *                              model/stylegan/op/conv2d_gradfix.py:104-227
 *   vt_modulate_weights_f32 <- ModulatedConv2d weight modulation/demodulation, model/stylegan/model.py:259-267
 *   vt_linear_f32           <- EqualLinear.forward (F.linear [+ fused_leaky_relu]), model/stylegan/model.py:153-162
 *   vt_instnorm_stats_nhwc / vt_adain_apply_nhwc <- AdaptiveInstanceNorm.forward, model/dualstylegan.py:16-21
 *   vt_fir_nhwc_f32         <- Blur.forward after the transposed conv + NoiseInjection + FusedLeakyReLU,
 *                              model/stylegan/model.py:74-90, 285, 315-320, 364-370
 *   vt_smalln_conv_f32      <- ToRGB / fusion_skip / Fusion.conv2 / encoder[-1] (Cout<=4 convs) + Upsample(skip) add,
 *                              model/stylegan/model.py:383-392, model/vtoonify.py:113,124-127,182,198
 *   vt_frame_u8_to_f32 / vt_f32_to_frame_u8 <- transforms.ToTensor+Normalize and util.tensor2cv2,
 *                              style_transfer.py:57-60,160, util.py:190-192
 */
#ifndef VTOONIFY_B200_H_
#define VTOONIFY_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VT_ABI_VERSION 7   /* 2: vt_conv_desc gained weight_bf16x3 / bf16x3_nstack / src_scale, vt_smalln_desc src_mask / tsum, vt_split_weights_bf16x3
                            * 3: face-parsing helpers (vt_frame_s2d_f32 .. vt_logits_readout_f32 with out_bstride), backward ops, frame pre-filter
                            * 4: row-strip kernels, vt_conv_desc gained split_fmt / acc_scale
                            * 5: vt_conv_desc gained stats_ws / stats_ws_floats (statistics of the conv output), vt_conv2d_tc_stats_chunks,
                            *    vt_instnorm_finalize_f32
                            * 6: sm_90a: vt_conv2d_rs takes the vt_conv2d_tc_tf32 weight split; the row-strip up-conv, vt_set_debug_buffer and
                            *    vt_selftest_tc_gemm are gone
                            * 7: instance-norm partials are pivoted: (pivot, sum and square sum of x - pivot) plus a per-chunk pixel
                            *    count, sized by vt_instnorm_partials_floats */

/* ---- library info / errors ------------------------------------------------------------- */
int         vt_abi_version(void);
const char* vt_last_error(void);          /* thread-local message of the last failing call   */
const char* vt_build_info(void);          /* "sm_90a ... " build string                        */
/* number of kernel launches issued by this library since process start (all threads)        */
int64_t     vt_launch_count(void);

/* ---- a1: upfirdn2d (planar / NCHW, any up/down/pad/kernel; index-exact) ------------------ */
/* in : [planes, in_h, in_w] fp32, out: [planes, out_h, out_w] fp32 with
 * out_h = (in_h*up_y + pad_y0 + pad_y1 - kh + down_y) / down_y   (same for w).
 * kernel: [kh, kw] fp32 (device). The kernel is flipped (true convolution), negative pads crop. */
int vt_upfirdn2d_out_size(int in_h, int in_w, int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                          int pad_x0, int pad_x1, int pad_y0, int pad_y1, int* out_h, int* out_w);
int vt_upfirdn2d_f32(const float* in, const float* kernel, float* out, int64_t planes, int in_h, int in_w,
                     int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                     int pad_x0, int pad_x1, int pad_y0, int pad_y1, void* stream);

/* ---- a2: fused bias + leaky-relu + gain (any layout; bias broadcast on dim 1) ------------ */
/* out[i] = lrelu(in[i] + bias[(i / step_b) % size_b], negative_slope) * scale; bias may be NULL. */
int vt_fused_bias_act_f32(const float* in, const float* bias, float* out, int64_t n, int64_t step_b,
                          int size_b, float negative_slope, float scale, void* stream);

/* f4 (training-side op surface): backward of the op above, fused_bias_act(grad=1) of fused_bias_act_kernel.cu:31-33 and
 * op/fused_act.py:20-53: out[i] = (ref[i] > 0 ? v : v * negative_slope) * scale with v = in[i] + bias[(i / step_b) % size_b]
 * (`in` = the incoming gradient, `ref` = the forward OUTPUT, bias = NULL in the first backward, gradgrad_bias in the second). */
int vt_fused_bias_act_grad_f32(const float* in, const float* bias, const float* ref, float* out, int64_t n, int64_t step_b,
                               int size_b, float negative_slope, float scale, void* stream);
/* deterministic per-channel sum of a contiguous [outer, C, inner] tensor (grad_bias = grad_input.sum over batch and space,
 * op/fused_act.py:33-41); workspace: vt_channel_sum_ws_floats(C) floats */
int64_t vt_channel_sum_ws_floats(int C);
int vt_channel_sum_f32(const float* in, float* out, float* workspace, int outer, int C, int64_t inner, void* stream);

/* ---- layout transforms (API boundary NCHW <-> internal NHWC) ------------------------------ */
/* out NHWC has `c_pad` >= C channels per pixel, the tail is zero-filled. round_tf32: cvt.rna.   */
int vt_nchw_to_nhwc_f32(const float* in, float* out, int B, int C, int H, int W, int c_pad, int round_tf32, void* stream);
int vt_nhwc_to_nchw_f32(const float* in, float* out, int B, int C, int H, int W, int c_stride, void* stream);

/* ---- a8: EqualLinear ---------------------------------------------------------------------- */
/* out[r, o] = act( sum_i in[r,i] * (W[o,i]*w_scale) + bias[o]*b_scale ), act: 0 none, 1 lrelu(0.2)*sqrt2 (fused_lrelu),
 * 2 lrelu(0.2) (nn.LeakyReLU), 3 relu, 4 sigmoid */
int vt_linear_f32(const float* in, const float* weight, const float* bias, float* out, int rows, int in_dim,
                  int out_dim, float w_scale, float b_scale, int act, void* stream);

/* PixelNorm (model/stylegan/model.py:13-18): out[r,:] = in[r,:] * rsqrt(mean(in[r,:]^2) + 1e-8) */
int vt_pixelnorm_f32(const float* in, float* out, int rows, int dim, void* stream);

/* ---- a3: weight modulation / demodulation and re-layout ---------------------------------- */
/* W: [Cout, Cin, kh, kw] fp32. style: [wB, Cin] (NULL => ones, wB must be 1). out: [wB][kh*kw][Cout][cin_pad]
 * out[b][t][n][c] = (scale*W[n][c][t]) * style[b][c] * demod[b][n], demod = rsqrt(sum_{c,t}(.)^2 + 1e-8) if demodulate.
 * pad channels [Cin, cin_pad) are zero. round_tf32 rounds to TF32 (rna) for the tensor-core path. */
int vt_modulate_weights_f32(const float* W, const float* style, float* out, int wB, int Cout, int Cin, int kh, int kw,
                            int cin_pad, float scale, int demodulate, int round_tf32, void* stream);

/* Fold Blur(4x4, pad (1,1)) o conv_transpose2d(stride 2, 3x3) into 4 phase-specific 3x3 kernels (SURVEY App. C):
 * w: [wB][9][Cout][cpad] (slab ky*3+kx, already modulated/demodulated), blur: [4,4] device,
 * out: [wB][9][4*Cout][cpad], slab = (dy+1)*3 + (dx+1), row = phase*Cout + n, phase = ry*2+rx (the 4 phases are stacked
 * along the GEMM N dimension):  out[2q+ry, 2p+rx] = sum_{dy,dx} x[q+dy, p+dx] * G[dy][dx][phase].
 * model/stylegan/model.py:273-286 (conv_transpose2d then self.blur). */
int vt_fold_upconv_weights_f32(const float* w, const float* blur, float* out, int wB, int Cout, int cpad, int round_tf32,
                               void* stream);

/* Split fp32 weight rows for the bf16x3 tensor-core mode: for every 32-channel chunk (128 bytes) of every row,
 * out = [bf16(w) x 32 | bf16(w - bf16(w)) x 32] (128 bytes). w, out: [rows][C] fp32-sized elements, C % 32 == 0.
 * nstack_rows > 0 (N-stacked form, rows % nstack_rows == 0): out has 2*rows rows; each group of nstack_rows input rows
 * becomes nstack_rows rows [hi|hi] followed by nstack_rows rows [lo|lo]. */
int vt_split_weights_bf16x3(const float* w, void* out, int64_t rows, int C, int nstack_rows, void* stream);
/* The same split with fp16 halves (11 + 11 mantissa bits): out = [half(w*scale) x 32 | half(w*scale - hi) x 32] per 32-channel chunk.
 * `scale` is a power of two that keeps the low halves out of fp16's subnormal range (undone by the consumer: the descriptor's acc_scale);
 * |w * scale| must stay below 65504. */
int vt_split_weights_f16x3(const float* w, void* out, int64_t rows, int C, float scale, void* stream);

/* ---- convolution descriptor (NHWC activations) -------------------------------------------- */
#define VT_MAX_TAPS 36     /* 9 taps x up to 4 output phases (folded up-conv) */
#define VT_ACT_NONE 0
#define VT_ACT_LRELU 1      /* lrelu(slope) * gain                                             */
#define VT_ACT_RELU_TANH 2  /* tanh(relu(v))      (Fusion mask, model/vtoonify.py:126)          */

typedef struct vt_conv_desc {
  int32_t struct_size;          /* sizeof(vt_conv_desc), ABI check                               */
  int32_t n_src;                /* 1 or 2: virtual channel concat of sources                     */
  const float* src[2];          /* NHWC [B, H, W, src_cstride[i]]                                */
  int32_t src_c[2];             /* logical channels taken from each source                      */
  int32_t src_cstride[2];       /* floats per pixel in memory (>= src_c)                         */
  int32_t B, H, W;              /* input batch / spatial                                         */
  int32_t Ho, Wo;               /* output spatial (of this call / phase)                         */
  int32_t stride;               /* in_y = oy*stride + tap_dy[t]                                  */
  int32_t taps;                 /* number of taps used by this call (<= 9)                       */
  int32_t tap_dy[VT_MAX_TAPS];
  int32_t tap_dx[VT_MAX_TAPS];
  int32_t tap_w[VT_MAX_TAPS];   /* index of the weight slab used by tap t                        */
  int32_t tap_phase[VT_MAX_TAPS]; /* reserved (must be 0)                                          */
  int32_t n_phase;              /* 1, or 4: weight rows are phase-major [n_phase*Cout] per tap and phase ph's Cout
                                   outputs go to the strided view at phase_off[ph] (folded stride-2 up-conv)       */
  int32_t out_cpitch;           /* floats per pixel of the dense tensor `out` points into (noise index = offset / out_cpitch) */
  int64_t phase_off[4];         /* element offset of each phase's strided output view             */
  const float* weight;          /* [wB][w_taps][Cout][w_cstride]; channel order = src0 then src1 */
  int32_t wB;                   /* 1 (shared) or B (per-sample, modulated)                       */
  int32_t w_taps;               /* slabs per sample in `weight`                                  */
  int32_t w_cstride;            /* floats per (tap, cout) row (>= src_c[0]+src_c[1])             */
  int32_t Cout;
  float*  out;                  /* strided NHWC view: out[b*out_sb + oy*out_sy + ox*out_sx + n]  */
  int64_t out_sb, out_sy, out_sx;   /* element strides                                           */
  /* epilogue: v = acc + bias[n] + noise_w[0]*noise[pixel]; v = act(v); v = v*alpha + beta*res
   * with pixel = (phase_off[ph] + b*out_sb + oy*out_sy + ox*out_sx) / out_cpitch                    */
  const float* bias;            /* [Cout] or NULL                                                */
  const float* noise;           /* planar [B, H_dense, W_dense] over the dense output tensor, or NULL */
  const float* noise_w;         /* device scalar or NULL                                         */
  int32_t act;                  /* VT_ACT_*                                                      */
  float   slope, gain;          /* lrelu params                                                  */
  const float* res;             /* residual with the same strided view as out, or NULL          */
  float   alpha, beta;
  int32_t round_tf32;           /* round outputs to TF32 (rna) for a tensor-core consumer       */
  int32_t reserved;
  /* optional fused ToRGB tail (tensor-core kernel only, needs Cout <= 256, n_phase == 1, dense output):
   * rgb_out[b,c,oy,ox] = sum_n out[b,oy,ox,n] * rgb_w[b,c,n] + rgb_bias[c] + upfirdn2d(rgb_skip, rgb_skip_kernel, up=2, pad=(2,1))
   * (model/stylegan/model.py:383-392 on the freshly computed activation, which is not re-read from HBM) */
  const float* rgb_w;           /* [wB][3][Cout] modulated 1x1 weights, or NULL                  */
  const float* rgb_bias;        /* [3]                                                           */
  const float* rgb_skip;        /* planar [B,3,Ho/2,Wo/2] or NULL                                */
  const float* rgb_skip_kernel; /* [4,4]                                                         */
  float*       rgb_out;         /* planar [B,3,Ho,Wo]                                            */
  const float* slope_vec;       /* optional [Cout] per-channel negative slopes (PReLU) used by VT_ACT_LRELU instead of `slope` */
  const void*  weight_bf16x3;   /* optional: `weight` split by vt_split_weights_bf16x3 (same shape/strides in bytes). When set, the
                                 * tensor-core kernel computes a*w as a_hi*w_hi + a_lo*w_hi + a_hi*w_lo with bf16 operands
                                 * (fp32-class accuracy, 1.5x the MMA work of TF32); ignored by the direct kernel          */
  int32_t bf16x3_nstack;        /* 1: weight_bf16x3 is the N-stacked form of vt_split_weights_bf16x3 (Cout == 32 only): per tap 32 rows
                                 * [w_hi|w_hi] then 32 rows [w_lo|w_lo]; 4 MMAs per tap instead of 6, all four hi/lo products        */
  int32_t reserved2;
  const float* src_scale[2];    /* optional planar [B,H,W] per-pixel multiplier of source i, applied while the operand is split
                                 * (bf16x3 tensor-core mode, stride 1 only): conv(cat[f_G, f_E * m_E]) without materialising
                                 * f_E * m_E (model/vtoonify.py:127). Rejected by the other kernels.                        */
  const float* src_affine[2];   /* optional [B][src_c[i]][2] = (scale, shift) per (sample, channel): in-image pixels of source i
                                 * become x*scale + shift while the operand is split (bf16x3 tensor-core mode, stride 1 only);
                                 * padding stays 0, exactly as the reference zero-pads the *normalised* tensor. Used to apply
                                 * AdaIN (model/dualstylegan.py:16-21) inside the convolution that consumes it
                                 * (vt_adain_affine_f32 builds the table). Rejected by the other kernels.                  */
  int32_t split_fmt;            /* format of the split operands (`weight_bf16x3` set): 0 = bf16 hi + lo (vt_split_weights_bf16x3),
                                 * 1 = fp16 hi + lo (vt_split_weights_f16x3: 11 + 11 mantissa bits, |activation| < 1.3e5)           */
  float   acc_scale;            /* accumulators are multiplied by this before the epilogue (0 = 1): the inverse of the power-of-two
                                 * `scale` given to vt_split_weights_f16x3                                                           */
  float*  stats_ws;             /* optional (tensor-core kernel, n_phase == 1, no fused ToRGB): instance-norm partials of the tensor
                                 * this launch WRITES, in the layout of vt_instnorm_finalize_f32 with chunks =
                                 * vt_conv2d_tc_stats_chunks(desc) and Cs = Cout; vt_instnorm_finalize_f32 turns them into (mean, rstd).
                                 * Replaces the separate statistics pass of AdaptiveInstanceNorm (model/dualstylegan.py:10-21) over a
                                 * conv output                                                                                        */
  int64_t stats_ws_floats;      /* capacity of stats_ws in floats: >= vt_instnorm_partials_floats(chunks, B, Cout)                   */
} vt_conv_desc;

/* fp32-exact CUDA-core implicit GEMM (FFMA). Any shape. */
int vt_conv2d_direct_f32(const vt_conv_desc* d, void* stream);
/* wgmma (TF32 or split 16-bit operands, fp32 accumulate in registers), TMA-staged tiles. Requires channel strides % 32 == 0,
 * Cout % 32 == 0, 16B-aligned views. */
int vt_conv2d_tc_tf32(const vt_conv_desc* d, void* stream);
int vt_conv2d_tc_supported(const vt_conv_desc* d);   /* 1 if vt_conv2d_tc_tf32 accepts the descriptor */
/* number of partial-sum chunks per (sample, channel) that vt_conv2d_tc_tf32 writes to desc->stats_ws for this descriptor under the current
 * options (-1 + vt_last_error() if the descriptor cannot produce statistics) */
int vt_conv2d_tc_stats_chunks(const vt_conv_desc* d);
/* Row-strip layers: full-resolution 3x3 / stride 1 / padding 1 convolutions with Cin, Cout in {32, 64} (StyledConv conv2 of the last
 * generator levels, model/stylegan/model.py:298-304 + 364-392).  Same descriptor and split weights as vt_conv2d_tc_tf32 (bf16x3 mode);
 * acc_scale > 0 overrides desc->acc_scale.  With the fused ToRGB tail `out` may be NULL: only `rgb_out` is written (the last
 * StyledConv of the synthesis network, whose activation has no reader: model/stylegan/model.py:549-556).  On sm_90a these layers run
 * on the wgmma kernel. */
int vt_conv2d_rs(const vt_conv_desc* d, float acc_scale, void* stream);
int vt_conv2d_rs_supported(const vt_conv_desc* d);
/* tuning knobs for experiments / tests: key in {"tc_mode","tc_mt","tc_tgroup","tc_transpose","smalln_is","fir4","upfirdn_tiled",
 * "tc_s2_halo","tc_stage_policy" (1: big halo boxes keep >= 5 weight stages), "tc_halo_pct" (halo staging threshold, % of the per-tap bytes),
 * "tc_m_major" (work-item order), "instnorm_chunks" (target chunks per sample on large maps, 0: small chunks)}; none of them changes results
 * beyond fp32 rounding of the instance-norm partial sums (tests/test_gpu_conv.py);
 * returns the previous value (-1 for an unknown key) */
int vt_set_option(const char* key, int value);

/* ---- weight gradient of a convolution (conv2d_gradfix backward, model/stylegan/op/conv2d_gradfix.py:104-227) ---------------
 * One reduction over pixels covers both ops:
 *   out[m][n][t] = sum over samples b and pixels p of the A grid of  A[b, p, m] * S[b, stride*p + (tap_dy[t], tap_dx[t]), n]
 * with S = 0 outside its image.
 *   conv2d:           A = grad_output (M = Cout), S = input (N = Cin), tap t = ky*kw+kx at (ky*dil - pad_y, kx*dil - pad_x)
 *   conv_transpose2d: A = input (M = Cin), S = grad_output (N = Cout), same tap offsets
 * so `out` is the PyTorch weight layout [M][N][kh][kw] (per_sample: [B*M][N][kh][kw], the weight gradient of the groups = batch
 * form of ModulatedConv2d, model/stylegan/model.py:273-304).  wgmma with operands split into bf16 hi + lo and three products
 * per algorithmic product (fp32 accumulate): the accuracy class of the forward kernel's bf16x3 mode, whatever the precision
 * setting.  The pixel reduction is split across CTAs only when the output has too few tiles to fill the GPU; the split count
 * depends on the descriptor alone and the partial results are added in index order (no atomics): results are bit-reproducible. */
typedef struct vt_conv_wgrad_desc {
  int32_t struct_size;          /* sizeof(vt_conv_wgrad_desc), ABI check                                              */
  int32_t B;                    /* samples                                                                            */
  int32_t per_sample;           /* 0: sum over samples, out [M][N][taps]; 1: one result per sample, out [B*M][N][taps] */
  int32_t stride;               /* 1 or 2                                                                             */
  const float* a;               /* NHWC [B, a_h, a_w, a_cstride]; channels [M, a_cstride) must be zero (padding)     */
  int32_t a_h, a_w, M, a_cstride;   /* a_cstride % 32 == 0                                                            */
  const float* s;               /* NHWC [B, s_h, s_w, s_cstride]                                                      */
  int32_t s_h, s_w, N, s_cstride;   /* s_cstride % 32 == 0                                                            */
  int32_t taps;                 /* 1 .. VT_MAX_TAPS                                                                   */
  int32_t tap_dy[VT_MAX_TAPS];
  int32_t tap_dx[VT_MAX_TAPS];
  float*  out;
  float*  ws;                   /* workspace of vt_conv2d_wgrad_ws_floats(desc) floats (NULL when that is 0)          */
  int64_t ws_floats;
} vt_conv_wgrad_desc;
/* workspace floats vt_conv2d_wgrad needs for this descriptor (0 when the reduction is not split); host only: plans without
 * touching the GPU.  -1 + vt_last_error() for a descriptor vt_conv2d_wgrad rejects. */
int64_t vt_conv2d_wgrad_ws_floats(const vt_conv_wgrad_desc* d);
int vt_conv2d_wgrad(const vt_conv_wgrad_desc* d, void* stream);

/* ---- small-N conv (Cout <= 4): planar output, optional planar extra source + skip upsample */
typedef struct vt_smalln_desc {
  int32_t struct_size;
  int32_t n_planar;             /* 0 or number of leading planar channels (<=4), e.g. skip (3)   */
  const float* planar;          /* [B, n_planar, H, W] or NULL                                   */
  const float* planar_weight;   /* [w_taps][Cout][n_planar] weights of the planar channels       */
  const float* src;             /* NHWC [B,H,W,src_cstride] (may be NULL if src_c == 0)          */
  int32_t src_c, src_cstride;
  const float* src2;            /* optional second NHWC source (same shape as src)                */
  int32_t src2_mode;            /* 0 none; 1: input = virtual concat [src | abs(src - src2)], weight rows hold 2*src_c */
  int32_t B, H, W;
  int32_t taps;
  int32_t tap_dy[VT_MAX_TAPS], tap_dx[VT_MAX_TAPS], tap_w[VT_MAX_TAPS];
  const float* weight;          /* [wB][w_taps][Cout][w_cstride]: weights of the NHWC source     */
  int32_t wB, w_taps, w_cstride, Cout;
  const float* bias;            /* [Cout] or NULL                                                */
  int32_t act;                  /* VT_ACT_NONE or VT_ACT_RELU_TANH                               */
  const float* skip;            /* optional [B,Cout,H/2,W/2] planar: out += upfirdn2d(skip, up=2, pad=(2,1), skip_kernel) */
  const float* skip_kernel;     /* [4,4] device                                                  */
  float* out;                   /* planar [B, Cout, H, W]                                        */
  float* mul_out;               /* optional NHWC [B,H,W,mul_c]: mul_src * out[:,0] (f_E * m_E)   */
  const float* mul_src;
  int32_t mul_c, round_tf32;
  const float* tap_const;       /* optional [wB][w_taps][Cout]: constant added per in-bounds tap (folded affine) */
  const float* src_mask;        /* optional planar [B,H,W]: the NHWC source is multiplied per pixel by it (f_E * m_E)        */
  const float* tsum;            /* optional NHWC [B,H,W,tsum_c] tensor of per-tap partial products T[.., t*Cout + n] computed by a
                                 * 1x1 tensor-core convolution: out[n] += sum over in-bounds taps t of T[p + shift_t][t*Cout + n]  */
  int32_t tsum_c, reserved;
} vt_smalln_desc;
int vt_smalln_conv_f32(const vt_smalln_desc* d, void* stream);
/* Fold a per-(b,c) affine (AdaIN: gamma*(x-mean)*rstd+beta, model/dualstylegan.py:16-21) into conv weights:
 * w: [taps_n][C2] (rows = tap*N+n), stats: [B][C2][2] (mean, rstd), gamma_beta: [B][2*C2] ->
 * out_w: [B][taps_n][C2] = w*gamma*rstd, out_k: [B][taps_n] = sum_c w*(beta - gamma*mean*rstd). */
int vt_affine_fold_weights_f32(const float* w, const float* stats, const float* gamma_beta, float* out_w, float* out_k,
                               int B, int taps_n, int C2, void* stream);

/* ---- FIR on NHWC (Blur after transposed conv) with fused noise + bias + leaky relu -------- */
/* in : [B, H, W, C] ; kernel [kh,kw] (device, flipped like upfirdn2d); pad (p0,p1) both axes.
 * out: [B, Ho, Wo, C], Ho = H + p0 + p1 - kh + 1. v = fir; v += noise_w*noise; v = lrelu(v+bias)*gain if act. */
int vt_fir_nhwc_f32(const float* in, const float* kernel, float* out, int B, int H, int W, int C, int kh, int kw,
                    int pad0, int pad1, const float* bias, const float* noise, const float* noise_w, int act,
                    float slope, float gain, int round_tf32, void* stream);

/* ---- a7: instance-norm statistics + AdaIN apply (NHWC) ------------------------------------ */
/* mode 0: x = in[b,p,c] (c < C). mode 1: virtual cat(in, |in - in2|) with 2C channels.
 * stats: [B, Cs, 2] = (mean, rstd) with biased variance, eps inside rsqrt.  Deterministic two-stage reduction (no
 * atomics): centred per-chunk partials, then vt_instnorm_finalize_f32; ws: caller-allocated scratch of vt_instnorm_ws_bytes() bytes. */
int64_t vt_instnorm_ws_bytes(int B, int64_t HW, int C, int mode);
int vt_instnorm_stats_nhwc(const float* in, const float* in2, int mode, int B, int64_t HW, int C, int c_stride,
                           float eps, float* stats, void* ws, void* stream);
/* second stage alone.  ws holds three float arrays of E = chunks * B * Cs entries (entry chunk * B * Cs + b * Cs + c): a pivot k
 * near the chunk's values (a value of the chunk, or its rounded mean), the sum of (x - k) and the sum of (x - k)^2; then int32
 * counts[chunks] = pixels of each chunk (the same for every entry; a chunk of 0 pixels has all partials 0), summing to HW.
 * -> stats [B, Cs, 2] = (mean, rstd).  The finalize adds the chunks in a fixed order in double precision: first the plane mean,
 * then each chunk's squared deviations from it.  Pivoted partials keep mean and rstd at fp32 accuracy on planes whose mean is
 * large next to their spread, where (sum, sum of squares) about zero cancels.
 * Used with vt_conv_desc.stats_ws (partials written by the producing conv). */
int vt_instnorm_finalize_f32(const float* ws, float* stats, int B, int Cs, int chunks, int64_t HW, float eps, void* stream);
/* floats of the vt_instnorm_finalize_f32 layout for (chunks, B, Cs): chunks * (B * Cs * 3 + 1); -1 for a non-positive argument */
int64_t vt_instnorm_partials_floats(int64_t chunks, int B, int Cs);
/* AdaIN as a per-(sample, channel) affine: affine[b][c] = (gamma*rstd, beta - gamma*mean*rstd); stats [B][Cs][2], gamma_beta [B][2*Cs] */
int vt_adain_affine_f32(const float* stats, const float* gamma_beta, float* affine, int B, int Cs, void* stream);
/* out[b,p,c] = gamma[b,c] * (x - mean) * rstd + beta[b,c]; gamma_beta: [B, 2*Cs] (gamma then beta) */
int vt_adain_apply_nhwc(const float* in, const float* in2, int mode, int B, int64_t HW, int C, int c_stride,
                        const float* stats, const float* gamma_beta, float* out, int round_tf32, void* stream);

/* ---- backward of the encoder path (NHWC [B, HW, C], C % 4 == 0, C <= 1024, 16-byte aligned tensors) --------------------- */
/* Both entry points follow the chunk plan of vt_instnorm_stats_nhwc (it depends on (HW, C) only) and reduce without atomics in
 * a fixed order, in double precision: the same inputs give bit-identical results.  ws: vt_act_grad_ws_bytes(B, HW, C) bytes. */
int64_t vt_act_grad_ws_bytes(int B, int64_t HW, int C);
/* Reduction half of the instance-norm backward: sums[b][c] = (sum_p g, sum_p g * xhat), xhat = (x - mean) * rstd with the
 * statistics the forward applied (stats [B][C][2] = (mean, rstd)).  The two sums are also dbeta and dgamma of the affine. */
int vt_adain_grad_stats_nhwc(const float* g, const float* x, const float* stats, int B, int64_t HW, int C, float* sums,
                             void* ws, void* stream);
/* Elementwise half: out = beta * res + gate(ref) * gain * T(g), gate(ref) = ref > 0 ? 1 : slope (ref NULL: 1), res may be NULL.
 * T(g) = g when x is NULL; otherwise the AdaIN backward gamma * rstd * ((g - m_g) - (x - mean) * rstd * m_gx) with
 * m_g, m_gx = sums / HW from vt_adain_grad_stats_nhwc and gamma from gamma_beta [B][2C] (gamma then beta).
 * bias_grad (may be NULL): [C] = sum over b and p of out, from per-chunk partials of the same pass.  With bias_grad, out may be
 * NULL: only the sums are produced (ops.channel_sum_nhwc). */
int vt_act_grad_nhwc(const float* g, const float* ref, float slope, float gain, const float* res, float beta, const float* x,
                     const float* stats, const float* gamma_beta, const float* sums, int B, int64_t HW, int C, float* out,
                     float* bias_grad, void* ws, void* stream);

/* ---- backward of the generator tail of VToonify.forward (G step), NHWC [B, HW, C], 16-byte aligned tensors ----------------- */
/* StyledConv gate with the ToRGB adjoint: out = gate(ref) * gain * (g + sum_k w_rgb[b][k][c] * g_rgb[b][k][p]); g may be NULL (0),
 * g_rgb planar [B][3][HW] (the image gradient, read directly), w_rgb [wB][3][w_cstride] (wB 1 or B), gate(ref) = ref > 0 ? 1 : slope. */
int vt_torgb_gate_grad_nhwc(const float* g, const float* g_rgb, const float* w_rgb, int wB, int w_cstride, const float* ref,
                            float slope, float gain, int B, int64_t HW, int C, float* out, void* stream);
/* bytes of the ws of vt_fusion_mask_grad_nhwc */
int64_t vt_fusion_mask_grad_ws_bytes(int B, int64_t HW);
/* Fusion mask head m = tanh(relu z): g_z[b][p] = (sum_c g_p * f_e + g_m[b][p]) * (1 - m^2) * [m > 0] (g_m planar, may be NULL), and
 * bias_grad[0] = sum of g_z.  g_p: gradient of f_E * m.  Fixed-order double reductions. */
int vt_fusion_mask_grad_nhwc(const float* g_p, const float* f_e, const float* m, const float* g_m, int B, int64_t HW, int C,
                             float* g_z, float* bias_grad, void* ws, void* stream);
/* AdaIN-backward sums of the mask head over the virtual concat A = cat(f_G, |f_G - f_E|) (2C channels, C <= 512): with
 * u = conv2's input gradient, u[p][c'] = sum_t w2[t][c'] * g_z[p - (t / 3 - 1, t % 3 - 1)], sums[b][c'] = (sum_p u, sum_p u * ahat),
 * ahat = (A - mean) * rstd, stats [B][2C][2].  w2 [9][2C] is conv2's weight tap-major.  u is never written.
 * ws: vt_act_grad_ws_bytes(B, H * W, 2C) bytes. */
int vt_fusion_adain_grad_stats_nhwc(const float* g_z, const float* w2, const float* f_g, const float* f_e, const float* stats,
                                    int B, int H, int W, int C, float* sums, void* ws, void* stream);
/* Elementwise pass of the mask head: T = the AdaIN backward of u (as vt_act_grad_nhwc with gamma_beta [B][4C]), s = sign(f_G - f_E)
 * (sign(0) = 0): g_fg = g_dir + T[c] + s * T[C + c], g_fe = g_p * m - s * T[C + c] (g_dir may be NULL). */
int vt_fusion_input_grad_nhwc(const float* g_z, const float* w2, const float* f_g, const float* f_e, const float* stats,
                              const float* gamma_beta, const float* sums, const float* g_dir, const float* g_p, const float* m,
                              int B, int H, int W, int C, float* g_fg, float* g_fe, void* stream);

/* ---- minibatch standard deviation of the StyleGAN discriminator (model/vtoonify.py:67-75), NHWC [B, HW, C] ------------------ */
/* group = min(B, 4) in the reference; B % group != 0 is an error.  Sample b is in column b % (B / group); per column the statistic
 * is the mean over (p, c) of sqrt(biased variance over the group + 1e-8).  Fixed-order double reductions, no atomics.
 * Forward: out [B, HW, c_out] = x in channels [0, C), the column's statistic in channel C, zeros in (C, c_out); c_out > C. */
int vt_mbstd_nhwc_f32(const float* x, float* out, int B, int group, int64_t HW, int C, int c_out, void* stream);
/* Backward: gin [B, HW, c_in] is the gradient of the forward's out (the forward's x is re-read) -> gx [B, HW, C] = gin's first C
 * channels plus the statistic's path, the column's sum of gin[..., C] times d(statistic)/dx. */
int vt_mbstd_grad_nhwc_f32(const float* gin, const float* x, float* gx, int B, int group, int64_t HW, int C, int c_in, void* stream);

/* ---- pSp encoder helpers (model/encoder/encoders/helpers.py:56-119, psp_encoders.py:72-88) ---------------- */
/* out[b,y,x,c] = x[b,y,x,c] * gate[b,c] + sc[b, y*sc_stride, x*sc_stride, c]   (SE gate + shortcut add; gate may be NULL = 1,
 * sc: NHWC [B, Hs, Ws, C] with Hs >= (H-1)*sc_stride+1; MaxPool2d(1, stride) shortcut == strided sampling) */
int vt_gate_shortcut_add_nhwc(const float* x, const float* gate, const float* sc, float* out, int B, int H, int W, int C,
                              int Hs, int Ws, int sc_stride, int round_tf32, void* stream);
/* out = bilinear_resize(x [B,h,w,C] -> [H,W], align_corners=True) + y [B,H,W,C]   (FPN _upsample_add) */
int vt_bilinear_add_nhwc(const float* x, const float* y, float* out, int B, int h, int w, int H, int W, int C,
                         int round_tf32, void* stream);

/* ---- face-parsing pre-network helpers (model/bisenet/model.py, style_transfer.py:171-174; next row of SURVEY 8f) ---- */
/* Space-to-depth input of the stride-2 7x7 stem: out[b,y,x,(py*2+px)*3+c] = X[b,c,2y+py,2x+px] (zero beyond X and in the pad
 * channels), X = in (upsample2 = 0) or 2 * F.interpolate(in, scale_factor=2, 'bilinear', align_corners=False) (upsample2 = 1).
 * in: planar [B,3,Hin,Win]; out: NHWC [B,Ho,Wo,cpad], Ho = ceil(XH/2). A 7x7/2 conv on X is a 4x4/1 conv on this tensor. */
int vt_frame_s2d_f32(const float* in, float* out, int B, int Hin, int Win, int Ho, int Wo, int cpad, int upsample2, void* stream);
/* nn.MaxPool2d(3, 2, 1) on NHWC: out [B, (H-1)/2+1, (W-1)/2+1, C] */
int vt_maxpool3x3s2_nhwc_f32(const float* in, float* out, int B, int H, int W, int C, void* stream);
/* ---- LPIPS perceptual loss (model/stylegan/lpips, VGG16 net-lin) ---- */
/* nn.MaxPool2d(2, 2) on NHWC: out [B, H/2, W/2, C] (floor; bit-identical to torch) */
int vt_maxpool2x2_nhwc_f32(const float* in, float* out, int B, int H, int W, int C, void* stream);
/* its adjoint: gx [B, H, W, C] = add + the gradient g [B, H/2, W/2, C] routed to the first maximal element of each window of the pool
 * input x in row-major order (torch's tie rule, recomputed from x); rows / columns dropped by the floor get add alone (add may be
 * NULL: 0) */
int vt_maxpool2x2_grad_nhwc_f32(const float* g, const float* x, const float* add, float* gx, int B, int H, int W, int C, void* stream);
/* bytes of the ws of vt_lpips_head_nhwc for taps of HW[k] pixels */
int64_t vt_lpips_head_ws_bytes(int B, int n_taps, const int64_t* HW);
/* out[b] = sum over the taps k of mean over the HW[k] pixels of sum_c w[k][c] (u0_c - u1_c)^2, u = f / (||f||_2 + 1e-10) with f0 the
 * row of sample b and f1 that of sample B + b in f[k] (NHWC [2B, HW[k], C[k]]); 1 to 8 taps, deterministic (double partials) */
int vt_lpips_head_nhwc(int n_taps, const float* const* f, const float* const* w, const int64_t* HW, const int* C, int B, float* out,
                       void* ws, void* stream);
/* the head's gradient for one tap, scaled by g_b[b] / HW: into the f0 rows (g_target, [B, HW, C]) and/or the f1 rows (g_pred); either may
 * be NULL; 0 at a pixel whose row is all zero */
int vt_lpips_head_grad_nhwc(const float* f, const float* w, const float* g_b, int B, int64_t HW, int C, float* g_target, float* g_pred,
                            void* stream);
/* F.interpolate(in, (H, W), mode='nearest') on NHWC */
int vt_resize_nearest_nhwc_f32(const float* in, float* out, int B, int h, int w, int H, int W, int C, void* stream);
/* out[b,c,y,x] = scale * F.interpolate(logits, (Hf, Wf), 'bilinear', align_corners=True)[b, c, step*y, step*x];
 * logits: NHWC [B,h,w,c_stride] (first n_classes channels used); out: planar [B,n_classes,Ho,Wo] with `out_bstride`
 * elements between samples (0 = dense), so the frame loop can write channels 3..21 of its [B,22,H,W] network input in place */
int vt_logits_readout_f32(const float* in, float* out, int B, int h, int w, int c_stride, int n_classes, int Hf, int Wf,
                          int Ho, int Wo, int step, float scale, int64_t out_bstride, void* stream);

/* ---- training-data augmentation (model/simple_augment.py random_apply_affine) ---- */
/* host only: the tile side (16 or 8) of vt_augment_affine_f32 for the per-sample warp coefficients coef (host, [B][6] double: x2-image
 * x = c0 + c1 j + c2 i, y = c3 + c4 j + c5 i at warp-grid column j, row i), chosen so the worst sample's footprint fits shared memory,
 * or 0 when none fits or a coordinate leaves +-2^22 (the caller then runs the unfused statements); win (may be NULL) receives the
 * x2-image window (width, height) to pass to the launch; -1 on bad arguments */
int vt_augment_affine_plan(const double* coef, int B, int H, int W, int* win);
/* out [B,C,H,W] = the 12-tap x2 down (flipped kernel, crop 1) of the bilinear warp (zeros outside) over the 2(H+6) x 2(W+6) warp grid
 * of the 12-tap x2 up (zeros beyond the padded extent) of in [B,C,H,W] reflect-padded to [Hp, Wp] with pads (pad_y, pad_x) at the
 * top-left; planar fp32, kernel: 12 device floats, coef: device [B][6] double; tile / win from vt_augment_affine_plan; one launch */
int vt_augment_affine_f32(const float* in, float* out, const float* kernel, const double* coef, int B, int C, int H, int W, int pad_x,
                          int pad_y, int Hp, int Wp, int tile, int win_w, int win_h, void* stream);

/* ---- RAFT optical flow (model/raft/core, full model, eval; vtoonify_b200.raft) ---- */
/* out [nB, H/2, W/2, cpad] (nB = B, or 2B when img2 is non-NULL: image2's rows follow image1's) = the space-to-depth tensor
 * Z[y, x, (py*2+px)*3 + c] of X = 2 * (img / 255) - 1 (planar [B, 3, H, W] in 0..255), zero pad channels; H, W even */
int vt_raft_input_s2d_f32(const float* img1, const float* img2, float* out, int B, int H, int W, int cpad, void* stream);
/* NHWC [B, HW, C]: out = relu((x - mean) * rstd), and with res: relu(that + s), s = res, or (res - mean') * rstd' when stats_res is
 * non-NULL; stats / stats_res: [B, C, 2] (mean, rstd) */
int vt_raft_norm_relu_nhwc(const float* x, const float* stats, const float* res, const float* stats_res, float* out, int B, int64_t HW,
                           int C, void* stream);
/* cnet [npix, 2C] -> net [npix, C] = tanh(cnet[:, :C]) and inp[p * inp_cpitch + c] = relu(cnet[p, C + c]) */
int vt_raft_context_f32(const float* cnet, float* net, float* inp, int64_t npix, int C, int inp_cpitch, void* stream);
/* F.avg_pool2d(2, 2) of N rows [h, w] (row stride in_stride floats) -> dense [N, h/2, w/2] (floor), torch's summation order */
int vt_raft_corr_pool_f32(const float* in, float* out, int64_t N, int h, int w, int64_t in_stride, void* stream);
/* CorrBlock lookup, radius 4, 4 levels: level l has size (h2 >> l, w2 >> l) per row (levels[l], row stride strides[l]; row p belongs to
 * the coords [npix, 2] (x, y) entry p); out[p * out_cpitch + l*81 + 9i + j] = bilinear sample at coords[p] / 2^l + (i - 4, j - 4),
 * zeros outside (grid_sample, align_corners=True) */
int vt_raft_corr_lookup_f32(const float* const* levels, const int64_t* strides, int h2, int w2, const float* coords, float* out,
                            int out_cpitch, int64_t npix, void* stream);
/* F.avg_pool2d(2, 2) of an NHWC feature map in [B, h, w, C] -> dense out [B, h/2, w/2, C] (floor), torch's summation order;
 * C % 4 == 0, both 16-byte aligned */
int vt_raft_fmap_pool_f32(const float* in, float* out, int B, int h, int w, int C, void* stream);
/* the lookup of vt_raft_corr_lookup_f32 without the correlation volume (AlternateCorrBlock): fmap1 [B, h, w, 256] (batch stride
 * fmap1_bstride floats, 0 allowed; rows dense), fmap2_levels[l] dense [B, h >> l, w >> l, 256] (fmap2 and its 2x2 mean pools),
 * coords [B, h, w, 2] (x, y) -> out[p * out_cpitch + l*81 + 9i + j] = the bilinear tap at coords[p] / 2^l + (i - 4, j - 4) of
 * fmap1[p] . fmap2_l / 16 (zeros outside), channels 324..out_cpitch-1 = 0; fp32 FMA in every precision mode; h, w >= 8 */
int vt_raft_corr_ondemand_f32(const float* fmap1, int64_t fmap1_bstride, const float* const* fmap2_levels, int B, int h, int w,
                              const float* coords, float* out, int out_cpitch, void* stream);
/* out [B, h, w, Cout] = relu(bias + 7x7 convolution (zero padding 3) of the flow coords - grid); w: [7*7][2][Cout] */
int vt_raft_convf1_f32(const float* coords, const float* w, const float* bias, float* out, int B, int h, int wd, int Cout, void* stream);
/* coords [B, h, w, 2] (x, y) = (init ? pixel grid : coords) + delta (planar [B, 2, h, w], may be NULL); flow_out (may be NULL) gets
 * coords - grid at channel pitch flow_cpitch */
int vt_raft_flow_f32(float* coords, const float* delta, int init, float* flow_out, int flow_cpitch, int B, int h, int w, void* stream);
/* rh [npix, C] = sigmoid(zr[:, C:2C]) * h, zr [npix, 2C] = (z | r) logits */
int vt_raft_gru_reset_f32(const float* zr, const float* h, float* rh, int64_t npix, int C, void* stream);
/* h = (1 - z) * h + z * tanh(q), z = sigmoid(zr[:, :C]), in place */
int vt_raft_gru_update_f32(const float* zr, const float* q, float* h, int64_t npix, int C, void* stream);
/* RAFT.upsample_flow: mask NHWC [B, h, w, mask_cpitch] (576 logits, already scaled), flow = coords - grid -> up planar [B, 2, 8h, 8w];
 * flow_low (may be NULL) planar [B, 2, h, w] = the flow */
int vt_raft_upsample_f32(const float* mask, int mask_cpitch, const float* coords, float* up, float* flow_low, int B, int h, int w,
                         void* stream);

/* ---- parsing-map smoothing (smooth_parsing_map.py warp and window fusion; vtoonify_b200.smooth_parsing) ---- */
/* the script's warp(x, flo): out [B, C, H, W] = grid_sample(x, grid + flow, align_corners=True, zeros) * mask and mask (may be NULL)
 * [B, C, H, W] = the sampled ones thresholded (< 0.9999 -> 0, then > 0 -> 1); flow planar [B, 2, H, W] in pixels (x, y) */
int vt_flow_warp_f32(const float* x, const float* flow, float* out, float* mask, int B, int C, int H, int W, void* stream);
/* one centre frame of the window fusion: nslot = 2 * window + 1 (at most 63) slots, host arrays of device pointers img[k] [3, H, W],
 * par[k] [C, H, W], flow[k] [2, H, W] (flow[window] is not read) and host temporal weights wt[k]; out [C, H, W] = sum_k par'_k * w_k /
 * sum_k w_k, with w_k = wt[k] * exp(-mean_c((I'_k - I_window)^2) / 0.08) * mask_k for the warped (') neighbours and w = wt[window] with
 * the unwarped par[window] at the centre */
int vt_parsing_fuse_f32(const float* const* img, const float* const* par, const float* const* flow, const float* wt, int nslot,
                        float* out, int C, int H, int W, void* stream);
/* B centres of the window fusion, each followed by Downsample([1, 3, 3, 1], 2) and a scale: img / par / flow are host arrays of
 * B * nslot device pointers (centre b's slot k at b * nslot + k, as for vt_parsing_fuse_f32); out + b * out_bstride [C, H / 2, W / 2]
 * (contiguous per sample) = scale * down(fuse_b), TF32-rounded when round_tf32.  Bit-identical to vt_parsing_fuse_f32, then
 * vt_upfirdn2d_f32 (kernel outer([1,3,3,1]) / 64, down 2, pad 1), then vt_axpby_f32 with the same scale and rounding; the fused map is
 * never written to memory */
int vt_parsing_fuse_down_f32(const float* const* img, const float* const* par, const float* const* flow, const float* wt, int nslot,
                             int B, float* out, int64_t out_bstride, int C, int H, int W, float scale, int round_tf32, void* stream);
/* the frame prep of smoothing from uint8 RGB frames [B, H, W, 3]: img planar [B, 3, 2H, 2W] = F.interpolate(Normalize(ToTensor(frame)),
 * scale_factor=2, mode='bilinear') (the up-sampling of vt_frame_s2d_f32, without its factor 2) and stem NHWC [B, H, W, cpad] = RAFT's
 * space-to-depth stem input (vt_raft_input_s2d_f32) of (img + 1) * 255 / 2, rounded after the add, the multiply and the divide */
int vt_smooth_frame_prep_u8(const uint8_t* frames, float* img, float* stem, int B, int H, int W, int cpad, void* stream);

/* ---- elementwise helpers ------------------------------------------------------------------ */
/* out = a * scale_a + b * scale_b (b may be NULL) */
int vt_axpby_f32(const float* a, const float* b, float* out, int64_t n, float scale_a, float scale_b, int round_tf32, void* stream);

/* ---- f3: pre-filter + resize of high-resolution frames (style_transfer.py:124-130, 151-156), bit-exact with OpenCV ------ */
/* out = cv2.sepFilter2D(in, -1, k, k), k = [1,3,3,1]/8: uint8 HWC [B,H,W,3] -> same shape (not in place) */
int vt_frame_blur4_u8(const uint8_t* in, uint8_t* out, int B, int H, int W, void* stream);
/* out = cv2.resize(in, (dw, dh))[top : top+Ho, left : left+Wo] (INTER_LINEAR on uint8): in [B,Hs,Ws,3] -> out [B,Ho,Wo,3].
 * xtab: device int32 [3][dw] = (source column, 2048-scaled weight of it, weight of the next column); ytab: [3][dh] likewise for
 * rows — built on the host exactly as cv::resize builds them (vtoonify_b200.ops.resize_tables) */
int vt_frame_resize_crop_u8(const uint8_t* in, uint8_t* out, int B, int Hs, int Ws, int dh, int dw, int top, int left,
                            int Ho, int Wo, const int* xtab, const int* ytab, void* stream);

/* ---- f2: FFHQ face alignment (align_all_parallel.py:108-147; vtoonify_b200.align), byte for byte with Pillow / NumPy / SciPy --- */
/* Images are uint8 RGB [H, W, 3] with a row pitch in bytes (a crop is a pointer offset); pad = host int[4] (left, top, right, bottom),
 * each >= 1; the padded image is [H + top + bottom, W + left + right, 3]. */
#define VT_ALIGN_MAX_RADIUS 127
/* one axis of Pillow resize(LANCZOS): horizontal -> out [H, out_size, 3], else out [out_size, W, 3] (contiguous).  tab: device int32
 * [out_size] first tap, [out_size] tap count, [out_size * ksize] 22-bit fixed-point taps (vtoonify_b200.align.lanczos_table) */
int vt_align_lanczos_u8(const uint8_t* in, int64_t in_pitch, int H, int W, uint8_t* out, int out_size, int horizontal, const int* tab,
                        int ksize, void* stream);
/* axis 0 of scipy.ndimage.gaussian_filter ('reflect') over np.pad(float32(in), pad, 'reflect'): out float32 [Hp, Wp, 3];
 * w: host double [r + 1], the centre tap first */
int vt_align_blur_rows_f32(const uint8_t* in, int64_t in_pitch, int H, int W, const int* pad, float* out, const double* w, int r,
                           void* stream);
/* axis 1 of the same Gaussian: in, out float32 [Hp, Wp, 3]; with img (the image under the pad; else NULL, and H, W, pad unread) out is
 * the first blend padded + (g - padded) * clip(3 mask + 1, 0, 1) instead of g */
int vt_align_blur_cols_f32(const float* in, float* out, int Hp, int Wp, const double* w, int r, const uint8_t* img, int64_t img_pitch,
                           int H, int W, const int* pad, void* stream);
/* device workspace of vt_align_median_f32 */
int64_t vt_align_median_ws_bytes(void);
/* med (device float32 [3]) = np.median(x, axis=0) of x [n, 3] float32 */
int vt_align_median_f32(const float* x, int64_t n, float* med, void* ws, void* stream);
/* out uint8 [Hp, Wp, 3] = clip(rint(x + (med - x) * clip(mask, 0, 1)), 0, 255); x float32 [Hp, Wp, 3], med device float32 [3] */
int vt_align_finish_u8(const float* x, const float* med, uint8_t* out, int Hp, int Wp, const int* pad, void* stream);
/* Pillow transform((size, size), QUAD, corners, BILINEAR): out [size, size, 3]; coef: host double[8], the QUAD coefficients */
int vt_align_warp_u8(const uint8_t* in, int64_t in_pitch, int H, int W, const double* coef, uint8_t* out, int size, void* stream);

/* ---- a11: frame loop transforms ----------------------------------------------------------- */
/* u8 HWC (RGB or BGR) -> fp32 NCHW in [-1,1]: (v/255 - 0.5)/0.5 ; style_transfer.py:57-60,110,160 */
int vt_frame_u8_to_f32(const uint8_t* in, float* out, int B, int H, int W, int swap_rb, int64_t out_batch_stride, void* stream);
/* fp32 NCHW (3ch) -> clamp(-1,1) -> ((v+1)*127.5) truncated to u8, HWC, optional RGB->BGR ; util.py:190-192 */
int vt_f32_to_frame_u8(const float* in, uint8_t* out, int B, int H, int W, int swap_rb, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VTOONIFY_B200_H_ */
