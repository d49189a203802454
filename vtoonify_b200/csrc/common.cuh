// common.cuh — shared helpers for libvtoonify_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/vtoonify_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libvtoonify_b200 is written for sm_90a (H100) only"
#endif

int vt_set_error(const char* fmt, ...);
void vt_count_launch(int n);

#define VT_CHECK(cond, ...)                          \
  do {                                               \
    if (!(cond)) return vt_set_error(__VA_ARGS__);   \
  } while (0)

#define VT_CUDA(call)                                                                     \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess)                                                               \
      return vt_set_error("%s:%d %s failed: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
  } while (0)

#define VT_LAUNCH_CHECK()                                                                 \
  do {                                                                                    \
    cudaError_t e__ = cudaGetLastError();                                                 \
    if (e__ != cudaSuccess)                                                               \
      return vt_set_error("%s:%d kernel launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
    vt_count_launch(1);                                                                   \
  } while (0)

static inline __host__ __device__ int64_t vt_cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Round fp32 to TF32 (round-to-nearest, ties away) keeping an fp32 container. The tensor core
// reads only the top 19 bits of the container, so pre-rounding in the producer makes the
// truncation unbiased.
__device__ __forceinline__ float vt_round_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

__device__ __forceinline__ float vt_lrelu(float v, float slope) { return v > 0.f ? v : v * slope; }

// ToTensor + Normalize(0.5, 0.5) of one uint8 sample: v / 255, then (v - 0.5) / 0.5 (torchvision's order)
__device__ __forceinline__ float vt_u8_unit(unsigned v) { return (((float)v / 255.f) - 0.5f) / 0.5f; }

// RAFT's input normalisation 2 * (x / 255) - 1 of a sample in 0..255
__device__ __forceinline__ float vt_raft_unit(float v) { return 2.f * (v / 255.f) - 1.f; }

// F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) of one [Hin, Win] plane at output pixel (Y, X); ld(offset) reads
// the plane.  Every kernel that up-samples frames calls this one function, so they agree bit for bit.  The roundings are explicit:
// left to the compiler, the contraction of w0*a + w1*b into an fma depends on the surrounding code (whether a product has other
// uses), and two kernels inlining the same expression computed different bits.  The fmas below are the ones frame_s2d_kernel was
// compiled to before this function existed (the sum h0*(w0*a + w1*b) + h1*(w0*c + w1*d) of ATen's upsample_bilinear2d).
template <class Load>
__device__ __forceinline__ float vt_bilinear_up2(Load ld, int Y, int X, int Hin, int Win) {
  // src = (dst + 0.5) / 2 - 0.5, clamped at 0 (the multiply by 0.5 is exact, so the fma rounds once like the expression)
  float sy = fmaf(__fadd_rn((float)Y, 0.5f), 0.5f, -0.5f), sx = fmaf(__fadd_rn((float)X, 0.5f), 0.5f, -0.5f);
  sy = sy < 0.f ? 0.f : sy; sx = sx < 0.f ? 0.f : sx;
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < Hin - 1 ? 1 : 0), x1 = x0 + (x0 < Win - 1 ? 1 : 0);
  const float ly = __fsub_rn(sy, (float)y0), lx = __fsub_rn(sx, (float)x0);
  const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  const float a = ld((int64_t)y0 * Win + x0), bq = ld((int64_t)y0 * Win + x1);
  const float cq = ld((int64_t)y1 * Win + x0), d = ld((int64_t)y1 * Win + x1);
  const float top = fmaf(lx, bq, __fmul_rn(hx, a));
  const float bot = fmaf(hx, cq, __fmul_rn(lx, d));
  return fmaf(hy, top, __fmul_rn(ly, bot));
}

// Rank-1 test of a (flipped) 4x4 FIR kernel held in shared memory: k = ay (x) bx, with bx normalised by the smallest non-zero entry of
// the pivot row so that integer-ratio filters (outer([1,3,3,1]), every StyleGAN blur) factor exactly.  Returns false for a full-rank
// kernel (the caller then applies the 16 taps directly).
__device__ __forceinline__ bool vt_rank1_4x4(const float* sk, float (&ay)[4], float (&bx)[4]) {
  int piv = 0;
  for (int i = 1; i < 16; ++i) if (fabsf(sk[i]) > fabsf(sk[piv])) piv = i;
  const float pv = fabsf(sk[piv]);
#pragma unroll
  for (int i = 0; i < 4; ++i) { ay[i] = 0.f; bx[i] = 0.f; }
  if (!(pv > 0.f)) return false;
  const int py = piv >> 2;
  int cs = piv & 3;
  for (int i = 0; i < 4; ++i) { const float a = fabsf(sk[py * 4 + i]); if (a > 0.f && a < fabsf(sk[py * 4 + cs])) cs = i; }
  const float den = sk[py * 4 + cs];
  float worst = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) { bx[i] = sk[py * 4 + i] / den; ay[i] = sk[i * 4 + cs]; }
  for (int j = 0; j < 4; ++j)
    for (int i = 0; i < 4; ++i) worst = fmaxf(worst, fabsf(sk[j * 4 + i] - ay[j] * bx[i]));
  return worst <= 2e-7f * pv;
}

int vt_num_sms();
