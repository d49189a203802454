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
