// tc_common.cuh — sm_90a building blocks: mbarrier, TMA (cp.async.bulk.tensor), wgmma descriptors.
// Inline PTX only; the descriptor bit layout follows the PTX ISA "matrix descriptor" table of the wgmma instructions.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "wgmma_sm90.cuh"

// 4-D tensor map (fp32 or bf16/fp16-sized 2-byte elements), SWIZZLE_128B, zero OOB fill; dims / box innermost first, strides in
// BYTES for dims 1..3 (defined in conv_tc.cu)
int vt_tc_make_map4(CUtensorMap* m, const void* base, const uint64_t dims[4], const uint64_t strides_b[3], const uint32_t box[4],
                    const char* what, bool bf16);

namespace vt_tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- mbarrier -----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}
// Bounded wait: a protocol bug becomes a trap instead of a hung GPU.  No message: a printf call anywhere in a kernel makes ptxas
// serialise every wgmma of that kernel.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (globaltimer_ns() - t0 > 2000000000ull) {
      __trap();
    }
  }
}

// ---- TMA ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---- wgmma shared-memory matrix descriptor (sm_90): K-major operand, SWIZZLE_128B, rows of 128 bytes.
//   [0,14)  start address >> 4        [16,30) leading byte offset >> 4 (unused for swizzled K-major)
//   [32,46) stride byte offset >> 4   [49,52) base offset              [62,64) layout type: 1 = SWIZZLE_128B
// sbo_bytes = distance between consecutive 8-row groups.  The swizzle is a function of the absolute shared-memory address (TMA
// writes with the same function), so a start address advanced by 32 bytes (one K step) or by whole 128-byte rows stays valid.
__host__ __device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | (1ull << 62);
}

// fp32 pair -> packed fp16 hi and fp16 residual lo (x ~= hi + lo to 2^-22); saturating converts: |x| beyond the fp16 range gives
// the largest finite halves instead of infinities (the pair then represents up to 131008)
__device__ __forceinline__ void split_f16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  float h0, h1;
  asm("{\n\t.reg .f16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, h;\n\t}" : "=f"(h0), "=f"(h1) : "r"(hi));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - h1), "f"(x0 - h0));
}

// Fused ToRGB, Upsample(skip) part for one output pixel (py, px) of sample b: upfirdn2d(up=2, pad=(2,1), 4x4 kernel) touches exactly
// 2x2 skip pixels per output pixel (taps with (y-2+ky) even).  Branch-free: clamped addresses + validity masks so the 12 loads
// issue together.  Loading (skip_taps_load) and summing (skip_taps_sum) are separate so that a kernel can issue the loads early.
struct SkipTaps {
  float v[3][4];   // skip values of the 4 taps per colour
  float w[4];      // masked flipped-kernel weights of the 4 taps (ky in {ky0, ky0+2}, kx in {kx0, kx0+2})
};
__device__ __forceinline__ void skip_taps_load(const float* rgb_skip, const float* kk, int b, int py, int px, int Ho, int Wo, SkipTaps& s) {
  const int hs = Ho >> 1, ws = Wo >> 1;
  const int ky0 = (py - 2) & 1, kx0 = (px - 2) & 1;
  const int iy0 = (py - 2 + ky0) >> 1, ix0 = (px - 2 + kx0) >> 1;        // second tap is +1
  const float my0 = iy0 >= 0 ? 1.f : 0.f, my1 = (iy0 + 1) < hs ? 1.f : 0.f;
  const float mx0 = ix0 >= 0 ? 1.f : 0.f, mx1 = (ix0 + 1) < ws ? 1.f : 0.f;
  const int cy0 = iy0 < 0 ? 0 : iy0, cy1 = (iy0 + 1) < hs ? iy0 + 1 : hs - 1;
  const int cx0 = ix0 < 0 ? 0 : ix0, cx1 = (ix0 + 1) < ws ? ix0 + 1 : ws - 1;
  s.w[0] = __ldg(kk + (3 - ky0) * 4 + (3 - kx0)) * my0 * mx0;
  s.w[1] = __ldg(kk + (3 - ky0) * 4 + (1 - kx0)) * my0 * mx1;
  s.w[2] = __ldg(kk + (1 - ky0) * 4 + (3 - kx0)) * my1 * mx0;
  s.w[3] = __ldg(kk + (1 - ky0) * 4 + (1 - kx0)) * my1 * mx1;
#pragma unroll
  for (int cc = 0; cc < 3; ++cc) {
    const float* sp = rgb_skip + ((int64_t)b * 3 + cc) * (int64_t)hs * ws;
    s.v[cc][0] = __ldg(sp + (int64_t)cy0 * ws + cx0);
    s.v[cc][1] = __ldg(sp + (int64_t)cy0 * ws + cx1);
    s.v[cc][2] = __ldg(sp + (int64_t)cy1 * ws + cx0);
    s.v[cc][3] = __ldg(sp + (int64_t)cy1 * ws + cx1);
  }
}
// same accumulation order as the reference loop (ky outer, kx inner)
__device__ __forceinline__ float skip_taps_sum(const SkipTaps& s, int cc) {
  float u = s.v[cc][0] * s.w[0];
  u = fmaf(s.v[cc][1], s.w[1], u);
  u = fmaf(s.v[cc][2], s.w[2], u);
  u = fmaf(s.v[cc][3], s.w[3], u);
  return u;
}

// Fused ToRGB, last step for one output pixel: rgb (the 1x1 modulated conv over the pixel's channels) + bias + Upsample(skip)
// (the taps in `st`, loaded by skip_taps_load when rgb_skip is set), written to the planar [B][3][Ho][Wo] image
__device__ __forceinline__ void torgb_store_taps(const float* rgb_bias, bool skip, const SkipTaps& st, float* rgb_out, const float rgb[3],
                                                 int b, int py, int px, int Ho, int Wo) {
  float o[3] = {rgb[0] + __ldg(rgb_bias), rgb[1] + __ldg(rgb_bias + 1), rgb[2] + __ldg(rgb_bias + 2)};
  if (skip) {
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) o[cc] += skip_taps_sum(st, cc);
  }
  const int64_t HW = (int64_t)Ho * Wo;
#pragma unroll
  for (int cc = 0; cc < 3; ++cc) rgb_out[((int64_t)b * 3 + cc) * HW + (int64_t)py * Wo + px] = o[cc];
}
__device__ __forceinline__ void torgb_store(const float* rgb_bias, const float* rgb_skip, const float* kk, float* rgb_out, const float rgb[3],
                                            int b, int py, int px, int Ho, int Wo) {
  SkipTaps st;
  if (rgb_skip) skip_taps_load(rgb_skip, kk, b, py, px, Ho, Wo, st);
  torgb_store_taps(rgb_bias, rgb_skip != nullptr, st, rgb_out, rgb, b, py, px, Ho, Wo);
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

}  // namespace vt_tc
