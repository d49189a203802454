// Parsing-map smoothing (smooth_parsing_map.py:38-74, 155-165): the flow warp and the temporal window fusion.
//   flow_warp     the script's warp(x, flo): grid_sample(x, grid + flo, align_corners=True, zeros) * mask and the thresholded mask
//   parsing_fuse  one centre frame: per pixel, the 2 * window + 1 slots' spatial weights exp(-mean((warp(I_s) - I_c)^2) / 0.08) * mask,
//                 times the temporal weights, normalised, and the weighted sum of the warped parsing maps (the centre slot unwarped
//                 with weight wt[window])
// Both sample through warp_taps, which restates the reference's fp32 coordinate arithmetic operation by operation (grid + flo, then
// 2 v / max(W - 1, 1) - 1, then grid_sample's ((g + 1) / 2) (W - 1)) with explicit round-to-nearest intrinsics, so nothing is
// contracted, and accumulates the mask over the in-bounds corners in ATen's order (nw, ne, sw, se): the mask is bit-identical to
// torch's grid_sample of a tensor of ones, which matters because the 0.9999 threshold is a discontinuity.
// One thread per output pixel, all channels; fixed summation order, no atomics, 64-bit offsets.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int MAX_SLOTS = 63;      // window <= 31

unsigned grid1(int64_t n, int threads) {
  int64_t blocks = vt_cdiv(n, threads);
  const int64_t cap = (int64_t)vt_num_sms() * 32;
  return (unsigned)(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}

struct Taps {
  int64_t off;         // offset of the nw corner in a plane (valid when any corner is in bounds)
  float w[4];          // nw, ne, sw, se bilinear weights
  unsigned in;         // bit k: corner k in bounds
  float mask;          // the thresholded mask: 0 or 1
};

// the sampling position of pixel (x, y) displaced by (fx, fy), as the script's warp and grid_sample (align_corners=True) compute it
__device__ __forceinline__ Taps warp_taps(int x, int y, float fx, float fy, int H, int W) {
  const float vx = __fadd_rn((float)x, fx), vy = __fadd_rn((float)y, fy);
  const float gx = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, vx), (float)max(W - 1, 1)), 1.0f);
  const float gy = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, vy), (float)max(H - 1, 1)), 1.0f);
  const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.f), 2.f), (float)(W - 1));
  const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.f), 2.f), (float)(H - 1));
  Taps t;
  t.in = 0;
  t.off = 0;
  t.mask = 0.f;
  t.w[0] = t.w[1] = t.w[2] = t.w[3] = 0.f;
  const float fxn = floorf(ix), fyn = floorf(iy);
  // a corner can be in bounds only when -1 <= floor < size; outside that (far samples, NaN) every corner is out and the weights are
  // never used, so the integer conversion below only ever sees small values
  if (!(fxn >= -1.f && fxn < (float)W && fyn >= -1.f && fyn < (float)H)) return t;
  const int x0 = (int)fxn, y0 = (int)fyn;
  const float x1f = (float)(x0 + 1), y1f = (float)(y0 + 1), x0f = (float)x0, y0f = (float)y0;
  t.w[0] = __fmul_rn(__fsub_rn(x1f, ix), __fsub_rn(y1f, iy));     // nw = (ix_se - ix) * (iy_se - iy)
  t.w[1] = __fmul_rn(__fsub_rn(ix, x0f), __fsub_rn(y1f, iy));     // ne = (ix - ix_sw) * (iy_sw - iy)
  t.w[2] = __fmul_rn(__fsub_rn(x1f, ix), __fsub_rn(iy, y0f));     // sw = (ix_ne - ix) * (iy - iy_ne)
  t.w[3] = __fmul_rn(__fsub_rn(ix, x0f), __fsub_rn(iy, y0f));     // se = (ix - ix_nw) * (iy - iy_nw)
  const bool xi0 = x0 >= 0, xi1 = x0 + 1 < W, yi0 = y0 >= 0, yi1 = y0 + 1 < H;
  t.in = (unsigned)(yi0 && xi0) | ((unsigned)(yi0 && xi1) << 1) | ((unsigned)(yi1 && xi0) << 2) | ((unsigned)(yi1 && xi1) << 3);
  t.off = (int64_t)y0 * W + x0;
  float m = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (t.in & (1u << k)) m = __fadd_rn(m, t.w[k]);
  // mask[mask < 0.9999] = 0; mask[mask > 0] = 1 (float32 comparisons, as torch makes them)
  if (m < 0.9999f) m = 0.f;
  if (m > 0.f) m = 1.f;
  t.mask = m;
  return t;
}

// the bilinear sample of one plane (zeros outside), corners added in ATen's order
__device__ __forceinline__ float sample(const float* __restrict__ plane, const Taps& t, int W) {
  float acc = 0.f;
  if (t.in & 1u) acc = fmaf(__ldg(plane + t.off), t.w[0], acc);
  if (t.in & 2u) acc = fmaf(__ldg(plane + t.off + 1), t.w[1], acc);
  if (t.in & 4u) acc = fmaf(__ldg(plane + t.off + W), t.w[2], acc);
  if (t.in & 8u) acc = fmaf(__ldg(plane + t.off + W + 1), t.w[3], acc);
  return acc;
}

// out [B, C, H, W] = warp(x) * mask, mask_out (may be NULL) [B, C, H, W] = the mask
__global__ void __launch_bounds__(256)
flow_warp_kernel(const float* __restrict__ x, const float* __restrict__ flow, float* __restrict__ out, float* __restrict__ mask_out, int C,
                 int H, int W, int64_t total) {
  const int64_t HW = (int64_t)H * W;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / HW, q = i % HW;
    const int px = (int)(q % W), py = (int)(q / W);
    const Taps t = warp_taps(px, py, __ldg(flow + 2 * b * HW + q), __ldg(flow + (2 * b + 1) * HW + q), H, W);
    for (int c = 0; c < C; ++c) {
      const int64_t o = (b * C + c) * HW;
      out[o + q] = __fmul_rn(sample(x + o, t, W), t.mask);
      if (mask_out) mask_out[o + q] = t.mask;
    }
  }
}

struct Slots {
  const float* img[MAX_SLOTS];    // [3, H, W] per slot
  const float* par[MAX_SLOTS];    // [C, H, W] per slot
  const float* flow[MAX_SLOTS];   // [2, H, W] per slot (the centre's is not read)
  float wt[MAX_SLOTS];            // temporal weights
};

// out [C, H, W]: the fused parsing map of the centre slot; per-slot normalised weights live in shared memory [nslot][blockDim]
__global__ void __launch_bounds__(128)
parsing_fuse_kernel(const Slots s, float* __restrict__ out, int nslot, int C, int H, int W) {
  extern __shared__ float s_w[];
  const int64_t HW = (int64_t)H * W;
  const int centre = nslot / 2;
  float* wp = s_w + threadIdx.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < HW; q += (int64_t)gridDim.x * blockDim.x) {
    const int px = (int)(q % W), py = (int)(q / W);
    const float* ic = s.img[centre];
    const float c0 = __ldg(ic + q), c1 = __ldg(ic + HW + q), c2 = __ldg(ic + 2 * HW + q);
    float wsum = 0.f;
    for (int k = 0; k < nslot; ++k) {
      float w;
      if (k == centre) {
        w = s.wt[k];                                         // ws[window] = 1.0, times wt
      } else {
        const float* f = s.flow[k];
        const Taps t = warp_taps(px, py, __ldg(f + q), __ldg(f + HW + q), H, W);
        const float* im = s.img[k];
        const float d0 = __fsub_rn(__fmul_rn(sample(im, t, W), t.mask), c0);
        const float d1 = __fsub_rn(__fmul_rn(sample(im + HW, t, W), t.mask), c1);
        const float d2 = __fsub_rn(__fmul_rn(sample(im + 2 * HW, t, W), t.mask), c2);
        const float mean = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2)), 3.f);
        const float ws = __fmul_rn(expf(__fdiv_rn(-mean, 0.08f)), t.mask);
        w = __fmul_rn(ws, s.wt[k]);
      }
      wp[k * blockDim.x] = w;
      wsum = __fadd_rn(wsum, w);
    }
    for (int k = 0; k < nslot; ++k) wp[k * blockDim.x] = __fdiv_rn(wp[k * blockDim.x], wsum);
    for (int c = 0; c < C; ++c) {
      const int64_t po = (int64_t)c * HW;
      float acc = 0.f;
      for (int k = 0; k < nslot; ++k) {
        float v;
        if (k == centre) {
          v = __ldg(s.par[k] + po + q);
        } else {
          const float* f = s.flow[k];
          const Taps t = warp_taps(px, py, __ldg(f + q), __ldg(f + HW + q), H, W);
          v = __fmul_rn(sample(s.par[k] + po, t, W), t.mask);
        }
        acc = __fadd_rn(acc, __fmul_rn(v, wp[k * blockDim.x]));
      }
      out[po + q] = acc;
    }
  }
}

}  // namespace

extern "C" int vt_flow_warp_f32(const float* x, const float* flow, float* out, float* mask, int B, int C, int H, int W, void* stream) {
  VT_CHECK(x && flow && out && B >= 1 && C >= 1 && H >= 1 && W >= 1, "flow_warp: bad args");
  const int64_t total = (int64_t)B * H * W;
  flow_warp_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(x, flow, out, mask, C, H, W, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_parsing_fuse_f32(const float* const* img, const float* const* par, const float* const* flow, const float* wt, int nslot,
                                   float* out, int C, int H, int W, void* stream) {
  VT_CHECK(img && par && flow && wt && out && nslot >= 1 && nslot <= MAX_SLOTS && nslot % 2 == 1 && C >= 1 && H >= 1 && W >= 1,
           "parsing_fuse: bad args (nslot = 2 * window + 1 <= %d)", MAX_SLOTS);
  Slots s;
  for (int k = 0; k < nslot; ++k) {
    VT_CHECK(img[k] && par[k] && (k == nslot / 2 || flow[k]), "parsing_fuse: slot %d has a NULL pointer", k);
    s.img[k] = img[k];
    s.par[k] = par[k];
    s.flow[k] = flow[k];
    s.wt[k] = wt[k];
  }
  for (int k = nslot; k < MAX_SLOTS; ++k) {
    s.img[k] = s.par[k] = s.flow[k] = nullptr;
    s.wt[k] = 0.f;
  }
  const int threads = 128;
  const int64_t HW = (int64_t)H * W;
  parsing_fuse_kernel<<<grid1(HW, threads), threads, (size_t)nslot * threads * sizeof(float), (cudaStream_t)stream>>>(s, out, nslot, C,
                                                                                                                        H, W);
  VT_LAUNCH_CHECK();
  return 0;
}
