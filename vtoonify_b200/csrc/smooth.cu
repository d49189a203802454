// Parsing-map smoothing (smooth_parsing_map.py:38-74, 155-165): the flow warp and the temporal window fusion.
//   flow_warp     the script's warp(x, flo): grid_sample(x, grid + flo, align_corners=True, zeros) * mask and the thresholded mask
//   parsing_fuse  one centre frame: per pixel, the 2 * window + 1 slots' spatial weights exp(-mean((warp(I_s) - I_c)^2) / 0.08) * mask,
//                 times the temporal weights, normalised, and the weighted sum of the warped parsing maps (the centre slot unwarped
//                 with weight wt[window])
//   parsing_fuse_down  the same fusion for B centres, then Downsample([1, 3, 3, 1], 2) and a scale, from a fused tile in shared memory
//   smooth_frame_prep  uint8 frames -> the 2x up-sampled image Is and RAFT's stem input of (Is + 1) * 255 / 2 (one-pass smoothing)
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

// The per-pixel fusion, shared by parsing_fuse_kernel and parsing_fuse_down_kernel so that both compute the same bits.  S holds the slot
// tables (img, par, flow, wt); centre e0's slot k is entry e0 + k of img / par / flow and k of wt.
// fuse_weights: the normalised weight of every slot of pixel q = (px, py) into wp[k * ws]
template <class S>
__device__ __forceinline__ void fuse_weights(const S& s, int e0, int nslot, int px, int py, int64_t q, int H, int W, float* wp, int ws) {
  const int64_t HW = (int64_t)H * W;
  const int centre = nslot / 2;
  const float* ic = s.img[e0 + centre];
  const float c0 = __ldg(ic + q), c1 = __ldg(ic + HW + q), c2 = __ldg(ic + 2 * HW + q);
  float wsum = 0.f;
  for (int k = 0; k < nslot; ++k) {
    float w;
    if (k == centre) {
      w = s.wt[k];                                         // ws[window] = 1.0, times wt
    } else {
      const float* f = s.flow[e0 + k];
      const Taps t = warp_taps(px, py, __ldg(f + q), __ldg(f + HW + q), H, W);
      const float* im = s.img[e0 + k];
      const float d0 = __fsub_rn(__fmul_rn(sample(im, t, W), t.mask), c0);
      const float d1 = __fsub_rn(__fmul_rn(sample(im + HW, t, W), t.mask), c1);
      const float d2 = __fsub_rn(__fmul_rn(sample(im + 2 * HW, t, W), t.mask), c2);
      const float mean = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2)), 3.f);
      const float ws_ = __fmul_rn(expf(__fdiv_rn(-mean, 0.08f)), t.mask);
      w = __fmul_rn(ws_, s.wt[k]);
    }
    wp[k * ws] = w;
    wsum = __fadd_rn(wsum, w);
  }
  for (int k = 0; k < nslot; ++k) wp[k * ws] = __fdiv_rn(wp[k * ws], wsum);
}

// fuse_channel: the fused value of channel plane offset po (c * H * W) at pixel q, from the weights fuse_weights wrote
template <class S>
__device__ __forceinline__ float fuse_channel(const S& s, int e0, int nslot, int px, int py, int64_t q, int64_t po, int H, int W,
                                              const float* wp, int ws) {
  const int64_t HW = (int64_t)H * W;
  const int centre = nslot / 2;
  float acc = 0.f;
  for (int k = 0; k < nslot; ++k) {
    float v;
    if (k == centre) {
      v = __ldg(s.par[e0 + k] + po + q);
    } else {
      const float* f = s.flow[e0 + k];
      const Taps t = warp_taps(px, py, __ldg(f + q), __ldg(f + HW + q), H, W);
      v = __fmul_rn(sample(s.par[e0 + k] + po, t, W), t.mask);
    }
    acc = __fadd_rn(acc, __fmul_rn(v, wp[k * ws]));
  }
  return acc;
}

// out [C, H, W]: the fused parsing map of the centre slot; per-slot normalised weights live in shared memory [nslot][blockDim]
__global__ void __launch_bounds__(128)
parsing_fuse_kernel(const Slots s, float* __restrict__ out, int nslot, int C, int H, int W) {
  extern __shared__ float s_w[];
  const int64_t HW = (int64_t)H * W;
  float* wp = s_w + threadIdx.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < HW; q += (int64_t)gridDim.x * blockDim.x) {
    const int px = (int)(q % W), py = (int)(q / W);
    fuse_weights(s, 0, nslot, px, py, q, H, W, wp, blockDim.x);
    for (int c = 0; c < C; ++c) {
      const int64_t po = (int64_t)c * HW;
      out[po + q] = fuse_channel(s, 0, nslot, px, py, q, po, H, W, wp, blockDim.x);
    }
  }
}

// ---- fusion + Downsample([1, 3, 3, 1], 2) + scale, for up to FD_MAX_ENTRIES / nslot centres per launch ----
constexpr int FD_MAX_ENTRIES = 126;      // slot entries per launch: keeps the parameter block under 4 KB
constexpr int FD_TOW = 32;               // output columns per CTA (one warp per output row)
constexpr int FD_THREADS = 256;
constexpr int FD_SMEM_CAP = 96 * 1024;   // the per-CTA budget the output-row count is chosen against

struct DownSlots {
  const float* img[FD_MAX_ENTRIES];
  const float* par[FD_MAX_ENTRIES];
  const float* flow[FD_MAX_ENTRIES];
  float wt[MAX_SLOTS];
};

// the fused 2x tile of a CTA: rows 2 * oy0 - 1 .. 2 * (oy0 + th) and columns 2 * ox0 - 1 .. 2 * (ox0 + FD_TOW), i.e. the outputs' 4 x 4
// taps with Downsample's padding of 1; pixels outside the map are the padding zeros
__host__ __device__ constexpr int fd_cols() { return 2 * FD_TOW + 2; }
__host__ __device__ inline int fd_pixels(int th) { return (2 * th + 2) * fd_cols(); }

// grid (tiles, centres); dynamic shared memory: nslot weight planes and two fused-channel planes of fd_pixels(th) floats.  Per channel:
// the CTA writes the fused channel of its tile (plus halo) to a plane, then each output sums its 16 taps in the order of
// upfirdn2d_stream_kernel<1, 2> (row by row, left to right, one fma chain from 0) and is scaled by `scale` (then TF32-rounded when
// round_tf32, as vt_axpby_f32 does).  The planes alternate, so one barrier per channel separates the writes from the reads.
__global__ void __launch_bounds__(FD_THREADS)
parsing_fuse_down_kernel(const __grid_constant__ DownSlots s, float* __restrict__ out, int64_t out_bstride, int nslot, int C, int H, int W,
                         int Ho, int Wo, int th, int tiles_x, float scale, int round_tf32) {
  extern __shared__ float smem[];
  const int P = fd_pixels(th), cols = fd_cols();
  float* s_w = smem;
  float* plane = smem + (size_t)nslot * P;
  const int e0 = blockIdx.y * nslot;
  const int oy0 = (blockIdx.x / tiles_x) * th, ox0 = (blockIdx.x % tiles_x) * FD_TOW;
  const int fy0 = 2 * oy0 - 1, fx0 = 2 * ox0 - 1;
  const int64_t HW = (int64_t)H * W;
  for (int p = threadIdx.x; p < P; p += FD_THREADS) {
    const int py = fy0 + p / cols, px = fx0 + p % cols;
    if (py >= 0 && py < H && px >= 0 && px < W) fuse_weights(s, e0, nslot, px, py, (int64_t)py * W + px, H, W, s_w + p, P);
  }
  // the Downsample kernel: outer([1, 3, 3, 1]) / 64, symmetric, so the flip of the true convolution changes nothing
  const float k1[4] = {1.f, 3.f, 3.f, 1.f};
  const int ty = threadIdx.x / FD_TOW, tx = threadIdx.x % FD_TOW;
  const int oy = oy0 + ty, ox = ox0 + tx;
  const bool writer = ty < th && oy < Ho && ox < Wo;
  float* ob = out + (int64_t)blockIdx.y * out_bstride;
  for (int c = 0; c < C; ++c) {
    float* pl = plane + (size_t)(c & 1) * P;
    const int64_t po = (int64_t)c * HW;
    for (int p = threadIdx.x; p < P; p += FD_THREADS) {
      const int py = fy0 + p / cols, px = fx0 + p % cols;
      float v = 0.f;
      if (py >= 0 && py < H && px >= 0 && px < W) v = fuse_channel(s, e0, nslot, px, py, (int64_t)py * W + px, po, H, W, s_w + p, P);
      pl[p] = v;
    }
    __syncthreads();
    if (writer) {
      const float* src = pl + (2 * ty) * cols + 2 * tx;
      float acc = 0.f;
#pragma unroll
      for (int ky = 0; ky < 4; ++ky)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc = fmaf(k1[ky] * k1[i] / 64.f, src[ky * cols + i], acc);
      const float v = acc * scale;
      ob[(int64_t)c * Ho * Wo + (int64_t)oy * Wo + ox] = round_tf32 ? vt_round_tf32(v) : v;
    }
  }
}

// ---- frame prep of smoothing: uint8 frames -> Is (2x bilinear of ToTensor + Normalize) and RAFT's stem input of (Is + 1) * 255 / 2 ----
// one thread per 2 x 2 block of Is pixels, i.e. per stem-input pixel (y, x) of the [B, H, W, cpad] space-to-depth tensor (grid.y = B)
__global__ void __launch_bounds__(256)
smooth_frame_prep_kernel(const uint8_t* __restrict__ frames, float* __restrict__ img, float* __restrict__ z, int H, int W, int cpad) {
  const int b = blockIdx.y;
  const int64_t HW = (int64_t)H * W, HW4 = 4 * HW;
  const uint8_t* fp = frames + (int64_t)b * HW * 3;
  float* ib = img + (int64_t)b * 3 * HW4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)(i / W);
    float v[12];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const uint8_t* pc = fp + c;
      const auto ld = [&](int64_t o) { return vt_u8_unit(__ldg(pc + 3 * o)); };
#pragma unroll
      for (int q = 0; q < 4; ++q) v[q * 3 + c] = vt_bilinear_up2(ld, 2 * y + (q >> 1), 2 * x + (q & 1), H, W);
      float* row = ib + (int64_t)c * HW4 + (int64_t)(2 * y) * (2 * W) + 2 * x;
      *reinterpret_cast<float2*>(row) = make_float2(v[c], v[3 + c]);
      *reinterpret_cast<float2*>(row + 2 * W) = make_float2(v[6 + c], v[9 + c]);
    }
    // the script's (I + 1) * 255.0 / 2, three roundings, then RAFT's 2 * (x / 255) - 1
#pragma unroll
    for (int k = 0; k < 12; ++k) v[k] = vt_raft_unit(__fdiv_rn(__fmul_rn(__fadd_rn(v[k], 1.f), 255.f), 2.f));
    float4* op = reinterpret_cast<float4*>(z + (((int64_t)b * H + y) * W + x) * cpad);
    op[0] = make_float4(v[0], v[1], v[2], v[3]);
    op[1] = make_float4(v[4], v[5], v[6], v[7]);
    op[2] = make_float4(v[8], v[9], v[10], v[11]);
    for (int k = 3; k < cpad / 4; ++k) op[k] = make_float4(0.f, 0.f, 0.f, 0.f);
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

extern "C" int vt_parsing_fuse_down_f32(const float* const* img, const float* const* par, const float* const* flow, const float* wt, int nslot,
                                        int B, float* out, int64_t out_bstride, int C, int H, int W, float scale, int round_tf32,
                                        void* stream) {
  VT_CHECK(img && par && flow && wt && out && nslot >= 1 && nslot <= MAX_SLOTS && nslot % 2 == 1 && B >= 1 && C >= 1 && H >= 2 && W >= 2,
           "parsing_fuse_down: bad args (nslot = 2 * window + 1 <= %d, H and W >= 2)", MAX_SLOTS);
  const int Ho = H / 2, Wo = W / 2;      // Downsample([1, 3, 3, 1], 2): pad 1 on each side, 4 taps, stride 2
  VT_CHECK(out_bstride >= (int64_t)C * Ho * Wo, "parsing_fuse_down: out_bstride %lld is smaller than one sample (%d x %d x %d)",
           (long long)out_bstride, C, Ho, Wo);
  for (int e = 0; e < B * nslot; ++e)
    VT_CHECK(img[e] && par[e] && (e % nslot == nslot / 2 || flow[e]), "parsing_fuse_down: centre %d slot %d has a NULL pointer", e / nslot,
             e % nslot);
  int th = 8;                             // output rows per CTA: the most that keeps the weight and channel planes in the budget
  while (th > 1 && (size_t)(nslot + 2) * fd_pixels(th) * sizeof(float) > (size_t)FD_SMEM_CAP) th /= 2;
  const size_t smem = (size_t)(nslot + 2) * fd_pixels(th) * sizeof(float);
  static bool attr_done = false;
  if (!attr_done) {
    VT_CUDA(cudaFuncSetAttribute(parsing_fuse_down_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FD_SMEM_CAP));
    attr_done = true;
  }
  const int tiles_x = (int)vt_cdiv(Wo, FD_TOW), tiles = tiles_x * (int)vt_cdiv(Ho, th);
  const int per = FD_MAX_ENTRIES / nslot;   // centres per launch
  for (int b0 = 0; b0 < B; b0 += per) {
    const int nb = B - b0 < per ? B - b0 : per;
    DownSlots s;
    for (int e = 0; e < FD_MAX_ENTRIES; ++e) {
      const bool on = e < nb * nslot;
      s.img[e] = on ? img[b0 * nslot + e] : nullptr;
      s.par[e] = on ? par[b0 * nslot + e] : nullptr;
      s.flow[e] = on ? flow[b0 * nslot + e] : nullptr;
    }
    for (int k = 0; k < MAX_SLOTS; ++k) s.wt[k] = k < nslot ? wt[k] : 0.f;
    parsing_fuse_down_kernel<<<dim3((unsigned)tiles, (unsigned)nb), FD_THREADS, smem, (cudaStream_t)stream>>>(
        s, out + (int64_t)b0 * out_bstride, out_bstride, nslot, C, H, W, Ho, Wo, th, tiles_x, scale, round_tf32);
    VT_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int vt_smooth_frame_prep_u8(const uint8_t* frames, float* img, float* stem, int B, int H, int W, int cpad, void* stream) {
  VT_CHECK(frames && img && stem && B >= 1 && B <= 65535 && H >= 1 && W >= 1, "smooth_frame_prep: bad args");
  VT_CHECK(cpad >= 12 && cpad % 4 == 0 && (((uintptr_t)stem | (uintptr_t)img) & 15) == 0,
           "smooth_frame_prep: cpad must be a multiple of 4 >= 12, img and stem 16-byte aligned");
  const int64_t n = (int64_t)H * W;
  smooth_frame_prep_kernel<<<dim3(grid1(n, 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(frames, img, stem, H, W, cpad);
  VT_LAUNCH_CHECK();
  return 0;
}
