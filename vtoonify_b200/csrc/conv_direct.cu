// conv_direct.cu — fp32-exact CUDA-core convolutions on NHWC activations.
//
//   vt_conv2d_direct_f32 : implicit-GEMM FFMA kernel (64 pixels x 64 couts x 16 k per CTA, 4x4 register tile).
//                          It is the fp32 reference-grade path ("precision=fp32") used to cross-check the wgmma
//                          kernel on the GPU and to run shapes the tensor-core kernel does not take.
//   vt_smalln_conv_f32   : Cout <= 4 convolutions (ToRGB 1x1, fusion_skip 3x3, Fusion mask 3x3, encoder[-1] 1x1).
//                          These are < 0.4 % of the FLOPs but read the largest tensors (SURVEY.md App. B), so they
//                          are written as HBM-streaming kernels: 8 lanes x float4 cover 32 channels of one pixel,
//                          weights live in shared memory, planar (NCHW) 3-channel output, with the skip-path
//                          `Upsample` (upfirdn2d up=2, model/stylegan/model.py:32-50,388-390) and the
//                          `f_E * m_E` product (model/vtoonify.py:127) fused into the epilogue.
//
// Both follow the arithmetic of F.conv2d / F.conv_transpose2d as called by the reference at
// model/stylegan/op/conv2d_gradfix.py:34-42,66-75 and model/vtoonify.py:96-97,111-113,162-182,195-198:
// a transposed stride-2 conv is issued as 4 polyphase calls (tap lists with dy,dx in {0,-1}) into a strided view.
#include "common.cuh"

int g_smalln_is = 1;   // input-stationary kernel for 3x3 small-N convolutions: 1 = automatic (Cout == 1 on large maps), 2 = always, 0 = never

namespace {

constexpr int BM = 64, BN = 64, BK = 16;
constexpr int LDA = BM + 4, LDB = BN + 4;

struct DirectArgs {
  vt_conv_desc d;
  int w_rows;   // weight rows per tap slab (n_phase * Cout)
  int w_row0;   // first row of this launch's phase
};

__global__ void __launch_bounds__(256)
conv_direct_kernel(const __grid_constant__ DirectArgs args) {
  const vt_conv_desc& d = args.d;
  __shared__ __align__(16) float As[BK][LDA];
  __shared__ __align__(16) float Bs[BK][LDB];

  const int tid = threadIdx.x;
  const int b = blockIdx.z;
  const int n0 = blockIdx.y * BN;
  const int64_t HoWo = (int64_t)d.Ho * d.Wo;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int wb = (d.wB > 1) ? b : 0;

  // loader role
  const int lp = tid >> 2;        // pixel (A) / cout (B) index within the tile
  const int lk = (tid & 3) * 4;   // k offset within the chunk
  const int64_t lm = m0 + lp;
  const bool lm_ok = lm < HoWo;
  const int loy = lm_ok ? (int)(lm / d.Wo) : 0;
  const int lox = lm_ok ? (int)(lm % d.Wo) : 0;
  const int ln = n0 + lp;
  const bool ln_ok = ln < d.Cout;

  // compute role
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  int coff = 0;
  for (int s = 0; s < d.n_src; ++s) {
    const float* sp = d.src[s];
    const int sc = d.src_c[s], scs = d.src_cstride[s];
    for (int t = 0; t < d.taps; ++t) {
      const int iy = loy * d.stride + d.tap_dy[t];
      const int ix = lox * d.stride + d.tap_dx[t];
      const bool pix_ok = lm_ok && iy >= 0 && iy < d.H && ix >= 0 && ix < d.W;
      const float* ap = sp + (((int64_t)b * d.H + iy) * d.W + ix) * scs;
      const float* wp = d.weight + (((int64_t)wb * d.w_taps + d.tap_w[t]) * args.w_rows + args.w_row0 + ln) * d.w_cstride + coff;
      for (int c0 = 0; c0 < sc; c0 += BK) {
        const int c = c0 + lk;
        float4 av = make_float4(0.f, 0.f, 0.f, 0.f), bv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (pix_ok && c < sc) av = *reinterpret_cast<const float4*>(ap + c);
        if (ln_ok && c < sc) bv = *reinterpret_cast<const float4*>(wp + c);
        __syncthreads();  // previous chunk fully consumed
        As[lk + 0][lp] = av.x; As[lk + 1][lp] = av.y; As[lk + 2][lp] = av.z; As[lk + 3][lp] = av.w;
        Bs[lk + 0][lp] = bv.x; Bs[lk + 1][lp] = bv.y; Bs[lk + 2][lp] = bv.z; Bs[lk + 3][lp] = bv.w;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
          const float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
          const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
          const float a[4] = {a4.x, a4.y, a4.z, a4.w};
          const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
      }
    }
    coff += sc;
  }

  // epilogue
  const float nw = (d.noise && d.noise_w) ? *d.noise_w : 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= HoWo) continue;
    const int oy = (int)(m / d.Wo), ox = (int)(m % d.Wo);
    const int64_t off = d.phase_off[0] + (int64_t)b * d.out_sb + (int64_t)oy * d.out_sy + (int64_t)ox * d.out_sx;
    const float nz = d.noise ? nw * d.noise[off / d.out_cpitch] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= d.Cout) continue;
      float v = acc[i][j];
      if (d.noise) v += nz;
      if (d.bias) v += d.bias[n];
      if (d.act == VT_ACT_LRELU) v = vt_lrelu(v, d.slope_vec ? d.slope_vec[n] : d.slope) * d.gain;
      else if (d.act == VT_ACT_RELU_TANH) v = tanhf(fmaxf(v, 0.f));
      if (d.res) v = v * d.alpha + d.beta * d.res[off + n];
      else if (d.alpha != 1.f) v = v * d.alpha;
      if (d.round_tf32) v = vt_round_tf32(v);
      d.out[off + n] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
struct SmallNArgs {
  vt_smalln_desc d;
};

// Per-pixel tail shared by both small-N kernels: lane L <-> pixel (y, x0 + L) of batch image b; `keep[n]` holds the NHWC-source
// part of the convolution.  Adds the planar-source taps, bias, activation, the up-sampled skip, stores planar outputs and (optionally)
// writes mul_src * out[:,0] for the whole warp row.  Must be called by all 32 lanes.
template <int N>
__device__ __forceinline__ void smalln_pixel_epilogue(const vt_smalln_desc& d, int b, int y, int x0, bool row_ok, float (&keep)[N],
                                                      const float* Wp, const float* Ks) {
  const int lane = threadIdx.x & 31;
  const int sub = lane & 7;
  const int grp = lane >> 3;
  const int64_t HW = (int64_t)d.H * d.W;
  const int hs = d.H / 2, ws = d.W / 2;
  // ---- per-pixel epilogue: lane L <-> pixel (y, x0 + L)
  const int x = x0 + lane;
  const bool p_ok = row_ok && x < d.W;
  const int64_t p = (int64_t)y * d.W + x;
  float m0v = 0.f;
  if (p_ok) {
    // Both tap loops are written branch-free (clamped address, 0/1 weight) over a compile-time 9 taps so that all loads of a
    // pixel are in flight together; this tail runs once per pixel with little other work to hide a serial chain of L2 latencies.
    if (d.tsum) {   // shifted sum of per-tap partial products (1x1 tensor-core conv output)
      float tv[9][N];
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int tt = t < d.taps ? t : 0;
        const int iy = y + d.tap_dy[tt], ix = x + d.tap_dx[tt];
        const bool ok = t < d.taps && iy >= 0 && iy < d.H && ix >= 0 && ix < d.W;
        const int cy = ok ? iy : y, cx = ok ? ix : x;
        const float* tp = d.tsum + (((int64_t)b * d.H + cy) * d.W + cx) * d.tsum_c + tt * N;
#pragma unroll
        for (int n = 0; n < N; ++n) tv[t][n] = ok ? __ldg(tp + n) : 0.f;
      }
#pragma unroll
      for (int t = 0; t < 9; ++t)
#pragma unroll
        for (int n = 0; n < N; ++n) keep[n] += tv[t][n];
      for (int t = 9; t < d.taps; ++t) {
        const int iy = y + d.tap_dy[t], ix = x + d.tap_dx[t];
        if (iy < 0 || iy >= d.H || ix < 0 || ix >= d.W) continue;
        const float* tp = d.tsum + (((int64_t)b * d.H + iy) * d.W + ix) * d.tsum_c + t * N;
#pragma unroll
        for (int n = 0; n < N; ++n) keep[n] += __ldg(tp + n);
      }
    }
    if (d.n_planar > 0) {
      for (int cp = 0; cp < d.n_planar; ++cp) {
        const float* pp = d.planar + ((int64_t)b * d.n_planar + cp) * HW;
        float av[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const int tt = t < d.taps ? t : 0;
          const int iy = y + d.tap_dy[tt], ix = x + d.tap_dx[tt];
          const bool ok = t < d.taps && iy >= 0 && iy < d.H && ix >= 0 && ix < d.W;
          av[t] = ok ? __ldg(pp + (int64_t)iy * d.W + ix) : 0.f;
        }
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          if (t < d.taps) {
#pragma unroll
            for (int n = 0; n < N; ++n) keep[n] = fmaf(av[t], Wp[(t * N + n) * d.n_planar + cp], keep[n]);
          }
        }
        for (int t = 9; t < d.taps; ++t) {
          const int iy = y + d.tap_dy[t], ix = x + d.tap_dx[t];
          if (iy < 0 || iy >= d.H || ix < 0 || ix >= d.W) continue;
          const float a = __ldg(pp + (int64_t)iy * d.W + ix);
#pragma unroll
          for (int n = 0; n < N; ++n) keep[n] = fmaf(a, Wp[(t * N + n) * d.n_planar + cp], keep[n]);
        }
      }
    }
#pragma unroll
    for (int n = 0; n < N; ++n) {
      float v = keep[n];
      if (d.bias) v += d.bias[n];
      if (d.act == VT_ACT_RELU_TANH) v = tanhf(fmaxf(v, 0.f));
      if (d.skip) {
        // upfirdn2d(skip, k, up=2, down=1, pad=(2,1)) at (y, x): taps with (y - 2 + ky) even
        const float* sp = d.skip + ((int64_t)b * N + n) * (int64_t)hs * ws;
        float u = 0.f;
        const int ty = y - 2, tx = x - 2;
        for (int ky = (ty & 1) ? 1 : 0; ky < 4; ky += 2) {
          const int iy = (ty + ky) >> 1;  // ty + ky is even; arithmetic shift == floor
          if (ty + ky < 0 || iy >= hs) continue;
          for (int kx = (tx & 1) ? 1 : 0; kx < 4; kx += 2) {
            const int ix = (tx + kx) >> 1;
            if (tx + kx < 0 || ix >= ws) continue;
            u = fmaf(__ldg(sp + (int64_t)iy * ws + ix), Ks[(3 - ky) * 4 + (3 - kx)], u);
          }
        }
        v += u;
      }
      d.out[((int64_t)b * N + n) * HW + p] = v;
      if (n == 0) m0v = v;
    }
  }
  if (d.mul_out) {
    for (int it = 0; it < 8; ++it) {
      const float m = __shfl_sync(0xffffffffu, m0v, it * 4 + grp);
      const int xx = x0 + it * 4 + grp;
      if (row_ok && xx < d.W) {
        const int64_t pp = (int64_t)y * d.W + xx;
        const float* ms = d.mul_src + ((int64_t)b * HW + pp) * d.mul_c;
        float* mo = d.mul_out + ((int64_t)b * HW + pp) * d.mul_c;
        for (int c = sub * 4; c < d.mul_c; c += 32) {
          float4 a = __ldg(reinterpret_cast<const float4*>(ms + c));
          a.x *= m; a.y *= m; a.z *= m; a.w *= m;
          if (d.round_tf32) { a.x = vt_round_tf32(a.x); a.y = vt_round_tf32(a.y); a.z = vt_round_tf32(a.z); a.w = vt_round_tf32(a.w); }
          *reinterpret_cast<float4*>(mo + c) = a;
        }
      }
    }
  }

}

template <int N>
__global__ void __launch_bounds__(256)
smalln_conv_kernel(const __grid_constant__ SmallNArgs args) {
  const vt_smalln_desc& d = args.d;
  extern __shared__ __align__(16) float smem[];
  const int CW = d.src2_mode ? 2 * d.src_c : d.src_c;           // weight-row channels (virtual concat doubles them)
  float* Ws = smem;                                              // [taps][N][CW]
  float* Wp = smem + (size_t)d.taps * N * CW;                    // [taps][N][n_planar]
  float* Ks = Wp + (size_t)d.taps * N * (d.n_planar > 0 ? d.n_planar : 0);  // [16] skip kernel
  float* Tc = Ks + 16;                                           // [taps][N] per-tap constants (affine fold), optional
  const int b = blockIdx.y;
  const int wb = d.wB > 1 ? b : 0;
  for (int i = threadIdx.x; i < d.taps * N * CW; i += blockDim.x) {
    const int c = i % CW;
    const int tn = i / CW;
    const int t = tn / N, n = tn % N;
    Ws[i] = d.weight[(((int64_t)wb * d.w_taps + d.tap_w[t]) * d.Cout + n) * d.w_cstride + c];
  }
  if (d.n_planar > 0) {
    for (int i = threadIdx.x; i < d.taps * N * d.n_planar; i += blockDim.x) {
      const int cp = i % d.n_planar;
      const int tn = i / d.n_planar;
      const int t = tn / N, n = tn % N;
      Wp[i] = d.planar_weight[((int64_t)d.tap_w[t] * d.Cout + n) * d.n_planar + cp];
    }
  }
  if (d.skip && threadIdx.x < 16) Ks[threadIdx.x] = d.skip_kernel[threadIdx.x];
  if (d.tap_const)
    for (int i = threadIdx.x; i < d.taps * N; i += blockDim.x)
      Tc[i] = d.tap_const[((int64_t)wb * d.w_taps + d.tap_w[i / N]) * d.Cout + (i % N)];
  __syncthreads();

  // A block owns a patch of 8 rows x 32 columns (warp w <-> row w): the vertical taps of neighbouring warps hit the
  // same L1 lines (1.25x re-read instead of 3x from L2).  Channels are walked in 32-wide chunks with the taps inside,
  // so the L1 working set is ~10 rows x 34 px x 128 B.  A warp processes its 32 pixels 4 at a time (8 lanes x float4 =
  // one pixel's 32-channel chunk per coalesced load); reduced results are handed to lane L <-> pixel L for the
  // epilogue, so planar stores and skip reads are coalesced.
  const int lane = threadIdx.x & 31;
  const int sub = lane & 7;      // channel slice
  const int grp = lane >> 3;     // pixel within the sub-iteration
  const int warp = threadIdx.x >> 5;
  const int64_t HW = (int64_t)d.H * d.W;
  const int patches_x = (d.W + 31) / 32;
  const int patches_y = (d.H + 7) / 8;
  const int hs = d.H / 2, ws = d.W / 2;
  for (int patch = blockIdx.x; patch < patches_x * patches_y; patch += gridDim.x) {
    const int y = (patch / patches_x) * 8 + warp;
    const int x0 = (patch % patches_x) * 32;
    const bool row_ok = y < d.H;
    float keep[N];
#pragma unroll
    for (int n = 0; n < N; ++n) keep[n] = 0.f;
    if (d.src_c > 0) {
      // acc[it][n]: the 8 sub-iterations (4 pixels each) are kept live together so that every (channel chunk, tap) step
      // issues 8 independent 16-byte loads per lane before any FMA consumes them (memory-level parallelism)
      float acc[8][N];
#pragma unroll
      for (int it = 0; it < 8; ++it)
#pragma unroll
        for (int n = 0; n < N; ++n) acc[it][n] = 0.f;
      if (row_ok) {
        for (int c = sub * 4; c < d.src_c; c += 32) {
          for (int t = 0; t < d.taps; ++t) {
            const int iy = y + d.tap_dy[t];
            if (iy < 0 || iy >= d.H) continue;
            const int ixb = x0 + grp + d.tap_dx[t];
            const int64_t rowo = (((int64_t)b * d.H + iy) * d.W) * d.src_cstride + c;
            float4 a[8], e[8];
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int ix = ixb + it * 4;
              const bool ok = ix >= 0 && ix < d.W && (ix - d.tap_dx[t]) < d.W;
              a[it] = ok ? __ldg(reinterpret_cast<const float4*>(d.src + rowo + (int64_t)ix * d.src_cstride))
                         : make_float4(0.f, 0.f, 0.f, 0.f);
              if (d.src_mask && ok) {
                const float mm = __ldg(d.src_mask + ((int64_t)b * d.H + iy) * d.W + ix);
                a[it].x *= mm; a[it].y *= mm; a[it].z *= mm; a[it].w *= mm;
              }
              if (d.src2_mode)
                e[it] = ok ? __ldg(reinterpret_cast<const float4*>(d.src2 + rowo + (int64_t)ix * d.src_cstride))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            const float* wt = Ws + (size_t)t * N * CW + c;
#pragma unroll
            for (int n = 0; n < N; ++n) {
              const float4 w = *reinterpret_cast<const float4*>(wt + n * CW);
#pragma unroll
              for (int it = 0; it < 8; ++it) {
                acc[it][n] = fmaf(a[it].x, w.x, acc[it][n]);
                acc[it][n] = fmaf(a[it].y, w.y, acc[it][n]);
                acc[it][n] = fmaf(a[it].z, w.z, acc[it][n]);
                acc[it][n] = fmaf(a[it].w, w.w, acc[it][n]);
              }
            }
            if (d.src2_mode) {   // second half of the virtual concat: |src - src2| (zero outside the image: a = e = 0)
#pragma unroll
              for (int n = 0; n < N; ++n) {
                const float4 w = *reinterpret_cast<const float4*>(wt + n * CW + d.src_c);
#pragma unroll
                for (int it = 0; it < 8; ++it) {
                  acc[it][n] = fmaf(fabsf(a[it].x - e[it].x), w.x, acc[it][n]);
                  acc[it][n] = fmaf(fabsf(a[it].y - e[it].y), w.y, acc[it][n]);
                  acc[it][n] = fmaf(fabsf(a[it].z - e[it].z), w.z, acc[it][n]);
                  acc[it][n] = fmaf(fabsf(a[it].w - e[it].w), w.w, acc[it][n]);
                }
              }
            }
          }
        }
        if (d.tap_const && sub == 0) {   // constant term of the folded affine (only in-bounds taps contribute)
          for (int t = 0; t < d.taps; ++t) {
            const int iy = y + d.tap_dy[t];
            if (iy < 0 || iy >= d.H) continue;
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int ix = x0 + it * 4 + grp + d.tap_dx[t];
              if (ix < 0 || ix >= d.W) continue;
#pragma unroll
              for (int n = 0; n < N; ++n) acc[it][n] += Tc[t * N + n];
            }
          }
        }
      }
#pragma unroll
      for (int it = 0; it < 8; ++it) {
#pragma unroll
        for (int n = 0; n < N; ++n) {
          float v = acc[it][n];
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          // lane 4*it+g takes the result of group g (held by lanes 8g..8g+7)
          const float r = __shfl_sync(0xffffffffu, v, (lane & 3) * 8);
          if ((lane >> 2) == it) keep[n] = r;
        }
      }
    }
    smalln_pixel_epilogue<N>(d, b, y, x0, row_ok, keep, Wp, Ks);
  }
}

// ---- input-stationary small-N 3x3 convolution --------------------------------------------------------------------------
// out[p] = sum_t <x[p + s_t], w_t>.  Instead of gathering 9 shifted pixels per output (9x L1 traffic, and |src - src2| of the
// virtual concat recomputed 9x), every input pixel of the patch (+1-pixel ring) is read ONCE: its 9*N partial dot products
// T[r][t][n] = <x[r], w_t[n]> go to shared memory, and each output pixel then sums 9 shifted T entries.  HBM traffic is the
// input read once (ring overlap 1.2x, served by L2); FMA work is unchanged (9*N*C per pixel).
// Block = 8 warps, output patch 16 rows x 32 columns; phase 1 walks the (16+2)x(32+2) region 4*IT pixels per warp step
// (8 lanes x float4 = one pixel's 32-channel chunk), phase 2 maps lane <-> column like smalln_conv_kernel.
constexpr int IS_TAPS = 9, IS_PH = 16, IS_PW = 32;

template <int N, int IT>
__global__ void __launch_bounds__(256)
smalln_is_kernel(const __grid_constant__ SmallNArgs args, int dy0, int dy1, int dx0, int dx1, int TS) {
  const vt_smalln_desc& d = args.d;
  extern __shared__ __align__(16) float smem[];
  constexpr int TN = IS_TAPS * N;
  const int CW = d.src2_mode ? 2 * d.src_c : d.src_c;
  float* Ws = smem;                                              // [TN][CW]
  float* Wp = Ws + (size_t)TN * CW;                              // [TN][n_planar]
  float* Ks = Wp + (size_t)TN * (d.n_planar > 0 ? d.n_planar : 0);
  float* Tc = Ks + 16;                                           // [TN] per-tap constants (0 if none)
  float* Ts = Tc + ((TN + 3) & ~3);                              // [RH*RW][TS]
  const int b = blockIdx.y;
  const int wb = d.wB > 1 ? b : 0;
  for (int i = threadIdx.x; i < TN * CW; i += blockDim.x) {
    const int c = i % CW, tn = i / CW;
    const int t = tn / N, n = tn % N;
    Ws[i] = d.weight[(((int64_t)wb * d.w_taps + d.tap_w[t]) * d.Cout + n) * d.w_cstride + c];
  }
  if (d.n_planar > 0)
    for (int i = threadIdx.x; i < TN * d.n_planar; i += blockDim.x) {
      const int cp = i % d.n_planar, tn = i / d.n_planar;
      Wp[i] = d.planar_weight[((int64_t)d.tap_w[tn / N] * d.Cout + (tn % N)) * d.n_planar + cp];
    }
  if (d.skip && threadIdx.x < 16) Ks[threadIdx.x] = d.skip_kernel[threadIdx.x];
  for (int i = threadIdx.x; i < TN; i += blockDim.x)
    Tc[i] = d.tap_const ? d.tap_const[((int64_t)wb * d.w_taps + d.tap_w[i / N]) * d.Cout + (i % N)] : 0.f;
  __syncthreads();

  const int lane = threadIdx.x & 31, sub = lane & 7, grp = lane >> 3, warp = threadIdx.x >> 5;
  const int RH = IS_PH + dy1 - dy0, RW = IS_PW + dx1 - dx0, npix = RH * RW;
  const int patches_x = (d.W + IS_PW - 1) / IS_PW, patches_y = (d.H + IS_PH - 1) / IS_PH;
  // shifted-sum offsets of the 9 taps inside Ts (phase 2)
  int toff[IS_TAPS];
#pragma unroll
  for (int t = 0; t < IS_TAPS; ++t) toff[t] = ((d.tap_dy[t] - dy0) * RW + (d.tap_dx[t] - dx0)) * TS + t * N;

  for (int patch = blockIdx.x; patch < patches_x * patches_y; patch += gridDim.x) {
    const int y0 = (patch / patches_x) * IS_PH, x0 = (patch % patches_x) * IS_PW;
    // ---- phase 1: T[r][t][n] for every input pixel r of the region
    for (int base = warp * 4 * IT; base < npix; base += 8 * 4 * IT) {
      const float* pa[IT];
      const float* pe[IT];
      bool ok[IT];
      int rr[IT];
      float pm[IT];
#pragma unroll
      for (int it = 0; it < IT; ++it) {
        const int r = base + it * 4 + grp;
        rr[it] = r;
        const int ry = r / RW, rx = r - ry * RW;
        const int iy = y0 + dy0 + ry, ix = x0 + dx0 + rx;
        ok[it] = r < npix && iy >= 0 && iy < d.H && ix >= 0 && ix < d.W;
        const int64_t o = ok[it] ? ((((int64_t)b * d.H + iy) * d.W + ix) * d.src_cstride) : 0;
        pa[it] = d.src + o;
        pe[it] = d.src2_mode ? d.src2 + o : nullptr;
        pm[it] = (d.src_mask && ok[it]) ? __ldg(d.src_mask + ((int64_t)b * d.H + iy) * d.W + ix) : 1.f;
      }
      float acc[IT][TN];
#pragma unroll
      for (int it = 0; it < IT; ++it)
#pragma unroll
        for (int tn = 0; tn < TN; ++tn) acc[it][tn] = 0.f;
      // software pipeline without extra registers: a's registers are dead after the |a - e| step, so the next trip's a is
      // requested there (covered by the e-half of the math), and the next e right after the e-half (covered by the next a-half).
      // The kernel is latency-bound (2 blocks x 8 warps per SM at 128 registers), not FMA-bound.
      const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
      float4 a[IT], e[IT];
      {
        const int c0 = sub * 4;
#pragma unroll
        for (int it = 0; it < IT; ++it) {
          a[it] = (ok[it] && c0 < d.src_c) ? __ldg(reinterpret_cast<const float4*>(pa[it] + c0)) : z4;
          e[it] = (d.src2_mode && ok[it] && c0 < d.src_c) ? __ldg(reinterpret_cast<const float4*>(pe[it] + c0)) : z4;
        }
      }
      for (int c = sub * 4; c < d.src_c; c += 32) {
        const int cn = c + 32;
        if (d.src_mask) {
#pragma unroll
          for (int it = 0; it < IT; ++it) { a[it].x *= pm[it]; a[it].y *= pm[it]; a[it].z *= pm[it]; a[it].w *= pm[it]; }
        }
#pragma unroll
        for (int tn = 0; tn < TN; ++tn) {
          const float4 w = *reinterpret_cast<const float4*>(Ws + (size_t)tn * CW + c);
#pragma unroll
          for (int it = 0; it < IT; ++it) {
            acc[it][tn] = fmaf(a[it].x, w.x, acc[it][tn]);
            acc[it][tn] = fmaf(a[it].y, w.y, acc[it][tn]);
            acc[it][tn] = fmaf(a[it].z, w.z, acc[it][tn]);
            acc[it][tn] = fmaf(a[it].w, w.w, acc[it][tn]);
          }
        }
        if (d.src2_mode) {   // second half of the virtual concat: |src - src2|, computed once per pixel
#pragma unroll
          for (int it = 0; it < IT; ++it) {
            e[it].x = fabsf(a[it].x - e[it].x); e[it].y = fabsf(a[it].y - e[it].y);
            e[it].z = fabsf(a[it].z - e[it].z); e[it].w = fabsf(a[it].w - e[it].w);
          }
        }
#pragma unroll
        for (int it = 0; it < IT; ++it)
          a[it] = (ok[it] && cn < d.src_c) ? __ldg(reinterpret_cast<const float4*>(pa[it] + cn)) : z4;
        if (d.src2_mode) {
#pragma unroll
          for (int tn = 0; tn < TN; ++tn) {
            const float4 w = *reinterpret_cast<const float4*>(Ws + (size_t)tn * CW + d.src_c + c);
#pragma unroll
            for (int it = 0; it < IT; ++it) {
              acc[it][tn] = fmaf(e[it].x, w.x, acc[it][tn]);
              acc[it][tn] = fmaf(e[it].y, w.y, acc[it][tn]);
              acc[it][tn] = fmaf(e[it].z, w.z, acc[it][tn]);
              acc[it][tn] = fmaf(e[it].w, w.w, acc[it][tn]);
            }
          }
#pragma unroll
          for (int it = 0; it < IT; ++it)
            e[it] = (ok[it] && cn < d.src_c) ? __ldg(reinterpret_cast<const float4*>(pe[it] + cn)) : z4;
        }
      }
      // reduce over the 8 channel-slice lanes; lane (tn & 7) of the pixel's group stores entry tn
#pragma unroll
      for (int it = 0; it < IT; ++it) {
#pragma unroll
        for (int tn = 0; tn < TN; ++tn) {
          float v = acc[it][tn];
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          if ((tn & 7) == sub && rr[it] < npix) Ts[(size_t)rr[it] * TS + tn] = ok[it] ? v + Tc[tn] : 0.f;
        }
      }
    }
    __syncthreads();
    // ---- phase 2: shifted sum + per-pixel tail; warp w owns rows w and w + 8 of the patch
#pragma unroll
    for (int h = 0; h < IS_PH / 8; ++h) {
      const int ly = warp + 8 * h, y = y0 + ly;
      const bool row_ok = y < d.H;
      float keep[N];
#pragma unroll
      for (int n = 0; n < N; ++n) keep[n] = 0.f;
      const float* tp = Ts + (size_t)(ly * RW + lane) * TS;
#pragma unroll
      for (int t = 0; t < IS_TAPS; ++t)
#pragma unroll
        for (int n = 0; n < N; ++n) keep[n] += tp[toff[t] + n];
      smalln_pixel_epilogue<N>(d, b, y, x0, row_ok, keep, Wp, Ks);
    }
    __syncthreads();
  }
}

// Fold the AdaIN affine of Fusion.forward (model/vtoonify.py:125-126) into the mask-conv weights:
//   conv(gamma*(x-mean)*rstd + beta, W) = conv(x, W*a) + sum_c W*bb   with a = gamma*rstd, bb = beta - gamma*mean*rstd,
// the constant only for taps that fall inside the image (the reference zero-pads the normalised tensor).
// grid (taps*N, B); w: [taps][N][C2]; stats: [B][C2][2]; gb: [B][2*C2]; out_w: [B][taps][N][C2]; out_k: [B][taps][N]
__global__ void __launch_bounds__(256)
affine_fold_kernel(const float* __restrict__ w, const float* __restrict__ stats, const float* __restrict__ gb,
                   float* __restrict__ out_w, float* __restrict__ out_k, int C2) {
  const int tn = blockIdx.x, b = blockIdx.y;
  const float* wr = w + (int64_t)tn * C2;
  const float* st = stats + (int64_t)b * C2 * 2;
  const float* gamma = gb + (int64_t)b * 2 * C2;
  const float* beta = gamma + C2;
  float* ow = out_w + ((int64_t)b * gridDim.x + tn) * C2;
  float k = 0.f;
  for (int c = threadIdx.x; c < C2; c += blockDim.x) {
    const float a = gamma[c] * st[c * 2 + 1];
    const float bb = beta[c] - a * st[c * 2];
    ow[c] = wr[c] * a;
    k = fmaf(wr[c], bb, k);
  }
  __shared__ float red[8];
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) k += __shfl_xor_sync(0xffffffffu, k, s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = k;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    out_k[(int64_t)b * gridDim.x + tn] = t;
  }
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

static int validate_conv_desc(const vt_conv_desc* d, const char* who) {
  VT_CHECK(d != nullptr, "%s: null descriptor", who);
  VT_CHECK(d->struct_size == (int)sizeof(vt_conv_desc), "%s: descriptor size mismatch (got %d, want %d)", who,
           d->struct_size, (int)sizeof(vt_conv_desc));
  VT_CHECK(d->n_src == 1 || d->n_src == 2, "%s: n_src must be 1 or 2", who);
  VT_CHECK(d->B >= 1 && d->H >= 1 && d->W >= 1 && d->Ho >= 1 && d->Wo >= 1, "%s: bad spatial shape", who);
  VT_CHECK(d->stride >= 1 && d->taps >= 1 && d->taps <= VT_MAX_TAPS, "%s: bad stride/taps", who);
  // out == NULL is the "image only" form of the fused ToRGB tail (row-strip kernel; the others reject it below)
  VT_CHECK(d->Cout >= 1 && d->weight && (d->out || (d->rgb_w && d->rgb_out)), "%s: bad weight/out", who);
  VT_CHECK(d->wB == 1 || d->wB == d->B, "%s: wB must be 1 or B", who);
  int ctot = 0;
  for (int s = 0; s < d->n_src; ++s) {
    VT_CHECK(d->src[s] != nullptr, "%s: null source %d", who, s);
    VT_CHECK(d->src_c[s] >= 4 && d->src_c[s] % 4 == 0, "%s: src_c[%d]=%d must be a multiple of 4", who, s, d->src_c[s]);
    VT_CHECK(d->src_cstride[s] >= d->src_c[s] && d->src_cstride[s] % 4 == 0, "%s: bad channel stride", who);
    VT_CHECK(aligned16(d->src[s]), "%s: source %d not 16-byte aligned", who, s);
    ctot += d->src_c[s];
  }
  VT_CHECK(d->w_cstride >= ctot && d->w_cstride % 4 == 0 && aligned16(d->weight), "%s: bad weight stride/alignment", who);
  VT_CHECK(d->n_phase == 1 || d->n_phase == 4, "%s: n_phase must be 1 or 4", who);
  VT_CHECK(d->out_cpitch >= d->Cout, "%s: out_cpitch (%d) must be >= Cout", who, d->out_cpitch);
  for (int t = 0; t < d->taps; ++t) {
    VT_CHECK(d->tap_w[t] >= 0 && d->tap_w[t] < d->w_taps, "%s: tap_w[%d] out of range", who, t);
    VT_CHECK(d->tap_phase[t] >= 0 && d->tap_phase[t] < d->n_phase, "%s: tap_phase[%d] out of range", who, t);
  }
  VT_CHECK(d->act >= 0 && d->act <= 2, "%s: bad act", who);
  if (d->noise) VT_CHECK(d->noise_w != nullptr, "%s: noise without noise_w", who);
  if (d->rgb_w) VT_CHECK(d->rgb_out && d->rgb_bias && (!d->rgb_skip || d->rgb_skip_kernel), "%s: incomplete fused ToRGB arguments", who);
  return 0;
}
int vt_validate_conv_desc(const vt_conv_desc* d, const char* who) { return validate_conv_desc(d, who); }

extern "C" int vt_conv2d_direct_f32(const vt_conv_desc* d, void* stream) {
  if (validate_conv_desc(d, "conv2d_direct")) return 1;
  VT_CHECK(d->B <= 65535 && vt_cdiv(d->Cout, BN) <= 65535, "conv2d_direct: grid too large");
  VT_CHECK(!d->rgb_w && d->out, "conv2d_direct: the fused ToRGB tail exists only in the tensor-core kernel");
  VT_CHECK(!d->src_scale[0] && !d->src_scale[1] && !d->src_affine[0] && !d->src_affine[1],
           "conv2d_direct: src_scale / src_affine are only implemented by the bf16x3 tensor-core kernel");
  const int64_t HoWo = (int64_t)d->Ho * d->Wo;
  dim3 grid((unsigned)vt_cdiv(HoWo, BM), (unsigned)vt_cdiv(d->Cout, BN), (unsigned)d->B);
  for (int ph = 0; ph < d->n_phase; ++ph) {   // one launch per output phase (weight rows ph*Cout.., view offset phase_off[ph])
    DirectArgs a;
    a.d = *d;
    a.w_rows = d->n_phase * d->Cout;
    a.w_row0 = ph * d->Cout;
    a.d.n_phase = 1;
    a.d.phase_off[0] = d->phase_off[ph];
    conv_direct_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
    VT_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int vt_smalln_conv_f32(const vt_smalln_desc* d, void* stream) {
  VT_CHECK(d != nullptr, "smalln_conv: null descriptor");
  VT_CHECK(d->struct_size == (int)sizeof(vt_smalln_desc), "smalln_conv: descriptor size mismatch (got %d, want %d)",
           d->struct_size, (int)sizeof(vt_smalln_desc));
  VT_CHECK(d->Cout >= 1 && d->Cout <= 4, "smalln_conv: Cout must be in [1,4]");
  VT_CHECK(d->B >= 1 && d->B <= 65535 && d->H >= 1 && d->W >= 1, "smalln_conv: bad shape");
  VT_CHECK(d->taps >= 1 && d->taps <= VT_MAX_TAPS, "smalln_conv: bad taps");
  VT_CHECK(d->src_c >= 0 && d->src_c % 4 == 0 && d->src_cstride % 4 == 0 && d->src_cstride >= d->src_c, "smalln_conv: src_c must be a multiple of 4");
  VT_CHECK(d->src_c == 0 || (d->src && aligned16(d->src)), "smalln_conv: bad src pointer");
  VT_CHECK(d->n_planar >= 0 && d->n_planar <= 4, "smalln_conv: n_planar must be <= 4");
  VT_CHECK(d->n_planar == 0 || (d->planar && d->planar_weight), "smalln_conv: planar source needs planar weights");
  VT_CHECK(d->src2_mode == 0 || (d->src2_mode == 1 && d->src2 && aligned16(d->src2)), "smalln_conv: bad src2 / src2_mode");
  VT_CHECK(d->wB == 1 || d->wB == d->B, "smalln_conv: wB must be 1 or B");
  VT_CHECK(d->weight || d->src_c == 0, "smalln_conv: null weight");
  VT_CHECK(d->act == VT_ACT_NONE || d->act == VT_ACT_RELU_TANH, "smalln_conv: bad act");
  VT_CHECK(d->out != nullptr, "smalln_conv: null out");
  VT_CHECK(!d->tsum || d->tsum_c >= d->taps * d->Cout, "smalln_conv: tsum_c must hold taps*Cout partial products");
  VT_CHECK(!d->src_mask || !d->src2_mode, "smalln_conv: src_mask cannot be combined with the virtual concat");
  if (d->skip) VT_CHECK(d->skip_kernel && d->H % 2 == 0 && d->W % 2 == 0, "smalln_conv: skip needs a 4x4 kernel and even H, W");
  if (d->mul_out) VT_CHECK(d->mul_src && d->mul_c % 4 == 0 && aligned16(d->mul_src) && aligned16(d->mul_out), "smalln_conv: bad mul_out args");
  for (int t = 0; t < d->taps; ++t) VT_CHECK(d->tap_w[t] >= 0 && d->tap_w[t] < d->w_taps, "smalln_conv: tap_w out of range");

  SmallNArgs a;
  a.d = *d;
  const int cw = d->src2_mode ? 2 * d->src_c : d->src_c;
  VT_CHECK(d->src_c == 0 || d->w_cstride >= cw, "smalln_conv: weight row shorter than the (virtual-concat) channel count");
  cudaStream_t st = (cudaStream_t)stream;
  // input-stationary kernel for 9-tap convolutions whose taps stay within +-2 pixels
  // (chosen automatically for Cout == 1 on maps of >= 64 patches only)
  const bool is_auto = d->Cout == 1 && vt_cdiv(d->W, IS_PW) * vt_cdiv(d->H, IS_PH) >= 64;   // per image: the choice must not depend on the batch size (frames are independent units)
  if ((g_smalln_is == 2 || (g_smalln_is == 1 && is_auto)) && d->taps == IS_TAPS && d->src_c >= 32) {
    int dy0 = 0, dy1 = 0, dx0 = 0, dx1 = 0;
    for (int t = 0; t < d->taps; ++t) {
      dy0 = d->tap_dy[t] < dy0 ? d->tap_dy[t] : dy0; dy1 = d->tap_dy[t] > dy1 ? d->tap_dy[t] : dy1;
      dx0 = d->tap_dx[t] < dx0 ? d->tap_dx[t] : dx0; dx1 = d->tap_dx[t] > dx1 ? d->tap_dx[t] : dx1;
    }
    const int tn = IS_TAPS * d->Cout;
    const int TS = tn | 1;   // odd pixel stride in Ts: conflict-free column-wise reads
    const int RH = IS_PH + dy1 - dy0, RW = IS_PW + dx1 - dx0;
    const size_t smem_is = ((size_t)tn * (cw + d->n_planar) + 16 + ((tn + 3) & ~3) + (size_t)RH * RW * TS) * sizeof(float);
    if (dy1 - dy0 <= 4 && dx1 - dx0 <= 4 && smem_is <= 200 * 1024) {
      const int64_t patches = vt_cdiv(d->W, IS_PW) * vt_cdiv(d->H, IS_PH);
      // persistent over patches: exactly one wave of resident blocks (a 1.5-wave grid ran its second half on half the slots)
#define VT_LAUNCH_IS(NN, ITT)                                                                                          \
  do {                                                                                                                 \
    if (smem_is > 48 * 1024)                                                                                           \
      VT_CUDA(cudaFuncSetAttribute(smalln_is_kernel<NN, ITT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_is)); \
    int occ = 0;                                                                                                       \
    VT_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, smalln_is_kernel<NN, ITT>, 256, smem_is));             \
    int64_t blocks = ((int64_t)vt_num_sms() * (occ > 0 ? occ : 1)) / d->B;                                             \
    if (blocks < 1) blocks = 1;                                                                                        \
    if (blocks > patches) blocks = patches;                                                                            \
    dim3 grid((unsigned)blocks, (unsigned)d->B);                                                                       \
    smalln_is_kernel<NN, ITT><<<grid, 256, smem_is, st>>>(a, dy0, dy1, dx0, dx1, TS);                                    \
  } while (0)
      switch (d->Cout) {
        case 1: VT_LAUNCH_IS(1, 4); break;
        case 2: VT_LAUNCH_IS(2, 2); break;
        case 3: VT_LAUNCH_IS(3, 2); break;
        default: VT_LAUNCH_IS(4, 1); break;
      }
#undef VT_LAUNCH_IS
      VT_LAUNCH_CHECK();
      return 0;
    }
  }
  const size_t smem = ((size_t)d->taps * d->Cout * (cw + d->n_planar + 1) + 16) * sizeof(float);
  VT_CHECK(smem <= 200 * 1024, "smalln_conv: weights (%zu B) do not fit in shared memory", smem);
  const int64_t HW = (int64_t)d->H * d->W;
  int64_t blocks = vt_cdiv(d->W, 32) * vt_cdiv(d->H, 8);
  const int64_t cap = (int64_t)vt_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  dim3 grid((unsigned)blocks, (unsigned)d->B);
#define VT_LAUNCH_SMALLN(NN)                                                                                   \
  do {                                                                                                         \
    if (smem > 48 * 1024)                                                                                      \
      VT_CUDA(cudaFuncSetAttribute(smalln_conv_kernel<NN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    smalln_conv_kernel<NN><<<grid, 256, smem, st>>>(a);                                                        \
  } while (0)
  switch (d->Cout) {
    case 1: VT_LAUNCH_SMALLN(1); break;
    case 2: VT_LAUNCH_SMALLN(2); break;
    case 3: VT_LAUNCH_SMALLN(3); break;
    default: VT_LAUNCH_SMALLN(4); break;
  }
#undef VT_LAUNCH_SMALLN
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_affine_fold_weights_f32(const float* w, const float* stats, const float* gamma_beta, float* out_w, float* out_k,
                                          int B, int taps_n, int C2, void* stream) {
  VT_CHECK(w && stats && gamma_beta && out_w && out_k && B >= 1 && B <= 65535 && taps_n >= 1 && C2 >= 1, "affine_fold_weights: bad args");
  dim3 grid((unsigned)taps_n, (unsigned)B);
  affine_fold_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, stats, gamma_beta, out_w, out_k, C2);
  VT_LAUNCH_CHECK();
  return 0;
}
