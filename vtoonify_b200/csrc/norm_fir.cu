// norm_fir.cu — instance-norm statistics, AdaIN apply, and the NHWC FIR (Blur) with fused StyledConv epilogue.
//
//   vt_instnorm_stats_nhwc / vt_adain_apply_nhwc : AdaptiveInstanceNorm.forward (model/dualstylegan.py:16-21):
//        nn.InstanceNorm2d(affine=False) = (x - mean) / sqrt(biased_var + 1e-5) per (b, c) plane, then gamma*x + beta.
//        mode 1 evaluates the virtual concat cat(f_G, |f_G - f_E|) of Fusion.forward (model/vtoonify.py:125-126)
//        without materialising it for the statistics pass.
//   vt_fir_nhwc_f32 : Blur.forward after the stride-2 transposed conv (model/stylegan/model.py:74-90,285) =
//        upfirdn2d(x, k, pad=(p0,p1)) with up=down=1, on NHWC, with NoiseInjection + FusedLeakyReLU
//        (model/stylegan/model.py:315-320,364-370) applied in the same pass. Each thread owns 4 channels (float4)
//        of a 1 x 4 vertical strip of outputs so every input row is loaded once per strip.
#include "common.cuh"

int g_fir4 = 1;   // 1: specialised 4x4 pad (1,1) FIR kernel; 0: generic kernel (tests / A-B)

namespace {

// Chan's merge of a group of nk values with sum sk and squared deviations m2k about their own mean into (n, s, m2):
// n*nk/(n+nk) * (mean_k - mean)^2 written with sums.  Groups are combined this way or, in the finalize, about the known plane mean, so no
// sum of squares about zero is ever formed: its rounding (u * E[x^2]) would swamp the variance of an offset plane.  An empty
// group (nk = 0, sk = m2k = 0) changes nothing.
__device__ __forceinline__ void chan_merge(double& n, double& s, double& m2, double nk, double sk, double m2k) {
  const double t = nk * s - n * sk;
  const float den = (float)(n * nk * (n + nk));
  m2 += (den > 0.f ? t * t * (double)__frcp_rn(den) : 0.0) + m2k;   // a positive term: fp32 reciprocal accuracy is plenty
  s += sk; n += nk;
}

// One thread's running statistics of one channel, about a pivot k (the thread's first value): s = sum of (x - k), m2 = squared
// deviations from the running mean.  Pixels arrive in blocks (a trip of 8 pixels, or the tail pixels) that accumulate
// (sum, sum of squares) of x - kb, kb = the block's first value: 3 flops per value, and the cancellation in the block's
// M2 = q - s^2 / nb stays within a factor of the block length (8).  Blocks are merged with Chan's update.
struct RunStat { float k, s, m2; };

// Weights of merging a block of nb values after n: 1/nb, 1/n (0 for the first block) and n nb / (n + nb); shared by the channels.
struct MergeW { float inv_nb, inv_n, w; };

__device__ __forceinline__ MergeW merge_weights(float n, float nb) {
  return MergeW{__frcp_rn(nb), n > 0.f ? __frcp_rn(n) : 0.f, n * nb * __frcp_rn(n + nb)};
}

// merge a block of nb values (deviation sum bs and square sum bq about its pivot kb) into r; the first block sets the pivot
__device__ __forceinline__ void run_merge(RunStat& r, float kb, float bs, float bq, float nb, const MergeW& mw) {
  if (mw.inv_n == 0.f) r.k = kb;
  const float m2b = fmaxf(fmaf(-bs, bs * mw.inv_nb, bq), 0.f);
  const float sb = fmaf(nb, kb - r.k, bs);                      // the block's deviation sum about r.k
  const float delta = sb * mw.inv_nb - r.s * mw.inv_n;
  r.m2 = fmaf(delta * mw.w, delta, r.m2 + m2b);
  r.s += sb;
}

// Deterministic two-stage reduction (no atomics) into the layout of vt_instnorm_finalize_f32: stage 1, grid (chunks, B): every
// thread owns one float4 channel group and every pstep-th pixel of its chunk; the pixel lanes' (pivot, deviation sum, M2) are
// merged in lane order through shared memory (Chan, double) into the chunk's entry, and block (chunk, 0) writes the chunk's
// pixel count.  Stage 2 merges the chunks (instnorm_finalize_kernel).  dyn smem: pstep * Cs * 3 floats.
template <int mode>
__global__ void __launch_bounds__(256)
instnorm_partial_kernel(const float* __restrict__ in, const float* __restrict__ in2, int64_t HW, int C, int c_stride, int64_t chunk,
                        float* __restrict__ ws) {
  extern __shared__ float sacc[];  // [pstep][Cs][3]
  const int Cs = mode ? 2 * C : C;
  const int b = blockIdx.y;
  const int nvec = C / 4;
  const int64_t p_begin = (int64_t)blockIdx.x * chunk;
  const int64_t p_end = (p_begin + chunk < HW) ? p_begin + chunk : HW;
  const float* ip = in + (int64_t)b * HW * c_stride;
  const float* ip2 = mode ? in2 + (int64_t)b * HW * c_stride : nullptr;
  const int pstep = blockDim.x / nvec;           // >= 1 (nvec <= 256 checked by the host)
  const int v = threadIdx.x % nvec, lane_p = threadIdx.x / nvec;
  if (lane_p < pstep) {
    RunStat r[4], r2[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) r[i] = r2[i] = RunStat{0.f, 0.f, 0.f};
    float n = 0.f;   // pixels merged so far (exact: < 2^24 per thread)
    int64_t p = p_begin + lane_p;
    // eight pixels per trip, one block: the loads are issued together (the kernel is latency-bound: one 16-byte load in flight
    // per thread gave 1.2 TB/s on L2-resident maps), the accumulation order stays the pixel order
    for (; p + 7 * (int64_t)pstep < p_end; p += 8 * (int64_t)pstep) {
      float4 a[8], e[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] = __ldg(reinterpret_cast<const float4*>(ip + (p + u * (int64_t)pstep) * c_stride + v * 4));
      if (mode) {
#pragma unroll
        for (int u = 0; u < 8; ++u) e[u] = __ldg(reinterpret_cast<const float4*>(ip2 + (p + u * (int64_t)pstep) * c_stride + v * 4));
      }
      const float kb[4] = {a[0].x, a[0].y, a[0].z, a[0].w};
      float kb2[4], bs[4] = {0, 0, 0, 0}, bq[4] = {0, 0, 0, 0}, bs2[4] = {0, 0, 0, 0}, bq2[4] = {0, 0, 0, 0};
      if (mode) {
        kb2[0] = fabsf(a[0].x - e[0].x); kb2[1] = fabsf(a[0].y - e[0].y); kb2[2] = fabsf(a[0].z - e[0].z); kb2[3] = fabsf(a[0].w - e[0].w);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float av[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float d = av[i] - kb[i]; bs[i] += d; bq[i] = fmaf(d, d, bq[i]); }
        if (mode) {
          const float ev[4] = {e[u].x, e[u].y, e[u].z, e[u].w};
#pragma unroll
          for (int i = 0; i < 4; ++i) { const float d = fabsf(av[i] - ev[i]) - kb2[i]; bs2[i] += d; bq2[i] = fmaf(d, d, bq2[i]); }
        }
      }
      const MergeW mw = merge_weights(n, 8.f);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        run_merge(r[i], kb[i], bs[i], bq[i], 8.f, mw);
        if (mode) run_merge(r2[i], kb2[i], bs2[i], bq2[i], 8.f, mw);
      }
      n += 8.f;
    }
    if (p < p_end) {   // the tail: fewer than 8 pixels of this lane left, one block
      float kb[4], kb2[4], bs[4] = {0, 0, 0, 0}, bq[4] = {0, 0, 0, 0}, bs2[4] = {0, 0, 0, 0}, bq2[4] = {0, 0, 0, 0};
      float nb = 0.f;
      for (; p < p_end; p += pstep) {
        const float4 a = *reinterpret_cast<const float4*>(ip + p * c_stride + v * 4);
        const float av[4] = {a.x, a.y, a.z, a.w};
        float ev[4] = {0, 0, 0, 0};
        if (mode) {
          const float4 e = *reinterpret_cast<const float4*>(ip2 + p * c_stride + v * 4);
          ev[0] = fabsf(a.x - e.x); ev[1] = fabsf(a.y - e.y); ev[2] = fabsf(a.z - e.z); ev[3] = fabsf(a.w - e.w);
        }
        if (nb == 0.f) {
#pragma unroll
          for (int i = 0; i < 4; ++i) { kb[i] = av[i]; kb2[i] = ev[i]; }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float d = av[i] - kb[i]; bs[i] += d; bq[i] = fmaf(d, d, bq[i]);
          if (mode) { const float d2 = ev[i] - kb2[i]; bs2[i] += d2; bq2[i] = fmaf(d2, d2, bq2[i]); }
        }
        nb += 1.f;
      }
      const MergeW mw = merge_weights(n, nb);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        run_merge(r[i], kb[i], bs[i], bq[i], nb, mw);
        if (mode) run_merge(r2[i], kb2[i], bs2[i], bq2[i], nb, mw);
      }
      n += nb;
    }
    float* row = sacc + (size_t)lane_p * Cs * 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float* e = row + (v * 4 + i) * 3;
      e[0] = r[i].k; e[1] = r[i].s; e[2] = r[i].m2;
      if (mode) {
        e = row + (C + v * 4 + i) * 3;
        e[0] = r2[i].k; e[1] = r2[i].s; e[2] = r2[i].m2;
      }
    }
  }
  __syncthreads();
  const int span = (int)(p_end - p_begin);   // < 2^24 (host check)
  const int64_t E = (int64_t)gridDim.x * gridDim.y * Cs, e0 = ((int64_t)blockIdx.x * gridDim.y + b) * Cs;
  for (int i = threadIdx.x; i < Cs; i += blockDim.x) {
    double n = 0.0, s = 0.0, m2 = 0.0;
    for (int l = 0; l < pstep && l < span; ++l) {   // lane l holds pixels p_begin + l, + pstep, ... of the chunk
      const float* e = sacc + ((size_t)l * Cs + i) * 3;
      const double nl = (double)((unsigned)(span - l + pstep - 1) / (unsigned)pstep);
      chan_merge(n, s, m2, nl, nl * e[0] + e[1], e[2]);
    }
    // pivot on the chunk mean rounded to fp32: the deviation sum keeps the rest of the mean, and the square sum about the pivot
    // is M2 plus a term of the size of that rounding
    const float k0 = (float)(s / n);
    const double dev = s - n * k0;
    ws[e0 + i] = k0;
    ws[E + e0 + i] = (float)dev;
    ws[2 * E + e0 + i] = (float)(m2 + dev * dev / n);
  }
  if (b == 0 && threadIdx.x == 0) reinterpret_cast<int*>(ws + 3 * E)[blockIdx.x] = span;
}

// block = 8 (b, c) entries x 32 chunk slices, two passes over the chunks (fixed order -> deterministic): slice ks adds the pixel
// counts and sums of chunks ks, ks + 32, ... in double, the 32 slice results are added in slice order into the plane mean; then
// slice ks adds each chunk's squared deviations from that mean, q_k + 2 (k - mean) d_k + n_k (k - mean)^2 for the chunk's pivot k,
// deviation sum d_k and square sum q_k about k, the same way.  Every addend of a pass is independent of the others
// (a Chan merge per chunk would chain a dozen dependent operations per step), so the loads stay in flight.  One thread per
// entry walking all chunks was a 140-step dependent chain of strided loads (57 us per call on the 72x128 maps once the
// partial kernel went to 144 chunks).
constexpr int FIN_ENTRIES = 8, FIN_SLICES = 32;   // 256 threads; more slices keep more SMs busy on few (b, c) entries

__global__ void __launch_bounds__(256)
instnorm_finalize_kernel(const float* __restrict__ ws, float* __restrict__ stats, int n, int chunks, double inv_hw, float eps) {
  __shared__ double red[3][FIN_SLICES][FIN_ENTRIES];
  const int li = threadIdx.x % FIN_ENTRIES, ks = threadIdx.x / FIN_ENTRIES;
  const int i = blockIdx.x * FIN_ENTRIES + li;   // i = b * Cs + c
  const int64_t E = (int64_t)chunks * n;
  const int* cnt = reinterpret_cast<const int*>(ws + 3 * E);
  double c = 0.0, s = 0.0;
  if (i < n) {
#pragma unroll 4
    for (int k = ks; k < chunks; k += FIN_SLICES) {
      const double ck = (double)__ldg(cnt + k);
      const int64_t j = (int64_t)k * n + i;
      c += ck;
      s += ck * __ldg(ws + j) + __ldg(ws + E + j);
    }
  }
  red[0][ks][li] = c; red[1][ks][li] = s;
  __syncthreads();
  double cc = 0.0, ss = 0.0;
#pragma unroll
  for (int k = 0; k < FIN_SLICES; ++k) { cc += red[0][k][li]; ss += red[1][k][li]; }
  const double mean = cc > 0.0 ? ss / cc : 0.0;
  double q = 0.0;
  if (i < n) {
#pragma unroll 4
    for (int k = ks; k < chunks; k += FIN_SLICES) {
      const double ck = (double)__ldg(cnt + k);
      const int64_t j = (int64_t)k * n + i;
      const double a = (double)__ldg(ws + j) - mean;   // a chunk of no pixels has all partials 0 and adds 0
      q += __ldg(ws + 2 * E + j) + a * (2.0 * __ldg(ws + E + j) + ck * a);
    }
  }
  red[2][ks][li] = q;
  __syncthreads();
  if (ks == 0 && i < n) {
    double qq = 0.0;
#pragma unroll
    for (int k = 0; k < FIN_SLICES; ++k) qq += red[2][k][li];
    stats[i * 2] = (float)(ss * inv_hw);
    stats[i * 2 + 1] = (float)(1.0 / sqrt(fmax(qq, 0.0) * inv_hw + (double)eps));
  }
}

// one thread per (pixel, float4 of the OUTPUT channels Cs)
__global__ void __launch_bounds__(256)
adain_apply_kernel(const float* __restrict__ in, const float* __restrict__ in2, int mode, int64_t HW, int C, int c_stride,
                   const float* __restrict__ stats, const float* __restrict__ gb, float* __restrict__ out, int round_tf32) {
  const int Cs = mode ? 2 * C : C;
  const int nvec = Cs / 4;
  const int b = blockIdx.y;
  const int64_t total = HW * nvec;
  const float* st = stats + (int64_t)b * Cs * 2;
  const float* gamma = gb + (int64_t)b * 2 * Cs;
  const float* beta = gamma + Cs;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / nvec;
    const int c = (int)(i % nvec) * 4;
    float x[4];
    if (!mode || c < C) {
      const float4 a = *reinterpret_cast<const float4*>(in + ((int64_t)b * HW + p) * c_stride + c);
      x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
    } else {
      const float4 a = *reinterpret_cast<const float4*>(in + ((int64_t)b * HW + p) * c_stride + (c - C));
      const float4 e = *reinterpret_cast<const float4*>(in2 + ((int64_t)b * HW + p) * c_stride + (c - C));
      x[0] = fabsf(a.x - e.x); x[1] = fabsf(a.y - e.y); x[2] = fabsf(a.z - e.z); x[3] = fabsf(a.w - e.w);
    }
    float y[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xn = (x[k] - st[(c + k) * 2]) * st[(c + k) * 2 + 1];
      float v = gamma[c + k] * xn + beta[c + k];
      y[k] = round_tf32 ? vt_round_tf32(v) : v;
    }
    *reinterpret_cast<float4*>(out + ((int64_t)b * HW + p) * Cs + c) = make_float4(y[0], y[1], y[2], y[3]);
  }
}

constexpr int FIR_R = 4;      // output rows per thread
constexpr int FIR_MAXK = 8;   // max kernel extent

__global__ void __launch_bounds__(256)
fir_nhwc_kernel(const float* __restrict__ in, const float* __restrict__ kernel, float* __restrict__ out, int H, int W,
                int C, int Ho, int Wo, int kh, int kw, int pad0, const float* __restrict__ bias,
                const float* __restrict__ noise, const float* __restrict__ noise_w, int act, float slope, float gain,
                int round_tf32) {
  __shared__ float sk[FIR_MAXK * FIR_MAXK];  // flipped kernel: sk[ky][kx] multiplies in[oy+ky-pad0][ox+kx-pad0]
  if (threadIdx.x < kh * kw) {
    const int ky = threadIdx.x / kw, kx = threadIdx.x % kw;
    sk[threadIdx.x] = kernel[(kh - 1 - ky) * kw + (kw - 1 - kx)];
  }
  __syncthreads();
  const int nvec = C / 4;
  const int b = blockIdx.z;
  const int strips = (Ho + FIR_R - 1) / FIR_R;
  const int64_t total = (int64_t)strips * Wo * nvec;
  const float nw = noise ? *noise_w : 0.f;
  const float* ip = in + (int64_t)b * H * W * C;
  float* op = out + (int64_t)b * Ho * Wo * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    const int64_t r = i / nvec;
    const int ox = (int)(r % Wo);
    const int oy0 = (int)(r / Wo) * FIR_R;
    float4 acc[FIR_R];
#pragma unroll
    for (int j = 0; j < FIR_R; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    // input rows oy0 - pad0 .. oy0 + FIR_R - 1 + kh - 1 - pad0
    for (int ry = 0; ry < FIR_R + kh - 1; ++ry) {
      const int iy = oy0 - pad0 + ry;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < kw; ++kx) {
        const int ix = ox - pad0 + kx;
        if (ix < 0 || ix >= W) continue;
        const float4 a = *reinterpret_cast<const float4*>(ip + ((int64_t)iy * W + ix) * C + v * 4);
#pragma unroll
        for (int j = 0; j < FIR_R; ++j) {
          const int ky = ry - j;
          if (ky >= 0 && ky < kh) {
            const float w = sk[ky * kw + kx];
            acc[j].x = fmaf(a.x, w, acc[j].x); acc[j].y = fmaf(a.y, w, acc[j].y);
            acc[j].z = fmaf(a.z, w, acc[j].z); acc[j].w = fmaf(a.w, w, acc[j].w);
          }
        }
      }
    }
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias) bv = *reinterpret_cast<const float4*>(bias + v * 4);
#pragma unroll
    for (int j = 0; j < FIR_R; ++j) {
      const int oy = oy0 + j;
      if (oy >= Ho) break;
      float o[4] = {acc[j].x, acc[j].y, acc[j].z, acc[j].w};
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
      const float nz = noise ? nw * noise[((int64_t)b * Ho + oy) * Wo + ox] : 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float t = o[k];
        if (noise) t += nz;
        if (act) t = vt_lrelu(t + bb[k], slope) * gain;
        else if (bias) t += bb[k];
        o[k] = round_tf32 ? vt_round_tf32(t) : t;
      }
      *reinterpret_cast<float4*>(op + ((int64_t)oy * Wo + ox) * C + v * 4) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

// 4x4 FIR, pad (1,1) (the Blur after a stride-2 transposed conv, model/stylegan/model.py:284-285): a thread owns 2 adjacent
// output columns x FIR4_R rows of one 4-channel group.  Per input row it issues 5 independent 16-byte loads (clamped address +
// zero mask, no branches), so 3.4 loads per output instead of 7 and all of them in flight together.
constexpr int FIR4_R = 8;

__global__ void __launch_bounds__(256)
fir4_nhwc_kernel(const float* __restrict__ in, const float* __restrict__ kernel, float* __restrict__ out, int H, int W,
                 int C, int Ho, int Wo, const float* __restrict__ bias, const float* __restrict__ noise,
                 const float* __restrict__ noise_w, int act, float slope, float gain, int round_tf32) {
  __shared__ float sk[16];  // flipped kernel: sk[ky][kx] multiplies in[oy+ky-1][ox+kx-1]
  if (threadIdx.x < 16) sk[threadIdx.x] = kernel[(3 - threadIdx.x / 4) * 4 + (3 - threadIdx.x % 4)];
  __syncthreads();
  float kk[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) kk[i] = sk[i];
  const int nvec = C / 4;
  const int b = blockIdx.z;
  const int strips = (Ho + FIR4_R - 1) / FIR4_R, pairs = (Wo + 1) / 2;
  const int64_t total = (int64_t)strips * pairs * nvec;
  const float nw = noise ? *noise_w : 0.f;
  const float* ip = in + (int64_t)b * H * W * C;
  float* op = out + (int64_t)b * Ho * Wo * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    const int64_t r = i / nvec;
    const int ox0 = (int)(r % pairs) * 2;
    const int oy0 = (int)(r / pairs) * FIR4_R;
    float4 acc[FIR4_R][2];
#pragma unroll
    for (int j = 0; j < FIR4_R; ++j) acc[j][0] = acc[j][1] = make_float4(0.f, 0.f, 0.f, 0.f);
    int cx[5];
    float mx[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int ix = ox0 - 1 + k;
      mx[k] = (ix >= 0 && ix < W) ? 1.f : 0.f;
      cx[k] = ix < 0 ? 0 : (ix >= W ? W - 1 : ix);
    }
#pragma unroll
    for (int ry = 0; ry < FIR4_R + 3; ++ry) {
      const int iy = oy0 - 1 + ry;
      const float my = (iy >= 0 && iy < H) ? 1.f : 0.f;
      const int cy = iy < 0 ? 0 : (iy >= H ? H - 1 : iy);
      const float* rowp = ip + (int64_t)cy * W * C + v * 4;
      float4 a[5];
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        a[k] = __ldg(reinterpret_cast<const float4*>(rowp + (int64_t)cx[k] * C));
        const float m = my * mx[k];
        a[k].x *= m; a[k].y *= m; a[k].z *= m; a[k].w *= m;
      }
#pragma unroll
      for (int j = 0; j < FIR4_R; ++j) {
        const int ky = ry - j;
        if (ky >= 0 && ky < 4) {
#pragma unroll
          for (int o = 0; o < 2; ++o)
#pragma unroll
            for (int kx = 0; kx < 4; ++kx) {
              const float w = kk[ky * 4 + kx];
              acc[j][o].x = fmaf(a[o + kx].x, w, acc[j][o].x); acc[j][o].y = fmaf(a[o + kx].y, w, acc[j][o].y);
              acc[j][o].z = fmaf(a[o + kx].z, w, acc[j][o].z); acc[j][o].w = fmaf(a[o + kx].w, w, acc[j][o].w);
            }
        }
      }
    }
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias) bv = *reinterpret_cast<const float4*>(bias + v * 4);
    const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
    for (int j = 0; j < FIR4_R; ++j) {
      const int oy = oy0 + j;
      if (oy >= Ho) break;
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        const int ox = ox0 + o;
        if (ox >= Wo) continue;
        float t4[4] = {acc[j][o].x, acc[j][o].y, acc[j][o].z, acc[j][o].w};
        const float nz = noise ? nw * noise[((int64_t)b * Ho + oy) * Wo + ox] : 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float t = t4[k];
          if (noise) t += nz;
          if (act) t = vt_lrelu(t + bb[k], slope) * gain;
          else if (bias) t += bb[k];
          t4[k] = round_tf32 ? vt_round_tf32(t) : t;
        }
        *reinterpret_cast<float4*>(op + ((int64_t)oy * Wo + ox) * C + v * 4) = make_float4(t4[0], t4[1], t4[2], t4[3]);
      }
    }
  }
}

}  // namespace

int g_instnorm_chunks = 296;   // target number of chunks per sample on large maps (0: always the small chunks)

static void instnorm_plan(int64_t HW, int C, int64_t* chunk, int64_t* chunks) {
  const int nvec = C / 4;
  const int plan = 256 / nvec;                      // pixels processed concurrently by a block
  int64_t ch = (int64_t)plan * 32;                  // 32 pixels per thread: several blocks per SM even on the 72x128 maps
  if (ch < 64) ch = 64;
  // Large maps: ~2 chunks per SM and sample instead of thousands of 8-trip blocks.  The partial pass itself is already
  // HBM-bound (ncu, [4,128,576,1024] x 2 sources: 2.42 GB in 344 us = 86 % DRAM throughput); what shrinks is the partial-sum
  // buffer and with it the finalize pass (2304 -> 296 chunks per entry).  The plan depends on (HW, C) only, never on the batch
  // size: a frame's statistics must not depend on the batch it travels in.
  if (g_instnorm_chunks > 0) {
    const int64_t unit = (int64_t)plan * 4;         // one trip of the main loop
    const int64_t want = vt_cdiv(vt_cdiv(HW, g_instnorm_chunks), unit) * unit;
    if (want > ch) ch = want;
  }
  *chunk = ch;
  *chunks = vt_cdiv(HW, ch);
}

extern "C" int64_t vt_instnorm_partials_floats(int64_t chunks, int B, int Cs) {
  if (chunks < 1 || B < 1 || Cs < 1) return -1;
  return chunks * ((int64_t)B * Cs * 3 + 1);
}

extern "C" int64_t vt_instnorm_ws_bytes(int B, int64_t HW, int C, int mode) {
  if (B < 1 || HW < 1 || C < 4 || C % 4 || C / 4 > 256) return -1;
  int64_t chunk, chunks;
  instnorm_plan(HW, C, &chunk, &chunks);
  return vt_instnorm_partials_floats(chunks, B, mode ? 2 * C : C) * (int64_t)sizeof(float);
}

extern "C" int vt_instnorm_stats_nhwc(const float* in, const float* in2, int mode, int B, int64_t HW, int C, int c_stride,
                                      float eps, float* stats, void* ws, void* stream) {
  VT_CHECK(in && stats && ws && (mode == 0 || (mode == 1 && in2)), "instnorm_stats: bad pointers/mode");
  VT_CHECK(B >= 1 && B <= 65535 && HW >= 1 && C >= 4 && C % 4 == 0 && c_stride >= C && c_stride % 4 == 0, "instnorm_stats: bad shape");
  VT_CHECK(C / 4 <= 256, "instnorm_stats: C must be <= 1024");
  const int Cs = mode ? 2 * C : C;
  cudaStream_t st = (cudaStream_t)stream;
  int64_t chunk, chunks;
  instnorm_plan(HW, C, &chunk, &chunks);
  VT_CHECK(chunk < (1LL << 24) && chunks < (1LL << 31), "instnorm_stats: plane too large (%lld pixels)", (long long)HW);
  const int pstep = 256 / (C / 4);
  dim3 grid((unsigned)chunks, (unsigned)B);
  const size_t smem = (size_t)pstep * Cs * 3 * sizeof(float);
  if (mode) instnorm_partial_kernel<1><<<grid, 256, smem, st>>>(in, in2, HW, C, c_stride, chunk, (float*)ws);
  else instnorm_partial_kernel<0><<<grid, 256, smem, st>>>(in, in2, HW, C, c_stride, chunk, (float*)ws);
  VT_LAUNCH_CHECK();
  const int n = B * Cs;
  instnorm_finalize_kernel<<<(unsigned)vt_cdiv(n, FIN_ENTRIES), 256, 0, st>>>((const float*)ws, stats, n, (int)chunks,
                                                                    1.0 / (double)HW, eps);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_instnorm_finalize_f32(const float* ws, float* stats, int B, int Cs, int chunks, int64_t HW, float eps, void* stream) {
  VT_CHECK(ws && stats && B >= 1 && Cs >= 1 && chunks >= 1 && HW >= 1, "instnorm_finalize: bad args");
  const int n = B * Cs;
  instnorm_finalize_kernel<<<(unsigned)vt_cdiv(n, FIN_ENTRIES), 256, 0, (cudaStream_t)stream>>>(ws, stats, n, chunks, 1.0 / (double)HW, eps);
  VT_LAUNCH_CHECK();
  return 0;
}

__global__ void adain_affine_kernel(const float* __restrict__ stats, const float* __restrict__ gb, float* __restrict__ aff, int B, int Cs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;   // i = b * Cs + c
  if (i >= B * Cs) return;
  const int b = i / Cs, c = i - b * Cs;
  const float gamma = gb[(int64_t)b * 2 * Cs + c], beta = gb[(int64_t)b * 2 * Cs + Cs + c];
  const float sc = gamma * stats[i * 2 + 1];
  aff[i * 2] = sc;
  aff[i * 2 + 1] = beta - sc * stats[i * 2];
}

extern "C" int vt_adain_affine_f32(const float* stats, const float* gamma_beta, float* affine, int B, int Cs, void* stream) {
  VT_CHECK(stats && gamma_beta && affine && B >= 1 && Cs >= 1, "adain_affine: bad args");
  adain_affine_kernel<<<(unsigned)vt_cdiv((int64_t)B * Cs, 128), 128, 0, (cudaStream_t)stream>>>(stats, gamma_beta, affine, B, Cs);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_adain_apply_nhwc(const float* in, const float* in2, int mode, int B, int64_t HW, int C, int c_stride,
                                   const float* stats, const float* gamma_beta, float* out, int round_tf32, void* stream) {
  VT_CHECK(in && stats && gamma_beta && out && (mode == 0 || (mode == 1 && in2)), "adain_apply: bad pointers/mode");
  VT_CHECK(B >= 1 && B <= 65535 && HW >= 1 && C >= 4 && C % 4 == 0 && c_stride >= C && c_stride % 4 == 0, "adain_apply: bad shape");
  const int Cs = mode ? 2 * C : C;
  const int64_t total = HW * (Cs / 4);
  int64_t blocks = vt_cdiv(total, 256);
  const int64_t cap = (int64_t)vt_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  dim3 grid((unsigned)blocks, (unsigned)B);
  adain_apply_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, in2, mode, HW, C, c_stride, stats, gamma_beta, out, round_tf32);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_fir_nhwc_f32(const float* in, const float* kernel, float* out, int B, int H, int W, int C, int kh, int kw,
                               int pad0, int pad1, const float* bias, const float* noise, const float* noise_w, int act,
                               float slope, float gain, int round_tf32, void* stream) {
  VT_CHECK(in && kernel && out, "fir_nhwc: null pointer");
  VT_CHECK(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0, "fir_nhwc: bad shape (C must be a multiple of 4)");
  VT_CHECK(kh >= 1 && kw >= 1 && kh <= FIR_MAXK && kw <= FIR_MAXK, "fir_nhwc: kernel extent must be <= %d", FIR_MAXK);
  VT_CHECK(pad0 >= 0 && pad1 >= 0, "fir_nhwc: negative pad not supported on the NHWC path");
  VT_CHECK(!noise || noise_w, "fir_nhwc: noise without noise_w");
  const int Ho = H + pad0 + pad1 - kh + 1, Wo = W + pad0 + pad1 - kw + 1;
  VT_CHECK(Ho >= 1 && Wo >= 1, "fir_nhwc: empty output");
  if (kh == 4 && kw == 4 && pad0 == 1 && pad1 == 1 && g_fir4) {
    const int64_t total4 = (int64_t)vt_cdiv(Ho, FIR4_R) * vt_cdiv(Wo, 2) * (C / 4);
    int64_t blocks4 = vt_cdiv(total4, 256);
    const int64_t cap4 = (int64_t)vt_num_sms() * 16;
    if (blocks4 > cap4) blocks4 = cap4;
    fir4_nhwc_kernel<<<dim3((unsigned)blocks4, 1, (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
        in, kernel, out, H, W, C, Ho, Wo, bias, noise, noise_w, act, slope, gain, round_tf32);
    VT_LAUNCH_CHECK();
    return 0;
  }
  const int strips = (Ho + FIR_R - 1) / FIR_R;
  const int64_t total = (int64_t)strips * Wo * (C / 4);
  int64_t blocks = vt_cdiv(total, 256);
  const int64_t cap = (int64_t)vt_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  dim3 grid((unsigned)blocks, 1, (unsigned)B);
  fir_nhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, kernel, out, H, W, C, Ho, Wo, kh, kw, pad0, bias, noise,
                                                         noise_w, act, slope, gain, round_tf32);
  VT_LAUNCH_CHECK();
  return 0;
}

// ---- backward of the encoder path (VToonify.forward(return_feat=True) under autograd) -------------------------------------
//   vt_adain_grad_stats_nhwc : per (b, c) the sums of g and of g * xhat, xhat = (x - mean) * rstd with the saved statistics
//   vt_act_grad_nhwc         : out = beta * res + gate(ref) * gain * T(g), T = identity or the AdaIN backward, and optionally the
//                              per-channel sums of out (a bias gradient) in the same pass
// Both walk the maps with the chunk plan of the statistics pass (instnorm_plan: it depends on (HW, C) only) and reduce without
// atomics: every block writes double partials for its (chunk, sample), a warp per output entry adds them in a fixed order.
namespace {

// per (chunk, b, c): (sum g, sum g * xhat) in double.  dyn smem: pstep * C * 2 doubles
__global__ void __launch_bounds__(256)
adain_grad_partial_kernel(const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ stats, int64_t HW,
                          int C, int64_t chunk, double* __restrict__ ws) {
  extern __shared__ double sred[];
  const int b = blockIdx.y, nvec = C / 4, pstep = blockDim.x / nvec;
  const int v = threadIdx.x % nvec, lane_p = threadIdx.x / nvec;
  const int64_t p_begin = (int64_t)blockIdx.x * chunk;
  const int64_t p_end = (p_begin + chunk < HW) ? p_begin + chunk : HW;
  if (lane_p < pstep) {
    float mean[4], rstd[4];
    double sg[4] = {0, 0, 0, 0}, sgx[4] = {0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      mean[i] = stats[((int64_t)b * C + v * 4 + i) * 2];
      rstd[i] = stats[((int64_t)b * C + v * 4 + i) * 2 + 1];
    }
    const float* gp = g + (int64_t)b * HW * C + v * 4;
    const float* xp = x + (int64_t)b * HW * C + v * 4;
#pragma unroll 4
    for (int64_t p = p_begin + lane_p; p < p_end; p += pstep) {
      const float4 gv = __ldg(reinterpret_cast<const float4*>(gp + p * C));
      const float4 xv = __ldg(reinterpret_cast<const float4*>(xp + p * C));
      const float ga[4] = {gv.x, gv.y, gv.z, gv.w}, xa[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float xh = (xa[i] - mean[i]) * rstd[i];
        sg[i] += (double)ga[i];
        sgx[i] = fma((double)ga[i], (double)xh, sgx[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      sred[((int64_t)lane_p * C + v * 4 + i) * 2] = sg[i];
      sred[((int64_t)lane_p * C + v * 4 + i) * 2 + 1] = sgx[i];
    }
  }
  __syncthreads();
  double* dst = ws + ((int64_t)blockIdx.x * gridDim.y + b) * C * 2;
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    double s = 0.0;
    for (int l = 0; l < pstep; ++l) s += sred[(int64_t)l * C * 2 + i];
    dst[i] = s;
  }
}

// out = beta * res + gate(ref) * gain * T(g); T(g) = g, or with ADAIN gamma * rstd * ((g - m_g) - (x - mean) * rstd * m_gx)
// (m_g, m_gx = plane means of g and g * xhat).  With ws: per (chunk, b, c) the double sum of out.  dyn smem: pstep * C doubles
template <bool ADAIN>
__global__ void __launch_bounds__(256)
act_grad_kernel(const float* __restrict__ g, const float* __restrict__ ref, float slope, float gain, const float* __restrict__ res,
                float beta, const float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gb,
                const float* __restrict__ sums, float inv_hw, int64_t HW, int C, int64_t chunk, float* __restrict__ out,
                double* __restrict__ ws) {
  extern __shared__ double sred[];
  const int b = blockIdx.y, nvec = C / 4, pstep = blockDim.x / nvec;
  const int v = threadIdx.x % nvec, lane_p = threadIdx.x / nvec;
  const int64_t p_begin = (int64_t)blockIdx.x * chunk;
  const int64_t p_end = (p_begin + chunk < HW) ? p_begin + chunk : HW;
  if (lane_p < pstep) {
    float mean[4] = {0, 0, 0, 0}, rstd[4] = {0, 0, 0, 0}, coef[4] = {0, 0, 0, 0}, mg[4] = {0, 0, 0, 0}, mgx[4] = {0, 0, 0, 0};
    if (ADAIN) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t e = (int64_t)b * C + v * 4 + i;
        mean[i] = stats[e * 2];
        rstd[i] = stats[e * 2 + 1];
        coef[i] = gb[(int64_t)b * 2 * C + v * 4 + i] * rstd[i];
        mg[i] = sums[e * 2] * inv_hw;
        mgx[i] = sums[e * 2 + 1] * inv_hw;
      }
    }
    double bs[4] = {0, 0, 0, 0};
    const int64_t base = (int64_t)b * HW * C + v * 4;
    for (int64_t p = p_begin + lane_p; p < p_end; p += pstep) {
      const int64_t o = base + p * C;
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g + o));
      float t[4] = {gv.x, gv.y, gv.z, gv.w};
      if (ADAIN) {
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x + o));
        const float xa[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) t[i] = coef[i] * ((t[i] - mg[i]) - (xa[i] - mean[i]) * rstd[i] * mgx[i]);
      }
      if (ref) {
        const float4 rv = __ldg(reinterpret_cast<const float4*>(ref + o));
        const float ra[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) t[i] = ra[i] > 0.f ? t[i] : t[i] * slope;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) t[i] *= gain;
      if (res) {
        const float4 sv = __ldg(reinterpret_cast<const float4*>(res + o));
        const float sa[4] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) t[i] = fmaf(beta, sa[i], t[i]);
      }
      if (out) *reinterpret_cast<float4*>(out + o) = make_float4(t[0], t[1], t[2], t[3]);
      if (ws) {
#pragma unroll
        for (int i = 0; i < 4; ++i) bs[i] += (double)t[i];
      }
    }
    if (ws) {
#pragma unroll
      for (int i = 0; i < 4; ++i) sred[(int64_t)lane_p * C + v * 4 + i] = bs[i];
    }
  }
  if (!ws) return;
  __syncthreads();
  double* dst = ws + ((int64_t)blockIdx.x * gridDim.y + b) * C;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    double s = 0.0;
    for (int l = 0; l < pstep; ++l) s += sred[(int64_t)l * C + i];
    dst[i] = s;
  }
}

// out[e] = scale * sum over parts of ws[part * n + e], one warp per entry: lane-strided sums, then a fixed shuffle tree
__global__ void __launch_bounds__(256)
partials_sum_kernel(const double* __restrict__ ws, int64_t parts, int64_t n, float scale, float* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (e >= n) return;
  double s = 0.0;
  for (int64_t k = lane; k < parts; k += 32) s += __ldg(ws + k * n + e);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[e] = (float)(s * (double)scale);
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

extern "C" int64_t vt_act_grad_ws_bytes(int B, int64_t HW, int C) {
  if (B < 1 || HW < 1 || C < 4 || C % 4 || C / 4 > 256) return -1;
  int64_t chunk, chunks;
  instnorm_plan(HW, C, &chunk, &chunks);
  return chunks * B * C * 2 * (int64_t)sizeof(double);
}

#define VT_GRAD_SHAPE_CHECK(name)                                                                                      \
  VT_CHECK(B >= 1 && B <= 65535 && HW >= 1 && C >= 4 && C % 4 == 0 && C / 4 <= 256, name ": bad shape (C must be a "   \
           "multiple of 4, at most 1024)")

extern "C" int vt_adain_grad_stats_nhwc(const float* g, const float* x, const float* stats, int B, int64_t HW, int C,
                                        float* sums, void* ws, void* stream) {
  VT_CHECK(g && x && stats && sums && ws, "adain_grad_stats: null pointer");
  VT_CHECK(aligned16(g) && aligned16(x) && aligned16(ws), "adain_grad_stats: g, x and ws must be 16-byte aligned");
  VT_GRAD_SHAPE_CHECK("adain_grad_stats");
  int64_t chunk, chunks;
  instnorm_plan(HW, C, &chunk, &chunks);
  VT_CHECK(chunks < (1LL << 31), "adain_grad_stats: plane too large");
  cudaStream_t st = (cudaStream_t)stream;
  const int pstep = 256 / (C / 4);
  adain_grad_partial_kernel<<<dim3((unsigned)chunks, (unsigned)B), 256, (size_t)pstep * C * 2 * sizeof(double), st>>>(
      g, x, stats, HW, C, chunk, (double*)ws);
  VT_LAUNCH_CHECK();
  const int64_t n = (int64_t)B * C * 2;
  partials_sum_kernel<<<(unsigned)vt_cdiv(n, 8), 256, 0, st>>>((const double*)ws, chunks, n, 1.f, sums);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_act_grad_nhwc(const float* g, const float* ref, float slope, float gain, const float* res, float beta,
                                const float* x, const float* stats, const float* gamma_beta, const float* sums, int B, int64_t HW,
                                int C, float* out, float* bias_grad, void* ws, void* stream) {
  VT_CHECK(g && (out || bias_grad), "act_grad: null pointer (out may be NULL only with bias_grad)");
  const bool adain = x != nullptr;
  VT_CHECK(!adain || (stats && gamma_beta && sums), "act_grad: the AdaIN form needs x, stats, gamma_beta and sums");
  VT_CHECK(!bias_grad || ws, "act_grad: bias_grad needs ws");
  VT_CHECK(aligned16(g) && (!out || aligned16(out)) && (!ref || aligned16(ref)) && (!res || aligned16(res)) && (!x || aligned16(x)) &&
           (!ws || aligned16(ws)), "act_grad: tensors must be 16-byte aligned");
  VT_GRAD_SHAPE_CHECK("act_grad");
  int64_t chunk, chunks;
  instnorm_plan(HW, C, &chunk, &chunks);
  VT_CHECK(chunks < (1LL << 31), "act_grad: plane too large");
  cudaStream_t st = (cudaStream_t)stream;
  const int pstep = 256 / (C / 4);
  double* part = bias_grad ? (double*)ws : nullptr;
  const size_t smem = part ? (size_t)pstep * C * sizeof(double) : 0;
  const dim3 grid((unsigned)chunks, (unsigned)B);
  const float inv_hw = (float)(1.0 / (double)HW);
  if (adain)
    act_grad_kernel<true><<<grid, 256, smem, st>>>(g, ref, slope, gain, res, beta, x, stats, gamma_beta, sums, inv_hw, HW, C,
                                                   chunk, out, part);
  else
    act_grad_kernel<false><<<grid, 256, smem, st>>>(g, ref, slope, gain, res, beta, x, stats, gamma_beta, sums, inv_hw, HW, C,
                                                    chunk, out, part);
  VT_LAUNCH_CHECK();
  if (bias_grad) {
    partials_sum_kernel<<<(unsigned)vt_cdiv(C, 8), 256, 0, st>>>(part, chunks * B, C, 1.f, bias_grad);
    VT_LAUNCH_CHECK();
  }
  return 0;
}

// ---- backward of the generator tail of VToonify.forward (the G step of both training scripts) -----------------------------------
//   vt_torgb_gate_grad_nhwc         : StyledConv gate with the ToRGB adjoint folded in, out = gate(ref) * gain * (g + w_rgb^T g_rgb)
//   vt_fusion_mask_grad_nhwc        : g_z of the mask head m = tanh(relu z), and conv2's bias gradient
//   vt_fusion_adain_grad_stats_nhwc : the AdaIN-backward sums over cat(f_G, |f_G - f_E|), the 2C-channel gradient recomputed per pixel
//                                     from g_z (conv2's transposed 3x3) instead of being written
//   vt_fusion_input_grad_nhwc       : g_{f_G} and g_{f_E} from the AdaIN backward, the |.| split and the f_E * m product
// The reductions follow act_grad's scheme: per-block double partials, then a warp per entry adds them in a fixed order.
namespace {

constexpr int MASK_CHUNK = 256;      // pixels per block of the mask-gradient pass

__global__ void __launch_bounds__(256)
torgb_gate_grad_kernel(const float* __restrict__ g, const float* __restrict__ grgb, const float* __restrict__ w, int wB,
                       int w_cstride, const float* __restrict__ ref, float slope, float gain, int B, int64_t HW, int C,
                       float* __restrict__ out) {
  const int nvec = C / 4;
  const int64_t total = (int64_t)B * HW * nvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    const int64_t bp = i / nvec;
    const int b = (int)(bp / HW);
    const int64_t p = bp - (int64_t)b * HW;
    const float* gr = grgb + (int64_t)b * 3 * HW + p;
    const float r0 = __ldg(gr), r1 = __ldg(gr + HW), r2 = __ldg(gr + 2 * HW);
    const float* wp = w + (int64_t)(wB == 1 ? 0 : b) * 3 * w_cstride + v * 4;
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + w_cstride));
    const float4 w2 = __ldg(reinterpret_cast<const float4*>(wp + 2 * w_cstride));
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    if (g) {
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g + bp * C + v * 4));
      t[0] = gv.x; t[1] = gv.y; t[2] = gv.z; t[3] = gv.w;
    }
    t[0] = fmaf(w2.x, r2, fmaf(w1.x, r1, fmaf(w0.x, r0, t[0])));
    t[1] = fmaf(w2.y, r2, fmaf(w1.y, r1, fmaf(w0.y, r0, t[1])));
    t[2] = fmaf(w2.z, r2, fmaf(w1.z, r1, fmaf(w0.z, r0, t[2])));
    t[3] = fmaf(w2.w, r2, fmaf(w1.w, r1, fmaf(w0.w, r0, t[3])));
    const float4 rv = __ldg(reinterpret_cast<const float4*>(ref + bp * C + v * 4));
    const float ra[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) t[k] = (ra[k] > 0.f ? t[k] : t[k] * slope) * gain;
    *reinterpret_cast<float4*>(out + bp * C + v * 4) = make_float4(t[0], t[1], t[2], t[3]);
  }
}

// One warp per pixel: s = sum_c g_p * f_e (double, lane-strided then a fixed shuffle tree); g_z = (s + g_m) * (1 - m^2) * [m > 0].
// Per (chunk, b) the double sum of g_z over the chunk's pixels, warps added in a fixed order.
__global__ void __launch_bounds__(256)
fusion_mask_grad_kernel(const float* __restrict__ gp, const float* __restrict__ fe, const float* __restrict__ m,
                        const float* __restrict__ gm, int64_t HW, int C, float* __restrict__ gz, double* __restrict__ ws) {
  __shared__ double sw[8];
  const int b = blockIdx.y, warp = threadIdx.x / 32, lane = threadIdx.x % 32, nvec = C / 4;
  const int64_t p_begin = (int64_t)blockIdx.x * MASK_CHUNK;
  const int64_t p_end = (p_begin + MASK_CHUNK < HW) ? p_begin + MASK_CHUNK : HW;
  double acc = 0.0;
  for (int64_t p = p_begin + warp; p < p_end; p += 8) {
    const int64_t o = ((int64_t)b * HW + p) * C;
    double s = 0.0;
    for (int v = lane; v < nvec; v += 32) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(gp + o + v * 4));
      const float4 e = __ldg(reinterpret_cast<const float4*>(fe + o + v * 4));
      s = fma((double)a.x, (double)e.x, s);
      s = fma((double)a.y, (double)e.y, s);
      s = fma((double)a.z, (double)e.z, s);
      s = fma((double)a.w, (double)e.w, s);
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
    const int64_t q = (int64_t)b * HW + p;
    const float mv = m[q];
    const float sg = (float)s + (gm ? gm[q] : 0.f);
    const float z = mv > 0.f ? sg * (1.f - mv * mv) : 0.f;
    if (lane == 0) gz[q] = z;
    acc += (double)z;
  }
  if (lane == 0) sw[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += sw[k];
    ws[(int64_t)blockIdx.x * gridDim.y + b] = t;
  }
}

// the 9 values g_z[p - (ky - 1, kx - 1)] that conv2's transposed 3x3 reads at pixel (y, x), 0 outside the map
__device__ __forceinline__ void fusion_taps(const float* __restrict__ gzb, int y, int x, int H, int W, float (&gt)[9]) {
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int yy = y - (t / 3 - 1), xx = x - (t % 3 - 1);
    gt[t] = (yy < 0 || yy >= H || xx < 0 || xx >= W) ? 0.f : __ldg(gzb + (int64_t)yy * W + xx);
  }
}

// u[c'] = sum over the taps of w2[t][c'] * gt[t]: the gradient at conv2's input, channels c' of the virtual concat
// cat(f_G, |f_G - f_E|) (C2 = 2C of them); ``w`` holds the thread's 4 channels for every tap
__device__ __forceinline__ void fusion_u4(const float (&gt)[9], const float4 (&w)[9], float (&u)[4]) {
  u[0] = u[1] = u[2] = u[3] = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    u[0] = fmaf(w[t].x, gt[t], u[0]);
    u[1] = fmaf(w[t].y, gt[t], u[1]);
    u[2] = fmaf(w[t].z, gt[t], u[2]);
    u[3] = fmaf(w[t].w, gt[t], u[3]);
  }
}

// the 4 virtual-concat values at channel c' (= 4 * v): f_G's for c' < C, |f_G - f_E| beyond
__device__ __forceinline__ void fusion_a4(const float* __restrict__ fg, const float* __restrict__ fe, int64_t o, int cc, bool second,
                                          float (&a)[4]) {
  const float4 gv = __ldg(reinterpret_cast<const float4*>(fg + o + cc));
  if (!second) {
    a[0] = gv.x; a[1] = gv.y; a[2] = gv.z; a[3] = gv.w;
    return;
  }
  const float4 ev = __ldg(reinterpret_cast<const float4*>(fe + o + cc));
  a[0] = fabsf(gv.x - ev.x); a[1] = fabsf(gv.y - ev.y); a[2] = fabsf(gv.z - ev.z); a[3] = fabsf(gv.w - ev.w);
}

// per (chunk, b, c'): (sum u, sum u * ahat) in double, ahat = (a - mean) * rstd.  dyn smem: pstep * C2 * 2 doubles
__global__ void __launch_bounds__(256)
fusion_adain_partial_kernel(const float* __restrict__ gz, const float* __restrict__ w2, const float* __restrict__ fg,
                            const float* __restrict__ fe, const float* __restrict__ stats, int H, int W, int C, int64_t chunk,
                            double* __restrict__ ws) {
  extern __shared__ double sred[];
  const int64_t HW = (int64_t)H * W;
  const int C2 = 2 * C, b = blockIdx.y, nvec = C2 / 4, pstep = blockDim.x / nvec;
  const int v = threadIdx.x % nvec, lane_p = threadIdx.x / nvec;
  const int64_t p_begin = (int64_t)blockIdx.x * chunk;
  const int64_t p_end = (p_begin + chunk < HW) ? p_begin + chunk : HW;
  if (lane_p < pstep) {
    const bool second = v * 4 >= C;
    const int cc = second ? v * 4 - C : v * 4;
    float4 w[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) w[t] = __ldg(reinterpret_cast<const float4*>(w2 + (int64_t)t * C2 + v * 4));
    float mean[4], rstd[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      mean[i] = stats[((int64_t)b * C2 + v * 4 + i) * 2];
      rstd[i] = stats[((int64_t)b * C2 + v * 4 + i) * 2 + 1];
    }
    double sg[4] = {0, 0, 0, 0}, sgx[4] = {0, 0, 0, 0};
    const float* gzb = gz + (int64_t)b * HW;
    for (int64_t p = p_begin + lane_p; p < p_end; p += pstep) {
      float gt[9], u[4], a[4];
      fusion_taps(gzb, (int)(p / W), (int)(p % W), H, W, gt);
      fusion_u4(gt, w, u);
      fusion_a4(fg, fe, ((int64_t)b * HW + p) * C, cc, second, a);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        sg[i] += (double)u[i];
        sgx[i] = fma((double)u[i], (double)((a[i] - mean[i]) * rstd[i]), sgx[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      sred[((int64_t)lane_p * C2 + v * 4 + i) * 2] = sg[i];
      sred[((int64_t)lane_p * C2 + v * 4 + i) * 2 + 1] = sgx[i];
    }
  }
  __syncthreads();
  double* dst = ws + ((int64_t)blockIdx.x * gridDim.y + b) * C2 * 2;
  for (int i = threadIdx.x; i < 2 * C2; i += blockDim.x) {
    double s = 0.0;
    for (int l = 0; l < pstep; ++l) s += sred[(int64_t)l * C2 * 2 + i];
    dst[i] = s;
  }
}

// g_fg = g_dir + T1 + sign(f_G - f_E) * T2,  g_fe = -sign(f_G - f_E) * T2 + g_p * m, with T1, T2 the AdaIN backward of the two halves
// of the concat (channel c and C + c): gamma * rstd * ((u - m_u) - ahat * m_ua)
__global__ void __launch_bounds__(256)
fusion_input_grad_kernel(const float* __restrict__ gz, const float* __restrict__ w2, const float* __restrict__ fg,
                         const float* __restrict__ fe, const float* __restrict__ stats, const float* __restrict__ gb,
                         const float* __restrict__ sums, float inv_hw, const float* __restrict__ gdir,
                         const float* __restrict__ gp, const float* __restrict__ m, int H, int W, int C, int64_t chunk,
                         float* __restrict__ gfg, float* __restrict__ gfe) {
  const int64_t HW = (int64_t)H * W;
  const int C2 = 2 * C, b = blockIdx.y, nvec = C / 4, pstep = blockDim.x / nvec;
  const int v = threadIdx.x % nvec, lane_p = threadIdx.x / nvec;
  if (lane_p >= pstep) return;
  const int64_t p_begin = (int64_t)blockIdx.x * chunk;
  const int64_t p_end = (p_begin + chunk < HW) ? p_begin + chunk : HW;
  float4 w1[9], w2b[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    w1[t] = __ldg(reinterpret_cast<const float4*>(w2 + (int64_t)t * C2 + v * 4));
    w2b[t] = __ldg(reinterpret_cast<const float4*>(w2 + (int64_t)t * C2 + C + v * 4));
  }
  float mean[2][4], rstd[2][4], coef[2][4], mu[2][4], mua[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = h * C + v * 4 + i;
      const int64_t e = (int64_t)b * C2 + c;
      mean[h][i] = stats[e * 2];
      rstd[h][i] = stats[e * 2 + 1];
      coef[h][i] = gb[(int64_t)b * 2 * C2 + c] * rstd[h][i];
      mu[h][i] = sums[e * 2] * inv_hw;
      mua[h][i] = sums[e * 2 + 1] * inv_hw;
    }
  const float* gzb = gz + (int64_t)b * HW;
  for (int64_t p = p_begin + lane_p; p < p_end; p += pstep) {
    const int y = (int)(p / W), x = (int)(p % W);
    const int64_t o = ((int64_t)b * HW + p) * C + v * 4;
    float gt[9], u1[4], u2[4];
    fusion_taps(gzb, y, x, H, W, gt);
    fusion_u4(gt, w1, u1);
    fusion_u4(gt, w2b, u2);
    const float4 gv = __ldg(reinterpret_cast<const float4*>(fg + o));
    const float4 ev = __ldg(reinterpret_cast<const float4*>(fe + o));
    const float4 pv = __ldg(reinterpret_cast<const float4*>(gp + o));
    float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gdir) dv = __ldg(reinterpret_cast<const float4*>(gdir + o));
    const float mv = __ldg(m + (int64_t)b * HW + p);
    const float ga[4] = {gv.x, gv.y, gv.z, gv.w}, ea[4] = {ev.x, ev.y, ev.z, ev.w}, pa[4] = {pv.x, pv.y, pv.z, pv.w};
    const float da[4] = {dv.x, dv.y, dv.z, dv.w};
    float rg[4], re[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float d = ga[i] - ea[i];
      const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
      const float t1 = coef[0][i] * ((u1[i] - mu[0][i]) - (ga[i] - mean[0][i]) * rstd[0][i] * mua[0][i]);
      const float t2 = coef[1][i] * ((u2[i] - mu[1][i]) - (fabsf(d) - mean[1][i]) * rstd[1][i] * mua[1][i]);
      rg[i] = da[i] + t1 + sgn * t2;
      re[i] = fmaf(pa[i], mv, -sgn * t2);
    }
    *reinterpret_cast<float4*>(gfg + o) = make_float4(rg[0], rg[1], rg[2], rg[3]);
    *reinterpret_cast<float4*>(gfe + o) = make_float4(re[0], re[1], re[2], re[3]);
  }
}

}  // namespace

extern "C" int vt_torgb_gate_grad_nhwc(const float* g, const float* g_rgb, const float* w_rgb, int wB, int w_cstride, const float* ref,
                                       float slope, float gain, int B, int64_t HW, int C, float* out, void* stream) {
  VT_CHECK(g_rgb && w_rgb && ref && out, "torgb_gate_grad: null pointer");
  VT_CHECK(B >= 1 && HW >= 1 && C >= 4 && C % 4 == 0 && w_cstride >= C && w_cstride % 4 == 0 && (wB == 1 || wB == B),
           "torgb_gate_grad: bad shape (C %% 4 == 0, w_cstride >= C, wB 1 or B)");
  VT_CHECK((!g || aligned16(g)) && aligned16(w_rgb) && aligned16(ref) && aligned16(out), "torgb_gate_grad: tensors must be 16-byte aligned");
  int64_t blocks = vt_cdiv((int64_t)B * HW * (C / 4), 256);
  const int64_t cap = (int64_t)vt_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  torgb_gate_grad_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(g, g_rgb, w_rgb, wB, w_cstride, ref, slope, gain, B, HW,
                                                                             C, out);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t vt_fusion_mask_grad_ws_bytes(int B, int64_t HW) {
  if (B < 1 || HW < 1) return -1;
  return vt_cdiv(HW, MASK_CHUNK) * B * (int64_t)sizeof(double);
}

extern "C" int vt_fusion_mask_grad_nhwc(const float* g_p, const float* f_e, const float* m, const float* g_m, int B, int64_t HW, int C,
                                        float* g_z, float* bias_grad, void* ws, void* stream) {
  VT_CHECK(g_p && f_e && m && g_z && bias_grad && ws, "fusion_mask_grad: null pointer");
  VT_CHECK(B >= 1 && B <= 65535 && HW >= 1 && C >= 4 && C % 4 == 0, "fusion_mask_grad: bad shape (C must be a multiple of 4)");
  VT_CHECK(aligned16(g_p) && aligned16(f_e) && aligned16(ws), "fusion_mask_grad: tensors must be 16-byte aligned");
  const int64_t chunks = vt_cdiv(HW, MASK_CHUNK);
  VT_CHECK(chunks < (1LL << 31), "fusion_mask_grad: plane too large");
  cudaStream_t st = (cudaStream_t)stream;
  fusion_mask_grad_kernel<<<dim3((unsigned)chunks, (unsigned)B), 256, 0, st>>>(g_p, f_e, m, g_m, HW, C, g_z, (double*)ws);
  VT_LAUNCH_CHECK();
  partials_sum_kernel<<<1, 256, 0, st>>>((const double*)ws, chunks * B, 1, 1.f, bias_grad);
  VT_LAUNCH_CHECK();
  return 0;
}

#define VT_FUSION_SHAPE_CHECK(name)                                                                                   \
  VT_CHECK(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0 && C <= 512, name ": bad shape (C must be a " \
           "multiple of 4, at most 512)")

extern "C" int vt_fusion_adain_grad_stats_nhwc(const float* g_z, const float* w2, const float* f_g, const float* f_e, const float* stats,
                                               int B, int H, int W, int C, float* sums, void* ws, void* stream) {
  VT_CHECK(g_z && w2 && f_g && f_e && stats && sums && ws, "fusion_adain_grad_stats: null pointer");
  VT_CHECK(aligned16(w2) && aligned16(f_g) && aligned16(f_e) && aligned16(ws), "fusion_adain_grad_stats: tensors must be 16-byte aligned");
  VT_FUSION_SHAPE_CHECK("fusion_adain_grad_stats");
  const int64_t HW = (int64_t)H * W;
  int64_t chunk, chunks;
  instnorm_plan(HW, 2 * C, &chunk, &chunks);
  VT_CHECK(chunks < (1LL << 31), "fusion_adain_grad_stats: plane too large");
  cudaStream_t st = (cudaStream_t)stream;
  const int pstep = 256 / (2 * C / 4);
  fusion_adain_partial_kernel<<<dim3((unsigned)chunks, (unsigned)B), 256, (size_t)pstep * 2 * C * 2 * sizeof(double), st>>>(
      g_z, w2, f_g, f_e, stats, H, W, C, chunk, (double*)ws);
  VT_LAUNCH_CHECK();
  const int64_t n = (int64_t)B * 2 * C * 2;
  partials_sum_kernel<<<(unsigned)vt_cdiv(n, 8), 256, 0, st>>>((const double*)ws, chunks, n, 1.f, sums);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_fusion_input_grad_nhwc(const float* g_z, const float* w2, const float* f_g, const float* f_e, const float* stats,
                                         const float* gamma_beta, const float* sums, const float* g_dir, const float* g_p, const float* m,
                                         int B, int H, int W, int C, float* g_fg, float* g_fe, void* stream) {
  VT_CHECK(g_z && w2 && f_g && f_e && stats && gamma_beta && sums && g_p && m && g_fg && g_fe, "fusion_input_grad: null pointer");
  VT_CHECK(aligned16(w2) && aligned16(f_g) && aligned16(f_e) && aligned16(g_p) && (!g_dir || aligned16(g_dir)) && aligned16(g_fg) &&
           aligned16(g_fe), "fusion_input_grad: tensors must be 16-byte aligned");
  VT_FUSION_SHAPE_CHECK("fusion_input_grad");
  const int64_t HW = (int64_t)H * W;
  int64_t chunk, chunks;
  instnorm_plan(HW, C, &chunk, &chunks);
  VT_CHECK(chunks < (1LL << 31), "fusion_input_grad: plane too large");
  fusion_input_grad_kernel<<<dim3((unsigned)chunks, (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
      g_z, w2, f_g, f_e, stats, gamma_beta, sums, (float)(1.0 / (double)HW), g_dir, g_p, m, H, W, C, chunk, g_fg, g_fe);
  VT_LAUNCH_CHECK();
  return 0;
}

// ---- minibatch standard deviation of the StyleGAN discriminator (model/vtoonify.py:67-75) --------------------------------------
// Sample b is in column m = b % M of its group (M = B / group, the reference's out.view(group, -1, ...)).  Per column the statistic
// is mean over (h, w, c) of sqrt(var_g + 1e-8), var_g the biased variance over the group; every sample of the column gets it as
// one more channel.  One block per column; every sum is in double and in a fixed order (thread-strided, then a shared-memory tree),
// so reruns are bit-identical.
namespace {

constexpr int MBSTD_THREADS = 256;
constexpr int MBSTD_MAX_GROUP = 4;

__device__ double mbstd_block_sum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = MBSTD_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

// x [B, HW, C] -> out [B, HW, c_out]: channels [0, C) = x, channel C = the column's statistic, (C, c_out) = 0
template <int G>
__global__ void __launch_bounds__(MBSTD_THREADS)
mbstd_kernel(const float* __restrict__ x, float* __restrict__ out, int M, int64_t HW, int C, int c_out, double inv_p) {
  __shared__ double sh[MBSTD_THREADS];
  const int m = blockIdx.x;
  const int P = (int)HW * C;
  double acc = 0.0;
  for (int i = threadIdx.x; i < P; i += MBSTD_THREADS) {
    const int p = i / C, c = i % C;
    double v[G], mean = 0.0;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int64_t b = (int64_t)g * M + m;
      v[g] = (double)__ldg(x + b * P + i);
      out[(b * HW + p) * c_out + c] = (float)v[g];
      mean += v[g];
    }
    mean *= 1.0 / G;
    double var = 0.0;
#pragma unroll
    for (int g = 0; g < G; ++g) var += (v[g] - mean) * (v[g] - mean);
    acc += (double)sqrtf((float)(var * (1.0 / G) + 1e-8));
  }
  const float s = (float)(mbstd_block_sum(acc, sh) * inv_p);
  const int tail = c_out - C;
  for (int i = threadIdx.x; i < G * (int)HW * tail; i += MBSTD_THREADS) {
    const int g = i / ((int)HW * tail), p = (i / tail) % (int)HW, c = i % tail;
    out[(((int64_t)g * M + m) * HW + p) * c_out + C + c] = c == 0 ? s : 0.f;
  }
}

// gin [B, HW, c_in] (the gradient of mbstd_kernel's output) -> gx [B, HW, C] = gin[..., :C] + d(statistic)/dx * (sum over the
// column's samples and pixels of gin[..., C]).  d sqrt(var + eps)/dx_g = (x_g - mean) / (G * sqrt(var + eps)).
template <int G>
__global__ void __launch_bounds__(MBSTD_THREADS)
mbstd_grad_kernel(const float* __restrict__ gin, const float* __restrict__ x, float* __restrict__ gx, int M, int64_t HW, int C,
                  int c_in, double inv_pg) {
  __shared__ double sh[MBSTD_THREADS];
  const int m = blockIdx.x;
  const int P = (int)HW * C;
  double part = 0.0;
  for (int i = threadIdx.x; i < G * (int)HW; i += MBSTD_THREADS) {
    const int64_t g = i / (int)HW, p = i % (int)HW;
    part += (double)__ldg(gin + ((g * M + m) * HW + p) * c_in + C);
  }
  const double coef = mbstd_block_sum(part, sh) * inv_pg;
  for (int i = threadIdx.x; i < P; i += MBSTD_THREADS) {
    const int p = i / C, c = i % C;
    double v[G], mean = 0.0;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      v[g] = (double)__ldg(x + ((int64_t)g * M + m) * P + i);
      mean += v[g];
    }
    mean *= 1.0 / G;
    double var = 0.0;
#pragma unroll
    for (int g = 0; g < G; ++g) var += (v[g] - mean) * (v[g] - mean);
    const double k = coef * (double)rsqrtf((float)(var * (1.0 / G) + 1e-8));
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int64_t b = (int64_t)g * M + m;
      gx[b * P + i] = (float)((double)__ldg(gin + (b * HW + p) * c_in + c) + k * (v[g] - mean));
    }
  }
}

}  // namespace

#define VT_MBSTD_CHECK(name, c_other)                                                                                  \
  VT_CHECK(B >= 1 && group >= 1 && group <= MBSTD_MAX_GROUP && HW >= 1 && C >= 1 && c_other > C &&                   \
           HW * c_other * MBSTD_MAX_GROUP < (1LL << 31), name ": bad shape (group 1..4, C < c_pad, small planes)");                                                                 \
  VT_CHECK(B % group == 0, name ": batch %d is not a multiple of the group size %d", B, group)

extern "C" int vt_mbstd_nhwc_f32(const float* x, float* out, int B, int group, int64_t HW, int C, int c_out, void* stream) {
  VT_CHECK(x && out, "mbstd: null pointer");
  VT_MBSTD_CHECK("mbstd", c_out);
  const int M = B / group;
  cudaStream_t st = (cudaStream_t)stream;
  switch (group) {
    case 1: mbstd_kernel<1><<<(unsigned)M, MBSTD_THREADS, 0, st>>>(x, out, M, HW, C, c_out, 1.0 / ((double)HW * C)); break;
    case 2: mbstd_kernel<2><<<(unsigned)M, MBSTD_THREADS, 0, st>>>(x, out, M, HW, C, c_out, 1.0 / ((double)HW * C)); break;
    case 3: mbstd_kernel<3><<<(unsigned)M, MBSTD_THREADS, 0, st>>>(x, out, M, HW, C, c_out, 1.0 / ((double)HW * C)); break;
    default: mbstd_kernel<4><<<(unsigned)M, MBSTD_THREADS, 0, st>>>(x, out, M, HW, C, c_out, 1.0 / ((double)HW * C)); break;
  }
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_mbstd_grad_nhwc_f32(const float* gin, const float* x, float* gx, int B, int group, int64_t HW, int C, int c_in,
                                      void* stream) {
  VT_CHECK(gin && x && gx, "mbstd_grad: null pointer");
  VT_MBSTD_CHECK("mbstd_grad", c_in);
  const int M = B / group;
  cudaStream_t st = (cudaStream_t)stream;
  switch (group) {
    case 1: mbstd_grad_kernel<1><<<(unsigned)M, MBSTD_THREADS, 0, st>>>(gin, x, gx, M, HW, C, c_in, 1.0 / ((double)HW * C * group)); break;
    case 2: mbstd_grad_kernel<2><<<(unsigned)M, MBSTD_THREADS, 0, st>>>(gin, x, gx, M, HW, C, c_in, 1.0 / ((double)HW * C * group)); break;
    case 3: mbstd_grad_kernel<3><<<(unsigned)M, MBSTD_THREADS, 0, st>>>(gin, x, gx, M, HW, C, c_in, 1.0 / ((double)HW * C * group)); break;
    default: mbstd_grad_kernel<4><<<(unsigned)M, MBSTD_THREADS, 0, st>>>(gin, x, gx, M, HW, C, c_in, 1.0 / ((double)HW * C * group)); break;
  }
  VT_LAUNCH_CHECK();
  return 0;
}
