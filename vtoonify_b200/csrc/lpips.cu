// The LPIPS head of the perceptual loss (model/stylegan/lpips/networks_basic.py:64-92 with net-lin, spatial=False), forward and
// backward, on NHWC VGG taps.  Per pixel of tap k, with f0 the target row and f1 the pred row (DistModel.forward(target, pred)):
//   u = f / (||f||_2 + eps)            (lpips/__init__.py:43-45: eps is added to the norm, not inside the square root)
//   d = sum_c w_c (u0_c - u1_c)^2      (lin_k, a 1x1 projection to one channel)
// and the loss of sample b is the sum over the taps of the spatial mean of d.  One warp per pixel; the per-pixel sums run in double
// (lane-strided, then a fixed shuffle tree), so the forward is a deterministic double reduction of exact fp32 inputs.  The spatial
// means follow act_grad's scheme: per-block double partials, then a warp per sample adds them in a fixed order.  No atomics.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int HEAD_CHUNK = 256;     // pixels per block (8 warps x 32 pixels)
constexpr int MAX_TAPS = 8;
constexpr double HEAD_EPS = 1e-10;

struct HeadArgs {
  const float* f[MAX_TAPS];
  const float* w[MAX_TAPS];
  int64_t hw[MAX_TAPS];
  int c[MAX_TAPS];
  int64_t part0[MAX_TAPS + 1];      // first block of tap k along gridDim.x
  int n;
};

__device__ __forceinline__ double warp_sum(double s) {
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
  return s;
}

// u0_c - u1_c with both products rounded (no FMA contraction), so equal rows give exactly 0
__device__ __forceinline__ double unit_diff(float f0, double r0, float f1, double r1) {
  return __dmul_rn((double)f0, r0) - __dmul_rn((double)f1, r1);
}

// the squared norms of the target row f0 and the pred row f1 of one pixel (every lane gets both)
__device__ __forceinline__ void row_norms2(const float* __restrict__ f0, const float* __restrict__ f1, int nvec, int lane, double& s0,
                                           double& s1) {
  s0 = 0.0; s1 = 0.0;
  for (int v = lane; v < nvec; v += 32) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(f0) + v), c = __ldg(reinterpret_cast<const float4*>(f1) + v);
    s0 = fma((double)a.x, (double)a.x, s0); s0 = fma((double)a.y, (double)a.y, s0);
    s0 = fma((double)a.z, (double)a.z, s0); s0 = fma((double)a.w, (double)a.w, s0);
    s1 = fma((double)c.x, (double)c.x, s1); s1 = fma((double)c.y, (double)c.y, s1);
    s1 = fma((double)c.z, (double)c.z, s1); s1 = fma((double)c.w, (double)c.w, s1);
  }
  s0 = warp_sum(s0); s1 = warp_sum(s1);
}

// blockIdx.x: a chunk of one tap's pixels (taps concatenated), blockIdx.y: the sample; ws[part * B + b] = (1 / HW) * sum of d
__global__ void __launch_bounds__(256)
lpips_head_kernel(HeadArgs a, int B, double* __restrict__ ws) {
  __shared__ double sw[8];
  const int b = blockIdx.y, warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  int k = 0;
  while (k + 1 < a.n && (int64_t)blockIdx.x >= a.part0[k + 1]) ++k;
  const int64_t HW = a.hw[k];
  const int C = a.c[k], nvec = C / 4;
  const float* __restrict__ w = a.w[k];
  const int64_t p_begin = ((int64_t)blockIdx.x - a.part0[k]) * HEAD_CHUNK;
  const int64_t p_end = (p_begin + HEAD_CHUNK < HW) ? p_begin + HEAD_CHUNK : HW;
  double acc = 0.0;
  for (int64_t p = p_begin + warp; p < p_end; p += 8) {
    const float* f0 = a.f[k] + ((int64_t)b * HW + p) * C;
    const float* f1 = a.f[k] + ((int64_t)(B + b) * HW + p) * C;
    double s0, s1;
    row_norms2(f0, f1, nvec, lane, s0, s1);
    const double r0 = 1.0 / (sqrt(s0) + HEAD_EPS), r1 = 1.0 / (sqrt(s1) + HEAD_EPS);
    double d = 0.0;
    for (int v = lane; v < nvec; v += 32) {
      const float4 x0 = __ldg(reinterpret_cast<const float4*>(f0) + v), x1 = __ldg(reinterpret_cast<const float4*>(f1) + v);
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + v);
      double t;
      t = unit_diff(x0.x, r0, x1.x, r1); d = fma((double)wv.x * t, t, d);
      t = unit_diff(x0.y, r0, x1.y, r1); d = fma((double)wv.y * t, t, d);
      t = unit_diff(x0.z, r0, x1.z, r1); d = fma((double)wv.z * t, t, d);
      t = unit_diff(x0.w, r0, x1.w, r1); d = fma((double)wv.w * t, t, d);
    }
    acc += warp_sum(d);
  }
  if (lane == 0) sw[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int j = 0; j < 8; ++j) t += sw[j];
    ws[(int64_t)blockIdx.x * B + b] = t / (double)HW;
  }
}

// out[b] = sum over parts of ws[part * B + b], one warp per sample in a fixed order
__global__ void __launch_bounds__(256)
lpips_sum_kernel(const double* __restrict__ ws, int64_t parts, int B, float* __restrict__ out) {
  const int b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (b >= B) return;
  double s = 0.0;
  for (int64_t k = lane; k < parts; k += 32) s += ws[k * B + b];
  s = warp_sum(s);
  if (lane == 0) out[b] = (float)s;
}

// Gradient of one tap, one warp per pixel: with a = n + eps, t = u0 - u1 and s = g_b[b] / HW,
//   g0 = s / a0 * (A0 - f0 (A0 . f0) / (n0 a0)),  A0 = +2 w t     (target rows)
//   g1 = s / a1 * (A1 - f1 (A1 . f1) / (n1 a1)),  A1 = -2 w t     (pred rows)
// and 0 for a side whose row is all zero (n = 0, where the ReLU in front of the tap passes no gradient anyway).
__global__ void __launch_bounds__(256)
lpips_head_grad_kernel(const float* __restrict__ f, const float* __restrict__ w, const float* __restrict__ gb, int B, int64_t HW, int C,
                       float* __restrict__ g0, float* __restrict__ g1) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, nvec = C / 4;
  const int64_t total = (int64_t)B * HW;
  for (int64_t q = (int64_t)blockIdx.x * 8 + warp; q < total; q += (int64_t)gridDim.x * 8) {
    const int b = (int)(q / HW);
    const int64_t p = q - (int64_t)b * HW;
    const float* f0 = f + q * C;
    const float* f1 = f + ((int64_t)(B + b) * HW + p) * C;
    double s0, s1;
    row_norms2(f0, f1, nvec, lane, s0, s1);
    const double n0 = sqrt(s0), n1 = sqrt(s1), a0 = n0 + HEAD_EPS, a1 = n1 + HEAD_EPS, r0 = 1.0 / a0, r1 = 1.0 / a1;
    double q0 = 0.0, q1 = 0.0;     // sum_c w t f0 and sum_c w t f1
    for (int v = lane; v < nvec; v += 32) {
      const float4 x0 = __ldg(reinterpret_cast<const float4*>(f0) + v), x1 = __ldg(reinterpret_cast<const float4*>(f1) + v);
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + v);
      const float e0[4] = {x0.x, x0.y, x0.z, x0.w}, e1[4] = {x1.x, x1.y, x1.z, x1.w}, ew[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double wt = (double)ew[j] * unit_diff(e0[j], r0, e1[j], r1);
        q0 = fma(wt, (double)e0[j], q0);
        q1 = fma(wt, (double)e1[j], q1);
      }
    }
    q0 = warp_sum(q0); q1 = warp_sum(q1);
    const double s = (double)__ldg(gb + b) / (double)HW;
    // g = s / a * (A - f * (A . f) / (n a)) = c * (+-2 w t) - f * k with c = s / a and k = c * (A . f) / (n a)
    const double c0 = s * r0, c1 = s * r1;
    const double k0 = n0 > 0.0 ? c0 * (2.0 * q0) / (n0 * a0) : 0.0;
    const double k1 = n1 > 0.0 ? c1 * (-2.0 * q1) / (n1 * a1) : 0.0;
    for (int v = lane; v < nvec; v += 32) {
      const float4 x0 = __ldg(reinterpret_cast<const float4*>(f0) + v), x1 = __ldg(reinterpret_cast<const float4*>(f1) + v);
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + v);
      const float e0[4] = {x0.x, x0.y, x0.z, x0.w}, e1[4] = {x1.x, x1.y, x1.z, x1.w}, ew[4] = {wv.x, wv.y, wv.z, wv.w};
      float o0[4], o1[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double wt2 = 2.0 * (double)ew[j] * unit_diff(e0[j], r0, e1[j], r1);
        o0[j] = n0 > 0.0 ? (float)(c0 * wt2 - (double)e0[j] * k0) : 0.f;
        o1[j] = n1 > 0.0 ? (float)(-c1 * wt2 - (double)e1[j] * k1) : 0.f;
      }
      if (g0) reinterpret_cast<float4*>(g0 + q * C)[v] = make_float4(o0[0], o0[1], o0[2], o0[3]);
      if (g1) reinterpret_cast<float4*>(g1 + q * C)[v] = make_float4(o1[0], o1[1], o1[2], o1[3]);
    }
  }
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

int64_t head_parts(int n_taps, const int64_t* HW, int64_t* part0) {
  int64_t parts = 0;
  for (int k = 0; k < n_taps; ++k) {
    if (part0) part0[k] = parts;
    parts += vt_cdiv(HW[k], HEAD_CHUNK);
  }
  if (part0) part0[n_taps] = parts;
  return parts;
}

}  // namespace

extern "C" int64_t vt_lpips_head_ws_bytes(int B, int n_taps, const int64_t* HW) {
  if (B < 1 || n_taps < 1 || n_taps > MAX_TAPS || !HW) return -1;
  for (int k = 0; k < n_taps; ++k)
    if (HW[k] < 1) return -1;
  return head_parts(n_taps, HW, nullptr) * B * (int64_t)sizeof(double);
}

extern "C" int vt_lpips_head_nhwc(int n_taps, const float* const* f, const float* const* w, const int64_t* HW, const int* C, int B,
                                  float* out, void* ws, void* stream) {
  VT_CHECK(n_taps >= 1 && n_taps <= MAX_TAPS && f && w && HW && C && out && ws, "lpips_head: bad args (1 to %d taps)", MAX_TAPS);
  VT_CHECK(B >= 1 && B <= 65535 && aligned16(ws), "lpips_head: bad batch or workspace");
  HeadArgs a{};
  a.n = n_taps;
  for (int k = 0; k < n_taps; ++k) {
    VT_CHECK(f[k] && w[k] && aligned16(f[k]) && aligned16(w[k]), "lpips_head: tap %d: null or unaligned tensor", k);
    VT_CHECK(HW[k] >= 1 && C[k] >= 4 && C[k] % 4 == 0, "lpips_head: tap %d: bad shape (C must be a multiple of 4)", k);
    a.f[k] = f[k]; a.w[k] = w[k]; a.hw[k] = HW[k]; a.c[k] = C[k];
  }
  const int64_t parts = head_parts(n_taps, HW, a.part0);
  VT_CHECK(parts < (1LL << 31), "lpips_head: maps too large");
  cudaStream_t st = (cudaStream_t)stream;
  lpips_head_kernel<<<dim3((unsigned)parts, (unsigned)B), 256, 0, st>>>(a, B, (double*)ws);
  VT_LAUNCH_CHECK();
  lpips_sum_kernel<<<(unsigned)vt_cdiv(B, 8), 256, 0, st>>>((const double*)ws, parts, B, out);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_lpips_head_grad_nhwc(const float* f, const float* w, const float* g_b, int B, int64_t HW, int C, float* g_target, float* g_pred, void* stream) {
  VT_CHECK(f && w && g_b && (g_target || g_pred), "lpips_head_grad: null pointer");
  VT_CHECK(B >= 1 && HW >= 1 && C >= 4 && C % 4 == 0, "lpips_head_grad: bad shape (C must be a multiple of 4)");
  VT_CHECK(aligned16(f) && aligned16(w) && aligned16(g_target) && aligned16(g_pred), "lpips_head_grad: tensors must be 16-byte aligned");
  int64_t blocks = vt_cdiv((int64_t)B * HW, 8);
  const int64_t cap = (int64_t)vt_num_sms() * 32;
  if (blocks > cap) blocks = cap;
  lpips_head_grad_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(f, w, g_b, B, HW, C, g_target, g_pred);
  VT_LAUNCH_CHECK();
  return 0;
}
