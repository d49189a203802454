// align.cu — f2: the image stages of the FFHQ face alignment (align_face, model/encoder/align_all_parallel.py:108-147) on the device,
// byte for byte with the libraries the reference calls (Pillow, NumPy, SciPy on x86-64):
//   lanczos  Pillow resize(LANCZOS) on RGB uint8: 22-bit fixed-point taps from host tables, acc = 2^21 + sum in * kk, out =
//            clamp(acc >> 22, 0, 255); one launch per axis, horizontal first, through a uint8 intermediate;
//   blur     scipy.ndimage.gaussian_filter(np.pad(float32(img), 'reflect'), [s, s, 0]): the reflect-101 pad is virtual, rows (axis 0)
//            then columns, each output w0 x0 + sum_{k=r..1} (x_-k + x_+k) w_k in double with SciPy's half-sample 'reflect' boundary on
//            the padded extent, stored as float32; the column pass can apply the first blend img += (g - img) * clip(3 mask + 1, 0, 1);
//   median   np.median per channel: an exact radix select (4 passes of 8 bits) on order-preserving keys of the float32 bits, with
//            device histograms, so the result never leaves the device;
//   finish   img += (med - img) * clip(mask, 0, 1), np.rint (half to even), clamp to uint8;
//   warp     Pillow transform(QUAD, BILINEAR): xs = a0 + a1 u + a2 v + a3 u v at pixel centres, 0 outside the image, bilinear lerp in
//            double, truncated to uint8.
// Every double and float step that the CPU rounds is written as an explicit __d*_rn / __f*_rn intrinsic: nvcc contracts a * b + c into
// an fma by default, the x86-64 builds of those libraries do not, and a single fused rounding changes output bytes.
// The blends' mask is the reference's float64 formula (NumPy 2 promotes float32 / int64 scalars to float64): the product with the
// float32 difference is float64, the sum is float64 rounded once to float32.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int ALIGN_THREADS = 256;
constexpr int MEDIAN_SEL = 6;           // (channel, rank) selections: ranks (n - 1) / 2 and n / 2 of each of the 3 channels

struct GaussTaps { double w[VT_ALIGN_MAX_RADIUS + 1]; };
struct QuadCoef { double a[8]; };
struct Pad4 { int l, t, r, b; };

unsigned grid_for(int64_t n) {
  int64_t blocks = vt_cdiv(n, ALIGN_THREADS);
  const int64_t cap = (int64_t)vt_num_sms() * 16;
  return (unsigned)(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}

// np.pad 'reflect' (reflect-101, repeated for pads wider than the image)
__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  const int p = 2 * n - 2;
  int j = i % p;
  if (j < 0) j += p;
  return j >= n ? p - j : j;
}

// scipy.ndimage mode 'reflect' (half-sample symmetric, period 2n)
__device__ __forceinline__ int reflect_half(int i, int n) {
  const int p = 2 * n;
  int j = i % p;
  if (j < 0) j += p;
  return j >= n ? p - 1 - j : j;
}

// the reference's mask of the padded image at (y, x), float64
__device__ __forceinline__ double pad_mask(int y, int x, int Hp, int Wp, Pad4 pd) {
  const double mx = __dsub_rn(1.0, fmin(__ddiv_rn((double)x, (double)pd.l), __ddiv_rn((double)(Wp - 1 - x), (double)pd.r)));
  const double my = __dsub_rn(1.0, fmin(__ddiv_rn((double)y, (double)pd.t), __ddiv_rn((double)(Hp - 1 - y), (double)pd.b)));
  return fmax(mx, my);
}

// img + (target - img) * weight: float32 difference, float64 product and sum, one rounding to float32
__device__ __forceinline__ float blend(float img, float target, double weight) {
  return __double2float_rn(__dadd_rn((double)img, __dmul_rn((double)__fsub_rn(target, img), weight)));
}

__device__ __forceinline__ double clip01(double v) { return fmin(fmax(v, 0.0), 1.0); }

// ---- Lanczos -------------------------------------------------------------------------------------------------------------------------
// horizontal: out [H, Wo, 3] from in [H, W, 3]; vertical: out [Ho, W, 3] from in [H, W, 3]; one thread per output pixel
template <bool HORIZONTAL>
__global__ void __launch_bounds__(ALIGN_THREADS)
lanczos_kernel(const uint8_t* __restrict__ in, int64_t in_pitch, uint8_t* __restrict__ out, int Ho, int Wo, const int* __restrict__ tab,
               int out_size, int ksize) {
  const int64_t n = (int64_t)Ho * Wo;
  const int* xmin = tab;
  const int* taps = tab + out_size;
  const int* kk = tab + 2 * out_size;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(i / Wo), ox = (int)(i - (int64_t)oy * Wo);
    const int o = HORIZONTAL ? ox : oy;
    const int lo = __ldg(xmin + o), nt = __ldg(taps + o);
    const int* k = kk + (int64_t)o * ksize;
    int acc[3] = {1 << 21, 1 << 21, 1 << 21};
    for (int t = 0; t < nt; ++t) {
      const int w = __ldg(k + t);
      const uint8_t* p = HORIZONTAL ? in + (int64_t)oy * in_pitch + (int64_t)(lo + t) * 3 : in + (int64_t)(lo + t) * in_pitch + (int64_t)ox * 3;
      acc[0] += (int)p[0] * w; acc[1] += (int)p[1] * w; acc[2] += (int)p[2] * w;
    }
    uint8_t* q = out + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int v = acc[c] >> 22;
      q[c] = (uint8_t)(acc[c] <= 0 ? 0 : (v > 255 ? 255 : v));
    }
  }
}

// ---- padded blur ---------------------------------------------------------------------------------------------------------------------
// axis 0 of the Gaussian over the virtual padded image: in [H, W, 3] uint8 (pitch), out [Hp, Wp, 3] float32
__global__ void __launch_bounds__(ALIGN_THREADS)
blur_rows_kernel(const uint8_t* __restrict__ in, int64_t in_pitch, int H, int W, Pad4 pd, float* __restrict__ out, int Hp, int Wp,
                 GaussTaps g, int r) {
  const int64_t n = (int64_t)Hp * Wp;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / Wp), x = (int)(i - (int64_t)y * Wp);
    const uint8_t* col = in + (int64_t)reflect101(x - pd.l, W) * 3;
    auto px = [&](int yy) { return col + (int64_t)reflect101(reflect_half(yy, Hp) - pd.t, H) * in_pitch; };
    const uint8_t* p0 = px(y);
    double acc[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] = __dmul_rn((double)p0[c], g.w[0]);
    for (int k = r; k >= 1; --k) {
      const uint8_t* a = px(y - k);
      const uint8_t* b = px(y + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] = __dadd_rn(acc[c], __dmul_rn(__dadd_rn((double)a[c], (double)b[c]), g.w[k]));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) out[i * 3 + c] = __double2float_rn(acc[c]);
  }
}

// axis 1 of the Gaussian: in, out [Hp, Wp, 3] float32; with img (the uint8 image under the virtual pad), out is the first blend instead
__global__ void __launch_bounds__(ALIGN_THREADS)
blur_cols_kernel(const float* __restrict__ in, float* __restrict__ out, int Hp, int Wp, GaussTaps g, int r,
                 const uint8_t* __restrict__ img, int64_t img_pitch, int H, int W, Pad4 pd) {
  const int64_t n = (int64_t)Hp * Wp;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / Wp), x = (int)(i - (int64_t)y * Wp);
    const float* row = in + (int64_t)y * Wp * 3;
    const float* p0 = row + (int64_t)x * 3;
    double acc[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] = __dmul_rn((double)p0[c], g.w[0]);
    for (int k = r; k >= 1; --k) {
      const float* a = row + (int64_t)reflect_half(x - k, Wp) * 3;
      const float* b = row + (int64_t)reflect_half(x + k, Wp) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] = __dadd_rn(acc[c], __dmul_rn(__dadd_rn((double)a[c], (double)b[c]), g.w[k]));
    }
    if (img == nullptr) {
#pragma unroll
      for (int c = 0; c < 3; ++c) out[i * 3 + c] = __double2float_rn(acc[c]);
    } else {
      const uint8_t* s = img + (int64_t)reflect101(y - pd.t, H) * img_pitch + (int64_t)reflect101(x - pd.l, W) * 3;
      const double m = clip01(__dadd_rn(__dmul_rn(pad_mask(y, x, Hp, Wp, pd), 3.0), 1.0));
#pragma unroll
      for (int c = 0; c < 3; ++c) out[i * 3 + c] = blend((float)s[c], __double2float_rn(acc[c]), m);
    }
  }
}

// ---- median --------------------------------------------------------------------------------------------------------------------------
struct MedianState {
  uint32_t hist[MEDIAN_SEL][256];
  uint32_t prefix[MEDIAN_SEL];
  uint32_t rank[MEDIAN_SEL];
};

// order-preserving key of a float's bits (negative values flipped, positive values above them)
__device__ __forceinline__ uint32_t float_key(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__global__ void median_init_kernel(MedianState* st, int64_t n) {
  uint32_t* h = &st->hist[0][0];
  for (int i = threadIdx.x; i < MEDIAN_SEL * 256; i += blockDim.x) h[i] = 0;
  if (threadIdx.x < MEDIAN_SEL) {
    st->prefix[threadIdx.x] = 0;
    st->rank[threadIdx.x] = (uint32_t)((threadIdx.x & 1) ? n / 2 : (n - 1) / 2);
  }
}

// histogram of digit `shift` of the keys that match each selection's prefix so far; x [n, 3]
__global__ void __launch_bounds__(ALIGN_THREADS)
median_hist_kernel(const float* __restrict__ x, int64_t n3, MedianState* st, int shift) {
  __shared__ uint32_t sh[MEDIAN_SEL][256];
  __shared__ uint32_t pre[MEDIAN_SEL];
  for (int i = threadIdx.x; i < MEDIAN_SEL * 256; i += blockDim.x) (&sh[0][0])[i] = 0;
  if (threadIdx.x < MEDIAN_SEL) pre[threadIdx.x] = st->prefix[threadIdx.x];
  __syncthreads();
  const uint32_t hi = shift == 24 ? 0u : (0xffffffffu << (shift + 8));
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n3; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t key = float_key(__ldg(x + i));
    const int c = (int)(i % 3);
    const uint32_t d = (key >> shift) & 255u;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int s = 2 * c + q;
      if (((key ^ pre[s]) & hi) == 0) atomicAdd(&sh[s][d], 1u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < MEDIAN_SEL * 256; i += blockDim.x) {
    const uint32_t v = (&sh[0][0])[i];
    if (v) atomicAdd(&st->hist[0][0] + i, v);
  }
}

// pick each selection's digit from its histogram and clear it; after the last digit, write np.median's value per channel
__global__ void median_select_kernel(MedianState* st, int shift, int64_t n, float* med) {
  const int s = threadIdx.x;
  if (s < MEDIAN_SEL) {
    uint32_t k = st->rank[s], cum = 0;
    int d = 0;
    for (; d < 255; ++d) {
      const uint32_t h = st->hist[s][d];
      if (cum + h > k) break;
      cum += h;
    }
    st->prefix[s] |= (uint32_t)d << shift;
    st->rank[s] = k - cum;
    for (int b = 0; b < 256; ++b) st->hist[s][b] = 0;
  }
  __syncwarp();
  if (shift == 0 && s < 3) {
    const float v0 = key_float(st->prefix[2 * s]), v1 = key_float(st->prefix[2 * s + 1]);
    med[s] = (n & 1) ? v0 : __fdiv_rn(__fadd_rn(v0, v1), 2.f);
  }
}

// ---- second blend, quantisation, warp --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ALIGN_THREADS)
finish_kernel(const float* __restrict__ x, const float* __restrict__ med, uint8_t* __restrict__ out, int Hp, int Wp, Pad4 pd) {
  const int64_t n = (int64_t)Hp * Wp;
  const float m0 = med[0], m1 = med[1], m2 = med[2];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / Wp), xx = (int)(i - (int64_t)y * Wp);
    const double m = clip01(pad_mask(y, xx, Hp, Wp, pd));
    const float md[3] = {m0, m1, m2};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = rintf(blend(x[i * 3 + c], md[c], m));     // round half to even
      out[i * 3 + c] = (uint8_t)(v <= 0.f ? 0 : (v >= 255.f ? 255 : (int)v));
    }
  }
}

__global__ void __launch_bounds__(ALIGN_THREADS)
warp_kernel(const uint8_t* __restrict__ in, int64_t in_pitch, int H, int W, QuadCoef q, uint8_t* __restrict__ out, int size) {
  const int64_t n = (int64_t)size * size;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(i / size), ox = (int)(i - (int64_t)oy * size);
    const double u = (double)ox + 0.5, v = (double)oy + 0.5;
    double xs = __dadd_rn(__dadd_rn(__dadd_rn(q.a[0], __dmul_rn(q.a[1], u)), __dmul_rn(q.a[2], v)), __dmul_rn(__dmul_rn(q.a[3], u), v));
    double ys = __dadd_rn(__dadd_rn(__dadd_rn(q.a[4], __dmul_rn(q.a[5], u)), __dmul_rn(q.a[6], v)), __dmul_rn(__dmul_rn(q.a[7], u), v));
    uint8_t* o = out + i * 3;
    if (!(xs >= 0.0 && xs < (double)W && ys >= 0.0 && ys < (double)H)) {
      o[0] = o[1] = o[2] = 0;
      continue;
    }
    xs = __dsub_rn(xs, 0.5);
    ys = __dsub_rn(ys, 0.5);
    const int x = (int)floor(xs), y = (int)floor(ys);
    const double dx = __dsub_rn(xs, (double)x), dy = __dsub_rn(ys, (double)y);
    const int x0 = min(max(x, 0), W - 1) * 3, x1 = min(max(x + 1, 0), W - 1) * 3;
    const uint8_t* r1 = in + (int64_t)min(max(y, 0), H - 1) * in_pitch;
    const bool second = y + 1 >= 0 && y + 1 < H;
    const uint8_t* r2 = in + (int64_t)(second ? y + 1 : 0) * in_pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double v1 = __dadd_rn((double)r1[x0 + c], __dmul_rn((double)((int)r1[x1 + c] - (int)r1[x0 + c]), dx));
      const double v2 = second ? __dadd_rn((double)r2[x0 + c], __dmul_rn((double)((int)r2[x1 + c] - (int)r2[x0 + c]), dx)) : v1;
      o[c] = (uint8_t)(int)__dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy));
    }
  }
}

bool pad_ok(const int* pad) { return pad && pad[0] >= 1 && pad[1] >= 1 && pad[2] >= 1 && pad[3] >= 1; }

}  // namespace

extern "C" {

int vt_align_lanczos_u8(const uint8_t* in, int64_t in_pitch, int H, int W, uint8_t* out, int out_size, int horizontal, const int* tab,
                        int ksize, void* stream) {
  VT_CHECK(in && out && tab && in != out, "vt_align_lanczos_u8: null pointer or in-place call");
  VT_CHECK(H >= 1 && W >= 1 && out_size >= 1 && ksize >= 1 && in_pitch >= 3 * (int64_t)W, "vt_align_lanczos_u8: bad shape");
  const int Ho = horizontal ? H : out_size, Wo = horizontal ? out_size : W;
  VT_CHECK((int64_t)Ho * Wo * 3 < 0x7fffffff && (int64_t)out_size * ksize < 0x7fffffff, "vt_align_lanczos_u8: too large");
  cudaStream_t st = (cudaStream_t)stream;
  if (horizontal) lanczos_kernel<true><<<grid_for((int64_t)Ho * Wo), ALIGN_THREADS, 0, st>>>(in, in_pitch, out, Ho, Wo, tab, out_size, ksize);
  else lanczos_kernel<false><<<grid_for((int64_t)Ho * Wo), ALIGN_THREADS, 0, st>>>(in, in_pitch, out, Ho, Wo, tab, out_size, ksize);
  VT_LAUNCH_CHECK();
  return 0;
}

int vt_align_blur_rows_f32(const uint8_t* in, int64_t in_pitch, int H, int W, const int* pad, float* out, const double* w, int r,
                           void* stream) {
  VT_CHECK(in && out && w && pad_ok(pad), "vt_align_blur_rows_f32: null pointer or a pad below 1");
  VT_CHECK(H >= 1 && W >= 1 && in_pitch >= 3 * (int64_t)W && r >= 0 && r <= VT_ALIGN_MAX_RADIUS, "vt_align_blur_rows_f32: bad shape or radius");
  const Pad4 pd{pad[0], pad[1], pad[2], pad[3]};
  const int64_t Hp = (int64_t)H + pd.t + pd.b, Wp = (int64_t)W + pd.l + pd.r;
  VT_CHECK(Hp * Wp * 3 < 0x7fffffff, "vt_align_blur_rows_f32: padded image too large");
  GaussTaps g;
  for (int k = 0; k <= r; ++k) g.w[k] = w[k];
  blur_rows_kernel<<<grid_for(Hp * Wp), ALIGN_THREADS, 0, (cudaStream_t)stream>>>(in, in_pitch, H, W, pd, out, (int)Hp, (int)Wp, g, r);
  VT_LAUNCH_CHECK();
  return 0;
}

int vt_align_blur_cols_f32(const float* in, float* out, int Hp, int Wp, const double* w, int r, const uint8_t* img, int64_t img_pitch,
                           int H, int W, const int* pad, void* stream) {
  VT_CHECK(in && out && w && in != out, "vt_align_blur_cols_f32: null pointer or in-place call");
  VT_CHECK(Hp >= 1 && Wp >= 1 && (int64_t)Hp * Wp * 3 < 0x7fffffff && r >= 0 && r <= VT_ALIGN_MAX_RADIUS, "vt_align_blur_cols_f32: bad shape or radius");
  Pad4 pd{0, 0, 0, 0};
  if (img) {
    VT_CHECK(pad_ok(pad) && H >= 1 && W >= 1 && img_pitch >= 3 * (int64_t)W, "vt_align_blur_cols_f32: bad blend image or pad");
    pd = Pad4{pad[0], pad[1], pad[2], pad[3]};
    VT_CHECK((int64_t)H + pd.t + pd.b == Hp && (int64_t)W + pd.l + pd.r == Wp, "vt_align_blur_cols_f32: pad does not give %d x %d", Hp, Wp);
  }
  GaussTaps g;
  for (int k = 0; k <= r; ++k) g.w[k] = w[k];
  blur_cols_kernel<<<grid_for((int64_t)Hp * Wp), ALIGN_THREADS, 0, (cudaStream_t)stream>>>(in, out, Hp, Wp, g, r, img, img_pitch, H, W, pd);
  VT_LAUNCH_CHECK();
  return 0;
}

int64_t vt_align_median_ws_bytes(void) { return (int64_t)sizeof(MedianState); }

int vt_align_median_f32(const float* x, int64_t n, float* med, void* ws, void* stream) {
  VT_CHECK(x && med && ws, "vt_align_median_f32: null pointer");
  VT_CHECK(n >= 1 && n * 3 < 0x7fffffff, "vt_align_median_f32: bad count %lld", (long long)n);
  cudaStream_t st = (cudaStream_t)stream;
  MedianState* s = (MedianState*)ws;
  median_init_kernel<<<1, ALIGN_THREADS, 0, st>>>(s, n);
  VT_LAUNCH_CHECK();
  for (int shift = 24; shift >= 0; shift -= 8) {
    median_hist_kernel<<<grid_for(n * 3), ALIGN_THREADS, 0, st>>>(x, n * 3, s, shift);
    VT_LAUNCH_CHECK();
    median_select_kernel<<<1, 32, 0, st>>>(s, shift, n, med);
    VT_LAUNCH_CHECK();
  }
  return 0;
}

int vt_align_finish_u8(const float* x, const float* med, uint8_t* out, int Hp, int Wp, const int* pad, void* stream) {
  VT_CHECK(x && med && out && pad_ok(pad), "vt_align_finish_u8: null pointer or a pad below 1");
  VT_CHECK(Hp >= 1 && Wp >= 1 && (int64_t)Hp * Wp * 3 < 0x7fffffff, "vt_align_finish_u8: bad shape");
  const Pad4 pd{pad[0], pad[1], pad[2], pad[3]};
  finish_kernel<<<grid_for((int64_t)Hp * Wp), ALIGN_THREADS, 0, (cudaStream_t)stream>>>(x, med, out, Hp, Wp, pd);
  VT_LAUNCH_CHECK();
  return 0;
}

int vt_align_warp_u8(const uint8_t* in, int64_t in_pitch, int H, int W, const double* coef, uint8_t* out, int size, void* stream) {
  VT_CHECK(in && coef && out, "vt_align_warp_u8: null pointer");
  VT_CHECK(H >= 1 && W >= 1 && in_pitch >= 3 * (int64_t)W && size >= 1 && size <= 4096, "vt_align_warp_u8: bad shape");
  QuadCoef q;
  for (int k = 0; k < 8; ++k) q.a[k] = coef[k];
  warp_kernel<<<grid_for((int64_t)size * size), ALIGN_THREADS, 0, (cudaStream_t)stream>>>(in, in_pitch, H, W, q, out, size);
  VT_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
