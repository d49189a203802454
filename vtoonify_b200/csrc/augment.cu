// augment.cu — the geometric training augmentation of model/simple_augment.py (random_apply_affine) in one launch:
//   out[b, c] = down2(warp_b(up2(reflect_pad(in[b, c]))))
// up2: x2 with the 12-tap kernel k as a true convolution, upfirdn2d(up=2, pad=(6, 5)) in x then y, zeros beyond the padded extent:
//        U[Y] = sum_r P[r] k[Y + 5 - 2r]                      (6 non-zero taps per output, their parity set by Y's)
// warp:  A[i][j] = bilinear sample of U at (x, y) = (c0 + c1 j + c2 i, c3 + c4 j + c5 i), zeros outside the x2 image
// down2: upfirdn2d(down=2, pad=(-1, -1)) with the flipped kernel, x then y:  out[n] = sum_t k[t] A[2n + 1 + t]
// so output pixel (oy, ox) reads the 12 x 12 warp-grid samples from (2oy + 1, 2ox + 1).  A block (sample, T x T output tile) owns the
// (2T + 10)^2 warp-grid block of its tile; it computes the block's bilinear indices and weights once and then, per channel, stages the
// reflect-padded input window that covers the block's footprint, builds the x2 window from it (x then y), warps, and runs both down
// passes in shared memory.  Nothing intermediate goes to global memory, sums run in a fixed order, and there are no atomics.
//
// The x2 window of a tile is the bounding box of its block's footprint; the host planner (vt_augment_affine_plan) sizes it for the
// worst sample of the call and picks the tile side so that it fits the shared-memory budget, or sends the call to the unfused route.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int AUG_TAPS = 12;
constexpr int AUG_THREADS = 256;
constexpr int AUG_SMEM_BUDGET = 112 * 1024;      // two blocks per SM
constexpr double AUG_COORD_LIMIT = 4194304.0;    // 2^22: window origins and offsets stay exact in int and fp32

// input rows / columns that cover a window of `win` x2 samples (each x2 sample reads 6 consecutive inputs)
__host__ __device__ inline int aug_in_extent(int win) { return win / 2 + 8; }

struct AugLayout {
  int buf1, buf2, pts, maps;   // floats
  __host__ __device__ AugLayout(int T, int win_w, int win_h) {
    const int nb = 2 * T + 10, in_w = aug_in_extent(win_w), in_h = aug_in_extent(win_h);
    buf1 = max(max(in_h * in_w, win_h * win_w), nb * T);   // input window, x2 window, x-down rows
    buf2 = max(in_h * win_w, nb * nb);                      // x-upsampled rows, warped block
    pts = 3 * nb * nb;                                      // per block point: window offset, x weight, y weight
    maps = in_h + in_w;                                     // source row / column of each input-window row / column
  }
  __host__ __device__ int64_t bytes() const { return 4 * (int64_t)(buf1 + buf2 + pts + maps); }
};

// padded index -> source index of the reflect pad, or -1 beyond the padded extent (where upfirdn2d sees zeros)
__device__ __forceinline__ int aug_src(int r, int n_pad, int pad0, int n) {
  if (r < 0 || r >= n_pad) return -1;
  int q = r - pad0;
  if (q < 0) q = -q;
  if (q >= n) q = 2 * n - 2 - q;
  return q;
}

template <int T>
__global__ void __launch_bounds__(AUG_THREADS)
augment_affine_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ kern,
                      const double* __restrict__ coef, int C, int H, int W, int pad_x, int pad_y, int Hp, int Wp, int tiles_x,
                      int win_w, int win_h) {
  constexpr int NB = 2 * T + 10;
  extern __shared__ float smem[];
  __shared__ float k[AUG_TAPS];
  const AugLayout L(T, win_w, win_h);
  const int in_w = aug_in_extent(win_w), in_h = aug_in_extent(win_h);
  float* buf1 = smem;
  float* buf2 = buf1 + L.buf1;
  int* pidx = reinterpret_cast<int*>(buf2 + L.buf2);
  float* pwx = reinterpret_cast<float*>(pidx + NB * NB);
  float* pwy = pwx + NB * NB;
  int* rmap = reinterpret_cast<int*>(pwy + NB * NB);
  int* cmap = rmap + in_h;

  const int tid = threadIdx.x, b = blockIdx.y;
  const int ty0 = (blockIdx.x / tiles_x) * T, tx0 = (blockIdx.x % tiles_x) * T;
  const double* cf = coef + 6 * (int64_t)b;
  const double c0 = cf[0], c1 = cf[1], c2 = cf[2], c3 = cf[3], c4 = cf[4], c5 = cf[5];
  // the block's first warp-grid sample in double, split into an integer and a fractional part; the per-point offsets from it
  // (at most ~2.5 (2T + 9) samples) are formed in fp32 on the fractional part, so the weights keep fp32 precision at any position
  const int j0 = 2 * tx0 + 1, i0 = 2 * ty0 + 1;
  const double xo = c0 + c1 * j0 + c2 * i0, yo = c3 + c4 * j0 + c5 * i0;
  const double ext = NB - 1;
  const int xw = (int)floor(xo + fmin(0.0, c1 * ext) + fmin(0.0, c2 * ext)) - 1;   // window origin, one sample of margin
  const int yw = (int)floor(yo + fmin(0.0, c4 * ext) + fmin(0.0, c5 * ext)) - 1;
  const double xo_i = floor(xo), yo_i = floor(yo);
  const float xo_f = (float)(xo - xo_i), yo_f = (float)(yo - yo_i);
  const int dx0 = (int)xo_i - xw, dy0 = (int)yo_i - yw;
  const float fc1 = (float)c1, fc2 = (float)c2, fc4 = (float)c4, fc5 = (float)c5;
  for (int p = tid; p < NB * NB; p += AUG_THREADS) {
    const float di = (float)(p / NB), dj = (float)(p % NB);
    const float fx = fmaf(fc2, di, fmaf(fc1, dj, xo_f)), fy = fmaf(fc5, di, fmaf(fc4, dj, yo_f));
    const float flx = floorf(fx), fly = floorf(fy);
    // inside [0, win - 2] by the planner's window bound; the clamp only keeps a mis-sized call inside shared memory
    const int x0 = min(max(dx0 + (int)flx, 0), win_w - 2), y0 = min(max(dy0 + (int)fly, 0), win_h - 2);
    pidx[p] = y0 * win_w + x0;
    pwx[p] = fx - flx;
    pwy[p] = fy - fly;
  }
  const int r0 = (yw - 6) >> 1, s0 = (xw - 6) >> 1;          // first padded input row / column of the input window
  for (int t = tid; t < in_h; t += AUG_THREADS) rmap[t] = aug_src(r0 + t, Hp, pad_y, H);
  for (int t = tid; t < in_w; t += AUG_THREADS) cmap[t] = aug_src(s0 + t, Wp, pad_x, W);
  if (tid < AUG_TAPS) k[tid] = kern[tid];
  __syncthreads();

  const int64_t plane = (int64_t)H * W;
  for (int c = 0; c < C; ++c) {
    const float* __restrict__ src = in + ((int64_t)b * C + c) * plane;
    for (int t = tid; t < in_h * in_w; t += AUG_THREADS) {
      const int sr = rmap[t / in_w], sc = cmap[t % in_w];
      buf1[t] = (sr >= 0 && sc >= 0) ? __ldg(src + (int64_t)sr * W + sc) : 0.f;
    }
    __syncthreads();
    // up, x: buf2[r][u] = x2 column X = xw + u of input-window row r
    for (int t = tid; t < in_h * win_w; t += AUG_THREADS) {
      const int r = t / win_w, u = t % win_w, X = xw + u, par = X & 1;
      const float* row = buf1 + r * in_w + (((X - 6 + par) >> 1) - s0);
      float acc = 0.f;
#pragma unroll
      for (int m = 0; m < 6; ++m) acc = fmaf(k[AUG_TAPS - 1 - 2 * m - par], row[m], acc);
      buf2[t] = acc;
    }
    __syncthreads();
    // up, y: buf1[v][u] = x2 sample (yw + v, xw + u), zero outside the x2 image (grid_sample's zeros padding)
    for (int t = tid; t < win_h * win_w; t += AUG_THREADS) {
      const int v = t / win_w, u = t % win_w, X = xw + u, Y = yw + v;
      float acc = 0.f;
      if (X >= 0 && X < 2 * Wp && Y >= 0 && Y < 2 * Hp) {
        const int par = Y & 1;
        const float* col = buf2 + (((Y - 6 + par) >> 1) - r0) * win_w + u;
#pragma unroll
        for (int m = 0; m < 6; ++m) acc = fmaf(k[AUG_TAPS - 1 - 2 * m - par], col[m * win_w], acc);
      }
      buf1[t] = acc;
    }
    __syncthreads();
    // warp: buf2[p] = bilinear sample of the block point p
    for (int p = tid; p < NB * NB; p += AUG_THREADS) {
      const float* q = buf1 + pidx[p];
      const float wx = pwx[p], wy = pwy[p];
      buf2[p] = (1.f - wx) * (1.f - wy) * q[0] + wx * (1.f - wy) * q[1] + (1.f - wx) * wy * q[win_w] + wx * wy * q[win_w + 1];
    }
    __syncthreads();
    // down, x: buf1[row][ox] = sum_t k[t] A[row][2 ox + t]
    for (int t = tid; t < NB * T; t += AUG_THREADS) {
      const int row = t / T, ox = t % T;
      const float* a = buf2 + row * NB + 2 * ox;
      float acc = 0.f;
#pragma unroll
      for (int m = 0; m < AUG_TAPS; ++m) acc = fmaf(k[m], a[m], acc);
      buf1[t] = acc;
    }
    __syncthreads();
    // down, y, and the store
    float* __restrict__ dst = out + ((int64_t)b * C + c) * plane;
    for (int t = tid; t < T * T; t += AUG_THREADS) {
      const int oy = t / T, ox = t % T;
      const float* d = buf1 + 2 * oy * T + ox;
      float acc = 0.f;
#pragma unroll
      for (int m = 0; m < AUG_TAPS; ++m) acc = fmaf(k[m], d[m * T], acc);
      if (ty0 + oy < H && tx0 + ox < W) dst[(int64_t)(ty0 + oy) * W + tx0 + ox] = acc;
    }
    __syncthreads();
  }
}

template <int T>
int aug_launch(const float* in, float* out, const float* kernel, const double* coef, int B, int C, int H, int W, int pad_x, int pad_y,
               int Hp, int Wp, int win_w, int win_h, cudaStream_t st) {
  const int tiles_x = (int)vt_cdiv(W, T), tiles_y = (int)vt_cdiv(H, T);
  VT_CHECK((int64_t)tiles_x * tiles_y <= 0x7fffffff, "vt_augment_affine_f32: %d x %d is too large", H, W);
  const int64_t smem = AugLayout(T, win_w, win_h).bytes();
  VT_CUDA(cudaFuncSetAttribute(augment_affine_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, AUG_SMEM_BUDGET));
  augment_affine_kernel<T><<<dim3(tiles_x * tiles_y, B), AUG_THREADS, smem, st>>>(in, out, kernel, coef, C, H, W, pad_x, pad_y, Hp, Wp,
                                                                                    tiles_x, win_w, win_h);
  VT_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" {

int vt_augment_affine_plan(const double* coef, int B, int H, int W, int* win) {
  if (coef == nullptr || B < 1 || H < 1 || W < 1) {
    vt_set_error("vt_augment_affine_plan: bad arguments (B=%d H=%d W=%d)", B, H, W);
    return -1;
  }
  for (int T = 16; T >= 8; T /= 2) {
    const int nb = 2 * T + 10;
    // the last warp-grid sample any tile computes, partial tiles included
    const double jmax = 2.0 * vt_cdiv(W, T) * T + 10, imax = 2.0 * vt_cdiv(H, T) * T + 10;
    double span_x = 0.0, span_y = 0.0;
    bool ok = true;
    for (int b = 0; b < B && ok; ++b) {
      const double* c = coef + 6 * (int64_t)b;
      for (int q = 0; q < 4; ++q) {
        const double j = (q & 1) ? jmax : 0.0, i = (q & 2) ? imax : 0.0;
        const double x = c[0] + c[1] * j + c[2] * i, y = c[3] + c[4] * j + c[5] * i;
        ok = ok && fabs(x) < AUG_COORD_LIMIT && fabs(y) < AUG_COORD_LIMIT;   // false for inf and NaN too
      }
      span_x = fmax(span_x, (fabs(c[1]) + fabs(c[2])) * (nb - 1));
      span_y = fmax(span_y, (fabs(c[4]) + fabs(c[5])) * (nb - 1));
    }
    if (!ok) return 0;
    // floor(max) - floor(min) <= ceil(span); plus the one-sample margin before the origin, the bilinear neighbour, and one sample for
    // the fp32 rounding of the per-point offsets
    const int win_w = (int)ceil(span_x) + 4, win_h = (int)ceil(span_y) + 4;
    if (AugLayout(T, win_w, win_h).bytes() <= AUG_SMEM_BUDGET) {
      if (win) { win[0] = win_w; win[1] = win_h; }
      return T;
    }
  }
  return 0;
}

int vt_augment_affine_f32(const float* in, float* out, const float* kernel, const double* coef, int B, int C, int H, int W, int pad_x,
                          int pad_y, int Hp, int Wp, int tile, int win_w, int win_h, void* stream) {
  VT_CHECK(in && out && kernel && coef, "vt_augment_affine_f32: null pointer");
  VT_CHECK(B >= 1 && B <= 65535 && C >= 1 && H >= 1 && W >= 1, "vt_augment_affine_f32: bad shape B=%d C=%d H=%d W=%d", B, C, H, W);
  VT_CHECK(pad_x >= 0 && pad_y >= 0 && pad_x < W && pad_y < H && Wp - W - pad_x >= 0 && Wp - W - pad_x < W && Hp - H - pad_y >= 0 &&
               Hp - H - pad_y < H,
           "vt_augment_affine_f32: reflect pads must be in [0, size - 1] (H=%d W=%d Hp=%d Wp=%d pad_x=%d pad_y=%d)", H, W, Hp, Wp,
           pad_x, pad_y);
  VT_CHECK(tile == 8 || tile == 16, "vt_augment_affine_f32: tile %d is not one vt_augment_affine_plan returns", tile);
  VT_CHECK(win_w >= 2 && win_h >= 2 && AugLayout(tile, win_w, win_h).bytes() <= AUG_SMEM_BUDGET,
           "vt_augment_affine_f32: window %d x %d does not fit tile %d", win_w, win_h, tile);
  cudaStream_t st = (cudaStream_t)stream;
  if (tile == 16) return aug_launch<16>(in, out, kernel, coef, B, C, H, W, pad_x, pad_y, Hp, Wp, win_w, win_h, st);
  return aug_launch<8>(in, out, kernel, coef, B, C, H, W, pad_x, pad_y, Hp, Wp, win_w, win_h, st);
}

}  // extern "C"
