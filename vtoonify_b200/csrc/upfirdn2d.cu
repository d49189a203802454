// upfirdn2d.cu — planar (NCHW) upsample / pad-crop / 2-D FIR / downsample in one pass.
//
// Semantics follow the reference CPU spec model/stylegan/op_cpu/upfirdn2d.py:19-60 and the CUDA
// op model/stylegan/op/upfirdn2d_kernel.cu:49-105 (generic kernel): zero-stuff by `up`, pad (negative
// pad crops), true convolution (kernel flipped), keep every `down`-th sample.  Written from the maths:
//   out[p,oy,ox] = sum_{ky,kx} U[p, oy*down_y + ky - pad_y0, ox*down_x + kx - pad_x0] * k[kh-1-ky][kw-1-kx]
//   U[p,u,v] = in[p,u/up_y,v/up_x] if up_y|u, up_x|v and inside, else 0.
// All offsets are 64-bit (the reference kernels overflow 32-bit ints at 576x1024 B>=8).
//
// Two kernels:
//   * upfirdn2d_generic_kernel : any (up, down, pad, kh, kw); one output per thread.
//   * upfirdn2d_tiled_kernel   : same semantics, the input window of a 32 x 64 output tile staged once in shared memory
//     (coalesced), division-free tap loops; used whenever the window fits (all hot-path instances).
#include "tc_common.cuh"

using namespace vt_tc;

int g_upfirdn_tiled = 2;   // 2: streaming kernel for the 4x4 instances (default); 1: staged-tile kernels; 0 forces the generic kernel (tests compare all)

namespace {

constexpr int kMaxSmemTaps = 1024;

__global__ void __launch_bounds__(256)
upfirdn2d_generic_kernel(const float* __restrict__ in, const float* __restrict__ kernel, float* __restrict__ out,
                         int64_t planes, int in_h, int in_w, int out_h, int out_w, int kh, int kw,
                         int up_x, int up_y, int down_x, int down_y, int pad_x0, int pad_y0, int taps_in_smem) {
  __shared__ float sk[kMaxSmemTaps];
  if (taps_in_smem) {
    for (int i = threadIdx.x; i < kh * kw; i += blockDim.x) sk[i] = kernel[i];
    __syncthreads();
  }
  const float* kp = taps_in_smem ? sk : kernel;
  const int64_t total = planes * (int64_t)out_h * out_w;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % out_w);
    const int64_t t1 = idx / out_w;
    const int oy = (int)(t1 % out_h);
    const int64_t p = t1 / out_h;
    const int ty = oy * down_y - pad_y0;  // position of tap ky=0 in the zero-stuffed signal
    const int tx = ox * down_x - pad_x0;
    int ky0, kx0;
    if (ty >= 0) { int r = ty % up_y; ky0 = r ? up_y - r : 0; } else { ky0 = -ty; }
    if (tx >= 0) { int r = tx % up_x; kx0 = r ? up_x - r : 0; } else { kx0 = -tx; }
    const float* ip = in + p * (int64_t)in_h * in_w;
    float acc = 0.f;
    for (int ky = ky0; ky < kh; ky += up_y) {
      const int iy = (ty + ky) / up_y;
      if (iy >= in_h) break;
      const float* row = ip + (int64_t)iy * in_w;
      const float* krow = kp + (kh - 1 - ky) * kw;
      for (int kx = kx0; kx < kw; kx += up_x) {
        const int ix = (tx + kx) / up_x;
        if (ix >= in_w) break;
        acc += __ldg(row + ix) * krow[kw - 1 - kx];
      }
    }
    out[idx] = acc;
  }
}

// ---- tiled fast path -----------------------------------------------------------------------------------------------
// A block owns a TOH x TOW output tile of one plane: the input window it needs (with zero halo) is staged once in
// shared memory by coalesced row reads, then each thread walks a column of the tile.  Tap index arithmetic is hoisted:
// the first contributing tap and its input column depend only on the thread's output column, (tx + kx) / up_x advances
// by exactly one input pixel per step of up_x taps, so there is no division in the tap loops.  HBM traffic is the
// algorithmic read-once / write-once (the generic kernel re-reads every input ~kh*kw/(up*up) times through L1/L2).
constexpr int T_OW = 64, T_OH = 32, T_ROWS_PER_THREAD = T_OH / 4;   // 256 threads = 64 columns x 4 row groups

__global__ void __launch_bounds__(256)
upfirdn2d_tiled_kernel(const float* __restrict__ in, const float* __restrict__ kernel, float* __restrict__ out,
                       int in_h, int in_w, int out_h, int out_w, int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                       int pad_x0, int pad_y0, int tiles_x, int tile_rows, int tile_cols) {
  extern __shared__ float smem[];
  float* sk = smem;                        // flipped kernel [kh][kw]
  float* S = smem + kh * kw;               // input window [tile_rows][tile_cols]
  for (int i = threadIdx.x; i < kh * kw; i += blockDim.x) sk[i] = kernel[(kh - 1 - i / kw) * kw + (kw - 1 - i % kw)];
  const int64_t plane = blockIdx.y;
  const int oy0 = (blockIdx.x / tiles_x) * T_OH, ox0 = (blockIdx.x % tiles_x) * T_OW;
  // first input row / column any output of this tile can touch (floor division, may be negative -> zero halo)
  const int uy0 = oy0 * down_y - pad_y0, ux0 = ox0 * down_x - pad_x0;
  const int iy_base = (uy0 >= 0) ? uy0 / up_y : -((-uy0 + up_y - 1) / up_y);
  const int ix_base = (ux0 >= 0) ? ux0 / up_x : -((-ux0 + up_x - 1) / up_x);
  const float* ip = in + plane * (int64_t)in_h * in_w;
  for (int i = threadIdx.x; i < tile_rows * tile_cols; i += blockDim.x) {
    const int r = i / tile_cols, c = i - r * tile_cols;
    const int iy = iy_base + r, ix = ix_base + c;
    S[i] = (iy >= 0 && iy < in_h && ix >= 0 && ix < in_w) ? __ldg(ip + (int64_t)iy * in_w + ix) : 0.f;
  }
  __syncthreads();
  const int c = threadIdx.x & (T_OW - 1), rg = threadIdx.x / T_OW;
  const int ox = ox0 + c;
  if (ox >= out_w) return;
  // column taps: kx = kx0, kx0 + up_x, ... ; input column (tx + kx) / up_x = sx0, sx0 + 1, ...  (relative to the window)
  const int tx = ox * down_x - pad_x0;
  int kx0;
  if (tx >= 0) { const int r = tx % up_x; kx0 = r ? up_x - r : 0; } else { const int r = (-tx) % up_x; kx0 = r; }
  // (tx + kx0) is a multiple of up_x; it may be negative (zero halo covers it)
  const int sx0 = ((tx + kx0) >= 0 ? (tx + kx0) / up_x : -((-(tx + kx0)) / up_x)) - ix_base;
  float* op = out + plane * (int64_t)out_h * out_w;
  for (int j = 0; j < T_ROWS_PER_THREAD; ++j) {
    const int oy = oy0 + rg * T_ROWS_PER_THREAD + j;
    if (oy >= out_h) break;
    const int ty = oy * down_y - pad_y0;
    int ky0;
    if (ty >= 0) { const int r = ty % up_y; ky0 = r ? up_y - r : 0; } else { ky0 = (-ty) % up_y; }
    int sy = ((ty + ky0) >= 0 ? (ty + ky0) / up_y : -((-(ty + ky0)) / up_y)) - iy_base;
    float acc = 0.f;
    for (int ky = ky0; ky < kh; ky += up_y, ++sy) {
      const float* srow = S + sy * tile_cols + sx0;
      const float* krow = sk + ky * kw;
      int sx = 0;
      for (int kx = kx0; kx < kw; kx += up_x, ++sx) acc = fmaf(srow[sx], krow[kx], acc);
    }
    op[(int64_t)oy * out_w + ox] = acc;
  }
}

// ---- 4x4-kernel specialisation (the hot-path instances: Blur pad(1,1)/(2,2), Upsample up=2 pad(2,1), Downsample down=2) ----
// 32 x 128 output tile per block, each thread owns a 4 x 4 output micro-tile.  UP/DOWN are compile-time (one of them is 1),
// the input window is staged in shared memory row by row (one warp per row, coalesced, no index division) and pulled
// into registers once per micro-tile, so a thread issues ~20-30 shared loads and 64-256 FMAs for 16 outputs.
constexpr int K4_OW = 128, K4_OH = 32;

template <int UP, int DOWN>
__global__ void __launch_bounds__(256)
upfirdn2d_k4_kernel(const float* __restrict__ in, const float* __restrict__ kernel, float* __restrict__ out, int in_h,
                    int in_w, int out_h, int out_w, int pad_x0, int pad_y0, int tiles_x) {
  constexpr int WR = ((K4_OH - 1) * DOWN + 3) / UP + 2;      // window rows / cols (upper bounds)
  constexpr int WC = (((K4_OW - 1) * DOWN + 3) / UP + 2 + 3) / 4 * 4;
  extern __shared__ __align__(16) float S[];                  // [WR][WC]
  __shared__ float sk[16];                                    // flipped kernel
  if (threadIdx.x < 16) sk[threadIdx.x] = kernel[(3 - threadIdx.x / 4) * 4 + (3 - threadIdx.x % 4)];
  const int64_t plane = blockIdx.y;
  const int oy0 = (blockIdx.x / tiles_x) * K4_OH, ox0 = (blockIdx.x % tiles_x) * K4_OW;
  const int uy0 = oy0 * DOWN - pad_y0, ux0 = ox0 * DOWN - pad_x0;      // first zero-stuffed coordinate of the tile
  // floor(u / UP) for possibly negative u (UP is 1 or 2)
  const int iy_base = (UP == 1) ? uy0 : (uy0 >> 1), ix_base = (UP == 1) ? ux0 : (ux0 >> 1);
  const float* ip = in + plane * (int64_t)in_h * in_w;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < WR; r += 8) {
    const int iy = iy_base + r;
    const bool row_ok = iy >= 0 && iy < in_h;
    const float* row = ip + (int64_t)iy * in_w;
    for (int c = lane; c < WC; c += 32) {
      const int ix = ix_base + c;
      S[r * WC + c] = (row_ok && ix >= 0 && ix < in_w) ? __ldg(row + ix) : 0.f;
    }
  }
  __syncthreads();
  float k[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) k[i] = sk[i];
  const int cg = threadIdx.x & 31, rg = threadIdx.x >> 5;     // 32 column groups x 8 row groups, 4 x 4 outputs each
  const int oxl = cg * 4, oyl = rg * 4;
  float acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[j][i] = 0.f;
  if (UP == 1) {
    // u = o*DOWN + k - pad  ->  window row (oyl+j)*DOWN + ky, window col (oxl+i)*DOWN + kx
    constexpr int NR = 3 * DOWN + 4, NC = 3 * DOWN + 4;        // 7 (blur) or 10 (downsample)
    float w[NR][NC];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      const float* sp = S + (oyl * DOWN + r) * WC + oxl * DOWN;   // oxl*DOWN is a multiple of 4: float4 loads
#pragma unroll
      for (int c4 = 0; c4 < NC / 4; ++c4) {
        const float4 v = *reinterpret_cast<const float4*>(sp + c4 * 4);
        w[r][c4 * 4] = v.x; w[r][c4 * 4 + 1] = v.y; w[r][c4 * 4 + 2] = v.z; w[r][c4 * 4 + 3] = v.w;
      }
#pragma unroll
      for (int c = NC / 4 * 4; c < NC; ++c) w[r][c] = sp[c];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int ky = 0; ky < 4; ++ky)
#pragma unroll
          for (int kx = 0; kx < 4; ++kx) acc[j][i] = fmaf(w[j * DOWN + ky][i * DOWN + kx], k[ky * 4 + kx], acc[j][i]);
  } else {
    // UP == 2, DOWN == 1: output o uses taps k = p, p + 2 with p = (o - pad) & 1 and inputs (o - pad + p) >> 1, +1
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ty = oy0 + oyl + j - pad_y0;
      const int py = ty & 1;
      const int sy = ((ty + py) >> 1) - iy_base;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int tx = ox0 + oxl + i - pad_x0;
        const int px = tx & 1;
        const int sx = ((tx + px) >> 1) - ix_base;
        const float* sp = S + sy * WC + sx;
        const float k00 = px ? (py ? k[5] : k[1]) : (py ? k[4] : k[0]);
        const float k01 = px ? (py ? k[7] : k[3]) : (py ? k[6] : k[2]);
        const float k10 = px ? (py ? k[13] : k[9]) : (py ? k[12] : k[8]);
        const float k11 = px ? (py ? k[15] : k[11]) : (py ? k[14] : k[10]);
        float a = sp[0] * k00;
        a = fmaf(sp[1], k01, a);
        a = fmaf(sp[WC], k10, a);
        a = fmaf(sp[WC + 1], k11, a);
        acc[j][i] = a;
      }
    }
  }
  float* op = out + plane * (int64_t)out_h * out_w;
  const int ox = ox0 + oxl;
  const bool vec = (out_w % 4 == 0) && ((reinterpret_cast<uintptr_t>(op) & 15) == 0) && (ox + 3 < out_w);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int oy = oy0 + oyl + j;
    if (oy >= out_h) break;
    float* orow = op + (int64_t)oy * out_w + ox;
    if (vec) {
      *reinterpret_cast<float4*>(orow) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (ox + i < out_w) orow[i] = acc[j][i];
    }
  }
}

template <int UP, int DOWN>
int launch_k4(const float* in, const float* kernel, float* out, int64_t planes, int in_h, int in_w, int out_h, int out_w,
              int pad_x0, int pad_y0, cudaStream_t st) {
  constexpr int WR = ((K4_OH - 1) * DOWN + 3) / UP + 2;
  constexpr int WC = (((K4_OW - 1) * DOWN + 3) / UP + 2 + 3) / 4 * 4;
  const size_t smem = (size_t)WR * WC * sizeof(float);
  if (smem > 48 * 1024)
    VT_CUDA(cudaFuncSetAttribute(upfirdn2d_k4_kernel<UP, DOWN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int tiles_x = (int)vt_cdiv(out_w, K4_OW), tiles_y = (int)vt_cdiv(out_h, K4_OH);
  dim3 grid((unsigned)(tiles_x * tiles_y), (unsigned)planes);
  upfirdn2d_k4_kernel<UP, DOWN><<<grid, 256, smem, st>>>(in, kernel, out, in_h, in_w, out_h, out_w, pad_x0, pad_y0, tiles_x);
  return 0;
}


// ---- streaming 4x4 kernel (default for the StyleGAN instances: Blur, Upsample x2, Downsample /2) ---------------------------
// The k4 kernel above stages a tile with per-lane 4-byte loads, waits, computes, stores: at most ~20 KB in flight per SM and
// 0.35 of the HBM roof.  Here a block walks a column strip of one plane from top to bottom:
//   * a producer warp streams the input rows of the strip into a shared-memory ring with 1-D bulk async copies
//     (cp.async.bulk, completion on an mbarrier; lane rr issues row rr of a stage): a row segment is contiguous in a planar
//     tensor, so no tensor map (and no 16-byte row pitch, which [.., 1025, 1025] planes do not have) is needed - the copy
//     starts at the 16-byte boundary below the segment and the consumers add the row's 0..3-float lead to their column
//     index.  ~68 KB are in flight per block, no registers or LSU slots are spent on the loads.  Rows in the zero padding
//     are written as zeros by the producer warp; a copy that would touch bytes outside the tensor (only the first / last
//     row of the whole tensor) is done with ordinary predicated loads instead.
//   * the consumer threads keep the vertical taps' partial sums in registers while the rows stream by, so every input
//     element comes from HBM once.  Blur and Upsample: a thread owns 4 (8) adjacent output columns, reads its 7 (6) inputs of
//     a row as three aligned 16-byte shared loads (the row's lead decides which of the 12 registers are used - a uniform
//     4-way branch) and stores 16 bytes per output row: 13 (6) instructions per output instead of 44 (the first, one
//     column per thread version was issue-bound at 0.46 of the HBM roof).  A rank-1 blur kernel (every StyleGAN filter:
//     outer([1,3,3,1])) is applied separably: 4 FMAs for the row filter + 4 for the column filter per output instead of 16.
//     Downsample: one output column per thread (4 scalar loads per input row, 2 input rows per output).
// Output rows go straight from registers to global memory (consecutive lanes -> consecutive 16-byte / 4-byte pieces).
constexpr int US_RS = 8;                   // input rows per ring stage
constexpr int US_STAGES = 4;

template <int UP, int DOWN> struct UsCfg;
template <> struct UsCfg<1, 1> { static constexpr int NCONS = 128, OWT = 512, COUNT = 515; };    // 4 output columns per thread
template <> struct UsCfg<2, 1> { static constexpr int NCONS = 128, OWT = 1024, COUNT = 514; };   // 8 output columns (4 inputs) per thread
template <> struct UsCfg<1, 2> { static constexpr int NCONS = 256, OWT = 256, COUNT = 514; };    // 1 output column per thread

struct UsArgs {
  const float* in; const float* kernel; float* out;
  int64_t planes, total_items;
  int in_h, in_w, out_h, out_w, pad_x0, pad_y0;
  int strips, chunks, rows_per_chunk;
  int row_stride;                          // ring: US_STAGES x US_RS rows x row_stride floats
};

__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// geometry of a work item (plane, row chunk, column strip): identical arithmetic in the producer and the consumers
template <int UP, int DOWN>
struct UsItem {
  int64_t plane;
  int oy_a, oy_b, ox0;       // output rows [oy_a, oy_b), first output column
  int iy_first, n_rows;      // input rows streamed: iy_first .. iy_first + n_rows - 1 (may lie in the padding)
  int ix0;                   // input column of ring column offset 0 (may be negative)
  int ix_lo, n_cols;         // columns actually copied: [ix_lo, ix_lo + n_cols) inside [0, in_w)
  int colbase;               // ring column of input column ix0 (before the per-row lead)
  __device__ __forceinline__ UsItem(const UsArgs& p, int64_t item) {
    using C = UsCfg<UP, DOWN>;
    const int strip = (int)(item % p.strips);
    const int64_t t = item / p.strips;
    const int chunk = (int)(t % p.chunks);
    plane = t / p.chunks;
    oy_a = chunk * p.rows_per_chunk;
    oy_b = min(oy_a + p.rows_per_chunk, p.out_h);
    ox0 = strip * C::OWT;
    if (UP == 1) {
      iy_first = oy_a * DOWN - p.pad_y0;
      n_rows = (oy_b - 1 - oy_a) * DOWN + 4;
      ix0 = ox0 * DOWN - p.pad_x0;
    } else {
      const int ty_a = oy_a - p.pad_y0, ty_l = oy_b - 1 - p.pad_y0;
      iy_first = (ty_a + (ty_a & 1)) >> 1;
      n_rows = ((ty_l + (ty_l & 1)) >> 1) + 1 - iy_first + 1;
      const int tx0 = ox0 - p.pad_x0;
      ix0 = (tx0 + (tx0 & 1)) >> 1;
    }
    ix_lo = max(ix0, 0);
    n_cols = min(ix0 + C::COUNT, p.in_w) - ix_lo;
    colbase = ((ix_lo - ix0 + 3) & ~3) - (ix_lo - ix0);   // D + (ix0 - ix_lo) with D = roundup(ix_lo - ix0, 4)
  }
};

// ---- Blur (UP = DOWN = 1), one input row, 4 adjacent output columns per thread.  u = three aligned float4 of the ring row, the
// thread's 7 inputs are u[SH .. SH + 6].  Input row r feeds the four output rows r - ky; the accumulator of an output row starts
// with its first tap (ky = 0: a multiply, no clearing needed) and is stored after its last (ky = 3).
template <bool SEP, int RR, int SH>
__device__ __forceinline__ void us_blur_row4(const float4* sp4, unsigned mbits, const float (&kf)[16], const float (&ay)[4],
                                             const float (&bx)[4], float (&acc)[4][4]) {
  float u[12];
  {
    const float4 a = sp4[0], b = sp4[1];
    u[0] = a.x; u[1] = a.y; u[2] = a.z; u[3] = a.w; u[4] = b.x; u[5] = b.y; u[6] = b.z; u[7] = b.w;
    if (SH >= 2) { const float4 c = sp4[2]; u[8] = c.x; u[9] = c.y; u[10] = c.z; u[11] = c.w; }
  }
  float v[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) v[i] = ((mbits >> i) & 1u) ? u[SH + i] : 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (SEP) {
      float h = bx[0] * v[c];
      h = fmaf(bx[1], v[c + 1], h); h = fmaf(bx[2], v[c + 2], h); h = fmaf(bx[3], v[c + 3], h);
      acc[c][RR & 3] = ay[0] * h;
#pragma unroll
      for (int ky = 1; ky < 4; ++ky) acc[c][(RR - ky) & 3] = fmaf(ay[ky], h, acc[c][(RR - ky) & 3]);
    } else {
#pragma unroll
      for (int ky = 0; ky < 4; ++ky) {
        float a = ky ? acc[c][(RR - ky) & 3] : 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) a = fmaf(kf[ky * 4 + i], v[c + i], a);
        acc[c][(RR - ky) & 3] = a;
      }
    }
  }
}

// ---- Upsample (UP = 2), one input row (the second of the two an output row needs), 8 adjacent output columns per thread.
// The thread's inputs are u[SH .. SH + 5] (cv) and the same columns of the previous row (pv).  Output column n of the thread:
// parity q = (tx0 + n) & 1, first input column f = (n + 1 - Q0) >> 1 (Q0 = tx0 & 1, the same for every thread of the launch).
// y[e][n]: e = 0 -> output row 2*iy - 3 + pad (taps ky = 1, 3), e = 1 -> the next one (ky = 0, 2);  w[e][q] = {kf[kyf][q], kf[kyf][q+2],
// kf[kys][q], kf[kys][q+2]}.
template <int Q0, int SH>
__device__ __forceinline__ void us_up_row8(const float4* sp4, unsigned mbits, const float (&w)[2][2][4], float (&pv)[6], float (&y)[2][8]) {
  float u[12];
  {
    const float4 a = sp4[0], b = sp4[1];
    u[0] = a.x; u[1] = a.y; u[2] = a.z; u[3] = a.w; u[4] = b.x; u[5] = b.y; u[6] = b.z; u[7] = b.w;
    if (SH >= 3) { const float4 c = sp4[2]; u[8] = c.x; u[9] = c.y; u[10] = c.z; u[11] = c.w; }
  }
  float cv[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) cv[i] = ((mbits >> i) & 1u) ? u[SH + i] : 0.f;
#pragma unroll
  for (int e = 0; e < 2; ++e)
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const int q = (Q0 + n) & 1, f = (n + 1 - Q0) >> 1;
      float t = w[e][q][0] * pv[f];
      t = fmaf(w[e][q][1], pv[f + 1], t); t = fmaf(w[e][q][2], cv[f], t); t = fmaf(w[e][q][3], cv[f + 1], t);
      y[e][n] = t;
    }
#pragma unroll
  for (int i = 0; i < 6; ++i) pv[i] = cv[i];
}

template <int UP, int DOWN>
__global__ void __launch_bounds__(UsCfg<UP, DOWN>::NCONS + 32)
upfirdn2d_stream_kernel(const __grid_constant__ UsArgs p) {
  using C = UsCfg<UP, DOWN>;
  constexpr int NCONS = C::NCONS;
  extern __shared__ __align__(128) float ring[];
  __shared__ __align__(8) uint64_t bars[2 * US_STAGES];
  __shared__ float sk[16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + (uint32_t)s * 8u; };
  auto empty_bar = [&](int s) { return bar0 + (uint32_t)(US_STAGES + s) * 8u; };
  if (threadIdx.x == 0) {
    // every thread that writes / reads a ring row through the generic proxy arrives itself (no lane-0 proxies: the ordering is then
    // explicit per thread, and compute-sanitizer's racecheck can follow it)
    for (int s = 0; s < US_STAGES; ++s) { mbar_init(full_bar(s), 32); mbar_init(empty_bar(s), NCONS); }
    fence_barrier_init();
  }
  if (threadIdx.x < 16) sk[threadIdx.x] = p.kernel[(3 - threadIdx.x / 4) * 4 + (3 - threadIdx.x % 4)];   // flipped: true convolution
  __syncthreads();
  const int64_t plane_elems = (int64_t)p.in_h * p.in_w;
  const int stage_floats = US_RS * p.row_stride;

  if (warp == NCONS / 32) {
    // ================= producer warp: lane rr prepares and issues the copy of row rr of the stage =================
    const uintptr_t t_begin = reinterpret_cast<uintptr_t>(p.in);
    const uintptr_t t_end = t_begin + (uintptr_t)(p.planes * plane_elems) * 4u;
    uint32_t it = 0;
    for (int64_t item = blockIdx.x; item < p.total_items; item += gridDim.x) {
      const UsItem<UP, DOWN> g(p, item);
      const int n_st = (g.n_rows + US_RS - 1) / US_RS;
      const int D = g.colbase + (g.ix_lo - g.ix0);         // multiple of 4 floats: the copies land 16-byte aligned
      const int64_t e_item = (g.plane * p.in_h + g.iy_first) * (int64_t)p.in_w + g.ix_lo;
      for (int s = 0; s < n_st; ++s, ++it) {
        const int slot = (int)(it % (uint32_t)US_STAGES);
        const uint32_t ph = (it / (uint32_t)US_STAGES) & 1u;
        mbar_wait(empty_bar(slot), ph ^ 1u);
        float* const sstage = ring + (size_t)slot * stage_floats;
        const int r = s * US_RS + lane;
        const int iy = g.iy_first + r;
        // 0: nothing (past the item: the consumers discard what they compute from the stale row), 1: bulk copy, 2: zero padding,
        // 3: copy that would touch bytes outside the tensor (its first / last row): ordinary loads
        int kind = 0;
        uint32_t nbytes = 0, lead = 0;
        int64_t e = 0;
        if (lane < US_RS && r < g.n_rows) {
          if (iy < 0 || iy >= p.in_h || g.n_cols <= 0) kind = 2;
          else {
            e = e_item + (int64_t)r * p.in_w;
            const uintptr_t addr = t_begin + (uintptr_t)e * 4u;
            const uintptr_t addr_al = addr & ~(uintptr_t)15;
            lead = (uint32_t)(addr - addr_al) >> 2;
            nbytes = ((lead + (uint32_t)g.n_cols) * 4u + 15u) & ~15u;
            if (addr_al >= t_begin && addr_al + nbytes <= t_end) {
              kind = 1;
              bulk_load_1d(smem_u32(sstage + (size_t)lane * p.row_stride + D), reinterpret_cast<const void*>(addr_al), nbytes, full_bar(slot));
            } else { kind = 3; nbytes = 0; }
          }
        }
        uint32_t bytes = kind == 1 ? nbytes : 0u;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);   // lanes 0..7 hold the rows
        unsigned zmask = __ballot_sync(0xffffffffu, kind == 2), emask = __ballot_sync(0xffffffffu, kind == 3);
        while (zmask) {
          const int rr = __ffs(zmask) - 1; zmask &= zmask - 1;
          float* srow = sstage + (size_t)rr * p.row_stride;
          for (int c = lane; c < p.row_stride; c += 32) srow[c] = 0.f;
        }
        while (emask) {
          const int rr = __ffs(emask) - 1; emask &= emask - 1;
          const int64_t er = __shfl_sync(0xffffffffu, e, rr);
          const int ld = (int)__shfl_sync(0xffffffffu, lead, rr);
          float* srow = sstage + (size_t)rr * p.row_stride + D + ld;
          for (int c = lane; c < g.n_cols; c += 32) srow[c] = __ldg(p.in + er + c);
        }
        if (lane == 0) mbar_arrive_expect_tx(full_bar(slot), bytes); else mbar_arrive(full_bar(slot));
      }
    }
    return;
  }

  // ================= consumers =================
  const int tid = threadIdx.x;
  float kf[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) kf[i] = sk[i];
  // rank-1 test (UP == DOWN == 1 only): kf = ay (x) bx with bx normalised by the smallest non-zero entry of the pivot row, so that
  // integer-ratio filters ([1,3,3,1]) factor exactly
  bool sep = false;
  float ay[4] = {0.f, 0.f, 0.f, 0.f}, bx[4] = {0.f, 0.f, 0.f, 0.f};
  if (UP == 1 && DOWN == 1) sep = vt_rank1_4x4(sk, ay, bx);
  const unsigned in_addr_lo = (unsigned)((reinterpret_cast<uintptr_t>(p.in) >> 2) & 3u);
  const bool out16 = (reinterpret_cast<uintptr_t>(p.out) & 15u) == 0 && (p.out_w & 3) == 0;

  uint32_t it = 0;
  for (int64_t item = blockIdx.x; item < p.total_items; item += gridDim.x) {
    const UsItem<UP, DOWN> g(p, item);
    const int n_st = (g.n_rows + US_RS - 1) / US_RS;
    // ring column of input column ix0 in row r: colbase + lead(r), lead(r) = ((in >> 2) + e_row) & 3 with
    // e_row = (plane*in_h + iy_first + r)*in_w + ix_lo; only the low two bits matter, so the running sum may wrap
    unsigned lead_acc = (unsigned)(((g.plane * p.in_h + g.iy_first) * (int64_t)p.in_w + g.ix_lo) & 3) + in_addr_lo;
    const unsigned in_w_u = (unsigned)p.in_w;
    float* const oplane = p.out + g.plane * (int64_t)p.out_h * p.out_w;

    if (UP == 1 && DOWN == 1) {
      const int ox = g.ox0 + 4 * tid;
      unsigned mbits = 0;
#pragma unroll
      for (int i = 0; i < 7; ++i) { const int ix = g.ix0 + 4 * tid + i; mbits |= (ix >= 0 && ix < p.in_w) ? (1u << i) : 0u; }
      float acc[4][4];
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[c][k] = 0.f;
      // input row r completes output row oy_a + r - 3: stored for 3 <= r < n_rows
      int64_t oidx = (int64_t)(g.oy_a - 3) * p.out_w + ox;
      const unsigned r_span = (unsigned)(g.n_rows - 3);
      const bool vec = out16 && ox + 3 < p.out_w;
      for (int s = 0; s < n_st; ++s, ++it) {
        const int slot = (int)(it % (uint32_t)US_STAGES);
        mbar_wait(full_bar(slot), (it / (uint32_t)US_STAGES) & 1u);
        const float* srow = ring + (size_t)slot * stage_floats + 4 * tid;
        const int r0 = s * US_RS - 3;
#define US_BLUR_ROW(SEPV, RRV)                                                                                   \
        switch (off & 3u) {                                                                                      \
          case 0: us_blur_row4<SEPV, RRV, 0>(sp4, mbits, kf, ay, bx, acc); break;                                \
          case 1: us_blur_row4<SEPV, RRV, 1>(sp4, mbits, kf, ay, bx, acc); break;                                \
          case 2: us_blur_row4<SEPV, RRV, 2>(sp4, mbits, kf, ay, bx, acc); break;                                \
          default: us_blur_row4<SEPV, RRV, 3>(sp4, mbits, kf, ay, bx, acc); break;                               \
        }
#pragma unroll
        for (int rr = 0; rr < US_RS; ++rr) {
          const unsigned off = (unsigned)g.colbase + (lead_acc & 3u);              // 0..6: float4 index off >> 2, shift off & 3
          const float4* sp4 = reinterpret_cast<const float4*>(srow + (off & ~3u));
          if (sep) {
            switch (rr & 3) {
              case 0: US_BLUR_ROW(true, 0) break;
              case 1: US_BLUR_ROW(true, 1) break;
              case 2: US_BLUR_ROW(true, 2) break;
              default: US_BLUR_ROW(true, 3) break;
            }
          } else {
            switch (rr & 3) {
              case 0: US_BLUR_ROW(false, 0) break;
              case 1: US_BLUR_ROW(false, 1) break;
              case 2: US_BLUR_ROW(false, 2) break;
              default: US_BLUR_ROW(false, 3) break;
            }
          }
          if ((unsigned)(r0 + rr) < r_span) {
            const int k = (rr - 3) & 3;
            float* op = oplane + oidx;
            if (vec) *reinterpret_cast<float4*>(op) = make_float4(acc[0][k], acc[1][k], acc[2][k], acc[3][k]);
            else {
#pragma unroll
              for (int c = 0; c < 4; ++c) if (ox + c < p.out_w) op[c] = acc[c][k];
            }
          }
          oidx += p.out_w; srow += p.row_stride; lead_acc += in_w_u;
        }
#undef US_BLUR_ROW
        mbar_arrive(empty_bar(slot));
      }
    } else if (UP == 1 && DOWN == 2) {
      const int ox = g.ox0 + tid;
      const bool col_ok = ox < p.out_w;
      const bool masked = g.ix0 < 0 || g.ix0 + C::COUNT > p.in_w;     // the strip touches the left / right zero padding
      bool m[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { const int ix = g.ix0 + 2 * tid + i; m[i] = ix >= 0 && ix < p.in_w; }
      float cur = 0.f, prev = 0.f;    // output rows q = oy_a + r/2 and q - 1
      // the odd input row r completes output row oy_a + (r >> 1) - 1: stored for 3 <= r < n_rows
      int64_t oidx = (int64_t)(g.oy_a - 1) * p.out_w + ox;
      const unsigned r_span = (unsigned)(g.n_rows - 3);
      for (int s = 0; s < n_st; ++s, ++it) {
        const int slot = (int)(it % (uint32_t)US_STAGES);
        mbar_wait(full_bar(slot), (it / (uint32_t)US_STAGES) & 1u);
        const float* srow = ring + (size_t)slot * stage_floats + g.colbase + 2 * tid;
        const int r0 = s * US_RS - 3;
#pragma unroll
        for (int rr = 0; rr < US_RS; ++rr) {
          const float* sp = srow + (lead_acc & 3u);
          float v[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) { v[i] = sp[i]; if (masked) v[i] = m[i] ? v[i] : 0.f; }
          // u = 2*oy_a + r: even rows carry taps ky = 0 (row q: its first tap) and 2 (row q - 1), odd rows ky = 1 and 3
          const int k0 = (rr & 1), k1 = (rr & 1) + 2;
          if (!(rr & 1)) cur = 0.f;
#pragma unroll
          for (int i = 0; i < 4; ++i) { cur = fmaf(kf[k0 * 4 + i], v[i], cur); prev = fmaf(kf[k1 * 4 + i], v[i], prev); }
          if (rr & 1) {
            if ((unsigned)(r0 + rr) < r_span && col_ok) oplane[oidx] = prev;
            oidx += p.out_w;
            prev = cur;
          }
          srow += p.row_stride; lead_acc += in_w_u;
        }
        mbar_arrive(empty_bar(slot));
      }
    } else {
      // UP == 2: thread t owns input columns ix0 + 4t .. +5 and output columns X = ox0 + 8t + n, n = 0..7
      const int X = g.ox0 + 8 * tid;
      const int q0 = (g.ox0 - p.pad_x0) & 1;
      unsigned mbits = 0;
#pragma unroll
      for (int i = 0; i < 6; ++i) { const int ix = g.ix0 + 4 * tid + i; mbits |= (ix >= 0 && ix < p.in_w) ? (1u << i) : 0u; }
      float pv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      // taps of the two output rows an input row completes (e = 0: ky = 1, 3; e = 1: ky = 0, 2) for both column parities
      float w[2][2][4];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kyf = e ? 0 : 1, kys = kyf + 2;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          w[e][q][0] = kf[kyf * 4 + q]; w[e][q][1] = kf[kyf * 4 + q + 2];
          w[e][q][2] = kf[kys * 4 + q]; w[e][q][3] = kf[kys * 4 + q + 2];
        }
      }
      // with iy = iy_first + r as the second input row: output rows oy = 2*iy - 3 + pad and oy + 1
      int oy = 2 * g.iy_first - 3 + p.pad_y0;
      int64_t oidx = (int64_t)oy * p.out_w + X;
      const bool vec = out16 && X + 7 < p.out_w;
      for (int s = 0; s < n_st; ++s, ++it) {
        const int slot = (int)(it % (uint32_t)US_STAGES);
        mbar_wait(full_bar(slot), (it / (uint32_t)US_STAGES) & 1u);
        const float* srow = ring + (size_t)slot * stage_floats + 4 * tid;
#define US_UP_ROW(Q0V)                                                                \
        switch (off & 3u) {                                                           \
          case 0: us_up_row8<Q0V, 0>(sp4, mbits, w, pv, y); break;                    \
          case 1: us_up_row8<Q0V, 1>(sp4, mbits, w, pv, y); break;                    \
          case 2: us_up_row8<Q0V, 2>(sp4, mbits, w, pv, y); break;                    \
          default: us_up_row8<Q0V, 3>(sp4, mbits, w, pv, y); break;                   \
        }
#pragma unroll
        for (int rr = 0; rr < US_RS; ++rr) {
          const unsigned off = (unsigned)g.colbase + (lead_acc & 3u);
          const float4* sp4 = reinterpret_cast<const float4*>(srow + (off & ~3u));
          float y[2][8];
          if (q0) { US_UP_ROW(1) } else { US_UP_ROW(0) }
          const bool first = (s == 0 && rr == 0);                    // no previous row yet
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (!first && oy + e >= g.oy_a && oy + e < g.oy_b) {
              float* op = oplane + oidx + (e ? p.out_w : 0);
              if (vec) {
                *reinterpret_cast<float4*>(op) = make_float4(y[e][0], y[e][1], y[e][2], y[e][3]);
                *reinterpret_cast<float4*>(op + 4) = make_float4(y[e][4], y[e][5], y[e][6], y[e][7]);
              } else {
#pragma unroll
                for (int n = 0; n < 8; ++n) if (X + n < p.out_w) op[n] = y[e][n];
              }
            }
          }
          oy += 2; oidx += 2 * (int64_t)p.out_w; srow += p.row_stride; lead_acc += in_w_u;
        }
#undef US_UP_ROW
        mbar_arrive(empty_bar(slot));
      }
    }
  }
}

template <int UP, int DOWN>
int launch_stream(const float* in, const float* kernel, float* out, int64_t planes, int in_h, int in_w, int out_h, int out_w,
                  int pad_x0, int pad_y0, cudaStream_t st) {
  using C = UsCfg<UP, DOWN>;
  UsArgs a;
  a.in = in; a.kernel = kernel; a.out = out; a.planes = planes;
  a.in_h = in_h; a.in_w = in_w; a.out_h = out_h; a.out_w = out_w; a.pad_x0 = pad_x0; a.pad_y0 = pad_y0;
  const int dmax = pad_x0 > 0 ? (((pad_x0 + UP - 1) / UP + 3) & ~3) : 0;
  // data + left pad + colbase / lead (<= 6) + the vector readers' overshoot (<= 12 floats past the last needed column) + copy tail
  a.row_stride = (C::COUNT + dmax + 6 + 12 + 4 + 3) & ~3;
  const size_t smem = (size_t)US_STAGES * US_RS * a.row_stride * sizeof(float);
  static bool attr_done[3] = {false, false, false};
  constexpr int which = (UP == 2) ? 2 : (DOWN == 2 ? 1 : 0);
  if (!attr_done[which]) {
    VT_CUDA(cudaFuncSetAttribute(upfirdn2d_stream_kernel<UP, DOWN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_done[which] = true;
  }
  int occ = 0;
  VT_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, upfirdn2d_stream_kernel<UP, DOWN>, C::NCONS + 32, smem));
  VT_CHECK(occ >= 1, "upfirdn2d: the streaming kernel does not fit (%zu B of shared memory)", smem);
  const int64_t slots = (int64_t)vt_num_sms() * occ;
  a.strips = (int)vt_cdiv(out_w, C::OWT);
  // enough items for ~4 rounds over the resident blocks, chunks of at least 32 output rows (3 halo rows are re-read per chunk)
  int64_t chunks = vt_cdiv(4 * slots, planes * a.strips);
  const int64_t max_chunks = vt_cdiv(out_h, 32);
  if (chunks > max_chunks) chunks = max_chunks;
  if (chunks < 1) chunks = 1;
  a.rows_per_chunk = (int)vt_cdiv(out_h, chunks);
  a.chunks = (int)vt_cdiv(out_h, a.rows_per_chunk);
  a.total_items = planes * a.chunks * a.strips;
  const int64_t grid = a.total_items < slots ? a.total_items : slots;
  upfirdn2d_stream_kernel<UP, DOWN><<<(unsigned)grid, C::NCONS + 32, smem, st>>>(a);
  return 0;
}

}  // namespace

extern "C" int vt_upfirdn2d_out_size(int in_h, int in_w, int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                                     int pad_x0, int pad_x1, int pad_y0, int pad_y1, int* out_h, int* out_w) {
  VT_CHECK(up_x >= 1 && up_y >= 1 && down_x >= 1 && down_y >= 1, "upfirdn2d: up/down must be >= 1");
  VT_CHECK(kh >= 1 && kw >= 1, "upfirdn2d: empty kernel");
  const int64_t nh = (int64_t)in_h * up_y + pad_y0 + pad_y1 - kh + down_y;
  const int64_t nw = (int64_t)in_w * up_x + pad_x0 + pad_x1 - kw + down_x;
  // floor division like Python's // (model/stylegan/op_cpu/upfirdn2d.py:58-59)
  auto fdiv = [](int64_t a, int64_t b) { int64_t q = a / b; if ((a % b != 0) && ((a < 0) != (b < 0))) --q; return q; };
  *out_h = (int)fdiv(nh, down_y);
  *out_w = (int)fdiv(nw, down_x);
  return 0;
}

extern "C" int vt_upfirdn2d_f32(const float* in, const float* kernel, float* out, int64_t planes, int in_h, int in_w,
                                int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                                int pad_x0, int pad_x1, int pad_y0, int pad_y1, void* stream) {
  int out_h = 0, out_w = 0;
  if (vt_upfirdn2d_out_size(in_h, in_w, kh, kw, up_x, up_y, down_x, down_y, pad_x0, pad_x1, pad_y0, pad_y1, &out_h, &out_w))
    return 1;
  VT_CHECK(in && kernel && out, "upfirdn2d: null pointer");
  VT_CHECK(planes >= 0 && in_h >= 1 && in_w >= 1, "upfirdn2d: bad input shape");
  VT_CHECK(out_h >= 1 && out_w >= 1, "upfirdn2d: empty output (%d x %d)", out_h, out_w);
  if (planes == 0) return 0;
  const bool hot4 = kh == 4 && kw == 4 && up_x == up_y && down_x == down_y && ((up_x == 1 && down_x <= 2) || (up_x == 2 && down_x == 1));
  if (g_upfirdn_tiled >= 2 && hot4 && pad_x0 >= -(1 << 20) && pad_x0 <= 64 && pad_y0 >= -(1 << 20) && pad_y0 <= (1 << 20) &&
      (reinterpret_cast<uintptr_t>(in) & 3) == 0) {
    int rc;
    if (up_x == 2) rc = launch_stream<2, 1>(in, kernel, out, planes, in_h, in_w, out_h, out_w, pad_x0, pad_y0, (cudaStream_t)stream);
    else if (down_x == 2) rc = launch_stream<1, 2>(in, kernel, out, planes, in_h, in_w, out_h, out_w, pad_x0, pad_y0, (cudaStream_t)stream);
    else rc = launch_stream<1, 1>(in, kernel, out, planes, in_h, in_w, out_h, out_w, pad_x0, pad_y0, (cudaStream_t)stream);
    if (rc) return rc;
    VT_LAUNCH_CHECK();
    return 0;
  }
  if (g_upfirdn_tiled && hot4 && planes <= 65535) {
    // the hot-path instances: compile-time up/down, 4 x 4 register micro-tiles
    int rc;
    if (up_x == 2) rc = launch_k4<2, 1>(in, kernel, out, planes, in_h, in_w, out_h, out_w, pad_x0, pad_y0, (cudaStream_t)stream);
    else if (down_x == 2) rc = launch_k4<1, 2>(in, kernel, out, planes, in_h, in_w, out_h, out_w, pad_x0, pad_y0, (cudaStream_t)stream);
    else rc = launch_k4<1, 1>(in, kernel, out, planes, in_h, in_w, out_h, out_w, pad_x0, pad_y0, (cudaStream_t)stream);
    if (rc) return rc;
    VT_LAUNCH_CHECK();
    return 0;
  }
  {
    // tiled fast path when the input window of a 32 x 64 output tile fits in shared memory
    const int tile_rows = ((T_OH - 1) * down_y + kh - 1) / up_y + 2;
    const int tile_cols = ((T_OW - 1) * down_x + kw - 1) / up_x + 2;
    const size_t smem = ((size_t)tile_rows * tile_cols + (size_t)kh * kw) * sizeof(float);
    if (g_upfirdn_tiled && smem <= 160 * 1024 && planes <= 65535) {
      const int tiles_x = (int)vt_cdiv(out_w, T_OW), tiles_y = (int)vt_cdiv(out_h, T_OH);
      if (smem > 48 * 1024)
        VT_CUDA(cudaFuncSetAttribute(upfirdn2d_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      dim3 grid((unsigned)(tiles_x * tiles_y), (unsigned)planes);
      upfirdn2d_tiled_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(in, kernel, out, in_h, in_w, out_h, out_w, kh, kw, up_x,
                                                                        up_y, down_x, down_y, pad_x0, pad_y0, tiles_x, tile_rows,
                                                                        tile_cols);
      VT_LAUNCH_CHECK();
      return 0;
    }
  }
  const int64_t total = planes * (int64_t)out_h * out_w;
  const int threads = 256;
  int64_t blocks = vt_cdiv(total, threads);
  const int64_t max_blocks = (int64_t)vt_num_sms() * 32;
  if (blocks > max_blocks) blocks = max_blocks;
  upfirdn2d_generic_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      in, kernel, out, planes, in_h, in_w, out_h, out_w, kh, kw, up_x, up_y, down_x, down_y, pad_x0, pad_y0,
      (kh * kw <= kMaxSmemTaps) ? 1 : 0);
  VT_LAUNCH_CHECK();
  return 0;
}
