// conv_wgrad.cu — weight gradient of a convolution on the Hopper tensor cores (wgmma):
//
//   D[m, n, t] = sum over samples b and pixels p of the A grid of  A[b, p, m] * S[b, stride*p + off_t, n]
//
// The GEMM's K dimension is pixels.  In NHWC the channels are contiguous, so both TMA tiles arrive MN-major (rows = pixels).
// wgmma takes MN-major shared-memory operands only for 16-bit types, and only the K-major form is wrapped in wgmma_sm90.cuh;
// the operand-transform warps split fp32 into bf16 hi + lo anyway, so they write the transposed (K-major) rows while they
// split, and the consumers use the same descriptors and MMA wrappers as conv_tc_kernel.
//
// One CTA per work item (tap t, 64 rows of M, 2 x NW columns of N, sample when per-sample, split of K), three warpgroups:
//   warp 0 (1 lane)  TMA producer : per K step of 32 pixels, boxes (32 ch, bx, 32/bx, 1) of A and of S shifted by the tap;
//                                   OOB zero fill is the padding of S and the tail of the A grid.  Stride 2 reads the parity
//                                   view of S that the tap lands on (as conv_tc.cu).
//   warps 1-3        transform    : fp32 [pixel][ch] boxes -> bf16 rows [ch][hi(32 px) | lo(32 px)] (128B swizzle), a second ring
//   warpgroups 1, 2  consumers    : both read the 64 A rows; warpgroup c owns N columns [c NW, c NW + NW).  6 MMAs m64nNk16 per
//                                   K step (a_hi b_hi + a_lo b_hi + a_hi b_lo), one commit group per step, one group in flight.
#include "tc_common.cuh"
#include <cuda_bf16.h>
#include <mutex>

using namespace vt_tc;

namespace {

constexpr int BM = 64;                 // M rows of a work item
constexpr int KPIX = 32;               // pixels per K step = one 128-byte operand row [hi(32) | lo(32)] of 16-bit values
constexpr int BOX_BYTES = KPIX * 128;  // one fp32 TMA box: 32 pixels x 32 channels
constexpr int MAX_SMEM = 227 * 1024;
constexpr int THREADS = 384;
constexpr int XFORM_WARPS = 3;
constexpr int RELEASE_ARRIVALS = 8;    // every consumer warp releases an operand stage it has read
constexpr int SPLIT_TARGET = 132;      // work items wanted before the pixel reduction is split (SMs of an H100 SXM)
constexpr int MIN_SPLIT_STEPS = 16;    // K steps per split at least

struct WgArgs {
  CUtensorMap a_map;
  CUtensorMap s_map[4];                // stride 1: [0] only; stride 2: parity view (py, px) at py * 2 + px
  int M, N, taps, nb, per_sample;
  int tiles_x, tiles_y, box_w;
  int64_t ksteps;                      // K steps of one output slice: B * tiles (shared weights) or tiles (per sample)
  int splits, m_tiles, n_tiles;
  int raw_stages, op_stages;
  int tap_view[VT_MAX_TAPS], tap_vx[VT_MAX_TAPS], tap_vy[VT_MAX_TAPS];
  float* out;                          // D, or the workspace [splits][nb * M][N][taps]
  int64_t split_stride;                // floats between the partial results of two splits (0: D itself)
};

template <int NW>
__device__ __forceinline__ void wgmma_bf16(float* acc, uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (NW == 32) wgmma_bf16_n32(acc, a, b, accumulate);
  else if constexpr (NW == 64) wgmma_bf16_n64(acc, a, b, accumulate);
  else wgmma_bf16_n128(acc, a, b, accumulate);
}

// NW: MMA N of one consumer warpgroup (the work item has 2 * NW columns of N)
template <int NW>
__global__ void __launch_bounds__(THREADS, 1)
conv_wgrad_kernel(const __grid_constant__ WgArgs p) {
  constexpr int BN = 2 * NW;
  constexpr int ROWS = BM + BN;                    // channels staged per K step (A rows, then S rows)
  constexpr uint32_t STAGE = ROWS * 128;           // bytes of a raw fp32 stage and of an operand stage alike
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t op_base = raw_base + (uint32_t)p.raw_stages * STAGE;
  const uint32_t bar_base = op_base + (uint32_t)p.op_stages * STAGE;
  auto raw_full = [&](int i) { return bar_base + 8u * i; };
  auto raw_empty = [&](int i) { return bar_base + 64u + 8u * i; };
  auto op_full = [&](int i) { return bar_base + 128u + 8u * i; };
  auto op_empty = [&](int i) { return bar_base + 192u + 8u * i; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;

  // work item: N tile fastest, then M tile, tap, sample, split (CTAs running together read the same pixels: L2 hits)
  int item = blockIdx.x;
  const int n_tile = item % p.n_tiles; item /= p.n_tiles;
  const int m_tile = item % p.m_tiles; item /= p.m_tiles;
  const int t = item % p.taps; item /= p.taps;
  const int bo = item % p.nb;
  const int split = item / p.nb;
  const int m0 = m_tile * BM, n0 = n_tile * BN;
  const int64_t k0 = p.ksteps * split / p.splits, k1 = p.ksteps * (split + 1) / p.splits;
  const int tiles_img = p.tiles_x * p.tiles_y;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.a_map);
    tma_prefetch_desc(&p.s_map[p.tap_view[t]]);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < p.raw_stages; ++i) { mbar_init(raw_full(i), 1); mbar_init(raw_empty(i), XFORM_WARPS); }
    for (int i = 0; i < p.op_stages; ++i) { mbar_init(op_full(i), XFORM_WARPS); mbar_init(op_empty(i), RELEASE_ARRIVALS); }
    fence_barrier_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (wg == 0) {
    if (warp == 0) {
      // ================= TMA producer =================
      const CUtensorMap* smap = &p.s_map[p.tap_view[t]];
      const int vx = p.tap_vx[t], vy = p.tap_vy[t];
      const int bw = p.box_w, bh = KPIX / p.box_w;
      int st = 0;
      uint32_t par = 0;
      for (int64_t k = k0; k < k1; ++k) {
        const int b = p.per_sample ? bo : (int)(k / tiles_img);
        const int rem = (int)(p.per_sample ? k : k % tiles_img);
        const int x0 = (rem % p.tiles_x) * bw, y0 = (rem / p.tiles_x) * bh;
        mbar_wait(raw_empty(st), par ^ 1);
        if (elect_one()) {
          const uint32_t dst = raw_base + (uint32_t)st * STAGE;
          mbar_arrive_expect_tx(raw_full(st), STAGE);
#pragma unroll
          for (int q = 0; q < BM / 32; ++q) tma_load_4d(dst + q * BOX_BYTES, &p.a_map, raw_full(st), m0 + 32 * q, x0, y0, b);
#pragma unroll
          for (int q = 0; q < BN / 32; ++q)
            tma_load_4d(dst + (BM / 32 + q) * BOX_BYTES, smap, raw_full(st), n0 + 32 * q, x0 + vx, y0 + vy, b);
        }
        __syncwarp();
        if (++st == p.raw_stages) { st = 0; par ^= 1; }
      }
    } else {
      // ================= operand transform: transpose + split =================
      // Task (channel ch, 8-pixel group g): the lanes of a warp take 32 consecutive channels of one box, so the fp32 reads
      // (one 128-byte box row per pixel) and the 16-byte stores (8 distinct swizzle phases per 8 lanes) are conflict-free.
      const int tid = (warp - 1) * 32 + lane;
      int rs = 0, os = 0;
      uint32_t rpar = 0, opar = 0;
      for (int64_t k = k0; k < k1; ++k) {
        mbar_wait(raw_full(rs), rpar);
        mbar_wait(op_empty(os), opar ^ 1);
        const uint32_t raw = raw_base + (uint32_t)rs * STAGE, op = op_base + (uint32_t)os * STAGE;
        for (int i = tid; i < ROWS * 4; i += 32 * XFORM_WARPS) {
          const int ch = i % ROWS, g = i / ROWS, c = ch & 31;
          // fp32 element (pixel r, channel c) of a box: row r, 16-byte chunk (c / 4) ^ (r & 7) (SWIZZLE_128B); r = 8 g + e
          const uint32_t src = raw + (uint32_t)(ch >> 5) * BOX_BYTES + (uint32_t)(8 * g) * 128u + (uint32_t)(c & 3) * 4u;
          float f[8];
#pragma unroll
          for (int e = 0; e < 8; ++e)
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(f[e]) : "r"(src + (uint32_t)e * 128u + ((uint32_t)((c >> 2) ^ e) << 4)));
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const __nv_bfloat162 h2 = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
            hi[j] = *reinterpret_cast<const uint32_t*>(&h2);
            const float r0 = f[2 * j] - __uint_as_float(hi[j] << 16), r1 = f[2 * j + 1] - __uint_as_float(hi[j] & 0xffff0000u);
            const __nv_bfloat162 l2 = __floats2bfloat162_rn(r0, r1);
            lo[j] = *reinterpret_cast<const uint32_t*>(&l2);
          }
          // operand row ch: [hi of pixels 0..31 | lo of pixels 0..31], 16-byte chunk j stored at j ^ (ch & 7)
          const uint32_t row = op + (uint32_t)ch * 128u, sw = (uint32_t)(ch & 7);
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(row + (((uint32_t)g ^ sw) << 4)), "r"(hi[0]), "r"(hi[1]), "r"(hi[2]), "r"(hi[3]) : "memory");
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(row + (((uint32_t)(g + 4) ^ sw) << 4)), "r"(lo[0]), "r"(lo[1]), "r"(lo[2]), "r"(lo[3]) : "memory");
        }
        // generic-proxy writes -> visible to the tensor core's async-proxy reads
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) { mbar_arrive(op_full(os)); mbar_arrive(raw_empty(rs)); }
        if (++rs == p.raw_stages) { rs = 0; rpar ^= 1; }
        if (++os == p.op_stages) { os = 0; opar ^= 1; }
      }
    }
  } else {
    // ================= consumers =================
    const int c = wg - 1;
    const int w = (threadIdx.x & 127) >> 5;
    float acc[NW / 2];
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
    int os = 0, rel = -1;
    uint32_t opar = 0, first = 1;
    for (int64_t k = k0; k < k1; ++k) {
      mbar_wait(op_full(os), opar);
      const uint32_t op = op_base + (uint32_t)os * STAGE;
      const uint64_t adesc = make_smem_desc_sw128(op, 1024);
      const uint64_t bdesc = make_smem_desc_sw128(op + (uint32_t)(BM + c * NW) * 128u, 1024);
      // +2 on a descriptor = +32 bytes = 16 pixels of K: a_hi b_hi, a_lo b_hi, a_hi b_lo (the a_lo b_lo term is ~2^-18 relative)
      constexpr int ao[6] = {0, 2, 4, 6, 0, 2};
      constexpr int bo6[6] = {0, 2, 0, 2, 4, 6};
      wgmma_fence();
#pragma unroll
      for (int i = 0; i < 6; ++i) wgmma_bf16<NW>(acc, adesc + (uint64_t)ao[i], bdesc + (uint64_t)bo6[i], i == 0 ? (first ^ 1u) : 1u);
      wgmma_commit();
      wgmma_wait<1>();   // this warp's share of the previous group has completed: its stage may be refilled
      if (lane == 0 && rel >= 0) mbar_arrive(op_empty(rel));
      rel = os;
      first = 0;
      if (++os == p.op_stages) { os = 0; opar ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_pin<NW / 2>(acc);
    // accumulator register i: row 16 w + lane / 4 + 8 ((i / 2) % 2) (an M channel), column 8 (i / 4) + 2 (lane % 4) + i % 2
    float* out = p.out + (int64_t)split * p.split_stride;
    const int qd = lane & 3;
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) {
      const int m = m0 + 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1);
      const int n = n0 + c * NW + 8 * (i >> 2) + 2 * qd + (i & 1);
      if (m < p.M && n < p.N) out[(((int64_t)bo * p.M + m) * p.N + n) * p.taps + t] = acc[i];
    }
  }
}

// D = sum over splits of the partial results, in split order
__global__ void conv_wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ out, int64_t n, int splits) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float s = ws[i];
    for (int k = 1; k < splits; ++k) s += ws[(int64_t)k * n + i];
    out[i] = s;
  }
}

struct WgPlan {
  int nw, box_w, tiles_x, tiles_y, m_tiles, n_tiles, nb, splits, raw_stages, op_stages, smem;
  int64_t ksteps, items, slice;
};

// host-only planning: validates the descriptor, picks the tiles and the split count (a function of the descriptor alone)
int plan(const vt_conv_wgrad_desc* d, WgPlan* pl) {
  VT_CHECK(d != nullptr && d->struct_size == (int)sizeof(vt_conv_wgrad_desc), "conv_wgrad: descriptor size mismatch (got %d, want %d)",
           d ? d->struct_size : -1, (int)sizeof(vt_conv_wgrad_desc));
  VT_CHECK(d->stride == 1 || d->stride == 2, "conv_wgrad: stride must be 1 or 2 (got %d)", d->stride);
  VT_CHECK(d->taps >= 1 && d->taps <= VT_MAX_TAPS, "conv_wgrad: taps must be 1..%d (got %d)", VT_MAX_TAPS, d->taps);
  VT_CHECK(d->a_cstride > 0 && d->a_cstride % 32 == 0 && d->s_cstride > 0 && d->s_cstride % 32 == 0,
           "conv_wgrad: channel strides must be positive multiples of 32 (got %d, %d)", d->a_cstride, d->s_cstride);
  VT_CHECK(d->M >= 1 && d->M <= d->a_cstride && d->N >= 1 && d->N <= d->s_cstride, "conv_wgrad: M / N out of range of the channel strides");
  VT_CHECK(d->B >= 1 && d->a_h >= 1 && d->a_w >= 1 && d->s_h >= 1 && d->s_w >= 1, "conv_wgrad: empty tensor");
  VT_CHECK(d->per_sample == 0 || d->per_sample == 1, "conv_wgrad: per_sample must be 0 or 1");
  VT_CHECK(d->stride == 1 || (d->s_h >= 2 && d->s_w >= 2), "conv_wgrad: stride 2 needs S of at least 2 x 2 pixels");
  for (int t = 0; t < d->taps; ++t)
    VT_CHECK(d->tap_dy[t] >= -4096 && d->tap_dy[t] <= 4096 && d->tap_dx[t] >= -4096 && d->tap_dx[t] <= 4096, "conv_wgrad: tap offset out of range");
  pl->nw = d->N <= 64 ? 32 : d->N <= 128 ? 64 : 128;
  pl->box_w = d->a_w > 16 ? 32 : d->a_w > 8 ? 16 : 8;
  pl->tiles_x = (int)vt_cdiv(d->a_w, pl->box_w);
  pl->tiles_y = (int)vt_cdiv(d->a_h, KPIX / pl->box_w);
  pl->m_tiles = (int)vt_cdiv(d->M, BM);
  pl->n_tiles = (int)vt_cdiv(d->N, 2 * pl->nw);
  pl->nb = d->per_sample ? d->B : 1;
  const int64_t tiles = (int64_t)pl->tiles_x * pl->tiles_y;
  pl->ksteps = d->per_sample ? tiles : tiles * d->B;
  const int64_t items0 = (int64_t)d->taps * pl->m_tiles * pl->n_tiles * pl->nb;
  int64_t s = 1;
  if (items0 < SPLIT_TARGET) {
    s = vt_cdiv(SPLIT_TARGET, items0);
    const int64_t cap = pl->ksteps / MIN_SPLIT_STEPS;
    s = s < cap ? s : cap;
    s = s < 1 ? 1 : s;
  }
  pl->splits = (int)s;
  pl->items = items0 * s;
  VT_CHECK(pl->items < (1LL << 31), "conv_wgrad: too many work items");
  pl->slice = (int64_t)pl->nb * d->M * d->N * d->taps;
  const int stage = (BM + 2 * pl->nw) * 128;
  const int fixed = 1024 /*barriers*/ + 1024 /*alignment slack*/;
  const int n_stages = (MAX_SMEM - fixed) / stage;
  pl->raw_stages = n_stages / 2 < 4 ? n_stages / 2 : 4;
  pl->op_stages = n_stages - pl->raw_stages < 4 ? n_stages - pl->raw_stages : 4;
  pl->smem = (pl->raw_stages + pl->op_stages) * stage + fixed;
  VT_CHECK(pl->raw_stages >= 2 && pl->op_stages >= 2 && pl->smem <= MAX_SMEM, "conv_wgrad: shared memory plan does not fit");
  return 0;
}

struct WgKernel {
  int nw;
  void (*fn)(WgArgs);
};
const WgKernel kWgKernels[] = {{32, conv_wgrad_kernel<32>}, {64, conv_wgrad_kernel<64>}, {128, conv_wgrad_kernel<128>}};

}  // namespace

extern "C" int64_t vt_conv2d_wgrad_ws_floats(const vt_conv_wgrad_desc* d) {
  WgPlan pl;
  if (plan(d, &pl)) return -1;
  return pl.splits > 1 ? pl.splits * pl.slice : 0;
}

extern "C" int vt_conv2d_wgrad(const vt_conv_wgrad_desc* d, void* stream) {
  WgPlan pl;
  if (plan(d, &pl)) return 1;
  VT_CHECK(d->a && d->s && d->out, "conv_wgrad: NULL tensor");
  VT_CHECK(((uintptr_t)d->a & 15) == 0 && ((uintptr_t)d->s & 15) == 0, "conv_wgrad: operands not 16-byte aligned");
  const int64_t ws_need = pl.splits > 1 ? pl.splits * pl.slice : 0;
  VT_CHECK(ws_need == 0 || (d->ws && d->ws_floats >= ws_need), "conv_wgrad: workspace too small (%lld floats, need %lld)",
           (long long)d->ws_floats, (long long)ws_need);

  static thread_local WgArgs a;
  memset(&a, 0, sizeof(a));
  a.M = d->M; a.N = d->N; a.taps = d->taps; a.nb = pl.nb; a.per_sample = d->per_sample;
  a.tiles_x = pl.tiles_x; a.tiles_y = pl.tiles_y; a.box_w = pl.box_w;
  a.ksteps = pl.ksteps; a.splits = pl.splits; a.m_tiles = pl.m_tiles; a.n_tiles = pl.n_tiles;
  a.raw_stages = pl.raw_stages; a.op_stages = pl.op_stages;
  a.out = pl.splits > 1 ? d->ws : d->out;
  a.split_stride = pl.splits > 1 ? pl.slice : 0;
  for (int t = 0; t < d->taps; ++t) {
    int view = 0, vx = d->tap_dx[t], vy = d->tap_dy[t];
    if (d->stride == 2) {
      const int px = vx & 1, py = vy & 1;
      view = py * 2 + px;
      vx = (vx - px) / 2;
      vy = (vy - py) / 2;
    }
    a.tap_view[t] = view; a.tap_vx[t] = vx; a.tap_vy[t] = vy;
  }
  // tensor maps: dims innermost first (channels, x, y, sample), strides in bytes
  const uint32_t box[4] = {32, (uint32_t)pl.box_w, (uint32_t)(KPIX / pl.box_w), 1};
  {
    const uint64_t cs = (uint64_t)d->a_cstride;
    const uint64_t dims[4] = {cs, (uint64_t)d->a_w, (uint64_t)d->a_h, (uint64_t)d->B};
    const uint64_t str[3] = {cs * 4, (uint64_t)d->a_w * cs * 4, (uint64_t)d->a_h * d->a_w * cs * 4};
    if (vt_tc_make_map4(&a.a_map, d->a, dims, str, box, "wgrad A", false)) return 1;
  }
  const uint64_t cs = (uint64_t)d->s_cstride;
  if (d->stride == 1) {
    const uint64_t dims[4] = {cs, (uint64_t)d->s_w, (uint64_t)d->s_h, (uint64_t)d->B};
    const uint64_t str[3] = {cs * 4, (uint64_t)d->s_w * cs * 4, (uint64_t)d->s_h * d->s_w * cs * 4};
    if (vt_tc_make_map4(&a.s_map[0], d->s, dims, str, box, "wgrad S", false)) return 1;
  } else {
    // parity views: view (py, px)[vy][vx] = S[2 vy + py][2 vx + px]
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        const uint64_t dims[4] = {cs, (uint64_t)((d->s_w - px + 1) / 2), (uint64_t)((d->s_h - py + 1) / 2), (uint64_t)d->B};
        const uint64_t str[3] = {2 * cs * 4, 2 * (uint64_t)d->s_w * cs * 4, (uint64_t)d->s_h * d->s_w * cs * 4};
        if (vt_tc_make_map4(&a.s_map[py * 2 + px], d->s + ((int64_t)py * d->s_w + px) * (int64_t)cs, dims, str, box, "wgrad S(parity)", false))
          return 1;
      }
  }
  static std::once_flag attr_once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once, [] {
    for (const WgKernel& k : kWgKernels)
      if (attr_err == cudaSuccess) attr_err = cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM);
  });
  VT_CHECK(attr_err == cudaSuccess, "conv_wgrad: cudaFuncSetAttribute failed: %s", cudaGetErrorString(attr_err));
  const WgKernel* kern = nullptr;
  for (const WgKernel& k : kWgKernels)
    if (k.nw == pl.nw) kern = &k;
  VT_CHECK(kern != nullptr, "conv_wgrad: no kernel for N = %d", pl.nw);
  kern->fn<<<(unsigned)pl.items, THREADS, pl.smem, (cudaStream_t)stream>>>(a);
  VT_LAUNCH_CHECK();
  if (pl.splits > 1) {
    const int64_t blocks = vt_cdiv(pl.slice, 256);
    conv_wgrad_reduce_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, (cudaStream_t)stream>>>(d->ws, d->out, pl.slice, pl.splits);
    VT_LAUNCH_CHECK();
  }
  return 0;
}
