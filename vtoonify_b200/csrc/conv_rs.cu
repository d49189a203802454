// conv_rs.cu — the full-resolution 3x3 / stride 1 layers with Cin, Cout in {32, 64} (row-strip entry point vt_conv2d_rs).
//
//   D[64 cout rows, 128 pixels] (registers, fp32) += W[64 cout rows, K] (smem, bf16 hi/lo) * X[128 pixels, K]^T (smem, bf16 hi/lo)
//
// conv_tc_kernel puts pixels on the wgmma M dimension (64 per warpgroup) and output channels on N, so these layers issue
// m64n32k16 / m64n64k16 MMAs that read more shared-memory bytes per clock than the port delivers.  Here the roles are swapped:
// output channels fill M = 64 and pixels are N = 128, and each m64n128k16 reads 6 KB per 64 clocks.
//
// One persistent CTA per SM, three warpgroups (the same roles as conv_tc_kernel):
//   warp 0 (1 lane)  TMA producer : one halo box of (8+2) x (16+2) pixels x 32 channels per K chunk (zero fill = the padding),
//                                   and the weights of every tap and K chunk, kept resident while the sample's weights stay the same.
//   warps 1-3        operand transform: fp32 rows -> [hi | lo] bf16 rows, in place.
//   warpgroups 1, 2  consumers    : a work item is an 8 x 16 pixel tile; the two warpgroups own alternate items, so one
//                                   warpgroup's epilogue overlaps the other's MMAs.  A staged halo row is one pixel's
//                                   [x_hi | x_lo] 128-byte row with K contiguous, i.e. already the K-major N x K layout of the
//                                   wgmma B operand: a tap is the B descriptor's start shifted by whole rows, with the halo row
//                                   pitch as stride byte offset (8 consecutive x pixels per 8-row group, 16 groups = 16 y rows).
//
// Products per 32-channel chunk and tap, as in conv_tc_kernel:
//   Cout = 64: rows [w_hi | w_lo]; w_hi*x_hi, w_hi*x_lo, w_lo*x_hi in 6 MMAs, in conv_tc_kernel's order.
//   Cout = 32: the N-stacked split (32 rows [w_hi | w_hi], then 32 rows [w_lo | w_lo]) is the 64-row A operand: 4 MMAs give all four
//              products, the w_hi ones in rows c, the w_lo ones in rows c + 32; the epilogue adds row c + 32 to row c.
//
// Shared memory (bytes; the limit is 232448):
//   Cin = 32: weights 9 x 64 x 128 = 73728, 3 halo stages x 23552, epilogue 2 x 34816, barriers + alignment 2048 = 216064
//   Cin = 64: weights 2 x 73728 = 147456, 3 halo stages x 23552, epilogue 2 x 4352, barriers + alignment 2048 = 228864
//
// Epilogue: the accumulators (a thread holds channel rows and pixel columns) go through a per-warpgroup [pixel][channel] shared
// tile: the whole 128-pixel tile in one pass (Cin = 32), or 16 pixels per pass (Cin = 64).  Every pixel is then read by 4 or 8
// neighbouring threads, each holding whole float4 channel groups: bias, noise, leaky ReLU * gain, 16-byte NHWC stores (a warp
// writes 8 whole pixels), and the fused ToRGB reduced over the pixel's threads by shuffles in a fixed order.  With 4 pixels per
// thread and pass (Cin = 32) or 1 pixel in each of 8 passes (Cin = 64), each of a pixel's threads finishes the ToRGB (bias +
// up-sampled skip) of a different pixel, once, after the last pass.  The epilogue is bound by global-memory latency, not by
// bandwidth, so its loads (noise, skip taps) are issued when the work item starts and land while the MMAs run.
#include "tc_common.cuh"
#include <cuda_bf16.h>
#include <mutex>

using namespace vt_tc;

int vt_validate_conv_desc(const vt_conv_desc* d, const char* who);
extern "C" int vt_conv2d_tc_supported(const vt_conv_desc* d);

int g_rs_kernel = 1;   // vt_set_option("rs_kernel"): 1 = conv_rs_kernel where it takes the launch, 0 = always conv_tc_kernel

namespace {

constexpr int RS_THREADS = 384;
constexpr int XFORM_WARPS = 3;
constexpr int TILE_W = 8, TILE_H = 16;                   // work item: 8 x 16 output pixels = MMA N 128
constexpr int HALO_W = TILE_W + 2, HALO_H = TILE_H + 2;
constexpr int HALO_ROWS = HALO_W * HALO_H;               // 180 rows of 128 bytes
constexpr uint32_t HALO_TX = HALO_ROWS * 128;            // 23040
constexpr uint32_t A_STAGE = (HALO_TX + 1023) / 1024 * 1024;
constexpr uint32_t W_TAP = 64 * 128;                     // 64 weight rows of one tap and K chunk
constexpr uint32_t W_CHUNK = 9 * W_TAP;
constexpr int EP = 68;                                   // floats per pixel of the epilogue tile (64 rows + 4: no bank conflicts on write)
constexpr int MAX_SMEM = 227 * 1024;

template <int CIN>
struct RsPlan {
  static constexpr int KC = CIN / 32;
  static constexpr uint32_t W_BYTES = KC * W_CHUNK;
  static constexpr int A_STAGES = 3;
  static constexpr int PJ = KC == 1 ? 16 : 2;            // 8-pixel rows per epilogue pass: all 16 when the tile fits
  static constexpr int TPP = KC == 1 ? 4 : 8;            // threads per pixel in the epilogue's read phase
  static constexpr int PPT = PJ * 8 * TPP / 128;         // pixels per thread and pass
  static constexpr uint32_t EPI_BYTES = PJ * 8 * EP * 4;
  static constexpr uint32_t SMEM = W_BYTES + A_STAGES * A_STAGE + 2 * EPI_BYTES + 1024 /*barriers*/ + 1024 /*alignment slack*/;
  static_assert(SMEM <= MAX_SMEM, "conv_rs shared-memory plan");
};

struct RsArgs {
  CUtensorMap in_map, w_map;
  int tiles_x, tiles_y, B, total_tiles, Ho, Wo, wB;
  const float* bias;
  const float* noise;
  const float* noise_w;
  float* out;
  int64_t out_off, out_sb, out_sy, out_sx;
  int64_t pix_off, pix_sb, pix_sy, pix_sx;   // the same view in dense-pixel units (noise index)
  int act, round_tf32;
  float slope, gain, acc_scale;
  const float* rgb_w; const float* rgb_bias; const float* rgb_skip; const float* rgb_skip_kernel; float* rgb_out;
};

// one tap of one 32-channel chunk: A = weight rows, B = pixel rows; +2 on a descriptor = +32 B = 16 elements of K
template <bool NSTACK>
__device__ __forceinline__ void rs_mma_step(float* acc, uint64_t wdesc, uint64_t xdesc, uint32_t first) {
  constexpr int xo[6] = {0, 2, 4, 6, 0, 2};   // pixel row [x_hi | x_lo]
  constexpr int wo[6] = {0, 2, 0, 2, 4, 6};   // weight row [w_hi | w_lo]; N-stacked rows pair with the pixel row as they are
#pragma unroll
  for (int i = 0; i < (NSTACK ? 4 : 6); ++i)
    wgmma_bf16_n128(acc, wdesc + (uint64_t)(NSTACK ? xo[i] : wo[i]), xdesc + (uint64_t)xo[i], i == 0 ? (first ^ 1u) : 1u);
}

template <int CIN, int COUT>
__global__ void __launch_bounds__(RS_THREADS, 1)
conv_rs_kernel(const __grid_constant__ RsArgs p) {
  using P = RsPlan<CIN>;
  constexpr int KC = P::KC, A_STAGES = P::A_STAGES, PJ = P::PJ;
  constexpr bool NSTACK = COUT == 32;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t w_base = (raw + 1023u) & ~1023u;
  const uint32_t a_base = w_base + P::W_BYTES;
  const uint32_t e_base = a_base + A_STAGES * A_STAGE;
  const uint32_t bar_base = e_base + 2 * P::EPI_BYTES;
  auto a_full = [&](int i) { return bar_base + 8u * i; };
  auto a_ready = [&](int i) { return bar_base + 64u + 8u * i; };   // stage converted to [hi|lo] bf16 rows
  auto a_empty = [&](int i) { return bar_base + 128u + 8u * i; };
  const uint32_t w_full = bar_base + 192u, w_empty = bar_base + 200u;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.in_map);
    tma_prefetch_desc(&p.w_map);
  }
  if (warp == 1 && lane == 0) {
    // every stage and the weights are released by all 8 consumer warps: the warpgroup that does not own an item releases its
    // stages at once, so both warpgroups walk the rings in lockstep
    for (int i = 0; i < A_STAGES; ++i) { mbar_init(a_full(i), 1); mbar_init(a_ready(i), XFORM_WARPS); mbar_init(a_empty(i), 8); }
    mbar_init(w_full, 1);
    mbar_init(w_empty, 8);
    fence_barrier_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  const int tiles_per_img = p.tiles_y * p.tiles_x;
  if (wg == 0) {
    if (warp == 0) {
      // ================= TMA producer =================
      int a_st = 0, last_wb = -1;
      uint32_t a_par = 0, w_par = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int b = tile / tiles_per_img, rem = tile % tiles_per_img;
        const int oy0 = (rem / p.tiles_x) * TILE_H, ox0 = (rem % p.tiles_x) * TILE_W;
        const int wb = p.wB > 1 ? b : 0;
        if (wb != last_wb) {   // work items are sample-major: a CTA loads each sample's weights once
          mbar_wait(w_empty, w_par ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(w_full, P::W_BYTES);
            for (int kc = 0; kc < KC; ++kc) tma_load_4d(w_base + kc * W_CHUNK, &p.w_map, w_full, kc * 64, 0, 0, wb);
          }
          __syncwarp();
          w_par ^= 1;
          last_wb = wb;
        }
        for (int kc = 0; kc < KC; ++kc) {
          mbar_wait(a_empty(a_st), a_par ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(a_full(a_st), HALO_TX);
            tma_load_4d(a_base + a_st * A_STAGE, &p.in_map, a_full(a_st), kc * 32, ox0 - 1, oy0 - 1, b);
          }
          __syncwarp();
          if (++a_st == A_STAGES) { a_st = 0; a_par ^= 1; }
        }
      }
    } else {
      // ================= operand transform: fp32 rows -> [hi(32) | lo(32)] bf16 rows, in place =================
      // 16-byte chunk j of a row lives at physical chunk j ^ ((addr >> 7) & 7) (SWIZZLE_128B as TMA wrote it, kept for the MMA)
      const int t = (warp - 1) * 32 + lane;
      int a_st = 0;
      uint32_t a_par = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        for (int kc = 0; kc < KC; ++kc) {
          mbar_wait(a_full(a_st), a_par);
          const uint32_t stage = a_base + a_st * A_STAGE;
          for (int r = t; r < HALO_ROWS; r += 32 * XFORM_WARPS) {
            const uint32_t row = stage + (uint32_t)r * 128u;
            const uint32_t ph = (row >> 7) & 7u;
            float f[32];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float4 v;
              asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(row + ((j ^ ph) << 4)));
              f[4 * j] = v.x; f[4 * j + 1] = v.y; f[4 * j + 2] = v.z; f[4 * j + 3] = v.w;
            }
            uint32_t hi[16], lo[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const __nv_bfloat162 h2 = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
              hi[i] = *reinterpret_cast<const uint32_t*>(&h2);
              const float r0 = f[2 * i] - __uint_as_float(hi[i] << 16), r1 = f[2 * i + 1] - __uint_as_float(hi[i] & 0xffff0000u);
              const __nv_bfloat162 l2 = __floats2bfloat162_rn(r0, r1);
              lo[i] = *reinterpret_cast<const uint32_t*>(&l2);
            }
#pragma unroll
            for (int m4 = 0; m4 < 4; ++m4) {
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(row + ((m4 ^ ph) << 4)), "r"(hi[4 * m4]), "r"(hi[4 * m4 + 1]), "r"(hi[4 * m4 + 2]), "r"(hi[4 * m4 + 3]) : "memory");
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(row + (((m4 + 4) ^ ph) << 4)), "r"(lo[4 * m4]), "r"(lo[4 * m4 + 1]), "r"(lo[4 * m4 + 2]), "r"(lo[4 * m4 + 3]) : "memory");
            }
          }
          fence_proxy_async_smem();   // generic-proxy writes -> visible to the tensor core's async-proxy reads
          __syncwarp();
          if (lane == 0) mbar_arrive(a_ready(a_st));
          if (++a_st == A_STAGES) { a_st = 0; a_par ^= 1; }
        }
      }
    }
    return;
  }

  // ================= consumers: warpgroup c owns the CTA's items k with k % 2 == c =================
  const int c = wg - 1;
  const int tw = warp & 3;                  // accumulator rows [16 tw, 16 tw + 16)
  const int qd = lane & 3;
  const bool leader = lane == 0;
  const float nw = (p.noise && p.noise_w) ? *p.noise_w : 0.f;
  float* epi = reinterpret_cast<float*>(smem_raw + (e_base - raw) + c * P::EPI_BYTES);
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  int a_st = 0, last_wb = -1;
  uint32_t a_par = 0, w_par = 0;
  for (int tile = blockIdx.x, k = 0; tile < p.total_tiles; tile += gridDim.x, ++k) {
    const int b = tile / tiles_per_img, rem = tile % tiles_per_img;
    const int oy0 = (rem / p.tiles_x) * TILE_H, ox0 = (rem % p.tiles_x) * TILE_W;
    const int wb = p.wB > 1 ? b : 0;
    if (wb != last_wb) {   // this warpgroup's MMAs on the previous weights have completed (wgmma_wait<0> after each item)
      if (last_wb >= 0 && leader) mbar_arrive(w_empty);
      mbar_wait(w_full, w_par);
      w_par ^= 1;
      last_wb = wb;
    }
    if ((k & 1) != c) {
      for (int kc = 0; kc < KC; ++kc) {
        mbar_wait(a_ready(a_st), a_par);
        if (leader) mbar_arrive(a_empty(a_st));
        if (++a_st == A_STAGES) { a_st = 0; a_par ^= 1; }
      }
      continue;
    }
    // The epilogue's global loads are issued now and complete while the MMAs run: the noise of every pixel this thread handles,
    // and the 2x2 up-sampled skip taps of the one pixel whose ToRGB it finishes.  Epilogue layout: pass q stages PJ tile rows;
    // thread et reads pixels pp + i * 128 / TPP (i < PPT) of each pass, channel groups t4 + kv * TPP.  Its ToRGB pixel is slot t4
    // (pass t4 / PPT, pixel t4 % PPT): NQ * PPT == TPP, so the TPP threads of a pixel finish TPP different pixels.
    constexpr int TPP = P::TPP, PPT = P::PPT, NQ = TILE_H / PJ;
    static_assert(NQ * PPT == TPP, "one ToRGB pixel per thread");
    const int et = threadIdx.x & 127;
    const int pp = et / TPP, t4 = et % TPP;
    float nzr[NQ][PPT];
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
      for (int i = 0; i < PPT; ++i) {
        const int px = pp + i * (128 / TPP), oy = oy0 + q * PJ + px / 8, ox = ox0 + px % 8;
        nzr[q][i] = (p.noise && oy < p.Ho && ox < p.Wo)
                        ? __ldg(p.noise + p.pix_off + (int64_t)b * p.pix_sb + (int64_t)oy * p.pix_sy + (int64_t)ox * p.pix_sx) : 0.f;
      }
    const int px_rgb = pp + (t4 % PPT) * (128 / TPP);
    const int oy_rgb = oy0 + (t4 / PPT) * PJ + px_rgb / 8, ox_rgb = ox0 + px_rgb % 8;
    const bool own_rgb = p.rgb_w && oy_rgb < p.Ho && ox_rgb < p.Wo;
    SkipTaps st = {};
    if (own_rgb && p.rgb_skip) skip_taps_load(p.rgb_skip, p.rgb_skip_kernel, b, oy_rgb, ox_rgb, p.Ho, p.Wo, st);
    float rgb_own[3] = {0.f, 0.f, 0.f};

    int rel_a = -1;   // stage the previous (still in flight) wgmma group reads, released once it has completed
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      mbar_wait(a_ready(a_st), a_par);
      const uint32_t xs = a_base + a_st * A_STAGE;
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int ky = t / 3, kx = t % 3;
        const uint64_t wdesc = make_smem_desc_sw128(w_base + kc * W_CHUNK + t * W_TAP, 1024);
        const uint64_t xdesc = make_smem_desc_sw128(xs + (uint32_t)(ky * HALO_W + kx) * 128u, HALO_W * 128);
        wgmma_fence();
        rs_mma_step<NSTACK>(acc, wdesc, xdesc, (kc == 0 && t == 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (leader && rel_a >= 0) mbar_arrive(a_empty(rel_a));
        rel_a = t == 8 ? a_st : -1;
      }
      if (++a_st == A_STAGES) { a_st = 0; a_par ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_pin<64>(acc);
    if (leader) mbar_arrive(a_empty(rel_a));

    // ---- epilogue.  Accumulator register i holds channel row 16 tw + lane/4 + 8 ((i/2)%2) and pixel column 8 (i/4) + 2 qd + (i%2),
    // i.e. tile row ty = i/4, x = 2 qd + (i%2).  Each pass stages PJ tile rows as [pixel][row] and then reads them per pixel.
    constexpr int NV = COUT / (4 * TPP);         // float4 channel groups per thread and pixel
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
#pragma unroll
      for (int jj = 0; jj < PJ; ++jj)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            epi[(jj * 8 + 2 * qd + e) * EP + 16 * tw + (lane >> 2) + 8 * h] = acc[4 * (q * PJ + jj) + 2 * h + e];
      named_bar_sync(1 + c, 128);
      int oy[PPT], ox[PPT];
      bool in_img[PPT];
      float nz[PPT], rgb[PPT][3];
#pragma unroll
      for (int i = 0; i < PPT; ++i) {
        const int px = pp + i * (128 / TPP);
        oy[i] = oy0 + q * PJ + px / 8; ox[i] = ox0 + px % 8;
        in_img[i] = oy[i] < p.Ho && ox[i] < p.Wo;
        nz[i] = (p.noise && in_img[i]) ? nw * nzr[q][i] : 0.f;
        rgb[i][0] = rgb[i][1] = rgb[i][2] = 0.f;
      }
#pragma unroll
      for (int i = 0; i < PPT; ++i) {
        const int px = pp + i * (128 / TPP);
        const int64_t off = p.out_off + (int64_t)b * p.out_sb + (int64_t)oy[i] * p.out_sy + (int64_t)ox[i] * p.out_sx;
#pragma unroll
        for (int kv = 0; kv < NV; ++kv) {
          const int ch = 4 * (kv * TPP + t4);
          float4 x = *reinterpret_cast<const float4*>(epi + px * EP + ch);
          if constexpr (NSTACK) {   // + the w_lo products of the same channels
            const float4 y = *reinterpret_cast<const float4*>(epi + px * EP + ch + 32);
            x.x += y.x; x.y += y.y; x.z += y.z; x.w += y.w;
          }
          float v[4] = {x.x * p.acc_scale, x.y * p.acc_scale, x.z * p.acc_scale, x.w * p.acc_scale};
          const float4 bq = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + ch)) : make_float4(0.f, 0.f, 0.f, 0.f);
          v[0] += bq.x + nz[i]; v[1] += bq.y + nz[i]; v[2] += bq.z + nz[i]; v[3] += bq.w + nz[i];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (p.act == VT_ACT_LRELU) v[u] = vt_lrelu(v[u], p.slope) * p.gain;
            if (p.round_tf32) v[u] = vt_round_tf32(v[u]);
          }
          if (p.rgb_w) {
            // 1x1 modulated conv to 3 channels on the values just produced (model/stylegan/model.py:384-385)
            const float* w0 = p.rgb_w + ((int64_t)(p.wB > 1 ? b : 0) * 3) * COUT + ch;
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) {
              const float4 wv = __ldg(reinterpret_cast<const float4*>(w0 + cc * COUT));
              rgb[i][cc] = fmaf(v[3], wv.w, fmaf(v[2], wv.z, fmaf(v[1], wv.y, fmaf(v[0], wv.x, rgb[i][cc]))));
            }
          }
          if (in_img[i] && p.out) *reinterpret_cast<float4*>(p.out + off + ch) = make_float4(v[0], v[1], v[2], v[3]);
        }
      }
      if (p.rgb_w) {
        // butterfly over the pixel's TPP threads (every one ends with the full sum); the thread of slot q * PPT + i keeps it
#pragma unroll
        for (int i = 0; i < PPT; ++i) {
#pragma unroll
          for (int cc = 0; cc < 3; ++cc)
#pragma unroll
            for (int o = 1; o < TPP; o <<= 1) rgb[i][cc] += __shfl_xor_sync(0xffffffffu, rgb[i][cc], o);
          if (t4 == q * PPT + i) { rgb_own[0] = rgb[i][0]; rgb_own[1] = rgb[i][1]; rgb_own[2] = rgb[i][2]; }
        }
      }
      named_bar_sync(1 + c, 128);
    }
    if (own_rgb) torgb_store_taps(p.rgb_bias, p.rgb_skip != nullptr, st, p.rgb_out, rgb_own, b, oy_rgb, ox_rgb, p.Ho, p.Wo);
  }
}

struct RsKernel {
  int cin, cout;
  uint32_t smem;
  void (*fn)(RsArgs);
};
#define VT_RS(CIN, COUT) {CIN, COUT, RsPlan<CIN>::SMEM, conv_rs_kernel<CIN, COUT>}
const RsKernel kRsKernels[] = {VT_RS(32, 32), VT_RS(32, 64), VT_RS(64, 32), VT_RS(64, 64)};
#undef VT_RS

}  // namespace

// Descriptors conv_rs_kernel takes (vt_conv2d_rs has already checked the row-strip shape: one source, 3x3, stride 1, one phase,
// Cin and Cout in {32, 64}, no residual / per-channel slope / source scaling): the bf16 split (N-stacked exactly when Cout == 32),
// the taps of a 3x3 / padding 1 cross-correlation in raster order on slabs 0..8, and no instance-norm statistics.
int vt_conv_rs_takes(const vt_conv_desc* d) {
  if (!d->weight_bf16x3 || d->split_fmt != 0 || (d->bf16x3_nstack != 0) != (d->Cout == 32) || d->stats_ws) return 0;
  if (d->taps != 9 || d->w_taps != 9) return 0;
  for (int t = 0; t < 9; ++t)
    if (d->tap_dy[t] != t / 3 - 1 || d->tap_dx[t] != t % 3 - 1 || d->tap_w[t] != t) return 0;
  if (d->noise && (d->out_sb % d->out_cpitch || d->out_sy % d->out_cpitch || d->out_sx % d->out_cpitch || d->phase_off[0] % d->out_cpitch)) return 0;
  return vt_conv2d_tc_supported(d);
}

int vt_conv_rs_run(const vt_conv_desc* d, void* stream) {
  if (vt_validate_conv_desc(d, "conv2d_rs")) return 1;
  static thread_local RsArgs a;
  memset(&a, 0, sizeof(a));
  const int cin = d->src_c[0];
  a.B = d->B; a.Ho = d->Ho; a.Wo = d->Wo; a.wB = d->wB;
  a.tiles_x = (int)vt_cdiv(d->Wo, TILE_W);
  a.tiles_y = (int)vt_cdiv(d->Ho, TILE_H);
  const int64_t total = (int64_t)a.tiles_x * a.tiles_y * d->B;
  VT_CHECK(total < (1LL << 31), "conv2d_rs: too many tiles");
  a.total_tiles = (int)total;
  a.bias = d->bias; a.noise = d->noise; a.noise_w = d->noise_w; a.out = d->out;
  a.out_off = d->phase_off[0]; a.out_sb = d->out_sb; a.out_sy = d->out_sy; a.out_sx = d->out_sx;
  if (d->noise) {
    a.pix_off = d->phase_off[0] / d->out_cpitch;
    a.pix_sb = d->out_sb / d->out_cpitch; a.pix_sy = d->out_sy / d->out_cpitch; a.pix_sx = d->out_sx / d->out_cpitch;
  }
  a.act = d->act; a.round_tf32 = d->round_tf32; a.slope = d->slope; a.gain = d->gain;
  a.acc_scale = d->acc_scale > 0.f ? d->acc_scale : 1.f;
  a.rgb_w = d->rgb_w; a.rgb_bias = d->rgb_bias; a.rgb_skip = d->rgb_skip; a.rgb_skip_kernel = d->rgb_skip_kernel; a.rgb_out = d->rgb_out;
  {
    // activations: (channels, x, y, batch) fp32, one (32, 10, 18, 1) halo box per K chunk; out-of-image pixels are zero-filled
    const uint64_t cs = (uint64_t)d->src_cstride[0];
    const uint64_t dims[4] = {cs, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->B};
    const uint64_t str[3] = {cs * 4, (uint64_t)d->W * cs * 4, (uint64_t)d->H * d->W * cs * 4};
    const uint32_t box[4] = {32, HALO_W, HALO_H, 1};
    if (vt_tc_make_map4(&a.in_map, d->src[0], dims, str, box, "input", false)) return 1;
  }
  {
    // weights: 64 bf16 rows per tap (Cout = 64 rows [w_hi | w_lo], or the N-stacked 2 x 32 rows), one (64, 64, 9, 1) box per K chunk
    VT_CHECK(((uintptr_t)d->weight_bf16x3 & 15) == 0, "conv2d_rs: weight_bf16x3 not 16-byte aligned");
    const uint64_t wc = (uint64_t)d->w_cstride;
    const uint64_t dims[4] = {2 * wc, 64, 9, (uint64_t)d->wB};
    const uint64_t str[3] = {wc * 4, 64 * wc * 4, 9 * 64 * wc * 4};
    const uint32_t box[4] = {64, 64, 9, 1};
    if (vt_tc_make_map4(&a.w_map, d->weight_bf16x3, dims, str, box, "weight(bf16x3)", true)) return 1;
  }
  static std::once_flag attr_once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once, [] {
    for (const RsKernel& k : kRsKernels)
      if (attr_err == cudaSuccess) attr_err = cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.smem);
  });
  VT_CHECK(attr_err == cudaSuccess, "conv2d_rs: cudaFuncSetAttribute failed: %s", cudaGetErrorString(attr_err));
  const RsKernel* kern = nullptr;
  for (const RsKernel& k : kRsKernels)
    if (k.cin == cin && k.cout == d->Cout) kern = &k;
  VT_CHECK(kern != nullptr, "conv2d_rs: no kernel for %d -> %d channels", cin, d->Cout);
  int grid = vt_num_sms();
  if (grid > a.total_tiles) grid = a.total_tiles;
  kern->fn<<<grid, RS_THREADS, kern->smem, (cudaStream_t)stream>>>(a);
  VT_LAUNCH_CHECK();
  return 0;
}
