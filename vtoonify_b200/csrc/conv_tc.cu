// conv_tc.cu — the hot kernel: NHWC convolution as an implicit GEMM on the Hopper tensor cores (wgmma).
//
//   D[128 pixels, N couts] (registers, fp32) += A[128 pixels, 32 ch] (smem, TF32) * W[N couts, 32 ch]^T (smem, TF32)
//
// One persistent CTA per SM, three warpgroups:
//   warp 0 (1 lane)  TMA producer : activation tiles are 4-D boxes (32 ch, 8 x, 16 y, 1 b) of the NHWC tensor, shifted by
//                                   the filter tap; out-of-image pixels are zero-filled by TMA == the conv's zero padding,
//                                   so there is no im2col buffer and no bounds code.  Weight tiles are (32 ch, N, 1 tap, 1 b)
//                                   boxes of the per-sample modulated/demodulated weights [b][tap][cout][cin].
//   warps 1-3        operand transform (bf16x3 only): fp32 rows -> [hi | lo] 16-bit rows, in place.
//   warpgroups 1, 2  consumers    : each owns 64 of the 128 pixels (8 rows of the 8 x 16 tile): wgmma m64nNk8 (tf32) or
//                                   m64nNk16 (bf16 / fp16 split operands, N <= 128), fp32 accumulators in registers, one wgmma group
//                                   kept in flight while the next stage is awaited; then the epilogue straight from the
//                                   accumulator registers (+noise, +bias, leaky-relu*gain, residual, TF32 rna, fused ToRGB,
//                                   instance-norm partial sums) with direct global stores.
//                                   conv_tc_pingpong_kernel: each warpgroup owns alternate work items whole (all 128 pixels),
//                                   so one item's epilogue runs under the other warpgroup's MMAs.
//
// A-operand reuse ("halo" mode, stride-1 convs): one TMA box of (8+2d) x (16+2d) pixels per 32-channel chunk serves all
// 9 taps; each tap's MMA reads it through a descriptor whose start address is shifted by whole 128-byte rows and whose
// stride-byte-offset is the halo row pitch, so the activations cross L2->smem once instead of nine times.
//
// The modulated convolution of the reference (model/stylegan/model.py:259-304: per-sample weights + grouped conv) and the
// plain convs (model/vtoonify.py:96-97,111-113,162-182) are the same GEMM here; a stride-2 transposed conv is 4 polyphase
// calls, a stride-2 conv reads 4 parity views of the input (see make_views()).
#include "tc_common.cuh"
#include <cuda_bf16.h>
#include <mutex>

using namespace vt_tc;

int vt_validate_conv_desc(const vt_conv_desc* d, const char* who);
extern int g_upfirdn_tiled;
extern int g_smalln_is;
extern int g_fir4;
extern int g_instnorm_chunks;
extern int g_rs_kernel;
int vt_conv_rs_takes(const vt_conv_desc* d);
int vt_conv_rs_run(const vt_conv_desc* d, void* stream);

namespace {

constexpr int TILE_W = 8, TILE_H = 16, TILE_M = 128;
constexpr int KCH = 32;                       // fp32 channels per K chunk = one 128-byte swizzle row
constexpr int MAX_SMEM = 227 * 1024;
constexpr int MAX_BLOCK_N = 128;              // largest N tile (wgmma N) of one work item under the flat register budget
constexpr int MAX_ACC_COLS = 128;             // accumulator columns per consumer thread group: mt * mma_n (64 registers) under the flat
                                              // budget of 168 registers per thread; 256 columns spill there
// The wide work item: 128 pixels x 256 output channels on m64n256k16 (bf16 split only, one M tile).  Its 256 accumulator
// columns (128 registers) fit because warpgroup 0 (producer + transform warps) hands registers to the two consumer
// warpgroups with setmaxnreg: 128 * WIDE_REGS_XFORM + 256 * WIDE_REGS_CONSUMER <= 384 * 168, the launch allocation.  The
// ping-pong item (two 64 x 128 accumulators per consumer thread) uses the same plan.
constexpr int WIDE_N = 256;
constexpr int WIDE_REGS_XFORM = 88;
constexpr int WIDE_REGS_CONSUMER = 208;
constexpr int STATS_WARPS = 8;                // instance-norm chunks per 128-pixel tile: one per consumer warp (16 pixels)

struct TcArgs {
  CUtensorMap in_map[2][4];
  CUtensorMap w_map;
  int n_src, kchunks[2], coff[2];
  // "B steps": one weight tile (tap of one phase) each; every step feeds `mt` accumulators (the M tiles of the work item)
  int n_steps;
  int8_t step_view[VT_MAX_TAPS], step_vx[VT_MAX_TAPS], step_vy[VT_MAX_TAPS];
  int16_t step_w[VT_MAX_TAPS];
  int step_aoff[VT_MAX_TAPS];                  // halo mode: byte offset of the tap's first row inside the halo box
  int n_phase;                                 // the N dimension is phase-major [n_phase][Cout] (folded up-conv), else 1
  int tgroup;                                  // taps per weight TMA box / pipeline step (consecutive slabs)
  int halo, halo_x0, halo_y0, halo_w;   // halo staging; x0/y0/w describe view 0's box (stride 1: the only one)
  // halo boxes of one K chunk: stride 1 has one, stride 2 one per parity view in use (each with its own extent and pitch)
  int n_hv, hv_view[4], hv_x0[4], hv_y0[4], hv_off[4], hv_bytes[4], a_rows;
  uint16_t step_sbo[VT_MAX_TAPS];   // halo mode: stride (bytes) between 8-pixel row groups of the tap's box
  int a_stages, b_stages, a_stage_bytes, b_stage_bytes, a_tx_bytes, b_tx_bytes;
  int block_n, n_tiles, tiles_x, tiles_y, B, total_tiles;
  int m_first;               // first pixel tile of this launch: a layer may run its pixel tiles as a wide and a narrow launch
  int Ho, Wo, Cout, wB, out_cpitch;
  const float* bias;
  const float* noise;
  const float* noise_w;
  const float* res;
  float* out;
  int64_t out_sb, out_sy, out_sx, phase_off[4];
  int64_t pix_sb, pix_sy, pix_sx, phase_pix[4];   // the same view in dense-pixel units (noise index), = offsets / out_cpitch
  int act, round_tf32;
  float slope, gain, alpha, beta;
  // fused ToRGB tail
  const float* rgb_w; const float* rgb_bias; const float* rgb_skip; const float* rgb_skip_kernel; float* rgb_out;
  const float* slope_vec;
  const float* src_scale[2]; // bf16x3: optional planar per-pixel multiplier of source s (kernel-space strides below)
  const float* src_affine[2];  // bf16x3: optional [B][C_s][2] (scale, shift) applied to in-image pixels of source s
  int src_cn[2];             // channels of source s (row length of src_affine)
  int64_t sc_sb, sc_sy, sc_sx;
  int in_w, in_h;            // kernel-space input extents
  int mma_n;                 // N of one MMA: block_n, or 2*block_n in the N-stacked bf16x3 form
  int m_major;               // work-item order: the N tiles of one pixel tile are neighbours (run on neighbouring SMs at the same
                             // time, so the second read of the activations hits L2) instead of N-tile-major
  float* stats_ws;           // optional instance-norm partials of the OUTPUT in the layout of vt_instnorm_finalize_f32 (pivot,
                             // deviation sum, square sum about the pivot), one chunk per (pixel tile, consumer warp)
  int64_t stats_e;           // entries per partial array: chunks * B * Cout
  int* stats_cnt;            // [chunk] in-image pixels of each chunk (after the three arrays)
  float acc_scale;           // accumulators are multiplied by this first (undoes the power-of-two weight scale of the fp16 split)
};

constexpr int TC_THREADS = 384;
constexpr int XFORM_WARPS = 3;
constexpr int CONSUMERS = 2;
// wgmma.wait_group covers the executing warp's share of a warpgroup MMA only: every consumer warp releases a stage it has read
constexpr int RELEASE_ARRIVALS = CONSUMERS * 4;

// Operand mode of the MMAs, a template parameter of the kernel together with N and the M tiles per work item: every tap step
// is then straight-line code (fence, the MMAs of all M tiles, commit) and compiles to one hardware wgmma group.  Runtime
// control flow between the fence and the commit makes ptxas split the step into several groups and close it with a
// placeholder group, so that waiting for "all but one" group waits for the step's own MMAs and drains the tensor pipe.
enum TcOp : int {
  OP_TF32 = 0,          // fp32 operands read as TF32: 4 MMAs m64nNk8 per 32-channel chunk
  OP_BF16 = 1,          // bf16 hi/lo split operands, 3 products: 6 MMAs m64nNk16
  OP_F16 = 2,           // fp16 hi/lo split operands (split_fmt = 1), 3 products
  OP_BF16_NSTACK = 3,   // bf16 split, Cout == 32: weight rows [w_hi|w_hi] x32 then [w_lo|w_lo] x32 -> 4 MMAs of N = 64, halves
                        // summed in the epilogue
};

template <int NW, bool F16>
__device__ __forceinline__ void wgmma_split(float* acc, uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (NW == 32) {
    if constexpr (F16) wgmma_f16_n32(acc, a, b, accumulate); else wgmma_bf16_n32(acc, a, b, accumulate);
  } else if constexpr (NW == 64) {
    if constexpr (F16) wgmma_f16_n64(acc, a, b, accumulate); else wgmma_bf16_n64(acc, a, b, accumulate);
  } else if constexpr (NW == 128) {
    if constexpr (F16) wgmma_f16_n128(acc, a, b, accumulate); else wgmma_bf16_n128(acc, a, b, accumulate);
  } else {
    static_assert(NW == WIDE_N && !F16, "the 256-wide MMA exists for the bf16 split only");
    wgmma_bf16_n256(acc, a, b, accumulate);
  }
}

// one K step of one accumulator: the products of a 32-channel chunk (4 tf32 MMAs, or the split-operand MMAs)
template <int NW, int OP>
__device__ __forceinline__ void mma_step(float* acc, uint64_t adesc, uint64_t bdesc, uint32_t first) {
  if constexpr (OP == OP_TF32) {
    if constexpr (NW == 32) {
      wgmma_tf32_n32(acc, adesc, bdesc, first ^ 1u); wgmma_tf32_n32(acc, adesc + 2, bdesc + 2, 1);
      wgmma_tf32_n32(acc, adesc + 4, bdesc + 4, 1); wgmma_tf32_n32(acc, adesc + 6, bdesc + 6, 1);
    } else if constexpr (NW == 64) {
      wgmma_tf32_n64(acc, adesc, bdesc, first ^ 1u); wgmma_tf32_n64(acc, adesc + 2, bdesc + 2, 1);
      wgmma_tf32_n64(acc, adesc + 4, bdesc + 4, 1); wgmma_tf32_n64(acc, adesc + 6, bdesc + 6, 1);
    } else {
      wgmma_tf32_n128(acc, adesc, bdesc, first ^ 1u); wgmma_tf32_n128(acc, adesc + 2, bdesc + 2, 1);
      wgmma_tf32_n128(acc, adesc + 4, bdesc + 4, 1); wgmma_tf32_n128(acc, adesc + 6, bdesc + 6, 1);
    }
  } else {
    // The A row is [a_hi(32)|a_lo(32)] and the B row [w_hi(32)|w_lo(32)] 16-bit; +2 on a descriptor = +32 B = 16 elements of K.
    //   nstack:  [a_hi|a_lo] (K = 64) x rows [w_hi|w_hi] (columns 0..31) and [w_lo|w_lo] (columns 32..63): all four products
    //   else:    a*w ~= a_hi*w_hi + a_lo*w_hi + a_hi*w_lo (the dropped a_lo*w_lo term is ~2^-18 relative)
    constexpr bool nstack = OP == OP_BF16_NSTACK;
    constexpr int ao[6] = {0, 2, 4, 6, 0, 2};
    constexpr int bo[6] = {0, 2, 0, 2, 4, 6};
#pragma unroll
    for (int i = 0; i < (nstack ? 4 : 6); ++i)
      wgmma_split<NW, OP == OP_F16>(acc, adesc + (uint64_t)ao[i], bdesc + (uint64_t)(nstack ? ao[i] : bo[i]), i == 0 ? (first ^ 1u) : 1u);
  }
}

// NW: MMA N (accumulator columns per M tile); MT: M tiles (accumulators) per work item; OP: operand mode (TcOp);
// PP: ping-pong (conv_tc_pingpong_kernel): each consumer warpgroup owns whole work items, both 64-row halves of every M tile
template <int NW, int MT, int OP, bool PP>
__device__ __forceinline__ void conv_tc_body(const TcArgs& p) {
  // The wide item and the ping-pong item hold 128 accumulator registers per consumer thread; they are the instantiations that
  // reallocate registers between the warpgroups.  Their epilogue leaves out the fused ToRGB and the tanh activation (the
  // planner never gives them those layers): with them, the fully unrolled 8-chunk epilogue made the wide kernel 11.6k
  // instructions, which no longer stay in the instruction cache, and every layer ran slower wide than 128-wide; without them
  // it is 7.0k, the size of the 128-wide kernel.
  constexpr bool WIDE = NW == WIDE_N;
  constexpr bool REALLOC = WIDE || PP;
  constexpr int HALVES = PP ? 2 : 1;   // 64-row halves of an M tile one consumer warpgroup computes
  static_assert((MT * NW <= MAX_ACC_COLS || (WIDE && MT == 1 && OP == OP_BF16)) && (MT == 1 || MT == 2 || MT == 4),
                "accumulators of one work item exceed the register plan");
  static_assert(!PP || (NW == MAX_BLOCK_N && MT == 1 && OP == OP_BF16), "the ping-pong item is the 128 x 128 bf16-split item");
  // ping-pong: a stage is released by the 4 warps of the warpgroup that owns the item reading it
  constexpr int RELEASES = PP ? 4 : RELEASE_ARRIVALS;
  static_assert(128 * WIDE_REGS_XFORM + 256 * WIDE_REGS_CONSUMER <= TC_THREADS * ((65536 / TC_THREADS) & ~7),
                "setmaxnreg plan exceeds the launch allocation");
  static_assert(OP != OP_BF16_NSTACK || NW == 64, "the N-stacked form is the Cout == 32 layer at MMA N = 64");
  constexpr bool SPLIT = OP != OP_TF32;   // operands split into 16-bit hi/lo rows in shared memory by the transform warps
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B swizzle atoms
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = a_base + (uint32_t)p.a_stages * p.a_stage_bytes;
  const uint32_t bar_base = b_base + (uint32_t)p.b_stages * p.b_stage_bytes;
  // barriers: a_full[8] a_empty[8] b_full[8] b_empty[8] a_ready[8]
  auto a_full = [&](int i) { return bar_base + 8u * i; };
  auto a_empty = [&](int i) { return bar_base + 64u + 8u * i; };
  auto b_full = [&](int i) { return bar_base + 128u + 8u * i; };
  auto b_empty = [&](int i) { return bar_base + 192u + 8u * i; };
  auto a_ready = [&](int i) { return bar_base + 256u + 8u * i; };   // bf16x3: A stage converted to [hi|lo] 16-bit rows
  auto turn = [&](int c) { return bar_base + 320u + 8u * c; };      // ping-pong: consumer warpgroup c may run its main loop

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < p.n_src; ++s)
      for (int v = 0; v < 4; ++v) tma_prefetch_desc(&p.in_map[s][v]);
    tma_prefetch_desc(&p.w_map);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < p.a_stages; ++i) { mbar_init(a_full(i), 1); mbar_init(a_empty(i), RELEASES); mbar_init(a_ready(i), XFORM_WARPS); }
    for (int i = 0; i < p.b_stages; ++i) { mbar_init(b_full(i), 1); mbar_init(b_empty(i), RELEASES); }
    if constexpr (PP) { mbar_init(turn(0), 4); mbar_init(turn(1), 4); }
    fence_barrier_init();
    fence_proxy_async_smem();
  }
  __syncthreads();

  const int m_tiles = p.total_tiles / p.n_tiles;   // pixel tiles of this launch, from p.m_first on
  const int tiles_per_img = p.tiles_y * p.tiles_x;
  constexpr int item_w = TILE_W * MT;   // a work item covers item_w x TILE_H output pixels

  if (wg == 0) {
    if constexpr (REALLOC) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WIDE_REGS_XFORM));
    if (warp == 0) {
      // ================= TMA producer (whole warp converged; one elected lane issues) =================
      int a_st = 0, b_st = 0;
      uint32_t a_par = 0, b_par = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int n_tile = p.m_major ? tile % p.n_tiles : tile / m_tiles, m = p.m_first + (p.m_major ? tile / p.n_tiles : tile % m_tiles);
        const int b = m / tiles_per_img, rem = m % tiles_per_img;
        const int oy0 = (rem / p.tiles_x) * TILE_H, ox0 = (rem % p.tiles_x) * item_w;
        const int n0 = n_tile * p.block_n;
        const int wb = p.wB > 1 ? b : 0;
        for (int s = 0; s < p.n_src; ++s) {
          for (int kc = 0; kc < p.kchunks[s]; ++kc) {
            const int c0 = kc * KCH;
            if (p.halo) {
              mbar_wait(a_empty(a_st), a_par ^ 1);
              if (elect_one()) {
                const uint32_t st = a_base + a_st * p.a_stage_bytes;
                mbar_arrive_expect_tx(a_full(a_st), (uint32_t)p.a_tx_bytes);
                for (int v = 0; v < p.n_hv; ++v)
                  tma_load_4d(st + p.hv_off[v], &p.in_map[s][p.hv_view[v]], a_full(a_st), c0, ox0 + p.hv_x0[v], oy0 + p.hv_y0[v], b);
              }
              __syncwarp();
              if (++a_st == p.a_stages) { a_st = 0; a_par ^= 1; }
            }
            int gj = 0;   // position inside the current tap group
            for (int j = 0; j < p.n_steps; ++j) {
              if (!p.halo) {
                mbar_wait(a_empty(a_st), a_par ^ 1);
                if (elect_one()) {
                  mbar_arrive_expect_tx(a_full(a_st), (uint32_t)p.a_tx_bytes);
                  tma_load_4d(a_base + a_st * p.a_stage_bytes, &p.in_map[s][p.step_view[j]], a_full(a_st), c0, ox0 + p.step_vx[j],
                              oy0 + p.step_vy[j], b);
                }
                __syncwarp();
                if (++a_st == p.a_stages) { a_st = 0; a_par ^= 1; }
              }
              if (gj == 0) {
                // one TMA box carries the weight tiles of `tgroup` consecutive taps: (32 ch, block_n, tgroup, 1)
                mbar_wait(b_empty(b_st), b_par ^ 1);
                if (elect_one()) {
                  // bf16x3: the weight row of a 32-channel chunk is one 128-byte 16-bit row [w_hi(32) | w_lo(32)]
                  const int wc = SPLIT ? (p.coff[s] + c0) * 2 : p.coff[s] + c0;
                  mbar_arrive_expect_tx(b_full(b_st), (uint32_t)p.b_tx_bytes);
                  tma_load_4d(b_base + b_st * p.b_stage_bytes, &p.w_map, b_full(b_st), wc, OP == OP_BF16_NSTACK ? 0 : n0, p.step_w[j], wb);
                }
                __syncwarp();
                if (++b_st == p.b_stages) { b_st = 0; b_par ^= 1; }
              }
              if (++gj == p.tgroup) gj = 0;
            }
          }
        }
      }
    } else if constexpr (SPLIT) {
      // ================= operand transform (bf16x3): fp32 rows -> [hi(32) | lo(32)] 16-bit rows, in place =================
      // A 32-channel fp32 row (128 B) becomes the K = 64 row [a_hi | a_lo] with a_hi = bf16(a), a_lo = bf16(a - a_hi);
      // 16-byte chunk j of the row lives at physical chunk j ^ ((addr >> 7) & 7) (SWIZZLE_128B as TMA wrote it, kept for the MMA).
      const int t = (warp - 1) * 32 + lane;   // 0 .. 32 * XFORM_WARPS
      const int rows = p.a_rows;
      int a_st = 0;
      uint32_t a_par = 0;
      const int bw = p.halo ? p.halo_w : TILE_W;   // pixels per box row
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int m = p.m_first + (p.m_major ? tile / p.n_tiles : tile % m_tiles);
        const int b = m / tiles_per_img, rem = m % tiles_per_img;
        const int oy0 = (rem / p.tiles_x) * TILE_H, ox0 = (rem % p.tiles_x) * item_w;
        for (int s = 0; s < p.n_src; ++s) {
          const float* sc = p.src_scale[s];
          const float* aff = p.src_affine[s];
          for (int kc = 0; kc < p.kchunks[s]; ++kc) {
            const float4* affp = aff ? reinterpret_cast<const float4*>(aff + ((int64_t)b * p.src_cn[s] + kc * KCH) * 2) : nullptr;
            const int loads = p.halo ? 1 : p.n_steps;
            for (int l = 0; l < loads; ++l) {
              mbar_wait(a_full(a_st), a_par);
              const uint32_t stage = a_base + a_st * p.a_stage_bytes;
              const int bx0 = ox0 + (p.halo ? p.halo_x0 : p.step_vx[l]), by0 = oy0 + (p.halo ? p.halo_y0 : p.step_vy[l]);
              for (int r = t; r < rows; r += 32 * XFORM_WARPS) {
                const uint32_t row = stage + (uint32_t)r * 128u;
                const uint32_t ph = (row >> 7) & 7u;
                float f[32];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  float4 v;
                  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(row + ((j ^ ph) << 4)));
                  f[4 * j] = v.x; f[4 * j + 1] = v.y; f[4 * j + 2] = v.z; f[4 * j + 3] = v.w;
                }
                if (sc || aff) {   // rows are box pixels in raster order
                  const int ry = r / bw, rx = r - ry * bw;
                  const int ix = bx0 + rx, iy = by0 + ry;
                  const bool inb = ix >= 0 && ix < p.in_w && iy >= 0 && iy < p.in_h;
                  if (aff && inb) {   // per-(sample, channel) affine (AdaIN) on real pixels; the zero padding stays zero
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                      const float4 q = __ldg(affp + j);   // (scale, shift) of channels 2j, 2j+1 (same address in every thread)
                      f[2 * j] = fmaf(f[2 * j], q.x, q.y);
                      f[2 * j + 1] = fmaf(f[2 * j + 1], q.z, q.w);
                    }
                  }
                  if (sc) {           // per-pixel multiplier of this source (f_E * m_E)
                    const float mm = inb ? __ldg(sc + (int64_t)b * p.sc_sb + (int64_t)iy * p.sc_sy + (int64_t)ix * p.sc_sx) : 0.f;
#pragma unroll
                    for (int i = 0; i < 32; ++i) f[i] *= mm;
                  }
                }
                uint32_t hi[16], lo[16];
                if constexpr (OP == OP_F16) {
#pragma unroll
                  for (int i = 0; i < 16; ++i) split_f16x2(f[2 * i], f[2 * i + 1], hi[i], lo[i]);
                } else {
#pragma unroll
                  for (int i = 0; i < 16; ++i) {
                    // packed converts (one cvt.rn.bf16x2.f32 per pair); a bf16 widened to fp32 is its bits shifted left by 16
                    const __nv_bfloat162 h2 = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
                    hi[i] = *reinterpret_cast<const uint32_t*>(&h2);
                    const float r0 = f[2 * i] - __uint_as_float(hi[i] << 16), r1 = f[2 * i + 1] - __uint_as_float(hi[i] & 0xffff0000u);
                    const __nv_bfloat162 l2 = __floats2bfloat162_rn(r0, r1);
                    lo[i] = *reinterpret_cast<const uint32_t*>(&l2);
                  }
                }
#pragma unroll
                for (int m4 = 0; m4 < 4; ++m4) {
                  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(row + ((m4 ^ ph) << 4)), "r"(hi[4 * m4]), "r"(hi[4 * m4 + 1]), "r"(hi[4 * m4 + 2]), "r"(hi[4 * m4 + 3]) : "memory");
                  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(row + (((m4 + 4) ^ ph) << 4)), "r"(lo[4 * m4]), "r"(lo[4 * m4 + 1]), "r"(lo[4 * m4 + 2]), "r"(lo[4 * m4 + 3]) : "memory");
                }
              }
              // generic-proxy writes -> visible to the tensor core's async-proxy reads
              fence_proxy_async_smem();
              __syncwarp();
              if (lane == 0) mbar_arrive(a_ready(a_st));
              if (++a_st == p.a_stages) { a_st = 0; a_par ^= 1; }
            }
          }
        }
      }
    }
  } else {
    // ================= consumers: wgmma main loop + epilogue =================
    // Cooperative (PP = false): both warpgroups work on every item, warpgroup c on pixel rows [8c, 8c + 8) of the 8 x 16 tile,
    // and every stage is released by all 8 consumer warps.
    // Ping-pong (PP = true): warpgroup c owns the CTA's items k with k % 2 == c and computes all 16 rows of them, so its
    // epilogue runs while the other warpgroup's MMAs keep the tensor cores busy.  Invariants:
    //   * the producer and the transform warps fill the stages in the cooperative order; a stage use is released once, by the
    //     4 warps of the warpgroup whose item reads it (empty barriers count 4);
    //   * the warpgroup that does not own item k reads none of its stages and does not wait for them: it only advances its
    //     ring indices and parities over them, by the stage counts the plan fixes per item (a_item halo or per-tap stages,
    //     b_item weight stages);
    //   * the main loops run in item order: warpgroup c waits on turn(c) before item k's first stage (k > 0) and arrives on
    //     turn(1 - c) after item k's last commit.  So every stage use before item k has been waited on (its full phase has
    //     completed) when item k's owner waits for its own phase: an mbarrier parity wait never sees a phase two steps away;
    //   * a CTA whose item count is odd, or 1, just leaves the last hand-off unwaited.
    if constexpr (REALLOC) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WIDE_REGS_CONSUMER));
    const int c = wg - 1;
    const int tw_ = (threadIdx.x & 127) >> 5;   // warp inside the warpgroup: accumulator rows [16 tw_, 16 tw_ + 16)
    const bool leader = lane == 0;   // one arrival per consumer warp
    const int qd = lane & 3;                    // column pair inside each 8-column group
    float acc[MT * HALVES][NW / 2];
#pragma unroll
    for (int g = 0; g < MT * HALVES; ++g)
#pragma unroll
      for (int i = 0; i < NW / 2; ++i) acc[g][i] = 0.f;
    const float nw = (p.noise && p.noise_w) ? *p.noise_w : 0.f;
    int a_st = 0, b_st = 0;
    uint32_t a_par = 0, b_par = 0;
    const uint32_t tile_bytes_n = (uint32_t)p.mma_n * 128u;   // bytes of one tap's weight rows
    int a_item = 0, b_item = 0;   // ping-pong: A and weight stages of one work item
    uint32_t t_par = 0;
    if constexpr (PP) {
      for (int s = 0; s < p.n_src; ++s) {
        a_item += p.halo ? p.kchunks[s] : p.kchunks[s] * p.n_steps;
        b_item += p.kchunks[s] * (p.n_steps / p.tgroup);
      }
    }
    for (int tile = blockIdx.x, item = 0; tile < p.total_tiles; tile += gridDim.x, ++item) {
      const int n_tile = p.m_major ? tile % p.n_tiles : tile / m_tiles, m = p.m_first + (p.m_major ? tile / p.n_tiles : tile % m_tiles);
      const int b = m / tiles_per_img, rem = m % tiles_per_img;
      const int oy0 = (rem / p.tiles_x) * TILE_H, ox0 = (rem % p.tiles_x) * item_w;
      const int n0 = n_tile * p.block_n;
      if constexpr (PP) {
        if ((item & 1) != c) {
          for (a_st += a_item; a_st >= p.a_stages; a_st -= p.a_stages) a_par ^= 1;
          for (b_st += b_item; b_st >= p.b_stages; b_st -= p.b_stages) b_par ^= 1;
          continue;
        }
        // The epilogue's global reads are requested now and land while the MMAs run: the noise of every pixel this thread
        // stores (each phase of a folded up-convolution is its own word) into L1, and the thread's 128-byte line of each
        // pixel's residual row into L2 (an item's residual is 64 KB, more than the L1 left beside the pipeline's shared memory).
        const int ph_first = n0 / p.Cout, ph_last = (n0 + p.block_n - 1) / p.Cout;
#pragma unroll
        for (int hh = 0; hh < HALVES; ++hh)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = 64 * hh + 16 * tw_ + (lane >> 2);
            const int oy = oy0 + r / TILE_W + h, ox = ox0 + r % TILE_W;
            if (oy >= p.Ho || ox >= p.Wo) continue;
            if (p.noise) {
              const int64_t pix = (int64_t)b * p.pix_sb + (int64_t)oy * p.pix_sy + (int64_t)ox * p.pix_sx;
              for (int ph = ph_first; ph <= ph_last; ++ph) asm volatile("prefetch.global.L1 [%0];" ::"l"(p.noise + p.phase_pix[ph] + pix));
            }
            if (p.res) {
              const int64_t off = p.phase_off[ph_first] + (int64_t)b * p.out_sb + (int64_t)oy * p.out_sy + (int64_t)ox * p.out_sx +
                                  (n0 - ph_first * p.Cout) + 32 * qd;
              asm volatile("prefetch.global.L2 [%0];" ::"l"(p.res + off));
            }
          }
        if (item > 0) { mbar_wait(turn(c), t_par); t_par ^= 1; }
      }
      uint32_t first = 1;   // first K step of this work item overwrites the accumulators
      int rel_a = -1, rel_b = -1;   // stages the previous (still in flight) wgmma group reads, released once it has completed
      for (int s = 0; s < p.n_src; ++s) {
        for (int kc = 0; kc < p.kchunks[s]; ++kc) {
          if (p.halo) mbar_wait(SPLIT ? a_ready(a_st) : a_full(a_st), a_par);
          int gj = 0;
          for (int j = 0; j < p.n_steps; ++j) {
            if (!p.halo) mbar_wait(SPLIT ? a_ready(a_st) : a_full(a_st), a_par);
            if (gj == 0) mbar_wait(b_full(b_st), b_par);
            uint32_t a_addr = a_base + a_st * p.a_stage_bytes;
            uint32_t sbo = 1024;
            if (p.halo) {
              // the 128B swizzle follows the absolute smem address bits (TMA wrote the halo box with the same function), so a
              // tap is just a start address shifted by whole 128-byte rows
              a_addr += (uint32_t)p.step_aoff[j];
              sbo = (uint32_t)p.step_sbo[j];
            }
            if constexpr (!PP) a_addr += 8u * (uint32_t)c * sbo;   // this warpgroup's 8 pixel rows = 8 row groups of 8 pixels
            const uint64_t bdesc = make_smem_desc_sw128(b_base + b_st * p.b_stage_bytes + (uint32_t)gj * tile_bytes_n, 1024);
            const bool last_of_group = (gj == p.tgroup - 1);
            wgmma_fence();
#pragma unroll
            for (int g = 0; g < MT; ++g)
#pragma unroll
              for (int hh = 0; hh < HALVES; ++hh) {
                const uint64_t adesc = make_smem_desc_sw128(a_addr + 8u * (uint32_t)hh * sbo + (uint32_t)(g * TILE_W * 128), sbo);
                mma_step<NW, OP>(acc[g * HALVES + hh], adesc, bdesc, first);
              }
            wgmma_commit();
            wgmma_wait<1>();   // this warp's share of the group before this one has completed: its stages may be refilled
            if (leader) {
              if (rel_a >= 0) mbar_arrive(a_empty(rel_a));
              if (rel_b >= 0) mbar_arrive(b_empty(rel_b));
            }
            rel_a = (!p.halo || j == p.n_steps - 1) ? a_st : -1;
            rel_b = last_of_group ? b_st : -1;
            first = 0;
            if (last_of_group) { gj = 0; if (++b_st == p.b_stages) { b_st = 0; b_par ^= 1; } } else { ++gj; }
            if (!p.halo || j == p.n_steps - 1) { if (++a_st == p.a_stages) { a_st = 0; a_par ^= 1; } }
          }
        }
      }
      if constexpr (PP) {
        if (leader) mbar_arrive(turn(c ^ 1));   // every stage of this item has been waited on: the other warpgroup's item may start
      }
      wgmma_wait<0>();
#pragma unroll
      for (int g = 0; g < MT * HALVES; ++g) wgmma_pin<NW / 2>(acc[g]);
      if (leader) {
        if (rel_a >= 0) mbar_arrive(a_empty(rel_a));
        if (rel_b >= 0) mbar_arrive(b_empty(rel_b));
      }

      // ---- epilogue. Accumulator register i of a thread holds row 16 tw_ + lane/4 + 8 ((i/2)%2) (a pixel of the tile) and
      // column 8 (i/4) + 2 qd + (i%2): every thread owns two pixels (same x, rows ty and ty + 1) and 2-channel pairs of them.
      // Half hh (ping-pong) or warpgroup c (cooperative) selects pixel rows [8 hh, 8 hh + 8) of the tile.
      const int ph0 = n0 / p.Cout, nb0 = n0 - ph0 * p.Cout;
      const int nchunks = p.block_n / 32;
#pragma unroll
      for (int gh = 0; gh < MT * HALVES; ++gh) {
        const int g = gh / HALVES, half = PP ? gh % HALVES : c;
        const int r0 = 64 * half + 16 * tw_ + (lane >> 2);
        const int ty = r0 / TILE_W, tx = r0 % TILE_W;   // second pixel: ty + 1
        int oy[2], ox[2];
        bool in_img[2];
        int64_t off0[2], pix0[2];
        float rgb[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          oy[h] = oy0 + ty + h; ox[h] = ox0 + g * TILE_W + tx;
          in_img[h] = oy[h] < p.Ho && ox[h] < p.Wo;
          off0[h] = (int64_t)b * p.out_sb + (int64_t)oy[h] * p.out_sy + (int64_t)ox[h] * p.out_sx;
          pix0[h] = (int64_t)b * p.pix_sb + (int64_t)oy[h] * p.pix_sy + (int64_t)ox[h] * p.pix_sx;   // dense-pixel index
        }
        // in-image pixels of this warp's 16 (lanes 4r hold pixel row r of both halves h), and 1 / 0 masks of this lane's two
        const int st_cnt = p.stats_ws ? __popc(__ballot_sync(0xffffffffu, in_img[0]) & 0x11111111u) +
                                            __popc(__ballot_sync(0xffffffffu, in_img[1]) & 0x11111111u) : 0;
        const float st_m0 = in_img[0] ? 1.f : 0.f, st_m1 = in_img[1] ? 1.f : 0.f;
        int ph = ph0, nb = nb0 - 32;
#pragma unroll
        for (int j = 0; j < NW / 32; ++j) {
          if (j >= nchunks) break;
          // column -> (phase, channel): the N dimension is phase-major [n_phase][Cout]; a 32-column chunk never straddles
          nb += 32;
          if (nb >= p.Cout) { nb -= p.Cout; ++ph; }
          float nz[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) nz[h] = (p.noise && in_img[h]) ? nw * __ldg(p.noise + p.phase_pix[ph] + pix0[h]) : 0.f;
          // v[h][k][e]: pixel h, channel nb + 8k + 2qd + e
          float v[2][4][2];
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int i = 16 * j + 4 * k + 2 * h + e;
                float x = acc[gh][i];
                if constexpr (OP == OP_BF16_NSTACK) x += acc[gh][(i + 16) % (NW / 2)];   // second column half: the w_lo products
                v[h][k][e] = x * p.acc_scale;
              }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int ch = nb + 8 * k + 2 * qd;
            float2 bq = make_float2(0.f, 0.f), sq = make_float2(p.slope, p.slope);
            if (p.bias) bq = __ldg(reinterpret_cast<const float2*>(p.bias + ch));
            if (p.slope_vec) sq = __ldg(reinterpret_cast<const float2*>(p.slope_vec + ch));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float v0 = v[h][k][0] + bq.x + nz[h], v1 = v[h][k][1] + bq.y + nz[h];
              if (p.act == VT_ACT_LRELU) {
                v0 = vt_lrelu(v0, sq.x) * p.gain; v1 = vt_lrelu(v1, sq.y) * p.gain;
              } else if (!REALLOC && p.act == VT_ACT_RELU_TANH) {
                v0 = tanhf(fmaxf(v0, 0.f)); v1 = tanhf(fmaxf(v1, 0.f));
              }
              const int64_t off = p.phase_off[ph] + off0[h] + ch;
              if (p.res) {
                if (in_img[h]) {
                  const float2 rv = __ldg(reinterpret_cast<const float2*>(p.res + off));
                  v0 = v0 * p.alpha + p.beta * rv.x; v1 = v1 * p.alpha + p.beta * rv.y;
                }
              } else if (p.alpha != 1.f) {
                v0 *= p.alpha; v1 *= p.alpha;
              }
              if (p.round_tf32) { v0 = vt_round_tf32(v0); v1 = vt_round_tf32(v1); }
              if (!REALLOC && p.rgb_w) {
                // 1x1 modulated conv to 3 channels on the values just produced (model/stylegan/model.py:384-385)
                const float* w0 = p.rgb_w + ((int64_t)(p.wB > 1 ? b : 0) * 3) * p.Cout + ch;
#pragma unroll
                for (int cc = 0; cc < 3; ++cc) {
                  const float2 wv = __ldg(reinterpret_cast<const float2*>(w0 + cc * p.Cout));
                  rgb[h][cc] = fmaf(v1, wv.y, fmaf(v0, wv.x, rgb[h][cc]));
                }
              }
              if (in_img[h] && p.out) *reinterpret_cast<float2*>(p.out + off) = make_float2(v0, v1);
              v[h][k][0] = in_img[h] ? v0 : 0.f; v[h][k][1] = in_img[h] ? v1 : 0.f;
            }
          }
          if (p.stats_ws) {
            // AdaptiveInstanceNorm statistics of the tensor this launch writes (model/dualstylegan.py:10-21): per channel over the
            // warp's in-image pixels, the sum and the sum of squares of x - pivot, both in a fixed butterfly order (no atomics).
            // The pivot is the chunk's first pixel (lane qd, h = 0: in the image whenever any pixel of the chunk is), so the
            // finalize's cancellation stays within a factor of the chunk's 16 pixels; about zero, or as an fp32 chunk sum, an
            // offset plane would lose its variance.  Pixels outside the image hold 0, so x - pivot * mask drops them.
            const int kchunk = ((rem * MT + g) * STATS_WARPS) + half * 4 + tw_;
            // every lane ends with the chunk's values: lanes 4c + qd store component c (pivot, deviation sum, square sum) of
            // both channels of their pair
            const int comp = lane >> 2;
            float2* wsp = reinterpret_cast<float2*>(p.stats_ws + comp * p.stats_e + ((int64_t)kchunk * p.B + b) * p.Cout + nb + 2 * qd);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              float out[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float piv = __shfl_sync(0xffffffffu, v[0][k][e], qd);
                const float d0 = fmaf(-piv, st_m0, v[0][k][e]), d1 = fmaf(-piv, st_m1, v[1][k][e]);
                float dsum = d0 + d1, dsq = fmaf(d0, d0, d1 * d1);
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                  dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
                  dsq += __shfl_xor_sync(0xffffffffu, dsq, o);
                }
                out[e] = comp == 0 ? piv : (comp == 1 ? dsum : dsq);
              }
              if (comp < 3) wsp[4 * k] = make_float2(out[0], out[1]);
            }
            if (b == 0 && n0 == 0 && j == 0 && lane == 0) p.stats_cnt[kchunk] = st_cnt;
          }
        }
        if (!REALLOC && p.rgb_w) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) {
              rgb[h][cc] += __shfl_xor_sync(0xffffffffu, rgb[h][cc], 1);
              rgb[h][cc] += __shfl_xor_sync(0xffffffffu, rgb[h][cc], 2);
            }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (qd != 0 || !in_img[h]) continue;
            torgb_store(p.rgb_bias, p.rgb_skip, p.rgb_skip_kernel, p.rgb_out, rgb[h], b, oy[h], ox[h], p.Ho, p.Wo);
          }
        }
      }
    }
  }
}

template <int NW, int MT, int OP>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ TcArgs p) { conv_tc_body<NW, MT, OP, false>(p); }

// The ping-pong form has its own name: it is the other instantiation besides the wide item whose warpgroups reallocate
// registers, and profiles tell the two schedules apart.
template <int NW, int MT, int OP>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_pingpong_kernel(const __grid_constant__ TcArgs p) { conv_tc_body<NW, MT, OP, true>(p); }

// The instantiations conv_tc_run can select: every (MMA N, M tiles) with MT * NW <= MAX_ACC_COLS in each operand mode, the
// N-stacked form only at N = 64 (Cout == 32), the wide item (N = 256, one M tile) in the bf16 split mode, and the ping-pong
// form of the 128 x 128 bf16-split item.
struct TcKernel {
  int nw, mt, op;
  bool pp;
  void (*fn)(TcArgs);
};
#define VT_TC_OPS(NW, MT) {NW, MT, OP_TF32, false, conv_tc_kernel<NW, MT, OP_TF32>}, {NW, MT, OP_BF16, false, conv_tc_kernel<NW, MT, OP_BF16>}, \
                          {NW, MT, OP_F16, false, conv_tc_kernel<NW, MT, OP_F16>}
const TcKernel kTcKernels[] = {
    VT_TC_OPS(128, 1), VT_TC_OPS(64, 1), VT_TC_OPS(64, 2), VT_TC_OPS(32, 1), VT_TC_OPS(32, 2), VT_TC_OPS(32, 4),
    {64, 1, OP_BF16_NSTACK, false, conv_tc_kernel<64, 1, OP_BF16_NSTACK>}, {64, 2, OP_BF16_NSTACK, false, conv_tc_kernel<64, 2, OP_BF16_NSTACK>},
    {WIDE_N, 1, OP_BF16, false, conv_tc_kernel<WIDE_N, 1, OP_BF16>},
    {MAX_BLOCK_N, 1, OP_BF16, true, conv_tc_pingpong_kernel<MAX_BLOCK_N, 1, OP_BF16>},
};
#undef VT_TC_OPS

}  // namespace

// ------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)f;
  });
  return fn;
}

// 4-D fp32 tensor map, SWIZZLE_128B, zero OOB fill. dims/strides innermost first; strides in BYTES for dims 1..3.
int vt_tc_make_map4(CUtensorMap* m, const void* base, const uint64_t dims[4], const uint64_t strides_b[3], const uint32_t box[4],
                    const char* what, bool bf16) {
  PFN_encodeTiled enc = get_encode();
  VT_CHECK(enc != nullptr, "conv_tc: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t gd[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gs[3] = {strides_b[0], strides_b[1], strides_b[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t es[4] = {1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) VT_CHECK(gd[i] >= 1 && bx[i] >= 1 && bx[i] <= 256, "conv_tc: bad %s map dim %d (dim=%llu box=%u)", what, i, (unsigned long long)gd[i], bx[i]);
  for (int i = 0; i < 3; ++i) VT_CHECK(gs[i] % 16 == 0 && gs[i] > 0, "conv_tc: %s map stride %d (%llu B) not a positive multiple of 16", what, i, (unsigned long long)gs[i]);
  VT_CHECK(((uintptr_t)base & 15) == 0, "conv_tc: %s base pointer not 16-byte aligned", what);
  CUresult r = enc(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(base), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VT_CHECK(r == CUDA_SUCCESS, "conv_tc: cuTensorMapEncodeTiled(%s) failed with CUresult %d", what, (int)r);
  return 0;
}


namespace {
inline int make_map4(CUtensorMap* m, const void* base, const uint64_t dims[4], const uint64_t strides_b[3], const uint32_t box[4],
                     const char* what, bool bf16 = false) { return vt_tc_make_map4(m, base, dims, strides_b, box, what, bf16); }

int g_tc_mode = 1;  // 0: one TMA box per tap; 1: one halo box per K chunk + row-shifted descriptors
int g_tc_mt = 0;    // 0: automatic M-tiles per work item; 1/2/4: forced
int g_tc_transpose = 1;   // 1: hand the problem over transposed when that wastes fewer tiles; 0: never; 2: always (tests)
int g_tc_tgroup = 0;  // 0: automatic taps per weight box (<= 36 KB); 1: one tap per box; n>1: KB budget
int g_tc_s2_halo = 0;  // 1: stride-2 layers may use halo staging (4 parity-view boxes per K chunk, 78 KB for a 3x3)
int g_tc_stage_policy = 1;  // big halo boxes (dilated 3x3): 0 = shrink the weight ring first (3 + 3 stages at dilation 4), 1 = keep >= 5 weight stages and drop to 2 halo stages
int g_tc_halo_pct = 60;    // halo staging must stage at most this percentage of the per-tap bytes (stride 1)
int g_tc_m_major = 1;      // work items ordered pixel-tile-major (the N tiles of a pixel tile run side by side: the activations' second read hits L2)
int g_tc_wide = 1;         // 128 x 256 work items: 0 = never, 1 = automatic (stride 1, with the wave-remainder split), 2 = whenever eligible, one launch
int g_tc_pingpong = 1;     // 128 x 128 bf16-split items owned by one consumer warpgroup each: 0 = never, 1 = automatic (>= 3 items per CTA), 2 = whenever eligible

int check_supported(const vt_conv_desc* d, bool set_err) {
#define VT_SUP(cond, ...) do { if (!(cond)) { if (set_err) vt_set_error(__VA_ARGS__); return 0; } } while (0)
  VT_SUP(d->Cout % 32 == 0, "conv_tc: Cout must be a multiple of 32 (got %d)", d->Cout);
  VT_SUP(d->out != nullptr || d->rgb_w != nullptr, "conv_tc: out may be NULL only with the fused ToRGB tail (image-only launch)");
  for (int s = 0; s < d->n_src; ++s) {
    VT_SUP(d->src_c[s] % KCH == 0, "conv_tc: src_c[%d]=%d must be a multiple of 32", s, d->src_c[s]);
    VT_SUP(d->src_cstride[s] % 4 == 0, "conv_tc: channel stride must be a multiple of 4");
  }
  VT_SUP(d->stride == 1 || d->stride == 2, "conv_tc: stride must be 1 or 2");
  VT_SUP(d->n_phase == 1 || (d->n_phase == 4 && d->stride == 1 && g_tc_mode != 0 && !d->res), "conv_tc: phases need stride 1, halo mode, no residual");
  for (int ph = 0; ph < d->n_phase; ++ph) VT_SUP(d->phase_off[ph] % 4 == 0, "conv_tc: phase offset must be a multiple of 4 floats");
  VT_SUP(d->out_sx % 4 == 0 && d->out_sy % 4 == 0 && d->out_sb % 4 == 0, "conv_tc: output strides must be multiples of 4 floats");
  VT_SUP(((uintptr_t)d->out & 15) == 0, "conv_tc: out not 16-byte aligned");
  VT_SUP(d->w_cstride % 4 == 0, "conv_tc: weight stride must be a multiple of 4");
  VT_SUP((!d->src_scale[0] && !d->src_scale[1] && !d->src_affine[0] && !d->src_affine[1]) || (d->weight_bf16x3 && d->stride == 1),
         "conv_tc: src_scale / src_affine need the bf16x3 mode and stride 1");
  for (int s = 0; s < 2; ++s) VT_SUP(!d->src_affine[s] || (((uintptr_t)d->src_affine[s] & 15) == 0), "conv_tc: src_affine not 16-byte aligned");
  VT_SUP(!d->bf16x3_nstack || (d->weight_bf16x3 && d->Cout == 32 && d->n_phase == 1 && d->split_fmt == 0), "conv_tc: the N-stacked bf16x3 form needs Cout == 32, one phase and the bf16 split");
  VT_SUP(d->split_fmt == 0 || d->split_fmt == 1, "conv_tc: split_fmt must be 0 (bf16) or 1 (fp16)");
  VT_SUP(!d->weight_bf16x3 || d->w_cstride % KCH == 0, "conv_tc: bf16x3 weights need a channel stride that is a multiple of 32");
  VT_SUP(!d->res || (((uintptr_t)d->res & 15) == 0), "conv_tc: res not 16-byte aligned");
  VT_SUP(!d->bias || (((uintptr_t)d->bias & 15) == 0), "conv_tc: bias not 16-byte aligned");
  VT_SUP(!d->slope_vec || (((uintptr_t)d->slope_vec & 15) == 0), "conv_tc: slope_vec not 16-byte aligned");
  // fused ToRGB: every channel of a pixel must be in one N tile (the 3-channel dot product is finished in the epilogue)
  VT_SUP(!d->rgb_w || (d->n_phase == 1 && d->Cout <= MAX_BLOCK_N && (d->Cout & (d->Cout - 1)) == 0 && (((uintptr_t)d->rgb_w & 15) == 0) &&
                       d->out_sx == d->Cout && d->out_sy == (int64_t)d->Wo * d->Cout && (!d->rgb_skip || (d->Ho % 2 == 0 && d->Wo % 2 == 0))),
         "conv_tc: fused ToRGB needs Cout a power of two <= 128, one phase, a dense output and even Ho/Wo for the skip");
  return 1;
#undef VT_SUP
}

}  // namespace

extern "C" int vt_set_option(const char* key, int value) {
  if (key && strcmp(key, "tc_mode") == 0) { int old = g_tc_mode; g_tc_mode = value; return old; }
  if (key && strcmp(key, "tc_mt") == 0) { int old = g_tc_mt; g_tc_mt = value; return old; }
  if (key && strcmp(key, "tc_tgroup") == 0) { int old = g_tc_tgroup; g_tc_tgroup = value; return old; }
  if (key && strcmp(key, "tc_s2_halo") == 0) { int old = g_tc_s2_halo; g_tc_s2_halo = value; return old; }
  if (key && strcmp(key, "tc_stage_policy") == 0) { int old = g_tc_stage_policy; g_tc_stage_policy = value; return old; }
  if (key && strcmp(key, "tc_halo_pct") == 0) { int old = g_tc_halo_pct; g_tc_halo_pct = value; return old; }
  if (key && strcmp(key, "tc_m_major") == 0) { int old = g_tc_m_major; g_tc_m_major = value; return old; }
  if (key && strcmp(key, "tc_transpose") == 0) { int old = g_tc_transpose; g_tc_transpose = value; return old; }
  if (key && strcmp(key, "tc_wide") == 0) { int old = g_tc_wide; g_tc_wide = value; return old; }
  if (key && strcmp(key, "tc_pingpong") == 0) { int old = g_tc_pingpong; g_tc_pingpong = value; return old; }
  if (key && strcmp(key, "rs_kernel") == 0) { int old = g_rs_kernel; g_rs_kernel = value; return old; }
  if (key && strcmp(key, "instnorm_chunks") == 0) { int old = g_instnorm_chunks; g_instnorm_chunks = value; return old; }
  if (key && strcmp(key, "fir4") == 0) { int old = g_fir4; g_fir4 = value; return old; }
  if (key && strcmp(key, "smalln_is") == 0) { int old = g_smalln_is; g_smalln_is = value; return old; }
  if (key && strcmp(key, "upfirdn_tiled") == 0) { int old = g_upfirdn_tiled; g_upfirdn_tiled = value; return old; }
  return -1;
}

extern "C" int vt_conv2d_tc_supported(const vt_conv_desc* d) {
  if (!d || d->struct_size != (int)sizeof(vt_conv_desc)) return 0;
  return check_supported(d, false);
}

// chunks_out != NULL: plan only — how many instance-norm partial-sum chunks this descriptor's launch writes per (sample, channel).
// m_first > 0: run only the pixel tiles from m_first on (the remainder launch of a wide layer); allow_wide = false: 128-wide N tiles.
static int conv_tc_run(const vt_conv_desc* d, void* stream, int* chunks_out, int m_first = 0, bool allow_wide = true) {
  if (vt_validate_conv_desc(d, "conv2d_tc")) return 1;
  if (!check_supported(d, true)) return 1;

  static thread_local TcArgs a;  // large (tensor maps); reused to avoid stack churn
  memset(&a, 0, sizeof(a));

  // ---- geometry view. The kernel's M tile is 8 pixels along "x" by 16 along "y". When that wastes fewer tiles the
  // problem is handed over transposed (x <-> y): only strides, extents and tap offsets swap roles, the data stays put.
  // (72x128 maps: 16x5 = 80 tiles as is, 9x8 = 72 transposed.)
  bool T = false;
  if (g_tc_transpose && d->stride == 1 && !d->rgb_w) {
    const int64_t t0 = vt_cdiv(d->Wo, TILE_W) * vt_cdiv(d->Ho, TILE_H), t1 = vt_cdiv(d->Ho, TILE_W) * vt_cdiv(d->Wo, TILE_H);
    T = (g_tc_transpose == 2) || (t1 < t0);
  }
  const int gH = T ? d->W : d->H, gW = T ? d->H : d->W, gHo = T ? d->Wo : d->Ho, gWo = T ? d->Ho : d->Wo;
  const int64_t g_out_sy = T ? d->out_sx : d->out_sy, g_out_sx = T ? d->out_sy : d->out_sx;

  a.n_phase = d->n_phase;
  a.Ho = gHo; a.Wo = gWo; a.Cout = d->Cout; a.wB = d->wB; a.out_cpitch = d->out_cpitch;
  a.bias = d->bias; a.noise = d->noise; a.noise_w = d->noise_w; a.res = d->res;
  a.out_sb = d->out_sb; a.out_sy = g_out_sy; a.out_sx = g_out_sx;
  for (int ph = 0; ph < 4; ++ph) a.phase_off[ph] = d->phase_off[ph < d->n_phase ? ph : 0];
  if (d->noise) {
    VT_CHECK(d->out_sb % d->out_cpitch == 0 && d->out_sy % d->out_cpitch == 0 && d->out_sx % d->out_cpitch == 0,
             "conv_tc: output strides must be multiples of out_cpitch when noise is used");
    a.pix_sb = d->out_sb / d->out_cpitch; a.pix_sy = g_out_sy / d->out_cpitch; a.pix_sx = g_out_sx / d->out_cpitch;
    // a view's noise pixel is its element offset over out_cpitch (as in the FFMA kernel): the remainder is the channel offset
    // of a channel slice, which has to keep the slice inside one pixel
    for (int ph = 0; ph < 4; ++ph) {
      VT_CHECK(a.phase_off[ph] >= 0 && a.phase_off[ph] % d->out_cpitch + d->Cout <= d->out_cpitch,
               "conv_tc: with noise, the output view's channels must lie inside one pixel of out_cpitch channels");
      a.phase_pix[ph] = a.phase_off[ph] / d->out_cpitch;
    }
  }
  a.out = d->out;
  a.slope_vec = d->slope_vec;
  a.rgb_w = d->rgb_w; a.rgb_bias = d->rgb_bias; a.rgb_skip = d->rgb_skip; a.rgb_skip_kernel = d->rgb_skip_kernel; a.rgb_out = d->rgb_out;
  a.act = d->act; a.round_tf32 = d->round_tf32; a.slope = d->slope; a.gain = d->gain; a.alpha = d->alpha; a.beta = d->beta;
  a.B = d->B;
  const bool split = d->weight_bf16x3 != nullptr;
  const bool nstack = split && d->bf16x3_nstack;
  const int op = !split ? OP_TF32 : nstack ? OP_BF16_NSTACK : d->split_fmt == 1 ? OP_F16 : OP_BF16;
  a.acc_scale = (split && d->acc_scale > 0.f) ? d->acc_scale : 1.f;
  a.src_scale[0] = d->src_scale[0]; a.src_scale[1] = d->src_scale[1];
  a.src_affine[0] = d->src_affine[0]; a.src_affine[1] = d->src_affine[1];
  a.src_cn[0] = d->src_c[0]; a.src_cn[1] = d->n_src > 1 ? d->src_c[1] : 0;
  a.in_w = gW; a.in_h = gH;
  a.sc_sb = (int64_t)d->H * d->W; a.sc_sy = T ? 1 : d->W; a.sc_sx = T ? d->W : 1;

  // ---- K iteration space
  a.n_src = d->n_src;
  int coff = 0;
  for (int s = 0; s < d->n_src; ++s) { a.kchunks[s] = d->src_c[s] / KCH; a.coff[s] = coff; coff += d->src_c[s]; }
  a.n_steps = d->taps;
  int dxmin = 1 << 30, dxmax = -(1 << 30), dymin = 1 << 30, dymax = -(1 << 30);
  for (int t = 0; t < d->taps; ++t) {
    const int tdx = T ? d->tap_dy[t] : d->tap_dx[t], tdy = T ? d->tap_dx[t] : d->tap_dy[t];
    int view = 0, vx = tdx, vy = tdy;
    if (d->stride == 2) {
      const int px = tdx & 1, py = tdy & 1;
      view = py * 2 + px;
      vx = (tdx - px) / 2;
      vy = (tdy - py) / 2;
    }
    VT_CHECK(vx >= -100 && vx <= 100 && vy >= -100 && vy <= 100, "conv_tc: tap offset out of range");
    a.step_view[t] = (int8_t)view; a.step_vx[t] = (int8_t)vx; a.step_vy[t] = (int8_t)vy;
    a.step_w[t] = (int16_t)d->tap_w[t];
    dxmin = vx < dxmin ? vx : dxmin; dxmax = vx > dxmax ? vx : dxmax;
    dymin = vy < dymin ? vy : dymin; dymax = vy > dymax ? vy : dymax;
  }

  // ---- N tile and accumulator plan (registers: mt * N <= 128 accumulator columns per consumer thread, or the wide item)
  // GEMM N = n_phase * Cout (phase-major rows of the weight tensor); N tile = largest power of two <= 128 dividing it, or 256
  // (the wide item) in the bf16 split mode when it divides N and its pipeline fits (below)
  const int n_eff = d->n_phase * d->Cout;
  int bn_narrow = MAX_BLOCK_N;
  while (bn_narrow > 32 && (n_eff % bn_narrow) != 0) bn_narrow /= 2;
  VT_CHECK(n_eff % bn_narrow == 0, "conv_tc: no N tile for N=%d", n_eff);
  // (automatic: stride 1 only; the stride-2 layers, which stage one box per tap, measured slower with wide items)
  const bool wide = allow_wide && (g_tc_wide == 2 || (g_tc_wide == 1 && d->stride == 1)) && op == OP_BF16 && n_eff % WIDE_N == 0 &&
                    !d->rgb_w && d->act != VT_ACT_RELU_TANH;
  const int bn = wide ? WIDE_N : bn_narrow;
  const int bnm = nstack ? 2 * bn : bn;  // MMA N = accumulator columns = weight rows per tile
  // halo staging: multi-tap layers (one box serves all taps) and small-N 1x1 layers (several M tiles per box and weight tile).
  // tc_mode 3: halo for stride 1 only (A/B tests)
  const bool can_halo = (g_tc_mode != 0) && (d->taps > 1 || (bn <= 64 && d->stride == 1)) && (d->stride == 1 || g_tc_mode != 3);
  // M tiles per work item: share each weight tile across `mt` pixel tiles when N is small (weights dominate L2->smem
  // traffic there); bounded by the accumulator registers and by the halo box fitting a pipeline stage.
  int mt = 1;
  if (can_halo && g_tc_mt != 1) {
    int want = (g_tc_mt > 0) ? g_tc_mt : (bn >= 128 ? 1 : (bn >= 64 ? 2 : 4));
    while (want > 1 && (want * bnm > MAX_ACC_COLS || gWo <= TILE_W * (want / 2))) want /= 2;
    mt = want;
  }
  const int fixed = 1024 /*barriers*/ + 1024 /*alignment slack*/;
  int smem_bytes = 0;
  // taps per weight box: as many consecutive slabs as fit ~36 KB, dividing the step count, never crossing a phase
  int tgroup = 1;
  if (g_tc_tgroup != 1) {
    for (int tg = d->taps; tg >= 2; --tg) {
      if (d->taps % tg != 0 || tg * bnm * 128 > (g_tc_tgroup > 1 ? g_tc_tgroup : 36) * 1024) continue;
      bool ok = true;
      for (int t = 0; t < d->taps && ok; ++t)
        if (t % tg != 0 && d->tap_w[t] != d->tap_w[t - 1] + 1) ok = false;
      if (ok) { tgroup = tg; break; }
    }
  }
  a.tgroup = tgroup;
  // per parity view (stride 1: view 0 only): offset ranges of the taps that read it
  int vx0[4], vx1[4], vy0[4], vy1[4];
  bool vused[4] = {false, false, false, false};
  for (int t = 0; t < d->taps; ++t) {
    const int v = a.step_view[t], vx = a.step_vx[t], vy = a.step_vy[t];
    if (!vused[v]) { vused[v] = true; vx0[v] = vx1[v] = vx; vy0[v] = vy1[v] = vy; }
    vx0[v] = vx < vx0[v] ? vx : vx0[v]; vx1[v] = vx > vx1[v] ? vx : vx1[v];
    vy0[v] = vy < vy0[v] ? vy : vy0[v]; vy1[v] = vy > vy1[v] ? vy : vy1[v];
  }
  int hv_w[4] = {0, 0, 0, 0}, hv_h[4] = {0, 0, 0, 0};
  for (;; mt /= 2) {
    // one halo box per view in use, each 1024-byte aligned inside the stage (the 128B swizzle phase follows address bits 7-9)
    int halo_bytes = 0, tx_bytes = 0;
    bool fits = true;
    a.n_hv = 0;
    for (int v = 0; v < 4; ++v) {
      if (!vused[v]) continue;
      const int w = TILE_W * mt + (vx1[v] - vx0[v]), h = TILE_H + (vy1[v] - vy0[v]);
      fits = fits && w <= 256 && h <= 256;
      const int i = a.n_hv++;
      a.hv_view[i] = v; a.hv_x0[i] = vx0[v]; a.hv_y0[i] = vy0[v]; a.hv_off[i] = halo_bytes; a.hv_bytes[i] = w * h * 128;
      hv_w[v] = w; hv_h[v] = h;
      tx_bytes += w * h * 128;
      halo_bytes = (int)(vt_cdiv(halo_bytes + w * h * 128, 1024) * 1024);
    }
    // staged bytes must pay off against one box per tap: at most half of it (stride 2 with tc_s2_halo: 0.6 - a 3x3 / stride-2 layer
    // stages 4 views x 9 x 17 pixels = 0.53 of the per-tap bytes, and the operand-transform warps touch every staged byte once)
    const int64_t tap_bytes = (int64_t)d->taps * TILE_M * 128;
    const bool pays = (d->stride == 2 && g_tc_s2_halo) ? (tx_bytes * 10 <= tap_bytes * 6) : ((int64_t)tx_bytes * 100 <= tap_bytes * g_tc_halo_pct);
    a.halo = can_halo && fits && halo_bytes <= 96 * 1024 && (mt > 1 || pays) &&
             2 * halo_bytes + 2 * bnm * 128 * tgroup + fixed <= MAX_SMEM;   // at least a 2+2 stage pipeline must fit
    if (!a.halo && mt > 1) continue;
    a.halo_x0 = a.hv_x0[0]; a.halo_y0 = a.hv_y0[0]; a.halo_w = hv_w[a.hv_view[0]];
    a.a_tx_bytes = a.halo ? tx_bytes : TILE_M * 128;
    a.a_rows = a.halo ? (a.hv_off[a.n_hv - 1] + a.hv_bytes[a.n_hv - 1]) / 128 : TILE_M;
    // shared memory plan: A ring (halo boxes or per-tap tiles) + B ring (weight tiles)
    a.a_stage_bytes = a.halo ? halo_bytes : TILE_M * 128;
    a.b_stage_bytes = bnm * 128 * tgroup;
    a.a_stages = a.halo ? 3 : 4;
    a.b_stages = tgroup > 1 ? 4 : 6;
    // a K chunk's MMAs (taps x 6 instructions) cover one halo stage; a weight stage covers one tap only: with big halo boxes a
    // deeper weight ring hides more TMA latency than a third halo stage (policy 1)
    const int b_floor = (g_tc_stage_policy == 1 && a.halo && a.a_stage_bytes >= 40 * 1024 && tgroup == 1) ? 5 : 3;
    while (a.a_stages * a.a_stage_bytes + a.b_stages * a.b_stage_bytes + fixed > MAX_SMEM) {
      if (a.b_stages > b_floor) --a.b_stages;
      else if (a.a_stages > 2) --a.a_stages;
      else if (a.b_stages > 2) --a.b_stages;
      else break;
    }
    if (b_floor > 3)
      while (a.b_stages < 8 && a.a_stages * a.a_stage_bytes + (a.b_stages + 1) * a.b_stage_bytes + fixed <= MAX_SMEM) ++a.b_stages;
    smem_bytes = a.a_stages * a.a_stage_bytes + a.b_stages * a.b_stage_bytes + fixed;
    if (smem_bytes <= MAX_SMEM || mt == 1) break;
  }
  // the wide item needs at least 2 A stages and 3 weight stages (32 KB each); otherwise the layer takes the 128-wide plan
  if (wide && !(smem_bytes <= MAX_SMEM && a.a_stages >= 2 && a.b_stages >= 3)) return conv_tc_run(d, stream, chunks_out, m_first, false);
  a.b_tx_bytes = bnm * 128 * tgroup;
  VT_CHECK(smem_bytes <= MAX_SMEM && a.a_stages >= 2 && a.b_stages >= 2 && a.a_stages <= 8 && a.b_stages <= 8,
           "conv_tc: shared memory plan does not fit (%d B, mt=%d, bn=%d)", smem_bytes, mt, bn);
  for (int t = 0; t < d->taps; ++t) {
    const int v = a.step_view[t];
    int i = 0;
    while (i < a.n_hv - 1 && a.hv_view[i] != v) ++i;
    a.step_aoff[t] = a.hv_off[i] + ((a.step_vy[t] - vy0[v]) * hv_w[v] + (a.step_vx[t] - vx0[v])) * 128;
    a.step_sbo[t] = (uint16_t)(hv_w[v] * 128);
  }
  a.block_n = bn;
  a.mma_n = bnm;
  a.n_tiles = n_eff / bn;
  VT_CHECK(!d->rgb_w || a.n_tiles == 1, "conv_tc: fused ToRGB needs one N tile (Cout = %d)", d->Cout);
  a.tiles_x = (int)vt_cdiv(gWo, TILE_W * mt);
  a.tiles_y = (int)vt_cdiv(gHo, TILE_H);
  const int64_t m_total = (int64_t)a.B * a.tiles_x * a.tiles_y;
  VT_CHECK(m_first < m_total, "conv_tc: first pixel tile %d out of range", m_first);
  const int64_t total = (int64_t)a.n_tiles * (m_total - m_first);
  VT_CHECK(total < (1LL << 31), "conv_tc: too many tiles");
  a.total_tiles = (int)total;
  a.m_first = m_first;
  a.m_major = g_tc_m_major ? 1 : 0;
  {
    // fused instance-norm statistics of the output: one chunk per (pixel tile of an image, consumer warp)
    const int64_t chunks = (int64_t)a.tiles_x * a.tiles_y * mt * STATS_WARPS;
    if (chunks_out) {
      VT_CHECK(d->n_phase == 1 && !d->rgb_w && chunks < (1 << 24), "conv_tc: output statistics need one phase and no fused ToRGB");
      *chunks_out = (int)chunks;
      return 0;
    }
    if (d->stats_ws) {
      VT_CHECK(d->n_phase == 1 && !d->rgb_w, "conv_tc: output statistics need one phase and no fused ToRGB");
      const int64_t need = vt_instnorm_partials_floats(chunks, d->B, d->Cout);
      VT_CHECK(d->stats_ws_floats >= need, "conv_tc: stats_ws too small (%lld floats, need %lld)", (long long)d->stats_ws_floats,
               (long long)need);
      VT_CHECK(((uintptr_t)d->stats_ws & 7) == 0, "conv_tc: stats_ws not 8-byte aligned");
      a.stats_ws = d->stats_ws;
      a.stats_e = chunks * d->B * d->Cout;
      a.stats_cnt = reinterpret_cast<int*>(d->stats_ws + 3 * a.stats_e);
    }
  }

  // ---- tensor maps (dims innermost first: channels, kernel-x, kernel-y, batch)
  for (int s = 0; s < d->n_src; ++s) {
    const uint64_t cs = (uint64_t)d->src_cstride[s];
    if (d->stride == 1) {
      const uint64_t real_sx = cs * 4, real_sy = (uint64_t)d->W * cs * 4;
      const uint64_t dims[4] = {cs, (uint64_t)gW, (uint64_t)gH, (uint64_t)d->B};
      const uint64_t str[3] = {T ? real_sy : real_sx, T ? real_sx : real_sy, (uint64_t)d->H * d->W * cs * 4};
      const uint32_t box[4] = {KCH, (uint32_t)(a.halo ? hv_w[0] : TILE_W), (uint32_t)(a.halo ? hv_h[0] : TILE_H), 1};
      if (make_map4(&a.in_map[s][0], d->src[s], dims, str, box, "input")) return 1;
      for (int v = 1; v < 4; ++v) a.in_map[s][v] = a.in_map[s][0];
    } else {
      // parity views: view (py,px)[vy][vx] = in[2*vy+py][2*vx+px]
      bool have0 = false;
      for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
          const int vw = (d->W - px + 1) / 2, vh = (d->H - py + 1) / 2;
          CUtensorMap* mp = &a.in_map[s][py * 2 + px];
          if (vw < 1 || vh < 1) { if (have0) *mp = a.in_map[s][0]; continue; }
          const uint64_t dims[4] = {cs, (uint64_t)vw, (uint64_t)vh, (uint64_t)d->B};
          const uint64_t str[3] = {2 * cs * 4, 2 * (uint64_t)d->W * cs * 4, (uint64_t)d->H * d->W * cs * 4};
          const int v = py * 2 + px;
          const uint32_t box[4] = {KCH, (uint32_t)((a.halo && vused[v]) ? hv_w[v] : TILE_W), (uint32_t)((a.halo && vused[v]) ? hv_h[v] : TILE_H), 1};
          if (make_map4(mp, d->src[s] + ((int64_t)py * d->W + px) * cs, dims, str, box, "input(parity)")) return 1;
          have0 = true;
        }
    }
  }
  {
    const uint64_t wc = (uint64_t)d->w_cstride;
    const uint64_t dims[4] = {wc, (uint64_t)n_eff, (uint64_t)d->w_taps, (uint64_t)d->wB};
    const uint64_t str[3] = {wc * 4, (uint64_t)n_eff * wc * 4, (uint64_t)d->w_taps * n_eff * wc * 4};
    if (split) {   // same byte layout as the fp32 tensor: every 32-channel chunk is [w_hi(32) | w_lo(32)] bf16
      VT_CHECK(((uintptr_t)d->weight_bf16x3 & 15) == 0, "conv_tc: weight_bf16x3 not 16-byte aligned");
      const uint64_t rows = (uint64_t)n_eff * (nstack ? 2 : 1);  // N-stacked: 32 [w_hi|w_hi] rows then 32 [w_lo|w_lo] rows per tap
      const uint64_t dims2[4] = {2 * wc, rows, (uint64_t)d->w_taps, (uint64_t)d->wB};
      const uint64_t str2[3] = {wc * 4, rows * wc * 4, (uint64_t)d->w_taps * rows * wc * 4};
      const uint32_t box[4] = {2 * KCH, (uint32_t)bnm, (uint32_t)a.tgroup, 1};
      if (make_map4(&a.w_map, d->weight_bf16x3, dims2, str2, box, "weight(bf16x3)", true)) return 1;
    } else {
      const uint32_t box[4] = {KCH, (uint32_t)bn, (uint32_t)a.tgroup, 1};
      if (make_map4(&a.w_map, d->weight, dims, str, box, "weight")) return 1;
    }
  }
  static std::once_flag attr_once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once, [] {
    for (const TcKernel& k : kTcKernels)
      if (attr_err == cudaSuccess) attr_err = cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM);
  });
  VT_CHECK(attr_err == cudaSuccess, "conv_tc: cudaFuncSetAttribute failed: %s", cudaGetErrorString(attr_err));
  // ping-pong: never with the fused ToRGB or tanh, which it leaves out.  Automatic: when every CTA gets at least 3 items.  Ping-pong
  // hides the epilogues of all but the last item of a CTA, but one warpgroup alone runs an item's main loop slower than two: one
  // item per CTA measured 3-9 % slower, two gave no clear gain, three or more 2-21 % faster (DESIGN.md section 4).
  const bool pingpong = (g_tc_pingpong == 2 || (g_tc_pingpong == 1 && a.total_tiles >= 3 * vt_num_sms())) && op == OP_BF16 &&
                        bnm == MAX_BLOCK_N && mt == 1 && !d->rgb_w && d->act != VT_ACT_RELU_TANH;
  const TcKernel* kern = nullptr;
  for (const TcKernel& k : kTcKernels)
    if (k.nw == bnm && k.mt == mt && k.op == op && k.pp == pingpong) kern = &k;
  if (!kern) return vt_set_error("conv_tc: no kernel for MMA N = %d, %d M tiles, operand mode %d", bnm, mt, op);
  int grid = vt_num_sms();
  // Wave remainder of a wide layer: its whole rounds of wide items (one per SM) run in this launch, the pixel tiles left over
  // in a second launch of 128-wide items, which fills the last partial round with half-length items.  Both use the same
  // tiling and statistics chunks and write disjoint outputs.
  int m_split = 0;
  if (wide && g_tc_wide == 1 && a.total_tiles >= grid && a.total_tiles % grid != 0)
    m_split = (a.total_tiles / grid) * grid / a.n_tiles;
  if (m_split > 0) a.total_tiles = m_split * a.n_tiles;
  if (grid > a.total_tiles) grid = a.total_tiles;
  kern->fn<<<grid, TC_THREADS, smem_bytes, (cudaStream_t)stream>>>(a);
  VT_LAUNCH_CHECK();
  return m_split > 0 ? conv_tc_run(d, stream, nullptr, m_split, false) : 0;
}

extern "C" int vt_conv2d_tc_tf32(const vt_conv_desc* d, void* stream) { return conv_tc_run(d, stream, nullptr); }

// Row-strip entry points: the full-resolution 3x3 / stride 1 layers with Cin, Cout in {32, 64}.  They run conv_rs_kernel
// (conv_rs.cu: output channels on the MMA's M, pixels on N) when it takes the descriptor, else the kernel above.
static bool rs_shape(const vt_conv_desc* d) {
  if (d->n_src != 1 || d->stride != 1 || d->taps != 9 || d->n_phase != 1 || d->res || d->slope_vec || !d->weight_bf16x3) return false;
  if (d->src_scale[0] || d->src_affine[0] || d->alpha != 1.f) return false;
  if ((d->Cout != 32 && d->Cout != 64) || (d->src_c[0] != 32 && d->src_c[0] != 64)) return false;
  return d->act == VT_ACT_NONE || d->act == VT_ACT_LRELU;
}

extern "C" int vt_conv2d_rs_supported(const vt_conv_desc* d) {
  if (!d || d->struct_size != (int)sizeof(vt_conv_desc)) return 0;
  return rs_shape(d) && check_supported(d, false);
}

extern "C" int vt_conv2d_rs(const vt_conv_desc* d, float acc_scale, void* stream) {
  VT_CHECK(d && d->struct_size == (int)sizeof(vt_conv_desc) && rs_shape(d), "conv2d_rs: not a row-strip layer (3x3, stride 1, Cin/Cout in {32, 64})");
  vt_conv_desc c = *d;
  if (acc_scale > 0.f) c.acc_scale = acc_scale;
  if (g_rs_kernel && vt_conv_rs_takes(&c)) return vt_conv_rs_run(&c, stream);
  return conv_tc_run(&c, stream, nullptr);
}

extern "C" int vt_conv2d_tc_stats_chunks(const vt_conv_desc* d) {
  int chunks = 0;
  if (conv_tc_run(d, nullptr, &chunks)) return -1;
  return chunks;
}

