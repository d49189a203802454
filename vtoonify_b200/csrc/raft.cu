// RAFT optical flow (model/raft/core, full model, test-time settings of smooth_parsing_map.py): the gather and elementwise steps around
// the convolutions.  The convolutions themselves (encoders, correlation volume, motion encoder, GRU, heads) run on conv_tc / conv_direct.
//   raft_input_s2d   2 * (x / 255) - 1 of image1 (and image2 behind it) as the space-to-depth input of the 7x7 / 2 stems
//   raft_norm_relu   instance norm + ReLU of a conv output, optionally + a (normalised) shortcut and a second ReLU
//   raft_context     cnet's split: tanh(net) into the GRU state, relu(inp) into the GRU input buffer
//   raft_corr_pool   F.avg_pool2d(corr, 2, 2) over the (h2, w2) axes of every correlation row (floor sizes, torch's summation order)
//   raft_corr_lookup CorrBlock.__call__: 4 levels x 81 bilinear taps (grid_sample, align_corners=True, zeros outside)
//   raft_fmap_pool   F.avg_pool2d(fmap, 2, 2) of an NHWC feature map (floor sizes, torch's summation order): the on-demand pyramid
//   raft_corr_ondemand  the same 4 x 81 taps without the all-pairs volume (AlternateCorrBlock): per pixel and level the dot products of
//                    fmap1 with the pooled fmap2 at the 10 x 10 integer positions around floor(coords / 2^l) - 4, combined bilinearly
//   raft_convf1      the motion encoder's 7x7 convolution of the 2-channel flow (49 taps: a direct kernel) + bias + ReLU
//   raft_flow        coords1 (+)= delta, or the flow coords1 - coords0 written into a channel slice of an NHWC buffer
//   raft_gru_reset / raft_gru_update   sigmoid(r) * h, and h = (1 - sigmoid(z)) h + sigmoid(z) tanh(q)
//   raft_upsample    RAFT.upsample_flow: softmax over 9 mask logits, convex combination of 8 * flow, planar [B, 2, 8h, 8w] store
// Every kernel writes each output element from one thread with a fixed summation order: no atomics, reruns are bit-identical.
// Offsets are 64-bit (the level-0 correlation volume holds more than 2^31 floats at the smoothing size).
#include <math.h>
#include "common.cuh"

namespace {

constexpr int RADIUS = 4;
constexpr int WIN = 2 * RADIUS + 1;        // 9
constexpr int LEVELS = 4;
constexpr int LOOKUP_C = LEVELS * WIN * WIN;  // 324

unsigned grid1(int64_t n, int threads) {
  int64_t blocks = vt_cdiv(n, threads);
  const int64_t cap = (int64_t)vt_num_sms() * 64;
  return (unsigned)(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

// out [nB, H/2, W/2, cpad]: Z[y, x, (py*2+px)*3 + c] = 2 * (X[c, 2y+py, 2x+px] / 255) - 1, zero pad channels; rows B.. come from img2
__global__ void __launch_bounds__(256)
raft_input_s2d_kernel(const float* __restrict__ img1, const float* __restrict__ img2, float* __restrict__ out, int B, int H, int W,
                      int cpad, int64_t total) {
  const int Ho = H / 2, Wo = W / 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % Wo);
    const int64_t t = i / Wo;
    const int y = (int)(t % Ho), n = (int)(t / Ho);
    const float* ip = n < B ? img1 + (int64_t)n * 3 * H * W : img2 + (int64_t)(n - B) * 3 * H * W;
    float* op = out + i * cpad;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int Y = 2 * y + (q >> 1), X = 2 * x + (q & 1);
#pragma unroll
      for (int c = 0; c < 3; ++c) op[q * 3 + c] = vt_raft_unit(__ldg(ip + ((int64_t)c * H + Y) * W + X));
    }
    for (int c = 12; c < cpad; ++c) op[c] = 0.f;
  }
}

// out = relu(relu((x - m) * r) + s), s = res (stats_res NULL) or (res - m') * r' (res non-NULL), or out = relu((x - m) * r) (res NULL);
// stats: [B, C, 2] (mean, rstd) per plane
__global__ void __launch_bounds__(256)
raft_norm_relu_kernel(const float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ res,
                      const float* __restrict__ stats_res, float* __restrict__ out, int64_t HW, int C, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t b = i / C / HW;
    const float2 st = __ldg(reinterpret_cast<const float2*>(stats) + b * C + c);
    float v = fmaxf((__ldg(x + i) - st.x) * st.y, 0.f);
    if (res) {
      float s = __ldg(res + i);
      if (stats_res) {
        const float2 sr = __ldg(reinterpret_cast<const float2*>(stats_res) + b * C + c);
        s = (s - sr.x) * sr.y;
      }
      v = fmaxf(v + s, 0.f);
    }
    out[i] = v;
  }
}

// cnet [npix, 2C] -> net [npix, C] = tanh(cnet[:, :C]), inp[p * inp_cpitch + c] = relu(cnet[:, C:])
__global__ void __launch_bounds__(256)
raft_context_kernel(const float* __restrict__ cnet, float* __restrict__ net, float* __restrict__ inp, int C, int inp_cpitch,
                    int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / C;
    const int c = (int)(i % C);
    net[i] = tanhf(__ldg(cnet + p * 2 * C + c));
    inp[p * inp_cpitch + c] = fmaxf(__ldg(cnet + p * 2 * C + C + c), 0.f);
  }
}

// out row n [h/2, w/2] (dense) = 2x2 means of in row n [h, w] (row stride in_stride); ((a00 + a01) + a10) + a11, then / 4, as ATen
__global__ void __launch_bounds__(256)
raft_corr_pool_kernel(const float* __restrict__ in, float* __restrict__ out, int h, int w, int64_t in_stride, int64_t total) {
  const int ho = h / 2, wo = w / 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % wo);
    const int64_t t = i / wo;
    const int y = (int)(t % ho);
    const int64_t n = t / ho;
    const float* p = in + n * in_stride + (int64_t)(2 * y) * w + 2 * x;
    float s = 0.f;
    s += __ldg(p);
    s += __ldg(p + 1);
    s += __ldg(p + w);
    s += __ldg(p + w + 1);
    out[i] = s / 4.f;
  }
}

struct Pyramid {
  const float* lvl[LEVELS];
  int64_t stride[LEVELS];
  int h[LEVELS], w[LEVELS];
};

// out[p * out_cpitch + l*81 + 9i + j] = bilinear sample of level l of row p at (x, y) = coords[p] / 2^l + (i - 4, j - 4); corners
// outside the map contribute 0 (grid_sample, zeros padding, align_corners=True on pixel coordinates)
__global__ void __launch_bounds__(256)
raft_corr_lookup_kernel(Pyramid pyr, const float* __restrict__ coords, float* __restrict__ out, int out_cpitch, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / LOOKUP_C;
    const int k = (int)(i % LOOKUP_C);
    const int l = k / (WIN * WIN), ij = k % (WIN * WIN);
    const int di = ij / WIN - RADIUS, dj = ij % WIN - RADIUS;
    const float2 cxy = __ldg(reinterpret_cast<const float2*>(coords) + p);
    const float inv = 1.f / (float)(1 << l);
    const float ix = cxy.x * inv + (float)di, iy = cxy.y * inv + (float)dj;
    const int H = pyr.h[l], W = pyr.w[l];
    const float* m = pyr.lvl[l] + p * pyr.stride[l];
    const float fx = floorf(ix), fy = floorf(iy);
    const float tx = ix - fx, ty = iy - fy;
    float v = 0.f;
    if (fx > -2.f && fx < (float)W && fy > -2.f && fy < (float)H) {
      const int x0 = (int)fx, y0 = (int)fy;
      const bool x0in = x0 >= 0 && x0 < W, x1in = x0 + 1 >= 0 && x0 + 1 < W;
      const bool y0in = y0 >= 0 && y0 < H, y1in = y0 + 1 >= 0 && y0 + 1 < H;
      if (y0in && x0in) v += __ldg(m + (int64_t)y0 * W + x0) * ((1.f - tx) * (1.f - ty));
      if (y0in && x1in) v += __ldg(m + (int64_t)y0 * W + x0 + 1) * (tx * (1.f - ty));
      if (y1in && x0in) v += __ldg(m + (int64_t)(y0 + 1) * W + x0) * ((1.f - tx) * ty);
      if (y1in && x1in) v += __ldg(m + (int64_t)(y0 + 1) * W + x0 + 1) * (tx * ty);
    }
    out[p * out_cpitch + k] = v;
  }
}

// out [B, h/2, w/2, C] = 2x2 means of in [B, h, w, C] (floor sizes, C % 4 == 0); ((a00 + a01) + a10) + a11, then / 4, as ATen
__global__ void __launch_bounds__(256)
raft_fmap_pool_kernel(const float4* __restrict__ in, float4* __restrict__ out, int h, int w, int C4, int64_t total) {
  const int ho = h / 2, wo = w / 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    int64_t t = i / C4;
    const int x = (int)(t % wo);
    t /= wo;
    const int y = (int)(t % ho);
    const int64_t b = t / ho;
    const float4* p = in + ((b * h + 2 * y) * w + 2 * x) * C4 + c;
    const float4 a = __ldg(p), bb = __ldg(p + C4), cc = __ldg(p + (int64_t)w * C4), d = __ldg(p + (int64_t)w * C4 + C4);
    float4 s;
    s.x = 0.f; s.x += a.x; s.x += bb.x; s.x += cc.x; s.x += d.x;
    s.y = 0.f; s.y += a.y; s.y += bb.y; s.y += cc.y; s.y += d.y;
    s.z = 0.f; s.z += a.z; s.z += bb.z; s.z += cc.z; s.z += d.z;
    s.w = 0.f; s.w += a.w; s.w += bb.w; s.w += cc.w; s.w += d.w;
    out[i] = make_float4(s.x / 4.f, s.y / 4.f, s.z / 4.f, s.w / 4.f);
  }
}

constexpr int FEAT_C = 256;                   // fnet's output channels
constexpr int OD_SIDE = WIN + 1;              // 10 integer positions per axis cover the 9 taps and their right / lower neighbours
constexpr int OD_POS = OD_SIDE * OD_SIDE;     // 100
constexpr int OD_WARPS = 8;

struct FeatPyramid {
  const float* lvl[LEVELS];                   // [B, h >> l, w >> l, 256] dense
  int h[LEVELS], w[LEVELS];
};

// one step of a reduce-scatter over the warp: lanes that differ in bit OFF exchange halves of v[0, 2 OFF) and keep v[s] = the pair's sum of
// slot s + (lane & OFF); after the steps 16, 8, 4, 2, 1, lane k holds in v[0] the warp's sum of slot k
template <int OFF>
__device__ __forceinline__ void butterfly_step(float (&v)[32], int lane) {
  const bool up = lane & OFF;
#pragma unroll
  for (int s = 0; s < OFF; ++s) {
    const float send = up ? v[s] : v[s + OFF];
    const float keep = up ? v[s + OFF] : v[s];
    v[s] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
  }
}

// One warp per pixel p (all four levels); lane k holds channels 4k..4k+3 and 128+4k..128+4k+3 of fmap1[p] in registers.  Per level the
// 100 dot products fmap1[p] . fmap2_l[by + i, bx + j] ((bx, by) = floor(coords / 2^l) - 4) are taken 32 at a time: each lane sums its
// 8 channels of every position (fp32 FMA chains), then a butterfly reduce-scatter over the lanes leaves position g*32 + k's sum in lane k
// (31 shuffles per 32 positions).  Positions outside the map are 0, as grid_sample's zero padding makes them.  The taps then combine
// four of the warp's dots with the lookup kernel's weights, in its order, and scale by 1/16.  The 8 warps of a CTA take consecutive
// pixels, so with coherent flows their windows share rows in L1.
__global__ void __launch_bounds__(OD_WARPS * 32)
raft_corr_ondemand_kernel(const float* __restrict__ f1, int64_t f1_bstride, FeatPyramid f2, const float* __restrict__ coords,
                          float* __restrict__ out, int out_cpitch, int64_t hw, int64_t npix) {
  __shared__ float dots[OD_WARPS][OD_POS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* dw = dots[warp];
  for (int64_t p = (int64_t)blockIdx.x * OD_WARPS + warp; p < npix; p += (int64_t)gridDim.x * OD_WARPS) {
    const int64_t b = p / hw;
    const float* a = f1 + b * f1_bstride + (p - b * hw) * FEAT_C;
    const float4 a0 = __ldg(reinterpret_cast<const float4*>(a) + lane), a1 = __ldg(reinterpret_cast<const float4*>(a + 128) + lane);
    const float2 cxy = __ldg(reinterpret_cast<const float2*>(coords) + p);
    float* o = out + p * out_cpitch;
    for (int l = 0; l < LEVELS; ++l) {
      const float inv = 1.f / (float)(1 << l);
      const float cx = cxy.x * inv, cy = cxy.y * inv;
      const float bxf = floorf(cx) - (float)RADIUS, byf = floorf(cy) - (float)RADIUS;
      const int H = f2.h[l], W = f2.w[l];
      // the window [bx, bx + 9] x [by, by + 9] misses the map (or the coordinate is not finite): every tap is 0
      if (!(bxf >= -(float)(OD_SIDE - 1) && bxf <= (float)(W - 1) && byf >= -(float)(OD_SIDE - 1) && byf <= (float)(H - 1))) {
        for (int k = lane; k < WIN * WIN; k += 32) o[l * (WIN * WIN) + k] = 0.f;
        continue;
      }
      const int bx = (int)bxf, by = (int)byf;
      const float* m = f2.lvl[l] + b * (int64_t)H * W * FEAT_C;
      for (int g = 0; g * 32 < OD_POS; ++g) {
        float v[32];
#pragma unroll
        for (int s = 0; s < 32; ++s) {
          const int q = g * 32 + s;
          const int Y = by + q / OD_SIDE, X = bx + q % OD_SIDE;
          float d = 0.f;
          if (q < OD_POS && Y >= 0 && Y < H && X >= 0 && X < W) {           // warp-uniform
            const float4* r = reinterpret_cast<const float4*>(m + ((int64_t)Y * W + X) * FEAT_C);
            const float4 b0 = __ldg(r + lane), b1 = __ldg(r + 32 + lane);
            d = a0.x * b0.x;
            d = fmaf(a0.y, b0.y, d); d = fmaf(a0.z, b0.z, d); d = fmaf(a0.w, b0.w, d);
            d = fmaf(a1.x, b1.x, d); d = fmaf(a1.y, b1.y, d); d = fmaf(a1.z, b1.z, d); d = fmaf(a1.w, b1.w, d);
          }
          v[s] = d;
        }
        butterfly_step<16>(v, lane);
        butterfly_step<8>(v, lane);
        butterfly_step<4>(v, lane);
        butterfly_step<2>(v, lane);
        butterfly_step<1>(v, lane);
        if (g * 32 + lane < OD_POS) dw[g * 32 + lane] = v[0];
      }
      __syncwarp();
      for (int k = lane; k < WIN * WIN; k += 32) {
        const int di = k / WIN - RADIUS, dj = k % WIN - RADIUS;
        const float ix = cx + (float)di, iy = cy + (float)dj;
        const float fx = floorf(ix), fy = floorf(iy);
        const float tx = ix - fx, ty = iy - fy;
        // floor(ix) is floor(cx) + di, or one more where ix rounded up to an integer: jx in [0, 9], and jx + 1 == 10 only where tx == 0
        const int jx = (int)fx - bx, jy = (int)fy - by;
        const bool xr = jx + 1 < OD_SIDE, yr = jy + 1 < OD_SIDE;
        const float* d = dw + jy * OD_SIDE + jx;
        float v = 0.f;
        v += d[0] * ((1.f - tx) * (1.f - ty));
        if (xr) v += d[1] * (tx * (1.f - ty));
        if (yr) v += d[OD_SIDE] * ((1.f - tx) * ty);
        if (xr && yr) v += d[OD_SIDE + 1] * (tx * ty);
        o[l * (WIN * WIN) + k] = v * (1.f / 16.f);                 // / sqrt(256), exact
      }
      __syncwarp();
    }
    for (int k = LOOKUP_C + lane; k < out_cpitch; k += 32) o[k] = 0.f;
  }
}

// out [B, h, w, Cout] = relu(bias + conv7x7(flow)), flow = coords1 - coords0 (2 channels, zero padding 3); w: [49][2][Cout]
__global__ void __launch_bounds__(256)
raft_convf1_kernel(const float* __restrict__ coords, const float* __restrict__ wt, const float* __restrict__ bias,
                   float* __restrict__ out, int h, int w, int Cout, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(i % Cout);
    const int64_t p = i / Cout;
    const int x = (int)(p % w);
    const int64_t t = p / w;
    const int y = (int)(t % h);
    const int64_t b = t / h;
    float acc = __ldg(bias + co);
    for (int ky = 0; ky < 7; ++ky) {
      const int yy = y + ky - 3;
      if (yy < 0 || yy >= h) continue;
      for (int kx = 0; kx < 7; ++kx) {
        const int xx = x + kx - 3;
        if (xx < 0 || xx >= w) continue;
        const float2 c = __ldg(reinterpret_cast<const float2*>(coords) + (b * h + yy) * w + xx);
        const float* wp = wt + (int64_t)((ky * 7 + kx) * 2) * Cout + co;
        acc = fmaf(c.x - (float)xx, __ldg(wp), acc);
        acc = fmaf(c.y - (float)yy, __ldg(wp + Cout), acc);
      }
    }
    out[i] = fmaxf(acc, 0.f);
  }
}

// coords [B, h, w, 2] (x, y): init -> the pixel grid; then + delta (planar [B, 2, h, w], may be NULL); flow_out (may be NULL) gets
// coords - grid at channel pitch flow_cpitch
__global__ void __launch_bounds__(256)
raft_flow_kernel(float* __restrict__ coords, const float* __restrict__ delta, int init, float* __restrict__ flow_out, int flow_cpitch,
                 int h, int w, int64_t total) {
  const int64_t hw = (int64_t)h * w;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(p % w);
    const int y = (int)((p / w) % h);
    const int64_t b = p / hw, q = p % hw;
    float cx, cy;
    if (init) { cx = (float)x; cy = (float)y; } else { cx = coords[2 * p]; cy = coords[2 * p + 1]; }
    if (delta) {
      cx = cx + __ldg(delta + (2 * b) * hw + q);
      cy = cy + __ldg(delta + (2 * b + 1) * hw + q);
    }
    coords[2 * p] = cx;
    coords[2 * p + 1] = cy;
    if (flow_out) {
      flow_out[p * flow_cpitch] = cx - (float)x;
      flow_out[p * flow_cpitch + 1] = cy - (float)y;
    }
  }
}

// rh [npix, C] = sigmoid(zr[:, C + c]) * h
__global__ void __launch_bounds__(256)
raft_gru_reset_kernel(const float* __restrict__ zr, const float* __restrict__ hs, float* __restrict__ rh, int C, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / C;
    const int c = (int)(i % C);
    rh[i] = sigmoidf_(__ldg(zr + p * 2 * C + C + c)) * __ldg(hs + i);
  }
}

// h = (1 - z) * h + z * tanh(q), z = sigmoid(zr[:, c]) (in place)
__global__ void __launch_bounds__(256)
raft_gru_update_kernel(const float* __restrict__ zr, const float* __restrict__ q, float* __restrict__ hs, int C, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / C;
    const int c = (int)(i % C);
    const float z = sigmoidf_(__ldg(zr + p * 2 * C + c));
    hs[i] = (1.f - z) * hs[i] + z * tanhf(__ldg(q + i));
  }
}

// up [B, 2, 8h, 8w]: at (8y + dy, 8x + dx) the softmax over k of mask[b, y, x, k*64 + dy*8 + dx] (k = 3x3 neighbour ky*3 + kx) weighting
// 8 * flow at (y + ky - 1, x + kx - 1) (0 outside); flow_low (may be NULL) [B, 2, h, w] = the flow itself
__global__ void __launch_bounds__(256)
raft_upsample_kernel(const float* __restrict__ mask, int mask_cpitch, const float* __restrict__ coords, float* __restrict__ up,
                     float* __restrict__ flow_low, int h, int w, int64_t total) {
  const int H = 8 * h, W = 8 * w;
  const int64_t HW = (int64_t)H * W, hw = (int64_t)h * w;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    const int Y = (int)((i / W) % H);
    const int64_t b = i / HW;
    const int x = X >> 3, dx = X & 7, y = Y >> 3, dy = Y & 7;
    const float* mp = mask + ((b * h + y) * w + x) * mask_cpitch + dy * 8 + dx;
    float lg[9];
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 9; ++k) { lg[k] = __ldg(mp + k * 64); mx = fmaxf(mx, lg[k]); }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) { lg[k] = expf(lg[k] - mx); s += lg[k]; }
    float u = 0.f, v = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
      float fx = 0.f, fy = 0.f;
      if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
        const float2 c = __ldg(reinterpret_cast<const float2*>(coords) + (b * h + yy) * w + xx);
        fx = 8.f * (c.x - (float)xx);
        fy = 8.f * (c.y - (float)yy);
      }
      const float wk = lg[k] / s;
      u += wk * fx;
      v += wk * fy;
    }
    up[(2 * b) * HW + (int64_t)Y * W + X] = u;
    up[(2 * b + 1) * HW + (int64_t)Y * W + X] = v;
    if (flow_low && dx == 0 && dy == 0) {
      const float2 c = __ldg(reinterpret_cast<const float2*>(coords) + (b * h + y) * w + x);
      flow_low[(2 * b) * hw + (int64_t)y * w + x] = c.x - (float)x;
      flow_low[(2 * b + 1) * hw + (int64_t)y * w + x] = c.y - (float)y;
    }
  }
}

bool al8(const void* p) { return ((uintptr_t)p & 7) == 0; }
bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

extern "C" int vt_raft_input_s2d_f32(const float* img1, const float* img2, float* out, int B, int H, int W, int cpad, void* stream) {
  VT_CHECK(img1 && out && B >= 1 && H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0 && cpad >= 12,
           "raft_input_s2d: bad args (even H, W and cpad >= 12 needed)");
  const int64_t total = (int64_t)(img2 ? 2 * B : B) * (H / 2) * (W / 2);
  raft_input_s2d_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(img1, img2, out, B, H, W, cpad, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_norm_relu_nhwc(const float* x, const float* stats, const float* res, const float* stats_res, float* out, int B,
                                      int64_t HW, int C, void* stream) {
  VT_CHECK(x && stats && out && B >= 1 && HW >= 1 && C >= 1 && al8(stats) && (!stats_res || (res && al8(stats_res))),
           "raft_norm_relu: bad args (stats_res needs res; stats 8-byte aligned)");
  const int64_t total = (int64_t)B * HW * C;
  raft_norm_relu_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(x, stats, res, stats_res, out, HW, C, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_context_f32(const float* cnet, float* net, float* inp, int64_t npix, int C, int inp_cpitch, void* stream) {
  VT_CHECK(cnet && net && inp && npix >= 1 && C >= 1 && inp_cpitch >= C, "raft_context: bad args");
  const int64_t total = npix * C;
  raft_context_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(cnet, net, inp, C, inp_cpitch, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_corr_pool_f32(const float* in, float* out, int64_t N, int h, int w, int64_t in_stride, void* stream) {
  VT_CHECK(in && out && N >= 1 && h >= 2 && w >= 2 && in_stride >= (int64_t)h * w, "raft_corr_pool: bad args (h, w >= 2)");
  const int64_t total = N * (h / 2) * (w / 2);
  raft_corr_pool_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, h, w, in_stride, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_corr_lookup_f32(const float* const* levels, const int64_t* strides, int h2, int w2, const float* coords, float* out,
                                       int out_cpitch, int64_t npix, void* stream) {
  VT_CHECK(levels && strides && coords && out && npix >= 1 && out_cpitch >= LOOKUP_C && al8(coords), "raft_corr_lookup: bad args");
  Pyramid pyr;
  int h = h2, w = w2;
  for (int l = 0; l < LEVELS; ++l) {
    VT_CHECK(levels[l] && h >= 1 && w >= 1 && strides[l] >= (int64_t)h * w, "raft_corr_lookup: level %d is empty or its stride too small", l);
    pyr.lvl[l] = levels[l]; pyr.stride[l] = strides[l]; pyr.h[l] = h; pyr.w[l] = w;
    h /= 2; w /= 2;
  }
  const int64_t total = npix * LOOKUP_C;
  raft_corr_lookup_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(pyr, coords, out, out_cpitch, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_fmap_pool_f32(const float* in, float* out, int B, int h, int w, int C, void* stream) {
  VT_CHECK(in && out && B >= 1 && h >= 2 && w >= 2 && C >= 4 && C % 4 == 0 && al16(in) && al16(out),
           "raft_fmap_pool: bad args (h, w >= 2, C a multiple of 4, 16-byte aligned rows)");
  const int64_t total = (int64_t)B * (h / 2) * (w / 2) * (C / 4);
  raft_fmap_pool_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(in),
                                                                               reinterpret_cast<float4*>(out), h, w, C / 4, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_corr_ondemand_f32(const float* fmap1, int64_t fmap1_bstride, const float* const* fmap2_levels, int B, int h,
                                         int w, const float* coords, float* out, int out_cpitch, void* stream) {
  VT_CHECK(fmap1 && fmap2_levels && coords && out && B >= 1 && (h >> (LEVELS - 1)) >= 1 && (w >> (LEVELS - 1)) >= 1 &&
               out_cpitch >= LOOKUP_C && al16(fmap1) && fmap1_bstride >= 0 && fmap1_bstride % 4 == 0 && al8(coords),
           "raft_corr_ondemand: bad args (h, w >= 8, fmap1 16-byte aligned with a batch stride of 0 or a multiple of 4)");
  FeatPyramid f2;
  for (int l = 0; l < LEVELS; ++l) {
    VT_CHECK(fmap2_levels[l] && al16(fmap2_levels[l]), "raft_corr_ondemand: fmap2 level %d is NULL or not 16-byte aligned", l);
    f2.lvl[l] = fmap2_levels[l]; f2.h[l] = h >> l; f2.w[l] = w >> l;
  }
  const int64_t npix = (int64_t)B * h * w;
  raft_corr_ondemand_kernel<<<grid1(npix, OD_WARPS), OD_WARPS * 32, 0, (cudaStream_t)stream>>>(fmap1, fmap1_bstride, f2, coords, out,
                                                                                            out_cpitch, (int64_t)h * w, npix);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_convf1_f32(const float* coords, const float* w, const float* bias, float* out, int B, int h, int wd, int Cout,
                                  void* stream) {
  VT_CHECK(coords && w && bias && out && B >= 1 && h >= 1 && wd >= 1 && Cout >= 1 && al8(coords), "raft_convf1: bad args");
  const int64_t total = (int64_t)B * h * wd * Cout;
  raft_convf1_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(coords, w, bias, out, h, wd, Cout, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_flow_f32(float* coords, const float* delta, int init, float* flow_out, int flow_cpitch, int B, int h, int w,
                                void* stream) {
  VT_CHECK(coords && B >= 1 && h >= 1 && w >= 1 && (!flow_out || flow_cpitch >= 2), "raft_flow: bad args");
  const int64_t total = (int64_t)B * h * w;
  raft_flow_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(coords, delta, init, flow_out, flow_cpitch, h, w, total);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_gru_reset_f32(const float* zr, const float* h, float* rh, int64_t npix, int C, void* stream) {
  VT_CHECK(zr && h && rh && npix >= 1 && C >= 1, "raft_gru_reset: bad args");
  raft_gru_reset_kernel<<<grid1(npix * C, 256), 256, 0, (cudaStream_t)stream>>>(zr, h, rh, C, npix * C);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_gru_update_f32(const float* zr, const float* q, float* h, int64_t npix, int C, void* stream) {
  VT_CHECK(zr && q && h && npix >= 1 && C >= 1, "raft_gru_update: bad args");
  raft_gru_update_kernel<<<grid1(npix * C, 256), 256, 0, (cudaStream_t)stream>>>(zr, q, h, C, npix * C);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_raft_upsample_f32(const float* mask, int mask_cpitch, const float* coords, float* up, float* flow_low, int B, int h,
                                    int w, void* stream) {
  VT_CHECK(mask && coords && up && B >= 1 && h >= 1 && w >= 1 && mask_cpitch >= 576 && al8(coords), "raft_upsample: bad args");
  const int64_t total = (int64_t)B * 64 * h * w;
  raft_upsample_kernel<<<grid1(total, 256), 256, 0, (cudaStream_t)stream>>>(mask, mask_cpitch, coords, up, flow_low, h, w, total);
  VT_LAUNCH_CHECK();
  return 0;
}
