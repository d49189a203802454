// elementwise.cu — HBM-bound streaming kernels: fused bias+leaky-relu, layout transforms, axpby, frame transforms.
//
//   fused_bias_act : y = lrelu(x + b[c], slope) * scale, written from the spec
//                    model/stylegan/op_cpu/fused_act.py:23-34 (== op/fused_bias_act_kernel.cu case act*10+grad == 30).
//                    float4 vectorised; the channel index is computed once per vector (no per-element div/mod).
//   nchw<->nhwc    : 32x32 smem-tiled transposes between the API layout (NCHW) and the internal NHWC layout.
//   frame u8<->f32 : ToTensor+Normalize(0.5,0.5) and util.tensor2cv2 (style_transfer.py:57-60, util.py:190-192).
#include "common.cuh"

namespace {

__global__ void __launch_bounds__(256)
fused_bias_act_vec4_kernel(const float4* __restrict__ in, const float* __restrict__ bias, float4* __restrict__ out,
                           int64_t n4, int64_t step_b4, int size_b, float slope, float scale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = __ldcs(in + i);
    float b = 0.f;
    if (bias) b = __ldg(bias + (int)((i / step_b4) % size_b));
    v.x = vt_lrelu(v.x + b, slope) * scale;
    v.y = vt_lrelu(v.y + b, slope) * scale;
    v.z = vt_lrelu(v.z + b, slope) * scale;
    v.w = vt_lrelu(v.w + b, slope) * scale;
    __stcs(out + i, v);
  }
}

__global__ void __launch_bounds__(256)
fused_bias_act_scalar_kernel(const float* __restrict__ in, const float* __restrict__ bias, float* __restrict__ out,
                             int64_t n, int64_t step_b, int size_b, float slope, float scale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float b = bias ? __ldg(bias + (int)((i / step_b) % size_b)) : 0.f;
    out[i] = vt_lrelu(in[i] + b, slope) * scale;
  }
}

// in: [B, C, HW] -> out: [B, HW, c_pad]; tile 32 (c) x 32 (hw)
__global__ void __launch_bounds__(256)
nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int64_t HW, int c_pad, int round_tf32) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int64_t hw0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const float* ip = in + (int64_t)b * C * HW;
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const int64_t hw = hw0 + tx;
    tile[j][tx] = (c < C && hw < HW) ? ip[(int64_t)c * HW + hw] : 0.f;
  }
  __syncthreads();
  float* op = out + (int64_t)b * HW * c_pad;
  for (int j = ty; j < 32; j += 8) {
    const int64_t hw = hw0 + j;
    const int c = c0 + tx;
    if (hw < HW && c < c_pad) {
      float v = tile[tx][j];
      op[hw * c_pad + c] = round_tf32 ? vt_round_tf32(v) : v;
    }
  }
}

// in: [B, HW, c_stride] -> out: [B, C, HW]
__global__ void __launch_bounds__(256)
nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int64_t HW, int c_stride) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int64_t hw0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float* ip = in + (int64_t)b * HW * c_stride;
  for (int j = ty; j < 32; j += 8) {
    const int64_t hw = hw0 + j;
    const int c = c0 + tx;
    tile[j][tx] = (hw < HW && c < C) ? ip[hw * c_stride + c] : 0.f;
  }
  __syncthreads();
  float* op = out + (int64_t)b * C * HW;
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const int64_t hw = hw0 + tx;
    if (c < C && hw < HW) op[(int64_t)c * HW + hw] = tile[tx][j];
  }
}

__global__ void __launch_bounds__(256)
axpby_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int64_t n,
             float sa, float sb, int round_tf32) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = a[i] * sa;
    if (b) v += b[i] * sb;
    out[i] = round_tf32 ? vt_round_tf32(v) : v;
  }
}

// u8 HWC -> f32 NCHW, one thread per pixel
__global__ void __launch_bounds__(256)
frame_u8_to_f32_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int64_t HW, int swap_rb,
                       int64_t out_batch_stride) {
  const int b = blockIdx.y;
  const uint8_t* ip = in + (int64_t)b * HW * 3;
  float* op = out + (int64_t)b * out_batch_stride;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (int64_t)gridDim.x * blockDim.x) {
    uint8_t c0 = ip[p * 3 + 0], c1 = ip[p * 3 + 1], c2 = ip[p * 3 + 2];
    if (swap_rb) { uint8_t t = c0; c0 = c2; c2 = t; }
    // ToTensor: v/255 ; Normalize(0.5, 0.5): (v - 0.5) / 0.5   (same op order as torchvision)
    op[p] = vt_u8_unit(c0);
    op[HW + p] = vt_u8_unit(c1);
    op[2 * HW + p] = vt_u8_unit(c2);
  }
}

// f32 NCHW (3ch) -> clamp -> u8 HWC ; tensor2cv2: ((x + 1) * 127.5).astype(uint8) (truncation), optional RGB->BGR
__global__ void __launch_bounds__(256)
f32_to_frame_u8_kernel(const float* __restrict__ in, uint8_t* __restrict__ out, int64_t HW, int swap_rb) {
  const int b = blockIdx.y;
  const float* ip = in + (int64_t)b * 3 * HW;
  uint8_t* op = out + (int64_t)b * HW * 3;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (int64_t)gridDim.x * blockDim.x) {
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float x = fminf(fmaxf(ip[(int64_t)c * HW + p], -1.f), 1.f);
      v[c] = (x + 1.0f) * 127.5f;
    }
    uint8_t r = (uint8_t)(int)v[0], g = (uint8_t)(int)v[1], bl = (uint8_t)(int)v[2];
    if (swap_rb) { uint8_t t = r; r = bl; bl = t; }
    op[p * 3 + 0] = r; op[p * 3 + 1] = g; op[p * 3 + 2] = bl;
  }
}

// SE gate * x + (strided) shortcut, float4 over channels
__global__ void __launch_bounds__(256)
gate_shortcut_add_kernel(const float* __restrict__ x, const float* __restrict__ gate, const float* __restrict__ sc,
                         float* __restrict__ out, int H, int W, int C, int Hs, int Ws, int sc_stride, int round_tf32) {
  const int b = blockIdx.y;
  const int nvec = C / 4;
  const int64_t total = (int64_t)H * W * nvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % nvec) * 4;
    const int64_t p = i / nvec;
    const int xx = (int)(p % W), yy = (int)(p / W);
    float4 v = *reinterpret_cast<const float4*>(x + (((int64_t)b * H + yy) * W + xx) * C + c);
    if (gate) {
      const float4 g = *reinterpret_cast<const float4*>(gate + (int64_t)b * C + c);
      v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
    }
    const float4 s = *reinterpret_cast<const float4*>(sc + (((int64_t)b * Hs + (int64_t)yy * sc_stride) * Ws + (int64_t)xx * sc_stride) * C + c);
    v.x += s.x; v.y += s.y; v.z += s.z; v.w += s.w;
    if (round_tf32) { v.x = vt_round_tf32(v.x); v.y = vt_round_tf32(v.y); v.z = vt_round_tf32(v.z); v.w = vt_round_tf32(v.w); }
    *reinterpret_cast<float4*>(out + (((int64_t)b * H + yy) * W + xx) * C + c) = v;
  }
}

// F.interpolate(x, size=(H,W), mode='bilinear', align_corners=True) + y  (psp_encoders.py:87-88)
__global__ void __launch_bounds__(256)
bilinear_add_kernel(const float* __restrict__ x, const float* __restrict__ y, float* __restrict__ out, int h, int w, int H,
                    int W, int C, int round_tf32) {
  const int b = blockIdx.y;
  const int nvec = C / 4;
  const int64_t total = (int64_t)H * W * nvec;
  const float sy = (H > 1) ? (float)(h - 1) / (float)(H - 1) : 0.f;
  const float sx = (W > 1) ? (float)(w - 1) / (float)(W - 1) : 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % nvec) * 4;
    const int64_t p = i / nvec;
    const int ox = (int)(p % W), oy = (int)(p / W);
    const float fy = oy * sy, fx = ox * sx;
    int y0 = (int)fy, x0 = (int)fx;
    const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const float* xb = x + (int64_t)b * h * w * C + c;
    const float4 v00 = *reinterpret_cast<const float4*>(xb + ((int64_t)y0 * w + x0) * C);
    const float4 v01 = *reinterpret_cast<const float4*>(xb + ((int64_t)y0 * w + x1) * C);
    const float4 v10 = *reinterpret_cast<const float4*>(xb + ((int64_t)y1 * w + x0) * C);
    const float4 v11 = *reinterpret_cast<const float4*>(xb + ((int64_t)y1 * w + x1) * C);
    const float4 yy = *reinterpret_cast<const float4*>(y + (((int64_t)b * H + oy) * W + ox) * C + c);
    const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
    float4 o;
    o.x = w00 * v00.x + w01 * v01.x + w10 * v10.x + w11 * v11.x + yy.x;
    o.y = w00 * v00.y + w01 * v01.y + w10 * v10.y + w11 * v11.y + yy.y;
    o.z = w00 * v00.z + w01 * v01.z + w10 * v10.z + w11 * v11.z + yy.z;
    o.w = w00 * v00.w + w01 * v01.w + w10 * v10.w + w11 * v11.w + yy.w;
    if (round_tf32) { o.x = vt_round_tf32(o.x); o.y = vt_round_tf32(o.y); o.z = vt_round_tf32(o.z); o.w = vt_round_tf32(o.w); }
    *reinterpret_cast<float4*>(out + (((int64_t)b * H + oy) * W + ox) * C + c) = o;
  }
}

inline unsigned grid_for(int64_t work_items, int threads) {
  int64_t blocks = vt_cdiv(work_items, threads);
  const int64_t cap = (int64_t)vt_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

}  // namespace

extern "C" int vt_fused_bias_act_f32(const float* in, const float* bias, float* out, int64_t n, int64_t step_b,
                                     int size_b, float negative_slope, float scale, void* stream) {
  VT_CHECK(in && out, "fused_bias_act: null pointer");
  VT_CHECK(n >= 0, "fused_bias_act: negative size");
  if (n == 0) return 0;
  if (bias) VT_CHECK(step_b >= 1 && size_b >= 1, "fused_bias_act: bad bias broadcast (step_b=%lld size_b=%d)", (long long)step_b, size_b);
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = (n % 4 == 0) && (!bias || step_b % 4 == 0) && (((uintptr_t)in & 15) == 0) && (((uintptr_t)out & 15) == 0);
  if (vec) {
    fused_bias_act_vec4_kernel<<<grid_for(n / 4, 256), 256, 0, st>>>((const float4*)in, bias, (float4*)out, n / 4,
                                                                    bias ? step_b / 4 : 1, bias ? size_b : 1,
                                                                    negative_slope, scale);
  } else {
    fused_bias_act_scalar_kernel<<<grid_for(n, 256), 256, 0, st>>>(in, bias, out, n, bias ? step_b : 1,
                                                                  bias ? size_b : 1, negative_slope, scale);
  }
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_nchw_to_nhwc_f32(const float* in, float* out, int B, int C, int H, int W, int c_pad, int round_tf32, void* stream) {
  VT_CHECK(in && out && B >= 1 && C >= 1 && H >= 1 && W >= 1 && c_pad >= C, "nchw_to_nhwc: bad args");
  const int64_t HW = (int64_t)H * W;
  VT_CHECK(B <= 65535 && vt_cdiv(c_pad, 32) <= 65535, "nchw_to_nhwc: grid too large");
  dim3 grid((unsigned)vt_cdiv(HW, 32), (unsigned)vt_cdiv(c_pad, 32), (unsigned)B);
  nchw_to_nhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, C, HW, c_pad, round_tf32);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_nhwc_to_nchw_f32(const float* in, float* out, int B, int C, int H, int W, int c_stride, void* stream) {
  VT_CHECK(in && out && B >= 1 && C >= 1 && H >= 1 && W >= 1 && c_stride >= C, "nhwc_to_nchw: bad args");
  const int64_t HW = (int64_t)H * W;
  VT_CHECK(B <= 65535 && vt_cdiv(C, 32) <= 65535, "nhwc_to_nchw: grid too large");
  dim3 grid((unsigned)vt_cdiv(HW, 32), (unsigned)vt_cdiv(C, 32), (unsigned)B);
  nhwc_to_nchw_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, C, HW, c_stride);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_axpby_f32(const float* a, const float* b, float* out, int64_t n, float scale_a, float scale_b,
                            int round_tf32, void* stream) {
  VT_CHECK(n >= 0, "axpby: negative size");
  if (n == 0) return 0;                 // empty tensors may have null data pointers
  VT_CHECK(a && out, "axpby: null pointer");
  axpby_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, out, n, scale_a, scale_b, round_tf32);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_gate_shortcut_add_nhwc(const float* x, const float* gate, const float* sc, float* out, int B, int H, int W,
                                         int C, int Hs, int Ws, int sc_stride, int round_tf32, void* stream) {
  VT_CHECK(x && sc && out && B >= 1 && B <= 65535 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0, "gate_shortcut_add: bad args");
  VT_CHECK(sc_stride >= 1 && (int64_t)(H - 1) * sc_stride < Hs && (int64_t)(W - 1) * sc_stride < Ws, "gate_shortcut_add: shortcut too small");
  dim3 grid(grid_for((int64_t)H * W * (C / 4), 256), (unsigned)B);
  gate_shortcut_add_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, gate, sc, out, H, W, C, Hs, Ws, sc_stride, round_tf32);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_bilinear_add_nhwc(const float* x, const float* y, float* out, int B, int h, int w, int H, int W, int C,
                                    int round_tf32, void* stream) {
  VT_CHECK(x && y && out && B >= 1 && B <= 65535 && h >= 1 && w >= 1 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0, "bilinear_add: bad args");
  dim3 grid(grid_for((int64_t)H * W * (C / 4), 256), (unsigned)B);
  bilinear_add_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, out, h, w, H, W, C, round_tf32);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_frame_u8_to_f32(const uint8_t* in, float* out, int B, int H, int W, int swap_rb,
                                  int64_t out_batch_stride, void* stream) {
  VT_CHECK(in && out && B >= 1 && B <= 65535 && H >= 1 && W >= 1, "frame_u8_to_f32: bad args");
  const int64_t HW = (int64_t)H * W;
  VT_CHECK(out_batch_stride >= 3 * HW, "frame_u8_to_f32: out_batch_stride too small");
  dim3 grid(grid_for(HW, 256), (unsigned)B);
  frame_u8_to_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, HW, swap_rb, out_batch_stride);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_f32_to_frame_u8(const float* in, uint8_t* out, int B, int H, int W, int swap_rb, void* stream) {
  VT_CHECK(in && out && B >= 1 && B <= 65535 && H >= 1 && W >= 1, "f32_to_frame_u8: bad args");
  const int64_t HW = (int64_t)H * W;
  dim3 grid(grid_for(HW, 256), (unsigned)B);
  f32_to_frame_u8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, HW, swap_rb);
  VT_LAUNCH_CHECK();
  return 0;
}

// ---- f4: backward of the fused bias + leaky-relu op (model/stylegan/op/fused_act.py:20-84, fused_bias_act_kernel.cu act*10+grad == 31)
namespace {

__global__ void __launch_bounds__(256)
fused_bias_act_grad_kernel(const float* __restrict__ in, const float* __restrict__ bias, const float* __restrict__ ref,
                           float* __restrict__ out, int64_t n, int64_t step_b, int size_b, float slope, float scale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float x = in[i];
    if (bias) x += __ldg(bias + (int)((i / step_b) % size_b));
    out[i] = (ref[i] > 0.f ? x : x * slope) * scale;
  }
}

// deterministic per-channel sum of a [outer, C, inner] tensor: stage 1 writes CH_SPLIT partial sums per channel (fixed
// assignment of elements to partials and fixed reduction trees), stage 2 adds them in order
constexpr int CH_SPLIT = 64;

__global__ void __launch_bounds__(256)
channel_sum_partial_kernel(const float* __restrict__ in, float* __restrict__ partial, int outer, int C, int64_t inner) {
  const int c = blockIdx.x, part = blockIdx.y;
  const int64_t total = (int64_t)outer * inner;
  float acc = 0.f;
  for (int64_t j = (int64_t)part * blockDim.x + threadIdx.x; j < total; j += (int64_t)CH_SPLIT * blockDim.x) {
    const int64_t o = j / inner, k = j - o * inner;
    acc += in[(o * C + c) * inner + k];
  }
  __shared__ float red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s2 = 128; s2 > 0; s2 >>= 1) {
    if ((int)threadIdx.x < s2) red[threadIdx.x] += red[threadIdx.x + s2];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[c * CH_SPLIT + part] = red[0];
}

__global__ void channel_sum_final_kernel(const float* __restrict__ partial, float* __restrict__ out, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc = 0.f;
  for (int i = 0; i < CH_SPLIT; ++i) acc += partial[c * CH_SPLIT + i];
  out[c] = acc;
}

}  // namespace

extern "C" int vt_fused_bias_act_grad_f32(const float* in, const float* bias, const float* ref, float* out, int64_t n,
                                          int64_t step_b, int size_b, float negative_slope, float scale, void* stream) {
  VT_CHECK(in && ref && out && n >= 1, "fused_bias_act_grad: null pointer / empty tensor");
  VT_CHECK(!bias || (step_b >= 1 && size_b >= 1), "fused_bias_act_grad: bad bias broadcast");
  int64_t blocks = vt_cdiv(n, 256);
  const int64_t cap = (int64_t)vt_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  fused_bias_act_grad_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(in, bias, ref, out, n, bias ? step_b : 1,
                                                                               bias ? size_b : 1, negative_slope, scale);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t vt_channel_sum_ws_floats(int C) { return (int64_t)C * CH_SPLIT; }

extern "C" int vt_channel_sum_f32(const float* in, float* out, float* workspace, int outer, int C, int64_t inner, void* stream) {
  VT_CHECK(in && out && workspace && outer >= 1 && C >= 1 && C <= 65535 && inner >= 1, "channel_sum: bad args");
  channel_sum_partial_kernel<<<dim3((unsigned)C, CH_SPLIT), 256, 0, (cudaStream_t)stream>>>(in, workspace, outer, C, inner);
  VT_LAUNCH_CHECK();
  channel_sum_final_kernel<<<(unsigned)vt_cdiv(C, 128), 128, 0, (cudaStream_t)stream>>>(workspace, out, C);
  VT_LAUNCH_CHECK();
  return 0;
}
