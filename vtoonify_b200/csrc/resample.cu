// Resampling helpers of the face-parsing pre-network (model/bisenet/model.py, style_transfer.py:171-174): frame preparation
// (2x bilinear up-sampling + space-to-depth for the stride-2 7x7 stem), 3x3/2 max-pool, nearest resize, and the final
// bilinear (align_corners=True) read-out of the logits.  All HBM-bound, float4 over channels where the layout allows.
#include "common.cuh"

namespace {

// out[b, y, x, (py*2+px)*3 + c] = X[b, c, 2y+py, 2x+px], X = in (mode 0) or 2 * bilinear_up2(in) (mode 1, align_corners=False);
// channels 12..cpad-1 are zero; rows/columns beyond X are zero.  in: planar [B,3,Hin,Win]; out: NHWC [B,Ho,Wo,cpad].
__global__ void __launch_bounds__(256)
frame_s2d_kernel(const float* __restrict__ in, float* __restrict__ out, int Hin, int Win, int Ho, int Wo, int cpad, int mode) {
  const int b = blockIdx.y;
  const int64_t total = (int64_t)Ho * Wo;
  const int XH = mode ? 2 * Hin : Hin, XW = mode ? 2 * Win : Win;
  const float* ip = in + (int64_t)b * 3 * Hin * Win;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % Wo), y = (int)(i / Wo);
    float v[12];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int Y = 2 * y + (q >> 1), X = 2 * x + (q & 1);
      const bool ok = Y < XH && X < XW;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float r = 0.f;
        if (ok) {
          const float* pl = ip + (int64_t)c * Hin * Win;
          if (mode == 0) {
            r = __ldg(pl + (int64_t)Y * Win + X);
          } else {
            // F.interpolate(scale_factor=2, mode='bilinear', align_corners=False): src = (dst + 0.5) / 2 - 0.5, clamped at 0
            float sy = (Y + 0.5f) * 0.5f - 0.5f, sx = (X + 0.5f) * 0.5f - 0.5f;
            sy = sy < 0.f ? 0.f : sy; sx = sx < 0.f ? 0.f : sx;
            const int y0 = (int)sy, x0 = (int)sx;
            const int y1 = y0 + (y0 < Hin - 1 ? 1 : 0), x1 = x0 + (x0 < Win - 1 ? 1 : 0);
            const float ly = sy - (float)y0, lx = sx - (float)x0;
            const float a = __ldg(pl + (int64_t)y0 * Win + x0), bq = __ldg(pl + (int64_t)y0 * Win + x1);
            const float cq = __ldg(pl + (int64_t)y1 * Win + x0), d = __ldg(pl + (int64_t)y1 * Win + x1);
            // same association as ATen's upsample_bilinear2d: h0*(w0*a + w1*b) + h1*(w0*c + w1*d)
            r = 2.f * ((1.f - ly) * ((1.f - lx) * a + lx * bq) + ly * ((1.f - lx) * cq + lx * d));
          }
        }
        v[q * 3 + c] = r;
      }
    }
    float4* op = reinterpret_cast<float4*>(out + (((int64_t)b * Ho + y) * Wo + x) * cpad);
    op[0] = make_float4(v[0], v[1], v[2], v[3]);
    op[1] = make_float4(v[4], v[5], v[6], v[7]);
    op[2] = make_float4(v[8], v[9], v[10], v[11]);
    for (int k = 3; k < cpad / 4; ++k) op[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// nn.MaxPool2d(3, 2, 1) on NHWC (padding acts as -inf)
__global__ void __launch_bounds__(256)
maxpool3x3s2_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int C, int Ho, int Wo) {
  const int b = blockIdx.y, nvec = C / 4;
  const int64_t total = (int64_t)Ho * Wo * nvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % nvec) * 4;
    const int64_t p = i / nvec;
    const int ox = (int)(p % Wo), oy = (int)(p / Wo);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = 2 * oy - 1 + ky;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = 2 * ox - 1 + kx;
        if (ix < 0 || ix >= W) continue;
        const float4 a = *reinterpret_cast<const float4*>(in + (((int64_t)b * H + iy) * W + ix) * C + c);
        m.x = fmaxf(m.x, a.x); m.y = fmaxf(m.y, a.y); m.z = fmaxf(m.z, a.z); m.w = fmaxf(m.w, a.w);
      }
    }
    *reinterpret_cast<float4*>(out + (((int64_t)b * Ho + oy) * Wo + ox) * C + c) = m;
  }
}

// nn.MaxPool2d(2, 2) on NHWC (VGG16 of the LPIPS loss); the last row / column of an odd map is dropped
__global__ void __launch_bounds__(256)
maxpool2x2_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int C, int Ho, int Wo) {
  const int b = blockIdx.y, nvec = C / 4;
  const int64_t total = (int64_t)Ho * Wo * nvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % nvec) * 4;
    const int64_t p = i / nvec;
    const int ox = (int)(p % Wo), oy = (int)(p / Wo);
    const float* r0 = in + (((int64_t)b * H + 2 * oy) * W + 2 * ox) * C + c;
    const float4 a = __ldg(reinterpret_cast<const float4*>(r0)), bq = __ldg(reinterpret_cast<const float4*>(r0 + C));
    const float4 cq = __ldg(reinterpret_cast<const float4*>(r0 + (int64_t)W * C));
    const float4 d = __ldg(reinterpret_cast<const float4*>(r0 + (int64_t)W * C + C));
    float4 m;
    m.x = fmaxf(fmaxf(a.x, bq.x), fmaxf(cq.x, d.x)); m.y = fmaxf(fmaxf(a.y, bq.y), fmaxf(cq.y, d.y));
    m.z = fmaxf(fmaxf(a.z, bq.z), fmaxf(cq.z, d.z)); m.w = fmaxf(fmaxf(a.w, bq.w), fmaxf(cq.w, d.w));
    *reinterpret_cast<float4*>(out + (((int64_t)b * Ho + oy) * Wo + ox) * C + c) = m;
  }
}

// the window element that receives the gradient: the first maximal one in row-major order, as ATen's max_pool2d records it
__device__ __forceinline__ void maxpool2x2_route(float a, float b, float c, float d, float g, float (&o)[4]) {
  const float m = fmaxf(fmaxf(a, b), fmaxf(c, d));
  const int k = a == m ? 0 : (b == m ? 1 : (c == m ? 2 : 3));
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = j == k ? g : 0.f;
}

// Adjoint of maxpool2x2_kernel, one thread per (window, 4 channels): the argmax is recomputed from the pool input x (no index
// tensor); add (may be NULL) is added to every input position, and rows / columns dropped by the floor get add (or 0) alone.
__global__ void __launch_bounds__(256)
maxpool2x2_grad_kernel(const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ add, float* __restrict__ gx,
                       int H, int W, int C, int Ho, int Wo) {
  const int b = blockIdx.y, nvec = C / 4;
  const int64_t total = (int64_t)Ho * Wo * nvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % nvec) * 4;
    const int64_t p = i / nvec;
    const int ox = (int)(p % Wo), oy = (int)(p / Wo);
    int64_t off[4];
    off[0] = (((int64_t)b * H + 2 * oy) * W + 2 * ox) * C + c;
    off[1] = off[0] + C;
    off[2] = off[0] + (int64_t)W * C;
    off[3] = off[2] + C;
    float4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = __ldg(reinterpret_cast<const float4*>(x + off[j]));
    const float4 gv = __ldg(reinterpret_cast<const float4*>(g + (((int64_t)b * Ho + oy) * Wo + ox) * C + c));
    float o[4][4];   // [channel][window element]
    maxpool2x2_route(v[0].x, v[1].x, v[2].x, v[3].x, gv.x, o[0]);
    maxpool2x2_route(v[0].y, v[1].y, v[2].y, v[3].y, gv.y, o[1]);
    maxpool2x2_route(v[0].z, v[1].z, v[2].z, v[3].z, gv.z, o[2]);
    maxpool2x2_route(v[0].w, v[1].w, v[2].w, v[3].w, gv.w, o[3]);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float4 r = make_float4(o[0][j], o[1][j], o[2][j], o[3][j]);
      if (add) {
        const float4 s = __ldg(reinterpret_cast<const float4*>(add + off[j]));
        r.x += s.x; r.y += s.y; r.z += s.z; r.w += s.w;
      }
      *reinterpret_cast<float4*>(gx + off[j]) = r;
    }
    // the floor's dropped last column / row (and their corner) are written by the windows next to them
    const bool col = (W & 1) && ox == Wo - 1, row = (H & 1) && oy == Ho - 1;
    auto pass = [&](int64_t o) {
      *reinterpret_cast<float4*>(gx + o) = add ? __ldg(reinterpret_cast<const float4*>(add + o)) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    if (col) { pass(off[1] + C); pass(off[3] + C); }
    if (row) { pass(off[2] + (int64_t)W * C); pass(off[3] + (int64_t)W * C); }
    if (col && row) pass(off[3] + (int64_t)W * C + C);
  }
}

// F.interpolate(x, (H, W), mode='nearest') on NHWC: src = min(floor(dst * in/out), in - 1) with the scale in fp32 (ATen)
__global__ void __launch_bounds__(256)
resize_nearest_kernel(const float* __restrict__ in, float* __restrict__ out, int h, int w, int H, int W, int C) {
  const int b = blockIdx.y, nvec = C / 4;
  const float fy = (float)h / (float)H, fx = (float)w / (float)W;
  const int64_t total = (int64_t)H * W * nvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % nvec) * 4;
    const int64_t p = i / nvec;
    const int x = (int)(p % W), y = (int)(p / W);
    int sy = (int)floorf((float)y * fy), sx = (int)floorf((float)x * fx);
    sy = sy < h - 1 ? sy : h - 1; sx = sx < w - 1 ? sx : w - 1;
    *reinterpret_cast<float4*>(out + (((int64_t)b * H + y) * W + x) * C + c) =
        *reinterpret_cast<const float4*>(in + (((int64_t)b * h + sy) * w + sx) * C + c);
  }
}

// out[b, c, y, x] = scale * bilinear(logits[b, :, :, c]) evaluated at pixel (step*y, step*x) of the (Hf, Wf) grid that
// F.interpolate(logits, (Hf, Wf), mode='bilinear', align_corners=True) would produce: src = dst * (h - 1) / (Hf - 1).
// step 2 = the frame loop's nearest x0.5 of the 2x-size parsing map (style_transfer.py:171-172) without materialising it.
__global__ void __launch_bounds__(256)
logits_readout_kernel(const float* __restrict__ in, float* __restrict__ out, int h, int w, int cs, int ncls, int Hf, int Wf,
                      int Ho, int Wo, int step, float scale, int64_t out_bstride) {
  const int b = blockIdx.y;
  const float ry = Hf > 1 ? (float)(h - 1) / (float)(Hf - 1) : 0.f, rx = Wf > 1 ? (float)(w - 1) / (float)(Wf - 1) : 0.f;
  const int64_t total = (int64_t)Ho * Wo;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % Wo), y = (int)(i / Wo);
    const float sy = ry * (float)(step * y), sx = rx * (float)(step * x);
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
    const float ly = sy - (float)y0, lx = sx - (float)x0;
    const float* p00 = in + (((int64_t)b * h + y0) * w + x0) * cs;
    const float* p01 = in + (((int64_t)b * h + y0) * w + x1) * cs;
    const float* p10 = in + (((int64_t)b * h + y1) * w + x0) * cs;
    const float* p11 = in + (((int64_t)b * h + y1) * w + x1) * cs;
    for (int c = 0; c < ncls; ++c) {
      const float v = (1.f - ly) * ((1.f - lx) * __ldg(p00 + c) + lx * __ldg(p01 + c)) + ly * ((1.f - lx) * __ldg(p10 + c) + lx * __ldg(p11 + c));
      out[(int64_t)b * out_bstride + ((int64_t)c * Ho + y) * Wo + x] = scale * v;
    }
  }
}

unsigned grid1(int64_t work, int threads) {
  int64_t blocks = vt_cdiv(work, threads);
  const int64_t cap = (int64_t)vt_num_sms() * 16;
  return (unsigned)(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}

}  // namespace

extern "C" int vt_frame_s2d_f32(const float* in, float* out, int B, int Hin, int Win, int Ho, int Wo, int cpad, int upsample2,
                                void* stream) {
  VT_CHECK(in && out && B >= 1 && B <= 65535 && Hin >= 1 && Win >= 1, "frame_s2d: bad args");
  VT_CHECK(cpad >= 12 && cpad % 4 == 0 && ((uintptr_t)out & 15) == 0, "frame_s2d: cpad must be a multiple of 4 >= 12, out 16-byte aligned");
  const int XH = upsample2 ? 2 * Hin : Hin, XW = upsample2 ? 2 * Win : Win;
  VT_CHECK(Ho == (XH + 1) / 2 && Wo == (XW + 1) / 2, "frame_s2d: output must be ceil(X/2) (got %dx%d for X %dx%d)", Ho, Wo, XH, XW);
  frame_s2d_kernel<<<dim3(grid1((int64_t)Ho * Wo, 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(in, out, Hin, Win, Ho, Wo, cpad,
                                                                                                      upsample2 ? 1 : 0);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_maxpool3x3s2_nhwc_f32(const float* in, float* out, int B, int H, int W, int C, void* stream) {
  VT_CHECK(in && out && B >= 1 && B <= 65535 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0, "maxpool3x3s2: bad args");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;   // floor((H + 2 - 3) / 2) + 1
  maxpool3x3s2_kernel<<<dim3(grid1((int64_t)Ho * Wo * (C / 4), 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(in, out, H, W, C, Ho, Wo);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_maxpool2x2_nhwc_f32(const float* in, float* out, int B, int H, int W, int C, void* stream) {
  VT_CHECK(in && out && B >= 1 && B <= 65535 && H >= 2 && W >= 2 && C >= 4 && C % 4 == 0, "maxpool2x2: bad args");
  VT_CHECK((((uintptr_t)in | (uintptr_t)out) & 15) == 0, "maxpool2x2: tensors must be 16-byte aligned");
  const int Ho = H / 2, Wo = W / 2;
  maxpool2x2_kernel<<<dim3(grid1((int64_t)Ho * Wo * (C / 4), 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(in, out, H, W, C, Ho, Wo);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_maxpool2x2_grad_nhwc_f32(const float* g, const float* x, const float* add, float* gx, int B, int H, int W, int C,
                                           void* stream) {
  VT_CHECK(g && x && gx && B >= 1 && B <= 65535 && H >= 2 && W >= 2 && C >= 4 && C % 4 == 0, "maxpool2x2_grad: bad args");
  VT_CHECK((((uintptr_t)g | (uintptr_t)x | (uintptr_t)add | (uintptr_t)gx) & 15) == 0, "maxpool2x2_grad: tensors must be 16-byte aligned");
  const int Ho = H / 2, Wo = W / 2;
  maxpool2x2_grad_kernel<<<dim3(grid1((int64_t)Ho * Wo * (C / 4), 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(g, x, add, gx, H, W,
                                                                                                                    C, Ho, Wo);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_resize_nearest_nhwc_f32(const float* in, float* out, int B, int h, int w, int H, int W, int C, void* stream) {
  VT_CHECK(in && out && B >= 1 && B <= 65535 && h >= 1 && w >= 1 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0, "resize_nearest: bad args");
  resize_nearest_kernel<<<dim3(grid1((int64_t)H * W * (C / 4), 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(in, out, h, w, H, W, C);
  VT_LAUNCH_CHECK();
  return 0;
}

extern "C" int vt_logits_readout_f32(const float* in, float* out, int B, int h, int w, int c_stride, int n_classes, int Hf, int Wf,
                                     int Ho, int Wo, int step, float scale, int64_t out_bstride, void* stream) {
  if (out_bstride == 0) out_bstride = (int64_t)n_classes * Ho * Wo;
  VT_CHECK(out_bstride >= (int64_t)n_classes * Ho * Wo, "logits_readout: out_bstride smaller than one sample");
  VT_CHECK(in && out && B >= 1 && B <= 65535 && h >= 1 && w >= 1 && n_classes >= 1 && c_stride >= n_classes, "logits_readout: bad args");
  VT_CHECK(step >= 1 && Ho >= 1 && Wo >= 1 && (int64_t)(Ho - 1) * step < Hf && (int64_t)(Wo - 1) * step < Wf,
           "logits_readout: the sampled pixels must lie inside the (Hf, Wf) grid");
  logits_readout_kernel<<<dim3(grid1((int64_t)Ho * Wo, 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(in, out, h, w, c_stride, n_classes,
                                                                                                          Hf, Wf, Ho, Wo, step, scale, out_bstride);
  VT_LAUNCH_CHECK();
  return 0;
}
