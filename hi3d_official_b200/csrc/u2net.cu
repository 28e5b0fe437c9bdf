// Kernels of the U^2-Net background-removal network (u2net.py) that the GEMM engine's epilogues cannot express: the RSU
// blocks' ceil-mode 2x2 max-pool, the size-matched bilinear resize (align_corners=False) that fills the upsample half of each
// decoder concat in place, and the fusion of the six side outputs into the sigmoid probability map.  The pool and the resize
// are HBM streams on NHWC fp16 with 16-byte accesses and channel strides on both sides, so that either end may be a channel
// slice of a concat buffer; see include/hi3d_b200.h for the reference call sites.
#include <cstring>

#include "common.cuh"

namespace hi3d {

constexpr int U2_MAX_SIDES = 8;

// MaxPool2d(2, 2, ceil_mode=True): one thread per (output pixel, 8 channels); a window that hangs over the bottom / right edge
// takes the max of its valid elements only.
__global__ void maxpool2x2_ceil_kernel(const __half* __restrict__ x, int x_ld, int H, int W, int C, int Ho, int Wo,
                                       long long total, __half* __restrict__ y, int y_ld) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int CV = C / 8;
  const long long pixel = idx / CV;
  const int c0 = (int)(idx - pixel * CV) * 8;
  const long long im = pixel / ((long long)Ho * Wo);
  const int pix = (int)(pixel - im * Ho * Wo), oy = pix / Wo, ox = pix - oy * Wo;
  const int iy0 = 2 * oy, ix0 = 2 * ox;
  const int ny = (iy0 + 1 < H) ? 2 : 1, nx = (ix0 + 1 < W) ? 2 : 1;
  const __half* base = x + ((im * H + iy0) * W + ix0) * (long long)x_ld + c0;
  Half8 m = *reinterpret_cast<const Half8*>(base);
  for (int dy = 0; dy < ny; dy++)
    for (int dx = 0; dx < nx; dx++) {
      if (dy == 0 && dx == 0) continue;
      const Half8 v = *reinterpret_cast<const Half8*>(base + ((long long)dy * W + dx) * x_ld);
#pragma unroll
      for (int q = 0; q < 4; q++) m.h[q] = __hmax2_nan(m.h[q], v.h[q]);
    }
  *reinterpret_cast<Half8*>(y + pixel * (long long)y_ld + c0) = m;
}

// Source coordinate of F.interpolate(mode='bilinear', align_corners=False) without a scale_factor: scale = in / out in fp32,
// src = max(scale * (dst + 0.5) - 0.5, 0) as one fused multiply-add, as PyTorch's CUDA kernel computes it; the lower tap, the
// clamped upper tap and the weight of the upper tap.
struct Tap1 {
  int i0, i1;
  float l1;
};

HI3D_DEVINL Tap1 bilinear_tap(int dst, int in, float scale) {
  float s = fmaf(scale, (float)dst + 0.5f, -0.5f);
  s = fmaxf(s, 0.f);
  Tap1 t;
  t.i0 = (int)s;
  t.i1 = t.i0 + (t.i0 < in - 1);
  t.l1 = s - (float)t.i0;
  return t;
}

// Bilinear resize Hs x Ws -> Ht x Wt (align_corners=False), one thread per (output pixel, 8 channels), fp32 with one rounding.
__global__ void resize_bilinear_kernel(const __half* __restrict__ x, int x_ld, int Hs, int Ws, int C, int Ht, int Wt, float sh,
                                       float sw, long long total, __half* __restrict__ y, int y_ld) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int CV = C / 8;
  const long long pixel = idx / CV;
  const int c0 = (int)(idx - pixel * CV) * 8;
  const long long im = pixel / ((long long)Ht * Wt);
  const int pix = (int)(pixel - im * Ht * Wt), oy = pix / Wt, ox = pix - oy * Wt;
  const Tap1 ty = bilinear_tap(oy, Hs, sh), tx = bilinear_tap(ox, Ws, sw);
  const float h1 = ty.l1, h0 = 1.f - h1, w1 = tx.l1, w0 = 1.f - w1;
  const __half* base = x + im * Hs * Ws * (long long)x_ld + c0;
  const Half8 v00 = *reinterpret_cast<const Half8*>(base + ((long long)ty.i0 * Ws + tx.i0) * x_ld);
  const Half8 v01 = *reinterpret_cast<const Half8*>(base + ((long long)ty.i0 * Ws + tx.i1) * x_ld);
  const Half8 v10 = *reinterpret_cast<const Half8*>(base + ((long long)ty.i1 * Ws + tx.i0) * x_ld);
  const Half8 v11 = *reinterpret_cast<const Half8*>(base + ((long long)ty.i1 * Ws + tx.i1) * x_ld);
  Half8 o;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const float2 a = __half22float2(v00.h[k]), b = __half22float2(v01.h[k]);
    const float2 c = __half22float2(v10.h[k]), d = __half22float2(v11.h[k]);
    const float fx = h0 * (w0 * a.x + w1 * b.x) + h1 * (w0 * c.x + w1 * d.x);
    const float fy = h0 * (w0 * a.y + w1 * b.y) + h1 * (w0 * c.y + w1 * d.y);
    o.h[k] = __floats2half2_rn(fx, fy);
  }
  *reinterpret_cast<Half8*>(y + pixel * (long long)y_ld + c0) = o;
}

struct U2Sides {
  const __half* src[U2_MAX_SIDES];
  int ld[U2_MAX_SIDES], h[U2_MAX_SIDES], w[U2_MAX_SIDES];
  float sh[U2_MAX_SIDES], sw[U2_MAX_SIDES];
};

// prob = sigmoid(b0 + sum_k resize(side_k)) at H x W: channel 0 of each side map, read through the same bilinear taps as
// resize_bilinear_kernel, summed in fp32.  One thread per output pixel.
__global__ void u2net_fuse_sides_kernel(U2Sides s, int n_sides, float b0, int H, int W, long long total, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const long long im = idx / ((long long)H * W);
  const int pix = (int)(idx - im * H * W), oy = pix / W, ox = pix - oy * W;
  float acc = b0;
  for (int k = 0; k < n_sides; k++) {
    const int hs = s.h[k], ws = s.w[k], ld = s.ld[k];
    const Tap1 ty = bilinear_tap(oy, hs, s.sh[k]), tx = bilinear_tap(ox, ws, s.sw[k]);
    const __half* base = s.src[k] + im * hs * ws * (long long)ld;
    const float a = __half2float(base[((long long)ty.i0 * ws + tx.i0) * ld]);
    const float b = __half2float(base[((long long)ty.i0 * ws + tx.i1) * ld]);
    const float c = __half2float(base[((long long)ty.i1 * ws + tx.i0) * ld]);
    const float d = __half2float(base[((long long)ty.i1 * ws + tx.i1) * ld]);
    const float h1 = ty.l1, h0 = 1.f - h1, w1 = tx.l1, w0 = 1.f - w1;
    acc += h0 * (w0 * a + w1 * b) + h1 * (w0 * c + w1 * d);
  }
  out[idx] = 1.f / (1.f + expf(-acc));
}

static unsigned u2_blocks(long long total) { return (unsigned)((total + 255) / 256); }

}  // namespace hi3d

using namespace hi3d;

extern "C" int hi3d_maxpool2x2_ceil(const void* x, int x_ld, int n, int H, int W, int C, void* y, int y_ld, void* stream) {
  if (!x || !y || n <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 || x_ld < C || x_ld % 8 || y_ld < C || y_ld % 8 ||
      ((uintptr_t)x & 15) || ((uintptr_t)y & 15)) {
    set_error("hi3d_maxpool2x2_ceil: bad arguments (n=%d H=%d W=%d C=%d x_ld=%d y_ld=%d)", n, H, W, C, x_ld, y_ld);
    return -2;
  }
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const long long total = (long long)n * Ho * Wo * (C / 8);
  maxpool2x2_ceil_kernel<<<u2_blocks(total), 256, 0, (cudaStream_t)stream>>>((const __half*)x, x_ld, H, W, C, Ho, Wo, total,
                                                                            (__half*)y, y_ld);
  return check_launch("hi3d_maxpool2x2_ceil");
}

extern "C" int hi3d_resize_bilinear(const void* x, int x_ld, int n, int Hs, int Ws, int C, void* y, int y_ld, int Ht, int Wt,
                                    void* stream) {
  if (!x || !y || n <= 0 || Hs <= 0 || Ws <= 0 || Ht <= 0 || Wt <= 0 || C <= 0 || C % 8 || x_ld < C || x_ld % 8 || y_ld < C ||
      y_ld % 8 || ((uintptr_t)x & 15) || ((uintptr_t)y & 15)) {
    set_error("hi3d_resize_bilinear: bad arguments (n=%d %dx%d -> %dx%d C=%d x_ld=%d y_ld=%d)", n, Hs, Ws, Ht, Wt, C, x_ld, y_ld);
    return -2;
  }
  const long long total = (long long)n * Ht * Wt * (C / 8);
  resize_bilinear_kernel<<<u2_blocks(total), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)x, x_ld, Hs, Ws, C, Ht, Wt, (float)Hs / (float)Ht, (float)Ws / (float)Wt, total, (__half*)y, y_ld);
  return check_launch("hi3d_resize_bilinear");
}

extern "C" int hi3d_u2net_fuse_sides(const void* const* sides, const int* side_ld, const int* side_h, const int* side_w,
                                     int n_sides, float b0, int n, int H, int W, float* out, void* stream) {
  if (!sides || !side_ld || !side_h || !side_w || n_sides <= 0 || n_sides > U2_MAX_SIDES || n <= 0 || H <= 0 || W <= 0 || !out) {
    set_error("hi3d_u2net_fuse_sides: bad arguments (sides=%d n=%d H=%d W=%d)", n_sides, n, H, W);
    return -2;
  }
  U2Sides s;
  memset(&s, 0, sizeof(s));
  for (int k = 0; k < n_sides; k++) {
    if (!sides[k] || side_ld[k] <= 0 || side_h[k] <= 0 || side_w[k] <= 0) {
      set_error("hi3d_u2net_fuse_sides: bad side %d (ld=%d %dx%d)", k, side_ld[k], side_h[k], side_w[k]);
      return -2;
    }
    s.src[k] = (const __half*)sides[k];
    s.ld[k] = side_ld[k];
    s.h[k] = side_h[k];
    s.w[k] = side_w[k];
    s.sh[k] = (float)side_h[k] / (float)H;
    s.sw[k] = (float)side_w[k] / (float)W;
  }
  const long long total = (long long)n * H * W;
  u2net_fuse_sides_kernel<<<u2_blocks(total), 256, 0, (cudaStream_t)stream>>>(s, n_sides, b0, H, W, total, out);
  return check_launch("hi3d_u2net_fuse_sides");
}
