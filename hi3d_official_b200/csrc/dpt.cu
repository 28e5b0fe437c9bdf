// Kernels of the conditioner's MiDaS DPT-Hybrid depth tower (midas.py) that the GEMM engine's epilogues cannot express: the
// BiT stem's patch rows and "same" max-pool, GroupNorm apply with a fused shortcut / ReLU, the fusion blocks' bilinear x2
// (align_corners=True) with a fused addend, and the ReLU copy of a residual conv unit's input.  All are HBM streams on NHWC
// fp16 with 16-byte accesses; see include/hi3d_b200.h for the reference call sites.
#include "common.cuh"

namespace hi3d {

constexpr int DPT_GROUPS = 32;

// One thread per 8 columns of one patch row: the 7x7 stride-2 stem conv of BiT (timm StdConv2dSame) as rows for a plain GEMM,
// K ordered (c, ky, kx) like weight.reshape(Co, 147), zero beyond K = 147 and outside the image (the TF "same" zero pad).
template <typename TI>
__global__ void dpt_stem_rows_kernel(const TI* __restrict__ img, int H, int W, int Ho, int Wo, int pad_t, int pad_l, int Kpad,
                                     long long total, __half* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cpr = Kpad / 8;
  const long long row = idx / cpr;
  const int k0 = (int)(idx - row * cpr) * 8;
  const long long im = row / ((long long)Ho * Wo);
  const int pix = (int)(row - im * Ho * Wo), oy = pix / Wo, ox = pix - oy * Wo;
  Half8 v;
#pragma unroll
  for (int e = 0; e < 8; e += 2) {
    float a[2];
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int k = k0 + e + u;
      float val = 0.f;
      if (k < 147) {
        const int c = k / 49, r = k - c * 49, ky = r / 7, kx = r - ky * 7;
        const int iy = 2 * oy + ky - pad_t, ix = 2 * ox + kx - pad_l;
        if ((unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W) val = (float)img[((im * 3 + c) * H + iy) * W + ix];
      }
      a[u] = val;
    }
    v.h[e / 2] = __floats2half2_rn(a[0], a[1]);
  }
  *reinterpret_cast<Half8*>(out + row * Kpad + k0) = v;
}

// 3x3 stride-2 max-pool, one thread per (output pixel, 8 channels); the "same" pad is -inf (timm MaxPool2dSame), so only
// pixels inside the image take part.
__global__ void maxpool3x3s2_kernel(const __half* __restrict__ x, int H, int W, int C, int Ho, int Wo, int pad_t, int pad_l,
                                    long long total, __half* __restrict__ y) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int CV = C / 8;
  const long long pixel = idx / CV;
  const int c0 = (int)(idx - pixel * CV) * 8;
  const long long im = pixel / ((long long)Ho * Wo);
  const int pix = (int)(pixel - im * Ho * Wo), oy = pix / Wo, ox = pix - oy * Wo;
  const __half2 ninf = __halves2half2(__ushort_as_half(0xfc00), __ushort_as_half(0xfc00));
  Half8 m;
#pragma unroll
  for (int q = 0; q < 4; q++) m.h[q] = ninf;
  for (int dy = 0; dy < 3; dy++) {
    const int iy = 2 * oy - pad_t + dy;
    if ((unsigned)iy >= (unsigned)H) continue;
    for (int dx = 0; dx < 3; dx++) {
      const int ix = 2 * ox - pad_l + dx;
      if ((unsigned)ix >= (unsigned)W) continue;
      const Half8 v = *reinterpret_cast<const Half8*>(x + ((im * H + iy) * W + ix) * C + c0);
#pragma unroll
      for (int q = 0; q < 4; q++) m.h[q] = __hmax2_nan(m.h[q], v.h[q]);
    }
  }
  *reinterpret_cast<Half8*>(y + pixel * C + c0) = m;
}

// y = [relu](GN(x) + addend), addend = a raw tensor, GN_a(a) or nothing.  Group statistics of each image come from the unit
// tables of hi3d_groupnorm_unit_stats; grid (row slabs, images), each thread owns one 8-channel column.
__global__ void __launch_bounds__(256)
gn_apply_add_kernel(const __half* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                    const float* __restrict__ beta, const __half* __restrict__ a, const float* __restrict__ a_stats,
                    const float* __restrict__ a_gamma, const float* __restrict__ a_beta, int C, int unit, long long rows,
                    long long rows_per_cta, float eps, int relu, __half* __restrict__ y, long long y_sample_rows,
                    long long y_row_off) {
  __shared__ float smean[2][DPT_GROUPS], srstd[2][DPT_GROUPS];
  const int tid = threadIdx.x, img = blockIdx.y;
  const int cpg = C / DPT_GROUPS, upg = cpg / unit, nu = C / unit;
  if (tid < 2 * DPT_GROUPS) {
    const int which = tid / DPT_GROUPS, g = tid % DPT_GROUPS;
    const float* st = which ? a_stats : stats;
    if (st != nullptr) {
      double s = 0.0, q = 0.0;
      for (int u = 0; u < upg; u++) {
        const float* e = st + ((long long)img * nu + g * upg + u) * 2;
        s += (double)e[0];
        q += (double)e[1];
      }
      const double cnt = (double)rows * (double)cpg;
      const double mean = s / cnt;
      double var = q / cnt - mean * mean;
      if (var < 0.0) var = 0.0;
      smean[which][g] = (float)mean;
      srstd[which][g] = (float)(1.0 / sqrt(var + (double)eps));
    }
  }
  __syncthreads();
  const int CV = C >> 3, cv = tid % CV, rl = tid / CV, RL = blockDim.x / CV;
  const int c0 = cv * 8;
  float A[8], B[8], A2[8], B2[8];
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const int c = c0 + e, g = c / cpg;
    A[e] = srstd[0][g] * gamma[c];
    B[e] = beta[c] - smean[0][g] * A[e];
    A2[e] = 1.f;
    B2[e] = 0.f;
    if (a_stats != nullptr) {
      A2[e] = srstd[1][g] * a_gamma[c];
      B2[e] = a_beta[c] - smean[1][g] * A2[e];
    }
  }
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  long long r1 = r0 + rows_per_cta;
  if (r1 > rows) r1 = rows;
  const __half* xb = x + (long long)img * rows * C + c0;
  const __half* ab = a ? a + (long long)img * rows * C + c0 : nullptr;
  __half* yb = y + ((long long)img * y_sample_rows + y_row_off) * C + c0;
  for (long long r = r0 + rl; r < r1; r += RL) {
    const Half8 v = *reinterpret_cast<const Half8*>(xb + r * C);
    Half8 w;
    if (ab) w = *reinterpret_cast<const Half8*>(ab + r * C);
    Half8 o;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      float2 f = __half22float2(v.h[k]);
      f.x = f.x * A[2 * k] + B[2 * k];
      f.y = f.y * A[2 * k + 1] + B[2 * k + 1];
      if (ab) {
        const float2 g = __half22float2(w.h[k]);
        f.x += g.x * A2[2 * k] + B2[2 * k];
        f.y += g.y * A2[2 * k + 1] + B2[2 * k + 1];
      }
      if (relu) {
        f.x = fmaxf(f.x, 0.f);
        f.y = fmaxf(f.y, 0.f);
      }
      o.h[k] = __floats2half2_rn(f.x, f.y);
    }
    *reinterpret_cast<Half8*>(yb + r * C) = o;
  }
}

// Bilinear x2 with align_corners=True (source coordinate = o * (in - 1) / (out - 1), as F.interpolate computes it in fp32),
// plus an optional addend of the output's shape; one thread per (output pixel, 8 channels).
__global__ void upsample2x_bilinear_ac_kernel(const __half* __restrict__ x, int H, int W, int C, const __half* __restrict__ add,
                                              long long total, __half* __restrict__ y) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int CV = C / 8, Ho = 2 * H, Wo = 2 * W;
  const long long pixel = idx / CV;
  const int c0 = (int)(idx - pixel * CV) * 8;
  const long long im = pixel / ((long long)Ho * Wo);
  const int pix = (int)(pixel - im * Ho * Wo), oy = pix / Wo, ox = pix - oy * Wo;
  const float sh = (float)(H - 1) / (float)(Ho - 1), sw = (float)(W - 1) / (float)(Wo - 1);
  const float fy = sh * (float)oy, fx = sw * (float)ox;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < H - 1), x1 = x0 + (x0 < W - 1);
  const float ly = fy - (float)y0, lx = fx - (float)x0;
  const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
  const __half* base = x + im * H * W * C + c0;
  const Half8 v00 = *reinterpret_cast<const Half8*>(base + ((long long)y0 * W + x0) * C);
  const Half8 v01 = *reinterpret_cast<const Half8*>(base + ((long long)y0 * W + x1) * C);
  const Half8 v10 = *reinterpret_cast<const Half8*>(base + ((long long)y1 * W + x0) * C);
  const Half8 v11 = *reinterpret_cast<const Half8*>(base + ((long long)y1 * W + x1) * C);
  Half8 ad;
  if (add) ad = *reinterpret_cast<const Half8*>(add + pixel * C + c0);
  Half8 o;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const float2 a = __half22float2(v00.h[k]), b = __half22float2(v01.h[k]);
    const float2 c = __half22float2(v10.h[k]), d = __half22float2(v11.h[k]);
    float2 f = make_float2(w00 * a.x + w01 * b.x + w10 * c.x + w11 * d.x, w00 * a.y + w01 * b.y + w10 * c.y + w11 * d.y);
    if (add) {
      const float2 g = __half22float2(ad.h[k]);
      f.x += g.x;
      f.y += g.y;
    }
    o.h[k] = __floats2half2_rn(f.x, f.y);
  }
  *reinterpret_cast<Half8*>(y + pixel * C + c0) = o;
}

__global__ void relu_copy_kernel(const __half* __restrict__ x, long long n8, __half* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  Half8 v = reinterpret_cast<const Half8*>(x)[i];
  const __half2 z = __float2half2_rn(0.f);
#pragma unroll
  for (int q = 0; q < 4; q++) v.h[q] = __hmax2_nan(v.h[q], z);
  reinterpret_cast<Half8*>(y)[i] = v;
}

// TF "same" padding before the first row / column of a k x k stride-2 window: ceil(in / 2) outputs, the odd pixel at the end
static int same_pad_lo(int in, int k) {
  const int out = (in + 1) / 2;
  const int total = (out - 1) * 2 + k - in;
  return total > 0 ? total / 2 : 0;
}

static unsigned blocks_for(long long total) { return (unsigned)((total + 255) / 256); }

}  // namespace hi3d

using namespace hi3d;

extern "C" int hi3d_dpt_stem_rows(const void* img, int img_is_fp32, int n, int H, int W, int Kpad, void* out, void* stream) {
  if (!img || !out || n <= 0 || H <= 0 || W <= 0 || Kpad < 147 || Kpad % 8 || ((uintptr_t)out & 15)) {
    set_error("hi3d_dpt_stem_rows: bad arguments (n=%d H=%d W=%d Kpad=%d)", n, H, W, Kpad);
    return -2;
  }
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const long long total = (long long)n * Ho * Wo * (Kpad / 8);
  if (img_is_fp32)
    dpt_stem_rows_kernel<float><<<blocks_for(total), 256, 0, (cudaStream_t)stream>>>(
        (const float*)img, H, W, Ho, Wo, same_pad_lo(H, 7), same_pad_lo(W, 7), Kpad, total, (__half*)out);
  else
    dpt_stem_rows_kernel<__half><<<blocks_for(total), 256, 0, (cudaStream_t)stream>>>(
        (const __half*)img, H, W, Ho, Wo, same_pad_lo(H, 7), same_pad_lo(W, 7), Kpad, total, (__half*)out);
  return check_launch("hi3d_dpt_stem_rows");
}

extern "C" int hi3d_maxpool3x3s2_same(const void* x, int n, int H, int W, int C, void* y, void* stream) {
  if (!x || !y || n <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 || ((uintptr_t)x & 15) || ((uintptr_t)y & 15)) {
    set_error("hi3d_maxpool3x3s2_same: bad arguments (n=%d H=%d W=%d C=%d)", n, H, W, C);
    return -2;
  }
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const long long total = (long long)n * Ho * Wo * (C / 8);
  maxpool3x3s2_kernel<<<blocks_for(total), 256, 0, (cudaStream_t)stream>>>((const __half*)x, H, W, C, Ho, Wo, same_pad_lo(H, 3),
                                                                          same_pad_lo(W, 3), total, (__half*)y);
  return check_launch("hi3d_maxpool3x3s2_same");
}

extern "C" int hi3d_groupnorm_apply_add(const void* x, const float* stats, const float* gamma, const float* beta, const void* add,
                                        const float* add_stats, const float* add_gamma, const float* add_beta, int C, int unit,
                                        int n_images, int64_t rows_per_image, float eps, int apply_relu, void* y,
                                        int64_t y_sample_rows, int64_t y_row_off, void* stream) {
  if (!x || !stats || !gamma || !beta || !y || C <= 0 || C % DPT_GROUPS || C % 8 || C > 2048 || unit <= 0 ||
      (C / DPT_GROUPS) % unit || n_images <= 0 || n_images > 65535 || rows_per_image <= 0 || ((uintptr_t)x & 15) ||
      ((uintptr_t)y & 15) || (add && ((uintptr_t)add & 15)) || (add_stats && (!add || !add_gamma || !add_beta)) ||
      (y_sample_rows > 0 && (y_row_off < 0 || y_row_off + rows_per_image > y_sample_rows))) {
    set_error("hi3d_groupnorm_apply_add: bad arguments (C=%d unit=%d n=%d rows=%lld y_sample_rows=%lld y_row_off=%lld)", C, unit,
              n_images, (long long)rows_per_image, (long long)y_sample_rows, (long long)y_row_off);
    return -2;
  }
  if (y_sample_rows <= 0) { y_sample_rows = rows_per_image; y_row_off = 0; }
  const int CV = C / 8, threads = (256 / CV) * CV, RL = threads / CV;
  long long slabs = (132 * 8 + n_images - 1) / n_images;
  const long long max_slabs = (rows_per_image + RL - 1) / RL;
  if (slabs > max_slabs) slabs = max_slabs;
  long long rows_per_cta = (rows_per_image + slabs - 1) / slabs;
  rows_per_cta = (rows_per_cta + RL - 1) / RL * RL;
  slabs = (rows_per_image + rows_per_cta - 1) / rows_per_cta;
  gn_apply_add_kernel<<<dim3((unsigned)slabs, n_images), threads, 0, (cudaStream_t)stream>>>(
      (const __half*)x, stats, gamma, beta, (const __half*)add, add_stats, add_gamma, add_beta, C, unit, rows_per_image,
      rows_per_cta, eps, apply_relu, (__half*)y, y_sample_rows, y_row_off);
  return check_launch("hi3d_groupnorm_apply_add");
}

extern "C" int hi3d_upsample2x_bilinear_ac(const void* x, int n, int H, int W, int C, const void* add, void* y, void* stream) {
  if (!x || !y || n <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 || ((uintptr_t)x & 15) || ((uintptr_t)y & 15) ||
      (add && ((uintptr_t)add & 15))) {
    set_error("hi3d_upsample2x_bilinear_ac: bad arguments (n=%d H=%d W=%d C=%d)", n, H, W, C);
    return -2;
  }
  const long long total = (long long)n * 4 * H * W * (C / 8);
  upsample2x_bilinear_ac_kernel<<<blocks_for(total), 256, 0, (cudaStream_t)stream>>>((const __half*)x, H, W, C,
                                                                                    (const __half*)add, total, (__half*)y);
  return check_launch("hi3d_upsample2x_bilinear_ac");
}

extern "C" int hi3d_relu_copy(const void* x, int64_t n, void* y, void* stream) {
  if (!x || !y || n <= 0 || n % 8 || ((uintptr_t)x & 15) || ((uintptr_t)y & 15)) {
    set_error("hi3d_relu_copy: bad arguments (n=%lld)", (long long)n);
    return -2;
  }
  relu_copy_kernel<<<blocks_for(n / 8), 256, 0, (cudaStream_t)stream>>>((const __half*)x, n / 8, (__half*)y);
  return check_launch("hi3d_relu_copy");
}
