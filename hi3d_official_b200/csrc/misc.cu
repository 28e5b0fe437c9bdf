// Sampler-side fused elementwise kernels and layout converters (all HBM-bound, vectorised where the
// layout allows).  See include/hi3d_b200.h for the reference call sites each one replaces.
#include "common.cuh"

namespace hi3d {

__global__ void timestep_embedding_kernel(const float* __restrict__ t, int n, int dim, float neg_log_period_over_half,
                                          __half* __restrict__ out) {
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half) return;
  const int i = idx / half, k = idx - i * half;
  const float freq = expf(neg_log_period_over_half * (float)k);
  const float a = t[i] * freq;
  out[(long long)i * dim + k] = __float2half_rn(cosf(a));
  out[(long long)i * dim + half + k] = __float2half_rn(sinf(a));
  if ((dim & 1) && k == 0) out[(long long)i * dim + dim - 1] = __float2half(0.f);
}

template <typename TC>
__global__ void sampler_pre_kernel(const float* __restrict__ x, const float* __restrict__ sigma,
                                   const TC* __restrict__ cuc, const TC* __restrict__ cc, int F, int Cx, int Cc, int HW,
                                   int Cpad, __half* __restrict__ out, float* __restrict__ c_noise_out) {
  // one thread per (sample n in [0, 2F), pixel): writes Cpad channels (16-byte vectors)
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)2 * F * HW) return;
  const int n = (int)(idx / HW), pix = (int)(idx - (long long)n * HW);
  const int f = n % F;
  const bool cond = n >= F;
  const float sg = sigma[f];
  const float c_in = rsqrtf(sg * sg + 1.f);
  if (pix == 0 && c_noise_out != nullptr) c_noise_out[n] = 0.25f * logf(sg);   // VScalingWithEDMcNoise c_noise
  const TC* cat = cond ? cc : cuc;
  __half* o = out + idx * Cpad;
  for (int c0 = 0; c0 < Cpad; c0 += 8) {
    Half8 v;
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      float a[2];
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int c = c0 + e + u;
        float val = 0.f;
        if (c < Cx) val = x[((long long)f * Cx + c) * HW + pix] * c_in;
        else if (c < Cx + Cc && cat != nullptr) val = (float)cat[((long long)f * Cc + (c - Cx)) * HW + pix];
        a[u] = val;
      }
      v.h[e / 2] = __floats2half2_rn(a[0], a[1]);
    }
    *reinterpret_cast<Half8*>(o + c0) = v;
  }
}

__global__ void sampler_post_kernel(const __half* __restrict__ net, int net_ld, const float* __restrict__ x,
                                    const float* __restrict__ sigma, const float* __restrict__ sigma_next,
                                    const float* __restrict__ scale, int T, int F, int Cx, int HW,
                                    float* __restrict__ x_out, float* __restrict__ den_out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)F * HW) return;
  const int f = (int)(idx / HW), pix = (int)(idx - (long long)f * HW);
  const float sg = sigma[f], sn = sigma_next[f];
  const float d2 = sg * sg + 1.f;
  const float c_skip = 1.f / d2, c_out = -sg * rsqrtf(d2);
  const float gs = scale[f % T];
  const __half* nu = net + ((long long)f * HW + pix) * net_ld;
  const __half* nc = net + ((long long)(F + f) * HW + pix) * net_ld;
  for (int c = 0; c < Cx; c++) {
    const long long xi = ((long long)f * Cx + c) * HW + pix;
    const float xv = x[xi];
    const float du = __half2float(nu[c]) * c_out + xv * c_skip;
    const float dc = __half2float(nc[c]) * c_out + xv * c_skip;
    const float den = du + gs * (dc - du);
    if (den_out) den_out[xi] = den;
    const float d = (xv - den) / sg;
    x_out[xi] = xv + d * (sn - sg);
  }
}

// The pre step of every sampler, guider and churn setting: `rows` = 2 (CFG batch, uc half first) or 1 (IdentityGuider, cond
// rows only).  With eps, the network sees the churned x_hat = x + (eps * s_noise) * sqrt(sigma^2 - sigma_from^2) (EDMSampler,
// sampling.py:94-97), which the first row of each frame also writes to x_hat_out for the post step.
template <typename TC>
__global__ void sampler_pre_ex_kernel(const float* __restrict__ x, const float* __restrict__ sigma,
                                      const float* __restrict__ sigma_from, const float* __restrict__ eps, float s_noise,
                                      const TC* __restrict__ cuc, const TC* __restrict__ cc, int rows, int F, int Cx, int Cc,
                                      int HW, int Cpad, __half* __restrict__ out, float* __restrict__ c_noise_out,
                                      float* __restrict__ x_hat_out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)rows * F * HW) return;
  const int n = (int)(idx / HW), pix = (int)(idx - (long long)n * HW);
  const int f = n % F;
  const bool cond = rows == 1 || n >= F;
  const float sg = sigma[f];
  const float c_in = rsqrtf(sg * sg + 1.f);
  float churn = 0.f;
  if (eps) {
    const float sf = sigma_from[f];
    churn = sqrtf(sg * sg - sf * sf);
  }
  if (pix == 0 && c_noise_out != nullptr) c_noise_out[n] = 0.25f * logf(sg);
  const TC* cat = cond ? cc : cuc;
  __half* o = out + idx * Cpad;
  for (int c0 = 0; c0 < Cpad; c0 += 8) {
    Half8 v;
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      float a[2];
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int c = c0 + e + u;
        float val = 0.f;
        if (c < Cx) {
          const long long xi = ((long long)f * Cx + c) * HW + pix;
          float xv = x[xi];
          if (eps) {
            xv = xv + (eps[xi] * s_noise) * churn;
            if (n == f) x_hat_out[xi] = xv;
          }
          val = xv * c_in;
        } else if (c < Cx + Cc && cat != nullptr) {
          val = (float)cat[((long long)f * Cc + (c - Cx)) * HW + pix];
        }
        a[u] = val;
      }
      v.h[e / 2] = __floats2half2_rn(a[0], a[1]);
    }
    *reinterpret_cast<Half8*>(o + c0) = v;
  }
}

// The post step with an ancestral update and an optional guider: scale == nullptr reads F network rows (IdentityGuider), else
// 2F rows combined with scale[f % T].  x_out = x + d (sigma_to - sigma), then + (eps * s_noise) * sigma_up where sigma_next > 0
// (AncestralSampler, sampling.py:158-170).
__global__ void sampler_post_ancestral_kernel(const __half* __restrict__ net, int net_ld, const float* __restrict__ x,
                                              const float* __restrict__ sigma, const float* __restrict__ sigma_to,
                                              const float* __restrict__ scale, int T, const float* __restrict__ eps,
                                              float s_noise, const float* __restrict__ sigma_up,
                                              const float* __restrict__ sigma_next, int F, int Cx, int HW,
                                              float* __restrict__ x_out, float* __restrict__ den_out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)F * HW) return;
  const int f = (int)(idx / HW), pix = (int)(idx - (long long)f * HW);
  const float sg = sigma[f], st = sigma_to[f];
  const float d2 = sg * sg + 1.f;
  const float c_skip = 1.f / d2, c_out = -sg * rsqrtf(d2);
  const bool noise = eps != nullptr && sigma_next[f] > 0.f;
  const float su = eps != nullptr ? sigma_up[f] : 0.f;
  const __half* nc = net + ((long long)((scale ? F : 0) + f) * HW + pix) * net_ld;
  const __half* nu = net + ((long long)f * HW + pix) * net_ld;
  const float gs = scale ? scale[f % T] : 1.f;
  for (int c = 0; c < Cx; c++) {
    const long long xi = ((long long)f * Cx + c) * HW + pix;
    const float xv = x[xi];
    float den = __half2float(nc[c]) * c_out + xv * c_skip;
    if (scale) {
      const float du = __half2float(nu[c]) * c_out + xv * c_skip;
      den = du + gs * (den - du);
    }
    if (den_out) den_out[xi] = den;
    const float d = (xv - den) / sg;
    float xn = xv + d * (st - sg);
    if (noise) xn = xn + (eps[xi] * s_noise) * su;
    x_out[xi] = xn;
  }
}

struct LincombTerms {
  const float* x[8];
  const float* c[8];
};

// out = sum_k c_k[f] x_k over up to 8 terms: linear multistep of order 4 over (x, D) pairs, DPM-Solver++(2S)'s selected update.
__global__ void lincomb_kernel(float* __restrict__ out, LincombTerms t, int nterms, int per_sample, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = (int)(i / per_sample);
  float v = t.c[0][f] * t.x[0][i];
#pragma unroll
  for (int k = 1; k < 8; k++)
    if (k < nterms) v += t.c[k][f] * t.x[k][i];
  out[i] = v;
}

// out = c0 x0 + c1 x1 + c2 x2 + c3 x3 with per-sample fp32 coefficients: the solver algebra of the multi-evaluation samplers
// (Heun's trapezoid update, DPM-Solver++(2M)'s extrapolated update) on the fp32 sampler state, one launch.
__global__ void lincomb4_kernel(float* __restrict__ out, const float* __restrict__ x0, const float* __restrict__ x1,
                                const float* __restrict__ x2, const float* __restrict__ x3, const float* __restrict__ c0,
                                const float* __restrict__ c1, const float* __restrict__ c2, const float* __restrict__ c3,
                                int per_sample, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = (int)(i / per_sample);
  float v = c0[f] * x0[i];
  if (x1) v += c1[f] * x1[i];
  if (x2) v += c2[f] * x2[i];
  if (x3) v += c3[f] * x3[i];
  out[i] = v;
}

__global__ void renoise_blend_kernel(float* __restrict__ lat, const float* __restrict__ init, const float* __restrict__ z,
                                     float alpha, float sigma, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) lat[i] = lat[i] * (1.f - alpha) + (init[i] * sigma + z[i]) * alpha;
}

// NCHW -> NHWC(fp16, Cpad) through a shared-memory transpose tile: 32 pixels x all channels per CTA
template <typename TI>
__global__ void __launch_bounds__(256)
nchw_to_nhwc_kernel(const TI* __restrict__ in, int C, int HW, int Cpad, float scale, __half* __restrict__ out) {
  extern __shared__ __half tile[];   // [32][Cpad + 2]
  const int pitch = Cpad + 2;
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int c = ty; c < Cpad; c += 8) {
    float v = 0.f;
    if (c < C && p0 + tx < HW) v = (float)in[((long long)n * C + c) * HW + p0 + tx] * scale;
    tile[tx * pitch + c] = __float2half_rn(v);
  }
  __syncthreads();
  const int total = 32 * Cpad;
  for (int i = threadIdx.x; i < total; i += 256) {
    const int p = i / Cpad, c = i - p * Cpad;
    if (p0 + p < HW) out[((long long)n * HW + p0 + p) * Cpad + c] = tile[p * pitch + c];
  }
}

template <typename TO>
__global__ void __launch_bounds__(256)
nhwc_to_nchw_kernel(const __half* __restrict__ in, int in_ld, int C, int HW, float scale, TO* __restrict__ out) {
  extern __shared__ __half tile[];   // [32][C + 2]
  const int pitch = C + 2;
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * 32;
  const int total = 32 * C;
  for (int i = threadIdx.x; i < total; i += 256) {
    const int p = i / C, c = i - p * C;
    tile[p * pitch + c] = (p0 + p < HW) ? in[((long long)n * HW + p0 + p) * in_ld + c] : __float2half(0.f);
  }
  __syncthreads();
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int c = ty; c < C; c += 8)
    if (p0 + tx < HW) out[((long long)n * C + c) * HW + p0 + tx] = (TO)(__half2float(tile[tx * pitch + c]) * scale);
}

__global__ void gaussian_sample_kernel(const __half* __restrict__ mom, int ld, const float* __restrict__ noise, int C,
                                       int HW, float scale, float* __restrict__ out, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over (n, c, pix) NCHW
  if (idx >= total) return;
  const int pix = (int)(idx % HW);
  const long long nc = idx / HW;
  const int c = (int)(nc % C);
  const long long n = nc / C;
  const __half* m = mom + (n * HW + pix) * ld;
  float v = __half2float(m[c]);
  if (noise) {
    float lv = __half2float(m[C + c]);
    lv = fminf(fmaxf(lv, -30.f), 20.f);
    v += expf(0.5f * lv) * noise[idx];
  }
  out[idx] = v * scale;
}


// ---- one-time weight packing (the C-ABI twin of hi3d_official_b200/pack.py) ---------------------------------------
// src: (Co, Ci, taps) row-major -- nn.Linear [Co, Ci] (taps 1), Conv2d OIHW (taps kh*kw), Conv3d (Co, Ci, 3, 1, 1) (taps 3).
// dst: fp16 [cout_pad, taps * cin_pad] with K ordered (tap, ci) = the segment order of the implicit-GEMM engine;
// geglu: destination rows interleave (value_j, gate_j) of the [value ; gate] row blocks (attention.py:87-94).
HI3D_DEVINL float to_float(float v) { return v; }
HI3D_DEVINL float to_float(__half v) { return __half2float(v); }

template <typename T>
__global__ void pack_weight_kernel(const T* __restrict__ w, int Co, int Ci, int taps, int cin_pad, int cout_pad, int geglu,
                                   __half* __restrict__ out, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int K = taps * cin_pad;
  const int n = (int)(idx / K), rem = (int)(idx - (long long)n * K);
  const int t = rem / cin_pad, ci = rem - t * cin_pad;
  int sn = n;
  if (geglu) sn = (n & 1) ? (Co >> 1) + (n >> 1) : (n >> 1);
  float v = 0.f;
  // rows >= Co are padding (zeros) also in the interleaved GEGLU order
  if (n < Co && sn < Co && ci < Ci) v = to_float(w[((long long)sn * Ci + ci) * taps + t]);
  out[idx] = __float2half_rn(v);
}
template <typename T>
__global__ void pack_bias_kernel(const T* __restrict__ b, int n, int n_pad, int geglu, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad) return;
  int si = i;
  if (geglu) si = (i & 1) ? (n >> 1) + (i >> 1) : (i >> 1);
  out[i] = (b != nullptr && i < n && si < n) ? to_float(b[si]) : 0.f;
}

}  // namespace hi3d

using namespace hi3d;

extern "C" int hi3d_timestep_embedding(const float* t, int n, int dim, float max_period, void* out, void* stream) {
  if (!t || !out || n <= 0 || dim < 2) { set_error("hi3d_timestep_embedding: bad arguments"); return -2; }
  const int half = dim / 2;
  const int total = n * half;
  timestep_embedding_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(t, n, dim, -logf(max_period) / (float)half,
                                                                                 (__half*)out);
  return check_launch("hi3d_timestep_embedding");
}

extern "C" int hi3d_sampler_pre(const float* x, const float* sigma, const void* concat_uc, const void* concat_c,
                                int concat_is_fp32, int F, int Cx, int Cc, int H, int W, int Cpad, void* out,
                                float* c_noise_out, void* stream) {
  if (!x || !sigma || !out || F <= 0 || Cx <= 0 || Cc < 0 || H <= 0 || W <= 0 || (Cpad % 8) || Cpad < Cx + Cc ||
      ((uintptr_t)out & 15) || (Cc > 0 && !concat_c)) {
    set_error("hi3d_sampler_pre: bad arguments (F=%d Cx=%d Cc=%d Cpad=%d)", F, Cx, Cc, Cpad);
    return -2;
  }
  const long long total = (long long)2 * F * H * W;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (concat_is_fp32)
    sampler_pre_kernel<float><<<blocks, 256, 0, (cudaStream_t)stream>>>(x, sigma, (const float*)concat_uc,
                                                                       (const float*)concat_c, F, Cx, Cc, H * W, Cpad,
                                                                       (__half*)out, c_noise_out);
  else
    sampler_pre_kernel<__half><<<blocks, 256, 0, (cudaStream_t)stream>>>(x, sigma, (const __half*)concat_uc,
                                                                        (const __half*)concat_c, F, Cx, Cc, H * W, Cpad,
                                                                        (__half*)out, c_noise_out);
  return check_launch("hi3d_sampler_pre");
}

extern "C" int hi3d_sampler_post(const void* net, int net_ld, const float* x, const float* sigma, const float* sigma_next,
                                 const float* scale, int T, int F, int Cx, int H, int W, float* x_out,
                                 float* denoised_out, void* stream) {
  if (!net || !x || !sigma || !sigma_next || !scale || !x_out || T <= 0 || F <= 0 || Cx <= 0 || net_ld < Cx) {
    set_error("hi3d_sampler_post: bad arguments");
    return -2;
  }
  const long long total = (long long)F * H * W;
  sampler_post_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)net, net_ld, x, sigma, sigma_next, scale, T, F, Cx, H * W, x_out, denoised_out);
  return check_launch("hi3d_sampler_post");
}

extern "C" int hi3d_sampler_lincomb4(float* out, const float* x0, const float* x1, const float* x2, const float* x3,
                                     const float* c0, const float* c1, const float* c2, const float* c3, int F,
                                     int64_t per_sample, void* stream) {
  if (!out || !x0 || !c0 || F <= 0 || per_sample <= 0 || per_sample > 2147483647LL || (x1 && !c1) || (x2 && !c2) || (x3 && !c3)) {
    set_error("hi3d_sampler_lincomb4: bad arguments");
    return -2;
  }
  const long long n = (long long)F * per_sample;
  lincomb4_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(out, x0, x1, x2, x3, c0, c1, c2, c3,
                                                                                (int)per_sample, n);
  return check_launch("hi3d_sampler_lincomb4");
}

extern "C" int hi3d_sampler_pre_ex(const float* x, const float* sigma, const float* sigma_from, const float* eps,
                                   float s_noise, const void* concat_uc, const void* concat_c, int concat_is_fp32, int guided,
                                   int F, int Cx, int Cc, int H, int W, int Cpad, void* out, float* c_noise_out,
                                   float* x_hat_out, void* stream) {
  if (!x || !sigma || !out || F <= 0 || Cx <= 0 || Cc < 0 || H <= 0 || W <= 0 || (Cpad % 8) || Cpad < Cx + Cc ||
      ((uintptr_t)out & 15) || (Cc > 0 && !concat_c) || (guided != 0 && guided != 1) ||
      (eps && (!sigma_from || !x_hat_out))) {
    set_error("hi3d_sampler_pre_ex: bad arguments (F=%d Cx=%d Cc=%d Cpad=%d guided=%d)", F, Cx, Cc, Cpad, guided);
    return -2;
  }
  const int rows = guided ? 2 : 1;
  const long long total = (long long)rows * F * H * W;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (concat_is_fp32)
    sampler_pre_ex_kernel<float><<<blocks, 256, 0, (cudaStream_t)stream>>>(
        x, sigma, sigma_from, eps, s_noise, (const float*)concat_uc, (const float*)concat_c, rows, F, Cx, Cc, H * W, Cpad,
        (__half*)out, c_noise_out, x_hat_out);
  else
    sampler_pre_ex_kernel<__half><<<blocks, 256, 0, (cudaStream_t)stream>>>(
        x, sigma, sigma_from, eps, s_noise, (const __half*)concat_uc, (const __half*)concat_c, rows, F, Cx, Cc, H * W, Cpad,
        (__half*)out, c_noise_out, x_hat_out);
  return check_launch("hi3d_sampler_pre_ex");
}

extern "C" int hi3d_sampler_post_ancestral(const void* net, int net_ld, const float* x, const float* sigma,
                                           const float* sigma_to, const float* scale, int T, const float* eps, float s_noise,
                                           const float* sigma_up, const float* sigma_next, int F, int Cx, int H, int W,
                                           float* x_out, float* denoised_out, void* stream) {
  if (!net || !x || !sigma || !sigma_to || !x_out || F <= 0 || Cx <= 0 || H <= 0 || W <= 0 || net_ld < Cx ||
      (scale && T <= 0) || (eps && (!sigma_up || !sigma_next))) {
    set_error("hi3d_sampler_post_ancestral: bad arguments (F=%d Cx=%d net_ld=%d T=%d)", F, Cx, net_ld, T);
    return -2;
  }
  const long long total = (long long)F * H * W;
  sampler_post_ancestral_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)net, net_ld, x, sigma, sigma_to, scale, T, eps, s_noise, sigma_up, sigma_next, F, Cx, H * W, x_out,
      denoised_out);
  return check_launch("hi3d_sampler_post_ancestral");
}

extern "C" int hi3d_sampler_lincomb(float* out, const float* const* xs, const float* const* cs, int nterms, int F,
                                    int64_t per_sample, void* stream) {
  bool ok = out && xs && cs && nterms >= 1 && nterms <= 8 && F > 0 && per_sample > 0 && per_sample <= 2147483647LL;
  LincombTerms t = {};
  for (int k = 0; ok && k < nterms; k++) {
    ok = xs[k] && cs[k];
    t.x[k] = xs[k];
    t.c[k] = cs[k];
  }
  if (!ok) {
    set_error("hi3d_sampler_lincomb: bad arguments (nterms=%d F=%d)", nterms, F);
    return -2;
  }
  const long long n = (long long)F * per_sample;
  lincomb_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(out, t, nterms, (int)per_sample, n);
  return check_launch("hi3d_sampler_lincomb");
}

extern "C" int hi3d_renoise_blend(float* lat, const float* init, const float* z, float alpha, float sigma, int64_t n,
                                  void* stream) {
  if (!lat || !init || !z || n <= 0) { set_error("hi3d_renoise_blend: bad arguments"); return -2; }
  renoise_blend_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(lat, init, z, alpha, sigma, n);
  return check_launch("hi3d_renoise_blend");
}

// One thread per 8 output columns of one patch row (a 16-byte store); row 0 of each image is the zero class-token slot.
template <typename TI>
__global__ void clip_patchify_kernel(const TI* __restrict__ img, int n, int H, int W, int patch, int normalize, int Kpad,
                                     __half* __restrict__ out) {
  const int Gx = W / patch, P = (H / patch) * Gx;
  const int cpr = Kpad / 8, K = 3 * patch * patch, pp = patch * patch;
  const long long total = (long long)n * (1 + P) * cpr;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const long long row = idx / cpr;
  const int k0 = (int)(idx - row * cpr) * 8;
  const int im = (int)(row / (1 + P)), t = (int)(row - (long long)im * (1 + P));
  const float mean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
  const float istd[3] = {1.f / 0.26862954f, 1.f / 0.26130258f, 1.f / 0.27577711f};
  Half8 v;
#pragma unroll
  for (int e = 0; e < 8; e += 2) {
    float a[2];
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int k = k0 + e + u;
      float val = 0.f;
      if (t > 0 && k < K) {
        const int c = k / pp, r = k - c * pp, ky = r / patch, kx = r - ky * patch;
        const int py = (t - 1) / Gx, px = (t - 1) - py * Gx;
        val = (float)img[(((long long)im * 3 + c) * H + py * patch + ky) * W + px * patch + kx];
        if (normalize) val = (val - mean[c]) * istd[c];
      }
      a[u] = val;
    }
    v.h[e / 2] = __floats2half2_rn(a[0], a[1]);
  }
  *reinterpret_cast<Half8*>(out + row * Kpad + k0) = v;
}

extern "C" int hi3d_clip_patchify(const void* img, int img_is_fp32, int n, int H, int W, int patch, int normalize, int Kpad,
                                  void* out, void* stream) {
  if (!img || !out || n <= 0 || patch <= 0 || H < patch || W < patch || H % patch || W % patch || Kpad % 8 ||
      Kpad < 3 * patch * patch || ((uintptr_t)out & 15)) {
    set_error("hi3d_clip_patchify: bad arguments (n=%d H=%d W=%d patch=%d Kpad=%d)", n, H, W, patch, Kpad);
    return -2;
  }
  const long long total = (long long)n * (1 + (H / patch) * (W / patch)) * (Kpad / 8);
  const int grid = (int)((total + 255) / 256);
  if (img_is_fp32)
    clip_patchify_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)img, n, H, W, patch, normalize, Kpad,
                                                                      (__half*)out);
  else
    clip_patchify_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)img, n, H, W, patch, normalize, Kpad,
                                                                       (__half*)out);
  return check_launch("hi3d_clip_patchify");
}

extern "C" int hi3d_nchw_to_nhwc(const void* in, int in_is_fp32, int N, int C, int H, int W, int Cpad, float scale,
                                 void* out, void* stream) {
  if (!in || !out || N <= 0 || C <= 0 || Cpad < C || (Cpad % 8) || Cpad > 512 || N > 65535) {
    set_error("hi3d_nchw_to_nhwc: bad arguments (N=%d C=%d Cpad=%d)", N, C, Cpad);
    return -2;
  }
  const int HW = H * W;
  dim3 grid((HW + 31) / 32, N);
  const size_t sm = (size_t)32 * (Cpad + 2) * sizeof(__half);
  if (in_is_fp32)
    nchw_to_nhwc_kernel<float><<<grid, 256, sm, (cudaStream_t)stream>>>((const float*)in, C, HW, Cpad, scale, (__half*)out);
  else
    nchw_to_nhwc_kernel<__half><<<grid, 256, sm, (cudaStream_t)stream>>>((const __half*)in, C, HW, Cpad, scale,
                                                                        (__half*)out);
  return check_launch("hi3d_nchw_to_nhwc");
}

extern "C" int hi3d_nhwc_to_nchw(const void* in, int in_ld, int N, int C, int H, int W, float scale, void* out,
                                 int out_is_fp32, void* stream) {
  if (!in || !out || N <= 0 || C <= 0 || in_ld < C || C > 512 || N > 65535) {
    set_error("hi3d_nhwc_to_nchw: bad arguments");
    return -2;
  }
  const int HW = H * W;
  dim3 grid((HW + 31) / 32, N);
  const size_t sm = (size_t)32 * (C + 2) * sizeof(__half);
  if (out_is_fp32)
    nhwc_to_nchw_kernel<float><<<grid, 256, sm, (cudaStream_t)stream>>>((const __half*)in, in_ld, C, HW, scale, (float*)out);
  else
    nhwc_to_nchw_kernel<__half><<<grid, 256, sm, (cudaStream_t)stream>>>((const __half*)in, in_ld, C, HW, scale,
                                                                        (__half*)out);
  return check_launch("hi3d_nhwc_to_nchw");
}

extern "C" int hi3d_gaussian_sample(const void* moments, int ld, const float* noise, int N, int C, int H, int W,
                                    float scale, float* out, void* stream) {
  if (!moments || !out || N <= 0 || C <= 0 || ld < 2 * C) { set_error("hi3d_gaussian_sample: bad arguments"); return -2; }
  const long long total = (long long)N * C * H * W;
  gaussian_sample_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const __half*)moments, ld,
                                                                                          noise, C, H * W, scale, out,
                                                                                          total);
  return check_launch("hi3d_gaussian_sample");
}

extern "C" int hi3d_pack_weight(const void* w, int w_is_fp32, int Co, int Ci, int taps, int cin_pad, int cout_pad,
                                int geglu_interleave, void* out, void* stream) {
  if (!w || !out || Co <= 0 || Ci <= 0 || taps <= 0 || cin_pad < Ci || cout_pad < Co || (geglu_interleave && (Co & 1))) {
    set_error("hi3d_pack_weight: bad arguments (Co=%d Ci=%d taps=%d cin_pad=%d cout_pad=%d)", Co, Ci, taps, cin_pad, cout_pad);
    return -2;
  }
  const long long total = (long long)cout_pad * taps * cin_pad;
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (w_is_fp32)
    pack_weight_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)w, Co, Ci, taps, cin_pad, cout_pad,
                                                                     geglu_interleave, (__half*)out, total);
  else
    pack_weight_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)w, Co, Ci, taps, cin_pad, cout_pad,
                                                                      geglu_interleave, (__half*)out, total);
  return check_launch("hi3d_pack_weight");
}

extern "C" int hi3d_pack_bias(const void* b, int b_is_fp32, int n, int n_pad, int geglu_interleave, float* out,
                              void* stream) {
  if (!out || n <= 0 || n_pad < n || (geglu_interleave && (n & 1))) {
    set_error("hi3d_pack_bias: bad arguments (n=%d n_pad=%d)", n, n_pad);
    return -2;
  }
  const unsigned grid = (unsigned)((n_pad + 255) / 256);
  if (b_is_fp32)
    pack_bias_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)b, n, n_pad, geglu_interleave, out);
  else
    pack_bias_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)b, n, n_pad, geglu_interleave, out);
  return check_launch("hi3d_pack_bias");
}
