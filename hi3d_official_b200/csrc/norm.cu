// GroupNorm(32) [+SiLU] and LayerNorm for channels-last fp16 activations.  Statistics in fp32 (final
// combine in fp64), matching the reference's fp32 GroupNorm32 / autocast-fp32 LayerNorm (SURVEY App. E).
// Both are pure HBM streams: every thread owns fixed 16-byte channel columns, keeps its per-channel
// constants in registers and walks rows with several independent 16-byte loads in flight; grids are sized to a
// few full waves of the 132 SMs.
#include "common.cuh"

namespace hi3d {

constexpr int GN_GROUPS = 32;
constexpr int GN_UNROLL = 4;

HI3D_DEVINL Half8 ld_stream(const __half* p) {
  Half8 v;
  uint4 u;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
               : "l"(p));
  *reinterpret_cast<uint4*>(&v) = u;
  return v;
}

// ---- GroupNorm apply: y = [silu]((x - mean) * rstd * gamma + beta) ----------------------------------
// grid (row_slabs, n_samples), blockDim = RL * CV.  Statistics: the unit tables stats1 / stats2 when stats1 != NULL, else the
// per-(sample, group) sums `fin` over `count` elements.
template <bool HALO,      // HALO = haloed output with peer stores / boundary zero fill (frame-sharded temporal GroupNorm only):
                          // a template so that the dense kernel keeps its 64 registers (2 CTAs per SM)
          bool OUT8>      // OUT8 = dense e4m3 output: each fp16 result the fp16 kernel would store, converted by half8_to_e4m3
__global__ void __launch_bounds__(512)
gn_apply_kernel(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2, long long rows_per_sample,
                long long rows_per_cta, const float* __restrict__ fin, double count, float eps,
                const float* __restrict__ gamma, const float* __restrict__ beta, int apply_silu, __half* __restrict__ y,
                long long y_sample_rows, long long y_row_off, __half* __restrict__ y_prev, __half* __restrict__ y_next,
                long long frame_rows, int zero_lead, int zero_trail, const float* __restrict__ stats1,
                const float* __restrict__ stats2, int unit, int ips) {
  __shared__ float smean[GN_GROUPS], srstd[GN_GROUPS];
  __shared__ float ssum[GN_GROUPS * 2];
  const int C = C1 + C2, CV = C >> 3, cpg = C / GN_GROUPS;
  const int tid = threadIdx.x, n = blockIdx.y;
  if (stats1 != nullptr) {
    // statistics from the unit tables hi3d_groupnorm_unit_stats accumulated over the inputs: group g of
    // sample n = units [g cpg / unit, (g+1) cpg / unit) of the channel concat, over the `ips` images of the sample.
    // 64 threads, one per (group, sum | sumsq), each adding its <= ips * upg table entries in registers (independent loads).
    if (tid < GN_GROUPS * 2) {
      const int g = tid >> 1, which = tid & 1;
      const int upg = cpg / unit, u1 = C1 / unit, u2 = C2 / unit;
      float acc = 0.f;
      for (int img = 0; img < ips; img++) {
        const long long im = (long long)n * ips + img;
        for (int uu = 0; uu < upg; uu++) {
          const int u = g * upg + uu;
          acc += (u < u1) ? __ldg(stats1 + (im * u1 + u) * 2 + which) : __ldg(stats2 + (im * u2 + (u - u1)) * 2 + which);
        }
      }
      ssum[tid] = acc;
    }
    __syncthreads();
    fin = ssum - (long long)n * (GN_GROUPS * 2);                   // so that the indexing below reads ssum[...]
  }
  if (tid < GN_GROUPS) {      // `count` = elements per (sample, group) over ALL ranks
    const double mean = (double)fin[(long long)n * (GN_GROUPS * 2) + 2 * tid] / count;
    double var = (double)fin[(long long)n * (GN_GROUPS * 2) + 2 * tid + 1] / count - mean * mean;
    if (var < 0.0) var = 0.0;
    smean[tid] = (float)mean;
    srstd[tid] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
  const int cv = tid % CV, rl = tid / CV, RL = blockDim.x / CV;
  const int c0 = cv * 8;
  float A[8], B[8];
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const int c = c0 + e, g = c / cpg;
    A[e] = srstd[g] * gamma[c];
    B[e] = beta[c] - smean[g] * A[e];
  }
  const __half* base;
  int ld;
  if (c0 < C1) { base = x1 + c0; ld = C1; } else { base = x2 + (c0 - C1); ld = C2; }
  const long long srow0 = (long long)n * rows_per_sample;
  base += srow0 * ld;
  __half* yb = y + ((long long)n * y_sample_rows + y_row_off) * C + c0;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  long long r1 = r0 + rows_per_cta;
  if (r1 > rows_per_sample) r1 = rows_per_sample;
  // (A variant with one shared reciprocal per four sigmoids -- 1.25 MUFU operations per element instead of 2 -- was measured
  // SLOWER: 128 us vs 76 us per launch in the ncu launch list of profiles/r02_*: the kernel is latency-bound at ~50 % issue /
  // MUFU / DRAM utilisation, and the extra multiplies plus the register squeeze cost more than the MUFU slots they free.)
  auto xform = [&](Half8 v) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      float2 f = __half22float2(v.h[k]);
      f.x = f.x * A[2 * k] + B[2 * k];
      f.y = f.y * A[2 * k + 1] + B[2 * k + 1];
      if (apply_silu) { f.x = silu_f(f.x); f.y = silu_f(f.y); }
      v.h[k] = __floats2half2_rn(f.x, f.y);
    }
    return v;
  };
  // Frame-sharded temporal GroupNorm (SURVEY 8e): y is a haloed [n, T_local + 2, frame_rows, C] buffer.  The first local
  // frame is ALSO stored into the trailing halo slot of the previous rank's buffer and the last local frame into the leading
  // halo slot of the next rank's (peer stores over NVLink): the one-frame halo exchange of the (3,1,1) conv rides on this
  // kernel's stores.  y_prev / y_next are the peers' buffer bases (NULL at the clip boundary: that slot stays zero = padding).
  const long long last0 = rows_per_sample - frame_rows;
  __half* yp = (HALO && y_prev) ? y_prev + ((long long)n * y_sample_rows + (y_sample_rows - frame_rows)) * C + c0 : nullptr;
  __half* yn = (HALO && y_next) ? y_next + ((long long)n * y_sample_rows - last0) * C + c0 : nullptr;
  // At a clip boundary (no previous / next rank) the halo slot of THIS rank is the Conv3d zero padding: the buffer is
  // shared by layers of different geometry, so it is re-zeroed here by the threads that own the matching boundary frame.
  __half* zl = (HALO && zero_lead) ? y + ((long long)n * y_sample_rows) * C + c0 : nullptr;                     // slot 0
  __half* zt = (HALO && zero_trail) ? y + ((long long)n * y_sample_rows + (y_sample_rows - frame_rows) - last0) * C + c0 : nullptr;
  Half8 zero8;
  zero8.u = make_uint4(0u, 0u, 0u, 0u);
  bool remote = false;
  uint8_t* yb8 = reinterpret_cast<uint8_t*>(y) + ((long long)n * y_sample_rows + y_row_off) * C + c0;
  auto put = [&](long long rr, const Half8& o) {
    if constexpr (OUT8) {
      *reinterpret_cast<uint2*>(yb8 + rr * C) = half8_to_e4m3(o);
      return;
    }
    *reinterpret_cast<Half8*>(yb + rr * C) = o;
    if (!HALO) return;
    if (rr < frame_rows) {
      if (yp != nullptr) { *reinterpret_cast<Half8*>(yp + rr * C) = o; remote = true; }
      if (zl != nullptr) *reinterpret_cast<Half8*>(zl + rr * C) = zero8;
    }
    if (rr >= last0) {
      if (yn != nullptr) { *reinterpret_cast<Half8*>(yn + rr * C) = o; remote = true; }
      if (zt != nullptr) *reinterpret_cast<Half8*>(zt + rr * C) = zero8;
    }
  };
  long long r = r0 + rl;
  for (; r + (long long)(GN_UNROLL - 1) * RL < r1; r += (long long)GN_UNROLL * RL) {
    Half8 v[GN_UNROLL];
#pragma unroll
    for (int u = 0; u < GN_UNROLL; u++) v[u] = ld_stream(base + (r + (long long)u * RL) * ld);
#pragma unroll
    for (int u = 0; u < GN_UNROLL; u++) put(r + (long long)u * RL, xform(v[u]));
  }
  for (; r < r1; r += RL) put(r, xform(ld_stream(base + r * ld)));
  if (remote) __threadfence_system();
}

// ---- LayerNorm: LPR lanes per row (32/LPR rows per warp pass), VPL 16-byte vectors per lane ------------------
// C = 8 * VPL * LPR exactly (C = 320 -> VPL 5, LPR 8; 640 -> 5 x 16; 1280 -> 5 x 32; 64 -> 1 x 8; 2560 -> 10 x 32).
// OUT8: y is e4m3, each fp16 result the fp16 kernel would store converted by half8_to_e4m3 (both LayerNorm kernels).
template <int VPL, int LPR, bool OUT8>
__global__ void __launch_bounds__(256)
layernorm_kernel(const __half* __restrict__ x, const __half* __restrict__ addvec, int add_div, int add_mod, long long M,
                 int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                 __half* __restrict__ y) {
  constexpr int RPW = 32 / LPR;                      // rows per warp pass
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR, rsel = lane / LPR;
  const long long wrow0 = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * RPW;
  const long long m = wrow0 + rsel;
  const bool live = m < M;
  const float invC = 1.f / (float)C;
  Half8 raw[VPL];
  if (live) {
#pragma unroll
    for (int i = 0; i < VPL; i++) raw[i] = ld_stream(x + m * C + (sub + LPR * i) * 8);
  }
  float v[VPL][8];
  float sum = 0.f;
  if (live) {
    const __half* av = addvec ? addvec + (long long)((m / add_div) % add_mod) * C : nullptr;
#pragma unroll
    for (int i = 0; i < VPL; i++) {
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const float2 f = __half22float2(raw[i].h[k]);
        v[i][2 * k] = f.x; v[i][2 * k + 1] = f.y;
      }
      if (av) {
        const Half8 a = *reinterpret_cast<const Half8*>(av + (sub + LPR * i) * 8);
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const float2 f = __half22float2(a.h[k]);
          v[i][2 * k] += f.x; v[i][2 * k + 1] += f.y;
        }
      }
#pragma unroll
      for (int e = 0; e < 8; e++) sum += v[i][e];
    }
  } else {
#pragma unroll
    for (int i = 0; i < VPL; i++)
#pragma unroll
      for (int e = 0; e < 8; e++) v[i][e] = 0.f;
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum * invC;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; i++)
#pragma unroll
    for (int e = 0; e < 8; e++) { const float d = v[i][e] - mean; sq += d * d; }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq * invC + eps);
  if (live) {
#pragma unroll
    for (int i = 0; i < VPL; i++) {
      const int c0 = (sub + LPR * i) * 8;
      Half8 o;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const float2 gm = *reinterpret_cast<const float2*>(gamma + c0 + 2 * k);
        const float2 bt = *reinterpret_cast<const float2*>(beta + c0 + 2 * k);
        o.h[k] = __floats2half2_rn((v[i][2 * k] - mean) * rstd * gm.x + bt.x, (v[i][2 * k + 1] - mean) * rstd * gm.y + bt.y);
      }
      if constexpr (OUT8) *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(y) + m * C + c0) = half8_to_e4m3(o);
      else *reinterpret_cast<Half8*>(y + m * C + c0) = o;
    }
  }
}

// generic fallback: one warp per row, up to 10 vectors per lane with masking (any C % 8 == 0, C <= 2560)
template <int VPL, bool OUT8>
__global__ void __launch_bounds__(256)
layernorm_generic_kernel(const __half* __restrict__ x, const __half* __restrict__ addvec, int add_div, int add_mod,
                         long long M, int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                         __half* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const long long m = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (m >= M) return;
  const int CV = C >> 3;
  const __half* av = addvec ? addvec + (long long)((m / add_div) % add_mod) * C : nullptr;
  float v[VPL][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; i++) {
    const int cv = lane + 32 * i;
#pragma unroll
    for (int e = 0; e < 8; e++) v[i][e] = 0.f;
    if (cv < CV) {
      const Half8 h = ld_stream(x + m * C + cv * 8);
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const float2 f = __half22float2(h.h[k]);
        v[i][2 * k] = f.x; v[i][2 * k + 1] = f.y;
      }
      if (av) {
        const Half8 a = *reinterpret_cast<const Half8*>(av + cv * 8);
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const float2 f = __half22float2(a.h[k]);
          v[i][2 * k] += f.x; v[i][2 * k + 1] += f.y;
        }
      }
#pragma unroll
      for (int e = 0; e < 8; e++) sum += v[i][e];
    }
  }
  const float mean = warp_sum(sum) / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; i++)
    if (lane + 32 * i < CV) {
#pragma unroll
      for (int e = 0; e < 8; e++) { const float d = v[i][e] - mean; sq += d * d; }
    }
  const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < VPL; i++) {
    const int cv = lane + 32 * i;
    if (cv < CV) {
      Half8 o;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int c = cv * 8 + 2 * k;
        o.h[k] = __floats2half2_rn((v[i][2 * k] - mean) * rstd * gamma[c] + beta[c],
                                   (v[i][2 * k + 1] - mean) * rstd * gamma[c + 1] + beta[c + 1]);
      }
      if constexpr (OUT8) *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(y) + m * C + cv * 8) = half8_to_e4m3(o);
      else *reinterpret_cast<Half8*>(y + m * C + cv * 8) = o;
    }
  }
}

}  // namespace hi3d

using namespace hi3d;

static int gn_check(const void* x1, int C1, const void* x2, int C2, int n_samples, int64_t rows_per_sample, const char* who) {
  const int C = C1 + C2;
  if (!x1 || n_samples <= 0 || rows_per_sample <= 0 || C1 <= 0 || (C1 % 8) || (C2 % 8) || (C % GN_GROUPS) || C > 4096 ||
      ((uintptr_t)x1 & 15) || (x2 && ((uintptr_t)x2 & 15)) || n_samples > 65535) {
    set_error("%s: bad arguments (C1=%d C2=%d n=%d rows=%lld)", who, C1, C2, n_samples, (long long)rows_per_sample);
    return -2;
  }
  return 0;
}

// The one launcher of gn_apply_kernel.  Statistics come from exactly one source: the unit tables stats1 / stats2 (`unit`
// channels per entry, `ips` images per sample) when stats1 != NULL, else `sums` [n_samples][32][2].  Either way they cover
// `count_rows` rows per sample: rows_per_sample on one GPU, the GLOBAL row count when the sums were all-reduced over ranks.
// Sample n of y starts at row n * y_sample_rows + y_row_off (haloed temporal buffers); 0, 0 -> dense like x.
// frame_rows > 0 selects the haloed form: a NULL neighbour then means "clip boundary", whose local halo slot is zero-filled.
static int gn_apply_launch(const char* who, const void* x1, int C1, const void* x2, int C2, int n_samples,
                           int64_t rows_per_sample, const float* sums, const float* stats1, const float* stats2, int unit, int ips,
                           int64_t count_rows, const float* gamma, const float* beta, float eps, int apply_silu, void* y,
                           int64_t y_sample_rows, int64_t y_row_off, void* y_prev_rank, void* y_next_rank, int64_t frame_rows,
                           void* stream, bool out8 = false) {
  int rc = gn_check(x1, C1, x2, C2, n_samples, rows_per_sample, who);
  if (rc) return rc;
  if ((y_prev_rank || y_next_rank || frame_rows > 0) &&
      (frame_rows <= 0 || rows_per_sample % frame_rows || y_sample_rows != rows_per_sample + 2 * frame_rows ||
       y_row_off != frame_rows || ((uintptr_t)y_prev_rank & 15) || ((uintptr_t)y_next_rank & 15))) {
    set_error("%s: the peer halo stores need y = [n, T_local + 2, frame_rows, C] with y_row_off = frame_rows (rows %lld, "
              "frame_rows %lld, y_sample_rows %lld, y_row_off %lld)", who, (long long)rows_per_sample, (long long)frame_rows,
              (long long)y_sample_rows, (long long)y_row_off);
    return -2;
  }
  if ((!sums && !stats1) || !gamma || !beta || !y || ((uintptr_t)y & 15) || count_rows <= 0) {
    set_error("%s: bad arguments", who);
    return -2;
  }
  if (y_sample_rows <= 0) { y_sample_rows = rows_per_sample; y_row_off = 0; }
  cudaStream_t st = (cudaStream_t)stream;
  const int C = C1 + C2, CV = C / 8;
  const int threads = (512 / CV) * CV;
  const int RL = threads / CV;
  const long long min_rows = (long long)RL * GN_UNROLL;
  const long long max_by_rows = (rows_per_sample + min_rows - 1) / min_rows;
  // 2 CTAs per SM x 3 waves: a CTA lives ~4x longer than with the statistics kernels' grid, so its prologue (group statistics
  // -> mean / rstd -> 16 coefficient registers) is amortised; measured 120 -> see profiles/r02 launch lists
  long long slabs = (132 * 2 * 3 + n_samples - 1) / n_samples;
  if (slabs > max_by_rows) slabs = max_by_rows;
  if (slabs < 1) slabs = 1;
  long long rows_per_cta = (rows_per_sample + slabs - 1) / slabs;
  rows_per_cta = (rows_per_cta + RL - 1) / RL * RL;
  slabs = (rows_per_sample + rows_per_cta - 1) / rows_per_cta;
  if (slabs > 2147483647LL) { set_error("%s: too many slabs", who); return -2; }
  if (frame_rows > 0)
    gn_apply_kernel<true, false><<<dim3((unsigned)slabs, n_samples), threads, 0, st>>>(
        (const __half*)x1, C1, (const __half*)x2, C2, rows_per_sample, rows_per_cta, sums,
        (double)count_rows * (double)(C / GN_GROUPS), eps, gamma, beta, apply_silu, (__half*)y, y_sample_rows, y_row_off,
        (__half*)y_prev_rank, (__half*)y_next_rank, frame_rows, !y_prev_rank ? 1 : 0, !y_next_rank ? 1 : 0, stats1, stats2,
        unit, ips);
  else if (out8)
    gn_apply_kernel<false, true><<<dim3((unsigned)slabs, n_samples), threads, 0, st>>>(
        (const __half*)x1, C1, (const __half*)x2, C2, rows_per_sample, rows_per_cta, sums,
        (double)count_rows * (double)(C / GN_GROUPS), eps, gamma, beta, apply_silu, (__half*)y, y_sample_rows, y_row_off,
        nullptr, nullptr, 0, 0, 0, stats1, stats2, unit, ips);
  else
    gn_apply_kernel<false, false><<<dim3((unsigned)slabs, n_samples), threads, 0, st>>>(
        (const __half*)x1, C1, (const __half*)x2, C2, rows_per_sample, rows_per_cta, sums,
        (double)count_rows * (double)(C / GN_GROUPS), eps, gamma, beta, apply_silu, (__half*)y, y_sample_rows, y_row_off,
        nullptr, nullptr, 0, 0, 0, stats1, stats2, unit, ips);
  return check_launch(who);
}

extern "C" int hi3d_groupnorm_apply_halo(const void* x1, int C1, const void* x2, int C2, int n_samples, int64_t rows_per_sample,
                                         const float* sums, int64_t count_rows, const float* gamma, const float* beta, float eps,
                                         int apply_silu, void* y, int64_t y_sample_rows, int64_t y_row_off, void* y_prev_rank,
                                         void* y_next_rank, int64_t frame_rows, void* stream) {
  if (!x2) C2 = 0;
  return gn_apply_launch("hi3d_groupnorm_apply_halo", x1, C1, x2, C2, n_samples, rows_per_sample, sums, nullptr, nullptr, 0, 1,
                         count_rows, gamma, beta, eps, apply_silu, y, y_sample_rows, y_row_off, y_prev_rank, y_next_rank,
                         frame_rows, stream);
}

// ---- unit statistics of an existing tensor: (sum, sumsq) per image and per `unit` consecutive channels, accumulated -------
// Every sum is taken in a fixed order that depends on (rows_per_image, C, unit) only, never on scheduling or on the other
// images of the launch: the same input gives the same table bits, and an image gives the same bits alone or in any batch.
// Each image is cut into `slices` channel slices (whole units, whole 32-byte sectors) x `ranks` row ranges.  One thread-block
// cluster of `ranks` CTAs owns one (image, slice):
//   1. each thread owns one 16-byte channel column of the slice and walks its rows of the CTA's range in order;
//   2. the CTA folds its row lanes with a fixed pairwise tree in shared memory, then each unit's channels in channel order;
//   3. after a cluster barrier, rank 0 adds the ranks' unit partials in rank order (distributed shared memory) and adds the
//      result to the table: one writer per entry per launch, no atomics.
// The plan (unit_stats_plan) sizes a CTA's share to ~GN_CTA_BYTES, so one large image (the VAE at 1024^2, called one frame at a
// time) still spreads over up to 8 x slices CTAs, each with GN_STATS_UNROLL 16-byte loads in flight per thread.
constexpr int GN_MAX_UNITS = 256;
constexpr int GN_STATS_THREADS = 512;
constexpr int GN_STATS_UNROLL = 8;
constexpr int GN_MAX_RANKS = 8;                       // the portable cluster size
constexpr long long GN_CTA_BYTES = 256 << 10;

HI3D_DEVINL void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

HI3D_DEVINL float ld_cluster_f32(const float* p, unsigned rank) {   // p's counterpart in CTA `rank` of this cluster
  const uint32_t local = (uint32_t)__cvta_generic_to_shared(p);
  uint32_t remote;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(remote) : "r"(local), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];\n" : "=f"(v) : "r"(remote) : "memory");
  return v;
}

// (2 CTAs per SM: without the minimum ptxas sinks each load to its use and only one load per thread is in flight)
__global__ void __launch_bounds__(GN_STATS_THREADS, 2)
gn_unit_stats_kernel(const __half* __restrict__ x, int C, long long rows_per_image, long long rows_per_rank, int slice_c,
                     int unit, float* __restrict__ stats) {
  __shared__ __align__(16) float red[GN_STATS_THREADS * 16];    // [row lane][column][sum 8 | sumsq 8]
  __shared__ float su[GN_MAX_UNITS * 2];                        // this CTA's unit partials of the slice
  unsigned rank;
  asm("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(rank));
  unsigned ranks;
  asm("mov.u32 %0, %%cluster_nctarank;\n" : "=r"(ranks));
  const int tid = threadIdx.x, n = blockIdx.y;
  const int slice = blockIdx.x / ranks;
  const int CVs = slice_c >> 3, cv = tid % CVs, rl = tid / CVs, RL = blockDim.x / CVs;   // blockDim.x == RL * CVs
  const long long r0 = (long long)rank * rows_per_rank;
  long long r1 = r0 + rows_per_rank;
  if (r1 > rows_per_image) r1 = rows_per_image;
  const __half* base = x + (long long)n * rows_per_image * C + slice * slice_c + cv * 8;
  float s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; e++) s[e] = q[e] = 0.f;
  auto add = [&](const Half8& v) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const float2 f = __half22float2(v.h[k]);
      s[2 * k] += f.x; q[2 * k] += f.x * f.x;
      s[2 * k + 1] += f.y; q[2 * k + 1] += f.y * f.y;
    }
  };
  long long r = r0 + rl;
  for (; r + (long long)(GN_STATS_UNROLL - 1) * RL < r1; r += (long long)GN_STATS_UNROLL * RL) {
    Half8 v[GN_STATS_UNROLL];
#pragma unroll
    for (int u = 0; u < GN_STATS_UNROLL; u++) v[u] = ld_stream(base + (r + (long long)u * RL) * C);
#pragma unroll
    for (int u = 0; u < GN_STATS_UNROLL; u++) add(v[u]);
  }
  for (; r < r1; r += RL) add(ld_stream(base + r * C));
  float4* mine = reinterpret_cast<float4*>(red + tid * 16);     // tid = rl * CVs + cv: row lane rl's block is contiguous
  mine[0] = make_float4(s[0], s[1], s[2], s[3]);
  mine[1] = make_float4(s[4], s[5], s[6], s[7]);
  mine[2] = make_float4(q[0], q[1], q[2], q[3]);
  mine[3] = make_float4(q[4], q[5], q[6], q[7]);
  __syncthreads();
  // row lanes: a fixed pairwise tree (lane i += lane i + h while more than one lane is left)
  const int W16 = CVs * 16;
  for (int m = RL; m > 1;) {
    const int h = (m + 1) >> 1, items = (m - h) * W16;
    for (int i = tid; i < items; i += blockDim.x) red[i] += red[i + h * W16];
    __syncthreads();
    m = h;
  }
  // channels -> units, in channel order
  const int nus = slice_c / unit;
  for (int i = tid; i < nus * 2; i += blockDim.x) {      // (a CTA may have fewer threads than 2 x units: C = 2560 has 320)
    const int u = i >> 1, which = i & 1;
    float acc = 0.f;
    for (int k = 0; k < unit; k++) {
      const int c = u * unit + k;
      acc += red[(c >> 3) * 16 + which * 8 + (c & 7)];
    }
    su[i] = acc;
  }
  cluster_sync_all();
  if (rank == 0) {
    for (int i = tid; i < nus * 2; i += blockDim.x) {
      float acc = 0.f;
      for (unsigned k = 0; k < ranks; k++) acc += ld_cluster_f32(su + i, k);
      stats[((long long)n * (C / unit) + (long long)slice * nus) * 2 + i] += acc;
    }
  }
  cluster_sync_all();                                   // the other CTAs' shared memory stays alive until rank 0 has read it
}

// unit tables -> (sum, sumsq) per (sample, group): sums[n][32][2].  One thread per (group, sum | sumsq), adding its entries
// image by image and unit by unit, the loop of gn_apply_kernel's prologue.
__global__ void __launch_bounds__(GN_GROUPS * 2)
gn_group_sums_kernel(const float* __restrict__ stats1, int C1, const float* __restrict__ stats2, int C2, int unit, int ips,
                     float* __restrict__ sums) {
  const int tid = threadIdx.x, n = blockIdx.x;
  const int g = tid >> 1, which = tid & 1;
  const int cpg = (C1 + C2) / GN_GROUPS, upg = cpg / unit, u1 = C1 / unit, u2 = C2 / unit;
  float acc = 0.f;
  for (int img = 0; img < ips; img++) {
    const long long im = (long long)n * ips + img;
    for (int uu = 0; uu < upg; uu++) {
      const int u = g * upg + uu;
      acc += (u < u1) ? __ldg(stats1 + (im * u1 + u) * 2 + which) : __ldg(stats2 + (im * u2 + (u - u1)) * 2 + which);
    }
  }
  sums[(long long)n * (GN_GROUPS * 2) + tid] = acc;
}

// The decomposition of one image for gn_unit_stats_kernel, from (rows_per_image, C, unit) alone.
struct GnStatsPlan {
  int slices, ranks, slice_c, threads;
  long long rows_per_rank;
};

static GnStatsPlan unit_stats_plan(long long rows, int C, int unit) {
  GnStatsPlan p;
  const long long bytes = rows * (long long)C * 2;
  long long want = (bytes + GN_CTA_BYTES - 1) / GN_CTA_BYTES;
  p.ranks = 1;
  while (p.ranks < GN_MAX_RANKS && 2LL * p.ranks <= want && rows >= 64LL * p.ranks) p.ranks *= 2;
  // channel slices: whole units, the fewest that reach `want` CTAs per image.  A slice is at least 64 bytes of a row (32
  // channels); 32-byte slices (16 channels) only while an image has fewer than 64 CTAs (on an H100 80GB HBM3 at 700 W, the
  // VAE's 1024^2 x 256 tensor, one frame per call, streamed at 1.45 TB/s in 32-byte slices and 2.69 TB/s in 64-byte ones)
  p.slices = 1;
  for (int s = 2; (long long)p.slices * p.ranks < want && s <= C / 16; s++)
    if (C % s == 0 && (C / s) % unit == 0 && (C / s) % 16 == 0 && ((C / s) >= 32 || (long long)p.slices * p.ranks < 64))
      p.slices = s;
  p.slice_c = C / p.slices;
  const int CVs = p.slice_c / 8;
  p.threads = (GN_STATS_THREADS / CVs) * CVs;
  p.rows_per_rank = (rows + p.ranks - 1) / p.ranks;
  return p;
}

static int unit_check(int C1, int C2, int unit, const char* who) {
  const int C = C1 + C2;
  if (unit <= 0 || (C % GN_GROUPS) || ((C / GN_GROUPS) % unit) || (C1 % unit) || (C2 % unit) || C1 / unit > GN_MAX_UNITS ||
      C2 / unit > GN_MAX_UNITS) {
    set_error("%s: unit %d must divide C1 = %d, C2 = %d and the channels per group %d (at most %d units per tensor)", who, unit,
              C1, C2, C / GN_GROUPS, GN_MAX_UNITS);
    return -2;
  }
  return 0;
}

extern "C" int hi3d_groupnorm_unit_stats(const void* x, int C, int n_images, int64_t rows_per_image, int unit, float* stats,
                                         void* stream) {
  if (!x || !stats || C <= 0 || (C % 8) || C > 8 * GN_STATS_THREADS || n_images <= 0 || n_images > 65535 ||
      rows_per_image <= 0 || unit <= 0 || (C % unit) || C / unit > GN_MAX_UNITS || ((uintptr_t)x & 15)) {
    set_error("hi3d_groupnorm_unit_stats: bad arguments (C=%d unit=%d n=%d rows=%lld)", C, unit, n_images, (long long)rows_per_image);
    return -2;
  }
  const GnStatsPlan p = unit_stats_plan(rows_per_image, C, unit);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(p.slices * p.ranks), (unsigned)n_images);
  cfg.blockDim = dim3((unsigned)p.threads);
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)p.ranks;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, gn_unit_stats_kernel, (const __half*)x, C, (long long)rows_per_image,
                                           p.rows_per_rank, p.slice_c, unit, stats);
  if (e != cudaSuccess) {
    set_error("hi3d_groupnorm_unit_stats: cluster launch failed: %s", cudaGetErrorString(e));
    return -1;
  }
  return check_launch("hi3d_groupnorm_unit_stats");
}

extern "C" int hi3d_groupnorm_group_sums(const float* stats1, int C1, const float* stats2, int C2, int unit, int n_samples,
                                         int imgs_per_sample, float* sums, void* stream) {
  if (!stats2) C2 = 0;
  if (!stats1 || !sums || n_samples <= 0 || imgs_per_sample <= 0) { set_error("hi3d_groupnorm_group_sums: bad arguments"); return -2; }
  int rc = unit_check(C1, C2, unit, "hi3d_groupnorm_group_sums");
  if (rc) return rc;
  gn_group_sums_kernel<<<n_samples, GN_GROUPS * 2, 0, (cudaStream_t)stream>>>(stats1, C1, stats2, C2, unit, imgs_per_sample, sums);
  return check_launch("hi3d_groupnorm_group_sums");
}

extern "C" int hi3d_groupnorm_apply_stats(const void* x1, int C1, const float* stats1, const void* x2, int C2, const float* stats2,
                                          int unit, int n_samples, int64_t rows_per_sample, int imgs_per_sample,
                                          int64_t count_rows, const float* gamma, const float* beta, float eps, int apply_silu,
                                          void* y, int64_t y_sample_rows, int64_t y_row_off, void* y_prev_rank, void* y_next_rank,
                                          int64_t frame_rows, void* stream) {
  if (!x2) { C2 = 0; stats2 = nullptr; }
  if (!stats1 || (x2 && !stats2) || imgs_per_sample <= 0) { set_error("hi3d_groupnorm_apply_stats: null statistics table"); return -2; }
  int rc = unit_check(C1, C2, unit, "hi3d_groupnorm_apply_stats");
  if (rc) return rc;
  return gn_apply_launch("hi3d_groupnorm_apply_stats", x1, C1, x2, C2, n_samples, rows_per_sample, nullptr, stats1, stats2, unit,
                         imgs_per_sample, count_rows, gamma, beta, eps, apply_silu, y, y_sample_rows, y_row_off, y_prev_rank,
                         y_next_rank, frame_rows, stream);
}

extern "C" int hi3d_groupnorm_apply_stats_fp8(const void* x1, int C1, const float* stats1, const void* x2, int C2,
                                              const float* stats2, int unit, int n_samples, int64_t rows_per_sample,
                                              int imgs_per_sample, int64_t count_rows, const float* gamma, const float* beta,
                                              float eps, int apply_silu, void* y, void* stream) {
  if (!x2) { C2 = 0; stats2 = nullptr; }
  if (!stats1 || (x2 && !stats2) || imgs_per_sample <= 0) {
    set_error("hi3d_groupnorm_apply_stats_fp8: null statistics table");
    return -2;
  }
  int rc = unit_check(C1, C2, unit, "hi3d_groupnorm_apply_stats_fp8");
  if (rc) return rc;
  return gn_apply_launch("hi3d_groupnorm_apply_stats_fp8", x1, C1, x2, C2, n_samples, rows_per_sample, nullptr, stats1, stats2,
                         unit, imgs_per_sample, count_rows, gamma, beta, eps, apply_silu, y, 0, 0, nullptr, nullptr, 0, stream,
                         true);
}

// The one launcher of the LayerNorm kernels; out8: e4m3 output.
static int layernorm_launch(const char* who, const void* x, const void* addvec, int add_div, int add_mod, int64_t M, int C,
                            const float* gamma, const float* beta, float eps, void* y, void* stream, bool out8) {
  if (!x || !y || !gamma || !beta || M <= 0 || C <= 0 || (C % 8) || C > 2560 || ((uintptr_t)x & 15) ||
      ((uintptr_t)y & 15) || ((uintptr_t)gamma & 7) || ((uintptr_t)beta & 7) ||
      (addvec && (add_div <= 0 || add_mod <= 0 || ((uintptr_t)addvec & 15)))) {
    set_error("%s: bad arguments (M=%lld C=%d)", who, (long long)M, C);
    return -2;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int CV = C / 8;
  const __half* xp = (const __half*)x;
  const __half* ap = (const __half*)addvec;
  __half* yp = (__half*)y;
#define HI3D_LN_LAUNCH(VPL, LPR)                                                                                        \
  do {                                                                                                                  \
    const long long rows_per_cta = 8 * (32 / LPR);                                                                      \
    const long long blocks = (M + rows_per_cta - 1) / rows_per_cta;                                                     \
    if (blocks > 2147483647LL) { set_error("%s: M too large", who); return -2; }                                 \
    if (out8) layernorm_kernel<VPL, LPR, true><<<(unsigned)blocks, 256, 0, st>>>(xp, ap, add_div, add_mod, M, C, gamma, beta, eps, yp); \
    else layernorm_kernel<VPL, LPR, false><<<(unsigned)blocks, 256, 0, st>>>(xp, ap, add_div, add_mod, M, C, gamma, beta, eps, yp); \
  } while (0)
#define HI3D_LN_GENERIC(VPL)                                                                                             \
  do {                                                                                                                  \
    const long long blocks = (M + 7) / 8;                                                                               \
    if (blocks > 2147483647LL) { set_error("%s: M too large", who); return -2; }                                 \
    if (out8) layernorm_generic_kernel<VPL, true><<<(unsigned)blocks, 256, 0, st>>>(xp, ap, add_div, add_mod, M, C, gamma, beta, eps, yp); \
    else layernorm_generic_kernel<VPL, false><<<(unsigned)blocks, 256, 0, st>>>(xp, ap, add_div, add_mod, M, C, gamma, beta, eps, yp); \
  } while (0)
  if (CV == 40) HI3D_LN_LAUNCH(5, 8);            // C = 320
  else if (CV == 80) HI3D_LN_LAUNCH(5, 16);      // C = 640
  else if (CV == 160) HI3D_LN_LAUNCH(5, 32);     // C = 1280
  else if (CV == 8) HI3D_LN_LAUNCH(1, 8);        // C = 64
  else if (CV == 16) HI3D_LN_LAUNCH(2, 8);       // C = 128
  else if (CV == 32) HI3D_LN_LAUNCH(2, 16);      // C = 256
  else if (CV == 64) HI3D_LN_LAUNCH(2, 32);      // C = 512
  else if (CV == 320) HI3D_LN_LAUNCH(10, 32);    // C = 2560
  else if (CV <= 64) HI3D_LN_GENERIC(2);
  else if (CV <= 160) HI3D_LN_GENERIC(5);
  else HI3D_LN_GENERIC(10);
#undef HI3D_LN_LAUNCH
#undef HI3D_LN_GENERIC
  return check_launch(who);
}


extern "C" int hi3d_layernorm(const void* x, const void* addvec, int add_div, int add_mod, int64_t M, int C,
                              const float* gamma, const float* beta, float eps, void* y, void* stream) {
  return layernorm_launch("hi3d_layernorm", x, addvec, add_div, add_mod, M, C, gamma, beta, eps, y, stream, false);
}

extern "C" int hi3d_layernorm_fp8(const void* x, const void* addvec, int add_div, int add_mod, int64_t M, int C,
                                  const float* gamma, const float* beta, float eps, void* y, void* stream) {
  return layernorm_launch("hi3d_layernorm_fp8", x, addvec, add_div, add_mod, M, C, gamma, beta, eps, y, stream, true);
}
