// VAE mid-block attention (AttnBlock, model.py:180-201): ONE head of dimension 512 over L = (H/8)(W/8) tokens, as a
// flash-attention kernel on Hopper (TMA + wgmma) -- no L x L score matrix in memory, scores and softmax in fp32.
//
// A 64-query x 512 fp32 accumulator would be 256 registers per thread, so a CTA (one warpgroup) owns 64 queries and HALF of
// the value dimension (256 columns): grid (L/64, 2, images); both halves compute the full S = Q K^T (contraction over
// 512) -- 1.5x the minimal tensor work, on a block that is ~1 % of a video.
//   S = sum over eight 64-wide chunks c of Q_c K_c^T: the 64 x 512 query tile (64 KB) stays RESIDENT in shared memory; the
//       64 x 512 key tile (64 KB) and this CTA's 64 x 256 value half (32 KB) have one buffer each, refilled by TMA as soon as
//       the MMAs that read them have retired (K(j+1) loads during softmax and P V(j), V(j+1) during S(j+1)).
//   softmax: online, in registers (rows g and g + 8 of each warp's 16 rows per thread).
//   O += P V: P from registers (the S accumulator fragment), V as four MN-major 64-column chunks.
#include <cuda.h>
#include <string.h>

#include "common.cuh"
#include "tc5.cuh"

namespace hi3d {

constexpr int F5_BM = 64, F5_BN = 64, F5_D = 512, F5_DV = 256;
constexpr int F5_THREADS = 128;
constexpr int F5_TILE = 64 * 128;                  // 64 rows x 64 fp16
constexpr int F5_SMEM = 8 * F5_TILE + 8 * F5_TILE + 4 * F5_TILE + 64 + 1024;

struct Fa512Params {
  CUtensorMap qkv_map;     // [rows, 1536] fp16 (q | k | v), box {64, 64}
  int L;
  float scale_log2;
  __half* out;             // [rows, 512]
};

__global__ void __launch_bounds__(F5_THREADS, 1) fmha512_tc5_kernel(const __grid_constant__ Fa512Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t sQ = base;                                    // 8 chunks [64 queries x 64], resident
  const uint32_t sK = sQ + 8 * F5_TILE;                        // 8 chunks [64 keys x 64]
  const uint32_t sV = sK + 8 * F5_TILE;                        // 4 chunks [64 keys x 64] of this CTA's value half
  const uint32_t bar_q = sV + 4 * F5_TILE;
  const uint32_t bar_k = bar_q + 8;
  const uint32_t bar_v = bar_k + 8;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q0 = blockIdx.x * F5_BM;
  const int dvh = blockIdx.y;
  const int row0 = blockIdx.z * p.L;
  const int nkv = p.L / F5_BN;

  auto load_k = [&](int j) {
    mbar_expect_tx(bar_k, 8 * F5_TILE);
    for (int c = 0; c < 8; c++) tma_load_2d(sK + c * F5_TILE, &p.qkv_map, bar_k, F5_D + c * 64, row0 + j * F5_BN);
  };
  auto load_v = [&](int j) {
    mbar_expect_tx(bar_v, 4 * F5_TILE);
    for (int c = 0; c < 4; c++)
      tma_load_2d(sV + c * F5_TILE, &p.qkv_map, bar_v, 2 * F5_D + dvh * F5_DV + c * 64, row0 + j * F5_BN);
  };
  if (tid == 0) {
    mbar_init(bar_q, 1);
    mbar_init(bar_k, 1);
    mbar_init(bar_v, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    mbar_expect_tx(bar_q, 8 * F5_TILE);
    for (int c = 0; c < 8; c++) tma_load_2d(sQ + c * F5_TILE, &p.qkv_map, bar_q, c * 64, row0 + q0);
    load_k(0);
    load_v(0);
  }
  __syncthreads();

  float o[4][32];
#pragma unroll
  for (int c = 0; c < 4; c++)
#pragma unroll
    for (int i = 0; i < 32; i++) o[c][i] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const float cl = p.scale_log2;
  mbar_wait(bar_q, 0);

  for (int j = 0; j < nkv; j++) {
    // ---- S = sum_c Q_c K_c^T ----
    mbar_wait(bar_k, j & 1);
    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const uint64_t qd = gmma_desc_sw128(sQ + c * F5_TILE), kd = gmma_desc_sw128(sK + c * F5_TILE);
#pragma unroll
      for (int k = 0; k < 4; k++) wgmma_ss<64>(sc, qd + (uint64_t)(2 * k), kd + (uint64_t)(2 * k), (c | k) ? 1 : 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    __syncthreads();                                           // every warp's MMAs on K(j) have retired
    if (tid == 0 && j + 1 < nkv) load_k(j + 1);
    // ---- online softmax ----
    uint32_t pa[4][4];
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; nt++) mx = fmaxf(mx, fmaxf(sc[4 * nt + 2 * hh], sc[4 * nt + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mnew = fmaxf(mrow[hh], mx);
      const float corr = exp2f((mrow[hh] - mnew) * cl);
      const float moff = mnew * cl;
      float rs = 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; nt++) {
        const float p0 = exp2f(sc[4 * nt + 2 * hh] * cl - moff);
        const float p1 = exp2f(sc[4 * nt + 2 * hh + 1] * cl - moff);
        rs += p0 + p1;
        pa[nt >> 1][(nt & 1) * 2 + hh] = pack_half2(p0, p1);
      }
      lrow[hh] = lrow[hh] * corr + rs;
      mrow[hh] = mnew;
#pragma unroll
      for (int c = 0; c < 4; c++)
#pragma unroll
        for (int dt = 0; dt < 8; dt++) {
          o[c][4 * dt + 2 * hh] *= corr;
          o[c][4 * dt + 2 * hh + 1] *= corr;
        }
    }
    // ---- O += P V ----
    mbar_wait(bar_v, j & 1);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; kk++)
#pragma unroll
      for (int c = 0; c < 4; c++) wgmma_rs_tb<64>(o[c], pa[kk], gmma_desc_sw128(sV + c * F5_TILE) + (uint64_t)(128 * kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < 4; c++) wgmma_fence_regs(o[c]);
    __syncthreads();                                           // every warp's MMAs on V(j) have retired
    if (tid == 0 && j + 1 < nkv) load_v(j + 1);
  }

  // ---- epilogue: O / l -> fp16, this CTA's 256 output columns of rows g and g + 8 ----
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int hh = 0; hh < 2; hh++) {
    float l = lrow[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    __half* dst = p.out + (long long)(row0 + q0 + warp * 16 + g + 8 * hh) * F5_D + dvh * F5_DV + 2 * t4;
#pragma unroll
    for (int c = 0; c < 4; c++)
#pragma unroll
      for (int dt = 0; dt < 8; dt++)
        *reinterpret_cast<uint32_t*>(dst + c * 64 + dt * 8) = pack_half2(o[c][4 * dt + 2 * hh] * inv, o[c][4 * dt + 2 * hh + 1] * inv);
  }
}

}  // namespace hi3d

using namespace hi3d;

extern "C" int hi3d_attention_d512_tc5(const void* qkv, int n_img, int L, float scale, void* out, void* stream) {
  if (!qkv || !out || n_img <= 0 || L <= 0 || (L % 128) || n_img > 65535 || ((uintptr_t)qkv & 15) || ((uintptr_t)out & 15)) {
    set_error("hi3d_attention_d512_tc5: bad arguments (n_img=%d L=%d; L must be a multiple of 128)", n_img, L);
    return -2;
  }
  Fa512Params fp;
  memset(&fp, 0, sizeof(fp));
  {
    cuuint64_t dims[2] = {(cuuint64_t)(3 * F5_D), (cuuint64_t)n_img * (cuuint64_t)L};
    cuuint64_t str[1] = {(cuuint64_t)(3 * F5_D) * 2};
    cuuint32_t box[2] = {64, 64};
    if (encode_map(&fp.qkv_map, qkv, 2, dims, str, box, nullptr)) return -1;
  }
  fp.L = L;
  fp.scale_log2 = scale * 1.4426950408889634f;
  fp.out = (__half*)out;
  static bool attr_done[HI3D_MAX_DEVICES];
  if (ensure_dyn_smem(fmha512_tc5_kernel, F5_SMEM, attr_done, "hi3d_attention_d512_tc5")) return -1;
  dim3 grid(L / F5_BM, 2, n_img);
  fmha512_tc5_kernel<<<grid, F5_THREADS, F5_SMEM, (cudaStream_t)stream>>>(fp);
  return check_launch("hi3d_attention_d512_tc5");
}
