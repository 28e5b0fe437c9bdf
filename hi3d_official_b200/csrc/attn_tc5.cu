// Spatial self-attention core (head dim 64) on Hopper: TMA operand staging through an mbarrier ring and wgmma for both
// products -- S = Q K^T with Q and K from shared memory, O += P V with P from registers (the S accumulator fragment is the
// A-operand fragment of the next product, so P never touches shared memory) and V as an MN-major shared-memory operand.
//
// CTA = 128 queries x one (image, head), two warpgroups of 64 query rows; keys stream in tiles of BN (64 or 128) through a
// ring of (K, V) tiles that both warpgroups read.  Thread 0 issues every TMA load; each warp releases a stage once its
// warpgroup's MMAs on it have retired.  The key tail (L not a multiple of BN: keys of the next image or TMA out-of-bounds
// zeros) is masked to -inf before the online softmax; query rows past L are computed and not stored.
//
// Variants (hi3d_attention_tc5_set_variant) choose the key tile and the ring depth; hi3d_attention_tc5_set_exp_emulation
// moves a fraction (quarters, or 1/8, 3/8, 5/8) of the softmax exponentials from the MUFU pipe to the FMA pipe (exp2 by range reduction and a
// cubic, relative error 1.6e-4 before the fp16 rounding of P).
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "tc5.cuh"

namespace hi3d {

constexpr int FA_BM = 128;                 // queries per CTA
constexpr int FA_MAX_STAGES = 5;
constexpr int FA_THREADS = 256;
constexpr int FA_QTILE = 64 * 128;         // 64 rows x 64 fp16

struct FaParams {
  CUtensorMap q_map;       // [n_img * L, 3C] fp16 (q | k | v), box {64, 64}
  CUtensorMap kv_map;      // the same matrix, box {64, BN}
  int L, C, stages, emu8;   // emu8: eighths of the exponentials on the FMA pipe
  float scale_log2;
  __half* out;             // [n_img * L, C]
};

// (key tile, ring depth) of each variant.  Default: variant 6 without exponential emulation, the fastest on an H100 at the
// benchmark's shapes (32 images x 5 heads, L = 16384: 290 TFLOP/s against 272 for (64, 3) and 225 for the 128-key tiles;
// L = 4096: 288 against 280).
constexpr int FA_NVARIANTS = 7;
constexpr int FA_VARIANT_BN[FA_NVARIANTS] = {64, 64, 64, 128, 128, 128, 64};
constexpr int FA_VARIANT_STAGES[FA_NVARIANTS] = {2, 4, 3, 2, 3, 4, 5};
constexpr int FA_VARIANT_DEFAULT = 6;
constexpr int FA_EMU_DEFAULT = 0;

// 2^x for x <= 0 on the FMA pipe: x = j + f, 2^f by a cubic (relative error 1.6e-4), 2^j added to the exponent bits.
HI3D_DEVINL float exp2_fma(float x) {
  x = fmaxf(x, -127.f);
  const float j = floorf(x);
  const float f = x - j;
  const float p = fmaf(fmaf(fmaf(0.07640766f, f, 0.22823162f), f, 0.6950504f), f, 1.0f);
  return __int_as_float(__float_as_int(p) + ((int)j << 23));
}

template <int BN>
__global__ void __launch_bounds__(FA_THREADS, 1) fmha_tc5_kernel(const __grid_constant__ FaParams p) {
  constexpr int KV_TILE = BN * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  const int STAGES = p.stages;
  const uint32_t sQ = base;                                  // [128 queries x 64]
  const uint32_t sR = base + 2 * FA_QTILE;                   // ring: STAGES x (K tile, V tile)
  const uint32_t bar_q = sR + STAGES * 2 * KV_TILE;
  const uint32_t bar_full = bar_q + 8;                       // [STAGES]
  const uint32_t bar_empty = bar_full + 8 * FA_MAX_STAGES;   // [STAGES], one arrive per warp

  const int tid = threadIdx.x, lane = tid & 31;
  const int cw = tid >> 7;                                   // warpgroup: query rows 64 cw .. + 63
  const int warp = (tid >> 5) & 3;
  const int q0 = blockIdx.x * FA_BM;
  const int h = blockIdx.y;
  const int row0 = blockIdx.z * p.L;
  const int nkv = (p.L + BN - 1) / BN;
  const int C = p.C;

  auto issue_kv = [&](int j, int s) {
    const uint32_t full = bar_full + 8 * s;
    mbar_expect_tx(full, 2 * KV_TILE);
    tma_load_2d(sR + s * 2 * KV_TILE, &p.kv_map, full, C + h * 64, row0 + j * BN);
    tma_load_2d(sR + s * 2 * KV_TILE + KV_TILE, &p.kv_map, full, 2 * C + h * 64, row0 + j * BN);
  };
  if (tid == 0) {
    mbar_init(bar_q, 1);
    for (int s = 0; s < STAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    mbar_expect_tx(bar_q, 2 * FA_QTILE);
    tma_load_2d(sQ, &p.q_map, bar_q, h * 64, row0 + q0);
    tma_load_2d(sQ + FA_QTILE, &p.q_map, bar_q, h * 64, row0 + q0 + 64);
    for (int j = 0; j < STAGES && j < nkv; j++) issue_kv(j, j);
  }
  __syncthreads();

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; i++) o[i] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const int t4 = lane & 3;
  const float c = p.scale_log2;
  const uint64_t qd = gmma_desc_sw128(sQ + cw * FA_QTILE);
  const int emu8 = p.emu8;
  mbar_wait(bar_q, 0);

  uint32_t s = 0, ph = 0;
  for (int j = 0; j < nkv; j++) {
    mbar_wait(bar_full + 8 * s, ph);
    const uint32_t sK = sR + s * 2 * KV_TILE, sV = sK + KV_TILE;
    // ---- S = Q K^T ----
    float sc[BN / 2];
    const uint64_t kd = gmma_desc_sw128(sK);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) wgmma_ss<BN>(sc, qd + (uint64_t)(2 * k), kd + (uint64_t)(2 * k), k);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    // ---- mask the key tail ----
    if ((j + 1) * BN > p.L) {
#pragma unroll
      for (int nt = 0; nt < BN / 8; nt++) {
        const int col = j * BN + nt * 8 + 2 * t4;
        if (col >= p.L) { sc[4 * nt] = -INFINITY; sc[4 * nt + 2] = -INFINITY; }
        if (col + 1 >= p.L) { sc[4 * nt + 1] = -INFINITY; sc[4 * nt + 3] = -INFINITY; }
      }
    }
    // ---- online softmax: this thread holds rows g (hh = 0) and g + 8 (hh = 1) of its warp's 16 rows ----
    uint32_t pa[BN / 16][4];
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < BN / 8; nt++) mx = fmaxf(mx, fmaxf(sc[4 * nt + 2 * hh], sc[4 * nt + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mnew = fmaxf(mrow[hh], mx);
      const float corr = exp2f((mrow[hh] - mnew) * c);
      const float moff = mnew * c;
      float rs = 0.f;
#pragma unroll
      for (int nt = 0; nt < BN / 8; nt++) {
        const float x0 = sc[4 * nt + 2 * hh] * c - moff, x1 = sc[4 * nt + 2 * hh + 1] * c - moff;
        const bool fma_pipe = (nt & 7) < emu8;       // emu8 eighths of the key columns
        const float p0 = fma_pipe ? exp2_fma(x0) : exp2f(x0);
        const float p1 = fma_pipe ? exp2_fma(x1) : exp2f(x1);
        rs += p0 + p1;
        // accumulator fragment -> A fragment: key columns 8 nt .. feed k16 step nt / 2, register (nt & 1) * 2 + hh
        pa[nt >> 1][(nt & 1) * 2 + hh] = pack_half2(p0, p1);
      }
      lrow[hh] = lrow[hh] * corr + rs;
      mrow[hh] = mnew;
#pragma unroll
      for (int dt = 0; dt < 8; dt++) {
        o[4 * dt + 2 * hh] *= corr;
        o[4 * dt + 2 * hh + 1] *= corr;
      }
    }
    // ---- O += P V (16 keys per MMA: V advances 16 rows = 2048 bytes) ----
    const uint64_t vd = gmma_desc_sw128(sV);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; kk++) wgmma_rs_tb<64>(o, pa[kk], vd + (uint64_t)(128 * kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
    if (tid == 0 && j + STAGES < nkv) {
      mbar_wait(bar_empty + 8 * s, ph);          // both warpgroups are done with this stage
      issue_kv(j + STAGES, s);
    }
    if (++s == (uint32_t)STAGES) { s = 0; ph ^= 1; }
  }

  // ---- finalize: O /= l, stage through this warpgroup's own Q rows, 16-byte stores ----
  const int g = lane >> 2;
  uint8_t* stage = smem + cw * FA_QTILE;
#pragma unroll
  for (int hh = 0; hh < 2; hh++) {
    float l = lrow[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    const int r = warp * 16 + g + 8 * hh;
#pragma unroll
    for (int dt = 0; dt < 8; dt++)
      *reinterpret_cast<uint32_t*>(stage + swz128(r, dt) + t4 * 4) = pack_half2(o[4 * dt + 2 * hh] * inv, o[4 * dt + 2 * hh + 1] * inv);
  }
  __syncwarp();
  __half* obase = p.out + (long long)row0 * C + h * 64;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int r = warp * 16 + (lane >> 3) + 4 * i;
    const int ch = lane & 7;
    const int q = q0 + cw * 64 + r;
    if (q < p.L) {
      const uint4 v = *reinterpret_cast<const uint4*>(stage + swz128(r, ch));
      *reinterpret_cast<uint4*>(obase + (long long)q * C + ch * 8) = v;
    }
  }
}

static int g_variant = -1;   // -1 unread: HI3D_FMHA_VARIANT, else FA_VARIANT_DEFAULT
static int g_emu = -1;       // -1 unread: HI3D_FMHA_EMU, else FA_EMU_DEFAULT
static void read_env_once() {
  if (g_variant < 0) {
    const char* e = getenv("HI3D_FMHA_VARIANT");
    g_variant = e ? atoi(e) : FA_VARIANT_DEFAULT;
    if (g_variant < 0 || g_variant >= FA_NVARIANTS) g_variant = FA_VARIANT_DEFAULT;
  }
  if (g_emu < 0) {
    const char* e = getenv("HI3D_FMHA_EMU");
    g_emu = e ? atoi(e) : FA_EMU_DEFAULT;
    if (g_emu < 0 || g_emu > 7) g_emu = FA_EMU_DEFAULT;
  }
}

template <int BN>
static int launch_fmha(FaParams& fp, const void* qkv, int n_img, int heads, cudaStream_t st) {
  {
    cuuint64_t dims[2] = {(cuuint64_t)(3 * fp.C), (cuuint64_t)n_img * (cuuint64_t)fp.L};
    cuuint64_t str[1] = {(cuuint64_t)(3 * fp.C) * 2};
    cuuint32_t box[2] = {64, 64};
    if (encode_map(&fp.q_map, qkv, 2, dims, str, box, nullptr)) return -1;
    box[1] = BN;
    if (encode_map(&fp.kv_map, qkv, 2, dims, str, box, nullptr)) return -1;
  }
  constexpr int smem_max = 2 * FA_QTILE + FA_MAX_STAGES * 2 * BN * 128 + 8 + 16 * FA_MAX_STAGES + 1024;
  const int smem = 2 * FA_QTILE + fp.stages * 2 * BN * 128 + 8 + 16 * FA_MAX_STAGES + 1024;
  static bool attr_done[HI3D_MAX_DEVICES];
  if (ensure_dyn_smem(fmha_tc5_kernel<BN>, smem_max, attr_done, "hi3d_attention_d64_tc5")) return -1;
  dim3 grid((fp.L + FA_BM - 1) / FA_BM, heads, n_img);
  fmha_tc5_kernel<BN><<<grid, FA_THREADS, smem, st>>>(fp);
  return check_launch("hi3d_attention_d64_tc5");
}

}  // namespace hi3d

using namespace hi3d;

extern "C" int hi3d_attention_d64_tc5(const void* qkv, int n_img, int L, int heads, float scale, void* out, void* stream) {
  if (!qkv || !out || n_img <= 0 || L <= 0 || heads <= 0 || ((uintptr_t)qkv & 15) || ((uintptr_t)out & 15)) {
    set_error("hi3d_attention_d64_tc5: bad arguments (n_img=%d L=%d heads=%d)", n_img, L, heads);
    return -2;
  }
  if (heads > 65535 || n_img > 65535) { set_error("hi3d_attention_d64_tc5: grid too large"); return -2; }
  read_env_once();
  FaParams fp;
  memset(&fp, 0, sizeof(fp));
  fp.L = L;
  fp.C = heads * 64;
  fp.stages = FA_VARIANT_STAGES[g_variant];
  fp.emu8 = g_emu <= 4 ? 2 * g_emu : (g_emu == 5 ? 3 : (g_emu == 6 ? 1 : 5));
  fp.scale_log2 = scale * 1.4426950408889634f;
  fp.out = (__half*)out;
  const cudaStream_t st = (cudaStream_t)stream;
  return FA_VARIANT_BN[g_variant] == 128 ? launch_fmha<128>(fp, qkv, n_img, heads, st) : launch_fmha<64>(fp, qkv, n_img, heads, st);
}

extern "C" int hi3d_attention_tc5_set_variant(int variant) {
  if (variant < 0 || variant >= FA_NVARIANTS) {
    set_error("hi3d_attention_tc5_set_variant: variant must be 0 .. %d", FA_NVARIANTS - 1);
    return -2;
  }
  read_env_once();
  g_variant = variant;
  return 0;
}

extern "C" int hi3d_attention_tc5_set_exp_emulation(int quarters) {
  if (quarters < 0 || quarters > 7) {
    set_error("hi3d_attention_tc5_set_exp_emulation: 0 .. 4 (quarters of the exponentials) or 5 / 6 / 7 (3/8, 1/8, 5/8)");
    return -2;
  }
  read_env_once();
  g_emu = quarters;
  return 0;
}
