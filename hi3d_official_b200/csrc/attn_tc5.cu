// Spatial self-attention core (head dim 64) on Hopper: a warp-specialised, software-pipelined flash-attention kernel.
// TMA stages the operands through mbarrier rings and wgmma runs both products -- S = Q K^T with Q and K from shared memory,
// O += P V with P from registers (the S accumulator fragment is the A-operand fragment of the next product, so P never
// touches shared memory) and V as an MN-major shared-memory operand.
//
// CTA = 64 NC queries x one (image, head): warpgroup 0 is the producer (one lane issues every TMA load and the warpgroup
// hands its registers to the consumers), warpgroups 1 .. NC each own 64 query rows.  Keys stream in tiles of BN (64 or
// 128) through two rings, one of K tiles and one of V tiles, each stage with its own full and empty barrier: S_j starts as
// soon as K_j has landed, K_j's slot goes back to the producer when S_j retires and V_j's when P_j V_j retires.
//
// At d = 64 the exponentials (MUFU) take as many cycles as the two products (tensor cores), so a consumer overlaps them:
//   issue S_j = Q K_j^T | O *= correction_{j-1} | issue O += P_{j-1} V_{j-1} | wait S_j | softmax(S_j) | wait P V | pack P_j
// -- the softmax of tile j runs while the tensor cores work on S_j's tail and on P_{j-1} V_{j-1}.  Only wgmma touches the
// registers of an in-flight product (P_j stays fp32 in the S registers until P_{j-1} V_{j-1} retires), so ptxas keeps the
// products asynchronous.
//
// The key tail (L not a multiple of BN: keys of the next image or TMA out-of-bounds zeros) is masked to -inf before the
// online softmax; tiles are visited in order, so the masked tile comes last and every row has a finite maximum by then.
// Query rows past L are computed and not stored.
//
// Variants (hi3d_attention_tc5_set_variant) choose the key tile, the consumer count and the ring depth;
// hi3d_attention_tc5_set_exp_emulation moves a fraction (quarters, or 1/8, 3/8, 5/8) of the softmax exponentials from the
// MUFU pipe to the FMA pipe (exp2 by range reduction and a cubic, relative error 1.6e-4 before the fp16 rounding of P).
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "attn_softmax.cuh"
#include "common.cuh"
#include "tc5.cuh"

namespace hi3d {

constexpr int FA_MAX_STAGES = 4;
constexpr int FA_QTILE = 64 * 128;         // 64 query rows x 64 fp16: one consumer warpgroup's Q tile

struct FaParams {
  CUtensorMap q_map;       // [n_img * L, 3C] fp16 (q | k | v), box {64, 64}
  CUtensorMap kv_map;      // the same matrix, box {64, BN}
  int L, C, stages;
  float scale_log2;
  __half* out;             // [n_img * L, C]
};

// (key tile, consumer warpgroups, ring depth) of each variant.  Default: variant 6 without exponential emulation.  On an
// H100 80GB HBM3 at 700 W (tools/time_attention.py, 32 images): L = 16384 x 5 heads 413 TFLOP/s (variant 5: 417, 4: 412,
// 2: 408, 3: 407, the two-stage 64-key variants 0 / 1: 350), L = 4096 x 10 heads 391 (5: 393), L = 1024 x 20 heads 334
// (5: 318), L = 256 x 20 heads 194 (5: 164) -- variant 6 is within 1 % of the fastest at every shape.  Moving 1/8 of the
// exponentials to the FMA pipe costs 8 % at L = 16384 and 3/8 costs 14 %: the tensor cores, not MUFU, set the pace now.
constexpr int FA_NVARIANTS = 7;
// 128-key tiles run with two consumers only: three need S (64) + P (32) + O (32) fp32 registers per thread in flight, and
// ptxas allocates to the 128-register cap of a 512-thread CTA (not to the setmaxnreg budget), so they spill.
constexpr int FA_VARIANT_BN[FA_NVARIANTS] = {64, 64, 64, 128, 128, 64, 128};
constexpr int FA_VARIANT_NC[FA_NVARIANTS] = {2, 2, 3, 2, 2, 3, 2};
constexpr int FA_VARIANT_STAGES[FA_NVARIANTS] = {2, 4, 2, 2, 4, 4, 3};
constexpr int FA_VARIANT_DEFAULT = 6;
constexpr int FA_EMU_DEFAULT = 0;

// accumulator fragment -> A fragment: key columns 8 nt .. feed k16 step nt / 2, registers (nt & 1) * 2 + hh
template <int BN>
HI3D_DEVINL void fa_pack(const float (&sc)[BN / 2], uint32_t (&pa)[BN / 16][4]) {
#pragma unroll
  for (int nt = 0; nt < BN / 8; nt++)
#pragma unroll
    for (int hh = 0; hh < 2; hh++) pa[nt >> 1][(nt & 1) * 2 + hh] = pack_half2(sc[4 * nt + 2 * hh], sc[4 * nt + 2 * hh + 1]);
}

template <int BN, int NC, int EMU8>
__global__ void __launch_bounds__(128 * (NC + 1), 1) fmha_tc5_kernel(const __grid_constant__ FaParams p) {
  constexpr int KV_TILE = BN * 128;
  constexpr int BM = 64 * NC;                                // queries per CTA
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  const int STAGES = p.stages;
  const uint32_t sQ = base;                                  // NC x [64 queries x 64]
  const uint32_t sK = sQ + NC * FA_QTILE;                    // STAGES K tiles
  const uint32_t sV = sK + STAGES * KV_TILE;                 // STAGES V tiles
  const uint32_t bar_q = sV + STAGES * KV_TILE;
  const uint32_t bar_kfull = bar_q + 8;                      // [STAGES] each: the producer's expect_tx arrive
  const uint32_t bar_vfull = bar_kfull + 8 * FA_MAX_STAGES;
  const uint32_t bar_kempty = bar_vfull + 8 * FA_MAX_STAGES; // [STAGES] each: one arrive per consumer warp
  const uint32_t bar_vempty = bar_kempty + 8 * FA_MAX_STAGES;

  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);      // warp-uniform role index
  const int q0 = blockIdx.x * BM;
  const int h = blockIdx.y;
  const int row0 = blockIdx.z * p.L;
  const int nkv = (p.L + BN - 1) / BN;
  const int C = p.C;

  if (tid == 0) {
    mbar_init(bar_q, 1);
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar_kfull + 8 * s, 1);
      mbar_init(bar_vfull + 8 * s, 1);
      mbar_init(bar_kempty + 8 * s, 4 * NC);
      mbar_init(bar_vempty + 8 * s, 4 * NC);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ======================= TMA producer: Q once, then K_0, and (K_{j+1}, V_j) in the order the consumers use them
    setmaxnreg_dec<NC == 2 ? 24 : 32>();
    if (tid == 0) {
      mbar_expect_tx(bar_q, NC * FA_QTILE);
      for (int c = 0; c < NC; c++) tma_load_2d(sQ + c * FA_QTILE, &p.q_map, bar_q, h * 64, row0 + q0 + 64 * c);
      uint32_t ks = 0, kph = 0, vs = 0, vph = 0;
      auto load_k = [&](int j) {
        mbar_wait(bar_kempty + 8 * ks, kph ^ 1);
        mbar_expect_tx(bar_kfull + 8 * ks, KV_TILE);
        tma_load_2d(sK + ks * KV_TILE, &p.kv_map, bar_kfull + 8 * ks, C + h * 64, row0 + j * BN);
        if (++ks == (uint32_t)STAGES) { ks = 0; kph ^= 1; }
      };
      load_k(0);
      for (int j = 0; j < nkv; j++) {
        if (j + 1 < nkv) load_k(j + 1);
        mbar_wait(bar_vempty + 8 * vs, vph ^ 1);
        mbar_expect_tx(bar_vfull + 8 * vs, KV_TILE);
        tma_load_2d(sV + vs * KV_TILE, &p.kv_map, bar_vfull + 8 * vs, 2 * C + h * 64, row0 + j * BN);
        if (++vs == (uint32_t)STAGES) { vs = 0; vph ^= 1; }
      }
    }
    return;
  }

  // ======================= consumers: warpgroup cw owns query rows 64 cw .. + 63 of the CTA's tile
  setmaxnreg_inc<NC == 2 ? 240 : 160>();
  const int cw = wg - 1;
  const int warp = (tid >> 5) & 3;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; i++) o[i] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f}, corr[2];
  const int t4 = lane & 3;
  const float c = p.scale_log2;
  const uint64_t qd = gmma_desc_sw128(sQ + cw * FA_QTILE);
  float sc[BN / 2];
  uint32_t pa[BN / 16][4];
  uint32_t ks = 0, kph = 0, vs = 0, vph = 0;
  auto issue_s = [&]() {       // S = Q K^T on K stage ks
    const uint64_t kd = gmma_desc_sw128(sK + ks * KV_TILE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) wgmma_ss<BN>(sc, qd + (uint64_t)(2 * k), kd + (uint64_t)(2 * k), k);
    wgmma_commit();
  };
  auto issue_pv = [&]() {      // O += P V on V stage vs (16 keys per MMA: V advances 16 rows = 2048 bytes)
    const uint64_t vd = gmma_desc_sw128(sV + vs * KV_TILE);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; kk++) wgmma_rs_tb<64>(o, pa[kk], vd + (uint64_t)(128 * kk), 1);
    wgmma_commit();
  };
  auto release = [&](uint32_t bar, uint32_t& s, uint32_t& ph) {
    __syncwarp();
    if (lane == 0) mbar_arrive(bar + 8 * s);
    if (++s == (uint32_t)STAGES) { s = 0; ph ^= 1; }
  };

  auto rescale_o = [&]() {
#pragma unroll
    for (int dt = 0; dt < 8; dt++) {
      o[4 * dt] *= corr[0];
      o[4 * dt + 1] *= corr[0];
      o[4 * dt + 2] *= corr[1];
      o[4 * dt + 3] *= corr[1];
    }
  };

  mbar_wait(bar_q, 0);
  mbar_wait(bar_kfull, 0);
  issue_s();
  wgmma_wait<0>();
  wgmma_fence_regs(sc);
  release(bar_kempty, ks, kph);
  fa_softmax<BN, EMU8>(sc, mrow, lrow, corr, 0, p.L, c, t4);
  fa_pack<BN>(sc, pa);
  for (int j = 1; j < nkv; j++) {
    mbar_wait(bar_kfull + 8 * ks, kph);
    issue_s();                                  // S_j
    rescale_o();                                // to tile j - 1's running max
    mbar_wait(bar_vfull + 8 * vs, vph);
    issue_pv();                                 // O += P_{j-1} V_{j-1}
    wgmma_wait<1>();                            // S_j has retired, P V may still run
    wgmma_fence_regs(sc);
    release(bar_kempty, ks, kph);
    fa_softmax<BN, EMU8>(sc, mrow, lrow, corr, j, p.L, c, t4);
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    release(bar_vempty, vs, vph);
    fa_pack<BN>(sc, pa);
  }
  rescale_o();
  mbar_wait(bar_vfull + 8 * vs, vph);
  issue_pv();
  wgmma_wait<0>();
  wgmma_fence_regs(o);

  // ---- finalize: O /= l, stage through this warpgroup's own Q rows (only its own S products read them), 16-byte stores
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

template <int BN, int NC, int EMU8>
static int launch_fmha(FaParams& fp, const void* qkv, int n_img, int heads, cudaStream_t st) {
  {
    cuuint64_t dims[2] = {(cuuint64_t)(3 * fp.C), (cuuint64_t)n_img * (cuuint64_t)fp.L};
    cuuint64_t str[1] = {(cuuint64_t)(3 * fp.C) * 2};
    cuuint32_t box[2] = {64, 64};
    if (encode_map(&fp.q_map, qkv, 2, dims, str, box, nullptr)) return -1;
    box[1] = BN;
    if (encode_map(&fp.kv_map, qkv, 2, dims, str, box, nullptr)) return -1;
  }
  constexpr int bars = 8 + 4 * 8 * FA_MAX_STAGES;
  constexpr int smem_max = NC * FA_QTILE + FA_MAX_STAGES * 2 * BN * 128 + bars + 1024;
  const int smem = NC * FA_QTILE + fp.stages * 2 * BN * 128 + bars + 1024;
  static bool attr_done[HI3D_MAX_DEVICES];
  if (ensure_dyn_smem(fmha_tc5_kernel<BN, NC, EMU8>, smem_max, attr_done, "hi3d_attention_d64_tc5")) return -1;
  dim3 grid((fp.L + 64 * NC - 1) / (64 * NC), heads, n_img);
  fmha_tc5_kernel<BN, NC, EMU8><<<grid, 128 * (NC + 1), smem, st>>>(fp);
  return check_launch("hi3d_attention_d64_tc5");
}

template <int EMU8>
static int launch_variant(FaParams& fp, const void* qkv, int n_img, int heads, cudaStream_t st) {
  const int bn = FA_VARIANT_BN[g_variant], nc = FA_VARIANT_NC[g_variant];
  if (bn == 128) return launch_fmha<128, 2, EMU8>(fp, qkv, n_img, heads, st);
  return nc == 3 ? launch_fmha<64, 3, EMU8>(fp, qkv, n_img, heads, st) : launch_fmha<64, 2, EMU8>(fp, qkv, n_img, heads, st);
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
  fp.scale_log2 = scale * 1.4426950408889634f;
  fp.out = (__half*)out;
  const cudaStream_t st = (cudaStream_t)stream;
  const int emu8 = g_emu <= 4 ? 2 * g_emu : (g_emu == 5 ? 3 : (g_emu == 6 ? 1 : 5));
  switch (emu8) {
    case 0: return launch_variant<0>(fp, qkv, n_img, heads, st);
    case 1: return launch_variant<1>(fp, qkv, n_img, heads, st);
    case 2: return launch_variant<2>(fp, qkv, n_img, heads, st);
    case 3: return launch_variant<3>(fp, qkv, n_img, heads, st);
    case 4: return launch_variant<4>(fp, qkv, n_img, heads, st);
    case 5: return launch_variant<5>(fp, qkv, n_img, heads, st);
    case 6: return launch_variant<6>(fp, qkv, n_img, heads, st);
    default: return launch_variant<8>(fp, qkv, n_img, heads, st);
  }
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
