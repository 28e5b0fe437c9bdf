// Spatial self-attention core (head dim 64) with e4m3 operands on Hopper: the flash-attention kernel of attn_tc5.cu with both
// products on the FP8 tensor cores.  Same structure: a TMA producer warpgroup that hands its registers to the consumers,
// separate K and V rings with a full and an empty mbarrier per stage, consumer warpgroups of 64 queries, and the softmax of key
// tile j overlapped with S_j and P_{j-1} V_{j-1}:
//   issue S_j = Q K_j^T | O *= correction_{j-1} | issue O += P_{j-1} V_{j-1} | wait S_j | softmax(S_j) | wait P V | pack P_j
//
// What changes against the fp16 kernel:
//  - Q and K tiles are 64-byte rows (64 e4m3) under SWIZZLE_64B; S = Q K^T is two k32 MMAs.
//  - FP8 wgmma takes only K-major B, so P V needs V with keys contiguous: V tiles come from vt, the per-(image, head)
//    transpose that hi3d_attention_vt_e4m3 writes, as {128 keys, 64 rows} boxes (128-byte rows, SWIZZLE_128B).  Its key
//    columns are permuted within each 32-block (see include/hi3d_b200.h) so that the f32 S fragment of a thread, keys
//    8 i + 2 t4 + {0, 1}, is exactly the thread's e4m3 A fragment of P V: P is converted in registers with
//    cvt.rn.satfinite.e4m3x2.f32 and no shuffles.
//  - P = exp2(s - m) in (0, 1] is computed scaled by 2^8 (a PLOG2 of the shared softmax), so that e4m3 keeps keys down to
//    2^-17 of the row maximum instead of flushing everything below 2^-9.  The row sum l is kept in fp32 from the unrounded
//    scaled P, and O / l removes the scale.
//
// One configuration: 128-key tiles, two consumer warpgroups, three stages per ring, every exponential on MUFU.  On an H100 80GB
// HBM3 at 700 W (tools/time_attention.py --fp8, 32 images x 16384 keys x 5 heads) the kernel takes 22.4 ms, 491 TFLOP/s against
// 454 for hi3d_attention_d64_tc5 in the same run; with 1/8 of the exponentials on the FMA pipe (exp2_fma) 22.6 ms, with 1/4
// 24.9 ms.  The tensor cores are idle most of the time: each consumer warp issues about 460 instructions per 128-key tile
// (66 MUFU.EX2, 68 FFMA, 66 FADD, 70 FMNMX, 34 FMUL, 32 F2FP, 16 PRMT, ...) for 2048 scores, and two such warps per scheduler
// hide little of the softmax's max / shuffle / exp / sum latency chain.
#include <cuda.h>
#include <string.h>

#include "attn_softmax.cuh"
#include "common.cuh"
#include "tc5.cuh"

namespace hi3d {

constexpr int FA8_BN = 128;                  // keys per tile
constexpr int FA8_NC = 2;                    // consumer warpgroups of 64 queries
constexpr int FA8_STAGES = 3;                // depth of the K ring and of the V ring
constexpr int FA8_EMU8 = 0;                  // eighths of the exponentials on the FMA pipe
constexpr int FA8_PLOG2 = 8;                 // P is scaled by 2^8 before its e4m3 rounding
constexpr int FA8_QSLOT = 64 * 128;          // per consumer: its Q tile (64 x 64 e4m3, 4 KiB), later its fp16 output staging
constexpr int FA8_QTILE = 64 * 64;
constexpr int FA8_KTILE = FA8_BN * 64;       // BN keys x 64 e4m3
constexpr int FA8_VTILE = 64 * FA8_BN;       // 64 rows (d) x BN keys
constexpr int FA8_VT_KEYS = 128;             // vt's key axis is padded to a multiple of this

struct Fa8Params {
  CUtensorMap q_map;       // qkv8 [n_img * L, 3C] e4m3 (q | k | v), box {64, 64}, SWIZZLE_64B
  CUtensorMap k_map;       // the same matrix, box {64, BN}
  CUtensorMap v_map;       // vt [n_img * heads * 64, Lp] e4m3, box {BN, 64}, SWIZZLE_128B
  int L, C;
  float scale_log2;
  __half* out;             // [n_img * L, C]
};

// Four fp32 values -> four e4m3 bytes, a0 in the lowest byte (cvt.rn.satfinite: nearest even, saturating to +-448).
HI3D_DEVINL uint32_t pack_e4m3x4(float a0, float a1, float a2, float a3) {
  uint32_t r;
  asm("{\n.reg .b16 lo, hi;\n"
      "cvt.rn.satfinite.e4m3x2.f32 lo, %2, %1;\n"
      "cvt.rn.satfinite.e4m3x2.f32 hi, %4, %3;\n"
      "mov.b32 %0, {lo, hi};\n}\n"
      : "=r"(r)
      : "f"(a0), "f"(a1), "f"(a2), "f"(a3));
  return r;
}

// S accumulator fragment -> e4m3 A fragments of P V, one k32 step per 32-key block kb.  A register r holds K columns
// 16 (r >> 1) + 4 t4 + 0..3 of row g + 8 (r & 1); here they are filled with the S columns 8 nt + 2 t4 + {0, 1} of
// nt = 4 kb + 2 (r >> 1) and nt + 1 -- so K column k of block kb is key 32 kb + pi(k), the permutation vt is written in.
HI3D_DEVINL void fa8_pack(const float (&sc)[FA8_BN / 2], uint32_t (&pa)[FA8_BN / 32][4]) {
#pragma unroll
  for (int kb = 0; kb < FA8_BN / 32; kb++)
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int nt = 4 * kb + 2 * (r >> 1), hh = r & 1;
      pa[kb][r] = pack_e4m3x4(sc[4 * nt + 2 * hh], sc[4 * nt + 2 * hh + 1], sc[4 * nt + 4 + 2 * hh], sc[4 * nt + 5 + 2 * hh]);
    }
}

__global__ void __launch_bounds__(128 * (FA8_NC + 1), 1) fmha_fp8_kernel(const __grid_constant__ Fa8Params p) {
  constexpr int BN = FA8_BN, NC = FA8_NC, STAGES = FA8_STAGES;
  constexpr int BM = 64 * NC;                                // queries per CTA
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  const uint32_t sQ = base;                                  // NC slots of FA8_QSLOT
  const uint32_t sK = sQ + NC * FA8_QSLOT;                   // STAGES K tiles
  const uint32_t sV = sK + STAGES * FA8_KTILE;               // STAGES V tiles
  const uint32_t bar_q = sV + STAGES * FA8_VTILE;
  const uint32_t bar_kfull = bar_q + 8;                      // [STAGES] each: the producer's expect_tx arrive
  const uint32_t bar_vfull = bar_kfull + 8 * STAGES;
  const uint32_t bar_kempty = bar_vfull + 8 * STAGES;        // [STAGES] each: one arrive per consumer warp
  const uint32_t bar_vempty = bar_kempty + 8 * STAGES;

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
    setmaxnreg_dec<24>();
    if (tid == 0) {
      const int vrow = (blockIdx.z * gridDim.y + h) * 64;    // this (image, head)'s 64 rows of vt
      mbar_expect_tx(bar_q, NC * FA8_QTILE);
      for (int c = 0; c < NC; c++) tma_load_2d(sQ + c * FA8_QSLOT, &p.q_map, bar_q, h * 64, row0 + q0 + 64 * c);
      uint32_t ks = 0, kph = 0, vs = 0, vph = 0;
      auto load_k = [&](int j) {
        mbar_wait(bar_kempty + 8 * ks, kph ^ 1);
        mbar_expect_tx(bar_kfull + 8 * ks, FA8_KTILE);
        tma_load_2d(sK + ks * FA8_KTILE, &p.k_map, bar_kfull + 8 * ks, C + h * 64, row0 + j * BN);
        if (++ks == (uint32_t)STAGES) { ks = 0; kph ^= 1; }
      };
      load_k(0);
      for (int j = 0; j < nkv; j++) {
        if (j + 1 < nkv) load_k(j + 1);
        mbar_wait(bar_vempty + 8 * vs, vph ^ 1);
        mbar_expect_tx(bar_vfull + 8 * vs, FA8_VTILE);
        tma_load_2d(sV + vs * FA8_VTILE, &p.v_map, bar_vfull + 8 * vs, j * BN, vrow);
        if (++vs == (uint32_t)STAGES) { vs = 0; vph ^= 1; }
      }
    }
    return;
  }

  // ======================= consumers: warpgroup cw owns query rows 64 cw .. + 63 of the CTA's tile
  setmaxnreg_inc<240>();
  const int cw = wg - 1;
  const int warp = (tid >> 5) & 3;
  // O in fp32 registers; each tile's P V is a fresh wgmma accumulator folded into it.  FP8 wgmma adds its products into the
  // accumulator with reduced precision, relative to the accumulator's magnitude: chained over all L keys, the late tiles'
  // products lose bits against the running sum (O came out up to 9 % small at L = 4096 when attention is spread wide).
  float o[32], pv[32];
#pragma unroll
  for (int i = 0; i < 32; i++) o[i] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f}, corr[2];
  const int t4 = lane & 3;
  const float c = p.scale_log2;
  const uint64_t qd = gmma_desc_sw64(sQ + cw * FA8_QSLOT);
  float sc[BN / 2];
  uint32_t pa[BN / 32][4];
  uint32_t ks = 0, kph = 0, vs = 0, vph = 0;
  auto issue_s = [&]() {       // S = Q K^T on K stage ks: two k32 steps of 32 bytes (+2 in the descriptors)
    const uint64_t kd = gmma_desc_sw64(sK + ks * FA8_KTILE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 2; k++) wgmma_ss_e4m3<BN>(sc, qd + (uint64_t)(2 * k), kd + (uint64_t)(2 * k), k);
    wgmma_commit();
  };
  auto issue_pv = [&]() {      // pv = P V on V stage vs: one k32 step per 32 keys, 32 bytes along vt's key rows
    const uint64_t vd = gmma_desc_sw128(sV + vs * FA8_VTILE);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < BN / 32; kb++) wgmma_rs_e4m3_64(pv, pa[kb], vd + (uint64_t)(2 * kb), kb);
    wgmma_commit();
  };
  auto release = [&](uint32_t bar, uint32_t& s, uint32_t& ph) {
    __syncwarp();
    if (lane == 0) mbar_arrive(bar + 8 * s);
    if (++s == (uint32_t)STAGES) { s = 0; ph ^= 1; }
  };
  auto add_pv = [&](float c0, float c1) {      // O = O * (rescale to the tile's running max) + P V
#pragma unroll
    for (int dt = 0; dt < 8; dt++) {
      o[4 * dt] = fmaf(o[4 * dt], c0, pv[4 * dt]);
      o[4 * dt + 1] = fmaf(o[4 * dt + 1], c0, pv[4 * dt + 1]);
      o[4 * dt + 2] = fmaf(o[4 * dt + 2], c1, pv[4 * dt + 2]);
      o[4 * dt + 3] = fmaf(o[4 * dt + 3], c1, pv[4 * dt + 3]);
    }
  };

  mbar_wait(bar_q, 0);
  mbar_wait(bar_kfull, 0);
  issue_s();
  wgmma_wait<0>();
  wgmma_fence_regs(sc);
  release(bar_kempty, ks, kph);
  fa_softmax<BN, FA8_EMU8, FA8_PLOG2>(sc, mrow, lrow, corr, 0, p.L, c, t4);
  fa8_pack(sc, pa);
  for (int j = 1; j < nkv; j++) {
    mbar_wait(bar_kfull + 8 * ks, kph);
    issue_s();                                  // S_j
    mbar_wait(bar_vfull + 8 * vs, vph);
    issue_pv();                                 // pv = P_{j-1} V_{j-1}
    const float c0 = corr[0], c1 = corr[1];     // to tile j - 1's running max
    wgmma_wait<1>();                            // S_j has retired, P V may still run
    wgmma_fence_regs(sc);
    release(bar_kempty, ks, kph);
    fa_softmax<BN, FA8_EMU8, FA8_PLOG2>(sc, mrow, lrow, corr, j, p.L, c, t4);
    wgmma_wait<0>();
    wgmma_fence_regs(pv);
    release(bar_vempty, vs, vph);
    add_pv(c0, c1);
    fa8_pack(sc, pa);
  }
  mbar_wait(bar_vfull + 8 * vs, vph);
  issue_pv();
  wgmma_wait<0>();
  wgmma_fence_regs(pv);
  add_pv(corr[0], corr[1]);

  // ---- finalize: O /= l (both carry the 2^8 of P), stage through this warpgroup's own Q slot (only its own S products read
  // it), 16-byte stores of the rows < L
  const int g = lane >> 2;
  uint8_t* stage = smem + cw * FA8_QSLOT;
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

// Position of key q (0 .. 31) inside its 32-block of vt: the inverse of pi(k) = (k & 16) + 8 ((k >> 1) & 1) + 2 ((k >> 2) & 3) + (k & 1).
HI3D_DEVINL int vt_slot(int q) { return (q & 16) + 4 * ((q >> 1) & 3) + 2 * ((q >> 3) & 1) + (q & 1); }

// One CTA per (128-key tile, head, image): the tile's V block [128 keys, 64] is read with 16-byte loads (zeros past L),
// scattered byte-wise into a [64, 128] shared tile at the permuted key positions, and written out as 128-byte rows.
__global__ void __launch_bounds__(128) vt_e4m3_kernel(const uint8_t* __restrict__ qkv8, int L, int heads, int Lp,
                                                      uint8_t* __restrict__ vt) {
  __shared__ __align__(16) uint8_t sT[64][FA8_VT_KEYS + 16];   // 144-byte rows: 16-byte aligned, fewer bank conflicts
  const int tile = blockIdx.x, h = blockIdx.y, img = blockIdx.z, tid = threadIdx.x;
  const long long ld = 3LL * heads * 64;
  const uint8_t* src = qkv8 + (long long)img * L * ld + 2LL * heads * 64 + h * 64;
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int i = tid + 128 * r, key = i >> 2, c = i & 3;
    const int gk = tile * FA8_VT_KEYS + key;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (gk < L) v = *reinterpret_cast<const uint4*>(src + gk * ld + 16 * c);
    const int pos = (key & ~31) | vt_slot(key & 31);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 16; e++) sT[16 * c + e][pos] = (uint8_t)(w[e >> 2] >> (8 * (e & 3)));
  }
  __syncthreads();
  uint8_t* dst = vt + (long long)(img * heads + h) * 64 * Lp + tile * FA8_VT_KEYS;
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int i = tid + 128 * r, d = i >> 3, ch = i & 7;
    *reinterpret_cast<uint4*>(dst + (long long)d * Lp + 16 * ch) = *reinterpret_cast<const uint4*>(&sT[d][16 * ch]);
  }
}

static int vt_keys(int L) { return (L + FA8_VT_KEYS - 1) / FA8_VT_KEYS * FA8_VT_KEYS; }

}  // namespace hi3d

using namespace hi3d;

extern "C" int64_t hi3d_attention_vt_e4m3_bytes(int n_img, int L, int heads) {
  if (n_img <= 0 || L <= 0 || heads <= 0) {
    set_error("hi3d_attention_vt_e4m3_bytes: bad arguments (n_img=%d L=%d heads=%d)", n_img, L, heads);
    return -2;
  }
  return (int64_t)n_img * heads * 64 * vt_keys(L);
}

extern "C" int hi3d_attention_vt_e4m3(const void* qkv8, int n_img, int L, int heads, void* vt, void* stream) {
  if (!qkv8 || !vt || n_img <= 0 || L <= 0 || heads <= 0 || ((uintptr_t)qkv8 & 15) || ((uintptr_t)vt & 15)) {
    set_error("hi3d_attention_vt_e4m3: bad arguments (n_img=%d L=%d heads=%d)", n_img, L, heads);
    return -2;
  }
  if (heads > 65535 || n_img > 65535) { set_error("hi3d_attention_vt_e4m3: grid too large"); return -2; }
  const int Lp = vt_keys(L);
  dim3 grid(Lp / FA8_VT_KEYS, heads, n_img);
  vt_e4m3_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const uint8_t*)qkv8, L, heads, Lp, (uint8_t*)vt);
  return check_launch("hi3d_attention_vt_e4m3");
}

extern "C" int hi3d_attention_d64_tc5_fp8(const void* qkv8, const void* vt, int n_img, int L, int heads, float scale, void* out,
                                          void* stream) {
  if (!qkv8 || !vt || !out || n_img <= 0 || L <= 0 || heads <= 0 || ((uintptr_t)qkv8 & 15) || ((uintptr_t)vt & 15) ||
      ((uintptr_t)out & 15)) {
    set_error("hi3d_attention_d64_tc5_fp8: bad arguments (n_img=%d L=%d heads=%d)", n_img, L, heads);
    return -2;
  }
  if (heads > 65535 || n_img > 65535 || (int64_t)n_img * heads * 64 > 0x7fffffff) {
    set_error("hi3d_attention_d64_tc5_fp8: grid too large");
    return -2;
  }
  Fa8Params fp;
  memset(&fp, 0, sizeof(fp));
  fp.L = L;
  fp.C = heads * 64;
  fp.scale_log2 = scale * 1.4426950408889634f;
  fp.out = (__half*)out;
  {
    cuuint64_t dims[2] = {(cuuint64_t)(3 * fp.C), (cuuint64_t)n_img * (cuuint64_t)L};
    cuuint64_t str[1] = {(cuuint64_t)(3 * fp.C)};
    cuuint32_t box[2] = {64, 64};
    if (encode_map(&fp.q_map, qkv8, 2, dims, str, box, nullptr, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return -1;
    box[1] = FA8_BN;
    if (encode_map(&fp.k_map, qkv8, 2, dims, str, box, nullptr, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return -1;
    const int Lp = vt_keys(L);
    cuuint64_t vdims[2] = {(cuuint64_t)Lp, (cuuint64_t)n_img * heads * 64};
    cuuint64_t vstr[1] = {(cuuint64_t)Lp};
    cuuint32_t vbox[2] = {FA8_BN, 64};
    if (encode_map(&fp.v_map, vt, 2, vdims, vstr, vbox, nullptr, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_UINT8))
      return -1;
  }
  constexpr int bars = 8 + 4 * 8 * FA8_STAGES;
  constexpr int smem = FA8_NC * FA8_QSLOT + FA8_STAGES * (FA8_KTILE + FA8_VTILE) + bars + 1024;
  static bool attr_done[HI3D_MAX_DEVICES];
  if (ensure_dyn_smem(fmha_fp8_kernel, smem, attr_done, "hi3d_attention_d64_tc5_fp8")) return -1;
  dim3 grid((L + 64 * FA8_NC - 1) / (64 * FA8_NC), heads, n_img);
  fmha_fp8_kernel<<<grid, 128 * (FA8_NC + 1), smem, (cudaStream_t)stream>>>(fp);
  return check_launch("hi3d_attention_d64_tc5_fp8");
}
