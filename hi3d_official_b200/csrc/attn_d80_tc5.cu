// Self-attention core for head dim 80 (OpenCLIP ViT-H/14: width 1280 = 16 heads x 80) on Hopper: the d = 64 kernel of
// attn_tc5.cu (TMA through an mbarrier ring, S = Q K^T and O += P V on wgmma, P fed back from registers) with the head
// dimension split 64 + 16.
//
// Staging: an 80-column fp16 row is 160 B, more than one 128-byte swizzle span.  Each Q / K / V tile is therefore loaded as
// two TMA boxes from the same tensor map geometry: columns 0..63 as a 64-column SWIZZLE_128B box (128-B rows) and columns
// 64..79 as a 16-column SWIZZLE_32B box (32-B rows).  Nothing is padded in memory or in shared memory.
//   S = Q K^T: four k16 steps on the 128-B tiles, the fifth on the 32-B tiles (one 32-B row = one k16 step).
//   O += P V : an m64n64 product on the 128-B V tile and an m64n16 product on the 32-B V tile, into two accumulators.
//
// CTA = 128 queries x one (image, head), two warpgroups of 64 query rows; keys stream in tiles of 64.  The key tail (L not a
// multiple of 64: keys of the next image or TMA out-of-bounds zeros) is masked to -inf; query rows past L are not stored.
#include <cuda.h>
#include <string.h>

#include "common.cuh"
#include "tc5.cuh"

namespace hi3d {

constexpr int D80_BM = 128;                  // queries per CTA
constexpr int D80_BN = 64;                   // keys per ring stage
constexpr int D80_STAGES = 3;                // ViT sequences are short (257 tokens = 5 key tiles)
constexpr int D80_THREADS = 256;
constexpr int D80_T64 = 64 * 128;            // 64 rows x 64 fp16, SWIZZLE_128B
constexpr int D80_T16 = 64 * 32;             // 64 rows x 16 fp16, SWIZZLE_32B
constexpr int D80_QWG = D80_T64 + D80_T16;   // one warpgroup's Q rows (10240 B; also its output staging area)
constexpr int D80_STAGE = 2 * D80_T64 + 2 * D80_T16;   // K64 | V64 | K16 | V16
constexpr int D80_SMEM = 2 * D80_QWG + D80_STAGES * D80_STAGE + 8 + 16 * D80_STAGES + 1024;

struct D80Params {
  CUtensorMap map64;       // [n_img * L, 3C] fp16 (q | k | v), box {64, 64}, SWIZZLE_128B
  CUtensorMap map16;       // the same matrix, box {16, 64}, SWIZZLE_32B
  int L, C;
  float scale_log2;
  __half* out;             // [n_img * L, C]
};

__global__ void __launch_bounds__(D80_THREADS, 1) fmha_d80_tc5_kernel(const __grid_constant__ D80Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  const uint32_t sQ = base;                                   // per warpgroup: [64 x 64] sw128 then [64 x 16] sw32
  const uint32_t sR = base + 2 * D80_QWG;                     // ring of D80_STAGES stages
  const uint32_t bar_q = sR + D80_STAGES * D80_STAGE;
  const uint32_t bar_full = bar_q + 8;                        // [D80_STAGES]
  const uint32_t bar_empty = bar_full + 8 * D80_STAGES;       // [D80_STAGES], one arrive per warp

  const int tid = threadIdx.x, lane = tid & 31;
  const int cw = tid >> 7;                                    // warpgroup: query rows 64 cw .. + 63
  const int warp = (tid >> 5) & 3;
  const int q0 = blockIdx.x * D80_BM;
  const int h = blockIdx.y;
  const int row0 = blockIdx.z * p.L;
  const int nkv = (p.L + D80_BN - 1) / D80_BN;
  const int C = p.C;

  auto issue_kv = [&](int j, int s) {
    const uint32_t full = bar_full + 8 * s, st = sR + s * D80_STAGE;
    const int r = row0 + j * D80_BN;
    mbar_expect_tx(full, D80_STAGE);
    tma_load_2d(st, &p.map64, full, C + h * 80, r);
    tma_load_2d(st + D80_T64, &p.map64, full, 2 * C + h * 80, r);
    tma_load_2d(st + 2 * D80_T64, &p.map16, full, C + h * 80 + 64, r);
    tma_load_2d(st + 2 * D80_T64 + D80_T16, &p.map16, full, 2 * C + h * 80 + 64, r);
  };
  if (tid == 0) {
    mbar_init(bar_q, 1);
    for (int s = 0; s < D80_STAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    mbar_expect_tx(bar_q, 2 * D80_QWG);
    for (int w = 0; w < 2; w++) {
      tma_load_2d(sQ + w * D80_QWG, &p.map64, bar_q, h * 80, row0 + q0 + 64 * w);
      tma_load_2d(sQ + w * D80_QWG + D80_T64, &p.map16, bar_q, h * 80 + 64, row0 + q0 + 64 * w);
    }
    for (int j = 0; j < D80_STAGES && j < nkv; j++) issue_kv(j, j);
  }
  __syncthreads();

  float o[32], o16[8];
#pragma unroll
  for (int i = 0; i < 32; i++) o[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; i++) o16[i] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const int t4 = lane & 3;
  const float c = p.scale_log2;
  const uint64_t qd = gmma_desc_sw128(sQ + cw * D80_QWG);
  const uint64_t qd16 = gmma_desc_sw32(sQ + cw * D80_QWG + D80_T64 + 0);
  mbar_wait(bar_q, 0);

  uint32_t s = 0, ph = 0;
  for (int j = 0; j < nkv; j++) {
    mbar_wait(bar_full + 8 * s, ph);
    const uint32_t st = sR + s * D80_STAGE;
    // ---- S = Q K^T: head columns 0..63 in four k16 steps, 64..79 in a fifth ----
    float sc[D80_BN / 2];
    const uint64_t kd = gmma_desc_sw128(st);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) wgmma_ss<D80_BN>(sc, qd + (uint64_t)(2 * k), kd + (uint64_t)(2 * k), k);
    wgmma_ss<D80_BN>(sc, qd16, gmma_desc_sw32(st + 2 * D80_T64), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    // ---- mask the key tail ----
    if ((j + 1) * D80_BN > p.L) {
#pragma unroll
      for (int nt = 0; nt < D80_BN / 8; nt++) {
        const int col = j * D80_BN + nt * 8 + 2 * t4;
        if (col >= p.L) { sc[4 * nt] = -INFINITY; sc[4 * nt + 2] = -INFINITY; }
        if (col + 1 >= p.L) { sc[4 * nt + 1] = -INFINITY; sc[4 * nt + 3] = -INFINITY; }
      }
    }
    // ---- online softmax: this thread holds rows g (hh = 0) and g + 8 (hh = 1) of its warp's 16 rows ----
    uint32_t pa[D80_BN / 16][4];
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < D80_BN / 8; nt++) mx = fmaxf(mx, fmaxf(sc[4 * nt + 2 * hh], sc[4 * nt + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mnew = fmaxf(mrow[hh], mx);
      const float corr = exp2f((mrow[hh] - mnew) * c);
      const float moff = mnew * c;
      float rs = 0.f;
#pragma unroll
      for (int nt = 0; nt < D80_BN / 8; nt++) {
        const float p0 = exp2f(sc[4 * nt + 2 * hh] * c - moff), p1 = exp2f(sc[4 * nt + 2 * hh + 1] * c - moff);
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
#pragma unroll
      for (int dt = 0; dt < 2; dt++) {
        o16[4 * dt + 2 * hh] *= corr;
        o16[4 * dt + 2 * hh + 1] *= corr;
      }
    }
    // ---- O += P V: 16 keys per MMA (V64 advances 16 rows = 2048 B, V16 16 rows = 512 B) ----
    const uint64_t vd = gmma_desc_sw128(st + D80_T64);
    const uint64_t vd16 = gmma_desc_sw32(st + 2 * D80_T64 + D80_T16);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D80_BN / 16; kk++) {
      wgmma_rs_tb<64>(o, pa[kk], vd + (uint64_t)(128 * kk), 1);
      wgmma_rs_tb<16>(o16, pa[kk], vd16 + (uint64_t)(32 * kk), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    wgmma_fence_regs(o16);
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
    if (tid == 0 && j + D80_STAGES < nkv) {
      mbar_wait(bar_empty + 8 * s, ph);          // both warpgroups are done with this stage
      issue_kv(j + D80_STAGES, s);
    }
    if (++s == (uint32_t)D80_STAGES) { s = 0; ph ^= 1; }
  }

  // ---- finalize: O /= l, staged as plain [16 rows x 80] per warp in this warpgroup's Q area, 16-byte stores ----
  named_bar_sync(1 + cw, 128);                   // no MMA of this warpgroup reads its Q rows any more
  const int g = lane >> 2;
  uint8_t* stage = smem + cw * D80_QWG + warp * (16 * 160);
#pragma unroll
  for (int hh = 0; hh < 2; hh++) {
    float l = lrow[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    uint8_t* rowp = stage + (g + 8 * hh) * 160 + t4 * 4;
#pragma unroll
    for (int dt = 0; dt < 8; dt++)
      *reinterpret_cast<uint32_t*>(rowp + dt * 16) = pack_half2(o[4 * dt + 2 * hh] * inv, o[4 * dt + 2 * hh + 1] * inv);
#pragma unroll
    for (int dt = 0; dt < 2; dt++)
      *reinterpret_cast<uint32_t*>(rowp + 128 + dt * 16) =
          pack_half2(o16[4 * dt + 2 * hh] * inv, o16[4 * dt + 2 * hh + 1] * inv);
  }
  __syncwarp();
  __half* obase = p.out + (long long)row0 * C + h * 80;
#pragma unroll
  for (int i = 0; i < 5; i++) {                  // 16 rows x 10 chunks of 16 B
    const int idx = lane + 32 * i;
    const int r = idx / 10, ch = idx - r * 10;
    const int q = q0 + cw * 64 + warp * 16 + r;
    if (q < p.L)
      *reinterpret_cast<uint4*>(obase + (long long)q * C + ch * 8) = *reinterpret_cast<const uint4*>(stage + r * 160 + ch * 16);
  }
}

}  // namespace hi3d

using namespace hi3d;

extern "C" int hi3d_attention_d80_tc5(const void* qkv, int n_img, int L, int heads, float scale, void* out, void* stream) {
  if (!qkv || !out || n_img <= 0 || L <= 0 || heads <= 0 || ((uintptr_t)qkv & 15) || ((uintptr_t)out & 15)) {
    set_error("hi3d_attention_d80_tc5: bad arguments (n_img=%d L=%d heads=%d)", n_img, L, heads);
    return -2;
  }
  if (heads > 65535 || n_img > 65535) { set_error("hi3d_attention_d80_tc5: grid too large"); return -2; }
  D80Params fp;
  memset(&fp, 0, sizeof(fp));
  fp.L = L;
  fp.C = heads * 80;
  fp.scale_log2 = scale * 1.4426950408889634f;
  fp.out = (__half*)out;
  cuuint64_t dims[2] = {(cuuint64_t)(3 * fp.C), (cuuint64_t)n_img * (cuuint64_t)L};
  cuuint64_t str[1] = {(cuuint64_t)(3 * fp.C) * 2};
  cuuint32_t box[2] = {64, 64};
  if (encode_map(&fp.map64, qkv, 2, dims, str, box, nullptr)) return -1;
  box[0] = 16;
  if (encode_map(&fp.map16, qkv, 2, dims, str, box, nullptr, CU_TENSOR_MAP_SWIZZLE_32B)) return -1;
  static bool attr_done[HI3D_MAX_DEVICES];
  if (ensure_dyn_smem(fmha_d80_tc5_kernel, D80_SMEM, attr_done, "hi3d_attention_d80_tc5")) return -1;
  dim3 grid((L + D80_BM - 1) / D80_BM, heads, n_img);
  fmha_d80_tc5_kernel<<<grid, D80_THREADS, D80_SMEM, (cudaStream_t)stream>>>(fp);
  return check_launch("hi3d_attention_d80_tc5");
}
