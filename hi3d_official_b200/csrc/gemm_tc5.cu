// Implicit-GEMM engine, Hopper-native variant: TMA (cp.async.bulk.tensor) operand staging into SWIZZLE_128B shared
// tiles through an mbarrier ring, wgmma (warpgroup MMA, fp32 accumulators in registers) on the tiles in place, and an
// epilogue staged through shared memory for coalesced 16-byte stores.  Same contract as hi3d_gemm (include/hi3d_b200.h);
// geometries this engine does not cover (upsample-fused convs, odd patch shapes, N < 32, > 4 distinct A sources) are
// forwarded to the mma.sync engine.
//
// The 128 rows of a tile are
//   PLAIN    : 128 consecutive rows
//   CONV2D   : a (tn images) x (th rows) x (tw columns) patch, tn*th*tw = 128 -- the 3x3 taps are the same TMA box
//              shifted by (dy, dx) and the zero padding is TMA out-of-bounds fill (stride 2: TMA element strides)
//   TEMPORAL : (tf frames) x (ts pixels), tf*ts = 128 -- the temporal taps shift the frame coordinate of a
//              [C, HW, T, B] view; clip boundaries zero-fill by OOB.
// Tiles are ordered n-tile fastest, so that CTAs running together share A rows through L2.  Two schedules share the TMA
// producer (t5_produce), the row mappings and the epilogue arithmetic (a register pass into a staging tile, then the GELU
// family, residual and blend on 16-byte chunks of it):
//
// gemm_tc5_kernel -- one CTA per 128 x BN output tile (BN in {64, 128, 192, 256}, chosen per call to cover N with the least
// padding and wave quantisation over the SMs).  Warp roles (128 + 256 NT threads): warpgroup 0 = TMA producer (one elected
// thread), then two MMA + epilogue warpgroups per 128-row tile (rows 0..63 and 64..127); the epilogue runs after the main loop,
// in the ring.  NT = 2 ("tile pairs", 16 epilogue warps) puts two consecutive row tiles in one CTA that share every B tile --
// half the B bytes from L2 per output row, for long-K shapes -- and is built for BN <= 128 (the register budget of 640
// threads).  The producer hands its registers to the MMA warpgroups (setmaxnreg): a 64 x 256 fp32 accumulator is 128
// registers per thread.
//
// gemm_tc5_pingpong_kernel -- fp16, short K: a persistent grid of min(tiles, SMs) CTAs; one producer fills one ring across all
// of a CTA's tiles, and two consumer warpgroups take its tiles in turn, each owning a whole 128 x BN tile (BN in {64, 128}) and
// its own staging tile.  Their MMA turns alternate, so one warpgroup's epilogue runs while the other's main loop has the tensor
// cores.  With K short the epilogue is as long as the main loop, and the single-tile kernel leaves the tensor cores idle for it.
// Its epilogue is specialised at compile time (GEGLU, residual / blend) and its staged tiles leave by TMA stores.
//
// Selection (tc5_choose, the only place): an fp16 GEMM with K <= 64 T5_PINGPONG_MAX_KT, M >= 128, at least one tile per SM and
// not GEGLU together with a residual or blend runs ping-pong; otherwise tile pairs for K >= 1920 with 4 pair tiles per SM, else
// single tiles.  The hooks hi3d_gemm_tc5_set_pair_mode / set_epilogue_warps force single tiles or pairs, and
// hi3d_gemm_tc5_schedule reports the choice.
// The kernels are templated on the operand type: hi3d_gemm_tc5 runs fp16 operands and hi3d_gemm_tc5_fp8 e4m3 ones (wgmma k32,
// SWIZZLE_64B stages, a per-column weight scale on the fp32 accumulator and an optional e4m3 output).  The e4m3 path keeps the
// single-tile / pair schedule: its chained accumulation (`part`, see T5_PROMOTE) needs registers beside the accumulator that a
// 128 x 128 consumer tile does not leave.
#include <cuda.h>
#include <cuda_fp8.h>
#include <stdlib.h>
#include <string.h>
#include <type_traits>

#include "common.cuh"
#include "tc5.cuh"

namespace hi3d {
int validate_gemm(const hi3d_gemm_params* p, const char* who);

constexpr int T5_BM = 128;
constexpr int T5_BK = 64;
constexpr int T5_MAX_MAPS = 4;
constexpr int T5_SMEM_BUDGET = 200 * 1024;

// Operand types.  fp16: a stage holds 64-element K rows of 128 bytes under SWIZZLE_128B, four k16 MMAs per stage.  e4m3: 64-element
// K rows of 64 bytes under SWIZZLE_64B (segment channel counts are multiples of 64, not of 128), two k32 MMAs per stage; the
// stages are half the bytes, so twice as many fit the same shared memory.
template <typename Op> struct T5Op;
template <> struct T5Op<__half> {
  static constexpr int ROW = 128, MAX_STAGES = 8;
  static constexpr CUtensorMapDataType DT = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  static constexpr CUtensorMapSwizzle SW = CU_TENSOR_MAP_SWIZZLE_128B;
};
template <> struct T5Op<__nv_fp8_e4m3> {
  static constexpr int ROW = 64, MAX_STAGES = 16;
  static constexpr CUtensorMapDataType DT = CU_TENSOR_MAP_DATA_TYPE_UINT8;
  static constexpr CUtensorMapSwizzle SW = CU_TENSOR_MAP_SWIZZLE_64B;
};

// FP8 accumulation: a wgmma chain covers T5_PROMOTE k-tiles (128 K elements, 4 k32 steps) before it is added into fp32
// registers.  Of 2, 4 and 8 k-tiles, 2 measured both the most accurate and the fastest (8 holds the whole ring of 8 stages).
// The chain runs on CW-column slices of the tile: the whole tile where the accumulator and the chain's registers fit the 168
// registers of the single-tile kernels (BN <= 128) or the pair kernel's 96 (BN = 64), else half of it (BN = 192) or 32 columns
// (BN = 256, and pairs at BN = 128).
constexpr int T5_PROMOTE = 2;
template <int BN, int NT> struct T5PromoteCols {
  static constexpr int value = NT == 2 ? (BN == 128 ? 32 : BN) : (BN == 192 ? 96 : (BN == 256 ? 32 : BN));
};

struct T5Seg {
  int map;       // index into amap[]
  int c_off, C;  // channel range
  int dy, dx, dt;
};

struct T5Params {
  CUtensorMap bmap;
  CUtensorMap amap[T5_MAX_MAPS];
  CUtensorMap omap;   // ping-pong schedule: the output tile's TMA store boxes (see t5_encode_out_map)
  T5Seg seg[HI3D_MAX_SEGS];
  int nseg;
  int M, N, K, mode;
  int stages, n_tiles, m_tiles;   // m_tiles: row tiles (ping-pong schedule's persistent grid)
  // tile -> rows
  int tw, th, tn;      // CONV2D patch (PLAIN: tw = 128, th = tn = 1; TEMPORAL: tw = ts, th = tf)
  int Wo, Ho, Nimg;    // CONV2D: output W, H, images.  TEMPORAL: Wo = HW, Ho = T, Nimg = B
  int tiles_x, tiles_y;  // tiles along W and H (CONV2D) / along HW and T (TEMPORAL)
  int cstride;           // CONV2D input stride (1 | 2): TMA element strides, box origin = tile origin * cstride + tap
  int out_up, out_py, out_px;   // parity-class output mapping (see hi3d_gemm_params::out_up)
  int t_off;                    // TEMPORAL: frame offset of output frame 0 inside the (haloed) source clip
  // epilogue
  const float* bias;
  const __half* rowbias;
  int rb_div, rb_mod, rb_ld, act;
  const __half* residual;
  int res_ld;
  const __half* blend_x;
  int blend_ld;
  float alpha;
  __half* out;
  int out_ld;
  const float* w_scale;   // e4m3 operands: per-column dequantisation scale of W, applied to the accumulator first
  int out_fp8;            // e4m3 operands: 1 -> out is e4m3 [M, out_ld]
};

struct T5Tile {
  int x0, y0, z0;   // TMA origin coordinates (CONV2D: x, y, image; TEMPORAL: pixel, frame, clip)
};

HI3D_DEVINL T5Tile t5_origin(const T5Params& p, int mt) {
  T5Tile t{0, 0, 0};
  if (p.mode != HI3D_ROWS_PLAIN) {
    const int tx = mt % p.tiles_x, rest = mt / p.tiles_x;
    t.x0 = tx * p.tw;
    t.y0 = (rest % p.tiles_y) * p.th;
    t.z0 = (rest / p.tiles_y) * p.tn;
  }
  return t;
}
// tile-local row -> global output row (or -1)
HI3D_DEVINL long long t5_row(const T5Params& p, int mt, const T5Tile& o, int r) {
  if (p.mode == HI3D_ROWS_PLAIN) {
    const long long m = (long long)mt * T5_BM + r;
    return m < p.M ? m : -1;
  }
  const int x = o.x0 + r % p.tw;
  const int y = o.y0 + (r / p.tw) % p.th;
  const int n = o.z0 + r / (p.tw * p.th);
  if (x >= p.Wo || y >= p.Ho || n >= p.Nimg) return -1;
  return ((long long)n * p.Ho + y) * p.Wo + x;
}

// The TMA producer's k-loop over one CTA tile (NT row tiles from mt0, origins o, columns from n0).  The whole calling warp walks
// the loop with warp-uniform values and one lane issues.  s / ph: ring position and phase, carried from one tile to the next by
// the persistent kernel.
template <int BN, int NT, typename Op>
HI3D_DEVINL void t5_produce(const T5Params& p, uint32_t base, uint32_t bar_full, uint32_t bar_empty, int mt0,
                            const T5Tile (&o)[NT], int n0, uint32_t& s, uint32_t& ph) {
  constexpr int ROW = T5Op<Op>::ROW;
  constexpr int A_BYTES = T5_BM * ROW;
  constexpr uint32_t stage_bytes = NT * A_BYTES + BN * ROW;
  const int lane = threadIdx.x & 31, KT = p.K / T5_BK, STAGES = p.stages;
  int si = 0, so = 0;
  T5Seg sg = p.seg[0];
  const CUtensorMap* am = &p.amap[sg.map];
  for (int kt = 0; kt < KT; kt++) {
    mbar_wait(bar_empty + 8 * s, ph ^ 1);
    if (lane == 0) {
      const uint32_t sB = base + s * stage_bytes + NT * A_BYTES;
      const uint32_t full = bar_full + 8 * s;
      const int c = sg.c_off + so;
      mbar_expect_tx(full, stage_bytes);
      // a second row tile past the last one loads out of bounds (zeros) and stores nothing
#pragma unroll
      for (int t = 0; t < NT; t++) {
        const uint32_t sA = base + s * stage_bytes + t * A_BYTES;
        if (p.mode == HI3D_ROWS_PLAIN)
          tma_load_2d(sA, am, full, c, (mt0 + t) * T5_BM);
        else if (p.mode == HI3D_ROWS_CONV2D)
          tma_load_4d(sA, am, full, c, o[t].x0 * p.cstride + sg.dx, o[t].y0 * p.cstride + sg.dy, o[t].z0);
        else
          tma_load_4d(sA, am, full, c, o[t].x0, o[t].y0 + p.t_off + sg.dt, o[t].z0);
      }
      tma_load_2d(sB, &p.bmap, full, kt * T5_BK, n0);
    }
    __syncwarp();
    so += T5_BK;
    if (so >= sg.C && kt + 1 < KT) { si++; so = 0; sg = p.seg[si]; am = &p.amap[sg.map]; }
    if (++s == (uint32_t)STAGES) { s = 0; ph ^= 1; }
  }
}

// Epilogue phase 1 for one thread's share of a 64-row accumulator fragment (wgmma m64nBN layout): rows rl and rl + 8 of the
// staging tile sC (row pitch BN + 8 halfs), global rows m[0] / m[1] (-1 past the end), columns from n0.  In fp32: the e4m3 weight
// scale, bias, rowbias, then SiLU or GEGLU; one fp16 rounding into sC.
template <int BN, bool FP8>
HI3D_DEVINL void t5_stage(const T5Params& p, const float (&acc)[BN / 2], __half* sC, int rl, const long long (&m)[2], int n0) {
  constexpr int pitch = BN + 8;
  const bool geglu = (p.act == HI3D_ACT_GEGLU);
  const int t4 = threadIdx.x & 3;
#pragma unroll
  for (int hh = 0; hh < 2; hh++) {
    const int r = rl + 8 * hh;
    const __half* rbp = nullptr;
    if (p.rowbias != nullptr && m[hh] >= 0) rbp = p.rowbias + (long long)((m[hh] / p.rb_div) % p.rb_mod) * p.rb_ld;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
      const int cl = j * 8 + 2 * t4;
      const int n = n0 + cl;
      float v0 = acc[4 * j + 2 * hh], v1 = acc[4 * j + 2 * hh + 1];
      if (n < p.N) {
        if constexpr (FP8) {
          const float2 ws = __ldg(reinterpret_cast<const float2*>(p.w_scale + n));
          v0 *= ws.x;
          v1 *= ws.y;
        }
        if (p.bias != nullptr) {
          v0 += __ldg(p.bias + n);
          v1 += __ldg(p.bias + n + 1);
        }
        if (rbp != nullptr) {
          const __half2 rbv = *reinterpret_cast<const __half2*>(rbp + n);
          v0 += __low2float(rbv);
          v1 += __high2float(rbv);
        }
      }
      if (geglu) {
        sC[r * pitch + (cl >> 1)] = __float2half_rn(v0 * gelu_erf_f(v1));
      } else {
        if (p.act == HI3D_ACT_SILU) {
          v0 = silu_f(v0);
          v1 = silu_f(v1);
        }
        *reinterpret_cast<uint32_t*>(sC + r * pitch + cl) = pack_half2(v0, v1);
      }
    }
  }
}

// Epilogue phase 2, split so that a caller can issue the global loads of several chunks before their stores.  out may alias
// residual or blend_x element for element (an in-place residual add), never partially: a chunk is only read by its own loads.
// t5_out_row: the output row of global row m (differs from m only for the parity-class upsample convs).
HI3D_DEVINL long long t5_out_row(const T5Params& p, long long m) {
  if (!p.out_up) return m;
  const int hw = p.Ho * p.Wo;
  const int n_ = (int)(m / hw), rem_ = (int)(m - (long long)n_ * hw);
  const int y_ = rem_ / p.Wo, x_ = rem_ - y_ * p.Wo;
  return ((long long)n_ * 2 * p.Ho + 2 * y_ + p.out_py) * (2 * p.Wo) + 2 * x_ + p.out_px;
}
HI3D_DEVINL void t5_load_chunk(const T5Params& p, long long mo, int nc, Half8& rr, Half8& xx) {
  if (p.residual != nullptr) rr = *reinterpret_cast<const Half8*>(p.residual + mo * p.res_ld + nc);
  if (p.blend_x != nullptr) xx = *reinterpret_cast<const Half8*>(p.blend_x + mo * p.blend_ld + nc);
}
// Eight staged halfs v with their chunk's residual rr / blend xx: the GELU family, then the residual add, then the blend.
HI3D_DEVINL void t5_finish_half8(const T5Params& p, Half8& v, const Half8& rr, const Half8& xx) {
  if (p.act >= HI3D_ACT_GELU) store_act_half8(p.act, v);
  if (p.residual != nullptr) {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const float2 a = __half22float2(v.h[q]), b = __half22float2(rr.h[q]);
      v.h[q] = __floats2half2_rn(a.x + b.x, a.y + b.y);
    }
  }
  if (p.blend_x != nullptr) {
    const float al = p.alpha, be = 1.f - p.alpha;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const float2 a = __half22float2(v.h[q]), b = __half22float2(xx.h[q]);
      v.h[q] = __floats2half2_rn(al * b.x + be * a.x, al * b.y + be * a.y);
    }
  }
}
// The 8 staged halfs v of output row mo, columns nc .. nc + 7, finished as above; one coalesced store.
template <bool FP8>
HI3D_DEVINL void t5_finish_chunk(const T5Params& p, Half8 v, long long mo, int nc, const Half8& rr, const Half8& xx) {
  t5_finish_half8(p, v, rr, xx);
  if constexpr (FP8) {
    if (p.out_fp8) {
      *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(p.out) + mo * p.out_ld + nc) = half8_to_e4m3(v);
      return;
    }
  }
  *reinterpret_cast<Half8*>(p.out + mo * p.out_ld + nc) = v;
}
// One chunk: the 8 staged halfs v of global row m (>= 0), output columns nc .. nc + 7.
template <bool FP8>
HI3D_DEVINL void t5_store_chunk(const T5Params& p, Half8 v, long long m, int nc) {
  const long long mo = t5_out_row(p, m);
  Half8 rr, xx;
  t5_load_chunk(p, mo, nc, rr, xx);
  t5_finish_chunk<FP8>(p, v, mo, nc, rr, xx);
}

template <int BN, int NT, typename Op>
__global__ void __launch_bounds__(128 + 256 * NT, 1) gemm_tc5_kernel(const __grid_constant__ T5Params p) {
  constexpr bool FP8 = sizeof(Op) == 1;
  constexpr int ROW = T5Op<Op>::ROW;             // bytes of one 64-element K row of a stage
  constexpr int A_BYTES = T5_BM * ROW;
  constexpr int MMA_THREADS = 256 * NT;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;          // SWIZZLE_128B atoms need 1024-byte alignment
  uint8_t* smem = smem_raw + (base - raw);
  const int STAGES = p.stages;
  constexpr uint32_t stage_bytes = NT * A_BYTES + BN * ROW;
  const uint32_t bar_full = base + STAGES * stage_bytes;   // STAGES x 8
  const uint32_t bar_empty = bar_full + 8 * T5Op<Op>::MAX_STAGES;

  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);    // provably warp-uniform role index
  const int KT = p.K / T5_BK;
  const int nt = blockIdx.x % p.n_tiles, mt0 = (blockIdx.x / p.n_tiles) * NT;
  const int n0 = nt * BN;
  T5Tile o[NT];
#pragma unroll
  for (int t = 0; t < NT; t++) o[t] = t5_origin(p, mt0 + t);

  if (tid == 0) {
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar_full + 8 * s, 1);        // the producer's expect_tx arrive
      mbar_init(bar_empty + 8 * s, 8 * NT);  // one arrive per MMA warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ======================= TMA producer =======================
    if (NT == 1) setmaxnreg_dec<40>();
    if (tid < 32) {
      uint32_t s = 0, ph = 0;
      t5_produce<BN, NT, Op>(p, base, bar_full, bar_empty, mt0, o, n0, s, ph);
    }
    return;
  }

  // ======================= MMA warpgroups: rows 64 (wg - 1) .. + 63 of the CTA's 128 NT rows =======================
  // 384 threads x 168 registers: the producer's 128 x 128 released registers raise the MMA threads to 232.  The pair
  // kernel (640 threads) fits its 64 x 128 accumulators in the 96 registers it is launched with.
  if (NT == 1) setmaxnreg_inc<232>();
  const int cw = wg - 1;                 // MMA warpgroup index
  const int ct = cw >> 1;                // its row tile
  const int warp = (tid >> 5) & 3;       // warp inside the warpgroup: accumulator rows 16 warp .. + 15
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
  if constexpr (FP8) {
    // FP8 wgmma adds its products into the accumulator with reduced precision, relative to the accumulator's magnitude: one
    // chain over a long K loses the late products' low bits against the running sum (measured on an H100: up to 549 x 2^-10
    // sum |a w| at K = 23040 when one large product comes first).  So each chain covers T5_PROMOTE k-tiles in `part`, which is
    // then added into the fp32 `acc`.  A chain runs over a slice of CW of the tile's columns at a time, so that acc and part fit
    // the registers; the slicing does not change any column's arithmetic, and every tile width and pair mode computes the same
    // bits.
    constexpr int CW = T5PromoteCols<BN, NT>::value;
    float part[CW / 2];
    uint32_t s = 0, ph = 0;
    // one interval: NK k-tiles from stage s, chained per slice and added into acc; then its stages go back to the producer
    auto interval = [&](auto nk_) {
      constexpr int NK = decltype(nk_)::value;
      {
        uint32_t s1 = s, ph1 = ph;
#pragma unroll
        for (int i = 0; i < NK; i++) {
          mbar_wait(bar_full + 8 * s1, ph1);
          if (++s1 == (uint32_t)STAGES) { s1 = 0; ph1 ^= 1; }
        }
      }
#pragma unroll
      for (int c = 0; c < BN / CW; c++) {
        wgmma_fence();
        uint32_t s1 = s;
#pragma unroll
        for (int i = 0; i < NK; i++) {
          const uint64_t ad = gmma_desc_sw64(base + s1 * stage_bytes + cw * 64 * ROW);
          const uint64_t bd = gmma_desc_sw64(base + s1 * stage_bytes + NT * A_BYTES + c * CW * ROW);
#pragma unroll
          for (int k = 0; k < T5_BK / 32; k++)   // +32 bytes along K inside the 64-byte swizzle atom
            wgmma_ss_e4m3<CW>(part, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (i | k) ? 1 : 0);
          if (++s1 == (uint32_t)STAGES) s1 = 0;
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(part);
#pragma unroll
        for (int i = 0; i < CW / 2; i++) acc[c * (CW / 2) + i] += part[i];
      }
#pragma unroll
      for (int i = 0; i < NK; i++) {
        if (lane == 0) mbar_arrive(bar_empty + 8 * s);
        if (++s == (uint32_t)STAGES) { s = 0; ph ^= 1; }
      }
    };
    int kt = 0;
    for (; kt + T5_PROMOTE <= KT; kt += T5_PROMOTE) interval(std::integral_constant<int, T5_PROMOTE>());
    for (; kt < KT; kt++) interval(std::integral_constant<int, 1>());   // the last KT % T5_PROMOTE k-tiles one by one
  } else {
    uint32_t s = 0, ph = 0, ps = 0;
    for (int kt = 0; kt < KT; kt++) {
      mbar_wait(bar_full + 8 * s, ph);
      const uint32_t sA = base + s * stage_bytes + cw * 64 * ROW;
      const uint32_t sB = base + s * stage_bytes + NT * A_BYTES;
      wgmma_fence();
      {
        const uint64_t ad = gmma_desc_sw128(sA), bd = gmma_desc_sw128(sB);
#pragma unroll
        for (int k = 0; k < T5_BK / 16; k++)   // +32 bytes along K inside the 128-byte swizzle atom
          wgmma_ss<BN>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kt | k) ? 1 : 0);
      }
      wgmma_commit();
      // keep one k-block of MMAs in flight: the previous one has retired, its stage goes back to the producer
      wgmma_wait<1>();
      if (kt > 0 && lane == 0) mbar_arrive(bar_empty + 8 * ps);
      ps = s;
      if (++s == (uint32_t)STAGES) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
  }
  // every MMA of all MMA warpgroups has read its operands: the ring becomes the epilogue's staging tile
  named_bar_sync(1, MMA_THREADS);

  // ---- epilogue phase 1: registers -> (bias, rowbias, activation) -> fp16 staging tile in smem ----
  const bool geglu = (p.act == HI3D_ACT_GEGLU);
  const int BNo = geglu ? BN / 2 : BN;          // staged tile width
  constexpr int pitch = BN + 8;                 // halfs
  __half* sC = reinterpret_cast<__half*>(smem);
  {
    const int rl = cw * 64 + warp * 16 + (lane >> 2);
    const T5Tile oc = ct == 0 ? o[0] : o[NT - 1];    // no dynamic index: o stays in registers
    const long long m[2] = {t5_row(p, mt0 + ct, oc, rl - ct * T5_BM), t5_row(p, mt0 + ct, oc, rl + 8 - ct * T5_BM)};
    t5_stage<BN, FP8>(p, acc, sC, rl, m, n0);
  }
  named_bar_sync(1, MMA_THREADS);

  // ---- epilogue phase 2: coalesced 16-byte stores with residual / blend ---------------------------
  const int cpr = BNo / 8;  // 16-byte chunks per staged row
  const int Nout = geglu ? p.N / 2 : p.N;
  const int nout0 = geglu ? n0 / 2 : n0;
  const int et = tid - 128;
  for (int idx = et; idx < NT * T5_BM * cpr; idx += MMA_THREADS) {
    const int r = idx / cpr, c = idx - r * cpr;
    const int nc = nout0 + c * 8;
    if (nc >= Nout) continue;
    const int t = r / T5_BM;
    const T5Tile ot = t == 0 ? o[0] : o[NT - 1];   // no dynamic index: o stays in registers
    const long long m = t5_row(p, mt0 + t, ot, r - t * T5_BM);
    if (m < 0) continue;
    t5_store_chunk<FP8>(p, *reinterpret_cast<const Half8*>(sC + r * pitch + c * 8), m, nc);
  }
}

// Ping-pong schedule (fp16 operands, short K): a persistent grid whose CTA c takes tiles c, c + grid, c + 2 grid, ... (tile
// order as gemm_tc5_kernel's CTA order, n-tile fastest).  Warpgroup 0 is the TMA producer; it fills ONE ring in tile order and
// never drains it between tiles.  Consumer warpgroups 1 and 2 take the CTA's tiles in turn (local tile j -> warpgroup 1 + j % 2),
// each owning a whole 128 x BN tile as two m64 wgmma rows per k16 step (BN <= 128: 2 x BN / 2 accumulator registers), with its
// own staging tile outside the ring.  The MMA turns are ordered by a pair of named barriers: a warpgroup starts the main loop of
// its next tile only once the other one has issued the whole main loop of the tile before it.  So the main loop of tile j + 1
// runs on the tensor cores while the epilogue of tile j runs on the other warpgroup.  The ordering is also what keeps the ring's
// parity waits exact: every k-tile a warpgroup waits for is at most one ring lap ahead of the last one consumed.  Each stage is
// consumed by exactly one warpgroup, so its empty barrier counts that warpgroup's 4 warps.  The k16 MMA sequence of every output
// element and the epilogue arithmetic are those of gemm_tc5_kernel: results are bit-identical to it.
//
// The epilogue is specialised on what the UNet's short-K GEMMs ask of it.  GEGLU is a template option, and so is PASS2, the
// chunk pass that adds the residual and the blend (and applies the GELU family, which follows the fp16 rounding): the register
// pass then carries no option branch but SiLU and rowbias, which are hoisted out of its unrolled loops.  The warpgroup copies
// the tile's BN bias values to shared memory once per tile, before the main loop.  The staged tile leaves by TMA stores (p.omap, one 128-row box per 64
// output columns) issued by one thread of the warpgroup, and is written in the boxes' swizzled layout (T5Stage).
constexpr int T5_PP_BATCH = 2;   // ping-pong chunk pass: chunks whose global loads are issued together (4 spills at BN = 128)

// The ping-pong staging tile of W fp16 columns: TMA store boxes of BOXC = min(W, 64) columns x 128 rows, one after the other,
// each row 2 BOXC bytes under the swizzle TMA applies to such rows (SWIZZLE_128B for 128-byte rows, SWIZZLE_64B for 64-byte
// rows: the 16-byte chunk index is XORed with bits 7.. of the byte offset).  The tile is 1024-byte aligned.
template <int W>
struct T5Stage {
  static constexpr int BOXC = W < 64 ? W : 64, ROWB = 2 * BOXC, BOX_BYTES = T5_BM * ROWB, BOXES = W / BOXC;
  // byte offset of element (r, c); c even for 4-byte and a multiple of 8 for 16-byte accesses
  static HI3D_DEVINL uint32_t off(int r, int c) {
    const uint32_t o = (uint32_t)((c / BOXC) * BOX_BYTES + r * ROWB + (c % BOXC) * 2);
    return o ^ (((o >> 7) & (ROWB == 128 ? 7u : 3u)) << 4);
  }
};

// Register pass of one ping-pong tile (wgmma m64nBN layout, two m64 rows h): accumulator + bias (sbias: the tile's BN bias
// values, -0 where there is none, as x + -0 = x for every x), rowbias, then SiLU or GEGLU; one fp16 rounding into the staging
// tile sC.
template <int BN, bool GEGLU, bool SILU, bool RB>
HI3D_DEVINL void t5_pp_stage(const T5Params& p, const float (&acc)[2][BN / 2], const float* sbias, uint8_t* sC, int mt,
                             const T5Tile& o, int n0) {
  using S = T5Stage<GEGLU ? BN / 2 : BN>;
  const int lane = threadIdx.x & 31, t4 = lane & 3, warp = (threadIdx.x >> 5) & 3;
  const int ncols = p.N - n0;   // columns of the tile inside N (rowbias reads stop there)
#pragma unroll
  for (int h = 0; h < 2; h++) {
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
      const int r = h * 64 + warp * 16 + (lane >> 2) + 8 * hh;
      const __half* rbp = nullptr;
      if constexpr (RB) {
        const long long m = t5_row(p, mt, o, r);   // rows past the end (-1) read row 0's rowbias and are not stored
        rbp = p.rowbias + (long long)(((m < 0 ? 0 : m) / p.rb_div) % p.rb_mod) * p.rb_ld + n0;
      }
#pragma unroll
      for (int j = 0; j < BN / 8; j++) {
        const int cl = j * 8 + 2 * t4;
        const float2 b = *reinterpret_cast<const float2*>(sbias + cl);
        float v0 = acc[h][4 * j + 2 * hh] + b.x, v1 = acc[h][4 * j + 2 * hh + 1] + b.y;
        if constexpr (RB) {
          if (j * 8 < ncols) {
            const __half2 rbv = *reinterpret_cast<const __half2*>(rbp + cl);
            v0 += __low2float(rbv);
            v1 += __high2float(rbv);
          }
        }
        if constexpr (GEGLU) {
          *reinterpret_cast<__half*>(sC + S::off(r, cl >> 1)) = __float2half_rn(v0 * gelu_erf_f(v1));
        } else {
          if constexpr (SILU) {
            v0 = silu_f(v0);
            v1 = silu_f(v1);
          }
          *reinterpret_cast<uint32_t*>(sC + S::off(r, cl)) = pack_half2(v0, v1);
        }
      }
    }
  }
}

// Chunk pass of one ping-pong tile (W = BN staged columns): the GELU family, the residual and the blend on the staged tile in
// place, with coalesced 16-byte residual / blend loads, T5_PP_BATCH chunks per thread in flight.
template <int W>
HI3D_DEVINL void t5_pp_pass2(const T5Params& p, uint8_t* sC, int mt, const T5Tile& o, int nout0, int Nout) {
  using S = T5Stage<W>;
  constexpr int CPR = W / 8;   // 16-byte chunks per staged row
  static_assert((T5_BM * CPR) % (128 * T5_PP_BATCH) == 0, "whole batches");
#pragma unroll 1
  for (int idx0 = threadIdx.x & 127; idx0 < T5_BM * CPR; idx0 += 128 * T5_PP_BATCH) {
    long long mo[T5_PP_BATCH];
    uint32_t so[T5_PP_BATCH];
    Half8 rr[T5_PP_BATCH], xx[T5_PP_BATCH];
#pragma unroll
    for (int u = 0; u < T5_PP_BATCH; u++) {
      const int idx = idx0 + u * 128, r = idx / CPR, c = (idx % CPR) * 8;
      so[u] = S::off(r, c);
      const long long m = nout0 + c < Nout ? t5_row(p, mt, o, r) : -1;
      mo[u] = m < 0 ? -1 : t5_out_row(p, m);
      if (mo[u] >= 0) t5_load_chunk(p, mo[u], nout0 + c, rr[u], xx[u]);
    }
#pragma unroll
    for (int u = 0; u < T5_PP_BATCH; u++) {
      if (mo[u] < 0) continue;
      Half8 v = *reinterpret_cast<const Half8*>(sC + so[u]);
      t5_finish_half8(p, v, rr[u], xx[u]);
      *reinterpret_cast<Half8*>(sC + so[u]) = v;
    }
  }
}

template <int BN, bool GEGLU, bool PASS2>
__global__ void __launch_bounds__(384, 1) gemm_tc5_pingpong_kernel(const __grid_constant__ T5Params p) {
  static_assert(!(GEGLU && PASS2), "GEGLU GEMMs with a residual or blend take the single-tile schedule");
  constexpr int ROW = T5Op<__half>::ROW;
  constexpr int A_BYTES = T5_BM * ROW;
  constexpr uint32_t stage_bytes = A_BYTES + BN * ROW;
  using S = T5Stage<GEGLU ? BN / 2 : BN>;
  constexpr uint32_t STAGING_BYTES = T5_BM * BN * sizeof(__half);   // one consumer's staging tile (GEGLU uses half of it)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;          // SWIZZLE_128B atoms need 1024-byte alignment
  uint8_t* smem = smem_raw + (base - raw);
  const int STAGES = p.stages;
  float* const sbias_all = reinterpret_cast<float*>(smem + STAGES * stage_bytes + 2 * STAGING_BYTES);   // 2 x BN floats
  const uint32_t bar_full = base + STAGES * stage_bytes + 2 * STAGING_BYTES + 2 * BN * (uint32_t)sizeof(float);
  const uint32_t bar_empty = bar_full + 8 * T5Op<__half>::MAX_STAGES;

  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);    // provably warp-uniform role index
  const int KT = p.K / T5_BK;
  const int tiles = p.m_tiles * p.n_tiles;
  const int n_local = (tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (tid == 0) {
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar_full + 8 * s, 1);        // the producer's expect_tx arrive
      mbar_init(bar_empty + 8 * s, 4);       // one arrive per warp of the consuming warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ======================= TMA producer: every tile of this CTA through one ring =======================
    setmaxnreg_dec<40>();
    if (tid < 32) {
      uint32_t s = 0, ph = 0;
      for (int j = 0; j < n_local; j++) {
        const int tile = blockIdx.x + j * gridDim.x;
        const int mt = tile / p.n_tiles;
        const T5Tile o[1] = {t5_origin(p, mt)};
        t5_produce<BN, 1, __half>(p, base, bar_full, bar_empty, mt, o, (tile % p.n_tiles) * BN, s, ph);
      }
    }
    return;
  }

  // ======================= consumer warpgroups: tiles cw, cw + 2, ... of this CTA =======================
  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const bool leader = (tid & 127) == 0;   // issues and waits for this warpgroup's TMA stores
  const uint32_t sC_addr = base + STAGES * stage_bytes + cw * STAGING_BYTES;
  uint8_t* const sC = smem + (sC_addr - base);
  float* const sbias = sbias_all + cw * BN;
  const int Nout = GEGLU ? p.N / 2 : p.N;
  const bool silu = !GEGLU && p.act == HI3D_ACT_SILU;
  const bool rowbias = p.rowbias != nullptr;
  for (int j = cw; j < n_local; j += 2) {
    const int tile = blockIdx.x + j * gridDim.x;
    const int mt = tile / p.n_tiles, n0 = (tile % p.n_tiles) * BN;
    const T5Tile o = t5_origin(p, mt);
    // the tile's bias columns, loaded under the main loop (the register pass of tile j - 2 has read them: barrier 4 + cw)
    for (int c = tid & 127; c < BN; c += 128) sbias[c] = (p.bias != nullptr && n0 + c < p.N) ? __ldg(p.bias + n0 + c) : -0.f;
    float acc[2][BN / 2];
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int i = 0; i < BN / 2; i++) acc[h][i] = 0.f;
    // our MMA turn: the other warpgroup has issued the main loop of tile j - 1
    if (j > 0) named_bar_sync(2 + cw, 256);
    uint32_t it = (uint32_t)j * KT;
    uint32_t s = it % STAGES, ph = (it / STAGES) & 1, ps = 0;
    for (int kt = 0; kt < KT; kt++) {
      mbar_wait(bar_full + 8 * s, ph);
      const uint32_t sA = base + s * stage_bytes;
      wgmma_fence();
      {
        const uint64_t ad0 = gmma_desc_sw128(sA), ad1 = gmma_desc_sw128(sA + 64 * ROW);
        const uint64_t bd = gmma_desc_sw128(sA + A_BYTES);
#pragma unroll
        for (int k = 0; k < T5_BK / 16; k++) {   // +32 bytes along K inside the 128-byte swizzle atom
          wgmma_ss<BN>(acc[0], ad0 + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kt | k) ? 1 : 0);
          wgmma_ss<BN>(acc[1], ad1 + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kt | k) ? 1 : 0);
        }
      }
      wgmma_commit();
      // keep one k-block of MMAs in flight: the previous one has retired, its stage goes back to the producer
      wgmma_wait<1>();
      if (kt > 0 && lane == 0) mbar_arrive(bar_empty + 8 * ps);
      ps = s;
      if (++s == (uint32_t)STAGES) { s = 0; ph ^= 1; }
    }
    // hand the tensor cores to the other warpgroup's next tile, then finish ours
    if (j + 1 < n_local) named_bar_arrive(2 + (cw ^ 1), 256);
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (lane == 0) mbar_arrive(bar_empty + 8 * ps);

    // the TMA stores of this warpgroup's previous tile (issued a whole main loop ago) have read the staging tile, and sbias
    // is written
    if (leader && j > cw) bulk_wait_read();
    named_bar_sync(4 + cw, 128);
    // ---- register pass: accumulators -> (bias, rowbias, SiLU / GEGLU) -> staging tile ----
    if (rowbias) {
      if (silu) t5_pp_stage<BN, GEGLU, true, true>(p, acc, sbias, sC, mt, o, n0);
      else t5_pp_stage<BN, GEGLU, false, true>(p, acc, sbias, sC, mt, o, n0);
    } else {
      if (silu) t5_pp_stage<BN, GEGLU, true, false>(p, acc, sbias, sC, mt, o, n0);
      else t5_pp_stage<BN, GEGLU, false, false>(p, acc, sbias, sC, mt, o, n0);
    }
    const int nout0 = GEGLU ? n0 / 2 : n0;
    if constexpr (PASS2) {
      named_bar_sync(4 + cw, 128);
      t5_pp_pass2<BN>(p, sC, mt, o, nout0, Nout);
    }
    // ---- the staged tile leaves by TMA; rows past M and columns past Nout fall outside the map and are not written ----
    fence_proxy_async_smem();
    named_bar_sync(4 + cw, 128);
    if (leader) {
#pragma unroll
      for (int b = 0; b < S::BOXES; b++) {
        const int c0 = nout0 + b * S::BOXC;
        if (c0 >= Nout) break;
        if (p.mode == HI3D_ROWS_PLAIN) tma_store_2d(&p.omap, sC_addr + b * S::BOX_BYTES, c0, mt * T5_BM);
        else tma_store_4d(&p.omap, sC_addr + b * S::BOX_BYTES, c0, o.x0, o.y0, o.z0);
      }
      bulk_commit();
    }
  }
  if (leader) bulk_wait();
}

// ---- host: tensor maps ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(f);
  }
  return fn;
}

int encode_map(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, const cuuint32_t* elem_strides, CUtensorMapSwizzle swizzle, CUtensorMapDataType dtype) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("hi3d_gemm_tc5: cuTensorMapEncodeTiled entry point unavailable"); return -1; }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  if (elem_strides) for (int i = 0; i < rank; i++) estr[i] = elem_strides[i];
  CUresult r = enc(m, dtype, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("hi3d_gemm_tc5: cuTensorMapEncodeTiled failed (%d) rank=%d dims=%llu,%llu box=%u,%u", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return -1;
  }
  return 0;
}

static bool pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }

// Test / tuning hooks: -1 automatic, else forced single tiles (pair 0 / 8 epilogue warps) or tile pairs (pair 1 / 16
// epilogue warps); read once from HI3D_TC5_PAIR / HI3D_TC5_EW.
static int g_pair_mode = -2;   // -2 unread
static int g_ew_mode = -2;
static void read_env_once() {
  if (g_pair_mode == -2) { const char* e = getenv("HI3D_TC5_PAIR"); g_pair_mode = e ? atoi(e) : -1; }
  if (g_pair_mode < -1 || g_pair_mode > 1) g_pair_mode = -1;
  if (g_ew_mode == -2) { const char* e = getenv("HI3D_TC5_EW"); g_ew_mode = e ? atoi(e) : -1; }
  if (g_ew_mode != 8 && g_ew_mode != 16) g_ew_mode = -1;
}

template <int BN, int NT, typename Op>
static int launch_tc5(const T5Params& tp, int grid, int smem, cudaStream_t st) {
  static bool attr_done[HI3D_MAX_DEVICES];
  if (ensure_dyn_smem(gemm_tc5_kernel<BN, NT, Op>, smem, attr_done, "hi3d_gemm_tc5")) return -1;
  gemm_tc5_kernel<BN, NT, Op><<<grid, 128 + 256 * NT, smem, st>>>(tp);
  return check_launch("hi3d_gemm_tc5");
}

template <int BN, bool GEGLU, bool PASS2>
static int launch_pingpong(const T5Params& tp, int grid, int smem, cudaStream_t st) {
  static bool attr_done[HI3D_MAX_DEVICES];
  if (ensure_dyn_smem(gemm_tc5_pingpong_kernel<BN, GEGLU, PASS2>, smem, attr_done, "hi3d_gemm_tc5")) return -1;
  gemm_tc5_pingpong_kernel<BN, GEGLU, PASS2><<<grid, 384, smem, st>>>(tp);
  return check_launch("hi3d_gemm_tc5");
}

// The ping-pong kernels: tile width x epilogue (GEGLU; bias / rowbias / SiLU only; with the chunk pass for residual, blend and
// the GELU family).  A GEGLU GEMM with a residual or blend does not run ping-pong (tc5_choose).
static int launch_pingpong(const T5Params& tp, int BN, int grid, int smem, cudaStream_t st) {
  const bool geglu = tp.act == HI3D_ACT_GEGLU;
  const bool pass2 = tp.residual != nullptr || tp.blend_x != nullptr || tp.act >= HI3D_ACT_GELU;
  if (BN == 64) {
    if (geglu) return launch_pingpong<64, true, false>(tp, grid, smem, st);
    return pass2 ? launch_pingpong<64, false, true>(tp, grid, smem, st) : launch_pingpong<64, false, false>(tp, grid, smem, st);
  }
  if (geglu) return launch_pingpong<128, true, false>(tp, grid, smem, st);
  return pass2 ? launch_pingpong<128, false, true>(tp, grid, smem, st) : launch_pingpong<128, false, false>(tp, grid, smem, st);
}

// The ping-pong output map: the output in the geometry of a tile's rows, boxes of W = min(staged tile width, 64) columns x the
// tile's 128 rows (t5_row's order), swizzled as T5Stage lays the staging tile out.  Its row strides are out_ld, so a column
// slice of a wider buffer is written in place; a parity-class upsample conv starts at its class's first output row and steps two
// output columns / rows per tile column / row.
static int t5_encode_out_map(const hi3d_gemm_params* p, const T5Params& tp, int BN, CUtensorMap* m) {
  const bool geglu = p->act == HI3D_ACT_GEGLU;
  const int W = geglu ? BN / 2 : BN;
  const cuuint32_t boxc = W < 64 ? W : 64;
  const CUtensorMapSwizzle sw = boxc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  const cuuint64_t nout = (cuuint64_t)(geglu ? p->N / 2 : p->N), ld = (cuuint64_t)p->out_ld * sizeof(__half);
  if (p->mode == HI3D_ROWS_PLAIN) {
    cuuint64_t dims[2] = {nout, (cuuint64_t)p->M};
    cuuint64_t str[1] = {ld};
    cuuint32_t box[2] = {boxc, (cuuint32_t)T5_BM};
    return encode_map(m, p->out, 2, dims, str, box, nullptr, sw);
  }
  const cuuint64_t Wo = (cuuint64_t)tp.Wo, Ho = (cuuint64_t)tp.Ho, up = p->out_up ? 2 : 1;
  const __half* o = (const __half*)p->out;
  if (p->out_up) o += ((long long)p->out_py * 2 * tp.Wo + p->out_px) * p->out_ld;
  cuuint64_t dims[4] = {nout, Wo, Ho, (cuuint64_t)tp.Nimg};
  cuuint64_t str[3] = {up * ld, up * up * Wo * ld, up * up * Wo * Ho * ld};
  cuuint32_t box[4] = {boxc, (cuuint32_t)tp.tw, (cuuint32_t)tp.th, (cuuint32_t)tp.tn};
  return encode_map(m, o, 4, dims, str, box, nullptr, sw);
}

// The ping-pong schedule runs fp16 GEMMs of at most T5_PINGPONG_MAX_KT k-tiles (K <= 1280).  Measured with tools/time_gemm.py on
// every shape of the stage-2 UNet forward (H100 80GB HBM3, 700 W), ping-pong against the schedule otherwise chosen: 1.02x to
// 1.37x faster at K = 320 .. 1280 (5 .. 20 k-tiles); 0.82x and 0.90x at the plan's next K, 1920 (30 k-tiles), and slower
// at nearly every longer K, where tile pairs halve the B traffic and the epilogue is a small part of a tile.  M >= 128: a GEMM of
// fewer rows is a stream of W through mostly-padding tiles, which the 256-wide single tiles move in half the tiles.
constexpr int T5_PINGPONG_MAX_KT = 20;

// Schedules (hi3d_gemm_tc5_schedule returns schedule * 1000 + tile width).
enum { T5_SCHED_MMA_SYNC = 0, T5_SCHED_SINGLE = 1, T5_SCHED_PAIR = 2, T5_SCHED_PINGPONG = 3 };
struct T5Choice {
  int sched, BN, ntile;
};

// The one place that picks a covered GEMM's schedule and tile width (m_tiles from tc5_geometry).
template <bool FP8>
static T5Choice tc5_choose(const hi3d_gemm_params* p, int m_tiles) {
  const int sm_count = device_sm_count();
  read_env_once();
  // tile-N in {64, .., max_bn}.  Cost model = waves of one-CTA-per-SM tiles x time per tile, where a tile costs its MMA columns
  // plus a fixed term (A-operand traffic / epilogue set-up); this accounts both for the padding of N and for wave quantisation
  // over the SMs.  Ties go to the wider tile.
  auto pick_bn = [&](int max_bn, int m_units) {
    int bn = max_bn;
    long long best = -1;
    for (int cand = max_bn; cand >= 64; cand -= 64) {
      const long long ntl = (p->N + cand - 1) / cand;
      const long long waves = ((long long)m_units * ntl + sm_count - 1) / sm_count;
      const long long cost = waves * (cand + 48);
      if (best < 0 || cost < best) { best = cost; bn = cand; }
    }
    return bn;
  };
  const bool forced = g_ew_mode > 0 || g_pair_mode >= 0;
  const bool geglu_res = p->act == HI3D_ACT_GEGLU && (p->residual != nullptr || p->blend_x != nullptr);
  if (!FP8 && !forced && !geglu_res && p->K / T5_BK <= T5_PINGPONG_MAX_KT && p->M >= T5_BM) {
    const int bn = pick_bn(128, m_tiles);
    if ((long long)m_tiles * ((p->N + bn - 1) / bn) >= sm_count) return {T5_SCHED_PINGPONG, bn, 1};
  }
  // Tile pairs (NT = 2): two row tiles share each B tile, halving the B bytes per output row; worth it once the main loop
  // dominates (long K) and there are enough tiles to fill the SMs with pairs.  The hooks force either choice.
  int ntile = (p->K >= 1920 && (long long)m_tiles * ((p->N + 127) / 128) >= 4LL * sm_count) ? 2 : 1;
  if (g_ew_mode > 0) ntile = g_ew_mode / 8;
  if (g_pair_mode >= 0) ntile = g_pair_mode + 1;
  const int bn = pick_bn(ntile == 2 ? 128 : 256, (m_tiles + ntile - 1) / ntile);
  return {ntile == 2 ? T5_SCHED_PAIR : T5_SCHED_SINGLE, bn, ntile};
}

}  // namespace hi3d

using namespace hi3d;

extern "C" int hi3d_gemm_tc5_set_pair_mode(int mode) {
  if (mode < -1 || mode > 1) { set_error("hi3d_gemm_tc5_set_pair_mode: mode must be -1 (auto), 0 or 1"); return -2; }
  read_env_once();
  g_pair_mode = mode;
  return 0;
}

extern "C" int hi3d_gemm_tc5_set_epilogue_warps(int warps) {
  if (warps != -1 && warps != 8 && warps != 16) { set_error("hi3d_gemm_tc5_set_epilogue_warps: -1 (auto), 8 or 16"); return -2; }
  read_env_once();
  g_ew_mode = warps;
  return 0;
}

// The tiling of one GEMM on this engine, from its geometry alone: tile -> rows mapping, row tiles, and the distinct A sources
// (srcs / lds, T5_MAX_MAPS entries) that become tensor maps.  False when the engine does not cover the geometry.
static bool tc5_geometry(const hi3d_gemm_params* p, T5Params& tp, int& m_tiles, const void** srcs, int* lds, int& nmaps) {
  memset(&tp, 0, sizeof(tp));
  tp.M = p->M; tp.N = p->N; tp.K = p->K; tp.mode = p->mode; tp.nseg = p->nseg;
  tp.cstride = (p->mode == HI3D_ROWS_CONV2D) ? p->stride : 1;
  tp.out_up = p->out_up; tp.out_py = p->out_py; tp.out_px = p->out_px;
  tp.t_off = p->t_off;
  m_tiles = 0;
  bool ok = (p->N >= 32) && (p->N % 8 == 0);
  ok = ok && (p->rowbias == nullptr || ((uintptr_t)p->rowbias % 4 == 0 && p->rb_ld % 2 == 0));
  if (p->mode == HI3D_ROWS_PLAIN) {
    tp.tw = 128; tp.th = 1; tp.tn = 1;
    m_tiles = (p->M + T5_BM - 1) / T5_BM;
  } else if (p->mode == HI3D_ROWS_CONV2D) {
    ok = ok && p->ups == 0 && ((p->stride == 1 && p->Ho == p->Hs && p->Wo == p->Ws) ||
                               (p->stride == 2 && p->Hs == 2 * p->Ho && p->Ws == 2 * p->Wo && !p->out_up));
    const int Nimg = ok ? p->M / (p->Ho * p->Wo) : 0;
    int tw = 1;
    while (tw * 2 <= 16 && (p->Wo % (tw * 2)) == 0) tw *= 2;
    int th = 1;
    while (tw * th * 2 <= 128 && (p->Ho % (th * 2)) == 0) th *= 2;
    int tn = ok ? 128 / (tw * th) : 1;
    ok = ok && pow2(tn) && tw * th * tn == 128 && (Nimg % tn) == 0;
    tp.tw = tw; tp.th = th; tp.tn = tn; tp.Wo = p->Wo; tp.Ho = p->Ho; tp.Nimg = Nimg;
    tp.tiles_x = p->Wo / tw; tp.tiles_y = p->Ho / th;
    m_tiles = ok ? tp.tiles_x * tp.tiles_y * (Nimg / tn) : 0;
  } else {
    const int HW = p->Ho * p->Wo, T = p->T, B = p->M / (HW * T);
    int ts = 1;
    while (ts * 2 <= 128 && (HW % (ts * 2)) == 0) ts *= 2;
    int tf = 128 / ts;
    ok = ok && (T % tf) == 0;
    tp.tw = ts; tp.th = tf; tp.tn = 1; tp.Wo = HW; tp.Ho = T; tp.Nimg = B;
    tp.tiles_x = HW / ts; tp.tiles_y = ok ? T / tf : 1;
    m_tiles = ok ? tp.tiles_x * tp.tiles_y * B : 0;
  }
  // distinct A sources -> tensor maps
  nmaps = 0;
  for (int i = 0; ok && i < p->nseg; i++) {
    const hi3d_seg& s = p->seg[i];
    int mi = -1;
    for (int j = 0; j < nmaps; j++)
      if (srcs[j] == s.src && lds[j] == s.ld) mi = j;
    if (mi < 0) {
      if (nmaps == T5_MAX_MAPS) { ok = false; break; }
      srcs[nmaps] = s.src; lds[nmaps] = s.ld; mi = nmaps++;
    }
    tp.seg[i].map = mi; tp.seg[i].c_off = s.c_off; tp.seg[i].C = s.C;
    tp.seg[i].dy = s.dy; tp.seg[i].dx = s.dx; tp.seg[i].dt = s.dt;
  }
  return ok && m_tiles > 0;
}

// One GEMM on the engine, with fp16 or e4m3 operands.  fp16: geometries the engine does not cover go to the mma.sync engine
// (same results).  e4m3: there is no other engine, so such a geometry is an error.
template <typename Op>
static int tc5_gemm(const hi3d_gemm_params* p, const float* w_scale, int out_fp8, void* stream, const char* who) {
  constexpr bool FP8 = sizeof(Op) == 1;
  constexpr int ROW = T5Op<Op>::ROW, ESIZE = sizeof(Op), MAX_STAGES = T5Op<Op>::MAX_STAGES;
  int rc = validate_gemm(p, who);
  if (rc) return rc;
  if (FP8) {
    // TMA global strides are multiples of 16 bytes
    for (int i = 0; i < p->nseg; i++)
      if (p->seg[i].ld % 16) { set_error("%s: e4m3 segment %d has ld %d, not a multiple of 16", who, i, p->seg[i].ld); return -2; }
    if (w_scale == nullptr || ((uintptr_t)w_scale & 7)) { set_error("%s: w_scale null or misaligned", who); return -2; }
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // ---- geometry this engine covers ----
  T5Params tp;
  const void* srcs[T5_MAX_MAPS];
  int lds[T5_MAX_MAPS];
  int m_tiles = 0, nmaps = 0;
  const bool ok = tc5_geometry(p, tp, m_tiles, srcs, lds, nmaps);
  if (!ok) {
    if (!FP8) return hi3d_gemm(p, stream);
    set_error("%s: geometry not covered by the e4m3 engine (mode %d, M %d, N %d, Ho %d, Wo %d, T %d, stride %d, ups %d, %d segments)",
              who, p->mode, p->M, p->N, p->Ho, p->Wo, p->T, p->stride, p->ups, p->nseg);
    return -2;
  }

  const T5Choice ch = tc5_choose<FP8>(p, m_tiles);
  const int BN = ch.BN, ntile = ch.ntile;
  const bool pingpong = ch.sched == T5_SCHED_PINGPONG;
  const int stage_bytes = ntile * T5_BM * ROW + BN * ROW;
  // the ping-pong schedule keeps one staging tile and the tile's bias per consumer warpgroup outside the ring
  const int staging_bytes = pingpong ? 2 * (T5_BM * BN * (int)sizeof(__half) + BN * (int)sizeof(float)) : 0;
  int stages = (T5_SMEM_BUDGET - staging_bytes) / stage_bytes;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  tp.stages = stages;
  tp.n_tiles = (p->N + BN - 1) / BN;
  tp.m_tiles = m_tiles;
  const int m_units = (m_tiles + ntile - 1) / ntile;
  long long grid = (long long)m_units * tp.n_tiles;
  if (grid > 2147483647LL) { set_error("%s: too many tiles", who); return -2; }
  if (pingpong && grid > device_sm_count()) grid = device_sm_count();

  for (int j = 0; j < nmaps; j++) {
    const cuuint64_t ld = (cuuint64_t)lds[j];
    if (p->mode == HI3D_ROWS_PLAIN) {
      cuuint64_t dims[2] = {ld, (cuuint64_t)p->M};
      cuuint64_t str[1] = {ld * ESIZE};
      cuuint32_t box[2] = {64, 128};
      if (encode_map(&tp.amap[j], srcs[j], 2, dims, str, box, nullptr, T5Op<Op>::SW, T5Op<Op>::DT)) return -1;
    } else if (p->mode == HI3D_ROWS_CONV2D) {
      cuuint64_t dims[4] = {ld, (cuuint64_t)p->Ws, (cuuint64_t)p->Hs, (cuuint64_t)tp.Nimg};
      cuuint64_t str[3] = {ld * ESIZE, ld * ESIZE * p->Ws, ld * ESIZE * p->Ws * p->Hs};
      const cuuint32_t cs = (cuuint32_t)tp.cstride;   // stride 2: box spans 2*tw x 2*th input pixels, every 2nd loaded
      cuuint32_t box[4] = {64, (cuuint32_t)tp.tw * cs, (cuuint32_t)tp.th * cs, (cuuint32_t)tp.tn};
      cuuint32_t est[4] = {1, cs, cs, 1};
      if (encode_map(&tp.amap[j], srcs[j], 4, dims, str, box, est, T5Op<Op>::SW, T5Op<Op>::DT)) return -1;
    } else {
      const cuuint64_t HW = (cuuint64_t)tp.Wo, T = (cuuint64_t)(p->Tin > 0 ? p->Tin : tp.Ho);   // source frames per clip
      cuuint64_t dims[4] = {ld, HW, T, (cuuint64_t)tp.Nimg};
      cuuint64_t str[3] = {ld * ESIZE, ld * ESIZE * HW, ld * ESIZE * HW * T};
      cuuint32_t box[4] = {64, (cuuint32_t)tp.tw, (cuuint32_t)tp.th, 1};
      if (encode_map(&tp.amap[j], srcs[j], 4, dims, str, box, nullptr, T5Op<Op>::SW, T5Op<Op>::DT)) return -1;
    }
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)p->K, (cuuint64_t)p->N};
    cuuint64_t str[1] = {(cuuint64_t)p->K * ESIZE};
    cuuint32_t box[2] = {64, (cuuint32_t)BN};
    if (encode_map(&tp.bmap, p->W, 2, dims, str, box, nullptr, T5Op<Op>::SW, T5Op<Op>::DT)) return -1;
  }
  tp.bias = p->bias; tp.rowbias = (const __half*)p->rowbias; tp.rb_div = p->rb_div; tp.rb_mod = p->rb_mod;
  tp.rb_ld = p->rb_ld; tp.act = p->act; tp.residual = (const __half*)p->residual; tp.res_ld = p->res_ld;
  tp.blend_x = (const __half*)p->blend_x; tp.blend_ld = p->blend_ld; tp.alpha = p->alpha;
  tp.out = (__half*)p->out; tp.out_ld = p->out_ld;
  tp.w_scale = w_scale; tp.out_fp8 = out_fp8;

  const int smem = stages * stage_bytes + staging_bytes + 16 * MAX_STAGES + 1024;
  if constexpr (!FP8) {
    if (pingpong) {
      if (t5_encode_out_map(p, tp, BN, &tp.omap)) return -1;
      return launch_pingpong(tp, BN, (int)grid, smem, st);
    }
  }
  if (ntile == 2)
    return BN == 64 ? launch_tc5<64, 2, Op>(tp, (int)grid, smem, st) : launch_tc5<128, 2, Op>(tp, (int)grid, smem, st);
  switch (BN) {
    case 64: return launch_tc5<64, 1, Op>(tp, (int)grid, smem, st);
    case 128: return launch_tc5<128, 1, Op>(tp, (int)grid, smem, st);
    case 192: return launch_tc5<192, 1, Op>(tp, (int)grid, smem, st);
    default: return launch_tc5<256, 1, Op>(tp, (int)grid, smem, st);
  }
}

extern "C" int hi3d_gemm_tc5(const hi3d_gemm_params* p, void* stream) {
  return tc5_gemm<__half>(p, nullptr, 0, stream, "hi3d_gemm_tc5");
}

extern "C" int hi3d_gemm_tc5_fp8(const hi3d_gemm_params* p, const float* w_scale, int out_fp8, void* stream) {
  return tc5_gemm<__nv_fp8_e4m3>(p, w_scale, out_fp8 ? 1 : 0, stream, "hi3d_gemm_tc5_fp8");
}

extern "C" int hi3d_gemm_tc5_fp8_covers(const hi3d_gemm_params* p) {
  if (p == nullptr || p->M <= 0 || p->N <= 0 || p->nseg <= 0 || p->nseg > HI3D_MAX_SEGS ||
      (p->mode == HI3D_ROWS_CONV2D && (p->Ho <= 0 || p->Wo <= 0)) ||
      (p->mode == HI3D_ROWS_TEMPORAL && (p->Ho <= 0 || p->Wo <= 0 || p->T <= 0))) {
    set_error("hi3d_gemm_tc5_fp8_covers: bad parameters");
    return -2;
  }
  T5Params tp;
  const void* srcs[T5_MAX_MAPS];
  int lds[T5_MAX_MAPS];
  int m_tiles = 0, nmaps = 0;
  return tc5_geometry(p, tp, m_tiles, srcs, lds, nmaps) ? 1 : 0;
}

extern "C" int hi3d_gemm_tc5_schedule(const hi3d_gemm_params* p) {
  int rc = validate_gemm(p, "hi3d_gemm_tc5_schedule");
  if (rc) return rc;
  T5Params tp;
  const void* srcs[T5_MAX_MAPS];
  int lds[T5_MAX_MAPS];
  int m_tiles = 0, nmaps = 0;
  if (!tc5_geometry(p, tp, m_tiles, srcs, lds, nmaps)) return T5_SCHED_MMA_SYNC;
  const T5Choice ch = tc5_choose<false>(p, m_tiles);
  return ch.sched * 1000 + ch.BN;
}
