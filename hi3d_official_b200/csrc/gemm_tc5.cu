// Implicit-GEMM engine, Hopper-native variant: TMA (cp.async.bulk.tensor) operand staging into SWIZZLE_128B shared
// tiles through an mbarrier ring, wgmma (warpgroup MMA, fp32 accumulators in registers) on the tiles in place, and an
// epilogue staged through shared memory for coalesced 16-byte stores.  Same contract as hi3d_gemm (include/hi3d_b200.h);
// geometries this engine does not cover (upsample-fused convs, odd patch shapes, N < 32, > 4 distinct A sources) are
// forwarded to the mma.sync engine.
//
// One CTA per 128 x BN output tile (BN in {64, 128, 192, 256}, chosen per call to cover N with the least padding and
// wave quantisation over the SMs; n-tile fastest so that CTAs running together share A rows through L2).  The 128 rows of
// a tile are
//   PLAIN    : 128 consecutive rows
//   CONV2D   : a (tn images) x (th rows) x (tw columns) patch, tn*th*tw = 128 -- the 3x3 taps are the same TMA box
//              shifted by (dy, dx) and the zero padding is TMA out-of-bounds fill (stride 2: TMA element strides)
//   TEMPORAL : (tf frames) x (ts pixels), tf*ts = 128 -- the temporal taps shift the frame coordinate of a
//              [C, HW, T, B] view; clip boundaries zero-fill by OOB.
// Warp roles (128 + 256 NT threads): warpgroup 0 = TMA producer (one elected thread), then two MMA + epilogue warpgroups
// per 128-row tile (rows 0..63 and 64..127).  NT = 2 ("tile pairs", 16 epilogue warps) puts two consecutive row tiles in
// one CTA that share every B tile -- half the B bytes from L2 per output row, for long-K shapes -- and is built for
// BN <= 128 (the register budget of 640 threads).  The producer hands its registers to the MMA warpgroups (setmaxnreg):
// a 64 x 256 fp32 accumulator is 128 registers per thread.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "tc5.cuh"

namespace hi3d {
int validate_gemm(const hi3d_gemm_params* p, const char* who);
int gemm_gn_stats_pass(const hi3d_gemm_params* p, void* stream);

constexpr int T5_BM = 128;
constexpr int T5_BK = 64;
constexpr int T5_MAX_MAPS = 4;
constexpr int T5_MAX_STAGES = 8;
constexpr int T5_A_BYTES = T5_BM * 128;
constexpr int T5_SMEM_BUDGET = 200 * 1024;

struct T5Seg {
  int map;       // index into amap[]
  int c_off, C;  // channel range
  int dy, dx, dt;
};

struct T5Params {
  CUtensorMap bmap;
  CUtensorMap amap[T5_MAX_MAPS];
  T5Seg seg[HI3D_MAX_SEGS];
  int nseg;
  int M, N, K, mode;
  int stages, n_tiles;
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

template <int BN, int NT>
__global__ void __launch_bounds__(128 + 256 * NT, 1) gemm_tc5_kernel(const __grid_constant__ T5Params p) {
  constexpr int MMA_THREADS = 256 * NT;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;          // SWIZZLE_128B atoms need 1024-byte alignment
  uint8_t* smem = smem_raw + (base - raw);
  const int STAGES = p.stages;
  constexpr uint32_t stage_bytes = NT * T5_A_BYTES + BN * 128;
  const uint32_t bar_full = base + STAGES * stage_bytes;   // STAGES x 8
  const uint32_t bar_empty = bar_full + 8 * T5_MAX_STAGES;

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
      // the whole warp walks the loop with warp-uniform values and one lane issues
      uint32_t s = 0, ph = 0;
      int si = 0, so = 0;
      T5Seg sg = p.seg[0];
      const CUtensorMap* am = &p.amap[sg.map];
      for (int kt = 0; kt < KT; kt++) {
        mbar_wait(bar_empty + 8 * s, ph ^ 1);
        if (lane == 0) {
          const uint32_t sB = base + s * stage_bytes + NT * T5_A_BYTES;
          const uint32_t full = bar_full + 8 * s;
          const int c = sg.c_off + so;
          mbar_expect_tx(full, stage_bytes);
          // a second row tile past the last one loads out of bounds (zeros) and stores nothing
          for (int t = 0; t < NT; t++) {
            const uint32_t sA = base + s * stage_bytes + t * T5_A_BYTES;
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
  {
    uint32_t s = 0, ph = 0, ps = 0;
    for (int kt = 0; kt < KT; kt++) {
      mbar_wait(bar_full + 8 * s, ph);
      const uint32_t sA = base + s * stage_bytes + cw * 64 * 128;
      const uint32_t sB = base + s * stage_bytes + NT * T5_A_BYTES;
      const uint64_t ad = gmma_desc_sw128(sA), bd = gmma_desc_sw128(sB);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < T5_BK / 16; k++)   // +32 bytes along K inside the 128-byte swizzle atom
        wgmma_ss<BN>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kt | k) ? 1 : 0);
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
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int hh = 0; hh < 2; hh++) {
    const int rl = cw * 64 + warp * 16 + g + 8 * hh;
    const long long m = t5_row(p, mt0 + ct, o[ct], rl - ct * T5_BM);
    const __half* rbp = nullptr;
    if (p.rowbias != nullptr && m >= 0) rbp = p.rowbias + (long long)((m / p.rb_div) % p.rb_mod) * p.rb_ld;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
      const int cl = j * 8 + 2 * t4;
      const int n = n0 + cl;
      float v0 = acc[4 * j + 2 * hh], v1 = acc[4 * j + 2 * hh + 1];
      if (n < p.N) {
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
        sC[rl * pitch + (cl >> 1)] = __float2half_rn(v0 * gelu_erf_f(v1));
      } else {
        if (p.act == HI3D_ACT_SILU) {
          v0 = silu_f(v0);
          v1 = silu_f(v1);
        }
        *reinterpret_cast<uint32_t*>(sC + rl * pitch + cl) = pack_half2(v0, v1);
      }
    }
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
    const long long m = t5_row(p, mt0 + t, o[t], r - t * T5_BM);
    if (m < 0) continue;
    long long mo = m;                       // output row (differs from m only for the parity-class upsample convs)
    if (p.out_up) {
      const int hw = p.Ho * p.Wo;
      const int n_ = (int)(m / hw), rem_ = (int)(m - (long long)n_ * hw);
      const int y_ = rem_ / p.Wo, x_ = rem_ - y_ * p.Wo;
      mo = ((long long)n_ * 2 * p.Ho + 2 * y_ + p.out_py) * (2 * p.Wo) + 2 * x_ + p.out_px;
    }
    Half8 v = *reinterpret_cast<const Half8*>(sC + r * pitch + c * 8);
    if (p.act >= HI3D_ACT_GELU) clip_act_half8(p.act, v);
    if (p.residual != nullptr) {
      const Half8 rr = *reinterpret_cast<const Half8*>(p.residual + mo * p.res_ld + nc);
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const float2 a = __half22float2(v.h[q]), b = __half22float2(rr.h[q]);
        v.h[q] = __floats2half2_rn(a.x + b.x, a.y + b.y);
      }
    }
    if (p.blend_x != nullptr) {
      const Half8 xx = *reinterpret_cast<const Half8*>(p.blend_x + mo * p.blend_ld + nc);
      const float al = p.alpha, be = 1.f - p.alpha;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const float2 a = __half22float2(v.h[q]), b = __half22float2(xx.h[q]);
        v.h[q] = __floats2half2_rn(al * b.x + be * a.x, al * b.y + be * a.y);
      }
    }
    *reinterpret_cast<Half8*>(p.out + mo * p.out_ld + nc) = v;
  }
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
               const cuuint32_t* box, const cuuint32_t* elem_strides, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("hi3d_gemm_tc5: cuTensorMapEncodeTiled entry point unavailable"); return -1; }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  if (elem_strides) for (int i = 0; i < rank; i++) estr[i] = elem_strides[i];
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box,
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

template <int BN, int NT>
static int launch_tc5(const T5Params& tp, int grid, int smem, cudaStream_t st) {
  static bool attr_done[HI3D_MAX_DEVICES];
  if (ensure_dyn_smem(gemm_tc5_kernel<BN, NT>, smem, attr_done, "hi3d_gemm_tc5")) return -1;
  gemm_tc5_kernel<BN, NT><<<grid, 128 + 256 * NT, smem, st>>>(tp);
  return check_launch("hi3d_gemm_tc5");
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

extern "C" int hi3d_gemm_tc5(const hi3d_gemm_params* p, void* stream) {
  int rc = validate_gemm(p, "hi3d_gemm_tc5");
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // ---- geometry this engine covers; everything else goes to the mma.sync engine (same results) ----
  T5Params tp;
  memset(&tp, 0, sizeof(tp));
  tp.M = p->M; tp.N = p->N; tp.K = p->K; tp.mode = p->mode; tp.nseg = p->nseg;
  tp.cstride = (p->mode == HI3D_ROWS_CONV2D) ? p->stride : 1;
  tp.out_up = p->out_up; tp.out_py = p->out_py; tp.out_px = p->out_px;
  tp.t_off = p->t_off;
  int m_tiles = 0;
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
  const void* srcs[T5_MAX_MAPS];
  int lds[T5_MAX_MAPS];
  int nmaps = 0;
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
  if (!ok || m_tiles <= 0) return hi3d_gemm(p, stream);
  if (p->gn_stats != nullptr) {
    const int hw = (p->mode == HI3D_ROWS_PLAIN) ? p->gn_rows : p->Ho * p->Wo;
    if (p->gn_unit <= 0 || (p->N % p->gn_unit) || p->gn_rows <= 0 || (p->M % p->gn_rows) || p->act == HI3D_ACT_GEGLU ||
        (p->mode != HI3D_ROWS_PLAIN && p->gn_rows != hw)) {
      set_error("hi3d_gemm_tc5: bad gn_stats arguments (unit %d, rows %d, N %d, M %d)", p->gn_unit, p->gn_rows, p->N, p->M);
      return -2;
    }
  }

  // Tile pairs (NT = 2): two row tiles share each B tile, halving the B bytes per output row; worth it once the main loop
  // dominates (long K) and there are enough tiles to fill the SMs with pairs.  The hooks force either choice.
  const int sm_count = device_sm_count();
  read_env_once();
  int ntile = (p->K >= 1920 && (long long)m_tiles * ((p->N + 127) / 128) >= 4LL * sm_count) ? 2 : 1;
  if (g_ew_mode > 0) ntile = g_ew_mode / 8;
  if (g_pair_mode >= 0) ntile = g_pair_mode + 1;
  const int m_units = (m_tiles + ntile - 1) / ntile;
  // tile-N in {64, 128, 192, 256} ({64, 128} for pairs).  Cost model = waves of one-CTA-per-SM tiles x time per tile,
  // where a tile costs its MMA columns plus a fixed term (A-operand traffic / epilogue set-up); this accounts both for the
  // padding of N and for wave quantisation over the SMs.  Ties go to the wider tile.
  int BN = ntile == 2 ? 128 : 256;
  {
    long long best = -1;
    for (int cand = BN; cand >= 64; cand -= 64) {
      const long long ntl = (p->N + cand - 1) / cand;
      const long long waves = ((long long)m_units * ntl + sm_count - 1) / sm_count;
      const long long cost = waves * (cand + 48);
      if (best < 0 || cost < best) { best = cost; BN = cand; }
    }
  }
  const int stage_bytes = ntile * T5_A_BYTES + BN * 128;
  int stages = T5_SMEM_BUDGET / stage_bytes;
  if (stages > T5_MAX_STAGES) stages = T5_MAX_STAGES;
  tp.stages = stages;
  tp.n_tiles = (p->N + BN - 1) / BN;
  const long long grid = (long long)m_units * tp.n_tiles;
  if (grid > 2147483647LL) { set_error("hi3d_gemm_tc5: too many tiles"); return -2; }

  for (int j = 0; j < nmaps; j++) {
    const cuuint64_t ld = (cuuint64_t)lds[j];
    if (p->mode == HI3D_ROWS_PLAIN) {
      cuuint64_t dims[2] = {ld, (cuuint64_t)p->M};
      cuuint64_t str[1] = {ld * 2};
      cuuint32_t box[2] = {64, 128};
      if (encode_map(&tp.amap[j], srcs[j], 2, dims, str, box, nullptr)) return -1;
    } else if (p->mode == HI3D_ROWS_CONV2D) {
      cuuint64_t dims[4] = {ld, (cuuint64_t)p->Ws, (cuuint64_t)p->Hs, (cuuint64_t)tp.Nimg};
      cuuint64_t str[3] = {ld * 2, ld * 2 * p->Ws, ld * 2 * p->Ws * p->Hs};
      const cuuint32_t cs = (cuuint32_t)tp.cstride;   // stride 2: box spans 2*tw x 2*th input pixels, every 2nd loaded
      cuuint32_t box[4] = {64, (cuuint32_t)tp.tw * cs, (cuuint32_t)tp.th * cs, (cuuint32_t)tp.tn};
      cuuint32_t est[4] = {1, cs, cs, 1};
      if (encode_map(&tp.amap[j], srcs[j], 4, dims, str, box, est)) return -1;
    } else {
      const cuuint64_t HW = (cuuint64_t)tp.Wo, T = (cuuint64_t)(p->Tin > 0 ? p->Tin : tp.Ho);   // source frames per clip
      cuuint64_t dims[4] = {ld, HW, T, (cuuint64_t)tp.Nimg};
      cuuint64_t str[3] = {ld * 2, ld * 2 * HW, ld * 2 * HW * T};
      cuuint32_t box[4] = {64, (cuuint32_t)tp.tw, (cuuint32_t)tp.th, 1};
      if (encode_map(&tp.amap[j], srcs[j], 4, dims, str, box, nullptr)) return -1;
    }
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)p->K, (cuuint64_t)p->N};
    cuuint64_t str[1] = {(cuuint64_t)p->K * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)BN};
    if (encode_map(&tp.bmap, p->W, 2, dims, str, box, nullptr)) return -1;
  }
  tp.bias = p->bias; tp.rowbias = (const __half*)p->rowbias; tp.rb_div = p->rb_div; tp.rb_mod = p->rb_mod;
  tp.rb_ld = p->rb_ld; tp.act = p->act; tp.residual = (const __half*)p->residual; tp.res_ld = p->res_ld;
  tp.blend_x = (const __half*)p->blend_x; tp.blend_ld = p->blend_ld; tp.alpha = p->alpha;
  tp.out = (__half*)p->out; tp.out_ld = p->out_ld;

  const int smem = stages * stage_bytes + 16 * T5_MAX_STAGES + 1024;
  if (ntile == 2) {
    rc = BN == 64 ? launch_tc5<64, 2>(tp, (int)grid, smem, st) : launch_tc5<128, 2>(tp, (int)grid, smem, st);
  } else {
    switch (BN) {
      case 64: rc = launch_tc5<64, 1>(tp, (int)grid, smem, st); break;
      case 128: rc = launch_tc5<128, 1>(tp, (int)grid, smem, st); break;
      case 192: rc = launch_tc5<192, 1>(tp, (int)grid, smem, st); break;
      default: rc = launch_tc5<256, 1>(tp, (int)grid, smem, st);
    }
  }
  if (rc || p->gn_stats == nullptr) return rc;
  // hi3d_gemm_params::gn_stats: a statistics pass over the stored tensor, as on the mma.sync engine
  return gemm_gn_stats_pass(p, stream);
}
