// Shared device helpers for the Hi3D H100 kernels (sm_90a).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/hi3d_b200.h"

#define HI3D_DEVINL __device__ __forceinline__

namespace hi3d {

// ---- error plumbing (host) -------------------------------------------------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);
// One process may drive several GPUs: one-time per-device state (opt-in shared memory attributes, SM count) is
// indexed by the CURRENT device, never kept in a single process-wide flag.
constexpr int HI3D_MAX_DEVICES = 64;
int current_device();                       // cudaGetDevice(), clamped to [0, HI3D_MAX_DEVICES)
int device_sm_count();                      // SM count of the current device (cached per device)
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device); `done` = a static bool[HI3D_MAX_DEVICES]
template <typename K>
int ensure_dyn_smem(K kernel, int bytes, bool* done, const char* who) {
  const int d = current_device();
  if (done[d]) return 0;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) { set_error("%s: cudaFuncSetAttribute: %s", who, cudaGetErrorString(e)); return -1; }
  done[d] = true;
  return 0;
}

// ---- async copy / ldmatrix / mma ---------------------------------------------------------------
HI3D_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 16-byte cp.async with zero-fill when !valid (src must still be a legal address)
HI3D_DEVINL void cp_async16(uint32_t dst, const void* src, bool valid) {
  int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(sz));
}
HI3D_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
HI3D_DEVINL void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

HI3D_DEVINL void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
HI3D_DEVINL void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}

// D(16x8,f32) += A(16x16,f16,row) * B(16x8,f16,col)
HI3D_DEVINL void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 128-byte-row shared tile with the 128B XOR swizzle (16-byte chunk index ^= row & 7).  This is the
// same physical layout TMA SWIZZLE_128B writes and wgmma SWIZZLE_128B descriptors read.
HI3D_DEVINL uint32_t swz128(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

HI3D_DEVINL uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// x * sigmoid(x) with ex2.approx + rcp.approx (2 MUFU + 3 FMA-class instructions; the IEEE division of `x / (1 + e)`
// alone was ~10 instructions and made the GroupNorm apply pass issue-bound).  Relative error ~1e-6, output is fp16.
HI3D_DEVINL float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
HI3D_DEVINL float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
// QuickGELU of OpenAI CLIP (clip/model.py QuickGELU): x * sigmoid(1.702 x), in the form of silu_f.
HI3D_DEVINL float quick_gelu_f(float x) { return __fdividef(x, 1.0f + __expf(-1.702f * x)); }

HI3D_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
HI3D_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Eight fp16 values = one 16-byte access.  __half2 has user-provided copy operations, so a plain struct of four of them is
// copied member by member and nvcc emits four 32-bit loads / stores per access (every epilogue, GroupNorm and LayerNorm
// store in round 1 went out as 4-byte writes: partial sectors, ~30 % of HBM bandwidth).  The copy operations below move
// the uint4 view instead, which compiles to LDG.128 / STG.128 / LDS.128 / STS.128.
struct alignas(16) Half8 {
  union {
    uint4 u;
    __half2 h[4];
  };
  __host__ __device__ Half8() {}
  __host__ __device__ Half8(const Half8& o) : u(o.u) {}
  __host__ __device__ Half8& operator=(const Half8& o) {
    u = o.u;
    return *this;
  }
};

// HI3D_ACT_GELU / HI3D_ACT_QUICKGELU (the CLIP towers' MLP activations) on eight staged fp16 GEMM outputs.  Both GEMM
// engines apply them in their store pass, on the fp16 tile, before the residual: the register pass that produces the tile
// (bias, SiLU, GEGLU) is shared by every UNet GEMM, and code added to that unrolled loop slowed those GEMMs down.
HI3D_DEVINL void clip_act_half8(int act, Half8& v) {
#pragma unroll
  for (int q = 0; q < 4; q++) {
    float2 a = __half22float2(v.h[q]);
    if (act == HI3D_ACT_GELU) {
      a.x = gelu_erf_f(a.x);
      a.y = gelu_erf_f(a.y);
    } else {
      a.x = quick_gelu_f(a.x);
      a.y = quick_gelu_f(a.y);
    }
    v.h[q] = __floats2half2_rn(a.x, a.y);
  }
}

}  // namespace hi3d
