// Online softmax of the d = 64 flash-attention kernels (attn_tc5.cu in fp16, attn_fp8_tc5.cu in e4m3): the exponentials and
// the per-tile max / sum / correction update, on the wgmma f32 accumulator fragment of S.
#pragma once
#include "common.cuh"

namespace hi3d {

// 2^x for x < 128 on the FMA pipe:x = j + f, 2^f by a cubic (relative error 1.6e-4), 2^j added to the exponent bits.
HI3D_DEVINL float exp2_fma(float x) {
  x = fmaxf(x, -127.f);
  const float j = floorf(x);
  const float f = x - j;
  const float p = fmaf(fmaf(fmaf(0.07640766f, f, 0.22823162f), f, 0.6950504f), f, 1.0f);
  return __int_as_float(__float_as_int(p) + ((int)j << 23));
}

// 2^x on the MUFU pipe.  exp2f adds a range test and two multiplies around MUFU.EX2 to produce denormal results; P is
// rounded to fp16 or e4m3 (which flush them to zero anyway) and the row sums are >= 1, so the flush-to-zero form loses nothing.
HI3D_DEVINL float exp2_mufu(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}

// Online softmax of one S tile (key tile j) in place: masks the key tail, updates the running max / sum of this thread's
// rows g (hh = 0) and g + 8 (hh = 1) of its warp's 16, leaves P (fp32) in the S registers and returns the factor by which
// the accumulator must be rescaled.  P is packed into the A fragments of P V separately, once the previous P V that reads
// those registers has retired.
// EMU8: eighths of the key columns whose exponentials run on the FMA pipe -- a template parameter, so that each column's
// pipe is fixed at compile time (a run-time fraction made every exponential compute both forms and select one).
// PLOG2: P comes out scaled by 2^PLOG2 (exp2(s c - m c + PLOG2)), and so does the running sum; the e4m3 kernel uses it to keep
// small probabilities above e4m3's underflow.  The final O / l is unchanged.
template <int BN, int EMU8, int PLOG2 = 0>
HI3D_DEVINL void fa_softmax(float (&sc)[BN / 2], float (&mrow)[2], float (&lrow)[2], float (&corr)[2], int j, int L,
                            float c, int t4) {
  if ((j + 1) * BN > L) {
#pragma unroll
    for (int nt = 0; nt < BN / 8; nt++) {
      const int col = j * BN + nt * 8 + 2 * t4;
      if (col >= L) { sc[4 * nt] = -INFINITY; sc[4 * nt + 2] = -INFINITY; }
      if (col + 1 >= L) { sc[4 * nt + 1] = -INFINITY; sc[4 * nt + 3] = -INFINITY; }
    }
  }
#pragma unroll
  for (int hh = 0; hh < 2; hh++) {
    float mx = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < BN / 8; nt++) mx = fmaxf(mx, fmaxf(sc[4 * nt + 2 * hh], sc[4 * nt + 2 * hh + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float mnew = fmaxf(mrow[hh], mx);
    corr[hh] = exp2_mufu((mrow[hh] - mnew) * c);
    float moff;
    if constexpr (PLOG2 == 0) moff = mnew * c;
    else moff = fmaf(mnew, c, -(float)PLOG2);
    float rs = 0.f;
#pragma unroll
    for (int nt = 0; nt < BN / 8; nt++) {
      const float x0 = sc[4 * nt + 2 * hh] * c - moff, x1 = sc[4 * nt + 2 * hh + 1] * c - moff;
      const bool fma_pipe = (nt & 7) < EMU8;
      const float p0 = fma_pipe ? exp2_fma(x0) : exp2_mufu(x0);
      const float p1 = fma_pipe ? exp2_fma(x1) : exp2_mufu(x1);
      rs += p0 + p1;
      sc[4 * nt + 2 * hh] = p0;
      sc[4 * nt + 2 * hh + 1] = p1;
    }
    lrow[hh] = lrow[hh] * corr[hh] + rs;
    mrow[hh] = mnew;
  }
}

}  // namespace hi3d
