// Depthwise-stage math shared by the fused depthwise + pointwise producers (ctn_wgmma.cu).
#pragma once
#include "ctn_common.cuh"

// ---- depthwise producer math (PRO_DW) -------------------------------------------------------------------------
// One channel, 4 consecutive time steps.  q0,q1,q2: the three aligned 128-bit loads (d >= 4: taps t-d, t, t+d;
// d < 4: the window [t-4, t+8)).  DCLS in {1, 2, 4(=d>=4)} selects the tap positions at compile time.
// INTERIOR tiles (every tap of every element inside [0, frames)) fold gLN1 into the taps: 3 FMA per output.
// KEEP_PRE (training forward): also returns the PRE-activation (dwconv + bias, zero at the padded positions) through `pre`.
template <int DCLS, bool INTERIOR, bool KEEP_PRE = false>
__device__ __forceinline__ float4 dw_channel(const float4 q0, const float4 q1, const float4 q2, float gsc, float gsh, float w0,
                                             float w1, float w2, float bd, float slope, int first, int step, int tbase,
                                             int frames, bool cvalid, float2& ls, float2& lss, float4* pre = nullptr) {
  const float win[12] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w};
  constexpr int i0 = DCLS == 4 ? 0 : (DCLS == 2 ? 2 : 3);
  constexpr int i1 = 4;
  constexpr int i2 = DCLS == 4 ? 8 : (DCLS == 2 ? 6 : 5);
  float o[4];
  if (INTERIOR) {
    const float a0 = gsc * w0, a1 = gsc * w1, a2 = gsc * w2;
    const float cst = fmaf(gsh, (w0 + w1) + w2, bd);
#pragma unroll
    for (int e = 0; e < 4; ++e) o[e] = fmaf(a2, win[i2 + e], fmaf(a1, win[i1 + e], fmaf(a0, win[i0 + e], cst)));
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      // absolute time of the three taps of element e
      const int t0 = DCLS == 4 ? first + e : first + i0 + e;
      const int t1 = DCLS == 4 ? first + step + e : first + i1 + e;
      const int t2 = DCLS == 4 ? first + 2 * step + e : first + i2 + e;
      const float h0 = (t0 >= 0 && t0 < frames) ? fmaf(win[i0 + e], gsc, gsh) : 0.f;
      const float h1 = (t1 >= 0 && t1 < frames) ? fmaf(win[i1 + e], gsc, gsh) : 0.f;
      const float h2 = (t2 >= 0 && t2 < frames) ? fmaf(win[i2 + e], gsc, gsh) : 0.f;
      o[e] = fmaf(w2, h2, fmaf(w1, h1, fmaf(w0, h0, bd)));
    }
  }
  if (KEEP_PRE) {
    float pz[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) pz[e] = (!INTERIOR && (tbase + e >= frames || !cvalid)) ? 0.f : o[e];
    *pre = make_float4(pz[0], pz[1], pz[2], pz[3]);
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float u = prelu_f(o[e], slope);
    if (!INTERIOR && (tbase + e >= frames || !cvalid)) u = 0.f;
    o[e] = u;
  }
  ls.x += o[0] + o[2];
  ls.y += o[1] + o[3];
  lss.x = fmaf(o[2], o[2], fmaf(o[0], o[0], lss.x));
  lss.y = fmaf(o[3], o[3], fmaf(o[1], o[1], lss.y));
  return make_float4(o[0], o[1], o[2], o[3]);
}

