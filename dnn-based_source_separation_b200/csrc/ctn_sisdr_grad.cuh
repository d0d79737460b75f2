// Gradient of one SI-SDR pair w.r.t. its estimate, from the pair statistics (src/criterion/sdr.py:135-137):
//   SI-SDR = k (ln P - ln Q),  P = alpha^2 |t|^2 + eps,  Q = |alpha t - x|^2 + eps,  alpha = <x,t> / (|t|^2 + eps)
//   g * dSI-SDR/dx = ct * t + cx * x
//   ct = g k { 2 alpha tt / ((tt+eps) P)  -  (2 (alpha tt - xt)/(tt+eps) - 2 alpha) / Q },   cx = g k (-2 / Q)
// xt = <x,t>, den = |alpha t - x|^2 (explicit residual), tt = |t|^2, all accumulated in double by the forward.
// Shared by the PIT backward (ctn_loss.cu) and the ORPIT / SinkPIT backward (ctn_pitx.cu).  The weight g is taken as a
// callable evaluated after the pair terms, the order k_sisdr_pit_bwd has always computed them in.
#pragma once

template <class Weight>
__device__ __forceinline__ void sisdr_grad_coef(double xt, double den, double tt, double e, Weight weight, float& ct, float& cx) {
  const double alpha = xt / (tt + e), P = alpha * alpha * tt + e, Q = den + e;
  const double k10 = 4.342944819032518;  // 10 / ln 10
  const double g = weight();
  ct = (float)(g * k10 * (2.0 * alpha * tt / ((tt + e) * P) - (2.0 * (alpha * tt - xt) / (tt + e) - 2.0 * alpha) / Q));
  cx = (float)(g * k10 * (-2.0 / Q));
}
