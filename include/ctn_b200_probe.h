/* ctn_b200_probe.h -- verification hook: the library's 1x1 contraction kernels called one at a time.
 *
 * The pipelines reach the pointwise contraction kernels (ctn_wgmma.cu, ctn_tcn_simt.cu) and the weight-gradient kernel
 * (ctn_wgrad_wgmma.cu) only inside whole models, where normalisations and nonlinearities dilute a kernel's error before any
 * output is compared.  These entry points expose those kernels directly so that a test can compare one contraction with a
 * high-precision reference.  No pipeline calls them; they add no kernels.  Conventions as in ctn_b200.h.
 */
#ifndef CTN_B200_PROBE_H
#define CTN_B200_PROBE_H

#include "ctn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* prologue / epilogue selectors (ctn_internal.h) */
enum { CTN_PRO_NONE = 0, CTN_PRO_PRELU = 1, CTN_PRO_DW = 2, CTN_PRO_RES = 3 };
enum { CTN_EPI_RAW = 0, CTN_EPI_HEAD = 1, CTN_EPI_H = 2, CTN_EPI_MASK = 3, CTN_EPI_MASKDEC = 4 };

/* One contraction D[b][n][t] = epi( sum_k W[n][k] pro(A[b][k][t]) ).  Field for field the library's internal argument block
 * (PwArgs, ctn_internal.h), in plain C types; every pointer is nullable where the prologue / epilogue does not read it. */
typedef struct ctn_pw_probe {
  const float* A;
  const float* W;
  float* D;
  int32_t B, M, K, frames, pitch;
  const float* pro_slope;
  const float* dw_norm_g;
  const float* dw_norm_b;
  const float* dw_w;
  const float* dw_b;
  const double* dw_stats_in;
  double* dw_stats_out;
  int32_t dw_dilation, dw_pad_left;
  float dw_eps;
  const float* bias;
  const float* slope;
  const float* v1;
  const float* v2;
  const double* stats_in;
  double n_in;
  float eps;
  double* stats_out;
  int32_t store_pre;
  const float* wenc;
  int32_t Nb;
  float* mask_out;
  int32_t mask_logits;
  const float* dec_w;
  int32_t dec_crop_left, dec_T_out;
  const float* res_r;
  int32_t res_Mt;
  const float* res_v1;
  const float* res_v2;
  const double* res_stats;
  double res_n;
  float res_eps;
  float* res_x_out;
  const float* act_scale;
  const float* dw_in_slope;
  float* dw_u_pre_out;
} ctn_pw_probe_t;

/* route 0: the weight image of W is built into wimg on every call (the per-call builders);
 * route 1: the batched builders prepare wimg first (operand scale present = fp16 pieces allowed), then the kernel reads it.
 * Returns the contraction's status unchanged (CTN_EALIGN, CTN_EUNSUPPORTED, ...).  math CTN_MATH_FP32 ignores wimg. */
int ctn_probe_pw(const ctn_pw_probe_t* p, int pro, int epi, int math, int route, void* wimg, size_t wimg_bytes, ctn_stream_t stream);
/* bytes of the weight image of an (M, K) contraction */
size_t ctn_probe_pw_wimg_bytes(int M, int K, int math);
/* dW (M, K) += sum_{b, t < frames} dY[b][m][t] X[b][k][t]: rows [0, split_row) to dWa, the rest to dWb (nullable);
 * dY_b = dy + b * dy_bs, X_b = x + b * x_bs (floats).  dWa / dWb must be zeroed by the caller. */
int ctn_probe_wgrad(const float* dy, size_t dy_bs, const float* x, size_t x_bs, float* dWa, float* dWb, int split_row, int M, int K,
                    int B, int frames, int pitch, int math, ctn_stream_t stream);

#ifdef __cplusplus
}
#endif

#endif /* CTN_B200_PROBE_H */
