/* ctn_b200_probe.h -- verification hook: the library's 1x1 contraction kernels, the training path's streaming kernels and the
 * inference forward's gLN folds, depthwise, residual / skip and statistics kernels called one at a time.
 *
 * The pipelines reach the pointwise contraction kernels (ctn_wgmma.cu, ctn_tcn_simt.cu), the weight-gradient kernels
 * (ctn_wgrad_wgmma.cu, ctn_train.cu), the training path's streaming kernels (ctn_train.cu) and the forward's streaming kernels
 * (ctn_tcn_simt.cu, ctn_causal.cu, ctn_norm.cu, ctn_api.cu) only inside whole models, where normalisations and nonlinearities
 * dilute a kernel's error before any output is compared.  These entry points expose those kernels directly, through the launchers
 * the pipelines call, so that a test can compare one operation with a high-precision reference.  No pipeline calls them; they add
 * no kernels.  Conventions as in ctn_b200.h.
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

/* route 0: the contraction builds the weight image of W into wimg on every call;
 * route 1: the pipelines' batched preparation builds wimg first (operand scale present = fp16 pieces allowed), then the kernel
 * reads it.  Both reach the same image builders.
 * Returns the contraction's status unchanged (CTN_EALIGN, CTN_EUNSUPPORTED, ...).  math CTN_MATH_FP32 ignores wimg. */
int ctn_probe_pw(const ctn_pw_probe_t* p, int pro, int epi, int math, int route, void* wimg, size_t wimg_bytes, ctn_stream_t stream);
/* bytes of the weight image of an (M, K) contraction */
size_t ctn_probe_pw_wimg_bytes(int M, int K, int math);
/* dW (M, K) += sum_{b, t < frames} dY[b][m][t] X[b][k][t]: rows [0, split_row) to dWa, the rest to dWb (nullable);
 * dY_b = dy + b * dy_bs, X_b = x + b * x_bs (floats).  dWa / dWb must be zeroed by the caller.  The training backward's launcher:
 * CTN_MATH_FP32 runs the FFMA split-K kernel, the other modes the wgmma kernel. */
int ctn_probe_wgrad(const float* dy, size_t dy_bs, const float* x, size_t x_bs, float* dWa, float* dWb, int split_row, int M, int K,
                    int B, int frames, int pitch, int math, ctn_stream_t stream);

/* The training path's streaming and filter-bank gradient kernels (ctn_train.cu), one operation per entry point, through the same
 * launchers ctn_convtasnet_fwd_train / ctn_convtasnet_bwd use.  Tensors are (B, C, pitch) floats with pitch % 4 == 0 and
 * 16-byte-aligned rows; stats / sums are (B, 2) doubles; "+=" outputs are accumulated, never cleared.  Nullable pointers are
 * the ones the pipeline passes as null. */
/* y = y + bias[c] in place ; stats[b] += (sum, sumsq) of PReLU(y; slope) over t < frames */
int ctn_probe_bias_prelu_stats(float* y, const float* bias, const float* slope, double* stats, int B, int C, int frames, int pitch,
                               ctn_stream_t stream);
/* upre = dwconv(gLN1(PReLU(hpre; slope1)), wd (C, P), dilation dil, pad_left) + bd ; stats2[b] += (sum, sumsq) of PReLU(upre; slope2).
 * gLN1 from stats1 over n1 elements. */
int ctn_probe_dw_train_fwd(const float* hpre, float* upre, const float* g1, const float* b1, const float* wd, const float* bd,
                           const float* slope1, const float* slope2, const double* stats1, double* stats2, int B, int C, int frames,
                           int pitch, int P, int dil, int pad_left, double n1, float eps, ctn_stream_t stream);
/* y = gLN(act(pre)) from stats over n elements; act = PReLU(slope), identity when slope is null */
int ctn_probe_act_norm(const float* pre, float* y, const float* slope, const float* g, const float* bt, const double* stats, double n,
                       float eps, int B, int C, int frames, int pitch, ctn_stream_t stream);
/* gLN (+ PReLU) backward: dpre (may alias dy); += dgamma, dbeta (phase 1, and sums = per-sample (sum g dy, sum g dy xhat), cleared
 * first) unless reduced; += dslope, dbias (both nullable) */
int ctn_probe_gln_prelu_bwd(const float* dy, const float* pre, float* dpre, const float* slope, const float* g, const double* stats,
                            double n, float eps, double* sums, float* dgamma, float* dbeta, float* dslope, float* dbias, int B, int C,
                            int frames, int pitch, int reduced, ctn_stream_t stream);
/* depthwise backward: dhn = dwconv^T(dupre) ; dwd += taps' gradients ; phase 1 of the gLN1 backward on dhn (+= sums, dgamma, dbeta) */
int ctn_probe_dw_bwd(const float* dupre, const float* hpre, float* dhn, const float* slope1, const float* g1, const float* b1,
                     const double* stats1, double n1, float eps, const float* wd, float* dwd, double* sums, float* dgamma, float* dbeta,
                     int B, int C, int frames, int pitch, int P, int dil, int pad_left, ctn_stream_t stream);
/* sigmoid-mask backward: dwhat (B, S*N, pitch) -> d_mpre in place ; dwprod (B, N, pitch) = sum_s dwhat * mask */
int ctn_probe_mask_bwd(float* dwhat, const float* w, const float* mask, float* dwprod, int B, int S, int N, int frames, int pitch,
                       ctn_stream_t stream);
/* softmax-mask backward (softmax over all S*N channels of a frame): dwprod (B, N, pitch) = sum_s dwhat * mask ; dwhat -> d_z =
 * mask * (dwhat * w - dot) in place, dot = sum_n w * dwprod per frame.  Pad lanes [frames, pitch) of both are written as 0.
 * pitch % 32 == 0 (else CTN_EINVAL) */
int ctn_probe_softmax_mask_bwd(float* dwhat, const float* w, const float* mask, float* dwprod, int B, int S, int N, int frames,
                               int pitch, ctn_stream_t stream);
int ctn_probe_prelu_apply(const float* x, float* y, const float* slope, int B, int C, int frames, int pitch, ctn_stream_t stream);
/* dpre = dy * (pre > 0 ? 1 : slope) (may alias dy) ; dslope += sum_{pre <= 0} dy * pre */
int ctn_probe_prelu_bwd(const float* dy, const float* pre, float* dpre, const float* slope, float* dslope, int B, int C, int frames,
                        int pitch, ctn_stream_t stream);
/* dw = dw + dwprod, and 0 where !(w > 0) when relu */
int ctn_probe_dw_combine(float* dw, const float* dwprod, const float* w, int relu, int B, int C, int frames, int pitch,
                         ctn_stream_t stream);
/* dW (N, L) += sum_{r < R, f < frames} act[r][n][f] * sig[r][f*stride + k - pad_left] (0 outside [0, T)); act (R, N, pitch) */
int ctn_probe_encdec_wgrad(const float* act, const float* sig, float* dW, int R, int N, int frames, int pitch, int T, int L,
                           int stride, int pad_left, ctn_stream_t stream);
/* the same over C signal channels per act row: dW (N, C, L) += sum_{r,f} act[r][n][f] * sig[r*C + c][f*stride + k - pad_left];
 * sig (R*C, T).  C = 1 is ctn_probe_encdec_wgrad. */
int ctn_probe_encdec_wgrad_mc(const float* act, const float* sig, float* dW, int R, int N, int C, int frames, int pitch, int T,
                              int L, int stride, int pad_left, ctn_stream_t stream);
/* out[c] += sum_{b, t < frames} dy[b * bs + c * pitch + t] */
int ctn_probe_rowsum(const float* dy, size_t bs, int C, int B, int frames, int pitch, float* out, ctn_stream_t stream);
/* dst[b][c] (+)= src[b][c], c < C, batch strides dst_bs / src_bs floats; columns [frames, pitch) of dst are written as 0 */
int ctn_probe_rows(float* dst, size_t dst_bs, const float* src, size_t src_bs, int C, int B, int accumulate, int frames, int pitch,
                   ctn_stream_t stream);
/* Wt (K, M) = W (M, K)^T */
int ctn_probe_transpose(const float* W, float* Wt, int M, int K, ctn_stream_t stream);

/* The activation envelope of the fp16-piece mode as a forward computed it (ctn_act_scales), read back from the workspace that
 * forward ran in; call it after the forward, on the same stream.  path: which forward carved the workspace (B, frames, cfg as
 * given to it):
 *   CTN_ENV_TCN    ctn_tcn_fwd, or ctn_tcn_blocks_fwd with cfg.num_blocks = 1, cfg.num_layers = n_blocks;
 *   CTN_ENV_MODEL  ctn_convtasnet_fwd (frames = ctn_frames of its T) or ctn_separator_fwd;
 *   CTN_ENV_TRAIN  ctn_convtasnet_fwd_train (CTN_EUNSUPPORTED when the config does not run the fused TCN forward).
 * With n = num_blocks * num_layers, Hp = hidden rounded up to 16 and Mt = bottleneck + skip, device buffers receive:
 *   scales_out [2n + 1]   the operand scales: [2i] pw1 of block i (x_i), [2i + 1] pw2 (u_i), [2n] the mask contraction;
 *   dwp_out    [n][Hp][8] the packed depthwise parameters (written by the forward only when sep_kernel == 3);
 *   vb_out     [n][Mt]    each block's row bounds of its [out; skip] contraction (skip rows first when it has no out head;
 *                         the Bc rows past them are then not written by the forward);
 *   x0_out     the |x_0| candidates: [1] the measured max |x| (CTN_ENV_TCN), [bottleneck] the head's row bounds otherwise. */
enum { CTN_ENV_TCN = 0, CTN_ENV_MODEL = 1, CTN_ENV_TRAIN = 2 };
int ctn_probe_tcn_envelope(const ctn_config_t* cfg, int B, int frames, int path, void* workspace, float* scales_out, float* dwp_out,
                           float* vb_out, float* x0_out, ctn_stream_t stream);
/* *out = max(*out, max |x| over rows x frames of a pitched (rows, pitch) tensor); *out must hold a non-negative float */
int ctn_probe_absmax_pitch(const float* x, int rows, int frames, int pitch, float* out, ctn_stream_t stream);

/* The inference forward's streaming kernels, through the launchers ctn_convtasnet_fwd / ctn_separator_fwd / ctn_tcn_fwd /
 * ctn_tcn_blocks_fwd and the causal pipeline call.  Tensors (B, C, pitch) floats as above; stats (B, 2) doubles, "+=". */
/* One gLN fold into rows [row_offset, row_offset + M) of (Wf, v1, v2, vb):  Wf[m][k] = W[m][k] gamma[k],
 * v1[m] = sum_k W[m][k] beta[k] + bias[m],  v2[m] = sum_k Wf[m][k],  vb[m] = sum_k |W[m][k]| (|gamma[k]| R + |beta[k]|) + |bias[m]|.
 * bias and vb nullable. */
typedef struct ctn_fold_probe {
  const float* W;
  const float* bias;
  const float* gamma;
  const float* beta;
  int32_t M, K, row_offset;
  float R;
  float* Wf;
  float* v1;
  float* v2;
  float* vb;
} ctn_fold_probe_t;
/* n >= 1 jobs in one call; more than one launch's worth are split the way the pipelines' preparation splits them */
int ctn_probe_fold(const ctn_fold_probe_t* jobs, int n, ctn_stream_t stream);
/* u = PReLU(dwconv(gLN1(h)) + bd; slope) with gLN1 from stats_in over H frames elements, P taps at dilation dil, pad_left
 * ((P-1) dil) / 2 ; stats_out[b] += (sum, sumsq) of u */
int ctn_probe_dw_fwd(const float* h, float* u, const float* norm_g, const float* norm_b, const float* dw_w, const float* dw_b,
                     const float* slope, const double* stats_in, double* stats_out, int B, int H, int frames, int pitch, int P, int dil,
                     float eps, ctn_stream_t stream);
/* x (B, Bc, pitch) += rstd2 r[:, :Bc] + (v1 - mean2 rstd2 v2), r (B, Bc + Sc, pitch), (mean2, rstd2) from stats2 over n2 elements */
int ctn_probe_finish(const float* r, const float* v1, const float* v2, const double* stats2, double n2, float eps, float* x, int B,
                     int Bc, int Sc, int frames, int pitch, ctn_stream_t stream);
/* One block's share of the skip sum: rows [off, off + Sc) of r (B, Mt, pitch), folded constants v1 / v2 (indexed like r's rows) */
typedef struct ctn_skip_probe {
  const float* r;
  const float* v1;
  const float* v2;
  const double* stats2;
  int32_t off, Mt;
} ctn_skip_probe_t;
/* skip (B, Sc, pitch) = sum_i rstd2_i r_i[:, off_i:off_i + Sc] + (v1_i - mean2_i rstd2_i v2_i)[off_i:], 1 <= n <= 64 jobs */
int ctn_probe_skip_reduce(const ctn_skip_probe_t* jobs, int n, double n2, float eps, float* skip, int B, int Sc, int frames, int pitch,
                          ctn_stream_t stream);
/* stats[b] += (sum, sumsq) over c < C, t < frames, in double */
int ctn_probe_stats_pitch(const float* x, int B, int C, int frames, int pitch, double* stats, ctn_stream_t stream);
/* u = PReLU(sum_k wd[c][k] h[c][t + k dil - pad_left] + bd[c]; slope), h = 0 outside [0, frames) */
int ctn_probe_dw_plain(const float* h, float* u, const float* wd, const float* bd, const float* slope, int B, int C, int frames,
                       int pitch, int P, int dil, int pad_left, ctn_stream_t stream);
/* rows of r (B, Mt, pitch): m < Bc (has_out): xout = xin + r + bo[m] (xin == xout: in place); else skip (+)= r + bs[m - Bc]
 * (skip_init: =) */
int ctn_probe_res_skip(const float* r, int Mt, const float* xin, float* xout, float* skip, const float* bo, const float* bs, int Bc,
                       int Sc, int has_out, int skip_init, int B, int frames, int pitch, ctn_stream_t stream);
/* y[b][c][t] += bias[c] */
int ctn_probe_bias_rows(float* y, const float* bias, int C, int B, int frames, int pitch, ctn_stream_t stream);
/* cLN over the first frames columns (in place allowed); scratch double[B][frames][2] */
int ctn_probe_cln_pitch(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int frames, int pitch, float eps,
                        double* scratch, ctn_stream_t stream);

/* The causal training path's streaming kernels (ctn_norm.cu, ctn_causal_train.cu), through the launchers ctn_causal_fwd_train /
 * ctn_causal_bwd call.  mi: float[B][frames][2], the (mean_t, 1 / (std_t + eps)) table of a cLN. */
/* st double[B][frames][2] = inclusive prefix sums over frames of (sum_c, sum_c of squares) of PReLU(x; slope) (slope nullable:
 * of x); mi nullable */
int ctn_probe_cln_stats(const float* x, const float* slope, int B, int C, int frames, int pitch, float eps, double* st, float* mi,
                        ctn_stream_t stream);
/* cLN (+ PReLU(slope) in front, slope nullable) backward from the forward's st: dpre (may alias dy); += dgamma, dbeta, dslope,
 * dbias (the last two nullable).  scratch: 144 * B * frames bytes, 16-byte aligned. */
int ctn_probe_cln_bwd(const float* dy, const float* pre, float* dpre, const float* slope, const float* gamma, const double* st,
                      float eps, void* scratch, float* dgamma, float* dbeta, float* dslope, float* dbias, int B, int C, int frames,
                      int pitch, ctn_stream_t stream);
/* upre = dwconv(cLN1(PReLU(hpre; slope1)), wd (C, P), dilation dil, all (P - 1) dil of the padding on the left) + bd */
int ctn_probe_cdw_train_fwd(const float* hpre, float* upre, const float* mi, const float* g1, const float* b1, const float* wd,
                            const float* bd, const float* slope1, int B, int C, int frames, int pitch, int P, int dil,
                            ctn_stream_t stream);
/* dhn = dwconv^T(dupre) ; dwd += the taps' gradients against hn = cLN1(PReLU(hpre; slope1)) */
int ctn_probe_cdw_bwd(const float* dupre, const float* hpre, float* dhn, const float* mi, const float* g1, const float* b1,
                      const float* slope1, const float* wd, float* dwd, int B, int C, int frames, int pitch, int P, int dil,
                      ctn_stream_t stream);
/* The batched tiled Cholesky of BSS Eval on nmat row-major N x N matrices (N a multiple of 64): the factor overwrites the lower
 * triangle of A, W (nmat, N/64, 64, 64) receives the inverses of its diagonal tiles, flag (nmat) 1 where a pivot was not positive
 * and finite.  Then G X = B for nrhs <= 8 right-hand sides with the factor: route 0 is the one-CTA-per-column solve of
 * ctn_bss_eval_sources, rhs (nmat, nrhs, N); route 1 the all-columns solve of ctn_bss_eval_images, rhs (nmat, N, nrhs) with tmp
 * of the same size.  X overwrites rhs. */
int ctn_probe_chol_factor(double* A, double* W, int32_t* flag, int N, int nmat, ctn_stream_t stream);
int ctn_probe_chol_solve(const double* A, const double* W, double* rhs, double* tmp, int N, int nmat, int nrhs, int route,
                         ctn_stream_t stream);

#ifdef __cplusplus
}
#endif

#endif /* CTN_B200_PROBE_H */
