// Verification hook (include/ctn_b200_probe.h): thin C entry points over the 1x1 contraction internals and the training and
// inference paths' launchers (ctn_internal.h), so that tests can compare one operation with a high-precision reference.  No
// kernels here and no pipeline calls these.
#include <vector>

#include "ctn_internal.h"
#include "ctn_b200_probe.h"

static_assert((int)CTN_PRO_NONE == (int)PRO_NONE && (int)CTN_PRO_PRELU == (int)PRO_PRELU && (int)CTN_PRO_DW == (int)PRO_DW &&
                  (int)CTN_PRO_RES == (int)PRO_RES,
              "prologue selectors");
static_assert((int)CTN_EPI_RAW == (int)EPI_RAW && (int)CTN_EPI_HEAD == (int)EPI_HEAD && (int)CTN_EPI_H == (int)EPI_H &&
                  (int)CTN_EPI_MASK == (int)EPI_MASK && (int)CTN_EPI_MASKDEC == (int)EPI_MASKDEC,
              "epilogue selectors");

namespace {
PwArgs to_pw_args(const ctn_pw_probe_t& p) {
  PwArgs a{};
  a.A = p.A; a.W = p.W; a.D = p.D;
  a.B = p.B; a.M = p.M; a.K = p.K; a.frames = p.frames; a.pitch = p.pitch;
  a.pro_slope = p.pro_slope;
  a.dw_norm_g = p.dw_norm_g; a.dw_norm_b = p.dw_norm_b; a.dw_w = p.dw_w; a.dw_b = p.dw_b;
  a.dw_stats_in = p.dw_stats_in; a.dw_stats_out = p.dw_stats_out;
  a.dw_dilation = p.dw_dilation; a.dw_pad_left = p.dw_pad_left; a.dw_eps = p.dw_eps;
  a.bias = p.bias; a.slope = p.slope; a.v1 = p.v1; a.v2 = p.v2;
  a.stats_in = p.stats_in; a.n_in = p.n_in; a.eps = p.eps; a.stats_out = p.stats_out; a.store_pre = p.store_pre;
  a.wenc = p.wenc; a.Nb = p.Nb; a.mask_out = p.mask_out; a.mask_logits = p.mask_logits;
  a.dec_w = p.dec_w; a.dec_crop_left = p.dec_crop_left; a.dec_T_out = p.dec_T_out;
  a.res_r = p.res_r; a.res_Mt = p.res_Mt; a.res_v1 = p.res_v1; a.res_v2 = p.res_v2;
  a.res_stats = p.res_stats; a.res_n = p.res_n; a.res_eps = p.res_eps; a.res_x_out = p.res_x_out;
  a.wimg = nullptr;
  a.act_scale = p.act_scale;
  a.dw_params = nullptr;  // read by no kernel of ctn_pw (ctn_act_scales fills it for the pipelines)
  a.dw_in_slope = p.dw_in_slope; a.dw_u_pre_out = p.dw_u_pre_out;
  return a;
}
}  // namespace

extern "C" int ctn_probe_pw(const ctn_pw_probe_t* p, int pro, int epi, int math, int route, void* wimg, size_t wimg_bytes,
                            ctn_stream_t stream) {
  if (!p || (route != 0 && route != 1)) return CTN_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  PwArgs a = to_pw_args(*p);
  if (math != CTN_MATH_FP32 && (!wimg || wimg_bytes < ctn_pw_wimg_bytes(a.M, a.K, math))) return CTN_EWORKSPACE;
  if (route == 0) return ctn_pw(a, pro, epi, math, static_cast<float*>(wimg), st);
  WimgJob job{a.W, static_cast<float*>(wimg), a.M, a.K};
  CTN_TRY(ctn_pw_prepare_batch(&job, 1, math, a.act_scale != nullptr, st));
  a.wimg = static_cast<const float*>(wimg);
  return ctn_pw(a, pro, epi, math, nullptr, st);
}

extern "C" size_t ctn_probe_pw_wimg_bytes(int M, int K, int math) { return ctn_pw_wimg_bytes(M, K, math); }

extern "C" int ctn_probe_wgrad(const float* dy, size_t dy_bs, const float* x, size_t x_bs, float* dWa, float* dWb, int split_row, int M,
                               int K, int B, int frames, int pitch, int math, ctn_stream_t stream) {
  return ctn_wgrad(math, dy, dy_bs, x, x_bs, dWa, dWb, split_row, M, K, B, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_bias_prelu_stats(float* y, const float* bias, const float* slope, double* stats, int B, int C, int frames,
                                          int pitch, ctn_stream_t stream) {
  return ctn_bias_prelu_stats(y, bias, slope, stats, B, C, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_dw_train_fwd(const float* hpre, float* upre, const float* g1, const float* b1, const float* wd,
                                      const float* bd, const float* slope1, const float* slope2, const double* stats1, double* stats2,
                                      int B, int C, int frames, int pitch, int P, int dil, int pad_left, double n1, float eps,
                                      ctn_stream_t stream) {
  return ctn_dw_train_fwd(hpre, upre, g1, b1, wd, bd, slope1, slope2, stats1, stats2, B, C, frames, pitch, P, dil, pad_left, n1, eps,
                          (cudaStream_t)stream);
}

extern "C" int ctn_probe_act_norm(const float* pre, float* y, const float* slope, const float* g, const float* bt, const double* stats,
                                  double n, float eps, int B, int C, int frames, int pitch, ctn_stream_t stream) {
  return ctn_act_norm(pre, y, slope, g, bt, stats, n, eps, B, C, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_gln_prelu_bwd(const float* dy, const float* pre, float* dpre, const float* slope, const float* g,
                                       const double* stats, double n, float eps, double* sums, float* dgamma, float* dbeta,
                                       float* dslope, float* dbias, int B, int C, int frames, int pitch, int reduced,
                                       ctn_stream_t stream) {
  return ctn_gln_prelu_bwd(dy, pre, dpre, slope, g, stats, n, eps, sums, dgamma, dbeta, dslope, dbias, B, C, frames, pitch,
                           (cudaStream_t)stream, reduced != 0);
}

extern "C" int ctn_probe_dw_bwd(const float* dupre, const float* hpre, float* dhn, const float* slope1, const float* g1, const float* b1,
                                const double* stats1, double n1, float eps, const float* wd, float* dwd, double* sums, float* dgamma,
                                float* dbeta, int B, int C, int frames, int pitch, int P, int dil, int pad_left, ctn_stream_t stream) {
  return ctn_dw_bwd(dupre, hpre, dhn, slope1, g1, b1, stats1, n1, eps, wd, dwd, sums, dgamma, dbeta, B, C, frames, pitch, P, dil,
                    pad_left, (cudaStream_t)stream);
}

extern "C" int ctn_probe_mask_bwd(float* dwhat, const float* w, const float* mask, float* dwprod, int B, int S, int N, int frames,
                                  int pitch, ctn_stream_t stream) {
  return ctn_mask_bwd(dwhat, w, mask, dwprod, B, S, N, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_softmax_mask_bwd(float* dwhat, const float* w, const float* mask, float* dwprod, int B, int S, int N,
                                          int frames, int pitch, ctn_stream_t stream) {
  LaunchScope scope(dwhat);
  return ctn_softmax_mask_bwd(dwhat, w, mask, dwprod, B, S, N, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_prelu_apply(const float* x, float* y, const float* slope, int B, int C, int frames, int pitch,
                                     ctn_stream_t stream) {
  return ctn_prelu_apply(x, y, slope, B, C, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_prelu_bwd(const float* dy, const float* pre, float* dpre, const float* slope, float* dslope, int B, int C,
                                   int frames, int pitch, ctn_stream_t stream) {
  return ctn_prelu_bwd(dy, pre, dpre, slope, dslope, B, C, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_dw_combine(float* dw, const float* dwprod, const float* w, int relu, int B, int C, int frames, int pitch,
                                    ctn_stream_t stream) {
  return ctn_dw_combine(dw, dwprod, w, relu, B, C, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_encdec_wgrad(const float* act, const float* sig, float* dW, int R, int N, int frames, int pitch, int T, int L,
                                      int stride, int pad_left, ctn_stream_t stream) {
  return ctn_encdec_wgrad(act, sig, dW, R, N, 1, frames, pitch, T, L, stride, pad_left, (cudaStream_t)stream);
}

extern "C" int ctn_probe_encdec_wgrad_mc(const float* act, const float* sig, float* dW, int R, int N, int C, int frames, int pitch, int T,
                                         int L, int stride, int pad_left, ctn_stream_t stream) {
  if (C < 1) return CTN_EINVAL;
  return ctn_encdec_wgrad(act, sig, dW, R, N, C, frames, pitch, T, L, stride, pad_left, (cudaStream_t)stream);
}

extern "C" int ctn_probe_rowsum(const float* dy, size_t bs, int C, int B, int frames, int pitch, float* out, ctn_stream_t stream) {
  return ctn_rowsum(dy, bs, C, B, frames, pitch, out, (cudaStream_t)stream);
}

extern "C" int ctn_probe_rows(float* dst, size_t dst_bs, const float* src, size_t src_bs, int C, int B, int accumulate, int frames,
                              int pitch, ctn_stream_t stream) {
  return ctn_rows(dst, dst_bs, src, src_bs, C, B, accumulate, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_transpose(const float* W, float* Wt, int M, int K, ctn_stream_t stream) {
  return ctn_transpose(W, Wt, M, K, (cudaStream_t)stream);
}

static_assert((int)CTN_ENV_TCN == (int)ENV_TCN && (int)CTN_ENV_MODEL == (int)ENV_MODEL && (int)CTN_ENV_TRAIN == (int)ENV_TRAIN,
              "envelope paths");

extern "C" int ctn_probe_tcn_envelope(const ctn_config_t* cfg, int B, int frames, int path, void* workspace, float* scales_out,
                                      float* dwp_out, float* vb_out, float* x0_out, ctn_stream_t stream) {
  if (!scales_out || !dwp_out || !vb_out || !x0_out) return CTN_EINVAL;
  EnvelopeView v;
  CTN_TRY(ctn_envelope_view(cfg, B, frames, path, workspace, &v));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t dwp_n = (size_t)ctn_round_up(cfg->hidden, 16) * 8, vb_n = (size_t)cfg->bottleneck + cfg->skip;
  const cudaMemcpyKind d2d = cudaMemcpyDeviceToDevice;
  cudaError_t e = cudaMemcpyAsync(scales_out, v.scales, sizeof(float) * (2 * v.n + 1), d2d, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(x0_out, v.x0_bound, sizeof(float) * v.x0_n, d2d, st);
  for (int i = 0; i < v.n && e == cudaSuccess; ++i) {
    e = cudaMemcpyAsync(dwp_out + i * dwp_n, v.dwp[i], sizeof(float) * dwp_n, d2d, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(vb_out + i * vb_n, v.vb[i], sizeof(float) * vb_n, d2d, st);
  }
  return (int)e;
}

extern "C" int ctn_probe_absmax_pitch(const float* x, int rows, int frames, int pitch, float* out, ctn_stream_t stream) {
  return ctn_absmax_pitch(x, rows, frames, pitch, out, (cudaStream_t)stream);
}

extern "C" int ctn_probe_fold(const ctn_fold_probe_t* jobs, int n, ctn_stream_t stream) {
  if (!jobs || n <= 0) return CTN_EINVAL;
  std::vector<FoldJob> fj((size_t)n);
  for (int i = 0; i < n; ++i) {
    const ctn_fold_probe_t& p = jobs[i];
    fj[i] = FoldJob{p.W, p.bias, p.gamma, p.beta, FoldedConv{p.Wf, p.v1, p.v2, p.vb}, p.M, p.K, p.row_offset, p.R};
  }
  return ctn_fold_batch(fj.data(), n, (cudaStream_t)stream);
}

extern "C" int ctn_probe_dw_fwd(const float* h, float* u, const float* norm_g, const float* norm_b, const float* dw_w, const float* dw_b,
                                const float* slope, const double* stats_in, double* stats_out, int B, int H, int frames, int pitch, int P,
                                int dil, float eps, ctn_stream_t stream) {
  return ctn_dw_fwd(h, u, norm_g, norm_b, dw_w, dw_b, slope, stats_in, stats_out, B, H, frames, pitch, P, dil, eps, (cudaStream_t)stream);
}

extern "C" int ctn_probe_finish(const float* r, const float* v1, const float* v2, const double* stats2, double n2, float eps, float* x,
                                int B, int Bc, int Sc, int frames, int pitch, ctn_stream_t stream) {
  const FoldedConv f{nullptr, const_cast<float*>(v1), const_cast<float*>(v2), nullptr};  // k_finish reads v1 / v2 only
  return ctn_finish_fwd(r, f, stats2, n2, eps, x, B, Bc, Sc, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_skip_reduce(const ctn_skip_probe_t* jobs, int n, double n2, float eps, float* skip, int B, int Sc, int frames,
                                     int pitch, ctn_stream_t stream) {
  if (!jobs || n <= 0 || n > CTN_MAX_BLOCKS) return CTN_EINVAL;
  SkipJobs sj;
  sj.n = n;
  for (int i = 0; i < n; ++i) sj.j[i] = SkipJob{jobs[i].r, jobs[i].v1, jobs[i].v2, jobs[i].stats2, jobs[i].off, jobs[i].Mt};
  return ctn_skip_reduce(sj, n2, eps, skip, B, Sc, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_stats_pitch(const float* x, int B, int C, int frames, int pitch, double* stats, ctn_stream_t stream) {
  return ctn_stats_pitch(x, B, C, frames, pitch, stats, (cudaStream_t)stream);
}

extern "C" int ctn_probe_dw_plain(const float* h, float* u, const float* wd, const float* bd, const float* slope, int B, int C, int frames,
                                  int pitch, int P, int dil, int pad_left, ctn_stream_t stream) {
  return ctn_dw_plain_fwd(h, u, wd, bd, slope, B, C, frames, pitch, P, dil, pad_left, (cudaStream_t)stream);
}

extern "C" int ctn_probe_res_skip(const float* r, int Mt, const float* xin, float* xout, float* skip, const float* bo, const float* bs,
                                  int Bc, int Sc, int has_out, int skip_init, int B, int frames, int pitch, ctn_stream_t stream) {
  return ctn_res_skip_fwd(r, Mt, xin, xout, skip, bo, bs, Bc, Sc, has_out, skip_init, B, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_bias_rows(float* y, const float* bias, int C, int B, int frames, int pitch, ctn_stream_t stream) {
  return ctn_bias_rows_fwd(y, bias, C, B, frames, pitch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_cln_pitch(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int frames, int pitch,
                                   float eps, double* scratch, ctn_stream_t stream) {
  return ctn_cln_pitch_fwd(x, gamma, beta, y, B, C, frames, pitch, eps, scratch, (cudaStream_t)stream);
}

extern "C" int ctn_probe_cln_stats(const float* x, const float* slope, int B, int C, int frames, int pitch, float eps, double* st,
                                   float* mi, ctn_stream_t stream) {
  return ctn_cln_stats(x, slope, B, C, frames, pitch, eps, st, reinterpret_cast<float2*>(mi), (cudaStream_t)stream);
}

extern "C" int ctn_probe_cln_bwd(const float* dy, const float* pre, float* dpre, const float* slope, const float* gamma, const double* st,
                                 float eps, void* scratch, float* dgamma, float* dbeta, float* dslope, float* dbias, int B, int C,
                                 int frames, int pitch, ctn_stream_t stream) {
  if (!scratch || (((uintptr_t)scratch) & 15)) return CTN_EALIGN;
  double* part = static_cast<double*>(scratch);
  float4* tab = reinterpret_cast<float4*>(part + ctn_cln_bwd_part_doubles(B, frames));
  return ctn_cln_bwd_pitch(dy, pre, dpre, slope, gamma, st, eps, part, tab, dgamma, dbeta, dslope, dbias, B, C, frames, pitch,
                           (cudaStream_t)stream);
}

extern "C" int ctn_probe_cdw_train_fwd(const float* hpre, float* upre, const float* mi, const float* g1, const float* b1, const float* wd,
                                       const float* bd, const float* slope1, int B, int C, int frames, int pitch, int P, int dil,
                                       ctn_stream_t stream) {
  return ctn_cdw_train_fwd(hpre, upre, reinterpret_cast<const float2*>(mi), g1, b1, wd, bd, slope1, B, C, frames, pitch, P, dil,
                           (cudaStream_t)stream);
}

extern "C" int ctn_probe_cdw_bwd(const float* dupre, const float* hpre, float* dhn, const float* mi, const float* g1, const float* b1,
                                 const float* slope1, const float* wd, float* dwd, int B, int C, int frames, int pitch, int P, int dil,
                                 ctn_stream_t stream) {
  return ctn_cdw_bwd(dupre, hpre, dhn, reinterpret_cast<const float2*>(mi), g1, b1, slope1, wd, dwd, B, C, frames, pitch, P, dil,
                     (cudaStream_t)stream);
}

extern "C" int ctn_probe_chol_factor(double* A, double* W, int32_t* flag, int N, int nmat, ctn_stream_t stream) {
  LaunchScope scope(A);
  if (!A || !W || !flag || N < BSS_NB || N % BSS_NB || nmat < 1 || nmat > 65535) return CTN_EINVAL;
  return ctn_chol_factor(MatSet{A, W, flag, N, N / BSS_NB, nmat}, (cudaStream_t)stream);
}

extern "C" int ctn_probe_chol_solve(const double* A, const double* W, double* rhs, double* tmp, int N, int nmat, int nrhs, int route,
                                    ctn_stream_t stream) {
  LaunchScope scope(A);
  if (!A || !W || !rhs || N < BSS_NB || N % BSS_NB || nmat < 1 || nmat > 65535 || nrhs < 1 || nrhs > 8) return CTN_EINVAL;
  const MatSet s{const_cast<double*>(A), const_cast<double*>(W), nullptr, N, N / BSS_NB, nmat};
  if (route == 0) return ctn_chol_solve_cols(s, rhs, nrhs, (cudaStream_t)stream);
  if (route == 1 && tmp) return ctn_chol_solve_multi(s, rhs, tmp, nrhs, (cudaStream_t)stream);
  return CTN_EINVAL;
}
