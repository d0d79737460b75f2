// Verification hook (include/ctn_b200_probe.h): thin C entry points over the 1x1 contraction internals, so that tests can
// compare one contraction with a high-precision reference.  No kernels here and no pipeline calls these.
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
  return ctn_wgrad_wgmma(dy, dy_bs, x, x_bs, dWa, dWb, split_row, M, K, B, frames, pitch, math, (cudaStream_t)stream);
}
