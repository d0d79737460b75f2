// GALRNet stages.  Reference: src/models/galr.py:135-197 (LowDimensionGloballyAttentiveBlock), src/models/galrnet.py:222-240
// (Separator head).
//
// The dual-path state is channels-last, X (B, S, K, F), as on the DPTNet path; the intra-chunk block is the DPRNN one unchanged
// (ctn_bilstm_proj_fwd + ctn_dprnn_norm_res2_fwd, swap = 0).  One LowDimensionGloballyAttentiveBlock is
//   * down-map (k_galr_down, one CTA per (b, s)): fc_map along the chunk axis, K -> Q, in fp32 FMAs; LayerNorm over the F channels
//     of each of the Q tokens, mean then centred variance in double; plus the sinusoidal encoding of position p = s Q + q, feature
//     f < F/2: sin(p / d[f]), else cos(p / d[f - F/2]) (concatenated, not interleaved).  The divisors d = 10000^(j / F) come from
//     the caller, formed on the host with the reference's own fp32 expression: in-kernel powf would move arguments of a few
//     thousand radians by 1e-4.  p / d is an IEEE division and sinf / cosf are the full-precision ones (no fast math here).
//     The result is stored Zt (B, Q, S, F): every attention sequence (b, q) of S tokens is contiguous;
//   * attention: ctn_mha_fwd over the B Q sequences, as it is;
//   * gLN statistics of Y + Zt per sample, over (Q, S, F), in double over fixed slices (ctn_sample_gln_stats), no atomics;
//   * up-map (k_galr_up, one CTA per (b, s)): the gLN of the Q x F slab of Y + Zt of chunk s, fc_inv (Q -> K) and the block input.
#include <math.h>

#include "ctn_internal.h"

namespace {

constexpr int GT = 256;              // threads per CTA of the down- and up-map
constexpr int GR = 8;                // output rows per thread and pass
constexpr int GKT = 32;              // reduction rows staged in shared memory per tile
constexpr int GMAX_F = 128;
constexpr int GROWS = GT / 32 * GR;  // most output rows per pass (F = 32)

bool galr_ok(int F, int K, int Q) { return (F == 32 || F == 64 || F == 128) && K >= 1 && Q >= 1 && Q <= K; }

size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }

// x (B, S, K, F) -> zt (B, Q, S, F) = LN_F(fc_map(x) along K) + pe.  grid (S, B), block 256.  Thread (grp, f): grp = tid / F,
// rows grp + r (256 / F) of each pass of (256 / F) * 8 tokens; the K reduction runs over tiles of 32 rows of x and of fc_map in
// shared memory (k ascending), then one warp per token normalises it.
__global__ void __launch_bounds__(GT) k_galr_down(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ bias,
                                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                                  const float* __restrict__ pe_div, float* __restrict__ zt, int S, int K, int Q, int F,
                                                  float eps) {
  __shared__ float xs[GKT][GMAX_F];
  __shared__ float ws[GROWS][GKT + 1];
  __shared__ float res[GROWS * 32];
  const int s = blockIdx.x, b = blockIdx.y;
  const int groups = GT / F, f = threadIdx.x % F, grp = threadIdx.x / F, QP = groups * GR;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* xt = x + ((size_t)b * S + s) * K * F;
  for (int q0 = 0; q0 < Q; q0 += QP) {
    float acc[GR];
#pragma unroll
    for (int r = 0; r < GR; ++r) acc[r] = 0.f;
    for (int k0 = 0; k0 < K; k0 += GKT) {
      const int nk = K - k0 < GKT ? K - k0 : GKT;
      __syncthreads();  // the previous tiles (and the previous pass's res) are consumed
      for (int i = threadIdx.x; i < nk * F; i += GT) xs[i / F][i % F] = xt[(size_t)k0 * F + i];
      for (int i = threadIdx.x; i < QP * GKT; i += GT) {
        const int r = i / GKT, kk = i % GKT, q = q0 + r;
        ws[r][kk] = (q < Q && kk < nk) ? __ldg(W + (size_t)q * K + k0 + kk) : 0.f;
      }
      __syncthreads();
      for (int kk = 0; kk < nk; ++kk) {
        const float xv = xs[kk][f];
#pragma unroll
        for (int r = 0; r < GR; ++r) acc[r] = fmaf(ws[grp + r * groups][kk], xv, acc[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < GR; ++r) {
      const int row = grp + r * groups, q = q0 + row;
      if (q < Q) res[row * F + f] = acc[r] + __ldg(bias + q);
    }
    __syncthreads();
    const int nq = Q - q0 < QP ? Q - q0 : QP;
    for (int row = warp; row < nq; row += GT / 32) {
      const int q = q0 + row, per = F / 32;
      float v[GMAX_F / 32];
      double sum = 0.0;
#pragma unroll
      for (int j = 0; j < GMAX_F / 32; ++j) {
        v[j] = j < per ? res[row * F + lane + 32 * j] : 0.f;
        sum += (double)v[j];
      }
      const double mean = warp_sum_d(sum) / F;
      double var = 0.0;
#pragma unroll
      for (int j = 0; j < GMAX_F / 32; ++j) {
        const double d = j < per ? (double)v[j] - mean : 0.0;
        var = fma(d, d, var);
      }
      const double rstd = 1.0 / sqrt(warp_sum_d(var) / F + (double)eps);
      const float p = (float)(s * Q + q);
      const int half = F / 2;
      float* dst = zt + (((size_t)b * Q + q) * S + s) * F;
#pragma unroll
      for (int j = 0; j < GMAX_F / 32; ++j) {
        if (j >= per) break;
        const int ff = lane + 32 * j;
        const float xn = (float)(((double)v[j] - mean) * rstd);
        const float pe = ff < half ? sinf(p / __ldg(pe_div + ff)) : cosf(p / __ldg(pe_div + ff - half));
        dst[ff] = fmaf(xn, __ldg(gamma + ff), __ldg(beta + ff)) + pe;
      }
    }
  }
}

// out (B, S, K, F) = fc_inv(gLN(Y + Zt)) along Q + x, for chunk s of sample b: the Q x F slab of Y + Zt normalised with the
// sample's statistics (G partials summed in slice order) as it is staged, 32 rows at a time; q ascending.  grid (S, B),
// block 256, rows of K split into passes as in k_galr_down.  out may alias x (each element is read, then written, by one thread).
__global__ void __launch_bounds__(GT) k_galr_up(const float* __restrict__ Y, const float* __restrict__ zt, const double* __restrict__ part,
                                                int G, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                const float* __restrict__ W, const float* __restrict__ bias, const float* x, float* out,
                                                int S, int K, int Q, int F, float eps) {
  __shared__ float gs[GKT][GMAX_F];
  __shared__ float ws[GROWS][GKT + 1];
  __shared__ double st[2];
  const int s = blockIdx.x, b = blockIdx.y;
  const int groups = GT / F, f = threadIdx.x % F, grp = threadIdx.x / F, KP = groups * GR;
  const float2 mr = sample_gln_mean_rstd(part, G, b, (double)Q * S * F, eps, st);
  const float gf = __ldg(gamma + f), bf = __ldg(beta + f);
  const size_t xo = ((size_t)b * S + s) * K * F;
  for (int k0 = 0; k0 < K; k0 += KP) {
    float acc[GR];
#pragma unroll
    for (int r = 0; r < GR; ++r) acc[r] = 0.f;
    for (int q0 = 0; q0 < Q; q0 += GKT) {
      const int nq = Q - q0 < GKT ? Q - q0 : GKT;
      __syncthreads();
      for (int i = threadIdx.x; i < nq * F; i += GT) {
        const int qq = i / F, c = i % F;  // c == f: F divides 256
        const size_t at = (((size_t)b * Q + q0 + qq) * S + s) * F + c;
        gs[qq][c] = fmaf((Y[at] + zt[at] - mr.x) * mr.y, gf, bf);
      }
      for (int i = threadIdx.x; i < KP * GKT; i += GT) {
        const int r = i / GKT, qq = i % GKT, k = k0 + r;
        ws[r][qq] = (k < K && qq < nq) ? __ldg(W + (size_t)k * Q + q0 + qq) : 0.f;
      }
      __syncthreads();
      for (int qq = 0; qq < nq; ++qq) {
        const float gv = gs[qq][f];
#pragma unroll
        for (int r = 0; r < GR; ++r) acc[r] = fmaf(ws[grp + r * groups][qq], gv, acc[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < GR; ++r) {
      const int k = k0 + grp + r * groups;
      if (k < K) {
        const size_t at = xo + (size_t)k * F + f;
        out[at] = acc[r] + __ldg(bias + k) + x[at];
      }
    }
  }
}

}  // namespace

// ---- one LowDimensionGloballyAttentiveBlock -----------------------------------------------------------------------------------
extern "C" int ctn_galr_supported(int F, int K, int Q, int heads) { return galr_ok(F, K, Q) && ctn_mha_supported(F, heads) ? 1 : 0; }

extern "C" size_t ctn_galr_inter_workspace_bytes(int B, int S, int K, int Q, int F) {
  if (B <= 0 || S <= 0 || K <= 0 || Q <= 0 || F <= 0) return 0;
  const size_t n = (size_t)Q * S * F;
  return 2 * up256((size_t)B * n * sizeof(float)) + up256(ctn_mha_workspace_bytes(B * Q, S, F)) +
         up256((size_t)B * ctn_sample_gln_parts(n) * 2 * sizeof(double)) + 256;
}

extern "C" int ctn_galr_inter_fwd(const float* x, const float* map_w, const float* map_b, const float* ln_g, const float* ln_b,
                                  const float* pe_div, int heads, const float* in_w, const float* in_b, const float* out_w, const float* out_b,
                                  const float* gn_g, const float* gn_b, const float* inv_w, const float* inv_b, float* out, int B, int S,
                                  int K, int Q, int F, float ln_eps, float gn_eps, void* workspace, size_t workspace_bytes,
                                  ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !map_w || !map_b || !ln_g || !ln_b || !pe_div || !in_w || !in_b || !out_w || !out_b || !gn_g || !gn_b || !inv_w || !inv_b ||
      !out || !workspace || B <= 0 || S <= 0 || K <= 0 || Q <= 0 || F <= 0 || heads <= 0)
    return CTN_EINVAL;
  if (!ctn_galr_supported(F, K, Q, heads)) return CTN_EUNSUPPORTED;
  // the grids of the down- and up-map and of the gLN statistics, and positions s Q + q exact in fp32
  if (B > 65535 || S > 65535 || (long long)S * Q > (1LL << 24)) return CTN_EUNSUPPORTED;
  if (((uintptr_t)workspace) & 255) return CTN_EALIGN;
  if (workspace_bytes < ctn_galr_inter_workspace_bytes(B, S, K, Q, F)) return CTN_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)Q * S * F;
  const int G = ctn_sample_gln_parts(n);
  Carver cv(workspace);
  float* zt = cv.take<float>((size_t)B * n);
  float* y = cv.take<float>((size_t)B * n);
  const size_t mha_bytes = ctn_mha_workspace_bytes(B * Q, S, F);
  void* mha_ws = cv.take<char>(mha_bytes);
  double* part = cv.take<double>((size_t)B * G * 2);
  k_galr_down<<<dim3(S, B), GT, 0, st>>>(x, map_w, map_b, ln_g, ln_b, pe_div, zt, S, K, Q, F, ln_eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  CTN_TRY(ctn_mha_fwd(zt, B * Q, S, F, heads, in_w, in_b, out_w, out_b, y, mha_ws, mha_bytes, stream));
  CTN_TRY(ctn_sample_gln_stats(y, zt, n, B, part, G, st));
  k_galr_up<<<dim3(S, B), GT, 0, st>>>(y, zt, part, G, gn_g, gn_b, inv_w, inv_b, x, out, S, K, Q, F, gn_eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- separator head: pad + Segment1d (channels-last) + gLN over the segmented tensor, no bottleneck -----------------------------
extern "C" size_t ctn_galr_head_workspace_bytes(int B, int S, int K, int F) {
  if (B <= 0 || S <= 0 || K <= 0 || F <= 0) return 0;
  return up256((size_t)B * ctn_sample_gln_parts((size_t)S * K * F) * 2 * sizeof(double)) + 256;
}

extern "C" int ctn_galr_head_fwd(const float* w, const float* norm_g, const float* norm_b, float* z, int B, int F, int frames, int pitch,
                                 int chunk_size, int hop_size, int pad_left, int pad_right, float eps, void* workspace,
                                 size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(w);
  if (!w || !norm_g || !norm_b || !z || !workspace || B <= 0 || F <= 0 || frames <= 0 || pitch < frames || chunk_size <= 0 ||
      hop_size <= 0 || pad_left < 0 || pad_right < 0)
    return CTN_EINVAL;
  const int Tp = frames + pad_left + pad_right;
  if (Tp < chunk_size) return CTN_EINVAL;
  if (B > 65535) return CTN_EUNSUPPORTED;
  if (((uintptr_t)workspace) & 255) return CTN_EALIGN;
  const int S = (Tp - chunk_size) / hop_size + 1;
  if (workspace_bytes < ctn_galr_head_workspace_bytes(B, S, chunk_size, F)) return CTN_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)S * chunk_size * F;
  const int G = ctn_sample_gln_parts(n);
  double* part = Carver(workspace).take<double>((size_t)B * G * 2);
  CTN_TRY(ctn_segment_fwd(w, z, B, F, frames, pitch, chunk_size, hop_size, pad_left, pad_right, 1, stream));
  CTN_TRY(ctn_sample_gln_stats(z, nullptr, n, B, part, G, st));
  return ctn_sample_gln_apply(z, n, B, F, part, G, norm_g, norm_b, eps, st);
}
