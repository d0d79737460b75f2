// DPTNet (dual-path transformer) stages.  Reference: src/models/dptnet.py:319-348 (Separator), :482-525 (MultiheadAttentionBlock),
// :527-572 (FeedForwardBlock), src/models/gtu.py:10-44 (GTU1d).
//
// The dual-path state is channels-last, Z (B, D1, D2, F), as on the DPRNN-TasNet path: a "sequence" of the current path is one
// (b, d1) row of D2 tokens of F features (intra: D1 = S chunks, D2 = K frames; inter: D1 = K, D2 = S).
//   * multi-head self-attention (nn.MultiheadAttention, no mask): the QKV projection, the attention and the output projection are
//     three launches; the attention streams keys in tiles of 64 with an online softmax (running max and sum in fp32), so any
//     sequence length runs in fixed shared memory.  All products are fp32 FMAs.
//   * the norm of both sub-blocks is GroupNorm(1, F) over each SEQUENCE (dptnet.py:519-521 / 566-568), applied to x + residual:
//     one CTA per (b, d1) row sums the row in double in a fixed order (no atomics: repeated calls give the same bits), then
//     normalises it, storing the intra <-> inter swap on the way out.
//   * the head's gLN (dptnet.py:337) is per SAMPLE over the segmented tensor, duplicated overlap frames and padding zeros included.
//   * the head (bottleneck 1x1, optional: GALRNet has none) and the tail are shared by DPTNet, GALRNet and SepFormer.  The tail is
//     PReLU -> map 1x1 -> GTU1d (map and map_gate in one 1x1 of 2N rows) [-> bottleneck_conv1d_out, SepFormer] -> mask
//     nonlinearity -> w * mask -> decoder; all weight images of a call are built in one batch.
#include <math.h>

#include "ctn_internal.h"

namespace {

constexpr int PROJ_ROWS = 32;    // token rows per CTA of the row projection
constexpr int PROJ_MAX_K = 128;  // input features the row projection stages in shared memory
constexpr int ATT_Q = 64;        // queries per attention CTA (one per thread)
constexpr int ATT_KT = 64;       // keys per shared-memory tile
constexpr int ATT_SUB = 16;      // keys per online-softmax update

// Y[r][m] = bias[m] + sum_k X[r][k] W[m][k]  (nn.Linear on channels-last rows), k ascending.  grid ceil(R / 32), block 128
__global__ void __launch_bounds__(128) k_rowproj(const float* __restrict__ X, const float* __restrict__ W, const float* __restrict__ bias,
                                                 float* __restrict__ Y, long long R, int K, int M) {
  __shared__ float xs[PROJ_ROWS][PROJ_MAX_K + 1];
  const long long r0 = (long long)blockIdx.x * PROJ_ROWS;
  for (int i = threadIdx.x; i < PROJ_ROWS * K; i += blockDim.x) {
    const int r = i / K, k = i % K;
    xs[r][k] = r0 + r < R ? X[(r0 + r) * K + k] : 0.f;
  }
  __syncthreads();
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    float acc[PROJ_ROWS];
    const float b = __ldg(bias + m);
#pragma unroll
    for (int r = 0; r < PROJ_ROWS; ++r) acc[r] = b;
    for (int k = 0; k < K; ++k) {
      const float w = __ldg(W + (size_t)m * K + k);
#pragma unroll
      for (int r = 0; r < PROJ_ROWS; ++r) acc[r] = fmaf(xs[r][k], w, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < PROJ_ROWS; ++r)
      if (r0 + r < R) Y[(r0 + r) * M + m] = acc[r];
  }
}

// O[seq][t][h D + c] = sum_j softmax_j(q_t . k_j / sqrt(D)) v_j[c] for head h, qkv (NSEQ, T, 3F) = [q | k | v] per token.
// grid (NSEQ, ceil(T / 64), heads), block 64: one query per thread, q and the running output in registers; keys and values of
// a 64-key tile in shared memory (every thread reads the same key: broadcast).  The sequences are on x, whose limit is 2^31 - 1,
// so a batch of any size runs (DPTNet's inter path has B * chunk_size sequences).  Per 16 keys the running max m and sum l are
// updated: the old terms are rescaled by exp(m_old - m_new), exactly as in a one-pass softmax.
template <int D>
__global__ void __launch_bounds__(ATT_Q) k_attn(const float* __restrict__ qkv, float* __restrict__ O, int T, int F, float scale) {
  __shared__ float ks[ATT_KT][D], vs[ATT_KT][D];
  const int seq = blockIdx.x, hd = blockIdx.z, t = blockIdx.y * ATT_Q + threadIdx.x;
  const size_t base = (size_t)seq * T;
  const int F3 = 3 * F;
  float q[D], acc[D];
#pragma unroll
  for (int c = 0; c < D; ++c) {
    q[c] = t < T ? __ldg(qkv + (base + t) * F3 + hd * D + c) * scale : 0.f;
    acc[c] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < T; k0 += ATT_KT) {
    const int nk = T - k0 < ATT_KT ? T - k0 : ATT_KT;
    __syncthreads();  // the previous tile is consumed
    for (int i = threadIdx.x; i < nk * D; i += ATT_Q) {
      const int j = i / D, c = i % D;
      const float* row = qkv + (base + k0 + j) * F3 + hd * D + c;
      ks[j][c] = __ldg(row + F);
      vs[j][c] = __ldg(row + 2 * F);
    }
    __syncthreads();
    for (int j0 = 0; j0 < nk; j0 += ATT_SUB) {
      float s[ATT_SUB];
      float mt = m;
#pragma unroll
      for (int jj = 0; jj < ATT_SUB; ++jj) {
        const int j = j0 + jj;
        float dot = -INFINITY;
        if (j < nk) {
          dot = 0.f;
#pragma unroll
          for (int c = 0; c < D; ++c) dot = fmaf(q[c], ks[j][c], dot);
        }
        s[jj] = dot;
        mt = fmaxf(mt, dot);
      }
      const float corr = expf(m - mt);  // m = -inf before the first key: corr = 0 rescales the empty sums
      l *= corr;
#pragma unroll
      for (int c = 0; c < D; ++c) acc[c] *= corr;
#pragma unroll
      for (int jj = 0; jj < ATT_SUB; ++jj) {
        const int j = j0 + jj;
        if (j < nk) {
          const float p = expf(s[jj] - mt);
          l += p;
#pragma unroll
          for (int c = 0; c < D; ++c) acc[c] = fmaf(p, vs[j][c], acc[c]);
        }
      }
      m = mt;
    }
  }
  if (t < T) {
    const float inv = 1.f / l;
#pragma unroll
    for (int c = 0; c < D; ++c) O[(base + t) * F + hd * D + c] = acc[c] * inv;
  }
}

// x = Y0 + Y1 + bias + R (the last three nullable), out = GroupNorm(1, F) of each (b, d1) row of D2 x F values (gamma, beta per
// feature), stored as (B, D2, D1, F) when swap.  grid (D1, B), block 256.  Each thread sums its elements in double in index
// order; the block reduction is a fixed shuffle tree: the statistics do not depend on scheduling.
__device__ __forceinline__ float seq_val(const float* __restrict__ Y0, const float* __restrict__ Y1, const float* __restrict__ bias,
                                         const float* __restrict__ R, size_t i, int f) {
  float x = Y0[i];
  if (Y1) x += Y1[i];
  if (bias) x += __ldg(bias + f);
  if (R) x += R[i];
  return x;
}
__global__ void __launch_bounds__(256) k_seq_norm(const float* Y0, const float* Y1, const float* __restrict__ bias, const float* R,
                                                  const float* __restrict__ gamma, const float* __restrict__ beta, float* out, int D1,
                                                  int D2, int F, float eps, int swap) {
  __shared__ double red[64];
  __shared__ double st[2];
  const int b = blockIdx.y, d1 = blockIdx.x;
  const size_t row = ((size_t)b * D1 + d1) * D2 * F, n = (size_t)D2 * F;
  double s = 0.0, ss = 0.0;
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double x = seq_val(Y0, Y1, bias, R, row + i, (int)(i % F));
    s += x;
    ss = fma(x, x, ss);
  }
  block_sum2_d(s, ss, red);
  if (threadIdx.x == 0) { st[0] = s; st[1] = ss; }
  __syncthreads();
  const float2 mr = gln_mean_rstd(st, (double)n, eps);
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int f = (int)(i % F), d2 = (int)(i / F);
    const float x = seq_val(Y0, Y1, bias, R, row + i, f);
    const size_t dst = swap ? (((size_t)b * D2 + d2) * D1 + d1) * F + f : row + i;
    out[dst] = fmaf((x - mr.x) * mr.y, __ldg(gamma + f), __ldg(beta + f));
  }
}

// gLN per sample over n values of x = z + z2 (B, n), z2 nullable: partial (sum, sumsq) of G slices -> part[b][g][2] ...
__global__ void __launch_bounds__(256) k_sample_part(const float* __restrict__ z, const float* __restrict__ z2, size_t n,
                                                     double* __restrict__ part) {
  __shared__ double red[64];
  const int b = blockIdx.y, G = gridDim.x;
  const size_t lo = n * blockIdx.x / G, hi = n * (blockIdx.x + 1) / G;
  double s = 0.0, ss = 0.0;
  for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    float v = z[(size_t)b * n + i];
    if (z2) v += z2[(size_t)b * n + i];
    const double x = v;
    s += x;
    ss = fma(x, x, ss);
  }
  block_sum2_d(s, ss, red);
  if (threadIdx.x == 0) { part[((size_t)b * G + blockIdx.x) * 2] = s; part[((size_t)b * G + blockIdx.x) * 2 + 1] = ss; }
}
// ... and z = (z - mean) rstd gamma[f] + beta[f] in place, f = i % F, the G partials summed in slice order by every CTA
__global__ void __launch_bounds__(256) k_sample_apply(float* __restrict__ z, size_t n, int F, const double* __restrict__ part, int G,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta, float eps) {
  __shared__ double st[2];
  const int b = blockIdx.y;
  const float2 mr = sample_gln_mean_rstd(part, G, b, (double)n, eps, st);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int f = (int)(i % F);
    float* p = z + (size_t)b * n + i;
    *p = fmaf((*p - mr.x) * mr.y, __ldg(gamma + f), __ldg(beta + f));
  }
}

// GTU1d and the mask, one or both per launch, on the (R = B S, ., pitch) layout, columns [frames, pitch) = 0:
//   GTU:  v = tanh(g[n]) sigmoid(g[N + n]) from g (R, 2N, pitch) = [map; map_gate] (x) + bias;  otherwise v = x (R, N, pitch);
//   MASK: out[r][n][t] = act(v) w[r / S][n][t], act = ReLU (mask_relu) or sigmoid;  otherwise out = v.
// grid (<= 256, R), block 256.
template <bool GTU, bool MASK>
__global__ void __launch_bounds__(256) k_gtu_mask(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ out, int S,
                                                  int N, int frames, int pitch, int mask_relu) {
  const int r = blockIdx.y, b = r / S;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)N * pitch; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / pitch), t = (int)(i % pitch);
    float v = 0.f;
    if (t < frames) {
      if (GTU) {
        const float a = x[((size_t)r * 2 * N + n) * pitch + t], gt = x[((size_t)r * 2 * N + N + n) * pitch + t];
        v = tanhf(a) * (1.f / (1.f + expf(-gt)));
      } else {
        v = x[(size_t)r * N * pitch + i];
      }
      if (MASK) {
        const float mk = mask_relu ? fmaxf(v, 0.f) : 1.f / (1.f + expf(-v));
        v = mk * w[((size_t)b * N + n) * pitch + t];
      }
    }
    out[(size_t)r * N * pitch + i] = v;
  }
}
template <bool GTU, bool MASK>
int launch_gtu_mask(const float* x, const float* w, float* out, int R, int S, int N, int frames, int pitch, int mask_relu, cudaStream_t st) {
  int gx = (int)(((size_t)N * pitch + 255) / 256);
  if (gx > 256) gx = 256;
  k_gtu_mask<GTU, MASK><<<dim3(gx, R), 256, 0, st>>>(x, w, out, S, N, frames, pitch, mask_relu);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

bool mha_ok(int F, int heads) {
  if (F <= 0 || heads <= 0 || F % heads || F > PROJ_MAX_K || (F & 3)) return false;
  const int D = F / heads;
  return D == 8 || D == 16 || D == 32 || D == 64;
}

struct MhaWs { float *qkv, *o; };
void carve_mha(Carver& cv, int NSEQ, int T, int F, MhaWs* ws) {
  const size_t tok = (size_t)NSEQ * T;
  ws->qkv = cv.take<float>(tok * 3 * F);
  ws->o = cv.take<float>(tok * F);
}

// the head's workspace: the bottleneck's output, its weight image (tf32x3-sized: any mode fits) and statistics, the gLN partials
struct HeadWs {
  float *x0, *wimg;
  double *stats, *part;
};
void carve_head(Carver& cv, int B, int N, int Bc, int pitch, int S, int K, HeadWs* ws) {
  ws->x0 = cv.take<float>((size_t)B * Bc * pitch);
  ws->wimg = cv.take<float>(ctn_pw_wimg_bytes(Bc, N, CTN_MATH_TF32X3) / sizeof(float));
  ws->stats = cv.take<double>(2 * (size_t)B);
  ws->part = cv.take<double>((size_t)B * ctn_sample_gln_parts((size_t)S * K * Bc) * 2);
}

// the tail's workspace; u and img_out only with bottleneck_conv1d_out
struct TailWs {
  float *yp, *m, *u, *g, *wcat, *bcat, *img_map, *img_gtu, *img_out;
  double* stats;
};
void carve_tail(Carver& cv, int B, int N, int Bc, int S, int pitch, bool bout, TailWs* ws) {
  const size_t R = (size_t)B * S;
  ws->yp = cv.take<float>((size_t)B * Bc * pitch);
  ws->m = cv.take<float>(R * N * pitch);
  ws->u = bout ? cv.take<float>(R * N * pitch) : nullptr;
  ws->g = cv.take<float>(R * 2 * N * pitch);
  ws->wcat = cv.take<float>((size_t)2 * N * N);
  ws->bcat = cv.take<float>((size_t)2 * N);
  ws->img_map = cv.take<float>(ctn_pw_wimg_bytes(S * N, Bc, CTN_MATH_TF32X3) / sizeof(float));
  ws->img_gtu = cv.take<float>(ctn_pw_wimg_bytes(2 * N, N, CTN_MATH_TF32X3) / sizeof(float));
  ws->img_out = bout ? cv.take<float>(ctn_pw_wimg_bytes(N, N, CTN_MATH_TF32X3) / sizeof(float)) : nullptr;
  ws->stats = cv.take<double>(2 * R);
}

bool math_ok(int math) {
  return math == CTN_MATH_FP32 || math == CTN_MATH_TF32 || math == CTN_MATH_TF32X3 || math == CTN_MATH_F16X3;
}

}  // namespace

// ---- per-sample gLN over a contiguous tensor (ctn_internal.h) -------------------------------------------------------------------
int ctn_sample_gln_parts(size_t n) {
  size_t g = (n + 256 * 16 - 1) / (256 * 16);
  return g < 1 ? 1 : (g > 128 ? 128 : (int)g);
}

int ctn_sample_gln_stats(const float* z, const float* z2, size_t n, int B, double* part, int G, cudaStream_t st) {
  k_sample_part<<<dim3(G, B), 256, 0, st>>>(z, z2, n, part);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int ctn_sample_gln_apply(float* z, size_t n, int B, int F, const double* part, int G, const float* gamma, const float* beta, float eps,
                         cudaStream_t st) {
  int ga = (int)((n + 255) / 256);
  if (ga > 512) ga = 512;
  k_sample_apply<<<dim3(ga, B), 256, 0, st>>>(z, n, F, part, G, gamma, beta, eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- multi-head self-attention --------------------------------------------------------------------------------------------------
extern "C" int ctn_mha_supported(int F, int heads) { return mha_ok(F, heads) ? 1 : 0; }

extern "C" size_t ctn_mha_workspace_bytes(int NSEQ, int T, int F) {
  if (NSEQ <= 0 || T <= 0 || F <= 0) return 0;
  Carver cv(nullptr);
  MhaWs ws;
  carve_mha(cv, NSEQ, T, F, &ws);
  return cv.off + 256;
}

extern "C" int ctn_mha_fwd(const float* z, int NSEQ, int T, int F, int heads, const float* in_w, const float* in_b, const float* out_w,
                           const float* out_b, float* y, void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(z);
  if (!z || !in_w || !in_b || !out_w || !out_b || !y || !workspace || NSEQ <= 0 || T <= 0 || F <= 0 || heads <= 0) return CTN_EINVAL;
  if (!mha_ok(F, heads) || (T + ATT_Q - 1) / ATT_Q > 65535) return CTN_EUNSUPPORTED;
  if (((uintptr_t)workspace) & 255) return CTN_EALIGN;
  if (workspace_bytes < ctn_mha_workspace_bytes(NSEQ, T, F)) return CTN_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const long long tok = (long long)NSEQ * T;
  Carver cv(workspace);
  MhaWs ws;
  carve_mha(cv, NSEQ, T, F, &ws);
  float *qkv = ws.qkv, *o = ws.o;
  const unsigned gproj = (unsigned)((tok + PROJ_ROWS - 1) / PROJ_ROWS);
  k_rowproj<<<gproj, 128, 0, st>>>(z, in_w, in_b, qkv, tok, F, 3 * F);
  CTN_COUNT_LAUNCH();
  const int D = F / heads;
  const float scale = (float)(1.0 / sqrt((double)D));
  const dim3 ga(NSEQ, (T + ATT_Q - 1) / ATT_Q, heads);
  if (D == 8) k_attn<8><<<ga, ATT_Q, 0, st>>>(qkv, o, T, F, scale);
  if (D == 16) k_attn<16><<<ga, ATT_Q, 0, st>>>(qkv, o, T, F, scale);
  if (D == 32) k_attn<32><<<ga, ATT_Q, 0, st>>>(qkv, o, T, F, scale);
  if (D == 64) k_attn<64><<<ga, ATT_Q, 0, st>>>(qkv, o, T, F, scale);
  CTN_COUNT_LAUNCH();
  k_rowproj<<<gproj, 128, 0, st>>>(o, out_w, out_b, y, tok, F, F);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- per-sequence gLN of x + residual, with the path swap ----------------------------------------------------------------------
extern "C" int ctn_seq_norm_fwd(const float* Y0, const float* Y1, const float* bias, const float* R, const float* gamma, const float* beta,
                                float* out, int B, int D1, int D2, int F, float eps, int swap, ctn_stream_t stream) {
  LaunchScope scope(Y0);
  if (!Y0 || !gamma || !beta || !out || B <= 0 || D1 <= 0 || D2 <= 0 || F <= 0) return CTN_EINVAL;
  if (B > 65535) return CTN_EUNSUPPORTED;
  if (swap && (out == Y0 || out == Y1 || out == R)) return CTN_EINVAL;  // the swap cannot run in place
  k_seq_norm<<<dim3(D1, B), 256, 0, (cudaStream_t)stream>>>(Y0, Y1, bias, R, gamma, beta, out, D1, D2, F, eps, swap);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- separator head: [bottleneck 1x1 ->] pad + segment (channels-last) -> gLN over the segmented tensor --------------------------
extern "C" size_t ctn_dpt_head_workspace_bytes(int B, int N, int Bc, int pitch, int S, int K) {
  if (B <= 0 || N <= 0 || Bc <= 0 || pitch <= 0 || S <= 0 || K <= 0) return 0;
  Carver cv(nullptr);
  HeadWs ws;
  carve_head(cv, B, N, Bc, pitch, S, K, &ws);
  return cv.off + 256;
}

extern "C" int ctn_dpt_head_fwd(const float* w, const float* bn_w, const float* bn_b, const float* norm_g, const float* norm_b, float* z,
                                int B, int N, int Bc, int frames, int pitch, int chunk_size, int hop_size, int pad_left, int pad_right,
                                float eps, int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(w);
  if (!w || !norm_g || !norm_b || !z || !workspace || B <= 0 || N <= 0 || Bc <= 0 || frames <= 0 || chunk_size <= 0 || hop_size <= 0 ||
      pad_left < 0 || pad_right < 0)
    return CTN_EINVAL;
  if (!bn_w != !bn_b || (!bn_w && Bc != N) || !math_ok(math)) return CTN_EINVAL;
  if (pitch < frames || pitch % CTN_TILE_T != 0 || (((uintptr_t)workspace) & 255) || (((uintptr_t)w) & 15)) return CTN_EALIGN;
  const int Tp = frames + pad_left + pad_right;
  if (Tp < chunk_size) return CTN_EINVAL;
  if (B > 65535) return CTN_EUNSUPPORTED;  // the grids of the segmentation and the gLN
  const int S = (Tp - chunk_size) / hop_size + 1;
  if (workspace_bytes < ctn_dpt_head_workspace_bytes(B, N, Bc, pitch, S, chunk_size)) return CTN_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)S * chunk_size * Bc;
  const int G = ctn_sample_gln_parts(n);
  Carver cv(workspace);
  HeadWs ws;
  carve_head(cv, B, N, Bc, pitch, S, chunk_size, &ws);
  const float* x = w;
  if (bn_w) {
    const float* one = ctn_device_one();
    if (!one) return CTN_ENOTBUILT;
    cudaError_t e = cudaMemsetAsync(ws.stats, 0, sizeof(double) * 2 * B, st);
    if (e != cudaSuccess) return (int)e;
    const WimgJob job{bn_w, ws.wimg, Bc, N};
    CTN_TRY(ctn_pw_prepare_batch(&job, 1, math, false, st));
    CTN_TRY(ctn_pw_run(w, bn_w, ws.wimg, ws.x0, B, Bc, N, frames, pitch, math, bn_b, one, ws.stats, st));
    x = ws.x0;
  }
  CTN_TRY(ctn_segment_fwd(x, z, B, Bc, frames, pitch, chunk_size, hop_size, pad_left, pad_right, 1, stream));
  CTN_TRY(ctn_sample_gln_stats(z, nullptr, n, B, ws.part, G, st));
  return ctn_sample_gln_apply(z, n, B, Bc, ws.part, G, norm_g, norm_b, eps, st);
}

// ---- separator tail + decoder: PReLU -> map -> GTU1d [-> bottleneck_conv1d_out] -> mask nonlinearity -> w * mask -> decoder ------
extern "C" size_t ctn_dpt_tail_workspace_bytes(int B, int N, int Bc, int S, int pitch, int bout) {
  if (B <= 0 || N <= 0 || Bc <= 0 || S <= 0 || pitch <= 0) return 0;
  Carver cv(nullptr);
  TailWs ws;
  carve_tail(cv, B, N, Bc, S, pitch, bout != 0, &ws);
  return cv.off + 256;
}

extern "C" int ctn_dpt_tail_fwd(const float* y, const float* w, const float* prelu, const float* map_w, const float* map_b,
                                const float* gtu_w, const float* gtu_b, const float* gate_w, const float* gate_b, const float* bout_w,
                                const float* bout_b, const float* dec_w, float* out, float* latent, float* what, int B, int N, int Bc,
                                int S, int frames, int pitch, int L, int stride, int crop_left, int T, int mask_relu, int math,
                                void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(y);
  if (!y || !w || !prelu || !map_w || !map_b || !gtu_w || !gtu_b || !gate_w || !gate_b || !dec_w || !out || !what || !workspace || B <= 0 ||
      N <= 0 || Bc <= 0 || S <= 0 || frames <= 0)
    return CTN_EINVAL;
  if (!bout_w != !bout_b || !math_ok(math)) return CTN_EINVAL;
  const bool bout = bout_w != nullptr;
  if (pitch < frames || pitch % CTN_TILE_T != 0 || (((uintptr_t)workspace) & 255)) return CTN_EALIGN;
  if ((((uintptr_t)y) | ((uintptr_t)w) | ((uintptr_t)what)) & 15) return CTN_EALIGN;
  if (workspace_bytes < ctn_dpt_tail_workspace_bytes(B, N, Bc, S, pitch, bout)) return CTN_EWORKSPACE;
  if ((long long)B * S > 65535) return CTN_EUNSUPPORTED;
  CTN_TRY(ctn_decoder_check(B * S, N, frames, pitch, L, stride, crop_left, T));
  const float* one = ctn_device_one();
  if (!one) return CTN_ENOTBUILT;
  cudaStream_t st = (cudaStream_t)stream;
  const int R = B * S;
  Carver cv(workspace);
  TailWs ws;
  carve_tail(cv, B, N, Bc, S, pitch, bout, &ws);
  const bool tc = math != CTN_MATH_FP32;
  cudaError_t e;
  // [map; map_gate] as one 2N x N contraction
  if ((e = cudaMemcpyAsync(ws.wcat, gtu_w, sizeof(float) * N * N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpyAsync(ws.wcat + (size_t)N * N, gate_w, sizeof(float) * N * N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpyAsync(ws.bcat, gtu_b, sizeof(float) * N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpyAsync(ws.bcat + N, gate_b, sizeof(float) * N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(ws.stats, 0, sizeof(double) * 2 * R, st)) != cudaSuccess) return (int)e;
  if (tc) {  // every weight image of the call in one batch
    const WimgJob jobs[3] = {{map_w, ws.img_map, S * N, Bc}, {ws.wcat, ws.img_gtu, 2 * N, N}, {bout_w, ws.img_out, N, N}};
    CTN_TRY(ctn_pw_prepare_batch(jobs, bout ? 3 : 2, math, false, st));
  }
  CTN_TRY(ctn_prelu_apply(y, ws.yp, prelu, B, Bc, frames, pitch, st));
  CTN_TRY(ctn_pw_run(ws.yp, map_w, ws.img_map, ws.m, B, S * N, Bc, frames, pitch, math, map_b, one, ws.stats, st));
  CTN_TRY(ctn_pw_run(ws.m, ws.wcat, ws.img_gtu, ws.g, R, 2 * N, N, frames, pitch, math, ws.bcat, one, ws.stats, st));
  if (bout) {
    CTN_TRY((launch_gtu_mask<true, false>(ws.g, nullptr, ws.u, R, S, N, frames, pitch, mask_relu, st)));
    CTN_TRY(ctn_pw_run(ws.u, bout_w, ws.img_out, ws.m, R, N, N, frames, pitch, math, bout_b, one, ws.stats, st));
    CTN_TRY((launch_gtu_mask<false, true>(ws.m, w, what, R, S, N, frames, pitch, mask_relu, st)));
  } else {
    CTN_TRY((launch_gtu_mask<true, true>(ws.g, w, what, R, S, N, frames, pitch, mask_relu, st)));
  }
  CTN_TRY(ctn_decoder_fwd(what, dec_w, out, R, N, frames, pitch, L, stride, crop_left, T, stream));
  if (latent) CTN_TRY(ctn_copy_from_pitch(what, latent, R * N, frames, pitch, st));
  return CTN_OK;
}
