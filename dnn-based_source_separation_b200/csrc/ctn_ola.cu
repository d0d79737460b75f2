// Separation of recordings of any length with a model that only sees fixed-size chunks (ConvTasNet.separate_long):
// chunk gather, permutation alignment of neighbouring chunks, windowed overlap-add, and the call that strings them around
// ctn_convtasnet_fwd.  The reference has no counterpart (its separate scripts run the whole signal through the model).
//
// Chunk plan (chunk_plan below, the only place that knows it): Lc = min(chunk, T) samples per chunk; chunk k starts at k*hop,
// the last one at T - Lc, so no chunk reads past the signal.  chunk/2 <= hop <= chunk (integer division) bounds the chunks
// that cover one sample by four: three regular ones (two when 2*hop >= chunk) and the last.
#include <math.h>

#include "ctn_internal.h"

#define OLA_MAX_S 6       // alignment enumerates S! permutations, like the fused PIT loss
#define OLA_MAX_SPLIT 16  // CTAs that share one pair's overlap
#define OLA_TILE 1024     // pairs composed per shared-memory tile

struct ChunkPlan {
  int T, Lc, hop, K;
  __host__ __device__ int start(int k) const { return k == K - 1 ? T - Lc : k * hop; }
  // samples chunk k shares with chunk k + 1 (0 <= k < K - 1)
  __host__ __device__ int overlap(int k) const { const int o = start(k) + Lc - start(k + 1); return o > 0 ? o : 0; }
};

static int chunk_plan(int T, int chunk, int hop, ChunkPlan* p) {
  if (T <= 0 || chunk <= 0 || hop <= 0 || hop < chunk / 2 || hop > chunk) return CTN_EINVAL;
  p->T = T; p->hop = hop;
  p->Lc = T < chunk ? T : chunk;
  p->K = T <= chunk ? 1 : (int)(((long long)T - chunk + hop - 1) / hop) + 1;
  return CTN_OK;
}

extern "C" int ctn_chunk_plan(int T, int chunk, int hop, int* starts, int capacity) {
  ChunkPlan p;
  CTN_TRY(chunk_plan(T, chunk, hop, &p));
  if (starts) {
    if (capacity < p.K) return CTN_EINVAL;
    for (int k = 0; k < p.K; ++k) starts[k] = p.start(k);
  }
  return p.K;
}

// CTAs per pair of the scoring kernel: a function of the chunk size alone, so the scratch size does not depend on T
static int score_split(int Lc) {
  const int g = (Lc + 4095) / 4096;
  return g < 1 ? 1 : (g > OLA_MAX_SPLIT ? OLA_MAX_SPLIT : g);
}

// ---- gather: xc[j] = x[b][start(k) .. + Lc), chunk index first + j = b*K + k ----------------------------------------------
__global__ void __launch_bounds__(256) k_chunk_gather(const float* __restrict__ x, float* __restrict__ xc, ChunkPlan p, int first) {
  const int g = first + blockIdx.y, b = g / p.K, k = g - b * p.K;
  const float* src = x + (size_t)b * p.T + p.start(k);
  float* dst = xc + (size_t)blockIdx.y * p.Lc;
  const int t = (blockIdx.x * 256 + threadIdx.x) * 4;
  if (t >= p.Lc) return;
  if (t + 3 < p.Lc && ((((uintptr_t)(src + t)) | ((uintptr_t)(dst + t))) & 15) == 0) {
    st4(dst + t, ld4(src + t));
  } else {
    for (int i = t; i < t + 4 && i < p.Lc; ++i) dst[i] = src[i];
  }
}

// ---- alignment scores: partial[pair][g][i*S + j] = sum over CTA g's slice of the overlap of e_k[i] * e_{k+1}[j] ------------
// Every product and sum in double, summed in a fixed order (thread-strided slice, warp shuffles, warps in order): no atomics.
template <int S>
__global__ void __launch_bounds__(256) k_overlap_scores(const float* __restrict__ est, double* __restrict__ partial, ChunkPlan p) {
  __shared__ double red[8][S * S];
  const int pair = blockIdx.y, b = pair / (p.K - 1), k = pair - b * (p.K - 1);
  const int ov = p.overlap(k), G = gridDim.x;
  const int slice = (ov + G - 1) / G;
  const int q0 = blockIdx.x * slice, q1 = min(ov, q0 + slice);
  const float* ea = est + ((size_t)(b * p.K + k) * S) * p.Lc + (p.Lc - ov);
  const float* eb = ea + (size_t)S * p.Lc - (p.Lc - ov);
  double acc[S][S];
#pragma unroll
  for (int i = 0; i < S; ++i)
#pragma unroll
    for (int j = 0; j < S; ++j) acc[i][j] = 0.0;
  for (int q = q0 + threadIdx.x; q < q1; q += 256) {
    double vb[S];
#pragma unroll
    for (int j = 0; j < S; ++j) vb[j] = (double)eb[(size_t)j * p.Lc + q];
#pragma unroll
    for (int i = 0; i < S; ++i) {
      const double va = (double)ea[(size_t)i * p.Lc + q];
#pragma unroll
      for (int j = 0; j < S; ++j) acc[i][j] = fma(va, vb[j], acc[i][j]);
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < S; ++i)
#pragma unroll
    for (int j = 0; j < S; ++j) {
      const double v = warp_sum_d(acc[i][j]);
      if (lane == 0) red[wid][i * S + j] = v;
    }
  __syncthreads();
  if (threadIdx.x < S * S) {
    double v = 0.0;
    for (int w = 0; w < 8; ++w) v += red[w][threadIdx.x];
    partial[((size_t)pair * G + blockIdx.x) * (S * S) + threadIdx.x] = v;
  }
}

// ---- permutations: local argmax per pair, then the composition along each recording ----------------------------------------
// One CTA per recording.  Per tile of pairs: a thread per pair sums the pair's partial scores (in CTA order), walks the S!
// permutations in itertools order and keeps the first maximum of sum_i c[i][pi(i)]; then thread s < S follows source s through
// the tile: P_{k+1}(s) = pi_k(P_k(s)), P_0 = identity.  partial == nullptr: identity permutations.
__global__ void __launch_bounds__(256) k_compose_perms(const double* __restrict__ partial, int G, int S, int K, int32_t* __restrict__ perms) {
  __shared__ unsigned char local[OLA_TILE][OLA_MAX_S];
  const int b = blockIdx.x;
  int32_t* P = perms + (size_t)b * K * S;
  if (!partial) {
    for (int i = threadIdx.x; i < K * S; i += 256) P[i] = i % S;
    return;
  }
  int cur = threadIdx.x;  // P_k(s) of thread s
  if (threadIdx.x < S) P[threadIdx.x] = cur;
  for (int k0 = 0; k0 < K - 1; k0 += OLA_TILE) {
    const int n = min(OLA_TILE, K - 1 - k0);
    for (int r = threadIdx.x; r < n; r += 256) {
      const double* pp = partial + ((size_t)b * (K - 1) + k0 + r) * G * (S * S);
      double c[OLA_MAX_S * OLA_MAX_S];
      for (int e = 0; e < S * S; ++e) {
        double v = 0.0;
        for (int g = 0; g < G; ++g) v += pp[(size_t)g * (S * S) + e];
        c[e] = v;
      }
      int pi[OLA_MAX_S], best[OLA_MAX_S];
      for (int i = 0; i < S; ++i) pi[i] = best[i] = i;
      double best_v = 0.0;
      for (int i = 0; i < S; ++i) best_v += c[i * S + i];
      for (;;) {
        // next permutation in lexicographic order
        int i = S - 2;
        while (i >= 0 && pi[i] > pi[i + 1]) --i;
        if (i < 0) break;
        int j = S - 1;
        while (pi[j] < pi[i]) --j;
        int tmp = pi[i]; pi[i] = pi[j]; pi[j] = tmp;
        for (int lo = i + 1, hi = S - 1; lo < hi; ++lo, --hi) { tmp = pi[lo]; pi[lo] = pi[hi]; pi[hi] = tmp; }
        double v = 0.0;
        for (int s = 0; s < S; ++s) v += c[s * S + pi[s]];
        if (v > best_v) {
          best_v = v;
          for (int s = 0; s < S; ++s) best[s] = pi[s];
        }
      }
      for (int s = 0; s < S; ++s) local[r][s] = (unsigned char)best[s];
    }
    __syncthreads();
    if (threadIdx.x < S)
      for (int r = 0; r < n; ++r) {
        cur = local[r][cur];
        P[(size_t)(k0 + r + 1) * S + threadIdx.x] = cur;
      }
    __syncthreads();
  }
}

// ---- overlap-add, gather form: one thread per output time t, all S sources (they share the weights) ---------------------------
// w_k(t) = rise * fall: rise = sin^2(pi/2 (r + 1/2) / a) over the first a samples (a = overlap with chunk k - 1), fall =
// cos^2(pi/2 (q + 1/2) / n) over the last n (n = overlap with chunk k + 1), 1 elsewhere; the two ramps of one overlap sum to 1
// and the half-sample offset keeps them positive.  out = sum_k w_k e_k[P_k(s)] / sum_k w_k, k ascending, in double.
__device__ __forceinline__ double ola_weight(const ChunkPlan& p, int k, int r) {
  double w = 1.0;
  if (k > 0) {
    const int a = p.overlap(k - 1);
    if (r < a) { const double s = sinpi(0.5 * ((double)r + 0.5) / (double)a); w = s * s; }
  }
  if (k < p.K - 1) {
    const int n = p.overlap(k), q = r - (p.Lc - n);
    if (q >= 0) { const double c = cospi(0.5 * ((double)q + 0.5) / (double)n); w *= c * c; }
  }
  return w;
}

__global__ void __launch_bounds__(256) k_overlap_add(const float* __restrict__ est, const int32_t* __restrict__ perms, float* __restrict__ out,
                                                     ChunkPlan p, int S) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= p.T) return;
  // regular chunks 0 .. K-2 that cover t, then the last one
  int ks[4];
  double w[4], den = 0.0;
  int nc = 0;
  const int k_lo = t >= p.Lc ? (t - p.Lc) / p.hop + 1 : 0;
  const int k_hi = min(t / p.hop, p.K - 2);
  for (int k = k_lo; k <= k_hi; ++k) { ks[nc] = k; w[nc] = ola_weight(p, k, t - p.start(k)); den += w[nc]; ++nc; }
  if (t >= p.T - p.Lc) { ks[nc] = p.K - 1; w[nc] = ola_weight(p, p.K - 1, t - (p.T - p.Lc)); den += w[nc]; ++nc; }
  const double rden = 1.0 / den;
  for (int s = 0; s < S; ++s) {
    double num = 0.0;
    for (int c = 0; c < nc; ++c) {
      const size_t g = (size_t)b * p.K + ks[c];
      const int src = perms ? perms[g * S + s] : s;
      num = fma(w[c], (double)est[(g * S + src) * p.Lc + (t - p.start(ks[c]))], num);
    }
    out[((size_t)b * S + s) * p.T + t] = (float)(num * rden);
  }
}

// ---- launchers ---------------------------------------------------------------------------------------------------------------
static int launch_gather(const float* x, float* xc, const ChunkPlan& p, int first, int n, cudaStream_t st) {
  k_chunk_gather<<<dim3((p.Lc + 1023) / 1024, n), 256, 0, st>>>(x, xc, p, first);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

static size_t align_scratch_bytes(int B, int S, const ChunkPlan& p) {
  return sizeof(double) * (size_t)B * (p.K - 1) * score_split(p.Lc) * S * S;
}

static int launch_compose(const double* partial, int G, int B, int S, int K, int32_t* perms, cudaStream_t st) {
  k_compose_perms<<<B, 256, 0, st>>>(partial, G, S, K, perms);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// perms (B, K, S) from the chunk estimates; S == 1 or K == 1: identity, nothing to score
static int launch_align(const float* est, int B, int S, const ChunkPlan& p, int32_t* perms, double* partial, cudaStream_t st) {
  if (S == 1 || p.K == 1) return launch_compose(nullptr, 0, B, S, p.K, perms, st);
  const int G = score_split(p.Lc);
  const dim3 grid(G, B * (p.K - 1));
  switch (S) {
    case 2: k_overlap_scores<2><<<grid, 256, 0, st>>>(est, partial, p); break;
    case 3: k_overlap_scores<3><<<grid, 256, 0, st>>>(est, partial, p); break;
    case 4: k_overlap_scores<4><<<grid, 256, 0, st>>>(est, partial, p); break;
    case 5: k_overlap_scores<5><<<grid, 256, 0, st>>>(est, partial, p); break;
    default: k_overlap_scores<6><<<grid, 256, 0, st>>>(est, partial, p); break;
  }
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return launch_compose(partial, G, B, S, p.K, perms, st);
}

static int launch_ola(const float* est, const int32_t* perms, float* out, int B, int S, const ChunkPlan& p, cudaStream_t st) {
  k_overlap_add<<<dim3((p.T + 255) / 256, B), 256, 0, st>>>(est, perms, out, p, S);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// the grids put B (recordings), pairs and chunks of a batch on gridDim.y
static bool fits_grid_y(long long n) { return n > 0 && n <= 65535; }

// ---- the three steps on their own ---------------------------------------------------------------------------------------------
extern "C" int ctn_chunk_gather(const float* x, int B, int T, int chunk, int hop, int first, int n, float* xc, ctn_stream_t stream) {
  LaunchScope scope(x);
  ChunkPlan p;
  CTN_TRY(chunk_plan(T, chunk, hop, &p));
  if (!x || !xc || B <= 0 || first < 0 || n <= 0 || (long long)first + n > (long long)B * p.K) return CTN_EINVAL;
  if (!fits_grid_y(n)) return CTN_EUNSUPPORTED;
  return launch_gather(x, xc, p, first, n, (cudaStream_t)stream);
}

extern "C" size_t ctn_chunk_align_scratch_bytes(int B, int S, int T, int chunk, int hop) {
  ChunkPlan p;
  if (chunk_plan(T, chunk, hop, &p) != CTN_OK || B <= 0 || S <= 1 || S > OLA_MAX_S) return 0;
  return align_scratch_bytes(B, S, p);
}

extern "C" int ctn_chunk_align(const float* est, int B, int S, int T, int chunk, int hop, int32_t* perms, void* scratch,
                               size_t scratch_bytes, ctn_stream_t stream) {
  LaunchScope scope(est);
  ChunkPlan p;
  CTN_TRY(chunk_plan(T, chunk, hop, &p));
  if (!est || !perms || B <= 0 || S <= 0) return CTN_EINVAL;
  if (S > OLA_MAX_S) return CTN_EUNSUPPORTED;
  if (S > 1 && hop >= chunk) return CTN_EINVAL;  // neighbouring chunks must share samples
  if (S > 1 && p.K > 1) {
    if (!scratch) return CTN_EINVAL;
    if (((uintptr_t)scratch) & 7) return CTN_EALIGN;
    if (scratch_bytes < align_scratch_bytes(B, S, p)) return CTN_EWORKSPACE;
    if (!fits_grid_y((long long)B * (p.K - 1))) return CTN_EUNSUPPORTED;
  }
  if (!fits_grid_y(B)) return CTN_EUNSUPPORTED;
  return launch_align(est, B, S, p, perms, (double*)scratch, (cudaStream_t)stream);
}

extern "C" int ctn_chunk_overlap_add(const float* est, const int32_t* perms, int B, int S, int T, int chunk, int hop, float* out,
                                     ctn_stream_t stream) {
  LaunchScope scope(est);
  ChunkPlan p;
  CTN_TRY(chunk_plan(T, chunk, hop, &p));
  if (!est || !out || B <= 0 || S <= 0) return CTN_EINVAL;
  if (!fits_grid_y(B)) return CTN_EUNSUPPORTED;
  return launch_ola(est, perms, out, B, S, p, (cudaStream_t)stream);
}

// ---- the whole call -------------------------------------------------------------------------------------------------------------
struct LongWs {
  int32_t* perms;   // (B, K, S)
  double* partial;  // alignment scores, (B (K-1), split, S, S)
  float* xc;        // (nb, 1, Lc) one gathered chunk batch
  float* est;       // (B K, S, Lc) chunk estimates
  void* model;      // workspace of ctn_convtasnet_fwd for one chunk batch
  size_t model_bytes;
  int nb;           // chunks per batch
};

static int carve_long(Carver& cv, const ctn_config_t* c, int B, const ChunkPlan& p, int chunk_batch, LongWs* ws) {
  const int S = c->n_sources;
  const long long chunks = (long long)B * p.K;
  ws->nb = (int)(chunks < chunk_batch ? chunks : chunk_batch);
  if (ws->nb > 65535) ws->nb = 65535;  // a batch's chunks ride on gridDim.y
  CTN_TRY(ctn_workspace_bytes(c, ws->nb, p.Lc, &ws->model_bytes));
  ws->perms = cv.take<int32_t>((size_t)chunks * S);
  ws->partial = nullptr; ws->xc = nullptr; ws->est = nullptr;
  if (p.K > 1) {
    if (S > 1 && S <= OLA_MAX_S) ws->partial = cv.take<double>(align_scratch_bytes(B, S, p) / sizeof(double));
    ws->xc = cv.take<float>((size_t)ws->nb * p.Lc);
    ws->est = cv.take<float>((size_t)chunks * S * p.Lc);
  }
  ws->model = cv.take<char>(ws->model_bytes);
  return CTN_OK;
}

static int check_long(const ctn_config_t* c, int B, int T, int chunk, int hop, int chunk_batch, ChunkPlan* p) {
  CTN_TRY(check_model_cfg(c));
  if (B <= 0 || chunk_batch <= 0) return CTN_EINVAL;
  CTN_TRY(chunk_plan(T, chunk, hop, p));
  if (c->in_channels > 1) return CTN_EUNSUPPORTED;
  if (!fits_grid_y(B) || (long long)B * p->K > INT32_MAX) return CTN_EUNSUPPORTED;
  return CTN_OK;
}

extern "C" int ctn_separate_long_workspace_bytes(const ctn_config_t* cfg, int B, int T, int chunk, int hop, int chunk_batch, size_t* bytes) {
  ChunkPlan p;
  CTN_TRY(check_long(cfg, B, T, chunk, hop, chunk_batch, &p));
  if (!bytes) return CTN_EINVAL;
  Carver cv(nullptr);
  LongWs ws;
  CTN_TRY(carve_long(cv, cfg, B, p, chunk_batch, &ws));
  *bytes = cv.off + 256;
  return CTN_OK;
}

extern "C" int ctn_convtasnet_separate_long(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, int chunk,
                                            int hop, int chunk_batch, int align, float* out, int32_t* perms_out, void* workspace,
                                            size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(x);
  ChunkPlan p;
  CTN_TRY(check_long(cfg, B, T, chunk, hop, chunk_batch, &p));
  if (!params || !params->blocks || !x || !out || !workspace) return CTN_EINVAL;
  const int S = cfg->n_sources;
  const bool scored = align && S > 1;
  if (scored && S > OLA_MAX_S) return CTN_EUNSUPPORTED;
  if (scored && hop >= chunk) return CTN_EINVAL;  // neighbouring chunks must share samples
  if (((uintptr_t)workspace) & 255) return CTN_EALIGN;
  size_t need = 0;
  CTN_TRY(ctn_separate_long_workspace_bytes(cfg, B, T, chunk, hop, chunk_batch, &need));
  if (workspace_bytes < need) return CTN_EWORKSPACE;
  if (scored && p.K > 1 && !fits_grid_y((long long)B * (p.K - 1))) return CTN_EUNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  Carver cv(workspace);
  LongWs ws;
  CTN_TRY(carve_long(cv, cfg, B, p, chunk_batch, &ws));
  if (p.K == 1) {
    // the recordings are the chunks: the plain forward on the caller's buffers, batch by batch
    for (int g0 = 0; g0 < B; g0 += ws.nb) {
      const int n = B - g0 < ws.nb ? B - g0 : ws.nb;
      CTN_TRY(ctn_convtasnet_fwd(cfg, params, x + (size_t)g0 * T, n, T, out + (size_t)g0 * S * T, nullptr, ws.model, ws.model_bytes, stream));
    }
    return perms_out ? launch_compose(nullptr, 0, B, S, 1, perms_out, st) : CTN_OK;
  }
  const int chunks = B * p.K;
  for (int g0 = 0; g0 < chunks; g0 += ws.nb) {
    const int n = chunks - g0 < ws.nb ? chunks - g0 : ws.nb;
    CTN_TRY(launch_gather(x, ws.xc, p, g0, n, st));
    CTN_TRY(ctn_convtasnet_fwd(cfg, params, ws.xc, n, p.Lc, ws.est + (size_t)g0 * S * p.Lc, nullptr, ws.model, ws.model_bytes, stream));
  }
  int32_t* perms = nullptr;
  if (scored) {
    perms = perms_out ? perms_out : ws.perms;
    CTN_TRY(launch_align(ws.est, B, S, p, perms, ws.partial, st));
  } else if (perms_out) {
    CTN_TRY(launch_compose(nullptr, 0, B, S, p.K, perms_out, st));
  }
  return launch_ola(ws.est, perms, out, B, S, p, st);
}
