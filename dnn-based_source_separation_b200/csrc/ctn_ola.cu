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
  // a batch's chunks ride on gridDim.y, and the forward's decoder puts their nb * S source rows there
  if ((long long)ws->nb * S > 65535) ws->nb = 65535 / S;
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

// =================================================================================================================================
// Whole tracks of a MUSDB18-style model (ConvTasNet.separate_track): every segment and channel standardised on its own before the
// forward, the estimates mapped back with the same statistics, then overlap-added.  The recipe's tester (egs/musdb18/conv-tasnet,
// adhoc_dataset.py / adhoc_driver.py) does this in Python around one forward per segment.
//
// Two layouts of the same ChunkPlan:
//  * tester (hop = 0): Lc = segment, K = ceil(T / segment), segment k starts at k * segment and samples at or past T read as zero
//    (the tester's zero padding, counted in the statistics).  The plan's T is the padded extent K * segment, so ChunkPlan::start
//    and ola_weight see K chunks that share no samples: every weight is 1 and the overlap-add is the tester's concatenate-and-crop.
//  * cross-faded (segment/2 <= hop <= segment): chunk_plan as it is; no chunk reads past T.
// TrackPlan::T is the signal's own length in both.
#define TRACK_SLICE 8192     // samples of one (segment, channel) per statistics CTA
#define TRACK_MAX_SPLIT 64

struct TrackPlan {
  ChunkPlan p;
  int T;
  // samples of chunk k that lie inside the signal (the rest are zeros)
  __host__ __device__ int valid(int k) const { const int v = T - p.start(k); return v < p.Lc ? v : p.Lc; }
};

static int track_plan(int T, int segment, int hop, TrackPlan* tp) {
  if (hop != 0) {
    CTN_TRY(chunk_plan(T, segment, hop, &tp->p));
    tp->T = T;
    return CTN_OK;
  }
  if (T <= 0 || segment <= 0) return CTN_EINVAL;
  const long long K = ((long long)T + segment - 1) / segment;
  if (K * segment > INT32_MAX) return CTN_EUNSUPPORTED;
  tp->p.T = (int)(K * segment); tp->p.Lc = segment; tp->p.hop = segment; tp->p.K = (int)K;
  tp->T = T;
  return CTN_OK;
}

extern "C" int ctn_track_plan(int T, int segment, int hop, int* starts, int capacity) {
  TrackPlan tp;
  CTN_TRY(track_plan(T, segment, hop, &tp));
  if (starts) {
    if (capacity < tp.p.K) return CTN_EINVAL;
    for (int k = 0; k < tp.p.K; ++k) starts[k] = tp.p.start(k);
  }
  return tp.p.K;
}

// statistics CTAs per (segment, channel): a function of the segment length alone
static int stats_split(int Lc) {
  const int g = (Lc + TRACK_SLICE - 1) / TRACK_SLICE;
  return g < 1 ? 1 : (g > TRACK_MAX_SPLIT ? TRACK_MAX_SPLIT : g);
}

// ---- statistics: partial[row][g] = (sum d, sum d^2) over CTA g's slice of row = (b K + k) C + c, d = x - x[start_k] -------------
// The shift by the segment's first sample keeps a large DC offset out of the squares.  Double throughout, fixed order (thread-
// strided slice, warp shuffles, warps in order); one flat grid of rows * G CTAs.
__global__ void __launch_bounds__(256) k_track_stats(const float* __restrict__ x, double* __restrict__ partial, TrackPlan tp, int C, int G) {
  __shared__ double red[8][2];
  const size_t blk = blockIdx.x, row = blk / G;
  const int g = (int)(blk - row * G);
  const int c = (int)(row % C);
  const size_t bk = row / C;
  const int b = (int)(bk / tp.p.K), k = (int)(bk - (size_t)b * tp.p.K);
  const float* src = x + ((size_t)b * C + c) * tp.T + tp.p.start(k);
  const int n_valid = tp.valid(k), Lc = tp.p.Lc;
  const double s = (double)src[0];
  const int slice = (Lc + G - 1) / G;
  const int q0 = g * slice, q1 = min(Lc, q0 + slice);
  double a1 = 0.0, a2 = 0.0;
  for (int q = q0 + threadIdx.x; q < q1; q += 256) {
    const double d = (q < n_valid ? (double)src[q] : 0.0) - s;
    a1 += d;
    a2 = fma(d, d, a2);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  a1 = warp_sum_d(a1);
  a2 = warp_sum_d(a2);
  if (lane == 0) { red[wid][0] = a1; red[wid][1] = a2; }
  __syncthreads();
  if (threadIdx.x < 2) {
    double v = 0.0;
    for (int w = 0; w < 8; ++w) v += red[w][threadIdx.x];
    partial[blk * 2 + threadIdx.x] = v;
  }
}

// stats[row] = (mean, unbiased std) over the Lc samples of the row (zeros past T included), the G partials summed in CTA order
__global__ void __launch_bounds__(256) k_track_stats_combine(const float* __restrict__ x, const double* __restrict__ partial,
                                                             double* __restrict__ stats, TrackPlan tp, int C, int G, size_t rows) {
  const size_t row = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (row >= rows) return;
  const int c = (int)(row % C);
  const size_t bk = row / C;
  const int b = (int)(bk / tp.p.K), k = (int)(bk - (size_t)b * tp.p.K);
  const double s = (double)x[((size_t)b * C + c) * tp.T + tp.p.start(k)];
  double s1 = 0.0, s2 = 0.0;
  for (int g = 0; g < G; ++g) { s1 += partial[(row * G + g) * 2]; s2 += partial[(row * G + g) * 2 + 1]; }
  const double n = (double)tp.p.Lc;
  const double var = fmax(s2 - s1 * (s1 / n), 0.0) / (n - 1.0);
  stats[row * 2] = s + s1 / n;
  stats[row * 2 + 1] = sqrt(var);
}

// ---- gather: xc[j][c][t] = (float)((x - mean) / (std + eps)) of chunk first + j = b K + k, zeros past T; rows (j, c) on gridDim.y -----
__global__ void __launch_bounds__(256) k_track_gather(const float* __restrict__ x, const double* __restrict__ stats, float* __restrict__ xc,
                                                      TrackPlan tp, int C, int first, double eps) {
  const int j = blockIdx.y / C, c = blockIdx.y - j * C;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= tp.p.Lc) return;
  const size_t g = (size_t)first + j;
  const int b = (int)(g / tp.p.K), k = (int)(g - (size_t)b * tp.p.K);
  const int at = tp.p.start(k) + t;
  const double v = at < tp.T ? (double)x[((size_t)b * C + c) * tp.T + at] : 0.0;
  const size_t row = g * C + c;
  xc[((size_t)j * C + c) * tp.p.Lc + t] = (float)((v - stats[row * 2]) / (stats[row * 2 + 1] + eps));
}

// ---- overlap-add, gather form: one thread per output time t of a (track, channel), all S sources ----------------------------------
// out[b][s][c][t] = sum_k w_k(t) (std_kc est_k[s][c](t - start_k) + mean_kc) / sum_k w_k(t), k ascending, in double; w_k = ola_weight
__global__ void __launch_bounds__(256) k_track_overlap_add(const float* __restrict__ est, const double* __restrict__ stats,
                                                           float* __restrict__ out, TrackPlan tp, int S, int C) {
  const int b = blockIdx.y / C, c = blockIdx.y - b * C;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= tp.T) return;
  const ChunkPlan& p = tp.p;
  int ks[4];
  double w[4], mu[4], sd[4], den = 0.0;
  int nc = 0;
  const int k_lo = t >= p.Lc ? (t - p.Lc) / p.hop + 1 : 0;
  const int k_hi = min(t / p.hop, p.K - 2);
  for (int k = k_lo; k <= k_hi; ++k) { ks[nc] = k; w[nc] = ola_weight(p, k, t - p.start(k)); den += w[nc]; ++nc; }
  if (t >= p.T - p.Lc) { ks[nc] = p.K - 1; w[nc] = ola_weight(p, p.K - 1, t - (p.T - p.Lc)); den += w[nc]; ++nc; }
  for (int i = 0; i < nc; ++i) {
    const size_t row = ((size_t)b * p.K + ks[i]) * C + c;
    mu[i] = stats[row * 2];
    sd[i] = stats[row * 2 + 1];
  }
  const double rden = 1.0 / den;
  for (int s = 0; s < S; ++s) {
    double num = 0.0;
    for (int i = 0; i < nc; ++i) {
      const size_t g = (size_t)b * p.K + ks[i];
      const double e = (double)est[((g * S + s) * C + c) * p.Lc + (t - p.start(ks[i]))];
      num = fma(w[i], fma(sd[i], e, mu[i]), num);
    }
    out[(((size_t)b * S + s) * C + c) * tp.T + t] = (float)(num * rden);
  }
}

// ---- launchers ---------------------------------------------------------------------------------------------------------------
static size_t track_rows(int B, int C, const TrackPlan& tp) { return (size_t)B * tp.p.K * C; }

static size_t stats_scratch_bytes(int B, int C, const TrackPlan& tp) {
  return sizeof(double) * 2 * track_rows(B, C, tp) * stats_split(tp.p.Lc);
}

static int launch_track_stats(const float* x, int B, int C, const TrackPlan& tp, double* stats, double* partial, cudaStream_t st) {
  const int G = stats_split(tp.p.Lc);
  const size_t rows = track_rows(B, C, tp);
  k_track_stats<<<(unsigned)(rows * G), 256, 0, st>>>(x, partial, tp, C, G);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  k_track_stats_combine<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(x, partial, stats, tp, C, G, rows);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

static int launch_track_gather(const float* x, const double* stats, float* xc, int C, const TrackPlan& tp, int first, int n, float eps,
                               cudaStream_t st) {
  k_track_gather<<<dim3((tp.p.Lc + 255) / 256, n * C), 256, 0, st>>>(x, stats, xc, tp, C, first, (double)eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

static int launch_track_ola(const float* est, const double* stats, float* out, int B, int S, int C, const TrackPlan& tp, cudaStream_t st) {
  k_track_overlap_add<<<dim3((tp.T + 255) / 256, B * C), 256, 0, st>>>(est, stats, out, tp, S, C);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// plan + shape checks shared by the steps: an unbiased std needs two samples per segment; the statistics grid is flat (rows * G
// CTAs on gridDim.x)
static int check_track_shape(int B, int C, int T, int segment, int hop, TrackPlan* tp) {
  CTN_TRY(track_plan(T, segment, hop, tp));
  if (B <= 0 || C <= 0 || C > 64) return CTN_EINVAL;
  if (tp->p.Lc < 2) return CTN_EINVAL;
  if ((long long)B * tp->p.K > INT32_MAX) return CTN_EUNSUPPORTED;
  if (track_rows(B, C, *tp) * stats_split(tp->p.Lc) > (size_t)INT32_MAX) return CTN_EUNSUPPORTED;
  return CTN_OK;
}

// ---- the three steps on their own ---------------------------------------------------------------------------------------------
extern "C" size_t ctn_track_stats_scratch_bytes(int B, int C, int T, int segment, int hop) {
  TrackPlan tp;
  if (check_track_shape(B, C, T, segment, hop, &tp) != CTN_OK) return 0;
  return stats_scratch_bytes(B, C, tp);
}

extern "C" int ctn_track_stats(const float* x, int B, int C, int T, int segment, int hop, double* stats, void* scratch, size_t scratch_bytes,
                               ctn_stream_t stream) {
  LaunchScope scope(x);
  TrackPlan tp;
  CTN_TRY(check_track_shape(B, C, T, segment, hop, &tp));
  if (!x || !stats || !scratch) return CTN_EINVAL;
  if ((((uintptr_t)stats) | ((uintptr_t)scratch)) & 7) return CTN_EALIGN;
  if (scratch_bytes < stats_scratch_bytes(B, C, tp)) return CTN_EWORKSPACE;
  return launch_track_stats(x, B, C, tp, stats, (double*)scratch, (cudaStream_t)stream);
}

extern "C" int ctn_track_gather(const float* x, const double* stats, int B, int C, int T, int segment, int hop, float eps, int first, int n,
                                float* xc, ctn_stream_t stream) {
  LaunchScope scope(x);
  TrackPlan tp;
  CTN_TRY(check_track_shape(B, C, T, segment, hop, &tp));
  if (!x || !stats || !xc || first < 0 || n <= 0 || (long long)first + n > (long long)B * tp.p.K) return CTN_EINVAL;
  if (!(eps >= 0.0f)) return CTN_EINVAL;
  if (((uintptr_t)stats) & 7) return CTN_EALIGN;
  if (!fits_grid_y((long long)n * C)) return CTN_EUNSUPPORTED;
  return launch_track_gather(x, stats, xc, C, tp, first, n, eps, (cudaStream_t)stream);
}

extern "C" int ctn_track_overlap_add(const float* est, const double* stats, int B, int S, int C, int T, int segment, int hop, float* out,
                                     ctn_stream_t stream) {
  LaunchScope scope(est);
  TrackPlan tp;
  CTN_TRY(check_track_shape(B, C, T, segment, hop, &tp));
  if (!est || !stats || !out || S <= 0) return CTN_EINVAL;
  if (((uintptr_t)stats) & 7) return CTN_EALIGN;
  if (!fits_grid_y((long long)B * C)) return CTN_EUNSUPPORTED;
  return launch_track_ola(est, stats, out, B, S, C, tp, (cudaStream_t)stream);
}

// ---- the whole call -------------------------------------------------------------------------------------------------------------
struct TrackWs {
  double* stats;    // (B K, C, 2) mean, std
  double* partial;  // statistics partials, (B K C, split, 2)
  float* xc;        // (nb, C, Lc) one standardised chunk batch
  float* est;       // (B K, S, C, Lc) chunk estimates
  void* model;      // workspace of ctn_convtasnet_fwd for one chunk batch
  size_t model_bytes;
  int nb;           // chunks per batch
};

static int track_channels(const ctn_config_t* c) { return c->in_channels > 1 ? c->in_channels : 1; }

static int carve_track(Carver& cv, const ctn_config_t* c, int B, const TrackPlan& tp, int chunk_batch, TrackWs* ws) {
  const int S = c->n_sources, C = track_channels(c);
  const long long chunks = (long long)B * tp.p.K;
  ws->nb = (int)(chunks < chunk_batch ? chunks : chunk_batch);
  // a batch's (chunk, channel) rows ride on gridDim.y, and so do the nb * S source rows of the forward's decoder
  const int rows = C > S ? C : S;
  if ((long long)ws->nb * rows > 65535) ws->nb = 65535 / rows;
  CTN_TRY(ctn_workspace_bytes(c, ws->nb, tp.p.Lc, &ws->model_bytes));
  ws->stats = cv.take<double>(track_rows(B, C, tp) * 2);
  ws->partial = cv.take<double>(stats_scratch_bytes(B, C, tp) / sizeof(double));
  ws->xc = cv.take<float>((size_t)ws->nb * C * tp.p.Lc);
  ws->est = cv.take<float>((size_t)chunks * S * C * tp.p.Lc);
  ws->model = cv.take<char>(ws->model_bytes);
  return CTN_OK;
}

static int check_track(const ctn_config_t* c, int B, int T, int segment, int hop, int chunk_batch, TrackPlan* tp) {
  CTN_TRY(check_model_cfg(c));
  if (chunk_batch <= 0) return CTN_EINVAL;
  const int C = track_channels(c);
  CTN_TRY(check_track_shape(B, C, T, segment, hop, tp));
  if (!fits_grid_y((long long)B * C)) return CTN_EUNSUPPORTED;
  return CTN_OK;
}

extern "C" int ctn_separate_track_workspace_bytes(const ctn_config_t* cfg, int B, int T, int segment, int hop, int chunk_batch, size_t* bytes) {
  TrackPlan tp;
  CTN_TRY(check_track(cfg, B, T, segment, hop, chunk_batch, &tp));
  if (!bytes) return CTN_EINVAL;
  Carver cv(nullptr);
  TrackWs ws;
  CTN_TRY(carve_track(cv, cfg, B, tp, chunk_batch, &ws));
  *bytes = cv.off + 256;
  return CTN_OK;
}

extern "C" int ctn_convtasnet_separate_track(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, int segment,
                                             int hop, int chunk_batch, float* out, void* workspace, size_t workspace_bytes,
                                             ctn_stream_t stream) {
  LaunchScope scope(x);
  TrackPlan tp;
  CTN_TRY(check_track(cfg, B, T, segment, hop, chunk_batch, &tp));
  if (!params || !params->blocks || !x || !out || !workspace) return CTN_EINVAL;
  if (((uintptr_t)workspace) & 255) return CTN_EALIGN;
  size_t need = 0;
  CTN_TRY(ctn_separate_track_workspace_bytes(cfg, B, T, segment, hop, chunk_batch, &need));
  if (workspace_bytes < need) return CTN_EWORKSPACE;
  const int S = cfg->n_sources, C = track_channels(cfg), Lc = tp.p.Lc;
  cudaStream_t st = (cudaStream_t)stream;
  Carver cv(workspace);
  TrackWs ws;
  CTN_TRY(carve_track(cv, cfg, B, tp, chunk_batch, &ws));
  CTN_TRY(launch_track_stats(x, B, C, tp, ws.stats, ws.partial, st));
  const int chunks = B * tp.p.K;
  for (int g0 = 0; g0 < chunks; g0 += ws.nb) {
    const int n = chunks - g0 < ws.nb ? chunks - g0 : ws.nb;
    CTN_TRY(launch_track_gather(x, ws.stats, ws.xc, C, tp, g0, n, cfg->eps, st));
    CTN_TRY(ctn_convtasnet_fwd(cfg, params, ws.xc, n, Lc, ws.est + (size_t)g0 * S * C * Lc, nullptr, ws.model, ws.model_bytes, stream));
  }
  return launch_track_ola(ws.est, ws.stats, out, B, S, C, tp, st);
}
