// One-and-rest PIT and Sinkhorn PIT over SI-SDR (src/criterion/pit.py:87-213).
// Both criteria need nothing but a table of per-pair SI-SDR statistics, so both share one two-pass pair kernel
// (k_pitx_stats, the numerics of k_pit_pass1/2 in ctn_loss.cu):
//   pass 1: dot[p] = <e_i, v_j>, tt[j] = |v_j|^2           pass 2: den[p] = |alpha_p v_j - e_i|^2 (explicit residual)
// where the "virtual" target rows v_j are
//   SinkPIT: the S target rows; pairs p = i*S + j cover every (estimate i, target j).
//   ORPIT:   t_0..t_{n-1} followed by the rests r_i = sum_{j<n_b, j!=i} t_j, formed on the fly in shared memory;
//            pairs p = 0..n-1 are (e_0, t_p), pairs p = n..2n-1 are (e_1, r_{p-n}).
// A CTA owns (sample, T-chunks): each chunk of every row is read from HBM once per pass and staged in shared memory, and
// each thread reduces one pair over a stride of the chunk (fp32 in groups of 4, double across groups and threads).
// The small per-sample work (candidate scores, the Sinkhorn iterations and their unrolled backward) runs in double with
// one CTA per sample, and both backward passes end in one streaming kernel: d_e_i = cx_i e_i + sum_j W_ij t_j.
#include <cmath>

#include "ctn_common.cuh"
#include "ctn_sisdr_grad.cuh"

#define PITX_MAX 16                            // S (SinkPIT) and n (ORPIT) limit of the fused path
#define PITX_C 256                             // T-chunk staged per row
#define PITX_CP (PITX_C + 1)                   // shared-memory row pitch (odd: pairs of one warp hit distinct banks)
#define PITX_ROWS (2 + 2 * PITX_MAX)           // ORPIT: e0, e1, n targets, n rests (SinkPIT: S + S)
#define PITX_CTAS 528                          // stats grid target: 4 CTAs on each of the H100 SXM's 132 SMs

// per-sample pair statistics (doubles): dot[P], den[P], tt[V]; P = ne*nt pairs, V virtual target rows
__host__ __device__ inline int pitx_pairs(int ne, int nt) { return ne * nt; }
__host__ __device__ inline int pitx_vrows(int nt, int orpit) { return orpit ? 2 * nt : nt; }
__host__ __device__ inline size_t pitx_stats_per_sample(int ne, int nt, int orpit) {
  return 2 * (size_t)pitx_pairs(ne, nt) + pitx_vrows(nt, orpit);
}

// sdr.py:135-137 from the pair statistics, in double
__device__ __forceinline__ double pitx_sisdr(const double* st, int P, int p, int v, double eps) {
  const double dot = st[p], den = st[P + p], tt = st[2 * P + v];
  const double alpha = dot / (tt + eps);
  return 10.0 * log10((alpha * alpha * tt + eps) / (den + eps));
}

// est (B, ne, T), tgt (B, nt, T), n_b (B) nullable: targets in use per sample (ORPIT; the rest of the rows are padding).
// grid (chunks, min(B, 65535)), block 256; samples loop over gridDim.y, so up to 65535 samples each CTA row owns one sample.
// PASS 1 accumulates dot and tt, PASS 2 den (needs the completed pass-1 sums).  Bounded to 6 CTAs per SM: 40 registers.
template <int PASS>
__global__ void __launch_bounds__(256, 6) k_pitx_stats(const float* __restrict__ est, const float* __restrict__ tgt,
                                                       const int* __restrict__ n_b, int B, int ne, int nt, int orpit, int T,
                                                       float eps, double* __restrict__ stats) {
  __shared__ float sh[PITX_ROWS * PITX_CP];
  const int tid = threadIdx.x;
  const int P = pitx_pairs(ne, nt);
  int KS = 32;  // threads per pair (consecutive lanes of one warp)
  while (KS > 1 && KS * P > 256) KS >>= 1;
  const int p = tid / KS, ks = tid % KS;
  const int nrow = ne + nt;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const int nb = n_b ? n_b[b] : nt;
    double* st = stats + (size_t)b * pitx_stats_per_sample(ne, nt, orpit);
    const bool act = p < P && (p % nt) < nb;
    const int er = act ? p / nt : 0, vr = act ? (orpit ? p : p % nt) : 0;
    const bool own_tt = act && (orpit || p < nt);
    const float* xe = sh + er * PITX_CP;
    const float* xv = sh + (ne + vr) * PITX_CP;
    float alpha = 0.f;
    if (PASS == 2 && act) alpha = (float)st[p] / ((float)st[2 * P + vr] + eps);  // sdr.py:135, as k_pit_pass2
    double acc0 = 0.0, acc1 = 0.0;
    for (int k0 = blockIdx.x * PITX_C; k0 < T; k0 += gridDim.x * PITX_C) {
      __syncthreads();
#pragma unroll 4
      for (int idx = tid; idx < nrow * PITX_C; idx += 256) {
        const int r = idx / PITX_C, k = idx % PITX_C, kk = k0 + k;
        const float* row = r < ne ? est + ((size_t)b * ne + r) * T : tgt + ((size_t)b * nt + (r - ne)) * T;
        sh[r * PITX_CP + k] = kk < T ? __ldg(row + kk) : 0.f;
      }
      if (orpit) {  // rests in the reference's order: sum over j of mask_rest * target (pit.py:135-138)
        __syncthreads();
        for (int idx = tid; idx < nb * PITX_C; idx += 256) {
          const int i = idx / PITX_C, k = idx % PITX_C;
          float r = 0.f;
          for (int j = 0; j < nb; ++j)
            if (j != i) r += sh[(ne + j) * PITX_CP + k];
          sh[(ne + nt + i) * PITX_CP + k] = r;
        }
      }
      __syncthreads();
      if (act) {
        float f0 = 0.f, f1 = 0.f;
        int m = 0;
#pragma unroll 4
        for (int k = ks; k < PITX_C; k += KS) {
          const float x = xe[k], v = xv[k];
          if (PASS == 1) {
            f0 += x * v;
            if (own_tt) f1 += v * v;
          } else {
            const float d = alpha * v - x;  // sdr.py:136 (alpha*target - input)
            f0 += d * d;
          }
          if ((++m & 3) == 0) { acc0 += (double)f0; acc1 += (double)f1; f0 = 0.f; f1 = 0.f; }
        }
        acc0 += (double)f0;
        acc1 += (double)f1;
      }
    }
    for (int o = KS >> 1; o > 0; o >>= 1) {
      acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
      acc1 += __shfl_xor_sync(0xffffffffu, acc1, o);
    }
    if (act && ks == 0) {
      if (PASS == 1) {
        atomicAdd(&st[p], acc0);
        if (own_tt) atomicAdd(&st[2 * P + vr], acc1);
      } else {
        atomicAdd(&st[P + p], acc0);
      }
    }
  }
}

static int launch_pitx_stats(const float* est, const float* tgt, const int* n_b, int B, int ne, int nt, int orpit, int T,
                             float eps, double* stats, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(stats, 0, sizeof(double) * (size_t)B * pitx_stats_per_sample(ne, nt, orpit), st);
  if (e != cudaSuccess) return (int)e;
  const int chunks = (T + PITX_C - 1) / PITX_C;
  int gx = (PITX_CTAS + B - 1) / B;
  if (gx > chunks) gx = chunks;
  const dim3 grid(gx, B < 65535 ? B : 65535);
  k_pitx_stats<1><<<grid, 256, 0, st>>>(est, tgt, n_b, B, ne, nt, orpit, T, eps, stats);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  k_pitx_stats<2><<<grid, 256, 0, st>>>(est, tgt, n_b, B, ne, nt, orpit, T, eps, stats);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// d_est (B, ne, T) = cx[b,i] * est_i + sum_j W[b,i,j] * tgt_j, W (B, ne, nt), cx (B, ne).  grid (chunks, min(B, 65535)),
// block 256; samples loop over gridDim.y as in k_pitx_stats, restaging w and c per sample.
__global__ void __launch_bounds__(256) k_pitx_pair_bwd(const float* __restrict__ est, const float* __restrict__ tgt,
                                                       const float* __restrict__ W, const float* __restrict__ cx, int B, int ne,
                                                       int nt, int T, float* __restrict__ d_est) {
  __shared__ float w[PITX_MAX * PITX_MAX], c[PITX_MAX];
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    __syncthreads();  // the previous sample's w and c are read until here
    for (int q = threadIdx.x; q < ne * nt; q += 256) w[(q / nt) * PITX_MAX + q % nt] = W[(size_t)b * ne * nt + q];
    if (threadIdx.x < ne) c[threadIdx.x] = cx[(size_t)b * ne + threadIdx.x];
    __syncthreads();
    const float* eb = est + (size_t)b * ne * T;
    const float* tb = tgt + (size_t)b * nt * T;
    float* db = d_est + (size_t)b * ne * T;
    for (int k = blockIdx.x * 256 + threadIdx.x; k < T; k += gridDim.x * 256) {
      float t[PITX_MAX];
#pragma unroll
      for (int j = 0; j < PITX_MAX; ++j) t[j] = j < nt ? __ldg(tb + (size_t)j * T + k) : 0.f;
      for (int i = 0; i < ne; ++i) {
        float a = c[i] * __ldg(eb + (size_t)i * T + k);
#pragma unroll
        for (int j = 0; j < PITX_MAX; ++j)
          if (j < nt) a = fmaf(w[i * PITX_MAX + j], t[j], a);
        db[(size_t)i * T + k] = a;
      }
    }
  }
}

static int launch_pitx_pair_bwd(const float* est, const float* tgt, const float* W, const float* cx, int B, int ne, int nt,
                                int T, float* d_est, cudaStream_t st) {
  int gx = (T + 1023) / 1024;
  if (gx > 64) gx = 64;
  k_pitx_pair_bwd<<<dim3(gx, B < 65535 ? B : 65535), 256, 0, st>>>(est, tgt, W, cx, B, ne, nt, T, d_est);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ------------------------------------------------------------------------------------------------------------------------
// ORPIT (pit.py:87-160).  Candidate i of sample b: v_i = SI-SDR(e0, t_i) + SI-SDR(e1, r_i) / (n_b - 1) in fp32; the
// reference takes the first min of -v_i for NegSISDR and the first max of v_i for SISDR, which is the same index.
// ------------------------------------------------------------------------------------------------------------------------
struct OrpitScratch {
  double* stats;  // B * pitx_stats_per_sample(2, n, 1)
  float* W;       // B * 2 * n
  float* cx;      // B * 2
};
static OrpitScratch orpit_carve(void* scratch, int B, int n) {
  OrpitScratch s;
  s.stats = (double*)scratch;
  s.W = (float*)(s.stats + (size_t)B * pitx_stats_per_sample(2, n, 1));
  s.cx = s.W + (size_t)B * 2 * n;
  return s;
}
extern "C" size_t ctn_orpit_scratch_bytes(int B, int n) {
  if (B <= 0 || n <= 0) return 0;
  return sizeof(double) * (size_t)B * pitx_stats_per_sample(2, n, 1) + sizeof(float) * (size_t)B * (2 * n + 2);
}

// one warp per sample, lane i = candidate i
__global__ void k_orpit_finalize(const double* __restrict__ stats, const int* __restrict__ n_b, int n, float eps, int maximize,
                                 float* __restrict__ loss_b, int64_t* __restrict__ indices) {
  const int b = blockIdx.x, i = threadIdx.x;
  const int nb = n_b ? n_b[b] : n, P = pitx_pairs(2, n);
  const double* st = stats + (size_t)b * pitx_stats_per_sample(2, n, 1);
  float v = -INFINITY;
  if (i < nb) {
    const float s0 = (float)pitx_sisdr(st, P, i, i, (double)eps);
    const float s1 = (float)pitx_sisdr(st, P, n + i, n + i, (double)eps);
    v = s0 + s1 / (float)(nb - 1);  // pit.py:142
  }
  int idx = i;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {  // first maximum (torch.max / torch.min, pit.py:150-153)
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  if (i == 0) {
    loss_b[b] = maximize ? v : -v;
    indices[b] = (int64_t)idx;
  }
}

// coefficients of the selected candidate: d loss_b / d SI-SDR(e0, t_i) = s, d / d SI-SDR(e1, r_i) = s / (n_b - 1),
// s = +-grad_loss_b; r_i's coefficient goes to every t_j it sums
__global__ void k_orpit_coef(const double* __restrict__ stats, const int* __restrict__ n_b, const int64_t* __restrict__ indices,
                             int B, int n, float eps, int maximize, const float* __restrict__ gl, float* __restrict__ W,
                             float* __restrict__ cx) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int nb = n_b ? n_b[b] : n, P = pitx_pairs(2, n), sel = (int)indices[b];
  const double* st = stats + (size_t)b * pitx_stats_per_sample(2, n, 1);
  const double g0 = (gl ? (double)gl[b] : 1.0) * (maximize ? 1.0 : -1.0), g1 = g0 / (double)(nb - 1);
  const double e = (double)eps;
  float ct0, cx0, ct1, cx1;
  sisdr_grad_coef(st[sel], st[P + sel], st[2 * P + sel], e, [=] { return g0; }, ct0, cx0);
  sisdr_grad_coef(st[n + sel], st[P + n + sel], st[2 * P + n + sel], e, [=] { return g1; }, ct1, cx1);
  float* w = W + (size_t)b * 2 * n;
  for (int j = 0; j < n; ++j) {
    w[j] = j == sel ? ct0 : 0.f;
    w[n + j] = (j != sel && j < nb) ? ct1 : 0.f;
  }
  cx[2 * b] = cx0;
  cx[2 * b + 1] = cx1;
}

// argument checks run before any CUDA call
static int orpit_check(const float* est, const float* tgt, const void* scratch, int B, int n, int T) {
  if (!est || !tgt || !scratch || B <= 0 || T <= 0 || n < 2) return CTN_EINVAL;
  if (n > PITX_MAX) return CTN_EUNSUPPORTED;
  return CTN_OK;
}

extern "C" int ctn_orpit_fwd(const float* est, const float* tgt, const int32_t* n_b, int B, int n, int T, float eps, int maximize,
                             float* loss_b, int64_t* indices, void* scratch, ctn_stream_t stream) {
  int rc = orpit_check(est, tgt, scratch, B, n, T);
  if (rc) return rc;
  if (!loss_b || !indices) return CTN_EINVAL;
  LaunchScope scope(est);
  cudaStream_t st = (cudaStream_t)stream;
  StageTimer tm(CTN_ST_LOSS, st);
  OrpitScratch s = orpit_carve(scratch, B, n);
  rc = launch_pitx_stats(est, tgt, n_b, B, 2, n, 1, T, eps, s.stats, st);
  if (rc) return rc;
  k_orpit_finalize<<<B, 32, 0, st>>>(s.stats, n_b, n, eps, maximize, loss_b, indices);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_orpit_bwd(const float* est, const float* tgt, const int32_t* n_b, const int64_t* indices, int B, int n, int T,
                             float eps, int maximize, void* scratch, const float* grad_loss_b, float* d_est, ctn_stream_t stream) {
  int rc = orpit_check(est, tgt, scratch, B, n, T);
  if (rc) return rc;
  if (!indices || !d_est) return CTN_EINVAL;
  LaunchScope scope(est);
  cudaStream_t st = (cudaStream_t)stream;
  StageTimer tm(CTN_ST_LOSS, st);
  OrpitScratch s = orpit_carve(scratch, B, n);
  k_orpit_coef<<<(B + 127) / 128, 128, 0, st>>>(s.stats, n_b, indices, B, n, eps, maximize, grad_loss_b, s.W, s.cx);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return launch_pitx_pair_bwd(est, tgt, s.W, s.cx, B, 2, n, T, d_est, st);
}

// ------------------------------------------------------------------------------------------------------------------------
// SinkPIT (pit.py:162-213).  L[i][j] = -SI-SDR(e_i, t_j) for both NegSISDR and SISDR (SISDR's table is negated, :177-178);
// Z = -coldness L, K times { Z -= logsumexp(Z, dim=1); Z -= logsumexp(Z, dim=2) }, P = exp(Z),
// loss_b = sign * sum (L + Z/coldness) P, sign = -1 for SISDR.  One CTA per sample, 16-lane segments: in the dim=1 phase
// segment j holds column j (lane = i), in the dim=2 phase segment i holds row i (lane = j).  Every logsumexp is kept in
// the scratch, which is all the backward needs to walk the K iterations back: Z_before = Z_after + lse.
// ------------------------------------------------------------------------------------------------------------------------
struct SinkScratch {
  double* stats;  // B * pitx_stats_per_sample(S, S, 0)
  double* Z;      // B * S * S: Z after the last iteration
  double* lse;    // B * 2K * S: logsumexp of every half-step
  float* W;       // B * S * S
  float* cx;      // B * S
};
static SinkScratch sink_carve(void* scratch, int B, int S, int K) {
  SinkScratch s;
  s.stats = (double*)scratch;
  s.Z = s.stats + (size_t)B * pitx_stats_per_sample(S, S, 0);
  s.lse = s.Z + (size_t)B * S * S;
  s.W = (float*)(s.lse + (size_t)B * 2 * K * S);
  s.cx = s.W + (size_t)B * S * S;
  return s;
}
extern "C" size_t ctn_sinkpit_scratch_bytes(int B, int S, int K) {
  if (B <= 0 || S <= 0 || K < 0) return 0;
  return sizeof(double) * (size_t)B * (pitx_stats_per_sample(S, S, 0) + (size_t)S * S + (size_t)2 * K * S) +
         sizeof(float) * (size_t)B * ((size_t)S * S + S);
}

__device__ __forceinline__ double seg16_max(double v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double seg16_sum(double v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block = 16 * S rounded up to a warp; smem tables [16][17] doubles
__global__ void k_sinkhorn_fwd(const double* __restrict__ stats, int S, int K, double coldness, float eps, int maximize,
                               double* __restrict__ Zout, double* __restrict__ lse_out, float* __restrict__ loss_b,
                               float* __restrict__ Pout, float* __restrict__ pair_sisdr) {
  __shared__ double L[PITX_MAX][PITX_MAX + 1], Z[PITX_MAX][PITX_MAX + 1], rowsum[PITX_MAX];
  const int b = blockIdx.x, seg = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const bool ok = seg < S && lane < S;
  const int P = S * S;
  const double* st = stats + (size_t)b * pitx_stats_per_sample(S, S, 0);
  if (ok) {  // row-phase mapping: i = seg, j = lane
    const double sd = pitx_sisdr(st, P, seg * S + lane, lane, (double)eps);
    L[seg][lane] = -sd;
    Z[seg][lane] = coldness * sd;
    if (pair_sisdr) pair_sisdr[(size_t)b * P + seg * S + lane] = (float)sd;
  }
  __syncthreads();
  double* lse_b = lse_out + (size_t)b * 2 * K * S;
  for (int it = 0; it < K; ++it) {
#pragma unroll
    for (int ph = 0; ph < 2; ++ph) {  // ph 0: dim=1 (over i, segment = column j), ph 1: dim=2 (over j, segment = row i)
      double& z = ph == 0 ? Z[ok ? lane : 0][ok ? seg : 0] : Z[ok ? seg : 0][ok ? lane : 0];
      const double v = ok ? z : -INFINITY;
      const double m = seg16_max(v);
      const double s = seg16_sum(ok ? exp(v - m) : 0.0);
      const double lse = m + log(s);
      if (ok) z = v - lse;
      if (ok && lane == 0) lse_b[(2 * it + ph) * S + seg] = lse;
      __syncthreads();
    }
  }
  double term = 0.0;
  if (ok) {
    const double z = Z[seg][lane], p = exp(z);
    term = (L[seg][lane] + z / coldness) * p;  // pit.py:191
    Zout[(size_t)b * P + seg * S + lane] = z;
    Pout[(size_t)b * P + seg * S + lane] = (float)p;
  }
  term = seg16_sum(term);
  if (ok && lane == 0) rowsum[seg] = term;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < S; ++i) tot += rowsum[i];
    loss_b[b] = (float)(maximize ? -tot : tot);
  }
}

// backward of k_sinkhorn_fwd through all K iterations: Z' = Z - lse(Z) along a dim  =>  dZ = dZ' - exp(Z') sum_dim dZ'.
// dL = g P - coldness dZ_0 (g = sign * grad_loss_b); writes dL and the pair-backward coefficients of -dL (L = -SI-SDR).
__global__ void k_sinkhorn_bwd(const double* __restrict__ stats, const double* __restrict__ Zin, const double* __restrict__ lse_in,
                               int S, int K, double coldness, float eps, int maximize, const float* __restrict__ gl,
                               const float* __restrict__ gP, float* __restrict__ dL, float* __restrict__ W, float* __restrict__ cx) {
  __shared__ double Z[PITX_MAX][PITX_MAX + 1], dZ[PITX_MAX][PITX_MAX + 1];
  __shared__ float cxs[PITX_MAX][PITX_MAX + 1];
  const int b = blockIdx.x, seg = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const bool ok = seg < S && lane < S;
  const int P = S * S;
  const double* st = stats + (size_t)b * pitx_stats_per_sample(S, S, 0);
  const double g = (gl ? (double)gl[b] : 1.0) * (maximize ? -1.0 : 1.0);
  double Ld = 0.0, Lv = 0.0;  // direct term g P and L of entry (seg, lane)
  if (ok) {
    const int q = seg * S + lane;
    const double z = Zin[(size_t)b * P + q], p = exp(z);
    Lv = -pitx_sisdr(st, P, q, lane, (double)eps);
    Ld = g * p;
    Z[seg][lane] = z;
    dZ[seg][lane] = g * (p / coldness + (Lv + z / coldness) * p) + (gP ? (double)gP[(size_t)b * P + q] * p : 0.0);
  }
  __syncthreads();
  const double* lse_b = lse_in + (size_t)b * 2 * K * S;
  for (int it = K - 1; it >= 0; --it) {
#pragma unroll
    for (int ph = 1; ph >= 0; --ph) {
      double& z = ph == 0 ? Z[ok ? lane : 0][ok ? seg : 0] : Z[ok ? seg : 0][ok ? lane : 0];
      double& dz = ph == 0 ? dZ[ok ? lane : 0][ok ? seg : 0] : dZ[ok ? seg : 0][ok ? lane : 0];
      const double za = ok ? z : 0.0, d = ok ? dz : 0.0;
      const double sd = seg16_sum(d);
      if (ok) {
        dz = d - exp(za) * sd;
        z = za + lse_b[(2 * it + ph) * S + seg];
      }
      __syncthreads();
    }
  }
  if (ok) {
    const int q = seg * S + lane;
    const double dl = Ld - coldness * dZ[seg][lane];
    dL[(size_t)b * P + q] = (float)dl;
    float ct, c;
    sisdr_grad_coef(st[q], st[P + q], st[2 * P + lane], (double)eps, [=] { return -dl; }, ct, c);
    W[(size_t)b * P + q] = ct;
    cxs[seg][lane] = c;
  }
  __syncthreads();
  if (threadIdx.x < S) {
    float a = 0.f;
    for (int j = 0; j < S; ++j) a += cxs[threadIdx.x][j];
    cx[(size_t)b * S + threadIdx.x] = a;
  }
}

static int sinkpit_check(const float* est, const float* tgt, const void* scratch, int B, int S, int T, int K, double coldness) {
  if (!est || !tgt || !scratch || B <= 0 || T <= 0 || S < 1 || K < 0 || !(coldness > 0.0) || !std::isfinite(coldness))
    return CTN_EINVAL;
  if (S > PITX_MAX) return CTN_EUNSUPPORTED;
  return CTN_OK;
}
static int sink_threads(int S) { return (16 * S + 31) / 32 * 32; }

extern "C" int ctn_sinkpit_fwd(const float* est, const float* tgt, int B, int S, int T, int K, double coldness, float eps,
                               int maximize, float* loss_b, float* P, float* pair_sisdr, void* scratch, ctn_stream_t stream) {
  int rc = sinkpit_check(est, tgt, scratch, B, S, T, K, coldness);
  if (rc) return rc;
  if (!loss_b || !P) return CTN_EINVAL;
  LaunchScope scope(est);
  cudaStream_t st = (cudaStream_t)stream;
  StageTimer tm(CTN_ST_LOSS, st);
  SinkScratch s = sink_carve(scratch, B, S, K);
  rc = launch_pitx_stats(est, tgt, nullptr, B, S, S, 0, T, eps, s.stats, st);
  if (rc) return rc;
  k_sinkhorn_fwd<<<B, sink_threads(S), 0, st>>>(s.stats, S, K, coldness, eps, maximize, s.Z, s.lse, loss_b, P, pair_sisdr);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_sinkpit_bwd(const float* est, const float* tgt, int B, int S, int T, int K, double coldness, float eps,
                               int maximize, void* scratch, const float* grad_loss_b, const float* grad_P, float* dL, float* d_est,
                               ctn_stream_t stream) {
  int rc = sinkpit_check(est, tgt, scratch, B, S, T, K, coldness);
  if (rc) return rc;
  if (!dL || !d_est) return CTN_EINVAL;
  LaunchScope scope(est);
  cudaStream_t st = (cudaStream_t)stream;
  StageTimer tm(CTN_ST_LOSS, st);
  SinkScratch s = sink_carve(scratch, B, S, K);
  k_sinkhorn_bwd<<<B, sink_threads(S), 0, st>>>(s.stats, s.Z, s.lse, S, K, coldness, eps, maximize, grad_loss_b, grad_P, dL, s.W,
                                                s.cx);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return launch_pitx_pair_bwd(est, tgt, s.W, s.cx, B, S, S, T, d_est, st);
}
