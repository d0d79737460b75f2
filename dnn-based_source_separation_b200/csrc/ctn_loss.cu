// SI-SDR + permutation-invariant training (PIT) loss.
//   reference: sisdr(), src/criterion/sdr.py:122-139; NegSISDR.forward :198-227; pit(), src/criterion/pit.py:9-44.
// The reference evaluates the criterion S! times on permuted targets (S! full passes over both tensors).  Here the
// S x S table of pairwise SI-SDR values is computed once in two streaming passes (HBM-bound, 128-bit loads along T):
//   pass 1: dot[i][j] = <e_i, t_j>, tt[j] = |t_j|^2                 -> alpha_ij = dot/(tt+eps)
//   pass 2: den[i][j] = |alpha_ij t_j - e_i|^2 (explicit residual, no cancellation), num = sum (alpha t)^2
// and a finalize kernel enumerates the permutations in itertools (lexicographic) order, takes the first minimum
// and writes the int64 permutation.  Accumulation is fp32 per thread-chunk, double across threads.
// PIT over plain SDR (further down) needs one pass only: its pair value is a function of |t_j|^2 and |t_j - e_i|^2, and it shares
// the permutation scoring through k_pit_finalize's Pair parameter.
#include "ctn_common.cuh"
#include "ctn_sisdr_grad.cuh"

#define CTN_MAX_S 6

// scratch layout per sample b (doubles): dot[S*S], den[S*S], tt[S]
__host__ __device__ inline size_t pit_scratch_per_sample(int S) { return (size_t)(2 * S * S + S); }

// Samples are looped over gridDim.y (at most 65535); up to that many samples each CTA row owns exactly one sample.
template <int S>
__global__ void __launch_bounds__(256) k_pit_pass1(const float* __restrict__ est, const float* __restrict__ tgt, int B, int T,
                                                   double* __restrict__ scratch) {
  __shared__ double red[64];
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const float* eb = est + (size_t)b * S * T;
    const float* tb = tgt + (size_t)b * S * T;
    double dot[S][S], tt[S];
#pragma unroll
    for (int i = 0; i < S; ++i) { tt[i] = 0.0;
#pragma unroll
      for (int j = 0; j < S; ++j) dot[i][j] = 0.0; }
    // 128-bit loads need every row 16-byte aligned: T % 4 == 0 and the sample's base (an offset view may start anywhere)
    const bool vec = (T % 4 == 0) && ((((uintptr_t)eb) | ((uintptr_t)tb)) & 15) == 0;
    const int nvec = vec ? T / 4 : 0;
    for (int v0 = blockIdx.x * 256 + threadIdx.x; v0 < nvec; v0 += gridDim.x * 256) {
      float4 e[S], t[S];
#pragma unroll
      for (int i = 0; i < S; ++i) {
        e[i] = __ldg(reinterpret_cast<const float4*>(eb + (size_t)i * T) + v0);
        t[i] = __ldg(reinterpret_cast<const float4*>(tb + (size_t)i * T) + v0);
      }
#pragma unroll
      for (int j = 0; j < S; ++j) {
        tt[j] += (double)((t[j].x * t[j].x + t[j].y * t[j].y) + (t[j].z * t[j].z + t[j].w * t[j].w));
#pragma unroll
        for (int i = 0; i < S; ++i)
          dot[i][j] += (double)((e[i].x * t[j].x + e[i].y * t[j].y) + (e[i].z * t[j].z + e[i].w * t[j].w));
      }
    }
    if (!vec) {
      for (int k = blockIdx.x * 256 + threadIdx.x; k < T; k += gridDim.x * 256) {
        float e[S], t[S];
#pragma unroll
        for (int i = 0; i < S; ++i) { e[i] = eb[(size_t)i * T + k]; t[i] = tb[(size_t)i * T + k]; }
#pragma unroll
        for (int j = 0; j < S; ++j) {
          tt[j] += (double)(t[j] * t[j]);
#pragma unroll
          for (int i = 0; i < S; ++i) dot[i][j] += (double)(e[i] * t[j]);
        }
      }
    }
    double* sc = scratch + (size_t)b * pit_scratch_per_sample(S);
#pragma unroll
    for (int j = 0; j < S; ++j) {
#pragma unroll
      for (int i = 0; i < S; i += 2) {
        double a = dot[i][j], c = (i + 1 < S) ? dot[i + 1][j] : 0.0;
        block_sum2_d(a, c, red);
        if (threadIdx.x == 0) {
          atomicAdd(&sc[i * S + j], a);
          if (i + 1 < S) atomicAdd(&sc[(i + 1) * S + j], c);
        }
        __syncthreads();
      }
    }
#pragma unroll
    for (int j = 0; j < S; j += 2) {
      double a = tt[j], c = (j + 1 < S) ? tt[j + 1] : 0.0;
      block_sum2_d(a, c, red);
      if (threadIdx.x == 0) {
        atomicAdd(&sc[2 * S * S + j], a);
        if (j + 1 < S) atomicAdd(&sc[2 * S * S + j + 1], c);
      }
      __syncthreads();
    }
  }
}

template <int S>
__global__ void __launch_bounds__(256) k_pit_pass2(const float* __restrict__ est, const float* __restrict__ tgt, int B, int T,
                                                   float eps, double* __restrict__ scratch) {
  __shared__ double red[64];
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const float* eb = est + (size_t)b * S * T;
    const float* tb = tgt + (size_t)b * S * T;
    double* sc = scratch + (size_t)b * pit_scratch_per_sample(S);
    float alpha[S][S];
#pragma unroll
    for (int i = 0; i < S; ++i)
#pragma unroll
      for (int j = 0; j < S; ++j) alpha[i][j] = (float)sc[i * S + j] / ((float)sc[2 * S * S + j] + eps);  // sdr.py:135
    double den[S][S];
#pragma unroll
    for (int i = 0; i < S; ++i)
#pragma unroll
      for (int j = 0; j < S; ++j) den[i][j] = 0.0;
    for (int k = blockIdx.x * 256 + threadIdx.x; k < T; k += gridDim.x * 256) {
      float e[S], t[S];
#pragma unroll
      for (int i = 0; i < S; ++i) { e[i] = __ldg(eb + (size_t)i * T + k); t[i] = __ldg(tb + (size_t)i * T + k); }
#pragma unroll
      for (int i = 0; i < S; ++i)
#pragma unroll
        for (int j = 0; j < S; ++j) {
          const float d = alpha[i][j] * t[j] - e[i];  // sdr.py:136 (alpha*target - input)
          den[i][j] += (double)(d * d);
        }
    }
#pragma unroll
    for (int i = 0; i < S; ++i) {
#pragma unroll
      for (int j = 0; j < S; j += 2) {
        double a = den[i][j], c = (j + 1 < S) ? den[i][j + 1] : 0.0;
        block_sum2_d(a, c, red);
        if (threadIdx.x == 0) {
          atomicAdd(&sc[S * S + i * S + j], a);
          if (j + 1 < S) atomicAdd(&sc[S * S + i * S + j + 1], c);
        }
        __syncthreads();
      }
    }
  }
}

// Pair value of the SI-SDR PIT: v[i][j] = SI-SDR(est_i, tgt_j) from the pass statistics (dot, den, tt).
struct SisdrPair {
  static __device__ size_t per_sample(int S) { return pit_scratch_per_sample(S); }
  static __device__ float value(const double* sc, int S, int p, float eps) {
    const int j = p % S;
    const float tt = (float)sc[2 * S * S + j];
    const float alpha = (float)sc[p] / (tt + eps);
    const float num = alpha * alpha * tt;  // sum((alpha*target)^2), sdr.py:136
    const float den = (float)sc[S * S + p];
    return 10.f * log10f((num + eps) / (den + eps));  // sdr.py:136-137
  }
};

// One block per sample, thread p = permutation index (lexicographic); block = 32*ceil(S!/32).  Pair supplies the sample's
// scratch stride and the value of pair p = i*S + j; everything after the pair table is shared by the SI-SDR and SDR PITs.
template <class Pair>
__global__ void k_pit_finalize(const double* __restrict__ scratch, int S, int nperm, float eps, float* __restrict__ loss_b,
                               int64_t* __restrict__ perm, float* __restrict__ pair_out) {
  __shared__ float sd[CTN_MAX_S * CTN_MAX_S];
  __shared__ float best_v[32];
  __shared__ int best_i[32];
  const int b = blockIdx.x, p = threadIdx.x;
  const double* sc = scratch + (size_t)b * Pair::per_sample(S);
  if (p < S * S) {
    const float v = Pair::value(sc, S, p, eps);
    sd[p] = v;
    if (pair_out) pair_out[(size_t)b * S * S + p] = v;
  }
  __syncthreads();
  float myloss = INFINITY;
  int pi[CTN_MAX_S];
  if (p < nperm) {
    // decode p-th lexicographic permutation (factoradic) -- itertools.permutations order, pit.py:55
    int avail[CTN_MAX_S];
    for (int i = 0; i < S; ++i) avail[i] = i;
    int fact = 1;
    for (int i = 2; i < S; ++i) fact *= i;  // (S-1)!
    int rem = p;
    for (int i = 0; i < S; ++i) {
      const int q = rem / fact;
      rem -= q * fact;
      pi[i] = avail[q];
      for (int k = q; k < S - 1 - i; ++k) avail[k] = avail[k + 1];
      if (S - 1 - i > 0) fact /= (S - 1 - i);
    }
    float acc = 0.f;
    for (int i = 0; i < S; ++i) acc += -sd[i * S + pi[i]];  // NegSISDR / NegSDR (sdr.py:212), target permuted (pit.py:30)
    myloss = acc / (float)S;                                // reduction='mean' over sources (sdr.py:216)
  }
  // first-minimum argmin over p (torch.min, pit.py:39)
  float v = myloss;
  int idx = p;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov < v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  const int lane = p & 31, wid = p >> 5, nw = blockDim.x >> 5;
  if (lane == 0) { best_v[wid] = v; best_i[wid] = idx; }
  __syncthreads();
  if (p == 0) {
    for (int w = 1; w < nw; ++w)
      if (best_v[w] < v || (best_v[w] == v && best_i[w] < idx)) { v = best_v[w]; idx = best_i[w]; }
    best_i[0] = idx;
    loss_b[b] = v;
  }
  __syncthreads();
  if (p == best_i[0] && p < nperm)
    for (int i = 0; i < S; ++i) perm[(size_t)b * S + i] = (int64_t)pi[i];
}

__global__ void k_batch_mean(const float* __restrict__ loss_b, int B, float* __restrict__ out) {
  // single warp, sequential-order-independent double sum (pit.py:41-42)
  double s = 0.0;
  for (int i = threadIdx.x; i < B; i += 32) s += (double)loss_b[i];
  s = warp_sum_d(s);
  if (threadIdx.x == 0) out[0] = (float)(s / (double)B);
}

// gridDim.y is at most 65535; the kernels loop over the rest of the rows
static unsigned grid_rows(int rows) { return rows < 65535 ? (unsigned)rows : 65535u; }

// permutation scoring (+ the batch mean when loss_mean is given) from the pair statistics in scratch
template <class Pair>
static int launch_pit_finalize(const double* scratch, int B, int S, float eps, float* loss_b, int64_t* perm, float* loss_mean,
                               float* pair_out, cudaStream_t st) {
  int nperm = 1;
  for (int i = 2; i <= S; ++i) nperm *= i;
  int threads = ((nperm > S * S ? nperm : S * S) + 31) / 32 * 32;
  k_pit_finalize<Pair><<<B, threads, 0, st>>>(scratch, S, nperm, eps, loss_b, perm, pair_out);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  if (loss_mean) {
    k_batch_mean<<<1, 32, 0, st>>>(loss_b, B, loss_mean);
    CTN_COUNT_LAUNCH();
    CTN_RETURN_IF_CUDA_ERR();
  }
  return CTN_OK;
}

template <int S>
static int launch_pit(const float* est, const float* tgt, int B, int T, float eps, double* scratch, cudaStream_t st) {
  int gx = (T / 4 + 255) / 256;
  if (gx < 1) gx = 1;
  if (gx > 32) gx = 32;
  k_pit_pass1<S><<<dim3(gx, grid_rows(B)), 256, 0, st>>>(est, tgt, B, T, scratch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  int gx2 = (T + 255) / 256;
  if (gx2 > 64) gx2 = 64;
  k_pit_pass2<S><<<dim3(gx2, grid_rows(B)), 256, 0, st>>>(est, tgt, B, T, eps, scratch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" size_t ctn_sisdr_pit_scratch_bytes(int B, int S) { return sizeof(double) * (size_t)B * pit_scratch_per_sample(S); }

extern "C" int ctn_sisdr_pit_fwd(const float* est, const float* tgt, int B, int S, int T, float eps, float* loss_b,
                                 int64_t* perm, float* loss_mean, float* pair_sisdr, double* scratch,
                                 ctn_stream_t stream) {
  LaunchScope scope(est);
  if (!est || !tgt || !loss_b || !perm || !scratch || B <= 0 || T <= 0) return CTN_EINVAL;
  if (S < 1 || S > CTN_MAX_S) return CTN_EUNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  StageTimer tm(CTN_ST_LOSS, st);
  cudaError_t e = cudaMemsetAsync(scratch, 0, ctn_sisdr_pit_scratch_bytes(B, S), st);
  if (e != cudaSuccess) return (int)e;
  int rc;
  switch (S) {
    case 1: rc = launch_pit<1>(est, tgt, B, T, eps, scratch, st); break;
    case 2: rc = launch_pit<2>(est, tgt, B, T, eps, scratch, st); break;
    case 3: rc = launch_pit<3>(est, tgt, B, T, eps, scratch, st); break;
    case 4: rc = launch_pit<4>(est, tgt, B, T, eps, scratch, st); break;
    case 5: rc = launch_pit<5>(est, tgt, B, T, eps, scratch, st); break;
    default: rc = launch_pit<6>(est, tgt, B, T, eps, scratch, st); break;
  }
  if (rc) return rc;
  return launch_pit_finalize<SisdrPair>(scratch, B, S, eps, loss_b, perm, loss_mean, pair_sisdr, st);
}

__global__ void k_sisdr_finalize(const double* __restrict__ scratch, int rows, float eps, float* __restrict__ out) {
  const int r = blockIdx.x * 128 + threadIdx.x;
  if (r >= rows) return;
  const double* sc = scratch + (size_t)r * 3;  // dot, den, tt
  const float tt = (float)sc[2];
  const float alpha = (float)sc[0] / (tt + eps);
  const float num = alpha * alpha * tt;
  out[r] = 10.f * log10f((num + eps) / ((float)sc[1] + eps));
}

// plain sisdr(est[r], tgt[r]) per row: reuse the S=1 kernels with B=rows
extern "C" int ctn_sisdr_fwd(const float* est, const float* tgt, int rows, int T, float eps, float* out, double* scratch,
                             ctn_stream_t stream) {
  LaunchScope scope(est);
  if (!est || !tgt || !out || !scratch || rows <= 0 || T <= 0) return CTN_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(scratch, 0, ctn_sisdr_pit_scratch_bytes(rows, 1), st);
  if (e != cudaSuccess) return (int)e;
  int rc = launch_pit<1>(est, tgt, rows, T, eps, scratch, st);
  if (rc) return rc;
  k_sisdr_finalize<<<(rows + 127) / 128, 128, 0, st>>>(scratch, rows, eps, out);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}


// ---- plain SDR (src/criterion/sdr.py:6-20): 10 log10((|t|^2 + eps) / (|t - x|^2 + eps)) per row -------------------------
// The residual is accumulated explicitly (not as |t|^2 - 2<x,t> + |x|^2, which cancels catastrophically at high SDR), in double.
__global__ void __launch_bounds__(256) k_sdr_partial(const float* __restrict__ est, const float* __restrict__ tgt, int rows, int T,
                                                     double* __restrict__ scratch) {
  __shared__ double red[64];
  for (int r = blockIdx.y; r < rows; r += gridDim.y) {
    const float* x = est + (size_t)r * T;
    const float* t = tgt + (size_t)r * T;
    double tt = 0.0, ee = 0.0;
    const bool vec = ((((uintptr_t)x) | ((uintptr_t)t)) & 15) == 0;
    const int n4 = vec ? T / 4 : 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(x) + i), b = __ldg(reinterpret_cast<const float4*>(t) + i);
      const float d0 = b.x - a.x, d1 = b.y - a.y, d2 = b.z - a.z, d3 = b.w - a.w;
      tt += (double)(fmaf(b.x, b.x, b.y * b.y) + fmaf(b.z, b.z, b.w * b.w));
      ee += (double)(fmaf(d0, d0, d1 * d1) + fmaf(d2, d2, d3 * d3));
    }
    for (int i = n4 * 4 + blockIdx.x * blockDim.x + threadIdx.x; i < T; i += gridDim.x * blockDim.x) {
      const float b = t[i], d = b - x[i];
      tt += (double)b * b;
      ee += (double)d * d;
    }
    block_sum2_d(tt, ee, red);
    if (threadIdx.x == 0) { atomicAdd(&scratch[2 * r], tt); atomicAdd(&scratch[2 * r + 1], ee); }
    if (r + gridDim.y < rows) __syncthreads();  // red is reused by the next row
  }
}
__global__ void k_sdr_finalize(const double* __restrict__ scratch, int rows, float eps, float* __restrict__ out) {
  const int r = blockIdx.x * 128 + threadIdx.x;
  if (r >= rows) return;
  out[r] = 10.f * log10f(((float)scratch[2 * r] + eps) / ((float)scratch[2 * r + 1] + eps));
}

extern "C" int ctn_sdr_fwd(const float* est, const float* tgt, int rows, int T, float eps, float* out, double* scratch, ctn_stream_t stream) {
  LaunchScope scope(est);
  if (!est || !tgt || !out || !scratch || rows <= 0 || T <= 0) return CTN_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * rows, st);
  if (e != cudaSuccess) return (int)e;
  int gx = (T / 4 + 1023) / 1024;
  if (gx < 1) gx = 1;
  if (gx > 64) gx = 64;
  k_sdr_partial<<<dim3(gx, grid_rows(rows)), 256, 0, st>>>(est, tgt, rows, T, scratch);
  CTN_COUNT_LAUNCH();
  k_sdr_finalize<<<(rows + 127) / 128, 128, 0, st>>>(scratch, rows, eps, out);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- SDR gradient and PIT over SDR -------------------------------------------------------------------------------------------
// d SDR(x, t) / d x = 20 / (ln 10 (|t - x|^2 + eps)) (t - x): one row coefficient, formed in double from the forward's residual
// sum, times the fp32 difference.  sdr_row_grad streams one row with 128-bit accesses when all three bases are 16-byte aligned
// (a view may start anywhere; T need not be a multiple of 4: the tail goes element by element).
__device__ __forceinline__ void sdr_row_grad(const float* __restrict__ x, const float* __restrict__ t, float* __restrict__ d, int T,
                                             float c) {
  const bool vec = ((((uintptr_t)x) | ((uintptr_t)t) | ((uintptr_t)d)) & 15) == 0;
  const int n4 = vec ? T / 4 : 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(x) + i), b = __ldg(reinterpret_cast<const float4*>(t) + i);
    reinterpret_cast<float4*>(d)[i] = make_float4(c * (b.x - a.x), c * (b.y - a.y), c * (b.z - a.z), c * (b.w - a.w));
  }
  for (int i = n4 * 4 + blockIdx.x * blockDim.x + threadIdx.x; i < T; i += gridDim.x * blockDim.x) d[i] = c * (__ldg(t + i) - __ldg(x + i));
}

__device__ __forceinline__ float sdr_grad_coef(double ee, double eps, double g) {
  return (float)(g * 8.685889638065035 / (ee + eps));  // 20 / ln 10
}

// grid (chunks, min(rows, 65535)), block 256; scratch = ctn_sdr_fwd's (|t|^2, |t - x|^2) per row
__global__ void __launch_bounds__(256) k_sdr_bwd(const float* __restrict__ est, const float* __restrict__ tgt, int rows, int T, float eps,
                                                 const double* __restrict__ scratch, const float* __restrict__ g, float coef,
                                                 float* __restrict__ d_est) {
  for (int r = blockIdx.y; r < rows; r += gridDim.y) {
    const float c = sdr_grad_coef(scratch[2 * r + 1], (double)eps, (g ? (double)g[r] : 1.0) * (double)coef);
    sdr_row_grad(est + (size_t)r * T, tgt + (size_t)r * T, d_est + (size_t)r * T, T, c);
  }
}

static int sdr_grad_chunks(int T) {
  int gx = (T / 4 + 1023) / 1024;
  if (gx < 1) gx = 1;
  return gx > 64 ? 64 : gx;
}

extern "C" int ctn_sdr_bwd(const float* est, const float* tgt, int rows, int T, float eps, const double* fwd_scratch, const float* grad_out,
                           float coef, float* d_est, ctn_stream_t stream) {
  LaunchScope scope(est);
  if (!est || !tgt || !fwd_scratch || !d_est || rows <= 0 || T <= 0) return CTN_EINVAL;
  k_sdr_bwd<<<dim3(sdr_grad_chunks(T), grid_rows(rows)), 256, 0, (cudaStream_t)stream>>>(est, tgt, rows, T, eps, fwd_scratch, grad_out,
                                                                                          coef, d_est);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// PIT over SDR.  Scratch per sample (doubles): ee[S*S] = |t_j - x_i|^2 at i*S + j, then tt[S] = |t_j|^2.  One streaming pass forms
// both with the explicit residual, in fp32 runs of at most four summed in double (k_sdr_partial's arithmetic); the finalize kernel
// is the SI-SDR PIT's with SdrPair's value.
__host__ __device__ inline size_t sdr_pit_scratch_per_sample(int S) { return (size_t)(S * S + S); }

struct SdrPair {
  static __device__ size_t per_sample(int S) { return sdr_pit_scratch_per_sample(S); }
  static __device__ float value(const double* sc, int S, int p, float eps) {
    return 10.f * log10f(((float)sc[S * S + p % S] + eps) / ((float)sc[p] + eps));  // k_sdr_finalize's expression
  }
};

template <int S>
__global__ void __launch_bounds__(256) k_sdr_pit_pass(const float* __restrict__ est, const float* __restrict__ tgt, int B, int T,
                                                      double* __restrict__ scratch) {
  __shared__ double red[64];
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const float* eb = est + (size_t)b * S * T;
    const float* tb = tgt + (size_t)b * S * T;
    double ee[S][S], tt[S];
#pragma unroll
    for (int i = 0; i < S; ++i) { tt[i] = 0.0;
#pragma unroll
      for (int j = 0; j < S; ++j) ee[i][j] = 0.0; }
    // 128-bit loads need every row of the sample 16-byte aligned: T % 4 == 0 and aligned sample bases
    const bool vec = (T % 4 == 0) && ((((uintptr_t)eb) | ((uintptr_t)tb)) & 15) == 0;
    const int nvec = vec ? T / 4 : 0;
    for (int v0 = blockIdx.x * 256 + threadIdx.x; v0 < nvec; v0 += gridDim.x * 256) {
      float4 e[S], t[S];
#pragma unroll
      for (int i = 0; i < S; ++i) {
        e[i] = __ldg(reinterpret_cast<const float4*>(eb + (size_t)i * T) + v0);
        t[i] = __ldg(reinterpret_cast<const float4*>(tb + (size_t)i * T) + v0);
      }
#pragma unroll
      for (int j = 0; j < S; ++j) {
        tt[j] += (double)(fmaf(t[j].x, t[j].x, t[j].y * t[j].y) + fmaf(t[j].z, t[j].z, t[j].w * t[j].w));
#pragma unroll
        for (int i = 0; i < S; ++i) {
          const float d0 = t[j].x - e[i].x, d1 = t[j].y - e[i].y, d2 = t[j].z - e[i].z, d3 = t[j].w - e[i].w;
          ee[i][j] += (double)(fmaf(d0, d0, d1 * d1) + fmaf(d2, d2, d3 * d3));
        }
      }
    }
    if (!vec) {
      for (int k = blockIdx.x * 256 + threadIdx.x; k < T; k += gridDim.x * 256) {
        float e[S], t[S];
#pragma unroll
        for (int i = 0; i < S; ++i) { e[i] = __ldg(eb + (size_t)i * T + k); t[i] = __ldg(tb + (size_t)i * T + k); }
#pragma unroll
        for (int j = 0; j < S; ++j) {
          tt[j] += (double)t[j] * t[j];
#pragma unroll
          for (int i = 0; i < S; ++i) {
            const float d = t[j] - e[i];
            ee[i][j] += (double)d * d;
          }
        }
      }
    }
    double* sc = scratch + (size_t)b * sdr_pit_scratch_per_sample(S);
#pragma unroll
    for (int i = 0; i < S; ++i) {
#pragma unroll
      for (int j = 0; j < S; j += 2) {
        double a = ee[i][j], c = (j + 1 < S) ? ee[i][j + 1] : 0.0;
        block_sum2_d(a, c, red);
        if (threadIdx.x == 0) {
          atomicAdd(&sc[i * S + j], a);
          if (j + 1 < S) atomicAdd(&sc[i * S + j + 1], c);
        }
        __syncthreads();
      }
    }
#pragma unroll
    for (int j = 0; j < S; j += 2) {
      double a = tt[j], c = (j + 1 < S) ? tt[j + 1] : 0.0;
      block_sum2_d(a, c, red);
      if (threadIdx.x == 0) {
        atomicAdd(&sc[S * S + j], a);
        if (j + 1 < S) atomicAdd(&sc[S * S + j + 1], c);
      }
      __syncthreads();
    }
  }
}

template <int S>
static int launch_sdr_pit(const float* est, const float* tgt, int B, int T, double* scratch, cudaStream_t st) {
  int gx = (T / 4 + 255) / 256;
  if (gx < 1) gx = 1;
  if (gx > 32) gx = 32;
  k_sdr_pit_pass<S><<<dim3(gx, grid_rows(B)), 256, 0, st>>>(est, tgt, B, T, scratch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" size_t ctn_sdr_pit_scratch_bytes(int B, int S) { return sizeof(double) * (size_t)B * sdr_pit_scratch_per_sample(S); }

extern "C" int ctn_sdr_pit_fwd(const float* est, const float* tgt, int B, int S, int T, float eps, float* loss_b, int64_t* perm,
                               float* loss_mean, float* pair_sdr, double* scratch, ctn_stream_t stream) {
  LaunchScope scope(est);
  if (!est || !tgt || !loss_b || !perm || !scratch || B <= 0 || T <= 0) return CTN_EINVAL;
  if (S < 1 || S > CTN_MAX_S) return CTN_EUNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  StageTimer tm(CTN_ST_LOSS, st);
  cudaError_t e = cudaMemsetAsync(scratch, 0, ctn_sdr_pit_scratch_bytes(B, S), st);
  if (e != cudaSuccess) return (int)e;
  int rc;
  switch (S) {
    case 1: rc = launch_sdr_pit<1>(est, tgt, B, T, scratch, st); break;
    case 2: rc = launch_sdr_pit<2>(est, tgt, B, T, scratch, st); break;
    case 3: rc = launch_sdr_pit<3>(est, tgt, B, T, scratch, st); break;
    case 4: rc = launch_sdr_pit<4>(est, tgt, B, T, scratch, st); break;
    case 5: rc = launch_sdr_pit<5>(est, tgt, B, T, scratch, st); break;
    default: rc = launch_sdr_pit<6>(est, tgt, B, T, scratch, st); break;
  }
  if (rc) return rc;
  return launch_pit_finalize<SdrPair>(scratch, B, S, eps, loss_b, perm, loss_mean, pair_sdr, st);
}

// backward through the selected permutation: row (b, i) reads ee[i][perm[b][i]] from the forward's scratch
__global__ void __launch_bounds__(256) k_sdr_pit_bwd(const float* __restrict__ est, const float* __restrict__ tgt,
                                                     const int64_t* __restrict__ perm, const double* __restrict__ scratch,
                                                     const float* __restrict__ gl, float coef, int B, int S, int T, float eps,
                                                     float* __restrict__ d_est) {
  for (int row = blockIdx.y; row < B * S; row += gridDim.y) {
    const int b = row / S, i = row % S;
    const int j = (int)perm[(size_t)b * S + i];
    const double ee = scratch[(size_t)b * sdr_pit_scratch_per_sample(S) + i * S + j];
    const float c = sdr_grad_coef(ee, (double)eps, (gl ? (double)gl[b] : 1.0) * (double)coef);
    sdr_row_grad(est + (size_t)row * T, tgt + ((size_t)b * S + j) * T, d_est + (size_t)row * T, T, c);
  }
}

extern "C" int ctn_sdr_pit_bwd(const float* est, const float* tgt, const int64_t* perm, int B, int S, int T, float eps,
                               const double* fwd_scratch, const float* grad_loss_b, float coef, float* d_est, ctn_stream_t stream) {
  LaunchScope scope(est);
  if (!est || !tgt || !perm || !fwd_scratch || !d_est || B <= 0 || T <= 0) return CTN_EINVAL;
  if (S < 1 || S > CTN_MAX_S) return CTN_EUNSUPPORTED;
  k_sdr_pit_bwd<<<dim3(sdr_grad_chunks(T), grid_rows(B * S)), 256, 0, (cudaStream_t)stream>>>(est, tgt, perm, fwd_scratch, grad_loss_b,
                                                                                               coef, B, S, T, eps, d_est);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ------------------------------------------------------------------------------------------------
// backward of PIT(NegSISDR) through the SELECTED permutation (pit.py:36-44: the indices carry no gradient).
// The per-pair coefficients (ct, cx) come from sisdr_grad_coef (ctn_sisdr_grad.cuh).
// The pair statistics <x,t>, |alpha t - x|^2, |t|^2 are the ones the forward left in its scratch (explicit residual,
// double), so the backward is one streaming pass.  grid (chunks, min(B*S, 65535)), block 256.
// ------------------------------------------------------------------------------------------------
// Bounded to six CTAs per SM (40 registers): the compiler versions the row loop on `gl`, which otherwise takes 48 (five CTAs).
__global__ void __launch_bounds__(256, 6) k_sisdr_pit_bwd(const float* __restrict__ est, const float* __restrict__ tgt,
                                                          const int64_t* __restrict__ perm, const double* __restrict__ scratch,
                                                          const float* __restrict__ gl, float coef, int B, int S, int T,
                                                          float eps, float* __restrict__ d_est) {
  for (int row = blockIdx.y; row < B * S; row += gridDim.y) {
    const int b = row / S, i = row % S;
    const int j = (int)perm[(size_t)b * S + i];
    const double* sc = scratch + (size_t)b * pit_scratch_per_sample(S);
    const double xt = sc[i * S + j], den = sc[S * S + i * S + j], tt = sc[2 * S * S + j];
    float ct, cx;
    sisdr_grad_coef(xt, den, tt, (double)eps, [&] { return (gl ? (double)gl[b] : 1.0) * (double)coef; }, ct, cx);
    const float* x = est + (size_t)row * T;
    const float* t = tgt + ((size_t)b * S + j) * T;
    float* d = d_est + (size_t)row * T;
    for (int k = blockIdx.x * 256 + threadIdx.x; k < T; k += gridDim.x * 256) d[k] = fmaf(ct, t[k], cx * x[k]);
  }
}

extern "C" int ctn_sisdr_pit_bwd(const float* est, const float* tgt, const int64_t* perm, int B, int S, int T, float eps,
                                 const double* fwd_scratch, const float* grad_loss_b, float coef, float* d_est,
                                 ctn_stream_t stream) {
  LaunchScope scope(est);
  if (!est || !tgt || !perm || !fwd_scratch || !d_est || B <= 0 || T <= 0) return CTN_EINVAL;
  if (S < 1 || S > CTN_MAX_S) return CTN_EUNSUPPORTED;
  int gx = (T + 1023) / 1024;
  if (gx > 64) gx = 64;
  k_sisdr_pit_bwd<<<dim3(gx, grid_rows(B * S)), 256, 0, (cudaStream_t)stream>>>(est, tgt, perm, fwd_scratch, grad_loss_b, coef, B, S, T,
                                                                                 eps, d_est);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
