// BSS Eval: mir_eval 0.7 `bss_eval_sources` (filter length 512) on the GPU in fp64, behind the reference's utils/bss.py.
//
// Per item: S references r_i (T samples, zero outside [0, T)) and K sets of S estimates.  With L = 512 and N = S L:
//   G[iL+k, jL+l] = c_ij(k-l),  c_ij(m) = sum_u r_i(u) r_j(u+m)       (Gram matrix of the delayed references, block-Toeplitz)
//   D_i[k]        = sum_u r_i(u) e(u+k)                                (one right-hand side per estimate e)
//   P_all e = sum_i sum_k C_i[k] r_i(t-k) with G C = D;  P_j e the same with block (j, j) of G and D_j alone
// and SDR = |P_j e|^2 / |e - P_j e|^2, SIR = |P_j e|^2 / |P_all e - P_j e|^2, SAR = |P_all e|^2 / |e - P_all e|^2 in dB.
//
// Stages (fixed launch sequence, no atomics, every sum in a fixed order: two calls give the same bits):
//   1. correlations: corr(x, y)[m] = sum_u x(u) y(u+m), m < L, for every ordered reference pair (c_ij(-m) = c_ji(m)) and every
//      (reference, estimate) pair, as partial sums over BSS_NCH time chunks, then summed chunk by chunk; G, its S diagonal
//      blocks and the right-hand sides are written from the table.
//   2. blocked right-looking Cholesky (64-wide tiles) of G and of the S blocks, with the inverse of every diagonal tile kept for
//      the solves; a pivot that is not positive and finite marks the matrix.  Then forward and back solves, one CTA per
//      (matrix, right-hand side).
//   3. projection: per output sample, P_all e and every P_j e from the same reference window; the energies are sums of squares
//      of explicit residual samples, never differences of energies (e - P_all e is rounding noise when e is the mixture).
//   4. per item: the S x S tables, the permutation with the largest mean SIR, the gather and the status word.
// The workspace is a function of (B, K, S) alone: the chunk and range counts of stages 1 and 3 are fixed.
#include <math.h>

#include "ctn_internal.h"

#define BSS_L 512
#define BSS_MAX_S 4
#define BSS_NCH 16     // time chunks of the correlation partial sums
#define BSS_TU 1024    // samples per shared-memory tile of the correlation kernel
#define BSS_LD 65      // padded row of a shared tile (conflict-free column reads)
#define BSS_NTT 64     // time ranges of the projection pass per estimate
#define BSS_PT 256     // output samples per projection sub-tile (one per thread)
#define BSS_WIN (BSS_PT + BSS_L - 1)

struct BssDims {
  int B, K, S, T;
  int J;   // correlation jobs per item: S*S reference pairs, then K*S*S (estimate, reference) pairs
  int N;   // S*L
  int KS;  // estimates per item
};

// ---- 1. correlations --------------------------------------------------------------------------------------------------------
// job < S*S: (x, y) = (r_{job/S}, r_{job%S});  else q = job - S*S: (x, y) = (r_{q%S}, e_{q/S}), estimate q/S = k*S + a of the item
__device__ __forceinline__ void bss_job(const BssDims& d, const float* ref, const float* est, int b, int job, const float** x,
                                        const float** y) {
  const size_t T = (size_t)d.T;
  if (job < d.S * d.S) {
    *x = ref + ((size_t)b * d.S + job / d.S) * T;
    *y = ref + ((size_t)b * d.S + job % d.S) * T;
  } else {
    const int q = job - d.S * d.S;
    *x = ref + ((size_t)b * d.S + q % d.S) * T;
    *y = est + ((size_t)b * d.KS + q / d.S) * T;
  }
}

// part[b][job][chunk][m] = sum over the chunk's u of x(u) y(u+m); thread owns lags tid + 128 q (conflict-free window reads)
__global__ void __launch_bounds__(128) k_bss_corr(const float* __restrict__ ref, const float* __restrict__ est, double* __restrict__ part,
                                                  BssDims d) {
  __shared__ double xs[BSS_TU];
  __shared__ double ys[BSS_TU + BSS_L - 1];
  const int c = blockIdx.x % BSS_NCH, job = blockIdx.x / BSS_NCH, b = blockIdx.y;
  const float *x, *y;
  bss_job(d, ref, est, b, job, &x, &y);
  const int TC = (d.T + BSS_NCH - 1) / BSS_NCH;
  const int u_lo = min(d.T, c * TC), u_hi = min(d.T, u_lo + TC);
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int u0 = u_lo; u0 < u_hi; u0 += BSS_TU) {
    const int n = min(BSS_TU, u_hi - u0);
    for (int v = threadIdx.x; v < n; v += 128) xs[v] = (double)x[u0 + v];
    for (int v = threadIdx.x; v < n + BSS_L - 1; v += 128) ys[v] = u0 + v < d.T ? (double)y[u0 + v] : 0.0;
    __syncthreads();
#pragma unroll 4
    for (int u = 0; u < n; ++u) {
      const double xv = xs[u];
      const double* yw = ys + u + threadIdx.x;
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = fma(xv, yw[128 * q], acc[q]);
    }
    __syncthreads();
  }
  double* out = part + (((size_t)b * d.J + job) * BSS_NCH + c) * BSS_L + threadIdx.x;
#pragma unroll
  for (int q = 0; q < 4; ++q) out[128 * q] = acc[q];
}

// chunks summed in order: reference pairs -> corr[b][job][m], estimate pairs -> the right-hand sides of G and of block i
__global__ void __launch_bounds__(BSS_L) k_bss_combine(const double* __restrict__ part, double* __restrict__ corr, double* __restrict__ rhsG,
                                                       double* __restrict__ rhsB, BssDims d) {
  const int job = blockIdx.x, b = blockIdx.y, m = threadIdx.x;
  const double* p = part + ((size_t)b * d.J + job) * BSS_NCH * BSS_L + m;
  double v = 0.0;
  for (int c = 0; c < BSS_NCH; ++c) v += p[(size_t)c * BSS_L];
  if (job < d.S * d.S) {
    corr[((size_t)b * d.S * d.S + job) * BSS_L + m] = v;
  } else {
    const int q = job - d.S * d.S, ka = q / d.S, i = q % d.S;
    rhsG[((size_t)b * d.KS + ka) * d.N + i * BSS_L + m] = v;
    rhsB[(((size_t)b * d.S + i) * d.KS + ka) * BSS_L + m] = v;
  }
}

// G (B, N, N) in full and its diagonal blocks (B S, L, L)
__global__ void __launch_bounds__(256) k_bss_build(const double* __restrict__ corr, double* __restrict__ G, double* __restrict__ Bk, BssDims d) {
  const int b = blockIdx.y;
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  const int row = (int)(idx / d.N), col = (int)(idx % d.N);
  const int i = row / BSS_L, k = row % BSS_L, j = col / BSS_L, l = col % BSS_L;
  const double* cb = corr + (size_t)b * d.S * d.S * BSS_L;
  const double v = k >= l ? cb[(i * d.S + j) * BSS_L + (k - l)] : cb[(j * d.S + i) * BSS_L + (l - k)];
  G[(size_t)b * d.N * d.N + idx] = v;
  if (i == j) Bk[(((size_t)b * d.S + i) * BSS_L + k) * BSS_L + l] = v;
}

// ---- 2. batched Cholesky and solves -------------------------------------------------------------------------------------------
// MatSet (ctn_internal.h): nmat row-major N x N matrices (N a multiple of 64), factor in the lower triangle, W the inverses of
// its diagonal tiles, flag[mat] = 1 when a pivot was not positive and finite.
#define BSS_TILE_SMEM (2 * BSS_NB * BSS_LD * sizeof(double))

__device__ __forceinline__ void bss_load_tile(double (*s)[BSS_LD], const double* g, int ld) {
  for (int e = threadIdx.x; e < BSS_NB * BSS_NB; e += 256) s[e >> 6][e & 63] = g[(size_t)(e >> 6) * ld + (e & 63)];
}

// acc[i][j] = sum_q a[ty + 16 i][q] b[tx + 16 j][q]   (A B^T of two shared tiles, 4 x 4 outputs per thread)
__device__ __forceinline__ void bss_tile_abt(const double (*a)[BSS_LD], const double (*b)[BSS_LD], double acc[4][4]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
#pragma unroll 4
  for (int q = 0; q < BSS_NB; ++q) {
    double av[4], bv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) av[i] = a[ty + 16 * i][q];
#pragma unroll
    for (int j = 0; j < 4; ++j) bv[j] = b[tx + 16 * j][q];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fma(av[i], bv[j], acc[i][j]);
  }
}

// diagonal tile kt: unblocked Cholesky in shared memory, then its triangular inverse (thread c walks column c).  Step j updates
// the trailing triangle from the unscaled column j (a_il -= a_ij a_lj / d_j), then scales column j by 1 / sqrt(d_j): the scaling
// touches only column j, which no later step reads or writes, so one barrier per step suffices.
__global__ void __launch_bounds__(256) k_chol_diag(MatSet s, int kt) {
  extern __shared__ double sm[];
  double (*a)[BSS_LD] = reinterpret_cast<double (*)[BSS_LD]>(sm);
  double (*w)[BSS_LD] = a + BSS_NB;
  const int mat = blockIdx.x, tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
  double* A = s.A + (size_t)mat * s.N * s.N + (size_t)kt * BSS_NB * s.N + kt * BSS_NB;
  bss_load_tile(a, A, s.N);
  for (int e = tid; e < BSS_NB * BSS_NB; e += 256) w[e >> 6][e & 63] = 0.0;
  int bad = 0;
  __syncthreads();
  for (int j = 0; j < BSS_NB; ++j) {
    const double dj = a[j][j];
    const double rd = 1.0 / dj;
    if (tx > j) {
      const double lx = a[tx][j] * rd;
      for (int ii = tx + ty; ii < BSS_NB; ii += 4) a[ii][tx] = fma(-a[ii][j], lx, a[ii][tx]);
    }
    __syncthreads();
    if (tid == 0) bad |= !(dj > 0.0) || !isfinite(dj);
    const double pj = sqrt(dj);
    if (tid >= j && tid < BSS_NB) a[tid][j] = tid == j ? pj : a[tid][j] / pj;
  }
  __syncthreads();
  if (tid < BSS_NB) {
    const int c = tid;
    w[c][c] = 1.0 / a[c][c];
    for (int i = c + 1; i < BSS_NB; ++i) {
      double acc[4] = {0.0, 0.0, 0.0, 0.0};
      int k = c;
      for (; k + 3 < i; k += 4)
#pragma unroll
        for (int u = 0; u < 4; ++u) acc[u] = fma(a[i][k + u], w[k + u][c], acc[u]);
      for (; k < i; ++k) acc[0] = fma(a[i][k], w[k][c], acc[0]);
      w[i][c] = -((acc[0] + acc[1]) + (acc[2] + acc[3])) / a[i][i];
    }
  }
  __syncthreads();
  double* Wt = s.W + ((size_t)mat * s.nt + kt) * BSS_NB * BSS_NB;
  for (int e = tid; e < BSS_NB * BSS_NB; e += 256) {
    const int r = e >> 6, c = e & 63;
    if (c <= r) A[(size_t)r * s.N + c] = a[r][c];
    Wt[e] = w[r][c];
  }
  if (tid == 0) {
    if (kt == 0) s.flag[mat] = bad;
    else if (bad) s.flag[mat] = 1;
  }
}

// panel: L[it][kt] = A[it][kt] W_kt^T for every tile row it > kt
__global__ void __launch_bounds__(256) k_chol_panel(MatSet s, int kt) {
  extern __shared__ double sm[];
  double (*a)[BSS_LD] = reinterpret_cast<double (*)[BSS_LD]>(sm);
  double (*w)[BSS_LD] = a + BSS_NB;
  const int it = kt + 1 + blockIdx.x, mat = blockIdx.y;
  double* A = s.A + (size_t)mat * s.N * s.N + (size_t)it * BSS_NB * s.N + kt * BSS_NB;
  bss_load_tile(a, A, s.N);
  bss_load_tile(w, s.W + ((size_t)mat * s.nt + kt) * BSS_NB * BSS_NB, BSS_NB);
  __syncthreads();
  double acc[4][4];
  bss_tile_abt(a, w, acc);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) A[(size_t)(ty + 16 * i) * s.N + tx + 16 * j] = acc[i][j];
}

// trailing update: A[it][jt] -= L[it][kt] L[jt][kt]^T for kt < jt <= it (tile pair p of the lower triangle)
__global__ void __launch_bounds__(256) k_chol_update(MatSet s, int kt) {
  extern __shared__ double sm[];
  double (*a)[BSS_LD] = reinterpret_cast<double (*)[BSS_LD]>(sm);
  double (*b)[BSS_LD] = a + BSS_NB;
  const int p = blockIdx.x, mat = blockIdx.y;
  int i = (int)((sqrt(8.0 * p + 1.0) - 1.0) * 0.5);
  while ((i + 1) * (i + 2) / 2 <= p) ++i;
  while (i * (i + 1) / 2 > p) --i;
  const int it = kt + 1 + i, jt = kt + 1 + (p - i * (i + 1) / 2);
  const double* M = s.A + (size_t)mat * s.N * s.N;
  bss_load_tile(a, M + (size_t)it * BSS_NB * s.N + kt * BSS_NB, s.N);
  bss_load_tile(b, M + (size_t)jt * BSS_NB * s.N + kt * BSS_NB, s.N);
  __syncthreads();
  double acc[4][4];
  bss_tile_abt(a, b, acc);
  double* C = s.A + (size_t)mat * s.N * s.N + (size_t)it * BSS_NB * s.N + jt * BSS_NB;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      double* g = C + (size_t)(ty + 16 * r) * s.N + tx + 16 * c;
      *g -= acc[r][c];
    }
}

// G x = b in place for right-hand side blockIdx.x of matrix blockIdx.y: L y = b tile by tile, then L^T x = y.  Row sums over a
// warp's lanes then shuffles, column sums over four row slices added in order.
__global__ void __launch_bounds__(256) k_chol_solve(MatSet s, double* __restrict__ rhs, int nrhs) {
  extern __shared__ double y[];
  __shared__ double r[BSS_NB];
  __shared__ double red[4][BSS_NB];
  const int mat = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double* A = s.A + (size_t)mat * s.N * s.N;
  const double* W = s.W + (size_t)mat * s.nt * BSS_NB * BSS_NB;
  double* v = rhs + ((size_t)mat * nrhs + blockIdx.x) * s.N;
  for (int e = tid; e < s.N; e += 256) y[e] = v[e];
  __syncthreads();
  for (int kt = 0; kt < s.nt; ++kt) {
    const int R0 = kt * BSS_NB;
    for (int rr = warp; rr < BSS_NB; rr += 8) {
      const double* Lr = A + (size_t)(R0 + rr) * s.N;
      double acc = 0.0;
      for (int p = lane; p < R0; p += 32) acc = fma(Lr[p], y[p], acc);
      acc = warp_sum_d(acc);
      if (lane == 0) r[rr] = y[R0 + rr] - acc;
    }
    __syncthreads();
    for (int rr = warp; rr < BSS_NB; rr += 8) {
      const double* Wr = W + ((size_t)kt * BSS_NB + rr) * BSS_NB;
      const double acc = warp_sum_d(fma(Wr[lane], r[lane], Wr[lane + 32] * r[lane + 32]));
      if (lane == 0) y[R0 + rr] = acc;
    }
    __syncthreads();
  }
  for (int kt = s.nt - 1; kt >= 0; --kt) {
    const int R0 = kt * BSS_NB, c = tid & 63, sl = tid >> 6;
    double acc = 0.0;
    for (int p = R0 + BSS_NB + sl; p < s.N; p += 4) acc = fma(A[(size_t)p * s.N + R0 + c], y[p], acc);
    red[sl][c] = acc;
    __syncthreads();
    if (tid < BSS_NB) r[tid] = y[R0 + tid] - (((red[0][tid] + red[1][tid]) + red[2][tid]) + red[3][tid]);
    __syncthreads();
    const double* Wk = W + (size_t)kt * BSS_NB * BSS_NB;
    acc = 0.0;
    for (int row = sl; row < BSS_NB; row += 4) acc = fma(Wk[row * BSS_NB + c], r[row], acc);
    red[sl][c] = acc;
    __syncthreads();
    if (tid < BSS_NB) y[R0 + tid] = ((red[0][tid] + red[1][tid]) + red[2][tid]) + red[3][tid];
    __syncthreads();
  }
  for (int e = tid; e < s.N; e += 256) v[e] = y[e];
}

int ctn_chol_factor(const MatSet& s, cudaStream_t st) {
  for (auto k : {(const void*)k_chol_diag, (const void*)k_chol_panel, (const void*)k_chol_update}) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BSS_TILE_SMEM);
    if (e != cudaSuccess) return (int)e;
  }
  for (int kt = 0; kt < s.nt; ++kt) {
    k_chol_diag<<<s.nmat, 256, BSS_TILE_SMEM, st>>>(s, kt);
    CTN_COUNT_LAUNCH();
    const int n = s.nt - 1 - kt;
    if (n == 0) break;
    k_chol_panel<<<dim3(n, s.nmat), 256, BSS_TILE_SMEM, st>>>(s, kt);
    CTN_COUNT_LAUNCH();
    k_chol_update<<<dim3(n * (n + 1) / 2, s.nmat), 256, BSS_TILE_SMEM, st>>>(s, kt);
    CTN_COUNT_LAUNCH();
  }
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int ctn_chol_solve_cols(const MatSet& s, double* rhs, int nrhs, cudaStream_t st) {
  k_chol_solve<<<dim3(nrhs, s.nmat), 256, sizeof(double) * s.N, st>>>(s, rhs, nrhs);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- 3. projection and energies ---------------------------------------------------------------------------------------------
// Energies of one estimate e, in this order: |P_all e|^2, |e - P_all e|^2, |e|^2, then per reference j:
// |P_j e|^2, |e - P_j e|^2, |P_all e - P_j e|^2.
#define BSS_NQ(S) (3 + 3 * (S))

template <int S>
__global__ void __launch_bounds__(256) k_bss_project(const float* __restrict__ ref, const float* __restrict__ est,
                                                     const double* __restrict__ rhsG, const double* __restrict__ rhsB,
                                                     double* __restrict__ epart, BssDims d) {
  constexpr int NQ = BSS_NQ(S);
  extern __shared__ double sm[];
  double2* cp = reinterpret_cast<double2*>(sm);  // [S][L]: (coefficient in P_all, coefficient in P_i)
  double* rw = sm + 2 * S * BSS_L;                // [S][WIN]: r_i(t0 - (L-1) + v)
  __shared__ double red[8][NQ];
  const int e = blockIdx.y, b = e / d.KS, ka = e % d.KS, tid = threadIdx.x;
  for (int idx = tid; idx < S * BSS_L; idx += 256) {
    const int i = idx / BSS_L, m = idx % BSS_L;
    cp[idx] = make_double2(rhsG[((size_t)b * d.KS + ka) * d.N + idx], rhsB[(((size_t)b * S + i) * d.KS + ka) * BSS_L + m]);
  }
  const size_t T = (size_t)d.T;
  const float* R = ref + (size_t)b * S * T;
  const float* E = est + (size_t)e * T;
  const int Tt = d.T + BSS_L - 1, span = (Tt + BSS_NTT - 1) / BSS_NTT;
  const int t_lo = min(Tt, (int)blockIdx.x * span), t_hi = min(Tt, t_lo + span);
  double en[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) en[q] = 0.0;
  for (int t0 = t_lo; t0 < t_hi; t0 += BSS_PT) {
    __syncthreads();
    for (int idx = tid; idx < S * BSS_WIN; idx += 256) {
      const int i = idx / BSS_WIN, g = t0 - (BSS_L - 1) + idx % BSS_WIN;
      rw[idx] = (g >= 0 && g < d.T) ? (double)R[(size_t)i * T + g] : 0.0;
    }
    __syncthreads();
    const int t = t0 + tid;
    if (t < t_hi) {
      double pa = 0.0, pj[S];
#pragma unroll
      for (int i = 0; i < S; ++i) {
        pj[i] = 0.0;
        const double* rwi = rw + i * BSS_WIN + tid + BSS_L - 1;
        const double2* ci = cp + i * BSS_L;
#pragma unroll 8
        for (int m = 0; m < BSS_L; ++m) {
          const double rv = rwi[-m];
          const double2 c = ci[m];
          pa = fma(c.x, rv, pa);
          pj[i] = fma(c.y, rv, pj[i]);
        }
      }
      const double ev = t < d.T ? (double)E[t] : 0.0, ra = ev - pa;
      en[0] = fma(pa, pa, en[0]);
      en[1] = fma(ra, ra, en[1]);
      en[2] = fma(ev, ev, en[2]);
#pragma unroll
      for (int j = 0; j < S; ++j) {
        const double dj = ev - pj[j], ij = pa - pj[j];
        en[3 + 3 * j] = fma(pj[j], pj[j], en[3 + 3 * j]);
        en[4 + 3 * j] = fma(dj, dj, en[4 + 3 * j]);
        en[5 + 3 * j] = fma(ij, ij, en[5 + 3 * j]);
      }
    }
  }
  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const double v = warp_sum_d(en[q]);
    if (lane == 0) red[warp][q] = v;
  }
  __syncthreads();
  if (tid < NQ) {
    double v = 0.0;
    for (int w = 0; w < 8; ++w) v += red[w][tid];
    epart[((size_t)e * BSS_NTT + blockIdx.x) * NQ + tid] = v;
  }
}

template <int S>
static int launch_project(const float* ref, const float* est, const double* rhsG, const double* rhsB, double* epart, const BssDims& d,
                          cudaStream_t st) {
  const size_t smem = sizeof(double) * (2 * S * BSS_L + S * BSS_WIN);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(k_bss_project<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  k_bss_project<S><<<dim3(BSS_NTT, d.B * d.KS), 256, smem, st>>>(ref, est, rhsG, rhsB, epart, d);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- 4. tables, permutation, status -----------------------------------------------------------------------------------------
__device__ __forceinline__ double bss_safe_db(double num, double den) { return den == 0.0 ? (double)INFINITY : 10.0 * log10(num / den); }

// one CTA per item.  The permutation maximises mean_j SIR[pi(j)][j] over itertools.permutations order, first maximum kept, a NaN
// mean counting as the maximum (numpy argmax); the mean is summed as numpy's add.reduce does (x0 + (x1 + x2 + ...)), then / S.
__global__ void __launch_bounds__(64) k_bss_select(const double* __restrict__ epart, const double* __restrict__ corr, const int* __restrict__ flagG,
                                                   const int* __restrict__ flagB, BssDims d, int compute_permutation, double* __restrict__ sdr,
                                                   double* __restrict__ sir, double* __restrict__ sar, int32_t* __restrict__ perm,
                                                   int32_t* __restrict__ status) {
  __shared__ double q[BSS_MAX_S * BSS_NQ(BSS_MAX_S)];
  const int b = blockIdx.x, tid = threadIdx.x, S = d.S, NQ = BSS_NQ(d.S);
  int st = 0;
  for (int k = 0; k < d.K; ++k) {
    __syncthreads();
    if (tid < S * NQ) {
      const int a = tid / NQ, qq = tid % NQ;
      const double* p = epart + ((size_t)(b * d.KS + k * S + a) * BSS_NTT) * NQ + qq;
      double v = 0.0;
      for (int t = 0; t < BSS_NTT; ++t) v += p[(size_t)t * NQ];
      q[tid] = v;
    }
    __syncthreads();
    if (tid == 0) {
      double SDR[BSS_MAX_S][BSS_MAX_S], SIR[BSS_MAX_S][BSS_MAX_S], SAR[BSS_MAX_S];
      for (int a = 0; a < S; ++a) {
        const double* qa = q + a * NQ;
        if (qa[2] == 0.0) st |= CTN_BSS_SILENT_EST;
        SAR[a] = bss_safe_db(qa[0], qa[1]);
        for (int j = 0; j < S; ++j) {
          SDR[a][j] = bss_safe_db(qa[3 + 3 * j], qa[4 + 3 * j]);
          SIR[a][j] = bss_safe_db(qa[3 + 3 * j], qa[5 + 3 * j]);
        }
      }
      int pi[BSS_MAX_S], best[BSS_MAX_S];
      for (int j = 0; j < S; ++j) pi[j] = best[j] = j;
      if (compute_permutation) {
        double best_v = 0.0;
        bool first = true;
        for (;;) {
          double rest = 0.0;
          for (int j = 1; j < S; ++j) rest += SIR[pi[j]][j];
          const double v = (SIR[pi[0]][0] + rest) / S;
          if (first || (!isnan(best_v) && (isnan(v) || v > best_v))) {
            best_v = v;
            for (int j = 0; j < S; ++j) best[j] = pi[j];
          }
          first = false;
          // next permutation in lexicographic (itertools) order
          int i = S - 2;
          while (i >= 0 && pi[i] > pi[i + 1]) --i;
          if (i < 0) break;
          int j = S - 1;
          while (pi[j] < pi[i]) --j;
          int tmp = pi[i]; pi[i] = pi[j]; pi[j] = tmp;
          for (int lo = i + 1, hi = S - 1; lo < hi; ++lo, --hi) { tmp = pi[lo]; pi[lo] = pi[hi]; pi[hi] = tmp; }
        }
      }
      for (int j = 0; j < S; ++j) {
        const size_t o = (size_t)(b * d.K + k) * S + j;
        sdr[o] = SDR[best[j]][j];
        sir[o] = SIR[best[j]][j];
        sar[o] = SAR[best[j]];
        perm[o] = best[j];
      }
    }
  }
  if (tid == 0) {
    for (int i = 0; i < S; ++i) {
      if (corr[((size_t)b * S * S + i * S + i) * BSS_L] == 0.0) st |= CTN_BSS_SILENT_REF;
      if (flagB[b * S + i]) st |= CTN_BSS_NOT_PD;
    }
    if (flagG[b]) st |= CTN_BSS_NOT_PD;
    status[b] = st;
  }
}

// ---- host -------------------------------------------------------------------------------------------------------------------
struct BssWs {
  double *part, *corr, *G, *Wg, *Bk, *Wb, *rhsG, *rhsB, *epart;
  int *flagG, *flagB;
};

static void carve_bss(Carver& cv, const BssDims& d, BssWs* w) {
  const size_t B = d.B, S = d.S, N = d.N, L = BSS_L;
  w->part = cv.take<double>(B * d.J * BSS_NCH * L);
  w->corr = cv.take<double>(B * S * S * L);
  w->G = cv.take<double>(B * N * N);
  w->Wg = cv.take<double>(B * N * BSS_NB);
  w->Bk = cv.take<double>(B * S * L * L);
  w->Wb = cv.take<double>(B * S * L * BSS_NB);
  w->rhsG = cv.take<double>(B * d.KS * N);
  w->rhsB = cv.take<double>(B * S * d.KS * L);
  w->epart = cv.take<double>(B * d.KS * BSS_NTT * BSS_NQ(S));
  w->flagG = cv.take<int>(B);
  w->flagB = cv.take<int>(B * S);
}

static int bss_dims(int B, int K, int S, int T, BssDims* d) {
  if (B < 1 || K < 1 || S < 1 || T < 1) return CTN_EINVAL;
  if (S > BSS_MAX_S) return CTN_EUNSUPPORTED;
  if ((long long)B * K * S > 65535) return CTN_EUNSUPPORTED;  // estimates ride on gridDim.y
  d->B = B; d->K = K; d->S = S; d->T = T;
  d->KS = K * S;
  d->J = S * S + K * S * S;
  d->N = S * BSS_L;
  return CTN_OK;
}

extern "C" int ctn_bss_workspace_bytes(int B, int K, int S, int T, size_t* bytes) {
  BssDims d;
  CTN_TRY(bss_dims(B, K, S, T, &d));
  if (!bytes) return CTN_EINVAL;
  Carver cv(nullptr);
  BssWs w;
  carve_bss(cv, d, &w);
  *bytes = cv.off + 256;
  return CTN_OK;
}

extern "C" int ctn_bss_eval_sources(const float* ref, const float* est, int B, int K, int S, int T, int compute_permutation, double* sdr,
                                    double* sir, double* sar, int32_t* perm, int32_t* status, void* ws, size_t ws_bytes,
                                    ctn_stream_t stream) {
  LaunchScope scope(ref);
  if (!ref || !est || !sdr || !sir || !sar || !perm || !status || !ws) return CTN_EINVAL;
  BssDims d;
  CTN_TRY(bss_dims(B, K, S, T, &d));
  if (((uintptr_t)ws) & 255) return CTN_EALIGN;
  size_t need = 0;
  CTN_TRY(ctn_bss_workspace_bytes(B, K, S, T, &need));
  if (ws_bytes < need) return CTN_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  Carver cv(ws);
  BssWs w;
  carve_bss(cv, d, &w);

  k_bss_corr<<<dim3(BSS_NCH * d.J, B), 128, 0, st>>>(ref, est, w.part, d);
  CTN_COUNT_LAUNCH();
  k_bss_combine<<<dim3(d.J, B), BSS_L, 0, st>>>(w.part, w.corr, w.rhsG, w.rhsB, d);
  CTN_COUNT_LAUNCH();
  k_bss_build<<<dim3((unsigned)((size_t)d.N * d.N / 256), B), 256, 0, st>>>(w.corr, w.G, w.Bk, d);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();

  const MatSet g{w.G, w.Wg, w.flagG, d.N, d.N / BSS_NB, B};
  const MatSet blk{w.Bk, w.Wb, w.flagB, BSS_L, BSS_L / BSS_NB, B * S};
  CTN_TRY(ctn_chol_factor(g, st));
  CTN_TRY(ctn_chol_factor(blk, st));
  CTN_TRY(ctn_chol_solve_cols(g, w.rhsG, d.KS, st));
  CTN_TRY(ctn_chol_solve_cols(blk, w.rhsB, d.KS, st));

  switch (S) {
    case 1: CTN_TRY(launch_project<1>(ref, est, w.rhsG, w.rhsB, w.epart, d, st)); break;
    case 2: CTN_TRY(launch_project<2>(ref, est, w.rhsG, w.rhsB, w.epart, d, st)); break;
    case 3: CTN_TRY(launch_project<3>(ref, est, w.rhsG, w.rhsB, w.epart, d, st)); break;
    default: CTN_TRY(launch_project<4>(ref, est, w.rhsG, w.rhsB, w.epart, d, st)); break;
  }
  k_bss_select<<<B, 64, 0, st>>>(w.epart, w.corr, w.flagG, w.flagB, d, compute_permutation, sdr, sir, sar, perm, status);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
