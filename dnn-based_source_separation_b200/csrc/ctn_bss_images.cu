// BSS Eval v4 of multichannel source images (museval 0.4 `evaluate(..., mode='v4')`) on the GPU in fp64.  DESIGN §10.
//
// J sources, I channels, T samples; reference rows m = (j, c), M = J I <= 8; distortion filters of L = 512 taps over all rows:
//   G[(m,k),(m',l)] = sum_u r_m(u-k) r_m'(u-l)          (block-Toeplitz, N = M L)
//   D[(m,k), (j,c)] = sum_u r_m(u) e_{j,c}(u+k)
//   (G + eps I) C = D over the whole track;  (G_jj + eps I) Ct_j = the rows of D of source j's own channels
// Per window w (win samples from w hop, every signal zero outside it), for t over win + L - 1 samples and every channel c:
//   P_all(t,c) = sum_{m,k} C[(m,k),(j,c)] r_m^w(t-k),  P_j(t,c) = sum_{c',k} Ct_j[(c',k),c] r_{j,c'}^w(t-k)
// and SDR / ISR / SIR / SAR of (source, window) from seven energies of explicit residuals summed over channels and samples.
//
// Stages (fixed launch sequence, no atomics, every sum in a fixed order: two calls give the same bits, a call can be captured):
//   1. k_mus_silent: per (window, source), whether the channel sum is zero over the window (references and estimates).
//   2. k_mus_corr<M>: corr(x = r_m, y)[k] = sum_u x(u) y(u+k), k < L, for every reference row m against every y row (the M
//      reference rows, then the M estimate rows), as partial sums over MUS_NCH time chunks; one CTA holds all M x rows, so each
//      y sample it loads feeds M rows.  k_mus_combine sums the chunks in order and writes the right-hand sides.
//   3. k_mus_build writes G + eps I and its J diagonal blocks; the tiled Cholesky of ctn_bss.cu factors them, and
//      k_mus_fwd_step / k_mus_bwd_step solve all right-hand sides of a matrix together (ctn_chol_solve_multi).
//   4. k_mus_project<M, I>: per (window, range of 512-sample output tiles), one shared-memory window of reference row m at a time
//      feeds P_all of all M columns and P_j of the I columns of m's source; the energies are accumulated per source.
//      k_mus_finish sums the ranges in order, forms the dB values and applies the +inf / NaN rules and the status word.
// The workspace is a function of (J, I) and nwin: the chunk counts of stage 2 are fixed, and stage 4 keeps at most MUS_MAXR
// partial energy sets per window.
#include <math.h>

#include "ctn_internal.h"

#define MUS_L 512
#define MUS_MAXM 8
#define MUS_NCH 128    // time chunks of the correlation partial sums
#define MUS_TU 512     // samples per shared-memory tile of the correlation kernel
#define MUS_PQ 4       // output samples per thread in the projection
#define MUS_PT (128 * MUS_PQ)
#define MUS_MAXR 64    // most partial energy sets per window
#define MUS_NE 7       // energies per (source, window)

struct MusDims {
  int J, I, M, T, win, hop, nwin;
  int N;      // M L
  int ntile;  // output tiles of MUS_PT samples per window, over win + L - 1 samples
  int per;    // tiles per range
  int R;      // ranges per window
};

// ---- 1. silence -------------------------------------------------------------------------------------------------------------
// silent[w][which] bit j: the channel sum of source j is zero at every sample of window w (which 0: references, 1: estimates)
__global__ void __launch_bounds__(256) k_mus_silent(const float* __restrict__ ref, const float* __restrict__ est, int* __restrict__ silent,
                                                    MusDims d) {
  const int w = blockIdx.x, which = blockIdx.y;
  const float* x = which ? est : ref;
  const size_t T = (size_t)d.T, s0 = (size_t)w * d.hop;
  int bits = 0;
  for (int j = 0; j < d.J; ++j) {
    int nz = 0;
    for (int t = threadIdx.x; t < d.win && !nz; t += 256) {
      double s = 0.0;
      for (int c = 0; c < d.I; ++c) s += (double)x[(size_t)(j * d.I + c) * T + s0 + t];
      nz = s != 0.0;
    }
    if (!__syncthreads_or(nz)) bits |= 1 << j;
  }
  if (threadIdx.x == 0) silent[w * 2 + which] = bits;
}

// ---- 2. correlations --------------------------------------------------------------------------------------------------------
// part[y][chunk][m][k] = sum over the chunk's u of r_m(u) y(u+k); y < M: reference row y, else estimate row y - M.  Thread owns
// lags tid + 128 q (conflict-free reads of the y window); the M x values of a sample are one broadcast row.
template <int M>
__global__ void __launch_bounds__(128) k_mus_corr(const float* __restrict__ ref, const float* __restrict__ est, double* __restrict__ part,
                                                  MusDims d) {
  constexpr int MP = (M + 1) & ~1;
  __shared__ __align__(16) double xs[MUS_TU * MP];
  __shared__ double ys[MUS_TU + MUS_L - 1];
  const int c = blockIdx.x, yr = blockIdx.y, tid = threadIdx.x;
  const size_t T = (size_t)d.T;
  const float* y = yr < M ? ref + (size_t)yr * T : est + (size_t)(yr - M) * T;
  const int TC = (d.T + MUS_NCH - 1) / MUS_NCH;
  const int u_lo = min(d.T, c * TC), u_hi = min(d.T, u_lo + TC);
  double acc[M][4];
#pragma unroll
  for (int m = 0; m < M; ++m)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[m][q] = 0.0;
  for (int u0 = u_lo; u0 < u_hi; u0 += MUS_TU) {
    const int n = min(MUS_TU, u_hi - u0);
    for (int v = tid; v < n * MP; v += 128) {
      const int u = v / MP, m = v % MP;
      xs[v] = m < M ? (double)ref[(size_t)m * T + u0 + u] : 0.0;
    }
    for (int v = tid; v < n + MUS_L - 1; v += 128) ys[v] = u0 + v < d.T ? (double)y[u0 + v] : 0.0;
    __syncthreads();
#pragma unroll 2
    for (int u = 0; u < n; ++u) {
      double xv[MP];
#pragma unroll
      for (int m = 0; m < MP; m += 2) {
        const double2 p = *reinterpret_cast<const double2*>(xs + u * MP + m);
        xv[m] = p.x;
        xv[m + 1] = p.y;
      }
      double yv[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) yv[q] = ys[u + tid + 128 * q];
#pragma unroll
      for (int m = 0; m < M; ++m)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[m][q] = fma(xv[m], yv[q], acc[m][q]);
    }
    __syncthreads();
  }
  double* out = part + (((size_t)yr * MUS_NCH + c) * M) * MUS_L + tid;
#pragma unroll
  for (int m = 0; m < M; ++m)
#pragma unroll
    for (int q = 0; q < 4; ++q) out[(size_t)m * MUS_L + 128 * q] = acc[m][q];
}

// chunks summed in order -> corr[y][m][k] (y < M), or the right-hand sides: rhsG[(m,k)][col] and, when col belongs to m's
// source j, rhsB[j][(c',k)][c] = rhsB[(m,k)][c]
__global__ void __launch_bounds__(MUS_L) k_mus_combine(const double* __restrict__ part, double* __restrict__ corr, double* __restrict__ rhsG,
                                                      double* __restrict__ rhsB, MusDims d) {
  const int m = blockIdx.x, yr = blockIdx.y, k = threadIdx.x;
  const double* p = part + ((size_t)yr * MUS_NCH * d.M + m) * MUS_L + k;
  double v = 0.0;
  for (int c = 0; c < MUS_NCH; ++c) v += p[(size_t)c * d.M * MUS_L];
  if (yr < d.M) {
    corr[((size_t)yr * d.M + m) * MUS_L + k] = v;
  } else {
    const int col = yr - d.M;
    rhsG[((size_t)m * MUS_L + k) * d.M + col] = v;
    if (col / d.I == m / d.I) rhsB[((size_t)m * MUS_L + k) * d.I + col % d.I] = v;
  }
}

// G + eps I (N x N) in full and its J diagonal blocks (I L x I L).  corr[y][m][k] = sum_u r_m(u) r_y(u+k), so
// G[(m,k),(m',l)] = corr[m'][m][k-l] for k >= l and corr[m][m'][l-k] otherwise.
__global__ void __launch_bounds__(256) k_mus_build(const double* __restrict__ corr, double* __restrict__ G, double* __restrict__ Bk, MusDims d) {
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (size_t)d.N * d.N) return;
  const int row = (int)(idx / d.N), col = (int)(idx % d.N);
  const int m = row / MUS_L, k = row % MUS_L, m2 = col / MUS_L, l = col % MUS_L;
  double v = k >= l ? corr[((size_t)m2 * d.M + m) * MUS_L + (k - l)] : corr[((size_t)m * d.M + m2) * MUS_L + (l - k)];
  if (row == col) v += 0x1p-52;  // museval: np.finfo(float).eps on the diagonal
  G[idx] = v;
  const int j = m / d.I;
  if (m2 / d.I == j) {
    const int NB = d.I * MUS_L, r = (m % d.I) * MUS_L + k, cc = (m2 % d.I) * MUS_L + l;
    Bk[((size_t)j * NB + r) * NB + cc] = v;
  }
}

// ---- 3. solves with all right-hand sides of a matrix together -----------------------------------------------------------------
// Forward sweep, step kt, CTA b of matrix blockIdx.y: y_kt = W_kt b_kt (b_kt final after steps < kt); CTA 0 stores y_kt, CTA b > 0
// updates b_it -= L[it][kt] y_kt for it = kt + b.  Thread (r = tid / 4, q = tid % 4 and + 4) owns two of the 64 x 8 outputs.
#define MUS_SLD 65
__device__ __forceinline__ void mus_load_tile(double (*s)[MUS_SLD], const double* g, int ld) {
  for (int e = threadIdx.x; e < BSS_NB * BSS_NB; e += 256) s[e >> 6][e & 63] = g[(size_t)(e >> 6) * ld + (e & 63)];
}

__global__ void __launch_bounds__(256) k_mus_fwd_step(MatSet s, double* __restrict__ rhs, double* __restrict__ sol, int nrhs, int kt) {
  __shared__ double a[BSS_NB][MUS_SLD];
  __shared__ double bk[BSS_NB][8], yk[BSS_NB][8];
  const int mat = blockIdx.y, b = blockIdx.x, tid = threadIdx.x, r = tid >> 2, q0 = tid & 3;
  const size_t mo = (size_t)mat * s.N * nrhs;
  mus_load_tile(a, s.W + ((size_t)mat * s.nt + kt) * BSS_NB * BSS_NB, BSS_NB);
  for (int e = tid; e < BSS_NB * 8; e += 256) {
    const int rr = e >> 3, q = e & 7;
    bk[rr][q] = q < nrhs ? rhs[mo + (size_t)(kt * BSS_NB + rr) * nrhs + q] : 0.0;
  }
  __syncthreads();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + 4 * h;
    double acc = 0.0;
    for (int p = 0; p <= r; ++p) acc = fma(a[r][p], bk[p][q], acc);
    yk[r][q] = acc;
  }
  __syncthreads();
  if (b == 0) {
    for (int e = tid; e < BSS_NB * nrhs; e += 256) {
      const int rr = e / nrhs, q = e % nrhs;
      sol[mo + (size_t)(kt * BSS_NB + rr) * nrhs + q] = yk[rr][q];
    }
    return;
  }
  const int it = kt + b;
  mus_load_tile(a, s.A + (size_t)mat * s.N * s.N + (size_t)it * BSS_NB * s.N + kt * BSS_NB, s.N);
  __syncthreads();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + 4 * h;
    if (q >= nrhs) continue;
    double acc = 0.0;
    for (int p = 0; p < BSS_NB; ++p) acc = fma(a[r][p], yk[p][q], acc);
    double* g = rhs + mo + (size_t)(it * BSS_NB + r) * nrhs + q;
    *g -= acc;
  }
}

// Back sweep, step kt (descending): x_kt = W_kt^T y_kt (y_kt final after steps > kt); CTA 0 stores x_kt into rhs, CTA b > 0
// updates y_jt -= L[kt][jt]^T x_kt for jt = b - 1.
__global__ void __launch_bounds__(256) k_mus_bwd_step(MatSet s, double* __restrict__ rhs, double* __restrict__ sol, int nrhs, int kt) {
  __shared__ double a[BSS_NB][MUS_SLD];
  __shared__ double yv[BSS_NB][8], xk[BSS_NB][8];
  const int mat = blockIdx.y, b = blockIdx.x, tid = threadIdx.x, r = tid >> 2, q0 = tid & 3;
  const size_t mo = (size_t)mat * s.N * nrhs;
  mus_load_tile(a, s.W + ((size_t)mat * s.nt + kt) * BSS_NB * BSS_NB, BSS_NB);
  for (int e = tid; e < BSS_NB * 8; e += 256) {
    const int rr = e >> 3, q = e & 7;
    yv[rr][q] = q < nrhs ? sol[mo + (size_t)(kt * BSS_NB + rr) * nrhs + q] : 0.0;
  }
  __syncthreads();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + 4 * h;
    double acc = 0.0;
    for (int p = r; p < BSS_NB; ++p) acc = fma(a[p][r], yv[p][q], acc);
    xk[r][q] = acc;
  }
  __syncthreads();
  if (b == 0) {
    for (int e = tid; e < BSS_NB * nrhs; e += 256) {
      const int rr = e / nrhs, q = e % nrhs;
      rhs[mo + (size_t)(kt * BSS_NB + rr) * nrhs + q] = xk[rr][q];
    }
    return;
  }
  const int jt = b - 1;
  mus_load_tile(a, s.A + (size_t)mat * s.N * s.N + (size_t)kt * BSS_NB * s.N + jt * BSS_NB, s.N);
  __syncthreads();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + 4 * h;
    if (q >= nrhs) continue;
    double acc = 0.0;
    for (int p = 0; p < BSS_NB; ++p) acc = fma(a[p][r], xk[p][q], acc);
    double* g = sol + mo + (size_t)(jt * BSS_NB + r) * nrhs + q;
    *g -= acc;
  }
}

int ctn_chol_solve_multi(const MatSet& s, double* rhs, double* tmp, int nrhs, cudaStream_t st) {
  if (nrhs < 1 || nrhs > 8) return CTN_EUNSUPPORTED;
  for (int kt = 0; kt < s.nt; ++kt) {
    k_mus_fwd_step<<<dim3(s.nt - kt, s.nmat), 256, 0, st>>>(s, rhs, tmp, nrhs, kt);
    CTN_COUNT_LAUNCH();
  }
  for (int kt = s.nt - 1; kt >= 0; --kt) {
    k_mus_bwd_step<<<dim3(kt + 1, s.nmat), 256, 0, st>>>(s, rhs, tmp, nrhs, kt);
    CTN_COUNT_LAUNCH();
  }
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- 4. projection and energies ---------------------------------------------------------------------------------------------
// Energies of (source j, window), summed over its channels and the window's win + L - 1 output samples, in this order:
// |s|^2, |e - s|^2, |P_j - s|^2, |P_j|^2, |P_all - P_j|^2, |P_all|^2, |e - P_all|^2   (s = r_{j,c}^w, e = e_{j,c}^w)
// C: rhsG solved, [(m,k)][col]; Ct: rhsB solved, [(m,k)][c].  Shared: cs[k][NCP] = (C[(m,k)][0..M), Ct[(m,k)][0..I), pad),
// rw[v] = r_m^w(t0 - (L-1) + v).
template <int M, int I>
__global__ void __launch_bounds__(128) k_mus_project(const float* __restrict__ ref, const float* __restrict__ est, const double* __restrict__ C,
                                                     const double* __restrict__ Ct, double* __restrict__ epart, MusDims d) {
  constexpr int J = M / I, NC = M + I, NCP = (NC + 1) & ~1;
  extern __shared__ __align__(16) double sm[];
  double* cs = sm;
  double* rw = sm + MUS_L * NCP;
  double* en = rw + MUS_PT + MUS_L - 1;  // [J * MUS_NE][128]: this thread's energies, kept out of registers
  const int w = blockIdx.x / d.R, rg = blockIdx.x % d.R, tid = threadIdx.x;
  const size_t T = (size_t)d.T, s0 = (size_t)w * d.hop;
  const int span = d.win + MUS_L - 1;
  const int tile_lo = rg * d.per, tile_hi = min(d.ntile, tile_lo + d.per);
  for (int e = 0; e < J * MUS_NE; ++e) en[e * 128 + tid] = 0.0;
  for (int tile = tile_lo; tile < tile_hi; ++tile) {
    const int t0 = tile * MUS_PT;
    double pa[MUS_PQ][M], pj[MUS_PQ][M];
#pragma unroll
    for (int q = 0; q < MUS_PQ; ++q)
#pragma unroll
      for (int col = 0; col < M; ++col) pa[q][col] = pj[q][col] = 0.0;
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const int jm = m / I;
      __syncthreads();
      for (int e = tid; e < MUS_L * NCP; e += 128) {
        const int k = e / NCP, q = e % NCP;
        const size_t row = (size_t)m * MUS_L + k;
        cs[e] = q < M ? C[row * M + q] : q < NC ? Ct[row * I + (q - M)] : 0.0;
      }
      for (int v = tid; v < MUS_PT + MUS_L - 1; v += 128) {
        const int tt = t0 - (MUS_L - 1) + v;
        rw[v] = (tt >= 0 && tt < d.win) ? (double)ref[(size_t)m * T + s0 + tt] : 0.0;
      }
      __syncthreads();
#pragma unroll 2
      for (int k = 0; k < MUS_L; ++k) {
        double cv[NCP];
#pragma unroll
        for (int q = 0; q < NCP; q += 2) {
          const double2 p = *reinterpret_cast<const double2*>(cs + k * NCP + q);
          cv[q] = p.x;
          cv[q + 1] = p.y;
        }
#pragma unroll
        for (int q = 0; q < MUS_PQ; ++q) {
          const double rv = rw[tid + 128 * q + MUS_L - 1 - k];
#pragma unroll
          for (int col = 0; col < M; ++col) pa[q][col] = fma(cv[col], rv, pa[q][col]);
#pragma unroll
          for (int c = 0; c < I; ++c) pj[q][jm * I + c] = fma(cv[M + c], rv, pj[q][jm * I + c]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < MUS_PQ; ++q) {
      const int t = t0 + tid + 128 * q;
      if (t >= span) continue;
#pragma unroll
      for (int col = 0; col < M; ++col) {
        const int j = col / I;
        const size_t g = (size_t)col * T + s0 + t;
        const double sv = t < d.win ? (double)ref[g] : 0.0, ev = t < d.win ? (double)est[g] : 0.0;
        const double p_j = pj[q][col], p_a = pa[q][col];
        const double r1 = ev - sv, r2 = p_j - sv, r4 = p_a - p_j, r6 = ev - p_a;
        double* ej = en + j * MUS_NE * 128 + tid;
        ej[0 * 128] = fma(sv, sv, ej[0 * 128]);
        ej[1 * 128] = fma(r1, r1, ej[1 * 128]);
        ej[2 * 128] = fma(r2, r2, ej[2 * 128]);
        ej[3 * 128] = fma(p_j, p_j, ej[3 * 128]);
        ej[4 * 128] = fma(r4, r4, ej[4 * 128]);
        ej[5 * 128] = fma(p_a, p_a, ej[5 * 128]);
        ej[6 * 128] = fma(r6, r6, ej[6 * 128]);
      }
    }
  }
  __syncthreads();
  if (tid < J * MUS_NE) {
    const double* p = en + tid * 128;
    double v = 0.0;
    for (int i = 0; i < 128; ++i) v += p[i];
    epart[((size_t)w * MUS_MAXR + rg) * J * MUS_NE + tid] = v;
  }
}

template <int M, int I>
static int launch_mus_project(const float* ref, const float* est, const double* C, const double* Ct, double* epart, const MusDims& d,
                              cudaStream_t st) {
  constexpr int NCP = (M + I + 1) & ~1;
  const size_t smem = sizeof(double) * (MUS_L * NCP + MUS_PT + MUS_L - 1 + (M / I) * MUS_NE * 128);
  cudaError_t e = cudaFuncSetAttribute(k_mus_project<M, I>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  k_mus_project<M, I><<<(unsigned)d.nwin * d.R, 128, smem, st>>>(ref, est, C, Ct, epart, d);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

__device__ __forceinline__ double mus_safe_db(double num, double den) { return den == 0.0 ? (double)INFINITY : 10.0 * log10(num / den); }

// one CTA per window, thread j per source: ranges summed in order, the four metrics, NaN for a window with a silent source;
// CTA 0 writes the status word
__global__ void __launch_bounds__(32) k_mus_finish(const double* __restrict__ epart, const int* __restrict__ silent, const int* __restrict__ flagG,
                                                   const int* __restrict__ flagB, MusDims d, double* __restrict__ sdr, double* __restrict__ isr,
                                                   double* __restrict__ sir, double* __restrict__ sar, int32_t* __restrict__ status) {
  const int w = blockIdx.x, j = threadIdx.x;
  if (j < d.J) {
    double e[MUS_NE];
    for (int q = 0; q < MUS_NE; ++q) {
      const double* p = epart + (size_t)w * MUS_MAXR * d.J * MUS_NE + j * MUS_NE + q;
      double v = 0.0;
      for (int r = 0; r < d.R; ++r) v += p[(size_t)r * d.J * MUS_NE];
      e[q] = v;
    }
    const bool nan = (silent[2 * w] | silent[2 * w + 1]) != 0;
    const size_t o = (size_t)j * d.nwin + w;
    sdr[o] = nan ? (double)NAN : mus_safe_db(e[0], e[1]);
    isr[o] = nan ? (double)NAN : mus_safe_db(e[0], e[2]);
    sir[o] = nan ? (double)NAN : mus_safe_db(e[3], e[4]);
    sar[o] = nan ? (double)NAN : mus_safe_db(e[5], e[6]);
  }
  if (w == 0 && j == 0) {
    int bad = flagG[0];
    for (int i = 0; i < d.J; ++i) bad |= flagB[i];
    *status = bad ? CTN_BSS_NOT_PD : 0;
  }
}

// ---- host -------------------------------------------------------------------------------------------------------------------
struct MusWs {
  double *part, *corr, *G, *Wg, *Bk, *Wb, *rhsG, *solG, *rhsB, *solB, *epart;
  int *silent, *flagG, *flagB;
};

static void carve_mus(Carver& cv, const MusDims& d, MusWs* w) {
  const size_t M = d.M, N = d.N, L = MUS_L, NB = (size_t)d.I * L;
  w->part = cv.take<double>(2 * M * MUS_NCH * M * L);
  w->corr = cv.take<double>(M * M * L);
  w->G = cv.take<double>(N * N);
  w->Wg = cv.take<double>(N * BSS_NB);
  w->Bk = cv.take<double>((size_t)d.J * NB * NB);
  w->Wb = cv.take<double>((size_t)d.J * NB * BSS_NB);
  w->rhsG = cv.take<double>(N * M);
  w->solG = cv.take<double>(N * M);
  w->rhsB = cv.take<double>(N * d.I);
  w->solB = cv.take<double>(N * d.I);
  w->epart = cv.take<double>((size_t)d.nwin * MUS_MAXR * d.J * MUS_NE);
  w->silent = cv.take<int>((size_t)d.nwin * 2);
  w->flagG = cv.take<int>(1);
  w->flagB = cv.take<int>(d.J);
}

static int mus_dims(int J, int I, int T, int win, int hop, MusDims* d) {
  if (J < 1 || I < 1 || T < 1 || win < 1 || hop < 1) return CTN_EINVAL;
  if ((long long)J * I > MUS_MAXM) return CTN_EUNSUPPORTED;
  const long long nwin = ((long long)T - win + hop) / hop;
  if ((long long)T - win + hop < hop || nwin < 1) return CTN_EINVAL;  // floor((T - win + hop) / hop) <= 0
  if (nwin * MUS_MAXR > 0x7fffffffLL) return CTN_EUNSUPPORTED;
  d->J = J; d->I = I; d->M = J * I; d->T = T; d->win = win; d->hop = hop; d->nwin = (int)nwin;
  d->N = d->M * MUS_L;
  d->ntile = (int)(((long long)win + MUS_L - 1 + MUS_PT - 1) / MUS_PT);
  d->per = (d->ntile + MUS_MAXR - 1) / MUS_MAXR;
  d->R = (d->ntile + d->per - 1) / d->per;
  return CTN_OK;
}

extern "C" int ctn_bss_images_workspace_bytes(int J, int I, int T, int win, int hop, size_t* bytes) {
  MusDims d;
  CTN_TRY(mus_dims(J, I, T, win, hop, &d));
  if (!bytes) return CTN_EINVAL;
  Carver cv(nullptr);
  MusWs w;
  carve_mus(cv, d, &w);
  *bytes = cv.off + 256;
  return CTN_OK;
}

// (J, I) with J I <= 8
static int mus_project_dispatch(const float* ref, const float* est, const MusWs& w, const MusDims& d, cudaStream_t st) {
#define MUS_CASE(J_, I_) \
  if (d.J == J_ && d.I == I_) return launch_mus_project<J_ * I_, I_>(ref, est, w.rhsG, w.rhsB, w.epart, d, st);
  MUS_CASE(1, 1) MUS_CASE(2, 1) MUS_CASE(3, 1) MUS_CASE(4, 1) MUS_CASE(5, 1) MUS_CASE(6, 1) MUS_CASE(7, 1) MUS_CASE(8, 1)
  MUS_CASE(1, 2) MUS_CASE(2, 2) MUS_CASE(3, 2) MUS_CASE(4, 2)
  MUS_CASE(1, 3) MUS_CASE(2, 3)
  MUS_CASE(1, 4) MUS_CASE(2, 4)
  MUS_CASE(1, 5) MUS_CASE(1, 6) MUS_CASE(1, 7) MUS_CASE(1, 8)
#undef MUS_CASE
  return CTN_EUNSUPPORTED;
}

static int mus_corr(const float* ref, const float* est, double* part, const MusDims& d, cudaStream_t st) {
  const dim3 grid(MUS_NCH, 2 * d.M);
  switch (d.M) {
    case 1: k_mus_corr<1><<<grid, 128, 0, st>>>(ref, est, part, d); break;
    case 2: k_mus_corr<2><<<grid, 128, 0, st>>>(ref, est, part, d); break;
    case 3: k_mus_corr<3><<<grid, 128, 0, st>>>(ref, est, part, d); break;
    case 4: k_mus_corr<4><<<grid, 128, 0, st>>>(ref, est, part, d); break;
    case 5: k_mus_corr<5><<<grid, 128, 0, st>>>(ref, est, part, d); break;
    case 6: k_mus_corr<6><<<grid, 128, 0, st>>>(ref, est, part, d); break;
    case 7: k_mus_corr<7><<<grid, 128, 0, st>>>(ref, est, part, d); break;
    default: k_mus_corr<8><<<grid, 128, 0, st>>>(ref, est, part, d); break;
  }
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_bss_eval_images(const float* ref, const float* est, int J, int I, int T, int win, int hop, double* sdr, double* isr,
                                   double* sir, double* sar, int32_t* status, void* ws, size_t ws_bytes, ctn_stream_t stream) {
  LaunchScope scope(ref);
  if (!ref || !est || !sdr || !isr || !sir || !sar || !status || !ws) return CTN_EINVAL;
  MusDims d;
  CTN_TRY(mus_dims(J, I, T, win, hop, &d));
  if (((uintptr_t)ws) & 255) return CTN_EALIGN;
  size_t need = 0;
  CTN_TRY(ctn_bss_images_workspace_bytes(J, I, T, win, hop, &need));
  if (ws_bytes < need) return CTN_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  Carver cv(ws);
  MusWs w;
  carve_mus(cv, d, &w);

  k_mus_silent<<<dim3(d.nwin, 2), 256, 0, st>>>(ref, est, w.silent, d);
  CTN_COUNT_LAUNCH();
  CTN_TRY(mus_corr(ref, est, w.part, d, st));
  k_mus_combine<<<dim3(d.M, 2 * d.M), MUS_L, 0, st>>>(w.part, w.corr, w.rhsG, w.rhsB, d);
  CTN_COUNT_LAUNCH();
  k_mus_build<<<(unsigned)(((size_t)d.N * d.N + 255) / 256), 256, 0, st>>>(w.corr, w.G, w.Bk, d);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();

  const MatSet g{w.G, w.Wg, w.flagG, d.N, d.N / BSS_NB, 1};
  const MatSet blk{w.Bk, w.Wb, w.flagB, d.I * MUS_L, d.I * MUS_L / BSS_NB, d.J};
  CTN_TRY(ctn_chol_factor(g, st));
  CTN_TRY(ctn_chol_factor(blk, st));
  CTN_TRY(ctn_chol_solve_multi(g, w.rhsG, w.solG, d.M, st));
  CTN_TRY(ctn_chol_solve_multi(blk, w.rhsB, w.solB, d.I, st));

  CTN_TRY(mus_project_dispatch(ref, est, w, d, st));
  k_mus_finish<<<d.nwin, 32, 0, st>>>(w.epart, w.silent, w.flagG, w.flagB, d, sdr, isr, sir, sar, status);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
