// CUDA-core (exact fp32 FFMA) implementation of the TCN stages + the stages shared with the wgmma path
// (weight folding, depthwise stage, finishing, pitch copies).
//
// Per ResidualBlock1d (src/models/tdcn.py:107-147 + 177-196), with d = dilation:
//   K_A  (pointwise, EPI_H):   h = PReLU_a1(W1 x + b1)                      + (sum, sumsq) of h        -> stats1
//   K_B  (ctn_dw_fwd):         u = PReLU_a2(dwconv_d(zero-pad(gLN1(h))) + bd) + (sum, sumsq) of u        -> stats2
//   K_C  (pointwise, EPI_RAW): r = [Wo;Ws] diag(gamma2) u                   (gLN2 folded, see ctn_internal.h)
//   K_F  (ctn_finish_fwd):     x += rstd2*r[:B] + c_o   (the skip rows: ctn_skip_reduce, once over all blocks)
#include "ctn_internal.h"

// ------------------------------------------------------------------------------------------------
// weight folding: one warp per output row
// ------------------------------------------------------------------------------------------------
// __restrict__ lets the compiler issue the loads of W, gamma and beta ahead of the stores to Wf; the pointers of a FoldJob carry
// no such promise, hence the helper.
__device__ __forceinline__ void fold_row(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ gamma,
                                         const float* __restrict__ beta, int K, int row, int row_offset, float* __restrict__ Wf,
                                         float* __restrict__ v1, float* __restrict__ v2, float* __restrict__ vb, float R) {
  const int lane = threadIdx.x & 31;
  float s1 = 0.f, s2 = 0.f, s3 = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float w = W[(size_t)row * K + k];
    const float wf = w * gamma[k];
    Wf[(size_t)(row + row_offset) * K + k] = wf;
    s1 = fmaf(w, beta[k], s1);
    s2 += wf;
    s3 = fmaf(fabsf(w), fmaf(fabsf(gamma[k]), R, fabsf(beta[k])), s3);
  }
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  s3 = warp_sum(s3);
  if (lane == 0) {
    v1[row + row_offset] = s1 + (bias ? bias[row] : 0.f);
    v2[row + row_offset] = s2;
    if (vb) vb[row + row_offset] = s3 + (bias ? fabsf(bias[row]) : 0.f);
  }
}

struct FoldJobs { FoldJob j[CTN_MAX_JOBS]; };
// grid ((rows of the largest job + 3) / 4, jobs): one warp per row of one job.  No grid-stride loop: with one, the loads lose
// their early issue and a single fold takes twice as long (H100).
__global__ void __launch_bounds__(128) k_fold_batch(const FoldJobs jobs) {
  const FoldJob& jb = jobs.j[blockIdx.y];
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= jb.M) return;
  fold_row(jb.W, jb.bias, jb.gamma, jb.beta, jb.K, row, jb.row_offset, jb.out.Wf, jb.out.v1, jb.out.v2, jb.out.vb, jb.R);
}

int ctn_fold_batch(const FoldJob* jobs, int n, cudaStream_t st) {
  for (int i0 = 0; i0 < n; i0 += CTN_MAX_JOBS) {
    FoldJobs fj;
    const int m = n - i0 < CTN_MAX_JOBS ? n - i0 : CTN_MAX_JOBS;
    int maxM = 1;
    for (int i = 0; i < m; ++i) { fj.j[i] = jobs[i0 + i]; if (jobs[i0 + i].M > maxM) maxM = jobs[i0 + i].M; }
    k_fold_batch<<<dim3((maxM + 3) / 4, m), 128, 0, st>>>(fj);
    CTN_COUNT_LAUNCH();
  }
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ------------------------------------------------------------------------------------------------
// activation envelope of the fp16-piece mode (see ctn_internal.h: ScaleJobs)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float pow2_scale_for(float bound) {
  // largest power of two s with bound * s <= 2^15 (fp16 max 65504); 1 for a zero / non-finite bound
  if (!(bound > 0.f) || !(bound < 3.0e38f)) return 1.f;
  int e;
  frexpf(bound, &e);  // bound = m 2^e, m in [0.5, 1)  =>  bound <= 2^e
  e = 15 - e;
  e = e < -100 ? -100 : (e > 100 ? 100 : e);
  return ldexpf(1.f, e);
}
__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) v = fmaxf(v, red[i]);
  return v;
}
// grid = number of residual blocks: block i packs dwp_i and writes its three partial bounds (U_i, D_out_i, D_skip_i)
__global__ void __launch_bounds__(256) k_scale_partials(const ScaleJobs jobs, float* __restrict__ part) {
  __shared__ float red[8];
  const ScaleJob& jb = jobs.j[blockIdx.x];
  const int H = jobs.H, P = jobs.P;
  const float a2 = fmaxf(1.f, fabsf(jb.slope2[0]));
  float u = 0.f;
  const int Hp = (H + 15) & ~15;
  for (int c = threadIdx.x; c < Hp; c += blockDim.x) {
    float g = 0.f, b = 0.f, bd = 0.f, w[3] = {0.f, 0.f, 0.f}, wsum = 0.f;
    if (c < H) {
      g = jb.g1[c]; b = jb.b1[c]; bd = jb.dw_b[c];
      for (int k = 0; k < P; ++k) { const float wk = jb.dw_w[c * P + k]; wsum += fabsf(wk); if (k < 3) w[k] = wk; }
      u = fmaxf(u, a2 * fmaf(fmaf(fabsf(g), jobs.R, fabsf(b)), wsum, fabsf(bd)));
    }
    if (jb.dwp && P == 3) {
      float4* d = reinterpret_cast<float4*>(jb.dwp + (size_t)c * 8);
      d[0] = make_float4(g, b, w[0], w[1]);
      d[1] = make_float4(w[2], bd, 0.f, 0.f);
    }
  }
  u = block_max(u, red);
  float dout = 0.f, dskip = 0.f;
  const int Mt = jb.has_out ? jobs.Bc + jobs.Sc : jobs.Sc;
  for (int n = threadIdx.x; n < Mt; n += blockDim.x) {
    const float v = jb.vb[n];
    if (jb.has_out && n < jobs.Bc) dout = fmaxf(dout, v); else dskip = fmaxf(dskip, v);
  }
  dout = block_max(dout, red);
  dskip = block_max(dskip, red);
  if (threadIdx.x == 0) { part[3 * blockIdx.x] = u; part[3 * blockIdx.x + 1] = dout; part[3 * blockIdx.x + 2] = dskip; }
}
__global__ void __launch_bounds__(256) k_scale_chain(const ScaleJobs jobs, const float* __restrict__ part) {
  // stage everything the serial chain needs in shared memory first (the dependent global loads of a one-thread loop cost 12 us)
  __shared__ float sp[3 * CTN_MAX_BLOCKS];
  __shared__ float sx[8];
  for (int i = threadIdx.x; i < 3 * jobs.n; i += blockDim.x) sp[i] = part[i];
  float X = 0.f;
  for (int i = threadIdx.x; i < jobs.x0_n; i += blockDim.x) X = fmaxf(X, fabsf(jobs.x0_bound[i]));
  X = block_max(X, sx);
  __syncthreads();
  if (threadIdx.x != 0) return;
  float S = 0.f;
  for (int i = 0; i < jobs.n; ++i) {
    jobs.scales[2 * i] = pow2_scale_for(X);
    jobs.scales[2 * i + 1] = pow2_scale_for(sp[3 * i]);
    X += sp[3 * i + 1];
    S += sp[3 * i + 2];
  }
  const float am = jobs.mask_slope ? fmaxf(1.f, fabsf(jobs.mask_slope[0])) : 1.f;
  jobs.scales[2 * jobs.n] = pow2_scale_for(am * S);
}
int ctn_act_scales(const ScaleJobs& jobs, cudaStream_t st) {
  if (jobs.n <= 0 || jobs.n > CTN_MAX_BLOCKS) return CTN_EINVAL;
  float* part = jobs.scales + 2 * jobs.n + 1;  // scratch behind the scales: 3 floats per block
  k_scale_partials<<<jobs.n, 256, 0, st>>>(jobs, part);
  CTN_COUNT_LAUNCH();
  k_scale_chain<<<1, 256, 0, st>>>(jobs, part);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

__global__ void __launch_bounds__(256) k_absmax_pitch(const float* __restrict__ x, int rows, int frames, int pitch, float* __restrict__ out) {
  __shared__ float red[8];
  float m = 0.f;
  for (int r = blockIdx.x; r < rows; r += gridDim.x)
    for (int t = threadIdx.x; t < frames; t += blockDim.x) m = fmaxf(m, fabsf(x[(size_t)r * pitch + t]));
  m = block_max(m, red);
  if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(m));  // non-negative floats order like uints
}
int ctn_absmax_pitch(const float* x, int rows, int frames, int pitch, float* out, cudaStream_t st) {
  k_absmax_pitch<<<rows < 1024 ? rows : 1024, 256, 0, st>>>(x, rows, frames, pitch, out);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ------------------------------------------------------------------------------------------------
// pointwise (1x1) contraction, fp32 FFMA:  D[b][m][t] = epi( sum_k W[m][k] * pro(A[b][k][t]) )
// 64(m) x 64(t) x 16(k) tiles, 256 threads, 4x4 micro-tiles, 128-bit loads/stores along t.
// ------------------------------------------------------------------------------------------------
template <int PRO, int EPI>
__global__ void __launch_bounds__(256) k_pw_simt(const PwArgs a) {
  __shared__ __align__(16) float As[16][64 + 4];  // [k][m]  (weights, transposed)
  __shared__ __align__(16) float Bs[16][64];      // [k][t]
  __shared__ double red[64];
  const int b = blockIdx.z, m0 = blockIdx.y * 64, t0 = blockIdx.x * 64;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const float* Ab = a.A + (size_t)b * a.K * a.pitch;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float pslope = 0.f;
  if (PRO == PRO_PRELU) pslope = a.pro_slope[0];

  const int lm = tid >> 2, lk = (tid & 3) * 4;   // W tile: row lm (0..63), k offset lk
  const int bk = tid >> 4, bt = (tid & 15) * 4;  // A tile: row bk (0..15), t offset bt
  for (int k0 = 0; k0 < a.K; k0 += 16) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + lm, k = k0 + lk + i;
      As[lk + i][lm] = (m < a.M && k < a.K) ? a.W[(size_t)m * a.K + k] : 0.f;
    }
    {
      const int k = k0 + bk;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k < a.K) v = *reinterpret_cast<const float4*>(Ab + (size_t)k * a.pitch + t0 + bt);
      if (PRO == PRO_PRELU) {
        v.x = prelu_f(v.x, pslope); v.y = prelu_f(v.y, pslope); v.z = prelu_f(v.z, pslope); v.w = prelu_f(v.w, pslope);
      }
      *reinterpret_cast<float4*>(&Bs[bk][bt]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 w4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 x4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
      const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(wv[i], xv[j], acc[i][j]);
    }
    __syncthreads();
  }

  // ---- epilogue ----
  float2 mr = make_float2(0.f, 1.f);
  if (EPI == EPI_HEAD) mr = gln_mean_rstd(a.stats_in + 2 * b, a.n_in, a.eps);
  float eslope = 0.f;
  if (EPI == EPI_H) eslope = a.slope[0];
  float ls = 0.f, lss = 0.f;
  const int t = t0 + tx * 4;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= a.M) continue;
    float o[4];
    float wv[4] = {0.f, 0.f, 0.f, 0.f};
    if (EPI == EPI_MASK) {
      const float4 w4 = *reinterpret_cast<const float4*>(a.wenc + ((size_t)b * a.Nb + (m % a.Nb)) * a.pitch + t);
      wv[0] = w4.x; wv[1] = w4.y; wv[2] = w4.z; wv[3] = w4.w;
    }
    float mk[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v = acc[i][j];
      if (EPI == EPI_HEAD) v = mr.y * v + (a.v1[m] - mr.x * mr.y * a.v2[m]);
      if (EPI == EPI_H) v = prelu_f(v + a.bias[m], eslope);
      if (EPI == EPI_MASK) {
        if (a.mask_logits) {
          v += a.bias[m];
          mk[j] = v;
        } else {
          v = 1.f / (1.f + expf(-(v + a.bias[m])));
          mk[j] = v;
          v *= wv[j];
        }
      }
      if (t + j >= a.frames) { v = 0.f; mk[j] = 0.f; }
      o[j] = v;
      if (EPI == EPI_H) { ls += v; lss += v * v; }
    }
    *reinterpret_cast<float4*>(a.D + ((size_t)b * a.M + m) * a.pitch + t) = make_float4(o[0], o[1], o[2], o[3]);
    if (EPI == EPI_MASK && a.mask_out)
      *reinterpret_cast<float4*>(a.mask_out + ((size_t)b * a.M + m) * a.pitch + t) = make_float4(mk[0], mk[1], mk[2], mk[3]);
  }
  if (EPI == EPI_H) {
    double s = ls, ss = lss;
    block_sum2_d(s, ss, red);
    if (tid == 0) { atomicAdd(&a.stats_out[2 * b], s); atomicAdd(&a.stats_out[2 * b + 1], ss); }
  }
}

int ctn_pw_simt(const PwArgs& a, int pro, int epi, cudaStream_t st) {
  if (a.pitch % 64 != 0) return CTN_EALIGN;
  dim3 grid(a.pitch / 64, (a.M + 63) / 64, a.B);
#define PW_LAUNCH(P, E)                               \
  if (pro == P && epi == E) {                         \
    k_pw_simt<P, E><<<grid, 256, 0, st>>>(a);         \
    CTN_COUNT_LAUNCH();                               \
    CTN_RETURN_IF_CUDA_ERR();                         \
    return CTN_OK;                                    \
  }
  PW_LAUNCH(PRO_NONE, EPI_RAW)
  PW_LAUNCH(PRO_NONE, EPI_HEAD)
  PW_LAUNCH(PRO_NONE, EPI_H)
  PW_LAUNCH(PRO_PRELU, EPI_MASK)
#undef PW_LAUNCH
  return CTN_EUNSUPPORTED;
}

// softmax over ALL M = S*N mask channels per frame, then * w: thread = one frame (coalesced along t), three passes over the channels
__global__ void __launch_bounds__(128) k_softmax_mask(float* __restrict__ x, const float* __restrict__ wenc, float* __restrict__ mask_out, int M,
                                                      int Nb, int frames, int pitch) {
  const int b = blockIdx.y, t = blockIdx.x * 128 + threadIdx.x;
  if (t >= pitch) return;
  float* col = x + (size_t)b * M * pitch + t;
  if (t >= frames) {
    for (int m = 0; m < M; ++m) { col[(size_t)m * pitch] = 0.f; if (mask_out) mask_out[((size_t)b * M + m) * pitch + t] = 0.f; }
    return;
  }
  float mx = -INFINITY;
  for (int m = 0; m < M; ++m) mx = fmaxf(mx, col[(size_t)m * pitch]);
  float sum = 0.f;
  for (int m = 0; m < M; ++m) sum += expf(col[(size_t)m * pitch] - mx);
  const float inv = 1.f / sum;
  const float* wc = wenc + (size_t)b * Nb * pitch + t;
  for (int m = 0; m < M; ++m) {
    const float p = expf(col[(size_t)m * pitch] - mx) * inv;
    if (mask_out) mask_out[((size_t)b * M + m) * pitch + t] = p;
    col[(size_t)m * pitch] = p * wc[(size_t)(m % Nb) * pitch];
  }
}
int ctn_softmax_mask(float* logits_what, const float* wenc, float* mask_out, int B, int M, int Nb, int frames, int pitch, cudaStream_t st) {
  k_softmax_mask<<<dim3((pitch + 127) / 128, B), 128, 0, st>>>(logits_what, wenc, mask_out, M, Nb, frames, pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ------------------------------------------------------------------------------------------------
// depthwise stage:  u[c][t] = PReLU( sum_k wd[c][k] * hn[c][t + k*d - pl] + bd[c] ),
//   hn = gLN1(h) inside [0,frames), exactly 0 outside (F.pad after the norm, tdcn.py:123-132),
//   pl = ((P-1)d)//2.   + (sum, sumsq) of u -> stats_out.
// thread = 4 consecutive frames of one channel; grid (pitch/512, H, B), block 128.
// ------------------------------------------------------------------------------------------------
template <int P>
__global__ void __launch_bounds__(128) k_dw(const float* __restrict__ h, float* __restrict__ u, const float* __restrict__ norm_g,
                                            const float* __restrict__ norm_b, const float* __restrict__ dw_w,
                                            const float* __restrict__ dw_b, const float* __restrict__ slope,
                                            const double* __restrict__ stats_in, double* __restrict__ stats_out, int H,
                                            int frames, int pitch, int Pdyn, int dilation, int pad_left, float eps) {
  __shared__ double red[64];
  const int b = blockIdx.z, c = blockIdx.y;
  const int t = (blockIdx.x * 128 + threadIdx.x) * 4;
  const int taps = P > 0 ? P : Pdyn;
  const float2 mr = gln_mean_rstd(stats_in + 2 * b, (double)H * (double)frames, eps);
  const float g = norm_g[c] * mr.y, sh = norm_b[c] - mr.x * mr.y * norm_g[c];
  const float a2 = slope[0], bd = dw_b[c];
  const float* hr = h + ((size_t)b * H + c) * pitch;
  float o[4] = {bd, bd, bd, bd};
  if (t < pitch) {
    for (int k = 0; k < taps; ++k) {
      const float wk = dw_w[c * taps + k];
      const int off = k * dilation - pad_left;
      const int ts = t + off;
      if ((off & 3) == 0 && ts >= 0 && ts + 3 < frames) {
        const float4 v = *reinterpret_cast<const float4*>(hr + ts);
        o[0] = fmaf(wk, fmaf(v.x, g, sh), o[0]);
        o[1] = fmaf(wk, fmaf(v.y, g, sh), o[1]);
        o[2] = fmaf(wk, fmaf(v.z, g, sh), o[2]);
        o[3] = fmaf(wk, fmaf(v.w, g, sh), o[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int tj = ts + j;
          if (tj >= 0 && tj < frames) o[j] = fmaf(wk, fmaf(hr[tj], g, sh), o[j]);
        }
      }
    }
  }
  float ls = 0.f, lss = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float v = prelu_f(o[j], a2);
    if (t + j >= frames) v = 0.f;
    o[j] = v;
    ls += v;
    lss += v * v;
  }
  if (t < pitch) *reinterpret_cast<float4*>(u + ((size_t)b * H + c) * pitch + t) = make_float4(o[0], o[1], o[2], o[3]);
  double s = ls, ss = lss;
  block_sum2_d(s, ss, red);
  if (threadIdx.x == 0) { atomicAdd(&stats_out[2 * b], s); atomicAdd(&stats_out[2 * b + 1], ss); }
}

int ctn_dw_fwd(const float* h, float* u, const float* norm_g, const float* norm_b, const float* dw_w, const float* dw_b,
               const float* slope, const double* stats_in, double* stats_out, int B, int H, int frames, int pitch, int P,
               int dilation, float eps, cudaStream_t st) {
  const int pad_left = ((P - 1) * dilation) / 2;
  dim3 grid((pitch + 511) / 512, H, B);
  if (P == 3)
    k_dw<3><<<grid, 128, 0, st>>>(h, u, norm_g, norm_b, dw_w, dw_b, slope, stats_in, stats_out, H, frames, pitch, P, dilation, pad_left, eps);
  else
    k_dw<0><<<grid, 128, 0, st>>>(h, u, norm_g, norm_b, dw_w, dw_b, slope, stats_in, stats_out, H, frames, pitch, P, dilation, pad_left, eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ------------------------------------------------------------------------------------------------
// finishing: residual update with the deferred gLN2 scale/shift, x += rstd2*r[:Bc] + c (the skip rows go to k_skip_reduce)
// grid (pitch/512, Bc, B), block 128
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_finish(const float* __restrict__ outraw, const float* __restrict__ v1,
                                                const float* __restrict__ v2, const double* __restrict__ stats2, double n2,
                                                float eps, float* __restrict__ x, int Bc, int Sc, int frames, int pitch) {
  const int b = blockIdx.z, m = blockIdx.y;
  const int t = (blockIdx.x * 128 + threadIdx.x) * 4;
  if (t >= pitch) return;
  const float2 mr = gln_mean_rstd(stats2 + 2 * b, n2, eps);
  const float c = v1[m] - mr.x * mr.y * v2[m];
  float4 r = *reinterpret_cast<const float4*>(outraw + ((size_t)b * (Bc + Sc) + m) * pitch + t);
  r.x = fmaf(mr.y, r.x, c); r.y = fmaf(mr.y, r.y, c); r.z = fmaf(mr.y, r.z, c); r.w = fmaf(mr.y, r.w, c);
  float* dst = x + ((size_t)b * Bc + m) * pitch + t;
  const float4 o = *reinterpret_cast<const float4*>(dst);
  r.x += o.x; r.y += o.y; r.z += o.z; r.w += o.w;
  if (t + 0 >= frames) r.x = 0.f;
  if (t + 1 >= frames) r.y = 0.f;
  if (t + 2 >= frames) r.z = 0.f;
  if (t + 3 >= frames) r.w = 0.f;
  *reinterpret_cast<float4*>(dst) = r;
}

int ctn_finish_fwd(const float* outraw, const FoldedConv f, const double* stats2, double n2, float eps, float* x, int B, int Bc,
                   int Sc, int frames, int pitch, cudaStream_t st) {
  dim3 grid((pitch + 511) / 512, Bc, B);
  k_finish<<<grid, 128, 0, st>>>(outraw, f.v1, f.v2, stats2, n2, eps, x, Bc, Sc, frames, pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// grid (pitch/512, Sc, B), block 128: thread = 4 consecutive frames of one skip channel, loops over the blocks
__global__ void __launch_bounds__(128) k_skip_reduce(const SkipJobs jobs, double n2, float eps, float* __restrict__ skip, int Sc,
                                                     int frames, int pitch) {
  // per residual block the (rstd, folded constant) of this (sample, channel) -- computed ONCE per thread block (the fp64 mean /
  // rstd evaluation used to run 24 times in every thread and out-weighed the 24 loads it accompanied)
  __shared__ float s_rstd[CTN_MAX_BLOCKS], s_c[CTN_MAX_BLOCKS];
  const int b = blockIdx.z, m = blockIdx.y;
  if (threadIdx.x < jobs.n) {
    const SkipJob& jb = jobs.j[threadIdx.x];
    const float2 mr = gln_mean_rstd(jb.stats2 + 2 * b, n2, eps);
    s_rstd[threadIdx.x] = mr.y;
    s_c[threadIdx.x] = __ldg(jb.v1 + jb.off + m) - mr.x * mr.y * __ldg(jb.v2 + jb.off + m);
  }
  __syncthreads();
  const int t = (blockIdx.x * 128 + threadIdx.x) * 4;
  if (t >= pitch) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
  for (int i = 0; i < jobs.n; ++i) {
    const SkipJob& jb = jobs.j[i];
    const float4 r = __ldg(reinterpret_cast<const float4*>(jb.r + ((size_t)b * jb.Mt + jb.off + m) * pitch + t));
    const float rs = s_rstd[i], c = s_c[i];
    acc.x += fmaf(rs, r.x, c); acc.y += fmaf(rs, r.y, c); acc.z += fmaf(rs, r.z, c); acc.w += fmaf(rs, r.w, c);
  }
  if (t + 0 >= frames) acc.x = 0.f;
  if (t + 1 >= frames) acc.y = 0.f;
  if (t + 2 >= frames) acc.z = 0.f;
  if (t + 3 >= frames) acc.w = 0.f;
  *reinterpret_cast<float4*>(skip + ((size_t)b * Sc + m) * pitch + t) = acc;
}

int ctn_skip_reduce(const SkipJobs& jobs, double n2, float eps, float* skip, int B, int Sc, int frames, int pitch, cudaStream_t st) {
  dim3 grid((pitch + 511) / 512, Sc, B);
  k_skip_reduce<<<grid, 128, 0, st>>>(jobs, n2, eps, skip, Sc, frames, pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ------------------------------------------------------------------------------------------------
// pitch copies (module-level API <-> internal padded layout)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_copy_to_pitch(const float* __restrict__ src, float* __restrict__ dst, int frames, int pitch) {
  const size_t row = blockIdx.y;
  for (int t = blockIdx.x * 256 + threadIdx.x; t < pitch; t += gridDim.x * 256)
    dst[row * pitch + t] = t < frames ? src[row * frames + t] : 0.f;
}
__global__ void __launch_bounds__(256) k_copy_from_pitch(const float* __restrict__ src, float* __restrict__ dst, int frames, int pitch) {
  const size_t row = blockIdx.y;
  for (int t = blockIdx.x * 256 + threadIdx.x; t < frames; t += gridDim.x * 256) dst[row * frames + t] = src[row * pitch + t];
}
int ctn_copy_to_pitch(const float* src, float* dst, int rows, int frames, int pitch, cudaStream_t st) {
  int gx = (pitch + 255) / 256; if (gx > 16) gx = 16;
  for (int r0 = 0; r0 < rows; r0 += 65535) {
    const int nr = rows - r0 < 65535 ? rows - r0 : 65535;
    k_copy_to_pitch<<<dim3(gx, nr), 256, 0, st>>>(src + (size_t)r0 * frames, dst + (size_t)r0 * pitch, frames, pitch);
    CTN_COUNT_LAUNCH();
  }
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
int ctn_copy_from_pitch(const float* src, float* dst, int rows, int frames, int pitch, cudaStream_t st) {
  int gx = (frames + 255) / 256; if (gx > 16) gx = 16;
  for (int r0 = 0; r0 < rows; r0 += 65535) {
    const int nr = rows - r0 < 65535 ? rows - r0 : 65535;
    k_copy_from_pitch<<<dim3(gx, nr), 256, 0, st>>>(src + (size_t)r0 * pitch, dst + (size_t)r0 * frames, frames, pitch);
    CTN_COUNT_LAUNCH();
  }
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
