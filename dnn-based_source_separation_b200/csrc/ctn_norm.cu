// Stand-alone normalisation entry points (module-level API parity): GlobalLayerNorm and CumulativeLayerNorm1d
// on PyTorch-contiguous (B,C,T) tensors.  Inside the fused forward the gLN statistics are produced by the
// epilogue of the producing kernel and the affine normalisation is folded into the consumer (ctn_tcn_*.cu).
#include "ctn_common.cuh"

// ---- gLN: GroupNorm(1,C,eps), src/modules/norm.py:18,32 -------------------------------------------------
// Every element is summed in double: the square of an fp32 value is exact there, so var = E[x^2] - mean^2 keeps its digits
// under a DC offset.  With fp32 partial sums the variance error grows with offset^2, and at |mean| / std ~ 1e3 the output
// was 3x outside the fp32 forward-error bound.  The input here is user data, not a normalised activation.
__global__ void __launch_bounds__(256) k_gln_stats(const float* __restrict__ x, size_t per_sample, double* __restrict__ stats) {
  __shared__ double red[64];
  const int b = blockIdx.y;
  const float* xb = x + (size_t)b * per_sample;
  double s = 0.0, ss = 0.0;
  for (size_t i0 = (size_t)blockIdx.x * 256 * 8; i0 < per_sample; i0 += (size_t)gridDim.x * 256 * 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const size_t i = i0 + (size_t)j * 256 + threadIdx.x;
      const double v = i < per_sample ? (double)xb[i] : 0.0;
      s += v;
      ss = fma(v, v, ss);
    }
  }
  block_sum2_d(s, ss, red);
  if (threadIdx.x == 0) { atomicAdd(&stats[2 * b], s); atomicAdd(&stats[2 * b + 1], ss); }
}

__global__ void __launch_bounds__(256) k_gln_apply(const float* __restrict__ x, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, float* __restrict__ y, int C, int T,
                                                   float eps, const double* __restrict__ stats) {
  const int b = blockIdx.z, c = blockIdx.y;
  const float2 mr = gln_mean_rstd(stats + 2 * b, (double)C * (double)T, eps);
  const float g = gamma[c] * mr.y, sh = beta[c] - mr.x * mr.y * gamma[c];
  const size_t off = ((size_t)b * C + c) * T;
  for (int t = blockIdx.x * 256 + threadIdx.x; t < T; t += gridDim.x * 256) {
    // (x - mean) * rstd * gamma + beta, evaluated as in ATen's fused scale/shift form
    y[off + t] = fmaf(x[off + t], g, sh);
  }
}

extern "C" int ctn_gln_fwd(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int T,
                           float eps, double* scratch, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !gamma || !beta || !y || !scratch || B <= 0 || C <= 0 || T <= 0) return CTN_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * B, st);
  if (e != cudaSuccess) return (int)e;
  const size_t per = (size_t)C * T;
  int chunks = (int)((per + 2047) / 2048);
  if (chunks > 296) chunks = 296;
  k_gln_stats<<<dim3(chunks, B), 256, 0, st>>>(x, per, scratch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  int gx = (T + 255) / 256;
  if (gx > 64) gx = 64;
  k_gln_apply<<<dim3(gx, C, B), 256, 0, st>>>(x, gamma, beta, y, C, T, eps, scratch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- cLN: src/modules/norm.py:78-90 --------------------------------------------------------------------
// x rows are `pitch` floats apart (pitch == T for PyTorch-contiguous tensors, the padded pitch inside the fused forward)
__global__ void __launch_bounds__(128) k_cln_step(const float* __restrict__ x, int C, int T, int pitch, double* __restrict__ st) {
  const int b = blockIdx.y, t = blockIdx.x * 128 + threadIdx.x;
  if (t >= T) return;
  const float* xb = x + (size_t)b * C * pitch + t;
  double s = 0.0, ss = 0.0;
  for (int c = 0; c < C; ++c) {
    const double v = (double)xb[(size_t)c * pitch];
    s += v;
    ss += v * v;
  }
  st[((size_t)b * T + t) * 2] = s;
  st[((size_t)b * T + t) * 2 + 1] = ss;
}

// inclusive scan along t, one block (1024 threads) per sample
__global__ void __launch_bounds__(1024) k_cln_scan(double* __restrict__ st, int T) {
  __shared__ double wsum[2][32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  double* sb = st + (size_t)b * T * 2;
  const int per = (T + 1023) / 1024;
  const int t0 = tid * per, t1 = min(T, t0 + per);
  double s = 0.0, ss = 0.0;
  for (int t = t0; t < t1; ++t) { s += sb[2 * t]; ss += sb[2 * t + 1]; }
  // exclusive scan of (s, ss) over threads
  double ps = s, pss = ss;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double a = __shfl_up_sync(0xffffffffu, ps, o), c = __shfl_up_sync(0xffffffffu, pss, o);
    if (lane >= o) { ps += a; pss += c; }
  }
  if (lane == 31) { wsum[0][wid] = ps; wsum[1][wid] = pss; }
  __syncthreads();
  if (wid == 0) {
    double a = wsum[0][lane], c = wsum[1][lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double a2 = __shfl_up_sync(0xffffffffu, a, o), c2 = __shfl_up_sync(0xffffffffu, c, o);
      if (lane >= o) { a += a2; c += c2; }
    }
    wsum[0][lane] = a;
    wsum[1][lane] = c;
  }
  __syncthreads();
  double base_s = (ps - s) + (wid > 0 ? wsum[0][wid - 1] : 0.0);
  double base_ss = (pss - ss) + (wid > 0 ? wsum[1][wid - 1] : 0.0);
  for (int t = t0; t < t1; ++t) {
    base_s += sb[2 * t];
    base_ss += sb[2 * t + 1];
    sb[2 * t] = base_s;
    sb[2 * t + 1] = base_ss;
  }
}

// y may alias x.  Columns [T, pitch) of y are written as zero (padded layout).
__global__ void __launch_bounds__(128) k_cln_apply(const float* x, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, float* y, int C, int T, int pitch,
                                                   float eps, const double* __restrict__ st) {
  const int b = blockIdx.z, t = blockIdx.x * 128 + threadIdx.x;
  if (t >= pitch) return;
  if (t >= T) {
    for (int c = blockIdx.y; c < C; c += gridDim.y) y[((size_t)b * C + c) * pitch + t] = 0.f;
    return;
  }
  const double n = (double)C * (double)(t + 1);
  const double mean = st[((size_t)b * T + t) * 2] / n;
  double var = st[((size_t)b * T + t) * 2 + 1] / n - mean * mean;
  var = var > 0.0 ? var : 0.0;  // the reference can go NaN here (SURVEY.md 8a-6); we clamp
  const float m = (float)mean, inv = 1.f / ((float)sqrt(var) + eps);  // eps OUTSIDE the sqrt (norm.py:90)
  for (int c = blockIdx.y; c < C; c += gridDim.y) {
    const size_t i = ((size_t)b * C + c) * pitch + t;
    y[i] = (x[i] - m) * inv * gamma[c] + beta[c];
  }
}

// internal: cLN on a (B, C, pitch) tensor with `frames` valid columns (in place allowed); scratch double[B][frames][2]
int ctn_cln_pitch_fwd(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int frames, int pitch,
                      float eps, double* scratch, cudaStream_t st) {
  k_cln_step<<<dim3((frames + 127) / 128, B), 128, 0, st>>>(x, C, frames, pitch, scratch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  k_cln_scan<<<B, 1024, 0, st>>>(scratch, frames);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  int gy = C < 64 ? C : 64;
  k_cln_apply<<<dim3((pitch + 127) / 128, gy, B), 128, 0, st>>>(x, gamma, beta, y, C, frames, pitch, eps, scratch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_cln_fwd(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int T,
                           float eps, double* scratch, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !gamma || !beta || !y || !scratch || B <= 0 || C <= 0 || T <= 0) return CTN_EINVAL;
  return ctn_cln_pitch_fwd(x, gamma, beta, y, B, C, T, T, eps, scratch, (cudaStream_t)stream);
}
