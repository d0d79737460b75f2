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
// x rows are `pitch` floats apart (pitch == T for PyTorch-contiguous tensors, the padded pitch inside the fused forward).
// slope (nullable) in every kernel below: the normalised tensor is PReLU(x; slope), applied on load.
__global__ void __launch_bounds__(128) k_cln_step(const float* __restrict__ x, const float* __restrict__ slope, int C, int T, int pitch,
                                                  double* __restrict__ st) {
  const int b = blockIdx.y, t = blockIdx.x * 128 + threadIdx.x;
  if (t >= T) return;
  const float* xb = x + (size_t)b * C * pitch + t;
  const bool act = slope != nullptr;
  const float a = act ? slope[0] : 1.f;
  double s = 0.0, ss = 0.0;
  for (int c = 0; c < C; ++c) {
    float xf = xb[(size_t)c * pitch];
    if (act) xf = prelu_f(xf, a);
    const double v = (double)xf;
    s += v;
    ss += v * v;
  }
  st[((size_t)b * T + t) * 2] = s;
  st[((size_t)b * T + t) * 2 + 1] = ss;
}

// Inclusive scan along t of `st` (B, T, 2), one block (1024 threads) per sample.  A thread owns `per` consecutive frames; the
// scan over threads is shared by the forward scan and the backward's reverse scan (which walks the frames last to first).
__device__ __forceinline__ void cln_scan_base(double& s, double& ss, double (*wsum)[32]) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
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
  s = (ps - s) + (wid > 0 ? wsum[0][wid - 1] : 0.0);
  ss = (pss - ss) + (wid > 0 ? wsum[1][wid - 1] : 0.0);
}

// mi (nullable): (B, T) table of (mean_t, 1 / (std_t + eps)) for kernels that normalise on load (the causal training depthwise)
__global__ void __launch_bounds__(1024) k_cln_scan(double* __restrict__ st, int T, float2* __restrict__ mi, int C, float eps) {
  __shared__ double wsum[2][32];
  const int b = blockIdx.x, tid = threadIdx.x;
  double* sb = st + (size_t)b * T * 2;
  const int per = (T + 1023) / 1024;
  const int t0 = tid * per, t1 = min(T, t0 + per);
  double s = 0.0, ss = 0.0;
  for (int t = t0; t < t1; ++t) { s += sb[2 * t]; ss += sb[2 * t + 1]; }
  cln_scan_base(s, ss, wsum);
  double base_s = s, base_ss = ss;
  for (int t = t0; t < t1; ++t) {
    base_s += sb[2 * t];
    base_ss += sb[2 * t + 1];
    sb[2 * t] = base_s;
    sb[2 * t + 1] = base_ss;
    if (mi) mi[(size_t)b * T + t] = cln_mean_inv(sb + 2 * t, (double)C * (double)(t + 1), eps);
  }
}

// y may alias x.  Columns [T, pitch) of y are written as zero (padded layout).
__global__ void __launch_bounds__(128) k_cln_apply(const float* x, const float* __restrict__ slope, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, float* y, int C, int T, int pitch,
                                                   float eps, const double* __restrict__ st) {
  const int b = blockIdx.z, t = blockIdx.x * 128 + threadIdx.x;
  if (t >= pitch) return;
  if (t >= T) {
    for (int c = blockIdx.y; c < C; c += gridDim.y) y[((size_t)b * C + c) * pitch + t] = 0.f;
    return;
  }
  const float2 mi = cln_mean_inv(st + ((size_t)b * T + t) * 2, (double)C * (double)(t + 1), eps);
  const bool act = slope != nullptr;
  const float a = act ? slope[0] : 1.f;
  for (int c = blockIdx.y; c < C; c += gridDim.y) {
    const size_t i = ((size_t)b * C + c) * pitch + t;
    const float xv = act ? prelu_f(x[i], a) : x[i];
    y[i] = cln_affine(xv, mi, gamma[c], beta[c]);
  }
}

int ctn_cln_stats(const float* x, const float* slope, int B, int C, int frames, int pitch, float eps, double* st, float2* mi,
                  cudaStream_t stream) {
  k_cln_step<<<dim3((frames + 127) / 128, B), 128, 0, stream>>>(x, slope, C, frames, pitch, st);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  k_cln_scan<<<B, 1024, 0, stream>>>(st, frames, mi, C, eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int ctn_cln_apply(const float* x, const float* slope, const float* gamma, const float* beta, float* y, int B, int C, int frames,
                  int pitch, float eps, const double* st, cudaStream_t stream) {
  const int gy = C < 64 ? C : 64;
  k_cln_apply<<<dim3((pitch + 127) / 128, gy, B), 128, 0, stream>>>(x, slope, gamma, beta, y, C, frames, pitch, eps, st);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// internal: cLN on a (B, C, pitch) tensor with `frames` valid columns (in place allowed); scratch double[B][frames][2]
int ctn_cln_pitch_fwd(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int frames, int pitch,
                      float eps, double* scratch, cudaStream_t st) {
  CTN_TRY(ctn_cln_stats(x, nullptr, B, C, frames, pitch, eps, scratch, nullptr, st));
  return ctn_cln_apply(x, nullptr, gamma, beta, y, B, C, frames, pitch, eps, scratch, st);
}

extern "C" int ctn_cln_fwd(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int T,
                           float eps, double* scratch, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !gamma || !beta || !y || !scratch || B <= 0 || C <= 0 || T <= 0) return CTN_EINVAL;
  return ctn_cln_pitch_fwd(x, gamma, beta, y, B, C, T, T, eps, scratch, (cudaStream_t)stream);
}

// ---- cLN backward.  With n_t = C (t + 1), m_t = S_t / n_t, v_t = Q_t / n_t - m_t^2, s_t = sqrt(max(v_t, 0)), r_t = 1 / (s_t + eps),
// x = PReLU(pre) (or pre), y = (x - m_t) r_t gamma_c + beta_c and g = dy gamma_c:
//   a_t = sum_c g            b_t = sum_c g (x - m_t)           e_t = dL/dv_t = -r_t^2 b_t / (2 s_t)
//   dS_t = (-r_t a_t - 2 m_t e_t) / n_t     dQ_t = e_t / n_t    U_tau = sum_{t >= tau} dS_t    V_tau = sum_{t >= tau} dQ_t
//   dx[c][tau] = g r_tau + U_tau + 2 x V_tau        dgamma_c = sum dy (x - m_t) r_t        dbeta_c = sum dy
// Where the forward clamped v_t to 0 the derivative of the square root does not exist (the reference's autograd yields
// inf / NaN there); e_t = 0 is taken for those frames: the clamped variance is a constant.
// Phase 1: per frame (sum_c g, sum_c g x) in double -- the products of two floats are exact there, and b_t = sum g x - m_t a_t is
// formed in the scan, so this pass needs no statistics.  The channels are cut into CLN_BWD_SLICES strided slices, one thread per
// (slice, frame) summing its channels in order; the scan adds the slices in order: deterministic.
#define CLN_BWD_SLICES 8
__global__ void __launch_bounds__(128) k_cln_bwd_sums(const float* __restrict__ dy, const float* __restrict__ pre,
                                                      const float* __restrict__ slope, const float* __restrict__ gamma, int C, int T,
                                                      int pitch, double* __restrict__ part) {
  const int b = blockIdx.z, s = blockIdx.y, t = blockIdx.x * 128 + threadIdx.x;
  if (t >= T) return;
  const bool act = slope != nullptr;
  const float a = act ? slope[0] : 1.f;
  double sa = 0.0, sb = 0.0;
#pragma unroll 4
  for (int c = s; c < C; c += gridDim.y) {
    const size_t i = ((size_t)b * C + c) * pitch + t;
    const float g = dy[i] * gamma[c];
    const float xv = act ? prelu_f(pre[i], a) : pre[i];
    sa += (double)g;
    sb = fma((double)g, (double)xv, sb);
  }
  double* o = part + (((size_t)b * gridDim.y + s) * T + t) * 2;
  o[0] = sa;
  o[1] = sb;
}

// Phase 2: (dS_t, dQ_t) per frame and their suffix sums, one block per sample: the forward scan run over the frames in reverse.
// tab[b][t] = (m_t, r_t, U_t, V_t) as floats for the apply kernel; the sums themselves stay in double.  Slice 0 of `part` is
// reused to hold (dS_t, dQ_t) between the two passes.
__global__ void __launch_bounds__(1024) k_cln_bwd_scan(const double* __restrict__ st, double* __restrict__ part, int slices,
                                                       float4* __restrict__ tab, int C, int T, float eps) {
  __shared__ double wsum[2][32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const double* sb = st + (size_t)b * T * 2;
  double* pb = part + (size_t)b * slices * T * 2;
  const int per = (T + 1023) / 1024;
  const int j0 = tid * per, j1 = min(T, j0 + per);  // reversed frame index j = T - 1 - t
  double s = 0.0, ss = 0.0;
  for (int j = j0; j < j1; ++j) {
    const int t = T - 1 - j;
    double at = 0.0, bx = 0.0;
    for (int q = 0; q < slices; ++q) { at += pb[((size_t)q * T + t) * 2]; bx += pb[((size_t)q * T + t) * 2 + 1]; }
    const double n = (double)C * (double)(t + 1);
    const double mean = sb[2 * t] / n, var = sb[2 * t + 1] / n - mean * mean;
    const double sd = var > 0.0 ? sqrt(var) : 0.0, r = 1.0 / (sd + (double)eps);
    const double e = var > 0.0 ? -r * r * (bx - mean * at) / (2.0 * sd) : 0.0;
    const double dS = (-r * at - 2.0 * mean * e) / n, dQ = e / n;
    pb[2 * t] = dS;
    pb[2 * t + 1] = dQ;
    s += dS;
    ss += dQ;
  }
  cln_scan_base(s, ss, wsum);
  for (int j = j0; j < j1; ++j) {
    const int t = T - 1 - j;
    s += pb[2 * t];
    ss += pb[2 * t + 1];
    const float2 mi = cln_mean_inv(sb + 2 * t, (double)C * (double)(t + 1), eps);
    tab[(size_t)b * T + t] = make_float4(mi.x, mi.y, (float)s, (float)ss);
  }
}

// Phase 3: dx, and with a slope the PReLU backward behind it: d_pre = dx (pre > 0 ? 1 : a), dslope += sum_{pre <= 0} dx pre,
// dbias[c] += sum d_pre (the bias of the conv that produced `pre`).  dgamma, dbeta += per-row sums.  dpre may alias dy (a thread
// loads its four frames before it stores them).  Columns [T, pitch) of dpre are written as zero.  grid (C, B)
__global__ void __launch_bounds__(256) k_cln_bwd_apply(const float* dy, const float* __restrict__ pre, float* dpre,
                                                       const float* __restrict__ slope, const float* __restrict__ gamma,
                                                       const float4* __restrict__ tab, float* __restrict__ dgamma,
                                                       float* __restrict__ dbeta, float* __restrict__ dslope,
                                                       float* __restrict__ dbias, int C, int T, int pitch) {
  __shared__ double red[2][64];
  const int c = blockIdx.x, b = blockIdx.y;
  const bool act = slope != nullptr;
  const float a = act ? slope[0] : 1.f;
  const float gc = gamma[c];
  const float* d = dy + ((size_t)b * C + c) * pitch;
  const float* p = pre + ((size_t)b * C + c) * pitch;
  float* o = dpre + ((size_t)b * C + c) * pitch;
  const float4* tb = tab + (size_t)b * T;
  // 128-bit row access on the padded layout; a PyTorch-contiguous tensor (pitch == T, any T) may not allow it
  const bool vec = (pitch & 3) == 0 && (((uintptr_t)dy | (uintptr_t)pre | (uintptr_t)dpre) & 15) == 0;
  float sg = 0.f, sbt = 0.f, sa = 0.f, sbi = 0.f;
  for (int t = threadIdx.x * 4; t < pitch; t += 1024) {
    float ov[4] = {0.f, 0.f, 0.f, 0.f};
    if (t < T) {
      float dvv[4], pvv[4];
      if (vec) {
        const float4 dv = ld4(d + t), pv = ld4(p + t);
        dvv[0] = dv.x; dvv[1] = dv.y; dvv[2] = dv.z; dvv[3] = dv.w;
        pvv[0] = pv.x; pvv[1] = pv.y; pvv[2] = pv.z; pvv[3] = pv.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          dvv[j] = t + j < T ? d[t + j] : 0.f;
          pvv[j] = t + j < T ? p[t + j] : 0.f;
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (t + j < T) {
          const float4 q = tb[t + j];
          const float x = act ? prelu_f(pvv[j], a) : pvv[j];
          const float dx = fmaf(dvv[j] * gc, q.y, fmaf(2.f * x, q.w, q.z));
          sg = fmaf(dvv[j], (x - q.x) * q.y, sg);
          sbt += dvv[j];
          float r = dx;
          if (act) {
            r = pvv[j] > 0.f ? dx : a * dx;
            if (!(pvv[j] > 0.f)) sa = fmaf(dx, pvv[j], sa);
          }
          ov[j] = r;
          sbi += r;
        }
      }
    }
    if (vec) {
      st4(o + t, make_float4(ov[0], ov[1], ov[2], ov[3]));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (t + j < pitch) o[t + j] = ov[j];
    }
  }
  double d0 = sg, d1 = sbt;
  block_sum2_d(d0, d1, red[0]);
  if (threadIdx.x == 0) {
    atomicAdd(&dgamma[c], (float)d0);
    atomicAdd(&dbeta[c], (float)d1);
  }
  if (dslope || dbias) {
    double d2 = sa, d3 = sbi;
    block_sum2_d(d2, d3, red[1]);
    if (threadIdx.x == 0) {
      if (act && dslope) atomicAdd(dslope, (float)d2);
      if (dbias) atomicAdd(&dbias[c], (float)d3);
    }
  }
}

size_t ctn_cln_bwd_part_doubles(int B, int frames) { return (size_t)B * CLN_BWD_SLICES * frames * 2; }

// 3 launches
int ctn_cln_bwd_pitch(const float* dy, const float* pre, float* dpre, const float* slope, const float* gamma, const double* st,
                      float eps, double* part, float4* tab, float* dgamma, float* dbeta, float* dslope, float* dbias, int B, int C,
                      int frames, int pitch, cudaStream_t stream) {
  const int slices = C < CLN_BWD_SLICES ? C : CLN_BWD_SLICES;
  k_cln_bwd_sums<<<dim3((frames + 127) / 128, slices, B), 128, 0, stream>>>(dy, pre, slope, gamma, C, frames, pitch, part);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  k_cln_bwd_scan<<<B, 1024, 0, stream>>>(st, part, slices, tab, C, frames, eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  k_cln_bwd_apply<<<dim3(C, B), 256, 0, stream>>>(dy, pre, dpre, slope, gamma, tab, dgamma, dbeta, dslope, dbias, C, frames, pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_cln_bwd(const float* dy, const float* x, const float* gamma, void* scratch, float* dx, float* dgamma,
                           float* dbeta, int B, int C, int T, float eps, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!dy || !x || !gamma || !scratch || !dx || !dgamma || !dbeta || B <= 0 || C <= 0 || T <= 0) return CTN_EINVAL;
  if (((uintptr_t)scratch) & 15) return CTN_EALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  double* stq = static_cast<double*>(scratch);
  double* part = stq + (size_t)B * T * 2;
  float4* tab = reinterpret_cast<float4*>(part + ctn_cln_bwd_part_doubles(B, T));
  CTN_TRY(ctn_cln_stats(x, nullptr, B, C, T, T, eps, stq, nullptr, st));
  return ctn_cln_bwd_pitch(dy, x, dx, nullptr, gamma, stq, eps, part, tab, dgamma, dbeta, nullptr, nullptr, B, C, T, T, st);
}
