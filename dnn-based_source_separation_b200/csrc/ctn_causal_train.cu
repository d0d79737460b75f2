// Depthwise convolution of the causal (cLN) training path: the forward that keeps its pre-activation and normalises its input
// on load, and the backward.  All of the padding sits on the left (src/models/tdcn.py:125-127): pad_left = (P - 1) dil, so
// tap k of output frame t reads input frame t - (P - 1 - k) dil, never a later one.
//
// cLN statistics differ per frame, so the normalised input hn = cLN1(PReLU(h_pre)) is rebuilt from the (mean_t, 1/(std_t+eps))
// table the forward's scan left behind (k_cln_scan, ctn_norm.cu), in the expression every cLN forward evaluates (cln_affine).
// Layout (B, C, pitch) as in ctn_train.cu; pad columns are written as zero.
#include "ctn_internal.h"

namespace {

// u_pre[c][t] = bd[c] + sum_k wd[c][k] hn[c][t + k dil - pad_left], hn = 0 before frame 0.  Taps in the order of the inference
// kernel (k_dw_plain, ctn_causal.cu), which applies the PReLU this one leaves to its consumers.
__global__ void __launch_bounds__(256) k_cdw_train_fwd(const float* __restrict__ hpre, float* __restrict__ upre,
                                                       const float2* __restrict__ mi, const float* __restrict__ g1,
                                                       const float* __restrict__ b1, const float* __restrict__ wd,
                                                       const float* __restrict__ bd, const float* __restrict__ slope1, int C,
                                                       int frames, int pitch, int P, int dil) {
  const int b = blockIdx.y, pad_left = (P - 1) * dil;
  const float a1 = slope1[0];
  const float2* mb = mi + (size_t)b * frames;
  for (int c = blockIdx.x; c < C; c += gridDim.x) {
    const float* h = hpre + ((size_t)b * C + c) * pitch;
    float* u = upre + ((size_t)b * C + c) * pitch;
    const float gc = g1[c], bc = b1[c], bias = bd[c];
    for (int t = threadIdx.x; t < pitch; t += 256) {
      float acc = 0.f;
      if (t < frames) {
        acc = bias;
        for (int k = 0; k < P; ++k) {
          const int tt = t + k * dil - pad_left;
          if (tt >= 0 && tt < frames) acc = fmaf(wd[c * P + k], cln_affine(prelu_f(h[tt], a1), mb[tt], gc, bc), acc);
        }
      }
      u[t] = acc;
    }
  }
}

// dU = d_u_pre:   d_hn[c][t] = sum_k wd[c][k] dU[c][t - k dil + pad_left]     (zero beyond the last frame)
//                 dwd[c][k] += sum_{b,t} dU[c][t] hn[c][t + k dil - pad_left]  (hn = 0 before frame 0)
// A dilation beyond the frame count leaves only tap P - 1 inside.  grid (C, B)
__global__ void __launch_bounds__(256) k_cdw_bwd(const float* __restrict__ dupre, const float* __restrict__ hpre,
                                                 float* __restrict__ dhn, const float2* __restrict__ mi,
                                                 const float* __restrict__ g1, const float* __restrict__ b1,
                                                 const float* __restrict__ slope1, const float* __restrict__ wd,
                                                 float* __restrict__ dwd, int C, int frames, int pitch, int P, int dil) {
  __shared__ float part[8][CTN_MAX_P];
  const int c = blockIdx.x, b = blockIdx.y, pad_left = (P - 1) * dil;
  const float a1 = slope1[0], gc = g1[c], bc = b1[c];
  const float2* mb = mi + (size_t)b * frames;
  const float* du = dupre + ((size_t)b * C + c) * pitch;
  const float* h = hpre + ((size_t)b * C + c) * pitch;
  float* o = dhn + ((size_t)b * C + c) * pitch;
  float w[CTN_MAX_P], acc[CTN_MAX_P];
#pragma unroll
  for (int k = 0; k < CTN_MAX_P; ++k) { w[k] = k < P ? wd[c * P + k] : 0.f; acc[k] = 0.f; }
  for (int t = threadIdx.x; t < pitch; t += 256) {
    float v = 0.f;
    if (t < frames) {
      const float dut = du[t];
#pragma unroll
      for (int k = 0; k < CTN_MAX_P; ++k) {
        if (k < P) {
          const int off = pad_left - k * dil;  // >= 0
          if (off < frames - t) v = fmaf(w[k], du[t + off], v);  // u[t + off] read hn[t] through tap k
          if (t >= off) acc[k] = fmaf(dut, cln_affine(prelu_f(h[t - off], a1), mb[t - off], gc, bc), acc[k]);
        }
      }
    }
    o[t] = v;
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < CTN_MAX_P; ++k) {
    if (k < P) {
      const float s = warp_sum(acc[k]);
      if (lane == 0) part[wid][k] = s;
    }
  }
  __syncthreads();
  if (threadIdx.x < P) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < 8; ++q) s += (double)part[q][threadIdx.x];
    atomicAdd(&dwd[c * P + threadIdx.x], (float)s);
  }
}

}  // namespace

int ctn_cdw_train_fwd(const float* hpre, float* upre, const float2* mi, const float* g1, const float* b1, const float* wd,
                      const float* bd, const float* slope1, int B, int C, int frames, int pitch, int P, int dil, cudaStream_t st) {
  k_cdw_train_fwd<<<grid_cb(C, B), 256, 0, st>>>(hpre, upre, mi, g1, b1, wd, bd, slope1, C, frames, pitch, P, dil);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int ctn_cdw_bwd(const float* dupre, const float* hpre, float* dhn, const float2* mi, const float* g1, const float* b1,
                const float* slope1, const float* wd, float* dwd, int B, int C, int frames, int pitch, int P, int dil,
                cudaStream_t st) {
  if (P > CTN_MAX_P) return CTN_EUNSUPPORTED;
  k_cdw_bwd<<<dim3(C, B), 256, 0, st>>>(dupre, hpre, dhn, mi, g1, b1, slope1, wd, dwd, C, frames, pitch, P, dil);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
