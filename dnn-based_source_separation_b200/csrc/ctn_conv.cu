// Plain depthwise-separable convolution of src/modules/conv.py:13-29 (DepthwiseSeparableConv1d: depthwise Conv1d(groups = C,
// kernel K, stride, padding, dilation, bias) followed by a pointwise 1x1 Conv1d with bias).  Not on Conv-TasNet's hot path
// (SURVEY.md 8a row a11'); exposed for API completeness.  The depthwise stage is an HBM-bound streaming kernel; the pointwise
// stage reuses the dense-contraction kernels of the path (wgmma or FFMA, selected by `math`) on the padded layout.
#include <string.h>
#include "ctn_internal.h"

namespace {
// y[b][c][to] = bias[c] + sum_k w[c][k] * xpad[b][c][to*stride + k*dilation - padding]   (zeros outside [0, T))
__global__ void __launch_bounds__(256) k_depthwise1d(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                     float* __restrict__ y, int C, int T, int To, int K, int stride, int padding, int dilation,
                                                     int y_pitch) {
  const int c = blockIdx.y, b = blockIdx.z;
  const float* xr = x + ((size_t)b * C + c) * T;
  float* yr = y + ((size_t)b * C + c) * y_pitch;
  const float bv = bias ? bias[c] : 0.f;
  for (int to = blockIdx.x * blockDim.x + threadIdx.x; to < y_pitch; to += gridDim.x * blockDim.x) {
    float acc = 0.f;
    if (to < To) {
      acc = bv;
      for (int k = 0; k < K; ++k) {
        const int t = to * stride + k * dilation - padding;
        if (t >= 0 && t < T) acc = fmaf(w[c * K + k], xr[t], acc);
      }
    }
    yr[to] = acc;  // columns [To, y_pitch) are written as zero (padded-layout invariant)
  }
}
}  // namespace

extern "C" int ctn_depthwise_conv1d_fwd(const float* x, const float* w, const float* bias, float* y, int B, int C, int T, int K, int stride,
                                        int padding, int dilation, int y_pitch, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !w || !y || B <= 0 || C <= 0 || T <= 0 || K <= 0 || stride <= 0 || padding < 0 || dilation <= 0) return CTN_EINVAL;
  const int span = dilation * (K - 1) + 1;
  if (T + 2 * padding < span) return CTN_EINVAL;
  const int To = (T + 2 * padding - span) / stride + 1;
  if (y_pitch < To) return CTN_EINVAL;
  if (C > 65535 || B > 65535) return CTN_EUNSUPPORTED;
  int gx = (y_pitch + 255) / 256;
  if (gx > 64) gx = 64;
  k_depthwise1d<<<dim3(gx, C, B), 256, 0, (cudaStream_t)stream>>>(x, w, bias, y, C, T, To, K, stride, padding, dilation, y_pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// Pointwise Conv1d(K -> M, kernel 1) with optional bias on a PADDED-layout input: x (B,K,pitch) with `frames` valid columns,
// y (B,M,frames) contiguous.  workspace: (B*M*pitch floats) + ctn_stage_workspace_bytes(M, K).
extern "C" int ctn_pointwise_conv1d_fwd(const float* x, const float* W, const float* bias, float* y, int B, int M, int K, int frames,
                                        int pitch, int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !W || !y || !workspace || B <= 0 || M <= 0 || K <= 0 || frames <= 0) return CTN_EINVAL;
  if (pitch < frames || pitch % CTN_TILE_T != 0 || (((uintptr_t)workspace) & 255)) return CTN_EALIGN;
  if (((uintptr_t)x) & 15) return CTN_EALIGN;  // 128-bit operand loads
  const size_t ybytes = ((size_t)B * M * pitch * sizeof(float) + 255) & ~(size_t)255;
  const size_t wbytes = math != CTN_MATH_FP32 ? ctn_pw_wimg_bytes(M, K, math) + 256 : 0;
  if (workspace_bytes < ybytes + wbytes + (size_t)B * 2 * sizeof(double) + 512) return CTN_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  float* yp = (float*)workspace;
  float* wimg = (float*)((char*)workspace + ybytes);
  double* stats = (double*)((char*)workspace + ybytes + ((wbytes + 255) & ~(size_t)255));
  PwArgs a;
  memset(&a, 0, sizeof(a));
  a.A = x; a.W = W; a.D = yp; a.B = B; a.M = M; a.K = K; a.frames = frames; a.pitch = pitch;
  int epi = EPI_RAW;
  if (bias) {  // bias add = the EPI_H epilogue with a PReLU slope of 1 (identity); its statistics go to scratch
    const float* one = ctn_device_one();
    if (!one) return CTN_ENOTBUILT;
    cudaError_t e = cudaMemsetAsync(stats, 0, sizeof(double) * 2 * B, st);
    if (e != cudaSuccess) return (int)e;
    a.bias = bias; a.slope = one; a.stats_out = stats;
    epi = EPI_H;
  }
  CTN_TRY(ctn_pw(a, PRO_NONE, epi, math, wimg, st));  // arbitrary operand magnitudes, no operand scale: tf32 pieces in f16x3
  return ctn_copy_from_pitch(yp, y, B * M, frames, pitch, st);
}
