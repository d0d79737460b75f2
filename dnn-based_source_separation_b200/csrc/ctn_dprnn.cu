// DPRNN-TasNet data-movement kernels (BASELINE cfg4): segmentation, overlap-add and the gLN + residual (+ intra/inter
// permute) step of a dual-path block.  Reference: src/models/transform.py:6-65 (Segment1d / OverlapAdd1d),
// src/models/dprnn_tasnet.py:335-351 (pad -> segment -> dprnn -> overlap-add -> crop), src/models/dprnn.py:82-94, 134-148
// (permute -> LSTM -> Linear -> permute -> gLN -> permute -> + residual).
//
// All of it is HBM-bound gather / scatter work (no arithmetic worth a tensor core).  The dual-path state is kept
// CHANNELS-LAST, Z (B, D1, D2, F) with F contiguous: that is exactly the (batch*D1, D2, F) batch_first tensor the LSTM of
// the current path consumes (intra: D1 = S chunks, D2 = K frames; inter: D1 = K, D2 = S), so the reference's four
// permute().contiguous() copies per block disappear -- the D1 <-> D2 swap for the other path is folded into the store
// indexing of the gLN + residual kernel, which moves whole F-vectors (F*4 bytes contiguous) per (d1, d2) cell.
#include "ctn_internal.h"

namespace {

// ---- segmentation ---------------------------------------------------------------------------------------------------
// xp = zero-pad(x, pad_left, .) (dprnn_tasnet.py:339-345); chunk s covers padded frames [s*P, s*P + K) (transform.py:25).
// channels-last (layout 1): Z[b][s][k][f].
// grid (ceil(Tp/32), ceil(F/32), B), block (32, 8): a 32 (frames) x 32 (channels) tile is transposed through shared memory
// so that both the reads (frames contiguous) and the channels-last writes (channels contiguous) are coalesced.
__global__ void __launch_bounds__(256) k_segment_cl(const float* __restrict__ x, float* __restrict__ Z, int F, int frames, int pitch,
                                                    int pad_left, int S, int K, int P, int Tp) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, f0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int f = f0 + j, tp = t0 + threadIdx.x, t = tp - pad_left;
    tile[j][threadIdx.x] = (f < F && t >= 0 && t < frames) ? x[((size_t)b * F + f) * pitch + t] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int tp = t0 + j, f = f0 + threadIdx.x;
    if (tp >= Tp || f >= F) continue;
    const float v = tile[threadIdx.x][j];
    // chunks covering padded frame tp: s in [ceil((tp-K+1)/P), floor(tp/P)] clipped to [0, S)
    int s_hi = tp / P;
    if (s_hi > S - 1) s_hi = S - 1;
    for (int s = s_hi; s >= 0 && s * P + K > tp; --s) Z[(((size_t)b * S + s) * K + (tp - s * P)) * F + f] = v;
  }
}
// channel-first (rows of z_pitch >= S K): Z[b][f][s K + k] = xp[b][f][s P + k], columns [S K, z_pitch) = 0.  grid
// (ceil(z_pitch / 256), min(B F, 65535)), the (b, f) rows strided over y, so no channel count is refused.
__global__ void __launch_bounds__(256) k_segment_cf(const float* __restrict__ x, float* __restrict__ Z, long long BF, int frames, int pitch,
                                                    int pad_left, int S, int K, int P, long long z_pitch) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= z_pitch) return;
  for (long long bf = blockIdx.y; bf < BF; bf += gridDim.y) {
    float v = 0.f;
    if (i < (long long)S * K) {
      const int s = (int)(i / K), k = (int)(i % K), tt = s * P + k - pad_left;
      if (tt >= 0 && tt < frames) v = __ldg(x + bf * pitch + tt);
    }
    Z[bf * z_pitch + i] = v;
  }
}

// ---- overlap-add (+ crop) -------------------------------------------------------------------------------------------
// y[b][f][t] = sum_{s : s*P <= tp < s*P + K} Z[b][s][tp - s*P][f],  tp = t + crop_left  (transform.py:58-62, F.fold sums
// the overlapping chunks in increasing s; dprnn_tasnet.py:347 crops the padding).  Columns [T_out, out_pitch) are zeroed.
__global__ void __launch_bounds__(256) k_overlap_add_cl(const float* __restrict__ Z, float* __restrict__ y, int F, int S, int K, int P,
                                                        int crop_left, int T_out, int out_pitch) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, f0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int t = t0 + j, f = f0 + threadIdx.x;
    float acc = 0.f;
    if (t < T_out && f < F) {
      const int tp = t + crop_left;
      int s_lo = (tp - K + P) / P;  // ceil((tp - K + 1) / P) for tp - K + 1 > 0
      if (tp - K + 1 <= 0) s_lo = 0;
      int s_hi = tp / P;
      if (s_hi > S - 1) s_hi = S - 1;
      for (int s = s_lo; s <= s_hi; ++s) acc += Z[(((size_t)b * S + s) * K + (tp - s * P)) * F + f];
    }
    tile[j][threadIdx.x] = acc;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int f = f0 + j, t = t0 + threadIdx.x;
    if (f < F && t < out_pitch) y[((size_t)b * F + f) * out_pitch + t] = t < T_out ? tile[threadIdx.x][j] : 0.f;
  }
}
// channel-first: chunk s of row (b, f) at Z[b][f][s K .. s K + K) of a z_pitch row; grid as k_segment_cf over out_pitch
__global__ void __launch_bounds__(256) k_overlap_add_cf(const float* __restrict__ Z, float* __restrict__ y, long long BF, int S, int K, int P,
                                                        long long z_pitch, int crop_left, int T_out, int out_pitch) {
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= out_pitch) return;
  for (long long bf = blockIdx.y; bf < BF; bf += gridDim.y) {
    float acc = 0.f;
    if (t < T_out) {
      const int tp = t + crop_left;
      int s_lo = (tp - K + 1 <= 0) ? 0 : (tp - K + P) / P;
      int s_hi = tp / P;
      if (s_hi > S - 1) s_hi = S - 1;
      const float* z = Z + bf * z_pitch;
      for (int s = s_lo; s <= s_hi; ++s) acc += __ldg(z + (size_t)s * K + tp - s * P);
    }
    y[bf * out_pitch + t] = acc;
  }
}

// ---- gLN + residual (+ path swap) -----------------------------------------------------------------------------------
// Y, R: (B, D1, D2, F) channels-last.  gLN statistics per sample over all D1*D2*F values (GroupNorm(1, F), norm.py:18):
//   out[b][..][f] = (Y - mean_b) * rstd_b * gamma[f] + beta[f] + R
// swap = 1 writes out as (B, D2, D1, F) -- the layout of the OTHER path (dprnn.py:91-92 / 144-146 fold into this store).
__global__ void __launch_bounds__(256) k_sample_stats(const float* __restrict__ Y, size_t n, double* __restrict__ stats) {
  __shared__ double red[64];
  const int b = blockIdx.y;
  const float4* p = reinterpret_cast<const float4*>(Y + (size_t)b * n);
  // 128-bit loads only when every sample starts 16-byte aligned (Y is; sample b sits b*n floats further): else all scalar
  const size_t n4 = (n & 3) ? 0 : n / 4;
  double s = 0.0, ss = 0.0;
  // every element in double before it is added: fp32 partials lose the variance under a DC offset
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x; i0 < n4; i0 += (size_t)gridDim.x * blockDim.x * 4) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const size_t i = i0 + (size_t)u * gridDim.x * blockDim.x + threadIdx.x;
      if (i < n4) {
        const float4 v = __ldg(p + i);
        const double x = v.x, y = v.y, z = v.z, w = v.w;
        s += (x + y) + (z + w);
        ss = fma(x, x, fma(y, y, fma(z, z, fma(w, w, ss))));
      }
    }
  }
  for (size_t i = n4 * 4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = Y[(size_t)b * n + i];
    s += v;
    ss += (double)v * v;
  }
  block_sum2_d(s, ss, red);
  if (threadIdx.x == 0) { atomicAdd(&stats[2 * b], s); atomicAdd(&stats[2 * b + 1], ss); }
}

// one warp per (d1, d2) cell: F-vector in, F-vector out (F % 4 == 0: 128-bit accesses)
__global__ void __launch_bounds__(256) k_norm_res(const float* __restrict__ Y, const float* __restrict__ R, const float* __restrict__ gamma,
                                                  const float* __restrict__ beta, float* __restrict__ out, const double* __restrict__ stats,
                                                  int D1, int D2, int F, float eps, int swap) {
  const int b = blockIdx.y;
  const float2 mr = gln_mean_rstd(stats + 2 * b, (double)D1 * (double)D2 * (double)F, eps);
  const size_t cells = (size_t)D1 * D2;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const bool vec = (F & 3) == 0;
  for (size_t c = (size_t)blockIdx.x * wpb + (threadIdx.x >> 5); c < cells; c += (size_t)gridDim.x * wpb) {
    const int d1 = (int)(c / D2), d2 = (int)(c % D2);
    const size_t src = ((size_t)b * cells + c) * F;
    const size_t dst = swap ? (((size_t)b * D2 + d2) * D1 + d1) * F : src;
    if (vec) {
      for (int f = lane * 4; f < F; f += 128) {
        const float4 y = __ldg(reinterpret_cast<const float4*>(Y + src + f)), r = __ldg(reinterpret_cast<const float4*>(R + src + f));
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + f)), be = __ldg(reinterpret_cast<const float4*>(beta + f));
        float4 o;
        o.x = fmaf((y.x - mr.x) * mr.y, g.x, be.x) + r.x;
        o.y = fmaf((y.y - mr.x) * mr.y, g.y, be.y) + r.y;
        o.z = fmaf((y.z - mr.x) * mr.y, g.z, be.z) + r.z;
        o.w = fmaf((y.w - mr.x) * mr.y, g.w, be.w) + r.w;
        *reinterpret_cast<float4*>(out + dst + f) = o;
      }
    } else {
      for (int f = lane; f < F; f += 32) out[dst + f] = fmaf((Y[src + f] - mr.x) * mr.y, gamma[f], beta[f]) + R[src + f];
    }
  }
}

}  // namespace

// rows of the channel-first grid: (b, f) strided over at most 65535 CTAs of y
static unsigned cf_rows(long long BF) { return (unsigned)(BF < 65535 ? BF : 65535); }

// the row pitch a layout argument selects for S chunks of K frames: 0 for channels-last (1), S K for the dense channel-first
// layout (0), the argument itself from S K on; -1 for any other value
static long long row_pitch(int layout, int S, int K) {
  const long long n = (long long)S * K;
  if (layout == 1) return 0;
  if (layout == 0) return n;
  return layout >= n ? layout : -1;
}

extern "C" int ctn_segment_fwd(const float* x, float* Z, int B, int F, int frames, int pitch, int chunk_size, int hop_size,
                               int pad_left, int pad_right, int layout, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !Z || B <= 0 || F <= 0 || frames <= 0 || pitch < frames || chunk_size <= 0 || hop_size <= 0 || pad_left < 0 || pad_right < 0)
    return CTN_EINVAL;
  const int Tp = frames + pad_left + pad_right;
  if (Tp < chunk_size) return CTN_EINVAL;
  const int S = (Tp - chunk_size) / hop_size + 1;  // F.unfold drops a ragged tail (transform.py:21)
  const long long z_pitch = row_pitch(layout, S, chunk_size);
  if (z_pitch < 0) return CTN_EINVAL;
  if (B > 65535) return CTN_EUNSUPPORTED;  // the batch is the channels-last grid's z axis
  cudaStream_t st = (cudaStream_t)stream;
  if (!z_pitch) {
    const int Tc = (S - 1) * hop_size + chunk_size;  // frames that land in some chunk
    if (hop_size > chunk_size) {  // gaps between chunks: not every cell is written by the scatter below
      cudaError_t e = cudaMemsetAsync(Z, 0, sizeof(float) * (size_t)B * S * chunk_size * F, st);
      if (e != cudaSuccess) return (int)e;
    }
    k_segment_cl<<<dim3((Tc + 31) / 32, (F + 31) / 32, B), dim3(32, 8), 0, st>>>(x, Z, F, frames, pitch, pad_left, S, chunk_size, hop_size, Tc);
  } else {
    const long long BF = (long long)B * F;
    k_segment_cf<<<dim3((unsigned)((z_pitch + 255) / 256), cf_rows(BF)), 256, 0, st>>>(x, Z, BF, frames, pitch, pad_left, S, chunk_size, hop_size,
                                                                            z_pitch);
  }
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_overlap_add_fwd(const float* Z, float* y, int B, int F, int S, int chunk_size, int hop_size, int crop_left,
                                   int T_out, int out_pitch, int layout, ctn_stream_t stream) {
  LaunchScope scope(Z);
  if (!Z || !y || B <= 0 || F <= 0 || S <= 0 || chunk_size <= 0 || hop_size <= 0 || crop_left < 0 || T_out <= 0 || out_pitch < T_out)
    return CTN_EINVAL;
  if (crop_left + T_out > (S - 1) * hop_size + chunk_size) return CTN_EINVAL;
  const long long z_pitch = row_pitch(layout, S, chunk_size);
  if (z_pitch < 0) return CTN_EINVAL;
  if (B > 65535) return CTN_EUNSUPPORTED;  // the batch is the channels-last grid's z axis
  cudaStream_t st = (cudaStream_t)stream;
  if (!z_pitch) {
    k_overlap_add_cl<<<dim3((out_pitch + 31) / 32, (F + 31) / 32, B), dim3(32, 8), 0, st>>>(Z, y, F, S, chunk_size, hop_size, crop_left, T_out,
                                                                                        out_pitch);
  } else {
    const long long BF = (long long)B * F;
    k_overlap_add_cf<<<dim3((out_pitch + 255) / 256, cf_rows(BF)), 256, 0, st>>>(Z, y, BF, S, chunk_size, hop_size, z_pitch, crop_left, T_out,
                                                                                 out_pitch);
  }
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_dprnn_norm_res_fwd(const float* Y, const float* R, const float* gamma, const float* beta, float* out, int B, int D1,
                                      int D2, int F, float eps, int swap, double* scratch, ctn_stream_t stream) {
  LaunchScope scope(Y);
  if (!Y || !R || !gamma || !beta || !out || !scratch || B <= 0 || D1 <= 0 || D2 <= 0 || F <= 0) return CTN_EINVAL;
  if (B > 65535) return CTN_EUNSUPPORTED;  // the batch is the grid's y axis
  if (swap && (out == Y || out == R)) return CTN_EINVAL;  // the path swap cannot run in place
  if ((((uintptr_t)Y) | ((uintptr_t)R) | ((uintptr_t)out) | ((uintptr_t)gamma) | ((uintptr_t)beta)) & 15) return CTN_EALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * B, st);
  if (e != cudaSuccess) return (int)e;
  const size_t n = (size_t)D1 * D2 * F;
  int gx = (int)((n / 4 + 256 * 4 - 1) / (256 * 4));
  {  // ~8 resident blocks per SM over the WHOLE batch: longer per-thread streams, 2 double atomics per block on 2B addresses
    const int cap = 1184 / B > 1 ? 1184 / B : 1;
    if (gx > cap) gx = cap;
  }
  if (gx < 1) gx = 1;
  k_sample_stats<<<dim3(gx, B), 256, 0, st>>>(Y, n, scratch);
  CTN_COUNT_LAUNCH();
  const size_t cells = (size_t)D1 * D2;
  int gy = (int)((cells + 7) / 8);
  if (gy > 2368) gy = 2368;
  k_norm_res<<<dim3(gy, B), 256, 0, st>>>(Y, R, gamma, beta, out, scratch, D1, D2, F, eps, swap);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
