// LSTM-TasNet stages.  Reference: src/models/tasnet.py:146-189 (TasNet.extract_latent), :324-381 (Separator),
// src/models/filterbank.py:325-346 (GatedEncoder).
//
// Layout: every activation is CHANNEL-FIRST and pitched, (B, C, pitch) with pitch = ctn_pitch(frames), so each LSTM gate row is
// contiguous in time and every Linear is one ctn_pw contraction with the frames as columns.
//   * the gated encoder: ||x|| per sample in double (k_tas_sig_norm), then one CTA per tile of TAS_TF frames forms both
//     contractions, ReLU(U x) sigmoid(V x), and the frame norm over the N channels from the tile it keeps in shared memory.
//   * a bi-LSTM layer: the input projections W_ih x + b_ih + b_hh of both directions are one ctn_pw contraction (M = dirs 4H);
//     the recurrence is one cooperative launch (k_tas_lstm).  Each direction owns ceil(H / U) CTAs, CTA c owning hidden units
//     [c U, c U + U) with all four gates; its 4U rows of W_hh stay in shared memory in fp32 for the whole call.  Per step a CTA
//     reads h_{t-1} of its direction from a double-buffered global array, forms its gate rows with fp32 FMAs, adds the input
//     projection (prefetched TAS_PF steps ahead with cp.async), updates c (in a register of the owning thread) and h, publishes
//     its h slice and meets the other CTAs of its direction at a release / acquire counter barrier.  The two directions never
//     wait for each other.  Every sum has a fixed order: a repeated call gives the same bits.
//   * the tail: fc as ctn_pw with the sigmoid mask and w * mask in its epilogue, or its logits and a softmax over the SOURCES
//     (tasnet.py:312-316, nn.Softmax(dim=1) of (B, S, N, T')), then the transposed-conv decoder with the crop.
#include <math.h>
#include <string.h>

#include "ctn_internal.h"

namespace {

constexpr int TAS_TF = 8;        // frames per encoder / frame-norm CTA (one warp per frame in the norm)
constexpr int TAS_THREADS = 256;
constexpr int TAS_PF = 16;       // steps of input projection prefetched per tile
constexpr int TAS_GMAX = 16;     // most sequences one pass of the recurrence carries
constexpr int TAS_RB = 4, TAS_SB = 4;  // gate rows x sequences per warp register tile

__device__ const float k_tas_one = 1.f;  // the PReLU slope that makes the pro/epilogue PReLU of ctn_pw an identity

// ---- encoder ------------------------------------------------------------------------------------------------------------------
// nrm[b] = ||x_b||_2 over the T samples (zero padding adds nothing), summed in double, fixed reduction tree.  grid B, block 256.
__global__ void __launch_bounds__(256) k_tas_sig_norm(const float* __restrict__ x, double* __restrict__ nrm, int T) {
  __shared__ double red[64];
  const float* xb = x + (size_t)blockIdx.x * T;
  double s = 0.0, dummy = 0.0;
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    const double v = xb[i];
    s = fma(v, v, s);
  }
  block_sum2_d(s, dummy, red);
  if (threadIdx.x == 0) nrm[blockIdx.x] = sqrt(s);
}

// Per-frame norm of a tile wt[n][TAS_TF] held in shared memory (tasnet.py:356-359): warp f normalises frame f0 + f over the N
// channels, mean and then the centred variance in double (lanes stride the channels, fixed shuffle tree), so an all-zero frame
// gives exactly beta.  xn[b][n][f0 + f] = gamma_n (w - mean) / (sqrt(var) + eps) + beta_n; frames at or past `frames` get 0.
__device__ void tas_frame_norm_tile(const float* wt, const float* __restrict__ gamma, const float* __restrict__ beta, float* xn, int N,
                                    int f0, int frames, int pitch, float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int f = warp; f < TAS_TF; f += TAS_THREADS / 32) {
    const int t = f0 + f;
    if (t >= pitch) continue;
    float* col = xn + t;
    if (t >= frames) {
      for (int n = lane; n < N; n += 32) col[(size_t)n * pitch] = 0.f;
      continue;
    }
    double s = 0.0;
    for (int n = lane; n < N; n += 32) s += (double)wt[n * TAS_TF + f];
    const double mean = warp_sum_d(s) / N;
    double v = 0.0;
    for (int n = lane; n < N; n += 32) {
      const double d = (double)wt[n * TAS_TF + f] - mean;
      v = fma(d, d, v);
    }
    const double denom = sqrt(warp_sum_d(v) / N) + (double)eps;
    for (int n = lane; n < N; n += 32)
      col[(size_t)n * pitch] = (float)((double)__ldg(gamma + n) * (((double)wt[n * TAS_TF + f] - mean) / denom) + (double)__ldg(beta + n));
  }
}

// GatedEncoder + frame norm: w[b][n][t] = ReLU(U x~)[n][t] sigmoid(V x~)[n][t], x~ = x / (||x|| + enc_eps) zero-padded by pad_left;
// xn = the frame norm of w.  Columns [frames, pitch) of both are 0.  grid (pitch / TAS_TF, B), block 256; dynamic shared memory:
// the tile's samples, then wt[N][TAS_TF].
__global__ void __launch_bounds__(TAS_THREADS) k_tas_enc_gated(const float* __restrict__ x, const double* __restrict__ nrm,
                                                               const float* __restrict__ Uw, const float* __restrict__ Vw,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                                               float* __restrict__ w, float* __restrict__ xn, int T, int pad_left,
                                                               int N, int L, int stride, int frames, int pitch, float enc_eps,
                                                               float eps) {
  extern __shared__ float sm[];
  const int b = blockIdx.y, f0 = blockIdx.x * TAS_TF;
  const int nsamp = (TAS_TF - 1) * stride + L;
  float* xs = sm;
  float* wt = sm + ((nsamp + 3) & ~3);
  const double scale = nrm[b] + (double)enc_eps;
  const float* xb = x + (size_t)b * T;
  for (int i = threadIdx.x; i < nsamp; i += TAS_THREADS) {
    const long long p = (long long)f0 * stride + i - pad_left;
    xs[i] = (p >= 0 && p < T) ? (float)((double)xb[p] / scale) : 0.f;
  }
  __syncthreads();
  float* wb = w + (size_t)b * N * pitch;
  for (int idx = threadIdx.x; idx < N * TAS_TF; idx += TAS_THREADS) {
    const int n = idx / TAS_TF, f = idx % TAS_TF, t = f0 + f;
    float o = 0.f;
    if (t < frames) {
      const float* xf = xs + f * stride;
      const float* u = Uw + (size_t)n * L;
      const float* v = Vw + (size_t)n * L;
      float au = 0.f, av = 0.f;
      for (int k = 0; k < L; ++k) {
        au = fmaf(__ldg(u + k), xf[k], au);
        av = fmaf(__ldg(v + k), xf[k], av);
      }
      o = fmaxf(au, 0.f) * (1.f / (1.f + expf(-av)));
    }
    wt[idx] = o;
    if (t < pitch) wb[(size_t)n * pitch + t] = o;
  }
  __syncthreads();
  tas_frame_norm_tile(wt, gamma, beta, xn + (size_t)b * N * pitch, N, f0, frames, pitch, eps);
}

// the frame norm alone, from w (B, N, pitch) (the plain Encoder's output).  grid (pitch / TAS_TF, B), dynamic smem wt[N][TAS_TF]
__global__ void __launch_bounds__(TAS_THREADS) k_tas_frame_norm(const float* __restrict__ w, const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, float* __restrict__ xn, int N,
                                                                int frames, int pitch, float eps) {
  extern __shared__ float wt[];
  const int b = blockIdx.y, f0 = blockIdx.x * TAS_TF;
  const float* wb = w + (size_t)b * N * pitch;
  for (int idx = threadIdx.x; idx < N * TAS_TF; idx += TAS_THREADS) {
    const int n = idx / TAS_TF, t = f0 + idx % TAS_TF;
    wt[idx] = t < frames ? wb[(size_t)n * pitch + t] : 0.f;
  }
  __syncthreads();
  tas_frame_norm_tile(wt, gamma, beta, xn + (size_t)b * N * pitch, N, f0, frames, pitch, eps);
}

// ---- bi-LSTM layer ------------------------------------------------------------------------------------------------------------
// wcat (dirs 4H, F) = [W_ih; W_ih_reverse], bcat (dirs 4H) = b_ih + b_hh per direction.  grid-stride, 1 launch.
struct TasW { const float* w_ih[2]; const float* b_ih[2]; const float* b_hh[2]; };
__global__ void __launch_bounds__(256) k_tas_lstm_prep(TasW p, float* __restrict__ wcat, float* __restrict__ bcat, int F, int H4,
                                                       int dirs) {
  const size_t nw = (size_t)H4 * F;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nw * dirs; i += (size_t)gridDim.x * blockDim.x) {
    wcat[i] = (i < nw ? p.w_ih[0] : p.w_ih[1])[i % nw];
  }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)H4 * dirs; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i % H4);
    const bool rev = i >= (size_t)H4;  // kernel parameters indexed by a register would be copied to the stack
    bcat[i] = (rev ? p.b_ih[1] : p.b_ih[0])[r] + (rev ? p.b_hh[1] : p.b_hh[0])[r];
  }
}

struct LstmArgs {
  const float* G;       // (B, dirs 4H, pitch): W_ih x + b_ih + b_hh, row d 4H + g H + j
  const float* whh[2];  // (4H, H) per direction, gate order i, f, g, o
  float* out;           // (B, dirs H, pitch): forward direction rows [0, H), reverse [H, 2H)
  const float* skip_in; // nullable: skip_out = out + skip_in
  float* skip_out;      // nullable
  float* hbuf;          // [dirs][2][gmax][H]
  unsigned* bar;        // dirs counters, 32 words apart
  int B, H, T, pitch, dirs, U, cpd, gmax, Hs;
};

__device__ __forceinline__ void cp_async4(float* s, const float* g) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(s);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(a), "l"(g) : "memory");
}
__device__ __forceinline__ float sigm(float a) { return 1.f / (1.f + expf(-a)); }

// shared-memory floats of one recurrence CTA: W_hh slice [4U][Hs], h [gmax][Hs], gate sums [4U][gmax], prefetch [2][4U][gmax][PF]
size_t lstm_smem_bytes(int H, int U, int gmax) {
  const size_t Hs = (size_t)((H + 3) & ~3);
  return sizeof(float) * (4 * U * Hs + gmax * Hs + (size_t)4 * U * gmax + (size_t)2 * 4 * U * gmax * TAS_PF);
}

__global__ void __launch_bounds__(TAS_THREADS, 1) k_tas_lstm(const LstmArgs a) {
  extern __shared__ __align__(16) float sm[];
  const int d = blockIdx.x / a.cpd, c = blockIdx.x % a.cpd;
  const int H = a.H, T = a.T, Hs = a.Hs, gmax = a.gmax;
  const int j0 = c * a.U, nu = min(a.U, H - j0), R = 4 * nu;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float* ws = sm;                          // local row r = g nu + u  <->  W_hh row g H + j0 + u
  float* hs = ws + (size_t)4 * a.U * Hs;
  float* gs = hs + (size_t)gmax * Hs;
  float* pre = gs + 4 * a.U * gmax;
  const float* whh = d ? a.whh[1] : a.whh[0];
  for (int i = tid; i < R * H; i += TAS_THREADS) {
    const int r = i / H, k = i % H, g = r / nu, u = r % nu;
    ws[r * Hs + k] = __ldg(whh + ((size_t)g * H + j0 + u) * H + k);
  }
  // pad columns [T, pitch) of the rows this CTA owns
  const int npad = a.pitch - T;
  for (int i = tid; i < a.B * nu * npad; i += TAS_THREADS) {
    const int bb = i / (nu * npad), u = (i / npad) % nu, t = T + i % npad;
    const size_t o = ((size_t)bb * a.dirs * H + (size_t)d * H + j0 + u) * a.pitch + t;
    a.out[o] = 0.f;
    if (a.skip_out) a.skip_out[o] = 0.f;
  }
  unsigned* bar = a.bar + 32 * d;
  float* hb = a.hbuf + (size_t)d * 2 * gmax * H;
  const int G4 = a.dirs * 4 * H;
  unsigned epoch = 0;
  for (int b0 = 0; b0 < a.B; b0 += gmax) {
    const int nb = min(gmax, a.B - b0);
    const bool owner = tid < nu * nb;
    const int uo = owner ? tid % nu : 0, bo = owner ? tid / nu : 0;
    float cst = 0.f;
    // input projections of steps [tile PF, tile PF + PF) into prefetch buffer tile & 1: pre[buf][(r nb + b) PF + p]
    auto prefetch = [&](int tile) {
      float* dst = pre + (size_t)(tile & 1) * 4 * a.U * gmax * TAS_PF;
      for (int i = tid; i < R * nb * TAS_PF; i += TAS_THREADS) {
        const int p = i % TAS_PF, bb = (i / TAS_PF) % nb, r = i / (TAS_PF * nb);
        const int s = tile * TAS_PF + p;
        if (s < T) {
          const int t = d ? T - 1 - s : s, g = r / nu, u = r % nu;
          cp_async4(dst + i, a.G + ((size_t)(b0 + bb) * G4 + (size_t)d * 4 * H + (size_t)g * H + j0 + u) * a.pitch + t);
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    prefetch(0);
    for (int s = 0; s < T; ++s) {
      const int t = d ? T - 1 - s : s, slot = s % TAS_PF, tile = s / TAS_PF;
      if (slot == 0) {
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();
        if (s + TAS_PF < T) prefetch(tile + 1);
      }
      // h_{s-1} of the group (zero at the first step)
      const float* hprev = hb + (size_t)((s + 1) & 1) * gmax * H;
      for (int i = tid; i < nb * H; i += TAS_THREADS) {
        const int bb = i / H, k = i % H;
        hs[bb * Hs + k] = s ? __ldcg(hprev + (size_t)bb * H + k) : 0.f;
      }
      __syncthreads();
      // gate rows: warp tiles of TAS_RB rows x TAS_SB sequences, lanes stride k, then a fixed shuffle tree
      for (int rb = warp * TAS_RB; rb < R; rb += (TAS_THREADS / 32) * TAS_RB) {
        for (int sb = 0; sb < nb; sb += TAS_SB) {
          float acc[TAS_RB][TAS_SB];
#pragma unroll
          for (int r = 0; r < TAS_RB; ++r)
#pragma unroll
            for (int q = 0; q < TAS_SB; ++q) acc[r][q] = 0.f;
          const float* wr[TAS_RB];
          const float* hr[TAS_SB];
#pragma unroll
          for (int r = 0; r < TAS_RB; ++r) wr[r] = ws + min(rb + r, R - 1) * Hs;
#pragma unroll
          for (int q = 0; q < TAS_SB; ++q) hr[q] = hs + min(sb + q, nb - 1) * Hs;
          for (int k = lane; k < H; k += 32) {
            float hv[TAS_SB];
#pragma unroll
            for (int q = 0; q < TAS_SB; ++q) hv[q] = hr[q][k];
#pragma unroll
            for (int r = 0; r < TAS_RB; ++r) {
              const float wv = wr[r][k];
#pragma unroll
              for (int q = 0; q < TAS_SB; ++q) acc[r][q] = fmaf(wv, hv[q], acc[r][q]);
            }
          }
#pragma unroll
          for (int r = 0; r < TAS_RB; ++r)
#pragma unroll
            for (int q = 0; q < TAS_SB; ++q)
              if (rb + r < R && sb + q < nb) {
                const float v = warp_sum(acc[r][q]);
                if (lane == 0) gs[(rb + r) * gmax + sb + q] = v;
              }
        }
      }
      __syncthreads();
      if (owner) {
        const float* pb = pre + (size_t)(tile & 1) * 4 * a.U * gmax * TAS_PF;
        float gv[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int r = g * nu + uo;
          gv[g] = gs[r * gmax + bo] + pb[((size_t)r * nb + bo) * TAS_PF + slot];
        }
        cst = fmaf(sigm(gv[1]), cst, sigm(gv[0]) * tanhf(gv[2]));
        const float h = sigm(gv[3]) * tanhf(cst);
        const size_t o = ((size_t)(b0 + bo) * a.dirs * H + (size_t)d * H + j0 + uo) * a.pitch + t;
        a.out[o] = h;
        if (a.skip_out) a.skip_out[o] = h + a.skip_in[o];
        __stcg(hb + (size_t)(s & 1) * gmax * H + (size_t)bo * H + j0 + uo, h);
      }
      // every CTA of this direction has published h_s (and finished reading h_{s-1})
      __syncthreads();
      ++epoch;
      if (tid == 0) {
        __threadfence();
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
        const unsigned target = epoch * (unsigned)a.cpd;
        unsigned v;
        do {
          asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
        } while ((int)(v - target) < 0);
        __threadfence();
      }
      __syncthreads();
    }
  }
}

// recurrence geometry on the current device: U units per CTA, cpd CTAs per direction, gmax sequences per pass
struct LstmGeo { int U, cpd, gmax; size_t smem; };

int device_limits(int* nsm, int* smem_optin) {
  int dev = 0, coop = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return 0; }
  if (cudaDeviceGetAttribute(nsm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaDeviceGetAttribute(smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return coop;
}

// false when H does not fit: one CTA per SM, each direction on its own half of the SMs
bool lstm_geo(int H, int dirs, int nsm, int smem_optin, LstmGeo* g) {
  if (H <= 0 || (dirs != 1 && dirs != 2)) return false;
  const int per_dir = nsm / dirs;
  if (per_dir <= 0) return false;
  g->U = (H + per_dir - 1) / per_dir;
  g->cpd = (H + g->U - 1) / g->U;
  if (g->U > TAS_THREADS) return false;
  g->gmax = TAS_GMAX < TAS_THREADS / g->U ? TAS_GMAX : TAS_THREADS / g->U;
  while (g->gmax >= 1 && lstm_smem_bytes(H, g->U, g->gmax) > (size_t)smem_optin) --g->gmax;
  if (g->gmax < 1) return false;
  g->smem = lstm_smem_bytes(H, g->U, g->gmax);
  return true;
}

bool lstm_geo_here(int H, int dirs, LstmGeo* g) {
  int nsm = 0, smem = 0;
  if (!device_limits(&nsm, &smem)) return false;
  return lstm_geo(H, dirs, nsm, smem, g);
}

size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }

bool math_ok(int math) {
  return math == CTN_MATH_FP32 || math == CTN_MATH_TF32 || math == CTN_MATH_TF32X3 || math == CTN_MATH_F16X3;
}

const float* one_ptr() {
  void* p = nullptr;
  if (cudaGetSymbolAddress(&p, k_tas_one) != cudaSuccess) return nullptr;
  return (const float*)p;
}

size_t enc_smem_bytes(int N, int L, int stride) {
  const int nsamp = (TAS_TF - 1) * stride + L;
  return sizeof(float) * ((size_t)((nsamp + 3) & ~3) + (size_t)N * TAS_TF);
}

int set_smem(const void* fn, size_t bytes) {
  if (bytes <= 48 * 1024) return CTN_OK;
  const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  return e == cudaSuccess ? CTN_OK : (int)e;
}

// softmax over the S sources of each (b, n, t) of the fc logits (B, S N, pitch), times w: in place
__global__ void __launch_bounds__(256) k_tas_softmax_src(float* __restrict__ what, const float* __restrict__ w, int S, int N, int frames,
                                                         int pitch) {
  const int b = blockIdx.y;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)N * pitch; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / pitch), t = (int)(i % pitch);
    float* col = what + ((size_t)b * S * N + n) * pitch + t;
    if (t >= frames) {
      for (int s = 0; s < S; ++s) col[(size_t)s * N * pitch] = 0.f;
      continue;
    }
    float m = -INFINITY;
    for (int s = 0; s < S; ++s) m = fmaxf(m, col[(size_t)s * N * pitch]);
    float sum = 0.f;
    for (int s = 0; s < S; ++s) sum += expf(col[(size_t)s * N * pitch] - m);
    const float wv = w[((size_t)b * N + n) * pitch + t];
    for (int s = 0; s < S; ++s) col[(size_t)s * N * pitch] = expf(col[(size_t)s * N * pitch] - m) / sum * wv;
  }
}

}  // namespace

// ---- encoder + frame norm ----------------------------------------------------------------------------------------------------------
extern "C" int ctn_tas_enc_gated_fwd(const float* x, const float* u_w, const float* v_w, const float* gamma, const float* beta, float* w,
                                     float* xn, double* nrm, int B, int T, int pad_left, int pad_right, int N, int L, int stride, int pitch,
                                     float enc_eps, float eps, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !u_w || !v_w || !gamma || !beta || !w || !xn || !nrm || B <= 0 || T <= 0 || N <= 0 || L <= 0 || stride <= 0 || pad_left < 0 ||
      pad_right < 0)
    return CTN_EINVAL;
  const long long Tp = (long long)T + pad_left + pad_right;
  if (Tp < L) return CTN_EINVAL;
  const int frames = (int)((Tp - L) / stride + 1);  // Conv1d: a ragged tail makes no frame (but counts in the norm)
  if (pitch < frames || pitch % CTN_TILE_T != 0) return CTN_EALIGN;
  if (B > 65535) return CTN_EUNSUPPORTED;
  int nsm = 0, smem_optin = 0;
  device_limits(&nsm, &smem_optin);
  const size_t smem = enc_smem_bytes(N, L, stride);
  if (smem > (size_t)(smem_optin > 48 * 1024 ? smem_optin : 48 * 1024)) return CTN_EUNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  CTN_TRY(set_smem((const void*)k_tas_enc_gated, smem));
  k_tas_sig_norm<<<B, 256, 0, st>>>(x, nrm, T);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  k_tas_enc_gated<<<dim3(pitch / TAS_TF, B), TAS_THREADS, smem, st>>>(x, nrm, u_w, v_w, gamma, beta, w, xn, T, pad_left, N, L, stride, frames,
                                                                       pitch, enc_eps, eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_tas_frame_norm_fwd(const float* w, const float* gamma, const float* beta, float* xn, int B, int N, int frames, int pitch,
                                      float eps, ctn_stream_t stream) {
  LaunchScope scope(w);
  if (!w || !gamma || !beta || !xn || B <= 0 || N <= 0 || frames <= 0) return CTN_EINVAL;
  if (pitch < frames || pitch % CTN_TILE_T != 0) return CTN_EALIGN;
  if (w == xn) return CTN_EINVAL;
  if (B > 65535) return CTN_EUNSUPPORTED;
  int nsm = 0, smem_optin = 0;
  device_limits(&nsm, &smem_optin);
  const size_t smem = sizeof(float) * (size_t)N * TAS_TF;
  if (smem > (size_t)(smem_optin > 48 * 1024 ? smem_optin : 48 * 1024)) return CTN_EUNSUPPORTED;
  CTN_TRY(set_smem((const void*)k_tas_frame_norm, smem));
  k_tas_frame_norm<<<dim3(pitch / TAS_TF, B), TAS_THREADS, smem, (cudaStream_t)stream>>>(w, gamma, beta, xn, N, frames, pitch, eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- one (bi-)LSTM layer --------------------------------------------------------------------------------------------------------------
extern "C" int ctn_tas_lstm_max_hidden(int dirs) {
  int nsm = 0, smem = 0;
  if (!device_limits(&nsm, &smem) || (dirs != 1 && dirs != 2)) return 0;
  LstmGeo g;
  int lo = 0, hi = 1 << 16;  // lstm_geo is monotone in H: the smem of one pass only grows with it
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (lstm_geo(mid, dirs, nsm, smem, &g)) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

extern "C" int ctn_tas_lstm_supported(int F, int H, int dirs) {
  LstmGeo g;
  return F > 0 && lstm_geo_here(H, dirs, &g) ? 1 : 0;
}

extern "C" int ctn_tas_lstm_group(int H, int dirs) {
  LstmGeo g;
  return lstm_geo_here(H, dirs, &g) ? g.gmax : 0;
}

extern "C" size_t ctn_tas_lstm_workspace_bytes(int B, int F, int H, int dirs, int pitch, int math) {
  if (B <= 0 || F <= 0 || H <= 0 || (dirs != 1 && dirs != 2) || pitch <= 0) return 0;
  const size_t M = (size_t)dirs * 4 * H;
  const size_t img = math == CTN_MATH_FP32 ? 0 : up256(ctn_pw_wimg_bytes((int)M, F, math));
  return up256(M * F * 4) + up256(M * 4) + img + up256((size_t)B * M * pitch * 4) + up256((size_t)2 * B * 8) +
         up256((size_t)dirs * 2 * TAS_GMAX * H * 4) + up256((size_t)dirs * 32 * 4) + 256;
}

extern "C" int ctn_tas_lstm_fwd(const float* x, const float* const* w, float* out, const float* skip_in, float* skip_out, int B, int F, int H,
                                int dirs, int frames, int pitch, int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !w || !out || !workspace || B <= 0 || F <= 0 || H <= 0 || frames <= 0 || (dirs != 1 && dirs != 2)) return CTN_EINVAL;
  for (int i = 0; i < 4 * dirs; ++i)
    if (!w[i]) return CTN_EINVAL;
  if ((skip_in == nullptr) != (skip_out == nullptr)) return CTN_EINVAL;
  if (out == x || (skip_out && (skip_out == x || skip_out == out))) return CTN_EINVAL;
  if (!math_ok(math)) return CTN_EINVAL;
  if (pitch < frames || pitch % CTN_TILE_T != 0 || (((uintptr_t)workspace) & 255) || (((uintptr_t)x) & 15)) return CTN_EALIGN;
  if (workspace_bytes < ctn_tas_lstm_workspace_bytes(B, F, H, dirs, pitch, math)) return CTN_EWORKSPACE;
  LstmGeo geo;
  if (!lstm_geo_here(H, dirs, &geo)) return CTN_EUNSUPPORTED;
  const long long ngroups = (B + geo.gmax - 1) / geo.gmax;
  if (ngroups * frames * geo.cpd >= 0x7fffffffLL) return CTN_EUNSUPPORTED;  // the barrier counters are 32-bit
  const float* one = one_ptr();
  if (!one) return CTN_ENOTBUILT;
  int occ = 0, nsm = 0, smem_optin = 0;
  device_limits(&nsm, &smem_optin);
  cudaError_t e = cudaFuncSetAttribute((const void*)k_tas_lstm, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)geo.smem);
  if (e != cudaSuccess) return (int)e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_tas_lstm, TAS_THREADS, geo.smem)) != cudaSuccess) return (int)e;
  if ((long long)occ * nsm < (long long)dirs * geo.cpd) return CTN_EUNSUPPORTED;  // the spinning CTAs could not all be resident
  cudaStream_t st = (cudaStream_t)stream;
  const int M = dirs * 4 * H;
  Carver cv(workspace);
  float* wcat = cv.take<float>((size_t)M * F);
  float* bcat = cv.take<float>(M);
  float* img = math == CTN_MATH_FP32 ? nullptr : cv.take<float>(ctn_pw_wimg_bytes(M, F, math) / 4);
  float* G = cv.take<float>((size_t)B * M * pitch);
  double* stats = cv.take<double>((size_t)2 * B);
  float* hbuf = cv.take<float>((size_t)dirs * 2 * TAS_GMAX * H);
  unsigned* bar = cv.take<unsigned>((size_t)dirs * 32);
  if ((e = cudaMemsetAsync(bar, 0, sizeof(unsigned) * 32 * dirs, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(stats, 0, sizeof(double) * 2 * B, st)) != cudaSuccess) return (int)e;
  TasW p;
  for (int d = 0; d < 2; ++d) {
    const int dd = d < dirs ? d : 0;
    p.w_ih[d] = w[4 * dd + 0];
    p.b_ih[d] = w[4 * dd + 2];
    p.b_hh[d] = w[4 * dd + 3];
  }
  int gp = (int)(((size_t)M * F + 255) / 256);
  if (gp > 1024) gp = 1024;
  k_tas_lstm_prep<<<gp, 256, 0, st>>>(p, wcat, bcat, F, 4 * H, dirs);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  // G = W_ih x + (b_ih + b_hh) for both directions: EPI_H with a slope of 1 is the bias add alone
  PwArgs a;
  memset(&a, 0, sizeof(a));
  a.A = x; a.W = wcat; a.D = G; a.B = B; a.M = M; a.K = F; a.frames = frames; a.pitch = pitch;
  a.bias = bcat; a.slope = one; a.stats_out = stats;
  if (img) {
    const WimgJob job{wcat, img, M, F};
    CTN_TRY(ctn_pw_prepare_batch(&job, 1, math, false, st));
    a.wimg = img;
  }
  CTN_TRY(ctn_pw(a, PRO_NONE, EPI_H, math, nullptr, st));
  LstmArgs la;
  la.G = G;
  la.whh[0] = w[1];
  la.whh[1] = dirs == 2 ? w[5] : w[1];
  la.out = out; la.skip_in = skip_in; la.skip_out = skip_out; la.hbuf = hbuf; la.bar = bar;
  la.B = B; la.H = H; la.T = frames; la.pitch = pitch; la.dirs = dirs; la.U = geo.U; la.cpd = geo.cpd; la.gmax = geo.gmax;
  la.Hs = (H + 3) & ~3;
  // the CTAs of a direction spin on each other: a cooperative launch guarantees they are co-resident, or fails
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(dirs * geo.cpd);
  cfg.blockDim = dim3(TAS_THREADS);
  cfg.dynamicSmemBytes = geo.smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if ((e = cudaLaunchKernelEx(&cfg, k_tas_lstm, la)) != cudaSuccess) {
    cudaGetLastError();
    return (int)e;
  }
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- separator tail + decoder ----------------------------------------------------------------------------------------------------
extern "C" size_t ctn_tas_tail_workspace_bytes(int N, int Hd, int S, int math) {
  if (N <= 0 || Hd <= 0 || S <= 0) return 0;
  return (math == CTN_MATH_FP32 ? 0 : up256(ctn_pw_wimg_bytes(S * N, Hd, math))) + 256;
}

extern "C" int ctn_tas_tail_fwd(const float* skip, const float* w, const float* fc_w, const float* fc_b, const float* dec_w, float* out,
                                float* latent, float* what, int B, int N, int Hd, int S, int frames, int pitch, int L, int stride,
                                int crop_left, int T, int softmax, int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(skip);
  if (!skip || !w || !fc_w || !fc_b || !dec_w || !out || !what || !workspace || B <= 0 || N <= 0 || Hd <= 0 || S <= 0 || frames <= 0)
    return CTN_EINVAL;
  if (!math_ok(math)) return CTN_EINVAL;
  if (pitch < frames || pitch % CTN_TILE_T != 0 || (((uintptr_t)workspace) & 255)) return CTN_EALIGN;
  if ((((uintptr_t)skip) | ((uintptr_t)w) | ((uintptr_t)what)) & 15) return CTN_EALIGN;
  if (workspace_bytes < ctn_tas_tail_workspace_bytes(N, Hd, S, math)) return CTN_EWORKSPACE;
  if ((long long)B * S > 65535) return CTN_EUNSUPPORTED;
  CTN_TRY(ctn_decoder_check(B * S, N, frames, pitch, L, stride, crop_left, T));
  const float* one = one_ptr();
  if (!one) return CTN_ENOTBUILT;
  cudaStream_t st = (cudaStream_t)stream;
  PwArgs m;
  memset(&m, 0, sizeof(m));
  m.A = skip; m.W = fc_w; m.D = what; m.B = B; m.M = S * N; m.K = Hd; m.frames = frames; m.pitch = pitch;
  m.pro_slope = one; m.bias = fc_b; m.wenc = w; m.Nb = N; m.mask_logits = softmax ? 1 : 0;
  if (math != CTN_MATH_FP32) {
    Carver cv(workspace);
    float* img = cv.take<float>(ctn_pw_wimg_bytes(S * N, Hd, math) / 4);
    const WimgJob job{fc_w, img, S * N, Hd};
    CTN_TRY(ctn_pw_prepare_batch(&job, 1, math, false, st));
    m.wimg = img;
  }
  CTN_TRY(ctn_pw(m, PRO_PRELU, EPI_MASK, math, nullptr, st));
  if (softmax) {
    int gx = (int)(((size_t)N * pitch + 255) / 256);
    if (gx > 256) gx = 256;
    k_tas_softmax_src<<<dim3(gx, B), 256, 0, st>>>(what, w, S, N, frames, pitch);
    CTN_COUNT_LAUNCH();
    CTN_RETURN_IF_CUDA_ERR();
  }
  CTN_TRY(ctn_decoder_fwd(what, dec_w, out, B * S, N, frames, pitch, L, stride, crop_left, T, stream));
  if (latent) CTN_TRY(ctn_copy_from_pitch(what, latent, B * S * N, frames, pitch, st));
  return CTN_OK;
}
