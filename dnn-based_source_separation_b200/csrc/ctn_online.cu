// Online (chunk-by-chunk) inference of the causal Conv-TasNet (include/ctn_b200.h, ctn_online_*).
//
// Every operation of the causal model is per frame except three: cLN (statistics over all frames <= t), the causal dilated
// depthwise conv (reads (P-1)*d earlier frames) and the two filter banks (a frame spans L samples; an output sample sums
// L/S frames).  So a push carries exactly that state, and everything else runs on the chunk's frames alone:
//   encoder over [carry | chunk] -> cLN0 (carried sums) -> bottleneck 1x1 (+ bias)
//   per block: pw1 1x1 (+ bias, PReLU) -> k_online_block -> [Wo; Ws] 1x1 -> residual / skip
//   mask 1x1 (+ softmax) -> decoder over [history | chunk] -> commit the sample counter
// The 1x1 contractions, the bias / residual kernels and the softmax are the offline causal path's own (ctn_causal.cu), with
// weight images built once at init; each produces a frame's column from that frame's column alone, so a frame computed
// online gets the offline bits.  The new kernels keep the offline operation order: the depthwise taps, the cLN apply
// formula and the decoder's summation order (split across channel quarters like k_decoder) are the same.  Only the cLN
// prefix sums are added in another order, in double.
//
// Each stream's chunk goes through the cLN kernels in ONE CTA: the prefix sum over frames crosses every channel and every
// frame of the chunk, and one CTA does it with __syncthreads alone.  The chunk is walked in tiles of 32 frames (lane =
// frame, warp = channel group), the scan carried from tile to tile.  With B streams the grid is B CTAs.
//
// Counters (OnlineHdr, push_frames in ctn_internal.h, shared with the online LSTM-TasNet): the state's header holds T0, the
// samples pushed since the reset.  Every kernel of a push reads it; the decoder,
// the push's last kernel, advances it once all its CTAs have read it (ticket).  Frames done before the push:
// F0 = T0 >= L ? (T0 - L) / S + 1 : 0; the push completes F1 - F0 of its n / S columns.
#include <string.h>
#include <vector>
#include "ctn_internal.h"

namespace {

constexpr int OT = 512;          // threads of the per-stream cLN kernels
constexpr int NW = OT / 32;      // channel groups
constexpr int TF = 32;           // frames per tile

struct OnlineState {
  OnlineHdr* hdr;
  double* cln;                 // [B][1 + 2RX][2] running (sum, sumsq) of cLN0, then norm1 / norm2 of every block
  float* enc_carry;            // [B][L - S] the last L - S input samples
  float* dec_hist;             // [B][S*N][L/S - 1] w_hat of the last L/S - 1 frames
  std::vector<float*> ring;    // per block: [B][H][(P-1) d] cLN1 output, frame g at slot g mod (P-1) d
  double* dummy;               // [B][2] sink for the unused gLN statistics of the EPI_H epilogue
  size_t carry_bytes;          // the bytes above: zeroed by init and reset
  std::vector<float*> wcat;    // per block: [Wo; Ws] (Bc+Sc, H)
  std::vector<float*> wimg1, wimg2;
  float *wimg_head, *wimg_mask;
  float* dec_w;                // (N, L) decoder basis: the flush has no parameter argument
  // one chunk, (B, rows, pitch)
  float *w, *wn, *x, *skip, *h, *u, *r, *what;
};

int ring_frames(const ctn_config_t* c, int i) { return (c->sep_kernel - 1) * (1 << (i % c->num_layers)); }

void carve(Carver& cv, const ctn_config_t* c, int B, int pitch, OnlineState* s) {
  const int RX = c->num_blocks * c->num_layers, H = c->hidden, Bc = c->bottleneck, Sc = c->skip, N = c->n_basis;
  const int S = c->n_sources, D = c->kernel_size - c->stride, R = c->kernel_size / c->stride;
  s->hdr = cv.take<OnlineHdr>(1);
  s->cln = cv.take<double>((size_t)B * (1 + 2 * RX) * 2);
  s->enc_carry = cv.take<float>((size_t)B * D);
  s->dec_hist = cv.take<float>((size_t)B * S * N * (R - 1));
  size_t ring_total = 0;
  for (int i = 0; i < RX; ++i) ring_total += (size_t)B * H * ring_frames(c, i);
  float* ring = cv.take<float>(ring_total);  // B H (P-1) sum_i d_i floats in all
  s->ring.assign(RX, nullptr);
  for (int i = 0; i < RX; ++i) {
    s->ring[i] = ring;
    if (ring) ring += (size_t)B * H * ring_frames(c, i);
  }
  s->dummy = cv.take<double>((size_t)B * 2);
  cv.off = (cv.off + 255) & ~(size_t)255;
  s->carry_bytes = cv.off;
  s->wcat.assign(RX, nullptr);
  s->wimg1.assign(RX, nullptr);
  s->wimg2.assign(RX, nullptr);
  for (int i = 0; i < RX; ++i) {
    s->wcat[i] = cv.take<float>((size_t)(Bc + Sc) * H);
    if (c->math != CTN_MATH_FP32) {
      s->wimg1[i] = cv.take<float>(ctn_pw_wimg_bytes(H, Bc, c->math) / sizeof(float));
      s->wimg2[i] = cv.take<float>(ctn_pw_wimg_bytes(Bc + Sc, H, c->math) / sizeof(float));
    }
  }
  s->wimg_head = s->wimg_mask = nullptr;
  if (c->math != CTN_MATH_FP32) {
    s->wimg_head = cv.take<float>(ctn_pw_wimg_bytes(Bc, N, c->math) / sizeof(float));
    s->wimg_mask = cv.take<float>(ctn_pw_wimg_bytes(S * N, Sc, c->math) / sizeof(float));
  }
  s->dec_w = cv.take<float>((size_t)N * c->kernel_size);
  const size_t bp = (size_t)B * pitch;
  s->w = cv.take<float>(bp * N);
  s->wn = cv.take<float>(bp * N);
  s->x = cv.take<float>(bp * Bc);
  s->skip = cv.take<float>(bp * Sc);
  s->h = cv.take<float>(bp * H);
  s->u = cv.take<float>(bp * H);
  s->r = cv.take<float>(bp * (Bc + Sc));
  s->what = cv.take<float>(bp * S * N);
}

int check_cfg(const ctn_config_t* c) {
  if (c && (c->causal != 1 || c->in_channels > 1)) return CTN_EUNSUPPORTED;  // gLN needs the whole utterance; monaural only
  CTN_TRY(check_model_cfg(c));
  if ((size_t)c->n_basis * (c->kernel_size / c->stride - 1) * sizeof(float) > 48 * 1024) return CTN_EUNSUPPORTED;  // decoder history
  return CTN_OK;
}

// Encoder over [carry | chunk]: w[b][c][f] = sum_k W[c][k] xcat[base + f S + k] (k ascending, as k_encoder), f < nv; zero up to pitch.
// One CTA per stream: the carry is read into shared memory before it is overwritten.
__global__ void __launch_bounds__(256) k_online_enc(const float* __restrict__ x, const float* __restrict__ W, float* __restrict__ carry,
                                                    float* __restrict__ w, const OnlineHdr* __restrict__ hdr, int N, int L, int S, int n,
                                                    int pitch, int relu) {
  extern __shared__ float xs[];  // [D + n]
  const int b = blockIdx.x, D = L - S;
  const OnlineFrames fr = push_frames(hdr, L, S, n);
  float* cb = carry + (size_t)b * D;
  for (int i = threadIdx.x; i < D; i += 256) xs[i] = cb[i];
  for (int i = threadIdx.x; i < n; i += 256) xs[D + i] = x[(size_t)b * n + i];
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += 256) cb[i] = xs[n + i];
  // frame F0 + f starts at sample (F0 + f) S, at xcat position (F0 + f) S - (T0 - D): 0 once L samples were seen
  const int base = (int)(fr.F0 * S - (fr.T0 - D));
  for (int i = threadIdx.x; i < N * pitch; i += 256) {
    const int c = i / pitch, f = i - c * pitch;
    float v = 0.f;
    if (f < fr.nv) {
      const float* xf = xs + base + f * S;
      float acc = 0.f;
      for (int k = 0; k < L; ++k) acc = fmaf(W[c * L + k], xf[k], acc);
      v = relu ? fmaxf(acc, 0.f) : acc;
    }
    w[((size_t)b * N + c) * pitch + f] = v;
  }
}

// cLN of the frames [t0, t0 + TF) of one stream's (C, pitch) rows, in place allowed: per-frame channel sums in double, an
// inclusive scan seeded with the running sums `run` (shared, advanced here), then k_cln_apply's formula.  Frames >= nv are
// written as zero and left out of the sums.  Called by all OT threads.
__device__ void cln_tile(const float* src, float* dst, int C, int pitch, int t0, int nv, long long F0, double* run,
                         const float* __restrict__ gamma, const float* __restrict__ beta, float eps, double (*red)[TF][2],
                         float2* mi) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, t = t0 + lane;
  const bool valid = t < nv;
  double s = 0.0, ss = 0.0;
  if (valid)
    for (int c = wid; c < C; c += NW) {
      const double v = (double)src[(size_t)c * pitch + t];
      s += v;
      ss += v * v;
    }
  red[wid][lane][0] = s;
  red[wid][lane][1] = ss;
  __syncthreads();
  if (wid == 0) {
    s = 0.0; ss = 0.0;
    for (int g = 0; g < NW; ++g) { s += red[g][lane][0]; ss += red[g][lane][1]; }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double a = __shfl_up_sync(0xffffffffu, s, o), b = __shfl_up_sync(0xffffffffu, ss, o);
      if (lane >= o) { s += a; ss += b; }
    }
    const double cs = run[0] + s, css = run[1] + ss;
    const double nn = (double)C * (double)(F0 + t + 1);
    const double mean = cs / nn;
    double var = css / nn - mean * mean;
    var = var > 0.0 ? var : 0.0;
    mi[lane] = make_float2((float)mean, 1.f / ((float)sqrt(var) + eps));  // eps outside the sqrt, as k_cln_apply
    __syncwarp();
    if (lane == 31) { run[0] = cs; run[1] = css; }  // frames >= nv added zeros
  }
  __syncthreads();
  const float m = mi[lane].x, inv = mi[lane].y;
  for (int c = wid; c < C; c += NW) {
    const size_t i = (size_t)c * pitch + t;
    dst[i] = valid ? (src[i] - m) * inv * gamma[c] + beta[c] : 0.f;
  }
}

// cLN0 of the encoder output: wn = cLN(w), running sums carried in run_g (double[2] of this norm, stride `rstride` per stream)
__global__ void __launch_bounds__(OT) k_online_cln(const float* __restrict__ w, float* __restrict__ wn, double* __restrict__ run_g,
                                                   int rstride, const OnlineHdr* __restrict__ hdr, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, int C, int L, int S, int n, int F, int pitch,
                                                   float eps) {
  __shared__ double red[NW][TF][2];
  __shared__ float2 mi[TF];
  __shared__ double run[2];
  const int b = blockIdx.x;
  const OnlineFrames fr = push_frames(hdr, L, S, n);
  double* rg = run_g + (size_t)b * rstride;
  if (threadIdx.x < 2) run[threadIdx.x] = rg[threadIdx.x];
  __syncthreads();
  const float* src = w + (size_t)b * C * pitch;
  float* dst = wn + (size_t)b * C * pitch;
  for (int t0 = 0; t0 < F; t0 += TF) {
    cln_tile(src, dst, C, pitch, t0, fr.nv, fr.F0, run, gamma, beta, eps, red, mi);
    __syncthreads();
  }
  if (threadIdx.x < 2) rg[threadIdx.x] = run[threadIdx.x];
}

// The middle of residual block i on one stream's chunk, in place on h:
//   hn = cLN1(h) -> u = PReLU(causal dilated depthwise conv over [ring | hn] + bd) (k_dw_plain's tap order) -> u = cLN2(u)
// then the ring takes the last (P-1) d frames of hn.  run_g: double[2][2] (norm1, norm2) of this block, `rstride` per stream.
__global__ void __launch_bounds__(OT) k_online_block(float* __restrict__ h, float* __restrict__ u, float* __restrict__ ring_g,
                                                     double* __restrict__ run_g, int rstride, const OnlineHdr* __restrict__ hdr,
                                                     const float* __restrict__ g1, const float* __restrict__ b1,
                                                     const float* __restrict__ wd, const float* __restrict__ bd,
                                                     const float* __restrict__ slope, const float* __restrict__ g2,
                                                     const float* __restrict__ b2, int H, int P, int dil, int L, int S, int n,
                                                     int F, int pitch, float eps) {
  __shared__ double red[NW][TF][2];
  __shared__ float2 mi[TF];
  __shared__ double run[4];
  const int b = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int Rd = (P - 1) * dil;
  const OnlineFrames fr = push_frames(hdr, L, S, n);
  double* rg = run_g + (size_t)b * rstride;
  if (threadIdx.x < 4) run[threadIdx.x] = rg[threadIdx.x];
  __syncthreads();
  float* hb = h + (size_t)b * H * pitch;
  float* ub = u + (size_t)b * H * pitch;
  float* ring = ring_g + (size_t)b * H * Rd;
  const float a = slope[0];
  const int head = Rd > 0 ? (int)(fr.F0 % Rd) : 0;  // ring slot of frame F0
  for (int t0 = 0; t0 < F; t0 += TF) {
    cln_tile(hb, hb, H, pitch, t0, fr.nv, fr.F0, run, g1, b1, eps, red, mi);
    __syncthreads();  // this tile's hn is read by other threads' taps
    const int t = t0 + lane;
    const long long g = fr.F0 + t;
    for (int c = wid; c < H; c += NW) {
      float v = 0.f;
      if (t < fr.nv) {
        float acc = bd[c];
        for (int k = 0; k < P; ++k) {
          const long long gt = g - (long long)(P - 1 - k) * dil;  // tt = t + k d - pad_left of k_dw_plain, in stream frames
          if (gt < 0) continue;                                   // the causal left padding
          const int tt = (int)(gt - fr.F0);                       // > -Rd
          const float hv = tt >= 0 ? hb[(size_t)c * pitch + tt] : ring[(size_t)c * Rd + (head + tt + Rd) % Rd];
          acc = fmaf(wd[c * P + k], hv, acc);
        }
        v = prelu_f(acc, a);
      }
      ub[(size_t)c * pitch + t] = v;
    }
    cln_tile(ub, ub, H, pitch, t0, fr.nv, fr.F0, run + 2, g2, b2, eps, red, mi);
    __syncthreads();
  }
  // ring <- hn of frames [max(F0, F1 - Rd), F1), after every tap of the chunk has read the ring
  if (Rd > 0) {
    const int first = fr.nv > Rd ? fr.nv - Rd : 0, cnt = fr.nv - first;
    for (int i = threadIdx.x; i < H * cnt; i += OT) {
      const int c = i / cnt, t = first + i - c * cnt;
      ring[(size_t)c * Rd + (head + t) % Rd] = hb[(size_t)c * pitch + t];
    }
  }
  if (threadIdx.x < 4) rg[threadIdx.x] = run[threadIdx.x];
}

// Decoder over [history | chunk] with the crop of the offline model: output position p is sample g = T0 - D + p (< 0: the
// delay, zero) = segment j = g / S, phase q = g % S, summed over the frames j - r, r < L/S, that exist.  split: the order of
// k_decoder<S, 2> (channel quarters, r inner, quarters added in order); else k_decoder_generic's.  One CTA per (stream,
// source) row block.  push = 1: the history takes the last L/S - 1 frames and the last CTA advances T0 by n.  push = 0
// (flush): nout = D samples from the history alone, nothing advanced.
__global__ void __launch_bounds__(256) k_online_dec(const float* __restrict__ what, const float* __restrict__ Wd, float* __restrict__ hist_g,
                                                    float* __restrict__ y, OnlineHdr* __restrict__ hdr, int N, int L, int S, int n,
                                                    int nout, int pitch, int split, int push) {
  extern __shared__ float hs[];  // [N][R-1] new history
  const int bs = blockIdx.x, R = L / S, D = L - S;
  const OnlineFrames fr = push_frames(hdr, L, S, push ? n : 0);
  const long long F1 = fr.F0 + fr.nv, Fh = fr.F0 - (R - 1);  // frames [Fh, F0) in the history
  const float* wb = what + (size_t)bs * N * pitch;
  float* hist = hist_g + (size_t)bs * N * (R - 1);
  for (int p = threadIdx.x; p < nout; p += 256) {
    const long long g = fr.T0 - D + p;
    float out = 0.f;
    if (g >= 0) {
      const long long j = g / S;
      const int q = (int)(g - j * S);
      // frame j - r: a chunk column (stride pitch) or a history slot (stride R - 1); absent frames read as 0
      auto frame = [&](int r, const float*& src, size_t& step) {
        const long long f = j - r;
        step = f >= fr.F0 ? (size_t)pitch : (size_t)(R - 1);
        src = f >= fr.F0 ? wb + (f - fr.F0) : hist + (f - Fh);
        return f >= 0 && f < F1;
      };
      if (split) {  // R == 2
        const float *s0, *s1;
        size_t st0, st1;
        const bool ok0 = frame(0, s0, st0), ok1 = frame(1, s1, st1);
        const int nper = (N + 3) / 4;
        for (int pp = 0; pp < 4; ++pp) {
          float acc = 0.f;
          const int n_end = min(N, (pp + 1) * nper);
#pragma unroll 8
          for (int c = pp * nper; c < n_end; ++c) {
            const float v0 = ok0 ? s0[c * st0] : 0.f, v1 = ok1 ? s1[c * st1] : 0.f;
            acc = fmaf(v0, Wd[c * L + q], acc);
            acc = fmaf(v1, Wd[c * L + S + q], acc);
          }
          out = pp == 0 ? acc : out + acc;  // ((q0 + q1) + q2) + q3
        }
      } else {
        float acc = 0.f;
        for (int r = 0; r < R; ++r) {
          const float* sr;
          size_t str;
          if (!frame(r, sr, str)) continue;
#pragma unroll 8
          for (int c = 0; c < N; ++c) acc = fmaf(sr[c * str], Wd[c * L + r * S + q], acc);
        }
        out = acc;
      }
    }
    y[(size_t)bs * nout + p] = out;
  }
  if (!push) return;
  // history <- frames [F1 - (R-1), F1)
  const long long Fn = F1 - (R - 1);
  for (int i = threadIdx.x; i < N * (R - 1); i += 256) {
    const int c = i / (R - 1);
    const long long f = Fn + (i - c * (R - 1));
    hs[i] = f < 0 ? 0.f : (f >= fr.F0 ? wb[(size_t)c * pitch + (f - fr.F0)] : hist[c * (R - 1) + (int)(f - Fh)]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N * (R - 1); i += 256) hist[i] = hs[i];
  // every thread of this CTA read T0 before the barrier above; the last CTA to get here advances it
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned tk = atomicAdd(&hdr->ticket, 1u);
    if (tk == gridDim.x - 1) {
      hdr->T0 = fr.T0 + n;
      hdr->ticket = 0u;
      __threadfence();
    }
  }
}

bool decoder_split(int L, int S) { return L == 2 * S && (S == 8 || S == 1 || S == 10 || S == 2); }  // ctn_decoder_fwd's k_decoder cases

}  // namespace

size_t ctn_online_enc_smem(int L, int S, int n) { return sizeof(float) * ((size_t)L - S + n); }

int ctn_online_enc(const float* x, const float* W, float* carry, float* w, const OnlineHdr* hdr, int B, int N, int L, int S, int n,
                   int pitch, int relu, cudaStream_t st) {
  const size_t smem = ctn_online_enc_smem(L, S, n);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(k_online_enc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  k_online_enc<<<B, 256, smem, st>>>(x, W, carry, w, hdr, N, L, S, n, pitch, relu);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int ctn_online_dec(const float* what, const float* Wd, float* hist, float* y, OnlineHdr* hdr, int BS, int N, int L, int S, int n, int pitch,
                   int push, cudaStream_t st) {
  const int R = L / S;
  k_online_dec<<<BS, 256, sizeof(float) * (size_t)N * (R - 1), st>>>(what, Wd, hist, y, hdr, N, L, S, push ? n : 0, push ? n : L - S,
                                                                     pitch, decoder_split(L, S) ? 1 : 0, push);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_online_state_bytes(const ctn_config_t* cfg, int B, int max_chunk_frames, size_t* bytes) {
  CTN_TRY(check_cfg(cfg));
  if (B <= 0 || max_chunk_frames <= 0 || !bytes) return CTN_EINVAL;
  if (ctn_online_enc_smem(cfg->kernel_size, cfg->stride, max_chunk_frames * cfg->stride) > 200 * 1024) return CTN_EUNSUPPORTED;
  Carver cv(nullptr);
  OnlineState s;
  carve(cv, cfg, B, ctn_pitch(max_chunk_frames), &s);
  *bytes = cv.off + 256;
  return CTN_OK;
}

extern "C" int ctn_online_init(const ctn_config_t* cfg, const ctn_params_t* params, int B, int max_chunk_frames, void* state,
                               size_t state_bytes, ctn_stream_t stream) {
  CTN_TRY(check_cfg(cfg));
  if (!params || !params->blocks || !state || B <= 0 || max_chunk_frames <= 0) return CTN_EINVAL;
  if (((uintptr_t)state) & 255) return CTN_EALIGN;
  size_t need = 0;
  CTN_TRY(ctn_online_state_bytes(cfg, B, max_chunk_frames, &need));
  if (state_bytes < need) return CTN_EWORKSPACE;
  const int RX = cfg->num_blocks * cfg->num_layers, Bc = cfg->bottleneck, H = cfg->hidden, Sc = cfg->skip, N = cfg->n_basis;
  for (int i = 0; i < RX; ++i)
    if (!params->blocks[i].out_w && i != RX - 1) return CTN_EINVAL;
  LaunchScope scope(state);
  cudaStream_t st = (cudaStream_t)stream;
  Carver cv(state);
  OnlineState s;
  carve(cv, cfg, B, ctn_pitch(max_chunk_frames), &s);
  cudaError_t e = cudaMemsetAsync(state, 0, s.carry_bytes, st);
  if (e != cudaSuccess) return (int)e;
  // the offline path copies [Wo; Ws] and builds every image on each call; here once
  for (int i = 0; i < RX; ++i) {
    const ctn_block_params_t& q = params->blocks[i];
    const int Mt = q.out_w ? Bc + Sc : Sc;
    CTN_TRY(ctn_block_wcat(q, Bc, Sc, H, s.wcat[i], st));
    PwArgs a;
    memset(&a, 0, sizeof(a));
    a.W = q.bottleneck_w; a.M = H; a.K = Bc;
    CTN_TRY(ctn_pw_prepare(a, cfg->math, s.wimg1[i], st));
    a.W = s.wcat[i]; a.M = Mt; a.K = H;
    CTN_TRY(ctn_pw_prepare(a, cfg->math, s.wimg2[i], st));
  }
  PwArgs a;
  memset(&a, 0, sizeof(a));
  a.W = params->bn_w; a.M = Bc; a.K = N;
  CTN_TRY(ctn_pw_prepare(a, cfg->math, s.wimg_head, st));
  a.W = params->mask_w; a.M = cfg->n_sources * N; a.K = Sc;
  CTN_TRY(ctn_pw_prepare(a, cfg->math, s.wimg_mask, st));
  e = cudaMemcpyAsync(s.dec_w, params->dec_w, sizeof(float) * (size_t)N * cfg->kernel_size, cudaMemcpyDeviceToDevice, st);
  return e == cudaSuccess ? CTN_OK : (int)e;
}

extern "C" int ctn_online_reset(const ctn_config_t* cfg, void* state, int B, ctn_stream_t stream) {
  CTN_TRY(check_cfg(cfg));
  if (!state || B <= 0) return CTN_EINVAL;
  if (((uintptr_t)state) & 255) return CTN_EALIGN;
  LaunchScope scope(state);
  Carver cv(nullptr);
  OnlineState s;
  carve(cv, cfg, B, CTN_TILE_T, &s);
  cudaError_t e = cudaMemsetAsync(state, 0, s.carry_bytes, (cudaStream_t)stream);
  return e == cudaSuccess ? CTN_OK : (int)e;
}

extern "C" int ctn_online_push(const ctn_config_t* cfg, const ctn_params_t* params, void* state, const float* x, int B,
                               int max_chunk_frames, int n, float* y, ctn_stream_t stream) {
  CTN_TRY(check_cfg(cfg));
  if (!params || !params->blocks || !state || !x || !y || B <= 0 || max_chunk_frames <= 0) return CTN_EINVAL;
  const int L = cfg->kernel_size, S = cfg->stride;
  if (n <= 0 || n % S != 0 || n / S > max_chunk_frames) return CTN_EINVAL;
  if (((uintptr_t)state) & 255) return CTN_EALIGN;
  const int RX = cfg->num_blocks * cfg->num_layers, Bc = cfg->bottleneck, H = cfg->hidden, Sc = cfg->skip, N = cfg->n_basis;
  const int Ns = cfg->n_sources, P = cfg->sep_kernel;
  for (int i = 0; i < RX; ++i)
    if (!params->blocks[i].out_w && i != RX - 1) return CTN_EINVAL;
  LaunchScope scope(state);
  cudaStream_t st = (cudaStream_t)stream;
  const int F = n / S, pitch = ctn_pitch(F);  // the chunk's layout: every scratch tensor is rewritten by each push
  Carver cv(state);
  OnlineState s;
  carve(cv, cfg, B, pitch, &s);
  const int rstride = (1 + 2 * RX) * 2;
  {
    StageTimer tm(CTN_ST_ENC, st);
    CTN_TRY(ctn_online_enc(x, params->enc_w, s.enc_carry, s.w, s.hdr, B, N, L, S, n, pitch, cfg->enc_relu, st));
  }
  {
    StageTimer tm(CTN_ST_HEAD, st);
    k_online_cln<<<B, OT, 0, st>>>(s.w, s.wn, s.cln, rstride, s.hdr, params->norm0_g, params->norm0_b, N, L, S, n, F, pitch, cfg->eps);
    CTN_COUNT_LAUNCH();
    CTN_RETURN_IF_CUDA_ERR();
    PwArgs a;
    memset(&a, 0, sizeof(a));
    a.A = s.wn; a.W = params->bn_w; a.D = s.x; a.B = B; a.M = Bc; a.K = N; a.frames = F; a.pitch = pitch; a.wimg = s.wimg_head;
    CTN_TRY(ctn_pw(a, PRO_NONE, EPI_RAW, cfg->math, nullptr, st));
    CTN_TRY(ctn_bias_rows_fwd(s.x, params->bn_b, Bc, B, F, pitch, st));
  }
  for (int i = 0; i < RX; ++i) {
    const ctn_block_params_t& q = params->blocks[i];
    const bool has_out = q.out_w != nullptr;
    const int Mt = has_out ? Bc + Sc : Sc;
    PwArgs a;
    memset(&a, 0, sizeof(a));
    a.A = s.x; a.W = q.bottleneck_w; a.D = s.h; a.B = B; a.M = H; a.K = Bc; a.frames = F; a.pitch = pitch;
    a.bias = q.bottleneck_b; a.slope = q.prelu1; a.stats_out = s.dummy; a.wimg = s.wimg1[i];
    { StageTimer tm(CTN_ST_PW1, st); CTN_TRY(ctn_pw(a, PRO_NONE, EPI_H, cfg->math, nullptr, st)); }
    {
      StageTimer tm(CTN_ST_DW, st);
      k_online_block<<<B, OT, 0, st>>>(s.h, s.u, s.ring[i], s.cln + 2 + 4 * i, rstride, s.hdr, q.norm1_g, q.norm1_b, q.dw_w, q.dw_b,
                                       q.prelu2, q.norm2_g, q.norm2_b, H, P, 1 << (i % cfg->num_layers), L, S, n, F, pitch, cfg->eps_tcn);
      CTN_COUNT_LAUNCH();
      CTN_RETURN_IF_CUDA_ERR();
    }
    memset(&a, 0, sizeof(a));
    a.A = s.u; a.W = s.wcat[i]; a.D = s.r; a.B = B; a.M = Mt; a.K = H; a.frames = F; a.pitch = pitch; a.wimg = s.wimg2[i];
    { StageTimer tm(CTN_ST_PW2, st); CTN_TRY(ctn_pw(a, PRO_NONE, EPI_RAW, cfg->math, nullptr, st)); }
    { StageTimer tm(CTN_ST_FIN, st);
      CTN_TRY(ctn_res_skip_fwd(s.r, Mt, s.x, s.x, s.skip, q.out_b, q.skip_b, Bc, Sc, has_out ? 1 : 0, i == 0 ? 1 : 0, B, F, pitch, st)); }
  }
  {
    StageTimer tm(CTN_ST_MASK, st);
    PwArgs m;
    memset(&m, 0, sizeof(m));
    m.A = s.skip; m.W = params->mask_w; m.D = s.what; m.B = B; m.M = Ns * N; m.K = Sc; m.frames = F; m.pitch = pitch;
    m.pro_slope = params->prelu_out; m.bias = params->mask_b; m.wenc = s.w; m.Nb = N; m.wimg = s.wimg_mask;
    m.mask_logits = cfg->mask_softmax ? 1 : 0;
    CTN_TRY(ctn_pw(m, PRO_PRELU, EPI_MASK, cfg->math, nullptr, st));
    if (cfg->mask_softmax) CTN_TRY(ctn_softmax_mask(s.what, s.w, nullptr, B, Ns * N, N, F, pitch, st));
  }
  {
    StageTimer tm(CTN_ST_DEC, st);
    CTN_TRY(ctn_online_dec(s.what, s.dec_w, s.dec_hist, y, s.hdr, B * Ns, N, L, S, n, pitch, 1, st));
  }
  return CTN_OK;
}

extern "C" int ctn_online_flush(const ctn_config_t* cfg, void* state, int B, float* y_tail, ctn_stream_t stream) {
  CTN_TRY(check_cfg(cfg));
  const int L = cfg->kernel_size, S = cfg->stride, D = L - S, N = cfg->n_basis;
  // a zero-delay model (kernel_size == stride) has no tail: y_tail holds 0 samples and may be null
  if (!state || (D > 0 && !y_tail) || B <= 0) return CTN_EINVAL;
  if (((uintptr_t)state) & 255) return CTN_EALIGN;
  LaunchScope scope(state);
  cudaStream_t st = (cudaStream_t)stream;
  Carver cv(state);
  OnlineState s;
  carve(cv, cfg, B, CTN_TILE_T, &s);
  long long T0 = 0;
  cudaError_t e = cudaMemcpyAsync(&T0, &s.hdr->T0, sizeof(T0), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return (int)e;
  if (T0 < L) return CTN_EINVAL;  // no frame yet: the offline model needs T >= kernel_size
  if (D == 0) return CTN_OK;
  // the tail segments read the history only; `what` is not touched (pitch is unused)
  return ctn_online_dec(s.what, s.dec_w, s.dec_hist, y_tail, s.hdr, B * cfg->n_sources, N, L, S, 0, CTN_TILE_T, 0, st);
}
