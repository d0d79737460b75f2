// SepFormer stages.  Reference: src/models/sepformer.py:281-361 (Separator), :438-520 (IntraTransformer / InterTransformer),
// src/models/transformer.py:7-43 (PositionalEncoding), torch.nn.TransformerEncoderLayer (post-norm, ReLU) and src/models/gtu.py.
//
// The dual-path state is CHANNEL-FIRST and pitched: X (B, F, pitch), token s*C + k for chunk s and frame k, pitch =
// ctn_pitch(S*C) -- the reference's own (B, F, S, C) layout with padded rows.  Every Linear of an encoder layer is then one ctn_pw
// contraction with the tokens as columns, and the two paths only differ in which tokens form a sequence:
//   sequence j of sample b = tokens j*seq_stride + t*tok_stride, t < len
//   intra: nseq = S, len = C, seq_stride = C, tok_stride = 1;   inter: nseq = C, len = S, seq_stride = 1, tok_stride = C.
// Nothing is permuted between the paths.
//   * attention reads the channel-first QKV (B, 3F, pitch) ctn_pw leaves (without the in-projection bias, which is added on load);
//     one query per thread (intra: neighbouring threads read neighbouring tokens), keys streamed in tiles of 64 through an online
//     softmax (running max and sum in fp32), so any sequence length runs in fixed shared memory.  fp32 FMAs.
//   * the post-norm LayerNorm of each sub-layer, LN(x + y + bias) over the F features of a token: one thread per token, mean and
//     centred variance in double (two passes), so a token whose features are all equal comes out exactly beta.
//   * the end of each Intra/InterTransformer: GroupNorm(1, F) per SEQUENCE (F x len values, summed in double in a fixed order,
//     no atomics) plus the outer residual, the block input without the positional encoding (sepformer.py:468, 476).
//   * the tail: PReLU -> map -> GTU1d -> bottleneck_conv1d_out -> ReLU / sigmoid -> w * mask -> decoder.
#include <math.h>
#include <string.h>

#include "ctn_internal.h"

namespace {

constexpr int ATT_Q = 64;    // queries per attention CTA (one per thread)
constexpr int ATT_KT = 64;   // keys per shared-memory tile
constexpr int ATT_SUB = 16;  // keys per online-softmax update
constexpr int LN_T = 128;    // tokens per LayerNorm CTA
constexpr int SFM_PE_MAX = 5000;  // rows of the reference's positional-encoding buffer (transformer.py:8)
constexpr int SFM_LAYER_PTRS = 12;

struct Seqs {
  int nseq, len, seq_stride, tok_stride;
  __host__ __device__ size_t tok(int j, int t) const { return (size_t)j * seq_stride + (size_t)t * tok_stride; }
};

// O[b][h D + c][tok(j, t)] = sum_i softmax_i(q_t . k_i / sqrt(D)) v_i[c] over the tokens i of sequence j, q/k/v = qkv rows
// [0,F) / [F,2F) / [2F,3F) + in_b.  grid (B * nseq, ceil(len / 64), heads), block 64: one query per thread, q and the running
// output in registers; a 64-key tile of k and v in shared memory (every thread reads the same key: broadcast).  Rows of the tile
// are D + 4 floats: 16-byte aligned for the vector reads, and the tile stores (keys fastest) spread over the banks.
template <int D>
__global__ void __launch_bounds__(ATT_Q) k_sfm_attn(const float* __restrict__ qkv, const float* __restrict__ in_b, float* __restrict__ O,
                                                    int F, int pitch, Seqs q_, float scale) {
  __shared__ __align__(16) float ks[ATT_KT][D + 4];
  __shared__ __align__(16) float vs[ATT_KT][D + 4];
  const int b = blockIdx.x / q_.nseq, j = blockIdx.x % q_.nseq, hd = blockIdx.z;
  const int t = blockIdx.y * ATT_Q + threadIdx.x, T = q_.len;
  const float* base = qkv + (size_t)b * 3 * F * pitch;
  const size_t qtok = q_.tok(j, t < T ? t : 0);
  float q[D], acc[D];
#pragma unroll
  for (int c = 0; c < D; ++c) {
    const int row = hd * D + c;
    q[c] = t < T ? (__ldg(base + (size_t)row * pitch + qtok) + __ldg(in_b + row)) * scale : 0.f;
    acc[c] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < T; k0 += ATT_KT) {
    const int nk = T - k0 < ATT_KT ? T - k0 : ATT_KT;
    __syncthreads();  // the previous tile is consumed
    for (int i = threadIdx.x; i < ATT_KT * D; i += ATT_Q) {
      const int kk = i % ATT_KT, c = i / ATT_KT;
      if (kk < nk) {
        const size_t tk = q_.tok(j, k0 + kk);
        const int rk = F + hd * D + c, rv = 2 * F + hd * D + c;
        ks[kk][c] = __ldg(base + (size_t)rk * pitch + tk) + __ldg(in_b + rk);
        vs[kk][c] = __ldg(base + (size_t)rv * pitch + tk) + __ldg(in_b + rv);
      }
    }
    __syncthreads();
    for (int j0 = 0; j0 < nk; j0 += ATT_SUB) {
      float s[ATT_SUB];
      float mt = m;
#pragma unroll
      for (int jj = 0; jj < ATT_SUB; ++jj) {
        const int kk = j0 + jj;
        float dot = -INFINITY;
        if (kk < nk) {
          dot = 0.f;
#pragma unroll
          for (int c = 0; c < D; ++c) dot = fmaf(q[c], ks[kk][c], dot);
        }
        s[jj] = dot;
        mt = fmaxf(mt, dot);
      }
      const float corr = expf(m - mt);  // m = -inf before the first key: corr = 0 rescales the empty sums
      l *= corr;
#pragma unroll
      for (int c = 0; c < D; ++c) acc[c] *= corr;
#pragma unroll
      for (int jj = 0; jj < ATT_SUB; ++jj) {
        const int kk = j0 + jj;
        if (kk < nk) {
          const float p = expf(s[jj] - mt);
          l += p;
#pragma unroll
          for (int c = 0; c < D; ++c) acc[c] = fmaf(p, vs[kk][c], acc[c]);
        }
      }
      m = mt;
    }
  }
  if (t < T) {
    const float inv = 1.f / l;
    float* o = O + (size_t)b * F * pitch + qtok;
#pragma unroll
    for (int c = 0; c < D; ++c) o[(size_t)(hd * D + c) * pitch] = acc[c] * inv;
  }
}

// out[b][f][t] = LN_f(X + (Y + bias)) over the F features of token t (nn.LayerNorm(F, eps) of the post-norm layer,
// x = norm(x + sublayer(x))), gamma, beta per feature; Y, bias nullable; out may alias X.  Columns [ntok, pitch) = 0.
// grid (ceil(pitch / 128), B), block 128, one token per thread: neighbouring threads read neighbouring columns.
__device__ __forceinline__ float ln_val(const float* X, const float* Y, const float* __restrict__ bias, size_t i, int f) {
  float y = Y ? Y[i] : 0.f;
  if (bias) y += __ldg(bias + f);
  return X[i] + y;
}
__global__ void __launch_bounds__(LN_T) k_token_ln(const float* X, const float* Y, const float* __restrict__ bias, const float* __restrict__ gamma,
                                                  const float* __restrict__ beta, float* out, int F, int ntok, int pitch, float eps) {
  const int b = blockIdx.y, t = blockIdx.x * LN_T + threadIdx.x;
  if (t >= pitch) return;
  const size_t col = (size_t)b * F * pitch + t;
  if (t >= ntok) {
    for (int f = 0; f < F; ++f) out[col + (size_t)f * pitch] = 0.f;
    return;
  }
  double s = 0.0;
  for (int f = 0; f < F; ++f) s += ln_val(X, Y, bias, col + (size_t)f * pitch, f);
  const double mean = s / F;
  double v = 0.0;
  for (int f = 0; f < F; ++f) {
    const double d = ln_val(X, Y, bias, col + (size_t)f * pitch, f) - mean;
    v = fma(d, d, v);
  }
  const double rstd = 1.0 / sqrt(v / F + (double)eps);
  for (int f = 0; f < F; ++f) {
    const size_t i = col + (size_t)f * pitch;
    const float xn = (float)((ln_val(X, Y, bias, i, f) - mean) * rstd);
    out[i] = fmaf(xn, __ldg(gamma + f), __ldg(beta + f));
  }
}

// out = GroupNorm(1, F)(sequence j of X; gamma, beta) + R over the F x len values of each sequence (LayerNormWrapper('gLN') as the
// encoder's final norm, then the outer residual).  grid (nseq, B), block 256.  Each thread sums its elements in double in index
// order and the block reduction is a fixed shuffle tree: the statistics do not depend on scheduling.  The CTA of sequence 0 also
// zeroes the pad columns [ntok, pitch) of its sample.  out may alias R.
__global__ void __launch_bounds__(256) k_sfm_seq_norm(const float* X, const float* R, const float* __restrict__ gamma,
                                                      const float* __restrict__ beta, float* out, int F, int pitch, int ntok, Seqs q_,
                                                      float eps) {
  __shared__ double red[64];
  __shared__ double st[2];
  const int j = blockIdx.x, b = blockIdx.y, T = q_.len;
  const size_t n = (size_t)F * T, sb = (size_t)b * F * pitch;
  double s = 0.0, ss = 0.0;
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int f = (int)(i / T), t = (int)(i % T);
    const double x = X[sb + (size_t)f * pitch + q_.tok(j, t)];
    s += x;
    ss = fma(x, x, ss);
  }
  block_sum2_d(s, ss, red);
  if (threadIdx.x == 0) { st[0] = s; st[1] = ss; }
  __syncthreads();
  const float2 mr = gln_mean_rstd(st, (double)n, eps);
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int f = (int)(i / T), t = (int)(i % T);
    const size_t at = sb + (size_t)f * pitch + q_.tok(j, t);
    out[at] = fmaf((X[at] - mr.x) * mr.y, __ldg(gamma + f), __ldg(beta + f)) + R[at];
  }
  if (j == 0) {
    const int pad = pitch - ntok;
    for (int i = threadIdx.x; i < F * pad; i += blockDim.x) out[sb + (size_t)(i / pad) * pitch + ntok + i % pad] = 0.f;
  }
}

// out = X + (X + pe[t]) at token tok(j, t): the encoder input of sepformer.py:471-472, where PositionalEncoding.forward already
// returns input + encoding (transformer.py:39) and the caller adds the input once more.  pe (>= len, F) as the module's buffer
// (5000, 1, F), read bit for bit.  Columns [ntok, pitch) = 0.  grid (ceil(pitch / 128), F, B), block 128.
__global__ void __launch_bounds__(128) k_sfm_pos_enc(const float* __restrict__ X, const float* __restrict__ pe, float* __restrict__ out,
                                                     int F, int pitch, int ntok, int C, int intra) {
  const int f = blockIdx.y, b = blockIdx.z, t = blockIdx.x * 128 + threadIdx.x;
  if (t >= pitch) return;
  const size_t i = ((size_t)b * F + f) * pitch + t;
  if (t >= ntok) { out[i] = 0.f; return; }
  const int pos = intra ? t % C : t / C;  // frame within its chunk (intra) or chunk index (inter)
  const float x = X[i];
  out[i] = x + (x + __ldg(pe + (size_t)pos * F + f));
}

// segmentation into the pitched channel-first layout: Z[b][f][s C + k] = xpad[b][f][s P + k] (xpad = x zero-padded by pad_left on
// the left), columns [S C, z_pitch) = 0.  grid (ceil(z_pitch / 256), F, B)
__global__ void __launch_bounds__(256) k_sfm_segment(const float* __restrict__ x, float* __restrict__ Z, int F, int frames, int pitch,
                                                     int pad_left, int S, int C, int P, int z_pitch) {
  const int f = blockIdx.y, b = blockIdx.z, i = blockIdx.x * 256 + threadIdx.x;
  if (i >= z_pitch) return;
  float v = 0.f;
  if (i < S * C) {
    const int s = i / C, k = i % C, tt = s * P + k - pad_left;
    if (tt >= 0 && tt < frames) v = __ldg(x + ((size_t)b * F + f) * pitch + tt);
  }
  Z[((size_t)b * F + f) * z_pitch + i] = v;
}

// overlap-add + crop from the pitched layout: y[b][f][t] = sum over the chunks s covering padded frame tp = t + crop_left, s
// ascending, of Z[b][f][s C + tp - s P]; columns [T_out, out_pitch) = 0.  grid (ceil(out_pitch / 256), F, B)
__global__ void __launch_bounds__(256) k_sfm_overlap_add(const float* __restrict__ Z, float* __restrict__ y, int F, int S, int C, int P,
                                                         int z_pitch, int crop_left, int T_out, int out_pitch) {
  const int f = blockIdx.y, b = blockIdx.z, t = blockIdx.x * 256 + threadIdx.x;
  if (t >= out_pitch) return;
  float acc = 0.f;
  if (t < T_out) {
    const int tp = t + crop_left;
    int s_lo = (tp - C + 1 <= 0) ? 0 : (tp - C + P) / P;
    int s_hi = tp / P;
    if (s_hi > S - 1) s_hi = S - 1;
    const float* z = Z + ((size_t)b * F + f) * z_pitch;
    for (int s = s_lo; s <= s_hi; ++s) acc += __ldg(z + (size_t)s * C + tp - s * P);
  }
  y[((size_t)b * F + f) * out_pitch + t] = acc;
}

// PReLU on the (B, C, pitch) layout (columns [frames, pitch) = 0); thread 0 of CTA 0 also stores the device scalar 1.0 the
// bias-only contractions of the tail take as their PReLU slope
__global__ void __launch_bounds__(256) k_sfm_prelu(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ slope,
                                                   size_t n, int frames, int pitch, float* one) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *one = 1.f;
  const float a = __ldg(slope);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    y[i] = (int)(i % pitch) < frames ? prelu_f(x[i], a) : 0.f;
}

// GTU1d: g (R, 2N, pitch) = [map; map_gate] m + bias -> u (R, N, pitch) = tanh(g[n]) sigmoid(g[N + n]); columns [frames, pitch) = 0
__global__ void __launch_bounds__(256) k_sfm_gtu(const float* __restrict__ g, float* __restrict__ u, int N, int frames, int pitch) {
  const int r = blockIdx.y;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)N * pitch; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / pitch), t = (int)(i % pitch);
    float v = 0.f;
    if (t < frames) {
      const float a = g[((size_t)r * 2 * N + n) * pitch + t], gt = g[((size_t)r * 2 * N + N + n) * pitch + t];
      v = tanhf(a) * (1.f / (1.f + expf(-gt)));
    }
    u[(size_t)r * N * pitch + i] = v;
  }
}

// what[b s][n][t] = act(v[b s][n][t]) w[b][n][t], act = ReLU (mask_relu) or sigmoid; columns [frames, pitch) = 0
__global__ void __launch_bounds__(256) k_sfm_mask(const float* __restrict__ v, const float* __restrict__ w, float* __restrict__ what, int S,
                                                  int N, int frames, int pitch, int mask_relu) {
  const int bs = blockIdx.y, b = bs / S;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)N * pitch; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / pitch), t = (int)(i % pitch);
    float o = 0.f;
    if (t < frames) {
      const float x = v[(size_t)bs * N * pitch + i];
      const float mk = mask_relu ? fmaxf(x, 0.f) : 1.f / (1.f + expf(-x));
      o = mk * w[((size_t)b * N + n) * pitch + t];
    }
    what[(size_t)bs * N * pitch + i] = o;
  }
}

bool attn_ok(int F, int heads) {
  if (F <= 0 || heads <= 0 || F % heads) return false;
  const int D = F / heads;
  return D == 8 || D == 16 || D == 32 || D == 64;
}

// the sequence set of one path over S chunks of C frames
Seqs path_seqs(int S, int C, int intra) {
  Seqs q;
  if (intra) { q.nseq = S; q.len = C; q.seq_stride = C; q.tok_stride = 1; }
  else { q.nseq = C; q.len = S; q.seq_stride = 1; q.tok_stride = C; }
  return q;
}

// refusals shared by the stages on the pitched dual-path state
int state_check(int B, int F, int S, int C, int pitch) {
  if (B <= 0 || F <= 0 || S <= 0 || C <= 0 || pitch <= 0) return CTN_EINVAL;
  if ((long long)S * C > pitch) return CTN_EINVAL;
  if (B > 65535 || F > 65535) return CTN_EUNSUPPORTED;
  return CTN_OK;
}

int launch_attn(const float* qkv, const float* in_b, float* O, int B, int F, int heads, int pitch, const Seqs& q, cudaStream_t st) {
  const int D = F / heads;
  const float scale = (float)(1.0 / sqrt((double)D));
  const dim3 g((unsigned)((long long)B * q.nseq), (q.len + ATT_Q - 1) / ATT_Q, heads);
  if (D == 8) k_sfm_attn<8><<<g, ATT_Q, 0, st>>>(qkv, in_b, O, F, pitch, q, scale);
  if (D == 16) k_sfm_attn<16><<<g, ATT_Q, 0, st>>>(qkv, in_b, O, F, pitch, q, scale);
  if (D == 32) k_sfm_attn<32><<<g, ATT_Q, 0, st>>>(qkv, in_b, O, F, pitch, q, scale);
  if (D == 64) k_sfm_attn<64><<<g, ATT_Q, 0, st>>>(qkv, in_b, O, F, pitch, q, scale);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int launch_token_ln(const float* X, const float* Y, const float* bias, const float* gamma, const float* beta, float* out, int B, int F,
                    int ntok, int pitch, float eps, cudaStream_t st) {
  k_token_ln<<<dim3((pitch + LN_T - 1) / LN_T, B), LN_T, 0, st>>>(X, Y, bias, gamma, beta, out, F, ntok, pitch, eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int launch_seq_norm(const float* X, const float* R, const float* gamma, const float* beta, float* out, int B, int F, int pitch, int ntok,
                    const Seqs& q, float eps, cudaStream_t st) {
  k_sfm_seq_norm<<<dim3(q.nseq, B), 256, 0, st>>>(X, R, gamma, beta, out, F, pitch, ntok, q, eps);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// one 1x1 contraction of the pitched state through ctn_pw from a prebuilt weight image (none in the fp32 mode): EPI_RAW, or
// EPI_H with the PReLU slope and the statistics scratch the caller passes (ReLU: a device slope of 0)
int pw_run(const float* A, const float* W, const float* wimg, float* D, int B, int M, int K, int frames, int pitch, int math,
           const float* bias, const float* slope, double* stats, cudaStream_t st) {
  PwArgs a;
  memset(&a, 0, sizeof(a));
  a.A = A; a.W = W; a.D = D; a.B = B; a.M = M; a.K = K; a.frames = frames; a.pitch = pitch;
  a.wimg = wimg;
  if (bias) { a.bias = bias; a.slope = slope; a.stats_out = stats; }
  return ctn_pw(a, PRO_NONE, bias ? EPI_H : EPI_RAW, math, nullptr, st);
}

size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t tf_img_bytes(int F, int d_ff, int math, int k) {  // image of contraction k of a layer: QKV, out_proj, linear1, linear2
  if (math == CTN_MATH_FP32) return 0;
  const int shapes[4][2] = {{3 * F, F}, {F, F}, {d_ff, F}, {F, d_ff}};
  return up256(ctn_pw_wimg_bytes(shapes[k][0], shapes[k][1], math));
}

}  // namespace

// ---- attention over a strided sequence set ---------------------------------------------------------------------------------------
extern "C" int ctn_sfm_attn_supported(int F, int heads) { return attn_ok(F, heads) ? 1 : 0; }

extern "C" int ctn_sfm_attn_fwd(const float* qkv, const float* in_b, float* O, int B, int F, int heads, int S, int C, int pitch, int intra,
                                ctn_stream_t stream) {
  LaunchScope scope(qkv);
  if (!qkv || !in_b || !O || heads <= 0) return CTN_EINVAL;
  CTN_TRY(state_check(B, F, S, C, pitch));
  if (!attn_ok(F, heads)) return CTN_EUNSUPPORTED;
  const Seqs q = path_seqs(S, C, intra);
  if ((long long)B * q.nseq > 0x7fffffffLL || (q.len + ATT_Q - 1) / ATT_Q > 65535) return CTN_EUNSUPPORTED;
  return launch_attn(qkv, in_b, O, B, F, heads, pitch, q, (cudaStream_t)stream);
}

// ---- post-norm LayerNorm of a token --------------------------------------------------------------------------------------------
extern "C" int ctn_sfm_token_ln_fwd(const float* X, const float* Y, const float* bias, const float* gamma, const float* beta, float* out,
                                    int B, int F, int ntok, int pitch, float eps, ctn_stream_t stream) {
  LaunchScope scope(X);
  if (!X || !gamma || !beta || !out || B <= 0 || F <= 0 || ntok <= 0 || pitch < ntok) return CTN_EINVAL;
  if (B > 65535) return CTN_EUNSUPPORTED;
  if (Y && out == Y) return CTN_EINVAL;  // only X may be overwritten
  return launch_token_ln(X, Y, bias, gamma, beta, out, B, F, ntok, pitch, eps, (cudaStream_t)stream);
}

// ---- the encoder's final gLN per sequence + the outer residual -------------------------------------------------------------------
extern "C" int ctn_sfm_seq_norm_res_fwd(const float* X, const float* R, const float* gamma, const float* beta, float* out, int B, int F,
                                        int S, int C, int pitch, int intra, float eps, ctn_stream_t stream) {
  LaunchScope scope(X);
  if (!X || !R || !gamma || !beta || !out) return CTN_EINVAL;
  CTN_TRY(state_check(B, F, S, C, pitch));
  if (out == X) return CTN_EINVAL;  // X is read again after other sequences' stores could land
  return launch_seq_norm(X, R, gamma, beta, out, B, F, pitch, S * C, path_seqs(S, C, intra), eps, (cudaStream_t)stream);
}

// ---- positional encoding ---------------------------------------------------------------------------------------------------------
extern "C" int ctn_sfm_pos_enc_fwd(const float* X, const float* pe, float* out, int B, int F, int S, int C, int pitch, int intra,
                                   ctn_stream_t stream) {
  LaunchScope scope(X);
  if (!X || !pe || !out) return CTN_EINVAL;
  CTN_TRY(state_check(B, F, S, C, pitch));
  if ((intra ? C : S) > SFM_PE_MAX) return CTN_EINVAL;
  k_sfm_pos_enc<<<dim3((pitch + 127) / 128, F, B), 128, 0, (cudaStream_t)stream>>>(X, pe, out, F, pitch, S * C, C, intra);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- segmentation / overlap-add on the pitched channel-first layout -------------------------------------------------------------
extern "C" int ctn_sfm_segment_fwd(const float* x, float* Z, int B, int F, int frames, int pitch, int chunk_size, int hop_size, int pad_left,
                                   int pad_right, int z_pitch, ctn_stream_t stream) {
  LaunchScope scope(x);
  if (!x || !Z || B <= 0 || F <= 0 || frames <= 0 || pitch < frames || chunk_size <= 0 || hop_size <= 0 || pad_left < 0 || pad_right < 0)
    return CTN_EINVAL;
  const int Tp = frames + pad_left + pad_right;
  if (Tp < chunk_size) return CTN_EINVAL;
  const int S = (Tp - chunk_size) / hop_size + 1;
  if ((long long)S * chunk_size > z_pitch) return CTN_EINVAL;
  if (B > 65535 || F > 65535) return CTN_EUNSUPPORTED;
  k_sfm_segment<<<dim3((z_pitch + 255) / 256, F, B), 256, 0, (cudaStream_t)stream>>>(x, Z, F, frames, pitch, pad_left, S, chunk_size, hop_size,
                                                                                  z_pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

extern "C" int ctn_sfm_overlap_add_fwd(const float* Z, float* y, int B, int F, int S, int chunk_size, int hop_size, int z_pitch,
                                       int crop_left, int T_out, int out_pitch, ctn_stream_t stream) {
  LaunchScope scope(Z);
  if (!Z || !y || B <= 0 || F <= 0 || S <= 0 || chunk_size <= 0 || hop_size <= 0 || crop_left < 0 || T_out <= 0 || out_pitch < T_out)
    return CTN_EINVAL;
  if ((long long)S * chunk_size > z_pitch || crop_left + T_out > (S - 1) * hop_size + chunk_size) return CTN_EINVAL;
  if (B > 65535 || F > 65535) return CTN_EUNSUPPORTED;
  k_sfm_overlap_add<<<dim3((out_pitch + 255) / 256, F, B), 256, 0, (cudaStream_t)stream>>>(Z, y, F, S, chunk_size, hop_size, z_pitch,
                                                                                        crop_left, T_out, out_pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// ---- one IntraTransformer / InterTransformer ---------------------------------------------------------------------------------------
extern "C" size_t ctn_sfm_transformer_workspace_bytes(int B, int F, int d_ff, int layers, int pitch, int math) {
  if (B <= 0 || F <= 0 || d_ff <= 0 || layers <= 0 || pitch <= 0) return 0;
  const size_t big = (size_t)(3 * F > d_ff ? 3 * F : d_ff);
  size_t img = 0;
  for (int k = 0; k < 4; ++k) img += tf_img_bytes(F, d_ff, math, k);
  return up256((size_t)B * F * pitch * 4) * 2 + up256((size_t)B * big * pitch * 4) + img * layers + up256((size_t)2 * B * 8) + up256(4) +
         256;
}

extern "C" int ctn_sfm_transformer_fwd(const float* X, float* out, const float* const* w, int B, int F, int heads, int d_ff, int layers,
                                       int S, int C, int pitch, int intra, float eps, int math, void* workspace, size_t workspace_bytes,
                                       ctn_stream_t stream) {
  LaunchScope scope(X);
  if (!X || !out || !w || !workspace || heads <= 0 || d_ff <= 0 || layers <= 0) return CTN_EINVAL;
  CTN_TRY(state_check(B, F, S, C, pitch));
  for (int i = 0; i < SFM_LAYER_PTRS * layers + 3; ++i)
    if (!w[i]) return CTN_EINVAL;
  if (out == X) return CTN_EINVAL;
  if (math != CTN_MATH_FP32 && math != CTN_MATH_TF32 && math != CTN_MATH_TF32X3 && math != CTN_MATH_F16X3) return CTN_EINVAL;
  if (!attn_ok(F, heads)) return CTN_EUNSUPPORTED;
  const Seqs q = path_seqs(S, C, intra);
  if ((long long)B * q.nseq > 0x7fffffffLL || (q.len + ATT_Q - 1) / ATT_Q > 65535) return CTN_EUNSUPPORTED;
  if (q.len > SFM_PE_MAX) return CTN_EINVAL;  // past the positional encoding's rows
  if (pitch % CTN_TILE_T != 0 || (((uintptr_t)workspace) & 255) || (((uintptr_t)X) & 15)) return CTN_EALIGN;
  if (workspace_bytes < ctn_sfm_transformer_workspace_bytes(B, F, d_ff, layers, pitch, math)) return CTN_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int ntok = S * C;
  const size_t big = (size_t)(3 * F > d_ff ? 3 * F : d_ff);
  Carver cv(workspace);
  float* x = cv.take<float>((size_t)B * F * pitch);   // the residual stream of the layers
  float* o = cv.take<float>((size_t)B * F * pitch);   // attention output, then linear2's output
  float* g = cv.take<float>((size_t)B * big * pitch); // QKV, then out_proj's output, then linear1's
  float* imgs = nullptr;
  size_t per_layer = 0;
  for (int k = 0; k < 4; ++k) per_layer += tf_img_bytes(F, d_ff, math, k);
  if (per_layer) imgs = cv.take<float>(per_layer * layers / sizeof(float));
  double* stats = cv.take<double>((size_t)2 * B);
  float* zero = cv.take<float>(1);
  auto img = [&](int l, int k) -> float* {
    if (!imgs) return nullptr;
    size_t off = per_layer * l;
    for (int i = 0; i < k; ++i) off += tf_img_bytes(F, d_ff, math, i);
    return reinterpret_cast<float*>(reinterpret_cast<char*>(imgs) + off);
  };
  cudaError_t e;
  if ((e = cudaMemsetAsync(stats, 0, sizeof(double) * 2 * B, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(zero, 0, sizeof(float), st)) != cudaSuccess) return (int)e;
  // every weight image of the call in one batch (CTN_MAX_JOBS per launch)
  if (imgs) {
    WimgJob jobs[4 * 64];
    for (int l0 = 0; l0 < layers; l0 += 64) {
      const int nl = layers - l0 < 64 ? layers - l0 : 64;
      for (int l = 0; l < nl; ++l) {
        const float* const* p = w + SFM_LAYER_PTRS * (l0 + l);
        jobs[4 * l + 0] = WimgJob{p[0], img(l0 + l, 0), 3 * F, F};
        jobs[4 * l + 1] = WimgJob{p[2], img(l0 + l, 1), F, F};
        jobs[4 * l + 2] = WimgJob{p[4], img(l0 + l, 2), d_ff, F};
        jobs[4 * l + 3] = WimgJob{p[6], img(l0 + l, 3), F, d_ff};
      }
      CTN_TRY(ctn_pw_prepare_batch(jobs, 4 * nl, math, false, st));
    }
  }
  const float* const* fin = w + SFM_LAYER_PTRS * layers;  // pe, final norm gamma, beta
  k_sfm_pos_enc<<<dim3((pitch + 127) / 128, F, B), 128, 0, st>>>(X, fin[0], x, F, pitch, ntok, C, intra);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  for (int l = 0; l < layers; ++l) {
    const float* const* p = w + SFM_LAYER_PTRS * l;
    // x = norm1(x + out_proj(attention(in_proj(x))))
    CTN_TRY(pw_run(x, p[0], img(l, 0), g, B, 3 * F, F, ntok, pitch, math, nullptr, nullptr, nullptr, st));
    CTN_TRY(launch_attn(g, p[1], o, B, F, heads, pitch, q, st));
    CTN_TRY(pw_run(o, p[2], img(l, 1), g, B, F, F, ntok, pitch, math, nullptr, nullptr, nullptr, st));
    CTN_TRY(launch_token_ln(x, g, p[3], p[8], p[9], x, B, F, ntok, pitch, eps, st));
    // x = norm2(x + linear2(relu(linear1(x))))
    CTN_TRY(pw_run(x, p[4], img(l, 2), g, B, d_ff, F, ntok, pitch, math, p[5], zero, stats, st));
    CTN_TRY(pw_run(g, p[6], img(l, 3), o, B, F, d_ff, ntok, pitch, math, nullptr, nullptr, nullptr, st));
    CTN_TRY(launch_token_ln(x, o, p[7], p[10], p[11], x, B, F, ntok, pitch, eps, st));
  }
  return launch_seq_norm(x, X, fin[1], fin[2], out, B, F, pitch, ntok, q, eps, st);
}

// ---- separator tail + decoder ----------------------------------------------------------------------------------------------------
extern "C" size_t ctn_sfm_tail_workspace_bytes(int B, int N, int Bc, int S, int pitch) {
  if (B <= 0 || N <= 0 || Bc <= 0 || S <= 0 || pitch <= 0) return 0;
  const size_t R = (size_t)B * S;
  return up256((size_t)B * Bc * pitch * 4) + up256(R * N * pitch * 4) * 2 + up256(R * 2 * N * pitch * 4) + up256((size_t)2 * N * N * 4) +
         up256((size_t)2 * N * 4) + up256(ctn_pw_wimg_bytes(S * N, Bc, CTN_MATH_TF32X3)) + up256(ctn_pw_wimg_bytes(2 * N, N, CTN_MATH_TF32X3)) +
         up256(ctn_pw_wimg_bytes(N, N, CTN_MATH_TF32X3)) + up256(2 * R * 8) + up256(4) + 256;
}

extern "C" int ctn_sfm_tail_fwd(const float* y, const float* w, const float* prelu, const float* map_w, const float* map_b,
                                const float* gtu_w, const float* gtu_b, const float* gate_w, const float* gate_b, const float* bout_w,
                                const float* bout_b, const float* dec_w, float* out, float* latent, float* what, int B, int N, int Bc,
                                int S, int frames, int pitch, int L, int stride, int crop_left, int T, int mask_relu, int math,
                                void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(y);
  if (!y || !w || !prelu || !map_w || !map_b || !gtu_w || !gtu_b || !gate_w || !gate_b || !bout_w || !bout_b || !dec_w || !out || !what ||
      !workspace || B <= 0 || N <= 0 || Bc <= 0 || S <= 0 || frames <= 0)
    return CTN_EINVAL;
  if (math != CTN_MATH_FP32 && math != CTN_MATH_TF32 && math != CTN_MATH_TF32X3 && math != CTN_MATH_F16X3) return CTN_EINVAL;
  if (pitch < frames || pitch % CTN_TILE_T != 0 || (((uintptr_t)workspace) & 255)) return CTN_EALIGN;
  if ((((uintptr_t)y) | ((uintptr_t)w) | ((uintptr_t)what)) & 15) return CTN_EALIGN;
  if (workspace_bytes < ctn_sfm_tail_workspace_bytes(B, N, Bc, S, pitch)) return CTN_EWORKSPACE;
  if ((long long)B * S > 65535) return CTN_EUNSUPPORTED;
  CTN_TRY(ctn_decoder_check(B * S, N, frames, pitch, L, stride, crop_left, T));
  cudaStream_t st = (cudaStream_t)stream;
  const int R = B * S;
  Carver cv(workspace);
  float* yp = cv.take<float>((size_t)B * Bc * pitch);
  float* m = cv.take<float>((size_t)R * N * pitch);
  float* u = cv.take<float>((size_t)R * N * pitch);
  float* g = cv.take<float>((size_t)R * 2 * N * pitch);
  float* wcat = cv.take<float>((size_t)2 * N * N);
  float* bcat = cv.take<float>((size_t)2 * N);
  float* img_map = cv.take<float>(ctn_pw_wimg_bytes(S * N, Bc, CTN_MATH_TF32X3) / 4);
  float* img_gtu = cv.take<float>(ctn_pw_wimg_bytes(2 * N, N, CTN_MATH_TF32X3) / 4);
  float* img_out = cv.take<float>(ctn_pw_wimg_bytes(N, N, CTN_MATH_TF32X3) / 4);
  double* stats = cv.take<double>((size_t)2 * R);
  float* one = cv.take<float>(1);
  const bool tc = math != CTN_MATH_FP32;
  cudaError_t e;
  // [map; map_gate] as one 2N x N contraction
  if ((e = cudaMemcpyAsync(wcat, gtu_w, sizeof(float) * N * N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpyAsync(wcat + (size_t)N * N, gate_w, sizeof(float) * N * N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpyAsync(bcat, gtu_b, sizeof(float) * N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpyAsync(bcat + N, gate_b, sizeof(float) * N, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(stats, 0, sizeof(double) * 2 * R, st)) != cudaSuccess) return (int)e;
  if (tc) {
    const WimgJob jobs[3] = {{map_w, img_map, S * N, Bc}, {wcat, img_gtu, 2 * N, N}, {bout_w, img_out, N, N}};
    CTN_TRY(ctn_pw_prepare_batch(jobs, 3, math, false, st));
  }
  const size_t n = (size_t)B * Bc * pitch;
  int gp = (int)((n + 255) / 256);
  if (gp > 1024) gp = 1024;
  k_sfm_prelu<<<gp, 256, 0, st>>>(y, yp, prelu, n, frames, pitch, one);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  CTN_TRY(pw_run(yp, map_w, tc ? img_map : nullptr, m, B, S * N, Bc, frames, pitch, math, map_b, one, stats, st));
  CTN_TRY(pw_run(m, wcat, tc ? img_gtu : nullptr, g, R, 2 * N, N, frames, pitch, math, bcat, one, stats, st));
  int gx = (int)(((size_t)N * pitch + 255) / 256);
  if (gx > 256) gx = 256;
  k_sfm_gtu<<<dim3(gx, R), 256, 0, st>>>(g, u, N, frames, pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  CTN_TRY(pw_run(u, bout_w, tc ? img_out : nullptr, m, R, N, N, frames, pitch, math, bout_b, one, stats, st));
  k_sfm_mask<<<dim3(gx, R), 256, 0, st>>>(m, w, what, S, N, frames, pitch, mask_relu);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  CTN_TRY(ctn_decoder_fwd(what, dec_w, out, R, N, frames, pitch, L, stride, crop_left, T, stream));
  if (latent) CTN_TRY(ctn_copy_from_pitch(what, latent, R * N, frames, pitch, st));
  return CTN_OK;
}
