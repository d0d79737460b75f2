// Internal (non-ABI) declarations shared by the .cu translation units.
#pragma once
#include "ctn_common.cuh"

// ---- folded / derived parameters (built per forward by ctn_prep_*; weights may change every step) ----------
// For a 1x1 conv applied to a gLN output,  W (gamma*(u-mu)*rstd + beta) + b  ==  rstd * (W diag(gamma)) u
//   + (b + W beta) - mu*rstd * (W gamma):   Wf = W diag(gamma),  v1 = b + W beta,  v2 = W gamma.
struct FoldedConv {
  float* Wf;  // (M, K)
  float* v1;  // (M)
  float* v2;  // (M)
  float* vb;  // (M) nullable: bound of |W gLN(u) + b| per row = sum_k |W[m][k]| (|gamma_k| R + |beta_k|) + |b_m|, R = sqrt(#elements
              // of the gLN group) >= max |normalised value|  (activation envelope of the fp16-piece mode)
};

inline size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }

// Workspace carving: 256-byte aligned sub-buffers of one allocation.  base == nullptr only measures (off = bytes needed), so an
// entry's workspace query is its carve run on Carver(nullptr) and cannot drift from the carve itself.
struct Carver {
  char* base;
  size_t off;
  explicit Carver(void* b) : base((char*)b), off(0) {}
  template <typename T>
  T* take(size_t count) {
    off = up256(off);
    T* p = base ? (T*)(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};

#define CTN_MAX_BLOCKS 64
#define CTN_MAX_P 8  // most depthwise taps the training path takes

// Config checks shared by every pipeline (ctn_api.cu): CTN_EINVAL for a value no pipeline accepts, CTN_EUNSUPPORTED for one
// outside the stack's envelope.  check_tcn_cfg covers the separator stack's fields; max_layers is the longest run of layers
// with dilations 2^l (20), or CTN_MAX_BLOCKS where the caller passes the dilations itself.  check_model_cfg adds the
// encoder / mask / decoder fields.  Each pipeline adds its own envelope refusals after these.
int check_tcn_cfg(const ctn_config_t* c, int max_layers = 20);
int check_model_cfg(const ctn_config_t* c);

// launch grid of the (B, C, pitch) streaming kernels: a block walks channels c = blockIdx.x, += gridDim.x
inline dim3 grid_cb(int C, int B) { return dim3(C < 1024 ? C : 1024, B); }
// epilogue / prologue selectors of the pointwise (1x1) contraction kernels
enum { PRO_NONE = 0, PRO_PRELU = 1, PRO_DW = 2, PRO_RES = 3 };
enum { EPI_RAW = 0, EPI_HEAD = 1, EPI_H = 2, EPI_MASK = 3, EPI_MASKDEC = 4 };

struct PwArgs {
  const float* A;      // (B, K, pitch) activations
  const float* W;      // (M, K) row-major weights
  float* D;            // (B, M, pitch)
  int B, M, K, frames, pitch;
  // prologue
  const float* pro_slope;  // PRO_PRELU / PRO_DW: PReLU slope (1)
  // PRO_DW (tensor-core path): A is h (B,K,pitch); the producer computes u = PReLU(dwconv3(gLN1(h)) + bd) on the fly
  const float* dw_norm_g;  // (K) gLN1 gamma
  const float* dw_norm_b;  // (K) gLN1 beta
  const float* dw_w;       // (K,3) depthwise taps
  const float* dw_b;       // (K)
  const double* dw_stats_in;   // (B,2) (sum, sumsq) of h
  double* dw_stats_out;        // (B,2) += (sum, sumsq) of u
  int dw_dilation, dw_pad_left;
  float dw_eps;
  // epilogue
  const float* bias;       // EPI_H / EPI_MASK: (M)
  const float* slope;      // EPI_H: PReLU slope (1)
  const float* v1;         // EPI_HEAD
  const float* v2;         // EPI_HEAD
  const double* stats_in;  // EPI_HEAD: (B,2) of the input tensor
  double n_in;             // EPI_HEAD: element count of a gLN group of the input
  float eps;               // EPI_HEAD
  double* stats_out;       // EPI_H: (B,2) += (sum, sumsq) over valid outputs
  int store_pre;           // EPI_H (tensor-core path only): store W A + bias (pre-activation) instead of PReLU(.); stats unchanged
  const float* wenc;       // EPI_MASK: encoder output (B, Nb, pitch)
  int Nb;                  // EPI_MASK: n_basis
  float* mask_out;         // EPI_MASK: optional raw mask output (B, M, pitch)
  int mask_logits;         // EPI_MASK: 1 = store the LOGITS (W A + bias) to D, no sigmoid, no w product (softmax masks take a second pass)
  // EPI_MASKDEC: mask 1x1 + sigmoid + w*mask + transposed-conv decoder + crop in one epilogue; w_hat is never
  // materialised.  D = estimates (B, M/Nb, dec_T_out) contiguous, ZERO-initialised by the caller (tile seams are red.add'ed)
  const float* dec_w;      // (Nb, 1, 16) decoder basis, kernel 16 / stride 8
  int dec_crop_left, dec_T_out;
  // PRO_RES (tensor-core path): the operand is the UPDATED residual stream  x_new = A + rstd*res_r[:K] + (v1 - mean*rstd*v2)
  // (the deferred gLN2 of the previous block); CTAs with n-tile 0 also store x_new to res_x_out (ping-pong buffer).
  const float* res_r;       // (B, res_Mt, pitch) raw [out;skip] contraction of the previous block; rows [0,K) are used
  int res_Mt;
  const float* res_v1;      // (>=K) folded bias vectors of the previous block
  const float* res_v2;
  const double* res_stats;  // (B,2) stats2 of the previous block
  double res_n;
  float res_eps;
  float* res_x_out;         // (B, K, pitch)
  // tensor-core path only
  const float* wimg;       // pre-swizzled hi/lo weight images (ctn_pw_prepare)
  // fp16-piece mode: power-of-two scale of the activation operand (device scalar, nullable = 1), chosen per forward from a
  // bound on |operand| derived from the weights alone (ctn_act_scales) so that fp16 can never saturate; undone in the epilogue
  const float* act_scale;
  const float* dw_params;  // PRO_DW: packed per-channel parameters [ceil16(K)][8] (ctn_act_scales)
  // PRO_DW, training forward : A holds the PRE-activation h_pre = W1 x + b1 (the backward needs it), the producer
  // applies PReLU(dw_in_slope) on load; the depthwise pre-activation u_pre is stored to dw_u_pre_out (B, K, pitch)
  const float* dw_in_slope;
  float* dw_u_pre_out;
};

// gLN per sample over the n contiguous values of each of B samples (ctn_dptnet.cu): ctn_sample_gln_stats sums x = z + z2 (z2
// nullable) in double over G = ctn_sample_gln_parts(n) slices per sample into part double[B][G][2] [1 launch, no atomics];
// ctn_sample_gln_apply normalises z in place, f = i % F [1 launch].  Every reader of part sums the G partials in slice order
// (sample_gln_mean_rstd), so repeated calls give the same bits.
int ctn_sample_gln_parts(size_t n);
int ctn_sample_gln_stats(const float* z, const float* z2, size_t n, int B, double* part, int G, cudaStream_t st);
int ctn_sample_gln_apply(float* z, size_t n, int B, int F, const double* part, int G, const float* gamma, const float* beta, float eps,
                         cudaStream_t st);
// (mean, rstd) of sample b from its G partials, summed in slice order by thread 0 into st (shared, double[2]); the caller's
// whole CTA must reach it (it holds a barrier)
__device__ __forceinline__ float2 sample_gln_mean_rstd(const double* __restrict__ part, int G, int b, double n, float eps, double* st) {
  if (threadIdx.x == 0) {
    double s = 0.0, ss = 0.0;
    for (int g = 0; g < G; ++g) { s += part[((size_t)b * G + g) * 2]; ss += part[((size_t)b * G + g) * 2 + 1]; }
    st[0] = s; st[1] = ss;
  }
  __syncthreads();
  return gln_mean_rstd(st, n, eps);
}

// One 1x1 contraction (ctn_wgmma.cu).  math is the model's mode: fp32 runs the FFMA kernel; the tensor-core modes run the wgmma
// kernel, on fp16 pieces in the f16x3 mode exactly when the operand has a static bound (a.act_scale), on tf32 pieces otherwise.
// wimg_scratch == nullptr: a.wimg already holds the weight image (ctn_pw_prepare / ctn_pw_prepare_batch with the same
// math); otherwise the image of a.W is built into wimg_scratch (ctn_pw_wimg_bytes) first.
int ctn_pw(const PwArgs& a, int pro, int epi, int math, float* wimg_scratch, cudaStream_t st);
size_t ctn_pw_wimg_bytes(int M, int K, int math);
// weight image of a.W (a.M, a.K) for ctn_pw(a, .., math, nullptr, ..); nothing to do in the fp32 mode
int ctn_pw_prepare(const PwArgs& a, int math, float* wimg, cudaStream_t st);
// device scalar 1.0 of the current device (one __device__ constant, ctn_wgmma.cu): the PReLU slope that turns the PReLU of the
// EPI_H epilogue or the PRO_PRELU prologue into an identity.  nullptr when the symbol cannot be resolved.
const float* ctn_device_one();
// One 1x1 contraction of a pitched (B, K, pitch) operand from a prebuilt weight image (wimg; none in the fp32 mode): EPI_RAW
// without bias; with bias, EPI_H with the PReLU slope (ctn_device_one(): a plain bias add) and its statistics in stats (double[2 B],
// accumulated, never read back by the callers).
int ctn_pw_run(const float* A, const float* W, const float* wimg, float* D, int B, int M, int K, int frames, int pitch, int math,
               const float* bias, const float* slope, double* stats, cudaStream_t st);
// EPI_MASKDEC (PRO_PRELU) applies to this contraction: fp16-piece mode, n_basis a multiple of 128, K <= 128 (the operand stays
// resident in shared memory), decoder kernel 16 / stride 8 (caller)
int ctn_pw_maskdec_supported(const PwArgs& a, int math);

// wgmma weight gradient of a 1x1 conv (ctn_wgrad_wgmma.cu): dW (M,K) += sum_{b,t} dY[b][m][t] X[b][k][t]; rows
// [0,split_row) -> dWa, rest -> dWb (nullable).  dW must be zero-initialised by the caller (split-K partials are added).
int ctn_wgrad_wgmma(const float* dy, size_t dy_bs, const float* x, size_t x_bs, float* dWa, float* dWb, int split_row, int M,
                    int K, int B, int frames, int pitch, int math, cudaStream_t st);

// weight preparation of one or many convs: gLN folds into rows [row_offset, row_offset + M) of a FoldedConv (R as in its vb),
// weight images for ctn_pw; up to CTN_MAX_JOBS jobs per launch (they travel in the kernel parameter block)
struct FoldJob { const float *W, *bias, *gamma, *beta; FoldedConv out; int M, K, row_offset; float R; };
struct WimgJob { const float* W; float* wimg; int M, K; };
#define CTN_MAX_JOBS 48
int ctn_fold_batch(const FoldJob* jobs, int n, cudaStream_t st);
// weight images of the jobs, one launch per job when they take different pieces; bounded: every one of these contractions
// carries an operand scale (see ctn_pw)
int ctn_pw_prepare_batch(const WimgJob* jobs, int n, int math, bool bounded, cudaStream_t st);
// largest ctn_pw_wimg_bytes over n (M, K) shapes; 256 in the fp32 mode, which builds no images
size_t ctn_pw_wimg_max_bytes(const int (*shapes)[2], int n, int math);

// Activation envelope of the fp16-piece mode.  Per residual block i the two operands that meet the tensor core as fp16
// pieces are x_i (pw1) and u_i (fused depthwise output, pw2); the mask contraction sees PReLU(skip sum).  From the weights
// alone:  |gLN(.)| <= |gamma| R + |beta| with R = sqrt(#elements of the group);  |u_c| <= max(1,|a2|) ((|g1_c| R + |b1_c|) sum_k |wd_ck| + |bd_c|);
// |x_{i+1}| <= |x_i| + max_n vb_out_i[n];  |skip| <= sum_i max_n vb_skip_i[n].  scales[2i] / [2i+1] / [2n] receive the powers of two
// that map those bounds to <= 2^15; dwp_i receives the packed depthwise parameters {g1, b1, w0, w1, w2, bd, 0, 0} per channel.
struct ScaleJob { const float *vb, *g1, *b1, *dw_w, *dw_b, *slope2; float* dwp; int has_out; };
struct ScaleJobs {
  ScaleJob j[CTN_MAX_BLOCKS];
  int n, Bc, Sc, H, P;
  const float* x0_bound;  // device: x0_n candidates whose max bounds |x_0|
  int x0_n;
  const float* mask_slope;  // nullable
  float R;
  float* scales;  // [2n + 1]
};
int ctn_act_scales(const ScaleJobs& jobs, cudaStream_t st);
// max |x| over rows x frames of a pitched tensor -> *out (float, must be zeroed by the caller)
int ctn_absmax_pitch(const float* x, int rows, int frames, int pitch, float* out, cudaStream_t st);
// Where a forward left its activation envelope: the workspace re-carved the way the forward carved it (ctn_api.cu), for the
// verification hook to read back.  path ENV_TCN: ctn_tcn_fwd, or ctn_tcn_blocks_fwd with num_blocks = 1, num_layers = n_blocks;
// ENV_MODEL: ctn_convtasnet_fwd / ctn_separator_fwd; ENV_TRAIN: ctn_convtasnet_fwd_train (fused TCN only).  x0_bound holds the
// x0_n candidates the scales took |x_0| from (the measured max |x| of a stand-alone TCN, the head's row bounds of a model).
enum { ENV_TCN = 0, ENV_MODEL = 1, ENV_TRAIN = 2 };
struct EnvelopeView { const float* scales; const float* dwp[CTN_MAX_BLOCKS]; const float* vb[CTN_MAX_BLOCKS]; const float* x0_bound; int n, x0_n; };
int ctn_envelope_view(const ctn_config_t* c, int B, int frames, int path, void* mem, EnvelopeView* v);
// training workspace (ctn_train.cu): the region of the fused TCN forward (nullptr when the config does not fuse it) and the head's
// row bounds
void ctn_train_tcn_region(const ctn_config_t* c, int B, int frames, void* mem, void** tcn_mem, const float** head_vb);

// training forward of the TCN through the fused inference kernels (ctn_api.cu); per-block buffers owned by the training workspace
struct TcnTrainHooks { float* const* x_keep; float* const* hpre; float* const* upre; };
size_t ctn_tcn_train_ws_bytes(const ctn_config_t* c, int B, int pitch);
int ctn_tcn_train_fwd(const ctn_config_t* c, const ctn_block_params_t* blocks, void* mem, size_t mem_bytes, const TcnTrainHooks* hooks,
                      double* stats, float* skip, const float* x0_bound, int x0_n, const float* mask_slope, const float** mask_scale,
                      int B, int frames, int pitch, cudaStream_t st);

// mask_nonlinear = 'softmax' (src/models/conv_tasnet.py:345-357, 375-376: nn.Softmax(dim=1) over ALL S*N channels before the view):
// in place on the logits (B, M, pitch): what = softmax_m(logits) * w[m % Nb]; mask_out (nullable) receives the softmax itself
int ctn_softmax_mask(float* logits_what, const float* wenc, float* mask_out, int B, int M, int Nb, int frames, int pitch, cudaStream_t st);

// depthwise stage: u = PReLU(dwconv(gLN1(h))) (+ stats2), all (B,H,pitch)
int ctn_dw_fwd(const float* h, float* u, const float* norm_g, const float* norm_b, const float* dw_w, const float* dw_b,
               const float* slope, const double* stats_in, double* stats_out, int B, int H, int frames, int pitch, int P,
               int dilation, float eps, cudaStream_t st);

// finishing of a block with an output head: x += rstd2*outraw[:Bc] + c, outraw (B, Bc + Sc, pitch); its skip rows are reduced
// by ctn_skip_reduce
int ctn_finish_fwd(const float* outraw, const FoldedConv f, const double* stats2, double n2, float eps, float* x, int B, int Bc,
                   int Sc, int frames, int pitch, cudaStream_t st);

// deferred skip reduction: skip[b][m][t] = sum_i ( rstd2_i[b] * r_i[b][off_i + m][t] + (v1_i[off_i+m] - mean_i rstd_i v2_i[off_i+m]) )
// over all residual blocks i -- reads every block's skip rows ONCE instead of read-modify-writing the accumulator per block
struct SkipJob { const float* r; const float* v1; const float* v2; const double* stats2; int off; int Mt; };
struct SkipJobs { SkipJob j[CTN_MAX_BLOCKS]; int n; };
int ctn_skip_reduce(const SkipJobs& jobs, double n2, float eps, float* skip, int B, int Sc, int frames, int pitch, cudaStream_t st);

// Online (chunk-by-chunk) inference, shared by causal Conv-TasNet (ctn_online.cu) and causal LSTM-TasNet (ctn_tasnet.cu).  The
// state's header holds T0, the samples pushed since the reset.  Every kernel of a push reads it; the decoder, the push's last
// kernel, advances it once all its CTAs have read it (ticket).
struct OnlineHdr {
  long long T0;     // samples pushed since the reset
  unsigned ticket;  // CTAs of the decoder that have finished reading T0
  unsigned pad;
};
struct OnlineFrames { long long T0, F0; int nv; };
// frames done before this push (F0) and completed by it (nv), from the device counter
__device__ __forceinline__ OnlineFrames push_frames(const OnlineHdr* hdr, int L, int S, int n) {
  OnlineFrames f;
  f.T0 = *(const volatile long long*)&hdr->T0;
  const long long T1 = f.T0 + n;
  f.F0 = f.T0 >= L ? (f.T0 - L) / S + 1 : 0;
  const long long F1 = T1 >= L ? (T1 - L) / S + 1 : 0;
  f.nv = (int)(F1 - f.F0);
  return f;
}
// Encoder over [carry | chunk] of B streams (k_online_enc, ctn_encoder_fwd's order): w (B, N, pitch), columns [nv, pitch) zero;
// carry [B][L - S] takes the last L - S samples.  Shared memory (L - S + n) floats, at most 200 KB.  1 launch.
size_t ctn_online_enc_smem(int L, int S, int n);
int ctn_online_enc(const float* x, const float* W, float* carry, float* w, const OnlineHdr* hdr, int B, int N, int L, int S, int n,
                   int pitch, int relu, cudaStream_t st);
// Decoder over [history | chunk] of BS rows (k_online_dec, ctn_decoder_fwd's summation order) with the offline crop.  push = 1:
// y (BS, n), the history [BS][N][L/S - 1] takes the last frames and the decoder advances T0 by n; push = 0 (flush): y (BS, D)
// from the history alone, nothing advanced.  N (L/S - 1) floats of shared memory, at most 48 KB.  1 launch.
int ctn_online_dec(const float* what, const float* Wd, float* hist, float* y, OnlineHdr* hdr, int BS, int N, int L, int S, int n, int pitch,
                   int push, cudaStream_t st);

// the refusals of ctn_decoder_fwd, for callers that must refuse before their own launches (ctn_sep_tail_fwd)
int ctn_decoder_check(int BS, int N, int frames, int in_pitch, int L, int stride, int crop_left, int T_out);

int ctn_copy_to_pitch(const float* src, float* dst, int rows, int frames, int pitch, cudaStream_t st);
int ctn_copy_from_pitch(const float* src, float* dst, int rows, int frames, int pitch, cudaStream_t st);

// cLN (src/modules/norm.py:78-90) on the padded (B, C, pitch) layout, in place allowed; scratch double[B][frames][2]
int ctn_cln_pitch_fwd(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int frames, int pitch,
                      float eps, double* scratch, cudaStream_t st);

// cLN in pieces, for the causal training path: the prefix sums (S_t, Q_t) of act(x) (act = PReLU(slope), identity when slope is
// null) into st double[B][frames][2] [2 launches], with mi (nullable, float2[B][frames]) the table of (mean_t, 1 / (std_t + eps));
// and the normalisation y = cLN(act(x)) from st [1 launch].  ctn_cln_pitch_fwd is the two in a row without a slope.
int ctn_cln_stats(const float* x, const float* slope, int B, int C, int frames, int pitch, float eps, double* st, float2* mi,
                  cudaStream_t stream);
int ctn_cln_apply(const float* x, const float* slope, const float* gamma, const float* beta, float* y, int B, int C, int frames,
                  int pitch, float eps, const double* st, cudaStream_t stream);
// cLN (+ PReLU(slope) in front, slope nullable) backward from the forward's st: dy -> dpre (may alias dy); += dgamma, dbeta, dslope,
// dbias (the last two nullable).  Scratch: part double[ctn_cln_bwd_part_doubles(B, frames)], tab float4[B][frames].  3 launches.
size_t ctn_cln_bwd_part_doubles(int B, int frames);
int ctn_cln_bwd_pitch(const float* dy, const float* pre, float* dpre, const float* slope, const float* gamma, const double* st,
                      float eps, double* part, float4* tab, float* dgamma, float* dbeta, float* dslope, float* dbias, int B, int C,
                      int frames, int pitch, cudaStream_t stream);
// Depthwise conv of the causal training path (ctn_causal_train.cu), pad_left = (P - 1) dil; mi: the cLN1 table of ctn_cln_stats.
// upre = dwconv(cLN1(PReLU(hpre; slope1))) + bd
int ctn_cdw_train_fwd(const float* hpre, float* upre, const float2* mi, const float* g1, const float* b1, const float* wd,
                      const float* bd, const float* slope1, int B, int C, int frames, int pitch, int P, int dil, cudaStream_t st);
// dhn = dwconv^T(dupre) ; dwd += the taps' gradients, hn = cLN1(PReLU(hpre)) rebuilt on load.  P <= CTN_MAX_P
int ctn_cdw_bwd(const float* dupre, const float* hpre, float* dhn, const float2* mi, const float* g1, const float* b1,
                const float* slope1, const float* wd, float* dwd, int B, int C, int frames, int pitch, int P, int dil,
                cudaStream_t st);

// Causal (cLN) models: un-fused pipeline in the reference's operation order (ctn_causal.cu).  The cumulative statistics of
// cLN depend on every earlier frame, so the gLN tricks of the fused stack (statistics from the producing epilogue, affine
// folded into the next contraction) do not apply; each block is contraction -> cLN -> causal depthwise -> cLN -> contraction.
size_t ctn_causal_ws_bytes(const ctn_config_t* c, int B, int pitch);
// x: (B, Bc, pitch) block-0 input (updated in place); skip: (B, Sc, pitch) result; h, u: (B, H, pitch) scratch
int ctn_causal_tcn(const ctn_config_t* c, const ctn_block_params_t* blocks, float* x, float* skip, float* h, float* u, int B,
                   int frames, int pitch, void* cws, cudaStream_t st);
// separator head for causal models: x0 = Wb cLN0(w) + bb;  tmp: (B, N, pitch) scratch
int ctn_causal_head(const ctn_config_t* c, const ctn_params_t* p, const float* w, float* tmp, float* x0, int B, int frames,
                    int pitch, void* cws, cudaStream_t st);
// The un-folded pipelines' per-frame kernels on their own (causal, online, un-fused training forward):  rows of r (B, Mt, pitch):
// m < Bc (has_out): xout = xin + r + bo[m] (xin == xout: in place); else skip (+)= r + bs[j] (skip_init: =);  and
// y[b][c][t] += bias[c].  Columns [frames, pitch) are written as zero.
int ctn_res_skip_fwd(const float* r, int Mt, const float* xin, float* xout, float* skip, const float* bo, const float* bs, int Bc, int Sc,
                     int has_out, int skip_init, int B, int frames, int pitch, cudaStream_t st);
int ctn_bias_rows_fwd(float* y, const float* bias, int C, int B, int frames, int pitch, cudaStream_t st);
// u = PReLU(dwconv(h) + bd), P taps at dilation dil, h = 0 outside [0, frames) (the causal layout passes pad_left = (P-1) dil)
int ctn_dw_plain_fwd(const float* h, float* u, const float* wd, const float* bd, const float* slope, int B, int C, int frames, int pitch,
                     int P, int dil, int pad_left, cudaStream_t st);
// stats[b] += (sum, sumsq) over c < C, t < frames of a (B, C, pitch) tensor, every element summed in double (ctn_api.cu)
int ctn_stats_pitch(const float* x, int B, int C, int frames, int pitch, double* stats, cudaStream_t st);
// a block's [out_w; skip_w] (skip_w alone when it has no output head) -> wcat (Mt, H), stream-ordered device copies
int ctn_block_wcat(const ctn_block_params_t& q, int Bc, int Sc, int H, float* wcat, cudaStream_t st);

// Streaming and filter-bank gradient kernels of the training path (ctn_train.cu), one launcher each.  ctn_convtasnet_fwd_train /
// ctn_convtasnet_bwd and the verification hook (ctn_probe.cu) launch them only through these, so both run the same grid shapes
// and split counts.  Layout (B, C, pitch) as in the kernels' comments there; "+=" outputs accumulate with atomics.
// y = y + bias[c] in place ; stats[b] += (sum, sumsq) of PReLU(y)
int ctn_bias_prelu_stats(float* y, const float* bias, const float* slope, double* stats, int B, int C, int frames, int pitch,
                         cudaStream_t st);
// upre = dwconv(gLN1(PReLU(hpre; slope1))) + bd (P taps, dilation dil) ; stats2[b] += (sum, sumsq) of PReLU(upre; slope2)
int ctn_dw_train_fwd(const float* hpre, float* upre, const float* g1, const float* b1, const float* wd, const float* bd,
                     const float* slope1, const float* slope2, const double* stats1, double* stats2, int B, int C, int frames,
                     int pitch, int P, int dil, int pad_left, double n1, float eps, cudaStream_t st);
// y = gLN(act(pre)), act = PReLU(slope) or identity (slope == nullptr)
int ctn_act_norm(const float* pre, float* y, const float* slope, const float* g, const float* bt, const double* stats, double n,
                 float eps, int B, int C, int frames, int pitch, cudaStream_t st);
// gLN (+ PReLU(slope) in front, slope nullable) backward: dy -> dpre (may alias dy); += dgamma, dbeta, dslope, dbias (the last
// two nullable).  reduced: sums / dgamma / dbeta were already accumulated by the producer of dy (ctn_dw_bwd), only the apply runs.
int ctn_gln_prelu_bwd(const float* dy, const float* pre, float* dpre, const float* slope, const float* g, const double* stats,
                      double n, float eps, double* sums, float* dgamma, float* dbeta, float* dslope, float* dbias, int B, int C,
                      int frames, int pitch, cudaStream_t st, bool reduced = false);
// depthwise conv backward: d_hn, += dwd, and phase 1 of the gLN1 backward on d_hn (+= sums, dgamma, dbeta)
int ctn_dw_bwd(const float* dupre, const float* hpre, float* dhn, const float* slope1, const float* g1, const float* b1,
               const double* stats1, double n1, float eps, const float* wd, float* dwd, double* sums, float* dgamma, float* dbeta,
               int B, int C, int frames, int pitch, int P, int dil, int pad_left, cudaStream_t st);
// sigmoid-mask backward: dwhat (B, S*N, pitch) -> d_mpre in place ; dwprod (B, N, pitch) = sum_s dwhat * mask
int ctn_mask_bwd(float* dwhat, const float* w, const float* mask, float* dwprod, int B, int S, int N, int frames, int pitch,
                 cudaStream_t st);
// softmax-mask backward (softmax over all S*N channels of a frame): dwhat (B, S*N, pitch) -> d_z = m * (dwhat * w - dot) in place,
// dot = sum_n w * dwprod ; dwprod (B, N, pitch) = sum_s dwhat * mask.  Pad lanes [frames, pitch) of both are written as 0
int ctn_softmax_mask_bwd(float* dwhat, const float* w, const float* mask, float* dwprod, int B, int S, int N, int frames, int pitch,
                         cudaStream_t st);
int ctn_prelu_apply(const float* x, float* y, const float* slope, int B, int C, int frames, int pitch, cudaStream_t st);
// dpre = dy * (pre > 0 ? 1 : a) (may alias dy) ; dslope += sum_{pre <= 0} dy * pre
int ctn_prelu_bwd(const float* dy, const float* pre, float* dpre, const float* slope, float* dslope, int B, int C, int frames,
                  int pitch, cudaStream_t st);
// dw = dw + dwprod, zeroed where !(w > 0) when relu
int ctn_dw_combine(float* dw, const float* dwprod, const float* w, int relu, int B, int C, int frames, int pitch, cudaStream_t st);
// dst[b][c] (+)= src[b][c] for c < C with independent batch strides (floats)
int ctn_rows(float* dst, size_t dst_bs, const float* src, size_t src_bs, int C, int B, int accumulate, int frames, int pitch,
             cudaStream_t st);
// Wt (K, M) = W (M, K)^T
int ctn_transpose(const float* W, float* Wt, int M, int K, cudaStream_t st);
// dW (M, K) += sum dY X^T; rows [0, split_row) -> dWa, the rest -> dWb (nullable).  math: the model's numeric mode (fp32: the
// FFMA split-K kernel; otherwise ctn_wgrad_wgmma)
int ctn_wgrad(int math, const float* dy, size_t dy_bs, const float* x, size_t x_bs, float* dWa, float* dWb, int split_row, int M,
              int K, int B, int frames, int pitch, cudaStream_t st);
// filter-bank weight gradient dW (N, C, L) += sum_{r,f} act[r][n][f] * sig[r*C + c][f*stride + k - pad_left] (signal rows of T
// samples, C per act row)
int ctn_encdec_wgrad(const float* act, const float* sig, float* dW, int R, int N, int C, int frames, int pitch, int T, int L, int stride,
                     int pad_left, cudaStream_t st);
// out[c] += sum_{b, t < frames} dy[b][c][t]
int ctn_rowsum(const float* dy, size_t bs, int C, int B, int frames, int pitch, float* out, cudaStream_t st);

// Batched tiled Cholesky of BSS Eval (ctn_bss.cu).  nmat row-major N x N matrices (N a multiple of BSS_NB); the factor L
// overwrites the lower triangle.  W: the inverse of every diagonal tile of L, (nmat, N/64, 64, 64), zero above the diagonal.
// flag[mat] = 1 when a pivot was not positive and finite.
#define BSS_NB 64
struct MatSet {
  double* A;
  double* W;
  int* flag;
  int N, nt, nmat;
};
// factor every matrix of s: 3 nt - 2 launches
int ctn_chol_factor(const MatSet& s, cudaStream_t st);
// G x = b in place for nrhs right-hand sides per matrix, rhs (nmat, nrhs, N): one CTA per (matrix, right-hand side), 1 launch
int ctn_chol_solve_cols(const MatSet& s, double* rhs, int nrhs, cudaStream_t st);
// G X = B for nrhs <= 8 right-hand sides per matrix, rhs (nmat, N, nrhs) row-major: X overwrites rhs, tmp (same size) holds the
// forward sweep's result.  Each sweep reads every factor tile once for all columns (ctn_bss_images.cu), 2 nt launches
int ctn_chol_solve_multi(const MatSet& s, double* rhs, double* tmp, int nrhs, cudaStream_t st);
