/* ctn_b200.h -- C ABI of the H100-native (sm_90a) Conv-TasNet separation path.
 *
 * The reference (tky823/DNN-based_source_separation) has NO native/FFI layer: the path sits behind
 * Python nn.Module classes (SURVEY.md section 8b).  This header is therefore the boundary a maintainer would
 * bind from those classes (ctypes stub shown in INTEGRATION.md).  Each entry point names the reference
 * interface it replaces (file:line relative to the reference root).
 *
 * Conventions
 *   - plain C types only; device pointers are raw `float*` / `int64_t*`; `ctn_stream_t` is a cudaStream_t.
 *   - every call is asynchronous on `stream`, never allocates or frees, never retains pointers.
 *   - return 0 on success, negative CTN_E* for argument / envelope errors, positive = cudaError_t.
 *   - activations inside the library use (batch, channels, pitch) fp32 with pitch = ctn_pitch(frames)
 *     (frames rounded up to 128) so every row is 512-byte aligned; tensors crossing the boundary are
 *     PyTorch-contiguous.
 *   - there is no CPU fallback.  Unsupported configurations return CTN_EUNSUPPORTED.
 */
#ifndef CTN_B200_H
#define CTN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* ctn_stream_t; /* cudaStream_t */

#define CTN_VERSION 100 /* 0.1.0 */

enum ctn_status {
  CTN_OK = 0,
  CTN_EINVAL = -1,       /* bad shape / null pointer              -> Python ValueError        */
  CTN_EUNSUPPORTED = -2, /* outside the kernel envelope           -> Python NotImplementedError */
  CTN_EALIGN = -3,       /* pointer / pitch alignment             -> Python ValueError        */
  CTN_EWORKSPACE = -4,   /* workspace too small                   -> Python RuntimeError      */
  CTN_ENOTBUILT = -5     /* kernel family not compiled into lib   -> Python RuntimeError      */
};

/* numeric mode of the dense 1x1 contractions */
enum ctn_math {
  CTN_MATH_FP32 = 0,   /* CUDA-core FFMA, exact fp32 products (verification mode)          */
  CTN_MATH_TF32X3 = 1, /* wgmma tf32, 3-pass hi/lo split, fp32 accumulate (default)      */
  CTN_MATH_TF32 = 2,   /* wgmma tf32 single pass (fast mode, looser tolerance)           */
  CTN_MATH_F16X3 = 3   /* wgmma f16, 3-pass fp16 hi/lo split (11-bit pieces like TF32, twice the MMA rate), fp32
                          accumulate; default of the Python classes.  Weight rows are rescaled by powers of two inside the
                          library (any magnitude is fine); activations must stay below 65504 in magnitude (conversion
                          saturates beyond) -- always true behind the normalisations of this network; the separator head
                          (un-normalised encoder output) and all gradient contractions use the TF32 pieces regardless */
};

/* Constructor arguments of ConvTasNet / Separator (src/models/conv_tasnet.py:57-66, 322-328). */
typedef struct ctn_config {
  int32_t n_basis;      /* N  */
  int32_t kernel_size;  /* L  */
  int32_t stride;       /* L/2 by default */
  int32_t bottleneck;   /* B  (sep_bottleneck_channels) */
  int32_t hidden;       /* H  (sep_hidden_channels)     */
  int32_t skip;         /* Sc (sep_skip_channels)       */
  int32_t sep_kernel;   /* P  (sep_kernel_size)         */
  int32_t num_blocks;   /* R  */
  int32_t num_layers;   /* X  */
  int32_t n_sources;    /* S  */
  int32_t causal;       /* 0: gLN (supported), 1: cLN (CTN_EUNSUPPORTED in the fused path) */
  int32_t enc_relu;     /* enc_nonlinear == 'relu' */
  int32_t mask_softmax; /* mask_nonlinear == 'softmax'; trains through ctn_softmax_* (the other training entries: CTN_EUNSUPPORTED) */
  int32_t math;         /* enum ctn_math */
  float eps;            /* Separator head norm eps (ConvTasNet eps)            */
  float eps_tcn;        /* eps of the norms inside the TDCN (reference passes the default 1e-12) */
  int32_t in_channels;  /* C = n_mics of the 4-D input form (conv_tasnet.py:75,138-141); 0 or 1: monaural.  > 1: trains through ctn_multichannel_* */
} ctn_config_t;

/* Parameters of one ResidualBlock1d (+ its DepthwiseSeparableConv1d), src/models/tdcn.py:77-196.
 * state_dict names (prefix separator.tdcn.net.{r}.net.{x}.) are given per field. */
typedef struct ctn_block_params {
  const float* bottleneck_w; /* bottleneck_conv1d.weight (H,B,1)                       */
  const float* bottleneck_b; /* bottleneck_conv1d.bias   (H)                           */
  const float* prelu1;       /* nonlinear1d.weight (1)                                 */
  const float* norm1_g;      /* norm1d.norm.weight (H)                                 */
  const float* norm1_b;      /* norm1d.norm.bias   (H)                                 */
  const float* dw_w;         /* separable_conv1d.depthwise_conv1d.weight (H,1,P)       */
  const float* dw_b;         /* separable_conv1d.depthwise_conv1d.bias   (H)           */
  const float* prelu2;       /* separable_conv1d.nonlinear1d.weight (1)                */
  const float* norm2_g;      /* separable_conv1d.norm1d.norm.weight (H)                */
  const float* norm2_b;      /* separable_conv1d.norm1d.norm.bias   (H)                */
  const float* out_w;        /* separable_conv1d.output_pointwise_conv1d.weight (B,H,1) or NULL (last block) */
  const float* out_b;        /* ...bias (B) or NULL                                    */
  const float* skip_w;       /* separable_conv1d.skip_pointwise_conv1d.weight (Sc,H,1) */
  const float* skip_b;       /* ...bias (Sc)                                           */
} ctn_block_params_t;

typedef struct ctn_params {
  const float* enc_w;      /* encoder.conv1d.weight (N,1,L)                  */
  const float* norm0_g;    /* separator.norm1d.norm.weight (N)               */
  const float* norm0_b;    /* separator.norm1d.norm.bias   (N)               */
  const float* bn_w;       /* separator.bottleneck_conv1d.weight (B,N,1)     */
  const float* bn_b;       /* separator.bottleneck_conv1d.bias   (B)         */
  const ctn_block_params_t* blocks; /* HOST array of R*X entries (device pointers inside) */
  const float* prelu_out;  /* separator.prelu.weight (1)                      */
  const float* mask_w;     /* separator.mask_conv1d.weight (S*N,Sc,1)        */
  const float* mask_b;     /* separator.mask_conv1d.bias   (S*N)             */
  const float* dec_w;      /* decoder.conv_transpose1d.weight (N,1,L)        */
} ctn_params_t;

/* ---- introspection ------------------------------------------------------------------------- */
int ctn_version(void);
const char* ctn_strerror(int status);
/* 1 if the tensor-core (wgmma, sm_90a) kernel family is compiled in */
int ctn_has_tcgen05(void);

/* ---- geometry helpers (host only) ----------------------------------------------------------
 * ConvTasNet.extract_latent padding rule, src/models/conv_tasnet.py:145-149. */
int ctn_frames(int T, int kernel_size, int stride, int* pad_left, int* pad_right); /* returns T' or <0 */
int ctn_pitch(int frames);                                                         /* frames rounded up to 128 */
/* bytes of device workspace ctn_convtasnet_fwd needs for (batch, T) */
int ctn_workspace_bytes(const ctn_config_t* cfg, int batch, int T, size_t* bytes);

/* ---- module-level entry points -------------------------------------------------------------- */

/* Encoder.forward, src/models/filterbank.py:222-229 (Conv1d(1,N,L,stride,bias=False) [+ReLU]).
 * x (B,1,T) contiguous; virtual zero padding pad_left/pad_right; w (B,N,w_pitch) with frames valid columns,
 * columns [frames,w_pitch) are written as zero.  stats (nullable): double[B][2] += (sum, sumsq) over valid. */
int ctn_encoder_fwd(const float* x, const float* enc_w, float* w, int B, int T, int pad_left, int pad_right,
                    int N, int L, int stride, int relu, int w_pitch, double* stats, ctn_stream_t stream);

/* Decoder.forward, src/models/filterbank.py:245-247 (ConvTranspose1d(N,1,L,stride,bias=False)), fused with the
 * crop of conv_tasnet.py:169: y[bs][t] = full[bs][t + crop_left], t in [0,T_out).  w_hat (BS,N,in_pitch). */
int ctn_decoder_fwd(const float* w_hat, const float* dec_w, float* y, int BS, int N, int frames, int in_pitch,
                    int L, int stride, int crop_left, int T_out, ctn_stream_t stream);
/* Multichannel filter banks, src/models/filterbank.py:212,241 with in_channels = C > 1 (the 4-D input of conv_tasnet.py:138-141):
 * x (B,C,T), enc_w (N,C,L) -> w (B,N,w_pitch) [+ gLN statistics]; w_hat (BS,N,in_pitch), dec_w (N,C,L) -> y (BS,C,T_out), cropped. */
int ctn_encoder_mc_fwd(const float* x, const float* enc_w, float* w, int B, int C, int T, int pad_left, int pad_right, int N, int L,
                       int stride, int relu, int w_pitch, double* stats, ctn_stream_t stream);
int ctn_decoder_mc_fwd(const float* w_hat, const float* dec_w, float* y, int BS, int C, int N, int frames, int in_pitch, int L,
                       int stride, int crop_left, int T_out, ctn_stream_t stream);

/* GlobalLayerNorm.forward, src/modules/norm.py:18,32 (GroupNorm(1,C,eps)).  x,y (B,C,T) contiguous.
 * scratch: double[B][2], zero-initialised by the callee. */
int ctn_gln_fwd(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int T, float eps,
                double* scratch, ctn_stream_t stream);

/* CumulativeLayerNorm1d.forward, src/modules/norm.py:78-90.  x,y (B,C,T) contiguous; scratch double[B][T][2]. */
int ctn_cln_fwd(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int T, float eps,
                double* scratch, ctn_stream_t stream);
/* Backward of ctn_cln_fwd: dy (B,C,T) -> dx (B,C,T) (dx may alias dy); dgamma, dbeta (C) are ACCUMULATED (zero them first).
 * scratch: 160 * B * T bytes, 16-byte aligned (the forward's prefix sums are recomputed there).  Frames whose cumulative
 * variance the forward clamped to 0 take the variance as a constant (the reference's autograd yields inf / NaN there). */
int ctn_cln_bwd(const float* dy, const float* x, const float* gamma, void* scratch, float* dx, float* dgamma, float* dbeta,
                int B, int C, int T, float eps, ctn_stream_t stream);

/* TimeDilatedConvNet.forward == TemporalConvNet.forward, src/models/tdcn.py:29-41 (src/models/tcn.py:37-49).
 * x (B,bottleneck,frames) contiguous -> skip sum (B,skip,frames) contiguous.  Uses cfg fields bottleneck, hidden,
 * skip, sep_kernel, num_blocks, num_layers, causal, math, eps_tcn.  workspace sized by ctn_tcn_workspace_bytes. */
int ctn_tcn_workspace_bytes(const ctn_config_t* cfg, int batch, int frames, size_t* bytes);
int ctn_tcn_fwd(const ctn_config_t* cfg, const ctn_block_params_t* blocks, const float* x, float* skip_out, int B,
                int frames, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* ResidualBlock1d.forward (src/models/tdcn.py:107-147, n_blocks = 1) / TimeDilatedConvBlock1d.forward (tdcn.py:65-75): a run of
 * residual blocks with EXPLICIT dilations returning both heads.  x (B,bottleneck,frames) -> x_out (nullable; the residual stream
 * after the last block, which must then have the output head) and skip_out (B,skip,frames) = sum of the blocks' skip heads.
 * cfg as for ctn_tcn_fwd (num_blocks / num_layers are ignored); workspace: ctn_tcn_workspace_bytes with num_blocks = 1,
 * num_layers = n_blocks.  Non-causal (gLN) only. */
int ctn_tcn_blocks_fwd(const ctn_config_t* cfg, const ctn_block_params_t* blocks, int n_blocks, const int* dilations, const float* x,
                       float* x_out, float* skip_out, int B, int frames, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* ConvTasNet.forward / extract_latent, src/models/conv_tasnet.py:116-171.
 * x (B,1,T) -> out (B,S,T); latent (nullable) (B,S,N,frames) contiguous. */
int ctn_convtasnet_fwd(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, float* out,
                       float* latent, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* ---- online (chunk-by-chunk) inference of the causal model ---------------------------------------------------
 * B streams advance together; each push takes n new samples per stream and returns n samples per source, delayed by
 * D = kernel_size - stride samples.  With x = everything pushed since the last init / reset (T samples), Y = the
 * concatenated push outputs and Z = the flush output: Y[..., :D] == 0 and cat(Y[..., D:], Z) == ctn_convtasnet_fwd(x).
 * Envelope: causal = 1, in_channels <= 1 (else CTN_EUNSUPPORTED); sigmoid or softmax mask; every math mode.
 * `state`: one device buffer of ctn_online_state_bytes(cfg, B, max_chunk_frames) bytes, 256-byte aligned, owned by the
 * caller.  It holds the carried state (sample counter, running cLN sums, the depthwise history of every block, the
 * filter-bank carries), the weight images of every contraction (built by ctn_online_init, kept by ctn_online_reset) and
 * the scratch of one chunk.  Pushes read the counters from the state on the device, so a captured push replays.
 * ctn_online_init: builds the images from `params` and zeroes the carries.  The weights must not change afterwards.
 * ctn_online_reset: back to zero history / statistics / samples (images kept).
 * ctn_online_push: x (B,1,n) -> y (B,S,n), contiguous; n % stride == 0, 0 < n <= max_chunk_frames * stride.  A push
 * computes the frames its samples complete; its launch sequence depends on cfg alone.
 * ctn_online_flush: y_tail (B,S,D) = the last D samples of the offline output.  CTN_EINVAL when fewer than kernel_size
 * samples were pushed since the reset; reads that count from the device (synchronises the stream once).  y_tail must be
 * non-null when D > 0; a zero-delay model (kernel_size == stride) writes nothing, so y_tail may then be null. */
int ctn_online_state_bytes(const ctn_config_t* cfg, int B, int max_chunk_frames, size_t* bytes);
int ctn_online_init(const ctn_config_t* cfg, const ctn_params_t* params, int B, int max_chunk_frames, void* state, size_t state_bytes,
                    ctn_stream_t stream);
int ctn_online_reset(const ctn_config_t* cfg, void* state, int B, ctn_stream_t stream);
int ctn_online_push(const ctn_config_t* cfg, const ctn_params_t* params, void* state, const float* x, int B, int max_chunk_frames, int n,
                    float* y, ctn_stream_t stream);
int ctn_online_flush(const ctn_config_t* cfg, void* state, int B, float* y_tail, ctn_stream_t stream);

/* ---- recordings of any length through a model that sees fixed-size chunks (no counterpart in the reference) -----------
 * Plan: chunk/2 <= hop <= chunk (integer division), else CTN_EINVAL.  K = 1 chunk of T samples when T <= chunk; otherwise
 * K = ceil((T - chunk) / hop) + 1 chunks of `chunk` samples, chunk k starting at k*hop and the last one at T - chunk, so it
 * ends at T and no chunk sees padding the signal does not contain.  Chunk index g = b*K + k throughout.
 * ctn_chunk_plan (host only): returns K (or < 0); starts (nullable) receives the K chunk starts, capacity >= K.
 * ctn_chunk_gather: x (B,1,T) -> xc (n,1,Lc), Lc = min(chunk, T): chunks first .. first + n - 1; n <= 65535.
 * ctn_chunk_align: est (B*K,S,Lc) chunk estimates -> perms (B,K,S) int32: row perms[b][k][s] of chunk k carries source s.
 *   For each neighbouring pair, over the samples both chunks cover, c[i][j] = <e_k[i], e_{k+1}[j]> in double; the local
 *   permutation maximises sum_i c[i][pi(i)] (itertools.permutations order, first maximum on ties, as in ctn_sisdr_pit_fwd);
 *   perms[b][0] = identity, perms[b][k+1][s] = pi_k(perms[b][k][s]).  Two launches (scores of every pair; one scan per
 *   recording), no atomics.  S <= 6 (else CTN_EUNSUPPORTED); S > 1 needs hop < chunk (CTN_EINVAL) and, when K > 1, scratch
 *   of ctn_chunk_align_scratch_bytes() bytes, 8-byte aligned; B*(K-1) <= 65535.
 * ctn_chunk_overlap_add: out (B,S,T), out[b][s][t] = sum_k w_k(t) est[b*K+k][perms[b][k][s]][t - start_k] / sum_k w_k(t) over the
 *   chunks covering t, k ascending, accumulated in double (gather form: deterministic).  w_k = rise * fall, rise =
 *   sin^2(pi/2 (r + 1/2)/a) over the first a samples of the chunk (a = samples shared with chunk k-1), fall = cos^2(pi/2 (q + 1/2)/n)
 *   over its last n (shared with chunk k+1), 1 elsewhere.  perms nullable (identity).  Any S. */
int ctn_chunk_plan(int T, int chunk, int hop, int* starts, int capacity);
int ctn_chunk_gather(const float* x, int B, int T, int chunk, int hop, int first, int n, float* xc, ctn_stream_t stream);
size_t ctn_chunk_align_scratch_bytes(int B, int S, int T, int chunk, int hop);
int ctn_chunk_align(const float* est, int B, int S, int T, int chunk, int hop, int32_t* perms, void* scratch, size_t scratch_bytes,
                    ctn_stream_t stream);
int ctn_chunk_overlap_add(const float* est, const int32_t* perms, int B, int S, int T, int chunk, int hop, float* out,
                          ctn_stream_t stream);
/* The whole call: x (B,1,T) -> out (B,S,T).  The B*K chunks are gathered into batches of at most chunk_batch and run through
 * ctn_convtasnet_fwd (a smaller last batch runs at its own size), then aligned (align != 0 and S > 1; needs hop < chunk and
 * S <= 6) and overlap-added.  T <= chunk: ctn_convtasnet_fwd on x itself, in batches of chunk_batch recordings.  perms_out
 * (nullable) (B,K,S) int32 receives the permutations used.  Every launch goes to `stream`, nothing is read back to the host.
 * Envelope: whatever ctn_convtasnet_fwd accepts with in_channels <= 1.  Workspace (256-byte aligned), for T > chunk:
 * the forward's workspace for min(chunk_batch, B*K) chunks + one gathered batch + 4*B*K*S*chunk bytes of chunk estimates
 * + B*K*S*4 (permutations) + the alignment scratch: only the last three grow with T. */
int ctn_separate_long_workspace_bytes(const ctn_config_t* cfg, int B, int T, int chunk, int hop, int chunk_batch, size_t* bytes);
int ctn_convtasnet_separate_long(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, int chunk, int hop,
                                 int chunk_batch, int align, float* out, int32_t* perms_out, void* workspace, size_t workspace_bytes,
                                 ctn_stream_t stream);

/* ---- whole tracks through a model trained on standardised segments (the MUSDB18 recipe's tester) -----------------------------
 * Each segment and channel is standardised on its own, (x - mean) / (std + eps) with the unbiased std, run through the model,
 * mapped back with std * est + mean (the mixture's statistics for every source) and overlap-added.  x (B,C,T), C = in_channels.
 * Plan: hop = 0 is the tester's layout: Lc = segment, K = ceil(T / segment), segment k starts at k*segment, samples at or past T
 *   read as zero (and count in the statistics), segments share no samples.  segment/2 <= hop <= segment (integer division) is
 *   the cross-faded layout of ctn_chunk_plan (Lc = min(segment, T), the last chunk ends at T).  Anything else CTN_EINVAL.
 *   Chunk index g = b*K + k, row (g, c) throughout.  Lc >= 2 (an unbiased std needs two samples), 1 <= C <= 64, else CTN_EINVAL.
 * ctn_track_plan (host only): returns K (or < 0); starts (nullable) receives the K segment starts, capacity >= K.
 * ctn_track_stats: stats (B,K,C,2) double = (mean, unbiased std) of every row, in double: per row several CTAs write partial sums
 *   of x - x[start] and its square into scratch (ctn_track_stats_scratch_bytes(), 8-byte aligned), a second launch sums them
 *   in a fixed order.  No atomics: the same input gives the same bits.  2 launches.
 * ctn_track_gather: xc (n,C,Lc) = (float)((x - mean) / (std + eps)) of chunks first .. first + n - 1, computed in double and
 *   rounded once; an all-zero segment gives zeros when eps > 0.  n*C <= 65535 (else CTN_EUNSUPPORTED).
 * ctn_track_overlap_add: est (B*K,S,C,Lc) -> out (B,S,C,T), out[b][s][c][t] = sum_k w_k(t) (std_kc est_k[s][c][t - start_k] +
 *   mean_kc) / sum_k w_k(t), k ascending, in double; w_k as in ctn_chunk_overlap_add (every w_k = 1 in the tester layout, where
 *   this is concatenate-and-crop).  No permutation alignment: the stems have a fixed order.  B*C <= 65535. */
int ctn_track_plan(int T, int segment, int hop, int* starts, int capacity);
size_t ctn_track_stats_scratch_bytes(int B, int C, int T, int segment, int hop);
int ctn_track_stats(const float* x, int B, int C, int T, int segment, int hop, double* stats, void* scratch, size_t scratch_bytes,
                    ctn_stream_t stream);
int ctn_track_gather(const float* x, const double* stats, int B, int C, int T, int segment, int hop, float eps, int first, int n, float* xc,
                     ctn_stream_t stream);
int ctn_track_overlap_add(const float* est, const double* stats, int B, int S, int C, int T, int segment, int hop, float* out,
                          ctn_stream_t stream);
/* The whole call: x (B,C,T) -> out (B,S,C,T) (C = 1: (B,1,T) -> (B,S,T)).  Statistics; per batch of at most chunk_batch chunks
 * the standardising gather (eps = cfg->eps) and ctn_convtasnet_fwd (a smaller last batch runs at its own size); then the
 * overlap-add.  Every launch goes to `stream`, nothing is read back to the host (CUDA-graph capturable).  Envelope: whatever
 * ctn_convtasnet_fwd accepts (1 <= in_channels <= 64, causal or not, sigmoid or softmax mask, every math mode); B*C <= 65535.
 * Workspace (256-byte aligned): the forward's workspace for min(chunk_batch, B*K) chunks + one standardised batch
 * + 4*B*K*S*C*Lc bytes of chunk estimates + the statistics and their partials: only the last two grow with T. */
int ctn_separate_track_workspace_bytes(const ctn_config_t* cfg, int B, int T, int segment, int hop, int chunk_batch, size_t* bytes);
int ctn_convtasnet_separate_track(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, int segment, int hop,
                                  int chunk_batch, float* out, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* Separator.forward, src/models/conv_tasnet.py:359-378: w (B,N,frames) -> mask (B,S,N,frames), both contiguous. */
int ctn_separator_fwd(const ctn_config_t* cfg, const ctn_params_t* params, const float* w, int B, int frames,
                      float* mask, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* ---- DPRNN-TasNet path (BASELINE cfg4): segment / dual-path glue / overlap-add, and the separator stages around it ----
 *
 * Segment1d.forward, src/models/transform.py:15-29, fused with the zero padding of src/models/dprnn_tasnet.py:339-345:
 * x (B,F,pitch) with `frames` valid columns (pitch == frames for a contiguous tensor) -> chunks of `chunk_size` frames every
 * `hop_size` of the padded sequence, S = (frames + pad_left + pad_right - chunk_size) / hop_size + 1.
 * channels_last = 0: Z (B,F,S,chunk) -- the reference layout;  1: Z (B,S,chunk,F) -- the batch_first layout the intra-chunk
 * LSTM consumes, i.e. the permute of src/models/dprnn.py:83-84 folded in. */
int ctn_segment_fwd(const float* x, float* Z, int B, int F, int frames, int pitch, int chunk_size, int hop_size, int pad_left,
                    int pad_right, int channels_last, ctn_stream_t stream);
/* OverlapAdd1d.forward, src/models/transform.py:46-62, fused with the crop of dprnn_tasnet.py:347: y (B,F,out_pitch),
 * y[..][t] = sum of the chunks covering padded frame t + crop_left, t < T_out; columns [T_out,out_pitch) = 0.
 * Z laid out as above (channels_last). */
int ctn_overlap_add_fwd(const float* Z, float* y, int B, int F, int S, int chunk_size, int hop_size, int crop_left, int T_out,
                        int out_pitch, int channels_last, ctn_stream_t stream);
/* Tail of IntraChunkRNN / InterChunkRNN.forward, src/models/dprnn.py:87-94 / 140-148: out = gLN(Y; gamma, beta) + R on
 * channels-last tensors (B,D1,D2,F) (gLN = GroupNorm(1,F): per-sample statistics over D1*D2*F values).  swap = 1 stores out as
 * (B,D2,D1,F) -- the layout of the other path (the permutes of dprnn.py:83, 91, 136, 144-146).  scratch: double[B][2]. */
int ctn_dprnn_norm_res_fwd(const float* Y, const float* R, const float* gamma, const float* beta, float* out, int B, int D1, int D2,
                           int F, float eps, int swap, double* scratch, ctn_stream_t stream);
/* Bidirectional LSTM + the 2H -> F Linear of a dual-path block, src/models/dprnn.py:85-87 / 138-139 (nn.LSTM(batch_first,
 * bidirectional) followed by nn.Linear), on wgmma, 3xTF32 (csrc/ctn_lstm.cu).
 * z (NSEQ,T,F) fp32, batch_first; w[8] = host array of device pointers in torch.nn.LSTM order: weight_ih_l0 (4H,F), weight_hh_l0
 * (4H,H), bias_ih_l0, bias_hh_l0 (4H), then the four *_reverse tensors; gate order i,f,g,o; zero initial state.
 * w_fc (Fo,2H) nullable.  P (2,NSEQ,T,Fo): partial projections W_fc[:, dir*H:(dir+1)*H] h_dir WITHOUT the Linear's bias -- the
 * Linear output is P[0] + P[1] + bias (ctn_dprnn_norm_res2_fwd consumes it in that form).  hout (NSEQ,T,2H) nullable: the LSTM
 * output itself (forward direction in [:H], reverse in [H:]).  Envelope: F, H in {32,64,128}, Fo in {32,64,96,128}
 * (ctn_bilstm_supported); workspace >= ctn_bilstm_workspace_bytes(F,H,Fo), 256-byte aligned.  z_absmax (nullable): device word holding
 * the bit pattern of max|z| (the fp16 operand scale of x is derived from it); null = measured here with one more pass over z. */
int ctn_bilstm_supported(int F, int H, int Fo);
size_t ctn_bilstm_workspace_bytes(int F, int H, int Fo);
int ctn_bilstm_proj_fwd(const float* z, int NSEQ, int T, int F, int H, const float* const* w, const float* w_fc, int Fo, float* P,
                        float* hout, const unsigned* z_absmax, void* workspace, size_t workspace_bytes, ctn_stream_t stream);
/* ctn_dprnn_norm_res_fwd with Y = P[0] + P[1] + fc_bias, P (2,B,D1,D2,F) as ctn_bilstm_proj_fwd leaves it (F % 4 == 0).
 * out_absmax (nullable): receives the bit pattern of max|out| -- the z_absmax of the next ctn_bilstm_proj_fwd. */
int ctn_dprnn_norm_res2_fwd(const float* P, const float* fc_bias, const float* R, const float* gamma, const float* beta, float* out,
                            int B, int D1, int D2, int F, float eps, int swap, double* scratch, unsigned* out_absmax, ctn_stream_t stream);
/* ---- DPTNet path: the dual-path transformer (src/models/dptnet.py) ----
 *
 * ctn_bilstm_proj_fwd with w_fc required and ReLU applied to the projection's operand only: P = W_fc ReLU(h) per direction (the
 * ReLU between the LSTM and the Linear of FeedForwardBlock, dptnet.py:560-562); the recurrence and hout use the raw h. */
int ctn_bilstm_relu_proj_fwd(const float* z, int NSEQ, int T, int F, int H, const float* const* w, const float* w_fc, int Fo, float* P,
                             float* hout, void* workspace, size_t workspace_bytes, ctn_stream_t stream);
/* nn.MultiheadAttention(F, heads)(z, z, z) without mask (dptnet.py:512), on channels-last sequences: z (NSEQ,T,F) -> y (NSEQ,T,F) =
 * out_proj(attention) + out_b, no residual.  in_w (3F,F), in_b (3F), out_w (F,F), out_b (F); scale 1/sqrt(F/heads).  fp32 FMAs, keys
 * streamed through an online softmax: any T up to 65535 tiles of 64.  Envelope (ctn_mha_supported): F <= 128, F % 4 == 0,
 * F/heads in {8,16,32,64}; any NSEQ (the sequences are the grid's x).  workspace >= ctn_mha_workspace_bytes(NSEQ,T,F), 256-byte aligned.  3 launches. */
int ctn_mha_supported(int F, int heads);
size_t ctn_mha_workspace_bytes(int NSEQ, int T, int F);
int ctn_mha_fwd(const float* z, int NSEQ, int T, int F, int heads, const float* in_w, const float* in_b, const float* out_w,
                const float* out_b, float* y, void* workspace, size_t workspace_bytes, ctn_stream_t stream);
/* The norm of MultiheadAttentionBlock / FeedForwardBlock (dptnet.py:513-521 / 563-568): x = Y0 + Y1 + bias[f] + R (Y1, bias, R
 * nullable; all (B,D1,D2,F) channels-last), out = GroupNorm(1,F) of each SEQUENCE, i.e. each (b, d1) row of D2*F values, with
 * gamma, beta (F).  swap = 1 stores out as (B,D2,D1,F) and then must not alias an input.  The statistics are summed in double in a
 * fixed order: repeated calls give the same bits.  1 launch. */
int ctn_seq_norm_fwd(const float* Y0, const float* Y1, const float* bias, const float* R, const float* gamma, const float* beta,
                     float* out, int B, int D1, int D2, int F, float eps, int swap, ctn_stream_t stream);
/* Separator head, dptnet.py:334-337: z (B,S,chunk,Bc) = gLN(Segment1d(pad(Wb w + bb))) with the gLN per sample over the segmented
 * tensor (overlap duplicates and padding zeros included).  w (B,N,pitch) pitched, 16-byte aligned; S = (frames + pad_left +
 * pad_right - chunk) / hop + 1.  The 1x1 follows ctn_pw's numeric mode `math`.  workspace >= ctn_dpt_head_workspace_bytes(B, N, Bc,
 * pitch, S, chunk), 256-byte aligned.  Every refusal comes before the first launch. */
size_t ctn_dpt_head_workspace_bytes(int B, int N, int Bc, int pitch, int S, int chunk_size);
int ctn_dpt_head_fwd(const float* w, const float* bn_w, const float* bn_b, const float* norm_g, const float* norm_b, float* z, int B,
                     int N, int Bc, int frames, int pitch, int chunk_size, int hop_size, int pad_left, int pad_right, float eps, int math,
                     void* workspace, size_t workspace_bytes, ctn_stream_t stream);
/* Separator tail + decoder, dptnet.py:341-346 and 136-143: PReLU -> map 1x1 (Bc -> S*N) -> GTU1d per source (tanh(map) *
 * sigmoid(map_gate), N -> N, gtu.py:37-42) -> ReLU (mask_relu = 1) or sigmoid -> w * mask -> ConvTranspose1d -> crop.
 * y (B,Bc,pitch), w (B,N,pitch); out (B,S,T); latent nullable (B,S,N,frames); what (B,S*N,pitch) scratch; B*S <= 65535.
 * workspace >= ctn_dpt_tail_workspace_bytes(B,N,Bc,S,pitch), 256-byte aligned.  Every refusal comes before the first launch. */
size_t ctn_dpt_tail_workspace_bytes(int B, int N, int Bc, int S, int pitch);
int ctn_dpt_tail_fwd(const float* y, const float* w, const float* prelu, const float* map_w, const float* map_b, const float* gtu_w,
                     const float* gtu_b, const float* gate_w, const float* gate_b, const float* dec_w, float* out, float* latent, float* what,
                     int B, int N, int Bc, int S, int frames, int pitch, int L, int stride, int crop_left, int T, int mask_relu, int math,
                     void* workspace, size_t workspace_bytes, ctn_stream_t stream);
/* Separator head on the padded layout, src/models/conv_tasnet.py:370-371 == src/models/dprnn_tasnet.py:335-336:
 * x0 (B,Bc,pitch) = Wb gLN(w) + bb; w (B,N,pitch), stats0 double[B][2] = (sum, sumsq) of w (as ctn_encoder_fwd leaves them).
 * workspace >= ctn_stage_workspace_bytes(Bc, N), 256-byte aligned; w and x0 16-byte aligned.  Every refusal comes before the first launch. */
size_t ctn_stage_workspace_bytes(int M, int K);
int ctn_sep_head_fwd(const float* w, const double* stats0, const float* norm_g, const float* norm_b, const float* bn_w,
                     const float* bn_b, float* x0, int B, int N, int Bc, int frames, int pitch, float eps, int math, void* workspace,
                     size_t workspace_bytes, ctn_stream_t stream);
/* Separator tail + decoder, conv_tasnet.py:373-376,158-169 == dprnn_tasnet.py:348-350,141-153: PReLU -> mask 1x1 -> sigmoid ->
 * w*mask -> ConvTranspose1d -> crop.  y (B,Bc,pitch), w (B,N,pitch); out (B,S,T); latent nullable (B,S,N,frames);
 * what (B,S*N,pitch) scratch; workspace >= ctn_stage_workspace_bytes(S*N, Bc), 256-byte aligned; y, w and what 16-byte aligned.
 * Every refusal, the decoder's included (crop_left + T past the full length, L % stride != 0), comes before the first launch. */
int ctn_sep_tail_fwd(const float* y, const float* w, const float* prelu, const float* mask_w, const float* mask_b,
                     const float* dec_w, float* out, float* latent, float* what, int B, int N, int Bc, int S, int frames, int pitch,
                     int L, int stride, int crop_left, int T, int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* ---- SepFormer path: the dual-path transformer of src/models/sepformer.py (csrc/ctn_sepformer.cu) ----
 *
 * The dual-path state is channel-first and pitched: X (B,F,pitch), token s*C + k for chunk s < S and frame k < C, pitch >= S*C
 * (ctn_pitch(S*C) in the model); columns [S*C, pitch) are zero wherever these entries write the state.  intra = 1 selects the
 * sequences of IntraTransformer (the C tokens of one chunk), intra = 0 those of InterTransformer (the S tokens of one frame, C apart).
 * Every entry refuses before its first launch and is CUDA-graph capturable.
 *
 * Segment1d / OverlapAdd1d on that layout (sepformer.py:348-352): Z (B,F,z_pitch), Z[b][f][s*C + k] = the zero-padded x at frame
 * s*hop + k - pad_left, columns [S*C, z_pitch) = 0; the overlap-add sums the chunks covering frame t + crop_left in ascending s into
 * y (B,F,out_pitch), columns [T_out, out_pitch) = 0.  1 launch each. */
int ctn_sfm_segment_fwd(const float* x, float* Z, int B, int F, int frames, int pitch, int chunk_size, int hop_size, int pad_left,
                        int pad_right, int z_pitch, ctn_stream_t stream);
int ctn_sfm_overlap_add_fwd(const float* Z, float* y, int B, int F, int S, int chunk_size, int hop_size, int z_pitch, int crop_left,
                            int T_out, int out_pitch, ctn_stream_t stream);
/* Scaled dot-product attention of nn.MultiheadAttention(F, heads) over every sequence of the path: qkv (B,3F,pitch) = the
 * in-projection WITHOUT its bias (as ctn_pw leaves it, channel-first), in_b (3F) added on load; O (B,F,pitch) receives the
 * concatenated heads before out_proj; its columns outside the sequences are not written.  Scale 1/sqrt(F/heads), online softmax
 * over 64-key tiles (any length), fp32 FMAs.  Envelope (ctn_sfm_attn_supported): F/heads in {8,16,32,64}.  1 launch. */
int ctn_sfm_attn_supported(int F, int heads);
int ctn_sfm_attn_fwd(const float* qkv, const float* in_b, float* O, int B, int F, int heads, int S, int C, int pitch, int intra,
                     ctn_stream_t stream);
/* The post-norm LayerNorm of nn.TransformerEncoderLayer: out = LayerNorm_F(X + (Y + bias); gamma, beta, eps) per token (column) of
 * (B,F,pitch) tensors, statistics in double (mean, then the centred variance).  Y, bias nullable; out may alias X (not Y).  Columns
 * [ntok, pitch) of out = 0.  1 launch. */
int ctn_sfm_token_ln_fwd(const float* X, const float* Y, const float* bias, const float* gamma, const float* beta, float* out, int B,
                         int F, int ntok, int pitch, float eps, ctn_stream_t stream);
/* The end of IntraTransformer / InterTransformer (sepformer.py:473-476 / 515-518): out = GroupNorm(1,F) of each SEQUENCE of X (its F x
 * len values; gamma, beta per feature) + R, R the block input without the positional encoding.  Summed in double in a fixed order,
 * no atomics: repeated calls give the same bits.  out may alias R, not X.  1 launch. */
int ctn_sfm_seq_norm_res_fwd(const float* X, const float* R, const float* gamma, const float* beta, float* out, int B, int F, int S,
                             int C, int pitch, int intra, float eps, ctn_stream_t stream);
/* The encoder input of sepformer.py:471-472: out = X + (X + pe[p]) with p the token's position in its sequence (PositionalEncoding
 * returns input + encoding and the caller adds the input again).  pe = the module's (5000,1,F) buffer, read as it is.  1 launch. */
int ctn_sfm_pos_enc_fwd(const float* X, const float* pe, float* out, int B, int F, int S, int C, int pitch, int intra, ctn_stream_t stream);
/* One IntraTransformer (intra = 1) or InterTransformer (intra = 0): positional encoding, `layers` post-norm ReLU encoder layers
 * (heads, d_ff, LayerNorm eps) and the final per-sequence gLN + residual.  X, out (B,F,pitch), distinct, X 16-byte aligned.
 * w: host array of 12*layers + 3 device pointers: per layer in_proj_weight (3F,F), in_proj_bias, out_proj.weight (F,F),
 * out_proj.bias, linear1.weight (d_ff,F), linear1.bias, linear2.weight (F,d_ff), linear2.bias, norm1.weight, norm1.bias,
 * norm2.weight, norm2.bias; then the positional-encoding buffer and the final gLN's weight and bias.  The four contractions of a
 * layer run through ctn_pw in the numeric mode `math`; every weight image of the call is built in one batch first.  Sequences
 * longer than 5000 tokens: CTN_EINVAL.  workspace >= ctn_sfm_transformer_workspace_bytes(), 256-byte aligned.
 * Launches: 7*layers + 2, plus, outside the fp32 mode, ceil(4*n / 48) weight-image launches for each batch of n <= 64 layers. */
size_t ctn_sfm_transformer_workspace_bytes(int B, int F, int d_ff, int layers, int pitch, int math);
int ctn_sfm_transformer_fwd(const float* X, float* out, const float* const* w, int B, int F, int heads, int d_ff, int layers, int S, int C,
                            int pitch, int intra, float eps, int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream);
/* Separator tail + decoder, sepformer.py:353-359 and 142-155: PReLU -> map 1x1 (Bc -> S*N) -> GTU1d per source -> bottleneck_conv1d_out
 * (N -> N, bias) -> ReLU (mask_relu = 1) or sigmoid -> w * mask -> ConvTranspose1d -> crop.  y (B,Bc,pitch), w (B,N,pitch);
 * out (B,S,T); latent nullable (B,S,N,frames); what (B,S*N,pitch) scratch; B*S <= 65535.  The three weight images are built in one
 * batch.  workspace >= ctn_sfm_tail_workspace_bytes(B,N,Bc,S,pitch), 256-byte aligned.  Launches: 6 + the decoder's (+ 1 weight-image
 * launch outside the fp32 mode, + 1 with latent). */
size_t ctn_sfm_tail_workspace_bytes(int B, int N, int Bc, int S, int pitch);
int ctn_sfm_tail_fwd(const float* y, const float* w, const float* prelu, const float* map_w, const float* map_b, const float* gtu_w,
                     const float* gtu_b, const float* gate_w, const float* gate_b, const float* bout_w, const float* bout_b,
                     const float* dec_w, float* out, float* latent, float* what, int B, int N, int Bc, int S, int frames, int pitch, int L,
                     int stride, int crop_left, int T, int mask_relu, int math, void* workspace, size_t workspace_bytes,
                     ctn_stream_t stream);

/* ---- LSTM-TasNet path (src/models/tasnet.py, csrc/ctn_tasnet.cu) ----
 *
 * GatedEncoder (filterbank.py:325-346) + the Separator's frame norm (tasnet.py:356-359): x (B,1,T) -> w (B,N,pitch) =
 * ReLU(U x~) * sigmoid(V x~) with x~ = x / (||x||_2 + enc_eps), the norm over the whole padded signal of each sample (nrm: double[B]
 * scratch), and xn (B,N,pitch) = gamma (w - mean) / (sqrt(var) + eps) + beta over the N channels of each frame, mean and centred
 * variance in double (an all-zero frame gives exactly beta).  u_w, v_w (N,1,L); virtual zero padding pad_left / pad_right, frames =
 * (T + pad_left + pad_right - L) / stride + 1 (a ragged tail makes no frame but counts in the norm); columns [frames, pitch) of w and xn are 0.  2 launches.
 * ctn_tas_frame_norm_fwd: the frame norm alone, w (B,N,pitch) -> xn (as ctn_encoder_fwd leaves w for the plain Encoder).  1 launch. */
int ctn_tas_enc_gated_fwd(const float* x, const float* u_w, const float* v_w, const float* gamma, const float* beta, float* w, float* xn,
                          double* nrm, int B, int T, int pad_left, int pad_right, int N, int L, int stride, int pitch, float enc_eps,
                          float eps, ctn_stream_t stream);
int ctn_tas_frame_norm_fwd(const float* w, const float* gamma, const float* beta, float* xn, int B, int N, int frames, int pitch,
                           float eps, ctn_stream_t stream);
/* One nn.LSTM layer (batch_first, bidirectional when dirs = 2) on the channel-first layout: x (B,F,pitch) -> out (B,dirs*H,pitch),
 * forward direction in rows [0,H), reverse in [H,2H) (torch's concat order), zero initial state, gate order i,f,g,o.
 * w[4*dirs] = host array of device pointers in torch order: weight_ih_l{k} (4H,F), weight_hh_l{k} (4H,H), bias_ih_l{k}, bias_hh_l{k}
 * (4H), then the *_reverse tensors.  skip_in / skip_out (both or neither, (B,dirs*H,pitch)): skip_out = out + skip_in, in place
 * allowed.  The input projections of both directions are one ctn_pw contraction in the numeric mode `math`; the recurrence is one
 * cooperative launch whose CTAs keep their rows of W_hh resident in shared memory (fp32 FMAs, expf / tanhf gates, fixed summation
 * order: repeated calls give the same bits).  Envelope (ctn_tas_lstm_supported): any F, 1 <= H <= ctn_tas_lstm_max_hidden(dirs)
 * (from the current device's SM count and shared memory), any B (ctn_tas_lstm_group(H, dirs) sequences per pass), any frames.
 * workspace >= ctn_tas_lstm_workspace_bytes(), 256-byte aligned.  Every refusal comes before the first launch; a refused
 * cooperative launch returns its error.  Launches: 3 (+ 1 weight-image launch outside the fp32 mode). */
int ctn_tas_lstm_max_hidden(int dirs);
int ctn_tas_lstm_supported(int F, int H, int dirs);
int ctn_tas_lstm_group(int H, int dirs);
size_t ctn_tas_lstm_workspace_bytes(int B, int F, int H, int dirs, int pitch, int math);
int ctn_tas_lstm_fwd(const float* x, const float* const* w, float* out, const float* skip_in, float* skip_out, int B, int F, int H, int dirs,
                     int frames, int pitch, int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream);
/* Separator tail + decoder, tasnet.py:365-381 and 177-184: fc (Hd -> S*N, bias; row s*N + n) -> sigmoid (softmax = 0) or softmax
 * over the S sources of each (n, t) (softmax = 1) -> w * mask -> ConvTranspose1d -> crop.  skip (B,Hd,pitch), w (B,N,pitch);
 * out (B,S,T); latent nullable (B,S,N,frames); what (B,S*N,pitch) scratch; B*S <= 65535.  workspace >=
 * ctn_tas_tail_workspace_bytes(N,Hd,S,math), 256-byte aligned.  Launches: 1 (+1 softmax, +1 weight image outside the fp32 mode,
 * +1 with latent) + the decoder's. */
size_t ctn_tas_tail_workspace_bytes(int N, int Hd, int S, int math);
int ctn_tas_tail_fwd(const float* skip, const float* w, const float* fc_w, const float* fc_b, const float* dec_w, float* out, float* latent,
                     float* what, int B, int N, int Hd, int S, int frames, int pitch, int L, int stride, int crop_left, int T, int softmax,
                     int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* ---- GALRNet path (src/models/galrnet.py, src/models/galr.py, csrc/ctn_galr.cu) ----
 *
 * The dual-path state is channels-last, (B,S,K,F); the intra-chunk block is ctn_bilstm_proj_fwd + ctn_dprnn_norm_res2_fwd with
 * swap = 0, and the tail is ctn_dpt_tail_fwd with Bc = N.
 *
 * Separator head, galrnet.py:233-239: z (B,S,chunk,F) = gLN(Segment1d(pad(w))) with the gLN per sample over the segmented tensor
 * (overlap duplicates and padding zeros included), no bottleneck.  w (B,F,pitch) with `frames` valid columns; S = (frames +
 * pad_left + pad_right - chunk) / hop + 1.  workspace >= ctn_galr_head_workspace_bytes(B,S,chunk,F), 256-byte aligned.  Every
 * refusal comes before the first launch.  3 launches. */
size_t ctn_galr_head_workspace_bytes(int B, int S, int chunk_size, int F);
int ctn_galr_head_fwd(const float* w, const float* norm_g, const float* norm_b, float* z, int B, int F, int frames, int pitch, int chunk_size,
                      int hop_size, int pad_left, int pad_right, float eps, void* workspace, size_t workspace_bytes, ctn_stream_t stream);
/* LowDimensionGloballyAttentiveBlock.forward, galr.py:161-197, on x (B,S,K,F) channels-last -> out (B,S,K,F); out may alias x.
 * zt = LN_F(fc_map(x) along K) + pe, then y = MultiheadAttention(zt) over the S chunks of each of the B*Q down-sampled frames,
 * out = fc_inv(gLN(y + zt)) along Q + x with the gLN per sample over (Q,S,F).  map_w (Q,K), map_b (Q); ln_g, ln_b (F) of
 * norm2d_in (eps ln_eps); in_w, in_b, out_w, out_b as ctn_mha_fwd; gn_g, gn_b (F) of norm2d_out (eps gn_eps); inv_w (K,Q),
 * inv_b (K).  pe_div (F/2): the divisors 10000^(j/F) of the positional encoding, formed as the reference forms them (fp32); the
 * encoding of position p = s*Q + q is sin(p / pe_div[f]) for f < F/2 and cos(p / pe_div[f - F/2]) above.  LayerNorm and gLN
 * statistics are summed in double in a fixed order: repeated calls give the same bits.  Envelope (ctn_galr_supported): F in
 * {32,64,128}, 1 <= Q <= K, F/heads in ctn_mha_supported's; B, S <= 65535, S*Q <= 2^24.  workspace >=
 * ctn_galr_inter_workspace_bytes(B,S,K,Q,F), 256-byte aligned.  Every refusal comes before the first launch.  6 launches. */
int ctn_galr_supported(int F, int K, int Q, int heads);
size_t ctn_galr_inter_workspace_bytes(int B, int S, int K, int Q, int F);
int ctn_galr_inter_fwd(const float* x, const float* map_w, const float* map_b, const float* ln_g, const float* ln_b, const float* pe_div,
                       int heads, const float* in_w, const float* in_b, const float* out_w, const float* out_b, const float* gn_g,
                       const float* gn_b, const float* inv_w, const float* inv_b, float* out, int B, int S, int K, int Q, int F, float ln_eps,
                       float gn_eps, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* modules.conv.DepthwiseSeparableConv1d.forward, src/modules/conv.py:24-28 (not on Conv-TasNet's path; API completeness).
 * Depthwise stage: x (B,C,T) contiguous, w (C,1,K), bias nullable -> y (B,C,y_pitch) with T_out = (T + 2 padding - dilation (K-1) - 1)
 * / stride + 1 valid columns, the rest zero.  Pointwise stage: x (B,K,pitch) padded layout with `frames` valid columns, W (M,K,1),
 * bias nullable -> y (B,M,frames) contiguous, x 16-byte aligned; workspace >= 4*B*M*pitch + ctn_stage_workspace_bytes(M,K) + 16*B + 4096
 * bytes, 256-byte aligned.  Both stages refuse before any launch. */
int ctn_depthwise_conv1d_fwd(const float* x, const float* w, const float* bias, float* y, int B, int C, int T, int K, int stride, int padding,
                             int dilation, int y_pitch, ctn_stream_t stream);
int ctn_pointwise_conv1d_fwd(const float* x, const float* W, const float* bias, float* y, int B, int M, int K, int frames, int pitch,
                             int math, void* workspace, size_t workspace_bytes, ctn_stream_t stream);

/* sisdr, src/criterion/sdr.py:122-139: est,tgt (rows,T) contiguous -> out (rows). scratch double[rows][4].  Any row count and
 * any 4-byte-aligned base: 128-bit loads are used only where T % 4 == 0 and both bases are 16-byte aligned. */
int ctn_sisdr_fwd(const float* est, const float* tgt, int rows, int T, float eps, float* out, double* scratch,
                  ctn_stream_t stream);
/* sdr(), src/criterion/sdr.py:6-20: out[r] = 10 log10((|tgt_r|^2 + eps) / (|tgt_r - est_r|^2 + eps)); est, tgt (rows,T) contiguous;
 * any row count; scratch: double[rows][2]. */
int ctn_sdr_fwd(const float* est, const float* tgt, int rows, int T, float eps, float* out, double* scratch, ctn_stream_t stream);

/* PIT1d(NegSISDR(reduction='mean')), src/criterion/pit.py:9-44,71-77 + src/criterion/sdr.py:198-227.
 * est,tgt (B,S,T) contiguous.  loss_b (B) = min over permutations of -mean_i SI-SDR(est_i, tgt_perm[i]);
 * perm (B,S) int64, estimate i <-> target perm[i] (first minimum on ties, lexicographic permutation order);
 * loss_mean (1) = mean over the batch.  pair_sisdr (nullable) (B,S,S) = SI-SDR(est_i, tgt_j).
 * scratch: double[B][S*S*2 + S], zero-initialised by the callee.  S <= 6, any B.  est/tgt need no alignment beyond float's:
 * 128-bit loads are used only for samples whose rows are all 16-byte aligned (T % 4 == 0 and aligned sample bases). */
int ctn_sisdr_pit_fwd(const float* est, const float* tgt, int B, int S, int T, float eps, float* loss_b,
                      int64_t* perm, float* loss_mean, float* pair_sisdr, double* scratch, ctn_stream_t stream);
size_t ctn_sisdr_pit_scratch_bytes(int B, int S);

/* End-to-end call with HOST buffers (the "e2e" leg): copies x_host (B,1,T) and tgt_host (B,S,T) (pinned or
 * pageable) to the device staging areas, runs ctn_convtasnet_fwd + ctn_sisdr_pit_fwd, copies back out_host
 * (nullable, (B,S,T)), loss_mean_host (1), perm_host (B,S).  All on `stream`; the caller synchronises.
 * dev_io: device staging of dev_io_bytes >= ctn_host_io_bytes() (checked); loss_eps: eps of the SI-SDR (sdr.py:122, 1e-12). */
size_t ctn_host_io_bytes(const ctn_config_t* cfg, int B, int T);
int ctn_convtasnet_loss_host(const ctn_config_t* cfg, const ctn_params_t* params, const float* x_host,
                             const float* tgt_host, int B, int T, float* out_host, float* loss_mean_host,
                             int64_t* perm_host, void* dev_io, size_t dev_io_bytes, void* workspace,
                             size_t workspace_bytes, float loss_eps, ctn_stream_t stream);

/* ---- training path: what `loss.backward()` does in the reference trainer (egs/wsj0-mix/common/src/driver.py:146-150) ----
 * ctn_convtasnet_fwd_train == ctn_convtasnet_fwd (same estimate) but keeps, inside `train_ws`, what the backward needs:
 * encoder output, mask, every residual block's input and the two pre-activations (W1 x + b1, dwconv(..) + bd) and the gLN
 * statistics.  ctn_convtasnet_bwd then turns d_out (B,S,T), the gradient of the estimate, into the gradients of all
 * parameters.  `grads` has the layout of ctn_params_t (same shapes as the parameters); every gradient tensor must be
 * ZERO on entry (kernels accumulate with atomics) and is complete on return.  The gradient w.r.t. the mixture is not
 * produced (the reference trainer never asks for it).  train_ws: ctn_train_workspace_bytes(), 256-byte aligned, must
 * be left untouched between the two calls.  Envelope: non-causal gLN, sigmoid mask, sep_kernel <= 8. */
typedef ctn_params_t ctn_grads_t;
int ctn_train_workspace_bytes(const ctn_config_t* cfg, int batch, int T, size_t* bytes);
int ctn_convtasnet_fwd_train(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, float* out,
                             void* train_ws, size_t train_ws_bytes, ctn_stream_t stream);
int ctn_convtasnet_bwd(const ctn_config_t* cfg, const ctn_params_t* params, const ctn_grads_t* grads, const float* x,
                       const float* d_out, int B, int T, void* train_ws, size_t train_ws_bytes, ctn_stream_t stream);
/* The same three calls for causal (cLN) models, with the same arguments and the same contract: the estimate of
 * ctn_convtasnet_fwd on a causal config, and what the backward needs kept in train_ws (per block as above, with the cumulative
 * prefix sums of every cLN in double in place of the gLN statistics).  Envelope: causal = 1, sigmoid mask, in_channels = 1,
 * sep_kernel <= 8; anything else CTN_EUNSUPPORTED (non-causal configs train through the three calls above). */
int ctn_causal_train_workspace_bytes(const ctn_config_t* cfg, int batch, int T, size_t* bytes);
int ctn_causal_fwd_train(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, float* out,
                         void* train_ws, size_t train_ws_bytes, ctn_stream_t stream);
int ctn_causal_bwd(const ctn_config_t* cfg, const ctn_params_t* params, const ctn_grads_t* grads, const float* x,
                   const float* d_out, int B, int T, void* train_ws, size_t train_ws_bytes, ctn_stream_t stream);
/* The same three calls for multichannel models (in_channels = C, the 4-D input form of conv_tasnet.py:138-141,167-168; the
 * MUSDB18 recipes): x (B,C,T), out and d_out (B,S,C,T); enc_w and dec_w (N,C,L).  One pipeline with ctn_convtasnet_fwd_train /
 * ctn_convtasnet_bwd: the same separator, the same launch count and the same workspace; the filter banks, the decoder's adjoint
 * and the two filter-bank weight gradients run over C channels.  Envelope: causal = 0, sigmoid mask, 2 <= in_channels <= 64,
 * sep_kernel <= 8; an invalid field is CTN_EINVAL, causal, softmax or in_channels <= 1 CTN_EUNSUPPORTED. */
int ctn_multichannel_train_workspace_bytes(const ctn_config_t* cfg, int batch, int T, size_t* bytes);
int ctn_multichannel_fwd_train(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, float* out,
                               void* train_ws, size_t train_ws_bytes, ctn_stream_t stream);
int ctn_multichannel_bwd(const ctn_config_t* cfg, const ctn_params_t* params, const ctn_grads_t* grads, const float* x,
                         const float* d_out, int B, int T, void* train_ws, size_t train_ws_bytes, ctn_stream_t stream);
/* The same three calls for softmax-mask models (mask_nonlinear='softmax': nn.Softmax(dim=1) over ALL S*N mask channels of a frame,
 * conv_tasnet.py:345-357; the ORPIT and Sinkhorn PIT recipes).  The forward is ctn_convtasnet_fwd's estimate (mask logits, then one
 * softmax pass that keeps the mask in train_ws): one launch more than the sigmoid step.  The workspace equals
 * ctn_train_workspace_bytes of the same config with mask_softmax = 0.  ctn_softmax_bwd takes one more argument, d_x (B,1,T),
 * nullable: when given it is OVERWRITTEN with the gradient w.r.t. the mixture (the encoder's adjoint, one more launch), which a
 * recursive fine-tune step needs when the mixture is an earlier estimate; null skips it.  Envelope: mask_softmax = 1, causal = 0,
 * in_channels <= 1, sep_kernel <= 8; an invalid field is CTN_EINVAL, mask_softmax = 0, causal or in_channels > 1 CTN_EUNSUPPORTED;
 * a null pointer other than d_x is CTN_EINVAL before any CUDA call. */
int ctn_softmax_train_workspace_bytes(const ctn_config_t* cfg, int batch, int T, size_t* bytes);
int ctn_softmax_fwd_train(const ctn_config_t* cfg, const ctn_params_t* params, const float* x, int B, int T, float* out,
                          void* train_ws, size_t train_ws_bytes, ctn_stream_t stream);
int ctn_softmax_bwd(const ctn_config_t* cfg, const ctn_params_t* params, const ctn_grads_t* grads, const float* x,
                    const float* d_out, float* d_x, int B, int T, void* train_ws, size_t train_ws_bytes, ctn_stream_t stream);

/* Backward of ctn_sisdr_pit_fwd through the selected permutation (src/criterion/pit.py:36-44; sdr.py:135-137):
 * d_est (B,S,T) = grad_loss_b[b] * coef * dSI-SDR(est_i, tgt_perm[i])/d est_i.  fwd_scratch = the scratch buffer the
 * forward call filled (pair statistics), perm = its permutation output.  grad_loss_b (B) nullable (= 1);
 * coef = -1/S for NegSISDR(reduction='mean'), -1 for 'sum'. */
int ctn_sisdr_pit_bwd(const float* est, const float* tgt, const int64_t* perm, int B, int S, int T, float eps,
                      const double* fwd_scratch, const float* grad_loss_b, float coef, float* d_est, ctn_stream_t stream);

/* Backward of ctn_sdr_fwd (src/criterion/sdr.py:6-20): d_est (rows,T) = coef * grad_out[r] * 20 / (ln 10 (|tgt_r - est_r|^2 + eps))
 * * (tgt_r - est_r), the row coefficient in double from fwd_scratch, the buffer the forward call filled (|t|^2, |t - x|^2 per
 * row).  grad_out (rows) nullable (= 1).  Any row count, any T; 128-bit accesses where est, tgt and d_est rows are 16-byte aligned. */
int ctn_sdr_bwd(const float* est, const float* tgt, int rows, int T, float eps, const double* fwd_scratch, const float* grad_out,
                float coef, float* d_est, ctn_stream_t stream);

/* PIT1d(NegSDR(reduction='mean')), src/criterion/pit.py:9-44 + src/criterion/sdr.py:6-20,72-110.  est,tgt (B,S,T) contiguous.
 * loss_b (B) = min over permutations of -mean_i SDR(est_i, tgt_perm[i]); perm (B,S) int64 (first minimum on ties, lexicographic
 * permutation order); loss_mean (1, nullable) = mean over the batch; pair_sdr (nullable) (B,S,S) = SDR(est_i, tgt_j).
 * One pass forms |t_j|^2 and the explicit residual table |t_j - est_i|^2, then ctn_sisdr_pit_fwd's permutation scoring.
 * scratch: ctn_sdr_pit_scratch_bytes(B, S) = double[B][S*S + S], zero-initialised by the callee.  S <= 6, any B, any T.
 * ctn_sdr_pit_bwd: d_est (B,S,T) = grad_loss_b[b] (nullable: 1) * coef * dSDR(est_i, tgt_perm[i])/d est_i from the forward's
 * scratch and perm; coef = -1/S for NegSDR(reduction='mean'), -1 for 'sum'. */
size_t ctn_sdr_pit_scratch_bytes(int B, int S);
int ctn_sdr_pit_fwd(const float* est, const float* tgt, int B, int S, int T, float eps, float* loss_b, int64_t* perm, float* loss_mean,
                    float* pair_sdr, double* scratch, ctn_stream_t stream);
int ctn_sdr_pit_bwd(const float* est, const float* tgt, const int64_t* perm, int B, int S, int T, float eps, const double* fwd_scratch,
                    const float* grad_loss_b, float coef, float* d_est, ctn_stream_t stream);

/* ORPIT(NegSISDR | SISDR), one-and-rest PIT, src/criterion/pit.py:87-160.  est (B,2,T), tgt (B,n,T) contiguous (any T, no
 * alignment needed); n_b (B) int32 device array, nullable (= n for every sample): sample b uses targets 0..n_b[b]-1, each n_b in
 * [2, n] (checked by the caller, the rows past n_b are ignored).  Candidate i scores
 *   v_i = SI-SDR(est_0, tgt_i) + SI-SDR(est_1, sum_{j<n_b, j!=i} tgt_j) / (n_b - 1)
 * loss_b (B) = -v (maximize = 0, NegSISDR) or v (maximize = 1, SISDR) at the first best candidate, indices (B) int64.
 * scratch: ctn_orpit_scratch_bytes(B, n), 8-byte aligned; ctn_orpit_bwd reads what the forward left there.
 * d_est (B,2,T) = grad_loss_b[b] (nullable: 1) * d loss_b / d est through the selected candidate.  n <= 16. */
size_t ctn_orpit_scratch_bytes(int B, int n);
int ctn_orpit_fwd(const float* est, const float* tgt, const int32_t* n_b, int B, int n, int T, float eps, int maximize,
                  float* loss_b, int64_t* indices, void* scratch, ctn_stream_t stream);
int ctn_orpit_bwd(const float* est, const float* tgt, const int32_t* n_b, const int64_t* indices, int B, int n, int T, float eps,
                  int maximize, void* scratch, const float* grad_loss_b, float* d_est, ctn_stream_t stream);

/* sinkpit(NegSISDR | SISDR), Sinkhorn PIT, src/criterion/pit.py:162-213.  est, tgt (B,S,T) contiguous (any T).
 * L[b,i,j] = -SI-SDR(est_i, tgt_j); Z = -coldness L; K times: Z -= logsumexp(Z, dim=1), Z -= logsumexp(Z, dim=2);
 * P (B,S,S) = exp(Z); loss_b (B) = sign * sum_ij (L + Z/coldness) P, sign = -1 when maximize (SISDR), else 1.
 * pair_sisdr (nullable) (B,S,S) = SI-SDR(est_i, tgt_j).  Iterations run in double, one CTA per sample.
 * scratch: ctn_sinkpit_scratch_bytes(B, S, K), 8-byte aligned, holds the pair statistics and every logsumexp for the backward.
 * ctn_sinkpit_bwd: grad_loss_b (B) nullable (= 1), grad_P (B,S,S) nullable (= 0) -> dL (B,S,S) = d loss / d L through all K
 * iterations (the unrolled gradient, not the converged P), and d_est (B,S,T).  S <= 16, K >= 0, coldness > 0. */
size_t ctn_sinkpit_scratch_bytes(int B, int S, int K);
int ctn_sinkpit_fwd(const float* est, const float* tgt, int B, int S, int T, int K, double coldness, float eps, int maximize,
                    float* loss_b, float* P, float* pair_sisdr, void* scratch, ctn_stream_t stream);
int ctn_sinkpit_bwd(const float* est, const float* tgt, int B, int S, int T, int K, double coldness, float eps, int maximize,
                    void* scratch, const float* grad_loss_b, const float* grad_P, float* dL, float* d_est, ctn_stream_t stream);

/* Training-step remainder, egs/wsj0-mix/common/src/driver.py:152-155 (clip_grad_norm_(max_norm) + Adam.step()), on the flat
 * gradient bucket of ctn_convtasnet_bwd: g *= min(1, max_norm/(||g||+1e-6)) (max_norm <= 0: no clipping), then torch.optim.Adam
 * arithmetic (amsgrad off).  params: device array of n_tensors parameter pointers; flat_off / numel: element offset of each
 * tensor's gradient inside flat_grad / its size; exp_avg, exp_avg_sq: Adam state laid out like flat_grad; lr (float) and step
 * (int64, advanced by one) are DEVICE scalars (graph-replayable); chunk_table: int32 pairs (tensor, offset) from
 * ctn_clip_adam_chunks (host helper: returns the chunk count; pass null outputs to size the table); norm_out nullable (1).
 * ||g|| is the norm over the listed tensors only, so flat_grad may hold other values between or around them (padding, the
 * gradients of frozen tensors); flat_numel is not read. */
int ctn_clip_adam_chunks(const int* numel, int n_tensors, int* chunk_tensor, int* chunk_offset, int capacity);
int ctn_clip_adam_step(const int32_t* chunk_table, int n_chunks, float* const* params, const long long* flat_off,
                       const int32_t* numel, int n_tensors, const float* flat_grad, size_t flat_numel, float* exp_avg,
                       float* exp_avg_sq, double* sumsq_scratch, const float* lr, long long* step, float beta1, float beta2, float eps,
                       float weight_decay, float max_norm, float* norm_out, ctn_stream_t stream);

/* BSS Eval, src/utils/bss.py:4-30 (mir_eval 0.7 bss_eval_sources, filter length 512) in fp64.  ref (B,S,T) references,
 * est (B,K,S,T): K sets of S estimates scored against the same references (the tester's estimate and repeated mixture share the
 * Gram matrix of the references and its factorisations).  Outputs (B,K,S), indexed by reference j: sdr, sir, sar of the estimate
 * perm[j] assigned to reference j.  compute_permutation = 1: perm maximises the mean SIR over itertools.permutations order (first
 * maximum); 0: perm is the identity.  status (B) int32: 0, or the CTN_BSS_* bits of the item (its outputs are then undefined).
 * A Gram matrix that is not numerically positive definite is reported (CTN_BSS_NOT_PD), where mir_eval falls back to lstsq.
 * All arithmetic in double, no atomics: the same inputs give the same bits.  S <= 4 and B*K*S <= 65535 (else CTN_EUNSUPPORTED).
 * ws: ctn_bss_workspace_bytes(), 256-byte aligned; it depends on (B, K, S) only, not on T.  No host synchronisation inside. */
enum ctn_bss_status { CTN_BSS_SILENT_REF = 1, CTN_BSS_SILENT_EST = 2, CTN_BSS_NOT_PD = 4 };
int ctn_bss_workspace_bytes(int B, int K, int S, int T, size_t* bytes);
int ctn_bss_eval_sources(const float* ref, const float* est, int B, int K, int S, int T, int compute_permutation, double* sdr,
                         double* sir, double* sar, int32_t* perm, int32_t* status, void* ws, size_t ws_bytes, ctn_stream_t stream);

/* BSS Eval v4 of multichannel source images: museval 0.4 `evaluate(references, estimates, win, hop, mode='v4')` in fp64
 * (distortion filters of 512 taps over all sources and channels, computed once over the whole track; SDR / ISR / SIR / SAR per
 * window).  ref, est (J, I, T): J sources of I channels, time-contiguous, estimate j scored against reference j (no permutation).
 * Outputs sdr, isr, sir, sar (J, nwin) with nwin = floor((T - win + hop) / hop); a window in which the channel sum of some source
 * is zero throughout, in the references or in the estimates, is NaN for every source; a zero denominator gives +inf.
 * status (1) int32: 0, or CTN_BSS_NOT_PD when a Cholesky pivot of G + eps I or of a diagonal block was not positive and finite
 * (museval would fall back to lstsq; the outputs are then undefined), e.g. when J I 512 > T + 511.
 * J I <= 8 (else CTN_EUNSUPPORTED); J, I, T, win, hop >= 1 and nwin >= 1 (else CTN_EINVAL).  All arithmetic in double, no
 * atomics and no host synchronisation: the same inputs give the same bits, and a call can be captured in a CUDA graph.
 * ws: ctn_bss_images_workspace_bytes(), 256-byte aligned; it depends on (J, I) and nwin, not otherwise on T. */
int ctn_bss_images_workspace_bytes(int J, int I, int T, int win, int hop, size_t* bytes);
int ctn_bss_eval_images(const float* ref, const float* est, int J, int I, int T, int win, int hop, double* sdr, double* isr,
                        double* sir, double* sar, int32_t* status, void* ws, size_t ws_bytes, ctn_stream_t stream);

/* number of kernel launches the last ctn_* call on this thread enqueued (for bench.py's gpu_launches) */
int ctn_last_launch_count(void);
/* kernels launched by this thread through the library since it was loaded (paths made of several entry calls: DPRNN) */
long long ctn_total_launch_count(void);

/* Stage timing with CUDA events recorded on the launching stream (bench.py's roofline leg).  ctn_profile_enable(1)
 * makes every following ctn_* call on this thread bracket its kernel groups with events; ctn_profile_read
 * synchronises on them, ADDS per-stage milliseconds / launch counts into the caller's arrays (length CTN_NSTAGES)
 * and recycles the events. */
enum ctn_stage {
  CTN_ST_PREP = 0,   /* weight folding / operand images           */
  CTN_ST_ENC = 1,    /* encoder                                   */
  CTN_ST_HEAD = 2,   /* gLN0 + bottleneck 1x1                     */
  CTN_ST_PW1 = 3,    /* per block: 1x1 B->H (+PReLU, stats)       */
  CTN_ST_DW = 4,     /* per block: gLN1 + depthwise + PReLU       */
  CTN_ST_PW2 = 5,    /* per block: [out;skip] 1x1 H->B+Sc         */
  CTN_ST_FIN = 6,    /* per block: residual / skip accumulation   */
  CTN_ST_MASK = 7,   /* PReLU + mask 1x1 + sigmoid + w*mask       */
  CTN_ST_DEC = 8,    /* decoder                                   */
  CTN_ST_LOSS = 9,   /* SI-SDR + PIT                              */
  CTN_NSTAGES = 10
};
int ctn_profile_enable(int enable);
int ctn_profile_read(double* ms, int* launches);

#ifdef __cplusplus
}
#endif
#endif /* CTN_B200_H */
