// Hopper (sm_90a) wgmma implementation of the dense 1x1 "pointwise" contractions of the Conv-TasNet path.
//
//   D[b][n][t] = epi( sum_k W[n][k] * pro(A[b][k][t]) )        A: (B,K,pitch) fp32, time contiguous
//
// TIME runs along the wgmma M dimension (64 rows per warpgroup), output channels along N = 128 per warpgroup.  A CTA computes
// 128 time steps x 1 n-tile (time split over the two warpgroups) or, for the fp16-piece TCN block contractions, 64 time steps
// x 2 n-tiles (channel split, see chan_split):
//   * the activation operand is formed by the CTA's own threads (global -> registers -> prologue -> hi/lo split) and stored
//     swizzled: fp16 pieces MN-major (rows of 64 time steps of one input channel, read with wgmma's transpose), tf32 pieces
//     K-major (rows of one time step, 32 input channels per slab);
//   * the weight operand is K-major (PyTorch (out,in,1) layout), pre-arranged once per forward into the exact swizzled
//     shared-memory image of a slab, so that one 1-D bulk async copy (TMA engine) brings a 32-channel slab of an n-tile in;
//   * the accumulator stays in registers; the fused epilogue runs on it directly.
// fp32-parity numerics: x = hi + lo with 11-bit pieces, D = A_hi W_hi + A_lo W_hi + A_hi W_lo accumulated in fp32 (the dropped
// lo*lo term is ~2^-22 relative).  Pieces are TF32 ("3xTF32", SWIZZLE_128B rows of 32 x 4 B) or FP16 ("3xFP16", weights in
// SWIZZLE_64B rows of 32 x 2 B, twice the tensor rate, weights pre-scaled per 16-row group, see wimg_f16_group) -- template
// parameter F16.
//
// Pipeline: two shared-memory stages.  While the tensor core works on slab ks (wgmma is asynchronous), all 256 threads form
// and stage slab ks + 1, whose global loads went out one slab earlier, and one thread issues the bulk copy of its weights.
#include "ctn_internal.h"
#include "ctn_wgmma_ptx.cuh"
#include "ctn_dw_math.cuh"
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

// FFMA kernels of the fp32 mode (ctn_tcn_simt.cu)
int ctn_pw_simt(const PwArgs& a, int pro, int epi, cudaStream_t st);

namespace {

constexpr int TM = 128;        // time steps per tile of the time-split kernels (2 warpgroups x wgmma M = 64)
constexpr int KS = 32;         // input channels per smem slab
constexpr int NT = 128;        // output channels per n-tile (wgmma N)
constexpr int THREADS = 256;   // 8 warps: warp w stages channels [4w, 4w+4) of every slab, each lane 4 consecutive time steps
constexpr int CPW = 4;         // channels of a slab per warp
constexpr int STAGES = 2;
constexpr int SMEM_HEADER = 1024;   // mbarriers
constexpr int F16_MAX_ROWS = 2048;  // fp16-piece mode: padded output channels of one contraction (see eff_math)

// Tiling.  The fp16-piece TCN block contractions (PRO_DW, and EPI_H) split OUTPUT CHANNELS over the two warpgroups: a CTA owns 64
// frames x 2 n-tiles, warpgroup w n-tile 2p + w, and both consume the same activation slab, so h and its depthwise stage (or the
// residual update) are formed once per frame tile instead of once per n-tile.  With an odd n-tile count (e.g. the last block's
// [out; skip] contraction, M = 128) the last CTA's second warpgroup has no n-tile: it still forms its share of each slab, and skips
// its MMAs and epilogue.  Every other kernel splits TIME: 128 frames x 1 n-tile, warpgroup w frames [64w, 64w + 64): tf32 pieces
// are K-major only (see the operand store).  The fused mask + decoder (k_maskdec) and the fp16-piece EPI_H contractions with K <=
// P1_MAX_K (pw1, k_pw1_resident) have kernels of their own; the channel-split EPI_H tile here serves K > P1_MAX_K.
template <int PRO, int EPI, bool F16>
__host__ __device__ constexpr bool chan_split() { return F16 && (PRO == PRO_DW || EPI == EPI_H); }
template <int PRO, int EPI, bool F16>
__host__ __device__ constexpr int tile_frames() { return chan_split<PRO, EPI, F16>() ? 64 : TM; }

struct TcArgs {
  PwArgs a;
  const float* wimg;    // [n_tiles][k_slabs][NPREC][NT*KS] swizzled images
  const float* oscale;  // fp16-piece mode: [n_tiles*NT] per-output-channel scale 2^-e (stored behind the images)
  int n_tiles, k_slabs, t_tiles;
  int n_groups;    // CTAs per (sample, time tile)
  // n-tiles a CTA walks back to back, always 1: a runtime loop count on purpose.  With the loop flattened the compiler lays the
  // block contractions out differently: pw1 6.87-7.15 -> 7.20-7.44 ms and pw2 7.25-7.50 -> 7.65-7.89 ms per cfg2 step (H100,
  // three runs each, alternated); with the loop kept their SASS is unchanged.
  int nt_per_cta;
};

// A thread's global loads for one slab: CPT channels x 4 time steps, NQ float4 per channel (PRO_DW: the 3 depthwise taps; PRO_RES:
// x and r).  They are issued one slab ahead of their use, so that their latency overlaps the store and the MMAs of the previous slab.
template <int PRO>
__host__ __device__ constexpr int raw_q() { return PRO == PRO_DW ? 3 : PRO == PRO_RES ? 2 : 1; }
template <int PRO, int CPT>
struct Raw { float4 q[CPT][raw_q<PRO>()]; };

// channels [c0, c0 + CPT) of the operand, time steps [tbase, tbase + 4).  PRO_DW: taps at first + k * step (clamped to the row
// outside interior tiles).
template <int PRO, int CPT>
__device__ __forceinline__ void load_raw(const PwArgs& a, int b, int c0, int tbase, int first, int step, bool interior, Raw<PRO, CPT>& r) {
#pragma unroll
  for (int j = 0; j < CPT; ++j) {
    const int c = c0 + j;
    if constexpr (PRO == PRO_DW) {
      const int cc = interior ? c : (c < a.K ? c : a.K - 1);
      const float* hr = a.A + ((size_t)b * a.K + cc) * a.pitch;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        int ts = first + k * step;
        if (!interior) ts = ts < 0 ? 0 : (ts > a.pitch - 4 ? a.pitch - 4 : ts);
        r.q[j][k] = __ldg(reinterpret_cast<const float4*>(hr + ts));
      }
    } else {
      const bool ok = c < a.K;
      r.q[j][0] = ok ? __ldg(reinterpret_cast<const float4*>(a.A + ((size_t)b * a.K + c) * a.pitch + tbase)) : make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (PRO == PRO_RES)
        r.q[j][1] = ok ? __ldg(reinterpret_cast<const float4*>(a.res_r + ((size_t)b * a.res_Mt + c) * a.pitch + tbase))
                       : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// x_new = x + rstd2*r + (v1 - mean2*rstd2*v2) for channels [c0, c0 + CPT): the previous block's deferred residual update, 0 past
// frames and past K.  `store`: also write x_new (to res_x_out, for the block after next).
template <int CPT>
__device__ __forceinline__ void res_form(const PwArgs& a, int b, int c0, int tbase, float2 mr_res, bool store, const Raw<PRO_RES, CPT>& cur,
                                         float4 (&v)[CPT]) {
#pragma unroll
  for (int j = 0; j < CPT; ++j) {
    const int k = c0 + j;
    const int kc = k < a.K ? k : a.K - 1;
    const float4 x = cur.q[j][0], r = cur.q[j][1];
    const float cst = __ldg(a.res_v1 + kc) - mr_res.x * mr_res.y * __ldg(a.res_v2 + kc);
    float4 xn;
    xn.x = fmaf(mr_res.y, r.x, x.x + cst); xn.y = fmaf(mr_res.y, r.y, x.y + cst);
    xn.z = fmaf(mr_res.y, r.z, x.z + cst); xn.w = fmaf(mr_res.y, r.w, x.w + cst);
    if (tbase + 0 >= a.frames) xn.x = 0.f;
    if (tbase + 1 >= a.frames) xn.y = 0.f;
    if (tbase + 2 >= a.frames) xn.z = 0.f;
    if (tbase + 3 >= a.frames) xn.w = 0.f;
    if (k >= a.K) xn = make_float4(0.f, 0.f, 0.f, 0.f);
    v[j] = xn;
    if (store && k < a.K) *reinterpret_cast<float4*>(a.res_x_out + ((size_t)b * a.K + k) * a.pitch + tbase) = xn;
  }
}

// Byte offset of (frame f, channel c) in a 32-channel slab of fp16 pieces, MN-major SWIZZLE_128B (ptx::wg_desc_mn128): row =
// slab channel, 128 B = 64 consecutive frames, 16-byte chunk index XOR channel % 8; 8 channels per 1 KB atom, 4 atoms down the
// slab; each 64-frame column of a 128-frame tile is its own column of atoms (4 KB apart).  A thread's 4 frames are one 8-byte store
// per piece, and a warp's store covers two 128-byte rows.
__device__ __forceinline__ uint32_t mn128_offset(uint32_t f, uint32_t c) {
  return (f >> 6) * 4096u + (c >> 3) * 1024u + (c & 7) * 128u + ((((f >> 3) & 7) ^ (c & 7)) << 4) + (f & 7) * 2u;
}

// u = PReLU(dwconv3(gLN1(h)) + bd) for channels [c0, c0 + CPT) from their loaded taps.
// TRAIN: A holds the pre-activation of h; PReLU(dw_in_slope) is applied here and the depthwise pre-activation is stored by the
// CTA that holds n-tile 0 (store_side).
template <int DCLS, bool INTERIOR, bool TRAIN, int CPT>
__device__ __forceinline__ void dw_form(const PwArgs& a, int b, int c0, int tbase, int first, int step, float2 mr1, float pslope,
                                        bool store_side, Raw<PRO_DW, CPT>& r, float4 (&v)[CPT], float2& dls, float2& dlss) {
  const float islope = TRAIN ? __ldg(a.dw_in_slope) : 0.f;
#pragma unroll
  for (int j = 0; j < CPT; ++j) {
    const int c = c0 + j;
    const int cc = INTERIOR ? c : (c < a.K ? c : a.K - 1);
    float4* q = r.q[j];
    if (TRAIN) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        q[k].x = prelu_f(q[k].x, islope); q[k].y = prelu_f(q[k].y, islope); q[k].z = prelu_f(q[k].z, islope); q[k].w = prelu_f(q[k].w, islope);
      }
    }
    const float pg = __ldg(a.dw_norm_g + cc), pb = __ldg(a.dw_norm_b + cc), pbd = __ldg(a.dw_b + cc);
    const float w0 = __ldg(a.dw_w + cc * 3), w1 = __ldg(a.dw_w + cc * 3 + 1), w2 = __ldg(a.dw_w + cc * 3 + 2);
    const float gsc = pg * mr1.y, gsh = pb - mr1.x * mr1.y * pg;
    float4 pre;
    v[j] = dw_channel<DCLS, INTERIOR, TRAIN>(q[0], q[1], q[2], gsc, gsh, w0, w1, w2, pbd, pslope, first, step, tbase, a.frames, c < a.K,
                                             dls, dlss, &pre);
    if (TRAIN && store_side && c < a.K) *reinterpret_cast<float4*>(a.dw_u_pre_out + ((size_t)b * a.K + c) * a.pitch + tbase) = pre;
  }
}

// F16 kernels fit two CTAs per SM (82 KB of shared memory for the channel-split tile, 66 KB for the time-split one).  The tf32
// kernels need 130 KB, so one CTA per SM and no register cap.
template <int PRO, int EPI, int NPASS, bool F16, bool TRAIN>
__global__ void __launch_bounds__(THREADS, F16 ? 2 : 1) k_pw_wgmma(const TcArgs g) {
  constexpr bool CSPLIT = chan_split<PRO, EPI, F16>();
  constexpr int TMC = tile_frames<PRO, EPI, F16>();          // frames of the CTA tile
  constexpr int NWG = CSPLIT ? 2 : 1;                          // n-tiles staged per slab
  constexpr int LPR = TMC / 4;                                 // lanes per channel (4 time steps per lane)
  constexpr int CPT = CPW * LPR / 32;                          // channels a thread forms per slab: 4, or 2 with the channel split
  constexpr int NPREC = NPASS == 3 ? 2 : 1;                    // precisions staged per operand (hi [, lo])
  constexpr uint32_t ROWB = F16 ? 64u : 128u;                  // bytes of 32 channels
  constexpr uint32_t A_BYTES = TMC * ROWB, W_BYTES = NT * ROWB;  // one precision of a slab
  constexpr uint32_t STAGE_BYTES = NPREC * (A_BYTES + NWG * W_BYTES);
  static_assert(F16 || CPT == CPW, "the K-major tf32 store takes a warp's 4 channels per time step");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;  // swizzle atoms need 1024-byte alignment
  uint8_t* smem = smem_raw + (base - raw);
  uint64_t* wbar = reinterpret_cast<uint64_t*>(smem);
  const uint32_t stage0 = base + SMEM_HEADER;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const PwArgs& a = g.a;

  // item -> (group of output-channel tiles, time tile, sample); the groups of one time tile are adjacent (activations shared in L2)
  const int n_groups = g.n_groups;
  const int ngrp = (int)blockIdx.x % n_groups;
  const int tt = ((int)blockIdx.x / n_groups) % g.t_tiles;
  const int b = (int)blockIdx.x / (n_groups * g.t_tiles);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) ptx::mbar_init(ptx::smem_u32(&wbar[s]), 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();

  // fp16 pieces: power-of-two scale of the activation operand (|operand| * act_s <= 2^15 by construction, ctn_act_scales),
  // undone together with the weight-group scales in the epilogue
  float act_s = 1.f;
  if (F16 && a.act_scale) act_s = __ldg(a.act_scale);
  float pslope = 0.f;
  if (PRO == PRO_PRELU || PRO == PRO_DW) pslope = __ldg(a.pro_slope);
  const int c_thr = warp * CPW + (lane / LPR) * CPT;  // first of this thread's CPT channels within a slab
  const int tbase = tt * TMC + (lane % LPR) * 4;      // first of this thread's 4 time steps
  float2 mr1 = make_float2(0.f, 1.f), mr_res = make_float2(0.f, 1.f);
  if (PRO == PRO_DW) mr1 = gln_mean_rstd(a.dw_stats_in + 2 * b, (double)a.K * (double)a.frames, a.dw_eps);
  if (PRO == PRO_RES) mr_res = gln_mean_rstd(a.res_stats + 2 * b, a.res_n, a.res_eps);
  int dcls = 4, first = tbase, step = 0;
  bool dw_interior = false;
  if (PRO == PRO_DW) {
    const int d = a.dw_dilation;
    dcls = d >= 4 ? 4 : d;
    step = dcls == 4 ? d : 4;  // d < 4: the aligned window [t - 4, t + 8)
    first = dcls == 4 ? tbase - a.dw_pad_left : tbase - 4;
    const int reach = d >= 4 ? d : 4;  // furthest sample touched on either side of the tile
    dw_interior = (tt * TMC - reach >= 0) && (tt * TMC + TMC - 1 + reach + 3 < a.frames) && (a.K % KS == 0) && (a.dw_pad_left == d);
  }

  for (int ntl = 0; ntl < g.nt_per_cta; ++ntl) {
  // nt0: first n-tile of the CTA (the CTA holding n-tile 0 also stores the prologue's side outputs); nt: this warpgroup's n-tile
  const int nt0 = CSPLIT ? 2 * ngrp : ngrp * g.nt_per_cta + ntl;
  const int nt = CSPLIT ? nt0 + wg : nt0;
  const bool wg_live = nt < g.n_tiles;  // false only for the second warpgroup of the last CTA at an odd n-tile count
  const int nw = CSPLIT ? min(2, g.n_tiles - nt0) : 1;  // n-tiles whose weights a stage holds
  const bool store_side = nt0 == 0;
  const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(g.wimg) + (size_t)nt0 * g.k_slabs * NPREC * W_BYTES;
  float2 dls = make_float2(0.f, 0.f), dlss = make_float2(0.f, 0.f);
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  Raw<PRO, CPT> cur;
  load_raw<PRO, CPT>(a, b, c_thr, tbase, first, step, dw_interior, cur);
  for (int ks = 0; ks < g.k_slabs; ++ks) {
    const int gk = ntl * g.k_slabs + ks;  // slab counter of the CTA: stage and mbarrier phase
    const int s = gk & 1;
    const uint32_t st_base = stage0 + (uint32_t)s * STAGE_BYTES;
    // the stage was last read by the MMAs of slab ks - 2, complete in both warpgroups (wait + barrier at the end of ks - 1)
    if (threadIdx.x == 0) {
      const uint32_t fb = ptx::smem_u32(&wbar[s]);
      ptx::mbar_arrive_expect_tx(fb, (uint32_t)nw * NPREC * W_BYTES);
      for (int w = 0; w < nw; ++w)
        ptx::bulk_g2s(st_base + NPREC * (A_BYTES + w * W_BYTES), wsrc + ((size_t)w * g.k_slabs + ks) * NPREC * W_BYTES, NPREC * W_BYTES, fb);
    }
    const int c0 = ks * KS + c_thr;
    float4 v[CPT];
    if constexpr (PRO == PRO_DW) {
      if (dw_interior) {
        if (dcls == 4) dw_form<4, true, TRAIN>(a, b, c0, tbase, first, step, mr1, pslope, store_side, cur, v, dls, dlss);
        else if (dcls == 2) dw_form<2, true, TRAIN>(a, b, c0, tbase, first, step, mr1, pslope, store_side, cur, v, dls, dlss);
        else dw_form<1, true, TRAIN>(a, b, c0, tbase, first, step, mr1, pslope, store_side, cur, v, dls, dlss);
      } else {
        if (dcls == 4) dw_form<4, false, TRAIN>(a, b, c0, tbase, first, step, mr1, pslope, store_side, cur, v, dls, dlss);
        else if (dcls == 2) dw_form<2, false, TRAIN>(a, b, c0, tbase, first, step, mr1, pslope, store_side, cur, v, dls, dlss);
        else dw_form<1, false, TRAIN>(a, b, c0, tbase, first, step, mr1, pslope, store_side, cur, v, dls, dlss);
      }
    } else {
#pragma unroll
      for (int j = 0; j < CPT; ++j) v[j] = cur.q[j][0];
      // the CTA holding n-tile 0 of each time tile also writes x_new
      if constexpr (PRO == PRO_RES) res_form<CPT>(a, b, c0, tbase, mr_res, store_side, cur, v);
      if (PRO == PRO_PRELU) {
#pragma unroll
        for (int j = 0; j < CPT; ++j) {
          v[j].x = prelu_f(v[j].x, pslope); v[j].y = prelu_f(v[j].y, pslope);
          v[j].z = prelu_f(v[j].z, pslope); v[j].w = prelu_f(v[j].w, pslope);
        }
      }
    }
    // the next slab's loads go out as soon as this slab's are consumed: they are in flight during its store and MMAs.  (Issuing
    // them before the forming would keep two slabs of loads in registers, which PRO_DW cannot afford under the 128-register cap.)
    if (ks + 1 < g.k_slabs) load_raw<PRO, CPT>(a, b, (ks + 1) * KS + c_thr, tbase, first, step, dw_interior, cur);
    uint8_t* sa = smem + SMEM_HEADER + (size_t)s * STAGE_BYTES;
    if (F16) {
      const uint32_t f = (uint32_t)(tbase - tt * TMC);
#pragma unroll
      for (int j = 0; j < CPT; ++j) {
        const uint32_t off = mn128_offset(f, (uint32_t)(c_thr + j));
        uint2 h2, l2;
        ptx::split_f16x2(v[j].x * act_s, v[j].y * act_s, h2.x, l2.x);
        ptx::split_f16x2(v[j].z * act_s, v[j].w * act_s, h2.y, l2.y);
        *reinterpret_cast<uint2*>(sa + off) = h2;
        *reinterpret_cast<uint2*>(sa + A_BYTES + off) = l2;
      }
    } else {
      // K-major SWIZZLE_128B (wgmma reads tf32 K-major only): row = time step, 128 B = 32 channels, 16-byte chunk (this warp's 4
      // channels) index XOR row % 8
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int t = lane * 4 + e;
        float x[CPW];
#pragma unroll
        for (int j = 0; j < CPW; ++j) x[j] = e == 0 ? v[j].x : e == 1 ? v[j].y : e == 2 ? v[j].z : v[j].w;
        const uint32_t off = (uint32_t)t * 128u + (((uint32_t)warp ^ (uint32_t)(t & 7)) << 4);
        float4 hi, lo;
        hi.x = ptx::hi_tf32(x[0]); hi.y = ptx::hi_tf32(x[1]); hi.z = ptx::hi_tf32(x[2]); hi.w = ptx::hi_tf32(x[3]);
        lo.x = x[0] - hi.x; lo.y = x[1] - hi.y; lo.z = x[2] - hi.z; lo.w = x[3] - hi.w;
        *reinterpret_cast<float4*>(sa + off) = hi;
        if (NPASS == 3) *reinterpret_cast<float4*>(sa + A_BYTES + off) = lo;
      }
    }
    ptx::fence_proxy_async_smem();
    __syncthreads();
    ptx::mbar_wait(ptx::smem_u32(&wbar[s]), (uint32_t)(gk >> 1) & 1u);
    if (wg_live) {
      // time split: warpgroup wg reads frames [64 wg, 64 wg + 64) (4 KB column / 64 K-major rows on); channel split: the whole slab
      const uint32_t a_hi = st_base + (CSPLIT ? 0u : (uint32_t)wg * 64u * ROWB), a_lo = a_hi + A_BYTES;
      const uint32_t w_hi = st_base + NPREC * (A_BYTES + (CSPLIT ? (uint32_t)wg * W_BYTES : 0u)), w_lo = w_hi + W_BYTES;
      ptx::wg_fence();
#pragma unroll
      for (int kk = 0; kk < (F16 ? KS / 16 : KS / 8); ++kk) {  // 16 fp16 / 8 tf32 channels per instruction
        if (F16) {
          // A: 16 channels = 2 atoms per step (SBO 1 KB between 8-channel atoms; LBO, the next 64 frames, is never reached at M = 64)
          const uint64_t dah = ptx::wg_desc_mn128(a_hi + kk * 2048, 4096u, 1024u), dwh = ptx::wg_desc(w_hi + kk * 32, 8 * ROWB, ptx::SW64);
          ptx::wg_mma_f16(acc, dah, dwh);
          if (NPASS == 3) {
            const uint64_t dal = ptx::wg_desc_mn128(a_lo + kk * 2048, 4096u, 1024u), dwl = ptx::wg_desc(w_lo + kk * 32, 8 * ROWB, ptx::SW64);
            ptx::wg_mma_f16(acc, dal, dwh);
            ptx::wg_mma_f16(acc, dah, dwl);
          }
        } else {
          const uint64_t dah = ptx::wg_desc(a_hi + kk * 32, 8 * ROWB, ptx::SW128), dwh = ptx::wg_desc(w_hi + kk * 32, 8 * ROWB, ptx::SW128);
          ptx::wg_mma_tf32(acc, dah, dwh);
          if (NPASS == 3) {
            const uint64_t dal = ptx::wg_desc(a_lo + kk * 32, 8 * ROWB, ptx::SW128), dwl = ptx::wg_desc(w_lo + kk * 32, 8 * ROWB, ptx::SW128);
            ptx::wg_mma_tf32(acc, dal, dwh);
            ptx::wg_mma_tf32(acc, dah, dwl);
          }
        }
      }
      ptx::wg_commit();
      ptx::wg_wait<1>();  // the MMAs of slab ks - 1 are done: its stage may be refilled
    }
    __syncthreads();
  }
  ptx::wg_wait<0>();

  if (PRO == PRO_DW && store_side) {
    const double sd = warp_sum_d((double)dls.x + (double)dls.y), ssd = warp_sum_d((double)dlss.x + (double)dlss.y);
    if (lane == 0) { atomicAdd(&a.dw_stats_out[2 * b], sd); atomicAdd(&a.dw_stats_out[2 * b + 1], ssd); }
  }
  if (!wg_live) continue;  // idle warpgroup (odd n-tile count): no outputs
  // n0 reaches the epilogue through an opaque move: otherwise the compiler forms the epilogue's per-column addresses before the
  // slab loop and spills them across it
  int n0 = nt * NT;
  asm volatile("" : "+r"(n0));

  // ===================================== EPILOGUE (on the accumulator fragment) =====================================
  float eslope = 0.f;
  if (EPI == EPI_H) eslope = __ldg(a.slope);
  const bool store_pre = EPI == EPI_H && a.store_pre != 0;  // training forward: keep the PRE-activation, statistics of PReLU(.)
  float2 mr = make_float2(0.f, 1.f);
  if (EPI == EPI_HEAD) mr = gln_mean_rstd(a.stats_in + 2 * b, a.n_in, a.eps);
  const float inv_act = 1.f / act_s;
  const int row0 = (CSPLIT ? 0 : wg * 64) + (warp & 3) * 16 + (lane >> 2);  // frame within the tile
  float ls = 0.f, lss = 0.f;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int row = row0 + 8 * ((i >> 1) & 1);
    const int n = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    const int t = tt * TMC + row;
    if (n >= a.M) continue;
    const bool tvalid = t < a.frames;
    // F16: v * osc undoes the power-of-two row scaling of the weights and the activation scale (exact)
    const float osc = F16 ? __ldg(g.oscale + n) * inv_act : 1.f;
    float v = acc[i];
    float* q = a.D + ((size_t)b * a.M + n) * a.pitch + t;
    if (EPI == EPI_RAW) {
      if (F16) v *= osc;
    } else if (EPI == EPI_HEAD) {
      const float pv = __ldg(a.v1 + n) - mr.x * mr.y * __ldg(a.v2 + n);
      v = F16 ? fmaf(mr.y * osc, v, pv) : fmaf(mr.y, v, pv);
    } else if (EPI == EPI_H) {
      const float pre = F16 ? fmaf(v, osc, __ldg(a.bias + n)) : v + __ldg(a.bias + n);
      const float act = prelu_f(pre, eslope);
      v = store_pre ? pre : act;
      if (tvalid) { ls += act; lss = fmaf(act, act, lss); }  // gLN statistics are always those of PReLU(.)
    } else if (EPI == EPI_MASK) {
      const float logit = F16 ? fmaf(v, osc, __ldg(a.bias + n)) : v + __ldg(a.bias + n);
      float mk;
      if (a.mask_logits) {  // softmax masks: the normalisation over all S*N channels is a second pass (ctn_softmax_mask)
        mk = logit;
        v = logit;
      } else {
        mk = __fdividef(1.f, 1.f + __expf(-logit));
        v = tvalid ? mk * __ldg(a.wenc + ((size_t)b * a.Nb + n % a.Nb) * a.pitch + t) : 0.f;
      }
      if (a.mask_out) a.mask_out[((size_t)b * a.M + n) * a.pitch + t] = tvalid ? mk : 0.f;
    }
    *q = tvalid ? v : 0.f;
  }
  if (EPI == EPI_H) {
    const double s = warp_sum_d((double)ls), ss = warp_sum_d((double)lss);
    if (lane == 0) { atomicAdd(&a.stats_out[2 * b], s); atomicAdd(&a.stats_out[2 * b + 1], ss); }
  }
  }  // n-tiles of the CTA
}

// ---- fused mask + decoder ----------------------------------------------------------------------------------------
// estimates[b][s][8 t + k - crop] = sum_t' sum_n w[b][n][t'] * sigmoid(logit[b][s N + n][t']) * Dec[n][k'] (ConvTranspose1d(N, 1, 16,
// stride 8), filterbank.py:245-247), logit = Wm PReLU(skip) + bm: mask 1x1, sigmoid, w * mask and the decoder in one launch, w_hat
// never reaches HBM.  fp16 pieces, time split (warpgroup w frames [64 w, 64 w + 64)).  One CTA per (sample, 128-frame tile) walks
// every n-tile of every source:
//   * the operand PReLU(skip) * act_s is formed once, and the hi / lo pieces of all its K <= MD_MAX_K channels stay resident in
//     shared memory (MN-major SWIZZLE_128B, as in k_pw_wgmma, one 16 KB slab after the other);
//   * weight slabs stream through a ring of MD_STAGES bulk-copy stages that runs on across n-tile and source boundaries: while an
//     n-tile's epilogue runs, the next n-tile's slabs are already in flight;
//   * each thread loads its 64 encoder values of an n-tile before issuing that n-tile's MMAs, so their HBM latency hides behind the
//     tensor core instead of stalling the epilogue; the n-tile's decoder taps, scales and biases go into a shared-memory table,
//     so the epilogue issues no global loads.  About 158 KB of shared memory: one CTA per SM.
// The MMAs are not overlapped with the epilogue: at cfg2 (H100) the launch takes 0.59 ms, 0.56 ms of it with the MMAs removed.
// The logits come from the same 3-piece wgmma sequence as k_pw_wgmma's (slab, then kk, then hi.hi, lo.hi, hi.lo), and w_hat and
// the decoder sums from the same float operations in the same order: per source, n-tiles ascending; per n-tile each thread's
// columns in fragment order, then the quad reduction (lane ^ 1, then lane ^ 2), then the add into the tile sums.
constexpr int MD_MAX_K = 128;  // resident operand: 4 slabs x hi / lo x 128 frames x 64 B = 64 KB
constexpr int MD_STAGES = 4;
constexpr int MD_ROW = 20;     // floats per frame row of the tile sums: 16 taps + 4 of padding, see the quad reduction
constexpr uint32_t MD_A_BYTES = TM * 64u, MD_W_BYTES = NT * 64u;  // one fp16 piece of an operand / weight slab
constexpr int MD_TAB = NT * 16 + 2 * NT;  // floats of an n-tile's epilogue table: decoder taps [tap / 4][column] (float4), scale, bias
constexpr size_t MD_SMEM = 1024 + SMEM_HEADER + (size_t)(MD_MAX_K / KS) * 2 * MD_A_BYTES + (size_t)MD_STAGES * 2 * MD_W_BYTES +
                           (size_t)TM * MD_ROW * sizeof(float) + 2 * (size_t)MD_TAB * sizeof(float);

__global__ void __launch_bounds__(THREADS, 1) k_maskdec(const TcArgs g) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  uint64_t* wbar = reinterpret_cast<uint64_t*>(smem);
  const uint32_t op0 = base + SMEM_HEADER;                                                 // resident operand
  const uint32_t ring0 = op0 + (uint32_t)(MD_MAX_K / KS) * 2 * MD_A_BYTES;                 // weight ring
  float* dacc = reinterpret_cast<float*>(smem + (ring0 - base) + MD_STAGES * 2 * MD_W_BYTES);  // [frame][MD_ROW] tile sums
  float* tab0 = dacc + TM * MD_ROW;  // two epilogue tables, n-tile parity
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const PwArgs& a = g.a;
  const int tt = (int)blockIdx.x % g.t_tiles, b = (int)blockIdx.x / g.t_tiles;
  const int ntps = a.Nb / NT, n_tiles = g.n_tiles, k_slabs = g.k_slabs;
  const int total = n_tiles * k_slabs;  // weight slabs of the launch, in image order (n-tile major)
  const uint8_t* wimg = reinterpret_cast<const uint8_t*>(g.wimg);

  for (int i = threadIdx.x; i < TM * MD_ROW; i += THREADS) dacc[i] = 0.f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < MD_STAGES; ++s) ptx::mbar_init(ptx::smem_u32(&wbar[s]), 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  // slab q goes to stage q % MD_STAGES; it may be issued once slab q - MD_STAGES has been consumed by both warpgroups
  int issued = 0;
  auto refill = [&](int consumed) {
    for (; issued < total && issued < consumed + MD_STAGES; ++issued) {
      const uint32_t fb = ptx::smem_u32(&wbar[issued % MD_STAGES]);
      ptx::mbar_arrive_expect_tx(fb, 2 * MD_W_BYTES);
      ptx::bulk_g2s(ring0 + (uint32_t)(issued % MD_STAGES) * 2 * MD_W_BYTES, wimg + (size_t)issued * 2 * MD_W_BYTES, 2 * MD_W_BYTES, fb);
    }
  };
  if (threadIdx.x == 0) refill(0);

  // ---- the operand, once: warp w forms channels [4 w, 4 w + 4) of every slab, lane l frames [4 l, 4 l + 4) of the tile
  const float act_s = __ldg(a.act_scale), pslope = __ldg(a.pro_slope);
  {
    const int tbase = tt * TM + lane * 4;
    float4 v[MD_MAX_K / KS][CPW];
#pragma unroll
    for (int ks = 0; ks < MD_MAX_K / KS; ++ks)
#pragma unroll
      for (int j = 0; j < CPW; ++j) {
        const int c = ks * KS + warp * CPW + j;
        v[ks][j] = ks < k_slabs && c < a.K ? __ldg(reinterpret_cast<const float4*>(a.A + ((size_t)b * a.K + c) * a.pitch + tbase))
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    const uint32_t f = (uint32_t)lane * 4u;
#pragma unroll
    for (int ks = 0; ks < MD_MAX_K / KS; ++ks) {
      if (ks >= k_slabs) break;
      uint8_t* sa = smem + (op0 - base) + (size_t)ks * 2 * MD_A_BYTES;
#pragma unroll
      for (int j = 0; j < CPW; ++j) {
        float4 x = v[ks][j];
        x.x = prelu_f(x.x, pslope); x.y = prelu_f(x.y, pslope); x.z = prelu_f(x.z, pslope); x.w = prelu_f(x.w, pslope);
        const uint32_t off = mn128_offset(f, (uint32_t)(warp * CPW + j));
        uint2 h2, l2;
        ptx::split_f16x2(x.x * act_s, x.y * act_s, h2.x, l2.x);
        ptx::split_f16x2(x.z * act_s, x.w * act_s, h2.y, l2.y);
        *reinterpret_cast<uint2*>(sa + off) = h2;
        *reinterpret_cast<uint2*>(sa + MD_A_BYTES + off) = l2;
      }
    }
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();

  const float inv_act = 1.f / act_s;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // frame within the tile (and row0 + 8)
  const int t0 = tt * TM + row0;
  const int S = a.M / a.Nb;
  for (int nt = 0; nt < n_tiles; ++nt) {
    const int src = nt / ntps, nb0 = (nt - src * ntps) * NT;  // source, first basis channel of the n-tile
    // this thread's encoder values, in flight during the MMAs (pitch columns are always readable; those past frames are not used)
    float wv[64];
    {
      const float* wr = a.wenc + ((size_t)b * a.Nb + nb0 + 2 * (lane & 3)) * a.pitch + t0;
#pragma unroll
      for (int i = 0; i < 64; ++i) wv[i] = __ldg(wr + (size_t)(8 * (i >> 2) + (i & 1)) * a.pitch + 8 * ((i >> 1) & 1));
    }
    // this thread's share of the n-tile's epilogue table (column threadIdx.x % 128: taps [8 h, 8 h + 8), h = threadIdx.x / 128,
    // and the scale (h = 0) or the bias (h = 1)); loaded now, stored after the MMAs
    const int tc = threadIdx.x & (NT - 1), th = threadIdx.x >> 7;
    const float4* dsrc = reinterpret_cast<const float4*>(a.dec_w + (size_t)(nb0 + tc) * 16) + 2 * th;
    const float4 td0 = __ldg(dsrc), td1 = __ldg(dsrc + 1);
    const float tsb = th == 0 ? __ldg(g.oscale + nt * NT + tc) * inv_act : __ldg(a.bias + nt * NT + tc);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int ks = 0; ks < k_slabs; ++ks) {
      const int q = nt * k_slabs + ks;
      const uint32_t w_hi = ring0 + (uint32_t)(q % MD_STAGES) * 2 * MD_W_BYTES, w_lo = w_hi + MD_W_BYTES;
      const uint32_t a_hi = op0 + (uint32_t)ks * 2 * MD_A_BYTES + (uint32_t)wg * 4096u, a_lo = a_hi + MD_A_BYTES;
      ptx::mbar_wait(ptx::smem_u32(&wbar[q % MD_STAGES]), (uint32_t)(q / MD_STAGES) & 1u);
      ptx::wg_fence();
#pragma unroll
      for (int kk = 0; kk < KS / 16; ++kk) {
        const uint64_t dah = ptx::wg_desc_mn128(a_hi + kk * 2048, 4096u, 1024u), dwh = ptx::wg_desc(w_hi + kk * 32, 8 * 64, ptx::SW64);
        const uint64_t dal = ptx::wg_desc_mn128(a_lo + kk * 2048, 4096u, 1024u), dwl = ptx::wg_desc(w_lo + kk * 32, 8 * 64, ptx::SW64);
        ptx::wg_mma_f16(acc, dah, dwh);
        ptx::wg_mma_f16(acc, dal, dwh);
        ptx::wg_mma_f16(acc, dah, dwl);
      }
      ptx::wg_commit();
    }
    ptx::wg_wait<0>();
    // the table of parity nt & 1 was last read in the epilogue of n-tile nt - 2, which every thread left before the barrier of nt - 1
    float* tab = tab0 + (nt & 1) * MD_TAB;
    float4* tdec = reinterpret_cast<float4*>(tab);  // [q4][column]: a warp's 4 distinct columns 2 apart, on distinct banks
    tdec[(2 * th) * NT + tc] = td0;
    tdec[(2 * th + 1) * NT + tc] = td1;
    tab[NT * 16 + th * NT + tc] = tsb;
    __syncthreads();  // both warpgroups are done with this n-tile's slabs (and with the previous source's flush); the table is in
    if (threadIdx.x == 0) refill((nt + 1) * k_slabs);

    // w_hat[n][t] = w[n][t] * sigmoid(logit), contracted on the spot with the decoder taps: frame t adds w_hat[n][t] * Dec[n][k] to
    // sample 8 t + k.  dpart: sum over this thread's columns, rows row0 and row0 + 8
    float dpart[2][16];
#pragma unroll
    for (int k = 0; k < 32; ++k) dpart[k >> 4][k & 15] = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int c = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      const bool tvalid = t0 + 8 * ((i >> 1) & 1) < a.frames;
      const float osc = tab[NT * 16 + c];
      const float logit = fmaf(acc[i], osc, tab[NT * 17 + c]);
      const float o = tvalid ? __fdividef(wv[i], 1.f + __expf(-logit)) : 0.f;
#pragma unroll
      for (int q4 = 0; q4 < 4; ++q4) {
        const float4 d4 = tdec[q4 * NT + c];
        float* dp = dpart[(i >> 1) & 1] + 4 * q4;
        dp[0] = fmaf(o, d4.x, dp[0]); dp[1] = fmaf(o, d4.y, dp[1]); dp[2] = fmaf(o, d4.z, dp[2]); dp[3] = fmaf(o, d4.w, dp[3]);
      }
    }
    // quad reduction as reduce-scatter: lane bit 0 keeps row row0 + 8 (bit set) or row0, lane bit 1 taps 8..15 or 0..7.  Every
    // kept sum is (v_q + v_q^1) + (v_q^2 + v_q^3), bit for bit the value a full butterfly leaves in every lane.  Row stride
    // MD_ROW = 20 floats puts the 32 lanes' 16-byte chunks on distinct banks.
    const bool hb0 = lane & 1, hb1 = lane & 2;
    float r1[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float keep = hb0 ? dpart[1][j] : dpart[0][j], send = hb0 ? dpart[0][j] : dpart[1][j];
      r1[j] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
    }
    float r2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float keep = hb1 ? r1[8 + j] : r1[j], send = hb1 ? r1[j] : r1[8 + j];
      r2[j] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    float4* dst = reinterpret_cast<float4*>(dacc + (row0 + (hb0 ? 8 : 0)) * MD_ROW + (hb1 ? 8 : 0));
    float4 u0 = dst[0], u1 = dst[1];
    u0.x += r2[0]; u0.y += r2[1]; u0.z += r2[2]; u0.w += r2[3];
    u1.x += r2[4]; u1.y += r2[5]; u1.z += r2[6]; u1.w += r2[7];
    dst[0] = u0; dst[1] = u1;

    if (nt - src * ntps == ntps - 1) {
      // the source is complete: sample 8 f + k of the tile = taps k < 8 of frame f + taps 8 + k of frame f - 1, then the crop
      // (conv_tasnet.py:169).  The first 8 samples also receive the previous tile's last frame and the 8 samples after the tile
      // belong to the next tile's first frame: those are added to the zero-initialised output with red.add, exactly two operands
      // each, so the result is order-independent.  Each tile sum is read by one thread, which clears it for the next source.  A
      // warp takes frames f, f + 2, f + 4, f + 6 (8 samples each): at the 20-float row stride their taps lie on distinct banks.
      __syncthreads();
      float* yo = a.D + ((size_t)b * S + src) * (size_t)a.dec_T_out;
      const long long tb = 8LL * tt * TM - a.dec_crop_left;
      for (int j = threadIdx.x; j < 2 * 32 * (TM / 8 + 1); j += THREADS) {
        const int u = j >> 5, f = (u >> 1) * 8 + 2 * ((j & 31) >> 3) + (u & 1), k = j & 7;
        if (f > TM) continue;
        const int sidx = 8 * f + k;
        float v = 0.f;
        if (f < TM) { v += dacc[f * MD_ROW + k]; dacc[f * MD_ROW + k] = 0.f; }
        if (f >= 1) { v += dacc[(f - 1) * MD_ROW + 8 + k]; dacc[(f - 1) * MD_ROW + 8 + k] = 0.f; }
        const long long tau = tb + sidx;
        if (tau < 0 || tau >= a.dec_T_out) continue;
        if (sidx < 8 || sidx >= 8 * TM) atomicAdd(yo + tau, v);
        else yo[tau] = v;
      }
    }
  }
}

// ---- pw1 on a resident operand -----------------------------------------------------------------------------------
// h = PReLU(W1 x + b1) with its gLN statistics (EPI_H), fp16 pieces, K <= P1_MAX_K; x is the block input (PRO_NONE) or the previous
// block's deferred residual update (PRO_RES, which also writes x_new).  One CTA per (sample, 64-frame tile) walks every n-tile:
//   * every global load of the tile's operand is issued before any of it is formed (at K = 128, 8 float4 of x and 8 of r per
//     thread); x_new is formed and stored once, and its hi / lo pieces stay resident in shared memory for every pass (32 KB,
//     the MN-major layout of mn128_offset);
//   * channel split as in k_pw_wgmma: warpgroup w computes n-tile 2p + w in pass p (at an odd n-tile count the second warpgroup
//     has one pass less).  Each warpgroup streams its own n-tile's weight slabs through a ring of P1_WST bulk-copy stages that
//     runs on across passes, so the next pass's first slabs arrive during this pass's epilogue; the warpgroups only meet again
//     at the end;
//   * each pass's output scales and biases are loaded while its MMAs run and go into a shared-memory table, so the epilogue
//     issues no global loads;
//   * the gLN statistics are reduced per CTA before the double atomics.
// h and x_new are bit for bit those of k_pw_wgmma's channel-split tile: the same prologue, the same 3-piece wgmma sequence
// (slab, then kk, then hi.hi, lo.hi, hi.lo) and the same epilogue operations.  Only the order of the double statistics sums differs.
// About 102 KB of shared memory: two CTAs per SM, so one CTA's loads overlap the other's epilogue stores.
constexpr int P1_MAX_K = 128;
constexpr int P1_TF = 64;   // frames per CTA
constexpr int P1_WST = 2;   // weight stages per warpgroup
constexpr uint32_t P1_A_BYTES = P1_TF * 64u, P1_W_BYTES = NT * 64u;  // one fp16 piece of an operand / weight slab
constexpr size_t P1_SMEM = 1024 + SMEM_HEADER + (size_t)(P1_MAX_K / KS) * 2 * P1_A_BYTES + (size_t)2 * P1_WST * 2 * P1_W_BYTES +
                           (size_t)2 * 2 * 2 * NT * sizeof(float) + (size_t)(THREADS / 32) * 2 * sizeof(double);

// the 128 threads of warpgroup wg
__device__ __forceinline__ void wg_bar(int wg) {
  if (wg == 0) ptx::named_bar_sync<1, 128>();
  else ptx::named_bar_sync<2, 128>();
}

template <int PRO>
__global__ void __launch_bounds__(THREADS, 2) k_pw1_resident(const TcArgs g) {
  static_assert(PRO == PRO_NONE || PRO == PRO_RES, "pw1 prologues");
  constexpr int NSL = P1_MAX_K / KS;
  constexpr int CPT = 2;  // channels a thread forms per slab: warp w channels [4 w, 4 w + 4), 16 lanes x 4 frames per channel
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  uint64_t* wbar = reinterpret_cast<uint64_t*>(smem);  // [warpgroup][stage]
  const uint32_t op0 = base + SMEM_HEADER;                                                  // resident operand
  const uint32_t ring0 = op0 + (uint32_t)NSL * 2 * P1_A_BYTES;                               // weight rings
  float* tab0 = reinterpret_cast<float*>(smem + (ring0 - base) + 2 * P1_WST * 2 * P1_W_BYTES);  // [warpgroup][parity][scale | bias]
  double* red = reinterpret_cast<double*>(tab0 + 2 * 2 * 2 * NT);                             // [warp][sum, sumsq]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2, lt = threadIdx.x & (NT - 1);
  const PwArgs& a = g.a;
  const int tt = (int)blockIdx.x % g.t_tiles, b = (int)blockIdx.x / g.t_tiles;
  const int k_slabs = g.k_slabs;
  const int passes = g.n_tiles > wg ? (g.n_tiles - wg + 1) / 2 : 0;  // this warpgroup's n-tiles 2p + wg
  const int total = passes * k_slabs;                                 // its weight slabs, pass-major
  const uint8_t* wimg = reinterpret_cast<const uint8_t*>(g.wimg);
  const uint32_t ring = ring0 + (uint32_t)wg * P1_WST * 2 * P1_W_BYTES;

  if (threadIdx.x == 0) {
    for (int s = 0; s < 2 * P1_WST; ++s) ptx::mbar_init(ptx::smem_u32(&wbar[s]), 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  // slab u of the warpgroup goes to stage u % P1_WST; it may be issued once slab u - P1_WST has been consumed by all 4 warps
  int issued = 0;
  auto refill = [&](int consumed) {
    for (; issued < total && issued < consumed + P1_WST; ++issued) {
      const int p = issued / k_slabs, ks = issued - p * k_slabs;
      const uint32_t fb = ptx::smem_u32(&wbar[wg * P1_WST + issued % P1_WST]);
      ptx::mbar_arrive_expect_tx(fb, 2 * P1_W_BYTES);
      ptx::bulk_g2s(ring + (uint32_t)(issued % P1_WST) * 2 * P1_W_BYTES, wimg + ((size_t)(2 * p + wg) * k_slabs + ks) * 2 * P1_W_BYTES,
                    2 * P1_W_BYTES, fb);
    }
  };
  if (lt == 0) refill(0);

  // ---- the operand, once
  const float act_s = __ldg(a.act_scale);
  {
    const int c_thr = warp * CPW + (lane / 16) * CPT;
    const int tbase = tt * P1_TF + (lane % 16) * 4;
    Raw<PRO, CPT> cur[NSL];
#pragma unroll
    for (int ks = 0; ks < NSL; ++ks)
      if (ks < k_slabs) load_raw<PRO, CPT>(a, b, ks * KS + c_thr, tbase, 0, 0, false, cur[ks]);
    float2 mr_res = make_float2(0.f, 1.f);
    if (PRO == PRO_RES) mr_res = gln_mean_rstd(a.res_stats + 2 * b, a.res_n, a.res_eps);
    const uint32_t f = (uint32_t)(tbase - tt * P1_TF);
#pragma unroll
    for (int ks = 0; ks < NSL; ++ks) {
      if (ks >= k_slabs) break;
      float4 v[CPT];
      if constexpr (PRO == PRO_RES) {
        res_form<CPT>(a, b, ks * KS + c_thr, tbase, mr_res, true, cur[ks], v);
      } else {
#pragma unroll
        for (int j = 0; j < CPT; ++j) v[j] = cur[ks].q[j][0];
      }
      uint8_t* sa = smem + (op0 - base) + (size_t)ks * 2 * P1_A_BYTES;
#pragma unroll
      for (int j = 0; j < CPT; ++j) {
        const uint32_t off = mn128_offset(f, (uint32_t)(c_thr + j));
        uint2 h2, l2;
        ptx::split_f16x2(v[j].x * act_s, v[j].y * act_s, h2.x, l2.x);
        ptx::split_f16x2(v[j].z * act_s, v[j].w * act_s, h2.y, l2.y);
        *reinterpret_cast<uint2*>(sa + off) = h2;
        *reinterpret_cast<uint2*>(sa + P1_A_BYTES + off) = l2;
      }
    }
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();

  const float inv_act = 1.f / act_s, eslope = __ldg(a.slope);
  const bool store_pre = a.store_pre != 0;  // training forward: keep the PRE-activation, statistics of PReLU(.)
  const int row0 = (warp & 3) * 16 + (lane >> 2);  // frame within the tile (and row0 + 8)
  double cs = 0.0, css = 0.0;
  for (int p = 0; p < passes; ++p) {
    const int nt = 2 * p + wg;
    // this thread's column of the pass's epilogue table, in flight during the MMAs
    const int tn = nt * NT + lt;
    const float tsc = tn < a.M ? __ldg(g.oscale + tn) * inv_act : 0.f;
    const float tbi = tn < a.M ? __ldg(a.bias + tn) : 0.f;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int ks = 0; ks < k_slabs; ++ks) {
      const int u = p * k_slabs + ks;
      const uint32_t w_hi = ring + (uint32_t)(u % P1_WST) * 2 * P1_W_BYTES, w_lo = w_hi + P1_W_BYTES;
      const uint32_t a_hi = op0 + (uint32_t)ks * 2 * P1_A_BYTES, a_lo = a_hi + P1_A_BYTES;
      ptx::mbar_wait(ptx::smem_u32(&wbar[wg * P1_WST + u % P1_WST]), (uint32_t)(u / P1_WST) & 1u);
      ptx::wg_fence();
#pragma unroll
      for (int kk = 0; kk < KS / 16; ++kk) {
        const uint64_t dah = ptx::wg_desc_mn128(a_hi + kk * 2048, 4096u, 1024u), dwh = ptx::wg_desc(w_hi + kk * 32, 8 * 64, ptx::SW64);
        const uint64_t dal = ptx::wg_desc_mn128(a_lo + kk * 2048, 4096u, 1024u), dwl = ptx::wg_desc(w_lo + kk * 32, 8 * 64, ptx::SW64);
        ptx::wg_mma_f16(acc, dah, dwh);
        ptx::wg_mma_f16(acc, dal, dwh);
        ptx::wg_mma_f16(acc, dah, dwl);
      }
      ptx::wg_commit();
      if (ks > 0) {
        ptx::wg_wait<1>();  // slab u - 1 is consumed in this warp ...
        wg_bar(wg);         // ... and in the warpgroup: its stage may be refilled
        if (lt == 0) refill(u);
      }
    }
    ptx::wg_wait<0>();
    // the table of parity p & 1 was last read in the epilogue of pass p - 2, which every warp of the warpgroup left before the
    // barrier of pass p - 1
    float* tab = tab0 + (wg * 2 + (p & 1)) * 2 * NT;
    tab[lt] = tsc;
    tab[NT + lt] = tbi;
    wg_bar(wg);  // the pass's slabs are consumed and the table is in
    if (lt == 0) refill((p + 1) * k_slabs);

    // n0 reaches the epilogue through an opaque move, so that the per-column addresses are not formed ahead of the slab loop
    int n0 = nt * NT;
    asm volatile("" : "+r"(n0));
    float ls = 0.f, lss = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int row = row0 + 8 * ((i >> 1) & 1);
      const int c = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      const int n = n0 + c;
      const int t = tt * P1_TF + row;
      if (n >= a.M) continue;
      const bool tvalid = t < a.frames;
      // v * scale undoes the power-of-two row scaling of the weights and the activation scale (exact)
      const float pre = fmaf(acc[i], tab[c], tab[NT + c]);
      const float act = prelu_f(pre, eslope);
      if (tvalid) { ls += act; lss = fmaf(act, act, lss); }  // gLN statistics are always those of PReLU(.)
      a.D[((size_t)b * a.M + n) * a.pitch + t] = tvalid ? (store_pre ? pre : act) : 0.f;
    }
    cs += warp_sum_d((double)ls);
    css += warp_sum_d((double)lss);
  }
  if (lane == 0) { red[2 * warp] = cs; red[2 * warp + 1] = css; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0, ss = 0.0;
    for (int w = 0; w < THREADS / 32; ++w) { s += red[2 * w]; ss += red[2 * w + 1]; }
    atomicAdd(&a.stats_out[2 * b], s);
    atomicAdd(&a.stats_out[2 * b + 1], ss);
  }
}

// ---- weight images ---------------------------------------------------------------------------------------------
// K-major SWIZZLE_128B image of an (n_tile x KS=32) tf32 weight slab: rows of 128 B, 8-row groups of 1024 B, 16-byte chunk
// index XOR (row & 7).  Float offset of element (row nl, k kl):
__host__ __device__ __forceinline__ int wimg_offset(int nl, int kl) {
  return (nl >> 3) * 256 + (nl & 7) * 32 + ((((kl >> 2) ^ (nl & 7)) << 2) | (kl & 3));
}

// fp16 variant ("3xFP16"): K-major SWIZZLE_64B rows of 32 k x 2 B; per slab a hi image then a lo image of n_tile*64 bytes.
// Every group of 16 weight ROWS (output channels) is first scaled by a power of two 2^e so that its largest entry lands in
// [2^9, 2^10) (one scale per 16 rows = per 16-column epilogue chunk, so the epilogue needs a single scalar per chunk):
// hi and lo pieces then sit in fp16's normal range whatever the magnitude of the weights (tiny gamma-folded rows would
// otherwise lose their lo piece to fp16's subnormal floor of 6e-8, huge ones would saturate); the epilogue multiplies the
// accumulator of channel n by the exact inverse 2^-e (oscale, stored behind the images).
// One warp per row; block = 16 warps = one 16-row scale group (the epilogue reads one scale per 16-column chunk).
__device__ __forceinline__ void wimg_f16_group(const float* __restrict__ W, int M, int K, int n_tile, int k_slabs, int nt, int grp,
                                               __half* __restrict__ img, float* __restrict__ oscale, float* smax) {
  static_assert(KS == 32, "one lane per channel of a slab");
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nl = grp * 16 + wid;
  const int n = nt * n_tile + nl;
  const bool live = nl < n_tile && n < M;
  const float* row = W + (size_t)n * K;
  float mx = 0.f;
  if (live)
    for (int k = lane; k < K; k += 32) mx = fmaxf(mx, fabsf(row[k]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) smax[wid] = mx;
  __syncthreads();
  mx = smax[lane & 15];
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __syncthreads();  // smax is reused by the next group of this block
  int e = 0;
  if (mx > 0.f && mx < INFINITY) e = 9 - ilogbf(mx);  // 2^e * (largest entry of the 16 rows) in [2^9, 2^10)
  e = max(-100, min(100, e));
  const float up = ldexpf(1.f, e), down = ldexpf(1.f, -e);
  if (nl >= n_tile) return;
  if (lane == 0) oscale[n] = down;
  const size_t per = (size_t)n_tile * KS;  // halves per precision
  for (int ks = 0; ks < k_slabs; ++ks) {
    const int kl = lane, k = ks * KS + kl;  // KS == 32 == warp size
    const float x = (live && k < K) ? row[k] * up : 0.f;
    __half* dst = img + ((size_t)nt * k_slabs + ks) * 2 * per;
    const int off = (nl >> 3) * 256 + (nl & 7) * 32 + ((((kl >> 3) ^ ((nl >> 1) & 3))) << 3) + (kl & 7);  // in halves
    const __half hi = __float2half_rn(x);
    dst[off] = hi;
    dst[per + off] = __float2half_rn(x - __half2float(hi));
  }
}
__host__ __device__ inline size_t wimg_f16_image_bytes(int n_tile, int n_tiles, int k_slabs) {
  return (size_t)n_tiles * k_slabs * 2 * n_tile * KS * sizeof(__half);
}

struct WimgJobs { WimgJob j[CTN_MAX_JOBS]; };
// tf32 image(s) of slab ks of n-tile nt.  __restrict__ lets the compiler issue the loads of W ahead of the image stores; the
// pointers of a WimgJob carry no such promise, hence the helper.
__device__ __forceinline__ void wimg_tf32_slab(const float* __restrict__ W, int M, int K, int k_slabs, int nt, int ks, int nprec,
                                               float* __restrict__ wimg) {
  const int n_tile = NT;
  const size_t per = (size_t)n_tile * KS;  // floats per precision
  float* dst = wimg + ((size_t)nt * k_slabs + ks) * nprec * per;
  for (int i = threadIdx.x; i < n_tile * KS; i += 256) {
    const int nl = i / KS, kl = i % KS;
    const int n = nt * n_tile + nl, k = ks * KS + kl;
    const float x = (n < M && k < K) ? W[(size_t)n * K + k] : 0.f;
    const int off = wimg_offset(nl, kl);
    const float hi = ptx::to_tf32(x);
    dst[off] = hi;
    if (nprec == 2) dst[per + off] = ptx::to_tf32(x - hi);
  }
}

// grid (blocks of the largest job, jobs): one block per (slab, n-tile) of one job.  No grid-stride loop: with one, the loads
// lose their early issue and a single image takes about three times as long to build (H100).
__global__ void __launch_bounds__(256) k_build_wimg_batch(const WimgJobs jobs, int nprec) {
  const WimgJob& jb = jobs.j[blockIdx.y];
  const int n_tiles = (jb.M + NT - 1) / NT, k_slabs = (jb.K + KS - 1) / KS;
  const int blk = blockIdx.x;
  if (blk >= n_tiles * k_slabs) return;
  const int nt = blk / k_slabs, ks = blk - nt * k_slabs;
  wimg_tf32_slab(jb.W, jb.M, jb.K, k_slabs, nt, ks, nprec, jb.wimg);
}

// grid (blocks of the largest job, jobs), block 512: blockIdx.x walks the (n-tile, 16-row group) pairs of its job
__global__ void __launch_bounds__(512) k_build_wimg_batch_f16(const WimgJobs jobs) {
  __shared__ float smax[16];
  const WimgJob& jb = jobs.j[blockIdx.y];
  const int n_tile = NT;
  const int n_tiles = (jb.M + n_tile - 1) / n_tile, k_slabs = (jb.K + KS - 1) / KS;
  const int groups = n_tile / 16;
  __half* img = reinterpret_cast<__half*>(jb.wimg);
  float* oscale = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(jb.wimg) + wimg_f16_image_bytes(n_tile, n_tiles, k_slabs));
  for (int blk = blockIdx.x; blk < n_tiles * groups; blk += gridDim.x)
    wimg_f16_group(jb.W, jb.M, jb.K, n_tile, k_slabs, blk / groups, blk % groups, img, oscale, smax);
}

// the fp16-piece mode keeps one scale per padded output channel: contractions with more than F16_MAX_ROWS padded output
// channels use the tf32 pieces instead (images and kernel are chosen by the same rule)
int eff_math(int M, int math) {
  if (math != CTN_MATH_F16X3) return math;
  return ((M + NT - 1) / NT) * NT > F16_MAX_ROWS ? CTN_MATH_TF32X3 : math;
}

template <int PRO, int EPI, int NPASS, bool F16, bool TRAIN>
int launch(const TcArgs& g0, cudaStream_t st) {
  constexpr int NPREC = NPASS == 3 ? 2 : 1;
  constexpr bool CSPLIT = chan_split<PRO, EPI, F16>();
  constexpr int TMC = tile_frames<PRO, EPI, F16>();
  constexpr size_t smem = SMEM_HEADER + 1024 + (size_t)STAGES * NPREC * (TMC + (CSPLIT ? 2 : 1) * NT) * (F16 ? 64 : 128);
  TcArgs g = g0;
  g.t_tiles = g.a.pitch / TMC;
  g.n_groups = CSPLIT ? (g.n_tiles + 1) / 2 : g.n_tiles / g.nt_per_cta;
  static bool attr_done[CTN_MAX_DEVICES] = {false};  // the opt-in is per device (context)
  const int dev = ctn_current_device();
  if (!attr_done[dev]) {
    cudaError_t e = cudaFuncSetAttribute(k_pw_wgmma<PRO, EPI, NPASS, F16, TRAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done[dev] = true;
  }
  const long long grid = (long long)g.a.B * g.t_tiles * g.n_groups;
  if (grid > 0x7fffffffLL) return CTN_EUNSUPPORTED;
  k_pw_wgmma<PRO, EPI, NPASS, F16, TRAIN><<<(unsigned)grid, THREADS, smem, st>>>(g);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

template <int PRO, int EPI, bool TRAIN = false>
int launch_math(const TcArgs& g, int math, cudaStream_t st) {
  if (math == CTN_MATH_F16X3) return launch<PRO, EPI, 3, true, TRAIN>(g, st);
  if (math == CTN_MATH_TF32) return launch<PRO, EPI, 1, false, TRAIN>(g, st);
  return launch<PRO, EPI, 3, false, TRAIN>(g, st);
}

// Pieces of one contraction in the model's mode `math`.  fp16 pieces have 5 exponent bits, so they are only safe on an
// operand with a static bound, i.e. a contraction that carries an operand scale (PwArgs::act_scale, from ctn_act_scales);
// every other contraction of the f16x3 mode runs on tf32 pieces.  Weight images and kernels follow the same rule.
int piece_math(int math, bool bounded) { return math == CTN_MATH_F16X3 && !bounded ? CTN_MATH_TF32X3 : math; }

// weight images of jobs that all take the pieces `math` (eff_math already applied), CTN_MAX_JOBS per launch
int build_images(const WimgJob* jobs, int n, int math, cudaStream_t st) {
  const bool f16 = math == CTN_MATH_F16X3;
  for (int i0 = 0; i0 < n; i0 += CTN_MAX_JOBS) {
    WimgJobs wj;
    const int m = n - i0 < CTN_MAX_JOBS ? n - i0 : CTN_MAX_JOBS;
    int maxb = 1;
    for (int i = 0; i < m; ++i) {
      const WimgJob& jb = jobs[i0 + i];
      wj.j[i] = jb;
      const int blocks = ((jb.M + NT - 1) / NT) * (f16 ? NT / 16 : (jb.K + KS - 1) / KS);
      if (blocks > maxb) maxb = blocks;
    }
    if (f16) k_build_wimg_batch_f16<<<dim3(maxb, m), 512, 0, st>>>(wj);
    else k_build_wimg_batch<<<dim3(maxb, m), 256, 0, st>>>(wj, math == CTN_MATH_TF32 ? 1 : 2);  // hi [, lo]
    CTN_COUNT_LAUNCH();
  }
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// fused mask + decoder (k_maskdec): fp16-piece mode, whole n-tiles per source, decoder basis (Nb, 1, 16) with kernel 16 /
// stride 8, and an operand small enough to stay resident (K <= MD_MAX_K); otherwise the caller runs EPI_MASK and the decoder
bool maskdec_ok(const PwArgs& a, int pmath) {
  return eff_math(a.M, pmath) == CTN_MATH_F16X3 && a.dec_w && a.Nb > 0 && a.Nb % NT == 0 && a.M % a.Nb == 0 && a.K <= MD_MAX_K &&
         (((uintptr_t)a.dec_w) & 15) == 0;
}

int launch_maskdec(const TcArgs& g0, cudaStream_t st) {
  TcArgs g = g0;
  g.t_tiles = g.a.pitch / TM;
  g.n_groups = 1;
  static bool attr_done[CTN_MAX_DEVICES] = {false};
  const int dev = ctn_current_device();
  if (!attr_done[dev]) {
    cudaError_t e = cudaFuncSetAttribute(k_maskdec, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MD_SMEM);
    if (e != cudaSuccess) return (int)e;
    attr_done[dev] = true;
  }
  const long long grid = (long long)g.a.B * g.t_tiles;
  if (grid > 0x7fffffffLL) return CTN_EUNSUPPORTED;
  k_maskdec<<<(unsigned)grid, THREADS, MD_SMEM, st>>>(g);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

template <int PRO>
int launch_pw1(const TcArgs& g0, cudaStream_t st) {
  TcArgs g = g0;
  g.t_tiles = g.a.pitch / P1_TF;
  g.n_groups = 1;
  static bool attr_done[CTN_MAX_DEVICES] = {false};
  const int dev = ctn_current_device();
  if (!attr_done[dev]) {
    cudaError_t e = cudaFuncSetAttribute(k_pw1_resident<PRO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P1_SMEM);
    if (e != cudaSuccess) return (int)e;
    attr_done[dev] = true;
  }
  const long long grid = (long long)g.a.B * g.t_tiles;
  if (grid > 0x7fffffffLL) return CTN_EUNSUPPORTED;
  k_pw1_resident<PRO><<<(unsigned)grid, THREADS, P1_SMEM, st>>>(g);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

// a.wimg holds the image of a.W in the pieces `pmath`
int launch_wgmma(const PwArgs& a, int pro, int epi, int pmath, cudaStream_t st) {
  if (!a.wimg) return CTN_EINVAL;
  const int math = eff_math(a.M, pmath);
  if (a.pitch % TM != 0) return CTN_EALIGN;
  if ((((uintptr_t)a.A) | ((uintptr_t)a.wimg)) & 15) return CTN_EALIGN;
  TcArgs g;
  g.a = a;
  g.wimg = a.wimg;
  g.n_tiles = (a.M + NT - 1) / NT;
  g.k_slabs = (a.K + KS - 1) / KS;
  g.oscale = math == CTN_MATH_F16X3
                 ? reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(a.wimg) + wimg_f16_image_bytes(NT, g.n_tiles, g.k_slabs))
                 : nullptr;
  g.nt_per_cta = 1;
  const bool train_dw = pro == PRO_DW && a.dw_u_pre_out != nullptr;
  if (pro == PRO_NONE && epi == EPI_RAW) return launch_math<PRO_NONE, EPI_RAW>(g, math, st);
  if (pro == PRO_DW && epi == EPI_RAW)
    return train_dw ? launch_math<PRO_DW, EPI_RAW, true>(g, math, st) : launch_math<PRO_DW, EPI_RAW>(g, math, st);
  if (pro == PRO_NONE && epi == EPI_HEAD) return launch_math<PRO_NONE, EPI_HEAD>(g, math, st);
  // pw1 on fp16 pieces: the resident-operand kernel up to P1_MAX_K input channels, k_pw_wgmma's channel-split tile beyond
  if (epi == EPI_H && math == CTN_MATH_F16X3 && a.K <= P1_MAX_K) {
    if (pro == PRO_NONE) return launch_pw1<PRO_NONE>(g, st);
    if (pro == PRO_RES) return launch_pw1<PRO_RES>(g, st);
  }
  if (pro == PRO_NONE && epi == EPI_H) return launch_math<PRO_NONE, EPI_H>(g, math, st);
  if (pro == PRO_RES && epi == EPI_H) return launch_math<PRO_RES, EPI_H>(g, math, st);
  if (pro == PRO_PRELU && epi == EPI_MASK) return launch_math<PRO_PRELU, EPI_MASK>(g, math, st);
  if (pro == PRO_PRELU && epi == EPI_MASKDEC) {
    if (!maskdec_ok(a, pmath)) return CTN_EUNSUPPORTED;
    return launch_maskdec(g, st);
  }
  return CTN_EUNSUPPORTED;
}

}  // namespace

// the tensor-core (hi/lo split) numeric modes are built
extern "C" int ctn_has_tcgen05(void) { return 1; }

size_t ctn_pw_wimg_bytes(int M, int K, int math) {
  const int nprec = math == CTN_MATH_TF32 ? 1 : 2;
  const int n_tiles = (M + NT - 1) / NT, k_slabs = (K + KS - 1) / KS;
  // fp16 images are half the size but carry the per-channel scale array behind them; the tf32x3 size + scales covers both
  return (size_t)n_tiles * k_slabs * nprec * NT * KS * sizeof(float) + (size_t)n_tiles * NT * sizeof(float) + 256;
}

size_t ctn_pw_wimg_max_bytes(const int (*shapes)[2], int n, int math) {
  if (math == CTN_MATH_FP32) return 256;
  size_t mx = 0;
  for (int i = 0; i < n; ++i) {
    const size_t b = ctn_pw_wimg_bytes(shapes[i][0], shapes[i][1], math);
    if (b > mx) mx = b;
  }
  return mx;
}

int ctn_pw_prepare(const PwArgs& a, int math, float* wimg, cudaStream_t st) {
  const WimgJob job{a.W, wimg, a.M, a.K};
  return ctn_pw_prepare_batch(&job, 1, math, a.act_scale != nullptr, st);
}

int ctn_pw_prepare_batch(const WimgJob* jobs, int n, int math, bool bounded, cudaStream_t st) {
  if (math == CTN_MATH_FP32) return CTN_OK;
  math = piece_math(math, bounded);
  bool uniform = true;
  for (int i = 0; i < n; ++i) uniform = uniform && eff_math(jobs[i].M, math) == math;
  if (uniform) return build_images(jobs, n, math, st);
  // f16x3 with some contraction past F16_MAX_ROWS (tf32 pieces): one launch per job, each in its own pieces
  for (int i = 0; i < n; ++i) CTN_TRY(build_images(jobs + i, 1, eff_math(jobs[i].M, math), st));
  return CTN_OK;
}

namespace {
__device__ const float k_one = 1.f;
}  // namespace

const float* ctn_device_one() {
  void* p = nullptr;
  if (cudaGetSymbolAddress(&p, k_one) != cudaSuccess) return nullptr;
  return (const float*)p;
}

int ctn_pw_run(const float* A, const float* W, const float* wimg, float* D, int B, int M, int K, int frames, int pitch, int math,
               const float* bias, const float* slope, double* stats, cudaStream_t st) {
  PwArgs a;
  memset(&a, 0, sizeof(a));
  a.A = A; a.W = W; a.D = D; a.B = B; a.M = M; a.K = K; a.frames = frames; a.pitch = pitch;
  a.wimg = wimg;
  if (bias) { a.bias = bias; a.slope = slope; a.stats_out = stats; }
  return ctn_pw(a, PRO_NONE, bias ? EPI_H : EPI_RAW, math, nullptr, st);
}

int ctn_pw_maskdec_supported(const PwArgs& a, int math) { return maskdec_ok(a, piece_math(math, a.act_scale != nullptr)); }

int ctn_pw(const PwArgs& a, int pro, int epi, int math, float* wimg_scratch, cudaStream_t st) {
  if (math == CTN_MATH_FP32) return ctn_pw_simt(a, pro, epi, st);
  const int pmath = piece_math(math, a.act_scale != nullptr);
  if (!wimg_scratch) return launch_wgmma(a, pro, epi, pmath, st);
  CTN_TRY(ctn_pw_prepare(a, math, wimg_scratch, st));
  PwArgs b = a;
  b.wimg = wimg_scratch;
  return launch_wgmma(b, pro, epi, pmath, st);
}
