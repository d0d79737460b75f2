// Bidirectional LSTM recurrence + output projection of a dual-path block (BASELINE cfg4) on Hopper wgmma.
// Reference: src/models/dprnn.py:82-90 / 134-142 (x -> nn.LSTM(bidirectional, batch_first) -> nn.Linear(2H, F)); the recurrence
// itself is torch.nn.LSTM: gates (i, f, g, o) = W_ih x_t + b_ih + W_hh h_{t-1} + b_hh, c_t = f c_{t-1} + i g, h_t = o tanh(c_t).
//
// One CTA (one warpgroup) = 64 sequences of ONE direction, all T steps.  Per step the pre-activations are ONE contraction
//   [x_t | h_{t-1}] (64 x (F + H))  x  [W_ih | W_hh]^T ((F + H) x 4H)
// run as 3xTF32 (hi/lo pieces, fp32 accumulate in registers; no operand scaling needed).  Gate columns are reordered unit-major (the
// 4 gates of a hidden unit adjacent) and cut into chunks of 32 units = 128 columns (wgmma N = 128), so that a chunk's accumulator
// holds whole units: the cell update runs on the fragment after one lane-pair exchange, with c_t in registers.
//   * [x_t | h_{t-1}]: K-major SWIZZLE_128B shared-memory slabs of 32 channels (hi + lo), rewritten every step;
//   * weights: pre-split / pre-swizzled 32 KB slab images (128 columns x 32 k, hi + lo), streamed from L2 through a ring of
//     shared-memory stages by 1-D bulk async copies on mbarriers (the whole set is larger than an SM's shared memory);
//   * the 2H -> F projection of the block (nn.Linear after the LSTM) rides along: per step one more contraction h_t x
//     W_fc[:, dir*H:(dir+1)*H]^T on the freshly written h slabs; each direction stores its partial projection (NSEQ, T, F) and the
//     gLN + residual kernel adds the two and the bias, so the (NSEQ, T, 2H) LSTM output is only materialised on request.
#include "ctn_internal.h"
#include "ctn_wgmma_ptx.cuh"

namespace {

constexpr int LSEQ = 64;              // sequences per CTA (wgmma M)
constexpr int LTHREADS = 128;         // one warpgroup
constexpr uint32_t SLAB = 32768;      // weight slab image: [hi 128 rows x 128 B][lo 128 rows x 128 B]
constexpr uint32_t ASLAB = 16384;     // operand slab: [hi 64 rows x 128 B][lo 64 rows x 128 B]
constexpr int MAX_NST = 4;
constexpr int SMEM_LIMIT = 232448;

struct LstmArgs {
  const float* z;        // (NSEQ, T, F)
  float* P;              // (2, NSEQ, T, Fo) or null
  float* hout;           // (NSEQ, T, 2H) or null
  const uint8_t* img;    // [2][per_step][SLAB]
  const float* bias;     // [2][4H] b_ih + b_hh, unit-major column order
  int NSEQ, T, Fo, per_step, nst;
};

__host__ __device__ inline int lstm_per_step(int F, int H, bool proj) { return (H / 32) * (F / 32 + H / 32) + (proj ? H / 32 : 0); }

__device__ __forceinline__ float sigmoid_(float a) { return 1.f / (1.f + expf(-a)); }

// float offset of element (row, k) in a K-major SWIZZLE_128B plane of 32-element rows
__device__ __forceinline__ int sw128(int row, int k) { return (row >> 3) * 256 + (row & 7) * 32 + ((((k >> 2) ^ (row & 7)) << 2) | (k & 3)); }

struct LstmWeights { const float* w[8]; };  // weight_ih, weight_hh, bias_ih, bias_hh, then the _reverse set

// grid (per_step, 2 directions), block 256: slab `sl` of a direction's image; bias in unit-major order
__global__ void __launch_bounds__(256) k_lstm_build(const LstmWeights wp, const float* __restrict__ w_fc, int F, int H, int Fo,
                                                    int per_step, uint8_t* __restrict__ img, float* __restrict__ bias) {
  const int sl = blockIdx.x, dir = blockIdx.y, NCH = H / 32, KT = F / 32 + H / 32;
  const float* wih = wp.w[4 * dir];
  const float* whh = wp.w[4 * dir + 1];
  float* dst = reinterpret_cast<float*>(img + ((size_t)dir * per_step + sl) * SLAB);
  for (int i = threadIdx.x; i < 128 * 32; i += 256) {
    const int nl = i >> 5, kl = i & 31;
    float v;
    if (sl < NCH * KT) {
      const int c = sl / KT, kk = sl % KT, u = c * 32 + (nl >> 2), row = (nl & 3) * H + u, k = kk * 32 + kl;
      v = k < F ? wih[(size_t)row * F + k] : whh[(size_t)row * H + (k - F)];
    } else {
      const int kk = sl - NCH * KT;
      v = nl < Fo ? w_fc[(size_t)nl * 2 * H + dir * H + kk * 32 + kl] : 0.f;
    }
    const float hi = ptx::to_tf32(v);
    dst[sw128(nl, kl)] = hi;
    dst[4096 + sw128(nl, kl)] = ptx::to_tf32(v - hi);
  }
  if (sl == 0)
    for (int n = threadIdx.x; n < 4 * H; n += 256) {
      const int u = n >> 2, gi = n & 3;
      bias[dir * 4 * H + n] = wp.w[4 * dir + 2][gi * H + u] + wp.w[4 * dir + 3][gi * H + u];
    }
}

// stores rows x 32-channel slab pieces: v (4 consecutive channels 4 c4 .. 4 c4 + 3 of one row) -> hi / lo planes of slab c4 / 8
__device__ __forceinline__ void put4(uint8_t* a_slabs, int slab0, int row, int c4, float4 v) {
  float* base = reinterpret_cast<float*>(a_slabs + (size_t)(slab0 + (c4 >> 3)) * ASLAB);
  const int off = sw128(row, (c4 & 7) * 4);
  float4 hi, lo;
  hi.x = ptx::hi_tf32(v.x); hi.y = ptx::hi_tf32(v.y); hi.z = ptx::hi_tf32(v.z); hi.w = ptx::hi_tf32(v.w);
  lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
  *reinterpret_cast<float4*>(base + off) = hi;
  *reinterpret_cast<float4*>(base + 2048 + off) = lo;
}

// 64 x 128 += A slab (hi/lo at a_addr) x weight slab (hi/lo at w_addr), 3xTF32
__device__ __forceinline__ void mma_slab(float (&acc)[64], uint32_t a_addr, uint32_t w_addr) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t dah = ptx::wg_desc(a_addr + kk * 32, 1024u, ptx::SW128), dal = ptx::wg_desc(a_addr + 8192 + kk * 32, 1024u, ptx::SW128);
    const uint64_t dwh = ptx::wg_desc(w_addr + kk * 32, 1024u, ptx::SW128), dwl = ptx::wg_desc(w_addr + 16384 + kk * 32, 1024u, ptx::SW128);
    ptx::wg_mma_tf32(acc, dah, dwh);
    ptx::wg_mma_tf32(acc, dal, dwh);
    ptx::wg_mma_tf32(acc, dah, dwl);
  }
}

// NCH = H / 32 gate chunks, KSX = F / 32 input slabs.  RELU_PROJ: the projection sees ReLU(h_t) (DPTNet's FeedForwardBlock,
// dptnet.py:560-562), the recurrence and hout the raw h_t
template <int NCH, int KSX, bool RELU_PROJ = false>
__global__ void __launch_bounds__(LTHREADS, 1) k_bilstm(const LstmArgs g) {
  constexpr int H = NCH * 32, F = KSX * 32, KT = KSX + NCH;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint8_t* a_slabs = smem + 1024;                                    // KT operand slabs
  float* hs = reinterpret_cast<float*>(a_slabs + KT * ASLAB);        // h_t, [64][H]
  const uint32_t a_addr = base + 1024, ring = base + 1024 + KT * ASLAB + LSEQ * H * 4;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q = lane & 3, p = q & 1;
  const int dir = blockIdx.y, seq0 = blockIdx.x * LSEQ;
  const uint8_t* img = g.img + (size_t)dir * g.per_step * SLAB;
  const float* bias = g.bias + dir * 4 * H;
  const long long total = (long long)g.T * g.per_step;
  if (tid == 0) {
    for (int s = 0; s < g.nst; ++s) ptx::mbar_init(ptx::smem_u32(&full[s]), 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  auto issue = [&](long long gs) {  // bulk copy of the gs-th slab of the whole call into its ring stage
    const int s = (int)(gs % g.nst);
    const uint32_t fb = ptx::smem_u32(&full[s]);
    ptx::mbar_arrive_expect_tx(fb, SLAB);
    ptx::bulk_g2s(ring + (uint32_t)s * SLAB, img + (size_t)(gs % g.per_step) * SLAB, SLAB, fb);
  };
  if (tid == 0)
    for (int s = 0; s < g.nst && s < total; ++s) issue(s);
  long long gs = 0;
  auto consume = [&](float (&acc)[64], int a_slab) {
    const int s = (int)(gs % g.nst);
    ptx::mbar_wait(ptx::smem_u32(&full[s]), (uint32_t)((gs / g.nst) & 1));
    ptx::wg_fence();
    mma_slab(acc, a_addr + (uint32_t)a_slab * ASLAB, ring + (uint32_t)s * SLAB);
    ptx::wg_commit();
    ptx::wg_wait<0>();
    __syncthreads();  // every warp's MMAs have read the stage
    if (tid == 0 && gs + g.nst < total) issue(gs + g.nst);
    ++gs;
  };
  // h_0 = 0
  for (int i = tid; i < NCH * ASLAB / 4; i += LTHREADS) reinterpret_cast<float*>(a_slabs + KSX * ASLAB)[i] = 0.f;
  float cst[NCH][16];
#pragma unroll
  for (int c = 0; c < NCH; ++c)
#pragma unroll
    for (int j = 0; j < 16; ++j) cst[c][j] = 0.f;
  const int r0 = warp * 16 + (lane >> 2);  // fragment rows r0, r0 + 8
  const int my_row = r0 + 8 * p, my_seq = seq0 + my_row;

  for (int step = 0; step < g.T; ++step) {
    const int t = dir == 0 ? step : g.T - 1 - step;
    for (int i = tid; i < LSEQ * F / 4; i += LTHREADS) {
      const int row = i / (F / 4), c4 = i % (F / 4), seq = seq0 + row;
      const float4 v = seq < g.NSEQ ? __ldg(reinterpret_cast<const float4*>(g.z + ((size_t)seq * g.T + t) * F) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      put4(a_slabs, 0, row, c4, v);
    }
    ptx::fence_proxy_async_smem();
    __syncthreads();
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      for (int kk = 0; kk < KT; ++kk) consume(acc, kk);
      // register i = 4 j + 2 hh + e: row r0 + 8 hh, column 8 j + 2 q + e = gate (2 (q & 1) + e) of unit 2 j + q / 2.  Lane pairs
      // (q, q ^ 1) swap halves: lane p = q & 1 ends up with all four gates of unit 2 j + q / 2 for row r0 + 8 p.
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int cb = c * 128 + 8 * j + 2 * q;
        const float b0 = __ldg(bias + cb), b1 = __ldg(bias + cb + 1);
        const float a0 = acc[4 * j] + b0, a1 = acc[4 * j + 1] + b1, a2 = acc[4 * j + 2] + b0, a3 = acc[4 * j + 3] + b1;
        const float s0 = p ? a0 : a2, s1 = p ? a1 : a3;
        const float r0v = __shfl_xor_sync(0xffffffffu, s0, 1), r1v = __shfl_xor_sync(0xffffffffu, s1, 1);
        const float gi = p ? r0v : a0, gf = p ? r1v : a1, gg = p ? a2 : r0v, go = p ? a3 : r1v;
        const float cc = fmaf(sigmoid_(gf), cst[c][j], sigmoid_(gi) * tanhf(gg));
        cst[c][j] = cc;
        const float h = sigmoid_(go) * tanhf(cc);
        const int u = c * 32 + 2 * j + (q >> 1);
        hs[my_row * H + u] = h;
        if (g.hout && my_seq < g.NSEQ) g.hout[((size_t)my_seq * g.T + t) * 2 * H + dir * H + u] = h;
      }
    }
    __syncthreads();
    for (int i = tid; i < LSEQ * H / 4; i += LTHREADS) {
      const int row = i / (H / 4), c4 = i % (H / 4);
      float4 v = *reinterpret_cast<const float4*>(hs + row * H + 4 * c4);
      if (RELU_PROJ) v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
      put4(a_slabs, KSX, row, c4, v);
    }
    ptx::fence_proxy_async_smem();
    __syncthreads();
    if (g.P) {
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      for (int kk = 0; kk < NCH; ++kk) consume(acc, KSX + kk);
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int row = r0 + 8 * ((i >> 1) & 1), o = 8 * (i >> 2) + 2 * q + (i & 1), seq = seq0 + row;
        if (o < g.Fo && seq < g.NSEQ) g.P[(((size_t)dir * g.NSEQ + seq) * g.T + t) * g.Fo + o] = acc[i];
      }
    }
    if (RELU_PROJ)  // the next step's gates read the raw h_t: every MMA on the slabs has completed (consume waits and syncs), and
                    // the next step's operand fence + barrier orders these stores before them
      for (int i = tid; i < LSEQ * H / 4; i += LTHREADS) {
        const int row = i / (H / 4), c4 = i % (H / 4);
        put4(a_slabs, KSX, row, c4, *reinterpret_cast<const float4*>(hs + row * H + 4 * c4));
      }
  }
}

template <int NCH, int KSX, bool RELU_PROJ>
int launch_bilstm(const LstmArgs& a, size_t smem, cudaStream_t st) {
  static bool done[CTN_MAX_DEVICES] = {};
  const int dev = ctn_current_device();
  if (!done[dev]) {
    cudaError_t e = cudaFuncSetAttribute(k_bilstm<NCH, KSX, RELU_PROJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) return (int)e;
    done[dev] = true;
  }
  k_bilstm<NCH, KSX, RELU_PROJ><<<dim3((a.NSEQ + LSEQ - 1) / LSEQ, 2), LTHREADS, smem, st>>>(a);
  return CTN_OK;
}

// Y = P0 + P1 + bias (the Linear of dprnn.py:87 / 139 split over the two directions): gLN statistics of it ...
// Every element goes into double before it is added (as k_sample_part of ctn_dptnet.cu): fp32 runs of 16 values lose the
// variance under a DC offset far above the spread (DESIGN 19 gives the rows that failed on an H100 before this).
__global__ void __launch_bounds__(256) k_sample_stats2(const float* __restrict__ P0, const float* __restrict__ P1,
                                                       const float* __restrict__ bias, size_t n, int F, double* __restrict__ stats) {
  __shared__ double red[64];
  const int b = blockIdx.y;
  const float4* p0 = reinterpret_cast<const float4*>(P0 + (size_t)b * n);
  const float4* p1 = reinterpret_cast<const float4*>(P1 + (size_t)b * n);
  const size_t n4 = n / 4;  // F % 4 == 0
  double s = 0.0, ss = 0.0;
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x * 4; i0 < n4; i0 += (size_t)gridDim.x * blockDim.x * 4) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const size_t i = i0 + (size_t)u * blockDim.x + threadIdx.x;
      if (i < n4) {
        const float4 a = __ldg(p0 + i), c = __ldg(p1 + i), bb = __ldg(reinterpret_cast<const float4*>(bias + (i * 4) % F));
        const double x = a.x + c.x + bb.x, y = a.y + c.y + bb.y, z = a.z + c.z + bb.z, w = a.w + c.w + bb.w;
        s += (x + y) + (z + w);
        ss = fma(x, x, fma(y, y, fma(z, z, fma(w, w, ss))));
      }
    }
  }
  block_sum2_d(s, ss, red);
  if (threadIdx.x == 0) { atomicAdd(&stats[2 * b], s); atomicAdd(&stats[2 * b + 1], ss); }
}

// ... and out = gLN(Y) + R, optionally stored with the two middle dimensions swapped (the layout of the other path).
// grid (D1, B), block (F/4, 256/(F/4)): one block per (b, d1) row of D2 x F floats (contiguous on the read side: a warp reads 512
// consecutive bytes of each operand); 4 independent cells per thread in flight; on the swapped side every cell is one 4F-byte run.
__global__ void __launch_bounds__(256) k_norm_res2(const float* __restrict__ P0, const float* __restrict__ P1, const float* __restrict__ bias,
                                                   const float* __restrict__ R, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, float* __restrict__ out, const double* __restrict__ stats,
                                                   int D1, int D2, int F, float eps, int swap, unsigned* __restrict__ absmax) {
  const int b = blockIdx.y, d1 = blockIdx.x, f = threadIdx.x * 4;
  float amax = 0.f;
  const float2 mr = gln_mean_rstd(stats + 2 * b, (double)D1 * (double)D2 * (double)F, eps);
  const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + f)), gm = __ldg(reinterpret_cast<const float4*>(gamma + f)),
               be = __ldg(reinterpret_cast<const float4*>(beta + f));
  // y_norm = (p0 + p1 + bias - mean) * rstd * gamma + beta  ==  (p0 + p1) * sc + sh
  const float4 sc = make_float4(mr.y * gm.x, mr.y * gm.y, mr.y * gm.z, mr.y * gm.w);
  const float4 sh = make_float4(fmaf(bb.x - mr.x, sc.x, be.x), fmaf(bb.y - mr.x, sc.y, be.y), fmaf(bb.z - mr.x, sc.z, be.z),
                                fmaf(bb.w - mr.x, sc.w, be.w));
  const size_t row = ((size_t)b * D1 + d1) * D2;
  const int TY = blockDim.y;
  for (int d20 = threadIdx.y; d20 < D2; d20 += 4 * TY) {
    float4 a[4], c[4], r[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int d2 = d20 + u * TY;
      if (d2 < D2) {
        const size_t src = (row + d2) * F + f;
        a[u] = __ldg(reinterpret_cast<const float4*>(P0 + src));
        c[u] = __ldg(reinterpret_cast<const float4*>(P1 + src));
        r[u] = __ldg(reinterpret_cast<const float4*>(R + src));
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int d2 = d20 + u * TY;
      if (d2 < D2) {
        const size_t dst = (swap ? ((size_t)b * D2 + d2) * D1 + d1 : row + d2) * F + f;
        float4 o;
        o.x = fmaf(a[u].x + c[u].x, sc.x, sh.x) + r[u].x;
        o.y = fmaf(a[u].y + c[u].y, sc.y, sh.y) + r[u].y;
        o.z = fmaf(a[u].z + c[u].z, sc.z, sh.z) + r[u].z;
        o.w = fmaf(a[u].w + c[u].w, sc.w, sh.w) + r[u].w;
        *reinterpret_cast<float4*>(out + dst) = o;
        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
      }
    }
  }
  if (absmax) {  // max|out|: the operand scale of the next path's LSTM (saves its own pass over the state)
    // (F/4) x TY need not be a multiple of 32 (F = 12, 48, 96, ...): the last warp is then partial and the reduction names only
    // its existing lanes.  amax >= 0, so the float order is the order of its bit patterns.
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, left = blockDim.x * blockDim.y - (tid & ~31);
    const unsigned m = __reduce_max_sync(left >= 32 ? 0xffffffffu : (1u << left) - 1u, __float_as_uint(amax));
    if ((tid & 31) == 0 && m != 0u) atomicMax(absmax, m);
  }
}


bool lstm_supported(int F, int H, int Fo) {
  if (!(H == 32 || H == 64 || H == 128) || !(F == 32 || F == 64 || F == 128)) return false;
  return Fo == 0 || (Fo % 32 == 0 && Fo >= 32 && Fo <= 128);
}
size_t lstm_fixed_smem(int F, int H) { return 2048 + (size_t)(F / 32 + H / 32) * ASLAB + (size_t)LSEQ * H * 4; }
size_t lstm_ws_bytes(int F, int H, int Fo) { return 256 + (size_t)2 * 4 * H * 4 + (size_t)2 * lstm_per_step(F, H, Fo > 0) * SLAB; }

}  // namespace

extern "C" int ctn_bilstm_supported(int F, int H, int Fo) { return lstm_supported(F, H, Fo) ? 1 : 0; }

extern "C" size_t ctn_bilstm_workspace_bytes(int F, int H, int Fo) { return lstm_supported(F, H, Fo) ? lstm_ws_bytes(F, H, Fo) : 0; }

namespace {
int bilstm_proj(const float* z, int NSEQ, int T, int F, int H, const float* const* w, const float* w_fc, int Fo, float* P, float* hout,
                bool relu_proj, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (!z || !w || !workspace || NSEQ <= 0 || T <= 0) return CTN_EINVAL;
  if (relu_proj && !w_fc) return CTN_EINVAL;
  for (int i = 0; i < 8; ++i)
    if (!w[i]) return CTN_EINVAL;
  if ((w_fc == nullptr) != (P == nullptr)) return CTN_EINVAL;
  if (!w_fc && !hout) return CTN_EINVAL;
  const int Fp = w_fc ? Fo : 0;
  // Fo = 0 names the envelope without a projection: with w_fc the image would hold projection slabs the workspace size omits
  if (!lstm_supported(F, H, Fp) || (w_fc && Fp == 0)) return CTN_EUNSUPPORTED;
  if (workspace_bytes < lstm_ws_bytes(F, H, Fp)) return CTN_EWORKSPACE;
  if ((((uintptr_t)z) | ((uintptr_t)P) | ((uintptr_t)hout) | ((uintptr_t)workspace)) & 15) return CTN_EALIGN;
  const size_t fixed = lstm_fixed_smem(F, H);
  int nst = (int)((SMEM_LIMIT - fixed) / SLAB);
  if (nst > MAX_NST) nst = MAX_NST;
  if (nst < 2) return CTN_EUNSUPPORTED;
  cudaStream_t st = stream;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  LstmWeights wts;
  for (int i = 0; i < 8; ++i) wts.w[i] = w[i];
  float* bias = reinterpret_cast<float*>(ws + 256);
  uint8_t* img = ws + 256 + (size_t)2 * 4 * H * 4;
  LstmArgs a;
  a.z = z; a.P = P; a.hout = hout; a.img = img; a.bias = bias;
  a.NSEQ = NSEQ; a.T = T; a.Fo = Fp; a.per_step = lstm_per_step(F, H, w_fc != nullptr); a.nst = nst;
  k_lstm_build<<<dim3(a.per_step, 2), 256, 0, st>>>(wts, w_fc, F, H, Fp, a.per_step, img, bias);
  CTN_COUNT_LAUNCH();
  const size_t smem = fixed + (size_t)nst * SLAB;
  int rc = CTN_EUNSUPPORTED;
  const int NCH = H / 32, KSX = F / 32;
#define CTN_LSTM_CASE(nch, ksx)                                                                       \
  if (NCH == nch && KSX == ksx)                                                                       \
    rc = relu_proj ? launch_bilstm<nch, ksx, true>(a, smem, st) : launch_bilstm<nch, ksx, false>(a, smem, st);
  CTN_LSTM_CASE(1, 1) CTN_LSTM_CASE(1, 2) CTN_LSTM_CASE(1, 4) CTN_LSTM_CASE(2, 1) CTN_LSTM_CASE(2, 2) CTN_LSTM_CASE(2, 4)
  CTN_LSTM_CASE(4, 1) CTN_LSTM_CASE(4, 2) CTN_LSTM_CASE(4, 4)
#undef CTN_LSTM_CASE
  if (rc != CTN_OK) return rc;
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
}  // namespace

extern "C" int ctn_bilstm_proj_fwd(const float* z, int NSEQ, int T, int F, int H, const float* const* w, const float* w_fc, int Fo, float* P,
                                   float* hout, const unsigned* z_absmax, void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(z);
  (void)z_absmax;  // 3xTF32 pieces keep fp32's exponent range: the recurrence needs no operand scale
  return bilstm_proj(z, NSEQ, T, F, H, w, w_fc, Fo, P, hout, false, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int ctn_bilstm_relu_proj_fwd(const float* z, int NSEQ, int T, int F, int H, const float* const* w, const float* w_fc, int Fo,
                                        float* P, float* hout, void* workspace, size_t workspace_bytes, ctn_stream_t stream) {
  LaunchScope scope(z);
  return bilstm_proj(z, NSEQ, T, F, H, w, w_fc, Fo, P, hout, true, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int ctn_dprnn_norm_res2_fwd(const float* P, const float* fc_bias, const float* R, const float* gamma, const float* beta,
                                       float* out, int B, int D1, int D2, int F, float eps, int swap, double* scratch, unsigned* out_absmax,
                                       ctn_stream_t stream) {
  LaunchScope scope(P);
  if (!P || !fc_bias || !R || !gamma || !beta || !out || !scratch || B <= 0 || D1 <= 0 || D2 <= 0 || F <= 0 || (F & 3)) return CTN_EINVAL;
  if (F > 1024 || D1 > 65535 * 32 || B > 65535) return CTN_EUNSUPPORTED;
  if (swap && out == R) return CTN_EINVAL;
  if ((((uintptr_t)P) | ((uintptr_t)R) | ((uintptr_t)out) | ((uintptr_t)gamma) | ((uintptr_t)beta) | ((uintptr_t)fc_bias)) & 15)
    return CTN_EALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * B, st);
  if (e != cudaSuccess) return (int)e;
  if (out_absmax && (e = cudaMemsetAsync(out_absmax, 0, sizeof(unsigned), st)) != cudaSuccess) return (int)e;
  const size_t n = (size_t)D1 * D2 * F;
  const float* P1 = P + (size_t)B * n;  // second direction
  int gx = (int)((n / 4 + 256 * 4 - 1) / (256 * 4));
  {  // ~8 resident blocks per SM over the WHOLE batch: longer per-thread streams, 2 double atomics per block on 2B addresses
    const int cap = 1184 / B > 1 ? 1184 / B : 1;
    if (gx > cap) gx = cap;
  }
  if (gx < 1) gx = 1;
  k_sample_stats2<<<dim3(gx, B), 256, 0, st>>>(P, P1, fc_bias, n, F, scratch);
  CTN_COUNT_LAUNCH();
  const int q = F / 4;
  k_norm_res2<<<dim3(D1, B), dim3(q, 256 / q >= 1 ? 256 / q : 1), 0, st>>>(P, P1, fc_bias, R, gamma, beta, out, scratch, D1, D2, F, eps, swap, out_absmax);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
