// Hopper (sm_90a) wgmma weight-gradient kernel of the 1x1 convolutions (training path):
//
//   dW[m][k] += sum_b sum_{t < frames} dY[b][m][t] * X[b][k][t]            dY: (B, M, pitch), X: (B, K, pitch)
//
// Both operands are reduced over TIME, which is the contiguous dimension of both tensors, so both are K-major wgmma
// operands in the canonical SWIZZLE_128B layout (rows of 32 time steps = 128 bytes): output channels m on the wgmma M
// dimension (two warpgroups of 64 rows), input channels k on N = 128, 32 time steps per pipeline stage (4 MMAs of K = 8).
// The reduction over B * frames (128 k at cfg2) is split across the CTAs of a tile ("split-K"): grid = tiles x splits
// ~ two CTAs per SM; every CTA accumulates its share of the time axis in registers and adds the tile to dW with fp32
// reductions at the end (dW must be zero on entry).
// fp32-parity numerics: the same 3xTF32 split as the forward kernels, applied to BOTH operands while staging
// (hi = x rounded to 10 mantissa bits, lo = x - hi exact; D += hi*hi + lo*hi + hi*lo, fp32 accumulate).
#include "ctn_internal.h"
#include "ctn_wgmma_ptx.cuh"
#include <stdlib.h>
#include <string.h>

namespace {

constexpr int WG_THREADS = 256;
constexpr int WG_KT = 32;              // time steps per stage
constexpr int WG_ROWS = 128;           // rows of each operand tile (m of dY, k of X)
constexpr uint32_t WG_A_BYTES = WG_ROWS * 128;  // 128 rows x 128 B per precision
constexpr int WG_HEADER = 1024;

struct WgArgs {
  const float* dy; size_t dy_bs;
  const float* x; size_t x_bs;
  float* dWa; float* dWb; int split_row;  // rows [0, split_row) -> dWa, rows [split_row, M) -> dWb (both (rows, K) row-major)
  int M, K, B, frames, pitch;
  int tiles_n, tiles, steps_per_split, chunks;
};

template <int NPASS>
__global__ void __launch_bounds__(WG_THREADS, 1) k_wgrad_wgmma(const WgArgs g) {
  constexpr int NPREC = NPASS == 3 ? 2 : 1;
  constexpr uint32_t STAGE_BYTES = 2u * NPREC * WG_A_BYTES;  // dY tile [hi, lo], X tile [hi, lo]
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  const uint32_t stage0 = base + WG_HEADER;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;

  const int tile = (int)blockIdx.x % g.tiles, split = (int)blockIdx.x / g.tiles;
  const int m0 = (tile / g.tiles_n) * WG_ROWS, n0 = (tile % g.tiles_n) * WG_ROWS;
  const long long total = (long long)g.B * g.chunks;
  const long long s0 = (long long)split * g.steps_per_split;
  const long long s1 = s0 + g.steps_per_split < total ? s0 + g.steps_per_split : total;
  const int nsteps = (int)(s1 - s0);
  if (nsteps <= 0) return;  // uniform over the CTA

  // staging: thread -> (row r = threadIdx / 8 + 32 i, 16-byte chunk ch = threadIdx % 8) of both operands, i < 4
  const int ch = threadIdx.x & 7, r0 = threadIdx.x >> 3;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  for (int it = 0; it < nsteps; ++it) {
    const int s = it & 1;
    const long long step = s0 + it;
    const int b = (int)(step / g.chunks), t = (int)(step % g.chunks) * WG_KT + ch * 4;
    uint8_t* st = smem + WG_HEADER + (size_t)s * STAGE_BYTES;
#pragma unroll
    for (int op = 0; op < 2; ++op) {
      const float* src = op == 0 ? g.dy + (size_t)b * g.dy_bs + (size_t)m0 * g.pitch : g.x + (size_t)b * g.x_bs + (size_t)n0 * g.pitch;
      const int lim = op == 0 ? g.M - m0 : g.K - n0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = r0 + 32 * i;
        float4 x = r < lim ? __ldg(reinterpret_cast<const float4*>(src + (size_t)r * g.pitch + t)) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (t + 0 >= g.frames) x.x = 0.f;  // pad columns never contribute (last chunk of a sample only)
        if (t + 1 >= g.frames) x.y = 0.f;
        if (t + 2 >= g.frames) x.z = 0.f;
        if (t + 3 >= g.frames) x.w = 0.f;
        float4 hi, lo;
        hi.x = ptx::hi_tf32(x.x); hi.y = ptx::hi_tf32(x.y); hi.z = ptx::hi_tf32(x.z); hi.w = ptx::hi_tf32(x.w);
        const uint32_t off = (uint32_t)op * NPREC * WG_A_BYTES + (uint32_t)r * 128u + (((uint32_t)ch ^ (uint32_t)(r & 7)) << 4);
        *reinterpret_cast<float4*>(st + off) = hi;
        if (NPASS == 3) {
          lo.x = x.x - hi.x; lo.y = x.y - hi.y; lo.z = x.z - hi.z; lo.w = x.w - hi.w;
          *reinterpret_cast<float4*>(st + off + WG_A_BYTES) = lo;  // the lo plane of an operand sits right behind its hi plane
        }
      }
    }
    ptx::fence_proxy_async_smem();
    __syncthreads();
    const uint32_t sb = stage0 + (uint32_t)s * STAGE_BYTES;
    const uint32_t a_hi = sb + (uint32_t)wg * 64u * 128u, a_lo = a_hi + WG_A_BYTES;
    const uint32_t b_hi = sb + NPREC * WG_A_BYTES, b_lo = b_hi + WG_A_BYTES;
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < WG_KT / 8; ++kk) {
      const uint64_t dah = ptx::wg_desc(a_hi + kk * 32, 1024u, ptx::SW128), dbh = ptx::wg_desc(b_hi + kk * 32, 1024u, ptx::SW128);
      ptx::wg_mma_tf32(acc, dah, dbh);
      if (NPASS == 3) {
        ptx::wg_mma_tf32(acc, ptx::wg_desc(a_lo + kk * 32, 1024u, ptx::SW128), dbh);
        ptx::wg_mma_tf32(acc, dah, ptx::wg_desc(b_lo + kk * 32, 1024u, ptx::SW128));
      }
    }
    ptx::wg_commit();
    ptx::wg_wait<1>();  // the MMAs of step it - 1 are done: its stage may be refilled
    __syncthreads();
  }
  ptx::wg_wait<0>();

  const int row0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int m = row0 + 8 * ((i >> 1) & 1);
    const int n = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    if (m >= g.M || n >= g.K) continue;
    float* row = m < g.split_row ? g.dWa + (size_t)m * g.K : g.dWb + (size_t)(m - g.split_row) * g.K;
    atomicAdd(row + n, acc[i]);
  }
}

int g_sms[CTN_MAX_DEVICES] = {0};  // per device ordinal
int sms() {
  const int dev = ctn_current_device();
  if (g_sms[dev] == 0) {
    cudaDeviceGetAttribute(&g_sms[dev], cudaDevAttrMultiProcessorCount, dev);
    if (g_sms[dev] <= 0) g_sms[dev] = 132;
  }
  return g_sms[dev];
}

template <int NPASS>
int launch_wg(const WgArgs& g, int grid, cudaStream_t st) {
  constexpr int NPREC = NPASS == 3 ? 2 : 1;
  constexpr size_t smem = WG_HEADER + 1024 + 2 * 2 * NPREC * (size_t)WG_A_BYTES;
  static bool attr_done[CTN_MAX_DEVICES] = {false};  // the opt-in is per device (context)
  const int dev = ctn_current_device();
  if (!attr_done[dev]) {
    cudaError_t e = cudaFuncSetAttribute(k_wgrad_wgmma<NPASS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done[dev] = true;
  }
  k_wgrad_wgmma<NPASS><<<grid, WG_THREADS, smem, st>>>(g);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

}  // namespace

// rows [0, split_row) of the (M, K) result go to dWa, the rest to dWb (pass split_row = M and dWb = nullptr for one tensor)
int ctn_wgrad_wgmma(const float* dy, size_t dy_bs, const float* x, size_t x_bs, float* dWa, float* dWb, int split_row, int M,
                    int K, int B, int frames, int pitch, int math, cudaStream_t st) {
  if (!dy || !x || !dWa || M <= 0 || K <= 0 || B <= 0 || frames <= 0) return CTN_EINVAL;
  if (pitch % 128 != 0 || (dy_bs % 4) != 0 || (x_bs % 4) != 0) return CTN_EALIGN;
  if ((((uintptr_t)dy) | ((uintptr_t)x)) & 15) return CTN_EALIGN;
  WgArgs g;
  memset(&g, 0, sizeof(g));
  g.dy = dy; g.dy_bs = dy_bs; g.x = x; g.x_bs = x_bs; g.dWa = dWa; g.dWb = dWb; g.split_row = dWb ? split_row : M;
  g.M = M; g.K = K; g.B = B; g.frames = frames; g.pitch = pitch;
  g.tiles_n = (K + WG_ROWS - 1) / WG_ROWS;
  g.tiles = ((M + WG_ROWS - 1) / WG_ROWS) * g.tiles_n;
  g.chunks = (frames + WG_KT - 1) / WG_KT;
  const long long total = (long long)B * g.chunks;
  long long splits = 2LL * sms() / g.tiles;
  if (splits < 1) splits = 1;
  if (splits > total) splits = total;
  g.steps_per_split = (int)((total + splits - 1) / splits);
  splits = (total + g.steps_per_split - 1) / g.steps_per_split;
  const int grid = g.tiles * (int)splits;
  // F16X3 forwards use the 3xTF32 weight-gradient kernel
  return math == CTN_MATH_TF32 ? launch_wg<1>(g, grid, st) : launch_wg<3>(g, grid, st);
}
