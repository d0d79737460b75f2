// Raw PTX wrappers for the Hopper (sm_90a) features the tensor-core kernels use: mbarrier, 1-D bulk async copy (TMA
// engine), clusters / distributed shared memory, wgmma, proxy fences.  No CUTLASS dependency.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}" ::"r"(bar), "r"(parity) : "memory");
}

// named barrier ID (1..15; 0 is __syncthreads) over THREADS threads, e.g. the 128 of one warpgroup.  Immediate operands: with a
// register id ptxas reserves all 16 barriers of the CTA.
template <uint32_t ID, uint32_t THREADS>
__device__ __forceinline__ void named_bar_sync() {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(THREADS) : "memory");
}

// ---- async proxy -----------------------------------------------------------------------------------------------
// generic-proxy st.shared writes -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// 1-D bulk copy global -> shared, completion on an mbarrier (complete_tx::bytes).  size % 16 == 0, 16-byte aligned.
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// same, multicast to every CTA of the cluster whose bit is set in cta_mask (same CTA-relative dst / mbarrier offsets)
__device__ __forceinline__ void bulk_g2s_multicast(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(dst_smem),
      "l"(src), "r"(bytes), "r"(bar), "h"(cta_mask)
      : "memory");
}

// one lane of a converged warp (elect.sync): code under this predicate is known single-threaded to the compiler, so
// uniform-datapath instructions are emitted without per-instruction election loops
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .b32 rx;\n\t"
      ".reg .pred px;\n\t"
      "elect.sync rx|px, 0xFFFFFFFF;\n\t"
      "@px mov.s32 %0, 1;\n\t"
      "}"
      : "+r"(pred));
  return pred != 0;
}

// ---- clusters ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {  // every thread of every CTA in the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// arrive on the mbarrier at the same CTA-relative address in CTA `rank` of the cluster (release at cluster scope)
__device__ __forceinline__ void mbar_arrive_remote(uint32_t local_bar, uint32_t rank) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t"
      "}" ::"r"(local_bar), "r"(rank)
      : "memory");
}
// wait with acquire at CLUSTER scope (the arrivals may come from the peer CTA)
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}" ::"r"(bar), "r"(parity) : "memory");
}

// bulk copy from this CTA's shared memory into the SAME offsets of CTA `rank` of the cluster (distributed shared memory), completing
// on the mbarrier at `bar` (CTA-relative address) in that CTA: the transfer runs in the async proxy on both sides, so the
// receiver's wgmma may read the data right after its mbarrier wait.  16-byte aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_s2peer(uint32_t dst_smem, uint32_t src_smem, uint32_t bytes, uint32_t bar, uint32_t rank) {
  asm volatile(
      "{\n\t"
      ".reg .b32 rd, rb;\n\t"
      "mapa.shared::cluster.u32 rd, %0, %4;\n\t"
      "mapa.shared::cluster.u32 rb, %3, %4;\n\t"
      "cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [rd], [%1], %2, [rb];\n\t"
      "}" ::"r"(dst_smem), "r"(src_smem), "r"(bytes), "r"(bar), "r"(rank)
      : "memory");
}

// 16-byte store into the shared memory of CTA `rank` of the cluster, same CTA-relative address (generic proxy, DSMEM)
__device__ __forceinline__ void st_peer_v4(uint32_t local_addr, uint32_t rank, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "st.shared::cluster.v4.b32 [ra], {%2, %3, %4, %5};\n\t"
      "}" ::"r"(local_addr), "r"(rank), "r"(a), "r"(b), "r"(c), "r"(d)
      : "memory");
}

// ---- wgmma (Hopper warpgroup MMA) -----------------------------------------------------------------------------------
// D (64 x 128, fp32, registers of the 128 threads of a warpgroup) += A (64 x K, shared memory) * B (128 x K, shared memory)^T.
// B K-major; A K-major (tf32) or MN-major (f16).  Accumulator fragment of thread (warp w of the group, lane l), register i:
//   row = 16 w + l / 4 + 8 ((i / 2) % 2),  column = 8 (i / 4) + 2 (l % 4) + i % 2.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void wg_mma_tf32(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db));
}
// fp16: A is MN-major (imm-trans-a = 1, descriptor from wg_desc_mn128), B K-major
__device__ __forceinline__ void wg_mma_f16(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db));
}

// round-to-nearest fp32 -> tf32 (result is an fp32 bit pattern with the low 13 mantissa bits cleared)
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// cheap hi/lo split for the 3xTF32 scheme (3 instructions per element instead of two emulated cvt.rna):
//   hi = x rounded to nearest (ties away) at 10 explicit mantissa bits via integer add + mask; lo = x - hi is EXACT in
//   fp32 and the tensor core consumes its leading tf32 bits (remaining error <= 2^-21 |x|).
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
  lo = x - hi;
}

// fp16 hi/lo split of two fp32 values ("3xFP16"): hi = rn_f16(x) (saturating, never inf), lo = rn_f16(x - hi).
// Both pieces carry 11 significant bits like TF32; packed as f16x2 (element 0 in the low half).
__device__ __forceinline__ void split_f16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  float h0, h1;
  asm("{\n\t.reg .f16 a, b;\n\tmov.b32 {a, b}, %2;\n\tcvt.f32.f16 %0, a;\n\tcvt.f32.f16 %1, b;\n\t}" : "=f"(h0), "=f"(h1) : "r"(hi));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - h1), "f"(x0 - h0));
}

__device__ __forceinline__ float hi_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }

// ---- descriptors -------------------------------------------------------------------------------------------------
// sm_90 shared-memory matrix descriptor of a K-major operand in a swizzled canonical layout:
//   bits [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused by swizzled K-major layouts) |
//   [32,46) stride byte offset >> 4 = bytes between 8-row groups | [62,64) layout: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B.
// Rows are 128 B (SWIZZLE_128B: 16-byte chunk index XOR row % 8) or 64 B (SWIZZLE_64B: chunk index XOR (row / 2) % 4); the
// start address of the k-th 32-byte column step is base + 32 k.
constexpr uint32_t SW128 = 1u, SW64 = 2u;
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr, uint32_t sbo_bytes, uint32_t layout) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) | ((uint64_t)layout << 62);
}

// Descriptor of an MN-major 16-bit operand in the canonical SWIZZLE_128B layout, ((T,8,m),(8,k)) : ((1,T,LBO),(8T,SBO)) with
// T = 8 elements (PTX ISA, "Shared Memory Matrix Layout"): a 128-byte row holds 64 consecutive M (or N) elements of one k, 16-byte
// chunk index XOR (row % 8); 8 rows of consecutive k form a 1 KB atom.  LBO = bytes between atoms along M (the next 64 elements),
// SBO = bytes between atoms along K (the next 8 k).  The k-th 16-deep instruction step starts 2 atoms further on.
__device__ __forceinline__ uint64_t wg_desc_mn128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) |
         ((uint64_t)SW128 << 62);
}

}  // namespace ptx
