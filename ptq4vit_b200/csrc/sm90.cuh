// Hopper (sm_90a) primitives of the wgmma kernels: shared-memory addresses, mbarriers, bulk copies, proxy fences,
// the K-major operand descriptor and the wgmma instructions.  Included by sweep_tc.cu, gram_gemm.cu and the three
// frozen-forward kernels (forward_tc.cu, forward_mm_tc.cu, forward_attn_tc.cu).
//
// Everything is __forceinline__ and makes no call: ptxas ignores setmaxnreg in a kernel that contains a call (C7507,
// the sweep kernel relies on it), and a call between wgmmas splits their pipeline (C7510).
// Everything sits in an anonymous namespace, so each translation unit has its own copy of the timeout word: the library
// links separately compiled objects without -rdc, where a non-static __device__ variable defined in a header would give
// every object the same host shadow symbol.
#pragma once
#include <stdint.h>
#include <cstdio>

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarriers ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(void* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// Makes the barrier initialisation visible to the async proxy (bulk copies) before the block barrier that follows it.
__device__ __forceinline__ void fence_mbarrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx_addr(uint32_t addr, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(addr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void* bar, uint32_t bytes) { mbar_expect_tx_addr(smem_u32(bar), bytes); }
__device__ __forceinline__ void mbar_arrive(void* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t addr, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\t"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
               "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped launch (cudaErrorLaunchFailure), never as a hung GPU.  The bound
// is ~10 s of SM clocks: clock64 keeps counting while a context is time-sliced, a legitimate wait of a sub-millisecond
// kernel must never reach it.  The wait is inline and makes no call (see above).  On timeout it leaves
// (block << 32 | thread << 20 | barrier smem address) in g_mbar_timeout for a debugger-free post-mortem; building with
// -DP4V_SWEEP_DEBUG_PRINTF also prints it.  The failing launch identifies the kernel.
__device__ unsigned long long g_mbar_timeout;
[[noreturn]] __device__ __forceinline__ void mbar_timeout(uint32_t addr, uint32_t parity) {
  g_mbar_timeout = ((unsigned long long)blockIdx.x << 32) | ((unsigned long long)threadIdx.x << 20) | (addr & 0xFFFFFu);
  __threadfence();
#ifdef P4V_SWEEP_DEBUG_PRINTF
  printf("ptq4vit: mbarrier wait timed out (block %d thread %d smem 0x%x parity %u)\n",
         (int)blockIdx.x, (int)threadIdx.x, addr, parity);
#endif
  __trap();
  while (true) {}
}
__device__ __forceinline__ void mbar_wait_slow(uint32_t addr, uint32_t parity) {
  const long long t0 = clock64();
  while (!mbar_try(addr, parity))
    if (clock64() - t0 > 20000000000ll) mbar_timeout(addr, parity);
}
__device__ __forceinline__ void mbar_wait_addr(uint32_t addr, uint32_t parity) {
  if (!mbar_try(addr, parity)) mbar_wait_slow(addr, parity);
}
__device__ __forceinline__ void mbar_wait(void* bar, uint32_t parity) { mbar_wait_addr(smem_u32(bar), parity); }

// ---- bulk copies -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bulk_g2s_addr(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, void* bar) {
  bulk_g2s_addr(dst, src, bytes, smem_u32(bar));
}
// Warp-uniform single-lane election for the bulk copies.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// One warp's arrival (barrier count = arriving warps) once all its lanes are past the point being signalled.
__device__ __forceinline__ void warp_arrive(void* bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}
// Orders this thread's generic-proxy shared-memory stores before later async-proxy (wgmma, bulk copy) accesses; issued
// by every writing thread before the block barrier that hands the data over.
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma -------------------------------------------------------------------------------------------------------
// K-major, no swizzle (the canonical layout of common.cuh, [16-byte K chunk][rows][16 B]): core matrix = 8 rows x 16 B;
// LBO = stride between the 16-byte chunks of K (rows x 16 B), SBO = stride between 8-row groups (128 B).  desc_const
// holds the constant fields only, for loops that OR a precomputed 14-bit start address (bits 0..13, units of 16 B) into
// it; make_desc is the whole descriptor of a shared-memory address.
__device__ __forceinline__ uint64_t desc_const(uint32_t rows) {
  return ((uint64_t)((rows * 16) >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);
}
__device__ __forceinline__ uint64_t make_desc(uint32_t addr, uint32_t rows) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | desc_const(rows);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// Operand lists of the 64- and 32-register accumulators (d[]); C = P4V_F (fp32) or P4V_R (s32).
#define P4V_WG_D64                                                                                                 \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29," \
  "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,"    \
  "%57,%58,%59,%60,%61,%62,%63}"
#define P4V_WG_D32                                                                                                 \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29," \
  "%30,%31}"
#define P4V_WG_OP8(C, i) C(d[i]), C(d[i + 1]), C(d[i + 2]), C(d[i + 3]), C(d[i + 4]), C(d[i + 5]), C(d[i + 6]), C(d[i + 7])
#define P4V_WG_OP32(C) P4V_WG_OP8(C, 0), P4V_WG_OP8(C, 8), P4V_WG_OP8(C, 16), P4V_WG_OP8(C, 24)
#define P4V_WG_OP64(C) P4V_WG_OP32(C), P4V_WG_OP8(C, 32), P4V_WG_OP8(C, 40), P4V_WG_OP8(C, 48), P4V_WG_OP8(C, 56)
#define P4V_F(x) "+f"(x)
#define P4V_R(x) "+r"(x)

// D[64 rows][128 cols] (+)= A[64][32 bytes of K] * B[128][32 bytes of K]^T, both K-major in shared memory; the
// accumulator type picks bf16 (fp32 accumulators) or int8 (s32) operands.  accumulate = 0 starts from zero.
__device__ __forceinline__ void wgmma_k32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " P4V_WG_D64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
               : P4V_WG_OP64(P4V_F) : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_k32(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 " P4V_WG_D64 ", %64, %65, p;\n\t}"
               : P4V_WG_OP64(P4V_R) : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 rows][64 cols] (+)= A[64][32 bytes of K] * B[64][32 bytes of K]^T.
__device__ __forceinline__ void wgmma_n64_k32(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " P4V_WG_D32 ", %32, %33, p, 1, 1, 0, 0;\n\t}"
               : P4V_WG_OP32(P4V_F) : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_n64_k32(uint32_t (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 " P4V_WG_D32 ", %32, %33, p;\n\t}"
               : P4V_WG_OP32(P4V_R) : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 rows][32 cols] (+)= A[64][32 bytes of K] * B[32][32 bytes of K]^T, int8 operands.
__device__ __forceinline__ void wgmma_n32_k32(uint32_t (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n\t}"
               : P4V_WG_OP8(P4V_R, 0), P4V_WG_OP8(P4V_R, 8) : "l"(da), "l"(db), "r"(accumulate));
}
// Barrier `id` (1..15; 0 is __syncthreads) over `threads` threads, e.g. the 128 of one warpgroup.
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// One stage = nk (1..4) k32 steps of m64n128 over 128-row operand tiles, issued as one committed batch.  Each count has
// its own straight-line sequence: a data-dependent branch between the wgmmas of a batch makes ptxas wait for each one
// before issuing the next (C7520).  nk must be provably warp-uniform (callers broadcast it with __shfl_sync).
template <int N, typename AccT>
__device__ __forceinline__ void wgmma_seq(AccT (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  wgmma_k32(d, da, db, accumulate);
#pragma unroll
  for (int k = 1; k < N; ++k) wgmma_k32(d, da + 256 * k, db + 256 * k, 1u);   // +32 bytes of K = 2 x 128 rows x 16 B
}
template <typename AccT>
__device__ __forceinline__ void wgmma_stage(AccT (&d)[64], uint32_t nk, uint64_t da, uint64_t db, uint32_t accumulate) {
  wg_fence();
  switch (nk) {
    case 1: wgmma_seq<1>(d, da, db, accumulate); break;
    case 2: wgmma_seq<2>(d, da, db, accumulate); break;
    case 3: wgmma_seq<3>(d, da, db, accumulate); break;
    default: wgmma_seq<4>(d, da, db, accumulate); break;
  }
  wg_commit();
}

}  // namespace
