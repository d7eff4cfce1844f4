// Gram GEMM of the normal-equation weight search (gram.cu):   H[o][pair] = sum_m (gs*g[m,o])^2 * Xq[m,k] * Xq[m,k']
// for ALL column blocks of a search round in one launch.  Both operands are exact two-term bf16 splits
//   A = (gs*g)^2 = A_hi + A_lo   (rows = output channels, K = tokens; image of 128-row tiles)
//   Z = Xq_k*Xq_k' = Z_hi + Z_lo (rows = (block, pair),   K = tokens; image of 256-row tiles)
// and the product keeps the three significant combinations hi*hi + hi*lo + lo*hi, accumulated in ONE fp32 wgmma
// accumulator.  A CTA computes a 128 x 128 output tile (one half of a 256-row pair tile); a stage of the shared-memory
// ring carries 64 bytes of K of all four term tiles, so every byte pulled from L2 feeds three tensor-core passes.
// The tensor core adds into the fp32 accumulator with truncation, so a long contraction of same-signed terms (the
// diagonal of H: 6304 tokens x 3 products) drifts by ~1e-5 relative.  The contraction is therefore cut into splits of
// `kSplitChunks` stages (256 tokens): each split starts a fresh accumulator and the consumer adds the splits in
// registers with round-to-nearest fp32 adds.  With `accumulate` (row chunks of a chunked search) that running sum starts
// from the stored H, so chunks whose boundaries fall on multiples of 256 tokens add in the order of one pass.
// Roles: warp 0 = bulk-copy producer; warpgroups 1-2 = consumers, each issuing wgmma m64n128 for 64 of the 128 output
// channels of the tile.
#include "gram.cuh"
#include <cstdio>

namespace {

constexpr int kThreads = 128 + 256;
constexpr int kConsumerWarps = 8;
constexpr int kSplitChunks = 8;                                     // stages (64 B of K = 32 tokens each) per accumulation split
constexpr int kStages = 6;
constexpr uint32_t kStageKB = 64;                                   // bytes of K per row and stage
constexpr uint32_t kTerm = kStageKB * 128;                          // bytes of one 128-row term tile in a stage
constexpr uint32_t kStageBytes = 4 * kTerm;                         // R hi, R lo, C hi, C lo: 32 KB

struct Ctl {
  alignas(8) unsigned long long full[kStages], empty[kStages];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(void* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ bool mbar_try(uint32_t addr, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded: a protocol bug traps, never hangs.  Inline and call-free (a call splits the wgmma pipeline, C7510); on timeout
// (block << 32 | thread << 20 | barrier smem address) is left in g_gram_timeout, and printed with -DP4V_SWEEP_DEBUG_PRINTF.
__device__ unsigned long long g_gram_timeout;
[[noreturn]] __device__ __forceinline__ void mbar_timeout(uint32_t addr, uint32_t parity) {
  g_gram_timeout = ((unsigned long long)blockIdx.x << 32) | ((unsigned long long)threadIdx.x << 20) | (addr & 0xFFFFFu);
  __threadfence();
#ifdef P4V_SWEEP_DEBUG_PRINTF
  printf("ptq4vit gram gemm: mbarrier wait timed out (block %d thread %d smem 0x%x parity %u)\n", (int)blockIdx.x,
         (int)threadIdx.x, addr, parity);
#endif
  __trap();
  while (true) {}
}
__device__ __forceinline__ void mbar_wait_slow(uint32_t addr, uint32_t parity) {
  const long long t0 = clock64();
  while (!mbar_try(addr, parity))
    if (clock64() - t0 > 20000000000ll) mbar_timeout(addr, parity);
}
__device__ __forceinline__ void mbar_wait(void* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  if (!mbar_try(addr, parity)) mbar_wait_slow(addr, parity);
}
__device__ __forceinline__ void mbar_arrive(void* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, void* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// K-major, no swizzle (same canonical layout as the sweep kernel): core matrix = 8 rows x 16 B, SBO = 128 B between
// 8-row groups, LBO = 128 rows x 16 B between the 16-byte K chunks of a stage tile.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  constexpr uint64_t lbo = (128 * 16) >> 4, sbo = 128 >> 4;
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (lbo << 16) | (sbo << 32);
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
      "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,"
      "%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}

__global__ void __launch_bounds__(kThreads, 1) gram_gemm_kernel(const __grid_constant__ GramGemmArgs a) {
  extern __shared__ uint8_t smem_raw[];
  // 128-byte aligned base, formed by pointer arithmetic on the __shared__ array (not an integer round trip) so that
  // the compiler keeps the shared state space: LDS / STS instead of generic loads and stores with 64-bit addresses.
  uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
  Ctl& S = *reinterpret_cast<Ctl*>(smem + (size_t)kStages * kStageBytes);
  const uint32_t ring = smem_u32(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(&S.full[i], 1); mbar_init(&S.empty[i], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int tiles = a.tiles_o * a.tiles_p * 2;                      // (output-channel tile, pair tile, pair half)
  const uint32_t term = a.term_bytes;
  const int n_chunks = (int)((term + kStageKB - 1) / kStageKB);

  if (warp < 4) {
    if (warp != 0) return;
    // ---------------- producer ----------------
    uint32_t stage = 0, phase = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      const int q = t / a.tiles_o;
      const uint8_t* rt = a.R + (size_t)(t % a.tiles_o) * a.R_tile_bytes;
      const uint8_t* ct = a.C + (size_t)(q >> 1) * a.C_tile_bytes + (size_t)(q & 1) * 128 * 16;
      for (int ch = 0; ch < n_chunks; ++ch) {
        const uint32_t k0 = ch * kStageKB, kb = (term - k0 < kStageKB) ? term - k0 : kStageKB;
        mbar_wait(&S.empty[stage], phase ^ 1);
        if (elect_one()) {
          const uint32_t s0 = ring + stage * kStageBytes;
          mbar_expect_tx(&S.full[stage], kb * 128 * 4);
          bulk_g2s(s0, rt + (size_t)k0 * 128, kb * 128, &S.full[stage]);
          bulk_g2s(s0 + kTerm, rt + ((size_t)term + k0) * 128, kb * 128, &S.full[stage]);
          // pair image rows of this half: 2 KB per 16-byte K chunk (chunk stride 256 rows x 16 B)
          for (uint32_t c16 = 0; c16 < kb / 16; ++c16) {
            bulk_g2s(s0 + 2 * kTerm + c16 * 2048, ct + ((size_t)k0 / 16 + c16) * 4096, 2048, &S.full[stage]);
            bulk_g2s(s0 + 3 * kTerm + c16 * 2048, ct + ((size_t)term + k0) * 256 + (size_t)c16 * 4096, 2048, &S.full[stage]);
          }
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  // ---------------- consumers: wgmma -> registers (sum of the splits) -> H ----------------
  const int et = threadIdx.x - 128;
  const int wg = et >> 7;                         // 64-channel half of the tile
  const int frow = (et >> 5) * 16 + (lane >> 2);  // fragment rows frow, frow + 8; columns 8 * i + 2 * (lane % 4) + {0, 1}
  const uint64_t a_off = (uint64_t)wg * 64;       // 64 rows x 16 B, in 16-byte units
  uint32_t stage = 0, phase = 0;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int q = t / a.tiles_o;
    const int o = (t % a.tiles_o) * 128 + frow;
    float sum[64], acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) { sum[j] = 0.f; acc[j] = 0.f; }
    float* hbase = a.H + (size_t)(q >> 1) * 256 + (q & 1) * 128 + 2 * (lane & 3);
    if (a.accumulate) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int oo = o + 8 * h;
        if (oo < a.O) {
          const float* hrow = hbase + (size_t)oo * a.ldH;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float2 v = *reinterpret_cast<const float2*>(hrow + 8 * i);
            sum[4 * i + 2 * h] = v.x; sum[4 * i + 2 * h + 1] = v.y;
          }
        }
      }
    }
    for (int ch = 0; ch < n_chunks; ++ch) {
      const bool first = ch % kSplitChunks == 0, last = (ch % kSplitChunks == kSplitChunks - 1) || ch == n_chunks - 1;
      const uint32_t k0 = ch * kStageKB, kb = (term - k0 < kStageKB) ? term - k0 : kStageKB;
      mbar_wait(&S.full[stage], phase);
      const uint32_t s0 = ring + stage * kStageBytes;
      const uint64_t rhi = make_desc(s0) + a_off, rlo = make_desc(s0 + kTerm) + a_off;
      const uint64_t chi = make_desc(s0 + 2 * kTerm), clo = make_desc(s0 + 3 * kTerm);
      // one K step = 16 bf16 = two 16-byte chunks; a stage holds two (kb = 64) or, at the end of a term, one (kb = 32).
      // Each case is one straight-line batch: a loop or branch between the wgmmas of a batch makes ptxas wait for each
      // one before issuing the next (C7520).
      auto kstep = [&](const uint32_t ks, const uint32_t accumulate) {
        const uint64_t k16 = ks * ((2u * 128 * 16) >> 4);
        wgmma_bf16(acc, rhi + k16, chi + k16, accumulate);
        wgmma_bf16(acc, rhi + k16, clo + k16, 1u);
        wgmma_bf16(acc, rlo + k16, chi + k16, 1u);
      };
      // (the count is broadcast from lane 0 after the per-lane spin wait, so that ptxas can prove the branch warp-uniform)
      const bool two = __shfl_sync(0xffffffffu, kb == kStageKB ? 1 : 0, 0) != 0;
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
      if (two) { kstep(0, first ? 0u : 1u); kstep(1, 1u); }
      else     { kstep(0, first ? 0u : 1u); }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(&S.empty[stage]);
      if (++stage == kStages) { stage = 0; phase ^= 1; }
      if (last) {
#pragma unroll
        for (int j = 0; j < 64; ++j) sum[j] += acc[j];
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int oo = o + 8 * h;
      if (oo < a.O) {
        float* hrow = hbase + (size_t)oo * a.ldH;
#pragma unroll
        for (int i = 0; i < 16; ++i) *reinterpret_cast<float2*>(hrow + 8 * i) = make_float2(sum[4 * i + 2 * h], sum[4 * i + 2 * h + 1]);
      }
    }
  }
}

}  // namespace

int p4v_gram_gemm(const GramGemmArgs& a, cudaStream_t st) {
  P4V_REQUIRE(a.term_bytes % 32 == 0 && a.ldH % 4 == 0, "gram gemm: bad operand geometry");
  const int tiles = a.tiles_o * a.tiles_p * 2;
  if (tiles < 1) return 0;
  const int grid = tiles < p4v_num_sms() ? tiles : p4v_num_sms();
  const size_t smem = (size_t)kStages * kStageBytes + sizeof(Ctl) + 256;
  P4V_CUDA_OK(cudaFuncSetAttribute(gram_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaEvent_t e0 = nullptr;
  if (p4v_prof_on()) p4v_prof_begin(st, &e0);
  gram_gemm_kernel<<<grid, kThreads, smem, st>>>(a); p4v_count_launch();
  // three bf16 term products per (output channel, pair, token): 128x256 pair tiles over term_bytes/2 tokens
  if (p4v_prof_on()) p4v_prof_end(st, e0, 2, 3.0 * 2.0 * 128.0 * 256.0 * (double)a.tiles_o * a.tiles_p * (double)(a.term_bytes / 2));
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}
