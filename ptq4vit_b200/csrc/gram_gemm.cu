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
#include "sm90.cuh"

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
    fence_mbarrier_init();
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
      const uint64_t rhi = make_desc(s0, 128) + a_off, rlo = make_desc(s0 + kTerm, 128) + a_off;
      const uint64_t chi = make_desc(s0 + 2 * kTerm, 128), clo = make_desc(s0 + 3 * kTerm, 128);
      // one K step = 16 bf16 = two 16-byte chunks; a stage holds two (kb = 64) or, at the end of a term, one (kb = 32).
      // Each case is one straight-line batch: a loop or branch between the wgmmas of a batch makes ptxas wait for each
      // one before issuing the next (C7520).
      auto kstep = [&](const uint32_t ks, const uint32_t accumulate) {
        const uint64_t k16 = ks * ((2u * 128 * 16) >> 4);
        wgmma_k32(acc, rhi + k16, chi + k16, accumulate);
        wgmma_k32(acc, rhi + k16, clo + k16, 1u);
        wgmma_k32(acc, rlo + k16, chi + k16, 1u);
      };
      // (the count is broadcast from lane 0 after the per-lane spin wait, so that ptxas can prove the branch warp-uniform)
      const bool two = __shfl_sync(0xffffffffu, kb == kStageKB ? 1 : 0, 0) != 0;
      wg_fence();
      if (two) { kstep(0, first ? 0u : 1u); kstep(1, 1u); }
      else     { kstep(0, first ? 0u : 1u); }
      wg_commit();
      wg_wait0();
      warp_arrive(&S.empty[stage], lane);
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
