// Fused forward of a frozen MatMul on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces, for a module whose step sizes were packed once (p4v_matmul_pack), the reference's
//   out = quant_input(A, A_interval) @ quant_input(B, B_interval)      (quant_layers/matmul.py:40-45, :140-145;
//   split-of-softmax A operand :595-598, :628-629)
// in one launch: both operands are quantised from FP32 straight into shared memory and never exist in HBM.
//
// A CTA owns one output tile: problem p = image * heads + head, 128 rows of A[p], BN columns of B[p] (BN = 64 when
// S3 <= 64, else 128).  All 256 threads (two warpgroups of 64 rows) walk K in slabs of 64 elements through two
// shared-memory stages:
//   1. quantise slab s + 1 into the free stage while the wgmma of slab s (m64nBNk32 s32.s8.s8, two k32 steps; both
//      split-of-softmax planes into their own accumulator) runs on the other one; fence.proxy.async, then one block
//      barrier hands the stage to the async proxy;
//   2. epilogue in the order of the sweep's forward branch (sweep_tc.cu): r = 0, r = fmaf(-scale[g][head], (float)acc_g, r)
//      for the groups in order (plain: one; split-of-softmax: high then low part), out = -r.  The tile goes through
//      shared memory so that each warp stores whole row segments (lanes along the columns): the output rows of S3 = 197
//      floats are not 8-byte aligned, and fragment-order stores would touch 8 rows per instruction.
// Loads are lanes-along-the-unit-stride-dimension scalar loads, coalesced for any row alignment:
//   * A and a K-contiguous B (matmul1's k^T view): a warp reads 64 consecutive floats of one row (2 x 128 B) and writes
//     the quantised bytes into the K-major canonical layout [16-byte K chunk][rows][16 B];
//   * an N-contiguous B (matmul2's v): one thread reads 16 K rows of one column (lanes along N, 128 B per load),
//     quantises them and stores one 16-byte K chunk: the transpose int8 wgmma needs happens in registers.
// The quantisers are the operand-image kernel's (p4v_quant_plain / p4v_quant_sos, prep.cu), so the integers are those
// of the unfrozen forward; where that forward multiplies bf16 images (S2 < 64) its fp32 accumulator holds the same
// integer (every partial sum is below 2^24), so the output is bit-identical to p4v_matmul_quant_forward.
// Shared memory does not depend on S2: any sequence length takes this path.
#include "forward.cuh"
#include "sm90.cuh"
#include <climits>

namespace {

constexpr int kThreads = 256;                 // two warpgroups; every thread quantises, both warpgroups multiply
constexpr int kSlab = 64;                     // K elements (int8 bytes per row) of one stage: two wgmma k32 steps
constexpr int kAPlane = P4V_TILE * kSlab;     // one plane of the A slab: [4 chunks][128 rows][16 B]

template <int BN, bool SOS> struct MMLayout {
  static constexpr int a_bytes = (SOS ? 2 : 1) * kAPlane;
  static constexpr int stage = a_bytes + BN * kSlab;
  static constexpr int ld_out = BN + 8;      // staged output row, padded: the float2 fragment stores of a warp hit 2 wavefronts
  static constexpr int out_bytes = P4V_TILE * ld_out * 4;
  static constexpr int smem = (2 * stage > out_bytes ? 2 * stage : out_bytes) + 128;
};

// D[64 rows][BN cols] += A[64][32 int8 of K] * B[BN][32 int8 of K]^T.  The accumulators start at 0, so scale-d is the
// constant 1 here rather than the register predicate of wgmma_k32 / wgmma_n64_k32 (sm90.cuh): with a register, ptxas
// allocates forward_mm_kernel<64, false> differently.
__device__ __forceinline__ void mma_k32(uint32_t (&d)[64], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 " P4V_WG_D64 ", %64, %65, p;\n\t}"
               : P4V_WG_OP64(P4V_R) : "l"(da), "l"(db));
}
__device__ __forceinline__ void mma_k32(uint32_t (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 " P4V_WG_D32 ", %32, %33, p;\n\t}"
               : P4V_WG_OP32(P4V_R) : "l"(da), "l"(db));
}

// Two CTAs per SM (128 registers) overlap one tile's quantisation with another's MMAs and stores; the split-of-softmax
// kernel with 128-column tiles holds 2 x 64 accumulator registers and runs one CTA per SM.
template <int BN, bool SOS>
__global__ void __launch_bounds__(kThreads, (SOS && BN == 128) ? 1 : 2) forward_mm_kernel(const __grid_constant__ FwdMMParams P) {
  using L = MMLayout<BN, SOS>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;

  // the CTA's tile: column tiles fastest (they share the A rows, read again from L2), then row tiles, then problems
  const int tn = blockIdx.x % P.tiles_n;
  const int rest = blockIdx.x / P.tiles_n;
  const int tm = rest % P.tiles_m, p = rest / P.tiles_m;
  const int img = p / P.heads, h = p % P.heads;
  const int rowsA = min(P4V_TILE, P.S1 - tm * P4V_TILE), colsB = min(BN, P.S3 - tn * BN);
  const float* Ap = P.A + img * P.sA_b + h * P.sA_h + (long long)tm * P4V_TILE * P.sA_m;
  const float* Bp = P.B + img * P.sB_b + h * P.sB_h + (long long)tn * BN * P.sB_n;
  const bool b_kmajor = P.sB_k == 1;

  // the quantisers of the operand images (prep.cu: quant_image_kernel), step sizes of this head
  const float dA = SOS ? 1.f : __ldg(P.dA + h), dB = __ldg(P.dB + h);
  const bool fastA = p4v_rint_div_ok(dA), fastB = p4v_rint_div_ok(dB);
  const float rcpA = fastA ? __frcp_rn(dA) : 0.f, rcpB = fastB ? __frcp_rn(dB) : 0.f;
  const float split = SOS ? __ldg(P.split) : 0.f;
  auto qB = [&](float v) { return p4v_qbyte(p4v_quant_plain(v, dB, fastB, rcpB, false, 0.f, P.B_lo, P.B_hi)); };
  auto qA = [&](float v, int part) {
    return p4v_qbyte(SOS ? p4v_quant_sos(v, split, P.qm1, part) : p4v_quant_plain(v, dA, fastA, rcpA, false, 0.f, P.A_lo, P.A_hi));
  };

  // quantise K slab s into stage `buf`; elements outside the problem are 0 (not the quantised 0: the high
  // split-of-softmax part of 0 is not 0)
  auto load_slab = [&](int s, int buf) {
    const int k0 = s * kSlab;
    uint8_t* sa = smem + buf * L::stage;
    uint8_t* sb = sa + L::a_bytes;
    // A: warp rows warp + 8 i, lanes along K; in passes of 8 rows (split-of-softmax: 4) to bound the registers in flight
    constexpr int kRows = SOS ? 4 : 8;
#pragma unroll 1
    for (int pass = 0; pass < 16 / kRows; ++pass) {
      float v[kRows][2];
#pragma unroll
      for (int i = 0; i < kRows; ++i) {
        const int r = warp + 8 * (i + kRows * pass);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int k = k0 + lane + 32 * j;
          v[i][j] = (r < rowsA && k < P.S2) ? __ldg(Ap + (long long)r * P.sA_m + k) : 0.f;
        }
      }
#pragma unroll
      for (int i = 0; i < kRows; ++i) {
        const int r = warp + 8 * (i + kRows * pass);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int kk = lane + 32 * j;
          const bool in = r < rowsA && k0 + kk < P.S2;
          uint8_t* dst = sa + ((kk >> 4) * P4V_TILE + r) * 16 + (kk & 15);
          dst[0] = (uint8_t)(in ? qA(v[i][j], 1) : 0u);
          if (SOS) dst[kAPlane] = (uint8_t)(in ? qA(v[i][j], 2) : 0u);
        }
      }
    }
    if (b_kmajor) {        // B rows (output columns) are K-contiguous: as A
#pragma unroll 1
      for (int pass = 0; pass < BN / 64; ++pass) {
        float v[8][2];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int n = warp + 8 * (i + 8 * pass);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int k = k0 + lane + 32 * j;
            v[i][j] = (n < colsB && k < P.S2) ? __ldg(Bp + (long long)n * P.sB_n + k) : 0.f;
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int n = warp + 8 * (i + 8 * pass);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int kk = lane + 32 * j;
            sb[((kk >> 4) * BN + n) * 16 + (kk & 15)] = (uint8_t)((n < colsB && k0 + kk < P.S2) ? qB(v[i][j]) : 0u);
          }
        }
      }
    } else {               // N-contiguous: one thread = one column x one 16-byte K chunk, lanes along N
#pragma unroll
      for (int u = threadIdx.x; u < 4 * BN; u += kThreads) {
        const int n = u % BN, kc = u / BN;
        const int kb = k0 + 16 * kc;
        float v[16];
#pragma unroll
        for (int e = 0; e < 16; ++e)
          v[e] = (n < colsB && kb + e < P.S2) ? __ldg(Bp + (long long)(kb + e) * P.sB_k + n) : 0.f;
        uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int e = 0; e < 16; ++e)
          if (n < colsB && kb + e < P.S2) w[e >> 2] |= qB(v[e]) << ((e & 3) * 8);
        *reinterpret_cast<uint4*>(sb + (kc * BN + n) * 16) = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
  };

  uint32_t acc0[BN / 2], acc1[SOS ? BN / 2 : 1];
#pragma unroll
  for (int v = 0; v < BN / 2; ++v) { acc0[v] = 0u; if (SOS) acc1[v] = 0u; }

  const int n_slabs = (P.S2 + kSlab - 1) / kSlab;
  load_slab(0, 0);
  fence_proxy_async();   // generic-proxy stores -> wgmma (async proxy) reads
  __syncthreads();
  const uint32_t base = smem_u32(smem);
  for (int s = 0; s < n_slabs; ++s) {
    const uint32_t sa = base + (s & 1) * L::stage + wg * 64 * 16, sb = base + (s & 1) * L::stage + L::a_bytes;
    wg_fence();
#pragma unroll
    for (int k = 0; k < 2; ++k) {             // +32 bytes of K = 2 chunks
      mma_k32(acc0, make_desc(sa + k * 2 * kAPlane / 4, P4V_TILE), make_desc(sb + k * 2 * BN * 16, BN));
      if constexpr (SOS) mma_k32(acc1, make_desc(sa + kAPlane + k * 2 * kAPlane / 4, P4V_TILE), make_desc(sb + k * 2 * BN * 16, BN));
    }
    wg_commit();
    if (s + 1 < n_slabs) load_slab(s + 1, (s + 1) & 1);   // under the MMAs of slab s
    wg_wait0();
    fence_proxy_async();
    __syncthreads();                           // slab s + 1 visible; every warpgroup is done with stage s & 1
  }

  // ---- epilogue: the sweep's forward order, staged through shared memory (the stages are free) ----
  const float s0 = __ldg(P.scale + h), s1 = SOS ? __ldg(P.scale + P.heads + h) : 0.f;
  float* stg = reinterpret_cast<float*>(smem) + warp * 16 * L::ld_out;     // this warp's 16 fragment rows
#pragma unroll
  for (int v = 0; v < BN / 2; v += 2) {
    float o[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float r = 0.f;
      r = fmaf(-s0, __int2float_rn((int)acc0[v + e]), r);
      if constexpr (SOS) r = fmaf(-s1, __int2float_rn((int)acc1[v + e]), r);
      o[e] = -r;
    }
    const int row = (lane >> 2) + 8 * ((v >> 1) & 1), col = 8 * (v >> 2) + 2 * (lane & 3);
    *reinterpret_cast<float2*>(stg + row * L::ld_out + col) = make_float2(o[0], o[1]);
  }
  __syncwarp();
  const int row0 = tm * P4V_TILE + warp * 16;
  float* out = P.out + ((size_t)p * P.S1 + row0) * P.S3 + (size_t)tn * BN;
#pragma unroll 4
  for (int rr = 0; rr < 16; ++rr) {
    if (row0 + rr >= P.S1) break;
#pragma unroll
    for (int c = lane; c < BN; c += 32)
      if (c < colsB) out[(size_t)rr * P.S3 + c] = stg[rr * L::ld_out + c];
  }
}

template <int BN, bool SOS>
int launch(const FwdMMParams& p_in, cudaStream_t st) {
  constexpr int smem = MMLayout<BN, SOS>::smem;
  FwdMMParams p = p_in;
  p.tiles_m = p4v_cdiv(p.S1, P4V_TILE); p.tiles_n = p4v_cdiv(p.S3, BN);
  const long long ctas = (long long)p.batch * p.heads * p.tiles_m * p.tiles_n;
  P4V_REQUIRE(ctas <= INT_MAX, "matmul_frozen_forward: grid too large (%lld tiles)", ctas);
  P4V_CUDA_OK(cudaFuncSetAttribute(forward_mm_kernel<BN, SOS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  forward_mm_kernel<BN, SOS><<<(unsigned)ctas, kThreads, smem, st>>>(p);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace

// BN = 64 column tiles when S3 <= 64 (matmul2 of every model here: head dim 64 or 32), 128 otherwise
int p4v_launch_forward_mm_tc(const FwdMMParams& p, bool sos, cudaStream_t st) {
  if (p.S3 <= 64) return sos ? launch<64, true>(p, st) : launch<64, false>(p, st);
  return sos ? launch<128, true>(p, st) : launch<128, false>(p, st);
}
