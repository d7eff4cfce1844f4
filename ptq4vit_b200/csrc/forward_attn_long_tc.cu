// Fused frozen attention core for long sequences (ViT / DeiT at 384 pixels: 577 tokens) on Hopper tensor cores (wgmma,
// sm_90a).
//
// The same computation as forward_attn_tc.cu for the ViT / DeiT block (utils/models.py:10-26):
//   attn = matmul1(q, k^T) * scale;  out = matmul2(attn.softmax(-1), v).transpose(1, 2).reshape(B, N, C)
// for 1 <= N <= 1024, bit-identical to that sequence on the frozen modules and torch's softmax.  Where the short kernel
// stages a query tile's FP32 score rows in shared memory (so N <= 256), this one keeps only the quantised operands
// resident and recomputes the scores of each 32-key chunk in three passes.
//
// A CTA (256 threads) owns one problem p = image * heads + head and all its 64-row query tiles.  All threads quantise every key row and v (transposed in registers) into shared memory once, with the loaders
// and frozen quantisers the short kernel uses (forward.cuh).  Then each warpgroup loops over its own query tiles
// (t = wg + 2i), with its own q tile, and for each tile makes three passes over the keys in 32-key
// chunks (matmul1: m64n32k32 s32.s8.s8, frozen matmul1's epilogue, then __fmul_rn(s, scale)):
//   1. the row maxima, in the accumulator layout (a max does not depend on the order);
//   2. the per-lane sums of torch's warp softmax.  softmax_warp_forward (rows of at most 1024 floats) gives lane l the
//      elements it * 32 + l and adds their expf(x - max) in `it` order, then xor-butterfly adds over offsets 16 .. 1.
//      The chunk's expf values go through a per-warp 16 x 32 staging tile so that lane l adds element c * 32 + l of
//      chunk c; chunks are visited in order, so every lane's sum has torch's order.  Padding (and torch's iterations
//      past the padded keys) adds +0, which changes no sum; the extra butterfly level that rows shorter than 32 meet
//      adds +0 too;
//   3. expf(x - max) / sum (IEEE division) quantised at once into a 32-key chunk of matmul2's A plane(s) (double
//      buffered), which matmul2 (m64n64k32, two accumulators with split-of-softmax) accumulates straight away.
// s32 sums are exact and the epilogue is deterministic, so every pass sees the same FP32 scores and the same expf values.
// The output goes through frozen matmul2's epilogue to out[b][i][h * D + d].  The key axis is padded to 32 (zero key
// rows and zero v rows), the head dimension to 32 for matmul1 and 64 for matmul2 (zero bytes).
#include "forward.cuh"
#include "sm90.cuh"
#include <climits>

namespace {

constexpr int kThreads = 256;                 // two warpgroups, each with its own query tiles
constexpr int kRows = 64;                     // query rows of a tile: the M of one wgmma
constexpr int kQBytes = kRows * 64;           // a q tile at the largest padded head dimension
constexpr int kPlane = 2 * kRows * 16;        // one 32-key chunk of a matmul2 A plane
constexpr int kWgBytes = kQBytes + 4 * kPlane;   // q tile | staging tiles (pass 2), aliased by 2 buffers x 2 planes (pass 3)

// byte offsets: k [kd/16][sp][16] | v^T [sp/16][64][16] | warpgroup 0 | warpgroup 1
__host__ __device__ inline int long_wg_offset(int sp, int kd) { return sp * kd + sp * 64; }

// matmul1 of the tile's q (at aQ) with keys [32c, 32c + 32) (k at aK), the s32 sums in the m64n32 accumulator layout
__device__ __forceinline__ void chunk_scores(uint32_t (&acc)[16], uint32_t aQ, uint32_t aK, int c, int sp, int kd) {
  wg_fence();
#pragma unroll 1
  for (int ks = 0; ks < kd / 32; ++ks)
    wgmma_n32_k32(acc, make_desc(aQ + ks * 2 * kRows * 16, kRows), make_desc(aK + (c * 32 + ks * 2 * sp) * 16, sp), ks > 0);
  wg_commit();
  wg_wait0();
}

// the named barrier of warpgroup wg (barrier 0 is __syncthreads); immediate ids keep the CTA at two hardware barriers
__device__ __forceinline__ void wg_bar(int wg) {
  if (wg == 0) named_bar_sync(1, 128);
  else named_bar_sync(2, 128);
}

// the XOR swizzle of staging row r: the 32 lanes' stores of one accumulator element land in 32 banks
__device__ __forceinline__ int stage_swz(int r) { return ((r & 3) << 3) | ((r >> 2) & 1); }

template <bool SOS>
__global__ void __launch_bounds__(kThreads, 1) forward_attn_long_kernel(const __grid_constant__ FwdAttnParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int p = blockIdx.x;
  const int img = p / P.heads, h = p % P.heads;
  const float* q = P.qkv + img * P.s_b + h * P.s_h;
  const float* k = q + P.s_p;
  const float* v = q + 2 * P.s_p;
  uint8_t* sK = smem;
  uint8_t* sV = smem + P.sp * P.kd;
  uint8_t* sQ = smem + long_wg_offset(P.sp, P.kd) + wg * kWgBytes;
  uint8_t* sP = sQ + kQBytes;
  float* sT = reinterpret_cast<float*>(sP) + (warp & 3) * 16 * 32;   // this warp's 16 x 32 FP32 staging tile

  // ---- keys and v, once for all the CTA's query tiles
  {
    const AttnSteps S = p4v_attn_steps<SOS>(P, h);
    p4v_attn_load_k(P, S, k, sK, warp, lane);
    p4v_attn_load_vt(P, S, v, sV);
  }
  fence_proxy_async();   // generic-proxy stores -> wgmma (async proxy) reads
  __syncthreads();

  const uint32_t aK = smem_u32(sK), aV = smem_u32(sV), aQ = smem_u32(sQ), aP = smem_u32(sP);
  const float s1 = __ldg(P.scale1 + h), scale = P.scale;
  const int wrow = (warp & 3) * 16, rl = lane >> 2;   // the warp's 16 rows; this lane's rows rl and rl + 8 of them
  const int chunks = P.sp / 32, tiles = (P.N + kRows - 1) / kRows;

#pragma unroll 1
  for (int t = wg; t < tiles; t += 2) {
    const int row0 = t * kRows, rows = min(kRows, P.N - row0);
    wg_bar(wg);      // every wgmma of the warpgroup's previous tile has retired: the q tile may be replaced
    const AttnSteps S = p4v_attn_steps<SOS>(P, h);     // read again per tile: fewer registers live across the passes
    p4v_attn_load_q<4>(P, S, q, sQ, row0, rows, warp & 3, lane);
    fence_proxy_async();
    wg_bar(wg);

    // ---- pass 1: row maxima
    float m[2] = {__int_as_float(0xff800000), __int_as_float(0xff800000)};
#pragma unroll 1
    for (int c = 0; c < chunks; ++c) {
      uint32_t acc[16];
      chunk_scores(acc, aQ, aK, c, P.sp, P.kd);
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        const int j = c * 32 + 8 * (e >> 2) + 2 * (lane & 3) + (e & 1), hh = (e >> 1) & 1;
        if (j < P.N) {
          const float x = __fmul_rn(p4v_attn_mm1(acc[e], s1), scale);
          m[hh] = (m[hh] > x) ? m[hh] : x;
        }
      }
    }
#pragma unroll
    for (int off = 1; off < 4; off <<= 1)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float o = __shfl_xor_sync(0xffffffffu, m[hh], off);
        m[hh] = (m[hh] < o) ? o : m[hh];
      }

    // ---- pass 2: torch's per-lane sums of expf(x - max), then its butterfly
    float ls[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) ls[r] = 0.f;
#pragma unroll 1
    for (int c = 0; c < chunks; ++c) {
      uint32_t acc[16];
      chunk_scores(acc, aQ, aK, c, P.sp, P.kd);
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        const int col = 8 * (e >> 2) + 2 * (lane & 3) + (e & 1), hh = (e >> 1) & 1, r = rl + 8 * hh;
        const float x = c * 32 + col < P.N ? expf(__fsub_rn(__fmul_rn(p4v_attn_mm1(acc[e], s1), scale), m[hh])) : 0.f;
        sT[r * 32 + (col ^ stage_swz(r))] = x;
      }
      __syncwarp();
#pragma unroll
      for (int r = 0; r < 16; ++r) ls[r] = __fadd_rn(ls[r], sT[r * 32 + (lane ^ stage_swz(r))]);
      __syncwarp();
    }
#pragma unroll
    for (int r = 0; r < 16; ++r)
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) ls[r] = __fadd_rn(ls[r], __shfl_xor_sync(0xffffffffu, ls[r], off));
    float sum[2] = {ls[0], ls[8]};
#pragma unroll
    for (int r = 1; r < 8; ++r)
      if (rl == r) { sum[0] = ls[r]; sum[1] = ls[r + 8]; }
    wg_bar(wg);      // every warp is done with its staging tile, which the probability planes overwrite

    // ---- pass 3: probabilities quantised chunk by chunk into matmul2's A planes, multiplied with v at once
    const float split = SOS ? __ldg(P.split2) : 0.f;
    uint32_t acc0[32], acc1[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) { acc0[e] = 0u; acc1[e] = 0u; }
#pragma unroll 1
    for (int c = 0; c < chunks; ++c) {
      uint32_t acc[16];
      chunk_scores(acc, aQ, aK, c, P.sp, P.kd);
      const int buf = (c & 1) * 2 * kPlane;      // double buffered: chunk c - 1's wgmma may still read the other one
#pragma unroll
      for (int e = 0; e < 16; e += 2) {
        const int col = 8 * (e >> 2) + 2 * (lane & 3), hh = (e >> 1) & 1, r = wrow + rl + 8 * hh;
        uint32_t b1 = 0u, b2 = 0u;
#pragma unroll
        for (int f = 0; f < 2; ++f) {
          const bool in = c * 32 + col + f < P.N;
          const float x = in ? expf(__fsub_rn(__fmul_rn(p4v_attn_mm1(acc[e + f], s1), scale), m[hh])) : 0.f;
          const float pr = __fdiv_rn(x, sum[hh]);
          b1 |= (uint32_t)p4v_attn_prob_byte<SOS>(P, S, pr, in, split, 1) << (8 * f);
          if (SOS) b2 |= (uint32_t)p4v_attn_prob_byte<SOS>(P, S, pr, in, split, 2) << (8 * f);
        }
        const int off = buf + ((col >> 4) * kRows + r) * 16 + (col & 15);
        *reinterpret_cast<uint16_t*>(sP + off) = (uint16_t)b1;
        if (SOS) *reinterpret_cast<uint16_t*>(sP + kPlane + off) = (uint16_t)b2;
      }
      fence_proxy_async();
      wg_bar(wg);
      wg_fence();
      const uint64_t db = make_desc(aV + c * 2 * 64 * 16, 64);
      wgmma_n64_k32(acc0, make_desc(aP + buf, kRows), db, 1u);
      if constexpr (SOS) wgmma_n64_k32(acc1, make_desc(aP + buf + kPlane, kRows), db, 1u);
      wg_commit();
      wg_wait0();
    }

    // ---- frozen matmul2's epilogue, stored in the proj input's [B, N, C] order
    const float t0 = __ldg(P.scale2 + h), t1 = SOS ? __ldg(P.scale2 + P.heads + h) : 0.f;
    const long long C = (long long)P.heads * P.D;
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int r = wrow + rl + 8 * ((e >> 1) & 1), col = 8 * (e >> 2) + 2 * (lane & 3);
      if (r >= rows || col >= P.D) continue;
      const float o0 = p4v_attn_mm2<SOS>(acc0[e], acc1[e], t0, t1), o1 = p4v_attn_mm2<SOS>(acc0[e + 1], acc1[e + 1], t0, t1);
      *reinterpret_cast<float2*>(P.out + ((long long)img * P.N + row0 + r) * C + (long long)h * P.D + col) = make_float2(o0, o1);
    }
  }
}

template <bool SOS>
int launch(const FwdAttnParams& p_in, cudaStream_t st) {
  FwdAttnParams p = p_in;
  p.sp = (p.N + 31) / 32 * 32;
  p.kd = (p.D + 31) / 32 * 32;
  const int smem = (int)p4v_attn_long_smem_bytes(p.sp, p.kd);
  const long long ctas = (long long)p.batch * p.heads;
  P4V_REQUIRE(ctas <= INT_MAX, "attention_frozen_forward_long: grid too large (%lld CTAs)", ctas);
  P4V_CUDA_OK(cudaFuncSetAttribute(forward_attn_long_kernel<SOS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  forward_attn_long_kernel<SOS><<<(unsigned)ctas, kThreads, smem, st>>>(p);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace

size_t p4v_attn_long_smem_bytes(int sp, int kd) { return (size_t)long_wg_offset(sp, kd) + 2 * kWgBytes + 128; }

int p4v_launch_forward_attn_long_tc(const FwdAttnParams& p, bool sos, cudaStream_t st) {
  return sos ? launch<true>(p, st) : launch<false>(p, st);
}
