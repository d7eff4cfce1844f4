// Fused forward of a frozen Linear layer on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces, for a layer whose integer weights were packed once (p4v_linear_pack), the reference's
//   out = F.linear(quant_input(x), quant_weight, bias)        (quant_layers/linear.py:62-67, :164-169, :601-607)
// in one launch: the quantised activations never exist in HBM.
//
// A CTA owns one 128-row tile of x and a contiguous share of the layer's 128-column output tiles.
//   1. All threads read the tile's FP32 rows (float4) and quantise them with the operand-image sequence
//      (p4v_quant_plain, prep.cu: quant_image_kernel) straight into shared memory, in the wgmma K-major canonical layout
//      [16-byte K chunk][128 rows][16 B] -- the tile of the activation image the unfrozen forward builds in HBM.
//      Post-GELU layers write a second plane with the negative part.  The stores go through the generic proxy, so every
//      thread fences them towards the async proxy (fence.proxy.async) before the block barrier that releases the MMAs.
//   2. Warp 8 streams the weight slabs of each column tile from the packed image through a cp.async.bulk ring (the
//      image of a ViT-B layer is L2 resident across the CTAs).  Warps 0-7 (two warpgroups, 64 rows each) run the forward
//      step's job list: wgmma m64n128k32 s32.s8.s8 of the resident row slab with the ring stage, one accumulator per
//      segment group, folded into r after its last job exactly as the sweep's forward branch does (sweep_tc.cu):
//      r = -bias, r = fmaf(-scale[g][col / 16], (float)acc, r) in the step's group order, out = -r.  Same integers, same
//      fp32 operations in the same order: the output is bit-identical to p4v_linear_quant_forward.
// 288 threads leave 224 registers per thread without setmaxnreg; the bounded mbarrier wait is inline, and the k32 steps of
// a stage are one straight-line batch selected by a warp-uniform count (ptxas C7520, see sweep_tc.cu).
#include "forward.cuh"
#include <cstdio>

namespace {

constexpr int kConsumers = 256;
constexpr int kConsumerWarps = kConsumers / 32;
constexpr int kThreads = kConsumers + 32;     // warps 0-7: consumers (two warpgroups); warp 8: bulk-copy producer

struct Chunk { int k0; short n, a; };         // a 16-byte K chunk of a plane: first source column, valid elements (0..16), step-size index

struct FwdCtl {
  alignas(16) P4VJob jobs[P4V_MAX_JOBS];
  float scale[P4V_MAX_GROUPS][P4V_TILE_CG];
  Chunk chunks[P4V_FWD_MAX_CHUNKS];
  alignas(8) unsigned long long full[P4V_FWD_MAX_STAGES];
  unsigned long long empty[P4V_FWD_MAX_STAGES];
};
static_assert(sizeof(FwdCtl) + 256 <= P4V_FWD_CTL_BYTES, "control block outgrew its shared-memory reserve");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(void* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(void* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t addr, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded: a protocol bug traps, never hangs (~10 s of SM clocks).  Inline; on timeout (block << 32 | thread << 20 |
// barrier smem address) is left in g_forward_timeout, and printed with -DP4V_SWEEP_DEBUG_PRINTF.
__device__ unsigned long long g_forward_timeout;
[[noreturn]] __device__ __forceinline__ void mbar_timeout(uint32_t addr, uint32_t parity) {
  g_forward_timeout = ((unsigned long long)blockIdx.x << 32) | ((unsigned long long)threadIdx.x << 20) | (addr & 0xFFFFFu);
  __threadfence();
#ifdef P4V_SWEEP_DEBUG_PRINTF
  printf("ptq4vit forward: mbarrier wait timed out (block %d thread %d smem 0x%x parity %u)\n", (int)blockIdx.x,
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
__device__ __forceinline__ void mbar_wait_addr(uint32_t addr, uint32_t parity) {
  if (!mbar_try(addr, parity)) mbar_wait_slow(addr, parity);
}
__device__ __forceinline__ void mbar_expect_tx_addr(uint32_t addr, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(addr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s_addr(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void warp_arrive(void* bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}

// K-major, no swizzle (the canonical layout of common.cuh): LBO = 128 rows x 16 B between the 16-byte K chunks,
// SBO = 128 B between 8-row groups; the 14-bit start address (16-byte units) is added per use.
__device__ __forceinline__ uint64_t desc_const() {
  constexpr uint64_t lbo = (P4V_TILE * 16) >> 4, sbo = 128 >> 4;
  return (lbo << 16) | (sbo << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define P4V_WG_D64                                                                                                 \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29," \
  "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,"    \
  "%57,%58,%59,%60,%61,%62,%63}"
#define P4V_WG_OP8(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), "+r"(d[i + 6]), "+r"(d[i + 7])
#define P4V_WG_OP64 P4V_WG_OP8(0), P4V_WG_OP8(8), P4V_WG_OP8(16), P4V_WG_OP8(24), P4V_WG_OP8(32), P4V_WG_OP8(40), P4V_WG_OP8(48), P4V_WG_OP8(56)

// D[64 rows][128 cols] (+)= A[64][32 int8 of K] * B[128][32 int8 of K]^T, both K-major in shared memory.
__device__ __forceinline__ void wgmma_k32(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 " P4V_WG_D64 ", %64, %65, p;\n\t}"
               : P4V_WG_OP64 : "l"(da), "l"(db), "r"(accumulate));
}
template <int N>
__device__ __forceinline__ void wgmma_seq(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  wgmma_k32(d, da, db, accumulate);
#pragma unroll
  for (int k = 1; k < N; ++k) wgmma_k32(d, da + 256 * k, db + 256 * k, 1u);   // +32 bytes of K = 2 x 128 rows x 16 B
}
__device__ __forceinline__ void wgmma_stage(uint32_t (&d)[64], uint32_t nk, uint64_t da, uint64_t db, uint32_t accumulate) {
  wg_fence();
  switch (nk) {
    case 1: wgmma_seq<1>(d, da, db, accumulate); break;
    case 2: wgmma_seq<2>(d, da, db, accumulate); break;
    case 3: wgmma_seq<3>(d, da, db, accumulate); break;
    default: wgmma_seq<4>(d, da, db, accumulate); break;
  }
  wg_commit();
}

// 16 quantised values -> one 16-byte chunk of int8
__device__ __forceinline__ void pack16(uint32_t (&w)[4], int e, float q) {
  w[e >> 2] |= (uint32_t)((int)q & 0xff) << ((e & 3) * 8);
}

__global__ void __launch_bounds__(kThreads, 1) forward_tc_kernel(const __grid_constant__ FwdParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  // carve: [resident activation tile][weight ring][control]
  const uint32_t nst = P.n_stages, sC = P.stage_bytes;
  const uint32_t resA = smem_u32(smem), ring = resA + P.a_bytes;
  FwdCtl& S = *reinterpret_cast<FwdCtl*>(smem + P.a_bytes + (size_t)nst * sC);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // the CTA's row tile and its share of the column tiles
  const int csplit = gridDim.x / P.tiles_m;
  const int tm = blockIdx.x / csplit, cs = blockIdx.x % csplit;
  const int tn0 = cs * P.tiles_n / csplit, tn1 = (cs + 1) * P.tiles_n / csplit;

  // ---- setup: jobs, chunk table, barriers ----
  for (int i = threadIdx.x; i < P.n_jobs; i += kThreads) S.jobs[i] = P.jobs[i];
  for (int s = threadIdx.x; s < P.nseg; s += kThreads) {
    const P4VSeg sg = P.segs[s];
    const int c0 = sg.dst_off / (P4V_TILE * 16), nch = ((sg.klen + 31) / 32) * 2;      // every segment is padded to 32 B
    for (int c = 0; c < nch; ++c)
      S.chunks[c0 + c] = Chunk{sg.k0 + 16 * c, (short)max(0, min(16, sg.klen - 16 * c)), (short)sg.didx};
  }
  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < nst; ++i) { mbar_init(&S.full[i], 1); mbar_init(&S.empty[i], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // ---- quantise the row tile into shared memory: one thread = one (16-byte chunk, row), rows fastest ----
  {
    const float rcp_neg = __frcp_rn(P.d_neg), rcp_neg_scalar = __fdiv_rn(1.f, P.d_neg);
    const bool fast_neg = p4v_rint_div_ok(P.d_neg);
    for (int u = threadIdx.x; u < (int)P.n_chunks * P4V_TILE; u += kThreads) {
      const int r = u & (P4V_TILE - 1), c = u >> 7;
      const Chunk ch = S.chunks[c];
      const int row = tm * P4V_TILE + r;
      uint32_t wp[4] = {0u, 0u, 0u, 0u}, wn[4] = {0u, 0u, 0u, 0u};
      if (row < P.M && ch.n > 0) {
        float vals[16];
        const float* src = P.x + (size_t)row * P.ld + ch.k0;
        if (ch.n == 16 && ((P.ld | ch.k0) & 3) == 0) {
          const float4* src4 = reinterpret_cast<const float4*>(src);
#pragma unroll
          for (int e = 0; e < 4; ++e) { const float4 t4 = __ldg(src4 + e); vals[4 * e] = t4.x; vals[4 * e + 1] = t4.y; vals[4 * e + 2] = t4.z; vals[4 * e + 3] = t4.w; }
        } else {
#pragma unroll
          for (int e = 0; e < 16; ++e) vals[e] = e < ch.n ? src[e] : 0.f;
        }
        const float delta = P.dX[ch.a];
        const bool fast = p4v_rint_div_ok(delta);
        const float rcp = fast ? __frcp_rn(delta) : 0.f;
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          if (e < ch.n) {
            float q = p4v_quant_plain(vals[e], delta, fast, rcp, false, 0.f, P.lo, P.hi);
            if (!(q == q)) q = 0.f;          // NaN (0/0) cannot be represented in the integer operand
            pack16(wp, e, q);
            if (P.twin) {
              float qn = p4v_quant_plain(vals[e], P.d_neg, fast_neg, rcp_neg, !P.ieee_div, rcp_neg_scalar, P.neg_lo, 0.f);
              if (!(qn == qn)) qn = 0.f;
              pack16(wn, e, qn);
            }
          }
        }
      }
      uint8_t* dst = smem + ((size_t)c * P4V_TILE + r) * 16;
      *reinterpret_cast<uint4*>(dst) = make_uint4(wp[0], wp[1], wp[2], wp[3]);
      if (P.twin) *reinterpret_cast<uint4*>(dst + P.plane_bytes) = make_uint4(wn[0], wn[1], wn[2], wn[3]);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> wgmma (async proxy) reads
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ======================= bulk-copy producer: the weight slabs of every job of every column tile =======================
    uint32_t stage = 0, phase = 0;
    const uint32_t full0 = smem_u32(&S.full[0]), empty0 = smem_u32(&S.empty[0]);
    for (int tn = tn0; tn < tn1; ++tn) {
      const uint8_t* wt = P.W + (size_t)tn * P.W_tile_bytes;
      for (int j = 0; j < P.n_jobs; ++j) {
        const P4VJob jb = S.jobs[j];
        mbar_wait_addr(empty0 + stage * 8, phase ^ 1);
        if (elect_one()) {
          const uint32_t fb = full0 + stage * 8, bytes = p4v_job_bytes(jb);
          mbar_expect_tx_addr(fb, bytes);
          bulk_g2s_addr(ring + stage * sC, wt + jb.c_off, bytes, fb);
        }
        if (++stage == nst) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ======================= consumers (2 warpgroups x 64 rows of the tile) =======================
  const int et = threadIdx.x;                        // 0..255
  const int wg = et >> 7;                            // row half of the tile
  const int frow = warp * 16 + (lane >> 2);          // fragment rows frow, frow + 8 (inside the tile)
  const int fcol = 2 * (lane & 3);                   // fragment columns 8 * i + fcol + {0, 1}
  const uint64_t dconst = desc_const();
  const uint32_t sC16 = sC >> 4;
  const uint32_t resA16 = ((resA & 0x3FFFF) >> 4) + wg * 64, ring16 = (ring & 0x3FFFF) >> 4;   // +64 rows x 16 B
  const uint32_t full0 = smem_u32(&S.full[0]);
  const int gm = tm * P4V_TILE + frow;               // global rows gm, gm + 8
  uint32_t stage = 0, phase = 0;
  uint32_t acc[64];
  float r[64];

  for (int tn = tn0; tn < tn1; ++tn) {
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers));   // previous column tile done with the scale rows
    for (int i = et; i < P.n_groups * P4V_TILE_CG; i += kConsumers)
      S.scale[i >> 3][i & 7] = P.scale[(size_t)(i >> 3) * P.nsg + tn * P4V_TILE_CG + (i & 7)];
    const int gc = tn * P4V_TILE + fcol;               // global columns gc + 8 * i + {0, 1}
#pragma unroll
    for (int v = 0; v < 64; ++v) {
      const int col = gc + 8 * (v >> 2) + (v & 1);
      r[v] = (P.bias && col < P.N) ? -P.bias[col] : 0.f;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers));   // scale rows visible

    int gi = 0;
    for (int j = 0; j < P.n_jobs; ++j) {
      const P4VJob jb = S.jobs[j];
      const uint32_t flags = jb.flags, kb = jb.kb, nsub = p4v_job_nsub(jb);
      mbar_wait_addr(full0 + stage * 8, phase);
      uint32_t a16 = resA16 + (jb.r_off >> 4), b16 = ring16 + stage * sC16;
      for (uint32_t sub = 0; sub < nsub; ++sub) {
        const uint64_t da = dconst | (uint64_t)a16, db = dconst | (uint64_t)b16;
        const uint32_t nk = __shfl_sync(0xffffffffu, kb >> 5, 0);   // warp-uniform for ptxas (C7520)
        wgmma_stage(acc, nk, da, db, (flags & P4V_JOB_FIRST) ? 0u : 1u);
        wg_wait0();
        if (sub + 1 == nsub) warp_arrive(&S.empty[stage], lane);
        if (flags & P4V_JOB_LAST) {
#pragma unroll
          for (int v = 0; v < 64; ++v) r[v] = fmaf(-S.scale[gi][v >> 3], __int2float_rn((int)acc[v]), r[v]);
          ++gi;
        }
        a16 += kb * 8; b16 += kb * 8;        // kb * 128 bytes, in 16-byte units
      }
      if (++stage == nst) { stage = 0; phase ^= 1; }
    }
    const bool pairs = (P.N & 1) == 0;       // even row stride: the fragment's column pairs are 8-byte aligned
#pragma unroll
    for (int v = 0; v < 64; v += 2) {
      const int row = gm + 8 * ((v >> 1) & 1), col = gc + 8 * (v >> 2);
      if (row < P.M) {
        float* o = P.out + (size_t)row * P.N + col;
        if (pairs) { if (col < P.N) *reinterpret_cast<float2*>(o) = make_float2(-r[v], -r[v + 1]); }
        else { if (col < P.N) o[0] = -r[v]; if (col + 1 < P.N) o[1] = -r[v + 1]; }
      }
    }
  }
}

}  // namespace

int p4v_launch_forward_tc(const FwdParams& p, int num_sms, cudaStream_t st) {
  P4V_REQUIRE(p.n_jobs >= 1 && p.n_jobs <= P4V_MAX_JOBS && p.n_groups <= P4V_MAX_GROUPS, "forward: too many K segments");
  P4V_REQUIRE(p.n_stages >= 2 && p.n_stages <= P4V_FWD_MAX_STAGES && p.n_chunks <= P4V_FWD_MAX_CHUNKS &&
              p.stage_bytes % 128 == 0 && p.a_bytes % 128 == 0, "forward: bad shared-memory plan");
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(p.out) & 7) == 0 && (reinterpret_cast<uintptr_t>(p.x) & 15) == 0,
              "forward: x must be 16-byte and out 8-byte aligned");
  const size_t smem = (size_t)p.a_bytes + (size_t)p.n_stages * p.stage_bytes + sizeof(FwdCtl) + 128;
  P4V_REQUIRE(smem <= P4V_FWD_SMEM, "forward: shared-memory plan too large (%zu bytes)", smem);
  // Fewer row tiles than SMs: split the column tiles of a row tile over several CTAs (each quantises the row tile again,
  // from L2) so that the whole GPU writes output.
  int csplit = num_sms / p.tiles_m;
  csplit = csplit < 1 ? 1 : (csplit > p.tiles_n ? p.tiles_n : csplit);
  P4V_CUDA_OK(cudaFuncSetAttribute(forward_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  forward_tc_kernel<<<p.tiles_m * csplit, kThreads, smem, st>>>(p);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}
