// The hot kernel: candidate sweep on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces, for one search step, the reference's loop
//   for c in candidates: out = F.linear(x_sim, w_sim_c) ; sim = -(g*(y-out))**2 ; mean/sum
// (quant_layers/linear.py:466-488, :507-526; quant_layers/matmul.py:500-514, :541-555)
// without ever writing a candidate output to HBM.
//
// One persistent CTA per SM.  Work = (output tile 128x128) x (candidates).  Whole tiles are dealt
// round-robin in waves of gridDim.x (CTAs that run together share operand tiles in L2); the last partial
// wave is split at candidate granularity so that every SM finishes together.  Per tile fragment:
//   1. every consumer thread loads r = y - bias and g = grad * 2^k for the 64 elements of its accumulator fragment:
//      r into registers; g into registers (single-segment steps) or into this thread's slice of shared memory
//      (multi-segment steps, where it is needed once per candidate);
//   2. "fixed" segments (everything the candidate does not change) are multiplied on the tensor cores and
//      subtracted: r -= scale * acc;
//   3. per candidate only the segment(s) touched by the candidate step size are multiplied (bulk copy
//      -> smem ring -> wgmma -> registers); the consumer forms (g * (r - scale_c * acc))^2 straight from the
//      accumulator registers and writes one partial per (row quarter, 16 columns), or per row (row_keys).
// A job = one ring stage = up to 128 bytes of K of both operands, possibly several adjacent K slabs with an
// accumulator each (P4VJob::nsub); operands that do not change between candidates stay resident in shared memory.
// Roles: warp 0 = bulk-copy producer; warpgroups 1-2 = consumers, each issuing wgmma m64n128 for its 64 rows of the
// tile and running the epilogue on the fragment it holds.  The two consumer warpgroups share the tensor cores: while
// one runs its epilogue the other's MMAs proceed.  The launch budget is 168 registers per thread (384 threads); setmaxnreg
// moves it to the consumers (warpgroup 0: 56, consumers: 224), which hold r and the accumulator (128 registers) without
// spilling (ptxas -v: 0 bytes).  That needs a kernel without calls (ptxas drops setmaxnreg otherwise, C7507): the
// bounded mbarrier wait is inline and the scheduler divides in 32 bits.  The k32 steps of a stage are issued as one
// straight-line batch selected by a warp-uniform count, so ptxas pipelines them instead of waiting on each (C7520).
#include "common.cuh"
#include "sm90.cuh"
#include <algorithm>
#include <cstdlib>
#include <type_traits>

namespace {

constexpr int kMaxStages = 16;
constexpr int kConsumers = 256;
constexpr int kConsumerWarps = kConsumers / 32;
constexpr int kThreads = 128 + kConsumers;    // warpgroup 0: producer (+3 idle warps); warpgroups 1-2: consumers
constexpr int kSmemBudget = 208 * 1024;       // ring + resident operands + score reduction + parked tiles (227 KB per block in all)
// Score reduction: the two warps of a 32-row quarter each reduce their 16 rows per column group; the pair adds its two
// values through shared memory every kRedBatch candidates.  Layout [buffer][quarter][candidate][warp of pair][group].
constexpr int kRedBatch = 8;
constexpr int kRedBytes = 2 * 4 * kRedBatch * 2 * P4V_TILE_CG * 4;
constexpr int kTileBytes = P4V_TILE * P4V_TILE * 4;   // one fp32 tile parked in shared memory, [value pair][consumer thread]

struct SmemCtl {
  alignas(16) P4VJob jobs[P4V_MAX_JOBS];
  float fixs[P4V_MAX_GROUPS][P4V_TILE_CG];
  float candA[P4V_MAX_CAND][P4V_TILE_CG];
  float candB[P4V_MAX_GROUPS][P4V_TILE_CG];
  alignas(8) unsigned long long full[kMaxStages];
  unsigned long long empty[kMaxStages];
  unsigned long long res_full[2];
  unsigned long long res_empty[2];
  unsigned long long cres_full, cres_empty;
};

// Phase clocks (build with -DP4V_SWEEP_PHASE_CLOCKS, tools/sweep_phases.py): consumer warp 0 of each warpgroup and the
// producer add their clock64() cycles per phase into g_sweep_phases[kernel instantiation][phase]; p4v_sweep_phase_clocks
// reads them back.  Without the flag PhaseClock is empty and the kernel compiles to the same code as without it.
enum { kPhFull, kPhWgWait, kPhFixed, kPhCand, kPhFinal, kPhReduce, kPhConsumer, kPhEmpty, kPhProducer, kPhases };
#ifdef P4V_SWEEP_PHASE_CLOCKS
__device__ unsigned long long g_sweep_phases[6][kPhases];
struct PhaseClock {
  long long t0, mark;
  uint32_t t[kPhases];
  __device__ __forceinline__ void start() {
    t0 = mark = clock64();
#pragma unroll
    for (int k = 0; k < kPhases; ++k) t[k] = 0;
  }
  __device__ __forceinline__ void skip() { mark = clock64(); }   // the time since the last mark is not attributed
  __device__ __forceinline__ void lap(int k) { const long long n = clock64(); t[k] += (uint32_t)(n - mark); mark = n; }
  __device__ __forceinline__ void flush(int kind, int total, bool writer) {
    t[total] = (uint32_t)(clock64() - t0);
    if (writer)
#pragma unroll
      for (int k = 0; k < kPhases; ++k)
        if (t[k]) atomicAdd(&g_sweep_phases[kind][k], (unsigned long long)t[k]);
  }
};
#else
struct PhaseClock {
  __device__ __forceinline__ void start() {}
  __device__ __forceinline__ void skip() {}
  __device__ __forceinline__ void lap(int) {}
  __device__ __forceinline__ void flush(int, int, bool) {}
};
#endif

// Pair steps run one column half at a time (wgmma m64n64).  One stage of a pair step: the same nk k32 steps of the
// shared column slab against both row parts (d0: part 0, d1: part 1), one committed straight-line batch per count as in
// wgmma_stage.
template <int N, typename AccT>
__device__ __forceinline__ void wgmma_pair_seq(AccT (&d0)[32], AccT (&d1)[32], uint64_t da0, uint64_t da1, uint64_t db,
                                               uint32_t accumulate) {
#pragma unroll
  for (int k = 0; k < N; ++k) wgmma_n64_k32(d0, da0 + 256 * k, db + 256 * k, k ? 1u : accumulate);
#pragma unroll
  for (int k = 0; k < N; ++k) wgmma_n64_k32(d1, da1 + 256 * k, db + 256 * k, k ? 1u : accumulate);
}
template <typename AccT>
__device__ __forceinline__ void wgmma_pair_stage(AccT (&d0)[32], AccT (&d1)[32], uint32_t nk, uint64_t da0, uint64_t da1,
                                                 uint64_t db, uint32_t accumulate) {
  wg_fence();
  switch (nk) {
    case 1: wgmma_pair_seq<1>(d0, d1, da0, da1, db, accumulate); break;
    case 2: wgmma_pair_seq<2>(d0, d1, da0, da1, db, accumulate); break;
    case 3: wgmma_pair_seq<3>(d0, d1, da0, da1, db, accumulate); break;
    default: wgmma_pair_seq<4>(d0, d1, da0, da1, db, accumulate); break;
  }
  wg_commit();
}

// Register reallocation between the warpgroups (all four warps of a warpgroup execute it): the producer warpgroup
// gives registers back, the consumer warpgroups take them.  128 * 56 + 256 * 224 = 384 * 168, the launch budget.
// ptxas -v: no spills in any instantiation (40 / 232 leaves the producer spilling 12-20 bytes).
constexpr int kProducerRegs = 56, kConsumerRegs = 224;
__device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs)); }
__device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs)); }

// ---- work distribution -------------------------------------------------------------------------
struct Frag { int tile, p, tm, tn, c0, c1; };
// The tail wave has fewer than gridDim.x (<= SM count) tiles of at most P4V_MAX_CAND candidates, so its unit arithmetic
// fits 32 bits (and compiles to inline code: a 64-bit division is a subroutine call, which would void setmaxnreg).
struct Sched {
  int waves, k;                 // whole-tile waves, next wave index
  unsigned u, u_end;            // candidate-granular units of the tail wave
  int tail_tile0;
};
__device__ __forceinline__ void sched_init(const SweepParams& P, Sched& s) {
  const int tiles = P.P * P.tiles_m * P.tiles_n;
  const int G = gridDim.x;
  s.waves = tiles / G; s.k = 0;
  const unsigned tail_units = (unsigned)(tiles % G) * (unsigned)P.n_cand;
  s.u = tail_units * blockIdx.x / G; s.u_end = tail_units * (blockIdx.x + 1) / G;
  s.tail_tile0 = s.waves * G;
}
__device__ __forceinline__ bool next_frag(const SweepParams& P, Sched& s, Frag& f) {
  if (s.k < s.waves) {
    f.tile = s.k * gridDim.x + blockIdx.x; f.c0 = 0; f.c1 = P.n_cand; ++s.k;
  } else {
    if (s.u >= s.u_end) return false;
    f.tile = s.tail_tile0 + (int)(s.u / P.n_cand);
    f.c0 = (int)(s.u % P.n_cand);
    const unsigned rem = s.u_end - s.u;
    f.c1 = (rem < (unsigned)(P.n_cand - f.c0)) ? f.c0 + (int)rem : P.n_cand;
    s.u += f.c1 - f.c0;
  }
  const int per_p = P.tiles_m * P.tiles_n;
  f.p = f.tile / per_p;
  const int t = f.tile % per_p;
  if (P.order == 0) { f.tm = t % P.tiles_m; f.tn = t / P.tiles_m; }
  else              { f.tn = t % P.tiles_n; f.tm = t / P.tiles_n; }
  return true;
}

// Predicated read-only load (0 when !ok): a predicated instruction, not a branch around a load.
__device__ __forceinline__ float ldg_if(const float* p, bool ok) {
  float x;
  asm("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\tmov.b32 %0, 0;\n\t@q ld.global.nc.f32 %0, [%1];\n\t}"
      : "=f"(x) : "l"(p), "r"((uint32_t)ok));
  return x;
}

__device__ __forceinline__ float acc_to_float(uint32_t a) { return __int2float_rn((int)a); }
__device__ __forceinline__ float acc_to_float(float a) { return a; }

// Accumulator fragment of wgmma m64n128 (per thread 64 values): value v sits at
//   row = 16 * (warp in warpgroup) + lane / 4 + 8 * ((v >> 1) & 1),   column = 8 * (v >> 2) + 2 * (lane % 4) + (v & 1),
// so the 16-column scale / score group of value v is v >> 3.
// Reduce 8 per-lane values (one per column group) over the 32 lanes of the warp; lane l ends with the total of group
// (l >> 2) & 7 (reduce-scatter: 4 + 2 + 1 + 2 shuffles, fixed order).
__device__ __forceinline__ float reduce8_over_warp(float (&p)[8], int lane) {
  const unsigned full = 0xffffffffu;
#pragma unroll
  for (int half = 4, m = 16; half >= 1; half >>= 1, m >>= 1) {
    const bool hi = lane & m;
#pragma unroll
    for (int k = 0; k < half; ++k) {
      const float keep = hi ? p[k + half] : p[k], send = hi ? p[k] : p[k + half];
      p[k] = keep + __shfl_xor_sync(full, send, m);
    }
  }
  float t = p[0];
  t += __shfl_xor_sync(full, t, 2);
  t += __shfl_xor_sync(full, t, 1);
  return t;
}

// Consumer modes, chosen per launch by p4v_launch_sweep_tc:
//   kModeSingle: one candidate group; r stays in registers, g is parked.
//   kModeMulti:  several candidate groups, evaluated one job at a time; the residual is parked and restored per
//                candidate, g is read from global memory per candidate.
//   kModePair:   two candidate groups over the same candidate column slabs with different resident row parts (twin
//                activations of post-GELU weight steps, hi/lo parts of split-of-softmax B steps): one ring stage per
//                job pair, both parts multiplied per 64-column half, r stays in registers, g is parked.
//   kModeX8:     the int8 activation step of a bf16 layer (linear_api.cu build_plan, x8): a multi-segment step whose job
//                list is fixed, so the consumer runs it without reading the jobs.  Every candidate group is one K32 slab,
//                four per ring stage in group order, the column operand is the resident weight tile and there are no
//                fixed groups.  Same arithmetic as kModeMulti, group by group; launches report it as kModeMulti.
//   kModeFwdRes: a forward (out, no candidates) whose store adds the residual res: out = fl(-r + res), a block's
//                residual add folded into the frozen Linear that produces it (DESIGN §4.11).  The searches and the
//                plain forward never take it; launches report it as kModeMulti.
enum { kModeMulti = 0, kModeSingle = 1, kModePair = 2, kModeX8 = 3, kModeFwdRes = 4 };

template <bool kInt8, int kMode>
__global__ void __launch_bounds__(kThreads, 1) sweep_tc_kernel(const __grid_constant__ SweepParams P) {
  using AccT = typename std::conditional<kInt8, uint32_t, float>::type;
  constexpr bool kX8 = kMode == kModeX8;                       // parks the residual and reads g like kModeMulti
  constexpr bool kFwdRes = kMode == kModeFwdRes;              // stops after the forward store: the rest is dead code
  constexpr bool kPair = kMode == kModePair, kMulti = kMode == kModeMulti || kX8 || kFwdRes;
  static_assert(kInt8 || !kX8, "the x8 loop runs int8 operands only");
  // phase-clock row: x8 and the residual forward count as multi
  constexpr int kPhaseKind = (kInt8 ? 3 : 0) + (kX8 || kFwdRes ? kModeMulti : kMode);
  extern __shared__ uint8_t smem_raw[];
  // 128-byte aligned base, formed by pointer arithmetic on the __shared__ array (not an integer round trip) so that
  // the compiler keeps the shared state space: LDS / STS instead of generic loads and stores with 64-bit addresses.
  uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
  // carve: [ring R stages][ring C stages][resident R x bufs][resident C][control][score reduction][gradient tile]
  const uint32_t sR = P.stage_r_bytes, sC = P.stage_c_bytes, nst = P.n_stages, resB = P.resident_bytes, cresB = P.cres_bytes;
  const uint32_t ringR = smem_u32(smem), ringC = ringR + nst * sR, resR = ringC + nst * sC, resC = resR + P.resident_bufs * resB;
  const size_t ctl_off = (size_t)nst * (sR + sC) + (size_t)P.resident_bufs * resB + cresB;
  SmemCtl& S = *reinterpret_cast<SmemCtl*>(smem + ctl_off);
  float* const red = reinterpret_cast<float*>(smem + ctl_off + ((sizeof(SmemCtl) + 127) & ~size_t(127)));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // ---- one-time setup ----
  const int n_jobs = P.n_fixed_jobs + P.n_cand_jobs;
  for (int i = threadIdx.x; i < n_jobs; i += kThreads) S.jobs[i] = P.jobs[i];
  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < nst; ++i) { mbar_init(&S.full[i], 1); mbar_init(&S.empty[i], kConsumerWarps); }
    for (int i = 0; i < 2; ++i) { mbar_init(&S.res_full[i], 1); mbar_init(&S.res_empty[i], kConsumerWarps); }
    mbar_init(&S.cres_full, 1); mbar_init(&S.cres_empty, kConsumerWarps);
    fence_mbarrier_init();
  }
  __syncthreads();

  Sched sched; sched_init(P, sched);
  Frag f;

  if (warp < 4) {
    regs_dec();
    if (warp != 0) return;
    // ======================= bulk-copy producer (whole warp runs the loop, one elected lane issues) =======================
    uint32_t stage = 0, phase = 0, rbuf = 0, rphase = 0, cphase = 0;
    const uint32_t full0 = smem_u32(&S.full[0]), empty0 = smem_u32(&S.empty[0]);
    PhaseClock pc; pc.start();
    while (next_frag(P, sched, f)) {
      const size_t rt = P.R_shared ? (size_t)f.tm : (size_t)(f.p * P.tiles_m + f.tm), ct = (size_t)(f.p * P.tiles_n + f.tn);
      const uint8_t* r_cur = P.R_cur + rt * P.R_tile_bytes;
      const uint8_t* c_cur = P.C_cur + ct * P.C_tile_bytes;
      if (cresB) {     // the tile's whole current column image: once per fragment (single buffer: wait for the previous tile's MMAs)
        mbar_wait(&S.cres_empty, cphase ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&S.cres_full, cresB);
          for (uint32_t o = 0; o < cresB; o += 32768u)
            bulk_g2s(resC + o, c_cur + o, (cresB - o < 32768u) ? cresB - o : 32768u, &S.cres_full);
        }
        cphase ^= 1;
      }
      if (resB) {      // row operand of the candidate jobs: once per fragment, reused by every candidate
        mbar_wait(&S.res_empty[rbuf], rphase ^ 1);
        uint32_t total = 0;
        for (int j = 0; j < P.n_cand_jobs; ++j) total += p4v_job_bytes(S.jobs[P.n_fixed_jobs + j]);
        if (elect_one()) {
          mbar_expect_tx(&S.res_full[rbuf], total);
          for (int j = 0; j < P.n_cand_jobs; ++j) {
            const P4VJob jb = S.jobs[P.n_fixed_jobs + j];
            bulk_g2s(resR + rbuf * resB + jb.res_off, r_cur + jb.r_off, p4v_job_bytes(jb), &S.res_full[rbuf]);
          }
        }
        if (++rbuf == P.resident_bufs) { rbuf = 0; rphase ^= 1; }
      }
      auto issue = [&](const P4VJob j, const uint8_t* rr, const uint8_t* cc) {
        pc.skip();
        mbar_wait_addr(empty0 + stage * 8, phase ^ 1);
        pc.lap(kPhEmpty);
        const uint32_t bytes = p4v_job_bytes(j);
        if (elect_one()) {
          const uint32_t fb = full0 + stage * 8;
          const uint32_t nload = ((j.flags & P4V_JOB_RRES) ? 0u : 1u) + ((j.flags & P4V_JOB_CRES) ? 0u : 1u);
          mbar_expect_tx_addr(fb, nload * bytes);
          if (!(j.flags & P4V_JOB_RRES)) bulk_g2s_addr(ringR + stage * sR, rr + j.r_off, bytes, fb);
          if (!(j.flags & P4V_JOB_CRES)) bulk_g2s_addr(ringC + stage * sC, cc + j.c_off, bytes, fb);
        }
        if (++stage == nst) { stage = 0; phase ^= 1; }
      };
      for (int j = 0; j < P.n_fixed_jobs; ++j) issue(S.jobs[j], r_cur, c_cur);
      const uint8_t* r_cand = P.R_cand + rt * P.R_cand_tile_bytes + (size_t)f.c0 * P.R_cand_stride;
      const uint8_t* c_cand = P.C_cand + ct * P.C_cand_tile_bytes + (size_t)f.c0 * P.C_cand_stride;
      const int stage_jobs = kPair ? P.n_cand_jobs / 2 : P.n_cand_jobs;   // pair: job i + n/2 shares job i's column slab
      for (int c = f.c0; c < f.c1; ++c) {
        for (int jj = 0; jj < stage_jobs; ++jj) {
          const P4VJob j = S.jobs[P.n_fixed_jobs + jj];
          issue(j, (j.flags & P4V_JOB_RCAND) ? r_cand : r_cur, (j.flags & P4V_JOB_CCAND) ? c_cand : c_cur);
        }
        r_cand += P.R_cand_stride; c_cand += P.C_cand_stride;
      }
    }
    pc.flush(kPhaseKind, kPhProducer, lane == 0);
    return;
  }

  // ======================= consumers (2 warpgroups x 64 rows of the tile) =======================
  // Registers hold the residual r and the accumulator fragment.  This thread's slice of shared memory ([fragment value
  // pair][consumer thread] float2) parks g in single-segment and pair steps and, in multi-segment steps, the residual
  // every candidate starts from (g is then read from global memory once per candidate).
  regs_inc();
  const int et = threadIdx.x - 128;                  // 0..255
  const int wg = et >> 7;                            // row half of the tile
  const int cw = et >> 5;                            // consumer warp 0..7 = 16-row slice
  const int quarter = cw >> 1;                       // 32-row quarter (two warps)
  const int frow = cw * 16 + (lane >> 2);            // fragment rows frow, frow + 8 (inside the tile)
  const int fcol = 2 * (lane & 3);                   // fragment columns 8 * i + fcol + {0, 1}
  const float gs = (P.out && !P.out_residual) ? 1.f : *P.gscale;
  const uint64_t dconst = desc_const(P4V_TILE);
  const uint32_t sR16 = sR >> 4, sC16 = sC >> 4;
  const uint32_t ringR16 = ((ringR & 0x3FFFF) >> 4) + wg * 64, ringC16 = (ringC & 0x3FFFF) >> 4;   // +64 rows x 16 B
  const uint32_t resC16 = (resC & 0x3FFFF) >> 4;
  // x8: candidate group 0's slab in the resident weight tile, in 16-byte units (the groups' slabs follow it 32 bytes of K apart)
  const uint32_t x8_b16 = kX8 ? resC16 + (S.jobs[0].c_off >> 4) : 0;
  const uint32_t full0 = smem_u32(&S.full[0]);
  float2* const park = reinterpret_cast<float2*>(red + kRedBytes / 4) + et;  // values (v, v+1) at park[(v / 2) * 256]
  uint32_t stage = 0, phase = 0, rbuf = 0, rphase = 0, cphase = 0;
  int nb = 0, rb = 0;                                // score reduction: candidates in the open batch, buffer
  AccT acc[64];
  float r[64];
  PhaseClock pc; pc.start();

  // One job = one stage: wait for its bytes; per sub-accumulator run its K steps (a FIRST job starts from zero) and call
  // on_last() after a LAST one; the stage goes back to the producer with the last sub-accumulator.
  auto run = [&](const P4VJob jb, const uint32_t ra16, auto&& on_last) {
    const uint32_t flags = jb.flags, kb = jb.kb, nsub = p4v_job_nsub(jb);
    pc.skip();
    mbar_wait_addr(full0 + stage * 8, phase);
    pc.lap(kPhFull);
    uint32_t a16 = (flags & P4V_JOB_RRES) ? ra16 : ringR16 + stage * sR16;
    uint32_t b16 = (flags & P4V_JOB_CRES) ? resC16 + (jb.c_off >> 4) : ringC16 + stage * sC16;
    for (uint32_t sub = 0; sub < nsub; ++sub) {
      const uint64_t da = dconst | (uint64_t)a16, db = dconst | (uint64_t)b16;
      // k32 steps, broadcast from lane 0 right before the batch so that ptxas can prove the dispatch warp-uniform
      // (neither a value read from shared memory nor code behind the per-lane spin wait is, and a possibly divergent
      // branch around a wgmma batch serialises it, C7520)
      const uint32_t nk = __shfl_sync(0xffffffffu, kb >> 5, 0);
      wgmma_stage(acc, nk, da, db, (flags & P4V_JOB_FIRST) ? 0u : 1u);
      pc.skip();
      wg_wait0();
      pc.lap(kPhWgWait);
      if (sub + 1 == nsub) warp_arrive(&S.empty[stage], lane);
      if (flags & P4V_JOB_LAST) on_last();
      a16 += kb * 8; b16 += kb * 8;        // kb * 128 bytes, in 16-byte units
    }
    if (++stage == nst) { stage = 0; phase ^= 1; }
  };

  while (next_frag(P, sched, f)) {
    if constexpr (kPair) {   // acc must not stay live into the candidates, whose column halves use a0/a1 (see there)
#pragma unroll
      for (int v = 0; v < 64; ++v) acc[v] = 0;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers));   // previous fragment done with the tables
    {
      const int sg0 = (P.sg_mode == P4V_SG_COLUMN) ? f.tn * P4V_TILE_CG : (f.p % P.nsg);
      const int sgs = (P.sg_mode == P4V_SG_COLUMN) ? 1 : 0;
      for (int i = et; i < P.n_fixed_groups * P4V_TILE_CG; i += kConsumers)
        S.fixs[i >> 3][i & 7] = P.fix_scale[(size_t)(i >> 3) * P.nsg + sg0 + (i & 7) * sgs];
      for (int i = et; i < P.n_cand_groups * P4V_TILE_CG; i += kConsumers)
        S.candB[i >> 3][i & 7] = P.candB[(size_t)(i >> 3) * P.nsg + sg0 + (i & 7) * sgs];
      for (int i = et + f.c0 * P4V_TILE_CG; i < f.c1 * P4V_TILE_CG; i += kConsumers)
        S.candA[i >> 3][i & 7] = P.candA[(size_t)(i >> 3) * P.nsg + sg0 + (i & 7) * sgs];
    }
    const int gm = f.tm * P4V_TILE + frow;               // global rows gm, gm + 8
    const int gc = f.tn * P4V_TILE + fcol;               // global columns gc + 8 * i + {0, 1}
    const size_t pbase = (size_t)f.p * P.prob_stride;
    // -- residual target (and gradient) of this thread's fragment --
    if (P.out != nullptr && !P.out_residual) {           // quant_forward: r starts at -bias, output = -r
#pragma unroll
      for (int v = 0; v < 64; ++v) {
        const int col = gc + 8 * (v >> 2) + (v & 1);
        r[v] = (P.bias && col < P.N) ? -P.bias[col] : 0.f;
      }
    } else {
      const bool want_g = P.out == nullptr;
      const bool vec = ((P.ld | P.prob_stride) & 1) == 0 && (f.tn + 1) * P4V_TILE <= P.N &&
                       ((reinterpret_cast<uintptr_t>(P.Y) | (want_g ? reinterpret_cast<uintptr_t>(P.Gr) : 0) |
                         (P.bias ? reinterpret_cast<uintptr_t>(P.bias) : 0)) & 7) == 0;
#pragma unroll
      for (int v = 0; v < 64; v += 2) {
        const int row = gm + 8 * ((v >> 1) & 1), col = gc + 8 * (v >> 2);
        const size_t off = pbase + (size_t)row * P.ld + col;
        float y0 = 0.f, y1 = 0.f, g0 = 0.f, g1 = 0.f, b0 = 0.f, b1 = 0.f;
        if (row < P.M) {
          if (vec) {
            const float2 yv = *reinterpret_cast<const float2*>(P.Y + off);
            y0 = yv.x; y1 = yv.y;
            if (want_g) { const float2 gv = *reinterpret_cast<const float2*>(P.Gr + off); g0 = gv.x; g1 = gv.y; }
            if (P.bias) { const float2 bv = *reinterpret_cast<const float2*>(P.bias + col); b0 = bv.x; b1 = bv.y; }
          } else {
            if (col < P.N) { y0 = P.Y[off]; if (want_g) g0 = P.Gr[off]; if (P.bias) b0 = P.bias[col]; }
            if (col + 1 < P.N) { y1 = P.Y[off + 1]; if (want_g) g1 = P.Gr[off + 1]; if (P.bias) b1 = P.bias[col + 1]; }
          }
        }
        r[v] = y0 - b0; r[v + 1] = y1 - b1;
        if (!kMulti && want_g) park[(v >> 1) * kConsumers] = make_float2(g0 * gs, g1 * gs);
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers));   // tables visible
    if (cresB) { mbar_wait(&S.cres_full, cphase); cphase ^= 1; }

    // -- fixed segments: r -= scale * acc --
    {
      int gi = 0;
      for (int j = 0; j < P.n_fixed_jobs; ++j)
        run(S.jobs[j], 0u, [&] {
          pc.skip();
#pragma unroll
          for (int v = 0; v < 64; ++v) r[v] = fmaf(-S.fixs[gi][v >> 3], acc_to_float(acc[v]), r[v]);
          ++gi;
          pc.lap(kPhFixed);
        });
    }
    if (kFwdRes || P.out != nullptr) {
      if (cresB) warp_arrive(&S.cres_empty, lane);
      if constexpr (kFwdRes) {
        // out = fl(-r + res): torch's FP32 add of the stored value and the shortcut, read as the pairs it writes
        const bool pairs = ((P.ld | P.N | (long long)pbase) & 1) == 0;
#pragma unroll
        for (int v = 0; v < 64; v += 2) {
          const int row = gm + 8 * ((v >> 1) & 1), col = gc + 8 * (v >> 2);
          if (row < P.M) {
            const size_t off = pbase + (size_t)row * P.ld + col;
            if (pairs) {
              if (col < P.N) {
                const float2 sv = __ldg(reinterpret_cast<const float2*>(P.res + off));
                *reinterpret_cast<float2*>(P.out + off) = make_float2(__fadd_rn(-r[v], sv.x), __fadd_rn(-r[v + 1], sv.y));
              }
            } else {
              if (col < P.N) P.out[off] = __fadd_rn(-r[v], __ldg(P.res + off));
              if (col + 1 < P.N) P.out[off + 1] = __fadd_rn(-r[v + 1], __ldg(P.res + off + 1));
            }
          }
        }
      } else {
#pragma unroll
        for (int v = 0; v < 64; ++v) {
          const int row = gm + 8 * ((v >> 1) & 1), col = gc + 8 * (v >> 2) + (v & 1);
          if (row < P.M && col < P.N) P.out[pbase + (size_t)row * P.ld + col] = P.out_residual ? r[v] : -r[v];
        }
      }
      continue;
    }
    if constexpr (kMulti) {
#pragma unroll
      for (int v = 0; v < 64; v += 2) park[(v >> 1) * kConsumers] = make_float2(r[v], r[v + 1]);
    }
    // g of values (v, v + 1): parked (single-segment and pair steps) or, in multi-segment steps, read from global memory
    // (L2) once per candidate.  Those reads are predicated scalar loads with no branch around them: with a branch per
    // pair, ptxas puts each load and its use in a reconvergence region of its own, so the 32 L2 round trips of a
    // candidate's final epilogue ran one after another (a third of the consumer's time in the int8 activation steps).
    const float* const g0p = P.Gr + pbase + (size_t)gm * P.ld + gc;   // row gm; row gm + 8 below
    const float* const g8p = g0p + 8 * P.ld;
    const bool g0ok = gm < P.M, g8ok = gm + 8 < P.M;
    auto gpair = [&](const int v) -> float2 {
      if constexpr (!kMulti) {
        return park[(v >> 1) * kConsumers];
      } else {
        const int h = (v >> 1) & 1, dc = 8 * (v >> 2);
        const bool row = h ? g8ok : g0ok;
        const bool ok0 = row & (gc + dc < P.N), ok1 = row & (gc + dc + 1 < P.N);
        const float* const gp = (h ? g8p : g0p) + dc;
        const float x0 = ldg_if(gp, ok0), x1 = ldg_if(gp + 1, ok1);
        return make_float2(ok0 ? x0 * gs : 0.f, ok1 ? x1 * gs : 0.f);
      }
    };
    // The same loads in the x8 loop, with the predicates folded into one column limit per fragment row (0 when the row
    // is outside the problem): value (v, v + 1) loads when its column offset dc (+ 1), a compile-time constant, is below it.
    // gs is a power of two in [2^-100, 2^100] (p4v_make_gscale), so a value that is not loaded gives 0 * gs = +0, the
    // 0.f that gpair selects.
    const int glim0 = g0ok ? P.N - gc : 0, glim8 = g8ok ? P.N - gc : 0;
    auto gpair_x8 = [&](const int v) -> float2 {
      const int h = (v >> 1) & 1, dc = 8 * (v >> 2);
      const int lim = h ? glim8 : glim0;
      const float* const gp = (h ? g8p : g0p) + dc;
      return make_float2(ldg_if(gp, dc < lim) * gs, ldg_if(gp + 1, dc + 1 < lim) * gs);
    };

    // -- candidates --
    uint32_t res16 = 0;
    if (resB) {
      mbar_wait(&S.res_full[rbuf], rphase);
      res16 = ((resR + rbuf * resB) & 0x3FFFF) >> 4;
    }
    // Pair steps: the two column-half accumulators.  Defined here, and acc above at the start of the fragment, so that
    // ptxas sees neither live across the other's use (a wgmma reads its accumulators: an undefined one stays live
    // around the loops, which spills).
    AccT a0[32], a1[32];
    if constexpr (kPair) {
#pragma unroll
      for (int v = 0; v < 32; ++v) { a0[v] = 0; a1[v] = 0; }
    }
    for (int c = f.c0; c < f.c1; ++c) {
      if constexpr (kMulti) {
        if (kX8 || c > f.c0) {   // x8: on the first candidate too, so that r is dead after each final epilogue
#pragma unroll
          for (int v = 0; v < 64; v += 2) { const float2 x = park[(v >> 1) * kConsumers]; r[v] = x.x; r[v + 1] = x.y; }
        }
      }
      float ph[P4V_TILE_CG][2];                    // sum of (g * e)^2 per column group and fragment row
      float p[P4V_TILE_CG];                        // ... and per column group (this thread's two rows)
      if constexpr (kPair) {
        // The candidate's np stages (job i: part 0 = job i, part 1 = job i + np, same column slab).  A column half's two
        // accumulators run over all of them before its epilogue, so all np stages are held until the second half is
        // done (the launcher guarantees np + 1 ring stages).  Same fp32 operations in the same order as the
        // multi-segment path: t = r - s0 * acc0, then (g * (t - s1 * acc1))^2.
        const int np = P.n_cand_jobs >> 1;
        const bool noA0 = P.cand_noA_mask & 1ull, noA1 = (P.cand_noA_mask >> 1) & 1ull;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          uint32_t s = stage, sp = phase;
          for (int i = 0; i < np; ++i) {
            if (half == 0) mbar_wait_addr(full0 + s * 8, sp);
            const P4VJob j0 = S.jobs[P.n_fixed_jobs + i], j1 = S.jobs[P.n_fixed_jobs + np + i];
            const uint64_t da0 = dconst | (uint64_t)(res16 + (j0.res_off >> 4) + wg * 64);
            const uint64_t da1 = dconst | (uint64_t)(res16 + (j1.res_off >> 4) + wg * 64);
            const uint64_t db = dconst | (uint64_t)(ringC16 + s * sC16 + half * 64);   // +64 rows x 16 B
            const uint32_t nk = __shfl_sync(0xffffffffu, (uint32_t)j0.kb >> 5, 0);   // warp-uniform, see run()
            wgmma_pair_stage(a0, a1, nk, da0, da1, db, (j0.flags & P4V_JOB_FIRST) ? 0u : 1u);
            if (++s == nst) { s = 0; sp ^= 1; }
          }
          wg_wait0();
          // a0[v] / a1[v] of this half = fragment value 32 * half + v of the m64n128 layout (column groups 4 * half ..)
#pragma unroll
          for (int k = 0; k < P4V_TILE_CG / 2; ++k) {
            const int kk = (P4V_TILE_CG / 2) * half + k;
            const float s0 = noA0 ? S.candB[0][kk] : S.candA[c][kk] * S.candB[0][kk];
            const float s1 = noA1 ? S.candB[1][kk] : S.candA[c][kk] * S.candB[1][kk];
            float q[2] = {0.f, 0.f};
#pragma unroll
            for (int e = 0; e < 8; e += 2) {
              const int v = 8 * k + e, V = 32 * half + v;
              const float2 gv = gpair(V);
              const float w0 = gv.x * fmaf(-s1, acc_to_float(a1[v]), fmaf(-s0, acc_to_float(a0[v]), r[V]));
              const float w1 = gv.y * fmaf(-s1, acc_to_float(a1[v + 1]), fmaf(-s0, acc_to_float(a0[v + 1]), r[V + 1]));
              q[(e >> 1) & 1] = fmaf(w0, w0, q[(e >> 1) & 1]);
              q[(e >> 1) & 1] = fmaf(w1, w1, q[(e >> 1) & 1]);
            }
            p[kk] = q[0] + q[1];                   // added at once: half 0 keeps 4 values live, not 8
          }
        }
        for (int i = 0; i < np; ++i) {
          warp_arrive(&S.empty[stage], lane);
          if (++stage == nst) { stage = 0; phase ^= 1; }
        }
      } else if constexpr (kX8) {
        // Group gi is the K32 slab gi of the candidate's activation rows (ring stage gi / 4, 32 * (gi % 4) bytes in) against
        // the same slab of the resident weight tile, accumulated from zero.  Per group: one wgmma, its wait, the
        // epilogue; nothing is read from the job list and no count is dispatched at run time.  The operations per value
        // are those of the run() path: r = fmaf(-s, acc, r) per candidate group in group order, then
        // (g * fmaf(-s, acc, r))^2 for the last group.
        // A group's 8 scales candA[c][k] * candB[gi][k] come from four 16-byte shared loads.  (With the candidate's candA
        // row held in registers across its groups instead, ptxas -v reports 28 bytes of spill stores.)
        const int G = P.n_cand_groups;
        auto scales = [&](const int gi, float (&s)[P4V_TILE_CG]) {
          const float4* const a4 = reinterpret_cast<const float4*>(S.candA[c]);
          const float4* const b4 = reinterpret_cast<const float4*>(S.candB[gi]);
          const float4 a0 = a4[0], a1 = a4[1], b0 = b4[0], b1 = b4[1];
          const float a[P4V_TILE_CG] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
          const float b[P4V_TILE_CG] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
          const bool noA = (P.cand_noA_mask >> gi) & 1ull;
#pragma unroll
          for (int k = 0; k < P4V_TILE_CG; ++k) s[k] = noA ? b[k] : a[k] * b[k];
        };
        auto mma = [&](const uint32_t a16, const uint32_t b16) {
          wg_fence();
          wgmma_k32(acc, dconst | (uint64_t)a16, dconst | (uint64_t)b16, 0u);
          wg_commit();
          pc.skip();
          wg_wait0();
          pc.lap(kPhWgWait);
        };
        auto cand_epilogue = [&](const int gi) {
          pc.skip();
          float s[P4V_TILE_CG];
          scales(gi, s);
#pragma unroll
          for (int k = 0; k < P4V_TILE_CG; ++k)
#pragma unroll
            for (int e = 0; e < 8; ++e) r[8 * k + e] = fmaf(-s[k], acc_to_float(acc[8 * k + e]), r[8 * k + e]);
          pc.lap(kPhCand);
        };
        auto wait_stage = [&]() -> uint32_t {                // the stage's row slab, in 16-byte units
          pc.skip();
          mbar_wait_addr(full0 + stage * 8, phase);
          pc.lap(kPhFull);
          return ringR16 + stage * sR16;
        };
        int gi = 0;
        for (; gi + 4 < G; gi += 4) {                          // stages of four candidate groups
          const uint32_t a16 = wait_stage(), b16 = x8_b16 + 256 * gi;   // +32 bytes of K = 256 16-byte units
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            mma(a16 + 256 * q, b16 + 256 * q);
            if (q == 3) warp_arrive(&S.empty[stage], lane);
            cand_epilogue(gi + q);
          }
          if (++stage == nst) { stage = 0; phase ^= 1; }
        }
        {                                                     // the last stage: groups gi .. G - 1, the last one final
          const uint32_t a16 = wait_stage(), b16 = x8_b16 + 256 * gi;
          const int nq = G - gi;
          for (int q = 0; q + 1 < nq; ++q) {
            mma(a16 + 256 * q, b16 + 256 * q);
            cand_epilogue(gi + q);
          }
          mma(a16 + 256 * (nq - 1), b16 + 256 * (nq - 1));
          warp_arrive(&S.empty[stage], lane);
          if (++stage == nst) { stage = 0; phase ^= 1; }
          // the scales one column group at a time, from shared memory: the 64 g loads in flight leave no room for 8 more
          // live registers
          pc.skip();
          const bool noA = (P.cand_noA_mask >> (G - 1)) & 1ull;
#pragma unroll
          for (int k = 0; k < P4V_TILE_CG; ++k) {
            const float s = noA ? S.candB[G - 1][k] : S.candA[c][k] * S.candB[G - 1][k];
            float q[2] = {0.f, 0.f};
#pragma unroll
            for (int e = 0; e < 8; e += 2) {
              const int v = 8 * k + e;
              const float2 gv = gpair_x8(v);
              const float w0 = gv.x * fmaf(-s, acc_to_float(acc[v]), r[v]);
              const float w1 = gv.y * fmaf(-s, acc_to_float(acc[v + 1]), r[v + 1]);
              q[(e >> 1) & 1] = fmaf(w0, w0, q[(e >> 1) & 1]);
              q[(e >> 1) & 1] = fmaf(w1, w1, q[(e >> 1) & 1]);
            }
            ph[k][0] = q[0]; ph[k][1] = q[1];
          }
          pc.lap(kPhFinal);
        }
      } else {
        int gi = 0;
        for (int jj = 0; jj < P.n_cand_jobs; ++jj) {
          const P4VJob jb = S.jobs[P.n_fixed_jobs + jj];
          run(jb, res16 + (jb.res_off >> 4) + wg * 64, [&] {
            pc.skip();
            const bool noA = (P.cand_noA_mask >> gi) & 1ull;
            if (gi + 1 < P.n_cand_groups) {
              if constexpr (kMulti) {
#pragma unroll
                for (int k = 0; k < P4V_TILE_CG; ++k) {
                  const float s = noA ? S.candB[gi][k] : S.candA[c][k] * S.candB[gi][k];
#pragma unroll
                  for (int e = 0; e < 8; ++e) r[8 * k + e] = fmaf(-s, acc_to_float(acc[8 * k + e]), r[8 * k + e]);
                }
              }
              pc.lap(kPhCand);
            } else {
              // final segment: (g * (r - s*acc))^2; r itself is not modified
#pragma unroll
              for (int k = 0; k < P4V_TILE_CG; ++k) {
                const float s = noA ? S.candB[gi][k] : S.candA[c][k] * S.candB[gi][k];
                float q[2] = {0.f, 0.f};
#pragma unroll
                for (int e = 0; e < 8; e += 2) {
                  const int v = 8 * k + e;
                  const float2 gv = gpair(v);
                  const float w0 = gv.x * fmaf(-s, acc_to_float(acc[v]), r[v]);
                  const float w1 = gv.y * fmaf(-s, acc_to_float(acc[v + 1]), r[v + 1]);
                  q[(e >> 1) & 1] = fmaf(w0, w0, q[(e >> 1) & 1]);
                  q[(e >> 1) & 1] = fmaf(w1, w1, q[(e >> 1) & 1]);
                }
                ph[k][0] = q[0]; ph[k][1] = q[1];
              }
              pc.lap(kPhFinal);
            }
            ++gi;
          });
        }
      }
      if (!kPair && !kX8 && P.row_keys) {
        // one score per ROW (channel-wise conv search): [tile][candidate][column half][128 rows].  The quad of lanes
        // holding rows (frow, frow + 8) reduces its four (row, column half) totals and scatters them over its lanes.
        float k4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < P4V_TILE_CG; ++k) { k4[(k >> 2) * 2] += ph[k][0]; k4[(k >> 2) * 2 + 1] += ph[k][1]; }
        const bool hi2 = lane & 2, hi1 = lane & 1;
        const float a0 = (hi2 ? k4[2] : k4[0]) + __shfl_xor_sync(0xffffffffu, hi2 ? k4[0] : k4[2], 2);
        const float a1 = (hi2 ? k4[3] : k4[1]) + __shfl_xor_sync(0xffffffffu, hi2 ? k4[1] : k4[3], 2);
        const float tot = (hi1 ? a1 : a0) + __shfl_xor_sync(0xffffffffu, hi1 ? a0 : a1, 1);
        P.partial[((size_t)f.tile * P.n_cand + c) * 256 + (hi2 ? P4V_TILE : 0) + frow + (hi1 ? 8 : 0)] = tot;
        continue;
      }
      // per warp: totals of its 16 rows per column group; the two warps of a quarter add theirs every kRedBatch candidates
      pc.skip();
      if constexpr (!kPair) {
#pragma unroll
        for (int k = 0; k < P4V_TILE_CG; ++k) p[k] = ph[k][0] + ph[k][1];
      }
      const float tot = reduce8_over_warp(p, lane);
      float* const rbase = red + (size_t)(rb * 4 + quarter) * kRedBatch * 2 * P4V_TILE_CG;
      if ((lane & 3) == 0) rbase[(nb * 2 + (cw & 1)) * P4V_TILE_CG + (lane >> 2)] = tot;
      if (++nb == kRedBatch || c + 1 == f.c1) {
        asm volatile("bar.sync %0, 64;" ::"r"(2 + quarter));
        const int t64 = (cw & 1) * 32 + lane, j = t64 >> 3, k = t64 & 7;
        if (j < nb)
          P.partial[((size_t)f.tile * P.n_cand + (c + 1 - nb + j)) * 32 + quarter * 8 + k] =
              rbase[(j * 2) * P4V_TILE_CG + k] + rbase[(j * 2 + 1) * P4V_TILE_CG + k];
        rb ^= 1; nb = 0;
      }
      pc.lap(kPhReduce);
    }
    if (resB) {
      warp_arrive(&S.res_empty[rbuf], lane);       // every MMA reading the resident buffer has completed
      if (++rbuf == P.resident_bufs) { rbuf = 0; rphase ^= 1; }
    }
    if (cresB) warp_arrive(&S.cres_empty, lane);
  }
  pc.flush(kPhaseKind, kPhConsumer, lane == 0 && (cw & 3) == 0);
}

}  // namespace

#ifdef P4V_SWEEP_PHASE_CLOCKS
// Phase clocks since the last reset: out[kernel][phase] (kernel = 3 * int8 + consumer mode, phases in kPh* order), clock64
// cycles summed over consumer warp 0 of each warpgroup (consumer phases) or the producer warp (kPhEmpty, kPhProducer)
// of every CTA.
extern "C" __attribute__((visibility("default"))) int p4v_sweep_phase_clocks(unsigned long long* out, int reset) {
  P4V_CUDA_OK(cudaDeviceSynchronize());
  P4V_CUDA_OK(cudaMemcpyFromSymbol(out, g_sweep_phases, sizeof(g_sweep_phases)));
  if (reset) {
    static const unsigned long long zero[6][kPhases] = {};
    P4V_CUDA_OK(cudaMemcpyToSymbol(g_sweep_phases, zero, sizeof(zero)));
  }
  return 0;
}
#endif

int p4v_launch_sweep_tc(const SweepParams& p_in, const P4VJob* host_jobs, int num_sms, cudaStream_t st,
                        P4VLaunchDecision* decision) {
  SweepParams p = p_in;
  const int n_jobs = p.n_fixed_jobs + p.n_cand_jobs;
  P4V_REQUIRE(n_jobs <= P4V_MAX_JOBS, "sweep: too many jobs (%d)", n_jobs);
  P4V_REQUIRE(p.n_fixed_groups <= P4V_MAX_GROUPS && p.n_cand_groups <= P4V_MAX_GROUPS, "sweep: too many segment groups");
  P4V_REQUIRE(p.n_cand <= P4V_MAX_CAND && p.n_cand >= 1, "sweep: bad candidate count");
  P4V_REQUIRE(p.out != nullptr ? (p.n_cand == 1 && p.n_cand_jobs == 0) : p.n_cand_groups >= 1, "sweep: bad mode");
  P4V_REQUIRE(!p.row_keys || (p.n_cand_groups == 1 && p.out == nullptr), "sweep: per-row scores need a single-segment step");
  P4V_REQUIRE(!p.res || (p.out && !p.out_residual && p.is_int8 &&
                         ((reinterpret_cast<uintptr_t>(p.res) | reinterpret_cast<uintptr_t>(p.out)) & 7) == 0),
              "sweep: a residual needs an int8 forward with 8-byte aligned out and residual");
  const long long tiles = (long long)p.P * p.tiles_m * p.tiles_n;
  const long long units = tiles * p.n_cand;
  int grid = (int)(units < num_sms ? units : num_sms);
  if (grid < 1) return 0;
  // smem plan: stage size = largest job; resident row operand when the host marked the candidate jobs P4V_JOB_RRES
  uint32_t max_kb = 32, res_bytes = 0;
  bool any_r_stream = false, any_c_stream = false, any_cres = false;
  for (int j = 0; j < n_jobs; ++j) {
    const uint32_t kb_total = host_jobs[j].kb * p4v_job_nsub(host_jobs[j]);
    P4V_REQUIRE(host_jobs[j].kb % 32 == 0 && kb_total >= 32 && kb_total <= P4V_JOB_KB, "sweep: bad job size");
    if (kb_total > max_kb) max_kb = kb_total;
    if (host_jobs[j].flags & P4V_JOB_RRES) res_bytes = std::max(res_bytes, host_jobs[j].res_off + kb_total * P4V_TILE);
    else any_r_stream = true;
    if (host_jobs[j].flags & P4V_JOB_CRES) any_cres = true; else any_c_stream = true;
  }
  p.stage_r_bytes = any_r_stream ? max_kb * P4V_TILE : 0;
  p.stage_c_bytes = any_c_stream ? max_kb * P4V_TILE : 0;
  p.resident_bytes = res_bytes;
  p.cres_bytes = any_cres ? (unsigned int)p.C_tile_bytes : 0;
  P4V_REQUIRE(p.cres_bytes % 16 == 0 && p.cres_bytes <= 128 * 1024, "sweep: resident column image too large");
  const uint32_t per_stage = p.stage_r_bytes + p.stage_c_bytes;
  P4V_REQUIRE(per_stage > 0, "sweep: no streamed operand");
  const bool single = p.n_cand_groups == 1 && p.out == nullptr;
  const long long red_bytes = p.out != nullptr ? 0 : kRedBytes + kTileBytes;   // score reduction, parked g / residual tile
  p.resident_bufs = 2;                      // double buffered when that leaves a useful ring, else one buffer (a bubble per tile)
  if ((kSmemBudget - 2 * (long long)res_bytes - red_bytes - (long long)p.cres_bytes) / per_stage < 3) p.resident_bufs = 1;
  int nst = (int)((kSmemBudget - (long long)p.resident_bufs * res_bytes - red_bytes - (long long)p.cres_bytes) / per_stage);
  if (nst > kMaxStages) nst = kMaxStages;
  P4V_REQUIRE(nst >= 2, "sweep: operand tiles do not fit the shared-memory ring");
  p.n_stages = nst;
  const size_t smem = (size_t)nst * per_stage + (size_t)p.resident_bufs * res_bytes + p.cres_bytes + ((sizeof(SmemCtl) + 127) & ~size_t(127)) + (size_t)red_bytes + 256;
  P4V_REQUIRE(smem <= 227 * 1024, "sweep: shared-memory plan too large (%zu bytes)", smem);
  // Pair step: two candidate groups whose jobs i and i + n/2 multiply the same candidate column slab (same offsets and
  // flags, one accumulator each) with two resident row parts, each half one accumulator chain.  The pair consumer holds
  // a candidate's n/2 stages at once, so the ring must have one more.  P4V_NO_PAIR=1 keeps such steps on the
  // multi-segment path (A/B comparison).
  bool pair = false;
  if (!single && p.out == nullptr && p.n_cand_groups == 2 && p.n_cand_jobs % 2 == 0 && p.n_cand_jobs / 2 + 1 <= nst &&
      getenv("P4V_NO_PAIR") == nullptr) {
    const int np = p.n_cand_jobs / 2;
    const P4VJob* cj = host_jobs + p.n_fixed_jobs;
    pair = true;
    for (int i = 0; i < np; ++i) {
      const P4VJob &a = cj[i], &b = cj[np + i];
      const uint32_t need = P4V_JOB_CCAND | P4V_JOB_RRES;
      pair = pair && a.c_off == b.c_off && a.kb == b.kb && p4v_job_nsub(a) == 1 && p4v_job_nsub(b) == 1 &&
             a.flags == b.flags && (a.flags & (need | P4V_JOB_RCAND | P4V_JOB_CRES)) == need &&
             ((a.flags & P4V_JOB_FIRST) != 0) == (i == 0) && ((a.flags & P4V_JOB_LAST) != 0) == (i + 1 == np);
    }
  }
  const int mode = single ? kModeSingle : pair ? kModePair : kModeMulti;
  // The int8 activation step of a bf16 layer (build_plan's x8 jobs) runs the multi-segment arithmetic on its own loop
  // (kModeX8): no fixed groups, and candidate job j is groups 4j .. 4j + 3 (fewer in the last job), K32 slabs that
  // follow each other in both operand images, the activation slab from the candidate plane, the weight slab from the
  // tile's resident image, each slab its own accumulator.  Its launches are reported as multi-segment.
  bool x8 = false;
  if (mode == kModeMulti && p.is_int8 && !p.row_keys && p.n_fixed_jobs == 0 && p.n_cand_groups >= 2 &&
      p.n_cand_jobs == (p.n_cand_groups + 3) / 4) {
    const P4VJob* cj = host_jobs;
    const uint32_t flags = P4V_JOB_FIRST | P4V_JOB_LAST | P4V_JOB_RCAND | P4V_JOB_CRES;
    x8 = true;
    for (int j = 0; j < p.n_cand_jobs; ++j)
      x8 = x8 && cj[j].flags == flags && cj[j].kb == 32 &&
           p4v_job_nsub(cj[j]) == (unsigned)std::min(4, p.n_cand_groups - 4 * j) && cj[j].group == 4 * j &&
           cj[j].r_off == cj[0].r_off + j * 4 * 32 * P4V_TILE && cj[j].c_off == cj[0].c_off + j * 4 * 32 * P4V_TILE;
  }
  if (decision) *decision = P4VLaunchDecision{mode, nst, (int)p.resident_bufs, p.resident_bytes, p.cres_bytes, grid};
#define P4V_LAUNCH(I8, MODE)                                                                           \
  do {                                                                                                 \
    P4V_CUDA_OK(cudaFuncSetAttribute(sweep_tc_kernel<I8, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    sweep_tc_kernel<I8, MODE><<<grid, kThreads, smem, st>>>(p);                                        \
  } while (0)
#define P4V_LAUNCH_MODE(I8)                                                                            \
  do {                                                                                                 \
    if (mode == kModeSingle) P4V_LAUNCH(I8, kModeSingle);                                              \
    else if (mode == kModePair) P4V_LAUNCH(I8, kModePair);                                             \
    else P4V_LAUNCH(I8, kModeMulti);                                                                   \
  } while (0)
  if (p.res)          P4V_LAUNCH(true, kModeFwdRes);
  else if (x8)        P4V_LAUNCH(true, kModeX8);
  else if (p.is_int8) P4V_LAUNCH_MODE(true);
  else                P4V_LAUNCH_MODE(false);
#undef P4V_LAUNCH_MODE
#undef P4V_LAUNCH
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}
