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
// The kernel is a template on the fold mask of forward.cuh; each fold adds to the plain forward above (DESIGN §4.5):
// P4V_FOLD_MLP: the same kernel is fc1 of a fused frozen MLP: step 2's epilogue applies torch's GELU and fc2's activation
//   quantiser and writes fc2's int8 activation image instead of FP32 (see the epilogue below, DESIGN §4.8).
// P4V_FOLD_NORM: a LayerNorm is folded into step 1: the CTA first computes each row's mean and rstd with torch's exact
//   reduction (forward.cuh, p4v_ln_row_stats) and the quantise loop normalises every value before quantising it
//   (DESIGN §4.10).
// P4V_FOLD_RES: a block's residual add is folded into the FP32 store: each value goes to its destination row (the
//   identity, or Swin's window reverse and reverse shift, p4v_window_row) as fl(value + shortcut) (DESIGN §4.11).
// P4V_FOLD_GATHER (with NORM): the LayerNorm prologue and the quantise loop read each row from elsewhere in an image:
//   Swin's shifted window partition (p4v_window_row) or PatchMerging's 2x2 neighbourhood (p4v_merge_row) (DESIGN §4.12).
// P4V_FOLD_QKV8: the layer is an attention block's qkv; the epilogue quantises q, k and v with the attention's step sizes
//   and stores them as the int8 planes the attention kernel reads, instead of the FP32 output (DESIGN §4.14).
// p4v_launch_forward_tc instantiates the nine fold sets the host uses: none, MLP, NORM, MLP|NORM, RES, NORM|GATHER, QKV8,
// NORM|QKV8 and NORM|GATHER|QKV8.
// 288 threads leave 224 registers per thread without setmaxnreg; the bounded mbarrier wait is inline, and the k32 steps of
// a stage are one straight-line batch selected by a warp-uniform count (ptxas C7520, see sm90.cuh).
#include "../../include/ptq4vit_b200.h"
#include "forward.cuh"
#include "sm90.cuh"

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

// 16 quantised values -> one 16-byte chunk of int8
__device__ __forceinline__ void pack16(uint32_t (&w)[4], int e, float q) {
  w[e >> 2] |= (uint32_t)((int)q & 0xff) << ((e & 3) * 8);
}

// ---- the epilogue of mlp_fc1_kernel: GELU, fc2's activation quantiser, fc2's image --------------------------------
// Shared memory: [staged tile: planes2 x 128 rows x P4V_MLP_STAGE_LD][step size, reciprocal of the 128 columns][chunk table]
// The bytes of a 16-byte chunk of fc2's image have source columns that need not lie in one 128-column tile of fc1 (a
// segment of fc2 may start anywhere), and the column tiles of a row tile may belong to different CTAs.  A byte belongs
// to the column tile of its source column; a padding byte to that of its segment's last column.  Every byte of the image
// then has exactly one owner, and a CTA stores whole chunks it owns as one 16-byte store and the owned bytes of a chunk
// that straddles two column tiles one by one.
__device__ __forceinline__ uint8_t* mlp_epi(const FwdParams& P, uint8_t* smem) {
  return smem + P.a_bytes + (size_t)P.n_stages * P.stage_bytes;
}
__device__ __forceinline__ float* mlp_steps(const FwdParams& P, uint8_t* epi) {
  return reinterpret_cast<float*>(epi + P.planes2 * P4V_TILE * P4V_MLP_STAGE_LD);
}
__device__ __forceinline__ P4VMlpChunk* mlp_chunks(const FwdParams& P, uint8_t* epi) {
  return reinterpret_cast<P4VMlpChunk*>(mlp_steps(P, epi) + 2 * P4V_TILE);
}

// fc2's chunk table (one plane of a row of its image), by the whole CTA before the setup barrier
__device__ __forceinline__ void mlp_chunk_table(const FwdParams& P, uint8_t* epi) {
  P4VMlpChunk* tab = mlp_chunks(P, epi);
  for (int s = threadIdx.x; s < P.nseg2; s += kThreads) {
    const P4VSeg sg = P.segs2[s];
    const int c0 = sg.dst_off / (P4V_TILE * 16), nch = ((sg.klen + 31) / 32) * 2, last = sg.k0 + sg.klen - 1;
    for (int c = 0; c < nch; ++c) tab[c0 + c] = P4VMlpChunk{min(sg.k0 + 16 * c, last), max(0, min(16, sg.klen - 16 * c))};
  }
}

// fc2's step size of each column of tile tn and its reciprocal (0 where p4v_rint_div_ok fails: the exact division), by
// the consumers between the barriers that open a column tile
__device__ __forceinline__ void mlp_column_steps(const FwdParams& P, uint8_t* epi, int tn, int et) {
  float* d = mlp_steps(P, epi);
  for (int lc = et; lc < P4V_TILE; lc += kConsumers) {
    const int col = tn * P4V_TILE + lc;
    const float delta = col < P.N ? __ldg(P.dX2 + col / P.crb_acts2) : 1.f;
    d[lc] = delta;
    d[P4V_TILE + lc] = p4v_rint_div_ok(delta) ? __frcp_rn(delta) : 0.f;
  }
}

// The thread's 64 fc1 values (r = -value, fragment layout of forward_tc_body) -> GELU -> fc2's bytes, staged by column
// (quant_image_kernel's sequence for fc2's segments: p4v_quant_plain, the negative plane with d_neg, NaN -> 0)
__device__ __forceinline__ void mlp_stage_tile(const FwdParams& P, uint8_t* epi, const float (&r)[64], int frow, int fcol) {
  const float* d = mlp_steps(P, epi);
  const float rcp_neg = __frcp_rn(P.d_neg2), rcp_neg_scalar = __fdiv_rn(1.f, P.d_neg2);
  const bool fast_neg = p4v_rint_div_ok(P.d_neg2), twin = P.planes2 == 2;
#pragma unroll
  for (int v = 0; v < 64; v += 2) {
    const int row = frow + 8 * ((v >> 1) & 1), lc = fcol + 8 * (v >> 2);
    uint32_t bp = 0u, bn = 0u;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const float g = p4v_gelu(-r[v + t]);
      const float rcp = d[P4V_TILE + lc + t];
      bp |= p4v_qbyte(p4v_quant_plain(g, d[lc + t], rcp != 0.f, rcp, false, 0.f, P.lo2, P.hi2)) << (8 * t);
      if (twin) bn |= p4v_qbyte(p4v_quant_plain(g, P.d_neg2, fast_neg, rcp_neg, !P.ieee_div, rcp_neg_scalar, P.neg_lo2, 0.f)) << (8 * t);
    }
    uint8_t* st = epi + row * P4V_MLP_STAGE_LD + lc;
    *reinterpret_cast<uint16_t*>(st) = (uint16_t)bp;
    if (twin) *reinterpret_cast<uint16_t*>(st + P4V_TILE * P4V_MLP_STAGE_LD) = (uint16_t)bn;
  }
}

// The bytes of fc2's image that column tile tn of row tile tm owns, from the staged tile; rows past M are zeros
__device__ __forceinline__ void mlp_store_tile(const FwdParams& P, uint8_t* epi, int tm, int tn, int et) {
  const P4VMlpChunk* tab = mlp_chunks(P, epi);
  const int c0 = tn * P4V_TILE, c1 = min(c0 + P4V_TILE, P.N);
  // the chunks with a byte in [c0, c1): kf and the owner of the last byte grow with the chunk index
  int lo = 0, hi = P.n_chunks2;
  while (lo < hi) { const int m = (lo + hi) >> 1; const P4VMlpChunk c = tab[m]; if (c.kf + max(c.n - 1, 0) >= c0) hi = m; else lo = m + 1; }
  const int cb = lo;
  hi = P.n_chunks2;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (tab[m].kf >= c1) hi = m; else lo = m + 1; }
  const int nc = lo - cb;
  for (int u = et; u < P.planes2 * nc * P4V_TILE; u += kConsumers) {
    const int r = u & (P4V_TILE - 1), pc = u >> 7, plane = pc / nc, c = cb + pc % nc;
    const P4VMlpChunk ch = tab[c];
    const bool in = tm * P4V_TILE + r < P.M;
    const uint8_t* srow = epi + (plane * P4V_TILE + r) * P4V_MLP_STAGE_LD - c0;   // indexed by source column
    uint8_t* dst = P.X2 + (size_t)tm * P.X2_tile_bytes + (size_t)plane * P.X2_plane_bytes + ((size_t)c * P4V_TILE + r) * 16;
    if (ch.n == 16 && ch.kf >= c0 && ch.kf + 16 <= c1 && ((ch.kf - c0) & 15) == 0) {
      *reinterpret_cast<uint4*>(dst) = in ? *reinterpret_cast<const uint4*>(srow + ch.kf) : make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    const int kl = ch.kf + max(ch.n - 1, 0);
    uint32_t w[4] = {0u, 0u, 0u, 0u}, own = 0u;
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      const int k = e < ch.n ? ch.kf + e : kl;
      if (k >= c0 && k < c1) {
        own |= 1u << e;
        if (e < ch.n && in) w[e >> 2] |= (uint32_t)srow[k] << ((e & 3) * 8);
      }
    }
    if (own == 0xffffu) {
      *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
#pragma unroll
      for (int e = 0; e < 16; ++e)
        if ((own >> e) & 1u) dst[e] = (uint8_t)(w[e >> 2] >> ((e & 3) * 8));
    }
  }
}

// The LayerNorm prologue's row stats, the last P4V_NORM_STATS_BYTES before the control block: mean [128], then rstd [128]
__device__ __forceinline__ float* ln_stats(const FwdParams& P, unsigned folds, uint8_t* smem) {
  return reinterpret_cast<float*>(smem + P.a_bytes + (size_t)P.n_stages * P.stage_bytes +
                                  (p4v_fwd_extra_bytes(folds, P.epi_bytes) - P4V_NORM_STATS_BYTES));
}

// ---- the row gather of P4V_FOLD_GATHER (DESIGN §4.12) ----------------------------------------------------------------
// The source row of each tile row, right below the row stats: the window map's image row, or the merge's first row
__device__ __forceinline__ int* gather_rows(const FwdParams& P, unsigned folds, uint8_t* smem) {
  return reinterpret_cast<int*>(ln_stats(P, folds, smem)) - P4V_TILE;
}

// Mean and rstd of tile row r (global row `row`), read from its source rows; returns the source row
__device__ __forceinline__ int gather_row_stats(const FwdParams& P, int row, int lane, float& mean, float& rstd) {
  const int K = (int)P.ld;
  if (P.ga.mode == P4V_GATHER_WINDOW) {
    const int s = p4v_window_row(P.ga.win, row);
    p4v_ln_row_stats(P.x + (size_t)s * K, K, P.ln.eps, lane, mean, rstd);
    return s;
  }
  // merge: float4 i of the 4C row lies in quarter i / (C / 4), since C % 4 == 0
  const int s = p4v_merge_row(P.ga.win, row), c4 = K >> 4;
  const float4* x4 = reinterpret_cast<const float4*>(P.x);
  const p4v_window_layout win = P.ga.win;
  p4v_ln_row_stats_at([=](int i) {
    const int q = i / c4;
    return x4 + (size_t)(s + p4v_merge_quarter(win, q)) * c4 + (i - q * c4);
  }, K, P.ln.eps, lane, mean, rstd);
  return s;
}

// The chunk's FP32 values (ch.n of them, zeros after) of the tile row whose source row is s.  A merge chunk inside one
// quarter reads like a contiguous row; one that straddles two quarters (C % 16 != 0) reads element by element.
__device__ __forceinline__ void gather_chunk(const FwdParams& P, int s, int k0, int n, float (&vals)[16]) {
  const int K = (int)P.ld;
  const float* src;
  if (P.ga.mode == P4V_GATHER_WINDOW) {
    src = P.x + (size_t)s * K + k0;
  } else {
    const int C = K >> 2, q = k0 / C, c = k0 - q * C;
    if (c + n > C) {
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        const int k = k0 + e, qe = k / C;
        vals[e] = e < n ? __ldg(P.x + (size_t)(s + p4v_merge_quarter(P.ga.win, qe)) * C + (k - qe * C)) : 0.f;
      }
      return;
    }
    src = P.x + (size_t)(s + p4v_merge_quarter(P.ga.win, q)) * C + c;
  }
  if (n == 16 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    const float4* src4 = reinterpret_cast<const float4*>(src);
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float4 t4 = __ldg(src4 + e); vals[4 * e] = t4.x; vals[4 * e + 1] = t4.y; vals[4 * e + 2] = t4.z; vals[4 * e + 3] = t4.w; }
  } else {
#pragma unroll
    for (int e = 0; e < 16; ++e) vals[e] = e < n ? __ldg(src + e) : 0.f;
  }
}

// ---- the qkv epilogue of P4V_FOLD_QKV8 (DESIGN §4.14) ---------------------------------------------------------------
// Shared memory, in the place of the MLP epilogue's: [staged bytes: 128 rows x P4V_MLP_STAGE_LD][a Qkv8Group per 16-column
// group of the column tile].  A 16-byte chunk of a plane row is one 16-column group of one output row of one column tile,
// so every byte of the planes has exactly one owner and is stored in a whole 16-byte store.
struct Qkv8Group { float d, rcp, lo, hi; int scaled, pad; long long off; };   // off: planes + off + (b * heads * N + n) * D
__device__ __forceinline__ Qkv8Group* qkv8_groups(uint8_t* epi) {
  return reinterpret_cast<Qkv8Group*>(epi + P4V_TILE * P4V_MLP_STAGE_LD);
}

// The step size, reciprocal, clamp range, q-scaling and (part, head, j) offset of each 16-column group of tile tn, by the
// consumers between the barriers that open a column tile
__device__ __forceinline__ void qkv8_column_groups(const FwdParams& P, uint8_t* epi, int tn, int et) {
  if (et >= P4V_TILE / 16) return;
  const FwdQkv8& Q = P.q8;
  const int c = tn * P4V_TILE + 16 * et;
  Qkv8Group g{1.f, 1.f, 0.f, 0.f, 0, 0, 0};
  if (c < P.N) {
    const int part = c / Q.C, h = (c - part * Q.C) / Q.D, j = c - part * Q.C - h * Q.D;
    g.d = __ldg((part == 0 ? Q.dq : part == 1 ? Q.dk : Q.dv) + h);
    g.rcp = p4v_rint_div_ok(g.d) ? __frcp_rn(g.d) : 0.f;
    g.lo = part == 0 ? Q.q_lo : part == 1 ? Q.k_lo : Q.v_lo;
    g.hi = part == 0 ? Q.q_hi : part == 1 ? Q.k_hi : Q.v_hi;
    g.scaled = part == 0 && Q.scale_on_q;
    g.off = ((long long)part * Q.batch * Q.heads + h) * Q.N * Q.D + j;     // [part][b = 0][h][n = 0][j]
  }
  qkv8_groups(epi)[et] = g;
}

// The thread's 64 qkv values (r = -value, fragment layout of forward_tc_body) -> the attention kernel's bytes, staged by
// column: p4v_qbyte(p4v_quant_plain(...)) with the arguments of forward_attn_tc.cu's loaders
__device__ __forceinline__ void qkv8_stage_tile(const FwdParams& P, uint8_t* epi, const float (&r)[64], int frow, int fcol) {
  const Qkv8Group* grp = qkv8_groups(epi);
#pragma unroll
  for (int v = 0; v < 64; v += 2) {
    const int row = frow + 8 * ((v >> 1) & 1), lc = fcol + 8 * (v >> 2);
    const Qkv8Group g = grp[lc >> 4];
    uint32_t b = 0u;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const float y = -r[v + t];
      const float xs = g.scaled ? __fmul_rn(y, P.q8.scale) : y;
      b |= p4v_qbyte(p4v_quant_plain(xs, g.d, p4v_rint_div_ok(g.d), g.rcp, false, 0.f, g.lo, g.hi)) << (8 * t);
    }
    *reinterpret_cast<uint16_t*>(epi + row * P4V_MLP_STAGE_LD + lc) = (uint16_t)b;
  }
}

// The planes' 16-byte chunks of row tile tm and column tile tn from the staged tile: one (row, 16-column group) per
// item, groups fastest, so that a warp stores whole runs of a head's rows
__device__ __forceinline__ void qkv8_store_tile(const FwdParams& P, uint8_t* epi, int tm, int tn, int et) {
  const FwdQkv8& Q = P.q8;
  const Qkv8Group* grp = qkv8_groups(epi);
  const int ng = min(P4V_TILE, P.N - tn * P4V_TILE) / 16;
  for (int u = et; u < P4V_TILE * (P4V_TILE / 16); u += kConsumers) {
    const int g = u & 7, r = u >> 3, row = tm * P4V_TILE + r;
    if (g >= ng || row >= P.M) continue;
    const int b = row / Q.N, n = row - b * Q.N;
    uint8_t* dst = Q.planes + grp[g].off + ((long long)b * Q.heads * Q.N + n) * Q.D;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(epi + r * P4V_MLP_STAGE_LD + 16 * g);
  }
}

// kFolds = 0: the frozen Linear forward, FP32 output.  P4V_FOLD_MLP: fc1 of a frozen MLP, GELU-and-quantise epilogue
// into fc2's image.  P4V_FOLD_NORM: a LayerNorm prologue.  P4V_FOLD_RES: the plain forward whose store adds the
// shortcut.  P4V_FOLD_GATHER (with NORM): the LayerNorm's rows gathered from an image.
template <unsigned kFolds>
__global__ void __launch_bounds__(kThreads, 1) forward_tc_kernel(const __grid_constant__ FwdParams P) {
  constexpr bool kMlp = kFolds & P4V_FOLD_MLP;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  // carve: [resident activation tile][weight ring][MLP epilogue][LayerNorm row stats][control]
  const uint32_t nst = P.n_stages, sC = P.stage_bytes;
  const uint32_t resA = smem_u32(smem), ring = resA + P.a_bytes;
  FwdCtl& S = *reinterpret_cast<FwdCtl*>(smem + P.a_bytes + (size_t)nst * sC + p4v_fwd_extra_bytes(kFolds, P.epi_bytes));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // the CTA's row tile and its share of the column tiles
  const int csplit = gridDim.x / P.tiles_m;
  const int tm = blockIdx.x / csplit, cs = blockIdx.x % csplit;
  const int tn0 = cs * P.tiles_n / csplit, tn1 = (cs + 1) * P.tiles_n / csplit;

  // ---- LayerNorm prologue: mean and rstd of every row of the tile, one warp per row (released by the setup barrier) ----
  if constexpr ((kFolds & P4V_FOLD_NORM) != 0) {
    float* ln_mean = ln_stats(P, kFolds, smem);
    for (int r = warp; r < P4V_TILE; r += kThreads / 32) {
      const int row = tm * P4V_TILE + r;
      if (row >= P.M) break;
      float mean, rstd;
      if constexpr ((kFolds & P4V_FOLD_GATHER) != 0) {
        const int s = gather_row_stats(P, row, lane, mean, rstd);
        if (lane == 0) gather_rows(P, kFolds, smem)[r] = s;
      } else {
        p4v_ln_row_stats(P.x + (size_t)row * P.ld, (int)P.ld, P.ln.eps, lane, mean, rstd);
      }
      if (lane == 0) { ln_mean[r] = mean; ln_mean[P4V_TILE + r] = rstd; }
    }
  }

  // ---- setup: jobs, chunk table, barriers ----
  for (int i = threadIdx.x; i < P.n_jobs; i += kThreads) S.jobs[i] = P.jobs[i];
  for (int s = threadIdx.x; s < P.nseg; s += kThreads) {
    const P4VSeg sg = P.segs[s];
    const int c0 = sg.dst_off / (P4V_TILE * 16), nch = ((sg.klen + 31) / 32) * 2;      // every segment is padded to 32 B
    for (int c = 0; c < nch; ++c)
      S.chunks[c0 + c] = Chunk{sg.k0 + 16 * c, (short)max(0, min(16, sg.klen - 16 * c)), (short)sg.didx};
  }
  if constexpr (kMlp) mlp_chunk_table(P, mlp_epi(P, smem));
  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < nst; ++i) { mbar_init(&S.full[i], 1); mbar_init(&S.empty[i], kConsumerWarps); }
    fence_mbarrier_init();
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
        if constexpr ((kFolds & P4V_FOLD_GATHER) != 0) {
          gather_chunk(P, gather_rows(P, kFolds, smem)[r], ch.k0, ch.n, vals);
        } else {
          const float* src = P.x + (size_t)row * P.ld + ch.k0;
          if (ch.n == 16 && ((P.ld | ch.k0) & 3) == 0) {
            const float4* src4 = reinterpret_cast<const float4*>(src);
#pragma unroll
            for (int e = 0; e < 4; ++e) { const float4 t4 = __ldg(src4 + e); vals[4 * e] = t4.x; vals[4 * e + 1] = t4.y; vals[4 * e + 2] = t4.z; vals[4 * e + 3] = t4.w; }
          } else {
#pragma unroll
            for (int e = 0; e < 16; ++e) vals[e] = e < ch.n ? src[e] : 0.f;
          }
        }
        if constexpr ((kFolds & P4V_FOLD_NORM) != 0) {
          const float* ln_mean = ln_stats(P, kFolds, smem);
          const float mean = ln_mean[r], rstd = ln_mean[P4V_TILE + r];
          float g[16], b[16];
          if (ch.n == 16 && (ch.k0 & 3) == 0) {          // gamma and beta are 16-byte aligned at a multiple of 4
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float4 g4 = __ldg(reinterpret_cast<const float4*>(P.ln.gamma + ch.k0) + e);
              const float4 b4 = __ldg(reinterpret_cast<const float4*>(P.ln.beta + ch.k0) + e);
              g[4 * e] = g4.x; g[4 * e + 1] = g4.y; g[4 * e + 2] = g4.z; g[4 * e + 3] = g4.w;
              b[4 * e] = b4.x; b[4 * e + 1] = b4.y; b[4 * e + 2] = b4.z; b[4 * e + 3] = b4.w;
            }
          } else {
#pragma unroll
            for (int e = 0; e < 16; ++e) { g[e] = e < ch.n ? __ldg(P.ln.gamma + ch.k0 + e) : 0.f; b[e] = e < ch.n ? __ldg(P.ln.beta + ch.k0 + e) : 0.f; }
          }
#pragma unroll
          for (int e = 0; e < 16; ++e)
            if (e < ch.n) vals[e] = p4v_ln_apply(vals[e], mean, rstd, g[e], b[e]);
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
    fence_proxy_async();   // generic-proxy stores -> wgmma (async proxy) reads
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
  const uint64_t dconst = desc_const(P4V_TILE);
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
    if constexpr (kMlp) mlp_column_steps(P, mlp_epi(P, smem), tn, et);
    if constexpr ((kFolds & P4V_FOLD_QKV8) != 0) qkv8_column_groups(P, mlp_epi(P, smem), tn, et);
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
    if constexpr (kMlp) {
      mlp_stage_tile(P, mlp_epi(P, smem), r, frow, fcol);
      asm volatile("bar.sync 1, %0;" ::"n"(kConsumers));   // staged tile complete
      // the next column tile's first barrier orders these reads of the staging before it is written again
      mlp_store_tile(P, mlp_epi(P, smem), tm, tn, et);
    } else if constexpr ((kFolds & P4V_FOLD_QKV8) != 0) {
      qkv8_stage_tile(P, mlp_epi(P, smem), r, frow, fcol);
      asm volatile("bar.sync 1, %0;" ::"n"(kConsumers));   // staged tile complete
      // the next column tile's first barrier orders these reads of the staging before it is written again
      qkv8_store_tile(P, mlp_epi(P, smem), tm, tn, et);
    } else if constexpr ((kFolds & P4V_FOLD_RES) != 0) {
      // the residual add: out[dst] = fl(-r + res[dst]) (torch's FP32 add of the stored value and the shortcut), the
      // shortcut read at the destination rows as the pairs the plain store writes
      const bool pairs = (P.N & 1) == 0;
      const int d0 = gm < P.M ? p4v_window_row(P.rs.win, gm) : 0, d8 = gm + 8 < P.M ? p4v_window_row(P.rs.win, gm + 8) : 0;
#pragma unroll
      for (int v = 0; v < 64; v += 2) {
        const int row = gm + 8 * ((v >> 1) & 1), col = gc + 8 * (v >> 2);
        if (row < P.M) {
          const size_t off = (size_t)((v >> 1) & 1 ? d8 : d0) * P.N + col;
          float* o = P.out + off;
          const float* s = P.rs.res + off;
          if (pairs) {
            if (col < P.N) {
              const float2 sv = __ldg(reinterpret_cast<const float2*>(s));
              *reinterpret_cast<float2*>(o) = make_float2(__fadd_rn(-r[v], sv.x), __fadd_rn(-r[v + 1], sv.y));
            }
          } else {
            if (col < P.N) o[0] = __fadd_rn(-r[v], __ldg(s));
            if (col + 1 < P.N) o[1] = __fadd_rn(-r[v + 1], __ldg(s + 1));
          }
        }
      }
    } else {
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
}

__global__ void gelu_probe_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = p4v_gelu(x[i]);
}

}  // namespace

int p4v_launch_forward_tc(const FwdParams& p, unsigned folds, int num_sms, cudaStream_t st) {
  void (*kernel)(const FwdParams);
  switch (folds) {
    case 0: kernel = forward_tc_kernel<0>; break;
    case P4V_FOLD_MLP: kernel = forward_tc_kernel<P4V_FOLD_MLP>; break;
    case P4V_FOLD_NORM: kernel = forward_tc_kernel<P4V_FOLD_NORM>; break;
    case P4V_FOLD_MLP | P4V_FOLD_NORM: kernel = forward_tc_kernel<P4V_FOLD_MLP | P4V_FOLD_NORM>; break;
    case P4V_FOLD_RES: kernel = forward_tc_kernel<P4V_FOLD_RES>; break;
    case P4V_FOLD_NORM | P4V_FOLD_GATHER: kernel = forward_tc_kernel<P4V_FOLD_NORM | P4V_FOLD_GATHER>; break;
    case P4V_FOLD_QKV8: kernel = forward_tc_kernel<P4V_FOLD_QKV8>; break;
    case P4V_FOLD_NORM | P4V_FOLD_QKV8: kernel = forward_tc_kernel<P4V_FOLD_NORM | P4V_FOLD_QKV8>; break;
    case P4V_FOLD_NORM | P4V_FOLD_GATHER | P4V_FOLD_QKV8:
      kernel = forward_tc_kernel<P4V_FOLD_NORM | P4V_FOLD_GATHER | P4V_FOLD_QKV8>; break;
    default: P4V_REQUIRE(false, "forward: no kernel for the fold set 0x%x", folds);
  }
  if (folds & P4V_FOLD_MLP)
    P4V_REQUIRE(!p.twin && (p.planes2 == 1 || p.planes2 == 2) && p.epi_bytes == p4v_mlp_epi_bytes(p.planes2, p.n_chunks2) &&
                (reinterpret_cast<uintptr_t>(p.X2) & 15) == 0, "mlp forward: bad epilogue plan");
  if (folds & P4V_FOLD_NORM) P4V_REQUIRE(!p.twin && p.ld % 4 == 0 && p.ln.gamma && p.ln.beta, "forward: bad LayerNorm plan");
  if (folds & P4V_FOLD_RES) {
    const p4v_window_layout& w = p.rs.win;
    P4V_REQUIRE(p.rs.res && (reinterpret_cast<uintptr_t>(p.rs.res) & 7) == 0, "forward: residual must be 8-byte aligned");
    P4V_REQUIRE(w.window == 0 || ((long long)w.images * w.height * w.width == p.M && w.height % w.window == 0 &&
                                  w.width % w.window == 0 && w.shift >= 0 && w.shift < w.window), "forward: bad window layout");
  }
  if (folds & P4V_FOLD_GATHER) {
    const p4v_window_layout& w = p.ga.win;
    const bool window = p.ga.mode == P4V_GATHER_WINDOW && w.window > 0 && w.height % w.window == 0 &&
                        w.width % w.window == 0 && w.shift >= 0 && w.shift < w.window && p.ld % 4 == 0 &&
                        (long long)w.images * w.height * w.width == p.M;
    const bool merge = p.ga.mode == P4V_GATHER_MERGE && w.window == 0 && w.shift == 0 && w.height % 2 == 0 &&
                       w.width % 2 == 0 && p.ld % 16 == 0 && (long long)w.images * (w.height / 2) * (w.width / 2) == p.M;
    P4V_REQUIRE(w.images > 0 && w.height > 0 && w.width > 0 && (window || merge), "forward: bad gather layout");
  }
  if (folds & P4V_FOLD_QKV8) {
    const FwdQkv8& q = p.q8;
    P4V_REQUIRE(q.planes && (reinterpret_cast<uintptr_t>(q.planes) & 15) == 0 && q.dq && q.dk && q.dv,
                "forward: qkv planes must be 16-byte aligned");
    P4V_REQUIRE(q.D > 0 && q.D % 16 == 0 && q.heads > 0 && q.C == q.heads * q.D && p.N == 3 * q.C && q.N > 0 &&
                (long long)q.batch * q.N == p.M, "forward: bad qkv plane layout");
  }
  const unsigned extra = p4v_fwd_extra_bytes(folds, p.epi_bytes);
  P4V_REQUIRE(p.n_jobs >= 1 && p.n_jobs <= P4V_MAX_JOBS && p.n_groups <= P4V_MAX_GROUPS, "forward: too many K segments");
  P4V_REQUIRE(p.n_stages >= 2 && p.n_stages <= P4V_FWD_MAX_STAGES && p.n_chunks <= P4V_FWD_MAX_CHUNKS &&
              p.stage_bytes % 128 == 0 && p.a_bytes % 128 == 0 && extra % 128 == 0, "forward: bad shared-memory plan");
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(p.out) & 7) == 0 && (reinterpret_cast<uintptr_t>(p.x) & 15) == 0,
              "forward: x must be 16-byte and out 8-byte aligned");
  const size_t smem = (size_t)p.a_bytes + (size_t)p.n_stages * p.stage_bytes + extra + sizeof(FwdCtl) + 128;
  P4V_REQUIRE(smem <= P4V_FWD_SMEM, "forward: shared-memory plan too large (%zu bytes)", smem);
  // Fewer row tiles than SMs: split the column tiles of a row tile over several CTAs (each quantises the row tile again,
  // from L2) so that the whole GPU writes output.
  int csplit = num_sms / p.tiles_m;
  csplit = csplit < 1 ? 1 : (csplit > p.tiles_n ? p.tiles_n : csplit);
  P4V_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<p.tiles_m * csplit, kThreads, smem, st>>>(p);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}

// Diagnostic: y = p4v_gelu(x) elementwise (the GELU of mlp_fc1_kernel's epilogue)
extern "C" int p4v_gelu_probe(const float* x, float* y, long long n, void* stream) {
  P4V_REQUIRE(x && y && n >= 0, "gelu_probe: null pointer or negative count");
  if (n == 0) return 0;
  const long long blocks = (n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096;
  gelu_probe_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, y, n);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}

namespace {

// one warp per row
__global__ void layer_norm_probe_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                        const float* __restrict__ beta, float eps, long long M, int N, float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  for (long long row = blockIdx.x * (long long)(blockDim.x / 32) + (threadIdx.x >> 5); row < M;
       row += (long long)gridDim.x * (blockDim.x / 32)) {
    const float* xr = x + row * N;
    float mean, rstd;
    p4v_ln_row_stats(xr, N, eps, lane, mean, rstd);
    for (int k = lane; k < N; k += 32) y[row * N + k] = p4v_ln_apply(xr[k], mean, rstd, gamma[k], beta[k]);
  }
}

}  // namespace

// Diagnostic: y = LayerNorm(x) row by row for [M][N] x (the LayerNorm of the fused kernel's prologue)
extern "C" int p4v_layer_norm_probe(const float* x, const float* gamma, const float* beta, float eps, long long M, int N, float* y,
                                    void* stream) {
  P4V_REQUIRE(x && gamma && beta && y && M >= 0, "layer_norm_probe: null pointer or negative count");
  P4V_REQUIRE(N > 0 && N % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "layer_norm_probe: N must be a positive "
              "multiple of 4 and x 16-byte aligned");
  P4V_REQUIRE(eps >= 0.f && eps <= 3.4e38f, "layer_norm_probe: eps must be finite and non-negative");
  if (M == 0) return 0;
  const long long blocks = (M + 7) / 8 < 4096 ? (M + 7) / 8 : 4096;
  layer_norm_probe_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, gamma, beta, eps, M, N, y);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}
