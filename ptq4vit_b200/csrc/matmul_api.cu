// C-ABI for the head-wise MatMul scale-factor search (PTQSLBatchingQuantMatMul and the
// split-of-softmax variant).  Problem p = image * heads + head; the row operand is A[p]
// (S1 x S2), the column operand is B[p]^T (S3 x S2); one K segment (n_V = n_H = 1).
#include <algorithm>
#include <vector>

#include "../../include/ptq4vit_b200.h"
#include "prep.cuh"

void p4v_count_launch();
int p4v_run_sweep(const SweepParams& sp, const P4VJob* host_jobs, int kernel, cudaStream_t st);

namespace {

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
template <class T> T* at(void* ws, size_t off) { return reinterpret_cast<T*>(static_cast<uint8_t*>(ws) + off); }

struct MStep { int job_off, nfj, ncj, nfg, ncg, meta_fix, meta_cand; };

struct MMPlan {
  p4v_matmul_desc d;
  bool i8, sos;
  int ew, P, H, S1, S2, S3, tiles_m, tiles_n, A_qmax, B_qmax;
  int ipc;       // images per chunk (0: whole layer); the operand images hold Pc = ipc * heads problems
  int Pc;
  int kb;        // padded K bytes of one part in the search operand type
  int kb16;      // padded K bytes in bf16 (split-search images)
  int KB_A, KB_B;            // row bytes of Acur / Bcur  (sos: Acur = [hi|lo])
  int KB_As, KB_Bs;          // split search: Acand = [hi|lo] bf16, Bsplit = [b1|b2|b3] bf16
  std::vector<P4VJob> jobs; std::vector<GroupMeta> metas;
  std::vector<P4VSeg> segA, segB, segAs, segBs;
  MStep stepA, stepB, stepS, fwd;
  std::vector<float> factors, split_factors;
  int n_split;
  size_t o_factors, o_sfactors, o_keys, o_dA0, o_dA, o_dB0, o_dB, o_ones, o_aux, o_split, o_gscale, o_scores, o_best,
      o_fix, o_candA, o_candB, o_jobs, o_metas, o_segA, o_segB, o_segAs, o_segBs, o_partial, o_Acur, o_Bcur, o_Acand,
      o_Bcand, o_Ascand, o_Bsplit, total;
};

void push_jobs(MMPlan& p, int r_off, int c_off, int kb, uint8_t src, int group, bool first, bool last, int& n) {
  for (int b = 0; b < kb; b += P4V_JOB_KB) {
    P4VJob j{};
    const int len = std::min(P4V_JOB_KB, kb - b);
    j.r_off = (uint32_t)(r_off + b) * P4V_TILE; j.c_off = (uint32_t)(c_off + b) * P4V_TILE; j.kb = (uint8_t)len;
    j.flags = src | ((first && b == 0) ? P4V_JOB_FIRST : 0) | ((last && b + len >= kb) ? P4V_JOB_LAST : 0);
    j.group = (uint8_t)group;
    p.jobs.push_back(j); ++n;
  }
}

int build_plan(const p4v_matmul_desc* d, MMPlan& p, bool with_search) {
  P4V_REQUIRE(d != nullptr, "null desc");
  p.d = *d;
  P4V_REQUIRE(d->batch > 0 && d->heads > 0 && d->S1 > 0 && d->S2 > 0 && d->S3 > 0, "matmul: empty shape");
  P4V_REQUIRE(d->A_bit >= 2 && d->A_bit <= 8 && d->B_bit >= 2 && d->B_bit <= 8, "matmul: bit widths must be in [2,8]");
  P4V_REQUIRE(d->eq_n >= 1 && d->eq_n <= P4V_MAX_CAND, "matmul: eq_n must be in [1,%d]", P4V_MAX_CAND);
  P4V_REQUIRE(d->images_per_chunk >= 0 && d->images_per_chunk <= d->batch,
              "matmul: images_per_chunk must be in [0, batch=%d] (got %d; 0 = whole layer)", d->batch, d->images_per_chunk);
  p.sos = d->sos != 0;
  p.H = d->heads; p.P = d->batch * d->heads;
  p.ipc = with_search ? d->images_per_chunk : 0;
  p.Pc = p.ipc > 0 ? p.ipc * d->heads : p.P; p.S1 = d->S1; p.S2 = d->S2; p.S3 = d->S3;
  p.A_qmax = 1 << (d->A_bit - 1); p.B_qmax = 1 << (d->B_bit - 1);
  p.tiles_m = p4v_cdiv(p.S1, P4V_TILE); p.tiles_n = p4v_cdiv(p.S3, P4V_TILE);
  if (d->operand == P4V_OPERAND_INT8) p.i8 = true;
  else if (d->operand == P4V_OPERAND_BF16) p.i8 = false;
  else p.i8 = p.S2 >= 64;
  p.ew = p.i8 ? 1 : 2;
  p.kb = (int)align_up((size_t)p.S2 * p.ew, 32);
  p.kb16 = (int)align_up((size_t)p.S2 * 2, 32);
  p.KB_A = p.sos ? 2 * p.kb : p.kb; p.KB_B = p.kb;
  p.KB_As = 2 * p.kb16; p.KB_Bs = 3 * p.kb16;
  const float qa1 = (float)(p.A_qmax - 1);

  p.segA.clear(); p.segB.clear(); p.segAs.clear(); p.segBs.clear();
  if (p.sos) {
    p.segA.push_back(P4VSeg{0, p.S2, 0, 0, 0.f, 0.f, qa1, 1, qa1, 0, 0});
    p.segA.push_back(P4VSeg{0, p.S2, p.kb * P4V_TILE, 0, 0.f, 0.f, qa1, 2, qa1, 0, 0});
    p.segAs.push_back(P4VSeg{0, p.S2, 0, 0, 0.f, 0.f, qa1, 1, qa1, 0, 0});
    p.segAs.push_back(P4VSeg{0, p.S2, p.kb16 * P4V_TILE, 0, 0.f, 0.f, qa1, 2, qa1, 0, 0});
    for (int t = 0; t < 3; ++t) p.segBs.push_back(P4VSeg{0, p.S2, t * p.kb16 * P4V_TILE, 0, 0.f, 0.f, 0.f, 0, 0.f, t + 1, 0});
  } else {
    p.segA.push_back(P4VSeg{0, p.S2, 0, 0, 0.f, (float)-p.A_qmax, (float)(p.A_qmax - 1), 0, 0.f, 0, 0});
  }
  p.segB.push_back(P4VSeg{0, p.S2, 0, 0, 0.f, (float)-p.B_qmax, (float)(p.B_qmax - 1), 0, 0.f, 0, 0});

  p.factors.resize(d->eq_n + 1);
  for (int i = 0; i <= d->eq_n; ++i) p.factors[i] = (float)(d->eq_alpha + i * (d->eq_beta - d->eq_alpha) / d->eq_n);
  p.n_split = 20;                                         // matmul.py:636
  p.split_factors.resize(p.n_split);
  for (int i = 0; i < p.n_split; ++i) p.split_factors[i] = (float)(1.0 / (double)(1u << i));

  p.jobs.clear(); p.metas.clear();
  p.stepA = p.stepB = p.stepS = p.fwd = MStep{};
  auto begin = [&](MStep& s) { s = MStep{}; s.job_off = (int)p.jobs.size(); s.meta_fix = (int)p.metas.size(); };
  if (with_search) {
    if (!p.sos) {   // A step: candidates on the row operand
      begin(p.stepA); p.stepA.meta_cand = (int)p.metas.size();
      push_jobs(p, 0, 0, p.kb, P4V_JOB_RCAND, 0, true, true, p.stepA.ncj);
      p.metas.push_back(GroupMeta{0, 0, 0, 0}); p.stepA.ncg = 1;
    } else {        // split search: (hi,lo)_c x exact 3-term bf16 split of the unquantised B
      begin(p.stepS); p.stepS.meta_cand = (int)p.metas.size();
      for (int part = 0; part < 2; ++part) {
        for (int t = 0; t < 3; ++t)
          push_jobs(p, part * p.kb16, t * p.kb16, p.kb16, P4V_JOB_RCAND, part, t == 0, t == 2, p.stepS.ncj);
        p.metas.push_back(GroupMeta{0, 0, 0, 0});        // both parts use aux[0] = 1/(qmax-1); lo also the candidate split
        ++p.stepS.ncg;
      }
    }
    begin(p.stepB); p.stepB.meta_cand = (int)p.metas.size();
    if (!p.sos) {
      push_jobs(p, 0, 0, p.kb, P4V_JOB_CCAND, 0, true, true, p.stepB.ncj);
      p.metas.push_back(GroupMeta{0, 0, 0, 0}); p.stepB.ncg = 1;
    } else {
      for (int part = 0; part < 2; ++part) {
        push_jobs(p, part * p.kb, 0, p.kb, P4V_JOB_CCAND, part, true, true, p.stepB.ncj);
        p.metas.push_back(GroupMeta{0, (short)part, 0, 0}); ++p.stepB.ncg;     // aux[0] = 1/(qmax-1), aux[1] = A_interval
      }
    }
    {   // the row operand (A) of the B step is the same for every candidate: keep it resident when it is small
      uint32_t total = 0, off = 0;
      for (int j = 0; j < p.stepB.ncj; ++j) total += (uint32_t)p.jobs[p.stepB.job_off + j].kb * P4V_TILE;
      if (total <= 60 * 1024)
        for (int j = 0; j < p.stepB.ncj; ++j) {
          P4VJob& jb = p.jobs[p.stepB.job_off + j];
          jb.flags |= P4V_JOB_RRES; jb.res_off = off; off += (uint32_t)jb.kb * P4V_TILE;
        }
    }
  }
  begin(p.fwd);
  if (!p.sos) { push_jobs(p, 0, 0, p.kb, 0, 0, true, true, p.fwd.nfj); p.metas.push_back(GroupMeta{0, 0, 0, 0}); p.fwd.nfg = 1; }
  else for (int part = 0; part < 2; ++part) {
    push_jobs(p, part * p.kb, 0, p.kb, 0, part, true, true, p.fwd.nfj);
    p.metas.push_back(GroupMeta{0, (short)part, 0, 0}); ++p.fwd.nfg;
  }
  p.fwd.meta_cand = (int)p.metas.size();
  P4V_REQUIRE((int)p.jobs.size() <= 4 * P4V_MAX_JOBS && p.stepS.ncj <= P4V_MAX_JOBS && p.stepB.ncj <= P4V_MAX_JOBS &&
              p.stepA.ncj <= P4V_MAX_JOBS && p.fwd.nfj <= P4V_MAX_JOBS, "matmul: S2 too large");

  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
  const int n_c = std::max(d->eq_n, p.n_split);
  p.o_factors = take((d->eq_n + 1) * 4); p.o_sfactors = take(p.n_split * 4);
  p.o_keys = take((2 * p.H + 1) * 4);
  p.o_dA0 = take(p.H * 4); p.o_dA = take(p.H * 4); p.o_dB0 = take(p.H * 4); p.o_dB = take(p.H * 4);
  p.o_ones = take(p.H * 4); p.o_aux = take(2 * 4); p.o_split = take(4); p.o_gscale = take(4);
  p.o_scores = take((size_t)n_c * p.H * 8); p.o_best = take(p.H * 4);
  p.o_fix = take((size_t)2 * p.H * 4); p.o_candA = take((size_t)n_c * p.H * 4); p.o_candB = take((size_t)2 * p.H * 4);
  p.o_jobs = take(p.jobs.size() * sizeof(P4VJob)); p.o_metas = take(p.metas.size() * sizeof(GroupMeta));
  p.o_segA = take(p.segA.size() * sizeof(P4VSeg)); p.o_segB = take(p.segB.size() * sizeof(P4VSeg));
  p.o_segAs = take(std::max<size_t>(1, p.segAs.size()) * sizeof(P4VSeg));
  p.o_segBs = take(std::max<size_t>(1, p.segBs.size()) * sizeof(P4VSeg));
  const size_t tilesA = (size_t)p.Pc * p.tiles_m, tilesB = (size_t)p.Pc * p.tiles_n;   // one chunk of problems
  p.o_partial = take(with_search ? tilesA * p.tiles_n * n_c * 32 * 4 : 4);
  p.o_Acur = take(tilesA * P4V_TILE * p.KB_A);
  p.o_Bcur = take(tilesB * P4V_TILE * p.KB_B);
  p.o_Acand = take(with_search && !p.sos ? (size_t)d->eq_n * tilesA * P4V_TILE * p.KB_A : 4);
  p.o_Bcand = take(with_search ? (size_t)d->eq_n * tilesB * P4V_TILE * p.KB_B : 4);
  p.o_Ascand = take(with_search && p.sos ? (size_t)p.n_split * tilesA * P4V_TILE * p.KB_As : 4);
  p.o_Bsplit = take(with_search && p.sos ? tilesB * P4V_TILE * p.KB_Bs : 4);
  p.total = o;
  return 0;
}

int upload(const MMPlan& p, void* ws, cudaStream_t st) {
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_factors), p.factors.data(), p.factors.size() * 4, cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_sfactors), p.split_factors.data(), p.split_factors.size() * 4, cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_jobs), p.jobs.data(), p.jobs.size() * sizeof(P4VJob), cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_metas), p.metas.data(), p.metas.size() * sizeof(GroupMeta), cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segA), p.segA.data(), p.segA.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segB), p.segB.data(), p.segB.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  if (!p.segAs.empty()) P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segAs), p.segAs.data(), p.segAs.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  if (!p.segBs.empty()) P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segBs), p.segBs.data(), p.segBs.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  std::vector<float> ones(p.H, 1.f);
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_ones), ones.data(), p.H * 4, cudaMemcpyHostToDevice, st));
  return 0;
}

// problems [p0, p0 + n) of the layer: one chunk of whole images (or the whole layer)
struct Chunk { int p0, n; };
std::vector<Chunk> chunks(const MMPlan& p) {
  std::vector<Chunk> cs;
  for (int p0 = 0; p0 < p.P; p0 += p.Pc) cs.push_back(Chunk{p0, std::min(p.Pc, p.P - p0)});
  return cs;
}

// which: 0 Acur, 1 Acand, 2 Bcur, 3 Bcand, 4 A split-search candidates (bf16), 5 B exact split (bf16); of the problems of c
int quant(const MMPlan& p, void* ws, int which, const float* src, Chunk c, cudaStream_t st) {
  QuantImageArgs q{};
  const bool isA = which == 0 || which == 1 || which == 4;
  q.P = c.n; q.prob_stride = isA ? (long long)p.S1 * p.S2 : (long long)p.S2 * p.S3;
  q.src = src + (size_t)c.p0 * q.prob_stride;     // chunks start at an image: problem p of the chunk is head p % heads
  q.src_transposed = isA ? 0 : 1; q.ld = isA ? p.S2 : p.S3;
  q.rows = isA ? p.S1 : p.S3; q.tiles = isA ? p.tiles_m : p.tiles_n;
  q.rows_per_block = 0; q.d_mod = p.H; q.d_stride = 1;
  q.is_int8 = p.i8; q.n_planes = 1; q.factors = nullptr; q.split = at<float>(ws, p.o_split);
  int KB = 0;
  switch (which) {
    case 0: q.dst = at<uint8_t>(ws, p.o_Acur); KB = p.KB_A; q.delta = at<float>(ws, p.o_dA); q.segs = at<P4VSeg>(ws, p.o_segA); q.nseg = (int)p.segA.size(); break;
    case 1: q.dst = at<uint8_t>(ws, p.o_Acand); KB = p.KB_A; q.delta = at<float>(ws, p.o_dA0); q.segs = at<P4VSeg>(ws, p.o_segA); q.nseg = (int)p.segA.size();
            q.n_planes = p.d.eq_n; q.factors = at<float>(ws, p.o_factors); break;
    case 2: q.dst = at<uint8_t>(ws, p.o_Bcur); KB = p.KB_B; q.delta = at<float>(ws, p.o_dB); q.segs = at<P4VSeg>(ws, p.o_segB); q.nseg = 1; break;
    case 3: q.dst = at<uint8_t>(ws, p.o_Bcand); KB = p.KB_B; q.delta = at<float>(ws, p.o_dB0); q.segs = at<P4VSeg>(ws, p.o_segB); q.nseg = 1;
            q.n_planes = p.d.eq_n; q.factors = at<float>(ws, p.o_factors); break;
    case 4: q.dst = at<uint8_t>(ws, p.o_Ascand); KB = p.KB_As; q.delta = at<float>(ws, p.o_dA0); q.segs = at<P4VSeg>(ws, p.o_segAs); q.nseg = 2;
            q.n_planes = p.n_split; q.factors = at<float>(ws, p.o_sfactors); q.is_int8 = 0; break;
    default: q.dst = at<uint8_t>(ws, p.o_Bsplit); KB = p.KB_Bs; q.delta = at<float>(ws, p.o_dB0); q.segs = at<P4VSeg>(ws, p.o_segBs); q.nseg = 3; q.is_int8 = 0; break;
  }
  q.tile_bytes = (unsigned long long)P4V_TILE * KB;
  q.plane_stride = q.tile_bytes * q.tiles * c.n;
  return p4v_quant_image(q, st);
}
int quant(const MMPlan& p, void* ws, int which, const float* src, cudaStream_t st) { return quant(p, ws, which, src, Chunk{0, p.P}, st); }

void fill_sweep(const MMPlan& p, void* ws, const MStep& s, SweepParams& sp, Chunk c) {
  sp = SweepParams{};
  sp.R_cur = at<uint8_t>(ws, p.o_Acur); sp.C_cur = at<uint8_t>(ws, p.o_Bcur);
  sp.R_cand = at<uint8_t>(ws, p.o_Acand); sp.C_cand = at<uint8_t>(ws, p.o_Bcand);
  sp.R_tile_bytes = sp.R_cand_tile_bytes = (unsigned long long)P4V_TILE * p.KB_A;
  sp.C_tile_bytes = sp.C_cand_tile_bytes = (unsigned long long)P4V_TILE * p.KB_B;
  sp.R_cand_stride = sp.R_cand_tile_bytes * p.tiles_m * c.n; sp.C_cand_stride = sp.C_cand_tile_bytes * p.tiles_n * c.n;
  sp.P = c.n; sp.M = p.S1; sp.N = p.S3; sp.tiles_m = p.tiles_m; sp.tiles_n = p.tiles_n;
  sp.ld = p.S3; sp.prob_stride = (long long)p.S1 * p.S3;
  sp.gscale = at<float>(ws, p.o_gscale);
  sp.jobs = at<P4VJob>(ws, p.o_jobs) + s.job_off;
  sp.n_fixed_jobs = s.nfj; sp.n_cand_jobs = s.ncj; sp.n_fixed_groups = s.nfg; sp.n_cand_groups = s.ncg;
  sp.fix_scale = at<float>(ws, p.o_fix); sp.candA = at<float>(ws, p.o_candA); sp.candB = at<float>(ws, p.o_candB);
  sp.nsg = p.H; sp.sg_mode = P4V_SG_PROBLEM;
  sp.n_cand = p.d.eq_n; sp.partial = at<float>(ws, p.o_partial); sp.is_int8 = p.i8;
}
void fill_sweep(const MMPlan& p, void* ws, const MStep& s, SweepParams& sp) { fill_sweep(p, ws, s, sp, Chunk{0, p.P}); }

int run_sweep(const MMPlan& p, const MStep& s, const SweepParams& sp, cudaStream_t st) {
  return p4v_run_sweep(sp, p.jobs.data() + s.job_off, p.d.kernel, st);
}

// kind 2: searched operand tables (d0, cur other) per head ; kind 3: other operand = aux[meta.a]
int tables(const MMPlan& p, void* ws, const MStep& s, int kind, const float* d_search0, const float* d_fixed_w,
           const float* d_other, const float* factors, int n_cand, cudaStream_t st) {
  StepTablesArgs t{};
  t.kind = kind; t.target = 0;
  t.dW = d_fixed_w; t.dW0 = d_search0; t.n_V = p.H; t.n_H = 1; t.crb_rows = P4V_CG;
  t.dX = d_other; t.dX0 = d_other; t.n_a = 1; t.d_neg = 0.f;
  t.factors = factors; t.n_cand = n_cand;
  t.fixed_meta = at<GroupMeta>(ws, p.o_metas) + s.meta_fix; t.n_fixed_groups = s.nfg;
  t.cand_meta = at<GroupMeta>(ws, p.o_metas) + s.meta_cand; t.n_cand_groups = s.ncg;
  t.nsg = p.H;
  t.fix_scale = at<float>(ws, p.o_fix); t.candA = at<float>(ws, p.o_candA); t.candB = at<float>(ws, p.o_candB);
  return p4v_step_tables(t, st);
}

__global__ void sos_aux_kernel(const float* split, float qm1, float* aux, float* A_interval_out) {
  aux[0] = __fdiv_rn(1.f, qm1);
  aux[1] = __fdiv_rn(split[0], qm1);       // A_interval = split / (A_qmax - 1)   (matmul.py:629)
  if (A_interval_out) A_interval_out[0] = aux[1];
}
__global__ void set_scalar_kernel(float* p, float v) { p[0] = v; }

// scores of chunk c: the first chunk writes the fp64 table, later chunks add to it (fixed chunk order)
int reduce(const MMPlan& p, void* ws, const SweepParams& sp, int n_cand, bool accumulate, cudaStream_t st) {
  ReduceArgs r{};
  r.partial = sp.partial; r.n_cand = n_cand; r.P = sp.P; r.tiles_m = p.tiles_m; r.tiles_n = p.tiles_n; r.order = sp.order;
  r.mode = P4V_SG_PROBLEM; r.n_keys = p.H; r.sums = at<double>(ws, p.o_scores); r.accumulate = accumulate ? 1 : 0;
  return p4v_reduce_scores(r, st);
}

int finish(const MMPlan& p, void* ws, int n_cand, int n_groups, double inv_count, const float* factors, const float* d0,
           float* d, float* score_log, cudaStream_t st) {
  SelectArgs f{};     // no image commit: the current image is re-quantised from the fp32 source with the chosen step size
  f.sums = at<double>(ws, p.o_scores); f.n_cand = n_cand; f.n_keys = p.H; f.n_groups = n_groups; f.keys_per_group = n_groups == 1 ? p.H : 1;
  f.inv_count = inv_count; f.gscale = at<float>(ws, p.o_gscale); f.factors = factors;
  f.d0 = d0; f.d = d; f.d_stride = 1; f.d_col = 0; f.best = at<int>(ws, p.o_best); f.score_log = score_log;
  f.has_next = 0;
  return p4v_select_step(f, st);
}

// One search step over every chunk: [chunk images] -> sweep -> reduce (into the table).  Unchunked, the images are
// those begin() built and the previous step re-quantised.
template <class Images, class Setup>
int sweep_chunks(const MMPlan& p, void* ws, const MStep& s, const float* Y, const float* G, int n_cand, Images images,
                 Setup setup, cudaStream_t st) {
  int rc;
  const std::vector<Chunk> cs = chunks(p);
  for (size_t i = 0; i < cs.size(); ++i) {
    if (p.ipc && (rc = images(cs[i]))) return rc;
    const size_t off = (size_t)cs[i].p0 * p.S1 * p.S3;
    SweepParams sp; fill_sweep(p, ws, s, sp, cs[i]);
    sp.Y = Y + off; sp.Gr = G + off;
    setup(sp, cs[i]);
    if ((rc = run_sweep(p, s, sp, st))) return rc;
    if ((rc = reduce(p, ws, sp, n_cand, i > 0, st))) return rc;
  }
  return 0;
}

int search_A(const MMPlan& p, void* ws, const float* A, const float* B, const float* Y, const float* G, float* log, cudaStream_t st) {
  int rc;
  if ((rc = tables(p, ws, p.stepA, 2, at<float>(ws, p.o_dA0), at<float>(ws, p.o_dA), at<float>(ws, p.o_dB),
                   at<float>(ws, p.o_factors), p.d.eq_n, st))) return rc;
  auto images = [&](Chunk c) { int r = quant(p, ws, 1, A, c, st); return r ? r : quant(p, ws, 2, B, c, st); };
  if ((rc = sweep_chunks(p, ws, p.stepA, Y, G, p.d.eq_n, images, [](SweepParams& sp, Chunk) { sp.order = 1; }, st))) return rc;
  if ((rc = finish(p, ws, p.d.eq_n, p.H, 1.0 / ((double)p.S1 * p.S3), at<float>(ws, p.o_factors),
                   at<float>(ws, p.o_dA0), at<float>(ws, p.o_dA), log, st))) return rc;
  return p.ipc ? 0 : quant(p, ws, 0, A, st);
}

int search_B(const MMPlan& p, void* ws, const float* A, const float* B, const float* Y, const float* G, float* log, cudaStream_t st) {
  int rc;
  if ((rc = tables(p, ws, p.stepB, p.sos ? 3 : 2, at<float>(ws, p.o_dB0), at<float>(ws, p.o_dB),
                   p.sos ? at<float>(ws, p.o_aux) : at<float>(ws, p.o_dA), at<float>(ws, p.o_factors), p.d.eq_n, st))) return rc;
  auto images = [&](Chunk c) { int r = quant(p, ws, 0, A, c, st); return r ? r : quant(p, ws, 3, B, c, st); };
  if ((rc = sweep_chunks(p, ws, p.stepB, Y, G, p.d.eq_n, images, [](SweepParams& sp, Chunk) { sp.order = 0; }, st))) return rc;
  if ((rc = finish(p, ws, p.d.eq_n, p.H, 1.0 / ((double)p.S1 * p.S3), at<float>(ws, p.o_factors),
                   at<float>(ws, p.o_dB0), at<float>(ws, p.o_dB), log, st))) return rc;
  return p.ipc ? 0 : quant(p, ws, 2, B, st);
}

int search_split(const MMPlan& p, void* ws, const float* A, const float* B, const float* Y, const float* G, float* log, cudaStream_t st) {
  int rc;
  // candA[c][head] = split_c * 1, candB[g][head] = aux[0] = 1/(qmax-1); the high part ignores candA
  if ((rc = tables(p, ws, p.stepS, 3, at<float>(ws, p.o_ones), at<float>(ws, p.o_ones), at<float>(ws, p.o_aux),
                   at<float>(ws, p.o_sfactors), p.n_split, st))) return rc;
  auto images = [&](Chunk c) { int r = quant(p, ws, 4, A, c, st); return r ? r : quant(p, ws, 5, B, c, st); };
  auto setup = [&](SweepParams& sp, Chunk c) {
    sp.order = 1; sp.n_cand = p.n_split; sp.is_int8 = 0; sp.cand_noA_mask = 1ull;
    sp.R_cand = at<uint8_t>(ws, p.o_Ascand); sp.R_cand_tile_bytes = (unsigned long long)P4V_TILE * p.KB_As;
    sp.R_cand_stride = sp.R_cand_tile_bytes * p.tiles_m * c.n;
    sp.C_cur = at<uint8_t>(ws, p.o_Bsplit); sp.C_tile_bytes = (unsigned long long)P4V_TILE * p.KB_Bs;
  };
  if ((rc = sweep_chunks(p, ws, p.stepS, Y, G, p.n_split, images, setup, st))) return rc;
  // global score: mean over heads and rows (matmul.py:620-621)
  if ((rc = finish(p, ws, p.n_split, 1, 1.0 / ((double)p.H * p.S1 * p.S3), at<float>(ws, p.o_sfactors),
                   at<float>(ws, p.o_ones), at<float>(ws, p.o_split), log, st))) return rc;
  sos_aux_kernel<<<1, 1, 0, st>>>(at<float>(ws, p.o_split), (float)(p.A_qmax - 1), at<float>(ws, p.o_aux), nullptr);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return p.ipc ? 0 : quant(p, ws, 0, A, st);
}

int begin(const MMPlan& p, void* ws, const float* A, const float* B, const float* G, cudaStream_t st) {
  int rc;
  if ((rc = upload(p, ws, st))) return rc;
  int* keys = at<int>(ws, p.o_keys);
  if ((rc = p4v_keys_reset(keys, 2 * p.H + 1, st))) return rc;
  if ((rc = p4v_group_absmax(A, (long long)p.S1 * p.S2, p.P, p.H, keys, st))) return rc;
  if ((rc = p4v_group_absmax(B, (long long)p.S2 * p.S3, p.P, p.H, keys + p.H, st))) return rc;
  if ((rc = p4v_group_absmax(G, (long long)p.P * p.S1 * p.S3, 1, 1, keys + 2 * p.H, st))) return rc;
  if (p.d.init_layerwise) {       // matmul.py:430-432
    if ((rc = p4v_keys_broadcast_max(keys, p.H, st))) return rc;
    if ((rc = p4v_keys_broadcast_max(keys + p.H, p.H, st))) return rc;
  }
  if ((rc = p4v_keys_to_delta(keys, p.H, (float)p.A_qmax - 0.5f, at<float>(ws, p.o_dA0), at<float>(ws, p.o_dA), st))) return rc;
  if ((rc = p4v_keys_to_delta(keys + p.H, p.H, (float)p.B_qmax - 0.5f, at<float>(ws, p.o_dB0), at<float>(ws, p.o_dB), st))) return rc;
  if ((rc = p4v_make_gscale(keys + 2 * p.H, at<float>(ws, p.o_gscale), st))) return rc;
  if (p.sos) {
    set_scalar_kernel<<<1, 1, 0, st>>>(at<float>(ws, p.o_split), 0.01f);       // matmul.py:354-355 (dead: overwritten by the first search)
    sos_aux_kernel<<<1, 1, 0, st>>>(at<float>(ws, p.o_split), (float)(p.A_qmax - 1), at<float>(ws, p.o_aux), nullptr);
    P4V_CUDA_OK(cudaGetLastError());
  }
  if (p.ipc) return 0;            // chunked: every step builds its chunks' images
  if (p.sos) {
    if ((rc = quant(p, ws, 4, A, st))) return rc;
    if ((rc = quant(p, ws, 5, B, st))) return rc;
  } else {
    if ((rc = quant(p, ws, 1, A, st))) return rc;
  }
  if ((rc = quant(p, ws, 0, A, st))) return rc;
  if ((rc = quant(p, ws, 2, B, st))) return rc;
  if ((rc = quant(p, ws, 3, B, st))) return rc;
  return 0;
}

}  // namespace

extern "C" int p4v_matmul_workspace_bytes(const p4v_matmul_desc* d, size_t* bytes) {
  MMPlan p; int rc = build_plan(d, p, true);
  if (rc) return rc;
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = p.total;
  return 0;
}

extern "C" int p4v_matmul_score_log_floats(const p4v_matmul_desc* d, size_t* n) {
  P4V_REQUIRE(d && n, "null argument");
  *n = (size_t)d->search_round * ((d->sos ? (size_t)20 : (size_t)d->eq_n * d->heads) + (size_t)d->eq_n * d->heads);
  return 0;
}

extern "C" int p4v_matmul_calibrate(const p4v_matmul_desc* d, const float* A, const float* B, const float* raw_out,
                                    const float* raw_grad, void* workspace, size_t workspace_bytes, float* A_interval,
                                    float* B_interval, float* split, float* score_log, void* stream) {
  MMPlan p; int rc = build_plan(d, p, true);
  if (rc) return rc;
  P4V_REQUIRE(A && B && raw_out && raw_grad && workspace && A_interval && B_interval, "matmul_calibrate: null pointer");
  P4V_REQUIRE(!p.sos || split, "matmul_calibrate: sos needs the split output");
  P4V_REQUIRE(workspace_bytes >= p.total, "matmul_calibrate: workspace too small (%zu < %zu)", workspace_bytes, p.total);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = begin(p, workspace, A, B, raw_grad, st))) return rc;
  for (int e = 0; e < d->search_round; ++e) {
    if (p.sos) {
      if ((rc = search_split(p, workspace, A, B, raw_out, raw_grad, score_log, st))) return rc;
      if (score_log) score_log += p.n_split;
    } else {
      if ((rc = search_A(p, workspace, A, B, raw_out, raw_grad, score_log, st))) return rc;
      if (score_log) score_log += (size_t)d->eq_n * p.H;
    }
    if ((rc = search_B(p, workspace, A, B, raw_out, raw_grad, score_log, st))) return rc;
    if (score_log) score_log += (size_t)d->eq_n * p.H;
  }
  if (p.sos) {
    P4V_CUDA_OK(cudaMemcpyAsync(split, at<float>(workspace, p.o_split), 4, cudaMemcpyDeviceToDevice, st));
    P4V_CUDA_OK(cudaMemcpyAsync(A_interval, at<float>(workspace, p.o_aux) + 1, 4, cudaMemcpyDeviceToDevice, st));
  } else {
    P4V_CUDA_OK(cudaMemcpyAsync(A_interval, at<float>(workspace, p.o_dA), (size_t)p.H * 4, cudaMemcpyDeviceToDevice, st));
  }
  P4V_CUDA_OK(cudaMemcpyAsync(B_interval, at<float>(workspace, p.o_dB), (size_t)p.H * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" int p4v_matmul_quant_forward_workspace_bytes(const p4v_matmul_desc* d, size_t* bytes) {
  MMPlan p; int rc = build_plan(d, p, false);
  if (rc) return rc;
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = p.total;
  return 0;
}

extern "C" int p4v_matmul_quant_forward(const p4v_matmul_desc* d, const float* A, const float* B, const float* A_interval,
                                        const float* B_interval, const float* split, void* workspace, size_t workspace_bytes,
                                        float* out, void* stream) {
  MMPlan p; int rc = build_plan(d, p, false);
  if (rc) return rc;
  P4V_REQUIRE(A && B && A_interval && B_interval && workspace && out, "matmul_quant_forward: null pointer");
  P4V_REQUIRE(!p.sos || split, "matmul_quant_forward: sos needs split");
  P4V_REQUIRE(workspace_bytes >= p.total, "matmul_quant_forward: workspace too small (%zu < %zu)", workspace_bytes, p.total);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = upload(p, workspace, st))) return rc;
  P4V_CUDA_OK(cudaMemcpyAsync(at<float>(workspace, p.o_dB), B_interval, (size_t)p.H * 4, cudaMemcpyDeviceToDevice, st));
  if (p.sos) {
    P4V_CUDA_OK(cudaMemcpyAsync(at<float>(workspace, p.o_split), split, 4, cudaMemcpyDeviceToDevice, st));
    sos_aux_kernel<<<1, 1, 0, st>>>(at<float>(workspace, p.o_split), (float)(p.A_qmax - 1), at<float>(workspace, p.o_aux), nullptr);
    P4V_CUDA_OK(cudaGetLastError());
  } else {
    P4V_CUDA_OK(cudaMemcpyAsync(at<float>(workspace, p.o_dA), A_interval, (size_t)p.H * 4, cudaMemcpyDeviceToDevice, st));
  }
  if ((rc = quant(p, workspace, 0, A, st))) return rc;
  if ((rc = quant(p, workspace, 2, B, st))) return rc;
  // fixed scale per head: plain dA*dB ; sos: dB * aux[part]
  if ((rc = tables(p, workspace, p.fwd, p.sos ? 3 : 2, at<float>(workspace, p.o_dB0),
                   p.sos ? at<float>(workspace, p.o_dB) : at<float>(workspace, p.o_dA),
                   p.sos ? at<float>(workspace, p.o_aux) : at<float>(workspace, p.o_dB), at<float>(workspace, p.o_factors), 0, st))) return rc;
  SweepParams sp; fill_sweep(p, workspace, p.fwd, sp);
  sp.out = out; sp.n_cand = 1; sp.order = 0; sp.R_cand = nullptr; sp.C_cand = nullptr;
  return run_sweep(p, p.fwd, sp, st);
}
