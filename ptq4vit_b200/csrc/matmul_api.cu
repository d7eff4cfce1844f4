// C-ABI for the head-wise MatMul scale-factor search (PTQSLBatchingQuantMatMul and the
// split-of-softmax variant).  Problem p = image * heads + head; the row operand is A[p]
// (S1 x S2), the column operand is B[p]^T (S3 x S2); one K segment (n_V = n_H = 1).
#include "../../include/ptq4vit_b200.h"
#include "plan.cuh"

namespace {

// An operand image and how it is built: from A (rows S1) or from B (rows S3, read transposed), with the current step
// sizes (cur) or the initial ones, the candidate factors (none: one plane of the step sizes) and its segment table
struct Operand { Image im; bool B, cur; const Table<float>* factors; const Table<P4VSeg>* segs; };

struct MStep {
  int job_off, nfj, ncj, nfg, ncg, meta_fix, meta_cand;
  int order, n_cand; unsigned long long noA_mask;   // sweep order, candidates, candidate groups that ignore candA
  const Image *Rcur, *Rcand, *Ccur, *Ccand;         // the images the sweep reads: rows = A, columns = B^T
};

struct MMPlan {
  MMPlan() = default;
  MMPlan(const MMPlan&) = delete;                   // the steps and operands point at the plan's images and tables
  p4v_matmul_desc d;
  bool i8, sos;
  int ew, P, H, S1, S2, S3, tiles_m, tiles_n, A_qmax, B_qmax;
  int ipc;       // images per chunk (0: whole layer); the operand images hold Pc = ipc * heads problems
  int Pc;
  int kb;        // padded K bytes of one part in the search operand type
  int kb16;      // padded K bytes in bf16 (split-search images)
  Table<P4VJob> jobs; Table<GroupMeta> metas;
  Table<P4VSeg> segA, segB, segAs, segBs;
  Table<float> factors, split_factors;
  // Acur = [hi|lo] for sos; split search: Ascand = [hi|lo] bf16 candidates, Bsplit = [b1|b2|b3] exact bf16 split of B
  Operand Acur, Acand, Bcur, Bcand, Ascand, Bsplit;
  MStep stepA, stepB, stepS, fwd;
  int n_split;
  size_t o_keys, o_dA0, o_dA, o_dB0, o_dB, o_ones, o_aux, o_split, o_gscale, o_scores, o_best, o_fix, o_candA, o_candB,
      o_partial, total;
};

// the checks every entry point makes of the shape and the bit widths
int check_shape(const p4v_matmul_desc* d) {
  P4V_REQUIRE(d != nullptr, "null desc");
  P4V_REQUIRE(d->batch > 0 && d->heads > 0 && d->S1 > 0 && d->S2 > 0 && d->S3 > 0, "matmul: empty shape");
  P4V_REQUIRE(d->A_bit >= 2 && d->A_bit <= 8 && d->B_bit >= 2 && d->B_bit <= 8, "matmul: bit widths must be in [2,8]");
  return 0;
}

int build_plan(const p4v_matmul_desc* d, MMPlan& p, bool with_search) {
  if (int rc = check_shape(d)) return rc;
  p.d = *d;
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
  const float qa1 = (float)(p.A_qmax - 1);

  if (p.sos) {
    p.segA.host.push_back(P4VSeg{0, p.S2, 0, 0, 0.f, 0.f, qa1, 1, qa1, 0, 0});
    p.segA.host.push_back(P4VSeg{0, p.S2, p.kb * P4V_TILE, 0, 0.f, 0.f, qa1, 2, qa1, 0, 0});
    p.segAs.host.push_back(P4VSeg{0, p.S2, 0, 0, 0.f, 0.f, qa1, 1, qa1, 0, 0});
    p.segAs.host.push_back(P4VSeg{0, p.S2, p.kb16 * P4V_TILE, 0, 0.f, 0.f, qa1, 2, qa1, 0, 0});
    for (int t = 0; t < 3; ++t) p.segBs.host.push_back(P4VSeg{0, p.S2, t * p.kb16 * P4V_TILE, 0, 0.f, 0.f, 0.f, 0, 0.f, t + 1, 0});
  } else {
    p.segA.host.push_back(P4VSeg{0, p.S2, 0, 0, 0.f, (float)-p.A_qmax, (float)(p.A_qmax - 1), 0, 0.f, 0, 0});
  }
  p.segB.host.push_back(P4VSeg{0, p.S2, 0, 0, 0.f, (float)-p.B_qmax, (float)(p.B_qmax - 1), 0, 0.f, 0, 0});

  p.factors.host = cand_factors(d->eq_n, d->eq_alpha, d->eq_beta);
  p.n_split = 20;                                         // matmul.py:636
  p.split_factors.host.resize(p.n_split);
  for (int i = 0; i < p.n_split; ++i) p.split_factors.host[i] = (float)(1.0 / (double)(1u << i));

  const int KB_A = p.sos ? 2 * p.kb : p.kb;
  p.Acur = Operand{Image{0, KB_A, p.tiles_m, p.Pc, 1, p.i8}, false, true, nullptr, &p.segA};
  p.Acand = Operand{Image{0, KB_A, p.tiles_m, p.Pc, d->eq_n, p.i8}, false, false, &p.factors, &p.segA};
  p.Bcur = Operand{Image{0, p.kb, p.tiles_n, p.Pc, 1, p.i8}, true, true, nullptr, &p.segB};
  p.Bcand = Operand{Image{0, p.kb, p.tiles_n, p.Pc, d->eq_n, p.i8}, true, false, &p.factors, &p.segB};
  p.Ascand = Operand{Image{0, 2 * p.kb16, p.tiles_m, p.Pc, p.n_split, false}, false, false, &p.split_factors, &p.segAs};
  p.Bsplit = Operand{Image{0, 3 * p.kb16, p.tiles_n, p.Pc, 1, false}, true, false, nullptr, &p.segBs};

  std::vector<P4VJob>& jobs = p.jobs.host;
  std::vector<GroupMeta>& metas = p.metas.host;
  p.stepA = p.stepB = p.stepS = p.fwd = MStep{};
  auto begin = [&](MStep& s, int order, int n_cand) {
    s = MStep{};
    s.job_off = (int)jobs.size(); s.meta_fix = (int)metas.size(); s.order = order; s.n_cand = n_cand;
    s.Rcur = &p.Acur.im; s.Rcand = &p.Acand.im; s.Ccur = &p.Bcur.im; s.Ccand = &p.Bcand.im;
  };
  if (with_search) {
    if (!p.sos) {   // A step: candidates on the row operand
      begin(p.stepA, 1, d->eq_n); p.stepA.meta_cand = (int)metas.size();
      add_group(jobs, 0, 0, p.kb, P4V_JOB_RCAND, 0, true, true, p.stepA.ncj);
      metas.push_back(GroupMeta{0, 0, 0, 0}); p.stepA.ncg = 1;
    } else {        // split search: (hi,lo)_c x exact 3-term bf16 split of the unquantised B; the high part ignores candA
      begin(p.stepS, 1, p.n_split); p.stepS.meta_cand = (int)metas.size();
      p.stepS.noA_mask = 1ull; p.stepS.Rcand = &p.Ascand.im; p.stepS.Ccur = &p.Bsplit.im;
      for (int part = 0; part < 2; ++part) {
        for (int t = 0; t < 3; ++t)
          add_group(jobs, part * p.kb16, t * p.kb16, p.kb16, P4V_JOB_RCAND, part, t == 0, t == 2, p.stepS.ncj);
        metas.push_back(GroupMeta{0, 0, 0, 0});        // both parts use aux[0] = 1/(qmax-1); lo also the candidate split
        ++p.stepS.ncg;
      }
    }
    begin(p.stepB, 0, d->eq_n); p.stepB.meta_cand = (int)metas.size();
    if (!p.sos) {
      add_group(jobs, 0, 0, p.kb, P4V_JOB_CCAND, 0, true, true, p.stepB.ncj);
      metas.push_back(GroupMeta{0, 0, 0, 0}); p.stepB.ncg = 1;
    } else {
      for (int part = 0; part < 2; ++part) {
        add_group(jobs, part * p.kb, 0, p.kb, P4V_JOB_CCAND, part, true, true, p.stepB.ncj);
        metas.push_back(GroupMeta{0, (short)part, 0, 0}); ++p.stepB.ncg;     // aux[0] = 1/(qmax-1), aux[1] = A_interval
      }
    }
    mark_resident(jobs, p.stepB.job_off, p.stepB.ncj);   // the row operand (A) of the B step is the same for every candidate
  }
  begin(p.fwd, 0, 1);
  if (!p.sos) { add_group(jobs, 0, 0, p.kb, 0, 0, true, true, p.fwd.nfj); metas.push_back(GroupMeta{0, 0, 0, 0}); p.fwd.nfg = 1; }
  else for (int part = 0; part < 2; ++part) {
    add_group(jobs, part * p.kb, 0, p.kb, 0, part, true, true, p.fwd.nfj);
    metas.push_back(GroupMeta{0, (short)part, 0, 0}); ++p.fwd.nfg;
  }
  p.fwd.meta_cand = (int)metas.size();
  P4V_REQUIRE((int)jobs.size() <= 4 * P4V_MAX_JOBS && p.stepS.ncj <= P4V_MAX_JOBS && p.stepB.ncj <= P4V_MAX_JOBS &&
              p.stepA.ncj <= P4V_MAX_JOBS && p.fwd.nfj <= P4V_MAX_JOBS, "matmul: S2 too large");

  Carver c{0};
  const int n_c = std::max(d->eq_n, p.n_split);
  p.factors.off = c.take(p.factors.bytes()); p.split_factors.off = c.take(p.split_factors.bytes());
  p.o_keys = c.take((2 * p.H + 1) * 4);
  p.o_dA0 = c.take(p.H * 4); p.o_dA = c.take(p.H * 4); p.o_dB0 = c.take(p.H * 4); p.o_dB = c.take(p.H * 4);
  p.o_ones = c.take(p.H * 4); p.o_aux = c.take(2 * 4); p.o_split = c.take(4); p.o_gscale = c.take(4);
  p.o_scores = c.take((size_t)n_c * p.H * 8); p.o_best = c.take(p.H * 4);
  p.o_fix = c.take((size_t)2 * p.H * 4); p.o_candA = c.take((size_t)n_c * p.H * 4); p.o_candB = c.take((size_t)2 * p.H * 4);
  p.jobs.off = c.take(p.jobs.bytes()); p.metas.off = c.take(p.metas.bytes());
  p.segA.off = c.take(p.segA.bytes()); p.segB.off = c.take(p.segB.bytes());
  p.segAs.off = c.take(std::max(p.segAs.bytes(), sizeof(P4VSeg)));
  p.segBs.off = c.take(std::max(p.segBs.bytes(), sizeof(P4VSeg)));
  p.o_partial = c.take(with_search ? (size_t)p.Pc * p.tiles_m * p.tiles_n * n_c * 32 * 4 : 4);   // one chunk of problems
  p.Acur.im.off = c.take(p.Acur.im.bytes());
  p.Bcur.im.off = c.take(p.Bcur.im.bytes());
  p.Acand.im.off = c.take(with_search && !p.sos ? p.Acand.im.bytes() : 4);
  p.Bcand.im.off = c.take(with_search ? p.Bcand.im.bytes() : 4);
  p.Ascand.im.off = c.take(with_search && p.sos ? p.Ascand.im.bytes() : 4);
  p.Bsplit.im.off = c.take(with_search && p.sos ? p.Bsplit.im.bytes() : 4);
  p.total = c.end;
  return 0;
}

int upload(const MMPlan& p, void* ws, cudaStream_t st) {
  int rc;
  if ((rc = p.factors.upload(ws, st)) || (rc = p.split_factors.upload(ws, st)) || (rc = p.jobs.upload(ws, st)) ||
      (rc = p.metas.upload(ws, st)) || (rc = p.segA.upload(ws, st)) || (rc = p.segB.upload(ws, st)) ||
      (rc = p.segAs.upload(ws, st)) || (rc = p.segBs.upload(ws, st))) return rc;
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

// Build operand image o of the problems of chunk c from its source A or B
int quant(const MMPlan& p, void* ws, const Operand& o, const float* A, const float* B, Chunk c, cudaStream_t st) {
  QuantImageArgs q{};
  o.im.chunk(o.im.tiles, c.n).fill(q, ws);
  q.prob_stride = o.B ? (long long)p.S2 * p.S3 : (long long)p.S1 * p.S2;
  q.src = (o.B ? B : A) + (size_t)c.p0 * q.prob_stride;     // chunks start at an image: problem p of the chunk is head p % heads
  q.src_transposed = o.B ? 1 : 0; q.ld = o.B ? p.S3 : p.S2; q.rows = o.B ? p.S3 : p.S1;
  q.rows_per_block = 0; q.d_mod = p.H; q.d_stride = 1;
  q.factors = o.factors ? o.factors->dev(ws) : nullptr; q.split = at<float>(ws, p.o_split);
  q.delta = at<float>(ws, o.B ? (o.cur ? p.o_dB : p.o_dB0) : (o.cur ? p.o_dA : p.o_dA0));
  q.segs = o.segs->dev(ws); q.nseg = (int)o.segs->host.size();
  return p4v_quant_image(q, st);
}
int quant(const MMPlan& p, void* ws, const Operand& o, const float* A, const float* B, cudaStream_t st) {
  return quant(p, ws, o, A, B, Chunk{0, p.P}, st);
}

void fill_sweep(const MMPlan& p, void* ws, const MStep& s, SweepParams& sp, Chunk c) {
  sp = SweepParams{};
  auto part = [&](const Image* im) { return im->chunk(im->tiles, c.n); };
  fill_images(sp, ws, part(s.Rcur), part(s.Rcand), part(s.Ccur), part(s.Ccand));
  sp.P = c.n; sp.M = p.S1; sp.N = p.S3; sp.tiles_m = p.tiles_m; sp.tiles_n = p.tiles_n;
  sp.ld = p.S3; sp.prob_stride = (long long)p.S1 * p.S3;
  sp.gscale = at<float>(ws, p.o_gscale);
  sp.jobs = p.jobs.dev(ws) + s.job_off;
  sp.n_fixed_jobs = s.nfj; sp.n_cand_jobs = s.ncj; sp.n_fixed_groups = s.nfg; sp.n_cand_groups = s.ncg;
  sp.fix_scale = at<float>(ws, p.o_fix); sp.candA = at<float>(ws, p.o_candA); sp.candB = at<float>(ws, p.o_candB);
  sp.nsg = p.H; sp.sg_mode = P4V_SG_PROBLEM;
  sp.cand_noA_mask = s.noA_mask; sp.n_cand = s.n_cand; sp.order = s.order; sp.partial = at<float>(ws, p.o_partial);
}

int run_sweep(const MMPlan& p, const MStep& s, const SweepParams& sp, cudaStream_t st) {
  return p4v_run_sweep(sp, p.jobs.host.data() + s.job_off, p.d.kernel, st);
}

// kind 2: searched operand tables (d0, cur other) per head ; kind 3: other operand = aux[meta.a]
int tables(const MMPlan& p, void* ws, const MStep& s, int kind, const float* d_search0, const float* d_fixed_w,
           const float* d_other, const float* factors, int n_cand, cudaStream_t st) {
  StepTablesArgs t{};
  t.kind = kind; t.target = 0;
  t.dW = d_fixed_w; t.dW0 = d_search0; t.n_V = p.H; t.n_H = 1; t.crb_rows = P4V_CG;
  t.dX = d_other; t.dX0 = d_other; t.n_a = 1; t.d_neg = 0.f;
  t.factors = factors; t.n_cand = n_cand;
  t.fixed_meta = p.metas.dev(ws) + s.meta_fix; t.n_fixed_groups = s.nfg;
  t.cand_meta = p.metas.dev(ws) + s.meta_cand; t.n_cand_groups = s.ncg;
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
int reduce(const MMPlan& p, void* ws, const SweepParams& sp, bool accumulate, cudaStream_t st) {
  ReduceArgs r{};
  r.partial = sp.partial; r.n_cand = sp.n_cand; r.P = sp.P; r.tiles_m = p.tiles_m; r.tiles_n = p.tiles_n; r.order = sp.order;
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

// One search step over every chunk: [the chunk's images R and C] -> sweep -> reduce (into the table).  Unchunked, the
// images are those begin() built and the previous step re-quantised.
int sweep_chunks(const MMPlan& p, void* ws, const MStep& s, const Operand& R, const Operand& C, const float* A, const float* B,
                 const float* Y, const float* G, cudaStream_t st) {
  int rc;
  const std::vector<Chunk> cs = chunks(p);
  for (size_t i = 0; i < cs.size(); ++i) {
    if (p.ipc && ((rc = quant(p, ws, R, A, B, cs[i], st)) || (rc = quant(p, ws, C, A, B, cs[i], st)))) return rc;
    const size_t off = (size_t)cs[i].p0 * p.S1 * p.S3;
    SweepParams sp; fill_sweep(p, ws, s, sp, cs[i]);
    sp.Y = Y + off; sp.Gr = G + off;
    if ((rc = run_sweep(p, s, sp, st))) return rc;
    if ((rc = reduce(p, ws, sp, i > 0, st))) return rc;
  }
  return 0;
}

int search_A(const MMPlan& p, void* ws, const float* A, const float* B, const float* Y, const float* G, float* log, cudaStream_t st) {
  int rc;
  if ((rc = tables(p, ws, p.stepA, 2, at<float>(ws, p.o_dA0), at<float>(ws, p.o_dA), at<float>(ws, p.o_dB),
                   p.factors.dev(ws), p.d.eq_n, st))) return rc;
  if ((rc = sweep_chunks(p, ws, p.stepA, p.Acand, p.Bcur, A, B, Y, G, st))) return rc;
  if ((rc = finish(p, ws, p.d.eq_n, p.H, 1.0 / ((double)p.S1 * p.S3), p.factors.dev(ws),
                   at<float>(ws, p.o_dA0), at<float>(ws, p.o_dA), log, st))) return rc;
  return p.ipc ? 0 : quant(p, ws, p.Acur, A, B, st);
}

int search_B(const MMPlan& p, void* ws, const float* A, const float* B, const float* Y, const float* G, float* log, cudaStream_t st) {
  int rc;
  if ((rc = tables(p, ws, p.stepB, p.sos ? 3 : 2, at<float>(ws, p.o_dB0), at<float>(ws, p.o_dB),
                   p.sos ? at<float>(ws, p.o_aux) : at<float>(ws, p.o_dA), p.factors.dev(ws), p.d.eq_n, st))) return rc;
  if ((rc = sweep_chunks(p, ws, p.stepB, p.Acur, p.Bcand, A, B, Y, G, st))) return rc;
  if ((rc = finish(p, ws, p.d.eq_n, p.H, 1.0 / ((double)p.S1 * p.S3), p.factors.dev(ws),
                   at<float>(ws, p.o_dB0), at<float>(ws, p.o_dB), log, st))) return rc;
  return p.ipc ? 0 : quant(p, ws, p.Bcur, A, B, st);
}

int search_split(const MMPlan& p, void* ws, const float* A, const float* B, const float* Y, const float* G, float* log, cudaStream_t st) {
  int rc;
  // candA[c][head] = split_c * 1, candB[g][head] = aux[0] = 1/(qmax-1); the high part ignores candA
  if ((rc = tables(p, ws, p.stepS, 3, at<float>(ws, p.o_ones), at<float>(ws, p.o_ones), at<float>(ws, p.o_aux),
                   p.split_factors.dev(ws), p.n_split, st))) return rc;
  if ((rc = sweep_chunks(p, ws, p.stepS, p.Ascand, p.Bsplit, A, B, Y, G, st))) return rc;
  // global score: mean over heads and rows (matmul.py:620-621)
  if ((rc = finish(p, ws, p.n_split, 1, 1.0 / ((double)p.H * p.S1 * p.S3), p.split_factors.dev(ws),
                   at<float>(ws, p.o_ones), at<float>(ws, p.o_split), log, st))) return rc;
  sos_aux_kernel<<<1, 1, 0, st>>>(at<float>(ws, p.o_split), (float)(p.A_qmax - 1), at<float>(ws, p.o_aux), nullptr);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return p.ipc ? 0 : quant(p, ws, p.Acur, A, B, st);
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
    if ((rc = quant(p, ws, p.Ascand, A, B, st))) return rc;
    if ((rc = quant(p, ws, p.Bsplit, A, B, st))) return rc;
  } else {
    if ((rc = quant(p, ws, p.Acand, A, B, st))) return rc;
  }
  if ((rc = quant(p, ws, p.Acur, A, B, st))) return rc;
  if ((rc = quant(p, ws, p.Bcur, A, B, st))) return rc;
  if ((rc = quant(p, ws, p.Bcand, A, B, st))) return rc;
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
  if ((rc = quant(p, workspace, p.Acur, A, B, st))) return rc;
  if ((rc = quant(p, workspace, p.Bcur, A, B, st))) return rc;
  // fixed scale per head: plain dA*dB ; sos: dB * aux[part]
  if ((rc = tables(p, workspace, p.fwd, p.sos ? 3 : 2, at<float>(workspace, p.o_dB0),
                   p.sos ? at<float>(workspace, p.o_dB) : at<float>(workspace, p.o_dA),
                   p.sos ? at<float>(workspace, p.o_aux) : at<float>(workspace, p.o_dB), p.factors.dev(workspace), 0, st))) return rc;
  SweepParams sp; fill_sweep(p, workspace, p.fwd, sp, Chunk{0, p.P});
  sp.out = out; sp.R_cand = nullptr; sp.C_cand = nullptr;
  return run_sweep(p, p.fwd, sp, st);
}

// ---- frozen modules: step sizes and scale tables packed once, a forward that only enqueues one kernel -------------
namespace {

// The packed buffer of a module: [dA heads][dB heads][split][aux 2][scale groups x heads][group meta groups].  A function
// of heads and sos only.
struct Packed {
  int groups;
  size_t o_dA, o_dB, o_split, o_aux, o_scale, o_meta, bytes;
};
Packed packed_layout(const p4v_matmul_desc* d) {
  Packed k{};
  k.groups = d->sos ? 2 : 1;
  Carver c{0};
  k.o_dA = c.take((size_t)d->heads * 4); k.o_dB = c.take((size_t)d->heads * 4);
  k.o_split = c.take(4); k.o_aux = c.take(2 * 4);
  k.o_scale = c.take((size_t)k.groups * d->heads * 4);
  k.o_meta = c.take((size_t)k.groups * sizeof(GroupMeta));
  k.bytes = c.end;
  return k;
}

}  // namespace

extern "C" int p4v_matmul_pack_bytes(const p4v_matmul_desc* d, size_t* bytes) {
  if (int rc = check_shape(d)) return rc;
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = packed_layout(d).bytes;
  return 0;
}

extern "C" int p4v_matmul_pack(const p4v_matmul_desc* d, const float* A_interval, const float* B_interval, const float* split,
                               void* packed, size_t packed_bytes, void* stream) {
  if (int rc = check_shape(d)) return rc;
  const Packed k = packed_layout(d);
  P4V_REQUIRE(B_interval && packed && (d->sos ? split != nullptr : A_interval != nullptr), "matmul_pack: null pointer");
  P4V_REQUIRE(packed_bytes >= k.bytes, "matmul_pack: packed buffer too small (%zu < %zu)", packed_bytes, k.bytes);
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 15) == 0, "matmul_pack: packed must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int H = d->heads;
  const float qm1 = (float)((1 << (d->A_bit - 1)) - 1);
  // the forward step's groups as the unfrozen forward plans them (build_plan: one plain group; sos: high, low part)
  std::vector<GroupMeta> metas;
  for (int g = 0; g < k.groups; ++g) metas.push_back(GroupMeta{0, (short)g, 0, 0});
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(packed, k.o_meta), metas.data(), metas.size() * sizeof(GroupMeta), cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<float>(packed, k.o_dB), B_interval, (size_t)H * 4, cudaMemcpyDeviceToDevice, st));
  if (d->sos) {
    P4V_CUDA_OK(cudaMemcpyAsync(at<float>(packed, k.o_split), split, 4, cudaMemcpyDeviceToDevice, st));
    sos_aux_kernel<<<1, 1, 0, st>>>(at<float>(packed, k.o_split), qm1, at<float>(packed, k.o_aux), nullptr);
    p4v_count_launch();
    P4V_CUDA_OK(cudaGetLastError());
  } else {
    P4V_CUDA_OK(cudaMemcpyAsync(at<float>(packed, k.o_dA), A_interval, (size_t)H * 4, cudaMemcpyDeviceToDevice, st));
  }
  // the scale table of p4v_matmul_quant_forward: plain dA[h] * dB[h]; sos dB[h] * aux[part]
  StepTablesArgs t{};
  t.kind = d->sos ? 3 : 2; t.n_V = H; t.n_H = 1; t.crb_rows = P4V_CG; t.n_a = 1;
  t.dW = at<float>(packed, d->sos ? k.o_dB : k.o_dA);
  t.dX = at<float>(packed, d->sos ? k.o_aux : k.o_dB);
  t.fixed_meta = at<GroupMeta>(packed, k.o_meta); t.n_fixed_groups = k.groups;
  t.nsg = H; t.fix_scale = at<float>(packed, k.o_scale);
  return p4v_step_tables(t, st);
}

extern "C" int p4v_matmul_frozen_forward(const p4v_matmul_desc* d, const float* A, const long long* A_strides, const float* B,
                                         const long long* B_strides, const void* packed, float* out, void* stream) {
  if (int rc = check_shape(d)) return rc;
  P4V_REQUIRE(A && A_strides && B && B_strides && packed && out, "matmul_frozen_forward: null pointer");
  for (int i = 0; i < 4; ++i)
    P4V_REQUIRE(A_strides[i] >= 0 && B_strides[i] >= 0, "matmul_frozen_forward: negative stride");
  P4V_REQUIRE(A_strides[3] == 1, "matmul_frozen_forward: A must have unit stride along K (got %lld)", A_strides[3]);
  P4V_REQUIRE(B_strides[2] == 1 || B_strides[3] == 1,
              "matmul_frozen_forward: B must have unit stride along K or along N (got %lld, %lld)", B_strides[2], B_strides[3]);
  P4V_REQUIRE(((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(out)) & 3) == 0,
              "matmul_frozen_forward: A, B and out must be 4-byte aligned");
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 15) == 0, "matmul_frozen_forward: packed must be 16-byte aligned");
  const Packed k = packed_layout(d);
  const int A_qmax = 1 << (d->A_bit - 1), B_qmax = 1 << (d->B_bit - 1);
  FwdMMParams q{};
  q.A = A; q.sA_b = A_strides[0]; q.sA_h = A_strides[1]; q.sA_m = A_strides[2];
  q.B = B; q.sB_b = B_strides[0]; q.sB_h = B_strides[1]; q.sB_k = B_strides[2]; q.sB_n = B_strides[3];
  q.out = out;
  q.batch = d->batch; q.heads = d->heads; q.S1 = d->S1; q.S2 = d->S2; q.S3 = d->S3;
  void* pk = const_cast<void*>(packed);         // read only
  q.dA = at<float>(pk, k.o_dA); q.dB = at<float>(pk, k.o_dB); q.split = at<float>(pk, k.o_split);
  q.scale = at<float>(pk, k.o_scale);
  q.A_lo = (float)-A_qmax; q.A_hi = (float)(A_qmax - 1); q.B_lo = (float)-B_qmax; q.B_hi = (float)(B_qmax - 1);
  q.qm1 = (float)(A_qmax - 1);
  return p4v_launch_forward_mm_tc(q, d->sos != 0, (cudaStream_t)stream);
}

// ---- the fused attention core of two frozen MatMul modules (forward_attn_tc.cu) ------------------------------------
extern "C" int p4v_attention_fused_ok(int32_t tokens, int32_t head_dim, int* ok) {
  P4V_REQUIRE(ok != nullptr, "null output");
  *ok = tokens > 0 && tokens <= P4V_ATTN_MAX_TOKENS && head_dim > 0 && head_dim <= P4V_ATTN_MAX_DIM && head_dim % 16 == 0;
  return 0;
}

namespace {

// Validates every argument of an attention call and fills the kernel parameters; `long_seq` applies the long kernel's
// rules (N <= 1024; no q-scaling, bias or mask).  planes non-null: the int8 variant reads q, k and v from the planes of
// the qkv epilogue ([3][batch][heads][N][head_dim], 16-byte aligned, not overlapping out) instead of qkv (null, as are
// qkv_strides).
int attention_params(const p4v_attention_desc* a, const float* qkv, const long long* qkv_strides, const p4v_matmul_desc* mm1,
                     const void* pack1, size_t pack1_bytes, const p4v_matmul_desc* mm2, const void* pack2, size_t pack2_bytes,
                     const float* bias, const float* mask, float* out, bool long_seq, FwdAttnParams& q,
                     const int8_t* planes = nullptr) {
  const char* fn = planes ? "attention_frozen_forward_i8" : long_seq ? "attention_frozen_forward_long" : "attention_frozen_forward";
  P4V_REQUIRE(a && (planes || (qkv && qkv_strides)) && mm1 && pack1 && mm2 && pack2 && out, "%s: null pointer", fn);
  P4V_REQUIRE(a->batch > 0 && a->heads > 0 && a->tokens > 0 && a->head_dim > 0, "%s: empty shape", fn);
  const int max_tokens = long_seq ? P4V_ATTN_LONG_MAX_TOKENS : P4V_ATTN_MAX_TOKENS;
  int ok = 0;
  if (long_seq) p4v_attention_long_ok(a->tokens, a->head_dim, &ok);
  else p4v_attention_fused_ok(a->tokens, a->head_dim, &ok);
  P4V_REQUIRE(a->tokens <= max_tokens, "%s: %d tokens (at most %d)", fn, a->tokens, max_tokens);
  P4V_REQUIRE(ok, "%s: head_dim %d not supported (a multiple of 16, at most %d)", fn, a->head_dim, P4V_ATTN_MAX_DIM);
  if (int rc = check_shape(mm1)) return rc;
  if (int rc = check_shape(mm2)) return rc;
  P4V_REQUIRE(mm1->heads == a->heads && mm2->heads == a->heads,
              "%s: packs made for %d and %d heads, the call has %d", fn, mm1->heads, mm2->heads, a->heads);
  P4V_REQUIRE(!mm1->sos, "%s: matmul1 cannot be split-of-softmax", fn);
  const Packed k1 = packed_layout(mm1), k2 = packed_layout(mm2);
  P4V_REQUIRE(pack1_bytes == k1.bytes && pack2_bytes == k2.bytes,
              "%s: pack sizes %zu and %zu, expected %zu and %zu", fn, pack1_bytes, pack2_bytes, k1.bytes, k2.bytes);
  if (!planes)
    for (int i = 0; i < 4; ++i) P4V_REQUIRE(qkv_strides[i] >= 0, "%s: negative stride", fn);
  P4V_REQUIRE(!a->scale_on_q || a->scale_on_q == 1, "%s: scale_on_q must be 0 or 1", fn);
  if (long_seq) {
    P4V_REQUIRE(!a->scale_on_q, "%s: scale_on_q is not supported (scores * scale after matmul1 only)", fn);
    P4V_REQUIRE(bias == nullptr && mask == nullptr && a->n_windows == 0, "%s: bias and mask are not supported", fn);
  }
  P4V_REQUIRE(mask == nullptr ? a->n_windows == 0 : (a->n_windows > 0 && a->batch % a->n_windows == 0),
              "%s: a mask needs n_windows > 0 dividing batch (and no mask n_windows = 0); got %d for batch %d", fn,
              a->n_windows, a->batch);
  P4V_REQUIRE(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(bias) | reinterpret_cast<uintptr_t>(mask)) & 3) == 0,
              "%s: qkv, bias and mask must be 4-byte aligned", fn);
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(out) & 7) == 0, "%s: out must be 8-byte aligned", fn);
  P4V_REQUIRE(((reinterpret_cast<uintptr_t>(pack1) | reinterpret_cast<uintptr_t>(pack2)) & 15) == 0,
              "%s: packs must be 16-byte aligned", fn);
  if (planes) {
    P4V_REQUIRE((reinterpret_cast<uintptr_t>(planes) & 15) == 0, "%s: planes must be 16-byte aligned", fn);
    const uintptr_t n = (uintptr_t)a->batch * a->tokens * a->heads * a->head_dim, pa = reinterpret_cast<uintptr_t>(planes),
                    po = reinterpret_cast<uintptr_t>(out);
    P4V_REQUIRE(pa + 3 * n <= po || po + 4 * n <= pa, "%s: planes overlap out", fn);
  }
  q = FwdAttnParams{};
  if (planes) {
    q.planes = reinterpret_cast<const uint8_t*>(planes);
  } else {
    q.qkv = qkv; q.s_b = qkv_strides[0]; q.s_n = qkv_strides[1]; q.s_p = qkv_strides[2]; q.s_h = qkv_strides[3];
  }
  q.out = out;
  q.batch = a->batch; q.heads = a->heads; q.N = a->tokens; q.D = a->head_dim;
  q.scale = (float)a->scale; q.scale_on_q = a->scale_on_q;
  q.bias = bias; q.mask = mask; q.n_windows = a->n_windows;
  void* p1 = const_cast<void*>(pack1);          // read only
  void* p2 = const_cast<void*>(pack2);
  const int A1 = 1 << (mm1->A_bit - 1), B1 = 1 << (mm1->B_bit - 1), A2 = 1 << (mm2->A_bit - 1), B2 = 1 << (mm2->B_bit - 1);
  q.dA1 = at<float>(p1, k1.o_dA); q.dB1 = at<float>(p1, k1.o_dB); q.scale1 = at<float>(p1, k1.o_scale);
  q.A1_lo = (float)-A1; q.A1_hi = (float)(A1 - 1); q.B1_lo = (float)-B1; q.B1_hi = (float)(B1 - 1);
  q.dA2 = at<float>(p2, k2.o_dA); q.split2 = at<float>(p2, k2.o_split); q.dB2 = at<float>(p2, k2.o_dB);
  q.scale2 = at<float>(p2, k2.o_scale);
  q.A2_lo = (float)-A2; q.A2_hi = (float)(A2 - 1); q.B2_lo = (float)-B2; q.B2_hi = (float)(B2 - 1);
  q.qm1 = (float)(A2 - 1);
  return 0;
}

}  // namespace

extern "C" int p4v_attention_frozen_forward(const p4v_attention_desc* a, const float* qkv, const long long* qkv_strides,
                                            const p4v_matmul_desc* mm1, const void* pack1, size_t pack1_bytes,
                                            const p4v_matmul_desc* mm2, const void* pack2, size_t pack2_bytes,
                                            const float* bias, const float* mask, float* out, void* stream) {
  FwdAttnParams q;
  if (int rc = attention_params(a, qkv, qkv_strides, mm1, pack1, pack1_bytes, mm2, pack2, pack2_bytes, bias, mask, out, false, q))
    return rc;
  return p4v_launch_forward_attn_tc(q, mm2->sos != 0, (cudaStream_t)stream);
}

// ---- q, k and v as int8 planes from the qkv Linear's epilogue (DESIGN §4.14) ----------------------------------------
extern "C" int p4v_attention_frozen_forward_i8(const p4v_attention_desc* a, const int8_t* planes, const p4v_matmul_desc* mm1,
                                               const void* pack1, size_t pack1_bytes, const p4v_matmul_desc* mm2,
                                               const void* pack2, size_t pack2_bytes, const float* bias, const float* mask,
                                               float* out, void* stream) {
  P4V_REQUIRE(planes, "attention_frozen_forward_i8: null pointer");
  FwdAttnParams q;
  if (int rc = attention_params(a, nullptr, nullptr, mm1, pack1, pack1_bytes, mm2, pack2, pack2_bytes, bias, mask, out, false, q,
                                planes))
    return rc;
  return p4v_launch_forward_attn_tc(q, mm2->sos != 0, (cudaStream_t)stream, true);
}

int p4v_qkv8_steps(const char* fn, const p4v_attention_desc* a, const p4v_matmul_desc* mm1, const void* pack1,
                   size_t pack1_bytes, const p4v_matmul_desc* mm2, const void* pack2, size_t pack2_bytes, FwdQkv8& q) {
  P4V_REQUIRE(a && mm1 && pack1 && mm2 && pack2, "%s: null pointer", fn);
  P4V_REQUIRE(a->batch > 0 && a->heads > 0 && a->tokens > 0 && a->head_dim > 0, "%s: empty shape", fn);
  P4V_REQUIRE(!a->scale_on_q || a->scale_on_q == 1, "%s: scale_on_q must be 0 or 1", fn);
  if (int rc = check_shape(mm1)) return rc;
  if (int rc = check_shape(mm2)) return rc;
  P4V_REQUIRE(mm1->heads == a->heads && mm2->heads == a->heads,
              "%s: packs made for %d and %d heads, the call has %d", fn, mm1->heads, mm2->heads, a->heads);
  P4V_REQUIRE(!mm1->sos, "%s: matmul1 cannot be split-of-softmax", fn);
  const Packed k1 = packed_layout(mm1), k2 = packed_layout(mm2);
  P4V_REQUIRE(pack1_bytes == k1.bytes && pack2_bytes == k2.bytes,
              "%s: pack sizes %zu and %zu, expected %zu and %zu", fn, pack1_bytes, pack2_bytes, k1.bytes, k2.bytes);
  P4V_REQUIRE(((reinterpret_cast<uintptr_t>(pack1) | reinterpret_cast<uintptr_t>(pack2)) & 15) == 0,
              "%s: packs must be 16-byte aligned", fn);
  void* p1 = const_cast<void*>(pack1);          // read only
  void* p2 = const_cast<void*>(pack2);
  const int A1 = 1 << (mm1->A_bit - 1), B1 = 1 << (mm1->B_bit - 1), B2 = 1 << (mm2->B_bit - 1);
  q.N = a->tokens; q.heads = a->heads; q.D = a->head_dim; q.C = a->heads * a->head_dim; q.batch = a->batch;
  q.scale_on_q = a->scale_on_q; q.scale = (float)a->scale;
  q.dq = at<float>(p1, k1.o_dA); q.dk = at<float>(p1, k1.o_dB); q.dv = at<float>(p2, k2.o_dB);
  q.q_lo = (float)-A1; q.q_hi = (float)(A1 - 1); q.k_lo = (float)-B1; q.k_hi = (float)(B1 - 1);
  q.v_lo = (float)-B2; q.v_hi = (float)(B2 - 1);
  return 0;
}

// ---- the long-sequence variant (forward_attn_long_tc.cu) ---------------------------------------------------------
extern "C" int p4v_attention_long_ok(int32_t tokens, int32_t head_dim, int* ok) {
  P4V_REQUIRE(ok != nullptr, "null output");
  *ok = tokens > 0 && tokens <= P4V_ATTN_LONG_MAX_TOKENS && head_dim > 0 && head_dim <= P4V_ATTN_MAX_DIM && head_dim % 16 == 0;
  return 0;
}

extern "C" int p4v_attention_frozen_forward_long(const p4v_attention_desc* a, const float* qkv, const long long* qkv_strides,
                                                 const p4v_matmul_desc* mm1, const void* pack1, size_t pack1_bytes,
                                                 const p4v_matmul_desc* mm2, const void* pack2, size_t pack2_bytes,
                                                 const float* bias, const float* mask, float* out, void* stream) {
  FwdAttnParams q;
  if (int rc = attention_params(a, qkv, qkv_strides, mm1, pack1, pack1_bytes, mm2, pack2, pack2_bytes, bias, mask, out, true, q))
    return rc;
  return p4v_launch_forward_attn_long_tc(q, mm2->sos != 0, (cudaStream_t)stream);
}
