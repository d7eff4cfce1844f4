// C-ABI for the Linear scale-factor search: host-side planning (segments, jobs,
// workspace carving) + the per-step launch sequence.  See include/ptq4vit_b200.h.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <vector>

#include "../../include/ptq4vit_b200.h"
#include "prep.cuh"
#include "gram.cuh"

int p4v_num_sms();

// ---------------------------------------------------------------- error / misc
static thread_local char g_err[512] = "";
static long long g_launches = 0;
extern "C" __attribute__((visibility("default"))) void p4v_set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}
extern "C" const char* p4v_last_error(void) { return g_err; }
extern "C" int p4v_version(void) { return 100; }
extern "C" long long p4v_launch_count(void) { return g_launches; }
void p4v_count_launch() { ++g_launches; }

// ---- live kernel timing (bench.py's roofline) ---------------------------------
// While enabled every tensor-core launch (slab sweep, Gram GEMM) is bracketed by CUDA events on its own stream and
// recorded with its kind and the tensor-core operations (2*MAC) it executes.
enum { P4V_PROF_SWEEP_BF16 = 0, P4V_PROF_SWEEP_INT8 = 1, P4V_PROF_GRAM_GEMM = 2, P4V_PROF_KINDS = 3 };
static bool g_prof = false;
struct ProfRec { cudaEvent_t e0, e1; int kind; double ops; int n_cand, nfg, ncg, nfj, ncj, out; long long tiles; };
static std::vector<ProfRec> g_prof_recs;
static std::vector<cudaEvent_t> g_prof_pool;
static cudaEvent_t prof_event() {
  if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}
bool p4v_prof_on() { return g_prof; }
void p4v_prof_begin(cudaStream_t st, cudaEvent_t* e0) { *e0 = prof_event(); cudaEventRecord(*e0, st); }
void p4v_prof_end(cudaStream_t st, cudaEvent_t e0, int kind, double ops) {
  cudaEvent_t e1 = prof_event(); cudaEventRecord(e1, st);
  g_prof_recs.push_back(ProfRec{e0, e1, kind, ops, 0, 0, 0, 0, 0, 0, 0});
}
extern "C" int p4v_profile_enable(int on) { g_prof = on != 0; return 0; }
// out[0..2] ms per kind (bf16 sweep, int8 sweep, Gram GEMM), out[3..5] executed ops, out[6..8] launches,
// out[9..11] the longest single launch: ms, ops, kind.  Synchronises the recorded events and clears the record.
extern "C" int p4v_profile_collect_kinds(double* out, int n) {
  P4V_REQUIRE(out && n >= 12, "profile_collect_kinds: need 12 doubles");
  for (int i = 0; i < 12; ++i) out[i] = 0.0;
  static const bool log_each = getenv("P4V_PROFILE_LOG") != nullptr;   // debug: one stderr line per launch
  for (auto& r : g_prof_recs) {
    P4V_CUDA_OK(cudaEventSynchronize(r.e1));
    float t = 0.f;
    P4V_CUDA_OK(cudaEventElapsedTime(&t, r.e0, r.e1));
    out[r.kind] += t; out[3 + r.kind] += r.ops; out[6 + r.kind] += 1.0;
    if (t > out[9]) { out[9] = t; out[10] = r.ops; out[11] = r.kind; }
    if (log_each)
      fprintf(stderr, "[p4v launch] %8.1f us kind=%d cand=%d fixed_groups=%d cand_groups=%d fixed_jobs=%d cand_jobs=%d out=%d tiles=%lld  %.1f TOP/s\n",
              t * 1e3, r.kind, r.n_cand, r.nfg, r.ncg, r.nfj, r.ncj, r.out, r.tiles, r.ops / (t * 1e-3) / 1e12);
    g_prof_pool.push_back(r.e0); g_prof_pool.push_back(r.e1);
  }
  g_prof_recs.clear();
  return 0;
}
extern "C" int p4v_profile_collect(double* sweep_ms, long long* sweep_launches, double* executed_ops) {
  double o[12];
  int rc = p4v_profile_collect_kinds(o, 12);
  if (rc) return rc;
  if (sweep_ms) *sweep_ms = o[0] + o[1];
  if (sweep_launches) *sweep_launches = (long long)(o[6] + o[7]);
  if (executed_ops) *executed_ops = o[3] + o[4];
  return 0;
}
// tensor-core work of one sweep launch: every job multiplies a 128x128 tile over kb bytes of K
static double sweep_ops(const SweepParams& sp, const P4VJob* host_jobs) {
  double kf = 0.0, kc = 0.0;
  const double ew = sp.is_int8 ? 1.0 : 2.0;
  for (int j = 0; j < sp.n_fixed_jobs; ++j) kf += host_jobs[j].kb * p4v_job_nsub(host_jobs[j]) / ew;
  for (int j = 0; j < sp.n_cand_jobs; ++j) kc += host_jobs[sp.n_fixed_jobs + j].kb * p4v_job_nsub(host_jobs[sp.n_fixed_jobs + j]) / ew;
  const double tiles = (double)sp.P * sp.tiles_m * sp.tiles_n;
  return 2.0 * P4V_TILE * P4V_TILE * tiles * (kf + kc * sp.n_cand);
}
int p4v_run_sweep(const SweepParams& sp, const P4VJob* host_jobs, int kernel, cudaStream_t st) {
  ++g_launches;
  cudaEvent_t e0 = nullptr;
  if (g_prof) p4v_prof_begin(st, &e0);
  int rc = kernel == P4V_KERNEL_SIMT ? p4v_launch_sweep_simt(sp, st) : p4v_launch_sweep_tc(sp, host_jobs, p4v_num_sms(), st);
  if (g_prof) {
    p4v_prof_end(st, e0, sp.is_int8 ? P4V_PROF_SWEEP_INT8 : P4V_PROF_SWEEP_BF16, sweep_ops(sp, host_jobs));
    ProfRec& r = g_prof_recs.back();
    r.n_cand = sp.n_cand; r.nfg = sp.n_fixed_groups; r.ncg = sp.n_cand_groups; r.nfj = sp.n_fixed_jobs; r.ncj = sp.n_cand_jobs;
    r.out = sp.out != nullptr; r.tiles = (long long)sp.P * sp.tiles_m * sp.tiles_n;
  }
  return rc;
}

int p4v_num_sms();
int p4v_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

namespace {

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
// bytes of K of one bf16 term of the Gram operands for n tokens
inline unsigned gram_term(int n) { return (unsigned)align_up((size_t)n * 2, 32); }

struct BSeg { int k0, klen, h, a, kb; int woff, xoff_p, xoff_n, xcoff; };   // offsets: bytes in the padded row
struct Step { int job_off, nfj, ncj, nfg, ncg, meta_fix, meta_cand, commit_off, ncommit, commit_chunks; };

struct LinPlan {
  p4v_linear_desc d;
  bool i8, twin;
  int ew, M, K, O, tiles_m, tiles_o, nsg, crb_rows, crb_cols, crb_acts, w_qmax, a_qmax;
  bool chunked; int chunk_rows, tiles_mc;   // rows of one chunk (M unchunked) and their 128-row tiles: the X images hold one chunk
  float d_neg;
  std::vector<BSeg> segs;
  int KB_W, KB_X, KB_Xc;
  std::vector<P4VJob> jobs; std::vector<GroupMeta> metas; std::vector<CommitSeg> commits;
  std::vector<P4VSeg> segsW, segsX, segsXc;
  std::vector<Step> wsteps, xsteps;
  Step fwd;   // quant_forward: every segment is a fixed group
  // normal-equation W search (gram.cu)
  bool gram; int g_ks, g_Mp, g_npairs, g_tiles_p, g_ldH, g_nmblk; unsigned g_term_bytes;
  size_t o_E, o_XqT, o_G2T, o_Z, o_H, o_Upart, o_E2part, o_U, o_E2, o_dprev, o_D, o_segsG;
  int g_osplit, g_opb;
  std::vector<float> factors;
  int max_groups;
  // workspace offsets
  size_t o_factors, o_keys, o_dW0, o_dW, o_dX0, o_dX, o_gscale, o_scores, o_best, o_fix, o_candA, o_candB, o_jobs,
      o_metas, o_segsW, o_segsX, o_segsXc, o_commits, o_partial, o_Wcur, o_Xcur, o_Wcand, o_Xcand, total;
  // int8 activation step of a bf16 layer (build_plan): K bytes of its images, its jobs and segment tables, the step (same
  // groups and scale tables as xsteps[0], jobs in jobs8) and its buffers inside the bf16 candidate activation region
  bool x8; int KB8;
  std::vector<P4VJob> jobs8; std::vector<P4VSeg> segsW8, segsXc8;
  Step xstep8;
  size_t o_Xcand8, o_Wcur8, o_jobs8, o_segsW8, o_segsXc8;
};

void add_group(std::vector<P4VJob>& jobs, int r_off_bytes, int c_off_bytes, int kb, uint8_t src_flags, int group_idx, int& njobs) {
  for (int b = 0; b < kb; b += P4V_JOB_KB) {
    P4VJob j{};
    const int len = std::min(P4V_JOB_KB, kb - b);
    j.r_off = (uint32_t)(r_off_bytes + b) * P4V_TILE;
    j.c_off = (uint32_t)(c_off_bytes + b) * P4V_TILE;
    j.kb = (uint8_t)len;
    j.flags = src_flags | (b == 0 ? P4V_JOB_FIRST : 0) | (b + len >= kb ? P4V_JOB_LAST : 0);
    j.group = (uint8_t)group_idx;
    jobs.push_back(j);
    ++njobs;
  }
}

// Candidate jobs whose row operand does not depend on the candidate (W steps): keep it resident in shared memory.
void mark_resident(LinPlan& p, const Step& st) {
  uint32_t total = 0;
  for (int j = 0; j < st.ncj; ++j) total += (uint32_t)p.jobs[st.job_off + st.nfj + j].kb * P4V_TILE;
  if (total == 0 || total > 60 * 1024) return;
  uint32_t off = 0;
  for (int j = 0; j < st.ncj; ++j) {
    P4VJob& jb = p.jobs[st.job_off + st.nfj + j];
    if (jb.flags & P4V_JOB_RCAND) return;
    jb.flags |= P4V_JOB_RRES; jb.res_off = off; off += (uint32_t)jb.kb * P4V_TILE;
  }
}

// Merge runs of single-job accumulator groups whose K slabs are adjacent in BOTH operand images into one
// stage load with several sub-accumulators (one bulk copy / one stage handshake for up to 128 bytes of K).
void batch_jobs(std::vector<P4VJob>& jobs, int first, int& count) {
  std::vector<P4VJob> out;
  for (int j = 0; j < count; ++j) {
    const P4VJob jb = jobs[first + j];
    const bool single = (jb.flags & P4V_JOB_FIRST) && (jb.flags & P4V_JOB_LAST) && !(jb.flags & (P4V_JOB_RRES | P4V_JOB_CCAND));
    if (single && !out.empty()) {
      P4VJob& prev = out.back();
      const unsigned n = p4v_job_nsub(prev);
      const bool prev_single = (prev.flags & P4V_JOB_FIRST) && (prev.flags & P4V_JOB_LAST);
      if (prev_single && prev.flags == jb.flags && prev.kb == jb.kb && (n + 1) * jb.kb <= P4V_JOB_KB &&
          prev.r_off + n * jb.kb * P4V_TILE == jb.r_off && prev.c_off + n * jb.kb * P4V_TILE == jb.c_off &&
          prev.group + n == jb.group) {
        prev.nsub = (uint8_t)(n + 1);
        continue;
      }
    }
    out.push_back(jb);
  }
  std::copy(out.begin(), out.end(), jobs.begin() + first);
  jobs.erase(jobs.begin() + first + out.size(), jobs.begin() + first + count);
  count = (int)out.size();
}

// x8_ok: the caller passes the activations to every activation step (p4v_linear_calibrate), which the int8 activation
// step needs to rebuild the bf16 current activation image after its pick.
int build_plan(const p4v_linear_desc* d, LinPlan& p, bool with_search, bool x8_ok = false) {
  P4V_REQUIRE(d != nullptr, "null desc");
  p.d = *d;
  p.M = d->rows; p.K = d->in_features; p.O = d->out_features;
  P4V_REQUIRE(p.M > 0 && p.K > 0 && p.O > 0, "linear: empty shape (rows=%d in=%d out=%d)", p.M, p.K, p.O);
  P4V_REQUIRE(d->n_V >= 1 && d->n_H >= 1 && d->n_a >= 1, "linear: n_V/n_H/n_a must be >= 1");
  P4V_REQUIRE(p.K % d->n_H == 0 && p.K % d->n_a == 0 && p.O % d->n_V == 0,
              "linear: in_features must divide by n_H and n_a, out_features by n_V (reference views, linear.py:117-119)");
  P4V_REQUIRE(d->tokens >= 1 && p.M % d->tokens == 0, "linear: rows must be a multiple of tokens");
  P4V_REQUIRE(d->w_bit >= 2 && d->w_bit <= 8 && d->a_bit >= 2 && d->a_bit <= 8, "linear: bit widths must be in [2,8]");
  P4V_REQUIRE(d->eq_n >= 1 && d->eq_n <= P4V_MAX_CAND, "linear: eq_n must be in [1,%d]", P4V_MAX_CAND);
  P4V_REQUIRE(d->rows_per_chunk >= 0 && d->rows_per_chunk % P4V_TILE == 0 && d->rows_per_chunk <= p.M,
              "linear: rows_per_chunk must be a multiple of %d in [0, rows=%d] (got %d; 0 = whole layer)", P4V_TILE, p.M,
              d->rows_per_chunk);
  p.crb_rows = p.O / d->n_V; p.crb_cols = p.K / d->n_H; p.crb_acts = p.K / d->n_a;
  P4V_REQUIRE(d->n_V == 1 || p.crb_rows % P4V_CG == 0, "linear: out_features/n_V must be a multiple of 16 (got %d)", p.crb_rows);
  p.w_qmax = 1 << (d->w_bit - 1); p.a_qmax = 1 << (d->a_bit - 1);
  p.twin = d->post_gelu != 0;
  p.d_neg = (float)(0.16997124254703522 / (double)p.a_qmax);
  p.tiles_m = p4v_cdiv(p.M, P4V_TILE); p.tiles_o = p4v_cdiv(p.O, P4V_TILE);
  p.chunked = with_search && d->rows_per_chunk > 0;
  p.chunk_rows = p.chunked ? d->rows_per_chunk : p.M; p.tiles_mc = p4v_cdiv(p.chunk_rows, P4V_TILE);
  p.nsg = p.tiles_o * P4V_TILE_CG;

  // K segments = intersections of the weight column blocks and the activation chunks
  std::vector<int> cuts;
  for (int h = 0; h <= d->n_H; ++h) cuts.push_back(h * p.crb_cols);
  for (int a = 0; a <= d->n_a; ++a) cuts.push_back(a * p.crb_acts);
  std::sort(cuts.begin(), cuts.end());
  cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
  int min_len = p.K;
  for (size_t i = 0; i + 1 < cuts.size(); ++i) min_len = std::min(min_len, cuts[i + 1] - cuts[i]);
  if (d->operand == P4V_OPERAND_INT8) p.i8 = true;
  else if (d->operand == P4V_OPERAND_BF16) p.i8 = false;
  // Automatic choice: short K segments (< 64 elements) take integer-valued bf16 for the weight steps, the residual and the
  // quantised forward.  The activation step of such a layer may still run on int8 images (x8 below).
  else p.i8 = min_len >= 64;
  p.ew = p.i8 ? 1 : 2;
  p.segs.clear();
  int off = 0;
  for (size_t i = 0; i + 1 < cuts.size(); ++i) {
    BSeg s{};
    s.k0 = cuts[i]; s.klen = cuts[i + 1] - cuts[i];
    s.h = s.k0 / p.crb_cols; s.a = s.k0 / p.crb_acts;
    s.kb = (int)align_up((size_t)s.klen * p.ew, 32);
    s.woff = off; s.xoff_p = off; s.xcoff = off;
    off += s.kb;
    p.segs.push_back(s);
  }
  p.KB_W = off; p.KB_Xc = off;
  p.KB_X = p.twin ? 2 * off : off;
  for (auto& s : p.segs) s.xoff_n = p.twin ? off + s.xoff_p : -1;
  P4V_REQUIRE((size_t)p.KB_X * P4V_TILE < (1ull << 32), "linear: in_features too large");

  // quantisation segment tables
  p.segsW.clear(); p.segsX.clear(); p.segsXc.clear();
  for (auto& s : p.segs) {
    P4VSeg w{s.k0, s.klen, s.woff * P4V_TILE, s.h, 0.f, (float)-p.w_qmax, (float)(p.w_qmax - 1), 0, 0.f, 0, 0};
    p.segsW.push_back(w);
    P4VSeg x{s.k0, s.klen, s.xoff_p * P4V_TILE, s.a, 0.f, p.twin ? 0.f : (float)-p.a_qmax, (float)(p.a_qmax - 1), 0, 0.f, 0, 0};
    p.segsX.push_back(x);
    P4VSeg xc = x; xc.dst_off = s.xcoff * P4V_TILE;
    p.segsXc.push_back(xc);
  }
  if (p.twin)
    for (auto& s : p.segs) {
      P4VSeg n{s.k0, s.klen, s.xoff_n * P4V_TILE, s.a, p.d_neg, (float)-p.a_qmax, 0.f, 0, 0.f, 0, 0};
      p.segsX.push_back(n);
    }

  // candidate factors (python floats -> fp32, linear.py:544-545)
  p.factors.resize(d->eq_n + 1);
  for (int i = 0; i <= d->eq_n; ++i) p.factors[i] = (float)(d->eq_alpha + i * (d->eq_beta - d->eq_alpha) / d->eq_n);

  // steps
  p.jobs.clear(); p.metas.clear(); p.commits.clear(); p.wsteps.clear(); p.xsteps.clear();
  p.max_groups = 1;
  auto begin_step = [&](Step& st) { st = Step{}; st.job_off = (int)p.jobs.size(); st.commit_off = (int)p.commits.size(); };
  auto fixed_group = [&](Step& st, const BSeg& s, bool neg) {
    add_group(p.jobs, neg ? s.xoff_n : s.xoff_p, s.woff, s.kb, 0, st.nfg, st.nfj);
    p.metas.push_back(GroupMeta{(short)s.h, (short)s.a, (short)(neg ? 1 : 0), 0});
    ++st.nfg;
  };
  if (with_search) {
    for (int h = 0; h < d->n_H; ++h) {
      Step st; begin_step(st);
      st.meta_fix = (int)p.metas.size();
      for (auto& s : p.segs) if (s.h != h) { fixed_group(st, s, false); if (p.twin) fixed_group(st, s, true); }
      st.meta_cand = (int)p.metas.size();
      for (auto& s : p.segs) if (s.h == h) {
        add_group(p.jobs, s.xoff_p, s.woff, s.kb, P4V_JOB_CCAND, st.ncg, st.ncj);
        p.metas.push_back(GroupMeta{(short)s.h, (short)s.a, 0, 0}); ++st.ncg;
        if (p.twin) {
          add_group(p.jobs, s.xoff_n, s.woff, s.kb, P4V_JOB_CCAND, st.ncg, st.ncj);
          p.metas.push_back(GroupMeta{(short)s.h, (short)s.a, 1, 0}); ++st.ncg;
        }
        p.commits.push_back(CommitSeg{s.woff * P4V_TILE, s.woff * P4V_TILE, s.kb});
        st.commit_chunks += s.kb / 16; ++st.ncommit;
      }
      mark_resident(p, st);
      batch_jobs(p.jobs, st.job_off, st.nfj);
      p.wsteps.push_back(st);
    }
    for (int a = 0; a < d->n_a; ++a) {
      Step st; begin_step(st);
      st.meta_fix = (int)p.metas.size();
      for (auto& s : p.segs) { if (s.a != a) fixed_group(st, s, false); if (p.twin) fixed_group(st, s, true); }
      st.meta_cand = (int)p.metas.size();
      for (auto& s : p.segs) if (s.a == a) {
        add_group(p.jobs, s.xcoff, s.woff, s.kb, P4V_JOB_RCAND, st.ncg, st.ncj);
        p.metas.push_back(GroupMeta{(short)s.h, (short)s.a, 0, 0}); ++st.ncg;
        p.commits.push_back(CommitSeg{s.xcoff * P4V_TILE, s.xoff_p * P4V_TILE, s.kb});
        st.commit_chunks += s.kb / 16; ++st.ncommit;
      }
      {   // candidates change the row operand only: keep the tile's weight image resident when it fits
        int ncj = st.ncj; batch_jobs(p.jobs, st.job_off + st.nfj, ncj); st.ncj = ncj;
        batch_jobs(p.jobs, st.job_off, st.nfj);
        if ((size_t)p.KB_W * P4V_TILE <= 100 * 1024 && getenv("P4V_NO_CRES") == nullptr)
          for (int j = 0; j < st.nfj + st.ncj; ++j) p.jobs[st.job_off + j].flags |= P4V_JOB_CRES;
      }
      p.xsteps.push_back(st);
    }
  }
  {
    Step st; begin_step(st);
    st.meta_fix = (int)p.metas.size();
    for (auto& s : p.segs) { fixed_group(st, s, false); if (p.twin) fixed_group(st, s, true); }
    st.meta_cand = (int)p.metas.size();
    batch_jobs(p.jobs, st.job_off, st.nfj);
    p.fwd = st;
  }
  auto check = [&](const Step& st) {
    return st.nfj + st.ncj <= P4V_MAX_JOBS && st.nfg <= P4V_MAX_GROUPS && st.ncg <= P4V_MAX_GROUPS;
  };
  for (auto& st : p.wsteps) { P4V_REQUIRE(check(st), "linear: too many K segments for one step (n_H/n_a/in_features)"); p.max_groups = std::max(p.max_groups, std::max(st.nfg, st.ncg)); }
  for (auto& st : p.xsteps) { P4V_REQUIRE(check(st), "linear: too many K segments for one step (n_H/n_a/in_features)"); p.max_groups = std::max(p.max_groups, std::max(st.nfg, st.ncg)); }
  P4V_REQUIRE(check(p.fwd), "linear: too many K segments for quant_forward");
  p.max_groups = std::max(p.max_groups, p.fwd.nfg);

  // workspace carving
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
  const int n_c = d->eq_n;
  p.o_factors = take((n_c + 1) * 4);
  p.o_keys = take((d->n_V * d->n_H + d->n_a + 1) * 4);
  p.o_dW0 = take(d->n_V * d->n_H * 4); p.o_dW = take(d->n_V * d->n_H * 4);
  p.o_dX0 = take(d->n_a * 4); p.o_dX = take(d->n_a * 4);
  p.o_gscale = take(4);
  p.o_scores = take((size_t)n_c * (p.nsg + d->n_V * (size_t)(1 + p4v_cdiv(p.crb_rows, 2))) * 8);
  p.o_best = take(std::max(d->n_V, 1) * 4);
  p.o_fix = take((size_t)p.max_groups * p.nsg * 4);
  p.o_candA = take((size_t)n_c * p.nsg * 4);
  p.o_candB = take((size_t)p.max_groups * p.nsg * 4);
  p.o_jobs = take(p.jobs.size() * sizeof(P4VJob));
  p.o_metas = take(p.metas.size() * sizeof(GroupMeta));
  p.o_segsW = take(p.segsW.size() * sizeof(P4VSeg));
  p.o_segsX = take(p.segsX.size() * sizeof(P4VSeg));
  p.o_segsXc = take(p.segsXc.size() * sizeof(P4VSeg));
  p.o_commits = take(std::max<size_t>(1, p.commits.size()) * sizeof(CommitSeg));
  p.o_partial = take(with_search ? (size_t)p.tiles_mc * p.tiles_o * n_c * 32 * 4 : 4);
  p.o_Wcur = take((size_t)p.tiles_o * P4V_TILE * p.KB_W);
  p.o_Xcur = take((size_t)p.tiles_mc * P4V_TILE * p.KB_X);
  p.o_Wcand = take(with_search ? (size_t)n_c * p.tiles_o * P4V_TILE * p.KB_W : 4);
  p.o_Xcand = take(with_search ? (size_t)n_c * p.tiles_mc * P4V_TILE * p.KB_Xc : 4);
  // normal-equation W search: narrow column blocks inside one activation chunk, plain (non twin) activations.
  // Chunked: the residual e and the token-major activations stay whole-layer, the (gs*g)^2 and pair images hold one chunk
  // of rows; H, U and sum (g e)^2 accumulate over the chunks.
  p.gram = false;
  {
    const char* env = getenv("P4V_GRAM");
    const bool want = with_search && (env ? atoi(env) != 0 : true) && d->kernel == P4V_KERNEL_TCGEN05;
    const unsigned term = gram_term(p.chunk_rows);
    if (want && !p.twin && p.crb_cols <= 64 && p.crb_cols % 4 == 0 && p.crb_acts % p.crb_cols == 0) {
      p.gram = true;
      p.g_ks = p.crb_cols; p.g_term_bytes = term;
      p.g_Mp = (int)align_up((size_t)p.M, 16) + 16;
      p.g_npairs = p.g_ks * (p.g_ks + 1) / 2;
      p.g_tiles_p = p4v_cdiv(p.g_npairs * d->n_H, GRAM_PT); p.g_ldH = p.g_tiles_p * GRAM_PT;   // all column blocks side by side
      p.g_nmblk = p4v_gram_update_splits(p.O, p.chunk_rows);
      const size_t KBg = 2 * (size_t)term;
      p.o_E = take((size_t)p.M * p.O * 4);
      p.o_XqT = take((size_t)p.K * p.g_Mp);
      p.o_G2T = take((size_t)p.tiles_o * P4V_TILE * KBg);
      p.o_Z = take((size_t)p.g_tiles_p * GRAM_PT * KBg);
      p.o_H = take((size_t)p.O * p.g_ldH * 4);
      p.o_Upart = take((size_t)p.g_nmblk * p.O * p.g_ks * 4);
      p.o_E2part = take((size_t)p.g_nmblk * p.O * 4);
      p.o_U = take((size_t)p.O * p.g_ks * 4); p.o_E2 = take((size_t)p.O * 4);
      p.g_osplit = std::max(1, p4v_cdiv(p.crb_rows, 2)); p.g_opb = p4v_cdiv(p.crb_rows, p.g_osplit);
      p.o_dprev = take((size_t)d->n_V * 4);
      p.o_D = take((size_t)p.O * 64 * 4);
      p.o_segsG = take((p.chunked ? 4 : 2) * sizeof(P4VSeg));   // chunked: a full chunk and the last one
    }
  }
  // Activation step of a layer that chose bf16 automatically, when the step has no fixed groups (one activation chunk,
  // not post-GELU): run it on int8 images.  The tile's int8 weight image (half the bf16 bytes) then stays resident in
  // shared memory, only the candidate activation slab streams, and the tensor cores run at the int8 rate.  bf16 with
  // fp32 accumulators and int8 with s32 accumulators form the same exact integer products (below 2^24), and the
  // epilogue runs the same fp32 operations per group in the same order, so score tables and picks are bit-identical.
  // The int8 candidate planes, an int8 copy of the current weight image and the step's job and segment tables take the
  // place of the bf16 candidate activation planes, which only the activation steps read: the workspace does not grow.
  // The weight steps, the residual sweep and the quantised forward keep the bf16 images.
  p.x8 = false;
  if (x8_ok && d->operand == P4V_OPERAND_AUTO && !p.i8 && d->kernel == P4V_KERNEL_TCGEN05 && p.xsteps.size() == 1 &&
      p.xsteps[0].nfg == 0 && getenv("P4V_NO_CRES") == nullptr) {
    p.jobs8.clear(); p.segsW8.clear(); p.segsXc8.clear();
    Step& st = p.xstep8;
    st = p.xsteps[0]; st.job_off = 0; st.nfj = 0; st.ncj = 0;
    int off8 = 0;
    for (size_t i = 0; i < p.segs.size(); ++i) {   // one candidate group per segment, in the order of the bf16 step
      const int kb = (int)align_up((size_t)p.segs[i].klen, 32);
      P4VSeg w = p.segsW[i], x = p.segsXc[i];
      w.dst_off = x.dst_off = off8 * P4V_TILE;
      p.segsW8.push_back(w); p.segsXc8.push_back(x);
      add_group(p.jobs8, off8, off8, kb, P4V_JOB_RCAND, (int)i, st.ncj);
      off8 += kb;
    }
    p.KB8 = off8;
    batch_jobs(p.jobs8, 0, st.ncj);
    for (auto& j : p.jobs8) j.flags |= P4V_JOB_CRES;
    size_t o8 = p.o_Xcand;
    auto take8 = [&](size_t bytes) { size_t r = o8; o8 = align_up(o8 + bytes, 256); return r; };
    p.o_Xcand8 = take8((size_t)n_c * p.tiles_mc * P4V_TILE * p.KB8);
    p.o_Wcur8 = take8((size_t)p.tiles_o * P4V_TILE * p.KB8);
    p.o_jobs8 = take8(p.jobs8.size() * sizeof(P4VJob));
    p.o_segsW8 = take8(p.segsW8.size() * sizeof(P4VSeg));
    p.o_segsXc8 = take8(p.segsXc8.size() * sizeof(P4VSeg));
    const size_t region_end = align_up(p.o_Xcand + (size_t)n_c * p.tiles_mc * P4V_TILE * p.KB_Xc, 256);
    p.x8 = (size_t)p.KB8 * P4V_TILE <= 100 * 1024 && o8 <= region_end && st.ncj <= P4V_MAX_JOBS;
  }
  p.total = o;
  return 0;
}

template <class T> T* at(void* ws, size_t off) { return reinterpret_cast<T*>(static_cast<uint8_t*>(ws) + off); }

int upload_tables(const LinPlan& p, void* ws, cudaStream_t st) {
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_factors), p.factors.data(), p.factors.size() * 4, cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_jobs), p.jobs.data(), p.jobs.size() * sizeof(P4VJob), cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_metas), p.metas.data(), p.metas.size() * sizeof(GroupMeta), cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segsW), p.segsW.data(), p.segsW.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segsX), p.segsX.data(), p.segsX.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segsXc), p.segsXc.data(), p.segsXc.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  if (!p.commits.empty())
    P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_commits), p.commits.data(), p.commits.size() * sizeof(CommitSeg), cudaMemcpyHostToDevice, st));
  if (p.x8) {
    P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_jobs8), p.jobs8.data(), p.jobs8.size() * sizeof(P4VJob), cudaMemcpyHostToDevice, st));
    P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segsW8), p.segsW8.data(), p.segsW8.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
    P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segsXc8), p.segsXc8.data(), p.segsXc8.size() * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  }
  if (p.gram) {
    const int n_last = p.M - (p4v_cdiv(p.M, p.chunk_rows) - 1) * p.chunk_rows;
    const int nr[2] = {p.chunk_rows, n_last};
    P4VSeg sg[4];
    for (int i = 0; i < 2; ++i) {
      sg[2 * i] = P4VSeg{0, nr[i], 0, 0, 0.f, 0.f, 0.f, 0, 0.f, 1, 1};
      sg[2 * i + 1] = P4VSeg{0, nr[i], (int)(gram_term(nr[i]) * P4V_TILE), 0, 0.f, 0.f, 0.f, 0, 0.f, 2, 1};
    }
    P4V_CUDA_OK(cudaMemcpyAsync(at<void>(ws, p.o_segsG), sg, (p.chunked ? 4 : 2) * sizeof(P4VSeg), cudaMemcpyHostToDevice, st));
  }
  return 0;
}

// x8: the int8 current weight image of the int8 activation step (cand must be false)
int quant_W(const LinPlan& p, void* ws, const float* W, const float* delta, bool cand, cudaStream_t st, bool x8 = false) {
  QuantImageArgs q{};
  q.src = W; q.ld = p.K; q.prob_stride = 0; q.src_transposed = 0;
  q.P = 1; q.rows = p.O; q.tiles = p.tiles_o;
  q.dst = at<uint8_t>(ws, x8 ? p.o_Wcur8 : cand ? p.o_Wcand : p.o_Wcur);
  q.tile_bytes = (unsigned long long)P4V_TILE * (x8 ? p.KB8 : p.KB_W); q.plane_stride = q.tile_bytes * p.tiles_o;
  q.n_planes = cand ? p.d.eq_n : 1;
  q.factors = cand ? at<float>(ws, p.o_factors) : nullptr;
  q.delta = delta; q.rows_per_block = p.crb_rows; q.d_stride = p.d.n_H; q.d_mod = 1;
  q.segs = at<P4VSeg>(ws, x8 ? p.o_segsW8 : p.o_segsW); q.nseg = (int)p.segsW.size(); q.is_int8 = x8 || p.i8;
  return p4v_quant_image(q, st);
}

// rows [r0, r0 + n) of the layer: one chunk (or all rows)
struct Rows { int r0, n; };
Rows all_rows(const LinPlan& p) { return Rows{0, p.M}; }

// The candidate planes are int8 when the activation step runs on int8 images (p.x8)
int quant_X(const LinPlan& p, void* ws, const float* x, const float* delta, bool cand, Rows r, cudaStream_t st) {
  const bool x8 = cand && p.x8;
  QuantImageArgs q{};
  q.src = x + (size_t)r.r0 * p.K; q.ld = p.K; q.prob_stride = 0; q.src_transposed = 0;
  q.P = 1; q.rows = r.n; q.tiles = p4v_cdiv(r.n, P4V_TILE);
  q.dst = at<uint8_t>(ws, x8 ? p.o_Xcand8 : cand ? p.o_Xcand : p.o_Xcur);
  q.tile_bytes = (unsigned long long)P4V_TILE * (x8 ? p.KB8 : cand ? p.KB_Xc : p.KB_X); q.plane_stride = q.tile_bytes * q.tiles;
  q.n_planes = cand ? p.d.eq_n : 1;
  q.factors = cand ? at<float>(ws, p.o_factors) : nullptr;
  q.delta = delta; q.rows_per_block = p.M + P4V_TILE; q.d_stride = 0; q.d_mod = 1;   // single row block: any row range
  q.segs = at<P4VSeg>(ws, x8 ? p.o_segsXc8 : cand ? p.o_segsXc : p.o_segsX); q.nseg = (int)(cand ? p.segsXc.size() : p.segsX.size());
  q.is_int8 = x8 || p.i8;
  return p4v_quant_image(q, st);
}

void fill_sweep(const LinPlan& p, void* ws, const Step& s, SweepParams& sp, Rows r) {
  const int tiles_m = p4v_cdiv(r.n, P4V_TILE);
  sp = SweepParams{};
  sp.R_cur = at<uint8_t>(ws, p.o_Xcur); sp.R_cand = at<uint8_t>(ws, p.o_Xcand);
  sp.C_cur = at<uint8_t>(ws, p.o_Wcur); sp.C_cand = at<uint8_t>(ws, p.o_Wcand);
  sp.R_tile_bytes = (unsigned long long)P4V_TILE * p.KB_X; sp.C_tile_bytes = (unsigned long long)P4V_TILE * p.KB_W;
  sp.R_cand_tile_bytes = (unsigned long long)P4V_TILE * p.KB_Xc; sp.C_cand_tile_bytes = sp.C_tile_bytes;
  sp.R_cand_stride = sp.R_cand_tile_bytes * tiles_m; sp.C_cand_stride = sp.C_cand_tile_bytes * p.tiles_o;
  sp.P = 1; sp.M = r.n; sp.N = p.O; sp.tiles_m = tiles_m; sp.tiles_n = p.tiles_o;
  sp.ld = p.O; sp.prob_stride = 0;
  sp.gscale = at<float>(ws, p.o_gscale);
  sp.jobs = at<P4VJob>(ws, p.o_jobs) + s.job_off;
  sp.n_fixed_jobs = s.nfj; sp.n_cand_jobs = s.ncj; sp.n_fixed_groups = s.nfg; sp.n_cand_groups = s.ncg;
  sp.fix_scale = at<float>(ws, p.o_fix); sp.candA = at<float>(ws, p.o_candA); sp.candB = at<float>(ws, p.o_candB);
  sp.nsg = p.nsg; sp.sg_mode = P4V_SG_COLUMN;
  sp.n_cand = p.d.eq_n;
  sp.partial = at<float>(ws, p.o_partial);
  sp.is_int8 = p.i8;
}
void fill_sweep(const LinPlan& p, void* ws, const Step& s, SweepParams& sp) { fill_sweep(p, ws, s, sp, all_rows(p)); }

// The int8 activation step: int8 candidate activation planes against the resident int8 current weight image
void fill_sweep_x8(const LinPlan& p, void* ws, SweepParams& sp, Rows r) {
  fill_sweep(p, ws, p.xstep8, sp, r);
  sp.R_cand = at<uint8_t>(ws, p.o_Xcand8); sp.C_cur = at<uint8_t>(ws, p.o_Wcur8);
  sp.R_cand_tile_bytes = sp.C_tile_bytes = (unsigned long long)P4V_TILE * p.KB8;
  sp.R_cand_stride = sp.R_cand_tile_bytes * sp.tiles_m;
  sp.jobs = at<P4VJob>(ws, p.o_jobs8);
  sp.is_int8 = 1;
}

int run_sweep(const LinPlan& p, const Step& s, const SweepParams& sp, cudaStream_t st) {
  return p4v_run_sweep(sp, p.jobs.data() + s.job_off, p.d.kernel, st);
}

StepTablesArgs tables_args(const LinPlan& p, void* ws, const Step& s, int kind, int target) {
  StepTablesArgs t{};
  t.kind = kind < 0 ? 0 : kind; t.target = target;
  t.dW = at<float>(ws, p.o_dW); t.dW0 = at<float>(ws, p.o_dW0); t.n_V = p.d.n_V; t.n_H = p.d.n_H; t.crb_rows = p.crb_rows;
  t.dX = at<float>(ws, p.o_dX); t.dX0 = at<float>(ws, p.o_dX0); t.n_a = p.d.n_a; t.d_neg = p.d_neg;
  t.factors = at<float>(ws, p.o_factors); t.n_cand = kind < 0 ? 0 : p.d.eq_n;
  t.fixed_meta = at<GroupMeta>(ws, p.o_metas) + s.meta_fix; t.n_fixed_groups = s.nfg;
  t.cand_meta = at<GroupMeta>(ws, p.o_metas) + s.meta_cand; t.n_cand_groups = s.ncg;
  t.nsg = p.nsg;
  t.fix_scale = at<float>(ws, p.o_fix); t.candA = at<float>(ws, p.o_candA); t.candB = at<float>(ws, p.o_candB);
  return t;
}

int tables_for(const LinPlan& p, void* ws, const Step& s, int kind, int target, cudaStream_t st) {
  return p4v_step_tables(tables_args(p, ws, s, kind, target), st);
}

struct StepRef { bool is_w; int idx; };

// One search step: [scale tables] -> sweep -> reduce -> select (+ tables of the next step) -> commit.
// Chunked: per chunk of rows, the chunk's X images (current; X step: candidates) -> sweep -> reduce into the fp64 table;
// select after the last chunk; only the weight image is committed (the X images are rebuilt from the step sizes).
// An int8 activation step (p.x8) first quantises the current weights to int8 and, unchunked, rebuilds the bf16 current
// activation image from the chosen step size instead of committing a candidate slab.
int search_step(const LinPlan& p, void* ws, StepRef cur, const StepRef* next, bool tables_ready, const float* x, const float* W,
                const float* bias, const float* y, const float* g, float* score_log, cudaStream_t st) {
  const bool is_w = cur.is_w; const int idx = cur.idx;
  const bool x8 = !is_w && p.x8;
  const Step& s = is_w ? p.wsteps[idx] : p.xsteps[idx];
  int rc;
  if (!tables_ready && (rc = tables_for(p, ws, s, is_w ? 0 : 1, idx, st))) return rc;
  if (x8 && (rc = quant_W(p, ws, W, at<float>(ws, p.o_dW), false, st, true))) return rc;
  SweepParams sp;
  for (int r0 = 0; r0 < p.M; r0 += p.chunk_rows) {
    const Rows r{r0, std::min(p.chunk_rows, p.M - r0)};
    if (p.chunked) {
      if ((rc = quant_X(p, ws, x, at<float>(ws, p.o_dX), false, r, st))) return rc;
      if (!is_w && (rc = quant_X(p, ws, x, at<float>(ws, p.o_dX0), true, r, st))) return rc;
    }
    if (x8) fill_sweep_x8(p, ws, sp, r);
    else fill_sweep(p, ws, s, sp, r);
    sp.Y = y + (size_t)r0 * p.O; sp.Gr = g + (size_t)r0 * p.O; sp.bias = p.d.has_bias ? bias : nullptr;
    sp.order = is_w ? 0 : 1;
    if ((rc = x8 ? p4v_run_sweep(sp, p.jobs8.data(), p.d.kernel, st) : run_sweep(p, s, sp, st))) return rc;
    ReduceArgs ra{};
    ra.partial = sp.partial; ra.n_cand = p.d.eq_n; ra.P = 1; ra.tiles_m = sp.tiles_m; ra.tiles_n = p.tiles_o; ra.order = sp.order;
    ra.mode = P4V_SG_COLUMN; ra.n_keys = p.nsg; ra.sums = at<double>(ws, p.o_scores); ra.accumulate = r0 > 0;
    if ((rc = p4v_reduce_scores(ra, st))) return rc;
  }
  const int n_groups = is_w ? p.d.n_V : 1;
  SelectArgs f{};
  f.sums = at<double>(ws, p.o_scores); f.n_cand = p.d.eq_n; f.n_keys = p.nsg; f.n_groups = n_groups;
  f.keys_per_group = (is_w && p.d.n_V > 1) ? p.crb_rows / P4V_CG : p.nsg;
  f.inv_count = 1.0 / ((double)p.d.tokens * (double)(is_w ? p.crb_rows : p.O));
  f.gscale = at<float>(ws, p.o_gscale); f.factors = at<float>(ws, p.o_factors);
  if (is_w) { f.d0 = at<float>(ws, p.o_dW0); f.d = at<float>(ws, p.o_dW); f.d_stride = p.d.n_H; f.d_col = idx; }
  else      { f.d0 = at<float>(ws, p.o_dX0); f.d = at<float>(ws, p.o_dX); f.d_stride = 0; f.d_col = idx; }
  f.best = at<int>(ws, p.o_best); f.score_log = score_log;
  f.has_next = next != nullptr;
  if (next) f.next = tables_args(p, ws, next->is_w ? p.wsteps[next->idx] : p.xsteps[next->idx], next->is_w ? 0 : 1, next->idx);
  if ((rc = p4v_select_step(f, st))) return rc;
  if (p.chunked && !is_w) return 0;
  if (x8) return quant_X(p, ws, x, at<float>(ws, p.o_dX), false, all_rows(p), st);
  CommitArgs c{};
  c.best = f.best; c.n_groups = n_groups;
  c.cand = at<uint8_t>(ws, is_w ? p.o_Wcand : p.o_Xcand);
  c.cand_tile_bytes = (unsigned long long)P4V_TILE * (is_w ? p.KB_W : p.KB_Xc);
  c.cand_plane_stride = c.cand_tile_bytes * (is_w ? p.tiles_o : p.tiles_m);
  c.cur = at<uint8_t>(ws, is_w ? p.o_Wcur : p.o_Xcur);
  c.cur_tile_bytes = (unsigned long long)P4V_TILE * (is_w ? p.KB_W : p.KB_X);
  c.P = 1; c.tiles = is_w ? p.tiles_o : p.tiles_m;
  c.rows_per_group = is_w ? p.crb_rows : 0; c.problem_groups = 0;
  c.segs = at<CommitSeg>(ws, p.o_commits) + s.commit_off; c.nseg = s.ncommit; c.commit_chunks = s.commit_chunks;
  return p4v_commit_step(c, st);
}

// (gs*g)^2 image of the rows r: rows = output channels, K = the chunk's tokens, two exact bf16 terms (transposed read)
int gram_g2_image(const LinPlan& p, void* ws, const float* g, Rows r, cudaStream_t st) {
  const unsigned term = gram_term(r.n);
  QuantImageArgs q{};
  q.src = g + (size_t)r.r0 * p.O; q.ld = p.O; q.prob_stride = 0; q.src_transposed = 1;
  q.P = 1; q.rows = p.O; q.tiles = p.tiles_o;
  q.dst = at<uint8_t>(ws, p.o_G2T); q.tile_bytes = (unsigned long long)P4V_TILE * 2 * term; q.plane_stride = 0;
  q.n_planes = 1; q.factors = nullptr; q.delta = at<float>(ws, p.o_dW0); q.rows_per_block = p.O + P4V_TILE; q.d_stride = 0; q.d_mod = 1;
  q.segs = at<P4VSeg>(ws, p.o_segsG) + (r.n == p.chunk_rows ? 0 : 2); q.nseg = 2; q.is_int8 = 0; q.presc = at<float>(ws, p.o_gscale);
  return p4v_quant_image(q, st);
}

// Whole W search of one round in normal-equation form (gram.cu): residual once, then per column block
// (pair image + Gram GEMM for every column block, once) and per column block update pass -> candidate evaluation -> select -> commit.
// Chunked: the residual sweep, the (gs*g)^2 and pair images, the Gram GEMM (seeded from the stored H) and the update pass
// (U, sum (g e)^2 added over the chunks) run per chunk of rows; evaluation, select and commit once per column block.
int gram_wsearch(const LinPlan& p, void* ws, const float* x, const float* W, const float* bias, const float* y, const float* g,
                 int h_begin, int h_end, float* score_log, cudaStream_t st) {
  int rc;
  const float w_lo = (float)-p.w_qmax, w_hi = (float)(p.w_qmax - 1);
  std::vector<Rows> chunks;
  for (int r0 = 0; r0 < p.M; r0 += p.chunk_rows) chunks.push_back(Rows{r0, std::min(p.chunk_rows, p.M - r0)});
  // e = y - yhat(current step sizes), exact integer products (every segment as a fixed group)
  if ((rc = tables_for(p, ws, p.fwd, -1, 0, st))) return rc;
  for (const Rows& r : chunks) {
    if (p.chunked && (rc = quant_X(p, ws, x, at<float>(ws, p.o_dX), false, r, st))) return rc;
    SweepParams sp; fill_sweep(p, ws, p.fwd, sp, r);
    sp.Y = y + (size_t)r.r0 * p.O; sp.Gr = g + (size_t)r.r0 * p.O; sp.bias = p.d.has_bias ? bias : nullptr;
    sp.out = at<float>(ws, p.o_E) + (size_t)r.r0 * p.O; sp.out_residual = 1; sp.n_cand = 1; sp.order = 0;
    sp.R_cand = nullptr; sp.C_cand = nullptr;
    if ((rc = run_sweep(p, p.fwd, sp, st))) return rc;
  }
  if ((rc = p4v_xq_transpose(x, p.M, p.K, p.g_Mp, at<float>(ws, p.o_dX), p.crb_acts, (float)-p.a_qmax, (float)(p.a_qmax - 1),
                             at<int8_t>(ws, p.o_XqT), st))) return rc;
  // H for every column block of the range: one pair image + one tensor-core GEMM per chunk of rows (the activations do
  // not change during the weight steps of a round)
  {
    const int nblk = h_end - h_begin;
    const int tiles_p = p4v_cdiv(p.g_npairs * nblk, GRAM_PT);
    for (const Rows& r : chunks) {
      const unsigned term = gram_term(r.n);
      const unsigned long long z_tile = (unsigned long long)GRAM_PT * 2 * term;
      if (p.chunked && (rc = gram_g2_image(p, ws, g, r, st))) return rc;
      if ((rc = p4v_pair_image(at<int8_t>(ws, p.o_XqT) + r.r0, p.g_Mp, r.n, h_begin * p.g_ks, p.g_ks, p.g_npairs, nblk, tiles_p,
                               z_tile, term, at<uint8_t>(ws, p.o_Z), st))) return rc;
      GramGemmArgs gg{};
      gg.R = at<uint8_t>(ws, p.o_G2T); gg.R_tile_bytes = (unsigned long long)P4V_TILE * 2 * term;
      gg.C = at<uint8_t>(ws, p.o_Z); gg.C_tile_bytes = z_tile; gg.term_bytes = term;
      gg.tiles_o = p.tiles_o; gg.tiles_p = tiles_p; gg.O = p.O; gg.H = at<float>(ws, p.o_H); gg.ldH = p.g_ldH;
      gg.accumulate = r.r0 > 0;
      if ((rc = p4v_gram_gemm(gg, st))) return rc;
    }
  }
  for (int h = h_begin; h < h_end; ++h) {
    for (const Rows& r : chunks) {
      GramUpdateArgs u{};
      u.E = at<float>(ws, p.o_E) + (size_t)r.r0 * p.O; u.G = g + (size_t)r.r0 * p.O; u.gscale = at<float>(ws, p.o_gscale);
      u.W = W; u.M = r.n; u.O = p.O; u.K = p.K; u.XqT = at<int8_t>(ws, p.o_XqT) + r.r0; u.Mp = p.g_Mp;
      u.dX = at<float>(ws, p.o_dX); u.crb_acts = p.crb_acts;
      u.dW = at<float>(ws, p.o_dW); u.dW_prev = at<float>(ws, p.o_dprev); u.n_V = p.d.n_V; u.n_H = p.d.n_H; u.crb_rows = p.crb_rows;
      u.h_prev = h > h_begin ? h - 1 : -1; u.k_prev = (h - 1) * p.g_ks; u.k_next = h * p.g_ks; u.ks = p.g_ks;
      u.w_lo = w_lo; u.w_hi = w_hi; u.Upart = at<float>(ws, p.o_Upart); u.E2part = at<float>(ws, p.o_E2part);
      u.D = at<float>(ws, p.o_D); u.n_split = p.g_nmblk;
      if ((rc = p4v_gram_update(u, st))) return rc;
      if ((rc = p4v_gram_reduce(u.Upart, u.E2part, p.g_nmblk, p.O, p.g_ks, at<float>(ws, p.o_U), at<float>(ws, p.o_E2),
                                r.r0 > 0, st))) return rc;
    }
    GramEvalArgs ev{};
    ev.H = at<float>(ws, p.o_H) + (size_t)(h - h_begin) * p.g_npairs; ev.ldH = p.g_ldH; ev.npairs = p.g_npairs;
    ev.U = at<float>(ws, p.o_U); ev.E2 = at<float>(ws, p.o_E2);
    ev.W = W; ev.O = p.O; ev.K = p.K; ev.k_first = h * p.g_ks; ev.ks = p.g_ks;
    ev.dW = at<float>(ws, p.o_dW); ev.dW0 = at<float>(ws, p.o_dW0); ev.n_H = p.d.n_H; ev.h = h;
    ev.dX = at<float>(ws, p.o_dX); ev.crb_acts = p.crb_acts;
    ev.factors = at<float>(ws, p.o_factors); ev.n_cand = p.d.eq_n;
    ev.n_groups = p.d.n_V; ev.rows_per_group = p.crb_rows; ev.osplit = p.g_osplit; ev.rows_per_block = p.g_opb;
    ev.w_lo = w_lo; ev.w_hi = w_hi;
    ev.sums = at<double>(ws, p.o_scores) + (size_t)p.d.eq_n * p.d.n_V; ev.n_keys = p.d.n_V * p.g_osplit;
    ev.sums2 = at<double>(ws, p.o_scores);
    if ((rc = p4v_gram_eval(ev, st))) return rc;
    SelectArgs f{};
    f.sums = ev.sums2; f.n_cand = p.d.eq_n; f.n_keys = p.d.n_V; f.n_groups = p.d.n_V; f.keys_per_group = 1;
    f.inv_count = 1.0 / ((double)p.d.tokens * (double)p.crb_rows);
    f.gscale = at<float>(ws, p.o_gscale); f.factors = at<float>(ws, p.o_factors);
    f.d0 = at<float>(ws, p.o_dW0); f.d = at<float>(ws, p.o_dW); f.d_stride = p.d.n_H; f.d_col = h;
    f.best = at<int>(ws, p.o_best); f.score_log = score_log; f.d_prev = at<float>(ws, p.o_dprev); f.has_next = 0;
    if ((rc = p4v_select_step(f, st))) return rc;
    const Step& s = p.wsteps[h];
    CommitArgs c{};
    c.best = f.best; c.n_groups = p.d.n_V;
    c.cand = at<uint8_t>(ws, p.o_Wcand); c.cand_tile_bytes = (unsigned long long)P4V_TILE * p.KB_W;
    c.cand_plane_stride = c.cand_tile_bytes * p.tiles_o;
    c.cur = at<uint8_t>(ws, p.o_Wcur); c.cur_tile_bytes = c.cand_tile_bytes;
    c.P = 1; c.tiles = p.tiles_o; c.rows_per_group = p.crb_rows; c.problem_groups = 0;
    c.segs = at<CommitSeg>(ws, p.o_commits) + s.commit_off; c.nseg = s.ncommit; c.commit_chunks = s.commit_chunks;
    if ((rc = p4v_commit_step(c, st))) return rc;
    if (score_log) score_log += (size_t)p.d.eq_n * p.d.n_V;
  }
  return 0;
}

int begin_impl(const LinPlan& p, const float* x, const float* W, const float* g, void* ws, cudaStream_t st) {
  int rc;
  if ((rc = upload_tables(p, ws, st))) return rc;
  int* keys = at<int>(ws, p.o_keys);
  const int nW = p.d.n_V * p.d.n_H;
  if ((rc = p4v_keys_reset(keys, nW + p.d.n_a + 1, st))) return rc;
  if ((rc = p4v_block_max(W, p.K, p.O, p.crb_rows, p.d.n_V, p.crb_cols, p.d.n_H, 1, keys, st))) return rc;
  if ((rc = p4v_block_max(x, p.K, p.M, p.M, 1, p.crb_acts, p.d.n_a, p.twin ? 0 : 1, keys + nW, st))) return rc;
  if ((rc = p4v_block_max(g, p.O, p.M, p.M, 1, p.O, 1, 1, keys + nW + p.d.n_a, st))) return rc;
  if (p.d.init_layerwise) {       // linear.py:382-383, :393-394: one step size for the whole weight / activation tensor
    if ((rc = p4v_keys_broadcast_max(keys, nW, st))) return rc;
    if ((rc = p4v_keys_broadcast_max(keys + nW, p.d.n_a, st))) return rc;
  }
  if ((rc = p4v_keys_to_delta(keys, nW, (float)p.w_qmax - 0.5f, at<float>(ws, p.o_dW0), at<float>(ws, p.o_dW), st))) return rc;
  if ((rc = p4v_keys_to_delta(keys + nW, p.d.n_a, (float)p.a_qmax - 0.5f, at<float>(ws, p.o_dX0), at<float>(ws, p.o_dX), st))) return rc;
  if ((rc = p4v_make_gscale(keys + nW + p.d.n_a, at<float>(ws, p.o_gscale), st))) return rc;
  // (gs*g)^2 of all rows, built once; a chunked search builds it per chunk
  if (p.gram && !p.chunked && (rc = gram_g2_image(p, ws, g, all_rows(p), st))) return rc;
  if ((rc = quant_W(p, ws, W, at<float>(ws, p.o_dW0), false, st))) return rc;
  if ((rc = quant_W(p, ws, W, at<float>(ws, p.o_dW0), true, st))) return rc;
  if (p.chunked) return 0;         // every step builds its chunks' activation images
  if ((rc = quant_X(p, ws, x, at<float>(ws, p.o_dX0), false, all_rows(p), st))) return rc;
  if ((rc = quant_X(p, ws, x, at<float>(ws, p.o_dX0), true, all_rows(p), st))) return rc;
  return 0;
}

}  // namespace

extern "C" int p4v_linear_workspace_bytes(const p4v_linear_desc* d, size_t* bytes) {
  LinPlan p; int rc = build_plan(d, p, true);
  if (rc) return rc;
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = p.total;
  return 0;
}

extern "C" int p4v_linear_score_log_floats(const p4v_linear_desc* d, size_t* n) {
  P4V_REQUIRE(d && n, "null argument");
  *n = (size_t)d->search_round * ((size_t)d->n_H * d->eq_n * d->n_V + (size_t)d->n_a * d->eq_n);
  return 0;
}

extern "C" int p4v_linear_begin(const p4v_linear_desc* d, const float* x, const float* weight, const float* bias,
                                const float* raw_out, const float* raw_grad, void* workspace, size_t workspace_bytes, void* stream) {
  (void)bias; (void)raw_out;
  LinPlan p; int rc = build_plan(d, p, true);
  if (rc) return rc;
  P4V_REQUIRE(x && weight && raw_grad && workspace, "linear_begin: null pointer");
  P4V_REQUIRE(!p.chunked, "linear_begin: the step-wise surface searches whole layers (rows_per_chunk must be 0)");
  P4V_REQUIRE(workspace_bytes >= p.total, "linear_begin: workspace too small (%zu < %zu)", workspace_bytes, p.total);
  return begin_impl(p, x, weight, raw_grad, workspace, (cudaStream_t)stream);
}

extern "C" int p4v_linear_search_w(const p4v_linear_desc* d, const float* bias, const float* raw_out, const float* raw_grad,
                                   void* workspace, int32_t h_begin, int32_t h_end, float* score_log, void* stream) {
  LinPlan p; int rc = build_plan(d, p, true);
  if (rc) return rc;
  P4V_REQUIRE(raw_out && raw_grad && workspace, "linear_search_w: null pointer");
  P4V_REQUIRE(!p.chunked, "linear_search_w: the step-wise surface searches whole layers (rows_per_chunk must be 0)");
  P4V_REQUIRE(0 <= h_begin && h_begin <= h_end && h_end <= d->n_H, "linear_search_w: bad block range");
  for (int h = h_begin; h < h_end; ++h) {
    StepRef nx{true, h + 1};
    if ((rc = search_step(p, workspace, StepRef{true, h}, h + 1 < h_end ? &nx : nullptr, h > h_begin, nullptr, nullptr, bias, raw_out, raw_grad,
                          score_log, (cudaStream_t)stream))) return rc;
    if (score_log) score_log += (size_t)d->eq_n * d->n_V;
  }
  return 0;
}

extern "C" int p4v_linear_search_a(const p4v_linear_desc* d, const float* bias, const float* raw_out, const float* raw_grad,
                                   void* workspace, int32_t a_begin, int32_t a_end, float* score_log, void* stream) {
  LinPlan p; int rc = build_plan(d, p, true);
  if (rc) return rc;
  P4V_REQUIRE(raw_out && raw_grad && workspace, "linear_search_a: null pointer");
  P4V_REQUIRE(!p.chunked, "linear_search_a: the step-wise surface searches whole layers (rows_per_chunk must be 0)");
  P4V_REQUIRE(0 <= a_begin && a_begin <= a_end && a_end <= d->n_a, "linear_search_a: bad chunk range");
  for (int a = a_begin; a < a_end; ++a) {
    StepRef nx{false, a + 1};
    if ((rc = search_step(p, workspace, StepRef{false, a}, a + 1 < a_end ? &nx : nullptr, a > a_begin, nullptr, nullptr, bias, raw_out, raw_grad,
                          score_log, (cudaStream_t)stream))) return rc;
    if (score_log) score_log += d->eq_n;
  }
  return 0;
}

extern "C" int p4v_linear_intervals(const p4v_linear_desc* d, void* workspace, float* w_interval, float* a_interval, void* stream) {
  LinPlan p; int rc = build_plan(d, p, true);
  if (rc) return rc;
  P4V_REQUIRE(workspace && w_interval && a_interval, "linear_intervals: null pointer");
  P4V_CUDA_OK(cudaMemcpyAsync(w_interval, at<float>(workspace, p.o_dW), (size_t)d->n_V * d->n_H * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  P4V_CUDA_OK(cudaMemcpyAsync(a_interval, at<float>(workspace, p.o_dX), (size_t)d->n_a * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

extern "C" int p4v_linear_calibrate(const p4v_linear_desc* d, const float* x, const float* weight, const float* bias,
                                    const float* raw_out, const float* raw_grad, void* workspace, size_t workspace_bytes,
                                    float* w_interval, float* a_interval, float* score_log, void* stream) {
  LinPlan p; int rc = build_plan(d, p, true, true);
  if (rc) return rc;
  P4V_REQUIRE(x && weight && raw_out && raw_grad && workspace && w_interval && a_interval, "linear_calibrate: null pointer");
  P4V_REQUIRE(!d->has_bias || bias, "linear_calibrate: has_bias set but bias is null");
  P4V_REQUIRE(workspace_bytes >= p.total, "linear_calibrate: workspace too small (%zu < %zu)", workspace_bytes, p.total);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = begin_impl(p, x, weight, raw_grad, workspace, st))) return rc;
  if (p.gram) {
    for (int e = 0; e < d->search_round; ++e) {
      if ((rc = gram_wsearch(p, workspace, x, weight, bias, raw_out, raw_grad, 0, d->n_H, score_log, st))) return rc;
      if (score_log) score_log += (size_t)d->n_H * d->eq_n * d->n_V;
      for (int a = 0; a < d->n_a; ++a) {
        StepRef nx{false, a + 1};
        if ((rc = search_step(p, workspace, StepRef{false, a}, a + 1 < d->n_a ? &nx : nullptr, a > 0, x, weight, bias, raw_out, raw_grad,
                              score_log, st))) return rc;
        if (score_log) score_log += d->eq_n;
      }
    }
  } else {
    std::vector<StepRef> seq;
    for (int e = 0; e < d->search_round; ++e) {
      for (int h = 0; h < d->n_H; ++h) seq.push_back(StepRef{true, h});
      for (int a = 0; a < d->n_a; ++a) seq.push_back(StepRef{false, a});
    }
    for (size_t i = 0; i < seq.size(); ++i) {
      if ((rc = search_step(p, workspace, seq[i], i + 1 < seq.size() ? &seq[i + 1] : nullptr, i > 0, x, weight, bias, raw_out, raw_grad,
                            score_log, st))) return rc;
      if (score_log) score_log += seq[i].is_w ? (size_t)d->eq_n * d->n_V : (size_t)d->eq_n;
    }
  }
  P4V_CUDA_OK(cudaMemcpyAsync(w_interval, at<float>(workspace, p.o_dW), (size_t)d->n_V * d->n_H * 4, cudaMemcpyDeviceToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(a_interval, at<float>(workspace, p.o_dX), (size_t)d->n_a * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" int p4v_linear_quant_forward_workspace_bytes(const p4v_linear_desc* d, size_t* bytes) {
  LinPlan p; int rc = build_plan(d, p, false);
  if (rc) return rc;
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = p.total;
  return 0;
}

extern "C" int p4v_linear_quant_forward(const p4v_linear_desc* d, const float* x, const float* weight, const float* bias,
                                        const float* w_interval, const float* a_interval, void* workspace,
                                        size_t workspace_bytes, float* out, void* stream) {
  LinPlan p; int rc = build_plan(d, p, false);
  if (rc) return rc;
  P4V_REQUIRE(x && weight && w_interval && a_interval && workspace && out, "linear_quant_forward: null pointer");
  P4V_REQUIRE(workspace_bytes >= p.total, "linear_quant_forward: workspace too small (%zu < %zu)", workspace_bytes, p.total);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = upload_tables(p, workspace, st))) return rc;
  P4V_CUDA_OK(cudaMemcpyAsync(at<float>(workspace, p.o_dW), w_interval, (size_t)d->n_V * d->n_H * 4, cudaMemcpyDeviceToDevice, st));
  P4V_CUDA_OK(cudaMemcpyAsync(at<float>(workspace, p.o_dX), a_interval, (size_t)d->n_a * 4, cudaMemcpyDeviceToDevice, st));
  if ((rc = quant_W(p, workspace, weight, at<float>(workspace, p.o_dW), false, st))) return rc;
  if ((rc = quant_X(p, workspace, x, at<float>(workspace, p.o_dX), false, all_rows(p), st))) return rc;
  if ((rc = tables_for(p, workspace, p.fwd, -1, 0, st))) return rc;
  SweepParams sp; fill_sweep(p, workspace, p.fwd, sp);
  sp.bias = d->has_bias ? bias : nullptr;
  sp.out = out; sp.n_cand = 1; sp.order = 0;
  sp.R_cand = nullptr; sp.C_cand = nullptr;
  return run_sweep(p, p.fwd, sp, st);
}
