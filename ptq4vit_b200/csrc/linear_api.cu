// C-ABI for the Linear scale-factor search: host-side planning (segments, jobs,
// workspace carving) + the per-step launch sequence.  See include/ptq4vit_b200.h.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "../../include/ptq4vit_b200.h"
#include "plan.cuh"
#include "gram.cuh"

namespace {

// bytes of K of one bf16 term of the Gram operands for n tokens
inline unsigned gram_term(int n) { return (unsigned)align_up((size_t)n * 2, 32); }

struct BSeg { int k0, klen, h, a, kb; int woff, xoff_p, xoff_n, xcoff; };   // offsets: bytes in the padded row
struct Step {
  int job_off, nfj, ncj, nfg, ncg, meta_fix, meta_cand;
  int commit_off, ncommit, commit_chunks;   // no commit segments: the candidates are laid out unlike the current image
  const Table<P4VJob>* jobs;
  const Image *Rcur, *Rcand, *Ccur, *Ccand;  // the images the sweep reads: rows = activations, columns = weights
  const Table<P4VSeg>* Rcand_segs;          // segments of Rcand (an activation step builds it per chunk of rows)
  const Table<P4VSeg>* Ccur_segs;           // set when Ccur is the step's own image of the current weights
};

struct LinPlan {
  LinPlan() = default;
  LinPlan(const LinPlan&) = delete;         // the steps point at the plan's images and tables
  p4v_linear_desc d;
  bool i8, twin;
  int ew, M, K, O, tiles_m, tiles_o, nsg, crb_rows, crb_cols, crb_acts, w_qmax, a_qmax;
  bool chunked; int chunk_rows, tiles_mc;   // rows of one chunk (M unchunked) and their 128-row tiles: the X images hold one chunk
  float d_neg;
  std::vector<BSeg> segs;
  Table<float> factors;
  Table<P4VJob> jobs; Table<GroupMeta> metas; Table<CommitSeg> commits;
  Table<P4VSeg> segsW, segsX, segsXc;
  Image Wcur, Xcur, Wcand, Xcand;
  std::vector<Step> wsteps, xsteps;
  Step fwd;   // quant_forward: every segment is a fixed group
  // normal-equation W search (gram.cu)
  bool gram; int g_ks, g_Mp, g_npairs, g_tiles_p, g_ldH, g_nmblk; unsigned g_term_bytes;
  size_t o_E, o_XqT, o_G2T, o_Z, o_H, o_Upart, o_E2part, o_U, o_E2, o_dprev, o_D, o_segsG;
  int g_osplit, g_opb;
  int max_groups;
  // workspace offsets
  size_t o_keys, o_dW0, o_dW, o_dX0, o_dX, o_gscale, o_scores, o_best, o_fix, o_candA, o_candB, o_partial, total;
  // int8 activation step of a bf16 layer (build_plan; it then is xsteps[0]): its jobs, segment tables and images, carved
  // inside the bf16 candidate activation region
  bool x8;
  Table<P4VJob> jobs8; Table<P4VSeg> segsW8, segsXc8;
  Image Xcand8, Wcur8;
};

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
  const int KB_W = off, KB_Xc = off, KB_X = p.twin ? 2 * off : off;
  for (auto& s : p.segs) s.xoff_n = p.twin ? off + s.xoff_p : -1;
  P4V_REQUIRE((size_t)KB_X * P4V_TILE < (1ull << 32), "linear: in_features too large");
  p.Wcur = Image{0, KB_W, p.tiles_o, 1, 1, p.i8}; p.Wcand = Image{0, KB_W, p.tiles_o, 1, d->eq_n, p.i8};
  p.Xcur = Image{0, KB_X, p.tiles_mc, 1, 1, p.i8}; p.Xcand = Image{0, KB_Xc, p.tiles_mc, 1, d->eq_n, p.i8};

  // quantisation segment tables
  for (auto& s : p.segs) {
    P4VSeg w{s.k0, s.klen, s.woff * P4V_TILE, s.h, 0.f, (float)-p.w_qmax, (float)(p.w_qmax - 1), 0, 0.f, 0, 0};
    p.segsW.host.push_back(w);
    P4VSeg x{s.k0, s.klen, s.xoff_p * P4V_TILE, s.a, 0.f, p.twin ? 0.f : (float)-p.a_qmax, (float)(p.a_qmax - 1), 0, 0.f, 0, 0};
    p.segsX.host.push_back(x);
    P4VSeg xc = x; xc.dst_off = s.xcoff * P4V_TILE;
    p.segsXc.host.push_back(xc);
  }
  if (p.twin)
    for (auto& s : p.segs) {
      P4VSeg n{s.k0, s.klen, s.xoff_n * P4V_TILE, s.a, p.d_neg, (float)-p.a_qmax, 0.f, 0, 0.f, 0, 0};
      p.segsX.host.push_back(n);
    }

  p.factors.host = cand_factors(d->eq_n, d->eq_alpha, d->eq_beta);

  // steps
  std::vector<P4VJob>& jobs = p.jobs.host;
  std::vector<GroupMeta>& metas = p.metas.host;
  p.max_groups = 1;
  auto begin_step = [&](Step& st) {
    st = Step{};
    st.job_off = (int)jobs.size(); st.commit_off = (int)p.commits.host.size();
    st.jobs = &p.jobs; st.Rcur = &p.Xcur; st.Rcand = &p.Xcand; st.Ccur = &p.Wcur; st.Ccand = &p.Wcand;
    st.Rcand_segs = &p.segsXc;
  };
  auto fixed_group = [&](Step& st, const BSeg& s, bool neg) {
    add_group(jobs, neg ? s.xoff_n : s.xoff_p, s.woff, s.kb, 0, st.nfg, true, true, st.nfj);
    metas.push_back(GroupMeta{(short)s.h, (short)s.a, (short)(neg ? 1 : 0), 0});
    ++st.nfg;
  };
  if (with_search) {
    for (int h = 0; h < d->n_H; ++h) {
      Step st; begin_step(st);
      st.meta_fix = (int)metas.size();
      for (auto& s : p.segs) if (s.h != h) { fixed_group(st, s, false); if (p.twin) fixed_group(st, s, true); }
      st.meta_cand = (int)metas.size();
      for (auto& s : p.segs) if (s.h == h) {
        add_group(jobs, s.xoff_p, s.woff, s.kb, P4V_JOB_CCAND, st.ncg, true, true, st.ncj);
        metas.push_back(GroupMeta{(short)s.h, (short)s.a, 0, 0}); ++st.ncg;
        if (p.twin) {
          add_group(jobs, s.xoff_n, s.woff, s.kb, P4V_JOB_CCAND, st.ncg, true, true, st.ncj);
          metas.push_back(GroupMeta{(short)s.h, (short)s.a, 1, 0}); ++st.ncg;
        }
        p.commits.host.push_back(CommitSeg{s.woff * P4V_TILE, s.woff * P4V_TILE, s.kb});
        st.commit_chunks += s.kb / 16; ++st.ncommit;
      }
      mark_resident(jobs, st.job_off + st.nfj, st.ncj);
      batch_jobs(jobs, st.job_off, st.nfj);
      p.wsteps.push_back(st);
    }
    for (int a = 0; a < d->n_a; ++a) {
      Step st; begin_step(st);
      st.meta_fix = (int)metas.size();
      for (auto& s : p.segs) { if (s.a != a) fixed_group(st, s, false); if (p.twin) fixed_group(st, s, true); }
      st.meta_cand = (int)metas.size();
      for (auto& s : p.segs) if (s.a == a) {
        add_group(jobs, s.xcoff, s.woff, s.kb, P4V_JOB_RCAND, st.ncg, true, true, st.ncj);
        metas.push_back(GroupMeta{(short)s.h, (short)s.a, 0, 0}); ++st.ncg;
        p.commits.host.push_back(CommitSeg{s.xcoff * P4V_TILE, s.xoff_p * P4V_TILE, s.kb});
        st.commit_chunks += s.kb / 16; ++st.ncommit;
      }
      {   // candidates change the row operand only: keep the tile's weight image resident when it fits
        int ncj = st.ncj; batch_jobs(jobs, st.job_off + st.nfj, ncj); st.ncj = ncj;
        batch_jobs(jobs, st.job_off, st.nfj);
        if ((size_t)KB_W * P4V_TILE <= 100 * 1024)
          for (int j = 0; j < st.nfj + st.ncj; ++j) jobs[st.job_off + j].flags |= P4V_JOB_CRES;
      }
      p.xsteps.push_back(st);
    }
  }
  {
    Step st; begin_step(st);
    st.meta_fix = (int)metas.size();
    for (auto& s : p.segs) { fixed_group(st, s, false); if (p.twin) fixed_group(st, s, true); }
    st.meta_cand = (int)metas.size();
    batch_jobs(jobs, st.job_off, st.nfj);
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
  Carver c{0};
  const int n_c = d->eq_n;
  p.factors.off = c.take(p.factors.bytes());
  p.o_keys = c.take((d->n_V * d->n_H + d->n_a + 1) * 4);
  p.o_dW0 = c.take(d->n_V * d->n_H * 4); p.o_dW = c.take(d->n_V * d->n_H * 4);
  p.o_dX0 = c.take(d->n_a * 4); p.o_dX = c.take(d->n_a * 4);
  p.o_gscale = c.take(4);
  p.o_scores = c.take((size_t)n_c * (p.nsg + d->n_V * (size_t)(1 + p4v_cdiv(p.crb_rows, 2))) * 8);
  p.o_best = c.take(std::max(d->n_V, 1) * 4);
  p.o_fix = c.take((size_t)p.max_groups * p.nsg * 4);
  p.o_candA = c.take((size_t)n_c * p.nsg * 4);
  p.o_candB = c.take((size_t)p.max_groups * p.nsg * 4);
  p.jobs.off = c.take(p.jobs.bytes());
  p.metas.off = c.take(p.metas.bytes());
  p.segsW.off = c.take(p.segsW.bytes());
  p.segsX.off = c.take(p.segsX.bytes());
  p.segsXc.off = c.take(p.segsXc.bytes());
  p.commits.off = c.take(std::max(p.commits.bytes(), sizeof(CommitSeg)));
  p.o_partial = c.take(with_search ? (size_t)p.tiles_mc * p.tiles_o * n_c * 32 * 4 : 4);
  p.Wcur.off = c.take(p.Wcur.bytes());
  p.Xcur.off = c.take(p.Xcur.bytes());
  p.Wcand.off = c.take(with_search ? p.Wcand.bytes() : 4);
  p.Xcand.off = c.take(with_search ? p.Xcand.bytes() : 4);
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
      p.o_E = c.take((size_t)p.M * p.O * 4);
      p.o_XqT = c.take((size_t)p.K * p.g_Mp);
      p.o_G2T = c.take((size_t)p.tiles_o * P4V_TILE * KBg);
      p.o_Z = c.take((size_t)p.g_tiles_p * GRAM_PT * KBg);
      p.o_H = c.take((size_t)p.O * p.g_ldH * 4);
      p.o_Upart = c.take((size_t)p.g_nmblk * p.O * p.g_ks * 4);
      p.o_E2part = c.take((size_t)p.g_nmblk * p.O * 4);
      p.o_U = c.take((size_t)p.O * p.g_ks * 4); p.o_E2 = c.take((size_t)p.O * 4);
      p.g_osplit = std::max(1, p4v_cdiv(p.crb_rows, 2)); p.g_opb = p4v_cdiv(p.crb_rows, p.g_osplit);
      p.o_dprev = c.take((size_t)d->n_V * 4);
      p.o_D = c.take((size_t)p.O * 64 * 4);
      p.o_segsG = c.take((p.chunked ? 4 : 2) * sizeof(P4VSeg));   // chunked: a full chunk and the last one
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
      p.xsteps[0].nfg == 0) {
    Step st = p.xsteps[0];
    st.job_off = 0; st.nfj = 0; st.ncj = 0; st.ncommit = 0;
    st.jobs = &p.jobs8; st.Rcand = &p.Xcand8; st.Ccur = &p.Wcur8; st.Rcand_segs = &p.segsXc8; st.Ccur_segs = &p.segsW8;
    int off8 = 0;
    for (size_t i = 0; i < p.segs.size(); ++i) {   // one candidate group per segment, in the order of the bf16 step
      const int kb = (int)align_up((size_t)p.segs[i].klen, 32);
      P4VSeg w = p.segsW.host[i], x = p.segsXc.host[i];
      w.dst_off = x.dst_off = off8 * P4V_TILE;
      p.segsW8.host.push_back(w); p.segsXc8.host.push_back(x);
      add_group(p.jobs8.host, off8, off8, kb, P4V_JOB_RCAND, (int)i, true, true, st.ncj);
      off8 += kb;
    }
    batch_jobs(p.jobs8.host, 0, st.ncj);
    for (auto& j : p.jobs8.host) j.flags |= P4V_JOB_CRES;
    p.Xcand8 = Image{0, off8, p.tiles_mc, 1, n_c, true}; p.Wcur8 = Image{0, off8, p.tiles_o, 1, 1, true};
    Carver c8{p.Xcand.off};
    p.Xcand8.off = c8.take(p.Xcand8.bytes());
    p.Wcur8.off = c8.take(p.Wcur8.bytes());
    p.jobs8.off = c8.take(p.jobs8.bytes());
    p.segsW8.off = c8.take(p.segsW8.bytes());
    p.segsXc8.off = c8.take(p.segsXc8.bytes());
    p.x8 = (size_t)off8 * P4V_TILE <= 100 * 1024 && c8.end <= align_up(p.Xcand.off + p.Xcand.bytes(), 256) && st.ncj <= P4V_MAX_JOBS;
    if (p.x8) p.xsteps[0] = st;
  }
  p.total = c.end;
  return 0;
}

int upload_tables(const LinPlan& p, void* ws, cudaStream_t st) {
  int rc;
  if ((rc = p.factors.upload(ws, st)) || (rc = p.jobs.upload(ws, st)) || (rc = p.metas.upload(ws, st)) ||
      (rc = p.segsW.upload(ws, st)) || (rc = p.segsX.upload(ws, st)) || (rc = p.segsXc.upload(ws, st)) ||
      (rc = p.commits.upload(ws, st))) return rc;
  if (p.x8 && ((rc = p.jobs8.upload(ws, st)) || (rc = p.segsW8.upload(ws, st)) || (rc = p.segsXc8.upload(ws, st)))) return rc;
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

// rows [r0, r0 + n) of the layer: one chunk (or all rows)
struct Rows { int r0, n; };
Rows all_rows(const LinPlan& p) { return Rows{0, p.M}; }

// Quantise rows r of the weights (rows = output channels, one step-size row block per crb_rows rows) or of the
// activations (one row block) into image im with the step sizes delta; cand: one plane per candidate factor
int quant(const LinPlan& p, void* ws, const Image& im, const Table<P4VSeg>& segs, bool weights, const float* src, Rows r,
          const float* delta, bool cand, cudaStream_t st) {
  QuantImageArgs q{};
  im.chunk(p4v_cdiv(r.n, P4V_TILE), 1).fill(q, ws);
  q.src = src + (size_t)r.r0 * p.K; q.ld = p.K; q.prob_stride = 0; q.src_transposed = 0; q.rows = r.n;
  q.factors = cand ? p.factors.dev(ws) : nullptr;
  q.delta = delta; q.d_mod = 1;
  q.rows_per_block = weights ? p.crb_rows : p.M + P4V_TILE; q.d_stride = weights ? p.d.n_H : 0;   // activations: any row range
  q.segs = segs.dev(ws); q.nseg = (int)segs.host.size();
  return p4v_quant_image(q, st);
}

void fill_sweep(const LinPlan& p, void* ws, const Step& s, SweepParams& sp, Rows r) {
  const int tiles_m = p4v_cdiv(r.n, P4V_TILE);
  sp = SweepParams{};
  fill_images(sp, ws, s.Rcur->chunk(tiles_m, 1), s.Rcand->chunk(tiles_m, 1), *s.Ccur, *s.Ccand);
  sp.P = 1; sp.M = r.n; sp.N = p.O; sp.tiles_m = tiles_m; sp.tiles_n = p.tiles_o;
  sp.ld = p.O; sp.prob_stride = 0;
  sp.gscale = at<float>(ws, p.o_gscale);
  sp.jobs = s.jobs->dev(ws) + s.job_off;
  sp.n_fixed_jobs = s.nfj; sp.n_cand_jobs = s.ncj; sp.n_fixed_groups = s.nfg; sp.n_cand_groups = s.ncg;
  sp.fix_scale = at<float>(ws, p.o_fix); sp.candA = at<float>(ws, p.o_candA); sp.candB = at<float>(ws, p.o_candB);
  sp.nsg = p.nsg; sp.sg_mode = P4V_SG_COLUMN;
  sp.n_cand = p.d.eq_n;
  sp.partial = at<float>(ws, p.o_partial);
}

int run_sweep(const LinPlan& p, const Step& s, const SweepParams& sp, cudaStream_t st) {
  return p4v_run_sweep(sp, s.jobs->host.data() + s.job_off, p.d.kernel, st);
}

// Copy the chosen candidates' commit slabs of step s into the current image: a weight step one group of crb_rows rows
// per row block, an activation step one group
int commit(const LinPlan& p, void* ws, const Step& s, bool is_w, cudaStream_t st) {
  CommitArgs c{};
  if (is_w) fill_images(c, ws, *s.Ccand, *s.Ccur);
  else fill_images(c, ws, *s.Rcand, *s.Rcur);
  c.best = at<int>(ws, p.o_best); c.n_groups = is_w ? p.d.n_V : 1;
  c.rows_per_group = is_w ? p.crb_rows : 0; c.problem_groups = 0;
  c.segs = p.commits.dev(ws) + s.commit_off; c.nseg = s.ncommit; c.commit_chunks = s.commit_chunks;
  return p4v_commit_step(c, st);
}

StepTablesArgs tables_args(const LinPlan& p, void* ws, const Step& s, int kind, int target) {
  StepTablesArgs t{};
  t.kind = kind < 0 ? 0 : kind; t.target = target;
  t.dW = at<float>(ws, p.o_dW); t.dW0 = at<float>(ws, p.o_dW0); t.n_V = p.d.n_V; t.n_H = p.d.n_H; t.crb_rows = p.crb_rows;
  t.dX = at<float>(ws, p.o_dX); t.dX0 = at<float>(ws, p.o_dX0); t.n_a = p.d.n_a; t.d_neg = p.d_neg;
  t.factors = p.factors.dev(ws); t.n_cand = kind < 0 ? 0 : p.d.eq_n;
  t.fixed_meta = p.metas.dev(ws) + s.meta_fix; t.n_fixed_groups = s.nfg;
  t.cand_meta = p.metas.dev(ws) + s.meta_cand; t.n_cand_groups = s.ncg;
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
// A step with its own image of the current weights (the int8 activation step) builds it first; a step without commit
// segments rebuilds the current activation image from the chosen step size instead of committing a candidate slab.
int search_step(const LinPlan& p, void* ws, StepRef cur, const StepRef* next, bool tables_ready, const float* x, const float* W,
                const float* bias, const float* y, const float* g, float* score_log, cudaStream_t st) {
  const bool is_w = cur.is_w; const int idx = cur.idx;
  const Step& s = is_w ? p.wsteps[idx] : p.xsteps[idx];
  int rc;
  if (!tables_ready && (rc = tables_for(p, ws, s, is_w ? 0 : 1, idx, st))) return rc;
  if (s.Ccur_segs && (rc = quant(p, ws, *s.Ccur, *s.Ccur_segs, true, W, Rows{0, p.O}, at<float>(ws, p.o_dW), false, st))) return rc;
  SweepParams sp;
  for (int r0 = 0; r0 < p.M; r0 += p.chunk_rows) {
    const Rows r{r0, std::min(p.chunk_rows, p.M - r0)};
    if (p.chunked) {
      if ((rc = quant(p, ws, p.Xcur, p.segsX, false, x, r, at<float>(ws, p.o_dX), false, st))) return rc;
      if (!is_w && (rc = quant(p, ws, *s.Rcand, *s.Rcand_segs, false, x, r, at<float>(ws, p.o_dX0), true, st))) return rc;
    }
    fill_sweep(p, ws, s, sp, r);
    sp.Y = y + (size_t)r0 * p.O; sp.Gr = g + (size_t)r0 * p.O; sp.bias = p.d.has_bias ? bias : nullptr;
    sp.order = is_w ? 0 : 1;
    if ((rc = run_sweep(p, s, sp, st))) return rc;
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
  f.gscale = at<float>(ws, p.o_gscale); f.factors = p.factors.dev(ws);
  if (is_w) { f.d0 = at<float>(ws, p.o_dW0); f.d = at<float>(ws, p.o_dW); f.d_stride = p.d.n_H; f.d_col = idx; }
  else      { f.d0 = at<float>(ws, p.o_dX0); f.d = at<float>(ws, p.o_dX); f.d_stride = 0; f.d_col = idx; }
  f.best = at<int>(ws, p.o_best); f.score_log = score_log;
  f.has_next = next != nullptr;
  if (next) f.next = tables_args(p, ws, next->is_w ? p.wsteps[next->idx] : p.xsteps[next->idx], next->is_w ? 0 : 1, next->idx);
  if ((rc = p4v_select_step(f, st))) return rc;
  if (p.chunked && !is_w) return 0;
  if (s.ncommit == 0) return quant(p, ws, p.Xcur, p.segsX, false, x, all_rows(p), at<float>(ws, p.o_dX), false, st);
  return commit(p, ws, s, is_w, st);
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
    if (p.chunked && (rc = quant(p, ws, p.Xcur, p.segsX, false, x, r, at<float>(ws, p.o_dX), false, st))) return rc;
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
    ev.factors = p.factors.dev(ws); ev.n_cand = p.d.eq_n;
    ev.n_groups = p.d.n_V; ev.rows_per_group = p.crb_rows; ev.osplit = p.g_osplit; ev.rows_per_block = p.g_opb;
    ev.w_lo = w_lo; ev.w_hi = w_hi;
    ev.sums = at<double>(ws, p.o_scores) + (size_t)p.d.eq_n * p.d.n_V; ev.n_keys = p.d.n_V * p.g_osplit;
    ev.sums2 = at<double>(ws, p.o_scores);
    if ((rc = p4v_gram_eval(ev, st))) return rc;
    SelectArgs f{};
    f.sums = ev.sums2; f.n_cand = p.d.eq_n; f.n_keys = p.d.n_V; f.n_groups = p.d.n_V; f.keys_per_group = 1;
    f.inv_count = 1.0 / ((double)p.d.tokens * (double)p.crb_rows);
    f.gscale = at<float>(ws, p.o_gscale); f.factors = p.factors.dev(ws);
    f.d0 = at<float>(ws, p.o_dW0); f.d = at<float>(ws, p.o_dW); f.d_stride = p.d.n_H; f.d_col = h;
    f.best = at<int>(ws, p.o_best); f.score_log = score_log; f.d_prev = at<float>(ws, p.o_dprev); f.has_next = 0;
    if ((rc = p4v_select_step(f, st))) return rc;
    if ((rc = commit(p, ws, p.wsteps[h], true, st))) return rc;
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
  if ((rc = quant(p, ws, p.Wcur, p.segsW, true, W, Rows{0, p.O}, at<float>(ws, p.o_dW0), false, st))) return rc;
  if ((rc = quant(p, ws, p.Wcand, p.segsW, true, W, Rows{0, p.O}, at<float>(ws, p.o_dW0), true, st))) return rc;
  if (p.chunked) return 0;         // every step builds its chunks' activation images
  if ((rc = quant(p, ws, p.Xcur, p.segsX, false, x, all_rows(p), at<float>(ws, p.o_dX0), false, st))) return rc;
  const Step& xs = p.xsteps[0];   // the candidate activation image of the activation steps (int8 for the int8 step)
  if ((rc = quant(p, ws, *xs.Rcand, *xs.Rcand_segs, false, x, all_rows(p), at<float>(ws, p.o_dX0), true, st))) return rc;
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
  if ((rc = quant(p, workspace, p.Wcur, p.segsW, true, weight, Rows{0, p.O}, at<float>(workspace, p.o_dW), false, st))) return rc;
  if ((rc = quant(p, workspace, p.Xcur, p.segsX, false, x, all_rows(p), at<float>(workspace, p.o_dX), false, st))) return rc;
  if ((rc = tables_for(p, workspace, p.fwd, -1, 0, st))) return rc;
  SweepParams sp; fill_sweep(p, workspace, p.fwd, sp, all_rows(p));
  sp.bias = d->has_bias ? bias : nullptr;
  sp.out = out; sp.n_cand = 1; sp.order = 0;
  sp.R_cand = nullptr; sp.C_cand = nullptr;
  return run_sweep(p, p.fwd, sp, st);
}

// ---- frozen layers: integer weights packed once, forward without any FP32 weight ----------------------------------
namespace {

// The forward-only plan of the layer with int8 operands, its tables addressed inside the packed buffer:
//   [int8 weight image][scale table][activation step sizes][jobs][activation segments][weight segments][group meta]
struct FrozenPlan {
  LinPlan p;
  size_t o_dX, bytes;
  int stages, stage_kb;                 // fused kernel: ring stages (0 = streamed path) and bytes of K per row of a stage
  Image X;                              // streamed path: the int8 activation image in the caller's workspace
};

// for_pack: the rows of the descriptor are ignored (nothing in the packed buffer, nor the path, depends on them)
int build_frozen(const p4v_linear_desc* d, FrozenPlan& f, bool for_pack) {
  P4V_REQUIRE(d != nullptr, "null desc");
  p4v_linear_desc dd = *d;
  dd.operand = P4V_OPERAND_INT8; dd.kernel = P4V_KERNEL_TCGEN05; dd.rows_per_chunk = 0;
  if (for_pack) dd.rows = dd.tokens = 1;
  LinPlan& p = f.p;
  int rc = build_plan(&dd, p, false);
  if (rc) return rc;
  Carver c{0};
  p.Wcur.off = c.take(p.Wcur.bytes());
  p.o_fix = c.take((size_t)p.fwd.nfg * p.nsg * 4);
  f.o_dX = p.o_dX = c.take((size_t)dd.n_a * 4);
  p.jobs.off = c.take(p.jobs.bytes());
  p.segsX.off = c.take(p.segsX.bytes());
  p.segsW.off = c.take(p.segsW.bytes());
  p.metas.off = c.take(p.metas.bytes());
  f.bytes = c.end;
  f.stage_kb = 32;
  for (int j = 0; j < p.fwd.nfj; ++j) {
    const P4VJob& jb = p.jobs.host[p.fwd.job_off + j];
    f.stage_kb = std::max(f.stage_kb, (int)(jb.kb * p4v_job_nsub(jb)));
  }
  f.X = p.Xcur; f.X.off = 0;
  f.stages = frozen_ring_stages(f.X.tile_bytes(), (size_t)f.stage_kb * P4V_TILE, p.Wcur.kb / 16);
  return 0;
}

// The ring stages the fused kernel gets for a call of the layer f1 with the folds `folds` -- as fc1 of a fused MLP whose
// fc2 is f2 (P4V_FOLD_MLP), with a LayerNorm folded into its activation quantiser (NORM), with a row gather of
// gather_mode in front of that LayerNorm (GATHER), as an attention block's qkv writing int8 planes (QKV8) -- or 0 when
// the call does not take the fused kernel.  f1 must be on it
// itself; an MLP needs fc1's outputs to be fc2's inputs and a plain fc1, a LayerNorm a plain layer with K % 4 == 0, the
// merge gather C = K / 4 a multiple of 4, so that no float4 of the LayerNorm's walk straddles a quarter.  The epilogue,
// the gather's source rows and the row stats take their share of shared memory, which can only lower the count.
int fold_stages(const FrozenPlan& f1, const FrozenPlan* f2, unsigned folds, int gather_mode = 0) {
  const LinPlan& p1 = f1.p;
  if (f1.stages < 2 || (f2 && (p1.O != f2->p.K || p1.twin)) ||
      ((folds & P4V_FOLD_NORM) && (p1.twin || p1.K % 4 != 0)) ||
      ((folds & P4V_FOLD_GATHER) && gather_mode == P4V_GATHER_MERGE && p1.K % 16 != 0)) return 0;
  // a plane of fc2's activation image has the K layout of its weight image; a post-GELU fc2 has two
  const unsigned epi = f2 ? p4v_mlp_epi_bytes(f2->p.twin ? 2 : 1, f2->p.Wcur.kb / 16) : 0u;
  return frozen_ring_stages(f1.X.tile_bytes() + p4v_fwd_extra_bytes(folds, epi), (size_t)f1.stage_kb * P4V_TILE,
                            p1.Wcur.kb / 16);
}

}  // namespace

extern "C" int p4v_linear_pack_bytes(const p4v_linear_desc* d, size_t* bytes) {
  FrozenPlan f; int rc = build_frozen(d, f, true);
  if (rc) return rc;
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = f.bytes;
  return 0;
}

extern "C" int p4v_linear_pack(const p4v_linear_desc* d, const float* weight, const float* w_interval, const float* a_interval,
                               void* packed, size_t packed_bytes, void* stream) {
  FrozenPlan f; int rc = build_frozen(d, f, true);
  if (rc) return rc;
  const LinPlan& p = f.p;
  P4V_REQUIRE(weight && w_interval && a_interval && packed, "linear_pack: null pointer");
  P4V_REQUIRE(packed_bytes >= f.bytes, "linear_pack: packed buffer too small (%zu < %zu)", packed_bytes, f.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = p.jobs.upload(packed, st)) || (rc = p.segsX.upload(packed, st)) || (rc = p.segsW.upload(packed, st)) ||
      (rc = p.metas.upload(packed, st))) return rc;
  P4V_CUDA_OK(cudaMemcpyAsync(at<float>(packed, f.o_dX), a_interval, (size_t)d->n_a * 4, cudaMemcpyDeviceToDevice, st));
  if ((rc = quant(p, packed, p.Wcur, p.segsW, true, weight, Rows{0, p.O}, w_interval, false, st))) return rc;
  StepTablesArgs t = tables_args(p, packed, p.fwd, -1, 0);
  t.dW = w_interval; t.dX = a_interval;
  return p4v_step_tables(t, st);
}

extern "C" int p4v_linear_frozen_path(const p4v_linear_desc* d, int* path) {
  FrozenPlan f; int rc = build_frozen(d, f, true);
  if (rc) return rc;
  P4V_REQUIRE(path != nullptr, "null output");
  *path = fold_stages(f, nullptr, 0) ? 1 : 0;
  return 0;
}

extern "C" int p4v_linear_frozen_workspace_bytes(const p4v_linear_desc* d, size_t* bytes) {
  FrozenPlan f; int rc = build_frozen(d, f, false);
  if (rc) return rc;
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = fold_stages(f, nullptr, 0) ? 0 : f.X.bytes();
  return 0;
}

namespace {

// The fused kernel's parameters of a frozen layer whose path is the fused kernel
void fill_fwd(const FrozenPlan& f, const float* x, const float* bias, void* packed, float* out, FwdParams& q) {
  const LinPlan& p = f.p;
  q.x = x; q.ld = p.K; q.M = p.M; q.N = p.O; q.bias = p.d.has_bias ? bias : nullptr; q.out = out;
  q.W = p.Wcur.ptr(packed); q.W_tile_bytes = p.Wcur.tile_bytes(); q.tiles_m = p.tiles_m; q.tiles_n = p.tiles_o;
  q.scale = at<float>(packed, p.o_fix); q.nsg = p.nsg; q.n_groups = p.fwd.nfg;
  q.jobs = p.jobs.dev(packed) + p.fwd.job_off; q.n_jobs = p.fwd.nfj;
  q.segs = p.segsX.dev(packed); q.nseg = (int)p.segs.size();
  q.dX = at<float>(packed, f.o_dX);
  q.twin = p.twin; q.d_neg = p.d_neg; q.lo = p.twin ? 0.f : (float)-p.a_qmax; q.hi = (float)(p.a_qmax - 1);
  q.neg_lo = (float)-p.a_qmax; q.ieee_div = p4v_scalar_div_ieee();
  q.plane_bytes = (unsigned)p.Wcur.tile_bytes(); q.a_bytes = (unsigned)f.X.tile_bytes();
  q.stage_bytes = (unsigned)f.stage_kb * P4V_TILE; q.n_stages = (unsigned)f.stages; q.n_chunks = (unsigned)p.Wcur.kb / 16;
}

// fc2's part of a fused MLP's parameters: the epilogue writes fc2's activation image into the workspace
void fill_mlp(const FrozenPlan& f2, void* pack2, void* workspace, FwdParams& q) {
  const LinPlan& p2 = f2.p;
  q.X2 = f2.X.ptr(workspace); q.X2_tile_bytes = f2.X.tile_bytes(); q.X2_plane_bytes = (unsigned)p2.Wcur.tile_bytes();
  q.segs2 = p2.segsX.dev(pack2); q.nseg2 = (int)p2.segs.size();
  q.n_chunks2 = p2.Wcur.kb / 16; q.planes2 = p2.twin ? 2 : 1;
  q.dX2 = at<float>(pack2, f2.o_dX); q.crb_acts2 = p2.crb_acts;
  q.d_neg2 = p2.d_neg; q.lo2 = p2.twin ? 0.f : (float)-p2.a_qmax; q.hi2 = (float)(p2.a_qmax - 1); q.neg_lo2 = (float)-p2.a_qmax;
  q.epi_bytes = p4v_mlp_epi_bytes(q.planes2, q.n_chunks2);
}

// The second half of the streamed path: the sweep forward of the layer's int8 activation image in the workspace; with
// res, the store adds the residual (sweep_tc.cu, kModeFwdRes)
int streamed_sweep(const FrozenPlan& f, void* packed, void* workspace, const float* bias, const float* res, float* out,
                   cudaStream_t st) {
  const LinPlan& p = f.p;
  SweepParams sp; fill_sweep(p, packed, p.fwd, sp, all_rows(p));
  sp.R_cur = f.X.ptr(workspace);
  sp.bias = p.d.has_bias ? bias : nullptr;
  sp.out = out; sp.res = res; sp.n_cand = 1; sp.order = 0;
  sp.R_cand = nullptr; sp.C_cand = nullptr;
  return run_sweep(p, p.fwd, sp, st);
}

// The arguments of a folded LayerNorm
int check_norm(const char* what, const float* x, const float* gamma, const float* beta, float eps) {
  P4V_REQUIRE(x && gamma && beta, "%s: null pointer", what);
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(gamma) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(beta) & 15) == 0, "%s: x, gamma and beta must be 16-byte aligned", what);
  P4V_REQUIRE(eps >= 0.f && eps <= 3.4028234663852886e38f, "%s: eps must be finite and non-negative (got %g)", what, (double)eps);
  return 0;
}

// The window layout rule of a layer with `rows` output rows (DESIGN §4.11)
int check_layout(const char* fn, const p4v_window_layout& win, int rows) {
  P4V_REQUIRE(win.window > 0 && win.height > 0 && win.width > 0 && win.images > 0,
              "%s: window layout needs positive images, height, width and window (got %d, %d, %d, %d)", fn, win.images,
              win.height, win.width, win.window);
  P4V_REQUIRE(win.height % win.window == 0 && win.width % win.window == 0,
              "%s: window layout: height %d and width %d must be multiples of the window %d", fn, win.height, win.width,
              win.window);
  P4V_REQUIRE(win.shift >= 0 && win.shift < win.window, "%s: window layout: shift %d must lie in [0, window %d)", fn,
              win.shift, win.window);
  P4V_REQUIRE((long long)win.images * win.height * win.width == rows,
              "%s: window layout: images * height * width = %lld, the layer has %d rows", fn,
              (long long)win.images * win.height * win.width, rows);
  return 0;
}

// The layout of a non-null row gather (DESIGN §4.12) of a call with `rows` output rows and K = in_features, the image x
// apart from out (out_bytes: [rows][out_cols] FP32, or the int8 planes of a qkv fold); x's null pointer and alignment are
// check_norm's
int check_gather(const char* fn, const p4v_input_gather& g, const float* x, const void* out, size_t out_bytes, int rows, int K) {
  const p4v_window_layout& w = g.layout;
  if (g.mode == P4V_GATHER_WINDOW) {
    if (int rc = check_layout(fn, w, rows)) return rc;
  } else {
    P4V_REQUIRE(g.mode == P4V_GATHER_MERGE, "%s: gather mode must be P4V_GATHER_WINDOW or P4V_GATHER_MERGE (got %d)", fn,
                g.mode);
    P4V_REQUIRE(w.window == 0 && w.shift == 0, "%s: merge layout: window and shift must be 0 (got %d, %d)", fn, w.window,
                w.shift);
    P4V_REQUIRE(w.images > 0 && w.height > 0 && w.width > 0 && w.height % 2 == 0 && w.width % 2 == 0,
                "%s: merge layout needs positive images and even height and width (got %d, %d, %d)", fn, w.images,
                w.height, w.width);
    P4V_REQUIRE(K % 4 == 0, "%s: merge: in_features %d must be 4 C", fn, K);
    P4V_REQUIRE((long long)w.images * (w.height / 2) * (w.width / 2) == rows,
                "%s: merge layout: images * (height / 2) * (width / 2) = %lld, the layer has %d rows", fn,
                (long long)w.images * (w.height / 2) * (w.width / 2), rows);
  }
  // either way the image holds rows * K floats
  const uintptr_t xb = (uintptr_t)rows * (uintptr_t)K * 4, ob = out_bytes, a = reinterpret_cast<uintptr_t>(x),
                  b = reinterpret_cast<uintptr_t>(out);
  P4V_REQUIRE(a + xb <= b || b + ob <= a, "%s: x overlaps out", fn);
  return 0;
}

// The arguments of a folded residual add (res non-null) of a call whose output out is [rows][cols]: res 8-byte aligned
// and apart from out, and the window layout's rule (win.window == 0: identity rows).  Nothing to check without res.
int check_residual(const char* fn, const float* res, const float* out, int rows, int cols, const p4v_window_layout& win) {
  if (!res) return 0;
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(res) & 7) == 0, "%s: residual must be 8-byte aligned", fn);
  const uintptr_t bytes = (uintptr_t)rows * (uintptr_t)cols * 4, a = reinterpret_cast<uintptr_t>(res),
                  b = reinterpret_cast<uintptr_t>(out);
  P4V_REQUIRE(a + bytes <= b || b + bytes <= a, "%s: residual overlaps out", fn);
  if (win.window != 0 || win.images != 0 || win.height != 0 || win.width != 0 || win.shift != 0)
    return check_layout(fn, win, rows);
  return 0;
}

// One call of frozen layers: layer f1 on x, optionally with a LayerNorm folded into its activation quantiser (ln), with
// its rows gathered from an image in front of that LayerNorm (gather, *ga), as fc1 of a fused MLP whose epilogue writes
// the image of its fc2 (f2) into the workspace, which fc2's sweep forward then reads, and with a residual added by the
// last store (rs.res non-null; rs.win: Swin's window reverse, on f1's fused kernel only), or as an attention block's qkv
// whose epilogue writes the attention's int8 planes (q8 non-null; out null).
struct FrozenCall {
  const FrozenPlan* f1; const float* x; const float* bias1; const void* pack1; size_t pack1_bytes;
  const FwdNorm* ln;                                   // null: no LayerNorm
  bool gather; const p4v_input_gather* ga;
  const FrozenPlan* f2; const float* bias2; const void* pack2; size_t pack2_bytes;   // f2 null: no MLP
  FwdResidual rs;
  const FwdQkv8* q8;                                   // null: FP32 output
  void* workspace; size_t workspace_bytes;
  float* out;
};

FrozenCall linear_call(const FrozenPlan& f, const float* x, const float* bias, const void* packed, float* out) {
  FrozenCall c{};
  c.f1 = &f; c.x = x; c.bias1 = bias; c.pack1 = packed; c.out = out;
  return c;
}

FrozenCall mlp_call(const FrozenPlan& f1, const float* x, const float* bias1, const void* pack1, size_t pack1_bytes,
                    const FrozenPlan& f2, const float* bias2, const void* pack2, size_t pack2_bytes, void* workspace,
                    size_t workspace_bytes, float* out) {
  FrozenCall c = linear_call(f1, x, bias1, pack1, out);
  c.pack1_bytes = pack1_bytes; c.f2 = &f2; c.bias2 = bias2; c.pack2 = pack2; c.pack2_bytes = pack2_bytes;
  c.workspace = workspace; c.workspace_bytes = workspace_bytes;
  return c;
}

// Validates every argument of the call c of entry point fn (with its name in the messages), then runs it: the fused
// kernel with the call's folds (then fc2's sweep forward for an MLP), or, for a plain layer that is not on the fused
// kernel, the streamed path (the int8 activation image in the workspace, then the layer's sweep forward).
int frozen_call(const char* fn, const FrozenCall& c, cudaStream_t st) {
  const FrozenPlan& f1 = *c.f1;
  const bool mlp = c.f2 != nullptr, norm = c.ln != nullptr;
  const unsigned folds = (mlp ? P4V_FOLD_MLP : 0u) | (norm ? P4V_FOLD_NORM : 0u) | (c.gather ? P4V_FOLD_GATHER : 0u) |
                         (c.rs.res && !mlp ? P4V_FOLD_RES : 0u) | (c.q8 ? P4V_FOLD_QKV8 : 0u);
  if (norm) {
    if (int rc = check_norm(fn, c.x, c.ln->gamma, c.ln->beta, c.ln->eps)) return rc;
  }
  if (mlp)
    P4V_REQUIRE(f1.p.d.rows == c.f2->p.d.rows, "%s: fc1 and fc2 must have the same rows (%d != %d)", fn, f1.p.d.rows,
                c.f2->p.d.rows);
  P4V_REQUIRE(c.x && c.pack1 && (!mlp || (c.pack2 && c.workspace)) && (c.out || (c.q8 && c.q8->planes)), "%s: null pointer", fn);
  P4V_REQUIRE((!f1.p.d.has_bias || c.bias1) && (!mlp || !c.f2->p.d.has_bias || c.bias2), "%s: has_bias set but bias is null", fn);
  if (c.gather) P4V_REQUIRE(c.ga, "%s: null pointer", fn);
  const int stages = fold_stages(f1, c.f2, folds, c.gather ? c.ga->mode : 0);
  if (folds & ~P4V_FOLD_RES)
    P4V_REQUIRE(stages, "%s: %s", fn, c.q8 ? "the attention operands do not fold into this qkv (p4v_linear_qkv8_ok)"
                                    : mlp ? (norm ? "these layers do not fuse with the LayerNorm (p4v_mlp_norm_ok)"
                                                  : "these layers do not fuse (p4v_mlp_fused_ok)")
                                          : c.gather ? "the gather does not fold into this layer (p4v_linear_gather_ok)"
                                                     : "the LayerNorm does not fold into this layer (p4v_linear_norm_ok)");
  // the int8 planes of a qkv fold take the place of the FP32 output
  const void* dst = c.q8 ? static_cast<const void*>(c.q8->planes) : static_cast<const void*>(c.out);
  const size_t dst_bytes = (size_t)f1.p.M * (size_t)f1.p.O * (c.q8 ? 1 : 4);
  if (c.gather) {
    if (int rc = check_gather(fn, *c.ga, c.x, dst, dst_bytes, f1.p.M, f1.p.K)) return rc;
  } else if (c.q8) {
    const uintptr_t xb = (uintptr_t)f1.p.M * (uintptr_t)f1.p.K * 4, a = reinterpret_cast<uintptr_t>(c.x),
                    b = reinterpret_cast<uintptr_t>(dst);
    P4V_REQUIRE(a + xb <= b || b + dst_bytes <= a, "%s: x overlaps the planes", fn);
  }
  if (mlp) {
    P4V_REQUIRE(c.pack1_bytes >= f1.bytes && c.pack2_bytes >= c.f2->bytes, "%s: packed buffer too small "
                "(fc1 %zu < %zu or fc2 %zu < %zu)", fn, c.pack1_bytes, f1.bytes, c.pack2_bytes, c.f2->bytes);
    P4V_REQUIRE((reinterpret_cast<uintptr_t>(c.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.out) & 7) == 0 &&
                (reinterpret_cast<uintptr_t>(c.workspace) & 15) == 0,
                "%s: %sworkspace must be 16-byte and out 8-byte aligned", fn, norm ? "" : "x and ");   // check_norm took x
    P4V_REQUIRE(c.workspace_bytes >= c.f2->X.bytes(), "%s: workspace too small (%zu < %zu)", fn, c.workspace_bytes,
                c.f2->X.bytes());
  }
  if (!stages) {
    P4V_REQUIRE(c.workspace && c.workspace_bytes >= f1.X.bytes(), "%s: workspace too small (%zu < %zu)", fn,
                c.workspace ? c.workspace_bytes : (size_t)0, f1.X.bytes());
    P4V_REQUIRE(c.rs.win.window == 0, "%s: a window layout needs the fused path (p4v_linear_frozen_path 1)", fn);
  }
  if (int rc = check_residual(fn, c.rs.res, c.out, f1.p.M, mlp ? c.f2->p.O : f1.p.O, c.rs.win)) return rc;
  // the plan's accessors take the buffers they index; nothing writes them
  void* p1 = const_cast<void*>(c.pack1);
  void* p2 = const_cast<void*>(c.pack2);
  if (!stages) {
    const LinPlan& p = f1.p;
    QuantImageArgs qa{};
    f1.X.fill(qa, c.workspace);
    qa.src = c.x; qa.ld = p.K; qa.rows = p.M; qa.delta = at<float>(p1, f1.o_dX); qa.d_mod = 1;
    qa.rows_per_block = p.M + P4V_TILE; qa.segs = p.segsX.dev(p1); qa.nseg = (int)p.segsX.host.size();
    if (int rc = p4v_quant_image(qa, st)) return rc;
    return streamed_sweep(f1, p1, c.workspace, c.bias1, c.rs.res, c.out, st);
  }
  FwdParams q{};
  fill_fwd(f1, c.x, c.bias1, p1, mlp ? nullptr : c.out, q);
  q.n_stages = (unsigned)stages;
  if (mlp) fill_mlp(*c.f2, p2, c.workspace, q);
  if (norm) q.ln = *c.ln;
  if (folds & P4V_FOLD_RES) q.rs = c.rs;
  if (c.gather) q.ga = FwdGather{c.ga->mode, c.ga->layout};
  if (c.q8) q.q8 = *c.q8;
  const int rc = p4v_launch_forward_tc(q, folds, p4v_num_sms(), st);
  if (rc || !mlp) return rc;
  return streamed_sweep(*c.f2, p2, c.workspace, c.bias2, c.rs.res, c.out, st);
}

}  // namespace

extern "C" int p4v_linear_frozen_forward(const p4v_linear_desc* d, const float* x, const float* bias, const void* packed,
                                         void* workspace, size_t workspace_bytes, float* out, void* stream) {
  FrozenPlan f; int rc = build_frozen(d, f, false);
  if (rc) return rc;
  FrozenCall c = linear_call(f, x, bias, packed, out);
  c.workspace = workspace; c.workspace_bytes = workspace_bytes;
  return frozen_call("linear_frozen_forward", c, (cudaStream_t)stream);
}

// ---- fused frozen MLP: fc1 + GELU + fc2's activation quantiser in one kernel, then fc2's sweep forward -----------
namespace {

// for_rule: the rows of the descriptors are ignored (p4v_mlp_fused_ok, p4v_mlp_norm_ok)
int build_mlp(const p4v_linear_desc* d1, const p4v_linear_desc* d2, FrozenPlan& f1, FrozenPlan& f2, bool for_rule) {
  P4V_REQUIRE(d1 && d2, "mlp: null desc");
  if (int rc = build_frozen(d1, f1, for_rule)) return rc;
  return build_frozen(d2, f2, for_rule);
}

}  // namespace

extern "C" int p4v_mlp_fused_ok(const p4v_linear_desc* fc1, const p4v_linear_desc* fc2, int* ok) {
  FrozenPlan f1, f2; int rc = build_mlp(fc1, fc2, f1, f2, true);
  if (rc) return rc;
  P4V_REQUIRE(ok != nullptr, "null output");
  *ok = fold_stages(f1, &f2, P4V_FOLD_MLP) ? 1 : 0;
  return 0;
}

extern "C" int p4v_mlp_frozen_workspace_bytes(const p4v_linear_desc* fc1, const p4v_linear_desc* fc2, size_t* bytes) {
  FrozenPlan f1, f2; int rc = build_mlp(fc1, fc2, f1, f2, false);
  if (rc) return rc;
  P4V_REQUIRE(fc1->rows == fc2->rows, "mlp: fc1 and fc2 must have the same rows (%d != %d)", fc1->rows, fc2->rows);
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = f2.X.bytes();
  return 0;
}

extern "C" int p4v_mlp_frozen_forward(const p4v_linear_desc* fc1, const float* x, const float* bias1, const void* pack1,
                                      size_t pack1_bytes, const p4v_linear_desc* fc2, const float* bias2, const void* pack2,
                                      size_t pack2_bytes, void* workspace, size_t workspace_bytes, float* out, void* stream) {
  FrozenPlan f1, f2; int rc = build_mlp(fc1, fc2, f1, f2, false);
  if (rc) return rc;
  return frozen_call("mlp_frozen_forward", mlp_call(f1, x, bias1, pack1, pack1_bytes, f2, bias2, pack2, pack2_bytes,
                                                    workspace, workspace_bytes, out), (cudaStream_t)stream);
}

// ---- LayerNorm folded into the activation quantiser of the fused kernel (forward_tc.cu, DESIGN §4.10) -------------
extern "C" int p4v_linear_norm_ok(const p4v_linear_desc* d, int* ok) {
  FrozenPlan f; int rc = build_frozen(d, f, true);
  if (rc) return rc;
  P4V_REQUIRE(ok != nullptr, "null output");
  *ok = fold_stages(f, nullptr, P4V_FOLD_NORM) ? 1 : 0;
  return 0;
}

extern "C" int p4v_mlp_norm_ok(const p4v_linear_desc* fc1, const p4v_linear_desc* fc2, int* ok) {
  FrozenPlan f1, f2; int rc = build_mlp(fc1, fc2, f1, f2, true);
  if (rc) return rc;
  P4V_REQUIRE(ok != nullptr, "null output");
  *ok = fold_stages(f1, &f2, P4V_FOLD_MLP | P4V_FOLD_NORM) ? 1 : 0;
  return 0;
}

extern "C" int p4v_linear_frozen_forward_norm(const p4v_linear_desc* d, const float* x, const float* gamma, const float* beta,
                                              float eps, const float* bias, const void* packed, float* out, void* stream) {
  FrozenPlan f; int rc = build_frozen(d, f, false);
  if (rc) return rc;
  const FwdNorm ln{gamma, beta, eps};
  FrozenCall c = linear_call(f, x, bias, packed, out);
  c.ln = &ln;
  return frozen_call("linear_frozen_forward_norm", c, (cudaStream_t)stream);
}

extern "C" int p4v_mlp_frozen_forward_norm(const p4v_linear_desc* fc1, const float* x, const float* gamma, const float* beta,
                                           float eps, const float* bias1, const void* pack1, size_t pack1_bytes,
                                           const p4v_linear_desc* fc2, const float* bias2, const void* pack2, size_t pack2_bytes,
                                           void* workspace, size_t workspace_bytes, float* out, void* stream) {
  FrozenPlan f1, f2; int rc = build_mlp(fc1, fc2, f1, f2, false);
  if (rc) return rc;
  const FwdNorm ln{gamma, beta, eps};
  FrozenCall c = mlp_call(f1, x, bias1, pack1, pack1_bytes, f2, bias2, pack2, pack2_bytes, workspace, workspace_bytes, out);
  c.ln = &ln;
  return frozen_call("mlp_frozen_forward_norm", c, (cudaStream_t)stream);
}

// ---- a block's residual add folded into the store of the frozen Linear that produces it (DESIGN §4.11) -------------
// Each entry point replaces  residual + <the call without _res>  (torch's FP32 add; Swin's proj also the window reverse
// and the reverse roll before it, through the layout).  A null residual is an error here, not the call without it.
extern "C" int p4v_linear_frozen_forward_res(const p4v_linear_desc* d, const float* x, const float* bias, const void* packed,
                                             void* workspace, size_t workspace_bytes, const float* residual,
                                             const p4v_window_layout* layout, float* out, void* stream) {
  P4V_REQUIRE(residual, "linear_frozen_forward_res: null pointer");
  FrozenPlan f; int rc = build_frozen(d, f, false);
  if (rc) return rc;
  FrozenCall c = linear_call(f, x, bias, packed, out);
  c.workspace = workspace; c.workspace_bytes = workspace_bytes;
  c.rs = FwdResidual{residual, layout ? *layout : p4v_window_layout{}};
  return frozen_call("linear_frozen_forward_res", c, (cudaStream_t)stream);
}

extern "C" int p4v_mlp_frozen_forward_res(const p4v_linear_desc* fc1, const float* x, const float* bias1, const void* pack1,
                                          size_t pack1_bytes, const p4v_linear_desc* fc2, const float* bias2, const void* pack2,
                                          size_t pack2_bytes, void* workspace, size_t workspace_bytes, const float* residual,
                                          float* out, void* stream) {
  FrozenPlan f1, f2; int rc = build_mlp(fc1, fc2, f1, f2, false);
  if (rc) return rc;
  P4V_REQUIRE(residual, "mlp_frozen_forward_res: null pointer");
  FrozenCall c = mlp_call(f1, x, bias1, pack1, pack1_bytes, f2, bias2, pack2, pack2_bytes, workspace, workspace_bytes, out);
  c.rs.res = residual;
  return frozen_call("mlp_frozen_forward_res", c, (cudaStream_t)stream);
}

extern "C" int p4v_mlp_frozen_forward_norm_res(const p4v_linear_desc* fc1, const float* x, const float* gamma, const float* beta,
                                               float eps, const float* bias1, const void* pack1, size_t pack1_bytes,
                                               const p4v_linear_desc* fc2, const float* bias2, const void* pack2,
                                               size_t pack2_bytes, void* workspace, size_t workspace_bytes,
                                               const float* residual, float* out, void* stream) {
  FrozenPlan f1, f2; int rc = build_mlp(fc1, fc2, f1, f2, false);
  if (rc) return rc;
  P4V_REQUIRE(residual, "mlp_frozen_forward_norm_res: null pointer");
  const FwdNorm ln{gamma, beta, eps};
  FrozenCall c = mlp_call(f1, x, bias1, pack1, pack1_bytes, f2, bias2, pack2, pack2_bytes, workspace, workspace_bytes, out);
  c.ln = &ln; c.rs.res = residual;
  return frozen_call("mlp_frozen_forward_norm_res", c, (cudaStream_t)stream);
}

// ---- a row gather in front of the LayerNorm folded into its frozen Linear (DESIGN §4.12) ---------------------------
// Replaces  layer(LayerNorm(gather(x)))  with gather Swin's roll(-shift) + window partition, or PatchMerging's 2x2 cat.
extern "C" int p4v_linear_gather_ok(const p4v_linear_desc* d, const p4v_input_gather* g, int* ok) {
  FrozenPlan f; int rc = build_frozen(d, f, true);
  if (rc) return rc;
  P4V_REQUIRE(g && ok, "null argument");
  P4V_REQUIRE(g->mode == P4V_GATHER_WINDOW || g->mode == P4V_GATHER_MERGE,
              "linear_gather_ok: gather mode must be P4V_GATHER_WINDOW or P4V_GATHER_MERGE (got %d)", g->mode);
  *ok = fold_stages(f, nullptr, P4V_FOLD_NORM | P4V_FOLD_GATHER, g->mode) ? 1 : 0;
  return 0;
}

extern "C" int p4v_linear_frozen_forward_norm_gather(const p4v_linear_desc* d, const float* x, const float* gamma,
                                                     const float* beta, float eps, const float* bias, const void* packed,
                                                     const p4v_input_gather* g, float* out, void* stream) {
  FrozenPlan f; int rc = build_frozen(d, f, false);
  if (rc) return rc;
  const FwdNorm ln{gamma, beta, eps};
  FrozenCall c = linear_call(f, x, bias, packed, out);
  c.ln = &ln; c.gather = true; c.ga = g;
  return frozen_call("linear_frozen_forward_norm_gather", c, (cudaStream_t)stream);
}

// ---- the attention operands' quantisation folded into the frozen qkv (DESIGN §4.14) --------------------------------
namespace {

// The fold set of a qkv call for the rule: with a window gather NORM | GATHER; without one, NORM too when the layer can
// take a LayerNorm, so that the rule holds with and without it
unsigned qkv8_rule_folds(const FrozenPlan& f, int gather_mode) {
  if (gather_mode) return P4V_FOLD_QKV8 | P4V_FOLD_NORM | P4V_FOLD_GATHER;
  return P4V_FOLD_QKV8 | (!f.p.twin && f.p.K % 4 == 0 ? P4V_FOLD_NORM : 0u);
}

// The rule without the attention's own (p4v_attention_fused_ok): out_features == 3 C and the fused plan fits
bool qkv8_fits(const FrozenPlan& f, const p4v_attention_desc& a, int gather_mode) {
  return (long long)f.p.O == 3LL * a.heads * a.head_dim && fold_stages(f, nullptr, qkv8_rule_folds(f, gather_mode), gather_mode) > 0;
}

}  // namespace

extern "C" int p4v_linear_qkv8_ok(const p4v_linear_desc* d, const p4v_attention_desc* a, int gather_mode, int* ok) {
  FrozenPlan f; int rc = build_frozen(d, f, true);
  if (rc) return rc;
  P4V_REQUIRE(a && ok, "null argument");
  P4V_REQUIRE(gather_mode == 0 || gather_mode == P4V_GATHER_WINDOW,
              "linear_qkv8_ok: gather mode must be 0 or P4V_GATHER_WINDOW (got %d)", gather_mode);
  int attn = 0;
  p4v_attention_fused_ok(a->tokens, a->head_dim, &attn);
  *ok = attn && a->heads > 0 && qkv8_fits(f, *a, gather_mode) ? 1 : 0;
  return 0;
}

extern "C" int p4v_linear_frozen_forward_qkv8(const p4v_linear_desc* d, const float* x, const float* bias, const void* packed,
                                              const p4v_attention_desc* a, const p4v_matmul_desc* mm1, const void* pack1,
                                              size_t pack1_bytes, const p4v_matmul_desc* mm2, const void* pack2,
                                              size_t pack2_bytes, int8_t* planes, const float* gamma, const float* beta,
                                              float eps, const p4v_input_gather* g, void* stream) {
  const char* fn = "linear_frozen_forward_qkv8";
  FrozenPlan f; int rc = build_frozen(d, f, false);
  if (rc) return rc;
  P4V_REQUIRE(planes, "%s: null pointer", fn);
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(planes) & 15) == 0, "%s: planes must be 16-byte aligned", fn);
  P4V_REQUIRE(!g || g->mode == P4V_GATHER_WINDOW, "%s: gather mode must be P4V_GATHER_WINDOW (got %d)", fn, g->mode);
  P4V_REQUIRE(!g || gamma, "%s: a gather needs the LayerNorm (gamma, beta)", fn);
  FwdQkv8 q8{};
  if ((rc = p4v_qkv8_steps(fn, a, mm1, pack1, pack1_bytes, mm2, pack2, pack2_bytes, q8))) return rc;
  P4V_REQUIRE((long long)a->batch * a->tokens == d->rows, "%s: batch * tokens = %lld, the layer has %d rows", fn,
              (long long)a->batch * a->tokens, d->rows);
  int attn = 0;
  p4v_attention_fused_ok(a->tokens, a->head_dim, &attn);
  P4V_REQUIRE(attn && qkv8_fits(f, *a, g ? g->mode : 0), "%s: the attention operands do not fold into this qkv "
              "(p4v_linear_qkv8_ok)", fn);
  q8.planes = reinterpret_cast<uint8_t*>(planes);
  const FwdNorm ln{gamma, beta, eps};
  FrozenCall c = linear_call(f, x, bias, packed, nullptr);
  c.q8 = &q8;
  if (gamma) c.ln = &ln;
  if (g) { c.gather = true; c.ga = g; }
  return frozen_call(fn, c, (cudaStream_t)stream);
}
