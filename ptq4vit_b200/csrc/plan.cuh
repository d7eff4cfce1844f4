// Host-side planning shared by the Linear, MatMul and Conv searches: workspace carving, job emission, host tables and
// their upload, and the layout of the operand images in the workspace.  Host code only.
#pragma once
#include <algorithm>
#include <vector>

#include "forward.cuh"
#include "prep.cuh"

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
template <class T> T* at(void* ws, size_t off) { return reinterpret_cast<T*>(static_cast<uint8_t*>(ws) + off); }

// Workspace regions handed out in call order from `end` on, each starting 256-byte aligned
struct Carver {
  size_t end;
  size_t take(size_t bytes) { const size_t r = end; end = align_up(end + bytes, 256); return r; }
};

// A table built on the host and the workspace offset of its device copy
template <class T> struct Table {
  std::vector<T> host;
  size_t off = 0;
  size_t bytes() const { return host.size() * sizeof(T); }
  T* dev(void* ws) const { return at<T>(ws, off); }
  int upload(void* ws, cudaStream_t st) const {
    if (!host.empty()) P4V_CUDA_OK(cudaMemcpyAsync(dev(ws), host.data(), bytes(), cudaMemcpyHostToDevice, st));
    return 0;
  }
};

// Jobs of one accumulator group over kb bytes of K at byte offsets r_off / c_off of the row and column tile rows.
// first / last: the group starts / ends with these jobs (a group may chain several calls).
inline void add_group(std::vector<P4VJob>& jobs, int r_off, int c_off, int kb, uint8_t flags, int group, bool first, bool last,
                      int& count) {
  for (int b = 0; b < kb; b += P4V_JOB_KB) {
    P4VJob j{};
    const int len = std::min(P4V_JOB_KB, kb - b);
    j.r_off = (uint32_t)(r_off + b) * P4V_TILE;
    j.c_off = (uint32_t)(c_off + b) * P4V_TILE;
    j.kb = (uint8_t)len;
    j.flags = flags | ((first && b == 0) ? P4V_JOB_FIRST : 0) | ((last && b + len >= kb) ? P4V_JOB_LAST : 0);
    j.group = (uint8_t)group;
    jobs.push_back(j);
    ++count;
  }
}

// Candidate jobs [first, first + n) whose row operand does not depend on the candidate: keep that operand resident in
// shared memory when it fits
inline void mark_resident(std::vector<P4VJob>& jobs, int first, int n) {
  uint32_t total = 0;
  for (int j = first; j < first + n; ++j) {
    if (jobs[j].flags & P4V_JOB_RCAND) return;
    total += (uint32_t)jobs[j].kb * P4V_TILE;
  }
  if (total > 60 * 1024) return;
  uint32_t off = 0;
  for (int j = first; j < first + n; ++j) {
    jobs[j].flags |= P4V_JOB_RRES; jobs[j].res_off = off; off += (uint32_t)jobs[j].kb * P4V_TILE;
  }
}

// eq_n + 1 candidate factors alpha + i (beta - alpha) / eq_n (python floats -> fp32, linear.py:544-545)
inline std::vector<float> cand_factors(int eq_n, double alpha, double beta) {
  std::vector<float> f(eq_n + 1);
  for (int i = 0; i <= eq_n; ++i) f[i] = (float)(alpha + i * (beta - alpha) / eq_n);
  return f;
}

// An operand image in the workspace: `planes` planes (the candidates; 1 for a current image) of `problems` problems of
// `tiles` 128-row tiles, each row kb padded bytes of K, in the tile layout of common.cuh.  The only code that knows the
// strides of an image.
struct Image {
  size_t off;
  int kb, tiles, problems, planes;
  bool i8;
  unsigned long long tile_bytes() const { return (unsigned long long)P4V_TILE * kb; }
  unsigned long long plane_stride() const { return tile_bytes() * tiles * problems; }
  size_t bytes() const { return (size_t)plane_stride() * planes; }
  uint8_t* ptr(void* ws) const { return at<uint8_t>(ws, off); }
  // the image holding fewer tiles or problems than it was carved for (one chunk of a chunked search)
  Image chunk(int t, int n) const { Image c = *this; c.tiles = t; c.problems = n; return c; }
  void fill(QuantImageArgs& q, void* ws) const {
    q.P = problems; q.tiles = tiles; q.dst = ptr(ws); q.tile_bytes = tile_bytes(); q.plane_stride = plane_stride();
    q.n_planes = planes; q.is_int8 = i8;
  }
};

// The operand images a sweep reads.  Its operand type is that of the current column image: the images a step's jobs
// read share one type.
inline void fill_images(SweepParams& sp, void* ws, const Image& Rcur, const Image& Rcand, const Image& Ccur, const Image& Ccand) {
  sp.R_cur = Rcur.ptr(ws); sp.R_cand = Rcand.ptr(ws); sp.C_cur = Ccur.ptr(ws); sp.C_cand = Ccand.ptr(ws);
  sp.R_tile_bytes = Rcur.tile_bytes(); sp.C_tile_bytes = Ccur.tile_bytes();
  sp.R_cand_tile_bytes = Rcand.tile_bytes(); sp.C_cand_tile_bytes = Ccand.tile_bytes();
  sp.R_cand_stride = Rcand.plane_stride(); sp.C_cand_stride = Ccand.plane_stride();
  sp.is_int8 = Ccur.i8;
}

// Forward of a frozen Linear layer: weight-ring stages of stage_bytes that fit in shared memory beside the resident
// quantised activation tile and whatever else the kernel keeps there, a_bytes in all (the tile of all segments, both
// parts of a post-GELU layer, plus p4v_fwd_extra_bytes of an MLP epilogue or a LayerNorm).  At least two, and a plane
// whose 16-byte chunks fit the kernel's chunk table: the fused kernel (forward_tc.cu).  0: the call does not take it
// (a plain layer streams an int8 activation image through the sweep kernel instead).
inline int frozen_ring_stages(size_t a_bytes, size_t stage_bytes, size_t plane_chunks) {
  const size_t usable = P4V_FWD_SMEM - P4V_FWD_CTL_BYTES;
  if (plane_chunks > P4V_FWD_MAX_CHUNKS || a_bytes + 2 * stage_bytes > usable) return 0;
  return (int)std::min<size_t>((usable - a_bytes) / stage_bytes, P4V_FWD_MAX_STAGES);
}

// A commit copies the chosen candidate's slabs from the planes of cand into cur
inline void fill_images(CommitArgs& c, void* ws, const Image& cand, const Image& cur) {
  c.cand = cand.ptr(ws); c.cand_tile_bytes = cand.tile_bytes(); c.cand_plane_stride = cand.plane_stride();
  c.cur = cur.ptr(ws); c.cur_tile_bytes = cur.tile_bytes();
  c.P = cur.problems; c.tiles = cur.tiles;
}
