// Plain-CUDA (no tensor core) evaluation of the same candidate sweep, same inputs,
// same partial-score layout as sweep_tc.cu.  It exists for two reasons:
//   * bring-up / bisecting: tests compare oracle <-> simt <-> tensor-core kernel;
//   * geometries the tensor-core kernel does not take.
// It is a GPU path (selected with desc.kernel = 1), never a CPU fallback.
#include "common.cuh"

namespace {

template <bool kInt8>
__device__ __forceinline__ float dot_job(const uint8_t* rimg, const uint8_t* cimg, int row, int col, int kb) {
  // images: [chunk][128][16 bytes]
  float acc = 0.f;
  long long iacc = 0;
  const int nchunk = kb >> 4;
  for (int ch = 0; ch < nchunk; ++ch) {
    const uint8_t* a = rimg + ((size_t)ch * P4V_TILE + row) * 16;
    const uint8_t* b = cimg + ((size_t)ch * P4V_TILE + col) * 16;
    if constexpr (kInt8) {
      const int4 av = *reinterpret_cast<const int4*>(a);
      const int4 bv = *reinterpret_cast<const int4*>(b);
      int s = 0;
      s = __dp4a(av.x, bv.x, s); s = __dp4a(av.y, bv.y, s); s = __dp4a(av.z, bv.z, s); s = __dp4a(av.w, bv.w, s);
      iacc += s;
    } else {
      const __nv_bfloat16* ah = reinterpret_cast<const __nv_bfloat16*>(a);
      const __nv_bfloat16* bh = reinterpret_cast<const __nv_bfloat16*>(b);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc = fmaf(__bfloat162float(ah[i]), __bfloat162float(bh[i]), acc);
    }
  }
  return kInt8 ? (float)iacc : acc;
}

// grid: (tiles_total, candidate chunks); block: 256 threads; thread -> column t%128, rows (t/128) + 2*i
template <bool kInt8>
__global__ void __launch_bounds__(256) sweep_simt_kernel(const __grid_constant__ SweepParams P, int cand_per_block) {
  __shared__ float red[4][P4V_TILE][2];
  const int tile = blockIdx.x;
  const int c0 = blockIdx.y * cand_per_block;
  const int c1 = min(P.n_cand, c0 + cand_per_block);
  const int per_p = P.tiles_m * P.tiles_n;
  const int p = tile / per_p, t = tile % per_p;
  int tm, tn;
  if (P.order == 0) { tm = t % P.tiles_m; tn = t / P.tiles_m; } else { tn = t % P.tiles_n; tm = t / P.tiles_n; }
  const int col = threadIdx.x & 127, rpar = threadIdx.x >> 7;
  const int gcol = tn * P4V_TILE + col;
  const int cg = col >> 4;
  const int sg = (P.sg_mode == P4V_SG_COLUMN) ? tn * P4V_TILE_CG + cg : (p % P.nsg);
  const float gs = P.out ? 1.f : *P.gscale;
  const uint8_t* Rcur = P.R_cur + (size_t)(p * P.tiles_m + tm) * P.R_tile_bytes;
  const uint8_t* Ccur = P.C_cur + (size_t)(p * P.tiles_n + tn) * P.C_tile_bytes;

  for (int c = c0; c < c1; ++c) {
    const uint8_t* Rcand = P.R_cand ? P.R_cand + (size_t)c * P.R_cand_stride + (size_t)(p * P.tiles_m + tm) * P.R_cand_tile_bytes : nullptr;
    const uint8_t* Ccand = P.C_cand ? P.C_cand + (size_t)c * P.C_cand_stride + (size_t)(p * P.tiles_n + tn) * P.C_cand_tile_bytes : nullptr;
    float part[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i = 0; i < 64; ++i) {
      const int row = rpar + 2 * i;
      const int gm = tm * P4V_TILE + row;
      if (gm >= P.M || gcol >= P.N) continue;
      const size_t off = (size_t)p * P.prob_stride + (size_t)gm * P.ld + gcol;
      float r = ((P.out && !P.out_residual) ? 0.f : P.Y[off]) - (P.bias ? P.bias[gcol] : 0.f);
      const float g = P.out ? 0.f : P.Gr[off] * gs;
      // fixed groups
      float acc = 0.f;
      for (int j = 0; j < P.n_fixed_jobs; ++j) {
        const P4VJob jb = P.jobs[j];
        for (unsigned sub = 0; sub < p4v_job_nsub(jb); ++sub) {
          const size_t so = (size_t)sub * jb.kb * P4V_TILE;
          if (jb.flags & P4V_JOB_FIRST) acc = 0.f;
          acc += dot_job<kInt8>(Rcur + jb.r_off + so, Ccur + jb.c_off + so, row, col, jb.kb);
          if (jb.flags & P4V_JOB_LAST) r = fmaf(-P.fix_scale[(size_t)(jb.group + sub) * P.nsg + sg], acc, r);
        }
      }
      if (P.out) { P.out[off] = P.out_residual ? r : -r; continue; }
      for (int j = 0; j < P.n_cand_jobs; ++j) {
        const P4VJob jb = P.jobs[P.n_fixed_jobs + j];
        for (unsigned sub = 0; sub < p4v_job_nsub(jb); ++sub) {
          const size_t so = (size_t)sub * jb.kb * P4V_TILE;
          const unsigned grp = jb.group + sub;
          if (jb.flags & P4V_JOB_FIRST) acc = 0.f;
          const uint8_t* rr = ((jb.flags & P4V_JOB_RCAND) ? Rcand : Rcur) + jb.r_off + so;
          const uint8_t* cc = ((jb.flags & P4V_JOB_CCAND) ? Ccand : Ccur) + jb.c_off + so;
          acc += dot_job<kInt8>(rr, cc, row, col, jb.kb);
          if (jb.flags & P4V_JOB_LAST) {
            const float cb = P.candB[(size_t)grp * P.nsg + sg];
            const float s = ((P.cand_noA_mask >> grp) & 1ull) ? cb : P.candA[(size_t)c * P.nsg + sg] * cb;
            r = fmaf(-s, acc, r);
          }
        }
      }
      const float w = g * r;
      part[row >> 5] = fmaf(w, w, part[row >> 5]);
    }
    if (P.out) continue;
    __syncthreads();
    for (int q = 0; q < 4; ++q) red[q][col][rpar] = part[q];
    __syncthreads();
    if (threadIdx.x < 32) {
      const int q = threadIdx.x >> 3, g8 = threadIdx.x & 7;
      float s = 0.f;
      for (int k = 0; k < 16; ++k) s += red[q][g8 * 16 + k][0] + red[q][g8 * 16 + k][1];
      P.partial[((size_t)tile * P.n_cand + c) * 32 + q * 8 + g8] = s;
    }
  }
}

}  // namespace

int p4v_launch_sweep_simt(const SweepParams& p, cudaStream_t st) {
  const int tiles = p.P * p.tiles_m * p.tiles_n;
  if (tiles < 1 || p.n_cand < 1) return 0;
  const int cpb = 4;
  dim3 grid(tiles, p4v_cdiv(p.n_cand, cpb));
  if (p.is_int8) sweep_simt_kernel<true><<<grid, 256, 0, st>>>(p, cpb);
  else sweep_simt_kernel<false><<<grid, 256, 0, st>>>(p, cpb);
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}
