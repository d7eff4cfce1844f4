// Shared device/host declarations for the PTQ4ViT scale-factor search on sm_90a (H100).
//
// Data model (see DESIGN.md):
//   * "operand image": a quantised matrix [rows][K] stored tile-wise in the wgmma
//     no-swizzle K-major canonical layout so that one contiguous bulk copy (TMA 1-D,
//     cp.async.bulk) lands a ready-to-multiply tile in shared memory:
//         image[tile][chunk][128 rows][16 bytes]      (chunk = 16 bytes of K)
//     K is cut into "segments" (intersection of the weight column blocks and the
//     activation chunks, each padded to a multiple of 32 bytes) -- inside one
//     segment both step sizes are constant, so the integer accumulation is exact.
//   * "job": one <=128-byte-per-row slice of a segment = one shared-memory stage =
//     up to 4 wgmma K-steps.  Consecutive jobs of a segment accumulate into
//     one register accumulator ("group"); the epilogue consumes one accumulator at a time.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define P4V_TILE 128           // rows per operand tile == 2 x wgmma M == wgmma N
#define P4V_JOB_KB 128         // max bytes of K per row and job
#define P4V_MAX_JOBS 320
#define P4V_MAX_GROUPS 96
#define P4V_MAX_CAND 128
#define P4V_CG 16              // columns per scale / score group
#define P4V_TILE_CG (P4V_TILE / P4V_CG)   // 8

enum : uint8_t {
  P4V_JOB_FIRST  = 1,   // first job of an accumulator group
  P4V_JOB_LAST   = 2,   // last job of an accumulator group
  P4V_JOB_RCAND  = 4,   // row operand comes from the candidate plane
  P4V_JOB_CCAND  = 8,   // column operand comes from the candidate plane
  P4V_JOB_RRES   = 16,  // row operand is candidate independent: loaded once per tile fragment (resident), not per job
  P4V_JOB_CRES   = 32,  // column operand comes from the tile's resident copy of the current column image
};

struct __align__(16) P4VJob {
  uint32_t r_off;      // byte offset inside the row-operand tile image
  uint32_t c_off;      // byte offset inside the column-operand tile image
  uint8_t  kb;         // bytes of K per row and per sub-accumulator (multiple of 32; kb * nsub <= P4V_JOB_KB)
  uint8_t  nsub;       // 0/1: one accumulator (FIRST/LAST chain rules apply); n > 1: the stage holds n consecutive K slabs,
                       //      each its own accumulator (groups group .. group+n-1), operand offsets advance by kb*128 bytes
  uint8_t  flags;
  uint8_t  group;      // accumulator group index (row of the scale table) of the first sub-accumulator
  uint32_t res_off;    // byte offset inside the resident row-operand buffer (P4V_JOB_RRES)
};

// score-group mapping of the 16-column groups (used by the sweep for scales and by
// the reduction for the argmax groups)
enum { P4V_SG_COLUMN = 0,   // scale group = global 16-column group index (Linear)
       P4V_SG_PROBLEM = 1   // scale group = problem % nsg (head-wise MatMul)
};

struct SweepParams {
  const uint8_t* R_cur;  const uint8_t* R_cand;
  const uint8_t* C_cur;  const uint8_t* C_cand;
  unsigned long long R_tile_bytes, C_tile_bytes;            // 128 * padded K bytes (current planes)
  unsigned long long R_cand_tile_bytes, C_cand_tile_bytes;  // same for the candidate planes
  unsigned long long R_cand_stride, C_cand_stride;          // bytes between candidate planes
  int P, M, N, tiles_m, tiles_n;
  const float* Y; const float* Gr; const float* bias;   // bias may be null
  const float* gscale;                                  // device scalar: power-of-two gradient scale
  long long ld, prob_stride;
  const P4VJob* jobs;       // [n_fixed_jobs] then [n_cand_jobs]
  int n_fixed_jobs, n_cand_jobs, n_fixed_groups, n_cand_groups;
  const float* fix_scale;   // [n_fixed_groups][nsg]
  const float* candA;       // [n_cand][nsg]
  const float* candB;       // [n_cand_groups][nsg]
  int nsg, sg_mode;
  unsigned long long cand_noA_mask;   // bit g set: candidate group g ignores candA (scale = candB only)
  int n_cand;
  float* partial;           // [tiles_total][n_cand][4][8]
  float* out;               // if non-null: no candidates; write bias + sum(scale*acc) of the fixed groups (quant_forward)
  int out_residual;         // with out: write y - bias - sum(scale*acc) instead (the current residual e)
  int order;                // 0: tile_m fastest, 1: tile_n fastest
  int is_int8;
  int R_shared;             // the row operand does not depend on the problem index (conv: kernel planes shared by all images)
  int row_keys;             // single-segment steps: one score per ROW, partial = [tile][candidate][column half][128 rows]
  // shared-memory plan, filled by the launcher
  unsigned int stage_r_bytes, stage_c_bytes, n_stages, resident_bytes, resident_bufs, cres_bytes;
  const float* res = nullptr;   // with out (not out_residual): out = fl(forward + res), res [M][N] like out (kModeFwdRes)
};

static inline __host__ __device__ int p4v_cdiv(int a, int b) { return (a + b - 1) / b; }
static inline __host__ __device__ unsigned p4v_job_nsub(const P4VJob& j) { return j.nsub ? j.nsub : 1u; }
static inline __host__ __device__ unsigned p4v_job_bytes(const P4VJob& j) { return (unsigned)j.kb * p4v_job_nsub(j) * P4V_TILE; }   // per operand

#ifdef __CUDACC__
// ---- exact rounding division shared by the operand-image and the Gram kernels ----
// rintf(__fdiv_rn(v, delta)) without the general-purpose division: rcp must be __frcp_rn(delta).
// q1 = q0 + (v - delta*q0)*rcp differs from the correctly rounded quotient by at most one ulp, so rint(q1) equals
// rint(v/delta) unless q1 lies within a few ulps of a half-integer; those (one in ~10^4) and non-finite values
// take the exact division.  Only valid for 2^-100 < |delta| < 2^100 (p4v_rint_div_ok, checked once per step size).
__device__ __forceinline__ float p4v_rint_div(float v, float delta, float rcp) {
  const float q0 = v * rcp;
  const float q1 = fmaf(fmaf(-delta, q0, v), rcp, q0);
  const float n = rintf(q1);
  const float aq = fabsf(q1);
  const float dist = fabsf(fabsf(q1 - n) - 0.5f);
  if (!(aq <= 3.0e38f) || dist <= aq * 4.8e-7f) return rintf(__fdiv_rn(v, delta));
  return n;
}

__device__ __forceinline__ bool p4v_rint_div_ok(float delta) { const float ad = fabsf(delta); return ad > 7.9e-31f && ad < 1.2e30f; }

// One element of a plain operand image: clamp(rne(v / delta), lo, hi); fast / rcp = p4v_rint_div_ok(delta) /
// __frcp_rn(delta).  by_rcp: the step size is one the reference holds as a Python scalar, divided by as v * (1/delta)
// (rcp_scalar = __fdiv_rn(1, delta); see quant_image_kernel).  Shared by the operand-image kernel and the fused forward,
// whose integers must be the same.
__device__ __forceinline__ float p4v_quant_plain(float v, float delta, bool fast, float rcp, bool by_rcp, float rcp_scalar,
                                                 float lo, float hi) {
  if (by_rcp) return fminf(fmaxf(rintf(v * rcp_scalar), lo), hi);
  return fminf(fmaxf(fast ? p4v_rint_div(v, delta, rcp) : rintf(__fdiv_rn(v, delta)), lo), hi);
}

// One element of a split-of-softmax operand image (matmul.py:595-598): part 1 (high) = rne(clamp(v, split, 1) * qm1),
// part 2 (low) = rne(clamp(v, 0, split) / (split / qm1)), both clamped to [0, qm1].  Shared by the operand-image kernel
// and the fused MatMul forward, whose integers must be the same.
__device__ __forceinline__ float p4v_quant_sos(float v, float split, float qm1, int part) {
  if (part == 1) return fminf(fmaxf(rintf(fminf(fmaxf(v, split), 1.f) * qm1), 0.f), qm1);
  return fminf(fmaxf(rintf(__fdiv_rn(fminf(fmaxf(v, 0.f), split), __fdiv_rn(split, qm1))), 0.f), qm1);
}

// The export quantiser of a weight element (export.cu mode 0, utils/integer.py:15-17): clamp(rne(x / delta), -q, q-1)
// with q = 2^(bit-1).  Shared by the export and the frozen convolution's pack, whose integers must be the same.
__device__ __forceinline__ float p4v_quant_export(float x, float delta, float q) {
  return fminf(fmaxf(rintf(__fdiv_rn(x, delta)), -q), q - 1.f);
}

// The int8 operand byte of a quantised value q (p4v_quant_plain / p4v_quant_sos): the integer's low byte.  NaN (0/0)
// cannot be represented in the integer operand and becomes 0.
__device__ __forceinline__ uint32_t p4v_qbyte(float q) {
  if (!(q == q)) q = 0.f;
  return (uint32_t)((int)q & 0xff);
}

#endif

// ---- error plumbing (host) --------------------------------------------------
#ifdef __cplusplus
extern "C" void p4v_set_error(const char* fmt, ...);
#endif
#define P4V_CUDA_OK(expr)                                                            \
  do { cudaError_t _e = (expr);                                                      \
       if (_e != cudaSuccess) { p4v_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
                                return 2; } } while (0)
#define P4V_REQUIRE(cond, ...)                                                       \
  do { if (!(cond)) { p4v_set_error(__VA_ARGS__); return 1; } } while (0)

// ---- kernel launchers shared between translation units ----------------------
// What p4v_launch_sweep_tc decided for one launch (p4v_profile_collect_launches reports it).
struct P4VLaunchDecision {
  int mode;                       // consumer mode: 0 multi-segment, 1 single, 2 pair
  int n_stages, resident_bufs;    // shared-memory ring stages, resident row-operand buffers
  unsigned int resident_bytes;    // resident row operand of the tile (P4V_JOB_RRES jobs), 0 if streamed
  unsigned int cres_bytes;        // resident column image of the tile (P4V_JOB_CRES jobs), 0 if streamed
  int grid;                       // CTAs launched
};
int p4v_launch_sweep_tc(const SweepParams& p, const P4VJob* host_jobs, int num_sms, cudaStream_t st,
                        P4VLaunchDecision* decision = nullptr);
int p4v_launch_sweep_simt(const SweepParams& p, cudaStream_t st);

// ---- library runtime (runtime.cu) -------------------------------------------
void p4v_count_launch();                   // every kernel launch, for p4v_launch_count
int p4v_num_sms();
bool p4v_prof_on();                        // live kernel timing of the tensor-core launches (p4v_profile_enable)
void p4v_prof_begin(cudaStream_t st, cudaEvent_t* e0);
void p4v_prof_end(cudaStream_t st, cudaEvent_t e0, int kind, double ops);
// one slab sweep on the kernel `kernel` selects (P4V_KERNEL_*): counted and, while timing is on, timed
int p4v_run_sweep(const SweepParams& sp, const P4VJob* host_jobs, int kernel, cudaStream_t st);
