// Fused frozen attention core on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces, for an attention block whose two MatMul modules were frozen (p4v_matmul_pack), the reference's
//   attn = matmul1(q, k^T) * scale            (ViT / DeiT: utils/models.py:10-26)
//   attn = matmul1(q * scale, k^T) + bias [+ mask]   (Swin: utils/models.py:28-56)
//   out  = matmul2(attn.softmax(-1), v).transpose(1, 2).reshape(B, N, C)
// in one launch.  q, k and v are read in place from the qkv Linear's output [B, N, 3, H, D]; the score matrix lives in
// shared memory only; the output is stored in the [B, N, C] order the proj Linear reads.
//
// A CTA owns one problem p = image * heads + head and 64 query rows.  Both warpgroups share the rows:
//   1. all 256 threads quantise the q tile, every key row and v (transposed in registers, as forward_mm_tc.cu does) into
//      shared memory with the frozen MatMul quantisers (p4v_quant_plain / p4v_quant_sos);
//   2. matmul1: the keys are cut into 64-column chunks, warpgroup w multiplies chunks w, w + 2, ... (m64n64k32 s32.s8.s8;
//      s32 sums are exact, so the K order does not matter).  The epilogue is frozen matmul1's (r = 0;
//      r = fmaf(-scale[h], acc, r); s = -r), then the IEEE operations of the module around it, none contracted:
//      __fmul_rn(s, scale) (ViT), __fadd_rn(s, bias[h][i][j]) and __fadd_rn(., mask[w][i][j]) (Swin).  The FP32 rows go
//      to shared memory (columns XOR-swizzled by row so the fragment stores spread over the banks);
//   3. softmax, one warp per row, as torch's persistent warp softmax computes it for rows of at most 1024 floats: lane l
//      holds the elements it * 32 + l, a per-lane max then an xor-butterfly max, a per-lane sum of expf(x - max) in `it`
//      order then an xor-butterfly add (offsets 16 .. 1), x / sum with IEEE division.  Padding lanes hold -inf (exp 0),
//      and an extra butterfly level over lanes that hold only padding adds +0, so rows shorter than 32 give torch's bits
//      too.  The probabilities are quantised at once into matmul2's A planes (split-of-softmax: high and low part);
//   4. matmul2 on warpgroup 0 (m64n64k32 over the keys; two accumulators for split-of-softmax), frozen matmul2's epilogue
//      in the same group order, stored straight to out[b][i][h * D + d].
// The key axis is padded to 64 (zero key rows and zero v rows: padded probabilities meet zero v bytes), the head
// dimension to 32 for matmul1 and 64 for matmul2 (zero bytes).  Shared memory is a function of the padded key length:
// 112 KiB at 256 keys with split-of-softmax, so two CTAs share an SM.
// The int8 variant (I8, DESIGN §4.14) reads q, k and v as the bytes the qkv Linear's epilogue already quantised with the
// same quantisers (FwdQkv8): step 1 copies the q tile and the keys as 16-byte chunks and transposes v's bytes; steps 2-4
// are the same code.
#include "forward.cuh"
#include "sm90.cuh"
#include <climits>

namespace {

constexpr int kThreads = 256;                 // two warpgroups
constexpr int kRows = 64;                     // query rows of a CTA: the M of one wgmma, shared by both warpgroups

// byte offsets: [q tile | k] (later the probability planes) | v^T | scores
struct AttnLayout { int q, k, p, v, s, total; };
__host__ __device__ inline AttnLayout attn_layout(int sp, int kd, bool sos) {
  AttnLayout L;
  L.q = 0; L.k = kRows * kd; L.p = 0;
  const int qk = L.k + sp * kd, planes = (sos ? 2 : 1) * kRows * sp;
  L.v = ((qk > planes ? qk : planes) + 127) & ~127;
  L.s = L.v + kRows * sp;
  L.total = L.s + kRows * sp * 4;
  return L;
}

template <bool SOS, bool I8>
__global__ void __launch_bounds__(kThreads, 2) forward_attn_kernel(const __grid_constant__ FwdAttnParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const AttnLayout L = attn_layout(P.sp, P.kd, SOS);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int tiles = (P.N + kRows - 1) / kRows;
  const int tm = blockIdx.x % tiles, p = blockIdx.x / tiles;
  const int img = p / P.heads, h = p % P.heads;
  const int row0 = tm * kRows, rows = min(kRows, P.N - row0);
  const float* q = P.qkv + img * P.s_b + h * P.s_h;
  const float* k = q + P.s_p;
  const float* v = q + 2 * P.s_p;

  const float dA1 = __ldg(P.dA1 + h), dB1 = __ldg(P.dB1 + h), dB2 = __ldg(P.dB2 + h);
  const float dA2 = SOS ? 1.f : __ldg(P.dA2 + h);
  const bool fA1 = p4v_rint_div_ok(dA1), fB1 = p4v_rint_div_ok(dB1), fA2 = p4v_rint_div_ok(dA2), fB2 = p4v_rint_div_ok(dB2);
  const float rA1 = fA1 ? __frcp_rn(dA1) : 0.f, rB1 = fB1 ? __frcp_rn(dB1) : 0.f;
  const float rA2 = fA2 ? __frcp_rn(dA2) : 0.f, rB2 = fB2 ? __frcp_rn(dB2) : 0.f;

  uint8_t* sQ = smem + L.q;
  uint8_t* sK = smem + L.k;
  uint8_t* sP = smem + L.p;
  uint8_t* sV = smem + L.v;
  float* sS = reinterpret_cast<float*>(smem + L.s);

  if constexpr (I8) {
    // ---- 1. operands from the planes [3][batch][heads][N][D]: a thread copies one 16-byte chunk of a q or key row, or
    // gathers one column d of a 16-key chunk of v (64 threads read 64 consecutive bytes of a row)
    const long long plane = (long long)P.batch * P.heads * P.N * P.D;
    const uint8_t* q8 = P.planes + ((long long)img * P.heads + h) * P.N * P.D;
    const uint8_t* k8 = q8 + plane;
    const uint8_t* v8 = q8 + 2 * plane;
    const int nc = P.D / 16;
#pragma unroll 1
    for (int u = threadIdx.x; u < (P.kd / 16) * kRows; u += kThreads) {
      const int c = u / kRows, r = u % kRows;
      *reinterpret_cast<uint4*>(sQ + (c * kRows + r) * 16) =
          (r < rows && c < nc) ? __ldg(reinterpret_cast<const uint4*>(q8 + (long long)(row0 + r) * P.D) + c) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll 1
    for (int u = threadIdx.x; u < (P.kd / 16) * P.sp; u += kThreads) {
      const int c = u / P.sp, n = u % P.sp;
      *reinterpret_cast<uint4*>(sK + (c * P.sp + n) * 16) =
          (n < P.N && c < nc) ? __ldg(reinterpret_cast<const uint4*>(k8 + (long long)n * P.D) + c) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll 1
    for (int u = threadIdx.x; u < 4 * P.sp; u += kThreads) {
      const int d = u % 64, kb = 16 * (u / 64);
      uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int e = 0; e < 16; ++e)
        if (d < P.D && kb + e < P.N) w[e >> 2] |= (uint32_t)__ldg(v8 + (long long)(kb + e) * P.D + d) << ((e & 3) * 8);
      *reinterpret_cast<uint4*>(sV + (kb / 16 * 64 + d) * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  } else {
    // ---- 1. operands: lanes along d for q and k (a warp reads whole 128-byte row segments), v transposed in registers
#pragma unroll 1
    for (int j = 0; j < P.kd / 32; ++j) {
      const int d = lane + 32 * j;
      float x[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = warp + 8 * i;
        x[i] = (r < rows && d < P.D) ? __ldg(q + (long long)(row0 + r) * P.s_n + d) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = warp + 8 * i;
        const float xs = P.scale_on_q ? __fmul_rn(x[i], P.scale) : x[i];
        sQ[((d >> 4) * kRows + r) * 16 + (d & 15)] =
            (uint8_t)((r < rows && d < P.D) ? p4v_qbyte(p4v_quant_plain(xs, dA1, fA1, rA1, false, 0.f, P.A1_lo, P.A1_hi)) : 0u);
      }
    }
#pragma unroll 1
    for (int pass = 0; pass < (P.sp / 64) * (P.kd / 32); ++pass) {
      const int j = pass % (P.kd / 32), n0 = 64 * (pass / (P.kd / 32));
      const int d = lane + 32 * j;
      float x[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int n = n0 + warp + 8 * i;
        x[i] = (n < P.N && d < P.D) ? __ldg(k + (long long)n * P.s_n + d) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int n = n0 + warp + 8 * i;
        sK[((d >> 4) * P.sp + n) * 16 + (d & 15)] =
            (uint8_t)((n < P.N && d < P.D) ? p4v_qbyte(p4v_quant_plain(x[i], dB1, fB1, rB1, false, 0.f, P.B1_lo, P.B1_hi)) : 0u);
      }
    }
#pragma unroll 1
    for (int u = threadIdx.x; u < 4 * P.sp; u += kThreads) {     // one thread = one column d x one 16-key chunk
      const int d = u % 64, kb = 16 * (u / 64);
      float x[16];
#pragma unroll
      for (int e = 0; e < 16; ++e)
        x[e] = (d < P.D && kb + e < P.N) ? __ldg(v + (long long)(kb + e) * P.s_n + d) : 0.f;
      uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int e = 0; e < 16; ++e)
        if (d < P.D && kb + e < P.N) w[e >> 2] |= p4v_qbyte(p4v_quant_plain(x[e], dB2, fB2, rB2, false, 0.f, P.B2_lo, P.B2_hi)) << ((e & 3) * 8);
      *reinterpret_cast<uint4*>(sV + (kb / 16 * 64 + d) * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
  fence_proxy_async();   // generic-proxy stores -> wgmma (async proxy) reads
  __syncthreads();

  // ---- 2. matmul1 and the module's operations on the scores
  const uint32_t base = smem_u32(smem);
  const float s1 = __ldg(P.scale1 + h);
  const int wrow = (warp & 3) * 16;             // this warp's 16 rows of the warpgroup's 64
#pragma unroll 1
  for (int c = wg; c < P.sp / 64; c += 2) {
    uint32_t acc[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) acc[e] = 0u;
    wg_fence();
#pragma unroll 1
    for (int ks = 0; ks < P.kd / 32; ++ks)
      wgmma_n64_k32(acc, make_desc(base + L.q + ks * 2 * kRows * 16, kRows),
                    make_desc(base + L.k + (c * 64 + ks * 2 * P.sp) * 16, P.sp), 1u);
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < 32; ++e) {
      const int r = wrow + (lane >> 2) + 8 * ((e >> 1) & 1), j = c * 64 + 8 * (e >> 2) + 2 * (lane & 3) + (e & 1);
      if (r < rows && j < P.N) {
        const int i = row0 + r;
        float s = p4v_attn_mm1(acc[e], s1);
        if (!P.scale_on_q) s = __fmul_rn(s, P.scale);
        if (P.bias) s = __fadd_rn(s, __ldg(P.bias + ((long long)h * P.N + i) * P.N + j));
        if (P.mask) s = __fadd_rn(s, __ldg(P.mask + ((long long)(img % P.n_windows) * P.N + i) * P.N + j));
        sS[r * P.sp + (j ^ ((r & 7) << 3))] = s;
      }
    }
  }
  __syncthreads();            // scores complete; every wgmma reading q and k has retired: the planes may overwrite them

  // ---- 3. softmax (torch's persistent warp softmax) and matmul2's A planes
  const float split = SOS ? __ldg(P.split2) : 0.f;
  const int plane = kRows * P.sp;
#pragma unroll 1
  for (int r = warp; r < rows; r += 8) {
    const int swz = (r & 7) << 3;
    float x[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int j = it * 32 + lane;
      x[it] = j < P.N ? sS[r * P.sp + (j ^ swz)] : __int_as_float(0xff800000);   // -inf
    }
    float m = x[0];
#pragma unroll
    for (int it = 1; it < 8; ++it) m = (m > x[it]) ? m : x[it];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float o = __shfl_xor_sync(0xffffffffu, m, off);
      m = (m < o) ? o : m;
    }
    float sum = 0.f;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      x[it] = it * 32 + lane < P.N ? expf(__fsub_rn(x[it], m)) : 0.f;
      sum = __fadd_rn(sum, x[it]);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, off));
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int j = it * 32 + lane;
      if (j < P.sp) {
        const bool in = j < P.N;
        const float pr = __fdiv_rn(x[it], sum);
        uint8_t* dst = sP + ((j >> 4) * kRows + r) * 16 + (j & 15);
        if (SOS) {
          dst[0] = (uint8_t)(in ? p4v_qbyte(p4v_quant_sos(pr, split, P.qm1, 1)) : 0u);
          dst[plane] = (uint8_t)(in ? p4v_qbyte(p4v_quant_sos(pr, split, P.qm1, 2)) : 0u);
        } else {
          dst[0] = (uint8_t)(in ? p4v_qbyte(p4v_quant_plain(pr, dA2, fA2, rA2, false, 0.f, P.A2_lo, P.A2_hi)) : 0u);
        }
      }
    }
  }
  fence_proxy_async();
  __syncthreads();
  if (wg != 0) return;

  // ---- 4. matmul2 and its epilogue, stored in the proj input's [B, N, C] order
  uint32_t acc0[32], acc1[SOS ? 32 : 1];
#pragma unroll
  for (int e = 0; e < 32; ++e) { acc0[e] = 0u; if (SOS) acc1[e] = 0u; }
  wg_fence();
#pragma unroll 1
  for (int ks = 0; ks < P.sp / 32; ++ks) {
    const uint64_t db = make_desc(base + L.v + ks * 2 * 64 * 16, 64);
    wgmma_n64_k32(acc0, make_desc(base + L.p + ks * 2 * kRows * 16, kRows), db, 1u);
    if constexpr (SOS) wgmma_n64_k32(acc1, make_desc(base + L.p + plane + ks * 2 * kRows * 16, kRows), db, 1u);
  }
  wg_commit();
  wg_wait0();
  const float t0 = __ldg(P.scale2 + h), t1 = SOS ? __ldg(P.scale2 + P.heads + h) : 0.f;
  const long long C = (long long)P.heads * P.D;
#pragma unroll
  for (int e = 0; e < 32; e += 2) {
    const int r = wrow + (lane >> 2) + 8 * ((e >> 1) & 1), col = 8 * (e >> 2) + 2 * (lane & 3);
    if (r >= rows || col >= P.D) continue;
    float o[2];
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      o[f] = p4v_attn_mm2<SOS>(acc0[e + f], SOS ? acc1[e + f] : 0u, t0, t1);
    }
    *reinterpret_cast<float2*>(P.out + ((long long)img * P.N + row0 + r) * C + (long long)h * P.D + col) = make_float2(o[0], o[1]);
  }
}

template <bool SOS, bool I8>
int launch(const FwdAttnParams& p_in, cudaStream_t st) {
  FwdAttnParams p = p_in;
  p.sp = (p.N + 63) / 64 * 64;
  p.kd = (p.D + 31) / 32 * 32;
  const int smem = (int)p4v_attn_smem_bytes(p.sp, p.kd, SOS);
  const long long ctas = (long long)p.batch * p.heads * p4v_cdiv(p.N, kRows);
  P4V_REQUIRE(ctas <= INT_MAX, "attention_frozen_forward: grid too large (%lld tiles)", ctas);
  P4V_CUDA_OK(cudaFuncSetAttribute(forward_attn_kernel<SOS, I8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  forward_attn_kernel<SOS, I8><<<(unsigned)ctas, kThreads, smem, st>>>(p);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace

size_t p4v_attn_smem_bytes(int sp, int kd, bool sos) { return (size_t)attn_layout(sp, kd, sos).total + 128; }

int p4v_launch_forward_attn_tc(const FwdAttnParams& p, bool sos, cudaStream_t st, bool i8) {
  if (i8) return sos ? launch<true, true>(p, st) : launch<false, true>(p, st);
  return sos ? launch<true, false>(p, st) : launch<false, false>(p, st);
}
