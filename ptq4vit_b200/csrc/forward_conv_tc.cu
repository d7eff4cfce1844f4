// Forward of a frozen patch-embedding convolution on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces, for a module whose weight was packed once (p4v_conv_pack), the reference's
//   out = F.conv2d(x, fl(q * delta), bias, stride = kernel)        (quant_layers/conv.py:53-62, :69-74, a_bit >= 32)
// with one launch and no im2col matrix in HBM: each CTA gathers the patches of its output positions straight from the
// image into shared memory.  The sum is the conv search's product (conv_api.cu): the FP32 pixels split exactly into
// three bf16 terms, times the integer weights as bf16 (exact for w_bit <= 8), the three term products chained into one
// fp32 accumulator; the step size is applied once per output, out = fmaf(delta[o], S, bias[o]).
//
// A CTA owns one output tile: 128 positions (rows; two warpgroups of 64) x 128 output channels (columns), column tiles
// fastest so that the CTAs sharing a row tile's pixels run together and read them again from L2.  All 256 threads walk
// K = C * kh * kw in slabs of 32 elements through two shared-memory stages:
//   1. gather and split slab s + 1 into the free stage while the wgmma of slab s (m64n128k16 bf16, two k16 steps per
//      term, terms high, middle, low) runs on the other one; the slab's 8 KB of the packed weight image is copied beside
//      it with 16-byte loads; fence.proxy.async, then one block barrier hands the stage to the async proxy;
//   2. epilogue: the fp32 accumulators go through shared memory as [channel][position], so that each warp stores runs of
//      consecutive positions of one channel (the NCHW output is contiguous along the positions).  The token-major
//      epilogues (FwdConvPosParams, FwdConvNormParams; DESIGN §4.13) stage them as [position][channel] instead: a warp
//      takes one position at a time and its lanes store a float4 of 4 consecutive channels each, a run of the token row,
//      with pos_embed added (ViT) or the row normalised with torch's LayerNorm (Swin, the whole row in this CTA).
// Gather: a thread owns one position (lanes along consecutive positions) and one 8-element K chunk per unit.  A position's
// pixels of element k sit at pos_base + koff[k] (koff: c*H*W + i*W + j, a per-CTA table in shared memory), so the
// thread's 8 values are two float4 loads when kw and W are multiples of 4 and x is 16-byte aligned (one kernel row holds
// each group of 4), else 8 scalar loads.  For kernel == stride, consecutive positions of a patch row read consecutive
// runs of kw floats of the same image rows: the warp's loads cover whole image-row segments.
#include "forward.cuh"
#include "sm90.cuh"
#include <climits>

namespace {

constexpr int kThreads = 256;
constexpr int kSlab = P4V_CONV_SLAB;                 // bf16 elements of K per row and stage
constexpr int kChunks = kSlab / 8;                   // 16-byte K chunks per row and stage
constexpr int kPlane = P4V_TILE * kSlab * 2;         // one term plane of the pixel slab: [4 chunks][128 rows][16 B]
constexpr int kStage = 3 * kPlane + kPlane;          // three term planes, then the weight slab (same shape)
constexpr int kLdOut = P4V_TILE + 4;                 // staged output row (one channel): 4 mod 32 words, no bank conflict
constexpr int kOutBytes = P4V_TILE * kLdOut * 4;
constexpr int kMainBytes = (2 * kStage > kOutBytes ? 2 * kStage : kOutBytes);
constexpr int kUnits = P4V_TILE * kChunks / kThreads;   // (position, chunk) units per thread and slab
static_assert(kUnits * kThreads == P4V_TILE * kChunks, "units must cover the slab");
static_assert(kPlane % (16 * kThreads) == 0, "the weight slab is copied in whole 16-byte rounds");
// token-major staging: row = position, 8 mod 32 words, so that a half-warp's float2 stores (4 rows x 8 columns) and a
// warp's float4 reads of one row hit distinct banks
constexpr int kLdTok = P4V_TILE + 8;
constexpr int kTokBytes = P4V_TILE * kLdTok * 4;

template <class Par> constexpr bool kIsNchw = std::is_same<Par, FwdConvParams>::value;
template <class Par> __host__ __device__ constexpr int main_bytes() {
  return kIsNchw<Par> ? kMainBytes : (2 * kStage > kTokBytes ? 2 * kStage : kTokBytes);
}
template <class Par> __host__ __device__ constexpr int smem_bytes(int K) { return main_bytes<Par>() + ((K * 4 + 127) & ~127) + 128; }

__device__ __forceinline__ uint32_t bf16_pair(float a, float b) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(a)) | ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(b)) << 16);
}

// The token-major epilogue (DESIGN §4.13): stage the tile as [position][channel] (the stages are free), then each warp
// takes positions warp, warp + 8, ... and its lane l the channels o0 + 4l .. + 3 of the position's token row.  The value
// is the NCHW epilogue's, fmaf(delta[o], S, bias[o]) (delta[o] * S without a bias); ViT adds pos_embed's row and writes
// the image's cls row along with its position 0, Swin normalises the row with torch's exact LayerNorm (the §4.10 fold's
// p4v_ln_row_stats_at over the staged row and p4v_ln_apply).  O % 4 == 0: a lane's four channels are all in or all out.
template <class Par>
__device__ __forceinline__ void token_epilogue(const Par& P, float* stg, const float (&acc)[64], int r0, int tm, int tn,
                                               int warp, int lane) {
#pragma unroll
  for (int v = 0; v < 64; v += 2) {
    const int row = r0 + 8 * ((v >> 1) & 1), col = 8 * (v >> 2) + 2 * (lane & 3);
    *reinterpret_cast<float2*>(stg + row * kLdTok + col) = make_float2(acc[v], acc[v + 1]);
  }
  __syncthreads();
  const int L = P.Ph * P.Pw;
  const int o = tn * P4V_TILE + 4 * lane;
  const bool col_in = o < P.O;
  float4 d = make_float4(0.f, 0.f, 0.f, 0.f), bo = d, ga = d, be = d, head = d;
  if (col_in) {
    d = __ldg(reinterpret_cast<const float4*>(P.delta + o));
    if (P.bias) bo = make_float4(__ldg(P.bias + o), __ldg(P.bias + o + 1), __ldg(P.bias + o + 2), __ldg(P.bias + o + 3));
    if constexpr (kIsConvNorm<Par>) {
      ga = __ldg(reinterpret_cast<const float4*>(P.ln.gamma + o));
      be = __ldg(reinterpret_cast<const float4*>(P.ln.beta + o));
    } else {   // the cls row: fl(cls + pos_embed[0])
      const float4 c = __ldg(reinterpret_cast<const float4*>(P.cls + o)), p0 = __ldg(reinterpret_cast<const float4*>(P.pos + o));
      head = make_float4(__fadd_rn(c.x, p0.x), __fadd_rn(c.y, p0.y), __fadd_rn(c.z, p0.z), __fadd_rn(c.w, p0.w));
    }
  }
  auto conv_out = [&](float dd, float a, float b) { return P.bias ? fmaf(dd, a, b) : __fmul_rn(dd, a); };
#pragma unroll 1
  for (int r = warp; r < P4V_TILE; r += kThreads / 32) {
    const int g = tm * P4V_TILE + r;
    if (g >= P.M) break;                       // warp-uniform: the LayerNorm's shuffles see the whole warp
    const int b = g / L, l = g - b * L;
    float* row = stg + r * kLdTok;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (col_in) {
      const float4 a = *reinterpret_cast<const float4*>(row + 4 * lane);
      v = make_float4(conv_out(d.x, a.x, bo.x), conv_out(d.y, a.y, bo.y), conv_out(d.z, a.z, bo.z), conv_out(d.w, a.w, bo.w));
    }
    if constexpr (kIsConvNorm<Par>) {
      if (col_in) *reinterpret_cast<float4*>(row + 4 * lane) = v;
      __syncwarp();
      const float4* row4 = reinterpret_cast<const float4*>(row);
      float mean, rstd;
      p4v_ln_row_stats_at([row4](int i) { return row4[i]; }, P.O, P.ln.eps, lane, mean, rstd);
      if (col_in)
        *reinterpret_cast<float4*>(P.out + (long long)g * P.O + o) =
            make_float4(p4v_ln_apply(v.x, mean, rstd, ga.x, be.x), p4v_ln_apply(v.y, mean, rstd, ga.y, be.y),
                        p4v_ln_apply(v.z, mean, rstd, ga.z, be.z), p4v_ln_apply(v.w, mean, rstd, ga.w, be.w));
    } else if (col_in) {
      const long long t = (long long)g + b + 1;   // token row: the image's cls row, then its positions
      const float4 pe = __ldg(reinterpret_cast<const float4*>(P.pos + (long long)(l + 1) * P.O + o));
      *reinterpret_cast<float4*>(P.out + t * P.O + o) =
          make_float4(__fadd_rn(v.x, pe.x), __fadd_rn(v.y, pe.y), __fadd_rn(v.z, pe.z), __fadd_rn(v.w, pe.w));
      if (l == 0) *reinterpret_cast<float4*>(P.out + (t - 1) * P.O + o) = head;
    }
  }
}

// Two CTAs per SM: 128 registers, 2 x ~70-84 KB of shared memory.
template <class Par>
__global__ void __launch_bounds__(kThreads, 2) forward_conv_kernel(const __grid_constant__ Par P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  int* koff = reinterpret_cast<int*>(smem + main_bytes<Par>());
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int tn = blockIdx.x % P.tiles_n, tm = blockIdx.x / P.tiles_n;
  const int L = P.Ph * P.Pw;
  const int khw = P.kh * P.kw;
  const long long HW = (long long)P.H * P.W;

  // the offset of element k = (c, i, j) from its position's first pixel (fits int: K <= 4096 and the API bounds C*H*W)
  for (int k = threadIdx.x; k < P.K; k += kThreads) {
    const int c = k / khw, r = k - c * khw, i = r / P.kw;
    koff[k] = (int)(c * HW + (long long)i * P.W + (r - i * P.kw));
  }

  // this thread's position (row of the tile) and the offset of its first pixel
  const int m = threadIdx.x & (P4V_TILE - 1);
  const int gm = tm * P4V_TILE + m;
  const bool row_in = gm < P.M;
  long long pos_base = 0;
  if (row_in) {
    const int b = gm / L, l = gm - b * L, py = l / P.Pw, px = l - py * P.Pw;
    pos_base = (long long)b * P.C * HW + (long long)py * P.kh * P.W + (long long)px * P.kw;
  }
  const float* xp = P.x + pos_base;
  const bool vec = (P.kw & 3) == 0 && (P.W & 3) == 0 && (reinterpret_cast<uintptr_t>(P.x) & 15) == 0;
  const uint4* wsrc = reinterpret_cast<const uint4*>(P.Wq + (size_t)tn * P.n_slabs * kPlane);
  __syncthreads();                             // koff visible

  // gather, split and store K slab s into stage `buf`; elements outside the problem are 0
  auto load_slab = [&](int s, int buf) {
    uint8_t* st = smem + buf * kStage;
    float v[kUnits][8];
#pragma unroll
    for (int u = 0; u < kUnits; ++u) {
      const int k0 = s * kSlab + 8 * ((threadIdx.x >> 7) + 2 * u);
      if (vec) {
#pragma unroll
        for (int g = 0; g < 2; ++g) {        // K is a multiple of 4: a group of 4 is all in or all out
          const int k = k0 + 4 * g;
          float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
          if (row_in && k < P.K) f = __ldg(reinterpret_cast<const float4*>(xp + koff[k]));
          v[u][4 * g] = f.x; v[u][4 * g + 1] = f.y; v[u][4 * g + 2] = f.z; v[u][4 * g + 3] = f.w;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[u][e] = (row_in && k0 + e < P.K) ? __ldg(xp + koff[k0 + e]) : 0.f;
      }
    }
    uint4 w[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) w[r] = __ldg(wsrc + (size_t)s * (kPlane / 16) + threadIdx.x + r * kThreads);
#pragma unroll
    for (int u = 0; u < kUnits; ++u) {
      const int ch = (threadIdx.x >> 7) + 2 * u;
      uint32_t t1[4], t2[4], t3[4];
#pragma unroll
      for (int e = 0; e < 8; e += 2) {       // the exact split of quant_image_kernel's split3 mode (prep.cu)
        float h[2], mi[2], lo[2];
#pragma unroll
        for (int z = 0; z < 2; ++z) {
          const float x = v[u][e + z];
          h[z] = __bfloat162float(__float2bfloat16_rn(x));
          mi[z] = __bfloat162float(__float2bfloat16_rn(x - h[z]));
          lo[z] = (x - h[z]) - mi[z];
        }
        t1[e >> 1] = bf16_pair(h[0], h[1]); t2[e >> 1] = bf16_pair(mi[0], mi[1]); t3[e >> 1] = bf16_pair(lo[0], lo[1]);
      }
      uint8_t* dst = st + (ch * P4V_TILE + m) * 16;
      *reinterpret_cast<uint4*>(dst) = make_uint4(t1[0], t1[1], t1[2], t1[3]);
      *reinterpret_cast<uint4*>(dst + kPlane) = make_uint4(t2[0], t2[1], t2[2], t2[3]);
      *reinterpret_cast<uint4*>(dst + 2 * kPlane) = make_uint4(t3[0], t3[1], t3[2], t3[3]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) reinterpret_cast<uint4*>(st + 3 * kPlane)[threadIdx.x + r * kThreads] = w[r];
  };

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  load_slab(0, 0);
  fence_proxy_async();                         // generic-proxy stores -> wgmma (async proxy) reads
  __syncthreads();
  const uint32_t base = smem_u32(smem);
  for (int s = 0; s < P.n_slabs; ++s) {
    const uint32_t st = base + (s & 1) * kStage;
    const uint32_t sa = st + wg * 64 * 16, sb = st + 3 * kPlane;
    wg_fence();
#pragma unroll
    for (int k = 0; k < 2; ++k)                // +16 bf16 of K = 2 chunks of 128 rows x 16 B
#pragma unroll
      for (int t = 0; t < 3; ++t)
        wgmma_k32(acc, make_desc(sa + t * kPlane + k * 2 * P4V_TILE * 16, P4V_TILE), make_desc(sb + k * 2 * P4V_TILE * 16, P4V_TILE), 1u);
    wg_commit();
    if (s + 1 < P.n_slabs) load_slab(s + 1, (s + 1) & 1);   // under the MMAs of slab s
    wg_wait0();
    fence_proxy_async();
    __syncthreads();                           // slab s + 1 visible; every warpgroup is done with stage s & 1
  }

  float* stg = reinterpret_cast<float*>(smem);
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  if constexpr (!kIsNchw<Par>) {
    token_epilogue(P, stg, acc, r0, tm, tn, warp, lane);
  } else {
    // ---- epilogue: stage [channel][position] (the stages are free), then runs of positions per channel ----
#pragma unroll
    for (int v = 0; v < 64; ++v) {
      const int row = r0 + 8 * ((v >> 1) & 1), col = 8 * (v >> 2) + 2 * (lane & 3) + (v & 1);
      stg[col * kLdOut + row] = acc[v];
    }
    __syncthreads();
    long long obase[P4V_TILE / 32];              // out offset of position lane + 32 i without the channel term, -1 outside
#pragma unroll
    for (int i = 0; i < P4V_TILE / 32; ++i) {
      const int g = tm * P4V_TILE + lane + 32 * i;
      obase[i] = -1;
      if (g < P.M) { const int b = g / L; obase[i] = (long long)b * P.O * L + (g - b * L); }
    }
    const int o0 = tn * P4V_TILE;
#pragma unroll 1
    for (int c = warp; c < P4V_TILE; c += kThreads / 32) {
      const int o = o0 + c;
      if (o >= P.O) break;
      const float d = __ldg(P.delta + o);
      const float bo = P.bias ? __ldg(P.bias + o) : 0.f;
#pragma unroll
      for (int i = 0; i < P4V_TILE / 32; ++i) {
        if (obase[i] < 0) continue;
        const float a = stg[c * kLdOut + lane + 32 * i];
        P.out[obase[i] + (long long)o * L] = P.bias ? fmaf(d, a, bo) : __fmul_rn(d, a);
      }
    }
  }
}

// q image of the packed blob: unit u = ((tile * n_slabs + slab) * 4 + chunk) * 128 + row holds channel tile*128 + row,
// K elements slab*32 + chunk*8 .. +7 as bf16 of the export's integer (a zero is +0, as the int8 export has no -0);
// channels >= O and elements >= K are 0.  delta[o] = w_interval[o] (one step size repeated when layer-wise); the table's
// padding up to n_delta entries is 0, so equal integers and step sizes give equal bytes.
__global__ void conv_pack_kernel(const float* __restrict__ w, const float* __restrict__ wi, int layerwise, int O, int K,
                                 float qmax, int n_slabs, long long n_units, int n_delta, float* __restrict__ delta,
                                 uint4* __restrict__ Wq) {
  for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < n_units; u += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(u % P4V_TILE);
    const long long rest = u / P4V_TILE;
    const int chunk = (int)(rest % kChunks);
    const long long ts = rest / kChunks;
    const int slab = (int)(ts % n_slabs), tile = (int)(ts / n_slabs);
    const int o = tile * P4V_TILE + row, k0 = slab * kSlab + chunk * 8;
    uint32_t q[4] = {0u, 0u, 0u, 0u};
    if (slab == 0 && chunk == 0 && o >= O && o < n_delta) delta[o] = 0.f;
    if (o < O) {
      const float d = wi[layerwise ? 0 : o];
      if (slab == 0 && chunk == 0) delta[o] = d;
      float e8[8];
#pragma unroll
      for (int e = 0; e < 8; ++e)
        e8[e] = k0 + e < K ? __int2float_rn((int)p4v_quant_export(w[(long long)o * K + k0 + e], d, qmax)) : 0.f;
#pragma unroll
      for (int e = 0; e < 8; e += 2) q[e >> 1] = bf16_pair(e8[e], e8[e + 1]);
    }
    Wq[u] = make_uint4(q[0], q[1], q[2], q[3]);
  }
}

}  // namespace

template <class Par> int p4v_launch_forward_conv_tc(const Par& p, cudaStream_t st) {
  const int smem = smem_bytes<Par>(p.K);
  P4V_CUDA_OK(cudaFuncSetAttribute(forward_conv_kernel<Par>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  forward_conv_kernel<Par><<<(unsigned)(p.tiles_m * p.tiles_n), kThreads, smem, st>>>(p);
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}
template int p4v_launch_forward_conv_tc<FwdConvParams>(const FwdConvParams&, cudaStream_t);
template int p4v_launch_forward_conv_tc<FwdConvPosParams>(const FwdConvPosParams&, cudaStream_t);
template int p4v_launch_forward_conv_tc<FwdConvNormParams>(const FwdConvNormParams&, cudaStream_t);

int p4v_launch_conv_pack(const float* weight, const float* w_interval, int layerwise, int O, int K, int w_bit, int tiles_n,
                         int n_slabs, float* delta, uint8_t* Wq, cudaStream_t st) {
  const long long n_units = (long long)tiles_n * n_slabs * kChunks * P4V_TILE;
  long long blocks = (n_units + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  conv_pack_kernel<<<(int)blocks, 256, 0, st>>>(weight, w_interval, layerwise, O, K, (float)(1 << (w_bit - 1)), n_slabs, n_units,
                                                (int)(p4v_conv_delta_bytes(O) / 4), delta, reinterpret_cast<uint4*>(Wq));
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  return 0;
}
