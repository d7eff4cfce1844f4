// C-ABI for the channel-wise weight search of the patch-embedding convolution
// (ChannelwiseBatchingQuantConv2d with a_bit >= 32, reference quant_layers/conv.py:444-614, as wired by
// configs/PTQ4ViT.py:52-54): per output channel o the step size f_c * delta0[o] minimising
//     sum_images mean_positions ( g * (y - b - conv(x, fq(w, f_c * delta0))) )^2          (conv.py:526-557)
// The convolution is a product over the im2col matrix: for image p
//     D_p[o, l] = sum_k q_c[o, k] * cols_p[l, k] ,   yhat = b[o] + f_c * delta0[o] * D_p[o, l]
// rows = output channels (row operand: candidate planes of the integer kernel, shared by all images), columns = output
// positions (column operand: the FP32 im2col matrix split exactly into three bf16 terms -- the activations are not
// quantised), one accumulator per candidate, three term products chained into it.  The per-channel step size would be a
// per-ROW scale; the sweep's scales are per column group, so delta0[o] is folded into the targets once:
//     (g * (y - b - f*d0*D))^2 = (g*d0 * ((y - b)/d0 - f*D))^2
// and the candidate scale is the plain factor f_c.  Scores are kept per row (SweepParams::row_keys).
//
// Layer-wise mode (desc.layerwise = 1: BatchingEasyQuantConv2d with a_bit >= 32, conv.py:279-441, as wired by
// configs/BasePTQ.py:48-50): one step size for the whole kernel.  It is the channel-wise search with every row given the
// same delta0 = max|W| / (qmax - 0.5) (conv.py:313): one block over the kernel, the same planes, prescale, sweep and
// per-row sums; only the selection differs, summing the O per-channel keys of a candidate into one score
//     score_c = -sum_images mean_positions mean_channels (g * (y - yhat_c))^2                 (conv.py:387-394)
#include "../../include/ptq4vit_b200.h"
#include "plan.cuh"
#include <climits>

#define P4V_XSTR(x) #x
#define P4V_STR(x) P4V_XSTR(x)

namespace {

struct ConvPlan {
  p4v_conv_desc d;
  int P, O, K, L, tiles_o, tiles_l, kb, w_qmax;
  int n_d;             // step sizes searched: O (channel-wise) or 1 (layer-wise)
  Table<P4VJob> jobs; Table<P4VSeg> segW, segC; Table<float> factors;
  Image Wcand, Cimg;   // candidate planes of the integer kernel; the three-term split of the im2col matrix
  size_t o_keys, o_d0, o_d, o_gscale, o_ones, o_scores, o_best, o_candA, o_candB, o_fix, o_partial, o_Y, o_G, total;
};

int build_plan(const p4v_conv_desc* d, ConvPlan& p) {
  P4V_REQUIRE(d != nullptr, "null desc");
  p.d = *d;
  p.P = d->images; p.O = d->out_channels; p.K = d->K; p.L = d->positions;
  P4V_REQUIRE(p.P > 0 && p.O > 0 && p.K > 0 && p.L > 0, "conv: empty shape");
  P4V_REQUIRE(d->w_bit >= 2 && d->w_bit <= 8, "conv: w_bit must be in [2,8]");
  P4V_REQUIRE(d->eq_n >= 1 && d->eq_n <= P4V_MAX_CAND, "conv: eq_n must be in [1,%d]", P4V_MAX_CAND);
  P4V_REQUIRE(d->kernel == P4V_KERNEL_TCGEN05, "conv: the channel-wise search runs on the tensor-core kernel only");
  P4V_REQUIRE(d->layerwise == 0 || d->layerwise == 1, "conv: layerwise must be 0 or 1 (got %d)", d->layerwise);
  p.n_d = d->layerwise ? 1 : p.O;
  p.w_qmax = 1 << (d->w_bit - 1);
  p.tiles_o = p4v_cdiv(p.O, P4V_TILE); p.tiles_l = p4v_cdiv(p.L, P4V_TILE);
  p.kb = (int)align_up((size_t)p.K * 2, 32);                    // bf16 row bytes of one term
  P4V_REQUIRE(3 * (p.kb / 32) <= P4V_MAX_JOBS * 4 && 3 * p4v_cdiv(p.kb, P4V_JOB_KB) <= P4V_MAX_JOBS, "conv: kernel volume too large");
  p.segW.host = {P4VSeg{0, p.K, 0, 0, 0.f, (float)-p.w_qmax, (float)(p.w_qmax - 1), 0, 0.f, 0, 0}};
  for (int t = 0; t < 3; ++t) p.segC.host.push_back(P4VSeg{0, p.K, t * p.kb * P4V_TILE, 0, 0.f, 0.f, 0.f, 0, 0.f, t + 1, 0});
  p.factors.host = cand_factors(d->eq_n, d->eq_alpha, d->eq_beta);
  int n_jobs = 0;   // one accumulator: the three term products chained
  for (int t = 0; t < 3; ++t) add_group(p.jobs.host, 0, t * p.kb, p.kb, P4V_JOB_RCAND, 0, t == 0, t == 2, n_jobs);
  p.Wcand = Image{0, p.kb, p.tiles_o, 1, d->eq_n, false}; p.Cimg = Image{0, 3 * p.kb, p.tiles_l, p.P, 1, false};
  Carver c{0};
  const int n_c = d->eq_n;
  p.factors.off = c.take(p.factors.bytes()); p.o_keys = c.take((p.n_d + 1) * 4);
  p.o_d0 = c.take(p.n_d * 4); p.o_d = c.take(p.n_d * 4); p.o_gscale = c.take(4); p.o_ones = c.take(4);
  p.o_scores = c.take((size_t)n_c * p.O * 8); p.o_best = c.take(p.n_d * 4);
  p.o_candA = c.take((size_t)n_c * 4); p.o_candB = c.take(4); p.o_fix = c.take(4);
  p.jobs.off = c.take(p.jobs.bytes()); p.segW.off = c.take(p.segW.bytes()); p.segC.off = c.take(p.segC.bytes());
  p.o_partial = c.take((size_t)p.P * p.tiles_o * p.tiles_l * n_c * 256 * 4);
  p.Wcand.off = c.take(p.Wcand.bytes());
  p.Cimg.off = c.take(p.Cimg.bytes());
  p.o_Y = c.take((size_t)p.P * p.O * p.L * 4); p.o_G = c.take((size_t)p.P * p.O * p.L * 4);
  p.total = c.end;
  return 0;
}

// y' = (y - b[o]) / d0[o * d_stride] ,  g' = g * d0[o * d_stride]      ([P][O][L], one thread per element; d_stride 0:
// one step size for every channel)
__global__ void conv_prescale_kernel(const float* __restrict__ y, const float* __restrict__ g, const float* __restrict__ bias,
                                     const float* __restrict__ d0, int d_stride, int O, int L, long long n, float* __restrict__ yo,
                                     float* __restrict__ go) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)((i / L) % O);
    const float d = d0[o * d_stride];
    yo[i] = __fdiv_rn(y[i] - (bias ? bias[o] : 0.f), d);
    go[i] = g[i] * d;
  }
}

// sums[c][o] = sum over images, position tiles and column halves of the per-row partials (fixed order, fp64)
__global__ void conv_reduce_kernel(const float* __restrict__ partial, int P, int tiles_o, int tiles_l, int n_cand, int O, double* sums) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_cand * O) return;
  const int c = idx / O, o = idx % O;
  const int to = o / P4V_TILE, r = o % P4V_TILE;
  double acc = 0.0;
  for (int p = 0; p < P; ++p)
    for (int tl = 0; tl < tiles_l; ++tl) {
      // tile index of the sweep: order 0 -> t = tn * tiles_m + tm inside a problem
      const size_t tile = (size_t)p * tiles_o * tiles_l + (size_t)tl * tiles_o + to;
      const float* base = partial + (tile * n_cand + c) * 256;          // [column half][128 rows]
      acc += (double)base[r] + (double)base[128 + r];
    }
  sums[(size_t)c * O + o] = acc;
}

__global__ void conv_fill_kernel(float* candA, const float* factors, int n, float* ones) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) candA[i] = factors[i];
  if (i == 0) ones[0] = 1.f;
}

}  // namespace

extern "C" int p4v_conv_workspace_bytes(const p4v_conv_desc* d, size_t* bytes) {
  ConvPlan p; int rc = build_plan(d, p);
  if (rc) return rc;
  P4V_REQUIRE(bytes != nullptr, "null output");
  *bytes = p.total;
  return 0;
}

extern "C" int p4v_conv_calibrate(const p4v_conv_desc* d, const float* cols, const float* weight, const float* bias,
                                  const float* raw_out, const float* raw_grad, void* ws, size_t workspace_bytes,
                                  float* w_interval, float* score_log, void* stream) {
  ConvPlan p; int rc = build_plan(d, p);
  if (rc) return rc;
  P4V_REQUIRE(cols && weight && raw_out && raw_grad && ws && w_interval, "conv_calibrate: null pointer");
  P4V_REQUIRE(!d->has_bias || bias, "conv_calibrate: has_bias set but bias is null");
  P4V_REQUIRE(workspace_bytes >= p.total, "conv_calibrate: workspace too small (%zu < %zu)", workspace_bytes, p.total);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = p.factors.upload(ws, st)) || (rc = p.jobs.upload(ws, st)) || (rc = p.segW.upload(ws, st)) ||
      (rc = p.segC.upload(ws, st))) return rc;
  // min-max step size per output channel (conv.py:487) or of the whole kernel (conv.py:313), and the gradient scale
  const int rows_per_d = p.O / p.n_d;
  int* keys = at<int>(ws, p.o_keys);
  if ((rc = p4v_keys_reset(keys, p.n_d + 1, st))) return rc;
  if ((rc = p4v_block_max(weight, p.K, p.O, rows_per_d, p.n_d, p.K, 1, 1, keys, st))) return rc;
  if ((rc = p4v_group_absmax(raw_grad, (long long)p.P * p.O * p.L, 1, 1, keys + p.n_d, st))) return rc;
  if ((rc = p4v_keys_to_delta(keys, p.n_d, (float)p.w_qmax - 0.5f, at<float>(ws, p.o_d0), at<float>(ws, p.o_d), st))) return rc;
  if ((rc = p4v_make_gscale(keys + p.n_d, at<float>(ws, p.o_gscale), st))) return rc;
  conv_fill_kernel<<<p4v_cdiv(d->eq_n, 128), 128, 0, st>>>(at<float>(ws, p.o_candA), p.factors.dev(ws), d->eq_n, at<float>(ws, p.o_candB));
  p4v_count_launch();
  const long long n = (long long)p.P * p.O * p.L;
  conv_prescale_kernel<<<132 * 8, 256, 0, st>>>(raw_out, raw_grad, d->has_bias ? bias : nullptr, at<float>(ws, p.o_d0),
                                                 p.n_d == 1 ? 0 : 1, p.O, p.L, n, at<float>(ws, p.o_Y), at<float>(ws, p.o_G));
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  {   // candidate planes of the integer kernel: rows = channels, one step size per row (per kernel when layer-wise)
    QuantImageArgs q{};
    p.Wcand.fill(q, ws);
    q.src = weight; q.ld = p.K; q.prob_stride = 0; q.src_transposed = 0; q.rows = p.O;
    q.factors = p.factors.dev(ws); q.delta = at<float>(ws, p.o_d0);
    q.rows_per_block = rows_per_d; q.d_stride = 1; q.d_mod = 1; q.segs = p.segW.dev(ws); q.nseg = 1;
    if ((rc = p4v_quant_image(q, st))) return rc;
  }
  {   // exact three-term bf16 split of the FP32 im2col matrix: rows = output positions
    QuantImageArgs q{};
    p.Cimg.fill(q, ws);
    q.src = cols; q.ld = p.K; q.prob_stride = (long long)p.L * p.K; q.src_transposed = 0; q.rows = p.L;
    q.factors = nullptr; q.delta = at<float>(ws, p.o_d0); q.rows_per_block = 0; q.d_stride = 0; q.d_mod = 1;
    q.segs = p.segC.dev(ws); q.nseg = 3;
    if ((rc = p4v_quant_image(q, st))) return rc;
  }
  SweepParams sp{};
  fill_images(sp, ws, p.Wcand, p.Wcand, p.Cimg, p.Cimg);
  sp.R_shared = 1;                                          // the kernel planes do not depend on the image
  sp.P = p.P; sp.M = p.O; sp.N = p.L; sp.tiles_m = p.tiles_o; sp.tiles_n = p.tiles_l;
  sp.Y = at<float>(ws, p.o_Y); sp.Gr = at<float>(ws, p.o_G); sp.bias = nullptr;
  sp.ld = p.L; sp.prob_stride = (long long)p.O * p.L;
  sp.gscale = at<float>(ws, p.o_gscale);
  sp.jobs = p.jobs.dev(ws);
  sp.n_fixed_jobs = 0; sp.n_cand_jobs = (int)p.jobs.host.size(); sp.n_fixed_groups = 0; sp.n_cand_groups = 1;
  sp.fix_scale = at<float>(ws, p.o_fix); sp.candA = at<float>(ws, p.o_candA); sp.candB = at<float>(ws, p.o_candB);
  sp.nsg = 1; sp.sg_mode = P4V_SG_PROBLEM;                  // one scale group: the candidate factor
  sp.n_cand = d->eq_n; sp.partial = at<float>(ws, p.o_partial); sp.order = 0;
  sp.row_keys = 1;
  if ((rc = p4v_run_sweep(sp, p.jobs.host.data(), d->kernel, st))) return rc;
  conv_reduce_kernel<<<p4v_cdiv(d->eq_n * p.O, 256), 256, 0, st>>>(sp.partial, p.P, p.tiles_o, p.tiles_l, d->eq_n, p.O, at<double>(ws, p.o_scores));
  p4v_count_launch();
  P4V_CUDA_OK(cudaGetLastError());
  SelectArgs f{};
  f.sums = at<double>(ws, p.o_scores); f.n_cand = d->eq_n; f.n_keys = p.O; f.n_groups = p.n_d; f.keys_per_group = rows_per_d;
  // mean over the output positions, sum over the images (conv.py:548-549); layer-wise also the mean over the channels
  // (conv.py:387-389): the O per-channel sums of a candidate are added in a fixed order into its one score
  f.inv_count = 1.0 / ((double)rows_per_d * (double)p.L);
  f.gscale = at<float>(ws, p.o_gscale); f.factors = p.factors.dev(ws);
  f.d0 = at<float>(ws, p.o_d0); f.d = at<float>(ws, p.o_d); f.d_stride = 1; f.d_col = 0;
  f.best = at<int>(ws, p.o_best); f.score_log = score_log; f.has_next = 0;
  if ((rc = p4v_select_step(f, st))) return rc;
  P4V_CUDA_OK(cudaMemcpyAsync(w_interval, at<float>(ws, p.o_d), (size_t)p.n_d * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// ---- frozen patch-embedding convolution: integer weights packed once, forward on csrc/forward_conv_tc.cu -----------
namespace {

// The shape rule on the module's geometry (images, height and width are the forward's): nullptr when it qualifies, else
// the reason.
const char* conv_frozen_reason(const p4v_conv_frozen_desc* d) {
  if (d->in_channels < 1 || d->out_channels < 1 || d->kernel_h < 1 || d->kernel_w < 1) return "empty channel or kernel dimension";
  if (d->out_channels > P4V_CONV_MAX_O) return "out_channels above " P4V_STR(P4V_CONV_MAX_O);
  if ((long long)d->in_channels * d->kernel_h * d->kernel_w > P4V_CONV_MAX_K) return "K = in_channels * kh * kw above " P4V_STR(P4V_CONV_MAX_K);
  if (d->w_bit < 2 || d->w_bit > 8) return "w_bit must be in [2,8] (bf16 holds the integers exactly)";
  if ((d->layerwise != 0 && d->layerwise != 1) || (d->has_bias != 0 && d->has_bias != 1)) return "layerwise and has_bias must be 0 or 1";
  return nullptr;
}

struct ConvFrozen { int O, K, tiles_n, n_slabs; size_t delta_bytes, total; };

int build_conv_frozen(const p4v_conv_frozen_desc* d, ConvFrozen& f, const char* who) {
  P4V_REQUIRE(d != nullptr, "%s: null desc", who);
  const char* why = conv_frozen_reason(d);
  P4V_REQUIRE(why == nullptr, "%s: %s", who, why);
  f.O = d->out_channels; f.K = d->in_channels * d->kernel_h * d->kernel_w;
  f.tiles_n = p4v_cdiv(f.O, P4V_TILE); f.n_slabs = p4v_cdiv(f.K, P4V_CONV_SLAB);
  f.delta_bytes = p4v_conv_delta_bytes(f.O);
  f.total = f.delta_bytes + (size_t)f.tiles_n * f.n_slabs * p4v_conv_slab_bytes();
  return 0;
}

}  // namespace

extern "C" int p4v_conv_frozen_ok(const p4v_conv_frozen_desc* d, int* ok) {
  P4V_REQUIRE(d && ok, "conv_frozen_ok: null pointer");
  *ok = conv_frozen_reason(d) == nullptr;
  return 0;
}

extern "C" int p4v_conv_pack_bytes(const p4v_conv_frozen_desc* d, size_t* bytes) {
  ConvFrozen f; int rc = build_conv_frozen(d, f, "conv_pack_bytes");
  if (rc) return rc;
  P4V_REQUIRE(bytes != nullptr, "conv_pack_bytes: null output");
  *bytes = f.total;
  return 0;
}

extern "C" int p4v_conv_pack(const p4v_conv_frozen_desc* d, const float* weight, const float* w_interval, void* packed,
                             size_t packed_bytes, void* stream) {
  ConvFrozen f; int rc = build_conv_frozen(d, f, "conv_pack");
  if (rc) return rc;
  P4V_REQUIRE(weight && w_interval && packed, "conv_pack: null pointer");
  P4V_REQUIRE(packed_bytes >= f.total, "conv_pack: packed buffer too small (%zu < %zu)", packed_bytes, f.total);
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 15) == 0, "conv_pack: packed must be 16-byte aligned");
  uint8_t* base = static_cast<uint8_t*>(packed);
  return p4v_launch_conv_pack(weight, w_interval, d->layerwise, f.O, f.K, d->w_bit, f.tiles_n, f.n_slabs,
                              reinterpret_cast<float*>(base), base + f.delta_bytes, (cudaStream_t)stream);
}

namespace {

// Validates the arguments every frozen forward shares (in p4v_conv_frozen_forward's order, with fn's name in the
// messages) and fills the kernel's parameters
int conv_forward_params(const char* fn, const p4v_conv_frozen_desc* d, const float* x, const float* bias, const void* packed,
                        size_t packed_bytes, float* out, FwdConvParams& p) {
  ConvFrozen f; int rc = build_conv_frozen(d, f, fn);
  if (rc) return rc;
  P4V_REQUIRE(x && packed && out, "%s: null pointer", fn);
  P4V_REQUIRE(!d->has_bias || bias, "%s: has_bias set but bias is null", fn);
  P4V_REQUIRE(d->images >= 1 && d->height >= d->kernel_h && d->width >= d->kernel_w,
              "%s: bad geometry (images %d, input %dx%d, kernel %dx%d): need at least one image and one "
              "output position", fn, d->images, d->height, d->width, d->kernel_h, d->kernel_w);
  const long long chw = (long long)d->in_channels * d->height * d->width;
  const int Ph = d->height / d->kernel_h, Pw = d->width / d->kernel_w;
  const long long M = (long long)d->images * Ph * Pw;
  P4V_REQUIRE(chw <= INT_MAX && M <= INT_MAX - P4V_TILE && (long long)p4v_cdiv((int)M, P4V_TILE) * f.tiles_n <= INT_MAX,
              "%s: input too large (in_channels*height*width %lld, positions %lld)", fn, chw, M);
  P4V_REQUIRE(packed_bytes >= f.total, "%s: packed buffer too small (%zu < %zu)", fn, packed_bytes, f.total);
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 15) == 0 && (reinterpret_cast<uintptr_t>(x) & 3) == 0 &&
              (reinterpret_cast<uintptr_t>(out) & 3) == 0 && (reinterpret_cast<uintptr_t>(bias) & 3) == 0,
              "%s: packed must be 16-byte, x, bias and out 4-byte aligned", fn);
  p = FwdConvParams{};
  p.x = x; p.bias = d->has_bias ? bias : nullptr; p.out = out;
  p.delta = static_cast<const float*>(packed);
  p.Wq = static_cast<const uint8_t*>(packed) + f.delta_bytes;
  p.B = d->images; p.C = d->in_channels; p.H = d->height; p.W = d->width; p.O = f.O; p.kh = d->kernel_h; p.kw = d->kernel_w;
  p.Ph = Ph; p.Pw = Pw; p.K = f.K; p.M = (int)M;
  p.tiles_m = p4v_cdiv(p.M, P4V_TILE); p.tiles_n = f.tiles_n; p.n_slabs = f.n_slabs;
  return 0;
}

// The token epilogues' rule beyond the shape rule: nullptr when d qualifies, else the reason (norm: the LayerNorm's)
const char* conv_stem_reason(const p4v_conv_frozen_desc* d, bool norm) {
  if (const char* why = conv_frozen_reason(d)) return why;
  if (d->out_channels % 4 != 0) return "out_channels must be a multiple of 4 (a lane stores 4 channels of a token row)";
  if (norm && d->out_channels > P4V_TILE) return "out_channels above " P4V_STR(P4V_TILE) " (the LayerNorm needs the whole token row in one CTA)";
  return nullptr;
}

bool apart(const void* a, size_t abytes, const void* b, size_t bbytes) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return !a || !b || x + abytes <= y || y + bbytes <= x;
}

// The arguments of a token-major call (fn, rule `norm`) beyond conv_forward_params: the rule, out 16-byte aligned and
// apart from x, bias and packed; `tokens` token rows of out_channels per image
int check_tokens(const char* fn, const p4v_conv_frozen_desc* d, bool norm, const FwdConvParams& p, const void* packed,
                 size_t packed_bytes, const float* out, long long tokens) {
  const char* why = conv_stem_reason(d, norm);
  P4V_REQUIRE(why == nullptr, "%s: %s (%s)", fn, why, norm ? "p4v_conv_norm_ok" : "p4v_conv_pos_ok");
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "%s: out must be 16-byte aligned", fn);
  const size_t ob = (size_t)p.B * tokens * p.O * 4;
  P4V_REQUIRE(apart(out, ob, p.x, (size_t)p.B * p.C * p.H * p.W * 4) && apart(out, ob, p.bias, (size_t)p.O * 4) &&
              apart(out, ob, packed, packed_bytes), "%s: out overlaps x, bias or packed", fn);
  return 0;
}

}  // namespace

extern "C" int p4v_conv_frozen_forward(const p4v_conv_frozen_desc* d, const float* x, const float* bias, const void* packed,
                                       size_t packed_bytes, float* out, void* stream) {
  FwdConvParams p;
  if (int rc = conv_forward_params("conv_frozen_forward", d, x, bias, packed, packed_bytes, out, p)) return rc;
  return p4v_launch_forward_conv_tc(p, (cudaStream_t)stream);
}

extern "C" int p4v_conv_pos_ok(const p4v_conv_frozen_desc* d, int* ok) {
  P4V_REQUIRE(d && ok, "conv_pos_ok: null pointer");
  *ok = conv_stem_reason(d, false) == nullptr;
  return 0;
}

extern "C" int p4v_conv_norm_ok(const p4v_conv_frozen_desc* d, int* ok) {
  P4V_REQUIRE(d && ok, "conv_norm_ok: null pointer");
  *ok = conv_stem_reason(d, true) == nullptr;
  return 0;
}

// Replaces, with the conv frozen, VisionTransformer.forward's stem (reference: timm's VisionTransformer.forward_features,
// as utils/models.py:164 restates it):
//   x = patch_embed(x)                                  (proj(x).flatten(2).transpose(1, 2))
//   x = torch.cat((cls_token.expand(B, -1, -1), x), dim=1) + pos_embed
extern "C" int p4v_conv_frozen_forward_pos(const p4v_conv_frozen_desc* d, const float* x, const float* bias, const void* packed,
                                           size_t packed_bytes, const float* cls, size_t cls_numel, const float* pos,
                                           size_t pos_numel, float* out, void* stream) {
  const char* fn = "conv_frozen_forward_pos";
  FwdConvPosParams p;
  if (int rc = conv_forward_params(fn, d, x, bias, packed, packed_bytes, out, p)) return rc;
  P4V_REQUIRE(cls && pos, "%s: null pointer", fn);
  const long long tokens = 1 + (long long)p.Ph * p.Pw;
  P4V_REQUIRE(cls_numel == (size_t)p.O, "%s: cls has %zu elements, out_channels is %d", fn, cls_numel, p.O);
  P4V_REQUIRE(pos_numel == (size_t)(tokens * p.O), "%s: pos_embed has %zu elements, (1 + positions) * out_channels is %lld", fn,
              pos_numel, tokens * p.O);
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(cls) & 15) == 0 && (reinterpret_cast<uintptr_t>(pos) & 15) == 0,
              "%s: cls and pos_embed must be 16-byte aligned", fn);
  if (int rc = check_tokens(fn, d, false, p, packed, packed_bytes, out, tokens)) return rc;
  const size_t ob = (size_t)p.B * tokens * p.O * 4;
  P4V_REQUIRE(apart(out, ob, cls, cls_numel * 4) && apart(out, ob, pos, pos_numel * 4), "%s: out overlaps cls or pos_embed", fn);
  p.cls = cls; p.pos = pos;
  return p4v_launch_forward_conv_tc(p, (cudaStream_t)stream);
}

// Replaces, with the conv frozen, SwinTransformer.forward's stem (reference: timm's SwinTransformer.forward_features, as
// utils/models.py:390 restates it):  x = patch_norm(patch_embed(x))
extern "C" int p4v_conv_frozen_forward_norm(const p4v_conv_frozen_desc* d, const float* x, const float* bias, const void* packed,
                                            size_t packed_bytes, const float* gamma, const float* beta, size_t norm_numel,
                                            float eps, float* out, void* stream) {
  const char* fn = "conv_frozen_forward_norm";
  FwdConvNormParams p;
  if (int rc = conv_forward_params(fn, d, x, bias, packed, packed_bytes, out, p)) return rc;
  P4V_REQUIRE(gamma && beta, "%s: null pointer", fn);
  P4V_REQUIRE(norm_numel == (size_t)p.O, "%s: the LayerNorm has %zu features, out_channels is %d", fn, norm_numel, p.O);
  P4V_REQUIRE((reinterpret_cast<uintptr_t>(gamma) & 15) == 0 && (reinterpret_cast<uintptr_t>(beta) & 15) == 0,
              "%s: gamma and beta must be 16-byte aligned", fn);
  P4V_REQUIRE(eps >= 0.f && eps <= 3.4028234663852886e38f, "%s: eps must be finite and non-negative (got %g)", fn, (double)eps);
  const long long tokens = (long long)p.Ph * p.Pw;
  if (int rc = check_tokens(fn, d, true, p, packed, packed_bytes, out, tokens)) return rc;
  const size_t ob = (size_t)p.B * tokens * p.O * 4;
  P4V_REQUIRE(apart(out, ob, gamma, norm_numel * 4) && apart(out, ob, beta, norm_numel * 4), "%s: out overlaps gamma or beta", fn);
  p.ln = FwdNorm{gamma, beta, eps};
  return p4v_launch_forward_conv_tc(p, (cudaStream_t)stream);
}
