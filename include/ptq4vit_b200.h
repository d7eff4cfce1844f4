/* ptq4vit_b200 -- C ABI of the H100-native (sm_90a) PTQ4ViT scale-factor search.
 *
 * Drop-in boundary (SURVEY.md section 8b): the reference has no FFI; its operator
 * surface for this path is the Python classes in quant_layers/{linear,matmul}.py.
 * A maintainer binds these entry points with ctypes from those classes (see
 * INTEGRATION.md); each function names the reference method it replaces.
 *
 * Conventions: every pointer is a DEVICE pointer unless stated, fp32, row-major,
 * owned by the caller; nothing is allocated or freed by the library; work is
 * enqueued on `stream` (a cudaStream_t passed as void*) and the call returns
 * without synchronising.  Return value: 0 = ok, non-zero = error (message via
 * p4v_last_error()).  No exceptions cross the boundary.
 */
#ifndef PTQ4VIT_B200_H
#define PTQ4VIT_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define P4V_API __attribute__((visibility("default")))
#else
#define P4V_API
#endif

#define P4V_OPERAND_AUTO 0
#define P4V_OPERAND_INT8 1 /* wgmma .s8.s8, s32 accumulators                     */
#define P4V_OPERAND_BF16 2 /* integer-valued bf16, wgmma .bf16, exact f32 accum. */
#define P4V_KERNEL_TCGEN05 0 /* the tensor-core (wgmma) sweep; the name is historical */
#define P4V_KERNEL_SIMT 1 /* plain-CUDA cross-check kernel (bring-up / odd shapes) */

/* One wrapped Linear: mirrors the constructor of PTQSLQuantLinear /
 * PTQSLBatchingQuantLinear / PostGeluPTQSLBatchingQuantLinear
 * (quant_layers/linear.py:98-122, :350-363, :562-574). */
typedef struct p4v_linear_desc {
  int32_t rows;      /* M = images * tokens (all leading dims of x flattened)            */
  int32_t tokens;    /* tokens per image: rows / images (the reference means over them)  */
  int32_t in_features, out_features;
  int32_t n_V, n_H, n_a;
  int32_t w_bit, a_bit;
  int32_t eq_n;
  int32_t search_round;
  double eq_alpha, eq_beta; /* python floats in the reference: keep double */
  int32_t post_gelu; /* 1: twin-uniform activation quantizer (linear.py:557-642)         */
  int32_t has_bias;
  int32_t operand;   /* P4V_OPERAND_*  */
  int32_t kernel;    /* P4V_KERNEL_*   */
  int32_t init_layerwise; /* 1: every block starts from the layer-wise min-max step size (linear.py:382-383, :393-394) */
  int32_t rows_per_chunk; /* 0: search the whole layer at once.  > 0: a multiple of 128, at most rows: the search builds
                           * its row-dependent operand images (activations) for one chunk of rows at a time and adds the
                           * chunks' scores; the workspace holds one chunk (the reference's calib_batch_size batching,
                           * linear.py:365-378, :458-492). */
} p4v_linear_desc;

/* bytes of device workspace p4v_linear_* needs for this layer */
P4V_API int p4v_linear_workspace_bytes(const p4v_linear_desc* d, size_t* bytes);

/* number of floats of the optional score log: one [eq_n x groups] table per search
 * step in the reference's call order (W steps: groups = n_V, X steps: groups = 1). */
P4V_API int p4v_linear_score_log_floats(const p4v_linear_desc* d, size_t* n);

/* Replaces PTQSLBatchingQuantLinear.calibration_step2() (linear.py:536-555):
 *   _initialize_intervals (:380-397 / :576-599), candidate tables (:544-545),
 *   search_round x { _search_best_w_interval (:455-495), _search_best_a_interval
 *   (:497-533 / :609-642) }.
 * in : x [rows,in], weight [out,in], bias [out] or NULL, raw_out [rows,out], raw_grad [rows,out]
 * out: w_interval [n_V*n_H] (reference shape n_V,1,n_H,1), a_interval [n_a] (n_a,1),
 *      score_log (NULL or p4v_linear_score_log_floats floats).
 * With d->rows_per_chunk > 0 every search step loops over the row chunks: it quantises the chunk's activations (current
 * image, and the candidate planes in an activation step), sweeps them and adds the chunk's partial scores into the fp64
 * score table; the pick follows the last chunk.  The initial step sizes and the gradient scale are taken over all rows
 * first, so the result equals the unchunked search up to the order of the fp64 score sums.  The step-wise surface below
 * (begin / search_w / search_a) takes whole layers only. */
P4V_API int p4v_linear_calibrate(const p4v_linear_desc* d, const float* x, const float* weight, const float* bias,
                         const float* raw_out, const float* raw_grad, void* workspace, size_t workspace_bytes,
                         float* w_interval, float* a_interval, float* score_log, void* stream);

/* Step-wise surface (same workspace must be passed; begin() must come first):
 *   p4v_linear_begin      ~ _initialize_intervals + candidate tables
 *   p4v_linear_search_w   ~ _search_best_w_interval  (column blocks [h_begin,h_end))
 *   p4v_linear_search_a   ~ _search_best_a_interval  (activation chunks [a_begin,a_end))
 *   p4v_linear_intervals  -> copies the current step sizes out                          */
P4V_API int p4v_linear_begin(const p4v_linear_desc* d, const float* x, const float* weight, const float* bias,
                     const float* raw_out, const float* raw_grad, void* workspace, size_t workspace_bytes, void* stream);
P4V_API int p4v_linear_search_w(const p4v_linear_desc* d, const float* bias, const float* raw_out, const float* raw_grad,
                        void* workspace, int32_t h_begin, int32_t h_end, float* score_log, void* stream);
P4V_API int p4v_linear_search_a(const p4v_linear_desc* d, const float* bias, const float* raw_out, const float* raw_grad,
                        void* workspace, int32_t a_begin, int32_t a_end, float* score_log, void* stream);
P4V_API int p4v_linear_intervals(const p4v_linear_desc* d, void* workspace, float* w_interval, float* a_interval, void* stream);

/* Replaces quant_forward (linear.py:62-67 with quant_weight_bias :152-162 and
 * quant_input :164-169 / :601-607): out = fq(x) fq(W)^T + bias on the tensor cores. */
P4V_API int p4v_linear_quant_forward_workspace_bytes(const p4v_linear_desc* d, size_t* bytes);
P4V_API int p4v_linear_quant_forward(const p4v_linear_desc* d, const float* x, const float* weight, const float* bias,
                             const float* w_interval, const float* a_interval, void* workspace, size_t workspace_bytes,
                             float* out, void* stream);

/* Frozen Linear layer: the integer weights of a calibrated layer packed once, and a forward that reads no FP32 weight.
 * Replaces, per call of quant_forward (linear.py:62-67), the re-quantisation of the weight (quant_weight_bias, :46-55 /
 * :152-162) and the separate activation pass (quant_input, :57-60 / :164-169 / :601-607): the output is bit-identical to
 * p4v_linear_quant_forward with the same step sizes.
 * `packed` (p4v_linear_pack_bytes bytes, independent of d->rows; 256-byte aligned) holds what does not depend on the
 * batch: the int8 weight operand image (the layout the forward step uses with P4V_OPERAND_INT8: 128-row tiles, K-major
 * 16-byte chunks, segments padded to 32 B), the scale table step_W[v,h] * step_X[a] (post-GELU: also step_W[v,h] * the
 * constant negative-part step) per (segment group, 16-column group), the activation step sizes and the job and segment
 * tables of the forward step.  p4v_linear_pack may copy small tables from the host; p4v_linear_frozen_forward enqueues
 * kernels only -- no allocation, no host-to-device copy, no synchronisation -- so it can be captured in a CUDA graph.
 * p4v_linear_frozen_path: 1 = one fused kernel quantises each 128-row tile of x into shared memory and multiplies it
 * there (workspace 0 bytes); 0 = the quantised tile does not fit shared memory beside a two-stage weight ring (ViT-B
 * fc2: K = 3072, two parts): the activations are quantised into an int8 image in `workspace` and multiplied by the
 * sweep kernel.  A pure function of the descriptor without its rows. */
P4V_API int p4v_linear_pack_bytes(const p4v_linear_desc* d, size_t* bytes);
P4V_API int p4v_linear_pack(const p4v_linear_desc* d, const float* weight, const float* w_interval, const float* a_interval,
                    void* packed, size_t packed_bytes, void* stream);
P4V_API int p4v_linear_frozen_path(const p4v_linear_desc* d, int* path);
P4V_API int p4v_linear_frozen_workspace_bytes(const p4v_linear_desc* d, size_t* bytes);
P4V_API int p4v_linear_frozen_forward(const p4v_linear_desc* d, const float* x, const float* bias, const void* packed,
                              void* workspace, size_t workspace_bytes, float* out, void* stream);

/* One wrapped MatMul (head-wise groups, n_V = n_H = 1 per operand, as forced by
 * PTQSLBatchingQuantMatMul._get_padding_parameters, matmul.py:411-417, and used by
 * configs/PTQ4ViT.py:36-48).  A [batch,heads,S1,S2] @ B [batch,heads,S2,S3]. */
typedef struct p4v_matmul_desc {
  int32_t batch, heads, S1, S2, S3;
  int32_t A_bit, B_bit;
  int32_t eq_n;
  int32_t search_round;
  double eq_alpha, eq_beta;
  int32_t sos;       /* 1: split-of-softmax twin-uniform A (matmul.py:578-644)  */
  int32_t operand;
  int32_t kernel;
  int32_t init_layerwise; /* 1: every head starts from the layer-wise min-max step size (matmul.py:430-432) */
  int32_t images_per_chunk; /* 0: search the whole layer at once.  > 0 (at most batch): operand images are built for
                             * this many images at a time and the chunks' scores are added (matmul.py:396-409, :490-518) */
} p4v_matmul_desc;

P4V_API int p4v_matmul_workspace_bytes(const p4v_matmul_desc* d, size_t* bytes);
P4V_API int p4v_matmul_score_log_floats(const p4v_matmul_desc* d, size_t* n);
/* Replaces PTQSLBatchingQuantMatMul.calibration_step2() (matmul.py:565-576) and
 * SoSPTQSLBatchingQuantMatMul.calibration_step2() (matmul.py:633-644).
 * out: A_interval [heads] (sos: A_interval[0] = split/(qmax-1)), B_interval [heads], split [1] (sos)
 * With d->images_per_chunk > 0 every search step loops over the image chunks: it builds the chunk's A and B images
 * (current and candidate planes; split-of-softmax: the split candidates and the exact split of B), sweeps them and adds
 * the chunk's partial scores into the fp64 score table; the pick follows the last chunk.  Head-wise maxima and the
 * gradient scale are taken over all images first, so the result equals the unchunked search up to the order of the fp64
 * score sums. */
P4V_API int p4v_matmul_calibrate(const p4v_matmul_desc* d, const float* A, const float* B, const float* raw_out,
                         const float* raw_grad, void* workspace, size_t workspace_bytes, float* A_interval,
                         float* B_interval, float* split, float* score_log, void* stream);
/* Replaces quant_forward (matmul.py:140-145; SoS quant_input_A :595-598). */
P4V_API int p4v_matmul_quant_forward_workspace_bytes(const p4v_matmul_desc* d, size_t* bytes);
P4V_API int p4v_matmul_quant_forward(const p4v_matmul_desc* d, const float* A, const float* B, const float* A_interval,
                             const float* B_interval, const float* split, void* workspace, size_t workspace_bytes,
                             float* out, void* stream);

/* Frozen MatMul module: the step sizes and scale tables of a calibrated module packed once, and a forward that only
 * enqueues one kernel.  Replaces, per call of quant_forward (matmul.py:40-45 / :140-145; split-of-softmax quant_input_A
 * with A_interval = split / (A_qmax - 1), :595-598 / :628-629), the separate quantisation passes of both operands: the
 * output is bit-identical to p4v_matmul_quant_forward with the same step sizes.
 * `packed` (p4v_matmul_pack_bytes bytes; 16-byte aligned) depends on heads, the bit widths and sos only, not on batch
 * or the sequence lengths: the per-head step sizes A_interval [heads] (unused with sos) and B_interval [heads], split
 * [1] (sos), and the scale table of the unfrozen forward -- plain dA[h] * dB[h]; sos dB[h] * (1 / (A_qmax - 1)) and
 * dB[h] * (split / (A_qmax - 1)) -- computed by the same kernels.  p4v_matmul_pack copies a small table from the host.
 * p4v_matmul_frozen_forward reads A [batch,heads,S1,S2] and B [batch,heads,S2,S3] in place through element strides
 * (A_strides / B_strides: batch, head, then the two matrix dimensions, as torch's Tensor.stride()); A must have unit
 * stride along S2, B unit stride along S2 or S3 (the permuted q / k^T / v views of an attention block qualify).  `out` is
 * [batch,heads,S1,S3] contiguous.  No allocation, no host-to-device copy, no synchronisation, no workspace: it can be
 * captured in a CUDA graph.  Every argument is validated before the launch. */
P4V_API int p4v_matmul_pack_bytes(const p4v_matmul_desc* d, size_t* bytes);
P4V_API int p4v_matmul_pack(const p4v_matmul_desc* d, const float* A_interval, const float* B_interval, const float* split,
                    void* packed, size_t packed_bytes, void* stream);
P4V_API int p4v_matmul_frozen_forward(const p4v_matmul_desc* d, const float* A, const long long* A_strides, const float* B,
                              const long long* B_strides, const void* packed, float* out, void* stream);

/* Fused frozen attention core: one attention call of a block whose matmul1 and matmul2 modules are frozen.  Replaces the
 * reference's attention forward between the qkv and proj Linears (utils/models.py:10-26 for ViT / DeiT, :28-56 for
 * Swin windows) -- matmul1 (matmul.py:40-45), the `* scale`, relative-position bias and shifted-window mask, the softmax,
 * matmul2 (split-of-softmax A operand :595-598) and the transpose to [B, N, C] -- with one kernel
 * (csrc/forward_attn_tc.cu) whose output is bit-identical to that sequence on the frozen modules and torch's softmax.
 *   qkv        the qkv Linear's output as [batch, N, 3, heads, head_dim] with unit stride along head_dim; qkv_strides are
 *              the element strides of the batch, token, part (q / k / v) and head dimensions.  4-byte aligned.
 *   mm1, pack1 matmul1's descriptor and p4v_matmul_pack blob, as packed (heads must be a->heads; not split-of-softmax);
 *   mm2, pack2 matmul2's, likewise (plain or split-of-softmax).  pack*_bytes: the size of each blob.
 *   bias       [heads, N, N] contiguous, added to the scores, or NULL;
 *   mask       [n_windows, N, N] contiguous, added after the bias to image b's scores from window b % n_windows, or NULL.
 *   out        [batch, N, heads * head_dim] contiguous, 8-byte aligned.
 * Shapes: N <= 256 (the scores of one query tile stay in shared memory; p4v_attention_frozen_forward_long below takes
 * ViT / DeiT calls up to 1024 tokens), head_dim a multiple of 16, at most 64.
 * p4v_attention_fused_ok says whether a shape qualifies (a pure function of N and head_dim).  Every argument is validated
 * before the launch; no allocation, no copy, no synchronisation: the call can be captured in a CUDA graph. */
typedef struct p4v_attention_desc {
  int32_t batch;       /* images, or windows of all images (Swin)                                      */
  int32_t tokens;      /* N: queries = keys                                                              */
  int32_t heads, head_dim;
  int32_t scale_on_q;  /* 0: scores = matmul1 * scale (ViT, DeiT); 1: matmul1(q * scale, k^T) (Swin)     */
  int32_t n_windows;   /* rows of mask; 0 without a mask                                                 */
  double scale;        /* a Python float in the model: applied as (float)scale                           */
} p4v_attention_desc;
P4V_API int p4v_attention_fused_ok(int32_t tokens, int32_t head_dim, int* ok);
P4V_API int p4v_attention_frozen_forward(const p4v_attention_desc* a, const float* qkv, const long long* qkv_strides,
                                 const p4v_matmul_desc* mm1, const void* pack1, size_t pack1_bytes,
                                 const p4v_matmul_desc* mm2, const void* pack2, size_t pack2_bytes,
                                 const float* bias, const float* mask, float* out, void* stream);

/* The same attention core for longer sequences (ViT / DeiT at 384 pixels: 577 tokens), with its own kernel
 * (csrc/forward_attn_long_tc.cu) and the same bits.  A CTA quantises all keys and v of one (image, head) once and loops
 * over its 64-row query tiles, recomputing each tile's scores chunk by chunk instead of storing score rows, so shared
 * memory grows with N only through the quantised k and v.  The arguments are those of p4v_attention_frozen_forward,
 * validated the same way before the launch, with these differences: 1 <= N <= 1024 (torch's warp softmax, whose sum
 * order the kernel restates, covers rows of at most 1024 floats), and scale_on_q = 0, no bias, no mask (no windowed
 * model has more than 256 tokens).  head_dim: a multiple of 16, at most 64.  p4v_attention_long_ok is the shape rule.
 * One launch; no allocation, no copy, no synchronisation. */
P4V_API int p4v_attention_long_ok(int32_t tokens, int32_t head_dim, int* ok);
P4V_API int p4v_attention_frozen_forward_long(const p4v_attention_desc* a, const float* qkv, const long long* qkv_strides,
                                      const p4v_matmul_desc* mm1, const void* pack1, size_t pack1_bytes,
                                      const p4v_matmul_desc* mm2, const void* pack2, size_t pack2_bytes,
                                      const float* bias, const float* mask, float* out, void* stream);

/* Fused frozen MLP: one call of a transformer block's MLP (utils/models.py Mlp: fc2(act(fc1(x))), act = nn.GELU()) whose
 * fc1 and fc2 Linears are frozen (p4v_linear_pack).  Replaces the unfrozen sequence of quant_forward(fc1) (linear.py:62-67),
 * torch's GELU and quant_forward(fc2), whose activation quantiser (linear.py:62-67, post-GELU: :601-607) reads the GELU
 * output, with two launches:
 *   A. fc1 on the fused kernel (csrc/forward_tc.cu) with an epilogue that applies torch's fp32 GELU (approximate='none')
 *      to each output element and quantises it with fc2's activation quantiser into fc2's int8 activation image, the
 *      image of fc2's streamed path (p4v_linear_frozen_forward): the hidden activations reach HBM only as those bytes;
 *   B. fc2's sweep forward on that image.
 * Every byte of the image and every output bit equal those of p4v_linear_frozen_forward(fc1), torch.nn.functional.gelu
 * and p4v_linear_frozen_forward(fc2).  The descriptors are those fc1 and fc2 were packed with, their rows the rows of x.
 * p4v_mlp_fused_ok is the shape rule, a pure function of the descriptors without their rows: fc1.out_features ==
 * fc2.in_features, fc1 plain (not post-GELU) with the fused kernel as its frozen path, and the fused kernel's shared-memory
 * plan with the epilogue fits.  p4v_mlp_frozen_workspace_bytes: the size of fc2's image for the rows (the caller's
 * workspace).  p4v_mlp_frozen_forward validates every argument before it launches anything (null pointers, equal rows,
 * the shape rule, pack sizes, alignment: x 16 bytes, out 8 bytes, workspace 16 bytes; workspace size), then enqueues the
 * two kernels: no allocation, no copy, no synchronisation, so it can be captured in a CUDA graph. */
P4V_API int p4v_mlp_fused_ok(const p4v_linear_desc* fc1, const p4v_linear_desc* fc2, int* ok);
P4V_API int p4v_mlp_frozen_workspace_bytes(const p4v_linear_desc* fc1, const p4v_linear_desc* fc2, size_t* bytes);
P4V_API int p4v_mlp_frozen_forward(const p4v_linear_desc* fc1, const float* x, const float* bias1, const void* pack1,
                                   size_t pack1_bytes, const p4v_linear_desc* fc2, const float* bias2, const void* pack2,
                                   size_t pack2_bytes, void* workspace, size_t workspace_bytes, float* out, void* stream);
/* Diagnostic: y[i] = the GELU of the fused MLP's epilogue applied to x[i], for i < n (one launch on `stream`), so that it
 * can be compared with torch.nn.functional.gelu over every fp32 bit pattern. */
P4V_API int p4v_gelu_probe(const float* x, float* y, long long n, void* stream);

/* A LayerNorm folded into the frozen Linear that consumes it: out = layer(LayerNorm(x)) with torch's exact fp32 LayerNorm
 * (its vectorised kernel: weight and bias present, in_features % 4 == 0) computed in the fused kernel's activation
 * quantiser, so the normalised activations never reach HBM.  Bit-identical to torch's F.layer_norm followed by
 * p4v_linear_frozen_forward.
 * p4v_linear_norm_ok is the shape rule, a pure function of the descriptor without its rows: the layer is on the fused
 * path (p4v_linear_frozen_path), not post-GELU, in_features % 4 == 0, and the shared-memory plan with the per-row
 * statistics fits.  p4v_mlp_norm_ok: the same for fc1 of a fused MLP (p4v_mlp_fused_ok and the plan with the epilogue and
 * the statistics fits).
 * p4v_linear_frozen_forward_norm / p4v_mlp_frozen_forward_norm mirror p4v_linear_frozen_forward / p4v_mlp_frozen_forward
 * with the pre-norm x [rows][in_features] and the LayerNorm's gamma and beta [in_features] (contiguous, 16-byte aligned)
 * and eps (finite, >= 0).  Every argument is validated before the one launch of the folded layer (the MLP adds fc2's sweep);
 * nothing is allocated or copied, so both can be captured in a CUDA graph. */
P4V_API int p4v_linear_norm_ok(const p4v_linear_desc* d, int* ok);
P4V_API int p4v_mlp_norm_ok(const p4v_linear_desc* fc1, const p4v_linear_desc* fc2, int* ok);
P4V_API int p4v_linear_frozen_forward_norm(const p4v_linear_desc* d, const float* x, const float* gamma, const float* beta,
                                           float eps, const float* bias, const void* packed, float* out, void* stream);
P4V_API int p4v_mlp_frozen_forward_norm(const p4v_linear_desc* fc1, const float* x, const float* gamma, const float* beta,
                                        float eps, const float* bias1, const void* pack1, size_t pack1_bytes,
                                        const p4v_linear_desc* fc2, const float* bias2, const void* pack2, size_t pack2_bytes,
                                        void* workspace, size_t workspace_bytes, float* out, void* stream);
/* Diagnostic: y = the LayerNorm of the folded kernels applied to each row of x [M][N] (N % 4 == 0, x 16-byte aligned),
 * so that it can be compared with torch.nn.functional.layer_norm bit for bit. */
P4V_API int p4v_layer_norm_probe(const float* x, const float* gamma, const float* beta, float eps, long long M, int N, float* y,
                                 void* stream);

/* A block's residual add folded into the store of the frozen Linear that produces it: out[dst(r)] = fl(y[r] + residual[dst(r)])
 * for every output row r of the layer, y the output p4v_linear_frozen_forward computes.  Bit-identical to that call
 * followed by torch's elementwise FP32 add, signed zeros included; the Linear's FP32 output never reaches HBM.
 * dst is the identity, or for Swin's attention projection the window layout below: window row
 *   r = ((b * nH + wh) * nW + ww) * window^2 + i * window + j      (nH = height / window, nW = width / window)
 * is image row b * height * width + ((wh * window + i + shift) mod height) * width + (ww * window + j + shift) mod width,
 * which replaces  x + roll(window_reverse(proj(...)), (shift, shift))  of a (shifted) Swin block.  A layout needs
 * window > 0, height % window == 0, width % window == 0, 0 <= shift < window and images * height * width == rows, and the
 * layer on its fused path (p4v_linear_frozen_path 1): the streamed path takes the identity only.
 * p4v_linear_frozen_forward_res replaces  residual + p4v_linear_frozen_forward(...)  (either path); layout null = identity.
 * p4v_mlp_frozen_forward_res / p4v_mlp_frozen_forward_norm_res replace  residual + p4v_mlp_frozen_forward(...)  /
 * residual + p4v_mlp_frozen_forward_norm(...): the add is fc2's, always on its streamed sweep, in identity rows.
 * residual is [rows][out_features] FP32, contiguous, 8-byte aligned and must not overlap out.  Every argument of the
 * underlying call and the residual and layout are validated before anything is launched; the launches are those of the
 * underlying call, nothing is allocated or copied, so each can be captured in a CUDA graph. */
typedef struct p4v_window_layout {
  int32_t images, height, width, window, shift;
} p4v_window_layout;
P4V_API int p4v_linear_frozen_forward_res(const p4v_linear_desc* d, const float* x, const float* bias, const void* packed,
                                          void* workspace, size_t workspace_bytes, const float* residual,
                                          const p4v_window_layout* layout, float* out, void* stream);
P4V_API int p4v_mlp_frozen_forward_res(const p4v_linear_desc* fc1, const float* x, const float* bias1, const void* pack1,
                                       size_t pack1_bytes, const p4v_linear_desc* fc2, const float* bias2, const void* pack2,
                                       size_t pack2_bytes, void* workspace, size_t workspace_bytes, const float* residual,
                                       float* out, void* stream);
P4V_API int p4v_mlp_frozen_forward_norm_res(const p4v_linear_desc* fc1, const float* x, const float* gamma, const float* beta,
                                            float eps, const float* bias1, const void* pack1, size_t pack1_bytes,
                                            const p4v_linear_desc* fc2, const float* bias2, const void* pack2,
                                            size_t pack2_bytes, void* workspace, size_t workspace_bytes,
                                            const float* residual, float* out, void* stream);

/* A row gather in front of a LayerNorm folded into its frozen Linear: out = layer(LayerNorm(gather(x))), where the rows
 * the layer consumes are read from an image x [images][height][width][C] (contiguous, 16-byte aligned) instead of being
 * copied there by torch first.  LayerNorm is per row, so the normalised rows are those of the unfolded sequence; the
 * result is bit-identical to it and neither the normalised nor the gathered activations reach HBM.
 * P4V_GATHER_WINDOW (Swin's norm1 -> roll(-shift) -> window partition -> qkv): C = in_features, and output row r, in
 * window order
 *   r = ((b * nH + wh) * nW + ww) * window^2 + i * window + j      (nH = height / window, nW = width / window)
 * is computed from image row b * height * width + ((wh * window + i + shift) mod height) * width + (ww * window + j + shift)
 * mod width -- the window layout of p4v_linear_frozen_forward_res, read in the other direction.  The layout needs
 * window > 0, height % window == 0, width % window == 0, 0 <= shift < window and images * height * width == rows.
 * P4V_GATHER_MERGE (Swin's PatchMerging: cat(x[0::2, 0::2], x[1::2, 0::2], x[0::2, 1::2], x[1::2, 1::2]) -> norm ->
 * reduction): in_features = 4 C, and output row m = (b * (height / 2) + i) * (width / 2) + j takes its columns
 * [q C, (q + 1) C) from image row b * height * width + (2 i + (q & 1)) * width + 2 j + (q >> 1), q = 0 .. 3.  The layout
 * has window = shift = 0, height and width even and images * (height / 2) * (width / 2) == rows.
 * p4v_linear_gather_ok is the shape rule of a mode, a pure function of the descriptor without its rows: p4v_linear_norm_ok,
 * in_features % 16 == 0 for the merge, and the shared-memory plan with the 512-byte table of source rows fits.  A layer
 * on the streamed path (p4v_linear_frozen_path 0) never takes a gather.
 * p4v_linear_frozen_forward_norm_gather mirrors p4v_linear_frozen_forward_norm with the image x and the descriptor g.
 * Every argument is validated before its one launch (the LayerNorm's as there, g, the rule, the layout, x not
 * overlapping out); nothing is allocated or copied, so it can be captured in a CUDA graph. */
#define P4V_GATHER_WINDOW 1
#define P4V_GATHER_MERGE 2
typedef struct p4v_input_gather {
  int32_t mode;                  /* P4V_GATHER_WINDOW or P4V_GATHER_MERGE */
  p4v_window_layout layout;      /* the image: images, height, width; the window and shift (merge: 0, 0) */
} p4v_input_gather;
P4V_API int p4v_linear_gather_ok(const p4v_linear_desc* d, const p4v_input_gather* g, int* ok);
P4V_API int p4v_linear_frozen_forward_norm_gather(const p4v_linear_desc* d, const float* x, const float* gamma,
                                                  const float* beta, float eps, const float* bias, const void* packed,
                                                  const p4v_input_gather* g, float* out, void* stream);

/* The attention operands' quantisation folded into the frozen qkv Linear of an attention block whose matmul1 and matmul2
 * are frozen: the qkv kernel's epilogue quantises its output with the step sizes of the attention's operands and writes
 * int8 planes instead of the FP32 output, and the short attention kernel reads those planes instead of quantising q, k and
 * v from FP32.  Output row r = b * N + n and column c of qkv (torch's reshape(batch, N, 3, heads, head_dim)) go to
 *   planes[part][b][h][n][j]   ([3][batch][heads][N][head_dim] int8, contiguous), part = c / C, h = (c % C) / head_dim,
 *                              j = c % head_dim, C = heads * head_dim
 * as clamp(rne(y / delta), lo, hi) with, for q, y = fl(value * (float)scale) when scale_on_q and the value otherwise,
 * matmul1's A step size of head h; for k matmul1's B step size; for v matmul2's B step size -- the bytes the attention
 * kernel of p4v_attention_frozen_forward makes of them.  p4v_linear_frozen_forward_qkv8 followed by
 * p4v_attention_frozen_forward_i8 is bit-identical to p4v_linear_frozen_forward (or its LayerNorm / gather variants)
 * followed by p4v_attention_frozen_forward, and qkv's FP32 output never reaches HBM.
 * p4v_linear_qkv8_ok is the shape rule, a pure function of the descriptors without their rows: out_features == 3 heads
 * head_dim, p4v_attention_fused_ok(tokens, head_dim), the layer on its fused path (p4v_linear_frozen_path 1; a streamed
 * qkv never folds) and the shared-memory plan with the epilogue's staging fits beside a two-stage weight ring -- with the
 * LayerNorm's row statistics too when the layer can take a LayerNorm (p4v_linear_norm_ok's conditions), so the rule
 * holds with and without one.  gather_mode: 0, or P4V_GATHER_WINDOW for a call with a window gather (and the rule of
 * p4v_linear_gather_ok).
 * p4v_linear_frozen_forward_qkv8: qkv's descriptor (rows = batch * tokens), x, bias and pack as for
 * p4v_linear_frozen_forward; the attention descriptor and matmul1's and matmul2's descriptors and packs as for
 * p4v_attention_frozen_forward; planes (16-byte aligned, 3 * rows * C bytes); an optional LayerNorm (gamma, beta, eps as
 * p4v_linear_frozen_forward_norm; gamma null = none) and an optional window gather (g null = none; with the LayerNorm, as
 * p4v_linear_frozen_forward_norm_gather).  p4v_attention_frozen_forward_i8 takes the planes in place of qkv and its
 * strides, and otherwise the arguments of p4v_attention_frozen_forward (N <= 256).  Both validate every argument before
 * their one launch: null pointers, alignment, heads and head_dim against the descriptors, pack sizes, a split-of-softmax
 * matmul1 (refused), the rule, and x or out overlapping the planes.  Neither allocates, copies or synchronises: both can
 * be captured in a CUDA graph. */
P4V_API int p4v_linear_qkv8_ok(const p4v_linear_desc* d, const p4v_attention_desc* a, int gather_mode, int* ok);
P4V_API int p4v_linear_frozen_forward_qkv8(const p4v_linear_desc* d, const float* x, const float* bias, const void* packed,
                                           const p4v_attention_desc* a, const p4v_matmul_desc* mm1, const void* pack1,
                                           size_t pack1_bytes, const p4v_matmul_desc* mm2, const void* pack2,
                                           size_t pack2_bytes, int8_t* planes, const float* gamma, const float* beta,
                                           float eps, const p4v_input_gather* g, void* stream);
P4V_API int p4v_attention_frozen_forward_i8(const p4v_attention_desc* a, const int8_t* planes, const p4v_matmul_desc* mm1,
                                            const void* pack1, size_t pack1_bytes, const p4v_matmul_desc* mm2,
                                            const void* pack2, size_t pack2_bytes, const float* bias, const float* mask,
                                            float* out, void* stream);

/* The patch-embedding convolution: ChannelwiseBatchingQuantConv2d with a_bit >= 32 (quant_layers/conv.py:444-614, wired
 * by configs/PTQ4ViT.py:52-54): one weight step size per output channel, activations left in FP32.  The caller passes
 * the im2col matrix of the FP32 input (torch.nn.functional.unfold, [images, positions, K], K = in_channels*kh*kw in the
 * kernel's own order), the kernel as [out_channels, K] and raw_out / raw_grad as [images, out_channels, positions]. */
typedef struct p4v_conv_desc {
  int32_t images, out_channels, K, positions;
  int32_t w_bit;
  int32_t eq_n;
  double eq_alpha, eq_beta;
  int32_t has_bias;
  int32_t kernel;    /* P4V_KERNEL_TCGEN05 only */
  int32_t layerwise; /* 0: channel-wise (above).  1: BatchingEasyQuantConv2d with a_bit >= 32 (conv.py:279-441, wired by
                        configs/BasePTQ.py:48-50): ONE weight step size for the whole kernel, initial max|W| / (qmax - 0.5)
                        (:313), score -sum_images mean_positions mean_channels (g*(y - yhat))^2 (:387-394), first argmax
                        (:395-396).  The same search with every channel given that step size. */
} p4v_conv_desc;
P4V_API int p4v_conv_workspace_bytes(const p4v_conv_desc* d, size_t* bytes);
/* Replaces ChannelwiseBatchingQuantConv2d.calibration_step2() (conv.py:591-603): _initialize_intervals (:482-496) and
 * _search_best_w_interval (:526-557).  out: w_interval [out_channels] (reference shape oc,1,1,1), score_log NULL or
 * [eq_n][out_channels].  The search is the same in every round when the activations are not quantised: it runs once.
 * With desc.layerwise = 1 it replaces BatchingEasyQuantConv2d.calibration_step2() (conv.py:429-441): _initialize_intervals
 * (:312-320, weight part) and _search_best_w_interval (:365-396); out: w_interval [1] (reference shape 1,1,1,1),
 * score_log NULL or [eq_n]. */
P4V_API int p4v_conv_calibrate(const p4v_conv_desc* d, const float* cols, const float* weight, const float* bias,
                       const float* raw_out, const float* raw_grad, void* workspace, size_t workspace_bytes,
                       float* w_interval, float* score_log, void* stream);

/* Frozen patch-embedding convolution: the integer weights of a calibrated conv module with a_bit >= 32 packed once, and
 * a forward that reads no FP32 weight.  Replaces, per call of quant_forward (quant_layers/conv.py:69-74 with
 * quant_weight_bias :53-62; the activation quantiser :64-67 is off), the re-quantisation of the weight and
 * F.conv2d(x, fl(q * delta), bias) for kernel == stride, padding 0, dilation 1, groups 1 (the patch embedding of
 * ViT, DeiT and Swin; the Python layer checks stride, padding, dilation and groups, which the descriptor does not carry):
 *   out[b, o, py, px] = fmaf(delta[o], S, bias[o])      (delta[o] * S rounded once without a bias)
 *   S = sum_k (x_hi + x_mid + x_lo)[b, k at (py, px)] * q[o, k],   k = (c, i, j) in weight.reshape(O, K) order
 * q: the integers of the export quantiser (p4v_export_quantized mode 0) for this weight and w_interval; x_hi/mid/lo: the
 * exact three-term bf16 split of the FP32 pixel; bf16 wgmma products chained into one fp32 accumulator.  Not
 * bit-identical to cuDNN's convolution; the bound against fp64 (ref = fp64(sum_k x_k * fl(q * delta)[o, k] + bias[o])):
 *   |out - ref| <= (3K + 2) * 2^-23 * sum_k |x_k * fl(q * delta)[o, k]|  +  2^-23 * |ref|
 * Repeated calls give the same bits (fixed summation order). */
typedef struct p4v_conv_frozen_desc {
  int32_t images, in_channels, height, width;   /* x [images, in_channels, height, width], contiguous fp32        */
  int32_t out_channels, kernel_h, kernel_w;     /* stride = kernel; out [images, out_channels, height / kernel_h,
                                                   width / kernel_w], contiguous fp32 (what F.conv2d returns)      */
  int32_t w_bit;
  int32_t layerwise;                            /* 1: w_interval holds one step size (BatchingEasyQuantConv2d),
                                                   0: one per output channel (ChannelwiseBatchingQuantConv2d)      */
  int32_t has_bias;
} p4v_conv_frozen_desc;
/* The shape rule, a pure function of the descriptor's module geometry (images, height and width are not consulted):
 * 1 <= out_channels <= 4096, 1 <= K = in_channels * kernel_h * kernel_w <= 4096, 2 <= w_bit <= 8, flags 0 or 1. */
P4V_API int p4v_conv_frozen_ok(const p4v_conv_frozen_desc* d, int* ok);
/* `packed` (p4v_conv_pack_bytes bytes, independent of images, height and width; 16-byte aligned): the step size of every
 * output channel (one repeated when layer-wise) and the bf16 image of q in 128-channel tiles and 32-element K slabs.
 * p4v_conv_pack quantises weight [out_channels, K] fp32 with w_interval ([out_channels], or [1] when layer-wise). */
P4V_API int p4v_conv_pack_bytes(const p4v_conv_frozen_desc* d, size_t* bytes);
P4V_API int p4v_conv_pack(const p4v_conv_frozen_desc* d, const float* weight, const float* w_interval, void* packed,
                          size_t packed_bytes, void* stream);
/* One launch (csrc/forward_conv_tc.cu); every argument is validated first: null pointers, the shape rule, geometry
 * (images >= 1, height >= kernel_h, width >= kernel_w), packed_bytes, alignment (packed 16 bytes; x, bias, out 4 bytes).
 * No allocation, no copy, no synchronisation: it can be captured in a CUDA graph. */
P4V_API int p4v_conv_frozen_forward(const p4v_conv_frozen_desc* d, const float* x, const float* bias, const void* packed,
                                    size_t packed_bytes, float* out, void* stream);
/* The patch embedding's token epilogue folded into the frozen convolution: the kernel stores the token rows the model's
 * stem makes of the conv output, instead of the NCHW output torch then flattens, transposes and copies.  Each value is
 * the one p4v_conv_frozen_forward computes, v = conv[b, o, p] (p = py * (width / kernel_w) + px), and the result is
 * bit-identical to that call followed by torch's ops.  P = (height / kernel_h) * (width / kernel_w).
 * p4v_conv_frozen_forward_pos (ViT / DeiT): out [images][1 + P][out_channels],
 *   out[b][0][o] = fl(cls[o] + pos[0][o]),   out[b][1 + p][o] = fl(v + pos[1 + p][o])
 * which replaces  torch.cat((cls_token.expand(B, -1, -1), conv.flatten(2).transpose(1, 2)), 1) + pos_embed;
 * cls [out_channels] and pos [1 + P][out_channels] (cls_numel and pos_numel must be exactly that).
 * p4v_conv_frozen_forward_norm (Swin): out [images][P][out_channels], each token row normalised with torch's exact
 * LayerNorm (its vectorised kernel, the one the LayerNorm fold of p4v_linear_frozen_forward_norm reproduces), gamma and
 * beta [out_channels] (norm_numel must be exactly that), eps finite and >= 0; replaces
 * patch_norm(conv.flatten(2).transpose(1, 2)).
 * p4v_conv_pos_ok / p4v_conv_norm_ok are their shape rules, pure functions of the module geometry: p4v_conv_frozen_ok
 * and out_channels % 4 == 0; the LayerNorm also out_channels <= 128 (the whole token row in one CTA of the kernel).
 * Every argument is validated before the one launch: null pointers, the rule, geometry, packed_bytes, alignment (out,
 * cls, pos, gamma and beta 16 bytes; the rest as p4v_conv_frozen_forward), the element counts above and out not
 * overlapping any input.  No workspace, no allocation, no copy: each can be captured in a CUDA graph. */
P4V_API int p4v_conv_pos_ok(const p4v_conv_frozen_desc* d, int* ok);
P4V_API int p4v_conv_norm_ok(const p4v_conv_frozen_desc* d, int* ok);
P4V_API int p4v_conv_frozen_forward_pos(const p4v_conv_frozen_desc* d, const float* x, const float* bias, const void* packed,
                                        size_t packed_bytes, const float* cls, size_t cls_numel, const float* pos,
                                        size_t pos_numel, float* out, void* stream);
P4V_API int p4v_conv_frozen_forward_norm(const p4v_conv_frozen_desc* d, const float* x, const float* bias, const void* packed,
                                         size_t packed_bytes, const float* gamma, const float* beta, size_t norm_numel,
                                         float eps, float* out, void* stream);

/* Integer export of a calibrated module (utils/integer.py:8-129): src [rows, cols] fp32 -> dst one byte per element.
 * mode 0: int8 = clamp(rne(x / delta), -q, q-1) (quantize_int_weight :8-18, quantize_matmul_input :27-42, plain
 * activations :64-69); mode 1: the post-GELU twin uint8 layout (:51-62); mode 2: the split-of-softmax twin uint8 layout
 * (:78-87).  delta[((row / rows_per_block) % n_row_blocks) * n_col_blocks + col / cols_per_block] is the step size of an
 * element (rows_per_block = 0: one row block). */
P4V_API int p4v_export_quantized(const float* src, long long rows, long long cols, const float* delta, int rows_per_block,
                         int n_row_blocks, int cols_per_block, int n_col_blocks, int mode, int bit, float d_neg,
                         const float* split, void* dst, void* stream);

P4V_API const char* p4v_last_error(void);
P4V_API int p4v_version(void);
/* number of kernel launches issued by this library in this process so far (for bench.py's gpu_launches) */
P4V_API long long p4v_launch_count(void);
/* Optional live timing of the sweep kernel (bench.py's roofline): while enabled every sweep launch is
 * bracketed by CUDA events on its own stream.  p4v_profile_collect synchronises those events and returns
 * the summed device time (ms), the number of sweep launches and the tensor-core operations (2*MAC) they
 * executed, then clears the record. */
P4V_API int p4v_profile_enable(int on);
P4V_API int p4v_profile_collect(double* sweep_ms, long long* sweep_launches, double* executed_ops);
/* The same record split by launch kind: out[0..2] = device ms of the bf16 slab sweeps, the int8 slab sweeps and the Gram
 * GEMMs, out[3..5] = tensor-core operations they executed, out[6..8] = launches, out[9..11] = the longest single launch
 * (ms, operations, kind).  n must be >= 12. */
P4V_API int p4v_profile_collect_kinds(double* out, int n);
/* One row of P4V_LAUNCH_COLS doubles per launch recorded since profiling was enabled, in launch order, for tests that
 * pin the path a shape takes: kind (0 bf16 sweep, 1 int8 sweep, 2 Gram GEMM), the SIMT kernel ran (0/1), consumer mode
 * (0 multi-segment, 1 single, 2 pair; -1 for SIMT sweeps and Gram GEMMs), shared-memory ring stages, resident row-operand
 * buffers, resident row-operand bytes (0: streamed), resident column-image bytes (0: streamed), CTAs launched, tiles,
 * candidates, candidate groups, candidate jobs.  Writes at most max_rows rows, sets *n_rows to the number recorded and
 * does not clear the record (p4v_profile_collect_kinds does). */
#define P4V_LAUNCH_COLS 12
P4V_API int p4v_profile_collect_launches(double* out, int max_rows, int* n_rows);
/* Device self-test of the quantiser's division shortcut: evaluates round(v / delta) for n pseudo-random (v, delta)
 * pairs (plus pairs placed on and next to rounding ties) both with IEEE division, as the reference does
 * (quant_layers/linear.py:99-103 `(x / interval).round_()`), and with the reciprocal-based sequence the operand
 * image kernels use; writes the number of disagreements (must be 0).  Diagnostic only: unlike every other entry
 * point it allocates 8 bytes of device memory for the duration of the call and synchronises the stream. */
P4V_API int p4v_selftest_rint_div(unsigned long long n, unsigned long long seed, unsigned long long* mismatches, void* stream);

#ifdef __cplusplus
}
#endif
#endif
