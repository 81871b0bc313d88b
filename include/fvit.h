/* fvit.h — C ABI of libfvit_sm100.so: the H100 (sm_90a) kernels behind FasterViT.forward/backward.
 *
 * The reference (NVlabs/FasterViT) has no FFI: its hot path is torch.nn modules in
 * fastervit/models/faster_vit.py. Each entry point below replaces the ATen/cuDNN/cuBLAS call sequence
 * of the cited reference lines. Conventions:
 *   - plain device pointers + explicit sizes/strides; no C++/torch types cross the boundary;
 *   - every launch goes to the cudaStream_t passed as `stream` (a `void*`); nothing synchronises;
 *   - no allocation or free of caller memory; outputs/workspaces are caller-provided;
 *   - return 0 on success, non-zero on error; fvit_last_error() returns a per-thread message;
 *   - activations are row-major "token-major" (NHWC) matrices [rows, channels]; tensor-core operands
 *     are fp16 (or bf16) with fp32 accumulation, the residual stream and statistics are fp32.
 */
#ifndef FVIT_H_
#define FVIT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FVIT_ABI_VERSION 1

/* ---- library ------------------------------------------------------------------------------- */
int fvit_abi_version(void);
const char* fvit_last_error(void);
/* number of kernels launched by this library since load (or since last reset) — bench.py's
 * "gpu_launches" evidence. */
int64_t fvit_launch_count(void);
void fvit_reset_launch_count(void);
/* A launch list captured into a CUDA graph launches its kernels without passing through the entry points: the host side
 * adds the number of kernel nodes per replay so that fvit_launch_count() stays the number of kernels that really ran. */
void fvit_add_launch_count(int64_t n);
/* Persistent kernels (GEMM, attention) size their grids to the SM count; n > 0 caps that count for the launches that
 * follow (0 = no cap). Used while a gradient all-reduce is in flight: NCCL's CTAs cannot share an SM with a 227 KB GEMM
 * CTA, so a full-width grid would run its last CTAs as a second wave. */
void fvit_set_sm_limit(int32_t n);

/* ---- epilogue activation codes --------------------------------------------------------------- */
enum {
  FVIT_ACT_NONE = 0,
  FVIT_ACT_RELU = 1,
  FVIT_ACT_GELU = 2,     /* exact erf GELU (nn.GELU default; fv.py:379,491) */
  FVIT_ACT_GELU_BWD = 3, /* v *= gelu'(aux[row,col])  (backward of the above) */
  FVIT_ACT_RELU_BWD = 4, /* v *= (aux[row,col] > 0) */
  FVIT_ACT_MUL_AUX = 5   /* v *= aux[row,col]  (aux = gelu' saved by the forward GEMM, see pre_is_grad) */
};

/* ---- tensor-core GEMM with shifted-row taps and fused epilogue --------------------------------
 * D[m, n] = epilogue( sum_{t < ntaps} sum_{k < kc} A[plane_t][m + shift_t][k] * B[n][t*kc_pad + k] )
 *
 *  - linear layers (fv.py:401-404, 545-547, 559, 566, 927): ntaps = 1;
 *  - 3x3 convolutions on zero-bordered NHWC activations (fv.py:434, 458-461, 489-492) are the same
 *    kernel with 9 taps whose row shift is (dy*(W+2)+dx) in the flattened padded pixel index, i.e.
 *    im2col-free implicit GEMM: every tap is a plain 2-D TMA box of the activation matrix;
 *  - backward passes use a_mn_major / b_mn_major = 1 (operand stored [K, MN]) and split_k.
 *
 * Operands are 16-bit (fp16, or bf16 when `bf16` != 0), accumulated in fp32 in tensor memory.
 * Epilogue per element:  v = acc * alpha
 *                        v = v * col_scale[n] + col_shift[n]          (each optional)
 *                        out_pre16[m, n] = (half)v                     (optional: pre-activation copy)
 *                        v = act(v [, aux])                            (FVIT_ACT_*)
 *                        v = v * col_scale2[n] * row_scale[m]          (each optional, after act)
 *                        v += resid[orow, n]                           (optional, fp32)
 *                        out_f32[orow, n] = v ; out_f16[orow, n] = (half)v   (each optional)
 * with orow = row_map ? row_map[m] : m, rows with orow < 0 skipped. If col_sum/col_sumsq are given,
 * sum and sum-of-squares of v (after alpha/scale/shift, before act) over valid rows are atomically
 * added per column (train-mode BatchNorm statistics). With split_k > 1 the partial products are
 * atomically added into out_f32 (which the caller zeroed) and only `alpha` is applied.
 */
typedef struct fvit_gemm_args {
  /* A operand: K-major: [a_planes][a_rows][kc] with row stride lda (elements);
   *            MN-major: [a_rows = K][m] with row stride lda. */
  const void* a;
  int64_t a_rows;
  int64_t lda;
  int64_t a_plane_stride; /* elements; 0 if a_planes == 1 */
  int32_t a_planes;
  int32_t a_mn_major;
  /* B operand: K-major: [n][ntaps*kc_pad] row stride ldb; MN-major: [b_rows = K][n] row stride ldb */
  const void* b;
  int64_t b_rows;
  int64_t ldb;
  int32_t b_mn_major;
  int32_t bf16;
  /* problem */
  int32_t m, n, kc, ntaps;
  int32_t tap_shift[16]; /* row shift of A per tap */
  int32_t tap_plane[16]; /* plane of A per tap */
  int32_t a_row_off;     /* extra row offset on A K-rows (MN-major) */
  int32_t b_row_off;     /* extra row offset on B K-rows (MN-major) */
  int32_t split_k;       /* >= 1 */
  int32_t b_ntaps;       /* 0/1 = off. > 1 (conv weight gradient): the logical output has b_ntaps * n columns; column
                            block t is A^T-style product with B's K rows shifted by tap_shift[t] (A and B MN-major,
                            ntaps == 1): dW[co][t*n + ci] = sum_q dz[q][co] * x[q + tap_shift[t]][ci] */
  int32_t tile_n;        /* 0 = auto; else multiple of 16 in [16, 256] (wider than 128: split into two tiles) */
  /* epilogue */
  float alpha;
  int32_t act;
  const float* col_scale;
  const float* col_shift;
  const float* col_scale2;
  const void* aux; /* fp16 [m, n] indexed by m (not orow), row stride ld_aux */
  int64_t ld_aux;
  const float* resid;
  int64_t ld_resid;
  const int32_t* row_map;
  float* out_f32;
  int64_t ld_out_f32;
  void* out_f16;
  int64_t ld_out_f16;
  float* col_sum;
  float* col_sumsq;
  /* training-path extras (all optional) */
  const float* alpha_ptr; /* device scalar multiplied into alpha (gradient un-scaling without a host sync) */
  const float* row_scale; /* fp32 [m]: v *= row_scale[m] together with col_scale2 (stochastic depth masks,
                             per-row layer-scale in weight-gradient GEMMs) */
  void* out_pre16;        /* fp16 [m, n] (indexed by m): value after scale/shift, before act / col_scale2 /
                             row_scale / resid (pre-GELU activations; un-scaled branch outputs) */
  int64_t ld_out_pre16;
  float* out_colsum;      /* optional fp32 [n]: += *out_colsum_alpha * sum over rows of the rounded out_f16 values
                             (dgrad GEMM producing dZ of the previous Linear -> that Linear's bias gradient) */
  const float* out_colsum_alpha; /* device scalar, NULL = 1 */
  const float* aux_scale; /* optional fp32 [n] pair: the *_BWD activations see aux * aux_scale + aux_shift (aux = saved raw */
  const float* aux_shift; /* convolution output, scale/shift = that BatchNorm's batch-statistics affine) */
  int32_t pre_is_grad;    /* with act == FVIT_ACT_GELU and out_pre16: store gelu'(v) there instead of v, so the
                             backward GEMM's epilogue is a plain multiply (FVIT_ACT_MUL_AUX) */
  int32_t cta_group;      /* 0, 1 or 2; accepted for source compatibility: sm_90a has no CTA-pair MMA, every call
                             runs one CTA per 128-row tile */
} fvit_gemm_args;

int fvit_gemm(const fvit_gemm_args* args, void* stream);

/* ---- weight preparation (fp32 nn.Parameter -> packed fp16 tensor-core operands) ---------------- */
/* dst[r][0:cols_pad] = (half)src[r][0:cols], zero padded; nn.Linear weights [out, in] (fv.py:393-395,
 * 545-547, 927) become K-major B operands with a 16-byte aligned row stride. */
int fvit_cast_pad_f16(const float* src, int64_t lds, void* dst, int64_t ldd, int32_t rows,
                      int32_t cols, int32_t cols_pad, void* stream);
/* head-padded variants for the tensor-core attention path: blocks of `hd` rows / columns become
 * blocks of `hdp` (zero filled), so every head slice of q, k, v and of the attention output is a
 * 16-byte aligned TMA box (fv4: head_dim 49 -> 64). */
int fvit_cast_headpad_f16(const float* src, int64_t lds, void* dst, int64_t ldd, int32_t rows_dst,
                          int32_t cols_dst, int32_t hd, int32_t hdp, int32_t pad_rows, int32_t pad_cols,
                          void* stream);
int fvit_vec_headpad_f32(const float* src, float* dst, int32_t n_dst, int32_t hd, int32_t hdp, void* stream);
/* nn.Conv2d weight [cout][cin][3][3] (fv.py:434, 461, 489, 492) -> [cout][9][kc_pad] fp16, tap-major;
 * transpose_io != 0 builds the data-gradient operand [cin][9 flipped][kc_pad >= cout]. */
int fvit_pack_conv3x3_f16(const float* w, void* dst, int32_t cout, int32_t cin, int32_t kc_pad,
                          int32_t transpose_io, void* stream);
/* explicit tap list (no flip): dst[co][j][ci] = w[co][ci][t_j], or with transpose_io dst[ci][j][co]; used for the
 * data gradient of the stride-2 convolutions (one GEMM per input parity plane). */
int fvit_pack_conv3x3_taps_f16(const float* w, void* dst, int32_t cout, int32_t cin, int32_t kc_pad,
                               int32_t transpose_io, int32_t ntaps, int32_t t0, int32_t t1, int32_t t2, int32_t t3,
                               int32_t t4, int32_t t5, int32_t t6, int32_t t7, int32_t t8, void* stream);
/* scale/shift so that acc*scale+shift == layer_scale * BN_eval(acc + bias) (fv.py:504-510) or
 * layer_scale * (acc + bias) (fv.py:679-680, 690-691). Any of the BN / bias / layer_scale inputs may
 * be NULL. */
int fvit_affine_fold(float* scale, float* shift, int32_t n, const float* bn_w, const float* bn_b,
                     const float* bn_mean, const float* bn_var, float eps, const float* bias,
                     const float* layer_scale, void* stream);

/* ---- PatchEmbed first convolution (fv.py:458-460): 3x3 stride 2 pad 1 on the fp32 NCHW image ----
 * (element strides sb, sc, sh, sw), y = relu?(conv * scale + shift) as fp16 rows of `cout` channels at
 * out_row_map[b*Ho*Wo + oh*Wo + ow]. With col_sum/col_sumsq: adds per-channel sum / sum of squares of
 * the raw convolution (train-mode BatchNorm statistics); `out` may then be NULL. */
int fvit_stem_conv_fwd(const float* x, int64_t sb, int64_t sc, int64_t sh, int64_t sw, int32_t B,
                       int32_t cin, int32_t H, int32_t W, const float* wgt, int32_t cout,
                       const float* scale, const float* shift, int32_t relu, const int32_t* out_row_map,
                       void* out, int64_t ldo, float* col_sum, float* col_sumsq, void* stream);

/* im2col of the same convolution for the tensor-core path: out[pixel][c*9 + r*3 + s] = (half) input tap
 * (zero outside the image and in the padding columns up to ldo); the 9*cin-deep contraction then runs as a
 * plain fvit_gemm with the BatchNorm/ReLU epilogue (kc = stem_ld, one K block up to cin = 7). Any channel count
 * 1 <= cin <= FVIT_STEM_MAX_CIN; ldo must be a multiple of 8 and at least stem_ld = round_up(9*cin, 32) (32 for
 * RGB). cin == 3 has a kernel of its own (one thread per pixel row); every other cin writes one 16-byte piece of a
 * row per thread. */
#define FVIT_STEM_MAX_CIN 64
int fvit_stem_im2col(const float* x, int64_t sb, int64_t sc, int64_t sh, int64_t sw, int32_t B, int32_t cin,
                     int32_t H, int32_t W, void* out, int32_t ldo, void* stream);

/* ---- LayerNorm forward over the channel dim of token rows (nn.LayerNorm eps 1e-5 fv.py:615,631,
 * 643-644, 690-691; timm LayerNorm2d eps 1e-6 fv.py:432,438), fused with the positional-embedding add
 * of PosEmbMLPSwinv1D (fv.py:366, 665, 676), with row gather (window partition / ct_dewindow,
 * fv.py:83-101) on the input and row scatter on the output.
 *   v   = x[in_map ? in_map[r] : r] + ( (r % group) >= skip ? add[(r % group) - skip] : 0 )
 *   wb[r] = v (optional fp32 write-back of the updated residual stream)
 *   out[out_map ? out_map[r] : r] = (half)((v - mean) * rstd * gamma + beta)
 * mean_out / rstd_out (optional) receive the row statistics and xhat_out (optional, fp16 [rows, ldxh])
 * the normalised pre-affine rows for the backward pass. */
int fvit_ln_fwd(const float* x, int64_t ldx, const int32_t* in_map, int32_t rows, int32_t C,
                const float* add, int32_t group, int32_t skip, float* wb, int64_t ldwb,
                const float* gamma, const float* beta, float eps, void* out, int64_t ldo,
                const int32_t* out_map, float* mean_out, float* rstd_out, void* xhat_out, int64_t ldxh,
                void* stream);

/* ---- attention core of WindowAttention.forward (fv.py:559-565) on a packed qkv matrix -------------
 * qkv fp16 [groups*S, 3*heads*head_dim] (q | k | v); for every group of S consecutive tokens and every
 * head: out = softmax(q k^T * scale + bias[head]) v, written fp16 to out[row, head*head_dim + d].
 * bias fp32 [heads, S, S] or NULL. probs_out (optional, fp32 [groups, heads, S, S]) saves P. */
int fvit_attn_core_fwd(const void* qkv, int64_t ldq, int32_t groups, int32_t S, int32_t heads,
                       int32_t head_dim, const float* bias, float scale, void* out, int64_t ldo,
                       float* probs_out, void* stream);

/* Tensor-core version of the same attention core (wgmma: S = QK^T and O = PV with fp32 accumulators
 * staged in shared memory, TMA-staged head slices, per-row softmax; scores and probabilities never
 * leave the SM). qkv fp16 [groups*S, 3*heads*hdp] with head_dim zero-padded to
 * hdp in {32, 64}; out fp16 [groups*S, heads*hdp]; S <= 128. bias fp32 [heads, S, S] or NULL. */
int fvit_attn_tc_fwd(const void* qkv, int64_t ldq, int32_t groups, int32_t S, int32_t heads, int32_t hdp,
                     const float* bias, float scale, void* out, int64_t ldo, void* stream);

/* The fused hierarchical-attention kernel (north star; WindowAttention.forward faster_vit.py:557-565 with the qkv Linear
 * of faster_vit.py:546): out = softmax((x Wq^T + bq)(x Wk^T + bk)^T * scale + bias)(x Wv^T + bv) per window and head
 * in ONE wgmma kernel. xn16 [groups*S, C] is the LayerNorm-ed fp16 activation (norm1 / hat_norm1 output, row stride
 * ldx), wqkv16 the head-padded packed qkv weight [3*heads*hdp, C] (fvit_cast_headpad_f16; row stride ldw), qkv_bias
 * its padded bias [3*heads*hdp] or NULL, bias the relative-position bias [heads, S, S] or NULL. S <= 128, hdp in
 * {32, 64}. out [groups*S, heads*hdp] as fvit_attn_tc_fwd. qkv_out (optional, [groups*S, 3*heads*hdp] fp16) receives
 * the projected q | k | v for the backward pass; when NULL the qkv matrix never exists in HBM. */
int fvit_hat_attn_fwd(const void* xn16, int64_t ldx, int32_t C, const void* wqkv16, int64_t ldw, const float* qkv_bias,
                      int32_t groups, int32_t S, int32_t heads, int32_t hdp, const float* bias, float scale, void* out,
                      int64_t ldo, void* qkv_out, int64_t ldq, void* stream);

/* Key-loop tensor-core attention core for window sequences longer than one 128-row tile (any-res level 2:
 * S = 12*12 + 4 = 148, faster_vit_any_res.py:805-817; 21k windows S = 196 .. 2304, faster_vit.py:1253-1418):
 * work item = (window, head, 128 query rows); key tiles of 128 are visited twice (row maxima, then probabilities and
 * O += P V in an fp32 shared-memory accumulator). Same qkv / out layout as fvit_attn_tc_fwd; bias [heads, S, S] fp32 is staged by TMA, so
 * S % 4 == 0 is required when a bias is given. lse (optional, [groups*S, heads] fp32) receives the log2-domain
 * log-sum-exp of the scaled, biased scores (saved for the backward pass). */
int fvit_attn_loop_fwd(const void* qkv, int64_t ldq, int32_t groups, int32_t S, int32_t heads, int32_t hdp,
                       const float* bias, float scale, void* out, int64_t ldo, float* lse, void* stream);

/* ---- training-mode BatchNorm2d (batch statistics; fv.py:459-462, 490-493, 925 under module.train()) ----
 * fvit_colstats_f32: sum[c] += sum_r x[rows[r]][c]; sumsq likewise (fp32 input, optional row list).
 * fvit_bn_finalize : from (sum, sumsq, count) -> biased var for normalisation, running statistics
 *   update (momentum, unbiased var), epilogue vectors scale = w*rstd*[ls], shift = (b - mean*w*rstd)*[ls],
 *   and mean / rstd for the backward pass.
 * fvit_affine_rows : y = act(x16[row]*scale + shift) * row_scale[row] (+ resid32[row]) over a row list,
 *   fp32/fp16 out (normalise + ReLU/GELU (+ stochastic-depth mask, + residual) of a raw convolution output). */
int fvit_colstats_f32(const float* x, int64_t ldx, const int32_t* rows, int32_t nrows, int32_t C, float* sum,
                      float* sumsq, void* stream);
int fvit_bn_finalize(const float* sum, const float* sumsq, float count, const float* w, const float* b, float eps,
                     float momentum, float* running_mean, float* running_var, const float* layer_scale,
                     float* scale, float* shift, float* mean_out, float* rstd_out, int32_t C, void* stream);
int fvit_affine_rows(const void* x16, int64_t ldx, const int32_t* rows, int32_t nrows, int32_t C,
                     const float* scale, const float* shift, int32_t act, const float* resid, int64_t ldr,
                     float* out32, int64_t ldo32, void* out16, int64_t ldo16, const float* row_scale, void* stream);
/* Pivoted statistics. One-pass fp32 sums of x and x^2 lose about 2^-24 * (mean/std)^2 of the variance per summed
 * term, which is percents once a channel's offset is ~100 std. Summing d = x - K with K near the batch mean removes
 * that loss:
 * fvit_colstats_pivot_f32: as fvit_colstats_f32 over d = x - K with K[c] = x[rows[0]][c], written to pivot[c].
 * fvit_bn_col_shift      : col_shift = (bias ? bias : 0) - pivot, the GEMM epilogue vector that makes a convolution
 *   GEMM write and sum d = conv + bias - pivot.
 * fvit_bn_finalize_pivot : fvit_bn_finalize from moments of d: batch mean = pivot + sum/n, var = sumsq/n - (sum/n)^2;
 *   the running statistics use the batch mean. shifted != 0: the rows later normalised are d themselves (a GEMM
 *   output whose col_shift subtracted the pivot), so shift and mean_out use sum/n; shifted == 0: they use the batch
 *   mean. */
int fvit_colstats_pivot_f32(const float* x, int64_t ldx, const int32_t* rows, int32_t nrows, int32_t C, float* pivot,
                            float* sum, float* sumsq, void* stream);
int fvit_bn_col_shift(const float* bias, const float* pivot, int32_t C, float* col_shift, void* stream);
int fvit_bn_finalize_pivot(const float* sum, const float* sumsq, const float* pivot, int32_t shifted, float count,
                           const float* w, const float* b, float eps, float momentum, float* running_mean,
                           float* running_var, const float* layer_scale, float* scale, float* shift, float* mean_out,
                           float* rstd_out, int32_t C, void* stream);

/* ---- positional MLPs (cpb_mlp: Linear(2,512)+ReLU+Linear(512,D, no bias); fv.py:223-225, 322-324) --
 * out[p][d] for P coordinate pairs; hidden_out (optional, [P,512]) saves the ReLU output. */
int fvit_cpb_mlp_fwd(const float* coords, int32_t P, const float* w0, const float* b0, const float* w1,
                     int32_t D, float* out, float* hidden_out, void* stream);
/* bias[h][r][c] = 16*sigmoid(table[index[(r-ng)*L + (c-ng)]][h]) for r,c >= ng = S-L, else 0
 * (PosEmbMLPSwinv2D.forward fv.py:276-299). S < L (ng < 0) crops the top-left of the L x L table. */
int fvit_attn_bias_fwd(const float* table, const int64_t* index, int32_t heads, int32_t S, int32_t L,
                       float* bias, void* stream);

/* ---- TokenInitializer.forward (fv.py:733-738; fvar.py:729-750): depthwise 3x3 (+bias) then AvgPool
 * (kh x kw, stride sh x sw) -> oh x ow carrier tokens per image, written to rows ct_row_map[...] of
 * `out`. The feature map is read through pix_map[(b*Hp + y)*Wp + x] -> row of xs (-1: zero pixel). */
int fvit_token_init_fwd(const float* xs, int64_t ldx, const int32_t* pix_map, int32_t B, int32_t Hp,
                        int32_t Wp, int32_t C, const float* w, const float* bias, int32_t kh, int32_t kw,
                        int32_t sh, int32_t sw, int32_t oh, int32_t ow, const int32_t* ct_row_map,
                        float* out, int64_t ldo, void* stream);
/* The same pooled values stored as the detection backbone reads them (dino/models/dino/fastervit.py:591): image b's
 * NCHW map reinterpreted as [oh*ow, C] tokens, value (c, p) -> token t, channel k with c*oh*ow + p = t*C + k, written to
 * row ct_row_map[b*oh*ow + t] of `out`. */
int fvit_token_init_nchw_fwd(const float* xs, int64_t ldx, const int32_t* pix_map, int32_t B, int32_t Hp,
                             int32_t Wp, int32_t C, const float* w, const float* bias, int32_t kh, int32_t kw,
                             int32_t sh, int32_t sw, int32_t oh, int32_t ow, const int32_t* ct_row_map,
                             float* out, int64_t ldo, void* stream);

/* ---- carrier -> window propagation (fv.py:697-700): xs[r] += gamma * xs[src_map[r]] (src_map < 0:
 * row untouched; gamma NULL = 1). */
int fvit_propagate_fwd(float* xs, int64_t ldx, const int32_t* src_map, int32_t rows, int32_t C,
                       const float* gamma, void* stream);

/* ---- head (fv.py:953-958): BatchNorm2d folded into AdaptiveAvgPool2d(1):
 * out[b][c] = (half)(mean_t xs[row_map[b*T + t]][c] * scale[c] + shift[c]) */
int fvit_pool_affine_fwd(const float* xs, int64_t ldx, const int32_t* row_map, int32_t B, int32_t T,
                         int32_t C, const float* scale, const float* shift, void* out, int64_t ldo,
                         void* stream);

/* forward_features (faster_vit.py:949-953): the BatchNorm-ed (scale/shift folded) last-level activation in the
 * reference's NCHW fp32 layout: out[b][c][t] = xs[row_map[b*T+t]][c] * scale[c] + shift[c]. */
int fvit_feature_map_fwd(const float* xs, int64_t ldx, const int32_t* row_map, int32_t B, int32_t T, int32_t C,
                         const float* scale, const float* shift, float* out_nchw, void* stream);

/* Backward of fvit_feature_map_fwd with a batch-statistics BatchNorm2d folded in: autograd of the level norms
 * (downstream/object_detection/dino/models/dino/fastervit.py:816-827 `norm_layer(xo)` under .train()) and of the
 * final `norm` (faster_vit.py:953) in forward_features. dy is the NCHW fp32 gradient [B, C, T] of the map; xs / row_map
 * address the token-major level activation as in the forward. Two passes:
 * fvit_feature_map_bwd_stats: s1[c] += sum_{b,t} dy, s2[c] += sum dy * xhat (xhat = (xs[row][c] - mean[c]) * rstd[c]),
 *   *amax = max(*amax, max |dy|) (fp32 bits compared as integers; zero it before the first output). mean == NULL is
 *   the mode without a BatchNorm (raw forward_levels maps): only amax; xs, rstd, s1, s2 may be NULL.
 * fvit_feature_map_bwd: g[row_map[b*T+t]][c] += S * dx with S = gs[0] and, BatchNorm mode, dx = w*rstd*(dy - s1/N -
 *   xhat*s2/N) (N = B*T), else dx = dy; rows outside row_map are untouched. dw[c] += s2*(*scalar), dbeta[c] +=
 *   s1*(*scalar) (BatchNorm mode, optional, scalar NULL = 1). g NULL: only dw / dbeta.
 * fvit_grad_scale_finalize: gs = {S, 1/S}, S = 2^floor(log2(target / *amax)) (the fvit_grad_scale_init rule over the
 *   maximum the stats passes of every requested output gathered). */
int fvit_feature_map_bwd_stats(const float* dy, const float* xs, int64_t ldx, const int32_t* row_map, int32_t B,
                               int32_t T, int32_t C, const float* mean, const float* rstd, float* s1, float* s2,
                               float* amax, void* stream);
int fvit_feature_map_bwd(const float* dy, const float* xs, int64_t ldx, const int32_t* row_map, int32_t B, int32_t T,
                         int32_t C, const float* mean, const float* rstd, const float* w, const float* s1,
                         const float* s2, const float* gs, const float* scalar, float* g, int64_t ldg, float* dw,
                         float* dbeta, void* stream);
int fvit_grad_scale_finalize(const float* amax, float target, float* gs, void* stream);
/* Backward of fvit_feature_map_fwd with a running-statistics BatchNorm2d folded in (eval-mode gradients of the level
 * norms and of `norm` in forward_features): g[row_map[b*T+t]][c] += S * w[c] * rstd[c] * dy[b][c][t] (S = gs[0], rstd
 * = rsqrt(running_var + eps)); w == rstd == NULL is the raw map (g += S * dy). Rows outside row_map are untouched.
 * dw[c] += s2[c] * (*scalar), dbeta[c] += s1[c] * (*scalar) with s1 = sum dy, s2 = sum dy * xhat from
 * fvit_feature_map_bwd_stats run with the running mean / rstd (scalar NULL = 1). g NULL: only dw / dbeta. Same 32 x 32
 * transposed tiles as fvit_feature_map_bwd; the apply reads no activation. */
int fvit_feature_map_eval_bwd(const float* dy, const int32_t* row_map, int32_t B, int32_t T, int32_t C,
                              const float* rstd, const float* w, const float* s1, const float* s2, const float* gs,
                              const float* scalar, float* g, int64_t ldg, float* dw, float* dbeta, void* stream);
/* Level outputs through a channel LayerNorm (timm LayerNorm2d, the MOTRv2 tracking backbone's output norms), in train
 * and eval mode alike. Pixel p = b*T + t reads the fp32 row xs[row_map[p]] (row_map NULL: row p; row stride ldx >= C).
 * fvit_feature_map_ln_fwd: out[b][c][t] = (x[c] - mean_p) * rstd_p * w[c] + b[c] with mean_p / rstd_p =
 *   rsqrt(var_p + eps) over the C channels of the pixel (biased variance, fp32, moments about the pixel's channel 0);
 *   mean[p], rstd[p] are written when given (both or neither: NULL in inference).
 * fvit_feature_map_ln_bwd: from the NCHW map gradient dy and the forward's mean / rstd, with xhat = (x - mean_p) * rstd_p:
 *   g[row_map[p]][c] += S * rstd_p * (w[c]*dy - mean_c(w*dy) - xhat * mean_c(w*dy*xhat)) (S = gs[0]; g NULL: none);
 *   dw[c] += (*scalar) * sum_p dy * xhat, dbeta[c] += (*scalar) * sum_p dy (both or neither; scalar NULL = 1), summed
 *   with float atomics. C <= 6144. */
int fvit_feature_map_ln_fwd(const float* xs, int64_t ldx, const int32_t* row_map, int32_t B, int32_t T, int32_t C,
                            const float* w, const float* b, float eps, float* out_nchw, float* mean, float* rstd,
                            void* stream);
int fvit_feature_map_ln_bwd(const float* dy, const float* xs, int64_t ldx, const int32_t* row_map, int32_t B,
                            int32_t T, int32_t C, const float* mean, const float* rstd, const float* w, const float* gs,
                            const float* scalar, float* g, int64_t ldg, float* dw, float* dbeta, void* stream);
/* Backward of forward_head (faster_vit.py:955-958: AdaptiveAvgPool2d(1) + flatten + Linear), fp32 throughout, from
 * dlogits [B, ncls] (row stride ldl). feats: the fp32 input, NCHW [B, C, T] (T = H*W) or pooled [B, C] (T = 1).
 * dfeats[b][c][t] = (sum_k dlogits[b][k] * W[k][c]) / T (written); dW[k][c] += sum_b dlogits[b][k] * pooled[b][c] with
 * pooled = mean_t feats, recomputed into pooled_ws [B*C] when T > 1; db[k] += sum_b dlogits[b][k]. W NULL: an
 * identity head (num_classes = 0, ncls == C), the pooling backward alone. Any of dfeats / dW / db may be NULL. */
int fvit_head_eval_bwd(const float* dlogits, int64_t ldl, int32_t B, int32_t ncls, const float* feats, int32_t C,
                       int32_t T, const float* W, float* pooled_ws, float* dfeats, float* dW, float* db, void* stream);

/* forward_head (faster_vit.py:955-958): AdaptiveAvgPool2d(1) + flatten of an NCHW fp32 map into the fp16 operand
 * [B, ldo] of the classifier GEMM. */
int fvit_nchw_pool_f16(const float* x, int32_t B, int32_t C, int32_t T, void* out16, int64_t ldo, void* stream);

/* ==== backward pass (fv.py has no backward code: the reference relies on autograd, train.py:879-896) ====
 * Activation gradients are fp16 tensors (or the fp32 residual-stream gradient) multiplied by a
 * power-of-two scale S kept in device memory, gs = {S, 1/S}; parameter gradients are fp32, un-scaled by
 * the `scalar` / alpha_ptr device scalars. Nothing synchronises with the host. */
/* gs[0] = 2^floor(log2(target / max|x|)), gs[1] = 1/gs[0] (x = d loss / d logits, n elements), clamped to
 * [2^-24, 2^40]; S = 1 when the maximum is 0 or inf. NaN elements are skipped (the maximum is that of the others):
 * a NaN loss gradient is left to the optimizer's non-finite check. */
int fvit_grad_scale_init(const float* x, int32_t n, float target, float* gs, void* stream);
/* out[i] = a[i*a_stride] * b[i*b_stride] (vectors of device scalars). */
int fvit_vec_mul(const float* a, int32_t a_stride, const float* b, int32_t b_stride, float* out, int32_t n,
                 void* stream);
/* out = {s, 1/s} with s = 2^-floor(log2(max|v|)) (normaliser of a layer-scale vector gamma, fv.py:637-655,
 * so that gamma*s is O(1) and fp16 products with gamma = 1e-5 do not underflow). */
int fvit_pow2_norm(const float* v, int32_t n, float* out, void* stream);
/* out16[r][c] = (half)(x[rows ? rows[r] : r][c] * colmul[c] * *scalar * row_scale[r]): tensor-core operand copy
 * of a fp32 gradient (colmul = layer scale, scalar = its normaliser, row_scale = stochastic-depth mask/keep;
 * all optional). fvit_colsum and fvit_bn_bwd take the same optional row_scale (indexed by r / by the g row). */
int fvit_cast_scale_f16(const float* x, int64_t ldx, const int32_t* rows, int32_t nrows, int32_t C,
                        const float* colmul, const float* scalar, void* out, int64_t ldo, const float* row_scale,
                        void* stream);
/* out[c] += *scalar * colmul[c] * sum_r a[a_rows ? a_rows[r] : r][c] * (b16 ? b16[r][c] : 1): bias, LayerNorm /
 * BatchNorm affine and layer-scale gradients. a is fp32 or fp16 (a_is_f16). */
int fvit_colsum(const void* a, int32_t a_is_f16, int64_t lda, const int32_t* a_rows, const void* b16, int64_t ldb,
                int32_t nrows, int32_t C, const float* colmul, const float* scalar, float* out, const float* row_scale,
                void* stream);
/* Entry of a residual-branch backward x += gamma * f(LN(x)) (fv.py:637-655) in one pass over the fp32 gradient
 * g [rows, C]: dz16 = half(g * colmul * *scalar * row_scale) (operand of the branch's last Linear), dbias[c] +=
 * *bias_alpha * sum_r dz16 (its bias gradient), dgamma[c] += *gamma_alpha * sum_r g * u16 * row_scale (layer-scale
 * gradient; u16 = saved branch output). dbias / u16+dgamma optional. Needs C % 8 == 0. */
int fvit_branch_grad(const float* g, int64_t ldg, int32_t rows, int32_t C, const float* colmul, const float* scalar,
                     const float* row_scale, void* dz16, int64_t lddz, const float* bias_alpha, float* dbias,
                     const void* u16, int64_t ldu, const float* gamma_alpha, float* dgamma, void* stream);
/* out[t - skip][c] += *scalar * sum_w a[w*group + t][c], skip <= t < group: gradient of a positional
 * embedding broadcast-added to every window (fv.py:366). */
int fvit_group_sum(const float* a, int64_t lda, int32_t ngroups, int32_t group, int32_t skip, int32_t C,
                   const float* scalar, float* out, void* stream);
/* LayerNorm backward for the forward of fvit_ln_fwd (same row maps): with gv = (use_g ? g[r] : 0) +
 * rstd[r]*(gamma*dy - mean(gamma*dy) - xhat*mean(gamma*dy*xhat)):  g[in_map ? in_map[r] : r] = gv (with
 * clear_moved, g[r] is zeroed when the source is another row — r must then index rows of g); dgamma[c] += *scalar*sum dy*xhat; dbeta[c] += *scalar*sum dy.
 * dy16 rows through dy_map (rows with dy_map < 0 are skipped). */
int fvit_ln_bwd(const void* dy16, int64_t lddy, const int32_t* dy_map, const void* xhat16, int64_t ldxh,
                const float* rstd, const float* gamma, int32_t rows, int32_t C, float* g, int64_t ldg,
                const int32_t* in_map, int32_t use_g, int32_t clear_moved, const float* scalar, float* dgamma,
                float* dbeta, void* stream);
/* Backward of the attention core (either forward kernel): recomputes P from q, k, bias; writes dq, dk, dv
 * (fp16, head-padded layout [rows, 3*heads*hdp], padding columns zero) and accumulates dbias[h][S][S]. */
int fvit_attn_core_bwd(const void* qkv, int64_t ldq, const void* dout, int64_t lddo, int32_t groups, int32_t S,
                       int32_t heads, int32_t head_dim, int32_t hdp, const float* bias, float scale, void* dqkv,
                       int64_t lddq, float* dbias, void* stream);
/* Tensor-core version for S <= 64 and hdp in {32, 64} (wgmma: S = QK^T, dP = dO V^T, then dV = P^T dO,
 * dK = dS^T Q, dQ = dS K with the P / dS tiles read as MN-major / K-major operands); same contract. */
int fvit_attn_tc_bwd(const void* qkv, int64_t ldq, const void* dout, int64_t lddo, int32_t groups, int32_t S,
                     int32_t heads, int32_t head_dim, int32_t hdp, const float* bias, float scale, void* dqkv,
                     int64_t lddq, float* dbias, void* stream);
/* Tensor-core backward for windows longer than the tile kernel takes, the mirror of fvit_attn_loop_fwd (any S with
 * S % 4 == 0; the training plans use it from 65 tokens on): any-res S = 148, the 24 x 24 / 32 x 32 / 48 x 48 windows of
 * the 21k models (fv.py:1253-1418, WindowAttention.forward fv.py:557-568 differentiated). Needs the forward's output
 * `out` (for delta = rowsum(dO * O)) and its log-sum-exp vector `lse`. Key tiles outside, query tiles inside; dV_j /
 * dK_j accumulate in registers over the query loop, the per-pair partial dQ_i = dS K_j is added to the row of the fp32
 * scratch matrix dq_scratch[groups * S, ld_scratch >= heads * hdp] its owning thread keeps (16-byte stores for the
 * first key tile, 16-byte reductions afterwards: no initialisation needed) and converted to fp16 at the end of the
 * item. Same dqkv / dbias contract as fvit_attn_core_bwd; dq_scratch holds no result afterwards. */
int fvit_attn_loop_bwd_long(const void* qkv, int64_t ldq, const void* dout, int64_t lddo, const void* out, int64_t ldo,
                            const float* lse, int32_t groups, int32_t S, int32_t heads, int32_t hdp, const float* bias,
                            float scale, void* dqkv, int64_t lddq, float* dbias, float* dq_scratch, int64_t ld_scratch,
                            void* stream);
/* dst (+)= *scalar * src with head padding removed from rows and/or columns (inverse of
 * fvit_cast_headpad_f16 for gradients). */
int fvit_unpad_heads_f32(const float* src, int64_t lds, float* dst, int64_t ldd, int32_t rows_src, int32_t cols_src,
                         int32_t hd, int32_t hdp, int32_t pad_rows, int32_t pad_cols, const float* scalar,
                         void* stream);
/* Backward of fvit_attn_bias_fwd: dtable[index][h] += *scalar * dbias * b*(1 - b/16), b = 16 sigmoid(table); with
 * S < L only the entries the forward kept. */
int fvit_attn_bias_bwd(const float* dbias, const float* bias, const int64_t* index, int32_t heads, int32_t S,
                       int32_t L, const float* scalar, float* dtable, void* stream);
/* Backward of fvit_cpb_mlp_fwd (needs the saved hidden activations): accumulates dw0 [512,2], db0 [512],
 * dw1 [D,512] from dout [P,D] * *scalar. */
int fvit_cpb_mlp_bwd(const float* coords, int32_t P, const float* w1, const float* hidden, const float* dout,
                     int32_t D, const float* scalar, float* dw0, float* db0, float* dw1, void* stream);
/* Backward of the head's BatchNorm2d (batch statistics) + AdaptiveAvgPool2d(1) (fv.py:953-958): from
 * dpool [B,C] writes g[row(b,t)] and accumulates the BN weight/bias gradients; s1/s2 are [C] scratch. */
int fvit_pool_bn_bwd(const float* xs, int64_t ldx, const int32_t* rows, int32_t B, int32_t T, int32_t C,
                     const float* mean, const float* rstd, const float* w, const float* dpool, int64_t lddp,
                     float* s1, float* s2, const float* scalar, float* g, int64_t ldg, float* dw, float* dbeta,
                     void* stream);
/* dst[map[r]] += src[r] (fp32 rows; ct_dewindow backward, fv.py:96-101); rows with map[r] < 0 are skipped. The add is
 * a plain read-modify-write (no atomics): `map` must be injective on its non-negative entries. */
int fvit_scatter_add_rows(const float* src, int64_t lds, float* dst, int64_t ldd, const int32_t* map, int32_t rows,
                          int32_t C, void* stream);
/* BatchNorm2d (batch statistics) backward over row lists: dy = gin (fp32 or fp16) * colmul, masked by the
 * ReLU derivative when act == FVIT_ACT_RELU (sign of xhat*w + b); out16[o_rows[r]] = w*rstd*(dy - mean(dy) -
 * xhat*mean(dy*xhat)); dw += *scalar * sum dy*xhat; db += *scalar * sum dy. s1/s2: [C] scratch. */
int fvit_bn_bwd(const void* gin, int32_t g_is_f16, int64_t ldg, const int32_t* g_rows, const void* raw16, int64_t ldr,
                const int32_t* r_rows, int32_t nrows, int32_t C, const float* mean, const float* rstd, const float* w,
                const float* b, int32_t act, const float* colmul, float* s1, float* s2, const float* scalar, void* out16,
                int64_t ldo, const int32_t* o_rows, float* dw, float* db, const float* row_scale, void* stream);

/* ---- Eval-mode gradients: the backward of model(x) under .eval() ----
 * An eval forward with grad enabled runs the inference launch list unchanged and records the input; its backward
 * recomputes that forward as a saving train-style forward whose BatchNorms use their running statistics (no drop
 * path, no statistics update), then runs the training backward with the three entry points below. The cost of one
 * backward is therefore one extra forward on top of a training step's forward + backward; a forward with no backward
 * costs what an inference forward costs. */
/* BatchNorm2d on running statistics, backward over row lists: xhat = (raw - mean) * rsqrt(var + eps),
 * dy = gin (fp32 or fp16) * colmul, masked by the ReLU derivative when act == FVIT_ACT_RELU (sign of xhat*w + b);
 * out16[o_rows[r]] = w*rsqrt(var+eps)*dy; dw += *scalar * sum dy*xhat; db += *scalar * sum dy. One pass, no scratch.
 * With C % 4 == 0, 16-byte aligned rows and every leading dimension a multiple of 8 elements (4 for fp32 gin), the
 * padding columns of an out16 row up to the next multiple of 8 are written as zeros. */
int fvit_bn_eval_bwd(const void* gin, int32_t g_is_f16, int64_t ldg, const int32_t* g_rows, const void* raw16,
                     int64_t ldr, const int32_t* r_rows, int32_t nrows, int32_t C, const float* mean, const float* var,
                     float eps, const float* w, const float* b, int32_t act, const float* colmul, const float* scalar,
                     void* out16, int64_t ldo, const int32_t* o_rows, float* dw, float* db, void* stream);
/* Backward of the head's running-statistics BatchNorm2d + AdaptiveAvgPool2d(1) (fv.py:953-958 under .eval()):
 * g[row(b,t)][c] = dpool[b][c] / T * w[c] * rsqrt(var[c] + eps) (written); dw += *scalar * sum_b dpool * mean_t xhat;
 * dbeta += *scalar * sum_b dpool. Row conventions as fvit_pool_bn_bwd. */
int fvit_pool_bn_eval_bwd(const float* xs, int64_t ldx, const int32_t* rows, int32_t B, int32_t T, int32_t C,
                          const float* mean, const float* var, float eps, const float* w, const float* dpool,
                          int64_t lddp, const float* scalar, float* g, int64_t ldg, float* dw, float* dbeta,
                          void* stream);
/* Image gradient of the stem's first convolution (3x3, stride 2, pad 1, 3 input channels, fv.py:458):
 * dx[b][ci][y][x] = *scalar * sum w[co][ci][ky][kx] * dz[(b*H1 + oy)*W1 + ox][co] over y = 2*oy - 1 + ky,
 * x = 2*ox - 1 + kx, with H1 = (H+1)/2, W1 = (W+1)/2. dz: fp16 rows of stride lddz; w: fp32 [cout, 3, 3, 3],
 * cout <= 512; dx: fp32 NCHW [B, 3, H, W], every element written. A gather (no atomics): deterministic. */
int fvit_stem_conv_dgrad(const void* dz16, int64_t lddz, int32_t B, int32_t H, int32_t W, const float* wgt,
                         int32_t cout, const float* scalar, float* dx, void* stream);
/* The image gradient of the same convolution for any channel count, second half: the tap products come as fp32 rows
 * dcol[(b*H1 + oy)*W1 + ox][ci*9 + ky*3 + kx] (row stride ldc >= 9*cin; the fvit_gemm dz . W1 with W1 the conv weight
 * viewed as [cout, 9*cin], scaled as the gradient needs), and dx[b][ci][y][x] = sum of the 1, 2 or 4 entries whose
 * tap reads (y, x). dx: fp32 NCHW [B, cin, H, W], every element written, 1 <= cin <= FVIT_STEM_MAX_CIN. A gather
 * (no atomics): deterministic. The plans use it for in_chans != 3 and fvit_stem_conv_dgrad for 3. */
int fvit_stem_col2im(const float* dcol, int64_t ldc, int32_t B, int32_t cin, int32_t H, int32_t W, float* dx,
                     void* stream);
/* dst[co][ci][tap] += src[co][tap * cin + ci] (row stride ld): the b_ntaps weight-gradient GEMM output ->
 * nn.Conv2d layout. */
int fvit_unpack_conv_grad(const float* src, int32_t ld, float* dst, int32_t cout, int32_t cin, void* stream);
/* TokenInitializer backward (fv.py:733-738): gx[pixel rows] += d/dx, dw [C,9], dbias [C] from the carrier-row
 * gradients g[ct_row_map[...]]; x16 = fp16 copy of the level input tokens (same row layout as xs). */
int fvit_token_init_bwd(const float* g, int64_t ldg, const void* x16, int64_t ldx, const int32_t* pix_map,
                        const int32_t* ct_row_map, int32_t B, int32_t Hp, int32_t Wp, int32_t C, const float* w,
                        int32_t kh, int32_t kw, int32_t sh, int32_t sw, int32_t oh, int32_t ow, const float* scalar,
                        float* gx, int64_t ldgx, float* dw, float* dbias, void* stream);
/* Backward of fvit_propagate_fwd (fv.py:697-700): g[src_map[r]] += gamma*g[r]; dgamma += *scalar*sum g[r]*xs[src_map[r]]. */
int fvit_propagate_bwd(float* g, int64_t ldg, const float* xs, int64_t ldx, const int32_t* src_map, int32_t rows, int32_t C,
                       const float* gamma, const float* scalar, float* dgamma, void* stream);

/* ---- Data-only backward: the activation gradient through a stage whose parameters get no gradient ----
 * (a frozen prefix that an image gradient crosses; an eval-mode input gradient with the parameters frozen). The plans
 * then emit the data-gradient GEMMs and the attention-core backward (dbias = NULL) as they are, fvit_cast_scale_f16
 * for the branch entry, fvit_propagate_bwd with dgamma = NULL, and the three entry points below in place of
 * fvit_bn_eval_bwd / fvit_ln_bwd / fvit_token_init_bwd: the same arithmetic for the data gradient, no parameter sums. */
/* Running-statistics BatchNorm2d, data gradient alone: out16[o_rows[r]][c] = scale[c] * colmul[c] * *scalar * dy with
 * dy = gin[g_rows[r]][c] (fp32 or fp16), zeroed where act == FVIT_ACT_RELU and raw16[r_rows[r]][c] * scale[c] +
 * shift[c] <= 0. scale / shift are the forward's folded BatchNorm (fvit_affine_fold: w * rsqrt(var + eps) and
 * b - mean * scale); colmul, scalar, the row maps optional; raw16 / shift only read for the ReLU mask. A row whose map
 * entry is negative is skipped. One streaming pass, no reductions, no atomics; 16-byte accesses and zeroed padding
 * columns under the layout conditions of fvit_bn_eval_bwd. */
int fvit_bn_eval_dgrad(const void* gin, int32_t g_is_f16, int64_t ldg, const int32_t* g_rows, const void* raw16,
                       int64_t ldr, const int32_t* r_rows, int32_t nrows, int32_t C, const float* scale,
                       const float* shift, int32_t act, const float* colmul, const float* scalar, void* out16,
                       int64_t ldo, const int32_t* o_rows, void* stream);
/* The g update of fvit_ln_bwd without dgamma / dbeta (same dy_map / in_map / use_g / clear_moved conventions). */
int fvit_ln_dgrad(const void* dy16, int64_t lddy, const int32_t* dy_map, const void* xhat16, int64_t ldxh,
                  const float* rstd, const float* gamma, int32_t rows, int32_t C, float* g, int64_t ldg,
                  const int32_t* in_map, int32_t use_g, int32_t clear_moved, void* stream);
/* The gx update of fvit_token_init_bwd without dw / dbias (and so without the fp16 copy of the level input). */
int fvit_token_init_dgrad(const float* g, int64_t ldg, const int32_t* pix_map, const int32_t* ct_row_map, int32_t B,
                          int32_t Hp, int32_t Wp, int32_t C, const float* w, int32_t kh, int32_t kw, int32_t sh,
                          int32_t sw, int32_t oh, int32_t ow, float* gx, int64_t ldgx, void* stream);
/* fvit_token_init_bwd / fvit_token_init_dgrad for the carrier tokens of fvit_token_init_nchw_fwd: the gradient of pooled
 * value (c, p) of image b is channel (c*oh*ow + p) % C of row ct_row_map[b*oh*ow + (c*oh*ow + p) / C]. */
int fvit_token_init_nchw_bwd(const float* g, int64_t ldg, const void* x16, int64_t ldx, const int32_t* pix_map,
                             const int32_t* ct_row_map, int32_t B, int32_t Hp, int32_t Wp, int32_t C, const float* w,
                             int32_t kh, int32_t kw, int32_t sh, int32_t sw, int32_t oh, int32_t ow, const float* scalar,
                             float* gx, int64_t ldgx, float* dw, float* dbias, void* stream);
int fvit_token_init_nchw_dgrad(const float* g, int64_t ldg, const int32_t* pix_map, const int32_t* ct_row_map, int32_t B,
                               int32_t Hp, int32_t Wp, int32_t C, const float* w, int32_t kh, int32_t kw, int32_t sh,
                               int32_t sw, int32_t oh, int32_t ow, float* gx, int64_t ldgx, void* stream);

/* ---- optimizer step on the flat gradient buffer (SURVEY §8 f.1; train.py:879-899) -----------------------
 * Replaces, for the training loop either side of loss.backward(): GradScaler.unscale_ + the non-finite check,
 * dispatch_clip_grad(..., mode='norm') (`--clip-grad 5.0`), optimizer.step() for `--opt adamw` / `--opt lamb`
 * (TRAINING.md:28,105) and ModelEmaV2.update (train.py:898-899).
 *
 * Every parameter is a segment s: gradients and moments live in flat fp32 buffers at element offset seg_off[s]
 * (the layout the backward pass produces), parameters / EMA copies are addressed through per-segment device
 * pointer tables (seg_p / seg_ema: int64 addresses). `chunks` is a device int32 [nchunks][4] table
 * {segment, first element within the segment, element count (<= 2^31), 0}; one CTA per chunk. seg_hp is fp32
 * [nseg][2] = {lr, weight_decay}. scal is a persistent device fp32 [8] block: [0] gradient norm, [1] skip flag
 * (non-finite gradients), [2] gradient multiplier (unscale * clip), [3] steps taken, [4] 1-beta1^t, [5] 1-beta2^t. */
/* flat[seg_off[s] + i] = ((float*)seg_src[s])[i]: gathers per-tensor gradients that are not already flat. */
int fvit_optim_gather_f32(const int32_t* chunks, int32_t nchunks, const int64_t* seg_src, const int64_t* seg_off,
                          float* flat, void* stream);
/* partials[2c] = sum of squares of chunk c of g, partials[2c+1] = count of non-finite values. */
int fvit_optim_sqnorm(const int32_t* chunks, int32_t nchunks, const int64_t* seg_off, const float* g, float* partials,
                      void* stream);
/* Reduces the partials (nchunks may be 0: no norm) and updates scal: norm = sqrt(sum)/ *grad_scale; skip if any
 * non-finite or *found_inf != 0; multiplier = (1 / *grad_scale) * min(1, max_norm / (norm + clip_eps)) (max_norm <= 0:
 * no clipping; clip_eps = 1e-6 is torch.nn.utils.clip_grad_norm_, 0 is timm Lamb's max_grad_norm); the step
 * counter and bias corrections advance unless skipped. grad_scale / found_inf: optional device scalars
 * (torch.amp.GradScaler's). */
int fvit_optim_prepare(const float* partials, int32_t nchunks, const float* grad_scale, const float* found_inf,
                       float max_norm, float clip_eps, double beta1, double beta2, float* scal, void* stream);
/* torch.optim.AdamW step (decoupled weight decay, bias correction); seg_ema != NULL additionally applies
 * ema = ema_decay * ema + (1 - ema_decay) * p_new in the same pass. */
int fvit_optim_adamw(const int32_t* chunks, int32_t nchunks, const int64_t* seg_p, const int64_t* seg_off,
                     const float* seg_hp, const float* g, float* m, float* v, float beta1, float beta2, float eps,
                     const float* scal, const int64_t* seg_ema, float ema_decay, void* stream);
/* timm.optim.Lamb step in two passes: stage 1 updates the moments, writes the un-trusted update u (own flat
 * buffer) and accumulates per-segment sum p^2 / sum u^2 into seg_norms [nseg][2] (zeroed by the caller);
 * stage 2 applies p -= lr * trust * u with trust = ||p||/||u|| (segments with weight decay, or all with
 * always_adapt; min(trust, 1) with trust_clip) and the optional fused EMA. */
int fvit_optim_lamb_stage1(const int32_t* chunks, int32_t nchunks, const int64_t* seg_p, const int64_t* seg_off,
                           const float* seg_hp, const float* g, float* u, float* m, float* v, float beta1,
                           float beta2, float eps, const float* scal, float* seg_norms, void* stream);
int fvit_optim_lamb_stage2(const int32_t* chunks, int32_t nchunks, const int64_t* seg_p, const int64_t* seg_off,
                           const float* seg_hp, const float* u, const float* seg_norms, int32_t trust_clip,
                           int32_t always_adapt, const float* scal, const int64_t* seg_ema, float ema_decay,
                           void* stream);
/* ModelEmaV2.update: ((float*)seg_ema[s])[i] = decay * ema + (1 - decay) * ((float*)seg_src[s])[i]. */
int fvit_optim_ema(const int32_t* chunks, int32_t nchunks, const int64_t* seg_ema, const int64_t* seg_src, float decay,
                   void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FVIT_H_ */
