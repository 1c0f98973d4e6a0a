/* ns2_b200.h — C ABI of libns2b200.so: the sm_90a kernels behind the NaturalSpeech2 denoiser hot path.
 *
 * The reference (lucidrains/naturalspeech2-pytorch @ 659bec7) has no FFI of its own; its boundary for this
 * path is Python (nn.Module classes).  Each entry point below replaces the PyTorch library calls the
 * reference makes at the cited lines (paths relative to the reference repo; ns2.py =
 * naturalspeech2_pytorch/naturalspeech2_pytorch.py).  INTEGRATION.md shows the ctypes binding.
 *
 * Conventions
 *  - plain pointers and sizes only; all pointers are DEVICE pointers owned by the caller;
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*), never allocates device
 *    memory, never synchronises, and is re-entrant;
 *  - return value 0 = success, negative = error (ns2_last_error() gives a thread-local message);
 *  - activations are token-major (batch, position, channel) with the channel contiguous;
 *  - "bf16" buffers hold IEEE bfloat16, "f32" IEEE binary32, codes are int64 (as in the reference).
 */
#ifndef NS2_H100_H_
#define NS2_H100_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NS2_ABI_VERSION 9

typedef void* ns2_stream_t; /* cudaStream_t */

const char* ns2_last_error(void);
int ns2_abi_version(void);
/* Size the persistent grids of every kernel for at most `sms` SMs (rounded down to an even count; 0 = all SMs, the
 * default).  The GEMM / attention kernels run one CTA per SM for the whole launch, so a concurrent kernel that
 * holds a few SMs - NCCL's all-reduce of the gradients during the backward pass (ns2.py:1723-1726, 1886) - would delay
 * whole CTAs by a full tile loop; leaving those SMs out of the grid avoids that.  Returns the previous limit. */
int ns2_set_sm_limit(int sms);

/* ------------------------------------------------------------------------------------------------
 * 1. Segmented wgmma GEMM with fused epilogues.
 *
 * Computes, for every group g, batch b, position n and output channel j
 *     acc_a[b,n,j] = sum over segments s with segs[s].acc == a, k < segs[s].k_len of
 *                    A[b, n - segs[s].shift_units*dil[g], g*a_group_col_stride + segs[s].a_col_off + k]
 *                  * B[g*b_group_row_stride + j, segs[s].b_col_off + k]
 * where rows of A with a negative (or >= a_rows) position read as zero — this is the causal left padding
 * of CausalConv1d (ns2.py:583-595): a k=3 dilated causal conv is three segments with shift_units 2,1,0.
 * A Linear layer (nn.Linear: ns2.py:1021,1024,1051-1053,783) is one segment with shift 0.  A "same"-padded Conv1d
 * (kernel 2p+1, padding p: SpeechPromptEncoder ns2.py:316-320) is 2p+1 segments with shift_units p, p-1, ..., -p.
 *
 * Epilogues (all accumulate in fp32):
 *   NS2_EPI_BF16     out_bf16 = acc0 + bias
 *   NS2_EPI_F32      out_f32  = acc0 + bias (+ resid_f32)           residual add of ns2.py:799,805,809;
 *                    with resid == out (same row stride) the sum is formed by a TMA reduce-add into out
 *                    (one fp32 add of the same operands) and resid is never loaded
 *   NS2_EPI_GEGLU    out_bf16[j] = gelu_erf(acc0[gate j] + bias) * (acc0[val j] + bias)   ns2.py:1004-1007;
 *                    B rows must be packed so that each 256-row tile holds 128 value rows followed by
 *                    the 128 matching gate rows (see pack_geglu_weight in the Python host code);
 *                    `n` counts packed B rows (2x the number of output channels)
 *   NS2_EPI_WAVENET  y = (acc0 + bias)*gamma[b,j] + beta[b,j]; out_bf16 = tanh(y)*sigmoid(y) + acc1 + bias1
 *                    the WavenetResBlock body ns2.py:619-636 (acc0 = dilated conv, acc1 = res_conv);
 *                    gamma = film[b*film_batch_stride + g*film_group_stride + j], beta = gamma + n;
 *                    bias1 = bias + bias1_off.
 * All k_len must be multiples of 64 unless the segment ends at the last column of A and B.
 *
 * row_lens: a batch of sequences of different lengths, padded at the end: batch b's rows [0, row_lens[b]) are the
 * sample, the rest padding.  Device int32 (a_batches), each value clamped to [1, a_rows]; NULL = every row.  Only the
 * 128-row tiles that start before row_lens[b] are computed and stored (ceil(row_lens[b] / 128) tiles of batch b per
 * group and n-tile); every row of those tiles, including the rows at or past row_lens[b] inside the last one, is
 * bit-identical to the call without row_lens.  Rows of the other tiles are left untouched: neither written nor, with
 * the F32 epilogue's in-place residual, reduce-added.  A computed row reads A rows of its own tile and, through causal
 * shifts, earlier ones, so rows in untouched tiles (whatever they hold, NaN included) reach no computed row unless a
 * negative shift_units (an anti-causal tap) reads past the tile; callers must not pass such segments with padding that
 * is not finite.  With row_lens, a_batches must be <= NS2_GEMM_ROW_LENS_MAX_BATCHES (the lengths and their prefix sums
 * live in the kernel's shared memory); a larger batch is an error and nothing is launched.
 * ------------------------------------------------------------------------------------------------ */
enum { NS2_EPI_BF16 = 0, NS2_EPI_F32 = 1, NS2_EPI_GEGLU = 2, NS2_EPI_WAVENET = 3 };
#define NS2_GEMM_MAX_SEGS 12 /* a k=9 convolution (SpeechPromptEncoder, ns2.py:316-320) is 9 segments */
#define NS2_GEMM_MAX_GROUPS 8
#define NS2_GEMM_ROW_LENS_MAX_BATCHES 64

typedef struct ns2_gemm_seg {
  int32_t a_col_off;   /* first A column of this segment (within the group's column window) */
  int32_t b_col_off;   /* first B column (K index in the packed weight) */
  int32_t k_len;       /* reduction length */
  int32_t shift_units; /* row shift = shift_units * dil[group] */
  int32_t acc;         /* accumulator id, 0 or 1 */
} ns2_gemm_seg;

typedef struct ns2_gemm_args {
  const void* A;           /* bf16 (a_batches, a_rows, a_cols) */
  int64_t a_row_stride;    /* elements */
  int64_t a_batch_stride;  /* elements */
  int32_t a_batches, a_rows, a_cols;
  const void* B;           /* bf16 packed weights (b_rows, b_cols), K contiguous */
  int64_t b_row_stride;    /* elements */
  int32_t b_rows, b_cols;
  int32_t n;               /* B rows (accumulator columns) per group */
  int32_t groups;          /* >= 1; independent problems sharing the launch */
  int32_t a_group_col_stride;
  int32_t b_group_row_stride;
  int32_t out_group_col_stride;
  int32_t dil[NS2_GEMM_MAX_GROUPS];
  int32_t num_segs;
  ns2_gemm_seg segs[NS2_GEMM_MAX_SEGS];
  int32_t epilogue;
  const float* bias;       /* indexed like B rows (group offset = g*b_group_row_stride); may be NULL */
  int32_t bias1_off;       /* WAVENET: offset of the res_conv bias inside `bias` */
  void* out;               /* bf16 or f32, row (b*a_rows + n) */
  int64_t out_row_stride;  /* elements */
  const float* resid;      /* F32 epilogue: optional residual, same row indexing as out */
  int64_t resid_row_stride;
  const float* film;       /* WAVENET: FiLM table */
  int64_t film_batch_stride;
  int32_t film_group_stride;
  int32_t flags;           /* 0, or NS2_GEMM_FLAG_*; any other bit is an error */
  const int32_t* row_lens; /* optional (a_batches) row counts; NULL = every row */
} ns2_gemm_args;

#define NS2_GEMM_FLAG_SKIP_EPILOGUE 1  /* measurement aid: run the TMA/MMA mainloop only, write nothing */
#define NS2_GEMM_FLAG_SILU 4 /* BF16 / F32 epilogues: out = silu(acc + bias) (+ resid) — Conv1d + nn.SiLU of the prompt
                               encoder (ns2.py:316-320) and CausalConv1d + SiLU of the phoneme encoder (ns2.py:255-257) */

int ns2_gemm(const ns2_gemm_args* args, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 1b. Weight gradient of a Linear / CausalConv1d tap (autograd's grad_weight = grad_output^T @ input; the reference
 *     reaches it through loss.backward(), README.md:63, ns2.py:1886):
 *        dW[g][n, k] += sum_{b, m} dY[b, m, g*dy_group_col_stride + n] * X[b, m - shift_units*dil[g], g*x_group_col_stride + x_col_off + k]
 *     dY / X: bf16 token-major activations (batches, rows, cols); dW: fp32, ACCUMULATED into (reduce-add), row stride
 *     dw_row_stride, group g at row g*dw_group_row_stride.  n, k multiples of 32 (n a multiple of 128 when groups > 1).
 *     Positions outside [0, rows) of a shifted tap contribute zero (the conv's causal padding).  splits = 0: automatic.
 * ------------------------------------------------------------------------------------------------ */
typedef struct ns2_wgrad_args {
  const void* dY; int64_t dy_row_stride, dy_batch_stride; int32_t dy_cols;
  const void* X;  int64_t x_row_stride, x_batch_stride;  int32_t x_cols;
  int32_t batches, rows;
  int32_t n, k;
  int32_t groups, dy_group_col_stride, x_group_col_stride, x_col_off;
  int32_t dil[NS2_GEMM_MAX_GROUPS];
  int32_t shift_units;
  float* dW; int64_t dw_row_stride; int32_t dw_group_row_stride;
  int32_t splits;
} ns2_wgrad_args;

int ns2_wgrad(const ns2_wgrad_args* args, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 1c. A conv followed by a Linear with nothing between them, folded into one conv pack: the transformer feed-forward's
 *     CausalConv1d and output projection (FeedForward, ns2.py:1019-1024).  For each of `layers` stacked layers
 *        out[l][o, t*i_pad + c] = bf16( sum_d w2[l][o, d] * wc[l][d, c, t] )   (0 for i <= c < i_pad)
 *        bias_out[l][o]         = sum_d w2[l][o, d] * bc[l][d] + b2[l][o]
 *     w2 (layers, o, k), wc (layers, k, i, taps) (Conv1d's (out, in, taps) layout), bc (layers, k), b2 (layers, o):
 *     contiguous fp32.  out: bf16 (layers, o, taps*i_pad), tap-major like every conv pack; bias_out fp32 (layers, o).
 *     fp32 FMA accumulation (no TF32), one rounding to bf16.
 * ------------------------------------------------------------------------------------------------ */
int ns2_fold_conv_linear(const float* w2, const float* wc, const float* bc, const float* b2, int32_t layers, int32_t o,
                         int32_t k, int32_t i, int32_t taps, int32_t i_pad, void* out_bf16, float* bias_out,
                         ns2_stream_t stream);

/* One dropout site's parameters (training only): seed, site and drop probability p.  The attention calls of section 2
 * take them through a pointer in their argument structs (NULL = no dropout); section 2b gives the keep rule. */
typedef struct ns2_dropout {
  uint64_t seed;
  uint32_t site;
  float p;
} ns2_dropout;

/* ------------------------------------------------------------------------------------------------
 * 2. Non-causal flash attention forward (Attend.forward, attend.py:112-155 with causal=False).
 *    q/k/v: bf16, head h lives in columns [h*64, h*64+64) of each row; dim_head must be 64.
 *    out[b, i, h*64:(h+1)*64] = softmax_j(q_i . k_j * scale) @ v   (bf16)
 *    With kv_lens, q_lens and dropout NULL (a zero-initialised struct's optional fields) this is the unmasked,
 *    dropout-free attention the denoiser runs (mask=None, dropout=0, SURVEY T9).
 *  kv_lens: key padding for a batch of sequences of different lengths: sample b attends to keys [0, kv_lens[b]) only —
 *    Attend with a key-padding mask (attend.py:123-129, 140-142: masked scores -> -max, i.e. probability 0), the `mask`
 *    that PhonemeEncoder (ns2.py:275), SpeechPromptEncoder's Transformer (ns2.py:1110-1115) and the perceiver /
 *    predictor cross attentions (ns2.py:572-577, 457-466) would pass for padded batches.
 *    Device int32 (batches); each value is clamped to [1, kv_len] (callers should reject others).
 *    K / V rows at or past kv_lens[b] are never weighted, but they must be FINITE: their probability is exactly 0 and
 *    0 * V is still formed (V = NaN or inf there would reach the output).
 *    Query rows are not masked: rows a caller treats as padding get finite, meaningless output.
 *    Sample b's output rows are bit-identical to a call on that sample alone with kv_len = kv_lens[b] and no kv_lens.
 *  q_lens: query padding: sample b's queries [0, q_lens[b]) are the sample, the rest padding (device int32 (batches),
 *    each value clamped to [1, q_len]).  A 128-query tile that starts at or past q_lens[b] does nothing: its out rows
 *    and lse entries are left untouched.  Every row of the other tiles, including rows at or past q_lens[b] inside the
 *    last one, is bit-identical to the call without q_lens and the same kv_lens (or none).  Self-attention over padded
 *    sequences passes the same lengths as kv_lens and q_lens; cross-attention to unpadded keys passes q_lens only.
 *    Q rows of skipped tiles are never loaded, so they may hold anything.
 *  q_lens / kv_lens with a dropout of p > 0 is an error, nothing launched.
 *  dropout: dropout on the softmax probabilities (Attend, attend.py:106 SDPA dropout_p, attend.py:149 attn_dropout):
 *    out = ((P (.) M) V) / (1 - p); lse as without dropout (undropped probabilities, bit-identical).  p = 0 gives the
 *    bits of dropout == NULL.
 * ------------------------------------------------------------------------------------------------ */
typedef struct ns2_attn_args {
  const void* q; int64_t q_row_stride, q_batch_stride;
  const void* k; int64_t k_row_stride, k_batch_stride;
  const void* v; int64_t v_row_stride, v_batch_stride;
  void* out;     int64_t o_row_stride, o_batch_stride;
  int32_t batches, heads, q_len, kv_len, dim_head;
  float scale;
  float* lse;    /* optional (batches, heads, q_len) f32: log2-domain log-sum-exp of the scaled score rows,
                    saved for ns2_attn_bwd */
  const int32_t* kv_lens;       /* optional (batches) key counts; NULL = every key */
  const ns2_dropout* dropout;   /* optional; NULL = no dropout */
  const int32_t* q_lens;        /* optional (batches) query counts; NULL = every query */
} ns2_attn_args;

int ns2_attn_fwd(const ns2_attn_args* args, ns2_stream_t stream);

/* Backward of the above (autograd of F.scaled_dot_product_attention, reached from loss.backward(), ns2.py:1886):
 *   dq_accum (batches, q_len, heads*64) f32, contiguous: dQ is ADDED to it (every key tile adds its share; zero it for
 *   a plain gradient);
 *   dk / dv: bf16, same layout conventions as k / v;  lse from ns2_attn_fwd;  delta: scratch (batches, heads, q_len) f32.
 *   dropout: the forward's dropout parameters; the mask is regenerated from (seed, site, b, h, q, k):
 *   dV = (P (.) M)^T dO / (1 - p), dP = (dO V^T) (.) M / (1 - p), dS = P (.) (dP - D), D from the dropped output o.
 *   p = 0 gives the bits of dropout == NULL.
 *   kv_lens: the forward's kv_lens.  Sample b's dk / dv rows [0, kv_lens[b]) are bit-identical to a call on that sample
 *   alone with kv_len = kv_lens[b]; its rows past kv_lens[b] are written as exact zeros, and nothing from them reaches
 *   dq_accum.  K / V rows past kv_lens[b] must be finite (as for the forward).  With a dropout of p > 0 an error. */
typedef struct ns2_attn_bwd_args {
  const void* q; int64_t q_row_stride, q_batch_stride;
  const void* k; int64_t k_row_stride, k_batch_stride;
  const void* v; int64_t v_row_stride, v_batch_stride;
  const void* o; int64_t o_row_stride, o_batch_stride;
  const void* d_o; int64_t do_row_stride, do_batch_stride;
  const float* lse;
  float* delta;
  float* dq_accum;
  void* dk; int64_t dk_row_stride, dk_batch_stride;
  void* dv; int64_t dv_row_stride, dv_batch_stride;
  int32_t batches, heads, q_len, kv_len, dim_head;
  float scale;
  const ns2_dropout* dropout;   /* optional; NULL = no dropout */
  const int32_t* kv_lens;       /* optional (batches) key counts; NULL = every key */
} ns2_attn_bwd_args;

int ns2_attn_bwd(const ns2_attn_bwd_args* args, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 2b. Dropout (training only).  One site's parameters: a 64-bit seed (Philox4x32-10 key = its low / high 32 bits),
 *     the site number (one per dropout site of a forward call, reused by its backward) and the drop probability p.
 *     An element is kept iff its Philox word is >= min(floor(p 2^32 + 0.5), 2^32 - 1) (computed in double from the
 *     float p); kept values are scaled by (float)(1 / (1 - p)).  p must be in [0, 1); p = 0 is the same as no dropout.
 *     Counter layouts (csrc/philox.cuh):
 *       attention element (b, h, q, k), q' = q & ~8, k' = k & ~8:  ctr = ((k' >> 4) 8 + (k' & 7), (q' >> 4) 8 + (q' & 7),
 *           b heads + h, site); its four words belong to (q', k'), (q', k' + 8), (q' + 8, k'), (q' + 8, k' + 8)
 *       element-wise element i:  ctr = ((i >> 2) & 0xffffffff, i >> 34, 0xffffffff, site); word i & 3
 *    ns2_dropout_f32      : x (n f32, in place) = x * keep * scale — the phoneme encoder's conv dropout
 *                           (nn.Dropout, ns2.py:258) and its backward on the gradient
 * ------------------------------------------------------------------------------------------------ */
int ns2_dropout_f32(float* x, int64_t n, const ns2_dropout* dropout, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 3. RMSNorm (+ learned gamma) (+ FiLM) : RMSNorm.forward ns2.py:736-746.
 *    out_bf16[r, :] = x[r,:] / max(||x[r,:]||_2, 1e-12) * sqrt(dim) * gamma * film_gamma[b] + film_beta[b]
 *    gamma may be NULL (=1); film may be NULL (no FiLM); b = r / rows_per_batch;
 *    film_gamma = film + b*film_batch_stride, film_beta = film_gamma + dim.
 *    lens: NULL = every row, or per-batch row counts: device int32 (rows / rows_per_batch), each value clamped to
 *    [1, rows_per_batch].  Row r of batch b is normalized only if r % rows_per_batch < lens[b], by the same per-row
 *    code as without lens (bit-identical); the other rows are neither read nor written.
 * ------------------------------------------------------------------------------------------------ */
int ns2_rmsnorm_film(const float* x, int64_t x_row_stride, int64_t rows, int32_t dim,
                     int32_t rows_per_batch, const float* gamma, const float* film,
                     int64_t film_batch_stride, void* out_bf16, int64_t out_row_stride,
                     const int32_t* lens, ns2_stream_t stream);

/* Same, fp32 output (PerceiverResampler.norm, ns2.py:566,579). */
int ns2_rmsnorm_f32(const float* x, int64_t x_row_stride, int64_t rows, int32_t dim,
                    const float* gamma, float* out, int64_t out_row_stride, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 4. Small dense layers on the conditioning vector (M <= 64 rows), fp32 end to end.
 *    ns2_time_cond : LearnedSinusoidalPosEmb + Linear + SiLU (ns2.py:108-120, 839-843)
 *        out[b, :] = silu(W @ [t_b, sin(2 pi t_b w), cos(2 pi t_b w)] + bias),  W is (n_out, 2*half+1)
 *    ns2_small_linear : out[b,:] = act(W @ x[b,:] + bias), act 0 = none, 1 = SiLU (ns2.py:858-862)
 * ------------------------------------------------------------------------------------------------ */
int ns2_time_cond(const float* times, int32_t batch, const float* freqs, int32_t half_dim,
                  const float* W, const float* bias, int32_t n_out, float* out,
                  int64_t out_row_stride, ns2_stream_t stream);
int ns2_small_linear(const float* x, int64_t x_row_stride, int32_t batch, int32_t k, const float* W,
                     const float* bias, int32_t n_out, int32_t act, float* out,
                     int64_t out_row_stride, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 5. Layout / cast helpers (what `rearrange` + autocast do in the reference, ns2.py:972-997).
 *    ns2_cast_bf16        : out_bf16 = (bf16) (x [+ add]) ; add is broadcast over nothing (same shape) or NULL
 *    ns2_mean_rows        : out[b,:] = mean over n < L_b of x[b,n,:]   (Reduce('b n d -> b d','mean'), ns2.py:859);
 *                           L_b = n when lens is NULL, else lens[b] (device int32 (batch), clamped to [1, n]), summed
 *                           in row order either way — with lens, the prompt mean-pool of each sample run alone
 *    ns2_transpose_cast   : (B, C, L) f32 channel-first -> (B, L, C) bf16 token-major
 * ------------------------------------------------------------------------------------------------ */
int ns2_cast_bf16(const float* x, const float* add, int64_t count, void* out_bf16,
                  ns2_stream_t stream);
int ns2_mean_rows(const float* x, int32_t batch, int32_t n, int32_t dim, float* out, const int32_t* lens,
                  ns2_stream_t stream);
/*    ns2_mask_rows        : x[b, r, 0:cols] = 0 for lens[b] <= r < rows (lens clamped to [0, rows]), in place; x is f32
 *                           (f32 != 0) or bf16 with element strides row_stride / batch_stride — the zero padding past a
 *                           sample's end that a "same" convolution (ns2.py:316-320, 345-365) reads
 *    ns2_pack_rows        : bf16 out[b, r, 0:cols] = a[b, r, :] for r < La, b[b, r - La, :] for La <= r < La + Lb,
 *                           0 up to out_rows (La = a_lens[b] clamped to [0, a_rows], Lb = b_lens[b] clamped to
 *                           [0, b_rows]; out_rows >= a_rows + b_rows): the keys [norm(x) ; prompts] of the predictor's
 *                           cross attention (ns2.py:1060-1061) as one prefix of length La + Lb.  cols and every stride
 *                           a multiple of 4, pointers 8-byte aligned. */
int ns2_mask_rows(void* x, int32_t f32, int64_t row_stride, int64_t batch_stride, int32_t batch, int32_t rows,
                  int32_t cols, const int32_t* lens, ns2_stream_t stream);
int ns2_pack_rows(const void* a, int64_t a_row_stride, int64_t a_batch_stride, int32_t a_rows, const int32_t* a_lens,
                  const void* b, int64_t b_row_stride, int64_t b_batch_stride, int32_t b_rows, const int32_t* b_lens,
                  int32_t batch, int32_t cols, void* out, int64_t out_row_stride, int64_t out_batch_stride,
                  int32_t out_rows, ns2_stream_t stream);
/*    ns2_cond_inject      : out_bf16[b,n,:] = bf16(x[b,n,:] + c), c = 0 for n >= L_b (zero padding, ns2.py:70-77),
 *                           null_cond[:] where drop_mask[b] (uint8, may be NULL = keep all), else cproj[b,n,:]
 *                           (cproj: projected aligned condition, token-major (batch, cond_len, dim) f32; ns2.py:978-992).
 *                           L_b = cond_len when cond_lens is NULL, else min(cond_len, cond_lens[b]) (device int32
 *                           (batch), negative = 0): sample b's frames at or past it get nothing, null-substituted or
 *                           not — the zero padding after the projection of a sample run alone (ns2.py:978-992)
 *    ns2_select_rows      : out[b,:] = drop_mask[b] ? null_row[:] : src[b,:]  (f32 or bf16 out; ns2.py:954-968) */
int ns2_cond_inject(const float* x, const float* cproj, const uint8_t* drop_mask, const float* null_cond,
                    int32_t batch, int32_t n, int32_t cond_len, int32_t dim, void* out_bf16, const int32_t* cond_lens,
                    ns2_stream_t stream);
int ns2_select_rows(const uint8_t* drop_mask, const float* null_row, const float* src, int64_t src_row_stride,
                    int32_t batch, int32_t row_len, void* out, int64_t out_row_stride, int32_t out_bf16,
                    ns2_stream_t stream);
int ns2_transpose_cast(const float* x, int32_t batch, int32_t channels, int32_t length,
                       void* out_bf16, ns2_stream_t stream);
/*    ns2_embedding_bf16   : out_bf16[r,:] = bf16(table[ids[r] < 0 ? pad_id : ids[r], :]) — nn.Embedding of the phoneme
 *                           encoder with its padding substitution (ns2.py:253, 279-282); ids int64, table f32 */
int ns2_embedding_bf16(const int64_t* ids, int64_t rows, const float* table, int32_t num_rows, int32_t dim,
                       int32_t pad_id, void* out_bf16, ns2_stream_t stream);

/*    ns2_groupnorm_silu   : y = silu(GroupNorm(groups, channels)(x)) (+ resid) on token-major f32 x (batch, rows, channels):
 *                           statistics per (batch element, group) over rows x channels/groups values, biased variance,
 *                           eps inside the square root, per-channel affine (nn.GroupNorm) - Block.forward of the
 *                           duration / pitch predictor (ns2.py:345-365) with the ResnetBlock residual (ns2.py:399-401).
 *                           Writes out_f32 and/or out_bf16 (either may be NULL).  lens: NULL = every row, or sample b
 *                           has lens[b] rows (device int32 (batch), clamped to [1, rows]): the statistics cover rows
 *                           [0, lens[b]) in the order a call on a tensor of that many rows walks them (bit-identical to
 *                           it), and rows at or past lens[b] are written as exact zeros to out_f32 and out_bf16 (resid
 *                           is not read there) — Block's GroupNorm over a sample's own phonemes (ns2.py:345-365)
 *    ns2_rowdot           : out[r] = (relu ?) max(0, .) : (.) of dot(x[r,:], w) + bias[0] - Linear(dim, 1) + ReLU heads
 *                           (ns2.py:452-456) */
int ns2_groupnorm_silu(const float* x, int32_t batch, int32_t rows, int32_t channels, int32_t groups,
                       const float* weight, const float* bias, float eps, const float* resid, float* out_f32,
                       void* out_bf16, const int32_t* lens, ns2_stream_t stream);
int ns2_rowdot(const float* x, int64_t rows, int32_t dim, const float* w, const float* bias, int32_t relu, float* out,
               ns2_stream_t stream);
/*    ns2_expand_encodings : length regulation, NaturalSpeech2.expand_encodings (ns2.py:1449-1455) with the hard alignment
 *                           given as one text index per frame: out[b, d, n] = phon[b, m, d] + pitch_table[coarse[b, m], d],
 *                           m = idx[b, n] (int32; negative = frame past the sample's length -> 0).  phon f32 (batch, t_text,
 *                           dim) token-major, coarse int32 (batch, t_text) = f0_to_coarse bins, out f32 (batch, dim, length)
 *                           channel-first (the `cond` layout of Model.forward, ns2.py:929-937). */
int ns2_expand_encodings(const float* phon, const int32_t* coarse, const float* pitch_table, int32_t table_rows,
                         const int32_t* idx, int32_t batch, int32_t t_text, int32_t dim, int32_t length, float* out,
                         ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 6. Diffusion element-wise steps, fp32 (NaturalSpeech2.forward ns2.py:1621-1666; ddim_sample 1392-1429).
 *    All take per-sample scalars as device arrays of length `batch`; `per_sample` = N*D elements.
 *    `objective` selects the parameterisation (ns2.py:1637-1644, 1412-1421): NS2_OBJ_V / NS2_OBJ_EPS / NS2_OBJ_X0.
 *    ns2_q_sample   : x_t = alpha*x0 + sigma*noise ; target = alpha*noise - sigma*x0 (v) | noise (eps) | x0 (x0)
 *    ns2_mse_rows   : out[b] = mean((pred-target)^2) over the sample          (ns2.py:1646-1647);
 *                     deterministic two-level reduction through caller-provided scratch; optionally
 *                     also the batch mean of those per-sample values (one more tiny launch).
 *                     lens: NULL = every element, or a batch padded at the end: sample b is its first lens[b] rows of
 *                     row_elems elements (device int32 (batch), each clamped to [1, per_sample / row_elems]; row_elems
 *                     a multiple of 4 dividing per_sample, read only with lens).  out[b] is the mean over those
 *                     lens[b] * row_elems elements, reduced in the order a call on the unpadded sample uses:
 *                     bit-identical to it.  Elements past them are not read (they may hold anything).
 *    ns2_ddim_step  : x0 = alpha*x - sigma*out (v) | (x - sigma*out)/max(alpha,1e-10) (eps) | out (x0) ;
 *                     eps = (x - alpha*x0)/max(sigma,1e-10) ;
 *                     x <- x0*alpha_next + eps*sigma_next                     (ns2.py:1420-1429)
 *    ns2_cfg_combine: out = null + (cond - null)*scale                        (ns2.py:927)
 * ------------------------------------------------------------------------------------------------ */
#define NS2_MSE_SCRATCH_PER_SAMPLE 64
#define NS2_OBJ_V 0
#define NS2_OBJ_EPS 1
#define NS2_OBJ_X0 2
int ns2_q_sample(const float* x0, const float* noise, const float* alpha, const float* sigma,
                 int32_t batch, int64_t per_sample, float* x_t, float* target, int32_t objective,
                 ns2_stream_t stream);
int ns2_mse_rows(const float* pred, const float* target, int32_t batch, int64_t per_sample,
                 float* scratch /* batch * NS2_MSE_SCRATCH_PER_SAMPLE floats */, float* out,
                 float* mean_out /* optional: mean over the batch of out[], ns2.py:1666 */,
                 int64_t row_elems, const int32_t* lens, ns2_stream_t stream);
int ns2_ddim_step(float* x, const float* v, const float* alpha, const float* sigma,
                  const float* alpha_next, const float* sigma_next, int32_t batch,
                  int64_t per_sample, int32_t objective, ns2_stream_t stream);
int ns2_cfg_combine(const float* cond, const float* null_, float scale, int64_t count, float* out,
                    ns2_stream_t stream);
/*    ns2_x_start    : x_start implied by the model output `pred` (ns2.py:1673-1680): alpha*x - sigma*pred (v) |
 *                     (x - sigma*pred)/max(alpha,1e-10) (eps) | pred (x0) */
int ns2_x_start(const float* x, const float* pred, const float* alpha, const float* sigma, int32_t batch,
                int64_t per_sample, float* out, int32_t objective, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 7. Residual vector quantisation (Encodec RVQ encode/decode; third-party code reached from
 *    ns2.py:1445,1611 via audiolm_pytorch.EncodecWrapper -> encodec ResidualVectorQuantizer).
 *    ns2_rvq_prepare : codebooks f32 (Q, K, d) -> cb_f16: NS2_RVQ_PREPARED_HALFS(Q, K, d) fp16 values = the copy
 *                      (Q, K, d) scaled by 2^-e_q, codes permuted inside each 128-code chunk, followed by the (Q, K, 16) norm blocks (||c||^2 as an fp16 hi/lo pair,
 *                      laid out for the tensor core); ||c||^2 f32 (Q, K); meta f32 (Q, 2) = {max_k ||c_k||, 2^e_q}
 *    ns2_rvq_encode  : frames f32 (F, d) -> codes int64 (F, Q); residual chain in fp32, nearest
 *                      codeword by exact squared L2 distance, ties -> lowest index.  d must be 128,
 *                      K a multiple of 128.
 *    ns2_rvq_decode  : emb f32 (F, d) = sum_q codebooks[q, codes[f,q], :]  (summed in order q = 0..Q-1); a code
 *                      outside [0, K) reads the nearest valid codeword (< 0 -> 0, >= K -> K - 1).  d must be 128;
 *                      codebooks and emb 16-byte aligned.
 * ------------------------------------------------------------------------------------------------ */
#define NS2_RVQ_PREPARED_HALFS(q, k, d) ((long long)(q) * (k) * ((d) + 16))
#define NS2_RVQ_STATS_LEN 4
int ns2_rvq_prepare(const float* codebooks, int32_t q, int32_t k, int32_t d, void* cb_f16,
                    float* cb_norm2, float* cb_meta, ns2_stream_t stream);
int ns2_rvq_encode(const float* frames, int64_t num_frames, int32_t d, const float* codebooks,
                   const void* cb_f16, const float* cb_norm2, const float* cb_meta, int32_t q,
                   int32_t k, int64_t* codes,
                   int64_t* stats /* optional NS2_RVQ_STATS_LEN int64 counters, accumulated with atomics:
                                     {lookups, near-ties re-scored, full scans, sub-chunk scans} */,
                   ns2_stream_t stream);
int ns2_rvq_decode(const int64_t* codes, int64_t num_frames, int32_t q, int32_t k, int32_t d,
                   const float* codebooks, float* emb, ns2_stream_t stream);
/*    ns2_rvq_ce      : cross-entropy head of the residual VQ, `codec.rq(x_start, codes)` (ns2.py:1670-1684;
 *                      vector-quantize-pytorch ResidualVQ.forward(x, indices)).  Per stage the logits are the negative
 *                      Euclidean distances -||r_q - c_k||; loss = sum_q mean_{f: target != -1} CE(logits, target[f,q]);
 *                      the residual chain follows `own_codes` (the codec's own nearest codewords, from ns2_rvq_encode).
 *                      d must be 128, k >= 32.  ce_scratch: num_frames * q floats, left holding each frame's CE of
 *                      each stage at [f * q + stage] (0 where the target is -1); loss: 1 float. */
int ns2_rvq_ce(const float* frames, int64_t num_frames, int32_t d, const float* codebooks,
               const float* cb_norm2, int32_t q, int32_t k, const int64_t* own_codes,
               const int64_t* target_codes, float* ce_scratch, float* loss, ns2_stream_t stream);
/*    ns2_rvq_ce_bwd  : gradient of ns2_rvq_ce's loss with respect to `frames` (ns2.py:1682, `codec.rq(x_start, codes)`
 *                      differentiated through x_start).  The subtracted codewords are constants (vector-quantize-pytorch
 *                      subtracts `quantized.detach()`), so every stage's residual has d r_q / d frames = I and
 *                        d_frames[f] = row_scale[f / rows_per_sample] * sum_q d_loss / count_q * (u_t - sum_k p_k u_k),
 *                      u_k = (r_q - c_k) / ||r_q - c_k|| (0 where the distance is 0, torch.cdist's convention),
 *                      p = softmax(-||r_q - c_k||), t = target_codes[f, q]; stages whose target is -1 add nothing, a
 *                      stage with no valid target (count_q = 0) adds nothing.  `d_loss` (1 float) and the counts are read
 *                      on the device: no host synchronisation.  row_scale: optional (num_frames / rows_per_sample) f32,
 *                      NULL = 1 (NaturalSpeech2 folds d x_start / d pred into it).  coef_scratch: q floats.
 *                      d_frames: num_frames rows of out_stride floats (>= 128, multiple of 4, 16-byte aligned); only the
 *                      first 128 columns of valid rows are written.  Deterministic (no atomics). */
int ns2_rvq_ce_bwd(const float* frames, int64_t num_frames, int32_t d, const float* codebooks,
                   const float* cb_norm2, int32_t q, int32_t k, const int64_t* own_codes,
                   const int64_t* target_codes, const float* d_loss, const float* row_scale,
                   int64_t rows_per_sample, float* coef_scratch, float* d_frames, int64_t out_stride,
                   ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 8. Backward pass (what autograd runs for the reference's loss.backward(), README.md:63, ns2.py:1886).
 *    Matrix products: ns2_gemm with transposed weight packs (dgrad; negative shift_units = anti-causal taps) and
 *    ns2_wgrad.  Between them:
 *    ns2_rmsnorm_film_bwd : backward of RMSNorm (+learned gamma | +FiLM), ns2.py:736-746.  dxr (fp32 residual-stream
 *                           gradient) += dx IN PLACE, its bf16 copy is written to dxr_bf16; dfilm[b, :dim] += d(gamma_b),
 *                           dfilm[b, dim:2dim] += d(beta_b) (atomics); dgamma[:] += d(learned gamma)
 *    ns2_geglu_bwd        : pre (rows, 2*dp) bf16 in the packed [128 value | 128 gate] tile layout is OVERWRITTEN by its
 *                           gradient given dg (rows, dp) bf16   (GEGLU, ns2.py:1004-1007)
 *    ns2_wavenet_gate_bwd : dz of y = tanh(z) sigmoid(z) + res, z = c*gamma_b + beta_b (ns2.py:625-630): dc = dz*gamma_b,
 *                           dfilm += [sum dz*c | sum dz] per batch / group
 *    ns2_colsum_bf16      : out[c] += sum_r t[r, c]            (bias gradients)
 *    ns2_group_sum_bf16   : out[r, c] = sum_g t[r, g*dim + c]  (gradient of an input shared by all dilation columns)
 *    ns2_mse_bwd          : out = coef[b] * (pred - target), bf16 and/or f32   (seed of the backward pass, ns2.py:1646-1666);
 *                           row_elems / lens as for ns2_mse_rows: the first lens[b] rows of row_elems elements of
 *                           sample b are bit-identical to the call without lens, every element past them is written as
 *                           an exact zero (pred / target are not read there)
 *    ns2_film_wgrad       : dw[r, c] (+)= sum_b dfilm[b, r] * t[b, c]  (FiLM projection weights; batch <= 32 per call)
 *    ns2_attn_bwd         : flash-attention backward (dq, dk, dv) from (q, k, v, o, lse, do)
 * ------------------------------------------------------------------------------------------------ */
int ns2_rmsnorm_film_bwd(const float* x, const void* dh_bf16, int64_t rows, int32_t dim, int32_t rows_per_batch,
                         const float* gamma, const float* film, int64_t film_batch_stride, float* dfilm,
                         int64_t dfilm_batch_stride, float* dgamma, float* dxr, void* dxr_bf16, ns2_stream_t stream);
int ns2_geglu_bwd(void* pre_bf16, const void* dg_bf16, int64_t rows, int32_t dp, ns2_stream_t stream);
int ns2_wavenet_gate_bwd(const void* c_bf16, int64_t c_row_stride, const void* dy_bf16, int64_t dy_row_stride,
                         void* dc_bf16, int64_t dc_row_stride, int32_t batches, int32_t rows_per_batch, int32_t dim,
                         int32_t groups, const float* film, int64_t film_batch_stride, int32_t film_group_stride,
                         float* dfilm, int64_t dfilm_batch_stride, ns2_stream_t stream);
int ns2_colsum_bf16(const void* t_bf16, int64_t rows, int32_t cols, int64_t row_stride, float* out, ns2_stream_t stream);
int ns2_group_sum_bf16(const void* t_bf16, int64_t rows, int32_t dim, int32_t groups, void* out_bf16, ns2_stream_t stream);
int ns2_mse_bwd(const float* pred, const float* target, const float* coef, int32_t batch, int64_t per_sample,
                void* out_bf16 /* optional */, float* out_f32 /* optional */, int64_t row_elems, const int32_t* lens,
                ns2_stream_t stream);
int ns2_film_wgrad(const float* dfilm, int64_t dfilm_batch_stride /* elements between batch rows of dfilm (>= rows): a
                   column window of the stacked FiLM gradient can be reduced as soon as its layer is final */,
                   const float* t, int32_t batch, int64_t rows, int32_t cols, float* dw,
                   int32_t accumulate /* 0: dw = ..., dw need not be initialised; 1: dw += ... */, ns2_stream_t stream);
/*    ns2_accum_bf16       : acc (f32) += t (bf16); acc_bf16 (optional) = bf16(acc)   (joins a branch gradient) */
int ns2_accum_bf16(float* acc, const void* t_bf16, int64_t count, void* acc_bf16, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 8b. Backward of the conditioning front end (SpeechPromptEncoder ns2.py:289-341, PhonemeEncoder 228-287, pitch
 *     embedding and length regulation 1449-1455, 1581-1583): the diffusion loss reaches them through
 *     Model(prompt=prompt_enc, cond=cond) (ns2.py:1635, 1886).  Convolution dgrad / wgrad are ns2_gemm / ns2_wgrad
 *     ("same" padding: negative shift_units); attention, RMSNorm(gamma) and GEGLU reuse section 8.
 *    ns2_silu_bwd             : dpre = dout * s * (1 + pre * (1 - s)), s = sigmoid(pre), all bf16, `count` elements
 *                               (even); dpre may alias pre.  nn.SiLU after each k=9 conv (ns2.py:255-257, 316-320)
 *    ns2_embedding_bwd        : dtable[id(r), :] += de[r, :] (f32, atomics), id(r) = ids[r] < 0 ? pad_id : ids[r]
 *                               — nn.Embedding backward of the phoneme table (ns2.py:253, 279-282); the pad row
 *                               receives gradient (the reference's table has no padding_idx)
 *    ns2_expand_encodings_bwd : transpose of ns2_expand_encodings given d cond token-major f32 (batch, length, dim)
 *                               with row stride dcond_row_stride:  dphon[b, m, :] += sum over frames n with
 *                               idx[b, n] == m of dcond[b, n, :];  dtable[coarse[b, m], :] += the same sums (atomics).
 *                               Frames with idx < 0 add nothing; either output may be NULL
 *    ns2_add_rows_bcast       : x[b, r, :] += scale * v[b, :] for f32 x (batch, rows, dim) — the gradient of a
 *                               mean over rows (prompt mean-pool, ns2.py:858-862) added to a per-row gradient
 * ------------------------------------------------------------------------------------------------ */
int ns2_silu_bwd(const void* pre_bf16, const void* dout_bf16, int64_t count, void* dpre_bf16, ns2_stream_t stream);
int ns2_embedding_bwd(const int64_t* ids, int64_t rows, const float* de, int32_t num_rows, int32_t dim, int32_t pad_id,
                      float* dtable, ns2_stream_t stream);
int ns2_expand_encodings_bwd(const float* dcond, int64_t dcond_row_stride, const int32_t* coarse, int32_t table_rows,
                             const int32_t* idx, int32_t batch, int32_t t_text, int32_t dim, int32_t length, float* dphon,
                             float* dtable, ns2_stream_t stream);
int ns2_add_rows_bcast(float* x, int32_t batch, int32_t rows, int32_t dim, const float* v, float scale,
                       ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 8c. Backward of the duration / pitch predictor (DurationPitchPredictor ns2.py:345-527, trained through the L1
 *     losses of ns2.py:1579-1590).  Its k=3 "same" convs use ns2_gemm / ns2_wgrad (shifts +1..-1), its cross
 *     attention and RMSNorm(gamma) section 8.  Both entries are deterministic: per-CTA partial sums in a caller-provided
 *     workspace, then a second launch adds them in a fixed order (no atomics).
 *    ns2_groupnorm_silu_bwd : backward of ns2_groupnorm_silu (without its residual, an identity the caller adds) given
 *                             dy f32 (batch, rows, channels): with xh = (x - mean) * rstd (statistics recomputed as the
 *                             forward computes them), z = xh * weight + bias, dz = dy * silu'(z), dxh = dz * weight,
 *                               dx = rstd * (dxh - mean(dxh) - xh * mean(dxh * xh))   (means over the group of a sample)
 *                             written as bf16; dweight[c] = sum dz * xh, dbias[c] = sum dz (overwritten).  channels /
 *                             groups a multiple of 4 and <= 1024, batch <= 65535.  partial: 2 * batch * channels floats.
 *    ns2_rowdot_bwd         : backward of ns2_rowdot with relu: dpre[r] = pred[r] > 0 ? dpred[r] : 0 (0 at pred == 0,
 *                             as torch's threshold_backward); dx[r, :] += dpre[r] * w (f32, in place); dw[:] =
 *                             sum_r dpre[r] * x[r, :], db[0] = sum_r dpre[r] (overwritten).  partial:
 *                             ceil(rows / NS2_ROWDOT_BWD_ROWS) * (dim + 4) floats.
 * ------------------------------------------------------------------------------------------------ */
#define NS2_ROWDOT_BWD_ROWS 32
int ns2_groupnorm_silu_bwd(const float* x, int32_t batch, int32_t rows, int32_t channels, int32_t groups,
                           const float* weight, const float* bias, float eps, const float* dy, void* dx_bf16,
                           float* partial, float* dweight, float* dbias, ns2_stream_t stream);
int ns2_rowdot_bwd(const float* x, int64_t rows, int32_t dim, const float* w, const float* pred, const float* dpred,
                   float* dx, float* partial, float* dw, float* db, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 9. Monotonic alignment search: `maximum_path(value, mask)` of naturalspeech2_pytorch/aligner.py:88-122 (called from
 *    Aligner.forward aligner.py:214, reached from NaturalSpeech2.forward ns2.py:1578 in conditional training).
 *    value, mask: f32 (batch, t_x, t_y) contiguous (t_x text positions <= 1024, t_y mel frames); mask holds 0/1.
 *    Viterbi recursion over the frames with the reference's exact fp32 operations and tie rule, then the backtrack:
 *      idx[b, j]     (int32, batch x t_y)  = text position aligned to frame j
 *      path[b, i, j] (f32, optional)       = (idx[b, j] == i) * mask[b, i, j]      — bit-identical to the reference
 *    neg_const = the reference's `const` (default -inf).  workspace: ns2_maximum_path_workspace_bytes() bytes of
 *    scratch (1-bit decisions, batch x t_y x 128 B).
 * ------------------------------------------------------------------------------------------------ */
int64_t ns2_maximum_path_workspace_bytes(int32_t batch, int32_t t_x, int32_t t_y);
int ns2_maximum_path(const float* value, const float* mask, int32_t batch, int32_t t_x, int32_t t_y, float neg_const,
                     void* workspace, int64_t workspace_bytes, int32_t* idx, float* path, ns2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * 10. Encodec's SEANet decoder, 24 kHz model (`codec.decode(audio)`, ns2.py:1496-1499, reached through
 *     audiolm_pytorch.EncodecWrapper.decode -> encodec SEANetDecoder; transformers' EncodecDecoder has the same
 *     layers), and its SEANet encoder (`codec(raw_audio)`, transformers' EncodecEncoder).  Convolutions with >= 64
 *     channels, the transposed and strided convolutions and the LSTM input projections are ns2_gemm calls; these
 *     four entry points cover the rest.  Activations are token-major (batch, time, channel).
 *    ns2_lstm_seq    : one layer of nn.LSTM(512, 512) over `steps` time steps with zero initial state (the decoder's
 *                      SLSTM: encodec/modules/lstm.py, transformers EncodecLSTM), gate order i, f, g, o:
 *                        gates = xproj[b, t, :] + W_hh h_{t-1};  c = f c + i g;  h_t = o tanh(c)
 *                      xproj (batch, steps, 2048) f32 = x W_ih^T + b_ih + b_hh with its columns (and W_hh's rows)
 *                      permuted to the kernel's order: column 128 c + 64 hf + 16 w + 8 i + q holds gate 2 hf + i of
 *                      hidden unit 32 c + 8 w + q.  w_hh: those 2048 permuted rows x 512, bf16.  h_{t-1} enters the
 *                      recurrence as bf16.  Writes out[b, t, :] = h_t (+ skip[b, t, :] when skip != NULL: the
 *                      `lstm(x)[0] + x` of SLSTM) as f32 and/or bf16 (either may be NULL).  hidden must be 512.  One
 *                      16-CTA cluster per 64 batch rows (needs a device that can hold such a cluster, else an error).
 *    ns2_elu_pad     : out_bf16[b, r, 0:C] = bf16(act(xpad[b, r - pad])), r in [0, pad + length), act = ELU
 *                      (nn.ELU, alpha 1) with NS2_ELU_PAD_ELU else identity; xpad is x reflect-padded on the left by
 *                      `pad` (StreamableConv1d / EncodecConv1d causal padding, with their rule for inputs no longer
 *                      than the pad: zeros are appended before reflecting).  NS2_ELU_PAD_RAW also writes bf16(xpad) in
 *                      columns [C, 2C) (the un-activated input of a ResnetBlock shortcut).  C % 4 == 0.
 *    ns2_seanet_tail : the decoder's last 32-channel stage at the sample rate, f32 throughout:
 *                        z = shortcut(x) + conv1x1(ELU(conv3(ELU(x))))   (SEANetResnetBlock 32 -> 16 -> 32)
 *                        out[b, t] = conv7(ELU(z))[t]                    (final StreamableConv1d 32 -> 1)
 *                      causal, reflect-padded like ns2_elu_pad.  x: (batch, length, 32) f32.  params:
 *                      NS2_SEANET_TAIL_PARAMS f32 (weight norm folded):  w3 [tap 3][in 32][out 16], b3 [16],
 *                      w_shortcut [in 32][out 32], w_conv1 [in 16][out 32], b_shortcut + b_conv1 [32],
 *                      w_final [tap 7][in 32], b_final, 3 zeros.
 *    ns2_seanet_head : the encoder's first 32-channel stage at the sample rate (transformers EncodecEncoder layers
 *                      0-2), f32 throughout, bf16 output:
 *                        z0 = conv7(x)                                    (StreamableConv1d 1 -> 32)
 *                        z1 = shortcut(z0) + conv1x1(ELU(conv3(ELU(z0)))) (SEANetResnetBlock 32 -> 16 -> 32)
 *                        out_bf16[b, r, 0:32] = bf16(ELU(z1pad[b, r - 2])), r in [0, length + 2)
 *                      causal, reflect-padded like ns2_elu_pad; z1pad is z1 reflect-padded by 2, so `out` is
 *                      ns2_elu_pad(z1, pad = 2) and directly the A operand of the encoder's k4 stride-2 conv.
 *                      x: (batch, length) f32 with batch stride x_batch_stride.  out: 16-byte aligned, row and batch
 *                      strides multiples of 8.  params: NS2_SEANET_HEAD_PARAMS f32 (weight norm folded):
 *                      w0 [tap 7][out 32], b0 [32], w3 [tap 3][in 32][out 16], b3 [16], w_shortcut [in 32][out 32],
 *                      w_conv1 [in 16][out 32], b_shortcut + b_conv1 [32].
 *    The encoder's strided convs (k = 2s, stride s, reflect left pad s) are 2-segment ns2_gemm calls: ns2_elu_pad
 *    (pad = s) writes a contiguous (batch, L + s, C) buffer, viewed as (batch, L/s + 1, s C) rows; the weight packed
 *    tap-major (C_out, 2 s C); segments {a 0, b 0, k sC, shift 1}, {a 0, b sC, k sC, shift 0}; output row m + 1 is
 *    conv output m (row 0 is scratch).
 * ------------------------------------------------------------------------------------------------ */
#define NS2_ELU_PAD_ELU 1
#define NS2_ELU_PAD_RAW 2
#define NS2_SEANET_TAIL_PARAMS 3348
#define NS2_SEANET_HEAD_PARAMS 3376
int ns2_lstm_seq(const float* xproj, int64_t xp_row_stride, int64_t xp_batch_stride, const void* w_hh, int32_t batch,
                 int32_t steps, int32_t hidden, const float* skip, int64_t skip_row_stride, int64_t skip_batch_stride,
                 float* out, int64_t out_row_stride, int64_t out_batch_stride, void* out_bf16, int64_t outbf_row_stride,
                 int64_t outbf_batch_stride, ns2_stream_t stream);
int ns2_elu_pad(const float* x, int64_t x_row_stride, int64_t x_batch_stride, int32_t batch, int32_t length,
                int32_t channels, int32_t pad, int32_t flags, void* out_bf16, int64_t out_row_stride,
                int64_t out_batch_stride, ns2_stream_t stream);
int ns2_seanet_tail(const float* x, int64_t x_row_stride, int64_t x_batch_stride, int32_t batch, int32_t length,
                    const float* params, float* out, int64_t out_batch_stride, ns2_stream_t stream);
int ns2_seanet_head(const float* x, int64_t x_batch_stride, int32_t batch, int32_t length, const float* params,
                    void* out_bf16, int64_t out_row_stride, int64_t out_batch_stride, ns2_stream_t stream);

/* Number of kernel launches issued through this library since load (for bench.py's gpu_launches). */
int64_t ns2_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* NS2_H100_H_ */
