/* mmfb200.h - C ABI of the H100-native (sm_90a) multimodal-fusion block (libmmfb200.so).
 *
 * The reference (facebookresearch/mmf) has no FFI for this path: the boundary is the Python-level
 * module contract of
 *   BertSelfAttention/BertAttention/BertLayer/BertEncoder.forward   mmf/modules/hf_layers.py:161-355
 *   BertBiAttention/BertBiOutput/BertConnectionLayer.forward         mmf/models/vilbert.py:388-556
 *   BertVisioLinguisticEmbeddings.forward                            mmf/modules/embeddings.py:423-459
 *   BertImageFeatureEmbeddings.forward                               mmf/models/vilbert.py:904-913
 *   ModalEmbeddings.forward                                          mmf/models/mmbt.py:84-129
 *   HuggingfaceEmbeddings.forward                                    mmf/models/transformers/backends/huggingface.py:131-159
 * and their autograd backward (mmf/trainers/core/training_loop.py:211-213).  This header is what a
 * binding for that path calls (mmf_b200/lib.py is the ctypes binding; INTEGRATION.md shows the stub).
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless stated; bf16 = 16-bit bfloat, row-major, explicit
 *     leading dimensions in ELEMENTS; the caller owns every buffer (outputs, saved-for-backward,
 *     workspace); functions never allocate, never synchronise, enqueue on `stream` only
 *   - return value: 0 = ok, otherwise an mmfb_status; mmfb_last_error() gives the message of the
 *     last failure on the calling thread; no C++ exception crosses the ABI
 *   - there is no CPU fallback: without an sm_90 device every compute entry point fails
 */
#ifndef MMFB200_H_
#define MMFB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* mmfb_stream; /* cudaStream_t */

typedef enum {
  MMFB_OK = 0,
  MMFB_ERR_ARG = 1,     /* bad shape / alignment / null pointer  -> ValueError in the binding */
  MMFB_ERR_CUDA = 2,    /* CUDA runtime / driver failure         -> RuntimeError */
  MMFB_ERR_DEVICE = 3   /* no sm_90 device                       -> RuntimeError */
} mmfb_status;

/* epilogues of mmfb_gemm */
enum {
  MMFB_EPI_BIAS = 0,            /* C = acc + bias                      (bias may be NULL)            */
  MMFB_EPI_BIAS_GELU = 1,       /* C = acc + bias ; C2 = gelu_erf(C)   BertIntermediate              */
  MMFB_EPI_BIAS_DROP_RESID = 2, /* C = dropout(acc + bias) + aux       BertSelfOutput/BertOutput pre-LN */
  MMFB_EPI_GELU_BWD = 3,        /* C = acc * gelu_erf'(aux)            dgrad through BertIntermediate */
  MMFB_EPI_ADD_AUX = 4,         /* C = acc + aux                       dgrad + residual gradient     */
  MMFB_EPI_ATOMIC_F32 = 5,      /* C(fp32) += acc                      split-K weight gradient       */
  MMFB_EPI_BIAS_RELU = 6,       /* C = relu(acc + bias)                FinetuneFasterRcnnFpnFc7, encoders.py:176-179 */
  MMFB_EPI_BIAS_GELU_DROP = 7,  /* C = u = acc + bias ; C2 = keep * scale * gelu_erf(u)   timm Mlp fc1 -> GELU -> Dropout */
  MMFB_EPI_GELU_DROP_BWD = 8    /* C = acc * keep * scale * gelu_erf'(aux)               its dgrad (aux = u)           */
};
/* MMFB_EPI_BIAS_GELU_DROP runs with (a_mn, b_mn) = (0, 0) and MMFB_EPI_GELU_DROP_BWD with (0, 1).  Both read the keep bits
 * drop_mask (bit n % 32 of word n / 32 of row m keeps element (m, n); mmfb_dropout_bits) and scale kept values by drop_scale:
 * drop_mask NULL or not 4-byte aligned, ldmask < ceil(N/32), drop_scale not positive and finite, C2 NULL (_GELU_DROP) or aux
 * NULL (_GELU_DROP_BWD) is MMFB_ERR_ARG before any launch.  Dropped elements of C2 / C are exact zeros. */

/* C[M,N] = epi( A[M,K] * B[N,K]^T ).  a_mn/b_mn = 0: operand stored [rows,K] (K contiguous);
 * = 1: operand stored [K,rows] (rows contiguous), i.e. the transposed view of a row-major tensor. */
typedef struct {
  const void* A; int64_t lda; int a_mn;
  const void* B; int64_t ldb; int b_mn;
  void* C; int64_t ldc;          /* bf16 [M,N]; fp32 [M,N] for MMFB_EPI_ATOMIC_F32 */
  void* C2;                      /* second bf16 output (MMFB_EPI_BIAS_GELU), same ldc */
  const void* bias;              /* bf16 [N] or NULL */
  const void* aux; int64_t ldaux;/* bf16 [M,N] residual / pre-activation or NULL; the epilogues that read it (2, 3, 4)
                                  * load it by TMA: 16-byte aligned, ldaux % 8 == 0, else MMFB_ERR_ARG */
  const uint32_t* drop_mask; int64_t ldmask; float drop_scale; /* keep-bits [M, ldmask] words or NULL */
  int M, N, K;
  int epi;
  int splits;                    /* split-K factor, MMFB_EPI_ATOMIC_F32 only (0/1 = none) */
  int block_n;                   /* 0 = auto, else 128 or 256 */
  int cluster;                   /* 0, 1 or 2; kept for ABI compatibility: every GEMM runs as single-CTA tiles */
  void* workspace;               /* MMFB_EPI_ATOMIC_F32 only: NULL and 0 = fp32 vector reductions (see below) */
  int64_t workspace_bytes;
} mmfb_gemm_args;

int mmfb_gemm(const mmfb_gemm_args* args, mmfb_stream stream);

/* Ordered split-K (MMFB_EPI_ATOMIC_F32 with a workspace).  By default the S = splits units of an output tile add their
 * fp32 partial tiles into C with vector reductions, in whatever order they finish, so the low bits of C vary from run to
 * run whenever the GEMM actually runs S > 1 splits.  With `workspace` set, unit (tile, s) instead STORES its partial P_s
 * (the product over split s's k-blocks, accumulated from zero) into slice s of the fp32 workspace [S, M, N], and a second
 * kernel computes  C = ((C + P_0) + P_1) + ... + P_{S-1}  in fp32, split by split: the same bits on every run.
 * mmfb_gemm_workspace_bytes(M, N, K, splits) (host only, no device needed) gives the bytes this takes: S * M * N * 4 for the
 * split factor the GEMM will run (splits is lowered until every split owns a k-block of 64), or 0 when that factor is 1 -
 * a single unit per tile adds C + acc once, which is already deterministic, and the workspace is not touched.
 * An ordered call (workspace or workspace_bytes non-zero) whose workspace is NULL, smaller than that size or not 16-byte
 * aligned is MMFB_ERR_ARG before any launch.  The workspace is the caller's; nothing in it is kept between calls. */
int64_t mmfb_gemm_workspace_bytes(int M, int N, int K, int splits);

/* mmfb_gemm with device bounds.  m_dev: NULL, or a DEVICE int32 row bound: only the 128-row tiles that start below
 * min(M, *m_dev) are computed and stored.  k_dev: NULL, or a DEVICE int32 bound on K: only the 64-deep k-blocks that start
 * below min(K, *k_dev) are summed.  Both NULL is mmfb_gemm.  A masked-LM head captured in a CUDA graph runs its vocabulary GEMMs on a fixed
 * capacity of rows of which only a prefix, counted on the device, is labelled (mmfb_select_rows).  The bounds are read
 * when the kernel runs, after the kernel before it has finished; the grid is still sized from M, N, K and the CTAs with no
 * work left exit at once.  With b = clamp(*m_dev, 0, M), rows [0, ceil(b/128)*128) of C are computed and stored exactly as
 * an unbounded call computes them, and no row at or past that is read or written.  With b = clamp(*k_dev, 0, K) (the
 * weight gradient, where K is the row count), the k-blocks [0, ceil(b/64)) are shared among the launched splits the way an
 * unbounded call with K = b shares them; a split left without a k-block adds nothing, or with a workspace stores a zero
 * partial.  So the operand rows between b and the rounded bound are read: the caller keeps them zero.  Supported for
 * MMFB_EPI_BIAS with (a_mn, b_mn) = (0, 0) or (0, 1), for MMFB_EPI_ATOMIC_F32 with (1, 1), with or without a
 * workspace, and for the encoder layer's epilogues: MMFB_EPI_BIAS_GELU and MMFB_EPI_BIAS_DROP_RESID with (0, 0),
 * MMFB_EPI_GELU_BWD and MMFB_EPI_ADD_AUX with (0, 1).  Their per-row operands (aux, the dropout keep bits) are read only
 * for the row tiles below the rounded bound, like A; C and C2 are written only there.  A row between b and the rounded
 * bound is computed from whatever its operand rows hold and affects no other row (with one, the ordered reduce also covers only the rows below the rounded M bound: the rows of C past it
 * are not read or written, and the workspace rows past it are not read); anything else is MMFB_ERR_ARG before a launch.
 * A bound of 0 adds nothing to C. */
int mmfb_gemm_bounded(const mmfb_gemm_args* args, const int32_t* m_dev, const int32_t* k_dev, mmfb_stream stream);

/* Fused multi-head attention core (everything between the Q/K/V projections and the output projection):
 *   ctx = dropout(softmax(Q K^T / sqrt(d) + mask)) V        BertSelfAttentionJit.forward hf_layers.py:182-210,
 *   BertBiAttention.forward vilbert.py:421-461 (cross: q from one stream, k/v from the other).
 * q [B*Sq, ldq], k/v [B*Skv, ld*]: bf16, head h in columns [h*head_dim, (h+1)*head_dim); usually three
 * column slices of one fused projection buffer.  mask: additive fp32 [B, Skv] (the reference's
 * [B,1,1,Skv] tensor) or NULL; values below -10000 (finfo(dtype).min, -inf) act exactly like -10000, so a fully
 * masked row gives the softmax of its raw scores and stays finite.  lse2 [B, heads, Sq] fp32 receives the log2-domain row log-sum-exp
 * (saved for backward).  drop_mask: keep bits [B, heads, Sq, ceil(Skv/32)] (bit kv%32) or NULL.
 * Limits: head_dim 64 or 128; Skv <= 384 (d=64) / 256 (d=128) - MMF's path has S <= 324.
 * causal_len (self-attention only): T > 0 makes the last T keys a causal tail - the prefix-LM mask of M4C's multimodal
 * transformer (mmf/models/m4c.py:418-437).  With P = Skv - T, key k < P takes mask[b, k] as above (clamp included), and
 * key k >= P takes 0 when k <= q and -10000 otherwise, in place of mask[b, k], which is not read for those keys.  So the
 * first P queries never see the tail, and query P + t sees tail keys P .. P + t.  0 (what a zero-initialised struct
 * holds) means no tail.  Requires Sq == Skv and T <= Skv; a negative T is MMFB_ERR_ARG, and so is any T != 0 in the
 * packed (varlen) entry points and mmfb_attention_probs: packed attention with a tail is
 * mmfb_attention_varlen_causal_fwd / _bwd.  Every refusal happens before a launch. */
typedef struct {
  const void* q; int64_t ldq;
  const void* k; int64_t ldk;
  const void* v; int64_t ldv;
  const float* mask;
  void* ctx; int64_t ldo;            /* bf16 [B*Sq, ldo]: output of fwd, input of bwd */
  float* lse2;
  const uint32_t* drop_mask; float drop_scale;
  void* ctx_lo;                      /* optional bf16 [B*Sq, heads*head_dim], contiguous: bf16(O - float(ctx)), the part of the
                                        fp32 output the bf16 ctx drops; written by fwd, read by bwd (delta = rowsum(dO*(ctx+ctx_lo))) */
  /* backward only */
  const void* dctx; int64_t ld_dctx; /* bf16 [B*Sq, ld_dctx] */
  float* delta;                      /* fp32 scratch [B, heads, Sq] */
  void* dq; int64_t ld_dq;           /* bf16 outputs, same head layout as q/k/v */
  void* dk; int64_t ld_dk;
  void* dv; int64_t ld_dv;
  int B, heads, Sq, Skv, head_dim;
  int causal_len;                    /* keys in the causal tail, 0 = none (see above) */
} mmfb_attn_args;

int mmfb_attention_fwd(const mmfb_attn_args* args, mmfb_stream stream);
int mmfb_attention_bwd(const mmfb_attn_args* args, mmfb_stream stream);

/* Variable-length (packed) self-attention: padded tokens are removed before the call, so no work is spent on them.
 * cu_seqlens: int32 [B+1] on the DEVICE, a non-decreasing prefix sum with cu_seqlens[0] = 0 and cu_seqlens[B] = total;
 * sample b owns the packed rows [cu_seqlens[b], cu_seqlens[b+1]) of every row buffer (queries and keys share it).
 * A sample of length 0 is legal: nothing is computed or written for it.  The lengths are never read on the host.
 *   args->B = samples; args->Sq = args->Skv = max_len >= every length (sets the grid; rows past max_len are not used);
 *   args->mask must be NULL (MMFB_ERR_ARG otherwise): packing has already removed the masked keys;
 *   q, k, v, ctx, ctx_lo, dctx, dq, dk, dv: [total, ld] rows, same head-column layout as mmfb_attention_fwd;
 *   lse2, delta: fp32 [heads, total];
 *   drop_mask: keep bits int32 [heads, total, ceil(max_len/32)], bit kv%32 of word kv/32 for key kv WITHIN the sample.
 * Limits: head_dim 64 or 128; max_len <= 384 (d=64) / 256 (d=128).  total = 0 returns MMFB_OK without a launch. */
int mmfb_attention_varlen_fwd(const mmfb_attn_args* args, const int32_t* cu_seqlens, int total, mmfb_stream stream);
int mmfb_attention_varlen_bwd(const mmfb_attn_args* args, const int32_t* cu_seqlens, int total, mmfb_stream stream);

/* Variable-length (packed) self-attention with a causal tail: the packing of mmfb_attention_varlen_fwd / _bwd (same
 * arguments, buffers and keep-bit layout) with causal_len = T, the packed form of M4C's prefix-LM mask.  The tail of
 * sample b is its last T rows: with len_b = cu_seqlens[b+1] - cu_seqlens[b] and P_b = max(len_b - T, 0), counted within
 * the sample, key k >= P_b takes 0 for queries q >= k and -10000 for the others (the dense causal rule with len_b in
 * place of Skv), and keys below P_b take 0.  The lengths are read on the device only, so a sample shorter than T is all
 * tail.  Each sample computes bit for bit what mmfb_attention_fwd / _bwd compute for it alone (B = 1, Sq = Skv = len_b,
 * mask NULL, causal_len = min(T, len_b)).
 * Requires 0 < causal_len <= max_len, Sq == Skv == max_len, mask == NULL and a non-null cu_seqlens; any other call is
 * MMFB_ERR_ARG before a launch.  total = 0 returns MMFB_OK without a launch.  Limits as mmfb_attention_varlen_fwd. */
int mmfb_attention_varlen_causal_fwd(const mmfb_attn_args* args, const int32_t* cu_seqlens, int total, mmfb_stream stream);
int mmfb_attention_varlen_causal_bwd(const mmfb_attn_args* args, const int32_t* cu_seqlens, int total, mmfb_stream stream);

/* Variable-length (packed) cross-attention: the queries come from one packed stream and the keys / values from another
 * (ViLBERT co-attention, LXMERT cross-modality layers).  cu_q, cu_kv: int32 [B+1] on the DEVICE, each a non-decreasing
 * prefix sum from 0 to total_q / total_kv; sample b's queries are rows [cu_q[b], cu_q[b+1]) of q, ctx, ctx_lo, dctx, dq
 * and its keys rows [cu_kv[b], cu_kv[b+1]) of k, v, dk, dv.  The lengths are never read on the host.
 *   args->B = samples; args->Sq = max_q >= every query length (sets the grid), args->Skv = max_kv >= every key length;
 *   args->mask must be NULL (MMFB_ERR_ARG otherwise): packing has already removed the masked keys;
 *   q, ctx, ctx_lo, dctx, dq: [total_q, ld] rows; k, v, dk, dv: [total_kv, ld] rows; same head-column layout as
 *   mmfb_attention_fwd;
 *   lse2, delta: fp32 [heads, total_q];
 *   drop_mask: keep bits int32 [heads, total_q, ceil(max_kv/32)], bit kv%32 of word kv/32 for key kv WITHIN the sample.
 * Empty sides are defined and never produce NaN:
 *   a sample with queries but no keys writes ctx = ctx_lo = 0 and dq = 0 on its query rows, and lse2 = -inf (the log of an
 *   empty sum; the backward does not read it);
 *   a sample with keys but no queries writes dk = dv = 0 on its key rows (so the backward runs even when total_q = 0).
 * Every query row in [0, total_q) gets ctx / lse2 / dq, every key row in [0, total_kv) gets dk / dv, as long as the
 * lengths respect max_q / max_kv; lengths are clamped to them and to the totals, so a bad cu never reaches outside the
 * buffers.  Sq / Skv / totals of 0 are legal; the forward returns MMFB_OK without a launch when total_q = 0, the backward
 * when both totals are 0.  Packed self-attention is this call with cu_kv = cu_q and computes bit for bit what
 * mmfb_attention_varlen_fwd / _bwd do.
 * Limits: head_dim 64 or 128; max_kv <= 384 (d=64) / 256 (d=128); max_q only by the grid. */
int mmfb_attention_varlen_cross_fwd(const mmfb_attn_args* args, const int32_t* cu_q, int total_q, const int32_t* cu_kv,
                                    int total_kv, mmfb_stream stream);
int mmfb_attention_varlen_cross_bwd(const mmfb_attn_args* args, const int32_t* cu_q, int total_q, const int32_t* cu_kv,
                                    int total_kv, mmfb_stream stream);

/* Attention probabilities of one DENSE mmfb_attention_fwd call, for inspection (the reference's output_attentions /
 * ViLBERT visualization outputs, hf_layers.py:196-210, vilbert.py:94-112, 419-475):
 *   probs[b, h, q, k] = exp2(S[b,h,q,k] * log2(e)/sqrt(d) + M'[b,k] - lse2[b,h,q])      (* keep(b,h,q,k) * drop_scale)
 * S = Q K^T of the call's q / k head slices, M' = log2(e) * max(mask[b,k], -10000) (the clamp of the forward and backward),
 * lse2 the row statistics that forward wrote.  Pass the inputs of that forward: q, ldq, k, ldk, mask, lse2, drop_mask,
 * drop_scale, B, heads, Sq, Skv, head_dim; v, ctx and the backward fields are not read.
 *   probs: DEVICE buffer, contiguous [B, heads, Sq, Skv], fp32 (probs_dtype = MMFB_PROBS_F32) or bf16 (MMFB_PROBS_BF16),
 *   aligned to its element size.  Every element is written and nothing outside it.
 *   Without drop_mask a row sums to 1 (up to rounding).  With drop_mask (the keep bits the forward used) it is the
 *   post-dropout probability the reference returns in train mode: dropped entries are exactly 0 and kept ones are
 *   scaled by drop_scale = 1/(1-p).
 * Returns MMFB_ERR_ARG for a bad dtype, a null pointer or a shape mmfb_attention_fwd rejects.  One kernel launch; limits as
 * mmfb_attention_fwd.  There is no packed (varlen) variant. */
enum { MMFB_PROBS_F32 = 0, MMFB_PROBS_BF16 = 1 };
int mmfb_attention_probs(const mmfb_attn_args* args, void* probs, int probs_dtype, mmfb_stream stream);

/* LayerNorm over the last dimension (eps 1e-12 on this path), one warp per row.
 * fwd: x = LN(y)*gamma + beta, optional dropout on x (embeddings), saves mean / rstd (fp32 [M]).
 * bwd: dy = dLN(dx (+dx2)); dz = dropout-backward(dy) for the dense branch that fed y = dropout(dense)+resid;
 *      dgamma/dbeta/dbias (fp32 [H]) are ACCUMULATED (+=).  dz may equal dy (no dropout) or be NULL.
 * Limits (MMFB_ERR_ARG otherwise): H a multiple of 8 and <= 2048; rows are read and written as 16-byte vectors, so every
 * row tensor the call uses starts 16-byte aligned and, when M > 1, has a leading dimension that is a multiple of 8;
 * gamma and beta are 16-byte aligned in the forward, gamma in the backward when H > 1024. */
typedef struct {
  const void* y; int64_t ldy;        /* bf16 [M,H] pre-LN input */
  const void* gamma; const void* beta; /* bf16 [H] */
  void* x; int64_t ldx;              /* fwd output bf16 [M,H] */
  float* mean; float* rstd;          /* fp32 [M]: written by fwd, read by bwd */
  const uint32_t* drop_mask; int64_t ldmask; float drop_scale;
  float eps;
  /* backward */
  const void* dx; int64_t lddx;      /* bf16 [M,H] gradient wrt LN output */
  const void* dx2; int64_t lddx2;    /* optional second gradient term added to dx, or NULL */
  void* dy; int64_t lddy;            /* bf16 [M,H] gradient wrt y (residual branch) */
  void* dz; int64_t lddz;            /* bf16 [M,H] gradient wrt the dropped dense output */
  float* dgamma; float* dbeta; float* dbias;
  int M, H;
  float* workspace;                  /* backward: NULL and 0 = fp32 atomics for dgamma/dbeta/dbias (see below) */
  int64_t workspace_bytes;
} mmfb_ln_args;

int mmfb_layernorm_fwd(const mmfb_ln_args* args, mmfb_stream stream);
int mmfb_layernorm_bwd(const mmfb_ln_args* args, mmfb_stream stream);

/* The LayerNorm calls with a DEVICE int32 row bound m_dev (non-NULL, 4-byte aligned): with b = clamp(*m_dev, 0, M), read
 * when the kernel runs, only rows [0, b) of every row tensor (y, x, mean, rstd, dx, dx2, dy, dz, the keep bits) are read
 * or written; the rows at and past b keep what they held.  Every shape the unbounded calls take is covered, with the
 * same limits.  Row outputs equal those of the unbounded call with M = b, bit for bit.  dgamma / dbeta / dbias sum the
 * rows below b only.  With a workspace (sized for M) the chunks at and past b store zero partials, so the result equals
 * an unbounded ordered call with M = b (the same 128-row chunks) bit for bit.  An encoder layer captured in a CUDA graph
 * runs its LayerNorms this way on a fixed capacity of packed rows, of which the first b are tokens. */
int mmfb_layernorm_fwd_bounded(const mmfb_ln_args* args, const int32_t* m_dev, mmfb_stream stream);
int mmfb_layernorm_bwd_bounded(const mmfb_ln_args* args, const int32_t* m_dev, mmfb_stream stream);

/* Ordered reductions over rows.  The rows are cut into chunks of 128 (chunk k = rows [128k, 128k + 128)), a number that
 * depends on M alone.  Each chunk sums its rows in a fixed order (8 warps, warp w taking rows w, w + 8, ... of the chunk,
 * the warps' sums added in warp order) and STORES that partial into the workspace; a second kernel then adds the partials
 * to the destination in chunk order:  out[n] += ((part_0[n] + part_1[n]) + ...) + part_{K-1}[n].
 * The result has the same bits on every run and does not depend on the number of SMs.
 *   mmfb_layernorm_bwd with workspace set: dgamma / dbeta / dbias are accumulated this way; dy and dz are computed row by
 *   row exactly as without it (the same bits).  Size: mmfb_layernorm_bwd_workspace_bytes(M, H) = ceil(M/128) * 3 * H * 4.
 *   mmfb_colsum_ordered: the column sum of mmfb_colsum.  Size: mmfb_colsum_workspace_bytes(M, N) = ceil(M/128) * N * 4.
 * The size queries are host only (no device needed) and return 0 for an empty shape.  A layernorm_bwd with workspace or
 * workspace_bytes non-zero is an ordered call; an ordered call whose workspace is NULL, smaller than the size above or not
 * 16-byte aligned is MMFB_ERR_ARG before any launch. */
int64_t mmfb_layernorm_bwd_workspace_bytes(int M, int H);
int64_t mmfb_colsum_workspace_bytes(int M, int N);

/* out[n] += sum_m X[m,n]   (bias gradients), X bf16 [M,N], out fp32 [N].
 * Like the LayerNorm calls, the column sums, embed_compose / embed_scatter / embed_scatter_sorted and dropout_apply read
 * and write bf16 rows as 16-byte vectors: every row tensor they use starts 16-byte aligned and, when M > 1, has a leading
 * dimension that is a multiple of 8 (the gathered src / dsrc rows whatever M is); MMFB_ERR_ARG otherwise. */
int mmfb_colsum(const void* X, int64_t ldx, float* out, int M, int N, mmfb_stream stream);
/* mmfb_colsum with the chunk-ordered sum described above; workspace fp32, mmfb_colsum_workspace_bytes(M, N) bytes */
int mmfb_colsum_ordered(const void* X, int64_t ldx, float* out, int M, int N, float* workspace, int64_t workspace_bytes,
                        mmfb_stream stream);

/* Philox keep-bits for nn.Dropout(p): word w bit j <-> element 32*w+j, P(bit=1) = 1-p (16-bit resolution) */
int mmfb_dropout_bits(uint32_t* out, int64_t nwords, uint64_t seed, uint64_t offset, float p, mmfb_stream stream);
/* the same with a step counter in DEVICE memory mixed into the Philox counter (counter += *epoch << 40): a CUDA-graph replay of a
 * captured training step draws fresh masks as long as the graph increments *epoch (mmf_b200/graphs.py) */
int mmfb_dropout_bits_epoch(uint32_t* out, int64_t nwords, uint64_t seed, uint64_t offset, const uint64_t* epoch, float p,
                            mmfb_stream stream);
/* Keep bits for dropout(p) followed by stochastic depth (timm DropPath(p_path)) on an activation of M rows of H columns,
 * M = batch * rows_per_sample: out [M, ceil(H/32)] words.  Element (m, n) is kept when its element draw keeps it - the
 * draws of mmfb_dropout_bits(out, M * ceil(H/32), seed, offset, p) - AND sample m / rows_per_sample is kept, with
 * probability 1 - p_path from one draw per sample at Philox counter offset + 4 * M * ceil(H/32) + sample (16-bit
 * resolution), shared by the sample's rows.  Kept values are scaled by 1 / ((1 - p)(1 - p_path)).  The call uses the
 * counters [offset, offset + 4 * M * ceil(H/32) + batch).  M, H or rows_per_sample <= 0, M % rows_per_sample != 0, p or
 * p_path outside [0, 1) is MMFB_ERR_ARG. */
int mmfb_dropout_path_bits(uint32_t* out, int M, int H, int rows_per_sample, uint64_t seed, uint64_t offset, float p,
                           float p_path, mmfb_stream stream);
/* the same with the device step counter of mmfb_dropout_bits_epoch mixed into every counter it uses */
int mmfb_dropout_path_bits_epoch(uint32_t* out, int M, int H, int rows_per_sample, uint64_t seed, uint64_t offset,
                                 const uint64_t* epoch, float p, float p_path, mmfb_stream stream);

/* Embedding row composer (K1): y[r] = src0[src_row0[r]] + src1[src_row1[r]] + tab0[idx0[r]] + tab1[idx1[r]] +
 * tab2[idx2[r]]; a NULL pointer or a negative index drops the term.  src*: bf16 [*, ldsrc] dense rows (e.g. the
 * region-feature projection), tab*: bf16 [*, H] embedding tables.  Index arrays are int32 [M] on the device.
 * Covers BertVisioLinguisticEmbeddings (embeddings.py:329-370), ModalEmbeddings (mmbt.py:92-129),
 * HuggingfaceEmbeddings (huggingface.py:131-159) and BertImageFeatureEmbeddings (vilbert.py:904-913). */
typedef struct {
  const void* src[2]; int64_t ldsrc[2]; const int32_t* src_row[2];
  const void* tab[3]; const int32_t* tab_idx[3];
  void* y; int64_t ldy;
  int M, H;
} mmfb_compose_args;
int mmfb_embed_compose(const mmfb_compose_args* args, mmfb_stream stream);

/* backward of the composer: dsrc_k[src_row_k[r]] = dy[r] (bf16 store), dtab_k[idx_k[r]] += dy[r] (fp32 atomics) */
typedef struct {
  void* dsrc[2]; int64_t ldsrc[2]; const int32_t* src_row[2];
  float* dtab[3]; const int32_t* tab_idx[3];
  const void* dy; int64_t lddy;
  int M, H;
} mmfb_scatter_args;
int mmfb_embed_scatter(const mmfb_scatter_args* args, mmfb_stream stream);

/* table gradient with run aggregation: `sorted_idx` = the table indices in ascending order (negative = skip),
 * `order[k]` = the row of dy that sorted position k came from.  dtab[sorted_idx[k]] += dy[order[k]].
 * Equal indices are summed in registers first (one atomic per run of <= 32 rows instead of one per row). */
int mmfb_embed_scatter_sorted(const void* dy, int64_t lddy, const int32_t* order, const int32_t* sorted_idx, float* dtab,
                              int M, int H, mmfb_stream stream);
/* The same sum in an order fixed by the index vector alone.  Sorted positions are cut into chunks of 32 (one warp each);
 * a chunk sums each of its runs of equal indices in position order.  A run that lies inside one chunk has no other
 * contributor and is added to its table row directly.  A run that crosses chunk boundaries leaves one partial per chunk
 * in the workspace, and a second kernel adds  ((piece_first + piece_next) + ...) + piece_last  to the row, chunks in
 * position order.  Same bits on every run.  workspace: fp32, mmfb_embed_scatter_sorted_workspace_bytes(M, H) =
 * ceil(M/32) * 2 * H * 4 bytes (host only); NULL, smaller or not 16-byte aligned is MMFB_ERR_ARG before any launch. */
int64_t mmfb_embed_scatter_sorted_workspace_bytes(int M, int H);
int mmfb_embed_scatter_sorted_ordered(const void* dy, int64_t lddy, const int32_t* order, const int32_t* sorted_idx,
                                      float* dtab, int M, int H, float* workspace, int64_t workspace_bytes,
                                      mmfb_stream stream);

/* dz = dy where y > 0 else 0 (backward of the ReLU epilogue); contiguous bf16 buffers of n elements */
int mmfb_relu_bwd(const void* dy, const void* y, void* dz, int64_t n, mmfb_stream stream);

/* du = dh * GELU'(u) (erf GELU, the arithmetic of the MMFB_EPI_GELU_BWD epilogue) for a GELU that is NOT followed by a GEMM:
 * BertPredictionHeadTransform (dense -> gelu -> LayerNorm), HF modeling_bert via mmf/models/visual_bert.py:205-214.
 * Contiguous bf16 buffers of n elements. */
int mmfb_gelu_bwd(const void* dh, const void* u, void* du, int64_t n, mmfb_stream stream);

/* Cross-entropy over vocabulary-sized rows, forward and backward in ONE kernel: for every row m of the bf16 logits [M, V]
 * (row stride ldl, V % 8 == 0) with label[m] != ignore_index,  loss_m = logsumexp(z_m) - z_m[label[m]]  is added to
 * *loss_sum (and stored in row_loss[m] when given) and the row is OVERWRITTEN by
 * d(logits) = (softmax(z_m) - onehot(label[m])) * grad_scale;  ignored rows are overwritten by zeros.  A label outside
 * [0, V) that is not ignore_index is treated like ignore_index: zero gradient, row_loss 0, nothing added to *loss_sum.
 * *loss_sum takes one fp32 atomic per row, so its low bits depend on the order the rows finish; loss_sum may be NULL, and a
 * caller that needs the same bits on every run sums row_loss in a fixed order instead (d(logits) is per row and exact).
 * Replaces CrossEntropyLoss(ignore_index=-1) over prediction_scores.view(-1, vocab_size) of the masked-LM heads
 * (mmf/models/visual_bert.py:215,269-277; mmf/models/transformers/heads/mlm.py:46-97) inside the chunked
 * linear + cross-entropy head: the full [tokens, 30522] logits tensor never exists in HBM. */
int mmfb_ce_rows(void* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index, int M, int V, float grad_scale,
                 float* loss_sum, float* row_loss, mmfb_stream stream);

/* Static-rows masked-LM loss: the labelled rows of a batch, selected and counted on the device, so that a CUDA graph can
 * capture the head.  The head works on a fixed capacity of M rows (every row of its labels); rows [0, count) are the
 * labelled rows in row-major order, rows [count, M) hold zero features, ignore_index labels and zero gradients.
 *
 * mmfb_select_rows: labels int64 [M] (DEVICE).  One CTA, an ordered scan with no atomics (the same bits on every run).
 * A row is selected when its label != ignore_index (a label outside [0, V) is selected too; the loss kernel ignores it).
 *   state: DEVICE int32 [2 + 2M]: state[0] = count; state[1] = the fp32 bits of 1 / max(count, 1), the double reciprocal
 *          rounded once to fp32; pos = state + 2: pos[i] = the source row of output row i, -1 for i >= count;
 *          inv = state + 2 + M: inv[r] = the output row of source row r, -1 when r is not selected.
 *   labels_out: DEVICE int64 [M]: labels[pos[i]], ignore_index for i >= count.
 * mmfb_gather_rows: out[r] = idx[r] >= 0 ? x[idx[r]] : 0 for r < M (bf16 rows of H, H % 8 == 0, 16-byte aligned rows).
 *   With idx = pos it gathers the selected rows [M, H] (zeros past count); with idx = inv it is the backward, the full
 *   [M, H] input gradient (the gathered gradient at selected rows, zero elsewhere), with no atomics.
 * mmfb_ce_rows_bounded: mmfb_ce_rows on the rows below *m_dev rounded up to 128 (the GEMM's row tile) and with
 *   grad_scale = *scale_dev, both read from DEVICE memory when the kernel runs; rows at and past the rounded bound are
 *   not read or written (row_loss included).  The rows between *m_dev and the rounded bound must carry ignore_index.
 * mmfb_colsum_bounded: out[n] += sum over the rows below min(M, *m_dev) of X[m, n]; with a workspace
 *   (mmfb_colsum_workspace_bytes(M, N) bytes) the chunk-ordered sum of mmfb_colsum_ordered, which then adds the same
 *   partials as mmfb_colsum_ordered on the rows below the bound, followed by zero partials. */
int mmfb_select_rows(const int64_t* labels, int64_t ignore_index, int M, int32_t* state, int64_t* labels_out,
                     mmfb_stream stream);
int mmfb_gather_rows(const void* x, int64_t ldx, const int32_t* idx, void* out, int64_t ldo, int M, int H, mmfb_stream stream);
int mmfb_ce_rows_bounded(void* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index, int M, int V,
                         const int32_t* m_dev, const float* scale_dev, float* loss_sum, float* row_loss, mmfb_stream stream);
int mmfb_colsum_bounded(const void* X, int64_t ldx, float* out, int M, int N, const int32_t* m_dev, float* workspace,
                        int64_t workspace_bytes, mmfb_stream stream);

/* Static-rows region losses of masked region classification (MRC) and feature regression (MRFR): the rows of a fixed
 * capacity M of which the first count = clamp(*m_dev, 0, M) (DEVICE int32) are the masked regions, selected on the
 * device (mmfb_select_rows); row r < count takes its target from row tgt_idx[r] (DEVICE int32 [M]) of tgt (fp32, row
 * stride ldt).  Both write the gradient of their bf16 input IN PLACE, scaled by *scale_dev (DEVICE fp32, read when the
 * kernel runs), and the fp32 loss of row r to row_loss[r] (the caller sums the rows in a fixed order and multiplies by
 * the same scale).  Rows in [count, ceil(count / 128) * 128) get a zero gradient and a zero row loss, as the bounded
 * GEMMs that read them next require; rows at and past that are not read or written.  A count of 0 writes nothing.
 * mmfb_kl_rows_bounded: logits [M, V] (ldl >= V rounded up to 8): with p = softmax(z) and q the target row,
 *   row loss sum_j xlogy(q_j, q_j) - q_j log p_j, gradient (p_j sum_k q_k - q_j) * scale; columns [V, round8(V)) - the
 *   GEMM's zero padding - get a zero gradient.  F.kl_div(F.log_softmax(z), q, reduction="batchmean") with scale =
 *   1 / count (mmf/models/transformers/heads/mrc.py).
 * mmfb_mse_rows_bounded: pred [M, D]: row loss sum_j (z_j - t_j)^2, gradient 2 (z_j - t_j) * scale; F.mse_loss(z, t)
 *   with scale = 1 / (count * D) (heads/mrfr.py). */
int mmfb_kl_rows_bounded(void* logits, int64_t ldl, int M, int V, const float* tgt, int64_t ldt, const int32_t* tgt_idx,
                         const int32_t* m_dev, const float* scale_dev, float* row_loss, mmfb_stream stream);
int mmfb_mse_rows_bounded(void* pred, int64_t ldp, int M, int D, const float* tgt, int64_t ldt, const int32_t* tgt_idx,
                          const int32_t* m_dev, const float* scale_dev, float* row_loss, mmfb_stream stream);

/* out = a + b; contiguous bf16 buffers of n elements.  The residual-gradient join of a pre-LN layer (ViT: the residual
 * branches off BEFORE the LayerNorm, mmf/modules/vit.py:96-108), which a post-LN layer gets for free from the GEMM epilogue. */
int mmfb_add_bf16(const void* a, const void* b, void* out, int64_t n, mmfb_stream stream);

/* out[m, h] = keep-bit(m, h) ? x[m, h] * scale : 0  (bf16 [M, H] with row strides, bits = int32 words [M, ldm] as produced by
 * mmfb_dropout_bits).  Backward of a dropout that no LayerNorm follows: HF ViTSelfOutput / ViTOutput via vit.py:66-68. */
int mmfb_dropout_apply(const void* x, int64_t ldx, const uint32_t* bits, int64_t ldm, float scale, void* out, int64_t ldo,
                       int M, int H, mmfb_stream stream);

/* fp32 -> bf16 cast of a flat (parameter) buffer */
int mmfb_cast_f32_bf16(const float* in, void* out, int64_t n, mmfb_stream stream);

/* Fused AdamW step over a FLAT fp32 parameter / gradient buffer (the engine's ParamPack), optionally refreshing the
 * bf16 compute copy in the same pass.  SURVEY.md 8(f) item 2 - staged: parity tests exist, not yet run on the GPU.
 * Replaces the per-tensor loop of the reference's optimizer "adam_w" (mmf/modules/optimizers.py:8-17):
 *   mode 0: transformers AdamW arithmetic as restated in the reference (optimizers.py:60-84):
 *           m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= step_size * m / (sqrt(v) + eps);  p -= lr * wd * p
 *           with step_size = lr * sqrt(1-b2^t)/(1-b1^t) (or lr when correct_bias is off), computed by the host
 *   mode 1: torch.optim.AdamW arithmetic (the reference's fallback when transformers has no AdamW):
 *           p *= 1 - lr wd;  m += (g-m)(1-b1);  v = b2 v + (1-b2) g^2;  p -= step_size * m / (sqrt(v)/bc2_sqrt + eps)
 *           with step_size = lr/(1-b1^t), bc2_sqrt = sqrt(1-b2^t)
 * `group` (nullable) gives the hyper-parameter group of every 8-element block (parameters are padded to multiples of
 * 8 in the flat buffer); grad_scale multiplies the gradient first (1/loss_scale, clipping coefficient).  When
 * grad_scale_dev is set, the factor is grad_scale * *grad_scale_dev, the fp32 read from DEVICE memory when the kernel
 * runs (the clip coefficient mmfb_grad_norm writes), so a clipped step needs no device-to-host read.
 * When hp_dev is set, group g's lr / weight_decay / step_size / bc2_sqrt and beta1 / beta2 / eps are read from the
 * DEVICE table entry hp_dev[g] (written by mmfb_adamw_hparams) and the corresponding launch fields are ignored, so the
 * launch can be captured in a CUDA graph and replayed at later steps and learning rates.
 * Loss scaling (torch.amp.GradScaler), both nullable: when found_inf is set and *found_inf is non-zero, the launch writes
 * nothing (param, param_bf16, exp_avg, exp_avg_sq keep their bits).  When loss_scale_dev is set, every gradient is first
 * multiplied by inv = (float)(1.0 / (double)*loss_scale_dev) - GradScaler.unscale_'s factor - and then by the factor
 * above, as a second fp32 multiply: the bits of unscale_ followed by a step, for any scale. */
#define MMFB_ADAMW_MAX_GROUPS 8
typedef struct {
  float lr, weight_decay, step_size, bc2_sqrt;
  float beta1, beta2, eps, pad_;
} mmfb_adamw_hp;
typedef struct {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  void* param_bf16;          /* nullable */
  const uint8_t* group;      /* nullable: all blocks use group 0 */
  int64_t n;                 /* elements, multiple of 8 */
  int n_groups;
  float lr[MMFB_ADAMW_MAX_GROUPS];
  float weight_decay[MMFB_ADAMW_MAX_GROUPS];
  float step_size[MMFB_ADAMW_MAX_GROUPS];
  float bc2_sqrt[MMFB_ADAMW_MAX_GROUPS];
  float beta1, beta2, eps, grad_scale;
  int mode;
  const float* loss_scale_dev;   /* nullable: DEVICE fp32 loss scale S; gradients are multiplied by 1/S first */
  const float* found_inf;        /* nullable: DEVICE fp32; non-zero makes the launch a no-op */
  const float* grad_scale_dev;   /* nullable: DEVICE fp32 factor applied on top of grad_scale */
  const mmfb_adamw_hp* hp_dev;   /* nullable: DEVICE [n_groups] hyper-parameters replacing the launch fields (last) */
} mmfb_adamw_args;
int mmfb_adamw(const mmfb_adamw_args* args, mmfb_stream stream);

/* Device-side AdamW hyper-parameters, one CTA: for every slot s (a parameter, or a pack's parameter group) that is not
 * MMFB_ADAMW_SLOT_FROZEN, step[s] += 1 and, with t = step[s] and g = groups[slots[s].group], in fp64 then rounded once
 * to fp32 (the formulas of mmf_b200.optim.B200AdamW._group_hp):
 *   mode 0: step_size = lr * sqrt(1 - b2^t) / (1 - b1^t) with MMFB_ADAMW_SLOT_CORRECT_BIAS, lr without; bc2_sqrt = 1
 *   mode 1: step_size = lr / (1 - b1^t);  bc2_sqrt = sqrt(1 - b2^t)
 * hp[s] = {lr, weight_decay, step_size, bc2_sqrt, b1, b2, eps}.  A frozen slot (pack parameters the optimizer does not
 * own) keeps its step and gets lr = weight_decay = step_size = 0, bc2_sqrt = 1.  `groups` is the table the host stages
 * before each step (the values a learning-rate scheduler writes); `slots`, `step` and `hp` stay put.
 * found_inf (nullable, DEVICE fp32): when *found_inf is non-zero the launch writes nothing - no step count advances, as a
 * step that GradScaler skips does not count in torch's fused Adam. */
#define MMFB_ADAMW_SLOT_CORRECT_BIAS 1
#define MMFB_ADAMW_SLOT_FROZEN 2
typedef struct {
  double lr, weight_decay, beta1, beta2, eps;
} mmfb_adamw_group_hp;
typedef struct {
  int group;                 /* index into groups */
  int flags;                 /* MMFB_ADAMW_SLOT_* */
} mmfb_adamw_slot;
typedef struct {
  const mmfb_adamw_group_hp* groups;   /* DEVICE [groups used by slots] */
  const mmfb_adamw_slot* slots;        /* DEVICE [n_slots] */
  int64_t* step;                       /* DEVICE [n_slots] step counts */
  mmfb_adamw_hp* hp;                   /* DEVICE [n_slots] */
  int n_slots;
  int mode;                            /* 0 transformers, 1 torch (as mmfb_adamw) */
  const float* found_inf;              /* nullable: DEVICE fp32; non-zero makes the launch a no-op */
} mmfb_adamw_hparams_args;
int mmfb_adamw_hparams(const mmfb_adamw_hparams_args* args, mmfb_stream stream);

/* One AdamW launch over any number of separate fp32 tensors (parameters outside the flat packs), with the per-element
 * arithmetic of mmfb_adamw (the same device function: bit-identical results element for element).  Segment s updates
 * n elements at param / grad / exp_avg / exp_avg_sq (contiguous fp32, any 4-byte alignment) with hyper-parameters
 * hp[slot].  head: 0-3 elements before the first element at which all four pointers are 16-byte aligned, or -1 when
 * they never are together (every element is then accessed singly).  The segment owns the CTAs [first_block,
 * first_block + ceil((n + lead) / MMFB_ADAMW_SEGMENT_BLOCK)), lead = (8 - head) % 8 for head > 0 and 0 otherwise;
 * first_block is the running sum over the segments before it and n_blocks the total.  Gradients are multiplied by
 * grad_scale (times *grad_scale_dev when set) first; loss_scale_dev and found_inf act as in mmfb_adamw. */
#define MMFB_ADAMW_SEGMENT_BLOCK 2048
typedef struct {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t n;
  int slot;
  int first_block;
  int head;
  int pad_;
} mmfb_adamw_segment;
typedef struct {
  const mmfb_adamw_segment* segments;  /* DEVICE [n_segments] */
  int n_segments;
  int n_blocks;
  const mmfb_adamw_hp* hp;             /* DEVICE, indexed by the segments' slots */
  float grad_scale;
  int mode;
  const float* grad_scale_dev;         /* nullable */
  const float* loss_scale_dev;         /* nullable: DEVICE fp32 loss scale, as in mmfb_adamw */
  const float* found_inf;              /* nullable: DEVICE fp32 skip flag, as in mmfb_adamw */
} mmfb_adamw_segments_args;
int mmfb_adamw_segments(const mmfb_adamw_segments_args* args, mmfb_stream stream);

/* Global L2 norm of a list of gradient segments and torch's clip coefficient, on the device, in two launches:
 *   total_norm = sqrt(sum over every element x of every segment of x^2)
 *   clip_coef  = min(max_norm / (total_norm + 1e-6), 1)   (fp32, as torch.nn.utils.clip_grad_norm_; NaN stays NaN)
 * out[0] = total_norm, out[1] = clip_coef (DEVICE fp32 [2]); clip_coef is what mmfb_adamw's grad_scale_dev reads.
 * `segments` is a DEVICE array: segment s covers n elements (fp32 or bf16, contiguous) at ptr and owns the partial-sum
 * blocks [first_block, first_block + ceil(n / MMFB_GRAD_NORM_BLOCK)); first_block is the running sum of the blocks of the
 * segments before it and n_blocks the total (the table is not checked on the device).  `partials` is DEVICE fp64
 * workspace [n_blocks].  Block b sums the squares of its MMFB_GRAD_NORM_BLOCK elements in fp64 in a fixed order into
 * partials[b]; the second launch adds the partials in a fixed order: no atomics, and the result depends only on the
 * segment lengths and dtypes, so repeated calls give the same bits in every mode.  The fp32 norm is within one fp32 ulp of
 * the exact norm.  Non-finite gradients give an inf / NaN norm, as torch's with error_if_nonfinite=False.
 * norm_type must be 2 (MMFB_ERR_ARG otherwise).  max_norm_scale_dev (nullable, DEVICE fp32 S) makes the threshold
 * max_norm * S, one fp32 multiply when the kernel runs: the clip of loss-scaled gradients at max_norm times the loss
 * scale, without reading S on the host. */
#define MMFB_GRAD_NORM_BLOCK 16384
#define MMFB_GRAD_F32 0
#define MMFB_GRAD_BF16 1
typedef struct {
  const void* ptr;
  int64_t n;
  int dtype;                 /* MMFB_GRAD_F32 or MMFB_GRAD_BF16 */
  int first_block;
} mmfb_grad_segment;
typedef struct {
  const mmfb_grad_segment* segments;   /* DEVICE [n_segments] */
  int n_segments;
  int n_blocks;
  double* partials;                    /* DEVICE fp64 [n_blocks] */
  float* out;                          /* DEVICE fp32 [2] */
  float max_norm;
  float norm_type;
  const float* max_norm_scale_dev;     /* nullable: DEVICE fp32 factor on max_norm */
} mmfb_grad_norm_args;
int mmfb_grad_norm(const mmfb_grad_norm_args* args, mmfb_stream stream);

/* Optimal-transport distance of word-region alignment (UNITER's WRA loss): cosine cost, the IPOT transport plan and
 * trace(C T) in ONE kernel, one CTA per sample; the gradient through the cosine cost in a second one.  Replaces
 * optimal_transport_dist (mmf/modules/ot.py:80-102: cost_matrix_cosine :15-25, ipot :37-77, trace :28-34) as called by
 * the WRA head (mmf/models/transformers/heads/wra.py:64-76) and follows it operation for operation in fp32:
 *   C[m,n] = 1 - x^[m] . y^[n],  x^ = x / max(|x|, 1e-5);  0 where m >= x_len or n >= y_len
 *   sigma = 1 / x_len (0 on padding), T = 1, A = exp(-C^T / beta) (both 0 on padded pairs)
 *   iterations x { Q = A * T;  k x { delta = 1 / (y_len * Q sigma + 1e4 * y_pad);  sigma = 1 / (x_len * delta Q + 1e4 * x_pad) };
 *                  T = delta * Q * sigma };   T = 0 on padded pairs;   dist = sum_{m,n} C[m,n] T[n,m]
 * (k > 1 raises a shape error in the reference unless M = 1; the inner pass above is its evident intent.)
 * x: bf16 text rows, sample b row m at x + b * bsx + m * ldx (elements); y: bf16 region rows likewise - both may be views
 * into one [B, M + N, H] encoder output.  x_len / y_len: int32 [B] in HOST memory (they are validated and travel to the
 * kernel as launch parameters): the valid rows of a sample are its first x_len / y_len rows; rows past them are not read.
 * fwd writes dist fp32 [B], plan fp32 [B, N, M] (exact zeros on padded pairs), optionally cost fp32 [B, M, N], and
 * saved fp32 [B, 2 * (M + N)] for the backward (the clamped row norms and each row's x^ . dx^ term).
 * bwd: the reference detaches the plan (ot.py:98-101), so d dist / d C = T^T.  Given g = d loss / d dist fp32 [B] and
 * plan / saved of the forward it writes dx, dy (bf16, addressed like x and y; all M / N rows, exact zeros at padded rows):
 *   dx[m] = (d - x^[m] (x^[m] . d)) / |x_m|,  d = -g * sum_n T[n,m] y^[n]   (no projection term where |x_m| was clamped).
 * Limits (MMFB_ERR_ARG otherwise): 1 <= M, N <= 128; H a multiple of 64 up to 1024; 1 <= x_len <= M, 1 <= y_len <= N;
 * beta > 0, iterations >= 1, k >= 1; x, y, dx, dy 16-byte aligned with row and sample pitches that are multiples of 8.
 * One launch per 256 samples. */
typedef struct {
  const void* x; int64_t ldx; int64_t bsx;
  const void* y; int64_t ldy; int64_t bsy;
  const int32_t* x_len; const int32_t* y_len;   /* HOST int32 [B] */
  float* dist;                                  /* fp32 [B] (fwd) */
  float* plan;                                  /* fp32 [B, N, M]: written by fwd, read by bwd */
  float* cost;                                  /* fp32 [B, M, N] or NULL (fwd) */
  float* saved;                                 /* fp32 [B, 2 * (M + N)]: written by fwd, read by bwd */
  /* backward only */
  const float* g;                               /* fp32 [B] */
  void* dx; int64_t lddx; int64_t bsdx;
  void* dy; int64_t lddy; int64_t bsdy;
  int B, M, N, H;
  float beta; int iterations; int k;            /* fwd; the reference's defaults are 0.5, 50, 1 */
} mmfb_ot_args;
int mmfb_ot_fwd(const mmfb_ot_args* args, mmfb_stream stream);
int mmfb_ot_bwd(const mmfb_ot_args* args, mmfb_stream stream);

/* library / diagnostics */
const char* mmfb_last_error(void);
int mmfb_version(void);
int mmfb_device_ok(void);          /* 1 if the current device is sm_90 */
int64_t mmfb_launch_count(void);   /* number of kernels this library has launched in this process */

#ifdef __cplusplus
}
#endif

/* the device planner of skip-padding packings (mmfb_plan_packing) */
#include "mmfb200_plan.h"
/* the device update: learning-rate schedules and the fused non-finite check (mmfb_lr_schedule, mmfb_grad_*check) */
#include "mmfb200_update.h"
/* the capturable AdamW step gated per slot (mmfb_adamw_active, mmfb_adamw_hparams_active, mmfb_adamw_segments_active) */
#include "mmfb200_active.h"

#endif /* MMFB200_H_ */
