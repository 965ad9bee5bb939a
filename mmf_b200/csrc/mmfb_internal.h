// Internal host-side declarations shared by the translation units of libmmfb200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mmfb200.h"

namespace mmfb {

enum {
  EPI_BIAS = MMFB_EPI_BIAS,
  EPI_BIAS_GELU = MMFB_EPI_BIAS_GELU,
  EPI_BIAS_DROP_RESID = MMFB_EPI_BIAS_DROP_RESID,
  EPI_GELU_BWD = MMFB_EPI_GELU_BWD,
  EPI_ADD_AUX = MMFB_EPI_ADD_AUX,
  EPI_ATOMIC_F32 = MMFB_EPI_ATOMIC_F32,
  EPI_BIAS_RELU = MMFB_EPI_BIAS_RELU,
  EPI_BIAS_GELU_DROP = MMFB_EPI_BIAS_GELU_DROP,
  EPI_GELU_DROP_BWD = MMFB_EPI_GELU_DROP_BWD,
  // internal: the ordered split-K weight gradient - unit (tile, split s) stores its fp32 partial into slice s of the
  // caller's workspace [S, M, N] (plain stores), and a second kernel adds the slices into C in split order
  EPI_PARTIAL_F32 = 100
};

// Rows per chunk of the ordered column sums (colsum, LayerNorm parameter gradients): chunk k holds rows
// [k * ORDER_ROWS, (k + 1) * ORDER_ROWS), so the number of chunks and every partial depend on M alone.
constexpr int ORDER_ROWS = 128;
// Sorted positions per chunk of the ordered embedding-table scatter (the run-aggregation window of one warp).
constexpr int SCATTER_CHUNK = 32;
inline int order_chunks(int M) { return (M + ORDER_ROWS - 1) / ORDER_ROWS; }
// Rows a device-bounded row kernel (ce_rows_bounded) covers: the device count rounded up to this, the GEMM's row tile,
// so that every row a bounded GEMM tile reads next has been written (include/mmfb200.h, "Device bounds").
constexpr int BOUNDED_ROW_TILE = 128;

// split-K factor the GEMM actually runs for K and the requested `splits`: every split owns at least one k-block
int gemm_effective_splits(int K, int splits);
int64_t gemm_workspace_bytes(int M, int N, int K, int splits);
int64_t ln_bwd_workspace_bytes(int M, int H);
int64_t colsum_workspace_bytes(int M, int N);
int64_t scatter_sorted_workspace_bytes(int M, int H);

// records a thread-local error message and returns `code`
int set_error(int code, const char* fmt, ...);
int num_sms();
void count_launch(int n = 1);

// bf16 2-D tensor map: tensor [outer, inner] with row stride `ld` elements, box {box_inner, box_outer},
// SWIZZLE_128B (box_inner must be 64), out-of-bounds elements read as zero / are not written.
int make_tmap_2d(CUtensorMap* map, const void* ptr, int64_t inner, int64_t outer, int64_t ld, int box_inner,
                 int box_outer);
// bf16 3-D tensor map: tensor [d2, d1, inner] with strides ld1 (rows) and ld2 (batches) in elements
int make_tmap_3d(CUtensorMap* map, const void* ptr, int64_t inner, int64_t d1, int64_t d2, int64_t ld1,
                 int64_t ld2, int box_inner, int box_d1);

// Launch with the programmatic-stream-serialization attribute (common.cuh: griddep_launch / griddep_wait).
template <typename... KArgs, typename... Args>
cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#define MMFB_LAUNCH(kern, grid, block, smem, stream, ...) \
  (void)::mmfb::launch_k(kern, dim3(grid), dim3(block), static_cast<size_t>(smem), stream, __VA_ARGS__)

// m_dev / k_dev: the device bounds of mmfb_gemm_bounded (NULL: none)
int gemm(const mmfb_gemm_args& a, cudaStream_t stream, const int32_t* m_dev = nullptr, const int32_t* k_dev = nullptr);
int attn_fwd(const mmfb_attn_args& a, cudaStream_t stream);
int attn_bwd(const mmfb_attn_args& a, cudaStream_t stream);
int attn_varlen_fwd(const mmfb_attn_args& a, const int32_t* cu, int total, cudaStream_t stream);
int attn_varlen_bwd(const mmfb_attn_args& a, const int32_t* cu, int total, cudaStream_t stream);
int attn_varlen_cross_fwd(const mmfb_attn_args& a, const int32_t* cu_q, int total_q, const int32_t* cu_kv, int total_kv,
                          cudaStream_t stream);
int attn_varlen_cross_bwd(const mmfb_attn_args& a, const int32_t* cu_q, int total_q, const int32_t* cu_kv, int total_kv,
                          cudaStream_t stream);
int attn_probs(const mmfb_attn_args& a, void* probs, int probs_dtype, cudaStream_t stream);
// dense self-attention with a causal tail (attention_causal.cu), called by attn_fwd / attn_bwd after their checks
int attn_causal_fwd(const mmfb_attn_args& a, cudaStream_t stream);
int attn_causal_bwd(const mmfb_attn_args& a, cudaStream_t stream);
// packed self-attention with a causal tail (attention_varlen_causal.cu)
int attn_varlen_causal_fwd(const mmfb_attn_args& a, const int32_t* cu, int total, cudaStream_t stream);
int attn_varlen_causal_bwd(const mmfb_attn_args& a, const int32_t* cu, int total, cudaStream_t stream);
// m_dev: the device row bound of mmfb_layernorm_*_bounded (NULL: none)
int ln_fwd(const mmfb_ln_args& a, cudaStream_t s, const int32_t* m_dev = nullptr);
int ln_bwd(const mmfb_ln_args& a, cudaStream_t s, const int32_t* m_dev = nullptr);
int colsum(const void* X, int64_t ldx, float* out, int M, int N, cudaStream_t s);
int colsum_ordered(const void* X, int64_t ldx, float* out, int M, int N, float* ws, int64_t ws_bytes, cudaStream_t s);
int dropout_bits(uint32_t* out, int64_t nwords, uint64_t seed, uint64_t offset, float p, const uint64_t* epoch, cudaStream_t s);
int dropout_path_bits(uint32_t* out, int M, int H, int rows_per_sample, uint64_t seed, uint64_t offset, float p, float p_path,
                      const uint64_t* epoch, cudaStream_t s);
int compose(const mmfb_compose_args& a, cudaStream_t s);
int scatter(const mmfb_scatter_args& a, cudaStream_t s);
int cast_params(const float* in, void* out, int64_t n, cudaStream_t s);
int relu_bwd(const void* dy, const void* y, void* dz, int64_t n, cudaStream_t s);
int adamw(const mmfb_adamw_args& a, cudaStream_t s);
int adamw_hparams(const mmfb_adamw_hparams_args& a, cudaStream_t s);
int adamw_segments(const mmfb_adamw_segments_args& a, cudaStream_t s);
int grad_norm(const mmfb_grad_norm_args& a, float* found_inf, cudaStream_t s);
int grad_check(const mmfb_grad_segment* segs, int n_segs, int n_blocks, double* flags, float* found_inf, cudaStream_t s);
int lr_schedule(const mmfb_lr_schedule_args& a, cudaStream_t s);
int ce_rows(void* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index, int M, int V, float grad_scale,
            float* loss_sum, float* row_loss, cudaStream_t s);
int ce_rows_bounded(void* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index, int M, int V,
                    const int32_t* m_dev, const float* scale_dev, float* loss_sum, float* row_loss, cudaStream_t s);
int colsum_bounded(const void* X, int64_t ldx, float* out, int M, int N, const int32_t* m_dev, float* ws, int64_t ws_bytes,
                   cudaStream_t s);
int kl_rows_bounded(void* logits, int64_t ldl, int M, int V, const float* tgt, int64_t ldt, const int32_t* tgt_idx,
                    const int32_t* m_dev, const float* scale_dev, float* row_loss, cudaStream_t s);
int mse_rows_bounded(void* pred, int64_t ldp, int M, int D, const float* tgt, int64_t ldt, const int32_t* tgt_idx,
                     const int32_t* m_dev, const float* scale_dev, float* row_loss, cudaStream_t s);
int select_rows(const int64_t* labels, int64_t ignore_index, int M, int32_t* state, int64_t* labels_out, cudaStream_t s);
int gather_rows(const void* x, int64_t ldx, const int32_t* idx, void* out, int64_t ldo, int M, int H, cudaStream_t s);
int add_bf16(const void* a, const void* b, void* out, int64_t n, cudaStream_t s);
int dropout_apply(const void* x, int64_t ldx, const uint32_t* bits, int64_t ldm, float scale, void* out, int64_t ldo, int M,
                  int H, cudaStream_t s);
int gelu_bwd(const void* dh, const void* u, void* du, int64_t n, cudaStream_t s);
int scatter_sorted(const void* dy, int64_t lddy, const int32_t* order, const int32_t* sorted_idx, float* dtab, int M,
                   int H, cudaStream_t s);
int scatter_sorted_ordered(const void* dy, int64_t lddy, const int32_t* order, const int32_t* sorted_idx, float* dtab, int M,
                           int H, float* ws, int64_t ws_bytes, cudaStream_t s);
int ot_fwd(const mmfb_ot_args& a, cudaStream_t s);
int ot_bwd(const mmfb_ot_args& a, cudaStream_t s);

}  // namespace mmfb
