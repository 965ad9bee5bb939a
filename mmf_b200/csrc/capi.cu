// extern "C" surface of libmmfb200.so + host utilities (error state, device query, tensor maps).
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <atomic>

#include "mmfb_internal.h"

namespace mmfb {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// libcuda is resolved at first use through the runtime, so the library loads on a CPU-only host
static encode_tiled_fn get_encode() {
  static encode_tiled_fn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<encode_tiled_fn>(p);
  }
  return fn;
}

int make_tmap_2d(CUtensorMap* map, const void* ptr, int64_t inner, int64_t outer, int64_t ld, int box_inner,
                 int box_outer) {
  encode_tiled_fn enc = get_encode();
  if (!enc) return set_error(MMFB_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld % 8))
    return set_error(MMFB_ERR_ARG, "tensor map: base must be 16-byte aligned and ld a multiple of 8 (ptr=%p ld=%lld)",
                     ptr, (long long)ld);
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(MMFB_ERR_CUDA, "cuTensorMapEncodeTiled(2d inner=%lld outer=%lld ld=%lld box=%dx%d) failed: %d",
                     (long long)inner, (long long)outer, (long long)ld, box_inner, box_outer, (int)r);
  return MMFB_OK;
}

int make_tmap_3d(CUtensorMap* map, const void* ptr, int64_t inner, int64_t d1, int64_t d2, int64_t ld1, int64_t ld2,
                 int box_inner, int box_d1) {
  encode_tiled_fn enc = get_encode();
  if (!enc) return set_error(MMFB_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld1 % 8) || (ld2 % 8))
    return set_error(MMFB_ERR_ARG, "tensor map: base must be 16-byte aligned and strides multiples of 8");
  cuuint64_t dims[3] = {(cuuint64_t)inner, (cuuint64_t)d1, (cuuint64_t)d2};
  cuuint64_t strides[2] = {(cuuint64_t)ld1 * 2, (cuuint64_t)ld2 * 2};
  cuuint32_t box[3] = {(cuuint32_t)box_inner, (cuuint32_t)box_d1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(MMFB_ERR_CUDA, "cuTensorMapEncodeTiled(3d) failed: %d", (int)r);
  return MMFB_OK;
}

static int check_device() {
  static int ok = -1;
  if (ok < 0) {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
      cudaGetLastError();
      return 0;  // not cached: a device may appear later (e.g. after CUDA_VISIBLE_DEVICES changes)
    }
    ok = (major == 9) ? 1 : 0;
  }
  return ok;
}

}  // namespace mmfb

using namespace mmfb;

#define MMFB_REQUIRE_DEVICE()                                                                              \
  do {                                                                                                     \
    if (!check_device())                                                                                   \
      return set_error(MMFB_ERR_DEVICE, "libmmfb200 needs an sm_90 (H100) device; there is no CPU fallback"); \
  } while (0)

extern "C" {

const char* mmfb_last_error(void) { return g_err; }
int mmfb_version(void) { return 100; }
int mmfb_device_ok(void) { return check_device(); }
int64_t mmfb_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int mmfb_gemm(const mmfb_gemm_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_gemm: null args");
  MMFB_REQUIRE_DEVICE();
  return gemm(*args, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_gemm_bounded(const mmfb_gemm_args* args, const int32_t* m_dev, const int32_t* k_dev, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_gemm_bounded: null args");
  MMFB_REQUIRE_DEVICE();
  return gemm(*args, reinterpret_cast<cudaStream_t>(stream), m_dev, k_dev);
}

int mmfb_attention_fwd(const mmfb_attn_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_fwd: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_fwd(*args, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_attention_bwd(const mmfb_attn_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_bwd: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_bwd(*args, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_attention_varlen_fwd(const mmfb_attn_args* args, const int32_t* cu_seqlens, int total, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_varlen_fwd: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_varlen_fwd(*args, cu_seqlens, total, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_attention_varlen_bwd(const mmfb_attn_args* args, const int32_t* cu_seqlens, int total, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_varlen_bwd: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_varlen_bwd(*args, cu_seqlens, total, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_attention_varlen_causal_fwd(const mmfb_attn_args* args, const int32_t* cu_seqlens, int total, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_varlen_causal_fwd: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_varlen_causal_fwd(*args, cu_seqlens, total, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_attention_varlen_causal_bwd(const mmfb_attn_args* args, const int32_t* cu_seqlens, int total, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_varlen_causal_bwd: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_varlen_causal_bwd(*args, cu_seqlens, total, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_attention_varlen_cross_fwd(const mmfb_attn_args* args, const int32_t* cu_q, int total_q, const int32_t* cu_kv,
                                    int total_kv, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_varlen_cross_fwd: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_varlen_cross_fwd(*args, cu_q, total_q, cu_kv, total_kv, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_attention_varlen_cross_bwd(const mmfb_attn_args* args, const int32_t* cu_q, int total_q, const int32_t* cu_kv,
                                    int total_kv, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_varlen_cross_bwd: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_varlen_cross_bwd(*args, cu_q, total_q, cu_kv, total_kv, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_attention_probs(const mmfb_attn_args* args, void* probs, int probs_dtype, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_attention_probs: null args");
  MMFB_REQUIRE_DEVICE();
  return attn_probs(*args, probs, probs_dtype, reinterpret_cast<cudaStream_t>(stream));
}

int mmfb_layernorm_fwd(const mmfb_ln_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_layernorm_fwd: null args");
  MMFB_REQUIRE_DEVICE();
  return ln_fwd(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_layernorm_bwd(const mmfb_ln_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_layernorm_bwd: null args");
  MMFB_REQUIRE_DEVICE();
  return ln_bwd(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_layernorm_fwd_bounded(const mmfb_ln_args* args, const int32_t* m_dev, mmfb_stream stream) {
  if (!args || !m_dev) return set_error(MMFB_ERR_ARG, "mmfb_layernorm_fwd_bounded: null pointer");
  MMFB_REQUIRE_DEVICE();
  return ln_fwd(*args, reinterpret_cast<cudaStream_t>(stream), m_dev);
}
int mmfb_layernorm_bwd_bounded(const mmfb_ln_args* args, const int32_t* m_dev, mmfb_stream stream) {
  if (!args || !m_dev) return set_error(MMFB_ERR_ARG, "mmfb_layernorm_bwd_bounded: null pointer");
  MMFB_REQUIRE_DEVICE();
  return ln_bwd(*args, reinterpret_cast<cudaStream_t>(stream), m_dev);
}
int mmfb_colsum(const void* X, int64_t ldx, float* out, int M, int N, mmfb_stream stream) {
  if (!X || !out) return set_error(MMFB_ERR_ARG, "mmfb_colsum: null pointer");
  MMFB_REQUIRE_DEVICE();
  return colsum(X, ldx, out, M, N, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_colsum_ordered(const void* X, int64_t ldx, float* out, int M, int N, float* workspace, int64_t workspace_bytes,
                        mmfb_stream stream) {
  if (!X || !out) return set_error(MMFB_ERR_ARG, "mmfb_colsum_ordered: null pointer");
  MMFB_REQUIRE_DEVICE();
  return colsum_ordered(X, ldx, out, M, N, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}
int64_t mmfb_gemm_workspace_bytes(int M, int N, int K, int splits) { return gemm_workspace_bytes(M, N, K, splits); }
int64_t mmfb_layernorm_bwd_workspace_bytes(int M, int H) { return ln_bwd_workspace_bytes(M, H); }
int64_t mmfb_colsum_workspace_bytes(int M, int N) { return colsum_workspace_bytes(M, N); }
int64_t mmfb_embed_scatter_sorted_workspace_bytes(int M, int H) { return scatter_sorted_workspace_bytes(M, H); }
int mmfb_dropout_bits(uint32_t* out, int64_t nwords, uint64_t seed, uint64_t offset, float p, mmfb_stream stream) {
  if (!out) return set_error(MMFB_ERR_ARG, "mmfb_dropout_bits: null pointer");
  MMFB_REQUIRE_DEVICE();
  return dropout_bits(out, nwords, seed, offset, p, nullptr, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_dropout_bits_epoch(uint32_t* out, int64_t nwords, uint64_t seed, uint64_t offset, const uint64_t* epoch, float p,
                            mmfb_stream stream) {
  if (!out || !epoch) return set_error(MMFB_ERR_ARG, "mmfb_dropout_bits_epoch: null pointer");
  MMFB_REQUIRE_DEVICE();
  return dropout_bits(out, nwords, seed, offset, p, epoch, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_dropout_path_bits(uint32_t* out, int M, int H, int rows_per_sample, uint64_t seed, uint64_t offset, float p,
                           float p_path, mmfb_stream stream) {
  if (!out) return set_error(MMFB_ERR_ARG, "mmfb_dropout_path_bits: null pointer");
  MMFB_REQUIRE_DEVICE();
  return dropout_path_bits(out, M, H, rows_per_sample, seed, offset, p, p_path, nullptr,
                           reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_dropout_path_bits_epoch(uint32_t* out, int M, int H, int rows_per_sample, uint64_t seed, uint64_t offset,
                                 const uint64_t* epoch, float p, float p_path, mmfb_stream stream) {
  if (!out || !epoch) return set_error(MMFB_ERR_ARG, "mmfb_dropout_path_bits_epoch: null pointer");
  MMFB_REQUIRE_DEVICE();
  return dropout_path_bits(out, M, H, rows_per_sample, seed, offset, p, p_path, epoch,
                           reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_embed_compose(const mmfb_compose_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_embed_compose: null args");
  MMFB_REQUIRE_DEVICE();
  return compose(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_embed_scatter(const mmfb_scatter_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_embed_scatter: null args");
  MMFB_REQUIRE_DEVICE();
  return scatter(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_embed_scatter_sorted(const void* dy, int64_t lddy, const int32_t* order, const int32_t* sorted_idx, float* dtab,
                              int M, int H, mmfb_stream stream) {
  if (!dy || !order || !sorted_idx || !dtab) return set_error(MMFB_ERR_ARG, "mmfb_embed_scatter_sorted: null pointer");
  MMFB_REQUIRE_DEVICE();
  return scatter_sorted(dy, lddy, order, sorted_idx, dtab, M, H, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_embed_scatter_sorted_ordered(const void* dy, int64_t lddy, const int32_t* order, const int32_t* sorted_idx,
                                      float* dtab, int M, int H, float* workspace, int64_t workspace_bytes,
                                      mmfb_stream stream) {
  if (!dy || !order || !sorted_idx || !dtab)
    return set_error(MMFB_ERR_ARG, "mmfb_embed_scatter_sorted_ordered: null pointer");
  MMFB_REQUIRE_DEVICE();
  return scatter_sorted_ordered(dy, lddy, order, sorted_idx, dtab, M, H, workspace, workspace_bytes,
                                reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_relu_bwd(const void* dy, const void* y, void* dz, int64_t n, mmfb_stream stream) {
  if (!dy || !y || !dz) return set_error(MMFB_ERR_ARG, "mmfb_relu_bwd: null pointer");
  MMFB_REQUIRE_DEVICE();
  return relu_bwd(dy, y, dz, n, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_gelu_bwd(const void* dh, const void* u, void* du, int64_t n, mmfb_stream stream) {
  if (!dh || !u || !du) return set_error(MMFB_ERR_ARG, "mmfb_gelu_bwd: null pointer");
  MMFB_REQUIRE_DEVICE();
  return gelu_bwd(dh, u, du, n, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_ce_rows(void* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index, int M, int V, float grad_scale,
                 float* loss_sum, float* row_loss, mmfb_stream stream) {
  if (!logits || !labels) return set_error(MMFB_ERR_ARG, "mmfb_ce_rows: null pointer");
  MMFB_REQUIRE_DEVICE();
  return ce_rows(logits, ldl, labels, ignore_index, M, V, grad_scale, loss_sum, row_loss, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_ce_rows_bounded(void* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index, int M, int V,
                         const int32_t* m_dev, const float* scale_dev, float* loss_sum, float* row_loss, mmfb_stream stream) {
  if (!logits || !labels || !m_dev || !scale_dev) return set_error(MMFB_ERR_ARG, "mmfb_ce_rows_bounded: null pointer");
  MMFB_REQUIRE_DEVICE();
  return ce_rows_bounded(logits, ldl, labels, ignore_index, M, V, m_dev, scale_dev, loss_sum, row_loss,
                         reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_colsum_bounded(const void* X, int64_t ldx, float* out, int M, int N, const int32_t* m_dev, float* workspace,
                        int64_t workspace_bytes, mmfb_stream stream) {
  if (!X || !out || !m_dev) return set_error(MMFB_ERR_ARG, "mmfb_colsum_bounded: null pointer");
  MMFB_REQUIRE_DEVICE();
  return colsum_bounded(X, ldx, out, M, N, m_dev, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_kl_rows_bounded(void* logits, int64_t ldl, int M, int V, const float* tgt, int64_t ldt, const int32_t* tgt_idx,
                         const int32_t* m_dev, const float* scale_dev, float* row_loss, mmfb_stream stream) {
  if (!logits || !tgt || !tgt_idx || !m_dev || !scale_dev || !row_loss)
    return set_error(MMFB_ERR_ARG, "mmfb_kl_rows_bounded: null pointer");
  MMFB_REQUIRE_DEVICE();
  return kl_rows_bounded(logits, ldl, M, V, tgt, ldt, tgt_idx, m_dev, scale_dev, row_loss, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_mse_rows_bounded(void* pred, int64_t ldp, int M, int D, const float* tgt, int64_t ldt, const int32_t* tgt_idx,
                          const int32_t* m_dev, const float* scale_dev, float* row_loss, mmfb_stream stream) {
  if (!pred || !tgt || !tgt_idx || !m_dev || !scale_dev || !row_loss)
    return set_error(MMFB_ERR_ARG, "mmfb_mse_rows_bounded: null pointer");
  MMFB_REQUIRE_DEVICE();
  return mse_rows_bounded(pred, ldp, M, D, tgt, ldt, tgt_idx, m_dev, scale_dev, row_loss, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_select_rows(const int64_t* labels, int64_t ignore_index, int M, int32_t* state, int64_t* labels_out,
                     mmfb_stream stream) {
  if (!labels || !state || !labels_out) return set_error(MMFB_ERR_ARG, "mmfb_select_rows: null pointer");
  MMFB_REQUIRE_DEVICE();
  return select_rows(labels, ignore_index, M, state, labels_out, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_gather_rows(const void* x, int64_t ldx, const int32_t* idx, void* out, int64_t ldo, int M, int H, mmfb_stream stream) {
  if (!x || !idx || !out) return set_error(MMFB_ERR_ARG, "mmfb_gather_rows: null pointer");
  MMFB_REQUIRE_DEVICE();
  return gather_rows(x, ldx, idx, out, ldo, M, H, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_add_bf16(const void* a, const void* b, void* out, int64_t n, mmfb_stream stream) {
  if (!a || !b || !out) return set_error(MMFB_ERR_ARG, "mmfb_add_bf16: null pointer");
  MMFB_REQUIRE_DEVICE();
  return add_bf16(a, b, out, n, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_dropout_apply(const void* x, int64_t ldx, const uint32_t* bits, int64_t ldm, float scale, void* out, int64_t ldo,
                       int M, int H, mmfb_stream stream) {
  if (!x || !bits || !out) return set_error(MMFB_ERR_ARG, "mmfb_dropout_apply: null pointer");
  MMFB_REQUIRE_DEVICE();
  return dropout_apply(x, ldx, bits, ldm, scale, out, ldo, M, H, reinterpret_cast<cudaStream_t>(stream));
}
// the loss-scaling fields of the optimizer launches: nullable DEVICE fp32 scalars
static bool misaligned_f32(const float* p) { return (reinterpret_cast<uintptr_t>(p) & 3) != 0; }

int mmfb_adamw(const mmfb_adamw_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_adamw: null args");
  if (misaligned_f32(args->loss_scale_dev) || misaligned_f32(args->found_inf))
    return set_error(MMFB_ERR_ARG, "mmfb_adamw: loss_scale_dev and found_inf must be 4-byte aligned");
  MMFB_REQUIRE_DEVICE();
  return adamw(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_adamw_hparams(const mmfb_adamw_hparams_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_adamw_hparams: null args");
  if (misaligned_f32(args->found_inf)) return set_error(MMFB_ERR_ARG, "mmfb_adamw_hparams: found_inf must be 4-byte aligned");
  MMFB_REQUIRE_DEVICE();
  return adamw_hparams(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_adamw_segments(const mmfb_adamw_segments_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_adamw_segments: null args");
  if (misaligned_f32(args->loss_scale_dev) || misaligned_f32(args->found_inf))
    return set_error(MMFB_ERR_ARG, "mmfb_adamw_segments: loss_scale_dev and found_inf must be 4-byte aligned");
  MMFB_REQUIRE_DEVICE();
  return adamw_segments(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_grad_norm(const mmfb_grad_norm_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_grad_norm: null args");
  if (args->norm_type != 2.0f)
    return set_error(MMFB_ERR_ARG, "mmfb_grad_norm: only norm_type 2 is supported (got %g)", args->norm_type);
  if (misaligned_f32(args->max_norm_scale_dev))
    return set_error(MMFB_ERR_ARG, "mmfb_grad_norm: max_norm_scale_dev must be 4-byte aligned");
  MMFB_REQUIRE_DEVICE();
  return grad_norm(*args, nullptr, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_grad_norm_check(const mmfb_grad_norm_args* args, float* found_inf, mmfb_stream stream) {
  if (!args || !found_inf) return set_error(MMFB_ERR_ARG, "mmfb_grad_norm_check: null pointer");
  if (args->norm_type != 2.0f)
    return set_error(MMFB_ERR_ARG, "mmfb_grad_norm_check: only norm_type 2 is supported (got %g)", args->norm_type);
  if (misaligned_f32(args->max_norm_scale_dev) || misaligned_f32(found_inf))
    return set_error(MMFB_ERR_ARG, "mmfb_grad_norm_check: max_norm_scale_dev and found_inf must be 4-byte aligned");
  MMFB_REQUIRE_DEVICE();
  return grad_norm(*args, found_inf, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_grad_check(const mmfb_grad_segment* segments, int n_segments, int n_blocks, double* flags, float* found_inf,
                    mmfb_stream stream) {
  if (!segments || !flags || !found_inf) return set_error(MMFB_ERR_ARG, "mmfb_grad_check: null pointer");
  if (n_segments < 1 || n_blocks < 1)
    return set_error(MMFB_ERR_ARG, "mmfb_grad_check: need at least one segment and one block (got %d, %d)", n_segments,
                     n_blocks);
  if (misaligned_f32(found_inf)) return set_error(MMFB_ERR_ARG, "mmfb_grad_check: found_inf must be 4-byte aligned");
  MMFB_REQUIRE_DEVICE();
  return grad_check(segments, n_segments, n_blocks, flags, found_inf, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_lr_schedule(const mmfb_lr_schedule_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_lr_schedule: null args");
  if (!args->counter || !args->base_lr || !args->lr) return set_error(MMFB_ERR_ARG, "mmfb_lr_schedule: null pointer");
  if (args->desc.kind < MMFB_LR_WARMUP_LINEAR || args->desc.kind > MMFB_LR_PYTHIA)
    return set_error(MMFB_ERR_ARG, "mmfb_lr_schedule: unknown schedule kind %d", args->desc.kind);
  MMFB_REQUIRE_DEVICE();
  return lr_schedule(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_cast_f32_bf16(const float* in, void* out, int64_t n, mmfb_stream stream) {
  if (!in || !out) return set_error(MMFB_ERR_ARG, "mmfb_cast_f32_bf16: null pointer");
  MMFB_REQUIRE_DEVICE();
  return cast_params(in, out, n, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_ot_fwd(const mmfb_ot_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_ot_fwd: null args");
  MMFB_REQUIRE_DEVICE();
  return ot_fwd(*args, reinterpret_cast<cudaStream_t>(stream));
}
int mmfb_ot_bwd(const mmfb_ot_args* args, mmfb_stream stream) {
  if (!args) return set_error(MMFB_ERR_ARG, "mmfb_ot_bwd: null args");
  MMFB_REQUIRE_DEVICE();
  return ot_bwd(*args, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
