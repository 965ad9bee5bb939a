// Cross-entropy over vocabulary-sized rows, forward AND backward in one pass over each row (sm_90a).
//
//   loss_i  = logsumexp(z_i) - z_i[label_i]                      (rows with label == ignore_index contribute nothing)
//   dz_i    = (softmax(z_i) - onehot(label_i)) * grad_scale      written IN PLACE over the logits (bf16)
//
// This is the row kernel of the chunked "linear + cross-entropy" head (mmf_b200/ops.py linear_cross_entropy): the
// vocabulary GEMM produces a CHUNK of logits [rows, V], this kernel turns it into d(logits) and the summed loss, and the
// dgrad / wgrad GEMMs consume it at once - the [B*S, 30522] logits of the reference's masked-LM head
// (mmf/models/visual_bert.py:269-277: CrossEntropyLoss(ignore_index=-1) over prediction_scores.view(-1, vocab)) never
// exist in HBM as a whole.  HBM-bound: one block per row, the row (61 KB at V = 30528) is read from HBM once, re-read from
// L1/L2 for the second and third sweep, and written once.
#include "common.cuh"
#include "mmfb_internal.h"

namespace mmfb {

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float t = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, t) : v + t;
  }
  __syncthreads();                    // red[] may still be read from the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

// BOUNDED: the rows come from a fixed capacity of which only a prefix, counted on the device, is labelled: rows at or
// past *m_dev rounded up to BOUNDED_ROW_TILE are not touched (the rows between carry ignore_index and are zeroed, which
// is what the bounded GEMMs that read them next need), and grad_scale is *scale_dev.
template <bool BOUNDED = false>
__global__ void __launch_bounds__(256)
ce_rows_kernel(bf16* __restrict__ z, int64_t ldz, const int64_t* __restrict__ labels, int64_t ignore_index, int M, int V,
               float grad_scale, float* __restrict__ loss_sum, float* __restrict__ row_loss,
               const int32_t* __restrict__ m_dev = nullptr, const float* __restrict__ scale_dev = nullptr) {
  griddep_launch();
  griddep_wait();
  __shared__ float red[8];
  const int row = blockIdx.x;
  if (row >= M) return;
  if constexpr (BOUNDED) {
    const int b = max(*m_dev, 0);
    if (row >= (b + BOUNDED_ROW_TILE - 1) / BOUNDED_ROW_TILE * BOUNDED_ROW_TILE) return;
    grad_scale = *scale_dev;
  }
  bf16* zr = z + static_cast<int64_t>(row) * ldz;
  const int64_t label = labels[row];
  const bool active = label != ignore_index && label >= 0 && label < V;
  const int nvec = V >> 3;            // V is a multiple of 8 (the GEMM's N granularity)
  if (!active) {
    // the row takes no part in the loss: its gradient is zero
    const uint4 zero = make_uint4(0, 0, 0, 0);
    for (int i = threadIdx.x; i < nvec; i += 256) reinterpret_cast<uint4*>(zr)[i] = zero;
    if (row_loss != nullptr && threadIdx.x == 0) row_loss[row] = 0.0f;
    return;
  }
  const uint4* z4 = reinterpret_cast<const uint4*>(zr);
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < nvec; i += 256) {
    const uint4 u = z4[i];
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(a.x, a.y), fmaxf(b.x, b.y)), fmaxf(fmaxf(c.x, c.y), fmaxf(d.x, d.y))));
  }
  mx = block_reduce(mx, red, true);
  const float mx2 = mx * 1.4426950408889634f;
  float sum = 0.0f;
  for (int i = threadIdx.x; i < nvec; i += 256) {
    const uint4 u = z4[i];
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    sum += exp2f(fmaf(a.x, 1.4426950408889634f, -mx2)) + exp2f(fmaf(a.y, 1.4426950408889634f, -mx2)) +
           exp2f(fmaf(b.x, 1.4426950408889634f, -mx2)) + exp2f(fmaf(b.y, 1.4426950408889634f, -mx2)) +
           exp2f(fmaf(c.x, 1.4426950408889634f, -mx2)) + exp2f(fmaf(c.y, 1.4426950408889634f, -mx2)) +
           exp2f(fmaf(d.x, 1.4426950408889634f, -mx2)) + exp2f(fmaf(d.y, 1.4426950408889634f, -mx2));
  }
  sum = block_reduce(sum, red, false);
  const float zl = __bfloat162float(zr[label]);      // read before the row is overwritten (every thread: same address)
  __syncthreads();
  const float inv = grad_scale / sum;
  const int lvec = static_cast<int>(label >> 3), lsub = static_cast<int>(label & 7);
  for (int i = threadIdx.x; i < nvec; i += 256) {
    const uint4 u = z4[i];
    float v[8];
    float2 t;
    t = unpack_bf16x2(u.x); v[0] = t.x; v[1] = t.y;
    t = unpack_bf16x2(u.y); v[2] = t.x; v[3] = t.y;
    t = unpack_bf16x2(u.z); v[4] = t.x; v[5] = t.y;
    t = unpack_bf16x2(u.w); v[6] = t.x; v[7] = t.y;
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = exp2f(fmaf(v[e], 1.4426950408889634f, -mx2)) * inv;
    if (i == lvec) v[lsub] -= grad_scale;
    uint4 o;
    o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
    o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
    reinterpret_cast<uint4*>(zr)[i] = o;
  }
  if (threadIdx.x == 0) {
    const float li = mx + logf(sum) - zl;
    if (row_loss != nullptr) row_loss[row] = li;
    if (loss_sum != nullptr) atomicAdd(loss_sum, li);
  }
}

int ce_rows(void* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index, int M, int V, float grad_scale,
            float* loss_sum, float* row_loss, cudaStream_t s) {
  if (M <= 0 || V <= 0 || (V % 8) || (ldl % 8)) return set_error(MMFB_ERR_ARG, "ce_rows: bad shape %dx%d (ld %lld)", M, V, (long long)ldl);
  if (reinterpret_cast<uintptr_t>(logits) & 15) return set_error(MMFB_ERR_ARG, "ce_rows: logits must be 16-byte aligned");
  MMFB_LAUNCH(ce_rows_kernel<false>, M, 256, 0, s, reinterpret_cast<bf16*>(logits), ldl, labels, ignore_index, M, V, grad_scale,
              loss_sum, row_loss, nullptr, nullptr);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "ce_rows launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

int ce_rows_bounded(void* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index, int M, int V,
                    const int32_t* m_dev, const float* scale_dev, float* loss_sum, float* row_loss, cudaStream_t s) {
  if (M <= 0 || V <= 0 || (V % 8) || (ldl % 8)) return set_error(MMFB_ERR_ARG, "ce_rows_bounded: bad shape %dx%d (ld %lld)", M, V, (long long)ldl);
  if (reinterpret_cast<uintptr_t>(logits) & 15) return set_error(MMFB_ERR_ARG, "ce_rows_bounded: logits must be 16-byte aligned");
  if ((reinterpret_cast<uintptr_t>(m_dev) | reinterpret_cast<uintptr_t>(scale_dev)) & 3)
    return set_error(MMFB_ERR_ARG, "ce_rows_bounded: m_dev / scale_dev must be 4-byte aligned");
  MMFB_LAUNCH(ce_rows_kernel<true>, M, 256, 0, s, reinterpret_cast<bf16*>(logits), ldl, labels, ignore_index, M, V, 0.0f,
              loss_sum, row_loss, m_dev, scale_dev);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "ce_rows_bounded launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

// The region heads' losses on a fixed capacity of rows (masked region classification / feature regression of UNITER,
// mmf/models/transformers/heads/mrc.py and mrfr.py), bounded by a device count like ce_rows_bounded: row r < count is
// the r-th masked region, its target is row tgt_idx[r] of `tgt`; rows in [count, rounded bound) get a zero gradient and
// a zero row loss (the bounded GEMMs after this read them); rows at and past the rounded bound are not touched.
//
// kl:  q = target row (soft labels), p = softmax(z):  loss_r = sum_j xlogy(q_j, q_j) - q_j log p_j
//      dz_j = (p_j sum_k q_k - q_j) * scale                  (F.kl_div(F.log_softmax(z), q) per row)
//      columns [V, ldz-rounded-to-8) are the GEMM's zero padding: their gradient is written as 0
// mse: loss_r = sum_j (z_j - t_j)^2,  dz_j = 2 (z_j - t_j) * scale    (F.mse_loss per row)
// The gradient is written in place over z (bf16); row_loss[r] gets the fp32 row loss, summed by the caller.
__device__ __forceinline__ int bounded_rows(const int32_t* m_dev, int M, int* count) {
  const int b = min(max(*m_dev, 0), M);
  *count = b;
  return min(M, (b + BOUNDED_ROW_TILE - 1) / BOUNDED_ROW_TILE * BOUNDED_ROW_TILE);
}

__global__ void __launch_bounds__(256)
kl_rows_bounded_kernel(bf16* __restrict__ z, int64_t ldz, int M, int V, int Vp, const float* __restrict__ tgt, int64_t ldt,
                       const int32_t* __restrict__ tgt_idx, const int32_t* __restrict__ m_dev,
                       const float* __restrict__ scale_dev, float* __restrict__ row_loss) {
  griddep_launch();
  griddep_wait();
  __shared__ float red[8];
  const int row = blockIdx.x;
  int count;
  if (row >= bounded_rows(m_dev, M, &count)) return;
  bf16* zr = z + static_cast<int64_t>(row) * ldz;
  if (row >= count) {
    for (int i = threadIdx.x; i < Vp; i += 256) zr[i] = __float2bfloat16(0.0f);
    if (threadIdx.x == 0) row_loss[row] = 0.0f;
    return;
  }
  const float* q = tgt + static_cast<int64_t>(tgt_idx[row]) * ldt;
  float mx = -INFINITY, qs = 0.0f, qlq = 0.0f, qz = 0.0f;
  for (int i = threadIdx.x; i < V; i += 256) {
    const float zi = __bfloat162float(zr[i]), qi = q[i];
    mx = fmaxf(mx, zi);
    qs += qi;
    qlq += qi == 0.0f ? 0.0f : qi * logf(qi);
    qz += qi * zi;
  }
  mx = block_reduce(mx, red, true);
  qs = block_reduce(qs, red, false);
  qlq = block_reduce(qlq, red, false);
  qz = block_reduce(qz, red, false);
  const float mx2 = mx * 1.4426950408889634f;
  float se = 0.0f;
  for (int i = threadIdx.x; i < V; i += 256) se += exp2f(fmaf(__bfloat162float(zr[i]), 1.4426950408889634f, -mx2));
  se = block_reduce(se, red, false);
  const float scale = *scale_dev, f = qs / se;
  for (int i = threadIdx.x; i < Vp; i += 256) {
    float g = 0.0f;
    if (i < V) g = (exp2f(fmaf(__bfloat162float(zr[i]), 1.4426950408889634f, -mx2)) * f - q[i]) * scale;
    zr[i] = __float2bfloat16(g);
  }
  if (threadIdx.x == 0) row_loss[row] = qlq - qz + (mx + logf(se)) * qs;
}

__global__ void __launch_bounds__(256)
mse_rows_bounded_kernel(bf16* __restrict__ z, int64_t ldz, int M, int D, const float* __restrict__ tgt, int64_t ldt,
                        const int32_t* __restrict__ tgt_idx, const int32_t* __restrict__ m_dev,
                        const float* __restrict__ scale_dev, float* __restrict__ row_loss) {
  griddep_launch();
  griddep_wait();
  __shared__ float red[8];
  const int row = blockIdx.x;
  int count;
  if (row >= bounded_rows(m_dev, M, &count)) return;
  bf16* zr = z + static_cast<int64_t>(row) * ldz;
  if (row >= count) {
    for (int i = threadIdx.x; i < D; i += 256) zr[i] = __float2bfloat16(0.0f);
    if (threadIdx.x == 0) row_loss[row] = 0.0f;
    return;
  }
  const float* t = tgt + static_cast<int64_t>(tgt_idx[row]) * ldt;
  const float scale2 = 2.0f * *scale_dev;
  float s = 0.0f;
  for (int i = threadIdx.x; i < D; i += 256) {
    const float d = __bfloat162float(zr[i]) - t[i];
    s += d * d;
    zr[i] = __float2bfloat16(d * scale2);
  }
  s = block_reduce(s, red, false);
  if (threadIdx.x == 0) row_loss[row] = s;
}

static int region_rows_check(const char* what, const void* z, int64_t ldz, int M, int cols, int padded_cols,
                             const void* tgt, int64_t ldt, const void* tgt_idx, const void* m_dev, const void* scale_dev) {
  if (M <= 0 || cols <= 0 || ldz < padded_cols || ldt < cols)
    return set_error(MMFB_ERR_ARG, "%s: bad shape %dx%d (ldz %lld, ldt %lld)", what, M, cols, (long long)ldz, (long long)ldt);
  if ((reinterpret_cast<uintptr_t>(z) & 1) || (reinterpret_cast<uintptr_t>(tgt) & 3) || (reinterpret_cast<uintptr_t>(tgt_idx) & 3) ||
      ((reinterpret_cast<uintptr_t>(m_dev) | reinterpret_cast<uintptr_t>(scale_dev)) & 3))
    return set_error(MMFB_ERR_ARG, "%s: misaligned buffer", what);
  return MMFB_OK;
}

int kl_rows_bounded(void* logits, int64_t ldl, int M, int V, const float* tgt, int64_t ldt, const int32_t* tgt_idx,
                    const int32_t* m_dev, const float* scale_dev, float* row_loss, cudaStream_t s) {
  const int Vp = (V + 7) / 8 * 8;
  int rc = region_rows_check("kl_rows_bounded", logits, ldl, M, V, Vp, tgt, ldt, tgt_idx, m_dev, scale_dev);
  if (rc != MMFB_OK) return rc;
  MMFB_LAUNCH(kl_rows_bounded_kernel, M, 256, 0, s, reinterpret_cast<bf16*>(logits), ldl, M, V, Vp, tgt, ldt, tgt_idx,
              m_dev, scale_dev, row_loss);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "kl_rows_bounded launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

int mse_rows_bounded(void* pred, int64_t ldp, int M, int D, const float* tgt, int64_t ldt, const int32_t* tgt_idx,
                     const int32_t* m_dev, const float* scale_dev, float* row_loss, cudaStream_t s) {
  int rc = region_rows_check("mse_rows_bounded", pred, ldp, M, D, D, tgt, ldt, tgt_idx, m_dev, scale_dev);
  if (rc != MMFB_OK) return rc;
  MMFB_LAUNCH(mse_rows_bounded_kernel, M, 256, 0, s, reinterpret_cast<bf16*>(pred), ldp, M, D, tgt, ldt, tgt_idx, m_dev,
              scale_dev, row_loss);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "mse_rows_bounded launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

}  // namespace mmfb
