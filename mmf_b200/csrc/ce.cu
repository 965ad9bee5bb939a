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

}  // namespace mmfb
