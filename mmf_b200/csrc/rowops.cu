// Row-wise (HBM-bound) kernels of the fusion block: LayerNorm forward/backward (with the dropout
// backward and bias-gradient column sums folded in), bias-gradient column sums, Philox dropout keep-bit
// generation, the embedding "compose + LayerNorm" kernel (region-feature / token gather + type /
// position add + LN) and its scatter backward, fp32 -> bf16 parameter cast.
//
// All of them are one-warp-per-row, 16-byte vectorised, fully coalesced; nothing here is GEMM-shaped.
// Reference ops: nn.LayerNorm(eps=1e-12) in HF BertSelfOutput/BertOutput (called at
// mmf/modules/hf_layers.py:248,290) and mmf/models/vilbert.py:254,303,483,490,911; nn.Dropout at the same
// sites; embeddings mmf/modules/embeddings.py:329-370,423-459, mmf/models/mmbt.py:92-129,
// mmf/models/transformers/backends/huggingface.py:131-159, mmf/models/vilbert.py:904-913.
#include "common.cuh"
#include "mmfb_internal.h"

#include <initializer_list>

namespace mmfb {

constexpr int MAXV = 8;         // per-lane 8-element vectors: rows up to 8*256 = 2048 columns
constexpr int ROW_WARPS = 8;    // warps per block

__device__ __forceinline__ void ld8(const bf16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 t;
  t = unpack_bf16x2(u.x); f[0] = t.x; f[1] = t.y;
  t = unpack_bf16x2(u.y); f[2] = t.x; f[3] = t.y;
  t = unpack_bf16x2(u.z); f[4] = t.x; f[5] = t.y;
  t = unpack_bf16x2(u.w); f[6] = t.x; f[7] = t.y;
}
__device__ __forceinline__ void st8(bf16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// ----------------------------------------------------------------------------------------------
// LayerNorm forward:  x = LN(y) * gamma + beta  (+ optional dropout on the OUTPUT, used by the embeddings)
// BOUNDED (all LayerNorm kernels): only the rows below min(M, *m_dev) are read and written - an encoder layer's rows on a
// fixed capacity of which a device-counted prefix is valid (packed skip-padding under CUDA-graph capture).
// ----------------------------------------------------------------------------------------------
template <int NV, bool BOUNDED = false>
__global__ void __launch_bounds__(ROW_WARPS * 32)
ln_fwd_kernel(const bf16* __restrict__ y, int64_t ldy, const bf16* __restrict__ gamma,
              const bf16* __restrict__ beta, bf16* __restrict__ x, int64_t ldx, float* __restrict__ mean,
              float* __restrict__ rstd, const uint32_t* __restrict__ dmask, int64_t ldmask, float dscale, int M,
              int H, float eps, const int32_t* __restrict__ m_dev = nullptr) {
  griddep_launch();
  griddep_wait();
  if constexpr (BOUNDED) M = min(M, max(*m_dev, 0));
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * ROW_WARPS + (threadIdx.x >> 5);
  if (row >= M) return;
  float v[NV][8];
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int col = i * 256 + lane * 8;
    if (col < H) {
      ld8(y + row * ldy + col, v[i]);
#pragma unroll
      for (int e = 0; e < 8; ++e) s += v[i][e];
    }
  }
  const float mu = warp_sum(s) / H;
  float ss = 0.0f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int col = i * 256 + lane * 8;
    if (col < H) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float d = v[i][e] - mu; ss += d * d; }
    }
  }
  const float rs = rsqrtf(warp_sum(ss) / H + eps);
  if (lane == 0) {
    if (mean) mean[row] = mu;
    if (rstd) rstd[row] = rs;
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int col = i * 256 + lane * 8;
    if (col < H) {
      float g[8], b[8], o[8];
      ld8(gamma + col, g);
      ld8(beta + col, b);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mu) * rs * g[e] + b[e];
      if (dmask != nullptr) {
        const uint32_t w = __ldg(dmask + row * ldmask + (col >> 5));
        const uint32_t bits = (w >> (col & 31)) & 0xFFu;
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = ((bits >> e) & 1u) ? o[e] * dscale : 0.0f;
      }
      st8(x + row * ldx + col, o);
    }
  }
}

// ----------------------------------------------------------------------------------------------
// LayerNorm backward (+ dropout backward of the pre-LN dense branch + bias gradient)
//   dy    = gamma*rstd * (dx - mean_h(dx*gamma) ... ) standard LN backward wrt the pre-LN sum y = z + resid
//   dz    = dy * keep * dscale        (gradient of the dense output that was dropped)   [== dy when no dropout]
//   dgamma += sum_rows dx * xhat ; dbeta += sum_rows dx ; dbias += sum_rows dz
// dx_in may carry an extra additive term dx2 (the residual gradient arriving from a later consumer).
// A persistent grid (grid-stride over row groups) keeps the number of fp32 atomics at 3*H per block.
// Two kernels, chosen by H: ln_bwd_stream_kernel for H <= 1024, ln_bwd_kernel for 1024 < H <= 2048.
// ----------------------------------------------------------------------------------------------
// ORDERED (both kernels): block b owns the rows of chunk b (ORDER_ROWS rows, warp w taking rows w, w + ROW_WARPS, ...) and
// stores its three column-sum sets to ws[b][which][H] instead of adding them to dgamma / dbeta / dbias; chunk_reduce_kernel
// adds them up in chunk order.  The row outputs dy / dz do not depend on which block computes a row.
// BOUNDED (both kernels): M becomes min(M, *m_dev) on the device.  The grid stays sized from M: an ordered chunk at or past
// the bound stores zero partials, so the reduce adds what an unbounded ordered call with M = bound adds, then zeros.
// Rows of up to MAXV * 256 columns: a warp loads, computes and stores a row held in registers, and only the other warps
// of the SM cover its load latency.
template <bool ORDERED, bool BOUNDED = false>
__global__ void __launch_bounds__(ROW_WARPS * 32)
ln_bwd_kernel(const bf16* __restrict__ dx, int64_t lddx, const bf16* __restrict__ dx2, int64_t lddx2,
              const bf16* __restrict__ y, int64_t ldy, const float* __restrict__ mean,
              const float* __restrict__ rstd, const bf16* __restrict__ gamma, bf16* __restrict__ dy, int64_t lddy,
              bf16* __restrict__ dz, int64_t lddz, const uint32_t* __restrict__ dmask, int64_t ldmask, float dscale,
              float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int M, int H,
              float* __restrict__ ws, const int32_t* __restrict__ m_dev = nullptr) {
  griddep_launch();
  griddep_wait();
  if constexpr (BOUNDED) M = min(M, max(*m_dev, 0));
  __shared__ float red[ROW_WARPS][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float ag[MAXV][8], ab[MAXV][8], az[MAXV][8];
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) { ag[i][e] = 0.0f; ab[i][e] = 0.0f; az[i][e] = 0.0f; }

  const int64_t row_end = ORDERED ? min(static_cast<int64_t>(M), (static_cast<int64_t>(blockIdx.x) + 1) * ORDER_ROWS) : M;
  const int64_t stride = ORDERED ? ROW_WARPS : static_cast<int64_t>(gridDim.x) * ROW_WARPS;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * (ORDERED ? ORDER_ROWS : ROW_WARPS) + warp; row < row_end;
       row += stride) {
    const float mu = mean[row], rs = rstd[row];
    float g[MAXV][8], d[MAXV][8], xh[MAXV][8];
    float s1 = 0.0f, s2 = 0.0f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int col = i * 256 + lane * 8;
      if (col < H) {
        float yy[8];
        ld8(dx + row * lddx + col, d[i]);
        if (dx2 != nullptr) {
          float t[8];
          ld8(dx2 + row * lddx2 + col, t);
#pragma unroll
          for (int e = 0; e < 8; ++e) d[i][e] += t[e];
        }
        ld8(y + row * ldy + col, yy);
        ld8(gamma + col, g[i]);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          xh[i][e] = (yy[e] - mu) * rs;
          const float dg = d[i][e] * g[i][e];
          s1 += dg;
          s2 += dg * xh[i][e];
          ag[i][e] += d[i][e] * xh[i][e];
          ab[i][e] += d[i][e];
        }
      }
    }
    s1 = warp_sum(s1) / H;
    s2 = warp_sum(s2) / H;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int col = i * 256 + lane * 8;
      if (col < H) {
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = rs * (d[i][e] * g[i][e] - s1 - xh[i][e] * s2);
        if (dy != nullptr) st8(dy + row * lddy + col, o);
        if (dmask != nullptr) {
          const uint32_t w = __ldg(dmask + row * ldmask + (col >> 5));
          const uint32_t bits = (w >> (col & 31)) & 0xFFu;
#pragma unroll
          for (int e = 0; e < 8; ++e) o[e] = ((bits >> e) & 1u) ? o[e] * dscale : 0.0f;
          st8(dz + row * lddz + col, o);
        } else if (dz != nullptr && dz != dy) {
          st8(dz + row * lddz + col, o);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) az[i][e] += o[e];
      }
    }
  }
  // block reduction of the three column-sum sets, 256 columns at a time, then one atomic per column
#pragma unroll
  for (int which = 0; which < 3; ++which) {
    float* dst = which == 0 ? dgamma : (which == 1 ? dbeta : dbias);
    if (dst == nullptr) continue;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      if (i * 256 >= H) break;
      __syncthreads();
#pragma unroll
      for (int e = 0; e < 8; ++e) red[warp][lane * 8 + e] = which == 0 ? ag[i][e] : (which == 1 ? ab[i][e] : az[i][e]);
      __syncthreads();
      const int c = threadIdx.x;  // 256 threads <-> 256 columns
      float t = 0.0f;
#pragma unroll
      for (int w = 0; w < ROW_WARPS; ++w) t += red[w][c];
      if (i * 256 + c < H) {
        if (ORDERED) ws[(static_cast<int64_t>(blockIdx.x) * 3 + which) * H + i * 256 + c] = t;
        else atomicAdd(dst + i * 256 + c, t);
      }
    }
  }
}

// bf16x2 word -> the two values as a packed fp32 pair (exact: a bf16 is the top half of an fp32)
__device__ __forceinline__ uint64_t unpack2(uint32_t w) {
  return pk2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}
__device__ __forceinline__ uint32_t pack2(uint64_t v) {
  float lo, hi;
  upk2(v, lo, hi);
  return pack_bf16x2(lo, hi);
}

// Single-pass streaming LayerNorm backward for rows of up to 4 * 256 columns.  Every warp owns a private ring of ST row
// slots in shared memory that its lane 0 fills with bulk async copies (cp.async.bulk, one per tensor row, completion on a
// per-slot mbarrier) ST rows ahead, so ST x 16 warps x 3 KB are in flight per SM whatever the warps are doing, and the
// row lives in shared memory across the two phases (no row registers).  Rows are read from HBM once; dy / dz are stored
// straight from registers.
// Instruction diet (a first version issued ~42 instructions per element and was issue-bound at 0.48 of the HBM peak):
// all arithmetic on packed fp32 pairs (common.cuh: pk2 / fma2), xhat as ONE fma (y * rstd - mean * rstd), the output as
// two (d * (gamma * rstd) - rstd * m1, then - rstd * m2 * xhat), gamma as fp32 in shared memory (LDS.128, no unpack),
// dropout applied to the PACKED bf16 result with an AND mask looked up per 8 keep-bits (256 x 16 B table in shared
// memory) instead of eight bit tests + selects; dbias sums the bf16 values that are stored (what the consumer reads).
__device__ __forceinline__ void bulk_load_1d(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
template <int NV, bool HAS_DX2, int ST, bool ORDERED, bool BOUNDED = false>
__global__ void __launch_bounds__(ROW_WARPS * 32, 2)
ln_bwd_stream_kernel(const bf16* __restrict__ dx, int64_t lddx, const bf16* __restrict__ dx2, int64_t lddx2,
                     const bf16* __restrict__ y, int64_t ldy, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const bf16* __restrict__ gamma, bf16* __restrict__ dy, int64_t lddy,
                     bf16* __restrict__ dz, int64_t lddz, const uint32_t* __restrict__ dmask, int64_t ldmask, float dscale,
                     float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int M_rows, int H,
                     float* __restrict__ ws, const int32_t* __restrict__ m_dev = nullptr) {
  griddep_launch();
  griddep_wait();
  if constexpr (BOUNDED) M_rows = min(M_rows, max(*m_dev, 0));
  // the bound of the rows this block visits: its chunk's end when ORDERED
  const int M = ORDERED ? min(M_rows, static_cast<int>(blockIdx.x + 1) * ORDER_ROWS) : M_rows;
  constexpr int NT = HAS_DX2 ? 3 : 2;                 // tensors per slot: dx, y (, dx2)
  constexpr int ROWB = NV * 512;                      // bytes reserved per tensor row in a slot
  extern __shared__ __align__(128) uint8_t ln_smem[];
  uint8_t* ring = ln_smem;                                                        // [ROW_WARPS][ST][NT][ROWB]
  float* red = reinterpret_cast<float*>(ring + ROW_WARPS * ST * NT * ROWB);       // [ROW_WARPS][256]
  float* sG = red + ROW_WARPS * 256;                                              // [NV * 256]
  uint32_t* sKeep = reinterpret_cast<uint32_t*>(sG + NV * 256);                   // [256][4]
  uint64_t* full = reinterpret_cast<uint64_t*>(sKeep + 1024);                     // [ROW_WARPS][ST]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = threadIdx.x; c < NV * 256; c += ROW_WARPS * 32) sG[c] = c < H ? __bfloat162float(gamma[c]) : 0.0f;
  {
    const uint32_t b = threadIdx.x;          // 256 threads <-> the 256 patterns of 8 keep-bits
#pragma unroll
    for (int k = 0; k < 4; ++k)
      sKeep[b * 4 + k] = (((b >> (2 * k)) & 1u) ? 0x0000ffffu : 0u) | (((b >> (2 * k + 1)) & 1u) ? 0xffff0000u : 0u);
  }
  if (threadIdx.x < ROW_WARPS * ST) mbar_init(&full[threadIdx.x], 1);
  fence_barrier_init();
  __syncthreads();
  uint8_t* my = ring + warp * (ST * NT * ROWB);
  uint64_t* my_full = full + warp * ST;
  const uint32_t row_bytes = static_cast<uint32_t>(H) * 2u;
  const int64_t stride = ORDERED ? ROW_WARPS : static_cast<int64_t>(gridDim.x) * ROW_WARPS;
  const int64_t row_first = static_cast<int64_t>(blockIdx.x) * (ORDERED ? ORDER_ROWS : ROW_WARPS) + warp;
  auto fill = [&](int slot, int64_t row) {            // lane 0
    uint8_t* d = my + slot * (NT * ROWB);
    mbar_expect_tx(&my_full[slot], NT * row_bytes);
    bulk_load_1d(d, dx + row * lddx, row_bytes, &my_full[slot]);
    bulk_load_1d(d + ROWB, y + row * ldy, row_bytes, &my_full[slot]);
    if (HAS_DX2) bulk_load_1d(d + 2 * ROWB, dx2 + row * lddx2, row_bytes, &my_full[slot]);
  };
  if (lane == 0) {
#pragma unroll
    for (int s0 = 0; s0 < ST; ++s0)
      if (row_first + s0 * stride < M) fill(s0, row_first + s0 * stride);
  }
  uint64_t ag[NV][4], ab[NV][4], az[NV][4];
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) { ag[i][k] = 0ull; ab[i][k] = 0ull; az[i][k] = 0ull; }
  const float invH = 1.0f / static_cast<float>(H);
  const uint64_t ds2 = pk2(dscale, dscale);
  float mu_n = 0.0f, rs_n = 0.0f;
  if (row_first < M) { mu_n = mean[row_first]; rs_n = rstd[row_first]; }
  int slot = 0;
  uint32_t phase = 0;
  for (int64_t row = row_first; row < M; row += stride) {
    const float mu = mu_n, rs = rs_n;
    if (row + stride < M) { mu_n = mean[row + stride]; rs_n = rstd[row + stride]; }   // one row ahead
    uint32_t keepw[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int col = i * 256 + lane * 8;
      keepw[i] = 0xFFu;
      if (dmask != nullptr && col < H) keepw[i] = (__ldg(dmask + row * ldmask + (col >> 5)) >> (col & 31)) & 0xFFu;
    }
    const float nmr = -mu * rs;
    const uint64_t rs2 = pk2(rs, rs), nmr2 = pk2(nmr, nmr);
    const uint8_t* sl = my + slot * (NT * ROWB);
    mbar_wait(&my_full[slot], phase);
    uint64_t s1 = 0ull, s2 = 0ull;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int col = i * 256 + lane * 8;
      if (col < H) {
        const uint4 dwv = *reinterpret_cast<const uint4*>(sl + col * 2);
        const uint4 ywv = *reinterpret_cast<const uint4*>(sl + ROWB + col * 2);
        const uint32_t da[4] = {dwv.x, dwv.y, dwv.z, dwv.w};
        const uint32_t ya[4] = {ywv.x, ywv.y, ywv.z, ywv.w};
        uint32_t xa[4] = {0u, 0u, 0u, 0u};
        if (HAS_DX2) {
          const uint4 t = *reinterpret_cast<const uint4*>(sl + 2 * ROWB + col * 2);
          xa[0] = t.x; xa[1] = t.y; xa[2] = t.z; xa[3] = t.w;
        }
        const float4 ga = *reinterpret_cast<const float4*>(sG + col), gb = *reinterpret_cast<const float4*>(sG + col + 4);
        const uint64_t g2[4] = {pk2(ga.x, ga.y), pk2(ga.z, ga.w), pk2(gb.x, gb.y), pk2(gb.z, gb.w)};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          uint64_t d2 = unpack2(da[k]);
          if (HAS_DX2) d2 = add2(d2, unpack2(xa[k]));
          const uint64_t xh2 = fma2(unpack2(ya[k]), rs2, nmr2);
          const uint64_t dg2 = mul2(d2, g2[k]);
          s1 = add2(s1, dg2);
          s2 = fma2(dg2, xh2, s2);
          ag[i][k] = fma2(d2, xh2, ag[i][k]);
          ab[i][k] = add2(ab[i][k], d2);
        }
      }
    }
    float s1a, s1b, s2a, s2b;
    upk2(s1, s1a, s1b);
    upk2(s2, s2a, s2b);
    const float m1 = warp_sum(s1a + s1b) * invH, m2 = warp_sum(s2a + s2b) * invH;
    const uint64_t nA2 = pk2(-rs * m1, -rs * m1), nB2 = pk2(-rs * m2, -rs * m2);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int col = i * 256 + lane * 8;
      if (col < H) {
        const uint4 dwv = *reinterpret_cast<const uint4*>(sl + col * 2);
        const uint4 ywv = *reinterpret_cast<const uint4*>(sl + ROWB + col * 2);
        const uint32_t da[4] = {dwv.x, dwv.y, dwv.z, dwv.w};
        const uint32_t ya[4] = {ywv.x, ywv.y, ywv.z, ywv.w};
        uint32_t xa[4] = {0u, 0u, 0u, 0u};
        if (HAS_DX2) {
          const uint4 t = *reinterpret_cast<const uint4*>(sl + 2 * ROWB + col * 2);
          xa[0] = t.x; xa[1] = t.y; xa[2] = t.z; xa[3] = t.w;
        }
        const float4 ga = *reinterpret_cast<const float4*>(sG + col), gb = *reinterpret_cast<const float4*>(sG + col + 4);
        const uint64_t g2[4] = {pk2(ga.x, ga.y), pk2(ga.z, ga.w), pk2(gb.x, gb.y), pk2(gb.z, gb.w)};
        uint32_t keep[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
        if (dmask != nullptr) {
          const uint4 kk = *reinterpret_cast<const uint4*>(sKeep + keepw[i] * 4);
          keep[0] = kk.x; keep[1] = kk.y; keep[2] = kk.z; keep[3] = kk.w;
        }
        uint32_t ow[4], zw[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          uint64_t d2 = unpack2(da[k]);
          if (HAS_DX2) d2 = add2(d2, unpack2(xa[k]));
          const uint64_t xh2 = fma2(unpack2(ya[k]), rs2, nmr2);
          const uint64_t o2 = fma2(nB2, xh2, fma2(d2, mul2(g2[k], rs2), nA2));
          ow[k] = pack2(o2);
          if (dmask != nullptr) {
            zw[k] = pack2(mul2(o2, ds2)) & keep[k];
            az[i][k] = add2(az[i][k], unpack2(zw[k]));
          } else {
            zw[k] = ow[k];
            az[i][k] = add2(az[i][k], o2);
          }
        }
        if (dy != nullptr) *reinterpret_cast<uint4*>(dy + row * lddy + col) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        if (dz != nullptr && (dmask != nullptr || dz != dy))
          *reinterpret_cast<uint4*>(dz + row * lddz + col) = make_uint4(zw[0], zw[1], zw[2], zw[3]);
      }
    }
    // the slot has been read by every lane: refill it with the row ST steps ahead
    __syncwarp();
    if (lane == 0 && row + ST * stride < M) {
      fence_proxy_async();
      fill(slot, row + ST * stride);
    }
    if (++slot == ST) { slot = 0; phase ^= 1u; }
  }
  // block reduction of the three column-sum sets, 256 columns at a time, then one atomic per column
#pragma unroll
  for (int which = 0; which < 3; ++which) {
    float* dst = which == 0 ? dgamma : (which == 1 ? dbeta : dbias);
    if (dst == nullptr) continue;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (i * 256 >= H) break;
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float lo, hi;
        upk2(which == 0 ? ag[i][k] : (which == 1 ? ab[i][k] : az[i][k]), lo, hi);
        red[warp * 256 + lane * 8 + 2 * k] = lo;
        red[warp * 256 + lane * 8 + 2 * k + 1] = hi;
      }
      __syncthreads();
      const int c = threadIdx.x;  // 256 threads <-> 256 columns
      float t = 0.0f;
#pragma unroll
      for (int w = 0; w < ROW_WARPS; ++w) t += red[w * 256 + c];
      if (i * 256 + c < H) {
        if (ORDERED) ws[(static_cast<int64_t>(blockIdx.x) * 3 + which) * H + i * 256 + c] = t;
        else atomicAdd(dst + i * 256 + c, t);
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// column sums (bias gradients):  out[n] += sum_m X[m, n]
// ORDERED: block (x, k) sums the rows of chunk k and stores the partial to ws[k][N]; chunk_reduce_kernel adds them up.
// BOUNDED: only the rows below min(M, *m_dev) are summed (the grid is sized from M): an atomic block with no row there
// exits, an ordered chunk with no row there stores a zero partial, so the reduce adds exactly what an unbounded call on
// the rows below the bound adds, then zeros.
// ----------------------------------------------------------------------------------------------
template <bool ORDERED, bool BOUNDED = false>
__global__ void __launch_bounds__(256)
colsum_kernel(const bf16* __restrict__ X, int64_t ldx, float* __restrict__ out, int M, int N, float* __restrict__ ws,
              const int32_t* __restrict__ m_dev = nullptr) {
  griddep_launch();
  griddep_wait();
  if constexpr (BOUNDED) {
    M = min(M, max(*m_dev, 0));
    if (!ORDERED && static_cast<int64_t>(blockIdx.y) * 8 >= M) return;
  }
  __shared__ float red[8][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.0f;
  if (col < N) {
    // four independent 16-byte loads in flight per lane (the one-load-per-iteration loop reached 0.57 of the HBM peak),
    // packed fp32 adds
    uint64_t a2[4] = {0ull, 0ull, 0ull, 0ull};
    const int64_t stride = ORDERED ? 8 : static_cast<int64_t>(gridDim.y) * 8;
    const int64_t row_end = ORDERED ? min(static_cast<int64_t>(M), (static_cast<int64_t>(blockIdx.y) + 1) * ORDER_ROWS) : M;
    for (int64_t row = static_cast<int64_t>(blockIdx.y) * (ORDERED ? ORDER_ROWS : 8) + warp; row < row_end;
         row += 4 * stride) {
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int64_t r = row + k * stride;
        u[k] = r < row_end ? *reinterpret_cast<const uint4*>(X + r * ldx + col) : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        a2[0] = add2(a2[0], unpack2(u[k].x));
        a2[1] = add2(a2[1], unpack2(u[k].y));
        a2[2] = add2(a2[2], unpack2(u[k].z));
        a2[3] = add2(a2[3], unpack2(u[k].w));
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) upk2(a2[k], acc[2 * k], acc[2 * k + 1]);
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[warp][lane * 8 + e] = acc[e];
  __syncthreads();
  float t = 0.0f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x];
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < N) {
    if (ORDERED) ws[static_cast<int64_t>(blockIdx.y) * N + c] = t;
    else atomicAdd(out + c, t);
  }
}

// Second kernel of the ordered column sums: ws holds `chunks` partial rows of width segs * n, segment j of which belongs to
// out.p[j] (skipped when null).  out[c] += ((part_0[c] + part_1[c]) + ...) + part_{chunks-1}[c], one thread per column.
struct ChunkOuts {
  float* p[3];
};
__global__ void __launch_bounds__(256)
chunk_reduce_kernel(const float* __restrict__ ws, int chunks, int n, int segs, ChunkOuts out) {
  griddep_launch();
  griddep_wait();
  const int c = blockIdx.x * 256 + threadIdx.x;
  const int width = segs * n;
  if (c >= width) return;
  float* dst = out.p[c / n];
  if (dst == nullptr) return;
  float t = 0.0f;
  int k = 0;
  for (; k + 16 <= chunks; k += 16) {     // sixteen loads in flight, added in chunk order
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = ws[static_cast<int64_t>(k + j) * width + c];
#pragma unroll
    for (int j = 0; j < 16; ++j) t += v[j];
  }
  for (; k < chunks; ++k) t += ws[static_cast<int64_t>(k) * width + c];
  dst[c % n] += t;
}

// ----------------------------------------------------------------------------------------------
// dropout keep-bits: word w, bit j keeps element 32*w + j with probability 1-p (16-bit resolution)
// ----------------------------------------------------------------------------------------------
// Bit-sliced comparison: the 16 Philox words of a thread are read as 16 bit-PLANES of 32 sixteen-bit uniforms r_e (bit e of
// plane b = bit b of r_e), and r_e >= thresh16 is evaluated for the 32 elements at once, most significant plane first
// (<= 2 logic operations per plane; the branch on the threshold bit is uniform).  Same distribution and resolution as
// comparing 16-bit fields one by one (the round-1 form: ~3 extract / compare / insert operations per ELEMENT).
// `epoch` (optional, device memory): a step counter added to the Philox counter as epoch << 40, so that a CUDA-graph replay of a
// captured step (host arguments frozen at capture) still draws fresh masks once the graph itself increments the counter.
__global__ void dropout_bits_kernel(uint32_t* __restrict__ out, int64_t nwords, uint64_t seed, uint64_t offset,
                                    uint32_t thresh16, const unsigned long long* __restrict__ epoch) {
  griddep_launch();
  griddep_wait();
  const int64_t w = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (w >= nwords) return;
  if (epoch != nullptr) offset += static_cast<uint64_t>(*epoch) << 40;
  uint32_t gt = 0u, eq = 0xFFFFFFFFu;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint4 r = philox4x32(seed, offset + static_cast<uint64_t>(w) * 4 + i);
    const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int b = 15 - (i * 4 + k);              // plane of bit b, most significant first
      if ((thresh16 >> b) & 1u) {
        eq &= rr[k];                               // threshold bit 1: equal so far only where the uniform's bit is 1 too
      } else {
        gt |= eq & rr[k];                          // threshold bit 0, uniform bit 1: greater from here on
        eq &= ~rr[k];
      }
    }
  }
  out[w] = gt | eq;                                // keep where r >= thresh16
}

// word w of dropout_bits_kernel at the same (seed, offset), for the stochastic-depth kernel below
__device__ __forceinline__ uint32_t keep_word(uint64_t seed, uint64_t offset, int64_t w, uint32_t thresh16) {
  uint32_t gt = 0u, eq = 0xFFFFFFFFu;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint4 r = philox4x32(seed, offset + static_cast<uint64_t>(w) * 4 + i);
    const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int b = 15 - (i * 4 + k);              // plane of bit b, most significant first
      if ((thresh16 >> b) & 1u) {
        eq &= rr[k];                               // threshold bit 1: equal so far only where the uniform's bit is 1 too
      } else {
        gt |= eq & rr[k];                          // threshold bit 0, uniform bit 1: greater from here on
        eq &= ~rr[k];
      }
    }
  }
  return gt | eq;                                  // keep where r >= thresh16
}


// Dropout AND stochastic depth (timm DropPath): word w of row m = w / words is the element keep word of dropout_bits_kernel
// at the same counter, cleared unless sample m / rows_per_sample survives its own draw - the high 16 bits of the first
// Philox word at counter offset + 4 * nwords + sample against thresh_path16.  Every thread of a sample repeats that draw,
// so no thread waits for another.
__global__ void dropout_path_bits_kernel(uint32_t* __restrict__ out, int64_t nwords, int words, int rows_per_sample,
                                         uint64_t seed, uint64_t offset, uint32_t thresh16, uint32_t thresh_path16,
                                         const unsigned long long* __restrict__ epoch) {
  griddep_launch();
  griddep_wait();
  const int64_t w = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (w >= nwords) return;
  if (epoch != nullptr) offset += static_cast<uint64_t>(*epoch) << 40;
  const int64_t sample = w / words / rows_per_sample;
  const uint4 r = philox4x32(seed, offset + static_cast<uint64_t>(nwords) * 4 + static_cast<uint64_t>(sample));
  const bool sample_kept = (r.x >> 16) >= thresh_path16;
  out[w] = sample_kept ? keep_word(seed, offset, w, thresh16) : 0u;
}

// ----------------------------------------------------------------------------------------------
// embedding compose:  y[r] = src0[s0[r]] + src1[s1[r]] + tab0[i0[r]] + tab1[i1[r]] + tab2[i2[r]]   (absent terms: index < 0)
// followed by LayerNorm (+dropout) -> x[r]; y (pre-LN) is saved for the backward.
// ----------------------------------------------------------------------------------------------
struct ComposeDev {
  const bf16* src[2]; int64_t ldsrc[2]; const int32_t* srow[2];
  const bf16* tab[3]; const int32_t* tidx[3];
};

__global__ void __launch_bounds__(ROW_WARPS * 32)
compose_kernel(ComposeDev c, bf16* __restrict__ y, int64_t ldy, int M, int H) {
  griddep_launch();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * ROW_WARPS + (threadIdx.x >> 5);
  if (row >= M) return;
  int sidx[2], tix[3];
#pragma unroll
  for (int k = 0; k < 2; ++k) sidx[k] = (c.src[k] != nullptr && c.srow[k] != nullptr) ? c.srow[k][row] : -1;
#pragma unroll
  for (int k = 0; k < 3; ++k) tix[k] = (c.tab[k] != nullptr && c.tidx[k] != nullptr) ? c.tidx[k][row] : -1;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int col = i * 256 + lane * 8;
    if (col < H) {
      float a[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] = 0.0f;
#pragma unroll
      for (int k = 0; k < 2; ++k)
        if (sidx[k] >= 0) {
          float t[8];
          ld8(c.src[k] + static_cast<int64_t>(sidx[k]) * c.ldsrc[k] + col, t);
#pragma unroll
          for (int e = 0; e < 8; ++e) a[e] += t[e];
        }
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (tix[k] >= 0) {
          float t[8];
          ld8(c.tab[k] + static_cast<int64_t>(tix[k]) * H + col, t);
#pragma unroll
          for (int e = 0; e < 8; ++e) a[e] += t[e];
        }
      st8(y + row * ldy + col, a);
    }
  }
}

struct ScatterDev {
  bf16* dsrc[2]; int64_t ldsrc[2]; const int32_t* srow[2];
  float* dtab[3]; const int32_t* tidx[3];
};

// backward of compose: dsrc_k[s_k[r]] = dy[r]  (rows are unique) ; dtab_k[i_k[r]] += dy[r]  (fp32 atomics)
__global__ void __launch_bounds__(ROW_WARPS * 32)
scatter_kernel(ScatterDev c, const bf16* __restrict__ dy, int64_t lddy, int M, int H) {
  griddep_launch();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * ROW_WARPS + (threadIdx.x >> 5);
  if (row >= M) return;
  int sidx[2], tix[3];
#pragma unroll
  for (int k = 0; k < 2; ++k) sidx[k] = (c.dsrc[k] != nullptr && c.srow[k] != nullptr) ? c.srow[k][row] : -1;
#pragma unroll
  for (int k = 0; k < 3; ++k) tix[k] = (c.dtab[k] != nullptr && c.tidx[k] != nullptr) ? c.tidx[k][row] : -1;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int col = i * 256 + lane * 8;
    if (col < H) {
      float a[8];
      ld8(dy + row * lddy + col, a);
#pragma unroll
      for (int k = 0; k < 2; ++k)
        if (sidx[k] >= 0) st8(c.dsrc[k] + static_cast<int64_t>(sidx[k]) * c.ldsrc[k] + col, a);
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (tix[k] >= 0) {
          float* d = c.dtab[k] + static_cast<int64_t>(tix[k]) * H + col;
#pragma unroll
          for (int e = 0; e < 8; ++e) atomicAdd(d + e, a[e]);
        }
    }
  }
}

// Table-gradient scatter over SORTED indices: warp w owns sorted positions [32w, 32w+32); rows with equal index are
// summed in registers and flushed with one atomic per column per run, so an index shared by thousands of rows (type /
// position embeddings) costs M/32 atomics per address instead of M.
// ORDERED: a run piece that is the whole run (nothing before or after it in other chunks) is added to its table row with
// a plain read-modify-write - no other warp touches that row.  A piece of a run that crosses a chunk boundary is stored to
// the workspace instead: slot ws[w][0] when the run began before this chunk, ws[w][1] when it begins here and goes on
// past it; scatter_runs_kernel adds the pieces of each crossing run in chunk order.
template <int NV, bool ORDERED>
__global__ void __launch_bounds__(ROW_WARPS * 32)
scatter_sorted_kernel(const bf16* __restrict__ dy, int64_t lddy, const int32_t* __restrict__ order,
                      const int32_t* __restrict__ sorted_idx, float* __restrict__ dtab, int M, int H,
                      float* __restrict__ ws) {
  griddep_launch();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const int64_t w = static_cast<int64_t>(blockIdx.x) * ROW_WARPS + (threadIdx.x >> 5);
  const int64_t p0 = w * 32;
  if (p0 >= M) return;
  float acc[NV][8];
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[i][e] = 0.0f;
  int cur = -1;
  int run_start = 0;
  const int n = (M - p0) < 32 ? static_cast<int>(M - p0) : 32;
  for (int k = 0; k <= n; ++k) {
    const int id = (k < n) ? sorted_idx[p0 + k] : -2;
    if (id != cur) {
      if (cur >= 0) {
        float* piece = nullptr;       // ORDERED: the workspace slot of a crossing run's piece
        if (ORDERED) {
          if (run_start == 0 && p0 > 0 && sorted_idx[p0 - 1] == cur) piece = ws + (w * 2) * H;
          else if (k == n && p0 + n < M && sorted_idx[p0 + n] == cur) piece = ws + (w * 2 + 1) * H;
        }
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const int col = i * 256 + lane * 8;
          if (col < H) {
            float* d = dtab + static_cast<int64_t>(cur) * H + col;
            if (!ORDERED) {
#pragma unroll
              for (int e = 0; e < 8; ++e) atomicAdd(d + e, acc[i][e]);
            } else if (piece != nullptr) {
              *reinterpret_cast<float4*>(piece + col) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
              *reinterpret_cast<float4*>(piece + col + 4) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
            } else {
#pragma unroll
              for (int e = 0; e < 8; ++e) d[e] += acc[i][e];
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[i][e] = 0.0f;
          }
        }
      }
      cur = id;
      run_start = k;
    }
    if (k < n && id >= 0) {
      const int64_t r = order[p0 + k];
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int col = i * 256 + lane * 8;
        if (col < H) {
          float t[8];
          ld8(dy + r * lddy + col, t);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[i][e] += t[e];
        }
      }
    }
  }
}

// Second kernel of the ordered scatter: block w adds up the run that begins in chunk w and crosses into chunk w + 1, if
// there is one: its piece ws[w][1], then ws[c][0] of every later chunk c the run reaches, in chunk order, and adds the sum
// to the run's table row.  The run's end is found by a binary search of the sorted indices, so the pieces' loads do not
// wait on each other.
__global__ void __launch_bounds__(256)
scatter_runs_kernel(const int32_t* __restrict__ sorted_idx, const float* __restrict__ ws, float* __restrict__ dtab, int M,
                    int H) {
  griddep_launch();
  griddep_wait();
  const int64_t w = blockIdx.x;
  const int64_t p0 = w * SCATTER_CHUNK;
  const int64_t last = min(static_cast<int64_t>(M), p0 + SCATTER_CHUNK) - 1;
  if (last + 1 >= M) return;
  const int id = sorted_idx[last];
  if (id < 0 || sorted_idx[last + 1] != id) return;                          // nothing crosses out of this chunk
  if (sorted_idx[p0] == id && p0 > 0 && sorted_idx[p0 - 1] == id) return;    // the run began in an earlier chunk
  int64_t lo = last + 1, hi = M;                                              // first position past the run
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (sorted_idx[mid] == id) lo = mid + 1;
    else hi = mid;
  }
  const int64_t c_last = (lo - 1) / SCATTER_CHUNK;                            // chunk of the run's last position
  for (int col = threadIdx.x * 4; col < H; col += 256 * 4) {
    float4 t = *reinterpret_cast<const float4*>(ws + (w * 2 + 1) * H + col);
    int64_t c = w + 1;
    for (; c + 8 <= c_last + 1; c += 8) {       // eight loads in flight, added in chunk order
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = *reinterpret_cast<const float4*>(ws + ((c + j) * 2) * H + col);
#pragma unroll
      for (int j = 0; j < 8; ++j) { t.x += v[j].x; t.y += v[j].y; t.z += v[j].z; t.w += v[j].w; }
    }
    for (; c <= c_last; ++c) {
      const float4 v = *reinterpret_cast<const float4*>(ws + (c * 2) * H + col);
      t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
    }
    float* d = dtab + static_cast<int64_t>(id) * H + col;
    d[0] += t.x; d[1] += t.y; d[2] += t.z; d[3] += t.w;
  }
}

// backward of the ReLU epilogue: dz = (y > 0) ? dy : 0, 16-byte vectors
__global__ void relu_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ y, bf16* __restrict__ dz, int64_t n) {
  griddep_launch();
  griddep_wait();
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    float a[8], b[8];
    ld8(dy + i, a);
    ld8(y + i, b);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] = b[e] > 0.0f ? a[e] : 0.0f;
    st8(dz + i, a);
  } else {
    for (int64_t j = i; j < n; ++j) dz[j] = __bfloat162float(y[j]) > 0.0f ? dy[j] : __float2bfloat16_rn(0.0f);
  }
}

// out = a + b (bf16, 16-byte vectors): the residual-gradient join of the pre-LN (ViT) layer, mmf/modules/vit.py:96-108
__global__ void add_bf16_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ out, int64_t n) {
  griddep_launch();
  griddep_wait();
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    float x[8], y[8];
    ld8(a + i, x);
    ld8(b + i, y);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] += y[e];
    st8(out + i, x);
  } else {
    for (int64_t j = i; j < n; ++j) out[j] = __float2bfloat16_rn(__bfloat162float(a[j]) + __bfloat162float(b[j]));
  }
}

// out[m, h] = keep-bit(m, h) ? x[m, h] * scale : 0 : the backward of a dropout that is NOT followed by a LayerNorm
// (whose backward kernel otherwise applies the mask): one warp per row, 8 columns per lane and step
__global__ void dropout_apply_kernel(const bf16* __restrict__ x, int64_t ldx, const uint32_t* __restrict__ bits, int64_t ldm,
                                     float scale, bf16* __restrict__ out, int64_t ldo, int M, int H) {
  griddep_launch();
  griddep_wait();
  const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  for (int col = lane * 8; col < H; col += 256) {
    float v[8];
    ld8(x + row * ldx + col, v);
    const uint32_t w = __ldg(bits + row * ldm + (col >> 5));
    const uint32_t b8 = (w >> (col & 31)) & 0xFFu;
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = ((b8 >> e) & 1u) ? v[e] * scale : 0.0f;
    st8(out + row * ldo + col, v);
  }
}

// fp32 -> bf16 cast of the flat parameter buffer (done every forward, like autocast does)
__global__ void cast_f32_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, int64_t n) {
  griddep_launch();
  griddep_wait();
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const float4 a = *reinterpret_cast<const float4*>(in + i);
    const float4 b = *reinterpret_cast<const float4*>(in + i + 4);
    uint4 u;
    u.x = pack_bf16x2(a.x, a.y); u.y = pack_bf16x2(a.z, a.w);
    u.z = pack_bf16x2(b.x, b.y); u.w = pack_bf16x2(b.z, b.w);
    *reinterpret_cast<uint4*>(out + i) = u;
  } else {
    for (int64_t j = i; j < n; ++j) out[j] = __float2bfloat16_rn(in[j]);
  }
}

// ----------------------------------------------------------------------------------------------
// host
// ----------------------------------------------------------------------------------------------
static int check_rows(int M, int H, const char* who) {
  if (M <= 0 || H <= 0) return set_error(MMFB_ERR_ARG, "%s: empty problem", who);
  if (H % 8 || H > MAXV * 256) return set_error(MMFB_ERR_ARG, "%s: hidden size %d must be a multiple of 8 and <= %d", who, H, MAXV * 256);
  return MMFB_OK;
}
static int launch_ok(const char* who) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

// The row kernels (LayerNorm, column sums, embedding compose / scatter, dropout apply) move rows as 16-byte vectors (the
// streaming LayerNorm backward with cp.async.bulk), so every row a kernel reads or writes must start on a 16-byte
// boundary: the base pointer aligned and, when there is more than one row, the leading dimension a multiple of 8
// elements.  Null tensors are not used by the call and are skipped.  A misaligned view is refused with MMFB_ERR_ARG
// before anything is launched, instead of faulting in the kernel.
struct RowTensor {
  const void* p;
  int64_t ld;        // 0 for the [H] vectors
  const char* name;
};
static int check_aligned(const char* who, int M, std::initializer_list<RowTensor> ts) {
  for (const RowTensor& t : ts) {
    if (t.p == nullptr) continue;
    if (reinterpret_cast<uintptr_t>(t.p) & 15) return set_error(MMFB_ERR_ARG, "%s: %s must be 16-byte aligned", who, t.name);
    if (M > 1 && t.ld % 8)
      return set_error(MMFB_ERR_ARG, "%s: ld%s = %lld must be a multiple of 8", who, t.name, static_cast<long long>(t.ld));
  }
  return MMFB_OK;
}

int ln_fwd(const mmfb_ln_args& a, cudaStream_t s, const int32_t* m_dev) {
  int rc = check_rows(a.M, a.H, "layernorm_fwd");
  if (rc) return rc;
  if (!a.y || !a.gamma || !a.beta || !a.x) return set_error(MMFB_ERR_ARG, "layernorm_fwd: null pointer");
  rc = check_aligned("layernorm_fwd", a.M, {{a.y, a.ldy, "y"}, {a.x, a.ldx, "x"}, {a.gamma, 0, "gamma"}, {a.beta, 0, "beta"}});
  if (rc) return rc;
  if (reinterpret_cast<uintptr_t>(m_dev) & 3) return set_error(MMFB_ERR_ARG, "layernorm_fwd: m_dev must be 4-byte aligned");
#define LN_FWD(NV, BND)                                                                                    \
  MMFB_LAUNCH((ln_fwd_kernel<NV, BND>), (a.M + ROW_WARPS - 1) / ROW_WARPS, ROW_WARPS * 32, 0, s,                    \
      (const bf16*)a.y, a.ldy, (const bf16*)a.gamma, (const bf16*)a.beta, (bf16*)a.x, a.ldx, a.mean, a.rstd, \
      a.drop_mask, a.ldmask, a.drop_scale, a.M, a.H, a.eps, m_dev)
  const int nv = (a.H + 255) / 256;
  if (m_dev != nullptr) {
    if (nv <= 1) LN_FWD(1, true); else if (nv == 2) LN_FWD(2, true); else if (nv == 3) LN_FWD(3, true);
    else if (nv == 4) LN_FWD(4, true); else LN_FWD(8, true);
  } else {
    if (nv <= 1) LN_FWD(1, false); else if (nv == 2) LN_FWD(2, false); else if (nv == 3) LN_FWD(3, false);
    else if (nv == 4) LN_FWD(4, false); else LN_FWD(8, false);
  }
#undef LN_FWD
  return launch_ok("layernorm_fwd");
}

// Both backward kernels stride over the rows: a grid of at most two blocks per SM.
static int ln_bwd_grid(int M) {
  const int grid = (M + ROW_WARPS - 1) / ROW_WARPS, cap = num_sms() * 2;
  return grid < cap ? grid : cap;
}

int64_t ln_bwd_workspace_bytes(int M, int H) {
  return (M > 0 && H > 0) ? static_cast<int64_t>(order_chunks(M)) * 3 * H * 4 : 0;
}
int64_t colsum_workspace_bytes(int M, int N) {
  return (M > 0 && N > 0) ? static_cast<int64_t>(order_chunks(M)) * N * 4 : 0;
}
int64_t scatter_sorted_workspace_bytes(int M, int H) {
  return (M > 0 && H > 0) ? static_cast<int64_t>((M + SCATTER_CHUNK - 1) / SCATTER_CHUNK) * 2 * H * 4 : 0;
}
static int check_workspace(const char* who, const float* ws, int64_t ws_bytes, int64_t need) {
  if (ws == nullptr || ws_bytes < need || (reinterpret_cast<uintptr_t>(ws) & 15))
    return set_error(MMFB_ERR_ARG, "%s: the ordered reduction needs a 16-byte aligned workspace of %lld bytes (got %p, %lld)",
                     who, static_cast<long long>(need), static_cast<const void*>(ws), static_cast<long long>(ws_bytes));
  return MMFB_OK;
}
// adds the `chunks` partial rows of ws (segments of n columns, segment j for out[j]) to their destinations
static int chunk_reduce(const float* ws, int chunks, int n, float* out0, float* out1, float* out2, int segs, cudaStream_t s,
                        const char* who) {
  ChunkOuts o;
  o.p[0] = out0; o.p[1] = out1; o.p[2] = out2;
  MMFB_LAUNCH(chunk_reduce_kernel, (segs * n + 255) / 256, 256, 0, s, ws, chunks, n, segs, o);
  return launch_ok(who);
}

template <int NV, bool HAS_DX2, int ST, bool ORDERED, bool BOUNDED>
static int ln_bwd_stream(const mmfb_ln_args& a, cudaStream_t s, const int32_t* m_dev) {
  constexpr size_t smem = static_cast<size_t>(ROW_WARPS) * ST * (HAS_DX2 ? 3 : 2) * NV * 512 + ROW_WARPS * 256 * 4 +
                          NV * 256 * 4 + 4096 + ROW_WARPS * ST * 8;
  auto kern = ln_bwd_stream_kernel<NV, HAS_DX2, ST, ORDERED, BOUNDED>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "cudaFuncSetAttribute(layernorm_bwd): %s", cudaGetErrorString(e));
    attr_set = true;
  }
  MMFB_LAUNCH(kern, ORDERED ? order_chunks(a.M) : ln_bwd_grid(a.M), ROW_WARPS * 32, smem, s, (const bf16*)a.dx, a.lddx,
              (const bf16*)a.dx2, a.lddx2, (const bf16*)a.y, a.ldy, a.mean, a.rstd, (const bf16*)a.gamma, (bf16*)a.dy, a.lddy,
              (bf16*)a.dz, a.lddz, a.drop_mask, a.ldmask, a.drop_scale, a.dgamma, a.dbeta, a.dbias, a.M, a.H, a.workspace,
              m_dev);
  return launch_ok("layernorm_bwd");
}

// ln_bwd_stream<NV, HAS_DX2, ST, ORDERED, BOUNDED> indexed by [dx2 given][NV - 1]; NV = 256-column slabs per row, ST = ring
// depth (the same depths with and without the bound)
template <bool ORDERED, bool BOUNDED>
static int ln_bwd_stream_dispatch(const mmfb_ln_args& a, cudaStream_t s, const int32_t* m_dev) {
  static int (*const stream[2][4])(const mmfb_ln_args&, cudaStream_t, const int32_t*) = {
      {ln_bwd_stream<1, false, 4, ORDERED, BOUNDED>, ln_bwd_stream<2, false, 4, ORDERED, BOUNDED>,
       ln_bwd_stream<3, false, 3, ORDERED, BOUNDED>, ln_bwd_stream<4, false, 2, ORDERED, BOUNDED>},
      {ln_bwd_stream<1, true, 3, ORDERED, BOUNDED>, ln_bwd_stream<2, true, 3, ORDERED, BOUNDED>,
       ln_bwd_stream<3, true, 2, ORDERED, BOUNDED>, ln_bwd_stream<4, true, 2, ORDERED, BOUNDED>}};
  return stream[a.dx2 != nullptr][(a.H + 255) / 256 - 1](a, s, m_dev);
}

// The ordered LayerNorm backward: the kernels above with one block per chunk of rows, then the chunk partials of dgamma,
// dbeta and dbias added in chunk order.  Same ring depths as the atomic path.
template <bool BOUNDED>
static int ln_bwd_ordered(const mmfb_ln_args& a, bool wide, cudaStream_t s, const int32_t* m_dev) {
  const int chunks = order_chunks(a.M);
  if (wide) {
    MMFB_LAUNCH((ln_bwd_kernel<true, BOUNDED>), chunks, ROW_WARPS * 32, 0, s, (const bf16*)a.dx, a.lddx,
                (const bf16*)a.dx2, a.lddx2, (const bf16*)a.y, a.ldy, a.mean, a.rstd, (const bf16*)a.gamma, (bf16*)a.dy,
                a.lddy, (bf16*)a.dz, a.lddz, a.drop_mask, a.ldmask, a.drop_scale, a.dgamma, a.dbeta, a.dbias, a.M, a.H,
                a.workspace, m_dev);
    int rc = launch_ok("layernorm_bwd");
    if (rc) return rc;
  } else {
    int rc = ln_bwd_stream_dispatch<true, BOUNDED>(a, s, m_dev);
    if (rc) return rc;
  }
  if (!a.dgamma && !a.dbeta && !a.dbias) return MMFB_OK;
  return chunk_reduce(a.workspace, chunks, a.H, a.dgamma, a.dbeta, a.dbias, 3, s, "layernorm_bwd reduce");
}

int ln_bwd(const mmfb_ln_args& a, cudaStream_t s, const int32_t* m_dev) {
  int rc = check_rows(a.M, a.H, "layernorm_bwd");
  if (rc) return rc;
  if (!a.dx || !a.y || !a.mean || !a.rstd || !a.gamma) return set_error(MMFB_ERR_ARG, "layernorm_bwd: null pointer");
  if (a.drop_mask && !a.dz) return set_error(MMFB_ERR_ARG, "layernorm_bwd: dropout mask given without dz");
  const bool wide = a.H > 1024;
  // dz is written only when it is a separate output; only the wide kernel reads gamma as 16-byte vectors
  const void* dz = (a.drop_mask || a.dz != a.dy) ? a.dz : nullptr;
  rc = check_aligned("layernorm_bwd", a.M, {{a.dx, a.lddx, "dx"}, {a.dx2, a.lddx2, "dx2"}, {a.y, a.ldy, "y"},
                                            {a.dy, a.lddy, "dy"}, {dz, a.lddz, "dz"}, {wide ? a.gamma : nullptr, 0, "gamma"}});
  if (rc) return rc;
  if (reinterpret_cast<uintptr_t>(m_dev) & 3) return set_error(MMFB_ERR_ARG, "layernorm_bwd: m_dev must be 4-byte aligned");
  const bool bounded = m_dev != nullptr;
  if (a.workspace != nullptr || a.workspace_bytes != 0) {
    rc = check_workspace("layernorm_bwd", a.workspace, a.workspace_bytes, ln_bwd_workspace_bytes(a.M, a.H));
    if (rc) return rc;
    return bounded ? ln_bwd_ordered<true>(a, wide, s, m_dev) : ln_bwd_ordered<false>(a, wide, s, nullptr);
  }
  if (wide) {
    auto kern = bounded ? ln_bwd_kernel<false, true> : ln_bwd_kernel<false, false>;
    MMFB_LAUNCH(kern, ln_bwd_grid(a.M), ROW_WARPS * 32, 0, s, (const bf16*)a.dx, a.lddx, (const bf16*)a.dx2,
                a.lddx2, (const bf16*)a.y, a.ldy, a.mean, a.rstd, (const bf16*)a.gamma, (bf16*)a.dy, a.lddy, (bf16*)a.dz,
                a.lddz, a.drop_mask, a.ldmask, a.drop_scale, a.dgamma, a.dbeta, a.dbias, a.M, a.H, nullptr, m_dev);
    return launch_ok("layernorm_bwd");
  }
  return bounded ? ln_bwd_stream_dispatch<false, true>(a, s, m_dev) : ln_bwd_stream_dispatch<false, false>(a, s, nullptr);
}

int colsum(const void* X, int64_t ldx, float* out, int M, int N, cudaStream_t s) {
  if (M <= 0 || N <= 0 || N % 8) return set_error(MMFB_ERR_ARG, "colsum: bad shape %dx%d", M, N);
  const int rc = check_aligned("colsum", M, {{X, ldx, "x"}});
  if (rc) return rc;
  dim3 grid((N + 255) / 256, 1);
  int rows_blocks = (M + 63) / 64;
  const int cap = (num_sms() * 4 + grid.x - 1) / grid.x;
  grid.y = rows_blocks < cap ? rows_blocks : cap;
  if (grid.y < 1) grid.y = 1;
  MMFB_LAUNCH(colsum_kernel<false>, grid, 256, 0, s, (const bf16*)X, ldx, out, M, N, nullptr, nullptr);
  return launch_ok("colsum");
}

int colsum_ordered(const void* X, int64_t ldx, float* out, int M, int N, float* ws, int64_t ws_bytes, cudaStream_t s) {
  if (M <= 0 || N <= 0 || N % 8) return set_error(MMFB_ERR_ARG, "colsum_ordered: bad shape %dx%d", M, N);
  int rc = check_aligned("colsum_ordered", M, {{X, ldx, "x"}});
  if (rc) return rc;
  if ((rc = check_workspace("colsum_ordered", ws, ws_bytes, colsum_workspace_bytes(M, N)))) return rc;
  const int chunks = order_chunks(M);
  MMFB_LAUNCH(colsum_kernel<true>, dim3((N + 255) / 256, chunks), 256, 0, s, (const bf16*)X, ldx, out, M, N, ws, nullptr);
  if ((rc = launch_ok("colsum_ordered"))) return rc;
  return chunk_reduce(ws, chunks, N, out, nullptr, nullptr, 1, s, "colsum_ordered reduce");
}

// colsum / colsum_ordered (ws non-null) of the rows below min(M, *m_dev); grid and workspace sized from M
int colsum_bounded(const void* X, int64_t ldx, float* out, int M, int N, const int32_t* m_dev, float* ws, int64_t ws_bytes,
                   cudaStream_t s) {
  if (M <= 0 || N <= 0 || N % 8) return set_error(MMFB_ERR_ARG, "colsum_bounded: bad shape %dx%d", M, N);
  int rc = check_aligned("colsum_bounded", M, {{X, ldx, "x"}});
  if (rc) return rc;
  if (reinterpret_cast<uintptr_t>(m_dev) & 3) return set_error(MMFB_ERR_ARG, "colsum_bounded: m_dev must be 4-byte aligned");
  if (ws != nullptr || ws_bytes != 0) {
    if ((rc = check_workspace("colsum_bounded", ws, ws_bytes, colsum_workspace_bytes(M, N)))) return rc;
    const int chunks = order_chunks(M);
    MMFB_LAUNCH((colsum_kernel<true, true>), dim3((N + 255) / 256, chunks), 256, 0, s, (const bf16*)X, ldx, out, M, N, ws,
                m_dev);
    if ((rc = launch_ok("colsum_bounded"))) return rc;
    return chunk_reduce(ws, chunks, N, out, nullptr, nullptr, 1, s, "colsum_bounded reduce");
  }
  dim3 grid((N + 255) / 256, 1);
  int rows_blocks = (M + 63) / 64;
  const int cap = (num_sms() * 4 + grid.x - 1) / grid.x;
  grid.y = rows_blocks < cap ? rows_blocks : cap;
  if (grid.y < 1) grid.y = 1;
  MMFB_LAUNCH((colsum_kernel<false, true>), grid, 256, 0, s, (const bf16*)X, ldx, out, M, N, nullptr, m_dev);
  return launch_ok("colsum_bounded");
}

// Row selection of a static-rows masked-LM head (one CTA; the labels of one batch are a few ten thousand int64).  Thread t
// owns the consecutive labels [t * per, (t + 1) * per): it counts its labelled ones, an exclusive scan over the threads in
// thread order gives its first output slot, and a second pass writes them.  No atomics: the same bits on every run.
// state (int32 [2 + 2M]): [0] = count, [1] = the fp32 bits of 1 / max(count, 1) (the double reciprocal rounded once, as
// the host computes it), [2, 2 + M) = pos (output row -> source row, -1 past count), [2 + M, 2 + 2M) = inv (source row ->
// output row, -1 for an unlabelled row).  labels_out[i] = labels[pos[i]], ignore_index past count.
constexpr int SELECT_THREADS = 1024;
__global__ void __launch_bounds__(SELECT_THREADS)
select_rows_kernel(const int64_t* __restrict__ labels, int64_t ignore_index, int M, int32_t* __restrict__ state,
                   int64_t* __restrict__ labels_out) {
  griddep_launch();
  griddep_wait();
  __shared__ int warp_tot[SELECT_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int per = (M + SELECT_THREADS - 1) / SELECT_THREADS;
  const int b = min(M, static_cast<int>(threadIdx.x) * per), e = min(M, b + per);
  int n = 0;
  for (int i = b; i < e; ++i) n += labels[i] != ignore_index;
  int incl = n;                                   // inclusive scan within the warp
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  int before = 0, total = 0;
  for (int w = 0; w < SELECT_THREADS / 32; ++w) {
    const int t = warp_tot[w];
    if (w < warp) before += t;
    total += t;
  }
  int slot = before + incl - n;
  int32_t* pos = state + 2;
  int32_t* inv = state + 2 + M;
  for (int i = b; i < e; ++i) {
    const int64_t l = labels[i];
    if (l != ignore_index) {
      pos[slot] = i;
      inv[i] = slot;
      labels_out[slot] = l;
      ++slot;
    } else {
      inv[i] = -1;
    }
  }
  for (int i = total + threadIdx.x; i < M; i += SELECT_THREADS) {
    pos[i] = -1;
    labels_out[i] = ignore_index;
  }
  if (threadIdx.x == 0) {
    state[0] = total;
    state[1] = __float_as_int(__double2float_rn(1.0 / static_cast<double>(max(total, 1))));
  }
}

// out[r] = idx[r] >= 0 ? x[idx[r]] : 0, one warp per output row, 16-byte vectors.  With pos this is the forward gather of
// the selected rows; with inv it is its backward (each source row takes its gathered row's gradient, or zero): no atomics.
__global__ void __launch_bounds__(ROW_WARPS * 32)
gather_rows_kernel(const bf16* __restrict__ x, int64_t ldx, const int32_t* __restrict__ idx, bf16* __restrict__ out,
                   int64_t ldo, int M, int H) {
  griddep_launch();
  griddep_wait();
  const int row = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const int src = idx[row];
  uint4* dst = reinterpret_cast<uint4*>(out + static_cast<int64_t>(row) * ldo);
  const uint4* from = reinterpret_cast<const uint4*>(x + static_cast<int64_t>(src < 0 ? 0 : src) * ldx);
  for (int v = lane; v < H / 8; v += 32) dst[v] = src >= 0 ? from[v] : make_uint4(0u, 0u, 0u, 0u);
}

int select_rows(const int64_t* labels, int64_t ignore_index, int M, int32_t* state, int64_t* labels_out, cudaStream_t s) {
  if (M <= 0) return set_error(MMFB_ERR_ARG, "select_rows: empty problem");
  if ((reinterpret_cast<uintptr_t>(labels) | reinterpret_cast<uintptr_t>(labels_out)) & 7 ||
      reinterpret_cast<uintptr_t>(state) & 3)
    return set_error(MMFB_ERR_ARG, "select_rows: misaligned buffer");
  MMFB_LAUNCH(select_rows_kernel, 1, SELECT_THREADS, 0, s, labels, ignore_index, M, state, labels_out);
  return launch_ok("select_rows");
}

int gather_rows(const void* x, int64_t ldx, const int32_t* idx, void* out, int64_t ldo, int M, int H, cudaStream_t s) {
  if (M <= 0 || H <= 0 || H % 8) return set_error(MMFB_ERR_ARG, "gather_rows: bad shape %dx%d", M, H);
  int rc = check_aligned("gather_rows", 2, {{x, ldx, "x"}, {out, ldo, "out"}});
  if (rc) return rc;
  if (reinterpret_cast<uintptr_t>(idx) & 3) return set_error(MMFB_ERR_ARG, "gather_rows: idx must be 4-byte aligned");
  MMFB_LAUNCH(gather_rows_kernel, (M + ROW_WARPS - 1) / ROW_WARPS, ROW_WARPS * 32, 0, s, (const bf16*)x, ldx, idx, (bf16*)out,
              ldo, M, H);
  return launch_ok("gather_rows");
}

int dropout_bits(uint32_t* out, int64_t nwords, uint64_t seed, uint64_t offset, float p, const uint64_t* epoch, cudaStream_t s) {
  if (nwords <= 0) return set_error(MMFB_ERR_ARG, "dropout_bits: empty");
  if (!(p >= 0.0f && p < 1.0f)) return set_error(MMFB_ERR_ARG, "dropout_bits: p must be in [0,1), got %f", p);
  uint32_t thresh = static_cast<uint32_t>(p * 65536.0f + 0.5f);
  if (thresh > 65535u) thresh = 65535u;          // 16 planes: p within 2^-16 of 1 keeps one element in 65536
  MMFB_LAUNCH(dropout_bits_kernel, static_cast<unsigned>((nwords + 255) / 256), 256, 0, s, out, nwords, seed, offset, thresh,
              reinterpret_cast<const unsigned long long*>(epoch));
  return launch_ok("dropout_bits");
}

int dropout_path_bits(uint32_t* out, int M, int H, int rows_per_sample, uint64_t seed, uint64_t offset, float p, float p_path,
                      const uint64_t* epoch, cudaStream_t s) {
  if (M <= 0 || H <= 0 || rows_per_sample <= 0 || M % rows_per_sample)
    return set_error(MMFB_ERR_ARG, "dropout_path_bits: bad shape M=%d H=%d rows_per_sample=%d (M must be a multiple of it)",
                     M, H, rows_per_sample);
  if (!(p >= 0.0f && p < 1.0f) || !(p_path >= 0.0f && p_path < 1.0f))
    return set_error(MMFB_ERR_ARG, "dropout_path_bits: p and p_path must be in [0,1), got %f, %f", p, p_path);
  const auto thresh = [](float q) {
    const uint32_t t = static_cast<uint32_t>(q * 65536.0f + 0.5f);
    return t > 65535u ? 65535u : t;
  };
  const int words = (H + 31) / 32;
  const int64_t nwords = static_cast<int64_t>(M) * words;
  MMFB_LAUNCH(dropout_path_bits_kernel, static_cast<unsigned>((nwords + 255) / 256), 256, 0, s, out, nwords, words,
              rows_per_sample, seed, offset, thresh(p), thresh(p_path), reinterpret_cast<const unsigned long long*>(epoch));
  return launch_ok("dropout_path_bits");
}

int compose(const mmfb_compose_args& a, cudaStream_t s) {
  int rc = check_rows(a.M, a.H, "embed_compose");
  if (rc) return rc;
  if (!a.y) return set_error(MMFB_ERR_ARG, "embed_compose: null output");
  // a term is read only when both its tensor and its index vector are given; the gathered source rows can be any rows
  // of their buffer, so their leading dimension is checked whatever M is (the row count 2 below)
  auto used_src = [&](int k) { return a.src_row[k] != nullptr ? a.src[k] : nullptr; };
  auto used_tab = [&](int k) { return a.tab_idx[k] != nullptr ? a.tab[k] : nullptr; };
  rc = check_aligned("embed_compose", 2, {{used_src(0), a.ldsrc[0], "src0"}, {used_src(1), a.ldsrc[1], "src1"},
                                          {used_tab(0), a.H, "tab0"}, {used_tab(1), a.H, "tab1"}, {used_tab(2), a.H, "tab2"}});
  if (rc) return rc;
  rc = check_aligned("embed_compose", a.M, {{a.y, a.ldy, "y"}});
  if (rc) return rc;
  ComposeDev c;
  for (int k = 0; k < 2; ++k) { c.src[k] = (const bf16*)a.src[k]; c.ldsrc[k] = a.ldsrc[k]; c.srow[k] = a.src_row[k]; }
  for (int k = 0; k < 3; ++k) { c.tab[k] = (const bf16*)a.tab[k]; c.tidx[k] = a.tab_idx[k]; }
  MMFB_LAUNCH(compose_kernel, (a.M + ROW_WARPS - 1) / ROW_WARPS, ROW_WARPS * 32, 0, s, c, (bf16*)a.y, a.ldy, a.M, a.H);
  return launch_ok("embed_compose");
}

int scatter(const mmfb_scatter_args& a, cudaStream_t s) {
  int rc = check_rows(a.M, a.H, "embed_scatter");
  if (rc) return rc;
  if (!a.dy) return set_error(MMFB_ERR_ARG, "embed_scatter: null input");
  // the fp32 table gradients take scalar atomics and need no 16-byte rows; the dense-source gradients are stored to
  // gathered rows (any row of their buffer: leading dimension checked whatever M is)
  rc = check_aligned("embed_scatter", a.M, {{a.dy, a.lddy, "dy"}});
  if (rc) return rc;
  rc = check_aligned("embed_scatter", 2, {{a.src_row[0] != nullptr ? a.dsrc[0] : nullptr, a.ldsrc[0], "dsrc0"},
                                          {a.src_row[1] != nullptr ? a.dsrc[1] : nullptr, a.ldsrc[1], "dsrc1"}});
  if (rc) return rc;
  ScatterDev c;
  for (int k = 0; k < 2; ++k) { c.dsrc[k] = (bf16*)a.dsrc[k]; c.ldsrc[k] = a.ldsrc[k]; c.srow[k] = a.src_row[k]; }
  for (int k = 0; k < 3; ++k) { c.dtab[k] = a.dtab[k]; c.tidx[k] = a.tab_idx[k]; }
  MMFB_LAUNCH(scatter_kernel, (a.M + ROW_WARPS - 1) / ROW_WARPS, ROW_WARPS * 32, 0, s, c, (const bf16*)a.dy, a.lddy, a.M, a.H);
  return launch_ok("embed_scatter");
}

int scatter_sorted(const void* dy, int64_t lddy, const int32_t* order, const int32_t* sorted_idx, float* dtab, int M,
                   int H, cudaStream_t s) {
  int rc = check_rows(M, H, "embed_scatter_sorted");
  if (rc) return rc;
  if (H > 1024) return set_error(MMFB_ERR_ARG, "embed_scatter_sorted: hidden size %d > 1024", H);
  rc = check_aligned("embed_scatter_sorted", M, {{dy, lddy, "dy"}});
  if (rc) return rc;
  const int warps = (M + 31) / 32;
  const int grid = (warps + ROW_WARPS - 1) / ROW_WARPS;
  const int nv = (H + 255) / 256;
#define SS(NV) MMFB_LAUNCH((scatter_sorted_kernel<NV, false>), grid, ROW_WARPS * 32, 0, s, (const bf16*)dy, lddy, order, sorted_idx, dtab, M, H, nullptr)
  if (nv <= 1) SS(1); else if (nv == 2) SS(2); else if (nv == 3) SS(3); else SS(4);
#undef SS
  return launch_ok("embed_scatter_sorted");
}

int scatter_sorted_ordered(const void* dy, int64_t lddy, const int32_t* order, const int32_t* sorted_idx, float* dtab, int M,
                           int H, float* ws, int64_t ws_bytes, cudaStream_t s) {
  int rc = check_rows(M, H, "embed_scatter_sorted_ordered");
  if (rc) return rc;
  if (H > 1024) return set_error(MMFB_ERR_ARG, "embed_scatter_sorted_ordered: hidden size %d > 1024", H);
  if ((rc = check_aligned("embed_scatter_sorted_ordered", M, {{dy, lddy, "dy"}}))) return rc;
  if ((rc = check_workspace("embed_scatter_sorted_ordered", ws, ws_bytes, scatter_sorted_workspace_bytes(M, H)))) return rc;
  const int chunks = (M + SCATTER_CHUNK - 1) / SCATTER_CHUNK;
  const int grid = (chunks + ROW_WARPS - 1) / ROW_WARPS;
  const int nv = (H + 255) / 256;
#define SS(NV) MMFB_LAUNCH((scatter_sorted_kernel<NV, true>), grid, ROW_WARPS * 32, 0, s, (const bf16*)dy, lddy, order, sorted_idx, dtab, M, H, ws)
  if (nv <= 1) SS(1); else if (nv == 2) SS(2); else if (nv == 3) SS(3); else SS(4);
#undef SS
  if ((rc = launch_ok("embed_scatter_sorted_ordered"))) return rc;
  MMFB_LAUNCH(scatter_runs_kernel, chunks, 256, 0, s, sorted_idx, (const float*)ws, dtab, M, H);
  return launch_ok("embed_scatter_sorted_ordered runs");
}

int relu_bwd(const void* dy, const void* y, void* dz, int64_t n, cudaStream_t s) {
  if (n <= 0) return set_error(MMFB_ERR_ARG, "relu_bwd: empty");
  if ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(dz)) & 15)
    return set_error(MMFB_ERR_ARG, "relu_bwd: buffers must be 16-byte aligned");
  const int64_t thr = (n + 7) / 8;
  MMFB_LAUNCH(relu_bwd_kernel, static_cast<unsigned>((thr + 255) / 256), 256, 0, s, (const bf16*)dy, (const bf16*)y, (bf16*)dz, n);
  return launch_ok("relu_bwd");
}

int add_bf16(const void* a, const void* b, void* out, int64_t n, cudaStream_t s) {
  if (n <= 0) return set_error(MMFB_ERR_ARG, "add_bf16: empty");
  if ((reinterpret_cast<uintptr_t>(a) & 15) || (reinterpret_cast<uintptr_t>(b) & 15) || (reinterpret_cast<uintptr_t>(out) & 15))
    return set_error(MMFB_ERR_ARG, "add_bf16: buffers must be 16-byte aligned");
  const int64_t thr = (n + 7) / 8;
  MMFB_LAUNCH(add_bf16_kernel, static_cast<unsigned>((thr + 255) / 256), 256, 0, s, (const bf16*)a, (const bf16*)b, (bf16*)out, n);
  return launch_ok("add_bf16");
}

int dropout_apply(const void* x, int64_t ldx, const uint32_t* bits, int64_t ldm, float scale, void* out, int64_t ldo, int M,
                  int H, cudaStream_t s) {
  int rc = check_rows(M, H, "dropout_apply");
  if (rc) return rc;
  // the keep-bit words are read one 4-byte word at a time: no row constraint on them
  rc = check_aligned("dropout_apply", M, {{x, ldx, "x"}, {out, ldo, "out"}});
  if (rc) return rc;
  const int64_t threads = static_cast<int64_t>(M) * 32;
  MMFB_LAUNCH(dropout_apply_kernel, static_cast<unsigned>((threads + 255) / 256), 256, 0, s, (const bf16*)x, ldx, bits, ldm, scale,
                                                                                   (bf16*)out, ldo, M, H);
  return launch_ok("dropout_apply");
}

int cast_params(const float* in, void* out, int64_t n, cudaStream_t s) {
  if (n <= 0) return set_error(MMFB_ERR_ARG, "cast: empty");
  if ((reinterpret_cast<uintptr_t>(in) & 15) || (reinterpret_cast<uintptr_t>(out) & 15))
    return set_error(MMFB_ERR_ARG, "cast: buffers must be 16-byte aligned");
  const int64_t thr = (n + 7) / 8;
  MMFB_LAUNCH(cast_f32_bf16_kernel, static_cast<unsigned>((thr + 255) / 256), 256, 0, s, in, (bf16*)out, n);
  return launch_ok("cast_f32_bf16");
}

}  // namespace mmfb
