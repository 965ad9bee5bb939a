// Fused multi-head (self / cross) attention for the fusion block, forward and backward (sm_90a).
//
// Reference semantics (mmf/modules/hf_layers.py:182-210; mmf/models/vilbert.py:81-103, 421-461):
//     scores = Q K^T / sqrt(d) + M        M = additive mask [B, Skv] (0 / -10000); lower values count as -10000
//     probs  = dropout(softmax(scores))   a fully masked row is the softmax of its raw scores, never NaN
//     ctx    = probs V, heads merged back to [B, Sq, h*d]
//
// Every kernel works on 64-row tiles of one (batch, head): one warpgroup of four warps, each owning 16 rows of the
// resident tile, and a loop over 64-row blocks of the other sequence.  TMA stages the head slices straight out of the
// fused [tokens, 3*H] projection buffers (3-D tensor maps: sequence tails are zero-filled, never read from the next
// sample) into 128-byte-swizzled shared memory; the looped blocks go through a two-stage ring signalled by mbarriers, so
// the load of block i+2 overlaps the math of block i+1.  The products run on the tensor cores with wgmma m64nNk16 (bf16
// in, fp32 accumulate).  A product of two staged tiles reads both through shared-memory descriptors of the swizzled
// layout TMA wrote (no ldmatrix, no operand fragments in registers); a probability / gradient tile computed in registers
// is the A operand of the next product as it stands - the accumulator layout of two adjacent n8 tiles is the A layout
// of one k16 step - with the staged tile as the MN-major B operand.  Every wgmma group is waited for before its
// accumulators are read, and the last one of a block before the stage is refilled.
//
// Forward: online softmax over the key blocks in the log2 domain (the 1/sqrt(d) scale folded into log2(e)); the row
// log-sum-exp is saved for the backward.
// Backward: the probabilities are recomputed from Q, K and the saved row statistics (nothing of size S x S ever touches
// HBM).  Two kernels, no atomics, deterministic:
//   dq kernel : CTA owns 64 query rows, loops over key blocks:    dQ = scale * dS K
//   dkv kernel: CTA owns 64 key rows, loops over query blocks:    dV = P^T dO,  dK = scale * dS^T Q
//               (computed as S^T = K Q^T and dP^T = V dO^T, so the key rows stay the rows of every register tile)
// VARLEN instantiations (packed self- and cross-attention, include/mmfb200.h): the samples' rows are packed back to back,
// so a tile may run into the next sample; those rows are masked (keys), not stored (queries) or given P = 0 (dk/dv), and
// every CTA stays within its own sample's blocks.  Queries and keys each have their own packing (cu / total for the query
// side, cu_kv / total_kv for the key side); packed self-attention passes the same one twice.
// CAUSAL instantiations (dense self-attention with causal_len = T > 0, M4C's prefix-LM mask, m4c.py:418-437): keys from
// P = Skv - T on are a causal tail.  Where a score takes its mask value, a tail key k takes 0 if k <= q and -10000
// otherwise (the staged mask holds 0 there, mask[b, k] is not read); keys below P keep the additive mask.  No key block is
// skipped: M4C's tails (12 / 30 keys) sit inside one 64-key block, and every value stays finite, so a query whose other
// keys are all padding still gets the softmax of its raw scores, as in the reference.
// VARLEN && CAUSAL instantiations (packed self-attention with causal_len = T > 0, attention_varlen_causal.cu): the tail of
// sample b is its last T rows, from P_b = max(len_b - T, 0) on (counted within the sample; a sample shorter than T is all
// tail), found from cu after griddep_wait.  The rule is CAUSAL's with len_b in place of Skv: a tail key k takes 0 for
// queries q >= k and -10000 otherwise, keys below P_b take 0 (packing has removed the padded ones), and keys past the end
// of the sample keep the packed mode's -inf.
#include <stdlib.h>

#include "common.cuh"
#include "mmfb_internal.h"

namespace mmfb {

constexpr float LOG2E = 1.4426950408889634f;
constexpr int AT_ROWS = 64;       // rows of every staged tile
constexpr int AT_THREADS = 128;   // four warps x 16 rows

// An additive mask value as staged in shared memory (log2 domain).  Values below -10000 (HF's finfo(dtype).min, -inf)
// are clamped to -10000 first: their product with log2(e) would be -inf in fp32, and a query whose first key block is
// fully masked would then compute -inf - (-inf) = NaN in the online softmax.  -10000 is the reference's own convention
// and stays finite, so such a row keeps a finite log-sum-exp (softmax of its raw scores).  Masks at or above -10000 are
// unchanged bit for bit.
__device__ __forceinline__ float staged_mask(float m) { return fmaxf(m, -10000.0f) * LOG2E; }

// CAUSAL: the mask value (log2 domain) of query q and key kv; `staged` is the staged value of kv (0 for tail keys).  Tail
// keys past the query take -10000, the value staged_mask gives a padded key.
__device__ __forceinline__ float causal_mask(float staged, int q, int kv, int P, int Skv) {
  return (kv >= P && kv < Skv && kv > q) ? -10000.0f * LOG2E : staged;
}

// TMA of one [ROWS x D] head slice into `dst`, credited to `bar`: D/64 boxes {64, ROWS}, each a 64-column panel of
// ROWS x 128 B lines, SWIZZLE_128B (16-byte chunk index XOR row % 8) - the layout the wgmma descriptors name
template <int D, int ROWS>
__device__ __forceinline__ void load_tile(uint8_t* dst, const CUtensorMap* m, uint64_t* bar, int col0, int row0, int b) {
#pragma unroll
  for (int c = 0; c < D / 64; ++c) tma_load_3d(dst + c * ROWS * 128, m, bar, col0 + c * 64, row0, b);
}

// Issues acc[64 x 8 NT] = A[64 rows of tile a, D] * B[8 NT rows of tile b, D]^T, one wgmma per k16 step (both tiles K-major
// along D: a step is 32 B further along the 128-byte lines, the second 64-column panel follows the first).  The first
// step overwrites acc.  The caller fences before and commits / waits after.
template <int D, int NT, int AROWS, int BROWS>
__device__ __forceinline__ void wg_abt(float (&acc)[NT][4], uint32_t a, uint32_t b) {
#pragma unroll
  for (int ks = 0; ks < D / 16; ++ks) {
    const uint64_t da = gmma_desc_sw128(a + (ks >> 2) * (AROWS * 128) + (ks & 3) * 32, 16, 1024);
    const uint64_t db = gmma_desc_sw128(b + (ks >> 2) * (BROWS * 128) + (ks & 3) * 32, 16, 1024);
    wgmma_ss(acc, da, db, ks > 0 ? 1u : 0u);
  }
}

// Issues acc[64 x D] += P[64 x 16 KS] * B[16 KS rows of tile b, D]   (P: bf16 A fragments in registers; B is read MN-major:
// its rows are the k dimension, a k16 step is 16 lines = 2048 B, LBO the stride of its 64-column panels)
template <int D, int KS, int BROWS>
__device__ __forceinline__ void wg_pb(float (&acc)[D / 8][4], const uint32_t (&pf)[KS][4], uint32_t b) {
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wgmma_rs(acc, pf[ks], gmma_desc_sw128(b + ks * 2048, BROWS * 128, 1024), 1u);
}

// accumulator tile [16 x 8 NT] (fp32) -> bf16 A fragments of NT/2 k16 steps
template <int NT>
__device__ __forceinline__ void acc_to_a(const float (&c)[NT][4], uint32_t (&pf)[NT / 2][4]) {
#pragma unroll
  for (int k = 0; k < NT / 2; ++k) {
    pf[k][0] = pack_bf16x2(c[2 * k][0], c[2 * k][1]);
    pf[k][1] = pack_bf16x2(c[2 * k][2], c[2 * k][3]);
    pf[k][2] = pack_bf16x2(c[2 * k + 1][0], c[2 * k + 1][1]);
    pf[k][3] = pack_bf16x2(c[2 * k + 1][2], c[2 * k + 1][3]);
  }
}

// ----------------------------------------------------------------------------------------------
// forward
// ----------------------------------------------------------------------------------------------
struct AttnFwdDev {
  int B, H, Sq, Skv;
  const float* mask;      // [B, Skv] additive, or null
  bf16* ctx;              // [B*Sq, ldo]
  int64_t ldo;
  bf16* ctx_lo;           // optional [B*Sq, H*D] (training): bf16(O - float(ctx)), the part of O the bf16 output drops.
                          // The backward's delta = rowsum(dO * (ctx + ctx_lo)): with the bf16 O alone every dS of a row
                          // inherits the same rounding error
  float* lse2;            // [B, H, Sq]  log2-domain log-sum-exp of the scaled+masked scores
  const uint32_t* dmask;  // keep bits [B, H, Sq, W] (bit kv%32 of word kv/32) or null
  int W;
  float dscale;           // 1/(1-p)
  float scale2;           // log2(e)/sqrt(d)
  const int* cu;          // VARLEN: [B+1] first packed query row of every sample (Sq = max_q)
  int total;              // VARLEN: packed query rows
  const int* cu_kv;       // VARLEN: [B+1] first packed key row of every sample (Skv = max_kv; self-attention: cu)
  int total_kv;           // VARLEN: packed key rows
  int P;                  // CAUSAL: first key of the causal tail (Skv - causal_len); VARLEN && CAUSAL: Skv = max_len, and
                          // the kernels take causal_len = Skv - P to find each sample's own tail
};

// VARLEN: sample b owns the packed rows [cu[b], cu[b+1]) of one side's row buffers (clamped to [0, total] and to max_len
// rows); returns that range as (first row, length), the length never negative.  Read after griddep_wait, like every other
// global read.
__device__ __forceinline__ int2 varlen_rows(const int* cu, int b, int total, int max_len) {
  const int s0 = min(max(__ldg(cu + b), 0), total);
  return make_int2(s0, max(min(min(__ldg(cu + b + 1), total) - s0, max_len), 0));
}

// VARLEN && CAUSAL: the first key of the causal tail of a sample of `len` rows, within the sample: its last Skv - P rows
// (the causal_len), all of them when it is shorter.
__device__ __forceinline__ int varlen_tail(int len, int P, int Skv) { return max(len - (Skv - P), 0); }

// PACKED_ROW / PACKED_KV_ROW: tile row coordinate of a query / key tile (dense: within batch b; packed: sample b starts at
// query row seq0 and key row kv0).
// HEAD_ROW: first row of (batch-head bh, head h) in lse2 / delta / the keep bits: [B, H, Sq] dense, [H, total] packed (query
// rows).  Macros so that the dense kernels keep the exact expressions (and code) they had before the packed mode existed.
#define PACKED_ROW(r) (VARLEN ? seq0 + (r) : (r))
#define PACKED_KV_ROW(r) (VARLEN ? kv0 + (r) : (r))
#define HEAD_ROW(bh) (VARLEN ? static_cast<int64_t>(h) * p.total + seq0 : static_cast<int64_t>(bh) * p.Sq)

// grid (query tiles, heads, batch); smem: Q tile, two stages of (K block, V block), the key mask (log2 domain).
// VARLEN: packed attention (no additive mask); the tensor maps span each side's packed rows with a batch extent of 1, tiles
// load at row cu[b] + block * 64 (queries) / cu_kv[b] + block * 64 (keys), and rows past the end of the sample (the next
// sample's rows) are masked / not stored.  A sample without keys writes ctx = ctx_lo = 0 and lse2 = -inf (empty sum).
template <int D, bool VARLEN, bool CAUSAL>
__global__ void __launch_bounds__(AT_THREADS)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, AttnFwdDev p) {
  constexpr int TB = D / 64 * AT_ROWS * 128;   // bytes of one staged tile
  constexpr int DT = D / 8;                    // n8 tiles of the output
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + TB;                    // stage s: K at sKV + 2 s TB, V at sKV + (2 s + 1) TB
  const int NKB = (p.Skv + AT_ROWS - 1) / AT_ROWS;
  float* sMask = reinterpret_cast<float*>(sKV + 4 * TB);   // [NKB * 64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sMask + NKB * AT_ROWS);   // [0] Q, [1..2] K/V stages

  griddep_launch();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_ROWS, h = blockIdx.y, b = blockIdx.z;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  // dense: the sample's rows start at row 0 of batch b; VARLEN: at packed query row seq0 / key row kv0 of the single batch
  int seq0 = 0, len = p.Skv, nkb = NKB;
  int kv0 = 0, kvlen = p.Skv;
  int tail0 = 0;                               // VARLEN && CAUSAL: first tail key of this sample
  if constexpr (VARLEN) {
    const int2 r = varlen_rows(p.cu, b, p.total, p.Sq);
    seq0 = r.x;
    len = r.y;
    if (q0 >= len) return;                     // no query of this tile exists (empty samples: every tile)
    const int2 rk = varlen_rows(p.cu_kv, b, p.total_kv, p.Skv);
    kv0 = rk.x;
    kvlen = rk.y;
    nkb = (kvlen + AT_ROWS - 1) / AT_ROWS;     // the sample's own key blocks only (none without keys)
    if constexpr (CAUSAL) tail0 = varlen_tail(kvlen, p.P, p.Skv);
  }
  const int tb = VARLEN ? 0 : b;
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bars[0], TB);
    load_tile<D, AT_ROWS>(sQ, &tmQ, &bars[0], h * D, PACKED_ROW(q0), tb);
    for (int kb = 0; kb < 2 && kb < nkb; ++kb) {
      mbar_expect_tx(&bars[1 + kb], 2 * TB);
      load_tile<D, AT_ROWS>(sKV + 2 * kb * TB, &tmK, &bars[1 + kb], h * D, PACKED_KV_ROW(kb * AT_ROWS), tb);
      load_tile<D, AT_ROWS>(sKV + (2 * kb + 1) * TB, &tmV, &bars[1 + kb], h * D, PACKED_KV_ROW(kb * AT_ROWS), tb);
    }
  }
  // additive mask in the log2 domain; padded key columns (VARLEN: keys past the sample) get -inf so that exp2 yields
  // exactly 0
  for (int i = threadIdx.x; i < nkb * AT_ROWS; i += AT_THREADS) {
    if constexpr (VARLEN)
      sMask[i] = (i < kvlen) ? 0.0f : -INFINITY;
    else if constexpr (CAUSAL)
      sMask[i] = (i < p.Skv) ? (p.mask != nullptr && i < p.P ? staged_mask(p.mask[static_cast<int64_t>(b) * p.Skv + i]) : 0.0f)
                             : -INFINITY;
    else
      sMask[i] = (i < p.Skv) ? (p.mask != nullptr ? staged_mask(p.mask[static_cast<int64_t>(b) * p.Skv + i]) : 0.0f) : -INFINITY;
  }
  __syncthreads();

  const int g = lane >> 2, t4 = lane & 3;
  const int r0 = warp * 16;                    // this warp's rows of the tile
  float o[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.0f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.0f, 0.0f};
  const uint32_t* dm[2] = {nullptr, nullptr};
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = q0 + r0 + g + hr * 8;
    if (p.dmask != nullptr && q < (VARLEN ? len : p.Sq)) dm[hr] = p.dmask + (HEAD_ROW(b * p.H + h) + q) * p.W;
  }
  mbar_wait(&bars[0], 0);
  const uint32_t uQ = smem_u32(sQ);

  for (int kb = 0; kb < nkb; ++kb) {
    const int st = kb & 1;
    mbar_wait(&bars[1 + st], (kb >> 1) & 1);
    const uint32_t uK = smem_u32(sKV + 2 * st * TB), uV = uK + TB;
    float s[8][4];
    wgmma_fence();
    wg_abt<D, 8, AT_ROWS, AT_ROWS>(s, uQ, uK);
    wgmma_commit();
    wgmma_wait<0>();
    // scale + mask, block row max (the four threads of a quad share a row)
    float bmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float2 mk = *reinterpret_cast<const float2*>(sMask + kb * AT_ROWS + nt * 8 + 2 * t4);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float m = (e & 1) ? mk.y : mk.x;
        if constexpr (CAUSAL)
          m = causal_mask(m, q0 + r0 + g + (e >> 1) * 8, kb * AT_ROWS + nt * 8 + 2 * t4 + (e & 1), VARLEN ? tail0 : p.P,
                          VARLEN ? kvlen : p.Skv);
        s[nt][e] = fmaf(s[nt][e], p.scale2, m);
        bmax[e >> 1] = fmaxf(bmax[e >> 1], s[nt][e]);
      }
    }
    float corr[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      bmax[hr] = fmaxf(bmax[hr], __shfl_xor_sync(0xffffffffu, bmax[hr], 1));
      bmax[hr] = fmaxf(bmax[hr], __shfl_xor_sync(0xffffffffu, bmax[hr], 2));
      const float mn = fmaxf(mrow[hr], bmax[hr]);   // finite: every key block holds at least one real key
      corr[hr] = ex2_approx(mrow[hr] - mn);         // 0 on the first block
      mrow[hr] = mn;
      lrow[hr] *= corr[hr];
    }
#pragma unroll
    for (int i = 0; i < DT; ++i) {
      o[i][0] *= corr[0]; o[i][1] *= corr[0];
      o[i][2] *= corr[1]; o[i][3] *= corr[1];
    }
    uint32_t bits[2] = {0xFFFFFFFFu, 0xFFFFFFFFu}, bits2[2] = {0xFFFFFFFFu, 0xFFFFFFFFu};
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      if (dm[hr] != nullptr) {
        const int w0 = kb * 2;
        bits[hr] = __ldg(dm[hr] + w0);
        if (w0 + 1 < p.W) bits2[hr] = __ldg(dm[hr] + w0 + 1);
      }
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hr = e >> 1;
        const float pe = ex2_approx(s[nt][e] - mrow[hr]);   // 0 for padded columns
        lrow[hr] += pe;
        const int col = nt * 8 + 2 * t4 + (e & 1);          // key within the block
        const uint32_t w = col < 32 ? bits[hr] : bits2[hr];
        s[nt][e] = ((w >> (col & 31)) & 1u) ? pe : 0.0f;
      }
    }
    uint32_t pf[4][4];
    acc_to_a<8>(s, pf);
    wgmma_fence();
    wg_pb<D, 4, AT_ROWS>(o, pf, uV);
    wgmma_commit();
    wgmma_wait<0>();
    // every warp's wgmmas on this stage have retired: thread 0 may refill it (wgmma and TMA are both async-proxy accesses,
    // so the barrier orders them)
    __syncthreads();
    if (threadIdx.x == 0 && kb + 2 < nkb) {
      mbar_expect_tx(&bars[1 + st], 2 * TB);
      load_tile<D, AT_ROWS>(sKV + 2 * st * TB, &tmK, &bars[1 + st], h * D, PACKED_KV_ROW((kb + 2) * AT_ROWS), tb);
      load_tile<D, AT_ROWS>(sKV + (2 * st + 1) * TB, &tmV, &bars[1 + st], h * D, PACKED_KV_ROW((kb + 2) * AT_ROWS), tb);
    }
  }

#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float l = lrow[hr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int q = q0 + r0 + g + hr * 8;
    if (q >= (VARLEN ? len : p.Sq)) continue;
    if (t4 == 0) p.lse2[HEAD_ROW(b * p.H + h) + q] = mrow[hr] + log2f(l);   // VARLEN without keys: -inf + log2(0)
    const float inv = (VARLEN && kvlen == 0) ? 0.0f : p.dscale / l;         // no keys: o = 0 and l = 0, the row is 0
    const int64_t row = VARLEN ? static_cast<int64_t>(seq0) + q : static_cast<int64_t>(b) * p.Sq + q;
    bf16* dst = p.ctx + row * p.ldo + h * D;
    bf16* dlo = p.ctx_lo != nullptr ? p.ctx_lo + row * (p.H * D) + h * D : nullptr;
#pragma unroll
    for (int i = 0; i < DT; ++i) {
      const int c = i * 8 + 2 * t4;
      const float v0 = o[i][hr * 2] * inv, v1 = o[i][hr * 2 + 1] * inv;
      const uint32_t hi = pack_bf16x2(v0, v1);
      *reinterpret_cast<uint32_t*>(dst + c) = hi;
      if (dlo != nullptr) {
        const float2 hf = unpack_bf16x2(hi);
        *reinterpret_cast<uint32_t*>(dlo + c) = pack_bf16x2(v0 - hf.x, v1 - hf.y);
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// backward
// ----------------------------------------------------------------------------------------------
struct AttnBwdDev {
  int B, H, Sq, Skv;
  const float* mask;
  const float* lse2;      // [B, H, Sq]
  const float* delta;     // [B, H, Sq]
  const uint32_t* dmask;
  int W;
  float dscale, scale, scale2;
  bf16* out0; int64_t ld0;   // dq (dq kernel) / dk (dkv kernel)
  bf16* out1; int64_t ld1;   // dv (dkv kernel)
  const int* cu;             // VARLEN, as in AttnFwdDev
  int total;
  const int* cu_kv;
  int total_kv;
  int P;                     // CAUSAL, as in AttnFwdDev
};

// dQ for 64 query rows.  smem: Q, dO tiles; two stages of (K block, V block).  VARLEN and CAUSAL as in the forward (a
// sample without keys writes dq = 0).
template <int D, bool DROP, bool VARLEN, bool CAUSAL>
__global__ void __launch_bounds__(AT_THREADS)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                   const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, AttnBwdDev p) {
  constexpr int TB = D / 64 * AT_ROWS * 128;
  constexpr int DT = D / 8;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sdO = smem + TB;
  uint8_t* sKV = smem + 2 * TB;
  const int NKB = (p.Skv + AT_ROWS - 1) / AT_ROWS;
  float* sMask = reinterpret_cast<float*>(sKV + 4 * TB);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sMask + NKB * AT_ROWS);

  griddep_launch();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_ROWS, h = blockIdx.y, b = blockIdx.z;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmdO);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  int seq0 = 0, len = p.Skv, nkb = NKB;
  int kv0 = 0, kvlen = p.Skv;
  int tail0 = 0;
  if constexpr (VARLEN) {
    const int2 r = varlen_rows(p.cu, b, p.total, p.Sq);
    seq0 = r.x;
    len = r.y;
    if (q0 >= len) return;
    const int2 rk = varlen_rows(p.cu_kv, b, p.total_kv, p.Skv);
    kv0 = rk.x;
    kvlen = rk.y;
    nkb = (kvlen + AT_ROWS - 1) / AT_ROWS;
    if constexpr (CAUSAL) tail0 = varlen_tail(kvlen, p.P, p.Skv);
  }
  const int tb = VARLEN ? 0 : b;
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bars[0], 2 * TB);
    load_tile<D, AT_ROWS>(sQ, &tmQ, &bars[0], h * D, PACKED_ROW(q0), tb);
    load_tile<D, AT_ROWS>(sdO, &tmdO, &bars[0], h * D, PACKED_ROW(q0), tb);
    for (int kb = 0; kb < 2 && kb < nkb; ++kb) {
      mbar_expect_tx(&bars[1 + kb], 2 * TB);
      load_tile<D, AT_ROWS>(sKV + 2 * kb * TB, &tmK, &bars[1 + kb], h * D, PACKED_KV_ROW(kb * AT_ROWS), tb);
      load_tile<D, AT_ROWS>(sKV + (2 * kb + 1) * TB, &tmV, &bars[1 + kb], h * D, PACKED_KV_ROW(kb * AT_ROWS), tb);
    }
  }
  for (int i = threadIdx.x; i < nkb * AT_ROWS; i += AT_THREADS) {
    if constexpr (VARLEN)
      sMask[i] = (i < kvlen) ? 0.0f : -INFINITY;
    else if constexpr (CAUSAL)
      sMask[i] = (i < p.Skv) ? (p.mask != nullptr && i < p.P ? staged_mask(p.mask[static_cast<int64_t>(b) * p.Skv + i]) : 0.0f)
                             : -INFINITY;
    else
      sMask[i] = (i < p.Skv) ? (p.mask != nullptr ? staged_mask(p.mask[static_cast<int64_t>(b) * p.Skv + i]) : 0.0f) : -INFINITY;
  }
  __syncthreads();

  const int g = lane >> 2, t4 = lane & 3;
  const int r0 = warp * 16;
  const int64_t bh = static_cast<int64_t>(b) * p.H + h;
  float lse[2], dlt[2];
  const uint32_t* dm[2] = {nullptr, nullptr};
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = q0 + r0 + g + hr * 8;
    const bool ok = q < (VARLEN ? len : p.Sq);
    lse[hr] = ok ? p.lse2[HEAD_ROW(bh) + q] : INFINITY;      // rows past the sequence: P = 0
    dlt[hr] = ok ? p.delta[HEAD_ROW(bh) + q] : 0.0f;
    if (DROP && ok) dm[hr] = p.dmask + (HEAD_ROW(bh) + q) * p.W;
  }
  float dq[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.0f;
  mbar_wait(&bars[0], 0);
  const uint32_t uQ = smem_u32(sQ), udO = smem_u32(sdO);

  for (int kb = 0; kb < nkb; ++kb) {
    const int st = kb & 1;
    mbar_wait(&bars[1 + st], (kb >> 1) & 1);
    const uint32_t uK = smem_u32(sKV + 2 * st * TB), uV = uK + TB;
    float s[8][4], dp[8][4];
    wgmma_fence();
    wg_abt<D, 8, AT_ROWS, AT_ROWS>(s, uQ, uK);
    wg_abt<D, 8, AT_ROWS, AT_ROWS>(dp, udO, uV);
    wgmma_commit();
    wgmma_wait<0>();
    uint32_t bits[2][2] = {{0xFFFFFFFFu, 0xFFFFFFFFu}, {0xFFFFFFFFu, 0xFFFFFFFFu}};
    if (DROP) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        if (dm[hr] != nullptr) {
          bits[hr][0] = __ldg(dm[hr] + kb * 2);
          if (kb * 2 + 1 < p.W) bits[hr][1] = __ldg(dm[hr] + kb * 2 + 1);
        }
      }
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float2 mk = *reinterpret_cast<const float2*>(sMask + kb * AT_ROWS + nt * 8 + 2 * t4);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hr = e >> 1;
        float m = (e & 1) ? mk.y : mk.x;
        if constexpr (CAUSAL)
          m = causal_mask(m, q0 + r0 + g + hr * 8, kb * AT_ROWS + nt * 8 + 2 * t4 + (e & 1), VARLEN ? tail0 : p.P,
                          VARLEN ? kvlen : p.Skv);
        const float pe = ex2_approx(fmaf(s[nt][e], p.scale2, m) - lse[hr]);
        float dpe = dp[nt][e];
        if (DROP) {
          const int col = nt * 8 + 2 * t4 + (e & 1);
          dpe = ((bits[hr][col >> 5] >> (col & 31)) & 1u) ? dpe * p.dscale : 0.0f;
        }
        s[nt][e] = pe * (dpe - dlt[hr]);                    // dS
      }
    }
    uint32_t sf[4][4];
    acc_to_a<8>(s, sf);
    wgmma_fence();
    wg_pb<D, 4, AT_ROWS>(dq, sf, uK);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();
    if (threadIdx.x == 0 && kb + 2 < nkb) {
      mbar_expect_tx(&bars[1 + st], 2 * TB);
      load_tile<D, AT_ROWS>(sKV + 2 * st * TB, &tmK, &bars[1 + st], h * D, PACKED_KV_ROW((kb + 2) * AT_ROWS), tb);
      load_tile<D, AT_ROWS>(sKV + (2 * st + 1) * TB, &tmV, &bars[1 + st], h * D, PACKED_KV_ROW((kb + 2) * AT_ROWS), tb);
    }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = q0 + r0 + g + hr * 8;
    if (q >= (VARLEN ? len : p.Sq)) continue;
    const int64_t row = VARLEN ? static_cast<int64_t>(seq0) + q : static_cast<int64_t>(b) * p.Sq + q;
    bf16* dst = p.out0 + row * p.ld0 + h * D;
#pragma unroll
    for (int i = 0; i < DT; ++i)
      *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t4) = pack_bf16x2(dq[i][hr * 2] * p.scale, dq[i][hr * 2 + 1] * p.scale);
  }
}

// dK, dV for 64 key rows.  smem: K, V tiles; two stages of (Q block, dO block) of QB query rows.  The register tiles are
// transposed products (rows = keys, columns = queries).  VARLEN as in the forward; query rows past the end of the sample
// take lse = +inf and delta = 0 (P = 0), like rows past Sq, and a sample without queries writes dk = dv = 0.  CAUSAL as in
// the forward, with the key of a row and the query of a column.
template <int D, bool DROP, int QB, bool VARLEN, bool CAUSAL>
__global__ void __launch_bounds__(AT_THREADS)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO, AttnBwdDev p) {
  constexpr int TB = D / 64 * AT_ROWS * 128;    // resident key tile
  constexpr int QTB = D / 64 * QB * 128;        // streamed query block
  constexpr int DT = D / 8, NT = QB / 8;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* sK = smem;
  uint8_t* sV = smem + TB;
  uint8_t* sQd = smem + 2 * TB;                 // stage s: Q at sQd + 2 s QTB, dO at sQd + (2 s + 1) QTB
  float* sMask = reinterpret_cast<float*>(sQd + 4 * QTB);   // [64] this tile's keys
  uint64_t* bars = reinterpret_cast<uint64_t*>(sMask + AT_ROWS);

  griddep_launch();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = blockIdx.x * AT_ROWS, h = blockIdx.y, b = blockIdx.z;
  const int NQB = (p.Sq + QB - 1) / QB;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmdO);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  int seq0 = 0, len = p.Skv, nqb = NQB;
  int kv0 = 0, kvlen = p.Skv;
  int tail0 = 0;
  if constexpr (VARLEN) {
    const int2 rk = varlen_rows(p.cu_kv, b, p.total_kv, p.Skv);
    kv0 = rk.x;
    kvlen = rk.y;
    if (k0 >= kvlen) return;                    // no key of this tile exists
    const int2 r = varlen_rows(p.cu, b, p.total, p.Sq);
    seq0 = r.x;
    len = r.y;
    nqb = (len + QB - 1) / QB;                  // the sample's own query blocks only (none without queries)
    if constexpr (CAUSAL) tail0 = varlen_tail(kvlen, p.P, p.Skv);
  }
  const int tb = VARLEN ? 0 : b;
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bars[0], 2 * TB);
    load_tile<D, AT_ROWS>(sK, &tmK, &bars[0], h * D, PACKED_KV_ROW(k0), tb);
    load_tile<D, AT_ROWS>(sV, &tmV, &bars[0], h * D, PACKED_KV_ROW(k0), tb);
    for (int qb = 0; qb < 2 && qb < nqb; ++qb) {
      mbar_expect_tx(&bars[1 + qb], 2 * QTB);
      load_tile<D, QB>(sQd + 2 * qb * QTB, &tmQ, &bars[1 + qb], h * D, PACKED_ROW(qb * QB), tb);
      load_tile<D, QB>(sQd + (2 * qb + 1) * QTB, &tmdO, &bars[1 + qb], h * D, PACKED_ROW(qb * QB), tb);
    }
  }
  for (int i = threadIdx.x; i < AT_ROWS; i += AT_THREADS) {
    const int kv = k0 + i;
    if constexpr (VARLEN)
      sMask[i] = (kv < kvlen) ? 0.0f : -INFINITY;
    else if constexpr (CAUSAL)
      sMask[i] = (kv < p.Skv) ? (p.mask != nullptr && kv < p.P ? staged_mask(p.mask[static_cast<int64_t>(b) * p.Skv + kv]) : 0.0f)
                              : -INFINITY;
    else
      sMask[i] = (kv < p.Skv) ? (p.mask != nullptr ? staged_mask(p.mask[static_cast<int64_t>(b) * p.Skv + kv]) : 0.0f) : -INFINITY;
  }
  __syncthreads();

  const int g = lane >> 2, t4 = lane & 3;
  const int r0 = warp * 16;
  const int64_t bh = static_cast<int64_t>(b) * p.H + h;
  const float mk[2] = {sMask[r0 + g], sMask[r0 + g + 8]};
  // keys r0 + g and r0 + g + 8 share one keep-bit word (16-aligned group of keys)
  const int kw = (k0 + r0) >> 5, ksh0 = (k0 + r0 + g) & 31;
  float dk[DT][4], dv[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.0f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.0f;
  }
  mbar_wait(&bars[0], 0);
  const uint32_t uK = smem_u32(sK), uV = smem_u32(sV);

  for (int qb = 0; qb < nqb; ++qb) {
    const int st = qb & 1;
    mbar_wait(&bars[1 + st], (qb >> 1) & 1);
    const uint32_t uQ = smem_u32(sQd + 2 * st * QTB), udO = uQ + QTB;
    float s[NT][4], dp[NT][4];
    wgmma_fence();
    wg_abt<D, NT, AT_ROWS, QB>(s, uK, uQ);                  // S^T  [keys x queries]
    wg_abt<D, NT, AT_ROWS, QB>(dp, uV, udO);                // dP^T
    wgmma_commit();
    wgmma_wait<0>();
    float pd[NT][4];                                        // dropped probabilities P^T * keep * dscale
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int q = qb * QB + nt * 8 + 2 * t4 + j;
        const bool ok = q < (VARLEN ? len : p.Sq);
        const float lse = ok ? __ldg(p.lse2 + HEAD_ROW(bh) + q) : INFINITY;
        const float dlt = ok ? __ldg(p.delta + HEAD_ROW(bh) + q) : 0.0f;
        uint32_t w = 0xFFFFFFFFu;
        if (DROP && ok && k0 + r0 < (VARLEN ? kvlen : p.Skv)) w = __ldg(p.dmask + (HEAD_ROW(bh) + q) * p.W + kw);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int e = hr * 2 + j;
          float m = mk[hr];
          if constexpr (CAUSAL) m = causal_mask(m, q, k0 + r0 + g + hr * 8, VARLEN ? tail0 : p.P, VARLEN ? kvlen : p.Skv);
          const float pe = ex2_approx(fmaf(s[nt][e], p.scale2, m) - lse);
          const bool keep = !DROP || ((w >> (ksh0 + hr * 8)) & 1u);
          const float dpe = keep ? dp[nt][e] * p.dscale : 0.0f;
          pd[nt][e] = keep ? pe * p.dscale : 0.0f;
          s[nt][e] = pe * (dpe - dlt);                      // dS^T
        }
      }
    }
    uint32_t pf[NT / 2][4], sf[NT / 2][4];
    acc_to_a<NT>(pd, pf);
    acc_to_a<NT>(s, sf);
    wgmma_fence();
    wg_pb<D, NT / 2, QB>(dv, pf, udO);
    wg_pb<D, NT / 2, QB>(dk, sf, uQ);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();
    if (threadIdx.x == 0 && qb + 2 < nqb) {
      mbar_expect_tx(&bars[1 + st], 2 * QTB);
      load_tile<D, QB>(sQd + 2 * st * QTB, &tmQ, &bars[1 + st], h * D, PACKED_ROW((qb + 2) * QB), tb);
      load_tile<D, QB>(sQd + (2 * st + 1) * QTB, &tmdO, &bars[1 + st], h * D, PACKED_ROW((qb + 2) * QB), tb);
    }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int kv = k0 + r0 + g + hr * 8;
    if (kv >= (VARLEN ? kvlen : p.Skv)) continue;
    const int64_t row = VARLEN ? static_cast<int64_t>(kv0) + kv : static_cast<int64_t>(b) * p.Skv + kv;
    bf16* dK = p.out0 + row * p.ld0 + h * D;
    bf16* dV = p.out1 + row * p.ld1 + h * D;
#pragma unroll
    for (int i = 0; i < DT; ++i) {
      *reinterpret_cast<uint32_t*>(dK + i * 8 + 2 * t4) = pack_bf16x2(dk[i][hr * 2] * p.scale, dk[i][hr * 2 + 1] * p.scale);
      *reinterpret_cast<uint32_t*>(dV + i * 8 + 2 * t4) = pack_bf16x2(dv[i][hr * 2], dv[i][hr * 2 + 1]);
    }
  }
}

// delta[b,h,q] = sum_d dO[b,q,h,d] * O[b,q,h,d].  One warp per token row, 16-byte vector loads; a head of D
// elements is owned by D/8 consecutive lanes and reduced with shuffles (coalesced 512 B / 1 KB per warp access).
// Every row is a query row of some sample, so the packed layout [H, total] is this kernel's own with B = 1, Sq = total:
// the varlen backward launches it unchanged (it is defined once, in the dense translation unit).
#if defined(MMFB_ATTN_VARLEN_TU) || defined(MMFB_ATTN_PROBS_TU) || defined(MMFB_ATTN_CAUSAL_TU) || \
    defined(MMFB_ATTN_VARLEN_CAUSAL_TU)
__global__ void attn_delta_kernel(const bf16* __restrict__ dO, int64_t ld_do, const bf16* __restrict__ O,
                                  int64_t ld_o, const bf16* __restrict__ Olo, float* __restrict__ delta, int B, int H,
                                  int Sq, int D);
#else
__global__ void attn_delta_kernel(const bf16* __restrict__ dO, int64_t ld_do, const bf16* __restrict__ O,
                                  int64_t ld_o, const bf16* __restrict__ Olo, float* __restrict__ delta, int B, int H,
                                  int Sq, int D) {
  griddep_launch();
  griddep_wait();
  const int64_t tok = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (tok >= static_cast<int64_t>(B) * Sq) return;
  const int W = H * D;
  const int lanes_per_head = D / 8;           // 8 (d=64) or 16 (d=128)
  const int b = tok / Sq, q = tok % Sq;
  for (int base = 0; base < W; base += 256) {   // warp-uniform trip count: every lane takes part in the shuffles
    const int col = base + lane * 8;
    const bool act = col < W;
    float x[8];
    float s = 0.0f;
    if (act) {
      const uint4 u = *reinterpret_cast<const uint4*>(dO + tok * ld_do + col);
      float2 t;
      t = unpack_bf16x2(u.x); x[0] = t.x; x[1] = t.y;
      t = unpack_bf16x2(u.y); x[2] = t.x; x[3] = t.y;
      t = unpack_bf16x2(u.z); x[4] = t.x; x[5] = t.y;
      t = unpack_bf16x2(u.w); x[6] = t.x; x[7] = t.y;
    }
    if (act) {
      const uint4 u = *reinterpret_cast<const uint4*>(O + tok * ld_o + col);
      float2 t;
      float o[8];
      t = unpack_bf16x2(u.x); o[0] = t.x; o[1] = t.y;
      t = unpack_bf16x2(u.y); o[2] = t.x; o[3] = t.y;
      t = unpack_bf16x2(u.z); o[4] = t.x; o[5] = t.y;
      t = unpack_bf16x2(u.w); o[6] = t.x; o[7] = t.y;
      if (Olo != nullptr) {      // O = ctx + ctx_lo (the forward's fp32 value to ~2^-17)
        const uint4 l = *reinterpret_cast<const uint4*>(Olo + tok * static_cast<int64_t>(W) + col);
        t = unpack_bf16x2(l.x); o[0] += t.x; o[1] += t.y;
        t = unpack_bf16x2(l.y); o[2] += t.x; o[3] += t.y;
        t = unpack_bf16x2(l.z); o[4] += t.x; o[5] += t.y;
        t = unpack_bf16x2(l.w); o[6] += t.x; o[7] += t.y;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) s += x[e] * o[e];
    }
    // reduce over the lanes of this head (lanes_per_head is a power of two dividing 32; W % 256 may leave idle lanes)
    for (int o = lanes_per_head >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (act && (lane % lanes_per_head) == 0) delta[(static_cast<int64_t>(b) * H + col / D) * Sq + q] = s;
  }
}

#endif  // MMFB_ATTN_VARLEN_TU || MMFB_ATTN_PROBS_TU || MMFB_ATTN_CAUSAL_TU || MMFB_ATTN_VARLEN_CAUSAL_TU

// ----------------------------------------------------------------------------------------------
// host
// ----------------------------------------------------------------------------------------------
static int check_attn_common(const mmfb_attn_args& a, const char* who) {
  if (a.B <= 0 || a.heads <= 0 || a.Sq <= 0 || a.Skv <= 0) return set_error(MMFB_ERR_ARG, "%s: empty problem", who);
  if (a.head_dim != 64 && a.head_dim != 128)
    return set_error(MMFB_ERR_ARG, "%s: head_dim must be 64 or 128 (got %d)", who, a.head_dim);
  const int max_kv = a.head_dim == 64 ? 384 : 256;
  if (a.Skv > max_kv)
    return set_error(MMFB_ERR_ARG, "%s: Skv=%d exceeds the single-pass limit %d for head_dim %d", who, a.Skv, max_kv,
                     a.head_dim);
  if (a.causal_len < 0) return set_error(MMFB_ERR_ARG, "%s: negative causal_len (%d)", who, a.causal_len);
  if (a.causal_len > 0 && (a.Sq != a.Skv || a.causal_len > a.Skv))
    return set_error(MMFB_ERR_ARG, "%s: a causal tail needs self-attention (Sq=%d, Skv=%d) and causal_len (%d) <= Skv", who,
                     a.Sq, a.Skv, a.causal_len);
  return MMFB_OK;
}

// the packed entry points and the probabilities kernel have no causal tail
static inline int check_no_causal(const mmfb_attn_args& a, const char* who) {
  if (a.causal_len != 0) return set_error(MMFB_ERR_ARG, "%s: causal_len must be 0 (got %d)", who, a.causal_len);
  return MMFB_OK;
}

static int set_smem(const void* kern, int bytes, const char* who) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "%s smem attr (%d B): %s", who, bytes, cudaGetErrorString(e));
  return MMFB_OK;
}

// A tensor map over the [rows, heads * D] head columns of one operand: dense = B batches of S rows; packed (VARLEN) =
// one batch of `total` rows of its side, so that a tile at cu[b] + block * 64 never depends on B.  A packed side with no
// rows has no valid map; the caller then passes the other side's map, which no CTA loads through (every sample's loop over
// the empty side has no blocks).
static int head_map(CUtensorMap* m, const void* ptr, int W, int64_t ld, int rows, int batches, int box_rows) {
  return make_tmap_3d(m, ptr, W, rows, batches, ld, ld * rows, 64, box_rows);
}

template <int D, bool VARLEN, bool CAUSAL = false>
static int attn_fwd_launch(const mmfb_attn_args& a, const int32_t* cu, int total, const int32_t* cu_kv, int total_kv,
                           cudaStream_t stream) {
  const int W = a.heads * D;
  const int nb = VARLEN ? 1 : a.B, rq = VARLEN ? total : a.Sq, rkv = VARLEN ? total_kv : a.Skv;
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  if ((rc = head_map(&tmQ, a.q, W, a.ldq, rq, nb, AT_ROWS))) return rc;
  if (rkv > 0) {
    if ((rc = head_map(&tmK, a.k, W, a.ldk, rkv, nb, AT_ROWS))) return rc;
    if ((rc = head_map(&tmV, a.v, W, a.ldv, rkv, nb, AT_ROWS))) return rc;
  } else {
    tmK = tmV = tmQ;                         // no keys at all: every sample writes zeros without loading a key block
  }
  const int NKB = (a.Skv + AT_ROWS - 1) / AT_ROWS;
  const int smem = 5 * (D / 64) * AT_ROWS * 128 + NKB * AT_ROWS * 4 + 64 + 1024;
  AttnFwdDev p;
  p.B = a.B; p.H = a.heads; p.Sq = a.Sq; p.Skv = a.Skv;
  p.mask = a.mask;
  p.ctx = reinterpret_cast<bf16*>(a.ctx); p.ldo = a.ldo;
  p.lse2 = a.lse2;
  p.ctx_lo = reinterpret_cast<bf16*>(a.ctx_lo);
  p.dmask = a.drop_mask; p.W = (a.Skv + 31) / 32; p.dscale = a.drop_mask ? a.drop_scale : 1.0f;
  p.scale2 = LOG2E / sqrtf(static_cast<float>(D));
  p.cu = cu; p.total = total;
  p.cu_kv = cu_kv; p.total_kv = total_kv;
  p.P = a.Skv - a.causal_len;
  auto kern = attn_fwd_kernel<D, VARLEN, CAUSAL>;
  static int smem_set = 0;
  if (smem > smem_set) {
    if ((rc = set_smem(reinterpret_cast<const void*>(kern), smem, "attn_fwd"))) return rc;
    smem_set = smem;
  }
  dim3 grid((a.Sq + AT_ROWS - 1) / AT_ROWS, a.heads, a.B);
  MMFB_LAUNCH(kern, grid, AT_THREADS, smem, stream, tmQ, tmK, tmV, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "attn_fwd launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

template <int D, bool DROP, bool VARLEN, bool CAUSAL>
static int attn_bwd_kernels(const mmfb_attn_args& a, const AttnBwdDev& base, int total, int total_kv, cudaStream_t stream) {
  constexpr int QB = (D == 64) ? 64 : 32;   // query block of the dK/dV kernel: d = 128 keeps its tiles in registers
  const int W = a.heads * D;
  const int nb = VARLEN ? 1 : a.B, rq = VARLEN ? total : a.Sq, rkv = VARLEN ? total_kv : a.Skv;
  CUtensorMap tmQ, tmK, tmV, tmdO, tmQc, tmdOc;
  int rc;
  // a packed side without rows borrows the other side's maps (never loaded through, see head_map); rq + rkv > 0
  if (rq > 0) {
    if ((rc = head_map(&tmQ, a.q, W, a.ldq, rq, nb, AT_ROWS))) return rc;
    if ((rc = head_map(&tmdO, a.dctx, W, a.ld_dctx, rq, nb, AT_ROWS))) return rc;
  }
  if (rkv > 0) {
    if ((rc = head_map(&tmK, a.k, W, a.ldk, rkv, nb, AT_ROWS))) return rc;
    if ((rc = head_map(&tmV, a.v, W, a.ldv, rkv, nb, AT_ROWS))) return rc;
  } else {
    tmK = tmV = tmQ;
  }
  if (rq <= 0) tmQ = tmdO = tmK;
  tmQc = tmQ;
  tmdOc = tmdO;
  if (QB != AT_ROWS && rq > 0) {
    if ((rc = head_map(&tmQc, a.q, W, a.ldq, rq, nb, QB))) return rc;
    if ((rc = head_map(&tmdOc, a.dctx, W, a.ld_dctx, rq, nb, QB))) return rc;
  }
  const int TB = (D / 64) * AT_ROWS * 128;
  const int NKB = (a.Skv + AT_ROWS - 1) / AT_ROWS;
  const int smem_q = 6 * TB + NKB * AT_ROWS * 4 + 64 + 1024;
  const int smem_kv = 2 * TB + 4 * (D / 64) * QB * 128 + AT_ROWS * 4 + 64 + 1024;
  static int set_q = 0;
  static bool set_kv = false;
  if (smem_q > set_q) {
    if ((rc = set_smem(reinterpret_cast<const void*>(attn_bwd_dq_kernel<D, DROP, VARLEN, CAUSAL>), smem_q, "attn_bwd_dq"))) return rc;
    set_q = smem_q;
  }
  if (!set_kv) {
    if ((rc = set_smem(reinterpret_cast<const void*>(attn_bwd_dkv_kernel<D, DROP, QB, VARLEN, CAUSAL>), smem_kv, "attn_bwd_dkv")))
      return rc;
    set_kv = true;
  }
  AttnBwdDev p = base;
  // dense: both always launch.  Packed: no query rows -> no dq kernel (the dk/dv kernel still writes every key row, as 0),
  // no key rows -> no dk/dv kernel (the dq kernel writes every query row, as 0)
  if (rq > 0 && a.Sq > 0) {
    p.out0 = reinterpret_cast<bf16*>(a.dq); p.ld0 = a.ld_dq; p.out1 = nullptr; p.ld1 = 0;
    MMFB_LAUNCH((attn_bwd_dq_kernel<D, DROP, VARLEN, CAUSAL>), dim3((a.Sq + AT_ROWS - 1) / AT_ROWS, a.heads, a.B), AT_THREADS, smem_q,
                stream, tmQ, tmdO, tmK, tmV, p);
    count_launch();
  }
  if (rkv > 0 && a.Skv > 0) {
    p.out0 = reinterpret_cast<bf16*>(a.dk); p.ld0 = a.ld_dk;
    p.out1 = reinterpret_cast<bf16*>(a.dv); p.ld1 = a.ld_dv;
    MMFB_LAUNCH((attn_bwd_dkv_kernel<D, DROP, QB, VARLEN, CAUSAL>), dim3((a.Skv + AT_ROWS - 1) / AT_ROWS, a.heads, a.B), AT_THREADS,
                smem_kv, stream, tmK, tmV, tmQc, tmdOc, p);
    count_launch();
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "attn_bwd launch: %s", cudaGetErrorString(e));
  return MMFB_OK;
}

template <int D, bool VARLEN, bool CAUSAL = false>
static int attn_bwd_launch(const mmfb_attn_args& a, const int32_t* cu, int total, const int32_t* cu_kv, int total_kv,
                           cudaStream_t stream) {
  // delta = rowsum(dO * O); packed rows are one batch of `total` query rows
  if (!VARLEN || total > 0) {
    const int nb = VARLEN ? 1 : a.B, rq = VARLEN ? total : a.Sq;
    const int64_t warps = static_cast<int64_t>(nb) * rq;
    const int threads = 256;
    const int64_t blocks = (warps * 32 + threads - 1) / threads;
    MMFB_LAUNCH(attn_delta_kernel, static_cast<unsigned>(blocks), threads, 0, stream,
        reinterpret_cast<const bf16*>(a.dctx), a.ld_dctx, reinterpret_cast<const bf16*>(a.ctx), a.ldo, reinterpret_cast<const bf16*>(a.ctx_lo), a.delta,
        nb, a.heads, rq, D);
    count_launch();
  }
  AttnBwdDev p;
  p.B = a.B; p.H = a.heads; p.Sq = a.Sq; p.Skv = a.Skv;
  p.mask = a.mask; p.lse2 = a.lse2; p.delta = a.delta;
  p.dmask = a.drop_mask; p.W = (a.Skv + 31) / 32; p.dscale = a.drop_mask ? a.drop_scale : 1.0f;
  p.scale = 1.0f / sqrtf(static_cast<float>(D));
  p.scale2 = LOG2E * p.scale;
  p.cu = cu; p.total = total;
  p.cu_kv = cu_kv; p.total_kv = total_kv;
  p.P = a.Skv - a.causal_len;
  return a.drop_mask != nullptr ? attn_bwd_kernels<D, true, VARLEN, CAUSAL>(a, p, total, total_kv, stream)
                                : attn_bwd_kernels<D, false, VARLEN, CAUSAL>(a, p, total, total_kv, stream);
}

// The dense entry points instantiate the dense kernels only, attention_varlen.cu (which includes this file) the packed
// ones, attention_causal.cu the dense ones with a causal tail and attention_varlen_causal.cu the packed ones with a causal
// tail: instantiated in one translation unit, they share inlined helpers that the compiler then schedules differently,
// and the dense d = 64 forward would not keep the code it has without the other modes.  attention_probs.cu includes this
// file for its helpers only and instantiates none.
#if !defined(MMFB_ATTN_VARLEN_TU) && !defined(MMFB_ATTN_PROBS_TU) && !defined(MMFB_ATTN_CAUSAL_TU) && \
    !defined(MMFB_ATTN_VARLEN_CAUSAL_TU)
int attn_fwd(const mmfb_attn_args& a, cudaStream_t stream) {
  int rc = check_attn_common(a, "attn_fwd");
  if (rc) return rc;
  if (!a.q || !a.k || !a.v || !a.ctx || !a.lse2) return set_error(MMFB_ERR_ARG, "attn_fwd: null pointer");
  if (a.causal_len != 0) return attn_causal_fwd(a, stream);
  return a.head_dim == 64 ? attn_fwd_launch<64, false>(a, nullptr, 0, nullptr, 0, stream)
                          : attn_fwd_launch<128, false>(a, nullptr, 0, nullptr, 0, stream);
}

int attn_bwd(const mmfb_attn_args& a, cudaStream_t stream) {
  int rc = check_attn_common(a, "attn_bwd");
  if (rc) return rc;
  if (!a.q || !a.k || !a.v || !a.ctx || !a.lse2 || !a.dctx || !a.delta || !a.dq || !a.dk || !a.dv)
    return set_error(MMFB_ERR_ARG, "attn_bwd: null pointer");
  if (a.causal_len != 0) return attn_causal_bwd(a, stream);
  return a.head_dim == 64 ? attn_bwd_launch<64, false>(a, nullptr, 0, nullptr, 0, stream)
                          : attn_bwd_launch<128, false>(a, nullptr, 0, nullptr, 0, stream);
}

#elif defined(MMFB_ATTN_VARLEN_TU)

// Packed self-attention: Sq = Skv = max_len (the grid extent), no additive mask, `cu` on the device and never read here.
static int check_varlen(const mmfb_attn_args& a, const int32_t* cu, int total, const char* who) {
  int rc = check_attn_common(a, who);
  if (rc) return rc;
  if ((rc = check_no_causal(a, who))) return rc;
  if (a.Sq != a.Skv) return set_error(MMFB_ERR_ARG, "%s: self-attention only, Sq (%d) must equal Skv (%d) = max_len", who, a.Sq, a.Skv);
  if (a.mask != nullptr) return set_error(MMFB_ERR_ARG, "%s: mask must be NULL (packing has removed the masked keys)", who);
  if (!cu) return set_error(MMFB_ERR_ARG, "%s: null cu_seqlens", who);
  if (total < 0) return set_error(MMFB_ERR_ARG, "%s: negative total (%d)", who, total);
  return MMFB_OK;
}

int attn_varlen_fwd(const mmfb_attn_args& a, const int32_t* cu, int total, cudaStream_t stream) {
  int rc = check_varlen(a, cu, total, "attn_varlen_fwd");
  if (rc) return rc;
  if (total == 0) return MMFB_OK;           // every sample is empty: nothing to compute or write
  if (!a.q || !a.k || !a.v || !a.ctx || !a.lse2) return set_error(MMFB_ERR_ARG, "attn_varlen_fwd: null pointer");
  return a.head_dim == 64 ? attn_fwd_launch<64, true>(a, cu, total, cu, total, stream)
                          : attn_fwd_launch<128, true>(a, cu, total, cu, total, stream);
}

int attn_varlen_bwd(const mmfb_attn_args& a, const int32_t* cu, int total, cudaStream_t stream) {
  int rc = check_varlen(a, cu, total, "attn_varlen_bwd");
  if (rc) return rc;
  if (total == 0) return MMFB_OK;
  if (!a.q || !a.k || !a.v || !a.ctx || !a.lse2 || !a.dctx || !a.delta || !a.dq || !a.dk || !a.dv)
    return set_error(MMFB_ERR_ARG, "attn_varlen_bwd: null pointer");
  return a.head_dim == 64 ? attn_bwd_launch<64, true>(a, cu, total, cu, total, stream)
                          : attn_bwd_launch<128, true>(a, cu, total, cu, total, stream);
}

// Packed cross-attention: queries from one packing (cu_q / total_q, Sq = max_q), keys and values from another (cu_kv /
// total_kv, Skv = max_kv).  Either side of a sample may be empty, and so may a whole side; Sq / Skv = 0 are legal then.
static int check_varlen_cross(const mmfb_attn_args& a, const int32_t* cu_q, int total_q, const int32_t* cu_kv, int total_kv,
                              const char* who) {
  if (a.B <= 0 || a.heads <= 0 || a.Sq < 0 || a.Skv < 0)
    return set_error(MMFB_ERR_ARG, "%s: B and heads must be positive, Sq and Skv not negative", who);
  if (a.head_dim != 64 && a.head_dim != 128)
    return set_error(MMFB_ERR_ARG, "%s: head_dim must be 64 or 128 (got %d)", who, a.head_dim);
  const int max_kv = a.head_dim == 64 ? 384 : 256;
  if (a.Skv > max_kv)
    return set_error(MMFB_ERR_ARG, "%s: Skv=%d exceeds the single-pass limit %d for head_dim %d", who, a.Skv, max_kv,
                     a.head_dim);
  if (a.mask != nullptr) return set_error(MMFB_ERR_ARG, "%s: mask must be NULL (packing has removed the masked keys)", who);
  int rc = check_no_causal(a, who);
  if (rc) return rc;
  if (!cu_q || !cu_kv) return set_error(MMFB_ERR_ARG, "%s: null cu_q / cu_kv", who);
  if (total_q < 0 || total_kv < 0) return set_error(MMFB_ERR_ARG, "%s: negative total (%d, %d)", who, total_q, total_kv);
  return MMFB_OK;
}

int attn_varlen_cross_fwd(const mmfb_attn_args& a, const int32_t* cu_q, int total_q, const int32_t* cu_kv, int total_kv,
                          cudaStream_t stream) {
  int rc = check_varlen_cross(a, cu_q, total_q, cu_kv, total_kv, "attn_varlen_cross_fwd");
  if (rc) return rc;
  if (total_q == 0 || a.Sq == 0) return MMFB_OK;   // no query row: nothing to write
  if (!a.q || !a.ctx || !a.lse2 || (total_kv > 0 && (!a.k || !a.v)))
    return set_error(MMFB_ERR_ARG, "attn_varlen_cross_fwd: null pointer");
  return a.head_dim == 64 ? attn_fwd_launch<64, true>(a, cu_q, total_q, cu_kv, total_kv, stream)
                          : attn_fwd_launch<128, true>(a, cu_q, total_q, cu_kv, total_kv, stream);
}

int attn_varlen_cross_bwd(const mmfb_attn_args& a, const int32_t* cu_q, int total_q, const int32_t* cu_kv, int total_kv,
                          cudaStream_t stream) {
  int rc = check_varlen_cross(a, cu_q, total_q, cu_kv, total_kv, "attn_varlen_cross_bwd");
  if (rc) return rc;
  if (total_q == 0 && total_kv == 0) return MMFB_OK;
  if ((total_q > 0 && (!a.q || !a.ctx || !a.lse2 || !a.dctx || !a.delta || !a.dq)) ||
      (total_kv > 0 && (!a.k || !a.v || !a.dk || !a.dv)))
    return set_error(MMFB_ERR_ARG, "attn_varlen_cross_bwd: null pointer");
  return a.head_dim == 64 ? attn_bwd_launch<64, true>(a, cu_q, total_q, cu_kv, total_kv, stream)
                          : attn_bwd_launch<128, true>(a, cu_q, total_q, cu_kv, total_kv, stream);
}
#elif defined(MMFB_ATTN_CAUSAL_TU)

// Dense self-attention with a causal tail; attn_fwd / attn_bwd have checked the arguments (causal_len != 0 here).
int attn_causal_fwd(const mmfb_attn_args& a, cudaStream_t stream) {
  return a.head_dim == 64 ? attn_fwd_launch<64, false, true>(a, nullptr, 0, nullptr, 0, stream)
                          : attn_fwd_launch<128, false, true>(a, nullptr, 0, nullptr, 0, stream);
}

int attn_causal_bwd(const mmfb_attn_args& a, cudaStream_t stream) {
  return a.head_dim == 64 ? attn_bwd_launch<64, false, true>(a, nullptr, 0, nullptr, 0, stream)
                          : attn_bwd_launch<128, false, true>(a, nullptr, 0, nullptr, 0, stream);
}
#elif defined(MMFB_ATTN_VARLEN_CAUSAL_TU)

// Packed self-attention with a causal tail: the packed entry points' arguments, and 0 < causal_len <= max_len (the
// lengths are device data, so a sample shorter than the tail is all tail, see varlen_tail).
static int check_varlen_causal(const mmfb_attn_args& a, const int32_t* cu, int total, const char* who) {
  int rc = check_attn_common(a, who);     // also: Sq == Skv and causal_len <= Skv when causal_len > 0
  if (rc) return rc;
  if (a.causal_len <= 0)
    return set_error(MMFB_ERR_ARG, "%s: causal_len must be in [1, max_len=%d] (got %d)", who, a.Skv, a.causal_len);
  if (a.mask != nullptr) return set_error(MMFB_ERR_ARG, "%s: mask must be NULL (packing has removed the masked keys)", who);
  if (!cu) return set_error(MMFB_ERR_ARG, "%s: null cu_seqlens", who);
  if (total < 0) return set_error(MMFB_ERR_ARG, "%s: negative total (%d)", who, total);
  return MMFB_OK;
}

int attn_varlen_causal_fwd(const mmfb_attn_args& a, const int32_t* cu, int total, cudaStream_t stream) {
  int rc = check_varlen_causal(a, cu, total, "attn_varlen_causal_fwd");
  if (rc) return rc;
  if (total == 0) return MMFB_OK;
  if (!a.q || !a.k || !a.v || !a.ctx || !a.lse2) return set_error(MMFB_ERR_ARG, "attn_varlen_causal_fwd: null pointer");
  return a.head_dim == 64 ? attn_fwd_launch<64, true, true>(a, cu, total, cu, total, stream)
                          : attn_fwd_launch<128, true, true>(a, cu, total, cu, total, stream);
}

int attn_varlen_causal_bwd(const mmfb_attn_args& a, const int32_t* cu, int total, cudaStream_t stream) {
  int rc = check_varlen_causal(a, cu, total, "attn_varlen_causal_bwd");
  if (rc) return rc;
  if (total == 0) return MMFB_OK;
  if (!a.q || !a.k || !a.v || !a.ctx || !a.lse2 || !a.dctx || !a.delta || !a.dq || !a.dk || !a.dv)
    return set_error(MMFB_ERR_ARG, "attn_varlen_causal_bwd: null pointer");
  return a.head_dim == 64 ? attn_bwd_launch<64, true, true>(a, cu, total, cu, total, stream)
                          : attn_bwd_launch<128, true, true>(a, cu, total, cu, total, stream);
}
#endif  // MMFB_ATTN_VARLEN_TU / MMFB_ATTN_CAUSAL_TU / MMFB_ATTN_VARLEN_CAUSAL_TU

}  // namespace mmfb
