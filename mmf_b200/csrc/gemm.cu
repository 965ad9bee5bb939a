// wgmma GEMM family for the fusion block (sm_90a).
//
//   C[M,N] = epilogue( A[M,K] * B[N,K]^T )       bf16 operands, fp32 accumulation in registers
//
// Persistent: min(work units, SMs) CTAs, a work unit being one (128 x BN output tile, K split) pair; CTA b runs units
// b, b + gridDim.x, ...  384 threads = three warpgroups:
//   warpgroup 0    : TMA producer (one thread) - fills a STAGES-deep smem ring of 128x64 A tiles and BNx64 B tiles
//                    (SWIZZLE_128B), signalling `full[s]` with complete_tx bytes; it runs ahead into the next unit
//                    while the consumers run the current unit's epilogue
//   warpgroups 1,2 : consumers - each owns 64 rows of the tile and issues wgmma m64nBNk16 straight from the smem
//                    ring (one k-block in flight while the previous one retires and its slot is released through
//                    `empty[s]`), then runs the fused elementwise epilogue from its accumulator registers into smem
//                    staging boxes that one thread writes out with TMA bulk tensor stores (or fp32 vector reductions
//                    for the split-K weight-gradient GEMM).  That thread also fills the boxes with the epilogue's aux
//                    operand by TMA loads, issued while the unit's wgmmas run.
//
// Operand layouts: each of A and B may be K-major (row-major [rows, K]) or MN-major (row-major
// [K, rows]); the latter is what the backward pass needs (dgrad reads W[out,in] as B[N=in,K=out],
// wgrad reads dY[tokens,out] as A[M=out,K=tokens] and X[tokens,in] as B[N=in,K=tokens]) without
// ever materialising a transpose in HBM: wgmma reads MN-major bf16 tiles directly (transpose bits).
//
// Reference ops this replaces (mmf): the nn.Linear calls in mmf/modules/hf_layers.py:169-180 (Q,K,V),
// HF BertSelfOutput/BertIntermediate/BertOutput invoked at hf_layers.py:248,289-290,
// mmf/models/vilbert.py:77-79,127,144-145,396-412,504-509 and their autograd backward
// (mmf/trainers/core/training_loop.py:211-213).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "mmfb_internal.h"

namespace mmfb {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int NUM_THREADS = 384;

struct GemmDev {
  int M, N, K;
  int splits;
  bf16* c;               // bf16 destination [M, ldc]
  bf16* c2;              // second bf16 destination (EPI_BIAS_GELU)
  float* c32;            // EPI_ATOMIC_F32 destination; EPI_PARTIAL_F32: the workspace [splits, M, N]
  int64_t ldc;
  const bf16* bias;      // [N] or null
  const bf16* aux;       // residual / pre-activation, [M, ldaux], or null; read through the aux tensor map
  const uint32_t* dmask; // dropout keep-bits, [M, ldmask] words (bit n%32 of word n/32), or null
  int64_t ldmask;
  float dscale;          // 1/(1-p)
  const int32_t* m_dev;  // BOUNDED: device row bound (tiles starting at or past min(M, *m_dev) are skipped), or null
  const int32_t* k_dev;  // BOUNDED: device bound on K (only the k-blocks below min(K, *k_dev) are summed), or null
};

// epilogues that read a per-element bf16 operand (aux): it is loaded by TMA into the output staging boxes
__host__ __device__ constexpr bool epi_reads_aux(int epi) {
  return epi == EPI_BIAS_DROP_RESID || epi == EPI_GELU_BWD || epi == EPI_ADD_AUX;
}
// epilogues that write fp32 pairs straight from the accumulators (split-K weight gradient)
__host__ __device__ constexpr bool epi_f32(int epi) { return epi == EPI_ATOMIC_F32 || epi == EPI_PARTIAL_F32; }

template <int BN>
struct Cfg {
  // 192 KB of operand ring either way: 6 stages of 32 KB (BN = 128) or 4 stages of 48 KB (BN = 256)
  static constexpr int STAGES = (BN == 256) ? 4 : 6;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // epilogue staging, separate from the ring: per consumer warpgroup STG_BOXES buffers of one 64 x 64 bf16 TMA store
  // box (8 KB, SWIZZLE_128B), used round-robin.  Two boxes (not four on a 3-stage ring) measured faster for the aux
  // epilogues too, where they hold the aux boxes of the first two chunks, loaded during the K loop.
  static constexpr int BOX_BYTES = 64 * 64 * 2;
  static constexpr int STG_BOXES = 2;
  static constexpr int STG_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = STG_OFFSET + 2 * STG_BOXES * BOX_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFFSET + 256 + 1024;
  static_assert(STG_BOXES >= 2, "the store of one box must be able to overlap the writes of the next");
  static_assert((2 * STAGES + 2 * STG_BOXES) * 8 <= 256, "ring and aux mbarriers fit the barrier area");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget of one CTA per SM");
};

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BN == 256) wgmma_n256<TA, TB>(acc, da, db, accumulate);
  else wgmma_n128<TA, TB>(acc, da, db, accumulate);
}

// Work unit u = (tile, split), in (m, n, split) order: the CTAs running at one time share A row-blocks in L2.
struct Unit {
  int m0, n0, kb0, kb1;
};
template <int BN>
__device__ __forceinline__ Unit decode_unit(int u, const GemmDev& p, int tiles_n, int kb_total, int kb_per_split) {
  const int split = u % p.splits;
  const int t = u / p.splits;
  Unit w;
  w.m0 = (t / tiles_n) * BM;
  w.n0 = (t % tiles_n) * BN;
  w.kb0 = split * kb_per_split;
  w.kb1 = min(kb_total, w.kb0 + kb_per_split);
  return w;
}

// BOUNDED: the extents come from device memory (GemmDev::m_dev / k_dev), read after griddep_wait - the masked-LM head's
// vocabulary GEMMs run on a fixed capacity of rows of which only a device-counted prefix is labelled (DESIGN.md 4.1).
template <int BN, bool A_MN, bool B_MN, int EPI, bool BOUNDED = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmC2,
            const __grid_constant__ CUtensorMap tmX, GemmDev p) {
  using C = Cfg<BN>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::BAR_OFFSET);
  uint64_t* full = bars;                  // [STAGES]
  uint64_t* empty = bars + STAGES;        // [STAGES]
  uint64_t* auxb = bars + 2 * STAGES;     // [2][STG_BOXES]: aux box loaded into staging buffer b of a warpgroup
  const bool has_aux = epi_reads_aux(EPI) && p.aux != nullptr;

  griddep_launch();
  const int wg = threadIdx.x >> 7;
  const int tiles_n = (p.N + BN - 1) / BN;
  int kb_total = (p.K + BK - 1) / BK;
  int kb_per_split = (kb_total + p.splits - 1) / p.splits;
  int units = ((p.M + BM - 1) / BM) * tiles_n * p.splits;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (!epi_f32(EPI)) tma_prefetch_desc(&tmC);
    if (EPI == EPI_BIAS_GELU) tma_prefetch_desc(&tmC2);
    if (has_aux) tma_prefetch_desc(&tmX);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 256);          // every consumer thread releases the slot after its wgmma retired
    }
    if (epi_reads_aux(EPI))
      for (int b = 0; b < 2 * C::STG_BOXES; ++b) mbar_init(&auxb[b], 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();        // operands / aux / bias of this GEMM may come from the kernel that is still finishing
  if constexpr (BOUNDED) {
    // row tiles at or past the bound are not units at all (m is the outermost unit index); the k-blocks below the K bound
    // are shared among the launched splits as an unbounded call with K = bound would share them, and a unit left
    // without one adds nothing (EPI_ATOMIC_F32) or stores a zero partial (EPI_PARTIAL_F32, so the reduce is unchanged)
    if (p.m_dev != nullptr) units = ((min(p.M, max(*p.m_dev, 0)) + BM - 1) / BM) * tiles_n * p.splits;
    if (p.k_dev != nullptr) {
      kb_total = (min(p.K, max(*p.k_dev, 0)) + BK - 1) / BK;
      kb_per_split = (kb_total + p.splits - 1) / p.splits;
    }
  }

  // The ring position (slot s, phase ph) runs on over all k-blocks of all units of this CTA, in the same order in the
  // producer and in both consumers, and is never reset between units: the producer fills the next unit's first slots
  // while the consumers run the current unit's epilogue.
  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const Unit w = decode_unit<BN>(u, p, tiles_n, kb_total, kb_per_split);
        for (int kb = w.kb0; kb < w.kb1; ++kb) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* sa = smem + s * C::STAGE_BYTES;
          uint8_t* sb = sa + C::A_BYTES;
          mbar_expect_tx(&full[s], C::STAGE_BYTES);
          if (!A_MN) {
            tma_load_2d(sa, &tmA, &full[s], kb * BK, w.m0);
          } else {
#pragma unroll
            for (int pnl = 0; pnl < BM / 64; ++pnl) tma_load_2d(sa + pnl * 8192, &tmA, &full[s], w.m0 + pnl * 64, kb * BK);
          }
          if (!B_MN) {
            tma_load_2d(sb, &tmB, &full[s], kb * BK, w.n0);
          } else {
#pragma unroll
            for (int pnl = 0; pnl < BN / 64; ++pnl) tma_load_2d(sb + pnl * 8192, &tmB, &full[s], w.n0 + pnl * 64, kb * BK);
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ------------------------------ consumers ------------------------------
  const int half = wg - 1;                       // rows [64 half, 64 half + 64) of the tile
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool issuer = (threadIdx.x & 127) == 0;  // issues this warpgroup's TMA stores
  uint8_t* stg = smem + C::STG_OFFSET + half * C::STG_BOXES * C::BOX_BYTES;
  int s = 0;
  uint32_t ph = 0;
  uint32_t box = 0;                              // staging boxes this warpgroup has stored so far (all units)
  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    const Unit w = decode_unit<BN>(u, p, tiles_n, kb_total, kb_per_split);
    // 64-column chunks of this warpgroup's rows that are not wholly clipped: a prefix of the unit's chunks
    const int nch = w.m0 + half * 64 < p.M ? min(BN / 64, (p.N - w.n0 + 63) / 64) : 0;
    // TMA load of chunk cb's aux box into the staging buffer of box `bi`, where the chunk's results will be written:
    // each thread finds its aux pair at the swizzled address it stores the result to.  Rows past M and columns past N
    // are zero-filled and their results clipped by the store.
    const auto load_aux = [&](int cb, uint32_t bi) {
      const uint32_t b = half * C::STG_BOXES + bi % C::STG_BOXES;
      mbar_expect_tx(&auxb[b], C::BOX_BYTES);
      tma_load_2d(stg + (bi % C::STG_BOXES) * C::BOX_BYTES, &tmX, &auxb[b], w.n0 + cb * 64, w.m0 + half * 64);
    };
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
    {
      int prev = -1;
      for (int kb = w.kb0; kb < w.kb1; ++kb) {
        mbar_wait(&full[s], ph);
        const uint32_t sa = smem_u32(smem + s * C::STAGE_BYTES) + half * 8192;   // K-major: 64 rows x 128 B; MN-major: panel
        const uint32_t sb = smem_u32(smem + s * C::STAGE_BYTES) + C::A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) {
          const uint64_t da = A_MN ? gmma_desc_sw128(sa + kk * 2048, 8192, 1024) : gmma_desc_sw128(sa + kk * 32, 16, 1024);
          const uint64_t db = B_MN ? gmma_desc_sw128(sb + kk * 2048, 8192, 1024) : gmma_desc_sw128(sb + kk * 32, 16, 1024);
          wgmma_tile<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (kb > w.kb0 || kk > 0) ? 1u : 0u);
        }
        wgmma_commit();
        if (has_aux && issuer && kb == w.kb0) {
          // while the first k-block's wgmmas run: once the previous unit's stores have read their boxes out, prefetch
          // the aux boxes of this unit's first STG_BOXES chunks, hidden behind the rest of the K loop
          tma_store_wait_read<0>();
          for (int cb = 0; cb < min(nch, C::STG_BOXES); ++cb) load_aux(cb, box + cb);
        }
        wgmma_wait<1>();                   // the previous k-block's wgmmas have retired: its slot may be refilled
        if (prev >= 0) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      if (!BOUNDED || prev >= 0) mbar_arrive(&empty[prev]);   // every unbounded unit owns at least one k-block
    }

    if (epi_f32(EPI)) {
      // ------------- split-K epilogue: fp32 vector reductions into C, or plain stores of the split's partial -------------
      if (BOUNDED && EPI == EPI_ATOMIC_F32 && w.kb0 >= w.kb1) continue;   // no k-block below the bound: nothing to add
      float* dst = p.c32;
      if (EPI == EPI_PARTIAL_F32) dst += static_cast<int64_t>(u % p.splits) * p.M * p.N;   // ldc = N
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        const int m = w.m0 + half * 64 + warp * 16 + (lane >> 2) + rh * 8;
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = w.n0 + j * 8 + (lane & 3) * 2;
          if (n >= p.N) continue;                // N % 8 == 0: n < N implies n + 1 < N
          if (EPI == EPI_ATOMIC_F32) {
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + static_cast<int64_t>(m) * p.ldc + n),
                         "f"(acc[j * 4 + rh * 2]), "f"(acc[j * 4 + rh * 2 + 1])
                         : "memory");
          } else {
            *reinterpret_cast<float2*>(dst + static_cast<int64_t>(m) * p.ldc + n) =
                make_float2(acc[j * 4 + rh * 2], acc[j * 4 + rh * 2 + 1]);
          }
        }
      }
      continue;
    }

    // ------------------ epilogue: registers -> smem staging -> TMA bulk tensor stores ------------------
    // One 64-column chunk of this warpgroup's 64 rows at a time (one box per output).  Rows past M and columns past N
    // are computed without reading mask / bias (aux reads there find TMA's zero fill) and clipped by the store's tensor
    // map.  With aux, each box's buffer already holds the chunk's aux box, which the results overwrite in place.
    // Box i goes to buffer i % STG_BOXES, which box i - STG_BOXES used last: before the barrier of box i - 1 the issuer
    // waited until that store had read its source out.  C's box of a chunk is written as it is computed; C2's values
    // (EPI_BIAS_GELU) wait in registers until C's box has been handed to the TMA unit.
    const auto store_box = [&](const CUtensorMap* tm, uint8_t* bx, int c0, int c1) {
      fence_proxy_async();
      if (issuer) tma_store_wait_read<C::STG_BOXES - 2>();   // frees the buffer of the box after this one
      named_bar_sync(1 + half, 128);
      if (issuer) {
        tma_store_2d(tm, bx, c0, c1);
        tma_store_commit();
      }
      ++box;
    };
    // SWIZZLE_128B: 16-byte chunk jj of row r sits at chunk jj ^ (r % 8); the 32 lanes of a warp hit 32 banks
    const uint32_t st_row0 = (warp * 16 + (lane >> 2)) * 128 + (lane & 3) * 4;
    // Epilogues that read aux / mask store with a plain C++ store, which the compiler may move below the loads of later
    // pairs so that their latencies overlap.  EPI_BIAS_GELU reads no per-element operand; there the ordered asm store
    // keeps the compiler from holding many u and gelu(u) values at once (it would spill).
    const auto pair_at = [&](uint8_t* bx, int rh, int jj) {
      return reinterpret_cast<uint32_t*>(bx + st_row0 + rh * 8 * 128 + ((jj ^ (lane >> 2)) << 4));
    };
    const auto st_pair = [&](uint8_t* bx, int rh, int jj, uint32_t v) {
      uint32_t* dst = pair_at(bx, rh, jj);
      if (EPI == EPI_BIAS_GELU) asm volatile("st.shared.b32 [%0], %1;" ::"r"(smem_u32(dst)), "r"(v) : "memory");
      else *dst = v;
    };
#pragma unroll
    for (int cb = 0; cb < BN / 64; ++cb) {
      if (cb >= nch) continue;                   // the whole box is clipped (warpgroup-uniform)
      uint8_t* bx = stg + (box % C::STG_BOXES) * C::BOX_BYTES;
      if constexpr (C::STG_BOXES < BN / 64) {
        // chunks past the prefetched ones: chunk cb + STG_BOXES - 1 takes the buffer of chunk cb - 1, whose store the
        // issuer waits to have read out; its aux load then runs while this chunk is computed
        if (has_aux && issuer && cb >= 1 && cb + C::STG_BOXES - 1 < nch) {
          tma_store_wait_read<0>();
          load_aux(cb + C::STG_BOXES - 1, box + C::STG_BOXES - 1);
        }
      }
      // every box of a kernel with aux has had exactly one aux load: box / STG_BOXES loads used this buffer before
      if (has_aux) mbar_wait(&auxb[half * C::STG_BOXES + box % C::STG_BOXES], (box / C::STG_BOXES) & 1);
      uint32_t h[2][8];                          // gelu(u) of EPI_BIAS_GELU
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        const int m = w.m0 + half * 64 + warp * 16 + (lane >> 2) + rh * 8;
        const bool row_in = m < p.M;
        const uint32_t* mrow = (EPI == EPI_BIAS_DROP_RESID && p.dmask != nullptr && row_in)
                                   ? p.dmask + static_cast<int64_t>(m) * p.ldmask
                                   : nullptr;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = cb * 8 + jj;
          const int n = w.n0 + j * 8 + (lane & 3) * 2;
          float v0 = acc[j * 4 + rh * 2], v1 = acc[j * 4 + rh * 2 + 1];
          if (EPI == EPI_BIAS || EPI == EPI_BIAS_GELU || EPI == EPI_BIAS_DROP_RESID || EPI == EPI_BIAS_RELU) {
            if (p.bias != nullptr && n < p.N) {
              const float2 b = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + n)));
              v0 += b.x;
              v1 += b.y;
            }
          }
          if (EPI == EPI_BIAS_RELU) {
            v0 = fmaxf(v0, 0.0f);
            v1 = fmaxf(v1, 0.0f);
          }
          if (EPI == EPI_BIAS_DROP_RESID && mrow != nullptr && n < p.N) {
            const uint32_t bits = __ldg(mrow + (n >> 5)) >> (n & 31);
            v0 = (bits & 1u) ? v0 * p.dscale : 0.0f;
            v1 = (bits & 2u) ? v1 * p.dscale : 0.0f;
          }
          if (has_aux) {
            const float2 x = unpack_bf16x2(*pair_at(bx, rh, jj));
            if (EPI == EPI_GELU_BWD) {
              v0 *= gelu_erf_grad(x.x);
              v1 *= gelu_erf_grad(x.y);
            } else {
              v0 += x.x;
              v1 += x.y;
            }
          }
          st_pair(bx, rh, jj, pack_bf16x2(v0, v1));
          if (EPI == EPI_BIAS_GELU) h[rh][jj] = pack_bf16x2(gelu_erf(v0), gelu_erf(v1));
        }
      }
      store_box(&tmC, bx, w.n0 + cb * 64, w.m0 + half * 64);
      if (EPI == EPI_BIAS_GELU) {
        bx = stg + (box % C::STG_BOXES) * C::BOX_BYTES;
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) st_pair(bx, rh, jj, h[rh][jj]);
        store_box(&tmC2, bx, w.n0 + cb * 64, w.m0 + half * 64);
      }
    }
  }
  if (!epi_f32(EPI) && issuer) tma_store_wait_all();   // the staging smem must outlive the reads of the stores
}

// Second kernel of the ordered split-K GEMM:  C = ((C + P_0) + P_1) + ... + P_{S-1}  for the partials P_s = ws[s] [M, N].
// Four consecutive columns per thread (N % 8 == 0: they lie in one row).
// BOUNDED (a device row bound m_dev on the GEMM): the partial kernel stored no partial for the row tiles at or past
// min(M, *m_dev) rounded up to BM, so those rows of C are neither read nor written here either.
template <bool BOUNDED = false>
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ ws, int S, int M, int N, float* __restrict__ c, int64_t ldc,
                     const int32_t* __restrict__ m_dev = nullptr) {
  griddep_launch();
  griddep_wait();
  const int64_t mn = static_cast<int64_t>(M) * N;
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x) * 4;
  if (i >= mn) return;
  if constexpr (BOUNDED) {
    if (m_dev != nullptr && i / N >= min(M, (max(*m_dev, 0) + BM - 1) / BM * BM)) return;
  }
  float2* dst = reinterpret_cast<float2*>(c + (i / N) * ldc + (i % N));
  const float2 c0 = dst[0], c1 = dst[1];
  float4 r = make_float4(c0.x, c0.y, c1.x, c1.y);
  for (int s = 0; s < S; ++s) {
    const float4 v = *reinterpret_cast<const float4*>(ws + s * mn + i);
    r.x += v.x; r.y += v.y; r.z += v.z; r.w += v.w;
  }
  dst[0] = make_float2(r.x, r.y);
  dst[1] = make_float2(r.z, r.w);
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
int gemm_effective_splits(int K, int splits) {
  int s = splits > 0 ? splits : 1;
  const int kb_total = (K + BK - 1) / BK;
  if (s > kb_total) s = kb_total;
  // every split must own at least one k-block
  while (s > 1 && ((kb_total + s - 1) / s) * (s - 1) >= kb_total) --s;
  return s;
}

int64_t gemm_workspace_bytes(int M, int N, int K, int splits) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  const int s = gemm_effective_splits(K, splits);
  return s > 1 ? static_cast<int64_t>(s) * M * N * 4 : 0;
}

template <int BN, bool A_MN, bool B_MN, int EPI, bool BOUNDED = false>
static int launch(const mmfb_gemm_args& a, cudaStream_t stream, const int32_t* m_dev = nullptr,
                  const int32_t* k_dev = nullptr) {
  using C = Cfg<BN>;
  constexpr bool AUX = epi_reads_aux(EPI);
  CUtensorMap tmA, tmB;
  // operand maps: K-major -> tensor [rows, K] (inner = K), box {64, rows_per_tile}
  //               MN-major -> tensor [K, rows] (inner = rows), box {64, 64}
  int rc;
  if (!A_MN) rc = make_tmap_2d(&tmA, a.A, a.K, a.M, a.lda, 64, BM);
  else rc = make_tmap_2d(&tmA, a.A, a.M, a.K, a.lda, 64, 64);
  if (rc) return rc;
  if (!B_MN) rc = make_tmap_2d(&tmB, a.B, a.K, a.N, a.ldb, 64, BN);
  else rc = make_tmap_2d(&tmB, a.B, a.N, a.K, a.ldb, 64, 64);
  if (rc) return rc;
  if (EPI == EPI_BIAS_GELU && a.C2 == nullptr) return set_error(MMFB_ERR_ARG, "gemm: this epilogue needs the C2 output");
  if (((reinterpret_cast<uintptr_t>(a.C) | reinterpret_cast<uintptr_t>(a.C2) | reinterpret_cast<uintptr_t>(a.bias) |
        reinterpret_cast<uintptr_t>(a.aux)) & 3) ||
      (a.aux != nullptr && (a.ldaux % 2)))
    return set_error(MMFB_ERR_ARG, "gemm: C / C2 / bias / aux must be 4-byte aligned");
  // the epilogues that read aux load it by TMA in 64 x 64 boxes, like C's stores
  if (AUX && a.aux != nullptr && ((reinterpret_cast<uintptr_t>(a.aux) & 15) || (a.ldaux % 8)))
    return set_error(MMFB_ERR_ARG, "gemm: aux must be 16-byte aligned with ldaux a multiple of 8 (aux=%p ldaux=%lld)",
                     a.aux, (long long)a.ldaux);
  // bf16 outputs are written by TMA stores of 64 x 64 boxes: tensor [M, N] with row pitch ldc (C and C2 need 16-byte
  // alignment, which make_tmap_2d checks); columns past N and rows past M are not written
  CUtensorMap tmC, tmC2, tmX;
  memset(&tmC, 0, sizeof(tmC));
  memset(&tmC2, 0, sizeof(tmC2));
  memset(&tmX, 0, sizeof(tmX));
  if (!epi_f32(EPI) && (rc = make_tmap_2d(&tmC, a.C, a.N, a.M, a.ldc, 64, 64))) return rc;
  if (EPI == EPI_BIAS_GELU && (rc = make_tmap_2d(&tmC2, a.C2, a.N, a.M, a.ldc, 64, 64))) return rc;
  if (AUX && a.aux != nullptr && (rc = make_tmap_2d(&tmX, a.aux, a.N, a.M, a.ldaux, 64, 64))) return rc;
  GemmDev p;
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.splits = epi_f32(EPI) ? gemm_effective_splits(a.K, a.splits) : 1;
  p.c = reinterpret_cast<bf16*>(a.C);
  p.c2 = reinterpret_cast<bf16*>(a.C2);
  p.c32 = reinterpret_cast<float*>(EPI == EPI_PARTIAL_F32 ? a.workspace : a.C);
  p.ldc = EPI == EPI_PARTIAL_F32 ? a.N : a.ldc;
  p.bias = reinterpret_cast<const bf16*>(a.bias);
  p.aux = reinterpret_cast<const bf16*>(a.aux);
  p.dmask = a.drop_mask;
  p.ldmask = a.ldmask;
  p.dscale = a.drop_scale;
  p.m_dev = BOUNDED ? m_dev : nullptr;
  p.k_dev = BOUNDED ? k_dev : nullptr;

  auto kern = gemm_kernel<BN, A_MN, B_MN, EPI, BOUNDED>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "cudaFuncSetAttribute(gemm): %s", cudaGetErrorString(e));
    attr_set = true;
  }
  // persistent: at most one CTA per SM, each striding over the (tile, split) work units
  const int units = ((a.M + BM - 1) / BM) * ((a.N + BN - 1) / BN) * p.splits;
  MMFB_LAUNCH(kern, units < num_sms() ? units : num_sms(), NUM_THREADS, C::SMEM_BYTES, stream, tmA, tmB, tmC, tmC2, tmX,
              p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "gemm launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

template <int BN>
static int dispatch(const mmfb_gemm_args& a, cudaStream_t s) {
  const int key = (a.a_mn ? 100 : 0) + (a.b_mn ? 10 : 0) + a.epi;
  switch (key) {
    case 0 + EPI_BIAS: return launch<BN, false, false, EPI_BIAS>(a, s);
    case 0 + EPI_BIAS_GELU: return launch<BN, false, false, EPI_BIAS_GELU>(a, s);
    case 0 + EPI_BIAS_DROP_RESID: return launch<BN, false, false, EPI_BIAS_DROP_RESID>(a, s);
    case 0 + EPI_BIAS_RELU: return launch<BN, false, false, EPI_BIAS_RELU>(a, s);
    case 10 + EPI_BIAS: return launch<BN, false, true, EPI_BIAS>(a, s);
    case 10 + EPI_GELU_BWD: return launch<BN, false, true, EPI_GELU_BWD>(a, s);
    case 10 + EPI_ADD_AUX: return launch<BN, false, true, EPI_ADD_AUX>(a, s);
    case 110 + EPI_ATOMIC_F32: return launch<BN, true, true, EPI_ATOMIC_F32>(a, s);
    // test-only layout combinations (kept small: plain store epilogue)
    case 100 + EPI_BIAS: return launch<BN, true, false, EPI_BIAS>(a, s);
    case 110 + EPI_BIAS: return launch<BN, true, true, EPI_BIAS>(a, s);
    default:
      return set_error(MMFB_ERR_ARG, "gemm: unsupported (a_mn=%d, b_mn=%d, epi=%d)", a.a_mn, a.b_mn, a.epi);
  }
}

// The device-bounded instantiations (m_dev / k_dev set): the masked-LM head's vocabulary GEMM, its dgrad and its wgrad,
// and the encoder layer's GEMMs on a fixed capacity of packed rows (QKV / O-proj / FFN-up / FFN-down and their dgrads).
// A row tile at or past the rounded bound is no unit, so nothing of it is loaded (A, the aux box) or stored (C, C2).
template <int BN>
static int dispatch_bounded(const mmfb_gemm_args& a, cudaStream_t s, const int32_t* m_dev, const int32_t* k_dev) {
  const int key = (a.a_mn ? 100 : 0) + (a.b_mn ? 10 : 0) + a.epi;
  switch (key) {
    case 0 + EPI_BIAS: return launch<BN, false, false, EPI_BIAS, true>(a, s, m_dev, k_dev);
    case 0 + EPI_BIAS_GELU: return launch<BN, false, false, EPI_BIAS_GELU, true>(a, s, m_dev, k_dev);
    case 0 + EPI_BIAS_DROP_RESID: return launch<BN, false, false, EPI_BIAS_DROP_RESID, true>(a, s, m_dev, k_dev);
    case 10 + EPI_BIAS: return launch<BN, false, true, EPI_BIAS, true>(a, s, m_dev, k_dev);
    case 10 + EPI_GELU_BWD: return launch<BN, false, true, EPI_GELU_BWD, true>(a, s, m_dev, k_dev);
    case 10 + EPI_ADD_AUX: return launch<BN, false, true, EPI_ADD_AUX, true>(a, s, m_dev, k_dev);
    case 110 + EPI_ATOMIC_F32: return launch<BN, true, true, EPI_ATOMIC_F32, true>(a, s, m_dev, k_dev);
    default:
      return set_error(MMFB_ERR_ARG, "gemm: a device bound (m_dev / k_dev) is not supported for (a_mn=%d, b_mn=%d, epi=%d)",
                       a.a_mn, a.b_mn, a.epi);
  }
}

// Ordered split-K: every (tile, split) unit stores its partial into the workspace, then one more kernel adds the
// partials into C in split order.  No unit waits for another, so this is safe whatever number of CTAs is resident.
// BOUNDED: units without a k-block below the K bound store zero partials, so the reduce adds the same partials as an
// unbounded call with K = bound, then zeros; with an M bound the reduce skips the rows whose tiles stored no partial.
template <int BN, bool BOUNDED>
static int gemm_ordered(const mmfb_gemm_args& a, int splits, cudaStream_t stream, const int32_t* m_dev,
                        const int32_t* k_dev) {
  int rc = launch<BN, true, true, EPI_PARTIAL_F32, BOUNDED>(a, stream, m_dev, k_dev);
  if (rc) return rc;
  const int64_t quads = static_cast<int64_t>(a.M) * a.N / 4;
  MMFB_LAUNCH(splitk_reduce_kernel<BOUNDED>, static_cast<unsigned>((quads + 255) / 256), 256, 0, stream,
              reinterpret_cast<const float*>(a.workspace), splits, a.M, a.N, reinterpret_cast<float*>(a.C), a.ldc,
              BOUNDED ? m_dev : nullptr);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "gemm split-K reduce launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

int gemm(const mmfb_gemm_args& a, cudaStream_t stream, const int32_t* m_dev, const int32_t* k_dev) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return set_error(MMFB_ERR_ARG, "gemm: empty problem %dx%dx%d", a.M, a.N, a.K);
  // only CONTIGUOUS extents need 16-byte granularity (TMA row pitch / vector epilogue); K of an MN-major operand
  // (= the token count in the weight-gradient GEMM) is a row count and may be anything
  if (a.N % 8) return set_error(MMFB_ERR_ARG, "gemm: N must be a multiple of 8 (got %d)", a.N);
  if ((!a.a_mn || !a.b_mn) && (a.K % 8))
    return set_error(MMFB_ERR_ARG, "gemm: K must be a multiple of 8 for K-major operands (got %d)", a.K);
  if (a.a_mn && (a.M % 8)) return set_error(MMFB_ERR_ARG, "gemm: M must be a multiple of 8 for MN-major A (got %d)", a.M);
  if ((a.lda % 8) || (a.ldb % 8) || (a.epi != EPI_ATOMIC_F32 && (a.ldc % 8)))
    return set_error(MMFB_ERR_ARG, "gemm: leading dimensions must be multiples of 8 elements");
  const int bn = a.block_n > 0 ? a.block_n : (a.N >= 256 ? 256 : 128);
  const bool ordered = a.epi == EPI_ATOMIC_F32 && (a.workspace != nullptr || a.workspace_bytes != 0);
  const bool bounded = m_dev != nullptr || k_dev != nullptr;
  if ((reinterpret_cast<uintptr_t>(m_dev) | reinterpret_cast<uintptr_t>(k_dev)) & 3)
    return set_error(MMFB_ERR_ARG, "gemm: m_dev / k_dev must be 4-byte aligned");
  const int splits = gemm_effective_splits(a.K, a.splits);
  if (ordered && splits > 1 && (bn == 128 || bn == 256) && a.a_mn && a.b_mn) {
    const int64_t need = gemm_workspace_bytes(a.M, a.N, a.K, a.splits);
    if (a.workspace == nullptr || a.workspace_bytes < need || (reinterpret_cast<uintptr_t>(a.workspace) & 15))
      return set_error(MMFB_ERR_ARG, "gemm: ordered split-K needs a 16-byte aligned workspace of %lld bytes (got %p, %lld)",
                       (long long)need, a.workspace, (long long)a.workspace_bytes);
    if ((reinterpret_cast<uintptr_t>(a.C) & 7) || (a.ldc % 2))
      return set_error(MMFB_ERR_ARG, "gemm: ordered split-K needs an 8-byte aligned C with an even ldc");
    if (bounded)
      return bn == 256 ? gemm_ordered<256, true>(a, splits, stream, m_dev, k_dev)
                       : gemm_ordered<128, true>(a, splits, stream, m_dev, k_dev);
    return bn == 256 ? gemm_ordered<256, false>(a, splits, stream, nullptr, nullptr)
                     : gemm_ordered<128, false>(a, splits, stream, nullptr, nullptr);
  }
  if (bounded) {
    if (bn == 256) return dispatch_bounded<256>(a, stream, m_dev, k_dev);
    if (bn == 128) return dispatch_bounded<128>(a, stream, m_dev, k_dev);
  }
  if (bn == 256) return dispatch<256>(a, stream);
  if (bn == 128) return dispatch<128>(a, stream);
  return set_error(MMFB_ERR_ARG, "gemm: block_n must be 128 or 256");
}

}  // namespace mmfb
