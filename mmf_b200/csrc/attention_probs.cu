// Attention probabilities of one dense attention call, written out for inspection (output_attentions, ViLBERT
// visualization):
//     P[b, h, q, k] = exp2(fma(S, scale2, staged_mask(mask[b, k])) - lse2[b, h, q])  (* keep(b, h, q, k) * drop_scale)
// with S = Q K^T of the call's q / k head slices and lse2 the row statistics its forward saved.  This is the dq kernel's
// probability recompute (attention.cu) with the store of P in place of the gradient products: the same tiles, the same
// staged mask (clamped at -10000, keys past Skv at -inf), the same keep bits, so P is the post-dropout probability the
// reference returns.  It reads Q and K only, and its cost is the HBM write of P, so its one product stays on mma.sync
// m16n8k16 with ldmatrix fragments (each warp its own 16 rows).
//
// Its own translation unit (it includes attention.cu for the shared helpers and instantiates none of its kernels), so that
// the existing attention kernels keep their code.
#define MMFB_ATTN_PROBS_TU
#include "attention.cu"

namespace mmfb {

constexpr int AP_PITCH = AT_ROWS + 4;   // fp32 pitch of a staged row: 272 B, 16-byte aligned, rows start 4 banks apart

// byte offset of the 16-byte chunk holding column c (a multiple of 8) of row r in a staged tile: 64-column panels of
// ROWS x 128 B, SWIZZLE_128B (chunk index XOR row % 8), as written by a TMA box {64, ROWS}
template <int ROWS>
__device__ __forceinline__ uint32_t tile_off(int r, int c) {
  return (c >> 6) * (ROWS * 128) + r * 128 + ((((c >> 3) & 7) ^ (r & 7)) << 4);
}

// acc[16 x 8 NT] (+)= A[16 rows from r0 of tile a, D] * B[8 NT rows of tile b, D]^T   (both tiles K-major along D)
template <int D, int NT, int AROWS, int BROWS>
__device__ __forceinline__ void mma_abt(float (&acc)[NT][4], uint32_t a, int r0, uint32_t b, int lane) {
  const int mi = lane >> 3, lr = lane & 7;
#pragma unroll
  for (int ks = 0; ks < D / 16; ++ks) {
    uint32_t af[4];
    ldsm_x4(af, a + tile_off<AROWS>(r0 + (mi & 1) * 8 + lr, ks * 16 + (mi >> 1) * 8));
#pragma unroll
    for (int np = 0; np < NT / 2; ++np) {
      uint32_t bf[4];
      ldsm_x4(bf, b + tile_off<BROWS>(np * 16 + (mi >> 1) * 8 + lr, ks * 16 + (mi & 1) * 8));
      mma_bf16_16816(acc[2 * np], af, bf[0], bf[1]);
      mma_bf16_16816(acc[2 * np + 1], af, bf[2], bf[3]);
    }
  }
}

struct AttnProbsDev {
  int B, H, Sq, Skv;
  const float* mask;      // [B, Skv] additive, or null
  const float* lse2;      // [B, H, Sq] from the forward that used the same q, k, mask and keep bits
  const uint32_t* dmask;  // keep bits [B, H, Sq, W] or null
  int W;
  float dscale;
  float scale2;           // log2(e)/sqrt(d), as in the forward
  void* out;              // [B, H, Sq, Skv] contiguous, float or bf16
  int vec;                // rows can be stored as 16-byte vectors (base aligned, Skv a multiple of 16 B / element size)
};

// grid (query tiles, heads, batch).  smem: Q tile, two stages of K blocks, the key mask (log2 domain), and a 64 x 64 fp32
// staging tile (each warp owns its 16 rows, so staging needs warp synchronisation only).  The staged block is stored row by
// row: with `vec` as 16-byte vectors (a warp writes 2 rows of fp32 / 4 rows of bf16 per instruction), else as scalars
// (128 B / 64 B per warp instruction).  Only elements with q < Sq and k < Skv are written.
template <int D, typename T>
__global__ void __launch_bounds__(AT_THREADS)
attn_probs_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, AttnProbsDev p) {
  constexpr int TB = D / 64 * AT_ROWS * 128;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sK = smem + TB;                     // stage s at sK + s TB
  float* sP = reinterpret_cast<float*>(sK + 2 * TB);        // [64][AP_PITCH]
  const int NKB = (p.Skv + AT_ROWS - 1) / AT_ROWS;
  float* sMask = sP + AT_ROWS * AP_PITCH;                   // [NKB * 64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sMask + NKB * AT_ROWS);   // [0] Q, [1..2] K stages

  griddep_launch();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_ROWS, h = blockIdx.y, b = blockIdx.z;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bars[0], TB);
    load_tile<D, AT_ROWS>(sQ, &tmQ, &bars[0], h * D, q0, b);
    for (int kb = 0; kb < 2 && kb < NKB; ++kb) {
      mbar_expect_tx(&bars[1 + kb], TB);
      load_tile<D, AT_ROWS>(sK + kb * TB, &tmK, &bars[1 + kb], h * D, kb * AT_ROWS, b);
    }
  }
  for (int i = threadIdx.x; i < NKB * AT_ROWS; i += AT_THREADS)
    sMask[i] = (i < p.Skv) ? (p.mask != nullptr ? staged_mask(p.mask[static_cast<int64_t>(b) * p.Skv + i]) : 0.0f) : -INFINITY;
  __syncthreads();

  const int g = lane >> 2, t4 = lane & 3;
  const int r0 = warp * 16;
  const int64_t bh = static_cast<int64_t>(b) * p.H + h;
  float lse[2];
  const uint32_t* dm[2] = {nullptr, nullptr};
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = q0 + r0 + g + hr * 8;
    const bool ok = q < p.Sq;
    lse[hr] = ok ? p.lse2[bh * p.Sq + q] : INFINITY;        // rows past Sq: P = 0, never stored
    if (p.dmask != nullptr && ok) dm[hr] = p.dmask + (bh * p.Sq + q) * p.W;
  }
  float* myP = sP + r0 * AP_PITCH;
  T* out = reinterpret_cast<T*>(p.out);
  mbar_wait(&bars[0], 0);
  const uint32_t uQ = smem_u32(sQ);

  for (int kb = 0; kb < NKB; ++kb) {
    const int st = kb & 1;
    mbar_wait(&bars[1 + st], (kb >> 1) & 1);
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.0f;
    mma_abt<D, 8, AT_ROWS, AT_ROWS>(s, uQ, r0, smem_u32(sK + st * TB), lane);
    // every warp is done with this K stage: order its ldmatrix reads before the refill (see the forward kernel)
    fence_proxy_async();
    __syncthreads();
    if (threadIdx.x == 0 && kb + 2 < NKB) {
      mbar_expect_tx(&bars[1 + st], TB);
      load_tile<D, AT_ROWS>(sK + st * TB, &tmK, &bars[1 + st], h * D, (kb + 2) * AT_ROWS, b);
    }
    uint32_t bits[2][2] = {{0xFFFFFFFFu, 0xFFFFFFFFu}, {0xFFFFFFFFu, 0xFFFFFFFFu}};
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      if (dm[hr] != nullptr) {
        bits[hr][0] = __ldg(dm[hr] + kb * 2);
        if (kb * 2 + 1 < p.W) bits[hr][1] = __ldg(dm[hr] + kb * 2 + 1);
      }
    }
    __syncwarp();                              // the previous block's rows of this warp have been stored
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float2 mk = *reinterpret_cast<const float2*>(sMask + kb * AT_ROWS + nt * 8 + 2 * t4);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float v[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int e = hr * 2 + j;
          const float pe = ex2_approx(fmaf(s[nt][e], p.scale2, j ? mk.y : mk.x) - lse[hr]);
          const int col = nt * 8 + 2 * t4 + j;
          v[j] = dm[hr] == nullptr ? pe : (((bits[hr][col >> 5] >> (col & 31)) & 1u) ? pe * p.dscale : 0.0f);
        }
        *reinterpret_cast<float2*>(myP + (g + hr * 8) * AP_PITCH + nt * 8 + 2 * t4) = make_float2(v[0], v[1]);
      }
    }
    __syncwarp();
    const int k0 = kb * AT_ROWS;
    if (p.vec) {
      constexpr int EPV = 16 / sizeof(T);      // elements per 16-byte vector: 4 fp32 / 8 bf16
      constexpr int LPR = AT_ROWS / EPV;       // lanes per row
#pragma unroll
      for (int it = 0; it < 16 * LPR / 32; ++it) {
        const int rl = it * (32 / LPR) + lane / LPR, c = (lane % LPR) * EPV;
        const int q = q0 + r0 + rl;
        if (q >= p.Sq || k0 + c >= p.Skv) continue;   // Skv is a multiple of EPV: a vector is wholly in or out
        const float* src = myP + rl * AP_PITCH + c;
        T* dst = out + (bh * p.Sq + q) * p.Skv + k0 + c;
        if constexpr (sizeof(T) == 4) {
          __stcs(reinterpret_cast<float4*>(dst), *reinterpret_cast<const float4*>(src));
        } else {
          const float4 a = *reinterpret_cast<const float4*>(src), z = *reinterpret_cast<const float4*>(src + 4);
          __stcs(reinterpret_cast<uint4*>(dst), make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w),
                                                           pack_bf16x2(z.x, z.y), pack_bf16x2(z.z, z.w)));
        }
      }
    } else {
      for (int rl = 0; rl < 16; ++rl) {
        const int q = q0 + r0 + rl;
        if (q >= p.Sq) break;
        T* dst = out + (bh * p.Sq + q) * p.Skv + k0;
#pragma unroll
        for (int c = lane; c < AT_ROWS; c += 32) {
          if (k0 + c >= p.Skv) break;
          const float v = myP[rl * AP_PITCH + c];
          if constexpr (sizeof(T) == 4)
            dst[c] = v;
          else
            dst[c] = __float2bfloat16_rn(v);
        }
      }
    }
  }
}

template <int D, typename T>
static int attn_probs_launch(const mmfb_attn_args& a, void* probs, cudaStream_t stream) {
  const int W = a.heads * D;
  CUtensorMap tmQ, tmK;
  int rc;
  if ((rc = head_map(&tmQ, a.q, W, a.ldq, a.Sq, a.B, AT_ROWS))) return rc;
  if ((rc = head_map(&tmK, a.k, W, a.ldk, a.Skv, a.B, AT_ROWS))) return rc;
  const int TB = (D / 64) * AT_ROWS * 128;
  const int NKB = (a.Skv + AT_ROWS - 1) / AT_ROWS;
  const int smem = 3 * TB + AT_ROWS * AP_PITCH * 4 + NKB * AT_ROWS * 4 + 64 + 1024;
  AttnProbsDev p;
  p.B = a.B; p.H = a.heads; p.Sq = a.Sq; p.Skv = a.Skv;
  p.mask = a.mask;
  p.lse2 = a.lse2;
  p.dmask = a.drop_mask; p.W = (a.Skv + 31) / 32; p.dscale = a.drop_mask ? a.drop_scale : 1.0f;
  p.scale2 = LOG2E / sqrtf(static_cast<float>(D));
  p.out = probs;
  p.vec = (reinterpret_cast<uintptr_t>(probs) % 16 == 0) && ((a.Skv * sizeof(T)) % 16 == 0);
  auto kern = attn_probs_kernel<D, T>;
  static int smem_set = 0;
  if (smem > smem_set) {
    if ((rc = set_smem(reinterpret_cast<const void*>(kern), smem, "attn_probs"))) return rc;
    smem_set = smem;
  }
  MMFB_LAUNCH(kern, dim3((a.Sq + AT_ROWS - 1) / AT_ROWS, a.heads, a.B), AT_THREADS, smem, stream, tmQ, tmK, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "attn_probs launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

int attn_probs(const mmfb_attn_args& a, void* probs, int probs_dtype, cudaStream_t stream) {
  int rc = check_attn_common(a, "attn_probs");
  if (rc) return rc;
  if ((rc = check_no_causal(a, "attn_probs"))) return rc;
  if (probs_dtype != MMFB_PROBS_F32 && probs_dtype != MMFB_PROBS_BF16)
    return set_error(MMFB_ERR_ARG, "attn_probs: probs_dtype must be MMFB_PROBS_F32 or MMFB_PROBS_BF16 (got %d)", probs_dtype);
  if (!a.q || !a.k || !a.lse2 || !probs) return set_error(MMFB_ERR_ARG, "attn_probs: null pointer");
  const uintptr_t esize = probs_dtype == MMFB_PROBS_F32 ? 4 : 2;
  if (reinterpret_cast<uintptr_t>(probs) % esize)
    return set_error(MMFB_ERR_ARG, "attn_probs: probs must be aligned to its element size");
  if (probs_dtype == MMFB_PROBS_F32)
    return a.head_dim == 64 ? attn_probs_launch<64, float>(a, probs, stream) : attn_probs_launch<128, float>(a, probs, stream);
  return a.head_dim == 64 ? attn_probs_launch<64, bf16>(a, probs, stream) : attn_probs_launch<128, bf16>(a, probs, stream);
}

}  // namespace mmfb
