// Word-region alignment's optimal-transport distance (sm_90a): cosine cost, the IPOT plan and trace(C T) in ONE kernel
// per call, and the gradient through the cosine cost in a second one.
//
// The reference (mmf/modules/ot.py:15-102, called by mmf/models/transformers/heads/wra.py:74-76) builds the plan from
// 50 iterations of tiny batched torch ops on [B, regions, tokens] matrices - about ten launches per iteration.  The whole
// state of one sample (cost, kernel A = exp(-C^T/beta) and plan T, fp32, at most 128 x 128 each) fits the shared memory of
// one CTA, so here one CTA owns one sample from the dot products to the distance and nothing but the results reaches HBM.
//
//   forward, per sample:  S = x y^T on mma.sync (bf16 operands, fp32 accumulation) -> C = 1 - S / (|x| |y|), 0 on padded
//                         pairs -> A, T, sigma as ot.py:51-59 -> `iterations` x { Q = A*T; k x { delta; sigma };
//                         T = delta*Q*sigma } (ot.py:69-75) -> T zeroed on padded pairs -> dist = sum C[m,n] T[n,m].
//   backward:             the reference detaches T (ot.py:98-101), so d dist / d C = T^T and with x^ = x / max(|x|, eps)
//                           dx[m] = -g / |x_m| * (sum_n T[n,m] y^[n] - x^[m] * sum_n T[n,m] (1 - C[m,n]))
//                         (the second sum is x^[m] . d x^[m]; the forward saves it per row), dy likewise.
#include "common.cuh"
#include "mmfb_internal.h"

namespace mmfb {

namespace {

constexpr int OT_THREADS = 256;
constexpr int OT_MAX = 128;          // rows per side
constexpr int OT_KC = 64;            // hidden columns per staged chunk
constexpr int OT_LDS = OT_KC + 8;    // bf16 row pitch of a staged chunk: fragment loads hit 32 different banks
constexpr int OT_CHUNK = 256;        // samples per launch (their lengths travel as kernel parameters)
constexpr float OT_EPS = 1e-5f;      // F.normalize(eps=1e-5) of cost_matrix_cosine (ot.py:15-22)

struct OtLens {
  uint8_t x[OT_CHUNK];
  uint8_t y[OT_CHUNK];
};

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.0f;
#pragma unroll
  for (int w = 0; w < OT_THREADS / 32; ++w) r += red[w];
  return r;
}

// max(|row|, eps) of `rows` bf16 rows of H columns, one warp per row; rows at or past `len` get 1
__device__ __forceinline__ void row_norms(const bf16* __restrict__ p, int64_t ld, int rows, int len, int H, float* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < rows; r += OT_THREADS / 32) {
    float ss = 0.0f;
    if (r < len) {
      const uint4* v = reinterpret_cast<const uint4*>(p + r * ld);
      for (int i = lane; i < (H >> 3); i += 32) {
        const uint4 u = v[i];
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
        ss += a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y + c.x * c.x + c.y * c.y + d.x * d.x + d.y * d.y;
      }
    }
    ss = warp_sum(ss);
    if (lane == 0) out[r] = r < len ? fmaxf(sqrtf(ss), OT_EPS) : 1.0f;
  }
}

// columns [c0, c0 + 64) of `rows_pad` rows into shared memory (pitch OT_LDS); rows at or past `len` are zeros
__device__ __forceinline__ void stage_chunk(bf16* dst, const bf16* __restrict__ src, int64_t ld, int rows_pad, int len, int c0) {
  for (int i = threadIdx.x; i < rows_pad * (OT_KC / 8); i += OT_THREADS) {
    const int r = i >> 3, v = i & 7;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (r < len) u = *reinterpret_cast<const uint4*>(src + r * ld + c0 + v * 8);
    *reinterpret_cast<uint4*>(dst + r * OT_LDS + v * 8) = u;
  }
}

__global__ void __launch_bounds__(OT_THREADS)
ot_fwd_kernel(const bf16* __restrict__ x, int64_t ldx, int64_t bsx, const bf16* __restrict__ y, int64_t ldy, int64_t bsy,
              const OtLens lens, int b0, int M, int N, int H, float beta, int iterations, int k, float* __restrict__ dist,
              float* __restrict__ plan, float* __restrict__ cost, float* __restrict__ saved) {
  griddep_launch();
  griddep_wait();
  extern __shared__ __align__(16) uint8_t ot_smem[];
  const int b = b0 + blockIdx.x;
  const int xl = lens.x[blockIdx.x], yl = lens.y[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Mp = (M + 15) & ~15, Np = (N + 7) & ~7;

  float* Cs = reinterpret_cast<float*>(ot_smem);                 // [M][N]
  float* sig = Cs + ((M * N + 3) & ~3);                          // [128]
  float* del = sig + OT_MAX;                                     // [128]
  float* nx = del + OT_MAX;                                      // [128]
  float* ny = nx + OT_MAX;                                       // [128]
  float* red = ny + OT_MAX;                                      // [8]
  float* As = red + 8;                                           // [N][M], after the dot products
  float* Ts = As + M * N;                                        // [N][M]
  bf16* xs = reinterpret_cast<bf16*>(As);                        // staged chunks share the A / T space
  bf16* ys = xs + Mp * OT_LDS;

  x += b * bsx;
  y += b * bsy;
  row_norms(x, ldx, M, xl, H, nx);
  row_norms(y, ldy, N, yl, H, ny);

  // ---- S = x y^T: warp w owns rows [16 w, 16 w + 16), all Np columns (m16n8k16 tiles)
  float acc[OT_MAX / 8][4];
#pragma unroll
  for (int nt = 0; nt < OT_MAX / 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.0f;
  const int g = lane >> 2, t = lane & 3, r0 = warp * 16;
  for (int c0 = 0; c0 < H; c0 += OT_KC) {
    __syncthreads();
    stage_chunk(xs, x, ldx, Mp, xl, c0);
    stage_chunk(ys, y, ldy, Np, yl, c0);
    __syncthreads();
    if (r0 < Mp) {
#pragma unroll
      for (int kk = 0; kk < OT_KC; kk += 16) {
        uint32_t a[4];
        a[0] = *reinterpret_cast<const uint32_t*>(xs + (r0 + g) * OT_LDS + kk + 2 * t);
        a[1] = *reinterpret_cast<const uint32_t*>(xs + (r0 + g + 8) * OT_LDS + kk + 2 * t);
        a[2] = *reinterpret_cast<const uint32_t*>(xs + (r0 + g) * OT_LDS + kk + 8 + 2 * t);
        a[3] = *reinterpret_cast<const uint32_t*>(xs + (r0 + g + 8) * OT_LDS + kk + 8 + 2 * t);
#pragma unroll
        for (int nt = 0; nt < OT_MAX / 8; ++nt) {
          if (nt * 8 < Np) {
            const uint32_t b0r = *reinterpret_cast<const uint32_t*>(ys + (nt * 8 + g) * OT_LDS + kk + 2 * t);
            const uint32_t b1r = *reinterpret_cast<const uint32_t*>(ys + (nt * 8 + g) * OT_LDS + kk + 8 + 2 * t);
            mma_bf16_16816(acc[nt], a, b0r, b1r);
          }
        }
      }
    }
  }
  // ---- C = 1 - S / (|x| |y|), zero on padded pairs (ot.py:23-24, 92-93)
#pragma unroll
  for (int nt = 0; nt < OT_MAX / 8; ++nt) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int m = r0 + g + ((e >> 1) << 3), n = nt * 8 + 2 * t + (e & 1);
      if (m < M && n < N) Cs[m * N + n] = (m < xl && n < yl) ? 1.0f - acc[nt][e] / (nx[m] * ny[n]) : 0.0f;
    }
  }
  __syncthreads();            // every warp is done with the staged chunks: A and T may overwrite them

  // ---- sigma = 1 / x_len, T = 1, A = exp(-C^T / beta), all zero on padding (ot.py:51-59)
  for (int i = tid; i < N * M; i += OT_THREADS) {
    const int n = i / M, m = i - n * M;
    const bool valid = m < xl && n < yl;
    As[i] = valid ? expf(-Cs[m * N + n] / beta) : 0.0f;
    Ts[i] = valid ? 1.0f : 0.0f;
  }
  const float fxl = static_cast<float>(xl), fyl = static_cast<float>(yl);
  if (tid < OT_MAX) {
    sig[tid] = tid < xl ? 1.0f / fxl : 0.0f;
    del[tid] = 0.0f;
  }
  __syncthreads();

  // ---- IPOT (ot.py:69-75).  Ts holds T before the first iteration and Q = A * T afterwards; T = delta * Q * sigma of
  // iteration i is formed where iteration i + 1 (or the final pass) reads it.
  for (int it = 0; it < iterations; ++it) {
    for (int kk = 0; kk < k; ++kk) {
      // rows of Q, one warp per region n: delta[n] = 1 / (y_len * (Q sigma)[n] + 1e4 * y_pad[n])
      for (int n = warp; n < N; n += OT_THREADS / 32) {
        const float d_old = del[n];
        float s = 0.0f;
        for (int m = lane; m < M; m += 32) {
          float q = Ts[n * M + m];
          if (kk == 0) {
            if (it > 0) q = (d_old * q) * sig[m];
            q = As[n * M + m] * q;
            Ts[n * M + m] = q;
          }
          s += q * sig[m];
        }
        s = warp_sum(s);
        if (lane == 0) del[n] = 1.0f / (fyl * s + (n < yl ? 0.0f : 1e4f));
      }
      __syncthreads();
      // columns of Q, one thread per token m: sigma[m] = 1 / (x_len * (delta Q)[m] + 1e4 * x_pad[m])
      float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
      if (tid < M) {
        int n = 0;
        for (; n + 4 <= N; n += 4) {
          s0 += del[n] * Ts[n * M + tid];
          s1 += del[n + 1] * Ts[(n + 1) * M + tid];
          s2 += del[n + 2] * Ts[(n + 2) * M + tid];
          s3 += del[n + 3] * Ts[(n + 3) * M + tid];
        }
        for (; n < N; ++n) s0 += del[n] * Ts[n * M + tid];
      }
      if (tid < M) sig[tid] = 1.0f / (fxl * ((s0 + s1) + (s2 + s3)) + (tid < xl ? 0.0f : 1e4f));
      __syncthreads();
    }
  }

  // ---- T = delta * Q * sigma, zeroed on padded pairs (ot.py:75-76); dist = sum_{m,n} C[m,n] T[n,m] (trace, ot.py:101)
  float part = 0.0f;
  float* plan_b = plan + static_cast<int64_t>(b) * N * M;
  for (int i = tid; i < N * M; i += OT_THREADS) {
    const int n = i / M, m = i - n * M;
    float tv = (del[n] * Ts[i]) * sig[m];
    if (!(m < xl && n < yl)) tv = 0.0f;
    Ts[i] = tv;
    plan_b[i] = tv;
    part += Cs[m * N + n] * tv;
  }
  const float total = block_sum(part, red);      // its barriers also publish the final Ts
  if (tid == 0) dist[b] = total;
  if (cost != nullptr) {
    float* cost_b = cost + static_cast<int64_t>(b) * M * N;
    for (int i = tid; i < M * N; i += OT_THREADS) cost_b[i] = Cs[i];
  }
  // saved for the backward: |x| [M], |y| [N], then x^ . d x^ / (-g) [M] and y^ . d y^ / (-g) [N]
  float* sv = saved + static_cast<int64_t>(b) * 2 * (M + N);
  if (tid < M) {
    float s = 0.0f;
    for (int n = 0; n < N; ++n) s += Ts[n * M + tid] * (1.0f - Cs[tid * N + n]);
    sv[tid] = nx[tid];
    sv[M + N + tid] = s;
  }
  for (int n = warp; n < N; n += OT_THREADS / 32) {
    float s = 0.0f;
    for (int m = lane; m < M; m += 32) s += Ts[n * M + m] * (1.0f - Cs[m * N + n]);
    s = warp_sum(s);
    if (lane == 0) {
      sv[M + n] = ny[n];
      sv[2 * M + N + n] = s;
    }
  }
}

// One CTA per (sample, side).  Side 0 writes du = dx from v = y, side 1 writes du = dy from v = x:
//   du[i] = -g / |u_i| * (sum_j W[j][i] v^[j] - u^[i] * proj[i]),   W[j][i] = T[n][m] with (i, j) = (m, n) or (n, m);
// a row whose norm was clamped to eps has a constant denominator, so it gets no projection term.
__global__ void __launch_bounds__(OT_THREADS, 1)
ot_bwd_kernel(const bf16* __restrict__ x, int64_t ldx, int64_t bsx, const bf16* __restrict__ y, int64_t ldy, int64_t bsy,
              const OtLens lens, int b0, int M, int N, int H, const float* __restrict__ gout, const float* __restrict__ plan,
              const float* __restrict__ saved, bf16* __restrict__ dx, int64_t lddx, int64_t bsdx, bf16* __restrict__ dy,
              int64_t lddy, int64_t bsdy) {
  griddep_launch();
  griddep_wait();
  extern __shared__ __align__(16) uint8_t ot_smem[];
  const int b = b0 + blockIdx.x, side = blockIdx.y;
  const int tid = threadIdx.x;
  const int I = side == 0 ? M : N, J = side == 0 ? N : M;
  const int il = side == 0 ? lens.x[blockIdx.x] : lens.y[blockIdx.x];
  const int jl = side == 0 ? lens.y[blockIdx.x] : lens.x[blockIdx.x];
  const bf16* u = side == 0 ? x + b * bsx : y + b * bsy;
  const bf16* v = side == 0 ? y + b * bsy : x + b * bsx;
  const int64_t ldu = side == 0 ? ldx : ldy, ldv = side == 0 ? ldy : ldx;
  bf16* du = side == 0 ? dx + b * bsdx : dy + b * bsdy;
  const int64_t lddu = side == 0 ? lddx : lddy;
  const float* sv = saved + static_cast<int64_t>(b) * 2 * (M + N);
  const float* nu = side == 0 ? sv : sv + M;
  const float* nv = side == 0 ? sv + M : sv;
  const float* proj = side == 0 ? sv + M + N : sv + 2 * M + N;
  const float* plan_b = plan + static_cast<int64_t>(b) * N * M;
  const float gneg = -gout[b];

  const int Ip = (I + 3) & ~3;
  float* W = reinterpret_cast<float*>(ot_smem);     // [J][Ip], zero in the pad columns
  float* vs = W + J * Ip;                           // [J][64] fp32 v^ chunk
  for (int e = tid; e < J * Ip; e += OT_THREADS) {
    const int j = e / Ip, i = e - j * Ip;
    W[e] = i < I ? (side == 0 ? plan_b[j * M + i] : plan_b[i * M + j]) : 0.0f;
  }
  const int i0 = (tid >> 3) * 4, tc = tid & 7;      // 4 rows x (4 + 4) columns per thread
  for (int c0 = 0; c0 < H; c0 += OT_KC) {
    __syncthreads();
    for (int e = tid; e < jl * (OT_KC / 8); e += OT_THREADS) {
      const int j = e >> 3, q = e & 7;
      const uint4 raw = *reinterpret_cast<const uint4*>(v + j * ldv + c0 + q * 8);
      const float n = nv[j];
      const float2 a = unpack_bf16x2(raw.x), bb = unpack_bf16x2(raw.y), c = unpack_bf16x2(raw.z), d = unpack_bf16x2(raw.w);
      float4* o = reinterpret_cast<float4*>(vs + j * OT_KC + q * 8);
      o[0] = make_float4(a.x / n, a.y / n, bb.x / n, bb.y / n);
      o[1] = make_float4(c.x / n, c.y / n, d.x / n, d.y / n);
    }
    __syncthreads();
    if (i0 >= I) continue;
    float acc[4][8];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[r][c] = 0.0f;
    for (int j = 0; j < jl; ++j) {
      const float4 w = *reinterpret_cast<const float4*>(W + j * Ip + i0);
      const float4 p = *reinterpret_cast<const float4*>(vs + j * OT_KC + tc * 4);
      const float4 q = *reinterpret_cast<const float4*>(vs + j * OT_KC + 32 + tc * 4);
      const float wr[4] = {w.x, w.y, w.z, w.w};
      const float vc[8] = {p.x, p.y, p.z, p.w, q.x, q.y, q.z, q.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(wr[r], vc[c], acc[r][c]);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = i0 + r;
      if (i >= I) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int col = c0 + h * 32 + tc * 4;
        uint2 o = make_uint2(0, 0);                     // padded rows get exact zeros
        if (i < il) {
          const float n = nu[i];
          const float pr = n > OT_EPS ? proj[i] : 0.0f;
          const uint2 raw = *reinterpret_cast<const uint2*>(u + i * ldu + col);
          const float2 u01 = unpack_bf16x2(raw.x), u23 = unpack_bf16x2(raw.y);
          const float cf = gneg / n;
          o.x = pack_bf16x2(cf * (acc[r][4 * h + 0] - (u01.x / n) * pr), cf * (acc[r][4 * h + 1] - (u01.y / n) * pr));
          o.y = pack_bf16x2(cf * (acc[r][4 * h + 2] - (u23.x / n) * pr), cf * (acc[r][4 * h + 3] - (u23.y / n) * pr));
        }
        *reinterpret_cast<uint2*>(du + i * lddu + col) = o;
      }
    }
  }
}

size_t ot_fwd_smem(int M, int N) {
  const size_t Mp = (M + 15) & ~15, Np = (N + 7) & ~7;
  const size_t stage = (Mp + Np) * OT_LDS * sizeof(bf16), at = static_cast<size_t>(2) * M * N * sizeof(float);
  return (((static_cast<size_t>(M) * N + 3) & ~static_cast<size_t>(3)) + 4 * OT_MAX + 8) * sizeof(float) + (stage > at ? stage : at);
}

size_t ot_bwd_smem(int M, int N) {
  const size_t a = static_cast<size_t>(N) * ((M + 3) & ~3) + static_cast<size_t>(N) * OT_KC;
  const size_t c = static_cast<size_t>(M) * ((N + 3) & ~3) + static_cast<size_t>(M) * OT_KC;
  return (a > c ? a : c) * sizeof(float);
}

bool misaligned(const void* p, int64_t ld, int64_t bs) {
  return (reinterpret_cast<uintptr_t>(p) & 15) || (ld % 8) || (bs % 8);
}

int ot_check(const mmfb_ot_args& a, const char* who) {
  if (a.B < 1 || a.M < 1 || a.M > OT_MAX || a.N < 1 || a.N > OT_MAX)
    return set_error(MMFB_ERR_ARG, "%s: B >= 1 and 1 <= M, N <= %d are supported (B=%d M=%d N=%d)", who, OT_MAX, a.B, a.M, a.N);
  if (a.H < 64 || a.H > 1024 || (a.H % 64))
    return set_error(MMFB_ERR_ARG, "%s: H must be a multiple of 64 up to 1024, got %d", who, a.H);
  if (!a.x || !a.y || !a.x_len || !a.y_len || !a.plan || !a.saved)
    return set_error(MMFB_ERR_ARG, "%s: null pointer", who);
  if (misaligned(a.x, a.ldx, a.bsx) || misaligned(a.y, a.ldy, a.bsy))
    return set_error(MMFB_ERR_ARG, "%s: x and y must be 16-byte aligned with row and sample pitches that are multiples of 8", who);
  if (a.ldx < a.H || a.ldy < a.H) return set_error(MMFB_ERR_ARG, "%s: row pitch below H", who);
  for (int b = 0; b < a.B; ++b)
    if (a.x_len[b] < 1 || a.x_len[b] > a.M || a.y_len[b] < 1 || a.y_len[b] > a.N)
      return set_error(MMFB_ERR_ARG, "%s: sample %d has lengths %d / %d; 1 <= x_len <= M = %d and 1 <= y_len <= N = %d are supported",
                       who, b, a.x_len[b], a.y_len[b], a.M, a.N);
  return MMFB_OK;
}

// opt in to more than 48 KB of dynamic shared memory, once per size reached
template <typename Kern>
int ot_smem_attr(Kern kern, size_t smem, size_t& allowed, const char* who) {
  if (smem <= 48 * 1024 || smem <= allowed) return MMFB_OK;
  allowed = smem;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "%s: shared memory %zu: %s", who, smem, cudaGetErrorString(e));
  return MMFB_OK;
}

OtLens chunk_lens(const mmfb_ot_args& a, int b0, int nb) {
  OtLens l = {};
  for (int i = 0; i < nb; ++i) {
    l.x[i] = static_cast<uint8_t>(a.x_len[b0 + i]);
    l.y[i] = static_cast<uint8_t>(a.y_len[b0 + i]);
  }
  return l;
}

}  // namespace

int ot_fwd(const mmfb_ot_args& a, cudaStream_t s) {
  if (int rc = ot_check(a, "ot_fwd")) return rc;
  if (!a.dist) return set_error(MMFB_ERR_ARG, "ot_fwd: null pointer");
  if (!(a.beta > 0.0f) || a.iterations < 1 || a.k < 1)
    return set_error(MMFB_ERR_ARG, "ot_fwd: beta > 0, iterations >= 1 and k >= 1 are supported (beta=%g iterations=%d k=%d)",
                     a.beta, a.iterations, a.k);
  const size_t smem = ot_fwd_smem(a.M, a.N);
  static size_t allowed = 0;
  if (int rc = ot_smem_attr(ot_fwd_kernel, smem, allowed, "ot_fwd")) return rc;
  for (int b0 = 0; b0 < a.B; b0 += OT_CHUNK) {
    const int nb = a.B - b0 < OT_CHUNK ? a.B - b0 : OT_CHUNK;
    MMFB_LAUNCH(ot_fwd_kernel, nb, OT_THREADS, smem, s, reinterpret_cast<const bf16*>(a.x), a.ldx, a.bsx,
                reinterpret_cast<const bf16*>(a.y), a.ldy, a.bsy, chunk_lens(a, b0, nb), b0, a.M, a.N, a.H, a.beta, a.iterations,
                a.k, a.dist, a.plan, a.cost, a.saved);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "ot_fwd launch: %s", cudaGetErrorString(e));
    count_launch();
  }
  return MMFB_OK;
}

int ot_bwd(const mmfb_ot_args& a, cudaStream_t s) {
  if (int rc = ot_check(a, "ot_bwd")) return rc;
  if (!a.g || !a.dx || !a.dy) return set_error(MMFB_ERR_ARG, "ot_bwd: null pointer");
  if (misaligned(a.dx, a.lddx, a.bsdx) || misaligned(a.dy, a.lddy, a.bsdy) || a.lddx < a.H || a.lddy < a.H)
    return set_error(MMFB_ERR_ARG, "ot_bwd: dx and dy must be 16-byte aligned with row (>= H) and sample pitches that are multiples of 8");
  const size_t smem = ot_bwd_smem(a.M, a.N);
  static size_t allowed = 0;
  if (int rc = ot_smem_attr(ot_bwd_kernel, smem, allowed, "ot_bwd")) return rc;
  for (int b0 = 0; b0 < a.B; b0 += OT_CHUNK) {
    const int nb = a.B - b0 < OT_CHUNK ? a.B - b0 : OT_CHUNK;
    MMFB_LAUNCH(ot_bwd_kernel, dim3(nb, 2), OT_THREADS, smem, s, reinterpret_cast<const bf16*>(a.x), a.ldx, a.bsx,
                reinterpret_cast<const bf16*>(a.y), a.ldy, a.bsy, chunk_lens(a, b0, nb), b0, a.M, a.N, a.H, a.g, a.plan, a.saved,
                reinterpret_cast<bf16*>(a.dx), a.lddx, a.bsdx, reinterpret_cast<bf16*>(a.dy), a.lddy, a.bsdy);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "ot_bwd launch: %s", cudaGetErrorString(e));
    count_launch();
  }
  return MMFB_OK;
}

}  // namespace mmfb
