// Packing plan of a skip-padding encoder call, computed on the device so that a CUDA graph can capture the call
// (include/mmfb200.h, mmfb_plan_packing).  One launch plans one stream (BERT, M4C's multimodal transformer with its causal
// tail) or the two streams of a ViLBERT / LXMERT call, from their additive fp32 masks.
//
// One CTA per stream, three phases:
//   1. one warp per sample counts the kept positions of its row (mask exactly 0, or inside the causal tail); a two-stream
//      sample with no kept position while the other stream has one keeps its whole row instead (the one-sided rule);
//   2. an exclusive scan of the B lengths over the CTA's threads, in thread order, gives cu;
//   3. one warp per sample walks its row again in 32-position chunks: a ballot and a population count give each kept
//      position its packed row, written to unpack_map, and its flat index, written to pack_map at that row.
// The rows past cu[B] of pack_map get -1.  No atomics: every output is the same on every run.
#include "common.cuh"
#include "mmfb_internal.h"

namespace mmfb {

namespace {

constexpr int PLAN_THREADS = 1024;
constexpr int PLAN_WARPS = PLAN_THREADS / 32;
constexpr int PLAN_MAX_B = 4096;       // lengths of one stream in shared memory: 16 KB

struct PlanStream {
  const float* mask;                   // [B, S], NULL: an unpadded stream, planned by nobody
  int S;
  int32_t* cu;                         // [B + 1]
  int32_t* pack_map;                   // [B * S]
  int32_t* unpack_map;                 // [B * S]
};

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(PLAN_THREADS)
plan_packing_kernel(PlanStream s0, PlanStream s1, int B, int causal_len, int two_streams) {
  griddep_launch();
  griddep_wait();
  __shared__ int len[PLAN_MAX_B + 1];
  __shared__ int warp_tot[PLAN_WARPS];
  const PlanStream me = blockIdx.x == 0 ? s0 : s1;
  const PlanStream other = blockIdx.x == 0 ? s1 : s0;
  if (me.mask == nullptr) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int S = me.S, P = me.S - causal_len;          // positions >= P are the causal tail: always kept

  // 1. lengths
  for (int b = warp; b < B; b += PLAN_WARPS) {
    const float* row = me.mask + static_cast<int64_t>(b) * S;
    int n = 0;
    for (int s = lane; s < P; s += 32) n += row[s] == 0.0f;
    n = warp_sum(n) + causal_len;
    if (two_streams && n == 0) {
      // one-sided: this stream is empty where the other is not, and keeps every row so the other's queries see them
      int any = 1;
      if (other.mask != nullptr) {
        const float* orow = other.mask + static_cast<int64_t>(b) * other.S;
        int o = 0;
        for (int s = lane; s < other.S; s += 32) o |= orow[s] == 0.0f;
        any = __any_sync(0xffffffffu, o);
      }
      if (any) n = S;
    }
    if (lane == 0) len[b] = n;
  }
  __syncthreads();

  // 2. cu: thread t owns the consecutive samples [t * per, (t + 1) * per)
  const int per = (B + PLAN_THREADS - 1) / PLAN_THREADS;
  const int b0 = min(B, static_cast<int>(threadIdx.x) * per), b1 = min(B, b0 + per);
  int mine = 0;
  for (int b = b0; b < b1; ++b) mine += len[b];
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  int start = incl - mine, total = 0;
  for (int w = 0; w < PLAN_WARPS; ++w) {
    const int t = warp_tot[w];
    if (w < warp) start += t;
    total += t;
  }
  __syncthreads();                                    // every length is read before the starts replace them
  for (int b = b0; b < b1; ++b) {
    const int n = len[b];
    len[b] = start;
    me.cu[b] = start;
    start += n;
  }
  if (threadIdx.x == 0) {
    len[B] = total;
    me.cu[B] = total;
  }
  __syncthreads();

  // 3. the maps
  for (int b = warp; b < B; b += PLAN_WARPS) {
    const float* row = me.mask + static_cast<int64_t>(b) * S;
    const int64_t flat0 = static_cast<int64_t>(b) * S;
    int next = len[b];
    const bool all = len[b + 1] - next == S;          // every position kept: all valid, or one-sided
    for (int c = 0; c < S; c += 32) {
      const int s = c + lane;
      const bool kept = s < S && (all || s >= P || row[s] == 0.0f);
      const unsigned ballot = __ballot_sync(0xffffffffu, kept);
      const int dst = next + __popc(ballot & ((1u << lane) - 1u));
      if (s < S) me.unpack_map[flat0 + s] = kept ? dst : -1;
      if (kept) me.pack_map[dst] = static_cast<int32_t>(flat0 + s);
      next += __popc(ballot);
    }
  }
  const int C = B * S;
  for (int i = total + threadIdx.x; i < C; i += PLAN_THREADS) me.pack_map[i] = -1;
}

int plan_check(const char* who, const PlanStream& st, int B, int k) {
  if (st.S <= 0) return set_error(MMFB_ERR_ARG, "%s: stream %d has S = %d", who, k, st.S);
  if (static_cast<int64_t>(B) * st.S > INT32_MAX)
    return set_error(MMFB_ERR_ARG, "%s: stream %d has B * S = %lld rows, more than an int32 indexes", who, k,
                     static_cast<long long>(B) * st.S);
  if (st.mask == nullptr) {
    if (st.cu || st.pack_map || st.unpack_map)
      return set_error(MMFB_ERR_ARG, "%s: stream %d has no mask, so it takes no outputs", who, k);
    return MMFB_OK;
  }
  if (!st.cu || !st.pack_map || !st.unpack_map) return set_error(MMFB_ERR_ARG, "%s: stream %d: null output", who, k);
  if ((reinterpret_cast<uintptr_t>(st.mask) | reinterpret_cast<uintptr_t>(st.cu) |
       reinterpret_cast<uintptr_t>(st.pack_map) | reinterpret_cast<uintptr_t>(st.unpack_map)) & 3)
    return set_error(MMFB_ERR_ARG, "%s: stream %d: buffers must be 4-byte aligned", who, k);
  return MMFB_OK;
}

}  // namespace

}  // namespace mmfb

extern "C" int mmfb_plan_packing(const float* mask0, int S0, int32_t* cu0, int32_t* pack_map0, int32_t* unpack_map0,
                                 const float* mask1, int S1, int32_t* cu1, int32_t* pack_map1, int32_t* unpack_map1,
                                 int B, int causal_len, mmfb_stream stream) {
  using namespace mmfb;
  const char* who = "mmfb_plan_packing";
  if (B <= 0 || B > PLAN_MAX_B) return set_error(MMFB_ERR_ARG, "%s: B = %d must be in [1, %d]", who, B, PLAN_MAX_B);
  const PlanStream s0{mask0, S0, cu0, pack_map0, unpack_map0};
  const PlanStream s1{mask1, S1, cu1, pack_map1, unpack_map1};
  const int two = S1 != 0;
  int rc = plan_check(who, s0, B, 0);
  if (rc) return rc;
  if (two) {
    rc = plan_check(who, s1, B, 1);
    if (rc) return rc;
  } else if (mask1 || cu1 || pack_map1 || unpack_map1) {
    return set_error(MMFB_ERR_ARG, "%s: S1 = 0 plans one stream; stream 1's pointers must be NULL", who);
  }
  if (!mask0 && !mask1) return set_error(MMFB_ERR_ARG, "%s: no stream has a mask, so there is nothing to plan", who);
  if (causal_len < 0 || causal_len > S0)
    return set_error(MMFB_ERR_ARG, "%s: causal_len = %d must be in [0, S0 = %d]", who, causal_len, S0);
  if (causal_len && two) return set_error(MMFB_ERR_ARG, "%s: a causal tail is planned for one stream only", who);
  MMFB_LAUNCH(plan_packing_kernel, two ? 2 : 1, PLAN_THREADS, 0, reinterpret_cast<cudaStream_t>(stream), s0, s1, B,
              causal_len, two);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}
