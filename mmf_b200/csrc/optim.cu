// Fused AdamW over the flat fp32 parameter / gradient buffers of the engine (include/mmfb200.h: mmfb_adamw).
// HBM-bound: 4 fp32 streams read + 3 written (+ the bf16 compute copy) = 30 bytes per parameter, one pass.
// Arithmetic follows the reference's optimizer exactly, operation by operation (mmf/modules/optimizers.py:60-84 for the
// transformers variant, torch/optim/adamw.py single-tensor path for the fallback), so that parity is an fp32 statement.
#include "common.cuh"
#include "mmfb_internal.h"

namespace mmfb {

struct AdamWDev {
  float* p; const float* g; float* m; float* v; bf16* pb; const uint8_t* grp; int64_t n;
  float lr[MMFB_ADAMW_MAX_GROUPS], wd[MMFB_ADAMW_MAX_GROUPS], step[MMFB_ADAMW_MAX_GROUPS], bc2s[MMFB_ADAMW_MAX_GROUPS];
  float b1, b2, eps, gscale;
  const float* gscale_dev;   // read only by the SCALE_DEV instantiations (a device-side clipping coefficient)
  const mmfb_adamw_hp* hp;   // read only by the HP_DEV instantiations (mmfb_adamw_hparams' table)
  const float* loss_scale_dev;   // read only by the AMP instantiations (nullable there too)
  const float* found_inf;        // read only by the AMP instantiations (nullable there too)
};

// GradScaler's unscale factor of a loss scale S: (float)(1.0 / (double)S), as torch's _scale.double().reciprocal().float().
__device__ __forceinline__ float amp_inv_scale(const float* s) {
  return __double2float_rn(__ddiv_rn(1.0, static_cast<double>(*s)));
}

// A non-zero found_inf (GradScaler's flag of non-finite gradients) makes the whole update a no-op.
__device__ __forceinline__ bool amp_skip(const float* found_inf) { return found_inf != nullptr && *found_inf != 0.0f; }

// One element of the AdamW step, shared by adamw_kernel and adamw_segments_kernel so that both give the same bits.
// gr = g * gs is the scaled gradient; step = step_size, bc2s = bc2_sqrt.
template <int MODE>
__device__ __forceinline__ void adamw_elem(float& p, float& m, float& v, float g, float gs, float lr, float wd, float step,
                                           float bc2s, float b1, float b2, float eps) {
  const float gr = g * gs;
  if (MODE == 0) {
    // exp_avg.mul_(b1).add_(g, alpha=1-b1); exp_avg_sq.mul_(b2).addcmul_(g, g, value=1-b2)
    m = __fmaf_rn(gr, 1.0f - b1, m * b1);
    v = __fmaf_rn(gr * gr, 1.0f - b2, v * b2);
    const float denom = __fsqrt_rn(v) + eps;
    p = __fmaf_rn(-step, __fdiv_rn(m, denom), p);                          // p.addcdiv_(m, denom, value=-step_size)
    if (wd > 0.0f) p = __fmaf_rn(p, -lr * wd, p);                          // p.add_(p, alpha=-lr*wd)
  } else {
    p = p * (1.0f - lr * wd);                                              // p.mul_(1 - lr*wd)
    m = __fmaf_rn(gr - m, 1.0f - b1, m);                                   // m.lerp_(g, 1-b1)
    v = __fmaf_rn(gr * gr, 1.0f - b2, v * b2);
    const float denom = __fdiv_rn(__fsqrt_rn(v), bc2s) + eps;
    p = __fmaf_rn(-step, __fdiv_rn(m, denom), p);
  }
}

// SCALE_DEV: the gradient factor is gscale * *gscale_dev, read once per thread after the previous kernel has completed.
// HP_DEV: the group's hyper-parameters come from the device table a.hp instead of the launch parameters.
// AMP: loss scaling on the device - nothing is written when *found_inf is non-zero, and every gradient is first multiplied
// by amp_inv_scale(loss_scale_dev) (each pointer nullable), then by the factor above: GradScaler.unscale_, then step().
// The instantiations without any of the three are the kernels this file always had.
template <int MODE, bool SCALE_DEV, bool HP_DEV, bool AMP>
__global__ void __launch_bounds__(256)
adamw_kernel(const __grid_constant__ AdamWDev a) {
  griddep_launch();
  griddep_wait();
  if (AMP && amp_skip(a.found_inf)) return;
  const int64_t blk = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;     // 8-element block
  const int64_t i = blk * 8;
  if (i >= a.n) return;
  const int gi = a.grp != nullptr ? a.grp[blk] : 0;
  float lr, wd, step, bc2s, b1, b2, eps;
  if (HP_DEV) {
    const mmfb_adamw_hp h = a.hp[gi];
    lr = h.lr; wd = h.weight_decay; step = h.step_size; bc2s = h.bc2_sqrt; b1 = h.beta1; b2 = h.beta2; eps = h.eps;
  } else {
    lr = a.lr[gi]; wd = a.wd[gi]; step = a.step[gi]; bc2s = a.bc2s[gi]; b1 = a.b1; b2 = a.b2; eps = a.eps;
  }
  const float gs = SCALE_DEV ? a.gscale * *a.gscale_dev : a.gscale;
  float p[8], g[8], m[8], v[8];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float4 tp = *reinterpret_cast<const float4*>(a.p + i + 4 * h);
    const float4 tg = *reinterpret_cast<const float4*>(a.g + i + 4 * h);
    const float4 tm = *reinterpret_cast<const float4*>(a.m + i + 4 * h);
    const float4 tv = *reinterpret_cast<const float4*>(a.v + i + 4 * h);
    p[4 * h] = tp.x; p[4 * h + 1] = tp.y; p[4 * h + 2] = tp.z; p[4 * h + 3] = tp.w;
    g[4 * h] = tg.x; g[4 * h + 1] = tg.y; g[4 * h + 2] = tg.z; g[4 * h + 3] = tg.w;
    m[4 * h] = tm.x; m[4 * h + 1] = tm.y; m[4 * h + 2] = tm.z; m[4 * h + 3] = tm.w;
    v[4 * h] = tv.x; v[4 * h + 1] = tv.y; v[4 * h + 2] = tv.z; v[4 * h + 3] = tv.w;
  }
  if (AMP && a.loss_scale_dev != nullptr) {
    const float inv = amp_inv_scale(a.loss_scale_dev);
#pragma unroll
    for (int e = 0; e < 8; ++e) g[e] = g[e] * inv;
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) adamw_elem<MODE>(p[e], m[e], v[e], g[e], gs, lr, wd, step, bc2s, b1, b2, eps);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    *reinterpret_cast<float4*>(a.p + i + 4 * h) = make_float4(p[4 * h], p[4 * h + 1], p[4 * h + 2], p[4 * h + 3]);
    *reinterpret_cast<float4*>(a.m + i + 4 * h) = make_float4(m[4 * h], m[4 * h + 1], m[4 * h + 2], m[4 * h + 3]);
    *reinterpret_cast<float4*>(a.v + i + 4 * h) = make_float4(v[4 * h], v[4 * h + 1], v[4 * h + 2], v[4 * h + 3]);
  }
  if (a.pb != nullptr) {
    uint4 o;
    o.x = pack_bf16x2(p[0], p[1]); o.y = pack_bf16x2(p[2], p[3]);
    o.z = pack_bf16x2(p[4], p[5]); o.w = pack_bf16x2(p[6], p[7]);
    *reinterpret_cast<uint4*>(a.pb + i) = o;
  }
}

int adamw(const mmfb_adamw_args& a, cudaStream_t s) {
  if (!a.param || !a.grad || !a.exp_avg || !a.exp_avg_sq) return set_error(MMFB_ERR_ARG, "adamw: null pointer");
  if (a.n <= 0 || (a.n % 8)) return set_error(MMFB_ERR_ARG, "adamw: n must be a positive multiple of 8 (got %lld)", (long long)a.n);
  if (a.n_groups < 1 || a.n_groups > MMFB_ADAMW_MAX_GROUPS)
    return set_error(MMFB_ERR_ARG, "adamw: n_groups must be in [1, %d]", MMFB_ADAMW_MAX_GROUPS);
  if (a.mode != 0 && a.mode != 1) return set_error(MMFB_ERR_ARG, "adamw: mode must be 0 (transformers) or 1 (torch)");
  if ((reinterpret_cast<uintptr_t>(a.param) | reinterpret_cast<uintptr_t>(a.grad) | reinterpret_cast<uintptr_t>(a.exp_avg) |
       reinterpret_cast<uintptr_t>(a.exp_avg_sq) | reinterpret_cast<uintptr_t>(a.param_bf16)) & 15)
    return set_error(MMFB_ERR_ARG, "adamw: buffers must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(a.hp_dev) & 15) return set_error(MMFB_ERR_ARG, "adamw: hp_dev must be 16-byte aligned");
  AdamWDev d;
  d.p = a.param; d.g = a.grad; d.m = a.exp_avg; d.v = a.exp_avg_sq; d.pb = reinterpret_cast<bf16*>(a.param_bf16);
  d.grp = a.group; d.n = a.n;
  for (int i = 0; i < MMFB_ADAMW_MAX_GROUPS; ++i) {
    const int j = i < a.n_groups ? i : 0;
    d.lr[i] = a.lr[j]; d.wd[i] = a.weight_decay[j]; d.step[i] = a.step_size[j]; d.bc2s[i] = a.bc2_sqrt[j];
  }
  d.b1 = a.beta1; d.b2 = a.beta2; d.eps = a.eps; d.gscale = a.grad_scale; d.gscale_dev = a.grad_scale_dev;
  d.hp = a.hp_dev;
  d.loss_scale_dev = a.loss_scale_dev; d.found_inf = a.found_inf;
  const int64_t blocks8 = a.n / 8;
  const unsigned grid = static_cast<unsigned>((blocks8 + 255) / 256);
  const bool amp = a.loss_scale_dev != nullptr || a.found_inf != nullptr;
  const int variant = (amp ? 8 : 0) + a.mode * 4 + (a.grad_scale_dev != nullptr ? 2 : 0) + (a.hp_dev != nullptr ? 1 : 0);
  switch (variant) {
    case 0: MMFB_LAUNCH((adamw_kernel<0, false, false, false>), grid, 256, 0, s, d); break;
    case 1: MMFB_LAUNCH((adamw_kernel<0, false, true, false>), grid, 256, 0, s, d); break;
    case 2: MMFB_LAUNCH((adamw_kernel<0, true, false, false>), grid, 256, 0, s, d); break;
    case 3: MMFB_LAUNCH((adamw_kernel<0, true, true, false>), grid, 256, 0, s, d); break;
    case 4: MMFB_LAUNCH((adamw_kernel<1, false, false, false>), grid, 256, 0, s, d); break;
    case 5: MMFB_LAUNCH((adamw_kernel<1, false, true, false>), grid, 256, 0, s, d); break;
    case 6: MMFB_LAUNCH((adamw_kernel<1, true, false, false>), grid, 256, 0, s, d); break;
    case 7: MMFB_LAUNCH((adamw_kernel<1, true, true, false>), grid, 256, 0, s, d); break;
    case 8: MMFB_LAUNCH((adamw_kernel<0, false, false, true>), grid, 256, 0, s, d); break;
    case 9: MMFB_LAUNCH((adamw_kernel<0, false, true, true>), grid, 256, 0, s, d); break;
    case 10: MMFB_LAUNCH((adamw_kernel<0, true, false, true>), grid, 256, 0, s, d); break;
    case 11: MMFB_LAUNCH((adamw_kernel<0, true, true, true>), grid, 256, 0, s, d); break;
    case 12: MMFB_LAUNCH((adamw_kernel<1, false, false, true>), grid, 256, 0, s, d); break;
    case 13: MMFB_LAUNCH((adamw_kernel<1, false, true, true>), grid, 256, 0, s, d); break;
    case 14: MMFB_LAUNCH((adamw_kernel<1, true, false, true>), grid, 256, 0, s, d); break;
    default: MMFB_LAUNCH((adamw_kernel<1, true, true, true>), grid, 256, 0, s, d); break;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "adamw launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Device-side hyper-parameters (include/mmfb200.h: mmfb_adamw_hparams): one CTA, one slot per thread and pass.  fp64
// operation by operation as the host's B200AdamW._group_hp evaluates it (Python float ** int is C pow), rounded once.
// ---------------------------------------------------------------------------------------------------------------------
// SKIP: a non-zero *found_inf makes the launch a no-op (no step count advances, the table keeps its values), as a
// step that GradScaler skips does not count in torch's fused Adam.
constexpr int HP_THREADS = 256;

template <bool SKIP>
__global__ void __launch_bounds__(HP_THREADS)
adamw_hparams_kernel(const mmfb_adamw_group_hp* __restrict__ groups, const mmfb_adamw_slot* __restrict__ slots,
                     int64_t* __restrict__ steps, mmfb_adamw_hp* __restrict__ out, int n_slots, int mode,
                     const float* __restrict__ found_inf) {
  griddep_launch();
  griddep_wait();
  if (SKIP && *found_inf != 0.0f) return;
  for (int s = threadIdx.x; s < n_slots; s += HP_THREADS) {
    const mmfb_adamw_slot sl = slots[s];
    const mmfb_adamw_group_hp g = groups[sl.group];
    mmfb_adamw_hp h;
    h.beta1 = __double2float_rn(g.beta1); h.beta2 = __double2float_rn(g.beta2); h.eps = __double2float_rn(g.eps);
    h.pad_ = 0.0f;
    if (sl.flags & MMFB_ADAMW_SLOT_FROZEN) {
      h.lr = 0.0f; h.weight_decay = 0.0f; h.step_size = 0.0f; h.bc2_sqrt = 1.0f;
    } else {
      const int64_t t = steps[s] + 1;
      steps[s] = t;
      const double td = static_cast<double>(t);
      const double bc1 = __dsub_rn(1.0, pow(g.beta1, td));               // 1 - b1 ** t
      const double bc2s = __dsqrt_rn(__dsub_rn(1.0, pow(g.beta2, td)));  // math.sqrt(1 - b2 ** t)
      double ss, b2c;
      if (mode == 0) {
        ss = (sl.flags & MMFB_ADAMW_SLOT_CORRECT_BIAS) ? __ddiv_rn(__dmul_rn(g.lr, bc2s), bc1) : g.lr;
        b2c = 1.0;
      } else {
        ss = __ddiv_rn(g.lr, bc1);
        b2c = bc2s;
      }
      h.lr = __double2float_rn(g.lr); h.weight_decay = __double2float_rn(g.weight_decay);
      h.step_size = __double2float_rn(ss); h.bc2_sqrt = __double2float_rn(b2c);
    }
    out[s] = h;
  }
}

int adamw_hparams(const mmfb_adamw_hparams_args& a, cudaStream_t s) {
  if (!a.groups || !a.slots || !a.step || !a.hp) return set_error(MMFB_ERR_ARG, "adamw_hparams: null pointer");
  if (a.n_slots < 1) return set_error(MMFB_ERR_ARG, "adamw_hparams: need at least one slot (got %d)", a.n_slots);
  if (a.mode != 0 && a.mode != 1) return set_error(MMFB_ERR_ARG, "adamw_hparams: mode must be 0 (transformers) or 1 (torch)");
  if ((reinterpret_cast<uintptr_t>(a.groups) | reinterpret_cast<uintptr_t>(a.step)) & 7 ||
      reinterpret_cast<uintptr_t>(a.slots) & 7 || reinterpret_cast<uintptr_t>(a.hp) & 15)
    return set_error(MMFB_ERR_ARG, "adamw_hparams: groups / slots / step must be 8-byte aligned, hp 16-byte aligned");
  if (a.found_inf != nullptr)
    MMFB_LAUNCH(adamw_hparams_kernel<true>, 1, HP_THREADS, 0, s, a.groups, a.slots, a.step, a.hp, a.n_slots, a.mode,
                a.found_inf);
  else
    MMFB_LAUNCH(adamw_hparams_kernel<false>, 1, HP_THREADS, 0, s, a.groups, a.slots, a.step, a.hp, a.n_slots, a.mode,
                a.found_inf);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "adamw_hparams launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// AdamW over a table of separate fp32 tensors (include/mmfb200.h: mmfb_adamw_segments).  CTA b finds the segment whose
// first_block <= b is largest; thread t of its chunk c owns the 8-element group k = c * 256 + t, elements
// [8k - lead, 8k - lead + 8) of the segment clipped to [0, n).  A group inside the segment whose four streams are
// 16-byte aligned (head >= 0) moves as float4 pairs; the head group, the tail group and segments that are not co-aligned
// are read and written element by element.  Elements go through adamw_elem, as in adamw_kernel; AMP as there.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int AS_THREADS = MMFB_ADAMW_SEGMENT_BLOCK / 8;
static_assert(AS_THREADS == 256, "one 8-element group per thread");

template <int MODE, bool SCALE_DEV, bool AMP>
__global__ void __launch_bounds__(AS_THREADS)
adamw_segments_kernel(const mmfb_adamw_segment* __restrict__ segs, int n_segs, const mmfb_adamw_hp* __restrict__ hp,
                      float gscale, const float* __restrict__ gscale_dev, const float* __restrict__ loss_scale_dev,
                      const float* __restrict__ found_inf) {
  __shared__ int s_seg;
  griddep_launch();
  griddep_wait();
  if (AMP && amp_skip(found_inf)) return;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n_segs - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (segs[mid].first_block <= b) lo = mid; else hi = mid - 1;
    }
    s_seg = lo;
  }
  __syncthreads();
  const mmfb_adamw_segment sg = segs[s_seg];
  const int lead = sg.head > 0 ? 8 - sg.head : 0;
  const int64_t start = (static_cast<int64_t>(b - sg.first_block) * AS_THREADS + threadIdx.x) * 8 - lead;
  if (start >= sg.n) return;
  const mmfb_adamw_hp h = hp[sg.slot];
  const float gs = SCALE_DEV ? gscale * *gscale_dev : gscale;
  const bool vec = sg.head >= 0 && start >= 0 && start + 8 <= sg.n;
  float p[8], g[8], m[8], v[8];
  if (vec) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const float4 tp = *reinterpret_cast<const float4*>(sg.param + start + 4 * q);
      const float4 tg = *reinterpret_cast<const float4*>(sg.grad + start + 4 * q);
      const float4 tm = *reinterpret_cast<const float4*>(sg.exp_avg + start + 4 * q);
      const float4 tv = *reinterpret_cast<const float4*>(sg.exp_avg_sq + start + 4 * q);
      p[4 * q] = tp.x; p[4 * q + 1] = tp.y; p[4 * q + 2] = tp.z; p[4 * q + 3] = tp.w;
      g[4 * q] = tg.x; g[4 * q + 1] = tg.y; g[4 * q + 2] = tg.z; g[4 * q + 3] = tg.w;
      m[4 * q] = tm.x; m[4 * q + 1] = tm.y; m[4 * q + 2] = tm.z; m[4 * q + 3] = tm.w;
      v[4 * q] = tv.x; v[4 * q + 1] = tv.y; v[4 * q + 2] = tv.z; v[4 * q + 3] = tv.w;
    }
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int64_t j = start + e;
      const bool in = j >= 0 && j < sg.n;
      p[e] = in ? sg.param[j] : 0.0f; g[e] = in ? sg.grad[j] : 0.0f;
      m[e] = in ? sg.exp_avg[j] : 0.0f; v[e] = in ? sg.exp_avg_sq[j] : 0.0f;
    }
  }
  if (AMP && loss_scale_dev != nullptr) {
    const float inv = amp_inv_scale(loss_scale_dev);
#pragma unroll
    for (int e = 0; e < 8; ++e) g[e] = g[e] * inv;
  }
#pragma unroll
  for (int e = 0; e < 8; ++e)
    adamw_elem<MODE>(p[e], m[e], v[e], g[e], gs, h.lr, h.weight_decay, h.step_size, h.bc2_sqrt, h.beta1, h.beta2, h.eps);
  if (vec) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      *reinterpret_cast<float4*>(sg.param + start + 4 * q) = make_float4(p[4 * q], p[4 * q + 1], p[4 * q + 2], p[4 * q + 3]);
      *reinterpret_cast<float4*>(sg.exp_avg + start + 4 * q) = make_float4(m[4 * q], m[4 * q + 1], m[4 * q + 2], m[4 * q + 3]);
      *reinterpret_cast<float4*>(sg.exp_avg_sq + start + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int64_t j = start + e;
      if (j >= 0 && j < sg.n) { sg.param[j] = p[e]; sg.exp_avg[j] = m[e]; sg.exp_avg_sq[j] = v[e]; }
    }
  }
}

int adamw_segments(const mmfb_adamw_segments_args& a, cudaStream_t s) {
  if (!a.segments || !a.hp) return set_error(MMFB_ERR_ARG, "adamw_segments: null pointer");
  if (a.n_segments < 1 || a.n_blocks < 1)
    return set_error(MMFB_ERR_ARG, "adamw_segments: need at least one segment and one block (got %d, %d)", a.n_segments,
                     a.n_blocks);
  if (a.mode != 0 && a.mode != 1) return set_error(MMFB_ERR_ARG, "adamw_segments: mode must be 0 (transformers) or 1 (torch)");
  if (reinterpret_cast<uintptr_t>(a.segments) & 7 || reinterpret_cast<uintptr_t>(a.hp) & 15 ||
      reinterpret_cast<uintptr_t>(a.grad_scale_dev) & 3)
    return set_error(MMFB_ERR_ARG, "adamw_segments: segments must be 8-byte aligned, hp 16-byte, grad_scale_dev 4-byte");
  const bool amp = a.loss_scale_dev != nullptr || a.found_inf != nullptr;
  const int variant = (amp ? 4 : 0) + a.mode * 2 + (a.grad_scale_dev != nullptr ? 1 : 0);
#define MMFB_AS_LAUNCH(MODE, SCALE_DEV, AMP)                                                                       \
  MMFB_LAUNCH((adamw_segments_kernel<MODE, SCALE_DEV, AMP>), a.n_blocks, AS_THREADS, 0, s, a.segments, a.n_segments, \
              a.hp, a.grad_scale, a.grad_scale_dev, a.loss_scale_dev, a.found_inf)
  switch (variant) {
    case 0: MMFB_AS_LAUNCH(0, false, false); break;
    case 1: MMFB_AS_LAUNCH(0, true, false); break;
    case 2: MMFB_AS_LAUNCH(1, false, false); break;
    case 3: MMFB_AS_LAUNCH(1, true, false); break;
    case 4: MMFB_AS_LAUNCH(0, false, true); break;
    case 5: MMFB_AS_LAUNCH(0, true, true); break;
    case 6: MMFB_AS_LAUNCH(1, false, true); break;
    default: MMFB_AS_LAUNCH(1, true, true); break;
  }
#undef MMFB_AS_LAUNCH
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "adamw_segments launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Global L2 norm of a list of gradient segments (include/mmfb200.h: mmfb_grad_norm), two launches, no atomics.
// grad_norm_partial_kernel: block b owns elements [c * BLOCK, (c + 1) * BLOCK) (BLOCK = MMFB_GRAD_NORM_BLOCK) of the segment whose first_block <= b
// is largest, c = b - first_block.  Thread t owns the 8-element groups t, t + 256, ... of that chunk (GN_GROUPS of them)
// and adds x^2 element by element in fp64; the 256 thread sums are added by a fixed shuffle tree, and the 8 warp sums in
// warp order, into partial[b].  The element-to-thread map does not depend on alignment (an unaligned or short group is
// read element by element in the same order), so the order depends on the segment lengths and dtypes alone.
// grad_norm_final_kernel: one block of 1024 threads; thread t adds partials t, t + 1024, ... in index order, then the same
// fixed tree.  Squares of fp32 / bf16 values are exact in fp64, so the fp64 sum has a relative error below ~1e-14 for any
// realistic length, and the fp32 result is a faithful rounding of the exact norm (within one fp32 ulp).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int GN_THREADS = 256;
constexpr int GN_GROUPS = MMFB_GRAD_NORM_BLOCK / (GN_THREADS * 8);
static_assert(GN_GROUPS * GN_THREADS * 8 == MMFB_GRAD_NORM_BLOCK, "grad-norm chunk must be whole 8-element groups");
constexpr int GN_FINAL_THREADS = 1024;

__device__ __forceinline__ double gn_block_sum(double acc, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  double tot = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) tot += red[w];
  return tot;
}

__device__ __forceinline__ double gn_load(const void* p, int dtype, int64_t i) {
  return dtype == MMFB_GRAD_BF16 ? static_cast<double>(__bfloat162float(static_cast<const bf16*>(p)[i]))
                                 : static_cast<double>(static_cast<const float*>(p)[i]);
}

// Non-finite test of one fp32 value (a bf16 value widens to the same exponent): all exponent bits set is inf or NaN.
__device__ __forceinline__ bool gn_nonfinite(float x) { return (__float_as_uint(x) & 0x7f800000u) == 0x7f800000u; }

// KIND: GN_NORM sums the squares (the kernel this file always had); GN_NORM_CHECK also tests every element for
// inf / NaN and writes the block's flag (1.0 or 0.0) to flags[b]; GN_CHECK only tests and writes flags[b].
enum { GN_NORM = 0, GN_NORM_CHECK = 1, GN_CHECK = 2 };

template <int KIND>
__global__ void __launch_bounds__(GN_THREADS)
grad_norm_partial_kernel(const mmfb_grad_segment* __restrict__ segs, int n_segs, double* __restrict__ partial,
                         double* __restrict__ flags) {
  __shared__ int s_seg;
  __shared__ double red[GN_THREADS / 32];
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {                         // largest s with first_block <= b (empty segments are skipped over)
    int lo = 0, hi = n_segs - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (segs[mid].first_block <= b) lo = mid; else hi = mid - 1;
    }
    s_seg = lo;
  }
  __syncthreads();
  const mmfb_grad_segment sg = segs[s_seg];
  const int64_t start = static_cast<int64_t>(b - sg.first_block) * MMFB_GRAD_NORM_BLOCK;
  const int64_t len = min(static_cast<int64_t>(MMFB_GRAD_NORM_BLOCK), sg.n - start);
  double acc = 0.0;
  bool bad = false;
  if (sg.dtype == MMFB_GRAD_BF16) {
    const bf16* p = static_cast<const bf16*>(sg.ptr) + start;
    const bool vec = (reinterpret_cast<uintptr_t>(p) & 15) == 0;
#pragma unroll 4
    for (int k = 0; k < GN_GROUPS; ++k) {
      const int64_t j = (static_cast<int64_t>(k) * GN_THREADS + threadIdx.x) * 8;
      if (j >= len) break;
      if (vec && j + 8 <= len) {
        const uint4 u = __ldcs(reinterpret_cast<const uint4*>(p + j));
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = unpack_bf16x2(w[q]);
          if (KIND != GN_CHECK) {
            acc = fma(static_cast<double>(f.x), static_cast<double>(f.x), acc);
            acc = fma(static_cast<double>(f.y), static_cast<double>(f.y), acc);
          }
          if (KIND != GN_NORM) bad |= gn_nonfinite(f.x) | gn_nonfinite(f.y);
        }
      } else {
        for (int64_t e = j; e < min(j + 8, len); ++e) {
          const double x = gn_load(p, MMFB_GRAD_BF16, e);
          if (KIND != GN_CHECK) acc = fma(x, x, acc);
          if (KIND != GN_NORM) bad |= gn_nonfinite(static_cast<float>(x));
        }
      }
    }
  } else {
    const float* p = static_cast<const float*>(sg.ptr) + start;
    const bool vec = (reinterpret_cast<uintptr_t>(p) & 15) == 0;
#pragma unroll 4
    for (int k = 0; k < GN_GROUPS; ++k) {
      const int64_t j = (static_cast<int64_t>(k) * GN_THREADS + threadIdx.x) * 8;
      if (j >= len) break;
      if (vec && j + 8 <= len) {
        const float4 u = __ldcs(reinterpret_cast<const float4*>(p + j));
        const float4 v = __ldcs(reinterpret_cast<const float4*>(p + j + 4));
        const float f[8] = {u.x, u.y, u.z, u.w, v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (KIND != GN_CHECK) acc = fma(static_cast<double>(f[q]), static_cast<double>(f[q]), acc);
          if (KIND != GN_NORM) bad |= gn_nonfinite(f[q]);
        }
      } else {
        for (int64_t e = j; e < min(j + 8, len); ++e) {
          const double x = gn_load(p, MMFB_GRAD_F32, e);
          if (KIND != GN_CHECK) acc = fma(x, x, acc);
          if (KIND != GN_NORM) bad |= gn_nonfinite(static_cast<float>(x));
        }
      }
    }
  }
  if (KIND != GN_NORM) {
    bad = __syncthreads_or(bad);                  // an OR: the flag does not depend on which element or thread found it
    if (threadIdx.x == 0) flags[b] = bad ? 1.0 : 0.0;
  }
  if (KIND != GN_CHECK) {
    const double tot = gn_block_sum(acc, red);
    if (threadIdx.x == 0) partial[b] = tot;
  }
}

// Writes *found_inf = 1.0f when any of flags[0, n) is non-zero and 0.0f otherwise (one block of GN_FINAL_THREADS): an
// OR over the blocks' flags, so the value does not depend on the order in which they were written.
__device__ __forceinline__ void gn_found_inf(const double* __restrict__ flags, int n, float* __restrict__ found_inf) {
  bool any = false;
  for (int i = threadIdx.x; i < n; i += GN_FINAL_THREADS) any |= flags[i] != 0.0;
  any = __syncthreads_or(any);
  if (threadIdx.x == 0) *found_inf = any ? 1.0f : 0.0f;
}

// SCALE_DEV: the threshold is max_norm * *max_norm_scale in fp32 (MMF's clip of loss-scaled gradients at max_norm * S).
// CHECK: also writes *found_inf from the blocks' non-finite flags at partial + n_blocks.
template <bool SCALE_DEV, bool CHECK>
__global__ void __launch_bounds__(GN_FINAL_THREADS)
grad_norm_final_kernel(const double* __restrict__ partial, int n_blocks, float max_norm, float* __restrict__ out,
                       const float* __restrict__ max_norm_scale, float* __restrict__ found_inf) {
  __shared__ double red[GN_FINAL_THREADS / 32];
  griddep_launch();
  griddep_wait();
  double acc = 0.0;
  for (int i = threadIdx.x; i < n_blocks; i += GN_FINAL_THREADS) acc += partial[i];
  const double tot = gn_block_sum(acc, red);
  if (threadIdx.x == 0) {
    // torch.nn.utils.clip_grad_norm_: clip_coef = max_norm / (total_norm + 1e-6), clamped to at most 1, in fp32; torch
    // evaluates `float / Tensor` as reciprocal(Tensor) * float, and so does this.  The comparison form keeps a NaN
    // coefficient NaN (fminf would return 1).
    const float norm = static_cast<float>(sqrt(tot));
    const float mn = SCALE_DEV ? __fmul_rn(max_norm, *max_norm_scale) : max_norm;
    const float c = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), mn);
    out[0] = norm;
    out[1] = c > 1.0f ? 1.0f : c;
  }
  if (CHECK) gn_found_inf(partial + n_blocks, n_blocks, found_inf);
}

__global__ void __launch_bounds__(GN_FINAL_THREADS)
grad_check_final_kernel(const double* __restrict__ flags, int n_blocks, float* __restrict__ found_inf) {
  griddep_launch();
  griddep_wait();
  gn_found_inf(flags, n_blocks, found_inf);
}

static int grad_table_args(const mmfb_grad_segment* segs, int n_segs, int n_blocks, const void* partials, const char* who) {
  if (!segs || !partials) return set_error(MMFB_ERR_ARG, "%s: null pointer", who);
  if (n_segs < 1 || n_blocks < 1)
    return set_error(MMFB_ERR_ARG, "%s: need at least one segment and one block (got %d, %d)", who, n_segs, n_blocks);
  if (reinterpret_cast<uintptr_t>(segs) & 7 || reinterpret_cast<uintptr_t>(partials) & 7)
    return set_error(MMFB_ERR_ARG, "%s: segments / partials must be 8-byte aligned", who);
  return MMFB_OK;
}

int grad_norm(const mmfb_grad_norm_args& a, float* found_inf, cudaStream_t s) {
  const char* who = found_inf ? "grad_norm_check" : "grad_norm";
  if (!a.segments || !a.partials || !a.out) return set_error(MMFB_ERR_ARG, "%s: null pointer", who);
  if (a.norm_type != 2.0f) return set_error(MMFB_ERR_ARG, "%s: only norm_type 2 is supported (got %g)", who, a.norm_type);
  if (a.n_segments < 1 || a.n_blocks < 1)
    return set_error(MMFB_ERR_ARG, "%s: need at least one segment and one block (got %d, %d)", who, a.n_segments, a.n_blocks);
  if (reinterpret_cast<uintptr_t>(a.segments) & 7 || reinterpret_cast<uintptr_t>(a.partials) & 7 ||
      reinterpret_cast<uintptr_t>(a.out) & 3 || reinterpret_cast<uintptr_t>(found_inf) & 3)
    return set_error(MMFB_ERR_ARG, "%s: segments / partials must be 8-byte aligned, out and found_inf 4-byte aligned", who);
  if (found_inf)
    MMFB_LAUNCH(grad_norm_partial_kernel<GN_NORM_CHECK>, a.n_blocks, GN_THREADS, 0, s, a.segments, a.n_segments,
                a.partials, a.partials + a.n_blocks);
  else
    MMFB_LAUNCH(grad_norm_partial_kernel<GN_NORM>, a.n_blocks, GN_THREADS, 0, s, a.segments, a.n_segments, a.partials,
                static_cast<double*>(nullptr));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
#define MMFB_GN_FINAL(SCALE_DEV, CHECK)                                                                                 \
  MMFB_LAUNCH((grad_norm_final_kernel<SCALE_DEV, CHECK>), 1, GN_FINAL_THREADS, 0, s, static_cast<const double*>(a.partials), \
              a.n_blocks, a.max_norm, a.out, a.max_norm_scale_dev, found_inf)
  if (a.max_norm_scale_dev != nullptr) {
    if (found_inf) MMFB_GN_FINAL(true, true); else MMFB_GN_FINAL(true, false);
  } else {
    if (found_inf) MMFB_GN_FINAL(false, true); else MMFB_GN_FINAL(false, false);
  }
#undef MMFB_GN_FINAL
  e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  count_launch(2);
  return MMFB_OK;
}

int grad_check(const mmfb_grad_segment* segs, int n_segs, int n_blocks, double* flags, float* found_inf, cudaStream_t s) {
  int st = grad_table_args(segs, n_segs, n_blocks, flags, "grad_check");
  if (st != MMFB_OK) return st;
  if (!found_inf) return set_error(MMFB_ERR_ARG, "grad_check: null pointer");
  if (reinterpret_cast<uintptr_t>(found_inf) & 3) return set_error(MMFB_ERR_ARG, "grad_check: found_inf must be 4-byte aligned");
  MMFB_LAUNCH(grad_norm_partial_kernel<GN_CHECK>, n_blocks, GN_THREADS, 0, s, segs, n_segs, static_cast<double*>(nullptr),
              flags);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "grad_check launch: %s", cudaGetErrorString(e));
  MMFB_LAUNCH(grad_check_final_kernel, 1, GN_FINAL_THREADS, 0, s, static_cast<const double*>(flags), n_blocks, found_inf);
  e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "grad_check launch: %s", cudaGetErrorString(e));
  count_launch(2);
  return MMFB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Learning-rate schedules (include/mmfb200.h: mmfb_lr_schedule): one warp.  Every thread reads the counter t (plus one
// when advancing), evaluates MMF's schedule at t in fp64 with explicitly rounded operations (no contraction into fma,
// so each line is the host's Python expression), and writes base_lr[g] * lambda(t) for its groups; thread 0 then
// stores the advanced counter.  The powers lr_ratio ** i come from the descriptor, computed on the host.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int LR_THREADS = 32;

// bisect.bisect_right(lr_steps, t), the binary search itself (so an unsorted list gives the host's index as well)
__device__ __forceinline__ int lr_bisect_right(const mmfb_lr_schedule_desc& d, int64_t t) {
  int lo = 0, hi = d.n_lr_steps;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (t < d.lr_steps[mid]) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// The factor on base_lr.  The multi-step kinds return it as warmup_factor * (1 - alpha) + alpha or lr_ratio ** idx;
// base_lr * factor is then the reference's `base_lr * lr_ratio` (MultiStepScheduler.get_lr) and `base_lr * lmbda(t)`
// (LambdaLR over lr_lambda_update) alike.
__device__ __forceinline__ double lr_factor(const mmfb_lr_schedule_desc& d, int64_t t) {
  if (d.kind == MMFB_LR_WARMUP_LINEAR || d.kind == MMFB_LR_WARMUP_COSINE) {
    const int64_t w = d.warmup_iterations, n = d.total_steps;
    if (t < w) return __ddiv_rn(static_cast<double>(t), static_cast<double>(w > 1 ? w : 1));
    const int64_t span = n - w > 1 ? n - w : 1;
    if (d.kind == MMFB_LR_WARMUP_LINEAR) {
      const double x = __ddiv_rn(static_cast<double>(n - t), static_cast<double>(span));
      return x > 0.0 ? x : 0.0;                                                    // max(0.0, x)
    }
    const double progress = __ddiv_rn(static_cast<double>(t - w), static_cast<double>(span));
    const double arg = __dmul_rn(__dmul_rn(__dmul_rn(3.141592653589793, d.num_cycles), 2.0), progress);  // math.pi
    const double y = __dmul_rn(0.5, __dadd_rn(1.0, cos(arg)));
    return y > 0.0 ? y : 0.0;
  }
  if (d.use_warmup && t <= d.warmup_iterations) {
    const double alpha = __ddiv_rn(static_cast<double>(t), static_cast<double>(d.warmup_iterations));
    return __dadd_rn(__dmul_rn(d.warmup_factor, __dsub_rn(1.0, alpha)), alpha);
  }
  return d.ratio_pow[lr_bisect_right(d, t)];
}

__global__ void __launch_bounds__(LR_THREADS)
lr_schedule_kernel(const __grid_constant__ mmfb_lr_schedule_args a) {
  griddep_launch();
  griddep_wait();
  const int64_t t = *a.counter + (a.advance ? 1 : 0);
  const double f = lr_factor(a.desc, t);
  for (int g = threadIdx.x; g < a.n_groups; g += LR_THREADS)
    a.lr[static_cast<int64_t>(g) * a.lr_stride] = __dmul_rn(a.base_lr[g], f);
  __syncwarp();                                   // every lane has read the counter
  if (a.advance && threadIdx.x == 0) *a.counter = t;
}

int lr_schedule(const mmfb_lr_schedule_args& a, cudaStream_t s) {
  const mmfb_lr_schedule_desc& d = a.desc;
  if (!a.counter || !a.base_lr || !a.lr) return set_error(MMFB_ERR_ARG, "lr_schedule: null pointer");
  if ((reinterpret_cast<uintptr_t>(a.counter) | reinterpret_cast<uintptr_t>(a.base_lr) | reinterpret_cast<uintptr_t>(a.lr)) & 7)
    return set_error(MMFB_ERR_ARG, "lr_schedule: counter, base_lr and lr must be 8-byte aligned");
  if (a.n_groups < 1 || a.lr_stride < 1)
    return set_error(MMFB_ERR_ARG, "lr_schedule: need n_groups >= 1 and lr_stride >= 1 (got %d, %d)", a.n_groups, a.lr_stride);
  if (d.kind < MMFB_LR_WARMUP_LINEAR || d.kind > MMFB_LR_PYTHIA)
    return set_error(MMFB_ERR_ARG, "lr_schedule: unknown schedule kind %d", d.kind);
  if (d.n_lr_steps < 0 || d.n_lr_steps > MMFB_LR_MAX_MILESTONES)
    return set_error(MMFB_ERR_ARG, "lr_schedule: n_lr_steps must be in [0, %d] (got %d)", MMFB_LR_MAX_MILESTONES, d.n_lr_steps);
  if ((d.kind == MMFB_LR_MULTI_STEP || d.kind == MMFB_LR_PYTHIA) && d.use_warmup && d.warmup_iterations < 1)
    return set_error(MMFB_ERR_ARG, "lr_schedule: warmup needs warmup_iterations >= 1 (got %lld)",
                     static_cast<long long>(d.warmup_iterations));
  MMFB_LAUNCH(lr_schedule_kernel, 1, LR_THREADS, 0, s, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "lr_schedule launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

// du = dh * GELU'(u), 16-byte vectors (staged with the MLM head, SURVEY.md 8f item 1)
__global__ void gelu_bwd_kernel(const bf16* __restrict__ dh, const bf16* __restrict__ u, bf16* __restrict__ du, int64_t n) {
  griddep_launch();
  griddep_wait();
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const uint4 a = *reinterpret_cast<const uint4*>(dh + i);
    const uint4 b = *reinterpret_cast<const uint4*>(u + i);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint32_t ow[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 d = unpack_bf16x2(aw[k]), x = unpack_bf16x2(bw[k]);
      ow[k] = pack_bf16x2(d.x * gelu_erf_grad(x.x), d.y * gelu_erf_grad(x.y));
    }
    *reinterpret_cast<uint4*>(du + i) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
  } else {
    for (int64_t j = i; j < n; ++j)
      du[j] = __float2bfloat16_rn(__bfloat162float(dh[j]) * gelu_erf_grad(__bfloat162float(u[j])));
  }
}

int gelu_bwd(const void* dh, const void* u, void* du, int64_t n, cudaStream_t s) {
  if (n <= 0) return set_error(MMFB_ERR_ARG, "gelu_bwd: empty");
  if ((reinterpret_cast<uintptr_t>(dh) | reinterpret_cast<uintptr_t>(u) | reinterpret_cast<uintptr_t>(du)) & 15)
    return set_error(MMFB_ERR_ARG, "gelu_bwd: buffers must be 16-byte aligned");
  const int64_t thr = (n + 7) / 8;
  MMFB_LAUNCH(gelu_bwd_kernel, static_cast<unsigned>((thr + 255) / 256), 256, 0, s, (const bf16*)dh, (const bf16*)u, (bf16*)du, n);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MMFB_ERR_CUDA, "gelu_bwd launch: %s", cudaGetErrorString(e));
  count_launch();
  return MMFB_OK;
}

}  // namespace mmfb
