/* libmmfb200 - the device side of MMF's update beyond the AdamW step: learning-rate schedules and GradScaler's
 * non-finite check fused into the gradient-norm pass.  Included by mmfb200.h; the types it uses (mmfb_stream,
 * mmfb_grad_norm_args, mmfb_grad_segment) are declared there.  Their NaN and sentinel checks are in
 * tests/test_device_update_gpu.py. */
#ifndef MMFB200_UPDATE_H_
#define MMFB200_UPDATE_H_

#include "mmfb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The same norm and coefficient as mmfb_grad_norm, and GradScaler's non-finite check of the same gradients in the same
 * read: *found_inf (DEVICE fp32, GradScaler's dtype) is written 1.0f when any element of any segment is inf or NaN and
 * 0.0f otherwise.  The test is on each element's exponent bits, never on the norm: a finite fp32 gradient above ~1.8e19
 * squares to inf in fp32 but is not a skip for GradScaler.  Each block ORs its elements' flags, and the second launch
 * ORs the blocks' flags, so the result does not depend on launch order.  `partials` is DEVICE fp64 workspace
 * [2 * n_blocks] here (the block flags follow the partial sums).  Arguments otherwise as mmfb_grad_norm; a null or
 * misaligned found_inf is MMFB_ERR_ARG before any launch. */
int mmfb_grad_norm_check(const mmfb_grad_norm_args* args, float* found_inf, mmfb_stream stream);

/* The non-finite check alone, over a segment table of mmfb_grad_norm (for updates without clipping): *found_inf is
 * written 1.0f when any element is inf or NaN and 0.0f otherwise, in two launches as above.  flags: DEVICE fp64
 * workspace [n_blocks]. */
int mmfb_grad_check(const mmfb_grad_segment* segments, int n_segments, int n_blocks, double* flags, float* found_inf,
                    mmfb_stream stream);

/* MMF's learning-rate schedules on the device (mmf/modules/schedulers.py), one launch of one warp.  With t = *counter +
 * advance (LambdaLR's last_epoch after the step), group g gets lr[g * lr_stride] = base_lr[g] * f(t) in fp64, and with
 * advance set *counter = t.  f, in fp64 with every operation rounded as the host's Python expression:
 *   WARMUP_LINEAR (transformers' get_linear_schedule_with_warmup; W = warmup_iterations, N = total_steps):
 *     t < W: t / max(1, W);  else max(0, (N - t) / max(1, N - W))
 *   WARMUP_COSINE (get_cosine_schedule_with_warmup): t < W as above; else with p = (t - W) / max(1, N - W),
 *     max(0, 0.5 * (1 + cos(pi * num_cycles * 2 * p)))  - the device cos: within 2 ulp of the host's cosine
 *     term, so within base_lr * 2^-53 (plus 2 ulp) of the host's lr; 1 + cos cancels near the end of a half cycle
 *   MULTI_STEP (MultiStepScheduler.get_lr) and PYTHIA (lr_lambda_update under LambdaLR): with use_warmup and
 *     t <= warmup_iterations, alpha = t / warmup_iterations and f = warmup_factor * (1 - alpha) + alpha; otherwise
 *     f = ratio_pow[bisect_right(lr_steps, t)], the host's lr_ratio ** i.
 * lr is typically the mmfb_adamw_group_hp table of mmfb_adamw_hparams (lr_stride 5), so the next AdamW step reads the
 * scheduled lr on the device.  The descriptor travels by value (a captured launch freezes it).  MMFB_ERR_ARG before a
 * launch: a null or misaligned pointer, n_groups or lr_stride < 1, an unknown kind, n_lr_steps outside
 * [0, MMFB_LR_MAX_MILESTONES], or a multi-step warmup with warmup_iterations < 1 (the host divides by zero). */
#define MMFB_LR_WARMUP_LINEAR 0
#define MMFB_LR_WARMUP_COSINE 1
#define MMFB_LR_MULTI_STEP 2
#define MMFB_LR_PYTHIA 3
#define MMFB_LR_MAX_MILESTONES 32
typedef struct {
  int kind;                  /* MMFB_LR_* */
  int use_warmup;            /* MULTI_STEP / PYTHIA */
  int64_t warmup_iterations; /* num_warmup_steps for the transformers kinds */
  int64_t total_steps;       /* num_training_steps (WARMUP_LINEAR / WARMUP_COSINE) */
  double warmup_factor;
  double num_cycles;
  int n_lr_steps;
  int pad_;
  int64_t lr_steps[MMFB_LR_MAX_MILESTONES];
  double ratio_pow[MMFB_LR_MAX_MILESTONES + 1];   /* lr_ratio ** i, i = 0..n_lr_steps */
} mmfb_lr_schedule_desc;
typedef struct {
  int64_t* counter;          /* DEVICE int64 [1] */
  const double* base_lr;     /* DEVICE fp64 [n_groups] */
  double* lr;                /* DEVICE fp64, group g at lr[g * lr_stride] */
  int n_groups;
  int lr_stride;
  int advance;               /* 0: evaluate at *counter; 1: advance the counter first */
  int pad_;
  mmfb_lr_schedule_desc desc;
} mmfb_lr_schedule_args;
int mmfb_lr_schedule(const mmfb_lr_schedule_args* args, mmfb_stream stream);

#ifdef __cplusplus
}
#endif

#endif /* MMFB200_UPDATE_H_ */
