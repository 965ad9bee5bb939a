/* libmmfb200: the device planner of skip-padding packings, part of the C ABI of include/mmfb200.h (which includes this
 * file).  Its NaN and sentinel checks are in tests/test_device_plan_gpu.py. */
#ifndef MMFB200_PLAN_H_
#define MMFB200_PLAN_H_

#include "mmfb200.h"   /* mmfb_stream, mmfb_status */

#ifdef __cplusplus
extern "C" {
#endif
/* Packing plan of a skip-padding encoder call, planned on the device at the fixed capacity B * S_k rows per stream, so
 * that a CUDA graph can capture the call.  One launch plans one stream (S1 = 0: mask1 and stream 1's outputs NULL) or
 * two (S1 > 0).  mask_k: DEVICE fp32 [B, S_k], additive; a position is valid where it is exactly 0, and any other value
 * is padding.  A stream whose mask is NULL (S_k > 0 still) is unpadded: nothing is written for it, and for the
 * one-sided rule below it holds a valid row in every sample.  At least one mask must be set.  Per planned stream:
 *   cu_k:         DEVICE int32 [B + 1]: cu_k[b] = the packed rows before sample b; cu_k[B] is the device row count;
 *   pack_map_k:   DEVICE int32 [B * S_k]: the flat source index (b * S_k + s) of each packed row, in sample order and in
 *                 position order within a sample, then -1 from cu_k[B] on;
 *   unpack_map_k: DEVICE int32 [B * S_k]: the packed row of each position, or -1 where the position is not kept.
 * Kept positions: the valid ones; with causal_len = T > 0 (one stream only) also the last T positions of every sample, the
 * causal tail, so every sample keeps at least T rows and its tail is its last T packed rows.  Two streams: a sample
 * with no valid position in one stream and at least one in the other keeps EVERY position of the empty stream (the
 * other stream's queries attend over all of them, as in the dense path, where they all carry the same mask value); a
 * sample with none in either stream keeps nothing.  With one stream and no tail the three outputs equal those of the
 * torch plan of the single-stream encoders bit for bit.
 * Launch: one CTA of 1024 threads per planned stream, no dynamic shared memory, no atomics (the same bits on every run).
 * Limits: 1 <= B <= 4096, S_k >= 1, B * S_k < 2^31, 0 <= causal_len <= S0, every buffer 4-byte aligned; anything else is
 * MMFB_ERR_ARG before any launch. */
int mmfb_plan_packing(const float* mask0, int S0, int32_t* cu0, int32_t* pack_map0, int32_t* unpack_map0,
                      const float* mask1, int S1, int32_t* cu1, int32_t* pack_map1, int32_t* unpack_map1,
                      int B, int causal_len, mmfb_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* MMFB200_PLAN_H_ */
