/* libmmfb200 - the capturable AdamW step gated per slot: the parameters a step updates are chosen on the device, so one
 * captured update can serve micro-batches whose tasks reach different parameters (UNITER's heads under
 * training.update_frequency).  Included by mmfb200.h; the argument structs are declared there.  Their NaN and sentinel
 * checks are in tests/test_uniter_graphs_update_gpu.py.
 *
 * `active` is DEVICE uint8, one byte per slot of the mmfb_adamw_hparams slot table (for mmfb_adamw_active: one per
 * entry of hp_dev, i.e. the pack's slots).  A slot whose byte is 0 behaves as a parameter whose grad is None behaves in
 * torch.optim.AdamW: its parameters (and bf16 copy), exp_avg and exp_avg_sq are neither read nor written, its step
 * count is neither read nor advanced, and its hp row is written as a frozen slot's (lr = weight_decay = step_size = 0,
 * bc2_sqrt = 1).  A non-zero byte is the ungated launch, bit for bit.  A non-zero *found_inf still makes the whole
 * launch a no-op.  Every other argument is as for the ungated entry point; a null `active`, or mmfb_adamw_active without
 * hp_dev, is MMFB_ERR_ARG before any launch. */
#ifndef MMFB200_ACTIVE_H_
#define MMFB200_ACTIVE_H_

#include "mmfb200.h"

#ifdef __cplusplus
extern "C" {
#endif

int mmfb_adamw_active(const mmfb_adamw_args* args, const uint8_t* active, mmfb_stream stream);
int mmfb_adamw_hparams_active(const mmfb_adamw_hparams_args* args, const uint8_t* active, mmfb_stream stream);
int mmfb_adamw_segments_active(const mmfb_adamw_segments_args* args, const uint8_t* active, mmfb_stream stream);

#ifdef __cplusplus
}
#endif

#endif /* MMFB200_ACTIVE_H_ */
