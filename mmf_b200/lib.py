"""ctypes binding of libmmfb200.so (the C ABI declared in include/mmfb200.h).

The library is loaded eagerly and loudly: if it is missing it is built in-tree with nvcc; if that is
impossible an ImportError is raised.  There is no Python/CPU fallback for any compute entry point.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# MMFB_LIB: measure another build of the SAME ABI (A/B runs of kernel changes on one box); never a fallback
_LIB_PATH = os.environ.get("MMFB_LIB") or os.path.join(_HERE, "csrc", "libmmfb200.so")

MMFB_OK, MMFB_ERR_ARG, MMFB_ERR_CUDA, MMFB_ERR_DEVICE = 0, 1, 2, 3

EPI_BIAS = 0
EPI_BIAS_GELU = 1
EPI_BIAS_DROP_RESID = 2
EPI_GELU_BWD = 3
EPI_ADD_AUX = 4
EPI_ATOMIC_F32 = 5
EPI_BIAS_RELU = 6
EPI_BIAS_GELU_DROP = 7
EPI_GELU_DROP_BWD = 8


class GemmArgs(ctypes.Structure):
    _fields_ = [
        ("A", ctypes.c_void_p), ("lda", ctypes.c_int64), ("a_mn", ctypes.c_int),
        ("B", ctypes.c_void_p), ("ldb", ctypes.c_int64), ("b_mn", ctypes.c_int),
        ("C", ctypes.c_void_p), ("ldc", ctypes.c_int64),
        ("C2", ctypes.c_void_p),
        ("bias", ctypes.c_void_p),
        ("aux", ctypes.c_void_p), ("ldaux", ctypes.c_int64),
        ("drop_mask", ctypes.c_void_p), ("ldmask", ctypes.c_int64), ("drop_scale", ctypes.c_float),
        ("M", ctypes.c_int), ("N", ctypes.c_int), ("K", ctypes.c_int),
        ("epi", ctypes.c_int),
        ("splits", ctypes.c_int),
        ("block_n", ctypes.c_int),
        ("cluster", ctypes.c_int),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_int64),
    ]


class AttnArgs(ctypes.Structure):
    _fields_ = [
        ("q", ctypes.c_void_p), ("ldq", ctypes.c_int64),
        ("k", ctypes.c_void_p), ("ldk", ctypes.c_int64),
        ("v", ctypes.c_void_p), ("ldv", ctypes.c_int64),
        ("mask", ctypes.c_void_p),
        ("ctx", ctypes.c_void_p), ("ldo", ctypes.c_int64),
        ("lse2", ctypes.c_void_p),
        ("drop_mask", ctypes.c_void_p), ("drop_scale", ctypes.c_float),
        ("ctx_lo", ctypes.c_void_p),
        ("dctx", ctypes.c_void_p), ("ld_dctx", ctypes.c_int64),
        ("delta", ctypes.c_void_p),
        ("dq", ctypes.c_void_p), ("ld_dq", ctypes.c_int64),
        ("dk", ctypes.c_void_p), ("ld_dk", ctypes.c_int64),
        ("dv", ctypes.c_void_p), ("ld_dv", ctypes.c_int64),
        ("B", ctypes.c_int), ("heads", ctypes.c_int), ("Sq", ctypes.c_int), ("Skv", ctypes.c_int),
        ("head_dim", ctypes.c_int),
        ("causal_len", ctypes.c_int),
    ]


class LnArgs(ctypes.Structure):
    _fields_ = [
        ("y", ctypes.c_void_p), ("ldy", ctypes.c_int64),
        ("gamma", ctypes.c_void_p), ("beta", ctypes.c_void_p),
        ("x", ctypes.c_void_p), ("ldx", ctypes.c_int64),
        ("mean", ctypes.c_void_p), ("rstd", ctypes.c_void_p),
        ("drop_mask", ctypes.c_void_p), ("ldmask", ctypes.c_int64), ("drop_scale", ctypes.c_float),
        ("eps", ctypes.c_float),
        ("dx", ctypes.c_void_p), ("lddx", ctypes.c_int64),
        ("dx2", ctypes.c_void_p), ("lddx2", ctypes.c_int64),
        ("dy", ctypes.c_void_p), ("lddy", ctypes.c_int64),
        ("dz", ctypes.c_void_p), ("lddz", ctypes.c_int64),
        ("dgamma", ctypes.c_void_p), ("dbeta", ctypes.c_void_p), ("dbias", ctypes.c_void_p),
        ("M", ctypes.c_int), ("H", ctypes.c_int),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_int64),
    ]


class ComposeArgs(ctypes.Structure):
    _fields_ = [
        ("src", ctypes.c_void_p * 2), ("ldsrc", ctypes.c_int64 * 2), ("src_row", ctypes.c_void_p * 2),
        ("tab", ctypes.c_void_p * 3), ("tab_idx", ctypes.c_void_p * 3),
        ("y", ctypes.c_void_p), ("ldy", ctypes.c_int64),
        ("M", ctypes.c_int), ("H", ctypes.c_int),
    ]


class AdamWArgs(ctypes.Structure):
    _fields_ = [
        ("param", ctypes.c_void_p), ("grad", ctypes.c_void_p), ("exp_avg", ctypes.c_void_p),
        ("exp_avg_sq", ctypes.c_void_p), ("param_bf16", ctypes.c_void_p), ("group", ctypes.c_void_p),
        ("n", ctypes.c_int64), ("n_groups", ctypes.c_int),
        ("lr", ctypes.c_float * 8), ("weight_decay", ctypes.c_float * 8), ("step_size", ctypes.c_float * 8),
        ("bc2_sqrt", ctypes.c_float * 8),
        ("beta1", ctypes.c_float), ("beta2", ctypes.c_float), ("eps", ctypes.c_float), ("grad_scale", ctypes.c_float),
        ("mode", ctypes.c_int),
        ("loss_scale_dev", ctypes.c_void_p), ("found_inf", ctypes.c_void_p),
        ("grad_scale_dev", ctypes.c_void_p),
        ("hp_dev", ctypes.c_void_p),
    ]


MMFB_ADAMW_SLOT_CORRECT_BIAS, MMFB_ADAMW_SLOT_FROZEN = 1, 2
MMFB_ADAMW_SEGMENT_BLOCK = 2048
ADAMW_HP_FLOATS = 8          # floats per mmfb_adamw_hp entry
ADAMW_GROUP_HP_DOUBLES = 5   # doubles per mmfb_adamw_group_hp entry


class AdamWSlot(ctypes.Structure):
    _fields_ = [("group", ctypes.c_int), ("flags", ctypes.c_int)]


class AdamWHparamsArgs(ctypes.Structure):
    _fields_ = [
        ("groups", ctypes.c_void_p), ("slots", ctypes.c_void_p), ("step", ctypes.c_void_p), ("hp", ctypes.c_void_p),
        ("n_slots", ctypes.c_int), ("mode", ctypes.c_int),
        ("found_inf", ctypes.c_void_p),
    ]


class AdamWSegment(ctypes.Structure):
    _fields_ = [
        ("param", ctypes.c_void_p), ("grad", ctypes.c_void_p), ("exp_avg", ctypes.c_void_p), ("exp_avg_sq", ctypes.c_void_p),
        ("n", ctypes.c_int64), ("slot", ctypes.c_int), ("first_block", ctypes.c_int), ("head", ctypes.c_int),
        ("pad_", ctypes.c_int),
    ]


class AdamWSegmentsArgs(ctypes.Structure):
    _fields_ = [
        ("segments", ctypes.c_void_p), ("n_segments", ctypes.c_int), ("n_blocks", ctypes.c_int),
        ("hp", ctypes.c_void_p), ("grad_scale", ctypes.c_float), ("mode", ctypes.c_int),
        ("grad_scale_dev", ctypes.c_void_p),
        ("loss_scale_dev", ctypes.c_void_p), ("found_inf", ctypes.c_void_p),
    ]


MMFB_GRAD_NORM_BLOCK = 16384
MMFB_GRAD_F32, MMFB_GRAD_BF16 = 0, 1


class GradSegment(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("n", ctypes.c_int64), ("dtype", ctypes.c_int), ("first_block", ctypes.c_int)]


class GradNormArgs(ctypes.Structure):
    _fields_ = [
        ("segments", ctypes.c_void_p), ("n_segments", ctypes.c_int), ("n_blocks", ctypes.c_int),
        ("partials", ctypes.c_void_p), ("out", ctypes.c_void_p),
        ("max_norm", ctypes.c_float), ("norm_type", ctypes.c_float),
        ("max_norm_scale_dev", ctypes.c_void_p),
    ]


MMFB_LR_WARMUP_LINEAR, MMFB_LR_WARMUP_COSINE, MMFB_LR_MULTI_STEP, MMFB_LR_PYTHIA = 0, 1, 2, 3
MMFB_LR_MAX_MILESTONES = 32


class LrScheduleDesc(ctypes.Structure):
    _fields_ = [
        ("kind", ctypes.c_int), ("use_warmup", ctypes.c_int),
        ("warmup_iterations", ctypes.c_int64), ("total_steps", ctypes.c_int64),
        ("warmup_factor", ctypes.c_double), ("num_cycles", ctypes.c_double),
        ("n_lr_steps", ctypes.c_int), ("pad_", ctypes.c_int),
        ("lr_steps", ctypes.c_int64 * MMFB_LR_MAX_MILESTONES),
        ("ratio_pow", ctypes.c_double * (MMFB_LR_MAX_MILESTONES + 1)),
    ]


class LrScheduleArgs(ctypes.Structure):
    _fields_ = [
        ("counter", ctypes.c_void_p), ("base_lr", ctypes.c_void_p), ("lr", ctypes.c_void_p),
        ("n_groups", ctypes.c_int), ("lr_stride", ctypes.c_int), ("advance", ctypes.c_int), ("pad_", ctypes.c_int),
        ("desc", LrScheduleDesc),
    ]


class ScatterArgs(ctypes.Structure):
    _fields_ = [
        ("dsrc", ctypes.c_void_p * 2), ("ldsrc", ctypes.c_int64 * 2), ("src_row", ctypes.c_void_p * 2),
        ("dtab", ctypes.c_void_p * 3), ("tab_idx", ctypes.c_void_p * 3),
        ("dy", ctypes.c_void_p), ("lddy", ctypes.c_int64),
        ("M", ctypes.c_int), ("H", ctypes.c_int),
    ]


class OtArgs(ctypes.Structure):
    _fields_ = [
        ("x", ctypes.c_void_p), ("ldx", ctypes.c_int64), ("bsx", ctypes.c_int64),
        ("y", ctypes.c_void_p), ("ldy", ctypes.c_int64), ("bsy", ctypes.c_int64),
        ("x_len", ctypes.c_void_p), ("y_len", ctypes.c_void_p),
        ("dist", ctypes.c_void_p), ("plan", ctypes.c_void_p), ("cost", ctypes.c_void_p), ("saved", ctypes.c_void_p),
        ("g", ctypes.c_void_p),
        ("dx", ctypes.c_void_p), ("lddx", ctypes.c_int64), ("bsdx", ctypes.c_int64),
        ("dy", ctypes.c_void_p), ("lddy", ctypes.c_int64), ("bsdy", ctypes.c_int64),
        ("B", ctypes.c_int), ("M", ctypes.c_int), ("N", ctypes.c_int), ("H", ctypes.c_int),
        ("beta", ctypes.c_float), ("iterations", ctypes.c_int), ("k", ctypes.c_int),
    ]


def _load():
    if not os.path.exists(_LIB_PATH):
        try:
            from .csrc.build import build
            build()
        except Exception as e:  # pragma: no cover - build environment problem
            raise ImportError(
                "libmmfb200.so is missing and could not be built (%s); run `python -m mmf_b200.csrc.build`" % (e,)
            )
    lib = ctypes.CDLL(_LIB_PATH)
    lib.mmfb_last_error.restype = ctypes.c_char_p
    lib.mmfb_launch_count.restype = ctypes.c_int64
    lib.mmfb_colsum.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                ctypes.c_void_p]
    lib.mmfb_colsum_ordered.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    lib.mmfb_embed_scatter_sorted_ordered.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                                      ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                      ctypes.c_int64, ctypes.c_void_p]
    lib.mmfb_gemm_workspace_bytes.argtypes = [ctypes.c_int] * 4
    for name in ("mmfb_layernorm_bwd_workspace_bytes", "mmfb_colsum_workspace_bytes",
                 "mmfb_embed_scatter_sorted_workspace_bytes"):
        getattr(lib, name).argtypes = [ctypes.c_int, ctypes.c_int]
    for name in ("mmfb_gemm_workspace_bytes", "mmfb_layernorm_bwd_workspace_bytes", "mmfb_colsum_workspace_bytes",
                 "mmfb_embed_scatter_sorted_workspace_bytes"):
        getattr(lib, name).restype = ctypes.c_int64
    lib.mmfb_dropout_bits.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint64, ctypes.c_uint64,
                                      ctypes.c_float, ctypes.c_void_p]
    lib.mmfb_dropout_bits_epoch.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p,
                                            ctypes.c_float, ctypes.c_void_p]
    lib.mmfb_dropout_path_bits.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_uint64,
                                           ctypes.c_uint64, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]
    lib.mmfb_dropout_path_bits_epoch.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_uint64,
                                                 ctypes.c_uint64, ctypes.c_void_p, ctypes.c_float, ctypes.c_float,
                                                 ctypes.c_void_p]
    lib.mmfb_embed_scatter_sorted.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                              ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.mmfb_gelu_bwd.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    lib.mmfb_relu_bwd.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    lib.mmfb_ce_rows.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                 ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.mmfb_gemm_bounded.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.mmfb_layernorm_fwd_bounded.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.mmfb_layernorm_bwd_bounded.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.mmfb_ce_rows_bounded.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                         ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                         ctypes.c_void_p]
    lib.mmfb_colsum_bounded.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    for name in ("mmfb_kl_rows_bounded", "mmfb_mse_rows_bounded"):
        getattr(lib, name).argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                       ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_void_p]
    lib.mmfb_select_rows.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                     ctypes.c_void_p]
    lib.mmfb_gather_rows.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                     ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.mmfb_plan_packing.argtypes = ([ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3) * 2 + \
        [ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.mmfb_add_bf16.argtypes =[ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    lib.mmfb_dropout_apply.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_float,
                                       ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.mmfb_cast_f32_bf16.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
    for name in ("mmfb_attention_varlen_fwd", "mmfb_attention_varlen_bwd", "mmfb_attention_varlen_causal_fwd",
                 "mmfb_attention_varlen_causal_bwd"):
        getattr(lib, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    for name in ("mmfb_attention_varlen_cross_fwd", "mmfb_attention_varlen_cross_bwd"):
        getattr(lib, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.c_void_p]
    lib.mmfb_attention_probs.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.mmfb_grad_norm_check.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.mmfb_grad_check.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                    ctypes.c_void_p]
    lib.mmfb_lr_schedule.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    for name in ("mmfb_adamw_active", "mmfb_adamw_hparams_active", "mmfb_adamw_segments_active"):
        getattr(lib, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    for name in ("mmfb_ot_fwd", "mmfb_ot_bwd"):
        getattr(lib, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    return lib


MMFB_PROBS_F32, MMFB_PROBS_BF16 = 0, 1

LIB = _load()
LIB_PATH = _LIB_PATH


def last_error():
    return LIB.mmfb_last_error().decode("utf-8", "replace")


def check(status):
    """Turns an mmfb_status into the exception the reference path would raise."""
    if status == MMFB_OK:
        return
    msg = last_error()
    if status == MMFB_ERR_ARG:
        raise ValueError(msg)
    raise RuntimeError(msg)


def launch_count():
    return int(LIB.mmfb_launch_count())


def device_ok():
    return bool(LIB.mmfb_device_ok())


def header_symbols():
    """Function names declared in include/mmfb200.h (used by the export test)."""
    import re
    hdr = os.path.join(os.path.dirname(_HERE), "include", "mmfb200.h")
    with open(hdr) as fh:
        txt = fh.read()
    return sorted(set(re.findall(r"\b(mmfb_[a-z0-9_]+)\s*\(", txt)))


def _stream_ptr(stream=None):
    import torch
    s = stream if stream is not None else torch.cuda.current_stream()
    return ctypes.c_void_p(s.cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
