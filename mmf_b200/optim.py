"""Fused AdamW for the fusion block's parameters (SURVEY.md 8f item 2; STAGED: CPU-verified host logic + parity tests
against the reference's arithmetic, the CUDA kernel has not run on the GPU yet).

Drop-in for the reference's optimizer `adam_w` (mmf/modules/optimizers.py:8-17: transformers' AdamW, or
torch.optim.AdamW when transformers ships none), taking the same parameter groups
(mmf/utils/modeling.py:18-46 `get_bert_configured_parameters`: weight decay 0.01 / 0 for bias + LayerNorm).  Parameters
that live in an engine ParamPack are updated by ONE kernel over the pack's flat fp32 master / gradient buffers
(`mmfb_adamw`: 4 streams read, 3 written, hyper-parameter group looked up per 8-element block); the per-parameter
`state[p]["exp_avg"]` / `["exp_avg_sq"]` tensors are views of flat state buffers, so `state_dict()` keeps torch's layout.
Parameters outside any pack (task heads, poolers) fall back to the same arithmetic in torch ops.

Gradient clipping: `clip_grad_norm(max_norm)` is the hook MMF's trainer calls when the optimizer has one
(mmf/utils/general.py `clip_gradients`, `clip_norm_mode: all`).  The global L2 norm and torch's clip coefficient are
computed on the device (`mmfb_grad_norm`, one read of the gradients, fixed summation order); the next `step()` multiplies
every gradient by the coefficient it reads from device memory - inside the AdamW kernel for the packs, as a tensor factor
on the torch-op path - so nothing waits for the host and the clipped step can be captured in a CUDA graph.

Capturable steps: `B200AdamW(..., capturable=True)` steps every parameter with library launches and reads nothing on the
host, so clip + step can be captured in a CUDA graph (mmf_b200.graphs.GraphedStep(..., optimizer=opt)).  The step counts
live on the device (`state[p]["step"]` is a 0-d int64 CUDA tensor, shared by the parameters of one pack and group) and
one launch (`mmfb_adamw_hparams`) advances them and computes each slot's step size and bias corrections from the group
values, which stay Python floats in `param_groups` (schedulers keep working) and are staged by one pinned host-to-device
copy per step.  Packs get one `mmfb_adamw` each reading that table; every other parameter goes into one
`mmfb_adamw_segments` launch.  `state_dict()` reports the step counts as ints (one device read).

Loss scaling: a capturable B200AdamW implements torch's fused-optimizer protocol (`_step_supports_amp_scaling`), the path
MMF's trainer takes with `training.fp16` (mmf/trainers/core/training_loop.py: `scaler.step(optimizer)`).  GradScaler then
neither unscales the gradients nor reads `found_inf` on the host: it hands `step()` its scale and found_inf tensors, and
every launch of the step reads them on the device - the kernels multiply each gradient by fp32(1 / fp64(scale)) before
the clip factor, GradScaler.unscale_'s arithmetic, and a non-zero found_inf makes the launches write nothing, step counts
included.  So `.grad` keeps the scaled gradients after `scaler.step`, as with torch's fused optimizers.
`clip_grad_norm(max_norm, scale=scaler._get_scale_async())` clips the scaled gradients at max_norm times the device scale.
The default mode keeps its step counts on the host and keeps GradScaler's unscale_ path.

Learning-rate schedules on the device: `DeviceLRScheduler(opt, kind, **params)` (registered under MMF's scheduler names
warmup_linear, warmup_cosine, multi_step and pythia) keeps LambdaLR's counter on the device and writes each group's
scheduled lr into the fp64 group table the capturable step reads (`mmfb_lr_schedule`), so `sched.step()` is one launch
that a CUDA graph can hold.  While it is attached, stage_hparams copies weight decay, betas and eps but not lr.

Fused non-finite check: `B200AdamW(..., capturable=True, fused_inf_check=True)` with
`clip_grad_norm(c, scaler=scaler)` (or `check_finite(scaler)` without clipping) tests every gradient for inf / NaN in
the library's own launch and hands the flag to GradScaler as the result of an unscale, so `scaler.step` does not run
its foreach check and unscale pass.  It relies on GradScaler internals, as `_get_scale_async` does: the per-optimizer
state `_per_optimizer_states[id(opt)]` with its "stage" (torch.amp.grad_scaler.OptState) and "found_inf_per_device"
entries, and step()'s handling of an optimizer with `_step_supports_amp_scaling` in stage UNSCALED: it reads
found_inf_per_device instead of calling `_check_inf_per_device`, and sets `grad_scale` to None, so the optimizer keeps
the scale tensor itself to unscale inside its kernels.

torch.optim.Adam: with arithmetic="torch" and weight_decay=0 the step is torch.optim.Adam's (amsgrad and maximize off):
AdamW's decoupled decay multiplies the parameter by exactly 1, and the remaining operations - m.lerp_(g, 1-b1),
v.mul_(b2).addcmul_(g, g, 1-b2), p.addcdiv_(m, sqrt(v)/sqrt(1-b2^t) + eps, -lr/(1-b1^t)) - are Adam's.  Pass Adam's
eps (1e-8) explicitly: this class defaults to the reference's 1e-6.  That is how M4C's `optimizer.type: Adam` runs here.
"""
import math
import numbers
import weakref

import torch

from . import engine as E
from . import functional as F
from . import lib
from .registry import registry


def _capturing():
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def _read_steps(steps):
    """ints of a list of step counts (ints or 0-d tensors), with one device read per device"""
    out = list(steps)
    by_dev = {}
    for i, t in enumerate(out):
        if torch.is_tensor(t):
            by_dev.setdefault(t.device, []).append(i)
    for idx in by_dev.values():
        vals = torch.stack([out[i].reshape(()).to(torch.int64) for i in idx]).tolist()
        for i, v in zip(idx, vals):
            out[i] = int(v)
    return [int(v) for v in out]


def _h2d(t, device, out=None):
    """a host tensor on `device` (into `out` if given): one non-blocking copy from pinned memory (the caching host
    allocator keeps the pinned block until the copy has run)"""
    if device.type == "cuda":
        t = t.pin_memory()
    if out is None:
        return t.to(device, non_blocking=True)
    return out.copy_(t, non_blocking=True)


class _CapturablePlan:
    """What a capturable step launches: the slots (a pack's parameter group, or a loose parameter) with their device
    step counts and hyper-parameter table, the pack launches, and the segment table of the loose parameters."""

    def __init__(self, layout_key, device, mode):
        self.layout_key, self.device, self.mode = layout_key, device, mode
        self.packs = []          # (pack, flat state entry, first slot, slots, betas, eps)
        self.loose = []          # (param, slot)
        self.slots = []          # (group index, flags)
        self.table_key, self.table = None, None


def _reference_arithmetic():
    """what `adam_w` resolves to in the reference (optimizers.py:8-14)"""
    try:
        from transformers.optimization import AdamW  # noqa: F401
        return "transformers"
    except Exception:
        return "torch"


class B200AdamW(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True,
                 arithmetic="auto", capturable=False, fused_inf_check=False):
        if lr < 0.0 or eps < 0.0 or not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid AdamW hyper-parameters: lr=%s betas=%s eps=%s" % (lr, betas, eps))
        if arithmetic == "auto":
            arithmetic = _reference_arithmetic()
        if arithmetic not in ("transformers", "torch"):
            raise ValueError("arithmetic must be 'transformers', 'torch' or 'auto'")
        self.arithmetic = arithmetic
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay,
                                      correct_bias=correct_bias))
        self._flat = {}        # id(pack) -> {"pack": weakref, "m", "v", "groups": uint8 [total/8], "gids": {...}}
        self._clip_table = None   # (key of the gradient buffers, F.GradNormTable) of clip_grad_norm
        self._clip_coef = None    # 0-d fp32 CUDA tensor: the coefficient the next step() applies, then drops
        self.capturable = bool(capturable)   # fixed at construction, as the arithmetic mode and correct_bias are
        self._cap = None          # _CapturablePlan of the last capturable step
        if fused_inf_check and not self.capturable:
            raise ValueError("B200AdamW: fused_inf_check=True needs capturable=True (the steps that read GradScaler's "
                             "scale and found_inf on the device)")
        self.fused_inf_check = bool(fused_inf_check)
        self._found_inf = None    # fp32 [1] CUDA: the flag the fused check writes and hands to GradScaler
        self._amp_scale = None    # GradScaler's scale tensor registered by the fused check, read by the next step
        self._lr_sched = None     # the DeviceLRScheduler writing the groups' lr on the device, if one is attached
        if self.capturable:
            # torch.amp.GradScaler.step then passes its scale and found_inf tensors (attributes `grad_scale` and
            # `found_inf` during the call) instead of unscaling on the device and reading found_inf on the host
            self._step_supports_amp_scaling = True

    # ---------------------------------------------------------------------------------------------------------
    def _group_hp(self, group, step):
        b1, b2 = group["betas"]
        lr, wd = float(group["lr"]), float(group["weight_decay"])
        if self.arithmetic == "transformers":
            ss = lr
            if group.get("correct_bias", True):
                ss = lr * math.sqrt(1.0 - b2 ** step) / (1.0 - b1 ** step)
            return {"lr": lr, "weight_decay": wd, "step_size": ss, "bc2_sqrt": 1.0}
        return {"lr": lr, "weight_decay": wd, "step_size": lr / (1.0 - b1 ** step), "bc2_sqrt": math.sqrt(1.0 - b2 ** step)}

    def _torch_update(self, p, g, st, group, grad_scale, coef=None):
        """same arithmetic, operation by operation, on one tensor (parameters outside the packs)"""
        b1, b2 = group["betas"]
        hp = self._group_hp(group, st["step"])
        if coef is not None:                           # the kernel's factor: grad_scale * coef in fp32, then g * factor
            g = g.float() * (coef * grad_scale)
        else:
            g = g.float() * grad_scale if grad_scale != 1.0 else g.float()
        m, v, x = st["exp_avg"], st["exp_avg_sq"], p.data
        if self.arithmetic == "transformers":
            m.mul_(b1).add_(g, alpha=1.0 - b1)
            v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
            x.addcdiv_(m, v.sqrt().add_(group["eps"]), value=-hp["step_size"])
            if hp["weight_decay"] > 0.0:
                x.add_(x, alpha=-hp["lr"] * hp["weight_decay"])
        else:
            x.mul_(1.0 - hp["lr"] * hp["weight_decay"])
            m.lerp_(g, 1.0 - b1)
            v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
            x.addcdiv_(m, (v.sqrt() / hp["bc2_sqrt"]).add_(group["eps"]), value=-hp["step_size"])

    def _flat_state(self, pack, group_of):
        ent = self._flat.get(id(pack))
        if ent is not None and ent["pack"]() is pack and ent["master_ptr"] == pack.master.data_ptr():
            return ent
        m = torch.zeros_like(pack.master, dtype=torch.float32)
        v = torch.zeros_like(m)
        gid = torch.full((pack.total // 8,), 255, dtype=torch.uint8)
        for p, o in zip(pack.params, pack.offsets):
            gi = group_of.get(id(p))
            n8 = (p.numel() + 7) // 8
            if gi is not None:
                gid[o // 8:o // 8 + n8] = gi
            old = self.state.get(p, {})
            mv, vv = m[o:o + p.numel()].view(p.shape), v[o:o + p.numel()].view(p.shape)
            if "exp_avg" in old:                       # state that existed before the pack did (load_state_dict, ...)
                mv.copy_(old["exp_avg"])
                vv.copy_(old["exp_avg_sq"])
            if gi is not None:
                st = self.state[p]
                st.setdefault("step", 0)
                st["exp_avg"], st["exp_avg_sq"] = mv, vv
        frozen = int(gid.max()) == 255
        n_groups = len(self.param_groups) + (1 if frozen else 0)
        if n_groups > 8:
            raise ValueError("B200AdamW: at most 8 hyper-parameter groups per parameter pack (got %d)" % n_groups)
        if frozen:                                     # pack parameters the optimizer was not given: a no-op group
            gid[gid == 255] = len(self.param_groups)
        ent = {"pack": weakref.ref(pack), "m": m, "v": v, "groups": gid.to(pack.master.device), "frozen": frozen,
               "master_ptr": pack.master.data_ptr()}
        self._flat[id(pack)] = ent
        return ent

    def _clip_grads(self):
        """The gradient buffers clip_grad_norm covers, in parameter-group order: a pack's whole flat gradient buffer where
        the optimizer owns every parameter of the pack and each .grad is its slice (the padding between slices is zero),
        each other parameter's .grad on its own."""
        pack_of = {}
        for pack in list(E.ParamPack._live or ()):
            for p in pack.params:
                pack_of[id(p)] = pack
        owned = {id(p) for g in self.param_groups for p in g["params"]}
        grads, seen = [], set()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None or id(p) in seen:
                    continue
                pack = pack_of.get(id(p))
                if (pack is not None and pack.dtype == torch.float32 and pack.intact() and
                        all(id(q) in owned and q.grad is not None and q.grad.dtype == torch.float32 and
                            q.grad.data_ptr() == gp for q, gp in zip(pack.params, pack._gptrs))):
                    grads.append(pack.grad)
                    seen.update(id(q) for q in pack.params)
                else:
                    grads.append(p.grad)
                    seen.add(id(p))
        return grads

    def _grad_table(self):
        """the F.GradNormTable over _clip_grads(), rebuilt (never during capture) when a gradient buffer moves"""
        grads = self._clip_grads()
        if not grads:
            return None
        key = tuple((g.data_ptr(), g.numel(), g.dtype) for g in grads)
        if self._clip_table is None or self._clip_table[0] != key:
            if _capturing():
                raise RuntimeError("B200AdamW.clip_grad_norm: the gradient buffers changed during CUDA-graph capture; "
                                   "call clip_grad_norm once eagerly with the same gradients before capturing")
            self._clip_table = (key, F.grad_norm_table(grads))
            if self.fused_inf_check and (self._found_inf is None or self._found_inf.device != grads[0].device):
                self._found_inf = torch.zeros(1, dtype=torch.float32, device=grads[0].device)
        return self._clip_table[1]

    def _fused_scaler(self, scaler, who):
        """the GradScaler whose non-finite check this call replaces (None when it is disabled); refuses one whose
        optimizer state is past READY, as GradScaler.unscale_ does"""
        if not self.fused_inf_check:
            raise ValueError("B200AdamW.%s: scaler= needs B200AdamW(..., capturable=True, fused_inf_check=True)" % who)
        if not scaler.is_enabled():
            return None
        from torch.amp.grad_scaler import OptState
        if scaler._scale is None:
            raise RuntimeError("B200AdamW.%s: the scaler has no scale yet; call scaler.scale(loss) first" % who)
        if scaler._per_optimizer_states[id(self)]["stage"] is not OptState.READY:
            raise RuntimeError("B200AdamW.%s: the scaler already unscaled or stepped this optimizer since the last "
                               "update()" % who)
        return scaler

    def _register_found_inf(self, scaler):
        """GradScaler's per-optimizer state as after unscale_: found_inf on its device, stage UNSCALED, so that
        scaler.step passes it to step() and scaler.update() reads it, and neither checks the gradients again"""
        from torch.amp.grad_scaler import OptState
        st = scaler._per_optimizer_states[id(self)]
        st["found_inf_per_device"] = {self._found_inf.device: self._found_inf}
        st["stage"] = OptState.UNSCALED
        self._amp_scale = scaler._get_scale_async()

    @torch.no_grad()
    def check_finite(self, scaler):
        """GradScaler's non-finite check of this optimizer's gradients in one library launch pair, for an fp16 update
        without clipping (MMF's clip_gradients false): the flag goes to the scaler as clip_grad_norm(..., scaler=)
        hands it over.  Needs fused_inf_check=True.  Returns the fp32 [1] flag (None when the scaler is disabled)."""
        scaler = self._fused_scaler(scaler, "check_finite")
        if scaler is None:
            return None
        table = self._grad_table()
        if table is None:
            raise RuntimeError("B200AdamW.check_finite: no parameter of the optimizer has a gradient")
        F.grad_check(table, self._found_inf)
        self._register_found_inf(scaler)
        return self._found_inf

    @torch.no_grad()
    def clip_grad_norm(self, max_norm, norm_type=2.0, scale=None, scaler=None):
        """Clips the gradients of every parameter of the optimizer's groups to a global L2 norm of at most max_norm, as
        torch.nn.utils.clip_grad_norm_(params, max_norm) does, and returns the norm before clipping as a 0-d fp32 CUDA
        tensor - without a host synchronisation.  The gradients are not rewritten: the next step() (and only that one)
        multiplies them by min(max_norm / (norm + 1e-6), 1), so read .grad before the step to see unclipped values.
        Non-finite gradients give an inf / NaN norm and the same parameters as torch with error_if_nonfinite=False.
        Only norm_type 2 is supported.  The device table of gradient buffers is rebuilt only when a gradient moves; a
        step captured in a CUDA graph needs one eager call with the same gradients before the capture.
        scale: None or a 0-d fp32 CUDA tensor S (GradScaler's `_get_scale_async()`); the threshold is then max_norm * S,
        computed in fp32 when the kernel runs - MMF's clip of loss-scaled gradients, `max_norm * scaler.get_scale()`,
        without the host read.
        scaler: a torch.amp.GradScaler (needs fused_inf_check=True): the same read of the gradients also tests every
        element for inf / NaN, and the flag is handed to the scaler as unscale_ would (see the module docstring), so
        scaler.step runs no check of its own; scale defaults to the scaler's device scale."""
        if float(norm_type) != 2.0:
            raise ValueError("B200AdamW.clip_grad_norm supports norm_type 2 only, got %s" % (norm_type,))
        if scaler is not None:
            scaler = self._fused_scaler(scaler, "clip_grad_norm")
            if scaler is not None and scale is None:
                scale = scaler._get_scale_async()
        self._clip_coef = None
        table = self._grad_table()
        if table is None:
            return torch.tensor(0.0)
        kw = {} if scale is None else {"max_norm_scale_dev": scale}
        if scaler is None:
            out = F.grad_norm(table, max_norm, norm_type, **kw)
        else:
            out = F.grad_norm_check(table, max_norm, self._found_inf, norm_type, **kw)
            self._register_found_inf(scaler)
        self._clip_coef = out[1]
        return out[0]

    @torch.no_grad()
    def step(self, closure=None, grad_scale=1.0):
        """grad_scale multiplies every gradient first (1 / loss scale, gradient-clipping coefficient).  After
        clip_grad_norm, the gradients are multiplied by grad_scale * (its device-side coefficient) in this step only.
        In capturable mode under GradScaler.step, the scaler's `grad_scale` and `found_inf` tensors (set on the
        optimizer for the call) are read by every launch on the device; see the module docstring."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        coef, self._clip_coef = self._clip_coef, None
        clip = {} if coef is None else {"grad_scale_dev": coef}
        if self.capturable:
            amp = {}                               # set by GradScaler.step for this call only
            for key, attr in (("loss_scale_dev", "grad_scale"), ("found_inf", "found_inf")):
                if getattr(self, attr, None) is not None:
                    amp[key] = getattr(self, attr)
            fused_scale, self._amp_scale = self._amp_scale, None
            if fused_scale is not None and "loss_scale_dev" not in amp:
                amp["loss_scale_dev"] = fused_scale  # GradScaler passes grad_scale=None after the fused check
            self._step_capturable(grad_scale, clip, amp)
            return loss
        group_of = {id(p): gi for gi, g in enumerate(self.param_groups) for p in g["params"]}
        done = set()
        mode = 0 if self.arithmetic == "transformers" else 1
        for pack in list(E.ParamPack._live or ()):
            mine = [p for p in pack.params if id(p) in group_of]
            if not mine or pack.dtype != torch.float32 or not pack.intact():
                continue
            gidx = {id(p): i for i, p in enumerate(pack.params)}
            if not all(p.grad is not None and p.grad.dtype == torch.float32 and
                       p.grad.data_ptr() == pack._gptrs[gidx[id(p)]] for p in mine):
                continue                               # gradients not (all) in the flat buffer: per-parameter path below
            b = {(g["betas"], g["eps"]) for g in self.param_groups if any(id(p) in gidx for p in g["params"])}
            ent = self._flat_state(pack, group_of)
            steps = {}
            for p in mine:
                steps.setdefault(group_of[id(p)], set()).add(int(self.state[p]["step"]))
            if len(b) != 1 or any(len(s) != 1 for s in steps.values()):
                continue                               # mixed betas / eps or step counts inside the pack: per parameter
            (betas, eps), = b
            hps = []
            for gi, g in enumerate(self.param_groups):
                t = next(iter(steps[gi])) + 1 if gi in steps else 1
                hps.append(self._group_hp(g, t))
            if ent["frozen"]:
                hps.append({"lr": 0.0, "weight_decay": 0.0, "step_size": 0.0, "bc2_sqrt": 1.0})
            F.adamw(pack.master, pack.grad, ent["m"], ent["v"], hps, beta1=betas[0], beta2=betas[1], eps=eps, mode=mode,
                    grad_scale=grad_scale, group_of_block=ent["groups"], **clip)
            for p in mine:
                self.state[p]["step"] += 1
                done.add(id(p))
        for group in self.param_groups:
            for p in group["params"]:
                if id(p) in done or p.grad is None:
                    continue
                st = self.state[p]
                if "exp_avg" not in st:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p.data, dtype=torch.float32)
                    st["exp_avg_sq"] = torch.zeros_like(p.data, dtype=torch.float32)
                st["step"] += 1
                self._torch_update(p, p.grad, st, group, grad_scale, coef)
        return loss

    def load_state_dict(self, state_dict):
        """Takes the state of a B200AdamW in either mode or of torch.optim.AdamW / Adam (tensor step counts)."""
        super().load_state_dict(state_dict)
        self._clip_coef = None
        self._flat = {}                                # re-adopt the loaded per-parameter tensors into flat buffers
        if self.capturable:
            self._cap = None
            for st in self.state.values():
                if torch.is_tensor(st.get("step")):
                    st["step"] = int(st["step"].item())

    def state_dict(self):
        """torch's layout; in capturable mode the device step counts are read back (once) and reported as ints."""
        sd = super().state_dict()
        if not self.capturable:
            return sd
        state = {k: dict(v) for k, v in sd["state"].items()}
        keys = [k for k, v in state.items() if "step" in v]
        for k, v in zip(keys, _read_steps([state[k]["step"] for k in keys])):
            state[k]["step"] = v
        sd["state"] = state
        return sd

    # ---------------------------------------------------------------------------------------------------------
    # capturable mode
    def _capturable_plan(self):
        """The plan of the next capturable step: rebuilt when the stepped parameters or the packs change (this reads the
        step counts on the host), its segment table when a loose gradient or state tensor moves; neither may happen
        during stream capture."""
        group_of = {id(p): gi for gi, g in enumerate(self.param_groups) for p in g["params"]}
        stepped, seen = [], set()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is not None and id(p) not in seen:
                    seen.add(id(p))
                    stepped.append(p)
        if not stepped:
            return None
        order = {id(p): i for i, p in enumerate(stepped)}
        packs = []
        for pack in list(E.ParamPack._live or ()):
            owned = [p for p in pack.params if id(p) in group_of]
            mine = [p for p in owned if id(p) in seen]
            if not mine:
                continue
            ok = (pack.dtype == torch.float32 and pack.intact() and len(mine) == len(owned) and
                  all(p.grad.dtype == torch.float32 and p.grad.data_ptr() == pack._gptrs[pack._index[id(p)]]
                      for p in mine) and
                  len({(self.param_groups[group_of[id(p)]]["betas"], self.param_groups[group_of[id(p)]]["eps"])
                       for p in mine}) == 1)
            packs.append((min(order[id(p)] for p in mine), pack, mine, ok))
        packs.sort(key=lambda t: t[0])
        layout_key = (tuple(id(p) for p in stepped), tuple((id(pk), pk.master.data_ptr(), ok) for _, pk, _, ok in packs))
        plan = self._cap
        if plan is None or plan.layout_key != layout_key:
            if _capturing():
                raise RuntimeError("B200AdamW(capturable=True): the parameters with gradients changed during CUDA-graph "
                                   "capture; run one eager step with the same gradients before capturing")
            plan = self._cap = self._build_layout(layout_key, stepped, packs, group_of)
        table_key = tuple((p.data_ptr(), p.grad.data_ptr(), self.state[p]["exp_avg"].data_ptr(),
                           self.state[p]["exp_avg_sq"].data_ptr()) for p, _ in plan.loose)
        if plan.loose and plan.table_key != table_key:
            if _capturing():
                raise RuntimeError("B200AdamW(capturable=True): a gradient or optimizer-state buffer moved during "
                                   "CUDA-graph capture; run one eager step with the same gradients before capturing")
            for p, _ in plan.loose:
                if not p.grad.is_contiguous() or p.grad.dtype != torch.float32:
                    raise ValueError("B200AdamW(capturable=True): gradients must be contiguous fp32 tensors; a parameter "
                                     "of shape %s has a %s%s gradient" % (tuple(p.shape), p.grad.dtype,
                                                                          "" if p.grad.is_contiguous() else
                                                                          " non-contiguous"))
            plan.table = F.adamw_segment_table([(p.data, p.grad, self.state[p]["exp_avg"], self.state[p]["exp_avg_sq"], s)
                                                for p, s in plan.loose])
            plan.table_key = table_key
        return plan

    def _build_layout(self, layout_key, stepped, packs, group_of):
        device = stepped[0].device
        plan = _CapturablePlan(layout_key, device, 0 if self.arithmetic == "transformers" else 1)
        steps = dict(zip((id(p) for p in stepped), _read_steps([self.state[p].get("step", 0) if p in self.state else 0
                                                                  for p in stepped])))
        cb = lambda gi: lib.MMFB_ADAMW_SLOT_CORRECT_BIAS if self.param_groups[gi].get("correct_bias", True) else 0
        counts, slot_of = [], {}
        in_pack = set()
        for _, pack, mine, ok in packs:
            by_group = {}
            for p in mine:
                by_group.setdefault(group_of[id(p)], set()).add(steps[id(p)])
            if not ok or any(len(v) != 1 for v in by_group.values()):
                continue                               # mixed step counts or betas: its parameters go to the segments
            ent = self._flat_state(pack, group_of)
            s0, g0 = len(plan.slots), min(by_group)
            for gi in range(len(self.param_groups)):
                if gi in by_group:
                    plan.slots.append((gi, cb(gi)))
                    counts.append(next(iter(by_group[gi])))
                else:                                  # a group without parameters here: its entry is never read
                    plan.slots.append((g0, lib.MMFB_ADAMW_SLOT_FROZEN))
                    counts.append(0)
            if ent["frozen"]:                          # pack parameters the optimizer was not given
                plan.slots.append((g0, lib.MMFB_ADAMW_SLOT_FROZEN))
                counts.append(0)
            g = self.param_groups[g0]
            plan.packs.append((pack, ent, s0, len(plan.slots) - s0, g["betas"], g["eps"]))
            for p in mine:
                slot_of[id(p)] = s0 + group_of[id(p)]
                in_pack.add(id(p))
        for p in stepped:
            if id(p) in in_pack:
                continue
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise ValueError("B200AdamW(capturable=True): parameters outside the engine's packs must be contiguous "
                                 "fp32 tensors; got a %s%s parameter of shape %s"
                                 % ("" if p.is_contiguous() else "non-contiguous ", p.dtype, tuple(p.shape)))
            st = self.state[p]
            for k in ("exp_avg", "exp_avg_sq"):
                t = st.get(k)
                if t is None or t.dtype != torch.float32 or not t.is_contiguous() or t.device != p.device:
                    st[k] = torch.zeros_like(p.data, dtype=torch.float32) if t is None else \
                        t.to(device=p.device, dtype=torch.float32).contiguous()
            slot_of[id(p)] = len(plan.slots)
            plan.loose.append((p, len(plan.slots)))
            plan.slots.append((group_of[id(p)], cb(group_of[id(p)])))
            counts.append(steps[id(p)])
        plan.step = _h2d(torch.tensor(counts, dtype=torch.int64), device)
        plan.slot_table = F.adamw_slot_table(plan.slots, device)
        plan.hp = torch.zeros(len(plan.slots), lib.ADAMW_HP_FLOATS, dtype=torch.float32, device=device)
        if self._lr_sched is not None:                 # the scheduler's table: its lr column is written on the device
            plan.groups = self._lr_sched._table_for(self, device)
        else:
            plan.groups = torch.zeros(len(self.param_groups), lib.ADAMW_GROUP_HP_DOUBLES, dtype=torch.float64,
                                      device=device)
        for p in stepped:
            self.state[p]["step"] = plan.step[slot_of[id(p)]]
        return plan

    def _group_values(self):
        """the staged table: (lr, weight_decay, beta1, beta2, eps) of every group, fp64"""
        return torch.tensor([[float(g["lr"]), float(g["weight_decay"]), float(g["betas"][0]), float(g["betas"][1]),
                              float(g["eps"])] for g in self.param_groups], dtype=torch.float64)

    def stage_hparams(self, plan=None):
        """Copy the groups' current lr / weight_decay / betas / eps to the device table the next (eager or replayed)
        capturable step reads: one non-blocking copy from pinned memory on the current stream.  An eager step() does
        this itself; GraphedStep does it before every replay.  With a DeviceLRScheduler attached the lr is the one
        the scheduler wrote on the device and is not copied (one copy per group of the other four values)."""
        plan = plan if plan is not None else self._cap
        if plan is None:
            return
        if self._lr_sched is None:
            _h2d(self._group_values(), plan.device, out=plan.groups)
            return
        # a DeviceLRScheduler owns the lr column: one copy per group of its weight_decay, beta1, beta2, eps
        host = self._group_values()[:, 1:].contiguous()
        if plan.device.type == "cuda":
            host = host.pin_memory()
        for g in range(host.shape[0]):
            plan.groups[g, 1:].copy_(host[g], non_blocking=True)

    def _step_capturable(self, grad_scale, clip, amp):
        plan = self._capturable_plan()
        if plan is None:
            return
        if not _capturing():
            self.stage_hparams(plan)
        F.adamw_hparams(plan.groups, plan.slot_table, plan.step, plan.hp, plan.mode,
                        **({"found_inf": amp["found_inf"]} if "found_inf" in amp else {}))
        for pack, ent, s0, n, betas, eps in plan.packs:
            F.adamw(pack.master, pack.grad, ent["m"], ent["v"], None, beta1=betas[0], beta2=betas[1], eps=eps,
                    mode=plan.mode, grad_scale=grad_scale, group_of_block=ent["groups"], hp_dev=plan.hp[s0:s0 + n],
                    **clip, **amp)
        if plan.loose:
            F.adamw_segments(plan.table, plan.hp, mode=plan.mode, grad_scale=grad_scale, **clip, **amp)


# ---------------------------------------------------------------------------------------------------------------------
# learning-rate schedules on the device
_SCHEDULE_KINDS = {"warmup_linear": lib.MMFB_LR_WARMUP_LINEAR, "warmup_cosine": lib.MMFB_LR_WARMUP_COSINE,
                   "multi_step": lib.MMFB_LR_MULTI_STEP, "pythia": lib.MMFB_LR_PYTHIA}


def _cfg(obj, key):
    """obj.key or obj[key] (an omegaconf / namespace config or a dict); KeyError when it has neither"""
    if isinstance(obj, dict):
        return obj[key]
    try:
        return getattr(obj, key)
    except AttributeError:
        raise KeyError(key)


def _milestones(lr_steps, who):
    steps = list(lr_steps)
    if len(steps) > lib.MMFB_LR_MAX_MILESTONES:
        raise ValueError("%s: at most %d lr_steps (got %d)" % (who, lib.MMFB_LR_MAX_MILESTONES, len(steps)))
    out = []
    for x in steps:
        if isinstance(x, bool) or not (isinstance(x, numbers.Integral) or (isinstance(x, float) and x.is_integer())):
            raise ValueError("%s: lr_steps must be whole update counts, got %r" % (who, x))
        out.append(int(x))
    return out


def schedule_desc(kind, num_warmup_steps=None, num_training_steps=None, num_cycles=0.5, use_warmup=False, lr_steps=(),
                  lr_ratio=0.1, warmup_iterations=0, warmup_factor=1.0):
    """The lib.LrScheduleDesc of one of MMF's schedules (mmf/modules/schedulers.py), with the host's powers
    lr_ratio ** i.  use_warmup counts only when it `is True`, as in the reference's tests."""
    if kind not in _SCHEDULE_KINDS:
        raise ValueError("DeviceLRScheduler: unknown schedule %r (MMF's are %s)" % (kind, ", ".join(_SCHEDULE_KINDS)))
    d = lib.LrScheduleDesc()
    d.kind = _SCHEDULE_KINDS[kind]
    if kind in ("warmup_linear", "warmup_cosine"):
        if num_warmup_steps is None or num_training_steps is None:
            raise TypeError("DeviceLRScheduler(%r) needs num_warmup_steps and num_training_steps" % kind)
        d.warmup_iterations, d.total_steps = int(num_warmup_steps), int(num_training_steps)
        d.num_cycles = float(num_cycles)
        return d
    steps = _milestones(lr_steps, "DeviceLRScheduler(%r)" % kind)
    d.use_warmup = 1 if use_warmup is True else 0
    d.warmup_iterations = int(warmup_iterations) if use_warmup else 0
    if d.use_warmup and d.warmup_iterations < 1:
        raise ValueError("DeviceLRScheduler(%r): use_warmup needs warmup_iterations >= 1 (the reference divides by it)"
                         % kind)
    d.warmup_factor = float(warmup_factor)
    d.n_lr_steps = len(steps)
    for i, x in enumerate(steps):
        d.lr_steps[i] = x
    for i in range(len(steps) + 1):
        d.ratio_pow[i] = float(lr_ratio ** i)          # pow(lr_ratio, idx) of the reference, on the host
    return d


class DeviceLRScheduler:
    """MMF's learning-rate schedulers with LambdaLR's counter and arithmetic on the device, for a capturable B200AdamW:

        sched = DeviceLRScheduler(opt, "warmup_linear", num_warmup_steps=2000, num_training_steps=88000)
        ... opt.step(); sched.step()        # or GraphedStep(..., optimizer=opt, lr_scheduler=sched)

    kind and the keyword arguments are those of the reference's schedulers (mmf/modules/schedulers.py): warmup_linear
    and warmup_cosine (transformers' get_*_schedule_with_warmup: num_warmup_steps, num_training_steps, num_cycles),
    multi_step (use_warmup, lr_steps, lr_ratio, warmup_iterations, warmup_factor) and pythia (lr_lambda_update over
    the registered config's training.* values).  The counter is LambdaLR's last_epoch, an int64 on the device; step()
    is one launch that advances it and writes every group's base_lr * f(last_epoch) into the fp64 group table the
    optimizer's next step reads, so it can be captured.  As LambdaLR does on construction, the lr is the schedule at
    step 0 before the first step().  The counter is separate from the AdamW step counts: it advances on updates that
    GradScaler skips, as MMF's trainer steps its scheduler on every update.

    LambdaLR's surface: step(), get_last_lr() (one device read), last_epoch (one device read), state_dict() and
    load_state_dict(), which resumes at the saved counter in place (graphs captured with this scheduler stay valid).
    The groups' "lr" in param_groups stays the base lr ("initial_lr"): the scheduled lr lives on the device.  One
    schedule for all groups, as LambdaLR with one lambda."""

    def __init__(self, optimizer, kind, **params):
        if not isinstance(optimizer, B200AdamW) or not optimizer.capturable:
            raise TypeError("DeviceLRScheduler: the optimizer must be mmf_b200.optim.B200AdamW(..., capturable=True), "
                            "whose steps read the lr from the device table this scheduler writes; use torch's "
                            "LambdaLR schedulers with other optimizers")
        if optimizer._lr_sched is not None:
            raise RuntimeError("DeviceLRScheduler: the optimizer already has a device scheduler attached")
        if kind == "pythia":
            if params:
                raise TypeError("DeviceLRScheduler('pythia') reads training.* from the registered config, as the "
                                "reference does; got arguments %s" % sorted(params))
            cfg = registry.get("config")
            if cfg is None:
                raise RuntimeError("DeviceLRScheduler('pythia'): no config registered (registry.register('config', ...))")
            tr = _cfg(cfg, "training")
            params = {k: _cfg(tr, k) for k in ("use_warmup", "lr_steps", "lr_ratio", "warmup_iterations",
                                                "warmup_factor")}
        elif kind == "multi_step":
            for k in ("use_warmup", "lr_steps", "lr_ratio", "warmup_factor") + \
                    (("warmup_iterations",) if params.get("use_warmup") else ()):
                if k not in params:
                    raise TypeError("DeviceLRScheduler('multi_step') needs %s" % k)
            w = params["warmup_iterations"] if params["use_warmup"] else 0
            if not params["lr_steps"] or not w < params["lr_steps"][0]:
                raise ValueError("DeviceLRScheduler('multi_step'): warmup_iterations must be below the first of lr_steps")
        self.kind, self.params = kind, dict(params)
        self.desc = schedule_desc(kind, **params)
        self.optimizer = optimizer
        dev = next((p.device for g in optimizer.param_groups for p in g["params"]), None)
        if dev is None or dev.type != "cuda":
            raise RuntimeError("DeviceLRScheduler: the optimizer's parameters must be on a CUDA device")
        self.device = dev
        self.base_lrs = [float(g.setdefault("initial_lr", g["lr"])) for g in optimizer.param_groups]
        self.base_lr = _h2d(torch.tensor(self.base_lrs, dtype=torch.float64), dev)
        self.counter = torch.zeros(1, dtype=torch.int64, device=dev)
        plan = optimizer._cap
        if plan is not None and plan.groups.shape[0] == len(self.base_lrs):
            self.table = plan.groups                   # graphs captured before this read this table: keep it
        else:
            self.table = torch.zeros(len(self.base_lrs), lib.ADAMW_GROUP_HP_DOUBLES, dtype=torch.float64, device=dev)
        optimizer._lr_sched = self
        self._launch(advance=False)

    def _table_for(self, optimizer, device):
        if self.table.shape[0] != len(optimizer.param_groups) or self.table.device != device:
            raise RuntimeError("DeviceLRScheduler: the optimizer's parameter groups changed since the scheduler was "
                               "built; build a new scheduler")
        return self.table

    def _launch(self, advance):
        F.lr_schedule(self.counter, self.base_lr, self.table, self.desc, advance, lr_stride=lib.ADAMW_GROUP_HP_DOUBLES)

    def step(self):
        """advance the counter and write the next lr of every group, on the device (capturable)"""
        self._launch(advance=True)

    def refresh(self):
        """rewrite the groups' lr from the current counter (after the counter was set in place)"""
        self._launch(advance=False)

    @property
    def last_epoch(self):
        return int(self.counter.item())

    def get_last_lr(self):
        """the lr of every group that the next optimizer step uses, read from the device"""
        return self.table[:, 0].tolist()

    def state_dict(self):
        return {"kind": self.kind, "params": dict(self.params), "base_lrs": list(self.base_lrs),
                "last_epoch": self.last_epoch}

    def load_state_dict(self, state_dict):
        if state_dict["kind"] != self.kind:
            raise ValueError("DeviceLRScheduler.load_state_dict: a %r state for a %r scheduler"
                             % (state_dict["kind"], self.kind))
        if len(state_dict["base_lrs"]) != len(self.base_lrs):
            raise ValueError("DeviceLRScheduler.load_state_dict: %d base lrs for %d groups"
                             % (len(state_dict["base_lrs"]), len(self.base_lrs)))
        self.base_lrs = [float(x) for x in state_dict["base_lrs"]]
        _h2d(torch.tensor(self.base_lrs, dtype=torch.float64), self.device, out=self.base_lr)
        _h2d(torch.tensor([int(state_dict["last_epoch"])], dtype=torch.int64), self.device, out=self.counter)
        self.refresh()


def _registered(kind, name):
    def __init__(self, optimizer, *args, **kwargs):
        if args:
            raise TypeError("%s takes keyword arguments only (MMF's scheduler.params)" % name)
        DeviceLRScheduler.__init__(self, optimizer, kind, **kwargs)
    cls = type(name, (DeviceLRScheduler,), {"__init__": __init__, "__doc__": "DeviceLRScheduler(optimizer, %r, ...)"
                                                                           % kind})
    return registry.register_scheduler(kind)(cls)


DeviceWarmupLinearScheduler = _registered("warmup_linear", "DeviceWarmupLinearScheduler")
DeviceWarmupCosineScheduler = _registered("warmup_cosine", "DeviceWarmupCosineScheduler")
DeviceMultiStepScheduler = _registered("multi_step", "DeviceMultiStepScheduler")
DevicePythiaScheduler = _registered("pythia", "DevicePythiaScheduler")
