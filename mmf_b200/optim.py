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

torch.optim.Adam: with arithmetic="torch" and weight_decay=0 the step is torch.optim.Adam's (amsgrad and maximize off):
AdamW's decoupled decay multiplies the parameter by exactly 1, and the remaining operations - m.lerp_(g, 1-b1),
v.mul_(b2).addcmul_(g, g, 1-b2), p.addcdiv_(m, sqrt(v)/sqrt(1-b2^t) + eps, -lr/(1-b1^t)) - are Adam's.  Pass Adam's
eps (1e-8) explicitly: this class defaults to the reference's 1e-6.  That is how M4C's `optimizer.type: Adam` runs here.
"""
import math
import weakref

import torch

from . import engine as E
from . import functional as F


def _reference_arithmetic():
    """what `adam_w` resolves to in the reference (optimizers.py:8-14)"""
    try:
        from transformers.optimization import AdamW  # noqa: F401
        return "transformers"
    except Exception:
        return "torch"


class B200AdamW(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True,
                 arithmetic="auto"):
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

    @torch.no_grad()
    def clip_grad_norm(self, max_norm, norm_type=2.0):
        """Clips the gradients of every parameter of the optimizer's groups to a global L2 norm of at most max_norm, as
        torch.nn.utils.clip_grad_norm_(params, max_norm) does, and returns the norm before clipping as a 0-d fp32 CUDA
        tensor - without a host synchronisation.  The gradients are not rewritten: the next step() (and only that one)
        multiplies them by min(max_norm / (norm + 1e-6), 1), so read .grad before the step to see unclipped values.
        Non-finite gradients give an inf / NaN norm and the same parameters as torch with error_if_nonfinite=False.
        Only norm_type 2 is supported.  The device table of gradient buffers is rebuilt only when a gradient moves; a
        step captured in a CUDA graph needs one eager call with the same gradients before the capture."""
        if float(norm_type) != 2.0:
            raise ValueError("B200AdamW.clip_grad_norm supports norm_type 2 only, got %s" % (norm_type,))
        self._clip_coef = None
        grads = self._clip_grads()
        if not grads:
            return torch.tensor(0.0)
        key = tuple((g.data_ptr(), g.numel(), g.dtype) for g in grads)
        if self._clip_table is None or self._clip_table[0] != key:
            if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
                raise RuntimeError("B200AdamW.clip_grad_norm: the gradient buffers changed during CUDA-graph capture; "
                                   "call clip_grad_norm once eagerly with the same gradients before capturing")
            self._clip_table = (key, F.grad_norm_table(grads))
        out = F.grad_norm(self._clip_table[1], max_norm, norm_type)
        self._clip_coef = out[1]
        return out[0]

    @torch.no_grad()
    def step(self, closure=None, grad_scale=1.0):
        """grad_scale multiplies every gradient first (1 / loss scale, gradient-clipping coefficient).  After
        clip_grad_norm, the gradients are multiplied by grad_scale * (its device-side coefficient) in this step only."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        coef, self._clip_coef = self._clip_coef, None
        clip = {} if coef is None else {"grad_scale_dev": coef}
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
        super().load_state_dict(state_dict)
        self._clip_coef = None
        self._flat = {}                                # re-adopt the loaded per-parameter tensors into flat buffers
