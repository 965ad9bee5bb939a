"""Whole-step CUDA graph for the small configurations (BASELINE.json configs[0]: MMBT, batch 2, 40 kernel launches of a few
microseconds each - the host cannot issue them as fast as the GPU retires them).

    step = GraphedStep(model, loss_fn, example_batch)      # warm-up, then capture of forward + backward
    loss = step(batch)                                      # copies `batch` into the static inputs, replays the graph

The graph holds the library's kernels exactly as an eager step launches them (same C ABI calls, recorded by stream capture);
nothing is traced or compiled.  What a capture freezes and how it is kept correct:
  * dropout: the host-side (seed, offset) of every keep-bit draw is frozen, so the graph increments a device-resident step
    counter that the generator mixes into its Philox counter (functional.dropout_epoch): every replay draws fresh masks;
  * gradients: captured with `.grad` unset, so the flat gradient buffers are zeroed inside the graph and the parameters'
    `.grad` are views of them afterwards - an optimizer sees fresh gradients after every replay;
  * inputs: static device tensors, refreshed by `copy_` on the replay stream (shapes are fixed at capture);
  * deterministic mode: the graph records the reductions that torch.use_deterministic_algorithms selected AT CAPTURE
    (mmf_b200.functional reads the flag per call): a step captured under the flag replays the ordered kernels, and one
    captured without it replays the atomic ones, whatever the flag says at replay.  Capture under the mode you want;
  * masked-LM losses: their labelled rows are a data-dependent number, found on the host in an eager step.  Inside
    `static_rows()` the heads (mmf_b200.heads.masked_lm_loss "fused" / "masked", mmf_b200.mmft.MLMHead) select and count
    them on the device instead and bound the vocabulary-sized kernels by that count, so the step can be captured;
    `GraphedStep(..., static_rows=True)` captures under it.  Such a step returns no MLM logits;
  * skip-padding: a single-stream encoder with skip_padding set plans its packing on the host in an eager step.  Inside
    `static_rows()` it plans it on the device at the capacity B*S (mmf_b200.modules._plan_packing_static) and bounds
    every GEMM, LayerNorm and column sum of its layers by the device token count, so that step can be captured too.
    Runners switched on with set_skip_padding(..., device_plan=True) do the same for M4C's causal tail (pack_tail) and
    the ViLBERT / LXMERT streams (pack_streams): one kernel (functional.plan_packing) plans every stream of the call.
  * the optimizer: `GraphedStep(..., optimizer=opt, max_grad_norm=c)` with a `B200AdamW(..., capturable=True)` captures
    the whole step - gradients zeroed in place, forward, backward, `opt.clip_grad_norm(c)`, `opt.step()`.  The step
    counts and bias corrections advance on the device; the groups' lr / weight_decay / betas / eps are staged from
    `param_groups` before every replay, so a learning-rate scheduler stepped between replays takes effect.  What the
    capture freezes: which parameters have gradients, the gradient and state buffers (they keep their storage from the
    warm-up on), `grad_scale` 1, correct_bias and the arithmetic mode.  The warm-up steps are undone, so capturing does
    not change the parameters or the optimizer state;
  * loss scaling: `GraphedStep(..., optimizer=opt, scaler=torch.amp.GradScaler("cuda"))` captures MMF's fp16 update -
    `scaler.scale(loss).backward()`, `opt.clip_grad_norm(c, scale=scaler._get_scale_async())`, `scaler.step(opt)`,
    `scaler.update()`.  The capturable optimizer reads the scale and found_inf on the device, and GradScaler's
    non-finite check and scale update are device ops, so a step with non-finite gradients is skipped and the scale
    backs off or grows inside the replay.  What the capture freezes: the scaler's scale and growth-tracker tensors and
    its factors and interval.  Its warm-up updates are undone too;
  * learning-rate schedules: `GraphedStep(..., optimizer=opt, lr_scheduler=mmf_b200.optim.DeviceLRScheduler(opt, ...))`
    ends every captured update with the scheduler's device step, so the lr needs no host work between replays; the
    schedule descriptor (kind, warm-up, milestones, the powers of lr_ratio) and the base lrs' buffer are frozen;
  * gradient accumulation: `GraphedStep(..., optimizer=opt, update_frequency=K)` runs MMF's `training.update_frequency`
    (mmf/trainers/core/training_loop.py: zero_grad, K backwards of losses not divided by K, clip, step).  It
    captures a micro-batch graph (dropout epoch, forward, backward, no zeroing: every gradient adds in place) and an
    update graph (clip, step, or scaler.step and scaler.update) in one memory pool; each call replays the micro graph,
    the K-th of a group replays the update too, and `finish_update()` updates after a partial group.  The gradients are
    zeroed in place (a graph of one `_foreach_zero_`) before the first micro-batch of a group, never set to None: the
    optimizer's device tables point at them.  After an update `.grad` holds the group's sum, as after MMF's eager update.  It freezes what the one-graph step
    freezes, and every micro-batch draws fresh dropout masks and counts its own static rows;
  * host draws: a model that draws its task on the host in every forward (UNITER) is captured by GraphedTaskSteps, one
    graph per task, with the draws made on the host before each replay;
  * evaluation: GraphedForward(model.eval(), batch) captures the eval forward `model(batch)` under torch.no_grad() -
    scores and losses, for M4C and the M4C captioner every greedy decoding step - and returns the captured output,
    overwritten by the next call.  It refuses what GraphedStep refuses, and a model in training mode;
The reference has no counterpart (its trainer launches eagerly, mmf/trainers/core/training_loop.py:185-213); this is the
answer to SURVEY.md 8a's "at T = R = 36 everything is launch-bound"."""
import contextlib
import numbers
import random

import numpy as np
import torch

from . import functional as F

_STATIC_ROWS = [0]      # depth of nested static_rows() contexts


@contextlib.contextmanager
def static_rows():
    """Run the masked-LM heads in static-rows mode while the context is open: the labelled rows are selected on the device
    into a fixed capacity (every row of the labels), the vocabulary GEMM and loss are bounded by the device count, the loss
    is the same mean cross-entropy and `logits` is None.  Nothing is read on the host, so the step can be captured.  A
    batch with no labelled row gives a loss of exactly 0 and zero gradients.
    Single-stream skip_padding encoders (calls without a causal tail) plan their packing on the device in the same way
    (mmf_b200.modules.run_bert_encoder), and so do causal-tail and two-stream encoders whose runner has `device_plan`
    set (patch.set_skip_padding(..., device_plan=True))."""
    _STATIC_ROWS[0] += 1
    try:
        yield
    finally:
        _STATIC_ROWS[0] -= 1


_static_rows_context = static_rows     # GraphedStep's `static_rows` argument shadows the name


def static_rows_active():
    """whether a static_rows() context is open (read by the masked-LM heads on every forward)"""
    return _STATIC_ROWS[0] > 0


def _map(fn, x):
    if isinstance(x, dict):
        return {k: _map(fn, v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_map(fn, v) for v in x)
    return fn(x) if torch.is_tensor(x) else x


def _copy_into(dst, src):
    if isinstance(dst, dict):
        for k in dst:
            _copy_into(dst[k], src[k])
    elif isinstance(dst, (list, tuple)):
        for d, s in zip(dst, src):
            _copy_into(d, s)
    elif torch.is_tensor(dst):
        dst.copy_(src, non_blocking=True)


class GraphedStep:
    def __init__(self, model, loss_fn, example_batch, warmup=3, static_rows=False, optimizer=None, max_grad_norm=None,
                 scaler=None, update_frequency=1, lr_scheduler=None):
        """loss_fn(batch) -> scalar loss; `example_batch`: (nested dict / list of) CUDA tensors with the shapes of every later
        batch.  The model must be in the mode (train / eval) it will be replayed in.

        The batch must carry every input the forward would otherwise build from a Python value: a tensor made from a
        host value during capture is frozen into the graph or is a copy the capture refuses.  ViLT's `is_correct`, for
        one, is made by torch.tensor when the batch lacks it.

        static_rows=True: warm-up and capture run inside static_rows(), so a model whose only refusal is the masked-LM
        row gather (it declares `static_rows_capturable = True`: VinVL, ViLT with an `mlm` head) is accepted, and LXMERT's
        masked-LM loss is captured too.  Single-stream skip_padding encoders (patch.set_skip_padding(model)) plan their
        packing on the device there and are captured as well, at a fixed capacity of every row of the batch.  Those with
        `pack_tail` (set_skip_padding(..., causal=True)) and two-stream encoders with `pack_streams` are captured too
        when they were switched on with set_skip_padding(..., device_plan=True), and refused otherwise.
        Opt-in because the replayed step differs from an eager one: no MLM logits.

        optimizer: a B200AdamW(..., capturable=True) over the model's parameters; the graph then holds the whole training
        step: gradients zeroed, forward, backward, optimizer.clip_grad_norm(max_grad_norm) when max_grad_norm is set, and
        optimizer.step().  Each call stages the groups' current hyper-parameters, then replays; afterwards `.grad` holds
        the step's unclipped gradients, as after an eager step.

        scaler: a torch.amp.GradScaler (needs optimizer=); the graph then runs MMF's fp16 update: zero the gradients,
        loss_fn (put the autocast inside it, with cache_enabled=False as torch requires under capture),
        scaler.scale(loss).backward(), optimizer.clip_grad_norm(max_grad_norm, scale=<the device scale>) when
        max_grad_norm is set, scaler.step(optimizer), scaler.update().  A call returns the unscaled loss; afterwards
        `.grad` holds the scaled gradients (the optimizer unscales inside its kernels), and the scaler's scale and growth
        tracker are those of the replayed update.

        update_frequency: K > 1 (needs optimizer=) accumulates the gradients of K calls and updates once, as MMF's
        `training.update_frequency: K` does; the loss is not divided by K.  Two graphs are captured in one memory pool:
        a micro-batch graph (advance the dropout epoch, loss_fn, the backward - scaled with a scaler - adding into the
        gradients in place) and an update graph (the clip and optimizer or scaler calls above), with a small graph
        that zeroes the gradients in place.  Each call copies the batch, replays the micro graph and returns that
        micro-batch's loss, valid until the next call; the first call of a group first replays the zeroing, and the
        K-th stages the hyper-parameters and replays the update.  `pending` counts the
        micro-batches since the last update, and finish_update() updates after a partial group (MMF's last update of a
        run).  After an update `.grad` holds the group's summed gradients, unclipped and, with a scaler, scaled.
        Construction leaves the gradients zeroed.  K = 1 is the one-graph step above.

        lr_scheduler: a mmf_b200.optim.DeviceLRScheduler attached to `optimizer`; the update then ends with
        lr_scheduler.step() (after scaler.update() with a scaler), MMF's scheduler step, inside the graph: the next
        update's lr is computed on the device and the replay needs no host work for it.  It advances once per update
        (once per K calls), skipped fp16 updates included.  Warm-up and capture leave its counter as they found it.

        With a scaler and B200AdamW(..., fused_inf_check=True) the update checks the gradients for inf / NaN in the
        library's clip launch (optimizer.clip_grad_norm(max_grad_norm, scaler=scaler)), or in its check-only launch
        (optimizer.check_finite(scaler)) without max_grad_norm, instead of GradScaler's foreach pass."""
        _check_optimizer("GraphedStep", optimizer, max_grad_norm)
        _check_scheduler("GraphedStep", optimizer, lr_scheduler)
        if scaler is not None and optimizer is None:
            raise ValueError("GraphedStep: scaler= unscales and skips inside the captured optimizer step; pass "
                             "optimizer=B200AdamW(..., capturable=True) as well, or scale and step eagerly after each "
                             "replay")
        if not isinstance(update_frequency, numbers.Integral) or isinstance(update_frequency, bool) or \
                update_frequency < 1:
            raise ValueError("GraphedStep: update_frequency must be a positive int (MMF's training.update_frequency), "
                             "got %r" % (update_frequency,))
        if update_frequency > 1 and optimizer is None:
            raise ValueError("GraphedStep: update_frequency=%d accumulates gradients over %d calls and updates inside "
                             "the captured optimizer step; pass optimizer=B200AdamW(..., capturable=True) as well "
                             "(without one, every replay starts from fresh gradients)"
                             % (update_frequency, update_frequency))
        _check_capturable("GraphedStep", model, static_rows)
        self.model, self.loss_fn = model, loss_fn
        self.optimizer, self.max_grad_norm, self.scaler = optimizer, max_grad_norm, scaler
        self.lr_scheduler = lr_scheduler
        self.update_frequency = int(update_frequency)
        self.pending = 0          # micro-batches accumulated since the last update (update_frequency > 1)
        with _static_rows_context() if static_rows else contextlib.nullcontext():
            self._capture(model, loss_fn, example_batch, warmup)

    def _capture(self, model, loss_fn, example_batch, warmup):
        self.static = _map(lambda t: t.detach().clone(), example_batch)
        dev = next(t for t in _flatten(self.static) if t.is_cuda).device
        self.epoch = F.dropout_epoch(dev, create=True)
        opt = self.optimizer
        saved = _save_optimizer(opt) if opt is not None else None
        saved_scaler = _save_scaler(self.scaler) if self.scaler is not None else None
        saved_counter = self.lr_scheduler.counter.clone() if self.lr_scheduler is not None else None
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):              # lazy engine state, kernel attributes, library work buffers
                self._zero_grads()
                self.epoch.add_(1)
                self._backward(loss_fn(self.static))
                if opt is not None:                      # builds the optimizer's device tables on these gradients
                    self._optimizer_step()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        if opt is None:
            model.zero_grad(set_to_none=True)
        else:
            _restore_optimizer(opt, saved)
            if self.scaler is not None:
                _restore_scaler(self.scaler, saved_scaler)
            if self.lr_scheduler is not None:
                _restore_scheduler(self.lr_scheduler, saved_counter)
            if self.update_frequency > 1:
                self._zero_grads()
            torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        if self.update_frequency > 1:
            self._capture_accumulating(loss_fn, side)
            return
        # captured on the warm-up stream: autograd binds every parameter's gradient accumulator to the stream that was current
        # when the accumulator was created, i.e. this one, as long as no autograd graph from an earlier eager step on another
        # stream is still alive (it would keep the old accumulators - and their stream - in use)
        with torch.cuda.graph(self.graph, stream=side):
            if opt is not None:
                self._zero_grads()
            self.epoch.add_(1)
            self.loss = loss_fn(self.static)
            self._backward(self.loss)
            if opt is not None:
                self._optimizer_step()
        self._plan = opt._cap if opt is not None else None

    def _capture_accumulating(self, loss_fn, side):
        """update_frequency > 1: the micro-batch graph, then in its memory pool the in-place zeroing and the update.  Every
        .grad is bound to its final buffer here, so the packs' prepare_grads records no zeroing and loose gradients are
        added to in place by AccumulateGrad: both accumulate across replays.  The zeroing allocates nothing; the update
        may reuse pool blocks the micro graph freed, which holds because it replays after micro-batches and leaves nothing
        in the pool that a later replay reads."""
        with torch.cuda.graph(self.graph, stream=side):
            self.epoch.add_(1)
            self.loss = loss_fn(self.static)
            self._backward(self.loss)
        self.zero_graph, self.update_graph = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.zero_graph, pool=self.graph.pool(), stream=side):
            self._zero_grads()
        with torch.cuda.graph(self.update_graph, pool=self.graph.pool(), stream=side):
            self._optimizer_step()
        self._plan = self.optimizer._cap

    def _zero_grads(self):
        """without an optimizer: .grad unset (the flat buffers are zeroed inside the graph); with one: zeroed in place, so
        every gradient keeps the storage the optimizer's tables point at"""
        if self.optimizer is None:
            self.model.zero_grad(set_to_none=True)
            return
        grads = [p.grad for p in self.model.parameters() if p.grad is not None]
        if grads:
            torch._foreach_zero_(grads)

    def _backward(self, loss):
        (loss if self.scaler is None else self.scaler.scale(loss)).backward()

    def _optimizer_step(self):
        scaler, opt = self.scaler, self.optimizer
        if scaler is None:
            if self.max_grad_norm is not None:
                opt.clip_grad_norm(self.max_grad_norm)
            opt.step()
        else:
            fused = getattr(opt, "fused_inf_check", False)
            if self.max_grad_norm is not None:
                if fused:
                    opt.clip_grad_norm(self.max_grad_norm, scaler=scaler)
                else:
                    opt.clip_grad_norm(self.max_grad_norm, scale=scaler._get_scale_async())
            elif fused:
                opt.check_finite(scaler)
            scaler.step(opt)
            scaler.update()
        if self.lr_scheduler is not None:
            self.lr_scheduler.step()

    def __call__(self, batch=None):
        if batch is not None:
            _copy_into(self.static, batch)
        if self.update_frequency > 1:
            return self._micro_batch()
        if self.optimizer is not None:
            self.optimizer.stage_hparams(self._plan)
        self.graph.replay()
        return self.loss

    def _micro_batch(self):
        if not self.pending:
            self.zero_graph.replay()
        self.graph.replay()
        self.pending += 1
        if self.pending == self.update_frequency:
            self.finish_update()
        return self.loss

    def finish_update(self):
        """Replay the update for the micro-batches accumulated since the last one: clip, step (or scaler.step and
        scaler.update) with the groups' current hyper-parameters.  A call updates on its own on the update_frequency-th
        micro-batch of a group, so this is for a partial group, MMF's last update of a run.  Nothing happens when no
        micro-batch is pending."""
        if not self.pending:
            return
        self.optimizer.stage_hparams(self._plan)
        self.update_graph.replay()
        self.pending = 0


def _check_optimizer(who, optimizer, max_grad_norm):
    if max_grad_norm is not None and optimizer is None:
        raise ValueError("%s: max_grad_norm clips inside the captured optimizer step; pass optimizer= as well, "
                         "or clip and step eagerly after each replay" % who)
    if optimizer is not None and not getattr(optimizer, "capturable", False):
        raise ValueError("%s: the optimizer's step reads host values at every step and cannot be captured; "
                         "construct it as mmf_b200.optim.B200AdamW(..., capturable=True)" % who)


def _check_scheduler(who, optimizer, lr_scheduler):
    if lr_scheduler is None:
        return
    if optimizer is None:
        raise ValueError("%s: lr_scheduler= steps inside the captured update; pass optimizer=B200AdamW(..., "
                         "capturable=True) as well" % who)
    if getattr(lr_scheduler, "optimizer", None) is not optimizer or not callable(getattr(lr_scheduler, "refresh", None)):
        raise ValueError("%s: lr_scheduler must be a mmf_b200.optim.DeviceLRScheduler built on this optimizer (a host "
                         "LambdaLR is stepped between replays instead)" % who)


def _check_capturable(who, model, static_rows):
    """the refusals GraphedStep and GraphedForward share: skip-padding encoders that read token counts on the host, and
    modules that declare `graph_capturable = False` (unless static_rows covers their only refusal)"""
    _check_runners(who, model, static_rows)
    for m in model.modules():
        if getattr(m, "graph_capturable", True) is False and not (static_rows and getattr(m, "static_rows_capturable",
                                                                                       False)):
            reason = getattr(m, "graph_refusal", "does work on the host in every forward")
            raise RuntimeError("%s: %s %s, so its step cannot be captured" % (who, type(m).__name__, reason))


def _check_runners(who, model, static_rows):
    """the encoders' skip-padding modes that read token counts on the host, and so cannot be captured: under static_rows,
    pack_tail and pack_streams runners with `device_plan` set plan on the device and are accepted"""
    runners = [m.__dict__.get("_runner") for m in model.modules()]
    if not static_rows and any(getattr(r, "skip_padding", False) for r in runners):
        raise RuntimeError("%s: the model has skip_padding encoders, which read the token count on the host and "
                           "cannot be captured; turn them off with mmf_b200.patch.set_skip_padding(model, False)" % who)
    planned = lambda r: static_rows and getattr(r, "device_plan", False)      # counts planned on the device instead
    if static_rows and any(getattr(r, "skip_padding", False) and getattr(r, "pack_tail", False) and not planned(r)
                           for r in runners):
        raise RuntimeError("%s: the model has skip_padding encoders with pack_tail set, which read the token "
                           "count on the host for calls with a causal tail even under static_rows, so they cannot be "
                           "captured; turn them off with mmf_b200.patch.set_skip_padding(model, False)" % who)
    if any(getattr(r, "pack_streams", False) and not planned(r) for r in runners):
        raise RuntimeError("%s: the model has two-stream encoders with pack_streams set, which read the token "
                           "counts on the host%s and cannot be captured; turn them off with "
                           "mmf_b200.patch.set_skip_padding(model, False, two_stream=True)"
                           % (who, " even under static_rows" if static_rows else ""))


class GraphedForward:
    """An evaluation forward replayed as one CUDA graph:

        fwd = GraphedForward(model.eval(), example_batch)     # warm-up, then capture of model(batch) under no_grad
        out = fwd(batch)                                      # copies `batch` into the static inputs, replays the graph

    The graph records `model(static_batch)` - for a registered model BaseModel.__call__, so `scores` and, when the batch
    carries targets, `losses` are in it - as an eager `model.eval()` forward under torch.no_grad() launches it.  M4C and
    the M4C captioner run all their greedy decoding steps in that forward (a fixed trip count, nothing read on the host),
    so the whole decode is one graph.

    The returned output is the captured structure of static tensors: every call overwrites it, so it is valid until the
    next call; clone what must outlive it.  `example_batch` is a (nested dict / SampleList / list of) CUDA tensors with the
    shapes of every later batch; its mapping types are kept, so a SampleList stays one.  Non-tensor values (dataset
    names) are fixed at capture.  As for GraphedStep, the batch must carry every input the forward would otherwise build
    from a host value.  Every forward gets fresh containers over the static tensors, so a forward that replaces keys of
    its sample list (MMBT's token shift, VisualBERT's masks) does not replace the static inputs.  As for GraphedStep,
    the reductions are those torch.use_deterministic_algorithms selected at capture: the static-rows masked-LM loss adds
    its row losses with atomics unless captured under the flag.

    The model must be in eval mode: nothing is drawn, and the dropout step counter of GraphedStep is neither created nor
    advanced.  Refused before any warm-up, as GraphedStep refuses them: skip-padding encoders without static_rows,
    pack_tail and pack_streams encoders, and modules that declare `graph_capturable = False` (UNITER, whose forward draws
    its task on the host; VinVL and ViLT pretraining without static_rows); under static_rows pack_tail and pack_streams
    encoders switched on with device_plan=True are accepted.  Also refused: a model that returns attention
    probabilities or hidden states (output_attentions / output_hidden_states / visualization), and a model or batch off
    the GPU.

    static_rows=True: warm-up and capture run inside static_rows(), so pretraining validation losses (the masked-LM
    heads select their rows on the device, and return no MLM logits) and single-stream skip-padding encoders (packed at a
    fixed capacity of every row of the batch) are captured."""

    def __init__(self, model, example_batch, warmup=3, static_rows=False):
        if model.training:
            raise ValueError("GraphedForward: the model is in training mode; capture an evaluation forward after "
                             "model.eval(), and a training step with GraphedStep")
        _check_capturable("GraphedForward", model, static_rows)
        for m in model.modules():
            if getattr(m, "output_attentions", False) or getattr(m, "output_hidden_states", False) or \
                    getattr(getattr(m, "config", None), "visualization", False) is True:
                raise RuntimeError("GraphedForward: %s returns attention probabilities or hidden states, which are not "
                                   "captured; turn off output_attentions / output_hidden_states / visualization"
                                   % type(m).__name__)
        off = sorted({str(t.device) for t in list(model.parameters()) + list(_flatten(example_batch))
                      if not t.is_cuda})
        if off or not any(True for _ in _flatten(example_batch)):
            raise RuntimeError("GraphedForward: the model and every tensor of the batch must be on a CUDA device (found "
                               "%s); a CUDA graph replays device work only" % (", ".join(off) or "no tensor in the batch"))
        self.model = model
        with _static_rows_context() if static_rows else contextlib.nullcontext():
            self._capture(model, example_batch, warmup)

    def _capture(self, model, example_batch, warmup):
        self.static = _map_keep(lambda t: t.detach().clone(), example_batch)
        dev = next(t for t in _flatten(self.static) if t.is_cuda).device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.no_grad(), torch.cuda.stream(side):
            for _ in range(max(1, warmup)):              # lazy engine state, kernel attributes, library work buffers
                model(_map_keep(lambda t: t, self.static))
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph, stream=side):
            self.output = model(_map_keep(lambda t: t, self.static))

    def __call__(self, batch=None):
        if batch is not None:
            _copy_into(self.static, batch)
        self.graph.replay()
        return self.output


def _map_keep(fn, x):
    """_map that keeps each container's type (the models read a SampleList's fields as attributes)"""
    if isinstance(x, dict):
        return type(x)((k, _map_keep(fn, v)) for k, v in x.items())
    if isinstance(x, (list, tuple)):
        return type(x)(_map_keep(fn, v) for v in x)
    return fn(x) if torch.is_tensor(x) else x


class GraphedTaskSteps:
    """One CUDA graph per task for a model whose forward draws its task on the host (UNITER: the task with torch.randint,
    the region masks of mrc / mrfr with numpy and random).  The model defines `draw(sample_list, task=None)`, which makes
    those draws, stores them in the sample list under `model.draws_key` and returns the task's name, and a forward that
    finds them draws nothing.  So the draws stay on the host, where the reference makes them, and everything after them
    is captured:

        steps = GraphedTaskSteps(model, loss_fn, example_batch, optimizer=opt, max_grad_norm=1.0)
        loss = steps(batch)      # draws on the host, copies batch and draws into the static inputs, replays that task

    Every graph is captured inside static_rows() (the masked-LM and region heads select their rows on the device) with
    its task's draws fixed; all graphs share one memory pool, so a returned loss is valid until the next call.
    Constructing the object leaves the torch CPU, numpy and `random` generators as they were, although warm-up and
    capture draw too; each call then draws exactly what an eager forward draws.

    Gradients: each task's graph zeroes and fills the gradients of the parameters that task reaches, in buffers all
    graphs share; after a call `.grad` is set for those and None for the others, as after an eager step from
    zero_grad(set_to_none=True).  With a capturable B200AdamW every graph carries its own optimizer plan, so a replayed
    step of task t updates exactly the parameters an eager step of t updates: heads t does not reach keep their values,
    moments and step counts.  The step counts live in one device table that each graph reads before and writes after its
    optimizer step; step the optimizer only through this object while it is in use.  The warm-up steps are undone.
    lr_scheduler: a DeviceLRScheduler on the optimizer, stepped inside every task's graph after its optimizer step, as
    in GraphedStep; all graphs advance its one device counter, which warm-up and capture leave as they found it.
    Skip-padding and pack_streams encoders are refused as by GraphedStep without static_rows."""

    def __init__(self, model, loss_fn, example_batch, warmup=3, optimizer=None, max_grad_norm=None, lr_scheduler=None):
        if not callable(getattr(model, "draw", None)) or not getattr(model, "draws_key", None) or \
                not getattr(model, "tasks", None):
            raise TypeError("GraphedTaskSteps: the model must define draw(sample_list, task=None), draws_key and tasks; "
                            "capture a model that draws nothing on the host with GraphedStep")
        _check_optimizer("GraphedTaskSteps", optimizer, max_grad_norm)
        _check_scheduler("GraphedTaskSteps", optimizer, lr_scheduler)
        _check_runners("GraphedTaskSteps", model, False)
        for m in model.modules():
            if m is not model and getattr(m, "graph_capturable", True) is False and \
                    not getattr(m, "static_rows_capturable", False):
                raise RuntimeError("GraphedTaskSteps: %s %s, so its step cannot be captured"
                                   % (type(m).__name__, getattr(m, "graph_refusal", "does work on the host in every forward")))
        self.model, self.loss_fn = model, loss_fn
        self.optimizer, self.max_grad_norm, self.lr_scheduler = optimizer, max_grad_norm, lr_scheduler
        self.tasks = list(dict.fromkeys(model.tasks))
        self.task = None
        state = (torch.get_rng_state(), np.random.get_state(), random.getstate())
        try:
            with _static_rows_context():
                self._capture(example_batch, warmup)
        finally:
            torch.set_rng_state(state[0])
            np.random.set_state(state[1])
            random.setstate(state[2])

    def _batch(self, task):
        """a fresh top level over the static inputs (the forward adds and replaces keys) with the task's static draws"""
        b = dict(self.static)
        b[self.model.draws_key] = self.draws[task]
        return b

    def _capture(self, example_batch, warmup):
        model, opt = self.model, self.optimizer
        self.static = _map(lambda t: t.detach().clone(), example_batch)
        self.draws = {}
        for t in self.tasks:
            probe = dict(self.static)
            model.draw(probe, task=t)
            self.draws[t] = _map(lambda x: x.detach().clone(), probe[model.draws_key])
        dev = next(t for t in _flatten(self.static) if t.is_cuda).device
        self.epoch = F.dropout_epoch(dev, create=True)
        params = list(dict.fromkeys(model.parameters()))
        saved = _save_optimizer(opt) if opt is not None else None
        saved_counter = self.lr_scheduler.counter.clone() if self.lr_scheduler is not None else None
        self.grads, self.used, self.graphs, self.losses, self.plans, self._keep = {}, {}, {}, {}, {}, []
        pool = None
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        for t in self.tasks:
            with torch.cuda.stream(side):
                model.zero_grad(set_to_none=True)          # which parameters task t reaches: those that get a .grad
                self._step(self._batch(t))
                self.used[t] = [p for p in params if p.grad is not None]
                for p in self.used[t]:
                    self.grads.setdefault(p, p.grad)
                for _ in range(max(1, warmup)):            # on the shared buffers: the optimizer's tables point at them
                    self._bind_grads(t)
                    torch._foreach_zero_([self.grads[p] for p in self.used[t]])
                    self._step(self._batch(t))
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            plan = opt._cap if opt is not None else None
            counts = None
            if plan is not None:
                # the graph reads these device buffers at every replay: they must live as long as it does
                counts = (plan,) + self._step_slots(plan, params)
                self._keep.append((opt._clip_table, counts))
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, pool=pool, stream=side):
                torch._foreach_zero_([self.grads[p] for p in self.used[t]])
                self.epoch.add_(1)
                self.losses[t] = self._step(self._batch(t), counts)
            pool = graph.pool()
            self.graphs[t], self.plans[t] = graph, plan
        if opt is not None:
            _restore_optimizer(opt, saved)
            steps = [saved["state"].get(p, {}).get("step", 0) for p in params]
            from .optim import _read_steps
            self.steps.copy_(torch.tensor(_read_steps(steps) + [0], dtype=torch.int64))
            for i, p in enumerate(params):
                if p in opt.state:
                    opt.state[p]["step"] = self.steps[i]
            if self.lr_scheduler is not None:
                _restore_scheduler(self.lr_scheduler, saved_counter)
            torch.cuda.synchronize(dev)
        self._bind_grads(self.tasks[-1])

    def _step_slots(self, plan, params):
        """device index tables between the plan's step-count slots and the shared per-parameter table `self.steps`
        (one entry per parameter, then one spare for the slots no parameter reads)"""
        if not hasattr(self, "steps"):
            self.steps = torch.zeros(len(params) + 1, dtype=torch.int64, device=plan.device)
        index = {id(p): i for i, p in enumerate(params)}
        group_of = {id(p): gi for gi, g in enumerate(self.optimizer.param_groups) for p in g["params"]}
        slot_param = [len(params)] * len(plan.slots)
        written = []                                       # (parameter index, slot)
        for pack, _, s0, _, _, _ in plan.packs:
            for p in pack.params:
                if id(p) in group_of and p.grad is not None:
                    slot_param[s0 + group_of[id(p)]] = index[id(p)]
                    written.append((index[id(p)], s0 + group_of[id(p)]))
        for p, slot in plan.loose:
            slot_param[slot] = index[id(p)]
            written.append((index[id(p)], slot))
        to_dev = lambda v: torch.tensor(v, dtype=torch.int64).to(plan.device)
        return to_dev(slot_param), to_dev([s for _, s in written]), to_dev([i for i, _ in written])

    def _bind_grads(self, task):
        for p in self.grads:
            p.grad = None
        for p in self.used[task]:
            p.grad = self.grads[p]

    def _step(self, batch, counts=None):
        loss = self.loss_fn(batch)
        loss.backward()
        opt = self.optimizer
        if opt is not None:
            if self.max_grad_norm is not None:
                opt.clip_grad_norm(self.max_grad_norm)
            if counts is not None:                         # this graph's step counts from the shared table ...
                plan, gather, slots, idx = counts
                plan.step.copy_(self.steps.index_select(0, gather))
            opt.step()
            if counts is not None:                         # ... and back
                self.steps.index_copy_(0, idx, plan.step.index_select(0, slots))
            if self.lr_scheduler is not None:
                self.lr_scheduler.step()
        return loss

    def __call__(self, batch=None):
        if batch is not None:
            _copy_into(self.static, batch)
        probe = dict(self.static)
        task = self.model.draw(probe)
        _copy_into(self.draws[task], probe[self.model.draws_key])
        if self.optimizer is not None:
            self.optimizer.stage_hparams(self.plans[task])
        self.graphs[task].replay()
        self._bind_grads(task)
        self.task = task
        return self.losses[task]


def _save_optimizer(opt):
    """copies of the parameters and optimizer state that the warm-up steps change"""
    params = [p for g in opt.param_groups for p in g["params"]]
    return {"params": [(p, p.detach().clone()) for p in params],
            "state": {p: {k: (v.clone() if torch.is_tensor(v) else v) for k, v in opt.state[p].items()}
                      for p in params if p in opt.state},
            "flat": {k: (e["m"].clone(), e["v"].clone()) for k, e in opt._flat.items()}}


def _restore_optimizer(opt, saved):
    """undo the warm-up steps: parameters, moments (flat buffers included) and step counts as they were before"""
    for p, c in saved["params"]:
        p.detach().copy_(c)
    for k, e in opt._flat.items():
        if k in saved["flat"]:
            e["m"].copy_(saved["flat"][k][0])
            e["v"].copy_(saved["flat"][k][1])
        else:
            e["m"].zero_()
            e["v"].zero_()
    for p, st in opt.state.items():
        old = saved["state"].get(p, {})
        for k in ("exp_avg", "exp_avg_sq"):
            if k in st:
                st[k].copy_(old[k]) if k in old else st[k].zero_()
        if torch.is_tensor(st.get("step")):
            st["step"].copy_(old["step"]) if torch.is_tensor(old.get("step")) else st["step"].fill_(int(old.get("step", 0)))
        elif "step" in st:
            st["step"] = old.get("step", 0)


def _save_scaler(scaler):
    """copies of the GradScaler state the warm-up updates change (None before its first scale())"""
    scale, tracker = scaler._scale, scaler._growth_tracker
    return (scale.clone() if scale is not None else None, tracker.clone() if tracker is not None else None)


def _restore_scaler(scaler, saved):
    """undo the warm-up updates in place: the graph reads and writes these tensors at every replay.  A scaler whose
    tensors the warm-up created gets its initial scale and a zero growth tracker, the state it stands for."""
    scale, tracker = saved
    if scaler._scale is not None:
        scaler._scale.copy_(scale) if scale is not None else scaler._scale.fill_(scaler._init_scale)
    if scaler._growth_tracker is not None:
        scaler._growth_tracker.copy_(tracker) if tracker is not None else scaler._growth_tracker.zero_()


def _restore_scheduler(sched, counter):
    """undo the warm-up's scheduler steps in place (the graphs read the counter and the lr table at every replay)"""
    sched.counter.copy_(counter)
    sched.refresh()


def _flatten(x):
    if isinstance(x, dict):
        for v in x.values():
            yield from _flatten(v)
    elif isinstance(x, (list, tuple)):
        for v in x:
            yield from _flatten(v)
    elif torch.is_tensor(x):
        yield x
