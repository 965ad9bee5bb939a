"""Drop-in encoder modules: same constructor inputs, sub-module / parameter names, forward signatures and
return structure as the reference's encoders, computing on the B200 engine.

  B200BertEncoder     <->  BertEncoderJit           mmf/modules/hf_layers.py:295-355
  B200ViLBertEncoder  <->  vilbert.BertEncoder      mmf/models/vilbert.py:559-796

EncoderRunner runs a single-stream layer stack, TwoStreamRunner the ViLBERT and LXMERT (mmf_b200.lxmert) ones.

Parameter names are the reference's (`layer.{i}.attention.self.query.weight`, `c_layer.{i}.biattention.query1.bias`,
`c_layer.{i}.biOutput.q_dense1.weight` ... SURVEY.md 5 "Checkpoint / resume"), so zoo checkpoints and
`pretrained_state_mapping` keep loading.  The nn.Linear / nn.LayerNorm children below are parameter HOLDERS:
their own forward is never called.

The same runners can be attached to an EXISTING HuggingFace / MMF module tree (mmf_b200.patch), which is how
VisualBERT / MMBT / MMFTransformer pick the engine up without any registry indirection (SURVEY.md 8b).
"""
import os

import torch
from torch import nn

from . import engine as E
from . import graphs
from . import lib


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(
            "%s is on %s: the fusion path has no CPU fallback (move the model and inputs to an H100)" % (what, t.device))
    if not lib.device_ok():
        raise RuntimeError("libmmfb200 needs an sm_90 (H100) device: " + lib.last_error())


def _check_erf_gelu(layer):
    """The FFN epilogue IS the exact erf GELU of the reference configs (ACT2FN["gelu"]); an attached HuggingFace layer
    with any other activation (gelu_new, relu, swish ...) must not be rerouted silently."""
    fn = getattr(getattr(layer, "intermediate", None), "intermediate_act_fn", None)
    if fn is None:
        return
    name = getattr(fn, "__name__", None) or type(fn).__name__
    if name.lower() in ("gelu", "geluactivation"):
        return
    probe = torch.tensor([-1.5, -0.3, 0.7, 2.0])
    try:
        ok = torch.allclose(fn(probe), torch.nn.functional.gelu(probe), atol=1e-6)
    except Exception:
        ok = False
    if not ok:
        raise NotImplementedError("the B200 fusion block implements the erf GELU only; this encoder uses %s" % name)


_SEED_COUNTER = [0]


def _fresh_dropout_state():
    """One Philox stream per forward, derived from torch's seed so `torch.manual_seed` makes runs repeatable.
    (The bits are drawn on the compute stream: the GEMMs a side-stream generator would overlap occupy every SM.)"""
    _SEED_COUNTER[0] += 1
    seed = torch.initial_seed() * 1000003 + _SEED_COUNTER[0]
    return E.DropoutState(seed)


# ------------------------------------------------------------------------------------------------------
# single-stream BERT encoder
# ------------------------------------------------------------------------------------------------------
class _LayerStack:
    """Engine state of layers run in a fixed order, layer i with handles class Ws[i] (built lazily on the first CUDA
    forward): ONE ParamPack over the layers' parameters in execution order, so that data-parallel gradient buckets complete
    in reverse order, and each layer's handles."""

    def __init__(self, layers, Ws):
        self._stack = list(zip(layers, Ws))
        self._starts = None
        self.pack = None
        self.weights = None
        self.grad_ready_hook = None   # callable(step_index) - set by mmf_b200.ddp for bucket all-reduce overlap

    def ensure(self, device):
        if self.pack is not None and self.pack.intact() and self.pack.device == device:
            return
        for m, _ in self._stack:
            _check_erf_gelu(m)
        params = [p for m, W in self._stack for p in W.params(m)]
        for p in params:
            _require_cuda(p, "encoder parameter")
        self.pack = E.ParamPack(params, device)
        self.weights = [W(self.pack, m) for m, W in self._stack]

    @property
    def step_offsets(self):
        """offset in the pack's flat buffers where each layer's parameters start (the data-parallel bucket boundaries)"""
        if self._starts is None:
            self._starts = [0]
            for m, W in self._stack[:-1]:
                self._starts.append(self._starts[-1] + len(W.params(m)))
        return [self.pack.offsets[i] for i in self._starts]


class EncoderRunner(_LayerStack):
    """Engine state of one BERT-style layer stack."""

    W = E.BertLayerW                       # parameter handles and block functions of one layer

    def __init__(self, layers):
        self.layers = list(layers)
        super().__init__(self.layers, [self.W] * len(self.layers))
        # skip padded tokens: pack the valid rows once per encoder call and run variable-length attention (run_bert_encoder)
        self.skip_padding = False
        # with skip_padding: also pack calls with a causal tail (M4C's multimodal transformer), keeping every tail row
        self.pack_tail = False
        # with pack_tail: inside graphs.static_rows() plan those calls on the device (_static_packings) so they can be
        # captured
        self.device_plan = False

    def forward(self, x, add_mask, training, need_grad, probs=None):
        """probs: an engine.ProbsSink that receives every layer's attention probabilities, or None"""
        B, S, H = x.shape
        h = x.reshape(B * S, H)
        saved = []
        ds = _fresh_dropout_state() if training else None
        hiddens = []
        extra = {} if probs is None else {"probs": probs}
        for m, w in zip(self.layers, self.weights):
            ps = [p if training else 0.0 for p in self.W.dropout_p(m)]
            hiddens.append(h)
            h, s = self.W.fwd(h, add_mask, w, B, S, *ps, ds, **extra)
            saved.append(s if need_grad else None)
        return h, saved, hiddens

    def backward(self, dout, saved, add_mask, B, S):
        d = dout
        for i in range(len(saved) - 1, -1, -1):
            d = self.W.bwd(d, saved[i], add_mask, self.weights[i], B, S)
            saved[i] = None
            if self.grad_ready_hook is not None:
                self.grad_ready_hook(i)
        return d


class _Packing:
    """Valid rows of a padded [B, S] batch: `rows` (int64 [total]) are their flat indices in sample order, `varlen` the
    descriptor the engine's attention reads.  rows = None is the trivial packing of an unpadded stream (every row, in
    place), which packs and unpacks without a copy."""

    def __init__(self, rows, varlen):
        self.rows, self.varlen = rows, varlen

    def pack(self, t):
        """[B*S, H] -> [total, H]: the valid rows, in their original order within each sample"""
        return t if self.rows is None else t.index_select(0, self.rows)

    def unpack(self, t, BS):
        """[total, H] -> [B*S, H] with exact zero rows at padded positions"""
        return t if self.rows is None else t.new_zeros(BS, t.shape[1]).index_copy_(0, self.rows, t)


def _no_capture(what):
    if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
        raise RuntimeError("%s cannot run under CUDA-graph capture: packing needs the valid-token count on the host "
                           "(turn it off with mmf_b200.patch.set_skip_padding(model, False) before capturing)" % what)


def _mask_counts(mask):
    """device side of a packing plan: (valid [B, S], lens int32 [B], int64 [3] = soft values, total, max_len)"""
    valid = mask == 0
    lens = valid.sum(1, dtype=torch.int32)
    soft = ((mask != 0) & (mask > -10000.0)).sum()
    return valid, lens, torch.stack([soft.to(torch.int64), lens.sum(dtype=torch.int64), lens.max().to(torch.int64)])


def _check_soft(n_soft, what="skip_padding"):
    if n_soft:
        raise ValueError("%s needs a key-padding mask of 0 (token) and <= -10000 (padding); %d value(s) are a "
                         "soft bias, which cannot be packed away" % (what, n_soft))


def _plan_packing(mask, B, S, counts=None):
    """The packing of an additive [B, S] fp32 mask (0 = token, <= -10000 = padding), or None when no row is padded.
    One device-to-host copy fetches the counts; the row indices are built on the device without another one.  `counts` =
    (valid, lens, (n_soft, total, max_len) on the host) when the caller has already fetched them (two-stream plans fetch
    both streams' counts in one copy)."""
    if counts is None:
        _no_capture("skip_padding")
        valid, lens, st = _mask_counts(mask)
        counts = (valid, lens, tuple(int(v) for v in st.tolist()))
    valid, lens, (n_soft, total, max_len) = counts
    _check_soft(n_soft)
    if total == B * S:
        return None
    cu = torch.zeros(B + 1, dtype=torch.int32, device=mask.device)
    cu[1:] = torch.cumsum(lens, 0, dtype=torch.int32)
    flat = valid.reshape(-1)
    dest = torch.where(flat, torch.cumsum(flat, 0) - 1, torch.full_like(flat, total, dtype=torch.int64))
    rows = torch.empty(total + 1, dtype=torch.int64, device=mask.device)
    rows.scatter_(0, dest, torch.arange(B * S, device=mask.device))     # padded rows all land in the spare last slot
    return _Packing(rows[:total], E.Varlen(cu, B, total, max_len))


class _StaticPacking:
    """The packing of a padded [B, S] batch planned on the device, at the fixed capacity C = B*S (graphs.static_rows()):
    `pack_map` (int32 [C]) holds the flat indices of the valid rows in _plan_packing's order, then -1; `unpack_map` (int32
    [B*S]) holds each position's packed row, or -1 at padded positions.  Packing, unpacking and both backwards are one
    row-gather kernel each (mmfb_gather_rows), and every shape depends on B and S only, so a CUDA graph can capture it.
    `varlen` carries the device count cu[B] as Varlen.count, which bounds the layers' kernels."""

    def __init__(self, pack_map, unpack_map, varlen):
        self.pack_map, self.unpack_map, self.varlen = pack_map, unpack_map, varlen

    def pack(self, t):
        """[B*S, H] -> [C, H]: the valid rows first, in their original order within each sample, then zero rows"""
        return E.F.gather_rows(t, self.pack_map)

    def unpack(self, t, BS):
        """[C, H] -> [B*S, H] with exact zero rows at padded positions"""
        return E.F.gather_rows(t, self.unpack_map)


def _plan_packing_static(mask, B, S):
    """_plan_packing without a host read: the packing of an additive [B, S] fp32 mask (0 = token, anything else = padding)
    at capacity B*S.  Every row valid and every row padded are planned like any other batch, and the soft-mask check of
    _plan_packing cannot run: a mask value that is neither 0 nor <= -10000 is taken as padding without a check."""
    C = B * S
    valid = (mask == 0).reshape(-1)
    incl = torch.cumsum(valid, 0, dtype=torch.int32)                    # valid rows up to and including each position
    cu = torch.zeros(B + 1, dtype=torch.int32, device=mask.device)
    cu[1:] = incl.view(B, S)[:, -1]
    unpack_map = torch.where(valid, incl - 1, torch.full_like(incl, -1))
    # packed row i comes from the first position where `incl` reaches i + 1; past the count no position does
    pack_map = torch.searchsorted(incl, torch.arange(1, C + 1, dtype=torch.int32, device=mask.device), out_int32=True)
    pack_map = torch.where(pack_map < C, pack_map, torch.full_like(pack_map, -1))
    return _StaticPacking(pack_map, unpack_map, E.Varlen(cu, B, C, S, count=cu[B:]))


def _static_packings(masks, B, lens, causal_len=0):
    """The packings of one or two streams planned on the device by one kernel (functional.plan_packing), at the capacity
    B*S of each stream: a _StaticPacking per stream with a mask, whose Varlen carries the device count cu[B]; a stream
    without a mask keeps the trivial packing, unbounded.  With causal_len = T > 0 (one stream) the last T positions of
    every sample are kept whatever the mask holds there, as _tail_kept does.  Two streams: a sample with tokens in one
    stream and none in the other keeps every row of the empty one, so the other's queries attend over all of them - the
    dense path gives those keys one common mask value, so the function is the dense one up to rounding, where
    plan_two_stream falls back to the dense path.  A sample without tokens in either stream keeps no row (zero outputs
    and input gradients).  Nothing is read on the host, and a mask value that is neither 0 nor <= -10000 is padding."""
    device = next(m.device for m in masks if m is not None)
    out = []
    for S, plan in zip(lens, E.F.plan_packing(masks, B, lens, causal_len)):
        if plan is None:
            out.append(_trivial_packing(B, S, device))
            continue
        cu, pack_map, unpack_map = plan
        out.append(_StaticPacking(pack_map, unpack_map, E.Varlen(cu, B, B * S, S, causal_len, count=cu[B:])))
    return out


def _tail_kept(mask, causal_len):
    """the key-padding mask of a call with a causal tail, as packing reads it: the mask before the tail, and 0 (kept) on
    the last causal_len positions, which the dense path does not read the mask at either"""
    m = mask.clone()
    m[:, mask.shape[1] - causal_len:] = 0.0
    return m


def _trivial_packing(B, S, device):
    """every row of an unpadded [B, S] stream, as a packing: cu = arange(B+1) * S"""
    cu = (torch.arange(B + 1, dtype=torch.int32, device=device) * S).contiguous()
    return _Packing(None, E.Varlen(cu, B, B * S, S))


def plan_two_stream(mask_a, mask_b, B, Sa, Sb, device):
    """Packing of a two-stream encoder call (ViLBERT, LXMERT) from the additive key-padding masks of its streams ([B, Sa],
    [B, Sb] fp32, or None = no padding).  Returns
      None            - nothing is padded, or some sample has tokens in one stream and none in the other: the dense path
                        runs.  (There those queries attend over the other stream's padded rows and the valid outputs depend
                        on them, so packing would change the function, not just skip work);
      "empty"         - every row of both streams is padding: the outputs and input gradients are zeros;
      (pack_a, pack_b) - a packing per stream; an unpadded stream gets the trivial one.
    Both streams' counts reach the host in one device-to-host copy.  A soft mask raises ValueError; stream capture raises
    RuntimeError."""
    if mask_a is None and mask_b is None:
        return None
    _no_capture("pack_streams")
    counts, stats = [], []
    for m, S in ((mask_a, Sa), (mask_b, Sb)):
        if m is None:
            counts.append((None, torch.full((B,), S, dtype=torch.int32, device=device)))
            stats.append(torch.tensor([0, B * S, S], dtype=torch.int64, device=device))
        else:
            valid, lens, st = _mask_counts(m)
            counts.append((valid, lens))
            stats.append(st)
    one_sided = ((counts[0][1] > 0) != (counts[1][1] > 0)).sum().to(torch.int64).reshape(1)
    host = torch.cat(stats + [one_sided]).tolist()            # the one device-to-host copy
    st_a, st_b, n_one_sided = tuple(host[0:3]), tuple(host[3:6]), host[6]
    _check_soft(st_a[0], "pack_streams")
    _check_soft(st_b[0], "pack_streams")
    if st_a[1] == B * Sa and st_b[1] == B * Sb:
        return None
    if st_a[1] == 0 and st_b[1] == 0:
        return "empty"
    if n_one_sided:
        return None
    plans = []
    for m, S, (valid, lens), st in ((mask_a, Sa, counts[0], st_a), (mask_b, Sb, counts[1], st_b)):
        plan = None if m is None else _plan_packing(m, B, S, counts=(valid, lens, st))
        plans.append(plan if plan is not None else _trivial_packing(B, S, device))
    return tuple(plans)


def _probs_sink(*dtypes):
    """A ProbsSink whose kernel output dtype is the callers' hidden-state dtype when that is fp32 or bf16 (and the same for
    every stream); fp32 otherwise, cast on the host afterwards."""
    dt = dtypes[0] if len(set(dtypes)) == 1 and dtypes[0] in (torch.float32, torch.bfloat16) else torch.float32
    return E.ProbsSink(dt)


class _BertEncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, runner, add_mask, training, want_hiddens, want_attn, x, *params):
        B, S, H = x.shape
        need_grad = any(ctx.needs_input_grad)   # (grad mode itself is always off inside Function.forward)
        runner.pack.refresh()
        xb = x.detach().to(torch.bfloat16).contiguous()
        packing = add_mask if isinstance(add_mask, (_Packing, _StaticPacking)) else None
        probs = _probs_sink(x.dtype) if want_attn else None
        if packing is None:
            out, saved, hiddens = runner.forward(xb, add_mask, training, need_grad, probs=probs)
        else:                                   # the layers run on the [total, H] valid rows only
            vl = packing.varlen
            xp = packing.pack(xb.view(B * S, H)).view(1, vl.total, H)
            out, saved, hiddens = runner.forward(xp, vl, training, need_grad)
            out = packing.unpack(out, B * S)
            hiddens = [packing.unpack(h, B * S) for h in hiddens] if want_hiddens else hiddens
        ctx.runner, ctx.saved, ctx.add_mask, ctx.dims, ctx.in_dtype = runner, saved, add_mask, (B, S, H), x.dtype
        outs = [out.view(B, S, H).to(x.dtype)]
        if want_hiddens:
            outs += [h.view(B, S, H).to(x.dtype) for h in hiddens]
        if want_attn:
            outs += [p.to(x.dtype) for p in probs]
        if len(outs) > 1:
            ctx.mark_non_differentiable(*outs[1:])
        return tuple(outs)

    @staticmethod
    def backward(ctx, dout, *unused):
        runner = ctx.runner
        B, S, H = ctx.dims
        if ctx.saved is None or any(s is None for s in ctx.saved):
            raise RuntimeError("B200 encoder: backward called twice or activations were not saved")
        aliased = runner.pack.prepare_grads()
        d = dout.to(torch.bfloat16).contiguous().view(B * S, H)
        if isinstance(ctx.add_mask, (_Packing, _StaticPacking)):
            packing = ctx.add_mask
            dx = runner.backward(packing.pack(d), ctx.saved, packing.varlen, 1, packing.varlen.total)
            dx = packing.unpack(dx, B * S)
        else:
            dx = runner.backward(d, ctx.saved, ctx.add_mask, B, S)
        ctx.saved = None
        return (None, None, None, None, None, dx.view(B, S, H).to(ctx.in_dtype)) + tuple(runner.pack.autograd_grads(aliased))


def run_bert_encoder(runner, hidden_states, attention_mask, training, output_hidden_states=False, output_attentions=False,
                     causal_len=0):
    """hidden_states [B,S,H] (fp32 or bf16), attention_mask additive [B,1,1,S] / [B,S] / None.
    causal_len = T > 0 makes the last T positions a causal tail (engine.CausalTail, M4C's prefix-LM mask): every query
    attends to the keys before the tail that attention_mask keeps, the first S - T queries to no tail key, and tail query t
    to tail keys 0..t; attention_mask is not read for the tail keys.  Such a call cannot return probabilities.  With
    skip_padding alone it runs the dense path; with skip_padding and runner.pack_tail it packs the rows before the tail
    that attention_mask keeps plus every tail row (so the tail is the last T packed rows of each sample) and runs the
    packed kernels with the tail, unless no row before the tail is padded (then it runs the dense path).
    Returns (last,), then the L layer inputs if output_hidden_states, then the L layers' attention probabilities
    [B, heads, S, S] (hidden-state dtype, post-dropout in training) if output_attentions.  The hidden states and
    probabilities are outputs for inspection: they carry no gradient, so a loss that reads them back-propagates nothing
    through them.  A call that asks for probabilities runs the dense path even with skip_padding set, so they have the
    reference's [B, heads, S, S] shape, padded rows and keys included.
    Inside graphs.static_rows(), a call without a causal tail on a skip_padding runner plans its packing on the device
    (_plan_packing_static) instead: nothing is read on the host, so the call can be captured in a CUDA graph.  It runs the
    packed path at a fixed capacity of B*S rows whatever the mask holds (every row valid, or none: then the outputs and
    the input gradient are exact zeros), and its mask values other than 0 and <= -10000 are not checked.  A call with a
    causal tail on a pack_tail runner with `device_plan` set does the same there (_static_packings): it packs the same
    rows as the eager call, every tail row included, and runs the packed path even when no row is padded."""
    _require_cuda(hidden_states, "hidden_states")
    if hidden_states.dim() != 3:
        raise ValueError("hidden_states must be [batch, seq, hidden], got %s" % (tuple(hidden_states.shape),))
    B, S, H = hidden_states.shape
    runner.ensure(hidden_states.device)
    if H != runner.weights[0].hidden:
        raise ValueError("hidden size %d does not match the encoder's %d" % (H, runner.weights[0].hidden))
    mask = E.additive_mask_2d(attention_mask, B, S)
    causal_len = int(causal_len)
    if causal_len:
        if not 0 < causal_len <= S:
            raise ValueError("causal_len must be in [0, S=%d], got %d" % (S, causal_len))
        packing = None
        if runner.skip_padding and runner.pack_tail and mask is not None and not output_attentions:
            if graphs.static_rows_active() and runner.device_plan:
                if runner.W is not E.BertLayerW:
                    raise RuntimeError("skip_padding under static_rows() covers BERT layer stacks only")
                packing = _static_packings([mask], B, [S], causal_len)[0]
            else:
                packing = _plan_packing(_tail_kept(mask, causal_len), B, S)     # never empty: the tail rows stay
        if packing is not None:
            packing.varlen.causal_len = causal_len
            mask = packing
        else:
            mask = E.CausalTail(mask, causal_len)
    elif runner.skip_padding and mask is not None and not output_attentions and graphs.static_rows_active():
        if runner.W is not E.BertLayerW:
            raise RuntimeError("skip_padding under static_rows() covers BERT layer stacks only")
        mask = _plan_packing_static(mask, B, S)
    elif runner.skip_padding and mask is not None and not output_attentions:
        packing = _plan_packing(mask, B, S)
        if packing is not None and packing.varlen.total == 0:
            # every token is padding: nothing to compute, every output row (and every input-gradient row) is zero
            z = hidden_states * 0
            return (z,) + ((z.detach(),) * len(runner.layers) if output_hidden_states else ())
        if packing is not None:
            mask = packing
    outs = _BertEncoderFn.apply(runner, mask, training, output_hidden_states, bool(output_attentions), hidden_states,
                                *runner.pack.params)
    return outs


class TwoStreamRunner(_LayerStack):
    """Engine state of a two-stream layer stack (ViLBERT, LXMERT).  `steps` lists
    the layers in execution order as (module, W, streams): W is the layer's handles class (which also holds its block
    functions) and `streams` the stream indices the block function takes, in its argument order - (0,) or (1,) for a
    single-stream layer, both for a layer that joins them (ViLBERT's co-attention takes (image, text) = (1, 0), LXMERT's
    cross-modality layer (language, vision) = (0, 1)).  Stream 0 is text / language, stream 1 image / vision."""

    def __init__(self, steps):
        self.steps = list(steps)
        super().__init__([m for m, _, _ in self.steps], [W for _, W, _ in self.steps])
        # skip padded tokens in both streams: pack each stream's valid rows once per encoder call and run variable-length
        # self- and cross-attention (plan_two_stream)
        self.pack_streams = False
        # with pack_streams: inside graphs.static_rows() plan the packing on the device (_static_packings) so the call can
        # be captured
        self.device_plan = False

    def forward(self, xs, masks, lens, B, training, need_grad, block_states=None, probs=None):
        """xs: the two streams' [rows, H] activations, replaced by the outputs; masks: their additive masks, None or Varlen
        descriptors; lens: their sequence lengths.  Returns what the backward needs.  block_states: a list that receives
        (stream 0, stream 1) after every step that joins the streams, or None.  probs: an engine.ProbsSink that receives
        the attention probabilities in step order, or None."""
        ds = _fresh_dropout_state() if training else None
        extra = {} if probs is None else {"probs": probs}
        saved = []
        for (m, W, streams), w in zip(self.steps, self.weights):
            ps = [p if training else 0.0 for p in W.dropout_p(m)]
            *outs, s = W.fwd(*[xs[k] for k in streams], *[masks[k] for k in streams], w, B, *[lens[k] for k in streams],
                             *ps, ds, **extra)
            for k, o in zip(streams, outs):
                xs[k] = o
            if block_states is not None and len(streams) == 2:
                block_states.append(tuple(xs))
            saved.append(s if need_grad else None)
        return saved

    def backward(self, grads, saved, masks, lens, B):
        """grads: the two streams' output gradients, replaced by the input gradients"""
        for j in range(len(self.steps) - 1, -1, -1):
            _, W, streams = self.steps[j]
            d = W.bwd(*[grads[k] for k in streams], saved[j], *[masks[k] for k in streams], self.weights[j], B,
                      *[lens[k] for k in streams])
            for k, g in zip(streams, d if len(streams) == 2 else (d,)):
                grads[k] = g
            saved[j] = None
            if self.grad_ready_hook is not None:
                self.grad_ready_hook(j)


class _TwoStreamEncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, runner, masks, training, want_blocks, want_attn, x0, x1, *params):
        B = x0.shape[0]
        lens, Hs, dts = (x0.shape[1], x1.shape[1]), (x0.shape[2], x1.shape[2]), (x0.dtype, x1.dtype)
        need_grad = any(ctx.needs_input_grad)
        runner.pack.refresh()
        xs = [x.detach().to(torch.bfloat16).contiguous().view(B * S, H) for x, S, H in zip((x0, x1), lens, Hs)]
        packings = masks if isinstance(masks[0], (_Packing, _StaticPacking)) else None
        if packings is not None:                  # both streams run on their valid rows only
            xs, masks = [pk.pack(x) for pk, x in zip(packings, xs)], [pk.varlen for pk in packings]
        blocks = [] if want_blocks else None
        probs = _probs_sink(*dts) if want_attn else None
        saved = runner.forward(xs, list(masks), lens, B, training, need_grad, blocks, probs)
        ctx.runner, ctx.saved, ctx.masks, ctx.packings, ctx.dims = runner, saved, masks, packings, (B, lens, Hs, dts)
        states = [xs] + (blocks or [])
        outs = [_unpacked(packings, k, t, B, lens).view(B, lens[k], Hs[k]).to(dts[k]) for st in states
                for k, t in enumerate(st)]
        if want_attn:
            # step order, one per query stream (stream 0's first); each in its query stream's dtype
            it = iter(probs)
            outs += [next(it).to(dts[k]) for _, _, streams in runner.steps for k in sorted(streams)]
        if len(outs) > 2:
            ctx.mark_non_differentiable(*outs[2:])
        return tuple(outs)

    @staticmethod
    def backward(ctx, d0, d1, *unused):
        runner = ctx.runner
        B, lens, Hs, dts = ctx.dims
        if ctx.saved is None:
            raise RuntimeError("B200 two-stream encoder: backward called twice")
        aliased = runner.pack.prepare_grads()
        grads = [(d if d is not None else torch.zeros(B, S, H, device=runner.pack.device)).to(torch.bfloat16).contiguous()
                 .view(B * S, H) for d, S, H in zip((d0, d1), lens, Hs)]
        if ctx.packings is not None:
            grads = [pk.pack(d) for pk, d in zip(ctx.packings, grads)]
        runner.backward(grads, ctx.saved, ctx.masks, lens, B)
        ctx.saved = None
        dx = [_unpacked(ctx.packings, k, d, B, lens).view(B, lens[k], Hs[k]).to(dts[k]) for k, d in enumerate(grads)]
        return (None, None, None, None, None) + tuple(dx) + tuple(runner.pack.autograd_grads(aliased))


def _unpacked(packings, k, t, B, lens):
    return t if packings is None else packings[k].unpack(t, B * lens[k])


def run_two_stream_encoder(runner, x0, x1, mask0, mask1, training, want_blocks=False, want_attn=False):
    """x0 / x1: the streams' [B, S, H] states (fp32 or bf16), mask0 / mask1 their additive [B,1,1,S] / [B,S] / None masks.
    Returns the two outputs, then (stream 0, stream 1) after every step that joins the streams if want_blocks, then the
    attention probabilities in step order if want_attn; the block states and probabilities carry no gradient.  With
    `runner.pack_streams` set the layers run on the valid rows (a call that asks for probabilities runs the dense path);
    returns None when every token of both streams is padding, where every output and input-gradient row is zero.
    Inside graphs.static_rows() a runner with `device_plan` set plans the packing on the device instead
    (_static_packings), so the call can be captured: it always runs the packed path at the capacity of every row (never
    returns None), and a sample with tokens in one stream only keeps every row of the other."""
    B, S0, _ = x0.shape
    S1 = x1.shape[1]
    runner.ensure(x0.device)
    masks = (E.additive_mask_2d(mask0, B, S0), E.additive_mask_2d(mask1, B, S1))
    if runner.pack_streams and not want_attn and runner.device_plan and graphs.static_rows_active() and \
            any(m is not None for m in masks):
        masks = tuple(_static_packings(masks, B, (S0, S1)))
    elif runner.pack_streams and not want_attn:
        plan = plan_two_stream(*masks, B, S0, S1, x0.device)
        if plan == "empty":
            return None
        if plan is not None:
            masks = plan
    return _TwoStreamEncoderFn.apply(runner, masks, training, want_blocks, want_attn, x0, x1, *runner.pack.params)


def split_encoder_outputs(outs, n_layers, output_hidden_states, output_attentions):
    """(last, hidden states or None, attentions or None) of run_bert_encoder's outputs; the hidden states in the reference's
    layout: the L layer inputs, then the last output"""
    hidden = tuple(outs[1:1 + n_layers]) + (outs[0],) if output_hidden_states else None
    attn = tuple(outs[len(outs) - n_layers:]) if output_attentions else None
    return outs[0], hidden, attn


class _Holder(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter holder: computed by the B200 engine, not callable")


class B200BertSelfAttention(_Holder):
    def __init__(self, hidden, heads, p_attn, in_hidden=None):
        super().__init__()
        if hidden % heads != 0:
            raise ValueError("The hidden size (%d) is not a multiple of the number of attention heads (%d)" % (hidden, heads))
        self.num_attention_heads = heads
        self.attention_head_size = hidden // heads
        self.all_head_size = hidden
        self.query = nn.Linear(in_hidden or hidden, hidden)
        self.key = nn.Linear(in_hidden or hidden, hidden)
        self.value = nn.Linear(in_hidden or hidden, hidden)
        self.dropout = nn.Dropout(p_attn)


class B200BertSelfOutput(_Holder):
    def __init__(self, in_features, hidden, p_hidden, eps):
        super().__init__()
        self.dense = nn.Linear(in_features, hidden)
        self.LayerNorm = nn.LayerNorm(hidden, eps=eps)
        self.dropout = nn.Dropout(p_hidden)


class B200BertAttention(_Holder):
    def __init__(self, hidden, heads, p_attn, p_hidden, eps):
        super().__init__()
        self.self = B200BertSelfAttention(hidden, heads, p_attn)
        self.output = B200BertSelfOutput(hidden, hidden, p_hidden, eps)


class B200BertIntermediate(_Holder):
    def __init__(self, hidden, inter):
        super().__init__()
        self.dense = nn.Linear(hidden, inter)


class B200BertLayer(_Holder):
    def __init__(self, hidden, heads, inter, p_attn, p_hidden, eps):
        super().__init__()
        self.attention = B200BertAttention(hidden, heads, p_attn, p_hidden, eps)
        self.intermediate = B200BertIntermediate(hidden, inter)
        self.output = B200BertSelfOutput(inter, hidden, p_hidden, eps)


def _init_bert_weights(module, std):
    """normal(0, initializer_range) Linear/Embedding weights, zero biases, LayerNorm (1, 0):
    mmf/models/transformers/base.py:213-223 / HF _init_weights."""
    for m in module.modules():
        if isinstance(m, (nn.Linear, nn.Embedding)):
            m.weight.data.normal_(mean=0.0, std=std)
            if isinstance(m, nn.Linear) and m.bias is not None:
                m.bias.data.zero_()
        elif isinstance(m, nn.LayerNorm):
            m.weight.data.fill_(1.0)
            m.bias.data.zero_()


class B200BertEncoder(nn.Module):
    """BertEncoderJit with the B200 engine underneath.  `config`: a HF BertConfig-like object."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        eps = float(getattr(config, "layer_norm_eps", 1e-12))
        act = getattr(config, "hidden_act", "gelu")
        if act not in ("gelu",) and not callable(act):
            raise ValueError("B200 fusion block implements the erf GELU of the reference configs, got %r" % (act,))
        self.layer = nn.ModuleList([
            B200BertLayer(config.hidden_size, config.num_attention_heads, config.intermediate_size,
                          float(config.attention_probs_dropout_prob), float(config.hidden_dropout_prob), eps)
            for _ in range(config.num_hidden_layers)])
        _init_bert_weights(self, float(getattr(config, "initializer_range", 0.02)))
        self._runner = EncoderRunner(self.layer)
        self._runner.skip_padding = bool(getattr(config, "skip_padding", False))

    def forward(self, hidden_states, attention_mask=None, encoder_hidden_states=None, encoder_attention_mask=None,
                output_attentions=False, output_hidden_states=False, return_dict=False, head_mask=None):
        """Same contract as BertEncoderJit.forward (hf_layers.py:316-355): returns (last_hidden,), then
        (all_hidden_states) if output_hidden_states, then (attn_0, ..., attn_{L-1}) if output_attentions.  The
        probabilities are written by one extra kernel per layer only when asked for; like the hidden states they are
        outputs for inspection and carry no gradient."""
        if head_mask is not None and not (isinstance(head_mask, (list, tuple)) and all(h is None for h in head_mask)):
            raise NotImplementedError("head_mask is not supported on the B200 path")
        # `encoder_hidden_states` is ignored exactly as BertLayerJit ignores it (hf_layers.py:281-283; MMFT passes
        # `[None]*L` there, huggingface.py:229-235)
        outs = run_bert_encoder(self._runner, hidden_states, attention_mask, self.training, output_hidden_states,
                                output_attentions)
        return encoder_result(outs, len(self.layer), output_hidden_states, output_attentions)


def encoder_result(outs, n_layers, output_hidden_states, output_attentions):
    """BertEncoderJit.forward's return structure (hf_layers.py:349-355) from run_bert_encoder's outputs"""
    last, hidden, attn = split_encoder_outputs(outs, n_layers, output_hidden_states, output_attentions)
    return (last,) + ((hidden,) if output_hidden_states else ()) + ((attn,) if output_attentions else ())


# ------------------------------------------------------------------------------------------------------
# ViLBERT two-stream encoder
# ------------------------------------------------------------------------------------------------------
class B200BiAttention(_Holder):
    def __init__(self, cfg):
        super().__init__()
        bi, hv, ht = cfg.bi_hidden_size, cfg.v_hidden_size, cfg.hidden_size
        if bi % cfg.bi_num_attention_heads != 0:
            raise ValueError("The hidden size (%d) is not a multiple of the number of attention heads (%d)"
                             % (bi, cfg.bi_num_attention_heads))
        self.num_attention_heads = cfg.bi_num_attention_heads
        self.attention_head_size = bi // cfg.bi_num_attention_heads
        self.all_head_size = bi
        self.query1, self.key1, self.value1 = nn.Linear(hv, bi), nn.Linear(hv, bi), nn.Linear(hv, bi)
        self.dropout1 = nn.Dropout(cfg.v_attention_probs_dropout_prob)
        self.query2, self.key2, self.value2 = nn.Linear(ht, bi), nn.Linear(ht, bi), nn.Linear(ht, bi)
        self.dropout2 = nn.Dropout(cfg.attention_probs_dropout_prob)


class B200BiOutput(_Holder):
    def __init__(self, cfg):
        super().__init__()
        bi, hv, ht = cfg.bi_hidden_size, cfg.v_hidden_size, cfg.hidden_size
        self.dense1 = nn.Linear(bi, hv)
        self.LayerNorm1 = nn.LayerNorm(hv, eps=1e-12)
        self.dropout1 = nn.Dropout(cfg.v_hidden_dropout_prob)
        self.q_dense1 = nn.Linear(bi, hv)      # present in the reference, never used (vilbert.py:486-494): no grads
        self.q_dropout1 = nn.Dropout(cfg.v_hidden_dropout_prob)
        self.dense2 = nn.Linear(bi, ht)
        self.LayerNorm2 = nn.LayerNorm(ht, eps=1e-12)
        self.dropout2 = nn.Dropout(cfg.hidden_dropout_prob)
        self.q_dense2 = nn.Linear(bi, ht)
        self.q_dropout2 = nn.Dropout(cfg.hidden_dropout_prob)


class B200ConnectionLayer(_Holder):
    def __init__(self, cfg):
        super().__init__()
        self.biattention = B200BiAttention(cfg)
        self.biOutput = B200BiOutput(cfg)
        self.v_intermediate = B200BertIntermediate(cfg.v_hidden_size, cfg.v_intermediate_size)
        self.v_output = B200BertSelfOutput(cfg.v_intermediate_size, cfg.v_hidden_size, cfg.v_hidden_dropout_prob, 1e-12)
        self.t_intermediate = B200BertIntermediate(cfg.hidden_size, cfg.intermediate_size)
        # the text side is HF's BertOutput (config.layer_norm_eps); the image side and biOutput fix 1e-12
        # (vilbert.py:303, 483-490, 520-526)
        self.t_output = B200BertSelfOutput(cfg.intermediate_size, cfg.hidden_size, cfg.hidden_dropout_prob,
                                           float(getattr(cfg, "layer_norm_eps", 1e-12)))


def vilbert_schedule(v_ids, t_ids, n_t, n_v):
    """Layer interleaving of vilbert.BertEncoder.forward (vilbert.py:619-785) as ('t'|'v'|'c', index) steps."""
    steps, v_start, t_start = [], 0, 0
    for count, (v_end, t_end) in enumerate(zip(v_ids, t_ids)):
        steps += [("t", i) for i in range(t_start, t_end)]
        steps += [("v", i) for i in range(v_start, v_end)]
        steps.append(("c", count))
        v_start, t_start = v_end, t_end
    steps += [("v", i) for i in range(v_start, n_v)]
    steps += [("t", i) for i in range(t_start, n_t)]
    return steps


class B200ViLBertEncoder(nn.Module):
    """vilbert.BertEncoder (vilbert.py:559-796) on the B200 engine.  `config` carries the reference's ViLBERT keys
    (mmf/configs/models/vilbert/defaults.yaml).  dynamic_attention, in_batch_pairs, fast_mode and fixed_*_layer > 0
    are configuration corners the reference defaults leave off; they raise here instead of silently differing."""

    def __init__(self, config):
        super().__init__()
        for flag in ("dynamic_attention", "in_batch_pairs", "fast_mode"):
            if getattr(config, flag, False):
                raise NotImplementedError("ViLBERT option %s is not implemented on the B200 path" % flag)
        if getattr(config, "fixed_t_layer", 0) or getattr(config, "fixed_v_layer", 0):
            raise NotImplementedError("fixed_t_layer / fixed_v_layer > 0 are not implemented on the B200 path")
        if not getattr(config, "with_coattention", True):
            raise NotImplementedError("with_coattention=False is not implemented on the B200 path")
        self.config = config
        self.v_biattention_id = list(config.v_biattention_id)
        self.t_biattention_id = list(config.t_biattention_id)
        # text layers: vilbert.BertLayer over HF's BertSelfOutput / BertOutput (config.layer_norm_eps); image layers:
        # BertImageSelfOutput / BertImageOutput, which fix 1e-12 (vilbert.py:131-170, 254, 303)
        self.layer = nn.ModuleList([
            B200BertLayer(config.hidden_size, config.num_attention_heads, config.intermediate_size,
                          float(config.attention_probs_dropout_prob), float(config.hidden_dropout_prob),
                          float(getattr(config, "layer_norm_eps", 1e-12)))
            for _ in range(config.num_hidden_layers)])
        self.v_layer = nn.ModuleList([
            B200BertLayer(config.v_hidden_size, config.v_num_attention_heads, config.v_intermediate_size,
                          float(config.v_attention_probs_dropout_prob), float(config.v_hidden_dropout_prob), 1e-12)
            for _ in range(config.v_num_hidden_layers)])
        self.c_layer = nn.ModuleList([B200ConnectionLayer(config) for _ in range(len(self.v_biattention_id))])
        _init_bert_weights(self, float(getattr(config, "initializer_range", 0.02)))
        kinds = {"t": (self.layer, E.BertLayerW, (0,)), "v": (self.v_layer, E.BertLayerW, (1,)),
                 "c": (self.c_layer, E.ConnectionW, (1, 0))}
        self._runner = TwoStreamRunner([(kinds[k][0][i],) + kinds[k][1:] for k, i in vilbert_schedule(
            self.v_biattention_id, self.t_biattention_id, len(self.layer), len(self.v_layer))])
        self._runner.pack_streams = bool(getattr(config, "skip_padding", False))

    def forward(self, txt_embedding, image_embedding, txt_attention_mask, txt_attention_mask2, image_attention_mask,
                co_attention_mask=None, output_all_encoded_layers=True, output_all_attention_masks=False):
        """Same signature / return structure as vilbert.BertEncoder.forward (vilbert.py:590-796):
        ([text layers], [image layers], ([], [], [])).  co_attention_mask is accepted and, like in the reference
        (vilbert.py:424-425,448-449), not applied.  output_all_encoded_layers=True reproduces the reference's lists: ONE
        entry per co-attention block - the states right after that block - and NOT the final states (vilbert.py:761-763,
        787-790).  Those per-block tensors are outputs for inspection: they carry no gradient here (the reference would
        back-propagate through them); the differentiable result is the default output_all_encoded_layers=False path.

        output_all_attention_masks=True with `config.visualization` set returns the reference's third element
        (vilbert.py:611-795): the text layers' probabilities [B, h, T, T] and the image layers' [B, h, R, R] in schedule
        order, and per co-attention block the pair (attn1, attn2) = (text queries over image keys [B, h, T, R], image
        queries over text keys [B, h, R, T]); post-dropout in training, in the stream's dtype.  One extra kernel per
        attention call writes them, and like the per-block states they carry no gradient.  A call that asks for them runs
        the dense path even with skip_padding set.  Without `visualization` the lists are empty, as in the reference, and
        nothing extra runs."""
        _require_cuda(txt_embedding, "txt_embedding")
        want_attn = bool(output_all_attention_masks) and bool(getattr(self.config, "visualization", False))
        outs = run_two_stream_encoder(self._runner, txt_embedding, image_embedding, txt_attention_mask, image_attention_mask,
                                      self.training, bool(output_all_encoded_layers), want_attn)
        if outs is None:
            # every token of both streams is padding: every output (and input-gradient) row is zero
            zt, zi = txt_embedding * 0, image_embedding * 0
            if output_all_encoded_layers:
                n = len(self.c_layer)
                return [zt.detach()] * n, [zi.detach()] * n, ([], [], [])
            return [zt], [zi], ([], [], [])
        nb = 2 * len(self.c_layer) if output_all_encoded_layers else 0
        blocks, attn = outs[2:2 + nb], iter(outs[2 + nb:])
        att_t, att_v, att_c = [], [], []
        for _, _, streams in self._runner.steps if want_attn else ():
            if len(streams) == 2:
                att_c.append((next(attn), next(attn)))
            else:
                (att_v if streams == (1,) else att_t).append(next(attn))
        if output_all_encoded_layers:
            return list(blocks[0::2]), list(blocks[1::2]), (att_t, att_v, att_c)
        return [outs[0]], [outs[1]], (att_t, att_v, att_c)
