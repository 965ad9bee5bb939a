"""Layer-implementation swap by monkey-patch - the reference's own mechanism for this boundary:
`replace_with_jit()` / `undo_replace_with_jit()` (mmf/modules/hf_layers.py:48-93, mmf/utils/patch.py:198-244) rebind
`BertEncoder.forward` & co process-wide from model constructors.  `replace_with_b200()` rebinds the forward of
HuggingFace `BertEncoder` (and every subclass that overrides `forward`, e.g. MMF's `BertEncoderJit`) to the B200 engine
with the contract of `BertEncoderJit.forward` (hf_layers.py:316-355).  Parameters keep their names; their storage is
re-homed into the engine's flat pack on the first CUDA forward.

`set_skip_padding()` switches the single-stream encoders of a model to packed execution: padded tokens are removed once
per encoder call and attention runs over each sample's own tokens (variable-length kernels), so padding costs nothing.
With `two_stream=True` it also packs both streams of the ViLBERT and LXMERT encoders (variable-length cross-attention),
and with `causal=True` the calls with a causal tail (M4C's multimodal transformer: variable-length attention with a tail).
"""
import types

from .modules import EncoderRunner, TwoStreamRunner, encoder_result, run_bert_encoder

_saved = {}


def _b200_encoder_forward(self, hidden_states, attention_mask=None, encoder_hidden_states=None,
                          encoder_attention_mask=None, output_attentions=False, output_hidden_states=False,
                          return_dict=False, head_mask=None, **unused):
    if head_mask is not None and not (isinstance(head_mask, (list, tuple)) and all(h is None for h in head_mask)):
        raise NotImplementedError("head_mask is not supported on the B200 path")
    runner = _runner_of(self)
    outs = run_bert_encoder(runner, hidden_states, attention_mask, self.training, output_hidden_states, output_attentions)
    return encoder_result(outs, len(runner.layers), output_hidden_states, output_attentions)


def _runner_of(encoder):
    r = encoder.__dict__.get("_runner")
    if r is None:
        r = EncoderRunner(encoder.layer)
        object.__setattr__(encoder, "_runner", r)
    return r


def attach_encoder(encoder):
    """Route ONE encoder instance (anything with `.layer[i].attention.self.{query,key,value}` ...) through the engine."""
    _runner_of(encoder)
    encoder.forward = types.MethodType(_b200_encoder_forward, encoder)
    return encoder


def _all_subclasses(cls):
    out = []
    for sub in cls.__subclasses__():
        out.append(sub)
        out += _all_subclasses(sub)
    return out


def replace_with_b200():
    """Process-wide swap, mirroring replace_with_jit()."""
    from transformers.models.bert.modeling_bert import BertEncoder
    for cls in [BertEncoder] + _all_subclasses(BertEncoder):
        if "forward" in cls.__dict__ and cls not in _saved:
            _saved[cls] = cls.__dict__["forward"]
            cls.forward = _b200_encoder_forward


def undo_replace_with_b200():
    """mirrors undo_replace_with_jit()"""
    for cls, fwd in list(_saved.items()):
        cls.forward = fwd
        del _saved[cls]


def _routed(m):
    """True if `m`'s forward is the engine's (replace_with_b200 on its class, or attach_encoder on the instance)"""
    f = m.__dict__.get("forward", None) or getattr(type(m), "forward", None)
    return getattr(f, "__func__", f) is _b200_encoder_forward


def set_skip_padding(module, enabled=True, two_stream=False, causal=False, device_plan=False):
    """Sets `skip_padding` on every single-stream encoder runner under `module` (B200BertEncoder - and so VisualBERT, MMBT,
    UNITER, VinVL and the TransformerEncoder plugin -, VisualBERT's bypass `additional_layer`, encoders routed by
    attach_encoder / replace_with_b200) and returns how many it set.  ViLBERT, LXMERT and ViT runners are left alone unless
    `two_stream` is True: then `pack_streams` is set on every ViLBERT and LXMERT runner too, and they count as well.  ViT
    runners are always left alone.  With `causal` True, `pack_tail` is set as well on the single-stream runners (it counts
    nothing extra): their calls with a causal tail (run_bert_encoder's causal_len, the multimodal transformer of `m4c` and
    `m4c_captioner`) then pack too, keeping every tail row.  Without it such calls run the dense path.

    With the flag on, an encoder call with a key-padding mask runs on the valid rows only: its outputs (and the input
    gradient) are exactly zero at padded positions instead of the values the dense path computes there.  For any loss that
    does not read padded positions it computes the same function and gradients as the dense path, up to rounding and the
    dropout masks drawn.  An eager call reads the token count on the host.  Inside graphs.static_rows() a call without a
    causal tail plans its packing on the device instead, at a fixed capacity of every row, so
    `GraphedStep(..., static_rows=True)` captures such a model.  Calls with a causal tail (`causal`) and two-stream packing
    read the counts on the host there too, and cannot be captured, unless `device_plan` is True: it sets `device_plan` on
    every runner this call touches, and inside static_rows() those plan every stream of a call with one device kernel,
    at the capacity of every row (mmf_b200.modules._static_packings), so that GraphedStep and GraphedForward capture
    them.  Opt-in, because that plan costs the capacity (the packed layers run B*S rows' worth of grid whatever the mask)
    and because of the two-stream rule below.  Outside static_rows() it changes nothing.

    A two-stream call falls back to the dense path when some sample has tokens in one stream and none in the other: there
    the dense outputs of those tokens depend on the other stream's padded rows.  With `device_plan` inside static_rows()
    such a sample instead keeps every row of its empty stream, which the dense path masks uniformly, so its valid outputs
    are the dense ones up to rounding.

    The registered `lxmert` model refuses packed streams (ValueError): like the reference, it passes segment ids as the text
    attention mask, so its text "padding" includes [CLS] and the masked-LM positions.  B200LXMERTBase and
    B200LXMERTEncoder called with real masks keep the packed path.

    A call that asks for attention probabilities (output_attentions, or ViLBERT's output_all_attention_masks with
    `visualization`) also runs the dense path, whatever the flag: the probabilities then have the reference's
    [B, heads, S, S] shape, padded rows and keys included."""
    n = 0
    for m in module.modules():
        r = m.__dict__.get("_runner")
        if r is None and hasattr(m, "layer") and _routed(m):
            r = _runner_of(m)
        if type(r) is EncoderRunner:
            r.skip_padding = bool(enabled)
            if causal:
                r.pack_tail = bool(enabled)
            r.device_plan = bool(device_plan)
            n += 1
        elif two_stream and isinstance(r, TwoStreamRunner):
            r.pack_streams = bool(enabled)
            r.device_plan = bool(device_plan)
            n += 1
    return n
