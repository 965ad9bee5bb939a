"""Attention probabilities (output_attentions, ViLBERT visualization) on the CPU: the encoders' orchestration over the kernel
test double (tests/fake_kernels.py), with a torch restatement of functional.attention_probs injected next to it.  Checks the
return structures against the reference's own modules (BertEncoderJit, ViTEncoder, ViLBERT BertEncoder, loaded through
oracle.ref_loader), that asking for the probabilities changes no output or gradient, the keep bits in train mode, the
skip-padding dense fallback, VisualBERT's empty attention_weights, the wrapper's argument checks and the C ABI entry point
without a GPU.

The test double keeps activations in bf16 as the kernels do, so values are compared with the reference's fp32 modules at
bf16 tolerance; the structure (tuple layout, list lengths, order, shapes) must match exactly."""
import ctypes
import types

import pytest
import torch

from mmf_b200 import engine as E

import fake_kernels as FK

CALLS = {"probs": 0, "varlen": 0}
RECORD = []


def _attention_probs(q, k, lse2, B, heads, Sq, Skv, mask=None, drop_mask=None, drop_scale=1.0, dtype=torch.float32,
                     out=None):
    """contract of functional.attention_probs: exp2(S log2(e)/sqrt(d) + log2(e) max(mask, -10000) - lse2) (* keep * scale)"""
    CALLS["probs"] += 1
    assert dtype in (torch.float32, torch.bfloat16)
    assert tuple(lse2.shape) == (B, heads, Sq)
    m = mask.clamp_min(-10000.0) if mask is not None else None
    p = torch.exp2(FK._probs(q, k, B, heads, Sq, Skv, m) * FK.LOG2E - lse2.unsqueeze(-1))
    if drop_mask is not None:
        assert tuple(drop_mask.shape) == (B, heads, Sq, (Skv + 31) // 32)
        p = torch.where(FK.unpack_keep_bits(drop_mask, Skv), p * drop_scale, torch.zeros_like(p))
    RECORD.append((drop_mask, drop_scale))
    return p.to(dtype)


def _no_varlen(*a, **k):
    CALLS["varlen"] += 1
    raise AssertionError("a call that asks for attention probabilities must run the dense path")


@pytest.fixture()
def fake(monkeypatch):
    monkeypatch.setattr(FK, "attention_probs", _attention_probs, raising=False)
    for name in ("attention_varlen_fwd", "attention_varlen_cross_fwd"):
        monkeypatch.setattr(FK, name, _no_varlen, raising=False)
    monkeypatch.setattr(E, "F", FK)
    import mmf_b200.modules as M
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    CALLS["probs"] = CALLS["varlen"] = 0
    RECORD.clear()
    yield M


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-12)).item()


def _bf16_round_(module):
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(p.to(torch.bfloat16).float())


def _ref(name):
    """the reference's own module file through the loader; skipped where no reference tree can be found"""
    from oracle import ref_loader as RL
    try:
        return getattr(RL, name)()
    except (FileNotFoundError, ImportError) as e:        # pragma: no cover - depends on the machine
        pytest.skip("reference sources not available: %s" % e)


def _padding_mask(B, S):
    valid = torch.ones(B, S, dtype=torch.bool)
    valid[0, S - 3:] = False           # suffix padding
    valid[1, :2] = False               # left padding
    return (~valid).float() * -10000.0


# ---------------------------------------------------------------------------------------------------------------------
# BertEncoderJit
# ---------------------------------------------------------------------------------------------------------------------
def _bert_pair(output_attentions, output_hidden_states, layers=2):
    from transformers import BertConfig
    hf = _ref("hf_layers")
    cfg = BertConfig(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=layers,
                     hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, vocab_size=50,
                     output_attentions=output_attentions, output_hidden_states=output_hidden_states)
    torch.manual_seed(3)
    ref = hf.BertEncoderJit(cfg).eval()
    _bf16_round_(ref)
    return ref, cfg


@pytest.mark.parametrize("hidden", [False, True])
def test_bert_encoder_matches_reference_structure_and_values(fake, hidden):
    ref, cfg = _bert_pair(True, hidden)
    enc = fake.B200BertEncoder(cfg).eval()
    missing, _ = enc.load_state_dict(ref.state_dict(), strict=False)
    assert not missing
    x = torch.randn(3, 10, 64).to(torch.bfloat16).float()
    add = _padding_mask(3, 10)[:, None, None, :]
    with torch.no_grad():
        want = ref(x, add, output_attentions=True, output_hidden_states=hidden)
        got = enc(x, add, output_attentions=True, output_hidden_states=hidden)
    assert len(got) == len(want) == (3 if hidden else 2)
    attn_got, attn_want = got[-1], want[-1]
    assert isinstance(attn_got, tuple) and len(attn_got) == len(attn_want) == 2
    for g, w in zip(attn_got, attn_want):
        assert g.shape == w.shape == (3, 2, 10, 10) and g.dtype == w.dtype
        assert (g - w).abs().max().item() < 1e-2 and rel(g, w) < 1e-2
        assert torch.allclose(g.sum(-1), torch.ones(3, 2, 10), atol=1e-5)
    if hidden:
        assert len(got[1]) == len(want[1]) == 3
    assert rel(got[0], want[0]) < 2e-2
    assert CALLS["probs"] == 2


def test_patched_hf_encoder_returns_attentions(fake):
    from transformers import BertConfig
    from transformers.models.bert.modeling_bert import BertEncoder
    from mmf_b200.patch import attach_encoder
    cfg = BertConfig(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=3, vocab_size=50,
                     hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    enc = attach_encoder(BertEncoder(cfg)).eval()
    x = torch.randn(2, 7, 64)
    with torch.no_grad():
        out = enc(x, None, output_attentions=True, output_hidden_states=True)
        plain = enc(x, None)
    assert len(out) == 3 and len(out[1]) == 4 and len(out[2]) == 3
    assert all(a.shape == (2, 2, 7, 7) for a in out[2])
    assert torch.equal(out[0], plain[0]) and len(plain) == 1


def _run(enc, x, add, w, **kw):
    x = x.clone().requires_grad_(True)
    enc.zero_grad(set_to_none=True)
    outs = enc(x, add, **kw)
    (outs[0] * w).sum().backward()
    return outs, x.grad, {k: p.grad.clone() for k, p in enc.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_flag_changes_no_output_or_gradient(fake, p):
    from transformers import BertConfig
    cfg = BertConfig(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=2, vocab_size=50,
                     hidden_dropout_prob=p, attention_probs_dropout_prob=p)
    torch.manual_seed(5)
    enc = fake.B200BertEncoder(cfg).train(p > 0)
    x, w = torch.randn(2, 9, 64), torch.randn(2, 9, 64)
    add = _padding_mask(2, 9)
    fake._SEED_COUNTER[0] = 0
    off, dx_off, g_off = _run(enc, x, add, w)
    fake._SEED_COUNTER[0] = 0
    on, dx_on, g_on = _run(enc, x, add, w, output_attentions=True)
    assert torch.equal(off[0], on[0]) and torch.equal(dx_off, dx_on)
    assert g_off.keys() == g_on.keys() and all(torch.equal(g_off[k], g_on[k]) for k in g_off)
    assert len(on[1]) == 2 and not any(a.requires_grad for a in on[1])
    if p > 0:
        # train mode: the probabilities use the forward's own keep bits: dropped entries 0, kept ones scaled by 1/(1-p)
        for a, (bits, scale) in zip(on[1], RECORD):
            assert bits is not None and scale == pytest.approx(1.0 / (1.0 - p))
            keep = FK.unpack_keep_bits(bits, 9)
            real = (add == 0)[:, None, None, :].expand_as(keep)              # padded keys have P = 0 either way
            assert not a[~keep].any() and (a[keep & real] > 0).all()
            assert (~keep & real).any() and (a.sum(-1) < scale + 1e-5).all()


def test_eval_under_no_grad_and_bf16_inputs(fake):
    from transformers import BertConfig
    cfg = BertConfig(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=1, vocab_size=50,
                     hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    enc = fake.B200BertEncoder(cfg).eval()
    with torch.no_grad():
        out = enc(torch.randn(2, 5, 64).to(torch.bfloat16), None, output_attentions=True)
    assert out[1][0].dtype == torch.bfloat16 and RECORD[0][0] is None       # eval: no keep bits
    with torch.no_grad():
        out = enc(torch.randn(2, 5, 64).to(torch.float16), None, output_attentions=True)
    assert out[1][0].dtype == torch.float16                                 # other dtypes: cast on the host


def test_skip_padding_runs_dense_when_probabilities_are_asked_for(fake):
    from transformers import BertConfig
    cfg = BertConfig(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=2, vocab_size=50,
                     hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    torch.manual_seed(6)
    enc = fake.B200BertEncoder(cfg).eval()
    x, add = torch.randn(2, 8, 64), _padding_mask(2, 8)
    with torch.no_grad():
        dense = enc(x, add, output_attentions=True)
        enc._runner.skip_padding = True
        packed = enc(x, add, output_attentions=True)
    assert CALLS["varlen"] == 0
    assert torch.equal(dense[0], packed[0])
    assert all(torch.equal(a, b) and a.shape == (2, 2, 8, 8) for a, b in zip(dense[1], packed[1]))


# ---------------------------------------------------------------------------------------------------------------------
# ViT
# ---------------------------------------------------------------------------------------------------------------------
def test_vit_encoder_matches_reference(fake):
    from transformers import ViTConfig
    import mmf_b200.vit as VT
    vit = _ref("vit")
    cfg = ViTConfig(hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                    hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, image_size=32, patch_size=8,
                    layer_norm_eps=1e-12)
    cfg.chunk_size_feed_forward, cfg.is_decoder, cfg.position_embedding_type, cfg.max_position_embeddings = 0, False, "absolute", 64
    torch.manual_seed(7)
    ref = vit.ViTEncoder(cfg).eval()
    _bf16_round_(ref)
    enc = VT.B200ViTEncoder(cfg).eval()
    missing, _ = enc.load_state_dict(ref.state_dict(), strict=False)
    assert not missing
    x = torch.randn(2, 11, 128).to(torch.bfloat16).float()
    add = _padding_mask(2, 11)[:, None, None, :]
    with torch.no_grad():
        want = ref(x, add, output_attentions=True, output_hidden_states=True, return_dict=True)
        got = enc(x, add, output_attentions=True, output_hidden_states=True, return_dict=True)
        tup = enc(x, add, output_attentions=True, return_dict=False)
    assert len(got.attentions) == len(want.attentions) == 2 and len(got.hidden_states) == len(want.hidden_states)
    for g, w in zip(got.attentions, want.attentions):
        assert g.shape == w.shape == (2, 2, 11, 11)
        assert (g - w).abs().max().item() < 1e-2 and rel(g, w) < 1e-2
    assert len(tup) == 2 and len(tup[1]) == 2
    assert enc(x, add, return_dict=True).attentions is None


# ---------------------------------------------------------------------------------------------------------------------
# ViLBERT
# ---------------------------------------------------------------------------------------------------------------------
def _vilbert_cfg(visualization, p=0.0):
    return types.SimpleNamespace(
        hidden_size=64, num_attention_heads=1, intermediate_size=128, num_hidden_layers=3,
        v_hidden_size=128, v_num_attention_heads=2, v_intermediate_size=128, v_num_hidden_layers=2,
        bi_hidden_size=128, bi_num_attention_heads=2, v_biattention_id=[0, 1], t_biattention_id=[1, 2],
        hidden_act="gelu", v_hidden_act="gelu", hidden_dropout_prob=p, v_hidden_dropout_prob=p,
        attention_probs_dropout_prob=p, v_attention_probs_dropout_prob=p, layer_norm_eps=1e-12,
        fast_mode=False, with_coattention=True, in_batch_pairs=False, fixed_t_layer=0, fixed_v_layer=0,
        dynamic_attention=False, visualization=visualization, chunk_size_feed_forward=0, is_decoder=False,
        add_cross_attention=False, position_embedding_type="absolute", _attn_implementation="eager")


def _vilbert_inputs(B=2, T=7, R=5):
    g = torch.Generator().manual_seed(8)
    txt = torch.randn(B, T, 64, generator=g).to(torch.bfloat16).float()
    img = torch.randn(B, R, 128, generator=g).to(torch.bfloat16).float()
    tm, im = _padding_mask(B, T), _padding_mask(B, R)
    return txt, img, tm[:, None, None, :], im[:, None, None, :]


@pytest.mark.parametrize("all_layers", [False, True])
def test_vilbert_visualization_matches_reference(fake, all_layers):
    vb = _ref("vilbert")
    cfg = _vilbert_cfg(True)
    torch.manual_seed(9)
    ref = vb.BertEncoder(cfg).eval()
    _bf16_round_(ref)
    enc = fake.B200ViLBertEncoder(cfg).eval()
    missing, _ = enc.load_state_dict(ref.state_dict(), strict=False)
    assert not missing
    txt, img, tm, im = _vilbert_inputs()
    with torch.no_grad():
        want = ref(txt, img, tm, tm, im, None, output_all_encoded_layers=all_layers, output_all_attention_masks=True)
        got = enc(txt, img, tm, tm, im, None, output_all_encoded_layers=all_layers, output_all_attention_masks=True)
    (wt, wv, wc), (gt, gv, gc) = want[2], got[2]
    assert len(gt) == len(wt) == 3 and len(gv) == len(wv) == 2 and len(gc) == len(wc) == 2
    assert len(got[0]) == len(want[0]) and len(got[1]) == len(want[1])
    for g, w in list(zip(gt, wt)) + list(zip(gv, wv)):
        assert g.shape == w.shape
        assert (g - w).abs().max().item() < 2e-2 and rel(g, w) < 2e-2
    for (g1, g2), (w1, w2) in zip(gc, wc):
        assert g1.shape == w1.shape == (2, 2, 7, 5) and g2.shape == w2.shape == (2, 2, 5, 7)
        assert (g1 - w1).abs().max().item() < 2e-2 and (g2 - w2).abs().max().item() < 2e-2
    assert CALLS["probs"] == 3 + 2 + 2 * 2


def test_vilbert_without_visualization_gives_empty_lists(fake):
    vb = _ref("vilbert")
    cfg = _vilbert_cfg(False)
    ref = vb.BertEncoder(cfg).eval()
    enc = fake.B200ViLBertEncoder(cfg).eval()
    txt, img, tm, im = _vilbert_inputs()
    with torch.no_grad():
        want = ref(txt, img, tm, tm, im, None, output_all_encoded_layers=False, output_all_attention_masks=True)
        got = enc(txt, img, tm, tm, im, None, output_all_encoded_layers=False, output_all_attention_masks=True)
    assert want[2] == ([], [], []) and got[2] == ([], [], []) and CALLS["probs"] == 0


def test_vilbert_flag_changes_nothing_else_and_skips_packing(fake):
    cfg = _vilbert_cfg(True, p=0.1)
    torch.manual_seed(10)
    enc = fake.B200ViLBertEncoder(cfg).train()
    txt, img, tm, im = _vilbert_inputs()
    res = []
    for flag in (False, True):
        enc._runner.pack_streams = flag          # packing is skipped when the probabilities are asked for
        fake._SEED_COUNTER[0] = 0
        t, i = txt.clone().requires_grad_(True), img.clone().requires_grad_(True)
        enc.zero_grad(set_to_none=True)
        out = enc(t, i, tm, tm, im, None, output_all_encoded_layers=False, output_all_attention_masks=flag)
        (out[0][-1].sum() + out[1][-1].square().sum()).backward()
        res.append((out, t.grad, i.grad, {k: p.grad.clone() for k, p in enc.named_parameters() if p.grad is not None}))
    (o0, dt0, di0, g0), (o1, dt1, di1, g1) = res
    assert CALLS["varlen"] == 0
    assert torch.equal(o0[0][-1], o1[0][-1]) and torch.equal(o0[1][-1], o1[1][-1])
    assert torch.equal(dt0, dt1) and torch.equal(di0, di1)
    assert g0.keys() == g1.keys() and all(torch.equal(g0[k], g1[k]) for k in g0)
    assert all(bits is not None for bits, _ in RECORD)                      # train mode: the forward's keep bits
    gt, gv, gc = o1[2]
    assert len(gt) == 3 and len(gv) == 2 and len(gc) == 2


# ---------------------------------------------------------------------------------------------------------------------
# VisualBERT, wrapper, C ABI
# ---------------------------------------------------------------------------------------------------------------------
class _StubTrunk(torch.nn.Module):
    """stands in for the VisualBERT trunk: (sequence_output, pooled_output, attention list) of fixed zeros"""

    def __init__(self, *a):
        super().__init__()
        self.embeddings = torch.nn.Module()
        self.embeddings.word_embeddings = torch.nn.Embedding(11, 8)

    def forward(self, input_ids, *a):
        B = input_ids.shape[0]
        return torch.zeros(B, 4, 8), torch.zeros(B, 8), []


def test_visual_bert_attention_weights_is_the_empty_tuple(monkeypatch):
    """the reference's trunk calls its encoder without output_attentions (visual_bert.py:144-157): attention_weights is
    encoded_layers[1:] = () in both heads' output dicts (visual_bert.py:258-259, 378-379)"""
    import mmf_b200.visual_bert as VBT
    from mmf_b200 import models as MD
    monkeypatch.setattr(VBT, "B200VisualBERTBase", _StubTrunk)
    cfg = types.SimpleNamespace(hidden_size=8, vocab_size=11, output_attentions=True, output_hidden_states=False,
                                hidden_act="gelu", layer_norm_eps=1e-12, initializer_range=0.02)
    out = VBT.B200VisualBERTForPretraining(cfg)(torch.zeros(2, 4, dtype=torch.long), None)
    assert out == {"attention_weights": ()}
    ccfg = MD.ConfigNode({"output_attentions": True, "training_head_type": "classification", "num_labels": 3,
                          "hidden_size": 8, "num_hidden_layers": 1, "num_attention_heads": 1, "intermediate_size": 16})
    model = MD.B200VisualBERTForClassification(ccfg).eval()
    model.classifier = torch.nn.Linear(8, 3)          # the head's own GEMM runs on the GPU only
    out = model(torch.zeros(2, 4, dtype=torch.long), torch.ones(2, 4, dtype=torch.long))
    assert out["attention_weights"] == () and out["scores"].shape == (2, 3)


def test_wrapper_rejects_bad_arguments():
    from mmf_b200 import functional as F
    B, h, Sq, Skv, W = 2, 2, 5, 7, 128
    q = torch.zeros(B * Sq, W, dtype=torch.bfloat16)
    k = torch.zeros(B * Skv, W, dtype=torch.bfloat16)
    lse2 = torch.zeros(B, h, Sq)
    with pytest.raises(ValueError, match="dtype"):
        F.attention_probs(q, k, lse2, B, h, Sq, Skv, dtype=torch.float16)
    with pytest.raises(ValueError, match="row counts"):
        F.attention_probs(q, k, lse2, B, h, Sq + 1, Skv)
    with pytest.raises(ValueError, match="width"):
        F.attention_probs(q, k[:, :64], lse2, B, h, Sq, Skv)
    with pytest.raises(ValueError, match="bf16"):
        F.attention_probs(q.float(), k, lse2, B, h, Sq, Skv)
    with pytest.raises(ValueError, match="mask"):
        F.attention_probs(q, k, lse2, B, h, Sq, Skv, mask=torch.zeros(B, Sq))
    with pytest.raises(ValueError, match="drop_mask"):
        F.attention_probs(q, k, lse2, B, h, Sq, Skv, drop_mask=torch.zeros(B, h, Sq, 2, dtype=torch.int32))
    with pytest.raises(ValueError, match="lse2"):
        F.attention_probs(q, k, lse2[:, :, :-1], B, h, Sq, Skv)
    out = torch.zeros(B, h, Skv, Sq).transpose(-1, -2)
    with pytest.raises(ValueError, match="out"):
        F.attention_probs(q, k, lse2, B, h, Sq, Skv, out=out)
    with pytest.raises(ValueError, match="out"):
        F.attention_probs(q, k, lse2, B, h, Sq, Skv, dtype=torch.bfloat16, out=torch.zeros(B, h, Sq, Skv))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA"):          # valid layouts, but no device: no CPU fallback
            F.attention_probs(q, k, lse2, B, h, Sq, Skv)


def test_probs_symbol_exported_and_needs_a_device():
    from mmf_b200 import lib
    assert "mmfb_attention_probs" in lib.header_symbols() and hasattr(lib.LIB, "mmfb_attention_probs")
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = lib.AttnArgs()
    assert lib.LIB.mmfb_attention_probs(ctypes.byref(a), None, lib.MMFB_PROBS_F32, None) == lib.MMFB_ERR_DEVICE
    assert "no CPU fallback" in lib.last_error()
    assert lib.LIB.mmfb_attention_probs(None, None, 0, None) == lib.MMFB_ERR_ARG


def test_sink_refuses_packed_attention():
    sink = E.ProbsSink()
    vl = E.Varlen(torch.zeros(2, dtype=torch.int32), 1, 0, 0)
    with pytest.raises(ValueError, match="dense"):
        sink.add(None, None, None, 1, 1, 1, 1, vl, None, 1.0)
