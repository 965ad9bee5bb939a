"""On the CPU: (1) the generators of tests/operand_scales.py produce the regimes test_operand_scales_gpu.py claims for
them, checked in fp64 (a generator that drifted back to mild inputs would let those tests pass without looking there);
(2) every fused LayerNorm call of the trunks gets its own module's eps.  For (2) the encoders run one forward and
backward over the kernel test double (tests/fake_kernels.py) with a non-default layer_norm_eps; every nn.LayerNorm weight
is filled with its own constant, so a spy on layernorm_fwd / layernorm_bwd tells from gamma which module a call belongs
to."""
import copy
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402
import operand_scales as OS  # noqa: E402

HEADS = 2


# ------------------------------------------------------------------------------------------------------------------
# the generators
# ------------------------------------------------------------------------------------------------------------------
def _gen(kind, Sq, Skv, d, seed, gap=None, where="last"):
    g = torch.Generator().manual_seed(seed)
    q, k, v, keys = OS.attention_sample(kind, Sq, Skv, HEADS, d, g, gap=gap, where=where)
    return q, k, v, keys, OS.scores_log2(q, k, HEADS)


def _gap(Z, keys):
    """per row: the planted max minus the largest other score (log2 units)"""
    others = torch.ones(Z.shape[-1], dtype=torch.bool)
    others[keys] = False
    return Z[..., keys].amin(-1) - Z[..., others].amax(-1)


@pytest.mark.parametrize("d,S", [(64, 65), (64, 384), (128, 65), (128, 256)])
def test_peaked_rows_span_more_than_60_log2_units(d, S):
    _, _, _, _, Z = _gen("peaked", S, S, d, S + d)
    span = Z.amax(-1) - Z.amin(-1)
    assert span.min().item() > 60.0, span.min().item()
    std_nat = (Z / OS.LOG2E).std().item()
    assert 16.0 < std_nat < 24.0, std_nat


@pytest.mark.parametrize("gap,where", [(40.0, "last"), (40.0, "first"), (140.0, "last"), (140.0, "first")])
@pytest.mark.parametrize("d,S", [(64, 65), (64, 200), (64, 384), (128, 256)])
def test_planted_max_lies_in_its_block_and_clears_the_gap(d, S, gap, where):
    _, _, _, keys, Z = _gen("planted", S, S, d, S + d, gap=gap, where=where)
    j = keys[0]
    assert (j // 64 == (S - 1) // 64) if where == "last" else (j < 64)
    assert (Z.argmax(-1) == j).all()
    assert _gap(Z, keys).min().item() >= gap
    if where == "last" and gap > 126:
        # the running max of the earlier blocks is > 126 below: ex2.approx.ftz(m_old - m_new) flushes to exactly 0
        m_old = Z[..., :64 * ((S - 1) // 64)].amax(-1)
        assert (m_old - Z[..., j]).max().item() < -126.0


@pytest.mark.parametrize("d,S", [(64, 65), (64, 384), (128, 256)])
def test_onehot_rows_give_p_exactly_0_or_1_in_fp32(d, S):
    _, _, _, keys, Z = _gen("onehot", S, S, d, S + d)
    assert _gap(Z, keys).min().item() >= 150.0
    Zf = Z.float()
    p = torch.exp2(Zf - Zf.amax(-1, keepdim=True))
    assert ((p == 0) | (p == 1)).all() and (p.sum(-1) == 1).all()


@pytest.mark.parametrize("d,S", [(64, 65), (64, 200), (128, 256)])
def test_ties_share_the_row_max_exactly(d, S):
    q, k, _, keys, Z = _gen("tie", S, S, d, S + d)
    assert len(keys) == 2 and keys[0] < 64 and keys[1] // 64 == (S - 1) // 64
    assert torch.equal(k[keys[0]], k[keys[1]])
    assert torch.equal(Z[..., keys[0]], Z[..., keys[1]]) and (Z.argmax(-1) == keys[0]).all()
    assert _gap(Z, keys).min().item() >= 150.0
    Zf = Z.float()
    p = torch.exp2(Zf - Zf.amax(-1, keepdim=True))
    p = p / p.sum(-1, keepdim=True)
    assert (p[..., keys] == 0.5).all()


@pytest.mark.parametrize("d", [64, 128])
def test_delta_rows_cancel(d):
    """p of the planted key is close to 1 and dctx is its v: dP - delta is a small difference of large terms"""
    g = torch.Generator().manual_seed(d)
    S = 200
    q, k, v, keys = OS.attention_sample("delta", S, S, HEADS, d, g)
    dctx = OS.dctx_for("delta", S, v, keys, g)
    Z = OS.scores_log2(q, k, HEADS)
    P = torch.softmax(Z / OS.LOG2E, -1)
    assert (P[..., keys[0]] > 0.99).all() and (P[..., keys[0]] < 1).all()
    V = v.double().reshape(S, HEADS, d).permute(1, 0, 2)
    dO = dctx.double().reshape(S, HEADS, d).permute(1, 0, 2)
    dP = dO @ V.transpose(-1, -2)
    delta = (dO * (P @ V)).sum(-1, keepdim=True)
    cancel = (dP[..., keys[0]] - delta[..., 0]).abs() / dP[..., keys[0]].abs()
    assert cancel.max().item() < 0.05, cancel.max().item()


@pytest.mark.parametrize("H", [264, 1032, 2040])
def test_layernorm_row_generators(H):
    g = torch.Generator().manual_seed(H)
    M = 40
    for c in (16.0, 64.0):
        y = OS.ln_rows("offset", M, H, g, c=c).double()
        assert (y.mean(1) - c).abs().max() < 0.5 and (y.var(1) - 1).abs().max() < 0.5
        assert y.mean(1).abs().min() > 8 * y.std(1).max()          # the mean dominates the spread
    y = OS.ln_rows("outlier", M, H, g).double()
    big = y.abs() >= 50
    assert ((big.sum(1) >= 2) & (big.sum(1) <= 6)).all() and y.abs().max() <= 200.5
    y = OS.ln_rows("constant", M, H, g).double()
    assert (y == y[:, :1]).all() and (y[0] == 0).all() and (y[1:, 0] != 0).any()
    for eps in (1e-12, 1e-6, 1e-5):
        y = OS.ln_rows("near", M, H, g, eps=eps)
        assert torch.equal(y.float().to(torch.bfloat16), y)                 # exact in bf16 by construction
        var = y.double().var(1, unbiased=False)
        assert ((var >= eps / 10) & (var <= 10 * eps)).all(), (eps, var.min().item(), var.max().item())
        assert (y.double().mean(1) != 0).any()                               # offset rows as well as centred ones


# ------------------------------------------------------------------------------------------------------------------
# eps at every LayerNorm site
# ------------------------------------------------------------------------------------------------------------------
class _Spy:
    """wraps a kernel double's layernorm_fwd / layernorm_bwd; records (gamma value, eps) and gamma values"""

    def __init__(self, double):
        self.fwd_calls, self.bwd_calls = [], []
        fwd, bwd = double.layernorm_fwd, double.layernorm_bwd

        def layernorm_fwd(y, gamma, beta, eps=FK.LN_EPS, **kw):
            self.fwd_calls.append((_gamma_id(gamma), float(eps)))
            kw.pop("m_bound", None)
            return fwd(y, gamma, beta, eps, **kw)

        def layernorm_bwd(dx, y, mean, rstd, gamma, *a, **kw):
            self.bwd_calls.append(_gamma_id(gamma))
            kw.pop("m_bound", None)
            return bwd(dx, y, mean, rstd, gamma, *a, **kw)
        double.layernorm_fwd, double.layernorm_bwd = layernorm_fwd, layernorm_bwd


def _gamma_id(gamma):
    vals = gamma.detach().float().unique()
    assert vals.numel() == 1, "a LayerNorm weight that is not the label this test gave it: %s" % vals[:4].tolist()
    return float(vals[0])


def _label_layernorms(model):
    """fills every nn.LayerNorm weight with its own bf16-exact constant 1 + k / 128; returns {constant: (name, eps)}"""
    table = {}
    with torch.no_grad():
        for k, (name, m) in enumerate((n, m) for n, m in model.named_modules() if isinstance(m, torch.nn.LayerNorm)):
            assert k < 127
            c = 1.0 + (k + 1) / 128.0
            m.weight.fill_(c)
            table[c] = (name, float(m.eps))
    return table


def _assert_eps(spy, table, expect):
    """every fused LayerNorm call got its module's eps, every module had a forward and a backward call, and each module's
    eps is the one `expect(name)` says"""
    assert spy.fwd_calls, "no LayerNorm ran"
    for gid, eps in spy.fwd_calls:
        assert gid in table, "a LayerNorm call with a gamma of no nn.LayerNorm (%r)" % gid
        name, want = table[gid]
        assert eps == want, "%s: the kernel got eps %r, the module has %r" % (name, eps, want)
    seen_f, seen_b = {g for g, _ in spy.fwd_calls}, set(spy.bwd_calls)
    for gid, (name, eps) in table.items():
        assert gid in seen_f, "%s: no fused LayerNorm forward" % name
        assert gid in seen_b, "%s: no fused LayerNorm backward" % name
        assert eps == expect(name), "%s: eps %r, expected %r" % (name, eps, expect(name))


@pytest.fixture()
def double(monkeypatch):
    """the kernel double with the spies, swapped in for every module that launches kernels: tests/fake_kernels.py with
    the entry points the ALBEF ViT (test_albef_vit_cpu), M4C's causal tail (test_m4c_model_cpu) and UNITER's optimal
    transport (test_uniter_model_cpu) add"""
    import importlib
    import mmf_b200.embeddings as EM
    import mmf_b200.engine as E
    import mmf_b200.ops as OPS
    import test_albef_vit_cpu as ACPU
    import test_m4c_model_cpu as M4C
    import test_uniter_model_cpu as UNC
    d = ACPU._double()
    causal = M4C._causal_fake()
    d.attention_fwd, d.attention_bwd = causal.attention_fwd, causal.attention_bwd
    d.ot_fwd, d.ot_bwd = UNC.ot_fwd, UNC.ot_bwd
    monkeypatch.setattr(FK, "_probs", M4C._probs)
    spy = _Spy(d)
    for mod in (E, OPS, EM):
        monkeypatch.setattr(mod, "F", d)
    for name in ("albef_vit", "embeddings", "encoders", "heads", "lxmert", "m4c_model", "mmbt", "mmft_backend",
                 "modules", "uniter", "vilbert", "vinvl", "vit"):
        mod = importlib.import_module("mmf_b200." + name)
        if hasattr(mod, "_require_cuda"):
            monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    return spy


def _bert_cfg(eps, **kw):
    return types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=2,
                                 hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=eps, **kw)


def test_bert_encoder_layernorms_take_layer_norm_eps(double):
    from mmf_b200.modules import B200BertEncoder
    torch.manual_seed(0)
    enc = B200BertEncoder(_bert_cfg(1e-5))
    table = _label_layernorms(enc)
    x = torch.randn(2, 9, 64, requires_grad=True)
    enc(x, None)[0].square().sum().backward()
    _assert_eps(double, table, lambda n: 1e-5)


def test_hf_vit_encoder_layernorms_take_layer_norm_eps(double):
    from mmf_b200.vit import B200ViTEncoder
    torch.manual_seed(1)
    cfg = _bert_cfg(1e-6, hidden_act="gelu", initializer_range=0.02)
    enc = B200ViTEncoder(cfg)
    table = _label_layernorms(enc)
    x = torch.randn(2, 9, 64, requires_grad=True)
    enc(x, return_dict=False)[0].square().sum().backward()
    _assert_eps(double, table, lambda n: 1e-6)


def test_albef_vit_layernorms_take_their_eps(double):
    """ALBEF's VisionTransformer builds every LayerNorm with eps 1e-6 (albef_vit.py refuses others): blocks and the final
    norm"""
    from mmf_b200.encoders import build_encoder
    torch.manual_seed(2)
    enc = build_encoder({"type": "albef_vit_encoder", "params": dict(params=dict(
        img_size=32, patch_size=16, embed_dim=64, num_heads=2, depth=2))})
    table = _label_layernorms(enc)
    images = torch.randn(2, 3, 32, 32, requires_grad=True)
    enc(images).square().sum().backward()
    _assert_eps(double, table, lambda n: 1e-6)


def test_vinvl_layernorms_take_layer_norm_eps_and_img_layer_norm_eps(double):
    """VinVL: the trunk and the text embeddings take layer_norm_eps, the image projection's LayerNorm img_layer_norm_eps"""
    from mmf_b200.vinvl import B200VinVLBase
    torch.manual_seed(3)
    cfg = _bert_cfg(1e-5, vocab_size=50, max_position_embeddings=32, type_vocab_size=2, initializer_range=0.02,
                    img_feature_dim=40, use_img_layernorm=True, img_layer_norm_eps=1e-7)
    m = B200VinVLBase(cfg)
    table = _label_layernorms(m)
    ids = torch.randint(0, 50, (2, 6))
    feats = torch.randn(2, 5, 40, requires_grad=True)
    att = torch.ones(2, 11, dtype=torch.long)
    m(ids, feats, attention_mask=att).last_hidden_state.square().sum().backward()
    _assert_eps(double, table, lambda n: 1e-7 if n.startswith("img_embedding") else 1e-5)


def test_a_site_that_drops_its_eps_is_caught(double, monkeypatch):
    """the check itself: a runner that hands the kernels the library default (1e-12) instead of the module's eps fails it"""
    import mmf_b200.engine as E
    from mmf_b200.vit import B200ViTEncoder
    monkeypatch.setattr(E, "ln_eps", lambda m: 1e-12)
    torch.manual_seed(1)
    enc = B200ViTEncoder(_bert_cfg(1e-6, hidden_act="gelu", initializer_range=0.02))
    table = _label_layernorms(enc)
    x = torch.randn(2, 9, 64, requires_grad=True)
    enc(x, return_dict=False)[0].square().sum().backward()
    with pytest.raises(AssertionError, match="the kernel got eps"):
        _assert_eps(double, table, lambda n: 1e-6)


# ------------------------------------------------------------------------------------------------------------------
# the registered models: one training step each with non-default eps; the modules the reference builds with a fixed
# eps = 1e-12 keep it
# ------------------------------------------------------------------------------------------------------------------
EPS, IMG_EPS = 1e-5, 1e-7
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden(name):
    return torch.load(os.path.join(GOLD, name), weights_only=False)


def _models():
    import mmf_b200.mmft  # noqa: F401  (registers mmf_transformer and its heads)
    import mmf_b200.models as MD
    return MD


def _fixed(*patterns):
    """expect(): 1e-12 for the modules whose name contains one of `patterns`, EPS for every other"""
    return lambda n: 1e-12 if any(p in n for p in patterns) else EPS


def _step(spy, model, loss_fn, expect):
    model.train()
    table = _label_layernorms(model)
    loss_fn(model).backward()
    _assert_eps(spy, table, expect)
    return table


def test_visual_bert_layernorms_take_layer_norm_eps(double):
    import test_models_cpu as MC
    MD, g = _models(), _golden("models.pt")
    cfg = MD.load_model_config("visual_bert", overrides=dict(g["visual_bert_pretraining_default"]["config"],
                                                             layer_norm_eps=EPS))
    cfg.losses = [{"type": "cross_entropy"}]
    torch.manual_seed(0)
    _step(double, MD.build_model(cfg), lambda m: m(MC._sample_list(g))["losses"]["golden/train/masked_lm_loss"],
          _fixed())


def test_vilbert_layernorms_take_layer_norm_eps(double):
    """ViLBERT builds the image stream's LayerNorms with eps = 1e-12 whatever the config says (the reference's
    vilbert.py:254, 303, 483, 490, 837, 901): image embeddings, image layers, the co-attention biOutput and v_output,
    and the image prediction head's transform.  The text stream takes layer_norm_eps."""
    import test_models_cpu as MC
    MD, g = _models(), _golden("models.pt")
    cfg = MD.load_model_config("vilbert", overrides=dict(g["vilbert_pretraining"]["config"], layer_norm_eps=EPS))
    cfg.losses = [{"type": "cross_entropy"}]
    v = g["vilbert_inputs"]
    sl = MC._sample_list(g, {"image_labels": v["image_labels"].clone()})
    sl["image_info_0"] = {"max_features": g["visual_bert_inputs"]["max_features"].clone(), "bbox": v["bbox"].clone(),
                          "cls_prob": v["cls_prob"].numpy().copy()}
    torch.manual_seed(1)
    _step(double, MD.build_model(cfg), lambda m: sum(x.sum() for x in m(sl)["losses"].values()),
          _fixed("v_embeddings.", "v_layer.", "biOutput.LayerNorm", "v_output.", "imagePredictions."))


def test_mmbt_layernorms_take_layer_norm_eps(double):
    from mmf_b200.sample import SampleList
    MD, g = _models(), _golden("mmbt.pt")
    cfg = MD.load_model_config("mmbt", overrides={
        "training_head_type": "classification", "num_labels": 2, "direct_features_input": True, "modal_hidden_size": 40,
        "modal_encoder": {"type": "identity", "params": {"in_dim": 40}},
        "text_encoder": {"type": "transformer", "params": {
            "num_segments": 2, "bert_model_name": None, "hidden_size": 64, "num_hidden_layers": 1,
            "num_attention_heads": 1, "intermediate_size": 128, "vocab_size": 50, "max_position_embeddings": 64,
            "hidden_dropout_prob": 0.0,
            "attention_probs_dropout_prob": 0.0, "layer_norm_eps": EPS}},
        "losses": [{"type": "cross_entropy"}]})
    sl = SampleList(input_ids=g["ids"].clone(), input_mask=g["mask"].clone(), segment_ids=g["seg"].clone(),
                    image_feature_0=g["feats"].clone(), targets=torch.tensor([1, 0]), dataset_name="hm",
                    dataset_type="train")
    torch.manual_seed(2)
    _step(double, MD.build_model(cfg), lambda m: m(sl)["losses"]["train/hm/cross_entropy"].sum(), _fixed())


def test_lxmert_layernorms_take_layer_norm_eps(double):
    """LXMERT's visual feature and box LayerNorms and the answer heads' are built with eps = 1e-12 (the reference's
    lxmert.py:99, 146, 154, 209, 213); every layer, the embeddings and the prediction transforms take layer_norm_eps.
    Two pretraining tasks, so that both the VQA and the GQA answer heads run."""
    import test_lxmert_model_cpu as LXC
    MD, g = _models(), _golden("lxmert_model.pt")
    cfg = MD.load_model_config("lxmert", overrides=dict(g["pretraining_config"], layer_norm_eps=EPS))
    sls = [LXC._sample_list(g, case) for case in ("pretraining_masked_vqa2", "pretraining_masked_gqa")]
    torch.manual_seed(3)
    _step(double, MD.build_model(cfg), lambda m: sum(sum(x.sum() for x in m(sl)["losses"].values()) for sl in sls),
          _fixed("visn_layer_norm", "box_layer_norm", "answer_head."))


def test_mmf_transformer_layernorms_take_their_eps(double):
    """MMF transformer: the backend's encoder layers and every modality's embedding LayerNorm take their own
    layer_norm_eps, the heads theirs"""
    from mmf_b200.sample import SampleList
    MD = _models()
    small = dict(hidden_size=64, num_hidden_layers=1, num_attention_heads=1, intermediate_size=128, vocab_size=512,
                 max_position_embeddings=128, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                 layer_norm_eps=EPS)
    mods = [dict(type="text", key="text", embedding_dim=64, position_dim=128, segment_id=0, layer_norm_eps=EPS),
            dict(type="image", key="image", embedding_dim=48, position_dim=8, segment_id=1,
                 encoder=dict(type="identity"), layer_norm_eps=IMG_EPS)]
    heads = [{"type": "mlp", "hidden_size": 64, "num_labels": 3, "layer_norm_eps": 1e-6},
             {"type": "mlm", "hidden_size": 64, "vocab_size": 512, "layer_norm_eps": 1e-4}]
    cfg = MD.load_model_config("mmf_transformer", overrides={"modalities": mods, "num_labels": 3,
                                                             "transformer_config": small, "heads": heads})
    lab = torch.full((2, 10), -1)
    lab[0, 3], lab[1, 7] = 5, 9
    g = torch.Generator().manual_seed(4)
    sl = SampleList(input_ids=torch.randint(1, 512, (2, 10), generator=g),
                    input_mask=torch.ones(2, 10, dtype=torch.long), image=torch.rand(2, 6, 48, generator=g),
                    lm_label_ids=lab)
    torch.manual_seed(4)

    def loss(m):
        out = m(sl)
        return out["losses"]["masked_lm_loss"] + out["scores"].square().sum()
    def expect(n):
        if n.startswith("heads."):
            return 1e-6 if n.startswith("heads.0") else 1e-4
        return IMG_EPS if n.endswith("layer_norms.1") or ".token_embeddings.1." in n else EPS
    _step(double, MD.build_model(cfg), loss, expect)


def test_vinvl_model_layernorms_take_layer_norm_eps_and_img_layer_norm_eps(double):
    import test_vinvl_model_cpu as VVC
    MD, g = _models(), _golden("vinvl_model.pt")
    c = dict(g["pretraining"]["config"])
    c["bert_overrides"] = dict(c["bert_overrides"], layer_norm_eps=EPS)
    c["img_layer_norm_eps"] = IMG_EPS
    c["heads"] = {"mlm": dict(c["heads"]["mlm"], layer_norm_eps=EPS), "contrast": dict(c["heads"]["contrast"])}
    cfg = MD.load_model_config("vinvl", overrides=c)
    sl = VVC._sample_list(g, "pretraining")
    torch.manual_seed(5)
    _step(double, MD.build_model(cfg), lambda m: sum(x.sum() for x in m(sl)["losses"].values()),
          lambda n: IMG_EPS if "img_embedding" in n else EPS)


def test_vilt_layernorms_take_their_eps(double):
    """ViLT: the ViT trunk (shared by both modalities) takes the image encoder's layer_norm_eps, the text embeddings and
    the heads their own"""
    import test_vilt_model_cpu as VLC
    MD, g = _models(), _golden("vilt_model.pt")
    c = copy.deepcopy(dict(g["pretraining"]["config"]))
    c["image_encoder"]["params"]["layer_norm_eps"] = IMG_EPS
    c["text_embeddings"]["bert_overrides"]["layer_norm_eps"] = EPS
    c["heads"]["masked_coco"] = [dict(h, layer_norm_eps=EPS) for h in c["heads"]["masked_coco"]]
    cfg = MD.load_model_config("vilt", overrides=c)
    sl = VLC._sample_list(g, "pretraining")
    torch.manual_seed(6)
    _step(double, MD.build_model(cfg), lambda m: sum(x.sum() for x in m(sl)["losses"].values()),
          lambda n: EPS if n.startswith(("text_embeddings", "heads")) else IMG_EPS)


def test_uniter_layernorms_take_layer_norm_eps(double):
    """UNITER: text embeddings, encoder and the MLM head take layer_norm_eps, the region heads their `eps`; the image
    embeddings keep 1e-12 (the reference's uniter.py:56-68, built without an eps)"""
    import test_uniter_model_cpu as UNC
    MD, g = _models(), _golden("uniter_model.pt")
    c = copy.deepcopy(dict(g["pretraining_config"]))
    for k in ("text_embeddings", "encoder"):
        c[k]["layer_norm_eps"] = EPS
    c["heads"] = {k: dict(v, layer_norm_eps=EPS) for k, v in c["heads"].items()}
    for k in ("mrc", "mrfr"):                 # the region heads read `eps` (heads/mrc.py, mrfr.py), not layer_norm_eps
        c["heads"][k]["eps"] = 1e-6
    cfg = MD.load_model_config("uniter", overrides=c)
    torch.manual_seed(7)
    model = MD.build_model(cfg)

    def loss(m):              # the seeded draw of each golden case picks that pretraining task
        total = 0.0
        for task in ("mlm", "itm", "mrc", "mrfr"):
            sl = UNC._sample_list(g, task)
            UNC._seed_all(g[task].get("seed", 7))
            total = total + sum(x.sum() for x in m(sl)["losses"].values())
            assert sl["task"] == task
        return total
    _step(double, model, loss,
          lambda n: 1e-12 if "img_embeddings." in n else 1e-6 if ".heads.mr" in n else EPS)


@pytest.mark.parametrize("captioner", [False, True])
def test_m4c_layernorms_take_layer_norm_eps(double, captioner):
    import test_m4c_model_cpu as M4C
    MD, g = _models(), _golden("m4c_model.pt")
    M4C.register(g)
    c = copy.deepcopy(dict(g["captioner_config" if captioner else "config"]))
    c["mmt"]["layer_norm_eps"] = EPS
    c["text_bert"]["layer_norm_eps"] = IMG_EPS
    cfg = MD.load_model_config("m4c_captioner" if captioner else "m4c", overrides=c)
    torch.manual_seed(8)
    _step(double, MD.build_model(cfg), lambda m: M4C.loss_of(m(M4C.sample_list(g))).sum(),
          lambda n: IMG_EPS if n.startswith("text_bert") else EPS)
