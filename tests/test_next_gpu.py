"""GPU parity of the components SURVEY.md 8f lists after the trunk: the masked-LM pre-training head (+ mmfb_gelu_bwd), the
fused AdamW kernel, the UNITER trunk, the LXMERT encoder (shared cross-attention block), and VisualBERT's
bypass_transformer path - against goldens produced by the reference's own files / the oracle.  (These ran behind
MMFB_STAGED_TESTS in round 1; they are part of the default `-m gpu` suite now.)"""
import math
import os

import pytest
import torch

from oracle.golden_format import kept  # noqa: E402

pytestmark = pytest.mark.gpu


def rel(a, b):
    """relative L2 over the elements the golden b stores (a sampled golden gradient stores some of them)"""
    a, b = kept(a, b)
    a, b = a.double(), b.double()
    return ((a.to(b.device) - b).norm() / b.norm()).item()


@pytest.mark.parametrize("mode", [0, 1])
def test_adamw_kernel_matches_the_oracle(mode):
    """mmfb_adamw over a flat buffer with two hyper-parameter groups + a frozen one, 3 steps, vs the fp32 oracle"""
    import math
    from mmf_b200 import functional as F
    from oracle import fusion_oracle as O
    torch.manual_seed(mode)
    n = 8 * 1000
    p = torch.randn(n, device="cuda")
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    gid = torch.randint(0, 3, (n // 8,), device="cuda", dtype=torch.uint8)
    lr, b1, b2, eps = 3e-3, 0.9, 0.98, 1e-6
    wds = [0.01, 0.0, 0.0]
    ref_p, ref_m, ref_v = p.cpu().clone(), m.cpu().clone(), v.cpu().clone()
    sel = gid.cpu().long().repeat_interleave(8)
    for step in range(1, 4):
        g = torch.randn(n, device="cuda") * 0.1
        hps = []
        for gi in range(3):
            if gi == 2:
                hps.append({"lr": 0.0, "weight_decay": 0.0, "step_size": 0.0, "bc2_sqrt": 1.0})      # frozen group
            elif mode == 0:
                hps.append({"lr": lr, "weight_decay": wds[gi], "bc2_sqrt": 1.0,
                            "step_size": lr * math.sqrt(1 - b2 ** step) / (1 - b1 ** step)})
            else:
                hps.append({"lr": lr, "weight_decay": wds[gi], "step_size": lr / (1 - b1 ** step),
                            "bc2_sqrt": math.sqrt(1 - b2 ** step)})
        F.adamw(p, g, m, v, hps, beta1=b1, beta2=b2, eps=eps, mode=mode, grad_scale=0.5, group_of_block=gid)
        gc = g.cpu() * 0.5
        for gi in range(2):
            idx = sel == gi
            pp, mm, vv = ref_p[idx], ref_m[idx], ref_v[idx]
            (O.adamw_step_transformers if mode == 0 else O.adamw_step_torch)(pp, gc[idx], mm, vv, step, lr, b1, b2, eps, wds[gi])
            ref_p[idx], ref_m[idx], ref_v[idx] = pp, mm, vv
        torch.cuda.synchronize()
        idx = sel < 2
        assert (p.cpu()[idx] - ref_p[idx]).abs().max() <= 2e-6 * ref_p[idx].abs().max()
        assert torch.equal(p.cpu()[sel == 2], ref_p[sel == 2])          # frozen blocks are bit-identical


def test_uniter_model_base_vs_reference_golden():
    """SURVEY.md 8f item 3 (written after the round's GPU budget was spent; CPU-verified over the kernel test double)"""
    import types
    from mmf_b200.uniter import B200UNITERModelBase
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "uniter.pt"), weights_only=False)
    c = g["cfg"]
    cfg = types.SimpleNamespace(hidden_size=c["hidden"], num_attention_heads=c["heads"], intermediate_size=c["inter"],
                                num_hidden_layers=c["layers"], vocab_size=c["vocab"], max_position_embeddings=c["max_pos"],
                                type_vocab_size=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                                layer_norm_eps=1e-12, initializer_range=0.02)
    m = B200UNITERModelBase(cfg, img_dim=c["img_dim"])
    m.load_state_dict({k: v for k, v in g["state_dict"].items() if k in m.state_dict()})
    m = m.cuda().eval()
    cu = lambda k: g[k].cuda()
    feat = cu("feat").requires_grad_(True)
    out = m(cu("ids"), cu("pos_ids"), feat, cu("pos"), cu("att"))
    assert rel(out.final_layer, g["final"]) < 1e-2 and rel(out.hidden_layers[1], g["hidden_1"]) < 1e-2
    (out.final_layer * cu("w_rand")).sum().backward()
    assert rel(feat.grad, g["dfeat"]) < 3e-2
    with torch.no_grad():      # [1, T] position ids broadcast over the batch like HF BertEmbeddings (uniter.py:732-737)
        bc = m(cu("ids"), cu("pos_ids")[:1], cu("feat"), cu("pos"), cu("att")).final_layer
        assert torch.equal(bc, m(cu("ids"), cu("pos_ids"), cu("feat"), cu("pos"), cu("att")).final_layer)


def test_lxmert_encoder_vs_reference_golden():
    """SURVEY.md 8f item 3: cross-modality layers with the shared cross-attention block (CPU-verified over the test double)"""
    import types
    from mmf_b200.lxmert import B200LXMERTEncoder
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "lxmert.pt"), weights_only=False)
    c = g["cfg"]
    cfg = types.SimpleNamespace(hidden_size=c["hidden"], num_attention_heads=c["heads"], intermediate_size=c["inter"],
                                hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, visual_feat_dim=c["feat_dim"],
                                visual_pos_dim=c["pos_dim"], l_layers=c["l"], x_layers=c["x"], r_layers=c["r"])
    enc = B200LXMERTEncoder(cfg)
    enc.load_state_dict(g["state_dict"])
    enc = enc.cuda().eval()
    lang = g["lang"].cuda().requires_grad_(True)
    feats = g["feats"].cuda().requires_grad_(True)
    ladd = ((1.0 - g["lmask"][:, None, None, :].float()) * -10000.0).cuda()
    vadd = ((1.0 - g["vmask"][:, None, None, :].float()) * -10000.0).cuda()
    lo, vo = enc(lang, ladd, (feats, g["boxes"].cuda()), vadd)
    assert rel(lo, g["lang_out"]) < 1e-2 and rel(vo, g["visn_out"]) < 1e-2
    ((lo * g["wl"].cuda()).sum() + (vo * g["wv"].cuda()).sum()).backward()
    assert rel(lang.grad, g["dlang"]) < 3e-2 and rel(feats.grad, g["dfeats"]) < 3e-2
    k = "x_layers.0.visual_attention.att.query.weight"          # shared block: gradient = sum of both directions
    assert rel(dict(enc.named_parameters())[k].grad, g["grads"][k]) < 5e-2


def test_gelu_bwd_kernel_and_masked_lm_head():
    """SURVEY.md 8f item 1: mmfb_gelu_bwd against the fp32 formula, then the head + loss against the HF golden"""
    import math
    import types
    from mmf_b200 import functional as F
    from mmf_b200.heads import B200BertPreTrainingHeads, masked_lm_loss
    torch.manual_seed(0)
    u = (torch.randn(1000, 72, device="cuda") * 2).to(torch.bfloat16)
    dh = torch.randn(1000, 72, device="cuda").to(torch.bfloat16)
    du = F.gelu_bwd(dh, u)
    uf = u.float()
    ref = dh.float() * (0.5 * (1 + torch.erf(uf / math.sqrt(2))) + uf * torch.exp(-0.5 * uf * uf) / math.sqrt(2 * math.pi))
    assert ((du.float() - ref).norm() / ref.norm()).item() < 5e-3
    tail = F.gelu_bwd(dh.reshape(-1)[:13].contiguous(), u.reshape(-1)[:13].contiguous())      # scalar tail path
    assert ((tail.float() - ref.reshape(-1)[:13]).abs().max() < 2e-2)
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "mlm_head.pt"), weights_only=False)
    cfg = types.SimpleNamespace(hidden_size=g["cfg"]["hidden"], vocab_size=g["cfg"]["vocab"], layer_norm_eps=1e-12,
                                initializer_range=0.02)
    cls = B200BertPreTrainingHeads(cfg)
    sd = {k[len("cls."):]: v for k, v in g["state_dict"].items()}
    sd["predictions.decoder.bias"] = sd["predictions.bias"]
    cls.load_state_dict(sd)
    cls = cls.cuda().eval()
    seq = g["seq"].cuda().requires_grad_(True)
    loss, logits = masked_lm_loss(cls, seq, g["labels"].cuda())
    assert rel(logits, g["scores"]) < 1e-2 and abs(loss.item() - g["loss"].item()) < 1e-2 * abs(g["loss"].item())
    loss.backward()
    assert rel(seq.grad, g["dseq"]) < 3e-2


def test_visual_bert_bypass_transformer_vs_reference_golden():
    import types
    from mmf_b200.visual_bert import B200VisualBERTBase
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "visual_bert_bypass.pt"), weights_only=False)
    c = g["cfg"]
    cfg = types.SimpleNamespace(hidden_size=c["hidden"], num_attention_heads=c["heads"], intermediate_size=c["inter"],
                                num_hidden_layers=c["layers"], vocab_size=c["vocab"], max_position_embeddings=c["max_pos"],
                                type_vocab_size=2, visual_embedding_dim=c["vdim"], hidden_dropout_prob=0.0,
                                attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12, hidden_act="gelu",
                                initializer_range=0.02, bypass_transformer=True)
    m = B200VisualBERTBase(cfg)
    m.load_state_dict({k: v for k, v in g["state_dict"].items() if k in m.state_dict()})
    m = m.cuda().eval()
    feats = g["feats"].cuda().requires_grad_(True)
    seq, pooled, _ = m(g["ids"].cuda(), g["att"].cuda(), g["seg"].cuda(), feats, g["vtype"].cuda())
    assert rel(seq, g["seq"]) < 1e-2 and rel(pooled, g["pooled"]) < 1e-2
    (seq * g["w_rand"].cuda()).sum().backward()
    assert rel(feats.grad, g["dfeats"]) < 3e-2


def test_vit_pre_ln_model_vs_reference_golden():
    """SURVEY.md 8f item 3 / kernel row K7: pre-LN (ViT) layers on the B200 kernels vs mmf/modules/vit.py (golden)"""
    import types
    from mmf_b200.vit import B200ViTModel
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vit.pt"), weights_only=False)
    c = g["cfg"]
    cfg = types.SimpleNamespace(hidden_size=c["hidden"], num_attention_heads=c["heads"], intermediate_size=c["inter"],
                                num_hidden_layers=c["layers"], hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                                layer_norm_eps=1e-12, hidden_act="gelu", image_size=c["image_size"], patch_size=c["patch_size"],
                                num_channels=3, initializer_range=0.02)
    m = B200ViTModel(cfg)
    m.load_state_dict(g["state_dict"])
    m = m.cuda().eval()
    x = g["x"].cuda().requires_grad_(True)
    add = ((1.0 - g["mask"][:, None, None, :].float()) * -10000.0).cuda()
    out = m.encoder(x, attention_mask=add, output_hidden_states=True, return_dict=False)
    e_out, e_h = rel(out[0], g["out"]), rel(out[1][1], g["hidden_1"])
    (out[0] * g["w_rand"].cuda()).sum().backward()
    e_dx = rel(x.grad, g["dx"])
    named = dict(m.named_parameters())
    worst = max((rel(named[k].grad, gr), k) for k, gr in g["grads"].items() if "key.bias" not in k)
    print("vit golden: out %.2e hidden %.2e dx %.2e worst dW %.2e (%s)" % (e_out, e_h, e_dx, worst[0], worst[1]))
    assert e_out < 1e-2 and e_h < 1e-2 and e_dx < 1.5e-2 and worst[0] < 3e-2
    with torch.no_grad():
        seq, pooled = m(g["pixels"].cuda())
    assert rel(seq, g["seq_from_pixels"]) < 1e-2 and rel(pooled, g["pooled_from_pixels"]) < 1e-2
    # dropout on: finite, and the two new row kernels agree with torch on the same bits
    from mmf_b200 import functional as F
    xb = torch.randn(300, 768, device="cuda").to(torch.bfloat16)
    yb = torch.randn(300, 768, device="cuda").to(torch.bfloat16)
    assert torch.equal(F.add(xb, yb), (xb.float() + yb.float()).to(torch.bfloat16))
    bits = F.dropout_bits((300,), 768, 0.1, 5, 0, "cuda")
    keep = F.unpack_keep_bits(bits, 768)
    ref = torch.where(keep, xb.float() * (1 / 0.9), torch.zeros(1, device="cuda")).to(torch.bfloat16)
    assert torch.equal(F.dropout_apply(xb, bits, 1 / 0.9), ref)


def test_vinvl_base_vs_reference_golden():
    """SURVEY.md 8f item 3: VinVLBase (mmf/models/vinvl.py:43-122) on the B200 kernels; 46-wide region features exercise the
    same column padding as VinVL's 2054 (both = 6 mod 8)"""
    import types
    from mmf_b200.vinvl import B200VinVLBase
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vinvl.pt"), weights_only=False)
    c = g["cfg"]
    cfg = types.SimpleNamespace(hidden_size=c["hidden"], num_attention_heads=c["heads"], intermediate_size=c["inter"],
                                num_hidden_layers=c["layers"], vocab_size=c["vocab"], max_position_embeddings=c["max_pos"],
                                type_vocab_size=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                                layer_norm_eps=1e-12, initializer_range=0.02, img_feature_dim=c["img_dim"],
                                use_img_layernorm=True, img_layer_norm_eps=1e-12)
    m = B200VinVLBase(cfg)
    m.load_state_dict(g["state_dict"])
    m = m.cuda().eval()
    feats = g["feats"].cuda().requires_grad_(True)
    out = m(g["ids"].cuda(), feats, attention_mask=g["att"].cuda())
    e1, e2 = rel(out.last_hidden_state, g["last"]), rel(out.hidden_layers[1], g["hidden_1"])
    (out.last_hidden_state * g["w_rand"].cuda()).sum().backward()
    e3 = rel(feats.grad, g["dfeats"])
    print("vinvl golden: last %.2e hidden %.2e dfeats %.2e" % (e1, e2, e3))
    assert e1 < 1e-2 and e2 < 1e-2 and e3 < 3e-2


@pytest.mark.parametrize("M,V", [(300, 30528), (17, 208), (1, 8)])
def test_ce_rows_kernel_loss_and_gradient(M, V):
    """mmfb_ce_rows: summed loss and in-place d(logits) vs torch autograd in fp32 on the same bf16 logits"""
    from mmf_b200 import functional as F
    torch.manual_seed(M + V)
    z = (torch.randn(M, V, device="cuda") * 3).to(torch.bfloat16)
    labels = torch.randint(0, V, (M,), device="cuda")
    labels[::4] = -1
    zf = z.float().requires_grad_(True)
    n = int((labels != -1).sum())
    ref = torch.nn.functional.cross_entropy(zf, labels, ignore_index=-1, reduction="sum")
    loss_sum = torch.zeros((), device="cuda")
    row_loss = torch.empty(M, device="cuda")
    scale = 1.0 / max(n, 1)
    F.ce_rows(z, labels, -1, scale, loss_sum, row_loss)
    if n > 0:
        (ref * scale).backward()
        assert abs(loss_sum.item() - ref.item()) <= 2e-3 * abs(ref.item()) + 1e-4
        g = zf.grad
        assert ((z.float() - g).norm() / g.norm()).item() < 5e-3
    assert torch.equal(z[labels == -1].float(), torch.zeros_like(z[labels == -1].float()))       # ignored rows: zero gradient
    assert torch.equal(row_loss[labels == -1], torch.zeros_like(row_loss[labels == -1]))


def test_fused_masked_lm_loss_matches_the_materialised_head():
    """positions="fused" (gather -> transform -> chunked vocabulary GEMM + loss kernel + dgrad/wgrad) vs positions="all" (the
    reference's full logits) at the real vocabulary size: same loss, same gradients, no [tokens, 30522] tensor"""
    import types
    from mmf_b200 import heads as HD
    torch.manual_seed(0)
    cfg = types.SimpleNamespace(hidden_size=768, vocab_size=30522, layer_norm_eps=1e-12, initializer_range=0.02)
    emb = torch.nn.Embedding(cfg.vocab_size, cfg.hidden_size).cuda()
    emb.weight.data.normal_(0, 0.02)
    cls = HD.B200BertPreTrainingHeads(cfg, emb.weight).cuda().eval()
    B, S = 6, 40
    seq = torch.randn(B, S, 768, device="cuda")
    labels = torch.full((B, S), -1, device="cuda")
    labels[:, 3::7] = torch.randint(0, 30522, (B, len(range(3, S, 7))), device="cuda")
    out = {}
    for mode in ("all", "fused"):
        cls.zero_grad(set_to_none=True)
        x = seq.clone().requires_grad_(True)
        loss, logits = HD.masked_lm_loss(cls, x, labels, positions=mode)
        loss.backward()
        out[mode] = (loss.item(), x.grad.clone(), emb.weight.grad.clone(), cls.predictions.transform.dense.weight.grad.clone(),
                     cls.predictions.bias.grad.clone())
        assert (logits is None) == (mode == "fused")
    errs = [abs(out["fused"][0] - out["all"][0]) / abs(out["all"][0])] + [rel(a, b) for a, b in zip(out["fused"][1:], out["all"][1:])]
    print("fused vs materialised MLM head: loss %.2e dseq %.2e dW_vocab %.2e dW_transform %.2e dbias %.2e" % tuple(errs))
    assert max(errs) < 1e-2


def test_graphed_step_replays_the_eager_step_and_redraws_dropout():
    """mmf_b200.graphs.GraphedStep: forward + backward captured as one CUDA graph.  Without dropout a replay reproduces the
    eager loss bit for bit and the gradients to fp32 summation order (same kernels, same order); with dropout every replay draws new masks through the
    device-resident step counter (the host-side seeds are frozen at capture)."""
    import types
    from mmf_b200 import functional as F
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.modules import B200BertEncoder
    torch.manual_seed(0)

    def build(p):
        cfg = types.SimpleNamespace(hidden_size=128, num_attention_heads=2, intermediate_size=256, num_hidden_layers=2,
                                    hidden_dropout_prob=p, attention_probs_dropout_prob=p, layer_norm_eps=1e-12, hidden_act="gelu")
        return B200BertEncoder(cfg).cuda().train()
    B, S = 3, 40
    x = torch.randn(B, S, 128, device="cuda")
    mask = torch.zeros(B, 1, 1, S, device="cuda")
    mask[1, ..., 30:] = -10000.0
    w = torch.randn(B, S, 128, device="cuda")
    loss_fn_of = lambda enc: (lambda b: (enc(b["x"], b["mask"])[0].float() * w).sum())
    # --- no dropout: graph == eager ---
    enc = build(0.0)
    import copy
    twin = copy.deepcopy(enc)            # the eager reference runs on a copy: no autograd graph of `enc` from another stream
    ref = loss_fn_of(twin)({"x": x, "mask": mask})
    ref.backward()
    ref_grads = {n: p.grad.clone() for n, p in twin.named_parameters()}
    ref = ref.detach()
    step = GraphedStep(enc, loss_fn_of(enc), {"x": x, "mask": mask})
    for _ in range(2):
        loss = step({"x": x, "mask": mask})
    torch.cuda.synchronize()
    assert torch.equal(loss, ref)
    for n, p in enc.named_parameters():      # column sums (bias / LayerNorm gradients) are fp32 atomics: same values, free order
        assert (p.grad - ref_grads[n]).abs().max() <= 1e-5 * ref_grads[n].abs().max().clamp_min(1.0), n
    x2 = torch.randn_like(x)
    with torch.no_grad():
        ref2 = loss_fn_of(twin)({"x": x2, "mask": mask})
    assert torch.equal(step({"x": x2, "mask": mask}), ref2)         # new inputs are copied into the static buffers
    # --- dropout: replays differ, and the counter advances ---
    enc = build(0.3)
    step = GraphedStep(enc, loss_fn_of(enc), {"x": x, "mask": mask})
    e0 = int(F.dropout_epoch("cuda").item())
    l1 = step().clone()
    l2 = step().clone()
    torch.cuda.synchronize()
    assert int(F.dropout_epoch("cuda").item()) == e0 + 2
    assert l1.item() != l2.item() and torch.isfinite(l1) and torch.isfinite(l2)
    F._DROPOUT_EPOCH.clear()          # later tests draw their masks from the host-side counters alone
