"""Skip-padding of M4C's multimodal transformer on the H100: the packed encoder call with a causal tail against the dense
one (a 2-layer 768-wide encoder at S = 182, T = 12 over random prefix padding), and the registered `m4c` and
`m4c_captioner` models with set_skip_padding(model, causal=True) against tests/golden/m4c_model.pt and against their
dense path: the loss, every parameter gradient, and the teacher-forced scores at valid answer and OCR slots."""
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_m4c_model_cpu as C  # noqa: E402  (builders, sample lists and the golden checks shared with the CPU test)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(C.GOLD, "m4c_model.pt"), weights_only=False)


@pytest.fixture(scope="module")
def MD():
    import mmf_b200.models as MD
    return MD


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-12)).item()


def _grad_tol(k):
    return 5e-2 if ("attention.self.query." in k or "attention.self.key." in k) else 3e-2


@pytest.fixture()
def packed_calls(monkeypatch):
    """the causal_len of every packed self-attention forward"""
    from mmf_b200 import functional as F
    seen, orig = [], F.attention_varlen_fwd

    def fwd(*a, **k):
        seen.append(k.get("causal_len", 0))
        return orig(*a, **k)
    monkeypatch.setattr(F, "attention_varlen_fwd", fwd)
    return seen


def test_encoder_causal_tail_packed_vs_dense(packed_calls):
    """[text 20 | objects 100 | OCR 50 | 12 decoding steps] with random valid counts per segment, a loss over the kept
    rows: outputs at kept rows, dx and every parameter gradient agree with the dense causal call; padded rows before the
    tail are exactly zero in the output and dx"""
    from mmf_b200.modules import B200BertEncoder, run_bert_encoder
    cfg = types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=2,
                                hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12,
                                initializer_range=0.02)
    torch.manual_seed(0)
    enc = B200BertEncoder(cfg).cuda()
    g = torch.Generator().manual_seed(3)
    B, segs, T, H = 16, (20, 100, 50), 12, 768
    S = sum(segs) + T
    parts = []
    for n in segs:
        cnt = torch.randint(0, n + 1, (B,), generator=g)
        cnt[0] = n                                   # one sample without padding
        parts.append(torch.arange(n)[None] < cnt[:, None])
    parts.append(torch.ones(B, T, dtype=torch.bool))
    kept = torch.cat(parts, 1).cuda()
    add = torch.where(kept, 0.0, -10000.0).float()
    x0 = torch.randn(B, S, H, generator=g).cuda()
    w = torch.randn(B, S, H, generator=g).cuda() * kept[..., None]

    def run(pack):
        enc._runner.skip_padding = enc._runner.pack_tail = pack
        x = x0.clone().requires_grad_(True)
        enc.zero_grad(set_to_none=True)
        out = run_bert_encoder(enc._runner, x, add, True, causal_len=T)[0]
        (out.float() * w).sum().backward()
        return out.detach().float(), x.grad.float(), {k: p.grad.clone() for k, p in enc.named_parameters()}

    od, dxd, gd = run(False)
    assert packed_calls == []
    op, dxp, gp = run(True)
    assert packed_calls == [T, T]
    assert not op[~kept].any() and not dxp[~kept].any()
    e_out, e_dx = rel(op[kept], od[kept]), rel(dxp[kept], dxd[kept])
    e_grad = {k: rel(gp[k], gd[k]) for k in gd if ".key.bias" not in k}      # the key biases are analytically 0
    print("encoder causal packed vs dense: out %.2e dx %.2e grad %.2e" % (e_out, e_dx, max(e_grad.values())))
    assert e_out < 1e-2 and e_dx < 2e-2
    for k, e in e_grad.items():
        assert e < _grad_tol(k), (k, e)


def _step(model, sl):
    model.zero_grad(set_to_none=True)
    out = model(sl)
    loss = C.loss_of(out)
    loss.sum().backward()
    torch.cuda.synchronize()
    return float(loss.detach()), out["scores"].detach(), {n: p.grad.clone() for n, p in model.named_parameters()
                                                          if p.grad is not None}


@pytest.mark.parametrize("captioner", [False, True], ids=["m4c", "m4c_captioner"])
def test_registered_model_packed_vs_golden_and_dense(MD, golden, captioner, packed_calls):
    from mmf_b200.patch import set_skip_padding
    model = C.build(MD, golden, captioner=captioner, device="cuda").train()
    i = golden["inputs"]
    assert (i["ocr_max_features"] < i["context_feature_0"].shape[1]).any()    # the fixture pads OCR slots
    sl = C.sample_list(golden, "cuda")
    ld, sd, gd = _step(model, sl)
    assert packed_calls == []
    assert set_skip_padding(model, causal=True) == 2
    lp, sp, gp = _step(model, sl)
    assert packed_calls.count(i["train_prev_inds"].shape[1]) == len(model.mmt.encoder.layer)
    # against the dense path: the loss, every parameter gradient, the scores at valid answer and OCR slots
    assert abs(lp - ld) <= 1e-2 * abs(ld), (lp, ld)
    assert gp.keys() == gd.keys()
    worst = 0.0
    for k in gd:
        if gd[k].norm() <= 1e-6:
            assert gp[k].norm() <= 1e-5, k
            continue
        e = rel(gp[k], gd[k])
        worst = max(worst, e)
        assert e < _grad_tol(k), (k, e)
    O = i["context_feature_0"].shape[1]
    ocr_valid = (torch.arange(O)[None] < i["ocr_max_features"][:, None]).cuda()
    valid = torch.cat([torch.ones(sd.shape[0], sd.shape[-1] - O, dtype=torch.bool, device="cuda"), ocr_valid], 1)
    valid = valid[:, None, :].expand_as(sd) & (sd > -1000.0)                  # the captioner's <unk> is -1e10 in both
    e_scores = rel(sp[valid], sd[valid])
    assert e_scores < 1e-2, e_scores
    pad = ~ocr_valid[:, None, :].expand(-1, sd.shape[1], -1)
    assert (sp[..., -O:][pad] < -9000).all() and (sd[..., -O:][pad] < -9000).all()
    print("%s packed vs dense: loss %.2e scores %.2e grad %.2e" % ("m4c_captioner" if captioner else "m4c",
                                                                     abs(lp - ld) / abs(ld), e_scores, worst))
    # against the reference's own outputs
    if not captioner:
        model.zero_grad(set_to_none=True)
        worst = C.check_train(model, golden, "cuda", 1e-2, 1.5e-2, _grad_tol)
        print("m4c packed train vs golden: " + " ".join("%s=%.2e" % kv for kv in worst.items()))
    e = C.check_decoding(model, golden, "captioner" if captioner else "eval", "cuda", 1.5e-2)
    print("%s packed decoding vs golden: scores=%.2e" % ("m4c_captioner" if captioner else "m4c", e))
