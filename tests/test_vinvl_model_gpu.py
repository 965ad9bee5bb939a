"""The registered `vinvl` model on the GPU against tests/golden/vinvl_model.pt (the REFERENCE's own registered VinVL,
tools/make_golden_vinvl_model.py): classification, pretraining, and pretraining with every MLM label ignored.  Bars as for
the UNITER model (bf16 kernels against an fp32 reference): losses within 1e-2, scores within 1.5e-2, 2-D gradients within
3e-2 relative L2 - 5e-2 for the attention query / key weights; attention masks bit for bit.  Then one bert-base,
2054-feature pretraining step at a realistic shape, and skip-padding against the dense path on a padded batch."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_vinvl_model_cpu as C  # noqa: E402  (builders, sample lists and the golden check shared with the CPU test)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(C.GOLD, "vinvl_model.pt"), weights_only=False)


def _models():
    import mmf_b200.mmft  # noqa: F401
    import mmf_b200.models as MD
    return MD


@pytest.mark.parametrize("case", C.CASES)
def test_registered_model_vs_reference_golden_on_gpu(golden, case):
    from mmf_b200 import lib
    model = C._build(_models(), golden, case).cuda()
    n0 = lib.launch_count()
    _, worst = C.check_case(model, golden, case, "cuda", 1e-2, 1.5e-2,
                            lambda k: 5e-2 if ".self.query." in k or ".self.key." in k else 3e-2)
    torch.cuda.synchronize()
    assert lib.launch_count() > n0                       # the library's own kernels ran
    print("\nvinvl %s: " % case + "  ".join("%s %.2e" % kv for kv in worst.items()))


def test_pretraining_gradients_are_the_sum_of_both_trunk_passes_on_gpu(golden):
    MD = _models()
    g = golden["pretraining"]
    model = C._build(MD, golden, "pretraining").cuda()
    named = dict(model.named_parameters())
    own = {}
    for loss_name in g["losses"]:
        model.zero_grad(set_to_none=True)
        model(C._sample_list(golden, "pretraining", "cuda"))["losses"][loss_name].backward()
        own[loss_name] = {k: named[k].grad.clone() for k in g["by_loss"][loss_name]["grads"]}
        for k, ref in g["by_loss"][loss_name]["grads"].items():
            tol = 5e-2 if ".self.query." in k else 3e-2
            assert C.rel(own[loss_name][k].cpu(), ref) < tol, (loss_name, k, C.rel(own[loss_name][k].cpu(), ref))
    model.zero_grad(set_to_none=True)
    sum(model(C._sample_list(golden, "pretraining", "cuda"))["losses"].values()).backward()
    for k in own["masked_lm_loss"]:
        parts = own["masked_lm_loss"][k] + own["three_way_contrastive_loss"][k]
        assert C.rel(named[k].grad, parts) < 1e-3, k


def _padded_batch(B, T, R, feat, vocab, dev, seed):
    from mmf_b200.sample import SampleList
    g = torch.Generator().manual_seed(seed)

    def mask(n, lo):
        lens = torch.randint(lo, n + 1, (B,), generator=g)
        return lens, (torch.arange(n)[None] < lens[:, None]).long()

    _, m = mask(T, 3)
    _, mc = mask(T, 3)
    nreg, _ = mask(R, 1)
    ids = torch.randint(1, vocab, (B, T), generator=g)
    labels = torch.full((B, T), -1, dtype=torch.long)
    pick = (torch.rand(B, T, generator=g) < 0.2) & (m == 1)
    pick[:, 1] = True                                    # at least one labelled (valid) token per sample
    labels[pick] = ids[pick]
    return SampleList(input_ids=ids, input_ids_masked=torch.where(pick, torch.full_like(ids, 3), ids),
                      input_ids_corrupt=torch.randint(1, vocab, (B, T), generator=g), lm_label_ids=labels,
                      input_mask=m, input_mask_corrupt=mc, segment_ids=torch.zeros(B, T, dtype=torch.long),
                      segment_ids_corrupt=torch.zeros(B, T, dtype=torch.long),
                      image_feature_0=torch.randn(B, R, feat, generator=g), image_info_0={"max_features": nreg},
                      contrastive_labels=torch.randint(0, 3, (B, 1), generator=g),
                      labels=torch.randint(0, 7, (B,), generator=g), dataset_name="test", dataset_type="train").to(dev)


def test_bert_base_pretraining_step_is_finite():
    """one training step of the registered model at VinVL's shape: bert-base, 35 tokens + 50 regions x 2054, dropout 0.1"""
    MD = _models()
    from mmf_b200 import lib
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("vinvl", overrides={"do_pretraining": True, "heads": {}})).cuda().train()
    assert len(model.vinvl.bert.encoder.layer) == 12 and model.vinvl.bert.img_embedding[0].in_features == 2054
    sl = _padded_batch(32, 35, 50, 2054, 30522, "cuda", 11)
    n0 = lib.launch_count()
    out = model(sl)
    loss = sum(out["losses"].values())
    loss.backward()
    torch.cuda.synchronize()
    assert lib.launch_count() > n0
    assert all(torch.isfinite(v) and v > 0 for v in out["losses"].values()), out["losses"]
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert len(grads) > 190 and all(torch.isfinite(gr).all() for gr in grads)
    print("\nvinvl bert-base step: " + "  ".join("%s %.4f" % (k, float(v)) for k, v in out["losses"].items()))


@pytest.mark.parametrize("case", ["pretraining", "classification"])
def test_skip_padding_matches_the_dense_path(golden, case):
    """text and regions laid out [text | pad | regions | pad] pack as they stand; both losses read valid rows only
    (labelled text positions, row 0), so packed and dense agree up to rounding"""
    MD = _models()
    from mmf_b200.patch import set_skip_padding
    over = dict(golden[case]["config"])
    model = C._build(MD, golden, case).cuda()
    assert over["do_pretraining"] == (case == "pretraining")
    sl = _padded_batch(8, 12, 9, 46, 50, "cuda", 23)
    res, trunk_out = {}, []
    hook = model.vinvl.bert.register_forward_hook(lambda mod, a, o: trunk_out.append(o.last_hidden_state.detach()))
    image_mask = MD.image_mask_from_dim(sl["image_feature_0"], sl["image_info_0"]["max_features"].cuda())
    pad = torch.cat([sl["input_mask"], image_mask], dim=1) == 0
    assert pad.any()
    for mode in ("dense", "packed"):
        assert set_skip_padding(model, mode == "packed") == 1
        model.zero_grad(set_to_none=True)
        trunk_out.clear()
        out = model(sl)
        sum(out["losses"].values()).backward()
        # the packed path computes no padded row: its trunk output is exactly zero there, the dense path's is not
        assert (trunk_out[0][pad] == 0).all() == (mode == "packed"), mode
        res[mode] = ({k: float(v) for k, v in out["losses"].items()},
                     {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None})
    hook.remove()
    set_skip_padding(model, False)
    worst = {"loss": 0.0, "grad": 0.0}
    for k, v in res["dense"][0].items():
        e = abs(res["packed"][0][k] - v) / max(abs(v), 1e-3)
        worst["loss"] = max(worst["loss"], e)
        assert e < 1e-2, (k, res["packed"][0][k], v)
    assert res["dense"][1].keys() == res["packed"][1].keys()
    for n, gd in res["dense"][1].items():
        if gd.dim() == 2 and gd.norm() > 1e-6:
            e = C.rel(res["packed"][1][n], gd)
            worst["grad"] = max(worst["grad"], e)
            assert e < (5e-2 if ".self.query." in n or ".self.key." in n else 3e-2), (n, e)
    print("\nvinvl %s skip-padding vs dense: loss %.2e grad %.2e" % (case, worst["loss"], worst["grad"]))
