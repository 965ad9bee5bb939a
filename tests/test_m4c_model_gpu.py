"""The registered `m4c` and `m4c_captioner` models on the H100 against tests/golden/m4c_model.pt (the reference's own M4C
and M4CCaptioner, tools/make_golden_m4c_model.py), the causality of the decoding steps bit for bit, and one training step
at TextVQA shapes."""
import os
import sys

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


def _grad_tol(k):
    return 5e-2 if ("attention.self.query." in k or "attention.self.key." in k) else 3e-2


def test_training_step_vs_reference_golden(MD, golden):
    model = C.build(MD, golden, device="cuda")
    worst = C.check_train(model, golden, "cuda", 1e-2, 1.5e-2, _grad_tol)
    print("m4c train: " + " ".join("%s=%.2e" % kv for kv in worst.items()))


@pytest.mark.parametrize("case", ["eval", "captioner"])
def test_greedy_decoding_vs_reference_golden(MD, golden, case):
    model = C.build(MD, golden, captioner=case == "captioner", device="cuda")
    e = C.check_decoding(model, golden, case, "cuda", 1.5e-2)
    print("m4c %s: scores=%.2e" % (case, e))


def _mmt_outputs(model):
    seen = []
    hook = model.mmt.register_forward_hook(lambda mod, a, out: seen.append({k: v.detach().clone() for k, v in out.items()}))
    return seen, hook


def test_decoding_steps_are_causal_bit_for_bit(MD, golden):
    """dropout off: the scores of decoding steps <= t do not change by a bit when prev_inds[:, t+1:] change, and the OCR
    outputs of the MMT do not change by a bit when any decoding input changes (an exponential of a masked score underflows
    to exactly 0, so any leak through the tail would show)"""
    model = C.build(MD, golden, device="cuda").train()
    i = golden["inputs"]
    assert (i["text_len"] > 0).all()        # every sample has a valid encoding key
    A = golden["num_final_outputs"] - golden["config"]["classifier"]["ocr_max_num"]
    D = i["train_prev_inds"].shape[1]
    seen, hook = _mmt_outputs(model)
    with torch.no_grad():
        base = model(C.sample_list(golden, "cuda"))["scores"]
        for t in range(D - 1):
            prev = i["train_prev_inds"].clone()
            prev[:, t + 1:] = (prev[:, t + 1:] + 7) % (A + 5)
            scores = model(C.sample_list(golden, "cuda", train_prev_inds=prev))["scores"]
            assert not torch.equal(scores, base)
            assert torch.equal(scores[:, :t + 1], base[:, :t + 1]), t
            assert torch.equal(seen[-1]["mmt_ocr_output"], seen[0]["mmt_ocr_output"]), t
            assert torch.equal(seen[-1]["mmt_txt_output"], seen[0]["mmt_txt_output"]), t
    hook.remove()


def test_textvqa_shape_training_step(MD, golden):
    """the default configuration (bert-base text BERT, 4-layer 768-wide MMT, 5000 answers + 50 OCR copies) at TextVQA
    shapes: 20 question tokens, 100 objects, 50 OCR tokens, 12 decoding steps"""
    from mmf_b200.registry import registry
    from mmf_b200.sample import SampleList
    C.register(golden)
    registry.register(golden["dataset"] + "_num_final_outputs", 5050)
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c")).cuda().train()
    B, T, R, O, D = 32, 20, 100, 50, 12
    dev = "cuda"
    sl = SampleList(text=torch.randint(1, 30522, (B, T), device=dev), text_len=torch.randint(1, T + 1, (B,), device=dev),
                    image_feature_0=torch.randn(B, R, 2048, device=dev).relu(), obj_bbox_coordinates=torch.rand(B, R, 4, device=dev),
                    image_info_0={"max_features": torch.randint(10, R + 1, (B,), device=dev)},
                    context_feature_0=torch.randn(B, O, 300, device=dev), context_feature_1=torch.rand(B, O, 604, device=dev),
                    image_feature_1=torch.randn(B, O, 2048, device=dev).relu(), order_vectors=torch.zeros(B, O, 50, device=dev),
                    ocr_bbox_coordinates=torch.rand(B, O, 4, device=dev),
                    context_info_0={"max_features": torch.randint(0, O + 1, (B,), device=dev)},
                    train_prev_inds=torch.randint(0, 5050, (B, D), device=dev),
                    targets=(torch.rand(B, D, 5050, device=dev) < 0.001).float(),
                    train_loss_mask=(torch.rand(B, D, device=dev) < 0.7).float(), dataset_name="textvqa", dataset_type="train")
    out = model(sl)
    loss = C.loss_of(out)
    loss.sum().backward()
    assert out["scores"].shape == (B, D, 5050) and torch.isfinite(loss).all()
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert len(grads) > 0.9 * len(list(model.parameters()))
    assert all(torch.isfinite(g).all() for g in grads)
