"""The registered `vilt` model on the GPU against tests/golden/vilt_model.pt (the REFERENCE's own registered ViLT,
tools/make_golden_vilt_model.py): VQA classification with and without masks, masked-LM + ITM pretraining, and pretraining
with every masked-LM label ignored.  Bars as for the VinVL model (bf16 kernels against an fp32 reference): losses within
1e-2, scores within 1.5e-2, gradients within 3e-2 relative L2 - 5e-2 for the attention query / key weights; masks bit for
bit.  Then a training step at the real vit_b32_384 shape against oracle.fusion_oracle's fp32 ViT trunk, and a VQA step
captured by GraphedStep against the eager step, bit for bit under torch.use_deterministic_algorithms."""
import contextlib
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import test_vilt_model_cpu as C  # noqa: E402  (builders, sample lists and the golden check shared with the CPU test)
from oracle import fusion_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(C.GOLD, "vilt_model.pt"), weights_only=False)


def _models():
    import mmf_b200.mmft  # noqa: F401
    import mmf_b200.models as MD
    return MD


def _grad_tol(k):
    return 5e-2 if ".attention.query." in k or ".attention.key." in k else 3e-2


@pytest.mark.parametrize("case", C.CASES)
def test_registered_model_vs_reference_golden_on_gpu(golden, case):
    from mmf_b200 import lib
    model = C._build(_models(), golden, case).cuda()
    n0 = lib.launch_count()
    _, worst = C.check_case(model, golden, case, "cuda", 1e-2, 1.5e-2, _grad_tol)
    torch.cuda.synchronize()
    assert lib.launch_count() > n0                       # the library's own kernels ran
    print("\nvilt %s: " % case + "  ".join("%s %.2e" % kv for kv in worst.items()))


def test_pretraining_gradients_are_the_sum_of_both_trunk_passes_on_gpu(golden):
    g = golden["pretraining"]
    model = C._build(_models(), golden, "pretraining").cuda()
    named = dict(model.named_parameters())
    own = {}
    for loss_name in g["losses"]:
        model.zero_grad(set_to_none=True)
        model(C._sample_list(golden, "pretraining", "cuda"))["losses"][loss_name].backward()
        own[loss_name] = {k: named[k].grad.clone() for k in g["by_loss"][loss_name]["grads"]}
        for k, ref in g["by_loss"][loss_name]["grads"].items():
            e = C.rel(own[loss_name][k].cpu(), ref)
            assert e < _grad_tol(k), (loss_name, k, e)
    model.zero_grad(set_to_none=True)
    sum(model(C._sample_list(golden, "pretraining", "cuda"))["losses"].values()).backward()
    for k in own["masked_lm_loss"]:
        parts = own["masked_lm_loss"][k] + own["itm_loss"][k]
        assert C.rel(named[k].grad, parts) < (1e-2 if k.startswith("image_embeddings.") else 1e-3), k


def _vqa_batch(B, T, size, labels, dev, seed):
    from mmf_b200.sample import SampleList
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(4, T + 1, (B,), generator=g)
    return SampleList(input_ids=torch.randint(1, 30522, (B, T), generator=g),
                      segment_ids=torch.zeros(B, T, dtype=torch.long),
                      input_mask=(torch.arange(T)[None] < lens[:, None]).long(),
                      image=torch.randn(B, 3, size, size, generator=g),
                      targets=(torch.rand(B, labels, generator=g) < 0.01).float(),
                      dataset_name="vqa2", dataset_type="train").to(dev)


def test_vit_b32_384_step_matches_the_fp32_trunk(golden):
    """bert-base text, ViT-B/32 at 384 px (40 + 145 positions), 3129 answers, B = 8: a training step with dropout is
    finite; in eval the encoder's output and the gradient of its input equal oracle.fusion_oracle's fp32 ViT trunk (the
    pre-LN layers and the final LayerNorm) on the same embeddings and mask"""
    MD = _models()
    from mmf_b200 import lib
    torch.manual_seed(0)
    cfg = MD.load_model_config("vilt", overrides=dict(golden["yamls"]["vqa2/vit_b32_384"], tasks="vqa2"))
    model = MD.build_model(cfg).cuda().train()
    sl = _vqa_batch(8, 40, 384, 3129, "cuda", 5)
    n0 = lib.launch_count()
    out = model(sl)
    loss = sum(out["losses"].values())
    loss.backward()
    torch.cuda.synchronize()
    assert lib.launch_count() > n0
    assert torch.isfinite(loss) and float(loss) > 0
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert len(grads) > 200 and all(torch.isfinite(gr).all() for gr in grads)

    model.eval().zero_grad(set_to_none=True)
    seen = {}

    def grab(mod, a, kw):
        seen["x"] = a[0].detach().clone()
        seen["mask"] = kw["attention_mask"].detach().clone()
    hook = model.encoder.register_forward_pre_hook(grab, with_kwargs=True)
    with torch.no_grad():
        model(sl)
    hook.remove()
    assert tuple(seen["x"].shape) == (8, 185, 768)
    x = seen["x"].clone().requires_grad_(True)
    seq, _ = model.encoder(x, attention_mask=seen["mask"])
    w = torch.randn(seq.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    (seq.float() * w).sum().backward()

    sd = {k[len("encoder.module."):]: v.detach().float() for k, v in model.state_dict().items()
          if k.startswith("encoder.module.")}
    enc_sd = {k[len("encoder."):]: v for k, v in sd.items() if k.startswith("encoder.")}
    xr = seen["x"].clone().requires_grad_(True)
    add = O.extended_attention_mask(seen["mask"])
    ref = O.layer_norm(O.vit_encoder(xr, add, enc_sd, "", 12, 12), sd, "layernorm")
    (ref * w).sum().backward()
    e_out, e_dx = C.rel(seq, ref), C.rel(x.grad, xr.grad)
    print("\nvilt vit_b32_384 trunk vs fp32 oracle: out %.2e dx %.2e" % (e_out, e_dx))
    assert e_out < 1e-2 and e_dx < 2e-2


@contextlib.contextmanager
def _deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def test_graphed_vqa_step_is_the_eager_step_bit_for_bit(golden):
    """a VQA training step (dropout 0) captured by GraphedStep and replayed gives the eager step's loss and gradients,
    bit for bit with torch.use_deterministic_algorithms(True)"""
    MD = _models()
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.sample import SampleList
    model = C._build(MD, golden, "classification").cuda().train()
    i = golden["inputs"]
    batch = {"input_ids": i["ids"], "segment_ids": i["segment"], "input_mask": i["mask"], "image": i["image"],
             "targets": i["targets"]}
    batch = {k: v.cuda() for k, v in batch.items()}

    def loss_fn_of(m):
        def run(b):
            out = m(SampleList(dict(b), dataset_name="vqa2", dataset_type="train"))
            return sum(out["losses"].values()).sum()
        return run
    with _deterministic():
        twin = copy.deepcopy(model)          # the eager step runs on a copy: no autograd graph of `model` on another stream
        ref = loss_fn_of(twin)(batch)
        ref.backward()
        ref_grads = {n: p.grad.detach().clone() for n, p in twin.named_parameters() if p.grad is not None}
        step = GraphedStep(model, loss_fn_of(model), batch)
        for _ in range(2):
            loss = step(batch)
        torch.cuda.synchronize()
    assert torch.equal(loss.detach(), ref.detach()), (float(loss), float(ref))
    got = {n: p.grad for n, p in model.named_parameters() if p.grad is not None}
    assert got.keys() == ref_grads.keys() and len(got) > 20
    for n, gr in ref_grads.items():
        assert torch.equal(got[n], gr), n
