"""Training steps with dropout against fp64, fed the kernels' own keep bits: every layer type, dense and packed.

Every dropout site of the fused path draws its keep bits through engine.DropoutState.bits.  A fixture records each draw;
the decoder below turns it into a bool keep tensor of the reference's dense shape, from the layouts documented in
include/mmfb200.h (it never calls the product's packing helpers):
  dense attention            int32 [B, heads, Sq, ceil(Skv/32)]
  packed self-attention      int32 [heads, total, ceil(max_len/32)]      key j of the sample, query row cu[b] + i
  packed cross-attention     int32 [heads, total_q, ceil(max_kv/32)]
  hidden / embedding sites   int32 [rows, ceil(H/32)]                    rows = B*S dense, or the packed valid rows
with element j in bit j%32 of word j/32.  Positions a packed draw does not cover are padding and get keep = True: a padded
key carries -10000 in the additive mask, so its probability is exactly 0 in fp64, and a padded row has zero loss weight.

The oracle (oracle/fusion_oracle.py) then runs on the bf16-rounded weights and inputs with those masks, in fp64 (the
truth) and in bf16 (the drift bar).  The bar is that of test_depth_gpu.py: relative L2
err(product vs fp64) <= 1.5 * err(bf16 reference vs fp64) + 2e-3, with a ceiling of 2.5e-2 on the outputs, for the outputs
at valid rows, every input gradient and every parameter gradient (key biases: analytically zero, only bounded to be tiny),
and again per sample on each sample's output and input-gradient rows.  A discrimination guard recomputes the fp64
reference with one site's masks misrouted and requires the product to miss it by at least 5x the bar."""
import math
import types

import pytest
import torch

from oracle import fusion_oracle as O

pytestmark = pytest.mark.gpu

P = 0.1                 # hidden_dropout_prob = attention_probs_dropout_prob of every MMF training config
HEADS = 12              # BERT-base attention heads at 768 wide


# ----------------------------------------------------------------------------------------------------------------------
# recorder and layout decoder
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def draws(monkeypatch):
    """every keep-bit draw of the forward, in order: (rows_shape, ncols, p, words)"""
    from mmf_b200 import engine as E
    rec = []
    orig = E.DropoutState.bits

    def spy(self, rows_shape, ncols, p, device):
        out = orig(self, rows_shape, ncols, p, device)
        rec.append((tuple(int(r) for r in rows_shape), int(ncols), float(p), out.clone()))
        return out
    monkeypatch.setattr(E.DropoutState, "bits", spy)
    return rec


def nwords(n):
    return (n + 31) // 32


def unpack_bits(words, n):
    """int32 words [..., W] -> bool [..., n]: element j is bit j % 32 of word j // 32"""
    w = words.to(torch.int64) & 0xFFFFFFFF
    j = torch.arange(n, device=words.device)
    return ((w[..., j // 32] >> (j % 32)) & 1).bool()


def attn_site(heads, q_valid, kv_valid):
    return ("attn", heads, q_valid, kv_valid)


def hid_site(valid, H):
    return ("hid", valid, H)


def decode(draw, site, packed):
    """the keep mask of one draw in the reference's dense shape: [B, heads, Sq, Skv] or [B, S, H]"""
    shape, ncols, p, words = draw
    assert p == P, (p, site[0])
    if site[0] == "attn":
        _, heads, qv, kv = site
        B, Sq, Skv = qv.shape[0], qv.shape[1], kv.shape[1]
        if not packed:
            assert shape == (B, heads, Sq) and ncols == Skv and tuple(words.shape) == (B, heads, Sq, nwords(Skv)), shape
            return unpack_bits(words, Skv)
        lq, lk = qv.sum(1).tolist(), kv.sum(1).tolist()
        total, max_kv = sum(lq), max(lk)
        assert shape == (heads, total) and tuple(words.shape) == (heads, total, nwords(max_kv)), (shape, words.shape)
        assert ncols == max_kv, (ncols, max_kv)
        bits = unpack_bits(words, max_kv)
        keep = torch.ones(B, heads, Sq, Skv, dtype=torch.bool, device=words.device)
        row = 0
        for b in range(B):
            qp, kp = qv[b].nonzero().squeeze(1), kv[b].nonzero().squeeze(1)
            keep[b][:, qp[:, None], kp[None, :]] = bits[:, row:row + lq[b], :lk[b]]
            row += lq[b]
        return keep
    _, valid, H = site
    B, S = valid.shape
    rows = valid.reshape(-1).nonzero().squeeze(1) if packed else torch.arange(B * S, device=words.device)
    assert shape == (rows.numel(),) and ncols == H and tuple(words.shape) == (rows.numel(), nwords(H)), (shape, H)
    keep = torch.ones(B * S, H, dtype=torch.bool, device=words.device)
    keep[rows] = unpack_bits(words, H)
    return keep.view(B, S, H)


def decode_all(draws, sites, packed):
    """decoded masks of a whole forward, after the per-site statistics: the draw count, each site's kept fraction within
    5 sigma of 1 - p, and no two sites of the same shape with identical words (overlapping Philox counters)"""
    assert len(draws) == len(sites), "%d draws, the layer structure implies %d" % (len(draws), len(sites))
    fracs = []
    for (_, ncols, _, words), site in zip(draws, sites):
        bits = unpack_bits(words, ncols)
        n = bits.numel()
        frac = bits.float().mean().item()
        fracs.append(frac)
        assert abs(frac - (1 - P)) < 5 * math.sqrt(P * (1 - P) / n), (site[0], frac, n)
    for i in range(len(draws)):
        for j in range(i):
            a, b = draws[i][3], draws[j][3]
            assert a.shape != b.shape or not torch.equal(a, b), "sites %d and %d drew identical words" % (j, i)
    print("  %d draws, keep fractions: %s" % (len(draws), " ".join("%.4f" % f for f in fracs)))
    return [decode(d, s, packed) for d, s in zip(draws, sites)]


def bert_sites(heads, valid, H):
    return [attn_site(heads, valid, valid), hid_site(valid, H), hid_site(valid, H)]


def bert_masks(m):
    return {"attn": m[0], "self_out": m[1], "out": m[2]}


# ----------------------------------------------------------------------------------------------------------------------
# reference runs and the comparison
# ----------------------------------------------------------------------------------------------------------------------
def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def reference(fn, sd, inputs, ws, dtype):
    """fn(inputs, sd) -> outputs, run on the bf16-rounded weights / inputs in `dtype`; loss = sum(out * w).
    -> (outputs, input gradients, parameter gradients), all fp64"""
    sdc = {k: v.detach().to(torch.bfloat16).to(dtype).requires_grad_(True) for k, v in sd.items()}
    xs = [x.detach().to(torch.bfloat16).to(dtype).requires_grad_(True) for x in inputs]
    outs = fn(xs, sdc)
    sum((o.double() * w.double()).sum() for o, w in zip(outs, ws)).backward()
    return ([o.detach().double() for o in outs], [x.grad.double() for x in xs],
            {k: v.grad.double() for k, v in sdc.items() if v.grad is not None})


def _key_bias(n):
    return ".key.bias" in n or ".key1.bias" in n or ".key2.bias" in n


def _bar(drift):
    return 1.5 * drift + 2e-3


def check(name, prod, fn, sd, inputs, ws, valid, masks, wrong_masks):
    """prod: (outputs, input gradients, named parameters) of the product; valid: bool [B, S] per output.
    Compares against the fp64 reference, bounded by the bf16 reference's drift; then the discrimination guard."""
    p_out, p_dx, named = prod
    f = reference(lambda xs, s: fn(xs, s, masks), sd, inputs, ws, torch.float64)
    b = reference(lambda xs, s: fn(xs, s, masks), sd, inputs, ws, torch.bfloat16)
    quantities = {}                                   # name -> (product, fp64, bf16)
    for k, (po, fo, bo) in enumerate(zip(p_out, f[0], b[0])):
        quantities["out%d" % k] = (po[valid[k]], fo[valid[k]], bo[valid[k]])
    for k, (pd, fd, bd) in enumerate(zip(p_dx, f[1], b[1])):
        quantities["dx%d" % k] = (pd, fd, bd)
    for n, p in named.items():
        if n not in f[2]:                             # a parameter the reference never reads (ViLBERT's q_dense*)
            assert p.grad is None or not p.grad.any(), n
            continue
        if _key_bias(n):   # analytically zero gradient (softmax shift invariance): only required to be tiny
            qn = n.replace("key", "query")
            assert p.grad.float().norm() <= 0.05 * named[qn].grad.float().norm() + 1e-3, n
            continue
        quantities[n] = (p.grad, f[2][n], b[2][n])
    errs = {q: (rel(pv, fv), rel(bv, fv)) for q, (pv, fv, bv) in quantities.items()}
    outs = [q for q in errs if q.startswith("out")]
    dxs = [q for q in errs if q.startswith("dx")]
    params = [q for q in errs if q not in outs and q not in dxs]
    worst_p = max(params, key=lambda q: errs[q][0] / _bar(errs[q][1]))
    print("  product / bf16 reference vs fp64: %s | worst parameter gradient %s %.2e / %.2e" % (
        " ".join("%s=%.2e/%.2e" % (q, *errs[q]) for q in outs + dxs), worst_p, *errs[worst_p]))
    bad = [(q, e, d) for q, (e, d) in errs.items() if e > _bar(d)]
    bad += [(q, e, 2.5e-2) for q in outs if errs[q][0] > 2.5e-2]
    assert not bad, bad[:8]
    # per sample: a bug that touches one sample must not be averaged away
    worst_s = (0.0, "")
    for k in range(len(p_out)):
        for s in range(valid[k].shape[0]):
            rows = valid[k][s]
            if rows.any():
                e, d = rel(p_out[k][s][rows], f[0][k][s][rows]), rel(b[0][k][s][rows], f[0][k][s][rows])
                assert e <= _bar(d), ("out%d sample %d" % (k, s), e, d)
                worst_s = max(worst_s, (e / _bar(d), "out%d[%d]" % (k, s)))
    for k in range(len(p_dx)):
        for s in range(p_dx[k].shape[0]):
            if not f[1][k][s].any():                  # a sample with no valid row: its input gradient is exactly zero
                assert not p_dx[k][s].any(), ("dx%d sample %d" % (k, s))
                continue
            e, d = rel(p_dx[k][s], f[1][k][s]), rel(b[1][k][s], f[1][k][s])
            assert e <= _bar(d), ("dx%d sample %d" % (k, s), e, d)
            worst_s = max(worst_s, (e / _bar(d), "dx%d[%d]" % (k, s)))
    # discrimination guard: the same comparison against a reference given one misrouted site must fail by far
    w = reference(lambda xs, s: fn(xs, s, wrong_masks), sd, inputs, ws, torch.float64)
    wrong = {"out%d" % k: (po[valid[k]], wo[valid[k]]) for k, (po, wo) in enumerate(zip(p_out, w[0]))}
    wrong.update({"dx%d" % k: (pd, wd) for k, (pd, wd) in enumerate(zip(p_dx, w[1]))})
    wrong.update({n: (quantities[n][0], w[2][n]) for n in params})
    margin = max((rel(pv, wv) / _bar(errs[q][1]), q) for q, (pv, wv) in wrong.items())
    print("  %s: worst per-sample ratio %.2f (%s); guard margin %.1fx the bar (%s)" % (name, *worst_s, *margin))
    assert margin[0] >= 5.0, margin


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
def bert_cfg(layers, hidden=768, heads=12, inter=3072):
    return types.SimpleNamespace(hidden_size=hidden, num_attention_heads=heads, intermediate_size=inter,
                                 num_hidden_layers=layers, hidden_dropout_prob=P, attention_probs_dropout_prob=P,
                                 layer_norm_eps=1e-12, hidden_act="gelu", initializer_range=0.02)


def _perturb_1d(module):
    with torch.no_grad():
        for p in module.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.02)


def _additive(valid):
    return torch.where(valid, 0.0, -10000.0).float()[:, None, None, :]


def _lens_valid(lens, S):
    return torch.arange(S, device="cuda")[None] < torch.tensor(lens, device="cuda")[:, None]


def _swap01(m, a=0, b=1):
    m = m.clone()
    m[[a, b]] = m[[b, a]]
    return m


def _roll_row(m):
    """a [B, S, H] hidden mask shifted by one row"""
    return m.reshape(-1, m.shape[-1]).roll(1, 0).view_as(m)


def _bert_encoder_run(enc, x, add, valid, w, draws, packed, guard, name, L):
    xg = x.clone().requires_grad_(True)
    out = enc(xg, add)[0]
    (out * w).sum().backward()
    torch.cuda.synchronize()
    H = x.shape[-1]
    m = decode_all(draws, bert_sites(HEADS, valid, H) * L, packed)
    masks = [bert_masks(m[3 * i:3 * i + 3]) for i in range(L)]
    sd = enc.state_dict()

    def fn(xs, s, mk):
        return [O.bert_encoder(xs[0], add.to(xs[0].dtype), s, "", L, HEADS, mk, P, P)]
    check(name, ([out], [xg.grad], dict(enc.named_parameters())), fn, sd, [x], [w], [valid], masks, guard(masks))


def _bert_encoder(L, packed=False):
    from mmf_b200.modules import B200BertEncoder
    enc = B200BertEncoder(bert_cfg(L)).cuda().train()
    _perturb_1d(enc)
    enc._runner.skip_padding = packed
    return enc


def test_bert_post_ln_dense(draws):
    """2 layers at 768 / 12 heads, B = 4, S = 228, ragged key padding (lengths 64, 228, 1, 33)"""
    torch.manual_seed(101)
    enc = _bert_encoder(2)
    B, S, H = 4, 228, 768
    valid = _lens_valid([64, 228, 1, 33], S)
    x = torch.randn(B, S, H, device="cuda")
    w = torch.randn(B, S, H, device="cuda") * valid[..., None]

    def guard(masks):           # layer 0's attention keep bits of samples 0 and 1 swapped
        return [dict(masks[0], attn=_swap01(masks[0]["attn"]))] + masks[1:]
    _bert_encoder_run(enc, x, _additive(valid), valid, w, draws, False, guard, "BERT dense", 2)


def test_bert_post_ln_packed(draws):
    """skip_padding: [text | pad | regions | pad] rows, sample lengths 0, 1, 31, 32, 33, 90 (the longest, not first), 65,
    33; max_len = 90 is not a multiple of 32"""
    torch.manual_seed(102)
    enc = _bert_encoder(2, packed=True)
    T, R, H = 40, 60, 768
    lt = [0, 1, 20, 16, 33, 40, 25, 3]
    nr = [0, 0, 11, 16, 0, 50, 40, 30]
    B, S = len(lt), T + R
    valid = torch.cat([_lens_valid(lt, T), _lens_valid(nr, R)], 1)
    x = torch.randn(B, S, H, device="cuda")
    w = torch.randn(B, S, H, device="cuda") * valid[..., None]

    def guard(masks):           # layer 1's self-output mask shifted by one row
        return masks[:1] + [dict(masks[1], self_out=_roll_row(masks[1]["self_out"]))]
    _bert_encoder_run(enc, x, _additive(valid), valid, w, draws, True, guard, "BERT packed", 2)


def _causal_mask(enc_valid, T):
    """the [B, 1, S, S] additive prefix-LM mask of mmf/models/m4c.py:427-437 (as test_attention_causal_gpu restates it)"""
    B, Pn = enc_valid.shape
    S = Pn + T
    am = torch.cat([enc_valid.float(), torch.zeros(B, T, device=enc_valid.device)], dim=1)
    ext = am[:, None, None, :].repeat(1, 1, S, 1)
    ext[:, :, -T:, -T:] = torch.tril(torch.ones(T, T, device=enc_valid.device))
    return (1.0 - ext) * -10000.0


@pytest.mark.parametrize("T", [12, 30])
def test_bert_causal_tail(draws, T):
    """M4C's path: run_bert_encoder(causal_len=T) on 2 layers at 768, S = 182; random prefix padding, sample 1's prefix
    entirely padding"""
    from mmf_b200 import modules
    torch.manual_seed(103 + T)
    enc = _bert_encoder(2)
    B, S, H = 4, 182, 768
    Pn = S - T
    enc_valid = _lens_valid([Pn, 0, 57, 121], Pn)
    valid = torch.cat([enc_valid, torch.ones(B, T, dtype=torch.bool, device="cuda")], 1)
    x = torch.randn(B, S, H, device="cuda")
    w = torch.randn(B, S, H, device="cuda") * valid[..., None]
    xg = x.clone().requires_grad_(True)
    out = modules.run_bert_encoder(enc._runner, xg, _additive(valid), True, causal_len=T)[0]
    (out * w).sum().backward()
    torch.cuda.synchronize()
    all_rows = torch.ones(B, S, dtype=torch.bool, device="cuda")
    m = decode_all(draws, bert_sites(HEADS, all_rows, H) * 2, False)
    masks = [bert_masks(m[3 * i:3 * i + 3]) for i in range(2)]
    add = _causal_mask(enc_valid, T)

    def fn(xs, s, mk):
        return [O.bert_encoder(xs[0], add.to(xs[0].dtype), s, "", 2, HEADS, mk, P, P)]
    guard = [dict(masks[0], attn=_swap01(masks[0]["attn"]))] + masks[1:]
    check("causal T=%d" % T, ([out], [xg.grad], dict(enc.named_parameters())), fn, enc.state_dict(), [x], [w], [valid],
          masks, guard)


def test_vit_pre_ln(draws):
    """B200ViTEncoder: 2 layers at 768 / 12 heads, S = 197; dropout_apply and add_bf16 in vit_layer_bwd"""
    from mmf_b200.vit import B200ViTEncoder
    torch.manual_seed(104)
    enc = B200ViTEncoder(bert_cfg(2)).cuda().train()
    _perturb_1d(enc)
    B, S, H = 4, 197, 768
    valid = _lens_valid([197, 150, 197, 97], S)
    add = _additive(valid)
    x = torch.randn(B, S, H, device="cuda")
    w = torch.randn(B, S, H, device="cuda") * valid[..., None]
    xg = x.clone().requires_grad_(True)
    out = enc(xg, attention_mask=add).last_hidden_state
    (out * w).sum().backward()
    torch.cuda.synchronize()
    m = decode_all(draws, bert_sites(HEADS, valid, H) * 2, False)
    masks = [bert_masks(m[3 * i:3 * i + 3]) for i in range(2)]

    def fn(xs, s, mk):
        return [O.vit_encoder(xs[0], add.to(xs[0].dtype), s, "", 2, HEADS, mk, P, P)]
    guard = [dict(masks[0], out=_roll_row(masks[0]["out"]))] + masks[1:]     # ViTOutput's mask misplaced
    check("ViT", ([out], [xg.grad], dict(enc.named_parameters())), fn, enc.state_dict(), [x], [w], [valid], masks, guard)


# two-stream lengths: crossing 32-key words, sample 0 empty in both streams, no sample empty in one stream only
TXT_LENS = [0, 33, 36, 5, 31, 32]
IMG_LENS = [0, 40, 12, 33, 1, 36]


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
def test_vilbert_two_stream(draws, packed):
    """text 768 / 12 heads, image 1024 / 8 heads, co-attention 1024 / 8 heads; schedule: text layer, image layer,
    connection layer"""
    from mmf_b200.modules import B200ViLBertEncoder
    torch.manual_seed(105)
    c = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=1, v_hidden_size=1024,
             v_num_attention_heads=8, v_intermediate_size=1024, v_num_hidden_layers=1, bi_hidden_size=1024,
             bi_num_attention_heads=8, v_biattention_id=[1], t_biattention_id=[1])
    cfg = types.SimpleNamespace(hidden_dropout_prob=P, v_hidden_dropout_prob=P, attention_probs_dropout_prob=P,
                                v_attention_probs_dropout_prob=P, layer_norm_eps=1e-12, initializer_range=0.02,
                                skip_padding=packed, **c)
    enc = B200ViLBertEncoder(cfg).cuda().train()
    _perturb_1d(enc)
    B, T, R = len(TXT_LENS), 36, 40
    tv, iv = _lens_valid(TXT_LENS, T), _lens_valid(IMG_LENS, R)
    tadd, iadd = _additive(tv), _additive(iv)
    txt = torch.randn(B, T, 768, device="cuda")
    img = torch.randn(B, R, 1024, device="cuda")
    wt = torch.randn(B, T, 768, device="cuda") * tv[..., None]
    wi = torch.randn(B, R, 1024, device="cuda") * iv[..., None]
    tg, ig = txt.clone().requires_grad_(True), img.clone().requires_grad_(True)
    tl, vl, _ = enc(tg, ig, tadd, tadd, iadd, None, output_all_encoded_layers=False)
    ((tl[-1] * wt).sum() + (vl[-1] * wi).sum()).backward()
    torch.cuda.synchronize()
    assert O.vilbert_schedule([1], [1], 1, 1) == [("t", 0), ("v", 0), ("c", 0)]
    sites = (bert_sites(12, tv, 768) + bert_sites(8, iv, 1024) +
             [attn_site(8, tv, iv), attn_site(8, iv, tv), hid_site(iv, 1024), hid_site(tv, 768), hid_site(iv, 1024),
              hid_site(tv, 768)])
    m = decode_all(draws, sites, packed)
    conn = dict(zip(("attn1", "attn2", "bo1", "bo2", "v_out", "t_out"), m[6:]))
    masks = [bert_masks(m[0:3]), bert_masks(m[3:6]), conn]

    def fn(xs, s, mk):
        return list(O.vilbert_encoder(xs[0], xs[1], tadd.to(xs[0].dtype), iadd.to(xs[0].dtype), s, "", c, mk, P, P, P, P))
    guard = masks[:2] + [dict(conn, attn1=_swap01(conn["attn1"], 1, 2))]
    check("ViLBERT %s" % ("packed" if packed else "dense"), ([tl[-1], vl[-1]], [tg.grad, ig.grad],
          dict(enc.named_parameters())), fn, enc.state_dict(), [txt, img], [wt, wi], [tv, iv], masks, guard)


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
def test_lxmert_two_stream(draws, packed):
    """l_layers = r_layers = x_layers = 1 at 768 / 12 heads.  The visual feature encoder's own nn.Dropout draws from torch's
    generator, not from the fused path's keep bits, so it is set to p = 0 here; every other site runs at p = 0.1."""
    from mmf_b200.lxmert import B200LXMERTEncoder
    torch.manual_seed(106)
    cfg = types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, hidden_dropout_prob=P,
                                attention_probs_dropout_prob=P, visual_feat_dim=512, visual_pos_dim=4, l_layers=1,
                                x_layers=1, r_layers=1, initializer_range=0.02, skip_padding=packed)
    enc = B200LXMERTEncoder(cfg).cuda().train()
    enc.visn_fc.dropout.p = 0.0
    _perturb_1d(enc)
    B, T, R = len(TXT_LENS), 36, 40
    lv, vv = _lens_valid(TXT_LENS, T), _lens_valid(IMG_LENS, R)
    ladd, vadd = _additive(lv), _additive(vv)
    lang = torch.randn(B, T, 768, device="cuda")
    feats = torch.randn(B, R, 512, device="cuda")
    boxes = torch.rand(B, R, 4, device="cuda")
    wl = torch.randn(B, T, 768, device="cuda") * lv[..., None]
    wv = torch.randn(B, R, 768, device="cuda") * vv[..., None]
    lg, fg, bg = (t.clone().requires_grad_(True) for t in (lang, feats, boxes))
    lo, vo = enc(lg, ladd, (fg, bg), vadd)
    ((lo * wl).sum() + (vo * wv).sum()).backward()
    torch.cuda.synchronize()
    sites = (bert_sites(12, lv, 768) + bert_sites(12, vv, 768) +
             [attn_site(12, lv, vv), attn_site(12, vv, lv), hid_site(lv, 768), hid_site(vv, 768)] +
             bert_sites(12, lv, 768) + bert_sites(12, vv, 768))
    m = decode_all(draws, sites, packed)
    x = dict(zip(("x_attn_lang", "x_attn_visn", "x_out_lang", "x_out_visn"), m[6:10]),
             lang=bert_masks(m[10:13]), visn=bert_masks(m[13:16]))
    masks = {"l": [bert_masks(m[0:3])], "r": [bert_masks(m[3:6])], "x": [x]}

    def fn(xs, s, mk):
        dt = xs[0].dtype
        return list(O.lxmert_encoder(xs[0], ladd.to(dt), xs[1], xs[2], vadd.to(dt), s, "", 1, 1, 1, 12, mk, P, P))
    guard = dict(masks, x=[dict(x, x_attn_lang=_swap01(x["x_attn_lang"], 1, 2))])
    check("LXMERT %s" % ("packed" if packed else "dense"), ([lo, vo], [lg.grad, fg.grad, bg.grad],
          dict(enc.named_parameters())), fn, enc.state_dict(), [lang, feats, boxes], [wl, wv], [lv, vv], masks, guard)


@pytest.mark.parametrize("kind", ["visio_linguistic", "image_feature"])
def test_embeddings(draws, kind):
    """B200VisioLinguisticEmbeddings (LayerNorm forward with the keep bits, torch multiply in its backward) and ViLBERT's
    B200ImageFeatureEmbeddings (ops.compose_ln), including the table and projection gradients"""
    torch.manual_seed(107)
    B = 4
    if kind == "visio_linguistic":
        from mmf_b200.embeddings import B200VisioLinguisticEmbeddings
        cfg = types.SimpleNamespace(hidden_size=768, vocab_size=1000, max_position_embeddings=64, type_vocab_size=2,
                                    visual_embedding_dim=1024, hidden_dropout_prob=P, layer_norm_eps=1e-12,
                                    initializer_range=0.02)
        emb = B200VisioLinguisticEmbeddings(cfg).cuda().train()
        T, R, H = 20, 30, 768
        ids = torch.randint(0, 1000, (B, T), device="cuda")
        ids[:, -3:] = 0                                               # [PAD] rows: read, no gradient
        seg = torch.randint(0, 2, (B, T), device="cuda")
        vtype = torch.randint(0, 2, (B, R), device="cuda")
        inputs = [torch.randn(B, R, 1024, device="cuda")]

        def prod(xs):
            return emb(ids, seg, xs[0], vtype)

        def fn(xs, s, mk):
            return [O.visio_linguistic_embeddings(ids, seg, xs[0], vtype, s, "emb", keep=mk, p=P)]
    else:
        from mmf_b200.vilbert import B200ImageFeatureEmbeddings
        cfg = types.SimpleNamespace(v_feature_size=2048, v_hidden_size=1024, hidden_dropout_prob=P)
        emb = B200ImageFeatureEmbeddings(cfg).cuda().train()
        T, R, H = 0, 36, 1024
        inputs = [torch.randn(B, R, 2048, device="cuda"), torch.rand(B, R, 5, device="cuda")]

        def prod(xs):
            return emb(xs[0], xs[1])

        def fn(xs, s, mk):
            return [O.image_feature_embeddings(xs[0], xs[1], s, "emb", keep=mk, p=P)]
    _perturb_1d(emb)
    S = T + R
    valid = torch.ones(B, S, dtype=torch.bool, device="cuda")
    w = torch.randn(B, S, H, device="cuda")
    xs = [t.clone().requires_grad_(True) for t in inputs]
    out = prod(xs)
    (out.float() * w).sum().backward()
    torch.cuda.synchronize()
    (keep,) = decode_all(draws, [hid_site(valid, H)], False)
    sd = {"emb." + k: v for k, v in emb.state_dict().items()}
    named = {"emb." + k: v for k, v in emb.named_parameters()}
    check("embeddings " + kind, ([out], [x.grad for x in xs], named), fn, sd, inputs, [w], [valid], keep, _roll_row(keep))
