"""TEST HELPER - never imported by the product.  A CPU restatement of the packing plan of mmfb_plan_packing
(include/mmfb200.h), sample by sample in plain Python, so that the CPU tests can set it against the host plans of the
encoders and the GPU tests can set the kernel against it."""
import torch


def kept_positions(masks, B, lens, causal_len=0):
    """per stream (None for a stream without a mask) a bool [B, S] of the positions the plan keeps"""
    valid = []
    for m, S in zip(masks, lens):
        if m is None:
            valid.append(torch.ones(B, S, dtype=torch.bool))
            continue
        v = m.detach().cpu() == 0
        if causal_len:
            v[:, S - causal_len:] = True
        valid.append(v)
    kept = [v.clone() for v in valid]
    if len(masks) == 2:
        for b in range(B):
            has = [bool(v[b].any()) for v in valid]
            for k in range(2):
                if not has[k] and has[1 - k]:          # one-sided: the empty stream keeps every position
                    kept[k][b] = True
    return [None if m is None else k for m, k in zip(masks, kept)]


def plan(masks, B, lens, causal_len=0):
    """per stream (None without a mask): (cu int32 [B+1], pack_map int32 [B*S], unpack_map int32 [B*S])"""
    out = []
    for kept, S in zip(kept_positions(masks, B, lens, causal_len), lens):
        if kept is None:
            out.append(None)
            continue
        flat = kept.reshape(-1)
        n = int(flat.sum())
        cu = torch.zeros(B + 1, dtype=torch.int32)
        cu[1:] = torch.cumsum(kept.sum(1), 0).to(torch.int32)
        unpack_map = torch.full((B * S,), -1, dtype=torch.int32)
        unpack_map[flat] = torch.arange(n, dtype=torch.int32)
        pack_map = torch.full((B * S,), -1, dtype=torch.int32)
        pack_map[:n] = torch.nonzero(flat).reshape(-1).to(torch.int32)
        out.append((cu, pack_map, unpack_map))
    return out


def masks_of(valid, soft=None):
    """the additive mask of a bool [B, S] validity: 0 at valid positions, -10000 elsewhere (or `soft` values)"""
    m = (~valid).float() * -10000.0
    if soft is not None:
        m = torch.where(valid, m, torch.full_like(m, soft))
    return m


def random_valid(B, S, g, kinds=()):
    """a bool [B, S] with random prefix lengths; kinds: indices of samples to leave empty ("empty", b) or full ("full", b)"""
    lens = torch.randint(0, S + 1, (B,), generator=g)
    v = torch.arange(S)[None] < lens[:, None]
    v &= torch.rand(B, S, generator=g) < 0.9          # a few holes inside the prefixes too
    for kind, b in kinds:
        v[b] = kind == "full"
    return v
