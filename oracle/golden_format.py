"""TEST INFRASTRUCTURE - compact storage of the fixtures under tests/golden (written by oracle/make_golden.py).

A fixture is a plain torch.save of nested dicts; the large members are objects that pickle as a call of one of the
functions below, so torch.load(path, weights_only=False) hands back ordinary tensors and every file stays under 1 MB:
  * Q8: a tensor of values base + k / 1024 (|k| <= 127; make_golden draws fixture weights on that grid) as int8 - exact;
  * Sampled: a gradient as a fixed seeded sample of its elements plus its first row; loaded at full shape with NaN
    where nothing was stored - `kept` restricts a comparison to the stored elements;
  * Replay: a state_dict drawn by the former make_golden._perturb from a seed (normal 0.02, LayerNorm weights around 1),
    redrawn in key order; the entries the draw does not reproduce are stored as they are.
"""
import torch


def q8(q, base):
    return q.float() / 1024.0 + base


def sampled(shape, idx, values):
    t = torch.full(shape, float("nan"))
    t.view(-1)[idx.long()] = values
    return t


def replay(seed, order, kept):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for n, shape, dtype in order:
        if dtype.is_floating_point:
            lnw = "LayerNorm.weight" in n or n.endswith("layer_norms.0.weight") or n.endswith(".1.weight")
            v = (1.0 if (len(shape) < 2 and lnw) else 0.0) + torch.randn(shape, generator=g) * 0.02
            out[n] = kept.get(n, v)
        else:
            out[n] = kept[n]
    return out


class Q8:
    def __init__(self, q, base):
        self.q, self.base = q, base

    def __reduce__(self):
        return q8, (self.q, self.base)


class Sampled:
    def __init__(self, shape, idx, values):
        self.shape, self.idx, self.values = shape, idx, values

    def __reduce__(self):
        return sampled, (self.shape, self.idx, self.values)


class Replay:
    def __init__(self, seed, order, kept):
        self.seed, self.order, self.kept = seed, order, kept

    def __reduce__(self):
        return replay, (self.seed, self.order, self.kept)


def kept(a, b):
    """(a, b) restricted to the elements the golden b stores (all of them unless b is a sampled gradient)"""
    if torch.is_tensor(b) and b.is_floating_point():
        m = ~torch.isnan(b)
        if not bool(m.all()):
            return a.reshape(-1)[m.reshape(-1).to(a.device)], b.reshape(-1)[m.reshape(-1)]
    return a, b
