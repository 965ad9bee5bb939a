"""Guarded buffers for the kernel tests (a plain module, imported by the poison tests; not a conftest).

The element-wise comparisons with fp64 share one blind spot: the memory around each operand is finite, and a fresh
process mostly hands out zeros.  A kernel that over-reads a tail row and multiplies it by a masked zero, or that writes
one element past its output, then still passes.  The helpers here put every operand inside a larger allocation:

    view, base = embed(shape, dtype, rows_before=.., rows_after=.., slack_cols=.., fill=..)

`view` is an interior view of `base`; everything in `base` outside `view` holds `fill`.  For inputs that is the poison
(a quiet NaN for floats, so an over-read that is multiplied by zero still gives NaN; `inf` where a kernel squares its
input; valid but wrong indices for index tensors, so an over-read gives a wrong value and never a wild address; all ones
for keep-bit words).  For outputs `fill` is left at None, which writes SENTINEL: a quiet NaN with a distinctive payload
for floats and a fixed word for integers.  `untouched(base, *views)` then checks the bits of every element outside the
views and names the first one that changed.

Layout rules are those of the TMA loads and 16-byte vector accesses: `base` starts 16-byte aligned (torch's caching
allocator aligns to 512 bytes), the row pitch of a 2-D view is a multiple of 8 elements and of 16 bytes, and every guard
region lies inside the same allocation as its view, so nothing a correct kernel does with these buffers can fault.

`poison_cache(value, nbytes)` fills torch's caching allocator with `value` and frees it again, so that later
`torch.empty` calls return memory that holds `value` instead of whatever a fresh process happened to have.
"""
import math

import torch

# sentinel bit patterns of the output guards, by element size (floats: quiet NaNs with a payload no kernel produces)
SENTINEL_BITS = {torch.bfloat16: 0x7FE5, torch.float16: 0x7EA5, torch.float32: 0x7FC5A5A5,
                 torch.float64: 0x7FF8A5A5A5A5A5A5, torch.int32: 0x5EED5EED, torch.int64: 0x5EED5EED5EED5EED,
                 torch.int16: 0x5EED, torch.uint8: 0xA5}
_INT_OF = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
NAN = float("nan")


def _ints(t):
    """the bits of t as a same-shaped integer tensor"""
    return t.view(_INT_OF[t.element_size()]) if t.dtype != _INT_OF[t.element_size()] else t


def _signed(bits, nbytes):
    """an unsigned bit pattern as the signed integer of that width"""
    return bits - (1 << (8 * nbytes)) if nbytes > 1 and bits >= 1 << (8 * nbytes - 1) else bits


def fill_bits(dtype, fill=None):
    """the integer bit pattern `untouched` expects outside the views: SENTINEL_BITS[dtype] for fill=None, else the bits
    of `fill` stored as `dtype`"""
    nbytes = torch.empty((), dtype=dtype).element_size()
    if fill is None:
        return _signed(SENTINEL_BITS[dtype], nbytes)
    return int(_ints(torch.full((1,), fill, dtype=dtype))[0])


def _fill(base, fill):
    _ints(base).fill_(fill_bits(base.dtype, fill))


def pitch_of(cols, slack_cols, dtype):
    """row pitch in elements: at least cols + slack_cols, a multiple of 8 elements and of 16 bytes"""
    esz = torch.empty((), dtype=dtype).element_size()
    q = max(8, 16 // esz)
    return -(-(cols + slack_cols) // q) * q


def embed(shape, dtype, *, rows_before=0, rows_after=0, slack_cols=0, fill=None, device="cuda"):
    """(view, base): a `shape` view inside one larger allocation whose other elements hold `fill` (SENTINEL for None).

    2-D shapes [rows, cols]: base is [rows_before + rows + rows_after, pitch] with pitch = pitch_of(cols, slack_cols),
    and view = base[rows_before:rows_before + rows, :cols] (row stride `pitch`).
    1-D and >2-D shapes are contiguous views: rows_before / rows_after count guard ELEMENTS before and after the view
    (the leading count rounded up to 16 bytes); slack_cols must be 0."""
    shape = tuple(int(s) for s in shape)
    esz = torch.empty((), dtype=dtype).element_size()
    if len(shape) == 2:
        rows, cols = shape
        pitch = pitch_of(cols, slack_cols, dtype)
        base = torch.empty(rows_before + rows + rows_after, pitch, dtype=dtype, device=device)
        _fill(base, fill)
        view = base[rows_before:rows_before + rows, :cols]
    else:
        if slack_cols:
            raise ValueError("embed: slack_cols needs a 2-D shape")
        n = math.prod(shape)
        q = max(1, 16 // esz)
        lead = -(-rows_before // q) * q
        base = torch.empty(lead + n + rows_after, dtype=dtype, device=device)
        _fill(base, fill)
        view = base[lead:lead + n].view(shape)
    assert view.data_ptr() % 16 == 0 or view.numel() == 0
    return view, base


def place(t, **kw):
    """embed(t.shape, t.dtype, **kw) with t's values copied into the view; returns (view, base)"""
    view, base = embed(t.shape, t.dtype, device=t.device, **kw)
    view.copy_(t)
    return view, base


def _region(base, flat):
    """names the guard region of base's flat element index"""
    if base.dim() == 2:
        r, c = divmod(flat, base.shape[1])
        return "row %d, column %d of the [%d, %d] allocation" % (r, c, base.shape[0], base.shape[1])
    return "element %d of the %d-element allocation" % (flat, base.numel())


def inside_mask(base, *views):
    """bool [base.numel()]: the elements of base that belong to one of the views"""
    inside = torch.zeros(base.numel(), dtype=torch.bool, device=base.device)
    idx = torch.arange(base.numel(), device=base.device)
    off0 = base.storage_offset()
    for v in views:
        assert v.untyped_storage().data_ptr() == base.untyped_storage().data_ptr(), "view is not inside base"
        if v.numel():
            inside[torch.as_strided(idx, v.size(), v.stride(), v.storage_offset() - off0).reshape(-1)] = True
    return inside


def untouched(base, *views, fill=None, what="guard"):
    """Fails unless every element of base outside the views still holds fill_bits(base.dtype, fill), bit for bit.  The
    message names the first changed element (its row and column in the allocation), as kernel_check.assert_within
    names the worst one, and how many changed."""
    expect = fill_bits(base.dtype, fill)
    bits = _ints(base).reshape(-1)
    bad = (bits != expect) & ~inside_mask(base, *views)
    if not bool(bad.any()):
        return
    first = int(torch.nonzero(bad)[0].item())
    mask = (1 << (8 * base.element_size())) - 1
    raise AssertionError("%s: %d element(s) outside the view changed; first at %s: 0x%x, expected 0x%x" % (
        what, int(bad.sum().item()), _region(base, first), int(bits[first].item()) & mask, expect & mask))


def assert_finite(t, what="view"):
    """no NaN or inf inside a float view (an over-read of poison shows up here)"""
    t = t.detach()
    if t.dtype.is_floating_point and t.numel():
        bad = ~torch.isfinite(t.float())
        if bool(bad.any()):
            idx = tuple(int(i) for i in torch.nonzero(bad)[0])
            raise AssertionError("%s: %d non-finite element(s); first at %s = %r" % (
                what, int(bad.sum().item()), idx, t[idx].item()))


# ------------------------------------------------------------------------------------------------------------------
# caching-allocator poison
# ------------------------------------------------------------------------------------------------------------------
CACHE_CAP = 4 << 30          # the GPUs are shared: never hold more than this much poison
SMALL_CAP = 96 << 20         # ... and at most this much of it in the small pool (blocks up to 1 MiB)


def poison_cache(value, nbytes):
    """Leaves `value` in the free blocks of torch's caching allocator: empties the cache, allocates blocks of both pools
    (in the small pool every size class from 512 B to 1 MiB, min(nbytes / 8, SMALL_CAP) bytes in all, so at least 2 MiB
    per class; then 2 MiB and up to min(nbytes, CACHE_CAP) in the large one), fills them with
    `value` as bf16 (a bf16 NaN pair is also an fp32 NaN, and -3e38 stays about -3e38 either way) and frees them.  A
    later torch.empty on the same stream then lands on `value` rather than on a fresh process's zeros.  Note that
    under torch.use_deterministic_algorithms torch itself fills torch.empty with NaN unless
    torch.utils.deterministic.fill_uninitialized_memory is off."""
    nbytes = min(int(nbytes), CACHE_CAP)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    held = []
    classes = [512 << i for i in range(12)]        # 512 B .. 1 MiB
    per_class = max(2 << 20, min(nbytes // 8, SMALL_CAP) // len(classes))
    for size in classes:                            # small pool: the same number of bytes in every size class
        for _ in range(per_class // size):
            held.append(torch.empty(size // 2, dtype=torch.bfloat16, device="cuda"))
    for t in held:
        t.fill_(value)
    total, size = 0, 2 << 20
    while total < nbytes:                           # large pool: doubling blocks up to the step's peak
        size = min(size, nbytes - total) if nbytes - total >= (2 << 20) else 2 << 20
        held.append(torch.full((size // 2,), value, dtype=torch.bfloat16, device="cuda"))
        total += size
        size = min(size * 2, 256 << 20)
    torch.cuda.synchronize()
    del held
