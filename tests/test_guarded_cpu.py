"""tests/guarded.py without a GPU: embed's strides and alignment, untouched catching one flipped bit in every guard
region, and the coverage rule that every compute entry point of include/mmfb200.h has a poison case in
tests/test_poison_guard_gpu.py (read with ast, so that nothing here loads the CUDA library)."""
import ast
import os
import re

import pytest
import torch

import guarded as G

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "mmfb200.h")
# queries that compute nothing on the device: sizes, the version and the error / diagnostic state
NOT_COMPUTE = {"mmfb_last_error", "mmfb_version", "mmfb_device_ok", "mmfb_launch_count"}

DTYPES = [torch.bfloat16, torch.float32, torch.int32, torch.int64, torch.uint8]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,cols,before,after,slack", [(5, 3, 2, 3, 0), (1, 8, 0, 1, 5), (7, 100, 1, 0, 29),
                                                          (3, 16, 4, 4, 0)])
def test_embed_strides_and_alignment(dtype, rows, cols, before, after, slack):
    view, base = G.embed((rows, cols), dtype, rows_before=before, rows_after=after, slack_cols=slack, device="cpu")
    esz = view.element_size()
    pitch = view.stride(0)
    assert tuple(view.shape) == (rows, cols) and view.stride(1) == 1
    assert pitch >= cols + slack and pitch % 8 == 0 and (pitch * esz) % 16 == 0
    assert tuple(base.shape) == (before + rows + after, pitch)
    assert (view.data_ptr() - base.data_ptr()) == before * pitch * esz
    assert view.data_ptr() % 16 == 0
    # every element outside the view holds the sentinel, and writing the view changes nothing else
    view.copy_(torch.ones(rows, cols).to(dtype))
    G.untouched(base, view)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape,before,after", [((13,), 3, 5), ((2, 3, 5), 1, 1), ((8,), 0, 1)])
def test_embed_contiguous_views(dtype, shape, before, after):
    view, base = G.embed(shape, dtype, rows_before=before, rows_after=after, device="cpu")
    assert view.is_contiguous() and tuple(view.shape) == shape and view.data_ptr() % 16 == 0
    lead = (view.data_ptr() - base.data_ptr()) // view.element_size()
    assert lead >= before and base.numel() == lead + view.numel() + after
    G.untouched(base, view)


def test_fills_are_the_poison_and_the_sentinel():
    v, b = G.embed((3, 5), torch.float32, rows_before=1, fill=G.NAN, device="cpu")
    assert torch.isnan(b[0]).all() and torch.isnan(b[1:, 5:]).all()
    v, b = G.embed((3, 5), torch.bfloat16, rows_after=1, device="cpu")
    assert torch.isnan(b.float()[3]).all() and int(b.view(torch.int16)[3, 0]) == 0x7FE5
    v, b = G.embed((4,), torch.float32, rows_after=2, fill=float("inf"), device="cpu")
    assert torch.isinf(b[-2:]).all()
    v, b = G.embed((2, 3), torch.int32, slack_cols=1, fill=7, device="cpu")
    assert (b[:, 3:] == 7).all()
    G.untouched(b, v, fill=7)


def _regions(base, view):
    """one flat index per guard region of a 2-D embed: first and last leading-row element, a slack column of every row,
    the first and last trailing-row element (the final element of the allocation)"""
    pitch = base.shape[1]
    r0 = (view.data_ptr() - base.data_ptr()) // view.element_size() // pitch
    rows, cols = view.shape
    out = {"leading row (first element)": 0, "leading row (last element)": r0 * pitch - 1}
    for r in range(rows):
        out["slack column of row %d" % r] = (r0 + r) * pitch + cols + (r % (pitch - cols))
    out["trailing row (first element)"] = (r0 + rows) * pitch
    out["final element"] = base.numel() - 1
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_untouched_catches_one_flipped_bit_in_every_region(dtype):
    view, base = G.embed((4, 13), dtype, rows_before=2, rows_after=2, slack_cols=6, device="cpu")
    for name, flat in _regions(base, view).items():
        for bit in (0, 8 * base.element_size() - 2):
            v, b = G.embed((4, 13), dtype, rows_before=2, rows_after=2, slack_cols=6, device="cpu")
            G.untouched(b, v)
            ints = b.view(G._INT_OF[b.element_size()]).reshape(-1)
            ints[flat] ^= 1 << bit
            with pytest.raises(AssertionError, match="outside the view changed"):
                G.untouched(b, v)
    # the flat (1-D) layout: the element before and the element after the view
    for flat_of in (lambda lead, n: lead - 1, lambda lead, n: lead + n, lambda lead, n: lead + n + 2):
        v, b = G.embed((9,), dtype, rows_before=3, rows_after=3, device="cpu")
        lead = (v.data_ptr() - b.data_ptr()) // v.element_size()
        b.view(G._INT_OF[b.element_size()])[flat_of(lead, 9)] ^= 1
        with pytest.raises(AssertionError):
            G.untouched(b, v)


def test_untouched_names_the_first_changed_element():
    view, base = G.embed((3, 5), torch.float32, rows_before=1, rows_after=1, device="cpu")
    base[2, 6] = 1.0
    with pytest.raises(AssertionError, match=r"row 2, column 6 of the \[5, 8\] allocation"):
        G.untouched(base, view)


def test_untouched_accepts_several_views_of_one_allocation():
    view, base = G.embed((6, 24), torch.bfloat16, rows_after=2, slack_cols=8, fill=G.NAN, device="cpu")
    q, k, v = view[:, :8], view[:, 8:16], view[:, 16:24]
    for t in (q, k, v):
        t.fill_(1.0)
    G.untouched(base, q, k, v, fill=G.NAN)
    with pytest.raises(AssertionError):
        G.untouched(base, q, v, fill=G.NAN)                 # k's columns are not the poison any more


def _compute_symbols():
    # the pattern of mmf_b200.lib.header_symbols(), applied to the header text without loading the library
    with open(HEADER) as fh:
        names = set(re.findall(r"\b(mmfb_[a-z0-9_]+)\s*\(", fh.read()))
    return {n for n in names if not n.endswith("_workspace_bytes") and n not in NOT_COMPUTE}


def _cases_table():
    with open(os.path.join(HERE, "test_poison_guard_gpu.py")) as fh:
        tree = ast.parse(fh.read())
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "CASES" for t in node.targets):
            return ast.literal_eval(node.value), tree
    raise AssertionError("tests/test_poison_guard_gpu.py has no CASES table")


def test_every_compute_entry_point_has_a_poison_case():
    cases, tree = _cases_table()
    missing = sorted(_compute_symbols() - set(cases))
    assert not missing, "compute entry points without a poison case in CASES: %s" % missing
    unknown = sorted(set(cases) - _compute_symbols())
    assert not unknown, "CASES names functions the header does not declare: %s" % unknown
    # every case names test functions that exist in the file, or says where the entry point is poisoned instead
    tests = {n.name for n in tree.body if isinstance(n, ast.FunctionDef) and n.name.startswith("test_")}
    for name, how in cases.items():
        if isinstance(how, str) and how.startswith("covered by "):
            continue
        names = [how] if isinstance(how, str) else list(how)
        assert names and all(t in tests for t in names), (name, how)
