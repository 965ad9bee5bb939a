"""bench.py host logic that needs no GPU: the algorithmic FLOP counts the throughput / roofline figures are built on
(pinned to BASELINE.md's table), the workload registry, and the default launch mode per configuration."""
import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def bench():
    return importlib.import_module("bench")


@pytest.mark.parametrize("name,gf,tokens", [("visual_bert", 122.9, 228), ("vilbert", 45.7, 72), ("mmbt", None, 122),
                                            ("mmft", None, 324), ("uniter_large", None, 120)])
def test_workload_flops_match_the_baseline_table(bench, name, gf, tokens):
    """fwd+bwd GFLOP per sample = 3 x forward (BASELINE.md, hot-path table); tokens per sample as SURVEY.md 8a lists them"""
    wl = bench.WORKLOADS[name]()
    assert wl.tokens_per_sample() == tokens
    got = 3 * wl.fwd_flops() / 1e9
    assert got > 0
    if gf is not None:
        assert abs(got - gf) / gf < 2e-3, (name, got)


def test_reference_arm_and_multi_gpu_runs_are_eager(bench, monkeypatch):
    """the CUDA-graph launch mode is a single-GPU default for the workloads it was validated with; everything else is eager"""
    import argparse

    def decide(workload, world, profile=False, impl="b200"):
        # the expression of bench.main(), kept in one place there; mirrored here on its inputs
        return (world == 1 and not profile and impl == "b200" and workload in ("visual_bert", "mmbt", "vilbert"))
    assert decide("visual_bert", 1) and decide("mmbt", 1) and decide("vilbert", 1)
    assert not decide("visual_bert", 8) and not decide("mmft", 1) and not decide("visual_bert", 1, profile=True)
    assert not decide("visual_bert", 1, impl="reference")
    src = open(os.path.join(ROOT, "bench.py")).read()
    assert 'args.workload in ("visual_bert", "mmbt", "vilbert")' in src and 'not args.profile and args.impl == "b200"' in src
    assert isinstance(argparse.ArgumentParser(), argparse.ArgumentParser)
