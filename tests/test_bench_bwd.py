"""CPU checks of benchmark/bench_bwd.py: argument parsing and FLOP accounting (nothing is timed)."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mod():
    spec = importlib.util.spec_from_file_location("bench_bwd", os.path.join(ROOT, "benchmark", "bench_bwd.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_default_cases_are_headline_gqa_and_d64():
    args, cases = _mod().parse([])
    assert args.seq == 32768 and args.dump is None and not args.deterministic
    assert cases == [(32, 32, 128), (32, 8, 128), (32, 32, 64)]


def test_custom_cases_and_dump():
    args, cases = _mod().parse(["--seq", "4096", "--heads", "16/4", "--dims", "64", "--dump", "out", "--deterministic"])
    assert args.seq == 4096 and args.dump == "out" and args.deterministic
    assert cases == [(16, 4, 64)]


@pytest.mark.parametrize("argv", [["--heads", "32/5"], ["--heads", "0/1"], ["--dims", "96"]])
def test_rejects_bad_shapes(argv):
    with pytest.raises(SystemExit):
        _mod().parse(argv)


def test_flops_are_two_and_a_half_causal_forwards():
    m = _mod()
    s, hq, d = 32768, 32, 128
    fwd = 4.0 * s * s * hq * d / 2  # causal forward: two GEMMs over half the score matrix
    assert m.bwd_flops(s, hq, d) == pytest.approx(2.5 * fwd)
    assert m.bwd_flops(s, hq, d) == pytest.approx(2.2e13, rel=0.01)


def test_per_pass_times_splits_launches_evenly():
    times, n = _mod().per_pass_times([1000.0, 2000.0, 3000.0, 4000.0], 2)
    assert n == 2 and times == [3.0, 7.0]


@pytest.mark.parametrize("kernel_us", [[], [1.0, 2.0, 3.0]])
def test_per_pass_times_rejects_missing_launches(kernel_us):
    with pytest.raises(SystemExit):
        _mod().per_pass_times(kernel_us, 2)
