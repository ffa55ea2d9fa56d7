"""CPU check that every `sliders_b200.ops` wrapper hands the C ABI exactly what tests/golden/ops_calls.pt recorded:
for each case of tests/golden/make_golden_ops_calls.py, the C function, every argument (which input or wrapper-allocated
tensor a pointer points into, each scalar, the `sb200_lora` fields), the `launch_count` delta, the refusals, and under
a reported capture the `profile_log` and `record_calls` entries and what `replay_calls` reissues."""
import importlib.util
import os

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _maker():
    spec = importlib.util.spec_from_file_location("make_golden_ops_calls",
                                                  os.path.join(GOLDEN, "make_golden_ops_calls.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MAKER = _maker()


@pytest.fixture(scope="module")
def fixture():
    return torch.load(os.path.join(GOLDEN, "ops_calls.pt"))


def test_fixture_covers_every_case(fixture):
    assert sorted(fixture) == sorted((c, m) for c in MAKER.CASES for m in ("plain", "capture"))


@pytest.mark.parametrize("mode", ["plain", "capture"])
@pytest.mark.parametrize("case", MAKER.CASES)
def test_ops_calls_match_fixture(fixture, case, mode):
    want = fixture[(case, mode)]
    got = MAKER.record(case, mode)
    assert got == want
