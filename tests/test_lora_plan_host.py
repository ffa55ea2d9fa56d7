"""CPU check that the LoRA packing hands the kernels exactly what tests/golden/lora_plan.pt recorded: every `ops.Lora`
of the UNet walk (r, rt, group_n, scale, scale_dev's value, the per-sample vector, rows_per_sample, the bytes of down
and up) and every `lora_compose`, call by call, in every scenario of tests/golden/make_golden_lora_plan.py: eager
walks, a training walk with its tape's `scales` record, and the CUDA-graph capture and scale-baking modes with a
replay's refresh."""
import importlib.util
import os

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _maker():
    spec = importlib.util.spec_from_file_location("make_golden_lora_plan",
                                                  os.path.join(GOLDEN, "make_golden_lora_plan.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MAKER = _maker()


@pytest.fixture(scope="module")
def fixture():
    return torch.load(os.path.join(GOLDEN, "lora_plan.pt"))


@pytest.mark.parametrize("cfg", MAKER.CONFIGS)
@pytest.mark.parametrize("scenario", list(MAKER.SCENARIOS))
def test_lora_plan_matches_fixture(fixture, cfg, scenario, capsys):
    want = fixture[(cfg, scenario)]
    got = MAKER.record(cfg, scenario)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, g, w)
