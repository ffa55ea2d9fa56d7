"""Host-side checks of per-sample slider scales and the batched scale sweep: the ctypes struct against the header, the
scale-major tiling, the chunking of scale lists, the shared prefix of each scheduler and the --scales_per_batch flag."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lora_args_layout_matches_header():
    """struct sb200_lora field order and offsets: the two per-sample fields come after scale_dev, so the existing
    fields keep their offsets."""
    from sliders_b200._cabi import LoraArgs

    src = open(os.path.join(ROOT, "include", "sb200.h")).read()
    body = re.search(r"typedef struct sb200_lora \{(.*?)\} sb200_lora;", src, re.S).group(1)
    names = [re.search(r"(\w+);", line).group(1) for line in body.splitlines() if ";" in line]
    assert names == [f[0] for f in LoraArgs._fields_]
    sizes = {"down": 8, "up": 8, "r": 4, "rt": 4, "group_n": 4, "scale": 4, "scale_dev": 8, "sample_scale": 8,
             "rows_per_sample": 4}
    off = 0
    for name in names:  # C layout on x86-64: natural alignment
        off = -(-off // sizes[name]) * sizes[name]
        assert getattr(LoraArgs, name).offset == off, name
        off += sizes[name]
    assert LoraArgs.scale_dev.offset == 32 and LoraArgs.sample_scale.offset == 40
    assert ctypes.sizeof(LoraArgs) == 56


def test_lora_defaults_and_derived_rows(monkeypatch):
    from sliders_b200 import ops

    d, u = torch.zeros(16, 64, dtype=torch.bfloat16), torch.zeros(64, 4)
    la = ops.Lora(d, u, 4, 64, 1.0)
    assert la._c.sample_scale is None and la._c.rows_per_sample == 0
    la = ops.Lora(d, u, 4, 64, 1.0, sample_scale=torch.ones(4))
    la.ref(4 * 77)
    assert la._c.rows_per_sample == 77
    with pytest.raises(ValueError, match="do not divide"):
        la.ref(4 * 77 + 1)
    la = ops.Lora(d, u, 4, 64, 1.0, sample_scale=torch.ones(4), rows_per_sample=5)
    la.ref(4 * 77)
    assert la._c.rows_per_sample == 5  # explicit values go to the launcher, which validates them


def test_scale_major_tiling():
    from sliders_b200 import generate

    lat = torch.arange(3 * 2).view(3, 2).float()
    t = generate.tile_scale_major(lat, 4)
    assert t.shape == (12, 2)
    for k in range(4):
        for i in range(3):
            assert torch.equal(t[k * 3 + i], lat[i])
    pe = torch.cat([-lat - 1, lat])  # (negatives; positives)
    tc = generate.tile_cfg(pe, 4)
    assert torch.equal(tc, torch.cat([generate.tile_scale_major(lat, 4)] * 2) * torch.cat(
        [-torch.ones(12, 1), torch.ones(12, 1)]) - torch.cat([torch.ones(12, 2), torch.zeros(12, 2)]))
    # the UNet sees batch entry b of cat([latents] * 2) at per-sample value scale[b % (N k)]; scale c covers rows c*N..
    N, k, chunk = 3, 4, [-2.0, -1.0, 0.5, 2.0]
    vals = [s for s in chunk for _ in range(N)]
    for b in range(2 * N * k):
        assert vals[b % len(vals)] == chunk[(b % (N * k)) // N]


@pytest.mark.parametrize("scales,K,want", [
    ([-2, -1, 0, 1, 2], 2, [[-2, -1], [0, 1], [2]]),
    ([-2, -1, 0, 1, 2], 3, [[-2, -1, 0], [1, 2]]),
    ([-2, -1, 0, 1, 2], 5, [[-2, -1, 0, 1, 2]]),
    ([-2, -1, 0], 8, [[-2, -1, 0]]),
    ([], 3, []),
])
def test_sweep_chunks(scales, K, want):
    from sliders_b200 import generate

    assert generate.sweep_chunks(scales, K) == want


@pytest.mark.parametrize("kind,steps,start_noise,want", [
    ("euler", 50, 750, 12),    # leading spacing + offset 1: 981, 961, ..., 761
    ("ddim", 50, 750, 12),     # 980, 960, ..., 760
    ("euler_a", 50, 750, 13),  # linspace spacing: 999, 978.6, ..., 754.3
    ("lms", 50, 750, 13),
    ("ddpm", 50, 750, 12),
    ("euler", 8, -1, 8),       # every step before start_noise: nothing but the shared part
    ("ddim", 8, 1000, 0),
])
def test_shared_prefix_steps(kind, steps, start_noise, want):
    from sliders_b200 import generate
    from sliders_b200.scheduler import create_noise_scheduler

    sched = create_noise_scheduler(kind)
    n = generate.shared_prefix_steps(sched, steps, start_noise)
    ts = [float(t) for t in (getattr(sched, "timesteps_host", None) or sched.timesteps)]
    assert n == sum(int(t) > start_noise for t in ts) == want
    assert all(int(t) > start_noise for t in ts[:n])


def test_cli_scales_per_batch():
    from sliders_b200 import eval_sweep as es

    base = ["--model_name", "m.pt", "--prompts_path", "p.csv", "--save_path", "o"]
    assert es.parse_args(base).scales_per_batch == 1
    assert es.parse_args(base + ["--scales_per_batch", "5"]).scales_per_batch == 5
    assert es.parse_args(base + ["--compose", "b.pt:1.0"]).scales_per_batch == 1
    with pytest.raises(SystemExit):
        es.parse_args(base + ["--compose", "b.pt:1.0", "--scales_per_batch", "2"])
    with pytest.raises(SystemExit):
        es.parse_args(base + ["--scales_per_batch", "0"])


def test_set_lora_slider_values():
    from sliders_b200 import lora

    assert lora._per_sample_values(1.5) is None
    assert lora._per_sample_values(torch.tensor(2.0)) is None
    assert lora._per_sample_values([1, -2.5]) == (1.0, -2.5)
    assert lora._per_sample_values(torch.tensor([0.5, 1.0])) == (0.5, 1.0)
    with pytest.raises(ValueError):
        lora._per_sample_values([])
    with pytest.raises(ValueError):
        lora._per_sample_values(torch.ones(2, 2))


def test_scale_sweep_rejects_bad_batch_size():
    from sliders_b200 import generate

    with pytest.raises(ValueError, match="scales_per_batch"):
        generate.scale_sweep(None, None, None, torch.zeros(1, 4, 8, 8), torch.zeros(2, 77, 8), scales_per_batch=0)
