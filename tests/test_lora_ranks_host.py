"""CPU tests of the LoRA rank rule: an adaptor of rank 1-16 takes a slot of 4, 8 or 16 down rows / up columns in the
packed buffers of a fused call (ops.lora_slots), zero-padded past its rank, and the stacked down rows are padded to
rt = 16, 32 or 64.  The padded product equals the sum of the per-leaf deltas; rank 17 is refused; and the SDXL launch
plan at rank 16 equals the one at rank 4, with 64 LoRA-down rows on exactly the fused q|k|v projections."""
import collections
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

from oracle import unet as ounet
from sliders_b200 import lora as plora
from sliders_b200 import ops
from sliders_b200.unet import UNet2DConditionModel, UNetConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _slot(r):
    return 4 if r <= 4 else 8 if r <= 8 else 16


@pytest.mark.parametrize("r", range(1, 17))
@pytest.mark.parametrize("groups", [1, 2, 3])
def test_lora_slots_rule(r, groups):
    rp, rt = ops.lora_slots(r, groups)
    assert rp == _slot(r)
    assert rt == min(w for w in (16, 32, 64) if w >= groups * rp)


def test_lora_slots_keep_ranks_4_and_8_as_before():
    # the rt the fused kernels have always been given at ranks 4 and 8
    for r in (4, 8):
        for groups in (1, 2, 3):
            assert ops.lora_slots(r, groups) == (r, 16 if groups * r <= 16 else 32)
    assert ops.lora_slots(16, 1) == (16, 16)
    assert ops.lora_slots(16, 2) == (16, 32)  # attn2 to_k | to_v
    assert ops.lora_slots(16, 3) == (16, 64)  # attn1 to_q | to_k | to_v


@pytest.mark.parametrize("r", [0, 17, 32])
def test_rank_outside_1_to_16_is_refused(r):
    with pytest.raises(NotImplementedError, match="1-16"):
        ops.lora_slots(r)


def _leaves(r, groups, K=48, N=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    leaves, adaptors = [], []
    for i in range(groups):
        leaf = nn.Linear(K, N)
        a = plora.LoRAModule(f"leaf{i}", leaf, multiplier=1.0, lora_dim=r, alpha=float(r) / 2)
        with torch.no_grad():
            a.lora_down.weight.copy_(torch.randn(r, K, generator=g))
            a.lora_up.weight.copy_(torch.randn(N, r, generator=g))
        a.apply_to()
        leaves.append(leaf)
        adaptors.append(a)
    return leaves, adaptors


def _engine():
    return UNet2DConditionModel(UNetConfig.from_dict(ounet.UNetConfig.tiny_xl().__dict__))


@pytest.mark.parametrize("r", range(1, 17))
@pytest.mark.parametrize("groups", [1, 2, 3])
def test_pack_positions_zeros_and_product(r, groups):
    K, N = 48, 32
    leaves, adaptors = _leaves(r, groups, K, N, seed=100 * r + groups)
    la = _engine()._lora(leaves)
    rp, rt = _slot(r), ops.lora_slots(r, groups)[1]
    assert (la.r, la.rt, la.group_n) == (rp, rt, N)
    assert tuple(la.down.shape) == (rt, K) and tuple(la.up.shape) == (groups * N, rp)
    down, up = la.down.double(), la.up.double()
    for gi, a in enumerate(adaptors):
        rows = slice(gi * rp, gi * rp + r)
        assert torch.equal(down[rows], a.lora_down.weight.detach().to(torch.bfloat16).double())
        assert not down[gi * rp + r:(gi + 1) * rp].any()
        cols = slice(gi * N, (gi + 1) * N)
        assert torch.equal(up[cols, :r], a.lora_up.weight.detach().double())
        assert not up[cols, r:].any()
    assert not down[groups * rp:].any()
    # (x . down^T) . up^T through the pack, adaptor by adaptor (output column n uses rows [(n // group_n) * r, +r)),
    # equals the sum of the per-leaf deltas
    x = torch.randn(5, K, generator=torch.Generator().manual_seed(r), dtype=torch.float64)
    t = x @ down.t()
    got = torch.cat([t[:, gi * rp:(gi + 1) * rp] @ up[gi * N:(gi + 1) * N].t() for gi in range(groups)], dim=1)
    want = torch.cat([x @ a.lora_down.weight.detach().to(torch.bfloat16).double().t()
                      @ a.lora_up.weight.detach().double().t() for a in adaptors], dim=1)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    assert la.scale == adaptors[0].scale


def test_rank_17_is_refused_by_the_engine():
    leaves, _ = _leaves(17, 1)
    with pytest.raises(NotImplementedError, match="1-16"):
        _engine()._lora(leaves)


def test_sdxl_launch_plan_at_rank_16():
    """Same launches as at rank 4; rt = 64 on exactly the 70 fused q|k|v calls, 16 everywhere else (rank 4: 16
    everywhere)."""
    code = (
        "import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r + '/tools');"
        "import shape_trace as st;"
        "out = {}\n"
        "for r in (4, 16):\n"
        "    out[r] = [st.trace(2, rank=r), sorted(st.lora_rts.items())]\n"
        "print(json.dumps(out))" % (ROOT, ROOT))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    plans = json.loads(out.stdout.strip().splitlines()[-1])
    (plan4, rts4), (plan16, rts16) = plans["4"], plans["16"]
    assert plan4 == plan16 and len(plan4) == 1008
    assert [i for i, _ in rts4] == [i for i, _ in rts16]
    assert collections.Counter(rt for _, rt in rts4) == {16: len(rts4)}
    wide = [i for i, rt in rts16 if rt == 64]
    assert len(wide) == 70
    assert all(rt == 16 for _, rt in rts16 if _ not in wide)
    qkv = {"gemm M8192 N1920 K640 L", "gemm M2048 N3840 K1280 L"}  # attn1 of the 640 / 1280 levels at batch 2
    assert {plan16[i][1] for i in wide} == qkv
    assert sum(1 for _, d, _ in plan16 if d in qkv) == 70
