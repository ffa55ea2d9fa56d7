"""GPU tests of slider composition: the `lora_compose` kernel, SliderStacks on the tiny SDXL / SD1.x UNets against the
reference's chained LoRANetworks (tests/golden/compose.pt, tests/golden/make_golden_compose.py), per-slider scales
under CUDA-graph replay, and the denoise loop and eval sweep with a stack."""
import os

import pytest
import torch

from test_gpu_kernels import GUARD_ROWS, NAN_BITS, guarded_out
from test_gpu_unet import GOLDEN, dev, rel_rms  # noqa: F401  (fixture re-export)

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------------ kernel
def _guarded_f32(n, dev):
    """(buffer, out): a contiguous fp32 output of n values inside the bf16 guard-band buffer of `guarded_out` (one row
    of 2n bf16 columns, filled with NAN_BITS around it; 16-byte aligned when n is a multiple of 4)."""
    buf, view = guarded_out(1, 2 * n, dev)
    return buf, view.view(torch.float32)


def _assert_f32_guard_intact(buf, n):
    """assert_guard_intact's band check for an fp32 output (its NaN check of the interior reads bf16 halves, which the
    low halves of fp32 values can trip); that every value was written is the caller's equality check."""
    bits = buf.view(torch.int16)
    guard = torch.ones_like(bits, dtype=torch.bool)
    guard[GUARD_ROWS, :2 * n] = False
    bad = int((bits[guard] != NAN_BITS).sum())
    assert bad == 0, f"{bad} elements written outside the [{n}] fp32 output"


@pytest.mark.parametrize("rp", [4, 8, 16, 6])
def test_lora_compose_kernel_bitwise_with_guards(dev, rp):
    """Several packs of uneven row counts in one arena, composed in one launch and pack by pack: equal to torch's fp32
    product bit for bit, nothing written outside the output (rp 6 and a 4-byte offset take the scalar path)."""
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(rp)
    rows = [1, 37, 640, 3 * 1280 + 5, 77]
    R = sum(rows)
    raw = torch.randn(R, rp, generator=g).to(dev)
    mult = torch.randn(rp, generator=g)
    mult[1] = 0.0
    mult[-1] = -mult[-1]
    mult = mult.to(dev)
    want = raw * mult
    buf, flat = _guarded_f32(R * rp, dev)
    out = flat.view(R, rp)
    ops.lora_compose(raw, mult, out=out)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    _assert_f32_guard_intact(buf, R * rp)
    # pack by pack into a fresh buffer, and from a source that is only 4-byte aligned
    buf, flat = _guarded_f32(R * rp, dev)
    out = flat.view(R, rp)
    src = torch.empty(R * rp + 1, device=dev)
    src[1:].copy_(raw.flatten())
    n0 = 0
    for r in rows:
        ops.lora_compose(src[1 + n0 * rp:1 + (n0 + r) * rp].view(r, rp), mult, out=out[n0:n0 + r])
        n0 += r
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    _assert_f32_guard_intact(buf, R * rp)


def test_lora_compose_rejects_bad_arguments(dev):
    from sliders_b200 import _cabi, ops

    raw = torch.zeros(4, 8, device=dev)
    with pytest.raises(ValueError):
        ops.lora_compose(raw, torch.zeros(4, device=dev))
    with pytest.raises(_cabi.Sb200Error, match="distinct"):
        ops.lora_compose(raw, torch.zeros(8, device=dev), out=raw)


# ---------------------------------------------------------------------------------------- tiny UNets vs golden
def _inputs(f, dev):
    lat, ehs = f["latents"].to(dev), f["text_embeddings"].to(dev)
    added = None
    if "add_text_embeddings" in f:
        added = {"text_embeds": f["add_text_embeddings"].to(dev), "time_ids": f["add_time_ids"].to(dev)}
    return lat, ehs, added


def _unet(cfg_name, dev, weight_seed):
    from oracle import unet as ounet
    from sliders_b200 import synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    pm = UNet2DConditionModel(UNetConfig.from_dict(getattr(ounet.UNetConfig, cfg_name)().__dict__))
    synthetic.init_synthetic_(pm, seed=weight_seed)
    return pm.to(dev, BF).eval().requires_grad_(False)


def _stack(cfg_name, case, dev, weight_seed, up_std):
    from sliders_b200 import lora as plora
    from sliders_b200 import synthetic

    pm = _unet(cfg_name, dev, weight_seed)
    specs = [dict(rank=r, alpha=a, train_method=m, network_type=t) for r, a, m, t, _ in case["specs"]]
    stack = plora.SliderStack(pm, specs)
    for net, spec in zip(stack.sliders, case["specs"]):
        synthetic.init_lora_nonzero_(net, seed=spec[4], up_std=up_std, reseed_down=True)
    stack.to(dev, BF).requires_grad_(False)
    assert [len(n.unet_loras) for n in stack.sliders] == case["n_lora"]
    return pm, stack


def _eps(pm, f, dev):
    lat, ehs, added = _inputs(f, dev)
    with torch.no_grad():
        return pm(lat, f["timestep"], encoder_hidden_states=ehs, added_cond_kwargs=added).sample.float().cpu()


@pytest.mark.parametrize("cfg", ["tiny_xl", "tiny_sd"])
@pytest.mark.parametrize("case", ["two", "three"])
def test_stack_matches_reference_chained_networks(dev, cfg, case):
    fx = torch.load(os.path.join(GOLDEN, "compose.pt"))
    f, c = fx[cfg], fx[cfg][case]
    pm, stack = _stack(cfg, c, dev, fx["weight_seed"], fx["up_std"])
    scales = c["scales"]
    stack.__exit__(None, None, None)
    off = _eps(pm, f, dev)
    assert rel_rms(off, f["eps_off"]) < 2.5e-2
    for i in range(len(scales)):
        stack.set_lora_slider([s if j == i else 0.0 for j, s in enumerate(scales)])
        with stack:
            solo = _eps(pm, f, dev)
        err = rel_rms(solo, c[f"eps_solo{i}"])
        print(f"{cfg} {case} slider {i} alone: rel_rms {err:.3g}")
        assert err < 2.5e-2
    stack.set_lora_slider(scales)
    with stack:
        mix = _eps(pm, f, dev)
    err, derr = rel_rms(mix, c["eps_mix"]), rel_rms(mix - off, c["eps_mix"] - f["eps_off"])
    print(f"{cfg} {case} all sliders {scales}: eps rel_rms {err:.3g}, delta rel_rms {derr:.3g}")
    assert err < 2.5e-2
    assert derr < 5e-2


# ------------------------------------------------------------------------------------ scales and graph replay
def _plain(dev, fx, rank, alpha, method, conv, state):
    """A plain LoRANetwork on its own identical UNet holding `state` (adaptors it has and `state` lacks keep lora_up = 0,
    so they add nothing)."""
    from sliders_b200 import lora as plora

    pu = _unet("tiny_xl", dev, fx["weight_seed"])
    saved = list(plora.DEFAULT_TARGET_REPLACE)
    if conv:
        plora.DEFAULT_TARGET_REPLACE += plora.UNET_TARGET_REPLACE_MODULE_CONV
    try:
        net = plora.LoRANetwork(pu, rank=rank, alpha=alpha, train_method=method).to(dev, BF)
    finally:
        del plora.DEFAULT_TARGET_REPLACE[len(saved):]
    missing = set(state) - set(net.state_dict())
    assert not missing, missing
    net.load_state_dict(state, strict=False)
    return pu, net.requires_grad_(False)


def _plain_eps(pu, net, f, dev, scale, folded):
    """eps of the plain network at `scale`; `folded`: multiplier * alpha / r folded into the packed up weights (the
    walk's `bake` mode, taken under graph capture when the factors differ) instead of applied in the GEMM epilogue."""
    net.set_lora_slider(scale)
    with net:
        if not folded:
            return _eps(pu, f, dev)
        lat, ehs, added = _inputs(f, dev)
        t = torch.full((lat.shape[0],), float(f["timestep"]), device=dev)
        with torch.no_grad():
            return pu._walk(lat.contiguous(), t, ehs.to(BF).contiguous(), added, lat.dtype, bake=True).float().cpu()


def test_one_slider_on_matches_plain_network(dev):
    """One slider on, the other at 0, against that slider as a plain LoRANetwork on an identical UNet.

    A plain network has two paths for its scale multiplier * alpha / r: eager, with one factor common to every adaptor,
    it is applied in the GEMM epilogue; under graph capture with differing factors (the `bake` mode) it is folded into
    the packed up weights.  The stack always folds (per-slider scales cannot be one epilogue scalar), so it must equal
    the plain network's folded path bit for bit, both for the slider `alone` and for a `matched` network adapting
    exactly the stack's leaves (the slider's weights, lora_up = 0 elsewhere): the zero columns of the sliders at 0 and
    the per-block cross-attention K / V a stack with an xattn slider runs change nothing.  Against the plain network's
    epilogue path the stack differs by exactly what separates the plain network's own two paths (measured on an
    H100 80GB HBM3 at 700 W: 4.7e-3 for the noxattn slider, 7.4e-3 for the xattn slider, eps rel-RMS)."""
    fx = torch.load(os.path.join(GOLDEN, "compose.pt"))
    f, c = fx["tiny_xl"], fx["tiny_xl"]["two"]
    pm, stack = _stack("tiny_xl", c, dev, fx["weight_seed"], fx["up_std"])
    conv_any = any(t == "c3lier" for _, _, _, t, _ in c["specs"])
    union = {n for net in stack.sliders for n in (l.lora_name for l in net.unet_loras)}
    for i, (r, a, m, t, _) in enumerate(c["specs"]):
        stack.set_lora_slider([-1.5 if j == i else 0.0 for j in range(len(c["specs"]))])
        with stack:
            got = _eps(pm, f, dev)
        state = stack.sliders[i].state_dict()
        pa, alone = _plain(dev, fx, r, a, m, t == "c3lier", state)
        a_fold = _plain_eps(pa, alone, f, dev, -1.5, folded=True)
        a_epi = _plain_eps(pa, alone, f, dev, -1.5, folded=False)
        pu, matched = _plain(dev, fx, r, a, "full", conv_any, state)
        assert {l.lora_name for l in matched.unet_loras} == union
        m_fold = _plain_eps(pu, matched, f, dev, -1.5, folded=True)
        e_epi, e_own = rel_rms(got, a_epi), rel_rms(a_epi, a_fold)
        print(f"slider {i} ({m}, rank {r}) at -1.5: stack == plain folded {torch.equal(got, a_fold)}, == matched "
              f"folded {torch.equal(got, m_fold)}; stack vs plain epilogue {e_epi:.3g}; plain epilogue vs plain "
              f"folded {e_own:.3g}")
        assert torch.equal(got, a_fold)
        assert torch.equal(got, m_fold)
        assert abs(e_epi - e_own) <= 1e-4  # only the plain network's own choice of path remains
        del pu, matched, pa, alone


def test_scales_zero_and_graph_replay(dev):
    from sliders_b200 import generate
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "compose.pt"))
    f, c = fx["tiny_xl"], fx["tiny_xl"]["two"]
    pm, stack = _stack("tiny_xl", c, dev, fx["weight_seed"], fx["up_std"])
    bare = _unet("tiny_xl", dev, fx["weight_seed"])
    ref_off = _eps(bare, f, dev)

    # every slider at 0 is the un-adapted forward, bit for bit
    stack.set_lora_slider([0.0, 0.0])
    with stack:
        assert torch.equal(_eps(pm, f, dev), ref_off)
    stack.__exit__(None, None, None)
    assert torch.equal(_eps(pm, f, dev), ref_off)

    # graph replay == eager for three scale vectors, one composite graph for all of them
    vectors = ([1.0, -2.0], [0.0, 1.5], [-0.5, 0.0])
    eager = []
    for v in vectors:
        stack.set_lora_slider(v)
        with stack:
            eager.append(_eps(pm, f, dev))
    assert not torch.equal(eager[0], eager[1]) and not torch.equal(eager[1], eager[2])
    pm.use_cuda_graph = True
    pm._graphs.clear()
    for v, e in zip(vectors, eager):
        stack.set_lora_slider(v)
        with stack:
            assert torch.equal(_eps(pm, f, dev), e), v
    assert len(pm._graphs) == 1

    # the denoise loop's start_noise gating switches every slider off above start_noise: at most one more graph
    lat, ehs, added = _inputs(f, dev)
    sched = create_noise_scheduler("ddim")
    kw = dict(num_inference_steps=6, guidance_scale=3.0, start_noise=500)
    out = generate.denoise_loop(pm, stack, sched, lat[:1].clone(), ehs, added["text_embeds"], added["time_ids"],
                                scale=[2.0, -1.0], **kw)
    assert len(pm._graphs) == 2
    pm.use_cuda_graph = False
    ref = generate.denoise_loop(pm, stack, sched, lat[:1].clone(), ehs, added["text_embeds"], added["time_ids"],
                                scale=[2.0, -1.0], **kw)
    assert torch.isfinite(out).all()
    assert rel_rms(out, ref) < 1e-3
    off = generate.denoise_loop(pm, stack, sched, lat[:1].clone(), ehs, added["text_embeds"], added["time_ids"],
                                scale=0.0, **kw)
    assert rel_rms(out, off) > 1e-3  # the sliders act below start_noise


def test_eval_sweep_with_compose(dev, tmp_path):
    from sliders_b200 import eval_sweep as es
    from sliders_b200 import lora as plora
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "compose.pt"))
    age = tmp_path / "age_alpha1.0_rank4_noxattn_last.pt"
    smile = tmp_path / "smile_alpha1.0_rank8_noxattn_last.pt"
    # both names parse as rank / alpha 1 / noxattn + c3lier: retrain-free stand-ins with the layout the names imply
    src = plora.SliderStack(_unet("tiny_xl", dev, fx["weight_seed"]),
                            [dict(rank=4, alpha=1.0, train_method="noxattn", network_type="c3lier"),
                             dict(rank=8, alpha=1.0, train_method="noxattn", network_type="c3lier")])
    from sliders_b200 import synthetic
    for i, net in enumerate(src.sliders):
        synthetic.init_lora_nonzero_(net, seed=40 + i, up_std=0.1, reseed_down=True)
    src.sliders[0].save_weights(str(age), dtype=BF)
    src.sliders[1].save_weights(str(smile), dtype=BF)
    pm = _unet("tiny_xl", dev, fx["weight_seed"])
    pm.use_cuda_graph = True
    stack = plora.SliderStack.from_files(pm, [str(age), str(smile)], dev, BF)
    assert stack.ranks == (4, 8)
    csv_path = tmp_path / "p.csv"
    csv_path.write_text("case_number,prompt,evaluation_seed\n3,a,11\n")
    rows = es.read_prompts_csv(str(csv_path))
    g = torch.Generator().manual_seed(0)
    table = {"a": (torch.randn(2, 77, 256, generator=g), torch.randn(2, 128, generator=g))}
    save_dir = tmp_path / "out" / age.name
    kw = dict(scales=(-2, 0, 2), num_samples=1, num_inference_steps=6, guidance_scale=5.0, start_noise=750,
              image_size=256)
    n = es.sweep(pm, stack, create_noise_scheduler("euler"), rows, lambda p: table[p], str(save_dir),
                 fixed_scales=[-1.0], **kw)
    assert n == 3
    assert sorted(os.listdir(save_dir)) == ["-2", "0", "2"]
    lat = {s: torch.load(save_dir / str(s) / "3_0.pt") for s in (-2, 0, 2)}
    assert all(torch.isfinite(v).all() and v.shape == (4, 32, 32) for v in lat.values())
    assert not torch.equal(lat[-2], lat[2])
    # scale 0 of the swept slider still carries the composed one at -1: not the un-adapted model
    bare_dir = tmp_path / "bare"
    stack.set_lora_slider(0.0)
    es.sweep(pm, stack, create_noise_scheduler("euler"), rows, lambda p: table[p], str(bare_dir),
             **dict(kw, scales=(0,)))
    assert not torch.equal(lat[0], torch.load(bare_dir / "0" / "3_0.pt"))
