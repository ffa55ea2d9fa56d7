"""GPU parity tests of the whole hot path: sliders_b200.UNet2DConditionModel + LoRANetwork + train_util
(`predict_noise(_xl)`, `diffusion_xl`) through the C ABI versus (a) the committed golden vectors that the
reference's own unmodified lora.py / train_util.py produced on the oracle (tests/golden/make_golden.py) and (b) the
fp32 oracle run live on the same seeded weights / inputs.

Tolerance (BASELINE.json north_star: "within a stated fp16 tolerance"): the kernels compute in bf16 with fp32
accumulation, the oracle in fp32.  Stated bound: relative RMS error of the predicted noise <= 2.5e-2 for a single
conditioned pass and for guidance-combined eps (guidance g multiplies the difference of two passes, so the bound is
looser for g = 7.5: 0.1); max-abs error <= 0.15 on eps ~ N(0, 0.6).  For context, PyTorch's own bf16 autocast of
the oracle differs from the fp32 oracle by 0.9e-2 rel-RMS on the full SDXL UNet (profiles/r01_unet_sdxl.log), our
kernels by 0.75e-2."""
import os

import pytest
import torch

from conftest import c3lier

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
BF = torch.bfloat16


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def rel_rms(got, ref):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert torch.isfinite(got).all()
    return ((got - ref).norm() / ref.norm()).item()


def build_product(fx, dev):
    """Product UNet + LoRANetwork with the fixture's seeded weights (regenerated, not stored)."""
    from oracle import unet as ounet
    from sliders_b200 import lora as plora, synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    ocfg = getattr(ounet.UNetConfig, fx["config"])()
    pm = UNet2DConditionModel(UNetConfig.from_dict(ocfg.__dict__))
    synthetic.init_synthetic_(pm, seed=fx["weight_seed"])  # CPU generator: identical to the oracle's weights
    pm = pm.to(dev, BF).eval()
    pm.requires_grad_(False)
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=fx["rank"], multiplier=1.0, alpha=fx["alpha"], train_method="noxattn")
    synthetic.init_lora_nonzero_(net, seed=fx["lora_seed"], up_std=fx["up_std"], reseed_down=True)
    net = net.to(dev, BF)
    assert len(net.unet_loras) == fx["n_lora"]
    return pm, net


def test_golden_tiny_xl_reference_call_sites(dev):
    """predict_noise_xl / diffusion_xl / set_lora_slider semantics against what the reference's code produced."""
    from sliders_b200 import train_util
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    sched = create_noise_scheduler("ddim")
    lat, ehs = fx["latents"].to(dev), fx["text_embeddings"].to(dev)
    pooled, tids = fx["add_text_embeddings"].to(dev), fx["add_time_ids"].to(dev)
    t = fx["timestep"]
    sched.set_timesteps(1000)
    assert int(sched.timesteps[500]) == t
    with torch.no_grad():
        net.__exit__(None, None, None)  # multiplier 0 outside the context manager (lora.py:256-258)
        off1 = train_util.predict_noise_xl(pm, sched, t, lat, ehs, pooled, tids, guidance_scale=1)
        off3 = train_util.predict_noise_xl(pm, sched, t, lat, ehs, pooled, tids, guidance_scale=3)
        with net:
            on1 = train_util.predict_noise_xl(pm, sched, t, lat, ehs, pooled, tids, guidance_scale=1)
        net.set_lora_slider(-2.0)
        with net:
            onm2 = train_util.predict_noise_xl(pm, sched, t, lat, ehs, pooled, tids, guidance_scale=3)
        net.set_lora_slider(1.0)
        sched.set_timesteps(50)
        with net:
            den = train_util.diffusion_xl(pm, sched, lat, ehs, pooled, tids, guidance_scale=3, total_timesteps=3)
    assert rel_rms(off1, fx["eps_off_g1"]) < 2.5e-2
    assert rel_rms(off3, fx["eps_off_g3"]) < 2.5e-2
    assert rel_rms(on1, fx["eps_on_s1_g1"]) < 2.5e-2
    assert rel_rms(onm2, fx["eps_on_sm2_g3"]) < 2.5e-2
    assert rel_rms(den, fx["denoised_3of50_g3"]) < 2.5e-2
    assert (off1.float().cpu() - fx["eps_off_g1"]).abs().max() < 0.15
    # the adaptor's effect is resolved well above the error floor, with the right sign for a negative slider
    eff = fx["eps_on_s1_g1"] - fx["eps_off_g1"]
    got_eff = (on1 - off1).float().cpu()
    assert torch.nn.functional.cosine_similarity(got_eff.flatten(), eff.flatten(), dim=0) > 0.98
    # loss formula on the four predictions (prompt_util.py:123-135), enhance, guidance 4.  The loss is a mean of
    # squared differences in which the bf16 error of two predictions enters multiplied by the guidance scale 4 and
    # squared, so its relative tolerance is looser than the eps tolerance (measured: 9 %).
    loss = torch.nn.functional.mse_loss(on1.float(), off1.float() + 4.0 * (off3.float() - onm2.float()))
    assert abs(loss.item() - fx["loss_enhance_g4"].item()) / fx["loss_enhance_g4"].item() < 0.2


def test_golden_tiny_sd_predict_noise(dev):
    """SD1.x topology (conv projections, 4 levels, no text_time embedding), rank 8, alpha 4, batch 2."""
    from sliders_b200 import train_util
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_sd.pt"))
    pm, net = build_product(fx, dev)
    sched = create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    lat, ehs, t = fx["latents"].to(dev), fx["text_embeddings"].to(dev), fx["timestep"]
    with torch.no_grad():
        net.__exit__(None, None, None)
        off = train_util.predict_noise(pm, sched, t, lat, ehs, guidance_scale=7.5)
        with net:
            on = train_util.predict_noise(pm, sched, t, lat, ehs, guidance_scale=1)
    # guidance 7.5: eps = u + 7.5 (c - u) amplifies the independent bf16 errors of the two passes by ~7.5 * sqrt(2)
    # relative to a single pass (0.65e-2 measured) -> expected ~7e-2; bound 0.1
    assert rel_rms(off, fx["eps_off_g7.5"]) < 0.1
    assert rel_rms(on, fx["eps_on_s1_g1"]) < 2.5e-2


def test_identities_bit_exact(dev):
    """Zero-initialised LoRA == no LoRA; multiplier 0 == no LoRA; CUDA-graph replay == eager; run-to-run
    reproducibility — all bit-exact (no atomics anywhere on the path)."""
    from sliders_b200 import lora as plora, synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig
    from oracle import unet as ounet

    ocfg = ounet.UNetConfig.tiny_xl()
    with torch.device(dev):
        pm = UNet2DConditionModel(UNetConfig.from_dict(ocfg.__dict__)).to(BF)
    synthetic.init_synthetic_(pm, seed=3)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 32, 32, generator=g).to(dev)
    ehs = torch.randn(2, 77, 256, generator=g).to(dev, BF)
    added = {"text_embeds": torch.randn(2, 128, generator=g).to(dev, BF),
             "time_ids": torch.tensor([[256., 256, 0, 0, 256, 256]] * 2, device=dev)}
    with torch.no_grad():
        base = pm(x, 321, ehs, added_cond_kwargs=added).sample
        again = pm(x, 321, ehs, added_cond_kwargs=added).sample
        assert torch.equal(base, again)
        with c3lier(plora):
            net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
        with net:
            fresh = pm(x, 321, ehs, added_cond_kwargs=added).sample  # lora_up == 0
        assert torch.equal(fresh, base)
        synthetic.init_lora_nonzero_(net, seed=4, up_std=0.05)
        off = pm(x, 321, ehs, added_cond_kwargs=added).sample  # multiplier 0 after __exit__
        assert torch.equal(off, base)
        net.set_lora_slider(1.5)
        with net:
            on = pm(x, 321, ehs, added_cond_kwargs=added).sample
        assert not torch.equal(on, base)
        pm.use_cuda_graph = True
        with net:
            g_on = pm(x, 321, ehs, added_cond_kwargs=added).sample
        net.set_lora_slider(-0.5)
        with net:
            g_neg = pm(x, 321, ehs, added_cond_kwargs=added).sample  # same graph, slider read from device memory
        g_off = pm(x, 321, ehs, added_cond_kwargs=added).sample
        pm.use_cuda_graph = False
        with net:
            e_neg = pm(x, 321, ehs, added_cond_kwargs=added).sample
        assert torch.equal(g_on, on) and torch.equal(g_neg, e_neg) and torch.equal(g_off, base)
        # linearity in the slider value for small scales is a property of the folded epilogue: eps(s) - eps(0)
        # changes sign with s
        d_pos, d_neg = (on - base).float(), (e_neg - base).float()
        assert torch.nn.functional.cosine_similarity(d_pos.flatten(), d_neg.flatten(), dim=0) < -0.5


def _grad_report(net, golden):
    """Per-tensor rel-RMS of the LoRA gradients vs the reference's, plus the global (concatenated) figure, over the
    adaptors the fixture stores (a fixed subset, to keep the file small)."""
    num = den = 0.0
    worst = (0.0, None)
    compared = 0
    for k, p in net.named_parameters():
        if k not in golden:
            continue
        compared += 1
        ref = golden[k].float().to(p.device)
        assert p.grad is not None, k
        got = p.grad.float()
        assert torch.isfinite(got).all(), k
        e, n = (got - ref).pow(2).sum().item(), ref.pow(2).sum().item()
        num, den = num + e, den + n
        r = (e / max(n, 1e-30)) ** 0.5
        if r > worst[0]:
            worst = (r, k)
    assert compared == len(golden), (compared, len(golden))
    return (num / den) ** 0.5, worst


def test_golden_tiny_xl_lora_gradients(dev):
    """One text-slider step's `loss.backward()` (train_lora_xl.py:299-345) against the gradients the reference's own
    code produced (tests/golden/make_golden_grads.py): every lora_down / lora_up of the 178 adaptors.  Tolerance: the
    product back-propagates in bf16 (as the reference does on GPU), the fixture is fp32 -> global rel-RMS <= 5e-2."""
    from sliders_b200 import train_util
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    gg = torch.load(os.path.join(GOLDEN, "tiny_xl_grads.pt"))
    pm, net = build_product(fx, dev)
    net.requires_grad_(True)
    sched = create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    lat, ehs = fx["latents"].to(dev), fx["text_embeddings"].to(dev)
    pooled, tids = fx["add_text_embeddings"].to(dev), fx["add_time_ids"].to(dev)
    with net:
        target = train_util.predict_noise_xl(pm, sched, fx["timestep"], lat, ehs, pooled, tids, guidance_scale=1)
    assert target.requires_grad
    assert rel_rms(target, gg["target"]) < 3e-2
    # guidance 1: the UNet node was told that its unconditional sample gets a zero gradient (backward runs on the
    # conditional half only; the golden gradients below are the reference's full-batch autograd)
    node = target.grad_fn
    while node is not None and not type(node).__name__.startswith("_UNetFunction"):
        node = next((f for f, _ in node.next_functions if f is not None), None)
    assert node is not None and getattr(node, "zero_rows", 0) == 1
    pos, neu, unc = fx["eps_off_g3"].to(dev), fx["eps_off_g1"].to(dev), fx["eps_on_sm2_g3"].to(dev)
    loss = torch.nn.functional.mse_loss(target, neu + 4.0 * (pos - unc))  # prompt_util.py:123-135 (enhance)
    assert abs(loss.item() - gg["loss"].item()) < 0.1 * gg["loss"].item()
    loss.backward()
    torch.cuda.synchronize()
    total, worst = _grad_report(net, gg["grads"])
    assert total < 5e-2, (total, worst)
    assert worst[0] < 0.25, worst
    # a second forward / backward accumulates into .grad like torch does
    with net:
        target = train_util.predict_noise_xl(pm, sched, fx["timestep"], lat, ehs, pooled, tids, guidance_scale=1)
    torch.nn.functional.mse_loss(target, neu + 4.0 * (pos - unc)).backward()
    total2, _ = _grad_report(net, {k: 2 * v.float() for k, v in gg["grads"].items()})
    assert total2 < 5e-2


def test_golden_tiny_sd_lora_gradients(dev):
    """SD1.x topology, rank 8, negative slider, image-slider style loss (train_lora-scale-xl.py:338)."""
    from sliders_b200 import train_util
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_sd.pt"))
    gg = torch.load(os.path.join(GOLDEN, "tiny_sd_grads.pt"))
    pm, net = build_product(fx, dev)
    net.requires_grad_(True)
    sched = create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    net.set_lora_slider(-1.0)
    with net:
        pred = train_util.predict_noise(pm, sched, fx["timestep"], fx["latents"].to(dev),
                                        fx["text_embeddings"].to(dev), guidance_scale=1)
    assert rel_rms(pred, gg["pred"]) < 3e-2
    loss = torch.nn.functional.mse_loss(pred.float(), gg["noise"].to(dev).float())
    loss.backward()
    torch.cuda.synchronize()
    total, worst = _grad_report(net, gg["grads"])
    assert total < 5e-2, (total, worst)
    # outside `with network:` the multiplier is 0: no adaptor is active, the inference forward runs
    out = train_util.predict_noise(pm, sched, fx["timestep"], fx["latents"].to(dev), fx["text_embeddings"].to(dev),
                                   guidance_scale=1)
    assert not out.requires_grad


@pytest.mark.parametrize("batch", [2])
def test_full_sdxl_parity_vs_fp32_oracle(dev, batch):
    """BASELINE workload size: SDXL-base UNet (2.57 B parameters, synthetic seeded weights), 128x128 latents, rank-4
    LoRA on 346 leaves at slider 2.  The oracle runs in fp32 on the same device (plain PyTorch, TF32 off) with the
    LoRA delta folded into its weights; tests/test_oracle.py pins that folding to the reference's forward hook."""
    from oracle import unet as ounet
    from sliders_b200 import lora as plora, synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    with torch.device(dev):
        pm = UNet2DConditionModel(UNetConfig.sdxl()).to(BF)
        om = ounet.UNet2DConditionModel(ounet.UNetConfig.sdxl())
    synthetic.init_synthetic_(pm, seed=1)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om.eval()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(batch, 4, 128, 128, generator=g).to(dev, BF)
    ehs = torch.randn(batch, 77, 2048, generator=g).to(dev, BF)
    added = {"text_embeds": torch.randn(batch, 1280, generator=g).to(dev, BF),
             "time_ids": torch.tensor([[1024., 1024, 0, 0, 1024, 1024]] * batch, device=dev)}
    addf = {"text_embeds": added["text_embeds"].float(), "time_ids": added["time_ids"]}
    with torch.no_grad():
        got = pm(x, 500, ehs, added_cond_kwargs=added).sample
        ref = om(x.float(), 500, ehs.float(), added_cond_kwargs=addf).sample
    # SURVEY.md §4 bar for the full-size model: rel-RMS <= 1e-2, max-abs <= 3e-2 (bf16 product vs fp32 oracle; the
    # reference itself runs this path in fp16/bf16 autocast, so the oracle is the tighter of the two comparisons)
    print(f"full SDXL base: rel_rms {rel_rms(got, ref):.4g} max_abs {(got.float() - ref).abs().max().item():.4g} "
          f"ref_rms {ref.pow(2).mean().sqrt().item():.4g}")
    assert rel_rms(got, ref) < 1e-2
    assert (got.float() - ref).abs().max().item() < 3e-2          # measured 0.0221 (deterministic kernels, fixed seeds)
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
    assert len(net.unet_loras) == 346
    synthetic.init_lora_nonzero_(net, seed=2, up_std=0.05)
    mods = {("lora_unet_" + n.replace(".", "_")): m for n, m in om.named_modules()}
    sd = net.state_dict()
    with torch.no_grad():
        for l in net.unet_loras:
            up, down = sd[l.lora_name + ".lora_up.weight"].float(), sd[l.lora_name + ".lora_down.weight"].float()
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down) if down.dim() == 4 else up @ down
            mods[l.lora_name].weight.add_(delta * (2.0 * l.scale))
        ref_l = om(x.float(), 19, ehs.float(), added_cond_kwargs=addf).sample
        net.set_lora_slider(2.0)
        with net:
            got_l = pm(x, 19, ehs, added_cond_kwargs=added).sample
    print(f"full SDXL + LoRA(346, slider 2): rel_rms {rel_rms(got_l, ref_l):.4g} "
          f"max_abs {(got_l.float() - ref_l).abs().max().item():.4g} ref_max {ref_l.abs().max().item():.4g}")
    assert rel_rms(got_l, ref_l) < 1e-2
    assert (got_l.float() - ref_l).abs().max().item() < 3e-2      # measured 0.0234
    # the same forward with LayerNorm folded into the consuming projections (sb200_gemm_ln; off by default)
    pm.fuse_layernorm = True
    with torch.no_grad(), net:
        got_f = pm(x, 19, ehs, added_cond_kwargs=added).sample
    pm.fuse_layernorm = False
    print(f"  LayerNorm-folded: rel_rms {rel_rms(got_f, ref_l):.4g}")
    assert rel_rms(got_f, ref_l) < 1e-2


def test_denoise_loop_with_slider_gating(dev):
    """eval-scripts/generate_images_xl.py:325-364 restated for the oracle: 5 DDIM steps, guidance 5, slider -1.5
    gated by start_noise (adaptors off for t > start_noise).  Oracle: two fp32 UNets (base / LoRA-folded)."""
    import copy

    from oracle import ddim as oddim
    from oracle import unet as ounet
    from sliders_b200 import generate, synthetic
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    om = ounet.UNet2DConditionModel(ounet.UNetConfig.tiny_xl())
    synthetic.init_synthetic_(om, seed=fx["weight_seed"])
    om.eval()
    om_l = copy.deepcopy(om)
    slider = -1.5
    mods = {("lora_unet_" + n.replace(".", "_")): m for n, m in om_l.named_modules()}
    sd = {k: v.float().cpu() for k, v in net.state_dict().items()}
    with torch.no_grad():
        for l in net.unet_loras:
            up, down = sd[l.lora_name + ".lora_up.weight"], sd[l.lora_name + ".lora_down.weight"]
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down) if down.dim() == 4 else up @ down
            mods[l.lora_name].weight.add_(delta * (slider * l.scale))
    g = torch.Generator().manual_seed(7)
    lat = torch.randn(2, 4, 32, 32, generator=g)
    ehs = fx["text_embeddings"].repeat_interleave(2, dim=0)     # [neg, neg, pos, pos]
    pooled = fx["add_text_embeddings"].repeat_interleave(2, dim=0)
    tids = fx["add_time_ids"].repeat_interleave(2, dim=0)
    steps, start_noise, gs = 5, 500, 5.0
    # oracle loop
    sch = oddim.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                              num_train_timesteps=1000, clip_sample=False)
    sch.set_timesteps(steps)
    x = lat.clone()
    with torch.no_grad():
        for t in sch.timesteps:
            model = om if int(t) > start_noise else om_l
            out = model(torch.cat([x] * 2), int(t), ehs, added_cond_kwargs={"text_embeds": pooled, "time_ids": tids}).sample
            u, c = out.chunk(2)
            x = sch.step(u + gs * (c - u), int(t), x).prev_sample
    got = generate.denoise_loop(pm, net, create_noise_scheduler("ddim"), lat.to(dev), ehs.to(dev), pooled.to(dev),
                                tids.to(dev), num_inference_steps=steps, guidance_scale=gs, scale=slider,
                                start_noise=start_noise)
    assert rel_rms(got, x) < 4e-2  # five guided steps (g = 5) accumulate the per-step bf16 error
    # the same loop under CUDA-graph replay is bit-identical
    pm.use_cuda_graph = True
    got_g = generate.denoise_loop(pm, net, create_noise_scheduler("ddim"), lat.to(dev), ehs.to(dev), pooled.to(dev),
                                  tids.to(dev), num_inference_steps=steps, guidance_scale=gs, scale=slider,
                                  start_noise=start_noise)
    pm.use_cuda_graph = False
    assert torch.equal(got_g, got)


def test_full_sd15_parity_vs_fp32_oracle(dev):
    """BASELINE config 2: SD-1.x UNet (859.5 M parameters, head dims 40 / 80 / 160, 1x1-conv projections, 8x8
    bottleneck), 64x64 latents (512 px), rank-4 LoRA on 150 leaves, CFG pair through `predict_noise`."""
    from oracle import unet as ounet
    from sliders_b200 import lora as plora, synthetic, train_util
    from sliders_b200.scheduler import create_noise_scheduler
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    with torch.device(dev):
        pm = UNet2DConditionModel(UNetConfig.sd15()).to(BF)
        om = ounet.UNet2DConditionModel(ounet.UNetConfig.sd15())
    synthetic.init_synthetic_(pm, seed=5)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om.eval()
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
    assert len(net.unet_loras) == 150
    synthetic.init_lora_nonzero_(net, seed=6, up_std=0.05)
    mods = {("lora_unet_" + n.replace(".", "_")): m for n, m in om.named_modules()}
    sd = net.state_dict()
    with torch.no_grad():
        for l in net.unet_loras:
            up, down = sd[l.lora_name + ".lora_up.weight"].float(), sd[l.lora_name + ".lora_down.weight"].float()
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down) if down.dim() == 4 else up @ down
            mods[l.lora_name].weight.add_(delta * l.scale)
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(2, 4, 64, 64, generator=g).to(dev, BF)
    ehs = torch.randn(4, 77, 768, generator=g).to(dev, BF)  # [u, u, c, c]
    sched = create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    with torch.no_grad():
        out = om(torch.cat([lat.float()] * 2), 321, ehs.float()).sample
        u, c = out.chunk(2)
        ref = u + 1.0 * (c - u)
        with net:
            got = train_util.predict_noise(pm, sched, 321, lat, ehs, guidance_scale=1.0)
    assert rel_rms(got, ref) < 2.5e-2


def test_full_sdxl_lora_gradients_vs_fp32_oracle(dev):
    """BASELINE-size backward: SDXL UNet, 128x128 latents, CFG pair, rank-4 LoRA on 346 leaves.  The oracle is the
    fp32 restatement under torch autograd with W_eff = W + s * up @ down built from leaf tensors (the same function
    as the reference's forward hook, tests/test_oracle.py pins that), so its d/d(up, down) are the reference's
    gradients.  Tolerance: bf16 back-propagation through ~400 layers vs fp32 -> global rel-RMS <= 6e-2."""
    from oracle import unet as ounet
    from sliders_b200 import lora as plora, synthetic, train_util
    from sliders_b200.scheduler import create_noise_scheduler
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    with torch.device(dev):
        pm = UNet2DConditionModel(UNetConfig.sdxl()).to(BF)
        om = ounet.UNet2DConditionModel(ounet.UNetConfig.sdxl())
    synthetic.init_synthetic_(pm, seed=1)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om.eval().requires_grad_(False)
    pm.requires_grad_(False)
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
    synthetic.init_lora_nonzero_(net, seed=2, up_std=0.05)
    net.requires_grad_(True)
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(1, 4, 128, 128, generator=g).to(dev, BF)
    ehs = torch.randn(2, 77, 2048, generator=g).to(dev, BF)
    pooled = torch.randn(2, 1280, generator=g).to(dev, BF)
    tids = torch.tensor([[1024., 1024., 0., 0., 1024., 1024.]] * 2, device=dev)
    goal = torch.randn(1, 4, 128, 128, generator=g).to(dev)
    sched = create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    net.set_lora_slider(1.5)
    with net:
        pred = train_util.predict_noise_xl(pm, sched, 500, lat, ehs, pooled, tids, guidance_scale=1)
    loss = torch.nn.functional.mse_loss(pred.float(), goal)
    loss.backward()
    torch.cuda.synchronize()
    # ---- oracle
    names = {"lora_unet_" + n.replace(".", "_"): n for n, _ in om.named_modules()}
    params = dict(om.named_parameters())
    leaves, eff = {}, {}
    for l in net.unet_loras:
        down = l.lora_down.weight.detach().float().requires_grad_()
        up = l.lora_up.weight.detach().float().requires_grad_()
        leaves[l.lora_name] = (down, up)
        w = params[names[l.lora_name] + ".weight"]
        s = 1.5 * l.scale
        if down.dim() == 4:
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down)
        else:
            delta = up @ down
        eff[names[l.lora_name] + ".weight"] = w + s * delta
    full = {**params, **eff}
    out = torch.func.functional_call(om, full, (torch.cat([lat.float()] * 2), 500, ehs.float()),
                                     {"added_cond_kwargs": {"text_embeds": pooled.float(), "time_ids": tids}}).sample
    u, c = out.chunk(2)
    ref_pred = u + 1.0 * (c - u)
    assert rel_rms(pred, ref_pred) < 2.5e-2
    torch.nn.functional.mse_loss(ref_pred, goal).backward()
    num = den = 0.0
    worst = (0.0, None)
    for l in net.unet_loras:
        for got, ref in ((l.lora_down.weight.grad, leaves[l.lora_name][0].grad),
                         (l.lora_up.weight.grad, leaves[l.lora_name][1].grad)):
            assert got is not None and torch.isfinite(got).all(), l.lora_name
            e, n = (got.float() - ref).pow(2).sum().item(), ref.pow(2).sum().item()
            num, den = num + e, den + n
            r = (e / max(n, 1e-30)) ** 0.5
            if r > worst[0]:
                worst = (r, l.lora_name)
    total = (num / den) ** 0.5
    print(f"SDXL LoRA gradient rel-RMS vs fp32 oracle: global {total:.4f}, worst tensor {worst[0]:.4f} ({worst[1]})")
    assert total < 6e-2, (total, worst)


def _oracle_lora_grads(om, net, slider, call):
    """LoRA gradients of the fp32 oracle with W_eff = W + s * up @ down built from leaf tensors (the reference's
    forward hook as a weight fold).  `call(functional_params) -> loss`."""
    names = {"lora_unet_" + n.replace(".", "_"): n for n, _ in om.named_modules()}
    params = dict(om.named_parameters())
    leaves, eff = {}, {}
    for l in net.unet_loras:
        down = l.lora_down.weight.detach().float().requires_grad_()
        up = l.lora_up.weight.detach().float().requires_grad_()
        leaves[l.lora_name] = (down, up)
        w = params[names[l.lora_name] + ".weight"]
        if down.dim() == 4:
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down)
        else:
            delta = up @ down
        eff[names[l.lora_name] + ".weight"] = w + slider * l.scale * delta
    call({**params, **eff}).backward()
    return leaves


@pytest.mark.parametrize("method,n_expected", [("full", None), ("xattn", None), ("selfattn", None)])
def test_tiny_xl_gradients_other_train_methods(dev, method, n_expected):
    """train methods that adapt the cross-attention projections (lora.py:176-188): the text-side K / V adaptors get
    their gradients from the dK / dV pass of the attention backward; `selfattn` leaves every conv untouched."""
    from oracle import unet as ounet
    from sliders_b200 import lora as plora, synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    ocfg = ounet.UNetConfig.tiny_xl()
    pm = UNet2DConditionModel(UNetConfig.from_dict(ocfg.__dict__))
    synthetic.init_synthetic_(pm, seed=21)
    om = ounet.UNet2DConditionModel(ocfg)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om = om.to(dev).eval().requires_grad_(False)
    pm = pm.to(dev, BF).eval().requires_grad_(False)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})  # the bf16-rounded weights
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=2.0, train_method=method).to(dev, BF)
    synthetic.init_lora_nonzero_(net, seed=22, up_std=0.05, reseed_down=True)
    net.requires_grad_(True)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 32, 32, generator=g).to(dev, BF)
    ehs = torch.randn(2, 77, ocfg.cross_attention_dim, generator=g).to(dev, BF)
    added = {"text_embeds": torch.randn(2, 128, generator=g).to(dev, BF),
             "time_ids": torch.tensor([[256., 256., 0., 0., 256., 256.]] * 2, device=dev)}
    goal = torch.randn(2, 4, 32, 32, generator=g).to(dev)
    net.set_lora_slider(0.5)
    with net:
        pred = pm(x, 321, encoder_hidden_states=ehs, added_cond_kwargs=added).sample
    assert pred.requires_grad
    torch.nn.functional.mse_loss(pred.float(), goal).backward()
    torch.cuda.synchronize()

    def call(fp):
        out = torch.func.functional_call(om, fp, (x.float(), 321, ehs.float()),
                                         {"added_cond_kwargs": {k: v.float() for k, v in added.items()}}).sample
        assert rel_rms(pred, out) < 3e-2
        return torch.nn.functional.mse_loss(out, goal)

    leaves = _oracle_lora_grads(om, net, 0.5, call)
    num = den = 0.0
    for l in net.unet_loras:
        for got, ref in ((l.lora_down.weight.grad, leaves[l.lora_name][0].grad),
                         (l.lora_up.weight.grad, leaves[l.lora_name][1].grad)):
            assert got is not None and torch.isfinite(got).all(), l.lora_name
            num += (got.float() - ref).pow(2).sum().item()
            den += ref.pow(2).sum().item()
    assert (num / den) ** 0.5 < 5e-2, (method, (num / den) ** 0.5)
    if method != "selfattn":
        assert any("attn2_to_k" in l.lora_name for l in net.unet_loras)


@pytest.mark.parametrize("h,w", [(72, 88), (40, 104), (24, 36)])
def test_tiny_xl_bucket_resolutions_forward_and_gradients(dev, h, w):
    """`dynamic_resolution` draws latent sizes that are multiples of 8 but neither square nor powers of two
    (train_util.get_random_resolution_in_bucket: 64..120 for the 1024 bucket), and eval runs at e.g. 768x512: the
    3x3 convolutions tile such images in <= 128-pixel patches with TMA zero fill, the token counts (h*w, h*w/4, ...)
    are ragged for the attention tiles.  Forward and LoRA gradients against the fp32 oracle."""
    from oracle import unet as ounet
    from sliders_b200 import lora as plora, synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    ocfg = ounet.UNetConfig.tiny_xl()
    pm = UNet2DConditionModel(UNetConfig.from_dict(ocfg.__dict__))
    synthetic.init_synthetic_(pm, seed=31)
    om = ounet.UNet2DConditionModel(ocfg)
    pm = pm.to(dev, BF).eval().requires_grad_(False)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})  # the bf16-rounded weights
    om = om.to(dev).eval().requires_grad_(False)
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
    synthetic.init_lora_nonzero_(net, seed=32, up_std=0.05, reseed_down=True)
    net.requires_grad_(True)
    g = torch.Generator().manual_seed(h * 1000 + w)
    x = torch.randn(2, 4, h, w, generator=g).to(dev, BF)
    ehs = torch.randn(2, 77, ocfg.cross_attention_dim, generator=g).to(dev, BF)
    added = {"text_embeds": torch.randn(2, 128, generator=g).to(dev, BF),
             "time_ids": torch.tensor([[8. * h, 8. * w, 0., 0., 8. * h, 8. * w]] * 2, device=dev)}
    goal = torch.randn(2, 4, h, w, generator=g).to(dev)
    net.set_lora_slider(1.0)
    with net:
        pred = pm(x, 321, encoder_hidden_states=ehs, added_cond_kwargs=added).sample
    assert pred.shape == (2, 4, h, w) and pred.requires_grad
    torch.nn.functional.mse_loss(pred.float(), goal).backward()
    torch.cuda.synchronize()

    def call(fp):
        out = torch.func.functional_call(om, fp, (x.float(), 321, ehs.float()),
                                         {"added_cond_kwargs": {k: v.float() for k, v in added.items()}}).sample
        assert rel_rms(pred, out) < 3e-2
        return torch.nn.functional.mse_loss(out, goal)

    leaves = _oracle_lora_grads(om, net, 1.0, call)
    num = den = 0.0
    for l in net.unet_loras:
        for got, ref in ((l.lora_down.weight.grad, leaves[l.lora_name][0].grad),
                         (l.lora_up.weight.grad, leaves[l.lora_name][1].grad)):
            assert got is not None and torch.isfinite(got).all(), l.lora_name
            num += (got.float() - ref).pow(2).sum().item()
            den += ref.pow(2).sum().item()
    assert (num / den) ** 0.5 < 5e-2, ((h, w), (num / den) ** 0.5)


def test_full_size_inference_sweep_properties(dev):
    """BASELINE config 5 at full size: SDXL, 1024 px, 16 samples (32 conditioned passes per step), DDIM, the slider
    sweep of eval-scripts/generate_images_xl.py:495-508 under CUDA-graph replay — checked through size-independent
    properties (the fp32 oracle needs minutes per step at this size): (1) slider 0 == adaptors never applied, bit for
    bit; (2) with start_noise below every timestep the adaptors are gated off for any scale (generate_images_xl.py:
    327-330), bit for bit; (3) replays are deterministic; (4) +s and -s move the result in opposite directions."""
    from sliders_b200 import generate, lora as plora, synthetic
    from sliders_b200.scheduler import create_noise_scheduler
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    with torch.device(dev):
        pm = UNet2DConditionModel(UNetConfig.sdxl()).to(BF)
    synthetic.init_synthetic_(pm, seed=1)
    pm.requires_grad_(False)
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
    synthetic.init_lora_nonzero_(net, seed=2, up_std=0.02)
    pm.use_cuda_graph = True
    n, steps = 16, 3
    g = torch.Generator().manual_seed(5)
    lat = torch.randn(n, 4, 128, 128, generator=g).to(dev, BF)
    ehs = torch.randn(2 * n, 77, 2048, generator=g).to(dev, BF)
    pooled = torch.randn(2 * n, 1280, generator=g).to(dev, BF)
    tids = torch.tensor([[1024., 1024., 0., 0., 1024., 1024.]] * (2 * n), device=dev)
    sched = create_noise_scheduler("ddim")
    run = lambda scale, start_noise: generate.denoise_loop(pm, net, sched, lat.clone(), ehs, pooled, tids,
                                                           num_inference_steps=steps, guidance_scale=5.0, scale=scale,
                                                           start_noise=start_noise)
    base = run(0.0, 1000)
    assert torch.isfinite(base).all() and base.shape == lat.shape
    assert torch.equal(run(3.0, -1), base)          # gated off at every step
    pos, pos2, neg = run(3.0, 1000), run(3.0, 1000), run(-3.0, 1000)
    assert torch.equal(pos, pos2)
    assert not torch.equal(pos, base)
    d_pos, d_neg = (pos - base).float().flatten(), (neg - base).float().flatten()
    assert torch.nn.functional.cosine_similarity(d_pos, d_neg, dim=0) < -0.5
    net.__exit__(None, None, None)
    with torch.no_grad():  # adaptors inert outside `with network:`; same graph-replayed loop without LoRA at all
        off = generate.denoise_loop(pm, net, sched, lat.clone(), ehs, pooled, tids, num_inference_steps=steps,
                                    guidance_scale=5.0, scale=0.0, start_noise=1000)
    assert torch.equal(off, base)


def test_full_sd15_lora_gradients_vs_fp32_oracle(dev):
    """BASELINE configs 1-2 (SD-1.x text slider, rank 4, 512 px): one grad-carrying `predict_noise` (train_lora.py:
    263-275) + MSE loss; LoRA gradients of all 150 adaptors vs the fp32 oracle's autograd.  Exercises the
    attention backward at head dims 40 / 80 / 160 and the 8x8 bottleneck."""
    from oracle import unet as ounet
    from sliders_b200 import lora as plora, synthetic, train_util
    from sliders_b200.scheduler import create_noise_scheduler
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    with torch.device(dev):
        pm = UNet2DConditionModel(UNetConfig.sd15()).to(BF)
        om = ounet.UNet2DConditionModel(ounet.UNetConfig.sd15())
    synthetic.init_synthetic_(pm, seed=5)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om.eval().requires_grad_(False)
    pm.requires_grad_(False)
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
    assert len(net.unet_loras) == 150
    synthetic.init_lora_nonzero_(net, seed=6, up_std=0.05)
    net.requires_grad_(True)
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(1, 4, 64, 64, generator=g).to(dev, BF)
    ehs = torch.randn(2, 77, 768, generator=g).to(dev, BF)
    goal = torch.randn(1, 4, 64, 64, generator=g).to(dev)
    sched = create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    with net:
        pred = train_util.predict_noise(pm, sched, 321, lat, ehs, guidance_scale=1.0)
    torch.nn.functional.mse_loss(pred.float(), goal).backward()
    torch.cuda.synchronize()

    def call(fp):
        out = torch.func.functional_call(om, fp, (torch.cat([lat.float()] * 2), 321, ehs.float())).sample
        u, c = out.chunk(2)
        ref = u + 1.0 * (c - u)
        assert rel_rms(pred, ref) < 2.5e-2
        return torch.nn.functional.mse_loss(ref, goal)

    leaves = _oracle_lora_grads(om, net, 1.0, call)
    num = den = 0.0
    for l in net.unet_loras:
        for got, ref in ((l.lora_down.weight.grad, leaves[l.lora_name][0].grad),
                         (l.lora_up.weight.grad, leaves[l.lora_name][1].grad)):
            assert got is not None and torch.isfinite(got).all(), l.lora_name
            num += (got.float() - ref).pow(2).sum().item()
            den += ref.pow(2).sum().item()
    total = (num / den) ** 0.5
    print(f"SD1.5 LoRA gradient rel-RMS vs fp32 oracle: {total:.4f}")
    assert total < 6e-2, total


def test_euler_denoise_loop_matches_oracle(dev):
    """The eval loop of generate_images_xl.py:325-364 with the scheduler the SDXL pipeline ships (EulerDiscrete, leading
    spacing, offset 1): 5 steps, guidance 5, slider 1.5 on the tiny SDXL-topology model vs the fp32 oracle UNet driven
    by oracle/euler.py; the guidance + Euler update runs in the affine mode of `cfg_ddim_kernel`."""
    import copy

    from oracle import euler as oeuler
    from oracle import unet as ounet
    from sliders_b200 import generate, synthetic
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    om = ounet.UNet2DConditionModel(ounet.UNetConfig.tiny_xl())
    synthetic.init_synthetic_(om, seed=fx["weight_seed"])
    om.eval()
    slider = 1.5
    mods = {("lora_unet_" + n.replace(".", "_")): m for n, m in om.named_modules()}
    sd = {k: v.float().cpu() for k, v in net.state_dict().items()}
    with torch.no_grad():
        for l in net.unet_loras:
            up, down = sd[l.lora_name + ".lora_up.weight"], sd[l.lora_name + ".lora_down.weight"]
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down) if down.dim() == 4 else up @ down
            mods[l.lora_name].weight.add_(delta * (slider * l.scale))
    steps, gs = 5, 5.0
    sch = oeuler.EulerDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                                        timestep_spacing="leading", steps_offset=1)
    sch.set_timesteps(steps)
    g = torch.Generator().manual_seed(11)
    lat = torch.randn(2, 4, 32, 32, generator=g) * float(sch.init_noise_sigma)
    ehs = fx["text_embeddings"].repeat_interleave(2, dim=0)
    pooled = fx["add_text_embeddings"].repeat_interleave(2, dim=0)
    tids = fx["add_time_ids"].repeat_interleave(2, dim=0)
    x = lat.clone()
    with torch.no_grad():
        for t in sch.timesteps:
            xin = sch.scale_model_input(torch.cat([x] * 2), float(t))
            out = om(xin, float(t), ehs, added_cond_kwargs={"text_embeds": pooled, "time_ids": tids}).sample
            u, c = out.chunk(2)
            x = sch.step(u + gs * (c - u), float(t), x).prev_sample
    psch = create_noise_scheduler("euler")
    psch.set_timesteps(steps)  # init_noise_sigma refers to the current sigma grid (the pipeline sets timesteps first)
    assert abs(float(psch.init_noise_sigma) - float(sch.init_noise_sigma)) < 1e-3, (psch.init_noise_sigma, sch.init_noise_sigma)
    got = generate.denoise_loop(pm, net, psch, lat.to(dev), ehs.to(dev), pooled.to(dev), tids.to(dev),
                                num_inference_steps=steps, guidance_scale=gs, scale=slider, start_noise=1000)
    r = rel_rms(got, x)
    print(f"euler loop rel-RMS {r:.4f}")
    assert r < 6e-2, r  # five guided steps (g = 5) accumulate the per-step bf16 error
    # scheduler.step alone on device tensors == the host formula
    e = torch.randn(2, 4, 32, 32, generator=g)
    t0 = psch.timesteps_host[1]
    dev_step = psch.step(e.to(dev), t0, lat.to(dev)).prev_sample
    r2 = rel_rms(dev_step, sch.step(e, t0, lat).prev_sample)
    assert r2 < 1e-5, r2
