"""GPU tests of per-sample LoRA scales (sb200_lora.sample_scale / rows_per_sample): every fused LoRA consumer element
by element against float64 with a per-row factor, the exact identities (an all-ones vector, a constant vector against
the scalar slider, graph replay with a new vector), the UNet against the fp32 oracle one sample at a time, the batched
scale sweep against the sequential one, and the refusals."""
import os

import pytest
import torch

import test_gpu_forward_bounds as fb
import test_gpu_kernels as gk
from test_gpu_kernels import (PAIR, SINGLE, assert_guard_intact, assert_within_bound, epilogue_ref, gemm_case,
                              guarded_out, run_conv, run_gemm)
from test_gpu_lora_ranks import make_lora, rank16  # noqa: F401  (fixture re-export)
from test_gpu_unet import GOLDEN, build_product, dev, rel_rms  # noqa: F401  (fixture re-export)

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def sample_vector(n, dev, seed=0):
    """n per-sample factors with zeros, negatives and magnitudes from 1e-2 to 7."""
    base = torch.tensor([0.0, -1.5, 2.0, 0.25, -3e-2, 7.0, 1.0, -0.5], dtype=torch.float64)
    i = torch.arange(n)
    v = base[(i + seed) % 8] * (1.0 + 0.125 * (i // 8))
    return v.float().to(dev)


def with_vector(la, vec, rows_per_sample):
    from sliders_b200 import ops

    return ops.Lora(la.down, la.up, la.r, la.group_n, la.scale, scale_dev=la.scale_dev, sample_scale=vec,
                    rows_per_sample=rows_per_sample)


def gemm_reference_rows(c, fac):
    """gk.gemm_reference with LoRA row m scaled by c.scale * fac[m] (fac float64 [M])."""
    def product(f):
        xd = f(c.x)
        y = xd @ f(c.w).t()
        gk._lora_add(y, xd @ f(c.down).t(), f(c.up), c.r, c.group_n, f(c.scale * fac[:, None]))
        return y

    rb = c.rowbias[torch.arange(c.M, device=c.w.device) // c.rpb] if c.rowbias is not None else None
    return epilogue_ref(product, bias=c.bias, rowbias=rb, resid=c.resid, geglu=c.geglu)


def conv_reference_images(c, fac):
    """gk.conv_reference with the LoRA term of image b scaled by c.scale * fac[b]."""
    import torch.nn.functional as F

    def product(f):
        xn = f(c.x).permute(0, 3, 1, 2)
        y = F.conv2d(xn, f(c.w).permute(0, 3, 1, 2), stride=c.stride, padding=1).permute(0, 2, 3, 1).contiguous()
        dn = f(c.down).view(-1, 3, 3, c.Cin).permute(0, 3, 1, 2)
        t = F.conv2d(xn, dn, stride=c.stride, padding=1).permute(0, 2, 3, 1)
        gk._lora_add(y, t, f(c.up), c.r, c.group_n, f(c.scale * fac[:, None, None, None]))
        return y

    rb = c.rowbias[:, None, None, :] if c.rowbias is not None else None
    return epilogue_ref(product, bias=c.bias, rowbias=rb, resid=c.resid)


# (M, N, K), flags, lora (rank, group_n, scale), bn | ctas, rows_per_sample.  Sample boundaries fall inside the
# 128-row tiles wherever rows_per_sample is not a multiple of 128.
GEMM_ROWS = [
    ((616, 960, 320), "bL", (4, 320, 1.0), 64 | SINGLE, 77),        # fused q|k|v on the text context, rt 16
    ((616, 1280, 640), "bRL", (8, 640, -0.5), 128 | SINGLE, 77),    # rank 8, two adaptors
    ((600, 960, 320), "L", (16, 320, 1.0), 64 | SINGLE, 100),       # rank-16 q|k|v: rt = 64
    ((600, 960, 320), "RL", (16, 320, 0.5), 128 | PAIR, 100),       # rt = 64 on 128-wide CTA pairs
    ((1000, 1280, 1280), "bRL", (16, 1280, -1.0), 128 | PAIR, 200),
    ((616, 2560, 640), "L", (16, 1280, 1.0), 64 | PAIR, 77),        # rt = 32
    ((256, 640, 640), "tL", (8, 640, 2.0), 64 | SINGLE, 1),         # one factor per row
    ((8192, 640, 320), "RL", (4, 320, 0.5), 64 | SINGLE, 1024),     # two CTAs per SM (grid > 2 x 132)
    ((1232, 3840, 1280), "L", (4, 1280, 1.0), 256 | SINGLE, 77),    # gemm_wide_kernel, rank 4
    ((1200, 1280, 640), "bRL", (8, 1280, -0.5), 256 | SINGLE, 100), # gemm_wide_kernel, rank 8
    ((600, 3840, 640), "L", (8, 1280, 1.0), 256 | SINGLE, 1),       # gemm_wide_kernel, rt = 32
]


def _gid(row):
    shape, flags, lora, force, rps = row
    bn, ctas = gk.decode_force(force)
    return f"bn{bn}-ctas{ctas}-r{lora[0]}-" + "x".join(map(str, shape)) + f"-{flags}-rps{rps}"


@pytest.mark.parametrize("shape,flags,lora,force,rps", GEMM_ROWS, ids=[_gid(r) for r in GEMM_ROWS])
def test_gemm_sample_scale(dev, rank16, shape, flags, lora, force, rps):
    M, N, K = shape
    c = gemm_case(M, N, K, flags, lora, dev, M + N + K)
    vec = sample_vector(M // rps, dev, seed=M)
    la = with_vector(c.la, vec, rps)
    buf, out = guarded_out(M, c.nout, dev)
    run_gemm(c, force, out=out, lora=la)
    torch.cuda.synchronize()
    assert_guard_intact(buf, M, c.nout)
    fac = vec.double()[torch.arange(M, device=dev) // rps]
    assert_within_bound(out, *gemm_reference_rows(c, fac))
    # an all-ones vector is the same launch without one, bit for bit
    ones = run_gemm(c, force, lora=with_vector(c.la, torch.ones(M // rps, device=dev), rps))
    assert torch.equal(ones, run_gemm(c, force))


# (B, H, W, C0, C1, Cout, stride), flags, lora, bn | ctas; rows_per_sample = Ho * Wo
CONV_ROWS = [
    ((4, 16, 16, 128, 0, 320, 1), "btL", (4, 320, 0.5), 64 | SINGLE),
    ((3, 32, 32, 64, 0, 320, 2), "bL", (8, 320, 1.0), 128 | SINGLE),      # stride 2
    ((2, 16, 16, 128, 64, 640, 1), "bRL", (16, 640, -0.5), 128 | SINGLE), # skip concat, rank 16
    ((3, 10, 10, 64, 0, 256, 1), "bL", (4, 256, 1.0), 256 | SINGLE),      # gemm_wide_kernel, Ho * Wo = 100
    ((5, 20, 12, 64, 0, 512, 2), "L", (8, 512, 2.0), 256 | SINGLE),       # wide, stride 2, Ho * Wo = 60
]


@pytest.mark.parametrize("shape,flags,lora,force", CONV_ROWS)
def test_conv_sample_scale(dev, rank16, shape, flags, lora, force):
    B, H, W, C0, C1, Cout, stride = shape
    c = gk.conv_case(B, H, W, C0, C1, Cout, stride, flags, lora, dev, B * H + Cout)
    rps = c.Ho * c.Wo
    vec = sample_vector(B, dev, seed=H)
    la = with_vector(c.la, vec, rps)
    buf, out2 = guarded_out(B * rps, Cout, dev)
    out = run_conv(c, force, out=out2.view(B, c.Ho, c.Wo, Cout), lora=la)
    torch.cuda.synchronize()
    assert_guard_intact(buf, B * rps, Cout)
    assert_within_bound(out, *conv_reference_images(c, vec.double()))
    ones = run_conv(c, force, lora=with_vector(c.la, torch.ones(B, device=dev), rps))
    assert torch.equal(ones, run_conv(c, force))


@pytest.mark.parametrize("M,N,K,act_out,lora,resid,rps", [
    (10, 1280, 1280, 0, (4, 1280, 0.5), False, 1),     # time_emb_proj under c3lier: one factor per batch entry
    (8, 40, 1280, 2, (8, 20, -0.75), True, 2),          # two groups, act_out 2, two rows per factor
    (64, 320, 320, 1, (16, 320, 2.0), True, 1),
])
def test_small_linear_sample_scale(dev, rank16, M, N, K, act_out, lora, resid, rps):
    x, w, b, res, la, lref = fb._sl_case(dev, M, N, K, 0, True, lora, resid, M + N)
    vec = sample_vector(M // rps, dev, seed=N)
    out = fb.run_small_linear(x, w, b, True, act_out, with_vector(la, vec, rps), res)
    fac = vec.double()[torch.arange(M, device=dev) // rps][:, None]
    ref, abs_ = fb.small_linear_ref(x, w, b, True, act_out, lref, lora[2] * fac, res)
    fb.assert_no_violations(fb.small_linear_violations(out, ref, abs_), out, ref, "small_linear sample_scale")
    ones = fb.run_small_linear(x, w, b, True, act_out, with_vector(la, torch.ones(M // rps, device=dev), rps), res)
    assert torch.equal(ones, fb.run_small_linear(x, w, b, True, act_out, la, res))


@pytest.mark.parametrize("rps", [-77, 5])
def test_bad_rows_per_sample_is_refused_without_a_launch(dev, rps):
    """SB200_ERR_INVALID before any launch: the guarded output stays untouched."""
    from sliders_b200 import _cabi, ops

    c = gemm_case(616, 640, 640, "L", (4, 640, 1.0), dev, 3)
    vec = torch.ones(8, device=dev)
    la = ops.Lora(c.down, c.up, c.r, c.group_n, 1.0, sample_scale=vec, rows_per_sample=rps)
    buf, out = guarded_out(616, 640, dev)
    with pytest.raises(_cabi.Sb200Error, match="status -1"):
        ops.gemm(c.x, c.w, lora=la, out=out)
    cc = gk.conv_case(2, 8, 8, 64, 0, 64, 1, "L", (4, 64, 1.0), dev, 4)
    with pytest.raises(_cabi.Sb200Error, match="status -1"):
        ops.conv3x3(cc.x0, cc.w, lora=ops.Lora(cc.down, cc.up, 4, 64, 1.0, sample_scale=vec, rows_per_sample=rps))
    x, w, b, _, sl, _ = fb._sl_case(dev, 6, 64, 64, 0, False, (4, 64, 1.0), False, 5)
    with pytest.raises(_cabi.Sb200Error, match="status -1"):
        ops.small_linear(x, w, b, lora=ops.Lora(sl.down, sl.up, 4, 64, 1.0, sample_scale=vec, rows_per_sample=rps))
    torch.cuda.synchronize()
    assert (buf.view(torch.int16) == gk.NAN_BITS).all(), "a refused launch wrote to its output"


def test_zero_rows_per_sample_is_refused(dev):
    """rows_per_sample 0 through the C ABI (ops derives it from the call instead, and refuses a vector whose length
    does not divide the rows)."""
    from sliders_b200 import _cabi, ops

    x, w, b, _, sl, _ = fb._sl_case(dev, 6, 64, 64, 0, False, (4, 64, 1.0), False, 5)
    la = ops.Lora(sl.down, sl.up, 4, 64, 1.0, sample_scale=torch.ones(3, device=dev))
    _, o = guarded_out(6, 64, dev)
    lib = _cabi.load()
    status = lib.sb200_small_linear(ops._ctx(x), ops._stream(), ops._p(x), x.stride(0), ops._p(w), w.stride(0),
                                    ops._p(b), ops._p(o), o.stride(0), 6, 64, 64, 0, 0, la.ref(), None)
    assert status == -1
    torch.cuda.synchronize()
    assert (o.view(torch.int16) == gk.NAN_BITS).all(), "a refused launch wrote to its output"
    with pytest.raises(ValueError, match="do not divide"):
        ops.small_linear(x, w, b, lora=ops.Lora(sl.down, sl.up, 4, 64, 1.0, sample_scale=torch.ones(4, device=dev)))


# ------------------------------------------------------------------------------------------------------------------
# UNet
# ------------------------------------------------------------------------------------------------------------------
def _inputs(fx, dev, B, h, w, seed):
    from oracle import unet as ounet

    cfg = getattr(ounet.UNetConfig, fx["config"])()
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, h, w, generator=g).to(dev, BF)
    ehs = torch.randn(B, 77, cfg.cross_attention_dim, generator=g).to(dev, BF)
    added = None
    if cfg.addition_embed_type == "text_time":
        added = {"text_embeds": torch.randn(B, 128, generator=g).to(dev, BF),
                 "time_ids": torch.tensor([[8. * h, 8. * w, 0., 0., 8. * h, 8. * w]] * B, device=dev)}
    return cfg, x, ehs, added


@pytest.mark.parametrize("config,h,w", [("tiny_xl", 32, 32), ("tiny_xl", 24, 36), ("tiny_sd", 32, 32)])
def test_unet_per_sample_scales_vs_oracle(dev, config, h, w):
    """A batch of 3 samples at 3 slider values against the fp32 oracle run one sample at a time with the slider folded
    into its weights (test_gpu_unet's bound for the same quantity: rel-RMS 2.5e-2 on eps)."""
    from oracle import unet as ounet

    fx = torch.load(os.path.join(GOLDEN, f"{config}.pt"))
    pm, net = build_product(fx, dev)
    scales = (-2.0, 0.5, 1.5)
    cfg, x, ehs, added = _inputs(fx, dev, 3, h, w, 7)
    om = ounet.UNet2DConditionModel(cfg)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om = om.to(dev).eval().requires_grad_(False)
    names = {"lora_unet_" + n.replace(".", "_"): n for n, _ in om.named_modules()}
    params = dict(om.named_parameters())
    net.set_lora_slider(list(scales))
    with torch.no_grad(), net:
        got = pm(x, 321, encoder_hidden_states=ehs, added_cond_kwargs=added).sample
    for i, s in enumerate(scales):
        eff = {}
        for l in net.unet_loras:
            down, up = l.lora_down.weight.detach().float(), l.lora_up.weight.detach().float()
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down) if down.dim() == 4 else up @ down
            key = names[l.lora_name] + ".weight"
            eff[key] = params[key] + s * l.scale * delta
        kw = {}
        if added is not None:
            kw["added_cond_kwargs"] = {k: v[i:i + 1].float() for k, v in added.items()}
        with torch.no_grad():
            ref = torch.func.functional_call(om, {**params, **eff}, (x[i:i + 1].float(), 321, ehs[i:i + 1].float()),
                                             kw).sample
        assert rel_rms(got[i:i + 1], ref) < 2.5e-2, (config, s, rel_rms(got[i:i + 1], ref))


def test_unet_per_sample_identities(dev):
    """Bit-exact: a constant vector == the scalar slider at the same batch (the vector holds fp32(value * alpha / r),
    the fp32 factor the scalar path passes, so the products are formed identically); an all-zero vector == adaptors
    off; a graph replay with new values == an eager call with them; n values tile the batch as scale[b % n]."""
    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    _, x, ehs, added = _inputs(fx, dev, 4, 32, 32, 11)

    def run(scale):
        net.set_lora_slider(scale)
        with torch.no_grad(), net:
            return pm(x, 321, encoder_hidden_states=ehs, added_cond_kwargs=added).sample

    assert torch.equal(run([1.5] * 4), run(1.5))
    assert torch.equal(run(torch.tensor([1.5, 1.5])), run(1.5))
    assert torch.equal(run([0.0, 0.0]), run(0.0))
    mixed = run([-1.0, 2.0])
    halves = run([-1.0, 2.0, -1.0, 2.0])
    assert torch.equal(mixed, halves)
    assert not torch.equal(mixed[0], mixed[1])
    pm.use_cuda_graph = True
    try:
        for vals in ([0.5, -2.0], [1.0, 3.0], [-1.0, 2.0]):
            graphed = run(vals)
            pm.use_cuda_graph = False
            eager = run(vals)
            pm.use_cuda_graph = True
            assert torch.equal(graphed, eager), vals
        assert torch.equal(run(1.5), run([1.5, 1.5]))      # the scalar graph and the per-sample graph side by side
    finally:
        pm.use_cuda_graph = False


def test_refusals(dev):
    from sliders_b200 import lora as plora, synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig
    from oracle import unet as ounet

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    _, x, ehs, added = _inputs(fx, dev, 4, 32, 32, 13)
    net.set_lora_slider([1.0, 2.0, 3.0])
    with torch.no_grad(), net, pytest.raises(ValueError, match="multiple"):
        pm(x, 321, encoder_hidden_states=ehs, added_cond_kwargs=added)
    # a gradient through a per-sample forward
    net.requires_grad_(True)
    net.set_lora_slider([1.0, 2.0])
    with net, pytest.raises(NotImplementedError, match="per-sample"):
        pm(x, 321, encoder_hidden_states=ehs, added_cond_kwargs=added).sample.float().sum().backward()
    net.requires_grad_(False)
    # a SliderStack takes no per-sample vector
    sm = UNet2DConditionModel(UNetConfig.from_dict(ounet.UNetConfig.tiny_xl().__dict__))
    synthetic.init_synthetic_(sm, seed=5)
    sm = sm.to(dev, BF)
    stack = plora.SliderStack(sm, [dict(rank=4), dict(rank=4)]).to(dev, BF)
    with pytest.raises(NotImplementedError, match="SliderStack"):
        stack.set_lora_slider([[1.0, 2.0], 0.5])
    with pytest.raises(NotImplementedError, match="SliderStack"):
        stack.sliders[0].set_lora_slider([1.0, 2.0])


# ------------------------------------------------------------------------------------------------------------------
# batched sweep
# ------------------------------------------------------------------------------------------------------------------
SCALES = (-2.0, -1.0, 0.0, 1.0, 2.0)


def _sweep_case(dev, N=2):
    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    pm.use_cuda_graph = True
    g = torch.Generator().manual_seed(21)
    pe = torch.randn(2 * N, 77, 256, generator=g).to(dev, BF)
    ae = torch.randn(2 * N, 128, generator=g).to(dev, BF)
    ids = torch.tensor([[256., 256, 0, 0, 256, 256]], device=dev).repeat(2 * N, 1)
    lat = torch.randn(N, 4, 32, 32, generator=g).to(dev, BF)
    return pm, net, pe, ae, ids, lat


def _sequential(pm, net, sched, lat, pe, ae, ids, steps, start_noise, seed):
    from sliders_b200 import generate

    out = []
    for s in SCALES:
        gen = torch.Generator(device=lat.device).manual_seed(seed) if seed is not None else None
        out.append(generate.denoise_loop(pm, net, sched, lat.clone(), pe, ae, ids, num_inference_steps=steps,
                                         guidance_scale=5.0, scale=s, start_noise=start_noise, generator=gen))
    return out


# Bound on the final latents, batched vs sequential.  The two runs differ only in GroupNorm's summation order (its
# chunk count depends on the batch): a last-bit difference per statistic, which the remaining steps carry through the
# network.  Measured on an H100 80GB HBM3 at 700 W: 0 for this tiny model at K = 2 and 3 (its reductions happen to sum
# in the same order at these batches), 4.5e-3 for a full SDXL sweep after 38 batched Euler steps
# (tools/gpu_time_sweep.py).  3e-3 allows for that drift on the tiny model and stays below half the distance between
# neighbouring scales here (>= 5.9e-3), and a scale run at the wrong value would also sit closer to another scale's
# sequential run than to its own, which the test rules out separately.
SWEEP_BOUND = 3e-3


@pytest.mark.parametrize("kind", ["ddim", "euler", "euler_a"])
@pytest.mark.parametrize("K", [2, 3])
def test_batched_sweep_matches_sequential(dev, kind, K):
    from sliders_b200 import generate
    from sliders_b200.scheduler import create_noise_scheduler

    pm, net, pe, ae, ids, lat = _sweep_case(dev)
    sched = create_noise_scheduler(kind)
    steps, start_noise = 8, 600
    P = generate.shared_prefix_steps(sched, steps, start_noise)
    assert 0 < P < steps
    seed = 5 if kind == "euler_a" else None
    seq = _sequential(pm, net, sched, lat, pe, ae, ids, steps, start_noise, seed)
    gen = torch.Generator(device=dev).manual_seed(5) if seed is not None else None
    bat = generate.scale_sweep(pm, net, sched, lat.clone(), pe, ae, ids, scales=SCALES, scales_per_batch=K,
                               num_inference_steps=steps, guidance_scale=5.0, start_noise=start_noise, generator=gen)
    assert len(bat) == len(SCALES)
    for i, (s, a, b) in enumerate(zip(SCALES, seq, bat)):
        assert b.shape == a.shape and b.dtype == a.dtype
        err = rel_rms(b, a)
        others = [rel_rms(b, o) for j, o in enumerate(seq) if j != i]
        print(f"{kind} K={K} scale {s}: rel-RMS {err:.3g} to its sequential run, >= {min(others):.3g} to the others")
        assert err < SWEEP_BOUND and err < min(others), (kind, K, s, err, others)
    # every step before start_noise: the whole loop is the shared part, bit for bit the sequential run's
    seq_p = _sequential(pm, net, sched, lat, pe, ae, ids, steps, -1, seed)
    gen = torch.Generator(device=dev).manual_seed(5) if seed is not None else None
    bat_p = generate.scale_sweep(pm, net, sched, lat.clone(), pe, ae, ids, scales=SCALES, scales_per_batch=K,
                                 num_inference_steps=steps, guidance_scale=5.0, start_noise=-1, generator=gen)
    for a, b in zip(seq_p, bat_p):
        assert torch.equal(a, b)


def test_batched_sweep_prefix_is_bit_identical(dev):
    """The shared steps run at the sequential batch: the latents after them equal the sequential run's at that step."""
    from sliders_b200 import generate
    from sliders_b200.scheduler import create_noise_scheduler

    pm, net, pe, ae, ids, lat = _sweep_case(dev)
    sched = create_noise_scheduler("euler")
    steps, start_noise = 8, 600
    P = generate.shared_prefix_steps(sched, steps, start_noise)
    seen = {}
    generate.denoise_loop(pm, net, sched, lat.clone(), pe, ae, ids, num_inference_steps=steps, guidance_scale=5.0,
                          scale=2.0, start_noise=start_noise, callback=lambda i, t, x: seen.setdefault(i, x.clone()))
    sched.set_timesteps(steps, device=dev)
    got = generate._run_steps(pm, net, sched, lat.clone(), pe, {"text_embeds": ae, "time_ids": ids},
                              generate._host_steps(sched)[:P], 0, guidance_scale=5.0, scale=0.0,
                              start_noise=start_noise)
    assert torch.equal(got, seen[P - 1])


def test_eval_sweep_batched_same_tree(dev, tmp_path):
    from sliders_b200 import eval_sweep as es

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    pm.use_cuda_graph = True
    csv_path = tmp_path / "p.csv"
    csv_path.write_text("case_number,prompt,evaluation_seed,concept\n3,a,11,x\n")
    rows = es.read_prompts_csv(str(csv_path))
    g = torch.Generator().manual_seed(0)
    table = {"a": (torch.randn(2, 77, 256, generator=g), torch.randn(2, 128, generator=g))}
    from sliders_b200.scheduler import create_noise_scheduler

    trees = {}
    for K in (1, 3):
        out_dir = tmp_path / f"out{K}"
        n = es.sweep(pm, net, create_noise_scheduler("euler"), rows, lambda p: table[p], str(out_dir),
                     num_samples=2, num_inference_steps=6, guidance_scale=5.0, start_noise=500, image_size=256,
                     scales_per_batch=K)
        assert n == 5 * 2
        trees[K] = sorted(str(p.relative_to(out_dir)) for p in out_dir.rglob("*") if p.is_file())
    assert trees[1] == trees[3] and len(trees[1]) == 10
    for f in trees[1]:
        a, b = torch.load(tmp_path / "out1" / f), torch.load(tmp_path / "out3" / f)
        assert rel_rms(b, a) < SWEEP_BOUND, f
