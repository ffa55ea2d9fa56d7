"""GPU tests of null-text inversion and the gradient w.r.t. encoder_hidden_states: the query-split cross-attention
dK / dV, the fp32 split-K context-gradient GEMM, the fused guided-step loss, fp32 Adam, the UNet's d_ehs against the
fp32 oracle's autograd, CUDA-graph vs eager, the out-of-scope errors, NullInversion's early stop and the edit sweep
with per-step unconditional embeddings.

Tolerances: attention backward rounds P and dS to bf16 -> rel-RMS 3e-2 (as tests/test_gpu_backward.py); the split-K
GEMM reads bf16 operands and accumulates in fp32 on the tensor cores (up to ~18 000 products per split) -> rel-RMS
1e-4 against fp64 on the same bf16 inputs (measured 3.5e-5 at K = 153 600; a bf16 output alone would cost 2e-3); the d_ehs of a
bf16 UNet against the fp32 oracle -> rel-RMS 5e-2 (the LoRA-gradient bar of tests/test_gpu_unet.py)."""
import pytest
import torch

from conftest import c3lier

pytestmark = pytest.mark.gpu

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
    return ((got - ref).norm() / (ref.norm() + 1e-30)).item()


# ---------------------------------------------------------------------------------------------------------------------
# 1. query-split cross-attention dK / dV
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Sq", [4096, 1024, 256])
@pytest.mark.parametrize("d,heads", [(40, 8), (64, 10), (80, 8), (160, 8)])
@pytest.mark.parametrize("B", [1, 2])
def test_split_cross_attention_bwd(dev, B, Sq, d, heads):
    from sliders_b200 import ops

    Skv = 77
    g = torch.Generator().manual_seed(Sq + d + B)
    Cc = heads * d
    q = torch.randn(B * Sq, Cc, generator=g).to(dev, BF)
    kv = torch.randn(B * Skv, 2 * Cc, generator=g).to(dev, BF)
    k, v = kv[:, :Cc], kv[:, Cc:]
    dout = torch.randn(B * Sq, Cc, generator=g).to(dev, BF)
    scale = d ** -0.5
    lse = torch.empty(B, heads, Sq, device=dev, dtype=torch.float32)
    o = ops.attention(q, k, v, B, heads, Sq, Skv, scale, head_dim=d, lse=lse)
    assert ops.attn_bwd_splits(B, heads, Sq, Skv) > 1
    runs = []
    for _ in range(2):
        dq = torch.empty_like(q)
        dkv = torch.empty_like(kv)
        ops.attention_bwd_split(q, k, v, o, dout, lse, B, heads, Sq, Skv, scale, d, dq, dkv[:, :Cc], dkv[:, Cc:])
        runs.append((dq, dkv))
    dq0 = torch.empty_like(q)
    ops.attention_bwd(q, k, v, o, dout, lse, B, heads, Sq, Skv, scale, d, dq0)
    torch.cuda.synchronize()
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])  # bit-reproducible
    assert torch.equal(runs[0][0], dq0)  # dQ as from sb200_attention_bwd
    qf = q.float().reshape(B, Sq, heads, d).transpose(1, 2).requires_grad_()
    kf = k.float().reshape(B, Skv, heads, d).transpose(1, 2).requires_grad_()
    vf = v.float().reshape(B, Skv, heads, d).transpose(1, 2).requires_grad_()
    ref = (torch.softmax(qf @ kf.transpose(-1, -2) * scale, dim=-1) @ vf).transpose(1, 2).reshape(B * Sq, Cc)
    ref.backward(dout.float())
    back = lambda t, S: t.transpose(1, 2).reshape(B * S, Cc)
    dkv = runs[0][1]
    assert rel_rms(dkv[:, :Cc], back(kf.grad, Skv)) < 3e-2
    assert rel_rms(dkv[:, Cc:], back(vf.grad, Skv)) < 3e-2


# ---------------------------------------------------------------------------------------------------------------------
# 2. fp32 split-K GEMM
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,K", [(1, 768, 3200), (1, 768, 6400), (2, 768, 15360), (1, 768, 24960),
                                   (1, 2048, 12800), (2, 2048, 153600), (1, 2048, 166400)])
def test_gemm_splitk_f32(dev, B, N, K):
    from sliders_b200 import ops

    M = 77 * B
    g = torch.Generator().manual_seed(N + K + M)
    x = (0.1 * torch.randn(M, K, generator=g)).to(dev, BF)
    w = (0.02 * torch.randn(N, K, generator=g)).to(dev, BF)
    out = ops.gemm_splitk_f32(x, w)
    out2 = ops.gemm_splitk_f32(x, w)
    ref = x.double() @ w.double().t()
    torch.cuda.synchronize()
    assert out.dtype == torch.float32 and out.shape == (M, N)
    assert torch.equal(out, out2)
    assert rel_rms(out.double(), ref) < 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# 3. fused loss, fp32 Adam
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 4, 64, 64), (1, 4, 128, 128), (1, 4, 8, 8)])
def test_guided_step_loss(dev, shape):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(shape[-1])
    eu, ec, x, tg = (torch.randn(shape, generator=g).to(dev) for _ in range(4))
    gs, cx, ce = 7.5, 1.0137, -0.0421
    eu_ = eu.clone().requires_grad_()
    loss = ops.guided_step_loss(eu_, ec, gs, x, cx, ce, tg)
    (2.5 * loss).backward()
    ef = eu.double().requires_grad_()
    ref = torch.nn.functional.mse_loss(cx * x.double() + ce * (ef + gs * (ec.double() - ef)), tg.double())
    (2.5 * ref).backward()
    assert abs(loss.item() - ref.item()) / ref.item() < 1e-5
    assert rel_rms(eu_.grad.double(), ef.grad) < 1e-5
    assert torch.equal(ops.guided_step_loss(eu, ec, gs, x, cx, ce, tg), loss.detach())


def test_adam_f32_matches_torch(dev):
    """10 steps on a [1, 77, 768] fp32 parameter with the inversion's lr: max relative deviation of the parameters
    from torch.optim.Adam (foreach) <= 1e-6 of their scale (fp32 rounding order only)."""
    from sliders_b200 import optim

    g = torch.Generator().manual_seed(5)
    p0 = torch.randn(1, 77, 768, generator=g).to(dev)
    a, b = p0.clone().requires_grad_(), p0.clone().requires_grad_()
    oa = optim.Adam([a], lr=1e-2 * 0.97)
    ob = torch.optim.Adam([b], lr=1e-2 * 0.97)
    for i in range(10):
        grad = torch.randn(1, 77, 768, generator=g).to(dev) * (0.1 + i)
        a.grad, b.grad = grad.clone(), grad.clone()
        oa.step()
        ob.step()
    torch.cuda.synchronize()
    assert ((a - b).abs().max() / b.abs().max()).item() < 1e-6
    assert torch.allclose(oa.state[a]["exp_avg_sq"], ob.state[b]["exp_avg_sq"], rtol=1e-5, atol=0)


# ---------------------------------------------------------------------------------------------------------------------
# 4. gradient w.r.t. encoder_hidden_states
# ---------------------------------------------------------------------------------------------------------------------
def _models(cfg_name, seed, dev):
    from oracle import unet as ounet
    from sliders_b200 import synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    ocfg = getattr(ounet.UNetConfig, cfg_name)()
    pm = UNet2DConditionModel(UNetConfig.from_dict(ocfg.__dict__))
    synthetic.init_synthetic_(pm, seed=seed)
    pm = pm.to(dev, BF).eval().requires_grad_(False)
    om = ounet.UNet2DConditionModel(ocfg)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})  # the bf16-rounded weights
    om = om.to(dev).eval().requires_grad_(False)
    return ocfg, pm, om


def _network(pm, dev, method, seed, trainable):
    from sliders_b200 import lora as plora, synthetic

    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=2.0, train_method=method).to(dev, BF)
    synthetic.init_lora_nonzero_(net, seed=seed, up_std=0.05, reseed_down=True)
    net.requires_grad_(trainable)
    return net


def _oracle_params(om, net, slider):
    """fp32 oracle parameters with W_eff = W + s * scale * up @ down (the reference's forward hook as a weight fold),
    and the (down, up) leaves that carry the LoRA gradients."""
    names = {"lora_unet_" + n.replace(".", "_"): n for n, _ in om.named_modules()}
    params = dict(om.named_parameters())
    leaves, eff = {}, {}
    if net is not None:
        for l in net.unet_loras:
            down = l.lora_down.weight.detach().float().requires_grad_()
            up = l.lora_up.weight.detach().float().requires_grad_()
            leaves[l.lora_name] = (down, up)
            w = params[names[l.lora_name] + ".weight"]
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down) if down.dim() == 4 else up @ down
            eff[names[l.lora_name] + ".weight"] = w + slider * l.scale * delta
    return {**params, **eff}, leaves


@pytest.mark.parametrize("cfg_name", ["tiny_sd", "tiny_xl"])
@pytest.mark.parametrize("case", ["none", "frozen", "trainable"])
def test_ehs_gradient_vs_oracle(dev, cfg_name, case):
    """d loss / d encoder_hidden_states of the bf16 UNet vs the fp32 oracle's autograd: no adaptors, a frozen
    `noxattn` slider at multiplier 1.5, and a trainable one (LoRA gradients checked too)."""
    ocfg, pm, om = _models(cfg_name, 41, dev)
    net = None if case == "none" else _network(pm, dev, "noxattn", 42, case == "trainable")
    B = 2
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, 4, 32, 32, generator=g).to(dev)
    ehs0 = torch.randn(B, 77, ocfg.cross_attention_dim, generator=g).to(dev)
    goal = torch.randn(B, 4, 32, 32, generator=g).to(dev)
    kw, okw = {}, {}
    if cfg_name == "tiny_xl":
        added = {"text_embeds": torch.randn(B, 128, generator=g).to(dev),
                 "time_ids": torch.tensor([[256., 256., 0., 0., 256., 256.]] * B, device=dev)}
        kw, okw = {"added_cond_kwargs": added}, {"added_cond_kwargs": added}
    slider = 1.5
    ehs = ehs0.clone().requires_grad_()
    if net is not None:
        net.set_lora_slider(slider)
        with net:
            pred = pm(x, 321, encoder_hidden_states=ehs, **kw).sample
    else:
        pred = pm(x, 321, encoder_hidden_states=ehs, **kw).sample
    torch.nn.functional.mse_loss(pred.float(), goal).backward()
    torch.cuda.synchronize()
    assert ehs.grad is not None and ehs.grad.dtype == torch.float32 and ehs.grad.shape == ehs.shape

    params, leaves = _oracle_params(om, net, slider)
    oehs = ehs0.clone().requires_grad_()
    out = torch.func.functional_call(om, params, (x, 321, oehs), okw).sample
    assert rel_rms(pred, out) < 3e-2
    torch.nn.functional.mse_loss(out, goal).backward()
    err = rel_rms(ehs.grad, oehs.grad)
    print(f"{cfg_name} {case}: d_ehs rel-RMS vs fp32 oracle {err:.4f}")
    assert err < 5e-2
    if case == "trainable":
        num = den = 0.0
        for l in net.unet_loras:
            for got, ref in ((l.lora_down.weight.grad, leaves[l.lora_name][0].grad),
                             (l.lora_up.weight.grad, leaves[l.lora_name][1].grad)):
                assert got is not None and torch.isfinite(got).all(), l.lora_name
                num += (got.float() - ref).pow(2).sum().item()
                den += ref.pow(2).sum().item()
        assert (num / den) ** 0.5 < 5e-2


def test_ehs_gradient_full_sd15_vs_oracle(dev):
    """Full-size SD1.5 topology, 64x64 latents, batch 1, synthetic weights: d_ehs vs the fp32 oracle."""
    ocfg, pm, om = _models("sd15", 51, dev)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(1, 4, 64, 64, generator=g).to(dev)
    ehs0 = torch.randn(1, 77, 768, generator=g).to(dev)
    goal = torch.randn(1, 4, 64, 64, generator=g).to(dev)
    ehs = ehs0.clone().requires_grad_()
    pred = pm(x, 500, encoder_hidden_states=ehs).sample
    torch.nn.functional.mse_loss(pred, goal).backward()
    oehs = ehs0.clone().requires_grad_()
    torch.nn.functional.mse_loss(om(x, 500, oehs).sample, goal).backward()
    err = rel_rms(ehs.grad, oehs.grad)
    print(f"SD1.5 d_ehs rel-RMS vs fp32 oracle: {err:.4f}")
    assert err < 5e-2


def test_ehs_gradient_graph_equals_eager_and_zero_rows(dev):
    """CUDA-graph replay gives the eager bits; samples marked as receiving an exactly-zero gradient get d_ehs = 0."""
    ocfg, pm, _ = _models("tiny_sd", 61, dev)
    net = _network(pm, dev, "noxattn", 62, False)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 4, 32, 32, generator=g).to(dev)
    ehs0 = torch.randn(2, 77, ocfg.cross_attention_dim, generator=g).to(dev)
    goal = torch.randn(2, 4, 32, 32, generator=g).to(dev)

    def run(graph, zero_rows=0, slider=True):
        pm.use_cuda_graph = graph
        ehs = ehs0.clone().requires_grad_()
        net.set_lora_slider(0.8)
        if slider:
            with net:
                pred = pm(x, 400, encoder_hidden_states=ehs).sample
        else:  # no adaptor active: the null-text optimisation itself
            pred = pm(x, 400, encoder_hidden_states=ehs).sample
        if zero_rows:
            pred.grad_fn.zero_rows = zero_rows
        torch.nn.functional.mse_loss(pred[zero_rows:], goal[zero_rows:]).backward()
        torch.cuda.synchronize()
        return pred.detach(), ehs.grad

    try:
        e_out, e_g = run(False)
        for _ in range(2):  # capture, then replay
            g_out, g_g = run(True)
            assert torch.equal(e_out, g_out) and torch.equal(e_g, g_g)
        z_e = run(False, zero_rows=1)[1]
        z_g = run(True, zero_rows=1)[1]
        n_e = run(False, slider=False)
        for _ in range(2):
            n_g = run(True, slider=False)
            assert torch.equal(n_e[0], n_g[0]) and torch.equal(n_e[1], n_g[1])
    finally:
        pm.use_cuda_graph = False
    assert torch.equal(z_e, z_g)
    assert torch.count_nonzero(z_e[0]) == 0 and torch.count_nonzero(z_e[1]) > 0


def test_ehs_gradient_out_of_scope_raises(dev):
    ocfg, pm, _ = _models("tiny_xl", 71, dev)
    g = torch.Generator().manual_seed(10)
    x = torch.randn(1, 4, 32, 32, generator=g).to(dev)
    ehs = torch.randn(1, 77, ocfg.cross_attention_dim, generator=g).to(dev).requires_grad_()
    added = {"text_embeds": torch.randn(1, 128, generator=g).to(dev),
             "time_ids": torch.tensor([[256., 256., 0., 0., 256., 256.]], device=dev)}
    with pytest.raises(NotImplementedError, match="sample"):
        pm(x.clone().requires_grad_(), 300, encoder_hidden_states=ehs, added_cond_kwargs=added)
    with pytest.raises(NotImplementedError, match="text_embeds"):
        pm(x, 300, encoder_hidden_states=ehs,
           added_cond_kwargs={**added, "text_embeds": added["text_embeds"].clone().requires_grad_()})
    net = _network(pm, dev, "xattn", 72, False)
    net.set_lora_slider(1.0)
    with net:
        with pytest.raises(NotImplementedError, match="to_k"):
            pm(x, 300, encoder_hidden_states=ehs, added_cond_kwargs=added)


# ---------------------------------------------------------------------------------------------------------------------
# 6. early stop, 7. edit sweep
# ---------------------------------------------------------------------------------------------------------------------
def _inversion_setup(dev, steps):
    from sliders_b200.inversion import NullInversion
    from sliders_b200.scheduler import DDIMScheduler

    ocfg, pm, _ = _models("tiny_sd", 81, dev)
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          set_alpha_to_one=False)
    g = torch.Generator().manual_seed(11)
    lat = (0.8 * torch.randn(1, 4, 32, 32, generator=g)).to(dev)
    unc = torch.randn(1, 77, ocfg.cross_attention_dim, generator=g).to(dev)
    cond = torch.randn(1, 77, ocfg.cross_attention_dim, generator=g).to(dev)
    return pm, NullInversion(pm, sched, num_ddim_steps=steps), sched, lat, unc, cond


def test_null_inversion_early_stop_and_progress(dev):
    pm, inv, _, lat, unc, cond = _inversion_setup(dev, 4)
    x_t, ddim_latents, lst = inv.invert(lat, unc, cond, num_inner_steps=5, early_stop_epsilon=1e9)
    assert inv.unet_calls == 4 and all(len(l) == 1 for l in inv.losses)
    assert len(ddim_latents) == 5 and len(lst) == 4 and x_t is ddim_latents[-1]
    x_t, ddim_latents, lst = inv.invert(lat, unc, cond, num_inner_steps=5, early_stop_epsilon=0.0)
    assert inv.unet_calls == 20
    # Adam on the unconditional embedding lowers the reconstruction loss within every outer step
    assert sum(l[-1] < l[0] for l in inv.losses) >= 3
    assert all(e.shape == (1, 77, unc.shape[-1]) and e.dtype == torch.float32 for e in lst)


def test_denoise_loop_negative_embeds_per_step(dev):
    """The per-step unconditional embeddings through `denoise_loop` (graphed) equal the notebook's eager loop, and
    slider 0 equals no network bit for bit."""
    from sliders_b200 import generate, train_util
    from sliders_b200 import lora as plora

    pm, inv, sched, lat, unc, cond = _inversion_setup(dev, 4)
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
    from sliders_b200 import synthetic
    synthetic.init_lora_nonzero_(net, seed=3, up_std=0.05, reseed_down=True)
    net.requires_grad_(False)
    g = torch.Generator().manual_seed(12)
    negs = [unc + 0.1 * i * torch.randn(unc.shape, generator=g).to(dev) for i in range(4)]
    prompt = torch.cat([unc, cond])

    def ref_loop(scale, unet=pm, network=net):
        sched.set_timesteps(4)
        x = lat.clone()
        for i, t in enumerate(sched.timesteps_host):
            emb = torch.cat([negs[i], cond])
            with torch.no_grad():
                if network is None:
                    eps = unet(torch.cat([x] * 2), t, encoder_hidden_states=emb).sample
                else:
                    network.set_lora_slider(scale=0 if t > 500 else scale)
                    with network:
                        eps = unet(torch.cat([x] * 2), t, encoder_hidden_states=emb).sample
            x = train_util.guided_step(sched, eps, t, x, 7.5)
        return x

    try:
        pm.use_cuda_graph = True
        got = generate.denoise_loop(pm, net, sched, lat.clone(), prompt, num_inference_steps=4, guidance_scale=7.5,
                                    scale=2.0, start_noise=500, negative_embeds_per_step=negs)
        n_graphs = len(pm._graphs)
        got0 = generate.denoise_loop(pm, net, sched, lat.clone(), prompt, num_inference_steps=4, guidance_scale=7.5,
                                     scale=0.0, start_noise=500, negative_embeds_per_step=negs)
        assert len(pm._graphs) == n_graphs  # no capture per step or per embedding
    finally:
        pm.use_cuda_graph = False
    assert torch.equal(got, ref_loop(2.0))
    assert not torch.equal(got, got0)
    bare = _inversion_setup(dev, 4)[0]  # the same seeded weights, no network injected
    assert torch.equal(got0, ref_loop(0.0, bare, None))


# ---------------------------------------------------------------------------------------------------------------------
# 5. against the reference's own NullInversion (tests/golden/make_golden_null_text.py)
# ---------------------------------------------------------------------------------------------------------------------
def test_null_inversion_matches_reference_class(dev):
    """The notebook's NullInversion class, exec'd unmodified on the fp32 tiny SD oracle (5 DDIM steps, 5 inner
    iterations, epsilon 0), against sliders_b200.inversion.NullInversion on the bf16 kernels with the same weights and
    inputs.  Bounds:
      * ddim_latents: every latent within rel-RMS 2.5e-2 of the oracle's (the single-pass eps bar of
        tests/test_gpu_unet.py; each inversion step is affine in eps with coefficients <= 1);
      * inner losses: each within 10 % relative of the oracle's.  The loss is the squared distance between the guided
        reconstruction and a target; the bf16 eps error (<= 2.5e-2) enters it multiplied by the guidance scale and
        |ce| of the step, and the distance itself is O(1) here, so ~1-5 % is expected;
      * the per-step embedding updates (optimised minus starting embedding) agree in sign on > 0.9 of the elements
        wherever the oracle moved (Adam's first steps move every element by ~lr sign(grad)).  Excepted: the last step
        (t = 0), where prev_step goes from alpha_bar[0] to final_alpha_cumprod = alpha_bar[0] (set_alpha_to_one=False),
        so the reconstruction does not depend on eps (ce = 0) and the loss not on the embedding.  The oracle's gradient
        there is float rounding of an analytically zero value, which Adam's normalisation turns into lr-sized moves;
        ours is exactly zero, so the embedding must stay put;
      * reconstruction of x_0 from x_T with the optimised embeddings: at least half of the improvement over the plain
        unconditional embedding that the oracle recorded."""
    import os

    from sliders_b200 import train_util
    from sliders_b200.inversion import NullInversion
    from sliders_b200.scheduler import DDIMScheduler

    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "null_text_sd.pt"))
    ocfg, pm, _ = _models(fx["config"], fx["weight_seed"], dev)
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          set_alpha_to_one=False)
    n = fx["num_ddim_steps"]
    inv = NullInversion(pm, sched, num_ddim_steps=n, guidance_scale=fx["guidance_scale"])
    lat, unc, cond = fx["latent"].to(dev), fx["uncond"].to(dev), fx["cond"].to(dev)
    x_t, ddim_latents, lst = inv.invert(lat, unc, cond, num_inner_steps=fx["num_inner_steps"],
                                        early_stop_epsilon=fx["epsilon"])
    torch.cuda.synchronize()

    errs = [rel_rms(a, b) for a, b in zip(ddim_latents[1:], fx["ddim_latents"][1:])]
    print("ddim_latents rel-RMS per step:", ["%.4f" % e for e in errs])
    assert max(errs) < 2.5e-2

    got = torch.tensor(inv.losses, dtype=torch.float64)
    ref = fx["losses"]
    assert got.shape == ref.shape
    rel = ((got - ref).abs() / ref.abs()).max().item()
    print(f"inner losses: max relative deviation {rel:.4f}")
    assert rel < 0.1

    prev_ce = {int(r[0]): r[4] for r in fx["step_coeffs"][n].tolist()}  # [t, next cx, next ce, prev cx, prev ce]
    start_g, start_o = fx["uncond"], unc.cpu()
    for i, t in enumerate(sched.timesteps_host):
        d_ref = fx["uncond_list"][i] - start_g
        d_got = lst[i].cpu() - start_o
        moved = d_ref != 0
        if abs(prev_ce[t]) < 1e-6:
            assert torch.count_nonzero(d_got) == 0, t
        elif moved.any():
            agree = (torch.sign(d_got[moved]) == torch.sign(d_ref[moved])).float().mean().item()
            print(f"step {i}: sign agreement of the embedding update {agree:.4f}")
            assert agree > 0.9
        start_g, start_o = fx["uncond_list"][i], lst[i].cpu()

    def reconstruct(uncs):
        x = x_t.clone()
        for i, t in enumerate(sched.timesteps_host):
            with torch.no_grad():
                eps = pm(torch.cat([x] * 2), t, encoder_hidden_states=torch.cat([uncs[i], cond])).sample
            x = train_util.guided_step(sched, eps, t, x, fx["guidance_scale"])
        return torch.nn.functional.mse_loss(x, lat).item()

    sched.set_timesteps(n)
    err_opt, err_plain = reconstruct(lst), reconstruct([unc] * n)
    g_opt, g_plain = fx["recon_mse_optimised"], fx["recon_mse_plain"]
    print(f"x_0 reconstruction mse: optimised {err_opt:.4f} plain {err_plain:.4f} "
          f"(oracle: {g_opt:.4f} / {g_plain:.4f})")
    assert err_opt < err_plain - 0.5 * (g_plain - g_opt)
