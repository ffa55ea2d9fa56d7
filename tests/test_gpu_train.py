"""End-to-end optimisation steps of the three trainers (sliders_b200/trainer.py) on the tiny fixtures' models:
the text-slider step (train_lora_xl.py:162-356 / train_lora.py:155-309) and the image-slider step
(train_lora-scale-xl.py:178-384), forward and backward in sb200 kernels, AdamW fused."""
import os

import pytest
import torch

from test_gpu_unet import GOLDEN, build_product, dev  # noqa: F401  (fixture re-export)

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _xl_pair(trainer, fx, d, action="enhance", bs=1):
    g = torch.Generator().manual_seed(7)
    mk = lambda: trainer.PromptEmbedsXL(torch.randn(1, 77, 256, generator=g).to(d, BF),
                                        torch.randn(1, 128, generator=g).to(d, BF))
    unc, tgt, pos = mk(), mk(), mk()
    st = trainer.PromptSettings(guidance_scale=4.0, resolution=256, batch_size=bs, action=action)
    return trainer.PromptEmbedsPair(torch.nn.MSELoss(), tgt, pos, unc, unc, st)


def test_text_slider_steps_xl(dev):
    from sliders_b200 import trainer, train_util
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    net.requires_grad_(True)
    params = net.prepare_optimizer_params()
    opt = train_util.get_optimizer("AdamW")(params, lr=2e-3)
    lr_sched = train_util.get_lr_scheduler("constant", opt, 100, 1e-6)
    sched = create_noise_scheduler("ddim")
    pair = _xl_pair(trainer, fx, dev)
    before = {k: v.detach().clone() for k, v in net.named_parameters()}
    gen = torch.Generator().manual_seed(3)
    losses = []
    for it in range(6):
        gen.manual_seed(3)  # same initial noise / same timestep: the loss must go down as the slider learns it
        losses.append(float(trainer.text_slider_step_xl(pm, net, sched, opt, lr_sched, pair, max_denoising_steps=50,
                                                        timesteps_to=2, device=dev, weight_dtype=BF, generator=gen)))
    assert all(l == l and l < 1e4 for l in losses)
    assert losses[-1] < losses[0], losses
    changed = sum(int(not torch.equal(before[k], v.detach())) for k, v in net.named_parameters())
    assert changed == len(before)
    assert all(float(l.multiplier) == 0.0 for l in net.unet_loras)  # `with network:` closed (lora.py:256-258)
    # erase action, random timestep, batch 2
    pair2 = _xl_pair(trainer, fx, dev, action="erase", bs=2)
    l = trainer.text_slider_step_xl(pm, net, sched, opt, lr_sched, pair2, device=dev, weight_dtype=BF)
    assert torch.isfinite(l)


def test_text_slider_step_sd(dev):
    from sliders_b200 import trainer, train_util
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_sd.pt"))
    pm, net = build_product(fx, dev)
    net.requires_grad_(True)
    opt = train_util.get_optimizer("AdamW")(net.prepare_optimizer_params(), lr=1e-3)
    sched = create_noise_scheduler("ddim")
    g = torch.Generator().manual_seed(5)
    D = fx["text_embeddings"].shape[-1]
    unc, tgt, pos = (torch.randn(1, 77, D, generator=g).to(dev, BF) for _ in range(3))
    st = trainer.PromptSettings(guidance_scale=1.0, resolution=256, batch_size=1, action="erase")
    pair = trainer.PromptEmbedsPair(torch.nn.MSELoss(), tgt, pos, unc, unc, st)
    gen = torch.Generator()
    losses = []
    for _ in range(4):
        gen.manual_seed(1)
        losses.append(float(trainer.text_slider_step(pm, net, sched, opt, None, pair, timesteps_to=3, device=dev,
                                                     weight_dtype=BF, generator=gen)))
    assert losses[-1] < losses[0], losses


def test_image_slider_step_xl(dev):
    from sliders_b200 import trainer, train_util
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    pm, net = build_product(fx, dev)
    net.requires_grad_(True)
    opt = train_util.get_optimizer("AdamW")(net.prepare_optimizer_params(), lr=1e-3)
    sched = create_noise_scheduler("ddim")
    pair = _xl_pair(trainer, fx, dev)
    g = torch.Generator().manual_seed(9)
    low = torch.randn(1, 4, 32, 32, generator=g).to(dev)
    high = low + 0.3 * torch.randn(1, 4, 32, 32, generator=g).to(dev)
    first = last = None
    for _ in range(4):
        ls = trainer.image_slider_step_xl(pm, net, sched, opt, None, pair, low, high, 2.0, timesteps_to=20, seed=4,
                                          device=dev, weight_dtype=BF)
        tot = float(ls[0] + ls[1])
        first = tot if first is None else first
        last = tot
    assert last < first, (first, last)


def test_training_cuda_graphs_match_eager(dev):
    """`unet.use_cuda_graph = True` replays the training forward and backward as two CUDA graphs
    (sliders_b200/autograd.py::_TrainCapture): same kernels, same order -> bit-identical LoRA weights after two
    optimisation steps, including the second step that reuses the captured graphs with updated weights."""
    from sliders_b200 import trainer, train_util
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "tiny_xl.pt"))
    results = {}
    for mode in ("eager", "graph"):
        pm, net = build_product(fx, dev)
        net.requires_grad_(True)
        pm.use_cuda_graph = mode == "graph"
        opt = train_util.get_optimizer("AdamW")(net.prepare_optimizer_params(), lr=1e-3)
        sched = create_noise_scheduler("ddim")
        pair = _xl_pair(trainer, fx, dev)
        losses = []
        for it in range(3):
            losses.append(float(trainer.text_slider_step_xl(pm, net, sched, opt, None, pair, timesteps_to=2, device=dev,
                                                            weight_dtype=BF,
                                                            generator=torch.Generator().manual_seed(40 + it))))
        results[mode] = (losses, torch.cat([p.detach().float().reshape(-1) for p in net.parameters()]))
        if mode == "graph":
            assert len(pm.__dict__.get("_train_graphs", {})) == 1
    assert results["eager"][0] == results["graph"][0], (results["eager"][0], results["graph"][0])
    assert torch.equal(results["eager"][1], results["graph"][1])


# ------------------------------------------------------------------------------------------------------------------
# Whole-iteration parity (SURVEY.md §8 a8 / a9): tests/golden/iter_*.pt hold ONE optimisation step produced by exec'ing
# the reference's own loop-body source on the fp32 oracle (tests/golden/make_golden_iter.py).  The product step gets the
# same seeds and must reproduce the loss (5 %), the LoRA gradients (rel-RMS 5e-2 over all tensors; bf16 kernels and a
# bf16 partial denoise against fp32) and the direction of the AdamW move (|grad|-weighted sign agreement >= 0.97).
# ------------------------------------------------------------------------------------------------------------------
def _grad_rel_rms(net, golden):
    # over the adaptors the fixture stores (a fixed subset, to keep the file small)
    num = den = 0.0
    compared = 0
    for k, p in net.named_parameters():
        if k not in golden:
            continue
        compared += 1
        ref = golden[k].float().to(p.device)
        num += (p.grad.float() - ref).pow(2).sum().item()
        den += ref.pow(2).sum().item()
    assert compared == len(golden), (compared, len(golden))
    return (num / den) ** 0.5


def _move_agreement(net, before, golden_sign, golden_grads):
    agree = total = 0.0
    for k, p in net.named_parameters():
        if k not in golden_grads:
            continue
        w = golden_grads[k].float().abs().to(p.device)
        ours = torch.sign(p.detach().float() - before[k].float())
        agree += (w * (ours == golden_sign[k].to(p.device).float())).sum().item()
        total += w.sum().item()
    return agree / total


def _pair_from(trainer, fx, d):
    e = {k: trainer.PromptEmbedsXL(v[0].to(d, BF), v[1].to(d, BF)) for k, v in fx["embeds"].items()}
    st = trainer.PromptSettings(**fx["settings"])
    return trainer.PromptEmbedsPair(torch.nn.MSELoss(), e["target"], e["positive"], e["unconditional"], e["neutral"], st)


def test_text_slider_iteration_matches_reference_loop(dev):
    from sliders_b200 import trainer
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "iter_text_xl.pt"))
    pm, net = build_product(fx, dev)
    net.requires_grad_(True)
    opt = torch.optim.AdamW(net.prepare_optimizer_params(), lr=fx["lr"])  # the reference's optimizer class, on bf16
    before = {k: p.detach().clone() for k, p in net.named_parameters()}
    pair = _pair_from(trainer, fx, dev)
    # same seed, same order of draws as the reference loop (pair index, timesteps_to, initial noise): nothing is passed in
    torch.manual_seed(fx["seed"])
    torch.randint(0, 1, (1,))   # `prompt_pairs[torch.randint(0, len(prompt_pairs), (1,))]` (train_lora_xl.py:172-174)
    loss = trainer.text_slider_step_xl(pm, net, create_noise_scheduler("ddim"), opt, None, pair, max_denoising_steps=50,
                                       device=dev, weight_dtype=BF)
    assert abs(float(loss) - float(fx["loss"])) <= 0.05 * float(fx["loss"]), (float(loss), float(fx["loss"]))
    assert _grad_rel_rms(net, fx["grads"]) < 5e-2
    assert _move_agreement(net, before, fx["delta_sign"], fx["grads"]) > 0.97


def test_image_slider_iteration_matches_reference_loop(dev):
    from sliders_b200 import trainer
    from sliders_b200.scheduler import create_noise_scheduler

    fx = torch.load(os.path.join(GOLDEN, "iter_image_xl.pt"))
    pm, net = build_product(fx, dev)
    net.requires_grad_(True)
    opt = torch.optim.AdamW(net.prepare_optimizer_params(), lr=fx["lr"])
    before = {k: p.detach().clone() for k, p in net.named_parameters()}
    pair = _pair_from(trainer, fx, dev)
    torch.manual_seed(fx["seed"])
    torch.randint(0, 1, (1,))   # prompt-pair pick (train_lora-scale-xl.py:186-188); timesteps_to is drawn by the step
    ls = trainer.image_slider_step_xl(pm, net, create_noise_scheduler("ddim"), opt, None, pair, fx["latents_low"],
                                      fx["latents_high"], fx["scale_to_look"], max_denoising_steps=50,
                                      seed=fx["noise_seed"], device=dev, weight_dtype=BF)
    assert abs(float(ls[0]) - float(fx["loss_high"])) <= 0.05 * float(fx["loss_high"])
    assert abs(float(ls[1]) - float(fx["loss_low"])) <= 0.05 * float(fx["loss_low"])
    assert _grad_rel_rms(net, fx["grads"]) < 5e-2
    assert _move_agreement(net, before, fx["delta_sign"], fx["grads"]) > 0.97
