"""Generates tests/golden/iter_{text_xl,image_xl}.pt — run in the build container, where /root/reference exists:

    python tests/golden/make_golden_iter.py

ONE whole optimisation step of each reference trainer, executed from the reference's OWN source text: the `for i in
pbar:` loop body of
    trainscripts/textsliders/train_lora_xl.py      (:162-375)   SDXL text slider   (SURVEY.md §8 a8)
    [trainscripts/textsliders/train_lora.py :155-321 runs through the same harness, `text_iteration(False)`; its
     fixture is not committed — rank-8 tensors, 4 MB — the SD1.x step is covered by tiny_sd_grads.pt]
    trainscripts/imagesliders/train_lora-scale-xl.py (:178-404) SDXL image slider  (a9)
is read from the file, dedented and exec'd unmodified for a single iteration in a namespace that holds what `train()`
had set up before the loop — the oracle UNet (oracle/unet.py), the reference's own `LoRANetwork`, `train_util`,
`prompt_util`, `model_util.create_noise_scheduler("ddim")` (through oracle/reference_bridge.py), torch.optim.AdamW, a
stand-in VAE for `get_noisy_image` (image sliders), and a seeded RNG.  So the timestep bookkeeping, which UNet call sits
inside `with network:`, the slider sign, the two-backward accumulation and the optimizer step are the reference's, not a
restatement.  Stored: every random draw of the iteration, the inputs, the loss(es), the LoRA gradients and the
post-AdamW LoRA weights.  Model / LoRA weights are regenerated from seeds (sliders_b200.synthetic), like the other
fixtures.  fp32 on CPU; inputs are rounded to bf16-representable values so the bf16 kernels see identical numbers.
"""
import os
import random
import sys
import tempfile
import textwrap
from types import SimpleNamespace

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import reference_bridge as rb  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from sliders_b200 import synthetic  # noqa: E402
import make_golden as mg  # noqa: E402

LR = 1e-2  # large enough for one AdamW step (|delta| ~ lr) to be resolvable in bf16 weights of magnitude ~0.05-0.5
bf = lambda t: t.to(torch.bfloat16).float()


def loop_source(script: str) -> str:
    """The `for i in pbar:` statement of train(), up to (excluding) the final `print("Saving...")`."""
    lines = open(script).read().splitlines()
    start = lines.index("    for i in pbar:")
    end = next(i for i in range(start + 1, len(lines)) if lines[i].startswith('    print("Saving...")'))
    return textwrap.dedent("\n".join(lines[start:end])) + "\n"


class _Bar(list):
    def set_description(self, s):
        pass


def base_namespace(flavour, om, net, pairs, sched, tu, pu):
    opt = torch.optim.AdamW(net.prepare_optimizer_params(), lr=LR)
    return dict(
        torch=torch, train_util=tu, prompt_util=pu, PromptEmbedsPair=pu.PromptEmbedsPair, np=np, os=os, random=random,
        Image=Image, wandb=None, flush=lambda: None, debug_util=None,
        config=SimpleNamespace(train=SimpleNamespace(max_denoising_steps=50, iterations=10),
                               logging=SimpleNamespace(verbose=False, use_wandb=False),
                               save=SimpleNamespace(per_steps=500, name="x")),
        device=torch.device("cpu"), weight_dtype=torch.float32, save_weight_dtype=torch.float32, save_path=None,
        unet=om, network=net, noise_scheduler=sched, optimizer=opt,
        lr_scheduler=tu.get_lr_scheduler("constant", opt, max_iterations=10, lr_min=LR / 100),
        criteria=torch.nn.MSELoss(), prompt_pairs=pairs, pbar=_Bar([0]), loss=None)


def snapshot(net):
    return {k: v.detach().clone() for k, v in net.state_dict().items()}


def grads_of(net):
    return {k: p.grad.detach().to(torch.bfloat16) for k, p in net.named_parameters()}


def pick_seed(n_pairs, lo, hi, max_steps=50, image=False):
    """First seed whose draws give a short partial denoise (lo <= timesteps_to <= hi): keeps the CPU run and the bf16
    error accumulation of the comparison small.  The draws themselves are the reference's (torch.randint, in order)."""
    for seed in range(1000):
        torch.manual_seed(seed)
        torch.randint(0, n_pairs, (1,))
        tt = torch.randint(1, max_steps, (1,)).item()
        if lo <= tt <= hi:
            return seed, tt
    raise RuntimeError("no seed")


def text_iteration(xl: bool):
    lora, tu, mu, pu = rb.load("lora"), rb.load("train_util"), rb.load("model_util"), rb.load("prompt_util")
    cfg_name, rank, alpha = ("tiny_xl", 4, 1.0) if xl else ("tiny_sd", 8, 4.0)
    cfg, om, net = mg.build(cfg_name, lora, rank, alpha, "noxattn")
    net.requires_grad_(True)
    sched = mu.create_noise_scheduler("ddim")
    g = torch.Generator().manual_seed(77)
    D = cfg.cross_attention_dim

    def emb():
        if xl:
            return pu.PromptEmbedsXL(bf(torch.randn(1, 77, D, generator=g)), bf(torch.randn(1, 128, generator=g)))
        return bf(torch.randn(1, 77, D, generator=g))

    e = {k: emb() for k in ("target", "positive", "unconditional", "neutral")}
    settings = pu.PromptSettings(target="t", positive="p", unconditional="u", neutral="n", action="enhance",
                                 guidance_scale=4.0, resolution=256, batch_size=1)
    pair = pu.PromptEmbedsPair(torch.nn.MSELoss(), e["target"], e["positive"], e["unconditional"], e["neutral"], settings)
    ns = base_namespace("text", om, net, [pair], sched, tu, pu)
    seed, tt = pick_seed(1, 2, 3)
    captured = {}
    orig = tu.get_initial_latents

    def rounded_initial_latents(*a, **k):   # inputs of the comparison are bf16-representable
        captured["latents"] = bf(orig(*a, **k))
        return captured["latents"]

    tu.get_initial_latents = rounded_initial_latents
    before = snapshot(net)
    script = os.path.join(rb.REFERENCE_ROOT, "trainscripts", "textsliders", "train_lora_xl.py" if xl else "train_lora.py")
    try:
        torch.manual_seed(seed)
        exec(compile(loop_source(script), script, "exec"), ns)
    finally:
        tu.get_initial_latents = orig
    assert ns["timesteps_to"] == tt
    out = {"config": cfg_name, "weight_seed": mg.WEIGHT_SEED, "lora_seed": mg.LORA_SEED, "rank": rank, "alpha": alpha,
           "up_std": 0.05, "lr": LR, "seed": seed, "timesteps_to": tt, "current_timestep": int(ns["current_timestep"]),
           "n_lora": len(net.unet_loras), "latents": captured["latents"], "denoised_latents": ns["denoised_latents"].detach(),
           "embeds": {k: ((v.text_embeds, v.pooled_embeds) if xl else v) for k, v in e.items()},
           "settings": dict(action="enhance", guidance_scale=4.0, resolution=256, batch_size=1),
           "loss": ns["loss"].detach(), "grads": grads_of(net), "lora_before": before, "lora_after": snapshot(net)}
    if xl:
        out["add_time_ids"] = ns["add_time_ids"].detach()
    return out


class _FakeVAE:
    """Stand-in for AutoencoderKL in `get_noisy_image` (imagesliders/train_util.py:201-235): 8x average pooling and a
    fixed 3->4 channel mix; outputs are bf16-representable and the scaling factor is a power of two, so the latents
    the reference loop sees are exactly what the fixture stores."""
    device = torch.device("cpu")
    config = SimpleNamespace(block_out_channels=(1, 1, 1, 1), scaling_factor=0.125)
    mix = torch.tensor([[1.0, 0.5, -0.5], [-0.75, 1.0, 0.25], [0.5, -1.0, 0.75], [0.25, 0.5, 1.0]])

    def to(self, *a, **k):
        return self

    def encode(self, image):
        lat = torch.einsum("oc,bchw->bohw", self.mix, torch.nn.functional.avg_pool2d(image, 8))
        lat = bf(lat * 4.0)
        return SimpleNamespace(latent_dist=SimpleNamespace(sample=lambda generator=None: lat))


def image_iteration():
    lora = rb.load("lora", "image")
    tu, mu, pu = rb.load("train_util", "image"), rb.load("model_util", "image"), rb.load("prompt_util", "image")
    cfg, om, net = mg.build("tiny_xl", lora, 4, 1.0, "noxattn")
    net.requires_grad_(True)
    sched = mu.create_noise_scheduler("ddim")
    g = torch.Generator().manual_seed(78)
    D = cfg.cross_attention_dim
    emb = lambda: pu.PromptEmbedsXL(bf(torch.randn(1, 77, D, generator=g)), bf(torch.randn(1, 128, generator=g)))
    e = {k: emb() for k in ("target", "positive", "unconditional", "neutral")}
    settings = pu.PromptSettings(target="t", positive="p", unconditional="u", neutral="n", action="enhance",
                                 guidance_scale=4.0, resolution=512, batch_size=1)
    pair = pu.PromptEmbedsPair(torch.nn.MSELoss(), e["target"], e["positive"], e["unconditional"], e["neutral"], settings)
    ns = base_namespace("image", om, net, [pair], sched, tu, pu)
    vae = _FakeVAE()
    seed, tt = pick_seed(1, 10, 40)
    with tempfile.TemporaryDirectory() as folder_main:
        rng = np.random.RandomState(5)
        base = rng.randint(0, 256, (64, 64, 3)).astype(np.uint8)   # the loop resizes to 512 x 512
        folders, scales = ["low", "high"], [-1, 1]
        for name, shift in (("low", 0), ("high", 40)):
            os.makedirs(os.path.join(folder_main, name))
            img = np.clip(base.astype(np.int32) + shift, 0, 255).astype(np.uint8)
            Image.fromarray(img).save(os.path.join(folder_main, name, "a.png"))
        ns.update(vae=vae, folder_main=folder_main, folders=np.array(folders), scales=np.array(scales),
                  scales_unique=list(scales))
        before = snapshot(net)
        script = os.path.join(rb.REFERENCE_ROOT, "trainscripts", "imagesliders", "train_lora-scale-xl.py")
        torch.manual_seed(seed)
        random.seed(seed)
        exec(compile(loop_source(script), script, "exec"), ns)
        proc = sys.modules["diffusers.image_processor"].VaeImageProcessor(8)
        lat = {n: vae.config.scaling_factor * vae.encode(proc.preprocess(
            Image.open(os.path.join(folder_main, n, "a.png")).resize((512, 512)))).latent_dist.sample(None)
            for n in ("low", "high")}
    assert ns["timesteps_to"] == tt and ns["scale_to_look"] == 1
    return {"config": "tiny_xl", "weight_seed": mg.WEIGHT_SEED, "lora_seed": mg.LORA_SEED, "rank": 4, "alpha": 1.0,
            "up_std": 0.05, "lr": LR, "seed": seed, "timesteps_to": tt, "noise_seed": int(ns["seed"]),
            "n_lora": len(net.unet_loras),
            "scale_to_look": float(ns["scale_to_look"]), "current_timestep": int(ns["current_timestep"]),
            "latents_low": lat["low"], "latents_high": lat["high"],
            "noisy_low": ns["denoised_latents_low"].detach(), "noisy_high": ns["denoised_latents_high"].detach(),
            "embeds": {k: (v.text_embeds, v.pooled_embeds) for k, v in e.items()},
            "settings": dict(action="enhance", guidance_scale=4.0, resolution=512, batch_size=1),
            "add_time_ids": ns["add_time_ids"].detach(),
            "loss_high": ns["loss_high"].detach(), "loss_low": ns["loss_low"].detach(),
            "grads": grads_of(net), "lora_before": before, "lora_after": snapshot(net)}


def main():
    assert rb.available(), "needs /root/reference"
    for name, fn in (("iter_text_xl", lambda: text_iteration(True)), ("iter_image_xl", image_iteration)):
        fx = fn()
        # the first AdamW step moves every weight by ~ -lr * sign(grad): the sign of the move is what survives bf16
        # weights, so that is what is stored (int8), not two more copies of the 178 x 2 tensors; `lora_before` is
        # regenerated from the seeds by the tests (make_golden.build)
        before, after = fx.pop("lora_before"), fx.pop("lora_after")
        fx["delta_sign"] = {k: torch.sign(after[k] - before[k]).to(torch.int8) for k in after if "alpha" not in k}
        mg.save_grad_subset(fx, os.path.join(HERE, name + ".pt"))
        gn = sum(float(g.float().pow(2).sum()) for g in fx["grads"].values()) ** 0.5
        print(name, "seed", fx["seed"], "timesteps_to", fx["timesteps_to"], "t", fx["current_timestep"],
              {k: float(fx[k]) for k in fx if k.startswith("loss")}, "grad norm", gn, "tensors", len(fx["grads"]))


if __name__ == "__main__":
    main()
