"""Generates tests/golden/tiny_{xl,sd}_grads.pt — run in the build container, where /root/reference exists:

    python tests/golden/make_golden_grads.py

One text-slider optimisation step's gradient, produced by the REFERENCE'S OWN, UNMODIFIED code (same bridge as
make_golden.py): `with network: target = predict_noise_xl(...)` with autograd on (train_lora_xl.py:299-322),
`PromptEmbedsPair.loss` (prompt_util.py:123-148) against the committed no-grad predictions, `loss.backward()`
(:345).  The fixture stores d loss / d lora_{down,up}.weight for every adaptor, keyed by the state-dict name.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import reference_bridge as rb  # noqa: E402
import make_golden as mg  # noqa: E402


def main():
    assert rb.available(), "needs /root/reference"
    lora, tu, mu, pu = rb.load("lora"), rb.load("train_util"), rb.load("model_util"), rb.load("prompt_util")

    fx = torch.load(os.path.join(HERE, "tiny_xl.pt"))
    cfg, om, net = mg.build("tiny_xl", lora, 4, 1.0, "noxattn")
    sched = mu.create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    t = fx["timestep"]
    net.requires_grad_(True)
    with net:
        target = tu.predict_noise_xl(om, sched, t, fx["latents"], fx["text_embeddings"], fx["add_text_embeddings"],
                                     fx["add_time_ids"], guidance_scale=1)
    settings = pu.PromptSettings(target="t", positive="p", unconditional="u", neutral="n", action="enhance",
                                 guidance_scale=4.0, resolution=256, batch_size=1)
    pair = pu.PromptEmbedsPair(torch.nn.MSELoss(), None, None, None, None, settings)
    loss = pair.loss(target_latents=target, positive_latents=fx["eps_off_g3"], neutral_latents=fx["eps_off_g1"],
                     unconditional_latents=fx["eps_on_sm2_g3"])
    loss.backward()
    out = {"loss": loss.detach(), "target": target.detach(),
           "grads": {k: p.grad.to(torch.bfloat16) for k, p in net.named_parameters()}}
    assert all(torch.isfinite(g).all() and g.abs().sum() > 0 for g in out["grads"].values())
    mg.save_grad_subset(out, os.path.join(HERE, "tiny_xl_grads.pt"))
    print("tiny_xl_grads:", len(out["grads"]), "tensors, loss", float(loss))

    fx = torch.load(os.path.join(HERE, "tiny_sd.pt"))
    cfg, om, net = mg.build("tiny_sd", lora, 8, 4.0, "noxattn")
    sched = mu.create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    net.requires_grad_(True)
    net.set_lora_slider(-1.0)  # image sliders train both signs (train_lora-scale-xl.py:312-372)
    with net:
        pred = tu.predict_noise(om, sched, fx["timestep"], fx["latents"], fx["text_embeddings"], guidance_scale=1)
    noise = fx["eps_off_g7.5"] * 0.1
    loss = torch.nn.functional.mse_loss(pred.float(), noise.float())  # train_lora-scale-xl.py:338
    loss.backward()
    out = {"loss": loss.detach(), "pred": pred.detach(), "noise": noise,
           "grads": {k: p.grad.to(torch.bfloat16) for k, p in net.named_parameters()}}
    assert all(torch.isfinite(g).all() and g.abs().sum() > 0 for g in out["grads"].values())
    mg.save_grad_subset(out, os.path.join(HERE, "tiny_sd_grads.pt"))
    print("tiny_sd_grads:", len(out["grads"]), "tensors, loss", float(loss))


if __name__ == "__main__":
    main()
