"""Generates tests/golden/null_text_sd.pt — run in the build container, where /root/reference exists:

    python tests/golden/make_golden_null_text.py

The `NullInversion` class of the reference's demo_image_editing.ipynb is read from the notebook (the cell that defines
it, from `class NullInversion:` to the end of the class) and exec'd UNMODIFIED in a namespace that holds what the
notebook had set up before it: `NUM_DDIM_STEPS` (5 here, to keep the CPU run short), `GUIDANCE_SCALE = 7.5`,
torch.optim.Adam, a no-op `ptp_utils.register_attention_control`, a progress-bar stand-in, and `nnf` whose `mse_loss`
records every inner-step loss.  The stub `model` holds the tiny SD oracle UNet (oracle/unet.py, fp32 CPU, weights
regenerated from a seed through sliders_b200.synthetic and rounded to bf16 like the product's) and the oracle DDIM
scheduler built as the notebook builds it (scaled_linear, clip_sample=False, set_alpha_to_one=False).  `self.context`
is set from seeded embeddings and the class's own `ddim_loop` and `null_optimization` run with epsilon = 0, so that
bf16-vs-fp32 noise cannot flip an early stop.

Stored: the inputs, `ddim_latents`, every inner-step loss, the per-step `uncond_embeddings_list`, the oracle's
reconstruction error of x_0 when x_T is denoised by the class's own guided step (`get_noise_pred(..., False, ...)`) with
the optimised list and with the plain unconditional embedding, and the (cx, ce) coefficients of the class's `next_step`
/ `prev_step` (x_next = cx x + ce eps) at every timestep for 5, 7 and 50 DDIM steps.
"""
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ddim as oddim  # noqa: E402
from oracle import reference_bridge as rb  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from sliders_b200 import synthetic  # noqa: E402
from sliders_b200.unet import UNet2DConditionModel, UNetConfig  # noqa: E402

NOTEBOOK = os.path.join(rb.REFERENCE_ROOT, "demo_image_editing.ipynb")
WEIGHT_SEED, INPUT_SEED = 81, 11
STEPS, INNER = 5, 5


def class_source() -> str:
    """`class NullInversion:` ... up to the first top-level statement after it, from the notebook cell."""
    nb = json.load(open(NOTEBOOK))
    src = next("".join(c["source"]) for c in nb["cells"] if "class NullInversion" in "".join(c["source"]))
    lines = src.splitlines()
    start = next(i for i, l in enumerate(lines) if l.startswith("class NullInversion"))
    end = next((i for i in range(start + 1, len(lines)) if lines[i] and not lines[i][0].isspace()), len(lines))
    return "\n".join(lines[start:end]) + "\n"


class _Bar:
    def __init__(self, *a, **k):
        pass

    def update(self, *a):
        pass

    def close(self):
        pass


class _Unet:
    """`self.model.unet(...)["sample"]` and `self.model.unet.dtype` over the oracle UNet."""

    dtype = torch.float32

    def __init__(self, om):
        self.om = om

    def __call__(self, latents, t, encoder_hidden_states):
        return {"sample": self.om(latents, t, encoder_hidden_states).sample}


def tiny_sd_oracle():
    ocfg = ounet.UNetConfig.tiny_sd()
    pm = UNet2DConditionModel(UNetConfig.from_dict(ocfg.__dict__))
    synthetic.init_synthetic_(pm, seed=WEIGHT_SEED)
    om = ounet.UNet2DConditionModel(ocfg)
    om.load_state_dict({k: v.to(torch.bfloat16).float() for k, v in pm.state_dict().items()})
    return ocfg, om.eval().requires_grad_(False)


def scheduler():
    return oddim.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                               set_alpha_to_one=False)


def main():
    assert os.path.isfile(NOTEBOOK), "needs the reference tree"
    torch.manual_seed(0)
    ocfg, om = tiny_sd_oracle()
    losses = []

    def mse_loss(a, b):
        loss = torch.nn.functional.mse_loss(a, b)
        losses.append(loss.item())
        return loss

    model = SimpleNamespace(unet=_Unet(om), scheduler=scheduler(), tokenizer=None)
    ns = dict(torch=torch, np=np, Union=__import__("typing").Union, tqdm=_Bar, Adam=torch.optim.Adam,
              nnf=SimpleNamespace(mse_loss=mse_loss), DDIMScheduler=oddim.DDIMScheduler,
              ptp_utils=SimpleNamespace(register_attention_control=lambda *a: None),
              NUM_DDIM_STEPS=STEPS, GUIDANCE_SCALE=7.5, device=torch.device("cpu"))
    exec(compile(class_source(), NOTEBOOK, "exec"), ns)
    inv = ns["NullInversion"](model)

    g = torch.Generator().manual_seed(INPUT_SEED)
    bf = lambda t: t.to(torch.bfloat16).float()
    latent = bf(0.8 * torch.randn(1, 4, 32, 32, generator=g))
    uncond = bf(torch.randn(1, 77, ocfg.cross_attention_dim, generator=g))
    cond = bf(torch.randn(1, 77, ocfg.cross_attention_dim, generator=g))
    inv.context = torch.cat([uncond, cond])
    ddim_latents = inv.ddim_loop(latent)
    uncond_list = inv.null_optimization(ddim_latents, INNER, 0.0)
    assert len(losses) == STEPS * INNER

    def reconstruct(uncs):
        x = ddim_latents[-1]
        with torch.no_grad():
            for i in range(STEPS):
                t = model.scheduler.timesteps[i]
                x = inv.get_noise_pred(x, t, False, torch.cat([uncs[i], cond]))
        return torch.nn.functional.mse_loss(x, latent).item()

    err_opt = reconstruct(uncond_list)
    err_plain = reconstruct([uncond] * STEPS)
    print(f"x_0 reconstruction mse: optimised {err_opt:.3e}, plain {err_plain:.3e}")

    coeffs = {}
    for n in (5, 7, 50):
        model.scheduler.set_timesteps(n)
        rows = []
        for t in model.scheduler.timesteps:
            one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
            rows.append([int(t), inv.next_step(zero, t, one).item(), inv.next_step(one, t, zero).item(),
                         inv.prev_step(zero, t, one).item(), inv.prev_step(one, t, zero).item()])
        coeffs[n] = torch.tensor(rows, dtype=torch.float64)  # [t, next cx, next ce, prev cx, prev ce]

    out = {
        "weight_seed": WEIGHT_SEED, "config": "tiny_sd", "num_ddim_steps": STEPS, "num_inner_steps": INNER,
        "guidance_scale": 7.5, "epsilon": 0.0,
        "latent": latent, "uncond": uncond, "cond": cond,
        "ddim_latents": torch.stack([x.detach() for x in ddim_latents]),
        "losses": torch.tensor(losses, dtype=torch.float64).view(STEPS, INNER),
        "uncond_list": torch.stack([e.detach() for e in uncond_list]),
        "recon_mse_optimised": err_opt, "recon_mse_plain": err_plain,
        "step_coeffs": coeffs,
    }
    path = os.path.join(HERE, "null_text_sd.pt")
    torch.save(out, path)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
