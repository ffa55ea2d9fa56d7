"""Generates tests/golden/*.pt — run in the build container, where /root/reference exists:

    python tests/golden/make_golden.py

Every fixture is produced by the REFERENCE'S OWN, UNMODIFIED code driving the oracle UNet:
  * `LoRANetwork` / `LoRAModule.forward` from /root/reference/trainscripts/textsliders/lora.py (the real hook,
    lora.py:108-112 — not the folded-weight shortcut the GPU tests use),
  * `predict_noise_xl` / `predict_noise` / `diffusion_xl` from …/train_util.py (:145-171, :220-294),
  * `create_noise_scheduler("ddim")` from …/model_util.py:230-246 (constructing the oracle DDIM restatement),
  * `PromptEmbedsPair.loss` from …/prompt_util.py:108-148,
through oracle/reference_bridge.py (a stub `diffusers` module exposes oracle/unet.py and oracle/ddim.py under the
names the reference imports).  Model weights are NOT stored: they are regenerated from a seed with
sliders_b200.synthetic (deterministic CPU generator), only inputs and outputs are committed (a few hundred KB).
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import reference_bridge as rb  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from sliders_b200 import synthetic  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
WEIGHT_SEED, LORA_SEED = 11, 12


MAX_FIXTURE_BYTES = 1_000_000


def save_grad_subset(fx, path):
    """torch.save(fx) with the per-adaptor gradient dicts ("grads", and "delta_sign" where present) cut to every
    stride-th adaptor (sorted names, both lora_down and lora_up of a kept adaptor), the smallest stride that keeps the
    file under MAX_FIXTURE_BYTES.  "grad_keys" keeps the full key list for the adaptor-set checks."""
    import io

    def adaptor(k):
        return k.rsplit(".lora_", 1)[0]

    keys = list(fx["grads"].keys())
    names = sorted({adaptor(k) for k in keys})
    for stride in range(1, len(names) + 1):
        keep = {n for i, n in enumerate(names) if i % stride == 0}
        out = dict(fx, grad_keys=keys)
        for field in ("grads", "delta_sign"):
            if field in fx:
                out[field] = {k: v for k, v in fx[field].items() if adaptor(k) in keep}
        buf = io.BytesIO()
        torch.save(out, buf)
        if buf.tell() < MAX_FIXTURE_BYTES:
            break
    with open(path, "wb") as f:
        f.write(buf.getvalue())
    return stride


def build(cfg_name, lora, rank, alpha, method):
    cfg = getattr(ounet.UNetConfig, cfg_name)()
    torch.manual_seed(0)
    om = ounet.UNet2DConditionModel(cfg)
    synthetic.init_synthetic_(om, seed=WEIGHT_SEED)
    om.requires_grad_(False)
    om.eval()
    saved = list(lora.DEFAULT_TARGET_REPLACE)
    lora.DEFAULT_TARGET_REPLACE += lora.UNET_TARGET_REPLACE_MODULE_CONV
    try:
        net = lora.LoRANetwork(om, rank=rank, multiplier=1.0, alpha=alpha, train_method=method)
    finally:
        del lora.DEFAULT_TARGET_REPLACE[len(saved):]
    synthetic.init_lora_nonzero_(net, seed=LORA_SEED, up_std=0.05, reseed_down=True)
    return cfg, om, net


def main():
    assert rb.available(), "needs /root/reference"
    lora = rb.load("lora")
    tu = rb.load("train_util")
    mu = rb.load("model_util")
    pu = rb.load("prompt_util")
    g = torch.Generator().manual_seed(1234)

    # ------------------------------------------------------------------ SDXL topology (tiny_xl)
    cfg, om, net = build("tiny_xl", lora, 4, 1.0, "noxattn")
    sched = mu.create_noise_scheduler("ddim")
    lat = torch.randn(1, 4, 32, 32, generator=g)
    ehs = torch.randn(2, 77, cfg.cross_attention_dim, generator=g)  # [uncond ; cond]
    pooled = torch.randn(2, 128, generator=g)
    tids = tu.get_add_time_ids(256, 256).repeat(2, 1) if False else torch.tensor([[256., 256., 0., 0., 256., 256.]] * 2)
    lat, ehs, pooled = (t.to(torch.bfloat16).float() for t in (lat, ehs, pooled))
    fx = {"config": "tiny_xl", "weight_seed": WEIGHT_SEED, "lora_seed": LORA_SEED, "rank": 4, "alpha": 1.0,
          "train_method": "noxattn+c3lier", "up_std": 0.05, "latents": lat, "text_embeddings": ehs,
          "add_text_embeddings": pooled, "add_time_ids": tids, "n_lora": len(net.unet_loras)}
    with torch.no_grad():
        sched.set_timesteps(1000)
        t = int(sched.timesteps[500])
        fx["timestep"] = t
        # LoRA off (multiplier 0 after __exit__), guidance 1 and 3
        net.__exit__(None, None, None)
        fx["eps_off_g1"] = tu.predict_noise_xl(om, sched, t, lat, ehs, pooled, tids, guidance_scale=1)
        fx["eps_off_g3"] = tu.predict_noise_xl(om, sched, t, lat, ehs, pooled, tids, guidance_scale=3)
        # LoRA on at slider 1 and -2 (set_lora_slider + context manager, lora.py:249-258)
        with net:
            fx["eps_on_s1_g1"] = tu.predict_noise_xl(om, sched, t, lat, ehs, pooled, tids, guidance_scale=1)
        net.set_lora_slider(-2.0)
        with net:
            fx["eps_on_sm2_g3"] = tu.predict_noise_xl(om, sched, t, lat, ehs, pooled, tids, guidance_scale=3)
        net.set_lora_slider(1.0)
        # partial denoise: 3 of 50 DDIM steps, guidance 3, LoRA on (train_lora_xl.py:205-227)
        sched.set_timesteps(50)
        with net:
            fx["denoised_3of50_g3"] = tu.diffusion_xl(om, sched, lat, ehs, pooled, tids, guidance_scale=3,
                                                      total_timesteps=3)
        # the text-slider loss on four predictions (prompt_util.py:123-148), enhance, guidance 4
        settings = pu.PromptSettings(target="t", positive="p", unconditional="u", neutral="n", action="enhance",
                                     guidance_scale=4.0, resolution=256, batch_size=1)
        pair = pu.PromptEmbedsPair(torch.nn.MSELoss(), None, None, None, None, settings)
        fx["loss_enhance_g4"] = pair.loss(target_latents=fx["eps_on_s1_g1"], positive_latents=fx["eps_off_g3"],
                                          neutral_latents=fx["eps_off_g1"],
                                          unconditional_latents=fx["eps_on_sm2_g3"])
    torch.save(fx, os.path.join(OUT, "tiny_xl.pt"))
    print("tiny_xl:", {k: (tuple(v.shape) if torch.is_tensor(v) else v) for k, v in fx.items()})

    # ------------------------------------------------------------------ SD1.x topology (tiny_sd), rank 8
    cfg, om, net = build("tiny_sd", lora, 8, 4.0, "noxattn")
    sched = mu.create_noise_scheduler("ddim")
    lat = torch.randn(2, 4, 32, 32, generator=g).to(torch.bfloat16).float()
    ehs = torch.randn(2, 77, cfg.cross_attention_dim, generator=g).to(torch.bfloat16).float()
    ehs = tu.concat_embeddings(ehs[:1], ehs[1:], 2)  # [u,u,c,c]
    fx = {"config": "tiny_sd", "weight_seed": WEIGHT_SEED, "lora_seed": LORA_SEED, "rank": 8, "alpha": 4.0,
          "train_method": "noxattn+c3lier", "up_std": 0.05, "latents": lat, "text_embeddings": ehs,
          "n_lora": len(net.unet_loras)}
    with torch.no_grad():
        sched.set_timesteps(1000)
        t = int(sched.timesteps[19])
        fx["timestep"] = t
        net.__exit__(None, None, None)
        fx["eps_off_g7.5"] = tu.predict_noise(om, sched, t, lat, ehs, guidance_scale=7.5)
        with net:
            fx["eps_on_s1_g1"] = tu.predict_noise(om, sched, t, lat, ehs, guidance_scale=1)
    torch.save(fx, os.path.join(OUT, "tiny_sd.pt"))
    print("tiny_sd:", {k: (tuple(v.shape) if torch.is_tensor(v) else v) for k, v in fx.items()})


if __name__ == "__main__":
    main()
