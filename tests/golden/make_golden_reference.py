"""Generates tests/golden/reference_answers.pt and the data fixtures under tests/golden/reference/ — run where the
reference tree is present (oracle/reference_bridge.py finds it; SLIDERS_REFERENCE_ROOT overrides the location):

    python tests/golden/make_golden_reference.py

The reference's own, unmodified lora.py / prompt_util.py / config_util.py / train_util.py / model_util.py run on the
oracle UNet and their answers are stored, so the tests that compare this project with the reference need nothing
outside the repository:
  * LoRANetwork injection: leaf names, leaf and parameter counts (SDXL rank 4 / 8, SD1.x rank 4, noxattn + c3lier);
  * state-dict keys of every train_method on SDXL and SD1.x (SHA-256 of the newline-joined key list, and its length),
    and keys / shapes of a rank-4 noxattn network on a small UNet (what a slider file must hold to load strictly);
  * zero-init identity and multiplier semantics: predict_noise_xl on the tiny oracle UNet with the reference's hook
    (fresh adaptors, adaptors off, adaptors on; the adaptor weights are redrawn from a seed per key);
  * the parsed configs / prompt settings of the reference's YAML files (copied as fixtures, with the head of one of
    its prompt CSVs) and the
    PromptEmbedsPair losses for seeded inputs.
"""
import hashlib
import os
import shutil
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from conftest import c3lier  # noqa: E402
from oracle import reference_bridge as rb  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from sliders_b200 import synthetic  # noqa: E402

TRAIN_METHODS = ("noxattn", "full", "xattn", "selfattn", "innoxattn", "xattn-strict", "noxattn-hspace",
                 "noxattn-hspace-last")
YAML_FILES = ("config-xl.yaml", "config.yaml", "prompts-xl.yaml", "prompts.yaml", "prompts-person_age_slider_GPT.yaml")
PROMPT_ATTRIBUTES = {"prompts-xl.yaml": ["male", "female"], "prompts.yaml": [],
                     "prompts-person_age_slider_GPT.yaml": ["asian", "white"]}
SMALL_CFG = dict(block_out_channels=(64, 128), down_block_types=("DownBlock2D", "CrossAttnDownBlock2D"),
                 up_block_types=("CrossAttnUpBlock2D", "UpBlock2D"), transformer_layers_per_block=(1, 1),
                 attention_head_dim=(1, 2), cross_attention_dim=64)


def key_digest(keys):
    return hashlib.sha256("\n".join(keys).encode()).hexdigest(), len(keys)


def main():
    assert rb.available(), f"needs the reference tree at {rb.REFERENCE_ROOT}"
    lora, tu, mu = rb.load("lora"), rb.load("train_util"), rb.load("model_util")
    rc, rp = rb.load("config_util"), rb.load("prompt_util")
    out = {}

    # ---- injection counts and leaf names
    inj = {}
    for name, rank in (("sdxl", 4), ("sdxl", 8), ("sd15", 4)):
        with torch.device("meta"):
            m = ounet.UNet2DConditionModel(getattr(ounet.UNetConfig, name)())
            with c3lier(lora):
                net = lora.LoRANetwork(m, rank=rank, multiplier=1.0, alpha=1.0, train_method="noxattn")
        inj[(name, rank)] = {"n_params": sum(p.numel() for p in net.parameters())}
        inj[name] = [l.lora_name for l in net.unet_loras]  # the same leaves at every rank
    out["injection"] = inj

    # ---- state-dict keys per train_method
    keys = {}
    for name in ("sdxl", "sd15"):
        for method in TRAIN_METHODS:
            with torch.device("meta"):
                m = ounet.UNet2DConditionModel(getattr(ounet.UNetConfig, name)())
                with c3lier(lora):
                    net = lora.LoRANetwork(m, rank=4, multiplier=1.0, alpha=1.0, train_method=method)
            keys[(name, method)] = key_digest(list(net.state_dict().keys()))
    out["state_dict_keys"] = keys
    from sliders_b200.unet import UNetConfig

    om = ounet.UNet2DConditionModel(ounet.UNetConfig(**UNetConfig.from_dict(SMALL_CFG).__dict__))
    with c3lier(lora):
        net = lora.LoRANetwork(om, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn")
    out["small_noxattn"] = {"config": SMALL_CFG, "keys": [(k, tuple(v.shape)) for k, v in net.state_dict().items()]}

    # ---- zero-init identity and multiplier semantics through the reference's hook
    m = ounet.UNet2DConditionModel(ounet.UNetConfig.tiny_xl())
    synthetic.init_synthetic_(m, seed=11)
    m.eval().requires_grad_(False)
    g = torch.Generator().manual_seed(5)
    lat = torch.randn(1, 4, 16, 16, generator=g)
    ehs = torch.randn(2, 77, 256, generator=g)
    pooled = torch.randn(2, 128, generator=g)
    tids = torch.tensor([[128., 128, 0, 0, 128, 128]] * 2)
    sched = mu.create_noise_scheduler("ddim")
    sched.set_timesteps(1000)
    with torch.no_grad():
        base = tu.predict_noise_xl(m, sched, 500, lat, ehs, pooled, tids, guidance_scale=1)
        with c3lier(lora):
            net = lora.LoRANetwork(m, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn")
        with net:
            fresh = tu.predict_noise_xl(m, sched, 500, lat, ehs, pooled, tids, guidance_scale=1)
        synthetic.init_lora_nonzero_(net, seed=1, up_std=0.05, reseed_down=True)  # reproducible from the seed
        off = tu.predict_noise_xl(m, sched, 500, lat, ehs, pooled, tids, guidance_scale=1)
        with net:
            on = tu.predict_noise_xl(m, sched, 500, lat, ehs, pooled, tids, guidance_scale=1)
    out["hook_semantics"] = {
        "weight_seed": 11, "inputs": {"latents": lat, "text_embeddings": ehs, "add_text_embeddings": pooled,
                                      "add_time_ids": tids, "timestep": 500},
        "lora_seed": 1, "lora_up_std": 0.05,
        "base": base, "fresh": fresh, "off": off, "on": on}

    # ---- YAML parsing (fixtures copied beside this file) and the prompt-pair loss
    fix = os.path.join(HERE, "reference")
    os.makedirs(fix, exist_ok=True)
    data = os.path.join(rb.REFERENCE_ROOT, "trainscripts", "textsliders", "data")
    parsed = {}
    for name in YAML_FILES:
        shutil.copyfile(os.path.join(data, name), os.path.join(fix, name))
        if name.startswith("config"):
            parsed[name] = rc.load_config_from_yaml(os.path.join(fix, name)).dict()
        else:
            parsed[name] = [r.dict() for r in rp.load_prompts_from_yaml(os.path.join(fix, name), PROMPT_ATTRIBUTES[name])]
    out["yaml"] = {"attributes": PROMPT_ATTRIBUTES, "parsed": parsed}
    with open(os.path.join(rb.REFERENCE_ROOT, "prompts", "prompts-person.csv")) as f:  # header + the first 40 rows
        head = f.readlines()[:41]
    with open(os.path.join(fix, "prompts-person.csv"), "w") as f:
        f.writelines(head)

    g = torch.Generator().manual_seed(1)
    t, p, u, n = (torch.randn(2, 4, 8, 8, generator=g) for _ in range(4))
    losses = {}
    for action in ("erase", "enhance"):
        rs = rp.PromptSettings(target="t", positive="p", unconditional="u", neutral="n", action=action,
                               guidance_scale=2.5, resolution=512, batch_size=2)
        ref = rp.PromptEmbedsPair(torch.nn.MSELoss(), None, None, None, None, rs)
        losses[action] = {"loss": ref.loss(target_latents=t, positive_latents=p, unconditional_latents=u,
                                           neutral_latents=n),
                          "batch_size": ref.batch_size, "resolution": ref.resolution, "dynamic_crops": ref.dynamic_crops}
    out["prompt_pair"] = {"latents": {"target": t, "positive": p, "unconditional": u, "neutral": n},
                          "guidance_scale": 2.5, "losses": losses}

    torch.save(out, os.path.join(HERE, "reference_answers.pt"))


if __name__ == "__main__":
    main()
