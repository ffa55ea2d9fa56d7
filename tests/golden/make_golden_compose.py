"""Generates tests/golden/compose.pt — run in the build container, where /root/reference exists:

    python tests/golden/make_golden_compose.py

Composition the reference's way: its own, unmodified `LoRANetwork` (trainscripts/textsliders/lora.py) built two and
three times on the same oracle UNet, so each network's `apply_to` chains the previous one's hook (lora.py:103-112) and
every network adds `up(down(x)) * multiplier * scale` at its own multiplier.  Done on the tiny SDXL and tiny SD1.x
topologies; one network is `xattn`, so the cross-attention to_k / to_v leaves are adapted.  Weights are not stored:
the UNet is regenerated from WEIGHT_SEED and each network's adaptors from its own seed with
`synthetic.init_lora_nonzero_` (lora_up nonzero, lora_down redrawn per key), so the GPU test rebuilds them exactly.
Stored: the inputs, eps with every network off, eps with each network alone at its scale, and eps with all of them
at their (mixed-sign) scales.
"""
import io
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import reference_bridge as rb  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from sliders_b200 import synthetic  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
WEIGHT_SEED = 11
MAX_FIXTURE_BYTES = 1_000_000
UP_STD = 0.15  # large enough that every network moves eps well above the bf16 error floor

# (rank, alpha, train_method, network_type, lora seed); the scales are the mixed-sign strengths of the "all on" case
STACKS = {
    "two": ([(4, 1.0, "noxattn", "c3lier", 21), (8, 4.0, "xattn", "lierla", 22)], [1.5, -2.0]),
    "three": ([(4, 1.0, "noxattn", "c3lier", 31), (4, 2.0, "xattn", "lierla", 32), (2, 1.0, "full", "lierla", 33)],
              [2.0, -1.0, 1.0]),
}


def build_networks(lora, om, specs):
    nets = []
    for rank, alpha, method, ntype, seed in specs:
        saved = list(lora.DEFAULT_TARGET_REPLACE)
        if ntype == "c3lier":
            lora.DEFAULT_TARGET_REPLACE += lora.UNET_TARGET_REPLACE_MODULE_CONV
        try:
            net = lora.LoRANetwork(om, rank=rank, multiplier=1.0, alpha=alpha, train_method=method)
        finally:
            del lora.DEFAULT_TARGET_REPLACE[len(saved):]
        synthetic.init_lora_nonzero_(net, seed=seed, up_std=UP_STD, reseed_down=True)
        net.__exit__(None, None, None)
        nets.append(net)
    return nets


def run_config(lora, cfg_name, g):
    cfg = getattr(ounet.UNetConfig, cfg_name)()
    xl = cfg.addition_embed_type == "text_time"
    lat = torch.randn(2, 4, 32, 32, generator=g).to(torch.bfloat16).float()
    ehs = torch.randn(2, 77, cfg.cross_attention_dim, generator=g).to(torch.bfloat16).float()
    added = None
    fx = {"config": cfg_name, "latents": lat, "text_embeddings": ehs, "timestep": 500}
    if xl:
        pooled = torch.randn(2, cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim,
                             generator=g).to(torch.bfloat16).float()
        tids = torch.tensor([[256., 256., 0., 0., 256., 256.]] * 2)
        added = {"text_embeds": pooled, "time_ids": tids}
        fx.update(add_text_embeddings=pooled, add_time_ids=tids)
    for name, (specs, scales) in STACKS.items():
        torch.manual_seed(0)
        om = ounet.UNet2DConditionModel(cfg)
        synthetic.init_synthetic_(om, seed=WEIGHT_SEED)
        om.requires_grad_(False)
        om.eval()
        nets = build_networks(lora, om, specs)

        def eps():
            with torch.no_grad():
                return om(lat, fx["timestep"], ehs, added_cond_kwargs=added).sample

        case = {"specs": specs, "scales": scales, "n_lora": [len(n.unet_loras) for n in nets]}
        if "eps_off" not in fx:
            fx["eps_off"] = eps()
        for i, (net, s) in enumerate(zip(nets, scales)):
            net.set_lora_slider(s)
            with net:
                case[f"eps_solo{i}"] = eps()
        for net in nets:
            net.__enter__()
        case["eps_mix"] = eps()
        for net in nets:
            net.__exit__(None, None, None)
        fx[name] = case
    return fx


def main():
    assert rb.available(), "needs /root/reference"
    lora = rb.load("lora")
    g = torch.Generator().manual_seed(4321)
    fx = {"weight_seed": WEIGHT_SEED, "up_std": UP_STD,
          "tiny_xl": run_config(lora, "tiny_xl", g), "tiny_sd": run_config(lora, "tiny_sd", g)}
    buf = io.BytesIO()
    torch.save(fx, buf)
    assert buf.tell() < MAX_FIXTURE_BYTES, buf.tell()
    with open(os.path.join(OUT, "compose.pt"), "wb") as f:
        f.write(buf.getvalue())
    print(f"compose.pt: {buf.tell()} bytes")


if __name__ == "__main__":
    main()
