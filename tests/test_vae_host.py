"""CPU tests of the VAE's host side: the oracle's key layout against the diffusers config, the product tree against the
oracle, the deprecated attention-name conversion, known answers of the oracle's pad / clamp / postprocess, `--vae`
resolution, the image-slider CLI's image-pair listing, and that every VAE entry point of include/sb200_vae.h has an element-wise GPU test."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import vae as ovae  # noqa: E402
from sliders_b200 import vae as pvae  # noqa: E402


@pytest.mark.parametrize("cfg", ["sd15", "sdxl"])
def test_oracle_key_layout_and_parameter_count(cfg):
    om = ovae.AutoencoderKL(getattr(ovae.VAEConfig, cfg)())
    sd = om.state_dict()
    # stabilityai/sd-vae-ft-mse and sdxl-vae share the architecture: 248 tensors, 83 653 863 parameters
    assert len(sd) == 248 and sum(v.numel() for v in sd.values()) == 83_653_863
    assert om.config.scaling_factor == {"sd15": 0.18215, "sdxl": 0.13025}[cfg]
    want = {
        "encoder.conv_in.weight": (128, 3, 3, 3),
        "encoder.down_blocks.1.resnets.0.conv_shortcut.weight": (256, 128, 1, 1),
        "encoder.down_blocks.2.downsamplers.0.conv.weight": (512, 512, 3, 3),
        "encoder.mid_block.attentions.0.group_norm.weight": (512,),
        "encoder.mid_block.attentions.0.to_q.weight": (512, 512),
        "encoder.mid_block.attentions.0.to_out.0.bias": (512,),
        "encoder.conv_out.weight": (8, 512, 3, 3),
        "quant_conv.weight": (8, 8, 1, 1),
        "post_quant_conv.weight": (4, 4, 1, 1),
        "decoder.conv_in.weight": (512, 4, 3, 3),
        "decoder.up_blocks.0.resnets.2.conv2.weight": (512, 512, 3, 3),
        "decoder.up_blocks.2.resnets.0.conv_shortcut.weight": (256, 512, 1, 1),
        "decoder.up_blocks.2.upsamplers.0.conv.weight": (256, 256, 3, 3),
        "decoder.up_blocks.3.resnets.0.conv_shortcut.weight": (128, 256, 1, 1),
        "decoder.conv_norm_out.weight": (128,),
        "decoder.conv_out.weight": (3, 128, 3, 3),
    }
    for k, shape in want.items():
        assert tuple(sd[k].shape) == shape, k
    assert not any("downsamplers" in k for k in sd if k.startswith("encoder.down_blocks.3"))
    assert not any("upsamplers" in k for k in sd if k.startswith("decoder.up_blocks.3"))
    assert sum(1 for k in sd if k.startswith("decoder.up_blocks.0.resnets.") and k.endswith("conv1.weight")) == 3


@pytest.mark.parametrize("cfg", ["sd15", "sdxl", "tiny"])
def test_product_tree_matches_oracle(cfg):
    ocfg = getattr(ovae.VAEConfig, cfg)()
    o = ovae.AutoencoderKL(ocfg).state_dict()
    p = pvae.AutoencoderKL(pvae.VAEConfig(**ocfg.__dict__)).state_dict()
    assert list(o) == list(p)
    assert all(o[k].shape == p[k].shape for k in o)


def test_deprecated_attention_names_convert():
    sd = {"encoder.mid_block.attentions.0.query.weight": 1, "encoder.mid_block.attentions.0.query.bias": 2,
          "decoder.mid_block.attentions.0.key.weight": 3, "decoder.mid_block.attentions.0.value.bias": 4,
          "decoder.mid_block.attentions.0.proj_attn.weight": 5, "decoder.mid_block.attentions.0.group_norm.weight": 6,
          "encoder.down_blocks.0.resnets.0.conv1.weight": 7}
    out = pvae.convert_deprecated_attention(sd)
    assert out == {"encoder.mid_block.attentions.0.to_q.weight": 1, "encoder.mid_block.attentions.0.to_q.bias": 2,
                   "decoder.mid_block.attentions.0.to_k.weight": 3, "decoder.mid_block.attentions.0.to_v.bias": 4,
                   "decoder.mid_block.attentions.0.to_out.0.weight": 5,
                   "decoder.mid_block.attentions.0.group_norm.weight": 6,
                   "encoder.down_blocks.0.resnets.0.conv1.weight": 7}


def test_load_vae_converts_and_rejects(tmp_path):
    m = pvae.AutoencoderKL(pvae.VAEConfig.sd15())
    sd = {k: torch.zeros_like(v) for k, v in m.state_dict().items()}
    old = {k.replace(".to_q.", ".query.").replace(".to_out.0.", ".proj_attn."): v for k, v in sd.items()}
    torch.save(old, tmp_path / "old.pt")
    loaded = pvae.load_vae(str(tmp_path / "old.pt"), pvae.VAEConfig.sd15(), dtype=torch.float32)
    assert set(loaded.state_dict()) == set(sd)
    bad = dict(sd)
    bad["quant_conv.weight"] = torch.zeros(8, 8)
    torch.save(bad, tmp_path / "bad.pt")
    with pytest.raises(RuntimeError, match="quant_conv.weight has shape"):
        pvae.load_vae(str(tmp_path / "bad.pt"), pvae.VAEConfig.sd15())
    del bad["quant_conv.weight"]
    torch.save(bad, tmp_path / "missing.pt")
    with pytest.raises(RuntimeError, match="missing 1"):
        pvae.load_vae(str(tmp_path / "missing.pt"), pvae.VAEConfig.sd15())


def test_downsample_pads_bottom_right_only():
    d = ovae.Downsample2D(1)
    with torch.no_grad():
        d.conv.weight.fill_(1.0)
        d.conv.bias.zero_()
    out = d(torch.ones(1, 1, 4, 4))
    # taps read rows / cols 2i .. 2i+2: the last output row / column reaches the zero pad, the first does not
    assert out[0, 0].tolist() == [[9.0, 6.0], [6.0, 4.0]]


def test_logvar_clamp():
    m = ovae.AutoencoderKL(ovae.VAEConfig.tiny())
    with torch.no_grad():
        m.quant_conv.weight.zero_()
        m.quant_conv.bias.copy_(torch.tensor([0.5, 0, 0, 0, 100.0, -100.0, 3.0, 0]))
    mean, logvar = m.moments(torch.zeros(1, 3, 8, 8))
    assert logvar[0, :, 0, 0].tolist() == [20.0, -30.0, 3.0, 0.0]
    eps = torch.ones(1, 4, 4, 4)
    z = m.encode_scaled(torch.zeros(1, 3, 8, 8), eps)
    assert torch.allclose(z[0, :, 0, 0], (torch.tensor([0.5, 0, 0, 0]) + torch.exp(0.5 * torch.tensor(
        [20.0, -30.0, 3.0, 0.0]))) * 0.18215)


def test_pre_and_postprocess_known_answers():
    img = torch.tensor([[[[0, 255, 51]]]], dtype=torch.uint8)
    assert ovae.preprocess(img).flatten().tolist() == [-1.0, 1.0, 51 / 255 * 2 - 1]
    # clamp at both ends, plain rounding away from ties
    y = torch.tensor([-3.0, 3.0, 0.0, -0.5, 0.5], dtype=torch.float32).view(1, 5, 1, 1).expand(1, 5, 1, 3)
    y = y.permute(0, 3, 1, 2)  # NCHW [1, 3, 5, 1]
    assert ovae.postprocess(y)[0, :, 0, 0].tolist() == [0, 255, 128, 64, 191]   # 127.5 -> 128, 63.75, 191.25
    # exact ties of fp32 (y / 2 + 0.5) * 255 round half to even, as numpy's round in numpy_to_pil
    ties = []
    for k in range(255):
        yk = torch.tensor((k + 0.5) / 255 * 2 - 1, dtype=torch.float32)
        if ((yk / 2 + 0.5) * 255).item() == k + 0.5:
            ties.append((yk.item(), k))
    assert sum(k % 2 == 1 for _, k in ties) >= 3
    yt = torch.tensor([v for v, _ in ties], dtype=torch.float32).view(1, 1, -1, 1).expand(1, 3, -1, 1)
    got = ovae.postprocess(yt)[0, :, 0, 0].tolist()
    assert got == [k + (k % 2) for _, k in ties]
    assert ovae.postprocess(y).dtype == torch.uint8


def test_vae_source_resolution(tmp_path):
    assert pvae.resolve_vae_source("none", str(tmp_path)) is None
    assert pvae.resolve_vae_source(None, str(tmp_path)) is None
    assert pvae.resolve_vae_source("synthetic:3", "synthetic") == "synthetic:3"
    assert pvae.resolve_vae_source("auto", "synthetic") is None
    assert pvae.resolve_vae_source("auto", str(tmp_path)) is None            # a directory without vae/
    (tmp_path / "vae").mkdir()
    f = tmp_path / "vae" / "diffusion_pytorch_model.safetensors"
    f.write_bytes(b"")
    assert pvae.resolve_vae_source("auto", str(tmp_path)) == str(f)
    assert pvae.resolve_vae_source(str(tmp_path), "synthetic") == str(tmp_path)
    from sliders_b200 import eval_sweep as es

    args = es.parse_args(["--model_name", "x.pt", "--prompts_path", "p.csv", "--save_path", "o"])
    assert args.vae == "auto"
    assert es.parse_args(["--model_name", "x.pt", "--prompts_path", "p.csv", "--save_path", "o", "--vae",
                          "synthetic:2"]).vae == "synthetic:2"


def test_image_pair_listing(tmp_path):
    from sliders_b200 import cli

    for sub, names in (("low", ["b.png", "a.JPG", "c.webp", "notes.txt"]), ("high", ["a.JPG", "b.png", "c.webp"])):
        (tmp_path / sub).mkdir()
        for n in names:
            (tmp_path / sub / n).write_bytes(b"")
    assert cli.list_image_pairs(str(tmp_path), "low", "high") == ["a.JPG", "b.png", "c.webp"]
    (tmp_path / "high" / "c.webp").unlink()
    with pytest.raises(FileNotFoundError, match="no c.webp"):
        cli.list_image_pairs(str(tmp_path), "low", "high")
    # without a VAE the .pt listing keeps its error for image-only folders
    with pytest.raises(FileNotFoundError, match="encode them with the SD VAE"):
        cli.list_pairs(str(tmp_path), "low", "high")
    assert cli.build_parser("image_xl").parse_args(["--config_file", "x", "--folder_main", "d", "--alpha", "1"]).vae \
        == "auto"


VAE_COVERAGE = {
    "sb200_vae_conv_in_u8": ["test_gpu_vae.py::test_vae_conv_in_u8"],
    "sb200_vae_conv_out_u8": ["test_gpu_vae.py::test_vae_conv_out_u8"],
    "sb200_vae_moments": ["test_gpu_vae.py::test_vae_moments"],
    "sb200_vae_post_quant": ["test_gpu_vae.py::test_vae_post_quant"],
    "sb200_softmax_rows": ["test_gpu_vae.py::test_softmax_rows"],
}


def test_every_vae_entry_point_has_an_element_wise_test():
    """A new `int sb200_*(` entry point in include/sb200_vae.h cannot land without a line here naming its
    element-by-element test, every named test must exist, and every entry point is bound by _cabi."""
    import ast
    import re

    from sliders_b200 import _cabi

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "sb200_vae.h")) as f:
        declared = set(re.findall(r"\bint\s+(sb200_\w+)\s*\(", f.read()))
    assert declared == set(VAE_COVERAGE)
    assert declared <= set(_cabi.SIGNATURES)
    if not os.path.exists(_cabi.lib_path()):
        import __graft_entry__ as ge

        ge.build()
    lib = _cabi.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/sb200_vae.h but not exported by libsb200.so"
    with open(os.path.join(root, "tests", "test_gpu_vae.py")) as f:
        funcs = {n.name for n in ast.walk(ast.parse(f.read())) if isinstance(n, ast.FunctionDef)}
    for tests in VAE_COVERAGE.values():
        for ref in tests:
            assert ref.split("::")[1] in funcs, ref
