"""GPU tests of the VAE (sliders_b200/vae.py, csrc/vae.cu, the SB200_CONV_PAD_BR conv): every new kernel against a
float64 reference element by element, and whole encode / decode against the fp32 oracle (oracle/vae.py).

Per-element bounds: a bf16 output may differ from the float64 value by its own rounding (2^-8 relative, round to
nearest) plus the fp32 accumulation error, bounded by K * 2^-24 times the sum of |terms| (K the number of terms).
Each kernel's output buffer carries guard bands that must come back untouched."""
from __future__ import annotations

import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
U = 2.0 ** -24


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def _bf(t):
    return t.to(BF)


def _guarded(shape, dtype, dev, fill):
    """(buffer with 64 guard elements on each side, view of the middle)."""
    n = int(np.prod(shape))
    buf = torch.full((n + 128,), fill, dtype=dtype, device=dev)
    return buf, buf[64:64 + n].view(shape)


def _guard_intact(buf, fill):
    g = torch.cat([buf[:64], buf[-64:]])
    assert bool((g == fill).all()), "kernel wrote outside its output"


def _conv_ref(x_nhwc, w_packed, stride, pad):
    """float64 conv and the sum of |terms| per output: x NHWC, w [Cout, 3, 3, Cin]; pad = (l, r, t, b)."""
    x = x_nhwc.double().permute(0, 3, 1, 2)
    w = w_packed.double().permute(0, 3, 1, 2)
    xp = F.pad(x, pad)
    ref = F.conv2d(xp, w, stride=stride)
    absd = F.conv2d(xp.abs(), w.abs(), stride=stride)
    return ref.permute(0, 2, 3, 1), absd.permute(0, 2, 3, 1)


@pytest.mark.parametrize("B,H,W,C,Cout", [(2, 32, 32, 128, 128), (1, 64, 48, 256, 256), (1, 16, 24, 512, 512)])
def test_conv3x3_pad_bottom_right(dev, B, H, W, C, Cout):
    from sliders_b200 import ops

    g = torch.Generator(device=dev).manual_seed(B * H + C)
    x = _bf(torch.randn(B, H, W, C, device=dev, generator=g))
    w = _bf(torch.randn(Cout, 3, 3, C, device=dev, generator=g) * (9 * C) ** -0.5)
    bias = _bf(torch.randn(Cout, device=dev, generator=g) * 0.1)
    buf, out = _guarded((B, H // 2, W // 2, Cout), BF, dev, 7.0)
    ops.conv3x3(x, w, stride=2, bias=bias, pad_bottom_right=True, out=out)
    torch.cuda.synchronize()
    _guard_intact(buf, 7.0)
    ref, absd = _conv_ref(x, w, 2, (0, 1, 0, 1))
    ref = ref + bias.double()
    bound = ref.abs() * 2.0 ** -8 + 9 * C * U * (absd + bias.double().abs()) + 1e-30
    err = (out.double() - ref).abs()
    assert bool((err <= bound).all()), f"max err / bound {(err / bound).max().item():.3g}"
    # the flag changes which taps are read: the diffusers pad (0, 1, 0, 1) result differs from pad 1 on every side
    sym, _ = _conv_ref(x, w, 2, (1, 1, 1, 1))
    assert (sym + bias.double() - ref).abs().max().item() > 0.1
    # and a launch without it is still the symmetric-pad conv
    plain = ops.conv3x3(x, w, stride=2, bias=bias)
    assert ((plain.double() - sym - bias.double()).abs() <= (sym + bias.double()).abs() * 2.0 ** -8
            + 9 * C * U * (absd + 1) + 1e-30).all()


@pytest.mark.parametrize("rows,S,mag", [(64, 16384, 30.0), (200, 1024, 5.0), (3, 4096, 0.01)])
def test_softmax_rows(dev, rows, S, mag):
    from sliders_b200 import ops

    g = torch.Generator(device=dev).manual_seed(rows + S)
    C = 512
    scale = C ** -0.5
    s = torch.randn(rows, S, device=dev, generator=g) * (mag / scale)  # scaled scores of magnitude ~mag
    buf, p = _guarded((rows, S), BF, dev, 3.0)
    ops.softmax_rows(s, scale, out=p)
    torch.cuda.synchronize()
    _guard_intact(buf, 3.0)
    ref = torch.softmax(s.double() * scale, dim=-1)
    # bf16 rounding of P, plus fp32 exp of arguments up to |scale (s - max)| (their rounding: |arg| * 2^-24 relative)
    arg = ((s.double() - s.double().max(-1, keepdim=True).values) * scale).abs()
    bound = ref * (2.0 ** -8 + (arg + 8) * 4 * U + S * U) + 1e-38
    err = (p.double() - ref).abs()
    assert bool((err <= bound).all()), f"max err / bound {(err / bound).max().item():.3g}"


@pytest.mark.parametrize("B,H,W,Cout", [(2, 64, 64, 128), (1, 40, 24, 64)])
def test_vae_conv_in_u8(dev, B, H, W, Cout):
    from oracle import vae as ovae
    from sliders_b200 import ops

    g = torch.Generator(device=dev).manual_seed(H * W)
    img = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device=dev, generator=g)
    img[0, :2, :2] = 255
    img[0, -2:, -2:] = 0
    w = _bf(torch.randn(Cout, 3, 3, 3, device=dev, generator=g) * 0.2)
    bias = _bf(torch.randn(Cout, device=dev, generator=g) * 0.1)
    out = ops.vae_conv_in_u8(img, w, bias)
    torch.cuda.synchronize()
    x = ovae.preprocess(img).permute(0, 2, 3, 1)
    ref, absd = _conv_ref(x, w, 1, (1, 1, 1, 1))
    ref = ref + bias.double()
    bound = ref.abs() * 2.0 ** -8 + 30 * U * (absd + bias.double().abs() + 27) + 1e-30
    err = (out.double() - ref).abs()
    assert bool((err <= bound).all()), f"max err / bound {(err / bound).max().item():.3g}"


@pytest.mark.parametrize("B,H,W,Cin", [(2, 64, 64, 128), (1, 24, 40, 64)])
def test_vae_conv_out_u8(dev, B, H, W, Cin):
    from oracle import vae as ovae
    from sliders_b200 import ops

    g = torch.Generator(device=dev).manual_seed(H + Cin)
    x = _bf(torch.randn(B, H, W, Cin, device=dev, generator=g))
    w = _bf(torch.randn(3, 3, 3, Cin, device=dev, generator=g) * (9 * Cin) ** -0.5 * 1.5)
    bias = _bf(torch.randn(3, device=dev, generator=g) * 0.1)
    img, y = ops.vae_conv_out_u8(x, w, bias, return_float=True)
    torch.cuda.synchronize()
    ref, absd = _conv_ref(x, w, 1, (1, 1, 1, 1))
    ref = (ref + bias.double()).permute(0, 3, 1, 2)
    absd = absd.permute(0, 3, 1, 2)
    bound = 9 * Cin * U * (absd + 1) + 1e-30
    err = (y.double() - ref).abs()
    assert bool((err <= bound).all()), f"max err / bound {(err / bound).max().item():.3g}"
    # uint8: the float64 postprocess of the same conv output, except within rounding distance of a .5 boundary
    want = ovae.postprocess(ref).to(dev)
    t = ((ref / 2 + 0.5).clamp(0, 1) * 255).permute(0, 2, 3, 1)
    near = ((t - t.floor() - 0.5).abs() <= (bound.permute(0, 2, 3, 1) * 255 / 2 + 255 * 2 * U))
    ok = (img == want) | (near & ((img.double() - t).abs() <= 1.0))
    assert bool(ok.all()), f"{int((~ok).sum())} pixels differ from the postprocess"
    assert int((~near).sum()) > 0.5 * near.numel()   # the band is conservative; most pixels are still compared exactly
    assert bool((img == 0).any()) and bool((img == 255).any()), "the clamp is not exercised"


def _moments_ref(x, w, bias, qw, qb, eps, sf):
    ref, absd = _conv_ref(x, w, 1, (1, 1, 1, 1))
    h = (ref + bias.double()).permute(0, 3, 1, 2)                   # [B, 8, H, W]
    ha = (absd + bias.double().abs()).permute(0, 3, 1, 2)
    m = torch.einsum("ck,bkhw->bchw", qw.double(), h) + qb.double().view(1, 8, 1, 1)
    ma = torch.einsum("ck,bkhw->bchw", qw.double().abs(), ha) + qb.double().abs().view(1, 8, 1, 1)
    mean, logvar = m[:, :4], m[:, 4:].clamp(-30, 20)
    std = torch.exp(0.5 * logvar)
    z = mean if eps is None else mean + std * eps.double()
    # accumulation error of the conv (K = 9 Cin) carried through quant_conv; exp's error on std
    e_m = 9 * x.shape[-1] * U * ma[:, :4] * 2
    e_std = std * (0.5 * 9 * x.shape[-1] * U * ma[:, 4:] * 2 + 4 * U)
    bound = (e_m + (0 if eps is None else e_std * eps.double().abs()) + z.abs() * 4 * U) * sf + 1e-30
    return z * sf, bound


@pytest.mark.parametrize("sample", [False, True])
@pytest.mark.parametrize("B,H,W,Cin,lv_shift", [(2, 32, 32, 512, 0.0), (1, 24, 16, 128, 0.0),
                                                (1, 16, 16, 128, 100.0), (1, 16, 16, 128, -100.0)])
def test_vae_moments(dev, B, H, W, Cin, lv_shift, sample):
    from sliders_b200 import ops

    g = torch.Generator(device=dev).manual_seed(Cin + H + int(lv_shift))
    x = _bf(torch.randn(B, H, W, Cin, device=dev, generator=g))
    w = _bf(torch.randn(8, 3, 3, Cin, device=dev, generator=g) * (9 * Cin) ** -0.5)
    bias = _bf(torch.randn(8, device=dev, generator=g) * 0.1)
    qw = torch.randn(8, 8, device=dev, generator=g) * 8 ** -0.5
    qb = torch.randn(8, device=dev, generator=g) * 0.1
    qb[4:] += lv_shift                                                   # logvar far outside [-30, 20]: the clamp
    eps = torch.randn(B, 4, H, W, device=dev, generator=g) if sample else None
    sf = 0.13025
    z = ops.vae_moments(x, w, bias, qw, qb, eps, sf)
    torch.cuda.synchronize()
    ref, bound = _moments_ref(x, w, bias, qw, qb, eps, sf)
    err = (z.double() - ref).abs()
    assert bool((err <= bound).all()), f"max err / bound {(err / bound).max().item():.3g}"
    if sample and lv_shift != 0:
        std = (z.double() / sf - _moments_ref(x, w, bias, qw, qb, None, 1.0)[0]) / eps.double()
        want = np.exp(0.5 * (20.0 if lv_shift > 0 else -30.0))
        # at exp(-15) the noise term sits near the fp32 resolution of the mean, so the recovered std is only coarse
        assert abs(std.median().item() / want - 1) < (1e-3 if lv_shift > 0 else 5e-2)


def test_vae_post_quant(dev):
    from sliders_b200 import ops

    g = torch.Generator(device=dev).manual_seed(5)
    z = torch.randn(3, 4, 24, 40, device=dev, generator=g)
    pw, pb = torch.randn(4, 4, device=dev, generator=g) * 0.5, torch.randn(4, device=dev, generator=g) * 0.1
    out = ops.vae_post_quant(z, pw, pb, 0.18215)
    torch.cuda.synchronize()
    zz = z.double() / 0.18215
    ref = torch.einsum("ck,bkhw->bchw", pw.double(), zz) + pb.double().view(1, 4, 1, 1)
    absd = torch.einsum("ck,bkhw->bchw", pw.double().abs(), zz.abs()) + pb.double().abs().view(1, 4, 1, 1)
    assert bool(((out.double() - ref).abs() <= 8 * U * absd + 1e-30).all())


# ---------------------------------------------------------------------------------------------------------------------
# whole encode / decode against the fp32 oracle (run on the GPU in fp32, TF32 off)
# ---------------------------------------------------------------------------------------------------------------------
def _models(dev, which, seed=3):
    from oracle import vae as ovae
    from sliders_b200 import synthetic
    from sliders_b200 import vae as pvae

    ocfg = {"tiny": ovae.VAEConfig.tiny, "sd": ovae.VAEConfig.sd15, "sdxl": ovae.VAEConfig.sdxl}[which]()
    om = ovae.AutoencoderKL(ocfg)
    synthetic.init_synthetic_(om, seed=seed)
    om = om.to(dev).eval()
    pm = pvae.AutoencoderKL(pvae.VAEConfig(**ocfg.__dict__))
    pm.load_state_dict(om.state_dict())
    return om, pm.to(dev, BF).eval()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


# chunk: queries per mid-block attention chunk; 768 and 512 leave a partial last chunk (S = 2048 and 768 tokens)
@pytest.mark.parametrize("which,H,W,chunk", [("tiny", 64, 64, 1024), ("tiny", 64, 128, 768), ("sd", 256, 256, 1024),
                                             ("sdxl", 256, 256, 1024), ("sdxl", 256, 192, 512)])
def test_vae_matches_oracle(dev, monkeypatch, which, H, W, chunk):
    from oracle import vae as ovae
    from sliders_b200 import vae as pvae

    monkeypatch.setattr(pvae, "ATTN_CHUNK", chunk)
    om, pm = _models(dev, which)
    g = torch.Generator(device=dev).manual_seed(H + W)
    # a smooth image plus noise, so the encoder sees structure at every scale
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H, device=dev), torch.linspace(0, 1, W, device=dev), indexing="ij")
    base = torch.stack([yy, xx, (yy + xx) / 2], -1) * 200 + 20
    img = (base.unsqueeze(0).repeat(2, 1, 1, 1) + torch.randn(2, H, W, 3, device=dev, generator=g) * 20)
    img = img.clamp(0, 255).round().to(torch.uint8)
    f = pm.config.downscale
    with torch.no_grad():
        x = ovae.preprocess(img).float()
        mean = om.encode_scaled(x)
        got = pm.encode(img, sample=False)
        rel_mean = _rel(got, mean)
        gen = torch.Generator(device=dev).manual_seed(11)
        got_s = pm.encode(img, generator=gen)
        eps = torch.randn((2, 4, H // f, W // f), generator=torch.Generator(device=dev).manual_seed(11), device=dev)
        rel_sample = _rel(got_s, om.encode_scaled(x, eps))
        y_ref = om.decode_scaled(mean)
        u8, y = pm.decode(mean, return_float=True)
        rel_dec = _rel(y, y_ref)
        px = (u8.int() - ovae.postprocess(y_ref).to(dev).int()).abs()
        # the same model run by PyTorch in bf16 (what diffusers does with a bf16 VAE): the error bf16 activations cost
        ob = om.to(BF)
        rel_mean_bf = _rel(ob.encode_scaled(x.to(BF)).float(), mean)
        y_bf = ob.decode_scaled(mean.to(BF)).float()
        rel_dec_bf = _rel(y_bf, y_ref)
        px_bf = (ovae.postprocess(y_bf).int() - ovae.postprocess(y_ref).int()).abs()
    far, far_bf = (px > 2).float().mean().item(), (px_bf > 2).float().mean().item()
    print(f"{which} {H}x{W}: encode mean rel-RMS {rel_mean:.3g} (torch bf16 {rel_mean_bf:.3g}), sample {rel_sample:.3g}, "
          f"decode {rel_dec:.3g} (torch bf16 {rel_dec_bf:.3g}), pixels off by > 2 levels {far:.2e} (torch bf16 "
          f"{far_bf:.2e}), max {px.max().item()}")
    assert tuple(got.shape) == (2, 4, H // f, W // f) and tuple(u8.shape) == (2, H, W, 3)
    # The 1e-2 bar of the UNet holds for the encoder and the tiny decoder.  The full decoder measured 1.13e-2 to
    # 1.15e-2 rel-RMS, with 1.6-1.8 % of pixels more than 2 levels off (max 8), on an H100 80GB HBM3 at 700 W with
    # seeded synthetic weights.  The cause is the bf16 storage of the activations between its ~40 convolutions, not a
    # kernel: PyTorch running the oracle itself in bf16 is further off (1.47e-2, 3.6-3.9 % of pixels; printed above).
    # So the decoder may not exceed 1.3e-2 / 2 % nor the bf16 run's own distance.
    assert rel_mean <= 1e-2 and rel_sample <= 1e-2
    assert rel_dec <= max(1e-2, min(1.3e-2, rel_dec_bf))
    assert far <= max(1e-3, min(2e-2, far_bf))


def test_vae_rejects_cpu_and_bad_sizes(dev):
    from sliders_b200 import _cabi
    from sliders_b200 import vae as pvae

    m = pvae.load_vae("synthetic:2", pvae.VAEConfig.sdxl(), device=dev)
    with pytest.raises(_cabi.Sb200Error):
        pvae.load_vae("synthetic:2", pvae.VAEConfig.sdxl()).decode(torch.zeros(1, 4, 32, 32))
    with pytest.raises(ValueError):
        m.encode(torch.zeros(1, 100, 100, 3, dtype=torch.uint8, device=dev))
    imgs = m.decode(torch.randn(1, 4, 32, 32, device=dev))
    assert imgs.dtype == torch.uint8 and tuple(imgs.shape) == (1, 256, 256, 3)
    assert len(pvae.to_pil(imgs)) == 1


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def test_eval_script_writes_png_tree(dev, tmp_path):
    from sliders_b200 import lora, synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    unet = UNet2DConditionModel(UNetConfig.sdxl())
    saved = list(lora.DEFAULT_TARGET_REPLACE)
    lora.DEFAULT_TARGET_REPLACE += lora.UNET_TARGET_REPLACE_MODULE_CONV   # c3lier, as the file name says
    try:
        net = lora.LoRANetwork(unet, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn")
    finally:
        del lora.DEFAULT_TARGET_REPLACE[len(saved):]
    synthetic.init_lora_nonzero_(net, seed=1)
    ckpt = tmp_path / "ageslider_alpha1.0_rank4_noxattn_last.pt"
    torch.save(net.state_dict(), ckpt)
    csv = tmp_path / "p.csv"
    csv.write_text("case_number,prompt,evaluation_seed\n0,a photo of a person,7\n")
    out = tmp_path / "out"
    cmd = [sys.executable, os.path.join(ROOT, "eval-scripts", "generate_images_xl.py"), "--model_name", str(ckpt),
           "--prompts_path", str(csv), "--save_path", str(out), "--unet", "synthetic", "--vae", "synthetic"]
    proc = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert proc.returncode == 0, proc.stdout[-3000:]
    root = out / ckpt.name
    scales = sorted(p.name for p in root.iterdir())
    assert len(scales) == 5
    from PIL import Image

    for s in scales:
        assert (root / s / "0_0.pt").is_file()
        im = Image.open(root / s / "0_0.png")
        assert im.size == (1024, 1024) and im.mode == "RGB"


def _write_pngs(folder, names, seed):
    from PIL import Image

    folder.mkdir(parents=True, exist_ok=True)
    rng = np.random.default_rng(seed)
    for n in names:
        Image.fromarray(rng.integers(0, 256, (96, 80, 3), dtype=np.uint8)).save(folder / n)


def _image_slider_run(tmp_path, folder_main, tag, iterations, monkeypatch):
    """cli.main("image_xl") on synthetic SDXL with `--vae synthetic`; returns [(latents_low, latents_high, losses,
    lora state after the step)] per iteration."""
    import random

    import yaml

    from sliders_b200 import cli, trainer

    cfg = yaml.safe_load(open(os.path.join(ROOT, "trainscripts", "imagesliders", "data", "config-xl.yaml")))
    cfg["prompts_file"] = os.path.join(ROOT, "trainscripts", "imagesliders", "data", "prompts-xl.yaml")
    cfg["pretrained_model"]["name_or_path"] = "synthetic"
    cfg["save"].update(name=tag, path=str(tmp_path / "models"), per_steps=1000)
    cfg_file = tmp_path / f"{tag}.yaml"
    cfg_file.write_text(yaml.safe_dump(cfg))
    steps = []
    real = trainer.image_slider_step_xl

    def step(unet, network, *a, **k):
        low, high = a[4], a[5]
        losses = real(unet, network, *a, **k)
        torch.cuda.synchronize()
        steps.append((low.detach().float().cpu().clone(), high.detach().float().cpu().clone(),
                      [float(x) for x in losses], {n: p.detach().float().cpu().clone()
                                                   for n, p in network.state_dict().items()}))
        return losses

    monkeypatch.setattr(trainer, "image_slider_step_xl", step)
    random.seed(0)
    torch.manual_seed(0)
    cli.main("image_xl", ["--config_file", str(cfg_file), "--folder_main", str(folder_main), "--alpha", "1",
                          "--folders=low,high", "--scales=-1,1", "--vae", "synthetic",
                          "--iterations", str(iterations)])
    return steps


def test_image_slider_cli_trains_from_png_folders(dev, tmp_path, monkeypatch):
    imgs = tmp_path / "imgs"
    _write_pngs(imgs / "low", ["a.png"], 1)
    _write_pngs(imgs / "high", ["a.png"], 2)
    steps = _image_slider_run(tmp_path, imgs, "img", 2, monkeypatch)
    assert len(steps) == 2
    for low, high, losses, _ in steps:
        assert tuple(low.shape) == (1, 4, 64, 64) and tuple(high.shape) == (1, 4, 64, 64)   # 512 px images
        assert all(np.isfinite(losses))
    assert not torch.equal(steps[0][0], steps[1][0]), "each iteration encodes a fresh latent sample"
    ckpt = tmp_path / "models" / "img_alpha1.0_rank4_noxattn" / "img_alpha1.0_rank4_noxattn_last.pt"
    assert ckpt.is_file()

    # the first iteration's encoded latents, read back through the .pt path, give the same step bit for bit
    lats = tmp_path / "lats"
    (lats / "low").mkdir(parents=True)
    (lats / "high").mkdir(parents=True)
    torch.save(steps[0][0][0], lats / "low" / "a.pt")
    torch.save(steps[0][1][0], lats / "high" / "a.pt")
    again = _image_slider_run(tmp_path, lats, "lat", 1, monkeypatch)
    assert again[0][2] == steps[0][2]
    assert all(torch.equal(again[0][3][k], steps[0][3][k]) for k in steps[0][3])


def test_edit_example_encodes_photo_and_writes_png(dev, tmp_path):
    _write_pngs(tmp_path, ["photo.png"], 3)
    out = tmp_path / "edited"
    cmd = [sys.executable, os.path.join(ROOT, "examples", "edit_real_image_sd1.py"), "--synthetic", "--vae",
           "synthetic", "--image", str(tmp_path / "photo.png"), "--steps", "3", "--inner", "1", "--scales", "0", "2",
           "--out", str(out)]
    proc = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert proc.returncode == 0, proc.stdout[-3000:]
    from PIL import Image

    for s in ("0", "2"):
        assert (out / f"latent_scale{s}.pt").is_file()
        assert Image.open(out / f"edit_scale{s}.png").size == (512, 512)
