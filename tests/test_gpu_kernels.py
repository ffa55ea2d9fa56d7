"""GPU parity tests of the individual sm_90a kernels, called through the C ABI (sliders_b200.ops) and compared
with fp32 torch math on the same bf16 inputs.  Tolerances: outputs are bf16 (relative rounding 2^-9 = 0.2 %), so
rel-RMS <= 1e-2 catches any indexing / accumulation error while allowing output rounding; attention additionally
rounds P to bf16 (standard flash attention), tolerance 2e-2.  Both GEMM flavours (single CTA and the
two-CTA cluster that multicasts the weight tile) are forced explicitly."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
SINGLE, PAIR = 0x2000, 0x1000


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def rel_rms(got, ref):
    got, ref = got.float(), ref.float()
    assert torch.isfinite(got).all()
    return ((got - ref).norm() / (ref.norm() + 1e-12)).item()


def make_lora(K, N, r, group_n, dev, seed, conv_cin=None):
    from sliders_b200.ops import Lora

    g = torch.Generator().manual_seed(seed)
    groups = (N + group_n - 1) // group_n
    rt = 16 if groups * r <= 16 else 32
    down = torch.zeros(rt, K)
    down[: groups * r] = torch.randn(groups * r, K, generator=g) / K ** 0.5
    up = (torch.randn(N, r, generator=g) * 0.5).to(BF).float()
    down = down.to(dev, BF)
    up = up.to(dev)
    return down, up, rt


@pytest.mark.parametrize("force", [SINGLE, PAIR, 0])
@pytest.mark.parametrize("M,N,K,flags,split,lora", [
    (128, 64, 64, "", 0, None),                 # one tile, one k-block
    (1000, 640, 640, "bR", 0, None),            # ragged M, bias + residual
    (154, 1280, 2048, "", 0, None),             # cross-attention K/V projection shape (77 x 2)
    (2048, 2560, 640, "bG", 0, None),           # GEGLU
    (1024, 640, 1920, "b", 1280, None),         # skip-concat split K (conv_shortcut)
    (1024, 1280, 1280, "bL", 0, (4, 1280, 0.25)),
    (1024, 1920, 640, "L", 0, (4, 640, 1.0)),   # fused to_q|to_k|to_v, three adaptors
    (512, 640, 640, "bRL", 0, (8, 640, -2.0)),  # rank 8, negative slider
    (4096, 1280, 1280, "btR", 0, None),         # row bias (time embedding) + residual
    (300, 3840, 1280, "L", 0, (4, 1280, 1.0)),  # fused QKV at SDXL width: the pair interleaves W / LoRA halves
    (640, 2560, 640, "bRL", 0, (8, 1280, 0.5)), # rank 8, two adaptors, rt = 16: one adaptor per pair half
    (129, 320, 320, "bRL", 0, (4, 320, 1.0)),   # odd number of 128-row sub-tiles: phantom half of the last pair
])
def test_gemm(dev, force, M, N, K, flags, split, lora):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).to(dev, BF)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, BF)
    geglu = "G" in flags
    nout = N // 2 if geglu else N
    bias = torch.randn(N, generator=g).to(dev, BF) if "b" in flags else None
    rpb = max(1, M // 4)
    rowbias = torch.randn((M + rpb - 1) // rpb, nout, generator=g).to(dev, BF) if "t" in flags else None
    resid = torch.randn(M, nout, generator=g).to(dev, BF) if "R" in flags else None
    la = None
    if lora:
        r, group_n, scale = lora
        down, up, rt = make_lora(K, N, r, group_n, dev, 7)
        la = ops.Lora(down, up, r, group_n, scale)
    x0, x1 = (x[:, :split].contiguous(), x[:, split:].contiguous()) if split else (x, None)
    out = ops.gemm(x0, w, bias=bias, rowbias=rowbias, rows_per_batch=rpb, resid=resid, geglu=geglu, lora=la, x1=x1,
                   bn=force)
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t()
    if lora:
        t = x.float() @ down.float().t()
        for g0 in range(0, N, group_n):
            grp = g0 // group_n
            ref[:, g0:g0 + group_n] += (t[:, grp * r:(grp + 1) * r] @ up[g0:g0 + group_n].t()) * scale
    if bias is not None:
        ref = ref + bias.float()
    if geglu:
        a, gate = ref.chunk(2, dim=-1)
        ref = a * F.gelu(gate)
    if rowbias is not None:
        ref = ref + rowbias.float()[torch.arange(M, device=dev) // rpb]
    if resid is not None:
        ref = ref + resid.float()
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("force", [SINGLE, PAIR, 0])
@pytest.mark.parametrize("B,H,W,C0,C1,Cout,stride,flags,lora", [
    (1, 32, 32, 64, 0, 64, 1, "", None),
    (1, 64, 64, 320, 0, 320, 1, "bt", None),       # conv1 of a ResnetBlock2D: + time-embedding row bias
    (1, 128, 128, 320, 0, 320, 1, "bR", None),     # conv2: + residual, one image row per tile
    (2, 32, 32, 1280, 640, 1280, 1, "b", None),    # skip-connection concat as two sources
    (2, 64, 64, 320, 0, 320, 2, "b", None),        # Downsample2D (stride 2, parity planes)
    (2, 32, 32, 640, 0, 640, 1, "bL", (4, 0.5)),   # LoRA conv: down 3x3 folded in, up 1x1 in the epilogue
    (3, 8, 8, 128, 0, 128, 1, "b", None),          # 8x8 level: tiles span images, ragged M
    (1, 16, 16, 128, 64, 64, 1, "b", None),
    # patches that overhang the image (dynamic_resolution buckets, non-square eval sizes: ADVICE r1 #1)
    (1, 72, 72, 64, 0, 64, 1, "bR", None),         # W = 72: one 72-pixel row per 128-row tile
    (2, 36, 88, 128, 0, 128, 1, "bt", (4, 0.5)),   # 36 x 88, LoRA + time-embedding bias
    (1, 18, 18, 128, 64, 64, 1, "b", None),        # 18 x 18 with a skip concat (7 rows of 18 per tile)
    (3, 9, 11, 64, 0, 64, 1, "bR", None),          # 99-pixel images: one (ragged) image per tile
    (2, 72, 104, 64, 0, 64, 2, "b", None),         # stride 2 to 36 x 52
    (1, 96, 160, 64, 0, 64, 1, "b", None),         # W > 128 and not a multiple of it
    (5, 4, 4, 64, 0, 64, 1, "bt", None),           # 8 images per tile, 5 in the batch
])
def test_conv3x3(dev, force, B, H, W, C0, C1, Cout, stride, flags, lora):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(B * H + C0 + Cout)
    Cin = C0 + C1
    x = torch.randn(B, H, W, Cin, generator=g).to(dev, BF)
    w = (torch.randn(Cout, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5).to(dev, BF)
    Ho, Wo = H // stride, W // stride
    bias = torch.randn(Cout, generator=g).to(dev, BF) if "b" in flags else None
    rowbias = torch.randn(B, Cout, generator=g).to(dev, BF) if "t" in flags else None
    resid = torch.randn(B, Ho, Wo, Cout, generator=g).to(dev, BF) if "R" in flags else None
    la = None
    if lora:
        r, scale = lora
        down, up, rt = make_lora(9 * Cin, Cout, r, Cout, dev, 9)
        la = ops.Lora(down, up, r, Cout, scale)
    x0 = x[..., :C0].contiguous()
    x1 = x[..., C0:].contiguous() if C1 else None
    out = ops.conv3x3(x0, w, x1=x1, stride=stride, bias=bias, rowbias=rowbias, resid=resid, lora=la, bn=force)
    torch.cuda.synchronize()
    xn = x.float().permute(0, 3, 1, 2)
    ref = F.conv2d(xn, w.float().permute(0, 3, 1, 2), None, stride=stride, padding=1)
    if lora:
        dn = down.float().view(-1, 3, 3, Cin).permute(0, 3, 1, 2)
        t = F.conv2d(xn, dn, None, stride=stride, padding=1)
        ref = ref + torch.einsum("brhw,or->bohw", t[:, :r], up) * scale
    ref = ref.permute(0, 2, 3, 1)
    if bias is not None:
        ref = ref + bias.float()
    if rowbias is not None:
        ref = ref + rowbias.float()[:, None, None, :]
    if resid is not None:
        ref = ref + resid.float()
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("B,heads,Sq,Skv,fused", [
    (1, 1, 128, 128, False), (2, 5, 1024, 1024, True), (2, 4, 1024, 77, False),  # cross-attention: 77 keys
    (1, 2, 64, 64, True),      # Sq, Skv below one tile
    (1, 3, 320, 200, False),   # ragged queries and keys
    (1, 10, 4096, 4096, True),  # SDXL 64x64 level
    (1, 3, 700, 600, False),   # ping-pong kernel (two query tiles per CTA): ragged last CTA, partial last key tile
    (2, 2, 300, 520, False),   # second query tile of the last CTA entirely out of range
    (1, 2, 1024, 513, False),  # one key in the last tile
])
def test_attention(dev, B, heads, Sq, Skv, fused):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(Sq + Skv)
    Cc = heads * 64
    if fused:
        qkv = torch.randn(B * Sq, 3 * Cc, generator=g).to(dev, BF)
        q, k, v = qkv[:, :Cc], qkv[:, Cc:2 * Cc], qkv[:, 2 * Cc:]
    else:
        q = torch.randn(B * Sq, Cc, generator=g).to(dev, BF)
        kv = torch.randn(B * Skv, 2 * Cc, generator=g).to(dev, BF)
        k, v = kv[:, :Cc], kv[:, Cc:]
    out = ops.attention(q, k, v, B, heads, Sq, Skv, 0.125)
    torch.cuda.synchronize()
    qf = q.float().reshape(B, Sq, heads, 64).transpose(1, 2)
    kf = k.float().reshape(B, Skv, heads, 64).transpose(1, 2)
    vf = v.float().reshape(B, Skv, heads, 64).transpose(1, 2)
    ref = (torch.softmax(qf @ kf.transpose(-1, -2) * 0.125, dim=-1) @ vf).transpose(1, 2).reshape(B * Sq, Cc)
    assert rel_rms(out, ref) < 2e-2


def test_attention_softmax_rows_sum_to_one(dev):
    """Size-independent property: with V = 1 the output is exactly the row sum of P / l = 1."""
    from sliders_b200 import ops

    B, heads, S = 2, 4, 1024
    g = torch.Generator().manual_seed(0)
    q = (torch.randn(B * S, heads * 64, generator=g) * 3).to(dev, BF)
    k = (torch.randn(B * S, heads * 64, generator=g) * 3).to(dev, BF)
    v = torch.ones(B * S, heads * 64, device=dev, dtype=BF)
    out = ops.attention(q, k, v, B, heads, S, S, 0.125)
    assert (out.float() - 1).abs().max().item() < 2e-2


def test_attention_growing_logits_rescale(dev):
    """Keys ordered so the row maximum keeps growing tile after tile (by much more than the 2^8 lazy-rescale
    threshold): every key tile triggers the accumulator rescale, in both forward kernels, and the log-sum-exp the
    backward pass consumes matches."""
    from sliders_b200 import ops

    B, heads, S = 1, 2, 1024
    g = torch.Generator().manual_seed(5)
    q = torch.randn(B * S, heads * 64, generator=g).abs()
    k = torch.randn(B * S, heads * 64, generator=g).abs() * torch.linspace(0.2, 6.0, S).repeat(B)[:, None]
    v = torch.randn(B * S, heads * 64, generator=g)
    q, k, v = q.to(dev, BF), k.to(dev, BF), v.to(dev, BF)
    lse = torch.empty(B, heads, S, device=dev, dtype=torch.float32)
    out = ops.attention(q, k, v, B, heads, S, S, 0.125, lse=lse)
    qf = q.float().reshape(B, S, heads, 64).transpose(1, 2)
    kf = k.float().reshape(B, S, heads, 64).transpose(1, 2)
    vf = v.float().reshape(B, S, heads, 64).transpose(1, 2)
    sc = qf @ kf.transpose(-1, -2) * 0.125
    assert (sc.amax(-1)[..., None] - sc[..., :128].amax(-1)[..., None]).min().item() > 16   # the max really grows
    ref = (torch.softmax(sc, dim=-1) @ vf).transpose(1, 2).reshape(B * S, heads * 64)
    assert rel_rms(out, ref) < 2e-2
    ref_lse = torch.logsumexp(sc, dim=-1) * 1.4426950408889634
    assert (lse - ref_lse).abs().max().item() < 5e-2


@pytest.mark.parametrize("B,HW,C0,C1,silu,eps", [(2, 1024, 320, 0, True, 1e-5), (2, 4096, 640, 320, True, 1e-5),
                                                (1, 16384, 320, 0, False, 1e-6), (3, 64, 64, 64, True, 1e-5),
                                                (2, 256, 1280, 640, True, 1e-5)])  # 1920/32 = 60: groups straddle
def test_groupnorm(dev, B, HW, C0, C1, silu, eps):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(HW + C0)
    Cc = C0 + C1
    x = (torch.randn(B, HW, Cc, generator=g) * 2 + 0.5).to(dev, BF)
    gamma = (1 + 0.1 * torch.randn(Cc, generator=g)).to(dev, BF)
    beta = (0.1 * torch.randn(Cc, generator=g)).to(dev, BF)
    x0 = x[..., :C0].contiguous()
    x1 = x[..., C0:].contiguous() if C1 else None
    out = ops.groupnorm(x0, gamma, beta, 32, eps, silu, x1=x1)
    out2 = ops.groupnorm(x0, gamma, beta, 32, eps, silu, x1=x1)
    torch.cuda.synchronize()
    ref = F.group_norm(x.float().transpose(1, 2), 32, gamma.float(), beta.float(), eps).transpose(1, 2)
    if silu:
        ref = F.silu(ref)
    assert rel_rms(out, ref) < 1e-2
    assert torch.equal(out, out2)  # atomic-free reduction: bit-reproducible


@pytest.mark.parametrize("M,Cc", [(2048, 640), (1000, 1280), (77, 128), (33, 320)])
def test_layernorm(dev, M, Cc):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(M)
    x = (torch.randn(M, Cc, generator=g) * 3 - 1).to(dev, BF)
    gamma = (1 + 0.1 * torch.randn(Cc, generator=g)).to(dev, BF)
    beta = (0.1 * torch.randn(Cc, generator=g)).to(dev, BF)
    out = ops.layernorm(x, gamma, beta, 1e-5)
    ref = F.layer_norm(x.float(), (Cc,), gamma.float(), beta.float(), 1e-5)
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("M,N,K,act_in,act_out,lora,resid", [
    (2, 1280, 320, False, 1, None, False), (8, 1280, 2816, False, 1, None, False),
    (4, 640, 1280, True, 0, None, False), (16, 320, 1280, False, 0, (4, 0.5), False),
    (3, 1280, 1280, True, 0, (8, -1.5), False), (2, 1280, 1280, False, 2, None, True),
])
def test_small_linear(dev, M, N, K, act_in, act_out, lora, resid):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(M + N)
    x = torch.randn(M, K, generator=g).to(dev, BF)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, BF)
    b = torch.randn(N, generator=g).to(dev, BF)
    res = torch.randn(M, N, generator=g).to(dev, BF) if resid else None
    la = None
    if lora:
        r, scale = lora
        down, up, rt = make_lora(K, N, r, N, dev, 5)
        la = ops.Lora(down, up, r, N, scale)
    out = ops.small_linear(x, w, b, act_in=act_in, act_out=act_out, lora=la, resid=res)
    xin = F.silu(x.float()).to(BF).float() if act_in else x.float()
    ref = xin @ w.float().t() + b.float()
    if lora:
        ref = ref + (xin @ down.float()[:r].t()) @ up.t() * scale
    if act_out == 1:
        ref = F.silu(ref)
    if res is not None:
        ref = ref + res.float()
    if act_out == 2:
        ref = F.silu(ref.to(BF).float())
    assert rel_rms(out, ref) < 1e-2


def test_sinusoid_conv_in_out_upsample_cfg_ddim(dev):
    from sliders_b200 import ops

    vals = torch.tensor([0.0, 1.0, 500.0, 999.0, 1024.0], device=dev)
    out = ops.sinusoid(vals, 320)
    freqs = torch.exp(-math.log(10000.0) * torch.arange(160, device=dev, dtype=torch.float32) / 160)
    arg = vals[:, None] * freqs[None]
    assert rel_rms(out, torch.cat([torch.cos(arg), torch.sin(arg)], -1)) < 5e-3
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(2, 4, 32, 32, generator=g).to(dev)
    w = (torch.randn(320, 3, 3, 4, generator=g) / 6).to(dev, BF)
    b = torch.randn(320, generator=g).to(dev, BF)
    ref = F.conv2d(lat.to(BF).float(), w.float().permute(0, 3, 1, 2), b.float(), padding=1).permute(0, 2, 3, 1)
    assert rel_rms(ops.conv_in(lat, w, b), ref) < 1e-2
    assert rel_rms(ops.conv_in(lat.to(BF), w, b), ref) < 1e-2
    x = torch.randn(2, 32, 32, 320, generator=g).to(dev, BF)
    w = (torch.randn(4, 3, 3, 320, generator=g) / 54).to(dev, BF)
    b = torch.randn(4, generator=g).to(dev, BF)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b.float(), padding=1)
    assert rel_rms(ops.conv_out(x, w, b, out_dtype=torch.float32), ref) < 1e-5
    assert rel_rms(ops.conv_out(x, w, b), ref) < 1e-2
    x = torch.randn(2, 8, 8, 64, generator=g).to(dev, BF)
    assert torch.equal(ops.upsample2x(x), x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))
    n = 2 * 4 * 32 * 32
    eps2 = torch.randn(2, 2, 4, 32, 32, generator=g).reshape(4, 4, 32, 32).to(dev, BF)
    xx = torch.randn(2, 4, 32, 32, generator=g).to(dev)
    e, xp = ops.cfg_ddim(eps2, 3.0, xx, 0.3, 0.5)
    eu, ec = eps2[:2].float(), eps2[2:].float()
    er = eu + 3.0 * (ec - eu)
    assert rel_rms(e, er) < 1e-6
    x0 = (xx - (1 - 0.3) ** 0.5 * er) / 0.3 ** 0.5
    assert rel_rms(xp, 0.5 ** 0.5 * x0 + 0.5 ** 0.5 * er) < 1e-6
    # idempotence-style property: guidance 1 returns the conditional half (train_util.py:250-253)
    e1, _ = ops.cfg_ddim(eps2, 1.0)
    assert torch.allclose(e1.float(), ec, atol=1e-2)


def test_bad_arguments_return_errors_not_crashes(dev):
    from sliders_b200 import _cabi, ops

    x = torch.zeros(128, 60, device=dev, dtype=BF)  # K = 60 is not a multiple of 8
    w = torch.zeros(64, 60, device=dev, dtype=BF)
    with pytest.raises(_cabi.Sb200Error, match="multiples of 8"):
        ops.gemm(x, w)
    with pytest.raises(_cabi.Sb200Error, match="multiples of 64"):   # channels are the only conv shape constraint left
        ops.conv3x3(torch.zeros(1, 96, 96, 40, device=dev, dtype=BF), torch.zeros(64, 3, 3, 40, device=dev, dtype=BF))
    with pytest.raises(_cabi.Sb200Error, match="stride 2 needs even dims"):
        ops.conv3x3(torch.zeros(1, 9, 9, 64, device=dev, dtype=BF), torch.zeros(64, 3, 3, 64, device=dev, dtype=BF), stride=2)
    with pytest.raises(_cabi.Sb200Error, match="CUDA tensors"):
        ops.layernorm(torch.zeros(4, 64, dtype=BF), torch.zeros(64, dtype=BF), torch.zeros(64, dtype=BF))


@pytest.mark.parametrize("B,heads,Sq,Skv,d", [
    (2, 8, 4096, 4096, 40),   # SD1.x 64x64 level
    (2, 8, 1024, 77, 40),
    (2, 8, 1024, 1024, 80),   # 32x32 level
    (2, 8, 256, 256, 160),    # 16x16 level
    (3, 8, 64, 64, 160),      # 8x8 level: fewer queries / keys than a tile
    (2, 8, 256, 77, 160),
    (1, 5, 320, 200, 24),     # any multiple of 8 works
])
def test_attention_sd1_head_dims(dev, B, heads, Sq, Skv, d):
    """Head dims that are not 64: the kernel pads the head to 64 / 128 / 192 columns with TMA zero fill."""
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(Sq + d)
    Cc = heads * d
    q = torch.randn(B * Sq, Cc, generator=g).to(dev, BF)
    kv = torch.randn(B * Skv, 2 * Cc, generator=g).to(dev, BF)
    k, v = kv[:, :Cc], kv[:, Cc:]
    scale = d ** -0.5
    out = ops.attention(q, k, v, B, heads, Sq, Skv, scale, head_dim=d)
    torch.cuda.synchronize()
    qf = q.float().reshape(B, Sq, heads, d).transpose(1, 2)
    kf = k.float().reshape(B, Skv, heads, d).transpose(1, 2)
    vf = v.float().reshape(B, Skv, heads, d).transpose(1, 2)
    ref = (torch.softmax(qf @ kf.transpose(-1, -2) * scale, dim=-1) @ vf).transpose(1, 2).reshape(B * Sq, Cc)
    assert rel_rms(out, ref) < 2e-2


@pytest.mark.parametrize("force", [SINGLE, PAIR, 0])
@pytest.mark.parametrize("M,C_,N,geglu,lora,resid", [
    (1000, 640, 1920, False, (4, 640, 1.0), False),    # norm1 -> fused q|k|v with three adaptors
    (2048, 1280, 1280, False, None, True),             # norm2 -> attn2.to_q; the producer carries bias + residual
    (512, 640, 5120, True, None, True),                # norm3 -> GEGLU
    (300, 320, 960, False, (8, 320, -0.5), False),     # rank 8, ragged M
])
def test_layernorm_folded_into_projection(dev, force, M, C_, N, geglu, lora, resid):
    """sb200_gemm_ln: a GEMM leaves per-row (sum, sum of squares) of the stream it writes; the next projection consumes
    LayerNorm(stream) without a LayerNorm launch (gamma folded into W, mean / rstd applied in the epilogue)."""
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(M + C_ + N)
    # producer: stream = a @ wp^T + bp (+ r), written by the kernel together with its row statistics
    a = torch.randn(M, 256, generator=g).to(dev, BF)
    wp = (torch.randn(C_, 256, generator=g) / 16).to(dev, BF)
    bp = (torch.randn(C_, generator=g) * 3).to(dev, BF)          # a large row mean stresses E[x^2] - mean^2
    r = torch.randn(M, C_, generator=g).to(dev, BF) if resid else None
    cap = (C_ + 15) // 16
    stats = torch.full((M * cap * 2,), float("nan"), device=dev)
    x = ops.gemm(a, wp, bias=bp, resid=r, rowstats=stats, bn=force)
    parts = ops.last_rowstats_parts
    assert 0 < parts <= cap
    st = stats[: M * parts * 2].view(parts, M, 2).double().sum(0)
    xf = x.double()
    assert torch.allclose(st[:, 0], xf.sum(1), rtol=1e-4, atol=1e-2)
    assert torch.allclose(st[:, 1], (xf * xf).sum(1), rtol=1e-4, atol=1e-2)
    # consumer
    gamma = (1 + 0.3 * torch.randn(C_, generator=g)).to(dev)
    beta = (0.2 * torch.randn(C_, generator=g)).to(dev)
    w = (torch.randn(N, C_, generator=g) / C_ ** 0.5).to(dev, BF)
    b = torch.randn(N, generator=g).to(dev, BF).float()
    wq = (w.float() * gamma[None, :]).to(BF).contiguous()
    c = wq.float().sum(1).contiguous()
    d = (w.float() @ beta + b).contiguous()
    la = cl = dl = None
    if lora:
        rr, group_n, scale = lora
        down, up, rt = make_lora(C_, N, rr, group_n, dev, 5)
        downq = (down.float() * gamma[None, :]).to(BF).contiguous()
        la = ops.Lora(downq, up, rr, group_n, scale)
        cl, dl = downq.float().sum(1).contiguous(), (down.float() @ beta).contiguous()
    fold = ops.LnFold(stats, parts, C_, 1e-5, c, d, cl, dl)
    out = ops.gemm(x, wq, geglu=geglu, lora=la, ln=fold, bn=force)
    torch.cuda.synchronize()
    n = F.layer_norm(x.float(), (C_,), gamma, beta, 1e-5)
    ref = n @ w.float().t() + b
    if lora:
        t = n @ down.float().t()
        for g0 in range(0, N, group_n):
            grp = g0 // group_n
            ref[:, g0:g0 + group_n] += (t[:, grp * rr:(grp + 1) * rr] @ up[g0:g0 + group_n].t()) * scale
    if geglu:
        v, gate = ref.chunk(2, dim=-1)
        ref = v * F.gelu(gate)
    assert rel_rms(out, ref) < 1e-2
