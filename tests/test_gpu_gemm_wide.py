"""GPU tests of gemm_wide_kernel, the persistent 128 x 256-tile GEMM / implicit-GEMM conv (bn = 256 forced).

Each case checks the per-element bound of test_gpu_kernels, NaN guard bands around the output, that two identical
calls are equal bit for bit, and that the result equals gemm_kernel's single-CTA bn = 128 result bit for bit: both
kernels accumulate each element over the same k-steps in the same order and run the same epilogue arithmetic."""
import pytest
import torch

from test_gpu_kernels import (SINGLE, PAIR, cdiv, conv_case, conv_reference, conv_sub_tiles, gemm_case,  # noqa: F401
                              gemm_reference, guarded_out, assert_guard_intact, assert_within_bound, lora_args, rel_rms,
                              run_conv, run_gemm, split_of, dev)

pytestmark = pytest.mark.gpu

WIDE = 256 | SINGLE
NARROW = 128 | SINGLE


def wide_tiles_gemm(M, N, flags):
    return cdiv(M, 128) * (N // 256)


# (M, N, K), flags (as gemm_case; S: split sources), lora, tiles per CTA ("few": fewer tiles than SMs, "some": one to
# three per CTA, "many": at least 3 tiles per CTA and a tile count that is not a multiple of the SM count)
GEMM_CASES = [
    ((1000, 512, 640), "b", None, "few"),                     # M tail (1000 = 7 x 128 + 104)
    ((1024, 768, 1920), "bSX", None, "few"),                  # split sources, views of one wider x
    ((640, 1280, 640), "bRXY", None, "few"),                  # column views of x and the residual
    ((2048, 512, 640), "bG", None, "few"),                    # GEGLU, N 512: two output tiles of 128 columns
    ((2000, 10240, 1280), "bG", None, "many"),                # GEGLU at SDXL width, M tail
    ((1000, 3840, 1280), "L", (4, 1280, 1.0), "few"),         # fused QKV: three rank-4 adaptors, rt 16
    ((512, 1024, 640), "bRL", (8, 256, -0.5), "few"),         # four rank-8 adaptors, rt 32
    ((4096, 1280, 1280), "btR", None, "some"),                # row bias (time embedding) + residual
    ((8192, 2560, 640), "bRL", (4, 1280, 0.5), "many"),       # two adaptors, residual, 640 tiles
    ((12000, 1280, 2560), "bR", None, "many"),                # FF-out: deep K, M tail
]

# (B, H, W, C0, C1, Cout, stride), flags, lora
CONV_CASES = [
    ((2, 36, 88, 128, 0, 256, 1), "bt", (4, 256, 0.5)),       # patches that overhang the image, LoRA, row bias
    ((2, 32, 32, 128, 64, 512, 1), "bRX", None),              # two sources (skip concat) as channel views
    ((2, 72, 104, 64, 0, 256, 2), "b", None),                 # stride 2 to 36 x 52: overhanging patches
    ((2, 64, 64, 128, 0, 512, 2), "bL", (8, 128, 1.0)),      # stride 2, four rank-8 adaptors: rt 32
    ((3, 9, 11, 64, 0, 256, 1), "bR", None),                  # 99-pixel images: one ragged image per tile
    ((8, 32, 32, 640, 0, 1280, 1), "bRL", (4, 1280, 1.0)),    # SDXL 32 x 32 LoRA conv: 2.4 tiles per CTA
]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("shape,flags,lora,per_cta", GEMM_CASES,
                         ids=["x".join(map(str, r[0])) + "-" + r[1] for r in GEMM_CASES])
def test_gemm_wide(dev, shape, flags, lora, per_cta):
    M, N, K = shape
    tiles, sms = wide_tiles_gemm(M, N, flags), _sms()
    if per_cta == "few":
        assert tiles < sms
    elif per_cta == "some":
        assert sms < tiles < 3 * sms
    else:
        assert tiles >= 3 * sms and tiles % sms != 0
    c = gemm_case(M, N, K, flags, lora, dev, M + N + K, split=split_of(flags, K))
    bufs = [guarded_out(M, c.nout, dev) for _ in range(2)]
    for _, out in bufs:
        run_gemm(c, WIDE, out=out)
    narrow = run_gemm(c, NARROW)
    torch.cuda.synchronize()
    for buf, _ in bufs:
        assert_guard_intact(buf, M, c.nout)
    out = bufs[0][1]
    assert torch.equal(out, bufs[1][1])
    assert torch.equal(out, narrow)
    ref, proj, mag = gemm_reference(c)
    assert_within_bound(out, ref, proj, mag)
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("shape,flags,lora", CONV_CASES,
                         ids=["x".join(map(str, r[0])) + "-" + r[1] for r in CONV_CASES])
def test_conv3x3_wide(dev, shape, flags, lora):
    B, H, W, C0, C1, Cout, stride = shape
    c = conv_case(B, H, W, C0, C1, Cout, stride, flags, lora, dev, B * H + C0 + Cout)
    pixels = B * c.Ho * c.Wo
    bufs = [guarded_out(pixels, Cout, dev) for _ in range(2)]
    for _, out in bufs:
        run_conv(c, WIDE, out=out.view(B, c.Ho, c.Wo, Cout))
    narrow = run_conv(c, NARROW)
    torch.cuda.synchronize()
    for buf, _ in bufs:
        assert_guard_intact(buf, pixels, Cout)
    out = bufs[0][1].view(B, c.Ho, c.Wo, Cout)
    assert torch.equal(out, bufs[1][1].view(B, c.Ho, c.Wo, Cout))
    assert torch.equal(out, narrow)
    ref, proj, mag = conv_reference(c)
    assert_within_bound(out, ref, proj, mag)
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("op", ["gemm", "conv"])
def test_wide_lora_runtime_scale(dev, op):
    """Lora.scale_dev in the wide kernel: scale 0.5 x device -3 is bitwise the host scale -1.5, and a new device value
    takes effect."""
    if op == "gemm":
        c = gemm_case(640, 768, 320, "bR", (8, 256, 1.0), dev, 13)
        run = lambda la: run_gemm(c, WIDE, lora=la)  # noqa: E731
    else:
        c = conv_case(2, 32, 32, 128, 0, 512, 1, "bR", (8, 256, 1.0), dev, 14)
        run = lambda la: run_conv(c, WIDE, lora=la)  # noqa: E731
    t = torch.tensor([-3.0], device=dev)
    dyn = lora_args(c, scale=0.5, scale_dev=t)
    a = run(dyn)
    assert torch.equal(a, run(lora_args(c, scale=-1.5)))
    t.fill_(2.0)
    b = run(dyn)
    assert torch.equal(b, run(lora_args(c, scale=1.0)))
    assert not torch.equal(a, b)


def test_wide_ineligible_returns_errors(dev):
    """An explicit bn = 256 on a shape or flag the wide kernel does not take is an error, not a crash."""
    from sliders_b200 import _cabi, ops

    x = torch.zeros(256, 640, device=dev, dtype=torch.bfloat16)
    with pytest.raises(_cabi.Sb200Error, match="bn=256"):
        ops.gemm(x, torch.zeros(640, 640, device=dev, dtype=torch.bfloat16), bn=WIDE)      # N not a multiple of 256
    with pytest.raises(_cabi.Sb200Error, match="bn=256"):
        ops.gemm(x, torch.zeros(512, 640, device=dev, dtype=torch.bfloat16), bn=256 | PAIR)  # CTA pairs
    with pytest.raises(_cabi.Sb200Error, match="bn=256"):
        ops.conv3x3(torch.zeros(1, 16, 16, 64, device=dev, dtype=torch.bfloat16),
                    torch.zeros(320, 3, 3, 64, device=dev, dtype=torch.bfloat16), bn=WIDE)    # Cout 320
    torch.cuda.synchronize()
