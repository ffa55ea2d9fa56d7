"""GPU tests of gemm_wide_kernel at 128 x 160 tiles (bn = 160 forced), the width the 320- and 640-channel layers and
the LoRA convs of the SD / SDXL UNets run at, and of the LoRA-down rows folded into the main wgmma (one m64 x (BN + rt)
product per k-step on every gemm_kernel LoRA instantiation and at bn = 160).

Each bn = 160 case checks the per-element bound of test_gpu_kernels, NaN guard bands around the output, that two
identical calls are equal bit for bit, and that the result equals gemm_kernel's single-CTA bn = 128 result bit for
bit: both kernels accumulate each element over the same k-steps in the same order and run the same epilogue
arithmetic."""
import pytest
import torch
import torch.nn.functional as F

import test_gpu_lora_ranks as lr
from test_gpu_kernels import (SINGLE, PAIR, cdiv, conv_case, conv_reference, epilogue_ref, gemm_case,  # noqa: F401
                              gemm_reference, guarded_out, assert_guard_intact, assert_within_bound, lora_args,
                              rel_rms, run_conv, run_gemm, split_of, dev)
from test_gpu_sample_scales import sample_vector, with_vector

pytestmark = pytest.mark.gpu

W160 = 160 | SINGLE
NARROW = 128 | SINGLE


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check(out_fn, narrow_fn, rows, cols, dev, reference):
    bufs = [guarded_out(rows, cols, dev) for _ in range(2)]
    outs = [out_fn(out) for _, out in bufs]
    narrow = narrow_fn()
    torch.cuda.synchronize()
    for buf, _ in bufs:
        assert_guard_intact(buf, rows, cols)
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0], narrow)
    ref, proj, mag = reference()
    assert_within_bound(outs[0], ref, proj, mag)
    assert rel_rms(outs[0], ref) < 1e-2
    return outs[0]


# (M, N, K), flags (as gemm_case; S: split sources), lora, tiles per CTA ("few": fewer tiles than SMs, "some": one to
# three per CTA, "many": at least 3 tiles per CTA and a tile count that is not a multiple of the SM count)
GEMM_CASES = [
    ((1000, 320, 640), "", None, "few"),                      # no epilogue operand, M tail (1000 = 7 x 128 + 104)
    ((1000, 640, 640), "b", None, "few"),                     # bias
    ((1024, 480, 1920), "bSX", None, "few"),                  # split sources, views of one wider x
    ((640, 640, 640), "bRXY", None, "few"),                   # column views of x and the residual
    ((4096, 1280, 1280), "btR", None, "some"),                # row bias (time embedding) + residual
    ((1000, 1920, 640), "L", (4, 640, 1.0), "few"),           # q|k|v: three rank-4 adaptors, rt 16
    ((640, 1920, 640), "bL", (8, 640, 0.5), "few"),           # q|k|v: three rank-8 adaptors, rt 32
    ((640, 960, 320), "RL", (8, 240, 1.0), "few"),            # four rank-8 adaptors, group edges inside tiles
    ((512, 640, 640), "bRL", (4, 80, -0.5), "few"),           # eight rank-4 adaptors, two per tile
    ((8192, 1920, 640), "bRL", (4, 640, 0.5), "many"),        # 768 tiles
    ((30000, 320, 640), "bR", None, "many"),                  # 470 tiles, M tail
    ((14000, 640, 2560), "bR", None, "many"),                 # FF-out at 64 x 64: deep K
]

# (B, H, W, C0, C1, Cout, stride), flags, lora
CONV_CASES = [
    ((2, 36, 88, 128, 0, 320, 1), "bt", (4, 320, 0.5)),       # patches that overhang the image, LoRA, row bias
    ((2, 32, 32, 128, 64, 640, 1), "bRX", None),              # two sources (skip concat) as channel views
    ((2, 32, 32, 128, 64, 320, 1), "bRL", (8, 320, 1.0)),     # two sources with LoRA
    ((2, 72, 104, 64, 0, 320, 2), "b", None),                 # stride 2 to 36 x 52: overhanging patches
    ((2, 64, 64, 128, 0, 640, 2), "bL", (8, 160, 1.0)),       # stride 2, four rank-8 adaptors: rt 32
    ((3, 9, 11, 64, 0, 320, 1), "bR", None),                  # 99-pixel images: one ragged image per tile
    ((8, 32, 32, 640, 0, 640, 1), "bRL", (4, 640, 1.0)),      # 64 x 64-style LoRA conv, 256 tiles
    ((8, 64, 64, 64, 0, 320, 1), "bRL", (4, 320, 1.0)),       # 128 x 128-style LoRA conv, 512 tiles
]


@pytest.mark.parametrize("shape,flags,lora,per_cta", GEMM_CASES,
                         ids=["x".join(map(str, r[0])) + "-" + (r[1] or "plain") for r in GEMM_CASES])
def test_gemm_w160(dev, shape, flags, lora, per_cta):
    M, N, K = shape
    tiles, sms = cdiv(M, 128) * (N // 160), _sms()
    if per_cta == "few":
        assert tiles < sms
    elif per_cta == "some":
        assert sms < tiles < 3 * sms
    else:
        assert tiles >= 3 * sms and tiles % sms != 0
    c = gemm_case(M, N, K, flags, lora, dev, M + N + K, split=split_of(flags, K))
    _check(lambda out: run_gemm(c, W160, out=out), lambda: run_gemm(c, NARROW), M, c.nout, dev,
           lambda: gemm_reference(c))


@pytest.mark.parametrize("shape,flags,lora", CONV_CASES,
                         ids=["x".join(map(str, r[0])) + "-" + r[1] for r in CONV_CASES])
def test_conv3x3_w160(dev, shape, flags, lora):
    B, H, W, C0, C1, Cout, stride = shape
    c = conv_case(B, H, W, C0, C1, Cout, stride, flags, lora, dev, B * H + C0 + Cout)
    pixels = B * c.Ho * c.Wo
    _check(lambda out: run_conv(c, W160, out=out.view(B, c.Ho, c.Wo, Cout)).view(pixels, Cout),
           lambda: run_conv(c, NARROW).view(pixels, Cout), pixels, Cout, dev,
           lambda: tuple(t.reshape(pixels, Cout) for t in conv_reference(c)))


@pytest.mark.parametrize("lora", [None, (4, 320, 1.0)])
def test_conv3x3_padded_stride2_w160(dev, lora):
    """Stride 2 padded at the bottom / right only (the VAE encoder's Downsample2D)."""
    from sliders_b200 import ops

    c = conv_case(2, 64, 96, 128, 0, 320, 2, "bR", lora, dev, 77)
    pixels = 2 * c.Ho * c.Wo
    run = lambda bn, out=None: ops.conv3x3(c.x0, c.w, stride=2, bias=c.bias, resid=c.resid, lora=c.la, out=out,  # noqa
                                           bn=bn, pad_bottom_right=True)

    def reference():
        def product(f):
            xn = F.pad(f(c.x).permute(0, 3, 1, 2), (0, 1, 0, 1))
            y = F.conv2d(xn, f(c.w).permute(0, 3, 1, 2), stride=2).permute(0, 2, 3, 1).contiguous()
            if c.la is not None:
                t = F.conv2d(xn, f(c.down).view(-1, 3, 3, c.Cin).permute(0, 3, 1, 2), stride=2).permute(0, 2, 3, 1)
                for g0 in range(0, c.Cout, c.group_n):
                    i = g0 // c.group_n
                    y[..., g0:g0 + c.group_n] += (t[..., i * c.r:(i + 1) * c.r] @ f(c.up)[g0:g0 + c.group_n].t()) \
                        * f(torch.tensor(c.scale))
            return y

        return tuple(t.reshape(pixels, c.Cout) for t in epilogue_ref(product, bias=c.bias, resid=c.resid))

    _check(lambda out: run(W160, out.view(2, c.Ho, c.Wo, 320)).view(pixels, 320),
           lambda: run(NARROW).view(pixels, 320), pixels, 320, dev, reference)


@pytest.mark.parametrize("op", ["gemm", "conv"])
def test_w160_lora_runtime_scale(dev, op):
    """Lora.scale_dev at bn = 160: scale 0.5 x device -3 is bitwise the host scale -1.5, and a new device value takes
    effect."""
    if op == "gemm":
        c = gemm_case(640, 960, 320, "bR", (8, 320, 1.0), dev, 13)
        run = lambda la: run_gemm(c, W160, lora=la)  # noqa: E731
    else:
        c = conv_case(2, 32, 32, 128, 0, 640, 1, "bR", (8, 160, 1.0), dev, 14)
        run = lambda la: run_conv(c, W160, lora=la)  # noqa: E731
    t = torch.tensor([-3.0], device=dev)
    dyn = lora_args(c, scale=0.5, scale_dev=t)
    a = run(dyn)
    assert torch.equal(a, run(lora_args(c, scale=-1.5)))
    t.fill_(2.0)
    b = run(dyn)
    assert torch.equal(b, run(lora_args(c, scale=1.0)))
    assert not torch.equal(a, b)


@pytest.mark.parametrize("op", ["gemm", "conv"])
def test_w160_sample_scales(dev, op):
    """Per-sample LoRA scales at bn = 160 (sample edges inside tiles): bitwise the bn = 128 result, and each sample's
    rows bitwise the rows of a call with that sample's factor as the host scale."""
    if op == "gemm":
        c = gemm_case(1200, 640, 320, "bR", (4, 320, 1.0), dev, 21)
        rps, nsamples = 200, 6
        run = lambda bn, la: run_gemm(c, bn, lora=la)  # noqa: E731
    else:
        c = conv_case(4, 20, 24, 128, 0, 320, 1, "bR", (8, 160, 1.0), dev, 22)
        rps, nsamples = 480, 4
        run = lambda bn, la: run_conv(c, bn, lora=la).reshape(-1, 320)  # noqa: E731
    vec = sample_vector(nsamples, dev, seed=3)
    got = run(W160, with_vector(c.la, vec, rps))
    assert torch.equal(got, run(NARROW, with_vector(c.la, vec, rps)))
    for s in range(nsamples):
        one = run(W160, lora_args(c, scale=float(vec[s])))
        assert torch.equal(got[s * rps:(s + 1) * rps], one[s * rps:(s + 1) * rps])


def test_w160_ineligible_returns_errors(dev):
    """An explicit bn = 160 on a shape or flag that 160-wide tiles do not take is an error, not a crash."""
    from sliders_b200 import _cabi, ops

    x = torch.zeros(256, 640, device=dev, dtype=torch.bfloat16)
    w = lambda n: torch.zeros(n, 640, device=dev, dtype=torch.bfloat16)  # noqa: E731
    with pytest.raises(_cabi.Sb200Error, match="bn=160"):
        ops.gemm(x, w(512), bn=W160)                                     # N not a multiple of 160
    with pytest.raises(_cabi.Sb200Error, match="bn=160"):
        ops.gemm(x, w(640), bn=160 | PAIR)                               # CTA pairs
    with pytest.raises(_cabi.Sb200Error, match="bn=160"):
        ops.gemm(x, w(1280), geglu=True, bn=W160)                        # GEGLU
    c = gemm_case(256, 960, 640, "", (8, 320, 1.0), dev, 5)
    down = torch.zeros(64, 640, device=dev, dtype=torch.bfloat16)
    with pytest.raises(_cabi.Sb200Error, match="bn=160"):                # rank 16: 64 LoRA rows
        ops.gemm(c.x0, c.w, lora=ops.Lora(down, torch.zeros(960, 16, device=dev), 16, 320, 1.0), bn=W160)
    with pytest.raises(_cabi.Sb200Error, match="bn=160"):
        ops.conv3x3(torch.zeros(1, 16, 16, 64, device=dev, dtype=torch.bfloat16),
                    torch.zeros(256, 3, 3, 64, device=dev, dtype=torch.bfloat16), bn=W160)  # Cout 256
    torch.cuda.synchronize()


# One case per gemm_kernel LoRA instantiation (tile width x CTA flavour x LoRA rows), each of which now issues one
# m64 x (BN + rt) wgmma per k-step: (M, N, K), flags, lora (rank, group_n, scale), bn | ctas, rt
FOLDED = [
    ((1000, 960, 320), "bRL", (4, 320, 1.0), 64 | SINGLE, 16),
    ((640, 960, 640), "L", (8, 320, -0.5), 64 | SINGLE, 32),
    ((640, 960, 320), "RL", (16, 320, 0.75), 64 | SINGLE, 64),
    ((1000, 640, 320), "btL", (4, 320, 0.5), 64 | PAIR, 16),
    ((512, 960, 640), "bL", (8, 320, 1.0), 64 | PAIR, 32),
    ((512, 960, 320), "bRL", (16, 320, 1.0), 64 | PAIR, 64),
    ((1000, 1280, 640), "bRL", (4, 1280, 1.0), 128 | SINGLE, 16),
    ((640, 1920, 640), "L", (8, 640, 0.5), 128 | SINGLE, 32),
    ((512, 1920, 640), "RL", (16, 640, -1.0), 128 | SINGLE, 64),
    ((1000, 1280, 640), "btL", (4, 1280, 2.0), 128 | PAIR, 16),
    ((384, 960, 640), "bL", (8, 320, 1.0), 128 | PAIR, 32),
    ((384, 960, 200), "bRL", (16, 320, 0.5), 128 | PAIR, 64),
]


def test_folded_matrix_is_complete():
    cells = set()
    for shape, flags, lora, force, rt in FOLDED:
        assert lr.make_lora(shape[2], shape[1], lora[0], lora[1], "cpu", 0)[2] == rt
        cells.add((force, rt))
    assert cells == {(bn | f, rt) for bn in (64, 128) for f in (SINGLE, PAIR) for rt in (16, 32, 64)}


@pytest.mark.parametrize("shape,flags,lora,force,rt", FOLDED,
                         ids=[f"bn{r[3] & 0xFFF}-{'pair' if r[3] & PAIR else 'single'}-rt{r[4]}" for r in FOLDED])
def test_gemm_kernel_folded_lora(dev, rank16, shape, flags, lora, force, rt):
    """The LoRA-down rows in the main wgmma of gemm_kernel: per-element bound against float64, guard bands, and two
    identical calls equal."""
    M, N, K = shape
    c = gemm_case(M, N, K, flags, lora, dev, M + N + K)
    assert c.rt == rt
    bufs = [guarded_out(M, c.nout, dev) for _ in range(2)]
    outs = [run_gemm(c, force, out=out) for _, out in bufs]
    torch.cuda.synchronize()
    for buf, _ in bufs:
        assert_guard_intact(buf, M, c.nout)
    assert torch.equal(outs[0], outs[1])
    ref, proj, mag = gemm_reference(c)
    assert_within_bound(outs[0], ref, proj, mag)
    assert rel_rms(outs[0], ref) < 1e-2


rank16 = lr.rank16
