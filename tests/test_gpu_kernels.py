"""GPU parity tests of the GEMM-family sm_90a kernels, called through the C ABI (sliders_b200.ops) and compared with a
float64 reference computed from the same bf16 inputs, element by element (`bound_violations` derives the bound) and
by rel-RMS.  Every instantiation of `gemm_kernel` (tile width x single CTA / CTA pair x LoRA rows) is forced
explicitly, in each shared-memory regime it can launch in.  Also here: two attention property tests (softmax rows sum
to one; a row maximum that grows on every key tile) and the argument checks.  The other forward kernels (attention,
LayerNorm, GroupNorm, small_linear, sinusoid, conv_in / conv_out, upsample2x, the CFG step) are checked element by
element in test_gpu_forward_bounds.py, the backward kernels in test_gpu_backward_bounds.py."""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
SINGLE, PAIR = 0x2000, 0x1000
NAN_BITS = 0x7FA5  # a bf16 NaN payload no kernel produces: guard bands around GEMM outputs are filled with it
GUARD_ROWS, GUARD_COLS = 3, 24


def cdiv(a, b):
    return -(-a // b)


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


def bound_violations(out, ref, proj, mag):
    """Bool mask of the elements of a GEMM / conv output outside its per-element error bound (NaN is outside).

    ref:  float64 result computed from the same bf16 inputs;
    proj: float64 value before the residual is added (equal to ref without a residual);
    mag:  the same expression on absolute values, |x|.|w|^T + |s| (|x|.|down|^T).|up|^T + |bias| + |rowbias|
          (for a conv: the conv of |x| with |w|), which bounds every partial sum the kernel forms.
    |out - ref| <= 2^-8 (|ref| + |proj|) + 2^-12 mag, because:
    - the kernel rounds twice to bf16, the fp32 projection and then projection + residual (a bf16 add), each within
      2^-9 of its value; 2^-8 (|ref| + |proj|) covers both with a factor 2 to spare;
    - fp32 accumulation: each rounding step errs by at most 2^-24 of a partial sum, and no partial sum exceeds mag.
      2^-12 mag allows 4096 steps; the longest accumulation tested is K = 17280 (a conv over 1920 channels), 1080
      wgmma k-steps of 16 plus a few roundings inside each, and the epilogue's bias / LoRA / row-bias additions.
    GEGLU (a * gelu(g)) carries the accumulation errors of a and g through the product: the caller passes
    mag = |gelu(g)| mag_a + 1.2 |a| mag_g, where 1.2 bounds |gelu'| (its maximum is 1.129)."""
    err = (out.double() - ref).abs()
    return ~(err <= 2.0 ** -8 * (ref.abs() + proj.abs()) + 2.0 ** -12 * mag)


def assert_within_bound(out, ref, proj, mag):
    bad = bound_violations(out, ref, proj, mag)
    n = int(bad.sum())
    if n:
        where = [tuple(i) for i in bad.nonzero()[:6].tolist()]
        detail = "; ".join(f"{i}: got {out[i].item():.5g}, want {ref[i].item():.5g}" for i in where)
        raise AssertionError(f"{n} of {out.numel()} elements outside the error bound, first at {detail}")


def _lora_add(y, t, up, r, group_n, scale):
    """In place: y[..., columns of adaptor i] += scale * t[..., i*r:(i+1)*r] @ up[those columns]^T."""
    for g0 in range(0, y.shape[-1], group_n):
        i = g0 // group_n
        y[..., g0:g0 + group_n] += (t[..., i * r:(i + 1) * r] @ up[g0:g0 + group_n].t()) * scale


def epilogue_ref(product, *, bias=None, rowbias=None, resid=None, geglu=False):
    """float64 reference of the fused epilogue -> (ref, proj, mag) for `bound_violations`.  product(f) is the
    projection (+ LoRA) computed from f(every input), f = float64 or its absolute value; rowbias is already
    broadcastable to the output."""
    dbl, mag_of = (lambda t: t.double()), (lambda t: t.double().abs())
    y, m = product(dbl), product(mag_of)
    if bias is not None:
        y, m = y + dbl(bias), m + mag_of(bias)
    if geglu:
        assert rowbias is None, "the kernel adds a row bias before the GEGLU product; no caller combines them"
        (a, g), (ma, mg) = y.chunk(2, dim=-1), m.chunk(2, dim=-1)
        gl = F.gelu(g)
        y, m = a * gl, gl.abs() * ma + 1.2 * a.abs() * mg
    if rowbias is not None:
        y, m = y + dbl(rowbias), m + mag_of(rowbias)
    ref = y + dbl(resid) if resid is not None else y
    return ref, y, m


def _col_view(t, extra):
    """A copy of t as a view of the first columns of a wider buffer (row stride > last dim)."""
    wide = torch.zeros(t.shape[:-1] + (t.shape[-1] + extra,), device=t.device, dtype=t.dtype)
    wide[..., :t.shape[-1]] = t
    return wide[..., :t.shape[-1]]


def gemm_case(M, N, K, flags, lora, dev, seed, split=0):
    """Inputs of one ops.gemm call.  flags: b bias, t time-embedding row bias (4 row groups), R residual, G GEGLU,
    X x as a column view (ldx > K), Y residual as a column view (ldr > N); lora = (rank, group_n, scale) or None;
    split: x comes as two sources, columns [0, split) and [split, K)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(dev, BF)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, BF)
    geglu = "G" in flags
    nout = N // 2 if geglu else N
    c = SimpleNamespace(M=M, N=N, K=K, nout=nout, geglu=geglu, w=w, rpb=max(1, M // 4), la=None)
    c.bias = torch.randn(N, generator=g).to(dev, BF) if "b" in flags else None
    c.rowbias = torch.randn(cdiv(M, c.rpb), nout, generator=g).to(dev, BF) if "t" in flags else None
    c.resid = torch.randn(M, nout, generator=g).to(dev, BF) if "R" in flags else None
    if "Y" in flags:
        c.resid = _col_view(c.resid, 40)
    c.x = _col_view(x, 24) if "X" in flags else x
    c.x0, c.x1 = (c.x[:, :split], c.x[:, split:]) if split else (c.x, None)
    if split and "X" not in flags:
        c.x0, c.x1 = c.x0.contiguous(), c.x1.contiguous()
    if lora:
        c.r, c.group_n, c.scale = lora
        c.down, c.up, c.rt = make_lora(K, N, c.r, c.group_n, dev, seed + 1)
        c.la = lora_args(c)
    return c


def lora_args(c, scale=None, scale_dev=None):
    from sliders_b200 import ops

    return ops.Lora(c.down, c.up, c.r, c.group_n, c.scale if scale is None else scale, scale_dev=scale_dev)


def run_gemm(c, bn, out=None, lora=None, rows=None):
    """ops.gemm on case c (its first `rows` rows if given)."""
    from sliders_b200 import ops

    s = slice(0, rows or c.M)
    return ops.gemm(c.x0[s], c.w, bias=c.bias, rowbias=c.rowbias, rows_per_batch=c.rpb,
                    resid=c.resid[s] if c.resid is not None else None, geglu=c.geglu, lora=lora or c.la,
                    x1=c.x1[s] if c.x1 is not None else None, out=out, bn=bn)


def gemm_reference(c):
    def product(f):
        xd = f(c.x)
        y = xd @ f(c.w).t()
        if c.la is not None:
            _lora_add(y, xd @ f(c.down).t(), f(c.up), c.r, c.group_n, f(torch.tensor(c.scale)))
        return y

    rb = c.rowbias[torch.arange(c.M, device=c.w.device) // c.rpb] if c.rowbias is not None else None
    return epilogue_ref(product, bias=c.bias, rowbias=rb, resid=c.resid, geglu=c.geglu)


def conv_case(B, H, W, C0, C1, Cout, stride, flags, lora, dev, seed):
    """Inputs of one ops.conv3x3 call; flags and lora as in gemm_case (X: the sources are channel slices of a wider
    NHWC buffer)."""
    g = torch.Generator().manual_seed(seed)
    Cin = C0 + C1
    x = torch.randn(B, H, W, Cin, generator=g).to(dev, BF)
    w = (torch.randn(Cout, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5).to(dev, BF)
    Ho, Wo = H // stride, W // stride
    c = SimpleNamespace(B=B, Ho=Ho, Wo=Wo, Cin=Cin, Cout=Cout, stride=stride, w=w, la=None)
    c.bias = torch.randn(Cout, generator=g).to(dev, BF) if "b" in flags else None
    c.rowbias = torch.randn(B, Cout, generator=g).to(dev, BF) if "t" in flags else None
    c.resid = torch.randn(B, Ho, Wo, Cout, generator=g).to(dev, BF) if "R" in flags else None
    if "Y" in flags:
        c.resid = _col_view(c.resid, 40)
    c.x = _col_view(x, 64) if "X" in flags else x
    if "X" in flags:
        c.x0, c.x1 = c.x[..., :C0], (c.x[..., C0:] if C1 else None)
    else:
        c.x0, c.x1 = c.x[..., :C0].contiguous(), (c.x[..., C0:].contiguous() if C1 else None)
    if lora:
        c.r, c.group_n, c.scale = lora
        c.down, c.up, c.rt = make_lora(9 * Cin, Cout, c.r, c.group_n, dev, seed + 2)
        c.la = lora_args(c)
    return c


def run_conv(c, bn, out=None, lora=None, images=None):
    """ops.conv3x3 on case c (its first `images` images if given)."""
    from sliders_b200 import ops

    s = slice(0, images or c.B)
    pick = lambda t: t[s] if t is not None else None  # noqa: E731
    return ops.conv3x3(c.x0[s], c.w, x1=pick(c.x1), stride=c.stride, bias=c.bias, rowbias=pick(c.rowbias),
                       resid=pick(c.resid), lora=lora or c.la, out=out, bn=bn)


def conv_reference(c):
    def product(f):
        xn = f(c.x).permute(0, 3, 1, 2)
        y = F.conv2d(xn, f(c.w).permute(0, 3, 1, 2), stride=c.stride, padding=1).permute(0, 2, 3, 1).contiguous()
        if c.la is not None:
            dn = f(c.down).view(-1, 3, 3, c.Cin).permute(0, 3, 1, 2)
            t = F.conv2d(xn, dn, stride=c.stride, padding=1).permute(0, 2, 3, 1)
            _lora_add(y, t, f(c.up), c.r, c.group_n, f(torch.tensor(c.scale)))
        return y

    rb = c.rowbias[:, None, None, :] if c.rowbias is not None else None
    return epilogue_ref(product, bias=c.bias, rowbias=rb, resid=c.resid)


def guarded_out(rows, cols, dev):
    """(buffer, view): a [rows, cols] output inside a buffer with GUARD_ROWS more rows above and below and GUARD_COLS
    more columns, all filled with the NAN_BITS pattern."""
    buf = torch.full((rows + 2 * GUARD_ROWS, cols + GUARD_COLS), NAN_BITS, dtype=torch.int16, device=dev).view(BF)
    return buf, buf[GUARD_ROWS:GUARD_ROWS + rows, :cols]


def assert_guard_intact(buf, rows, cols):
    bits = buf.view(torch.int16)
    guard = torch.ones_like(bits, dtype=torch.bool)
    guard[GUARD_ROWS:GUARD_ROWS + rows, :cols] = False
    n = int((bits[guard] != NAN_BITS).sum())
    assert n == 0, f"{n} elements written outside the [{rows}, {cols}] output"
    assert not torch.isnan(buf[GUARD_ROWS:GUARD_ROWS + rows, :cols]).any(), "NaN in the output (unwritten?)"


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
    c = gemm_case(M, N, K, flags, lora, dev, M + N + K, split=split)
    out = run_gemm(c, force)
    torch.cuda.synchronize()
    ref, proj, mag = gemm_reference(c)
    assert_within_bound(out, ref, proj, mag)
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("force", [SINGLE, PAIR, 0])
@pytest.mark.parametrize("B,H,W,C0,C1,Cout,stride,flags,lora", [
    (1, 32, 32, 64, 0, 64, 1, "", None),
    (1, 64, 64, 320, 0, 320, 1, "bt", None),       # conv1 of a ResnetBlock2D: + time-embedding row bias
    (1, 128, 128, 320, 0, 320, 1, "bR", None),     # conv2: + residual, one image row per tile
    (2, 32, 32, 1280, 640, 1280, 1, "b", None),    # skip-connection concat as two sources
    (2, 64, 64, 320, 0, 320, 2, "b", None),        # Downsample2D (stride 2, parity planes)
    (2, 32, 32, 640, 0, 640, 1, "bL", (4, 640, 0.5)),  # LoRA conv: down 3x3 folded in, up 1x1 in the epilogue
    (3, 8, 8, 128, 0, 128, 1, "b", None),          # 8x8 level: tiles span images, ragged M
    (1, 16, 16, 128, 64, 64, 1, "b", None),
    # patches that overhang the image (dynamic_resolution buckets, non-square eval sizes: ADVICE r1 #1)
    (1, 72, 72, 64, 0, 64, 1, "bR", None),         # W = 72: one 72-pixel row per 128-row tile
    (2, 36, 88, 128, 0, 128, 1, "bt", (4, 128, 0.5)),  # 36 x 88, LoRA + time-embedding bias
    (1, 18, 18, 128, 64, 64, 1, "b", None),        # 18 x 18 with a skip concat (7 rows of 18 per tile)
    (3, 9, 11, 64, 0, 64, 1, "bR", None),          # 99-pixel images: one (ragged) image per tile
    (2, 72, 104, 64, 0, 64, 2, "b", None),         # stride 2 to 36 x 52
    (1, 96, 160, 64, 0, 64, 1, "b", None),         # W > 128 and not a multiple of it
    (5, 4, 4, 64, 0, 64, 1, "bt", None),           # 8 images per tile, 5 in the batch
])
def test_conv3x3(dev, force, B, H, W, C0, C1, Cout, stride, flags, lora):
    c = conv_case(B, H, W, C0, C1, Cout, stride, flags, lora, dev, B * H + C0 + Cout)
    out = run_conv(c, force)
    torch.cuda.synchronize()
    ref, proj, mag = conv_reference(c)
    assert_within_bound(out, ref, proj, mag)
    assert rel_rms(out, ref) < 1e-2


# ----------------------------------------------------------------------------------------------------------------
# Every gemm_kernel<BN, kCtas, RT> instantiation in every shared-memory regime it launches in.  launch_gemm gives a
# CTA the whole SM's shared memory ("ring1": a deep stage ring) when the grid has no more CTAs than the GPU has SMs,
# and half of it ("ring2") when the grid is larger and the instantiation is built for two CTAs per SM (gemm_slots).
# The labels hold on any H100 from 114 SMs (PCIe) to 132 (SXM): ring1 cases launch at most 114 CTAs, ring2 cases at
# least 264.
# ----------------------------------------------------------------------------------------------------------------
def gemm_slots(bn, rt):
    """CTAs per SM gemm_kernel<bn, *, rt> is built for (gemm_slots in gemm.cu)."""
    return 2 if bn == 64 or rt == 0 else 1


def decode_force(force):
    return force & 0xFFF, 2 if force & PAIR else 1


def regime(grid_ctas, bn, rt, num_sms):
    return "ring2" if grid_ctas > num_sms and gemm_slots(bn, rt) == 2 else "ring1"


def gemm_grid(M, N, flags, bn, ctas):
    """CTAs of one ops.gemm launch: (128 * ctas)-row tiles x output-column tiles x ctas, as in launch_gemm."""
    ncols, nout = (bn // 2, N // 2) if "G" in flags else (bn, N)
    return cdiv(cdiv(M, 128), ctas) * cdiv(nout, ncols) * ctas


def conv_sub_tiles(B, H, W):
    """128-row sub-tiles of a conv over B x H x W output pixels: the patch pick_patch in gemm.cu chooses."""
    best = None
    for bw in range(min(W, 128), 0, -1):
        bh = min(128 // bw, H)
        bb = max(1, min(128 // (bw * bh), B)) if (bw == W and bh == H) else 1
        tiles = cdiv(W, bw) * cdiv(H, bh) * cdiv(B, bb)
        if best is None or tiles < best:
            best = tiles
    return best


def conv_grid(B, H, W, stride, Cout, bn, ctas):
    return cdiv(conv_sub_tiles(B, H // stride, W // stride), ctas) * cdiv(Cout, bn) * ctas


def split_of(flags, K):
    """'S' in flags: x in two sources along K, split at 2/3 of K rounded down to a k-block (as a skip concat)."""
    return (2 * K // 3) // 64 * 64 if "S" in flags else 0


# (M, N, K), flags (as gemm_case; S: split sources), lora, bn | ctas, LoRA rows rt, regime
GEMM_MATRIX = [
    ((300, 336, 200), "bRXY", None, 64 | SINGLE, 0, "ring1"),             # N % 32 = 16, K % 64 = 8, ldx > K, ldr > N
    ((300, 8192, 2048), "b", None, 64 | SINGLE, 0, "ring2"),              # 33.5 MB of W: M-fastest tile order
    ((256, 240, 72), "bL", (4, 80, 0.5), 64 | SINGLE, 16, "ring1"),       # group_n 80, K = 72 with LoRA
    ((8192, 320, 640), "bLS", (4, 320, 1.0), 64 | SINGLE, 16, "ring2"),   # SDXL conv_shortcut / proj: split + LoRA
    ((640, 960, 320), "L", (8, 320, 1.0), 64 | SINGLE, 32, "ring1"),      # fused q|k|v, three rank-8 adaptors
    ((4096, 960, 200), "RL", (8, 320, -0.5), 64 | SINGLE, 32, "ring2"),   # K = 200 with LoRA
    ((1000, 160, 640), "bGX", None, 64 | PAIR, 0, "ring1"),               # GEGLU at BN 64: Nout 80, last tile 16
    ((2100, 1280, 320), "btR", None, 64 | PAIR, 0, "ring2"),              # 17 sub-tiles: phantom half
    ((384, 336, 576), "RL", (4, 112, 2.0), 64 | PAIR, 16, "ring1"),       # phantom half, group_n 112, N % 32 = 16
    ((8192, 320, 960), "bLSX", (4, 320, 1.0), 64 | PAIR, 16, "ring2"),    # split sources: views of one x
    ((300, 240, 72), "bL", (8, 80, -0.75), 64 | PAIR, 32, "ring1"),       # group_n 80, rank 8, K = 72
    ((4000, 960, 320), "RL", (8, 320, 0.5), 64 | PAIR, 32, "ring2"),      # ragged last row tile
    ((1000, 336, 72), "RY", None, 128 | SINGLE, 0, "ring1"),              # K = 72, last tile 80 columns
    ((2048, 2592, 320), "bG", None, 128 | SINGLE, 0, "ring2"),            # GEGLU Nout 1296: last tile 16 columns
    ((300, 3840, 1280), "LX", (4, 1280, 1.0), 128 | SINGLE, 16, "ring1"),  # fused QKV at SDXL width
    ((640, 1920, 640), "L", (8, 640, 1.0), 128 | SINGLE, 32, "ring1"),    # fused QKV, three rank-8 adaptors
    ((1024, 640, 1920), "bS", None, 128 | PAIR, 0, "ring1"),              # skip concat
    ((600, 8192, 2048), "b", None, 128 | PAIR, 0, "ring2"),               # M-fastest order, phantom half
    ((512, 2560, 640), "bRLY", (8, 1280, 0.5), 128 | PAIR, 16, "ring1"),  # one adaptor per pair half
    ((300, 960, 200), "LX", (8, 320, -1.0), 128 | PAIR, 32, "ring1"),     # three rank-8 adaptors, K = 200
]

# (B, H, W, C0, C1, Cout, stride), flags, lora, bn | ctas, LoRA rows rt, regime
CONV_MATRIX = [
    ((1, 16, 16, 64, 0, 336, 1), "bRXY", None, 64 | SINGLE, 0, "ring1"),       # Cout 336: last tile 16 columns
    ((2, 64, 64, 64, 0, 320, 1), "bt", None, 64 | SINGLE, 0, "ring2"),
    ((2, 32, 32, 128, 0, 320, 2), "bL", (4, 320, 0.5), 64 | SINGLE, 16, "ring1"),   # stride 2 with LoRA
    ((2, 64, 64, 64, 0, 320, 1), "bLR", (4, 320, 1.0), 64 | SINGLE, 16, "ring2"),
    ((1, 16, 16, 128, 0, 336, 1), "L", (8, 112, 1.0), 64 | SINGLE, 32, "ring1"),    # three rank-8 adaptors
    ((2, 64, 64, 64, 0, 336, 1), "bL", (8, 112, -0.5), 64 | SINGLE, 32, "ring2"),
    ((5, 4, 4, 64, 0, 128, 1), "bt", None, 64 | PAIR, 0, "ring1"),              # one sub-tile: phantom half
    ((1, 65, 64, 64, 0, 640, 1), "bR", None, 64 | PAIR, 0, "ring2"),            # 33 sub-tiles: phantom half
    ((1, 64, 64, 64, 0, 320, 2), "bL", (4, 320, 0.5), 64 | PAIR, 16, "ring1"),    # stride 2 with LoRA
    ((2, 32, 32, 128, 64, 1280, 1), "bLRX", (4, 1280, 1.0), 64 | PAIR, 16, "ring2"),  # skip concat + LoRA
    ((1, 16, 16, 64, 0, 240, 1), "bL", (8, 80, 1.0), 64 | PAIR, 32, "ring1"),     # group_n 80
    ((2, 64, 64, 64, 0, 336, 1), "LRY", (8, 112, 0.5), 64 | PAIR, 32, "ring2"),
    ((1, 32, 32, 128, 0, 336, 1), "bR", None, 128 | SINGLE, 0, "ring1"),        # last tile 80 columns
    ((4, 64, 64, 64, 0, 320, 1), "bt", None, 128 | SINGLE, 0, "ring2"),
    ((1, 32, 32, 320, 0, 640, 1), "bL", (4, 640, 0.5), 128 | SINGLE, 16, "ring1"),
    ((1, 32, 32, 128, 0, 336, 1), "bRL", (8, 112, 1.0), 128 | SINGLE, 32, "ring1"),
    ((2, 32, 32, 128, 64, 320, 1), "bX", None, 128 | PAIR, 0, "ring1"),         # skip concat, channel views
    ((4, 128, 128, 64, 0, 320, 2), "b", None, 128 | PAIR, 0, "ring2"),          # stride 2
    ((2, 32, 32, 128, 0, 640, 2), "bL", (4, 640, 0.5), 128 | PAIR, 16, "ring1"),  # stride 2 with LoRA
    ((3, 9, 11, 64, 0, 336, 1), "btL", (8, 112, 1.0), 128 | PAIR, 32, "ring1"),  # ragged 99-pixel images
]


def _matrix_id(row):
    shape, flags, lora, force, rt, reg = row
    bn, ctas = decode_force(force)
    return f"bn{bn}-ctas{ctas}-rt{rt}-{reg}-" + "x".join(map(str, shape)) + (f"-{flags}" if flags else "")


@pytest.mark.parametrize("shape,flags,lora,force,rt,reg", GEMM_MATRIX, ids=[_matrix_id(r) for r in GEMM_MATRIX])
def test_gemm_variant_matrix(dev, shape, flags, lora, force, rt, reg):
    """Per-element bound, guard bands around the output, two identical calls equal, and the other CTA flavour at the
    same tile width equal bit for bit (the pair runs the same k order and epilogue arithmetic)."""
    M, N, K = shape
    bn, ctas = decode_force(force)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert regime(gemm_grid(M, N, flags, bn, ctas), bn, rt, sms) == reg
    c = gemm_case(M, N, K, flags, lora, dev, M + N + K, split=split_of(flags, K))
    assert (c.rt if lora else 0) == rt
    bufs = [guarded_out(M, c.nout, dev) for _ in range(2)]
    for _, out in bufs:
        run_gemm(c, force, out=out)
    other = run_gemm(c, bn | (SINGLE if ctas == 2 else PAIR))
    torch.cuda.synchronize()
    for buf, _ in bufs:
        assert_guard_intact(buf, M, c.nout)
    out = bufs[0][1]
    assert torch.equal(out, bufs[1][1])
    assert torch.equal(out, other)
    ref, proj, mag = gemm_reference(c)
    assert_within_bound(out, ref, proj, mag)
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("shape,flags,lora,force,rt,reg", CONV_MATRIX, ids=[_matrix_id(r) for r in CONV_MATRIX])
def test_conv3x3_variant_matrix(dev, shape, flags, lora, force, rt, reg):
    """As test_gemm_variant_matrix, for the implicit-GEMM conv (output rows are pixels)."""
    B, H, W, C0, C1, Cout, stride = shape
    bn, ctas = decode_force(force)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert regime(conv_grid(B, H, W, stride, Cout, bn, ctas), bn, rt, sms) == reg
    c = conv_case(B, H, W, C0, C1, Cout, stride, flags, lora, dev, B * H + C0 + Cout)
    assert (c.rt if lora else 0) == rt
    pixels = B * c.Ho * c.Wo
    bufs = [guarded_out(pixels, Cout, dev) for _ in range(2)]
    for _, out in bufs:
        run_conv(c, force, out=out.view(B, c.Ho, c.Wo, Cout))
    other = run_conv(c, bn | (SINGLE if ctas == 2 else PAIR))
    torch.cuda.synchronize()
    for buf, _ in bufs:
        assert_guard_intact(buf, pixels, Cout)
    out = bufs[0][1].view(B, c.Ho, c.Wo, Cout)
    assert torch.equal(out, bufs[1][1].view(B, c.Ho, c.Wo, Cout))
    assert torch.equal(out, other)
    ref, proj, mag = conv_reference(c)
    assert_within_bound(out, ref, proj, mag)
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("op,force,lora", [("gemm", 64 | SINGLE, True), ("gemm", 128 | PAIR, False),
                                           ("conv", 64 | PAIR, True), ("conv", 128 | SINGLE, False)])
def test_rows_do_not_depend_on_regime(dev, op, force, lora):
    """The same rows computed in a grid larger than the GPU (ring2) and in one that fits it (ring1) are bitwise
    equal: the ring depth changes only how far the loads run ahead."""
    bn, ctas = decode_force(force)
    rt = 16 if lora else 0
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if op == "gemm":
        M, N, K, m = 8192, 640, 640, 1000
        assert regime(gemm_grid(M, N, "", bn, ctas), bn, rt, sms) == "ring2"
        assert regime(gemm_grid(m, N, "", bn, ctas), bn, rt, sms) == "ring1"
        c = gemm_case(M, N, K, "bR", (4, 640, 0.5) if lora else None, dev, 11)
        full, part = run_gemm(c, force), run_gemm(c, force, rows=m)
    else:
        B, H, W, C0, Cout, b = 8, 32, 32, 128, 320, 2
        assert regime(conv_grid(B, H, W, 1, Cout, bn, ctas), bn, rt, sms) == "ring2"
        assert regime(conv_grid(b, H, W, 1, Cout, bn, ctas), bn, rt, sms) == "ring1"
        c = conv_case(B, H, W, C0, 0, Cout, 1, "btR", (4, 320, 0.5) if lora else None, dev, 12)
        full, part = run_conv(c, force), run_conv(c, force, images=b)
    torch.cuda.synchronize()
    assert torch.equal(full[:part.shape[0]], part)


@pytest.mark.parametrize("op,force", [("gemm", 64 | PAIR), ("gemm", 128 | SINGLE), ("conv", 128 | PAIR)])
def test_lora_runtime_scale(dev, op, force):
    """Lora.scale_dev: the kernel reads the slider scale from device memory at run time and multiplies it by the
    host scale; scale 0.5 x device -3 is bitwise the host scale -1.5, and a new device value takes effect."""
    if op == "gemm":
        c = gemm_case(640, 960, 320, "bR", (8, 320, 1.0), dev, 13)
        run = lambda la: run_gemm(c, force, lora=la)  # noqa: E731
    else:
        c = conv_case(2, 32, 32, 128, 0, 336, 1, "bR", (8, 112, 1.0), dev, 14)
        run = lambda la: run_conv(c, force, lora=la)  # noqa: E731
    t = torch.tensor([-3.0], device=dev)
    dyn = lora_args(c, scale=0.5, scale_dev=t)
    a = run(dyn)
    assert torch.equal(a, run(lora_args(c, scale=-1.5)))
    t.fill_(2.0)
    b = run(dyn)
    assert torch.equal(b, run(lora_args(c, scale=1.0)))
    assert not torch.equal(a, b)


def test_attention_softmax_rows_sum_to_one(dev):
    """Size-independent property: with V = 1 every output element is sum(bf16(p)) / l, where l sums the unrounded
    p; the bf16 rounding of P moves it by at most 2^-8 (2^-7 with the output rounding)."""
    from sliders_b200 import ops

    B, heads, S = 2, 4, 1024
    g = torch.Generator().manual_seed(0)
    q = (torch.randn(B * S, heads * 64, generator=g) * 3).to(dev, BF)
    k = (torch.randn(B * S, heads * 64, generator=g) * 3).to(dev, BF)
    v = torch.ones(B * S, heads * 64, device=dev, dtype=BF)
    out = ops.attention(q, k, v, B, heads, S, S, 0.125)
    assert (out.float() - 1).abs().max().item() <= 2.0 ** -7


def test_attention_growing_logits_rescale(dev):
    """Keys ordered so the row maximum keeps growing from key tile to key tile: attention_kernel rescales the O
    accumulator and l by alpha = 2^(m_old - m_new) on every tile, and this makes those factors far from 1.  Checked
    element by element (o and the log-sum-exp the backward pass consumes) at ND = 1, 2 and 3."""
    from test_gpu_forward_bounds import check_attention_fwd, run_attention_fwd

    B, heads, S = 1, 2, 1024
    for d in (64, 128, 192):
        g = torch.Generator().manual_seed(5)
        q = torch.randn(B * S, heads * d, generator=g).abs()
        k = torch.randn(B * S, heads * d, generator=g).abs() * torch.linspace(0.2, 6.0, S).repeat(B)[:, None]
        v = torch.randn(B * S, heads * d, generator=g)
        q, k, v = q.to(dev, BF), k.to(dev, BF), v.to(dev, BF)
        scale = 8.0 / d  # 0.125 at d = 64: logits of the same size at every head width
        sc = q.double().view(S, heads, d).transpose(0, 1) @ k.double().view(S, heads, d).permute(1, 2, 0) * scale
        assert (sc.amax(-1) - sc[..., :64].amax(-1)).min().item() > 16   # the max really grows past the first tile
        o, lse = run_attention_fwd(q, k, v, B, heads, S, S, d, scale)
        check_attention_fwd(o, lse, q, k, v, B, heads, S, S, d, scale)


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
    # GroupNorm: the stats kernels' shared memory (8 C bytes once C > 4096) stays within the default 48 KB
    for C, ok in ((6144, True), (6152, False)):
        x = torch.randn(1, 4, 4, C, device=dev).to(BF)
        gm, bt = torch.ones(C, device=dev, dtype=BF), torch.zeros(C, device=dev, dtype=BF)
        ws = ops.gn_ws(1, 8, dev)
        if ok:
            y = ops.groupnorm(x, gm, bt, 8, 1e-5, False, stats_ws=ws)
            torch.cuda.synchronize()
            assert torch.isfinite(y.float()).all()
            # the backward's 768-thread blocks exceed what its kernels' registers allow (at most 640 on sm_90a):
            # refused before any launch
            with pytest.raises(_cabi.Sb200Error, match="too large"):
                ops.groupnorm_bwd(x, gm, bt, 8, False, x, ws)
            continue
        with pytest.raises(_cabi.Sb200Error, match="too large"):
            ops.groupnorm(x, gm, bt, 8, 1e-5, False, stats_ws=ws)
        with pytest.raises(_cabi.Sb200Error, match="too large"):
            ops.groupnorm_bwd(x, gm, bt, 8, False, x, ws)
    # attention backward: every operand row must hold heads x head_dim columns
    q = torch.zeros(64, 128, device=dev, dtype=BF)
    lse = torch.zeros(1, 2, 64, device=dev)
    with pytest.raises(_cabi.Sb200Error, match="exceeds a row"):
        ops.attention_bwd(q, q, q, q, q, lse, 1, 2, 64, 64, 0.125, 64, torch.zeros(128, 64, device=dev, dtype=BF))
    with pytest.raises(ValueError, match="row-strided"):
        ops.layernorm_bwd(q, q[0], q, out=q.t())


def test_splitk_and_optimizer_arguments_return_errors(dev):
    """The split-K GEMM stores 16-byte vectors to out and ws: a misaligned pointer is refused on the host, before any
    launch; the optimisers refuse more tensors than the grid's y dimension holds."""
    from sliders_b200 import _cabi, ops
    from test_gpu_backward_bounds import _lib_call

    M, N, K = 77, 64, 128
    x = torch.zeros(M, K, device=dev, dtype=BF)
    w = torch.zeros(N, K, device=dev, dtype=BF)
    wide = torch.zeros(M, N + 8, device=dev)
    with pytest.raises(_cabi.Sb200Error, match="16-byte aligned"):   # ldo = 72 is fine, the start 8 bytes off
        ops.gemm_splitk_f32(x, w, out=wide[:, 2:2 + N])
    n_ws = ops.splitk_ws_floats(M, N, K)
    ws = torch.zeros(n_ws + 4, device=dev)
    out = torch.zeros(M, N, device=dev)
    with pytest.raises(_cabi.Sb200Error, match="16-byte aligned"):
        _lib_call("sb200_gemm_splitk_f32", ops._p(x), K, ops._p(w), K, ops._p(out), N, M, N, K, ops._p(ws[1:]), n_ws)
    with pytest.raises(ValueError, match="row-strided"):
        ops.gemm_splitk_f32(x, w, out=torch.zeros(M, N, device=dev, dtype=BF))
    with pytest.raises(ValueError, match="row-strided"):
        ops.gemm_splitk_f32(x, w, out=torch.zeros(N, M, device=dev).t())
    with pytest.raises(ValueError, match="is on cpu"):
        ops.gemm_splitk_f32(x, w, out=torch.zeros(M, N))
    table = torch.zeros(1, 5, device=dev, dtype=torch.int64)
    with pytest.raises(_cabi.Sb200Error, match="65535"):
        ops.adamw(table, 65536, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1)
    with pytest.raises(_cabi.Sb200Error, match="65535"):
        ops.adam_f32(table, 65536, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1)
    torch.cuda.synchronize()
    assert torch.equal(out, torch.zeros_like(out)) and torch.equal(ws, torch.zeros_like(ws))
