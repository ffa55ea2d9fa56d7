"""Element-by-element tests of the kernels that write weights and the ones behind null-text inversion: the split-K fp32
GEMM (d loss / d encoder_hidden_states), the guided-step loss and its gradient, the fused bf16 AdamW and the fp32 Adam.

Every variant table row
- asserts the launch quantities it is listed for, with Python mirrors of the host formulas (`splitk_kb`, `loss_parts`,
  `adamw_bx`, `adam_grid`, ...), so a label cannot drift from what runs;
- writes its outputs between guard bands (fp32: F32_NAN_BITS, bf16: NAN_BITS) and checks that nothing outside them
  changed and that every output element was written;
- runs twice and checks that both runs agree bit for bit (every reduction here has a fixed order, no atomics).
Two data regimes:
- exact data (small integers, or half-integers for the loss): every partial sum is an integer (a multiple of 1/4)
  below 2^24, so fp32 arithmetic in any order is exact and the kernel must equal the float64 result bit for bit;
- Gaussian data, checked against per-element bounds derived from each kernel's fp32 chain (`chain_c`).
AdamW stays bit-exact against torch.optim.AdamW(foreach=True), as optim.py documents.
tests/test_inversion_optim_bounds.py checks, without a GPU, that the bounds accept a CPU emulation of each kernel's
roundings and reject planted local errors, that the exact regimes are exact, and that the tables cover every variant."""
import functools
import math

import pytest
import torch

from test_gpu_backward_bounds import (F32_NAN_BITS, _lib_call, _outside, assert_bitwise, assert_flat_guard,
                                      assert_no_violations, cdiv, chain_c, flat_guarded)
from test_gpu_kernels import GUARD_COLS, GUARD_ROWS, NAN_BITS

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
F32 = torch.float32

# ------------------------------------------------------------------------------------------------------------------
# the host code's launch formulas (include/sb200.h, gemm.cu, elementwise.cu, backward.cu)
# ------------------------------------------------------------------------------------------------------------------
def splitk_bn(N):
    """sb200_gemm_splitk_f32: 128-column tiles when N % 128 == 0, else 64 (the last one may be narrower than 64)."""
    return 128 if N % 128 == 0 else 64


def splitk_tiles(M, N):
    """SB200_GEMM_SPLITK_TILES."""
    return cdiv(M, 128) * (N // 128 if N % 128 == 0 else cdiv(N, 64))


def splitk_kb_unclamped(M, N, K):
    """SB200_GEMM_SPLITK_KB_: k-blocks per split for about one wave of 132 CTAs."""
    return cdiv(cdiv(K, 64), cdiv(132, splitk_tiles(M, N)))


def splitk_kb(M, N, K):
    """SB200_GEMM_SPLITK_KB: at least 8 k-blocks per split."""
    return max(8, splitk_kb_unclamped(M, N, K))


def splitk_splits(M, N, K):
    """SB200_GEMM_SPLITK_SPLITS."""
    return cdiv(cdiv(K, 64), splitk_kb(M, N, K))


def splitk_ranges(M, N, K):
    """[k0, k1) element ranges of the splits: split s runs k-blocks [s kb, min((s + 1) kb, kblocks)), the last one
    ending at K (the TMA zero-fills the K tail of the last k-block)."""
    kb, kbs = splitk_kb(M, N, K), cdiv(K, 64)
    return [(s * kb * 64, min(min((s + 1) * kb, kbs) * 64, K)) for s in range(splitk_splits(M, N, K))]


def loss_parts(n):
    """SB200_GUIDED_LOSS_BLOCKS: mode-0 blocks (and partial sums)."""
    return min(n // 2048 + 1, 256)


def loss_mode1_blocks(n):
    """Mode-1 grid of sb200_guided_step_loss: one thread per element, at most 1024 blocks (above 262 144 elements the
    grid-stride loop wraps)."""
    return min(cdiv(n, 256), 1024)


def loss_chain(n):
    """Dependent fp32 roundings of the mode-0 loss: a thread's strided FMAs, the 8-level block tree, the 8-level
    finalize tree over the partials, the division by n."""
    return cdiv(n, loss_parts(n) * 256) + 8 + 8 + 1


def adamw_bx(max_numel):
    """sb200_adamw: blocks per tensor, min(ceil(max_numel / 256), 64); a larger tensor wraps the grid-stride loop."""
    return min(cdiv(max_numel, 256), 64)


def adam_grid(max_numel, sms):
    """sb200_adam_f32: grid_for(max_numel, 256, sms), capped at 16 blocks per SM."""
    return max(1, min(cdiv(max_numel, 256), sms * 16))


KV_K = {"tiny_sd": 4992, "tiny_xl": 11776, "sd15": 24960, "sdxl": 166400}  # K of each UNet's stacked to_k | to_v


# ------------------------------------------------------------------------------------------------------------------
# variant tables
# ------------------------------------------------------------------------------------------------------------------
# (M, N, K, views, bn, kb, splits): views "x" / "w": the operand is a column view of a wider NaN-filled buffer
# (ld > K); "o": out is a column slice of a wider guarded fp32 buffer (ldo > N, starting 8 floats in)
SPLITK_MATRIX = [
    (1, 16, 520, "xwo", 64, 8, 2),            # one row, a 16-column tile, K % 64 = 8, last split one k-block
    (77, 48, 440, "", 64, 8, 1),              # K % 64 = 56 below 8 k-blocks: a single split
    (127, 80, 4096, "x", 64, 8, 8),           # kb clamped to 8 (1 wanted), two 64-column tiles, the second 16 wide
    (128, 1040, 2112, "wo", 64, 8, 5),        # 17 tiles of 64 (the last 16 wide), last split one k-block
    (616, 48, 1080, "xwo", 64, 8, 3),         # five row tiles, K % 64 = 56, short last split
    (129, 1040, 24968, "xw", 64, 98, 4),      # bn = 64 unclamped, K % 64 = 8, last split 97 k-blocks
    (154, 128, KV_K["tiny_sd"], "xo", 128, 8, 10),
    (77, 256, KV_K["tiny_xl"], "w", 128, 8, 23),
    (77, 768, KV_K["sd15"], "x", 128, 18, 22),
    (154, 768, KV_K["sd15"], "", 128, 36, 11),
    (616, 768, KV_K["sd15"], "o", 128, 78, 5),
    (616, 256, 3000, "xwo", 128, 8, 6),
    (1, 2048, 6400, "", 128, 12, 9),
    (77, 2048, KV_K["sdxl"], "", 128, 289, 9),
    (154, 2048, KV_K["sdxl"], "xwo", 128, 520, 5),
]

# (n, parts, mode-1 blocks, mode-1 wraps)
LOSS_MATRIX = [
    (1, 1, 1, False),
    (255, 1, 1, False),
    (257, 1, 2, False),
    (2047, 1, 8, False),
    (2048, 2, 8, False),
    (2049, 2, 9, False),
    (65536, 33, 256, False),     # SDXL latent [1, 4, 128, 128]
    (300000, 147, 1024, True),   # the mode-1 grid wraps
    (522240, 256, 1024, True),   # the smallest n whose parts cap at 256
    (600001, 256, 1024, True),
]

# (g, ce, dloss): the inversion's guidance and Euler-like step, then the edges
LOSS_PARAMS = [(7.5, -0.0421, 2.5), (0.0, 0.37, 1.0), (1.0, -0.0421, 1.0), (7.5, 0.0, -0.75)]

# (table, grads, weight_decay, betas, bx, wraps): table "sdxl-r<rank>-<method>" is the parameter list of that
# LoRANetwork (c3lier) on the full-size SDXL UNet; grads "bf16", "fp32" (optim.AdamW casts them) or "flat" (views at
# odd offsets into one flat buffer, as the all-reduce leaves them).  A second group with the other weight decay, twice
# the lr and some grads None rides along in every row.
ADAMW_MATRIX = [
    ("sdxl-r4-noxattn", "bf16", 1e-2, (0.9, 0.999), 64, True),
    ("sdxl-r4-full", "fp32", 0.0, (0.5, 0.99), 64, True),   # beta1 <= 0.5: torch's lerp takes its other branch
    ("sdxl-r16-noxattn", "flat", 1e-2, (0.3, 0.9), 64, True),
    ("sdxl-r16-full", "flat", 0.0, (0.9, 0.999), 64, True),
    ("small", "fp32", 1e-2, (0.9, 0.999), 45, False),
]
SMALL_SHAPES = [(4, 1280), (1280, 4), (4, 320, 3, 3), (640, 4, 1, 1), (8, 77), (1,)]

ADAM_STEPS = [1, 2, 10, 1000]
ADAM_WDS = [0.0, 0.1]


def adam_sizes(sms):
    """fp32 Adam table: one element, a partial block, the inversion's [1, 77, 768] embedding, and one tensor past the
    grid cap (the grid-stride loop wraps)."""
    return [1, 1000, 77 * 768, sms * 16 * 256 + 4097]


# ------------------------------------------------------------------------------------------------------------------
# inputs and float64 references (device-agnostic: the CPU tests run them too)
# ------------------------------------------------------------------------------------------------------------------
def splitk_exact_inputs(M, N, K, gen, device):
    """x [M, K], w [N, K] bf16 with integer values in [-2, 2]: every product and partial sum is an integer of magnitude
    at most 4 K < 2^24, so fp32 accumulation in any order is exact."""
    x = torch.randint(-2, 3, (M, K), generator=gen, device=device).to(BF)
    w = torch.randint(-2, 3, (N, K), generator=gen, device=device).to(BF)
    return x, w


def splitk_split_refs(x, w, ranges):
    """float64 (product, |x| |w|^T) of each split's k-range."""
    out = []
    for k0, k1 in ranges:
        xs, ws = x[:, k0:k1].double(), w[:, k0:k1].double()
        out.append((xs @ ws.t(), xs.abs() @ ws.abs().t()))
    return out


def splitk_split_chain(k0, k1):
    """Roundings allowed for one split tile: test_gpu_kernels.bound_violations allows 2^-12 / 2^-24 = 4096 roundings
    for 1080 wgmma k16 steps (about 4 per step); chain_c(2 steps) is the same 4 x 2^-24 per k16 step."""
    return 2 * cdiv(k1 - k0, 16)


def splitk_out_chain(M, N, K):
    """out = the in-order sum of the splits: the longest split's chain plus one rounding per added split."""
    return max(splitk_split_chain(k0, k1) for k0, k1 in splitk_ranges(M, N, K)) + splitk_splits(M, N, K)


def splitk_reduce(ws):
    """The kernel's claimed reduction: ((ws[0] + ws[1]) + ws[2]) + ... in fp32."""
    acc = ws[0].clone()
    for s in range(1, ws.shape[0]):
        acc = acc + ws[s]
    return acc


def loss_exact_inputs(n, gen, device):
    """eps_u, eps_c, x, target fp32 with values in {-1, 0, 1}: with cx = ce = 1, g = 0.5 every residual is a
    half-integer and every square a multiple of 1/4; E[(2 r)^2] = 20 / 3, so 4 S < 2^24 up to n of about 2.5 M."""
    return [torch.randint(-1, 2, (n,), generator=gen, device=device).float() for _ in range(4)]


def loss_exact_sum(eu, ec, x, t):
    """S = sum of the squared residuals at cx = ce = 1, g = 0.5, in float64 (exact)."""
    r = x.double() + 0.5 * eu.double() + 0.5 * ec.double() - t.double()
    return float((r * r).sum())


def f32(v):
    """v rounded to fp32, as the kernel receives its float arguments."""
    return float(torch.tensor(v, dtype=F32))


def guided_ref(eu, ec, g, x, cx, ce, t, dloss):
    """float64 (residual, its magnitude, k = dloss (1 - g) ce 2 / n) of the guided step, from the fp32 scalars."""
    eu, ec, x, t = eu.double(), ec.double(), x.double(), t.double()
    r = cx * x + ce * (eu + g * (ec - eu)) - t
    mag = abs(cx) * x.abs() + abs(ce) * (eu.abs() + abs(g) * (ec.abs() + eu.abs())) + t.abs()
    return r, mag, dloss * (1 - g) * ce * 2 / eu.numel()


def guided_loss_violation(loss, r, mag, n):
    """Is the scalar loss outside |loss - mean r^2| <= chain_c(loss_chain(n) + 16) mean(mag^2)?  Each residual takes 7
    fp32 roundings of terms bounded by mag, so r^2 errs by at most 15 2^-24 mag^2 before the reduction; the reduction
    chain adds loss_chain(n) roundings of partial sums of at most sum(mag^2).  This is the worst case, every rounding at
    its largest and of one sign; on Gaussian data the errors cancel like a random walk and stay about 100x below it
    (measured on an H100: 0.010 of the bound), while a dropped block partial is 1 / parts of the loss, far above it."""
    ref = (r * r).mean().reshape(1)
    bound = chain_c(loss_chain(n) + 16) * (mag * mag).mean().reshape(1)
    return bool(_outside((torch.as_tensor(loss, dtype=torch.float64).reshape(1).to(ref.device) - ref).abs(), bound,
                         "guided_loss")[0])


def guided_grad_violations(d, r, mag, k):
    """Bool mask of d_eps_u outside |d - k r| <= chain_c(12) |k| mag: k takes 4 roundings, r 7 (relative to mag), the
    product 1."""
    return _outside((d.double() - k * r).abs(), chain_c(12) * abs(k) * mag, "guided_grad")


def adam_f32_ref(p, g, m, v, lr, b1, b2, eps, wd, step):
    """float64 torch.optim.Adam step (L2 weight decay in the gradient) and per-element bounds on the error of the fp32
    kernel: returns (p', m', v', bound_p, bound_m, bound_v).
    - g' = g + wd p: 2 roundings of terms of at most G = |g| + wd |p|, so g' errs by 2 2^-24 G even when it cancels;
    - m' = m + (1 - b1)(g' - m): 3 more roundings and the fp32 (1 - b1): within 6 2^-24 mag_m,
      mag_m = |m| + (1 - b1)(G + |m|);
    - v' = b2 v + (1 - b2) g'^2: 4 roundings, 2 fp32 scalars and the error of g' squared (2 |g'| 2 2^-24 G <= 4 2^-24
      G^2): within 10 2^-24 mag_v, mag_v = b2 v + (1 - b2) G^2.  When g' cancels and v is tiny, v' is far below mag_v
      and this is a large relative error of v';
    - sqrt(v'): an absolute error dv of v' moves the root by at most min(dv / sqrt(v'), sqrt(dv)), plus its own
      rounding; denom = sqrt(v') / bc2 + eps adds 4 relative roundings (the fp32 bc2 and eps, the division, the add),
      so the kernel's denom is within dd of denom and at least lo = max(denom - dd, eps);
    - p' = p - step m' / denom: m' / denom errs by at most (err_m + |m'| dd / denom) / lo, and the division, the fp32
      step, the product and the add are 4 more roundings of terms of at most |p| + step mag_m / lo.
    Every term takes the factor 2 of `chain_c`."""
    U = 2.0 ** -24
    p, g, m, v = p.double(), g.double(), m.double(), v.double()
    gg = g + wd * p
    gmag = g.abs() + wd * p.abs()
    m1 = m + (1 - b1) * (gg - m)
    v1 = b2 * v + (1 - b2) * gg * gg
    bc2 = math.sqrt(1 - b2 ** step)
    root = v1.sqrt()
    denom = root / bc2 + eps
    ss = lr / (1 - b1 ** step)
    p1 = p - ss * m1 / denom
    mag_m = m.abs() + (1 - b1) * (gmag + m.abs())
    bound_m = chain_c(6) * mag_m
    bound_v = chain_c(10) * (b2 * v + (1 - b2) * gmag * gmag)
    droot = torch.minimum(bound_v / root.clamp(min=1e-300), bound_v.sqrt()) + chain_c(1) * (root + bound_v.sqrt())
    dd = droot / bc2 + chain_c(4) * (denom + droot / bc2)
    lo = torch.clamp(denom - dd, min=eps * (1 - chain_c(2)))
    bound_p = 2 * ss * (bound_m + mag_m * dd / denom) / lo + chain_c(4) * (p.abs() + ss * mag_m / lo)
    return p1, m1, v1, bound_p, bound_m, bound_v


def adam_f32_violations(p1, m1, v1, ref):
    """Bool masks of the fp32 Adam outputs outside the bounds of `adam_f32_ref`."""
    rp, rm, rv, bp, bm, bv = ref
    return (_outside((p1.double() - rp).abs(), bp, "adam_f32_p"),
            _outside((m1.double() - rm).abs(), bm, "adam_f32_m"),
            _outside((v1.double() - rv).abs(), bv, "adam_f32_v"))


def _fma(a, b, c):
    """fl32(a b + c) for fp32 operands: a b is exact in float64, so only the final roundings remain (float64, then fp32;
    the double rounding differs from a true fused multiply-add in about 2^-29 of the cases)."""
    return (torch.as_tensor(a, dtype=torch.float64) * b.double() + c.double()).float()


def adamw_emulation(p, g, m, v, lr, b1, b2, eps, wd, step, order="cuda", round_m=True):
    """torch.optim.AdamW on bf16 tensors (one step, every materialised tensor rounded to bf16) in fp32 with the fused
    multiply-adds of torch's kernels.  lerp is fma(w, g - m, m) for w = 1 - b1 < 0.5, else fma(-b1, g - m, g).  torch's
    CUDA kernels and adamw_kernel (order "cuda") compute addcmul as fma(1 - b2, g g, v) and addcdiv as
    fma(-step, m / denom, p); torch's CPU kernels (order "cpu") as fma((1 - b2) g, g, v) and p + (-step m) / denom.
    round_m=False plants the error of an exp_avg whose bf16 rounding is skipped before it reaches the parameter update.
    Returns bf16 (p', m', v')."""
    rb = lambda a: a.to(BF).float()  # noqa: E731
    pf, gf, mf, vf = p.float(), g.float(), m.float(), v.float()
    pf = rb(pf * f32(1 - lr * wd))
    w = 1 - b1
    m_full = _fma(f32(w), gf - mf, mf) if w < 0.5 else _fma(-f32(b1), gf - mf, gf)
    mf = rb(m_full)
    vb = rb(vf * f32(b2))
    vf = rb(_fma(f32(1 - b2), gf * gf, vb) if order == "cuda" else _fma(f32(1 - b2) * gf, gf, vb))
    denom = rb(rb(rb(vf.sqrt()) / f32(math.sqrt(1 - b2 ** step))) + f32(eps))
    ms = mf if round_m else m_full
    nss = f32(-lr / (1 - b1 ** step))
    pf = rb(_fma(nss, ms / denom, pf) if order == "cuda" else pf + (nss * ms) / denom)
    return pf.to(BF), mf.to(BF), vf.to(BF)


@functools.lru_cache(maxsize=None)
def sdxl_lora_shapes(rank, method):
    """Shapes of LoRANetwork(rank, train_method, c3lier).prepare_optimizer_params() on the full-size SDXL UNet, built
    on the meta device (no memory, no initialisation)."""
    from conftest import c3lier
    from oracle import unet as ounet
    from sliders_b200 import lora as plora
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    with torch.device("meta"), c3lier(plora):
        unet = UNet2DConditionModel(UNetConfig.from_dict(ounet.UNetConfig.sdxl().__dict__))
        net = plora.LoRANetwork(unet, rank=rank, multiplier=1.0, alpha=1.0, train_method=method)
    return tuple(tuple(p.shape) for grp in net.prepare_optimizer_params() for p in grp["params"])


def adamw_table_shapes(table):
    if table == "small":
        return tuple(SMALL_SHAPES)
    _, r, method = table.split("-")
    return sdxl_lora_shapes(int(r[1:]), method)


# ------------------------------------------------------------------------------------------------------------------
# GPU machinery
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def nan_col_view(t, pad):
    """t [rows, cols] bf16 as a column view of a wider buffer (row stride cols + pad, first column pad // 2 rounded
    down to 8) whose other columns hold NaN: a kernel that reads past the view's columns meets NaN."""
    if not pad:
        return t.contiguous()
    rows, cols = t.shape
    lo = (pad // 2) // 8 * 8
    buf = torch.full((rows, cols + pad), NAN_BITS, dtype=torch.int16, device=t.device).view(BF)
    buf[:, lo:lo + cols] = t
    return buf[:, lo:lo + cols]


def guarded_f32_slice(rows, cols, lo, dev):
    """(buffer, view): a [rows, cols] fp32 view starting at column lo of a buffer with GUARD_ROWS more rows above and
    below and GUARD_COLS more columns on the right, all F32_NAN_BITS."""
    buf = torch.full((rows + 2 * GUARD_ROWS, lo + cols + GUARD_COLS), F32_NAN_BITS, dtype=torch.int32,
                     device=dev).view(F32)
    return buf, buf[GUARD_ROWS:GUARD_ROWS + rows, lo:lo + cols]


def assert_guard_f32_slice(buf, rows, cols, lo):
    bits = buf.view(torch.int32)
    guard = torch.ones_like(bits, dtype=torch.bool)
    guard[GUARD_ROWS:GUARD_ROWS + rows, lo:lo + cols] = False
    n = int((bits[guard] != F32_NAN_BITS).sum())
    assert n == 0, f"{n} elements written outside the [{rows}, {cols}] output"
    assert not torch.isnan(buf[GUARD_ROWS:GUARD_ROWS + rows, lo:lo + cols]).any(), "NaN in the output (unwritten?)"


def packed_guarded(sizes, dtype, dev, gap=37):
    """(buffer, views, guard mask): contiguous 1-D views of the given sizes inside one buffer, each preceded and the
    last followed by `gap` guard elements (an odd gap: the views start at arbitrary alignments), all NaN bits."""
    ib = torch.int16 if dtype == BF else torch.int32
    pat = NAN_BITS if dtype == BF else F32_NAN_BITS
    total = sum(sizes) + gap * (len(sizes) + 1)
    buf = torch.full((total,), pat, dtype=ib, device=dev).view(dtype)
    guard = torch.ones(total, dtype=torch.bool, device=dev)
    views, off = [], gap
    for n in sizes:
        views.append(buf[off:off + n])
        guard[off:off + n] = False
        off += n + gap
    return buf, views, guard


def assert_packed_guard(buf, guard):
    bits = buf.view(torch.int16 if buf.dtype == BF else torch.int32)
    pat = NAN_BITS if buf.dtype == BF else F32_NAN_BITS
    n = int((bits[guard] != pat).sum())
    assert n == 0, f"{n} guard elements changed"
    assert not torch.isnan(buf[~guard]).any(), "NaN inside a tensor (unwritten?)"


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == BF else torch.int32)


# ------------------------------------------------------------------------------------------------------------------
# 1. split-K fp32 GEMM
# ------------------------------------------------------------------------------------------------------------------
def _splitk_id(row):
    M, N, K, views, *_ = row
    return f"{M}x{N}x{K}" + (f"-{views}" if views else "")


def _run_splitk(x, w, M, N, K, splits, views, dev):
    """Two calls, each into a fresh guarded out and a fresh NaN-filled ws; returns (out, ws [splits, M, N])."""
    from sliders_b200 import ops

    P = ops._p
    lo = 8 if "o" in views else 0
    n_ws = splits * M * N
    runs = []
    for _ in range(2):
        obuf, out = guarded_f32_slice(M, N, lo, dev)
        wbuf, ws = flat_guarded(n_ws, F32, dev)
        _lib_call("sb200_gemm_splitk_f32", P(x), x.stride(0), P(w), w.stride(0), P(out), out.stride(0), M, N, K,
                  P(ws), n_ws)
        torch.cuda.synchronize()
        assert_guard_f32_slice(obuf, M, N, lo)
        assert_flat_guard(wbuf, n_ws)  # also: no NaN left in ws, so every (s, m < M, n < N) was written
        runs.append((out.clone(), ws.view(splits, M, N).clone()))
    assert_bitwise(runs[0][0], runs[1][0], "gemm_splitk_f32 out")
    assert_bitwise(runs[0][1], runs[1][1], "gemm_splitk_f32 ws")
    return runs[0]


@pytest.mark.parametrize("M,N,K,views,bn,kb,splits", SPLITK_MATRIX, ids=[_splitk_id(r) for r in SPLITK_MATRIX])
def test_gemm_splitk_f32_bound(dev, M, N, K, views, bn, kb, splits):
    from sliders_b200 import ops

    assert (splitk_bn(N), splitk_kb(M, N, K), splitk_splits(M, N, K)) == (bn, kb, splits)
    assert ops.splitk_ws_floats(M, N, K) == splits * M * N
    ranges = splitk_ranges(M, N, K)
    gen = torch.Generator(device=dev).manual_seed(M * 7 + N + K)

    # exact data: each split tile and out equal the float64 products bit for bit
    xe, we = splitk_exact_inputs(M, N, K, gen, dev)
    x, w = nan_col_view(xe, 40 if "x" in views else 0), nan_col_view(we, 24 if "w" in views else 0)
    assert ("x" in views) == (x.stride(0) > K) and ("w" in views) == (w.stride(0) > K)
    out, ws = _run_splitk(x, w, M, N, K, splits, views, dev)
    for s, (ref, _) in enumerate(splitk_split_refs(x, w, ranges)):
        bad = ws[s].double() != ref
        assert not bad.any(), f"split {s} (k {ranges[s]}): {int(bad.sum())} elements differ from the exact product"
    ref = x.double() @ w.double().t()
    assert torch.equal(out.double(), ref), f"out: {int((out.double() != ref).sum())} elements differ (exact data)"
    # the wrapper passes the same strides: same bits into a column slice
    wrap = torch.full((M, N + 16), float("nan"), device=dev)[:, 8:8 + N]
    assert ops.gemm_splitk_f32(x, w, out=wrap) is wrap
    assert_bitwise(wrap, out, "ops.gemm_splitk_f32 vs the C ABI call")

    # Gaussian data: per-split bounds, and out is the in-order fp32 sum of the splits bit for bit
    x = nan_col_view(torch.randn(M, K, generator=gen, device=dev).to(BF), 40 if "x" in views else 0)
    w = nan_col_view((torch.randn(N, K, generator=gen, device=dev) * 0.05).to(BF), 24 if "w" in views else 0)
    out, ws = _run_splitk(x, w, M, N, K, splits, views, dev)
    for s, (ref, mag) in enumerate(splitk_split_refs(x, w, ranges)):
        bad = _outside((ws[s].double() - ref).abs(), chain_c(splitk_split_chain(*ranges[s])) * mag, "splitk_split")
        assert_no_violations(bad, ws[s], ref, f"split {s} of {splits}")
    assert torch.equal(_bits(out), _bits(splitk_reduce(ws))), "out is not the in-order fp32 sum of the splits"
    xd, wd = x.double(), w.double()
    ref, mag = xd @ wd.t(), xd.abs() @ wd.abs().t()
    bad = _outside((out.double() - ref).abs(), chain_c(splitk_out_chain(M, N, K)) * mag, "splitk_out")
    assert_no_violations(bad, out, ref, "gemm_splitk_f32 out")


# ------------------------------------------------------------------------------------------------------------------
# 2. guided-step loss (null-text inversion's inner loss)
# ------------------------------------------------------------------------------------------------------------------
def _guided_call(eu, ec, g, x, cx, ce, t, n, mode, dloss=None):
    """One call into guarded buffers; returns (loss, ws partials) for mode 0, d_eps_u for mode 1."""
    from sliders_b200 import ops

    P = ops._p
    dev = eu.device
    if mode == 0:
        parts = loss_parts(n)
        lbuf, loss = flat_guarded(1, F32, dev)
        wbuf, ws = flat_guarded(parts, F32, dev)
        _lib_call("sb200_guided_step_loss", P(eu), P(ec), g, P(x), cx, ce, P(t), n, 0, P(loss), P(ws), None, None)
        torch.cuda.synchronize()
        assert_flat_guard(lbuf, 1)
        assert_flat_guard(wbuf, parts)
        return loss.clone(), ws.clone()
    dbuf, d = flat_guarded(n, F32, dev)
    _lib_call("sb200_guided_step_loss", P(eu), P(ec), g, P(x), cx, ce, P(t), n, 1, None, None, P(dloss), P(d))
    torch.cuda.synchronize()
    assert_flat_guard(dbuf, n)
    return d.clone()


def _check_loss_row(n, parts, blocks1, wraps):
    assert (loss_parts(n), loss_mode1_blocks(n), n > blocks1 * 256) == (parts, blocks1, wraps)


@pytest.mark.parametrize("n,parts,blocks1,wraps", LOSS_MATRIX)
def test_guided_loss_exact(dev, n, parts, blocks1, wraps):
    """cx = ce = 1, g = 0.5, inputs in {-1, 0, 1}: the loss is float32(S) / float32(n) exactly and d_eps_u is
    fl(fl(dloss (1 - g) ce 2 / n) r) exactly, for every element, block partial and tail."""
    _check_loss_row(n, parts, blocks1, wraps)
    gen = torch.Generator(device=dev).manual_seed(n)
    eu, ec, x, t = loss_exact_inputs(n, gen, dev)
    S = loss_exact_sum(eu, ec, x, t)
    assert 4 * S < 2 ** 24
    want = torch.tensor(S, dtype=F32) / torch.tensor(float(n), dtype=F32)
    runs = [_guided_call(eu, ec, 0.5, x, 1.0, 1.0, t, n, 0) for _ in range(2)]
    assert_bitwise(runs[0][0], runs[1][0], "guided loss")
    assert_bitwise(runs[0][1], runs[1][1], "guided loss partials")
    assert _bits(runs[0][0].cpu()).item() == _bits(want).item(), f"loss {runs[0][0].item()!r}, want {want.item()!r}"
    dloss = torch.tensor([1.0], device=dev)
    ds = [_guided_call(eu, ec, 0.5, x, 1.0, 1.0, t, n, 1, dloss) for _ in range(2)]
    assert_bitwise(ds[0], ds[1], "guided loss d_eps_u")
    k = torch.tensor(1.0, dtype=F32) * 0.5 * 1.0 * 2.0 / torch.tensor(float(n), dtype=F32)
    r = x + 0.5 * eu + 0.5 * ec - t  # exact in fp32
    assert torch.equal(_bits(ds[0]), _bits(k.to(dev) * r)), "d_eps_u differs from fl(k r)"


def _guided_gauss(dev, n, g, ce, dl):
    gen = torch.Generator(device=dev).manual_seed(n + 1)
    eu, ec, x, t = (torch.randn(n, generator=gen, device=dev) for _ in range(4))
    g, cx, ce, dl = f32(g), f32(1.0137), f32(ce), f32(dl)
    r, mag, k = guided_ref(eu, ec, g, x, cx, ce, t, dl)
    runs = [_guided_call(eu, ec, g, x, cx, ce, t, n, 0) for _ in range(2)]
    assert_bitwise(runs[0][0], runs[1][0], "guided loss")
    assert not guided_loss_violation(runs[0][0].item(), r, mag, n), \
        f"loss {runs[0][0].item()!r}, want {(r * r).mean().item()!r}"
    dloss = torch.tensor([dl], device=dev)
    ds = [_guided_call(eu, ec, g, x, cx, ce, t, n, 1, dloss) for _ in range(2)]
    assert_bitwise(ds[0], ds[1], "guided loss d_eps_u")
    if g == 1.0 or ce == 0.0:
        assert bool((ds[0] == 0).all()), "d_eps_u must be exactly 0 when (1 - g) ce = 0"
    else:
        assert_no_violations(guided_grad_violations(ds[0], r, mag, k), ds[0], k * r, "d_eps_u")


@pytest.mark.parametrize("n,parts,blocks1,wraps", LOSS_MATRIX)
def test_guided_loss_bound(dev, n, parts, blocks1, wraps):
    _check_loss_row(n, parts, blocks1, wraps)
    _guided_gauss(dev, n, *LOSS_PARAMS[0])


@pytest.mark.parametrize("n", [257, 600001])
@pytest.mark.parametrize("g,ce,dl", LOSS_PARAMS[1:])
def test_guided_loss_edges(dev, n, g, ce, dl):
    """g = 0 (unguided), g = 1 (d_eps_u exactly 0), ce = 0 (x_rec = cx x: d_eps_u exactly 0), dloss != 1."""
    _guided_gauss(dev, n, g, ce, dl)


# ------------------------------------------------------------------------------------------------------------------
# 3. AdamW on bf16 (bit-exact against torch.optim.AdamW(foreach=True))
# ------------------------------------------------------------------------------------------------------------------
def _cat_bits(ts):
    return torch.cat([_bits(t).reshape(-1) for t in ts]) if ts else torch.empty(0)


def _assert_same(ref_ts, my_ts, what):
    a, b = _cat_bits(ref_ts), _cat_bits(my_ts)
    n = int((a != b).sum())
    assert n == 0, f"{what}: {n} of {a.numel()} elements differ from torch.optim.AdamW"


@pytest.mark.parametrize("table,grads,wd,betas,bx,wraps", ADAMW_MATRIX, ids=[r[0] + "-" + r[1] for r in ADAMW_MATRIX])
def test_adamw_matches_torch_bitwise(dev, table, grads, wd, betas, bx, wraps):
    """Three steps with an lr scheduler changing lr between them; group 0 takes `wd`, group 1 (every third tensor) the
    other weight decay and twice the lr, and every sixth tensor never gets a gradient (it and its state stay untouched).
    Parameters and both moments must equal torch's bit for bit after every step."""
    from sliders_b200 import optim

    shapes = adamw_table_shapes(table)
    numels = [math.prod(s) for s in shapes]
    assert adamw_bx(max(numels)) == bx and (max(numels) > bx * 256) == wraps
    gen = torch.Generator(device=dev).manual_seed(len(shapes) + int(1e4 * wd) + int(100 * betas[0]))
    p0 = [(torch.randn(s, generator=gen, device=dev) * 0.1).to(BF) for s in shapes]
    ref_p = [torch.nn.Parameter(p.clone()) for p in p0]
    my_p = [torch.nn.Parameter(p.clone()) for p in p0]
    idle = {i for i in range(len(shapes)) if i % 6 == 5}
    wd1 = 1e-2 if wd == 0 else 0.0

    def groups(ps):
        return [{"params": [p for i, p in enumerate(ps) if i % 3 != 2]},
                {"params": [p for i, p in enumerate(ps) if i % 3 == 2], "weight_decay": wd1, "lr": 4e-4}]

    ref_opt = torch.optim.AdamW(groups(ref_p), lr=2e-4, betas=betas, weight_decay=wd, foreach=True)
    my_opt = optim.AdamW(groups(my_p), lr=2e-4, betas=betas, weight_decay=wd)
    scheds = [torch.optim.lr_scheduler.LambdaLR(o, lambda s: 1.0 / (1 + 0.7 * s)) for o in (ref_opt, my_opt)]
    live = [i for i in range(len(shapes)) if i not in idle]
    total = sum(numels[i] for i in live)
    if grads == "fp32":
        for p in my_p:
            p.grad_dtype = None  # let the bf16 parameters hold fp32 gradients
    for step, scale in enumerate((1.0, 0.01, 3.0)):
        if grads == "flat":   # views into one flat buffer at odd offsets
            flat = (torch.randn(total + 7 * len(live), generator=gen, device=dev) * scale).to(BF)
            off, gs = 0, {}
            for j, i in enumerate(live):
                off += j % 7
                gs[i] = flat[off:off + numels[i]].view(shapes[i])
                off += numels[i]
            ref_g = my_g = gs
        else:
            my_g = {i: torch.randn(shapes[i], generator=gen, device=dev) * scale for i in live}
            if grads == "bf16":
                my_g = {i: v.to(BF) for i, v in my_g.items()}
            ref_g = {i: v.to(BF) for i, v in my_g.items()}
        for i in live:
            ref_p[i].grad, my_p[i].grad = ref_g[i], my_g[i]
        ref_opt.step()
        my_opt.step()
        for s in scheds:
            s.step()
        assert ref_opt.param_groups[1]["lr"] == my_opt.param_groups[1]["lr"] != 4e-4
        torch.cuda.synchronize()
        _assert_same([ref_p[i] for i in live], [my_p[i] for i in live], f"step {step}: parameters")
        for key in ("exp_avg", "exp_avg_sq"):
            _assert_same([ref_opt.state[ref_p[i]][key] for i in live], [my_opt.state[my_p[i]][key] for i in live],
                         f"step {step}: {key}")
    _assert_same([p0[i] for i in idle], [my_p[i] for i in idle], "tensors without a gradient")
    assert all(not my_opt.state.get(my_p[i]) for i in idle)


def test_adamw_resumed_at_step_10000(dev):
    """A state resumed at step 9 999: the bias corrections are 1 (bc1) and 1 - 4.5e-5 (bc2); two steps bit for bit."""
    from sliders_b200 import optim

    shapes = [(4, 1280), (20000,), (1280, 4), (3,)]
    gen = torch.Generator(device=dev).manual_seed(10000)
    p0 = [(torch.randn(s, generator=gen, device=dev) * 0.1).to(BF) for s in shapes]
    m0 = [(torch.randn(s, generator=gen, device=dev) * 0.01).to(BF) for s in shapes]
    v0 = [(torch.randn(s, generator=gen, device=dev) * 0.01).square().to(BF) for s in shapes]
    ref_p = [torch.nn.Parameter(p.clone()) for p in p0]
    my_p = [torch.nn.Parameter(p.clone()) for p in p0]
    ref_opt = torch.optim.AdamW(ref_p, lr=2e-4, foreach=True)
    my_opt = optim.AdamW(my_p, lr=2e-4)
    for a, b, m, v in zip(ref_p, my_p, m0, v0):
        ref_opt.state[a] = {"step": torch.tensor(9999.0), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
        my_opt.state[b] = {"step": 9999, "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
    for step in range(2):
        for a, b in zip(ref_p, my_p):
            a.grad = b.grad = (torch.randn(a.shape, generator=gen, device=dev) * 0.1).to(BF)
        ref_opt.step()
        my_opt.step()
        torch.cuda.synchronize()
        _assert_same(ref_p, my_p, f"step {10000 + step}: parameters")
        for key in ("exp_avg", "exp_avg_sq"):
            _assert_same([ref_opt.state[a][key] for a in ref_p], [my_opt.state[b][key] for b in my_p], key)


def _table(rows, dev):
    return torch.tensor([[p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel()] for p, g, m, v in rows],
                        dtype=torch.int64).to(dev)


def test_adamw_guarded_table(dev):
    """ops.adamw on a hand-built table whose p / m / v live between guard bands of one buffer (odd offsets), sizes 1,
    255, 257 and 16 385 (bx = 64: the last wraps the grid-stride loop by one element).  Nothing outside the tensors may
    change; two copies give the same bits; the result equals torch.optim.AdamW's from the same state."""
    from sliders_b200 import ops

    sizes = [1, 255, 257, 16385]
    assert adamw_bx(max(sizes)) == 64 and max(sizes) > 64 * 256
    gen = torch.Generator(device=dev).manual_seed(16385)
    p0 = [(torch.randn(n, generator=gen, device=dev) * 0.1).to(BF) for n in sizes]
    g0 = [(torch.randn(n, generator=gen, device=dev) * 0.1).to(BF) for n in sizes]
    m0 = [(torch.randn(n, generator=gen, device=dev) * 0.01).to(BF) for n in sizes]
    v0 = [(torch.randn(n, generator=gen, device=dev) * 0.01).square().to(BF) for n in sizes]
    lr, b1, b2, eps, wd, step = 3e-4, 0.9, 0.999, 1e-8, 1e-2, 3
    results = []
    for _ in range(2):
        buf, views, guard = packed_guarded(sizes * 3, BF, dev)
        ps, ms, vs = views[:4], views[4:8], views[8:]
        for dst, src in zip(views, p0 + m0 + v0):
            dst.copy_(src)
        gs = [g.clone() for g in g0]
        ops.adamw(_table(list(zip(ps, gs, ms, vs)), dev), 4, max(sizes), lr, b1, b2, eps, wd, step)
        torch.cuda.synchronize()
        assert_packed_guard(buf, guard)
        results.append((buf, ps, ms, vs))
    assert_bitwise(results[0][0], results[1][0], "adamw (guarded table)")
    ref_p = [torch.nn.Parameter(p.clone()) for p in p0]
    ref_opt = torch.optim.AdamW(ref_p, lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=True)
    for a, g, m, v in zip(ref_p, g0, m0, v0):
        ref_opt.state[a] = {"step": torch.tensor(float(step - 1)), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
        a.grad = g.clone()
    ref_opt.step()
    _, ps, ms, vs = results[0]
    _assert_same(ref_p, ps, "parameters")
    _assert_same([ref_opt.state[a]["exp_avg"] for a in ref_p], ms, "exp_avg")
    _assert_same([ref_opt.state[a]["exp_avg_sq"] for a in ref_p], vs, "exp_avg_sq")
    for i in range(len(sizes)):   # the CPU file's emulation, in the CUDA order, is this arithmetic too
        emu = adamw_emulation(p0[i], g0[i], m0[i], v0[i], lr, b1, b2, eps, wd, step)
        _assert_same(list(emu), [ps[i], ms[i], vs[i]], f"adamw_emulation of the {sizes[i]}-element tensor")


# ------------------------------------------------------------------------------------------------------------------
# 4. fp32 Adam (null-text inversion's optimiser)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wd", ADAM_WDS)
@pytest.mark.parametrize("step", ADAM_STEPS)
def test_adam_f32_bound(dev, sms, step, wd):
    """One step from random (p, g, m, v) on a table of four tensors whose p / m / v live between guard bands of one
    buffer, the largest past the grid cap, against the float64 recurrence element by element."""
    from sliders_b200 import ops

    sizes = adam_sizes(sms)
    assert adam_grid(max(sizes), sms) == sms * 16 and max(sizes) > sms * 16 * 256
    gen = torch.Generator(device=dev).manual_seed(100 * step + round(10 * wd))
    p0 = [torch.randn(n, generator=gen, device=dev) for n in sizes]
    g0 = [torch.randn(n, generator=gen, device=dev) * 0.3 for n in sizes]
    m0 = [torch.randn(n, generator=gen, device=dev) * 0.1 for n in sizes]
    v0 = [(torch.randn(n, generator=gen, device=dev) * 0.1).square() for n in sizes]
    lr, b1, b2, eps = 1e-2 * 0.97, 0.9, 0.999, 1e-8
    results = []
    for _ in range(2):
        buf, views, guard = packed_guarded(sizes * 3, F32, dev)
        ps, ms, vs = views[:4], views[4:8], views[8:]
        for dst, src in zip(views, p0 + m0 + v0):
            dst.copy_(src)
        ops.adam_f32(_table(list(zip(ps, g0, ms, vs)), dev), 4, max(sizes), lr, b1, b2, eps, wd, step)
        torch.cuda.synchronize()
        assert_packed_guard(buf, guard)
        results.append((buf, ps, ms, vs))
    assert_bitwise(results[0][0], results[1][0], "adam_f32")
    _, ps, ms, vs = results[0]
    for i, n in enumerate(sizes):
        ref = adam_f32_ref(p0[i], g0[i], m0[i], v0[i], lr, b1, b2, eps, wd, step)
        for bad, got, want, name in zip(adam_f32_violations(ps[i], ms[i], vs[i], ref), (ps[i], ms[i], vs[i]),
                                        ref[:3], ("p", "exp_avg", "exp_avg_sq")):
            assert_no_violations(bad, got, want, f"adam_f32 {name} of the {n}-element tensor")
