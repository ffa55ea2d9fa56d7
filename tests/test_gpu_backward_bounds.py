"""Element-by-element tests of the backward-to-LoRA kernels (csrc/backward.cu, csrc/attention_bwd.cu) against float64
references computed from the same bf16 / fp32 inputs.

Every row of the variant tables below
- writes its outputs twice, each time into a fresh guarded buffer (bf16: the NAN_BITS pattern of test_gpu_kernels.py,
  fp32: F32_NAN_BITS), and checks that no guard element changed, that no output element is NaN and that the two
  calls agree bit for bit (the kernels claim deterministic, atomic-free reductions);
- checks each output element against the bound of its kernel family (the `*_violations` functions, whose docstrings
  derive the constants);
- asserts the launch variant it is listed for, with the host code's own formulas (`ln_nv`, `attn_nd`, `gn_launch`,
  `wgrad_launch`, ...), so a label cannot drift from what runs.
Operands use the call forms of autograd.py: column views with a row stride larger than their width, two-source
(concat) inputs, gradients written into column slices of a wider buffer, and accumulation.
tests/test_backward_bounds.py checks, without a GPU, that the bounds accept a CPU emulation of each kernel's
roundings, reject planted local errors that rel-RMS accepts, and that the tables cover every variant."""
import math
import os

import pytest
import torch

from test_gpu_kernels import GUARD_COLS, GUARD_ROWS, NAN_BITS, assert_guard_intact, guarded_out

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
U = 2.0 ** -24          # fp32 unit roundoff
F32_NAN_BITS = 0x7FA1A5A5  # an fp32 NaN payload no kernel produces: guard bands around fp32 outputs
FLAT_GUARD = 64         # guard elements before and after a contiguous output


def cdiv(a, b):
    return -(-a // b)


MAX_RATIO = {}  # family -> largest err / bound seen in this process (how tight each bound is in practice)


def _outside(err, bound, family):
    ok = err <= bound
    r = err[ok] / bound[ok]
    if r.numel():
        key = (family, os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0])
        MAX_RATIO[key] = max(MAX_RATIO.get(key, 0.0), float(r.max()))
    return ~ok


# ------------------------------------------------------------------------------------------------------------------
# the host code's launch formulas (backward.cu / attention_bwd.cu / include/sb200.h)
# ------------------------------------------------------------------------------------------------------------------
def ln_nv(C):
    """layernorm_bwd_kernel<NV>: 8-channel vectors per lane (sb200_layernorm_bwd)."""
    return 1 if C <= 256 else 3 if C <= 768 else 5 if C <= 1280 else 8


def ln_wraps(M, sms):
    """The grid is capped at 16 blocks of 8 warps (one row each) per SM: more rows than that wrap the row loop."""
    return M > sms * 16 * 8


def attn_nd(d):
    """attention_bwd_kernel<ND>: the head padded to ND x 64 columns."""
    return 1 if d <= 64 else 2 if d <= 128 else 3


def attn_kt(d):
    """Streamed rows per tile (AttnBwdCfg<ND>::kT)."""
    return 32 if attn_nd(d) == 3 else 64


def attn_split(B, heads, Sq, Skv):
    """(nsplit, q_split) of the dK / dV launches of sb200_attention_bwd_ws (attention_bwd_nsplit)."""
    want = min(cdiv(132, B * heads), cdiv(Sq, 64)) if (Skv <= 128 and 2 * B * heads <= 132) else 1
    if want <= 1:
        return 1, 0
    per = cdiv(cdiv(Sq, want), 64) * 64
    return cdiv(Sq, per), per


def gn_launch(B, HW, C, sms):
    """(rows_par, chunks, rows_per_block) of the GroupNorm forward / backward launches (norm.cu, backward.cu)."""
    rows_par = max(1, 512 // (C // 8))
    chunks = min(cdiv(sms * 4, B), 128)
    rpb = max(cdiv(HW, chunks), rows_par * 8)
    return rows_par, cdiv(HW, rpb), rpb


def gn_smem_ok(C):
    """The stats kernels' [rows_par][C][2] fp32 shared memory must fit the default 48 KB."""
    return 8 * C * max(1, 512 // (C // 8)) <= 48 * 1024


def wgrad_launch(rows, C, taps=1):
    """(column blocks, chunks, rows per chunk) of lora_wgrad_kernel / lora_rank_update_kernel (wgrad_chunks); the conv
    form (taps = 9) has the taps in the grid's z dimension, so its chunk count is taken for 9 x the column blocks."""
    cblocks = cdiv(C // 8, 32)
    chunks = min(cdiv(264, cblocks * taps), 256)
    rpb = max(cdiv(rows, chunks), 32)
    return cblocks, cdiv(rows, rpb), rpb


# ------------------------------------------------------------------------------------------------------------------
# bounds
# ------------------------------------------------------------------------------------------------------------------
def pointwise_violations(out, ref, mag, c):
    """Bool mask of the elements outside |out - ref| <= 2^-7 |ref| + c mag (NaN is outside), for kernels that compute a
    few fp32 operations per element and round once to bf16 (geglu, geglu_bwd, add, upsample2x_bwd, conv_out_bwd, the
    rank-r input-gradient updates).  bf16 keeps 8 significant bits, so rounding errs by at most 2^-8 of the value:
    2^-7 |ref| leaves a factor 2.
    `mag` is the same expression on absolute values and c covers the fp32 work before the rounding:
    - a chain of n dependent fp32 roundings errs by at most n 2^-24 mag: sums take c = 2 n 2^-24 (`chain_c`);
    - __expf errs by at most (2 + 1.16 |x|) ulp and erff by 2 ulp; the GELU arguments tested stay below |x| = 40
      (|x| = g^2 / 2 for g up to 9), so 50 ulp covers every transcendental of one element: geglu takes c = 2^-16.
      Phi(g) = (1 + erff(g / sqrt 2)) / 2 cancels for negative g, so its magnitude is (1 + |erf|) / 2: the absolute
      error of erff near -1 is what the bound then allows."""
    err = (out.double() - ref).abs()
    return _outside(err, 2.0 ** -7 * ref.abs() + c * mag, "pointwise")


def chain_c(n):
    """c of a bound whose fp32 part is a chain of n dependent roundings, with a factor 2 to spare."""
    return 2 * n * U


def reduction_violations(out, ref, mag, chain):
    """Bool mask of the elements of an fp32-output reduction (lora_proj T, lora_wgrad / lora_conv_wgrad G, colsum)
    outside |out - ref| <= 2 chain 2^-24 mag.  No bf16 rounding (a = 0); each of the `chain` dependent fp32 roundings
    errs by at most 2^-24 of a partial sum, and no partial sum exceeds mag = the reduction over absolute values (plus
    |G| before an accumulation).  `chain` comes from the kernel's chunking: see `proj_chain`, `wgrad_chain`,
    `colsum_chain`."""
    err = (out.double() - ref).abs()
    return _outside(err, chain_c(chain) * mag, "reduction")


def proj_chain(C, sources=1):
    """lora_proj_kernel: a lane owns every 32nd 8-channel vector (8 FMAs each), then a 5-step shuffle tree; a second
    source adds its row sums to the first (one more rounding)."""
    return 8 * cdiv(C // 8, 32) + 5 + (sources - 1)


def wgrad_chain(rows, C, taps=1):
    """lora_wgrad_kernel: a thread walks every 4th row of its chunk (one FMA each), 3 adds merge the 4 row lanes, the
    reduce kernel adds the chunks in order, then the scale multiply and an optional accumulation."""
    _, chunks, rpb = wgrad_launch(rows, C, taps)
    return cdiv(rpb, 4) + 3 + chunks + 2


def colsum_chain(HW):
    """colsum_kernel: 64 row lanes each add every 64th row, then lane 0 adds the other 63 lanes in order."""
    return cdiv(HW, 64) + 63


def norm_violations(out, ref, add, mag, stat, chain):
    """Bool mask of the LayerNorm / GroupNorm backward outputs outside
        |out - ref| <= 2^-7 (|ref| + |add|) + 2 (chain + 32) 2^-24 stat mag.
    out = rstd (dy g' - m1 - xhat m2) + add cancels, so the bound is relative to magnitudes, not to |ref|:
    - 2^-7 (|ref| + |add|): the bf16 rounding of the result (2^-8 |ref|, factor 2) and, when a cancelling `add` makes
      |ref| small, of the add's share;
    - mag = rstd (g'a + (1 + |xhat|) (mean g'a + mean g'a |xhat|)) + |add| with g'a = |dy gamma| (SiLU:
      |dy gamma| (|silu'(z)| + |gamma| (1 + |xhat|)), since |silu''| < 1 carries an error of z = gamma xhat + beta into
      dy silu'(z)).  It bounds each term of the output and the error an error d in xhat induces in m1, m2 and the
      output, all of which are sums of these magnitudes times |d|;
    - mean and rstd come from fp32 sums (LayerNorm: an in-warp two-pass mean / variance; GroupNorm: the forward's
      E[x^2] - mean^2 over its chunks).  A chain of n roundings makes the mean err by n 2^-24 (|mean| + 1/rstd) and the
      variance by n 2^-24 (mean^2 + var), so xhat errs by n 2^-24 stat (1 + |xhat|) and rstd relatively by
      n 2^-24 stat, with stat = 1 + (mean rstd)^2 per row / group;
    - chain = the longest fp32 chain of the statistics and of m1 / m2 (`ln_chain`, `gn_chain`); 32 more roundings
      cover the per-element expression, rsqrtf (2 ulp) and __expf in silu' (< 16 ulp for |z| < 12)."""
    err = (out.double() - ref).abs()
    return _outside(err, 2.0 ** -7 * (ref.abs() + add.abs()) + chain_c(chain + 32) * stat * mag, "norm")


def ln_chain(C):
    """layernorm_bwd_kernel: a lane sums 8 NV values, then a 5-step shuffle tree (sum, variance, m1, m2 alike)."""
    return 8 * ln_nv(C) + 5


def gn_chain(B, HW, C, groups, sms):
    """GroupNorm stats (forward and backward alike): a thread sums its rows of the chunk, the block adds rows_par x
    channels-per-group shared-memory partials, the finalize kernel's lanes add every 32nd chunk and a 5-step tree."""
    rows_par, chunks, rpb = gn_launch(B, HW, C, sms)
    return cdiv(rpb, rows_par) + rows_par * (C // groups) + cdiv(chunks, 32) + 5


def attn_violations(out, ref, mag):
    """Bool mask of attention-backward outputs outside |out - ref| <= 2^-7 (|ref| + mag).
    The kernel rounds P (for dV) and dS (for dQ, dK) to bf16 before the second MMA, so every term of the output sum
    carries a relative error of at most 2^-8; summed, at most 2^-8 mag with
        mag_dV = |P|^T |dO|,   mag_dQ = scale (|P| o (|dO| |V|^T + |D|)) |K|,   mag_dK = its transpose with |Q|.
    2^-7 mag leaves a factor 2 for that and room for the fp32 parts (exp2.approx, the forward's fp32 log-sum-exp, the
    fp32 S / dP products, the split partial sums), each far below 2^-8 relatively.  2^-7 |ref|: the bf16 output
    rounding (2^-8) with a factor 2.  The reference takes D from the kernel's own bf16 o, as attn_bwd_prep_kernel does."""
    err = (out.double() - ref).abs()
    return _outside(err, 2.0 ** -7 * (ref.abs() + mag), "attention")


def assert_no_violations(bad, out, ref, what):
    n = int(bad.sum())
    if n:
        where = [tuple(i) for i in bad.nonzero()[:6].tolist()]
        detail = "; ".join(f"{i}: got {out[i].item():.6g}, want {ref[i].item():.6g}" for i in where)
        raise AssertionError(f"{what}: {n} of {bad.numel()} elements outside the bound ({detail})")


# ------------------------------------------------------------------------------------------------------------------
# float64 references (device-agnostic: the CPU tests run them too)
# ------------------------------------------------------------------------------------------------------------------
def silu_grad(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


def _norm_bwd_ref(x, gamma, beta, dy, add, silu, dims, eps, mean=None, var=None):
    """x, dy: float64 [..., n] grouped so that `dims` are the reduced axes; gamma / beta broadcast."""
    if mean is None:
        mean = x.mean(dims, keepdim=True)
        var = ((x - mean) ** 2).mean(dims, keepdim=True)
    rstd = 1 / torch.sqrt(var + eps)
    xh = (x - mean) * rstd
    if silu:
        sg = silu_grad(gamma * xh + beta)
        dg = dy * sg * gamma
        ga = (dy * gamma).abs() * (sg.abs() + gamma.abs() * (1 + xh.abs()))
    else:
        dg = dy * gamma
        ga = (dy * gamma).abs()
    m1, m2 = dg.mean(dims, keepdim=True), (dg * xh).mean(dims, keepdim=True)
    ref = rstd * (dg - m1 - xh * m2)
    mag = rstd * (ga + (1 + xh.abs()) * (ga.mean(dims, keepdim=True) + (ga * xh.abs()).mean(dims, keepdim=True)))
    stat = 1 + (mean * rstd) ** 2
    if add is not None:
        ref, mag = ref + add, mag + add.abs()
    return ref, mag, stat.expand_as(ref)


def layernorm_bwd_ref(x, gamma, dy, add, eps=1e-5):
    """(ref, mag, stat) of dx = LayerNorm'(x)^T dy (+ add), [M, C] float64."""
    a = add.double() if add is not None else None
    return _norm_bwd_ref(x.double(), gamma.double(), 0.0, dy.double(), a, False, (1,), eps)


def groupnorm_bwd_ref(x, gamma, beta, dy, add, groups, silu, eps=1e-5):
    """x, dy, add: [B, HW, C]; returns [B, HW, C] float64 (ref, mag, stat)."""
    B, HW, C = x.shape
    cpg = C // groups
    sh = (B, HW, groups, cpg)
    gm, bt = gamma.double().view(groups, cpg), beta.double().view(groups, cpg)
    a = add.double().reshape(sh) if add is not None else None
    ref, mag, stat = _norm_bwd_ref(x.double().reshape(sh), gm, bt, dy.double().reshape(sh), a, silu, (1, 3), eps)
    return ref.reshape(B, HW, C), mag.reshape(B, HW, C), stat.reshape(B, HW, C)


def geglu_ref(pre):
    """(ref, mag) of a * gelu(g) for pre = [a | g]."""
    a, g = pre.double().chunk(2, dim=-1)
    erf = torch.erf(g / math.sqrt(2))
    return a * g * 0.5 * (1 + erf), (a * g).abs() * 0.5 * (1 + erf.abs())


def geglu_bwd_ref(pre, dout):
    """(ref, mag) of [dout gelu(g) | dout a gelu'(g)]."""
    a, g = pre.double().chunk(2, dim=-1)
    d = dout.double()
    erf = torch.erf(g / math.sqrt(2))
    cdf, cdf_mag = 0.5 * (1 + erf), 0.5 * (1 + erf.abs())
    pdf = torch.exp(-0.5 * g * g) / math.sqrt(2 * math.pi)
    ref = torch.cat([d * g * cdf, d * a * (cdf + g * pdf)], dim=-1)
    mag = torch.cat([(d * g).abs() * cdf_mag, (d * a).abs() * (cdf_mag + (g * pdf).abs())], dim=-1)
    return ref, mag


def attention_bwd_ref(q, k, v, o, dout, B, heads, Sq, Skv, d, scale):
    """float64 (dq, dk, dv) and their mags, [B * S, heads * d] each, one (batch, head) at a time."""
    outs = [torch.zeros(B * S, heads * d, dtype=torch.float64, device=q.device)
            for S in (Sq, Sq, Skv, Skv, Skv, Skv)]
    dq, mq, dk, mk, dv, mv = outs
    for b in range(B):
        rq, rk = slice(b * Sq, (b + 1) * Sq), slice(b * Skv, (b + 1) * Skv)
        for h in range(heads):
            c = slice(h * d, (h + 1) * d)
            qh, kh, vh = q[rq, c].double(), k[rk, c].double(), v[rk, c].double()
            oh, gh = o[rq, c].double(), dout[rq, c].double()
            P = torch.softmax(qh @ kh.t() * scale, dim=-1)
            D = (gh * oh).sum(1, keepdim=True)
            dS = P * (gh @ vh.t() - D)
            A = P * (gh.abs() @ vh.abs().t() + D.abs())
            dq[rq, c] = scale * dS @ kh
            mq[rq, c] = scale * A @ kh.abs()
            dk[rk, c] = scale * dS.t() @ qh
            mk[rk, c] = scale * A.t() @ qh.abs()
            dv[rk, c] = P.t() @ gh
            mv[rk, c] = P.t() @ gh.abs()
            del P, dS, A
    return dq, mq, dk, mk, dv, mv


# ------------------------------------------------------------------------------------------------------------------
# variant tables
# ------------------------------------------------------------------------------------------------------------------
# (M, C, add, NV, wraps): x, dy and add are column views of wider buffers (ld > C); dx goes into a guarded column view
LN_MATRIX = [
    (7, 256, False, 1, False),       # NV = 1 at its largest C
    (1, 264, True, 3, False),        # NV = 3 at its smallest C, one row
    (1000, 768, True, 3, False),     # NV = 3 at its largest C
    (300, 776, False, 5, False),     # NV = 5 at its smallest C
    (2048, 1280, True, 5, False),    # NV = 5 at its largest C (SDXL)
    (20000, 320, True, 3, True),     # SD1.x width; more rows than the grid: the row loop wraps
    (517, 1288, True, 8, False),     # NV = 8 at its smallest C
    (64, 2048, False, 8, False),     # NV = 8 at its largest C
    (20000, 2048, True, 8, True),    # NV = 8, wrapping
]

# (B, H, W, C0, C1, groups, silu, add, rows_par, one_chunk): x0 / x1 are column views of wider buffers, add a column
# view, dx guarded
GN_MATRIX = [
    (2, 32, 32, 320, 0, 32, True, False, 12, False),     # SD1.x level 1
    (2, 16, 16, 1280, 640, 32, True, True, 2, False),    # up-block resnet norm1: concat input + shortcut gradient
    (1, 8, 8, 320, 0, 32, True, True, 12, True),         # small image: a single chunk
    (2, 8, 8, 1280, 1280, 32, True, True, 1, False),     # SDXL 2560-channel concat
    (1, 64, 64, 640, 0, 32, False, True, 6, False),      # Transformer2DModel.norm
    (1, 16, 12, 4608, 0, 32, False, True, 1, False),     # C > 4096, rectangular image
    (1, 12, 12, 5120, 0, 32, True, False, 1, False),     # 640 threads per block: the largest the backward launches
    (1, 2, 4, 4608, 0, 32, True, True, 1, True),         # C > 4096 in a single chunk
]

# (M, F): pre = [a | g] and dout are column views; out / dpre guarded
GEGLU_MATRIX = [(1, 1280), (300, 2560), (4096, 1280), (77, 5120)]

# (M, C, r, sources, ld_pad, accumulate): A = column view with row stride C + ld_pad (for sources = 2: two column
# blocks of one buffer, like [x0 | x1]); G written transposed into the matching column slices of one [r, C] gradient
WGRAD_MATRIX = [
    (1, 1280, 4, 1, 0, False),         # time-embedding adaptor: M = batch, one chunk
    (7, 320, 8, 1, 64, True),          # M < 32, partial column block (40 vectors), accumulate
    (4096, 1280, 4, 2, 2560, False),   # two-source input (conv_shortcut: [x0 | x1]); A = dqkv[:, i C:(i+1) C]-like
    (1024, 640, 8, 1, 1280, True),     # lda = 3C (fused q|k|v gradient)
    (20000, 264, 4, 1, 8, False),      # many chunks, 33 vectors (partial block)
    (154, 2048, 8, 2, 0, True),        # cross-attention K/V shape, two sources
]

# (B, H, W, C0, C1, stride, r, accumulate): lora_conv_proj / lora_conv_wgrad / lora_conv_rank_update
CONV_MATRIX = [
    (2, 16, 24, 320, 0, 1, 4, False),
    (1, 16, 16, 256, 128, 1, 8, True),    # concat input, accumulate
    (2, 16, 12, 128, 0, 2, 4, True),      # stride 2, rectangular
    (1, 8, 8, 1280, 1280, 1, 4, False),   # SDXL up-block concat
    (1, 32, 32, 64, 0, 2, 8, False),
]

# (B, heads, Sq, Skv, d, cross): self-attention reads q / k / v from one fused [B S, 3 C] buffer and writes dq / dk /
# dv into the column slices of one guarded dqkv; cross-attention reads k / v from one [B Skv, 2 C] buffer
ATTN_MATRIX = [
    (1, 2, 200, 200, 8, False),
    (1, 5, 320, 200, 24, True),
    (2, 4, 256, 256, 40, False),
    (1, 10, 4096, 4096, 64, False),   # SDXL 64x64 level
    (1, 3, 130, 77, 72, True),
    (2, 2, 256, 256, 128, False),     # the largest head of ND = 2
    (1, 2, 192, 100, 136, True),      # ND = 3 (kT = 32), smallest head
    (2, 8, 256, 256, 160, False),     # SD1.x 16x16 level
    (1, 2, 96, 96, 192, False),       # ND = 3 at its largest head
]

# (B, heads, Sq, Skv, d, nsplit): attention_bwd_split (dK / dV with query splits when the shape qualifies)
SPLIT_MATRIX = [
    (2, 8, 1024, 77, 40, 8),     # SD1.x cross-attention at the 32x32 level
    (1, 10, 1000, 77, 64, 8),    # Sq not a multiple of q_split (128) or of 64
    (1, 4, 700, 40, 64, 11),     # Skv <= 64: the second consumer warpgroup has no valid rows
    (1, 2, 333, 128, 80, 6),     # the largest Skv that still splits; ragged Sq
    (11, 6, 256, 77, 64, 2),     # B heads = 66: still splits
    (67, 1, 256, 77, 64, 1),     # B heads = 67: unsplit, ws untouched
    (1, 8, 300, 129, 64, 1),     # Skv = 129: unsplit
    (2, 4, 4096, 77, 160, 16),   # ND = 3 split
]


# ------------------------------------------------------------------------------------------------------------------
# GPU machinery
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def col_view(M, C, pad, dev, gen, scale=1.0, offset=0.0):
    """A [M, C] bf16 column view (row stride C + pad, starting `pad // 2` rounded to 8 columns in) of a wider buffer."""
    lo = (pad // 2) // 8 * 8
    buf = (torch.randn(M, C + pad, generator=gen) * scale + offset).to(dev, BF)
    return buf[:, lo:lo + C]


def flat_guarded(n, dtype, dev):
    """(buffer, view): n contiguous elements with FLAT_GUARD guard elements before and after, all NaN bits."""
    if dtype == BF:
        buf = torch.full((n + 2 * FLAT_GUARD,), NAN_BITS, dtype=torch.int16, device=dev).view(BF)
    else:
        buf = torch.full((n + 2 * FLAT_GUARD,), F32_NAN_BITS, dtype=torch.int32, device=dev).view(torch.float32)
    return buf, buf[FLAT_GUARD:FLAT_GUARD + n]


def assert_flat_guard(buf, n):
    bits = buf.view(torch.int16 if buf.dtype == BF else torch.int32)
    pat = NAN_BITS if buf.dtype == BF else F32_NAN_BITS
    g = torch.cat([bits[:FLAT_GUARD], bits[FLAT_GUARD + n:]])
    assert int((g != pat).sum()) == 0, f"{int((g != pat).sum())} elements written outside the {n}-element output"
    assert not torch.isnan(buf[FLAT_GUARD:FLAT_GUARD + n]).any(), "NaN in the output (unwritten?)"


def guarded_f32(rows, cols, dev):
    buf = torch.full((rows + 2 * GUARD_ROWS, cols + GUARD_COLS), F32_NAN_BITS, dtype=torch.int32,
                     device=dev).view(torch.float32)
    return buf, buf[GUARD_ROWS:GUARD_ROWS + rows, :cols]


def assert_guard_f32(buf, rows, cols, allow_nan=False):
    bits = buf.view(torch.int32)
    guard = torch.ones_like(bits, dtype=torch.bool)
    guard[GUARD_ROWS:GUARD_ROWS + rows, :cols] = False
    n = int((bits[guard] != F32_NAN_BITS).sum())
    assert n == 0, f"{n} elements written outside the [{rows}, {cols}] output"
    if not allow_nan:
        assert not torch.isnan(buf[GUARD_ROWS:GUARD_ROWS + rows, :cols]).any(), "NaN in the output (unwritten?)"


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == BF else torch.int32)


def assert_bitwise(a, b, what):
    assert torch.equal(bits(a), bits(b)), f"{what}: two identical calls differ"


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm / GroupNorm backward
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,C,with_add,nv,wraps", LN_MATRIX)
def test_layernorm_bwd_bound(dev, sms, M, C, with_add, nv, wraps):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(M + C)
    x = col_view(M, C, 64, dev, g, 2.0, 0.5)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dev, BF)
    dy = col_view(M, C, 128, dev, g)
    add = col_view(M, C, 2 * C, dev, g) if with_add else None
    assert ln_nv(C) == nv and ln_wraps(M, sms) == wraps and x.stride(0) > C
    outs = []
    for _ in range(2):
        buf, dx = guarded_out(M, C, dev)
        assert ops.layernorm_bwd(x, gamma, dy, 1e-5, add=add, out=dx) is dx
        torch.cuda.synchronize()
        assert_guard_intact(buf, M, C)
        outs.append(dx)
    assert_bitwise(outs[0], outs[1], "layernorm_bwd")
    ref, mag, stat = layernorm_bwd_ref(x, gamma, dy, add)
    a = add.double() if add is not None else torch.zeros_like(ref)
    assert_no_violations(norm_violations(outs[0], ref, a, mag, stat, ln_chain(C)), outs[0], ref, "layernorm_bwd")


@pytest.mark.parametrize("B,H,W,C0,C1,groups,silu,with_add,rows_par,one_chunk", GN_MATRIX)
def test_groupnorm_bwd_bound(dev, sms, B, H, W, C0, C1, groups, silu, with_add, rows_par, one_chunk):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(H + W + C0 + C1)
    C, HW = C0 + C1, H * W
    rp, chunks, _ = gn_launch(B, HW, C, sms)
    assert gn_smem_ok(C) and rp == rows_par and (chunks == 1) == one_chunk
    x0 = col_view(B * HW, C0, 16, dev, g, 1.5, 0.3).view(B, H, W, C0)
    x1 = col_view(B * HW, C1, 24, dev, g, 1.5, -0.2).view(B, H, W, C1) if C1 else None
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dev, BF)
    beta = (0.2 * torch.randn(C, generator=g)).to(dev, BF)
    dy = col_view(B * HW, C, 8, dev, g).view(B, H, W, C)
    add = col_view(B * HW, C, 64, dev, g).view(B, H, W, C) if with_add else None
    ws = ops.gn_ws(B, groups, dev)
    ops.groupnorm(x0, gamma, beta, groups, 1e-5, silu, x1=x1, stats_ws=ws)
    outs = []
    for _ in range(2):
        buf, dx = guarded_out(B * HW, C, dev)
        dx4 = dx.view(B, H, W, C)
        assert ops.groupnorm_bwd(x0, gamma, beta, groups, silu, dy, ws, x1=x1, add=add, out=dx4) is dx4
        torch.cuda.synchronize()
        assert_guard_intact(buf, B * HW, C)
        outs.append(dx)
    assert_bitwise(outs[0], outs[1], "groupnorm_bwd")
    x = torch.cat([x0, x1], -1) if x1 is not None else x0
    ref, mag, stat = groupnorm_bwd_ref(x.reshape(B, HW, C), gamma, beta, dy.reshape(B, HW, C),
                                       add.reshape(B, HW, C) if add is not None else None, groups, silu)
    a = add.double().reshape(B, HW, C) if add is not None else torch.zeros_like(ref)
    out = outs[0].view(B, HW, C)
    assert_no_violations(norm_violations(out, ref, a, mag, stat, gn_chain(B, HW, C, groups, sms)), out, ref,
                         "groupnorm_bwd")


# ------------------------------------------------------------------------------------------------------------------
# GEGLU and the pointwise helpers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,Fh", GEGLU_MATRIX)
def test_geglu_fwd_bwd_bound(dev, M, Fh):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(M + Fh)
    pre = col_view(M, 2 * Fh, 64, dev, g, 2.5)
    dout = col_view(M, Fh, 32, dev, g)
    fw, bw = [], []
    for _ in range(2):
        buf, o = guarded_out(M, Fh, dev)
        assert ops.geglu(pre, out=o) is o
        bbuf, dp = guarded_out(M, 2 * Fh, dev)
        assert ops.geglu_bwd(pre, dout, out=dp) is dp
        torch.cuda.synchronize()
        assert_guard_intact(buf, M, Fh)
        assert_guard_intact(bbuf, M, 2 * Fh)
        fw.append(o)
        bw.append(dp)
    assert_bitwise(fw[0], fw[1], "geglu")
    assert_bitwise(bw[0], bw[1], "geglu_bwd")
    ref, mag = geglu_ref(pre)
    assert_no_violations(pointwise_violations(fw[0], ref, mag, 2.0 ** -16), fw[0], ref, "geglu")
    ref, mag = geglu_bwd_ref(pre, dout)
    assert_no_violations(pointwise_violations(bw[0], ref, mag, 2.0 ** -16), bw[0], ref, "geglu_bwd")


def _lib_call(name, *args):
    from sliders_b200 import _cabi, ops

    _cabi.check(getattr(_cabi.load(), name)(ops._ctx(torch.empty(1, device="cuda")), ops._stream(), *args))


def test_pointwise_helpers_bound(dev):
    """add (three column views into a column view), upsample2x_bwd, zero_stuff (bit-exact), conv_out_bwd with fp32 and
    bf16 d_eps; contiguous outputs are written between flat guard bands."""
    from sliders_b200 import ops

    P = ops._p
    g = torch.Generator().manual_seed(4)
    a = torch.randn(300, 1920, generator=g).to(dev, BF)
    b = col_view(300, 640, 64, dev, g)
    c = col_view(300, 640, 8, dev, g, 1e-3)
    ref = a[:, 640:1280].double() + b.double() + c.double()
    mag = a[:, 640:1280].double().abs() + b.double().abs() + c.double().abs()
    outs = []
    for _ in range(2):
        buf, o = guarded_out(300, 640, dev)
        ops.add(a[:, 640:1280], b, c, out=o)
        torch.cuda.synchronize()
        assert_guard_intact(buf, 300, 640)
        outs.append(o)
    assert_bitwise(outs[0], outs[1], "add")
    assert_no_violations(pointwise_violations(outs[0], ref, mag, chain_c(2)), outs[0], ref, "add")

    for (B, H2, W2, Cc) in ((2, 16, 24, 64), (1, 2, 2, 1280), (3, 32, 32, 320)):
        dy = torch.randn(B, H2, W2, Cc, generator=g).to(dev, BF)
        n = dy.numel() // 4
        ref = dy.double().view(B, H2 // 2, 2, W2 // 2, 2, Cc).sum(dim=(2, 4))
        mag = dy.double().abs().view(B, H2 // 2, 2, W2 // 2, 2, Cc).sum(dim=(2, 4))
        outs = []
        for _ in range(2):
            buf, o = flat_guarded(n, BF, dev)
            _lib_call("sb200_upsample2x_bwd", P(dy), P(o), B, H2 // 2, W2 // 2, Cc)
            torch.cuda.synchronize()
            assert_flat_guard(buf, n)
            outs.append(o.view(ref.shape))
        assert_bitwise(outs[0], outs[1], "upsample2x_bwd")
        assert_no_violations(pointwise_violations(outs[0], ref, mag, chain_c(3)), outs[0], ref, "upsample2x_bwd")
        n = dy.numel() * 4
        buf, z = flat_guarded(n, BF, dev)
        _lib_call("sb200_zero_stuff", P(dy), P(z), B, H2, W2, Cc)
        torch.cuda.synchronize()
        assert_flat_guard(buf, n)
        zr = torch.zeros(B, 2 * H2, 2 * W2, Cc, device=dev, dtype=BF)
        zr[:, ::2, ::2] = dy
        assert torch.equal(bits(z.view(zr.shape)), bits(zr)), "zero_stuff is not bit-exact"

    for (B, H, W, Cc) in ((2, 24, 16, 320), (1, 1, 7, 64), (1, 9, 5, 1280)):
        w = (torch.randn(4, Cc, 3, 3, generator=g) / (9 * Cc) ** 0.5).to(dev, BF)
        wp = w.permute(0, 2, 3, 1).contiguous()
        for dt in (torch.float32, BF):
            deps = torch.randn(B, 4, H, W, generator=g).to(dev, dt)
            ref = torch.nn.grad.conv2d_input((B, Cc, H, W), w.double(), deps.double(), padding=1).permute(0, 2, 3, 1)
            mag = torch.nn.grad.conv2d_input((B, Cc, H, W), w.double().abs(), deps.double().abs(),
                                             padding=1).permute(0, 2, 3, 1)
            n = B * H * W * Cc
            outs = []
            for _ in range(2):
                buf, o = flat_guarded(n, BF, dev)
                _lib_call("sb200_conv_out_bwd", P(deps), int(dt == torch.float32), P(wp), P(o), B, H, W, Cc)
                torch.cuda.synchronize()
                assert_flat_guard(buf, n)
                outs.append(o.view(B, H, W, Cc))
            assert_bitwise(outs[0], outs[1], "conv_out_bwd")
            # 36 taps x channels: one FMA chain of at most 36 roundings
            assert_no_violations(pointwise_violations(outs[0], ref, mag, chain_c(36)), outs[0], ref, "conv_out_bwd")


@pytest.mark.parametrize("B,HW,Cc,pad", [(2, 1024, 1280, 0), (3, 1600, 320, 64), (1, 17, 2560, 8), (8, 64, 264, 0)])
def test_colsum_bound(dev, B, HW, Cc, pad):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(HW + Cc)
    dy = col_view(B * HW, Cc, pad, dev, g)
    ref = dy.double().view(B, HW, Cc).sum(1)
    mag = dy.double().abs().view(B, HW, Cc).sum(1)
    outs = []
    for _ in range(2):  # the kernel writes [B, C] contiguous: guarded flat
        fbuf, fo = flat_guarded(B * Cc, torch.float32, dev)
        _lib_call("sb200_colsum", ops._p(dy), dy.stride(0), ops._p(fo), B, HW, Cc)
        torch.cuda.synchronize()
        assert_flat_guard(fbuf, B * Cc)
        outs.append(fo.view(B, Cc))
    assert_bitwise(outs[0], outs[1], "colsum")
    assert_no_violations(reduction_violations(outs[0], ref, mag, colsum_chain(HW)), outs[0], ref, "colsum")


# ------------------------------------------------------------------------------------------------------------------
# LoRA rank-r reductions and updates
# ------------------------------------------------------------------------------------------------------------------
def split_cols(C, sources):
    """Column widths of the [x0 | x1] sources of a WGRAD_MATRIX row."""
    return [C] if sources == 1 else [C // 16 * 8, C - C // 16 * 8]


@pytest.mark.parametrize("M,C,r,sources,pad,acc", WGRAD_MATRIX)
def test_lora_linear_bound(dev, M, C, r, sources, pad, acc):
    """lora_proj (two-source accumulation through out=), lora_wgrad (G transposed into column slices of one guarded
    gradient, untransposed into a strided guarded G, accumulate), lora_rank_update (into a column view of dX)."""
    from sliders_b200 import ops

    P = ops._p
    g = torch.Generator().manual_seed(M + C + r)
    widths = split_cols(C, sources)
    xbuf = torch.randn(M, C + pad, generator=g).to(dev, BF)
    xs, k0 = [], 0
    for wdt in widths:
        xs.append(xbuf[:, k0:k0 + wdt])
        k0 += wdt
    assert all(x.stride(0) == C + pad for x in xs)
    down = (torch.randn(r, C + 16, generator=g) / C ** 0.5).to(dev, BF)[:, :C]   # ldb > C
    T0 = torch.randn(M, r, generator=g).to(dev)
    G0 = torch.randn(r, C, generator=g).to(dev)
    dX0 = torch.randn(M, C + 24, generator=g).to(dev, BF)
    s = -0.75

    # lora_proj: T = [x0 | x1] @ down^T, the second source accumulating through out=
    Ts = []
    for _ in range(2):
        fbuf, T = flat_guarded(M * r, torch.float32, dev)
        T = T.view(M, r)
        k0 = 0
        for i, x in enumerate(xs):
            _lib_call("sb200_lora_proj", P(x), x.stride(0), P(down[:, k0:]), down.stride(0), P(T), M, x.shape[1], r,
                      int(i > 0))
            k0 += x.shape[1]
        torch.cuda.synchronize()
        assert_flat_guard(fbuf, M * r)
        Ts.append(T)
    assert_bitwise(Ts[0], Ts[1], "lora_proj")
    xd = torch.cat([x.double() for x in xs], 1)
    ref, mag = xd @ down.double().t(), xd.abs() @ down.double().abs().t()
    assert_no_violations(reduction_violations(Ts[0], ref, mag, proj_chain(max(widths), sources)), Ts[0], ref,
                         "lora_proj")

    # lora_wgrad, transposed: G[r, C] column slices (autograd.py's g_down[:, k0:k0 + K])
    Gs = []
    for _ in range(2):
        gbuf, G = guarded_f32(r, C, dev)
        if acc:
            G.copy_(G0)
        k0 = 0
        for i, x in enumerate(xs):
            ops.lora_wgrad(x, T0, G[:, k0:k0 + x.shape[1]], True, s, accumulate=acc)
            torch.cuda.synchronize()
            if i == 0 and len(xs) > 1 and not acc:  # the first source leaves the second source's columns alone
                assert torch.equal(bits(G[:, x.shape[1]:]), torch.full_like(bits(G[:, x.shape[1]:]), F32_NAN_BITS))
            k0 += x.shape[1]
        assert_guard_f32(gbuf, r, C)
        Gs.append(G.clone())
    assert_bitwise(Gs[0], Gs[1], "lora_wgrad (transposed)")
    ref = s * (T0.double().t() @ xd)
    mag = abs(s) * (T0.double().abs().t() @ xd.abs())
    if acc:
        ref, mag = ref + G0.double(), mag + G0.double().abs()
    chain = max(wgrad_chain(M, wdt) for wdt in widths)
    assert_no_violations(reduction_violations(Gs[0], ref, mag, chain), Gs[0], ref, "lora_wgrad (transposed)")

    # lora_wgrad, untransposed: G [C, r] with a padded row stride (g_up)
    x = xs[0]
    Gs = []
    for _ in range(2):
        gbuf, G = guarded_f32(x.shape[1], r, dev)
        if acc:
            G.copy_(G0[:, :x.shape[1]].t())
        ops.lora_wgrad(x, T0, G, False, s, accumulate=acc)
        torch.cuda.synchronize()
        assert_guard_f32(gbuf, x.shape[1], r)
        Gs.append(G.clone())
    assert_bitwise(Gs[0], Gs[1], "lora_wgrad")
    ref = s * (x.double().t() @ T0.double())
    mag = abs(s) * (x.double().abs().t() @ T0.double().abs())
    if acc:
        ref, mag = ref + G0[:, :x.shape[1]].t().double(), mag + G0[:, :x.shape[1]].t().double().abs()
    assert_no_violations(reduction_violations(Gs[0], ref, mag, wgrad_chain(M, x.shape[1])), Gs[0], ref, "lora_wgrad")

    # lora_rank_update: dX (a column view, ldx > C) += s T0 @ down, from a known dX
    outs = []
    for _ in range(2):
        buf, dX = guarded_out(M, C, dev)
        dX.copy_(dX0[:, 8:8 + C])
        ops.lora_rank_update(dX, T0, down, s)
        torch.cuda.synchronize()
        assert_guard_intact(buf, M, C)
        outs.append(dX)
    assert_bitwise(outs[0], outs[1], "lora_rank_update")
    ref = dX0[:, 8:8 + C].double() + s * (T0.double() @ down.double())
    mag = dX0[:, 8:8 + C].double().abs() + abs(s) * (T0.double().abs() @ down.double().abs())
    assert_no_violations(pointwise_violations(outs[0], ref, mag, chain_c(r + 2)), outs[0], ref, "lora_rank_update")
    # the variant this row claims
    assert (wgrad_launch(M, widths[0])[1] == 1) == (M < 32)


@pytest.mark.parametrize("B,H,W,C0,C1,stride,r,acc", CONV_MATRIX)
def test_lora_conv_bound(dev, B, H, W, C0, C1, stride, r, acc):
    from sliders_b200 import ops

    P = ops._p
    g = torch.Generator().manual_seed(H + W + C0 + C1 + stride + r)
    Cin = C0 + C1
    Ho, Wo = H // stride, W // stride
    npix = B * Ho * Wo
    x0 = col_view(B * H * W, C0, 16, dev, g).view(B, H, W, C0)
    x1 = col_view(B * H * W, C1, 8, dev, g).view(B, H, W, C1) if C1 else None
    x = torch.cat([x0, x1], -1) if x1 is not None else x0
    D = (torch.randn(r, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5).to(dev, BF)
    U0 = torch.randn(npix, r, generator=g).to(dev)
    G0 = torch.randn(r, 3, 3, Cin, generator=g).to(dev)
    dX0 = torch.randn(B, H, W, Cin, generator=g).to(dev, BF)
    s = 1.25
    xd = x.double().permute(0, 3, 1, 2)
    Dd = D.double().permute(0, 3, 1, 2)

    Ts = []
    for _ in range(2):
        fbuf, T = flat_guarded(npix * r, torch.float32, dev)
        _lib_call("sb200_lora_conv_proj", P(x0), x0.stride(2), C0, P(x1), x1.stride(2) if x1 is not None else 0, C1,
                  P(D), P(T), B, H, W, stride, r)
        torch.cuda.synchronize()
        assert_flat_guard(fbuf, npix * r)
        Ts.append(T.view(npix, r))
    assert_bitwise(Ts[0], Ts[1], "lora_conv_proj")
    conv = torch.nn.functional.conv2d
    ref = conv(xd, Dd, stride=stride, padding=1).permute(0, 2, 3, 1).reshape(npix, r)
    mag = conv(xd.abs(), Dd.abs(), stride=stride, padding=1).permute(0, 2, 3, 1).reshape(npix, r)
    # a lane: 9 taps x its vectors x 8 FMAs, then the shuffle tree
    assert_no_violations(reduction_violations(Ts[0], ref, mag, 9 * proj_chain(Cin)), Ts[0], ref, "lora_conv_proj")

    Gs = []
    for _ in range(2):
        fbuf, G = flat_guarded(G0.numel(), torch.float32, dev)
        G = G.view(G0.shape)
        if acc:
            G.copy_(G0)
        ops.lora_conv_wgrad(x0, U0, G, s, stride, x1=x1, accumulate=acc)
        torch.cuda.synchronize()
        assert_flat_guard(fbuf, G0.numel())
        Gs.append(G)
    assert_bitwise(Gs[0], Gs[1], "lora_conv_wgrad")
    Ud = U0.double().view(B, Ho, Wo, r).permute(0, 3, 1, 2)
    wg = torch.nn.grad.conv2d_weight
    ref = s * wg(xd, (r, Cin, 3, 3), Ud, stride=stride, padding=1).permute(0, 2, 3, 1)
    mag = abs(s) * wg(xd.abs(), (r, Cin, 3, 3), Ud.abs(), stride=stride, padding=1).permute(0, 2, 3, 1)
    if acc:
        ref, mag = ref + G0.double(), mag + G0.double().abs()
    assert_no_violations(reduction_violations(Gs[0], ref, mag, wgrad_chain(npix, Cin, 9)), Gs[0], ref,
                         "lora_conv_wgrad")

    outs = []
    n = dX0.numel()
    for _ in range(2):
        fbuf, dX = flat_guarded(n, BF, dev)
        dX = dX.view(dX0.shape)
        dX.copy_(dX0)
        ops.lora_conv_rank_update(dX, U0, D, s, stride)
        torch.cuda.synchronize()
        assert_flat_guard(fbuf, n)
        outs.append(dX)
    assert_bitwise(outs[0], outs[1], "lora_conv_rank_update")
    gi = torch.nn.grad.conv2d_input
    ref = dX0.double() + s * gi((B, Cin, H, W), Dd, Ud, stride=stride, padding=1).permute(0, 2, 3, 1)
    mag = dX0.double().abs() + abs(s) * gi((B, Cin, H, W), Dd.abs(), Ud.abs(), stride=stride,
                                           padding=1).permute(0, 2, 3, 1)
    assert_no_violations(pointwise_violations(outs[0], ref, mag, chain_c(9 * r + 2)), outs[0], ref,
                         "lora_conv_rank_update")


# ------------------------------------------------------------------------------------------------------------------
# attention backward
# ------------------------------------------------------------------------------------------------------------------
def _attn_inputs(dev, B, heads, Sq, Skv, d, cross, seed):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(seed)
    Cc = heads * d
    if cross:
        q = torch.randn(B * Sq, Cc + 64, generator=g).to(dev, BF)[:, 32:32 + Cc]
        kv = torch.randn(B * Skv, 2 * Cc, generator=g).to(dev, BF)
        k, v = kv[:, :Cc], kv[:, Cc:]
    else:
        qkv = torch.randn(B * Sq, 3 * Cc, generator=g).to(dev, BF)
        q, k, v = qkv[:, :Cc], qkv[:, Cc:2 * Cc], qkv[:, 2 * Cc:]
    dout = torch.randn(B * Sq, Cc, generator=g).to(dev, BF)
    scale = d ** -0.5
    lse = torch.empty(B, heads, Sq, device=dev, dtype=torch.float32)
    o = ops.attention(q, k, v, B, heads, Sq, Skv, scale, head_dim=d, lse=lse)
    return q, k, v, o, dout, lse, scale


def _check_attn(outs, refs, names):
    for got, (ref, mag), name in zip(outs, refs, names):
        assert_no_violations(attn_violations(got, ref, mag), got, ref, name)


@pytest.mark.parametrize("B,heads,Sq,Skv,d,cross", ATTN_MATRIX)
def test_attention_bwd_bound(dev, B, heads, Sq, Skv, d, cross):
    from sliders_b200 import ops

    assert attn_nd(d) in (1, 2, 3) and attn_kt(d) == (32 if d > 128 else 64)
    q, k, v, o, dout, lse, scale = _attn_inputs(dev, B, heads, Sq, Skv, d, cross, Sq + Skv + d)
    Cc = heads * d
    runs = []
    for _ in range(2):
        if cross:
            qbuf, dq = guarded_out(B * Sq, Cc, dev)
            kvbuf, dkv = guarded_out(B * Skv, 2 * Cc, dev)
            ops.attention_bwd(q, k, v, o, dout, lse, B, heads, Sq, Skv, scale, d, dq, dkv[:, :Cc], dkv[:, Cc:])
            torch.cuda.synchronize()
            assert_guard_intact(qbuf, B * Sq, Cc)
            assert_guard_intact(kvbuf, B * Skv, 2 * Cc)
            runs.append((dq, dkv[:, :Cc], dkv[:, Cc:]))
        else:
            buf, dqkv = guarded_out(B * Sq, 3 * Cc, dev)
            ops.attention_bwd(q, k, v, o, dout, lse, B, heads, Sq, Skv, scale, d, dqkv[:, :Cc], dqkv[:, Cc:2 * Cc],
                              dqkv[:, 2 * Cc:])
            torch.cuda.synchronize()
            assert_guard_intact(buf, B * Sq, 3 * Cc)
            runs.append((dqkv[:, :Cc], dqkv[:, Cc:2 * Cc], dqkv[:, 2 * Cc:]))
    for a, b, name in zip(runs[0], runs[1], ("dq", "dk", "dv")):
        assert_bitwise(a, b, f"attention_bwd {name}")
    dq, mq, dk, mk, dv, mv = attention_bwd_ref(q, k, v, o, dout, B, heads, Sq, Skv, d, scale)
    _check_attn(runs[0], ((dq, mq), (dk, mk), (dv, mv)), ("dq", "dk", "dv"))


def _attn_bwd_ws(q, k, v, o, dout, lse, B, heads, Sq, Skv, scale, d, dq, dk, dv, ws, ws_n):
    from sliders_b200 import ops

    P = ops._p
    dsum = torch.empty(B * heads * Sq, device=q.device, dtype=torch.float32)
    _lib_call("sb200_attention_bwd_ws", P(q), q.stride(0), P(k), k.stride(0), P(v), v.stride(0), P(o), o.stride(0),
              P(dout), dout.stride(0), P(lse), P(dsum), P(dq), dq.stride(0), P(dk), dk.stride(0), P(dv), dv.stride(0),
              B, heads, Sq, Skv, int(d), float(scale), P(ws), ws_n)


@pytest.mark.parametrize("B,heads,Sq,Skv,d,nsplit", SPLIT_MATRIX)
def test_attention_bwd_split_bound(dev, B, heads, Sq, Skv, d, nsplit):
    from sliders_b200 import ops

    assert attn_split(B, heads, Sq, Skv)[0] == nsplit and nsplit <= ops.attn_bwd_splits(B, heads, Sq, Skv)
    q, k, v, o, dout, lse, scale = _attn_inputs(dev, B, heads, Sq, Skv, d, True, Sq + Skv + d + B)
    Cc = heads * d
    ws_n = 2 * nsplit * B * Skv * Cc if nsplit > 1 else 4096
    runs = []
    for _ in range(2):
        qbuf, dq = guarded_out(B * Sq, Cc, dev)
        kvbuf, dkv = guarded_out(B * Skv, 2 * Cc, dev)
        wbuf, ws = flat_guarded(ws_n, torch.float32, dev)
        _attn_bwd_ws(q, k, v, o, dout, lse, B, heads, Sq, Skv, scale, d, dq, dkv[:, :Cc], dkv[:, Cc:], ws,
                     ws_n if nsplit > 1 else 0)
        torch.cuda.synchronize()
        assert_guard_intact(qbuf, B * Sq, Cc)
        assert_guard_intact(kvbuf, B * Skv, 2 * Cc)
        wbits = wbuf.view(torch.int32)
        if nsplit > 1:
            assert int((torch.cat([wbits[:FLAT_GUARD], wbits[FLAT_GUARD + ws_n:]]) != F32_NAN_BITS).sum()) == 0
            assert not torch.isnan(ws).any(), "split partials not all written"
        else:
            assert int((wbits != F32_NAN_BITS).sum()) == 0, "an unsplit shape wrote to the scratch"
        runs.append((dq, dkv[:, :Cc], dkv[:, Cc:]))
    for a, b, name in zip(runs[0], runs[1], ("dq", "dk", "dv")):
        assert_bitwise(a, b, f"attention_bwd_split {name}")
    dq_plain = torch.empty(B * Sq, Cc, device=dev, dtype=BF)
    ops.attention_bwd(q, k, v, o, dout, lse, B, heads, Sq, Skv, scale, d, dq_plain)
    torch.cuda.synchronize()
    assert torch.equal(bits(dq_plain), bits(runs[0][0])), "dq differs from attention_bwd's"
    dq, mq, dk, mk, dv, mv = attention_bwd_ref(q, k, v, o, dout, B, heads, Sq, Skv, d, scale)
    _check_attn(runs[0], ((dq, mq), (dk, mk), (dv, mv)), ("dq", "dk", "dv"))
