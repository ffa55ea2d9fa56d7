"""Element-by-element tests of the forward kernels outside the GEMM (csrc/attention.cu, csrc/norm.cu,
csrc/elementwise.cu) against float64 references computed from the same bf16 / fp32 inputs.

Every row of the variant tables below, in the manner of test_gpu_backward_bounds.py,
- writes its outputs twice, each time into a fresh guarded buffer (bf16: NAN_BITS, fp32: F32_NAN_BITS), and checks
  that no guard element changed, that no output element is NaN and that the two calls agree bit for bit;
- where the C ABI takes an output row stride (attention, layernorm, groupnorm, small_linear, sinusoid), writes into a
  guarded column view of a wider buffer, and calls the `ops` wrapper once more, whose result must be bitwise equal
  (so the wrapper's argument mapping is covered too);
- checks each output element against the bound of its kernel family (the `*_bound` / `*_violations` functions, whose
  docstrings derive the constants);
- asserts the launch variant it is listed for with the host code's own formulas (`attn_nd`, `attn_fwd_kv`, `ln_nv`,
  `ln_wraps`, `gn_launch`, the grid caps of elementwise.cu), so a label cannot drift from what runs.
tests/test_forward_bounds.py checks, without a GPU, that the bounds accept a CPU emulation of each kernel's roundings,
reject planted local errors that rel-RMS accepts, and that the tables cover every variant."""
import math

import pytest
import torch

from test_gpu_backward_bounds import (BF, F32_NAN_BITS, MAX_RATIO, U, _lib_call, _outside, assert_bitwise,  # noqa: F401
                                      assert_flat_guard, assert_no_violations, attn_nd, attn_violations, bits, cdiv,
                                      chain_c, col_view, dev, flat_guarded, gn_chain, gn_launch, gn_smem_ok, ln_chain,
                                      ln_nv, ln_wraps, norm_violations, pointwise_violations, reduction_violations,
                                      sms)
from test_gpu_kernels import assert_guard_intact, guarded_out, make_lora

pytestmark = pytest.mark.gpu

LOG2E = 1.0 / math.log(2.0)


# ------------------------------------------------------------------------------------------------------------------
# the host code's launch formulas (attention.cu / elementwise.cu)
# ------------------------------------------------------------------------------------------------------------------
def attn_fwd_kv(d):
    """AttnCfg<ND>::kKV: keys per K / V tile of attention_kernel (the O accumulator of wider heads takes the
    registers of the second half)."""
    return 128 if d <= 64 else 64


def attn_ksteps(d):
    """16-wide k-steps of the Q K^T contraction that hold data; for d = 8 (mod 16) the last one is half zero fill."""
    return cdiv(d, 16)


def conv_in_wraps(B, H, W, Cout, sms):
    """conv_in: one thread per (pixel, 8 output channels), at most 8 blocks of 256 threads per SM."""
    return B * H * W * (Cout // 8) > 2048 * sms


def conv_out_wraps(B, H, W, sms):
    """conv_out: one warp per output pixel, at most 8 blocks of 8 warps per SM."""
    return B * H * W > 64 * sms


def upsample_wraps(B, H, W, C, sms):
    """upsample2x: one thread per 8-channel output vector, at most 16 blocks of 256 threads per SM."""
    return B * 4 * H * W * (C // 8) > 4096 * sms


def cfg_wraps(n, sms):
    """cfg_ddim_kernel: one thread per element, at most 8 blocks of 256 threads per SM."""
    return n > 2048 * sms


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------
def attn_lse_chain(Skv, d):
    """Dependent fp32 roundings of the row sum l: a thread adds kKV / 4 probabilities of its row per key tile and
    multiplies by the rescale factor once per tile, then 2 quad shuffles."""
    kv = attn_fwd_kv(d)
    return cdiv(Skv, kv) * (kv // 4 + 1) + 2


def attention_fwd_ref(q, k, v, B, heads, Sq, Skv, d, scale):
    """float64 (o, mag, lse, lse_bound), o / mag [B Sq, heads d], lse / lse_bound [B, heads, Sq].
    mag = |P| |V| (the `attn_violations` form).  lse = logsumexp(scale S) log2(e), the log2-domain value the kernel
    stores; its absolute bound, per row, with x = scale log2(e) S and X = max |x|:
    - x: the fp32 S carries at most d roundings of partial sums of |q| |k| (one per product, conservatively), and
      scale log2(e) and the product x round once each: E_x = 2^-24 (d |scale log2 e| max(|q| |k|) + 2 X).  The
      log-sum-exp moves by at most max |dx|.
    - l = sum 2^(x - m): every exponent rounds once (relative 2^-24 |x - m| <= 2^-23 X in x, ln 2 times that in p),
      ex2.approx errs by at most 2^-22 relatively (2^-21 taken), and so does every per-tile rescale factor alpha; the
      sum of positive terms is a chain of `attn_lse_chain` roundings.  rel(l) <= 2^-24 chain + (tiles + 1)
      (2^-21 + ln 2 2^-23 X), and log2 moves by rel(l) / ln 2;
    - __log2f errs by at most 2^-22 absolutely on [0.5, 2] and 2 ulp elsewhere (l <= Skv): 2^-22 (1 + log2 Skv);
    - m + log2(l) rounds once: 2^-24 |lse|.
    The bound is twice the sum."""
    dev = q.device
    o = torch.zeros(B * Sq, heads * d, dtype=torch.float64, device=dev)
    mag = torch.zeros_like(o)
    lse = torch.zeros(B, heads, Sq, dtype=torch.float64, device=dev)
    lb = torch.zeros_like(lse)
    sl2 = abs(scale) * LOG2E
    tiles = cdiv(Skv, attn_fwd_kv(d))
    for b in range(B):
        rq, rk = slice(b * Sq, (b + 1) * Sq), slice(b * Skv, (b + 1) * Skv)
        for h in range(heads):
            c = slice(h * d, (h + 1) * d)
            qh, kh, vh = q[rq, c].double(), k[rk, c].double(), v[rk, c].double()
            S = qh @ kh.t() * scale
            P = torch.softmax(S, dim=-1)
            o[rq, c] = P @ vh
            mag[rq, c] = P @ vh.abs()
            lse[b, h] = torch.logsumexp(S, dim=-1) * LOG2E
            X = (S * LOG2E).abs().amax(1)
            ex = U * (d * sl2 * (qh.abs() @ kh.abs().t()).amax(1) + 2 * X)
            rel_l = U * attn_lse_chain(Skv, d) + (tiles + 1) * (2.0 ** -21 + math.log(2) * 2.0 ** -23 * X)
            lb[b, h] = 2 * (ex + rel_l * LOG2E + 2.0 ** -22 * (1 + math.log2(Skv)) + U * lse[b, h].abs())
            del S, P
    return o, mag, lse, lb


def lse_violations(got, ref, bound):
    """Bool mask of the lse entries outside |got - ref| <= bound (`attention_fwd_ref`); NaN is outside."""
    return _outside((got.double() - ref).abs(), bound, "attention lse")


# (B, heads, Sq, Skv, d, layout, ND, kKV).  layout "qkv": q | k | v are column slices of one fused [B S, 3 C] buffer
# (self-attention, Sq = Skv); "kv": q is its own matrix, k | v column slices of one [B Skv, 2 C] buffer.  The output
# goes into a guarded column view (ldo > heads d), lse between flat guards.
ATTN_FWD_MATRIX = [
    (1, 1, 128, 128, 64, "qkv", 1, 128),      # one query tile, one key tile
    (2, 5, 1024, 1024, 64, "qkv", 1, 128),
    (2, 4, 1024, 77, 64, "kv", 1, 128),       # SDXL cross-attention: 77 keys in one 128-key tile
    (1, 2, 64, 64, 64, "qkv", 1, 128),        # Sq mod 128 = 64: the second warpgroup's rows all out of range
    (1, 3, 320, 200, 64, "kv", 1, 128),       # Sq mod 128 = 64, ragged last key tile
    (1, 10, 4096, 4096, 64, "qkv", 1, 128),   # SDXL 64x64 level
    (1, 3, 700, 600, 64, "kv", 1, 128),       # ragged last query tile and key tile
    (2, 2, 300, 520, 64, "kv", 1, 128),       # B = 2 with Sq mod 128 = 44: the next batch's rows would show
    (1, 2, 1024, 513, 64, "kv", 1, 128),      # Skv mod 128 = 1: one key in the last tile
    (2, 4, 129, 129, 8, "qkv", 1, 128),       # smallest head (half a k-step); Sq, Skv mod 128 = 1
    (2, 5, 65, 77, 40, "kv", 1, 128),         # Sq mod 128 = 65: one row of the second warpgroup in range
    (2, 4, 321, 321, 56, "qkv", 1, 128),      # d = 8 mod 16, Sq mod 128 = 65
    (1, 5, 320, 200, 24, "kv", 1, 128),       # any multiple of 8 works
    (2, 8, 4096, 4096, 40, "kv", 1, 128),     # SD1.x 64x64 level
    (2, 8, 1024, 77, 40, "kv", 1, 128),       # SD1.x cross-attention
    (2, 3, 193, 65, 72, "kv", 2, 64),         # ND = 2 at its smallest head; Sq mod 128 = 65, Skv mod 64 = 1
    (1, 4, 1, 77, 80, "kv", 2, 64),           # one query; Skv = 77 in 64-key tiles
    (2, 8, 1024, 1024, 80, "kv", 2, 64),      # SD1.x 32x32 level
    (1, 2, 256, 256, 128, "qkv", 2, 64),      # ND = 2 at its largest head, Skv mod 64 = 0
    (2, 2, 200, 77, 136, "kv", 3, 64),        # ND = 3 at its smallest head (d = 8 mod 16)
    (2, 8, 256, 256, 160, "kv", 3, 64),       # SD1.x 16x16 level
    (3, 8, 64, 64, 160, "kv", 3, 64),         # 8x8 level: fewer queries and keys than a tile
    (2, 8, 256, 77, 160, "kv", 3, 64),
    (1, 2, 192, 192, 192, "qkv", 3, 64),      # ND = 3 at its largest head, Sq mod 128 = 64
]


def _attn_fwd_inputs(dev, B, heads, Sq, Skv, d, layout, seed):
    g = torch.Generator().manual_seed(seed)
    Cc = heads * d
    if layout == "qkv":
        assert Sq == Skv
        qkv = torch.randn(B * Sq, 3 * Cc, generator=g).to(dev, BF)
        return qkv[:, :Cc], qkv[:, Cc:2 * Cc], qkv[:, 2 * Cc:]
    q = torch.randn(B * Sq, Cc, generator=g).to(dev, BF)
    kv = torch.randn(B * Skv, 2 * Cc, generator=g).to(dev, BF)
    return q, kv[:, :Cc], kv[:, Cc:]


def run_attention_fwd(q, k, v, B, heads, Sq, Skv, d, scale):
    """Two calls into guarded outputs (checked), one `ops.attention` call (bitwise equal); returns (o, lse)."""
    from sliders_b200 import ops

    P = ops._p
    Cc = heads * d
    n = B * heads * Sq
    runs = []
    for _ in range(2):
        buf, o = guarded_out(B * Sq, Cc, dev=q.device)
        lbuf, lse = flat_guarded(n, torch.float32, q.device)
        _lib_call("sb200_attention", P(q), q.stride(0), P(k), k.stride(0), P(v), v.stride(0), P(o), o.stride(0), B,
                  heads, Sq, Skv, int(d), float(scale), P(lse))
        torch.cuda.synchronize()
        assert o.stride(0) > Cc
        assert_guard_intact(buf, B * Sq, Cc)
        assert_flat_guard(lbuf, n)
        runs.append((o, lse.view(B, heads, Sq)))
    assert_bitwise(runs[0][0], runs[1][0], "attention o")
    assert_bitwise(runs[0][1], runs[1][1], "attention lse")
    lse_w = torch.empty(B, heads, Sq, device=q.device, dtype=torch.float32)
    o_w = ops.attention(q, k, v, B, heads, Sq, Skv, scale, head_dim=d, lse=lse_w)
    torch.cuda.synchronize()
    assert_bitwise(o_w, runs[0][0], "ops.attention vs the C ABI call")
    assert_bitwise(lse_w, runs[0][1], "ops.attention lse vs the C ABI call")
    return runs[0]


def check_attention_fwd(o, lse, q, k, v, B, heads, Sq, Skv, d, scale):
    ref, mag, lref, lb = attention_fwd_ref(q, k, v, B, heads, Sq, Skv, d, scale)
    assert_no_violations(attn_violations(o, ref, mag), o, ref, "attention o")
    assert_no_violations(lse_violations(lse, lref, lb), lse, lref, "attention lse")


@pytest.mark.parametrize("B,heads,Sq,Skv,d,layout,nd,kv", ATTN_FWD_MATRIX)
def test_attention_fwd_bound(dev, B, heads, Sq, Skv, d, layout, nd, kv):
    assert attn_nd(d) == nd and attn_fwd_kv(d) == kv
    q, k, v = _attn_fwd_inputs(dev, B, heads, Sq, Skv, d, layout, Sq + Skv + d + B)
    scale = d ** -0.5
    o, lse = run_attention_fwd(q, k, v, B, heads, Sq, Skv, d, scale)
    check_attention_fwd(o, lse, q, k, v, B, heads, Sq, Skv, d, scale)


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm / GroupNorm forward
# ------------------------------------------------------------------------------------------------------------------
def layernorm_ref(x, gamma, beta):
    """(ref, mag, stat) of gamma (x - mean) rstd + beta over the rows of x, float64, for `norm_violations` (add = 0).
    mag = |gamma| (1 + |xhat|) + |beta| bounds every term of the fp32 expression, and an error e in xhat moves the
    output by |gamma| e.  layernorm_kernel takes two passes over the row in registers (sum, then the squares of
    x - mean): a chain of n roundings makes the mean err by n 2^-24 (|mean| + sigma) and the variance by about
    n 2^-24 var, so xhat errs by n 2^-24 stat (1 + |xhat|) with stat = 1 + |mean| rstd (no mean^2 term: the
    variance does not cancel).  n = `ln_chain`."""
    xd = x.double()
    mean = xd.mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(((xd - mean) ** 2).mean(1, keepdim=True) + 1e-5)
    xh = (xd - mean) * rstd
    g, b = gamma.double(), beta.double()
    ref = g * xh + b
    mag = g.abs() * (1 + xh.abs()) + b.abs()
    return ref, mag, (1 + mean.abs() * rstd).expand_as(ref)


def groupnorm_ref(x, gamma, beta, groups, eps, silu):
    """x [B, HW, C] -> float64 (ref, mag, stat, mean, rstd, sigma) of GroupNorm(+SiLU), for `norm_violations`.
    The kernel computes var = E[x^2] - mean^2 in fp32, so a chain of n roundings makes the variance err by
    n 2^-24 (mean^2 + var): stat = 1 + (mean rstd)^2, as in norm_violations.  It applies the statistics as one fma
    x (rstd gamma) + (beta - mean rstd gamma), whose two terms of size |mean| rstd |gamma| cancel: |mean| rstd <= stat,
    so mag = |gamma| (1 + |xhat|) + |beta| covers them.  SiLU: |silu'| < 1.1 carries the error of z = gamma xhat + beta
    (mag x 1.1); __expf in silu_f stays within the 32 extra roundings of norm_violations for |z| < 12."""
    B, HW, C = x.shape
    cpg = C // groups
    xd = x.double().reshape(B, HW, groups, cpg)
    mean = xd.mean((1, 3), keepdim=True)
    var = ((xd - mean) ** 2).mean((1, 3), keepdim=True)
    rstd = 1 / torch.sqrt(var + eps)
    xh = (xd - mean) * rstd
    g, b = gamma.double().view(groups, cpg), beta.double().view(groups, cpg)
    z = g * xh + b
    mag = g.abs() * (1 + xh.abs()) + b.abs()
    ref = z * torch.sigmoid(z) if silu else z
    if silu:
        mag = 1.1 * mag
    stat = (1 + (mean * rstd) ** 2).expand_as(ref)
    sh = (B, HW, C)
    return (ref.reshape(sh), mag.reshape(sh), stat.reshape(sh), mean.view(B, groups), rstd.view(B, groups),
            var.sqrt().view(B, groups))


def gn_stats_violations(st, mean, rstd, sigma, chain):
    """Bool mask [B, groups, 2] of the workspace's (mean, rstd) outside
        |mean' - mean| <= c (|mean| + sigma),   |rstd' - rstd| <= c (1 + (mean rstd)^2) rstd,
    c = chain_c(chain + 8): the chain of the sums (`gn_chain`) plus the scaling by 1/n, the subtraction, + eps and
    rsqrtf (2 ulp).  E[x^2] - mean^2 errs by n 2^-24 (mean^2 + var), i.e. relatively n 2^-24 (1 + (mean rstd)^2)
    of var + eps, and rstd by half that."""
    c = chain_c(chain + 8)
    em = (st[..., 0].double() - mean).abs()
    er = (st[..., 1].double() - rstd).abs()
    bm = c * (mean.abs() + sigma)
    br = c * (1 + (mean * rstd) ** 2) * rstd
    return torch.stack([_outside(em, bm, "groupnorm stats"), _outside(er, br, "groupnorm stats")], -1)


# (M, C, offset, NV, wraps): x is a column view of a wider buffer; the output a guarded column view.  offset: the
# rows' common mean in units of their standard deviation
LN_FWD_MATRIX = [
    (7, 256, 0.0, 1, False),       # NV = 1 at its largest C
    (77, 128, 0.0, 1, False),
    (1, 264, 0.0, 3, False),       # NV = 3 at its smallest C, one row
    (33, 320, 0.0, 3, False),
    (1000, 768, 0.0, 3, False),    # NV = 3 at its largest C
    (2048, 640, 8.0, 3, False),    # |mean| / sigma = 8
    (300, 776, 0.0, 5, False),     # NV = 5 at its smallest C
    (1000, 1280, 0.0, 5, False),   # NV = 5 at its largest C (SDXL)
    (517, 1288, 0.0, 8, False),    # NV = 8 at its smallest C
    (64, 2048, 0.0, 8, False),     # NV = 8 at its largest C
    (20000, 320, 0.0, 3, True),    # more rows than 16 blocks x 8 warps per SM: the row loop wraps
    (20000, 2048, 0.0, 8, True),   # NV = 8, wrapping
]


@pytest.mark.parametrize("M,C,offset,nv,wraps", LN_FWD_MATRIX)
def test_layernorm_fwd_bound(dev, sms, M, C, offset, nv, wraps):
    from sliders_b200 import ops

    assert ln_nv(C) == nv and ln_wraps(M, sms) == wraps
    g = torch.Generator().manual_seed(M + C)
    x = col_view(M, C, 64, dev, g, 1.0 if offset else 2.0, offset or 0.5)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dev, BF)
    beta = (0.2 * torch.randn(C, generator=g)).to(dev, BF)
    assert x.stride(0) > C
    outs = []
    for _ in range(2):
        buf, o = guarded_out(M, C, dev)
        _lib_call("sb200_layernorm", ops._p(x), x.stride(0), ops._p(gamma), ops._p(beta), ops._p(o), o.stride(0), M, C,
                  1e-5)
        torch.cuda.synchronize()
        assert o.stride(0) > C
        assert_guard_intact(buf, M, C)
        outs.append(o)
    assert_bitwise(outs[0], outs[1], "layernorm")
    assert_bitwise(ops.layernorm(x, gamma, beta, 1e-5), outs[0], "ops.layernorm vs the C ABI call")
    ref, mag, stat = layernorm_ref(x, gamma, beta)
    bad = norm_violations(outs[0], ref, torch.zeros_like(ref), mag, stat, ln_chain(C))
    assert_no_violations(bad, outs[0], ref, "layernorm")


# (B, H, W, C0, C1, groups, silu, eps, offset, rows_par, one_chunk): x0 / x1 are column views of wider buffers (as the
# up-block resnets pass the skip concat); the output a guarded column view
GN_FWD_MATRIX = [
    (2, 32, 32, 320, 0, 32, True, 1e-5, 0.0, 12, False),     # SD1.x level 1
    (1, 8, 8, 320, 0, 32, True, 1e-5, 0.0, 12, True),        # small image: a single chunk
    (2, 64, 64, 640, 320, 32, True, 1e-5, 0.0, 4, False),    # up-block concat
    (1, 128, 128, 320, 0, 32, False, 1e-6, 0.0, 12, False),  # eps 1e-6, no SiLU, many rows per chunk
    (3, 8, 8, 64, 64, 32, True, 1e-5, 0.0, 32, True),        # concat of two 64-channel sources, one chunk
    (2, 16, 16, 1280, 640, 32, True, 1e-5, 0.0, 2, False),   # 1920 / 32 = 60: groups straddle vectors and x0 / x1
    (1, 64, 64, 640, 0, 32, False, 1e-6, 0.0, 6, False),     # Transformer2DModel.norm
    (2, 16, 16, 640, 0, 32, True, 1e-5, 8.0, 6, False),      # |mean| / sigma = 8: E[x^2] - mean^2 cancels
    (2, 32, 32, 1280, 1280, 32, True, 1e-5, 0.0, 1, False),  # SDXL 2560-channel concat
    (1, 2, 4, 1280, 1280, 32, False, 1e-6, 0.0, 1, True),    # rows_par = 1 in a single chunk
    (1, 16, 12, 4608, 0, 32, False, 1e-5, 0.0, 1, False),    # C > 4096, rectangular image
]


@pytest.mark.parametrize("B,H,W,C0,C1,groups,silu,eps,offset,rows_par,one_chunk", GN_FWD_MATRIX)
def test_groupnorm_fwd_bound(dev, sms, B, H, W, C0, C1, groups, silu, eps, offset, rows_par, one_chunk):
    from sliders_b200 import ops

    P = ops._p
    C, HW = C0 + C1, H * W
    rp, chunks, _ = gn_launch(B, HW, C, sms)
    assert gn_smem_ok(C) and rp == rows_par and (chunks == 1) == one_chunk
    g = torch.Generator().manual_seed(H + W + C0 + C1)
    sc, off = (1.0, offset) if offset else (1.5, 0.3)
    x0 = col_view(B * HW, C0, 16, dev, g, sc, off).view(B, H, W, C0)
    x1 = col_view(B * HW, C1, 24, dev, g, sc, -off).view(B, H, W, C1) if C1 else None
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dev, BF)
    beta = (0.2 * torch.randn(C, generator=g)).to(dev, BF)
    outs, stats = [], []
    for _ in range(2):
        buf, o = guarded_out(B * HW, C, dev)
        ws = ops.gn_ws(B, groups, dev)
        _lib_call("sb200_groupnorm", P(x0), x0.stride(-2), C0, P(x1), x1.stride(-2) if C1 else 0, C1, P(gamma),
                  P(beta), P(o), o.stride(0), B, HW, groups, float(eps), int(silu), P(ws))
        torch.cuda.synchronize()
        assert o.stride(0) > C
        assert_guard_intact(buf, B * HW, C)
        outs.append(o)
        stats.append(ops.gn_stats(ws, B, groups).clone())
    assert_bitwise(outs[0], outs[1], "groupnorm")
    assert_bitwise(stats[0], stats[1], "groupnorm (mean, rstd)")
    ws = ops.gn_ws(B, groups, dev)
    o_w = ops.groupnorm(x0, gamma, beta, groups, eps, silu, x1=x1, stats_ws=ws)
    torch.cuda.synchronize()
    assert_bitwise(o_w.view(B * HW, C), outs[0], "ops.groupnorm vs the C ABI call")
    assert_bitwise(ops.gn_stats(ws, B, groups), stats[0], "ops.groupnorm (mean, rstd) vs the C ABI call")
    x = torch.cat([x0, x1], -1) if x1 is not None else x0
    ref, mag, stat, mean, rstd, sigma = groupnorm_ref(x.reshape(B, HW, C), gamma, beta, groups, eps, silu)
    chain = gn_chain(B, HW, C, groups, sms)
    out = outs[0].view(B, HW, C)
    assert_no_violations(norm_violations(out, ref, torch.zeros_like(ref), mag, stat, chain), out, ref, "groupnorm")
    st = stats[0]
    ref_st = torch.stack([mean, rstd], -1)
    assert_no_violations(gn_stats_violations(st, mean, rstd, sigma, chain), st, ref_st, "groupnorm (mean, rstd)")


# ------------------------------------------------------------------------------------------------------------------
# small_linear
# ------------------------------------------------------------------------------------------------------------------
def small_linear_chain(K, lora):
    """Dependent fp32 roundings of y: dot8 adds 8 products in 4 steps of (a0 b0 + a1 b1) (3 roundings each) and the
    lane adds the result (13 per 8-channel vector); a lane takes every 32nd vector, then a 5-step shuffle tree and the
    bias.  LoRA: T has the same chain, then r products, the scale and the add."""
    dot = 13 * cdiv(K // 8, 32) + 5
    return dot + 1 + (dot + 8 + 3 if lora else 0)


def silu_tol(x):
    """Absolute error bound of the kernel's fp32 silu_f(x) = x / (1 + __expf(-x)): __expf errs by (2 + 1.16 |x|) ulp,
    the add and the division by one each; a factor 2 on top."""
    s = x * torch.sigmoid(x)
    return U * (8 + 2.32 * x.abs()) * s.abs()


def _bf16_flip(val, tol):
    """|bf16(val + tol) - bf16(val - tol)|: the size of the one-ulp flip a value known to within tol may take when it
    is rounded to bf16 (zero unless val lies within tol of a rounding midpoint)."""
    return ((val + tol).to(BF).double() - (val - tol).to(BF).double()).abs()


def small_linear_ref(x, w, b, act_in, act_out, lora, scale, resid):
    """float64 (ref, abs) of small_linear for `small_linear_violations`: |out - ref| <= 2^-7 |ref| + abs.
    The kernel rounds twice to bf16 on purpose, as the framework it replaces does: bf16(silu(x)) on the input
    (act_in) and bf16(y + resid) before the act_out = 2 SiLU.  The reference makes the same roundings of its float64
    values, which agree with the kernel's except where the kernel's value lies within its own fp32 error of a bf16
    rounding midpoint; there, and only there, a one-ulp flip (`_bf16_flip`) enters the bound:
    - act_in: flip_in [M, K] (silu_tol), which moves y by flip_in |W|^T (+ the LoRA path);
    - y: E_y = chain_c(small_linear_chain) mag_y + the input flips, mag_y = |x'| |W|^T + |b| + |s| (|x'| |D|^T) |U|^T;
    - act_out 1: silu(y) + resid: 1.1 E_y (|silu'| < 1.1), silu_tol, one rounding of the add;
    - act_out 2: silu(bf16(y + resid)): a flip of bf16(y + resid) where y + resid lies within E_y of a midpoint,
      times 1.1, and silu_tol.
    2^-7 |ref|: the output rounding with a factor 2."""
    xd = x.double()
    if act_in:
        s = xd * torch.sigmoid(xd)
        xin, flip_in = s.to(BF).double(), _bf16_flip(s, silu_tol(xd))
    else:
        xin, flip_in = xd, torch.zeros_like(xd)
    wd, wa = w.double(), w.double().abs()
    y = xin @ wd.t()
    mag = xin.abs() @ wa.t()
    fl = flip_in @ wa.t()
    if b is not None:
        y, mag = y + b.double(), mag + b.double().abs()
    if lora is not None:
        down, up, r, group_n = lora
        dd, ud = down.double(), up.double()
        t, tm, tf = xin @ dd.t(), xin.abs() @ dd.abs().t(), flip_in @ dd.abs().t()
        for g0 in range(0, y.shape[1], group_n):
            i = g0 // group_n
            cols, rows = slice(g0, g0 + group_n), slice(i * r, (i + 1) * r)
            y[:, cols] += scale * t[:, rows] @ ud[cols].t()
            mag[:, cols] += abs(scale) * tm[:, rows] @ ud[cols].abs().t()
            fl[:, cols] += abs(scale) * tf[:, rows] @ ud[cols].abs().t()
    ey = chain_c(small_linear_chain(x.shape[1], lora is not None)) * mag + fl
    rd = resid.double() if resid is not None else torch.zeros_like(y)
    if act_out == 0:
        return y + rd, ey + chain_c(1) * (y.abs() + rd.abs())
    if act_out == 1:
        sy = y * torch.sigmoid(y)
        return sy + rd, 1.1 * ey + silu_tol(y) + chain_c(1) * (sy.abs() + rd.abs())
    s = y + rd
    tol = ey + chain_c(1) * s.abs()
    u = s.to(BF).double()
    flip = _bf16_flip(s, tol)
    return u * torch.sigmoid(u), 1.1 * flip + silu_tol(u.abs() + flip)


def small_linear_violations(out, ref, abs_):
    err = (out.double() - ref).abs()
    return _outside(err, 2.0 ** -7 * ref.abs() + abs_, "small_linear")


# (M, N, K, xpad, act_in, act_out, lora (r, group_n, scale) or None, resid): x is a column view when xpad > 0; the
# output a guarded column view.  The kernel's blocks are 8 output columns.
SL_MATRIX = [
    (1, 1280, 320, 0, False, 1, None, False),          # time_embedding.linear_1 at batch 1
    (2, 1280, 320, 0, False, 1, None, False),
    (8, 1280, 2816, 64, False, 1, None, False),        # SDXL add_embedding.linear_1, column-view x
    (4, 640, 1280, 0, True, 0, None, False),           # time_emb_proj with SiLU on the input
    (16, 320, 1280, 0, False, 0, (4, 320, 0.5), False),
    (3, 1280, 1280, 8, True, 0, (8, 1280, -1.5), False),
    (2, 1280, 1280, 0, False, 2, None, True),          # add_embedding.linear_2: SiLU(bf16(y + emb))
    (7, 100, 8, 8, False, 1, None, True),              # N = 100: the last block has 4 columns; K = 8
    (9, 40, 320, 16, True, 0, (4, 20, 1.0), False),    # group_n 20: the block of columns 16..23 spans two groups
    (8, 40, 1280, 0, False, 2, (8, 20, -0.75), True),  # rank 8, two groups, act_out 2 with a residual
    (64, 1280, 1280, 24, False, 1, (1, 1280, 2.0), True),   # the largest M, rank 1, SiLU + residual
    (1, 1280, 2816, 0, False, 0, None, True),          # act_out 0 with a residual
]


def _sl_case(dev, M, N, K, xpad, act_in, lora, resid, seed):
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(seed)
    x = col_view(M, K, xpad, dev, g) if xpad else torch.randn(M, K, generator=g).to(dev, BF)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, BF)
    b = torch.randn(N, generator=g).to(dev, BF)
    res = torch.randn(M, N, generator=g).to(dev, BF) if resid else None
    la = lref = None
    if lora:
        r, group_n, scale = lora
        down, up, _ = make_lora(K, N, r, group_n, dev, seed + 1)
        la = ops.Lora(down, up, r, group_n, scale)
        lref = (down, up, r, group_n)
    return x, w, b, res, la, lref


def run_small_linear(x, w, b, act_in, act_out, la, res):
    from sliders_b200 import ops

    P = ops._p
    M, K = x.shape
    N = w.shape[0]
    outs = []
    for _ in range(2):
        buf, o = guarded_out(M, N, x.device)
        _lib_call("sb200_small_linear", P(x), x.stride(0), P(w), w.stride(0), P(b), P(o), o.stride(0), M, N, K,
                  int(act_in), int(act_out), la.ref() if la is not None else None, P(res))
        torch.cuda.synchronize()
        assert o.stride(0) > N
        assert_guard_intact(buf, M, N)
        outs.append(o)
    assert_bitwise(outs[0], outs[1], "small_linear")
    return outs[0]


@pytest.mark.parametrize("M,N,K,xpad,act_in,act_out,lora,resid", SL_MATRIX)
def test_small_linear_bound(dev, M, N, K, xpad, act_in, act_out, lora, resid):
    from sliders_b200 import ops

    x, w, b, res, la, lref = _sl_case(dev, M, N, K, xpad, act_in, lora, resid, M + N + K)
    assert (x.stride(0) > K) == (xpad > 0)
    out = run_small_linear(x, w, b, act_in, act_out, la, res)
    o_w = ops.small_linear(x, w, b, act_in=act_in, act_out=act_out, lora=la, resid=res)
    torch.cuda.synchronize()
    assert_bitwise(o_w, out, "ops.small_linear vs the C ABI call")
    ref, abs_ = small_linear_ref(x, w, b, act_in, act_out, lref, lora[2] if lora else 0.0, res)
    assert_no_violations(small_linear_violations(out, ref, abs_), out, ref, "small_linear")


def test_small_linear_scale_dev(dev):
    """Lora.scale_dev: the slider scale read from device memory at run time (times the host scale), across a
    device-side update; two LoRA groups so that one block of columns spans both."""
    from sliders_b200 import ops

    M, N, K, r, group_n = 5, 40, 320, 4, 20
    x, w, b, res, _, lref = _sl_case(dev, M, N, K, 8, False, (r, group_n, 1.0), True, 77)
    down, up = lref[0], lref[1]
    t = torch.tensor([-3.0], device=dev)
    dyn = ops.Lora(down, up, r, group_n, 0.5, scale_dev=t)
    for val in (-3.0, 2.0):
        t.fill_(val)   # a device-side update between calls, as a captured graph sees it
        out = run_small_linear(x, w, b, False, 1, dyn, res)
        host = run_small_linear(x, w, b, False, 1, ops.Lora(down, up, r, group_n, 0.5 * val), res)
        assert_bitwise(out, host, f"scale_dev = {val} vs the host scale")
        ref, abs_ = small_linear_ref(x, w, b, False, 1, lref, 0.5 * val, res)
        assert_no_violations(small_linear_violations(out, ref, abs_), out, ref, f"small_linear scale_dev {val}")


# ------------------------------------------------------------------------------------------------------------------
# sinusoid, conv_in, conv_out, upsample2x
# ------------------------------------------------------------------------------------------------------------------
def sinusoid_ref(values, dim):
    """float64 (ref, abs): [cos(t f_j) | sin(t f_j)], f_j = exp(-ln(10^4) j / (dim / 2)).  The kernel's fp32 f_j
    errs relatively by the expf (2 ulp), the division and the exponent's own rounding (ln(10^4) 2^-24 < 10 2^-24),
    so the argument t f_j by about 14 2^-24 |t f_j| and cosf / sinf add 2 ulp; abs = 2^-24 (32 |t f_j| + 16) takes
    a factor 2.  The output rounding is the 2^-7 |ref| of pointwise_violations."""
    half = dim // 2
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=values.device) / half)
    arg = values.double()[:, None] * f[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], -1)
    return ref, torch.cat([U * (32 * arg.abs() + 16)] * 2, -1)


def test_sinusoid_bound(dev):
    """The timestep embedding (dim 320) and the SDXL time-id embedding (dim 256), each written into a guarded column
    view."""
    from sliders_b200 import ops

    vals = torch.tensor([0.0, 1.0, 0.37, 17.25, 500.0, 999.0, 1024.0, 768.0, 0.0], device=dev)  # + SDXL time ids
    n = vals.numel()
    for dim in (320, 256):
        outs = []
        for _ in range(2):
            buf, o = guarded_out(n, dim, dev)
            _lib_call("sb200_sinusoid", ops._p(vals), n, dim, ops._p(o), o.stride(0))
            torch.cuda.synchronize()
            assert o.stride(0) > dim
            assert_guard_intact(buf, n, dim)
            outs.append(o)
        assert_bitwise(outs[0], outs[1], "sinusoid")
        assert_bitwise(ops.sinusoid(vals, dim), outs[0], "ops.sinusoid vs the C ABI call")
        ref, abs_ = sinusoid_ref(vals, dim)
        bad = _outside((outs[0].double() - ref).abs(), 2.0 ** -7 * ref.abs() + abs_, "pointwise")
        assert_no_violations(bad, outs[0], ref, f"sinusoid dim {dim}")


def conv_ref(x_nchw, w_oikk, bias):
    """float64 (ref, mag) of a 3x3 / pad 1 conv (x NCHW, w [Cout, Cin, 3, 3])."""
    conv = torch.nn.functional.conv2d
    ref = conv(x_nchw.double(), w_oikk.double(), bias.double() if bias is not None else None, padding=1)
    mag = conv(x_nchw.double().abs(), w_oikk.double().abs(), bias.double().abs() if bias is not None else None,
               padding=1)
    return ref, mag


# (B, H, W, Cout, latent dtype, wraps): conv_in writes contiguous NHWC between flat guards
CONV_IN_MATRIX = [
    (2, 32, 32, 320, torch.float32, False),
    (2, 32, 32, 320, BF, False),
    (1, 17, 23, 680, torch.float32, False),    # the largest Cout (36 Cout bf16 of shared memory <= 48 KB), odd H / W
    (3, 1, 9, 320, BF, False),                 # one image row: every pixel on the top and bottom border
    (8, 128, 128, 320, BF, True),              # SDXL latent at B = 8: the grid-stride loop wraps
    (1, 96, 160, 640, torch.float32, True),    # rectangular, wrapping
]


@pytest.mark.parametrize("B,H,W,Cout,dt,wraps", CONV_IN_MATRIX)
def test_conv_in_bound(dev, sms, B, H, W, Cout, dt, wraps):
    from sliders_b200 import ops

    P = ops._p
    assert conv_in_wraps(B, H, W, Cout, sms) == wraps
    g = torch.Generator().manual_seed(B + H + W + Cout)
    lat = (torch.randn(B, 4, H, W, generator=g) * 1.3).to(dev, dt)
    w = (torch.randn(Cout, 3, 3, 4, generator=g) / 6).to(dev, BF)
    b = torch.randn(Cout, generator=g).to(dev, BF)
    n = B * H * W * Cout
    outs = []
    for _ in range(2):
        buf, o = flat_guarded(n, BF, dev)
        _lib_call("sb200_conv_in", P(lat), int(dt == torch.float32), P(w), P(b), P(o), B, H, W, Cout)
        torch.cuda.synchronize()
        assert_flat_guard(buf, n)
        outs.append(o.view(B, H, W, Cout))
    assert_bitwise(outs[0], outs[1], "conv_in")
    assert_bitwise(ops.conv_in(lat, w, b), outs[0], "ops.conv_in vs the C ABI call")
    # the kernel rounds the latent to bf16 (the model dtype) before the taps
    ref, mag = conv_ref(lat.to(BF), w.permute(0, 3, 1, 2), b)
    ref, mag = ref.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)
    # 36 dependent FMAs onto the bias, one bf16 rounding
    assert_no_violations(pointwise_violations(outs[0], ref, mag, chain_c(37)), outs[0], ref, "conv_in")


def conv_out_chain(Cin):
    """conv_out_kernel: a lane adds dot8 (13 roundings, see small_linear_chain) per 8-channel vector it owns, over 9
    taps, then a 5-step shuffle tree and the bias."""
    return 9 * 13 * cdiv(Cin // 8, 32) + 6


# (B, H, W, Cin, out dtype, bias, wraps): contiguous NHWC input, NCHW output between flat guards
CONV_OUT_MATRIX = [
    (2, 32, 32, 320, torch.float32, True, False),
    (2, 32, 32, 320, BF, True, False),
    (1, 9, 7, 8, BF, True, False),              # one vector: lanes 1..31 idle
    (2, 11, 13, 264, torch.float32, False, False),  # 33 vectors: lane 0 takes two; no bias
    (1, 17, 5, 680, BF, False, False),          # the largest Cin
    (4, 64, 64, 320, torch.float32, True, True),    # more pixels than 8 blocks x 8 warps per SM: wraps
    (4, 64, 64, 264, BF, False, True),
]


@pytest.mark.parametrize("B,H,W,Cin,dt,with_bias,wraps", CONV_OUT_MATRIX)
def test_conv_out_bound(dev, sms, B, H, W, Cin, dt, with_bias, wraps):
    from sliders_b200 import ops

    P = ops._p
    assert conv_out_wraps(B, H, W, sms) == wraps
    g = torch.Generator().manual_seed(B + H + W + Cin)
    x = torch.randn(B, H, W, Cin, generator=g).to(dev, BF)
    w = (torch.randn(4, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5).to(dev, BF)
    b = torch.randn(4, generator=g).to(dev, BF) if with_bias else None
    n = B * 4 * H * W
    outs = []
    for _ in range(2):
        buf, o = flat_guarded(n, dt, dev)
        _lib_call("sb200_conv_out", P(x), P(w), P(b), P(o), int(dt == torch.float32), B, H, W, Cin)
        torch.cuda.synchronize()
        assert_flat_guard(buf, n)
        outs.append(o.view(B, 4, H, W))
    assert_bitwise(outs[0], outs[1], "conv_out")
    assert_bitwise(ops.conv_out(x, w, b, out_dtype=dt), outs[0], "ops.conv_out vs the C ABI call")
    ref, mag = conv_ref(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), b)
    if dt == torch.float32:
        bad = reduction_violations(outs[0], ref, mag, conv_out_chain(Cin))
    else:
        bad = pointwise_violations(outs[0], ref, mag, chain_c(conv_out_chain(Cin)))
    assert_no_violations(bad, outs[0], ref, "conv_out")


# (B, H, W, C, wraps)
UPSAMPLE_MATRIX = [(2, 8, 8, 64, False), (1, 5, 7, 8, False), (3, 9, 1, 320, False), (2, 64, 64, 320, True),
                   (1, 33, 65, 640, True)]


@pytest.mark.parametrize("B,H,W,C,wraps", UPSAMPLE_MATRIX)
def test_upsample2x_exact(dev, sms, B, H, W, C, wraps):
    from sliders_b200 import ops

    assert upsample_wraps(B, H, W, C, sms) == wraps
    g = torch.Generator().manual_seed(B + H + W + C)
    x = torch.randn(B, H, W, C, generator=g).to(dev, BF)
    n = B * 4 * H * W * C
    outs = []
    for _ in range(2):
        buf, o = flat_guarded(n, BF, dev)
        _lib_call("sb200_upsample2x", ops._p(x), ops._p(o), B, H, W, C)
        torch.cuda.synchronize()
        assert_flat_guard(buf, n)
        outs.append(o.view(B, 2 * H, 2 * W, C))
    ref = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    assert torch.equal(bits(outs[0]), bits(ref)), "upsample2x is not bit-exact"
    assert_bitwise(outs[1], outs[0], "upsample2x")
    assert_bitwise(ops.upsample2x(x), outs[0], "ops.upsample2x vs the C ABI call")


# ------------------------------------------------------------------------------------------------------------------
# CFG + DDIM / affine scheduler step
# ------------------------------------------------------------------------------------------------------------------
def cfg_ref(eps2, g, x, a, b, mode):
    """float64 (eps, eps_mag, x_prev, x_mag) of the guided eps and the step.  mode "ddim": x_prev = sqrt(b) x0 +
    sqrt(1 - b) eps with x0 = (x - sqrt(1 - a) eps) / sqrt(a); "affine": a x + b eps (sb200_cfg_step: the scheduler's
    cx, ce); "single": eps2 is one guided batch (g = 0) and the step is DDIM; "eps": no x.  The magnitudes are the
    same expressions on absolute values, so x_mag carries the 1 / sqrt(a) amplification of x0."""
    e2 = eps2.double()
    if mode == "single":
        eu = ec = e2
    else:
        eu, ec = e2.chunk(2)
    e = eu + g * (ec - eu)
    em = eu.abs() + abs(g) * (ec.abs() + eu.abs())
    if x is None:
        return e, em, None, None
    xd = x.double()
    if mode == "affine":
        return e, em, a * xd + b * e, abs(a) * xd.abs() + abs(b) * em
    sa, sb, pa, pb = math.sqrt(a), math.sqrt(1 - a), math.sqrt(b), math.sqrt(1 - b)
    return e, em, pa * (xd - sb * e) / sa + pb * e, pa * (xd.abs() + sb * em) / sa + pb * em


CFG_CHAIN = 12  # g (ec - eu) + eu: 3 roundings; sqrtf x 4, x - sb e, / sa, pa x0 + pb e: 9 more


def cfg_violations(out, ref, mag):
    """|out - ref| <= 2^-7 |ref| (bf16 outputs only: the output rounding, factor 2) + chain_c(CFG_CHAIN) mag."""
    a = 2.0 ** -7 if out.dtype == BF else 0.0
    return _outside((out.double() - ref).abs(), a * ref.abs() + chain_c(CFG_CHAIN) * mag, "cfg")


# (eps dtype, out dtype, g, mode, latent shape [B, 4, H, W], wraps): outputs between flat guards
CFG_MATRIX = [
    (torch.float32, torch.float32, 7.5, "ddim", (2, 4, 31, 33), False),   # n = 8184: not a multiple of 256
    (BF, BF, 7.5, "ddim", (8, 4, 128, 128), True),                         # SDXL latent at B = 8
    (torch.float32, BF, 1.0, "affine", (1, 4, 17, 19), False),
    (BF, torch.float32, 0.0, "affine", (8, 4, 128, 128), True),
    (torch.float32, torch.float32, 0.0, "single", (1, 4, 64, 64), False),
    (BF, BF, 0.0, "single", (2, 4, 9, 7), False),
    (torch.float32, BF, 7.5, "eps", (8, 4, 128, 128), True),
    (BF, torch.float32, 1.0, "eps", (3, 4, 5, 11), False),
    (torch.float32, torch.float32, 1.0, "affine", (2, 4, 64, 64), False),
    (BF, BF, 0.0, "eps", (2, 4, 32, 32), False),
]


@pytest.mark.parametrize("te,to,g,mode,shape,wraps", CFG_MATRIX)
def test_cfg_step_bound(dev, sms, te, to, g, mode, shape, wraps):
    from sliders_b200 import ops

    P = ops._p
    n = math.prod(shape)
    assert cfg_wraps(n, sms) == wraps
    gen = torch.Generator().manual_seed(n + int(g * 2))
    eps2 = torch.randn((shape if mode == "single" else (2 * shape[0],) + shape[1:]), generator=gen).to(dev, te)
    x = (torch.randn(shape, generator=gen) * 2).to(dev, to) if mode != "eps" else None
    a, b = (1.0, -0.0625) if mode == "affine" else (0.3, 0.5)   # affine: (cx, ce) of an Euler step
    outs = []
    for _ in range(2):
        ebuf, e = flat_guarded(n, to, dev)
        xbuf, xp = flat_guarded(n, to, dev) if x is not None else (None, None)
        fn = "sb200_cfg_step" if mode == "affine" else "sb200_cfg_ddim"
        _lib_call(fn, P(eps2), int(te == torch.float32), float(g), P(x), float(a), float(b), P(xp), P(e),
                  int(to == torch.float32), n)
        torch.cuda.synchronize()
        assert_flat_guard(ebuf, n)
        if x is not None:
            assert_flat_guard(xbuf, n)
        outs.append((e, xp))
    assert_bitwise(outs[0][0], outs[1][0], "cfg eps")
    e_w, x_w = ops.cfg_ddim(eps2, g, x, a, b, out_dtype=to, single=mode == "single", affine=mode == "affine")
    torch.cuda.synchronize()
    assert_bitwise(e_w.reshape(-1), outs[0][0], "ops.cfg_ddim eps vs the C ABI call")
    e_ref, e_mag, x_ref, x_mag = cfg_ref(eps2.reshape(-1), g, x.reshape(-1) if x is not None else None, a, b, mode)
    assert_no_violations(cfg_violations(outs[0][0], e_ref, e_mag), outs[0][0], e_ref, "cfg eps")
    if x is not None:
        assert_bitwise(outs[0][1], outs[1][1], "cfg x_prev")
        assert_bitwise(x_w.reshape(-1), outs[0][1], "ops.cfg_ddim x_prev vs the C ABI call")
        assert_no_violations(cfg_violations(outs[0][1], x_ref, x_mag), outs[0][1], x_ref, "cfg x_prev")
