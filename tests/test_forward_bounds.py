"""Host-side checks of the forward-kernel test machinery in test_gpu_forward_bounds.py: each per-element bound accepts
a CPU emulation of its kernel's roundings and rejects the local errors a forward kernel can make (which rel-RMS over
the whole output does not), the forward wrappers refuse layouts their kernels do not read, and the variant tables
cover every launch variant of the host code."""
import math

import pytest
import torch

from test_gpu_backward_bounds import BF, attn_nd, attn_violations, gn_chain, gn_launch, gn_smem_ok, ln_chain, ln_nv, \
    ln_wraps, norm_violations, pointwise_violations, reduction_violations
from test_gpu_forward_bounds import (ATTN_FWD_MATRIX, CFG_MATRIX, CONV_IN_MATRIX, CONV_OUT_MATRIX, GN_FWD_MATRIX, LOG2E,
                                     LN_FWD_MATRIX, SL_MATRIX, UPSAMPLE_MATRIX, attention_fwd_ref, attn_fwd_kv,
                                     attn_ksteps, cfg_ref, cfg_violations, cfg_wraps, conv_in_wraps, conv_out_chain,
                                     conv_out_wraps, conv_ref, gn_stats_violations, groupnorm_ref, layernorm_ref,
                                     lse_violations, _bf16_flip, silu_tol, small_linear_ref, small_linear_violations, upsample_wraps)
from test_gpu_kernels import rel_rms

SMS = (114, 132)  # H100 PCIe .. SXM


def _only(v, where):
    """v holds violations at `where` and nowhere else."""
    mask = torch.zeros_like(v)
    mask[where] = True
    return bool(v[where].any()) and not bool((v & ~mask).any())


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------
def _attn_head_emulation(qh, kh, vh, scale):
    """attention_kernel on one head: fp32 S and x = S scale log2(e), p = 2^(x - m), l summed from the unrounded p,
    P rounded to bf16 for the P V product; returns (o fp32, lse)."""
    x = (qh.float() @ kh.float().t()) * torch.tensor(scale * LOG2E, dtype=torch.float32)
    m = x.amax(1, keepdim=True)
    p = torch.exp2(x - m)
    l = p.sum(1, keepdim=True)
    return (p.to(BF).float() @ vh.float()) / l, (m + torch.log2(l)).squeeze(1)


def test_attention_fwd_bound_and_planted_errors():
    g = torch.Generator().manual_seed(3)
    heads, d, Sq, Skv = 2, 40, 4096, 129   # 129 keys: the last 128-key tile holds one key
    Cc = heads * d
    q, k, v = (torch.randn(S, Cc, generator=g).to(BF) for S in (Sq, Skv, Skv))
    scale = d ** -0.5
    ref, mag, lref, lb = attention_fwd_ref(q, k, v, 1, heads, Sq, Skv, d, scale)
    o = torch.empty(Sq, Cc)
    lse = torch.empty(1, heads, Sq)
    for h in range(heads):
        c = slice(h * d, (h + 1) * d)
        o[:, c], lse[0, h] = _attn_head_emulation(q[:, c], k[:, c], v[:, c], scale)
    o = o.to(BF)
    assert not attn_violations(o, ref, mag).any()
    assert not lse_violations(lse, lref, lb).any()

    # head 0 of one query row reads the 8 columns past its d = 40 into head 1 (a box not clipped at the head)
    row = 1000
    wide = slice(0, d + 8)
    bad, bad_lse = o.clone(), lse.clone()
    ob, lb0 = _attn_head_emulation(q[row:row + 1, wide], k[:, wide], v[:, wide], scale)
    bad[row, :d], bad_lse[0, 0, row] = ob[0, :d].to(BF), lb0[0]
    assert _only(attn_violations(bad, ref, mag), (row, slice(0, d)))
    assert _only(lse_violations(bad_lse, lref, lb), (0, 0, row))
    assert rel_rms(bad, ref) < 2e-2

    # the rows of one query tile drop the one key of the last key tile (a mask one key short)
    rows = slice(128, 256)
    bad, bad_lse = o.clone(), lse.clone()
    for h in range(heads):
        c = slice(h * d, (h + 1) * d)
        ob, lb0 = _attn_head_emulation(q[rows, c], k[:Skv - 1, c], v[:Skv - 1, c], scale)
        bad[rows, c], bad_lse[0, h, rows] = ob.to(BF), lb0
    va = attn_violations(bad, ref, mag)
    assert va[rows].any(1).float().mean() > 0.9 and not va[:128].any() and not va[256:].any()
    vl = lse_violations(bad_lse, lref, lb)
    assert vl[0, :, rows].all() and int(vl.sum()) == 2 * 128
    assert rel_rms(bad, ref) < 2e-2

    bad = o.clone()
    bad[7, 3] = float("nan")
    assert attn_violations(bad, ref, mag)[7, 3]
    bad_lse = lse.clone()
    bad_lse[0, 1, 5] = float("nan")
    assert lse_violations(bad_lse, lref, lb)[0, 1, 5]


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm / GroupNorm
# ------------------------------------------------------------------------------------------------------------------
def _plant_vector(out, row, vec):
    bad = out.clone()
    bad[row, 8 * vec:8 * vec + 8] = out[row + 1, 8 * vec:8 * vec + 8]
    return bad


def test_layernorm_fwd_bound():
    g = torch.Generator().manual_seed(0)
    M, C = 512, 1288
    x = torch.randn(M, C, generator=g) * 2 + 0.5
    x[256:] = torch.randn(256, C, generator=g) + 8.0    # |mean| / sigma = 8
    x = x.to(BF)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(BF)
    beta = (0.2 * torch.randn(C, generator=g)).to(BF)
    ref, mag, stat = layernorm_ref(x, gamma, beta)
    zero = torch.zeros_like(ref)
    # the kernel: two-pass fp32 statistics, fp32 expression, one bf16 store
    xf = x.float()
    mean = xf.mean(1, keepdim=True)
    rstd = torch.rsqrt(((xf - mean) ** 2).mean(1, keepdim=True) + 1e-5)
    out = ((xf - mean) * rstd * gamma.float() + beta.float()).to(BF)
    chain = ln_chain(C)
    assert not norm_violations(out, ref, zero, mag, stat, chain).any()
    for row in (100, 300):
        bad = _plant_vector(out, row, 31)
        assert _only(norm_violations(bad, ref, zero, mag, stat, chain), (row, slice(8 * 31, 8 * 32)))
        assert rel_rms(bad, ref) < 1e-2
    bad = out.clone()
    bad[3, 5] = float("nan")
    assert norm_violations(bad, ref, zero, mag, stat, chain)[3, 5]


def test_groupnorm_fwd_bound_and_stats():
    g = torch.Generator().manual_seed(1)
    B, HW, C, groups, eps = 2, 256, 1920, 32, 1e-5   # 60 channels per group: vector 7 straddles groups 0 and 1
    x = torch.randn(B, HW, C, generator=g) * 1.5 + 0.3
    x[1] = torch.randn(HW, C, generator=g) + 8.0       # batch 1: |mean| / sigma = 8
    x = x.to(BF)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(BF)
    beta = (0.2 * torch.randn(C, generator=g)).to(BF)
    ref, mag, stat, mean, rstd, sigma = groupnorm_ref(x, gamma, beta, groups, eps, True)
    zero = torch.zeros_like(ref)
    # the kernel: E[x^2] - mean^2 in fp32, folded into one fma per element, SiLU, one bf16 store
    cpg = C // groups
    xf = x.float().view(B, HW, groups, cpg)
    m = xf.mean((1, 3))
    r = torch.rsqrt(torch.clamp((xf * xf).mean((1, 3)) - m * m, min=0) + eps)
    st = torch.stack([m, r], -1)

    def apply(stats):
        mc = stats[..., 0].repeat_interleave(cpg, 1)[:, None]
        rc = stats[..., 1].repeat_interleave(cpg, 1)[:, None]
        sc = rc * gamma.float()
        z = torch.addcmul(beta.float() - mc * sc, x.float(), sc)
        return (z * torch.sigmoid(z)).to(BF)

    out = apply(st)
    chain = gn_chain(B, HW, C, groups, 132)
    assert not norm_violations(out, ref, zero, mag, stat, chain).any()
    assert not gn_stats_violations(st, mean, rstd, sigma, chain).any()
    flat = out.view(B * HW, C)
    for row in (100, 300):
        bad = _plant_vector(flat, row, 17).view(B, HW, C)
        v = norm_violations(bad, ref, zero, mag, stat, chain).view(B * HW, C)
        assert _only(v, (row, slice(8 * 17, 8 * 18)))
        assert rel_rms(bad, ref) < 1e-2
    # one vector that straddles two groups takes the first group's statistics for all eight channels
    for b in range(B):
        bad = out.clone()
        wrong = st.clone()
        wrong[b, 1] = st[b, 0]
        bad[b, 7, 56:64] = apply(wrong)[b, 7, 56:64]
        assert _only(norm_violations(bad, ref, zero, mag, stat, chain), (b, 7, slice(60, 64)))
    # the statistics of a neighbouring group
    wrong = st.clone()
    wrong[0, 5] = st[0, 6]
    assert _only(gn_stats_violations(wrong, mean, rstd, sigma, chain), (0, 5))
    bad = out.clone()
    bad[1, 2, 3] = float("nan")
    assert norm_violations(bad, ref, zero, mag, stat, chain)[1, 2, 3]


# ------------------------------------------------------------------------------------------------------------------
# small_linear
# ------------------------------------------------------------------------------------------------------------------
def _sl_emulation(x, w, b, act_in, act_out, down, up, r, group_n, scale, resid, swap_col=None):
    """small_linear_kernel in fp32 (bf16(silu(x)) on the input, bf16(y + resid) before the act_out = 2 SiLU);
    swap_col: that column takes the LoRA term of the next group."""
    xin = torch.nn.functional.silu(x.float()).to(BF).float() if act_in else x.float()
    y = xin @ w.float().t() + b.float()
    if down is not None:
        t = xin @ down.float().t()
        N = w.shape[0]
        for n in range(N):
            gi = n // group_n + (1 if n == swap_col else 0)
            y[:, n] += scale * (t[:, gi * r:(gi + 1) * r] @ up[n].float())
    rf = resid.float() if resid is not None else 0.0
    if act_out == 1:
        y = torch.nn.functional.silu(y)
    y = y + rf
    if act_out == 2:
        y = torch.nn.functional.silu(y.to(BF).float())
    return y.to(BF)


def test_small_linear_bound_and_wrong_group():
    g = torch.Generator().manual_seed(2)
    M, N, K, r, group_n, scale = 9, 1280, 320, 4, 20, 0.25   # 64 groups: the block of columns 16..23 spans two
    x = torch.randn(M, K, generator=g).to(BF)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(BF)
    b = torch.randn(N, generator=g).to(BF)
    down = (torch.randn(N // group_n * r, K, generator=g) / K ** 0.5).to(BF)
    up = (torch.randn(N, r, generator=g) * 0.5).to(BF).float()
    lora = (down, up, r, group_n)
    ref, abs_ = small_linear_ref(x, w, b, True, 0, lora, scale, None)
    out = _sl_emulation(x, w, b, True, 0, down, up, r, group_n, scale, None)
    assert not small_linear_violations(out, ref, abs_).any()
    bad = _sl_emulation(x, w, b, True, 0, down, up, r, group_n, scale, None, swap_col=19)
    v = small_linear_violations(bad, ref, abs_)
    assert v[:, 19].float().mean() > 0.5 and not v[:, :19].any() and not v[:, 20:].any()
    assert rel_rms(bad, ref) < 1e-2
    bad = out.clone()
    bad[0, 0] = float("nan")
    assert small_linear_violations(bad, ref, abs_)[0, 0]


@pytest.mark.parametrize("act_in,act_out", [(True, 1), (False, 2), (True, 2)])
def test_small_linear_rounding_flips_are_local(act_in, act_out):
    """The bound accepts the fp32 emulation, whose bf16(silu(x)) and bf16(y + resid) may round the other way than
    the float64 reference's, and allows a flip only at the few elements within fp32 error of a bf16 midpoint."""
    g = torch.Generator().manual_seed(10 + act_out)
    M, N, K = 64, 1280, 1280
    x = (torch.randn(M, K, generator=g) * 3).to(BF)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(BF)
    b = torch.randn(N, generator=g).to(BF)
    resid = torch.randn(M, N, generator=g).to(BF)
    ref, abs_ = small_linear_ref(x, w, b, act_in, act_out, None, 0.0, resid)
    out = _sl_emulation(x, w, b, act_in, act_out, None, None, 0, 1, 0.0, resid)
    assert not small_linear_violations(out, ref, abs_).any()
    # the flip allowance applies to few elements: the silu inputs, and the y + resid values, within fp32 error of a
    # bf16 rounding midpoint
    xd = x.double()
    assert (_bf16_flip(xd * torch.sigmoid(xd), silu_tol(xd)) > 0).float().mean() < 0.01
    y = (torch.nn.functional.silu(xd).to(BF).double() if act_in else xd) @ w.double().t() + b.double()
    s = y + resid.double()
    assert (_bf16_flip(s, 2.0 ** -18 * s.abs()) > 0).float().mean() < 0.01


# ------------------------------------------------------------------------------------------------------------------
# conv_in / conv_out / CFG step
# ------------------------------------------------------------------------------------------------------------------
def test_conv_in_bound_and_missing_border_tap():
    g = torch.Generator().manual_seed(4)
    B, H, W, Cout = 1, 64, 64, 64
    lat = (torch.randn(B, 4, H, W, generator=g) * 1.3).to(BF)
    w = (torch.randn(Cout, 4, 3, 3, generator=g) / 6).to(BF)
    bias = torch.randn(Cout, generator=g).to(BF)
    ref, mag = conv_ref(lat, w, bias)
    out = torch.nn.functional.conv2d(lat.float(), w.float(), bias.float(), padding=1).to(BF)
    c = 2 * 37 * 2.0 ** -24
    assert not pointwise_violations(out, ref, mag, c).any()
    # right-border pixel (0, W - 1) drops its in-image left tap (kh = 1, kw = 0): a border test off by one
    bad = out.float()
    bad[0, :, 0, W - 1] -= w.float()[:, :, 1, 0] @ lat.float()[0, :, 0, W - 2]
    bad = bad.to(BF)
    v = pointwise_violations(bad, ref, mag, c)
    assert v[0, :, 0, W - 1].float().mean() > 0.5 and int(v.sum()) == int(v[0, :, 0, W - 1].sum())
    assert rel_rms(bad, ref) < 1e-2


def test_conv_out_bound_and_missing_border_tap():
    g = torch.Generator().manual_seed(5)
    B, H, W, Cin = 1, 64, 64, 64
    x = torch.randn(B, Cin, H, W, generator=g).to(BF)
    w = (torch.randn(4, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).to(BF)
    bias = torch.randn(4, generator=g).to(BF)
    ref, mag = conv_ref(x, w, bias)
    out = torch.nn.functional.conv2d(x.float(), w.float(), bias.float(), padding=1)
    chain = conv_out_chain(Cin)
    assert not reduction_violations(out, ref, mag, chain).any()
    assert not pointwise_violations(out.to(BF), ref, mag, 2 * chain * 2.0 ** -24).any()
    # bottom-border pixel (H - 1, 0) drops its in-image top tap (kh = 0, kw = 1)
    bad = out.clone()
    bad[0, :, H - 1, 0] -= w.float()[:, :, 0, 1] @ x.float()[0, :, H - 2, 0]
    v = reduction_violations(bad, ref, mag, chain)
    assert v[0, :, H - 1, 0].all() and int(v.sum()) == 4
    assert rel_rms(bad, ref) < 1e-2


def test_cfg_bound_and_bf16_eps():
    g = torch.Generator().manual_seed(6)
    n, gs, a, b = 4 * 64 * 64, 7.5, 0.3, 0.5
    eps2 = torch.randn(2 * n, generator=g).to(BF)
    x = torch.randn(n, generator=g) * 2
    e_ref, e_mag, x_ref, x_mag = cfg_ref(eps2, gs, x, a, b, "ddim")
    eu, ec = eps2.float().chunk(2)
    e = eu + gs * (ec - eu)
    sa, sb = math.sqrt(a), math.sqrt(1 - a)
    pa, pb = math.sqrt(b), math.sqrt(1 - b)

    def step(ev):
        return torch.tensor(pa, dtype=torch.float32) * ((x - sb * ev) / sa) + pb * ev

    assert not cfg_violations(e, e_ref, e_mag).any() and not cfg_violations(e.to(BF), e_ref, e_mag).any()
    xp = step(e)
    assert not cfg_violations(xp, x_ref, x_mag).any() and not cfg_violations(xp.to(BF), x_ref, x_mag).any()
    bad = step(e.to(BF).float())   # x_prev from the bf16-rounded guided eps
    assert cfg_violations(bad, x_ref, x_mag).float().mean() > 0.5
    assert rel_rms(bad, x_ref) < 1e-2
    bad = xp.clone()
    bad[11] = float("nan")
    assert cfg_violations(bad, x_ref, x_mag)[11]


# ------------------------------------------------------------------------------------------------------------------
# layout checks of the forward wrappers (raised before any library call, so CPU tensors show them)
# ------------------------------------------------------------------------------------------------------------------
def test_forward_wrappers_refuse_layouts_their_kernels_misread():
    from sliders_b200 import ops

    z = lambda *s, dt=BF: torch.zeros(*s, dtype=dt)  # noqa: E731
    with pytest.raises(ValueError, match="small_linear: x"):
        ops.small_linear(z(64, 4).t(), z(8, 64))
    with pytest.raises(ValueError, match="small_linear: w"):
        ops.small_linear(z(4, 64), z(64, 8).t())
    with pytest.raises(ValueError, match="small_linear: resid"):
        ops.small_linear(z(4, 64), z(8, 64), resid=z(4, 16)[:, :8])
    with pytest.raises(ValueError, match="small_linear: resid"):
        ops.small_linear(z(4, 64), z(8, 64), resid=z(8, 4).t())
    q = z(128, 3 * 128)
    with pytest.raises(ValueError, match="attention: q"):
        ops.attention(z(127, 128), q[:, 128:256], q[:, 256:], 1, 2, 128, 128, 0.125)
    with pytest.raises(ValueError, match="attention: k"):
        ops.attention(q[:, :128], z(128, 64), q[:, 256:], 1, 2, 128, 128, 0.125)
    with pytest.raises(ValueError, match="attention: v"):
        ops.attention(q[:, :128], q[:, 128:256], z(128, 128).t(), 1, 2, 128, 128, 0.125)
    with pytest.raises(ValueError, match="attention: k"):
        ops.attention(q[:, :128], z(2 * 77, 128)[:77], z(154, 128), 2, 2, 64, 77, 0.125)
    with pytest.raises(ValueError, match="attention: lse"):
        ops.attention(q[:, :128], q[:, 128:256], q[:, 256:], 1, 2, 128, 128, 0.125,
                      lse=z(1, 128, 2, dt=torch.float32).transpose(1, 2))
    with pytest.raises(ValueError, match="attention: lse"):
        ops.attention(q[:, :128], q[:, 128:256], q[:, 256:], 1, 2, 128, 128, 0.125, lse=z(1, 2, 128))
    with pytest.raises(ValueError, match="layernorm: x"):
        ops.layernorm(z(64, 8).t(), z(64), z(64))
    x = z(2, 4, 4, 64)
    with pytest.raises(ValueError, match="groupnorm: x0"):
        ops.groupnorm(x.permute(0, 2, 1, 3), z(64), z(64), 8, 1e-5, False)
    with pytest.raises(ValueError, match="groupnorm: x0"):
        ops.groupnorm(z(2, 64, 4, 4).permute(0, 2, 3, 1), z(64), z(64), 8, 1e-5, False)
    with pytest.raises(ValueError, match="groupnorm: x1"):
        ops.groupnorm(x, z(128), z(128), 8, 1e-5, False, x1=z(1, 4, 4, 64))
    with pytest.raises(ValueError, match="groupnorm: x1"):
        ops.groupnorm(x, z(128), z(128), 8, 1e-5, False, x1=z(2, 8, 4, 64)[:, ::2])
    with pytest.raises(ValueError, match="conv_out: x"):
        ops.conv_out(z(1, 4, 4, 128)[..., :64], z(4, 3, 3, 64), None)
    with pytest.raises(ValueError, match="upsample2x: x"):
        ops.upsample2x(z(1, 4, 8, 64)[:, :, ::2])
    with pytest.raises(ValueError, match="cfg_ddim: eps2"):
        ops.cfg_ddim(z(2, 4, 8, 8, dt=torch.float32).transpose(2, 3), 7.5)
    with pytest.raises(ValueError, match="cfg_ddim: eps2"):
        ops.cfg_ddim(z(3, 4, 8, 8, dt=torch.float32), 7.5)
    with pytest.raises(ValueError, match="cfg_ddim: x"):
        ops.cfg_ddim(z(2, 4, 8, 8, dt=torch.float32), 7.5, z(1, 4, 8, 8, dt=torch.float32).transpose(2, 3))
    with pytest.raises(ValueError, match="cfg_ddim: x"):
        ops.cfg_ddim(z(2, 4, 8, 8, dt=torch.float32), 7.5, z(2, 4, 8, 8, dt=torch.float32))
    with pytest.raises(ValueError, match="cfg_ddim: x"):
        ops.cfg_ddim(z(1, 4, 8, 8, dt=torch.float32), 0.0, z(2, 4, 8, 8, dt=torch.float32), single=True)


def test_forward_wrappers_accept_the_layouts_the_unet_passes():
    """The same checks pass the call forms of unet.py; a CPU tensor then stops at the CUDA requirement."""
    from sliders_b200 import _cabi, ops

    z = lambda *s, dt=BF: torch.zeros(*s, dtype=dt)  # noqa: E731
    qkv = z(2 * 64, 3 * 80)
    kv = z(2 * 77, 2 * 80)
    calls = [
        lambda: ops.attention(qkv[:, :80], qkv[:, 80:160], qkv[:, 160:], 2, 2, 64, 64, 0.125, 40,
                              lse=z(2, 2, 64, dt=torch.float32)),
        lambda: ops.attention(z(128, 80), kv[:, :80], kv[:, 80:], 2, 2, 64, 77, 0.125, 40),
        lambda: ops.attention(z(1, 80), kv[:77, :80], kv[:77, 80:], 1, 2, 1, 77, 0.125, 40),
        lambda: ops.layernorm(z(16, 96)[:, 8:72], z(64), z(64)),
        lambda: ops.groupnorm(z(2 * 16, 96)[:, 8:72].view(2, 4, 4, 64), z(128), z(128), 8, 1e-5, True,
                              x1=z(2, 4, 4, 64)),
        lambda: ops.groupnorm(z(1, 1, 4, 64)[:, :, :, :], z(64), z(64), 8, 1e-5, True),
        lambda: ops.small_linear(z(4, 72)[:, 8:], z(8, 64), resid=z(4, 8)),
        lambda: ops.conv_out(z(1, 4, 4, 64), z(4, 3, 3, 64), None),
        lambda: ops.upsample2x(z(1, 4, 4, 64)),
        lambda: ops.cfg_ddim(z(2, 4, 8, 8, dt=torch.float32), 7.5, z(1, 4, 8, 8, dt=torch.float32), 0.3, 0.5),
        lambda: ops.cfg_ddim(z(1, 4, 8, 8, dt=torch.float32), 0.0, z(1, 4, 8, 8, dt=torch.float32), single=True),
    ]
    for call in calls:
        with pytest.raises(_cabi.Sb200Error, match="CUDA tensors"):
            call()


# ------------------------------------------------------------------------------------------------------------------
# the GPU variant tables cover every variant, and each row's label is what the host code launches
# ------------------------------------------------------------------------------------------------------------------
def test_attention_fwd_matrix_is_complete():
    cells, kv_tails, ds = set(), set(), set()
    for B, heads, Sq, Skv, d, layout, nd, kv in ATTN_FWD_MATRIX:
        assert attn_nd(d) == nd and attn_fwd_kv(d) == kv and d % 8 == 0 and (layout != "qkv" or Sq == Skv)
        cells.add((nd, kv))
        kv_tails.add((kv, Skv % kv))
        ds.add(d)
        if Skv == 77:
            kv_tails.add((kv, 77))
    assert cells == {(1, 128), (2, 64), (3, 64)}
    assert {8, 64, 72, 128, 136, 192, 40, 80, 160} <= ds
    assert {nd for nd in (1, 2, 3) if any(d % 16 == 8 and attn_nd(d) == nd for d in ds)} == {1, 2, 3}
    assert all(attn_ksteps(d) == (d + 15) // 16 for d in ds)
    assert {(128, 0), (128, 1), (64, 0), (64, 1), (128, 77), (64, 77)} <= kv_tails
    assert {1, 64, 65} <= {row[2] % 128 for row in ATTN_FWD_MATRIX}
    assert any(B >= 2 and Sq % 128 for B, _, Sq, *_ in ATTN_FWD_MATRIX)
    assert sum(1 for _, h, _, _, d, _, nd, _ in ATTN_FWD_MATRIX if h >= 2 and d < 64 * nd) >= 5
    assert (1, 10, 4096, 4096, 64) in {row[:5] for row in ATTN_FWD_MATRIX}
    assert {row[5] for row in ATTN_FWD_MATRIX} == {"qkv", "kv"}


def test_norm_fwd_matrices_are_complete():
    cells = set()
    for M, C, offset, nv, wraps in LN_FWD_MATRIX:
        assert ln_nv(C) == nv
        for sms in SMS:
            assert ln_wraps(M, sms) == wraps, (M, sms)
        cells.add((nv, wraps))
    assert {nv for nv, _ in cells} == {1, 3, 5, 8} and {(3, True), (8, True)} <= cells
    assert {256, 264, 768, 776, 1280, 1288, 2048} <= {row[1] for row in LN_FWD_MATRIX}
    assert any(row[2] >= 8 for row in LN_FWD_MATRIX)
    cells = set()
    for B, H, W, C0, C1, groups, silu, eps, offset, rows_par, one_chunk in GN_FWD_MATRIX:
        C = C0 + C1
        assert gn_smem_ok(C) and C % groups == 0
        for sms in SMS:
            rp, chunks, _ = gn_launch(B, H * W, C, sms)
            assert rp == rows_par and (chunks == 1) == one_chunk, (B, H, W, C, sms)
        cells.add((rows_par, one_chunk))
    assert {12, 6, 2, 1} <= {rp for rp, _ in cells} and (1, True) in cells and (12, True) in cells
    assert {(row[6], row[7]) for row in GN_FWD_MATRIX} >= {(True, 1e-5), (False, 1e-6)}
    # a two-source row whose groups straddle 8-channel vectors and the x0 / x1 boundary (cpg = 60)
    assert any(C1 and (C0 + C1) // g % 8 and C0 % ((C0 + C1) // g) for _, _, _, C0, C1, g, *_ in GN_FWD_MATRIX)
    assert any(row[3] + row[4] > 4096 for row in GN_FWD_MATRIX) and any(row[8] >= 8 for row in GN_FWD_MATRIX)


def test_small_linear_matrix_is_complete():
    def spans(N, group_n):
        return any((8 * b) // group_n != min(8 * b + 7, N - 1) // group_n for b in range((N + 7) // 8))

    rows = SL_MATRIX
    assert {1, 7, 8, 9, 64} <= {row[0] for row in rows} and max(row[0] for row in rows) <= 64
    assert 1280 in {row[1] for row in rows} and any(row[1] % 8 for row in rows)
    assert {8, 320, 1280, 2816} <= {row[2] for row in rows} and any(row[3] for row in rows)
    loras = [row[6] for row in rows if row[6]]
    assert {lo[0] for lo in loras} == {1, 4, 8}
    assert any(lo[1] == row[1] for row in rows if (lo := row[6])) and any(spans(row[1], row[6][1])
                                                                             for row in rows if row[6])
    assert any(row[4] for row in rows)
    assert {row[5] for row in rows if row[7]} == {0, 1, 2}


def test_elementwise_matrices_are_complete():
    for sms in SMS:
        assert {w for *_, w in CONV_IN_MATRIX} == {True, False}
        for B, H, W, Cout, _, wraps in CONV_IN_MATRIX:
            assert conv_in_wraps(B, H, W, Cout, sms) == wraps and Cout * 72 <= 48 * 1024
        for B, H, W, Cin, _, _, wraps in CONV_OUT_MATRIX:
            assert conv_out_wraps(B, H, W, sms) == wraps and Cin * 72 <= 48 * 1024
        for B, H, W, C, wraps in UPSAMPLE_MATRIX:
            assert upsample_wraps(B, H, W, C, sms) == wraps
        for *_, shape, wraps in CFG_MATRIX:
            assert cfg_wraps(math.prod(shape), sms) == wraps
    assert {row[4] for row in CONV_IN_MATRIX} == {torch.float32, BF} and {320, 680} <= {r[3] for r in CONV_IN_MATRIX}
    assert any(H % 2 and W % 2 for _, H, W, *_ in CONV_IN_MATRIX) and any(H != W for _, H, W, *_ in CONV_IN_MATRIX)
    assert {8, 264, 320, 680} <= {row[3] for row in CONV_OUT_MATRIX}
    assert {(row[4], row[5]) for row in CONV_OUT_MATRIX} >= {(torch.float32, True), (BF, False)}
    assert {w for *_, w in CONV_OUT_MATRIX} == {True, False}
    assert 8 in {row[3] for row in UPSAMPLE_MATRIX} and any(H % 2 and W % 2 for _, H, W, *_ in UPSAMPLE_MATRIX)
    assert {w for *_, w in UPSAMPLE_MATRIX} == {True, False}
    assert {(te, to) for te, to, *_ in CFG_MATRIX} == {(a, b) for a in (torch.float32, BF) for b in (torch.float32, BF)}
    assert {row[2] for row in CFG_MATRIX} == {0.0, 1.0, 7.5}
    assert {row[3] for row in CFG_MATRIX} == {"ddim", "affine", "single", "eps"}
    assert all(row[2] == 0.0 for row in CFG_MATRIX if row[3] == "single")
    assert any(math.prod(row[4]) % 256 for row in CFG_MATRIX) and any(row[5] for row in CFG_MATRIX)
