"""Host-side checks of the backward-kernel test machinery in test_gpu_backward_bounds.py: each per-element bound
accepts a CPU emulation of its kernel's roundings and rejects the local errors a backward kernel can make (which
rel-RMS over the whole output does not), and the variant tables cover every launch variant of the host code."""
import torch

from test_gpu_backward_bounds import (ATTN_MATRIX, BF, CONV_MATRIX, GEGLU_MATRIX, GN_MATRIX, LN_MATRIX, SPLIT_MATRIX,
                                      WGRAD_MATRIX, attention_bwd_ref, attn_kt, attn_nd, attn_split, attn_violations,
                                      gn_chain, gn_launch, gn_smem_ok, geglu_bwd_ref, groupnorm_bwd_ref, layernorm_bwd_ref,
                                      ln_chain, ln_nv, ln_wraps, norm_violations, pointwise_violations,
                                      reduction_violations, split_cols, wgrad_chain, wgrad_launch)
from test_gpu_kernels import rel_rms

SMS = (114, 132)  # H100 PCIe .. SXM


def _plant_vector(out, row, vec):
    """One 8-channel vector of one row replaced by the next row's (a wrong row / lane map)."""
    bad = out.clone()
    bad[row, 8 * vec:8 * vec + 8] = out[row + 1, 8 * vec:8 * vec + 8]
    return bad


def _assert_rejects_only(v, where):
    assert v[where].all() and int(v.sum()) == int(v[where].numel()), int(v.sum())


def test_layernorm_bwd_bound():
    g = torch.Generator().manual_seed(0)
    M, C = 512, 1288
    x = (torch.randn(M, C, generator=g) * 2 + 0.5).to(BF)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(BF)
    dy = torch.randn(M, C, generator=g).to(BF)
    add = torch.randn(M, C, generator=g).to(BF)
    ref, mag, stat = layernorm_bwd_ref(x, gamma, dy, add)
    # the kernel: fp32 statistics and output expression, one bf16 store
    xf = x.float()
    mean = xf.mean(1, keepdim=True)
    rstd = torch.rsqrt(((xf - mean) ** 2).mean(1, keepdim=True) + 1e-5)
    xh = (xf - mean) * rstd
    dg = dy.float() * gamma.float()
    out = (rstd * (dg - dg.mean(1, keepdim=True) - xh * (dg * xh).mean(1, keepdim=True)) + add.float()).to(BF)
    a = add.double()
    assert not norm_violations(out, ref, a, mag, stat, ln_chain(C)).any()
    bad = _plant_vector(out, 100, 31)  # lane 31's vector at k = 0
    v = norm_violations(bad, ref, a, mag, stat, ln_chain(C))
    _assert_rejects_only(v, (100, slice(8 * 31, 8 * 32)))
    assert rel_rms(bad, ref) < 1e-2
    bad = out.clone()
    bad[3, 5] = float("nan")
    assert norm_violations(bad, ref, a, mag, stat, ln_chain(C))[3, 5]


def test_groupnorm_bwd_bound():
    g = torch.Generator().manual_seed(1)
    B, HW, C, groups = 2, 256, 640, 32
    x = (torch.randn(B, HW, C, generator=g) * 1.5 + 0.3).to(BF)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(BF)
    beta = (0.2 * torch.randn(C, generator=g)).to(BF)
    dy = torch.randn(B, HW, C, generator=g).to(BF)
    add = torch.randn(B, HW, C, generator=g).to(BF)
    ref, mag, stat = groupnorm_bwd_ref(x, gamma, beta, dy, add, groups, True)
    # the kernel: forward statistics as E[x^2] - mean^2 in fp32, fp32 backward, one bf16 store
    cpg = C // groups
    xf = x.float().view(B, HW, groups, cpg)
    mean = xf.mean((1, 3), keepdim=True)
    rstd = torch.rsqrt(torch.clamp((xf * xf).mean((1, 3), keepdim=True) - mean * mean, min=0) + 1e-5)
    gm, bt = gamma.float().view(groups, cpg), beta.float().view(groups, cpg)
    xh = (xf - mean) * rstd
    z = gm * xh + bt
    s = torch.sigmoid(z)
    dg = dy.float().view(B, HW, groups, cpg) * s * (1 + z * (1 - s)) * gm
    o = rstd * (dg - dg.mean((1, 3), keepdim=True) - xh * (dg * xh).mean((1, 3), keepdim=True))
    out = (o.view(B, HW, C) + add.float()).to(BF)
    a = add.double()
    chain = gn_chain(B, HW, C, groups, 132)
    assert not norm_violations(out, ref, a, mag, stat, chain).any()
    flat = out.view(B * HW, C)
    bad = _plant_vector(flat, 300, 17).view(B, HW, C)
    v = norm_violations(bad, ref, a, mag, stat, chain).view(B * HW, C)
    _assert_rejects_only(v, (300, slice(8 * 17, 8 * 18)))
    assert rel_rms(bad, ref) < 1e-2
    # statistics of the wrong group (off by one group) for one vector
    bad = out.clone()
    bad[1, 7, 40:48] = (o.view(B, HW, C)[1, 7, 60:68] + add.float()[1, 7, 40:48]).to(BF)
    assert norm_violations(bad, ref, a, mag, stat, chain)[1, 7, 40:48].any()


def test_geglu_bwd_bound():
    g = torch.Generator().manual_seed(2)
    M, Fh = 300, 1280
    pre = (torch.randn(M, 2 * Fh, generator=g) * 2.5).to(BF)
    dout = torch.randn(M, Fh, generator=g).to(BF)
    ref, mag = geglu_bwd_ref(pre, dout)
    a, gt = pre.float().chunk(2, dim=-1)
    cdf = 0.5 * (1 + torch.erf(gt * 0.7071067811865475))
    pdf = 0.3989422804014327 * torch.exp(-0.5 * gt * gt)
    out = torch.cat([dout.float() * gt * cdf, dout.float() * a * (cdf + gt * pdf)], -1).to(BF)
    assert not pointwise_violations(out, ref, mag, 2.0 ** -16).any()
    bad = _plant_vector(out, 10, Fh // 8 + 3)   # a vector of the gate half
    v = pointwise_violations(bad, ref, mag, 2.0 ** -16)
    assert v[10, Fh + 24:Fh + 32].all() and int(v.sum()) == int(v[10].sum())
    assert rel_rms(bad, ref) < 1e-2
    bad = out.clone()
    bad[0, 0] = float("nan")
    assert pointwise_violations(bad, ref, mag, 2.0 ** -16)[0, 0]


def _attn_emulation(q, k, v, o, dout, scale):
    """One head: fp32 S / dP, P and dS rounded to bf16 before the second products, fp32 accumulation."""
    qf, kf, vf, of, gf = (t.float() for t in (q, k, v, o, dout))
    P = torch.softmax(qf @ kf.t() * scale, -1)
    D = (gf * of).sum(1, keepdim=True)
    dS = (P * (gf @ vf.t() - D) * scale).to(BF).float()
    Pb = P.to(BF).float()
    return dS @ kf, dS.t() @ qf, Pb.t() @ gf, dS, Pb


def test_attention_bwd_bound_and_planted_tiles():
    g = torch.Generator().manual_seed(3)
    Sq, Skv, d = 768, 512, 64
    q, k, v, dout = (torch.randn(S, d, generator=g).to(BF) for S in (Sq, Skv, Skv, Sq))
    scale = d ** -0.5
    o = (torch.softmax(q.double() @ k.double().t() * scale, -1) @ v.double()).to(BF)
    dq, mq, dk, mk, dv, mv = attention_bwd_ref(q, k, v, o, dout, 1, 1, Sq, Skv, d, scale)
    eq, ek, ev, dS, Pb = _attn_emulation(q, k, v, o, dout, scale)
    for got, ref, mag in ((eq, dq, mq), (ek, dk, mk), (ev, dv, mv)):
        assert not attn_violations(got.to(BF), ref, mag).any()
    # one 64-key tile missing from one query row of dQ
    row, t = 77, 2
    bad = eq.clone()
    bad[row] -= dS[row, 64 * t:64 * (t + 1)] @ k.float()[64 * t:64 * (t + 1)]
    v_ = attn_violations(bad.to(BF), dq, mq)
    assert v_[row].any() and int(v_.sum()) == int(v_[row].sum())
    assert rel_rms(bad.to(BF), dq) < 3e-2
    # one 64-query split missing from the dV and dK partial sums of one key row (the row where it weighs most)
    qs = slice(64 * 5, 64 * 6)
    miss_v = Pb[qs].t() @ dout.float()[qs]
    miss_k = dS[qs].t() @ q.float()[qs]
    for est, miss, ref, mag in ((ev, miss_v, dv, mv), (ek, miss_k, dk, mk)):
        row = int((miss.abs().sum(1) / mag.sum(1)).argmax())
        bad = est.clone()
        bad[row] -= miss[row]
        v_ = attn_violations(bad.to(BF), ref, mag)
        assert v_[row].any() and int(v_.sum()) == int(v_[row].sum())
    bad = eq.to(BF)
    bad[1, 1] = float("nan")
    assert attn_violations(bad, dq, mq)[1, 1]


def _wgrad_emulation(A, T, rows_per_chunk):
    """lora_wgrad: fp32 per-chunk partials (4 row lanes each), chunks summed in order in fp32."""
    Af, Tf = A.float(), T.float()
    total = torch.zeros(A.shape[1], T.shape[1])
    parts = []
    for r0 in range(0, A.shape[0], rows_per_chunk):
        p = Af[r0:r0 + rows_per_chunk].t() @ Tf[r0:r0 + rows_per_chunk]
        parts.append(p)
        total = total + p
    return total, parts


def test_lora_wgrad_bound_and_missing_chunk():
    g = torch.Generator().manual_seed(4)
    M, C, r = 4096, 640, 8
    A = torch.randn(M, C, generator=g).to(BF)
    T = torch.randn(M, r, generator=g)
    _, chunks, rpb = wgrad_launch(M, C)
    assert chunks > 1
    out, parts = _wgrad_emulation(A, T, rpb)
    ref, mag = A.double().t() @ T.double(), A.double().abs().t() @ T.double().abs()
    chain = wgrad_chain(M, C)
    assert not reduction_violations(out, ref, mag, chain).any()
    bad = out.clone()
    bad[:, 3] -= parts[chunks // 2][:, 3]   # one column misses one row chunk
    v = reduction_violations(bad, ref, mag, chain)
    assert v[:, 3].float().mean() > 0.9 and not v[:, :3].any() and not v[:, 4:].any()
    assert rel_rms(bad, ref) < 1e-1
    bad = out.clone()
    bad[C - 1, r - 1] = float("nan")
    assert reduction_violations(bad, ref, mag, chain)[C - 1, r - 1]


def test_lora_conv_wgrad_bound_and_missing_tap():
    g = torch.Generator().manual_seed(5)
    B, H, W, C, r, stride = 2, 32, 32, 128, 4, 1
    x = torch.randn(B, C, H, W, generator=g).to(BF)
    Ug = torch.randn(B, r, H, W, generator=g)
    wg = torch.nn.grad.conv2d_weight
    ref = wg(x.double(), (r, C, 3, 3), Ug.double(), padding=1)
    mag = wg(x.double().abs(), (r, C, 3, 3), Ug.double().abs(), padding=1)
    out = wg(x.float(), (r, C, 3, 3), Ug.float(), padding=1)
    chain = wgrad_chain(B * H * W, C, 9)
    assert not reduction_violations(out, ref, mag, chain).any()
    # output pixel (b, y, x) misses its tap (a, bb): a wrong padding test drops that product from G[:, :, a, bb]
    b, y, xo, a, bb = 1, 5, 9, 2, 0
    bad = out.clone()
    bad[:, :, a, bb] -= torch.outer(Ug[b, :, y, xo], x.float()[b, :, y + a - 1, xo + bb - 1])
    v = reduction_violations(bad, ref, mag, chain)
    assert v[:, :, a, bb].float().mean() > 0.5 and int(v.sum()) == int(v[:, :, a, bb].sum())
    assert rel_rms(bad, ref) < 1e-2


# ------------------------------------------------------------------------------------------------------------------
# the GPU variant tables cover every variant, and each row's label is what the host code launches
# ------------------------------------------------------------------------------------------------------------------
def test_layernorm_matrix_is_complete():
    cells = set()
    for M, C, _, nv, wraps in LN_MATRIX:
        assert ln_nv(C) == nv
        for sms in SMS:
            assert ln_wraps(M, sms) == wraps, (M, sms)
        cells.add((nv, wraps))
    assert {nv for nv, _ in cells} == {1, 3, 5, 8} and any(w for _, w in cells)
    Cs, Ms = {row[1] for row in LN_MATRIX}, {row[0] for row in LN_MATRIX}
    assert {256, 264, 768, 776, 1280, 1288, 2048} <= Cs and {1, 7} <= Ms and max(Ms) >= 20000


def test_groupnorm_matrix_is_complete():
    cells = set()
    for B, H, W, C0, C1, groups, _, _, rows_par, one_chunk in GN_MATRIX:
        C = C0 + C1
        assert gn_smem_ok(C) and C % groups == 0
        for sms in SMS:
            rp, chunks, _ = gn_launch(B, H * W, C, sms)
            assert rp == rows_par and (chunks == 1) == one_chunk, (B, H, W, C, sms)
        cells.add((rows_par == 1, one_chunk))
    assert cells == {(False, False), (False, True), (True, False), (True, True)}
    assert any(row[4] for row in GN_MATRIX)  # a two-source (concat) input
    assert max(r[3] + r[4] for r in GN_MATRIX) > 5000 and gn_smem_ok(6144) and not gn_smem_ok(6152)
    assert all(gn_smem_ok(C) for C in range(8, 6145, 8))


def test_attention_matrices_are_complete():
    ds = {row[4] for row in ATTN_MATRIX}
    assert {8, 24, 40, 64, 72, 128, 136, 160, 192} <= ds
    assert {(attn_nd(d), attn_kt(d)) for d in ds} == {(1, 64), (2, 64), (3, 32)}
    assert any(Sq % 64 and Skv % 64 for _, _, Sq, Skv, _, _ in ATTN_MATRIX)
    assert {cross for *_, cross in ATTN_MATRIX} == {False, True}
    cells = set()
    for B, heads, Sq, Skv, d, nsplit in SPLIT_MATRIX:
        n, per = attn_split(B, heads, Sq, Skv)
        assert n == nsplit
        if n > 1:
            assert per % 64 == 0 and (n - 1) * per < Sq <= n * per
            cells.add(("split", Sq % per != 0, Sq % 64 != 0, Skv <= 64, Skv == 128, B * heads == 66, attn_nd(d)))
        else:
            cells.add(("unsplit", Skv > 128, B * heads == 67))
    split = [c for c in cells if c[0] == "split"]
    assert any(c[1] for c in split) and any(c[2] for c in split) and any(c[3] for c in split)
    assert any(c[4] for c in split) and any(c[5] for c in split) and {c[6] for c in split} >= {1, 2, 3}
    assert ("unsplit", True, False) in cells and ("unsplit", False, True) in cells


def test_lora_matrices_are_complete():
    cells = set()
    for M, C, r, sources, pad, acc in WGRAD_MATRIX:
        for w in split_cols(C, sources):
            assert w % 8 == 0
            cblocks, chunks, _ = wgrad_launch(M, w)
            cells.add((chunks == 1, (w // 8) % 32 != 0))
        assert (wgrad_launch(M, split_cols(C, sources)[0])[1] == 1) == (M < 32)
    assert cells == {(True, True), (True, False), (False, True), (False, False)}
    assert {r for _, _, r, *_ in WGRAD_MATRIX} == {4, 8} and {s for _, _, _, s, *_ in WGRAD_MATRIX} == {1, 2}
    assert {1, 7} <= {M for M, *_ in WGRAD_MATRIX} and {True, False} == {row[-1] for row in WGRAD_MATRIX}
    conv = {(stride, H != W, C1 > 0, r, acc) for _, H, W, _, C1, stride, r, acc in CONV_MATRIX}
    assert {c[0] for c in conv} == {1, 2} and any(c[0] == 2 and c[1] for c in conv)
    assert any(c[2] for c in conv) and {c[3] for c in conv} == {4, 8} and {c[4] for c in conv} == {True, False}
    assert all(F % 8 == 0 for _, F in GEGLU_MATRIX) and 1 in {M for M, _ in GEGLU_MATRIX}
