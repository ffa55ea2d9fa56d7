"""Host-side checks of the split-K GEMM, guided-step loss, AdamW and fp32 Adam test machinery in
test_gpu_inversion_optim_bounds.py: each bound accepts a CPU emulation of its kernel's roundings and rejects the local
errors these kernels can make (which rel-RMS over the whole output does not), the exact-data regimes really are exact,
and the variant tables cover every launch variant of the host code.  Also the coverage guard: every kernel entry point
of include/sb200.h is named here with the test(s) that check it element by element or bit for bit."""
import ast
import math
import os
import re

import torch

from test_gpu_inversion_optim_bounds import (ADAM_STEPS, ADAM_WDS, ADAMW_MATRIX, BF, KV_K, LOSS_MATRIX, LOSS_PARAMS,
                                             SPLITK_MATRIX, adam_f32_ref, adam_f32_violations, adam_grid, adam_sizes,
                                             adamw_bx, adamw_emulation, adamw_table_shapes, chain_c, f32,
                                             guided_grad_violations, guided_loss_violation, guided_ref,
                                             loss_exact_inputs, loss_exact_sum, loss_mode1_blocks, loss_parts,
                                             splitk_bn, splitk_exact_inputs,
                                             splitk_kb, splitk_kb_unclamped, splitk_out_chain, splitk_ranges,
                                             splitk_reduce, splitk_split_chain, splitk_split_refs, splitk_splits)
from test_gpu_backward_bounds import _outside
from test_gpu_kernels import rel_rms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS = (114, 132)  # H100 PCIe .. SXM
F32 = torch.float32


# ------------------------------------------------------------------------------------------------------------------
# split-K GEMM
# ------------------------------------------------------------------------------------------------------------------
def _splitk_emulation(x, w, ranges):
    """Each split tile accumulated in fp32 one k16 step at a time (the 16 products of a step summed exactly, one
    rounding per step)."""
    ws = []
    for k0, k1 in ranges:
        acc = torch.zeros(x.shape[0], w.shape[0], dtype=F32)
        for k in range(k0, k1, 16):
            acc = (acc.double() + x[:, k:k + 16].double() @ w[:, k:k + 16].double().t()).float()
        ws.append(acc)
    return torch.stack(ws)


def test_splitk_bound_accepts_emulation_and_rejects_planted_errors():
    M, N, K = 127, 80, 4096
    assert (splitk_bn(N), splitk_kb(M, N, K), splitk_splits(M, N, K)) == (64, 8, 8)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(M, K, generator=g).to(BF)
    w = (torch.randn(N, K, generator=g) * 0.05).to(BF)
    ranges = splitk_ranges(M, N, K)
    ws = _splitk_emulation(x, w, ranges)
    refs = splitk_split_refs(x, w, ranges)
    for s, (ref, mag) in enumerate(refs):
        assert not _outside((ws[s].double() - ref).abs(), chain_c(splitk_split_chain(*ranges[s])) * mag, "t").any()
    out = splitk_reduce(ws)
    full, fmag = x.double() @ w.double().t(), x.double().abs() @ w.double().abs().t()
    assert not _outside((out.double() - full).abs(), chain_c(splitk_out_chain(M, N, K)) * fmag, "t").any()

    # one element of split 3 misses one of its 8 k-blocks
    s, m, n, kb0 = 3, 100, 70, ranges[3][0] + 5 * 64
    bad = ws[s].clone()
    bad[m, n] -= float(x[m, kb0:kb0 + 64].double() @ w[n, kb0:kb0 + 64].double())
    ref, mag = refs[s]
    v = _outside((bad.double() - ref).abs(), chain_c(splitk_split_chain(*ranges[s])) * mag, "t")
    assert v[m, n] and int(v.sum()) == 1
    # the same error in a 616 x 2048 output at the SD1.x K is below what rel-RMS (test_gpu_inversion's 1e-4) can see
    x2 = torch.randn(616, 24960, generator=g).to(BF).float()
    w2 = (torch.randn(2048, 24960, generator=g) * 0.05).to(BF).float()
    out2 = x2 @ w2.t()
    bad2 = out2.clone()
    bad2[m, n] -= float(x2[m, 64:128] @ w2[n, 64:128])
    assert rel_rms(bad2, out2) < 1e-4

    # the splits summed in another order: rel-RMS cannot tell, the bit-for-bit comparison with the in-order sum can
    order = [0, 2, 1] + list(range(3, ws.shape[0]))
    swapped = splitk_reduce(ws[order])
    assert not torch.equal(swapped.view(torch.int32), out.view(torch.int32))
    assert rel_rms(swapped, full) < 1e-6

    # the 16-wide second column tile (bn = 64) stored 16 columns to the left: every element of it is outside the bound
    bad = out.clone()
    bad[:, 64:80] = out[:, 48:64]
    v = _outside((bad.double() - full).abs(), chain_c(splitk_out_chain(M, N, K)) * fmag, "t")
    assert v[:, 64:80].all() and int(v.sum()) == M * 16


# ------------------------------------------------------------------------------------------------------------------
# guided-step loss
# ------------------------------------------------------------------------------------------------------------------
def _guided_emulation(eu, ec, g, x, cx, ce, t, n, dloss):
    """guided_loss_kernel in fp32: the residual, each thread's strided FMA chain over a grid of loss_parts(n) blocks of
    256 threads, the block tree, the finalize tree over the partials and the division; and mode 1's d_eps_u.
    Returns (loss, partials, d_eps_u)."""
    e = eu + g * (ec - eu)
    r = cx * x + ce * e - t
    stride = loss_parts(n) * 256
    it = -(-n // stride)
    sq = torch.zeros(it * stride, dtype=torch.float64)
    sq[:n] = r.double() ** 2
    acc = torch.zeros(stride, dtype=F32)
    for k in range(it):
        acc = (acc.double() + sq[k * stride:(k + 1) * stride]).float()
    red = acc.view(-1, 256)
    for wd in (128, 64, 32, 16, 8, 4, 2, 1):
        red = torch.cat([red[:, :wd] + red[:, wd:2 * wd], red[:, 2 * wd:]], 1)
    parts = red[:, 0].clone()
    fin = torch.zeros(256, dtype=F32)
    fin[:parts.numel()] = parts
    for wd in (128, 64, 32, 16, 8, 4, 2, 1):
        fin = torch.cat([fin[:wd] + fin[wd:2 * wd], fin[2 * wd:]])
    k = torch.tensor(dloss, dtype=F32) * (1 - torch.tensor(g, dtype=F32)) * ce * 2 / torch.tensor(float(n), dtype=F32)
    return fin[0] / torch.tensor(float(n), dtype=F32), parts, k * r


def test_guided_loss_bounds_accept_emulation_and_reject_a_dropped_partial():
    for n in (65536, 600001):
        gen = torch.Generator().manual_seed(n)
        eu, ec, x, t = (torch.randn(n, generator=gen) for _ in range(4))
        g, cx, ce, dl = f32(7.5), f32(1.0137), f32(-0.0421), f32(2.5)
        loss, parts, d = _guided_emulation(eu, ec, g, x, cx, ce, t, n, dl)
        r, mag, k = guided_ref(eu, ec, g, x, cx, ce, t, dl)
        assert not guided_loss_violation(loss.item(), r, mag, n)
        assert not guided_grad_violations(d, r, mag, k).any()
        # the finalize kernel reading one partial fewer (or a block's partial dropped)
        for drop in (0, parts.numel() - 1):
            short = torch.cat([parts[:drop], parts[drop + 1:]]).double().sum() / n
            assert guided_loss_violation(float(short), r, mag, n), (n, drop)
        # one element of d_eps_u taking its neighbour's residual
        bad = d.clone()
        bad[n // 2] = d[n // 2 + 1]
        v = guided_grad_violations(bad, r, mag, k)
        assert v[n // 2] and int(v.sum()) == 1 and rel_rms(bad, k * r) < 1e-2


# ------------------------------------------------------------------------------------------------------------------
# fp32 Adam and bf16 AdamW
# ------------------------------------------------------------------------------------------------------------------
def _adam_f32_emulation(p, g, m, v, lr, b1, b2, eps, wd, step):
    """adam_f32_kernel in fp32 with the host's fp32 scalars."""
    one_m_b1, b2f, one_m_b2 = f32(1 - b1), f32(b2), f32(1 - b2)
    nss, bc2 = f32(-lr / (1 - b1 ** step)), f32(math.sqrt(1 - b2 ** step))
    gg = g + f32(wd) * p
    m1 = m + one_m_b1 * (gg - m)
    v1 = v * b2f + one_m_b2 * gg * gg
    denom = v1.sqrt() / bc2 + f32(eps)
    return p + nss * (m1 / denom), m1, v1


def test_adam_f32_bound_accepts_emulation_and_rejects_a_skipped_element():
    n = 1 << 20
    gen = torch.Generator().manual_seed(7)
    p, g = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 0.3
    m, v = torch.randn(n, generator=gen) * 0.1, (torch.randn(n, generator=gen) * 0.1).square()
    lr, b1, b2, eps = 1e-2 * 0.97, 0.9, 0.999, 1e-8
    for step in ADAM_STEPS:
        for wd in ADAM_WDS:
            ref = adam_f32_ref(p, g, m, v, lr, b1, b2, eps, wd, step)
            p1, m1, v1 = _adam_f32_emulation(p, g, m, v, lr, b1, b2, eps, wd, step)
            assert not any(bad.any() for bad in adam_f32_violations(p1, m1, v1, ref)), (step, wd)
    # g' = g + wd p cancels and v is tiny: v' is far below its magnitude, so the rounding of wd p is a large relative
    # error of v', sqrt(v'), denom and the step.  The bound must accept the kernel's arithmetic there; a bound without
    # the error of denom would not.
    wd, step = 0.1, 1000
    pc = torch.randn(n, generator=gen) + 1.5
    gc = (-f32(wd) * pc).double() + torch.randn(n, generator=gen).double() * 1e-3
    gc, vc = gc.float(), torch.rand(n, generator=gen) * 1e-10
    ref_c = adam_f32_ref(pc, gc, m, vc, lr, b1, b2, eps, wd, step)
    emu_c = _adam_f32_emulation(pc, gc, m, vc, lr, b1, b2, eps, wd, step)
    assert not any(bad.any() for bad in adam_f32_violations(*emu_c, ref_c))
    ss = lr / (1 - b1 ** step)
    mag_m = m.double().abs() + (1 - b1) * (gc.double().abs() + wd * pc.double().abs() + m.double().abs())
    denom = ref_c[2].sqrt() / math.sqrt(1 - b2 ** step) + eps
    without_denom = chain_c(20) * (pc.double().abs() + ss * mag_m / denom)
    assert bool(((emu_c[0].double() - ref_c[0]).abs() > without_denom).any())
    # one element of the table not updated (a grid-stride loop that stops one short)
    bad = p1.clone()
    bad[n - 1] = p[n - 1]
    vp = adam_f32_violations(bad, m1, v1, ref)[0]
    assert vp[n - 1] and int(vp.sum()) == 1 and rel_rms(bad, ref[0]) < 1e-4


def test_adamw_emulation_is_torchs_arithmetic():
    """adamw_emulation in the order of torch's CPU kernels equals torch.optim.AdamW on bf16 CPU tensors bit for bit, on
    both branches of lerp (beta1 = 0.9; 0.5 and 0.3).  Its CUDA order is checked against the kernel, which matches
    torch.optim.AdamW, in test_gpu_inversion_optim_bounds.test_adamw_guarded_table."""
    n = 1 << 20
    gen = torch.Generator().manual_seed(8)
    p = (torch.randn(n, generator=gen) * 0.1).to(BF)
    g = (torch.randn(n, generator=gen) * 0.1).to(BF)
    m = (torch.randn(n, generator=gen) * 0.01).to(BF)
    v = (torch.randn(n, generator=gen) * 0.01).square().to(BF)
    for b1 in (0.9, 0.5, 0.3):
        a = torch.nn.Parameter(p.clone())
        opt = torch.optim.AdamW([a], lr=1e-3, betas=(b1, 0.999), eps=1e-8, weight_decay=1e-2, foreach=False)
        opt.state[a] = {"step": torch.tensor(2.0), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
        a.grad = g.clone()
        opt.step()
        st = opt.state[a]
        got = adamw_emulation(p, g, m, v, 1e-3, b1, 0.999, 1e-8, 1e-2, 3, order="cpu")
        for want, mine, name in zip((a.detach(), st["exp_avg"], st["exp_avg_sq"]), got, ("p", "exp_avg", "v")):
            assert torch.equal(want.view(torch.int16), mine.view(torch.int16)), (b1, name)


def test_adamw_bitwise_comparison_rejects_an_unrounded_moment():
    """Skipping one bf16 rounding of exp_avg changes a few parameters by one bf16 ulp: rel-RMS over the table stays
    tiny, the bit-for-bit comparison against torch.optim.AdamW catches it."""
    n = 1 << 20
    gen = torch.Generator().manual_seed(8)
    p = (torch.randn(n, generator=gen) * 0.1).to(BF)
    g = (torch.randn(n, generator=gen) * 0.1).to(BF)
    m = (torch.randn(n, generator=gen) * 0.01).to(BF)
    v = (torch.randn(n, generator=gen) * 0.01).square().to(BF)
    args = (1e-3, 0.9, 0.999, 1e-8, 1e-2, 3)
    good = adamw_emulation(p, g, m, v, *args)
    bad = adamw_emulation(p, g, m, v, *args, round_m=False)
    assert torch.equal(good[1], bad[1])   # the stored moment is the same
    diff = int((good[0].view(torch.int16) != bad[0].view(torch.int16)).sum())
    assert diff > 0 and rel_rms(bad[0], good[0].double()) < 1e-3


# ------------------------------------------------------------------------------------------------------------------
# exact-data regimes
# ------------------------------------------------------------------------------------------------------------------
def test_exact_regimes_are_exact():
    # split-K: integers in [-2, 2]; every partial sum of a tile is bounded by 4 K in magnitude
    x, w = splitk_exact_inputs(64, 48, 520, torch.Generator().manual_seed(1), "cpu")
    for t in (x, w):
        assert torch.equal(t.float(), t.float().round()) and int(t.float().abs().max()) == 2
    assert all(4 * K < 2 ** 24 for _, _, K, *_ in SPLITK_MATRIX)
    # every partial sum of the emulated split tiles is the exact float64 value
    ranges = splitk_ranges(64, 48, 520)
    ws = _splitk_emulation(x, w, ranges)
    for s, (ref, _) in enumerate(splitk_split_refs(x, w, ranges)):
        assert torch.equal(ws[s].double(), ref)
    # loss: squares are multiples of 1/4 and non-negative, so every partial sum is at most S; 4 S < 2^24 at the largest
    # n with a wide margin (the GPU test asserts it again for its own data)
    n = max(row[0] for row in LOSS_MATRIX)
    for seed in range(3):
        eu, ec, xx, t = loss_exact_inputs(n, torch.Generator().manual_seed(seed), "cpu")
        S = loss_exact_sum(eu, ec, xx, t)
        assert 4 * S < 2 ** 23 and S == int(4 * S) / 4
        loss, parts, d = _guided_emulation(eu, ec, 0.5, xx, 1.0, 1.0, t, n, 1.0)
        assert float(parts.double().sum()) == S
        assert loss.item() == (torch.tensor(S, dtype=F32) / torch.tensor(float(n), dtype=F32)).item()


# ------------------------------------------------------------------------------------------------------------------
# the GPU variant tables cover every variant, and each row's label is what the host code launches
# ------------------------------------------------------------------------------------------------------------------
def test_kv_plan_widths():
    """KV_K is the K of each UNet's d_ctx GEMM: twice the to_k width summed over its cross-attention blocks."""
    from oracle import unet as ounet
    from sliders_b200.unet import Attention, UNet2DConditionModel, UNetConfig

    for name, K in KV_K.items():
        with torch.device("meta"):
            unet = UNet2DConditionModel(UNetConfig.from_dict(getattr(ounet.UNetConfig, name)().__dict__))
        assert sum(2 * m.to_k.weight.shape[0] for m in unet.modules() if isinstance(m, Attention) and m.is_cross) == K


def test_splitk_matrix_is_complete():
    from sliders_b200 import ops

    cells = set()
    for M, N, K, views, bn, kb, splits in SPLITK_MATRIX:
        assert (splitk_bn(N), splitk_kb(M, N, K), splitk_splits(M, N, K)) == (bn, kb, splits)
        assert ops.splitk_ws_floats(M, N, K) == splits * M * N and K % 8 == 0 and N % 16 == 0
        ranges = splitk_ranges(M, N, K)
        assert ranges[0][0] == 0 and ranges[-1][1] == K and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
        kbs = -(-K // 64)
        cells.add(("splits", "one" if splits == 1 else "short last" if kbs % kb else "even"))
        cells.add(("kb", "clamped" if splitk_kb_unclamped(M, N, K) < 8 and splits > 1 else "wanted", bn))
        cells.add(("narrow tile", N % 64 != 0))
    assert {("splits", c) for c in ("one", "short last", "even")} <= cells
    assert {("kb", "clamped", 64), ("kb", "clamped", 128), ("kb", "wanted", 64), ("kb", "wanted", 128)} <= cells
    assert ("narrow tile", True) in cells
    assert {16, 48, 80, 1040, 128, 256, 768, 2048} <= {r[1] for r in SPLITK_MATRIX}
    assert {1, 77, 127, 128, 129, 154, 616} <= {r[0] for r in SPLITK_MATRIX}
    assert {8, 56} <= {r[2] % 64 for r in SPLITK_MATRIX} and set(KV_K.values()) <= {r[2] for r in SPLITK_MATRIX}
    assert all(any(c in r[3] for r in SPLITK_MATRIX) for c in "xwo") and any(r[3] == "xwo" for r in SPLITK_MATRIX)


def test_loss_matrix_is_complete():
    for n, parts, blocks1, wraps in LOSS_MATRIX:
        assert (loss_parts(n), loss_mode1_blocks(n), n > blocks1 * 256) == (parts, blocks1, wraps)
    ns = {r[0] for r in LOSS_MATRIX}
    assert {1, 255, 257, 2047, 2048, 2049, 65536} <= ns
    assert loss_parts(522239) == 255 and 522240 in ns and any(r[3] for r in LOSS_MATRIX)
    assert any(r[1] == 256 and r[0] % 256 for r in LOSS_MATRIX)
    gs, ces, dls = ({p[i] for p in LOSS_PARAMS} for i in range(3))
    assert {0.0, 1.0, 7.5} <= gs and 0.0 in ces and any(d != 1.0 for d in dls)


def test_optimizer_matrices_are_complete():
    counts = {}
    for table, grads, wd, betas, bx, wraps in ADAMW_MATRIX:
        numels = [math.prod(s) for s in adamw_table_shapes(table)]
        assert adamw_bx(max(numels)) == bx and (max(numels) > bx * 256) == wraps
        counts[table] = len(numels)
    assert counts["sdxl-r4-noxattn"] == 692 and counts["sdxl-r16-noxattn"] == 692
    assert counts["sdxl-r4-full"] == counts["sdxl-r16-full"] > 692
    assert {r[1] for r in ADAMW_MATRIX} == {"bf16", "fp32", "flat"} and {r[2] for r in ADAMW_MATRIX} == {0.0, 1e-2}
    assert any(r[3][0] <= 0.5 for r in ADAMW_MATRIX) and {r[5] for r in ADAMW_MATRIX} == {True, False}
    assert adamw_bx(16385) == 64 and adamw_bx(16384) * 256 == 16384
    for sms in SMS:
        sizes = adam_sizes(sms)
        assert adam_grid(max(sizes), sms) == sms * 16 and max(sizes) > sms * 16 * 256 and min(sizes) == 1
    assert set(ADAM_STEPS) == {1, 2, 10, 1000} and set(ADAM_WDS) == {0.0, 0.1}


# ------------------------------------------------------------------------------------------------------------------
# coverage guard: every kernel entry point has an element-by-element or bit-exact test
# ------------------------------------------------------------------------------------------------------------------
COVERAGE = {
    "sb200_gemm": ["test_gpu_kernels.py::test_gemm_variant_matrix", "test_gpu_kernels.py::test_gemm"],
    "sb200_conv3x3": ["test_gpu_kernels.py::test_conv3x3_variant_matrix", "test_gpu_kernels.py::test_conv3x3"],
    "sb200_attention": ["test_gpu_forward_bounds.py::test_attention_fwd_bound"],
    "sb200_attention_bwd": ["test_gpu_backward_bounds.py::test_attention_bwd_bound"],
    "sb200_attention_bwd_ws": ["test_gpu_backward_bounds.py::test_attention_bwd_split_bound"],
    "sb200_gemm_splitk_f32": ["test_gpu_inversion_optim_bounds.py::test_gemm_splitk_f32_bound"],
    "sb200_groupnorm_bwd": ["test_gpu_backward_bounds.py::test_groupnorm_bwd_bound"],
    "sb200_layernorm_bwd": ["test_gpu_backward_bounds.py::test_layernorm_bwd_bound"],
    "sb200_geglu": ["test_gpu_backward_bounds.py::test_geglu_fwd_bwd_bound"],
    "sb200_geglu_bwd": ["test_gpu_backward_bounds.py::test_geglu_fwd_bwd_bound"],
    "sb200_add": ["test_gpu_backward_bounds.py::test_pointwise_helpers_bound"],
    "sb200_upsample2x_bwd": ["test_gpu_backward_bounds.py::test_pointwise_helpers_bound"],
    "sb200_zero_stuff": ["test_gpu_backward_bounds.py::test_pointwise_helpers_bound"],
    "sb200_conv_out_bwd": ["test_gpu_backward_bounds.py::test_pointwise_helpers_bound"],
    "sb200_colsum": ["test_gpu_backward_bounds.py::test_colsum_bound"],
    "sb200_lora_proj": ["test_gpu_backward_bounds.py::test_lora_linear_bound"],
    "sb200_lora_wgrad": ["test_gpu_backward_bounds.py::test_lora_linear_bound"],
    "sb200_lora_rank_update": ["test_gpu_backward_bounds.py::test_lora_linear_bound"],
    "sb200_lora_conv_proj": ["test_gpu_backward_bounds.py::test_lora_conv_bound"],
    "sb200_lora_conv_wgrad": ["test_gpu_backward_bounds.py::test_lora_conv_bound"],
    "sb200_lora_conv_rank_update": ["test_gpu_backward_bounds.py::test_lora_conv_bound"],
    "sb200_adamw": ["test_gpu_inversion_optim_bounds.py::test_adamw_matches_torch_bitwise",
                    "test_gpu_inversion_optim_bounds.py::test_adamw_resumed_at_step_10000",
                    "test_gpu_inversion_optim_bounds.py::test_adamw_guarded_table"],
    "sb200_adam_f32": ["test_gpu_inversion_optim_bounds.py::test_adam_f32_bound"],
    "sb200_groupnorm": ["test_gpu_forward_bounds.py::test_groupnorm_fwd_bound"],
    "sb200_layernorm": ["test_gpu_forward_bounds.py::test_layernorm_fwd_bound"],
    "sb200_small_linear": ["test_gpu_forward_bounds.py::test_small_linear_bound"],
    "sb200_sinusoid": ["test_gpu_forward_bounds.py::test_sinusoid_bound"],
    "sb200_conv_in": ["test_gpu_forward_bounds.py::test_conv_in_bound"],
    "sb200_conv_out": ["test_gpu_forward_bounds.py::test_conv_out_bound"],
    "sb200_upsample2x": ["test_gpu_forward_bounds.py::test_upsample2x_exact"],
    "sb200_cfg_ddim": ["test_gpu_forward_bounds.py::test_cfg_step_bound"],
    "sb200_cfg_step": ["test_gpu_forward_bounds.py::test_cfg_step_bound"],
    "sb200_guided_step_loss": ["test_gpu_inversion_optim_bounds.py::test_guided_loss_exact",
                               "test_gpu_inversion_optim_bounds.py::test_guided_loss_bound",
                               "test_gpu_inversion_optim_bounds.py::test_guided_loss_edges"],
    "sb200_lora_compose": ["test_gpu_compose.py::test_lora_compose_kernel_bitwise_with_guards"],
}


def test_every_kernel_entry_point_has_an_element_wise_test():
    """A new `int sb200_*(` entry point in include/sb200.h (other than create / destroy) cannot land without a line here
    naming its element-by-element or bit-exact test, and every named test must exist."""
    with open(os.path.join(ROOT, "include", "sb200.h")) as f:
        declared = set(re.findall(r"\bint\s+(sb200_\w+)\s*\(", f.read())) - {"sb200_create", "sb200_destroy"}
    assert len(declared) == 34
    assert declared == set(COVERAGE), (sorted(declared - set(COVERAGE)), sorted(set(COVERAGE) - declared))
    funcs = {}
    for tests in COVERAGE.values():
        for ref in tests:
            fname, func = ref.split("::")
            if fname not in funcs:
                with open(os.path.join(ROOT, "tests", fname)) as f:
                    funcs[fname] = {n.name for n in ast.walk(ast.parse(f.read())) if isinstance(n, ast.FunctionDef)}
            assert func in funcs[fname], ref
