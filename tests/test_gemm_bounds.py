"""Host-side checks of the GEMM test machinery in test_gpu_kernels.py: the per-element error bound rejects the local
errors a GEMM epilogue can make (which rel-RMS over the whole output does not), and the variant matrix forces every
gemm_kernel instantiation into every shared-memory regime it can launch in."""
import torch

from test_gpu_kernels import (BF, CONV_MATRIX, GEMM_MATRIX, bound_violations, conv_grid, decode_force, gemm_grid,
                              gemm_slots, make_lora, regime, rel_rms)


def test_elementwise_bound_accepts_rounding_and_rejects_local_errors():
    g = torch.Generator().manual_seed(0)
    M, N, K = 2048, 640, 256
    x = torch.randn(M, K, generator=g).to(BF)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(BF)
    resid = torch.randn(M, N, generator=g).to(BF)
    proj = x.double() @ w.double().t()
    ref = proj + resid.double()
    mag = x.double().abs() @ w.double().abs().t()

    def kernel_like(p, r):
        """fp32 projection rounded to bf16, then a bf16 residual add: the two roundings of the GEMM epilogue."""
        return p.float().to(BF) + r

    out = kernel_like(proj, resid)
    assert not bound_violations(out, ref, proj, mag).any()

    # one epilogue thread's 16-column chunk of one row holds the next row's values (a wrong row map or swizzle)
    bad = out.clone()
    bad[100, 48:64] = out[101, 48:64]
    v = bound_violations(bad, ref, proj, mag)
    assert v[100, 48:64].all() and int(v.sum()) == 16
    assert rel_rms(bad, ref) < 1e-2  # the whole-output check alone passes this output

    # one element misses one 64-deep k-block (its largest)
    i, j = 7, 5
    blocks = (x[i].double() * w[j].double()).view(K // 64, 64).sum(1)
    kb = int(blocks.abs().argmax())
    bad = out.clone()
    bad[i, j] = kernel_like(proj[i, j] - blocks[kb], resid[i, j])
    v = bound_violations(bad, ref, proj, mag)
    assert v[i, j] and int(v.sum()) == 1

    # the residual read one row off
    v = bound_violations(kernel_like(proj, resid.roll(1, dims=0)), ref, proj, mag)
    assert v.double().mean() > 0.9

    # NaN never passes
    bad = out.clone()
    bad[3, 3] = float("nan")
    assert bound_violations(bad, ref, proj, mag)[3, 3]


def _cells():
    """(BN, kCtas, RT, regime) of every gemm_kernel instantiation and shared-memory regime it can launch in."""
    return {(bn, ctas, rt, reg) for bn in (64, 128) for ctas in (1, 2) for rt in (0, 16, 32)
            for reg in (("ring1", "ring2") if gemm_slots(bn, rt) == 2 else ("ring1",))}


def _check_row(grid, bn, rt, reg):
    for sms in (114, 132):  # H100 PCIe .. SXM
        assert regime(grid, bn, rt, sms) == reg, (grid, sms)
    if gemm_slots(bn, rt) == 2:  # margins: ring2 grids fill both slots of every SM, ring1 grids fit the smallest H100
        assert grid >= 2 * 132 if reg == "ring2" else grid <= 114, grid


def test_variant_matrix_is_complete():
    assert len(_cells()) == 20
    for matrix, grid_of in ((GEMM_MATRIX, lambda s, f, bn, c: gemm_grid(s[0], s[1], f, bn, c)),
                            (CONV_MATRIX, lambda s, f, bn, c: conv_grid(s[0], s[1], s[2], s[6], s[5], bn, c))):
        cells = set()
        for shape, flags, lora, force, rt, reg in matrix:
            bn, ctas = decode_force(force)
            assert "Y" not in flags or "R" in flags, "a strided residual needs a residual"
            n, k = (shape[1], shape[2]) if matrix is GEMM_MATRIX else (shape[5], 9 * (shape[3] + shape[4]))
            assert (make_lora(k, n, lora[0], lora[1], "cpu", 0)[2] if lora else 0) == rt, (shape, lora)
            _check_row(grid_of(shape, flags, bn, ctas), bn, rt, reg)
            cells.add((bn, ctas, rt, reg))
        assert cells == _cells()
