"""GPU tests of gemm_wide_kernel on long persistent walks: N = 256 (GEGLU: 512 W rows), so the grid has one column of
tiles and every CTA runs three or more tiles back to back, each epilogue staging its output while the producer already
streams the next tile.  Each case checks guard bands, repeatability, bit equality with gemm_kernel's single-CTA
bn = 128 result and the per-element bound of test_gpu_kernels, as test_gpu_gemm_wide does for its shapes."""
import pytest
import torch

from test_gpu_kernels import (SINGLE, cdiv, gemm_case, gemm_reference, guarded_out,  # noqa: F401
                              assert_guard_intact, assert_within_bound, rel_rms, run_gemm, dev)

pytestmark = pytest.mark.gpu

WIDE = 256 | SINGLE
NARROW = 128 | SINGLE

# M, N, K, flags (as gemm_case: b bias, t row bias in 4 groups of M // 4 rows, R residual, Y residual as a column view,
# G GEGLU, L LoRA), lora
CASES = [
    (51000, 256, 128, "", None),                    # no epilogue operand, M tail
    (51000, 256, 128, "bRY", None),                 # residual through a column view
    (51011, 256, 192, "btR", None),                 # row-bias group boundaries inside tiles (12 752 rows per group)
    (51000, 512, 128, "bG", None),                  # GEGLU: one 128-column output tile per row tile
    (50944, 256, 128, "bRL", (4, 128, 0.75)),       # two rank-4 adaptors, rt 16
    (50944, 256, 128, "btL", (8, 256, -0.5)),       # one rank-8 adaptor, rt 16, row bias
]


@pytest.mark.parametrize("M,N,K,flags,lora", CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{c[3] or 'plain'}" for c in CASES])
def test_wide_persistent_walk(dev, M, N, K, flags, lora):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = cdiv(M, 128)
    assert tiles >= 3 * sms and tiles % sms != 0
    c = gemm_case(M, N, K, flags, lora, dev, M + K)
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
