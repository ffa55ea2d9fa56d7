"""Host-side pieces of null-text inversion (sliders_b200/inversion.py, generate.denoise_loop) that need no GPU: the DDIM
coefficient pairs of `next_step` / `prev_step` against what the notebook's class computed (golden fixture), the inner
loop's learning-rate schedule and early-stop threshold, argument validation of `negative_embeds_per_step`, and the
new C ABI entry points of libsb200.so."""
import os
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


GOLDEN = os.path.join(ROOT, "tests", "golden", "null_text_sd.pt")


@pytest.mark.parametrize("n", [50, 5, 7])
def test_step_coefficients_match_notebook(n):
    """(cx, ce) of x' = cx x + ce eps for the notebook's `next_step` / `prev_step` at every timestep, as its own class
    computed them on the oracle scheduler (tests/golden/make_golden_null_text.py), against the alpha-bar pairs
    inversion.py hands to the DDIM kernel.  The last step (t - T/N < 0) takes final_alpha_cumprod."""
    from oracle import ddim as oddim
    from sliders_b200 import inversion
    from sliders_b200.scheduler import DDIMScheduler

    rows = torch.load(GOLDEN)["step_coeffs"][n]
    ours = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                         set_alpha_to_one=False)
    ours.set_timesteps(n)
    assert ours.timesteps_host == [int(t) for t in rows[:, 0]]
    assert min(ours.timesteps_host) - 1000 // n < 0
    for t, ncx, nce, pcx, pce in rows.tolist():
        t = int(t)
        cx, ce = inversion.ddim_affine(*inversion.next_step_alphas(ours, t))
        assert (cx, ce) == (pytest.approx(ncx, rel=1e-5, abs=1e-6), pytest.approx(nce, rel=1e-5, abs=1e-6)), t
        cx, ce = inversion.ddim_affine(*inversion.prev_step_alphas(ours, t))
        assert (cx, ce) == (pytest.approx(pcx, rel=1e-5, abs=1e-6), pytest.approx(pce, rel=1e-5, abs=1e-6)), t
    ref = oddim.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                              set_alpha_to_one=False)
    t0 = min(ours.timesteps_host)
    assert inversion.prev_step_alphas(ours, t0)[1] == pytest.approx(float(ref.final_alpha_cumprod))
    assert inversion.next_step_alphas(ours, t0)[0] == pytest.approx(float(ref.final_alpha_cumprod))


def test_lr_schedule_and_early_stop_threshold():
    from sliders_b200 import inversion

    assert inversion.NUM_DDIM_STEPS == 50 and inversion.GUIDANCE_SCALE == 7.5
    assert [inversion.lr_at(i) for i in (0, 1, 49)] == pytest.approx([1e-2, 0.99e-2, 0.51e-2])
    assert inversion.early_stop_threshold(1e-5, 0) == pytest.approx(1e-5)
    assert inversion.early_stop_threshold(1e-5, 49) == pytest.approx(1e-5 + 49 * 2e-5)
    assert inversion.early_stop_threshold(0.0, 10) == pytest.approx(2e-4)


def test_negative_embeds_per_step_validation():
    from sliders_b200.generate import check_negative_embeds_per_step

    prompt = torch.zeros(4, 77, 768)
    good = [torch.zeros(1, 77, 768) for _ in range(5)]
    check_negative_embeds_per_step(good, prompt, 5)
    check_negative_embeds_per_step([torch.zeros(77, 768)] * 5, prompt, 5)
    with pytest.raises(ValueError, match="5 entries for 4 steps"):
        check_negative_embeds_per_step(good, prompt, 4)
    with pytest.raises(ValueError, match=r"\[2\]"):
        check_negative_embeds_per_step(good[:2] + [torch.zeros(1, 77, 2048)] + good[3:], prompt, 5)
    with pytest.raises(ValueError, match=r"\[0\]"):
        check_negative_embeds_per_step([torch.zeros(2, 77, 768)] + good[1:], prompt, 5)
    with pytest.raises(ValueError, match=r"\[1\]"):
        check_negative_embeds_per_step([good[0], None] + good[2:], prompt, 5)


def test_library_exports_inversion_entries():
    lib = os.path.join(ROOT, "sliders_b200", "libsb200.so")
    if not os.path.exists(lib):
        pytest.skip("libsb200.so not built")
    if shutil.which("nm") is None:
        pytest.skip("nm not available")
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    for name in ("sb200_attention_bwd", "sb200_attention_bwd_ws", "sb200_gemm_splitk_f32", "sb200_adam_f32",
                 "sb200_guided_step_loss"):
        assert any(line.split()[-1] == name for line in syms.splitlines() if line.strip()), name


def test_host_sizes_match_header_macros():
    """ops mirrors the scratch-size macros of include/sb200.h."""
    from sliders_b200 import ops

    # SD1.x at batch 1: 8 heads -> 17 splits wanted; SDXL at batch 2 (20 heads) -> 7; self-attention: no split
    assert ops.attn_bwd_splits(1, 8, 4096, 77) == 17
    assert ops.attn_bwd_splits(2, 10, 1024, 77) == 7
    assert ops.attn_bwd_splits(1, 8, 256, 77) == 4
    assert ops.attn_bwd_splits(1, 8, 4096, 4096) == 1
    assert ops.attn_bwd_splits(16, 10, 4096, 77) == 1
    # d_ctx GEMM, SD1.x batch 1: 6 tiles of 128 x 128, K = 24 960 -> 390 k-blocks in 22 splits of 18
    assert ops.splitk_ws_floats(77, 768, 24960) == 22 * 77 * 768
    # SDXL batch 1: 16 tiles, K = 166 400 -> 2600 k-blocks in 9 splits of 289
    assert ops.splitk_ws_floats(77, 2048, 166400) == 9 * 77 * 2048
