"""GPU tests of LoRA ranks 1-16: the rank-16 fused kernels (gemm_kernel<*, *, 64>, the rank-16 epilogue at 16 / 32 /
64 LoRA-down rows, conv, small_linear, the six backward kernels) element by element against float64,
and on tiny UNets that an adaptor of rank r gives bit for bit what the same weights zero-padded to the slot width give
(forward eager and under graph replay, gradients, one AdamW step), rank 16 against the fp32 oracle, and a rank-1
slider file through the eval sweep."""
import pytest
import torch

import test_gpu_backward_bounds as bb
import test_gpu_forward_bounds as fb
import test_gpu_kernels as gk
from conftest import c3lier
from test_gpu_kernels import (PAIR, SINGLE, assert_guard_intact, assert_within_bound, conv_case, conv_grid,
                              conv_reference, decode_force, gemm_case, gemm_grid, gemm_reference, guarded_out,
                              rel_rms, run_conv, run_gemm)

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def make_lora(K, N, r, group_n, dev, seed, conv_cin=None):
    """test_gpu_kernels.make_lora with rt from ops.lora_slots, so up to 64 LoRA-down rows (r is the slot width 4, 8 or
    16); the same draws, hence the same operands, wherever the rank-4/8 helper applies."""
    from sliders_b200 import ops

    g = torch.Generator().manual_seed(seed)
    groups = (N + group_n - 1) // group_n
    rt = ops.lora_slots(r, groups)[1]
    down = torch.zeros(rt, K)
    down[: groups * r] = torch.randn(groups * r, K, generator=g) / K ** 0.5
    up = (torch.randn(N, r, generator=g) * 0.5).to(BF).float()
    return down.to(dev, BF), up.to(dev), rt


@pytest.fixture
def rank16(monkeypatch):
    """The kernel-test helpers of test_gpu_kernels / test_gpu_forward_bounds with the rank-16 make_lora."""
    monkeypatch.setattr(gk, "make_lora", make_lora)
    monkeypatch.setattr(fb, "make_lora", make_lora)


def gemm_slots(bn, rt):
    """gemm_slots in gemm.cu: 64 LoRA rows run one CTA per SM at either width."""
    return 1 if rt == 64 else gk.gemm_slots(bn, rt)


# (M, N, K), flags, lora (rank, group_n, scale), bn | ctas, rt, regime: every rank-16 LoRA-row count on every tile
# width and CTA flavour.  rt = 64 instantiations run one CTA per SM, so "ring1" is their only regime.
GEMM16_MATRIX = [
    ((640, 960, 320), "L", (16, 320, 1.0), 64 | SINGLE, 64, "ring1"),        # fused q|k|v, three rank-16 adaptors
    ((300, 3840, 1280), "bRLX", (16, 1280, -0.5), 64 | PAIR, 64, "ring1"),   # SDXL width, phantom half, x a view
    ((512, 1920, 640), "RLY", (16, 640, 0.75), 128 | SINGLE, 64, "ring1"),   # residual a view
    ((384, 960, 200), "btL", (16, 320, 2.0), 128 | PAIR, 64, "ring1"),       # row bias, K = 200
    ((256, 336, 576), "bRL", (16, 336, 1.0), 64 | SINGLE, 16, "ring1"),      # one rank-16 adaptor, N % 32 = 16
    ((8192, 320, 640), "bLS", (16, 320, 1.0), 64 | PAIR, 16, "ring2"),       # split sources, two CTAs per SM
    ((1000, 1280, 1280), "bRL", (16, 1280, -1.0), 128 | SINGLE, 16, "ring1"),
    ((4096, 640, 320), "RL", (16, 320, 0.5), 64 | SINGLE, 32, "ring2"),      # attn2 to_k | to_v: two adaptors
    ((154, 2560, 2048), "L", (16, 1280, 1.0), 128 | PAIR, 32, "ring1"),      # the cross-attention K / V shape
]

CONV16_MATRIX = [
    ((2, 32, 32, 128, 0, 320, 1), "btL", (16, 320, 0.5), 64 | SINGLE, 16, "ring1"),
    ((1, 64, 64, 64, 0, 320, 2), "bL", (16, 320, 1.0), 64 | PAIR, 16, "ring1"),        # stride 2
    ((2, 32, 32, 128, 64, 640, 1), "bLRX", (16, 640, -0.5), 128 | SINGLE, 16, "ring1"),  # skip concat, views
    ((1, 16, 16, 64, 0, 640, 2), "bL", (16, 640, 1.0), 128 | PAIR, 16, "ring1"),       # stride 2
]


def _id(row):
    shape, flags, lora, force, rt, reg = row
    bn, ctas = decode_force(force)
    return f"bn{bn}-ctas{ctas}-rt{rt}-{reg}-" + "x".join(map(str, shape)) + f"-{flags}"


def test_rank16_matrix_is_complete():
    """Every rt = 64 instantiation in every regime it launches in, and both other row counts at rank 16."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    cells = set()
    for shape, flags, lora, force, rt, reg in GEMM16_MATRIX:
        bn, ctas = decode_force(force)
        assert make_lora(shape[2], shape[1], lora[0], lora[1], "cpu", 0)[2] == rt
        grid = gemm_grid(shape[0], shape[1], flags, bn, ctas)
        assert ("ring2" if grid > sms and gemm_slots(bn, rt) == 2 else "ring1") == reg, shape
        cells.add((bn, ctas, rt, reg))
    assert {c for c in cells if c[2] == 64} == {(bn, ctas, 64, "ring1") for bn in (64, 128) for ctas in (1, 2)}
    assert {c[2] for c in cells} == {16, 32, 64}
    for shape, flags, lora, force, rt, reg in CONV16_MATRIX:
        bn, ctas = decode_force(force)
        assert conv_grid(shape[0], shape[1], shape[2], shape[6], shape[5], bn, ctas) <= 114
    assert {row[0][6] for row in CONV16_MATRIX} == {1, 2} and any(row[0][4] for row in CONV16_MATRIX)


@pytest.mark.parametrize("shape,flags,lora,force,rt,reg", GEMM16_MATRIX, ids=[_id(r) for r in GEMM16_MATRIX])
def test_gemm_rank16(dev, rank16, shape, flags, lora, force, rt, reg):
    M, N, K = shape
    bn, ctas = decode_force(force)
    c = gemm_case(M, N, K, flags, lora, dev, M + N + K, split=gk.split_of(flags, K))
    assert c.rt == rt
    bufs = [guarded_out(M, c.nout, dev) for _ in range(2)]
    for _, out in bufs:
        run_gemm(c, force, out=out)
    other = run_gemm(c, bn | (SINGLE if ctas == 2 else PAIR))
    auto = run_gemm(c, 0)
    torch.cuda.synchronize()
    for buf, _ in bufs:
        assert_guard_intact(buf, M, c.nout)
    out = bufs[0][1]
    assert torch.equal(out, bufs[1][1]) and torch.equal(out, other)
    ref, proj, mag = gemm_reference(c)
    assert_within_bound(out, ref, proj, mag)
    assert_within_bound(auto, ref, proj, mag)
    assert rel_rms(out, ref) < 1e-2


@pytest.mark.parametrize("shape,flags,lora,force,rt,reg", CONV16_MATRIX, ids=[_id(r) for r in CONV16_MATRIX])
def test_conv3x3_rank16(dev, rank16, shape, flags, lora, force, rt, reg):
    B, H, W, C0, C1, Cout, stride = shape
    bn, ctas = decode_force(force)
    c = conv_case(B, H, W, C0, C1, Cout, stride, flags, lora, dev, B * H + C0 + Cout)
    assert c.rt == rt
    pixels = B * c.Ho * c.Wo
    buf, out = guarded_out(pixels, Cout, dev)
    run_conv(c, force, out=out.view(B, c.Ho, c.Wo, Cout))
    other = run_conv(c, bn | (SINGLE if ctas == 2 else PAIR))
    torch.cuda.synchronize()
    assert_guard_intact(buf, pixels, Cout)
    out = out.view(B, c.Ho, c.Wo, Cout)
    assert torch.equal(out, other)
    ref, proj, mag = conv_reference(c)
    assert_within_bound(out, ref, proj, mag)
    assert rel_rms(out, ref) < 1e-2


def test_wide_tiles_refuse_rank16(dev, rank16):
    """gemm_wide_kernel's epilogue takes ranks 4 and 8: an explicit bn = 256 at rank 16 or rt = 64 is refused, and the
    cost model never picks it there (the automatic choice is checked against the reference above)."""
    from sliders_b200 import _cabi

    for lora in ((16, 1280, 1.0), (16, 256, 1.0)):
        c = gemm_case(512, 768 if lora[1] == 256 else 1280, 640, "L", lora, dev, 5)
        with pytest.raises(_cabi.Sb200Error, match="bn=256"):
            run_gemm(c, 256)


@pytest.mark.parametrize("M,N,K,xpad,act_in,act_out,lora,resid", [
    (4, 640, 1280, 8, True, 0, (16, 640, 0.5), False),    # time_emb_proj at rank 16
    (64, 1280, 1280, 0, False, 1, (16, 1280, -1.0), True),
    (9, 40, 320, 16, True, 0, (16, 20, 1.0), False),      # a block of 8 columns spanning two rank-16 adaptors
])
def test_small_linear_rank16(dev, rank16, M, N, K, xpad, act_in, act_out, lora, resid):
    fb.test_small_linear_bound(dev, M, N, K, xpad, act_in, act_out, lora, resid)


@pytest.mark.parametrize("M,C,sources,pad,acc", [
    (1, 1280, 1, 0, False),        # M = batch: one chunk
    (4096, 1280, 2, 2560, True),   # two sources, strided A, accumulate
    (1024, 640, 1, 1280, False),   # lda = 3C
    (154, 2048, 2, 0, True),
])
def test_lora_linear_backward_rank16(dev, M, C, sources, pad, acc):
    """lora_proj / lora_wgrad (transposed into column slices and untransposed into a strided G, accumulate; rank 16
    runs as two 8-column halves) / lora_rank_update at rank 16, with the checks of test_gpu_backward_bounds."""
    bb.test_lora_linear_bound(dev, M, C, 16, sources, pad, acc)


@pytest.mark.parametrize("B,H,W,C0,C1,stride,acc", [
    (2, 16, 24, 320, 0, 1, False),
    (1, 16, 16, 256, 128, 1, True),    # concat input, accumulate
    (2, 16, 12, 128, 0, 2, True),      # stride 2
])
def test_lora_conv_backward_rank16(dev, B, H, W, C0, C1, stride, acc):
    bb.test_lora_conv_bound(dev, B, H, W, C0, C1, stride, 16, acc)


def test_backward_entry_points_take_rank_16_only_as_slot(dev):
    from sliders_b200 import _cabi, ops

    A = torch.zeros(8, 64, device=dev, dtype=BF)
    with pytest.raises(_cabi.Sb200Error, match="r=12"):
        ops.lora_proj(A, torch.zeros(12, 64, device=dev, dtype=BF))


# ------------------------------------------------------------------------------------------------------------------
# UNet level
# ------------------------------------------------------------------------------------------------------------------
def _tiny(config, dev, seed):
    from oracle import unet as ounet
    from sliders_b200 import synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    ocfg = getattr(ounet.UNetConfig, config)()
    pm = UNet2DConditionModel(UNetConfig.from_dict(ocfg.__dict__))
    synthetic.init_synthetic_(pm, seed=seed)
    return ocfg, pm.to(dev, BF).eval().requires_grad_(False)


def _inputs(ocfg, dev, xl, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 4, 32, 32, generator=g).to(dev, BF)
    ehs = torch.randn(2, 77, ocfg.cross_attention_dim, generator=g).to(dev, BF)
    added = None
    if xl:
        added = {"text_embeds": torch.randn(2, 128, generator=g).to(dev, BF),
                 "time_ids": torch.tensor([[256., 256., 0., 0., 256., 256.]] * 2, device=dev)}
    goal = torch.randn(2, 4, 32, 32, generator=g).to(dev)
    return x, ehs, added, goal


def _call(pm, x, ehs, added):
    kw = {"added_cond_kwargs": added} if added is not None else {}
    return pm(x, 321, encoder_hidden_states=ehs, **kw).sample


def _network(pm, rank, alpha, method, dev):
    from sliders_b200 import lora as plora

    with c3lier(plora):
        return plora.LoRANetwork(pm, rank=rank, multiplier=1.0, alpha=alpha, train_method=method).to(dev, BF)


def _snapshot(net):
    return [(a.lora_name, a.lora_down.weight.detach().clone(), a.lora_up.weight.detach().clone(), a.scale)
            for a in net.unet_loras]


def _pad_into(src, dst):
    """dst's adaptors (slot width) hold the weights of snapshot src (rank r), zero-padded."""
    with torch.no_grad():
        for (name, down, up, scale), b in zip(src, dst.unet_loras):
            assert name == b.lora_name
            r = down.shape[0]
            b.lora_down.weight.zero_()
            b.lora_up.weight.zero_()
            b.lora_down.weight[:r].copy_(down)
            b.lora_up.weight[:, :r].copy_(up)
            assert scale == b.scale


def _slot(r):
    return 4 if r <= 4 else 8 if r <= 8 else 16


@pytest.mark.parametrize("config", ["tiny_xl", "tiny_sd"])
@pytest.mark.parametrize("r", [1, 2, 3, 5, 7, 12])
def test_low_rank_equals_zero_padded_slot_width(dev, config, r):
    """Rank r against the same weights zero-padded to rank 4 / 8 / 16 with alpha scaled so that alpha / r is equal:
    eps eager and under graph replay, the real rows of every LoRA gradient, and the weights after one AdamW step are
    bit-identical."""
    from sliders_b200 import synthetic
    from sliders_b200.optim import AdamW

    rp = _slot(r)
    xl = config == "tiny_xl"
    outs = {}
    for rank in (r, rp):
        ocfg, pm = _tiny(config, dev, seed=40 + r)
        net = _network(pm, rank, 2.0 * rank / r, "noxattn", dev)
        if rank == r:
            synthetic.init_lora_nonzero_(net, seed=41, up_std=0.05, reseed_down=True)
            src = _snapshot(net)  # before this network's AdamW step changes it
        else:
            _pad_into(src, net)
        x, ehs, added, goal = _inputs(ocfg, dev, xl)
        net.set_lora_slider(0.75)
        with torch.no_grad(), net:
            eager = _call(pm, x, ehs, added)
            pm.use_cuda_graph = True
            _call(pm, x, ehs, added)
            net.set_lora_slider(-1.5)
            graphed = _call(pm, x, ehs, added)   # replay with another slider value
            pm.use_cuda_graph = False
            eager_neg = _call(pm, x, ehs, added)
            net.set_lora_slider(0.75)
        assert torch.equal(graphed, eager_neg)
        net.requires_grad_(True)
        opt = AdamW(net.prepare_optimizer_params(), lr=1e-3)
        with net:
            pred = _call(pm, x, ehs, added)
        torch.nn.functional.mse_loss(pred.float(), goal).backward()
        grads = {a.lora_name: (a.lora_down.weight.grad[:r].clone(), a.lora_up.weight.grad[:, :r].clone())
                 for a in net.unet_loras}
        for a in net.unet_loras:
            if rank != r:  # the padded rows of the slot-width network get zero gradients
                assert not a.lora_down.weight.grad[r:].any() and not a.lora_up.weight.grad[:, r:].any()
        opt.step()
        torch.cuda.synchronize()
        after = {a.lora_name: (a.lora_down.weight.detach()[:r].clone(), a.lora_up.weight.detach()[:, :r].clone())
                 for a in net.unet_loras}
        outs[rank] = (eager, eager_neg, grads, after)
    (e1, n1, g1, w1), (e2, n2, g2, w2) = outs[r], outs[rp]
    assert torch.equal(e1, e2) and torch.equal(n1, n2)
    assert g1.keys() == g2.keys()
    for k in g1:
        assert torch.equal(g1[k][0], g2[k][0]) and torch.equal(g1[k][1], g2[k][1]), k
        assert torch.equal(w1[k][0], w2[k][0]) and torch.equal(w1[k][1], w2[k][1]), k


@pytest.mark.parametrize("config", ["tiny_xl", "tiny_sd"])
@pytest.mark.parametrize("method", ["noxattn", "full"])
def test_rank16_against_fp32_oracle(dev, config, method):
    """eps and every LoRA gradient at rank 16 against the fp32 oracle with the LoRA delta folded into its weights
    (the tolerances of the rank-4 tests in test_gpu_unet.py).  `full` adapts the attn2 to_k | to_v pair (32 LoRA
    rows), the feed-forward and proj_in / proj_out besides the fused q|k|v (64 rows)."""
    from oracle import unet as ounet
    from sliders_b200 import synthetic
    from test_gpu_unet import _oracle_lora_grads

    xl = config == "tiny_xl"
    ocfg, pm = _tiny(config, dev, seed=21)
    om = ounet.UNet2DConditionModel(ocfg)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om = om.to(dev).eval().requires_grad_(False)
    net = _network(pm, 16, 8.0, method, dev)
    synthetic.init_lora_nonzero_(net, seed=22, up_std=0.05, reseed_down=True)
    net.requires_grad_(True)
    x, ehs, added, goal = _inputs(ocfg, dev, xl)
    net.set_lora_slider(0.5)
    with net:
        pred = _call(pm, x, ehs, added)
    torch.nn.functional.mse_loss(pred.float(), goal).backward()
    torch.cuda.synchronize()

    def call(fp):
        kw = {"added_cond_kwargs": {k: v.float() for k, v in added.items()}} if xl else {}
        out = torch.func.functional_call(om, fp, (x.float(), 321, ehs.float()), kw).sample
        assert rel_rms(pred, out) < 3e-2
        return torch.nn.functional.mse_loss(out, goal)

    leaves = _oracle_lora_grads(om, net, 0.5, call)
    num = den = 0.0
    for l in net.unet_loras:
        for got, ref in ((l.lora_down.weight.grad, leaves[l.lora_name][0].grad),
                         (l.lora_up.weight.grad, leaves[l.lora_name][1].grad)):
            assert got is not None and torch.isfinite(got).all(), l.lora_name
            num += (got.float() - ref).pow(2).sum().item()
            den += ref.pow(2).sum().item()
    assert (num / den) ** 0.5 < 5e-2, (config, method, (num / den) ** 0.5)
    if method == "full":
        assert any("attn2_to_k" in l.lora_name for l in net.unet_loras)


def test_training_graphs_bit_identical_to_eager_at_rank16(dev):
    """Three AdamW steps at rank 16 with CUDA-graph training replay and without: same weights bit for bit."""
    from sliders_b200 import synthetic
    from sliders_b200.optim import AdamW

    weights = []
    for graphs in (False, True):
        ocfg, pm = _tiny("tiny_xl", dev, seed=51)
        net = _network(pm, 16, 1.0, "noxattn", dev)
        synthetic.init_lora_nonzero_(net, seed=52, up_std=0.05, reseed_down=True)
        net.requires_grad_(True)
        pm.use_cuda_graph = graphs
        opt = AdamW(net.prepare_optimizer_params(), lr=1e-3)
        x, ehs, added, goal = _inputs(ocfg, dev, True)
        for _ in range(3):
            opt.zero_grad()
            with net:
                pred = _call(pm, x, ehs, added)
            torch.nn.functional.mse_loss(pred.float(), goal).backward()
            opt.step()
        torch.cuda.synchronize()
        weights.append([p.detach().clone() for p in net.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*weights))


@pytest.mark.parametrize("ext", [".pt", ".safetensors"])
def test_rank1_slider_file_through_the_eval_sweep(dev, tmp_path, ext):
    """A slider file named the reference's way without rank4 / rank8 in its name is built at rank 1 (the reference's
    eval scripts do so); a two-step sweep gives the latents of the same weights zero-padded to rank 4."""
    from sliders_b200 import eval_sweep as es
    from sliders_b200 import synthetic
    from sliders_b200.scheduler import create_noise_scheduler

    name = f"smile_alpha1.0_noxattn_last{ext}"
    assert es.parse_slider_name(name)["rank"] == 1
    trained = _network(_tiny("tiny_xl", dev, seed=61)[1], 1, 1.0, "noxattn", dev)
    synthetic.init_lora_nonzero_(trained, seed=62, up_std=0.1, reseed_down=True)
    slider = tmp_path / name
    trained.save_weights(str(slider), dtype=BF)
    pm = _tiny("tiny_xl", dev, seed=61)[1]
    pm.use_cuda_graph = True
    net = es.build_network(pm, str(slider), dev, BF)
    assert net.unet_loras[0].lora_down.weight.shape[0] == 1
    padded_pm = _tiny("tiny_xl", dev, seed=61)[1]
    padded_pm.use_cuda_graph = True
    padded = _network(padded_pm, 4, 4.0 * net.unet_loras[0].scale, "noxattn", dev)
    _pad_into(_snapshot(net), padded)
    csv_path = tmp_path / "p.csv"
    csv_path.write_text("case_number,prompt,evaluation_seed,concept\n3,a,11,x\n")
    rows = es.read_prompts_csv(str(csv_path))
    g = torch.Generator().manual_seed(0)
    table = {"a": (torch.randn(2, 77, 256, generator=g), torch.randn(2, 128, generator=g))}
    lat = {}
    for tag, unet, network in (("r1", pm, net), ("r4", padded_pm, padded)):
        out_dir = tmp_path / tag
        n = es.sweep(unet, network, create_noise_scheduler("euler"), rows, lambda p: table[p], str(out_dir),
                     scales=(-2, 2), num_samples=1, num_inference_steps=2, guidance_scale=5.0, start_noise=750,
                     image_size=256)
        assert n == 2
        lat[tag] = [torch.load(out_dir / str(s) / "3_0.pt") for s in (-2, 2)]
    assert all(torch.isfinite(v).all() for v in lat["r1"])
    assert not torch.equal(lat["r1"][0], lat["r1"][1])
    assert all(torch.equal(a, b) for a, b in zip(lat["r1"], lat["r4"]))


def _remove_network(pm, net):
    """Takes a LoRANetwork off its UNet: every adapted leaf gets its own forward back."""
    for a in net.unet_loras:
        del a.org_forward.__self__.__dict__["forward"]
    pm.__dict__.pop("_adapted_cache", None)


def test_swapping_in_a_network_of_another_rank_under_cuda_graphs(dev):
    """A rank-16 network replacing a rank-4 one on the same UNet gets its own packs and graphs: the graph replay after
    the swap equals the eager forward of the rank-16 network, forward and gradients, and swapping back to the rank-4
    network reproduces its first output."""
    from sliders_b200 import synthetic

    ocfg, pm = _tiny("tiny_xl", dev, seed=71)
    x, ehs, added, goal = _inputs(ocfg, dev, True)
    pm.use_cuda_graph = True
    results = {}
    for rank, seed in ((4, 72), (16, 73), (4, 72)):
        net = _network(pm, rank, 1.0, "noxattn", dev)
        synthetic.init_lora_nonzero_(net, seed=seed, up_std=0.05, reseed_down=True)
        net.set_lora_slider(1.5)
        with torch.no_grad(), net:
            graphed = [_call(pm, x, ehs, added) for _ in range(2)]
        pm.use_cuda_graph = False
        with torch.no_grad(), net:
            eager = _call(pm, x, ehs, added)
        pm.use_cuda_graph = True
        assert torch.equal(graphed[0], eager) and torch.equal(graphed[1], eager), rank
        net.requires_grad_(True)
        grads = []
        for graphs in (True, False):
            pm.use_cuda_graph = graphs
            for p in net.parameters():
                p.grad = None
            with net:
                pred = _call(pm, x, ehs, added)
            torch.nn.functional.mse_loss(pred.float(), goal).backward()
            grads.append([p.grad.clone() for p in net.parameters()])
        pm.use_cuda_graph = True
        assert all(torch.equal(a, b) for a, b in zip(*grads)), rank
        results.setdefault(rank, []).append(eager)
        _remove_network(pm, net)
    assert not torch.equal(results[4][0], results[16][0])
    assert torch.equal(results[4][0], results[4][1])


def test_full_sdxl_rank16_parity_vs_fp32_oracle(dev):
    """SDXL-base at 1024 px (128 x 128 latents, batch 2), rank-16 LoRA on the 346 noxattn + c3lier leaves at slider 2,
    against the fp32 oracle with the LoRA delta folded into its weights: the production q|k|v shapes (8192 x 1920 x 640
    and 2048 x 3840 x 1280 at 64 LoRA-down rows) end to end, with the full-size bar (rel-RMS <= 1e-2, max-abs
    <= 3e-2)."""
    from oracle import unet as ounet
    from sliders_b200 import lora as plora, synthetic
    from sliders_b200.unet import UNet2DConditionModel, UNetConfig

    batch = 2
    with torch.device(dev):
        pm = UNet2DConditionModel(UNetConfig.sdxl()).to(BF)
        om = ounet.UNet2DConditionModel(ounet.UNetConfig.sdxl())
    synthetic.init_synthetic_(pm, seed=1)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om.eval().requires_grad_(False)
    pm.eval().requires_grad_(False)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(batch, 4, 128, 128, generator=g).to(dev, BF)
    ehs = torch.randn(batch, 77, 2048, generator=g).to(dev, BF)
    added = {"text_embeds": torch.randn(batch, 1280, generator=g).to(dev, BF),
             "time_ids": torch.tensor([[1024., 1024, 0, 0, 1024, 1024]] * batch, device=dev)}
    addf = {"text_embeds": added["text_embeds"].float(), "time_ids": added["time_ids"]}
    with c3lier(plora):
        net = plora.LoRANetwork(pm, rank=16, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, BF)
    assert len(net.unet_loras) == 346
    synthetic.init_lora_nonzero_(net, seed=2, up_std=0.05)
    mods = {("lora_unet_" + n.replace(".", "_")): m for n, m in om.named_modules()}
    sd = net.state_dict()
    with torch.no_grad():
        for l in net.unet_loras:
            up, down = sd[l.lora_name + ".lora_up.weight"].float(), sd[l.lora_name + ".lora_down.weight"].float()
            delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down) if down.dim() == 4 else up @ down
            mods[l.lora_name].weight.add_(delta * (2.0 * l.scale))
        ref = om(x.float(), 19, ehs.float(), added_cond_kwargs=addf).sample
        del om
        net.set_lora_slider(2.0)
        with net:
            got = pm(x, 19, ehs, added_cond_kwargs=added).sample
    err = (got.float() - ref).abs().max().item()
    print(f"full SDXL + rank-16 LoRA (346, slider 2): rel_rms {rel_rms(got, ref):.4g} max_abs {err:.4g}")
    assert rel_rms(got, ref) < 1e-2
    assert err < 3e-2


def test_text_slider_iteration_rank16_matches_port(dev):
    """test_gpu_train.py's one-iteration check at rank 16: `trainer.text_slider_step_xl` with the inputs and random
    draws of the iter_text_xl fixture (tiny SDXL topology, noxattn + c3lier, enhance, guidance 4) but a rank-16 network,
    against oracle/port.py's `text_slider_iteration` on the fp32 oracle UNet with `LoRAHooks(rank=16)` holding the same
    weights, latents and step count: loss within 5 %, LoRA gradients rel-RMS < 5e-2, AdamW move sign agreement
    (weighted by |gradient|) > 0.97."""
    import os

    from oracle import ddim as oddim
    from oracle import port
    from oracle import unet as ounet
    from sliders_b200 import trainer
    from sliders_b200.scheduler import create_noise_scheduler
    from test_gpu_unet import GOLDEN, build_product

    fx = torch.load(os.path.join(GOLDEN, "iter_text_xl.pt"))
    pm, net = build_product(dict(fx, rank=16), dev)
    net.requires_grad_(True)
    om = ounet.UNet2DConditionModel(getattr(ounet.UNetConfig, fx["config"])())
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om = om.to(dev).eval().requires_grad_(False)
    hooks = port.LoRAHooks(om, rank=16, alpha=fx["alpha"], c3lier=True).to(dev)
    state = {k: v.float() for k, v in net.state_dict().items()}
    assert {k for k, _ in hooks.named_parameters()} == {k for k, _ in net.named_parameters()}
    hooks.load_weights(state)
    hooks.__exit__()
    before = {k: p.detach().clone() for k, p in net.named_parameters()}
    hooks_before = {k: p.detach().clone() for k, p in hooks.named_parameters()}

    e = {k: trainer.PromptEmbedsXL(v[0].to(dev, BF), v[1].to(dev, BF)) for k, v in fx["embeds"].items()}
    pair = trainer.PromptEmbedsPair(torch.nn.MSELoss(), e["target"], e["positive"], e["unconditional"], e["neutral"],
                                    trainer.PromptSettings(**fx["settings"]))
    opt = torch.optim.AdamW(net.prepare_optimizer_params(), lr=fx["lr"])
    torch.manual_seed(fx["seed"])
    torch.randint(0, 1, (1,))   # the prompt-pair pick that precedes the step's draws (train_lora_xl.py:172-174)
    loss = trainer.text_slider_step_xl(pm, net, create_noise_scheduler("ddim"), opt, None, pair, max_denoising_steps=50,
                                       device=dev, weight_dtype=BF)

    osched = oddim.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                                 num_train_timesteps=1000, clip_sample=False)
    oopt = torch.optim.AdamW(hooks.prepare_optimizer_params(), lr=fx["lr"])
    tids = fx["add_time_ids"].to(dev)
    ref_loss = port.text_slider_iteration(
        om, hooks, osched, oopt, {k: v[0].float().to(dev) for k, v in fx["embeds"].items()},
        fx["latents"].float().to(dev), fx["timesteps_to"], guidance_scale=4.0, action="enhance",
        added={k: (v[1].float().to(dev), tids) for k, v in fx["embeds"].items()})
    ref = dict(hooks.named_parameters())
    num = den = agree = total = 0.0
    for k, p in net.named_parameters():
        rg = ref[k].grad.float()
        num += (p.grad.float() - rg).pow(2).sum().item()
        den += rg.pow(2).sum().item()
        w = rg.abs()
        ours = torch.sign(p.detach().float() - before[k].float())
        theirs = torch.sign(ref[k].detach() - hooks_before[k])
        agree += (w * (ours == theirs).float()).sum().item()
        total += w.sum().item()
    print(f"rank-16 text-slider iteration: loss {float(loss):.5g} vs {float(ref_loss):.5g}, grad rel-RMS "
          f"{(num / den) ** 0.5:.4g}, move-sign agreement {agree / total:.4f}")
    assert abs(float(loss) - float(ref_loss)) <= 0.05 * float(ref_loss), (float(loss), float(ref_loss))
    assert (num / den) ** 0.5 < 5e-2, (num / den) ** 0.5
    assert agree / total > 0.97, agree / total
