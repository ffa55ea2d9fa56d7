"""CPU tests of slider composition (sliders_b200.lora.SliderStack): the slot layout of the composite LoRA packs,
seeded weights and checkpoint keys equal to the reference's chained LoRANetworks, every refusal, the graph signature,
and the eval sweep's `--compose`."""
import os

import pytest
import torch
import torch.nn as nn

from oracle import reference_bridge as rb
from oracle import unet as ounet
from sliders_b200 import lora as plora
from sliders_b200 import lora_pack as lp
from sliders_b200 import ops
from sliders_b200.unet import UNet2DConditionModel, UNetConfig, _StackArena, _adaptor_of, _fill_composite, _hook_of

SPECS = [dict(rank=4, alpha=1.0, train_method="noxattn", network_type="c3lier"),
         dict(rank=8, alpha=4.0, train_method="xattn")]


def _unet(cfg="tiny_xl"):
    return UNet2DConditionModel(UNetConfig.from_dict(getattr(ounet.UNetConfig, cfg)().__dict__))


def _stack(specs=SPECS, seed=0, unet=None):
    pm = unet if unet is not None else _unet()
    torch.manual_seed(seed)
    return pm, plora.SliderStack(pm, specs)


def _randomise(stack, seed=1):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in stack.parameters():
            if p.dim() > 0:
                p.copy_(torch.randn(p.shape, generator=g))


def _pack(pm, stack, leaves):
    hooks = [_hook_of(l) for l in leaves]
    rp = ops.lora_slots(stack.total_rank)[0]
    _, rt = ops.lora_slots(rp, len(leaves))
    K = leaves[0].weight[0].numel()
    N = sum(l.weight.shape[0] for l in leaves)
    down = torch.zeros(rt, K, dtype=torch.bfloat16)
    raw = torch.zeros(N, rp)
    _fill_composite(down, raw, leaves, hooks, stack.offsets, rp)
    return down, raw, rp, rt


def _module(net, leaf_path):
    return getattr(net, "lora_unet_" + leaf_path.replace(".", "_"))


# ---------------------------------------------------------------------------------------------------------- layout
def test_slot_layout_windows_and_zeros():
    pm, stack = _stack()
    _randomise(stack)
    noxattn, xattn = stack.sliders
    assert stack.offsets == (0, 4) and stack.ranks == (4, 8)
    attn1 = pm.down_blocks[1].attentions[0].transformer_blocks[0].attn1
    attn2 = pm.down_blocks[1].attentions[0].transformer_blocks[0].attn2
    path1 = "down_blocks.1.attentions.0.transformer_blocks.0.attn1"
    path2 = "down_blocks.1.attentions.0.transformer_blocks.0.attn2"

    # attn1 q|k|v: only the noxattn slider (columns 0-3); slider 1's window [4, 12) stays zero
    leaves = [attn1.to_q, attn1.to_k, attn1.to_v]
    down, raw, rp, rt = _pack(pm, stack, leaves)
    assert (rp, rt) == (16, 64)
    C = attn1.to_q.weight.shape[0]
    for gi, name in enumerate(("to_q", "to_k", "to_v")):
        a = _module(noxattn, f"{path1}.{name}")
        assert torch.equal(down[gi * rp: gi * rp + 4], a.lora_down.weight.to(torch.bfloat16))
        assert not down[gi * rp + 4: (gi + 1) * rp].any()
        assert torch.equal(raw[gi * C:(gi + 1) * C, :4], a.lora_up.weight.float() * (1.0 / 4))
    assert not raw[:, 4:].any()

    # attn2 k|v: only the xattn slider (columns 4-11, alpha 4 / rank 8); slider 0's columns stay zero
    leaves = [attn2.to_k, attn2.to_v]
    down, raw, rp, rt = _pack(pm, stack, leaves)
    assert (rp, rt) == (16, 32)
    for gi, name in enumerate(("to_k", "to_v")):
        a = _module(xattn, f"{path2}.{name}")
        assert a.scale == 0.5
        assert torch.equal(down[gi * rp + 4: gi * rp + 12], a.lora_down.weight.to(torch.bfloat16))
        assert not down[gi * rp: gi * rp + 4].any() and not down[gi * rp + 12: (gi + 1) * rp].any()
        assert torch.equal(raw[gi * C:(gi + 1) * C, 4:12], a.lora_up.weight.float() * 0.5)
    assert not raw[:, :4].any() and not raw[:, 12:].any()

    # a 3x3 conv of the c3lier slider: down packed tap-major [r, 3, 3, Cin]
    conv = pm.down_blocks[0].resnets[0].conv1
    down, raw, rp, rt = _pack(pm, stack, [conv])
    a = _module(noxattn, "down_blocks.0.resnets.0.conv1")
    assert torch.equal(down[:4], a.lora_down.weight.permute(0, 2, 3, 1).reshape(4, -1).to(torch.bfloat16))
    assert torch.equal(raw[:, :4], a.lora_up.weight.reshape(-1, 4).float() * 0.25)
    assert not raw[:, 4:].any()
    # a leaf no slider adapts has no hook
    assert _hook_of(pm.conv_in) is None and _hook_of(pm.time_embedding.linear_1) is None


def test_conv_rank_clamp_folds_alpha_over_clamped_rank():
    """lora.py:78: a conv adaptor's rank is clamped to min(rank, Cin, Cout); alpha / (clamped rank) is folded into raw
    and the slider's columns past the clamped rank stay zero."""
    leaf = nn.Conv2d(2, 3, 3, padding=1)
    a = plora.LoRAModule("c", leaf, multiplier=1.0, lora_dim=4, alpha=3.0)
    assert a.lora_dim == 2 and a.scale == 1.5
    with torch.no_grad():
        a.lora_up.weight.copy_(torch.randn(a.lora_up.weight.shape))
    del a.org_module
    hook = plora.SliderHook(None, "c")
    hook.slider_entries.append((1, a))
    rp = 8
    down, raw = torch.zeros(16, 18, dtype=torch.bfloat16), torch.zeros(3, rp)
    _fill_composite(down, raw, [leaf], [hook], (0, 4), rp)
    assert torch.equal(raw[:, 4:6], a.lora_up.weight.reshape(3, 2) * 1.5)
    assert not raw[:, :4].any() and not raw[:, 6:].any()
    assert down[4:6].any() and not down[:4].any() and not down[6:].any()


@pytest.mark.parametrize("ranks", [(1,), (4,), (2, 2), (4, 4), (4, 8), (4, 4, 4, 4), (16,), (3, 5, 8)])
def test_slot_width_follows_total_rank(ranks):
    specs = [dict(rank=r, alpha=1.0, train_method="xattn") for r in ranks]
    pm, stack = _stack(specs)
    arena = _StackArena(stack, "cpu")
    assert arena.rp == ops.lora_slots(sum(ranks))[0]
    assert stack.offsets == tuple(sum(ranks[:i]) for i in range(len(ranks)))
    arena.load([float(i + 1) for i in range(len(ranks))])
    cols = arena.mult.tolist()
    for i, (o, r) in enumerate(zip(stack.offsets, ranks)):
        assert cols[o:o + r] == [float(i + 1)] * r
    assert cols[sum(ranks):] == [0.0] * (arena.rp - sum(ranks))
    attn2 = pm.mid_block.attentions[0].transformer_blocks[0].attn2
    _, _, rp, rt = _pack(pm, stack, [attn2.to_k, attn2.to_v])
    assert (rp, rt) == ops.lora_slots(sum(ranks), 2)


# ------------------------------------------------------------------------------------------- weights and keys
@pytest.mark.skipif(not rb.available(), reason="needs the reference's lora.py")
@pytest.mark.parametrize("cfg", ["tiny_xl", "tiny_sd"])
def test_seeded_weights_equal_reference_chained_networks(cfg):
    """Same seed, same order: the stack's sliders hold bit for bit the initial weights of the reference's own
    LoRANetworks built one after another on one UNet (duplicates built and discarded included)."""
    lora = rb.load("lora")
    specs = [dict(rank=4, alpha=1.0, train_method="noxattn", network_type="c3lier"),
             dict(rank=8, alpha=4.0, train_method="xattn"), dict(rank=2, alpha=1.0, train_method="full")]
    om = ounet.UNet2DConditionModel(getattr(ounet.UNetConfig, cfg)())
    torch.manual_seed(7)
    refs = []
    for s in specs:
        saved = list(lora.DEFAULT_TARGET_REPLACE)
        if s.get("network_type") == "c3lier":
            lora.DEFAULT_TARGET_REPLACE += lora.UNET_TARGET_REPLACE_MODULE_CONV
        try:
            refs.append(lora.LoRANetwork(om, rank=s["rank"], multiplier=1.0, alpha=s["alpha"],
                                         train_method=s["train_method"]))
        finally:
            del lora.DEFAULT_TARGET_REPLACE[len(saved):]
    pm, stack = _stack(specs, seed=7, unet=_unet(cfg))
    for ref, net in zip(refs, stack.sliders):
        rsd, sd = ref.state_dict(), net.state_dict()
        assert list(rsd.keys()) == list(sd.keys())
        for k in rsd:
            assert torch.equal(rsd[k], sd[k]), k


@pytest.mark.parametrize("ext", [".pt", ".safetensors"])
def test_slider_checkpoint_round_trip_in_reference_key_layout(tmp_path, ext):
    from sliders_b200 import io as sio

    pm, stack = _stack()
    _randomise(stack)
    plain_unet = _unet()
    for spec, net in zip(SPECS, stack.sliders):
        assert isinstance(net, plora.LoRANetwork)
        spec = dict(spec)
        conv = spec.pop("network_type", None) == "c3lier"
        saved = list(plora.DEFAULT_TARGET_REPLACE)
        if conv:
            plora.DEFAULT_TARGET_REPLACE += plora.UNET_TARGET_REPLACE_MODULE_CONV
        try:
            plain = plora.LoRANetwork(_unet(), **spec)
        finally:
            del plora.DEFAULT_TARGET_REPLACE[len(saved):]
        assert list(net.state_dict().keys()) == list(plain.state_dict().keys())
        assert all(k.startswith("lora_unet_") for k in net.state_dict())
        path = str(tmp_path / f"s{ext}")
        net.save_weights(path)
        sio.load_slider(plain, path)
        for k, v in net.state_dict().items():
            assert torch.equal(plain.state_dict()[k], v), k
        groups = net.prepare_optimizer_params()
        assert sum(p.numel() for p in groups[0]["params"]) == sum(p.numel() for p in net.parameters())
    _, other = _stack(unet=plain_unet)
    for src, dst in zip(stack.sliders, other.sliders):
        dst.load_state_dict(src.state_dict())
        assert all(torch.equal(a, b) for a, b in zip(src.state_dict().values(), dst.state_dict().values()))


# ---------------------------------------------------------------------------------------------------- refusals
def test_total_rank_over_16_is_refused():
    with pytest.raises(NotImplementedError, match="total rank 17"):
        _stack([dict(rank=8, train_method="xattn"), dict(rank=9, train_method="xattn")])


def test_stack_on_a_unet_with_a_network_is_refused():
    pm = _unet()
    plora.LoRANetwork(pm, rank=4, alpha=1.0, train_method="noxattn")
    with pytest.raises(RuntimeError, match="already carries a LoRANetwork"):
        plora.SliderStack(pm, SPECS)


def test_network_on_a_stack_is_refused():
    pm, stack = _stack()
    with pytest.raises(RuntimeError, match="cannot be built on a UNet that carries a SliderStack"):
        plora.LoRANetwork(pm, rank=4, alpha=1.0, train_method="noxattn")
    with pytest.raises(RuntimeError, match="already carries a SliderStack"):
        plora.SliderStack(pm, SPECS)
    # an adaptor hooked over the composite hook the way chained networks do (lora.py:103-106) is refused at lookup
    leaf = pm.mid_block.attentions[0].transformer_blocks[0].attn1.to_q
    a = plora.LoRAModule("chained", leaf, lora_dim=4)
    a.apply_to()
    with pytest.raises(RuntimeError, match="applied on top of a SliderStack"):
        _adaptor_of(leaf)


def test_slider_with_mixed_multipliers_is_refused():
    pm, stack = _stack()
    stack.sliders[1].name = "smile_rank8.pt"
    stack.sliders[1].unet_loras[3].multiplier = 0.5
    with pytest.raises(ValueError, match="smile_rank8.pt has modules with different multipliers"):
        stack.slider_multipliers()
    with pytest.raises(ValueError, match="smile_rank8.pt"):
        lp.scan(pm, 1)


def test_autograd_paths_with_an_active_stack_are_refused():
    from sliders_b200 import autograd as sb_autograd

    pm, stack = _stack()
    pm.requires_grad_(False)
    x = torch.zeros(1, 4, 32, 32)
    ehs = torch.zeros(1, 77, 256)
    added = {"text_embeds": torch.zeros(1, 128), "time_ids": torch.zeros(1, 6)}
    stack.set_lora_slider([1.0, -1.0])
    with stack:
        with pytest.raises(NotImplementedError, match="SliderStack slider is active"):
            pm(x, 1, encoder_hidden_states=ehs, added_cond_kwargs=added)           # trainable sliders
        stack.requires_grad_(False)
        with pytest.raises(NotImplementedError, match="SliderStack slider is active"):
            pm(x, 1, encoder_hidden_states=ehs.requires_grad_(True), added_cond_kwargs=added)
        with pytest.raises(NotImplementedError, match="active SliderStack"):
            sb_autograd._new_tape(lp.scan(pm, 1))
    # every slider off: nothing of the stack is active, so the engine would take the plain path
    snap = lp.scan(pm, 1)
    assert snap.stack_mults is None and not snap.needs_grad()


def test_composite_hook_raises_when_called_through_pytorch():
    pm, stack = _stack()
    leaf = pm.mid_block.attentions[0].transformer_blocks[0].attn2.to_k
    assert [i for i, _ in _hook_of(leaf).slider_entries] == [1]
    with pytest.raises(RuntimeError, match="called through PyTorch"):
        leaf(torch.zeros(1, leaf.in_features))


# ------------------------------------------------------------------------------------- scales and signatures
def test_stack_scales_and_context_manager():
    pm, stack = _stack()
    stack.set_lora_slider([2.0, -1.0])
    assert stack.slider_multipliers() == [1.0, 1.0]  # a fresh network runs at multiplier 1 until its first exit
    with stack:
        assert stack.slider_multipliers() == [2.0, -1.0]
    assert stack.slider_multipliers() == [0.0, 0.0]
    stack.set_lora_slider(scale=3.0)
    with stack:
        assert stack.slider_multipliers() == [3.0, 3.0]
    with pytest.raises(ValueError, match="3 scales for 2 sliders"):
        stack.set_lora_slider([1.0, 2.0, 3.0])


def _signature(pm):
    snap = lp.scan(pm, 1)
    return snap.signature, snap.common


def test_graph_signature_holds_structure_not_scales():
    pm, stack = _stack()
    plain_off = _signature(_unet())
    stack.__exit__(None, None, None)
    assert _signature(pm) == plain_off            # every slider at 0: the no-adaptor graph
    sigs = set()
    for scales in ([1.0, 0.0], [0.0, -2.0], [2.0, -1.0], [0.5, 0.5]):
        stack.set_lora_slider(scales)
        with stack:
            sig, common = _signature(pm)
            assert common is None
            sigs.add(sig)
    assert len(sigs) == 1 and sig != plain_off[0]


def test_cross_kv_sees_the_stack():
    pm, stack = _stack()
    stack.set_lora_slider([1.0, 0.0])
    with stack:
        # slider 1 (xattn) is at 0, but the composite graph is one for every scale: its to_k / to_v packs run
        assert pm._cross_kv_adapted()
    assert not pm._cross_kv_adapted()
    pm2, stack2 = _stack([dict(rank=4, alpha=1.0, train_method="noxattn")])
    with stack2:
        assert not pm2._cross_kv_adapted()


def test_shape_trace_stand_in_sees_the_composite_slot():
    import importlib.util

    spec = importlib.util.spec_from_file_location(
        "shape_trace", os.path.join(os.path.dirname(os.path.dirname(__file__)), "tools", "shape_trace.py"))
    st = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(st)
    pm, stack = _stack()
    pm._packer.begin(lp.scan(pm, 1), "cpu")
    lora = st._slot_plan(pm._packer)
    attn1 = pm.mid_block.attentions[0].transformer_blocks[0].attn1
    got = lora([attn1.to_q, attn1.to_k, attn1.to_v])
    assert (got.r, got.rt) == ops.lora_slots(12, 3)
    assert lora([pm.conv_in]) is None


# ------------------------------------------------------------------------------------------------ --compose
def test_compose_argument_parsing():
    from sliders_b200 import eval_sweep as es

    args = es.build_parser().parse_args(["--model_name", "age_rank4.pt", "--prompts_path", "p.csv", "--save_path", "o",
                                         "--compose", "smile_rank4.pt:-1.5", "--compose", "C:/m/x_rank8.pt:2"])
    assert args.compose == [("smile_rank4.pt", -1.5), ("C:/m/x_rank8.pt", 2.0)]
    assert es.build_parser().parse_args(["--model_name", "a", "--prompts_path", "p", "--save_path", "o"]).compose == []
    for bad in ("smile.pt", "smile.pt:x", ":1"):
        with pytest.raises(SystemExit):
            es.build_parser().parse_args(["--model_name", "a", "--prompts_path", "p", "--save_path", "o",
                                          "--compose", bad])


def test_compose_sweep_output_tree(tmp_path, monkeypatch):
    """The sweep with a stack: --model_name's scales make the tree, the composed sliders ride along at their fixed
    scales (the denoise loop is replaced by a recorder: this part runs without a GPU)."""
    from sliders_b200 import eval_sweep as es
    from sliders_b200 import generate

    pm = _unet()
    paths = []
    for name, spec in (("age_alpha1.0_rank4_noxattn_last.pt", SPECS[0]),
                       ("smile_alpha1.0_rank8_noxattn_last.pt", dict(rank=8, alpha=1.0, train_method="noxattn",
                                                                      network_type="c3lier"))):
        _, s = _stack([spec])
        _randomise(s)
        s.sliders[0].save_weights(str(tmp_path / name))
        paths.append(str(tmp_path / name))
    stack = plora.SliderStack.from_files(pm, paths)
    assert stack.ranks == (4, 8) and [n.name for n in stack.sliders] == paths
    seen = []

    def fake_loop(unet, network, scheduler, latents, *a, scale=0.0, **k):
        assert network is stack
        seen.append(scale)
        return latents + float(scale[0])

    monkeypatch.setattr(generate, "denoise_loop", fake_loop)
    csv_path = tmp_path / "p.csv"
    csv_path.write_text("case_number,prompt,evaluation_seed\n3,a,11\n")
    embeds = lambda p: (torch.zeros(2, 77, 256), torch.zeros(2, 128))  # noqa: E731
    from sliders_b200.scheduler import create_noise_scheduler

    save_dir = os.path.join(str(tmp_path / "out"), os.path.basename(paths[0]))
    n = es.sweep(pm, stack, create_noise_scheduler("euler"), es.read_prompts_csv(str(csv_path)), embeds, save_dir,
                 scales=(-2, 0, 2), num_samples=2, num_inference_steps=2, image_size=256, dtype=torch.float32,
                 fixed_scales=[-1.0])
    assert n == 6
    assert seen == [[-2, -1.0], [0, -1.0], [2, -1.0]]
    assert sorted(os.listdir(save_dir)) == ["-2", "0", "2"]
    assert sorted(os.listdir(os.path.join(save_dir, "2"))) == ["3_0.pt", "3_1.pt"]
