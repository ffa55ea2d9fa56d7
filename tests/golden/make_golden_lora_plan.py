"""Generates tests/golden/lora_plan.pt — runs on CPU, no reference needed:

    python tests/golden/make_golden_lora_plan.py

The LoRA launch plan of the UNet walk: for every kernel call of `UNet2DConditionModel._walk`, in order, the op name
and, when the call carries adaptors, every field of its `ops.Lora` (r, rt, group_n, scale, the value of scale_dev, the
per-sample vector, rows_per_sample and hashes of the down / up bytes), plus each `lora_compose` with a hash of what it
wrote.  The kernels are replaced by stand-ins that return correctly shaped tensors and `lora_compose` by
`out.copy_(raw * mult)`, so the walk runs on CPU and only the LoRA packing is real.  Scenarios: no adaptors, rank 4
at scales 1 and 0, ranks 3 and 16, differing per-module multipliers, c3lier with the conv rank clamp, per-sample
values at two batch sizes, a SliderStack at three scale vectors, a training walk with its tape's `scales` record, and
the capture and scale-baking modes after a warm eager walk, each followed by a graph replay's refresh at new scales.
tests/test_lora_plan_host.py replays every scenario and requires the same record.
"""
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import unet as ounet  # noqa: E402
from sliders_b200 import autograd as sb_autograd  # noqa: E402
from sliders_b200 import lora as plora  # noqa: E402
from sliders_b200 import lora_pack as lp  # noqa: E402
from sliders_b200 import ops  # noqa: E402
from sliders_b200.unet import UNet2DConditionModel, UNetConfig, _GraphInputs  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lora_plan.pt")
BF16 = torch.bfloat16

events = []


def _hash(t):
    return hashlib.sha1(t.detach().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()[:16]


def _note(name, lora):
    if lora is None:
        events.append(name)
        return
    events.append((name, lora.r, lora.rt, lora.group_n, lora.scale,
                   None if lora.scale_dev is None else lora.scale_dev.tolist(),
                   None if lora.sample_scale is None else lora.sample_scale.tolist(),
                   lora.rows_per_sample, _hash(lora.down), _hash(lora.up)))


# stand-ins for the kernels: output shapes only
def gemm(x, w, *, bias=None, rowbias=None, rows_per_batch=1, resid=None, geglu=False, lora=None, x1=None, out=None,
         bn=0):
    _note("gemm", lora)
    return torch.zeros(x.shape[0], w.shape[0] // 2 if geglu else w.shape[0], dtype=BF16)


def conv3x3(x0, w, *, x1=None, stride=1, bias=None, rowbias=None, resid=None, lora=None, bn=0):
    _note("conv3x3", lora)
    B, H, W, _ = x0.shape
    return torch.zeros(B, H // stride, W // stride, w.shape[0], dtype=BF16)


def small_linear(x, w, bias=None, *, act_in=False, act_out=0, lora=None, resid=None):
    _note("small_linear", lora)
    return torch.zeros(x.shape[0], w.shape[0], dtype=BF16)


def attention(q, k, v, B, heads, Sq, Skv, scale, head_dim=64, lse=None):
    return torch.zeros(B * Sq, q.shape[1], dtype=BF16)


def geglu(pre):
    return torch.zeros(pre.shape[0], pre.shape[1] // 2, dtype=BF16)


def groupnorm(x0, gamma, beta, groups, eps, silu, *, x1=None, stats_ws=None):
    C = x0.shape[-1] + (x1.shape[-1] if x1 is not None else 0)
    return torch.zeros(*x0.shape[:-1], C, dtype=BF16)


def layernorm(x, gamma, beta, eps=1e-5):
    return torch.zeros_like(x)


def sinusoid(values, dim):
    return torch.zeros(values.numel(), dim, dtype=BF16)


def conv_in(latent, w, bias):
    B, _, H, W = latent.shape
    return torch.zeros(B, H, W, w.shape[0], dtype=BF16)


def conv_out(x, w, bias, out_dtype=BF16):
    B, H, W, _ = x.shape
    return torch.zeros(B, 4, H, W, dtype=out_dtype)


def upsample2x(x):
    B, H, W, C = x.shape
    return torch.zeros(B, 2 * H, 2 * W, C, dtype=x.dtype)


def lora_compose(raw, col_mult, out=None):
    out.copy_(raw * col_mult)
    events.append(("lora_compose", _hash(out)))
    return out


STUBS = ("gemm", "conv3x3", "small_linear", "attention", "geglu", "groupnorm", "layernorm", "sinusoid", "conv_in",
         "conv_out", "upsample2x", "lora_compose")


class stubbed_ops:
    """Swaps the kernel wrappers of sliders_b200.ops for the stand-ins above while the block runs."""

    def __enter__(self):
        self.saved = {n: getattr(ops, n) for n in STUBS}
        for n in STUBS:
            setattr(ops, n, globals()[n])

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(ops, n, f)


# ------------------------------------------------------------------------------------------------ the UNet's modes
def walk(unet, inputs, tape=None, capture=False, bake=False):
    x, t, ehs, added = inputs
    unet._walk(x, t, ehs, added, torch.float32, tape, capture=capture, bake=bake)


def replay_load(unet, inputs, bake=False):
    """What a graph replay does before the graph runs."""
    x, t, ehs, added = inputs
    _GraphInputs(x, t, ehs, added).load(unet, x, t, ehs, added, lp.scan(unet, x.shape[0]), bake)


def new_tape(unet, B):
    return sb_autograd._new_tape(lp.scan(unet, B))


# ------------------------------------------------------------------------------------------------------ scenarios
def make_unet(cfg, micro=False):
    d = dict(getattr(ounet.UNetConfig, cfg)().__dict__)
    if micro:  # conv channels below rank 16, so c3lier's conv adaptors are clamped (lora.py:78)
        d.update(block_out_channels=(8,) + (16,) * (len(d["block_out_channels"]) - 1), norm_num_groups=4)
    torch.manual_seed(0)
    return UNet2DConditionModel(UNetConfig.from_dict(d))


def inputs(unet, B):
    c = unet.config
    g = torch.Generator().manual_seed(B)
    added = None
    if c.addition_embed_type == "text_time":
        added = {"text_embeds": torch.randn(B, c.projection_class_embeddings_input_dim - 6 * c.addition_time_embed_dim,
                                            generator=g).to(BF16),
                 "time_ids": torch.randn(B, 6, generator=g)}
    return (torch.randn(B, 4, 16, 16, generator=g), torch.full((B,), 500.0),
            torch.randn(B, 77, c.cross_attention_dim, generator=g).to(BF16), added)


def randomise(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if "lora_" in name:
                p.copy_(torch.randn(p.shape, generator=g).to(BF16).float())


def network(unet, rank, alpha=1.0, method="noxattn", conv=False, seed=1):
    saved = list(plora.DEFAULT_TARGET_REPLACE)
    if conv:
        plora.DEFAULT_TARGET_REPLACE += plora.UNET_TARGET_REPLACE_MODULE_CONV
    try:
        torch.manual_seed(seed)
        net = plora.LoRANetwork(unet, rank=rank, multiplier=1.0, alpha=alpha, train_method=method)
    finally:
        del plora.DEFAULT_TARGET_REPLACE[len(saved):]
    randomise(net, seed)
    return net.requires_grad_(False)


def scalar(cfg, rank, scale, method="noxattn", conv=False, alpha=1.0, micro=False):
    unet = make_unet(cfg, micro)
    net = network(unet, rank, alpha=alpha, method=method, conv=conv)
    net.set_lora_slider(scale)
    with net:
        walk(unet, inputs(unet, 2))


def no_adaptors(cfg):
    unet = make_unet(cfg)
    walk(unet, inputs(unet, 2))


def folded(cfg, capture=False):
    """Per-module multipliers: every third adaptor at 0.5, one at 0, the rest at 1.5."""
    unet = make_unet(cfg)
    net = network(unet, 4, method="full", conv=True)
    with net:
        for i, a in enumerate(net.unet_loras):
            a.multiplier = 0.0 if i == 1 else 0.5 if i % 3 == 0 else 1.5
        x = inputs(unet, 2)
        walk(unet, x)
        if capture:  # a graph with differing factors folds them into the packs
            walk(unet, x, bake=True)
            walk(unet, x, capture=True, bake=True)
            net.unet_loras[0].multiplier = -2.0
            replay_load(unet, x, bake=True)
            walk(unet, x, capture=True, bake=True)


def per_sample(cfg, capture=False):
    unet = make_unet(cfg)
    net = network(unet, 4, method="full")
    net.set_lora_slider([1.0, -2.0])
    with net:
        walk(unet, inputs(unet, 2))
        x = inputs(unet, 4)
        walk(unet, x)
        if capture:
            walk(unet, x, capture=True)
            net.set_lora_slider([0.5, 3.0])
            net.__enter__()
            replay_load(unet, x)
            walk(unet, x, capture=True)


def stack(cfg, capture=False):
    unet = make_unet(cfg)
    torch.manual_seed(3)
    st = plora.SliderStack(unet, [dict(rank=4, alpha=1.0, train_method="noxattn", network_type="c3lier"),
                                  dict(rank=8, alpha=4.0, train_method="xattn")])
    randomise(st, 3)
    x = inputs(unet, 2)
    for v in ([2.0, -1.0], [1.0, 0.0], [0.0, 0.0]):
        st.set_lora_slider(v)
        with st:
            walk(unet, x)
    if capture:
        st.set_lora_slider([2.0, -1.0])
        with st:
            walk(unet, x)
            walk(unet, x, capture=True)
        st.set_lora_slider([-0.5, 1.5])
        with st:
            replay_load(unet, x)
            walk(unet, x, capture=True)


def capture_scalar(cfg):
    unet = make_unet(cfg)
    net = network(unet, 4, conv=True)
    x = inputs(unet, 2)
    with net:
        walk(unet, x)
        walk(unet, x, capture=True)
        net.set_lora_slider(2.0)
        net.__enter__()
        replay_load(unet, x)
        walk(unet, x, capture=True)


def training(cfg):
    unet = make_unet(cfg)
    net = network(unet, 4, method="full", conv=True)
    net.unet_loras[2].requires_grad_(True)
    net.unet_loras[5].requires_grad_(True)
    x = inputs(unet, 2)
    net.set_lora_slider(1.5)
    with net:
        net.unet_loras[4].multiplier = 0.0
        tape = new_tape(unet, 2)
        walk(unet, x, tape)
    names = {id(m): n for n, m in unet.named_modules()}
    scales = tape[0][1]
    events.append(("scales", [(names[k], a.lora_name, s, tr) for k, (a, s, tr) in scales.items()]))
    events.append(("tape", [kind for kind, _ in tape]))


SCENARIOS = {
    "none": lambda cfg: no_adaptors(cfg),
    "rank4_scale1": lambda cfg: scalar(cfg, 4, 1.0),
    "rank4_scale0": lambda cfg: scalar(cfg, 4, 0.0),
    "rank3": lambda cfg: scalar(cfg, 3, -1.5, method="full", alpha=2.0),
    "rank16": lambda cfg: scalar(cfg, 16, 0.75, method="full", conv=True, alpha=4.0),
    "folded": lambda cfg: folded(cfg),
    "c3lier_clamp": lambda cfg: scalar(cfg, 16, 1.25, conv=True, alpha=8.0, micro=True),
    "per_sample": lambda cfg: per_sample(cfg),
    "stack": lambda cfg: stack(cfg),
    "training": lambda cfg: training(cfg),
    "capture_scalar": lambda cfg: capture_scalar(cfg),
    "capture_per_sample": lambda cfg: per_sample(cfg, capture=True),
    "capture_stack": lambda cfg: stack(cfg, capture=True),
    "bake_folded": lambda cfg: folded(cfg, capture=True),
}
CONFIGS = ("tiny_sd", "tiny_xl")


def record(cfg, name):
    events.clear()
    with stubbed_ops():
        SCENARIOS[name](cfg)
    return list(events)


def main():
    import contextlib
    import io

    fx = {}
    for cfg in CONFIGS:
        for name in SCENARIOS:
            with contextlib.redirect_stdout(io.StringIO()):
                fx[(cfg, name)] = record(cfg, name)
            print(cfg, name, len(fx[(cfg, name)]), "events")
    torch.save(fx, OUT)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
