"""Dry-run the UNet forward on the meta device to list every kernel call with its shape, then (optionally)
join it with an ncu launch list (gpu__time_duration per launch, same order) to get a per-shape time table.
`trace(batch, train=True)` lists the training walk instead (tape kept: GEGLU unfused, attention keeps its lse).

    python tools/shape_trace.py 8 gpurun_out/launches_b8.csv
"""
import collections
import csv
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sliders_b200 import lora as plora  # noqa: E402
from sliders_b200 import ops  # noqa: E402
from sliders_b200.unet import UNet2DConditionModel, UNetConfig  # noqa: E402

calls = []  # (kernel_name, description, flops)
lora_rts = {}  # index in `calls` -> LoRA-down rows (sb200_lora.rt) of a call that carries adaptors


def _note_lora(lora):
    if lora is not None:
        lora_rts[len(calls) - 1] = lora.rt


def _slot_plan(packer):
    """Stand-in for `packer.lora` that packs nothing: the (slot width r, rt) of each call from the packer's own slot
    rule (LoraPacker.slots), which reads the walk's snapshot."""
    def lora(leaves):
        slots = packer.slots(leaves)
        return None if slots is None else types.SimpleNamespace(r=slots[0], rt=slots[1])

    return lora


def _meta(*shape):
    return torch.empty(shape, device="meta", dtype=torch.bfloat16)


def gemm(x, w, *, bias=None, rowbias=None, rows_per_batch=1, resid=None, geglu=False, lora=None, x1=None, out=None, bn=0):
    M, K0 = x.shape
    N, K = w.shape
    # b bias, R residual, G GEGLU, L LoRA, S split-K sources
    tag = "".join(c for c, f in (("b", bias is not None), ("R", resid is not None), ("G", geglu), ("L", lora is not None),
                                 ("S", x1 is not None)) if f)
    calls.append(("gemm_kernel", f"gemm M{M} N{N} K{K} {tag}", 2.0 * M * N * K))
    _note_lora(lora)
    return _meta(M, N // 2 if geglu else N)


def conv3x3(x0, w, *, x1=None, stride=1, bias=None, rowbias=None, resid=None, lora=None, bn=0):
    B, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    Cout = w.shape[0]
    tag = "".join(c for c, f in (("t", rowbias is not None), ("R", resid is not None), ("L", lora is not None),
                                 ("S", x1 is not None)) if f)
    calls.append(("gemm_kernel", f"conv {H}x{W} C{C0 + C1}->{Cout} s{stride} {tag} (M{B * H * W // stride ** 2} K{9 * (C0 + C1)})",
                  2.0 * B * (H // stride) * (W // stride) * Cout * 9 * (C0 + C1)))
    _note_lora(lora)
    return _meta(B, H // stride, W // stride, Cout)


def attention(q, k, v, B, heads, Sq, Skv, scale, head_dim=64, lse=None):
    keep = " lse" if lse is not None else ""
    calls.append(("attention_kernel", f"attn B{B} h{heads} Sq{Sq} Skv{Skv}{keep}", 4.0 * B * heads * Sq * Skv * 64))
    return _meta(B * Sq, heads * 64)


def geglu(pre):
    M, F2 = pre.shape
    calls.append(("geglu_kernel", f"geglu M{M} N{F2 // 2}", 0.0))
    return _meta(M, F2 // 2)


def groupnorm(x0, gamma, beta, groups, eps, silu, *, x1=None, stats_ws=None):
    C = x0.shape[-1] + (x1.shape[-1] if x1 is not None else 0)
    d = f"gn {tuple(x0.shape[:-1])} C{C}"
    for k in ("gn_stats_kernel", "gn_finalize_kernel", "gn_apply_kernel"):
        calls.append((k, d, 0.0))
    return _meta(*x0.shape[:-1], C)


def layernorm(x, gamma, beta, eps=1e-5):
    calls.append(("layernorm_kernel", f"ln M{x.shape[0]} C{x.shape[1]}", 0.0))
    return _meta(*x.shape)


def small_linear(x, w, bias=None, *, act_in=False, act_out=0, lora=None, resid=None):
    tag = " L" if lora is not None else ""
    calls.append(("small_linear_kernel", f"small_linear M{x.shape[0]} N{w.shape[0]} K{x.shape[1]}{tag}", 0.0))
    _note_lora(lora)
    return _meta(x.shape[0], w.shape[0])


def sinusoid(values, dim):
    calls.append(("sinusoid_kernel", f"sinusoid n{values.numel()} dim{dim}", 0.0))
    return _meta(values.numel(), dim)


def conv_in(latent, w, bias):
    B, _, H, W = latent.shape
    calls.append(("conv_in_kernel", f"conv_in {H}x{W}", 0.0))
    return _meta(B, H, W, w.shape[0])


def conv_out(x, w, bias, out_dtype=torch.bfloat16):
    B, H, W, _ = x.shape
    calls.append(("conv_out_kernel", f"conv_out {H}x{W}", 0.0))
    return _meta(B, 4, H, W)


def upsample2x(x):
    B, H, W, C = x.shape
    calls.append(("upsample2x_kernel", f"upsample {H}x{W} C{C}", 0.0))
    return _meta(B, 2 * H, 2 * W, C)


def trace(batch, with_lora=True, train=False, extra_targets=(), rank=4):
    """The launch plan of one SDXL forward: the inference walk, or with `train` the training walk (tape kept).  The
    LoRA network is `noxattn` of rank `rank` on the default targets plus the conv targets (c3lier) plus
    `extra_targets`; `lora_rts` then maps each call that carries adaptors to its LoRA-down rows."""
    calls.clear()
    lora_rts.clear()
    for name in ("gemm", "conv3x3", "attention", "geglu", "groupnorm", "layernorm", "small_linear", "sinusoid",
                 "conv_in", "conv_out", "upsample2x"):
        setattr(ops, name, globals()[name])
    with torch.device("meta"):
        unet = UNet2DConditionModel(UNetConfig.sdxl()).to(torch.bfloat16)
        net = None
        if with_lora:
            saved = list(plora.DEFAULT_TARGET_REPLACE)
            plora.DEFAULT_TARGET_REPLACE += plora.UNET_TARGET_REPLACE_MODULE_CONV + list(extra_targets)
            net = plora.LoRANetwork(unet, rank=rank, multiplier=1.0, alpha=1.0, train_method="noxattn")
            del plora.DEFAULT_TARGET_REPLACE[len(saved):]
        unet._packer.lora = _slot_plan(unet._packer)
        x = torch.empty(batch, 4, 128, 128, dtype=torch.float32)
        t = torch.empty(batch, dtype=torch.float32)
        ehs = torch.empty(batch, 77, 2048, dtype=torch.bfloat16)
        added = {"text_embeds": torch.empty(batch, 1280, dtype=torch.bfloat16),
                 "time_ids": torch.empty(batch, 6, dtype=torch.float32)}
        unet._walk(x, t, ehs, added, torch.float32, [] if train else None)
    return list(calls)


def main():
    batch = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    tr = trace(batch)
    print(f"{len(tr)} kernel launches per forward at batch {batch}")
    if len(sys.argv) <= 2:
        agg = collections.Counter(d for _, d, _ in tr)
        for d, n in agg.most_common():
            print(f"{n:4d}  {d}")
        return
    rows = []
    with open(sys.argv[2]) as f:
        lines = [l for l in f if not l.startswith("==")]
    for row in csv.DictReader(lines):
        if row.get("Metric Name", "gpu__time_duration.sum") != "gpu__time_duration.sum":
            continue
        name = row["Kernel Name"].split("(")[0].replace("sb200::", "").replace("void ", "").split("<")[0]
        v = float(row["Metric Value"].replace(",", ""))
        v = v / 1e3 if row["Metric Unit"] == "ns" else (v * 1e3 if row["Metric Unit"] == "ms" else v)
        if name.startswith("at::"):
            continue
        rows.append((name, v))
    assert len(rows) == len(tr), (len(rows), len(tr))
    agg = collections.OrderedDict()
    for (kname, desc, fl), (nname, us) in zip(tr, rows):
        assert kname.startswith(nname) or nname.startswith(kname.split("_kernel")[0]), (kname, nname)
        a = agg.setdefault(desc if kname in ("gemm_kernel", "attention_kernel") else kname, [0, 0.0, 0.0])
        a[0] += 1
        a[1] += us
        a[2] += fl
    total = sum(a[1] for a in agg.values())
    print(f"total {total / 1e3:.2f} ms (ncu-serialised)")
    for d, (n, us, fl) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        tf = fl / us / 1e6 if fl else 0.0
        print(f"{n:4d} x {us / n:8.1f} us = {us / 1e3:7.2f} ms {100 * us / total:5.1f}%  {tf:6.0f} TF/s  {d}")


if __name__ == "__main__":
    main()
