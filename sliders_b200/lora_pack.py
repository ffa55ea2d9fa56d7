"""LoRA state of the UNet forward, between the adaptors of sliders_b200.lora and the `ops.Lora` the fused kernels read.

`scan` reads a UNet's adaptors once per forward into a `Snapshot` and raises on every state the kernels cannot run.  A
UNet's `LoraPacker` turns the snapshot into the `ops.Lora` of each fused call of the walk and owns the device buffers
behind them.  Both the reference lora.py and sliders_b200.lora replace `leaf.forward` by a bound method of the adaptor
(lora.py:103-106), which is how a leaf's adaptor is found; a SliderStack installs one composite hook per leaf instead.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import ops
from .ops import BF16, Lora


# --------------------------------------------------------------------------------------------------------- discovery
def adaptor_of(leaf: nn.Module):
    fwd = leaf.__dict__.get("forward")
    owner = getattr(fwd, "__self__", None)
    if owner is not None and hasattr(owner, "lora_down") and hasattr(owner, "lora_up"):
        inner = getattr(getattr(owner, "org_forward", None), "__self__", None)
        if inner is not None and hasattr(inner, "slider_entries"):
            raise RuntimeError(f"{getattr(owner, 'lora_name', 'leaf')}: a LoRANetwork was applied on top of a "
                               "SliderStack; the stack's composite hook owns this leaf, so add the slider to the stack")
        if inner is not None and hasattr(inner, "lora_down"):
            # the reference chains `org_forward`, so two networks on one UNet both apply there; the fused kernels carry
            # one adaptor per leaf — refuse loudly instead of silently dropping the first network
            raise RuntimeError(f"{getattr(owner, 'lora_name', 'leaf')}: a second LoRANetwork was applied to a UNet that "
                               "already carries one; merge the sliders' weights or build the second network on another "
                               "UNet2DConditionModel (parameters can be shared with load_state_dict(assign=True))")
        return owner
    return None


def hook_of(leaf: nn.Module):
    """The composite hook a SliderStack installed on `leaf` (sliders_b200.lora.SliderHook), or None."""
    owner = getattr(leaf.__dict__.get("forward"), "__self__", None)
    return owner if owner is not None and hasattr(owner, "slider_entries") else None


def adapted_leaves(model: nn.Module) -> List[tuple]:
    """(leaf, adaptor) of every adapted Linear / Conv2d of `model`, in module order (leaf list cached on the model)."""
    cache = model.__dict__.get("_adapted_cache")
    if cache is None:
        cache = [m for m in model.modules() if isinstance(m, (nn.Linear, nn.Conv2d))]
        model.__dict__["_adapted_cache"] = cache
    return [(m, a) for m in cache for a in (adaptor_of(m),) if a is not None]


def _common(factors) -> Optional[float]:
    """The factor all non-zero `factors` share, or None (all 0, or differing: per-module multipliers or a conv rank
    clamp changing alpha / r; `with network:` / `set_lora_slider` alone give one factor, lora.py:249-258)."""
    nz = [s for s in factors if s != 0.0]
    return nz[0] if nz and all(abs(s - nz[0]) < 1e-12 for s in nz) else None


# ---------------------------------------------------------------------------------------------------------- snapshot
@dataclass(frozen=True)
class Snapshot:
    """The adaptors of one UNet forward, read once by `scan`."""

    batch: Optional[int]              # samples of the call; None outside a call
    adaptors: Dict[int, tuple]        # id(leaf) -> (adaptor, multiplier * alpha / r, trainable), every adapted leaf
    sample_values: Optional[tuple]    # per-sample slider values of the active adaptors (set_lora_slider of a sequence)
    stack: object                     # the UNet's SliderStack, or None
    stack_mults: Optional[tuple]      # its per-slider multipliers; None when it is absent or every slider is at 0
    common: Optional[float]           # the factor shared by every active adaptor, or None
    # Which adaptors contribute is baked into a captured graph, and so are differing factors; a common factor is a
    # device-side scalar.  The ranks set the sizes of the packs a graph reads; a per-sample graph reads a vector the
    # scalar graph does not.  A stack's holds its layout, not its (device-side) multipliers: one graph for all scales.
    signature: tuple

    def active(self, leaf: nn.Module) -> bool:
        """True when `leaf` runs an adaptor: its own at a non-zero factor, or its composite hook while any slider is on
        (one composite graph serves every scale, so a hooked leaf runs its pack even with its slider at 0)."""
        if self.stack_mults is not None and hook_of(leaf) is not None:
            return True
        return id(leaf) in self.adaptors and self.adaptors[id(leaf)][1] != 0.0

    def needs_grad(self) -> bool:
        """True when an active adaptor (multiplier != 0, i.e. inside `with network:`) has trainable weights."""
        if any(s != 0.0 and trainable for _, s, trainable in self.adaptors.values()):
            return True
        return self.stack_mults is not None and any(m != 0.0 and any(p.requires_grad for p in net.parameters())
                                                    for net, m in zip(self.stack.sliders, self.stack_mults))


def scan(model: nn.Module, batch: Optional[int]) -> Snapshot:
    """The adaptors of `model` (a UNet, or any module holding adapted leaves) for a call with `batch` samples (None:
    outside a call, so the batch is not checked against per-sample values)."""
    adapted = adapted_leaves(model)
    stack = model.__dict__.get("_slider_stack")
    mults = None
    if stack is not None:
        if adapted:
            raise RuntimeError("sliders_b200: a LoRANetwork was applied to a UNet that carries a SliderStack; add the "
                               "slider to the stack instead")
        mults = tuple(stack.slider_multipliers())
        if all(m == 0.0 for m in mults):
            mults = None
    adaptors, values = {}, None
    for leaf, a in adapted:
        s = float(a.multiplier) * float(a.scale)
        adaptors[id(leaf)] = (a, s, bool(a.lora_down.weight.requires_grad))
        v = getattr(a, "sample_scales", None)
        if v is None or s == 0.0:
            continue
        if values is not None and v != values:
            raise ValueError("sliders_b200: active adaptors carry different per-sample slider values")
        values = v
    if values is not None and batch is not None and batch % len(values) != 0:
        raise ValueError(f"sliders_b200: a batch of {batch} is not a multiple of the {len(values)} per-sample slider "
                         "values")
    factors = [s for _, s, _ in adaptors.values()]
    on = tuple(s != 0.0 for s in factors)
    ranks = (tuple(int(a.lora_dim) for _, a in adapted),
             any(getattr(a, "sample_scales", None) is not None for _, a in adapted))
    common = _common(factors)
    if mults is not None:
        signature, common = (on, ranks, None, stack.structure), None
    else:
        signature = (on, ranks, tuple(factors) if common is None and any(on) else None)
    return Snapshot(batch, adaptors, values, stack, mults, common, signature)


# ------------------------------------------------------------------------------------------------------ pack buffers
def _fill_composite(down: torch.Tensor, raw: torch.Tensor, leaves, hooks, offsets, rp: int) -> None:
    """Writes the sliders of one fused call into zeroed packs: leaf gi's slider i takes down rows
    [gi * rp + o_i, + r) and raw up columns [o_i, o_i + r) of the leaf's output rows, with its alpha / r (the conv rank
    clamp of lora.py:78 included) folded in; r is the adaptor's own rank, so a leaf a slider does not adapt, and the
    columns past a clamped rank, keep zeros."""
    n0 = 0
    for gi, (leaf, h) in enumerate(zip(leaves, hooks)):
        n1 = n0 + leaf.weight.shape[0]
        for i, a in (h.slider_entries if h is not None else ()):
            d = a.lora_down.weight.detach()
            if d.dim() == 4:
                d = d.permute(0, 2, 3, 1)
            rr = d.shape[0]
            c0 = offsets[i]
            down[gi * rp + c0: gi * rp + c0 + rr].copy_(d.reshape(rr, -1))
            u = a.lora_up.weight.detach().reshape(leaf.weight.shape[0], -1)
            raw[n0:n1, c0:c0 + rr].copy_(u.float() * float(a.scale))
        n0 = n1


def _fill_sample_vec(vec: torch.Tensor, factor: float, values: tuple) -> None:
    """vec[b] = fp32(values[b % n] * factor), with one fill per run of equal entries: kernel launches with the value
    as an argument, so the host never waits for the stream (a copy from pageable host memory would)."""
    n = len(values)
    entries = [values[b % n] * factor for b in range(vec.numel())]
    b0 = 0
    for b in range(1, len(entries) + 1):
        if b == len(entries) or entries[b] != entries[b0]:
            vec[b0:b].fill_(entries[b0])
            b0 = b


class _LoraPack:
    """Packed (down [rt,K], up [N,r]) buffers of one fused call site over `leaves`; repacked only when a parameter
    changes.  A composite pack (SliderStack) also keeps `raw`: the sliders' up columns with alpha / r folded in, before
    the runtime multipliers; `up` is then the effective pack sb200_lora_compose writes."""

    def __init__(self, leaves):
        self.leaves = list(leaves)
        self.key = self.down = self.up = self.raw = None


class _StackArena:
    """Device state of a UNet's SliderStack.  Every composite pack's raw and effective up columns are row slices of one
    fp32 arena each, so a single sb200_lora_compose launch per forward applies the per-column multipliers `mult` (one
    fp32 value per slot column: slider i's multiplier on its columns [o_i, o_i + r_i), 0 on padding)."""

    def __init__(self, stack, device):
        self.stack = stack
        self.rp = ops.lora_slots(stack.total_rank)[0]
        self.mult = torch.zeros(self.rp, device=device, dtype=torch.float32)
        self.packs: List[_LoraPack] = []
        self.raw = self.eff = None
        self.dirty = False

    def load(self, mults) -> None:
        """Writes the multipliers into `mult` with one fill per slider: kernel launches with the value as an argument, so
        the host never waits for the stream (a copy from pageable host memory would)."""
        for o, r, m in zip(self.stack.offsets, self.stack.ranks, mults):
            self.mult[o:o + r].fill_(float(m))

    def settle(self) -> bool:
        """Moves packs built since the last call into a new arena; True when packs that a captured graph may read
        moved (there was an arena before)."""
        if not self.dirty:
            return False
        moved = self.raw is not None
        rows = sum(p.raw.shape[0] for p in self.packs)
        dev = self.packs[0].raw.device
        raw = torch.empty((rows, self.rp), device=dev, dtype=torch.float32)
        eff = torch.empty((rows, self.rp), device=dev, dtype=torch.float32)
        n0 = 0
        for p in self.packs:
            n1 = n0 + p.raw.shape[0]
            raw[n0:n1].copy_(p.raw)
            eff[n0:n1].copy_(p.up)
            p.raw, p.up = raw[n0:n1], eff[n0:n1]
            n0 = n1
        self.raw, self.eff, self.dirty = raw, eff, False
        return moved


# ------------------------------------------------------------------------------------------------------------ packer
class LoraPacker:
    """The packed LoRA buffers of one UNet.  A walk runs `begin`, `lora(leaves)` at every fused call, then `end`.
    Graph modes: under `capture` nothing new is allocated and the values a replay changes (common factor, per-sample
    vectors, slider multipliers) are left to `refresh`, run before every replay; under `bake` every factor is folded
    into the packed up weights and the kernels run with scale 1 (adaptors whose factors differ between call sites have
    no single device-side factor).  `drop_graphs` is called when buffers captured graphs read are replaced."""

    def __init__(self, drop_graphs: Callable[[], None]):
        self._drop_graphs = drop_graphs
        self.reset()

    def reset(self) -> None:
        """Forgets every buffer (the UNet's parameters were moved or converted)."""
        self.packs: Dict[tuple, _LoraPack] = {}
        self.scale_dev: Optional[torch.Tensor] = None
        # per-sample slider values: one fp32 vector per (batch, adaptor factor), entry b = value[b % n] * factor
        self.sample_vecs: Dict[tuple, torch.Tensor] = {}
        self.arena: Optional[_StackArena] = None
        self.snap: Optional[Snapshot] = None
        self.device = None
        self.capture = self.bake = False
        self.filled: set = set()

    def begin(self, snap: Snapshot, device, capture: bool = False, bake: bool = False) -> None:
        """Start of a walk: with the stack on, the current multipliers go to the device vector and, once the packs are
        in their arena, one sb200_lora_compose writes every effective up pack."""
        self.snap, self.device, self.capture, self.bake = snap, device, capture, bake
        self.filled = set()
        if snap.stack_mults is None:
            return
        if self.arena is None:
            self.arena = _StackArena(snap.stack, device)
        if not capture:  # replays get the vector from `refresh`
            self.arena.load(snap.stack_mults)
        if self.arena.raw is not None:
            ops.lora_compose(self.arena.raw, self.arena.mult, out=self.arena.eff)

    def end(self) -> None:
        """End of a walk: composite packs built during it move into the stack's arena."""
        if self.arena is not None and not self.capture and self.arena.settle():
            self._drop_graphs()  # graphs captured before hold the packs' old buffers
        self.snap = None

    def slots(self, leaves: List[nn.Module]) -> Optional[Tuple[int, int]]:
        """(slot width, LoRA-down rows) of the fused call over `leaves` (ops.lora_slots; a stack's slot is as wide as
        its total rank), or None when no leaf is adapted or every factor is 0 (outside `with network:`, lora.py:256)."""
        snap = self.snap
        if snap.stack_mults is not None:
            if all(hook_of(l) is None for l in leaves):
                return None
            rp = ops.lora_slots(snap.stack.total_rank)[0]
            return rp, ops.lora_slots(rp, len(leaves))[1]
        ents = [snap.adaptors.get(id(l)) for l in leaves]
        if all(e is None or e[1] == 0.0 for e in ents):
            return None
        return ops.lora_slots(max(int(e[0].lora_dim) for e in ents if e is not None), len(leaves))

    def lora(self, leaves: List[nn.Module]) -> Optional[Lora]:
        """sb200_lora for one fused call over `leaves` (all sharing the same input), or None when it runs no adaptor.
        Outside a walk the call reads the adaptors of its own leaves."""
        if self.snap is None:
            self.begin(scan(nn.ModuleList(leaves), None), leaves[0].weight.device)
            try:
                return self.lora(leaves)
            finally:
                self.snap = None
        group_n = leaves[0].weight.shape[0]
        if self.snap.stack_mults is not None:
            pack = self._composite(leaves)
            return None if pack is None else Lora(pack.down, pack.up, self.arena.rp, group_n, 1.0)
        site = self._plain(leaves)
        if site is None:
            return None
        pack, r, common = site
        if self.snap.sample_values is not None:
            # per-sample values: the factor common to the call site (1 when folded into `up`) goes into the vector, so
            # a constant vector reproduces the scalar path's fp32 scale exactly
            vec = self._sample_vec(common if common is not None else 1.0)
            return Lora(pack.down, pack.up, r, group_n, 1.0, sample_scale=vec)
        if self.scale_dev is None:
            self.scale_dev = torch.ones(1, device=leaves[0].weight.device, dtype=torch.float32)
        if self.capture and common is not None:
            # graph mode: the common scale is read from device memory at replay time
            return Lora(pack.down, pack.up, r, group_n, 1.0, self.scale_dev)
        return Lora(pack.down, pack.up, r, group_n, common if common is not None else 1.0)

    def refresh(self, snap: Snapshot, bake: bool = False) -> None:
        """Before a graph replay: the snapshot's factors go to the device buffers the graph reads, and packs whose
        adaptor weights the optimiser changed are rebuilt in place (same storage, so the graph sees them)."""
        if self.scale_dev is not None:
            self.scale_dev.fill_(1.0 if snap.common is None else snap.common)
        if snap.stack_mults is not None:
            self.arena.load(snap.stack_mults)  # the graph's own compose applies them
        if snap.sample_values is not None:
            for (B, factor), vec in self.sample_vecs.items():
                if B == snap.batch:
                    _fill_sample_vec(vec, factor, snap.sample_values)
        self.snap, self.capture, self.bake = snap, False, bake
        repack = self._composite if snap.stack_mults is not None else self._plain
        for pack in list(self.packs.values()):
            repack(pack.leaves)
        self.snap = None

    def _plain(self, leaves):
        """(pack, slot width, factor common to the call site or None) of a call site of plain adaptors, repacked if a
        weight, or a factor folded into `up`, changed; None when the call runs no adaptor."""
        slots = self.slots(leaves)
        if slots is None:
            return None
        r, rt = slots
        ents = [self.snap.adaptors.get(id(l), (None, 0.0)) for l in leaves]
        adaptors, scales = [e[0] for e in ents], [e[1] for e in ents]
        # with `bake`, every factor is folded into the packed up-weights instead and the kernels run with scale 1
        common = None if self.bake else _common(scales)
        pack = self.packs.setdefault(tuple(id(l) for l in leaves), _LoraPack(leaves))
        ver = tuple((a.lora_down.weight.data_ptr(), a.lora_down.weight._version, a.lora_up.weight.data_ptr(),
                     a.lora_up.weight._version) if a is not None else None for a in adaptors)
        ver = (ver, None if common is not None else tuple(scales))
        if pack.key != ver:
            dev = leaves[0].weight.device
            K = leaves[0].weight[0].numel()
            N = sum(l.weight.shape[0] for l in leaves)
            if pack.down is None or pack.down.shape != (rt, K) or pack.up.shape != (N, r):
                # adaptor gi takes down rows [gi * r, +r) and up columns [0, r) with r the slot width (ops.lora_slots);
                # the rows and columns beyond its own rank stay zero
                if pack.down is not None:  # another slot width: captured graphs hold the old buffers
                    if self.capture:
                        raise RuntimeError("sliders_b200: the LoRA slot width changed while a CUDA graph was captured")
                    self._drop_graphs()
                pack.down = torch.zeros((rt, K), device=dev, dtype=BF16)
                pack.up = torch.zeros((N, r), device=dev, dtype=torch.float32)  # sb200_lora.up is fp32
            else:
                pack.down.zero_()
                pack.up.zero_()
            n0 = 0
            for gi, (leaf, a) in enumerate(zip(leaves, adaptors)):
                n1 = n0 + leaf.weight.shape[0]
                if a is not None:
                    d = a.lora_down.weight.detach()
                    if d.dim() == 4:
                        d = d.permute(0, 2, 3, 1)
                    rr = d.shape[0]
                    pack.down[gi * r: gi * r + rr].copy_(d.reshape(rr, -1))
                    u = a.lora_up.weight.detach().reshape(leaf.weight.shape[0], -1)
                    if common is None:
                        u = u.float() * scales[gi]
                    pack.up[n0:n1, :rr].copy_(u)
                n0 = n1
            pack.key = ver
        return pack, r, common

    def _composite(self, leaves) -> Optional[_LoraPack]:
        """The pack of one fused call on a UNet with an active SliderStack: slider i's rows / columns [o_i, o_i + r_i)
        of every leaf's slot, alpha / r folded into the raw up pack, the runtime multipliers applied by
        sb200_lora_compose; the kernels run with scale 1.  None when no leaf is hooked."""
        hooks = [hook_of(l) for l in leaves]
        if all(h is None for h in hooks):
            return None
        arena = self.arena
        rp = arena.rp
        _, rt = ops.lora_slots(rp, len(leaves))
        pack = self.packs.setdefault(tuple(id(l) for l in leaves), _LoraPack(leaves))
        ver = tuple(tuple((i, a.lora_down.weight.data_ptr(), a.lora_down.weight._version, a.lora_up.weight.data_ptr(),
                           a.lora_up.weight._version) for i, a in h.slider_entries) if h is not None else None
                    for h in hooks)
        if pack.key != ver:
            if pack.raw is None:
                if self.capture:
                    raise RuntimeError("sliders_b200: a SliderStack call site was first met while a CUDA graph was "
                                       "captured")
                dev = leaves[0].weight.device
                K = leaves[0].weight[0].numel()
                N = sum(l.weight.shape[0] for l in leaves)
                pack.down = torch.zeros((rt, K), device=dev, dtype=BF16)
                pack.raw = torch.zeros((N, rp), device=dev, dtype=torch.float32)
                pack.up = torch.empty((N, rp), device=dev, dtype=torch.float32)
                arena.packs.append(pack)
                arena.dirty = True
            else:
                pack.down.zero_()
                pack.raw.zero_()
            _fill_composite(pack.down, pack.raw, leaves, hooks, arena.stack.offsets, rp)
            pack.key = ver
            # the walk's compose has run already: compose this pack now
            ops.lora_compose(pack.raw, arena.mult, out=pack.up)
        return pack

    def _sample_vec(self, factor: float) -> torch.Tensor:
        """The device vector of the walk's batch for adaptor factor `factor`, filled once per walk (a captured graph
        gets its values from `refresh` instead)."""
        B = self.snap.batch
        key = (B, factor)
        vec = self.sample_vecs.get(key)
        if vec is None:
            if self.capture:
                raise RuntimeError("sliders_b200: a per-sample scale vector was first needed while a CUDA graph was "
                                   "captured")
            vec = torch.empty(B, device=self.device, dtype=torch.float32)
            self.sample_vecs[key] = vec
        if not self.capture and key not in self.filled:
            _fill_sample_vec(vec, factor, self.snap.sample_values)
            self.filled.add(key)
        return vec
