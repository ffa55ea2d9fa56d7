"""Multi-GPU fan-out of conditioned eps-predictions (SURVEY.md §8e): one process per GPU (torchrun),
`torch.distributed` for the plumbing (NCCL over NVLink between GPUs, gloo in the CPU tests).

The reference is single-process (`--device N`, train_lora_xl.py:414).  What shards naturally is the batch of
*independent* conditioned passes: the 4 predictions x CFG halves of a text-slider iteration
(train_lora_xl.py:236-322), the (high, low) x CFG passes of an image-slider iteration
(train_lora-scale-xl.py:312-372), or the prompts x scales of the inference sweep
(generate_images_xl.py:495-508).  Weights and LoRA parameters are replicated; each rank runs its slice of the
passes through the same kernels and the eps tensors ([B,4,h,w], 128 KiB per sample at 1024 px) are
all-gathered so every rank can evaluate the loss.  The only other exchange on the training path is one
all-reduce(sum) of the flat LoRA-gradient buffer (8.64 MB at rank 4) — `allreduce_lora_grads`.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous slice [lo, hi) of n_items owned by `rank`; the first n_items % world ranks get one extra."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0)
    return lo, hi


def fanout_predict(predict: Callable[..., torch.Tensor], batch_args: Sequence[torch.Tensor],
                   group: Optional[dist.ProcessGroup] = None, **kwargs) -> torch.Tensor:
    """Run `predict(*batch_args_slice, **kwargs)` on this rank's slice of the leading (pass) dimension and
    all-gather the per-pass results, so that every rank returns the full [n_passes, ...] tensor in pass order —
    identical to what one rank computing all passes returns (passes are independent)."""
    if not dist.is_available() or not dist.is_initialized():
        return predict(*batch_args, **kwargs)
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    n = batch_args[0].shape[0]
    lo, hi = shard_range(n, rank, world)
    local = predict(*[a[lo:hi] for a in batch_args], **kwargs) if hi > lo else None
    counts = [shard_range(n, r, world) for r in range(world)]
    max_cnt = max(h - l for l, h in counts)
    # pad to a common size so a single all_gather suffices (counts differ by at most one)
    if local is None:
        probe_shape = None
    else:
        probe_shape = tuple(local.shape[1:])
    shape_list: List[Optional[tuple]] = [None] * world
    dist.all_gather_object(shape_list, (probe_shape, str(local.dtype) if local is not None else None), group=group)
    tail, dtype_s = next(s for s in shape_list if s[0] is not None)
    dtype = getattr(torch, dtype_s.split(".")[-1])
    dev = batch_args[0].device
    buf = torch.zeros((max_cnt,) + tuple(tail), device=dev, dtype=dtype)
    if local is not None:
        buf[: hi - lo].copy_(local)
    gathered = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(gathered, buf, group=group)
    return torch.cat([g[: h - l] for g, (l, h) in zip(gathered, counts)], dim=0)


def allreduce_lora_grads(params: Sequence[torch.nn.Parameter], group: Optional[dist.ProcessGroup] = None) -> None:
    """Sum LoRA gradients over ranks with ONE collective on a flat fp32 buffer (ranks that held no graph contribute
    zeros); afterwards every `.grad` is a view of the reduced buffer (cast to the parameter dtype), so the whole
    exchange is one concat, one all-reduce and one cast regardless of the number of tensors (692 at SDXL rank 4)."""
    if not dist.is_available() or not dist.is_initialized():
        return
    ps = [p for p in params if p.requires_grad]
    if not ps:
        return
    dev = ps[0].device
    if all(p.grad is None for p in ps):
        flat = torch.zeros(sum(p.numel() for p in ps), device=dev, dtype=torch.float32)
    else:
        flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in ps]).float()
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    by_dtype = {}
    off = 0
    for p in ps:
        n = p.numel()
        src = by_dtype.get(p.dtype)
        if src is None:
            src = by_dtype[p.dtype] = flat if p.dtype == torch.float32 else flat.to(p.dtype)
        p.grad = src[off:off + n].view_as(p)
        off += n


def cfg_split_eps(eps_half: torch.Tensor, group: Optional[dist.ProcessGroup] = None) -> torch.Tensor:
    """CFG-split of a serial denoise step over two (or more) ranks: even ranks computed the unconditional half of the
    CFG pair, odd ranks the conditional half; one all-gather (64 KiB per sample at 1024 px) gives every rank
    [uncond ; cond].  Ranks >= 2 duplicate the work of rank (rank % 2) — the loop is serial, there is nothing else to
    split — so any even world size works."""
    world = dist.get_world_size(group)
    eps_half = eps_half.contiguous()
    parts = [torch.empty_like(eps_half) for _ in range(world)]
    dist.all_gather(parts, eps_half, group=group)
    return torch.cat([parts[0], parts[1]], dim=0)


def sync_draws(values: Sequence[float], device, group: Optional[dist.ProcessGroup] = None) -> List[float]:
    """Everything an iteration draws from the host RNG (timesteps_to, bucketed height / width, the six add_time_ids of
    dynamic_crops, the prompt-pair index, the noise seed) travels in ONE small broadcast from group rank 0, so replicas
    stay in lock-step whatever their per-rank seeds are (a `seed + rank` convention would otherwise hand mismatched
    latent shapes to the next collective).  float64 carries ints up to 2**53 exactly."""
    vals = [float(v) for v in values]
    if group is False or not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return vals
    t = torch.tensor(vals, dtype=torch.float64, device=device)
    src = dist.get_global_rank(group, 0) if group is not None else 0
    dist.broadcast(t, src=src, group=group)
    return t.tolist()


def broadcast_lora_params(network: torch.nn.Module, group: Optional[dist.ProcessGroup] = None) -> None:
    """Once at setup: every replica starts from group rank 0's adaptor weights (one flat broadcast per dtype)."""
    if group is False or not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    src = dist.get_global_rank(group, 0) if group is not None else 0
    ps = list(network.parameters())
    for dtype in {p.dtype for p in ps}:
        same = [p for p in ps if p.dtype == dtype]
        flat = torch.cat([p.detach().reshape(-1) for p in same])
        dist.broadcast(flat, src=src, group=group)
        off = 0
        with torch.no_grad():
            for p in same:
                p.copy_(flat[off:off + p.numel()].view_as(p))
                off += p.numel()


def assert_replicas_equal(params: Sequence[torch.Tensor], group: Optional[dist.ProcessGroup] = None,
                          what: str = "LoRA parameters") -> None:
    """Cheap divergence check: (sum, sum of squares) of the flat fp64 parameter vector must agree on every rank."""
    if group is False or not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    flat = torch.cat([p.detach().reshape(-1).double() for p in params])
    sig = torch.stack([flat.sum(), (flat * flat).sum()])
    lo, hi = sig.clone(), sig.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=group)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=group)
    if not torch.equal(lo, hi):
        raise RuntimeError(f"{what} differ between ranks (checksum min {lo.tolist()} max {hi.tolist()}): broadcast them "
                           "once at setup (parallel.broadcast_lora_params)")


def slider_groups(ranks_per_slider: int = 4):
    """Splits the job into independent slider groups of `ranks_per_slider` consecutive ranks and returns
    (this rank's group, its index, number of groups).  One text-slider iteration is a serial chain of batch-1 forwards
    whose sharding stops paying at 4 ranks (CFG halves x {target, frozen predictions}; DESIGN.md §5), so a node with
    more GPUs trains several sliders (attributes / prompt files) side by side, each exactly as a 4-rank job would.
    Every rank must call this (dist.new_group is collective).  Without torch.distributed: (None, 0, 1)."""
    if not dist.is_available() or not dist.is_initialized():
        return None, 0, 1
    world, rank = dist.get_world_size(), dist.get_rank()
    size = max(1, min(int(ranks_per_slider), world))
    if world % size != 0:
        raise ValueError(f"world size {world} is not a multiple of ranks_per_slider={size}")
    n = world // size
    if n == 1:
        return None, 0, 1
    mine = None
    for g in range(n):
        grp = dist.new_group(list(range(g * size, (g + 1) * size)))
        if rank // size == g:
            mine = grp
    return mine, rank // size, n
