"""Backward-to-LoRA pass of the UNet: what `loss.backward()` does in the reference trainers
(trainscripts/textsliders/train_lora_xl.py:345, train_lora.py:298, imagesliders/train_lora-scale-xl.py:340,372) —
autograd through the frozen diffusers UNet down to every `lora_down.weight` / `lora_up.weight` (lora.py:97-112).

The frozen weights need no gradient, so the pass is
  * the input-gradient chain of every op (dense products on the same wgmma GEMM / implicit-GEMM conv kernels with
    transposed weights, flash-attention backward, GroupNorm / LayerNorm / GEGLU / SiLU backward), and
  * per adapted leaf  y = W x + s up (down x):  d_up = s dY^T (x down^T),  d_down = s (dY up)^T x,  dX += s (dY up) down
    as rank-r reductions (csrc/backward.cu).
`UNet2DConditionModel.forward` routes here (through `_UNetFunction`) whenever autograd is enabled and an active
adaptor requires grad or `encoder_hidden_states` requires grad; otherwise the inference forward runs.  Both run the one
forward walk `UNet2DConditionModel._walk`: given a tape it also keeps the activations the backward needs (about 7 GB for
an SDXL CFG pair at 1024 px), so the backward mirrors exactly the function inference computes, and it applies GEGLU
unfused so its pre-activation can be kept.  Every Linear / conv leaf the walk runs carries its adaptor, if active, in
both modes.
The gradient w.r.t. `encoder_hidden_states` (null-text inversion optimises the unconditional text embedding through the
UNet) is the transpose of the batched cross-attention K / V projection of the forward (`unet._kv_plan`): every
cross-attention block's dK | dV lands in its columns of one [B * 77, sum 2C] matrix, and one fp32 split-K GEMM against
the stacked to_k | to_v weights gives d_ctx = dKV_all . W_kv.  Frozen active adaptors (a slider applied while the
embedding is optimised) contribute to the input gradients; only trainable ones get weight gradients.
The gradient w.r.t. the latents is not produced (the reference detaches them: train_lora_xl.py:207-229 runs the
denoising under no_grad) — `sample.grad` stays None.
"""
from __future__ import annotations

import warnings
import weakref

from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from .unet import _GraphInputs

BF16 = torch.bfloat16


# ----------------------------------------------------------------------------------------------------------------
# transposed frozen weights (cached next to the forward packing in unet._packed)
# ----------------------------------------------------------------------------------------------------------------
def _wt(unet, leaf) -> torch.Tensor:
    """Input-gradient weight of a Linear / 1x1 conv leaf: [K, N] so that dX = gemm(dY, wt)."""
    key = ("wt", id(leaf))
    w = unet._packed.get(key)
    if w is None:
        w = unet._w(leaf).t().contiguous()
        unet._packed[key] = w
    return w


def _wt_fused(unet, leaves) -> torch.Tensor:
    key = ("wtf",) + tuple(id(l) for l in leaves)
    w = unet._packed.get(key)
    if w is None:
        w = unet._fused_w(leaves).t().contiguous()
        unet._packed[key] = w
    return w


def _w_dgrad(unet, conv) -> torch.Tensor:
    """3x3 conv: [Cin, 3, 3, Cout] with flipped taps, so that dX = conv3x3(dY, w_dgrad) (stride 1 / pad 1)."""
    key = ("wd", id(conv))
    w = unet._packed.get(key)
    if w is None:
        w = unet._w(conv).flip(1, 2).permute(3, 1, 2, 0).contiguous()
        unet._packed[key] = w
    return w


# ----------------------------------------------------------------------------------------------------------------
# LoRA leaf gradients
# ----------------------------------------------------------------------------------------------------------------
class _Grads:
    """fp32 gradient buffers per adaptor parameter, keyed by id(parameter), plus the (adaptor, multiplier * alpha / r,
    trainable) of every active leaf as it was when the FORWARD ran: `loss.backward()` is called after `with network:`
    has reset the multipliers to 0 (train_lora_xl.py:299-345, lora.py:256-258).  `dkv` / `kv_off`: the cross-attention
    dK | dV matrix of the encoder_hidden_states gradient and each block's column offset in it (None without it)."""

    def __init__(self, scales: Dict[int, tuple]):
        self.by_param: Dict[int, torch.Tensor] = {}
        self.slots: Dict[int, torch.Tensor] = {}
        self.scales = scales
        self.dkv: Optional[torch.Tensor] = None
        self.kv_off: Dict[int, int] = {}

    def active(self, leaf):
        return self.scales.get(id(leaf), (None, 0.0, False))[:2]

    def trainable(self, leaf) -> bool:
        return self.scales.get(id(leaf), (None, 0.0, False))[2]

    def any_trainable(self) -> bool:
        return any(v[2] for v in self.scales.values())

    def buf(self, param: torch.Tensor, shape, r: int, rank_dim: int) -> Tuple[torch.Tensor, bool]:
        """(fp32 gradient buffer of `param` in the kernels' layout `shape`, whose axis `rank_dim` has the slot width;
        whether it already holds a gradient).  by_param files its first r entries along that axis: the gradient in
        the parameter's own rank, without the padding."""
        g = self.slots.get(id(param))
        if g is None:
            g = torch.empty(shape, device=param.device, dtype=torch.float32)
            self.slots[id(param)] = g
            self.by_param[id(param)] = g.narrow(rank_dim, 0, r)
            return g, False
        return g, True


def _pad_rank(t: torch.Tensor, dim: int, rp: int) -> torch.Tensor:
    """t zero-padded along its rank axis `dim` to the slot width rp (t itself when it has that size already)."""
    r = t.shape[dim]
    if r == rp:
        return t
    shape = list(t.shape)
    shape[dim] = rp
    out = t.new_zeros(shape)
    out.narrow(dim, 0, r).copy_(t)
    return out


def _new_tape(snap) -> list:
    """A tape for `unet._walk`, opened with the active adaptors of the forward's snapshot (lora_pack.scan), which
    `_Grads` reads."""
    if snap.stack_mults is not None:
        # the backward kernels read one adaptor per leaf; a SliderStack's composite hooks carry several
        raise NotImplementedError("sliders_b200: a gradient through an active SliderStack is not implemented "
                                  "(stacks are for inference)")
    scales = {}
    for key, (a, s, trainable) in snap.adaptors.items():
        if s != 0.0:
            if getattr(a, "sample_scales", None) is not None:
                # the backward kernels (lora_wgrad, lora_rank_update and their conv forms) take one scale per launch
                raise NotImplementedError("sliders_b200: a gradient through a forward with per-sample slider scales is "
                                          "not implemented (per-sample scales are for inference; set a scalar with "
                                          "set_lora_slider, or run under torch.no_grad())")
            scales[key] = (a, s, trainable)
    return [("scales", scales)]


def _lora_linear_bwd(unet, grads: _Grads, leaf, xs: List[torch.Tensor], dY: torch.Tensor,
                     dX: Optional[torch.Tensor]) -> None:
    """xs: the leaf's 2-D input as one or two column blocks ([x0 | x1]); dY [M, N]; dX [M, K] updated in place."""
    a, s = grads.active(leaf)
    train = grads.trainable(leaf)
    if a is None or (not train and dX is None):
        return
    down = a.lora_down.weight.detach().reshape(a.lora_down.weight.shape[0], -1).to(BF16)   # [r, K]
    up = a.lora_up.weight.detach().reshape(a.lora_up.weight.shape[0], -1).to(BF16)         # [N, r]
    r, K = down.shape
    rp, _ = ops.lora_slots(r)  # the kernels take rank rp: zero rows / columns beyond r
    down, up = _pad_rank(down, 0, rp), _pad_rank(up, 1, rp)
    if not train:  # frozen adaptor: its share of the input gradient only
        ops.lora_rank_update(dX, ops.lora_proj(dY, up.t().contiguous()), down, s)
        return
    t = None
    k0 = 0
    for x in xs:
        t = ops.lora_proj(x, down[:, k0:k0 + x.shape[1]], out=t)
        k0 += x.shape[1]
    u = ops.lora_proj(dY, up.t().contiguous())
    g_up, acc = grads.buf(a.lora_up.weight, (up.shape[0], rp), r, 1)
    ops.lora_wgrad(dY, t, g_up, False, s, accumulate=acc)
    g_down, acc = grads.buf(a.lora_down.weight, (rp, K), r, 0)
    k0 = 0
    for x in xs:
        ops.lora_wgrad(x, u, g_down[:, k0:k0 + x.shape[1]], True, s, accumulate=acc)
        k0 += x.shape[1]
    if dX is not None:
        ops.lora_rank_update(dX, u, down, s)


def _lora_conv_bwd(unet, grads: _Grads, conv, x: torch.Tensor, dY: torch.Tensor, dX: Optional[torch.Tensor],
                   stride: int = 1) -> None:
    """x [B,H,W,Cin] NHWC input of the 3x3 leaf; dY [B,Ho,Wo,Cout]; dX [B,H,W,Cin] updated in place."""
    a, s = grads.active(conv)
    train = grads.trainable(conv)
    if a is None or (not train and dX is None):
        return
    D = a.lora_down.weight.detach().permute(0, 2, 3, 1).to(BF16).contiguous()             # [r, 3, 3, Cin]
    up = a.lora_up.weight.detach().reshape(a.lora_up.weight.shape[0], -1).to(BF16)        # [Cout, r]
    r = D.shape[0]
    rp, _ = ops.lora_slots(r)
    D, up = _pad_rank(D, 0, rp), _pad_rank(up, 1, rp)
    dY2 = dY.reshape(-1, dY.shape[-1])
    if not train:  # frozen adaptor: its share of the input gradient only
        ops.lora_conv_rank_update(dX, ops.lora_proj(dY2, up.t().contiguous()), D, s, stride)
        return
    t = ops.lora_conv_proj(x, D, stride)
    u = ops.lora_proj(dY2, up.t().contiguous())
    g_up, acc = grads.buf(a.lora_up.weight, (up.shape[0], rp), r, 1)
    ops.lora_wgrad(dY2, t, g_up, False, s, accumulate=acc)
    g_down, acc = grads.buf(a.lora_down.weight, tuple(D.shape), r, 0)
    ops.lora_conv_wgrad(x, u, g_down, s, stride, accumulate=acc)
    if dX is not None:
        ops.lora_conv_rank_update(dX, u, D, s, stride)


# ----------------------------------------------------------------------------------------------------------------
# the backward, block by block, of the records `UNet2DConditionModel._walk` leaves on the tape
# ----------------------------------------------------------------------------------------------------------------
def _resnet_bwd(unet, grads, rec, d_out, need_dx=True):
    """Returns (dx0, dx1): gradients w.r.t. the block input and the skip source (views of one concat buffer)."""
    blk, x0, x1, emb_act, ws1, h1, h2, ws2, h3 = rec
    B, H, W, Cout = d_out.shape
    n1, n2 = blk.norm1, blk.norm2
    # conv2
    d_h3 = ops.conv3x3(d_out, _w_dgrad(unet, blk.conv2))
    _lora_conv_bwd(unet, grads, blk.conv2, h3, d_out, d_h3)
    d_h2 = ops.groupnorm_bwd(h2, *unet._w_norm(n2), n2.num_groups, True, d_h3, ws2)
    # time_emb_proj: its output is broadcast over the pixels of conv1's output
    if grads.trainable(blk.time_emb_proj):
        d_temb = ops.colsum(d_h2).to(BF16)
        _lora_linear_bwd(unet, grads, blk.time_emb_proj, [emb_act], d_temb, None)
    # conv1
    first = not need_dx
    d_h1 = None if first else ops.conv3x3(d_h2, _w_dgrad(unet, blk.conv1))
    _lora_conv_bwd(unet, grads, blk.conv1, h1, d_h2, d_h1)
    # shortcut
    d_out2 = d_out.reshape(-1, Cout)
    x0v = x0.reshape(-1, x0.shape[-1])
    xs = [x0v] + ([x1.reshape(-1, x1.shape[-1])] if x1 is not None else [])
    if blk.conv_shortcut is not None:
        sc = blk.conv_shortcut
        d_xs = None if first else ops.gemm(d_out2, _wt(unet, sc))
        _lora_linear_bwd(unet, grads, sc, xs, d_out2, d_xs)
        if d_xs is not None:
            d_xs = d_xs.view(B, H, W, -1)
    else:
        d_xs = d_out
    if first:
        return None, None
    dx = ops.groupnorm_bwd(x0, *unet._w_norm(n1), n1.num_groups, True, d_h1, ws1, x1=x1, add=d_xs)
    C0 = x0.shape[-1]
    if x1 is None:
        return dx, None
    return dx[..., :C0], dx[..., C0:]


def _attn_bwd(unet, grads, attn, rec, x_norm, d_h, B, S):
    """Backward of `resid + to_out(attention(x_norm))` w.r.t. x_norm: returns d_x_norm [M, C] (the residual path
    is the caller's)."""
    q, k, v, o, lse, Skv, ctx = rec
    C_ = attn.to_q.weight.shape[0]
    scale = attn.dim_head ** -0.5
    out = attn.to_out[0]
    d_o = ops.gemm(d_h, _wt(unet, out))
    _lora_linear_bwd(unet, grads, out, [o], d_h, d_o)
    if ctx is None:
        dqkv = torch.empty((B * S, 3 * C_), device=d_h.device, dtype=BF16)
        ops.attention_bwd(q, k, v, o, d_o, lse, B, attn.heads, S, S, scale, attn.dim_head, dqkv[:, :C_],
                          dqkv[:, C_:2 * C_], dqkv[:, 2 * C_:])
        leaves = [attn.to_q, attn.to_k, attn.to_v]
        d_n = ops.gemm(dqkv, _wt_fused(unet, leaves))
        for i, leaf in enumerate(leaves):
            _lora_linear_bwd(unet, grads, leaf, [x_norm], dqkv[:, i * C_:(i + 1) * C_], d_n)
        return d_n
    dq = torch.empty((B * S, C_), device=d_h.device, dtype=BF16)
    if any(grads.trainable(l) for l in (attn.to_k, attn.to_v)):
        # train methods `xattn` / `full`: the text-side projections are adapted; encoder_hidden_states needs no grad
        dkv = torch.empty((B * Skv, 2 * C_), device=d_h.device, dtype=BF16)
        ops.attention_bwd_split(q, k, v, o, d_o, lse, B, attn.heads, S, Skv, scale, attn.dim_head, dq, dkv[:, :C_],
                                dkv[:, C_:])
        _lora_linear_bwd(unet, grads, attn.to_k, [ctx], dkv[:, :C_], None)
        _lora_linear_bwd(unet, grads, attn.to_v, [ctx], dkv[:, C_:], None)
    elif grads.dkv is not None:
        # encoder_hidden_states needs a gradient: dK | dV into this block's columns of the batched K / V layout
        off = grads.kv_off[id(attn)]
        ops.attention_bwd_split(q, k, v, o, d_o, lse, B, attn.heads, S, Skv, scale, attn.dim_head, dq,
                                grads.dkv[:, off:off + C_], grads.dkv[:, off + C_:off + 2 * C_])
    else:
        ops.attention_bwd(q, k, v, o, d_o, lse, B, attn.heads, S, Skv, scale, attn.dim_head, dq)
    d_n = ops.gemm(dq, _wt(unet, attn.to_q))
    _lora_linear_bwd(unet, grads, attn.to_q, [x_norm], dq, d_n)
    return d_n


def _transformer_bwd(unet, grads, rec, d_out):
    tr, x, ws, hn, blocks, h_last = rec
    B, H, W, C_ = x.shape
    S = H * W
    d_out2 = d_out.reshape(B * S, C_)
    d_h = ops.gemm(d_out2, _wt(unet, tr.proj_out))
    _lora_linear_bwd(unet, grads, tr.proj_out, [h_last], d_out2, d_h)
    for blk, h1, a1, h2, a2, h3, pre in reversed(blocks):
        ffp, ffo = blk.ff.net[0].proj, blk.ff.net[2]
        # feed-forward
        d_f = ops.gemm(d_h, _wt(unet, ffo))
        if grads.active(ffo)[0] is not None:  # a frozen adaptor needs only dY: its input is not rebuilt
            _lora_linear_bwd(unet, grads, ffo, [ops.geglu(pre)] if grads.trainable(ffo) else [], d_h, d_f)
        d_pre = ops.geglu_bwd(pre, d_f)
        d_n = ops.gemm(d_pre, _wt(unet, ffp))
        if grads.active(ffp)[0] is not None:
            n3 = ops.layernorm(h3, *unet._w_norm(blk.norm3), eps=blk.norm3.eps) if grads.trainable(ffp) else None
            _lora_linear_bwd(unet, grads, ffp, [n3] if n3 is not None else [], d_pre, d_n)
        d_h = ops.layernorm_bwd(h3, unet._w_norm(blk.norm3)[0], d_n, blk.norm3.eps, add=d_h)
        # cross-attention
        n2 = ops.layernorm(h2, *unet._w_norm(blk.norm2), eps=blk.norm2.eps)
        d_n = _attn_bwd(unet, grads, blk.attn2, a2, n2, d_h, B, S)
        d_h = ops.layernorm_bwd(h2, unet._w_norm(blk.norm2)[0], d_n, blk.norm2.eps, add=d_h)
        # self-attention
        n1 = ops.layernorm(h1, *unet._w_norm(blk.norm1), eps=blk.norm1.eps)
        d_n = _attn_bwd(unet, grads, blk.attn1, a1, n1, d_h, B, S)
        d_h = ops.layernorm_bwd(h1, unet._w_norm(blk.norm1)[0], d_n, blk.norm1.eps, add=d_h)
    d_hn = ops.gemm(d_h, _wt(unet, tr.proj_in))
    _lora_linear_bwd(unet, grads, tr.proj_in, [hn], d_h, d_hn)
    gn = tr.norm
    return ops.groupnorm_bwd(x, *unet._w_norm(gn), gn.num_groups, False, d_hn.view(B, H, W, C_), ws, add=d_out)


def slice_tape(obj, lo: int, hi: int, B: int):
    """The tape restricted to samples [lo, hi) of the batch: every saved activation is batch-major ([B, ...] or a
    token matrix [B * rows, C]), so a view suffices.  Used to skip samples whose incoming gradient is exactly zero —
    the unconditional half of a CFG pair at guidance_scale 1 (train_util.py:250-253: d eps / d uncond = 1 - g = 0;
    every grad-carrying prediction of the trainers is made at guidance 1)."""
    if torch.is_tensor(obj):
        if obj.dim() >= 3 and obj.shape[0] == B:
            return obj[lo:hi]
        if obj.dim() == 2 and obj.shape[0] % B == 0:
            rpb = obj.shape[0] // B
            return obj[lo * rpb:hi * rpb]
        raise RuntimeError(f"slice_tape: tensor of shape {tuple(obj.shape)} is not batch-major for B={B}")
    if isinstance(obj, tuple):
        return tuple(slice_tape(o, lo, hi, B) for o in obj)
    if isinstance(obj, list):
        return [slice_tape(o, lo, hi, B) for o in obj]
    return obj  # modules, ints, None, the scales snapshot


def _kv_plan_t(unet) -> Tuple[torch.Tensor, Dict[int, int]]:
    """The stacked to_k | to_v weights of every cross-attention block, all channel widths in `_kv_plan` order, transposed
    to [D_ctx, sum 2C] (packed once, like `_wt`), and each block's column offset in that order."""
    ent = unet._packed.get("kvplan_t")
    if ent is None:
        plan = unet._kv_plan()
        offs, base, ws = {}, 0, []
        for C_, (w, o, _) in plan.items():
            for aid, off in o.items():
                offs[aid] = base + off
            base += w.shape[0]
            ws.append(w)
        ent = (torch.cat(ws, 0).t().contiguous(), offs)
        unet._packed["kvplan_t"] = ent
    return ent


def backward(unet, tape, d_eps: torch.Tensor, need_ehs: bool = False) -> Dict:
    """Runs the tape in reverse; returns {id(parameter): fp32 gradient in the packed kernel layout}, plus under the key
    "ehs" the fp32 [B * 77, D_ctx] gradient w.r.t. encoder_hidden_states when `need_ehs`."""
    assert tape[0][0] == "scales"
    grads = _Grads(tape[0][1])
    d_skips: List[torch.Tensor] = []
    d_h = None
    first_res = next(i for i, (kind, _) in enumerate(tape) if kind == "res")
    stop_at = -1
    if need_ehs:
        first_tr = next(i for i, (kind, _) in enumerate(tape) if kind == "tr")
        if not grads.any_trainable():
            stop_at = first_tr  # nothing below the first transformer block needs a gradient
        Sctx = next(rec for kind, rec in tape if kind == "ctx")  # tokens per sample of encoder_hidden_states
        wt, grads.kv_off = _kv_plan_t(unet)
        grads.dkv = torch.empty((d_eps.shape[0] * Sctx, wt.shape[1]), device=d_eps.device, dtype=BF16)
    for idx in range(len(tape) - 1, -1, -1):
        kind, rec = tape[idx]
        if kind == "out":
            h, ws = rec
            gn = unet.conv_norm_out
            d_hn = ops.conv_out_bwd(d_eps, unet._w(unet.conv_out))
            d_h = ops.groupnorm_bwd(h, *unet._w_norm(gn), gn.num_groups, True, d_hn, ws)
        elif kind == "res":
            dx0, dx1 = _resnet_bwd(unet, grads, rec, d_h, need_dx=idx != first_res)
            if dx1 is not None:
                d_skips.append(dx1)
            d_h = dx0
        elif kind == "tr":
            d_h = _transformer_bwd(unet, grads, rec, d_h)
        elif kind == "up":
            conv, x_in = rec
            xu = ops.upsample2x(x_in)
            d_xu = ops.conv3x3(d_h, _w_dgrad(unet, conv))
            _lora_conv_bwd(unet, grads, conv, xu, d_h, d_xu)
            d_h = ops.upsample2x_bwd(d_xu)
        elif kind == "down":
            conv, x_in = rec
            d_x = ops.conv3x3(ops.zero_stuff(d_h), _w_dgrad(unet, conv))
            _lora_conv_bwd(unet, grads, conv, x_in, d_h, d_x, stride=2)
            d_h = d_x
        elif kind == "skip":
            ds = d_skips.pop()
            shp = d_h.shape
            d_h = ops.add(d_h.reshape(-1, shp[-1]), ds.reshape(-1, shp[-1])).view(shp)
        if d_h is None and kind == "res":
            break  # first resnet: nothing upstream carries an adaptor
        if idx == stop_at:
            break
    if need_ehs:
        grads.by_param["ehs"] = ops.gemm_splitk_f32(grads.dkv, _kv_plan_t(unet)[0])
    return grads.by_param


# ----------------------------------------------------------------------------------------------------------------
# torch.autograd bridge
# ----------------------------------------------------------------------------------------------------------------
def _param_grad(shape, dtype, g: torch.Tensor) -> torch.Tensor:
    """fp32 packed-layout gradient -> the parameter's own shape / dtype (lora.py:67-91 layouts)."""
    if len(shape) == 4 and shape[2] == 3:      # conv lora_down [r, Cin, 3, 3] <- [r, 3, 3, Cin]
        g = g.permute(0, 3, 1, 2)
    return g.reshape(shape).to(dtype)


class _TrainCapture(_GraphInputs):
    """Training forward + backward of one call signature as two CUDA graphs sharing a memory pool: the eager path is
    host-bound (~5 000 launches per CFG pair, 124 ms against ~75 ms of device time at SDXL size).  The activations
    of the tape live in the graph pool between the two replays; inputs, the incoming gradient and the flat gradient
    of all adaptor weights are static buffers.  The forward reads the slider factor from the device scalar the
    inference graphs use; the backward bakes it in, so the factor is part of the cache key."""

    def __init__(self, unet, sample, t, ehs, added, out_dtype, params, keys, snap, need_ehs=False):
        super().__init__(sample, t, ehs, added)
        self.need_ehs = need_ehs
        self.keys = keys
        self.meta = [(tuple(p.shape), p.dtype) for p in params]
        self.pending = False
        self.pending_token = None
        stream = torch.cuda.Stream(device=sample.device)
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):  # warm-up: weight / LoRA packing caches, transposed weights, TMA descriptors
            tape = _new_tape(snap)
            out = unet._walk(self.x, self.t, self.ehs, self.added, out_dtype, tape, snap)
            backward(unet, tape, torch.zeros_like(out), need_ehs)
            del tape
        torch.cuda.current_stream().wait_stream(stream)
        torch.cuda.synchronize()
        self.gf = torch.cuda.CUDAGraph()
        self.tape = _new_tape(snap)
        with torch.cuda.graph(self.gf):
            self.out = unet._walk(self.x, self.t, self.ehs, self.added, out_dtype, self.tape, snap, capture=True)
        self.d_out = torch.zeros_like(self.out)
        self.unet = unet
        self.bwd = {}  # dead leading samples -> (graph, flat fp32 gradient of every adaptor weight, d_ehs or None)

    def _capture_backward(self, dead: int):
        unet = self.unet
        B = self.out.shape[0]
        tape = slice_tape(self.tape, dead, B, B) if dead else self.tape
        d_live = self.d_out[dead:] if dead else self.d_out
        stream = torch.cuda.Stream(device=self.x.device)
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            backward(unet, tape, d_live, self.need_ehs)  # warm-up of this variant
        torch.cuda.current_stream().wait_stream(stream)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, pool=self.gf.pool()):
            by_param = backward(unet, tape, d_live, self.need_ehs)
            pieces = []
            for key, (shape, dtype) in zip(self.keys, self.meta):
                g = by_param.get(key)
                g = _param_grad(shape, dtype, g) if g is not None else torch.zeros(shape, device=self.x.device, dtype=dtype)
                pieces.append(g.reshape(-1).to(torch.float32))
            flat = torch.cat(pieces) if pieces else None
        self.bwd[dead] = (graph, flat, by_param.get("ehs"))

    def run_forward(self, unet, x, t, ehs, added, snap):
        self.load(unet, x, t, ehs, added, snap)
        self.gf.replay()
        self.pending = True
        return self.out.clone()

    def run_backward(self, d_out, dead: int = 0):
        self.d_out.copy_(d_out)
        if dead not in self.bwd:
            self._capture_backward(dead)
        graph, flat_static, d_ehs = self.bwd[dead]
        graph.replay()
        self.pending = False
        d_ehs = d_ehs.clone() if d_ehs is not None else None
        if flat_static is None:
            return [], d_ehs
        flat = flat_static.clone()
        grads, off = [], 0
        by_dtype = {}
        for shape, dtype in self.meta:
            n = 1
            for d in shape:
                n *= d
            src = by_dtype.get(dtype)
            if src is None:
                src = by_dtype[dtype] = flat if dtype == torch.float32 else flat.to(dtype)
            grads.append(src[off:off + n].view(shape))
            off += n
        return grads, d_ehs


def _capture_for(unet, sample, t, ehs, added, out_dtype, params, keys, snap, need_ehs=False):
    """Cached _TrainCapture for this call signature, or None when graphs are off / the signature cannot be captured
    (adaptors with different factors, or a second forward before the first one's backward)."""
    if not getattr(unet, "use_cuda_graph", False):
        return None
    sig, common = snap.signature, snap.common
    if common is None and any(sig[0]):
        return None
    key = (("train",) + _GraphInputs.key(sample, ehs, added, out_dtype)
           + (sig, round(common, 9) if common is not None else None, tuple(keys), bool(need_ehs)))
    cache = unet.__dict__.setdefault("_train_graphs", {})
    cap = cache.get(key)
    if cap is None:
        while len(cache) >= getattr(unet, "train_graph_max", 2):  # each capture pins its activations (19 GB at SDXL)
            cache.pop(next(iter(cache)))
        cap = _TrainCapture(unet, sample, t, ehs, added, out_dtype, params, keys, snap, need_ehs)
        cache[key] = cap
    if cap.pending and cap.pending_token is not None and cap.pending_token() is None:
        # the autograd node of the forward that was never back-propagated is gone (exception, loss only logged, skipped
        # step): its tape is dead, the graphs are free again
        cap.pending = False
    if cap.pending:
        global _warned_pending
        if not _warned_pending:
            _warned_pending = True
            warnings.warn("sliders_b200: a second grad-carrying UNet forward with the same signature ran before the first "
                          "one's backward; it takes the eager (un-graphed) path.  Release or back-propagate the first "
                          "prediction to return to CUDA-graph replay.")
        return None
    return cap


_warned_pending = False


class _Token:
    """Lives in the autograd node's __dict__; a dead weakref to it means the node (and its tape) has been freed."""
    __slots__ = ("__weakref__",)


class _UNetFunction(torch.autograd.Function):
    @staticmethod
    def forward(fctx, unet, call, ehs_in, *params):
        sample, t, added, out_dtype, keys, need_ehs, snap = call
        ehs = ehs_in.detach().to(device=sample.device, dtype=BF16).contiguous()
        fctx.unet, fctx.keys, fctx.need_ehs = unet, keys, need_ehs
        fctx.ehs_meta = (tuple(ehs_in.shape), ehs_in.dtype, ehs_in.device)
        fctx.meta = [(tuple(p.shape), p.dtype) for p in params]
        fctx.cap = _capture_for(unet, sample, t, ehs, added, out_dtype, params, keys, snap, need_ehs)
        if fctx.cap is not None:
            fctx.tape = True
            fctx.token = _Token()
            fctx.cap.pending_token = weakref.ref(fctx.token)
            return fctx.cap.run_forward(unet, sample, t, ehs, added, snap)
        fctx.tape = _new_tape(snap)
        return unet._walk(sample, t, ehs, added, out_dtype, fctx.tape, snap)

    @staticmethod
    def backward(fctx, d_out):
        if fctx.tape is None:
            raise RuntimeError("sliders_b200: backward through the same UNet call twice (retain_graph is not supported)")
        dead = int(getattr(fctx, "zero_rows", 0) or 0)  # leading samples whose incoming gradient is exactly zero
        if fctx.cap is not None:
            with torch.no_grad():
                grads, d_ctx = fctx.cap.run_backward(d_out, dead)
                d_ehs = _ehs_grad(fctx, d_ctx, dead)
            fctx.tape = None
            return (None, None, d_ehs, *grads)
        with torch.no_grad():
            tape, d_live = fctx.tape, d_out.contiguous()
            if dead:
                B = d_out.shape[0]
                tape, d_live = slice_tape(tape, dead, B, B), d_live[dead:]
            by_param = backward(fctx.unet, tape, d_live, fctx.need_ehs)
            d_ehs = _ehs_grad(fctx, by_param.get("ehs"), dead)
        fctx.tape = None  # free the activations
        out = [None, None, d_ehs]
        for key, (shape, dtype) in zip(fctx.keys, fctx.meta):
            g = by_param.get(key)
            out.append(_param_grad(shape, dtype, g) if g is not None else None)
        return tuple(out)


def _ehs_grad(fctx, d_ctx: Optional[torch.Tensor], dead: int) -> Optional[torch.Tensor]:
    """fp32 [B_live * 77, D] -> the gradient in encoder_hidden_states' own shape / dtype / device; the `dead` leading
    samples (exactly-zero incoming gradient) get zeros."""
    if not fctx.need_ehs:
        return None
    shape, dtype, device = fctx.ehs_meta
    if dead:
        full = torch.zeros(shape, device=d_ctx.device, dtype=torch.float32)
        full[dead:].copy_(d_ctx.view((shape[0] - dead,) + shape[1:]))
        d_ctx = full
    return d_ctx.view(shape).to(device=device, dtype=dtype)



def trainable_lora_params(snap) -> List[torch.Tensor]:
    ps = []
    for a, s, trainable in snap.adaptors.values():
        if s != 0.0 and trainable:
            ps += [a.lora_down.weight, a.lora_up.weight]
    return ps


def apply(unet, sample, t, ehs, added, out_dtype, snap, need_ehs: bool = False):
    """ehs: encoder_hidden_states as the caller passed it (any float dtype); with `need_ehs` it is an autograd input
    and its gradient comes back in its own dtype, shape and device.  `snap`: the forward's lora_pack.scan."""
    params = trainable_lora_params(snap)
    keys = [id(p) for p in params]  # the backward files gradients under id(adaptor parameter)
    if not need_ehs:
        ehs = ehs.detach()
    return _UNetFunction.apply(unet, (sample, t, added, out_dtype, keys, need_ehs, snap), ehs, *params)
