"""Thin torch-tensor wrappers over the C ABI (include/sb200.h).  Every function enqueues exactly the
kernels named in its docstring on torch's *current* stream, so the whole UNet forward can be captured in a
CUDA graph.  There is deliberately no PyTorch fallback: a missing extension or a CPU tensor raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _cabi
from ._cabi import EPI_BIAS, EPI_GEGLU, EPI_LORA, EPI_RESID, EPI_ROWBIAS, LnFoldArgs, LoraArgs

BF16 = torch.bfloat16

# launches issued through this module since import (bench.py reports it as gpu_launches)
launch_count = 0
_KERNELS_PER_CALL = {"groupnorm": 3, "groupnorm_bwd": 3, "lora_wgrad": 2}  # stats + finalize + apply; partial + reduce


def _p(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ctx(t: torch.Tensor):
    if not t.is_cuda:
        raise _cabi.Sb200Error("sliders_b200 kernels need CUDA tensors on an H100 (no CPU fallback)")
    return _cabi.handle(t.device.index if t.device.index is not None else torch.cuda.current_device())


# Optional per-call device timing (bench.py's roofline leg): when `profile_log` is a list every wrapper brackets
# its launch with CUDA events on the launching stream and appends (name, flops, start_event, end_event).
profile_log = None
_pending_start = None


# Optional call recording (bench.py's per-kernel-class timing): while `record_calls` is a list and the current stream is
# being captured into a CUDA graph, every C-ABI call is remembered as [fn, args, name, flops].  `replay_calls` re-issues
# a subset on the current stream (normally under a second capture): same kernels, same buffers (they live in the first
# graph's memory pool), so a class of kernels can be timed back to back as its own graph.
record_calls = None


class _Recorder:
    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*args):
            record_calls.append([fn, args, None, 0.0])
            return fn(*args)

        return call


def replay_calls(calls) -> None:
    stream = _stream()
    for fn, args, _, _ in calls:
        assert isinstance(args[1], C.c_void_p), "C-ABI convention: (handle, stream, ...)"
        _cabi.check(fn(args[0], stream, *args[2:]))


def _begin():
    global _pending_start
    if profile_log is not None:
        _pending_start = torch.cuda.Event(enable_timing=True)
        _pending_start.record()
    lib = _cabi.load()
    if record_calls is not None and torch.cuda.is_current_stream_capturing():
        return _Recorder(lib)
    return lib


def _count(name: str = "", flops: float = 0.0) -> None:
    global launch_count, _pending_start
    launch_count += _KERNELS_PER_CALL.get(name, 1)
    if record_calls and record_calls[-1][2] is None:
        record_calls[-1][2], record_calls[-1][3] = name or "other", flops
    if profile_log is not None and _pending_start is not None:
        end = torch.cuda.Event(enable_timing=True)
        end.record()
        profile_log.append((name or "other", flops, _pending_start, end))
        _pending_start = None


class Lora:
    """Packed LoRA side inputs of one fused GEMM/conv call (see struct sb200_lora)."""

    __slots__ = ("down", "up", "r", "rt", "group_n", "scale", "scale_dev", "_c")

    def __init__(self, down: torch.Tensor, up: torch.Tensor, r: int, group_n: int, scale: float,
                 scale_dev: Optional[torch.Tensor] = None):
        self.down, self.up, self.r, self.rt, self.group_n = down, up, r, down.shape[0], group_n
        self.scale, self.scale_dev = float(scale), scale_dev
        self._c = LoraArgs(down.data_ptr(), up.data_ptr(), r, self.rt, group_n, self.scale,
                           scale_dev.data_ptr() if scale_dev is not None else None)

    def ref(self):
        return C.byref(self._c)


class LnFold:
    """LayerNorm folded into the consuming projection (struct sb200_lnfold): `stats` [M, parts, 2] fp32 partial row
    sums left by the GEMM that produced x (its `rowstats=`), `c` / `d` the per-output-column terms of the fold."""

    __slots__ = ("keep", "_c")

    def __init__(self, stats: torch.Tensor, parts: int, C_: int, eps: float, c: torch.Tensor, d: torch.Tensor,
                 c_lora: Optional[torch.Tensor] = None, d_lora: Optional[torch.Tensor] = None):
        self.keep = (stats, c, d, c_lora, d_lora)
        self._c = LnFoldArgs(stats.data_ptr(), int(parts), int(C_), float(eps), c.data_ptr(), d.data_ptr(),
                             c_lora.data_ptr() if c_lora is not None else None,
                             d_lora.data_ptr() if d_lora is not None else None)

    def ref(self):
        return C.byref(self._c)


# slots per row the last `gemm(..., rowstats=...)` call wrote (host-side value, fixed by the tile choice)
last_rowstats_parts = 0
_parts_slot = C.c_int(0)  # module lifetime: recorded calls (bench.py's class graphs) re-issue with this pointer


def gemm(x: torch.Tensor, w: torch.Tensor, *, bias=None, rowbias=None, rows_per_batch: int = 1, resid=None,
         geglu: bool = False, lora: Optional[Lora] = None, x1: Optional[torch.Tensor] = None,
         out: Optional[torch.Tensor] = None, bn: int = 0, ln: Optional[LnFold] = None,
         rowstats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[M,N] = epilogue([x | x1] @ w.T): one wgmma `gemm_kernel` launch.  `ln`: the rows of x are un-normalised and
    w is gamma-scaled (LayerNorm fold); `rowstats` [M, cap, 2] fp32: leave per-row partial (sum, sum of squares) of the
    output for a later `ln` (the number of slots used is `ops.last_rowstats_parts`)."""
    M, K0 = x.shape
    N, K = w.shape
    flags = 0
    if bias is not None:
        flags |= EPI_BIAS
    if rowbias is not None:
        flags |= EPI_ROWBIAS
    if resid is not None:
        flags |= EPI_RESID
    if geglu:
        flags |= EPI_GEGLU
    if lora is not None:
        flags |= EPI_LORA
    nout = N // 2 if geglu else N
    if out is None:
        out = torch.empty((M, nout), device=x.device, dtype=BF16)
    lib = _begin()
    if ln is None and rowstats is None:
        _cabi.check(lib.sb200_gemm(
            _ctx(x), _stream(), _p(x), x.stride(0), _p(x1), x1.stride(0) if x1 is not None else 0, K0,
            _p(w), w.stride(0), _p(out), out.stride(0), M, N, K, flags, _p(bias), _p(rowbias), rows_per_batch,
            _p(resid), resid.stride(0) if resid is not None else 0, lora.ref() if lora is not None else None, bn))
    else:
        global last_rowstats_parts
        parts = _parts_slot
        _cabi.check(lib.sb200_gemm_ln(
            _ctx(x), _stream(), _p(x), x.stride(0), _p(x1), x1.stride(0) if x1 is not None else 0, K0,
            _p(w), w.stride(0), _p(out), out.stride(0), M, N, K, flags, _p(bias), _p(rowbias), rows_per_batch,
            _p(resid), resid.stride(0) if resid is not None else 0, lora.ref() if lora is not None else None, bn,
            ln.ref() if ln is not None else None, _p(rowstats),
            rowstats.numel() // (2 * M) if rowstats is not None else 0, C.cast(C.pointer(parts), C.c_void_p)))
        if rowstats is not None:
            last_rowstats_parts = parts.value
    _count("gemm", 2.0 * M * N * K)
    return out


def conv3x3(x0: torch.Tensor, w_packed: torch.Tensor, *, x1: Optional[torch.Tensor] = None, stride: int = 1,
            bias=None, rowbias=None, resid=None, lora: Optional[Lora] = None, bn: int = 0) -> torch.Tensor:
    """3x3 / pad 1 conv on NHWC bf16 ([B,H,W,C] tensors); w_packed is [Cout,3,3,Cin].  One `gemm_kernel`."""
    B, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    Cout = w_packed.shape[0]
    flags = 0
    if bias is not None:
        flags |= EPI_BIAS
    if rowbias is not None:
        flags |= EPI_ROWBIAS
    if resid is not None:
        flags |= EPI_RESID
    if lora is not None:
        flags |= EPI_LORA
    out = torch.empty((B, H // stride, W // stride, Cout), device=x0.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_conv3x3(
        _ctx(x0), _stream(), _p(x0), x0.stride(2), _p(x1), x1.stride(2) if x1 is not None else 0, C0, C1,
        _p(w_packed), _p(out), Cout, B, H, W, Cout, stride, flags, _p(bias), _p(rowbias), _p(resid),
        resid.stride(2) if resid is not None else 0, lora.ref() if lora is not None else None, bn))
    _count("conv3x3", 2.0 * B * (H // stride) * (W // stride) * Cout * 9 * (C0 + C1))
    return out


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, B: int, heads: int, Sq: int, Skv: int,
              scale: float, head_dim: int = 64, lse: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q/k/v: 2-D (possibly column-sliced) token matrices; head h = columns [h*head_dim, (h+1)*head_dim).
    One `attention_kernel`.  lse: optional fp32 [B, heads, Sq] output kept for `attention_bwd`."""
    out = torch.empty((B * Sq, heads * head_dim), device=q.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_attention(_ctx(q), _stream(), _p(q), q.stride(0), _p(k), k.stride(0), _p(v),
                                    v.stride(0), _p(out), out.stride(0), B, heads, Sq, Skv, int(head_dim),
                                    float(scale), _p(lse)))
    _count("attention", 4.0 * B * heads * Sq * Skv * head_dim)
    return out


def groupnorm(x0: torch.Tensor, gamma, beta, groups: int, eps: float, silu: bool, *,
              x1: Optional[torch.Tensor] = None, stats_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x0/x1: [B, HW, C] (or [B,H,W,C]) NHWC; returns the concatenated, normalised tensor."""
    shp = x0.shape
    B, C0 = shp[0], shp[-1]
    HW = x0.numel() // (B * C0)
    C1 = x1.shape[-1] if x1 is not None else 0
    out = torch.empty(shp[:-1] + (C0 + C1,), device=x0.device, dtype=BF16)
    if stats_ws is None:
        stats_ws = torch.empty(B * groups * 2 * 129, device=x0.device, dtype=torch.float32)  # SB200_GN_WS_FLOATS
    lib = _begin()
    _cabi.check(lib.sb200_groupnorm(_ctx(x0), _stream(), _p(x0), x0.stride(-2), C0, _p(x1),
                                    x1.stride(-2) if x1 is not None else 0, C1, _p(gamma), _p(beta), _p(out),
                                    C0 + C1, B, HW, groups, float(eps), int(silu), _p(stats_ws)))
    _count("groupnorm")
    return out


def layernorm(x: torch.Tensor, gamma, beta, eps: float = 1e-5) -> torch.Tensor:
    M, Cc = x.shape
    out = torch.empty((M, Cc), device=x.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_layernorm(_ctx(x), _stream(), _p(x), x.stride(0), _p(gamma), _p(beta), _p(out), Cc, M,
                                    Cc, float(eps)))
    _count("layernorm")
    return out


def small_linear(x: torch.Tensor, w: torch.Tensor, bias=None, *, act_in: bool = False, act_out: int = 0,
                 lora: Optional[Lora] = None, resid: Optional[torch.Tensor] = None) -> torch.Tensor:
    """act_out: 0 none, 1 SiLU(y) + resid, 2 SiLU(bf16(y + resid)) — see sb200_small_linear."""
    M, K = x.shape
    N = w.shape[0]
    out = torch.empty((M, N), device=x.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_small_linear(_ctx(x), _stream(), _p(x), x.stride(0), _p(w), w.stride(0), _p(bias),
                                       _p(out), N, M, N, K, int(act_in), int(act_out),
                                       lora.ref() if lora is not None else None, _p(resid)))
    _count("small_linear")
    return out


def sinusoid(values: torch.Tensor, dim: int) -> torch.Tensor:
    """values: fp32 [n] on device -> [n, dim] bf16 ([cos | sin])."""
    n = values.numel()
    out = torch.empty((n, dim), device=values.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_sinusoid(_ctx(values), _stream(), _p(values), n, dim, _p(out), dim))
    _count("sinusoid")
    return out


def conv_in(latent: torch.Tensor, w_packed: torch.Tensor, bias) -> torch.Tensor:
    """latent: NCHW fp32 or bf16 -> NHWC bf16 [B,H,W,Cout]."""
    B, Cc, H, W = latent.shape
    assert Cc == 4 and latent.is_contiguous()
    Cout = w_packed.shape[0]
    out = torch.empty((B, H, W, Cout), device=latent.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_conv_in(_ctx(latent), _stream(), _p(latent), int(latent.dtype == torch.float32),
                                  _p(w_packed), _p(bias), _p(out), B, H, W, Cout))
    _count("conv_in")
    return out


def conv_out(x: torch.Tensor, w_packed: torch.Tensor, bias, out_dtype=BF16) -> torch.Tensor:
    B, H, W, Cin = x.shape
    out = torch.empty((B, 4, H, W), device=x.device, dtype=out_dtype)
    lib = _begin()
    _cabi.check(lib.sb200_conv_out(_ctx(x), _stream(), _p(x), _p(w_packed), _p(bias), _p(out),
                                   int(out_dtype == torch.float32), B, H, W, Cin))
    _count("conv_out")
    return out


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    B, H, W, Cc = x.shape
    out = torch.empty((B, 2 * H, 2 * W, Cc), device=x.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_upsample2x(_ctx(x), _stream(), _p(x), _p(out), B, H, W, Cc))
    _count("upsample2x")
    return out


def cfg_ddim(eps2: torch.Tensor, guidance: float, x: Optional[torch.Tensor] = None, a_t: float = 1.0,
             a_prev: float = 1.0, out_dtype=None, single: bool = False, affine: bool = False):
    """eps2 = [uncond batch ; cond batch] (contiguous).  Returns (guided_eps, x_prev or None).
    single=True: eps2 is one already-guided eps batch and guidance must be 0 (plain DDIM step).
    affine=True: (a_t, a_prev) are the coefficients (cx, ce) of x_prev = cx x + ce eps (`sb200_cfg_step`)."""
    if single:
        assert guidance == 0.0
        n = eps2.numel()
        shape = tuple(eps2.shape)
    else:
        n = eps2.numel() // 2
        shape = (eps2.shape[0] // 2,) + tuple(eps2.shape[1:])
    if eps2.dtype not in (torch.float32, BF16):
        eps2 = eps2.to(torch.float32)
    out_dtype = out_dtype or (x.dtype if x is not None else eps2.dtype)
    eps_out = torch.empty(shape, device=eps2.device, dtype=out_dtype)
    x_prev = torch.empty(shape, device=eps2.device, dtype=out_dtype) if x is not None else None
    if x is not None and x.dtype != out_dtype:
        x = x.to(out_dtype)
    lib = _begin()
    fn = lib.sb200_cfg_step if affine else lib.sb200_cfg_ddim
    _cabi.check(fn(_ctx(eps2), _stream(), _p(eps2), int(eps2.dtype == torch.float32),
                                   float(guidance), _p(x), float(a_t), float(a_prev), _p(x_prev), _p(eps_out),
                                   int(out_dtype == torch.float32), n))
    _count("cfg_ddim")
    return eps_out, x_prev


# ----------------------------------------------------------------------------------------------------------------
# backward-to-LoRA pass (csrc/backward.cu, csrc/attention_bwd.cu)
# ----------------------------------------------------------------------------------------------------------------
GN_STATS_OFFSET = 128  # final (mean, rstd) block sits at stats_ws[B * groups * 2 * 128:]  (SB200_GN_STATS_OFFSET)


def gn_ws(B: int, groups: int, device) -> torch.Tensor:
    return torch.empty(B * groups * 2 * 129, device=device, dtype=torch.float32)


def gn_stats(ws: torch.Tensor, B: int, groups: int) -> torch.Tensor:
    """The [B, groups, 2] (mean, rstd) block `groupnorm` left in its workspace (a view: keeps `ws` alive)."""
    return ws[B * groups * 2 * GN_STATS_OFFSET:].view(B, groups, 2)


def attention_bwd(q, k, v, o, dout, lse, B: int, heads: int, Sq: int, Skv: int, scale: float, head_dim: int,
                  dq: torch.Tensor, dk: Optional[torch.Tensor] = None, dv: Optional[torch.Tensor] = None) -> None:
    """dq (and dk, dv) are 2-D (possibly column-sliced) outputs.  `attn_bwd_prep_kernel` + `attention_bwd_kernel`
    (x2 when dk/dv are requested)."""
    dsum = torch.empty(B * heads * Sq, device=q.device, dtype=torch.float32)
    lib = _begin()
    _cabi.check(lib.sb200_attention_bwd(
        _ctx(q), _stream(), _p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(o), o.stride(0),
        _p(dout), dout.stride(0), _p(lse), _p(dsum), _p(dq), dq.stride(0), _p(dk),
        dk.stride(0) if dk is not None else 0, _p(dv), dv.stride(0) if dv is not None else 0, B, heads, Sq, Skv,
        int(head_dim), float(scale)))
    global launch_count
    launch_count += 1 if dk is None else 2
    _count("attention_bwd", (6.0 if dk is None else 14.0) * B * heads * Sq * Skv * head_dim)


def attn_bwd_splits(B: int, heads: int, Sq: int, Skv: int) -> int:
    """SB200_ATTN_BWD_SPLITS: the query-split count bound of `attention_bwd_split` (1 = the unsplit launches)."""
    if Skv > 128 or 2 * B * heads > 132:
        return 1
    return min((132 + B * heads - 1) // (B * heads), (Sq + 63) // 64)


def attention_bwd_split(q, k, v, o, dout, lse, B: int, heads: int, Sq: int, Skv: int, scale: float, head_dim: int,
                        dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor) -> None:
    """`attention_bwd` with dK / dV through `sb200_attention_bwd_ws`: for a short key sequence on few (head, batch)
    pairs (cross-attention) the dV and dK launches split the queries over SB200_ATTN_BWD_SPLITS CTAs per pair, and
    `attn_bwd_reduce_kernel` sums their fp32 partials in order.  Other shapes run exactly as `attention_bwd`."""
    dsum = torch.empty(B * heads * Sq, device=q.device, dtype=torch.float32)
    nsplit = attn_bwd_splits(B, heads, Sq, Skv)
    ws_n = 2 * nsplit * B * Skv * heads * head_dim if nsplit > 1 else 0
    ws = torch.empty(max(ws_n, 1), device=q.device, dtype=torch.float32)
    lib = _begin()
    _cabi.check(lib.sb200_attention_bwd_ws(
        _ctx(q), _stream(), _p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(o), o.stride(0),
        _p(dout), dout.stride(0), _p(lse), _p(dsum), _p(dq), dq.stride(0), _p(dk), dk.stride(0), _p(dv), dv.stride(0),
        B, heads, Sq, Skv, int(head_dim), float(scale), _p(ws), ws_n))
    global launch_count
    launch_count += 2 if nsplit == 1 else 3
    _count("attention_bwd", 14.0 * B * heads * Sq * Skv * head_dim)


def splitk_ws_floats(M: int, N: int, K: int) -> int:
    """SB200_GEMM_SPLITK_WS_FLOATS."""
    tiles = ((M + 127) // 128) * (N // 128 if N % 128 == 0 else (N + 63) // 64)
    want = (132 + tiles - 1) // tiles
    kbs = (K + 63) // 64
    kb = max(8, (kbs + want - 1) // want)
    return ((kbs + kb - 1) // kb) * M * N


def gemm_splitk_f32(x: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 out[M, N] = x[M, K] @ w[N, K].T (bf16 operands): `gemm_kernel` in split-K mode + `splitk_reduce_kernel`."""
    M, K = x.shape
    N = w.shape[0]
    assert w.shape[1] == K
    if out is None:
        out = torch.empty((M, N), device=x.device, dtype=torch.float32)
    n_ws = splitk_ws_floats(M, N, K)
    ws = torch.empty(n_ws, device=x.device, dtype=torch.float32)
    lib = _begin()
    _cabi.check(lib.sb200_gemm_splitk_f32(_ctx(x), _stream(), _p(x), x.stride(0), _p(w), w.stride(0), _p(out),
                                          out.stride(0), M, N, K, _p(ws), n_ws))
    global launch_count
    launch_count += 1
    _count("gemm", 2.0 * M * N * K)
    return out


def guided_step_loss_fwd(eps_u, eps_c, g: float, x, cx: float, ce: float, target) -> torch.Tensor:
    """fp32 scalar mean((cx x + ce (eps_u + g (eps_c - eps_u)) - target)^2): `guided_loss_kernel` + finalize."""
    n = eps_u.numel()
    parts = min(256, n // 2048 + 1)  # SB200_GUIDED_LOSS_BLOCKS
    ws = torch.empty(parts, device=eps_u.device, dtype=torch.float32)
    loss = torch.empty((), device=eps_u.device, dtype=torch.float32)
    lib = _begin()
    _cabi.check(lib.sb200_guided_step_loss(_ctx(eps_u), _stream(), _p(eps_u), _p(eps_c), float(g), _p(x), float(cx),
                                           float(ce), _p(target), n, 0, _p(loss), _p(ws), None, None))
    global launch_count
    launch_count += 1
    _count()
    return loss


def guided_step_loss_bwd(eps_u, eps_c, g: float, x, cx: float, ce: float, target, dloss) -> torch.Tensor:
    """d loss / d eps_u scaled by the device scalar dloss: one `guided_loss_kernel` launch."""
    d = torch.empty_like(eps_u)
    lib = _begin()
    _cabi.check(lib.sb200_guided_step_loss(_ctx(eps_u), _stream(), _p(eps_u), _p(eps_c), float(g), _p(x), float(cx),
                                           float(ce), _p(target), eps_u.numel(), 1, None, None, _p(dloss), _p(d)))
    _count()
    return d


class GuidedStepLoss(torch.autograd.Function):
    """loss = mse(cx x + ce (eps_u + g (eps_c - eps_u)), target) with a gradient for eps_u only (the null-text inner
    step: eps_c, x and target are constants).  All tensors fp32 CUDA, contiguous, of one shape."""

    @staticmethod
    def forward(fctx, eps_u, eps_c, g, x, cx, ce, target):
        for t in (eps_u, eps_c, x, target):
            if t.dtype != torch.float32 or not t.is_contiguous() or t.shape != eps_u.shape:
                raise ValueError("guided_step_loss: eps_u, eps_c, x and target must be contiguous fp32 of one shape")
        fctx.save_for_backward(eps_u, eps_c, x, target)
        fctx.coef = (float(g), float(cx), float(ce))
        return guided_step_loss_fwd(eps_u, eps_c, g, x, cx, ce, target)

    @staticmethod
    def backward(fctx, dloss):
        eps_u, eps_c, x, target = fctx.saved_tensors
        g, cx, ce = fctx.coef
        d = guided_step_loss_bwd(eps_u, eps_c, g, x, cx, ce, target, dloss.to(torch.float32).contiguous())
        return d, None, None, None, None, None, None


def guided_step_loss(eps_u, eps_c, g: float, x, cx: float, ce: float, target) -> torch.Tensor:
    return GuidedStepLoss.apply(eps_u, eps_c, g, x, cx, ce, target)


def groupnorm_bwd(x0, gamma, beta, groups: int, silu: bool, dy, stats_ws, *, x1=None, add=None) -> torch.Tensor:
    """Input gradient of `groupnorm` (concat layout [.., C0 + C1]); stats_ws is the forward's workspace, or its
    (mean, rstd) block as a [B, groups, 2] tensor (`gn_stats` — sliceable along the batch)."""
    shp = x0.shape
    B, C0 = shp[0], shp[-1]
    HW = x0.numel() // (B * C0)
    C1 = x1.shape[-1] if x1 is not None else 0
    Cc = C0 + C1
    dx = torch.empty(shp[:-1] + (Cc,), device=x0.device, dtype=BF16)
    ws = gn_ws(B, groups, x0.device)
    fwd = stats_ws if stats_ws.dim() == 3 else stats_ws[B * groups * 2 * GN_STATS_OFFSET:]
    assert fwd.is_contiguous()
    lib = _begin()
    _cabi.check(lib.sb200_groupnorm_bwd(
        _ctx(x0), _stream(), _p(x0), x0.stride(-2), C0, _p(x1), x1.stride(-2) if x1 is not None else 0, C1,
        _p(gamma), _p(beta), _p(dy), dy.stride(-2), _p(add), add.stride(-2) if add is not None else 0, _p(dx), Cc,
        B, HW, groups, int(silu), _p(fwd), _p(ws)))
    _count("groupnorm_bwd")
    return dx


def layernorm_bwd(x, gamma, dy, eps: float = 1e-5, add=None) -> torch.Tensor:
    M, Cc = x.shape
    dx = torch.empty((M, Cc), device=x.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_layernorm_bwd(_ctx(x), _stream(), _p(x), x.stride(0), _p(gamma), _p(dy), dy.stride(0),
                                        _p(add), add.stride(0) if add is not None else 0, _p(dx), Cc, M, Cc,
                                        float(eps)))
    _count()
    return dx


def geglu(pre: torch.Tensor) -> torch.Tensor:
    M, F2 = pre.shape
    out = torch.empty((M, F2 // 2), device=pre.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_geglu(_ctx(pre), _stream(), _p(pre), pre.stride(0), _p(out), F2 // 2, M, F2 // 2))
    _count()
    return out


def geglu_bwd(pre: torch.Tensor, dout: torch.Tensor) -> torch.Tensor:
    M, F2 = pre.shape
    dpre = torch.empty((M, F2), device=pre.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_geglu_bwd(_ctx(pre), _stream(), _p(pre), pre.stride(0), _p(dout), dout.stride(0),
                                    _p(dpre), F2, M, F2 // 2))
    _count()
    return dpre


def add(a: torch.Tensor, b: torch.Tensor, c: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None):
    """a + b (+ c) on 2-D (row-strided) bf16 matrices."""
    M, Cc = a.shape
    if out is None:
        out = torch.empty((M, Cc), device=a.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_add(_ctx(a), _stream(), _p(a), a.stride(0), _p(b), b.stride(0), _p(c),
                              c.stride(0) if c is not None else 0, _p(out), out.stride(0), M, Cc))
    _count()
    return out


def upsample2x_bwd(dy: torch.Tensor) -> torch.Tensor:
    B, H2, W2, Cc = dy.shape
    dx = torch.empty((B, H2 // 2, W2 // 2, Cc), device=dy.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_upsample2x_bwd(_ctx(dy), _stream(), _p(dy), _p(dx), B, H2 // 2, W2 // 2, Cc))
    _count()
    return dx


def zero_stuff(dy: torch.Tensor) -> torch.Tensor:
    B, Ho, Wo, Cc = dy.shape
    z = torch.empty((B, 2 * Ho, 2 * Wo, Cc), device=dy.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_zero_stuff(_ctx(dy), _stream(), _p(dy), _p(z), B, Ho, Wo, Cc))
    _count()
    return z


def conv_out_bwd(deps: torch.Tensor, w_packed: torch.Tensor) -> torch.Tensor:
    """deps: NCHW [B,4,H,W] fp32 / bf16 -> NHWC bf16 [B,H,W,C]."""
    B, _, H, W = deps.shape
    Cc = w_packed.shape[-1]
    deps = deps.contiguous()
    dx = torch.empty((B, H, W, Cc), device=deps.device, dtype=BF16)
    lib = _begin()
    _cabi.check(lib.sb200_conv_out_bwd(_ctx(deps), _stream(), _p(deps), int(deps.dtype == torch.float32),
                                       _p(w_packed), _p(dx), B, H, W, Cc))
    _count()
    return dx


def colsum(dy: torch.Tensor) -> torch.Tensor:
    """dy [B, H, W, C] (or [B, HW, C]) -> fp32 [B, C]."""
    B, Cc = dy.shape[0], dy.shape[-1]
    HW = dy.numel() // (B * Cc)
    out = torch.empty((B, Cc), device=dy.device, dtype=torch.float32)
    lib = _begin()
    _cabi.check(lib.sb200_colsum(_ctx(dy), _stream(), _p(dy), dy.stride(-2), _p(out), B, HW, Cc))
    _count()
    return out


def _wgrad_ws(Cc: int, r: int, device) -> torch.Tensor:
    cblocks = (Cc // 8 + 31) // 32
    chunks = min(256, (264 + cblocks - 1) // cblocks)
    return torch.empty(chunks * Cc * r, device=device, dtype=torch.float32)


def lora_proj(A: torch.Tensor, Bt: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """A [M, C] bf16 (row-strided), Bt [r, C] bf16 (row-strided) -> fp32 [M, r] = A @ Bt.T; with `out` given the
    product is accumulated into it (two-source inputs: x = [x0 | x1])."""
    M, Cc = A.shape
    r = Bt.shape[0]
    T = out if out is not None else torch.empty((M, r), device=A.device, dtype=torch.float32)
    lib = _begin()
    _cabi.check(lib.sb200_lora_proj(_ctx(A), _stream(), _p(A), A.stride(0), _p(Bt), Bt.stride(0), _p(T), M, Cc, r,
                                    int(out is not None)))
    _count()
    return T


def lora_wgrad(A: torch.Tensor, T: torch.Tensor, G: torch.Tensor, transposed: bool, scale: float,
               accumulate: bool = False) -> None:
    """G (+)= scale * A.T @ T.  A [M, C] bf16, T [M, r] fp32; G fp32 (any strides, e.g. a column slice):
    [C, r] (transposed=False) or [r, C] (transposed=True)."""
    M, Cc = A.shape
    r = T.shape[1]
    gs_c, gs_r = (G.stride(1), G.stride(0)) if transposed else (G.stride(0), G.stride(1))
    ws = _wgrad_ws(Cc, r, A.device)
    lib = _begin()
    _cabi.check(lib.sb200_lora_wgrad(_ctx(A), _stream(), _p(A), A.stride(0), _p(T), _p(G), gs_c, gs_r, float(scale),
                                     int(accumulate), M, Cc, r, _p(ws)))
    _count("lora_wgrad")


def lora_rank_update(dX: torch.Tensor, U: torch.Tensor, D: torch.Tensor, scale: float) -> None:
    """dX += scale * U @ D   (dX [M, C] bf16 in place, U [M, r] fp32, D [r, C] bf16)."""
    M, Cc = dX.shape
    lib = _begin()
    _cabi.check(lib.sb200_lora_rank_update(_ctx(dX), _stream(), _p(dX), dX.stride(0), _p(U), _p(D), D.stride(0),
                                           float(scale), M, Cc, U.shape[1]))
    _count()


def lora_conv_proj(x0: torch.Tensor, D: torch.Tensor, stride: int = 1, x1: Optional[torch.Tensor] = None):
    """3x3 / pad 1 conv of NHWC x (= [x0 | x1]) with D [r, 3, 3, C] -> fp32 [B*Ho*Wo, r]."""
    B, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    r = D.shape[0]
    T = torch.empty((B * (H // stride) * (W // stride), r), device=x0.device, dtype=torch.float32)
    lib = _begin()
    _cabi.check(lib.sb200_lora_conv_proj(_ctx(x0), _stream(), _p(x0), x0.stride(2), C0, _p(x1),
                                         x1.stride(2) if x1 is not None else 0, C1, _p(D), _p(T), B, H, W, stride, r))
    _count()
    return T


def lora_conv_wgrad(x0: torch.Tensor, U: torch.Tensor, G: torch.Tensor, scale: float, stride: int = 1,
                    x1: Optional[torch.Tensor] = None, accumulate: bool = False) -> None:
    """G [r, 3, 3, C] fp32 (+)= scale * sum_p U[p, :] (x) patch(x, p)."""
    B, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    r = U.shape[1]
    ws = _wgrad_ws(9 * (C0 + C1), r, x0.device)
    lib = _begin()
    _cabi.check(lib.sb200_lora_conv_wgrad(_ctx(x0), _stream(), _p(x0), x0.stride(2), C0, _p(x1),
                                          x1.stride(2) if x1 is not None else 0, C1, _p(U), _p(G), float(scale),
                                          int(accumulate), B, H, W, stride, r, _p(ws)))
    _count("lora_wgrad")


def lora_conv_rank_update(dX: torch.Tensor, U: torch.Tensor, D: torch.Tensor, scale: float, stride: int = 1) -> None:
    """dX [B,H,W,C] (contiguous, in place) += scale * conv_transpose(U [B,Ho,Wo,r], D [r,3,3,C])."""
    B, H, W, Cc = dX.shape
    assert dX.is_contiguous()
    lib = _begin()
    _cabi.check(lib.sb200_lora_conv_rank_update(_ctx(dX), _stream(), _p(dX), _p(U), _p(D), float(scale), B, H, W, Cc,
                                                stride, U.shape[1]))
    _count()


def adamw(table: torch.Tensor, n_tensors: int, max_numel: int, lr: float, beta1: float, beta2: float, eps: float,
          weight_decay: float, step: int) -> None:
    """One fused `adamw_kernel` launch over a device table of (p, g, m, v, n) records (int64 [n_tensors, 5])."""
    lib = _begin()
    _cabi.check(lib.sb200_adamw(_ctx(table), _stream(), _p(table), n_tensors, int(max_numel), float(lr), float(beta1),
                                float(beta2), float(eps), float(weight_decay), int(step)))
    _count()


def adam_f32(table: torch.Tensor, n_tensors: int, max_numel: int, lr: float, beta1: float, beta2: float, eps: float,
             weight_decay: float, step: int) -> None:
    """One `adam_f32_kernel` launch over a device table of fp32 (p, g, m, v, n) records (int64 [n_tensors, 5])."""
    lib = _begin()
    _cabi.check(lib.sb200_adam_f32(_ctx(table), _stream(), _p(table), n_tensors, int(max_numel), float(lr),
                                   float(beta1), float(beta2), float(eps), float(weight_decay), int(step)))
    _count()
