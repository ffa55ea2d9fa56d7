"""Thin torch-tensor wrappers over the C ABI (include/sb200.h).  Every function enqueues exactly the
kernels named in its docstring on torch's *current* stream, so the whole UNet forward can be captured in a
CUDA graph.  There is deliberately no PyTorch fallback: a missing extension or a CPU tensor raises.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Tuple

import torch

from . import _cabi
from ._cabi import CONV_PAD_BR, EPI_BIAS, EPI_GEGLU, EPI_LORA, EPI_RESID, EPI_ROWBIAS, LoraArgs

BF16 = torch.bfloat16

# launches issued through this module since import (bench.py reports it as gpu_launches)
launch_count = 0


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


# Optional call recording (bench.py's per-kernel-class timing): while `record_calls` is a list and the current stream is
# being captured into a CUDA graph, every C-ABI call is remembered as [fn, args, name, flops].  `replay_calls` re-issues
# a subset on the current stream (normally under a second capture): same kernels, same buffers (they live in the first
# graph's memory pool), so a class of kernels can be timed back to back as its own graph.
record_calls = None


def replay_calls(calls) -> None:
    stream = _stream()
    for fn, args, _, _ in calls:
        assert isinstance(args[1], C.c_void_p), "C-ABI convention: (handle, stream, ...)"
        _cabi.check(fn(args[0], stream, *args[2:]))


def _call(fn: str, anchor: torch.Tensor, *args, kernels: int = 1, name: str = "other", flops: float = 0.0) -> None:
    """C-ABI function `fn`(handle of anchor's device, current stream, *args), which enqueues `kernels` launches, with
    the module's launch count, profiling and call recording."""
    global launch_count
    if profile_log is not None:
        start = torch.cuda.Event(enable_timing=True)
        start.record()
    f = getattr(_cabi.load(), fn)
    args = (_ctx(anchor), _stream()) + args
    entry = None
    if record_calls is not None and torch.cuda.is_current_stream_capturing():
        entry = [f, args, None, 0.0]
        record_calls.append(entry)
    _cabi.check(f(*args))
    launch_count += kernels
    if entry is not None:
        entry[2], entry[3] = name, flops
    if profile_log is not None:
        end = torch.cuda.Event(enable_timing=True)
        end.record()
        profile_log.append((name, flops, start, end))


def _epilogue(bias, rowbias, resid, lora, geglu: bool = False) -> int:
    """The SB200_EPI_* flag word of a `gemm` / `conv3x3` call."""
    return ((EPI_BIAS if bias is not None else 0) | (EPI_ROWBIAS if rowbias is not None else 0)
            | (EPI_RESID if resid is not None else 0) | (EPI_GEGLU if geglu else 0)
            | (EPI_LORA if lora is not None else 0))


LORA_MAX_RANK = 16


def lora_slots(r: int, groups: int = 1) -> Tuple[int, int]:
    """(rp, rt) of `groups` adaptors of rank up to r fused into one call: each adaptor takes a slot of rp = 4, 8 or 16
    down rows / up columns (the smallest that holds r; the rows and columns beyond r are zero, so the padded terms add
    exact zeros to every fp32 sum), and the stacked down rows are padded to rt = 16, 32 or 64 (sb200_lora.rt)."""
    if not 1 <= r <= LORA_MAX_RANK:
        raise NotImplementedError(f"LoRA rank {r}: the fused kernels support ranks 1-{LORA_MAX_RANK}")
    rp = next(w for w in (4, 8, 16) if r <= w)
    need = groups * rp
    if need > 64:
        raise NotImplementedError(f"{groups} adaptors of rank {r} in one fused call need {need} > 64 LoRA rows")
    rt = next(w for w in (16, 32, 64) if need <= w)
    return rp, rt


class Lora:
    """Packed LoRA side inputs of one fused GEMM/conv call (see struct sb200_lora).

    sample_scale: optional fp32 device vector of per-sample factors; output row m of the LoRA term is multiplied by
    sample_scale[m // rows_per_sample].  rows_per_sample 0 lets `gemm` / `conv3x3` / `small_linear` derive it from the
    call as M // sample_scale.numel() (the vector then has one entry per batch entry of that call)."""

    __slots__ = ("down", "up", "r", "rt", "group_n", "scale", "scale_dev", "sample_scale", "rows_per_sample", "_c")

    def __init__(self, down: torch.Tensor, up: torch.Tensor, r: int, group_n: int, scale: float,
                 scale_dev: Optional[torch.Tensor] = None, sample_scale: Optional[torch.Tensor] = None,
                 rows_per_sample: int = 0):
        self.down, self.up, self.r, self.rt, self.group_n = down, up, r, down.shape[0], group_n
        self.scale, self.scale_dev = float(scale), scale_dev
        self.sample_scale, self.rows_per_sample = sample_scale, int(rows_per_sample)
        self._c = LoraArgs(down.data_ptr(), up.data_ptr(), r, self.rt, group_n, self.scale,
                           scale_dev.data_ptr() if scale_dev is not None else None,
                           sample_scale.data_ptr() if sample_scale is not None else None, self.rows_per_sample)

    def ref(self, M: int = 0):
        """The struct for a launch with M output rows; fills a derived rows_per_sample (see the class docstring)."""
        if self.sample_scale is not None and self.rows_per_sample == 0:
            n = self.sample_scale.numel()
            if M % n != 0:
                raise ValueError(f"LoRA sample_scale: {n} per-sample factors do not divide the call's {M} rows")
            self._c.rows_per_sample = M // n
        return C.byref(self._c)


def gemm(x: torch.Tensor, w: torch.Tensor, *, bias=None, rowbias=None, rows_per_batch: int = 1, resid=None,
         geglu: bool = False, lora: Optional[Lora] = None, x1: Optional[torch.Tensor] = None,
         out: Optional[torch.Tensor] = None, bn: int = 0) -> torch.Tensor:
    """out[M,N] = epilogue([x | x1] @ w.T): one wgmma `gemm_kernel` launch."""
    M, K0 = x.shape
    N, K = w.shape
    flags = _epilogue(bias, rowbias, resid, lora, geglu)
    nout = N // 2 if geglu else N
    if out is None:
        out = torch.empty((M, nout), device=x.device, dtype=BF16)
    _call("sb200_gemm", x, _p(x), x.stride(0), _p(x1), x1.stride(0) if x1 is not None else 0, K0,
          _p(w), w.stride(0), _p(out), out.stride(0), M, N, K, flags, _p(bias), _p(rowbias), rows_per_batch,
          _p(resid), resid.stride(0) if resid is not None else 0, lora.ref(M) if lora is not None else None, bn,
          name="gemm", flops=2.0 * M * N * K)
    return out


def conv3x3(x0: torch.Tensor, w_packed: torch.Tensor, *, x1: Optional[torch.Tensor] = None, stride: int = 1,
            bias=None, rowbias=None, resid=None, lora: Optional[Lora] = None, out: Optional[torch.Tensor] = None,
            bn: int = 0, pad_bottom_right: bool = False) -> torch.Tensor:
    """3x3 / pad 1 conv on NHWC bf16 ([B,H,W,C] tensors); w_packed is [Cout,3,3,Cin].  One `gemm_kernel`.
    `out`: [B, Ho, Wo, Cout] whose pixels are rows of one 2-D matrix with row stride out.stride(2) (e.g. a column
    slice of a wider NHWC buffer).  pad_bottom_right (stride 2 only): the conv of F.pad(x, (0, 1, 0, 1)) with
    padding 0, as diffusers' Downsample2D in the VAE encoder (SB200_CONV_PAD_BR)."""
    B, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    Cout = w_packed.shape[0]
    flags = _epilogue(bias, rowbias, resid, lora) | (CONV_PAD_BR if pad_bottom_right else 0)
    Ho, Wo = H // stride, W // stride
    if out is None:
        out = torch.empty((B, Ho, Wo, Cout), device=x0.device, dtype=BF16)
    elif (tuple(out.shape) != (B, Ho, Wo, Cout) or out.stride(3) != 1 or out.stride(1) != Wo * out.stride(2)
          or out.stride(0) != Ho * out.stride(1)):
        raise ValueError(f"conv3x3: out {tuple(out.shape)} / strides {out.stride()} is not a [B*Ho*Wo, ldo] matrix "
                         f"of [{B}, {Ho}, {Wo}, {Cout}]")
    _call("sb200_conv3x3", x0, _p(x0), x0.stride(2), _p(x1), x1.stride(2) if x1 is not None else 0, C0, C1,
          _p(w_packed), _p(out), out.stride(2), B, H, W, Cout, stride, flags, _p(bias), _p(rowbias), _p(resid),
          resid.stride(2) if resid is not None else 0, lora.ref(B * Ho * Wo) if lora is not None else None, bn,
          name="conv3x3", flops=2.0 * B * Ho * Wo * Cout * 9 * (C0 + C1))
    return out


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, B: int, heads: int, Sq: int, Skv: int,
              scale: float, head_dim: int = 64, lse: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q/k/v: 2-D (possibly column-sliced) token matrices; head h = columns [h*head_dim, (h+1)*head_dim).
    One `attention_kernel`.  lse: optional fp32 [B, heads, Sq] output kept for `attention_bwd`.
    The kernel's TMA descriptors cover exactly B * Sq query and B * Skv key rows of at least heads * head_dim
    columns, so other layouts raise ValueError."""
    for name, t, rows in (("q", q, B * Sq), ("k", k, B * Skv), ("v", v, B * Skv)):
        if t.dim() != 2 or t.shape[0] != rows or t.shape[1] < heads * head_dim:
            raise ValueError(f"attention: {name} {tuple(t.shape)} is not a [{rows}, >= {heads * head_dim}] matrix")
        _row_matrix(t, t.shape, "attention", name)
    if lse is not None and (tuple(lse.shape) != (B, heads, Sq) or lse.dtype != torch.float32
                            or not lse.is_contiguous()):
        raise ValueError(f"attention: lse {tuple(lse.shape)} {lse.dtype} is not a contiguous fp32 [{B}, {heads}, {Sq}]")
    out = torch.empty((B * Sq, heads * head_dim), device=q.device, dtype=BF16)
    _call("sb200_attention", q, _p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(out), out.stride(0),
          B, heads, Sq, Skv, int(head_dim), float(scale), _p(lse),
          name="attention", flops=4.0 * B * heads * Sq * Skv * head_dim)
    return out


def groupnorm(x0: torch.Tensor, gamma, beta, groups: int, eps: float, silu: bool, *,
              x1: Optional[torch.Tensor] = None, stats_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x0/x1: [B, HW, C] (or [B,H,W,C]) NHWC; returns the concatenated, normalised tensor."""
    shp = x0.shape
    B, C0 = shp[0], shp[-1]
    HW = x0.numel() // (B * C0)
    C1 = x1.shape[-1] if x1 is not None else 0
    _row_matrix(x0, shp, "groupnorm", "x0")
    if x1 is not None:
        if tuple(x1.shape[:-1]) != tuple(shp[:-1]):
            raise ValueError(f"groupnorm: x1 {tuple(x1.shape)} has other batch / pixel dims than x0 {tuple(shp)}")
        _row_matrix(x1, x1.shape, "groupnorm", "x1")
    out = torch.empty(shp[:-1] + (C0 + C1,), device=x0.device, dtype=BF16)
    if stats_ws is None:
        stats_ws = gn_ws(B, groups, x0.device)
    _call("sb200_groupnorm", x0, _p(x0), x0.stride(-2), C0, _p(x1), x1.stride(-2) if x1 is not None else 0, C1,
          _p(gamma), _p(beta), _p(out), C0 + C1, B, HW, groups, float(eps), int(silu), _p(stats_ws),
          kernels=3, name="groupnorm")
    return out


def layernorm(x: torch.Tensor, gamma, beta, eps: float = 1e-5) -> torch.Tensor:
    M, Cc = x.shape
    _row_matrix(x, (M, Cc), "layernorm", "x")
    out = torch.empty((M, Cc), device=x.device, dtype=BF16)
    _call("sb200_layernorm", x, _p(x), x.stride(0), _p(gamma), _p(beta), _p(out), Cc, M, Cc, float(eps),
          name="layernorm")
    return out


def small_linear(x: torch.Tensor, w: torch.Tensor, bias=None, *, act_in: bool = False, act_out: int = 0,
                 lora: Optional[Lora] = None, resid: Optional[torch.Tensor] = None) -> torch.Tensor:
    """act_out: 0 none, 1 SiLU(y) + resid, 2 SiLU(bf16(y + resid)) — see sb200_small_linear.  The kernel reads
    resid[m * N + n], so resid must be a contiguous [M, N]."""
    M, K = x.shape
    N = w.shape[0]
    _row_matrix(x, (M, K), "small_linear", "x")
    _row_matrix(w, (N, K), "small_linear", "w")
    if resid is not None and (tuple(resid.shape) != (M, N) or resid.dtype != BF16 or not resid.is_contiguous()):
        raise ValueError(f"small_linear: resid {tuple(resid.shape)} {resid.dtype} / strides {resid.stride()} is not a "
                         f"contiguous [{M}, {N}] bf16 matrix")
    out = torch.empty((M, N), device=x.device, dtype=BF16)
    _call("sb200_small_linear", x, _p(x), x.stride(0), _p(w), w.stride(0), _p(bias), _p(out), N, M, N, K,
          int(act_in), int(act_out), lora.ref(M) if lora is not None else None, _p(resid), name="small_linear")
    return out


def sinusoid(values: torch.Tensor, dim: int) -> torch.Tensor:
    """values: fp32 [n] on device -> [n, dim] bf16 ([cos | sin])."""
    n = values.numel()
    out = torch.empty((n, dim), device=values.device, dtype=BF16)
    _call("sb200_sinusoid", values, _p(values), n, dim, _p(out), dim, name="sinusoid")
    return out


def conv_in(latent: torch.Tensor, w_packed: torch.Tensor, bias) -> torch.Tensor:
    """latent: NCHW fp32 or bf16 -> NHWC bf16 [B,H,W,Cout]."""
    B, Cc, H, W = latent.shape
    assert Cc == 4 and latent.is_contiguous()
    Cout = w_packed.shape[0]
    out = torch.empty((B, H, W, Cout), device=latent.device, dtype=BF16)
    _call("sb200_conv_in", latent, _p(latent), int(latent.dtype == torch.float32), _p(w_packed), _p(bias), _p(out),
          B, H, W, Cout, name="conv_in")
    return out


def conv_out(x: torch.Tensor, w_packed: torch.Tensor, bias, out_dtype=BF16) -> torch.Tensor:
    """x: contiguous NHWC bf16 [B, H, W, Cin] -> NCHW [B, 4, H, W]."""
    B, H, W, Cin = x.shape
    if x.dtype != BF16 or not x.is_contiguous():
        raise ValueError(f"conv_out: x {tuple(x.shape)} {x.dtype} / strides {x.stride()} is not contiguous NHWC bf16")
    out = torch.empty((B, 4, H, W), device=x.device, dtype=out_dtype)
    _call("sb200_conv_out", x, _p(x), _p(w_packed), _p(bias), _p(out), int(out_dtype == torch.float32), B, H, W, Cin,
          name="conv_out")
    return out


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    """x: contiguous NHWC bf16 [B, H, W, C] -> [B, 2H, 2W, C] (nearest)."""
    B, H, W, Cc = x.shape
    if x.dtype != BF16 or not x.is_contiguous():
        raise ValueError(f"upsample2x: x {tuple(x.shape)} {x.dtype} / strides {x.stride()} is not contiguous NHWC bf16")
    out = torch.empty((B, 2 * H, 2 * W, Cc), device=x.device, dtype=BF16)
    _call("sb200_upsample2x", x, _p(x), _p(out), B, H, W, Cc, name="upsample2x")
    return out


def _image_shape(t: torch.Tensor, what: str, name: str, dtype, C: Optional[int] = None):
    if t.dim() != 4 or t.dtype != dtype or not t.is_contiguous() or (C is not None and t.shape[-1] != C):
        raise ValueError(f"{what}: {name} {tuple(t.shape)} {t.dtype} / strides {t.stride()} is not a contiguous "
                         f"[B, H, W, {C if C is not None else 'C'}] {dtype} tensor")
    return t.shape


def vae_conv_in_u8(img: torch.Tensor, w_packed: torch.Tensor, bias) -> torch.Tensor:
    """uint8 [B, H, W, 3] pixels -> NHWC bf16 [B, H, W, Cout]: preprocess (v / 255 * 2 - 1) + the VAE encoder's
    conv_in.  One `vae_conv_in_u8_kernel`."""
    B, H, W, _ = _image_shape(img, "vae_conv_in_u8", "img", torch.uint8, 3)
    Cout = w_packed.shape[0]
    out = torch.empty((B, H, W, Cout), device=img.device, dtype=BF16)
    _call("sb200_vae_conv_in_u8", img, _p(img), _p(w_packed), _p(bias), _p(out), B, H, W, Cout,
          name="vae_conv_in_u8", flops=2.0 * B * H * W * Cout * 27)
    return out


def vae_conv_out_u8(x: torch.Tensor, w_packed: torch.Tensor, bias, return_float: bool = False):
    """NHWC bf16 [B, H, W, Cin] (normalised + SiLU) -> uint8 [B, H, W, 3]: the VAE decoder's conv_out + postprocess
    (rint(clamp(y / 2 + 0.5, 0, 1) * 255)).  return_float: (uint8, fp32 NCHW [B, 3, H, W] y).  One
    `vae_conv_out_u8_kernel`."""
    B, H, W, Cin = _image_shape(x, "vae_conv_out_u8", "x", BF16)
    img = torch.empty((B, H, W, 3), device=x.device, dtype=torch.uint8)
    y = torch.empty((B, 3, H, W), device=x.device, dtype=torch.float32) if return_float else None
    _call("sb200_vae_conv_out_u8", x, _p(x), _p(w_packed), _p(bias), _p(img), _p(y), B, H, W, Cin,
          name="vae_conv_out_u8", flops=2.0 * B * H * W * 3 * 9 * Cin)
    return (img, y) if return_float else img


def vae_moments(x: torch.Tensor, w_packed: torch.Tensor, bias, quant_w: torch.Tensor, quant_b: torch.Tensor,
                eps: Optional[torch.Tensor], scaling: float) -> torch.Tensor:
    """NHWC bf16 [B, h, w, Cin] -> fp32 [B, 4, h, w] scaled latents: the VAE encoder's conv_out (Cin -> 8), quant_conv
    (fp32 [8, 8] + [8]), logvar clamp, mean + exp(logvar / 2) * eps (eps None: the mean), times scaling.  One
    `vae_moments_kernel`."""
    B, H, W, Cin = _image_shape(x, "vae_moments", "x", BF16)
    if tuple(quant_w.shape) != (8, 8) or quant_w.dtype != torch.float32 or quant_b.dtype != torch.float32:
        raise ValueError("vae_moments: quant_w / quant_b must be fp32 [8, 8] / [8]")
    if eps is not None and (tuple(eps.shape) != (B, 4, H, W) or eps.dtype != torch.float32 or not eps.is_contiguous()):
        raise ValueError(f"vae_moments: eps {tuple(eps.shape)} {eps.dtype} is not a contiguous fp32 [{B}, 4, {H}, {W}]")
    z = torch.empty((B, 4, H, W), device=x.device, dtype=torch.float32)
    _call("sb200_vae_moments", x, _p(x), _p(w_packed), _p(bias), _p(quant_w.contiguous()), _p(quant_b.contiguous()),
          _p(eps), float(scaling), _p(z), B, H, W, Cin, name="vae_moments", flops=2.0 * B * H * W * 8 * 9 * Cin)
    return z


def vae_post_quant(z: torch.Tensor, post_w: torch.Tensor, post_b: torch.Tensor, scaling: float) -> torch.Tensor:
    """fp32 NCHW [B, 4, h, w] -> post_quant_conv(z / scaling) (fp32 [4, 4] + [4]).  One `vae_post_quant_kernel`."""
    if z.dim() != 4 or z.shape[1] != 4 or z.dtype != torch.float32 or not z.is_contiguous():
        raise ValueError(f"vae_post_quant: z {tuple(z.shape)} {z.dtype} is not a contiguous fp32 [B, 4, h, w]")
    if tuple(post_w.shape) != (4, 4) or post_w.dtype != torch.float32 or post_b.dtype != torch.float32:
        raise ValueError("vae_post_quant: post_w / post_b must be fp32 [4, 4] / [4]")
    out = torch.empty_like(z)
    _call("sb200_vae_post_quant", z, _p(z), _p(post_w.contiguous()), _p(post_b.contiguous()), float(scaling), _p(out),
          z.shape[0], z.shape[2] * z.shape[3], name="vae_post_quant")
    return out


def softmax_rows(s: torch.Tensor, scale: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 scores [rows, cols] (row-strided) -> bf16 softmax(scale * s) per row, max and sum in fp32.  One
    `softmax_rows_kernel`."""
    rows, cols = s.shape
    _row_matrix(s, (rows, cols), "softmax_rows", "s", dtype=torch.float32)
    p = _out(out, (rows, cols), "softmax_rows", s.device)
    _call("sb200_softmax_rows", s, _p(s), s.stride(0), _p(p), p.stride(0), rows, cols, float(scale),
          name="softmax_rows")
    return p


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
    if not eps2.is_contiguous() or (not single and eps2.shape[0] % 2):
        raise ValueError(f"cfg_ddim: eps2 {tuple(eps2.shape)} / strides {eps2.stride()} is not a contiguous "
                         f"{'eps' if single else '[uncond ; cond]'} batch")
    if x is not None and (not x.is_contiguous() or x.numel() != n):
        raise ValueError(f"cfg_ddim: x {tuple(x.shape)} / strides {x.stride()} is not contiguous with {n} elements")
    if eps2.dtype not in (torch.float32, BF16):
        eps2 = eps2.to(torch.float32)
    out_dtype = out_dtype or (x.dtype if x is not None else eps2.dtype)
    eps_out = torch.empty(shape, device=eps2.device, dtype=out_dtype)
    x_prev = torch.empty(shape, device=eps2.device, dtype=out_dtype) if x is not None else None
    if x is not None and x.dtype != out_dtype:
        x = x.to(out_dtype)
    _call("sb200_cfg_step" if affine else "sb200_cfg_ddim", eps2, _p(eps2), int(eps2.dtype == torch.float32),
          float(guidance), _p(x), float(a_t), float(a_prev), _p(x_prev), _p(eps_out), int(out_dtype == torch.float32), n,
          name="cfg_ddim")
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
    _call("sb200_attention_bwd", q, _p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(o), o.stride(0),
          _p(dout), dout.stride(0), _p(lse), _p(dsum), _p(dq), dq.stride(0), _p(dk),
          dk.stride(0) if dk is not None else 0, _p(dv), dv.stride(0) if dv is not None else 0, B, heads, Sq, Skv,
          int(head_dim), float(scale), kernels=2 if dk is None else 3, name="attention_bwd",
          flops=(6.0 if dk is None else 14.0) * B * heads * Sq * Skv * head_dim)


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
    _call("sb200_attention_bwd_ws", q, _p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(o), o.stride(0),
          _p(dout), dout.stride(0), _p(lse), _p(dsum), _p(dq), dq.stride(0), _p(dk), dk.stride(0), _p(dv), dv.stride(0),
          B, heads, Sq, Skv, int(head_dim), float(scale), _p(ws), ws_n, kernels=3 if nsplit == 1 else 4,
          name="attention_bwd", flops=14.0 * B * heads * Sq * Skv * head_dim)


def splitk_ws_floats(M: int, N: int, K: int) -> int:
    """SB200_GEMM_SPLITK_WS_FLOATS."""
    tiles = ((M + 127) // 128) * (N // 128 if N % 128 == 0 else (N + 63) // 64)
    want = (132 + tiles - 1) // tiles
    kbs = (K + 63) // 64
    kb = max(8, (kbs + want - 1) // want)
    return ((kbs + kb - 1) // kb) * M * N


def gemm_splitk_f32(x: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 out[M, N] = x[M, K] @ w[N, K].T (bf16 operands): `gemm_kernel` in split-K mode + `splitk_reduce_kernel`.
    `out`: an fp32 [M, N] row-strided matrix on x's device (e.g. a column slice of a wider buffer)."""
    M, K = x.shape
    N = w.shape[0]
    assert w.shape[1] == K
    out = _out(out, (M, N), "gemm_splitk_f32", x.device, torch.float32)
    if out.device != x.device:
        raise ValueError(f"gemm_splitk_f32: out is on {out.device}, x on {x.device}")
    n_ws = splitk_ws_floats(M, N, K)
    ws = torch.empty(n_ws, device=x.device, dtype=torch.float32)
    _call("sb200_gemm_splitk_f32", x, _p(x), x.stride(0), _p(w), w.stride(0), _p(out), out.stride(0), M, N, K, _p(ws),
          n_ws, kernels=2, name="gemm", flops=2.0 * M * N * K)
    return out


def guided_step_loss_fwd(eps_u, eps_c, g: float, x, cx: float, ce: float, target) -> torch.Tensor:
    """fp32 scalar mean((cx x + ce (eps_u + g (eps_c - eps_u)) - target)^2): `guided_loss_kernel` + finalize."""
    n = eps_u.numel()
    parts = min(256, n // 2048 + 1)  # SB200_GUIDED_LOSS_BLOCKS
    ws = torch.empty(parts, device=eps_u.device, dtype=torch.float32)
    loss = torch.empty((), device=eps_u.device, dtype=torch.float32)
    _call("sb200_guided_step_loss", eps_u, _p(eps_u), _p(eps_c), float(g), _p(x), float(cx), float(ce), _p(target), n,
          0, _p(loss), _p(ws), None, None, kernels=2)
    return loss


def guided_step_loss_bwd(eps_u, eps_c, g: float, x, cx: float, ce: float, target, dloss) -> torch.Tensor:
    """d loss / d eps_u scaled by the device scalar dloss: one `guided_loss_kernel` launch."""
    d = torch.empty_like(eps_u)
    _call("sb200_guided_step_loss", eps_u, _p(eps_u), _p(eps_c), float(g), _p(x), float(cx), float(ce), _p(target),
          eps_u.numel(), 1, None, None, _p(dloss), _p(d))
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


def _row_matrix(t: torch.Tensor, shape, what: str, name: str = "out", dtype=BF16) -> torch.Tensor:
    """t if its elements are the rows of one 2-D matrix of the given shape and dtype, else ValueError.  A row-strided
    matrix has unit column stride and every leading dimension packed over the next ones with the row stride
    t.stride(-2) the wrappers pass as the leading dimension (e.g. a column slice of a wider buffer, or an NHWC tensor
    whose pixels are the rows); a dimension of size 1 is never stepped, so its stride does not matter."""
    shape = tuple(shape)
    st = t.stride()
    ld = st[-2] if len(shape) > 1 else 0
    packed = all(shape[i] == 1 or st[i] == ld * math.prod(shape[i + 1:-1]) for i in range(len(shape) - 2))
    if tuple(t.shape) != shape or t.dtype != dtype or (shape[-1] > 1 and st[-1] != 1) or not packed:
        raise ValueError(f"{what}: {name} {tuple(t.shape)} {t.dtype} / strides {st} is not a row-strided "
                         f"{shape} {dtype} matrix")
    return t


def _out(out: Optional[torch.Tensor], shape, what: str, device, dtype=BF16) -> torch.Tensor:
    """An optional output: `out` checked by `_row_matrix`, or a new tensor of the shape when None."""
    if out is None:
        return torch.empty(shape, device=device, dtype=dtype)
    return _row_matrix(out, shape, what, "out", dtype)


def groupnorm_bwd(x0, gamma, beta, groups: int, silu: bool, dy, stats_ws, *, x1=None, add=None,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Input gradient of `groupnorm` (concat layout [.., C0 + C1]); stats_ws is the forward's workspace, or its
    (mean, rstd) block as a [B, groups, 2] tensor (`gn_stats` — sliceable along the batch).  `out`: a [.., C0 + C1]
    tensor whose pixels are rows of one 2-D matrix with row stride out.stride(-2) (e.g. a column slice)."""
    shp = x0.shape
    B, C0 = shp[0], shp[-1]
    HW = x0.numel() // (B * C0)
    C1 = x1.shape[-1] if x1 is not None else 0
    Cc = C0 + C1
    dx = _out(out, shp[:-1] + (Cc,), "groupnorm_bwd", x0.device)
    ws = gn_ws(B, groups, x0.device)
    fwd = stats_ws if stats_ws.dim() == 3 else stats_ws[B * groups * 2 * GN_STATS_OFFSET:]
    assert fwd.is_contiguous()
    _call("sb200_groupnorm_bwd", x0, _p(x0), x0.stride(-2), C0, _p(x1), x1.stride(-2) if x1 is not None else 0, C1,
          _p(gamma), _p(beta), _p(dy), dy.stride(-2), _p(add), add.stride(-2) if add is not None else 0, _p(dx),
          dx.stride(-2), B, HW, groups, int(silu), _p(fwd), _p(ws), kernels=3, name="groupnorm_bwd")
    return dx


def layernorm_bwd(x, gamma, dy, eps: float = 1e-5, add=None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`out`: an [M, C] row-strided matrix (e.g. a column slice of a wider buffer) to write dx into."""
    M, Cc = x.shape
    dx = _out(out, (M, Cc), "layernorm_bwd", x.device)
    _call("sb200_layernorm_bwd", x, _p(x), x.stride(0), _p(gamma), _p(dy), dy.stride(0), _p(add),
          add.stride(0) if add is not None else 0, _p(dx), dx.stride(0), M, Cc, float(eps))
    return dx


def geglu(pre: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`out`: an [M, F] row-strided matrix to write a * gelu(g) into."""
    M, F2 = pre.shape
    o = _out(out, (M, F2 // 2), "geglu", pre.device)
    _call("sb200_geglu", pre, _p(pre), pre.stride(0), _p(o), o.stride(0), M, F2 // 2)
    return o


def geglu_bwd(pre: torch.Tensor, dout: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`out`: an [M, 2F] row-strided matrix to write [da | dg] into."""
    M, F2 = pre.shape
    dpre = _out(out, (M, F2), "geglu_bwd", pre.device)
    _call("sb200_geglu_bwd", pre, _p(pre), pre.stride(0), _p(dout), dout.stride(0), _p(dpre), dpre.stride(0), M,
          F2 // 2)
    return dpre


def add(a: torch.Tensor, b: torch.Tensor, c: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None):
    """a + b (+ c) on 2-D (row-strided) bf16 matrices."""
    M, Cc = a.shape
    if out is None:
        out = torch.empty((M, Cc), device=a.device, dtype=BF16)
    _call("sb200_add", a, _p(a), a.stride(0), _p(b), b.stride(0), _p(c), c.stride(0) if c is not None else 0, _p(out),
          out.stride(0), M, Cc)
    return out


def lora_compose(raw: torch.Tensor, col_mult: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[n, j] = raw[n, j] * col_mult[j]: the effective lora_up of composite LoRA packs (fp32 [rows, rp], contiguous),
    one `lora_compose` launch."""
    if raw.dtype != torch.float32 or col_mult.dtype != torch.float32 or raw.dim() != 2 or not raw.is_contiguous():
        raise ValueError("lora_compose: raw must be a contiguous fp32 [rows, rp] matrix and col_mult fp32")
    rows, rp = raw.shape
    if col_mult.numel() != rp or not col_mult.is_contiguous():
        raise ValueError(f"lora_compose: col_mult has {col_mult.numel()} values for {rp} columns")
    if out is None:
        out = torch.empty_like(raw)
    elif out.shape != raw.shape or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError("lora_compose: out must be a contiguous fp32 matrix shaped like raw")
    _call("sb200_lora_compose", raw, _p(raw), _p(col_mult), _p(out), rows, rp, name="lora_compose")
    return out


def upsample2x_bwd(dy: torch.Tensor) -> torch.Tensor:
    B, H2, W2, Cc = dy.shape
    dx = torch.empty((B, H2 // 2, W2 // 2, Cc), device=dy.device, dtype=BF16)
    _call("sb200_upsample2x_bwd", dy, _p(dy), _p(dx), B, H2 // 2, W2 // 2, Cc)
    return dx


def zero_stuff(dy: torch.Tensor) -> torch.Tensor:
    B, Ho, Wo, Cc = dy.shape
    z = torch.empty((B, 2 * Ho, 2 * Wo, Cc), device=dy.device, dtype=BF16)
    _call("sb200_zero_stuff", dy, _p(dy), _p(z), B, Ho, Wo, Cc)
    return z


def conv_out_bwd(deps: torch.Tensor, w_packed: torch.Tensor) -> torch.Tensor:
    """deps: NCHW [B,4,H,W] fp32 / bf16 -> NHWC bf16 [B,H,W,C]."""
    B, _, H, W = deps.shape
    Cc = w_packed.shape[-1]
    deps = deps.contiguous()
    dx = torch.empty((B, H, W, Cc), device=deps.device, dtype=BF16)
    _call("sb200_conv_out_bwd", deps, _p(deps), int(deps.dtype == torch.float32), _p(w_packed), _p(dx), B, H, W, Cc)
    return dx


def colsum(dy: torch.Tensor) -> torch.Tensor:
    """dy [B, H, W, C] (or [B, HW, C]) -> fp32 [B, C]."""
    B, Cc = dy.shape[0], dy.shape[-1]
    HW = dy.numel() // (B * Cc)
    out = torch.empty((B, Cc), device=dy.device, dtype=torch.float32)
    _call("sb200_colsum", dy, _p(dy), dy.stride(-2), _p(out), B, HW, Cc)
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
    _call("sb200_lora_proj", A, _p(A), A.stride(0), _p(Bt), Bt.stride(0), _p(T), M, Cc, r, int(out is not None))
    return T


def lora_wgrad(A: torch.Tensor, T: torch.Tensor, G: torch.Tensor, transposed: bool, scale: float,
               accumulate: bool = False) -> None:
    """G (+)= scale * A.T @ T.  A [M, C] bf16, T [M, r] fp32; G fp32 (any strides, e.g. a column slice):
    [C, r] (transposed=False) or [r, C] (transposed=True)."""
    M, Cc = A.shape
    r = T.shape[1]
    gs_c, gs_r = (G.stride(1), G.stride(0)) if transposed else (G.stride(0), G.stride(1))
    ws = _wgrad_ws(Cc, r, A.device)
    _call("sb200_lora_wgrad", A, _p(A), A.stride(0), _p(T), _p(G), gs_c, gs_r, float(scale), int(accumulate), M, Cc, r,
          _p(ws), kernels=2, name="lora_wgrad")


def lora_rank_update(dX: torch.Tensor, U: torch.Tensor, D: torch.Tensor, scale: float) -> None:
    """dX += scale * U @ D   (dX [M, C] bf16 in place, U [M, r] fp32, D [r, C] bf16)."""
    M, Cc = dX.shape
    _call("sb200_lora_rank_update", dX, _p(dX), dX.stride(0), _p(U), _p(D), D.stride(0), float(scale), M, Cc,
          U.shape[1])


def lora_conv_proj(x0: torch.Tensor, D: torch.Tensor, stride: int = 1, x1: Optional[torch.Tensor] = None):
    """3x3 / pad 1 conv of NHWC x (= [x0 | x1]) with D [r, 3, 3, C] -> fp32 [B*Ho*Wo, r]."""
    B, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    r = D.shape[0]
    T = torch.empty((B * (H // stride) * (W // stride), r), device=x0.device, dtype=torch.float32)
    _call("sb200_lora_conv_proj", x0, _p(x0), x0.stride(2), C0, _p(x1), x1.stride(2) if x1 is not None else 0, C1,
          _p(D), _p(T), B, H, W, stride, r)
    return T


def lora_conv_wgrad(x0: torch.Tensor, U: torch.Tensor, G: torch.Tensor, scale: float, stride: int = 1,
                    x1: Optional[torch.Tensor] = None, accumulate: bool = False) -> None:
    """G [r, 3, 3, C] fp32 (+)= scale * sum_p U[p, :] (x) patch(x, p)."""
    B, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    r = U.shape[1]
    ws = _wgrad_ws(9 * (C0 + C1), r, x0.device)
    _call("sb200_lora_conv_wgrad", x0, _p(x0), x0.stride(2), C0, _p(x1), x1.stride(2) if x1 is not None else 0, C1,
          _p(U), _p(G), float(scale), int(accumulate), B, H, W, stride, r, _p(ws), kernels=2, name="lora_wgrad")


def lora_conv_rank_update(dX: torch.Tensor, U: torch.Tensor, D: torch.Tensor, scale: float, stride: int = 1) -> None:
    """dX [B,H,W,C] (contiguous, in place) += scale * conv_transpose(U [B,Ho,Wo,r], D [r,3,3,C])."""
    B, H, W, Cc = dX.shape
    assert dX.is_contiguous()
    _call("sb200_lora_conv_rank_update", dX, _p(dX), _p(U), _p(D), float(scale), B, H, W, Cc, stride, U.shape[1])


def adamw(table: torch.Tensor, n_tensors: int, max_numel: int, lr: float, beta1: float, beta2: float, eps: float,
          weight_decay: float, step: int) -> None:
    """One fused `adamw_kernel` launch over a device table of (p, g, m, v, n) records (int64 [n_tensors, 5])."""
    _call("sb200_adamw", table, _p(table), n_tensors, int(max_numel), float(lr), float(beta1), float(beta2), float(eps),
          float(weight_decay), int(step))


def adam_f32(table: torch.Tensor, n_tensors: int, max_numel: int, lr: float, beta1: float, beta2: float, eps: float,
             weight_decay: float, step: int) -> None:
    """One `adam_f32_kernel` launch over a device table of fp32 (p, g, m, v, n) records (int64 [n_tensors, 5])."""
    _call("sb200_adam_f32", table, _p(table), n_tensors, int(max_numel), float(lr), float(beta1), float(beta2),
          float(eps), float(weight_decay), int(step))
