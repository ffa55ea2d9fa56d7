"""Generates tests/golden/ops_calls.pt:

    python tests/golden/make_golden_ops_calls.py

What every `sliders_b200.ops` wrapper hands the C ABI, recorded on CPU tensors with no library and no GPU.
`_cabi.load` returns a stand-in whose every `sb200_*` function records its arguments and returns 0, `ops._ctx` /
`ops._stream` return constants and `torch.cuda.Event` is stubbed.  Each case in CASES runs twice:

- "plain": the call(s) the C ABI received and the `launch_count` delta;
- "capture": with `profile_log` and `record_calls` set and the stream reported as capturing, also the
  `profile_log` (name, flops) and `record_calls` [fn, args, name, flops] entries, and the calls `replay_calls`
  issues for them.

An argument is recorded as ("ctx",), ("stream",), ("null",), ("in", input index, byte offset) for a pointer into a
case's input, ("alloc", allocation index, shape, dtype, byte offset) for a pointer into a tensor the wrapper
allocated with torch.empty / torch.empty_like, ("lora", fields) for an `sb200_lora`, or (type name, value) for a
scalar.  A wrapper that raises records the exception's type and message.
"""
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from sliders_b200 import _cabi, ops  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ops_calls.pt")
BF, F32 = torch.bfloat16, torch.float32
_CTX, _STREAM = C.c_void_p(0x5B200), C.c_void_p(0x57EA)


def _t(*shape, dtype=BF):
    return torch.zeros(shape, dtype=dtype)


def _cases():
    """name -> (inputs, fn(*inputs)).  Inputs are made fresh per run; views of an input go through the fn."""
    cs = {}
    x, w, b, rb, res = _t(64, 96), _t(128, 96), _t(128), _t(2, 128), _t(64, 128)
    cs["gemm"] = ([x, w], lambda x, w: ops.gemm(x, w))
    cs["gemm_bias"] = ([x, w, b], lambda x, w, b: ops.gemm(x, w, bias=b))
    cs["gemm_rowbias"] = ([x, w, rb], lambda x, w, rb: ops.gemm(x, w, rowbias=rb, rows_per_batch=32))
    cs["gemm_resid"] = ([x, w, res], lambda x, w, r: ops.gemm(x, w, resid=r))
    cs["gemm_geglu"] = ([x, w], lambda x, w: ops.gemm(x, w, geglu=True, bn=64))
    cs["gemm_x1_out"] = ([_t(64, 128), w, _t(64, 256)],
                         lambda xx, w, o: ops.gemm(xx[:, :48], w, x1=xx[:, 64:112], out=o[:, 128:]))
    cs["gemm_all"] = ([x, w, b, rb, res, _t(16, 96), _t(128, 4, dtype=F32), _t(1, dtype=F32)],
                      lambda x, w, b, rb, r, d, u, sd: ops.gemm(
                          x, w, bias=b, rowbias=rb, rows_per_batch=32, resid=r,
                          lora=ops.Lora(d, u, 4, 128, 0.5, scale_dev=sd), bn=128))
    cs["gemm_lora_derived_rps"] = ([x, w, _t(16, 96), _t(128, 4, dtype=F32), _t(4, dtype=F32)],
                                   lambda x, w, d, u, ss: ops.gemm(x, w, lora=ops.Lora(d, u, 4, 128, 2.0,
                                                                                       sample_scale=ss)))
    cs["gemm_lora_bad_rps"] = ([x, w, _t(16, 96), _t(128, 4, dtype=F32), _t(3, dtype=F32)],
                               lambda x, w, d, u, ss: ops.gemm(x, w, lora=ops.Lora(d, u, 4, 128, 2.0,
                                                                                   sample_scale=ss)))
    xi = _t(2, 8, 8, 64)
    wp = _t(128, 3, 3, 64)
    cs["conv3x3"] = ([xi, wp], lambda x, w: ops.conv3x3(x, w))
    cs["conv3x3_flags"] = ([xi, wp, b, rb, _t(2, 8, 8, 128)],
                           lambda x, w, b, rb, r: ops.conv3x3(x, w, bias=b, rowbias=rb, resid=r))
    cs["conv3x3_x1_s2_pad"] = ([xi, _t(2, 8, 8, 32), _t(128, 3, 3, 96), b],
                               lambda x, x1, w, b: ops.conv3x3(x, w, x1=x1, stride=2, bias=b, pad_bottom_right=True))
    cs["conv3x3_lora_out"] = ([xi, wp, _t(16, 3, 3, 64), _t(128, 4, dtype=F32), _t(2, dtype=F32),
                               _t(2, 8, 8, 256)],
                              lambda x, w, d, u, ss, o: ops.conv3x3(x, w, lora=ops.Lora(d, u, 4, 128, 1.0,
                                                                                        sample_scale=ss),
                                                                    out=o[..., 64:192], bn=64))
    cs["conv3x3_bad_out"] = ([xi, wp, _t(2, 8, 8, 256)], lambda x, w, o: ops.conv3x3(x, w, out=o[:, :, :4, :128]))
    q = _t(2 * 16, 3 * 128)
    kv = _t(2 * 8, 2 * 128)
    cs["attention"] = ([q, kv], lambda q, kv: ops.attention(q[:, :128], kv[:, :128], kv[:, 128:], 2, 2, 16, 8, 0.125))
    cs["attention_lse"] = ([q, kv, _t(2, 2, 16, dtype=F32)],
                           lambda q, kv, l: ops.attention(q[:, 128:256], kv[:, :128], kv[:, 128:], 2, 2, 16, 8, 0.125,
                                                          lse=l))
    cs["attention_bad_q"] = ([q, kv], lambda q, kv: ops.attention(q[:16], kv[:, :128], kv[:, 128:], 2, 2, 16, 8, 0.1))
    g, bt = _t(96), _t(96)
    cs["groupnorm"] = ([_t(2, 16, 64), g, bt], lambda x, g, b: ops.groupnorm(x, g, b, 32, 1e-5, True))
    cs["groupnorm_x1_ws"] = ([_t(2, 4, 4, 64), _t(2, 4, 4, 32), g, bt, _t(2 * 32 * 2 * 129, dtype=F32)],
                             lambda x, x1, g, b, ws: ops.groupnorm(x, g, b, 32, 1e-6, False, x1=x1, stats_ws=ws))
    cs["groupnorm_bad_x1"] = ([_t(2, 16, 64), _t(2, 8, 32), g, bt],
                              lambda x, x1, g, b: ops.groupnorm(x, g, b, 32, 1e-5, True, x1=x1))
    cs["layernorm"] = ([_t(64, 128), _t(128), _t(128)], lambda x, g, b: ops.layernorm(x[:, :96], g, b, 1e-6))
    cs["small_linear"] = ([_t(2, 320), _t(1280, 320), _t(1280)],
                          lambda x, w, b: ops.small_linear(x, w, b, act_in=True))
    cs["small_linear_lora_resid"] = ([_t(2, 320), _t(1280, 320), _t(16, 320), _t(1280, 4, dtype=F32),
                                      _t(2, 1280)],
                                     lambda x, w, d, u, r: ops.small_linear(
                                         x, w, None, act_out=2, lora=ops.Lora(d, u, 4, 1280, 1.0), resid=r))
    cs["small_linear_bad_resid"] = ([_t(2, 320), _t(1280, 320), _t(2, 1280)],
                                    lambda x, w, r: ops.small_linear(x, w, None, act_out=1, resid=r.t().contiguous()))
    cs["sinusoid"] = ([_t(4, dtype=F32)], lambda v: ops.sinusoid(v, 320))
    cs["conv_in_f32"] = ([_t(2, 4, 8, 8, dtype=F32), _t(320, 3, 3, 4), _t(320)], ops.conv_in)
    cs["conv_in_bf16"] = ([_t(2, 4, 8, 8), _t(320, 3, 3, 4), _t(320)], ops.conv_in)
    cs["conv_out"] = ([_t(2, 8, 8, 320), _t(4, 3, 3, 320), _t(4)], ops.conv_out)
    cs["conv_out_f32"] = ([_t(2, 8, 8, 320), _t(4, 3, 3, 320), _t(4)],
                          lambda x, w, b: ops.conv_out(x, w, b, out_dtype=F32))
    cs["upsample2x"] = ([_t(2, 4, 4, 64)], ops.upsample2x)
    cs["upsample2x_bad"] = ([_t(2, 4, 4, 64)], lambda x: ops.upsample2x(x.transpose(1, 2)))
    cs["vae_conv_in_u8"] = ([_t(1, 8, 8, 3, dtype=torch.uint8), _t(128, 3, 3, 3), _t(128)], ops.vae_conv_in_u8)
    cs["vae_conv_out_u8"] = ([_t(1, 8, 8, 128), _t(3, 3, 3, 128), _t(3)], ops.vae_conv_out_u8)
    cs["vae_conv_out_u8_float"] = ([_t(1, 8, 8, 128), _t(3, 3, 3, 128), _t(3)],
                                   lambda x, w, b: ops.vae_conv_out_u8(x, w, b, return_float=True))
    qw, qb = _t(8, 8, dtype=F32), _t(8, dtype=F32)
    cs["vae_moments"] = ([_t(1, 4, 4, 512), _t(8, 3, 3, 512), _t(8), qw, qb],
                         lambda x, w, b, qw, qb: ops.vae_moments(x, w, b, qw, qb, None, 0.18215))
    cs["vae_moments_eps"] = ([_t(1, 4, 4, 512), _t(8, 3, 3, 512), _t(8), qw, qb, _t(1, 4, 4, 4, dtype=F32)],
                             lambda x, w, b, qw, qb, e: ops.vae_moments(x, w, b, qw, qb, e, 0.13025))
    cs["vae_post_quant"] = ([_t(1, 4, 4, 4, dtype=F32), _t(4, 4, dtype=F32), _t(4, dtype=F32)],
                            lambda z, pw, pb: ops.vae_post_quant(z, pw, pb, 0.18215))
    cs["softmax_rows"] = ([_t(8, 64, dtype=F32)], lambda s: ops.softmax_rows(s[:, :48], 0.5))
    cs["softmax_rows_out"] = ([_t(8, 64, dtype=F32), _t(8, 96)], lambda s, o: ops.softmax_rows(s, 0.5, out=o[:, 32:]))
    cs["softmax_rows_bad_out"] = ([_t(8, 64, dtype=F32), _t(64, 8)], lambda s, o: ops.softmax_rows(s, 0.5, out=o.t()))
    e2 = _t(4, 4, 8, 8, dtype=F32)
    cs["cfg_ddim"] = ([e2], lambda e: ops.cfg_ddim(e, 7.5))
    cs["cfg_ddim_x"] = ([e2, _t(2, 4, 8, 8, dtype=F32)], lambda e, x: ops.cfg_ddim(e, 7.5, x, 0.9, 0.95))
    cs["cfg_ddim_bf16_x32"] = ([_t(4, 4, 8, 8), _t(2, 4, 8, 8, dtype=F32)],
                               lambda e, x: ops.cfg_ddim(e, 3.0, x, 0.5, 0.7))
    cs["cfg_ddim_single"] = ([_t(2, 4, 8, 8), _t(2, 4, 8, 8)],
                             lambda e, x: ops.cfg_ddim(e, 0.0, x, 0.5, 0.7, single=True))
    cs["cfg_ddim_affine"] = ([e2, _t(2, 4, 8, 8, dtype=F32)],
                             lambda e, x: ops.cfg_ddim(e, 5.0, x, 1.1, -0.2, out_dtype=BF, affine=True))
    cs["cfg_ddim_bad"] = ([_t(3, 4, 8, 8, dtype=F32)], lambda e: ops.cfg_ddim(e, 7.5))
    qkv = _t(2 * 16, 3 * 128)
    akv = _t(2 * 8, 2 * 128)
    o, do, lse = _t(2 * 16, 128), _t(2 * 16, 128), _t(2, 2, 16, dtype=F32)
    dq, dkv = _t(2 * 16, 3 * 128), _t(2 * 8, 2 * 128)
    cs["attention_bwd"] = ([qkv, akv, o, do, lse, dq],
                           lambda q, kv, o, do, l, dq: ops.attention_bwd(q[:, :128], kv[:, :128], kv[:, 128:], o, do, l,
                                                                         2, 2, 16, 8, 0.125, 64, dq[:, :128]))
    cs["attention_bwd_dkdv"] = ([qkv, akv, o, do, lse, dq, dkv],
                                lambda q, kv, o, do, l, dq, dkv: ops.attention_bwd(
                                    q[:, :128], kv[:, :128], kv[:, 128:], o, do, l, 2, 2, 16, 8, 0.125, 64,
                                    dq[:, :128], dkv[:, :128], dkv[:, 128:]))
    sq = 256  # 4 query splits (attn_bwd_splits)
    cs["attention_bwd_split"] = ([_t(2 * sq, 3 * 128), akv, _t(2 * sq, 128), _t(2 * sq, 128), _t(2, 2, sq, dtype=F32),
                                  _t(2 * sq, 3 * 128), dkv],
                                 lambda q, kv, o, do, l, dq, dkv: ops.attention_bwd_split(
                                     q[:, :128], kv[:, :128], kv[:, 128:], o, do, l, 2, 2, sq, 8, 0.125, 64,
                                     dq[:, :128], dkv[:, :128], dkv[:, 128:]))
    bkv = _t(2 * 256, 2 * 128)
    cs["attention_bwd_unsplit"] = ([qkv, bkv, o, do, lse, dq, _t(2 * 256, 2 * 128)],
                                   lambda q, kv, o, do, l, dq, dkv: ops.attention_bwd_split(
                                       q[:, :128], kv[:, :128], kv[:, 128:], o, do, l, 2, 2, 16, 256, 0.125, 64,
                                       dq[:, :128], dkv[:, :128], dkv[:, 128:]))
    cs["gemm_splitk_f32"] = ([_t(64, 512), _t(96, 512)], lambda x, w: ops.gemm_splitk_f32(x, w))
    cs["gemm_splitk_f32_out"] = ([_t(64, 512), _t(96, 512), _t(64, 256, dtype=F32)],
                                 lambda x, w, o: ops.gemm_splitk_f32(x, w, out=o[:, 64:160]))
    cs["gemm_splitk_f32_bad_out"] = ([_t(64, 512), _t(96, 512), _t(64, 96)],
                                     lambda x, w, o: ops.gemm_splitk_f32(x, w, out=o))
    gl = [_t(2, 4, 8, 8, dtype=F32) for _ in range(4)]
    cs["guided_step_loss_fwd"] = (gl, lambda eu, ec, x, t: ops.guided_step_loss_fwd(eu, ec, 7.5, x, 0.9, -0.3, t))
    cs["guided_step_loss_bwd"] = (gl + [_t(dtype=F32)],
                                  lambda eu, ec, x, t, d: ops.guided_step_loss_bwd(eu, ec, 7.5, x, 0.9, -0.3, t, d))
    gws = _t(2 * 32 * 2 * 129, dtype=F32)
    cs["groupnorm_bwd"] = ([_t(2, 16, 64), g, bt, _t(2, 16, 64), gws],
                           lambda x, g, b, dy, ws: ops.groupnorm_bwd(x, g, b, 32, True, dy, ws))
    cs["groupnorm_bwd_x1_add_out"] = ([_t(2, 4, 4, 64), _t(2, 4, 4, 32), g, bt, _t(2, 4, 4, 96), _t(2, 4, 4, 96),
                                       _t(2, 32, 2, dtype=F32), _t(2, 4, 4, 160)],
                                      lambda x, x1, g, b, dy, a, st, o: ops.groupnorm_bwd(
                                          x, g, b, 32, False, dy, st, x1=x1, add=a, out=o[..., 32:128]))
    cs["groupnorm_bwd_bad_out"] = ([_t(2, 16, 64), g, bt, _t(2, 16, 64), gws, _t(2, 16, 64)],
                                   lambda x, g, b, dy, ws, o: ops.groupnorm_bwd(x, g, b, 32, True, dy, ws,
                                                                                out=o.transpose(1, 2)))
    cs["layernorm_bwd"] = ([_t(64, 128), _t(128), _t(64, 128)], lambda x, g, dy: ops.layernorm_bwd(x, g, dy))
    cs["layernorm_bwd_add_out"] = ([_t(64, 128), _t(128), _t(64, 128), _t(64, 128), _t(64, 256)],
                                   lambda x, g, dy, a, o: ops.layernorm_bwd(x, g, dy, 1e-6, add=a, out=o[:, 64:192]))
    cs["layernorm_bwd_bad_out"] = ([_t(64, 128), _t(128), _t(64, 128), _t(128, 64)],
                                   lambda x, g, dy, o: ops.layernorm_bwd(x, g, dy, out=o.t()))
    cs["geglu"] = ([_t(64, 256)], lambda p: ops.geglu(p))
    cs["geglu_out"] = ([_t(64, 256), _t(64, 192)], lambda p, o: ops.geglu(p, out=o[:, 64:]))
    cs["geglu_bad_out"] = ([_t(64, 256), _t(64, 128, dtype=F32)], lambda p, o: ops.geglu(p, out=o))
    cs["geglu_bwd"] = ([_t(64, 256), _t(64, 128)], lambda p, d: ops.geglu_bwd(p, d))
    cs["geglu_bwd_out"] = ([_t(64, 256), _t(64, 128), _t(64, 512)], lambda p, d, o: ops.geglu_bwd(p, d, out=o[:, 256:]))
    cs["geglu_bwd_bad_out"] = ([_t(64, 256), _t(64, 128), _t(64, 128)], lambda p, d, o: ops.geglu_bwd(p, d, out=o))
    cs["add"] = ([_t(64, 128), _t(64, 128)], lambda a, b: ops.add(a, b))
    cs["add_c_out"] = ([_t(64, 256), _t(64, 128), _t(64, 128), _t(64, 128)],
                       lambda a, b, c, o: ops.add(a[:, 128:], b, c, out=o))
    cs["lora_compose"] = ([_t(64, 4, dtype=F32), _t(4, dtype=F32)], lambda r, m: ops.lora_compose(r, m))
    cs["lora_compose_out"] = ([_t(64, 4, dtype=F32), _t(4, dtype=F32), _t(64, 4, dtype=F32)],
                              lambda r, m, o: ops.lora_compose(r, m, out=o))
    cs["lora_compose_bad_out"] = ([_t(64, 4, dtype=F32), _t(4, dtype=F32), _t(4, 64, dtype=F32)],
                                  lambda r, m, o: ops.lora_compose(r, m, out=o.t()))
    cs["upsample2x_bwd"] = ([_t(2, 8, 8, 64)], ops.upsample2x_bwd)
    cs["zero_stuff"] = ([_t(2, 4, 4, 64)], ops.zero_stuff)
    cs["conv_out_bwd"] = ([_t(2, 4, 8, 8, dtype=F32), _t(4, 3, 3, 320)], ops.conv_out_bwd)
    cs["conv_out_bwd_bf16"] = ([_t(2, 4, 8, 8), _t(4, 3, 3, 320)], ops.conv_out_bwd)
    cs["colsum"] = ([_t(2, 8, 8, 64)], ops.colsum)
    cs["colsum_3d"] = ([_t(2, 64, 128)], lambda d: ops.colsum(d[..., :64]))
    cs["lora_proj"] = ([_t(64, 128), _t(4, 128)], lambda a, bt: ops.lora_proj(a, bt))
    cs["lora_proj_accumulate"] = ([_t(64, 192), _t(4, 128), _t(64, 4, dtype=F32)],
                                  lambda a, bt, o: ops.lora_proj(a[:, 64:], bt, out=o))
    cs["lora_wgrad"] = ([_t(64, 128), _t(64, 4, dtype=F32), _t(128, 4, dtype=F32)],
                        lambda a, t, gg: ops.lora_wgrad(a, t, gg, False, 0.5))
    cs["lora_wgrad_t_acc"] = ([_t(64, 256), _t(64, 8, dtype=F32), _t(8, 512, dtype=F32)],
                              lambda a, t, gg: ops.lora_wgrad(a[:, :128], t, gg[:, 128:256], True, 2.0,
                                                              accumulate=True))
    cs["lora_rank_update"] = ([_t(64, 128), _t(64, 4, dtype=F32), _t(4, 256)],
                              lambda dx, u, d: ops.lora_rank_update(dx, u, d[:, 128:], 0.25))
    cs["lora_conv_proj"] = ([_t(2, 8, 8, 64), _t(4, 3, 3, 64)], lambda x, d: ops.lora_conv_proj(x, d))
    cs["lora_conv_proj_x1_s2"] = ([_t(2, 8, 8, 64), _t(2, 8, 8, 32), _t(8, 3, 3, 96)],
                                  lambda x, x1, d: ops.lora_conv_proj(x, d, stride=2, x1=x1))
    cs["lora_conv_wgrad"] = ([_t(2, 8, 8, 64), _t(128, 4, dtype=F32), _t(4, 3, 3, 64, dtype=F32)],
                             lambda x, u, gg: ops.lora_conv_wgrad(x, u, gg, 0.5))
    cs["lora_conv_wgrad_x1_s2_acc"] = ([_t(2, 8, 8, 64), _t(2, 8, 8, 32), _t(32, 8, dtype=F32),
                                        _t(8, 3, 3, 96, dtype=F32)],
                                       lambda x, x1, u, gg: ops.lora_conv_wgrad(x, u, gg, 1.5, stride=2, x1=x1,
                                                                                accumulate=True))
    cs["lora_conv_rank_update"] = ([_t(2, 8, 8, 64), _t(2, 8, 8, 4, dtype=F32), _t(4, 3, 3, 64)],
                                   lambda dx, u, d: ops.lora_conv_rank_update(dx, u, d, 0.5))
    cs["lora_conv_rank_update_s2"] = ([_t(2, 8, 8, 64), _t(2, 4, 4, 16, dtype=F32), _t(16, 3, 3, 64)],
                                      lambda dx, u, d: ops.lora_conv_rank_update(dx, u, d, 0.5, stride=2))
    tab = _t(3, 5, dtype=torch.int64)
    cs["adamw"] = ([tab], lambda t: ops.adamw(t, 3, 4096, 1e-3, 0.9, 0.999, 1e-8, 1e-2, 7))
    cs["adam_f32"] = ([tab], lambda t: ops.adam_f32(t, 3, 4096, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1))
    return cs


CASES = list(_cases())


class _Trace:
    """The stand-ins: a library whose functions record their arguments, and torch.empty / torch.empty_like that
    remember what the wrapper allocated."""

    def __init__(self, inputs):
        self.inputs = inputs
        self.allocs = []
        self.calls = []

    def ptr(self, v):
        if v is None or v == 0:
            return ("null",)
        for i, t in enumerate(self.inputs):
            if t.data_ptr() == v:
                return ("in", i, 0)
        for i, t in enumerate(self.allocs):
            if t.data_ptr() == v:
                return ("alloc", i, tuple(t.shape), str(t.dtype), 0)
        for i, t in enumerate(self.inputs):
            base = t.untyped_storage().data_ptr()
            if base <= v < base + t.untyped_storage().nbytes():
                return ("in", i, v - t.data_ptr())
        for i, t in enumerate(self.allocs):
            base = t.untyped_storage().data_ptr()
            if base <= v < base + t.untyped_storage().nbytes():
                return ("alloc", i, tuple(t.shape), str(t.dtype), v - t.data_ptr())
        return ("unknown",)

    def arg(self, a):
        if a is _CTX:
            return ("ctx",)
        if a is _STREAM:
            return ("stream",)
        if a is None:
            return ("null",)
        if isinstance(a, C.c_void_p):
            return self.ptr(a.value)
        if type(a).__name__ == "CArgObject":  # C.byref(LoraArgs)
            s = a._obj
            return ("lora", self.ptr(s.down), self.ptr(s.up), s.r, s.rt, s.group_n, s.scale, self.ptr(s.scale_dev),
                    self.ptr(s.sample_scale), s.rows_per_sample)
        return (type(a).__name__, a)

    def lib(self):
        trace = self

        class Lib:
            def __getattr__(self, name):
                def fn(*args):
                    trace.calls.append((name, tuple(trace.arg(a) for a in args)))
                    return 0

                fn.__name__ = name
                return fn

        return Lib()

    def empty(self, real):
        def f(*a, **k):
            t = real(*a, **k)
            self.allocs.append(t)
            return t

        return f


class _Event:
    def __init__(self, enable_timing=False):
        pass

    def record(self, stream=None):
        pass


def record(case, mode):
    """What the wrapper of CASES[case] hands the C ABI in `mode` ("plain" or "capture")."""
    inputs, fn = _cases()[case]
    tr = _Trace(inputs)
    lib = tr.lib()
    saved = (_cabi.load, ops._ctx, ops._stream, torch.cuda.Event, torch.cuda.is_current_stream_capturing,
             torch.empty, torch.empty_like, ops.profile_log, ops.record_calls)
    capture = mode == "capture"
    _cabi.load = lambda: lib
    ops._ctx = lambda t: _CTX
    ops._stream = lambda: _STREAM
    torch.cuda.Event = _Event
    torch.cuda.is_current_stream_capturing = lambda: capture
    torch.empty, torch.empty_like = tr.empty(saved[5]), tr.empty(saved[6])
    ops.profile_log = [] if capture else None
    ops.record_calls = [] if capture else None
    out = {}
    try:
        before = ops.launch_count
        try:
            fn(*inputs)
            out["error"] = None
        except Exception as e:  # noqa: BLE001 -- the refusals are part of what is recorded
            out["error"] = (type(e).__name__, str(e))
        out["launches"] = ops.launch_count - before
        out["calls"] = list(tr.calls)
        if capture:
            out["profile"] = [(name, flops) for name, flops, _, _ in ops.profile_log]
            out["record"] = [(f.__name__, tuple(tr.arg(a) for a in args), name, flops)
                             for f, args, name, flops in ops.record_calls]
            tr.calls.clear()
            ops.replay_calls(ops.record_calls)
            out["replay"] = list(tr.calls)
    finally:
        (_cabi.load, ops._ctx, ops._stream, torch.cuda.Event, torch.cuda.is_current_stream_capturing,
         torch.empty, torch.empty_like, ops.profile_log, ops.record_calls) = saved
    return out


def main():
    data = {(case, mode): record(case, mode) for case in CASES for mode in ("plain", "capture")}
    torch.save(data, OUT)
    print(f"wrote {OUT}: {len(CASES)} cases, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
