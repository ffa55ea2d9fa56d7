"""Null-text inversion timings on SD1.5 at 512 px (64x64 latents, synthetic weights), in one process:
  * cross-attention dQ + dK + dV per call, query-split vs unsplit, alternated, at the SD1.x and SDXL cross-attention
    shapes (batch 1 and 2);
  * the d_ctx GEMM, fp32 split-K vs the plain sb200_gemm (bf16 out) at M = 77, N = 768, K = 24 960;
  * ms per inner step (forward + backward + loss + Adam), eager and CUDA-graphed;
  * wall time of a full `invert` (N steps x I inner iterations, epsilon = 0 so the count is fixed).
Usage: gpu_time_inversion.py [N I]  (default 50 10)."""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import unet as ounet  # noqa: E402
from sliders_b200 import ops, optim, synthetic  # noqa: E402
from sliders_b200.inversion import NullInversion, ddim_affine, prev_step_alphas  # noqa: E402
from sliders_b200.scheduler import DDIMScheduler  # noqa: E402
from sliders_b200.unet import UNet2DConditionModel, UNetConfig  # noqa: E402

BF = torch.bfloat16
dev = torch.device("cuda:0")
N_STEPS, INNER = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (50, 10)


def card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


print(f"card: {card()}", flush=True)

# ---- cross-attention dK / dV: split vs unsplit, alternated
g = torch.Generator().manual_seed(0)
# SD1.x 512 px (8 heads) at batch 1 and 2; SDXL 1024 px (10 / 20 heads of 64) at batch 1 and 2
for Sq, d, heads, B in ((4096, 40, 8, 1), (1024, 80, 8, 1), (256, 160, 8, 1), (4096, 40, 8, 2), (1024, 80, 8, 2),
                        (256, 160, 8, 2), (4096, 64, 10, 1), (1024, 64, 20, 1), (4096, 64, 10, 2), (1024, 64, 20, 2)):
    Skv = 77
    Cc = heads * d
    q = torch.randn(B * Sq, Cc, generator=g).to(dev, BF)
    kv = torch.randn(B * Skv, 2 * Cc, generator=g).to(dev, BF)
    k, v = kv[:, :Cc], kv[:, Cc:]
    dout = torch.randn(B * Sq, Cc, generator=g).to(dev, BF)
    lse = torch.empty(B, heads, Sq, device=dev, dtype=torch.float32)
    o = ops.attention(q, k, v, B, heads, Sq, Skv, d ** -0.5, head_dim=d, lse=lse)
    dq, dkv = torch.empty_like(q), torch.empty_like(kv)
    split = lambda: ops.attention_bwd_split(q, k, v, o, dout, lse, B, heads, Sq, Skv, d ** -0.5, d, dq, dkv[:, :Cc],
                                            dkv[:, Cc:])
    plain = lambda: ops.attention_bwd(q, k, v, o, dout, lse, B, heads, Sq, Skv, d ** -0.5, d, dq, dkv[:, :Cc],
                                      dkv[:, Cc:])
    ts, tp = [], []
    for _ in range(5):
        ts.append(timed(split, 20))
        tp.append(timed(plain, 20))
    print(f"attention_bwd dQ+dK+dV B={B} Sq={Sq} Skv=77 heads={heads} d={d}: split ({ops.attn_bwd_splits(B, heads, Sq, Skv)} "
          f"splits) {min(ts) * 1e3:.1f} us  unsplit {min(tp) * 1e3:.1f} us", flush=True)

# ---- d_ctx GEMM
x = (0.1 * torch.randn(77, 24960, generator=g)).to(dev, BF)
w = (0.02 * torch.randn(768, 24960, generator=g)).to(dev, BF)
ts, tp = [], []
for _ in range(5):
    ts.append(timed(lambda: ops.gemm_splitk_f32(x, w), 20))
    tp.append(timed(lambda: ops.gemm(x, w), 20))
print(f"d_ctx GEMM 77 x 768 x 24960: split-K fp32 {min(ts) * 1e3:.1f} us  plain sb200_gemm {min(tp) * 1e3:.1f} us",
      flush=True)

# ---- SD1.5 inner step and full invert
cfg = ounet.UNetConfig.sd15()
unet = UNet2DConditionModel(UNetConfig.from_dict(cfg.__dict__))
synthetic.init_synthetic_(unet, seed=1)
unet = unet.to(dev, BF).eval().requires_grad_(False)
sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                      set_alpha_to_one=False)
lat = (0.8 * torch.randn(1, 4, 64, 64, generator=g)).to(dev)
unc = torch.randn(1, 77, 768, generator=g).to(dev)
cond = torch.randn(1, 77, 768, generator=g).to(dev)
target = torch.randn(1, 4, 64, 64, generator=g).to(dev)
eps_c = torch.randn(1, 4, 64, 64, generator=g).to(dev)
sched.set_timesteps(50)
cx, ce = ddim_affine(*prev_step_alphas(sched, 501))
for graph in (False, True):
    unet.use_cuda_graph = graph
    emb = unc.clone().requires_grad_()
    opt = optim.Adam([emb], lr=1e-2)

    def inner():
        eps_u = unet(lat, 501, encoder_hidden_states=emb).sample
        loss = ops.guided_step_loss(eps_u, eps_c, 7.5, lat, cx, ce, target)
        opt.zero_grad()
        loss.backward()
        opt.step()

    for _ in range(3):
        inner()
    torch.cuda.synchronize()
    print(f"inner step (fwd + bwd + loss + Adam), {'graphed' if graph else 'eager'}: {timed(inner, 10):.2f} ms",
          flush=True)

for graph in (False, True):
    unet.use_cuda_graph = graph
    inv = NullInversion(unet, sched, num_ddim_steps=N_STEPS)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    inv.invert(lat, unc, cond, num_inner_steps=INNER, early_stop_epsilon=0.0)
    torch.cuda.synchronize()
    print(f"invert {N_STEPS} steps x {INNER} inner ({inv.unet_calls} grad UNet calls), "
          f"{'graphed' if graph else 'eager'}: {time.perf_counter() - t0:.1f} s", flush=True)
unet.use_cuda_graph = False
