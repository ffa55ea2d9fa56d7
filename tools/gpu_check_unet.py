"""End-to-end bring-up on an H100: product UNet (sliders_b200 kernels) vs the fp32 oracle on identical
weights / inputs, with and without LoRA, eager and CUDA-graph; then a first timing."""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import unet as ounet  # noqa: E402
from sliders_b200 import lora as plora  # noqa: E402
from sliders_b200 import ops, synthetic  # noqa: E402
from sliders_b200.unet import UNet2DConditionModel, UNetConfig  # noqa: E402

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
dev = torch.device("cuda:0")


def make_inputs(cfg, B, hw, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, hw, hw, generator=g)
    ehs = torch.randn(B, 77, cfg.cross_attention_dim, generator=g)
    added = None
    if cfg.addition_embed_type == "text_time":
        pooled = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
        added = {"text_embeds": torch.randn(B, pooled, generator=g),
                 "time_ids": torch.tensor([[hw * 8, hw * 8, 0, 0, hw * 8, hw * 8]] * B, dtype=torch.float32)}
    return x, ehs, added


def to_dev(x, ehs, added, dtype):
    a = None
    if added is not None:
        a = {k: v.to(dev, dtype if k == "text_embeds" else torch.float32) for k, v in added.items()}
    return x.to(dev, dtype), ehs.to(dev, dtype), a


def stats(name, got, ref):
    got, ref = got.float(), ref.float()
    d = got - ref
    rel = (d.norm() / ref.norm()).item()
    print(f"  {name}: max_abs {d.abs().max().item():.4g} rel_rms {rel:.4g} ref_std {ref.std().item():.3g} "
          f"finite {bool(torch.isfinite(got).all())}", flush=True)
    return rel


def run(cfg_name, B, hw, t=500, with_lora=True, time_it=False):
    pcfg = getattr(UNetConfig, cfg_name)() if hasattr(UNetConfig, cfg_name) else None
    ocfg = getattr(ounet.UNetConfig, cfg_name)()
    if pcfg is None:
        pcfg = UNetConfig.from_dict(ocfg.__dict__)
    print(f"== {cfg_name} B={B} latent {hw}x{hw} t={t}", flush=True)
    t0 = time.time()
    with torch.device(dev):
        pm = UNet2DConditionModel(pcfg).to(torch.bfloat16)
    synthetic.init_synthetic_(pm, seed=1)
    om = None
    with torch.device(dev):
        om = ounet.UNet2DConditionModel(ocfg)
    om.load_state_dict({k: v.float() for k, v in pm.state_dict().items()})
    om.eval()
    print(f"  models built in {time.time() - t0:.1f}s", flush=True)
    x, ehs, added = make_inputs(ocfg, B, hw)
    xb, eb, ab = to_dev(x, ehs, added, torch.bfloat16)
    xf, ef, af = to_dev(x, ehs, added, torch.float32)
    # the oracle sees the same bf16-rounded inputs
    xf, ef = xb.float(), eb.float()
    if af is not None:
        af["text_embeds"] = ab["text_embeds"].float()
    with torch.no_grad():
        ref = om(xf, t, ef, added_cond_kwargs=af).sample
        got = pm(xb, t, eb, added_cond_kwargs=ab).sample
    torch.cuda.synchronize()
    ok = stats("no LoRA  kernels vs fp32 oracle", got, ref) < 3e-2
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        ref_bf = om(xb, t, eb, added_cond_kwargs=ab).sample
    stats("(context) torch bf16-autocast oracle vs fp32 oracle", ref_bf, ref)
    if with_lora:
        saved = list(plora.DEFAULT_TARGET_REPLACE)
        plora.DEFAULT_TARGET_REPLACE += plora.UNET_TARGET_REPLACE_MODULE_CONV
        try:
            net = plora.LoRANetwork(pm, rank=4, multiplier=1.0, alpha=1.0, train_method="noxattn").to(dev, torch.bfloat16)
        finally:
            del plora.DEFAULT_TARGET_REPLACE[len(saved):]
        synthetic.init_lora_nonzero_(net, seed=2, up_std=0.05)
        # oracle side: fold the same LoRA delta into fp32 weight copies:  W' = W + s * up @ down
        sd = net.state_dict()
        om2 = om
        leaves = dict(om2.named_modules())
        scale_by_leaf = {}
        for l in net.unet_loras:
            path = l.lora_name[len("lora_unet_"):]
            scale_by_leaf[l.lora_name] = l.scale
        name_map = {("lora_unet_" + n.replace(".", "_")): m for n, m in leaves.items()}
        slider = 2.0
        with torch.no_grad():
            for l in net.unet_loras:
                m = name_map[l.lora_name]
                up = sd[l.lora_name + ".lora_up.weight"].float()
                down = sd[l.lora_name + ".lora_down.weight"].float()
                if down.dim() == 4:
                    delta = torch.einsum("or,rikl->oikl", up[:, :, 0, 0], down)
                else:
                    delta = up @ down
                m.weight.add_(delta * (slider * l.scale))
            ref_l = om2(xf, t, ef, added_cond_kwargs=af).sample
            net.set_lora_slider(slider)
            with net:
                got_l = pm(xb, t, eb, added_cond_kwargs=ab).sample
            got_off = pm(xb, t, eb, added_cond_kwargs=ab).sample
        stats("LoRA x2.0 kernels vs fp32 oracle (folded weights)", got_l, ref_l)
        stats("LoRA effect size (oracle with vs without)", ref_l, ref)
        print(f"  multiplier 0 after exit == no-LoRA run bit-exact: {bool(torch.equal(got_off, got))}", flush=True)
        # CUDA graph
        pm.use_cuda_graph = True
        with torch.no_grad():
            with net:
                g1 = pm(xb, t, eb, added_cond_kwargs=ab).sample
                net.set_lora_slider(-1.0)
            with net:
                g2 = pm(xb, t, eb, added_cond_kwargs=ab).sample
            g0 = pm(xb, t, eb, added_cond_kwargs=ab).sample
        pm.use_cuda_graph = False
        with torch.no_grad():
            with net:
                e2 = pm(xb, t, eb, added_cond_kwargs=ab).sample
        print(f"  graph(slider 2) == eager bit-exact: {bool(torch.equal(g1, got_l))}; graph(slider -1) == eager: "
              f"{bool(torch.equal(g2, e2))}; graph(off) == eager: {bool(torch.equal(g0, got))}", flush=True)
        net.set_lora_slider(1.0)
    if time_it:
        ops.launch_count = 0
        with torch.no_grad():
            pm(xb, t, eb, added_cond_kwargs=ab)
        print(f"  launches per forward: {ops.launch_count}", flush=True)
        for graph in (False, True):
            pm.use_cuda_graph = graph
            ctx = net if with_lora else torch.no_grad()
            with torch.no_grad(), ctx:
                for _ in range(3):
                    pm(xb, t, eb, added_cond_kwargs=ab)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.time()
                e0.record()
                n = 10
                for _ in range(n):
                    pm(xb, t, eb, added_cond_kwargs=ab)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / n
            print(f"  {'graph' if graph else 'eager'}: {ms:.2f} ms / forward of {B} passes -> {B / ms * 1e3:.1f} passes/s "
                  f"(host wall {1e3 * (time.time() - t0) / n:.2f} ms)", flush=True)
        pm.use_cuda_graph = False
    return ok


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "tiny"
    print(torch.cuda.get_device_name(0), flush=True)
    ok = True
    if which in ("tiny", "all"):
        ok &= run("tiny_xl", 2, 32)
        ok &= run("tiny_xl", 1, 64, t=19)
    if which in ("sdxl", "all"):
        ok &= run("sdxl", 2, 128, time_it=True)
    if which == "sdxl8":
        ok &= run("sdxl", 8, 128, time_it=True, with_lora=True)
    if which == "prof":
        # one eager forward of 8 passes between cudaProfilerStart/Stop (run under `ncu --profile-from-start off`)
        sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        import bench
        nb = int(sys.argv[2]) if len(sys.argv) > 2 else 8
        unet, net = bench.build_product(dev)
        lat_h, ehs_h, pooled_h, tids_h = bench.make_host_inputs(nb, "sdxl", pin=False)
        args = (lat_h.to(dev), 500, ehs_h.to(dev))
        added = {"text_embeds": pooled_h.to(dev), "time_ids": tids_h.to(dev)}
        with torch.no_grad(), net:
            unet(*args, added_cond_kwargs=added)
            torch.cuda.synchronize()
            torch.cuda.profiler.start()
            unet(*args, added_cond_kwargs=added)
            torch.cuda.synchronize()
            torch.cuda.profiler.stop()
    print("ALL OK" if ok else "SOME BAD", flush=True)
    sys.exit(0 if ok else 1)
