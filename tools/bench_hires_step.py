"""One-GPU ViT-L/16 training step at high resolution: 2 global crops at 512^2 (1 029 tokens with 4 storage tokens,
streamed attention kernels) and 8 local crops at 112^2 (53 tokens), B = 8 images, K = 65536 prototypes.

Prints the card name and power limit, ms/step and global-crops/s (CUDA events over --steps device-resident steps after
--warmup), then, in a separate profiled window, the share of summed kernel time spent in attention launches.
usage: python tools/bench_hires_step.py [--steps 10] [--warmup 3] [--global-size 512] [--batch 8]"""
import argparse
import collections
import dataclasses
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch

from gpu_timing import card, cuda_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--global-size", type=int, default=512)
    ap.add_argument("--local-size", type=int, default=112)
    ap.add_argument("--arch", default="vit_large")
    ap.add_argument("--depth", type=int, default=0, help="blocks (0: the arch's own depth)")
    ap.add_argument("--prototypes", type=int, default=65536)
    args = ap.parse_args()

    from dinov3_jax import _native
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import init_reference_like, synthetic_batch
    _native.init(0)
    print(card(), flush=True)
    # vit_7b runs its recipe's blocks (configs/train/dinov3_vit7b16_*.yaml): SwiGLU64, layernormbf16, mask_k_bias
    recipe = dict(ffn_layer="swiglu", swiglu_align=64, ln_eps=1e-5, mask_k_bias=True) if args.arch == "vit_7b" else {}
    cfg = config_for(args.arch, patch=16, global_size=args.global_size, local_size=args.local_size, n_storage=4,
                     n_prototypes=args.prototypes, **recipe)
    if args.depth:
        cfg = dataclasses.replace(cfg, depth=args.depth)
    B = args.batch
    batch = synthetic_batch(cfg, B, seed=0, pin=True)
    eng = Engine(cfg, B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    init_reference_like(eng, seed=0)
    hyper = dict(teacher_temp=0.04, lr=1e-4, wd=0.04, last_layer_lr=0.0, momentum=0.996)
    eng.set_batch(batch)
    for _ in range(args.warmup):
        eng.train_step(None, **hyper)
    _native.reset_launch_count()
    ms = cuda_ms(lambda: eng.train_step(None, **hyper), args.steps, 0)     # warmed up above, before the count restarts
    launches = _native.launch_count() / args.steps
    loss = eng.read_metrics()["total_loss"]
    ntok = lambda s: (s // 16) ** 2 + 1 + cfg.n_storage
    print(f"{args.arch}/16 ({cfg.depth} blocks, K = {cfg.n_prototypes}), 2 x {args.global_size}^2 ({ntok(args.global_size)} tokens) + 8 x {args.local_size}^2 "
          f"({ntok(args.local_size)} tokens), B = {B}: {ms:.2f} ms/step, {2 * B * 1e3 / ms:.1f} global-crops/s, "
          f"{launches:.0f} launches/step, loss {loss:.4f}", flush=True)

    # ---- attention share: summed device time per kernel name over 2 profiled steps (a separate window: the profiler
    # slows the host); the engine overlaps weight-gradient GEMMs on a second stream, so this is a share of kernel time
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            eng.train_step(None, **hyper)
        torch.cuda.synchronize()
    agg = collections.Counter()
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA or getattr(ev, "self_device_time_total", 0) > 0:
            agg[ev.key] += getattr(ev, "self_device_time_total", 0) or getattr(ev, "self_cuda_time_total", 0)
    total = sum(agg.values())
    attn = {k: v for k, v in agg.items() if "attn" in k}
    print(f"attention: {100 * sum(attn.values()) / total:.1f}% of summed kernel time "
          f"({sum(attn.values()) / 2e3:.2f} of {total / 2e3:.2f} ms per step)")
    for k, v in sorted(attn.items(), key=lambda kv: -kv[1]):
        print(f"  {v / 2e3:8.2f} ms/step  {100 * v / total:5.1f}%  {k[:90]}")


if __name__ == "__main__":
    main()
