"""One-GPU ViT-L/16 training step at bench.py's workload (2 x 224^2 + 8 x 96^2 crops, B = 64 images) with two head
geometries, alternated in one run:

  shared   DINO and iBOT heads 65 536 prototypes / hidden 2048 / bottleneck 256 (ssl_default_config.yaml, bench.py)
  dinov3   DINO head 262 144 / 8192 / 512, iBOT head 98 304 / 4096 / 384 (the DINOv3 recipes' dino.head_* / ibot.head_*)

Prints the card name and power limit, then per round and geometry: ms/step (CUDA events over --steps device-resident
steps after --warmup) and torch.cuda.max_memory_allocated of the engine's whole life (buffers, parameters, steps).
With --profile, a separate run instead: one single-stream step with CUDA events around every GEMM launch (prototype
GEMMs: those with a prototype count among M / N / K), and two profiled steps (torch.profiler) summing the device time
of the Sinkhorn kernels (colmax, sk_colsum_part, sk_rowsum) and of the cross-entropy (ce_fwd_bwd, metric_rows).
usage: python tools/bench_recipe_heads.py [--steps 10] [--warmup 3] [--batch 64] [--rounds 2] [--profile]"""
import argparse
import collections
import dataclasses
import gc
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch

from gpu_timing import card, cuda_ms

HEADS = {"shared": {}, "dinov3": dict(n_prototypes=262144, head_hidden=8192, head_bottleneck=512, ibot_n_prototypes=98304,
                                      ibot_head_hidden=4096, ibot_head_bottleneck=384)}
HYPER = dict(teacher_temp=0.04, lr=1e-4, wd=0.04, last_layer_lr=0.0, momentum=0.996)      # bench.py's
SINKHORN = ("colmax_kernel", "sk_colsum_part_kernel", "sk_rowsum_kernel")
CROSS_ENTROPY = ("ce_fwd_bwd_kernel", "metric_rows_kernel")


def build(name, B):
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import init_reference_like, synthetic_batch
    cfg = config_for("vit_large", **HEADS[name])
    batch = synthetic_batch(cfg, B, seed=0, pin=True)
    eng = Engine(cfg, B, max_masked=int(batch["mask_indices_list"].shape[0]))
    init_reference_like(eng, seed=0)
    eng.set_batch(batch)
    return cfg, eng


def step_ms(name, B, steps, warmup):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    cfg, eng = build(name, B)
    ms = cuda_ms(lambda: eng.train_step(None, **HYPER), steps, warmup)
    m = eng.read_metrics()
    peak = torch.cuda.max_memory_allocated()
    del eng
    gc.collect()
    return ms, peak, m


def profiled(name, B):
    from torch.profiler import ProfilerActivity, profile
    from dinov3_jax import ops
    torch.cuda.empty_cache()
    cfg, eng = build(name, B)
    for _ in range(2):
        eng.train_step(None, **HYPER)
    # GEMMs: one single-stream step with an event pair per launch (as bench.py's roofline leg)
    overlap, eng.wgrad_overlap = eng.wgrad_overlap, False
    ops.PROFILE = []
    eng.train_step(None, **HYPER)
    torch.cuda.synchronize()
    prof, ops.PROFILE = ops.PROFILE, None
    eng.wgrad_overlap = overlap
    protos = {cfg.head_dims("dino_head")[2], cfg.head_dims("ibot_head")[2]}
    proto = [p for p in prof if protos & set(p[4][:3])]
    proto_ms = sum(p[2].elapsed_time(p[3]) for p in proto)
    all_ms = sum(p[2].elapsed_time(p[3]) for p in prof)
    # Sinkhorn / cross-entropy: summed device time per kernel over two profiled steps
    with profile(activities=[ProfilerActivity.CUDA]) as tp:
        for _ in range(2):
            eng.train_step(None, **HYPER)
        torch.cuda.synchronize()
    agg = collections.Counter()
    for ev in tp.key_averages():
        agg[ev.key] += getattr(ev, "self_device_time_total", 0) or getattr(ev, "self_cuda_time_total", 0)
    pick = lambda names: sum(v for k, v in agg.items() if any(n in k for n in names)) / 2e3      # ms per step
    del eng
    gc.collect()
    return dict(proto_gemm_ms=proto_ms, proto_gemms=len(proto), all_gemm_ms=all_ms, sinkhorn_ms=pick(SINKHORN),
                cross_entropy_ms=pick(CROSS_ENTROPY), kernel_ms=sum(agg.values()) / 2e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    from dinov3_jax import _native
    _native.init(0)
    print(card(), flush=True)
    B = args.batch
    if args.profile:
        for name in HEADS:
            r = profiled(name, B)
            print(f"{name:7s} B = {B}: prototype GEMMs {r['proto_gemm_ms']:.2f} ms ({r['proto_gemms']} launches; all GEMMs "
                  f"{r['all_gemm_ms']:.2f} ms, single stream), Sinkhorn {r['sinkhorn_ms']:.2f} ms, cross-entropy "
                  f"{r['cross_entropy_ms']:.2f} ms, summed kernel time {r['kernel_ms']:.2f} ms per step", flush=True)
        return
    for rnd in range(args.rounds):
        for name in HEADS:
            ms, peak, m = step_ms(name, B, args.steps, args.warmup)
            print(f"round {rnd} {name:7s} B = {B}: {ms:.2f} ms/step, max_memory_allocated {peak / 2**30:.2f} GiB, "
                  f"dino_local {m['dino_local_crops_loss']:.3f}, ibot {m['ibot_loss']:.3f}", flush=True)


if __name__ == "__main__":
    main()
