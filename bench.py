#!/usr/bin/env python
"""bench.py — DINOv3 SSL training step on H100: global-crops/sec, ViT-L/16, 224^2, 2 global + 8 local crops, bf16.

Contract (driver): `python bench.py --gpus N --steps K --warmup W` (torchrun launches N ranks for N > 1) prints ONE
JSON line on rank 0.  `--impl reference` times the CPU restatement of the reference step (oracle/, "port") on the
host cores instead (the reference's JAX stack is not installable here; see DESIGN.md).
`--dump-outputs DIR` writes what the last timed step computed (loss terms, seeded samples of the updated parameters
and of the gradients) as DIR/<name>.npy, so that two builds can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200"))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

ARCH_FLOPS = {}  # filled by block_flops()


def f_img(D, L, Ng, Nl, n_local=8):
    """Algorithmic attention+MLP FLOPs per image (BASELINE.md §3): teacher fwd on 2 global crops + 3x student."""
    f_blk = lambda N: 24 * N * D * D + 4 * N * N * D
    return L * (2 * f_blk(Ng) + 3 * (2 * f_blk(Ng) + n_local * f_blk(Nl)))


# NVIDIA H100 SXM data sheet (700 W part): dense bf16 tensor-core rate.  An upper bound, not reached.
H100_BF16_TFLOPS = 989.0


def dump_outputs(eng, out_dir, write, per_tensor=4096):
    """The last timed step's results as DIR/<name>.npy: every loss term / metric (float64), and for the student
    parameters, the teacher parameters and the student gradients a fixed sample of `per_tensor` elements of every
    tensor (float32, tensors in name order, indices drawn from a generator seeded by the tensor name).  Every rank
    takes part (under FSDP the export gathers the shards); only the one with `write` set writes."""
    import zlib

    import numpy as np
    metrics = eng.read_metrics()
    trees = {"param": eng.params.export_reference_tree("param"), "grad": eng.params.export_reference_tree("grad")}
    if not write:
        return
    os.makedirs(out_dir, exist_ok=True)
    for k, v in metrics.items():
        np.save(os.path.join(out_dir, f"metric_{k}.npy"), np.array([v], dtype=np.float64))
    for fname, what, prefix in (("student_params_sample", "param", "student_"), ("teacher_params_sample", "param", "teacher_"),
                                ("student_grads_sample", "grad", "student_")):
        parts = []
        for name in sorted(k for k in trees[what] if k.startswith(prefix)):
            flat = trees[what][name].reshape(-1)
            g = torch.Generator().manual_seed(zlib.crc32(name.split("_", 1)[1].encode()))
            idx = torch.randint(0, flat.numel(), (min(per_tensor, flat.numel()),), generator=g)
            parts.append(flat[idx.to(flat.device)].float().cpu())
        np.save(os.path.join(out_dir, f"{fname}.npy"), torch.cat(parts).numpy().astype(np.float32))


class ClockSampler:
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.rows, self.proc = [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(index)], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), line.strip()))

    def stop(self, t0, t1):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        for t, line in self.rows:
            if t < t0 or t > t1 + 0.2:
                continue
            f = [x.strip() for x in line.split(",")]
            try:
                sm.append(float(f[0])); mx = float(f[1])
            except Exception:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


def log(msg):
    if int(os.environ.get("RANK", "0")) == 0:
        print(f"[bench {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def hyper(it):
    # ssl_default_config.yaml:124-128,142-146 at iteration `it` of the default schedule (values only matter for parity)
    return dict(teacher_temp=0.04, lr=1e-4, wd=0.04, last_layer_lr=0.0, momentum=0.996)


def cpu_reference_rate(arch, threads, sample_B, steps=1, warmup=0, **cfg_kw):
    """Times oracle.step.train_step (CPU restatement of the reference step) on `sample_B` images per step."""
    from oracle import cfg_for
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    from oracle.step import init_opt_state, train_step
    threads = max(1, min(threads, 32))   # beyond ~32 threads the fp32 restatement stops scaling (many small ops)
    torch.set_num_threads(threads)
    cfg = cfg_for(arch, **cfg_kw)
    P = init_params(cfg, 0)
    st = init_opt_state(P)
    batch = synthetic_batch(cfg, sample_B, 0)
    times, first_loss = [], None
    for i in range(warmup + steps):
        t0 = time.time()
        P, st, loss, m, _ = train_step(P, st, batch, cfg, **hyper(i))
        times.append(time.time() - t0)
        if first_loss is None:
            first_loss = float(loss)         # loss of the un-updated parameters (what parity_check compares)
    dt = sum(times[warmup:]) / steps
    return 2 * sample_B / dt, dt, float(loss), threads, first_loss


def oracle_kw(args):
    return dict(n_prototypes=args.prototypes, patch=args.patch, local_size=args.local_size)


def parity_check(args, cfg, loss_cpu, local_rank):
    """Engine vs oracle on the cpu_baseline sample: same architecture, K, parameters (oracle.init_params seed 0) and
    batch (oracle.batch.synthetic_batch seed 0) — the loss of the un-updated parameters, relative difference."""
    from dinov3_jax.engine import Engine
    from oracle import cfg_for
    from oracle.batch import synthetic_batch as oracle_batch
    from oracle.model import init_params
    ocfg = cfg_for(args.arch, **oracle_kw(args))
    B = args.cpu_sample_batch
    batch = oracle_batch(ocfg, B, 0)
    eng = Engine(cfg, B, device=f"cuda:{local_rank}", max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    eng.params.load_reference_tree(init_params(ocfg, 0))
    eng.set_batch(batch)
    eng.forward_backward(hyper(0)["teacher_temp"])
    loss = eng.read_metrics()["total_loss"]
    rel = abs(loss - loss_cpu) / abs(loss_cpu)
    return {"engine_loss": loss, "oracle_loss": loss_cpu, "rel": rel, "ok": bool(rel < 1e-3),
            "what": f"{args.arch} full depth, K={cfg.n_prototypes}, {B} images, fp32 oracle vs bf16 engine, tolerance 1e-3"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--arch", default="vit_large")
    ap.add_argument("--batch", type=int, default=64, help="images per GPU (ssl_default_config.yaml:75)")
    ap.add_argument("--prototypes", type=int, default=65536)
    ap.add_argument("--patch", type=int, default=16)
    ap.add_argument("--local-size", type=int, default=96, help="98 for patch 14 (96 is not divisible, layers/patch_embed.py:48-49)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--gram", choices=["off", "ema", "frozen"], default="off",
                    help="add the Gram-anchoring term (gram.use_loss; SURVEY 8f.2): ema = EMA teacher's patches as targets, "
                         "frozen = a third backbone pass with a snapshot of the teacher; off = the BASELINE headline workload")
    ap.add_argument("--remat", action="store_true", help="activation rematerialisation (train.checkpointing): BASELINE configs[4]")
    ap.add_argument("--cpu-sample-batch", type=int, default=2, help="images per CPU-baseline step (bounded sample: ~15-25 s of CPU work)")
    ap.add_argument("--cpu-budget-s", type=float, default=150.0, help="wall-clock bound of the --impl reference arm")
    ap.add_argument("--no-checks", action="store_true", help="skip parity_check / fsdp_check")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's loss terms and seeded samples of parameters / gradients as DIR/<name>.npy")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    cores = os.cpu_count() or 1

    from dinov3_jax.engine.config import ARCHS
    D, L, H = ARCHS[args.arch]
    Ng, Nl = (224 // args.patch) ** 2 + 1, (args.local_size // args.patch) ** 2 + 1
    flops_per_gcrop = f_img(D, L, Ng, Nl) / 2
    cfg_desc = {"workload": f"{args.arch}/{args.patch} student+teacher, 2x224^2 + 8x{args.local_size}^2 crops, {args.batch} img/GPU, "
                            f"K={args.prototypes} prototypes, DINO+iBOT+KoLeo, clip+AdamW+EMA (BASELINE configs[3] per-GPU shape)",
                "global_batch": args.batch * world, "parallelism": f"fsdp{world}" if world > 1 else "single",
                "l2": "inputs+activations per step >> 50 MB L2 (no flush needed)"}

    if args.impl == "reference":
        if rank != 0:
            return
        # The reference's JAX stack cannot be installed offline (DESIGN.md §2), so this arm times the CPU restatement of
        # the same step (oracle/, kind "port") on a BOUNDED SAMPLE of the workload: `--cpu-sample-batch` images per
        # step instead of 64.  Everything printed describes what actually ran.
        budget = float(args.cpu_budget_s)
        t_probe = time.time()
        _, dt1, _, used, _ = cpu_reference_rate(args.arch, cores, args.cpu_sample_batch, steps=1, warmup=0, **oracle_kw(args))   # untimed probe = warm-up 1
        steps = max(1, min(args.steps, int((budget - (time.time() - t_probe)) / max(dt1, 1e-3)) - max(args.warmup - 1, 0)))
        warm = max(0, min(args.warmup - 1, int(budget / max(dt1, 1e-3)) - steps))
        val, dt, _, used, _ = cpu_reference_rate(args.arch, cores, args.cpu_sample_batch, steps=steps, warmup=warm, **oracle_kw(args))
        ref_cfg = dict(cfg_desc)
        ref_cfg.update({"sample": f"{args.cpu_sample_batch} images per step (bounded sample of the {args.batch}-img/GPU step; "
                                  f"crops/s on the CPU is taken as batch-size independent)",
                        "global_batch": args.cpu_sample_batch, "parallelism": "single host process", "same_config": False,
                        "extrapolated": True, "requested": {"gpus": args.gpus, "steps": args.steps, "warmup": args.warmup}})
        print(json.dumps({
            "impl": "reference", "metric": "global_crops_per_sec", "value": val, "unit": "global-crops/s",
            "n_gpus": 1, "steps": steps, "warmup": warm + 1, "ms_per_step": dt * 1e3,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": ref_cfg,
            "cpu_baseline": {"value": val, "unit": "global-crops/s", "cores": used, "kind": "port",
                             "sample": f"torch-CPU fp32 restatement of the reference train_step (oracle/), {args.arch}, "
                                       f"{args.cpu_sample_batch} images/step, {steps} timed steps after {warm + 1} warm-up; "
                                       f"the reference's JAX stack is not installable offline"},
            "e2e": {"value": val, "unit": "global-crops/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
        return

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device — the GPU engine has no CPU fallback (use --impl reference for the CPU arm)")
    torch.cuda.set_device(local_rank)
    comm = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
        from dinov3_jax.fsdp.runtime import Comm
        comm = Comm(dist.group.WORLD)
    from dinov3_jax import _native, ops
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import synthetic_batch, init_reference_like
    _native.init(local_rank)
    cfg = config_for(args.arch, n_prototypes=args.prototypes, patch=args.patch, local_size=args.local_size)
    if args.gram != "off":
        import dataclasses
        cfg = dataclasses.replace(cfg, gram_use_loss=True, gram_ema_teacher=args.gram == "ema", gram_it_load_ema_teacher=0,
                                  gram_remove_only_teacher_neg=True)
        cfg_desc["workload"] += f" + Gram anchoring ({args.gram} teacher)"
        cfg_desc["gram"] = args.gram
    B = args.batch
    log(f"building synthetic batch B={B}")
    batch = synthetic_batch(cfg, B, seed=rank, pin=True)
    M = int(batch["mask_indices_list"].shape[0])
    eng = Engine(cfg, B, device=f"cuda:{local_rank}", max_masked=M, comm=comm, remat=args.remat)
    cfg_desc["activation_remat"] = bool(args.remat)
    if world > 1:
        cfg_desc["grad_reduce_scatter"] = ("push over NVLink peer memory (GEMM epilogue + d3_scatter_add_peers)" if eng.fsdp.push else "nccl reduce_scatter")
    cfg_desc["wgrad_stream"] = bool(eng.wgrad_overlap)
    log(f"engine allocated ({torch.cuda.memory_allocated() / 2**30:.1f} GiB); initialising {eng.params.n_params() / 1e6:.1f} M student params")
    init_reference_like(eng, seed=0)
    log("params loaded")

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    def step_device(i):
        eng.train_step(None, **hyper(i))

    def step_e2e(i):
        eng.train_step(batch, **hyper(i))     # pinned host -> device copies inside
        return eng.read_metrics()["total_loss"]  # device -> host read of the loss

    # ---- warm-up (device-resident inputs)
    eng.set_batch(batch)
    for i in range(max(args.warmup, 3)):
        tw = time.time()
        step_device(i)
        torch.cuda.synchronize()
        log(f"warm-up step {i}: {time.time() - tw:.3f} s")
    barrier()
    sampler = ClockSampler(local_rank) if rank == 0 else None
    _native.reset_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.time()
    e0.record()
    for i in range(args.steps):
        step_device(i)
    e1.record()
    barrier()
    t1 = time.time()
    launches = _native.launch_count()
    ms = e0.elapsed_time(e1) / args.steps
    log(f"timed region: {ms:.2f} ms/step")
    clocks = sampler.stop(t0, t1) if sampler else None
    if args.dump_outputs:
        dump_outputs(eng, args.dump_outputs, write=rank == 0)
    # ---- end-to-end: host buffers, H2D inside, loss read back every step
    for i in range(2):
        step_e2e(i)
    barrier()
    e0.record()
    loss = 0.0
    for i in range(args.steps):
        loss = step_e2e(i)
    e1.record()
    barrier()
    ms_e2e = e0.elapsed_time(e1) / args.steps
    log(f"e2e: {ms_e2e:.2f} ms/step")
    if world > 1:
        t = torch.tensor([ms, ms_e2e], device="cuda")
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        ms, ms_e2e = t.tolist()
    h2d = sum(batch[k].numel() * batch[k].element_size() for k in ("collated_global_crops", "collated_local_crops", "collated_masks", "mask_indices_list"))
    # ---- roofline leg: one instrumented step, CUDA events around every tensor-core GEMM launch
    # (single stream for this step: with the weight-gradient stream active a launch's event pair would also time its
    # wait for SMs held by the other stream's kernel)
    overlap, eng.wgrad_overlap = eng.wgrad_overlap, False
    fwd_overlap, eng.fwd_overlap = eng.fwd_overlap, False
    ops.PROFILE = []
    step_device(0)
    torch.cuda.synchronize()
    prof, ops.PROFILE = ops.PROFILE, None
    eng.wgrad_overlap = overlap
    eng.fwd_overlap = fwd_overlap
    g_flops = sum(p[1] for p in prof)
    g_ms = sum(p[2].elapsed_time(p[3]) for p in prof)
    peak = H100_BF16_TFLOPS
    gemm_tf = g_flops / (g_ms * 1e-3) / 1e12 if g_ms else 0.0
    value = 2 * B * world / (ms * 1e-3)
    e2e_value = 2 * B * world / (ms_e2e * 1e-3)
    step_tf = value * flops_per_gcrop / world / 1e12
    out = {
        "metric": "global_crops_per_sec", "value": value, "unit": "global-crops/s", "n_gpus": world, "steps": args.steps,
        "warmup": max(args.warmup, 3), "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "bf16", "data": "synthetic", "config": cfg_desc, "clocks": clocks, "gpu_launches": int(launches),
        "e2e": {"value": e2e_value, "unit": "global-crops/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": 32,
                "ms_per_step": ms_e2e, "loss": loss},
        "roofline": {"bound": "tensor", "kernel": "gemm_kernel (every wgmma GEMM launch of one step)",
                     "achieved": gemm_tf, "peak": peak, "unit": "TFLOP/s", "frac": gemm_tf / peak,
                     "traffic": None, "traffic_unit": "not measured",
                     "peak_source": "H100 SXM data sheet, dense bf16 (not reached)", "launches": len(prof),
                     "share_of_step": g_ms / ms if ms else None},
        "step_roofline": {"achieved": step_tf, "peak": peak, "unit": "TFLOP/s", "frac": step_tf / peak,
                          "note": "attention+MLP algorithmic FLOPs (BASELINE.md §3) / step time / GPU"},
    }
    if world > 1 and not args.no_checks:
        from dinov3_jax.fsdp.selfcheck import fsdp_equals_single_gpu
        try:
            out["fsdp_check"] = fsdp_equals_single_gpu(comm, f"cuda:{local_rank}")
        except Exception as e:                      # the timed numbers above stand; the check reports its own failure
            out["fsdp_check"] = {"ok": False, "error": repr(e)[:300]}
        log(f"fsdp_check: {out['fsdp_check']}")
    if rank == 0:
        if world == 1 and not args.no_cpu_baseline:
            log("cpu baseline (oracle port) ...")
            v, dt, _, cores, loss_cpu = cpu_reference_rate(args.arch, cores, args.cpu_sample_batch, steps=2, warmup=0, **oracle_kw(args))
            log(f"cpu baseline: {dt:.1f} s/step")
            out["cpu_baseline"] = {"value": v, "unit": "global-crops/s", "cores": cores, "kind": "port",
                                   "sample": f"oracle train_step (torch-CPU fp32 restatement), {args.arch}, "
                                             f"{args.cpu_sample_batch} images per step, 2 steps of {dt:.1f} s"}
            if not args.no_checks:
                # the same sample through the engine (same parameters, same batch): full-size model, K prototypes
                try:
                    out["parity_check"] = parity_check(args, cfg, loss_cpu, local_rank)
                except Exception as e:
                    out["parity_check"] = {"ok": False, "error": repr(e)[:300]}
                log(f"parity_check: {out['parity_check']}")
        print(json.dumps(out))
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
