"""GPU: where the bench.py training step's time goes, kernel by kernel.

torch.profiler (CUDA activities) over a few Engine.train_step calls of the bench.py workload (ViT-L/16, B = 64,
K = 65 536 prototypes, device-resident batch): per-step time, share of the summed kernel time and launches per step of
every kernel name.  Then one single-stream step with CUDA events around every GEMM launch (as bench.py's roofline leg)
splits the GEMM time into forward, input-gradient, weight-gradient and prototype-head (a dimension of K) calls.  The
card name and power limit are read in the same run.  Prints only; writes nothing.
usage: python tools/step_kernel_times.py [--steps 3] [--warmup 3] [--batch 64] [--arch vit_large] [--top 40]"""
import argparse
import collections
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200"))
import torch  # noqa: E402

from gpu_timing import card, cuda_ms  # noqa: E402


def kernel_name(key):
    """'void d3::gemm_kernel<128, 0, 1, 1>(CUtensorMap_st, ...)' -> 'd3::gemm_kernel<128, 0, 1, 1>'"""
    name = key.split("(")[0].strip()
    return name[5:] if name.startswith("void ") else name


def gemm_class(shape, prototypes):
    M, N, K, a_mn, b_mn = shape
    if prototypes in (M, N, K):
        return "head (prototype layer)"
    return {(0, 1): "forward", (0, 0): "input gradient", (1, 1): "weight gradient"}.get((a_mn, b_mn), f"layout {a_mn}{b_mn}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="vit_large")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--prototypes", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--top", type=int, default=40)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_kernel_times.py: no CUDA device")
    from dinov3_jax import _native, ops
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import init_reference_like, synthetic_batch

    torch.cuda.set_device(0)
    _native.init(0)
    cfg = config_for(args.arch, n_prototypes=args.prototypes)
    batch = synthetic_batch(cfg, args.batch, seed=0)
    eng = Engine(cfg, args.batch, device="cuda:0", max_masked=int(batch["mask_indices_list"].shape[0]))
    init_reference_like(eng, seed=0)
    eng.set_batch(batch)
    hyper = dict(teacher_temp=0.04, lr=1e-4, wd=0.04, last_layer_lr=0.0, momentum=0.996)
    for _ in range(args.warmup):
        eng.train_step(None, **hyper)
    torch.cuda.synchronize()
    print(card())

    # ---- every kernel of `steps` steps
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        step_ms = cuda_ms(lambda: eng.train_step(None, **hyper), args.steps, 0)     # warmed up above, unprofiled
    t_us, n = collections.Counter(), collections.Counter()
    for ev in prof.key_averages():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = kernel_name(ev.key)
        t_us[name] += ev.self_device_time_total
        n[name] += ev.count
    tot = sum(t_us.values())
    print(f"{args.arch} B={args.batch} K={args.prototypes}: {step_ms:.2f} ms per step under the profiler, "
          f"kernels {tot / 1e3 / args.steps:.2f} ms per step (streams overlap), "
          f"{sum(n.values()) / args.steps:.0f} launches per step")
    gemm = sum(v for k, v in t_us.items() if "gemm_kernel" in k)
    print(f"  gemm_kernel: {gemm / 1e3 / args.steps:.2f} ms per step, {100 * gemm / tot:.1f}% of kernel time")
    for name, v in t_us.most_common(args.top):
        print(f"{v / 1e3 / args.steps:9.3f} ms {100 * v / tot:5.1f}%  n={n[name] / args.steps:6.1f}  {name[:110]}")

    # ---- GEMM time by call class: one step on one stream, CUDA events around every launch
    overlap, eng.wgrad_overlap = eng.wgrad_overlap, False
    fwd_overlap, eng.fwd_overlap = eng.fwd_overlap, False
    ops.PROFILE = []
    eng.train_step(None, **hyper)
    torch.cuda.synchronize()
    launches, ops.PROFILE = ops.PROFILE, None
    eng.wgrad_overlap, eng.fwd_overlap = overlap, fwd_overlap
    ms, fl, cnt = collections.Counter(), collections.Counter(), collections.Counter()
    for _, flops, s, e, shape in launches:
        c = gemm_class(shape, args.prototypes)
        ms[c] += s.elapsed_time(e)
        fl[c] += flops
        cnt[c] += 1
    print(f"GEMM launches of one single-stream step: {sum(ms.values()):.2f} ms, {len(launches)} launches")
    for c, v in ms.most_common():
        print(f"  {c:24s} {v:8.2f} ms  n={cnt[c]:4d}  {fl[c] / v / 1e9:6.1f} TFLOP/s")


if __name__ == "__main__":
    main()
