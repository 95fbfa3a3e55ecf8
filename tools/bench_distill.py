"""One-GPU distillation step: a ViT-L/16 student of the distilled recipe (layernormbf16, 4 storage tokens, mask_k_bias,
DINO head 262 144 / 8192 / 512, iBOT head 98 304 / 4096 / 384) taught by a frozen 40-block vit_7b teacher (swiglu64,
no qkv bias, 4 storage tokens, the same heads), 2 x 256^2 + 8 x 112^2 crops, random weights.

Prints the card name and power limit, then per batch size B (8, 16, 32 by default; a size that does not fit in memory
is reported as such):
  * ms/step: CUDA events over --steps device-resident train_step calls after --warmup;
  * the teacher pass alone (Engine.teacher_pass: 7B forward, heads, Sinkhorn), CUDA events over --steps calls;
  * torch.cuda.max_memory_allocated over the engine's life;
  * the teacher's GEMM shapes in TFLOP/s (2 M N K over CUDA-event time, --gemm-iters launches each).  The qkv
    projection without a bias is timed with its fixed-flag staged epilogue and with the run-time-flag epilogue,
    alternated: the latter is reached by adding a LayerScale of ones (a flag set dispatch() does not list), which
    keeps the vector loads and stores of an aligned output and adds one multiply per element.
usage: python tools/bench_distill.py [--batches 8 16 32] [--steps 5] [--warmup 2] [--gemm-iters 20]"""
import argparse
import gc
import math
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch

from gpu_timing import card, cuda_ms

HEADS = dict(n_prototypes=262144, head_hidden=8192, head_bottleneck=512, ibot_n_prototypes=98304, ibot_head_hidden=4096,
             ibot_head_bottleneck=384)
CROPS = dict(patch=16, global_size=256, local_size=112)
HYPER = dict(teacher_temp=0.04, lr=1e-4, wd=0.04, last_layer_lr=0.0, momentum=0.996)


def configs():
    from dinov3_jax.engine import config_for
    common = dict(n_storage=4, ln_eps=1e-5, mask_k_bias=True, **CROPS, **HEADS)
    return (config_for("vit_large", **common),
            config_for("vit_7b", ffn_layer="swiglu", swiglu_align=64, qkv_bias=False, **common))


def random_teacher(eng, seed=0):
    """Frozen teacher weights drawn on the device (lecun-normal matrices, LayerNorm 1 / 0, LayerScale 1e-5, small
    tokens): a host-side tree of 6.7 B fp32 values would only be rounded to bf16 again."""
    gen = torch.Generator(device=eng.device).manual_seed(seed)
    for store in eng.t_net.mods.values():
        for name, off in store.offsets.items():
            if off < store.n_mat:
                w = store.w(name)
                w.copy_((torch.randn(w.shape, generator=gen, device=eng.device) / math.sqrt(w.shape[0])).to(w.dtype))
            else:
                v = store.vec(name)
                if name.endswith("/scale"):
                    v.fill_(1.0)
                elif name.endswith("/gamma"):
                    v.fill_(1e-5)
                elif name in ("cls_token", "storage_tokens"):
                    v.copy_(torch.randn(v.shape, generator=gen, device=eng.device) * 0.02)
                else:
                    v.zero_()


def build(B):
    from dinov3_jax.engine import Engine
    from dinov3_jax.engine.synth import init_reference_like, synthetic_batch
    cfg, tcfg = configs()
    batch = synthetic_batch(cfg, B, seed=0, pin=True)
    eng = Engine(cfg, B, max_masked=int(batch["mask_indices_list"].shape[0]), distill=tcfg)
    init_reference_like(eng, seed=0)
    random_teacher(eng)
    eng.set_batch(batch)
    return eng


def step(B, steps, warmup):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    eng = build(B)
    ms = cuda_ms(lambda: eng.train_step(None, **HYPER), steps, warmup)
    t_ms = cuda_ms(lambda: eng.teacher_pass(HYPER["teacher_temp"]), steps, 0)     # the train steps ran the teacher pass
    m = eng.read_metrics()
    peak = torch.cuda.max_memory_allocated()
    T = eng.teacher.T
    del eng
    gc.collect()
    return ms, t_ms, peak, m, T


def gemms(T, iters, rounds=2):
    """TFLOP/s of the teacher's forward GEMMs at T teacher tokens (vit_7b: D 4096, SwiGLU hidden 8192)."""
    from dinov3_jax import ops
    dev, bf16, f32 = "cuda", torch.bfloat16, torch.float32
    D, Hs = 4096, 8192
    g = torch.Generator(device=dev).manual_seed(1)
    r = lambda *s, dt=bf16: (torch.randn(*s, generator=g, device=dev) * 0.05).to(dt)
    Y, Z, Hh, O = r(T, D), r(T, D), r(T, Hs), r(T, D)
    Wqkv, Wp, W1, W3 = r(D, 3 * D), r(D, D), r(D, Hs), r(Hs, D)
    QKV, X12, X, Xo = r(T, 3 * D), r(T, 2 * Hs), r(T, D, dt=f32), r(T, D, dt=f32)
    bD, bH, gam, ones = r(D, dt=f32), r(Hs, dt=f32), r(D, dt=f32), torch.ones(3 * D, device=dev)
    shapes = {
        "qkv (no bias), staged": (lambda: ops.gemm(Y, Wqkv, QKV, b_mn=True), 3 * D, D),
        "qkv (no bias), run-time flags": (lambda: ops.gemm(Y, Wqkv, QKV, b_mn=True, gamma=ones), 3 * D, D),
        "proj + LayerScale + residual": (lambda: ops.gemm(O, Wp, Xo, b_mn=True, bias=bD, gamma=gam, resid=X), D, D),
        "w1 / w2 (+ bias)": (lambda: ops.gemm(Z, W1, X12[:, :Hs], b_mn=True, bias=bH), Hs, D),
        "w3 + LayerScale + residual": (lambda: ops.gemm(Hh, W3, Xo, b_mn=True, bias=bD, gamma=gam, resid=X), D, Hs),
    }
    for fn, _, _ in shapes.values():
        fn()
    out = {k: [] for k in shapes}
    for _ in range(rounds):
        for k, (fn, N, K) in shapes.items():
            ms = cuda_ms(fn, iters, 0)     # every shape ran once above, so the rounds alternate warm shapes
            out[k].append(2.0 * T * N * K / (ms * 1e-3) / 1e12)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 16, 32])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gemm-iters", type=int, default=20)
    args = ap.parse_args()
    from dinov3_jax import _native
    _native.init(0)
    print(card(), flush=True)
    for B in args.batches:
        try:
            res = step(B, args.steps, args.warmup)
        except torch.cuda.OutOfMemoryError:
            res = None
        if res is None:                       # outside the handler: its traceback no longer holds the engine
            gc.collect()
            torch.cuda.empty_cache()
            print(f"B = {B}: does not fit in memory", flush=True)
            continue
        ms, t_ms, peak, m, T = res
        print(f"B = {B}: {ms:.1f} ms/step, teacher pass {t_ms:.1f} ms, max_memory_allocated {peak / 2**30:.2f} GiB, "
              f"dino_local {m['dino_local_crops_loss']:.3f}, ibot {m['ibot_loss']:.3f}", flush=True)
        for k, v in gemms(T, args.gemm_iters).items():
            print(f"  B = {B}, M = {T}: {k:32s} " + " / ".join(f"{x:.0f}" for x in v) + " TFLOP/s", flush=True)


if __name__ == "__main__":
    main()
