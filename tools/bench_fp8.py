"""FP8 block-linear kernels on one H100: e4m3 against bf16 GEMM rates, and the quantizers' bandwidth.

  python tools/bench_fp8.py [--iters 20] [--out FILE]

Prints one JSON line per measurement (and writes them to --out when given; nothing else is written):
  gemm       TFLOP/s of d3_gemm_e4m3 and d3_gemm_bf16 at the ViT-L block shapes (M = 44 160 student tokens, 25 216
             teacher tokens; (K, N) of qkv, proj, fc1, fc2) for the forward (x W) and the input gradient (dy W^T), and at
             7B-width shapes (K = 4096).  Operands are prepared outside the timed window: the GEMM alone.
  quant      GB/s of the quantizers (bytes read + written, from the shapes).
  step       ms per train_step of Engine(fp8=False) and Engine(fp8=True), ViT-L/16 B = 64, alternated `--runs` times
             (`--runs 0` skips it).
Each record carries the card's name, its power limit and its maximum SM clock, read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

from gpu_timing import card, cuda_ms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200"))

RECORDS = []


def emit(rec):
    rec.update(card())
    RECORDS.append(rec)
    print(json.dumps(rec), flush=True)


def bench_gemm(M, K, N, site, iters):
    """x [M, K] times W [K, N] (forward) and dy [M, N] times W^T (input gradient), bf16 against e4m3."""
    from dinov3_jax import ops
    dev = "cuda"
    x = torch.randn(M, K, device=dev).to(torch.bfloat16)
    W = (torch.randn(K, N, device=dev) * K ** -0.5).to(torch.bfloat16)
    dy = torch.randn(M, N, device=dev).to(torch.bfloat16)
    y = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
    dx = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
    u8, f32 = torch.uint8, torch.float32
    qx, sx = ops.quant_rows(x, torch.empty(M, K, dtype=u8, device=dev), torch.empty(M, dtype=f32, device=dev))
    qwt, swt = ops.quant_cols_t(W, torch.empty(N, K, dtype=u8, device=dev), torch.empty(N, dtype=f32, device=dev))
    qdy, sdy = ops.quant_rows(dy, torch.empty(M, N, dtype=u8, device=dev), torch.empty(M, dtype=f32, device=dev))
    qw, sw = ops.quant_rows(W, torch.empty(K, N, dtype=u8, device=dev), torch.empty(K, dtype=f32, device=dev))
    flops = 2.0 * M * N * K
    for kind, bf, f8 in (("forward", lambda: ops.gemm(x, W, y, b_mn=True), lambda: ops.gemm_e4m3(qx, sx, qwt, swt, y)),
                         ("input_grad", lambda: ops.gemm(dy, W, dx), lambda: ops.gemm_e4m3(qdy, sdy, qw, sw, dx))):
        t_bf, t_f8 = cuda_ms(bf, iters, 1), cuda_ms(f8, iters, 1)
        emit({"what": "gemm", "site": site, "kind": kind, "M": M, "K": K if kind == "forward" else N,
              "N": N if kind == "forward" else K, "bf16_tflops": round(flops / t_bf / 1e9, 1),
              "e4m3_tflops": round(flops / t_f8 / 1e9, 1), "bf16_ms": round(t_bf, 4), "e4m3_ms": round(t_f8, 4)})
    del x, W, dy, y, dx, qx, qwt, qdy, qw


def bench_quant(iters):
    from dinov3_jax import ops
    u8, f32, dev = torch.uint8, torch.float32, "cuda"
    for R, C in ((44160, 1024), (44160, 4096)):
        x = torch.randn(R, C, device=dev).to(torch.bfloat16)
        q, s = torch.empty(R, C, dtype=u8, device=dev), torch.empty(R, dtype=f32, device=dev)
        t = cuda_ms(lambda: ops.quant_rows(x, q, s), iters, 1)
        emit({"what": "quant", "kernel": "quant_rows", "R": R, "C": C, "ms": round(t, 4),
              "GB/s": round(R * C * 3 / t / 1e6, 1)})
    for R, C in ((1024, 4096), (4096, 1024), (4096, 12288)):
        W = torch.randn(R, C, device=dev).to(torch.bfloat16)
        q, s = torch.empty(C, R, dtype=u8, device=dev), torch.empty(C, dtype=f32, device=dev)
        t = cuda_ms(lambda: ops.quant_cols_t(W, q, s), iters, 1)
        emit({"what": "quant", "kernel": "quant_cols_t", "R": R, "C": C, "ms": round(t, 4),
              "GB/s": round(R * C * 3 / t / 1e6, 1)})


def bench_step(fp8, steps, warmup):
    sys.path.insert(0, ROOT)
    from bench import hyper
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import init_reference_like, synthetic_batch
    cfg = config_for("vit_large", n_prototypes=65536, patch=16, local_size=96)
    B = 64
    batch = synthetic_batch(cfg, B, seed=0, pin=True)
    eng = Engine(cfg, B, max_masked=int(batch["mask_indices_list"].shape[0]), fp8=fp8)
    init_reference_like(eng, seed=0)
    eng.train_step(batch, **hyper(0))
    for i in range(warmup):
        eng.train_step(None, **hyper(i))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        eng.train_step(None, **hyper(i))
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    emit({"what": "step", "fp8": fp8, "arch": "vit_large", "B": B, "ms_per_step": round(ms, 2),
          "total_loss": eng.read_metrics()["total_loss"], "peak_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)})
    del eng, batch
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="GEMM / quantizer launches per timing")
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8.py: no CUDA device")
    from dinov3_jax import _native
    _native.init()
    for M, who in ((44160, "student"), (25216, "teacher")):
        for (K, N), site in (((1024, 3072), "qkv"), ((1024, 1024), "proj"), ((1024, 4096), "fc1"), ((4096, 1024), "fc2")):
            bench_gemm(M, K, N, f"vitl_{who}_{site}", args.iters)
    for (K, N), site in (((4096, 12288), "qkv"), ((4096, 4096), "proj"), ((4096, 8192), "w1"), ((8192, 4096), "w3")):
        bench_gemm(25216, K, N, f"7b_width_{site}", args.iters)
    torch.cuda.empty_cache()
    bench_quant(args.iters)
    for _ in range(args.runs):
        for fp8 in (False, True):
            bench_step(fp8, args.steps, args.warmup)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in RECORDS) + "\n")


if __name__ == "__main__":
    main()
