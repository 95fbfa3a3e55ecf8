"""Isolated timing of the attention kernels at the ViT-L/16 B=64 shapes of the headline step (CUDA events, 20 launches
after 3 warm-ups, inputs larger than L2): python tools/bench_attention.py [fwd|bwd|all]."""
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch
from dinov3_jax import _native, ops

_native.init(0)
what = sys.argv[1] if len(sys.argv) > 1 else "all"
H, D = 16, 1024
bf = torch.bfloat16


def timeit(fn, n=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3     # us


for name, n, N in (("global 128 crops x 197", 128, 197), ("local 512 crops x 37", 512, 37)):
    T = n * N
    qkv = torch.randn(T, 3 * D, device="cuda").to(bf)
    o = torch.empty(T, D, device="cuda", dtype=bf)
    lse = torch.empty(n, H, N, device="cuda")
    flops = 4.0 * N * N * 64 * n * H
    if what in ("fwd", "all"):
        us = timeit(lambda: ops.attn_fwd(qkv, o, lse, n, N, D, H))
        byt = T * 3 * D * 2 + T * D * 2
        print(f"fwd {name}: {us:8.1f} us  {flops / us / 1e6:7.1f} TFLOP/s  {byt / us / 1e3:7.1f} GB/s (algorithmic qkv in + o out)")
    if what in ("bwd", "all"):
        ops.attn_fwd(qkv, o, lse, n, N, D, H)
        do = torch.randn(T, D, device="cuda").to(bf)
        dqkv = torch.empty(T, 3 * D, device="cuda", dtype=bf)
        delta = torch.empty(n, H, N, device="cuda")
        us = timeit(lambda: ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H))
        byt = T * 3 * D * 2 * 2 + 2 * T * D * 2
        print(f"bwd {name}: {us:8.1f} us  {2.5 * flops / us / 1e6:7.1f} TFLOP/s  {byt / us / 1e3:7.1f} GB/s (qkv + o + do in, dqkv out; includes delta)")
