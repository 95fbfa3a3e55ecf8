"""Isolated timing of the attention kernels at the ViT-L/16 B=64 shapes of the headline step, the ViT-g/16 global crops
(257 tokens, 24 heads), then the long crops of the high-resolution recipes (streamed kernels) at ViT-L heads (CUDA
events, 20 launches after 3 warm-ups, inputs larger than L2): python tools/bench_attention.py [fwd|bwd|all]."""
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch
from dinov3_jax import _native, ops

_native.init(0)
what = sys.argv[1] if len(sys.argv) > 1 else "all"
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


def card():
    """Card name and power limit, read in the same run as the numbers they belong to."""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or f"{torch.cuda.get_device_name(0)}, power limit not read"


print(card())
SHORT = (("global 128 crops x 197", 128, 197, 16, True), ("local 512 crops x 37", 512, 37, 16, True),
         ("ViT-g global 128 crops x 257", 128, 257, 24, True))
LONG = (("512^2 16 crops x 1029", 16, 1029, 16, True), ("768^2 16 crops x 2309", 16, 2309, 16, True),
        ("gram 1152^2 8 crops x 5189", 8, 5189, 16, False))        # B = 8 global crops, 4 storage tokens
for name, n, N, H, with_bwd in SHORT + LONG:
    D = 64 * H
    T = n * N
    qkv = torch.randn(T, 3 * D, device="cuda").to(bf)
    o = torch.empty(T, D, device="cuda", dtype=bf)
    lse = torch.empty(n, H, N, device="cuda")
    flops = 4.0 * N * N * 64 * n * H
    if what in ("fwd", "all"):
        us = timeit(lambda: ops.attn_fwd(qkv, o, lse, n, N, D, H))
        byt = T * 3 * D * 2 + T * D * 2
        print(f"fwd {name}: {us:8.1f} us  {flops / us / 1e6:7.1f} TFLOP/s  {byt / us / 1e3:7.1f} GB/s (algorithmic qkv in + o out)")
    if what in ("bwd", "all") and with_bwd:
        ops.attn_fwd(qkv, o, lse, n, N, D, H)
        do = torch.randn(T, D, device="cuda").to(bf)
        dqkv = torch.empty(T, 3 * D, device="cuda", dtype=bf)
        delta = torch.empty(n, H, N, device="cuda")
        us = timeit(lambda: ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H))
        byt = T * 3 * D * 2 * 2 + 2 * T * D * 2
        print(f"bwd {name}: {us:8.1f} us  {2.5 * flops / us / 1e6:7.1f} TFLOP/s  {byt / us / 1e3:7.1f} GB/s (qkv + o + do in, dqkv out; includes delta)")
