"""Isolated timing of the head_dim 128 attention kernels at the vit_7b shapes (32 heads): 256^2 global crops (261 tokens
with 4 storage tokens), 112^2 local crops (54 tokens, packed two per 128-row tile), and the 512^2 / 768^2 crops of the
Gram-anchoring / high-resolution recipes (1 029 / 2 309 tokens), B = 8 images.  Next to each row,
torch.nn.functional.scaled_dot_product_attention (bf16, [n, H, N, 128], PyTorch's own backend choice) at the same shape,
for context.  CUDA events, 20 launches after 3 warm-ups; prints the card name and power limit read in the same run.
usage: python tools/bench_attention_hd128.py"""
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F
from dinov3_jax import _native, ops

HD, H = 128, 32
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


def main():
    _native.init(0)
    print(card())
    shapes = (("global 256^2, 16 crops x 261", 16, 261), ("local 112^2, 64 crops x 54", 64, 54),
              ("gram 512^2, 16 crops x 1029", 16, 1029), ("hi-res 768^2, 16 crops x 2309", 16, 2309))
    for name, n, N in shapes:
        D, T = HD * H, n * N
        qkv = torch.randn(T, 3 * D, device="cuda").to(bf)
        o = torch.empty(T, D, device="cuda", dtype=bf)
        lse = torch.empty(n, H, N, device="cuda")
        do = torch.randn(T, D, device="cuda").to(bf)
        dqkv = torch.empty(T, 3 * D, device="cuda", dtype=bf)
        delta = torch.empty(n, H, N, device="cuda")
        flops = 4.0 * N * N * HD * n * H
        f_us = timeit(lambda: ops.attn_fwd(qkv, o, lse, n, N, D, H))
        ops.attn_fwd(qkv, o, lse, n, N, D, H)
        b_us = timeit(lambda: ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H))
        q, k, v = [t.contiguous().requires_grad_(True) for t in qkv.view(n, N, 3, H, HD).permute(2, 0, 3, 1, 4)]
        g = do.view(n, N, H, HD).transpose(1, 2).contiguous()
        sf_us = timeit(lambda: F.scaled_dot_product_attention(q, k, v))
        sfb_us = timeit(lambda: torch.autograd.grad(F.scaled_dot_product_attention(q, k, v), (q, k, v), g)) - sf_us
        print(f"{name}: fwd {f_us:8.1f} us {flops / f_us / 1e6:6.1f} TFLOP/s (sdpa {sf_us:8.1f} us "
              f"{flops / sf_us / 1e6:6.1f}) | bwd {b_us:8.1f} us {2.5 * flops / b_us / 1e6:6.1f} TFLOP/s, incl. delta "
              f"(sdpa {sfb_us:8.1f} us {2.5 * flops / sfb_us / 1e6:6.1f})", flush=True)
        del qkv, o, lse, do, dqkv, delta, q, k, v, g
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
