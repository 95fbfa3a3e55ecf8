"""Isolated timing of the attention kernels (CUDA events, 20 launches after 3 warm-ups, inputs larger than L2):
python tools/bench_attention.py [fwd|bwd|all|hd128].

fwd / bwd / all: head_dim 64 at the ViT-L/16 B=64 shapes of the headline step, the ViT-g/16 global crops (257 tokens,
24 heads), then the long crops of the high-resolution recipes (streamed kernels) at ViT-L heads.

hd128: head_dim 128 at the vit_7b shapes (32 heads): 256^2 global crops (261 tokens with 4 storage tokens), 112^2 local
crops (54 tokens, packed two per 128-row tile), and the 512^2 / 768^2 crops of the Gram-anchoring / high-resolution
recipes (1 029 / 2 309 tokens), B = 8 images.  Next to each row, torch.nn.functional.scaled_dot_product_attention (bf16,
[n, H, N, 128], PyTorch's own backend choice) at the same shape, for context."""
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F
from dinov3_jax import _native, ops

from gpu_timing import card, cuda_ms

bf = torch.bfloat16


def us(fn):
    return cuda_ms(fn, 20, 3) * 1e3


def head_dim_64(what):
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
            t = us(lambda: ops.attn_fwd(qkv, o, lse, n, N, D, H))
            byt = T * 3 * D * 2 + T * D * 2
            print(f"fwd {name}: {t:8.1f} us  {flops / t / 1e6:7.1f} TFLOP/s  {byt / t / 1e3:7.1f} GB/s (algorithmic qkv in + o out)")
        if what in ("bwd", "all") and with_bwd:
            ops.attn_fwd(qkv, o, lse, n, N, D, H)
            do = torch.randn(T, D, device="cuda").to(bf)
            dqkv = torch.empty(T, 3 * D, device="cuda", dtype=bf)
            delta = torch.empty(n, H, N, device="cuda")
            t = us(lambda: ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H))
            byt = T * 3 * D * 2 * 2 + 2 * T * D * 2
            print(f"bwd {name}: {t:8.1f} us  {2.5 * flops / t / 1e6:7.1f} TFLOP/s  {byt / t / 1e3:7.1f} GB/s (qkv + o + do in, dqkv out; includes delta)")


def head_dim_128():
    HD, H = 128, 32
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
        f_us = us(lambda: ops.attn_fwd(qkv, o, lse, n, N, D, H))
        ops.attn_fwd(qkv, o, lse, n, N, D, H)
        b_us = us(lambda: ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H))
        q, k, v = [t.contiguous().requires_grad_(True) for t in qkv.view(n, N, 3, H, HD).permute(2, 0, 3, 1, 4)]
        g = do.view(n, N, H, HD).transpose(1, 2).contiguous()
        sf_us = us(lambda: F.scaled_dot_product_attention(q, k, v))
        sfb_us = us(lambda: torch.autograd.grad(F.scaled_dot_product_attention(q, k, v), (q, k, v), g)) - sf_us
        print(f"{name}: fwd {f_us:8.1f} us {flops / f_us / 1e6:6.1f} TFLOP/s (sdpa {sf_us:8.1f} us "
              f"{flops / sf_us / 1e6:6.1f}) | bwd {b_us:8.1f} us {2.5 * flops / b_us / 1e6:6.1f} TFLOP/s, incl. delta "
              f"(sdpa {sfb_us:8.1f} us {2.5 * flops / sfb_us / 1e6:6.1f})", flush=True)
        del qkv, o, lse, do, dqkv, delta, q, k, v, g
        torch.cuda.empty_cache()


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what not in ("fwd", "bwd", "all", "hd128"):
        raise SystemExit(__doc__)
    _native.init(0)
    print(card())
    if what == "hd128":
        head_dim_128()
    else:
        head_dim_64(what)
