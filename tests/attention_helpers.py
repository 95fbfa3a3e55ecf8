"""Helpers of the attention tests (test_kernels_gpu.py, test_attention_short_bwd_gpu.py, test_attention_long_gpu.py,
test_attention_hd128_gpu.py): the PyTorch fp32 reference, and the library's forward and backward into buffers of NaN so
that every element the kernels leave unwritten fails the comparison.  head_dim `hd` is 64 or 128; D = hd * H."""
import torch

BF16_TOL = 6e-3      # norm-wise relative error of a bf16-stored result (2^-9 per element)


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def attn_ref(qkv, n, N, H, hd=64):
    """softmax(q k^T / sqrt(hd)) v as [n * N, D] and the natural-log LSE [n, H, N] of the scaled scores, in fp32."""
    q, k, v = qkv.float().reshape(n, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    o = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(n * N, H * hd)
    return o, torch.logsumexp(s, -1)


def fwd(qkv, n, N, H, hd=64):
    from dinov3_jax import ops
    D = hd * H
    o = torch.full((n * N, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    lse = torch.full((n, H, N), float("nan"), device="cuda")
    ops.attn_fwd(qkv, o, lse, n, N, D, H)
    return o, lse


def bwd(qkv, o, do, lse, n, N, H, hd=64, **rope):
    from dinov3_jax import ops
    D = hd * H
    dqkv = torch.full((n * N, 3 * D), float("nan"), device="cuda", dtype=torch.bfloat16)
    ops.attn_bwd(qkv, o, do, lse, torch.zeros(n, H, N, device="cuda"), dqkv, n, N, D, H, **rope)
    return dqkv
