"""The FP8 block-linear arithmetic of d3_quant_rows_e4m3 / d3_quant_cols_e4m3_t / d3_gemm_e4m3, written out for the CPU
oracle.

Row-wise e4m3 with a high-precision weight gradient:
  quantize   q = e4m3(x / s) per row of a bf16 matrix, s = 2^e with e the smallest integer such that the row's largest
             finite magnitude is <= 448 * 2^e (s = 1 for a row of zeros); round to nearest even (torch's conversion).
  forward    y = x W: x per token row, W per output column; y = sum_k qx qw * s_x[m] * s_w[n] (float64 here).
  dx         dy W^T: the bf16 dy per token row, W per input row.
  dW         x^T dy on the bf16 operands, unchanged.
`block_forward_fp8` is oracle.model.block_forward with these linears at the block sites (qkv, proj, fc1 / fc2 or
w1 / w2 / w3), and `fp8_oracle()` makes every oracle backbone use it; the patch embedding, the heads and attention stay
as they are.
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

E4M3 = torch.float8_e4m3fn


def row_scale(x: torch.Tensor) -> torch.Tensor:
    """float32 [R] power-of-two scales of the rows of a 2-D tensor."""
    xf = x.float()
    a = torch.where(torch.isfinite(xf), xf.abs(), torch.zeros_like(xf)).amax(dim=1)
    m, E = torch.frexp(a)                       # a = m 2^E, m in [0.5, 1); 448 = 0.875 * 2^9
    e = torch.where(m <= 0.875, E - 9, E - 8)
    s = torch.ldexp(torch.ones_like(a), e)
    return torch.where(a > 0, s, torch.ones_like(a))


def quant_rows(x: torch.Tensor):
    """(e4m3 bytes as uint8 [R, C], float32 scales [R]) of the bf16 values of x."""
    xb = x.detach().to(torch.bfloat16).float()
    s = row_scale(xb)
    return (xb / s[:, None]).to(E4M3).view(torch.uint8), s


def dequant(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """float64 q * s, row-wise."""
    return q.view(E4M3).double() * s.double()[:, None]


def fp8_matmul(a: torch.Tensor, bt: torch.Tensor) -> torch.Tensor:
    """float64 a bt^T with both operands quantized per row (bt: the [N, K] operand)."""
    return dequant(*quant_rows(a)) @ dequant(*quant_rows(bt)).T


class Fp8Linear(torch.autograd.Function):
    """y = x W (W [in, out]) in the FP8 arithmetic above, for x of any leading shape."""

    @staticmethod
    def forward(ctx, x, W):
        ctx.save_for_backward(x, W)
        x2 = x.reshape(-1, x.shape[-1])
        return fp8_matmul(x2, W.T).to(x.dtype).reshape(*x.shape[:-1], W.shape[1])

    @staticmethod
    def backward(ctx, dy):
        x, W = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        dx = fp8_matmul(dy2, W).to(x.dtype).reshape(x.shape)
        bf = lambda t: t.to(torch.bfloat16).double()
        dW = (bf(x.reshape(-1, x.shape[-1])).T @ bf(dy2)).to(W.dtype)
        return dx, dW


def block_forward_fp8(P: dict, b: str, x, sin, cos, cfg, emu, lin=Fp8Linear.apply):
    """oracle.model.block_forward with the block linears y = lin(x, W).  With lin(x, W) = x @ emu.w(W) it is
    oracle.model.block_forward bit for bit (tests/test_fp8_cpu.py pins that, so the two cannot drift apart)."""
    from oracle.model import attention, gelu, layer_norm
    y = emu.act(layer_norm(x, P[b + "norm1/scale"], P[b + "norm1/bias"], cfg.ln_eps))
    qkv_bias = P[b + "attn/qkv/bias"]
    if cfg.mask_k_bias:
        D_ = qkv_bias.shape[0] // 3
        qkv_bias = torch.cat([qkv_bias[:D_], torch.zeros_like(qkv_bias[D_:2 * D_]), qkv_bias[2 * D_:]])
    qkv = emu.act(lin(y, P[b + "attn/qkv/kernel"]) + qkv_bias)
    o = emu.act(attention(qkv, cfg.heads, sin, cos, emu))
    p = lin(o, P[b + "attn/proj/kernel"]) + P[b + "attn/proj/bias"]
    x = x + P[b + "ls1/gamma"] * emu.grad(p)
    z = emu.act(layer_norm(x, P[b + "norm2/scale"], P[b + "norm2/bias"], cfg.ln_eps))
    if cfg.ffn_layer == "swiglu":
        x1 = emu.grad(lin(z, P[b + "mlp/w1/kernel"]) + P[b + "mlp/w1/bias"])
        x2 = emu.grad(lin(z, P[b + "mlp/w2/kernel"]) + P[b + "mlp/w2/bias"])
        h = emu.act(F.silu(x1) * x2)
        m = emu.grad(lin(h, P[b + "mlp/w3/kernel"]) + P[b + "mlp/w3/bias"])
        return x + P[b + "ls2/gamma"] * m
    u1 = emu.grad(lin(z, P[b + "mlp/Dense_0/kernel"]) + P[b + "mlp/Dense_0/bias"])
    h = emu.act(gelu(u1))
    u2 = emu.grad(lin(h, P[b + "mlp/Dense_1/kernel"]) + P[b + "mlp/Dense_1/bias"])
    m = gelu(u2) if cfg.mlp_second_act else u2
    return x + P[b + "ls2/gamma"] * m



@contextlib.contextmanager
def fp8_oracle():
    """Every backbone the oracle runs (student, EMA / gram / distillation teachers) uses the FP8 block linears."""
    import oracle.model as om
    saved = om.block_forward
    om.block_forward = block_forward_fp8
    try:
        yield
    finally:
        om.block_forward = saved
