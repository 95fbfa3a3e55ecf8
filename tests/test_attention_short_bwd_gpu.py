"""-m gpu: the one-pass attention backward for crop groups of span <= 256 (attn_bwd_fused_kernel) against PyTorch fp32
autograd: the ViT-L/16 step shapes, every edge of the 64- and 128-row tiling, ragged last crop groups of packed short
crops, the fused inverse RoPE with 5 prefix tokens, and bit-identical repeats (dQ is summed in a fixed order)."""
import pytest
import torch

from attention_helpers import BF16_TOL, attn_ref, bwd, fwd, rel

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _seed(native):
    torch.manual_seed(0)


def fwd_bwd(qkv, do, n, N, H, **rope):
    o, lse = fwd(qkv, n, N, H)
    return bwd(qkv, o, do, lse, n, N, H, **rope)


def check_against_autograd(n, N, H):
    D = 64 * H
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    x = qkv.float().requires_grad_(True)
    attn_ref(x, n, N, H)[0].backward(do.float())
    dqkv = fwd_bwd(qkv, do, n, N, H)
    if N == 1:    # softmax over one key: the q and k gradients are 0, only the bf16 rounding of O and dO remains
        assert dqkv[:, :2 * D].float().abs().max().item() < 1e-3
        assert rel(dqkv[:, 2 * D:], x.grad[:, 2 * D:]) < 1e-2
        return
    for j in range(3):
        assert rel(dqkv[:, j * D:(j + 1) * D], x.grad[:, j * D:(j + 1) * D]) < 1e-2, "qkv"[j]


# the ViT-L/16 B = 64 step: 128 global crops of 197 tokens, 512 local crops of 37 tokens packed 3 per group
@pytest.mark.parametrize("n,N", [(128, 197), (512, 37)])
def test_vit_large_shapes(n, N):
    check_against_autograd(n, N, 16)


# spans across the 64-key halves and the 128-row tiles; N <= 64 packs G = 128 // N crops per group
@pytest.mark.parametrize("n,N,H", [(1, 1, 1), (3, 17, 2), (2, 64, 1), (3, 65, 2), (2, 128, 1), (2, 129, 1),
                                   (2, 200, 3), (2, 256, 2)])
def test_edge_spans(n, N, H):
    check_against_autograd(n, N, H)


# the last crop group holds fewer crops than the others (200 = 128 + 72, 9 = 7 + 2, 5 = 3 + 2)
@pytest.mark.parametrize("n,N", [(200, 1), (9, 17), (5, 37)])
def test_ragged_last_crop_group(n, N):
    check_against_autograd(n, N, 2)


@pytest.mark.parametrize("Hp", [4, 8, 15])
def test_fused_inverse_rope_with_prefix_tokens(Hp):
    """dqkv with rope tables == separate inverse RoPE of the plain backward, 5 prefix tokens (cls + 4 storage tokens):
    21 tokens (packed 6 per group), 69 and 230 tokens."""
    from dinov3_jax import ops
    from oracle.model import rope_sincos
    n, H, prefix = 7, 2, 5
    N, D = Hp * Hp + prefix, 64 * H
    sin, cos = [t.cuda().contiguous() for t in rope_sincos(Hp, Hp, 64, 100.0, torch.float32)]
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    d1 = fwd_bwd(qkv, do, n, N, H)
    ops.rope(d1, sin, cos, N, prefix, D, 64, inverse=True)
    d2 = fwd_bwd(qkv, do, n, N, H, rope_sin=sin, rope_cos=cos, rope_prefix=prefix)
    assert rel(d2, d1) < BF16_TOL          # d1 is rounded to bf16 twice, d2 once
    assert torch.equal(d2[:, 2 * D:], d1[:, 2 * D:])


@pytest.mark.parametrize("n,N", [(128, 197), (512, 37)])
def test_two_calls_give_identical_bits(n, N):
    from dinov3_jax import ops
    H = 16
    D = 64 * H
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    o = torch.empty(n * N, D, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(n, H, N, device="cuda")
    ops.attn_fwd(qkv, o, lse, n, N, D, H)
    delta = torch.zeros(n, H, N, device="cuda")
    d1 = torch.empty(n * N, 3 * D, device="cuda", dtype=torch.bfloat16)
    d2 = torch.full_like(d1, float("nan"))
    ops.attn_bwd(qkv, o, do, lse, delta, d1, n, N, D, H)
    ops.attn_bwd(qkv, o, do, lse, delta, d2, n, N, D, H)
    assert torch.equal(d1, d2)
