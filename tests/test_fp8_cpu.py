"""The FP8 block-linear arithmetic (tests/fp8_oracle.py) against its written definition, and the configuration keys that
select it.  No GPU."""
import numpy as np
import pytest
import torch

from fp8_oracle import E4M3, Fp8Linear, block_forward_fp8, dequant, fp8_matmul, quant_rows, row_scale


def _e4m3_table():
    """Every finite non-negative e4m3fn value by its code 0..126: subnormals m 2^-9, normals (1 + m/8) 2^(e-7)."""
    v = []
    for code in range(127):
        e, m = code >> 3, code & 7
        v.append(m * 2.0 ** -9 if e == 0 else (1 + m / 8) * 2.0 ** (e - 7))
    return np.array(v)


def _rne_e4m3(x: np.ndarray) -> np.ndarray:
    """Round to the nearest e4m3 value, ties to the even code, by search over the table (no torch involved)."""
    t = _e4m3_table()
    a = np.abs(x)
    d = np.abs(a[:, None] - t[None, :])
    best = d.min(axis=1, keepdims=True)
    cand = d == best
    codes = np.where(cand.sum(axis=1) > 1, np.argmax(cand & (np.arange(127) % 2 == 0)[None, :], axis=1),
                     np.argmax(cand, axis=1))
    return np.sign(x) * t[codes]


def test_quantizer_matches_round_to_nearest_even_over_the_bf16_range():
    g = torch.Generator().manual_seed(0)
    rows = []
    for e in range(-133, 128, 7):                 # row maxima across the whole bf16 range, subnormals included
        r = torch.randn(64, generator=g, dtype=torch.float64) * 2.0 ** e
        rows.append(r)
    x = torch.stack(rows).to(torch.bfloat16)
    q, s = quant_rows(x)
    a = x.float().abs().amax(1)
    assert torch.all(s == torch.ldexp(torch.ones_like(s), torch.frexp(s)[1] - 1))          # powers of two
    assert torch.all(a / s <= 448) and torch.all(a / s > 224)                             # the smallest such power
    want = _rne_e4m3((x.double() / s.double()[:, None]).numpy().reshape(-1))
    got = q.view(E4M3).double().numpy().reshape(-1)
    np.testing.assert_array_equal(got, want)


def test_quantizer_edge_cases():
    bf = torch.bfloat16
    # amax exactly 448 * 2^e keeps 2^e (and quantizes to 448); one bf16 ulp more takes 2^(e+1)
    x = torch.tensor([[448.0 * 2 ** -3, 1.0], [448.0 * 2 ** -3 * (1 + 2 ** -7), 1.0]], dtype=bf)
    q, s = quant_rows(x)
    assert s.tolist() == [2.0 ** -3, 2.0 ** -2]
    assert q[0, 0].item() == 0x7E
    # zero row: scale 1, zero bytes
    q, s = quant_rows(torch.zeros(2, 16, dtype=bf))
    assert s.tolist() == [1.0, 1.0] and int(q.sum()) == 0
    # ties to even at scale 1: 1.0625 -> 1.0, 1.1875 -> 1.25; subnormals 2^-9 -> code 1, 3 * 2^-10 -> 2^-8 (code 2)
    x = torch.tensor([[448.0, 1.0625, 1.1875, 2.0 ** -9, 3 * 2.0 ** -10, -2.0 ** -10]], dtype=bf)
    q, s = quant_rows(x)
    assert s.item() == 1.0
    assert q.view(E4M3).float()[0].tolist() == [448.0, 1.0, 1.25, 2.0 ** -9, 2.0 ** -8, -0.0]
    assert q[0, 3].item() == 1 and q[0, 4].item() == 2
    # non-finite elements do not set the scale and stay non-finite
    x = torch.tensor([[float("inf"), 3.0, float("nan")]], dtype=bf)
    q, s = quant_rows(x)
    assert s.item() == 2.0 ** -7
    assert torch.isnan(q.view(E4M3).float()[0, [0, 2]]).all() and q.view(E4M3).float()[0, 1].item() == 3.0 / 2 ** -7
    assert row_scale(torch.zeros(1, 3)).item() == 1.0


def test_linear_gradients_follow_the_definition():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(6, 48, generator=g, dtype=torch.float64, requires_grad=True)
    W = (torch.randn(48, 32, generator=g, dtype=torch.float64) * 0.1).requires_grad_(True)
    dy = torch.randn(6, 32, generator=g, dtype=torch.float64)
    y = Fp8Linear.apply(x, W)
    torch.testing.assert_close(y, dequant(*quant_rows(x)) @ dequant(*quant_rows(W.T)).T, rtol=0, atol=0)
    y.backward(dy)
    # dx from the row-quantized dy and the row-quantized W (per input row)
    qd, sd = quant_rows(dy)
    qw, sw = quant_rows(W)
    torch.testing.assert_close(x.grad, dequant(qd, sd) @ dequant(qw, sw).T, rtol=0, atol=0)
    # dW from the bf16 operands
    bf = lambda t: t.detach().to(torch.bfloat16).double()
    torch.testing.assert_close(W.grad, bf(x).T @ bf(dy), rtol=0, atol=0)
    # the FP8 product is not the bf16 one (the test would not see a bf16 fall-back otherwise)
    assert float((y.detach() - bf(x) @ bf(W)).abs().max()) > 1e-3


def test_layerscale_gradient_is_that_of_the_fp8_output():
    """x_mid = x + g1 * (o Wp + bp): dg1 = colsum(dx_mid * p) with p the FP8 product, not the bf16 identity."""
    g = torch.Generator().manual_seed(2)
    o = torch.randn(10, 32, generator=g, dtype=torch.float64)
    Wp = torch.randn(32, 32, generator=g, dtype=torch.float64) * 0.2
    bp = torch.randn(32, generator=g, dtype=torch.float64) * 0.1
    g1 = (torch.rand(32, generator=g, dtype=torch.float64) + 0.5).requires_grad_(True)
    dxm = torch.randn(10, 32, generator=g, dtype=torch.float64)
    p = Fp8Linear.apply(o, Wp) + bp
    (g1 * p).backward(dxm)
    torch.testing.assert_close(g1.grad, (dxm * (fp8_matmul(o, Wp.T) + bp)).sum(0), rtol=1e-12, atol=0)
    assert float((g1.grad - (dxm * (o @ Wp + bp)).sum(0)).abs().max()) > 1e-3


def test_block_forward_fp8_matches_the_bf16_block_within_fp8_error():
    from oracle import tiny_cfg
    from oracle.model import Emu, block_forward, init_params, rope_sincos, sub
    cfg = tiny_cfg()
    P = sub(init_params(cfg, 0, dtype=torch.float64, perturb=0.05), "student_backbone")
    x = torch.randn(2, cfg.prefix + 16, cfg.embed_dim, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    sin, cos = rope_sincos(4, 4, cfg.head_dim, cfg.rope_base, torch.float64)
    a = block_forward(P, "blocks_0/", x, sin, cos, cfg, Emu(False))
    b = block_forward_fp8(P, "blocks_0/", x, sin, cos, cfg, Emu(False))
    e = float((a - b).norm() / (a - x).norm())
    assert 1e-4 < e < 0.1, e


@pytest.mark.parametrize("cfg_kw", [{}, dict(embed_dim=256, heads=2, ffn_layer="swiglu", swiglu_align=64, n_storage=4,
                                             mask_k_bias=True, mlp_second_act=False)])
def test_block_forward_fp8_is_the_oracle_block_with_its_linears_swapped(cfg_kw):
    """With the plain linear, block_forward_fp8 gives oracle.model.block_forward's bits, forward and backward."""
    from oracle import tiny_cfg
    from oracle.model import Emu, block_forward, init_params, rope_sincos, sub
    cfg = tiny_cfg(**cfg_kw)
    P = sub(init_params(cfg, 0, perturb=0.05), "student_backbone")
    sin, cos = rope_sincos(4, 4, cfg.head_dim, cfg.rope_base, torch.float32)
    for emu in (Emu(False), Emu(True)):
        outs = []
        for fwd in (block_forward, lambda *a: block_forward_fp8(*a, lin=lambda x, W: x @ emu.w(W))):
            Q = {k: v.clone().requires_grad_(True) for k, v in P.items()}
            x = torch.randn(2, cfg.prefix + 16, cfg.embed_dim, generator=torch.Generator().manual_seed(3))
            y = fwd(Q, "blocks_0/", x, sin, cos, cfg, emu)
            keys = [k for k in Q if k.startswith("blocks_0/")]
            gs = torch.autograd.grad(y.square().sum(), [Q[k] for k in keys], allow_unused=True)
            outs.append((y.detach(), gs))
        assert torch.equal(outs[0][0], outs[1][0])
        for a, b in zip(outs[0][1], outs[1][1]):
            assert (a is None and b is None) or torch.equal(a, b)


@pytest.mark.parametrize("flt", ["", "mlp", "attn", "blocks.0"])
def test_fp8_filters_other_than_blocks_raise(flt):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train.ssl_meta_arch import SSLMetaArch, fp8_from_config
    cfg = setup_config(DinoV3SetupArgs(opts=["student.fp8_enabled=true", f"student.fp8_filter={flt}"]))
    with pytest.raises(NotImplementedError, match="blocks"):
        fp8_from_config(cfg)
    with pytest.raises(NotImplementedError, match="blocks"):
        SSLMetaArch(cfg)


def test_fp8_keys_are_read_and_default_off():
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train.ssl_meta_arch import SSLMetaArch, fp8_from_config
    assert fp8_from_config(setup_config(DinoV3SetupArgs(opts=[]))) is False
    assert fp8_from_config(setup_config(DinoV3SetupArgs(opts=["student.fp8_filter=mlp"]))) is False
    cfg = setup_config(DinoV3SetupArgs(opts=["student.fp8_enabled=true"]))
    assert fp8_from_config(cfg) is True and SSLMetaArch(cfg).fp8 is True


def test_fp8_refuses_contractions_that_are_not_multiples_of_16():
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    with pytest.raises(NotImplementedError, match="multiples of 16"):
        Engine(from_oracle_cfg(tiny_cfg(ffn_ratio=4.0625)), 2, max_masked=4, fp8=True)
