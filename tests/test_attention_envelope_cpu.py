"""The float64 attention reference and element-wise bounds of attention_envelope.py, without a GPU: the backward formula
against float64 autograd (with and without the inverse RoPE), the bound's teeth at the ViT-L/16 step shapes where the
norm-wise check is blind, and the property each input family is named for."""
import pytest
import torch

from attention_envelope import (INPUTS, LSE_LAYOUT, O_LAYOUT, backward, check, early_keys, forward, logits_of,
                                make_inputs, sink_key)
from attention_helpers import BF16_TOL, attn_ref, rel


def _attn64(q, k, v, hd):
    """softmax(q k^T / sqrt(hd)) v on [crop, head, token, column] float64 tensors"""
    return torch.softmax(q @ k.transpose(-1, -2) * hd ** -0.5, -1) @ v


@pytest.mark.parametrize("n,N,H,hd", [(3, 37, 2, 64), (2, 70, 1, 128)])
def test_backward_formula_matches_float64_autograd(n, N, H, hd):
    """With Delta from the exact O, the reference gradients are those of autograd in float64."""
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(n * N, 3 * H * hd, generator=g, dtype=torch.float64) * 1.5
    do = torch.randn(n * N, H * hd, generator=g, dtype=torch.float64)
    x = qkv.clone().requires_grad_(True)
    q, k, v = x.reshape(n, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    o = _attn64(q, k, v, hd).transpose(1, 2).reshape(n * N, H * hd)
    o.backward(do)
    ref = backward(qkv, o.detach(), do, n, N, H, hd)
    want = x.grad.reshape(n, N, 3, H, hd)
    for j, name in enumerate(("dq", "dk", "dv")):
        torch.testing.assert_close(ref[name], want[:, :, j], rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("hd,prefix", [(64, 1), (128, 5)])
def test_backward_inverse_rope_matches_float64_autograd(hd, prefix):
    """The fused inverse RoPE: rotating the reference gradients back equals autograd through oracle.model.rope_apply."""
    from oracle.model import rope_apply, rope_sincos
    n, H, Hp = 2, 2, 4
    N = Hp * Hp + prefix
    sin, cos = rope_sincos(Hp, Hp, hd, 100.0, torch.float32)
    s64, c64 = sin.double(), cos.double()
    g = torch.Generator().manual_seed(2)
    raw = torch.randn(n * N, 3 * H * hd, generator=g, dtype=torch.float64)
    do = torch.randn(n * N, H * hd, generator=g, dtype=torch.float64)
    x = raw.clone().requires_grad_(True)
    q, k, v = x.reshape(n, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    rot = lambda t: torch.cat([t[:, :, :prefix], rope_apply(t[:, :, prefix:], s64, c64)], 2)   # noqa: E731
    q, k = rot(q), rot(k)
    o = _attn64(q, k, v, hd).transpose(1, 2).reshape(n * N, H * hd)
    o.backward(do)
    rotated = torch.cat([t.detach().transpose(1, 2).reshape(n * N, H * hd) for t in (q, k, v)], 1)   # the kernel's qkv
    ref = backward(rotated, o.detach(), do, n, N, H, hd, rope=(sin, cos, prefix))
    want = x.grad.reshape(n, N, 3, H, hd)
    for j, name in enumerate(("dq", "dk", "dv")):
        torch.testing.assert_close(ref[name], want[:, :, j], rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("n,N,H", [(128, 197, 16), (512, 37, 16)])
def test_bound_sees_a_five_percent_slice_the_norm_check_misses(n, N, H):
    """At the ViT-L/16 step shapes the reference rounded to bf16 (the best a kernel can return) uses under half of the
    bound; a 5 % change of one (token, head) slice of O, here the last token of the last crop in the last head, fails
    the element-wise check and passes the norm-wise rel(o, ref) < BF16_TOL of the other attention tests."""
    hd = 64
    qkv = make_inputs("std", n, N, H, hd)
    ref = forward(qkv, n, N, H, hd)
    o = ref["o"].to(torch.bfloat16)
    assert check(o, ref["o"], ref["o_bound"], O_LAYOUT, "O") < 0.5
    assert check(ref["lse"].float(), ref["lse"], ref["lse_bound"], LSE_LAYOUT, "LSE") < 0.5
    bad = o.double()
    bad[n - 1, N - 1, H - 1] *= 1.05
    with pytest.raises(AssertionError, match=f"crop {n - 1}, token {N - 1}, head {H - 1}"):
        check(bad, ref["o"], ref["o_bound"], O_LAYOUT, "O")
    assert rel(bad.reshape(n * N, H * hd), attn_ref(qkv, n, N, H)[0]) < BF16_TOL


def test_check_reports_nan_and_the_worst_element():
    want = torch.ones(2, 3, 1, 4, dtype=torch.float64)
    bound = torch.full_like(want, 0.1)
    got = want.clone()
    got[1, 2, 0, 3] = 1.05
    assert check(got, want, bound, O_LAYOUT) == pytest.approx(0.5)
    got[0, 1, 0, 2] = float("nan")
    with pytest.raises(AssertionError, match="crop 0, token 1, head 0, column 2"):
        check(got, want, bound, O_LAYOUT)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("kind", INPUTS)
def test_input_family_has_its_property(kind, hd):
    """make_inputs asserts each family's property itself; here the properties are restated on small shapes, for packed
    crops (N = 37) and for crops of more than one 128-key tile (N = 300)."""
    for n, N, H in ((4, 37, 2), (2, 300, 1)):
        qkv = make_inputs(kind, n, N, H, hd, seed=3)
        s = logits_of(qkv, n, N, H, hd)                     # [crop, head, query, key], float64
        if kind == "std":
            assert 0.8 < float(s.std()) < 1.2
        elif kind.startswith("peaked"):
            sigma = float(kind[len("peaked"):])
            assert 0.8 * sigma < float(s.std()) < 1.2 * sigma and float(s.abs().max()) > 3 * sigma
        elif kind.startswith("late_"):
            sink = sink_key(kind, N)
            assert bool((s.argmax(-1) == sink).all())
            if kind == "late_last":
                assert sink == N - 1 and (N % 64 != 0)      # in the partial last 64-key block
            if kind == "late_tile" and N > 128:
                assert sink // 128 == (N - 1) // 128 > 0    # a later 128-key tile than the first queries'
            early = early_keys(N)
            early = early[early != sink]
            rest = torch.ones(N, dtype=torch.bool)
            rest[early_keys(N)], rest[sink] = False, False
            assert float((s[..., early].amax(-1) - s[..., rest].amax(-1)).min()) > 10
            assert float((s[..., sink] - s[..., early].amax(-1)).min()) > 10
        elif kind == "shifted":
            base = qkv.clone()
            base.reshape(n * N, 3, H, hd)[:, 1, :, 0] = 0    # k column 0 carries the shift
            assert float(s.min()) > 40
            a, b = forward(qkv, n, N, H, hd), forward(base, n, N, H, hd)
            torch.testing.assert_close(a["o"], b["o"], rtol=1e-12, atol=1e-12)
            shift = a["lse"] - b["lse"]
            assert float(shift.max() - shift.min()) < 1e-9 and 55 < float(shift.mean()) < 65
        elif kind == "uniform":
            p = torch.softmax(s, -1)
            assert bool((p == 1.0 / N).all())
            v = qkv.reshape(n, N, 3, H, hd)[:, :, 2].double()
            torch.testing.assert_close(forward(qkv, n, N, H, hd)["o"], v.mean(1, keepdim=True).expand_as(v),
                                       rtol=1e-12, atol=1e-12)
        elif kind == "bait":
            assert float(s.max()) <= -30
            q = qkv.reshape(n, N, 3, H, hd)[:, :, 0].double().transpose(1, 2)
            k = qkv.reshape(n, N, 3, H, hd)[:, :, 1].double().transpose(1, 2)
            for c in range(n - 1):
                assert float((q[c] @ k[c + 1].transpose(-1, -2)).min()) * hd ** -0.5 >= 30
                assert float((q[c + 1] @ k[c].transpose(-1, -2)).min()) * hd ** -0.5 >= 30


def test_input_families_reject_what_they_are_not():
    """The property checks have teeth: a bait tensor whose crop signs are made equal is refused."""
    from attention_envelope import _assert_property
    n, N, H, hd = 3, 37, 1, 64
    qkv = make_inputs("bait", n, N, H, hd)
    x = qkv.reshape(n, N, 3, H, hd)
    x[1, :, 0, :, 0] *= -1                                   # crop 1's q now agrees in sign with crops 0 and 2
    with pytest.raises(AssertionError, match="bait"):
        _assert_property("bait", qkv, n, N, H, hd)
    with pytest.raises(AssertionError, match="uniform"):
        _assert_property("uniform", make_inputs("std", n, N, H, hd), n, N, H, hd)
