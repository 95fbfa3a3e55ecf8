"""-m gpu: every attention kernel family against the float64 reference of attention_envelope.py, element by element, on
input families that leave the easy regime of randn logits: peaked rows, a running max that jumps late, a large common
shift, exact uniform rows and bait keys outside each row's crop.  Each case prints its worst error / bound ratio."""
import pytest
import torch

from attention_envelope import (INPUTS, LSE_LAYOUT, O_LAYOUT, backward, check, forward, grad_thirds, make_grad,
                                make_inputs)
from attention_helpers import bwd, fwd

pytestmark = pytest.mark.gpu

# resident hd64: span <= 448 forward, <= 256 backward (packed short crops, G = 128 // N, ragged last group); streamed
# hd64 above; hd128 at every span.  N = 257 ... 448 backward: the resident forward's LSE feeds the streamed backward.
FWD_SHAPES = {
    "resident": [(5, 37, 2), (3, 64, 2), (3, 65, 2), (2, 197, 3), (1, 448, 1)],
    "streamed": [(1, 449, 1), (2, 577, 2), (1, 2309, 1)],
    "hd128": [(5, 37, 2), (5, 54, 2), (3, 197, 2), (2, 449, 2), (1, 1029, 2)],
}
BWD_SHAPES = {
    "resident": [(5, 37, 2), (9, 17, 2), (3, 65, 2), (2, 197, 3), (2, 256, 2)],
    "streamed": [(2, 257, 2), (1, 385, 1), (1, 449, 1), (2, 1029, 2)],
    "hd128": FWD_SHAPES["hd128"],
}


def _cases(shapes):
    return [pytest.param(fam, *s, id=f"{fam}-{s[0]}x{s[1]}x{s[2]}") for fam, ss in shapes.items() for s in ss]


def _head_dim(family):
    return 128 if family == "hd128" else 64


def _served_by(family, direction, n, N):
    """the kernel family d3_attn_fwd / d3_attn_bwd pick for this shape (csrc/attention.cu: attn_shape, the dispatch)"""
    if family == "hd128":
        return "hd128"
    span = min(128 // N, n) * N if N <= 64 else N
    return "resident" if span <= (448 if direction == "fwd" else 256) else "streamed"


def _report(family, direction, kind, shape, worst):
    print(f"\nenvelope {family} {direction} {kind} {'x'.join(map(str, shape))} worst err/bound {worst:.3f}")


def run_forward(kind, n, N, H, hd):
    qkv = make_inputs(kind, n, N, H, hd, device="cuda")
    o, lse = fwd(qkv, n, N, H, hd)
    ref = forward(qkv, n, N, H, hd)
    return o.reshape(n, N, H, hd), lse, ref


def forward_worst(kind, n, N, H, hd):
    o, lse, ref = run_forward(kind, n, N, H, hd)
    return max(check(o, ref["o"], ref["o_bound"], O_LAYOUT, "O"),
               check(lse, ref["lse"], ref["lse_bound"], LSE_LAYOUT, "LSE"))


def run_backward(kind, n, N, H, hd, rope=None):
    qkv = make_inputs(kind, n, N, H, hd, device="cuda")
    do = make_grad(n, N, H, hd, device="cuda")
    o, lse = fwd(qkv, n, N, H, hd)
    kw = {} if rope is None else dict(rope_sin=rope[0], rope_cos=rope[1], rope_prefix=rope[2])
    got = grad_thirds(bwd(qkv, o, do, lse, n, N, H, hd, **kw), n, N, H, hd)
    return got, backward(qkv, o, do, n, N, H, hd, rope=rope)


def backward_worst(kind, n, N, H, hd, rope=None):
    got, ref = run_backward(kind, n, N, H, hd, rope)
    return max(check(g, ref[name], ref[name + "_bound"], O_LAYOUT, name) for g, name in zip(got, ("dq", "dk", "dv")))


@pytest.mark.parametrize("kind", INPUTS)
@pytest.mark.parametrize("family,n,N,H", _cases(FWD_SHAPES))
def test_forward_within_envelope(native, family, n, N, H, kind):
    assert _served_by(family, "fwd", n, N) == family
    _report(family, "fwd", kind, (n, N, H), forward_worst(kind, n, N, H, _head_dim(family)))


@pytest.mark.parametrize("kind", INPUTS)
@pytest.mark.parametrize("family,n,N,H", _cases(BWD_SHAPES))
def test_backward_within_envelope(native, family, n, N, H, kind):
    assert _served_by(family, "bwd", n, N) == family
    _report(family, "bwd", kind, (n, N, H), backward_worst(kind, n, N, H, _head_dim(family)))


# the ViT-L/16 step (224^2 global crops of 197 tokens, 96^2 local crops of 37, 16 heads) and vit_7b's 256^2 global crops
@pytest.mark.parametrize("kind", ["std", "peaked4", "peaked16"])
@pytest.mark.parametrize("n,N,H,hd", [(128, 197, 16, 64), (512, 37, 16, 64), (2, 261, 32, 128)])
def test_step_shapes_within_envelope(native, n, N, H, hd, kind):
    family = _served_by("hd128" if hd == 128 else "", "fwd", n, N)
    _report(family, "fwd", kind, (n, N, H), forward_worst(kind, n, N, H, hd))
    family = _served_by("hd128" if hd == 128 else "", "bwd", n, N)
    _report(family, "bwd", kind, (n, N, H), backward_worst(kind, n, N, H, hd))


# N = Hp^2 + prefix: packed 37-token crops, 201 (resident); 405 and 577 (streamed); packed 54, 257 (hd128)
@pytest.mark.parametrize("family,n,Hp,prefix", [("resident", 5, 6, 1), ("resident", 2, 14, 5), ("streamed", 2, 20, 5),
                                                ("streamed", 1, 24, 1), ("hd128", 5, 7, 5), ("hd128", 2, 16, 1)])
def test_backward_fused_inverse_rope_within_envelope(native, family, n, Hp, prefix):
    from oracle.model import rope_sincos
    H, hd = 2, _head_dim(family)
    N = Hp * Hp + prefix
    assert _served_by(family, "bwd", n, N) == family
    sin, cos = [t.cuda().contiguous() for t in rope_sincos(Hp, Hp, hd, 100.0, torch.float32)]
    _report(family, "bwd-rope", "peaked16", (n, N, H), backward_worst("peaked16", n, N, H, hd, (sin, cos, prefix)))


def test_check_rejects_five_percent_on_one_slice_of_kernel_output(native):
    """The bounds have teeth on H100 output: one (token, head) slice of the kernel's O or dK scaled by 1.05 fails."""
    n, N, H, hd = 2, 197, 3, 64
    o, _, ref = run_forward("std", n, N, H, hd)
    assert check(o, ref["o"], ref["o_bound"], O_LAYOUT) <= 1
    bad = o.double()
    bad[1, N - 1, 2] *= 1.05
    with pytest.raises(AssertionError, match=f"crop 1, token {N - 1}, head 2"):
        check(bad, ref["o"], ref["o_bound"], O_LAYOUT)
    (_, dk, _), ref = run_backward("std", n, N, H, hd)
    assert check(dk, ref["dk"], ref["dk_bound"], O_LAYOUT) <= 1
    bad = dk.double()
    bad[0, 100, 1] *= 1.05
    with pytest.raises(AssertionError, match="crop 0, token 100, head 1"):
        check(bad, ref["dk"], ref["dk_bound"], O_LAYOUT)
