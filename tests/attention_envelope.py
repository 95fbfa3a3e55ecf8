"""Float64 reference of the attention kernels, element-wise error bounds for their bf16 / fp32 results, and seeded input
families that push the online softmax and the crop masks out of the easy regime of `torch.randn` logits.

Reference.  `forward` gives O* = softmax(q k^T / sqrt(hd)) v, the natural-log LSE* of the scaled scores and the envelope
A = P* |v|.  `backward` gives dV* = P*^T dO, dK* = dS*^T q, dQ* = dS* k with dP* = dO v^T, Delta = rowsum(dO o O) and
dS* = P* o (dP* - Delta) * scale, where P* is the float64 softmax of the bf16 q and k and Delta uses the bf16 O the kernel
was given (the op's input, and what attn_delta_kernel reads): the cancellation of Delta against dP that a rounded O brings
is a property of the algorithm, not of a kernel.  Everything is computed in float64 on the inputs' device.

Bounds, with u = 2^-9 (unit roundoff of bf16, round to nearest) and C = 4:
    |O  - O* | <= C u (P*|v|                              + |O* |)
    |dV - dV*| <= C u (P*^T |dO|                          + |dV*|)
    |dK - dK*| <= C u (scale |P* o (|dP*| + |Delta|)|^T |q| + |dK*|)
    |dQ - dQ*| <= C u (scale |P* o (|dP*| + |Delta|)| |k|   + |dQ*|)
The kernels round in three places: P (forward) and dS (backward) to bf16 as the A operands of the tensor-core products,
one relative u per element, which the envelope term bounds after the fp32 sum; and the result on its store to bf16,
u |X*|.  That is 1 u of each term.  Everything else is far below u: the row sum l is accumulated from the unrounded p,
so it adds no bf16 rounding; S and dP are fp32 sums of exact bf16 products (relative error at most hd 2^-24 of
scale sum_d |q_d k_d|); ex2.approx has a relative error of about 2^-22; the fp32 sums over at most a few thousand keys
add N 2^-24 <= 0.1 u; and the LSE that the backward's P is rebuilt from is within the LSE bound below, which is a few
times 2^-24 of |lse|.  For scaled logits up to about +-100 these stay below 0.3 u together.  C = 4 so covers the
first-order 2 u with a factor of two for those terms, while a 5 % change of one (token, head) slice of O exceeds it
several times at the ViT step shapes (tests/test_attention_envelope_cpu.py).  Results below 2^-126 may be flushed to
zero (ex2.approx.ftz): TINY absorbs them.

LSE: |lse - lse*| <= eps (1 + |lse*|), eps = 2^-24 (N + 2 hd + 32).  The fp32 sum of l over N keys contributes N 2^-24
(absolute, after the log); ex2.approx 4 2^-24; the rounding of m * scale, of the exponent argument and of the final sum
a few 2^-24 |lse*|; the fp32 accumulation of S at most hd 2^-24 scale sum_d |q_d k_d|, which for the input families
here (the bias column of `make_inputs` included) is below 2 hd 2^-24 (1 + |lse*|).

The fused inverse RoPE of the backward rotates each pair (d, d + hd/2) of dQ / dK; the reference rotates the float64
gradients the same way (oracle.model.rope_apply with -sin: its transpose, the two halves of the tables being equal) and
the bounds by the absolute rotation |cos| b_d + |sin| b_{d +- hd/2}, at most sqrt(2) max(b_d, b_{d +- hd/2}).

Layouts: O-like results are [crop, token, head, column] (O_LAYOUT), the LSE [crop, head, token] (LSE_LAYOUT)."""
import math

import torch

U = 2.0 ** -9
C = 4.0
TINY = 2.0 ** -100
O_LAYOUT = ("crop", "token", "head", "column")
LSE_LAYOUT = ("crop", "head", "token")
INPUTS = ("std", "peaked4", "peaked16", "late_first", "late_last", "late_tile", "shifted", "uniform", "bait")
BIAS_Q = 8.0   # q column 0 of the bias families; k column 0 then sets a per-key scaled-logit offset b = 8 * scale * k_0


def lse_eps(N, hd):
    return 2.0 ** -24 * (N + 2 * hd + 32)


def split_qkv(qkv, n, N, H, hd):
    """qkv [n * N, 3 * H * hd] -> float64 q, k, v, each [crop, head, token, column]"""
    x = qkv.reshape(n, N, 3, H, hd).permute(2, 0, 3, 1, 4).double()
    return x[0], x[1], x[2]


def heads_first(t, n, N, H, hd):
    """[n * N, H * hd] -> float64 [crop, head, token, column]"""
    return t.reshape(n, N, H, hd).transpose(1, 2).double()


def grad_thirds(dqkv, n, N, H, hd):
    """the kernel's dqkv [n * N, 3 * H * hd] -> dq, dk, dv in O_LAYOUT"""
    x = dqkv.reshape(n, N, 3, H, hd)
    return x[:, :, 0], x[:, :, 1], x[:, :, 2]


def logits_of(qkv, n, N, H, hd):
    """float64 scaled scores [crop, head, query, key]"""
    q, k, _ = split_qkv(qkv, n, N, H, hd)
    return q @ k.transpose(-1, -2) * hd ** -0.5


def _chunks(n, H, N):
    """crop ranges whose [crops, H, N, N] float64 score tensors stay near 128 MB"""
    step = max(1, (1 << 24) // (H * N * N))
    return [(c, min(c + step, n)) for c in range(0, n, step)]


def forward(qkv, n, N, H, hd):
    """O*, LSE* and their bounds: dict(o, o_bound) in O_LAYOUT, dict(lse, lse_bound) in LSE_LAYOUT"""
    q, k, v = split_qkv(qkv, n, N, H, hd)
    scale = hd ** -0.5
    o, a, lse = torch.empty_like(v), torch.empty_like(v), q.new_empty(n, H, N)
    for c0, c1 in _chunks(n, H, N):
        s = q[c0:c1] @ k[c0:c1].transpose(-1, -2) * scale
        lse[c0:c1] = torch.logsumexp(s, -1)
        p = torch.exp(s - lse[c0:c1, ..., None])
        o[c0:c1] = p @ v[c0:c1]
        a[c0:c1] = p @ v[c0:c1].abs()
    bound = C * U * (a + o.abs()) + TINY
    return dict(o=o.transpose(1, 2), o_bound=bound.transpose(1, 2), lse=lse,
                lse_bound=lse_eps(N, hd) * (1 + lse.abs()))


def backward(qkv, o, do, n, N, H, hd, rope=None):
    """dQ*, dK*, dV* and their bounds (dict dq, dk, dv, dq_bound, dk_bound, dv_bound in O_LAYOUT) for the given bf16 O
    and dO ([n * N, H * hd]).  rope = (sin, cos, prefix): the gradients of the fused inverse RoPE (tokens >= prefix of dQ
    and dK rotated back with the tables [N - prefix, hd])."""
    q, k, v = split_qkv(qkv, n, N, H, hd)
    O, dO = heads_first(o, n, N, H, hd), heads_first(do, n, N, H, hd)
    scale = hd ** -0.5
    delta = (dO * O).sum(-1, keepdim=True)
    out = {name: torch.empty_like(q) for name in ("dq", "dk", "dv", "eq", "ek", "ev")}
    for c0, c1 in _chunks(n, H, N):
        sl = slice(c0, c1)
        p = torch.softmax(q[sl] @ k[sl].transpose(-1, -2) * scale, -1)
        dp = dO[sl] @ v[sl].transpose(-1, -2)
        ds = p * (dp - delta[sl]) * scale
        w = p * (dp.abs() + delta[sl].abs()) * scale
        out["dv"][sl] = p.transpose(-1, -2) @ dO[sl]
        out["ev"][sl] = p.transpose(-1, -2) @ dO[sl].abs()
        out["dk"][sl] = ds.transpose(-1, -2) @ q[sl]
        out["ek"][sl] = w.transpose(-1, -2) @ q[sl].abs()
        out["dq"][sl] = ds @ k[sl]
        out["eq"][sl] = w @ k[sl].abs()
    res = {}
    for g in ("dq", "dk", "dv"):
        res[g] = out[g]
        res[g + "_bound"] = C * U * (out["e" + g[1]] + out[g].abs()) + TINY
    if rope is not None:
        sin, cos, prefix = rope
        sin, cos = sin.to(q.device, torch.float64), cos.to(q.device, torch.float64)
        for g in ("dq", "dk"):
            res[g] = _rope_inverse(res[g], sin, cos, prefix)
            res[g + "_bound"] = _rope_abs(res[g + "_bound"], sin, cos, prefix)
    return {key: t.transpose(1, 2) for key, t in res.items()}


def _rope_inverse(x, sin, cos, prefix):
    """transpose of oracle.model.rope_apply on tokens >= prefix of x [crop, head, token, column]"""
    from oracle.model import rope_apply
    y = x.clone()
    y[:, :, prefix:] = rope_apply(x[:, :, prefix:], -sin, cos)
    return y


def _rope_abs(b, sin, cos, prefix):
    """bound of a rotated error whose parts are bounded by b: |cos| b_d + |sin| b_(d +- hd/2)"""
    h = b.shape[-1] // 2
    y = b.clone()
    t = b[:, :, prefix:]
    y[:, :, prefix:] = t * cos.abs() + torch.cat([t[..., h:], t[..., :h]], -1) * sin.abs()
    return y


def check(got, want, bound, layout, what="result"):
    """Asserts |got - want| <= bound element-wise (NaN fails) and returns the worst |got - want| / bound.  On failure the
    message names the worst element by `layout` (one name per dimension), its values, error, bound and ratio."""
    assert got.shape == want.shape == bound.shape and len(layout) == got.dim(), (got.shape, want.shape, bound.shape)
    err = (got.double() - want).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound).nan_to_num(nan=math.inf)
    flat = int(ratio.argmax())
    worst = float(ratio.reshape(-1)[flat])
    if worst > 1.0:
        idx, rest = [], flat
        for size in reversed(got.shape):
            idx.append(rest % size)
            rest //= size
        idx = tuple(reversed(idx))
        where = ", ".join(f"{name} {i}" for name, i in zip(layout, idx))
        raise AssertionError(
            f"{what} outside its bound at {where}: got {float(got[idx]):.6g}, want {float(want[idx]):.6g}, "
            f"error {float(err[idx]):.3e}, bound {float(bound[idx]):.3e}, ratio {worst:.2f} "
            f"({int((ratio > 1).sum())} of {ratio.numel()} elements outside)")
    return worst


# ------------------------------------------------------------------------------------------------ input families
def early_keys(N):
    """the key block that sits about +20 above the rest in the late-max families: the first 64 keys (half of a short
    crop)"""
    return torch.arange(min(64, max(N // 2, 1)))


def sink_key(kind, N):
    """the key about +40 above the rest: token 0, the crop's last token (in its partial last 64-key block and last
    128-key tile), or the middle of the last 128-key tile (a later tile than the queries of the first; the middle of a
    crop of at most 128 tokens)"""
    if kind == "late_first":
        return 0
    if kind == "late_last":
        return N - 1
    assert kind == "late_tile"
    last = (N - 1) // 128 * 128
    return last + (N - 1 - last) // 2


def make_inputs(kind, n, N, H, hd, seed=0, device="cpu"):
    """Seeded bf16 qkv [n * N, 3 * H * hd] of one input family; asserts the family's property on its float64 logits.
      std          randn: scaled logits of std 1.
      peaked<s>    q and k scaled by sqrt(s): scaled logits of std s (s = 16 reaches about +-80).
      late_<where> per crop the early_keys block about +20 above the rest and the sink_key about +40: the running max
                   jumps after o and l have accumulated.
      shifted      every logit of a row raised by about +60 through column 0 of q and k: O* equals the unshifted O*.
      uniform      q = 0: P = 1/N exactly, O* the mean of the crop's own v.
      bait         in-crop scaled logits about -40, the neighbouring crops' keys about +40 (crop signs alternate in
                   column 0), zero-filled rows past the tensor score 0: any key outside a row's crop dominates it.
    The scaled-logit offsets of the bias families come from q column 0 = BIAS_Q and k column 0 = b / (BIAS_Q scale)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, N, 3, H, hd, generator=g)
    q, k = x[:, :, 0], x[:, :, 1]                 # views [crop, token, head, column]
    kb = 1.0 / (BIAS_Q * hd ** -0.5)              # k column 0 per unit of scaled-logit offset
    if kind.startswith("peaked"):
        x[:, :, :2] *= math.sqrt(float(kind[len("peaked"):]))
    elif kind.startswith("late_"):
        b = torch.zeros(N)
        b[early_keys(N)] = 20.0
        b[sink_key(kind, N)] = 40.0
        q[..., 0] = BIAS_Q
        k[..., 0] = b[None, :, None] * kb
    elif kind == "shifted":
        q[..., 0] = BIAS_Q
        k[..., 0] = 60.0 * kb
    elif kind == "uniform":
        q.zero_()
    elif kind == "bait":
        sign = (1 - 2 * (torch.arange(n) % 2)).float()[:, None, None]   # +1, -1, +1, ... per crop
        q[..., 0] = BIAS_Q * sign
        k[..., 0] = -40.0 * kb * sign
    elif kind != "std":
        raise ValueError(kind)
    qkv = x.reshape(n * N, 3 * H * hd).to(torch.bfloat16).to(device)
    _assert_property(kind, qkv, n, N, H, hd)
    return qkv


def make_grad(n, N, H, hd, seed=0, device="cpu"):
    g = torch.Generator().manual_seed(seed + 1)
    return torch.randn(n * N, H * hd, generator=g).to(torch.bfloat16).to(device)


def _assert_property(kind, qkv, n, N, H, hd):
    q, k, _ = split_qkv(qkv, n, N, H, hd)
    scale = hd ** -0.5
    tot, tot2, top, cnt = 0.0, 0.0, 0.0, 0
    for c0, c1 in _chunks(n, H, N):
        s = q[c0:c1] @ k[c0:c1].transpose(-1, -2) * scale      # [crops, H, N queries, N keys]
        tot, tot2, cnt = tot + float(s.sum()), tot2 + float((s * s).sum()), cnt + s.numel()
        top = max(top, float(s.abs().max()))
        if kind.startswith("late_"):
            sink, early = sink_key(kind, N), early_keys(N)
            assert bool((s.argmax(-1) == sink).all()), f"{kind}: a row maximum is not at key {sink}"
            rest = torch.ones(N, dtype=torch.bool, device=s.device)
            rest[early], rest[sink] = False, False
            e = s[..., early[early != sink]].amax(-1)
            assert float((s[..., sink] - e).min()) >= 10, f"{kind}: the sink is not well above the early block"
            if bool(rest.any()):
                assert float((e - s[..., rest].amax(-1)).min()) >= 10, f"{kind}: the early block is not above the rest"
        elif kind == "shifted":
            assert float(s.min()) >= 40, "shifted: a logit below +40"
        elif kind == "uniform":
            assert bool((s == 0).all()), "uniform: a logit is not exactly 0"
        elif kind == "bait":
            assert float(s.max()) <= -30, "bait: an in-crop logit above -30"
    std = math.sqrt(max(tot2 / cnt - (tot / cnt) ** 2, 0.0))
    if kind == "std":
        assert 0.8 <= std <= 1.2, f"std: logit std {std}"
    elif kind.startswith("peaked"):
        sigma = float(kind[len("peaked"):])
        assert 0.8 * sigma <= std <= 1.2 * sigma and top >= 3 * sigma, f"{kind}: logit std {std}, max |s| {top}"
    elif kind == "bait":
        for c in range(n - 1):                                   # both directions between neighbouring crops
            for a, b in ((c, c + 1), (c + 1, c)):
                x = q[a] @ k[b].transpose(-1, -2) * scale
                assert float(x.min()) >= 30, f"bait: a key of crop {b} scores {float(x.min())} for crop {a}"
