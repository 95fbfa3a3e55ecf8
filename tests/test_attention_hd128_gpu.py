"""-m gpu: attention at head_dim 128 (vit_7b: embed 4096, 32 heads).  The kernels against PyTorch fp32 / autograd at every
crop length class (packed short crops with a ragged last group, one tile, ragged tiles, long crops), the fused inverse
RoPE, bit reproducibility, the engine step against the oracle at narrow width, and the 7B width itself."""
import dataclasses

import pytest
import torch

from attention_helpers import BF16_TOL, attn_ref, bwd, fwd, rel
from test_engine_gpu import HYPER, check, run_pair

pytestmark = pytest.mark.gpu

HD = 128
NS = [1, 37, 54, 64, 65, 128, 129, 197, 261, 449, 1029, 2309]


@pytest.fixture(autouse=True)
def _seed(native):
    torch.manual_seed(0)


def n_crops(N):
    # short crops: 5 crops leave a ragged last packed group (N = 37: groups of 3 and 2, N = 54: 2 + 2 + 1)
    return 5 if N <= 64 else 3 if N <= 449 else 2 if N <= 1029 else 1


@pytest.mark.parametrize("H", [1, 2, 32])
@pytest.mark.parametrize("N", NS)
def test_hd128_forward_and_backward(N, H):
    n, D = n_crops(N), HD * H
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    x = qkv.float().requires_grad_(True)
    ro, rl = attn_ref(x, n, N, H, HD)
    ro.backward(do.float())
    o, lse = fwd(qkv, n, N, H, HD)
    assert rel(o, ro.detach()) < BF16_TOL and rel(lse, rl.detach()) < 1e-5
    dqkv = bwd(qkv, o, do, lse, n, N, H, HD)
    # at N = 1 dq and dk are exactly zero (dP - Delta = 0): their error is measured against the scale of the whole dqkv
    floor = 1e-2 * x.grad.norm().item()
    for j in range(3):
        got, want = dqkv[:, j * D:(j + 1) * D].float(), x.grad[:, j * D:(j + 1) * D]
        assert (got - want).norm().item() / max(want.norm().item(), floor) < 1e-2, j


@pytest.mark.parametrize("Hp,prefix", [(3, 5), (7, 5), (16, 5), (24, 1)])
def test_hd128_backward_fused_inverse_rope(Hp, prefix):
    """dqkv with rope tables [P, 128] == d3_rope(inverse) of the plain backward: pairs (d, d + 64), tokens < prefix and
    the v third untouched (packed 14- / 54-token crops, 261 and 577 tokens)."""
    from dinov3_jax import ops
    from oracle.model import rope_sincos
    n, H = 3, 2
    N, D = Hp * Hp + prefix, HD * H
    sin, cos = [t.cuda().contiguous() for t in rope_sincos(Hp, Hp, HD, 100.0, torch.float32)]
    assert sin.shape == (Hp * Hp, HD)
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    o, lse = fwd(qkv, n, N, H, HD)
    d1 = bwd(qkv, o, do, lse, n, N, H, HD)
    ops.rope(d1, sin, cos, N, prefix, D, HD, inverse=True)
    d2 = bwd(qkv, o, do, lse, n, N, H, HD, rope_sin=sin, rope_cos=cos, rope_prefix=prefix)
    assert rel(d2, d1) < BF16_TOL          # d1 is rounded to bf16 twice, d2 once
    assert torch.equal(d2[:, 2 * D:], d1[:, 2 * D:])
    pre = torch.cat([torch.arange(c * N, c * N + prefix) for c in range(n)]).cuda()
    assert torch.equal(d2[pre, :2 * D], bwd(qkv, o, do, lse, n, N, H, HD)[pre, :2 * D])


def test_hd128_rope_forward_matches_oracle():
    """d3_rope at head_dim 128 against the oracle's rotation (layers/attention.py:14-20): q and k of patch tokens rotated,
    prefix tokens and v unchanged."""
    from dinov3_jax import ops
    from oracle.model import rope_apply, rope_sincos
    n, H, Hp, prefix = 2, 3, 7, 5
    N, D = Hp * Hp + prefix, HD * H
    sin, cos = rope_sincos(Hp, Hp, HD, 100.0, torch.float32)
    qkv = torch.randn(n * N, 3 * D).to(torch.bfloat16)
    got = ops.rope(qkv.cuda().contiguous(), sin.cuda().contiguous(), cos.cuda().contiguous(), N, prefix, D, HD).cpu()
    x = qkv.float().reshape(n, N, 3, H, HD)
    want = x.clone()
    want[:, prefix:, :2] = rope_apply(x[:, prefix:, :2], sin[None, :, None, None], cos[None, :, None, None])
    want = want.reshape(n * N, 3 * D)
    assert rel(got, want) < 4e-3
    assert torch.equal(got.reshape(n, N, 3 * D)[:, :prefix], qkv.reshape(n, N, 3 * D)[:, :prefix])
    assert torch.equal(got[:, 2 * D:], qkv[:, 2 * D:])


@pytest.mark.parametrize("n,N,H", [(10, 54, 32), (4, 261, 32), (2, 1029, 32)])
def test_hd128_attention_is_bit_reproducible(n, N, H):
    D = HD * H
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    (o1, l1), (o2, l2) = fwd(qkv, n, N, H, HD), fwd(qkv, n, N, H, HD)
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    assert torch.equal(bwd(qkv, o1, do, l1, n, N, H, HD), bwd(qkv, o1, do, l1, n, N, H, HD))


def test_other_head_dims_are_refused():
    from dinov3_jax import ops
    qkv = torch.zeros(37, 3 * 96, device="cuda", dtype=torch.bfloat16)
    o = torch.zeros(37, 96, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(Exception, match="64 or 128"):
        ops.attn_fwd(qkv, o, None, 1, 37, 96, 1)


# ------------------------------------------------------------------------------------------------ engine at head_dim 128
def hd128_cfg(**kw):
    from oracle import tiny_cfg
    return tiny_cfg(embed_dim=256, heads=2, **kw)


def test_hd128_tiny_step_matches_oracle():
    check(run_pair(hd128_cfg(), 2))


def test_hd128_7b_block_recipe_matches_oracle():
    """The 7B block recipe at narrow width: SwiGLU64 at ffn_ratio 3, layernormbf16, 4 storage tokens, mask_k_bias."""
    check(run_pair(hd128_cfg(ffn_layer="swiglu", swiglu_align=64, ffn_ratio=3.0, ln_eps=1e-5, n_storage=4,
                             mask_k_bias=True, layerscale=0.5), 2, seed=4))


def test_hd128_step_with_long_global_crops():
    check(run_pair(hd128_cfg(global_size=352), 2))          # 485-token global crops


def test_hd128_remat_equals_stashing():
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg = hd128_cfg(layerscale=0.5, depth=3)
    B = 2
    P = init_params(cfg, 0, perturb=0.05)
    batch = synthetic_batch(cfg, B, 1)
    out = []
    for remat in (False, True):
        eng = Engine(from_oracle_cfg(cfg), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1), remat=remat)
        eng.params.load_reference_tree(P)
        eng.set_batch(batch)
        eng.forward_backward(HYPER["teacher_temp"])
        out.append((eng.read_metrics()["total_loss"], {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}))
    (la, ga), (lb, gb) = out
    assert abs(la - lb) <= 1e-6 * abs(la)
    num = sum(float(((ga[k] - gb[k]) ** 2).sum()) for k in ga)
    den = sum(float((ga[k] ** 2).sum()) for k in ga)
    assert (num / den) ** 0.5 < 5e-3


def test_hd128_step_with_gram_anchoring():
    """EMA-teacher Gram anchoring at head_dim 128: loss and gradients against oracle.step.ssl_forward under autograd."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    from oracle.step import ssl_forward
    cfg = hd128_cfg(layerscale=0.5)
    B, W = 2, 25.0
    P = init_params(cfg, 6, perturb=0.05)
    batch = synthetic_batch(cfg, B, 6)
    ecfg = dataclasses.replace(from_oracle_cfg(cfg), gram_use_loss=True, gram_loss_weight=W, gram_ema_teacher=True,
                               gram_it_load_ema_teacher=0)
    eng = Engine(ecfg, B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    eng.params.load_reference_tree(P)
    full = dict(P)
    student = {k: v.detach().clone().requires_grad_(True) for k, v in P.items() if k.startswith("student_")}
    full.update(student)
    loss, m = ssl_forward(full, batch, HYPER["teacher_temp"], cfg,
                          gram=dict(weight=W, ema_teacher=True, normalized=True, img_level=False, remove_neg=False,
                                    remove_only_teacher_neg=False, tokens_used="all"))
    keys = list(student)
    gl = torch.autograd.grad(loss, [student[k] for k in keys], allow_unused=True)
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    met = eng.read_metrics()
    assert abs(met["gram_loss"] - float(m["gram_loss"])) < 2e-2 * float(m["gram_loss"])
    assert abs(met["total_loss"] - float(loss.detach())) < 2e-3 * abs(float(loss.detach()))
    ge = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
    num = sum(((ge[k].reshape(g_.shape) - g_) ** 2).sum() for k, g_ in zip(keys, gl) if g_ is not None)
    den = sum((g_ ** 2).sum() for g_ in gl if g_ is not None)
    assert float(torch.sqrt(num / den)) < 3e-2


def test_hd128_steps_are_bit_reproducible():
    """Two engines (packed local crops and streamed 485-token global crops at head_dim 128) run the same two steps:
    every gradient, parameter and metric is identical."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg = hd128_cfg(global_size=352)
    B = 2
    P = init_params(cfg, 0, perturb=0.05)
    batch = synthetic_batch(cfg, B, 0)
    runs = []
    for _ in range(2):
        eng = Engine(from_oracle_cfg(cfg), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
        eng.params.load_reference_tree(P)
        for _ in range(2):
            eng.train_step(batch, **HYPER)
        torch.cuda.synchronize()
        runs.append((eng.read_metrics(), {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()},
                     {k: v.cpu() for k, v in eng.params.export_reference_tree("param").items()}))
        del eng
    (m0, g0, p0), (m1, g1, p1) = runs
    assert m0 == m1
    assert all(torch.equal(g0[k], g1[k]) for k in g0), [k for k in g0 if not torch.equal(g0[k], g1[k])][:5]
    assert all(torch.equal(p0[k], p1[k]) for k in p0), [k for k in p0 if not torch.equal(p0[k], p1[k])][:5]


# ------------------------------------------------------------------------------------------------ at real 7B width
def _tree(flat):
    tree = {}
    for k, v in flat.items():
        cur = tree
        parts = k.split("/")
        for p in parts[:-1]:
            cur = cur.setdefault(p, {})
        cur[parts[-1]] = v
    return tree


def test_vit_7b_width_forward_matches_oracle():
    """dinov3_jax.models.DinoVisionTransformer at embed 4096 / 32 heads (one block, ffn_ratio 3, 4 storage tokens) on
    256^2 global and 112^2 local crops against the oracle's backbone forward (fp32, CPU)."""
    from dinov3_jax.models import DinoVisionTransformer
    from oracle.arch import ModelCfg
    from oracle.model import backbone_forward, init_params, sub
    cfg = ModelCfg(embed_dim=4096, depth=1, heads=32, ffn_ratio=3.0, global_size=256, local_size=112, n_storage=4,
                   layerscale=0.5, ln_eps=1e-5, n_prototypes=64, head_hidden=64, head_bottleneck=64)
    bp = sub(init_params(cfg, 0, perturb=0.05), "student_backbone")
    model = DinoVisionTransformer(_tree(bp), img_size=256, patch_size=16, embed_dim=4096, n_blocks=1, num_heads=32,
                                  ffn_ratio=3.0, layerscale_init=0.5, n_storage_tokens=4, norm_layer="layernormbf16")
    xg = torch.randn(1, 256, 256, 3).to(torch.bfloat16).float()
    xl = torch.randn(2, 112, 112, 3).to(torch.bfloat16).float()
    masks = torch.rand(1, 16 * 16) < 0.3
    got = model([xg, xl], masks=[masks, None], is_training=True)
    ref = backbone_forward(bp, [xg, xl], [masks, None], cfg)
    assert got[0]["x_norm_patchtokens"].shape[1] == 256 and got[1]["x_norm_patchtokens"].shape[1] == 49
    for g, r in zip(got, ref):
        for k in ("x_norm_clstoken", "x_storage_tokens", "x_norm_patchtokens"):
            assert rel(g[k].cpu(), r[k]) < 2e-2, k


def test_vit_7b_recipe_train_step_is_finite():
    """One Engine.train_step of the vit_7b recipe (head_dim 128, ffn_ratio 3, SwiGLU64, layernormbf16, mask_k_bias, 4
    storage tokens) on 256^2 global / 112^2 local crops (261 / 54 tokens), B = 1, small prototype heads, at the widest
    width the engine trains (1536 = 12 heads of 128); the 4096-wide engine is refused with a message."""
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import init_reference_like, synthetic_batch
    kw = dict(depth=1, global_size=256, local_size=112, n_storage=4, n_prototypes=1024, head_hidden=512,
              head_bottleneck=256, ffn_layer="swiglu", swiglu_align=64, ln_eps=1e-5, mask_k_bias=True)
    with pytest.raises(NotImplementedError, match="1536"):
        Engine(config_for("vit_7b", **kw), 1)
    cfg = config_for("vit_7b", embed_dim=1536, heads=12, **kw)
    assert (cfg.head_dim, cfg.ffn_ratio, cfg.tokens(256), cfg.tokens(112)) == (128, 3.0, 261, 54)
    batch = synthetic_batch(cfg, 1, seed=2)
    eng = Engine(cfg, 1, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    init_reference_like(eng)
    eng.train_step(batch, **HYPER)
    m = eng.read_metrics()
    assert all(v == v and abs(v) != float("inf") for v in m.values()), m
    assert abs(m["dino_local_crops_loss"] - 6.931) < 0.1       # log(1024) at init
