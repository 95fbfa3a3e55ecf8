"""-m gpu: attention on crops longer than the resident kernels hold (forward span > 448, backward span > 256), served by the
streamed kernels: against PyTorch fp32 / autograd, with the fused inverse RoPE, bit-reproducible, and through the
module forward and full training steps at high resolution against the oracle."""
import dataclasses

import pytest
import torch

from attention_helpers import BF16_TOL, attn_ref, bwd, fwd, rel
from test_engine_gpu import HYPER, check, run_pair

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _seed(native):
    torch.manual_seed(0)


# (16, 1029, 16): 512^2 crops at patch 16 with 4 storage tokens, ViT-L heads; (1, 5189, 2): a 1 152^2 gram teacher crop
@pytest.mark.parametrize("n,N,H", [(1, 449, 1), (2, 450, 2), (3, 513, 1), (2, 577, 4), (2, 1029, 2), (1, 2309, 1),
                                   (16, 1029, 16), (1, 5189, 2)])
def test_long_attention_forward(n, N, H):
    qkv = torch.randn(n * N, 3 * 64 * H, device="cuda").to(torch.bfloat16)
    o, lse = fwd(qkv, n, N, H)
    ro, rl = attn_ref(qkv, n, N, H)
    assert rel(o, ro) < BF16_TOL and rel(lse, rl) < 1e-5


# N = 385 ... 448: the resident forward's LSE feeds the streamed backward
@pytest.mark.parametrize("n,N,H", [(1, 385, 1), (2, 401, 2), (2, 448, 1), (1, 449, 1), (3, 577, 2), (2, 1029, 2), (1, 2309, 1)])
def test_long_attention_backward(n, N, H):
    D = 64 * H
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    x = qkv.float().requires_grad_(True)
    attn_ref(x, n, N, H)[0].backward(do.float())
    o, lse = fwd(qkv, n, N, H)
    dqkv = bwd(qkv, o, do, lse, n, N, H)
    for j in range(3):
        assert rel(dqkv[:, j * D:(j + 1) * D], x.grad[:, j * D:(j + 1) * D]) < 1e-2


@pytest.mark.parametrize("Hp,prefix", [(24, 1), (32, 5)])
def test_long_attention_backward_fused_inverse_rope(Hp, prefix):
    """dqkv with rope tables == separate inverse-RoPE of the plain backward (tokens < prefix untouched, v untouched)."""
    from dinov3_jax import ops
    from oracle.model import rope_sincos
    n, H = 2, 2
    N, D = Hp * Hp + prefix, 64 * H
    sin, cos = [t.cuda().contiguous() for t in rope_sincos(Hp, Hp, 64, 100.0, torch.float32)]
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    o, lse = fwd(qkv, n, N, H)
    d1 = bwd(qkv, o, do, lse, n, N, H)
    ops.rope(d1, sin, cos, N, prefix, D, 64, inverse=True)
    d2 = bwd(qkv, o, do, lse, n, N, H, rope_sin=sin, rope_cos=cos, rope_prefix=prefix)
    assert rel(d2, d1) < BF16_TOL          # d1 is rounded to bf16 twice, d2 once
    assert torch.equal(d2[:, 2 * D:], d1[:, 2 * D:])


def test_long_attention_is_bit_reproducible():
    n, N, H = 4, 1029, 16
    qkv = torch.randn(n * N, 3 * 64 * H, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, 64 * H, device="cuda").to(torch.bfloat16)
    (o1, l1), (o2, l2) = fwd(qkv, n, N, H), fwd(qkv, n, N, H)
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    assert torch.equal(bwd(qkv, o1, do, l1, n, N, H), bwd(qkv, o1, do, l1, n, N, H))


def test_vit_forward_at_512(native):
    """dinov3_jax.models.DinoVisionTransformer on 512^2 global crops (1 029 tokens with 4 storage tokens) against the
    oracle's backbone forward."""
    from dinov3_jax.models import DinoVisionTransformer
    from oracle import tiny_cfg
    from oracle.model import backbone_forward, init_params, sub
    cfg = tiny_cfg(global_size=512, n_storage=4, layerscale=0.5)
    bp = sub(init_params(cfg, 0, perturb=0.05), "student_backbone")
    tree = {}
    for k, v in bp.items():
        cur = tree
        parts = k.split("/")
        for p in parts[:-1]:
            cur = cur.setdefault(p, {})
        cur[parts[-1]] = v
    model = DinoVisionTransformer(tree, img_size=512, patch_size=16, embed_dim=128, n_blocks=2, num_heads=2,
                                  layerscale_init=0.5, n_storage_tokens=4)
    x = torch.randn(2, 512, 512, 3).to(torch.bfloat16).float()
    masks = torch.rand(2, 32 * 32) < 0.3
    got = model([x], masks=[masks], is_training=True)[0]
    ref = backbone_forward(bp, [x], [masks], cfg)[0]
    assert got["x_norm_patchtokens"].shape[1] == 1024
    for k in ("x_norm_clstoken", "x_storage_tokens", "x_norm_patchtokens"):
        assert rel(got[k].cpu(), ref[k]) < 2e-2, k


def test_step_with_streamed_forward_and_backward():
    from oracle import tiny_cfg
    check(run_pair(tiny_cfg(global_size=352), 2))          # 485-token global crops


def test_step_with_resident_forward_and_streamed_backward():
    from oracle import tiny_cfg
    check(run_pair(tiny_cfg(global_size=320), 2))          # 401-token global crops


@pytest.mark.parametrize("antialias", [False, True])
def test_gram_teacher_above_448_tokens(antialias):
    """Student global crops 160^2 (10x10 patches), frozen gram teacher on its own 400^2 crops (626 tokens), resized to
    the student's grid: loss and gradients against the oracle."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    from oracle.step import ssl_forward
    cfg = tiny_cfg(layerscale=0.5, global_size=160)
    B, W, GS = 2, 25.0, 400
    P = init_params(cfg, 8, perturb=0.05)
    batch = synthetic_batch(cfg, B, 8)
    g = torch.Generator().manual_seed(3)
    batch["collated_gram_teacher_crops"] = torch.randn(cfg.n_global * B, GS, GS, 3, generator=g).to(torch.bfloat16)
    ecfg = dataclasses.replace(from_oracle_cfg(cfg), gram_use_loss=True, gram_loss_weight=W, gram_it_load_ema_teacher=0,
                               gram_teacher_size=GS, gram_resize_antialias=antialias)
    eng = Engine(ecfg, B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    assert eng.g_sets[0].N == 626
    eng.params.load_reference_tree(P)
    P2 = init_params(cfg, 9, perturb=0.05)
    tree = {k[len("teacher_backbone/"):]: v for k, v in P2.items() if k.startswith("teacher_backbone/")}
    eng.gram_teacher_load(tree)
    full = dict(P)
    full.update({"gram_backbone/" + k: v for k, v in tree.items()})
    student = {k: v.detach().clone().requires_grad_(True) for k, v in P.items() if k.startswith("student_")}
    full.update(student)
    loss, m = ssl_forward(full, batch, HYPER["teacher_temp"], cfg,
                          gram=dict(weight=W, ema_teacher=False, remove_neg=False, remove_only_teacher_neg=False,
                                    resize_antialias=antialias))
    keys = list(student)
    gl = torch.autograd.grad(loss, [student[k] for k in keys], allow_unused=True)
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    met = eng.read_metrics()
    assert abs(met["gram_loss"] - float(m["gram_loss"])) < 2e-2 * float(m["gram_loss"]), (met["gram_loss"], float(m["gram_loss"]))
    assert abs(met["total_loss"] - float(loss.detach())) < 2e-3 * abs(float(loss.detach()))
    ge = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
    num = sum(((ge[k].reshape(g_.shape) - g_) ** 2).sum() for k, g_ in zip(keys, gl) if g_ is not None)
    den = sum((g_ ** 2).sum() for g_ in gl if g_ is not None)
    assert float(torch.sqrt(num / den)) < 3e-2


def test_high_resolution_steps_are_bit_reproducible():
    """Two engines at 352^2 global crops (streamed attention forward and backward) run the same two steps: every
    gradient, parameter and metric is identical."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg = tiny_cfg(global_size=352)
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
