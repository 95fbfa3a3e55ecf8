"""Pins the oracle (and the product's host-side mirrors) against golden vectors produced by EXECUTING reference files
(tests/golden/make_golden.py): masks / collate / schedules directly, losses / RoPE / param groups under the numpy
stand-in for jax+flax; DinoVisionTransformer (+ every layer under it) and DINOHead under the shim's mini flax.linen.
Nothing here reads the reference checkout."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import reference_vectors

G = reference_vectors()
T = lambda a: torch.from_numpy(np.asarray(a))


@pytest.mark.parametrize("impl", ["oracle", "product"])
@pytest.mark.parametrize("tag,n,grid,size", [("b8", 16, 14, 224), ("tiny", 8, 4, 64)])
def test_masks_bit_exact(impl, tag, n, grid, size):
    if impl == "oracle":
        from oracle.batch import MaskGen as Gen, collate_masks
    else:
        from dinov3_jax.data.masking import MaskingGenerator as Gen
        from dinov3_jax.data.collate import collate_masks
    random.seed(7); np.random.seed(7)
    gen = Gen(input_size=(grid, grid), max_num_patches=0.5 * size // 16 * size // 16)
    d = collate_masks(n, grid * grid, (0.1, 0.5), 0.5, gen)
    assert np.array_equal(d["collated_masks"].numpy(), G[f"masks_{tag}"])
    assert np.array_equal(d["mask_indices_list"].numpy(), G[f"mask_indices_{tag}"])
    assert np.array_equal(d["masks_weight"].numpy(), G[f"masks_weight_{tag}"])
    assert d["upperbound"] == int(G[f"upperbound_{tag}"])
    assert int(d["n_masked_patches"]) == len(G[f"mask_indices_{tag}"])


@pytest.mark.parametrize("impl", ["oracle", "product"])
def test_schedules_bit_exact(impl):
    if impl == "oracle":
        from oracle.step import cosine_schedule
    else:
        from dinov3_jax.train.cosine_lr_scheduler import CosineScheduler
        cosine_schedule = lambda *a, **k: CosineScheduler(*a, **k).gen()
    assert np.array_equal(cosine_schedule(1e-3, 1e-6, 500, warmup_iters=50, start_warmup_value=0), G["sched_lr"])
    assert np.array_equal(cosine_schedule(0.04, 0.4, 500), G["sched_wd"])
    assert np.array_equal(cosine_schedule(0.07, 0.07, 120, warmup_iters=120, start_warmup_value=0.04), G["sched_temp"])
    assert np.array_equal(cosine_schedule(1.0, 0.0, 60, warmup_iters=10, freeze_iters=5), G["sched_freeze"])


def test_sinkhorn_and_dino_loss_match_reference_code():
    from oracle.losses import dino_loss, sinkhorn_knopp
    B, K = 5, 48
    Q = sinkhorn_knopp(T(G["dino_t_logits"]), 0.05, B_total=2 * B)
    assert torch.allclose(Q, T(G["dino_probs"]), rtol=1e-10, atol=1e-14)
    Qr = T(G["dino_probs"]).reshape(2, B, K)
    assert abs(dino_loss(T(G["dino_s_local"]), Qr, 0.1, False).item() - float(G["dino_loss_local"])) < 1e-12
    assert abs(dino_loss(T(G["dino_s_global"]), Qr, 0.1, True).item() - float(G["dino_loss_global"])) < 1e-12


def test_ibot_matches_reference_code():
    from oracle.losses import ibot_loss_masked, sinkhorn_knopp
    M = G["ibot_t_logits"].shape[0]
    Q = sinkhorn_knopp(T(G["ibot_t_logits"]), 0.05, B_total=float(M))
    assert torch.allclose(Q, T(G["ibot_probs"]), rtol=1e-10, atol=1e-14)
    assert abs(ibot_loss_masked(T(G["ibot_s"]), T(G["ibot_probs"]), 0.1, n_mask_rows=10).item() - float(G["ibot_loss"])) < 1e-12


def test_koleo_matches_reference_code():
    from oracle.losses import koleo_loss
    assert abs(koleo_loss(T(G["koleo_x"])).item() - float(G["koleo_loss"])) < 1e-12


@pytest.mark.parametrize("H,W", [(14, 14), (6, 6), (3, 5)])
def test_rope_tables_match_reference_code(H, W):
    from oracle.model import rope_sincos
    sin, cos = rope_sincos(H, W, 64, 100.0, torch.float64)
    assert torch.allclose(sin, T(G[f"rope_sin_{H}x{W}"]), atol=1e-13) and torch.allclose(cos, T(G[f"rope_cos_{H}x{W}"]), atol=1e-13)
    from dinov3_jax.engine.core import rope_tables      # the product's table builder (host side, fp32 output)
    if H == W:
        s32, c32 = rope_tables(H, W, 64, 100.0, "cpu")
        assert torch.allclose(s32.double(), T(G[f"rope_sin_{H}x{W}"]), atol=1e-6)
        assert torch.allclose(c32.double(), T(G[f"rope_cos_{H}x{W}"]), atol=1e-6)


def test_rope_apply_matches_reference_code():
    from oracle.model import rope_apply, rope_sincos
    sin, cos = rope_sincos(3, 3, 64, 100.0, torch.float64)
    assert torch.allclose(rope_apply(T(G["rope_x"]), sin, cos), T(G["rope_y"]), atol=1e-13)


@pytest.mark.parametrize("impl", ["oracle", "product"])
def test_param_group_multipliers_match_reference_code(impl):
    names = [str(n) for n in G["pg_names"]]
    vals = G["pg_values"]
    if impl == "oracle":
        from oracle.step import param_multipliers
        got = param_multipliers(names, depth=4)
        rows = [got[n] for n in names]
    else:
        from dinov3_jax.engine.config import EngineConfig
        from dinov3_jax.engine.params import lr_wd_multipliers
        cfg = EngineConfig(depth=4)
        rows = [lr_wd_multipliers(n.split("/", 1)[0][len("student_"):], n.split("/", 1)[1], cfg) for n in names]
    for n, (lr, wd, last), want in zip(names, rows, vals):
        assert abs(lr - want[0]) < 1e-12 and wd == want[1] and float(last) == want[2], n


def _golden_tree(prefix):
    return {k[len(prefix):]: T(G[k]).double() for k in G if k.startswith(prefix)}


def test_backbone_matches_reference_module_code():
    """models/vision_transformer.py DinoVisionTransformer.__call__(is_training=True) on [global, local] crops with iBOT
    masks, executed from the reference sources, vs the oracle restatement in float64."""
    from oracle.arch import ModelCfg
    from oracle.model import backbone_forward
    cfg = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_prototypes=48, head_hidden=64,
                   head_bottleneck=32, layerscale=0.5)
    bp = _golden_tree("vit_param/")
    outs = backbone_forward(bp, [T(G["vit_global"]).double(), T(G["vit_local"]).double()], [T(G["vit_masks"]), None], cfg)
    for o, tag in zip(outs, ("g", "l")):
        assert np.abs(o["x_norm_clstoken"].numpy() - G[f"vit_{tag}_cls"]).max() < 1e-11
        assert np.abs(o["x_norm_patchtokens"].numpy() - G[f"vit_{tag}_patch"]).max() < 1e-11
    # the mask has to matter (mask_token substituted before the blocks) or the fixture pins nothing about a4
    nomask = backbone_forward(bp, [T(G["vit_global"]).double()], [None], cfg)[0]
    assert np.abs(nomask["x_norm_clstoken"].numpy() - G["vit_g_cls"]).max() > 1e-3


def test_head_matches_reference_module_code():
    from oracle.model import head_forward
    hp = _golden_tree("head_param/")
    x = T(G["head_x"]).double()
    assert np.abs(head_forward(hp, x).numpy() - G["head_logits"]).max() < 1e-12
    assert np.abs(head_forward(hp, x, last_layer=False).numpy() - G["head_bottleneck"]).max() < 1e-12


def ssl_case(case, dtype=torch.float64):
    """Rebuild the closed-form inputs of an SSLMetaArch fixture (tests/golden/make_golden.py)."""
    from oracle.arch import ModelCfg
    from oracle.model import formula_images, formula_params
    B, n_local, seed, n_storage, norm_bf16 = (int(v) for v in G[f"ssl_{case}_spec"])
    cfg = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_local=n_local, n_prototypes=48,
                   head_hidden=64, head_bottleneck=32, n_storage=n_storage, ln_eps=1e-5 if norm_bf16 else 1e-6)
    masks = T(G[f"ssl_{case}_masks"])
    idx = T(G[f"ssl_{case}_mask_indices"])
    batch = {"collated_global_crops": formula_images((2 * B, 64, 64, 3), 100 + seed, dtype),
             "collated_local_crops": formula_images((n_local * B, 32, 32, 3), 200 + seed, dtype),
             "collated_masks": masks, "mask_indices_list": idx,
             "masks_weight": (1 / masks.sum(-1).clamp(min=1.0)).unsqueeze(-1).expand_as(masks)[masks].to(torch.float32),
             "n_masked_patches": torch.tensor([idx.shape[0]]), "upperbound": int(idx.shape[0]), "global_batch_size": B}
    return cfg, formula_params(cfg, seed, dtype), batch, float(G[f"ssl_{case}_teacher_temp"])


def test_backbone_with_storage_tokens_matches_reference_module_code():
    """DinoVisionTransformer(n_storage_tokens=4, norm_layer="layernormbf16") from the reference sources (SURVEY §8f.1):
    register tokens sit between cls and the patches, are not rotated by RoPE and come back as x_storage_tokens."""
    from oracle.arch import ModelCfg
    from oracle.model import backbone_forward, formula_images, formula_params, sub
    cfg = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_prototypes=48, head_hidden=64,
                   head_bottleneck=32, n_storage=4, ln_eps=1e-5)
    bp = sub(formula_params(cfg, 9), "student_backbone")
    outs = backbone_forward(bp, [formula_images((2, 64, 64, 3), 31), formula_images((3, 32, 32, 3), 32)],
                            [T(G["vit_masks"]), None], cfg)
    for o, tag in zip(outs, ("g", "l")):
        assert o["x_storage_tokens"].shape[1] == 4
        for key, name in (("x_norm_clstoken", "cls"), ("x_storage_tokens", "storage"), ("x_norm_patchtokens", "patch")):
            assert np.abs(o[key].numpy() - G[f"vitr_{tag}_{name}"]).max() < 1e-10, (tag, name)


@pytest.mark.parametrize("case", ["a", "b", "c"])
def test_ssl_forward_matches_reference_meta_arch(case):
    """train/ssl_meta_arch.py SSLMetaArch.__call__ executed from the reference sources (teacher + student passes, four
    heads, iBOT gathers, both Sinkhorns, loss weights) vs oracle.step.ssl_forward, float64.  The gradient the oracle
    hands to the GPU parity tests is torch autograd of exactly this function."""
    from oracle.step import ssl_forward
    cfg, P, batch, temp = ssl_case(case)
    loss, metrics = ssl_forward(P, batch, temp, cfg, dtype=torch.float64)
    assert abs(float(loss) - float(G[f"ssl_{case}_loss"])) < 1e-9 * abs(float(G[f"ssl_{case}_loss"]))
    keys = [k.split("/", 1)[1] for k in G if k.startswith(f"ssl_{case}_metric/")]
    assert set(keys) == {"local_batch_size", "dino_local_crops_loss", "dino_local_loss_weight", "dino_global_crops_loss",
                         "koleo_loss", "ibot_loss"}
    for k in keys:
        want = float(G[f"ssl_{case}_metric/{k}"])
        assert abs(float(metrics[k]) - want) < 1e-9 * max(abs(want), 1.0), k


def test_build_schedulers_bit_exact_against_reference_function():
    """dinov3_jax.train.train.build_schedulers vs the reference's function (train/train.py:124-182) executed on its own
    default YAML with OFFICIAL_EPOCH_LENGTH=20, epochs=12, warmup 3, freeze-last-layer 1, teacher-temp warm-up 4."""
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train.train import build_schedulers
    cfg = setup_config(DinoV3SetupArgs(opts=["train.OFFICIAL_EPOCH_LENGTH=20", "optim.epochs=12", "optim.warmup_epochs=3",
                                             "optim.freeze_last_layer_epochs=1", "teacher.warmup_teacher_temp_epochs=4"]))
    for name, sc in zip(("lr", "wd", "momentum", "teacher_temp", "last_layer_lr"), build_schedulers(cfg)):
        assert np.array_equal(np.asarray(sc.schedule, dtype=np.float64), G[f"bs_{name}"]), name
        assert np.array_equal(np.array([sc[0], sc[7], sc[10 ** 6]], dtype=np.float64), G[f"bs_{name}_probe"]), name


def test_gradient_clipping_matches_reference_block():
    """train/train.py:516-541 (per top-level student submodule: g * min(1, 3 / (||g|| + 1e-6)), norm reported as
    `{module}_grad_norm`) executed from the reference text vs oracle.step.clip_by_module.  One module is above the
    threshold (scaled), one far below (untouched), one in between."""
    from oracle.step import clip_by_module
    grads = {}
    for m in ("student_backbone", "student_dino_head", "student_ibot_head"):
        flat = T(G[f"clip_in/{m}"])
        grads[f"{m}/a/kernel"], grads[f"{m}/a/bias"], grads[f"{m}/b"] = flat[:35].reshape(7, 5), flat[35:40], flat[40:]
    out, norms = clip_by_module(grads, 3.0)
    scaled = 0
    for m in ("student_backbone", "student_dino_head", "student_ibot_head"):
        got = torch.cat([out[f"{m}/a/kernel"].reshape(-1), out[f"{m}/a/bias"], out[f"{m}/b"]]).numpy()
        assert np.abs(got - G[f"clip_out/{m}"]).max() < 1e-12
        assert abs(float(norms[f"{m}_grad_norm"]) - float(G[f"clip_norm/{m}"])) < 1e-12
        scaled += int(float(G[f"clip_norm/{m}"]) > 3.0)
    assert scaled >= 1


def test_collate_data_and_cast_matches_reference_function():
    """dinov3_jax.data.collate.collate_data_and_cast vs the reference function called on the same samples / seeds:
    crop-major stacking, bf16 cast, NHWC layout, masks / flat indices / weights / counters — bit-exact."""
    from dinov3_jax.data.collate import collate_data_and_cast
    from dinov3_jax.data.masking import MaskingGenerator
    gen = torch.Generator().manual_seed(21)
    nB, gs, ls = 3, 32, 16
    samples = [({"global_crops": [torch.randn(3, gs, gs, generator=gen) for _ in range(2)],
                 "local_crops": [torch.randn(3, ls, ls, generator=gen) for _ in range(4)]}, None) for _ in range(nB)]
    random.seed(13); np.random.seed(13)
    mg = MaskingGenerator(input_size=(4, 4), max_num_patches=0.5 * 16)
    d = collate_data_and_cast(samples, (0.1, 0.5), 0.5, torch.bfloat16, n_tokens=16, mask_generator=mg)
    keys = {k.split("/", 1)[1] for k in G if k.startswith("collate/")}
    assert keys == set(d.keys())
    for k in keys:
        want = G[f"collate/{k}"]
        got = d[k]
        if torch.is_tensor(got):
            assert tuple(got.shape) == tuple(want.shape), k
            got = got.float().numpy() if got.dtype == torch.bfloat16 else got.numpy()
        assert np.array_equal(np.asarray(got), want), k
    assert d["collated_global_crops"].shape == (2 * nB, gs, gs, 3) and d["collated_global_crops"].dtype == torch.bfloat16


@pytest.mark.parametrize("n", [2, 3])
def test_shard_params_matches_reference_function(n, monkeypatch):
    """dinov3_jax.fsdp.utils.shard_params vs the reference function (fsdp/utils.py:19-53) run for every rank of an
    n-device "dp" axis: which axis is split (largest divisible; ties resolved like np.argsort(...)[::-1]), which leaves
    stay replicated (too small / no divisible axis) and the slice each rank keeps."""
    from dinov3_jax.fsdp import utils as fu
    names = ("w", "odd", "tiny", "cube/k", "cube/sq")
    tree = {"w": T(G["shard_in/w"]), "odd": T(G["shard_in/odd"]), "tiny": T(G["shard_in/tiny"]),
            "cube": {"k": T(G["shard_in/cube/k"]), "sq": T(G["shard_in/cube/sq"])}}
    for r in range(n):
        monkeypatch.setattr(fu, "_axis_index", lambda axis_name="dp", r=r: r)
        monkeypatch.setattr(fu, "_axis_size", lambda axis_name="dp": n)
        sh = fu.shard_params(tree, "dp", min_param_size=8)
        flat = {"w": sh["w"], "odd": sh["odd"], "tiny": sh["tiny"], "cube/k": sh["cube"]["k"], "cube/sq": sh["cube"]["sq"]}
        for k in names:
            want_axis = int(G[f"shard_axis/n{n}r{r}/{k}"])
            got = flat[k]
            if want_axis < 0:
                assert not isinstance(got, fu.Partitioned), k
                assert np.array_equal(got.numpy(), G[f"shard_out/n{n}r{r}/{k}"])
            else:
                assert isinstance(got, fu.Partitioned) and got.axis == want_axis, k
                assert np.array_equal(got.value.numpy(), G[f"shard_out/n{n}r{r}/{k}"]), k


def test_softmax_centering_matches_reference_code():
    """DINOLoss.softmax_center_teacher / apply_center_update (loss/dino_clstoken_loss.py:24-33,91-95): the center EMA is
    applied BEFORE the softmax of the same call; two successive calls pin the state evolution (SURVEY a27)."""
    from oracle.losses import center_update, softmax_center_teacher
    c = torch.zeros(1, G["center_logits1"].shape[1], dtype=torch.float64)
    for i, temp in ((1, 0.05), (2, 0.07)):
        x = T(G[f"center_logits{i}"])
        c = center_update(c, x, 0.9)
        assert np.abs(c.numpy() - G[f"center_state{i}"]).max() < 1e-14
        assert np.abs(softmax_center_teacher(x, c, temp).numpy() - G[f"center_probs{i}"]).max() < 1e-13


def test_gram_loss_matches_reference_code():
    """loss/gram_loss.py GramLoss (defaults: normalised features, negatives removed) per image and over the batch —
    oracle groundwork for SURVEY §8f.2; the gram teacher is not on the GPU path yet."""
    from oracle.losses import gram_loss
    s, t = T(G["gram_s"]), T(G["gram_t"])
    assert abs(float(gram_loss(s, t, img_level=True)) - float(G["gram_img"])) < 1e-14
    assert abs(float(gram_loss(s, t, img_level=False)) - float(G["gram_batch"])) < 1e-14


@pytest.mark.parametrize("n", [2, 3])
def test_ac_compile_parallelize_axes_match_reference_function(n, monkeypatch):
    """fsdp/ac_compile_parallelize.py:20-44 executed with recording stand-ins for the jax placement API: same leaves
    sharded, same axis chosen (1-D leaves never; >= 2-D leaves on the largest divisible axis, whatever their size)."""
    from dinov3_jax.fsdp import ac_compile_parallelize as acp
    from dinov3_jax.fsdp.utils import Partitioned
    tree = {"k": torch.zeros(6, 8), "bias": torch.zeros(16384), "odd": torch.zeros(3, 5), "cube": torch.zeros(4, 6, 2),
            "sq": torch.zeros(6, 6)}
    monkeypatch.setattr(acp, "_axis_index", lambda name="dp": 0)
    monkeypatch.setattr(acp, "_axis_size", lambda name="dp": n)
    out = acp.ac_compile_parallelize(tree, None, None)
    for k, v in out.items():
        want = int(G[f"acp_axis/n{n}/{k}"])
        if want < 0:
            assert not isinstance(v, Partitioned), k
        else:
            assert isinstance(v, Partitioned) and v.axis == want, k


def test_swiglu_ffn_matches_reference_class():
    """layers/ffn_layers.py SwiGLUFFN (w3(silu(w1 x) * w2 x), hidden = 2/3 * hidden_features rounded up to align_to)
    executed from the reference source vs the oracle's SwiGLU branch — groundwork for SURVEY §8f.1."""
    import torch.nn.functional as F
    x = T(G["swiglu_x"])
    w = {k.split("/", 1)[1]: T(G[k]) for k in G if k.startswith("swiglu_param/")}
    assert w["w1/kernel"].shape == (32, 64)
    y = (F.silu(x @ w["w1/kernel"] + w["w1/bias"]) * (x @ w["w2/kernel"] + w["w2/bias"])) @ w["w3/kernel"] + w["w3/bias"]
    assert np.abs(y.numpy() - G["swiglu_y"]).max() < 1e-13
    from oracle.arch import ModelCfg
    assert ModelCfg(embed_dim=20, heads=1, ffn_ratio=4.0, ffn_layer="swiglu", swiglu_align=64).swiglu_hidden == 64
