"""Distillation from a frozen teacher of another architecture, host side: the teacher configuration mapping, the
reference's asserts and the rejected combinations, the parameter layouts without a qkv bias, and the distillation
oracle (tests/distill_helpers.py) against the reference's SSLMetaArch.__call__ run with `distillation.enabled`
(tests/golden/make_distill_golden.py)."""
import dataclasses
import os

import numpy as np
import pytest
import torch
import yaml

from dinov3_jax.engine.config import config_from_reference_cfg, distill_config_from_reference_cfg
from dinov3_jax.engine.params import FrozenStore, backbone_spec

# the student / dino / ibot blocks of the DINOv3 7B pretraining recipe (dinov3_vit7b16_pretrain.yaml)
VIT7B_TEACHER = {
    "student": {"arch": "vit_7b", "patch_size": 16, "drop_path_rate": 0.4, "layerscale": 1.0e-5, "ffn_layer": "swiglu64",
                "ffn_ratio": 3, "qkv_bias": False, "proj_bias": True, "ffn_bias": True, "norm_layer": "layernormbf16",
                "n_storage_tokens": 4, "untie_cls_and_patch_norms": False, "untie_global_and_local_cls_norm": True,
                "mask_k_bias": True, "in_chans": 3, "pos_embed_type": "rope", "pos_embed_rope_base": 100},
    "dino": {"loss_weight": 1.0, "head_n_prototypes": 262144, "head_bottleneck_dim": 512, "head_nlayers": 3,
             "head_hidden_dim": 8192, "koleo_loss_weight": 0.1},
    "ibot": {"loss_weight": 1.0, "separate_head": True, "head_n_prototypes": 98304, "head_bottleneck_dim": 384,
             "head_nlayers": 3, "head_hidden_dim": 4096},
    # ignored: the teacher is frozen and sees the student's crops
    "optim": {"lr": 123.0, "epochs": 7}, "crops": {"global_crops_size": 512, "local_crops_number": 2},
    "train": {"batch_size_per_gpu": 1},
}
# the distilled ViT-L/16 student's heads (dinov3_vitl16_lvd1689m_distilled.yaml)
STUDENT_OPTS = ["student.arch=vit_large", "dino.head_n_prototypes=262144", "dino.head_hidden_dim=8192",
                "dino.head_bottleneck_dim=512", "ibot.head_n_prototypes=98304", "ibot.head_hidden_dim=4096",
                "ibot.head_bottleneck_dim=384", "crops.global_crops_size=256", "crops.local_crops_size=112"]


def _setup(opts):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    return setup_config(DinoV3SetupArgs(opts=list(opts)))


def _teacher_yaml(tmp_path, **edits):
    t = yaml.safe_load(yaml.safe_dump(VIT7B_TEACHER))
    for key, val in edits.items():
        block, leaf = key.split("__")
        t.setdefault(block, {})[leaf] = val
    p = tmp_path / "teacher.yaml"
    p.write_text(yaml.safe_dump(t))
    return str(p)


def _distill_cfg(tmp_path, extra=(), **edits):
    return _setup(STUDENT_OPTS + ["distillation.enabled=true", f"distillation.full_cfg_path={_teacher_yaml(tmp_path, **edits)}"]
                  + list(extra))


def test_vit7b_teacher_mapping(tmp_path):
    cfg = _distill_cfg(tmp_path)
    t = distill_config_from_reference_cfg(cfg)
    assert (t.embed_dim, t.depth, t.heads, t.head_dim) == (4096, 40, 32, 128)
    assert (t.ffn_layer, t.swiglu_align, t.ffn_ratio, t.swiglu_hidden) == ("swiglu", 64, 3.0, 8192)
    assert t.qkv_bias is False and t.mask_k_bias is True and t.n_storage == 4 and t.ln_eps == 1e-5
    assert t.head_dims("dino_head") == (8192, 512, 262144)
    assert t.head_dims("ibot_head") == (4096, 384, 98304)
    # the teacher sees the student's crops; its own crops / optim / train blocks are ignored
    assert (t.global_size, t.local_size, t.n_local) == (256, 112, 8)


def test_without_distillation_the_student_mapping_is_unchanged(tmp_path):
    plain = _setup(STUDENT_OPTS)
    assert distill_config_from_reference_cfg(plain) is None
    s = config_from_reference_cfg(plain)
    assert config_from_reference_cfg(_distill_cfg(tmp_path)) == s
    assert s.qkv_bias is True and s == dataclasses.replace(s, qkv_bias=True)
    # the student mapping still refuses a vit_7b student without a qkv bias
    with pytest.raises(NotImplementedError):
        config_from_reference_cfg(_setup(["student.arch=vit_7b", "student.qkv_bias=false"]))


@pytest.mark.parametrize("edits", [dict(ibot__separate_head=False), dict(ibot__head_n_prototypes=65536),
                                   dict(dino__head_n_prototypes=65536), dict(student__patch_size=14)])
def test_reference_asserts_raise(tmp_path, edits):
    with pytest.raises(ValueError):
        distill_config_from_reference_cfg(_distill_cfg(tmp_path, **edits))


def test_rejected_and_accepted_teacher_options(tmp_path):
    with pytest.raises(NotImplementedError):
        distill_config_from_reference_cfg(_distill_cfg(tmp_path, student__untie_cls_and_patch_norms=True))
    with pytest.raises(NotImplementedError):
        distill_config_from_reference_cfg(_distill_cfg(tmp_path, extra=["gram.use_loss=true", "gram.ema_teacher=true"]))
    t = distill_config_from_reference_cfg(_distill_cfg(tmp_path, student__untie_global_and_local_cls_norm=True,
                                                       student__qkv_bias=False))
    assert t.qkv_bias is False
    with pytest.raises(ValueError):
        distill_config_from_reference_cfg(_setup(STUDENT_OPTS + ["distillation.enabled=true"]))    # no full_cfg_path


def test_spec_without_qkv_bias_and_frozen_layout():
    from dinov3_jax.engine.config import config_for
    c = config_for("vit_small", depth=2)
    nob = dataclasses.replace(c, qkv_bias=False)
    names = [n for n, _, _ in backbone_spec(c)]
    names_nob = [n for n, _, _ in backbone_spec(nob)]
    assert [n for n in names if not n.endswith("attn/qkv/bias")] == names_nob and len(names) == len(names_nob) + 2
    fz = FrozenStore(backbone_spec(nob), "cpu")
    assert fz.bf16.dtype == torch.bfloat16 and fz.vecs.dtype == torch.float32
    assert tuple(fz.w("blocks_1/attn/qkv/kernel").shape) == (384, 3 * 384)
    assert fz.vec("norm/bias").numel() == 384
    with pytest.raises(KeyError):          # a tree with a qkv bias does not match a teacher without one
        fz.load({n: torch.zeros(s) for n, s, _ in backbone_spec(c)}, mask_k_bias=False)


def test_engine_refuses_unsupported_distillation_setups():
    from dinov3_jax.engine import Engine
    from dinov3_jax.engine.config import config_for
    s = config_for("vit_small", depth=1)
    with pytest.raises(NotImplementedError):
        Engine(dataclasses.replace(s, qkv_bias=False), 2, device="cpu")
    with pytest.raises(NotImplementedError):
        Engine(s, 2, device="cpu", comm=object(), distill=config_for("vit_base", depth=1))
    with pytest.raises(ValueError):
        Engine(s, 2, device="cpu", distill=config_for("vit_base", depth=1, n_prototypes=1024))


# ------------------------------------------------------------------------------------------------ golden
def distill_golden():
    from conftest import GOLDEN
    with np.load(os.path.join(GOLDEN, "distill_vectors.npz")) as z:
        return {k: z[k] for k in z.files}


def distill_case(G, case, dtype=torch.float64):
    """The closed-form inputs of a distill_vectors.npz case: (student ModelCfg, teacher ModelCfg, parameters, batch,
    teacher temperature)."""
    from distill_helpers import STUDENT, STUDENT_IBOT, TEACHER, TEACHER_IBOT, distill_params
    from oracle.model import formula_images
    B, n_local, seed = (int(v) for v in G[f"ssl_{case}_spec"])
    cfg = dataclasses.replace(STUDENT, n_local=n_local)
    P = distill_params(cfg, STUDENT_IBOT, TEACHER, TEACHER_IBOT, seed, qkv_bias=False, dtype=dtype)
    masks = torch.from_numpy(G[f"ssl_{case}_masks"])
    idx = torch.from_numpy(G[f"ssl_{case}_mask_indices"])
    batch = {"collated_global_crops": formula_images((2 * B, 64, 64, 3), 100 + seed, dtype),
             "collated_local_crops": formula_images((n_local * B, 32, 32, 3), 200 + seed, dtype),
             "collated_masks": masks, "mask_indices_list": idx,
             "n_masked_patches": torch.tensor([idx.shape[0]]), "upperbound": int(idx.shape[0]), "global_batch_size": B}
    return cfg, TEACHER, P, batch, float(G[f"ssl_{case}_teacher_temp"])


@pytest.mark.parametrize("case", ["a", "b"])
def test_oracle_matches_reference_meta_arch_with_distillation(case):
    from distill_helpers import distill_ssl_forward
    G = distill_golden()
    cfg, tcfg, P, batch, temp = distill_case(G, case)
    assert "distill_backbone/blocks_0/attn/qkv/bias" not in P and "distill_backbone/storage_tokens" in P
    loss, metrics = distill_ssl_forward(P, batch, temp, cfg, tcfg, dtype=torch.float64)
    want = float(G[f"ssl_{case}_loss"])
    assert abs(float(loss) - want) < 1e-9 * abs(want)
    for k in ("dino_local_crops_loss", "dino_global_crops_loss", "koleo_loss", "ibot_loss"):
        w = float(G[f"ssl_{case}_metric/{k}"])
        assert abs(float(metrics[k]) - w) < 1e-9 * max(abs(w), 1.0), k


def test_golden_depends_on_the_distillation_semantics():
    """The plain step (EMA teacher, masked student crops) does not reproduce the fixture: it pins distillation."""
    from oracle.step import ssl_forward
    G = distill_golden()
    cfg, tcfg, P, batch, temp = distill_case(G, "a")
    loss, _ = ssl_forward(P, batch, temp, cfg, dtype=torch.float64)
    assert abs(float(loss) - float(G["ssl_a_loss"])) > 1e-3
