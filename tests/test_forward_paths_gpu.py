"""-m gpu: the training engine and the feature model run one forward (engine/forward.py), so they agree bit for bit.

  (a) the engine's teacher pass (final-norm output and last block output) against DinoVisionTransformer.forward_features
      on the same global crops, with the teacher tree from export_reference_tree: an mlp block; swiglu64 + mask_k_bias
      + 4 storage tokens + layernormbf16; head_dim 128;
  (b) layers.DINOHead on the teacher's DINO-head inputs against the engine's teacher logits;
  (c) a distillation teacher without a qkv bias and of another width against the model built from its tree.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

CASES = {
    "mlp": dict(embed_dim=128, heads=2),
    "swiglu64_mask_k_bias_storage_ln_bf16": dict(embed_dim=128, heads=2, ffn_layer="swiglu", swiglu_align=64,
                                                 mask_k_bias=True, n_storage=4, ln_eps=1e-5),
    "head_dim_128": dict(embed_dim=256, heads=2),
}


def _cfg(**kw):
    from oracle.arch import ModelCfg
    base = dict(depth=2, global_size=64, local_size=32, n_local=2, n_prototypes=96, head_hidden=64, head_bottleneck=32,
                layerscale=0.5)
    return ModelCfg(**{**base, **kw})


def _model(cfg, tree):
    from dinov3_jax.models import DinoVisionTransformer
    ffn = "mlp" if cfg.ffn_layer == "mlp" else f"swiglu{cfg.swiglu_align if cfg.swiglu_align > 8 else ''}"
    return DinoVisionTransformer(tree, img_size=cfg.global_size, patch_size=cfg.patch, embed_dim=cfg.embed_dim,
                                 n_blocks=cfg.depth, num_heads=cfg.heads, ffn_ratio=cfg.ffn_ratio,
                                 n_storage_tokens=cfg.n_storage, mask_k_bias=cfg.mask_k_bias, ffn_layer=ffn,
                                 norm_layer="layernormbf16" if cfg.ln_eps == 1e-5 else "layernorm")


def _check_teacher_pass(eng, model, images):
    """The engine's teacher stream after teacher_pass against model.forward_features(images), bit for bit."""
    st = eng.teacher
    cs = st.sets[0]
    n, N, D = cs.n, cs.N, eng.t_net.cfg.embed_dim
    out = model.forward_features(images)
    R = model.n_storage_tokens
    Xn = st.Xn.view(n, N, D)
    assert torch.equal(out["x_norm_clstoken"], Xn[:, 0])
    assert torch.equal(out["x_storage_tokens"], Xn[:, 1:1 + R])
    assert torch.equal(out["x_norm_patchtokens"], Xn[:, 1 + R:])
    assert torch.equal(out["x_prenorm"], st.x_in(eng.t_net.cfg.depth).view(n, N, D))


@pytest.mark.parametrize("case", list(CASES))
def test_teacher_pass_equals_feature_model_and_head(native, case):
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from dinov3_jax.layers import DINOHead
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg = _cfg(**CASES[case])
    B = 3
    batch = synthetic_batch(cfg, B, 0)
    eng = Engine(from_oracle_cfg(cfg), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    eng.params.load_reference_tree(init_params(cfg, 0, perturb=0.05))
    eng.set_batch(batch)
    eng.teacher_pass(0.05)
    tree = eng.params.export_reference_tree()
    sub = lambda pre: {k[len(pre):]: v for k, v in tree.items() if k.startswith(pre)}
    _check_teacher_pass(eng, _model(cfg, sub("teacher_backbone/")), batch["collated_global_crops"])
    ng = cfg.n_global * B
    head = DINOHead(sub("teacher_dino_head/"), in_dim=cfg.embed_dim, out_dim=cfg.n_prototypes, hidden_dim=cfg.head_hidden,
                    bottleneck_dim=cfg.head_bottleneck)
    hb = eng.h_t_dino
    assert torch.equal(head(hb.A0[:ng]), hb.logits[:ng])
    assert torch.equal(head(hb.A0[:ng], no_last_layer=True), hb.Yn[:ng])


def test_distillation_teacher_without_qkv_bias_equals_feature_model(native):
    import dataclasses

    from dinov3_jax.engine import Engine, from_oracle_cfg
    from distill_helpers import STUDENT, STUDENT_IBOT, TEACHER, TEACHER_IBOT, distill_params, frozen_tree
    from oracle.batch import synthetic_batch
    ecfg = lambda c, ibot, qkv_bias=True: dataclasses.replace(from_oracle_cfg(c), ibot_n_prototypes=ibot[0],
                                                              ibot_head_hidden=ibot[1], ibot_head_bottleneck=ibot[2],
                                                              qkv_bias=qkv_bias)
    B = 2
    P = distill_params(STUDENT, STUDENT_IBOT, TEACHER, TEACHER_IBOT, 0, qkv_bias=False, formula=False)
    batch = synthetic_batch(STUDENT, B, 0)
    eng = Engine(ecfg(STUDENT, STUDENT_IBOT), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1),
                 distill=ecfg(TEACHER, TEACHER_IBOT, qkv_bias=False))
    eng.params.load_reference_tree({k: v.float() for k, v in P.items() if not k.startswith("distill_")})
    teacher = frozen_tree(P)
    eng.distill_teacher_load(teacher)
    eng.set_batch(batch)
    eng.teacher_pass(0.05)
    assert TEACHER.embed_dim != STUDENT.embed_dim and not any(k.endswith("qkv/bias") for k in teacher["backbone"])
    _check_teacher_pass(eng, _model(TEACHER, teacher["backbone"]), batch["collated_global_crops"])
