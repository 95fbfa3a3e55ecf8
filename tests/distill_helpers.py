"""Distillation from a frozen teacher of another architecture (train/ssl_meta_arch.py:257-286), restated on the oracle's
layers and losses for the distillation tests.  The `oracle/` package is unchanged.

Parameters: `student_*` and the student-shaped EMA copy `teacher_*` as everywhere in the oracle, plus the frozen teacher
under `distill_*` at its own configuration.  The forward follows the reference's __call__ with
`distillation.enabled`: the teacher outputs come from `distill_*`, the student's global crops get no mask tokens
(:416) and the iBOT loss is still taken at `mask_indices_list` (:432).  The EMA copy is updated from the student by
oracle.step.train_step as in plain self-distillation, and is not read by the forward."""
from __future__ import annotations

import dataclasses

import torch

from oracle import step
from oracle.arch import ModelCfg
from oracle.losses import dino_loss, ibot_loss_masked, koleo_loss, sinkhorn_knopp
from oracle.model import Emu, backbone_forward, formula_params, head_forward, init_params, sub

MODULES = ("backbone", "dino_head", "ibot_head")

# the golden fixture's geometry (tests/golden/make_distill_golden.py): (prototypes, hidden, bottleneck) per head
STUDENT = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_prototypes=48, head_hidden=64,
                   head_bottleneck=32)
STUDENT_IBOT = (40, 56, 24)
TEACHER = ModelCfg(embed_dim=256, depth=2, heads=4, global_size=64, local_size=32, n_prototypes=48, head_hidden=96,
                   head_bottleneck=40, n_storage=4, ln_eps=1e-5)
TEACHER_IBOT = (40, 80, 48)


def _with_ibot(tree_fn, cfg: ModelCfg, ibot, *args, **kw) -> dict:
    """tree_fn(cfg, ...) with the iBOT head's tensors taken at the sizes `ibot` = (prototypes, hidden, bottleneck)."""
    K, Hh, Bn = ibot
    P = tree_fn(cfg, *args, **kw)
    # depth 0: the heads' leaves do not depend on the blocks, which would only be built to be dropped
    Pi = tree_fn(dataclasses.replace(cfg, depth=0, n_prototypes=K, head_hidden=Hh, head_bottleneck=Bn), *args, **kw)
    P.update({k: v for k, v in Pi.items() if k.split("/", 1)[0].endswith("_ibot_head")})
    return P


def distill_params(cfg: ModelCfg, ibot, tcfg: ModelCfg, t_ibot, seed: int, qkv_bias: bool, formula: bool = True,
                   dtype=torch.float64) -> dict:
    """student_* / teacher_* of the student, and distill_* of the frozen teacher (without attn/qkv/bias when
    `qkv_bias` is false).  formula: closed-form leaves (oracle.model.formula_params), else init_params with perturbed
    vectors."""
    if formula:
        make = lambda c, s: formula_params(c, s, dtype)
    else:
        make = lambda c, s: {k: v.to(dtype) for k, v in init_params(c, s, perturb=0.05).items()}
    P = _with_ibot(make, cfg, ibot, seed)
    T = _with_ibot(make, tcfg, t_ibot, seed + 11)
    for k, v in T.items():
        if k.startswith("teacher_") and (qkv_bias or not k.endswith("attn/qkv/bias")):
            P["distill_" + k[len("teacher_"):]] = v
    return P


def frozen_tree(params: dict) -> dict:
    """{backbone, dino_head, ibot_head} of the frozen teacher, as Engine.distill_teacher_load takes it."""
    return {m: sub(params, f"distill_{m}") for m in MODULES}


def distill_ssl_forward(params: dict, batch: dict, teacher_temp: float, cfg: ModelCfg, tcfg: ModelCfg,
                        emu: Emu = Emu(False), dtype=torch.float32, return_aux: bool = False):
    n_g, n_l = cfg.n_global, cfg.n_local
    g = batch["collated_global_crops"].to(dtype)
    l = batch["collated_local_crops"].to(dtype)
    masks, idx = batch["collated_masks"], batch["mask_indices_list"]
    B = l.shape[0] // n_l
    with torch.no_grad():
        tb = sub(params, "distill_backbone")
        for i in range(tcfg.depth):       # qkv_bias: false is a zero bias in the oracle's block
            tb.setdefault(f"blocks_{i}/attn/qkv/bias", torch.zeros(3 * tcfg.embed_dim, dtype=dtype))
        t_out = backbone_forward(tb, [g], [None], tcfg, emu)[0]
        t_cls, t_patch = t_out["x_norm_clstoken"], t_out["x_norm_patchtokens"]
        t_patch_logits = head_forward(sub(params, "distill_ibot_head"), t_patch.reshape(-1, t_patch.shape[-1])[idx], emu)
        t_cls_logits = head_forward(sub(params, "distill_dino_head"), t_cls, emu)
        cls_centered = sinkhorn_knopp(t_cls_logits, teacher_temp, B_total=t_cls_logits.shape[0]).reshape(n_g, B, -1)
        n_masked = batch["n_masked_patches"].sum().to(dtype)
        patch_centered = sinkhorn_knopp(t_patch_logits, teacher_temp, B_total=n_masked)
    s_g, s_l = backbone_forward(sub(params, "student_backbone"), [g, l], [None, None], cfg, emu)      # :416
    g_cls, g_patch, l_cls = s_g["x_norm_clstoken"], s_g["x_norm_patchtokens"], s_l["x_norm_clstoken"]
    s_patch_logits = head_forward(sub(params, "student_ibot_head"), g_patch.reshape(-1, g_patch.shape[-1])[idx], emu)
    buf = head_forward(sub(params, "student_dino_head"), torch.cat([g_cls, l_cls], dim=0), emu)
    s_g_logits = buf[: g_cls.shape[0]].reshape(n_g, B, -1)
    s_l_logits = buf[g_cls.shape[0]:].reshape(n_l, B, -1)
    g_terms, l_terms = n_g * (n_g - 1), n_g * n_l
    g_scale, l_scale = g_terms / (g_terms + l_terms), l_terms / (g_terms + l_terms)
    L_local = dino_loss(s_l_logits, cls_centered, cfg.student_temp, ignore_diagonal=False)
    L_global = dino_loss(s_g_logits, cls_centered, cfg.student_temp, ignore_diagonal=True)
    L_koleo = sum(koleo_loss(x) for x in g_cls.reshape(n_g, B, -1)) / n_g
    L_ibot = ibot_loss_masked(s_patch_logits, patch_centered, cfg.student_temp, n_mask_rows=masks.shape[0])
    loss = (cfg.dino_loss_weight * l_scale * L_local + cfg.dino_loss_weight * g_scale * L_global
            + cfg.koleo_loss_weight * n_g * L_koleo + cfg.ibot_loss_weight * L_ibot)
    metrics = {"dino_local_crops_loss": L_local.detach(), "dino_global_crops_loss": L_global.detach(),
               "koleo_loss": L_koleo.detach(), "ibot_loss": L_ibot.detach()}
    if return_aux:
        return loss, metrics, {"t_cls_logits": t_cls_logits, "t_patch_logits": t_patch_logits}
    return loss, metrics


def distill_train_step(params: dict, opt_state: dict, batch: dict, cfg: ModelCfg, tcfg: ModelCfg, **kw):
    """oracle.step.train_step (gradient, clip, AdamW, EMA into teacher_*) around distill_ssl_forward.  The frozen
    distill_* tensors are carried through unchanged: train_step differentiates and updates student_* only."""
    plain = step.ssl_forward
    step.ssl_forward = lambda full, b, temp, c, emu, dtype: distill_ssl_forward(full, b, temp, c, tcfg, emu, dtype=dtype)
    try:
        return step.train_step(params, opt_state, batch, cfg, **kw)
    finally:
        step.ssl_forward = plain
