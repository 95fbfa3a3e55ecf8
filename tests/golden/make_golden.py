"""Regenerate tests/golden/reference_vectors_*.npz by EXECUTING reference files from a checkout of the reference
(Dhia-naouali/dinov3-jax) named by $DINOV3_JAX_REFERENCE.

  * data/masking.py, train/cosine_lr_scheduler.py      — imported as they are (pure numpy / random)
  * data/collate.py mask section                       — re-executed with the reference MaskingGenerator
  * loss/dino_clstoken_loss.py, loss/ibot_patch_loss.py, loss/koleo_loss.py, layers/rope_position_encoding.py,
    layers/attention.py (rope_rotate_half / rope_apply), train/param_groups.py
                                                       — imported UNMODIFIED under oracle.jaxshim (numpy stand-in for
                                                         jax / flax.linen; the real stack is not installable offline)
  * models/vision_transformer.py (DinoVisionTransformer + every layer it pulls in: patch_embed, block, attention,
    ffn_layers, layer_scale, rope) and layers/dino_head.py
                                                       — imported UNMODIFIED as the package `dinov3_jax` under the shim's
                                                         mini flax.linen (Module tree / param naming / Dense / LayerNorm /
                                                         Conv / dot_product_attention restated in numpy float64) and run
                                                         on a 2-block ViT with multi-crop input + iBOT masks
  * train/ssl_meta_arch.py (SSLMetaArch.setup + __call__: teacher / student passes, head routing, iBOT row gathers,
    both Sinkhorns, loss weights and the metrics dict)  — imported UNMODIFIED under the shim; the generator stubs the
                                                         absent `omegaconf` / `termcolor` imports, registers the package
                                                         `dinov3_jax.train` without running its __init__ (that pulls
                                                         train.py -> optax / orbax), reads the reference's own
                                                         ssl_default_config.yaml with PyYAML and registers a 2-block
                                                         `vit_test` factory next to the reference's vit_* factories.
                                                         Parameters / crops are closed-form (oracle.model.formula_*),
                                                         so the fixture stores only masks and results.
  * hubconf.py: the function `setup_checkpoint` (torch-hub state-dict key mapper, :40-70) is exec'ed from its source
    text (the module body around it downloads a model) on a synthetic state dict with Meta's key names; the produced
    key list and transpose decisions pin dinov3_jax.checkpointer.convert_torch_hub_state_dict.
  * train/train.py: `build_schedulers` (:124-182) exec'ed from its source text with the reference CosineScheduler on the
    reference's default YAML (epoch length / epochs shortened).
  * train/train.py: the per-submodule gradient clipping block of train_step (:516-541, nested helpers `global_norm`,
    `clip_grads` and the loop over student submodules) exec'ed from its source text on a random gradient tree.
  * data/collate.py: `collate_data_and_cast` called as it is (crop stacking order, bf16 cast, NCHW -> NHWC, masks,
    indices, weights, dlpack hand-over through the shim).
  * fsdp/utils.py: `shard_params` (:19-53) called for every rank of a 2- and 3-device axis (axis_index / psum patched).
  * fsdp/ac_compile_parallelize.py: called with recording stand-ins for NamedSharding / PartitionSpec / device_put.
Usage:  DINOV3_JAX_REFERENCE=<checkout> python tests/golden/make_golden.py
        (writes next to this file, in parts of under 1 MB; the .npz files are committed)
"""
from __future__ import annotations

import importlib.util
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF_ROOT = os.path.abspath(os.environ.get("DINOV3_JAX_REFERENCE", "dinov3-jax-reference"))
REF = os.path.join(REF_ROOT, "dinov3_jax")
sys.path.insert(0, ROOT)


def load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    assert os.path.isdir(REF), "reference checkout not found: set DINOV3_JAX_REFERENCE"
    import torch
    from oracle.jaxshim import install, Arr
    install()
    J = lambda a: np.array(a, copy=True).view(Arr)   # inputs enter the reference code as (stand-in) jax arrays
    out = {}

    # ---- masks (reference generator + the mask section of data/collate.py:41-70)
    masking = load("ref_masking", "data/masking.py")
    for tag, (n, grid, size) in {"b8": (16, 14, 224), "tiny": (8, 4, 64)}.items():
        random.seed(7); np.random.seed(7)
        gen = masking.MaskingGenerator(input_size=(grid, grid), max_num_patches=0.5 * size // 16 * size // 16)
        N = grid * grid
        n_masked = int(n * 0.5)
        probs = torch.linspace(0.1, 0.5, n_masked + 1)
        masks, upper = [], 0
        for i in range(n_masked):
            masks.append(torch.BoolTensor(gen(int(N * probs[i + 1])))); upper += int(N * probs[i + 1])
        for _ in range(n_masked, n):
            masks.append(torch.BoolTensor(gen(0)))
        random.shuffle(masks)
        cm = torch.stack(masks).flatten(1)
        out[f"masks_{tag}"] = cm.numpy()
        out[f"mask_indices_{tag}"] = cm.flatten().nonzero().flatten().numpy()
        out[f"masks_weight_{tag}"] = (1 / cm.sum(-1).clamp(min=1.0)).unsqueeze(-1).expand_as(cm)[cm].numpy()
        out[f"upperbound_{tag}"] = np.array(upper)

    # ---- schedules
    sched = load("ref_sched", "train/cosine_lr_scheduler.py")
    out["sched_lr"] = sched.CosineScheduler(base_value=1e-3, final_value=1e-6, total_iters=500, warmup_iters=50, start_warmup_value=0).gen()
    out["sched_wd"] = sched.CosineScheduler(base_value=0.04, final_value=0.4, total_iters=500).gen()
    out["sched_temp"] = sched.CosineScheduler(base_value=0.07, final_value=0.07, total_iters=120, warmup_iters=120, start_warmup_value=0.04).gen()
    out["sched_freeze"] = sched.CosineScheduler(base_value=1.0, final_value=0.0, total_iters=60, warmup_iters=10, freeze_iters=5).gen()

    # ---- losses / rope under the shim
    rng = np.random.default_rng(0)
    dino = load("ref_dino", "loss/dino_clstoken_loss.py")
    ibot = load("ref_ibot", "loss/ibot_patch_loss.py")
    koleo = load("ref_koleo", "loss/koleo_loss.py")
    rope = load("ref_rope", "layers/rope_position_encoding.py")
    attn = load("ref_attn", "layers/attention.py")
    K, B = 48, 5
    t_logits = rng.standard_normal((2 * B, K)) * 0.3
    s_global = rng.standard_normal((2, B, K))
    s_local = rng.standard_normal((8, B, K))
    dl = dino.DINOLoss(K)
    probs = dl.sinkhorn_knopp_teacher(J(t_logits), teacher_temp=0.05)
    out.update(dino_t_logits=t_logits, dino_s_global=s_global, dino_s_local=s_local, dino_probs=np.asarray(probs),
               dino_loss_local=np.asarray(dl(J(s_local), J(probs).reshape(2, B, K))),
               dino_loss_global=np.asarray(dl(J(s_global), J(probs).reshape(2, B, K), ignore_diagonal=True)))
    # optional softmax-centering path (dino_clstoken_loss.py:24-33,91-95): two successive calls, the center is state
    crng2 = np.random.default_rng(17)
    dlc = dino.DINOLoss(K)
    c_logits1, c_logits2 = crng2.standard_normal((6, K)), crng2.standard_normal((6, K)) + 0.5
    c_p1 = np.asarray(dlc.softmax_center_teacher(J(c_logits1), 0.05))
    c_center1 = np.asarray(dlc.center.value).copy()
    c_p2 = np.asarray(dlc.softmax_center_teacher(J(c_logits2), 0.07))
    out.update(center_logits1=c_logits1, center_logits2=c_logits2, center_probs1=c_p1, center_probs2=c_p2,
               center_state1=c_center1, center_state2=np.asarray(dlc.center.value))
    # gram loss (loss/gram_loss.py:13-50; SURVEY 8f.2 — oracle groundwork only)
    gram = load("ref_gram", "loss/gram_loss.py")
    grng = np.random.default_rng(23)
    g_s, g_t = grng.standard_normal((3, 9, 16)), grng.standard_normal((3, 9, 16))
    gl = gram.GramLoss()
    out.update(gram_s=g_s, gram_t=g_t, gram_img=np.asarray(gl(J(g_s), J(g_t), img_level=True)),
               gram_batch=np.asarray(gl(J(g_s), J(g_t), img_level=False)))
    M = 11
    p_logits = rng.standard_normal((M, K)) * 0.3
    s_patch = rng.standard_normal((M, K))
    il = ibot.iBOTPatchLoss(K)
    p_probs = il.sinkhorn_knopp_teacher(J(p_logits), teacher_temp=0.05, n_masked_patches_tensor=J(np.array([M])))
    masks_flat = np.zeros((2 * B, 16), dtype=bool)
    out.update(ibot_t_logits=p_logits, ibot_s=s_patch, ibot_probs=np.asarray(p_probs),
               ibot_loss=np.asarray(il.forward_masked(J(s_patch), J(p_probs), student_masks_flat=J(masks_flat),
                                                      n_masked_patches=M, masks_weight=np.ones(M))))
    x = rng.standard_normal((7, 32))
    out.update(koleo_x=x, koleo_loss=np.asarray(koleo.KoLeoLoss()(J(x))))
    for (H, W) in ((14, 14), (6, 6), (3, 5)):
        r = rope.RopePositionEmbedding(embed_dim=384, num_heads=6)
        sin, cos = r(H=H, W=W)
        out[f"rope_sin_{H}x{W}"], out[f"rope_cos_{H}x{W}"] = np.asarray(sin), np.asarray(cos)
    xr = rng.standard_normal((2, 3, 9, 64))
    sin, cos = rope.RopePositionEmbedding(embed_dim=128, num_heads=2)(H=3, W=3)
    out.update(rope_x=xr, rope_y=np.asarray(attn.rope_apply(J(xr), J(sin), J(cos))))

    # ---- param groups (layer-wise decay etc.)
    pg = load("ref_pg", "train/param_groups.py")
    depth = 4
    tree = {"patch_embed": {"proj": {"kernel": 0, "bias": 0}}, "cls_token": 0, "mask_token": 0, "storage_tokens": 0,
            "norm": {"scale": 0, "bias": 0}}
    for i in range(depth):
        tree[f"blocks_{i}"] = {"norm1": {"scale": 0, "bias": 0}, "attn": {"qkv": {"kernel": 0, "bias": 0}, "proj": {"kernel": 0, "bias": 0}},
                               "ls1": {"gamma": 0}, "norm2": {"scale": 0, "bias": 0},
                               "mlp": {"Dense_0": {"kernel": 0, "bias": 0}, "Dense_1": {"kernel": 0, "bias": 0}}, "ls2": {"gamma": 0}}
    head = {"mlp": {f"layers_{i}": {"kernel": 0, "bias": 0} for i in (0, 2, 4)}, "last_layer": {"kernel": 0}}
    names, vals = [], []
    from flax.traverse_util import flatten_dict
    for root, t in (("student_backbone", tree), ("student_dino_head", head), ("student_ibot_head", head)):
        g = pg.get_params_groups_with_decay_fsdp(t, lr_decay_rate=0.9, patch_embed_lr_mult=0.2, dino_head_wd_multiplier=1.0, root_name=root)
        for k, v in flatten_dict(g, sep="/").items():
            names.append(f"{root}/{k}"); vals.append((v.lr_multiplier, v.wd_multiplier, float(v.is_last_layer)))
    out["pg_names"] = np.array(names)
    out["pg_values"] = np.array(vals, dtype=np.float64)

    # ---- backbone + head wiring: the reference's own module code, parameters supplied by name
    import importlib
    from oracle import jaxshim
    from oracle.arch import ModelCfg
    from oracle.model import init_params, sub
    for k in [k for k in sys.modules if k == "dinov3_jax" or k.startswith("dinov3_jax.")]:
        del sys.modules[k]
    sys.path.insert(0, REF_ROOT)
    vt = importlib.import_module("dinov3_jax.models.vision_transformer")
    dh = importlib.import_module("dinov3_jax.layers.dino_head")
    assert vt.__file__.startswith(REF_ROOT + os.sep) and dh.__file__.startswith(REF_ROOT + os.sep)
    cfg = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_prototypes=48, head_hidden=64,
                   head_bottleneck=32, layerscale=0.5)
    P = {k: v.double() for k, v in init_params(cfg, 3, perturb=0.05, dtype=torch.float32).items()}   # f32-representable
    rng = np.random.default_rng(11)
    g = rng.standard_normal((2, 64, 64, 3)).astype(np.float32).astype(np.float64)
    l = rng.standard_normal((3, 32, 32, 3)).astype(np.float32).astype(np.float64)
    vmask = rng.random((2, 16)) < 0.4
    bp = sub(P, "student_backbone")
    jaxshim.PARAMS.clear(); jaxshim.PARAMS.update({k: v.numpy() for k, v in bp.items()})
    model = vt.DinoVisionTransformer(img_size=64, patch_size=16, embed_dim=cfg.embed_dim, n_blocks=cfg.depth, num_heads=cfg.heads,
                                     ffn_ratio=cfg.ffn_ratio, qkv_bias=True, layerscale_init=cfg.layerscale,
                                     norm_layer="layernorm", ffn_layer="mlp", pos_embed_rope_base=cfg.rope_base)
    og, ol = model([J(g), J(l)], masks=[J(vmask), None], is_training=True)
    for k, v in bp.items():
        out[f"vit_param/{k}"] = v.numpy().astype(np.float32)
    out.update(vit_global=g.astype(np.float32), vit_local=l.astype(np.float32), vit_masks=vmask,
               vit_g_cls=np.asarray(og["x_norm_clstoken"]), vit_g_patch=np.asarray(og["x_norm_patchtokens"]),
               vit_l_cls=np.asarray(ol["x_norm_clstoken"]), vit_l_patch=np.asarray(ol["x_norm_patchtokens"]))
    # same network with 4 storage (register) tokens and norm_layer="layernormbf16" (eps 1e-5); closed-form parameters
    from oracle.model import formula_images, formula_params
    cfg_r = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_prototypes=48, head_hidden=64,
                     head_bottleneck=32, n_storage=4, ln_eps=1e-5)
    Pr = sub(formula_params(cfg_r, 9), "student_backbone")
    jaxshim.PARAMS.clear(); jaxshim.PARAMS.update({k: v.numpy() for k, v in Pr.items()})
    model_r = vt.DinoVisionTransformer(img_size=64, patch_size=16, embed_dim=128, n_blocks=2, num_heads=2, ffn_ratio=4.0,
                                       qkv_bias=True, layerscale_init=0.5, norm_layer="layernormbf16", ffn_layer="mlp",
                                       n_storage_tokens=4)
    gr, lr_ = formula_images((2, 64, 64, 3), 31).numpy(), formula_images((3, 32, 32, 3), 32).numpy()
    ogr, olr = model_r([J(gr), J(lr_)], masks=[J(vmask), None], is_training=True)
    out.update(vitr_g_cls=np.asarray(ogr["x_norm_clstoken"]), vitr_g_storage=np.asarray(ogr["x_storage_tokens"]),
               vitr_g_patch=np.asarray(ogr["x_norm_patchtokens"]), vitr_l_cls=np.asarray(olr["x_norm_clstoken"]),
               vitr_l_storage=np.asarray(olr["x_storage_tokens"]), vitr_l_patch=np.asarray(olr["x_norm_patchtokens"]))
    # SwiGLU FFN (layers/ffn_layers.py:52-76) called directly with explicit feature sizes (oracle groundwork, SURVEY 8f.1)
    ffn = importlib.import_module("dinov3_jax.layers.ffn_layers")
    srng2 = np.random.default_rng(41)
    sw = {"w1/kernel": srng2.standard_normal((32, 64)) * 0.2, "w1/bias": srng2.standard_normal(64) * 0.1,
          "w2/kernel": srng2.standard_normal((32, 64)) * 0.2, "w2/bias": srng2.standard_normal(64) * 0.1,
          "w3/kernel": srng2.standard_normal((64, 32)) * 0.2, "w3/bias": srng2.standard_normal(32) * 0.1}
    jaxshim.PARAMS.clear(); jaxshim.PARAMS.update(sw)
    sx = srng2.standard_normal((5, 32))
    swiglu = ffn.SwiGLUFFN(hidden_features=80, out_features=32, align_to=64)      # int(80*2/3) = 53 -> 64
    out["swiglu_x"], out["swiglu_y"] = sx, np.asarray(swiglu(J(sx)))
    for k_, v_ in sw.items():
        out[f"swiglu_param/{k_}"] = v_
    # inference entry point (is_training=False returns the head(cls) path = Identity -> x_norm_clstoken)
    hp = sub(P, "student_dino_head")
    jaxshim.PARAMS.clear(); jaxshim.PARAMS.update({k: v.numpy() for k, v in hp.items()})
    head = dh.DINOHead(in_dim=cfg.embed_dim, out_dim=cfg.n_prototypes, hidden_dim=cfg.head_hidden,
                       bottleneck_dim=cfg.head_bottleneck, nlayers=3)
    hx = rng.standard_normal((5, cfg.embed_dim)).astype(np.float32).astype(np.float64)
    for k, v in hp.items():
        out[f"head_param/{k}"] = v.numpy().astype(np.float32)
    out.update(head_x=hx.astype(np.float32), head_logits=np.asarray(head(J(hx))),
               head_bottleneck=np.asarray(head(J(hx), no_last_layer=True)))

    # ---- SSLMetaArch.__call__: the whole forward of the training step as the reference assembles it
    import types
    import yaml
    from oracle.batch import collate_masks, make_mask_generator
    from oracle.model import formula_images, formula_params

    def stub(name, **attrs):
        mod = types.ModuleType(name); mod.__dict__.update(attrs); sys.modules[name] = mod
    stub("omegaconf", OmegaConf=type("OmegaConf", (), {"create": staticmethod(lambda x=None: x)}), DictConfig=dict)
    stub("termcolor", colored=lambda text, *a, **k: text)
    trainpkg = types.ModuleType("dinov3_jax.train"); trainpkg.__path__ = [REF + "/train"]
    sys.modules["dinov3_jax.train"] = trainpkg
    arch_mod = importlib.import_module("dinov3_jax.train.ssl_meta_arch")
    assert arch_mod.__file__.startswith(REF_ROOT + os.sep)
    vt.vit_test = lambda patch_size=16, **kw: vt.DinoVisionTransformer(patch_size=patch_size, embed_dim=128, n_blocks=2,
                                                                       num_heads=2, ffn_ratio=4, **kw)

    class AD(dict):
        __getattr__ = dict.__getitem__
        __setattr__ = dict.__setitem__
    ad = lambda x: AD({k: ad(v) for k, v in x.items()}) if isinstance(x, dict) else x
    for case, (B, n_local, temp, seed, n_storage, norm) in {"a": (4, 3, 0.05, 1, 0, "layernorm"), "b": (3, 8, 0.07, 2, 0, "layernorm"),
                                                            "c": (2, 4, 0.06, 3, 4, "layernormbf16")}.items():
        rcfg = ad(yaml.safe_load(open(REF + "/configs/ssl_default_config.yaml")))
        rcfg.student.arch = "vit_test"
        rcfg.student.n_storage_tokens, rcfg.student.norm_layer = n_storage, norm      # register tokens / eps 1e-5 (§8f.1)
        rcfg.crops.global_crops_size, rcfg.crops.local_crops_size, rcfg.crops.local_crops_number = 64, 32, n_local
        for h in (rcfg.dino, rcfg.ibot):
            h.head_n_prototypes, h.head_hidden_dim, h.head_bottleneck_dim = 48, 64, 32
        mc = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_local=n_local, n_prototypes=48,
                      head_hidden=64, head_bottleneck=32, n_storage=n_storage, ln_eps=1e-5 if norm == "layernormbf16" else 1e-6)
        P = formula_params(mc, seed)
        jaxshim.PARAMS.clear(); jaxshim.PARAMS.update({k: v.numpy() for k, v in P.items()})
        random.seed(seed); np.random.seed(seed)
        md = collate_masks(2 * B, mc.n_patches_global, mc.mask_ratio, mc.mask_probability, make_mask_generator(mc))
        data = {"collated_global_crops": J(formula_images((2 * B, 64, 64, 3), 100 + seed).numpy()),
                "collated_local_crops": J(formula_images((n_local * B, 32, 32, 3), 200 + seed).numpy()),
                "collated_masks": J(md["collated_masks"].numpy()), "mask_indices_list": J(md["mask_indices_list"].numpy()),
                "masks_weight": J(md["masks_weight"].numpy()), "n_masked_patches": J(md["n_masked_patches"].numpy()),
                "upperbound": md["upperbound"], "global_batch_size": B}
        loss, metrics = arch_mod.SSLMetaArch(rcfg)(data, teacher_temp=temp, iteration=0)
        out[f"ssl_{case}_spec"] = np.array([B, n_local, seed, n_storage, int(norm == "layernormbf16")], dtype=np.int64)
        out[f"ssl_{case}_teacher_temp"] = np.array(temp)
        out[f"ssl_{case}_masks"] = md["collated_masks"].numpy()
        out[f"ssl_{case}_mask_indices"] = md["mask_indices_list"].numpy()
        out[f"ssl_{case}_loss"] = np.asarray(loss, dtype=np.float64)
        for k, v in metrics.items():
            out[f"ssl_{case}_metric/{k}"] = np.asarray(v, dtype=np.float64)
        print(f"SSLMetaArch case {case}: loss {float(loss):.12f}", {k: float(np.asarray(v)) for k, v in metrics.items()})

    # ---- torch-hub key mapping (hubconf.py:40-70)
    import re as _re
    src = open(os.path.join(REF_ROOT, "hubconf.py")).read()
    fn_src = src[src.index("def setup_checkpoint("): src.index("checkpoint = setup_checkpoint(")]
    ns = {"re": _re, "t2j": lambda x: x.detach().cpu().numpy()}
    exec(fn_src, ns)
    D, p_ = 8, 2
    sd = {"cls_token": torch.zeros(1, 1, D), "mask_token": torch.zeros(1, D), "storage_tokens": torch.zeros(1, 4, D),
          "patch_embed.proj.weight": torch.arange(D * 3 * p_ * p_, dtype=torch.float32).reshape(D, 3, p_, p_),
          "patch_embed.proj.bias": torch.zeros(D), "rope_embed.periods": torch.zeros(2),
          "norm.weight": torch.ones(D), "norm.bias": torch.zeros(D)}
    for i in range(2):
        b = f"blocks.{i}."
        sd.update({b + "norm1.weight": torch.ones(D), b + "norm1.bias": torch.zeros(D),
                   b + "attn.qkv.weight": torch.arange(3 * D * D, dtype=torch.float32).reshape(3 * D, D),
                   b + "attn.qkv.bias": torch.zeros(3 * D), b + "attn.qkv.bias_mask": torch.zeros(3 * D),
                   b + "attn.proj.weight": torch.zeros(D, D), b + "attn.proj.bias": torch.zeros(D),
                   b + "ls1.gamma": torch.ones(D), b + "norm2.weight": torch.ones(D), b + "norm2.bias": torch.zeros(D),
                   b + "mlp.fc1.weight": torch.arange(4 * D * D, dtype=torch.float32).reshape(4 * D, D),
                   b + "mlp.fc1.bias": torch.zeros(4 * D), b + "mlp.fc2.weight": torch.zeros(D, 4 * D),
                   b + "mlp.fc2.bias": torch.zeros(D), b + "ls2.gamma": torch.ones(D)})
    mapped = ns["setup_checkpoint"](sd, {})
    out["hub_torch_keys"] = np.array(sorted(sd))
    out["hub_jax_keys"] = np.array(sorted(mapped))
    out["hub_qkv_kernel_b0"] = np.asarray(mapped["blocks_0.attn.qkv.kernel"])
    out["hub_fc1_kernel_b1"] = np.asarray(mapped["blocks_1.mlp.Dense_0.kernel"])

    # ---- fsdp/utils.py shard_params (:19-53) for every rank of a 2- and a 3-device "dp" axis
    import jax as _jx
    futils = importlib.import_module("dinov3_jax.fsdp.utils")
    assert futils.__file__.startswith(REF_ROOT + os.sep)
    srng = np.random.default_rng(3)
    ptree = {"w": J(srng.standard_normal((6, 8))), "odd": J(srng.standard_normal((3, 5))), "tiny": J(srng.standard_normal(4)),
             "cube": {"k": J(srng.standard_normal((9, 6, 4))), "sq": J(srng.standard_normal((6, 6)))}}
    for k_, v_ in (("w", ptree["w"]), ("odd", ptree["odd"]), ("tiny", ptree["tiny"]), ("cube/k", ptree["cube"]["k"]), ("cube/sq", ptree["cube"]["sq"])):
        out[f"shard_in/{k_}"] = np.asarray(v_)
    keep = (_jx.lax.axis_index, _jx.lax.psum)
    for n_ in (2, 3):
        for r_ in range(n_):
            _jx.lax.axis_index, _jx.lax.psum = (lambda name, r_=r_: r_), (lambda x, name, n_=n_: x * n_)
            sh = futils.shard_params(ptree, "dp", min_param_size=8)
            for k_, v_ in (("w", sh["w"]), ("odd", sh["odd"]), ("tiny", sh["tiny"]), ("cube/k", sh["cube"]["k"]), ("cube/sq", sh["cube"]["sq"])):
                boxed = hasattr(v_, "names")
                out[f"shard_out/n{n_}r{r_}/{k_}"] = np.asarray(v_.value if boxed else v_)
                out[f"shard_axis/n{n_}r{r_}/{k_}"] = np.array(v_.names.index("dp") if boxed else -1)
    _jx.lax.axis_index, _jx.lax.psum = keep

    # ---- fsdp/ac_compile_parallelize.py (:20-44): which axis every leaf is placed on, for 2 and 3 devices
    acp = importlib.import_module("dinov3_jax.fsdp.ac_compile_parallelize")
    assert acp.__file__.startswith(REF_ROOT + os.sep)

    class _Spec:
        def __init__(self, *axes): self.axes = axes
    class _Named:
        def __init__(self, mesh, spec): self.spec = spec
    acp.NamedSharding, acp.P = _Named, _Spec
    keep_j = {k_: getattr(_jx, k_, None) for k_ in ("device_count", "make_mesh", "device_put")}
    _jx.make_mesh = lambda shape, names: None
    _jx.device_put = lambda p_, sh_: ("placed", sh_.spec.axes)
    atree = {"k": J(np.zeros((6, 8))), "bias": J(np.zeros(16384)), "odd": J(np.zeros((3, 5))), "cube": J(np.zeros((4, 6, 2))),
             "sq": J(np.zeros((6, 6)))}
    for n_ in (2, 3):
        _jx.device_count = lambda n_=n_: n_
        placed = acp.ac_compile_parallelize(atree, None, None)
        for k_, v_ in placed.items():
            axes = v_[1] if isinstance(v_, tuple) and v_[0] == "placed" else None
            out[f"acp_axis/n{n_}/{k_}"] = np.array(-1 if axes is None or "dp" not in axes else axes.index("dp"))
            out[f"acp_placed/n{n_}/{k_}"] = np.array(axes is not None)
    for k_, v_ in keep_j.items():
        if v_ is not None:
            setattr(_jx, k_, v_)

    # ---- collate_data_and_cast (data/collate.py:16-93): the reference function itself, reference mask generator,
    #      bf16 cast, NCHW -> NHWC, dlpack hand-over (the shim turns the capsule into a numpy array)
    collate = load("ref_collate", "data/collate.py")
    crng = torch.Generator().manual_seed(21)
    nB, gs, ls = 3, 32, 16
    samples = [({"global_crops": [torch.randn(3, gs, gs, generator=crng) for _ in range(2)],
                 "local_crops": [torch.randn(3, ls, ls, generator=crng) for _ in range(4)]}, None) for _ in range(nB)]
    random.seed(13); np.random.seed(13)
    cgen = masking.MaskingGenerator(input_size=(gs // 16 * 2, gs // 16 * 2), max_num_patches=0.5 * 16)
    cd = collate.collate_data_and_cast(samples, (0.1, 0.5), 0.5, torch.bfloat16, n_tokens=16, mask_generator=cgen)
    for k, v in cd.items():
        out[f"collate/{k}"] = np.asarray(v)

    # ---- build_schedulers (train/train.py:124-182): the function text is exec'ed (the module imports optax / orbax)
    tsrc = open(REF + "/train/train.py").read()
    fn_src = tsrc[tsrc.index("def build_schedulers(config):"):]
    fn_src = fn_src[: fn_src.index("\n    return (")] + "\n    return (lr_schedule, wd_schedule, momentum_schedule, teacher_temp_schedule, last_layer_lr_schedule)\n"
    import logging as _logging
    ns2 = {"CosineScheduler": sched.CosineScheduler, "logger": _logging.getLogger("dinov3")}
    exec(fn_src, ns2)
    scfg = ad(yaml.safe_load(open(REF + "/configs/ssl_default_config.yaml")))
    scfg.train.OFFICIAL_EPOCH_LENGTH = 20
    scfg.optim.epochs, scfg.optim.warmup_epochs, scfg.optim.freeze_last_layer_epochs = 12, 3, 1
    scfg.teacher.warmup_teacher_temp_epochs = 4
    scfg.pop("schedules", None)
    for nm, sc_ in zip(("lr", "wd", "momentum", "teacher_temp", "last_layer_lr"), ns2["build_schedulers"](scfg)):
        out[f"bs_{nm}"] = np.asarray(sc_.schedule, dtype=np.float64)
        out[f"bs_{nm}_probe"] = np.array([sc_[0], sc_[7], sc_[10 ** 6]], dtype=np.float64)     # __getitem__ incl. past-the-end

    # ---- per-submodule gradient clipping (train/train.py:516-541): the two nested helpers + the loop, exec'ed from text
    blk = tsrc[tsrc.index("        def global_norm(grads):"): tsrc.index("        def min_rank_1(v):")]
    import textwrap
    import jax as _jax, jax.numpy as _jnp
    crng = np.random.default_rng(5)
    gtree = {m_: {"a": {"kernel": J(crng.standard_normal((7, 5)) * s_), "bias": J(crng.standard_normal(5) * s_)},
                  "b": J(crng.standard_normal(11) * s_)}
             for m_, s_ in (("student_backbone", 2.0), ("student_dino_head", 0.05), ("student_ibot_head", 0.6))}
    flat3 = lambda t: np.concatenate([np.asarray(t["a"]["kernel"]).ravel(), np.asarray(t["a"]["bias"]).ravel(), np.asarray(t["b"]).ravel()])
    clip_inputs = {m_: flat3(gtree[m_]).copy() for m_ in gtree}        # the reference loop overwrites grads[k] in place
    ns3 = {"jnp": _jnp, "jax": _jax, "config": ad({"optim": {"clip_grad": 3.0}}), "grads": gtree,
           "student_params": {k: None for k in gtree}, "metrics_dict": {}}
    exec(textwrap.dedent(blk), ns3)
    for m_ in gtree:
        out[f"clip_in/{m_}"] = clip_inputs[m_]
        out[f"clip_out/{m_}"] = flat3(ns3["grads"][m_])
        out[f"clip_norm/{m_}"] = np.asarray(ns3["metrics_dict"][f"{m_}_grad_norm"], dtype=np.float64)
    parts, cur, size = [], {}, 0
    for k, v in out.items():                 # parts of under 1 MB (tests/conftest.py: reference_vectors)
        if cur and size + np.asarray(v).nbytes > 800_000:
            parts.append(cur); cur, size = {}, 0
        cur[k] = v; size += np.asarray(v).nbytes
    parts.append(cur)
    for i, p in enumerate(parts):
        np.savez_compressed(os.path.join(HERE, f"reference_vectors_{i}.npz"), **p)
    print("wrote", len(parts), "parts,", len(out), "arrays")


if __name__ == "__main__":
    main()
