"""Regenerate tests/golden/distill_vectors.npz by EXECUTING the reference's SSLMetaArch.setup + __call__ (a checkout named
by $DINOV3_JAX_REFERENCE) with `distillation.enabled: true`.  Same mechanism as make_heads_golden.py: the reference's
train/ssl_meta_arch.py, models/ and layers/ are imported unmodified under oracle.jaxshim (numpy float64 stand-in for
jax / flax.linen), parameters and crops are closed-form (oracle.model.formula_*), so the fixture stores only masks and
results.

Only `SSLMetaArch._setup_distillation` is replaced.  The reference's own cannot run (:271 writes `self.teacher`, which
does not exist; :273-278 passes `out_dim=head_hidden_dim` and `bottlenech_dim`; :280 drops the iBOT head), so the
stand-in builds `teacher_backbone` / `teacher_dino_head` / `teacher_ibot_head` from the teacher's configuration the way
upstream DINOv3 does: `build_model_from_cfg(teacher_cfg, only_teacher=True)` and DINOHeads at the teacher's dino.* /
ibot.* sizes.  The teacher (tests/distill_helpers.TEACHER) is wider than the student, has qkv_bias: false, 4 storage
tokens against the student's 0, layernormbf16, and its own head hidden / bottleneck sizes.

Usage:  DINOV3_JAX_REFERENCE=<checkout> python tests/golden/make_distill_golden.py
"""
from __future__ import annotations

import copy
import importlib
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF_ROOT = os.path.abspath(os.environ.get("DINOV3_JAX_REFERENCE", "dinov3-jax-reference"))
REF = os.path.join(REF_ROOT, "dinov3_jax")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

# case -> (B, n_local, teacher_temp, seed)
CASES = {"a": (4, 3, 0.05, 1), "b": (2, 4, 0.06, 3)}


def main():
    assert os.path.isdir(REF), "reference checkout not found: set DINOV3_JAX_REFERENCE"
    import yaml
    from distill_helpers import STUDENT, STUDENT_IBOT, TEACHER, TEACHER_IBOT, distill_params
    from oracle import jaxshim
    from oracle.batch import collate_masks, make_mask_generator
    from oracle.model import formula_images
    jaxshim.install()
    J = lambda a: np.array(a, copy=True).view(jaxshim.Arr)
    for k in [k for k in sys.modules if k == "dinov3_jax" or k.startswith("dinov3_jax.")]:
        del sys.modules[k]
    sys.path.insert(0, REF_ROOT)
    vt = importlib.import_module("dinov3_jax.models.vision_transformer")

    def stub(name, **attrs):
        mod = types.ModuleType(name); mod.__dict__.update(attrs); sys.modules[name] = mod
    stub("omegaconf", OmegaConf=type("OmegaConf", (), {"create": staticmethod(lambda x=None: x)}), DictConfig=dict)
    stub("termcolor", colored=lambda text, *a, **k: text)
    trainpkg = types.ModuleType("dinov3_jax.train"); trainpkg.__path__ = [REF + "/train"]
    sys.modules["dinov3_jax.train"] = trainpkg
    arch_mod = importlib.import_module("dinov3_jax.train.ssl_meta_arch")
    assert arch_mod.__file__.startswith(REF_ROOT + os.sep) and vt.__file__.startswith(REF_ROOT + os.sep)
    s, t = STUDENT, TEACHER
    vt.vit_test = lambda patch_size=16, **kw: vt.DinoVisionTransformer(patch_size=patch_size, embed_dim=s.embed_dim,
                                                                       n_blocks=s.depth, num_heads=s.heads, ffn_ratio=4, **kw)
    vt.vit_test_teacher = lambda patch_size=16, **kw: vt.DinoVisionTransformer(
        patch_size=patch_size, embed_dim=t.embed_dim, n_blocks=t.depth, num_heads=t.heads, ffn_ratio=4, **kw)

    class AD(dict):
        __getattr__ = dict.__getitem__
        __setattr__ = dict.__setitem__
    ad = lambda x: AD({k: ad(v) for k, v in x.items()}) if isinstance(x, dict) else x
    default = yaml.safe_load(open(REF + "/configs/ssl_default_config.yaml"))

    def heads(c, dino, ibot):
        for h, (K, Hh, Bn) in ((c.dino, dino), (c.ibot, ibot)):
            h.head_n_prototypes, h.head_hidden_dim, h.head_bottleneck_dim = K, Hh, Bn

    tcfg = ad(copy.deepcopy(default))
    tcfg.student.arch, tcfg.student.qkv_bias = "vit_test_teacher", False
    tcfg.student.n_storage_tokens, tcfg.student.norm_layer = t.n_storage, "layernormbf16"
    heads(tcfg, (t.n_prototypes, t.head_hidden, t.head_bottleneck), TEACHER_IBOT)

    def setup_distillation(self):
        backbone, embed_dim = arch_mod.build_model_from_cfg(tcfg, only_teacher=True)
        self.teacher_backbone = backbone
        for name, h in (("teacher_dino_head", tcfg.dino), ("teacher_ibot_head", tcfg.ibot)):
            setattr(self, name, self.fsdp(arch_mod.DINOHead)(in_dim=embed_dim, out_dim=h.head_n_prototypes,
                                                             hidden_dim=h.head_hidden_dim,
                                                             bottleneck_dim=h.head_bottleneck_dim, nlayers=h.head_nlayers))
    arch_mod.SSLMetaArch._setup_distillation = setup_distillation

    out = {}
    for case, (B, n_local, temp, seed) in CASES.items():
        rcfg = ad(copy.deepcopy(default))
        rcfg.student.arch = "vit_test"
        rcfg.crops.global_crops_size, rcfg.crops.local_crops_size, rcfg.crops.local_crops_number = 64, 32, n_local
        heads(rcfg, (s.n_prototypes, s.head_hidden, s.head_bottleneck), STUDENT_IBOT)
        rcfg.distillation.enabled = True
        mc = s.__class__(**{**s.__dict__, "n_local": n_local})
        P = distill_params(mc, STUDENT_IBOT, t, TEACHER_IBOT, seed, qkv_bias=False)
        # the reference's teacher_* modules are the distillation teacher
        leaves = {k: v for k, v in P.items() if k.startswith("student_")}
        leaves.update({"teacher_" + k[len("distill_"):]: v for k, v in P.items() if k.startswith("distill_")})
        jaxshim.PARAMS.clear(); jaxshim.PARAMS.update({k: v.numpy() for k, v in leaves.items()})
        random.seed(seed); np.random.seed(seed)
        md = collate_masks(2 * B, mc.n_patches_global, mc.mask_ratio, mc.mask_probability, make_mask_generator(mc))
        data = {"collated_global_crops": J(formula_images((2 * B, 64, 64, 3), 100 + seed).numpy()),
                "collated_local_crops": J(formula_images((n_local * B, 32, 32, 3), 200 + seed).numpy()),
                "collated_masks": J(md["collated_masks"].numpy()), "mask_indices_list": J(md["mask_indices_list"].numpy()),
                "masks_weight": J(md["masks_weight"].numpy()), "n_masked_patches": J(md["n_masked_patches"].numpy()),
                "upperbound": md["upperbound"], "global_batch_size": B}
        loss, metrics = arch_mod.SSLMetaArch(rcfg)(data, teacher_temp=temp, iteration=0)
        out[f"ssl_{case}_spec"] = np.array([B, n_local, seed], dtype=np.int64)
        out[f"ssl_{case}_teacher_temp"] = np.array(temp)
        out[f"ssl_{case}_masks"] = md["collated_masks"].numpy()
        out[f"ssl_{case}_mask_indices"] = md["mask_indices_list"].numpy()
        out[f"ssl_{case}_loss"] = np.asarray(loss, dtype=np.float64)
        for k, v in metrics.items():
            out[f"ssl_{case}_metric/{k}"] = np.asarray(v, dtype=np.float64)
        print(f"distillation case {case}: loss {float(loss):.12f}", {k: float(np.asarray(v)) for k, v in metrics.items()})
    np.savez_compressed(os.path.join(HERE, "distill_vectors.npz"), **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
