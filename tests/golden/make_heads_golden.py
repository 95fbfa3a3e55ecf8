"""Regenerate tests/golden/heads_vectors.npz by EXECUTING the reference's SSLMetaArch.__call__ (a checkout named by
$DINOV3_JAX_REFERENCE) with a DINO head and an iBOT head of different sizes: dino.head_* 48 prototypes / hidden 64 /
bottleneck 32, ibot.head_* 40 / 56 / 24.  Same mechanism as the SSLMetaArch section of make_golden.py: the reference's
train/ssl_meta_arch.py, models/vision_transformer.py and layers/dino_head.py are imported unmodified under
oracle.jaxshim (numpy float64 stand-in for jax / flax.linen), parameters and crops are closed-form
(oracle.model.formula_*), so the fixture stores only masks and results.  The iBOT head's parameters are
formula_params at the iBOT sizes (`heads_params`).

Usage:  DINOV3_JAX_REFERENCE=<checkout> python tests/golden/make_heads_golden.py
"""
from __future__ import annotations

import dataclasses
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

DINO = (48, 64, 32)          # (n_prototypes, hidden, bottleneck)
IBOT = (40, 56, 24)
# case -> (B, n_local, teacher_temp, seed, n_storage, norm_layer)
CASES = {"a": (4, 3, 0.05, 1, 0, "layernorm"), "c": (2, 4, 0.06, 3, 4, "layernormbf16")}


def heads_params(cfg, ibot, seed, dtype=None):
    """formula_params of `cfg` (DINO head at cfg's sizes) with the iBOT head's tensors at the sizes `ibot`."""
    import torch
    from oracle.model import formula_params
    dtype = dtype or torch.float64
    K, Hh, Bn = ibot
    P = formula_params(cfg, seed, dtype)
    Pi = formula_params(dataclasses.replace(cfg, n_prototypes=K, head_hidden=Hh, head_bottleneck=Bn), seed, dtype)
    P.update({k: v for k, v in Pi.items() if k.split("/", 1)[0].endswith("_ibot_head")})
    return P


def main():
    assert os.path.isdir(REF), "reference checkout not found: set DINOV3_JAX_REFERENCE"
    import yaml
    from oracle import jaxshim
    from oracle.arch import ModelCfg
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
    vt.vit_test = lambda patch_size=16, **kw: vt.DinoVisionTransformer(patch_size=patch_size, embed_dim=128, n_blocks=2,
                                                                       num_heads=2, ffn_ratio=4, **kw)

    class AD(dict):
        __getattr__ = dict.__getitem__
        __setattr__ = dict.__setitem__
    ad = lambda x: AD({k: ad(v) for k, v in x.items()}) if isinstance(x, dict) else x
    out = {"dino_dims": np.array(DINO, dtype=np.int64), "ibot_dims": np.array(IBOT, dtype=np.int64)}
    for case, (B, n_local, temp, seed, n_storage, norm) in CASES.items():
        rcfg = ad(yaml.safe_load(open(REF + "/configs/ssl_default_config.yaml")))
        rcfg.student.arch = "vit_test"
        rcfg.student.n_storage_tokens, rcfg.student.norm_layer = n_storage, norm
        rcfg.crops.global_crops_size, rcfg.crops.local_crops_size, rcfg.crops.local_crops_number = 64, 32, n_local
        for h, (K, Hh, Bn) in ((rcfg.dino, DINO), (rcfg.ibot, IBOT)):
            h.head_n_prototypes, h.head_hidden_dim, h.head_bottleneck_dim = K, Hh, Bn
        mc = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_local=n_local, n_prototypes=DINO[0],
                      head_hidden=DINO[1], head_bottleneck=DINO[2], n_storage=n_storage,
                      ln_eps=1e-5 if norm == "layernormbf16" else 1e-6)
        P = heads_params(mc, IBOT, seed)
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
    np.savez_compressed(os.path.join(HERE, "heads_vectors.npz"), **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
