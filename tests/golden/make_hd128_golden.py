"""Regenerate tests/golden/hd128_vectors.npz by EXECUTING the reference's RopePositionEmbedding and DinoVisionTransformer
(a checkout named by $DINOV3_JAX_REFERENCE) at head_dim 128: embed 256, 2 heads.  Same mechanism as make_golden.py: the
reference modules are imported unmodified under oracle.jaxshim (numpy float64 stand-in for jax / flax.linen), parameters
and crops are closed-form (oracle.model.formula_*), so the fixture stores only masks and results.

The name does not match reference_vectors_*.npz on purpose: those parts are merged into one dict by tests/conftest.py.
Usage:  DINOV3_JAX_REFERENCE=<checkout> python tests/golden/make_hd128_golden.py
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF_ROOT = os.path.abspath(os.environ.get("DINOV3_JAX_REFERENCE", "dinov3-jax-reference"))
sys.path.insert(0, ROOT)

D, HEADS, DEPTH = 256, 2, 2
# case -> (n_storage, norm_layer, parameter seed, image keys)
CASES = {"r4": (4, "layernormbf16", 12, (41, 42)), "r0": (0, "layernorm", 13, (43, 44))}
ROPE_GRIDS = ((3, 5), (4, 4), (14, 14))


def main():
    assert os.path.isdir(os.path.join(REF_ROOT, "dinov3_jax")), "reference checkout not found: set DINOV3_JAX_REFERENCE"
    from oracle import jaxshim
    from oracle.arch import ModelCfg
    from oracle.model import formula_images, formula_params, sub
    jaxshim.install()
    J = lambda a: np.array(a, copy=True).view(jaxshim.Arr)
    for k in [k for k in sys.modules if k == "dinov3_jax" or k.startswith("dinov3_jax.")]:
        del sys.modules[k]
    sys.path.insert(0, REF_ROOT)
    rope = importlib.import_module("dinov3_jax.layers.rope_position_encoding")
    vt = importlib.import_module("dinov3_jax.models.vision_transformer")
    assert rope.__file__.startswith(REF_ROOT + os.sep) and vt.__file__.startswith(REF_ROOT + os.sep)
    out = {}
    for H, W in ROPE_GRIDS:
        sin, cos = rope.RopePositionEmbedding(embed_dim=D, num_heads=HEADS)(H=H, W=W)
        out[f"rope_sin_{H}x{W}"], out[f"rope_cos_{H}x{W}"] = np.asarray(sin), np.asarray(cos)
    rng = np.random.default_rng(5)
    vmask = rng.random((2, 16)) < 0.4
    out["vit_masks"] = vmask
    for case, (n_storage, norm, seed, (kg, kl)) in CASES.items():
        cfg = ModelCfg(embed_dim=D, depth=DEPTH, heads=HEADS, global_size=64, local_size=32, n_prototypes=16, head_hidden=16,
                       head_bottleneck=8, n_storage=n_storage, ln_eps=1e-5 if norm == "layernormbf16" else 1e-6)
        bp = sub(formula_params(cfg, seed), "student_backbone")
        jaxshim.PARAMS.clear(); jaxshim.PARAMS.update({k: v.numpy() for k, v in bp.items()})
        model = vt.DinoVisionTransformer(img_size=64, patch_size=16, embed_dim=D, n_blocks=DEPTH, num_heads=HEADS, ffn_ratio=4.0,
                                         qkv_bias=True, layerscale_init=0.5, norm_layer=norm, ffn_layer="mlp",
                                         n_storage_tokens=n_storage)
        g, l = formula_images((2, 64, 64, 3), kg).numpy(), formula_images((3, 32, 32, 3), kl).numpy()
        og, ol = model([J(g), J(l)], masks=[J(vmask), None], is_training=True)
        for tag, o in (("g", og), ("l", ol)):
            out[f"vit_{case}_{tag}_cls"] = np.asarray(o["x_norm_clstoken"])
            out[f"vit_{case}_{tag}_storage"] = np.asarray(o["x_storage_tokens"])
            out[f"vit_{case}_{tag}_patch"] = np.asarray(o["x_norm_patchtokens"])
    np.savez_compressed(os.path.join(HERE, "hd128_vectors.npz"), **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
