"""Model factories with the reference's names (dinov3_jax/models/__init__.py:17-72, vision_transformer.py:325-408).
On the GPU path a "model" is its static description (EngineConfig); parameters live in the engine's flat buffers."""
from __future__ import annotations

from dataclasses import replace

from ..engine.config import ARCHS, EngineConfig, config_for, config_from_reference_cfg
from .vision_transformer import DinoVisionTransformer


def _factory(name):
    def make(patch_size: int = 16, **kw) -> EngineConfig:
        return replace(config_for(name, patch=patch_size), **{k: v for k, v in kw.items() if k in EngineConfig.__dataclass_fields__})
    make.__name__ = name
    return make


vit_small, vit_base, vit_large = _factory("vit_small"), _factory("vit_base"), _factory("vit_large")
vit_so400m, vit_huge2, vit_giant2 = _factory("vit_so400m"), _factory("vit_huge2"), _factory("vit_giant2")


def build_model(args, only_teacher: bool = False, img_size: int = 224):
    """models/__init__.py:17-55: returns (student, teacher, embed_dim) — here two (equal) static descriptions."""
    if args.arch not in ARCHS:
        raise ValueError(f"unknown arch {args.arch!r} (ConvNeXt and vit_7b are not on the GPU path)")
    cfg = config_for(args.arch, patch=args.patch_size)
    if only_teacher:
        return cfg, cfg.embed_dim
    return cfg, cfg, cfg.embed_dim


def build_model_from_cfg(cfg, only_teacher: bool = False):
    e = config_from_reference_cfg(cfg)
    if only_teacher:
        return e, e.embed_dim
    return e, e, e.embed_dim
