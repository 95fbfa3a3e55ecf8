"""Synthetic inputs and reference-style initialisation for benchmarks / smoke runs (product side, no oracle import).

Batches follow the reference's collate contract (data/collate.py:72-93) with masks from the mirrored generator
(`dinov3_jax.data.masking.MaskingGenerator`); parameters follow the reference initialisers (flax lecun-normal
Dense/Conv, LayerNorm ones/zeros, cls N(0, 0.02), mask_token 0, LayerScale gamma, truncated-normal(0.02) heads).
"""
from __future__ import annotations

import math
import random

import numpy as np
import torch

from ..data.collate import collate_masks
from ..data.masking import MaskingGenerator
from .config import EngineConfig
from .params import backbone_spec, head_spec


def synthetic_batch(cfg: EngineConfig, B: int, seed: int = 0, pin: bool = False) -> dict:
    random.seed(seed)
    np.random.seed(seed)
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn((cfg.n_global * B, cfg.global_size, cfg.global_size, 3), generator=gen).to(torch.bfloat16)
    l = torch.randn((cfg.n_local * B, cfg.local_size, cfg.local_size, 3), generator=gen).to(torch.bfloat16)
    grid = cfg.global_size // cfg.patch
    mg = MaskingGenerator(input_size=(grid, grid),
                          max_num_patches=0.5 * cfg.global_size // cfg.patch * cfg.global_size // cfg.patch)
    out = {"collated_global_crops": g, "collated_local_crops": l}
    out.update(collate_masks(cfg.n_global * B, grid * grid, cfg.mask_ratio, cfg.mask_probability, mg))
    out["global_batch_size"] = B
    if pin and torch.cuda.is_available():
        for k, v in out.items():
            if torch.is_tensor(v):
                out[k] = v.pin_memory()
    return out


def _trunc_normal(shape, std, lo, hi, gen):
    t = torch.empty(shape, dtype=torch.float32)
    torch.nn.init.trunc_normal_(t, mean=0.0, std=1.0, a=lo, b=hi, generator=gen)
    return t * std


def reference_like_params(cfg: EngineConfig, seed: int = 0) -> dict:
    gen = torch.Generator().manual_seed(seed)
    out = {}

    def fill(module, spec):
        for name, shape, kind in spec:
            if name.endswith("/scale"):
                t = torch.ones(shape)
            elif name.endswith("/gamma"):
                t = torch.full(shape, cfg.layerscale)
            elif name.endswith("/bias") or name == "mask_token":
                t = torch.zeros(shape)
            elif name in ("cls_token", "storage_tokens"):
                t = torch.randn(shape, generator=gen) * 0.02
            elif module == "backbone":
                fan_in = int(np.prod(shape[:-1]))
                t = _trunc_normal(shape, math.sqrt(1.0 / fan_in) / 0.87962566103423978, -2.0, 2.0, gen)
            else:
                t = _trunc_normal(shape, 0.02, -1.0, 1.0, gen)
            out[f"student_{module}/{name}"] = t
            out[f"teacher_{module}/{name}"] = t.clone()

    fill("backbone", backbone_spec(cfg))
    fill("dino_head", head_spec(cfg, "dino_head"))
    fill("ibot_head", head_spec(cfg, "ibot_head"))
    return out


def init_reference_like(engine, seed: int = 0):
    engine.params.load_reference_tree(reference_like_params(engine.cfg, seed))
