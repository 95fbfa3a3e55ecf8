"""Batch collation with the reference's dict contract (dinov3_jax/data/collate.py:16-93), torch tensors out.

The reference converts to jax arrays through dlpack (:85-91); the GPU engine consumes the torch tensors directly
(NHWC, `compute_precision.param_dtype`), so that conversion is dropped — everything else keeps its key and meaning.
"""
from __future__ import annotations

import random

import torch


def collate_masks(n_crops: int, n_tokens: int, mask_ratio_tuple, mask_probability: float, mask_generator,
                  random_circular_shift: bool = False) -> dict:
    """Mask part of the collate (reference :41-70): the first int(n*p) crops get a growing masked fraction from
    linspace(*ratio), the rest none; the list is shuffled; flat indices / weights are derived from it."""
    n_masked = int(n_crops * mask_probability)
    fractions = torch.linspace(*mask_ratio_tuple, n_masked + 1)[1:]
    masks, upperbound = [], 0
    for frac in fractions:
        count = int(n_tokens * frac)
        m = torch.BoolTensor(mask_generator(count))
        if random_circular_shift:
            m = torch.roll(m, (random.randint(0, m.shape[0] - 1), random.randint(0, m.shape[1] - 1)), (0, 1))
        masks.append(m)
        upperbound += count
    masks.extend(torch.BoolTensor(mask_generator(0)) for _ in range(n_crops - n_masked))
    random.shuffle(masks)
    collated = torch.stack(masks).flatten(1)
    indices = collated.flatten().nonzero().flatten()
    per_crop = collated.sum(-1).clamp(min=1.0)
    weights = (1 / per_crop).unsqueeze(-1).expand_as(collated)[collated]
    return {"collated_masks": collated, "mask_indices_list": indices, "masks_weight": weights, "upperbound": upperbound,
            "n_masked_patches": torch.full((1,), indices.shape[0], dtype=torch.long)}


def collate_data_and_cast(samples_list, mask_ratio_tuple, mask_probability, dtype, n_tokens=None, mask_generator=None,
                          random_circular_shift=False, local_batch_size=None):
    """Same signature as the reference.  samples_list[i][0] is the dict produced by the DINO augmentation
    ({"global_crops": [CHW tensors], "local_crops": [...]}); crops are stacked crop-major and emitted NHWC."""
    first = samples_list[0][0]
    n_g, n_l = len(first["global_crops"]), len(first["local_crops"])
    stack = lambda key, n: torch.stack([s[0][key][i] for i in range(n) for s in samples_list])
    g, l = stack("global_crops", n_g), stack("local_crops", n_l)
    n_for_masks = n_g * local_batch_size if local_batch_size is not None else len(g)
    out = {"collated_global_crops": g.to(dtype), "collated_local_crops": l.to(dtype)}
    if "gram_teacher_crops" in first:
        out["collated_gram_teacher_crops"] = stack("gram_teacher_crops", n_g).to(dtype)
    out.update(collate_masks(n_for_masks, n_tokens, mask_ratio_tuple, mask_probability, mask_generator,
                             random_circular_shift))
    for k, v in list(out.items()):
        if torch.is_tensor(v) and v.dim() >= 3:
            out[k] = torch.movedim(v, -3, -1).contiguous()   # NCHW -> NHWC (reference :89)
    return out
