"""CPU: checkpoint / weight-format adapter (SURVEY §8f.4) — pytree <-> disk round trip with the reference's call
signatures, retention helpers, and the torch-hub key map pinned against the reference's hubconf mapper output."""
import os

import numpy as np
import pytest
import torch

from conftest import reference_vectors

G = reference_vectors()


def _hub_state_dict(D=8, p=2):
    sd = {"cls_token": torch.zeros(1, 1, D), "mask_token": torch.zeros(1, D), "storage_tokens": torch.zeros(1, 4, D),
          "patch_embed.proj.weight": torch.arange(D * 3 * p * p, dtype=torch.float32).reshape(D, 3, p, p),
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
    return sd


def test_torch_hub_key_map_matches_reference_mapper():
    from dinov3_jax.checkpointer import convert_torch_hub_state_dict, flat_from_tree, to_torch_hub_state_dict
    sd = _hub_state_dict()
    assert sorted(sd) == list(G["hub_torch_keys"])                       # same synthetic input as the generator
    params, consts = convert_torch_hub_state_dict(sd)
    flat = flat_from_tree(params, sep=".")
    flat.update({"rope_embed." + k: v for k, v in flat_from_tree(consts.get("rope_embed", {}), sep=".").items()})
    assert sorted(flat) == list(G["hub_jax_keys"])                       # names produced by hubconf.py's mapper
    assert np.array_equal(flat["blocks_0.attn.qkv.kernel"].numpy(), G["hub_qkv_kernel_b0"])     # [in, out] = weight.T
    assert np.array_equal(flat["blocks_1.mlp.Dense_0.kernel"].numpy(), G["hub_fc1_kernel_b1"])
    # conv kernel: flax layout [p_h, p_w, 3, D] (the reference's `.T` would swap the two spatial axes; intent followed)
    w = sd["patch_embed.proj.weight"]
    assert torch.equal(flat["patch_embed.proj.kernel"], w.permute(2, 3, 1, 0))
    back = to_torch_hub_state_dict(params)
    for k, v in sd.items():
        if "bias_mask" in k or k.startswith("rope_embed"):
            continue
        assert torch.equal(back[k], v), k


def test_save_load_round_trip_and_strictness(tmp_path):
    from dinov3_jax.checkpointer import (CheckpointRetentionPolicy, cleanup_checkpoint, find_latest_checkpoint,
                                        keep_last_n_checkpoints, load_checkpoint, save_checkpoint, tree_from_flat)
    from oracle import tiny_cfg
    from oracle.model import init_params
    P = init_params(tiny_cfg(), 0, perturb=0.05)
    params = tree_from_flat(P)
    opt = {"count": 7, "mu": tree_from_flat({k: v * 0.1 for k, v in P.items() if k.startswith("student_")}),
           "nu": tree_from_flat({k: v * v for k, v in P.items() if k.startswith("student_")})}
    for it in (10, 20, 30):
        save_checkpoint(tmp_path / str(it), iteration=it, params=params, optimizer_state=opt, teacher_temp=0.05)
    assert find_latest_checkpoint(tmp_path).name == "30"
    ck = load_checkpoint(tmp_path / "30", abstract_model_params=params, abstract_optimizer_state=opt)
    assert ck["iteration"] == 30 and ck["optimizer_state"]["count"] == 7 and ck["teacher_temp"] == 0.05
    for k, v in P.items():
        cur = ck["model_params"]
        for part in k.split("/"):
            cur = cur[part]
        assert torch.equal(cur, v)
    with pytest.raises(RuntimeError):
        save_checkpoint(tmp_path / "30", iteration=30, params=params, optimizer_state=None, overwrite=False)
    bad = tree_from_flat({**P, "student_backbone/extra": torch.zeros(3)})
    with pytest.raises(ValueError):
        load_checkpoint(tmp_path / "30", abstract_model_params=bad, abstract_optimizer_state=None)
    load_checkpoint(tmp_path / "30", abstract_model_params=bad, abstract_optimizer_state=None, strict_loading=False)
    keep_last_n_checkpoints(tmp_path, 2)
    assert sorted(p.name for p in tmp_path.iterdir()) == ["20", "30"]
    save_checkpoint(tmp_path / "final", iteration=30, params={"a": torch.ones(2)}, optimizer_state=None)
    cleanup_checkpoint(tmp_path, CheckpointRetentionPolicy.LAST)
    assert sorted(p.name for p in tmp_path.iterdir()) == ["final"]
