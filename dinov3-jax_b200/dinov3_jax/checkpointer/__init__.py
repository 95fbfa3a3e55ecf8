"""Checkpoint / weight-format adapter (SURVEY §8f.4): the engine's flat fp32 / bf16 buffers <-> the reference's named
parameter pytree, on-disk save / load with the reference's call signatures, and the torch-hub name map.

Reference interface mirrored here (dinov3_jax/checkpointer/checkpointer.py): `CheckpointRetentionPolicy` (:22-48),
`find_all_checkpoints` / `find_latest_checkpoint` (:61-76), `keep_last_n_checkpoints` (:79-91), `cleanup_checkpoint`
(:100-118), `save_checkpoint(ckpt_dir, *, iteration, params, optimizer_state, overwrite=True, **others)` (:122-152),
`load_checkpoint(ckpt_dir, *, abstract_model_params, abstract_optimizer_state, strict_loading=True, **others)`
(:157-184).  The reference serialises with orbax (not installable here, and its own call sites pass mismatching
keyword names, SURVEY A11); this adapter keeps the *pytree contract* — nested dicts whose leaves carry the reference's
names and layouts (`kernel` [in, out], conv kernel [p, p, 3, D], `scale`/`bias`/`gamma` vectors) — and stores it as one
`.npy` per leaf plus a JSON manifest, so a checkpoint is readable with numpy alone.

`convert_torch_hub_state_dict` restates the key mapping of the reference's hubconf.py:40-74 (Meta's PyTorch DINOv3
backbone state dict -> this tree): `weight` -> `scale` for norms, -> `kernel` (transposed) for linear layers,
`fc{n}` -> `Dense_{n-1}`, `blocks.{i}` -> `blocks_{i}`, conv weight [D,3,p,p] -> [p,p,3,D], `qkv.bias_mask` dropped,
`rope_embed.periods` split off as a constant.
"""
from __future__ import annotations

import json
import re
import shutil
from enum import Enum
from pathlib import Path

import numpy as np
import torch


class CheckpointRetentionPolicy(Enum):
    ALL = "all"
    BEST = "best"
    LAST = "last"
    LAST_AND_BEST = "last_and_best"
    NONE = "none"

    @property
    def keep_filters(self):
        return {CheckpointRetentionPolicy.LAST: {"final"}, CheckpointRetentionPolicy.BEST: {"best"},
                CheckpointRetentionPolicy.LAST_AND_BEST: {"final", "best"}}.get(self, set())

    @property
    def max_to_keep(self):
        return None if self == CheckpointRetentionPolicy.ALL else 1


def _is_int(s: str) -> bool:
    try:
        int(s)
        return True
    except ValueError:
        return False


def find_all_checkpoints(ckpt_dir):
    ckpt_dir = Path(ckpt_dir)
    if not ckpt_dir.is_dir():
        return []
    return sorted((p for p in ckpt_dir.iterdir() if p.is_dir() and _is_int(p.name)), key=lambda p: int(p.name))


def find_latest_checkpoint(ckpt_dir):
    cps = find_all_checkpoints(ckpt_dir)
    return cps[-1] if cps else None


def keep_last_n_checkpoints(ckpt_dir, n):
    """Intent of checkpointer.py:79-91 (the reference compares the directory with its own children and never deletes):
    remove all but the n newest step directories."""
    if n is None:
        return
    for p in find_all_checkpoints(ckpt_dir)[:-n] if n > 0 else find_all_checkpoints(ckpt_dir):
        shutil.rmtree(p, ignore_errors=True)


def keep_checkpoint_copy(src):
    src = Path(src)
    dst = src.parent / f"{src.name}_keep"
    if dst.exists():                  # re-saving the same iteration after a resume: replace the kept copy
        shutil.rmtree(dst)
    shutil.copytree(src, dst, copy_function=lambda a, b: (Path(b).hardlink_to(a) if not Path(b).exists() else None))
    return dst


def cleanup_checkpoint(ckpt_dir, checkpoint_retention_policy: CheckpointRetentionPolicy):
    """checkpointer.py:100-118 with the filter applied to directory *names* (the reference compares Path to str)."""
    ckpt_dir = Path(ckpt_dir)
    if not ckpt_dir.is_dir():
        return []
    keep = checkpoint_retention_policy.keep_filters
    removed = []
    for p in ckpt_dir.iterdir():
        if p.is_dir() and p.name not in keep and not p.name.endswith("_keep"):
            shutil.rmtree(p, ignore_errors=True)
            removed.append(p)
    return removed


# ------------------------------------------------------------------------------------------------------- pytrees
def tree_from_flat(flat: dict, sep: str = "/") -> dict:
    out = {}
    for k, v in flat.items():
        cur = out
        parts = k.split(sep)
        for p in parts[:-1]:
            cur = cur.setdefault(p, {})
        cur[parts[-1]] = v
    return out


def flat_from_tree(tree: dict, sep: str = "/", _pre: str = "") -> dict:
    out = {}
    for k, v in tree.items():
        key = f"{_pre}{sep}{k}" if _pre else str(k)
        if isinstance(v, dict):
            out.update(flat_from_tree(v, sep, key))
        else:
            out[key] = v
    return out


def _to_numpy(v):
    if torch.is_tensor(v):
        v = v.detach().cpu()
        return v.float().numpy() if v.dtype == torch.bfloat16 else v.numpy()
    return np.asarray(v)


def save_checkpoint(ckpt_dir, *, iteration, params, optimizer_state=None, overwrite: bool = True, **others):
    """Write {iteration, model_params, optimizer_state, **others} under ckpt_dir (one .npy per leaf + manifest.json)."""
    ckpt_dir = Path(ckpt_dir).absolute()
    if ckpt_dir.exists() and not overwrite:
        raise RuntimeError(f"Checkpoint already exists: {ckpt_dir}")
    tmp = ckpt_dir.with_name(ckpt_dir.name + ".partial")
    if tmp.exists():
        shutil.rmtree(tmp)
    tmp.mkdir(parents=True)
    state = {"model_params": params}
    if optimizer_state is not None:
        state["optimizer_state"] = optimizer_state
    state.update(others)
    manifest = {"iteration": int(iteration) if _is_int(str(iteration)) else str(iteration), "leaves": {}, "scalars": {}}
    for i, (key, leaf) in enumerate(sorted(flat_from_tree(state).items())):
        if isinstance(leaf, (int, float, str, bool)) or leaf is None:
            manifest["scalars"][key] = leaf
            continue
        arr = _to_numpy(leaf)
        fname = f"leaf_{i:05d}.npy"
        np.save(tmp / fname, arr, allow_pickle=False)
        manifest["leaves"][key] = {"file": fname, "shape": list(arr.shape), "dtype": str(arr.dtype)}
    (tmp / "manifest.json").write_text(json.dumps(manifest, indent=1))
    # swap: the new checkpoint is complete on disk before the old one goes away, so a crash at any point leaves
    # either the old or the new checkpoint (never neither) under a name find_latest_checkpoint accepts
    old = ckpt_dir.with_name(ckpt_dir.name + ".old")
    if old.exists():
        shutil.rmtree(old) if old.is_dir() else old.unlink()
    if ckpt_dir.exists():
        ckpt_dir.rename(old)
    tmp.rename(ckpt_dir)
    if old.exists():
        shutil.rmtree(old) if old.is_dir() else old.unlink()
    return ckpt_dir


def load_checkpoint(ckpt_dir, *, abstract_model_params=None, abstract_optimizer_state=None, strict_loading: bool = True,
                    **others) -> dict:
    """Read a checkpoint written by save_checkpoint.  The `abstract_*` trees (any nested dict with the expected leaf
    names; leaves may be shapes, tensors or None) are validated against the stored leaves when given: missing or
    shape-mismatching entries raise under strict_loading, are skipped otherwise."""
    ckpt_dir = Path(ckpt_dir).absolute()
    manifest = json.loads((ckpt_dir / "manifest.json").read_text())
    flat = {k: torch.from_numpy(np.load(ckpt_dir / v["file"], allow_pickle=False)) for k, v in manifest["leaves"].items()}
    flat.update(manifest["scalars"])
    expect = {}
    if abstract_model_params is not None:
        expect.update({f"model_params/{k}": v for k, v in flat_from_tree(abstract_model_params).items()})
    if abstract_optimizer_state is not None:
        expect.update({f"optimizer_state/{k}": v for k, v in flat_from_tree(abstract_optimizer_state).items()})
    for name, tree in others.items():
        if isinstance(tree, dict):
            expect.update({f"{name}/{k}": v for k, v in flat_from_tree(tree).items()})
    problems = []
    for k, want in expect.items():
        if k not in flat:
            problems.append(f"missing leaf {k}")
            continue
        shape = tuple(want) if isinstance(want, (tuple, list)) else (tuple(want.shape) if hasattr(want, "shape") else None)
        if shape is not None and torch.is_tensor(flat[k]) and tuple(flat[k].shape) != shape:
            problems.append(f"shape of {k}: stored {tuple(flat[k].shape)} != expected {shape}")
            flat.pop(k)
    if problems and strict_loading:
        raise ValueError("checkpoint does not match the abstract trees:\n  " + "\n  ".join(problems))
    out = tree_from_flat(flat)
    out["iteration"] = manifest["iteration"]
    return out


# ------------------------------------------------------------------------------------------------ engine <-> pytree
def engine_state(engine) -> dict:
    """(params tree, optimizer-state tree) of a dinov3_jax.engine.Engine with the reference's names: params has the six
    top-level modules (train/ssl_meta_arch.py:62-64,86-87,130-131); the optimizer state mirrors optax.adamw's
    (count, mu, nu) over the student modules (train/train.py:95-106).  Under FSDP every rank calls this (collective
    all-gathers of the shards); rank 0 writes."""
    flat = {k: v.cpu() for k, v in engine.params.export_reference_tree("param").items()}
    gram_params, gram_opt = engine.gram_state()
    flat.update(gram_params)              # the frozen gram teacher (SURVEY 8f.2)
    params = tree_from_flat(flat)
    mu = tree_from_flat({k: v.cpu() for k, v in engine.params.export_reference_tree("m").items()})
    nu = tree_from_flat({k: v.cpu() for k, v in engine.params.export_reference_tree("v").items()})
    opt = {"count": int(engine.step_count), "mu": mu, "nu": nu, **gram_opt}
    if getattr(engine, "centering", "sinkhorn_knopp") != "sinkhorn_knopp":
        # "state" collection of the optional softmax-centering path (loss/dino_clstoken_loss.py:19-22)
        opt["centers"] = {"dino": engine.center_dino.cpu(), "ibot": engine.center_ibot.cpu()}
    return params, opt


def load_engine_state(engine, params: dict, optimizer_state: dict | None = None):
    flat = flat_from_tree(params)
    engine.params.load_reference_tree(flat)
    engine.gram_load_state(flat, optimizer_state)
    if optimizer_state is not None:
        engine.step_count = int(optimizer_state["count"])
        engine.params.load_optimizer_tree(flat_from_tree(optimizer_state["mu"]), flat_from_tree(optimizer_state["nu"]))
        if "centers" in optimizer_state and hasattr(engine, "center_dino"):
            engine.center_dino.copy_(optimizer_state["centers"]["dino"])
            engine.center_ibot.copy_(optimizer_state["centers"]["ibot"])


# ------------------------------------------------------------------------------------------------ torch hub weights
def convert_torch_hub_state_dict(state_dict: dict) -> tuple:
    """Meta's PyTorch DINOv3 ViT backbone state dict -> (backbone params tree, constants tree), hubconf.py:40-74.

    Linear `weight` [out, in] -> `kernel` [in, out]; norm `weight` -> `scale`; `mlp.fc1/fc2` -> `mlp/Dense_0/Dense_1`;
    `blocks.i.` -> `blocks_i/`; `patch_embed.proj.weight` [D, 3, p, p] -> `kernel` [p, p, 3, D] (flax Conv layout,
    layers/patch_embed.py:38-42); `attn.qkv.bias_mask` dropped (the reference keeps the plain bias, hubconf.py:33-36);
    `rope_embed.periods` goes to the constants collection (layers/rope_position_encoding.py:48)."""
    params, consts = {}, {}
    for tk, v in state_dict.items():
        if "bias_mask" in tk:
            continue
        v = v.detach().cpu() if torch.is_tensor(v) else torch.as_tensor(v)
        parts = tk.split(".")
        transpose = False
        if parts[-1] == "weight":
            if "norm" in parts[-2]:
                parts[-1] = "scale"
            else:
                parts[-1] = "kernel"
                transpose = True
        jk = ".".join(parts)
        jk = re.sub(r"fc(\d+)", lambda m: f"Dense_{int(m.group(1)) - 1}", jk)
        jk = jk.replace("blocks.", "blocks_")
        if transpose:
            v = v.permute(2, 3, 1, 0) if v.dim() == 4 else v.t()
        key = jk.replace(".", "/")
        (consts if key.startswith("rope_embed/") else params)[key] = v.contiguous()
    return tree_from_flat(params), tree_from_flat(consts)


def to_torch_hub_state_dict(backbone_tree: dict) -> dict:
    """Inverse of convert_torch_hub_state_dict for the parameter tree (export towards the PyTorch ecosystem)."""
    out = {}
    for k, v in flat_from_tree(backbone_tree).items():
        parts = k.split("/")
        if parts[-1] == "kernel":
            parts[-1] = "weight"
            v = v.permute(3, 2, 0, 1) if v.dim() == 4 else v.t()
        elif parts[-1] == "scale":
            parts[-1] = "weight"
        tk = ".".join(parts)
        tk = re.sub(r"Dense_(\d+)", lambda m: f"fc{int(m.group(1)) + 1}", tk)
        tk = re.sub(r"blocks_(\d+)", lambda m: f"blocks.{m.group(1)}", tk)
        out[tk] = v.contiguous()
    return out


def convert_convnext_torch_hub_state_dict(state_dict: dict) -> dict:
    """Meta's PyTorch DINOv3 ConvNeXt state dict -> the reference's ConvNeXt params tree (models/convnext.py:155-206).

    `downsample_layers.i.j.` -> `downsample_layers_i/layers_j/`, `stages.i.j.` -> `stages_i/layers_j/`.  Conv weights
    [O, I, kh, kw] -> HWIO `kernel` (the depthwise [C, 1, 7, 7] -> [7, 7, 1, C]); Linear `weight` [out, in] -> `kernel`
    [in, out]; the blocks' and downsampling layers' LayerNorms keep `weight` / `bias` (the reference's own LayerNorm), the
    final `norm.weight` becomes `scale` (flax nn.LayerNorm).  `norms.3.*`, upstream's alias of the final norm, is dropped."""
    params = {}
    for tk, v in state_dict.items():
        if tk.startswith("norms."):
            continue
        v = v.detach().cpu() if torch.is_tensor(v) else torch.as_tensor(v)
        parts = tk.split(".")
        if parts[-1] == "weight" and v.dim() >= 2:
            parts[-1] = "kernel"
            v = v.permute(2, 3, 1, 0) if v.dim() == 4 else v.t()
        elif parts == ["norm", "weight"]:
            parts[-1] = "scale"
        jk = re.sub(r"^(downsample_layers|stages)\.(\d+)\.(\d+)\.", r"\1_\2/layers_\3/", ".".join(parts))
        params[jk.replace(".", "/")] = v.contiguous()
    return tree_from_flat(params)


def to_convnext_torch_hub_state_dict(tree: dict) -> dict:
    """Inverse of convert_convnext_torch_hub_state_dict, with upstream's `norms.3.*` alias of the final norm, so the
    result loads strictly into upstream's module."""
    out = {}
    for k, v in flat_from_tree(tree).items():
        parts = k.split("/")
        if parts[-1] == "kernel":
            parts[-1] = "weight"
            v = v.permute(3, 2, 0, 1) if v.dim() == 4 else v.t()
        elif parts[-1] == "scale":
            parts[-1] = "weight"
        tk = re.sub(r"^(downsample_layers|stages)_(\d+)\.layers_(\d+)\.", r"\1.\2.\3.", ".".join(parts))
        out[tk] = v.contiguous()
    for name in ("weight", "bias"):
        out[f"norms.3.{name}"] = out[f"norm.{name}"].clone()
    return out


__all__ = ["CheckpointRetentionPolicy", "cleanup_checkpoint", "find_all_checkpoints", "find_latest_checkpoint",
           "keep_checkpoint_copy", "keep_last_n_checkpoints", "load_checkpoint", "save_checkpoint", "engine_state",
           "load_engine_state", "tree_from_flat", "flat_from_tree", "convert_torch_hub_state_dict",
           "to_torch_hub_state_dict", "convert_convnext_torch_hub_state_dict", "to_convnext_torch_hub_state_dict"]
