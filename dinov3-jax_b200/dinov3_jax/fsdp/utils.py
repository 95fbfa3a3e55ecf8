"""The reference's FSDP helper names (dinov3_jax/fsdp/utils.py:19-110) on torch tensors + torch.distributed.

In the reference these run inside `shard_map` and `axis_name` ("dp") names the mesh axis; here `axis_name` names the
process group (None / "dp" = WORLD).  The training engine itself uses the flat per-unit layout of fsdp/layout.py and
fsdp/runtime.py; these leaf-wise functions keep the reference's semantics for tools that shard / gather named pytrees
(checkpoint conversion, tests): slice each leaf on its LARGEST axis divisible by the axis size (:36-47), leave leaves of
<= min_param_size elements replicated (:27-29), gather with a tiled all-gather (:66), mean-reduce replicated grads (:108).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch
import torch.distributed as dist


@dataclass
class Partitioned:
    """Counterpart of flax.linen.Partitioned: a local shard plus the axis it was split on."""
    value: torch.Tensor
    axis: int
    axis_name: str = "dp"


def _group(axis_name):
    return None


def _axis_size(axis_name="dp") -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _axis_index(axis_name="dp") -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def _map(fn, tree):
    if isinstance(tree, dict):
        return {k: _map(fn, v) for k, v in tree.items()}
    return fn(tree)


def shard_params(params, axis_name="dp", min_param_size=2 ** 18):
    idx, size = _axis_index(axis_name), _axis_size(axis_name)

    def split(x):
        if isinstance(x, Partitioned) or x.numel() <= min_param_size:
            return x
        for i in np.argsort(x.shape)[::-1]:
            if x.shape[i] % size == 0:
                s = x.shape[i] // size
                return Partitioned(x.narrow(int(i), idx * s, s).contiguous(), int(i), axis_name)
        return x                                   # no divisible axis: stays replicated (:48-49)
    return _map(split, params)


def fwd_gather_bwd_pmean_scatter(x: torch.Tensor, axis: int, axis_name="dp") -> torch.Tensor:
    """Forward half (tiled all-gather along `axis`); the backward half (psum_scatter / axis_size) is the
    reduce-scatter(mean) issued by fsdp/runtime.py after each unit's backward."""
    size = _axis_size(axis_name)
    if size == 1:
        return x
    parts = [torch.empty_like(x) for _ in range(size)]
    dist.all_gather(parts, x.contiguous())
    return torch.cat(parts, dim=axis)


def gather_params(params, axis_name="dp"):
    return _map(lambda p: fwd_gather_bwd_pmean_scatter(p.value, p.axis, p.axis_name) if isinstance(p, Partitioned) else p,
                params)


def sync_grads(grads, axis_name="dp"):
    size = _axis_size(axis_name)

    def sync(g):
        if isinstance(g, Partitioned) or size == 1:
            return g
        g = g.clone()
        dist.all_reduce(g)
        return g / size
    return _map(sync, grads)


def fsdp_wrapper(target, axis_name="dp", min_param_size=2 ** 4):
    """The reference returns nn.map_variables(target, gather on read, shard on write) (:87-94).  The GPU engine shards
    by FSDP unit inside Engine(comm=...); wrapping a module class is therefore the identity, kept for API compatibility."""
    return target
