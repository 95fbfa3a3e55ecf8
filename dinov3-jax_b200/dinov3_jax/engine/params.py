"""Flat parameter / gradient / optimiser-state storage for the GPU engine.

One `ModuleStore` per top-level module of the reference's parameter tree (`backbone`, `dino_head`, `ibot_head`;
train/ssl_meta_arch.py:62-64,86-87,130-131), holding the student (fp32 master, bf16 compute copy, fp32 gradient, Adam
m / v) and the teacher (fp32 EMA master, bf16 compute copy) as flat device buffers.  Tensors keep the reference's
names and layouts (SURVEY.md Appendix C: Dense kernels [in, out], conv kernel [p, p, 3, D]); matrices (GEMM operands)
come first in the flat buffer, vectors (biases, LayerNorm affine, LayerScale gamma, cls / mask tokens) after, so that
  * the bf16 compute copy covers exactly the leading matrix region,
  * vector grads accumulate atomically and matrix grads are (split-K) accumulations of the wgrad GEMMs into the
    zeroed gradient buffer,
  * clip-norm, AdamW and EMA run as one launch per module (train/train.py:516-541 clips per top-level module).
FSDP units (models/vision_transformer.py:93,137; train/ssl_meta_arch.py:77-78,122-123) are sub-ranges of these buffers.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops
from .config import EngineConfig

ALIGN = 64  # elements; keeps every tensor 128-byte (bf16) / 256-byte (fp32) aligned for TMA and float4 access

SEG_DTYPE = np.dtype([("start", "<i8"), ("lr_mult", "<f4"), ("wd_mult", "<f4"), ("is_last", "<i4"), ("pad", "<i4")])


def backbone_spec(cfg: EngineConfig):
    """(name, shape, kind) in creation order — models/vision_transformer.py:86-171."""
    D, p = cfg.embed_dim, cfg.patch
    spec = [("patch_embed/proj/kernel", (p, p, 3, D), "mat"), ("patch_embed/proj/bias", (D,), "vec"),
            ("cls_token", (1, 1, D), "vec"), ("mask_token", (1, D), "vec")]
    if cfg.n_storage:
        spec.insert(3, ("storage_tokens", (1, cfg.n_storage, D), "vec"))
    for i in range(cfg.depth):
        spec += block_spec(cfg, i)
    spec += [("norm/scale", (D,), "vec"), ("norm/bias", (D,), "vec")]
    return spec


def block_spec(cfg: EngineConfig, i: int):
    """(name, shape, kind) of block i — layers/block.py:22-214."""
    D, Hd = cfg.embed_dim, cfg.hidden
    b = f"blocks_{i}/"
    spec = [(b + "norm1/scale", (D,), "vec"), (b + "norm1/bias", (D,), "vec"), (b + "attn/qkv/kernel", (D, 3 * D), "mat")]
    if cfg.qkv_bias:
        spec += [(b + "attn/qkv/bias", (3 * D,), "vec")]
    spec += [(b + "attn/proj/kernel", (D, D), "mat"), (b + "attn/proj/bias", (D,), "vec"),
             (b + "ls1/gamma", (D,), "vec"),
             (b + "norm2/scale", (D,), "vec"), (b + "norm2/bias", (D,), "vec")]
    if cfg.ffn_layer == "swiglu":                                 # layers/ffn_layers.py:62-69
        Hs = cfg.swiglu_hidden
        spec += [(b + "mlp/w1/kernel", (D, Hs), "mat"), (b + "mlp/w1/bias", (Hs,), "vec"),
                 (b + "mlp/w2/kernel", (D, Hs), "mat"), (b + "mlp/w2/bias", (Hs,), "vec"),
                 (b + "mlp/w3/kernel", (Hs, D), "mat"), (b + "mlp/w3/bias", (D,), "vec")]
    else:
        spec += [(b + "mlp/Dense_0/kernel", (D, Hd), "mat"), (b + "mlp/Dense_0/bias", (Hd,), "vec"),
                 (b + "mlp/Dense_1/kernel", (Hd, D), "mat"), (b + "mlp/Dense_1/bias", (D,), "vec")]
    return spec + [(b + "ls2/gamma", (D,), "vec")]


def head_spec(cfg: EngineConfig, module: str = "dino_head"):
    """layers/dino_head.py:15-43,65-74, at the sizes of `module` ("dino_head" | "ibot_head")."""
    D = cfg.embed_dim
    Hh, Bn, K = cfg.head_dims(module)
    return [("mlp/layers_0/kernel", (D, Hh), "mat"), ("mlp/layers_0/bias", (Hh,), "vec"),
            ("mlp/layers_2/kernel", (Hh, Hh), "mat"), ("mlp/layers_2/bias", (Hh,), "vec"),
            ("mlp/layers_4/kernel", (Hh, Bn), "mat"), ("mlp/layers_4/bias", (Bn,), "vec"),
            ("last_layer/kernel", (Bn, K), "mat")]


def lr_wd_multipliers(module: str, name: str, cfg: EngineConfig):
    """Per-tensor (lr_mult, wd_mult, is_last_layer): train/param_groups.py:56-96 and :104-134."""
    is_backbone = module == "backbone"
    n_layers = cfg.depth if is_backbone else 0
    layer_id = n_layers + 1
    if is_backbone:
        if any(t in name for t in ("pos_embed", "patch_embed", "mask_token", "cls_token", "storage_tokens")):
            layer_id = 0
        elif "blocks_" in name:
            layer_id = int(name.split("blocks_")[1].split("/")[0]) + 1
    lr_mult = cfg.layerwise_decay ** (n_layers + 1 - layer_id)
    wd_mult = 1.0
    if "dino_head" in name:
        wd_mult = cfg.dino_head_wd_multiplier
    is_last = "last_layer" in name
    if name.endswith("bias") or "norm" in name or "gamma" in name:
        wd_mult = 0.0
    if "patch_embed" in name:
        lr_mult *= cfg.patch_embed_lr_mult
    return lr_mult, wd_mult, is_last


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def flat_layout(spec):
    """(offsets, shapes, kinds, padded sizes, n_mat, n) of `spec` in one flat buffer: matrices first, then vectors."""
    offsets, shapes, kinds, padded = {}, {}, {}, {}
    off = n_mat = 0
    for kind in ("mat", "vec"):
        for name, shape, k in spec:
            if k != kind:
                continue
            offsets[name], shapes[name], kinds[name] = off, tuple(shape), k
            padded[name] = _round_up(int(np.prod(shape)), ALIGN)
            off += padded[name]
        if kind == "mat":
            n_mat = off
    return offsets, shapes, kinds, padded, n_mat, off


def _flat_view(flat, offset, shape, as2d):
    v = flat[offset:offset + int(np.prod(shape))]
    return v.view(-1, shape[-1]) if as2d else v.view(shape)


class FrozenStore:
    """A module that only runs forward (the frozen distillation teacher): the bf16 matrix region and the fp32 vector
    region of `spec`'s layout, with no master, optimiser state or gradient.  `w` / `vec` take the `teacher` argument
    of ModuleStore's and ignore it, so the forward pieces read either store."""

    def __init__(self, spec, device):
        self.offsets, self.shapes, _, _, self.n_mat, self.n = flat_layout(spec)
        self.bf16 = torch.zeros(self.n_mat, dtype=torch.bfloat16, device=device)
        self.vecs = torch.zeros(self.n - self.n_mat, dtype=torch.float32, device=device)

    def w(self, name, teacher=True):
        return _flat_view(self.bf16, self.offsets[name], self.shapes[name], True)

    def vec(self, name, teacher=True):
        return _flat_view(self.vecs, self.offsets[name] - self.n_mat, self.shapes[name], False).reshape(-1)

    def load(self, tensors: dict, mask_k_bias: bool):
        """tensors: name -> array (reference layout).  Matrices are rounded to bf16 one tensor at a time (d3_cast_f32_bf16,
        the rounding of ModuleStore.refresh_bf16), so no fp32 copy of the whole module is held on the device."""
        missing = [n for n in self.offsets if n not in tensors]
        extra = [n for n in tensors if n not in self.offsets]
        if missing or extra:
            raise KeyError(f"teacher tensors do not match the configuration: missing {missing[:4]}, unexpected {extra[:4]}")
        dev = self.bf16.device
        for name, off in self.offsets.items():
            src = torch.as_tensor(tensors[name]).to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
            if src.numel() != int(np.prod(self.shapes[name])):
                raise ValueError(f"teacher tensor {name}: {src.numel()} elements, expected shape {self.shapes[name]}")
            if off < self.n_mat:
                ops.cast_f32_bf16(src, self.bf16[off:off + src.numel()])
            else:
                dst = self.vecs[off - self.n_mat:off - self.n_mat + src.numel()]
                dst.copy_(src)
                if mask_k_bias and name.endswith("attn/qkv/bias"):
                    third = src.numel() // 3
                    dst[third:2 * third].zero_()

    def export(self) -> dict:
        """name -> fp32 tensor (reference layout) of every weight: the inverse of `load`, matrices as stored in bf16."""
        full = torch.cat([self.bf16.float(), self.vecs])
        return {name: _flat_view(full, off, self.shapes[name], False).clone() for name, off in self.offsets.items()}


class ModuleStore:
    """Flat buffers of one top-level module on one rank.

    world == 1: every buffer is full size; `vecs` aliases the vector region of the fp32 master.
    world  > 1: persistent state (fp32 master, Adam m / v, teacher master, bf16 shard copies, gradient shard) holds the
    rank's 1/world slice of every FSDP unit (fsdp/layout.py); `bf16` / `vecs` / `t_bf16` / `t_vecs` are the full
    compute buffers the all-gathers fill, `grad` the full gradient buffer the reduce-scatters drain.
    """

    def __init__(self, module: str, spec, cfg: EngineConfig, device, world: int = 1, rank: int = 0):
        from ..fsdp.layout import ShardLayout
        self.module, self.spec, self.cfg = module, spec, cfg
        self.world, self.rank = world, rank
        self.offsets, self.shapes, self.kinds, padded, self.n_mat, self.n = flat_layout(spec)
        names_in_order = [name for name, _, _ in spec]
        self.layout = L = ShardLayout(module, names_in_order, self.offsets, padded, self.kinds, self.n_mat, self.n, world)
        f32, bf16 = torch.float32, torch.bfloat16
        z = lambda n, dt: torch.zeros(n, dtype=dt, device=device)
        ns, nms = L.n_shard, L.n_mat_shard
        self.master, self.t_master = z(ns, f32), z(ns, f32)
        self.m, self.v = z(ns, f32), z(ns, f32)
        self.grad = z(self.n, f32)
        self.sumsq = z(1, f32)
        self.bf16, self.t_bf16 = z(self.n_mat, bf16), z(self.n_mat, bf16)
        if world == 1:
            self.grad_shard = self.grad
            self.bf16_shard, self.t_bf16_shard = self.bf16, self.t_bf16
            self.vecs, self.t_vecs = self.master[self.n_mat:], self.t_master[self.n_mat:]
        else:
            self.grad_shard = z(ns, f32)
            self.bf16_shard, self.t_bf16_shard = z(nms, bf16), z(nms, bf16)
            self.vecs, self.t_vecs = z(self.n - self.n_mat, f32), z(self.n - self.n_mat, f32)
        # optimiser segment table of this rank's shard (sorted by start)
        mult = {nm: lr_wd_multipliers(module, nm, cfg) for nm in self.offsets}
        seg_list = L.shard_segments(rank, mult)
        segs = np.zeros(len(seg_list), dtype=SEG_DTYPE)
        for i, (st_, lr_m, wd_m, last) in enumerate(seg_list):
            segs[i] = (st_, lr_m, wd_m, int(last), 0)
        self.segs_host = segs
        self.nseg = len(seg_list)
        self.segs = torch.from_numpy(segs.view(np.uint8).copy()).to(device)
        self._shard_index = None

    # ---- views (full compute buffers) ---------------------------------------------------------------------------
    def _view(self, flat, name, as2d=False, base=0):
        o, shp = self.offsets[name] - base, self.shapes[name]
        n = int(np.prod(shp))
        v = flat[o:o + n]
        if as2d:
            return v.view(-1, shp[-1])
        return v.view(shp)

    def w(self, name, teacher=False):
        """bf16 compute copy of a matrix, as [in, out] (conv kernel flattened to [p*p*3, D])."""
        return self._view(self.t_bf16 if teacher else self.bf16, name, as2d=True)

    def vec(self, name, teacher=False):
        """fp32 vector (flattened) from the full vector buffer."""
        return self._view(self.t_vecs if teacher else self.vecs, name, base=self.n_mat).reshape(-1)

    def gw(self, name):
        return self._view(self.grad, name, as2d=True)

    def gv(self, name):
        return self._view(self.grad, name).reshape(-1)

    # ---- host <-> device ---------------------------------------------------------------------------------------
    def shard_index(self):
        if self._shard_index is None:
            self._shard_index = torch.from_numpy(self.layout.full_to_shard_index(self.rank)).to(self.master.device)
        return self._shard_index

    def load(self, tensors: dict, teacher: bool):
        """tensors: name -> full tensor (reference layout).  Fills this rank's fp32 shard and the compute copies."""
        dev = self.master.device
        full = torch.zeros(self.n, dtype=torch.float32, device=dev)
        for name in self.offsets:
            self._view(full, name).copy_(tensors[name].to(device=dev, dtype=torch.float32).reshape(self.shapes[name]))
            if self.cfg.mask_k_bias and name.endswith("attn/qkv/bias"):
                # LinearKMaskedBias: the k third never reaches the forward; it is held at zero (and its gradient is
                # zeroed every step, engine/core.py), which is the masked layer's arithmetic
                third = self.shapes[name][0] // 3
                self._view(full, name)[third:2 * third].zero_()
        master = self.t_master if teacher else self.master
        if self.world == 1:
            master.copy_(full)
        else:
            master.copy_(full[self.shard_index()])
            (self.t_vecs if teacher else self.vecs).copy_(full[self.n_mat:])
        self.refresh_bf16(teacher, full=full)

    def refresh_bf16(self, teacher: bool, full=None):
        if not self.n_mat:
            return
        master = self.t_master if teacher else self.master
        nms = self.layout.n_mat_shard
        ops.cast_f32_bf16(master[:nms], (self.t_bf16_shard if teacher else self.bf16_shard))
        if self.world > 1 and full is not None:
            ops.cast_f32_bf16(full[: self.n_mat].contiguous(), self.t_bf16 if teacher else self.bf16)

    def export_full(self, flat_full: torch.Tensor) -> dict:
        return {name: self._view(flat_full, name).detach().clone() for name in self.offsets}

    def zero_grads(self):
        """Vector gradients accumulate atomically and weight gradients are split-K reductions (fp32 atomics), so the
        whole gradient buffer starts each step at zero."""
        self.grad.zero_()
        self.sumsq.zero_()


class ParamStore:
    """Student + teacher parameters of the three top-level modules."""

    MODULES = ("backbone", "dino_head", "ibot_head")

    def __init__(self, cfg: EngineConfig, device, world: int = 1, rank: int = 0):
        self.cfg = cfg
        self.mods = {
            "backbone": ModuleStore("backbone", backbone_spec(cfg), cfg, device, world, rank),
            "dino_head": ModuleStore("dino_head", head_spec(cfg, "dino_head"), cfg, device, world, rank),
            "ibot_head": ModuleStore("ibot_head", head_spec(cfg, "ibot_head"), cfg, device, world, rank),
        }
        self.runtime = None     # set by the engine (fsdp.runtime.FsdpRuntime)

    def load_reference_tree(self, params: dict):
        """params: flat dict 'student_backbone/blocks_0/attn/qkv/kernel' -> tensor (reference names/layouts)."""
        for m, st in self.mods.items():
            for who, teacher in (("student", False), ("teacher", True)):
                pre = f"{who}_{m}/"
                st.load({k[len(pre):]: v for k, v in params.items() if k.startswith(pre)}, teacher)

    def load_optimizer_tree(self, mu: dict, nu: dict):
        """Adam moments with the reference's names ('student_backbone/...'): fills this rank's m / v shards."""
        for m, st in self.mods.items():
            pre = f"student_{m}/"
            for tree, dst in ((mu, st.m), (nu, st.v)):
                full = torch.zeros(st.n, dtype=torch.float32, device=dst.device)
                for name in st.offsets:
                    st._view(full, name).copy_(tree[pre + name].to(device=dst.device, dtype=torch.float32).reshape(st.shapes[name]))
                dst.copy_(full if st.world == 1 else full[st.shard_index()])

    def export_reference_tree(self, what: str = "param") -> dict:
        """Full (un-sharded) tensors with the reference's names; under FSDP this all-gathers the shards."""
        out = {}
        for m, st in self.mods.items():
            for who, teacher in (("student", False), ("teacher", True)):
                if teacher and what != "param":
                    continue
                if self.runtime is not None:
                    full = self.runtime.gather_full(m, what, teacher)
                else:
                    full = {"param": st.t_master if teacher else st.master, "grad": st.grad_shard, "m": st.m, "v": st.v}[what]
                for k, v in st.export_full(full).items():
                    out[f"{who}_{m}/{k}"] = v
        return out

    def n_params(self) -> int:
        return sum(int(np.prod(s)) for st in self.mods.values() for s in st.shapes.values())
