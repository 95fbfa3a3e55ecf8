"""`DinoVisionTransformer` with the reference's constructor fields and call signature
(dinov3_jax/models/vision_transformer.py:55-321), forward pass through the CUDA kernels.

This is the feature-extraction entry point (`model(x)` / `model([global, local], masks=[m, None], is_training=True)`).
The weights live in one FrozenStore in the training engine's flat backbone layout, and the forward runs the engine's
own pieces (engine/forward.py: `embed`, `block_fwd`, `backbone_fwd`) on one token stream per input, so a feature
and a training teacher pass launch the same kernels on the same bits.  Parameters arrive as the reference's nested dict
(`cls_token`, `mask_token`, `patch_embed/proj`, `blocks_i/...`, `norm`), any float dtype, CUDA or CPU; weights go
through fp32 on their way to bf16, as every engine load does.
"""
from __future__ import annotations

import torch

from .. import ops
from ..checkpointer import flat_from_tree
from ..engine.forward import CropSet, Net, Stream, backbone_fwd, block_fwd, embed
from ..engine.params import backbone_spec
from ..layers import RopePositionEmbedding, frozen_store, vit_config

bf16, f32 = torch.bfloat16, torch.float32


def pack_intermediate_layers(outputs, return_class_token: bool, return_extra_tokens: bool) -> tuple:
    """[(cls, storage, patches) per block] -> the four return forms of models/vision_transformer.py:305-312."""
    patches, cls, extra = [o[2] for o in outputs], [o[0] for o in outputs], [o[1] for o in outputs]
    if return_class_token and return_extra_tokens:
        return tuple(zip(patches, cls, extra))
    if return_class_token:
        return tuple(zip(patches, cls))
    if return_extra_tokens:
        return tuple(zip(patches, extra))
    return tuple(patches)


class DinoVisionTransformer:
    def __init__(self, params: dict, *, img_size: int = 224, patch_size: int = 16, in_chans: int = 3,
                 pos_embed_rope_base: float = 100.0, pos_embed_rope_min_period=None, pos_embed_rope_max_period=None,
                 pos_embed_rope_normalize_coords: str = "separate", pos_embed_rope_shift_coords=None,
                 pos_embed_rope_jitter_coords=None, pos_embed_rope_rescale_coords=None, pos_embed_rope_dtype: str = "bf16",
                 embed_dim: int = 768, n_blocks: int = 12, num_heads: int = 12, ffn_ratio: float = 4.0,
                 qkv_bias: bool = True, drop_path_rate: float = 0.0, layerscale_init=None, norm_layer: str = "layernorm",
                 ffn_layer: str = "mlp", ffn_bias: bool = True, proj_bias: bool = True, n_storage_tokens: int = 0,
                 mask_k_bias: bool = False, untie_cls_and_patch_norms: bool = False,
                 untie_global_and_local_cls_norm: bool = False, device="cuda"):
        if norm_layer not in ("layernorm", "layernormbf16"):
            raise NotImplementedError("GPU path: norm_layer layernorm | layernormbf16")
        if drop_path_rate:
            raise NotImplementedError("stochastic depth is not on the GPU path (reference default 0 is asserted upstream)")
        self.rope_embed = RopePositionEmbedding(embed_dim=embed_dim, num_heads=num_heads, base=pos_embed_rope_base,
                                                min_period=pos_embed_rope_min_period, max_period=pos_embed_rope_max_period,
                                                normalize_coords=pos_embed_rope_normalize_coords)
        dev = torch.device(device)
        flat = {k: torch.as_tensor(v) for k, v in flat_from_tree(params).items()}
        eps = 1e-5 if norm_layer == "layernormbf16" else 1e-6        # models/vision_transformer.py:38-42
        self.cfg = vit_config(flat, embed_dim, num_heads, ffn_ratio, eps, ffn_layer, mask_k_bias, depth=n_blocks,
                              patch=patch_size, rope_base=pos_embed_rope_base, n_storage=n_storage_tokens)
        self.net = Net(self.cfg, {"backbone": frozen_store(backbone_spec(self.cfg), flat, mask_k_bias, dev, ffn_bias)}, True)
        self.patch_size, self.embed_dim, self.n_blocks, self.num_heads = patch_size, embed_dim, n_blocks, num_heads
        self.n_storage_tokens, self.eps = n_storage_tokens, eps
        self.norm = (self.net.mods["backbone"].vec("norm/scale"), self.net.mods["backbone"].vec("norm/bias"))
        ln = lambda name: tuple(flat[f"{name}/{k}"].to(device=dev, dtype=f32).reshape(-1).contiguous() for k in ("scale", "bias"))
        # :156-164.  local_cls_norm is only read by the training branch (:225), so it is loaded and never applied here.
        self.cls_norm = ln("cls_norm") if untie_cls_and_patch_norms else None
        self.local_cls_norm = ln("local_cls_norm") if untie_global_and_local_cls_norm else None
        self.device = dev

    def _stream(self, x, masks=None):
        """One input batch -> (its bf16 NHWC images, uint8 masks or None, a token stream of one crop set)."""
        x = torch.as_tensor(x).to(self.device)
        n, H, W, _ = x.shape
        p = self.patch_size
        if H % p or W % p:
            raise AssertionError(f"Input image height {H} / width {W} is not a multiple of patch size {p}")   # layers/patch_embed.py:48-49
        cs = CropSet(self.cfg, n, H // p, W // p, 0, self.device)
        m8 = None if masks is None else torch.as_tensor(masks).to(self.device).reshape(n, cs.P).to(torch.uint8).contiguous()
        return x.to(bf16).contiguous(), m8, Stream(self.cfg, [cs], self.device, stash=False)

    # models/vision_transformer.py:205-247
    def forward_features_list(self, x_list, masks_list):
        out = []
        L, D, R = self.cfg.depth, self.embed_dim, self.n_storage_tokens
        for x, masks in zip(x_list, masks_list):
            img, m8, st = self._stream(x, masks)
            cs = st.sets[0]
            if self.cls_norm is None:
                backbone_fwd(self.net, st, [img], [m8])
                Y = st.Xn.view(cs.n, cs.N, D)
                cls, storage, patches = Y[:, 0], Y[:, 1:1 + R], Y[:, 1 + R:]
            else:       # :224-232: the 1 + R prefix rows take cls_norm, so no LayerNorm runs over every token
                embed(self.net, st, [img], [m8])
                for i in range(L):
                    block_fwd(self.net, st, i)
                cls, storage, patches = self._tokens_out(st.x_in(L).view(cs.n, cs.N, D), cs.Hp, cs.Wp, True, False, f32)
            out.append({"x_norm_clstoken": cls, "x_storage_tokens": storage, "x_norm_patchtokens": patches,
                        "x_prenorm": st.x_in(L).view(cs.n, cs.N, D), "masks": masks})
        return out

    def _tokens_out(self, X, Hp, Wp, norm: bool, reshape: bool, out_dtype):
        """One block output -> (cls [n, D], storage [n, R, D], patches [n, P, D] or [n, D, Hp, Wp]) in one kernel."""
        n, N, D = X.shape
        R = self.n_storage_tokens
        e = lambda *shape: torch.empty(*shape, dtype=out_dtype, device=self.device)
        cls, patches = e(n, D), (e(n, D, Hp, Wp) if reshape else e(n, Hp * Wp, D))
        storage = e(n, R, D) if R else None
        ops.layernorm_tokens_out(X, cls, storage, patches, Hp, Wp, norm=self.norm if norm else None, pre_norm=self.cls_norm,
                                 eps=self.eps, channels_first=reshape)
        return cls, (e(n, 0, D) if storage is None else storage), patches

    def forward_features(self, x, masks=None):
        if isinstance(x, (list, tuple)):
            return self.forward_features_list(list(x), list(masks) if masks is not None else [None] * len(x))
        return self.forward_features_list([x], [masks])[0]

    # models/vision_transformer.py:262-313, with the upstream DINOv3 semantics (the reference's own method cannot run,
    # DESIGN.md §2).  Each selected block's output goes through d3_layernorm_tokens_out as soon as the block has run, so
    # only the returned tensors stay in memory.
    def get_intermediate_layers(self, x, *, n=1, reshape: bool = False, return_class_token: bool = False,
                                return_extra_tokens: bool = False, norm: bool = True, out_dtype=f32):
        """x NHWC [B, H, W, 3]; n: the last n blocks (int) or a list of block indices.  Returns one entry per selected
        block, in block order: patch tokens [B, H/p * W/p, D] (reshape: [B, D, H/p, W/p]), zipped with the class token
        [B, D] and / or the storage tokens [B, R, D] when asked for.  out_dtype: torch.float32 or torch.bfloat16."""
        if out_dtype not in (f32, bf16):
            raise ValueError("out_dtype must be torch.float32 or torch.bfloat16")
        img, _, st = self._stream(x)
        cs, L = st.sets[0], self.cfg.depth
        take = range(L - n, L) if isinstance(n, int) else [int(i) for i in n]
        embed(self.net, st, [img], [None])
        outputs = []
        for i in range(min(max(take, default=-1) + 1, L)):     # later blocks feed no selected output
            block_fwd(self.net, st, i)
            if i in take:
                outputs.append(self._tokens_out(st.x_out(i).view(cs.n, cs.N, self.embed_dim), cs.Hp, cs.Wp, norm, reshape,
                                                out_dtype))
        assert len(outputs) == len(take), f"only {len(outputs)} / {len(take)} blocks found"
        return pack_intermediate_layers(outputs, return_class_token, return_extra_tokens)

    def __call__(self, *args, is_training: bool = False, deterministic: bool = True, **kwargs):
        ret = self.forward_features(*args, **kwargs)
        if is_training:
            return ret
        return ret["x_norm_clstoken"]          # head = Identity (models/vision_transformer.py:160,321)


__all__ = ["DinoVisionTransformer", "pack_intermediate_layers"]
