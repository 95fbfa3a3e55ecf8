"""`DinoVisionTransformer` with the reference's constructor fields and call signature
(dinov3_jax/models/vision_transformer.py:55-321), forward pass through the CUDA kernels.

This is the feature-extraction entry point (`model(x)` / `model([global, local], masks=[m, None], is_training=True)`);
training goes through engine/core.py, which runs the same kernels on packed multi-crop streams with the stash the
backward needs.  Parameters arrive as the reference's nested dict (`cls_token`, `mask_token`, `patch_embed/proj`,
`blocks_i/...`, `norm`), any float dtype, CUDA or CPU.
"""
from __future__ import annotations

import torch

from .. import ops
from ..layers import PatchEmbed, RopePositionEmbedding, SelfAttentionBlock

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
        if ffn_layer != "mlp" and ffn_layer not in SelfAttentionBlock.FFN_ALIGN:
            raise NotImplementedError(f"ffn_layer {ffn_layer!r}: mlp | swiglu | swiglu32 | swiglu64 | swiglu128")
        self.eps = 1e-5 if norm_layer == "layernormbf16" else 1e-6        # models/vision_transformer.py:38-42
        self.n_storage_tokens = n_storage_tokens
        if drop_path_rate:
            raise NotImplementedError("stochastic depth is not on the GPU path (reference default 0 is asserted upstream)")
        dev = torch.device(device)
        to = lambda t: torch.as_tensor(t).to(dev)
        mv = lambda tree: {k: (mv(v) if isinstance(v, dict) else to(v)) for k, v in tree.items()}
        params = mv(params)
        self.patch_size, self.embed_dim, self.n_blocks, self.num_heads = patch_size, embed_dim, n_blocks, num_heads
        self.patch_embed = PatchEmbed(params["patch_embed"], img_size=img_size, patch_size=patch_size, in_chans=in_chans,
                                      embed_dim=embed_dim)
        self.cls_token = params["cls_token"].to(f32).reshape(-1).contiguous()
        self.mask_token = params["mask_token"].to(f32).reshape(-1).contiguous()
        self.storage_tokens = params["storage_tokens"].to(f32).reshape(-1).contiguous() if n_storage_tokens else None
        self.rope_embed = RopePositionEmbedding(embed_dim=embed_dim, num_heads=num_heads, base=pos_embed_rope_base,
                                                min_period=pos_embed_rope_min_period, max_period=pos_embed_rope_max_period,
                                                normalize_coords=pos_embed_rope_normalize_coords)
        self.blocks = [SelfAttentionBlock(params[f"blocks_{i}"], dim=embed_dim, num_heads=num_heads, ffn_ratio=ffn_ratio,
                                          qkv_bias=qkv_bias, proj_bias=proj_bias, ffn_bias=ffn_bias, eps=self.eps,
                                          ffn_layer=ffn_layer, mask_k_bias=mask_k_bias)
                       for i in range(n_blocks)]
        ln = lambda p: (p["scale"].to(f32).reshape(-1).contiguous(), p["bias"].to(f32).reshape(-1).contiguous())
        self.norm = ln(params["norm"])
        # :156-164.  local_cls_norm is only read by the training branch (:225), so it is loaded and never applied here.
        self.cls_norm = ln(params["cls_norm"]) if untie_cls_and_patch_norms else None
        self.local_cls_norm = ln(params["local_cls_norm"]) if untie_global_and_local_cls_norm else None
        self.device = dev

    # models/vision_transformer.py:173-203
    def prepare_tokens_with_masks(self, x, masks=None):
        x = torch.as_tensor(x).to(self.device)
        tok = self.patch_embed(x)
        n, Hp, Wp, D = tok.shape
        X = torch.empty(n, 1 + self.n_storage_tokens + Hp * Wp, D, dtype=f32, device=self.device)
        m8 = None if masks is None else torch.as_tensor(masks).to(self.device).reshape(n, Hp * Wp).to(torch.uint8).contiguous()
        ops.assemble_tokens(tok.view(n * Hp * Wp, D), self.cls_token, self.mask_token, m8, X, n, Hp * Wp, D,
                            storage=self.storage_tokens)
        return X, (Hp, Wp)

    # models/vision_transformer.py:205-247
    def forward_features_list(self, x_list, masks_list):
        out = []
        for x, masks in zip(x_list, masks_list):
            X, (Hp, Wp) = self.prepare_tokens_with_masks(x, masks)
            rope = self.rope_embed(H=Hp, W=Wp, device=self.device)
            for blk in self.blocks:
                X = blk(X, rope=rope)
            n, N, D = X.shape
            R = self.n_storage_tokens
            if self.cls_norm is not None:       # :224-232: the 1 + R prefix rows take cls_norm
                cls, storage, patches = self._tokens_out(X, Hp, Wp, True, False, f32)
                out.append({"x_norm_clstoken": cls, "x_storage_tokens": storage, "x_norm_patchtokens": patches,
                            "x_prenorm": X, "masks": masks})
                continue
            Y = torch.empty(n * N, D, dtype=f32, device=self.device)
            ops.layernorm_fwd(X.view(n * N, D), self.norm[0], self.norm[1], Y, eps=self.eps)
            Y = Y.view(n, N, D)
            out.append({"x_norm_clstoken": Y[:, 0], "x_storage_tokens": Y[:, 1:1 + R], "x_norm_patchtokens": Y[:, 1 + R:],
                        "x_prenorm": X, "masks": masks})
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
        X, (Hp, Wp) = self.prepare_tokens_with_masks(x)
        L = len(self.blocks)
        take = range(L - n, L) if isinstance(n, int) else [int(i) for i in n]
        rope = self.rope_embed(H=Hp, W=Wp, device=self.device)
        outputs = []
        for i, blk in enumerate(self.blocks[:max(take, default=-1) + 1]):     # later blocks feed no selected output
            X = blk(X, rope=rope)
            if i in take:
                outputs.append(self._tokens_out(X, Hp, Wp, norm, reshape, out_dtype))
        assert len(outputs) == len(take), f"only {len(outputs)} / {len(take)} blocks found"
        return pack_intermediate_layers(outputs, return_class_token, return_extra_tokens)

    def __call__(self, *args, is_training: bool = False, deterministic: bool = True, **kwargs):
        ret = self.forward_features(*args, **kwargs)
        if is_training:
            return ret
        return ret["x_norm_clstoken"]          # head = Identity (models/vision_transformer.py:160,321)


__all__ = ["DinoVisionTransformer", "pack_intermediate_layers"]
