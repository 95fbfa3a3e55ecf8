"""Layer objects with the reference's names and constructor fields (dinov3_jax/layers/*.py), forward pass on CUDA
tensors through the CUDA kernels.  Parameters are passed as a dict with the reference's leaf names and layouts
(Dense `kernel` [in, out], `bias`; LayerNorm `scale`, `bias`; LayerScale `gamma`).  These are inference-style
wrappers for unit-level use and tests.  `SelfAttentionBlock` and `DINOHead` run the training engine's forward pieces
(engine/forward.py: `block_fwd`, `head_fwd`) on frozen weights; `PatchEmbed`, `SelfAttention`, `Mlp`, `SwiGLUFFN` and
`LayerScale` launch the kernels of one layer on their own.
"""
from __future__ import annotations

from dataclasses import replace

import torch

from .. import ops
from ..checkpointer import flat_from_tree
from ..engine.config import FFN_LAYERS, EngineConfig
from ..engine.forward import CropSet, HeadBufs, Net, Stream, block_fwd, head_fwd, rope_tables
from ..engine.params import FrozenStore, block_spec, head_spec

bf16, f32 = torch.bfloat16, torch.float32


def _w(p):   # matrix -> bf16 [in, out]
    return p.to(bf16).contiguous() if p.dim() == 2 else p.reshape(-1, p.shape[-1]).to(bf16).contiguous()


def _v(p):
    return p.to(f32).reshape(-1).contiguous()


def vit_config(flat: dict, dim: int, num_heads: int, ffn_ratio: float, eps: float, ffn_layer: str, mask_k_bias: bool,
               **kw) -> EngineConfig:
    """The EngineConfig of a ViT block / backbone from the reference's constructor arguments.  A tree `flat` without
    qkv biases runs without them, whatever the qkv_bias argument says."""
    if dim not in (num_heads * 64, num_heads * 128):
        raise NotImplementedError("head_dim must be 64 or 128")
    if ffn_layer not in FFN_LAYERS:
        raise NotImplementedError(f"ffn_layer {ffn_layer!r}: mlp | swiglu | swiglu32 | swiglu64 | swiglu128")
    ffn, align = FFN_LAYERS[ffn_layer]
    return EngineConfig(embed_dim=dim, heads=num_heads, ffn_ratio=ffn_ratio, ln_eps=eps, ffn_layer=ffn, swiglu_align=align,
                        mask_k_bias=mask_k_bias, qkv_bias="blocks_0/attn/qkv/bias" in flat, **kw)


def frozen_store(spec, flat: dict, mask_k_bias: bool, device, ffn_bias: bool = True) -> FrozenStore:
    """A FrozenStore of `spec` loaded from `flat` ('/'-joined reference names, any float dtype).  Names outside the spec
    are ignored; a SwiGLU bias is a zero vector where the tree has none or `ffn_bias` is off (SwiGLUFFN's use_bias)."""
    tensors = {}
    for name, shape, _ in spec:
        if name.endswith(("mlp/w1/bias", "mlp/w2/bias", "mlp/w3/bias")) and (not ffn_bias or name not in flat):
            tensors[name] = torch.zeros(shape)
        elif name in flat:
            tensors[name] = flat[name]
    store = FrozenStore(spec, device)
    store.load(tensors, mask_k_bias)
    return store


class RopePositionEmbedding:
    """layers/rope_position_encoding.py:17-123 (deterministic path, normalize_coords='separate')."""

    def __init__(self, embed_dim: int, num_heads: int, base: float | None = 100.0, min_period=None, max_period=None,
                 normalize_coords: str = "separate", shift_coords=None, jitter_coords=None, rescale_coords=None, dtype=None):
        assert embed_dim % (4 * num_heads) == 0
        if base is None or min_period is not None or max_period is not None:
            raise NotImplementedError("only the `base` parametrisation is on the GPU path")
        if normalize_coords != "separate":
            raise NotImplementedError("normalize_coords must be 'separate' (default)")
        self.head_dim, self.base = embed_dim // num_heads, base

    def __call__(self, *, H, W, deterministic=True, rng=None, device="cuda"):
        return rope_tables(H, W, self.head_dim, self.base, device)


class LayerScale:
    """layers/layer_scale.py:12-21.  gamma is applied in the epilogue of the producing GEMM (D3_EP_GAMMA)."""

    def __init__(self, params: dict):
        self.gamma = _v(params["gamma"])


class PatchEmbed:
    """layers/patch_embed.py:21-55: [n, H, W, 3] -> [n, H/p, W/p, D]."""

    def __init__(self, params: dict, img_size: int = 224, patch_size: int = 16, in_chans: int = 3, embed_dim: int = 768,
                 flatten_embedding: bool = False):
        self.p, self.D = patch_size, embed_dim
        self.kernel, self.bias = _w(params["proj"]["kernel"]), _v(params["proj"]["bias"])

    def __call__(self, x):
        n, H, W, c = x.shape
        if H % self.p or W % self.p:
            raise AssertionError(f"Input image height {H} / width {W} is not a multiple of patch size {self.p}")   # :48-49
        P = (H // self.p) * (W // self.p)
        kdim = self.p * self.p * c
        patches = torch.empty(n * P, (kdim + 7) // 8 * 8, dtype=bf16, device=x.device)[:, :kdim]
        ops.im2col(x.to(bf16).contiguous(), patches, self.p)
        out = torch.empty(n * P, self.D, dtype=f32, device=x.device)
        ops.gemm(patches, self.kernel, out, b_mn=True, bias=self.bias)
        return out.view(n, H // self.p, W // self.p, self.D)


class Mlp:
    """layers/ffn_layers.py:24-49: Dense -> GELU -> Dense -> GELU (the second activation is in the reference)."""

    def __init__(self, params: dict, hidden_features=None, out_features=None, use_bias: bool = True):
        self.w1, self.b1 = _w(params["Dense_0"]["kernel"]), _v(params["Dense_0"]["bias"])
        self.w2, self.b2 = _w(params["Dense_1"]["kernel"]), _v(params["Dense_1"]["bias"])

    def __call__(self, x, deterministic=True):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1]).to(bf16).contiguous()
        h = torch.empty(x2.shape[0], self.w1.shape[1], dtype=bf16, device=x.device)
        ops.gemm(x2, self.w1, h, b_mn=True, bias=self.b1, gelu=True)
        y = torch.empty(x2.shape[0], self.w2.shape[1], dtype=f32, device=x.device)
        ops.gemm(h, self.w2, y, b_mn=True, bias=self.b2, gelu=True)
        return y.view(*shp[:-1], self.w2.shape[1])


class SwiGLUFFN:
    """layers/ffn_layers.py:52-76: w3(silu(w1 x) * w2 x), hidden width int(2/3 hidden_features) rounded up to align_to.
    The engine's kernels (engine/forward.py): the w1 and w2 GEMMs write the two halves of one [T, 2 Hs] buffer, then
    d3_swiglu_fwd, then the w3 GEMM."""

    def __init__(self, params: dict, hidden_features=None, out_features=None, act_layer=None, drop: float = 0.0,
                 use_bias: bool = True, align_to: int = 8):
        self.w1, self.w2, self.w3 = (_w(params[k]["kernel"]) for k in ("w1", "w2", "w3"))
        Hs = self.w1.shape[1]
        if hidden_features is not None:
            d = int(hidden_features * 2 / 3)
            assert Hs == d + (-d % align_to), f"w1 has {Hs} columns, SwiGLUFFN({hidden_features}, align_to={align_to}) " \
                                              f"has {d + (-d % align_to)}"
        if Hs % 8:
            raise NotImplementedError("SwiGLU hidden width must be a multiple of 8 (align_to 8 / 32 / 64 / 128 all give one)")
        zero = lambda k: torch.zeros(k, dtype=f32, device=self.w1.device)
        bias = lambda k, w: _v(params[k]["bias"]) if use_bias and "bias" in params[k] else zero(w.shape[1])
        self.b1, self.b2, self.b3 = bias("w1", self.w1), bias("w2", self.w2), bias("w3", self.w3)
        self.Hs = Hs

    def __call__(self, x):
        shp = x.shape
        z = x.reshape(-1, shp[-1]).to(bf16).contiguous()
        T, Hs = z.shape[0], self.Hs
        x12 = torch.empty(T, 2 * Hs, dtype=bf16, device=z.device)
        ops.gemm(z, self.w1, x12[:, :Hs], b_mn=True, bias=self.b1)
        ops.gemm(z, self.w2, x12[:, Hs:], b_mn=True, bias=self.b2)
        h = torch.empty(T, Hs, dtype=bf16, device=z.device)
        ops.swiglu_fwd(x12, h)
        y = torch.empty(T, self.w3.shape[1], dtype=f32, device=x.device)
        ops.gemm(h, self.w3, y, b_mn=True, bias=self.b3)
        return y.view(*shp[:-1], self.w3.shape[1])


class SelfAttention:
    """layers/attention.py:49-118: fused qkv Dense -> RoPE on q,k (prefix tokens skipped) -> attention -> proj."""

    def __init__(self, params: dict, dim: int, num_heads: int = 8, qkv_bias: bool = False, proj_bias: bool = True,
                 attn_drop: float = 0.0, proj_drop: float = 0.0, mask_k_bias: bool = False):
        if dim not in (num_heads * 64, num_heads * 128):
            raise NotImplementedError("head_dim must be 64 or 128")
        self.dim, self.H = dim, num_heads
        self.wqkv = _w(params["qkv"]["kernel"])
        self.bqkv = _v(params["qkv"]["bias"]) if "bias" in params["qkv"] else torch.zeros(3 * dim, device=self.wqkv.device)
        if mask_k_bias:      # the engine's meaning (upstream DINOv3 LinearKMaskedBias): the k third of the bias is zero
            self.bqkv = self.bqkv.clone()
            self.bqkv[dim:2 * dim] = 0
        self.wp, self.bp = _w(params["proj"]["kernel"]), _v(params["proj"]["bias"])

    def compute_attention(self, qkv, attn_bias=None, rope=None, deterministic=True):
        assert attn_bias is None
        n, N, _ = qkv.shape
        q2 = qkv.reshape(n * N, 3 * self.dim).contiguous()
        if rope is not None:
            sin, cos = rope
            ops.rope(q2, sin, cos, N, N - sin.shape[0], self.dim, self.dim // self.H)
        o = torch.empty(n * N, self.dim, dtype=bf16, device=qkv.device)
        ops.attn_fwd(q2, o, None, n, N, self.dim, self.H)
        return o.view(n, N, self.dim)

    def __call__(self, x, attn_bias=None, rope=None, deterministic=True):
        n, N, D = x.shape
        x2 = x.reshape(n * N, D).to(bf16).contiguous()
        qkv = torch.empty(n * N, 3 * D, dtype=bf16, device=x.device)
        ops.gemm(x2, self.wqkv, qkv, b_mn=True, bias=self.bqkv)
        o = self.compute_attention(qkv.view(n, N, 3 * D), attn_bias, rope)
        y = torch.empty(n * N, D, dtype=f32, device=x.device)
        ops.gemm(o.reshape(n * N, D), self.wp, y, b_mn=True, bias=self.bp)
        return y.view(n, N, D)


class SelfAttentionBlock:
    """layers/block.py:22-214, deterministic branch :195-201: x + ls1(attn(norm1 x)); x + ls2(mlp(norm2 x)), as
    engine.forward.block_fwd on a one-block FrozenStore."""

    def __init__(self, params: dict, dim: int, num_heads: int, ffn_ratio: float = 4.0, qkv_bias: bool = True,
                 proj_bias: bool = True, ffn_bias: bool = True, init_values=None, eps: float = 1e-6,
                 ffn_layer: str = "mlp", mask_k_bias: bool = False, **unused):
        flat = {"blocks_0/" + k: v for k, v in flat_from_tree(params).items()}
        self.cfg = vit_config(flat, dim, num_heads, ffn_ratio, eps, ffn_layer, mask_k_bias, depth=1)
        self.store = frozen_store(block_spec(self.cfg, 0), flat, mask_k_bias, flat["blocks_0/attn/qkv/kernel"].device, ffn_bias)

    def __call__(self, x, rope=None, deterministic=True):
        """x [n, N, D]; rope: (sin, cos) of the last P tokens, or None: identity tables (cos 1, sin 0), unrotated bits."""
        n, N, D = x.shape
        if rope is None:
            rope = (torch.zeros(N - 1, self.cfg.head_dim, device=x.device), torch.ones(N - 1, self.cfg.head_dim, device=x.device))
        P = rope[0].shape[0]
        cfg = replace(self.cfg, n_storage=N - P - 1)          # the N - P tokens in front are not rotated
        st = Stream(cfg, [CropSet(cfg, n, P, 1, 0, x.device, rope=rope)], x.device, stash=False)
        st.x_in(0).copy_(x.reshape(n * N, D))
        block_fwd(Net(cfg, {"backbone": self.store}, True), st, 0)
        return st.x_out(0).view(n, N, D)


class DINOHead:
    """layers/dino_head.py:46-85: MLP(GELU) -> x / (||x|| + 1e-12) -> bias-free prototype layer, as
    engine.forward.head_fwd on a FrozenStore."""

    def __init__(self, params: dict, in_dim: int, out_dim: int, use_bn: bool = False, nlayers: int = 3,
                 hidden_dim: int = 2048, bottleneck_dim: int = 256, mlp_bias: bool = True):
        if use_bn or nlayers != 3:
            raise NotImplementedError("DINOHead on the GPU path: nlayers=3, no batch norm (reference defaults)")
        flat = flat_from_tree(params)
        self.cfg = EngineConfig(embed_dim=in_dim, n_prototypes=out_dim, head_hidden=hidden_dim, head_bottleneck=bottleneck_dim)
        self.net = Net(self.cfg, {"dino_head": frozen_store(head_spec(self.cfg), flat, False, flat["last_layer/kernel"].device)}, True)

    def __call__(self, x, no_last_layer=False, only_last_layer=False):
        R = x.shape[0]
        if only_last_layer:
            logits = torch.empty(R, self.cfg.n_prototypes, dtype=f32, device=x.device)
            ops.gemm(x.to(bf16).contiguous(), self.net.mods["dino_head"].w("last_layer/kernel"), logits, b_mn=True)
            return logits
        hb = HeadBufs(self.cfg, "dino_head", R, x.device, stash=False)
        hb.A0.copy_(x)
        head_fwd(self.net, hb, "dino_head", R, stash=False)
        return hb.Yn if no_last_layer else hb.logits


__all__ = ["RopePositionEmbedding", "LayerScale", "PatchEmbed", "Mlp", "SwiGLUFFN", "SelfAttention", "SelfAttentionBlock", "DINOHead"]
