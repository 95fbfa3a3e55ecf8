"""Layer objects with the reference's names and constructor fields (dinov3_jax/layers/*.py), forward pass on CUDA
tensors through the CUDA kernels.  Parameters are passed as a dict with the reference's leaf names and layouts
(Dense `kernel` [in, out], `bias`; LayerNorm `scale`, `bias`; LayerScale `gamma`).  These are inference-style
wrappers for unit-level use and tests; the training engine fuses the same kernels block-wise (engine/core.py).
"""
from __future__ import annotations

import torch

from .. import ops
from ..engine.core import rope_tables

bf16, f32 = torch.bfloat16, torch.float32


def _w(p):   # matrix -> bf16 [in, out]
    return p.to(bf16).contiguous() if p.dim() == 2 else p.reshape(-1, p.shape[-1]).to(bf16).contiguous()


def _v(p):
    return p.to(f32).reshape(-1).contiguous()


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

    def residual(self, z, xmid, gamma):
        """xmid + gamma * mlp(z) (z bf16 [T, D], xmid fp32 [T, D]): LayerScale and residual in the second GEMM's epilogue."""
        h = torch.empty(z.shape[0], self.w1.shape[1], dtype=bf16, device=z.device)
        ops.gemm(z, self.w1, h, b_mn=True, bias=self.b1, gelu=True)
        out = torch.empty_like(xmid)
        ops.gemm(h, self.w2, out, b_mn=True, bias=self.b2, gelu=True, gamma=gamma, resid=xmid)
        return out


class SwiGLUFFN:
    """layers/ffn_layers.py:52-76: w3(silu(w1 x) * w2 x), hidden width int(2/3 hidden_features) rounded up to align_to.
    The engine's kernels (engine/core.py): the w1 and w2 GEMMs write the two halves of one [T, 2 Hs] buffer, then
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

    def _hidden(self, z):
        T, Hs = z.shape[0], self.Hs
        x12 = torch.empty(T, 2 * Hs, dtype=bf16, device=z.device)
        ops.gemm(z, self.w1, x12[:, :Hs], b_mn=True, bias=self.b1)
        ops.gemm(z, self.w2, x12[:, Hs:], b_mn=True, bias=self.b2)
        h = torch.empty(T, Hs, dtype=bf16, device=z.device)
        ops.swiglu_fwd(x12, h)
        return h

    def __call__(self, x):
        shp = x.shape
        h = self._hidden(x.reshape(-1, shp[-1]).to(bf16).contiguous())
        y = torch.empty(h.shape[0], self.w3.shape[1], dtype=f32, device=x.device)
        ops.gemm(h, self.w3, y, b_mn=True, bias=self.b3)
        return y.view(*shp[:-1], self.w3.shape[1])

    def residual(self, z, xmid, gamma):
        """xmid + gamma * ffn(z): LayerScale and residual in the w3 GEMM's epilogue."""
        out = torch.empty_like(xmid)
        ops.gemm(self._hidden(z), self.w3, out, b_mn=True, bias=self.b3, gamma=gamma, resid=xmid)
        return out


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
    """layers/block.py:22-214, deterministic branch :195-201: x + ls1(attn(norm1 x)); x + ls2(mlp(norm2 x))."""

    FFN_ALIGN = {"swiglu": 8, "swiglu32": 32, "swiglu64": 64, "swiglu128": 128}     # models/vision_transformer.py:30-36

    def __init__(self, params: dict, dim: int, num_heads: int, ffn_ratio: float = 4.0, qkv_bias: bool = True,
                 proj_bias: bool = True, ffn_bias: bool = True, init_values=None, eps: float = 1e-6,
                 ffn_layer: str = "mlp", mask_k_bias: bool = False, **unused):
        self.dim, self.H, self.eps = dim, num_heads, eps
        self.attn = SelfAttention(params["attn"], dim, num_heads, qkv_bias=qkv_bias, mask_k_bias=mask_k_bias)
        if ffn_layer == "mlp":
            self.mlp = Mlp(params["mlp"])
        elif ffn_layer in self.FFN_ALIGN:
            self.mlp = SwiGLUFFN(params["mlp"], hidden_features=int(dim * ffn_ratio), out_features=dim, use_bias=ffn_bias,
                                 align_to=self.FFN_ALIGN[ffn_layer])
        else:
            raise NotImplementedError(f"ffn_layer {ffn_layer!r}: mlp | swiglu | swiglu32 | swiglu64 | swiglu128")
        self.n1 = (_v(params["norm1"]["scale"]), _v(params["norm1"]["bias"]))
        self.n2 = (_v(params["norm2"]["scale"]), _v(params["norm2"]["bias"]))
        self.g1, self.g2 = _v(params["ls1"]["gamma"]), _v(params["ls2"]["gamma"])

    def __call__(self, x, rope=None, deterministic=True):
        n, N, D = x.shape
        X = x.reshape(n * N, D).to(f32).contiguous()
        y = torch.empty(n * N, D, dtype=bf16, device=x.device)
        ops.layernorm_fwd(X, self.n1[0], self.n1[1], y, eps=self.eps)
        qkv = torch.empty(n * N, 3 * D, dtype=bf16, device=x.device)
        ops.gemm(y, self.attn.wqkv, qkv, b_mn=True, bias=self.attn.bqkv)
        o = self.attn.compute_attention(qkv.view(n, N, 3 * D), rope=rope).reshape(n * N, D)
        xmid = torch.empty_like(X)
        ops.gemm(o, self.attn.wp, xmid, b_mn=True, bias=self.attn.bp, gamma=self.g1, resid=X)
        z = torch.empty(n * N, D, dtype=bf16, device=x.device)
        ops.layernorm_fwd(xmid, self.n2[0], self.n2[1], z, eps=self.eps)
        return self.mlp.residual(z, xmid, self.g2).view(n, N, D)


class DINOHead:
    """layers/dino_head.py:46-85: MLP(GELU) -> x / (||x|| + 1e-12) -> bias-free prototype layer."""

    def __init__(self, params: dict, in_dim: int, out_dim: int, use_bn: bool = False, nlayers: int = 3,
                 hidden_dim: int = 2048, bottleneck_dim: int = 256, mlp_bias: bool = True):
        if use_bn or nlayers != 3:
            raise NotImplementedError("DINOHead on the GPU path: nlayers=3, no batch norm (reference defaults)")
        m = params["mlp"]
        self.w = [_w(m[f"layers_{i}"]["kernel"]) for i in (0, 2, 4)]
        self.b = [_v(m[f"layers_{i}"]["bias"]) for i in (0, 2, 4)]
        self.wl = _w(params["last_layer"]["kernel"])

    def __call__(self, x, no_last_layer=False, only_last_layer=False):
        R = x.shape[0]
        dev = x.device
        if not only_last_layer:
            a = x.to(bf16).contiguous()
            h1 = torch.empty(R, self.w[0].shape[1], dtype=bf16, device=dev)
            ops.gemm(a, self.w[0], h1, b_mn=True, bias=self.b[0], gelu=True)
            h2 = torch.empty(R, self.w[1].shape[1], dtype=bf16, device=dev)
            ops.gemm(h1, self.w[1], h2, b_mn=True, bias=self.b[1], gelu=True)
            u = torch.empty(R, self.w[2].shape[1], dtype=f32, device=dev)
            ops.gemm(h2, self.w[2], u, b_mn=True, bias=self.b[2])
            yn = torch.empty(R, u.shape[1], dtype=bf16, device=dev)
            ops.l2norm_fwd(u, yn, torch.empty(R, dtype=f32, device=dev), 1e-12)
            x = yn
        if no_last_layer:
            return x
        logits = torch.empty(R, self.wl.shape[1], dtype=f32, device=dev)
        ops.gemm(x.to(bf16).contiguous(), self.wl, logits, b_mn=True)
        return logits


__all__ = ["RopePositionEmbedding", "LayerScale", "PatchEmbed", "Mlp", "SwiGLUFFN", "SelfAttention", "SelfAttentionBlock", "DINOHead"]
