"""`ConvNeXt` with the reference's sizes and call signatures (dinov3_jax/models/convnext.py:130-335), forward pass
through the CUDA kernels.  The semantics are upstream DINOv3's ConvNeXt, which the reference transcribes; the
reference's own module cannot run (DESIGN.md §2).

Parameters arrive as the reference's nested dict, any float dtype, CUDA or CPU:
`downsample_layers_0/layers_0` (Conv 4x4 stride 4, HWIO `kernel`, `bias`) and `/layers_1` (LayerNorm `weight`, `bias`);
`downsample_layers_i/layers_0` (LayerNorm) and `/layers_1` (Conv 2x2 stride 2) for i = 1..3;
`stages_i/layers_j/{dwconv (HWIO [7, 7, 1, C]), norm, pwconv1, pwconv2 (Dense `kernel` [in, out]), gamma}`; the final
`norm` (flax nn.LayerNorm: `scale`, `bias`).  checkpointer.convert_convnext_torch_hub_state_dict gives this tree from
Meta's PyTorch state dict.

Per stage the residual stream is one fp32 NHWC map.  A block is d3_dwconv7_layernorm (bf16 operand), the pwconv1 GEMM
with the exact-GELU epilogue (bf16 hidden) and the pwconv2 GEMM with bias, LayerScale and the residual add into the
stream.  Input is NHWC [B, H, W, 3] like DinoVisionTransformer's; H and W must be multiples of 32.
"""
from __future__ import annotations

from functools import partial

import torch

from .. import ops

bf16, f32 = torch.bfloat16, torch.float32
EPS = 1e-6          # every LayerNorm of the model (models/convnext.py:106,195)


def _m(p):          # Dense / conv kernel -> bf16 [prod(leading dims), out]: the B operand, stored [K, N]
    return p.reshape(-1, p.shape[-1]).to(bf16).contiguous()


def _v(p):
    return p.to(f32).reshape(-1).contiguous()


class ConvNeXt:
    def __init__(self, params: dict, *, depths, dims, patch_size: int | None = None, drop_path_rate: float = 0.0,
                 layer_scale_init_value: float = 1e-6, in_chans: int = 3, device="cuda"):
        if drop_path_rate:
            raise NotImplementedError("stochastic depth is not on the GPU path (forward only)")
        if in_chans != 3 or len(depths) != 4 or len(dims) != 4:
            raise NotImplementedError("GPU path: 3 input channels, four stages")
        dev = torch.device(device)
        to = lambda t: torch.as_tensor(t).to(dev)
        mv = lambda tree: {k: (mv(v) if isinstance(v, dict) else to(v)) for k, v in tree.items()}
        params = mv(params)
        self.depths, self.dims, self.patch_size, self.device = list(depths), list(dims), patch_size, dev
        self.embed_dim, self.embed_dims = dims[-1], list(dims)          # :199-200
        self.n_blocks, self.n_storage_tokens = 4, 0                     # :201-203
        ln = lambda p, w="weight": (_v(p[w]), _v(p["bias"]))
        self.downsample = []
        for i in range(4):
            d = params[f"downsample_layers_{i}"]
            conv, norm = (d["layers_0"], d["layers_1"]) if i == 0 else (d["layers_1"], d["layers_0"])
            self.downsample.append({"w": _m(conv["kernel"]), "b": _v(conv["bias"]), "ln": ln(norm)})
        self.stages = []
        for i in range(4):
            s = params[f"stages_{i}"]
            self.stages.append([{"dw_w": s[f"layers_{j}"]["dwconv"]["kernel"].to(f32).reshape(49, dims[i]).contiguous(),
                                 "dw_b": _v(s[f"layers_{j}"]["dwconv"]["bias"]), "ln": ln(s[f"layers_{j}"]["norm"]),
                                 "w1": _m(s[f"layers_{j}"]["pwconv1"]["kernel"]), "b1": _v(s[f"layers_{j}"]["pwconv1"]["bias"]),
                                 "w2": _m(s[f"layers_{j}"]["pwconv2"]["kernel"]), "b2": _v(s[f"layers_{j}"]["pwconv2"]["bias"]),
                                 "gamma": _v(s[f"layers_{j}"]["gamma"])}
                                for j in range(depths[i])])
        self.norm = ln(params["norm"], "scale")

    # ------------------------------------------------------------------------------------------------ stages
    def _empty(self, *shape, dtype=f32):
        return torch.empty(*shape, dtype=dtype, device=self.device)

    def _downsample(self, i: int, x):
        """Stem (i = 0, image bf16 [n, H, W, 3]): Conv 4x4 stride 4 as im2col + GEMM, then the LayerNorm.  Layer i > 0:
        the LayerNorm written into the 2x2 conv's operand, then the GEMM.  Returns the fp32 map [n, h, w, C_i]."""
        d, C = self.downsample[i], self.dims[i]
        n, H, W, _ = x.shape
        if i == 0:
            h, w = H // 4, W // 4
            A = self._empty(n * h * w, 48, dtype=bf16)
            ops.im2col(x, A, 4)
            Y = self._empty(n * h * w, C)
            ops.gemm(A, d["w"], Y, b_mn=True, bias=d["b"])
            X = self._empty(n * h * w, C)
            ops.layernorm_fwd(Y, d["ln"][0], d["ln"][1], X, eps=EPS)
        else:
            h, w = H // 2, W // 2
            A = self._empty(n * h * w, 4 * x.shape[-1], dtype=bf16)
            ops.layernorm_patchify2(x, d["ln"][0], d["ln"][1], A, eps=EPS)
            X = self._empty(n * h * w, C)
            ops.gemm(A, d["w"], X, b_mn=True, bias=d["b"])
        return X.view(n, h, w, C)

    def _block(self, blk: dict, X):
        """x + gamma * pwconv2(GELU(pwconv1(LN(dwconv7x7(x))))) (models/convnext.py:82-95), X updated in place."""
        n, h, w, C = X.shape
        T = n * h * w
        A = self._empty(T, C, dtype=bf16)
        ops.dwconv7_layernorm(X, blk["dw_w"], blk["dw_b"], blk["ln"][0], blk["ln"][1], A, eps=EPS)
        Hid = self._empty(T, 4 * C, dtype=bf16)
        ops.gemm(A, blk["w1"], Hid, b_mn=True, bias=blk["b1"], gelu_erf=True)
        Xv = X.view(T, C)
        ops.gemm(Hid, blk["w2"], Xv, b_mn=True, bias=blk["b2"], gamma=blk["gamma"], resid=Xv)
        return X

    def _stage(self, i: int, x):
        X = self._downsample(i, x)
        for blk in self.stages[i]:
            X = self._block(blk, X)
        return X

    def _image(self, x):
        x = torch.as_tensor(x).to(self.device)
        if x.dim() != 4 or x.shape[-1] != 3:
            raise ValueError(f"ConvNeXt takes NHWC images [B, H, W, 3], got {tuple(x.shape)}")
        if x.shape[1] % 32 or x.shape[2] % 32:
            raise ValueError(f"ConvNeXt: image height {x.shape[1]} and width {x.shape[2]} must be multiples of 32 "
                             "(stem stride 4, then three 2x2 downsamplings)")
        return x.to(bf16).contiguous()

    def _tokens_out(self, buf, h, w, norm: bool, reshape: bool, out_dtype):
        """[n, 1 + h*w, C] (pooled row, tokens) -> (cls [n, C], patches [n, h*w, C] or [n, C, h, w]), one kernel."""
        n, _, C = buf.shape
        cls = self._empty(n, C, dtype=out_dtype)
        patches = self._empty(n, C, h, w, dtype=out_dtype) if reshape else self._empty(n, h * w, C, dtype=out_dtype)
        ops.layernorm_tokens_out(buf, cls, None, patches, h, w, norm=self.norm if norm else None, eps=EPS,
                                 channels_first=reshape)
        return cls, patches

    # ------------------------------------------------------------------------------------------------ public
    # models/convnext.py:210-235: x_pool = mean over H x W of the last stage, norm(cat[x_pool, tokens])
    def forward_features_list(self, x_list, masks_list):
        out = []
        for x, masks in zip(x_list, masks_list):
            X = self._image(x)
            for i in range(4):
                X = self._stage(i, X)
            n, h, w, C = X.shape
            tokens = X.view(n, h * w, C)
            buf = self._empty(n, 1 + h * w, C)
            ops.pool_tokens(tokens, buf)
            cls, patches = self._tokens_out(buf, h, w, True, False, f32)
            out.append({"x_norm_clstoken": cls, "x_storage_tokens": self._empty(n, 0, C), "x_norm_patchtokens": patches,
                        "x_prenorm": tokens, "masks": masks})
        return out

    def forward_features(self, x, masks=None):
        if isinstance(x, (list, tuple)):
            return self.forward_features_list(list(x), list(masks) if masks is not None else [None] * len(x))
        return self.forward_features_list([x], [masks])[0]

    # models/convnext.py:246-301 with upstream's semantics: "blocks" are the four stages; norms[i] is Identity for
    # i = 0..2 and the final LayerNorm for i = 3 (the reference's `norms[-n]` read as `norms[-n:]`).  The class token is
    # pooled from the stage's own map; with patch_size the map is resized (bilinear, antialiased) to (H/p, W/p) before
    # the norm.  Each selected stage's output goes through d3_layernorm_tokens_out as soon as the stage has run.
    def get_intermediate_layers(self, x, *, n=1, reshape: bool = False, return_class_token: bool = False,
                                norm: bool = True, out_dtype=f32):
        """x NHWC [B, H, W, 3]; n: the last n stages (int) or a list of stage indices.  Returns one entry per selected
        stage, in stage order: patch tokens [B, h*w, C] (reshape: [B, C, h, w]), with (h, w) the stage's map or, with
        patch_size, (H/p, W/p); zipped with the class token [B, C] when asked for.  out_dtype: float32 or bfloat16."""
        if out_dtype not in (f32, bf16):
            raise ValueError("out_dtype must be torch.float32 or torch.bfloat16")
        take = list(range(4 - n, 4)) if isinstance(n, int) else [int(i) for i in n]
        if not take or any(i < 0 or i > 3 for i in take):
            raise ValueError(f"n selects stages {take}; a ConvNeXt has stages 0..3")
        X = self._image(x)
        H, W = X.shape[1:3]
        outputs = []
        for i in range(max(take) + 1):           # later stages feed no selected output
            X = self._stage(i, X)
            if i not in take:
                continue
            B, h, w, C = X.shape
            hd, wd = (h, w) if self.patch_size is None else (H // self.patch_size, W // self.patch_size)
            buf = self._empty(B, 1 + hd * wd, C)
            if (hd, wd) == (h, w):               # the antialiased bilinear resize to the same size is the identity
                ops.pool_tokens(X.view(B, h * w, C), buf)
            else:
                ops.pool_tokens(X.view(B, h * w, C), buf, copy_tokens=False)
                ops.resize_tokens_bilinear_aa(X, buf, hd, wd, prefix=1)
            cls, patches = self._tokens_out(buf, hd, wd, norm and i == 3, reshape, out_dtype)
            outputs.append((patches, cls))
        if return_class_token:
            return tuple(outputs)
        return tuple(p for p, _ in outputs)

    def __call__(self, *args, is_training: bool = False, **kwargs):
        ret = self.forward_features(*args, **kwargs)
        if is_training:
            return ret
        return ret["x_norm_clstoken"]           # head = Identity (models/convnext.py:198,243)


convnext_sizes = {                               # models/convnext.py:304-321
    "tiny": dict(depths=[3, 3, 9, 3], dims=[96, 192, 384, 768]),
    "small": dict(depths=[3, 3, 27, 3], dims=[96, 192, 384, 768]),
    "base": dict(depths=[3, 3, 27, 3], dims=[128, 256, 512, 1024]),
    "large": dict(depths=[3, 3, 27, 3], dims=[192, 384, 768, 1536]),
}


def get_convnext_arch(arch_name: str):
    """models/convnext.py:324-335: "convnext_<size>" -> ConvNeXt with that size's depths and dims."""
    parts = arch_name.split("_")
    if len(parts) < 2 or parts[1] not in convnext_sizes:
        raise NotImplementedError(f"didn't recognize convnext size string in {arch_name!r}")
    return partial(ConvNeXt, **convnext_sizes[parts[1]])


__all__ = ["ConvNeXt", "convnext_sizes", "get_convnext_arch"]
