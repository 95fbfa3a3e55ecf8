"""Dense features (get_intermediate_layers) without a GPU: the CPU restatement of upstream DINOv3's semantics against
Hugging Face's `DINOv3ViTModel` in float64, the argument checks of d3_layernorm_tokens_out, and the upstream return forms."""
import ctypes

import pytest
import torch

from features_helpers import intermediate_layers

f64 = torch.float64


def _hf_state_dict(bp: dict, depth: int, D: int, swiglu: bool, mask_k_bias: bool) -> dict:
    sd = {"embeddings.cls_token": bp["cls_token"], "embeddings.mask_token": bp["mask_token"].reshape(1, 1, D),
          "embeddings.register_tokens": bp.get("storage_tokens", torch.zeros(1, 0, D, dtype=f64)),
          "embeddings.patch_embeddings.weight": bp["patch_embed/proj/kernel"].permute(3, 2, 0, 1).contiguous(),
          "embeddings.patch_embeddings.bias": bp["patch_embed/proj/bias"], "norm.weight": bp["norm/scale"],
          "norm.bias": bp["norm/bias"]}
    for i in range(depth):
        b, h = f"blocks_{i}/", f"model.layer.{i}."
        qkv_w, qkv_b = bp[b + "attn/qkv/kernel"], bp[b + "attn/qkv/bias"]
        for j, name in enumerate(("q_proj", "k_proj", "v_proj")):
            sd[h + f"attention.{name}.weight"] = qkv_w[:, j * D:(j + 1) * D].t().contiguous()
            if not (mask_k_bias and name == "k_proj"):      # HF has no key bias where upstream masks it to zero
                sd[h + f"attention.{name}.bias"] = qkv_b[j * D:(j + 1) * D]
        sd[h + "attention.o_proj.weight"] = bp[b + "attn/proj/kernel"].t().contiguous()
        sd[h + "attention.o_proj.bias"] = bp[b + "attn/proj/bias"]
        sd[h + "norm1.weight"], sd[h + "norm1.bias"] = bp[b + "norm1/scale"], bp[b + "norm1/bias"]
        sd[h + "norm2.weight"], sd[h + "norm2.bias"] = bp[b + "norm2/scale"], bp[b + "norm2/bias"]
        sd[h + "layer_scale1.lambda1"], sd[h + "layer_scale2.lambda1"] = bp[b + "ls1/gamma"], bp[b + "ls2/gamma"]
        ffn = (("w1", "gate_proj"), ("w2", "up_proj"), ("w3", "down_proj")) if swiglu else \
            (("Dense_0", "up_proj"), ("Dense_1", "down_proj"))
        for ours, theirs in ffn:
            sd[h + f"mlp.{theirs}.weight"] = bp[b + f"mlp/{ours}/kernel"].t().contiguous()
            sd[h + f"mlp.{theirs}.bias"] = bp[b + f"mlp/{ours}/bias"]
    return sd


CASES = [  # ffn_layer, swiglu_align, n_storage, mask_k_bias
    ("mlp", 8, 0, False),
    ("mlp", 8, 4, True),
    ("swiglu", 64, 4, True),
    ("swiglu", 8, 0, False),
]


@pytest.mark.parametrize("ffn,align,R,mask_k_bias", CASES)
def test_intermediate_layers_match_huggingface_float64(ffn, align, R, mask_k_bias):
    """Upstream semantics pinned against a second code base: HF's per-layer outputs (forward hooks on model.layer[i])
    plus its final norm.  HF builds its RoPE tables in float32 even for a float64 model, so the hook on
    rope_embeddings hands it the float64 tables (their float32 agreement is test_hf_crosscheck_cpu.py's)."""
    hf = pytest.importorskip("transformers.models.dinov3_vit")
    from oracle.arch import ModelCfg
    from oracle.model import formula_images, formula_params, rope_sincos, sub
    D, depth, heads, size = 128, 3, 2, 48
    cfg = ModelCfg(embed_dim=D, depth=depth, heads=heads, global_size=size, local_size=32, n_storage=R, ln_eps=1e-5,
                   mlp_second_act=False, mask_k_bias=mask_k_bias, ffn_layer=ffn, swiglu_align=align, n_prototypes=16,
                   head_hidden=16, head_bottleneck=8)
    bp = sub(formula_params(cfg, 11), "student_backbone")
    swiglu = ffn == "swiglu"
    hcfg = hf.DINOv3ViTConfig(patch_size=16, hidden_size=D, intermediate_size=cfg.swiglu_hidden if swiglu else 4 * D,
                              num_hidden_layers=depth, num_attention_heads=heads,
                              hidden_act="silu" if swiglu else "gelu_pytorch_tanh", layer_norm_eps=1e-5, rope_theta=100.0,
                              image_size=size, query_bias=True, key_bias=not mask_k_bias, value_bias=True, proj_bias=True,
                              mlp_bias=True, layerscale_value=1.0, num_register_tokens=R, use_gated_mlp=swiglu)
    model = hf.DINOv3ViTModel(hcfg).double().eval()
    missing, unexpected = model.load_state_dict(_hf_state_dict(bp, depth, D, swiglu, mask_k_bias), strict=False)
    assert not unexpected and all("inv_freq" in k for k in missing), (missing, unexpected)
    Hp = size // 16
    sin, cos = rope_sincos(Hp, Hp, D // heads, 100.0, f64)
    model.rope_embeddings.register_forward_hook(lambda mod, args, out: (cos, sin))
    layer_out = {}
    for i, layer in enumerate(model.model.layer):
        layer.register_forward_hook(lambda mod, args, out, i=i: layer_out.__setitem__(i, out[0] if isinstance(out, tuple) else out))
    x = formula_images((2, size, size, 3), 91)
    with torch.no_grad():
        model(pixel_values=x.permute(0, 3, 1, 2).contiguous())
    for n in (2, [0, 2]):
        idx = list(range(depth - n, depth)) if isinstance(n, int) else n
        for norm in (True, False):
            got = intermediate_layers(bp, x, n, cfg, norm=norm)
            assert len(got) == len(idx)
            for g, i in zip(got, idx):
                with torch.no_grad():
                    want = model.norm(layer_out[i]) if norm else layer_out[i]
                mine = torch.cat([g["cls"][:, None], g["storage"], g["patches"]], dim=1)
                assert mine.shape == want.shape == (2, 1 + R + Hp * Hp, D)
                err = ((mine - want).abs().max() / want.abs().max()).item()
                assert err < 1e-9, (n, norm, i, err)


def test_layernorm_tokens_out_argument_errors_without_gpu():
    """Every argument check of d3_layernorm_tokens_out runs before any CUDA call: D3_ERR_ARG (-1) and a message."""
    from dinov3_jax import _native
    lib = _native.lib()
    A = 1 << 20                                             # 16-byte aligned stand-in addresses (never dereferenced)
    n, R, Hp, Wp, D = 2, 4, 7, 9, 256
    N = 1 + R + Hp * Wp

    def call(X=A, sc=A, bi=A, psc=A, pbi=A, n=n, N=N, R=R, Hp=Hp, Wp=Wp, D=D, cls=A, st=A, pt=A, f32=1, cf=0):
        return lib.d3_layernorm_tokens_out(X, sc, bi, psc, pbi, ctypes.c_float(1e-6), n, N, R, Hp, Wp, D, cls, st, pt, f32, cf,
                                           None), lib.d3_last_error()

    for kw, msg in ((dict(X=None), b"null"), (dict(cls=None), b"null"), (dict(pt=None), b"null"), (dict(st=None), b"null"),
                    (dict(bi=None), b"all given"), (dict(psc=None, pbi=None), b"all given"),
                    (dict(N=N + 1), b"N != 1 + R + Hp*Wp"), (dict(R=R - 1), b"N != 1 + R + Hp*Wp"),
                    (dict(D=258), b"multiple of 4"), (dict(D=0), b"multiple of 4"), (dict(Hp=0, N=1 + R), b"Hp, Wp"),
                    (dict(X=A + 4), b"aligned"), (dict(sc=A + 8), b"aligned"), (dict(cls=A + 8), b"aligned"),
                    (dict(cls=A + 4, f32=0), b"aligned"), (dict(pt=A + 8), b"aligned"), (dict(pt=A + 2, cf=1), b"aligned"),
                    (dict(pt=A + 1, cf=1, f32=0), b"aligned")):
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)


@pytest.mark.parametrize("return_class_token", [False, True])
@pytest.mark.parametrize("return_extra_tokens", [False, True])
@pytest.mark.parametrize("reshape", [False, True])
def test_return_forms_follow_upstream(return_class_token, return_extra_tokens, reshape):
    """models/vision_transformer.py:294-312: one entry per selected block; a bare patch tensor, or a tuple (patches,
    cls), (patches, extra) or (patches, cls, extra); patches [B, P, D] or, reshaped, [B, D, H/p, W/p]."""
    from dinov3_jax.models.vision_transformer import pack_intermediate_layers
    from oracle.arch import ModelCfg
    from oracle.model import formula_images, formula_params, sub
    B, H, W, R, D = 2, 48, 32, 4, 128
    cfg = ModelCfg(embed_dim=D, depth=3, heads=2, n_storage=R, n_prototypes=16, head_hidden=16, head_bottleneck=8)
    bp = sub(formula_params(cfg, 3, dtype=torch.float32), "student_backbone")
    blocks = intermediate_layers(bp, formula_images((B, H, W, 3), 5, torch.float32), [0, 2], cfg)
    Hp, Wp = H // 16, W // 16
    per_block = [(o["cls"], o["storage"], o["patches"].reshape(B, Hp, Wp, D).permute(0, 3, 1, 2) if reshape else o["patches"])
                 for o in blocks]
    out = pack_intermediate_layers(per_block, return_class_token, return_extra_tokens)
    assert isinstance(out, tuple) and len(out) == 2
    shape_p = (B, D, Hp, Wp) if reshape else (B, Hp * Wp, D)
    for o, blk in zip(out, blocks):
        parts = o if (return_class_token or return_extra_tokens) else (o,)
        assert isinstance(parts, tuple) and len(parts) == 1 + return_class_token + return_extra_tokens
        assert parts[0].shape == shape_p
        if reshape:
            assert torch.equal(parts[0].permute(0, 2, 3, 1).reshape(B, Hp * Wp, D), blk["patches"])
        rest = list(parts[1:])
        if return_class_token:
            c = rest.pop(0)
            assert c.shape == (B, D) and torch.equal(c, blk["cls"])
        if return_extra_tokens:
            e = rest.pop(0)
            assert e.shape == (B, R, D) and torch.equal(e, blk["storage"])
