"""-m gpu: dense features from the backbone.  d3_layernorm_tokens_out bit for bit against d3_layernorm_fwd plus torch
slicing / permute; DinoVisionTransformer.get_intermediate_layers bit for bit against forward_features and against the
CPU restatement of upstream DINOv3 (tests/features_helpers.py); the SwiGLU / mask_k_bias / untied-norm blocks through a
torch-hub state-dict round trip."""
import pytest
import torch

from features_helpers import add_norm, intermediate_layers, tree

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16


def rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-30)).item()


# ------------------------------------------------------------------------------------------------ kernel, bit for bit
@pytest.mark.parametrize("D", [192, 384, 1024, 1280, 1536, 4096])
def test_layernorm_tokens_out_matches_layernorm_fwd_bitwise(native, D):
    from dinov3_jax import ops
    g = torch.Generator(device="cuda").manual_seed(D)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    sc, bi, psc, pbi = 1 + 0.3 * rnd(D), 0.2 * rnd(D), 1 + 0.3 * rnd(D), 0.2 * rnd(D)
    eps = 1e-5
    for R in (0, 4):
        for Hp, Wp in ((14, 14), (7, 9), (64, 64)):
            for n in (1, 3):
                P, N = Hp * Wp, 1 + R + Hp * Wp
                X = (rnd(n, N, D) * 2 + 0.5).contiguous()
                for norm in ("none", "tied", "untied"):
                    if norm == "none":
                        want_pre = want_pat = X
                    else:
                        want_pat = torch.empty_like(X)
                        ops.layernorm_fwd(X.view(-1, D), sc, bi, want_pat.view(-1, D), eps=eps)
                        want_pre = want_pat
                        if norm == "untied":
                            want_pre = torch.empty_like(X)
                            ops.layernorm_fwd(X.view(-1, D), psc, pbi, want_pre.view(-1, D), eps=eps)
                    for dt in (f32, bf16):
                        for cf in (False, True):
                            cls = torch.empty(n, D, dtype=dt, device="cuda")
                            st = torch.empty(n, R, D, dtype=dt, device="cuda") if R else None
                            pt = torch.empty(*((n, D, Hp, Wp) if cf else (n, P, D)), dtype=dt, device="cuda")
                            ops.layernorm_tokens_out(X, cls, st, pt, Hp, Wp, norm=None if norm == "none" else (sc, bi),
                                                     pre_norm=(psc, pbi) if norm == "untied" else None, eps=eps,
                                                     channels_first=cf)
                            wp = want_pat[:, 1 + R:].to(dt)
                            if cf:
                                wp = wp.reshape(n, Hp, Wp, D).permute(0, 3, 1, 2)
                            tag = (R, Hp, Wp, n, norm, dt, cf)
                            assert torch.equal(cls, want_pre[:, 0].to(dt)), tag
                            assert R == 0 or torch.equal(st, want_pre[:, 1:1 + R].to(dt)), tag
                            assert torch.equal(pt, wp), tag
    torch.cuda.synchronize()


def test_layernorm_tokens_out_argument_errors(native):
    from dinov3_jax import _native, ops
    X = torch.zeros(2, 1 + 4 + 9, 128, device="cuda")
    cls, st, pt = torch.empty(2, 128, device="cuda"), torch.empty(2, 4, 128, device="cuda"), torch.empty(2, 9, 128, device="cuda")
    with pytest.raises(AssertionError):            # patches shape does not match the grid
        ops.layernorm_tokens_out(X, cls, st, pt, 3, 4)
    with pytest.raises(_native.NativeError, match="16-byte"):
        ops.layernorm_tokens_out(X, torch.empty(2 * 128 + 1, device="cuda")[1:].view(2, 128), st, pt, 3, 3)


# ------------------------------------------------------------------------------------------------ the model
def _model(cfg, bp, **kw):
    from dinov3_jax.models import DinoVisionTransformer
    ffn = kw.pop("ffn_layer", "mlp" if cfg.ffn_layer == "mlp" else f"swiglu{cfg.swiglu_align if cfg.swiglu_align > 8 else ''}")
    return DinoVisionTransformer(tree(bp, "cuda"), img_size=cfg.global_size, patch_size=16, embed_dim=cfg.embed_dim,
                                 n_blocks=cfg.depth, num_heads=cfg.heads, ffn_ratio=cfg.ffn_ratio, n_storage_tokens=cfg.n_storage,
                                 norm_layer="layernormbf16" if cfg.ln_eps == 1e-5 else "layernorm", ffn_layer=ffn,
                                 mask_k_bias=cfg.mask_k_bias, **kw)


def _small(**kw):
    from oracle.arch import ModelCfg
    base = dict(embed_dim=128, depth=3, heads=2, global_size=64, n_storage=4, layerscale=0.5, n_prototypes=16,
                head_hidden=16, head_bottleneck=8)
    return ModelCfg(**{**base, **kw})


def _params(cfg, seed=0):
    from oracle.model import init_params, sub
    return sub(init_params(cfg, seed, perturb=0.05), "student_backbone")


@pytest.mark.parametrize("untie", [False, True])
def test_intermediate_layers_equal_forward_features_bitwise(native, untie):
    cfg = _small()
    bp = _params(cfg)
    if untie:
        bp = add_norm(bp, "cls_norm", cfg.embed_dim, 5, torch.float32)
    model = _model(cfg, bp, untie_cls_and_patch_norms=untie)
    x = torch.randn(3, 64, 80, 3)
    ff = model.forward_features(x)
    ((pt, cls, st),) = model.get_intermediate_layers(x, n=1, norm=True, return_class_token=True, return_extra_tokens=True)
    assert torch.equal(pt, ff["x_norm_patchtokens"]) and torch.equal(cls, ff["x_norm_clstoken"])
    assert torch.equal(st, ff["x_storage_tokens"])
    ((pt, cls, st),) = model.get_intermediate_layers(x, n=1, norm=False, return_class_token=True, return_extra_tokens=True)
    X = ff["x_prenorm"]
    assert torch.equal(pt, X[:, 5:]) and torch.equal(cls, X[:, 0]) and torch.equal(st, X[:, 1:5])
    (r,) = model.get_intermediate_layers(x, n=[2], reshape=True)
    assert r.shape == (3, 128, 4, 5) and torch.equal(r, ff["x_norm_patchtokens"].reshape(3, 4, 5, 128).permute(0, 3, 1, 2))
    (rb,) = model.get_intermediate_layers(x, n=1, reshape=True, out_dtype=bf16)
    assert rb.dtype == bf16 and torch.equal(rb, r.to(bf16))
    if not untie:      # the tied configuration keeps the forward path it had: layernorm_fwd over every token
        assert torch.equal(model(x), ff["x_norm_clstoken"])


ORACLE_CASES = {
    "vit_s_mlp": dict(embed_dim=384, heads=6, n_storage=0),
    "swiglu64_mask_k_bias": dict(embed_dim=256, heads=4, ffn_layer="swiglu", swiglu_align=64, mask_k_bias=True, n_storage=4,
                                 ln_eps=1e-5),
    "untied_norms": dict(untie=True),
}


@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_intermediate_layers_match_oracle(native, case):
    kw = dict(ORACLE_CASES[case])
    untie = kw.pop("untie", False)
    cfg = _small(**kw)
    bp = _params(cfg, 1)
    if untie:
        bp = add_norm(bp, "cls_norm", cfg.embed_dim, 6, torch.float32)
    model = _model(cfg, bp, untie_cls_and_patch_norms=untie)
    B, H, W = 2, 64, 48
    x = torch.randn(B, H, W, 3).to(bf16).float()
    R, D, Hp, Wp = cfg.n_storage, cfg.embed_dim, H // 16, W // 16
    for n in (2, [0, 2]):
        for norm in (True, False):
            ref = intermediate_layers(bp, x, n, cfg, norm=norm, untie_cls_and_patch_norms=untie)
            for rc in (False, True):
                for re_ in (False, True):
                    for reshape in (False, True):
                        out = model.get_intermediate_layers(x, n=n, reshape=reshape, return_class_token=rc,
                                                            return_extra_tokens=re_, norm=norm)
                        assert isinstance(out, tuple) and len(out) == len(ref)
                        for o, r in zip(out, ref):
                            parts = o if (rc or re_) else (o,)
                            assert len(parts) == 1 + rc + re_
                            want_p = r["patches"].reshape(B, Hp, Wp, D).permute(0, 3, 1, 2) if reshape else r["patches"]
                            assert parts[0].shape == want_p.shape and rel(parts[0], want_p) < 2e-2, (n, norm, reshape)
                            rest = list(parts[1:])
                            if rc:
                                c = rest.pop(0)
                                assert c.shape == (B, D) and rel(c, r["cls"]) < 2e-2
                            if re_:
                                e = rest.pop(0)
                                assert e.shape == (B, R, D) and (R == 0 or rel(e, r["storage"]) < 2e-2)


def test_vit_7b_width_intermediate_layers_at_512(native):
    """embed 4096 / 32 heads of 128, one block, 512^2 crop = 1 + 4 + 1024 = 1029 tokens: the streamed head_dim-128
    attention kernels, and the channels-first tile at its widest."""
    from oracle.arch import ModelCfg
    cfg = ModelCfg(embed_dim=4096, depth=1, heads=32, ffn_ratio=3.0, global_size=512, n_storage=4, layerscale=0.5,
                   ln_eps=1e-5, n_prototypes=16, head_hidden=16, head_bottleneck=8)
    assert cfg.tokens(512) == 1029
    bp = _params(cfg)
    model = _model(cfg, bp)
    x = torch.randn(1, 512, 512, 3).to(bf16).float()
    ((pt, cls, st),) = model.get_intermediate_layers(x, n=1, reshape=True, return_class_token=True, return_extra_tokens=True)
    (r,) = intermediate_layers(bp, x, 1, cfg)
    assert pt.shape == (1, 4096, 32, 32)
    assert rel(pt, r["patches"].reshape(1, 32, 32, 4096).permute(0, 3, 1, 2)) < 2e-2
    assert rel(cls, r["cls"]) < 2e-2 and rel(st, r["storage"]) < 2e-2


def test_hub_round_trip_gives_the_same_features(native):
    """A SwiGLU64 / mask_k_bias / untied-norm tree out through to_torch_hub_state_dict, with the hub's
    attn.qkv.bias_mask entries added, and back through convert_torch_hub_state_dict: the same bits."""
    from dinov3_jax.checkpointer import convert_torch_hub_state_dict, to_torch_hub_state_dict
    cfg = _small(ffn_layer="swiglu", swiglu_align=64, mask_k_bias=True, ln_eps=1e-5)
    bp = add_norm(add_norm(_params(cfg, 2), "cls_norm", 128, 7, torch.float32), "local_cls_norm", 128, 8, torch.float32)
    sd = to_torch_hub_state_dict(tree(bp))
    for i in range(cfg.depth):
        sd[f"blocks.{i}.attn.qkv.bias_mask"] = torch.cat([torch.ones(128), torch.zeros(128), torch.ones(128)])
    params, _ = convert_torch_hub_state_dict(sd)
    kw = dict(untie_cls_and_patch_norms=True, untie_global_and_local_cls_norm=True)
    a = _model(cfg, bp, **kw)
    from dinov3_jax.checkpointer import flat_from_tree
    b = _model(cfg, flat_from_tree(params), **kw)
    x = torch.randn(2, 64, 64, 3)
    for oa, ob in zip(a.get_intermediate_layers(x, n=3, reshape=True, return_class_token=True, return_extra_tokens=True),
                      b.get_intermediate_layers(x, n=3, reshape=True, return_class_token=True, return_extra_tokens=True)):
        for ta, tb in zip(oa, ob):
            assert torch.equal(ta, tb)
    fa, fb = a.forward_features(x), b.forward_features(x)
    for k in ("x_norm_clstoken", "x_storage_tokens", "x_norm_patchtokens"):
        assert torch.equal(fa[k], fb[k])
