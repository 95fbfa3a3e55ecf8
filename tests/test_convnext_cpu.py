"""ConvNeXt without a GPU: the float64 restatement of upstream DINOv3's ConvNeXt (tests/convnext_helpers.py) against Hugging
Face's DINOv3ConvNextModel, the torch-hub key converters, the return forms of get_intermediate_layers, and the argument
checks of the new C entry points."""
import ctypes
import re

import pytest
import torch

from convnext_helpers import forward_features, intermediate_layers, stages, upstream_state_dict

f64 = torch.float64
SHRUNK = dict(depths=[1, 1, 2, 1], dims=[32, 64, 128, 256])


def _hf_state_dict(sd: dict) -> dict:
    """Upstream names -> Hugging Face's (model.stages.i.downsample_layers.j, layers.j.depthwise_conv, ...)."""
    out = {}
    for k, v in sd.items():
        if k.startswith("norms."):
            continue
        if k.startswith("norm."):
            out["layer_norm." + k[5:]] = v
            continue
        k = re.sub(r"^downsample_layers\.(\d+)\.", r"model.stages.\1.downsample_layers.", k)
        m = re.match(r"^stages\.(\d+)\.(\d+)\.(.*)$", k)
        if m:
            rest = m.group(3)
            for ours, theirs in (("dwconv", "depthwise_conv"), ("norm", "layer_norm"), ("pwconv1", "pointwise_conv1"),
                                 ("pwconv2", "pointwise_conv2")):
                rest = re.sub(rf"^{ours}\.", f"{theirs}.", rest)
            k = f"model.stages.{m.group(1)}.layers.{m.group(2)}.{rest}"
        out[k] = v
    return out


def _tree(sd):
    from dinov3_jax.checkpointer import convert_convnext_torch_hub_state_dict
    return convert_convnext_torch_hub_state_dict(sd)


@pytest.mark.parametrize("size", ["shrunk", "tiny"])
def test_restatement_matches_huggingface_float64(size):
    """The restatement, on the tree converted from an upstream-named state dict, against HF's model loaded from the
    same weights under HF's names: last_hidden_state, pooler_output and every stage's output, to 1e-9."""
    hf = pytest.importorskip("transformers.models.dinov3_convnext")
    from dinov3_jax.models import convnext_sizes
    arch = SHRUNK if size == "shrunk" else convnext_sizes["tiny"]
    sd = upstream_state_dict(arch["depths"], arch["dims"], seed=3)
    model = hf.DINOv3ConvNextModel(hf.DINOv3ConvNextConfig(depths=arch["depths"], hidden_sizes=arch["dims"],
                                                           layer_norm_eps=1e-6, hidden_act="gelu")).double().eval()
    model.load_state_dict(_hf_state_dict(sd), strict=True)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 64, 96, 3, generator=g, dtype=f64)
    with torch.no_grad():
        ref = model(pixel_values=x.permute(0, 3, 1, 2).contiguous(), output_hidden_states=True)
    tree = _tree(sd)
    mine = forward_features(tree, x)
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    assert rel(mine["x_norm_clstoken"], ref.pooler_output) < 1e-9
    got = torch.cat([mine["x_norm_clstoken"][:, None], mine["x_norm_patchtokens"]], dim=1)
    assert got.shape == ref.last_hidden_state.shape == (2, 1 + 2 * 3, arch["dims"][3])
    assert rel(got, ref.last_hidden_state) < 1e-9
    maps = stages(tree, x)
    hidden = ref.hidden_states[1:]                # HF's first entry is the input image
    assert len(hidden) == 4
    for i, (m, h) in enumerate(zip(maps, hidden)):
        assert m.permute(0, 3, 1, 2).shape == h.shape, i
        assert rel(m.permute(0, 3, 1, 2), h) < 1e-9, i
    # get_intermediate_layers without resizing: Identity norms for stages 0-2, HF's stage outputs; the final norm on 3
    outs = intermediate_layers(tree, x, [0, 1, 2, 3], return_class_token=True)
    for i, ((tok, cls), h) in enumerate(zip(outs[:3], hidden[:3])):
        assert rel(tok, h.flatten(2).transpose(1, 2)) < 1e-9 and rel(cls, h.mean(dim=(2, 3))) < 1e-9, i
    assert rel(outs[3][0], ref.last_hidden_state[:, 1:]) < 1e-9 and rel(outs[3][1], ref.pooler_output) < 1e-9


def test_converter_round_trip_and_layouts():
    from dinov3_jax.checkpointer import convert_convnext_torch_hub_state_dict, to_convnext_torch_hub_state_dict
    d, C = SHRUNK["depths"], SHRUNK["dims"]
    sd = upstream_state_dict(d, C, seed=1)
    tree = convert_convnext_torch_hub_state_dict(sd)
    assert "norms" not in tree and set(tree) == {f"downsample_layers_{i}" for i in range(4)} | {f"stages_{i}" for i in range(4)} | {"norm"}
    assert tree["downsample_layers_0"]["layers_0"]["kernel"].shape == (4, 4, 3, C[0])
    assert tree["downsample_layers_0"]["layers_1"]["weight"].shape == (C[0],)
    assert tree["downsample_layers_2"]["layers_0"]["weight"].shape == (C[1],)
    assert tree["downsample_layers_2"]["layers_1"]["kernel"].shape == (2, 2, C[1], C[2])
    blk = tree["stages_2"]["layers_1"]
    assert blk["dwconv"]["kernel"].shape == (7, 7, 1, C[2]) and blk["pwconv1"]["kernel"].shape == (C[2], 4 * C[2])
    assert set(blk["norm"]) == {"weight", "bias"} and set(tree["norm"]) == {"scale", "bias"}
    assert torch.equal(blk["pwconv2"]["kernel"], sd["stages.2.1.pwconv2.weight"].t())
    back = to_convnext_torch_hub_state_dict(tree)
    assert set(back) == set(sd)
    for k in sd:
        assert torch.equal(back[k], sd[k]), k


def test_intermediate_layer_forms_and_shapes():
    """Upstream's forms: a tuple with one entry per selected stage, the patch tokens [B, h*w, C] or, reshaped,
    [B, C, h, w], paired (patches, cls) with return_class_token; with patch_size 16 every stage is resized to
    (H/16, W/16)."""
    d, C = SHRUNK["depths"], SHRUNK["dims"]
    tree = _tree(upstream_state_dict(d, C, seed=2))
    B, H, W = 2, 64, 96
    x = torch.randn(B, H, W, 3, generator=torch.Generator().manual_seed(0), dtype=f64)
    grid = {i: (H // (4 << i), W // (4 << i)) for i in range(4)}
    for n, idx in ((1, [3]), (3, [1, 2, 3]), ([0, 2], [0, 2])):
        for p in (None, 16):
            for norm in (True, False):
                for reshape in (False, True):
                    for rct in (False, True):
                        out = intermediate_layers(tree, x, n, patch_size=p, reshape=reshape, return_class_token=rct, norm=norm)
                        assert isinstance(out, tuple) and len(out) == len(idx)
                        for o, i in zip(out, idx):
                            tok, cls = o if rct else (o, None)
                            h, w = grid[i] if p is None else (H // 16, W // 16)
                            assert tok.shape == ((B, C[i], h, w) if reshape else (B, h * w, C[i])), (n, p, i)
                            assert cls is None or cls.shape == (B, C[i])
    plain = intermediate_layers(tree, x, [1, 3], norm=False)
    shaped = intermediate_layers(tree, x, [1, 3], norm=False, reshape=True)
    for a, b in zip(plain, shaped):
        assert torch.equal(b.flatten(2).transpose(1, 2), a)
    normed = intermediate_layers(tree, x, [1, 3], return_class_token=True)
    raw = intermediate_layers(tree, x, [1, 3], norm=False, return_class_token=True)
    assert torch.equal(normed[0][0], raw[0][0]) and torch.equal(normed[0][1], raw[0][1])     # stage 1: Identity
    assert not torch.allclose(normed[1][0], raw[1][0])                                      # stage 3: the final norm


def test_sizes_and_input_checks_without_gpu():
    from dinov3_jax.models import ConvNeXt, convnext_sizes, get_convnext_arch
    assert convnext_sizes["large"] == dict(depths=[3, 3, 27, 3], dims=[192, 384, 768, 1536])
    make = get_convnext_arch("convnext_base")
    assert make.func is ConvNeXt and make.keywords == convnext_sizes["base"]
    with pytest.raises(NotImplementedError):
        get_convnext_arch("convnext_huge")
    model = ConvNeXt(_tree(upstream_state_dict(SHRUNK["depths"], SHRUNK["dims"], seed=4)), **SHRUNK, device="cpu")
    with pytest.raises(ValueError, match="multiples of 32"):
        model.forward_features(torch.zeros(1, 48, 64, 3))
    with pytest.raises(ValueError, match="stages 0..3"):
        model.get_intermediate_layers(torch.zeros(1, 64, 64, 3), n=[4])
    with pytest.raises(ValueError, match="out_dtype"):
        model.get_intermediate_layers(torch.zeros(1, 64, 64, 3), out_dtype=torch.float16)


def test_build_model_still_rejects_convnext():
    """build_model follows the reference's builder, which never reaches ConvNeXt; the model is built directly."""
    from types import SimpleNamespace
    from dinov3_jax.models import build_model
    with pytest.raises(ValueError, match="ConvNeXt"):
        build_model(SimpleNamespace(arch="convnext_tiny", patch_size=16))


def test_convnext_argument_errors_without_gpu():
    """Every argument check of the ConvNeXt entry points runs before any CUDA call: D3_ERR_ARG (-1) and a message."""
    from dinov3_jax import _native
    lib = _native.lib()
    A = 1 << 20                                              # 16-byte aligned stand-in addresses (never dereferenced)
    eps = ctypes.c_float(1e-6)

    def dw(X=A, w=A, wb=A, sc=A, bi=A, Y=A, n=2, H=7, W=7, C=96):
        return lib.d3_dwconv7_layernorm(X, w, wb, sc, bi, eps, Y, n, H, W, C, None), lib.d3_last_error()

    for kw, msg in ((dict(X=None), b"null"), (dict(w=None), b"null"), (dict(Y=None), b"null"), (dict(C=100), b"multiple of 8"),
                    (dict(C=1544), b"multiple of 8"), (dict(H=0), b"H, W >= 1"), (dict(n=-1), b"n >= 0"),
                    (dict(X=A + 4), b"aligned"), (dict(sc=A + 8), b"aligned"), (dict(Y=A + 8), b"aligned"),
                    (dict(w=A + 2), b"aligned")):
        rc, err = dw(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)

    def ps(X=A, sc=A, bi=A, Y=A, n=2, H=8, W=8, C=96):
        return lib.d3_layernorm_patchify2(X, sc, bi, eps, Y, n, H, W, C, None), lib.d3_last_error()

    for kw, msg in ((dict(Y=None), b"null"), (dict(H=7), b"even H, W"), (dict(W=0), b"even H, W"), (dict(C=6), b"multiple of 4"),
                    (dict(X=A + 4), b"aligned"), (dict(Y=A + 4), b"aligned")):
        rc, err = ps(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)

    def pt(X=A, out=A, n=2, P=49, C=96, rows=50, copy=1):
        return lib.d3_pool_tokens(X, out, n, P, C, rows, copy, None), lib.d3_last_error()

    for kw, msg in ((dict(out=None), b"null"), (dict(P=0), b"P >= 1"), (dict(C=98), b"multiple of 4"),
                    (dict(rows=49), b"rows == 1 + P"), (dict(rows=0, copy=0), b"rows >= 1"), (dict(out=A + 4), b"aligned")):
        rc, err = pt(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)

    def rs(src=A, dst=A, n=2, Hs=56, Ws=56, Hd=14, Wd=14, C=96, prefix=1):
        return lib.d3_resize_tokens_bilinear_aa(src, dst, n, Hs, Ws, Hd, Wd, C, prefix, None), lib.d3_last_error()

    for kw, msg in ((dict(src=None), b"null"), (dict(Hd=0), b"positive sizes"), (dict(C=94), b"C % 4"),
                    (dict(prefix=-1), b"prefix"), (dict(dst=A + 8), b"aligned"), (dict(Hd=7), b"too large")):
        rc, err = rs(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)
