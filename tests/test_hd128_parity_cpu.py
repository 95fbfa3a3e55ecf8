"""CPU parity pins for head_dim 128 (vit_7b: embed 4096, 32 heads).

* the oracle's ViT forward at embed 256 / 2 heads against Hugging Face transformers' DINOv3ViTModel (an independent
  port of upstream DINOv3): RoPE frequencies 100^(2i/64), i < 32, rotation pairs (d, d + 64), attention scale 128^-0.5;
* the same against tests/golden/hd128_vectors.npz, produced by executing the reference's own RopePositionEmbedding and
  DinoVisionTransformer (tests/golden/make_hd128_golden.py);
* the vit_7b entries of the arch table, factory, build_model and the YAML mapping."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN

D, HEADS, DEPTH = 256, 2, 2


@pytest.mark.parametrize("n_storage", [4, 0])
def test_oracle_vit_hd128_matches_huggingface_dinov3(n_storage):
    hf = pytest.importorskip("transformers.models.dinov3_vit")
    from test_hf_crosscheck_cpu import _to_hf_state_dict
    from oracle.arch import ModelCfg
    from oracle.model import backbone_forward, formula_images, formula_params, sub
    size = 64
    cfg = ModelCfg(embed_dim=D, depth=DEPTH, heads=HEADS, global_size=size, local_size=32, n_storage=n_storage, ln_eps=1e-5,
                   mlp_second_act=False, n_prototypes=16, head_hidden=16, head_bottleneck=8)
    assert cfg.head_dim == 128
    bp = sub(formula_params(cfg, 6), "student_backbone")
    if not n_storage:
        bp["storage_tokens"] = torch.zeros(1, 0, D, dtype=torch.float64)
    hcfg = hf.DINOv3ViTConfig(patch_size=16, hidden_size=D, intermediate_size=4 * D, num_hidden_layers=DEPTH,
                              num_attention_heads=HEADS, hidden_act="gelu_pytorch_tanh", layer_norm_eps=1e-5, rope_theta=100.0,
                              image_size=size, query_bias=True, key_bias=True, value_bias=True, proj_bias=True, mlp_bias=True,
                              layerscale_value=1.0, num_register_tokens=n_storage, use_gated_mlp=False)
    model = hf.DINOv3ViTModel(hcfg).double().eval()
    missing, unexpected = model.load_state_dict(_to_hf_state_dict(bp, DEPTH, D), strict=False)
    assert not unexpected and all("inv_freq" in k for k in missing), (missing, unexpected)
    n, P = 3, (size // 16) ** 2
    x = formula_images((n, size, size, 3), 79)
    masks = (torch.arange(n * P).reshape(n, P) * 7 % 5 == 0)
    bp_o = bp if n_storage else {k: v for k, v in bp.items() if k != "storage_tokens"}
    for mk in (masks, None):
        want = backbone_forward(bp_o, [x], [mk], cfg)[0]
        with torch.no_grad():
            got = model(pixel_values=x.permute(0, 3, 1, 2).contiguous(), bool_masked_pos=mk).last_hidden_state
        ref = torch.cat([want["x_norm_clstoken"][:, None], want["x_storage_tokens"], want["x_norm_patchtokens"]], dim=1)
        assert got.shape == ref.shape
        err = (got - ref).abs().max().item() / ref.abs().max().item()
        assert err < 2e-6, err            # HF builds its sin / cos tables in float32 even for a float64 model


@pytest.fixture(scope="module")
def fixture():
    with np.load(os.path.join(GOLDEN, "hd128_vectors.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("H,W", [(3, 5), (4, 4), (14, 14)])
def test_rope_tables_hd128_match_reference(fixture, H, W):
    """RopePositionEmbedding(embed_dim=256, num_heads=2) of the reference: [H*W, 128] tables.  The oracle's tables and
    the engine's (what d3_rope and the fused inverse RoPE read) agree with it."""
    from dinov3_jax.engine.core import rope_tables
    from oracle.model import rope_sincos
    ws, wc = fixture[f"rope_sin_{H}x{W}"], fixture[f"rope_cos_{H}x{W}"]
    assert ws.shape == (H * W, 128)
    s, c = rope_sincos(H, W, 128, 100.0, torch.float64)
    assert np.abs(s.numpy() - ws).max() < 1e-6 and np.abs(c.numpy() - wc).max() < 1e-6
    es, ec = rope_tables(H, W, 128, 100.0, "cpu")
    assert np.abs(es.double().numpy() - ws).max() < 1e-6 and np.abs(ec.double().numpy() - wc).max() < 1e-6


@pytest.mark.parametrize("case,n_storage,ln_eps,seed,keys", [("r4", 4, 1e-5, 12, (41, 42)), ("r0", 0, 1e-6, 13, (43, 44))])
def test_oracle_vit_hd128_matches_reference_fixture(fixture, case, n_storage, ln_eps, seed, keys):
    from oracle.arch import ModelCfg
    from oracle.model import backbone_forward, formula_images, formula_params, sub
    cfg = ModelCfg(embed_dim=D, depth=DEPTH, heads=HEADS, global_size=64, local_size=32, n_prototypes=16, head_hidden=16,
                   head_bottleneck=8, n_storage=n_storage, ln_eps=ln_eps)
    bp = sub(formula_params(cfg, seed), "student_backbone")
    if not n_storage:
        bp = {k: v for k, v in bp.items() if k != "storage_tokens"}
    g, l = formula_images((2, 64, 64, 3), keys[0]), formula_images((3, 32, 32, 3), keys[1])
    masks = torch.as_tensor(fixture["vit_masks"])
    og, ol = backbone_forward(bp, [g, l], [masks, None], cfg)
    for tag, o in (("g", og), ("l", ol)):
        for name, k in (("cls", "x_norm_clstoken"), ("storage", "x_storage_tokens"), ("patch", "x_norm_patchtokens")):
            want = fixture[f"vit_{case}_{tag}_{name}"]
            got = o[k].numpy()
            assert got.shape == want.shape, (tag, name)
            if want.size:
                assert np.abs(got - want).max() <= 1e-9 * max(np.abs(want).max(), 1.0), (tag, name)


# ------------------------------------------------------------------------------------------------ vit_7b configuration
def test_vit_7b_arch_factory_and_build_model():
    from types import SimpleNamespace

    from dinov3_jax import models
    from dinov3_jax.engine.config import ARCHS, config_for
    assert ARCHS["vit_7b"] == (4096, 40, 32)
    c = config_for("vit_7b")
    assert (c.embed_dim, c.depth, c.heads, c.head_dim, c.ffn_ratio) == (4096, 40, 32, 128, 3.0)
    f = models.vit_7b(patch_size=16, n_storage=4)
    assert f == config_for("vit_7b", n_storage=4)
    student, teacher, dim = models.build_model(SimpleNamespace(arch="vit_7b", patch_size=16))
    assert student == teacher == config_for("vit_7b") and dim == 4096
    assert config_for("vit_large").ffn_ratio == 4.0                          # the other archs keep their defaults
    with pytest.raises(ValueError):
        models.build_model(SimpleNamespace(arch="convnext_base", patch_size=16))


def _cfg7b(*opts):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    return setup_config(DinoV3SetupArgs(opts=["student.arch=vit_7b", "student.ffn_layer=swiglu64", "student.ffn_ratio=3",
                                              "student.norm_layer=layernormbf16", "student.n_storage_tokens=4",
                                              "student.mask_k_bias=true", *opts]))


def test_vit_7b_yaml_mapping():
    from dinov3_jax.engine import config_from_reference_cfg
    e = config_from_reference_cfg(_cfg7b())
    assert (e.embed_dim, e.depth, e.heads, e.head_dim, e.ffn_ratio) == (4096, 40, 32, 128, 3.0)
    assert e.ffn_layer == "swiglu" and e.swiglu_align == 64 and e.mask_k_bias and e.n_storage == 4 and e.ln_eps == 1e-5
    assert e.swiglu_hidden == 8192
    e2 = config_from_reference_cfg(_cfg7b("student.fp8_enabled=true"))       # ignored, as the reference does
    assert e2 == e


@pytest.mark.parametrize("opt", ["student.qkv_bias=false", "student.untie_global_and_local_cls_norm=true",
                                 "student.untie_cls_and_patch_norms=true"])
def test_vit_7b_yaml_options_not_on_the_gpu_path_raise(opt):
    from dinov3_jax.engine import config_from_reference_cfg
    with pytest.raises(NotImplementedError):
        config_from_reference_cfg(_cfg7b(opt))


def test_qkv_bias_check_is_scoped_to_vit_7b():
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.engine import config_from_reference_cfg
    e = config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["student.qkv_bias=false"])))
    assert (e.embed_dim, e.heads) == (1024, 16)
