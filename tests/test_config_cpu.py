"""Host-side mirrors of the reference's config / schedule surface (CPU)."""
import math

import pytest

from dinov3_jax.configs import DinoV3SetupArgs, setup_config
from dinov3_jax.engine import config_from_reference_cfg
from dinov3_jax.train.train import build_schedulers, get_args_parser


def test_defaults_follow_reference_yaml_and_scaling_rule():
    cfg = setup_config(DinoV3SetupArgs())
    assert cfg.dino.head_n_prototypes == 65536 and cfg.crops.local_crops_number == 8 and cfg.optim.clip_grad == 3.0
    assert abs(cfg.optim.lr - 0.001 * 4 * math.sqrt(64 / 1024.0)) < 1e-12          # sqrt_wrt_1024 (configs/config.py:52-54)
    e = config_from_reference_cfg(cfg)
    assert (e.embed_dim, e.depth, e.heads) == (1024, 24, 16)


def test_overrides_and_linear_rule():
    cfg = setup_config(DinoV3SetupArgs(opts=["optim.scaling_rule=linear_wrt_256", "train.batch_size_per_gpu=32", "student.arch=vit_base"]))
    assert abs(cfg.optim.lr - 0.001 * 32 / 256) < 1e-12 and config_from_reference_cfg(cfg).embed_dim == 768
    with pytest.raises(ValueError):
        setup_config(DinoV3SetupArgs(opts=["novalue"]))


def test_schedulers_match_reference_construction():
    cfg = setup_config(DinoV3SetupArgs())
    lr, wd, mom, temp, last = build_schedulers(cfg)
    L = cfg.train.OFFICIAL_EPOCH_LENGTH
    assert len(lr.schedule) == 100 * L and len(temp.schedule) == 30 * L
    assert lr[0] == 0.0 and abs(lr[10 * L - 1] - cfg.optim.lr) < 1e-12
    assert (last.schedule[:L] == 0).all() and last[L] == lr[L]                      # frozen first epoch (train.py:169-173)
    assert abs(temp[0] - 0.04) < 1e-12 and abs(temp[10 ** 9] - 0.07) < 1e-12 and abs(mom[0] - 0.992) < 1e-12
    assert abs(wd[0] - 0.04) < 1e-12 and wd[100 * L - 1] < 0.4 + 1e-9


def test_cli_surface():
    a = get_args_parser().parse_args(["--config-file", "x.yaml", "--opts", "a.b=1", "c=2", "--output-dir", "out"])
    assert a.config_file == "x.yaml" and a.opts == ["a.b=1", "c=2"] and a.output_dir == "out"


def test_storage_tokens_and_norm_layer_map_onto_the_engine_config():
    """student.n_storage_tokens / student.norm_layer (models/vision_transformer.py:38-42,106-111) are on the GPU path;
    so are SwiGLU (all four alignments) and mask_k_bias (SURVEY §8f.1); RMSNorm is not and is rejected loudly."""
    cfg = setup_config(DinoV3SetupArgs(opts=["student.n_storage_tokens=4", "student.norm_layer=layernormbf16"]))
    e = config_from_reference_cfg(cfg)
    assert e.n_storage == 4 and e.prefix == 5 and e.ln_eps == 1e-5
    assert e.tokens(224) == 196 + 5 and e.tokens(96) == 36 + 5
    assert config_from_reference_cfg(setup_config(DinoV3SetupArgs())).ln_eps == 1e-6
    with pytest.raises(NotImplementedError):
        config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["student.norm_layer=rmsnorm"])))
    s = config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["student.ffn_layer=swiglu64", "student.mask_k_bias=true"])))
    assert s.ffn_layer == "swiglu" and s.swiglu_align == 64 and s.mask_k_bias and not s.mlp_second_act
    assert s.swiglu_hidden == 2752 and s.ffn_width == 2752                  # int(4096 * 2 / 3) = 2730 -> next multiple of 64
    assert config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["student.ffn_layer=swiglu"]))).swiglu_hidden == 2736


def test_parameter_spec_contains_storage_tokens_with_the_reference_multipliers():
    from dinov3_jax.engine.config import config_for
    from dinov3_jax.engine.params import backbone_spec, lr_wd_multipliers
    cfg = config_for("vit_small", n_storage=4)
    spec = {n: (s, k) for n, s, k in backbone_spec(cfg)}
    assert spec["storage_tokens"] == ((1, 4, 384), "vec")
    lr, wd, last = lr_wd_multipliers("backbone", "storage_tokens", cfg)
    lr_cls, wd_cls, _ = lr_wd_multipliers("backbone", "cls_token", cfg)
    assert (lr, wd, last) == (lr_cls, wd_cls, False)            # same layer-0 group as cls / mask tokens (param_groups.py:117-129)
    assert abs(lr - cfg.layerwise_decay ** (cfg.depth + 1)) < 1e-12


def test_gram_keys_map_onto_the_engine_config():
    """gram.* (configs/ssl_default_config.yaml:55-73; train/ssl_meta_arch.py:165-254): the batch-level Gram term with the
    EMA teacher or a frozen snapshot is on the GPU path (SURVEY 8f.2); the variants that are not raise."""
    e = config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.ema_teacher=true",
                                                                      "gram.loss_weight=2.0", "gram.remove_only_teacher_neg=true"])))
    assert e.gram_use_loss and e.gram_ema_teacher and e.gram_loss_weight == 2.0 and e.gram_remove_only_teacher_neg
    assert not e.gram_img_level and e.gram_tokens_used == "all" and e.gram_normalized
    e = config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.it_load_ema_teacher=0",
                                                                      "gram.update_frequency=100", "crops.gram_teacher_crops_size=224"])))
    assert e.gram_use_loss and not e.gram_ema_teacher and e.gram_it_load_ema_teacher == 0 and e.gram_update_frequency == 100
    assert not config_from_reference_cfg(setup_config(DinoV3SetupArgs())).gram_use_loss
    with pytest.raises(ValueError):              # no checkpoint and no load iteration (ssl_meta_arch.py:215-218)
        config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true"])))
    with pytest.raises(NotImplementedError):
        config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.ema_teacher=true", "gram.ckpt=/x"])))
    e = config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.ema_teacher=true",
                                                                      "gram.tokens_used=masked"])))
    assert e.gram_tokens_used == "masked"
    assert config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.ema_teacher=true",
                                                                         "gram.img_level=true"]))).gram_img_level
    with pytest.raises(ValueError):              # ssl_meta_arch.py:222-223
        config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.ema_teacher=true",
                                                                      "gram.tokens_used=unmasked", "gram.img_level=true"])))
    # a gram teacher at its own resolution: up to 448 tokens per crop (320^2 at patch 16), bicubic resize of its features
    frozen = ["gram.use_loss=true", "gram.it_load_ema_teacher=0"]
    e = config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=frozen + ["crops.gram_teacher_crops_size=320",
                                                                             "gram.global_teacher_resize_antialias=true"])))
    assert e.gram_teacher_size == 320 and e.gram_resize_antialias
    with pytest.raises(NotImplementedError):
        config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=frozen + ["crops.gram_teacher_crops_size=448"])))
    with pytest.raises(ValueError):              # ssl_meta_arch.py:243-244
        config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.ema_teacher=true",
                                                                      "crops.gram_teacher_crops_size=224"])))


def test_meta_arch_gram_attributes_and_errors():
    """SSLMetaArch mirrors the gram attributes and configuration errors of train/ssl_meta_arch.py:165-254."""
    from dinov3_jax.train import SSLMetaArch
    m = SSLMetaArch(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.ema_teacher=true"])))
    assert m.gram_use_loss and m.gram_ema_teacher and not m.has_gram_teacher and m.gram_loss_weight == 1.0
    assert not m.gram_teacher_initialized and m.engine_config.gram_use_loss
    m = SSLMetaArch(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.it_load_ema_teacher=0",
                                                        "crops.gram_teacher_crops_size=224"])))
    assert m.has_gram_teacher and m.engine_config.gram_teacher_size == 224
    with pytest.raises(ValueError, match="gram_teacher_crops_size must be set"):
        SSLMetaArch(setup_config(DinoV3SetupArgs(opts=["gram.use_loss=true", "gram.it_load_ema_teacher=0"])))
    assert not SSLMetaArch(setup_config(DinoV3SetupArgs())).gram_use_loss
