"""Config surface of the reference (dinov3_jax/configs/config.py:30-98) without OmegaConf: defaults ⊕ YAML file ⊕
`key=value` overrides, dotted attribute access, and the learning-rate scaling rules (:43-56).

The reference's own `ssl_default_config.yaml` / `configs/train/*.yaml` load unchanged (pass them as `config_file`);
`DEFAULTS` below only carries the keys the GPU engine honours, with the reference's default values
(ssl_default_config.yaml line numbers in SURVEY.md §5), so the package also runs without the reference checkout.
"""
from __future__ import annotations

import copy
import math
import os
from dataclasses import dataclass, field
from typing import Any, List

import yaml

from .. import distributed

DEFAULTS = {
    "compute_precision": {"param_dtype": "bf16", "reduce_dtype": "fp32", "sharding_strategy": "SHARD_GRAD_OP"},
    "dino": {"loss_weight": 1.0, "global_ignore_diagonal": True, "head_n_prototypes": 65536, "head_bottleneck_dim": 256,
             "head_nlayers": 3, "head_hidden_dim": 2048, "koleo_loss_weight": 0.1, "koleo_loss_distributed": False,
             "koleo_topk": 1, "koleo_distributed_replicas": 0, "koleo_distributed_loss_group_size": None,
             "koleo_distributed_loss_group_data": True, "reweight_dino_local_loss": False,
             "local_loss_weight_schedule": {"start": 0.5, "peak": 0.5, "end": 0.5, "warmup_epochs": 0}},
    "ibot": {"loss_weight": 1.0, "mask_sample_probability": 0.5, "mask_ratio_min_max": [0.1, 0.5],
             "mask_random_circular_shift": False, "separate_head": True, "head_n_prototypes": 65536,
             "head_bottleneck_dim": 256, "head_nlayers": 3, "head_hidden_dim": 2048},
    "gram": {"use_loss": False, "compute_stats": False, "loss_weight": 1.0, "ema_teacher": False, "ckpt": None,
             "it_load_ema_teacher": -1, "rep_update": True, "update_frequency": 50000, "it_first_update": 0,
             "max_updates": None, "normalized": True, "img_level": False, "remove_neg": False,
             "remove_only_teacher_neg": False, "tokens_used": "all", "global_teacher_resize_method": "bicubic",
             "global_teacher_resize_antialias": False, "loss_weight_schedule": None},   # ssl_default_config.yaml:55-73
    "train": {"batch_size_per_gpu": 64, "output_dir": ".", "seed": 0, "OFFICIAL_EPOCH_LENGTH": 1250,
              "centering": "sinkhorn_knopp", "checkpointing": False, "dataset_path": "synthetic", "num_workers": 0,
              "cache_dataset": False},
    "student": {"arch": "vit_large", "patch_size": 16, "drop_path_rate": 0.3, "layerscale": 1.0e-5, "ffn_layer": "mlp",
                "ffn_ratio": 4.0, "qkv_bias": True, "proj_bias": True, "ffn_bias": True, "norm_layer": "layernorm",
                "n_storage_tokens": 0, "mask_k_bias": False, "pos_embed_rope_base": 100.0},
    "teacher": {"momentum_teacher": 0.992, "final_momentum_teacher": 1, "warmup_teacher_temp": 0.04,
                "teacher_temp": 0.07, "warmup_teacher_temp_epochs": 30},
    "crops": {"global_crops_scale": [0.32, 1.0], "local_crops_number": 8, "local_crops_scale": [0.05, 0.32],
              "global_crops_size": 224, "local_crops_size": 96, "global_local_crop_pairs_ratios": 1.0,
              "gram_teacher_crops_size": None, "localcrops_subset_of_globalcrops": False, "share_color_jitter": False,
              "horizontal_flips": True, "gram_teacher_no_distortions": False, "rgb_mean": [0.485, 0.456, 0.406],
              "rgb_std": [0.229, 0.224, 0.225]},
    "optim": {"epochs": 100, "weight_decay": 0.04, "weight_decay_end": 0.4, "lr": 0.001, "warmup_epochs": 10,
              "min_lr": 1.0e-06, "schedule_trunc_extra": 0.0, "clip_grad": 3.0, "freeze_last_layer_epochs": 1,
              "scaling_rule": "sqrt_wrt_1024", "patch_embed_lr_mult": 0.2, "dino_head_wd_multiplier": 1.0,
              "layerwise_decay": 0.9, "multi_tensor_optim": True, "adamw_beta1": 0.9, "adamw_beta2": 0.999},
    "checkpointing": {"period": 3750, "max_to_keep": 3},
    "distillation": {"enabled": False, "full_cfg_path": "", "checkpoint_path": ""},   # ssl_default_config.yaml:130-133
    # k-NN (train.do_test), linear-probe (train.do_linear_eval), linear segmentation (train.do_seg_eval), linear depth
    # (train.do_depth_eval), video segmentation (train.do_video_eval, DINO's label-propagation protocol), keypoint
    # correspondence (train.do_correspondence_eval, SPair-71k PCK), unsupervised object discovery
    # (train.do_discovery_eval, TokenCut CorLoc on VOC), instance retrieval (train.do_retrieval_eval, revisited
    # Oxford / Paris mAP), logistic regression (train.do_logreg_eval; C_values null: 10^linspace(-6, 5, 45)) and
    # attentive-probe video classification (train.do_attentive_eval, a V-JEPA-style single-query probe; datasets are
    # `path label` list files or .npz) evaluations of the teacher backbone; empty dataset paths: nothing is evaluated.
    # `config_files` (the reference's list of evaluation configs) is accepted and not read.  The segmentation, depth
    # and attentive-probe schedules are this project's defaults, not a published recipe's.
    "evaluation": {"eval_period_iterations": 12500, "config_files": [],
                   "knn": {"train_dataset_path": "", "val_dataset_path": "", "nb_knn": [10, 20, 100, 200],
                           "temperature": 0.07, "batch_size": 256, "resize_size": 256, "crop_size": 224,
                           "num_workers": 8},
                   "linear": {"train_dataset_path": "", "val_dataset_path": "", "epochs": 10, "epoch_length": 1250,
                              "batch_size": 128,
                              "learning_rates": [1e-5, 2e-5, 5e-5, 1e-4, 2e-4, 5e-4, 1e-3, 2e-3, 5e-3, 1e-2, 2e-2,
                                                 5e-2, 0.1],
                              "n_last_blocks_list": [1, 4], "avgpools": [False, True], "crop_size": 224,
                              "resize_size": 256, "num_workers": 8, "seed": 0},
                   "segmentation": {"train_dataset_path": "", "val_dataset_path": "", "num_classes": 150,
                                    "n_last_blocks": 1, "batch_size": 16, "crop_size": 512, "iterations": 40000,
                                    "lr": 1e-3, "weight_decay": 1e-3, "warmup_iterations": 1500, "num_workers": 8,
                                    "seed": 0},
                   "depth": {"train_dataset_path": "", "val_dataset_path": "", "n_last_blocks": 1, "use_cls_token": True,
                             "n_bins": 256, "min_depth": 0.001, "max_depth": 10.0, "batch_size": 16,
                             "crop_size": [416, 544], "iterations": 38400, "lr": 1e-3, "weight_decay": 1e-3,
                             "warmup_iterations": 1500, "eval_crop": "eigen", "depth_scale": 1000, "num_workers": 8,
                             "seed": 0},
                   "video": {"dataset_path": "", "n_last_frames": 7, "size_mask_neighborhood": 12, "topk": 5,
                             "temperature": 0.1, "short_side": 480, "batch_size": 16, "num_workers": 4,
                             "save_masks": False},
                   "correspondence": {"dataset_path": "", "split": "test", "image_size": 512,
                                      "alphas": [0.01, 0.05, 0.1], "batch_size": 16, "num_workers": 4},
                   "discovery": {"dataset_path": "", "split": "trainval", "tau": 0.2, "eps": 1e-5,
                                 "remove_difficult": False, "batch_size": 16, "num_workers": 4, "save_boxes": False},
                   "retrieval": {"dataset_path": "", "dataset": "roxford5k", "image_size": 512,
                                 "scales": [1.0, 0.7071067811865476, 0.5], "batch_size": 16, "num_workers": 4,
                                 "save_ranks": False},
                   "logreg": {"train_dataset_path": "", "val_dataset_path": "", "C_values": None,
                              "holdout_fraction": 0.1, "max_iter": 1000, "tol": 1e-6, "history": 10,
                              "avgpool": False, "batch_size": 256, "resize_size": 256, "crop_size": 224,
                              "num_workers": 8, "seed": 0},
                   "attentive": {"train_dataset_path": "", "val_dataset_path": "",
                                 "learning_rates": [1e-4, 3e-4, 1e-3], "epochs": 20, "warmup_epochs": 0,
                                 "weight_decay": 0.01, "batch_size": 16, "num_frames": 16, "frame_step": 4,
                                 "num_segments": 2, "num_views": 3, "crop_size": 224, "num_workers": 8, "seed": 0}},
}


class Cfg(dict):
    """dict with attribute access (cfg.optim.lr) — the subset of OmegaConf behaviour the training code uses."""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError as e:
            raise AttributeError(k) from e
        return v

    def __setattr__(self, k, v):
        self[k] = v

    @staticmethod
    def wrap(d):
        if isinstance(d, dict):
            return Cfg({k: Cfg.wrap(v) for k, v in d.items()})
        if isinstance(d, list):
            return [Cfg.wrap(v) for v in d]
        return d


def _merge(base: dict, over: dict) -> dict:
    for k, v in over.items():
        if isinstance(v, dict) and isinstance(base.get(k), dict):
            _merge(base[k], v)
        else:
            base[k] = v
    return base


def _apply_opt(cfg: dict, opt: str):
    key, _, val = opt.partition("=")
    if not _:
        raise ValueError(f"override must be key=value, got {opt!r}")
    node = cfg
    parts = key.split(".")
    for p in parts[:-1]:
        node = node.setdefault(p, {})
    node[parts[-1]] = yaml.safe_load(val)


@dataclass
class DinoV3SetupArgs:
    config_file: str | None = None
    pretrained_weights: str | None = None
    shard_unsharded_model: bool = False
    output_dir: str = ""
    opts: List[Any] = field(default_factory=list)


def get_default_config() -> Cfg:
    return Cfg.wrap(copy.deepcopy(DEFAULTS))


def get_cfg_from_args(args: DinoV3SetupArgs, strict: bool = False) -> Cfg:
    cfg = copy.deepcopy(DEFAULTS)
    if args.config_file:
        with open(args.config_file) as f:
            _merge(cfg, yaml.safe_load(f) or {})
    for o in (args.opts or []):
        _apply_opt(cfg, o)
    if args.output_dir:
        cfg["train"]["output_dir"] = os.path.realpath(args.output_dir)
    return Cfg.wrap(cfg)


def apply_scaling_rules_to_cfg(config: Cfg) -> Cfg:
    """configs/config.py:43-56: lr scaling by global batch size."""
    if "schedules" in config:
        return config
    gbs = config.train.batch_size_per_gpu * distributed.get_world_size()
    if config.optim.scaling_rule == "linear_wrt_256":
        config.optim.lr *= gbs / 256.0
    elif config.optim.scaling_rule == "sqrt_wrt_1024":
        config.optim.lr *= 4 * math.sqrt(gbs / 1024.0)
    return config


def setup_config(args: DinoV3SetupArgs, strict_cfg: bool = False) -> Cfg:
    return apply_scaling_rules_to_cfg(get_cfg_from_args(args, strict=strict_cfg))
