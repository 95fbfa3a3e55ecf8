"""Training driver with the reference's entry points (dinov3_jax/train/train.py): `get_args_parser`, `main`,
`do_train`, `build_schedulers`, `build_optimizer`, `train_step`, `build_data_loader_from_cfg`,
`build_multi_resolution_data_loader_from_cfg`.

Launch one process per GPU:  torchrun --nproc-per-node N -m dinov3_jax.train.train --config-file cfg.yaml --opts k=v
The loop keeps the reference's shape (:622-706) minus its per-step host syncs: metrics are read every `print_freq`.

Two ways to run a step, same arithmetic:
  * `train_step(params, batch, optimizer_state, teacher_temp, iteration, root_rngs)` -> `(params, optimizer_state,
    loss, metrics_dict)` followed by `model.update_ema()(ema_params, params, mom)` — the reference's call contract
    (:491-565, :666, ssl_meta_arch.py:644-660).  `params` / `optimizer_state` are handles onto engine-resident flat
    buffers (the reference donates both arguments, :611, so in-place update is the same contract);
  * `engine.train_step(batch, ...)` — what `do_train` uses: the EMA is fused into the AdamW kernel.
"""
from __future__ import annotations

import argparse
import math
import os
import sys
import time
from functools import partial

import torch

from ..configs import DinoV3SetupArgs, setup_config
from .cosine_lr_scheduler import CosineScheduler
from .ssl_meta_arch import SSLMetaArch


def get_args_parser(add_help: bool = True):
    """Flags of the reference parser (train/train.py:51-72): same names, positional `seed` (optional here, default 12)."""
    p = argparse.ArgumentParser("DINOv3 training (GPU engine)", add_help=add_help)
    p.add_argument("--config-file", default="", metavar="FILE")
    p.add_argument("--no-resume", action="store_true")
    p.add_argument("--eval-only", action="store_true", help="eval only")
    p.add_argument("--eval", type=str, default="", help="eval type")
    p.add_argument("--eval-pretrained-weights", type=str, default="", help="path to weights")
    p.add_argument("--opts", default=None, nargs="+", help="key=value overrides")
    p.add_argument("--output-dir", default="./local_dino", type=str)
    p.add_argument("--benchmark-codebase", action="store_true")
    p.add_argument("seed", nargs="?", default=12, type=int, help="rng seed")
    p.add_argument("--seed", dest="seed", type=int, help=argparse.SUPPRESS)      # round-1 spelling, kept
    p.add_argument("--test-ibot", action="store_true")
    p.add_argument("--profiling", action="store_true")
    p.add_argument("--dump-fsdp-weights", action="store_true")
    p.add_argument("--record-ref-losses", action="store_true")
    p.add_argument("--ref-losses-path", default="", type=str)
    p.add_argument("--multi-distillation", action="store_true")
    # GPU-engine extras
    p.add_argument("--max-iters", default=0, type=int, help="stop after this many iterations (0 = full schedule)")
    p.add_argument("--print-freq", default=10, type=int)
    return p


def build_schedulers(config):
    """train/train.py:127-182: lr, weight decay, teacher momentum, teacher temperature, last-layer lr."""
    L = config.train.OFFICIAL_EPOCH_LENGTH
    total = config.optim["epochs"] * L
    lr = dict(base_value=config.optim["lr"], final_value=config.optim["min_lr"], total_iters=total,
              warmup_iters=config.optim["warmup_epochs"] * L, start_warmup_value=0,
              trunc_extra=config.optim["schedule_trunc_extra"])
    wd = dict(base_value=config.optim["weight_decay"], final_value=config.optim["weight_decay_end"], total_iters=total,
              trunc_extra=config.optim["schedule_trunc_extra"])
    mom = dict(base_value=config.teacher["momentum_teacher"], final_value=config.teacher["final_momentum_teacher"],
               total_iters=total, trunc_extra=config.optim["schedule_trunc_extra"])
    tw = config.teacher["warmup_teacher_temp_epochs"] * L
    temp = dict(base_value=config.teacher["teacher_temp"], final_value=config.teacher["teacher_temp"], total_iters=tw,
                warmup_iters=tw, start_warmup_value=config.teacher["warmup_teacher_temp"])
    lr_s, wd_s, mom_s, temp_s, last_s = (CosineScheduler(**lr), CosineScheduler(**wd), CosineScheduler(**mom),
                                         CosineScheduler(**temp), CosineScheduler(**lr))
    last_s.schedule[: config.optim["freeze_last_layer_epochs"] * L] = 0     # :169-173
    return lr_s, wd_s, mom_s, temp_s, last_s


def build_optimizer(config, param_groups, lr_schedule=None, wd_schedule=None, last_layer_lr_schedule=None):
    """train/train.py:75-122 builds optax.multi_transform(adamw per group) with the schedules injected as functions of
    the step count.  The GPU optimizer is the fused clip+AdamW(+EMA) kernel inside the engine; this returns the
    description it is driven by (the per-tensor multipliers come from `SSLMetaArch.get_params_groups`)."""
    return {"groups": param_groups, "lr": lr_schedule, "wd": wd_schedule, "last_layer_lr": last_layer_lr_schedule,
            "b1": config.optim.adamw_beta1, "b2": config.optim.adamw_beta2, "clip_grad": config.optim.clip_grad}


class EngineTree:
    """Handle onto engine-resident state with the reference's top-level keys (`student_backbone`, ... `teacher_ibot_head`,
    train/ssl_meta_arch.py:62-64,86-87,130-131).  `tree[key]` exports that module as {flax path: tensor} (a device
    copy in the reference's layouts); the step functions only pass the handle through, like a donated pytree."""

    KEYS = tuple(f"{r}_{m}" for r in ("student", "teacher") for m in ("backbone", "dino_head", "ibot_head"))

    def __init__(self, engine, what: str = "param", optimizer=None):
        self.engine, self.what, self.optimizer = engine, what, optimizer

    def keys(self):
        return [k for k in self.KEYS if self.what == "param" or k.startswith("student_")]

    def __contains__(self, k):
        return k in self.keys()

    def __iter__(self):
        return iter(self.keys())

    def __getitem__(self, key):
        flat = self.engine.params.export_reference_tree(self.what)
        out = {k[len(key) + 1:]: v for k, v in flat.items() if k.startswith(key + "/")}
        if not out:
            raise KeyError(key)
        return out

    def items(self):
        return [(k, self[k]) for k in self.keys()]


def train_step(params, batch, optimizer_state, teacher_temp, iteration, root_rngs=None, axis_name="dp", clip_grads=None):
    """One optimisation step with the reference's positional contract (train/train.py:491-565):
    `(params, batch, optimizer_state, teacher_temp, iteration, root_rngs)` -> `(params, optimizer_state, loss,
    metrics_dict)`.  `params` is an `EngineTree` (see `do_train` / `make_state`), `optimizer_state` the `EngineTree`
    over Adam m / v that carries the optimizer description of `build_optimizer`; lr / wd / last-layer lr are read from
    its schedules at `iteration` (the reference injects them as functions of the optimizer's step count, :95-106).
    The teacher is NOT touched here — the reference updates it with `update_ema()(ema_params, params, mom)` after
    the step (:666); `root_rngs` is accepted and unused (no dropout / drop-path on this path).  `loss` and the metrics
    are host floats (one device->host read per call, like the reference's per-step isnan check, :656)."""
    engine = params.engine
    opt = optimizer_state.optimizer
    if opt is None:
        raise ValueError("optimizer_state must come from make_state(engine, build_optimizer(...))")
    it = int(iteration)
    engine.set_batch(batch)
    engine.gram_schedule(it)                 # gram teacher refresh points (no-op unless gram.use_loss with a frozen teacher)
    engine.forward_backward(float(teacher_temp))
    if clip_grads is not None and float(clip_grads or 0.0) != float(engine.cfg.clip_grad or 0.0):
        raise ValueError("clip_grads differs from the engine configuration (optim.clip_grad)")
    engine.optimizer_step(float(opt["lr"][it]), float(opt["wd"][it]), float(opt["last_layer_lr"][it]), momentum=1.0)
    m = engine.read_metrics()
    loss = m.pop("total_loss")
    return params, optimizer_state, loss, m


def make_state(engine, optimizer):
    """(params, ema_params, optimizer_state) handles for the reference-style step functions."""
    params = EngineTree(engine, "param")
    return params, params, EngineTree(engine, "m", optimizer=optimizer)


def build_multi_resolution_data_loader_from_cfg(config, model, start_iter: int = 0, seed: int = 65537):
    """train/train.py:718-769: one loader per (global, local, gram-teacher) crop-size triple.  The engine's buffers, RoPE
    tables and kernels are laid out for ONE triple, so a single-entry configuration (ints, or lists of length one) is
    built exactly like the reference does (config copy with `train.seed + 1`) and anything longer raises: train each
    resolution stage with its own engine (what the reference's 7B recipe does stage by stage in its YAMLs)."""
    import copy
    as_list = lambda v: [v] if (v is None or isinstance(v, (int, float))) else list(v)
    gs, ls = as_list(config.crops.global_crops_size), as_list(config.crops.local_crops_size)
    gram = as_list(config.crops.get("gram_teacher_crops_size", None))
    ratios = as_list(config.crops.get("global_local_crop_pairs_ratios", 1.0))
    assert len(gs) == len(ls) == len(gram) == len(ratios)
    if len(gs) != 1:
        raise NotImplementedError("multi-resolution crop lists: the GPU engine is built for one (global, local, gram) size "
                                  "triple; run one engine per resolution stage")
    config_i = copy.deepcopy(config)
    config_i.crops.global_crops_size, config_i.crops.local_crops_size = gs[0], ls[0]
    config_i.crops.gram_teacher_crops_size = gram[0]
    config_i.train.seed = config.train.seed + 1
    return build_data_loader_from_cfg(config=config_i, model=model, start_iter=start_iter)


def build_data_loader_from_cfg(config, model, start_iter: int = 0):
    """train/train.py:772-846.  `train.dataset_path`:
      synthetic            one fixed random batch per rank (benchmarks / smoke runs) — announced loudly;
      synthetic:noise      the reference decoder's own image distribution (noise images) through the DINO augmentation
                           and `collate_data_and_cast` (the full host pipeline, no files needed);
      synthetic:gpu        the same image distribution generated in HBM (uint8 [B,224,224,3]) through the ON-GPU
                           augmentation + mask pipeline (data/gpu_augment.py, SURVEY §8f.3): no host pixel work at all;
      gpu:ImageNet:split=TRAIN:root=R, gpu:ImageFolder:root=R
                           image files decoded by PIL in DataLoader workers, cropped and augmented on the GPU at each
                           image's own size (data/image_loader.py); resumable: the indices and crops of an iteration
                           depend on (train.seed, rank, world, iteration) only;
      anything else        the reference's `make_dataset` / `make_data_loader` (data/loaders.py), which stay in the
                           reference checkout and resolve through the package overlay (needs that checkout + its deps).
    """
    from .. import distributed
    from ..data import MaskingGenerator, collate_data_and_cast
    path = str(config.train.dataset_path)
    B = config.train.batch_size_per_gpu
    rank, world = distributed.get_rank(), distributed.get_world_size()
    if path == "synthetic":
        from ..engine.synth import synthetic_batch
        if distributed.is_main_process():
            print("WARNING: train.dataset_path=synthetic — training on ONE fixed random batch per rank "
                  "(benchmark / smoke mode, not a real data pipeline)", file=sys.stderr, flush=True)
        fixed = synthetic_batch(model.engine_config, B, seed=rank, pin=torch.cuda.is_available())

        def forever():
            while True:
                yield fixed
        return forever()
    if path.startswith("synthetic:gpu"):
        from ..data.gpu_augment import GpuBatchPipeline
        pipe = GpuBatchPipeline(config, seed=config.train.seed + 1000 * rank + start_iter)
        dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
        gen = torch.Generator(device=dev).manual_seed(config.train.seed + 7919 * rank + start_iter)

        def gpu_batches():
            while True:
                noise = torch.randn((B, 224, 224, 3), device=dev, generator=gen)        # decoders.py:31-34 on the device
                lo, hi = noise.amin((1, 2, 3), keepdim=True), noise.amax((1, 2, 3), keepdim=True)
                yield pipe(((noise - lo) / (hi - lo) * 255).to(torch.uint8))
        return gpu_batches()
    if path.startswith("gpu:"):
        from ..data.image_loader import GpuImageLoader
        return GpuImageLoader(config, start_iter=start_iter, rank=rank, world=world)
    img_size, patch = config.crops.global_crops_size, config.student.patch_size
    grid = img_size // patch
    mask_generator = MaskingGenerator(input_size=(grid, grid), max_num_patches=0.5 * img_size // patch * img_size // patch)
    dtype = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}[config.compute_precision.param_dtype]
    collate_fn = partial(collate_data_and_cast, mask_ratio_tuple=config.ibot.mask_ratio_min_max,
                         mask_probability=config.ibot.mask_sample_probability, dtype=dtype, n_tokens=grid * grid,
                         mask_generator=mask_generator, random_circular_shift=config.ibot.mask_random_circular_shift,
                         local_batch_size=None)
    transform = model.build_data_augmentation_dino(config)
    seed = config.train.seed + start_iter + 1                        # :840
    if path.startswith("synthetic:noise"):
        from ..data.synthetic import NoiseImageDataset, SeededBatchSampler
        ds = NoiseImageDataset(transform=transform, target_transform=lambda _: (), seed=config.train.seed)
        sampler = SeededBatchSampler(len(ds), B, seed=seed, rank=rank, world=world, advance=start_iter * B)
        return torch.utils.data.DataLoader(ds, batch_sampler=sampler, num_workers=int(config.train.get("num_workers", 0)),
                                           collate_fn=collate_fn, pin_memory=torch.cuda.is_available())
    from ..data import SamplerType, make_data_loader, make_dataset      # reference loaders through the overlay
    dataset = make_dataset(dataset_str=path, transform=transform, target_transform=lambda _: ())
    return make_data_loader(dataset=dataset, batch_size=B, num_workers=int(config.train.get("num_workers", 0)), shuffle=True,
                            seed=seed, sampler_type=SamplerType.EPOCH, sampler_advance=start_iter * B, drop_last=True,
                            collate_fn=collate_fn)


def _knn_cfg(config) -> dict:
    """The `evaluation.knn` block, or {} when it names no train / val dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    knn = dict(ev.get("knn", None) or {})
    return knn if knn.get("train_dataset_path") and knn.get("val_dataset_path") else {}


def _linear_cfg(config) -> dict:
    """The `evaluation.linear` block, or {} when it names no train / val dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    linear = dict(ev.get("linear", None) or {})
    return linear if linear.get("train_dataset_path") and linear.get("val_dataset_path") else {}


def _seg_cfg(config) -> dict:
    """The `evaluation.segmentation` block, or {} when it names no train / val dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    seg = dict(ev.get("segmentation", None) or {})
    return seg if seg.get("train_dataset_path") and seg.get("val_dataset_path") else {}


def _depth_cfg(config) -> dict:
    """The `evaluation.depth` block, or {} when it names no train / val dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    depth = dict(ev.get("depth", None) or {})
    return depth if depth.get("train_dataset_path") and depth.get("val_dataset_path") else {}


def _video_cfg(config) -> dict:
    """The `evaluation.video` block, or {} when it names no dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    video = dict(ev.get("video", None) or {})
    return video if video.get("dataset_path") else {}


def _correspondence_cfg(config) -> dict:
    """The `evaluation.correspondence` block, or {} when it names no dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    corr = dict(ev.get("correspondence", None) or {})
    return corr if corr.get("dataset_path") else {}


def _discovery_cfg(config) -> dict:
    """The `evaluation.discovery` block, or {} when it names no dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    disc = dict(ev.get("discovery", None) or {})
    return disc if disc.get("dataset_path") else {}


def _retrieval_cfg(config) -> dict:
    """The `evaluation.retrieval` block, or {} when it names no dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    ret = dict(ev.get("retrieval", None) or {})
    return ret if ret.get("dataset_path") else {}


def _logreg_cfg(config) -> dict:
    """The `evaluation.logreg` block, or {} when it names no train / val dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    logreg = dict(ev.get("logreg", None) or {})
    return logreg if logreg.get("train_dataset_path") and logreg.get("val_dataset_path") else {}


def _attentive_cfg(config) -> dict:
    """The `evaluation.attentive` block, or {} when it names no train / val dataset (then nothing is evaluated)."""
    ev = config.get("evaluation", None) or {}
    att = dict(ev.get("attentive", None) or {})
    return att if att.get("train_dataset_path") and att.get("val_dataset_path") else {}


def eval_backbone(config, weights):
    """The frozen backbone k-NN evaluates, with the architecture of the run's `student.*` config (the depth is the
    number of blocks in the weights).  `weights`: a DinoVisionTransformer (returned as is); a `save_checkpoint`
    directory (its `teacher_backbone`); a torch-hub `.pth` state dict; or a live Engine / SSLMetaArch (its EMA teacher,
    through `engine_state`, which is collective under FSDP: every rank calls this)."""
    from ..checkpointer import convert_torch_hub_state_dict, engine_state, flat_from_tree, load_checkpoint
    from ..engine.config import config_from_reference_cfg
    from ..models import DinoVisionTransformer
    if isinstance(weights, DinoVisionTransformer):
        return weights
    engine = getattr(weights, "engine", None) if isinstance(weights, SSLMetaArch) else weights
    if hasattr(engine, "params") and hasattr(engine, "train_step"):
        tree = engine_state(engine)[0]["teacher_backbone"]
        device = engine.device
    else:
        path = str(weights)
        if os.path.isdir(path):
            tree = load_checkpoint(path)["model_params"]["teacher_backbone"]
        elif path.endswith(".pth"):
            tree = convert_torch_hub_state_dict(torch.load(path, map_location="cpu", weights_only=True))[0]
        else:
            raise FileNotFoundError(f"{path}: not a checkpoint directory or a .pth state dict")
        device = f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}"
    ec, st = config_from_reference_cfg(config), config.student
    depth = sum(1 for k in tree if str(k).startswith("blocks_"))
    ffn = st.ffn_layer
    return DinoVisionTransformer(tree, patch_size=ec.patch, pos_embed_rope_base=ec.rope_base, embed_dim=ec.embed_dim,
                                 n_blocks=depth, num_heads=ec.heads, ffn_ratio=ec.ffn_ratio, norm_layer=st.norm_layer,
                                 ffn_layer=ffn, n_storage_tokens=ec.n_storage, mask_k_bias=ec.mask_k_bias,
                                 device=device)


def do_test(config, model, header):
    """k-NN evaluation of the teacher backbone of `model` (see `eval_backbone`) on the `evaluation.knn` datasets; rank 0
    writes <output_dir>/eval/<header>/results_knn.json and returns {k: {"top1", "top5"}} ({} on other ranks).  Without
    configured datasets it logs one line and returns {}."""
    import json
    from .. import distributed
    knn = _knn_cfg(config)
    if not knn:
        if distributed.is_main_process():
            print(f"do_test({header}): no evaluation.knn train / val dataset configured, nothing evaluated", flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_knn, make_eval_dataset
    c = config.crops
    results = eval_knn(backbone, make_eval_dataset(knn["train_dataset_path"]), make_eval_dataset(knn["val_dataset_path"]),
                       nb_knn=knn.get("nb_knn", (10, 20, 100, 200)), temperature=float(knn.get("temperature", 0.07)),
                       batch_size=int(knn.get("batch_size", 256)), resize_size=int(knn.get("resize_size", 256)),
                       crop_size=int(knn.get("crop_size", 224)), num_workers=int(knn.get("num_workers", 8)),
                       rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)), rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)))
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_knn.json"), "w") as f:
        json.dump({str(k): v for k, v in results.items()}, f, indent=1)
    print(f"do_test({header}): " + ", ".join(f"{k}-NN top-1 {v['top1']:.2f} top-5 {v['top5']:.2f}"
                                             for k, v in results.items()), flush=True)
    return results


def do_linear_eval(config, model, header):
    """Linear-probe evaluation of the teacher backbone of `model` (see `eval_backbone`) on the `evaluation.linear`
    datasets; rank 0 writes <output_dir>/eval/<header>/results_linear.json and returns {classifier name: {"top1",
    "top5"}, "best_classifier": {"name", "top1", "top5"}} ({} on other ranks).  Without configured datasets it logs one
    line and returns {}."""
    import json
    from .. import distributed
    linear = _linear_cfg(config)
    if not linear:
        if distributed.is_main_process():
            print(f"do_linear_eval({header}): no evaluation.linear train / val dataset configured, nothing evaluated",
                  flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_linear, make_eval_dataset
    c = config.crops
    kw = {k: linear[k] for k in ("epochs", "epoch_length", "batch_size", "learning_rates", "n_last_blocks_list",
                                 "avgpools", "crop_size", "resize_size", "num_workers", "seed") if k in linear}
    results = eval_linear(backbone, make_eval_dataset(linear["train_dataset_path"]),
                          make_eval_dataset(linear["val_dataset_path"]), rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                          rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_linear.json"), "w") as f:
        json.dump(results, f, indent=1)
    best = results["best_classifier"]
    print(f"do_linear_eval({header}): best {best['name']} top-1 {best['top1']:.2f} top-5 {best['top5']:.2f}", flush=True)
    return results


def do_seg_eval(config, model, header):
    """Linear segmentation probe of the teacher backbone of `model` (see `eval_backbone`) on the
    `evaluation.segmentation` datasets; rank 0 writes <output_dir>/eval/<header>/results_segmentation.json and returns
    {"mIoU", "mAcc", "aAcc", "per_class_iou"} in percent ({} on other ranks).  Without configured datasets it logs one
    line and returns {}."""
    import json
    from .. import distributed
    seg = _seg_cfg(config)
    if not seg:
        if distributed.is_main_process():
            print(f"do_seg_eval({header}): no evaluation.segmentation train / val dataset configured, nothing evaluated",
                  flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_segmentation, make_seg_dataset
    c = config.crops
    kw = {k: seg[k] for k in ("num_classes", "n_last_blocks", "batch_size", "crop_size", "iterations", "lr",
                              "weight_decay", "warmup_iterations", "num_workers", "seed") if k in seg}
    results = eval_segmentation(backbone, make_seg_dataset(seg["train_dataset_path"], "train"),
                                make_seg_dataset(seg["val_dataset_path"], "val"),
                                rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                                rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_segmentation.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(f"do_seg_eval({header}): mIoU {results['mIoU']:.2f} mAcc {results['mAcc']:.2f} aAcc {results['aAcc']:.2f}",
          flush=True)
    return results


def do_depth_eval(config, model, header):
    """Linear depth probe of the teacher backbone of `model` (see `eval_backbone`) on the `evaluation.depth` datasets;
    rank 0 writes <output_dir>/eval/<header>/results_depth.json and returns {"abs_rel", "sq_rel", "rmse", "rmse_log",
    "log10", "a1", "a2", "a3", "config"} ({} on other ranks), "config" echoing the evaluation.depth block.  Without
    configured datasets it logs one line and returns {}."""
    import json
    from .. import distributed
    depth = _depth_cfg(config)
    if not depth:
        if distributed.is_main_process():
            print(f"do_depth_eval({header}): no evaluation.depth train / val dataset configured, nothing evaluated",
                  flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_depth, make_depth_dataset
    c = config.crops
    kw = {k: depth[k] for k in ("n_last_blocks", "use_cls_token", "n_bins", "min_depth", "max_depth", "batch_size",
                                "crop_size", "iterations", "lr", "weight_decay", "warmup_iterations", "eval_crop",
                                "num_workers", "seed") if k in depth}
    scale = depth.get("depth_scale", 1000)
    results = eval_depth(backbone, make_depth_dataset(depth["train_dataset_path"], "train", scale),
                         make_depth_dataset(depth["val_dataset_path"], "val", scale),
                         rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                         rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    results["config"] = {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in depth.items()}
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_depth.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(f"do_depth_eval({header}): abs_rel {results['abs_rel']:.4f} rmse {results['rmse']:.4f} "
          f"a1 {results['a1']:.4f}", flush=True)
    return results


def do_video_eval(config, model, header):
    """Video object segmentation by label propagation through the teacher backbone of `model` (see `eval_backbone`) on
    the `evaluation.video` dataset; rank 0 writes <output_dir>/eval/<header>/results_video.json and returns {"J&F-Mean",
    "J-Mean", "J-Recall", "J-Decay", "F-Mean", "F-Recall", "F-Decay", "sequences", "protocol", "config"} ({} on other
    ranks), "config" echoing the evaluation.video block; with save_masks the predicted masks go to
    <output_dir>/eval/<header>/Annotations/480p/<sequence>/.  Without a configured dataset it logs one line and
    returns {}."""
    import json
    from .. import distributed
    video = _video_cfg(config)
    if not video:
        if distributed.is_main_process():
            print(f"do_video_eval({header}): no evaluation.video dataset configured, nothing evaluated", flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_video_segmentation, make_video_dataset
    c = config.crops
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    kw = {k: video[k] for k in ("n_last_frames", "size_mask_neighborhood", "topk", "temperature", "short_side",
                                "batch_size", "num_workers", "save_masks") if k in video}
    results = eval_video_segmentation(backbone, make_video_dataset(video["dataset_path"]), output_dir=out_dir,
                                      rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                                      rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    results["config"] = {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in video.items()}
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_video.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(f"do_video_eval({header}): J&F-Mean {results['J&F-Mean']:.4f} J-Mean {results['J-Mean']:.4f} "
          f"F-Mean {results['F-Mean']:.4f}", flush=True)
    return results


def do_correspondence_eval(config, model, header):
    """Keypoint correspondence (nearest neighbour over the upsampled patch features, PCK) through the teacher backbone of
    `model` (see `eval_backbone`) on the `evaluation.correspondence` dataset; rank 0 writes
    <output_dir>/eval/<header>/results_correspondence.json and returns {"PCK@a", "PCK-image@a" per alpha, "categories",
    "n_pairs", "n_keypoints", "protocol", "config"} ({} on other ranks), "config" echoing the evaluation.correspondence
    block.  Without a configured dataset it logs one line and returns {}."""
    import json
    from .. import distributed
    corr = _correspondence_cfg(config)
    if not corr:
        if distributed.is_main_process():
            print(f"do_correspondence_eval({header}): no evaluation.correspondence dataset configured, nothing "
                  "evaluated", flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_correspondence, make_correspondence_dataset
    c = config.crops
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    kw = {k: corr[k] for k in ("image_size", "alphas", "batch_size", "num_workers") if k in corr}
    results = eval_correspondence(backbone, make_correspondence_dataset(corr["dataset_path"], corr.get("split", "test")),
                                  rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                                  rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    results["config"] = {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in corr.items()}
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_correspondence.json"), "w") as f:
        json.dump(results, f, indent=1)
    a = results["protocol"]["alphas"][-1]
    print(f"do_correspondence_eval({header}): PCK@{a:g} {results[f'PCK@{a:g}']:.4f} PCK-image@{a:g} "
          f"{results[f'PCK-image@{a:g}']:.4f} over {results['n_pairs']} pairs", flush=True)
    return results


def do_discovery_eval(config, model, header):
    """Unsupervised object discovery (TokenCut's normalized cut on the patch features, CorLoc) through the teacher
    backbone of `model` (see `eval_backbone`) on the `evaluation.discovery` dataset; rank 0 writes
    <output_dir>/eval/<header>/results_discovery.json and returns {"CorLoc", "n_images", "n_unconverged", "protocol",
    "config"} (and "boxes" with save_boxes; {} on other ranks), "config" echoing the evaluation.discovery block.
    Without a configured dataset it logs one line and returns {}."""
    import json
    from .. import distributed
    disc = _discovery_cfg(config)
    if not disc:
        if distributed.is_main_process():
            print(f"do_discovery_eval({header}): no evaluation.discovery dataset configured, nothing evaluated",
                  flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_object_discovery, make_discovery_dataset
    c = config.crops
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    kw = {k: disc[k] for k in ("tau", "eps", "batch_size", "num_workers", "save_boxes") if k in disc}
    dataset = make_discovery_dataset(disc["dataset_path"], disc.get("split", "trainval"),
                                     bool(disc.get("remove_difficult", False)))
    results = eval_object_discovery(backbone, dataset, rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                                    rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    results["config"] = {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in disc.items()}
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_discovery.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(f"do_discovery_eval({header}): CorLoc {results['CorLoc']:.4f} over {results['n_images']} images, "
          f"{results['n_unconverged']} unconverged", flush=True)
    return results


def do_retrieval_eval(config, model, header):
    """Instance retrieval (revisited Oxford / Paris mAP of the multi-scale class token) through the teacher backbone of
    `model` (see `eval_backbone`) on the `evaluation.retrieval` dataset; rank 0 writes
    <output_dir>/eval/<header>/results_retrieval.json and returns {"mAP", "mP@k", "n_empty", "n_queries",
    "n_database", "protocol", "config"} (and "ranks" with save_ranks; {} on other ranks), "config" echoing the
    evaluation.retrieval block.  Without a configured dataset it logs one line and returns {}."""
    import json
    from .. import distributed
    ret = _retrieval_cfg(config)
    if not ret:
        if distributed.is_main_process():
            print(f"do_retrieval_eval({header}): no evaluation.retrieval dataset configured, nothing evaluated",
                  flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_instance_retrieval, make_retrieval_dataset
    c = config.crops
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    kw = {k: ret[k] for k in ("image_size", "scales", "batch_size", "num_workers", "save_ranks") if k in ret}
    dataset = make_retrieval_dataset(ret["dataset_path"], ret.get("dataset", "roxford5k"))
    results = eval_instance_retrieval(backbone, dataset, rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                                      rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    results["config"] = {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in ret.items()}
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_retrieval.json"), "w") as f:
        json.dump(results, f, indent=1)
    m = results["mAP"]
    print(f"do_retrieval_eval({header}): mAP easy {m['easy']:.2f} medium {m['medium']:.2f} hard {m['hard']:.2f} over "
          f"{results['n_queries']} queries and {results['n_database']} database images", flush=True)
    return results


def do_logreg_eval(config, model, header):
    """Logistic-regression evaluation (L-BFGS over a grid of regularisation strengths) of the teacher backbone of
    `model` (see `eval_backbone`) on the `evaluation.logreg` datasets; rank 0 writes
    <output_dir>/eval/<header>/results_logreg.json and returns {"sweep" (per C: held-out top-1, iterations,
    evaluations, stop reason), "best_C", "refit", "top1", "top5", "mean_per_class", ..., "protocol", "config"} ({} on
    other ranks).  Without configured datasets it logs one line and returns {}."""
    import json
    from .. import distributed
    logreg = _logreg_cfg(config)
    if not logreg:
        if distributed.is_main_process():
            print(f"do_logreg_eval({header}): no evaluation.logreg train / val dataset configured, nothing evaluated",
                  flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_log_regression, make_eval_dataset
    c = config.crops
    kw = {k: logreg[k] for k in ("C_values", "holdout_fraction", "max_iter", "tol", "history", "avgpool", "batch_size",
                                 "resize_size", "crop_size", "num_workers", "seed") if k in logreg}
    results = eval_log_regression(backbone, make_eval_dataset(logreg["train_dataset_path"]),
                                  make_eval_dataset(logreg["val_dataset_path"]),
                                  rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                                  rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    results["protocol"] = ("multinomial logistic regression, c * sum CE + ||W||^2 / 2 (bias unpenalised), L-BFGS "
                           "from zero; C chosen by held-out top-1 on a stratified split of train, refit on all of "
                           "train, scored on val")
    results["config"] = {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in logreg.items()}
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_logreg.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(f"do_logreg_eval({header}): C {results['best_C']:.3g} top-1 {results['top1']:.2f} top-5 "
          f"{results['top5']:.2f} mean per-class {results['mean_per_class']:.2f}", flush=True)
    return results


def do_attentive_eval(config, model, header):
    """Attentive-probe video classification of the teacher backbone of `model` (see `eval_backbone`) on the
    `evaluation.attentive` datasets; rank 0 writes <output_dir>/eval/<header>/results_attentive.json and returns
    {"probes" (per learning rate: val top-1, top-5, mean per-class accuracy), "best_probe", "top1", "top5",
    "mean_per_class", the train / val video and clip counts, "protocol", "config"} ({} on other ranks).  Without
    configured datasets it logs one line and returns {}."""
    import json
    from .. import distributed
    att = _attentive_cfg(config)
    if not att:
        if distributed.is_main_process():
            print(f"do_attentive_eval({header}): no evaluation.attentive train / val dataset configured, nothing "
                  "evaluated", flush=True)
        return {}
    backbone = eval_backbone(config, model)            # collective for a live engine under FSDP
    if not distributed.is_main_process():
        return {}
    from ..eval import eval_attentive, make_video_class_dataset
    c = config.crops
    kw = {k: att[k] for k in ("learning_rates", "epochs", "warmup_epochs", "weight_decay", "batch_size", "num_frames",
                              "frame_step", "num_segments", "num_views", "crop_size", "num_workers", "seed") if k in att}
    results = eval_attentive(backbone, make_video_class_dataset(att["train_dataset_path"]),
                             make_video_class_dataset(att["val_dataset_path"]),
                             rgb_mean=c.get("rgb_mean", (0.485, 0.456, 0.406)),
                             rgb_std=c.get("rgb_std", (0.229, 0.224, 0.225)), **kw)
    results["protocol"] = ("attentive probe (one query, the backbone's heads, temporal embedding, MLP block, linear "
                           "classifier) on the last block's patch tokens of every frame; AdamW, cross-entropy, warm-up "
                           "then cosine; val: mean softmax over segments x views, best learning rate by val top-1")
    results["config"] = {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in att.items()}
    out_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "eval", header)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "results_attentive.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(f"do_attentive_eval({header}): {results['best_probe']['name']} top-1 {results['top1']:.2f} top-5 "
          f"{results['top5']:.2f} mean per-class {results['mean_per_class']:.2f}", flush=True)
    return results


def do_train(config, model: SSLMetaArch, resume: bool = False, data_loader=None, max_iters: int = 0,
             print_freq: int = 10):
    """train/train.py:319-713.  `data_loader` (optional) yields the reference's collate dicts; by default it is built
    from `train.dataset_path` (`build_data_loader_from_cfg`), positioned at the resume iteration."""
    from .. import distributed
    from ..engine.synth import init_reference_like
    comm = None
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if distributed.is_enabled() and distributed.get_world_size() > 1:
        from ..fsdp.runtime import Comm
        comm = Comm()
    engine = model.build_engine(device=f"cuda:{local_rank}", comm=comm)
    init_reference_like(engine, seed=config.train.seed)
    schedules = build_schedulers(config)
    lr_s, wd_s, mom_s, temp_s, last_s = schedules
    local_s, gram_s = (getattr(model, a, None) for a in ("dino_local_loss_schedule", "gram_loss_schedule"))
    total = len(lr_s.schedule)
    n_iters = min(total, max_iters) if max_iters else total
    # ---- resume / periodic checkpoints (train/train.py:447-469,695-706; <output_dir>/ckpt/<iteration>)
    from ..checkpointer import (engine_state, find_latest_checkpoint, keep_checkpoint_copy, keep_last_n_checkpoints,
                                load_checkpoint, load_engine_state, save_checkpoint)
    ckpt_dir = os.path.join(getattr(config.train, "output_dir", None) or ".", "ckpt")
    ck_cfg = config.get("checkpointing", None) if hasattr(config, "get") else getattr(config, "checkpointing", None)
    start_iter = 0
    last = find_latest_checkpoint(ckpt_dir) if resume else None
    if last is not None:
        abstract_p, abstract_o = engine_state(engine)            # shapes / names to validate the files against
        ck = load_checkpoint(last, abstract_model_params=abstract_p, abstract_optimizer_state=abstract_o,
                             strict_loading=False)
        load_engine_state(engine, ck["model_params"], ck.get("optimizer_state"))
        start_iter = int(ck["iteration"]) + 1
        if distributed.is_main_process():
            print(f"checkpoint found {last}: resuming at iteration {start_iter}", flush=True)
    user_loader = data_loader is not None
    if data_loader is None:
        data_loader = build_data_loader_from_cfg(config, model, start_iter)
    it_loader = iter(data_loader)
    if user_loader and start_iter:
        # a caller-supplied loader starts at its beginning: skip what the checkpointed run already consumed
        for _ in range(start_iter):
            next(it_loader)
    meters, nan_streak, t0 = {}, 0, time.time()
    ev = config.get("evaluation", None) or {}
    knn_on, linear_on, seg_on = bool(_knn_cfg(config)), bool(_linear_cfg(config)), bool(_seg_cfg(config))
    depth_on, video_on = bool(_depth_cfg(config)), bool(_video_cfg(config))
    corr_on, disc_on = bool(_correspondence_cfg(config)), bool(_discovery_cfg(config))
    ret_on, logreg_on, att_on = bool(_retrieval_cfg(config)), bool(_logreg_cfg(config)), bool(_attentive_cfg(config))
    any_on = (knn_on or linear_on or seg_on or depth_on or video_on or corr_on or disc_on or ret_on or logreg_on
              or att_on)
    eval_period = int(ev.get("eval_period_iterations", 0) or 0) if any_on else 0
    try:
        for it in range(start_iter, n_iters):
            try:
                data = next(it_loader)
            except StopIteration:
                break
            local_w, gram_w = (None if s is None else float(s[it]) for s in (local_s, gram_s))
            engine.train_step(data, teacher_temp=float(temp_s[it]), lr=float(lr_s[it]), wd=float(wd_s[it]),
                              last_layer_lr=float(last_s[it]), momentum=float(mom_s[it]), gram_loss_weight=gram_w,
                              dino_local_loss_weight=local_w, iteration=it)
            if ck_cfg is not None and (it + 1) % int(ck_cfg.period) == 0:
                params_tree, opt_tree = engine_state(engine)             # collective under FSDP (all-gathers the shards)
                if distributed.is_main_process():
                    save_checkpoint(os.path.join(ckpt_dir, str(it)), iteration=it, params=params_tree,
                                    optimizer_state=opt_tree, overwrite=True)
                    keep_last_n_checkpoints(ckpt_dir, ck_cfg.max_to_keep)
                    if "keep_every" in ck_cfg and (it + 1) % int(ck_cfg.keep_every) == 0:
                        keep_checkpoint_copy(os.path.join(ckpt_dir, str(it)))
            if eval_period > 0 and (it + 1) % eval_period == 0:      # train/train.py:689-692
                if knn_on:
                    do_test(config, engine, f"training_{it}")
                if linear_on:
                    do_linear_eval(config, engine, f"training_{it}")
                if seg_on:
                    do_seg_eval(config, engine, f"training_{it}")
                if depth_on:
                    do_depth_eval(config, engine, f"training_{it}")
                if video_on:
                    do_video_eval(config, engine, f"training_{it}")
                if corr_on:
                    do_correspondence_eval(config, engine, f"training_{it}")
                if disc_on:
                    do_discovery_eval(config, engine, f"training_{it}")
                if ret_on:
                    do_retrieval_eval(config, engine, f"training_{it}")
                if logreg_on:
                    do_logreg_eval(config, engine, f"training_{it}")
                if att_on:
                    do_attentive_eval(config, engine, f"training_{it}")
            if it % print_freq == 0 or it == n_iters - 1:
                m = engine.read_metrics()                  # the only device->host sync of the loop
                if math.isnan(m["total_loss"]):            # NaN guard of train/train.py:656-667, evaluated on read
                    nan_streak += 1
                    if nan_streak > 2:
                        raise RuntimeError("loss is NaN for more than 2 consecutive reads")
                else:
                    nan_streak = 0
                meters = m
                if distributed.is_main_process():
                    dt = (time.time() - t0) / (it - start_iter + 1)
                    print(f"it {it}: loss {m['total_loss']:.4f} dino_l {m['dino_local_crops_loss']:.4f} dino_g "
                          f"{m['dino_global_crops_loss']:.4f} koleo {m['koleo_loss']:.4f} ibot {m['ibot_loss']:.4f} "
                          f"({dt * 1e3:.1f} ms/it)", flush=True)
    finally:
        if not user_loader:                  # the loader's workers end with the run, whether it returns or raises
            for obj in (it_loader, data_loader):
                close = getattr(obj, "close", None)
                if callable(close):
                    close()
    return meters


def main(argv=None):
    args = get_args_parser().parse_args(argv)
    if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    config = setup_config(DinoV3SetupArgs(config_file=args.config_file or None, output_dir=args.output_dir, opts=args.opts or []))
    import random
    import numpy as np
    random.seed(args.seed); np.random.seed(args.seed); torch.manual_seed(args.seed)   # setup_job(seed=args.seed), :281
    if args.eval not in ("", "knn", "linear", "logreg", "attentive", "seg", "depth", "video", "correspondence",
                         "discovery", "retrieval"):
        raise NotImplementedError(f"--eval {args.eval!r}: the evaluations are k-NN (--eval knn, or empty), the linear "
                                  "probe (--eval linear), logistic regression (--eval logreg), attentive-probe video "
                                  "classification (--eval attentive), the linear "
                                  "segmentation probe (--eval seg), the linear "
                                  "depth probe (--eval depth), video object segmentation (--eval video) and keypoint "
                                  "correspondence (--eval correspondence), and unsupervised object discovery "
                                  "(--eval discovery), and instance retrieval (--eval retrieval)")
    if args.eval_only:                                 # train/train.py:304-311
        import json
        from ..checkpointer import find_latest_checkpoint
        weights = args.eval_pretrained_weights
        if not weights:
            weights = find_latest_checkpoint(os.path.join(config.train.output_dir, "ckpt"))
        if not weights:
            raise FileNotFoundError("--eval-only needs --eval-pretrained-weights (a checkpoint directory or a torch-hub "
                                    f".pth) or a checkpoint under {os.path.join(config.train.output_dir, 'ckpt')}")
        it = 0
        if os.path.isdir(str(weights)):
            stored = json.loads(open(os.path.join(str(weights), "manifest.json")).read())["iteration"]
            it = int(stored) + 1 if str(stored).lstrip("-").isdigit() else 0
        if args.eval == "linear":
            return do_linear_eval(config, str(weights), f"manual_{it}")
        if args.eval == "logreg":
            return do_logreg_eval(config, str(weights), f"manual_{it}")
        if args.eval == "attentive":
            return do_attentive_eval(config, str(weights), f"manual_{it}")
        if args.eval == "seg":
            return do_seg_eval(config, str(weights), f"manual_{it}")
        if args.eval == "depth":
            return do_depth_eval(config, str(weights), f"manual_{it}")
        if args.eval == "video":
            return do_video_eval(config, str(weights), f"manual_{it}")
        if args.eval == "correspondence":
            return do_correspondence_eval(config, str(weights), f"manual_{it}")
        if args.eval == "discovery":
            return do_discovery_eval(config, str(weights), f"manual_{it}")
        if args.eval == "retrieval":
            return do_retrieval_eval(config, str(weights), f"manual_{it}")
        return do_test(config, str(weights), f"manual_{it}")
    model = SSLMetaArch(config)
    return do_train(config, model, resume=not args.no_resume, max_iters=args.max_iters, print_freq=args.print_freq)


if __name__ == "__main__":
    main()
