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
    for it in range(start_iter, n_iters):
        try:
            data = next(it_loader)
        except StopIteration:
            break
        engine.train_step(data, teacher_temp=float(temp_s[it]), lr=float(lr_s[it]), wd=float(wd_s[it]),
                          last_layer_lr=float(last_s[it]), momentum=float(mom_s[it]), iteration=it)
        if ck_cfg is not None and (it + 1) % int(ck_cfg.period) == 0:
            params_tree, opt_tree = engine_state(engine)                 # collective under FSDP (all-gathers the shards)
            if distributed.is_main_process():
                save_checkpoint(os.path.join(ckpt_dir, str(it)), iteration=it, params=params_tree,
                                optimizer_state=opt_tree, overwrite=True)
                keep_last_n_checkpoints(ckpt_dir, ck_cfg.max_to_keep)
                if "keep_every" in ck_cfg and (it + 1) % int(ck_cfg.keep_every) == 0:
                    keep_checkpoint_copy(os.path.join(ckpt_dir, str(it)))
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
    model = SSLMetaArch(config)
    return do_train(config, model, resume=not args.no_resume, max_iters=args.max_iters, print_freq=args.print_freq)


if __name__ == "__main__":
    main()
