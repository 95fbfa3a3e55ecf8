"""`SSLMetaArch` with the reference's constructor and helper names (dinov3_jax/train/ssl_meta_arch.py:32-660).

The reference class is a Flax module whose `__call__` is traced by jax.jit; here it is a plain object that owns the
configuration and builds the GPU step executor.  The top-level parameter keys (`student_backbone`, `student_dino_head`,
`student_ibot_head`, `teacher_*`; :62-64,86-87,130-131) and the batch-dict contract are unchanged.
"""
from __future__ import annotations

from ..engine import Engine, config_from_reference_cfg, distill_config_from_reference_cfg
from ..engine.params import lr_wd_multipliers
from .cosine_lr_scheduler import linear_warmup_cosine_decay

FP8_FILTERS = ("blocks",)


def fp8_from_config(config) -> bool:
    """student.fp8_enabled / student.fp8_filter (ssl_default_config.yaml:121-122): whether the engine runs the block
    linears in FP8.  "blocks" (qkv, proj and the MLP linears of every block) is the only filter there is."""
    st = config.student
    if not bool(st.get("fp8_enabled", False)):
        return False
    flt = st.get("fp8_filter", "blocks")
    if flt not in FP8_FILTERS:
        raise NotImplementedError(f"student.fp8_filter={flt!r}: FP8 runs only the block linears (fp8_filter: blocks = "
                                  "attn.qkv, attn.proj and mlp fc1 / fc2 or w1 / w2 / w3 of every block)")
    return True


def loss_weight_schedule(config, sc) -> linear_warmup_cosine_decay:
    """A {start, peak, end, warmup_epochs[, cosine_epochs]} block over OFFICIAL_EPOCH_LENGTH * optim.epochs
    iterations (train/ssl_meta_arch.py:150-163,183-199)."""
    if not sc:
        raise ValueError("a loss-weight schedule needs {start, peak, end, warmup_epochs[, cosine_epochs]}")
    per_epoch = int(config.train.OFFICIAL_EPOCH_LENGTH)
    cosine = sc.get("cosine_epochs", None)
    return linear_warmup_cosine_decay(start=sc.start, peak=sc.peak, end=sc.end,
                                      warmup_iterations=per_epoch * int(sc.warmup_epochs),
                                      total_iterations=per_epoch * int(config.optim.epochs),
                                      cosine_iterations=None if cosine is None else per_epoch * int(cosine))


class SSLMetaArch:
    PARAM_MODULES = ("backbone", "dino_head", "ibot_head")

    def __init__(self, config):
        self.config = config
        self.engine_config = config_from_reference_cfg(config)       # raises on options the reference asserts on (:47-51)
        # distillation.enabled (:257-286): the frozen teacher's configuration, None without distillation
        self.distill_config = distill_config_from_reference_cfg(config)
        self.is_distillation_enabled = self.distill_config is not None
        self.fp8 = fp8_from_config(config)                           # student.fp8_enabled, fp8_filter: blocks
        self.n_local_crops = config.crops.local_crops_number
        self.embed_dim = self.engine_config.embed_dim
        self.dino_out_dim = config.dino.head_n_prototypes
        self.dino_loss_weight = config.dino.loss_weight
        self.dino_koleo_loss_weight = config.dino.koleo_loss_weight
        self.ibot_loss_weight = config.ibot.loss_weight
        # dino.local_loss_weight_schedule (:150-163) and gram.loss_weight_schedule (:183-199): per-iteration weights
        # that do_train passes to every step; None: the local weight is 1 and the gram weight gram.loss_weight
        self.dino_local_loss_schedule = (loss_weight_schedule(config, config.dino.local_loss_weight_schedule)
                                         if config.dino.get("reweight_dino_local_loss", False) else None)
        gs = config.gram.get("loss_weight_schedule", None)
        self.gram_loss_schedule = loss_weight_schedule(config, gs) if config.gram.use_loss and gs else None
        # gram anchoring (:165-254): same attribute names and the same configuration errors
        g = config.gram
        self.gram_use_loss = bool(g.use_loss)
        self.gram_ema_teacher = bool(g.get("ema_teacher", False)) if self.gram_use_loss else False
        self.has_gram_teacher = self.gram_use_loss and not self.gram_ema_teacher
        self.gram_loss_weight = g.get("loss_weight", None) if self.gram_use_loss else None
        self.gram_img_level = g.get("img_level", None) if self.gram_use_loss else None
        self.gram_tokens_used = g.get("tokens_used", None) if self.gram_use_loss else None
        self.gram_compute_stats = g.get("compute_stats", None) if self.gram_use_loss else None
        if self.gram_use_loss:
            if self.gram_ema_teacher and g.get("ckpt", None) is not None:
                raise ValueError("Cannot use both `gram.ema_teacher` and `gram.ckpt` at the same time. Please set one of them to False.")
            if config.crops.get("gram_teacher_crops_size", None) is None and self.has_gram_teacher:
                raise ValueError("config.crops.gram_teacher_crops_size must be set to use gram loss")          # :241-242
        self.engine = None

    @property
    def gram_teacher_initialized(self) -> bool:
        return bool(self.engine is not None and self.engine.gram_active and self.has_gram_teacher)

    # -- GPU engine -------------------------------------------------------------------------------------------------
    def build_engine(self, device="cuda", comm=None, max_masked=None) -> Engine:
        # train.checkpointing (ssl_default_config.yaml:88-89): activation rematerialisation of the student blocks
        remat = bool(self.config.train.get("checkpointing", False) or self.config.train.get("checkpointing_full", False))
        self.engine = Engine(self.engine_config, self.config.train.batch_size_per_gpu, device=device,
                             max_masked=max_masked, comm=comm, remat=remat, distill=self.distill_config,
                             fp8=self.fp8)
        if self.distill_config is not None:
            self.load_distillation_teacher(self.config.distillation.checkpoint_path)
        return self.engine

    def load_distillation_teacher(self, checkpoint_path):
        """The frozen teacher from a directory written by `checkpointer.save_checkpoint`: its teacher_* subtrees, the
        EMA teacher of the run being distilled.  It is not part of the training state, so every build (a resume
        included) loads it again."""
        from ..checkpointer import load_checkpoint
        if not checkpoint_path:
            raise ValueError("distillation.enabled needs distillation.checkpoint_path (a save_checkpoint directory)")
        params = load_checkpoint(checkpoint_path)["model_params"]
        self.engine.distill_teacher_load({m: params[f"teacher_{m}"] for m in self.PARAM_MODULES if f"teacher_{m}" in params})

    def __call__(self, data, *, teacher_temp=0, iteration=0, deterministic=True, init_phase=False):
        """Forward + backward of one batch (the reference returns (loss, metrics) and lets jax.grad differentiate it,
        :289-363; here the gradients are left in the engine's gradient buffers)."""
        if self.engine is None:
            self.build_engine()
        self.engine.set_batch(data)
        self.engine.forward_backward(float(teacher_temp))
        m = self.engine.read_metrics()
        return m["total_loss"], m

    def update_ema(self):
        """The reference returns `fn(ema_params, params, mom)` (:644-660) that the loop applies after every step
        (train/train.py:666).  Same contract: the returned callable applies teacher <- mom*teacher + (1-mom)*student on
        the engine-resident shards (d3_ema) and returns the (in-place updated) ema handle.  `do_train` itself uses the
        EMA fused into the optimizer kernel instead."""
        def _update_ema(ema_params, params=None, mom=None):
            engine = getattr(ema_params, "engine", None) or self.engine
            if engine is None:
                raise ValueError("update_ema: no engine (call build_engine / pass the EngineTree handles)")
            if mom is None:
                raise TypeError("update_ema(ema_params, params, mom): mom is required")
            engine.ema_update(float(mom))
            return ema_params
        return _update_ema

    def build_data_augmentation_dino(self, cfg):
        """:561-575 — the augmentation class stays in the reference's data package (torchvision host pipeline) and is
        resolved through the package overlay."""
        from ..data import DataAugmentationDINO
        c = cfg.crops
        return DataAugmentationDINO(
            c.global_crops_scale, c.local_crops_scale, c.local_crops_number, global_crops_size=c.global_crops_size,
            local_crops_size=c.local_crops_size, gram_teacher_crops_size=c.get("gram_teacher_crops_size", None),
            gram_teacher_no_distortions=c.get("gram_teacher_no_distortions", False),
            local_crops_subset_of_global_crops=c.get("localcrops_subset_of_globalcrops", False),
            share_color_jitter=c.get("share_color_jitter", False), horizontal_flips=c.get("horizontal_flips", True),
            mean=c.get("rgb_mean", (0.485, 0.456, 0.406)), std=c.get("rgb_std", (0.229, 0.224, 0.225)))

    def get_params_groups(self, params=None):
        """name -> (lr_multiplier, wd_multiplier, is_last_layer) for every student tensor (:577-598 / param_groups.py)."""
        from ..engine.params import backbone_spec, head_spec
        out = {}
        for module, spec in (("backbone", backbone_spec(self.engine_config)),
                             ("dino_head", head_spec(self.engine_config, "dino_head")),
                             ("ibot_head", head_spec(self.engine_config, "ibot_head"))):
            for name, _, _ in spec:
                out[f"student_{module}/{name}"] = lr_wd_multipliers(module, name, self.engine_config)
        return out

    def prepare_for_distributed_training(self, params=None):
        """:600-642 shards the six sub-trees with `ac_compile_parallelize`.  Engine-resident state is sharded when the
        engine is built with a communicator (`build_engine(comm=...)`: fsdp/layout.py), so a handle passes through;
        a plain reference-named pytree is sharded with the mirrored policy."""
        if params is None or hasattr(params, "engine"):
            return params
        from ..fsdp.ac_compile_parallelize import ac_compile_parallelize
        return {k: ac_compile_parallelize(v, None, self.config) for k, v in params.items()}
