"""Static description of one training configuration for the GPU engine (derived from the reference's YAML keys).

Field names follow dinov3_jax/configs/ssl_default_config.yaml; arch table follows
dinov3_jax/models/vision_transformer.py:325-408.
"""
from __future__ import annotations

from dataclasses import dataclass, replace

ARCHS = {  # name -> (embed_dim, depth, heads)
    "vit_small": (384, 12, 6),
    "vit_base": (768, 12, 12),
    "vit_large": (1024, 24, 16),
    "vit_so400m": (1152, 27, 18),
    "vit_huge2": (1280, 32, 20),
    "vit_giant2": (1536, 40, 24),
    "vit_7b": (4096, 40, 32),        # head_dim 128
}
# constructor defaults of a factory beyond the table (models/vision_transformer.py:400-408: vit_7b has ffn_ratio 3)
ARCH_DEFAULTS = {"vit_7b": {"ffn_ratio": 3.0}}
# student.ffn_layer -> (EngineConfig.ffn_layer, swiglu_align)   models/vision_transformer.py:30-36
FFN_LAYERS = {"mlp": ("mlp", 8), "swiglu": ("swiglu", 8), "swiglu32": ("swiglu", 32), "swiglu64": ("swiglu", 64),
              "swiglu128": ("swiglu", 128)}


@dataclass(frozen=True)
class EngineConfig:
    embed_dim: int = 384
    depth: int = 12
    heads: int = 6
    patch: int = 16
    ffn_ratio: float = 4.0
    global_size: int = 224
    local_size: int = 96
    n_global: int = 2
    n_local: int = 8
    n_prototypes: int = 65536        # the DINO head's sizes (dino.head_*)
    head_hidden: int = 2048
    head_bottleneck: int = 256
    # the iBOT head's sizes (ibot.head_*); None: the same as the DINO head.  No concrete defaults on purpose: then
    # config_for(..., n_prototypes=4096) would still build a 65 536-prototype iBOT head
    ibot_n_prototypes: int | None = None
    ibot_head_hidden: int | None = None
    ibot_head_bottleneck: int | None = None
    layerscale: float = 1e-5
    rope_base: float = 100.0
    student_temp: float = 0.1
    dino_loss_weight: float = 1.0
    koleo_loss_weight: float = 0.1
    # dino.koleo_loss_distributed: top-k neighbours over the class tokens of a loss group of koleo_group_size images
    # (None: every rank's), engine/koleo.py.  Off: the plain per-rank KoLeo (d3_koleo_fwd_bwd_rows)
    koleo_distributed: bool = False
    koleo_topk: int = 1
    koleo_group_size: int | None = None
    ibot_loss_weight: float = 1.0
    clip_grad: float = 3.0
    ln_eps: float = 1e-6             # norm_layer layernorm: 1e-6, layernormbf16: 1e-5 (models/vision_transformer.py:38-42)
    n_storage: int = 0               # student.n_storage_tokens (register tokens after cls, vision_transformer.py:106-111)
    mlp_second_act: bool = True      # reference applies GELU after fc2 too (layers/ffn_layers.py:47)
    ffn_layer: str = "mlp"           # "mlp" | "swiglu" (layers/ffn_layers.py:52-76; SURVEY 8f.1: the 7B recipe uses swiglu64)
    swiglu_align: int = 8            # swiglu / swiglu32 / swiglu64 / swiglu128 (models/vision_transformer.py:30-36)
    mask_k_bias: bool = False        # student.mask_k_bias: the k third of the qkv bias is masked to zero (upstream DINOv3)
    qkv_bias: bool = True            # student.qkv_bias; false only for a frozen distillation teacher (the 7B recipes)
    layerwise_decay: float = 0.9
    patch_embed_lr_mult: float = 0.2
    dino_head_wd_multiplier: float = 1.0
    adamw_beta1: float = 0.9
    adamw_beta2: float = 0.999
    mask_probability: float = 0.5
    mask_ratio: tuple = (0.1, 0.5)
    # Gram anchoring (SURVEY 8f.2; configs/ssl_default_config.yaml:55-73, loss/gram_loss.py, train/ssl_meta_arch.py:165-254)
    gram_use_loss: bool = False
    gram_loss_weight: float = 1.0
    gram_ema_teacher: bool = False    # true: the EMA teacher's patch tokens are the targets (no third backbone pass)
    gram_normalized: bool = True
    gram_img_level: bool = False
    gram_remove_neg: bool = False
    gram_remove_only_teacher_neg: bool = False
    gram_tokens_used: str = "all"     # all | masked | unmasked
    gram_it_load_ema_teacher: int = -1
    gram_rep_update: bool = True
    gram_update_frequency: int = 50000
    gram_it_first_update: int = 0
    gram_max_updates: int | None = None
    gram_teacher_size: int | None = None      # crops.gram_teacher_crops_size: the gram teacher's crop resolution (None: global_size)
    gram_resize_antialias: bool = False       # gram.global_teacher_resize_antialias (method: bicubic)

    @property
    def head_dim(self) -> int:
        return self.embed_dim // self.heads

    @property
    def hidden(self) -> int:
        return int(self.embed_dim * self.ffn_ratio)

    @property
    def swiglu_hidden(self) -> int:
        d = int(self.hidden * 2 / 3)                       # layers/ffn_layers.py:64-65
        return d + (-d % self.swiglu_align)

    @property
    def ffn_width(self) -> int:
        """Columns of the FFN's hidden activation h (what fc2 / w3 contracts over)."""
        return self.swiglu_hidden if self.ffn_layer == "swiglu" else self.hidden

    def head_dims(self, module: str) -> tuple:
        """(hidden, bottleneck, prototypes) of "dino_head" or "ibot_head" (layers/dino_head.py)."""
        if module == "dino_head":
            return self.head_hidden, self.head_bottleneck, self.n_prototypes
        if module == "ibot_head":
            own = lambda v, dino: dino if v is None else v
            return (own(self.ibot_head_hidden, self.head_hidden), own(self.ibot_head_bottleneck, self.head_bottleneck),
                    own(self.ibot_n_prototypes, self.n_prototypes))
        raise ValueError(f"no head named {module!r} (dino_head | ibot_head)")

    def patches(self, size: int) -> int:
        return (size // self.patch) ** 2

    @property
    def prefix(self) -> int:
        """Tokens in front of the patch tokens (cls + storage): they are not rotated by RoPE."""
        return 1 + self.n_storage

    def tokens(self, size: int) -> int:
        return self.patches(size) + self.prefix


def config_for(arch: str, **kw) -> EngineConfig:
    d, l, h = ARCHS[arch]
    return replace(EngineConfig(embed_dim=d, depth=l, heads=h), **{**ARCH_DEFAULTS.get(arch, {}), **kw})


def from_oracle_cfg(c) -> EngineConfig:
    """Build from any object with the same field names (tests pass oracle.arch.ModelCfg)."""
    names = EngineConfig.__dataclass_fields__.keys()
    return EngineConfig(**{k: getattr(c, k) for k in names if hasattr(c, k)})


def config_from_reference_cfg(cfg) -> EngineConfig:
    """Map the reference's YAML keys (configs/ssl_default_config.yaml) onto the engine configuration; unsupported
    options the reference asserts on (train/ssl_meta_arch.py:47-51) or that this engine does not implement raise."""
    if cfg.train.centering != "sinkhorn_knopp":
        raise NotImplementedError("train.centering must be sinkhorn_knopp (asserted by the reference, ssl_meta_arch.py:49)")
    if not cfg.ibot.separate_head:
        raise NotImplementedError("ibot.separate_head must be true (ssl_meta_arch.py:48)")
    if cfg.crops.local_crops_number <= 0:
        raise ValueError("crops.local_crops_number must be > 0 (ssl_meta_arch.py:47)")
    ffn_table = FFN_LAYERS
    if cfg.student.ffn_layer not in ffn_table or cfg.student.norm_layer not in ("layernorm", "layernormbf16"):
        raise NotImplementedError("ffn_layer must be mlp | swiglu[32|64|128] and norm_layer layernorm | layernormbf16 "
                                  "(RMSNorm is not on the GPU path, SURVEY 8f)")
    koleo_kw = koleo_config_from_reference_cfg(cfg)
    gram_kw = {}
    if cfg.gram.use_loss:
        gg = cfg.gram
        if str(gg.get("tokens_used", "all")) not in ("all", "masked", "unmasked"):
            raise ValueError("gram.tokens_used must be all | masked | unmasked (ssl_meta_arch.py:221)")
        if str(gg.get("tokens_used", "all")) != "all" and gg.get("img_level", False):
            raise ValueError("gram.tokens_used masked | unmasked needs gram.img_level: false (ssl_meta_arch.py:222-223)")
        if gg.get("compute_stats", False):
            import warnings
            warnings.warn("gram.compute_stats: the stats_only/* metrics are not produced by the GPU engine", stacklevel=2)
        if gg.get("ckpt", None) is not None:
            raise NotImplementedError("gram.ckpt: load the gram teacher with dinov3_jax.checkpointer and Engine.gram_teacher_load "
                                      "instead of a path in the config")
        gsz = cfg.crops.get("gram_teacher_crops_size", None)
        if gsz is not None and not isinstance(gsz, int):
            raise NotImplementedError("multi-resolution crops.gram_teacher_crops_size lists (train/train.py:718-769): the engine "
                                      "is built for one resolution triple")
        if gsz is not None and gg.get("ema_teacher", False):
            raise ValueError("crops.gram_teacher_crops_size should be None when gram.ema_teacher=True (ssl_meta_arch.py:243-244)")
        if gsz is not None and (int(gsz) // cfg.student.patch_size) ** 2 + 1 + int(cfg.student.n_storage_tokens) > 448:
            raise NotImplementedError("crops.gram_teacher_crops_size: the single-pass attention kernel holds at most 448 tokens "
                                      "per crop (gram teacher crops up to 320^2 at patch 16)")
        if gsz is not None and int(gsz) != int(cfg.crops.global_crops_size) and \
                str(gg.get("global_teacher_resize_method", "bicubic")) != "bicubic":
            raise NotImplementedError("gram.global_teacher_resize_method must be bicubic")
        if bool(gg.get("remove_neg", False)) and bool(gg.get("remove_only_teacher_neg", False)):
            raise ValueError("gram.remove_neg and gram.remove_only_teacher_neg are exclusive (loss/gram_loss.py:20)")
        if not gg.get("ema_teacher", False) and int(gg.get("it_load_ema_teacher", -1)) < 0:
            raise ValueError("if no gram checkpoint is provided, gram.it_load_ema_teacher must be >= 0 (ssl_meta_arch.py:215-218)")
        gram_kw = dict(gram_use_loss=True, gram_loss_weight=float(gg.loss_weight), gram_ema_teacher=bool(gg.ema_teacher),
                       gram_normalized=bool(gg.normalized), gram_img_level=bool(gg.get("img_level", False)), gram_remove_neg=bool(gg.remove_neg),
                       gram_remove_only_teacher_neg=bool(gg.remove_only_teacher_neg), gram_tokens_used=str(gg.tokens_used),
                       gram_it_load_ema_teacher=int(gg.it_load_ema_teacher), gram_rep_update=bool(gg.rep_update),
                       gram_update_frequency=int(gg.update_frequency), gram_it_first_update=int(gg.it_first_update),
                       gram_max_updates=gg.get("max_updates", None),
                       gram_teacher_size=None if gsz is None else int(gsz),
                       gram_resize_antialias=bool(gg.get("global_teacher_resize_antialias", False)))
    # options this engine does not implement must not be silently ignored (the run would differ from the request)
    g = lambda node, key, default: node.get(key, default) if hasattr(node, "get") else getattr(node, key, default)
    if "schedules" in cfg and cfg["schedules"]:
        raise NotImplementedError("schedules (v2) block: only the v1 optim.* / teacher.* schedule keys are honoured")
    if not g(cfg.dino, "global_ignore_diagonal", True):
        raise NotImplementedError("dino.global_ignore_diagonal=false: the pair tables implement the default (true)")
    if int(g(cfg.dino, "head_nlayers", 3)) != 3 or int(g(cfg.ibot, "head_nlayers", 3)) != 3:
        raise NotImplementedError("head_nlayers != 3 (layers/dino_head.py default) is not on the GPU path")
    if "multidistillation" in cfg and g(cfg["multidistillation"], "enabled", False):
        raise NotImplementedError("multidistillation is outside the training hot path (SURVEY §2 out of scope)")
    if float(g(cfg.student, "drop_path_rate", 0.0) or 0.0) > 0.0:
        import warnings
        warnings.warn("student.drop_path_rate > 0 is ignored: like the reference's deterministic branch "
                      "(layers/block.py:195-201, the only one its train_step traces: deterministic=True, "
                      "train/ssl_meta_arch.py:289), the engine applies no stochastic depth", stacklevel=2)
    arch = cfg.student.arch
    if arch not in ARCHS:
        raise ValueError(f"unknown student.arch {arch!r}")
    if arch == "vit_7b":
        # the shipped 7B recipes set these; the engine's blocks always carry a qkv bias and one shared cls norm
        if not g(cfg.student, "qkv_bias", True):
            raise NotImplementedError("student.qkv_bias=false is not on the GPU path (every block has a qkv bias)")
        for key in ("untie_cls_and_patch_norms", "untie_global_and_local_cls_norm"):
            if g(cfg.student, key, False):
                raise NotImplementedError(f"student.{key}=true is not on the GPU path (one final norm for every token)")
    # an ibot_* field is set only where the iBOT head differs, so equal heads map to the same EngineConfig as ever
    ibot_kw = {field: int(getattr(cfg.ibot, key)) for field, key in (("ibot_n_prototypes", "head_n_prototypes"),
                                                                     ("ibot_head_hidden", "head_hidden_dim"),
                                                                     ("ibot_head_bottleneck", "head_bottleneck_dim"))
               if getattr(cfg.ibot, key) != getattr(cfg.dino, key)}
    return config_for(
        arch, patch=cfg.student.patch_size, ffn_ratio=cfg.student.ffn_ratio, global_size=cfg.crops.global_crops_size,
        local_size=cfg.crops.local_crops_size, n_local=cfg.crops.local_crops_number,
        n_prototypes=cfg.dino.head_n_prototypes, head_hidden=cfg.dino.head_hidden_dim,
        head_bottleneck=cfg.dino.head_bottleneck_dim, layerscale=cfg.student.layerscale,
        rope_base=cfg.student.pos_embed_rope_base, dino_loss_weight=cfg.dino.loss_weight,
        koleo_loss_weight=cfg.dino.koleo_loss_weight, ibot_loss_weight=cfg.ibot.loss_weight,
        clip_grad=cfg.optim.clip_grad, layerwise_decay=cfg.optim.layerwise_decay,
        patch_embed_lr_mult=cfg.optim.patch_embed_lr_mult, dino_head_wd_multiplier=cfg.optim.dino_head_wd_multiplier,
        adamw_beta1=cfg.optim.adamw_beta1, adamw_beta2=cfg.optim.adamw_beta2,
        mask_probability=cfg.ibot.mask_sample_probability, mask_ratio=tuple(cfg.ibot.mask_ratio_min_max),
        n_storage=int(cfg.student.n_storage_tokens), ln_eps=1e-5 if cfg.student.norm_layer == "layernormbf16" else 1e-6,
        ffn_layer=ffn_table[cfg.student.ffn_layer][0], swiglu_align=ffn_table[cfg.student.ffn_layer][1],
        mask_k_bias=bool(cfg.student.get("mask_k_bias", False)),
        mlp_second_act=ffn_table[cfg.student.ffn_layer][0] == "mlp", **ibot_kw, **gram_kw, **koleo_kw)


def koleo_config_from_reference_cfg(cfg) -> dict:
    """dino.koleo_loss_distributed / koleo_topk / koleo_distributed_loss_group_size / _group_data /
    koleo_distributed_replicas (train/ssl_meta_arch.py:94-106) as EngineConfig fields.  A group size must be a
    multiple of train.batch_size_per_gpu (that it divides the global batch is checked when the engine knows the
    world size)."""
    from .koleo import MAX_TOPK
    d = cfg.dino
    g = lambda key, default: d.get(key, default) if hasattr(d, "get") else getattr(d, key, default)
    topk = int(g("koleo_topk", 1))
    if not g("koleo_loss_distributed", False):
        if topk != 1:
            raise ValueError("dino.koleo_topk > 1 needs dino.koleo_loss_distributed: true (ssl_meta_arch.py:105)")
        return {}
    if int(g("koleo_distributed_replicas", 0) or 0) != 0:
        raise ValueError("dino.koleo_distributed_replicas is no longer supported: it must be 0 (ssl_meta_arch.py:97)")
    if not g("koleo_distributed_loss_group_data", True):
        raise NotImplementedError("dino.koleo_distributed_loss_group_data: false: a loss group is always consecutive "
                                  "ranks' images")
    G = g("koleo_distributed_loss_group_size", None)
    B = int(cfg.train.batch_size_per_gpu)
    if G is not None:
        G = int(G)
        if G <= 0 or G % B:
            raise ValueError(f"dino.koleo_distributed_loss_group_size {G} must be a multiple of "
                             f"train.batch_size_per_gpu {B}")
    if not 1 <= topk <= MAX_TOPK or (G is not None and topk > G - 1):
        raise ValueError(f"dino.koleo_topk {topk} must be in [1, min({MAX_TOPK}, rows in the loss group - 1)]")
    return dict(koleo_distributed=True, koleo_topk=topk, koleo_group_size=G)


def distill_config_from_reference_cfg(cfg) -> EngineConfig | None:
    """The frozen teacher of `distillation.enabled` (train/ssl_meta_arch.py:257-286), or None without distillation.

    `distillation.full_cfg_path` is merged over the defaults like any run configuration, and its `student.*` block is
    read the way `build_model_from_cfg(only_teacher=True)` reads it; the heads take its `dino.*` / `ibot.*` sizes.  The
    teacher config's optim / schedules / crops / train blocks are ignored: the teacher is frozen and sees the student's
    global crops."""
    g = lambda node, key, default: node.get(key, default) if hasattr(node, "get") else getattr(node, key, default)
    dist = g(cfg, "distillation", None)
    if dist is None or not g(dist, "enabled", False):
        return None
    if cfg.gram.use_loss:
        raise NotImplementedError("distillation together with gram.use_loss is not on the GPU path")
    from ..configs.config import DinoV3SetupArgs, get_cfg_from_args
    path = str(g(dist, "full_cfg_path", "") or "")
    if not path:
        raise ValueError("distillation.enabled needs distillation.full_cfg_path (the teacher's config)")
    t = get_cfg_from_args(DinoV3SetupArgs(config_file=path))
    # the reference's asserts (train/ssl_meta_arch.py:264-267)
    if not t.ibot.separate_head:
        raise ValueError("the distillation teacher needs ibot.separate_head: true (ssl_meta_arch.py:264)")
    if t.ibot.head_n_prototypes != cfg.ibot.head_n_prototypes or t.dino.head_n_prototypes != cfg.dino.head_n_prototypes:
        raise ValueError("the distillation teacher's dino / ibot head_n_prototypes must equal the student's "
                         "(ssl_meta_arch.py:265-266)")
    if t.student.patch_size != cfg.student.patch_size:
        raise ValueError("the distillation teacher's patch_size must equal the student's (ssl_meta_arch.py:267)")
    s = t.student
    if s.arch not in ARCHS:
        raise ValueError(f"unknown teacher student.arch {s.arch!r}")
    if s.ffn_layer not in FFN_LAYERS or s.norm_layer not in ("layernorm", "layernormbf16"):
        raise NotImplementedError("teacher ffn_layer must be mlp | swiglu[32|64|128] and norm_layer layernorm | layernormbf16")
    if g(s, "untie_cls_and_patch_norms", False):
        raise NotImplementedError("teacher student.untie_cls_and_patch_norms=true is not on the GPU path")
    if not g(s, "proj_bias", True) or not g(s, "ffn_bias", True):
        raise NotImplementedError("teacher student.proj_bias / ffn_bias = false is not on the GPU path")
    if int(g(t.dino, "head_nlayers", 3)) != 3 or int(g(t.ibot, "head_nlayers", 3)) != 3:
        raise NotImplementedError("teacher head_nlayers != 3 is not on the GPU path")
    # untie_global_and_local_cls_norm is accepted: local_cls_norm applies only to local crops, which the teacher never
    # sees (models/vision_transformer.py:224-226)
    ibot_kw = {field: int(getattr(t.ibot, key)) for field, key in (("ibot_n_prototypes", "head_n_prototypes"),
                                                                   ("ibot_head_hidden", "head_hidden_dim"),
                                                                   ("ibot_head_bottleneck", "head_bottleneck_dim"))
               if getattr(t.ibot, key) != getattr(t.dino, key)}
    return config_for(
        s.arch, patch=s.patch_size, ffn_ratio=s.ffn_ratio, global_size=cfg.crops.global_crops_size,
        local_size=cfg.crops.local_crops_size, n_local=cfg.crops.local_crops_number,
        n_prototypes=t.dino.head_n_prototypes, head_hidden=t.dino.head_hidden_dim, head_bottleneck=t.dino.head_bottleneck_dim,
        layerscale=s.layerscale, rope_base=s.pos_embed_rope_base, n_storage=int(s.n_storage_tokens),
        ln_eps=1e-5 if s.norm_layer == "layernormbf16" else 1e-6, ffn_layer=FFN_LAYERS[s.ffn_layer][0],
        swiglu_align=FFN_LAYERS[s.ffn_layer][1], mask_k_bias=bool(g(s, "mask_k_bias", False)),
        qkv_bias=bool(g(s, "qkv_bias", True)), mlp_second_act=FFN_LAYERS[s.ffn_layer][0] == "mlp", **ibot_kw)
