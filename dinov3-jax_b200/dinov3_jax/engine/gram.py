"""Gram anchoring (SURVEY 8f.2; loss/gram_loss.py:13-50, train/ssl_meta_arch.py:165-254,527-541): MSE between the
patch-similarity matrices of the student's and a gram teacher's global-crop patch tokens over the rank's local batch.
The gram teacher is the EMA teacher (gram.ema_teacher) or a frozen snapshot of it, at the global-crop or its own size."""
from __future__ import annotations

import torch

from .. import ops
from .config import EngineConfig
from .forward import CropSet, Net, Stream, backbone_fwd
from .params import FrozenStore, backbone_spec

f32, bf16 = torch.float32, torch.bfloat16

METRIC = 4          # slot of the Gram term in the engine's metrics


def pad8(n: int) -> int:
    return (n + 7) // 8 * 8


def operands(feats, x, nrm, n: int, normalized: bool):
    """Gram GEMM operands x (bf16) from n feature rows: zero rows up to the kernels' 8-row granule (zero similarity on
    both sides: no contribution), then L2-normalised (`normalized`) or cast.  `feats` None: x already holds the rows."""
    npad = pad8(n)
    if npad > n:
        (x if feats is None else feats)[n:npad].zero_()
    if feats is None:
        return
    if normalized:
        ops.l2norm_fwd(feats[:npad], x[:npad], nrm[:npad], 1e-12)
    else:
        ops.cast_f32_bf16(feats[:npad].reshape(-1), x[:npad].reshape(-1))


def similarity_diff(xs, xt, Ss, St, G, mode: int, inv: float, loss, block: int = 0):
    """St = Xt Xt^T, Ss = Xs Xs^T, then d3_gram_diff: loss += inv * sum (s' - t')^2 and, with G, its gradient."""
    ops.gemm(xt, xt, St)
    ops.gemm(xs, xs, Ss)
    ops.gram_diff(Ss, St, G, mode, inv, loss, block=block)


def _patch_rows(cs: CropSet, prefix: int, device):
    return (torch.arange(cs.n, dtype=torch.int32)[:, None] * cs.N + prefix
            + torch.arange(cs.P, dtype=torch.int32)[None, :]).reshape(-1).to(device)


class GramAnchor:
    """The Gram term of the engine's step: buffers, gram teacher, targets, loss and backward.  `sg`: the global crops."""

    def __init__(self, cfg: EngineConfig, sg: CropSet, device, fp8: bool = False):
        assert cfg.gram_tokens_used in ("all", "masked", "unmasked")         # train/ssl_meta_arch.py:221
        if cfg.gram_tokens_used != "all" and cfg.gram_img_level:
            raise ValueError("gram.tokens_used masked | unmasked needs gram.img_level: false (train/ssl_meta_arch.py:222-223)")
        gs = cfg.gram_teacher_size
        hi = not cfg.gram_ema_teacher and gs is not None and gs != cfg.global_size
        if hi and cfg.gram_tokens_used != "all":
            raise NotImplementedError("gram.tokens_used masked | unmasked with a gram teacher at its own resolution")
        self.cfg, self.device, self._sg = cfg, device, sg
        self.active = bool(cfg.gram_ema_teacher)     # the EMA teacher is always there; a frozen one once loaded
        self.weight = float(cfg.gram_loss_weight)
        self.updates = 0
        self._snapshot_pending = False
        self.stream = self.img = None
        D = cfg.embed_dim
        self.rows_all = _patch_rows(sg, cfg.prefix, device)                  # token row of every global-crop patch
        self.rows = self.rows_all                                            # rows in use: all | masked | unmasked
        self.n = sg.n * sg.P                                                 # live row count; buffers hold the maximum
        self.block = sg.P if cfg.gram_img_level else 0                       # per-image Gram matrices: diagonal blocks
        self.mode = ops.GRAM_MODES[(bool(cfg.gram_remove_neg), bool(cfg.gram_remove_only_teacher_neg))]
        e = lambda *shape, dt: torch.empty(*shape, dtype=dt, device=device)
        npad = pad8(self.n)
        self.fs, self.ft = e(npad, D, dt=f32), e(npad, D, dt=f32)          # gathered final-norm patch tokens
        self.xs, self.xt = e(npad, D, dt=bf16), e(npad, D, dt=bf16)        # (normalised) GEMM operands
        self.nrm_s, self.nrm_t = e(npad, dt=f32), e(npad, dt=f32)
        self.Ss, self.St = e(npad * npad, dt=f32), e(npad * npad, dt=f32)
        self.G = e(npad * npad, dt=bf16)
        self.dX, self.dF = e(npad, D, dt=bf16), e(npad, D, dt=bf16)
        # a frozen gram teacher: a full copy on every rank, in the backbone's flat layout (a snapshot copies the EMA's)
        self.net = None if cfg.gram_ema_teacher else Net(cfg, {"backbone": FrozenStore(backbone_spec(cfg), device)}, True, fp8=fp8)
        if hi:
            # a stream at the gram teacher's own size, resized to the student's grid (upstream get_gram_teacher_output)
            gp = CropSet(cfg, sg.n, gs // cfg.patch, gs // cfg.patch, 0, device)
            self.stream = Stream(cfg, [gp], device, stash=False)
            self.rows_hi = _patch_rows(gp, cfg.prefix, device)
            self.hi = e(gp.n * gp.P, D, dt=f32)

    def teacher_load(self, tensors: dict):
        """Gram teacher weights: backbone tensor names (reference layout, e.g. 'blocks_0/attn/qkv/kernel') -> arrays."""
        assert self.net is not None
        store = self.net.mods["backbone"]
        store.load({name: tensors[name] for name in store.offsets}, self.cfg.mask_k_bias)
        self.active = True

    def schedule(self, iteration: int):
        """Gram teacher refreshes (upstream DINOv3 train loop): a copy of the EMA teacher at gram.it_load_ema_teacher, then
        every gram.update_frequency iterations (gram.rep_update), taken in the next step after the EMA teacher's forward."""
        cfg = self.cfg
        if self.net is None:
            return
        if iteration == cfg.gram_it_load_ema_teacher:
            self._snapshot_pending = True
        elif (cfg.gram_rep_update and self.active and iteration >= cfg.gram_it_first_update
              and (iteration + 1) % cfg.gram_update_frequency == 0
              and (cfg.gram_max_updates is None or self.updates < cfg.gram_max_updates)):
            self._snapshot_pending = True
            self.updates += 1

    def state(self) -> tuple:
        """Checkpoint entries of a frozen gram teacher, so that a resumed run keeps the Gram term: (params, opt state)."""
        if self.net is None or not self.active:
            return {}, {}
        return ({f"gram_backbone/{k}": v.cpu() for k, v in self.net.mods["backbone"].export().items()},
                {"gram_updates": int(self.updates)})

    def load_state(self, flat: dict, optimizer_state: dict | None):
        """The entries of `state` from a flat checkpoint tree (ignored with the EMA teacher)."""
        gram = {k[len("gram_backbone/"):]: v for k, v in flat.items() if k.startswith("gram_backbone/")}
        if gram and self.net is not None:
            self.teacher_load(gram)
            if optimizer_state is not None and "gram_updates" in optimizer_state:
                self.updates = int(optimizer_state["gram_updates"])

    def set_batch(self, batch: dict, rows_masked, M: int, masks_u8):
        """The gram teacher's crops; the rows of gram.tokens_used (ssl_meta_arch.py:221-223; upstream patches[~masks])."""
        if self.stream is not None and batch.get("collated_gram_teacher_crops", None) is not None:
            self.img = batch["collated_gram_teacher_crops"].to(device=self.device, dtype=bf16, non_blocking=True).contiguous()
        if self.cfg.gram_tokens_used == "masked":
            self.rows, self.n = rows_masked, M
        elif self.cfg.gram_tokens_used == "unmasked":
            # stable sort of the mask bits: unmasked patch positions first, in order (no host sync, count known)
            order = torch.argsort(masks_u8.reshape(-1).to(torch.int16), stable=True)[: self.rows_all.numel() - M]
            self.rows, self.n = self.rows_all[order].contiguous(), order.numel()

    def features(self, Xn, student: bool):
        """The selected global-crop patch tokens of a final-norm output -> the student's or the teacher's operands."""
        feats, x, nrm = (self.fs, self.xs, self.nrm_s) if student else (self.ft, self.xt, self.nrm_t)
        if self.n == 0:
            return
        norm = self.cfg.gram_normalized
        ops.gather_rows(Xn, self.rows, self.n, self.cfg.embed_dim, **({"dst_f32": feats} if norm else {"dst_bf16": x}))
        operands(feats if norm else None, x, nrm, self.n, norm)

    def teacher_targets(self, teacher: Stream, g_img, ema_backbone):
        """End of the teacher pass: the EMA teacher's outputs are in `teacher`, its gathered weights in `ema_backbone`."""
        if self._snapshot_pending:
            g = self.net.mods["backbone"]
            g.bf16.copy_(ema_backbone.t_bf16)
            g.vecs.copy_(ema_backbone.t_vecs)
            self._snapshot_pending, self.active = False, True
        if not self.active:
            return
        if self.stream is not None:
            if self.img is None:
                raise ValueError("no gram teacher crops in the data, have you set cfg.crops.gram_teacher_crops_size? "
                                 "(train/ssl_meta_arch.py:310-313)")
            backbone_fwd(self.net, self.stream, [self.img], [None])
            gp, sg, D = self.stream.sets[0], self._sg, self.cfg.embed_dim
            ops.gather_rows(self.stream.Xn, self.rows_hi, gp.n * gp.P, D, dst_f32=self.hi)
            ops.resize_tokens_bicubic(self.hi, self.ft[:sg.n * sg.P], gp.n, gp.Hp, gp.Wp, sg.Hp, sg.Wp, D,
                                      self.cfg.gram_resize_antialias)
            operands(self.ft, self.xt, self.nrm_t, self.n, self.cfg.gram_normalized)
            return
        if self.net is not None:      # the EMA teacher's kernels and buffers, reading the frozen weights
            backbone_fwd(self.net, teacher, [g_img], [None])
        self.features(teacher.Xn, student=False)

    def loss_bwd(self, dXn, metrics):
        """loss/gram_loss.py:38-50 into metrics[METRIC]; dXs = (4 w / count) G Xs (G symmetric), through l2norm, into dXn."""
        n, D = self.n, self.cfg.embed_dim
        if n == 0:
            return
        npad = pad8(n)
        inv = 1.0 / (float(n) * float(self.block or n))            # 1 / entries under the mean
        sq = lambda b: b[:npad * npad].view(npad, npad)
        similarity_diff(self.xs[:npad], self.xt[:npad], sq(self.Ss), sq(self.St), sq(self.G), self.mode, inv,
                        metrics[METRIC:METRIC + 1], block=self.block)
        ops.gemm(sq(self.G), self.xs[:npad], self.dX[:npad], b_mn=True, alpha=4.0 * self.weight * inv)
        if self.cfg.gram_normalized:
            ops.l2norm_bwd(self.dX[:npad], self.fs[:npad], self.nrm_s[:npad], self.dF[:npad])
        ops.scatter_add_rows(self.dF if self.cfg.gram_normalized else self.dX, self.rows, dXn, n, D)

    def read(self, m: list, out: dict) -> float:
        """The Gram entries of Engine.read_metrics (train/ssl_meta_arch.py:538-541); returns the weighted term."""
        out["gram_loss"], out["gram_loss_weight"] = m[METRIC], self.weight
        return self.weight * m[METRIC]
