"""GPU step executor for the DINOv3 SSL hot path (replaces the jitted `train_step` of the reference,
dinov3_jax/train/train.py:491-565, and `SSLMetaArch.__call__`, train/ssl_meta_arch.py:289-363).

There is no autograd and no PyTorch math here: the forward and the hand-derived backward are explicit sequences of
C-ABI kernel launches (`..ops`) on pre-allocated device buffers; torch only owns the memory and the stream.
Student tokens of the global and the local crops live in ONE row-concatenated stream [T_g + T_l, D] so every
token-wise op (LayerNorm, the four GEMMs of a block and their wgrads) is a single launch; only RoPE / attention see
the crop structure.  Activations needed by the backward are stashed per block (bf16 except the fp32 residual stream).
"""
from __future__ import annotations

import math
import os

import torch

from .. import ops
from .config import EngineConfig
from .params import ParamStore

f32, bf16 = torch.float32, torch.bfloat16


def rope_tables(Hp: int, Wp: int, head_dim: int, base: float, device):
    """sin / cos [Hp*Wp, head_dim] fp32 — layers/rope_position_encoding.py:36-40,64-73,117-123 (normalize 'separate').
    Host-side table construction (a few KB, once per crop size); the rotation itself is d3_rope."""
    dt = torch.float64
    periods = base ** (2.0 * torch.arange(head_dim // 4, dtype=dt) / (head_dim // 2))
    ch = torch.arange(0.5, Hp, dtype=dt) / Hp
    cw = torch.arange(0.5, Wp, dtype=dt) / Wp
    coords = torch.stack(torch.meshgrid(ch, cw, indexing="ij"), dim=-1).reshape(-1, 2)
    coords = 2.0 * coords - 1.0
    ang = 2 * math.pi * coords[:, :, None] / periods[None, None, :]
    ang = ang.reshape(ang.shape[0], -1)
    ang = torch.cat([ang, ang], dim=-1)
    # the reference computes the tables in fp32 (SURVEY A8); fp64 -> fp32 rounding differs by < 1 ulp
    return (torch.sin(ang).to(f32).to(device).contiguous(), torch.cos(ang).to(f32).to(device).contiguous())


class CropSet:
    """Static geometry of one crop resolution inside a token stream."""

    def __init__(self, cfg: EngineConfig, n_crops: int, size: int, row0: int, device):
        self.n = n_crops
        self.size = size
        self.Hp = size // cfg.patch
        self.P = self.Hp * self.Hp
        self.N = self.P + cfg.prefix
        self.T = n_crops * self.N
        self.row0 = row0
        self.sin, self.cos = rope_tables(self.Hp, self.Hp, cfg.head_dim, cfg.rope_base, device)
        kdim = cfg.patch * cfg.patch * 3
        kpad = (kdim + 7) // 8 * 8             # TMA needs 16-byte row strides (patch 14: 588 -> 592, padding zeroed)
        self.patches = torch.empty(n_crops * self.P, kpad, dtype=bf16, device=device)[:, :kdim]
        self.tok = torch.empty(n_crops * self.P, cfg.embed_dim, dtype=f32, device=device)
        self.lse = None


class Stream:
    """Activation buffers of one network pass over a list of crop sets (teacher: global only; student: global+local)."""

    def __init__(self, cfg: EngineConfig, sets, device, stash: bool, remat: bool = False):
        D, Hd, L = cfg.embed_dim, cfg.ffn_width, cfg.depth
        swiglu = cfg.ffn_layer == "swiglu"
        self.sets = sets
        self.T = sum(s.T for s in sets)
        T = self.T
        self.stash = stash                    # keep what the backward needs
        self.per_block = stash and not remat  # ... for every block (False: one scratch set, blocks are recomputed)
        nb = L if self.per_block else 1
        e = lambda *shape, dt=bf16: torch.empty(*shape, dtype=dt, device=device)
        self.X = [e(T, D, dt=f32) for _ in range(L + 1)] if stash else [e(T, D, dt=f32), e(T, D, dt=f32)]
        self.Xmid = [e(T, D, dt=f32) for _ in range(nb)]
        self.Y = [e(T, D) for _ in range(nb)]
        self.QKV = [e(T, 3 * D) for _ in range(nb)]
        self.O = [e(T, D) for _ in range(nb)]
        self.Z = [e(T, D) for _ in range(nb)]
        self.Hh = [e(T, Hd) for _ in range(nb)]
        self.Xn = e(T, D, dt=f32)
        self.X12 = e(T, 2 * Hd) if (swiglu and not stash) else None       # teacher pass: [x1 | x2] scratch
        self.LSE = [[e(s.n, cfg.heads, s.N, dt=f32) for s in sets] for _ in range(nb)]
        if stash:
            self.U1 = [e(T, 2 * Hd if swiglu else Hd) for _ in range(nb)]   # mlp: u1; swiglu: [x1 | x2]
            self.U2 = [e(T, D) for _ in range(nb)]
            self.stats = [[e(T, dt=f32) for _ in range(4)] for _ in range(nb)]   # mean1, rstd1, mean2, rstd2
            self.fstats = [e(T, dt=f32), e(T, dt=f32)]

    def x_in(self, i):
        return self.X[i] if self.stash else self.X[i % 2]

    def x_out(self, i):
        return self.X[i + 1] if self.stash else self.X[(i + 1) % 2]

    def b(self, lst, i):
        return lst[i] if self.per_block else lst[0]


class HeadBufs:
    def __init__(self, cfg: EngineConfig, R: int, device, stash: bool):
        D, Hh, Bn, K = cfg.embed_dim, cfg.head_hidden, cfg.head_bottleneck, cfg.n_prototypes
        e = lambda *shape, dt=bf16: torch.empty(*shape, dtype=dt, device=device)
        self.R = R
        self.A0 = e(R, D)
        self.H1, self.H2 = e(R, Hh), e(R, Hh)
        self.U3 = e(R, Bn, dt=f32)
        self.nrm = e(R, dt=f32)
        self.Yn = e(R, Bn)
        self.logits = e(R, K, dt=f32)
        if stash:
            self.Ua, self.Ub = e(R, Hh), e(R, Hh)
            self.dS = e(R, K)
            self.dYn, self.dU3 = e(R, Bn), e(R, Bn)
            self.dUb, self.dUa = e(R, Hh), e(R, Hh)
            self.dA0 = e(R, D, dt=f32)


class SinkhornBufs:
    """`mx`, `s`, `btot` may be views into buffers shared by the DINO and iBOT heads (`joint`): the cross-rank
    reductions of the two Sinkhorn normalisations then travel in ONE all-reduce per stage (Engine._sinkhorn_pair)."""

    def __init__(self, R: int, K: int, device, joint=None, slot: int = 0):
        if joint is None:
            self.mx = torch.empty(K, dtype=f32, device=device)  # per-prototype shift (column maxima / global max)
            self.s = torch.empty(K, dtype=f32, device=device)
            self.btot = torch.empty(1, dtype=f32, device=device)
        else:
            mx2, s2 = joint                                      # [2K], [2K + 4]: sums of both heads, then the two row totals
            self.mx = mx2[slot * K:(slot + 1) * K]
            self.s = s2[slot * K:(slot + 1) * K]
            self.btot = s2[2 * K + slot:2 * K + slot + 1]
        self.gmx = torch.empty(1, dtype=f32, device=device)
        self.a = torch.empty(R, dtype=f32, device=device)


class Engine:
    """One rank's training engine: parameters, buffers and the step.

    `B` = images per rank.  The number of masked tokens M varies per batch; buffers are sized for `max_masked`
    (default: the collate upper bound, data/collate.py:47-61) and the live M comes from `mask_indices_list`.
    """

    def __init__(self, cfg: EngineConfig, B: int, device="cuda", max_masked: int | None = None, comm=None,
                 centering: str = "sinkhorn_knopp", center_momentum: float = 0.9, remat: bool = False):
        assert cfg.head_dim == 64, "kernels are specialised for head_dim 64 (every BASELINE arch)"
        assert centering in ("sinkhorn_knopp", "softmax")
        self.centering, self.center_momentum = centering, center_momentum
        # activation rematerialisation (train.checkpointing, ssl_default_config.yaml:88): only the block inputs X[i] of
        # the student stream are kept; each block's forward is recomputed into one scratch set right before its backward
        self.remat = bool(remat)
        self.cfg, self.B, self.device = cfg, B, torch.device(device)
        self.comm = comm  # fsdp.runtime.Comm (None = single GPU)
        self.world = 1 if comm is None else comm.world
        self.rank = 0 if comm is None else comm.rank
        dev = self.device
        self.params = ParamStore(cfg, dev, self.world, self.rank)
        # the per-module squared gradient norms live in one buffer so that their cross-rank sum is one all-reduce
        self._sumsq_all = torch.zeros(len(self.params.mods), dtype=f32, device=dev)
        for i, st_ in enumerate(self.params.mods.values()):
            st_.sumsq = self._sumsq_all[i:i + 1]
        from ..fsdp.runtime import FsdpRuntime
        self.fsdp = FsdpRuntime(comm, self.params.mods, dev)
        self.params.runtime = self.fsdp
        ng, nl = cfg.n_global * B, cfg.n_local * B
        # teacher stream: global crops only; student stream: global then local rows
        self.t_sets = [CropSet(cfg, ng, cfg.global_size, 0, dev)]
        self.s_sets = [CropSet(cfg, ng, cfg.global_size, 0, dev)]
        self.s_sets.append(CropSet(cfg, nl, cfg.local_size, self.s_sets[0].T, dev))
        self.teacher = Stream(cfg, self.t_sets, dev, stash=False)
        self.student = Stream(cfg, self.s_sets, dev, stash=True, remat=self.remat)
        P = self.s_sets[0].P
        if max_masked is None:
            n_masked_crops = int(ng * cfg.mask_probability)
            max_masked = sum(int(P * (cfg.mask_ratio[0] + (cfg.mask_ratio[1] - cfg.mask_ratio[0]) * (i + 1) /
                                      max(n_masked_crops, 1))) for i in range(n_masked_crops)) + 8
        self.max_masked = max(int(max_masked), 1)
        K, D = cfg.n_prototypes, cfg.embed_dim
        self.Rc = ng + nl                         # student dino-head rows: concat(g_cls, l_cls)
        self.h_s_dino = HeadBufs(cfg, self.Rc, dev, stash=True)
        self.h_s_ibot = HeadBufs(cfg, self.max_masked, dev, stash=True)
        self.h_t_dino = HeadBufs(cfg, ng, dev, stash=False)
        self.h_t_ibot = HeadBufs(cfg, self.max_masked, dev, stash=False)
        self.sk_mx2 = torch.empty(2 * K, dtype=f32, device=dev)
        self.sk_s2 = torch.zeros(2 * K + 4, dtype=f32, device=dev)
        self.sk_btot_local = torch.zeros(4, dtype=f32, device=dev)
        # small cross-rank reductions (Sinkhorn vectors, gradient norms) over NVLink peer memory when the runtime has it
        self._ar_stage = self.fsdp.setup_small_allreduce(2 * K + 2 * (2 * K + 4) + 4) if comm is not None else None
        self.sk_dino = SinkhornBufs(ng, K, dev, joint=(self.sk_mx2, self.sk_s2), slot=0)
        self.sk_ibot = SinkhornBufs(self.max_masked, K, dev, joint=(self.sk_mx2, self.sk_s2), slot=1)
        # centers of the optional softmax-centering path ("state" collection of the reference: dino_clstoken_loss.py:19-22)
        self.center_dino = torch.zeros(K, dtype=f32, device=dev)
        self.center_ibot = torch.zeros(K, dtype=f32, device=dev)
        self._colsum = torch.zeros(K, dtype=f32, device=dev)
        i32 = torch.int32
        self.rows_masked_t = torch.empty(self.max_masked, dtype=i32, device=dev)
        self.rows_cls_t = torch.empty(ng, dtype=i32, device=dev)
        self.rows_cls_s = torch.empty(self.Rc, dtype=i32, device=dev)
        self.cls_f32 = torch.empty(self.Rc, D, dtype=f32, device=dev)     # student cls rows (fp32) for KoLeo
        self.dcls = torch.empty(self.Rc, D, dtype=f32, device=dev)
        self.koleo_xn = torch.empty(B, D, dtype=f32, device=dev)
        self.koleo_nrm = torch.empty(B, dtype=f32, device=dev)
        self.koleo_nn = torch.empty(B, dtype=i32, device=dev)
        self.koleo_coef = torch.empty(B, dtype=f32, device=dev)
        self.metrics = torch.zeros(8, dtype=f32, device=dev)   # 0 dino_local 1 dino_global 2 koleo 3 ibot
        # backward scratch over the student stream
        T, Hd = self.student.T, cfg.ffn_width
        self.swiglu = cfg.ffn_layer == "swiglu"
        e = lambda *shape, dt=bf16: torch.empty(*shape, dtype=dt, device=dev)
        self.dX = [e(T, D, dt=f32), e(T, D, dt=f32)]
        self.dXmid = e(T, D, dt=f32)
        self.dZ, self.dY, self.dO = e(T, D), e(T, D), e(T, D)
        # Weight-gradient GEMMs only feed the optimizer, so they run on a second stream and fill the tensor cores
        # while the main stream is in its HBM-bound kernels (LN / LayerScale backward, column sums).  The operands
        # they read (dU2, dU1, dP, dQKV) are double-buffered by block parity; events order reuse.
        # (with remat the weight-gradient GEMMs read the single scratch set that the next block's recompute overwrites,
        # so they stay on the main stream)
        self.wgrad_overlap = os.environ.get("D3_WGRAD_STREAM", "1") != "0" and not self.remat
        nbuf = 2 if self.wgrad_overlap else 1
        self.dU2, self.dP = [e(T, D) for _ in range(nbuf)], [e(T, D) for _ in range(nbuf)]
        self.dU1 = [e(T, 2 * Hd if self.swiglu else Hd) for _ in range(nbuf)]       # swiglu: [dx1 | dx2]
        if self.swiglu:
            self.dH = e(T, Hd)
            self.dZ32 = e(T, D, dt=f32)
        self.dQKV = [e(T, 3 * D) for _ in range(nbuf)]
        self.fwd_overlap = os.environ.get("D3_FWD_STREAMS", "0") == "1"   # off by default
        if self.fwd_overlap:
            self.tstream = torch.cuda.Stream(device=self.device)
            self._ev_fwd = [torch.cuda.Event(), torch.cuda.Event()]
        if self.wgrad_overlap:
            self.wstream = torch.cuda.Stream(device=self.device, priority=0)
            self._ev_in = [[torch.cuda.Event() for _ in range(4)] for _ in range(2)]     # main -> wgrad stream
            self._ev_done = [torch.cuda.Event() for _ in range(2)]                      # wgrad stream -> main
            self._ev_done_live = [False, False]
        self.delta = [e(s.n, cfg.heads, s.N, dt=f32) for s in self.s_sets]
        self.dTok = [e(s.n * s.P, D) for s in self.s_sets]
        self._build_ce_tables()
        self._build_rows()
        self.step_count = 0
        self._init_gram()
        self.masks_u8 = torch.zeros(ng, P, dtype=torch.uint8, device=dev)
        self.mask_idx = torch.zeros(self.max_masked, dtype=torch.int64, device=dev)
        self.M = 0

    # ------------------------------------------------------------------------------------------------ Gram anchoring
    def _init_gram(self):
        """Buffers of the Gram-anchoring term (SURVEY 8f.2; loss/gram_loss.py:13-50, train/ssl_meta_arch.py:165-254,527-541):
        MSE between the patch-similarity matrices of the student's and a gram teacher's global-crop patch tokens, over
        the rank's whole local batch (gram.img_level: false).  The gram teacher is the EMA teacher itself
        (gram.ema_teacher: true) or a frozen snapshot of it (`gram_teacher_load_from_ema`, scheduled by `gram_schedule`)
        run through the teacher path at the global-crop resolution."""
        cfg, dev = self.cfg, self.device
        self.gram_active = False
        self._gram_w = float(cfg.gram_loss_weight)
        self._gram_snapshot_pending = False
        self.gram_updates = 0
        self.gram_stream, self.gram_img = None, None
        if not cfg.gram_use_loss:
            return
        assert cfg.gram_tokens_used in ("all", "masked", "unmasked")         # train/ssl_meta_arch.py:221
        if cfg.gram_tokens_used != "all" and cfg.gram_img_level:
            raise ValueError("gram.tokens_used masked | unmasked needs gram.img_level: false (train/ssl_meta_arch.py:222-223)")
        sg = self.s_sets[0]
        D = cfg.embed_dim
        n = sg.n * sg.P
        rows = (torch.arange(sg.n, dtype=torch.int32)[:, None] * sg.N + cfg.prefix
                + torch.arange(sg.P, dtype=torch.int32)[None, :]).reshape(-1)
        self.gram_rows_all = rows.to(dev)                                    # token row of every global-crop patch
        self.gram_rows = self.gram_rows_all                                  # rows in use: all | masked | unmasked (set_batch)
        self.gram_n = n                                                      # live row count; buffers hold the maximum
        self.gram_block = sg.P if cfg.gram_img_level else 0                  # per-image Gram matrices: diagonal blocks
        e = lambda *shape, dt: torch.empty(*shape, dtype=dt, device=dev)
        npad = (n + 7) // 8 * 8
        self.gram_fs, self.gram_ft = e(npad, D, dt=f32), e(npad, D, dt=f32)  # gathered final-norm patch tokens
        self.gram_xs, self.gram_xt = e(npad, D, dt=bf16), e(npad, D, dt=bf16)  # (normalised) GEMM operands
        self.gram_nrm_s, self.gram_nrm_t = e(npad, dt=f32), e(npad, dt=f32)
        self.gram_Ss, self.gram_St = e(npad * npad, dt=f32), e(npad * npad, dt=f32)
        self.gram_G = e(npad * npad, dt=bf16)
        self.gram_dX, self.gram_dF = e(npad, D, dt=bf16), e(npad, D, dt=bf16)
        self.gram_mode = ops.GRAM_MODES[(bool(cfg.gram_remove_neg), bool(cfg.gram_remove_only_teacher_neg))]
        if cfg.gram_ema_teacher:
            self.gram_active = True
        else:
            bb = self.params.mods["backbone"]
            bb.g_bf16 = torch.zeros_like(bb.t_bf16)                          # frozen full copies on every rank
            bb.g_vecs = torch.zeros(bb.n - bb.n_mat, dtype=f32, device=dev)
            gs = cfg.gram_teacher_size
            if gs is not None and gs != cfg.global_size and cfg.gram_tokens_used != "all":
                raise NotImplementedError("gram.tokens_used masked | unmasked with a gram teacher at its own resolution")
            if gs is not None and gs != cfg.global_size:
                # the gram teacher sees its own (larger) crops: a third token stream at that resolution; its patch tokens are
                # resized to the student's grid before the similarity matrices (upstream get_gram_teacher_output)
                self.g_sets = [CropSet(cfg, sg.n, gs, 0, dev)]
                assert self.g_sets[0].N <= 448, "gram teacher crops: at most 448 tokens per crop (attention forward kernel)"
                self.gram_stream = Stream(cfg, self.g_sets, dev, stash=False)
                gp = self.g_sets[0]
                self.gram_rows_hi = (torch.arange(gp.n, dtype=torch.int32)[:, None] * gp.N + cfg.prefix
                                     + torch.arange(gp.P, dtype=torch.int32)[None, :]).reshape(-1).to(dev)
                self.gram_hi = e(gp.n * gp.P, D, dt=f32)

    def gram_teacher_load_from_ema(self):
        """The gram teacher becomes a frozen copy of the current EMA teacher.  The copy is taken inside the next step,
        right after the EMA teacher's forward, when its gathered full-size buffers are valid on every rank."""
        assert self.cfg.gram_use_loss and not self.cfg.gram_ema_teacher
        self._gram_snapshot_pending = True

    def gram_teacher_load(self, tensors: dict):
        """Gram teacher weights from a checkpoint: `tensors` maps the backbone's tensor names (reference layout, e.g.
        'blocks_0/attn/qkv/kernel', as in export_reference_tree without the 'teacher_backbone/' prefix) to arrays."""
        assert self.cfg.gram_use_loss and not self.cfg.gram_ema_teacher
        bb = self.params.mods["backbone"]
        full = torch.zeros(bb.n, dtype=f32, device=self.device)
        for name in bb.offsets:
            bb._view(full, name).copy_(torch.as_tensor(tensors[name]).to(device=self.device, dtype=f32).reshape(bb.shapes[name]))
            if self.cfg.mask_k_bias and name.endswith("attn/qkv/bias"):
                third = bb.shapes[name][0] // 3
                bb._view(full, name)[third:2 * third].zero_()
        ops.cast_f32_bf16(full[:bb.n_mat].contiguous(), bb.g_bf16)
        bb.g_vecs.copy_(full[bb.n_mat:])
        self.gram_active = True

    def gram_schedule(self, iteration: int):
        """When the gram teacher is refreshed (upstream DINOv3 train loop; the reference's loop has no such code):
        loaded from the EMA teacher at gram.it_load_ema_teacher, then, with gram.rep_update, every
        gram.update_frequency iterations from gram.it_first_update on, at most gram.max_updates times."""
        cfg = self.cfg
        if not cfg.gram_use_loss or cfg.gram_ema_teacher:
            return
        if iteration == cfg.gram_it_load_ema_teacher:
            self.gram_teacher_load_from_ema()
        elif (cfg.gram_rep_update and self.gram_active and iteration >= cfg.gram_it_first_update
              and (iteration + 1) % cfg.gram_update_frequency == 0
              and (cfg.gram_max_updates is None or self.gram_updates < cfg.gram_max_updates)):
            self.gram_teacher_load_from_ema()
            self.gram_updates += 1

    def _gram_features(self, Xn, feats, x_bf16, nrm):
        """The selected global-crop patch tokens of a final-norm output -> the Gram operands (L2-normalised rows).  The row
        count is padded to the kernels' 8-row granule with zero rows (zero similarity on both sides: no contribution)."""
        n, D = self.gram_n, self.cfg.embed_dim
        if n == 0:
            return
        npad = (n + 7) // 8 * 8
        if self.cfg.gram_normalized:
            ops.gather_rows(Xn, self.gram_rows, n, D, dst_f32=feats)
            if npad > n:
                feats[n:npad].zero_()
            ops.l2norm_fwd(feats[:npad], x_bf16[:npad], nrm[:npad], 1e-12)
        else:
            ops.gather_rows(Xn, self.gram_rows, n, D, dst_bf16=x_bf16)
            if npad > n:
                x_bf16[n:npad].zero_()

    def _gram_teacher_targets(self):
        """Called at the end of the teacher pass (the EMA teacher's outputs have been gathered into the head buffers)."""
        cfg, T_ = self.cfg, self.teacher
        if not cfg.gram_ema_teacher:
            bb = self.params.mods["backbone"]
            if self._gram_snapshot_pending:
                bb.g_bf16.copy_(bb.t_bf16)
                bb.g_vecs.copy_(bb.t_vecs)
                self._gram_snapshot_pending = False
                self.gram_active = True
            if not self.gram_active:
                return
            # the same kernels (and, at the global-crop resolution, the same buffers) as the EMA teacher's pass, reading
            # the frozen weights
            hi = self.gram_stream is not None
            if hi and self.gram_img is None:
                raise ValueError("no gram teacher crops in the data, have you set cfg.crops.gram_teacher_crops_size? "
                                 "(train/ssl_meta_arch.py:310-313)")
            keep = (bb.t_bf16, bb.t_vecs)
            bb.t_bf16, bb.t_vecs = bb.g_bf16, bb.g_vecs
            try:
                self._backbone_fwd(self.gram_stream if hi else T_, [self.gram_img if hi else self.g_img], [None], teacher=True)
            finally:
                bb.t_bf16, bb.t_vecs = keep
            if hi:
                gp, sg, D = self.g_sets[0], self.s_sets[0], cfg.embed_dim
                ops.gather_rows(self.gram_stream.Xn, self.gram_rows_hi, gp.n * gp.P, D, dst_f32=self.gram_hi)
                ops.resize_tokens_bicubic(self.gram_hi, self.gram_ft[:sg.n * sg.P], gp.n, gp.Hp, gp.Hp, sg.Hp, sg.Hp, D,
                                          cfg.gram_resize_antialias)
                n = self.gram_n                       # all patch tokens (a multiple of 8 is not guaranteed: pad with zero rows)
                npad = (n + 7) // 8 * 8
                if npad > n:
                    self.gram_ft[n:npad].zero_()
                if cfg.gram_normalized:
                    ops.l2norm_fwd(self.gram_ft[:npad], self.gram_xt[:npad], self.gram_nrm_t[:npad], 1e-12)
                else:
                    ops.cast_f32_bf16(self.gram_ft[:npad].reshape(-1), self.gram_xt[:npad].reshape(-1))
                return
        self._gram_features(T_.Xn, self.gram_ft, self.gram_xt, self.gram_nrm_t)

    def _gram_loss_bwd(self, dXn):
        """loss/gram_loss.py:38-50 on the tensor cores: St = Xt Xt^T, Ss = Xs Xs^T, elementwise negative removal + squared
        difference (d3_gram_diff; per-image blocks only with gram.img_level), dXs = (4 w / count) G Xs (G symmetric), back
        through the row normalisation, added to the gradient of the student's final-norm output."""
        n, D = self.gram_n, self.cfg.embed_dim
        if n == 0:
            return
        npad = (n + 7) // 8 * 8
        count = float(n) * float(self.gram_block) if self.gram_block else float(n) * float(n)   # entries under the mean
        inv = 1.0 / count
        xs, xt = self.gram_xs[:npad], self.gram_xt[:npad]
        Ss, St = self.gram_Ss[:npad * npad].view(npad, npad), self.gram_St[:npad * npad].view(npad, npad)
        G = self.gram_G[:npad * npad].view(npad, npad)
        ops.gemm(xt, xt, St)
        ops.gemm(xs, xs, Ss)
        ops.gram_diff(Ss, St, G, self.gram_mode, inv, self.metrics[4:5], block=self.gram_block)
        ops.gemm(G, xs, self.gram_dX[:npad], b_mn=True, alpha=4.0 * self._gram_w * inv)
        if self.cfg.gram_normalized:
            ops.l2norm_bwd(self.gram_dX[:npad], self.gram_fs[:npad], self.gram_nrm_s[:npad], self.gram_dF[:npad])
            src = self.gram_dF
        else:
            src = self.gram_dX
        ops.scatter_add_rows(src, self.gram_rows, dXn, n, D)

    # ------------------------------------------------------------------------------------------------ static tables
    def _build_rows(self):
        sg, sl = self.s_sets
        ops.token_rows(None, self.rows_cls_t, self.t_sets[0].n, self.t_sets[0].P, 1, prefix=self.cfg.prefix)
        # student cls rows: global crops then local crops (local rows offset by the global part)
        rows_g = torch.arange(sg.n, dtype=torch.int32) * sg.N
        rows_l = torch.arange(sl.n, dtype=torch.int32) * sl.N + sl.row0
        self.rows_cls_s.copy_(torch.cat([rows_g, rows_l]))

    def _build_ce_tables(self):
        """Per-student-row teacher pairing and weights (loss/dino_clstoken_loss.py:66-89; train/ssl_meta_arch.py:480-525)."""
        cfg, B = self.cfg, self.B
        ng, nl = cfg.n_global, cfg.n_local
        g_terms, l_terms = ng * (ng - 1), ng * nl
        g_scale, l_scale = g_terms / (g_terms + l_terms), l_terms / (g_terms + l_terms)
        R = self.Rc
        t0 = torch.full((R,), -1, dtype=torch.int32)
        t1 = torch.full((R,), -1, dtype=torch.int32)
        wm, wg = torch.zeros(R), torch.zeros(R)
        slot = torch.zeros(R, dtype=torch.int32)
        assert ng == 2, "pair tables are written for two global crops (n_global_crops = 2, ssl_meta_arch.py:296)"
        for i in range(R):
            s, b = divmod(i, B)
            if s < ng:      # global student crop s pairs with the OTHER teacher crop (ignore_diagonal)
                t0[i] = (1 - s) * B + b
                norm = B * ng * ng - B * min(ng, ng)
                wm[i] = 1.0 / norm
                wg[i] = cfg.dino_loss_weight * g_scale / norm
                slot[i] = 1
            else:           # local student crop pairs with both teacher crops
                t0[i], t1[i] = b, B + b
                norm = B * nl * ng
                wm[i] = 1.0 / norm
                wg[i] = cfg.dino_loss_weight * l_scale / norm
                slot[i] = 0
        dev = self.device
        self.ce_dino = tuple(x.to(dev) for x in (t0, t1, wm, wg, slot))
        Mx = self.max_masked
        n_rows = ng * B    # masks.shape[0] (loss/ibot_patch_loss.py:67)
        self.ce_ibot = (torch.arange(Mx, dtype=torch.int32, device=dev), torch.full((Mx,), -1, dtype=torch.int32, device=dev),
                        torch.full((Mx,), 1.0 / n_rows, device=dev), torch.full((Mx,), cfg.ibot_loss_weight / n_rows, device=dev),
                        torch.full((Mx,), 3, dtype=torch.int32, device=dev))

    # ------------------------------------------------------------------------------------------------ forward pieces
    def _embed(self, st: Stream, images, masks_list, teacher: bool):
        cfg, bb = self.cfg, self.params.mods["backbone"]
        self.fsdp.acquire("backbone", "embed", teacher)
        X0 = st.x_in(0)
        Wpe = bb.w("patch_embed/proj/kernel", teacher)
        for cs, img, masks in zip(st.sets, images, masks_list):
            ops.im2col(img, cs.patches, cfg.patch)
            ops.gemm(cs.patches, Wpe, cs.tok, b_mn=True, bias=bb.vec("patch_embed/proj/bias", teacher))
            ops.assemble_tokens(cs.tok, bb.vec("cls_token", teacher), bb.vec("mask_token", teacher), masks,
                                X0[cs.row0: cs.row0 + cs.T], cs.n, cs.P, cfg.embed_dim,
                                storage=bb.vec("storage_tokens", teacher) if cfg.n_storage else None)

    def _block_fwd(self, st: Stream, i: int, teacher: bool):
        cfg, bb = self.cfg, self.params.mods["backbone"]
        D, H = cfg.embed_dim, cfg.heads
        self.fsdp.acquire("backbone", f"blocks_{i}", teacher)
        p = f"blocks_{i}/"
        v = lambda n: bb.vec(p + n, teacher)
        w = lambda n: bb.w(p + n, teacher)
        X, Xmid, Xo = st.x_in(i), st.b(st.Xmid, i), st.x_out(i)
        Y, QKV, O, Z, Hh = st.b(st.Y, i), st.b(st.QKV, i), st.b(st.O, i), st.b(st.Z, i), st.b(st.Hh, i)
        stats = st.b(st.stats, i) if st.stash else [None] * 4
        ops.layernorm_fwd(X, v("norm1/scale"), v("norm1/bias"), Y, stats[0], stats[1], cfg.ln_eps)
        ops.gemm(Y, w("attn/qkv/kernel"), QKV, b_mn=True, bias=v("attn/qkv/bias"))
        lses = st.b(st.LSE, i)
        for cs, lse in zip(st.sets, lses):
            q = QKV[cs.row0: cs.row0 + cs.T]
            ops.rope(q, cs.sin, cs.cos, cs.N, cfg.prefix, D, cfg.head_dim)
            ops.attn_fwd(q, O[cs.row0: cs.row0 + cs.T], lse if st.stash else None, cs.n, cs.N, D, H)
        ops.gemm(O, w("attn/proj/kernel"), Xmid, b_mn=True, bias=v("attn/proj/bias"), gamma=v("ls1/gamma"), resid=X)
        ops.layernorm_fwd(Xmid, v("norm2/scale"), v("norm2/bias"), Z, stats[2], stats[3], cfg.ln_eps)
        if cfg.ffn_layer == "swiglu":
            # SwiGLUFFN (layers/ffn_layers.py:71-76): h = silu(z W1 + b1) * (z W2 + b2); x_out = x_mid + g2 * (h W3 + b3)
            Hs = cfg.swiglu_hidden
            X12 = st.b(st.U1, i) if st.stash else st.X12
            ops.gemm(Z, w("mlp/w1/kernel"), X12[:, :Hs], b_mn=True, bias=v("mlp/w1/bias"))
            ops.gemm(Z, w("mlp/w2/kernel"), X12[:, Hs:], b_mn=True, bias=v("mlp/w2/bias"))
            ops.swiglu_fwd(X12, Hh)
            ops.gemm(Hh, w("mlp/w3/kernel"), Xo, b_mn=True, bias=v("mlp/w3/bias"),
                     store_pre=st.b(st.U2, i) if st.stash else None, gamma=v("ls2/gamma"), resid=Xmid)
            return
        ops.gemm(Z, w("mlp/Dense_0/kernel"), Hh, b_mn=True, bias=v("mlp/Dense_0/bias"), gelu=True,
                 store_pre=st.b(st.U1, i) if st.stash else None)
        ops.gemm(Hh, w("mlp/Dense_1/kernel"), Xo, b_mn=True, bias=v("mlp/Dense_1/bias"), gelu=cfg.mlp_second_act,
                 store_pre=st.b(st.U2, i) if st.stash else None, gamma=v("ls2/gamma"), resid=Xmid)

    def _backbone_fwd(self, st: Stream, images, masks_list, teacher: bool):
        cfg, bb = self.cfg, self.params.mods["backbone"]
        self._embed(st, images, masks_list, teacher)
        for i in range(cfg.depth):
            self._block_fwd(st, i, teacher)
        XL = st.x_in(cfg.depth)
        self.fsdp.acquire("backbone", "norm", teacher)
        fs = st.fstats if st.stash else [None, None]
        ops.layernorm_fwd(XL, bb.vec("norm/scale", teacher), bb.vec("norm/bias", teacher), st.Xn, fs[0], fs[1], cfg.ln_eps)

    def _head_fwd(self, hb: HeadBufs, module: str, R: int, teacher: bool, stash: bool):
        hd = self.params.mods[module]
        w = lambda n: hd.w(n, teacher)
        v = lambda n: hd.vec(n, teacher)
        r = lambda t: t[:R]
        self.fsdp.acquire(module, "head", teacher)
        if R == 0:
            return
        ops.gemm(r(hb.A0), w("mlp/layers_0/kernel"), r(hb.H1), b_mn=True, bias=v("mlp/layers_0/bias"), gelu=True,
                 store_pre=r(hb.Ua) if stash else None)
        ops.gemm(r(hb.H1), w("mlp/layers_2/kernel"), r(hb.H2), b_mn=True, bias=v("mlp/layers_2/bias"), gelu=True,
                 store_pre=r(hb.Ub) if stash else None)
        ops.gemm(r(hb.H2), w("mlp/layers_4/kernel"), r(hb.U3), b_mn=True, bias=v("mlp/layers_4/bias"))
        ops.l2norm_fwd(r(hb.U3), r(hb.Yn), r(hb.nrm), 1e-12)
        ops.gemm(r(hb.Yn), w("last_layer/kernel"), r(hb.logits), b_mn=True)

    def _sinkhorn_pair(self, R_d: int, R_i: int, temp: float, n_iter: int = 3):
        """Both heads' Sinkhorn-Knopp normalisations (DINO cls logits, iBOT masked-patch logits) in lock step: the
        column maxima of the two heads share one all-reduce(max), and each iteration's column sums — with the two row
        totals B riding in the same buffer — one all-reduce(sum): 4 collectives per step instead of 10 (each is latency,
        not bandwidth: 2 x 256 KB).  With NVLink peer memory available the all-reduce is d3_allreduce_peers on inputs
        staged in symmetric memory (FsdpRuntime.small_allreduce), otherwise NCCL."""
        K = self.cfg.n_prototypes
        heads = [(0, self.sk_dino, self.h_t_dino.logits[:R_d], R_d)]
        if R_i:
            heads.append((1, self.sk_ibot, self.h_t_ibot.logits[:R_i], R_i))
        if getattr(self, "_sk_rows", None) != (R_d, R_i):       # local row counts: device copy refreshed when M changes
            self.sk_btot_local[0:1].fill_(float(R_d))
            self.sk_btot_local[1:2].fill_(float(R_i))
            self._sk_rows = (R_d, R_i)
        stage = self._ar_stage                                   # symmetric staging: [mx 2K | s 2K+4 | s 2K+4 | sumsq 4]
        mx_in = stage[:2 * K] if stage is not None else self.sk_mx2
        mx_in.fill_(float("-inf"))
        for slot, sk, L, R in heads:
            ops.colmax(L, mx_in[slot * K:(slot + 1) * K])
        if stage is not None:
            self.fsdp.small_allreduce(0, 2 * K, self.sk_mx2, "max")
        elif self.comm is not None:
            self.comm.all_reduce_max(self.sk_mx2)
        a = [None, None]
        for it in range(n_iter):
            # staged inputs alternate between two buffers: a peer may still be reading the previous iteration's
            off = 2 * K + (it & 1) * (2 * K + 4)
            s_in = stage[off:off + 2 * K + 4] if stage is not None else self.sk_s2
            s_in.zero_()
            s_in[2 * K:].copy_(self.sk_btot_local)
            for slot, sk, L, R in heads:
                ops.sinkhorn_colsum(L, sk.mx, temp, a[slot], s_in[slot * K:(slot + 1) * K])
            if stage is not None:
                self.fsdp.small_allreduce(off, 2 * K + 4, self.sk_s2, "sum")   # psum of the row sums (:53 / ibot :99), of B
            elif self.comm is not None:
                self.comm.all_reduce_sum(self.sk_s2)
            for slot, sk, L, R in heads:
                ops.sinkhorn_rowsum(L, sk.mx, temp, sk.s, sk.btot, sk.a[:R])
                a[slot] = sk.a[:R]

    def _softmax_center(self, sk: SinkhornBufs, center, logits, R: int, temp: float, rows_local: float):
        """softmax((x - center)/temp) after the center EMA update (loss/dino_clstoken_loss.py:24-33,91-95), expressed
        through the same (mx, s, a, btot) scalings the cross-entropy kernel consumes."""
        L = logits[:R]
        sk.gmx.fill_(float("-inf"))
        sk.btot.fill_(float(rows_local))
        ops.absmax(L, sk.gmx)
        self._colsum.zero_()
        ops.colsum_f32(L, self._colsum)
        if self.comm is not None:
            self.comm.all_reduce_max(sk.gmx)
            self.comm.all_reduce_sum(sk.btot)
            self.comm.all_reduce_sum(self._colsum)        # pmean of the local centers over "dp" (:93)
        sk.mx.copy_(sk.gmx.expand_as(sk.mx))              # one global shift for every prototype (device-side broadcast)
        ops.center_update(center, self._colsum, sk.btot, self.center_momentum, temp, sk.s)
        ops.sinkhorn_rowsum(L, sk.mx, temp, sk.s, sk.btot, sk.a[:R])

    # ------------------------------------------------------------------------------------------------ backward pieces
    def _head_bwd(self, hb: HeadBufs, module: str, R: int):
        hd = self.params.mods[module]
        w, gw, gv = (lambda n: hd.w(n)), hd.gw, hd.gv
        r = lambda t: t[:R]
        if R == 0:
            self.fsdp.grads_ready(module, "head")
            return
        # prototype layer: logits = Yn Wl
        ops.gemm(r(hb.dS), w("last_layer/kernel"), r(hb.dYn))                                   # dYn = dS Wl^T
        ops.gemm(r(hb.Yn), r(hb.dS), gw("last_layer/kernel"), a_mn=True, b_mn=True, accum=True)              # dWl = Yn^T dS
        ops.l2norm_bwd(r(hb.dYn), r(hb.U3), r(hb.nrm), r(hb.dU3), 1e-12)
        ops.colsum_bf16(r(hb.dU3), gv("mlp/layers_4/bias"))
        ops.gemm(r(hb.H2), r(hb.dU3), gw("mlp/layers_4/kernel"), a_mn=True, b_mn=True, accum=True)
        ops.gemm(r(hb.dU3), w("mlp/layers_4/kernel"), r(hb.dUb), dgelu_of=r(hb.Ub))
        ops.colsum_bf16(r(hb.dUb), gv("mlp/layers_2/bias"))
        ops.gemm(r(hb.H1), r(hb.dUb), gw("mlp/layers_2/kernel"), a_mn=True, b_mn=True, accum=True)
        ops.gemm(r(hb.dUb), w("mlp/layers_2/kernel"), r(hb.dUa), dgelu_of=r(hb.Ua))
        ops.colsum_bf16(r(hb.dUa), gv("mlp/layers_0/bias"))
        ops.gemm(r(hb.A0), r(hb.dUa), gw("mlp/layers_0/kernel"), a_mn=True, b_mn=True, accum=True)
        ops.gemm(r(hb.dUa), w("mlp/layers_0/kernel"), r(hb.dA0))                                 # fp32 [R, D]
        self.fsdp.grads_ready(module, "head")

    def _ls_tail(self, i: int):
        """Arguments that make a LayerNorm backward also emit the LayerScale/activation backward of block i's MLP
        branch (x_out = x_mid + g2 * act(h W2 + b2)) from the residual gradient it produces: dU2 -> self.dU2[parity]."""
        cfg, bb, st = self.cfg, self.params.mods["backbone"], self.student
        p = f"blocks_{i}/"
        par = (i & 1) if self.wgrad_overlap else 0
        if self.wgrad_overlap and self._ev_done_live[par]:
            torch.cuda.current_stream().wait_event(self._ev_done[par])   # weight gradients of block i+2 have read dU2[par]
            self._ev_done_live[par] = False
        out_bias = "mlp/w3/bias" if self.swiglu else "mlp/Dense_1/bias"
        return dict(ls_gamma=bb.vec(p + "ls2/gamma"), ls_u=st.b(st.U2, i), ls_gelu=cfg.mlp_second_act and not self.swiglu,
                    ls_du=self.dU2[par], ls_dgamma=bb.gv(p + "ls2/gamma"), ls_dbias=bb.gv(p + out_bias))

    def _block_bwd(self, i: int, dX, dXprev):
        """Backward of block i.  On entry dX is the gradient of the block output and self.dU2[parity(i)] already holds
        dU2 = dX * g2 * act'(u2) (written by the LayerNorm backward that produced dX, see _ls_tail)."""
        cfg, bb, st = self.cfg, self.params.mods["backbone"], self.student
        D, H = cfg.embed_dim, cfg.heads
        p = f"blocks_{i}/"
        v, w, gw, gv = (lambda n: bb.vec(p + n)), (lambda n: bb.w(p + n)), (lambda n: bb.gw(p + n)), (lambda n: bb.gv(p + n))
        m1, r1, m2, r2 = st.b(st.stats, i)
        par = (i & 1) if self.wgrad_overlap else 0
        dU2, dU1, dP, dQKV = self.dU2[par], self.dU1[par], self.dP[par], self.dQKV[par]
        main = torch.cuda.current_stream()
        if self.remat:
            # recompute this block's forward from its stashed input (writes the scratch activations, statistics, LSE and
            # x_out again), then the LayerScale / activation backward of its MLP branch, which the stashing path gets
            # for free from the LayerNorm backward of the block above (_ls_tail)
            self._block_fwd(st, i, teacher=False)
            t = self._ls_tail(i)
            ops.ls_act_bwd(dX, t["ls_u"], t["ls_gamma"], t["ls_du"], t["ls_dgamma"], t["ls_dbias"], t["ls_gelu"])

        def on_wstream(slot, fn):
            """Run fn on the weight-gradient stream once the main stream has reached this point."""
            if not self.wgrad_overlap:
                fn()
                return
            ev = self._ev_in[par][slot]
            ev.record(main)
            self.wstream.wait_event(ev)
            with torch.cuda.stream(self.wstream):
                fn()

        # multi-GPU: the three large weight gradients are reduce-scattered by the GEMM epilogue itself (each tile is
        # added into the owning rank's gradient shard over NVLink); the rest of the unit is pushed in grads_ready
        big = ("mlp/w3/kernel", "mlp/w1/kernel", "mlp/w2/kernel", "attn/qkv/kernel") if self.swiglu else \
              ("mlp/Dense_1/kernel", "mlp/Dense_0/kernel", "attn/qkv/kernel")
        fused = big if (self.fsdp.push and self.fsdp.push_gemm) else ()
        inv_world = 1.0 / self.fsdp.world

        def wgrad(slot, a, b, name):
            spec = self.fsdp.scatter_spec("backbone", f"blocks_{i}", p + name) if name in fused else None
            on_wstream(slot, lambda: ops.gemm(a, b, gw(name), a_mn=True, b_mn=True, accum=True, scatter=spec,
                                              alpha=inv_world if spec else 1.0))
        # ---- MLP branch: x_out = x_mid + g2 * act(u2), u2 = h W2 + b2, h = gelu(u1), u1 = z W1 + b1
        if self.swiglu:
            # x_out = x_mid + g2 * (h W3 + b3), h = silu(x1) * x2, x1 = z W1 + b1, x2 = z W2 + b2
            Hs = cfg.swiglu_hidden
            X12, dX12 = st.b(st.U1, i), dU1
            wgrad(0, st.b(st.Hh, i), dU2, "mlp/w3/kernel")                                           # dW3 = h^T dU2
            ops.gemm(dU2, w("mlp/w3/kernel"), self.dH)                                         # dh = dU2 W3^T
            ops.swiglu_bwd(X12, self.dH, dX12)                                                 # [dx1 | dx2]
            wgrad(1, st.b(st.Z, i), dX12[:, :Hs], "mlp/w1/kernel")                                   # dW1 = z^T dx1
            wgrad(1, st.b(st.Z, i), dX12[:, Hs:], "mlp/w2/kernel")                                   # dW2 = z^T dx2
            on_wstream(1, lambda: (ops.colsum_bf16(dX12[:, :Hs], gv("mlp/w1/bias")), ops.colsum_bf16(dX12[:, Hs:], gv("mlp/w2/bias"))))
            ops.gemm(dX12[:, :Hs], w("mlp/w1/kernel"), self.dZ32)                              # dz = dx1 W1^T + dx2 W2^T (fp32)
            ops.gemm(dX12[:, Hs:], w("mlp/w2/kernel"), self.dZ32, accum=True)
            dZ = self.dZ32
        else:
            wgrad(0, st.b(st.Hh, i), dU2, "mlp/Dense_1/kernel")                                      # dW2 = h^T dU2
            ops.gemm(dU2, w("mlp/Dense_1/kernel"), dU1, dgelu_of=st.b(st.U1, i))                     # dU1 = (dU2 W2^T) * gelu'(u1)
            wgrad(1, st.b(st.Z, i), dU1, "mlp/Dense_0/kernel")                                       # dW1 = z^T dU1
            # bias gradients are column sums that only feed the optimizer: they ride on the weight-gradient stream
            on_wstream(1, lambda: ops.colsum_bf16(dU1, gv("mlp/Dense_0/bias")))
            ops.gemm(dU1, w("mlp/Dense_0/kernel"), self.dZ)                                    # dZ = dU1 W1^T
            dZ = self.dZ
        # LN2 backward; its tail is the attention branch's LayerScale: x_mid = x_in + g1 * (o Wp + bp), dP = dXmid * g1
        ops.layernorm_bwd_ls(dZ, st.b(st.Xmid, i), m2, r2, v("norm2/scale"), self.dXmid, dx_add=dX,
                             dscale=gv("norm2/scale"), dbias=gv("norm2/bias"),
                             ls_gamma=v("ls1/gamma"), ls_du=dP, ls_dbias=gv("attn/proj/bias"))

        def proj_wgrad():
            ops.gemm(st.b(st.O, i), dP, gw("attn/proj/kernel"), a_mn=True, b_mn=True, accum=True)    # dWp = o^T dP
            # dg1 from dWp / dbp (no stash of the projection output needed)
            ops.ls_gamma_from_wgrad(w("attn/proj/kernel"), gw("attn/proj/kernel"), v("attn/proj/bias"),
                                    gv("attn/proj/bias"), v("ls1/gamma"), gv("ls1/gamma"))
        on_wstream(2, proj_wgrad)
        ops.gemm(dP, w("attn/proj/kernel"), self.dO)                                           # dO = dP Wp^T
        for cs, lse, delta in zip(st.sets, st.b(st.LSE, i), self.delta):
            sl = slice(cs.row0, cs.row0 + cs.T)
            # gradient w.r.t. the pre-RoPE projection: the inverse rotation is fused into the kernel's store stage
            ops.attn_bwd(st.b(st.QKV, i)[sl], st.b(st.O, i)[sl], self.dO[sl], lse, delta, dQKV[sl], cs.n, cs.N, D, H,
                         rope_sin=cs.sin, rope_cos=cs.cos, rope_prefix=cfg.prefix)
        wgrad(3, st.b(st.Y, i), dQKV, "attn/qkv/kernel")                                             # dWqkv = y^T dQKV

        def qkv_bias_grad():
            if cfg.mask_k_bias:      # LinearKMaskedBias: no gradient reaches the k third of the bias
                gb = gv("attn/qkv/bias")
                ops.colsum_bf16(dQKV[:, :D], gb[:D])
                ops.colsum_bf16(dQKV[:, 2 * D:], gb[2 * D:])
            else:
                ops.colsum_bf16(dQKV, gv("attn/qkv/bias"))
        on_wstream(3, qkv_bias_grad)
        ops.gemm(dQKV, w("attn/qkv/kernel"), self.dY)                                          # dY = dQKV Wqkv^T
        tail = self._ls_tail(i - 1) if (i > 0 and not self.remat) else {}
        ops.layernorm_bwd_ls(self.dY, st.X[i], m1, r1, v("norm1/scale"), dXprev, dx_add=self.dXmid,
                             dscale=gv("norm1/scale"), dbias=gv("norm1/bias"), **tail)
        scattered = tuple(p + n for n in fused)
        if self.wgrad_overlap:
            if self.fsdp.push:
                # the remaining ranges are pushed from the weight-gradient stream, after the main stream's last
                # contribution to this unit (the LayerNorm backward above)
                on_wstream(0, lambda: self.fsdp.grads_ready("backbone", f"blocks_{i}", scattered=scattered))
                self._ev_done[par].record(self.wstream)
            else:
                self._ev_done[par].record(self.wstream)
                self.fsdp.grads_ready("backbone", f"blocks_{i}", also_after=self._ev_done[par])
            self._ev_done_live[par] = True
        else:
            self.fsdp.grads_ready("backbone", f"blocks_{i}", scattered=scattered)

    def _gather_schedule(self):
        """(module, unit, teacher) in the order the step uses them: teacher pass, then student pass (student parameters
        stay gathered for the backward: SHARD_GRAD_OP, ssl_default_config.yaml:19)."""
        items = []
        for teacher in (True, False):
            bb = self.params.mods["backbone"].layout
            items += [("backbone", u, teacher) for u in bb.units]
            for m in (("dino_head", "ibot_head") if teacher else ("dino_head", "ibot_head")):
                items += [(m, u, teacher) for u in self.params.mods[m].layout.units]
        return items

    # ------------------------------------------------------------------------------------------------ the step
    def set_batch(self, batch: dict):
        """Accepts the reference's collate dict (data/collate.py:72-93): crop-major NHWC bf16 crops, bool masks
        [2B, P], int64 mask_indices_list [M].  Device tensors are used as they are; host tensors are copied
        (pinned + non_blocking when possible)."""
        dev = self.device
        to = lambda t, dt=None: t.to(device=dev, dtype=dt, non_blocking=True)
        self.g_img = to(batch["collated_global_crops"], bf16).contiguous()
        self.l_img = to(batch["collated_local_crops"], bf16).contiguous()
        if self.gram_stream is not None and batch.get("collated_gram_teacher_crops", None) is not None:
            self.gram_img = to(batch["collated_gram_teacher_crops"], bf16).contiguous()
        masks = batch["collated_masks"]
        self.masks_u8.copy_(masks.to(torch.uint8) if masks.dtype != torch.uint8 else masks, non_blocking=True)
        idx = batch["mask_indices_list"]
        self.M = int(idx.shape[0])
        assert self.M <= self.max_masked, f"M={self.M} exceeds max_masked={self.max_masked}"
        self.mask_idx[: self.M].copy_(idx, non_blocking=True)
        ops.token_rows(self.mask_idx, self.rows_masked_t, self.M, self.s_sets[0].P, 0, prefix=self.cfg.prefix)
        if self.cfg.gram_use_loss and self.cfg.gram_tokens_used != "all":
            # gram.tokens_used (train/ssl_meta_arch.py:221-223; upstream: student_patches[masks] / [~masks])
            n_all = self.gram_rows_all.numel()
            if self.cfg.gram_tokens_used == "masked":
                self.gram_rows, self.gram_n = self.rows_masked_t, self.M
            else:
                # stable sort of the mask bits: unmasked patch positions first, in order (no host sync, count known)
                order = torch.argsort(self.masks_u8.reshape(-1).to(torch.int16), stable=True)[: n_all - self.M]
                self.gram_rows, self.gram_n = self.gram_rows_all[order].contiguous(), n_all - self.M

    def forward_backward(self, teacher_temp: float):
        cfg, B, M = self.cfg, self.B, self.M
        D, K = cfg.embed_dim, cfg.n_prototypes
        ng = cfg.n_global * B
        self.metrics.zero_()
        for st in self.params.mods.values():
            st.zero_grads()
        self.fsdp.begin_step()
        self.fsdp.prefetch(self._gather_schedule())
        # ---- teacher (train/ssl_meta_arch.py:366-402).  It shares nothing with the student pass until the losses, so
        # it runs on its own stream: the HBM-bound kernels of one pass overlap the tensor-bound kernels of the other.
        T_ = self.teacher

        def teacher_pass():
            self._backbone_fwd(T_, [self.g_img], [None], teacher=True)
            ops.gather_rows(T_.Xn, self.rows_cls_t, ng, D, dst_bf16=self.h_t_dino.A0)
            ops.gather_rows(T_.Xn, self.rows_masked_t, M, D, dst_bf16=self.h_t_ibot.A0)
            self._head_fwd(self.h_t_dino, "dino_head", ng, teacher=True, stash=False)
            self._head_fwd(self.h_t_ibot, "ibot_head", M, teacher=True, stash=False)
            if self.centering == "sinkhorn_knopp":
                self._sinkhorn_pair(ng, M, teacher_temp)
            else:
                self._softmax_center(self.sk_dino, self.center_dino, self.h_t_dino.logits, ng, teacher_temp, ng)
                self._softmax_center(self.sk_ibot, self.center_ibot, self.h_t_ibot.logits, M, teacher_temp, M)
            if cfg.gram_use_loss:
                self._gram_teacher_targets()

        if self.fwd_overlap:
            main = torch.cuda.current_stream()
            self._ev_fwd[0].record(main)
            self.tstream.wait_event(self._ev_fwd[0])          # batch, zeroed metrics, parameters of the last update
            with torch.cuda.stream(self.tstream):
                teacher_pass()
                self._ev_fwd[1].record(self.tstream)
        else:
            teacher_pass()
        # ---- student (train/ssl_meta_arch.py:406-460)
        S_ = self.student
        self._backbone_fwd(S_, [self.g_img, self.l_img], [self.masks_u8, None], teacher=False)
        ops.gather_rows(S_.Xn, self.rows_cls_s, self.Rc, D, dst_bf16=self.h_s_dino.A0, dst_f32=self.cls_f32)
        ops.gather_rows(S_.Xn, self.rows_masked_t, M, D, dst_bf16=self.h_s_ibot.A0)
        if self.gram_active:
            self._gram_features(S_.Xn, self.gram_fs, self.gram_xs, self.gram_nrm_s)
        self._head_fwd(self.h_s_dino, "dino_head", self.Rc, teacher=False, stash=True)
        self._head_fwd(self.h_s_ibot, "ibot_head", M, teacher=False, stash=True)
        # ---- losses + d(logits) (train/ssl_meta_arch.py:463-525)
        if self.fwd_overlap:
            torch.cuda.current_stream().wait_event(self._ev_fwd[1])      # teacher targets ready
        t0, t1, wm, wg, slot = self.ce_dino
        ops.ce_fwd_bwd(self.h_s_dino.logits, cfg.student_temp, self.h_t_dino.logits, self.sk_dino.mx, teacher_temp,
                       self.sk_dino.s, self.sk_dino.a, self.sk_dino.btot, t0, t1, wm, wg, slot, self.metrics,
                       self.h_s_dino.dS)
        if M:
            t0, t1, wm, wg, slot = self.ce_ibot
            ops.ce_fwd_bwd(self.h_s_ibot.logits[:M], cfg.student_temp, self.h_t_ibot.logits[:M], self.sk_ibot.mx,
                           teacher_temp, self.sk_ibot.s, self.sk_ibot.a, self.sk_ibot.btot, t0, t1, wm, wg, slot,
                           self.metrics, self.h_s_ibot.dS[:M])
        # ---- backward: heads
        self._head_bwd(self.h_s_dino, "dino_head", self.Rc)
        self._head_bwd(self.h_s_ibot, "ibot_head", M)
        # KoLeo on the pre-head global cls tokens, per crop (train/ssl_meta_arch.py:513): loss weight
        # koleo_loss_weight * n_global * (1/n_global) per crop; metric = mean over crops
        for c in range(cfg.n_global):
            ops.koleo_fwd_bwd(self.cls_f32[c * B:(c + 1) * B], self.koleo_xn, self.koleo_nrm, self.koleo_nn,
                              self.koleo_coef, self.metrics[2:3], self.h_s_dino.dA0[c * B:(c + 1) * B],
                              1.0 / cfg.n_global, cfg.koleo_loss_weight)
        # ---- backward: final norm (dXn is zero except cls rows and masked-patch rows)
        dXn = self.dX[0]
        dXn.zero_()
        ops.scatter_add_rows(self.h_s_dino.dA0, self.rows_cls_s, dXn, self.Rc, D)
        ops.scatter_add_rows(self.h_s_ibot.dA0, self.rows_masked_t, dXn, M, D)
        if self.gram_active:
            self._gram_loss_bwd(dXn)
        bb = self.params.mods["backbone"]
        dXL = self.dX[1]
        ops.layernorm_bwd_ls(dXn, S_.X[cfg.depth], S_.fstats[0], S_.fstats[1], bb.vec("norm/scale"), dXL,
                             dscale=bb.gv("norm/scale"), dbias=bb.gv("norm/bias"),
                             **({} if self.remat else self._ls_tail(cfg.depth - 1)))
        self.fsdp.grads_ready("backbone", "norm")
        cur, nxt = 1, 0
        for i in reversed(range(cfg.depth)):
            self._block_bwd(i, self.dX[cur], self.dX[nxt])
            cur, nxt = nxt, cur
        # ---- backward: token assembly + patch embedding
        dX0 = self.dX[cur]
        first = True
        for cs, masks, dTok in zip(S_.sets, [self.masks_u8, None], self.dTok):
            ops.assemble_tokens_bwd(dX0[cs.row0: cs.row0 + cs.T], masks, dTok, bb.gv("cls_token"),
                                    bb.gv("mask_token"), cs.n, cs.P, D,
                                    dstorage=bb.gv("storage_tokens") if cfg.n_storage else None)
            ops.colsum_bf16(dTok, bb.gv("patch_embed/proj/bias"))
            ops.gemm(cs.patches, dTok, bb.gw("patch_embed/proj/kernel"), a_mn=True, b_mn=True, accum=True)
            first = False
        self.fsdp.grads_ready("backbone", "embed")
        if self.wgrad_overlap:
            torch.cuda.current_stream().wait_stream(self.wstream)     # the optimizer reads every weight gradient
            self._ev_done_live = [False, False]

    def optimizer_step(self, lr: float, wd: float, last_layer_lr: float, momentum: float):
        """Per-module clip (train/train.py:516-541) + AdamW (:95-106) + teacher EMA (ssl_meta_arch.py:650-652)."""
        cfg = self.cfg
        self.step_count += 1
        self.fsdp.finish_grads()
        # global gradient norm per module (SURVEY A4): sum over ranks of the shards' squares; the modules' scalars are
        # views of one buffer, so the cross-rank sum is one reduction
        if self._ar_stage is not None:
            K = cfg.n_prototypes
            off = 2 * K + 2 * (2 * K + 4)
            sq_in = self._ar_stage[off:off + 4]
            sq_in.zero_()
            for i, st in enumerate(self.params.mods.values()):
                ops.sumsq(st.grad_shard, sq_in[i:i + 1])
            self.fsdp.small_allreduce(off, len(self.params.mods), self._sumsq_all, "sum")
        else:
            for st in self.params.mods.values():
                ops.sumsq(st.grad_shard, st.sumsq)
            if self.comm is not None:
                self.comm.all_reduce_sum(self._sumsq_all)
        for st in self.params.mods.values():
            ops.adamw_ema(st.master, st.grad_shard, st.m, st.v, st.t_master, st.bf16_shard, st.t_bf16_shard,
                          st.layout.n_mat_shard, st.segs, st.nseg, st.sumsq, float(cfg.clip_grad or 0.0), lr,
                          last_layer_lr, wd, self.step_count, momentum, cfg.adamw_beta1, cfg.adamw_beta2)

    def ema_update(self, momentum: float):
        """Stand-alone teacher EMA (train/ssl_meta_arch.py:644-660) for callers that keep the reference's two-call
        step: `optimizer_step(..., momentum=1.0)` leaves the teacher untouched, then this applies the EMA."""
        for st in self.params.mods.values():
            ops.ema(st.t_master, st.master, st.t_bf16_shard, st.layout.n_mat_shard, float(momentum))

    def train_step(self, batch: dict | None, *, teacher_temp: float, lr: float, wd: float, last_layer_lr: float,
                   momentum: float, gram_loss_weight: float | None = None, iteration: int | None = None):
        if batch is not None:
            self.set_batch(batch)
        if self.cfg.gram_use_loss:
            if gram_loss_weight is not None:       # gram.loss_weight_schedule[iteration] (train/ssl_meta_arch.py:534-537)
                self._gram_w = float(gram_loss_weight)
            self.gram_schedule(self.step_count if iteration is None else int(iteration))
        self.forward_backward(teacher_temp)
        self.optimizer_step(lr, wd, last_layer_lr, momentum)

    # ------------------------------------------------------------------------------------------------ results
    def read_metrics(self) -> dict:
        """Device -> host read of the step's metrics (one small sync; callers do it every print_freq, not every step)."""
        cfg = self.cfg
        if self.comm is not None:       # pmean of the loss terms over "dp" (train/ssl_meta_arch.py:361, train/train.py:554-557)
            mt = self.metrics.clone()
            self.comm.all_reduce_mean(mt)
            m = mt.cpu().tolist()
        else:
            m = self.metrics.cpu().tolist()
        ng, nl = cfg.n_global, cfg.n_local
        g_terms, l_terms = ng * (ng - 1), ng * nl
        g_scale, l_scale = g_terms / (g_terms + l_terms), l_terms / (g_terms + l_terms)
        loss = (cfg.dino_loss_weight * l_scale * m[0] + cfg.dino_loss_weight * g_scale * m[1]
                + cfg.koleo_loss_weight * ng * m[2] + cfg.ibot_loss_weight * m[3])
        out = {"dino_local_crops_loss": m[0], "dino_local_loss_weight": 1.0, "dino_global_crops_loss": m[1],
               "koleo_loss": m[2], "ibot_loss": m[3], "local_batch_size": float(self.B)}
        if self.gram_active:                       # train/ssl_meta_arch.py:538-541
            loss += self._gram_w * m[4]
            out["gram_loss"], out["gram_loss_weight"] = m[4], self._gram_w
        out["total_loss"] = loss
        for name, st in self.params.mods.items():
            out[f"student_{name}_grad_norm"] = math.sqrt(max(st.sumsq.item(), 0.0))
        return out
