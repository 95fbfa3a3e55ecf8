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
from .forward import CropSet, HeadBufs, Net, Stream, backbone_fwd, block_fwd, dgrad, head_fwd
from .forward import rope_tables  # noqa: F401  (engine.core.rope_tables stays importable for existing callers)
from .gram import GramAnchor
from .losses import SinkhornBufs, SmallReduce, sinkhorn, softmax_center
from .params import FrozenStore, ParamStore, backbone_spec, head_spec

f32, bf16 = torch.float32, torch.bfloat16


class Engine:
    """One rank's training engine: parameters, buffers and the step.

    `B` = images per rank.  The number of masked tokens M varies per batch; buffers are sized for `max_masked`
    (default: the collate upper bound, data/collate.py:47-61) and the live M comes from `mask_indices_list`.
    """

    def __init__(self, cfg: EngineConfig, B: int, device="cuda", max_masked: int | None = None, comm=None,
                 centering: str = "sinkhorn_knopp", center_momentum: float = 0.9, remat: bool = False,
                 distill: EngineConfig | None = None, fp8: bool = False):
        """`distill`: the configuration of a frozen teacher of another architecture (distillation.enabled,
        train/ssl_meta_arch.py:257-286).  It replaces the EMA teacher in the forward; the EMA of the student is still
        kept in the teacher_* buffers.  Its weights come from `distill_teacher_load`.
        `fp8` (student.fp8_enabled, fp8_filter: blocks): the block linears (qkv, proj, fc1 / fc2 or w1 / w2 / w3) of
        every backbone the step runs compute their forward and input gradients in e4m3 with row-wise power-of-two
        scales (d3_gemm_e4m3); their weight gradients stay bf16.  The heads, patch embedding and attention stay bf16."""
        for c in (cfg, distill):
            if c is not None:
                assert c.head_dim in (64, 128), "attention kernels exist for head_dim 64 (ViT-S ... giant2) and 128 (vit_7b)"
        if not cfg.qkv_bias:
            raise NotImplementedError("a trained model without a qkv bias: qkv_bias=false is supported for a frozen "
                                      "distillation teacher only")
        if distill is not None:
            if comm is not None:
                raise NotImplementedError("distillation on more than one GPU")
            if cfg.gram_use_loss:
                raise NotImplementedError("distillation together with Gram anchoring")
            if (distill.patch, distill.n_prototypes, distill.head_dims("ibot_head")[2]) != \
                    (cfg.patch, cfg.n_prototypes, cfg.head_dims("ibot_head")[2]):
                raise ValueError("the distillation teacher needs the student's patch size and prototype counts "
                                 "(train/ssl_meta_arch.py:264-267)")
        if cfg.embed_dim > 1536:
            raise NotImplementedError(f"embed_dim {cfg.embed_dim}: the LayerNorm backward (d3_layernorm_bwd_ls) takes rows of "
                                      "at most 1536 columns, so training stops at ViT-giant2 width; vit_7b (4096) runs "
                                      "forward through dinov3_jax.models.DinoVisionTransformer")
        if fp8:
            for c in (cfg, distill):
                if c is not None and (c.embed_dim % 16 or c.ffn_width % 16):
                    raise NotImplementedError(f"fp8: the e4m3 GEMM contracts over multiples of 16; embed_dim "
                                              f"{c.embed_dim} / ffn width {c.ffn_width} is not")
        self.fp8 = bool(fp8)
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
        self.distill = distill
        self.student_net = Net(cfg, self.params.mods, False, self.fsdp, fp8=self.fp8)
        if distill is None:
            self.t_net = Net(cfg, self.params.mods, True, self.fsdp, fp8=self.fp8)
        else:
            self.t_net = Net(distill, {"backbone": FrozenStore(backbone_spec(distill), dev),
                                       "dino_head": FrozenStore(head_spec(distill, "dino_head"), dev),
                                       "ibot_head": FrozenStore(head_spec(distill, "ibot_head"), dev)}, True, fp8=self.fp8)
        tcfg = self.t_net.cfg
        ng, nl = cfg.n_global * B, cfg.n_local * B
        # teacher stream: global crops only (at the teacher's width); student stream: global then local rows
        gp, lp = cfg.global_size // cfg.patch, cfg.local_size // cfg.patch
        self.t_sets = [CropSet(tcfg, ng, gp, gp, 0, dev)]
        self.s_sets = [CropSet(cfg, ng, gp, gp, 0, dev)]
        self.s_sets.append(CropSet(cfg, nl, lp, lp, self.s_sets[0].T, dev))
        self.teacher = Stream(tcfg, self.t_sets, dev, stash=False)
        self.student = Stream(cfg, self.s_sets, dev, stash=True, remat=self.remat, fp8=self.fp8)
        P = self.s_sets[0].P
        if max_masked is None:
            n_masked_crops = int(ng * cfg.mask_probability)
            max_masked = sum(int(P * (cfg.mask_ratio[0] + (cfg.mask_ratio[1] - cfg.mask_ratio[0]) * (i + 1) /
                                      max(n_masked_crops, 1))) for i in range(n_masked_crops)) + 8
        self.max_masked = max(int(max_masked), 1)
        D = cfg.embed_dim
        Kd, Ki = cfg.head_dims("dino_head")[2], cfg.head_dims("ibot_head")[2]
        Ks = Kd + Ki
        self.Rc = ng + nl                         # student dino-head rows: concat(g_cls, l_cls)
        self.h_s_dino = HeadBufs(cfg, "dino_head", self.Rc, dev, stash=True)
        self.h_s_ibot = HeadBufs(cfg, "ibot_head", self.max_masked, dev, stash=True)
        self.h_t_dino = HeadBufs(tcfg, "dino_head", ng, dev, stash=False)
        self.h_t_ibot = HeadBufs(tcfg, "ibot_head", self.max_masked, dev, stash=False)
        # each Sinkhorn stage reduces both heads at once (4 collectives per step instead of 10): [K_d | K_i] in sk_mx2
        self.sk_dino, self.sk_ibot = SinkhornBufs.joint([(ng, Kd), (self.max_masked, Ki)], dev)
        self.sk_mx2 = self.sk_dino.shared["mx"]
        self.reduce = SmallReduce(comm, {"max": Ks, "sum0": Ks + 4, "sum1": Ks + 4, "sumsq": len(self.params.mods)},
                                  peer=self.fsdp.push, device=dev)
        # centers of the optional softmax-centering path ("state" collection of the reference: dino_clstoken_loss.py:19-22)
        self.center_dino = torch.zeros(Kd, dtype=f32, device=dev)
        self.center_ibot = torch.zeros(Ki, dtype=f32, device=dev)
        i32 = torch.int32
        self.rows_masked_t = torch.empty(self.max_masked, dtype=i32, device=dev)
        # the masked patches' rows in the teacher stream (another prefix when a distillation teacher has other storage tokens)
        self.rows_masked_tt = self.rows_masked_t if distill is None else torch.empty(self.max_masked, dtype=i32, device=dev)
        self.rows_cls_t = torch.empty(ng, dtype=i32, device=dev)
        self.rows_cls_s = torch.empty(self.Rc, dtype=i32, device=dev)
        self.cls_f32 = torch.empty(self.Rc, D, dtype=f32, device=dev)     # student cls rows (fp32) for KoLeo
        self.dcls = torch.empty(self.Rc, D, dtype=f32, device=dev)
        self.koleo_xn = torch.empty(B, D, dtype=f32, device=dev)
        self.koleo_nrm = torch.empty(B, dtype=f32, device=dev)
        self.koleo_nn = torch.empty(B, dtype=i32, device=dev)
        self.koleo_coef = torch.empty(B, dtype=f32, device=dev)
        if cfg.koleo_distributed:
            from .koleo import DistributedKoLeo
            self.koleo_dist = DistributedKoLeo(comm, B, D, cfg.n_global, cfg.koleo_topk, cfg.koleo_group_size, dev)
        elif cfg.koleo_topk != 1:
            raise ValueError("koleo_topk > 1 needs koleo_distributed (train/ssl_meta_arch.py:105)")
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
        self.wgrad_overlap = not self.remat
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
        # dino.reweight_dino_local_loss: the local rows' CE gradient weights are base * w (train_step sets w)
        self.dino_local_loss_weight = 1.0
        self._wg_local = self.ce_dino[3][ng:].clone()
        self._build_rows()
        self.step_count = 0
        self._gram = g = GramAnchor(cfg, self.s_sets[0], dev, self.fp8) if cfg.gram_use_loss else None
        self.gram_net = g.net if g is not None else None                  # the frozen gram teacher (None: EMA teacher)
        self.g_sets = g.stream.sets if g is not None and g.stream is not None else None   # its own-resolution crops
        self.masks_u8 = torch.zeros(ng, P, dtype=torch.uint8, device=dev)
        self.mask_idx = torch.zeros(self.max_masked, dtype=torch.int64, device=dev)
        self.M = 0

    # ------------------------------------------------------------------------------------------------ distillation
    def distill_teacher_load(self, tree: dict):
        """Weights of the frozen distillation teacher: {"backbone", "dino_head", "ibot_head"} trees (nested dicts or
        flat '/'-joined names) with the reference's names and layouts, e.g. the teacher_* subtrees of a checkpoint.
        `attn/qkv/bias` is expected exactly when the teacher has a qkv bias."""
        if self.distill is None:
            raise ValueError("distill_teacher_load: the engine was built without a distillation teacher")
        from ..checkpointer import flat_from_tree
        for m in ("dino_head", "ibot_head"):
            if m not in tree:
                raise ValueError(f"distillation teacher without its {m}: the teacher's DINO and iBOT heads produce the "
                                 "targets, so backbone weights alone (e.g. torch-hub weights) cannot drive distillation")
        if "backbone" not in tree:
            raise ValueError("distillation teacher without its backbone")
        for m, store in self.t_net.mods.items():
            store.load(flat_from_tree(tree[m]), self.distill.mask_k_bias)

    # ------------------------------------------------------------------------------------------------ Gram anchoring
    @property
    def gram_active(self) -> bool:
        return self._gram is not None and self._gram.active

    def gram_teacher_load(self, tensors: dict):
        self._gram.teacher_load(tensors)

    def gram_schedule(self, iteration: int):
        if self._gram is not None:
            self._gram.schedule(iteration)

    def gram_state(self) -> tuple:
        return self._gram.state() if self._gram is not None else ({}, {})

    def gram_load_state(self, flat: dict, optimizer_state: dict | None):
        if self._gram is not None:
            self._gram.load_state(flat, optimizer_state)

    # ------------------------------------------------------------------------------------------------ static tables
    def _build_rows(self):
        sg, sl = self.s_sets
        ops.token_rows(None, self.rows_cls_t, self.t_sets[0].n, self.t_sets[0].P, 1, prefix=self.t_net.cfg.prefix)
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
        dg = lambda dy, n, out, **ep: dgrad(self.student_net, dy, w(n), out, **ep)   # bf16 or e4m3 (fp8)
        if self.remat:
            # recompute this block's forward from its stashed input (writes the scratch activations, statistics, LSE and
            # x_out again), then the LayerScale / activation backward of its MLP branch, which the stashing path gets
            # for free from the LayerNorm backward of the block above (_ls_tail)
            block_fwd(self.student_net, st, i)
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
        fused = big if self.fsdp.push else ()
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
            dg(dU2, "mlp/w3/kernel", self.dH)                                                  # dh = dU2 W3^T
            ops.swiglu_bwd(X12, self.dH, dX12)                                                 # [dx1 | dx2]
            wgrad(1, st.b(st.Z, i), dX12[:, :Hs], "mlp/w1/kernel")                                   # dW1 = z^T dx1
            wgrad(1, st.b(st.Z, i), dX12[:, Hs:], "mlp/w2/kernel")                                   # dW2 = z^T dx2
            on_wstream(1, lambda: (ops.colsum_bf16(dX12[:, :Hs], gv("mlp/w1/bias")), ops.colsum_bf16(dX12[:, Hs:], gv("mlp/w2/bias"))))
            dg(dX12[:, :Hs], "mlp/w1/kernel", self.dZ32)                                       # dz = dx1 W1^T + dx2 W2^T (fp32)
            dg(dX12[:, Hs:], "mlp/w2/kernel", self.dZ32, accum=True)
            dZ = self.dZ32
        else:
            wgrad(0, st.b(st.Hh, i), dU2, "mlp/Dense_1/kernel")                                      # dW2 = h^T dU2
            dg(dU2, "mlp/Dense_1/kernel", dU1, dgelu_of=st.b(st.U1, i))                              # dU1 = (dU2 W2^T) * gelu'(u1)
            wgrad(1, st.b(st.Z, i), dU1, "mlp/Dense_0/kernel")                                       # dW1 = z^T dU1
            # bias gradients are column sums that only feed the optimizer: they ride on the weight-gradient stream
            on_wstream(1, lambda: ops.colsum_bf16(dU1, gv("mlp/Dense_0/bias")))
            dg(dU1, "mlp/Dense_0/kernel", self.dZ)                                             # dZ = dU1 W1^T
            dZ = self.dZ
        # LN2 backward; its tail is the attention branch's LayerScale: x_mid = x_in + g1 * p, p = o Wp + bp, dP = dXmid * g1.
        # With fp8, p is not o Wp + bp in high precision, so dg1 = colsum(dXmid * p) comes from the stashed p.
        ls1 = dict(ls_u=st.b(st.Pa, i), ls_dgamma=gv("ls1/gamma")) if self.fp8 else {}
        ops.layernorm_bwd_ls(dZ, st.b(st.Xmid, i), m2, r2, v("norm2/scale"), self.dXmid, dx_add=dX,
                             dscale=gv("norm2/scale"), dbias=gv("norm2/bias"),
                             ls_gamma=v("ls1/gamma"), ls_du=dP, ls_dbias=gv("attn/proj/bias"), **ls1)

        def proj_wgrad():
            ops.gemm(st.b(st.O, i), dP, gw("attn/proj/kernel"), a_mn=True, b_mn=True, accum=True)    # dWp = o^T dP
            if not self.fp8:   # dg1 from dWp / dbp (no stash of the projection output needed)
                ops.ls_gamma_from_wgrad(w("attn/proj/kernel"), gw("attn/proj/kernel"), v("attn/proj/bias"),
                                        gv("attn/proj/bias"), v("ls1/gamma"), gv("ls1/gamma"))
        on_wstream(2, proj_wgrad)
        dg(dP, "attn/proj/kernel", self.dO)                                                    # dO = dP Wp^T
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
        dg(dQKV, "attn/qkv/kernel", self.dY)                                                   # dY = dQKV Wqkv^T
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
        for teacher in ((False,) if self.distill is not None else (True, False)):   # a distillation teacher is resident
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
        masks = batch["collated_masks"]
        self.masks_u8.copy_(masks.to(torch.uint8) if masks.dtype != torch.uint8 else masks, non_blocking=True)
        idx = batch["mask_indices_list"]
        self.M = int(idx.shape[0])
        assert self.M <= self.max_masked, f"M={self.M} exceeds max_masked={self.max_masked}"
        self.mask_idx[: self.M].copy_(idx, non_blocking=True)
        ops.token_rows(self.mask_idx, self.rows_masked_t, self.M, self.s_sets[0].P, 0, prefix=self.cfg.prefix)
        if self.distill is not None:
            ops.token_rows(self.mask_idx, self.rows_masked_tt, self.M, self.s_sets[0].P, 0, prefix=self.distill.prefix)
        if self._gram is not None:
            self._gram.set_batch(batch, self.rows_masked_t, self.M, self.masks_u8)

    def teacher_pass(self, teacher_temp: float):
        """Teacher forward over the global crops, its heads and the centering of its logits (train/ssl_meta_arch.py:366-402)."""
        ng, M, T_ = self.cfg.n_global * self.B, self.M, self.teacher
        Dt = self.t_net.cfg.embed_dim
        backbone_fwd(self.t_net, T_, [self.g_img], [None])
        ops.gather_rows(T_.Xn, self.rows_cls_t, ng, Dt, dst_bf16=self.h_t_dino.A0)
        ops.gather_rows(T_.Xn, self.rows_masked_tt, M, Dt, dst_bf16=self.h_t_ibot.A0)
        head_fwd(self.t_net, self.h_t_dino, "dino_head", ng, stash=False)
        head_fwd(self.t_net, self.h_t_ibot, "ibot_head", M, stash=False)
        heads = [(self.h_t_dino.logits[:ng], self.sk_dino), (self.h_t_ibot.logits[:M], self.sk_ibot)]
        if self.centering == "sinkhorn_knopp":
            sinkhorn(heads, teacher_temp, 3, self.reduce)
        else:
            for (L, sk), center in zip(heads, (self.center_dino, self.center_ibot)):
                softmax_center(L, sk, center, teacher_temp, self.center_momentum, self.reduce)
        if self._gram is not None:
            self._gram.teacher_targets(T_, self.g_img, self.params.mods["backbone"])

    def forward_backward(self, teacher_temp: float):
        cfg, B, M = self.cfg, self.B, self.M
        D = cfg.embed_dim
        ng = cfg.n_global * B
        self.metrics.zero_()
        for st in self.params.mods.values():
            st.zero_grads()
        self.fsdp.begin_step()
        self.fsdp.prefetch(self._gather_schedule())
        # ---- teacher (train/ssl_meta_arch.py:366-402).  It shares nothing with the student pass until the losses, so
        # it runs on its own stream: the HBM-bound kernels of one pass overlap the tensor-bound kernels of the other.
        if self.fwd_overlap:
            main = torch.cuda.current_stream()
            self._ev_fwd[0].record(main)
            self.tstream.wait_event(self._ev_fwd[0])          # batch, zeroed metrics, parameters of the last update
            with torch.cuda.stream(self.tstream):
                self.teacher_pass(teacher_temp)
                self._ev_fwd[1].record(self.tstream)
        else:
            self.teacher_pass(teacher_temp)
        # ---- student (train/ssl_meta_arch.py:406-460)
        S_ = self.student
        gram = self._gram if self.gram_active else None
        # a distilling student's global crops get no mask tokens (train/ssl_meta_arch.py:416); the iBOT loss is still
        # taken at the masked positions
        g_masks = self.masks_u8 if self.distill is None else None
        backbone_fwd(self.student_net, S_, [self.g_img, self.l_img], [g_masks, None])
        ops.gather_rows(S_.Xn, self.rows_cls_s, self.Rc, D, dst_bf16=self.h_s_dino.A0, dst_f32=self.cls_f32)
        ops.gather_rows(S_.Xn, self.rows_masked_t, M, D, dst_bf16=self.h_s_ibot.A0)
        if gram is not None:
            gram.features(S_.Xn, student=True)
        head_fwd(self.student_net, self.h_s_dino, "dino_head", self.Rc, stash=True)
        head_fwd(self.student_net, self.h_s_ibot, "ibot_head", M, stash=True)
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
        if cfg.koleo_distributed:
            self.koleo_dist(self.cls_f32[:ng], self.metrics[2:3], self.h_s_dino.dA0, 1.0 / cfg.n_global,
                            cfg.koleo_loss_weight)
        for c in range(0 if cfg.koleo_distributed else cfg.n_global):
            ops.koleo_fwd_bwd(self.cls_f32[c * B:(c + 1) * B], self.koleo_xn, self.koleo_nrm, self.koleo_nn,
                              self.koleo_coef, self.metrics[2:3], self.h_s_dino.dA0[c * B:(c + 1) * B],
                              1.0 / cfg.n_global, cfg.koleo_loss_weight)
        # ---- backward: final norm (dXn is zero except cls rows and masked-patch rows)
        dXn = self.dX[0]
        dXn.zero_()
        ops.scatter_add_rows(self.h_s_dino.dA0, self.rows_cls_s, dXn, self.Rc, D)
        ops.scatter_add_rows(self.h_s_ibot.dA0, self.rows_masked_t, dXn, M, D)
        if gram is not None:
            gram.loss_bwd(dXn, self.metrics)
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
        for cs, masks, dTok in zip(S_.sets, [g_masks, None], self.dTok):
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
        sq_in = self.reduce.input("sumsq", self._sumsq_all)
        if self.reduce.stage is not None:
            sq_in.zero_()                 # d3_sumsq adds; the engine's own buffer was zeroed with the gradients
        for i, st in enumerate(self.params.mods.values()):
            ops.sumsq(st.grad_shard, sq_in[i:i + 1])
        self.reduce(self._sumsq_all, "sum", "sumsq")
        for st in self.params.mods.values():
            ops.adamw_ema(st.master, st.grad_shard, st.m, st.v, st.t_master, st.bf16_shard, st.t_bf16_shard,
                          st.layout.n_mat_shard, st.segs, st.nseg, st.sumsq, float(cfg.clip_grad or 0.0), lr,
                          last_layer_lr, wd, self.step_count, momentum, cfg.adamw_beta1, cfg.adamw_beta2)

    def ema_update(self, momentum: float):
        """Stand-alone teacher EMA (train/ssl_meta_arch.py:644-660) for callers that keep the reference's two-call
        step: `optimizer_step(..., momentum=1.0)` leaves the teacher untouched, then this applies the EMA."""
        for st in self.params.mods.values():
            ops.ema(st.t_master, st.master, st.t_bf16_shard, st.layout.n_mat_shard, float(momentum))

    def set_dino_local_loss_weight(self, w: float):
        """Multiply the local-crop DINO term (its loss in total_loss and its gradient) by w; the tables change only
        when w does."""
        w = float(w)
        if w != self.dino_local_loss_weight:
            torch.mul(self._wg_local, w, out=self.ce_dino[3][self.cfg.n_global * self.B:])
            self.dino_local_loss_weight = w

    def train_step(self, batch: dict | None, *, teacher_temp: float, lr: float, wd: float, last_layer_lr: float,
                   momentum: float, gram_loss_weight: float | None = None, dino_local_loss_weight: float | None = None,
                   iteration: int | None = None):
        if batch is not None:
            self.set_batch(batch)
        if gram_loss_weight is not None and self._gram is not None:   # gram.loss_weight_schedule[iteration] (:534-537)
            self._gram.weight = float(gram_loss_weight)
        if dino_local_loss_weight is not None:            # dino.local_loss_weight_schedule[iteration] (:495-501)
            self.set_dino_local_loss_weight(dino_local_loss_weight)
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
        w_local = self.dino_local_loss_weight
        loss = (cfg.dino_loss_weight * l_scale * w_local * m[0] + cfg.dino_loss_weight * g_scale * m[1]
                + cfg.koleo_loss_weight * ng * m[2] + cfg.ibot_loss_weight * m[3])
        out = {"dino_local_crops_loss": m[0], "dino_local_loss_weight": w_local, "dino_global_crops_loss": m[1],
               "koleo_loss": m[2], "ibot_loss": m[3], "local_batch_size": float(self.B)}
        if self.gram_active:
            loss += self._gram.read(m, out)
        out["total_loss"] = loss
        for name, st in self.params.mods.items():
            out[f"student_{name}_grad_norm"] = math.sqrt(max(st.sumsq.item(), 0.0))
        return out
