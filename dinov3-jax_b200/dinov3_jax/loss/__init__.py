"""Loss objects with the reference's class / method names (dinov3_jax/loss/*.py), forward values computed by the CUDA
kernels on CUDA tensors.  (The training engine uses the same kernels in their fused forward+backward form.)"""
from __future__ import annotations

import torch

from .. import ops
from ..engine.gram import operands, pad8, similarity_diff
from ..engine.losses import SinkhornBufs, SmallReduce, sinkhorn, softmax_center

f32 = torch.float32


def _teacher(teacher_output, owner=None):
    """fp32 logits and one head's normalisation buffers; `owner`'s center ("state" collection) is created on first use."""
    L = teacher_output.to(f32).contiguous()
    if owner is not None and owner.center is None:
        owner.center = torch.zeros(L.shape[1], device=L.device)
    return L, SinkhornBufs.joint([L.shape], L.device)[0]


def _probs(L, sk: SinkhornBufs, teacher_temp: float):
    Q = torch.empty_like(L)
    ops.sinkhorn_probs(L, sk.mx, teacher_temp, sk.s, sk.a, sk.btot, Q)
    return Q


def _ce(student: torch.Tensor, teacher_probs: torch.Tensor, student_temp: float, t0, t1, w):
    """sum_i w_i * CE(student_i, sum of teacher rows t0_i, t1_i) through d3_ce_fwd_bwd (forward only)."""
    S = student.to(f32).contiguous()
    T = teacher_probs.to(f32).contiguous()
    dev = S.device
    metric = torch.zeros(1, device=dev)
    slot = torch.zeros(S.shape[0], dtype=torch.int32, device=dev)
    ops.ce_fwd_bwd(S, student_temp, T, None, 1.0, None, None, None, t0.to(dev), t1.to(dev), w.to(dev), w.to(dev), slot, metric, None)
    return metric[0]


class DINOLoss:
    """loss/dino_clstoken_loss.py:14-95."""

    def __init__(self, out_dim: int, student_temp: float = 0.1, center_momentum: float = 0.9, comm=None):
        self.out_dim, self.student_temp, self.center_momentum, self.comm = out_dim, student_temp, center_momentum, comm
        self.center = None          # "state" collection of the reference (:19-22): [1, K] zeros, created on first use

    def sinkhorn_knopp_teacher(self, teacher_output, teacher_temp, n_iterations=3, init_phase=False):
        L, sk = _teacher(teacher_output)
        sinkhorn([(L, sk)], float(teacher_temp), n_iterations, SmallReduce(None if init_phase else self.comm))
        return _probs(L, sk, float(teacher_temp))

    def softmax_center_teacher(self, teacher_output, teacher_temp, update_centers=True):
        """loss/dino_clstoken_loss.py:24-33: (optionally) apply_center_update first, then softmax((x - center)/temp)."""
        L, sk = _teacher(teacher_output, self)
        softmax_center(L, sk, self.center, float(teacher_temp), self.center_momentum, SmallReduce(self.comm), update_centers)
        return _probs(L, sk, float(teacher_temp))

    def apply_center_update(self, teacher_output):
        """:91-95: center <- m*center + (1-m)*pmean(mean_rows(teacher_output))."""
        L, sk = _teacher(teacher_output, self)
        softmax_center(L, sk, self.center, 1.0, self.center_momentum, SmallReduce(self.comm), probs=False)

    def __call__(self, student_logits, teacher_probs, ignore_diagonal=False):
        S, B, K = student_logits.shape
        T = teacher_probs.shape[0]
        i = torch.arange(S * B)
        s_idx, b_idx = i // B, i % B
        if ignore_diagonal:
            assert T == 2 and S == 2, "ignore_diagonal pairs each global crop with the other one (S = T = 2)"
            t0 = ((1 - s_idx) * B + b_idx).to(torch.int32)
            t1 = torch.full_like(t0, -1)
            w = torch.full((S * B,), 1.0 / (B * S * T - B * min(S, T)))
        else:
            assert T == 2, "teacher has the two global crops"
            t0, t1 = b_idx.to(torch.int32), (B + b_idx).to(torch.int32)
            w = torch.full((S * B,), 1.0 / (B * S * T))
        return _ce(student_logits.reshape(S * B, K), teacher_probs.reshape(T * B, K), self.student_temp, t0, t1, w)


class iBOTPatchLoss:
    """loss/ibot_patch_loss.py:17-109."""

    def __init__(self, patch_out_dim: int, student_temp: float = 0.1, center_momentum: float = 0.9, comm=None):
        self.patch_out_dim, self.student_temp, self.comm = patch_out_dim, student_temp, comm
        self.center_momentum, self.center = center_momentum, None

    def softmax_center_teacher(self, teacher_patch_tokens, teacher_temp, update_centers=True):
        """loss/ibot_patch_loss.py:28-36 (same arithmetic as DINOLoss.softmax_center_teacher, rows = masked patches)."""
        return DINOLoss.softmax_center_teacher(self, teacher_patch_tokens, teacher_temp, update_centers)

    def sinkhorn_knopp_teacher(self, teacher_output, teacher_temp, n_masked_patches_tensor, n_iterations=3, init_phase=False):
        L, sk = _teacher(teacher_output)
        sinkhorn([(L, sk)], float(teacher_temp), n_iterations, SmallReduce(None if init_phase else self.comm),
                 rows=(float(n_masked_patches_tensor.sum()),))
        return _probs(L, sk, float(teacher_temp))

    def forward_masked(self, student_patch_tokens_masked, teacher_patch_tokens_masked, student_masks_flat,
                       n_masked_patches=None, masks_weight=None):
        M = student_patch_tokens_masked.shape[0] if n_masked_patches is None else int(n_masked_patches)
        t0 = torch.arange(M, dtype=torch.int32)
        w = torch.full((M,), 1.0 / student_masks_flat.shape[0])      # masks_weight is NOT applied by the reference (:66)
        return _ce(student_patch_tokens_masked[:M], teacher_patch_tokens_masked[:M], self.student_temp, t0,
                   torch.full_like(t0, -1), w)


class KoLeoLoss:
    """loss/koleo_loss.py:20-35."""

    def __call__(self, student_output, eps=1e-8):
        x = student_output.to(f32).contiguous()
        B, D = x.shape
        dev = x.device
        met, dx = torch.zeros(1, device=dev), torch.zeros(B, D, device=dev)
        ops.koleo_fwd_bwd(x, torch.empty(B, D, device=dev), torch.empty(B, device=dev),
                          torch.empty(B, dtype=torch.int32, device=dev), torch.empty(B, device=dev), met, dx, 1.0, 0.0, eps)
        return met[0]


class KoLeoLossDistributed:
    """loss/koleo_loss.py:39-70: nearest neighbours are searched over the rows of ALL ranks (all-gather over "dp"),
    the loss is the mean over the local rows.  The gathered matrix is tiny ([world*B, D]); the neighbour search runs in
    the same KoLeo kernels on the concatenated rows, and the rows of this rank are picked out of the per-row terms.
    With topk > 1 or a `loss_group_size` (images; a multiple of B dividing world*B) the search runs in
    d3_koleo_topk_rows over this rank's group: the mean over the local rows and their topk neighbours (engine/koleo.py
    states the semantics)."""

    def __init__(self, topk: int = 1, loss_group_size=None, comm=None):
        from ..engine.koleo import MAX_TOPK
        if not 1 <= int(topk) <= MAX_TOPK:
            raise ValueError(f"KoLeoLossDistributed: topk {topk} must be in [1, {MAX_TOPK}]")
        self.topk, self.comm, self.loss_group_size = int(topk), comm, loss_group_size

    def __call__(self, student_output, eps=1e-8):
        x = student_output.to(f32).contiguous()
        B, D = x.shape
        dev = x.device
        world, rank = (1, 0) if self.comm is None else (self.comm.world, self.comm.rank)
        if self.topk > 1 or self.loss_group_size is not None:
            from ..engine.koleo import ranks_per_group
            R = ranks_per_group(world, B, self.loss_group_size, self.topk)
            allx = x
            if world > 1:
                allx = torch.empty(world * B, D, device=dev)
                self.comm.all_gather(allx, x)
            n = world * B
            met = torch.zeros(1, device=dev)
            ops.koleo_topk(allx, ((rank // R) * R * B, R * B), rank * B, B, self.topk,
                           ops.koleo_topk_scratch(n, D, B, self.topk, dev), met, torch.zeros(n, D, device=dev), 1.0,
                           0.0, eps)
            return met[0]
        if world == 1:
            return KoLeoLoss()(x, eps)
        allx = torch.empty(world * B, D, device=dev)
        self.comm.all_gather(allx, x)
        n = world * B
        met, dx = torch.zeros(1, device=dev), torch.zeros(n, D, device=dev)
        ops.koleo_fwd_bwd(allx, torch.empty(n, D, device=dev), torch.empty(n, device=dev),
                          torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, device=dev), met, dx, 1.0, 0.0,
                          eps, row0=rank * B, nrows=B)
        return met[0]


class GramLoss:
    """loss/gram_loss.py:13-50 (SURVEY 8f.2): MSE between the patch-similarity (Gram) matrices of student and gram-teacher
    features.  The value is computed with the library: row normalisation (d3_l2norm_fwd), similarity matrices on the
    tensor cores (d3_gemm_bf16, bf16 operands / fp32 accumulate), negative removal + squared difference (d3_gram_diff).
    `img_level=True` takes the diagonal (per-image) blocks of the batch's similarity matrix.  The training engine uses the same kernels with the
    backward fused in (engine/gram.py:GramAnchor.loss_bwd)."""

    def __init__(self, apply_norm: bool = True, img_level: bool = True, remove_neg: bool = True,
                 remove_only_teacher_neg: bool = False):
        assert remove_neg != remove_only_teacher_neg          # gram_loss.py:20
        self.apply_norm, self.img_level = apply_norm, img_level
        self.remove_neg, self.remove_only_teacher_neg = remove_neg, remove_only_teacher_neg

    def _one(self, s: torch.Tensor, t: torch.Tensor, acc: torch.Tensor, inv: float, block: int = 0):
        n, D = s.shape
        pd = -D % 8                                           # kernels work in 8-column granules; zero columns add nothing
        npad = pad8(n)
        e = lambda *shape, dt=f32: torch.empty(*shape, dtype=dt, device=s.device)
        xs, xt, nrm = e(npad, D + pd, dt=torch.bfloat16), e(npad, D + pd, dt=torch.bfloat16), e(npad)
        for f, x in ((s, xs), (t, xt)):
            operands(torch.nn.functional.pad(f.to(f32), (0, pd, 0, npad - n)).contiguous(), x, nrm, n, self.apply_norm)
        similarity_diff(xs, xt, e(npad, npad), e(npad, npad), None,
                        ops.GRAM_MODES[(self.remove_neg, self.remove_only_teacher_neg)], inv, acc, block=block)

    def __call__(self, output_feats: torch.Tensor, target_feats: torch.Tensor, img_level: bool = True) -> torch.Tensor:
        acc = torch.zeros(1, dtype=f32, device=output_feats.device)
        s = output_feats.reshape(-1, output_feats.shape[-1])
        t = target_feats.reshape(-1, target_feats.shape[-1])
        if img_level:
            assert output_feats.dim() == 3 and target_feats.dim() == 3          # gram_loss.py:25-26
            Bn, n, _ = output_feats.shape
            if (Bn * n) % 8 == 0 and n % 4 == 0:
                self._one(s, t, acc, 1.0 / (Bn * n * n), block=n)
            else:                                             # odd sizes: one image at a time
                for b in range(Bn):
                    self._one(output_feats[b], target_feats[b], acc, 1.0 / (Bn * n * n))
        else:
            self._one(s, t, acc, 1.0 / (s.shape[0] * s.shape[0]))
        return acc[0]
