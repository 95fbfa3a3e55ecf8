"""Loss objects with the reference's class / method names (dinov3_jax/loss/*.py), forward values computed by the CUDA
kernels on CUDA tensors.  (The training engine uses the same kernels in their fused forward+backward form.)"""
from __future__ import annotations

import torch

from .. import ops

f32 = torch.float32


def _sinkhorn(teacher_output: torch.Tensor, teacher_temp: float, btot_local: float, n_iterations: int = 3, comm=None):
    L = teacher_output.to(f32).contiguous()
    R, K = L.shape
    dev = L.device
    mx = torch.full((K,), float("-inf"), device=dev)      # per-prototype shift (cancels exactly, see csrc/losses.cu)
    btot = torch.tensor([float(btot_local)], device=dev)
    ops.colmax(L, mx)
    if comm is not None:
        comm.all_reduce_max(mx)
        comm.all_reduce_sum(btot)
    s, a_buf, a = torch.zeros(K, device=dev), torch.empty(R, device=dev), None
    for _ in range(n_iterations):
        s.zero_()
        ops.sinkhorn_colsum(L, mx, teacher_temp, a, s)
        if comm is not None:
            comm.all_reduce_sum(s)
        ops.sinkhorn_rowsum(L, mx, teacher_temp, s, btot, a_buf)
        a = a_buf
    Q = torch.empty(R, K, device=dev)
    ops.sinkhorn_probs(L, mx, teacher_temp, s, a, btot, Q)
    return Q


def _softmax_center(obj, teacher_output, teacher_temp: float, update: bool, probs: bool = True):
    L = teacher_output.to(f32).contiguous()
    R, K = L.shape
    dev = L.device
    if obj.center is None:
        obj.center = torch.zeros(K, device=dev)
    gmx = torch.full((1,), float("-inf"), device=dev)
    rows = torch.tensor([float(R)], device=dev)
    ops.absmax(L, gmx)
    colsum = torch.zeros(K, device=dev)
    if update:
        ops.colsum_f32(L, colsum)
    if obj.comm is not None:
        obj.comm.all_reduce_max(gmx)
        obj.comm.all_reduce_sum(rows)
        if update:
            obj.comm.all_reduce_sum(colsum)
    s = torch.empty(K, device=dev)
    # momentum 1.0 leaves the center untouched and only produces s[k] = exp((center[k] - max center)/temp)/K
    ops.center_update(obj.center, colsum, rows, obj.center_momentum if update else 1.0, teacher_temp, s)
    if not probs:
        return None
    mx = gmx.expand(K).contiguous()
    a = torch.empty(R, device=dev)
    ops.sinkhorn_rowsum(L, mx, teacher_temp, s, rows, a)
    Q = torch.empty(R, K, device=dev)
    ops.sinkhorn_probs(L, mx, teacher_temp, s, a, rows, Q)
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
        world = 1 if (self.comm is None or init_phase) else self.comm.world
        return _sinkhorn(teacher_output, float(teacher_temp), teacher_output.shape[0], n_iterations,
                         None if init_phase else self.comm)

    def softmax_center_teacher(self, teacher_output, teacher_temp, update_centers=True):
        """loss/dino_clstoken_loss.py:24-33: (optionally) apply_center_update first, then softmax((x - center)/temp).
        Same kernels as the engine's optional centering path (engine/core.py::_softmax_center)."""
        return _softmax_center(self, teacher_output, float(teacher_temp), update_centers)

    def apply_center_update(self, teacher_output):
        """:91-95: center <- m*center + (1-m)*pmean(mean_rows(teacher_output))."""
        _softmax_center(self, teacher_output, 1.0, True, probs=False)

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
        return _softmax_center(self, teacher_patch_tokens, float(teacher_temp), update_centers)

    def sinkhorn_knopp_teacher(self, teacher_output, teacher_temp, n_masked_patches_tensor, n_iterations=3, init_phase=False):
        return _sinkhorn(teacher_output, float(teacher_temp), float(n_masked_patches_tensor.sum()), n_iterations,
                         None if init_phase else self.comm)

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
    the same KoLeo kernels on the concatenated rows, and the rows of this rank are picked out of the per-row terms."""

    def __init__(self, topk: int = 1, loss_group_size=None, comm=None):
        if topk != 1:
            raise NotImplementedError("KoLeoLossDistributed: topk > 1 is not on the GPU path")
        self.comm, self.loss_group_size = comm, loss_group_size

    def __call__(self, student_output, eps=1e-8):
        x = student_output.to(f32).contiguous()
        B, D = x.shape
        dev = x.device
        if self.comm is None or self.comm.world == 1:
            return KoLeoLoss()(x, eps)
        world, rank = self.comm.world, self.comm.rank
        allx = torch.empty(world * B, D, device=dev)
        self.comm.all_gather(allx, x)
        n = world * B
        met, dx = torch.zeros(1, device=dev), torch.zeros(n, D, device=dev)
        ops.koleo_fwd_bwd_rows(allx, torch.empty(n, D, device=dev), torch.empty(n, device=dev),
                               torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, device=dev), met, dx,
                               rank * B, B, 1.0, 0.0, eps)
        return met[0]


class GramLoss:
    """loss/gram_loss.py:13-50 (SURVEY 8f.2): MSE between the patch-similarity (Gram) matrices of student and gram-teacher
    features.  The value is computed with the library: row normalisation (d3_l2norm_fwd), similarity matrices on the
    tensor cores (d3_gemm_bf16, bf16 operands / fp32 accumulate), negative removal + squared difference (d3_gram_diff).
    `img_level=True` takes the diagonal (per-image) blocks of the batch's similarity matrix.  The training engine uses the same kernels with the
    backward fused in (engine/core.py:_gram_loss_bwd)."""

    def __init__(self, apply_norm: bool = True, img_level: bool = True, remove_neg: bool = True,
                 remove_only_teacher_neg: bool = False):
        assert remove_neg != remove_only_teacher_neg          # gram_loss.py:20
        self.apply_norm, self.img_level = apply_norm, img_level
        self.remove_neg, self.remove_only_teacher_neg = remove_neg, remove_only_teacher_neg

    def _one(self, s: torch.Tensor, t: torch.Tensor, acc: torch.Tensor, inv: float, block: int = 0):
        n, D = s.shape
        pn, pd = (0 if block else -n % 8), -D % 8             # kernels work in 8-element granules; zero padding adds nothing
        if pn or pd:
            s, t = torch.nn.functional.pad(s, (0, pd, 0, pn)), torch.nn.functional.pad(t, (0, pd, 0, pn))
        s, t = s.to(f32).contiguous(), t.to(f32).contiguous()
        m = s.shape[0]
        xs, xt = torch.empty_like(s, dtype=torch.bfloat16), torch.empty_like(t, dtype=torch.bfloat16)
        if self.apply_norm:
            nrm = torch.empty(m, dtype=f32, device=s.device)
            ops.l2norm_fwd(s, xs, nrm, 1e-12)
            ops.l2norm_fwd(t, xt, nrm, 1e-12)
        else:
            xs.copy_(s); xt.copy_(t)
        Ss, St = torch.empty(m, m, dtype=f32, device=s.device), torch.empty(m, m, dtype=f32, device=s.device)
        ops.gemm(xs, xs, Ss)
        ops.gemm(xt, xt, St)
        ops.gram_diff(Ss, St, None, ops.GRAM_MODES[(self.remove_neg, self.remove_only_teacher_neg)], inv, acc, block=block)

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
