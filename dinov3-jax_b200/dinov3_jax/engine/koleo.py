"""Distributed KoLeo inside the step (dino.koleo_loss_distributed, loss/koleo_loss.py:39-70): top-k neighbours over
the class tokens of every rank of a loss group, with the gradient of each row returned to the rank that owns it.

Semantics (parity unpinned: the reference's own distributed KoLeo does not run, it normalises without keepdims, so
these are upstream DINOv3's):
  * a loss group is `group_size` images (None: all world*B), i.e. R = group_size / B consecutive ranks; a rank
    searches neighbours only among its group's rows, gathered in rank order;
  * per global crop, rank r's term L_r = -mean over its B rows i and their k neighbours j of
    log(||xn_i - xn_j|| + eps + eps), xn = x / (||x|| + eps), neighbours = the k largest fp32 dots (ties: lower index);
  * rank q's class-token gradient is sum_r dL_r/dx_q, summed in rank order (the same bits on every run).
R = 1 (one GPU, or groups of one rank) needs no communication: the kernel runs on the rank's own rows.
"""
from __future__ import annotations

import torch

from .. import ops

f32 = torch.float32
MAX_TOPK = 16


def ranks_per_group(world: int, B: int, group_size: int | None, topk: int) -> int:
    """R, the ranks in one loss group; raises on a group size or topk the layout cannot take."""
    G = world * B if group_size is None else int(group_size)
    if G <= 0 or G % B:
        raise ValueError(f"koleo_distributed_loss_group_size {group_size} must be a multiple of the per-GPU batch {B}")
    if (world * B) % G:
        raise ValueError(f"koleo_distributed_loss_group_size {G} must divide the global batch {world * B} "
                         f"({world} ranks x {B})")
    if not 1 <= int(topk) <= min(MAX_TOPK, G - 1):
        raise ValueError(f"koleo_topk {topk} must be in [1, min({MAX_TOPK}, rows in the loss group - 1 = {G - 1})]")
    return G // B


def group_comm(comm, R: int):
    """The communicator of this rank's loss group: R consecutive ranks of `comm` (every rank builds every group, in
    the same order, as torch.distributed.new_group requires).  None when R == 1."""
    if R == 1:
        return None
    if R == comm.world:
        return comm
    import torch.distributed as dist
    from ..fsdp.runtime import Comm
    ranks = dist.get_process_group_ranks(comm.group)
    mine = None
    for g in range(comm.world // R):
        grp = dist.new_group(ranks[g * R:(g + 1) * R])
        if g == comm.rank // R:
            mine = grp
    return Comm(mine)


class DistributedKoLeo:
    """Buffers and the per-step sequence: gather the group's class rows, the kernel per crop, the exchange of the dx
    slabs and their sum, in rank order, into the class-token gradient."""

    def __init__(self, comm, B: int, D: int, n_global: int, topk: int, group_size: int | None, device):
        world = 1 if comm is None else comm.world
        self.R = ranks_per_group(world, B, group_size, topk)
        self.B, self.D, self.n_global, self.topk = B, D, n_global, int(topk)
        self.comm = group_comm(comm, self.R) if comm is not None else None
        self.m = 0 if self.comm is None else self.comm.rank        # position inside the group
        n = self.R * B
        self.scratch = ops.koleo_topk_scratch(n, D, B, self.topk, device)
        if self.R > 1:
            self.xg = torch.empty(n_global, n, D, dtype=f32, device=device)
            self.dxg = torch.empty(n_global, n, D, dtype=f32, device=device)
            self.recv = torch.empty(n_global, self.R, B, D, dtype=f32, device=device)
            self.rows = [torch.arange(c * B, (c + 1) * B, dtype=torch.int32, device=device) for c in range(n_global)]

    def exchange(self, c: int):
        """recv[c][r] = rank r's contribution to this rank's rows (its dxg[c] slab of this rank)."""
        self.comm.all_to_all(self.recv[c].view(self.R * self.B, self.D), self.dxg[c])
        return self.recv[c]

    def __call__(self, cls: torch.Tensor, metric: torch.Tensor, dcls: torch.Tensor, w_metric: float, w_grad: float):
        """cls [n_global * B, D] fp32 (crop-major) -> metric += w_metric * sum over crops of L_r;
        dcls [n_global * B, D] += w_grad * the summed gradient of this rank's rows."""
        B, k = self.B, self.topk
        if self.R == 1:
            for c in range(self.n_global):
                ops.koleo_topk(cls[c * B:(c + 1) * B], (0, B), 0, B, k, self.scratch, metric, dcls[c * B:(c + 1) * B],
                               w_metric, w_grad)
            return
        n = self.R * B
        for c in range(self.n_global):
            self.comm.all_gather(self.xg[c], cls[c * B:(c + 1) * B])
        self.dxg.zero_()
        for c in range(self.n_global):
            ops.koleo_topk(self.xg[c], (0, n), self.m * B, B, k, self.scratch, metric, self.dxg[c], w_metric, w_grad)
            recv = self.exchange(c)
            for r in range(self.R):                                  # rank order
                ops.scatter_add_rows(recv[r], self.rows[c], dcls, B, self.D)
