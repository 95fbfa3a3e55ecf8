"""Sinkhorn-Knopp (loss/dino_clstoken_loss.py:35-62, ibot_patch_loss.py:77-109) and softmax centering (:24-33,91-95) of
teacher logits, for the engine (both heads in lock step) and the loss classes (one head), as the scalings mx, s, a, btot."""
from __future__ import annotations

import itertools

import torch

from .. import ops

f32 = torch.float32


class SinkhornBufs:
    """One head's buffers.  Heads made by one `joint` call share `shared["mx"]` and `shared["s"]`: head j's K prototypes
    sit at [off, off + K) of both, its row total at s[Ks + j], so one reduction per stage covers every head."""

    def __init__(self, shared: dict, R: int, K: int, off: int, slot: int, device):
        self.shared, self.K, self.off = shared, K, off
        Ks = shared["mx"].numel()
        self.mx = shared["mx"][off:off + K]       # per-prototype shift (column maxima / global max)
        self.s = shared["s"][off:off + K]
        self.btot = shared["s"][Ks + slot:Ks + slot + 1]
        self.colsum = shared["colsum"][:K]        # softmax centering: column sums of one head at a time
        self.gmx = torch.empty(1, dtype=f32, device=device)
        self.a = torch.empty(R, dtype=f32, device=device)

    @classmethod
    def joint(cls, sizes: list, device) -> list:
        """One SinkhornBufs per (rows, prototypes) in `sizes` (at most 4 heads)."""
        Ks, z = sum(K for _, K in sizes), (lambda n: torch.zeros(n, dtype=f32, device=device))
        shared = {"mx": torch.empty(Ks, dtype=f32, device=device), "s": z(Ks + 4), "rows": z(4), "rows_set": None,
                  "colsum": z(max(K for _, K in sizes))}
        return [cls(shared, R, K, sum(k for _, k in sizes[:j]), j, device) for j, (R, K) in enumerate(sizes)]


class SmallReduce:
    """Cross-rank reductions of a few KB (Sinkhorn vectors, gradient norms: latency, not bandwidth).  With NVLink peer
    memory (`peer`) the inputs are written straight into a symmetric-memory staging buffer, one range per `part`, and
    pulled by d3_allreduce_peers; otherwise NCCL (`comm`), or nothing on one GPU."""

    def __init__(self, comm=None, parts: dict | None = None, peer: bool = False, device=None):
        self.comm, self.stage, parts = comm, None, parts or {}      # parts: name -> size of its staging range
        self.offsets = dict(zip(parts, itertools.accumulate(parts.values(), initial=0)))
        if peer:
            import torch.distributed._symmetric_memory as symm_mem
            self.stage = symm_mem.empty(sum(parts.values()), dtype=f32, device=device)
            self._hdl = symm_mem.rendezvous(self.stage, comm.group)
            self._ptrs = [int(p) for p in self._hdl.buffer_ptrs]
            self.stage.zero_()
            torch.cuda.synchronize()
            torch.distributed.barrier(group=comm.group)

    def input(self, part: str, out: torch.Tensor) -> torch.Tensor:
        """Where the inputs of `out`'s reduction go: `part`'s staging range, or `out` itself."""
        if self.stage is None:
            return out
        return self.stage[self.offsets[part]:self.offsets[part] + out.numel()]

    def __call__(self, out: torch.Tensor, op: str, part: str | None = None):
        """out = reduction over ranks (op "max" | "sum", the same bits on every rank) of `input(part, out)`.  Staged: a
        barrier (all inputs written; all reads of earlier reductions done, so a range is reusable two calls later)."""
        if part is not None and self.stage is not None:
            self._hdl.barrier(2)
            ops.allreduce_peers([p + 4 * self.offsets[part] for p in self._ptrs], out, out.numel(), op)
        elif self.comm is not None:
            (self.comm.all_reduce_max if op == "max" else self.comm.all_reduce_sum)(out)


def sinkhorn(heads: list, temp: float, n_iter: int, reduce: SmallReduce, rows: tuple | None = None):
    """Sinkhorn-Knopp over `heads` [(logits [R, K], SinkhornBufs of one `joint`)]: one all-reduce(max) of the column
    maxima, then per iteration one all-reduce(sum) of the column sums and row totals (`rows`, default R) of all heads."""
    shared = heads[0][1].shared
    mx2, s2 = shared["mx"], shared["s"]
    Ks = mx2.numel()
    rows = tuple(L.shape[0] for L, _ in heads) if rows is None else tuple(rows)
    if shared["rows_set"] != rows:               # device copy refreshed only when a row count changes
        for j, r in enumerate(rows):
            shared["rows"][j:j + 1].fill_(float(r))
        shared["rows_set"] = rows
    live = [(L, sk) for L, sk in heads if L.shape[0]]
    mx_in = reduce.input("max", mx2)
    mx_in.fill_(float("-inf"))
    for L, sk in live:
        ops.colmax(L, mx_in[sk.off:sk.off + sk.K])
    reduce(mx2, "max", "max")
    for it in range(n_iter):
        part = ("sum0", "sum1")[it & 1]          # a peer may still be reading the previous iteration's staged sums
        s_in = reduce.input(part, s2)
        s_in.zero_()
        s_in[Ks:].copy_(shared["rows"])
        for L, sk in live:             # the row scalings of the previous iteration (none in the first)
            ops.sinkhorn_colsum(L, sk.mx, temp, sk.a[:L.shape[0]] if it else None, s_in[sk.off:sk.off + sk.K])
        reduce(s2, "sum", part)                  # psum of the row sums (:53 / ibot :99) and of the row totals
        for L, sk in live:
            ops.sinkhorn_rowsum(L, sk.mx, temp, sk.s, sk.btot, sk.a[:L.shape[0]])


def softmax_center(L: torch.Tensor, sk: SinkhornBufs, center: torch.Tensor, temp: float, momentum: float,
                   reduce: SmallReduce, update: bool = True, probs: bool = True):
    """softmax((L - center)/temp) after the center EMA update, as one global shift sk.mx, sk.s and the row scalings
    sk.a.  `update` False leaves the center untouched (momentum 1); `probs` False stops after the center update."""
    R = L.shape[0]
    sk.gmx.fill_(float("-inf"))
    sk.btot.fill_(float(R))
    ops.absmax(L, sk.gmx)
    sk.colsum.zero_()
    if update:
        ops.colsum_f32(L, sk.colsum)
    reduce(sk.gmx, "max")
    reduce(sk.btot, "sum")
    if update:
        reduce(sk.colsum, "sum")                 # pmean of the local centers over "dp" (:93)
    sk.mx.copy_(sk.gmx.expand_as(sk.mx))         # one global shift for every prototype (device-side broadcast)
    ops.center_update(center, sk.colsum, sk.btot, momentum if update else 1.0, temp, sk.s)
    if probs:
        ops.sinkhorn_rowsum(L, sk.mx, temp, sk.s, sk.btot, sk.a[:R])
