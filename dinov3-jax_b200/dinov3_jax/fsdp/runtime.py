"""FSDP runtime: all-gather of each unit's parameters before use and reduce-scatter (mean) of its gradients after its
backward, issued on a side stream so they overlap the neighbouring unit's compute.

With NCCL and more than one rank both go through NVLink peer memory (torch symmetric memory): the bf16 matrices are
gathered by copy-engine copies out of the peers' shards, and every rank adds its gradients straight into the owners'
fp32 shards (the weight-gradient GEMM epilogue for the big matrices, d3_scatter_add_peers for the rest), fenced by a
symmetric-memory barrier.  NCCL all_gather / reduce_scatter is the fallback: on gloo (the CPU tests), where symmetric
memory is unavailable, and with D3_FSDP_PUSH=0.  The small vector ranges always take one all-gather per module.

Replaces `gather_params` / `fwd_gather_bwd_pmean_scatter` / `sync_grads` of the reference (dinov3_jax/fsdp/utils.py:
56-110), which lower to per-leaf jax.lax.all_gather / psum_scatter / pmean inside the jitted step.  torch.distributed
(backend "nccl"; "gloo" in the CPU tests) is the plumbing; payloads are the flat per-unit ranges of fsdp/layout.py.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


class Comm:
    """Thin wrapper over a process group ("dp" axis of the reference's 1-D mesh, train/train.py:322-325)."""

    def __init__(self, group=None):
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.backend = dist.get_backend(self.group)

    def all_reduce_sum(self, t):
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)

    def all_reduce_max(self, t):
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)

    def all_reduce_mean(self, t):
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        t.div_(self.world)

    def all_gather(self, out, inp, async_op=False):
        """out = concat over ranks of inp (tiled all-gather, fsdp/utils.py:66)."""
        return dist.all_gather_into_tensor(out, inp, group=self.group, async_op=async_op)

    def all_to_all(self, out, inp):
        """Slice q of inp (dim 0 cut into world equal slices) goes to rank q; out = the slices sent to this rank, in
        rank order."""
        dist.all_to_all_single(out, inp, group=self.group)

    def reduce_scatter_mean(self, out, inp, async_op=False):
        """out = this rank's slice of mean over ranks of inp (psum_scatter / axis_size, fsdp/utils.py:61-64)."""
        if self.backend == "nccl":
            return dist.reduce_scatter_tensor(out, inp, op=dist.ReduceOp.AVG, group=self.group, async_op=async_op)
        # gloo has no reduce_scatter: all-reduce a copy and keep our slice (CPU tests only)
        tmp = inp.clone()
        dist.all_reduce(tmp, op=dist.ReduceOp.SUM, group=self.group)
        n = out.numel()
        out.copy_(tmp[self.rank * n:(self.rank + 1) * n] / self.world)
        return None


class _EventWork:
    """`wait()` like a c10d Work: makes the current stream wait for an event recorded on the gather stream."""

    def __init__(self, ev):
        self.ev = ev

    def wait(self):
        torch.cuda.current_stream().wait_event(self.ev)


class FsdpRuntime:
    """Schedules the collectives of one rank.  `stores`: dict module -> ModuleStore (engine/params.py)."""

    def __init__(self, comm: Comm | None, stores: dict, device):
        self.comm = comm
        self.stores = stores
        self.world = 1 if comm is None else comm.world
        self.cuda = torch.device(device).type == "cuda"
        self.side = torch.cuda.Stream(device=device) if (self.cuda and self.world > 1) else None
        self._pending = {}       # (module, unit, teacher) -> [works]
        self._grad_works = []
        import os
        # Gradient reduce-scatter without NCCL: every rank ADDS its contribution straight into the owner's gradient
        # shard through NVLink peer mappings (torch symmetric memory provides the mappings) — from the weight-gradient
        # GEMM's epilogue for the big matrices (ops.gemm(scatter=...)), from d3_scatter_add_peers for the rest.
        self.push = False
        self._peer_views = {}
        self._peer_ptrs = {}
        # vector regions (LN / bias / LayerScale: ~1 MB per module): ONE all-gather per (module, teacher|student) and one
        # permutation kernel at step start instead of one NCCL kernel per unit — ~50 fewer NCCL launches co-running
        # with (and taking SMs from) the teacher pass's persistent GEMMs.
        self._vec_perm = {}
        self._vec_tmp = {}
        # On at every world size.  D3_FSDP_PUSH=0 selects the NCCL reduce-scatter and all-gather
        # (tools/check_fsdp_push.py compares the pushed shards with the NCCL reduce-scatter).
        if self.cuda and self.world > 1 and comm.backend == "nccl" and os.environ.get("D3_FSDP_PUSH", "1") != "0":
            self._setup_push()

    def _setup_push(self):
        import torch.distributed._symmetric_memory as symm_mem
        try:
            for name, st in self.stores.items():
                shard = symm_mem.empty(st.grad_shard.numel(), dtype=torch.float32, device=st.grad_shard.device)
                hdl = symm_mem.rendezvous(shard, self.comm.group)
                shard.zero_()
                st.grad_shard = shard
                self._peer_ptrs[name] = [int(p) for p in hdl.buffer_ptrs]
                st._symm_handle = hdl
                if st.bf16_shard.numel():
                    # bf16 matrix shards (student + teacher) in peer-mapped memory: the parameter all-gather becomes
                    # plain device-to-device copies out of the peers' shards (copy engines, no SM, no NCCL kernel
                    # taking SMs from the persistent GEMM grids)
                    hs = {}
                    for attr in ("bf16_shard", "t_bf16_shard"):
                        old = getattr(st, attr)
                        buf = symm_mem.empty(old.numel(), dtype=torch.bfloat16, device=old.device)
                        h = symm_mem.rendezvous(buf, self.comm.group)
                        buf.copy_(old)
                        setattr(st, attr, buf)
                        hs[attr] = h
                    st._symm_param_handles = hs
            torch.cuda.synchronize()
            torch.distributed.barrier(group=self.comm.group)
            self.push = True
        except Exception as e:            # no peer access on this box: keep the NCCL reduce-scatter
            import warnings
            warnings.warn(f"symmetric-memory gradient push disabled ({type(e).__name__}: {e}); using NCCL reduce-scatter")
            self.push = False

    def scatter_spec(self, module: str, unit_name: str, tensor: str):
        """(peer pointers at this unit's shard slice, offset of the tensor inside the unit's matrix range, shard length)
        for ops.gemm(scatter=...), or None when gradients go through NCCL."""
        if not self.push:
            return None
        st = self.stores[module]
        L = st.layout
        unit = next(u for u in L.units if u.name == unit_name)
        a, b = unit.mat
        s = (b - a) // self.world
        so, _ = L.shard_range(unit, "mat")
        return [p + 4 * so for p in self._peer_ptrs[module]], L.offsets[tensor] - a, s

    def begin_step(self):
        """Gradient shards accumulate pushes from every rank, so they start each step at zero.  Safe without a barrier:
        a peer can only push after its forward, which needs this rank's all-gathers, which are queued after this."""
        if self.push:
            for st in self.stores.values():
                st.grad_shard.zero_()

    def _push_ranges(self, module: str, unit, skip: tuple):
        """Push every gradient range of the unit that the GEMM epilogues did not already scatter."""
        from .. import ops
        st = self.stores[module]
        L = st.layout
        inv = 1.0 / self.world
        peers = self._peer_ptrs[module]
        for region in ("mat", "vec"):
            a, b = getattr(unit, region)
            if b <= a:
                continue
            s = (b - a) // self.world
            so, _ = L.shard_range(unit, region)
            pp = [p + 4 * so for p in peers]
            # maximal runs of the region not covered by `skip` tensors
            holes = sorted((L.offsets[t], L.offsets[t] + L.padded[t]) for t in skip if L.kinds[t] == ("mat" if region == "mat" else "vec"))
            cur = a
            for ha, hb in holes + [(b, b)]:
                if ha > cur:
                    ops.scatter_add_peers(st.grad[cur:ha], pp, cur - a, s, inv)
                cur = max(cur, hb)

    # ------------------------------------------------------------------------------------------ parameter gathers
    def _issue_gather(self, module: str, unit, teacher: bool):
        st = self.stores[module]
        L = st.layout
        works = []
        ma, mb = unit.mat
        if mb > ma:
            sa, sb = L.shard_range(unit, "mat")
            src = (st.t_bf16_shard if teacher else st.bf16_shard)[sa:sb]
            dst = (st.t_bf16 if teacher else st.bf16)[ma:mb]
            if self.push:
                # tiled all-gather (fsdp/utils.py:66) as world copies: slice r of the unit comes from rank r's shard
                n = sb - sa
                views = self._shard_views(module, st, teacher)
                for r in range(self.world):
                    dst[r * n:(r + 1) * n].copy_(views[r][sa:sb], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream())
                works.append(_EventWork(ev))
            else:
                works.append(self.comm.all_gather(dst, src, async_op=True))
        va, vb = unit.vec
        if vb > va:
            works.append(self._vec_done[(module, teacher)])
        self._pending[(module, unit.name, teacher)] = works

    def _gather_vecs(self, module: str, teacher: bool):
        """All vector regions of a module in one collective: rank r's vector shard is contiguous
        ([n_mat_shard, n_shard) of its shard buffer, fsdp/layout.py), so one all-gather gives [world][n_vec_shard];
        an index_select with a precomputed permutation lays it out unit-major like the single-GPU buffer."""
        st = self.stores[module]
        L = st.layout
        nv = L.n_shard - L.n_mat_shard
        dst = st.t_vecs if teacher else st.vecs
        if nv == 0:
            return None
        if module not in self._vec_perm:
            import numpy as np
            perm = np.empty(L.n - L.n_mat, dtype=np.int64)
            for u in L.units:
                va, vb = u.vec
                if vb <= va:
                    continue
                s_u = (vb - va) // self.world
                so = L.shard_vec_off[u.name] - L.n_mat_shard
                for r in range(self.world):
                    perm[va - L.n_mat + r * s_u: va - L.n_mat + (r + 1) * s_u] = r * nv + so + np.arange(s_u)
            self._vec_perm[module] = torch.from_numpy(perm).to(dst.device)
            self._vec_tmp[module] = torch.empty(self.world * nv, dtype=dst.dtype, device=dst.device)
        tmp = self._vec_tmp[module]
        self.comm.all_gather(tmp, (st.t_master if teacher else st.master)[L.n_mat_shard:L.n_shard])
        torch.index_select(tmp, 0, self._vec_perm[module], out=dst)
        if self.cuda:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            return _EventWork(ev)
        return None

    def _shard_views(self, module: str, st, teacher: bool):
        key = (module, teacher)
        if key not in self._peer_views:
            attr = "t_bf16_shard" if teacher else "bf16_shard"
            h = st._symm_param_handles[attr]
            n = getattr(st, attr).numel()
            self._peer_views[key] = [getattr(st, attr) if r == self.comm.rank else h.get_buffer(r, (n,), torch.bfloat16, 0)
                                     for r in range(self.world)]
        return self._peer_views[key]

    def prefetch(self, items):
        """items: iterable of (module, unit, teacher) in use order.  All gathers are queued on the side stream at once:
        NCCL executes them back to back while the compute stream works through earlier units."""
        if self.world == 1:
            return
        items = list(items)
        self._vec_done = {}

        def vecs_first():
            for module, teacher in dict.fromkeys((m, t) for m, _, t in items):
                self._vec_done[(module, teacher)] = self._gather_vecs(module, teacher)
        if self.side is not None:
            self.side.wait_stream(torch.cuda.current_stream())   # parameters come from the previous optimizer step
            with torch.cuda.stream(self.side):
                if self.push:
                    # the copies below read the PEERS' shards: every rank's optimizer step must have finished.  (The
                    # opposite hazard - a peer's next optimizer step overwriting a shard still being copied - is closed
                    # by the fence barrier of finish_grads: a rank reaches it only after its backward, i.e. after all
                    # of its gathers of this step were consumed.)
                    next(iter(self.stores.values()))._symm_handle.barrier(0)
                vecs_first()
                for module, unit, teacher in items:
                    self._issue_gather(module, unit, teacher)
        else:
            vecs_first()
            for module, unit, teacher in items:
                self._issue_gather(module, unit, teacher)

    def acquire(self, module: str, unit_name: str, teacher: bool):
        """Make the compute stream wait for this unit's gathered parameters."""
        if self.world == 1:
            return
        for w in self._pending.pop((module, unit_name, teacher), []):
            if w is not None:
                w.wait()

    # ------------------------------------------------------------------------------------------ gradient reduction
    def grads_ready(self, module: str, unit_name: str, also_after=None, scattered=()):
        """Called right after the kernels of this unit's backward were enqueued: reduce-scatter (mean) its gradient
        ranges into the rank's gradient shard, on the side stream."""
        if self.world == 1:
            return
        st = self.stores[module]
        L = st.layout
        unit = next(u for u in L.units if u.name == unit_name)
        if self.push:
            # the stand-alone pushes (proj matrices, vectors, heads, embed: 0.84 ms per ViT-L step at 2 ranks in the
            # kernel timeline) only feed the optimizer: they run on the side stream, off the backward's critical path;
            # finish_grads() joins it before the fence
            self.side.wait_stream(torch.cuda.current_stream())
            if also_after is not None:
                self.side.wait_event(also_after)
            with torch.cuda.stream(self.side):
                self._push_ranges(module, unit, tuple(scattered))
            return

        def issue():
            for region in ("mat", "vec"):
                a, b = getattr(unit, region)
                if b > a:
                    sa, sb = L.shard_range(unit, region)
                    w = self.comm.reduce_scatter_mean(st.grad_shard[sa:sb], st.grad[a:b], async_op=True)
                    if w is not None:
                        self._grad_works.append(w)
        if self.side is not None:
            self.side.wait_stream(torch.cuda.current_stream())
            if also_after is not None:       # kernels of this unit enqueued on another stream (weight gradients)
                self.side.wait_event(also_after)
            with torch.cuda.stream(self.side):
                issue()
        else:
            if also_after is not None:
                torch.cuda.current_stream().wait_event(also_after)
            issue()

    def finish_grads(self):
        for w in self._grad_works:
            w.wait()
        self._grad_works = []
        if self.push:
            torch.cuda.current_stream().wait_stream(self.side)
            # every rank's pushes are complete once its stream reaches this barrier; the barrier completes on a rank
            # only after all ranks have reached it, so afterwards every contribution has landed in the local shard
            next(iter(self.stores.values()))._symm_handle.barrier(1)

    # ------------------------------------------------------------------------------------------ utilities
    def gather_full(self, module: str, what: str, teacher: bool = False) -> torch.Tensor:
        """Full fp32 flat buffer of a module assembled from all ranks' shards (export / checkpoint / tests)."""
        st = self.stores[module]
        L = st.layout
        src = {"param": st.t_master if teacher else st.master, "grad": getattr(st, "grad_shard", None),
               "m": getattr(st, "m", None), "v": getattr(st, "v", None)}[what]
        if self.world == 1:
            return src
        full = torch.empty(L.n, dtype=src.dtype, device=src.device)
        for u in L.units:
            for region in ("mat", "vec"):
                a, b = getattr(u, region)
                if b > a:
                    sa, sb = L.shard_range(u, region)
                    self.comm.all_gather(full[a:b], src[sa:sb].contiguous())
        return full
