"""FSDP runtime: NCCL all-gather of each unit's parameters before use and reduce-scatter (mean) of its gradients after
its backward, issued on a side stream so they overlap the neighbouring unit's compute.

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
        self._debug = int(os.environ.get("D3_FSDP_DEBUG", "0"))   # diagnostics only: 1 = skip gathers, 2 = skip reduce-scatters
        # Gradient reduce-scatter without NCCL: every rank ADDS its contribution straight into the owner's gradient
        # shard through NVLink peer mappings (torch symmetric memory provides the mappings) — from the weight-gradient
        # GEMM's epilogue for the big matrices (ops.gemm(scatter=...)), from d3_scatter_add_peers for the rest.
        self.push = False
        self.push_gemm = os.environ.get("D3_FSDP_PUSH_GEMM", "1") != "0"     # 0: only the stand-alone push kernel
        # parameter all-gather of the bf16 matrices through the copy engines (peer-mapped shards) instead of NCCL kernels
        # that take SMs from the persistent GEMM grids; D3_FSDP_DMA_GATHER=0 keeps NCCL
        self.dma_gather = os.environ.get("D3_FSDP_DMA_GATHER", "1") != "0"
        self._peer_views = {}
        self._peer_ptrs = {}
        # vector regions (LN / bias / LayerScale: ~1 MB per module): ONE all-gather per (module, teacher|student) and one
        # permutation kernel at step start instead of one NCCL kernel per unit — ~50 fewer NCCL launches co-running
        # with (and taking SMs from) the teacher pass's persistent GEMMs.  D3_FSDP_VEC_BULK=0: per-unit gathers.
        self.vec_bulk = os.environ.get("D3_FSDP_VEC_BULK", "1") != "0"
        self._fence_barrier = os.environ.get("D3_FSDP_FENCE_BARRIER", "1") != "0"   # 0: NCCL all-reduce as the push fence
        self._push_side = os.environ.get("D3_FSDP_PUSH_SIDE", "1") != "0"          # 0: stand-alone pushes on the compute stream
        self._vec_perm = {}
        self._vec_tmp = {}
        # Default: on at every world size (tools/check_fsdp_push.py compares the pushed shards with the NCCL
        # reduce-scatter).  D3_FSDP_PUSH=0 selects the NCCL reduce-scatter.
        want = os.environ.get("D3_FSDP_PUSH", "auto")
        if self.cuda and self.world > 1 and comm.backend == "nccl" and want in ("1", "auto"):
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
                if self.dma_gather and st.bf16_shard.numel():
                    # bf16 matrix shards (student + teacher) in peer-mapped memory: the parameter all-gather becomes
                    # plain device-to-device copies out of the peers' shards (copy engines, no SM, no NCCL kernel)
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

    def setup_small_allreduce(self, n_floats: int):
        """Symmetric-memory staging buffer for small all-reduces over peer mappings (d3_allreduce_peers); None when the
        peer-memory path is not active (the caller then uses NCCL).  D3_FSDP_SMALL_AR=0 keeps NCCL."""
        import os
        if not self.push or os.environ.get("D3_FSDP_SMALL_AR", "1") == "0":
            return None
        import torch.distributed._symmetric_memory as symm_mem
        dev = next(iter(self.stores.values())).grad_shard.device
        buf = symm_mem.empty(n_floats, dtype=torch.float32, device=dev)
        hdl = symm_mem.rendezvous(buf, self.comm.group)
        buf.zero_()
        torch.cuda.synchronize()
        torch.distributed.barrier(group=self.comm.group)
        self._ar = (buf, hdl, [int(p) for p in hdl.buffer_ptrs])
        return buf

    def small_allreduce(self, off: int, n: int, out: torch.Tensor, op: str):
        """out[:n] = reduce over ranks of stage[off:off+n] (every rank gets identical bits).  One symmetric-memory barrier
        (all ranks have written their inputs; also: all ranks have finished the reads of every EARLIER reduction, which
        is what allows a staging range to be rewritten two calls later) + one pull kernel."""
        from .. import ops
        buf, hdl, ptrs = self._ar
        hdl.barrier(2)
        ops.allreduce_peers([p + 4 * off for p in ptrs], out, n, op)

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
            if self.push and self.dma_gather and hasattr(st, "_symm_param_handles"):
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
        if vb > va and self.vec_bulk:
            works.append(self._vec_done[(module, teacher)])
        elif vb > va:
            sa, sb = L.shard_range(unit, "vec")
            src = (st.t_master if teacher else st.master)[sa:sb]
            dst = (st.t_vecs if teacher else st.vecs)[va - L.n_mat: vb - L.n_mat]
            works.append(self.comm.all_gather(dst, src, async_op=True))
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
        if self.world == 1 or (self._debug & 1):
            return
        items = list(items)
        self._vec_done = {}

        def vecs_first():
            if self.vec_bulk:
                for module, teacher in dict.fromkeys((m, t) for m, _, t in items):
                    self._vec_done[(module, teacher)] = self._gather_vecs(module, teacher)
        if self.side is not None:
            self.side.wait_stream(torch.cuda.current_stream())   # parameters come from the previous optimizer step
            with torch.cuda.stream(self.side):
                if self.push and self.dma_gather:
                    # the copies below read the PEERS' shards: every rank's optimizer step must have finished.  (The
                    # opposite hazard - a peer's next optimizer step overwriting a shard still being copied - is closed
                    # by the fence all-reduce of finish_grads: a rank reaches it only after its backward, i.e. after all
                    # of its gathers of this step were consumed.)
                    st0 = next(iter(self.stores.values()))
                    if hasattr(st0, "_symm_handle"):
                        st0._symm_handle.barrier(0)
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
        if self.world == 1 or (self._debug & 2):
            return
        st = self.stores[module]
        L = st.layout
        unit = next(u for u in L.units if u.name == unit_name)
        if self.push:
            # the stand-alone pushes (proj matrices, vectors, heads, embed: 0.84 ms per ViT-L step at 2 ranks in the
            # kernel timeline) only feed the optimizer: they run on the side stream, off the backward's critical path;
            # finish_grads() joins it before the fence
            cur = torch.cuda.current_stream()
            ps = self.side if (self.side is not None and self._push_side) else cur
            if ps is not cur:
                ps.wait_stream(cur)
            if also_after is not None:
                ps.wait_event(also_after)
            with torch.cuda.stream(ps):
                self._push_ranges(module, unit, tuple(scattered))
            self._pushed_on_side = ps is not cur
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
            if getattr(self, "_pushed_on_side", False):
                torch.cuda.current_stream().wait_stream(self.side)
                self._pushed_on_side = False
            # every rank's pushes are complete once its stream reaches this collective; the all-reduce completes on a
            # rank only after all ranks have joined, so afterwards every contribution has landed in the local shard
            # (a symmetric-memory barrier on this stream has the same property at a fraction of an all-reduce's latency)
            st0 = next(iter(self.stores.values()))
            if self._fence_barrier and hasattr(st0, "_symm_handle"):
                st0._symm_handle.barrier(1)
                return
            self._fence = getattr(self, "_fence", None)
            if self._fence is None:
                self._fence = torch.zeros(1, device=st0.grad_shard.device)
            self.comm.all_reduce_sum(self._fence)

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
