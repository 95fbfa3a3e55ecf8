"""Host-side FSDP logic on CPU: shard layout invariants, per-rank optimiser segment tables, and the all-gather /
reduce-scatter(mean) plumbing over a world_size-2 gloo group (no CUDA kernels are called here)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from dinov3_jax.engine.config import EngineConfig
from dinov3_jax.engine.params import ALIGN, backbone_spec, head_spec, lr_wd_multipliers
from dinov3_jax.fsdp.layout import ShardLayout


def build_layout(module, spec, world):
    offsets, padded, kinds = {}, {}, {}
    off = 0
    n_mat = 0
    for kind in ("mat", "vec"):
        for name, shape, k in spec:
            if k != kind:
                continue
            offsets[name] = off
            kinds[name] = k
            padded[name] = (int(np.prod(shape)) + ALIGN - 1) // ALIGN * ALIGN
            off += padded[name]
        if kind == "mat":
            n_mat = off
    return ShardLayout(module, [n for n, _, _ in spec], offsets, padded, kinds, n_mat, off, world), offsets, padded


CFG = EngineConfig(embed_dim=128, depth=3, heads=2, n_prototypes=512, head_hidden=256, head_bottleneck=64)


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("module", ["backbone", "dino_head"])
def test_shards_partition_the_flat_buffer(world, module):
    spec = backbone_spec(CFG) if module == "backbone" else head_spec(CFG)
    L, offsets, padded = build_layout(module, spec, world)
    seen = np.zeros(L.n, dtype=np.int32)
    for r in range(world):
        idx = L.full_to_shard_index(r)
        assert len(idx) == L.n_shard
        seen[idx] += 1
    assert (seen == 1).all()                       # every element owned by exactly one rank
    assert L.n_shard * world == L.n
    names = [u.name for u in L.units]
    if module == "backbone":
        assert names == ["embed", "blocks_0", "blocks_1", "blocks_2", "norm"]   # FSDP units (vision_transformer.py:93,137)
    else:
        assert names == ["head"]


@pytest.mark.parametrize("world", [1, 2, 8])
def test_segment_tables_cover_each_tensor_once_with_its_multipliers(world):
    spec = backbone_spec(CFG)
    L, offsets, padded = build_layout("backbone", spec, world)
    mult = {n: lr_wd_multipliers("backbone", n, CFG) for n in offsets}
    covered = np.zeros(L.n, dtype=np.int32)
    for r in range(world):
        segs = L.shard_segments(r, mult)
        idx = L.full_to_shard_index(r)
        starts = [s[0] for s in segs] + [L.n_shard]
        assert starts == sorted(starts) and starts[0] == 0
        for (st, lr, wd, last), en in zip(segs, starts[1:]):
            full = idx[st:en]
            # all elements of a segment belong to one tensor whose multipliers match
            owner = [n for n in offsets if offsets[n] <= full[0] < offsets[n] + padded[n]]
            assert len(owner) == 1 and full[-1] < offsets[owner[0]] + padded[owner[0]]
            assert (lr, wd, last) == mult[owner[0]]
            covered[full] += 1
    assert (covered == 1).all()


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dinov3_jax.fsdp.runtime import Comm
        comm = Comm()
        spec = head_spec(CFG)
        L, offsets, padded = build_layout("dino_head", spec, world)
        torch.manual_seed(0)
        full = torch.randn(L.n)                                  # identical on all ranks
        shard = full[torch.from_numpy(L.full_to_shard_index(rank))]
        # all-gather of every unit range reproduces the full buffer
        out = torch.zeros(L.n)
        for u in L.units:
            for region in ("mat", "vec"):
                a, b = getattr(u, region)
                if b > a:
                    sa, sb = L.shard_range(u, region)
                    comm.all_gather(out[a:b], shard[sa:sb].contiguous())
        ok_gather = torch.equal(out, full)
        # reduce-scatter(mean) of rank-dependent gradients lands the mean slice in the shard layout
        g = full * (rank + 1)
        gs = torch.zeros(L.n_shard)
        for u in L.units:
            for region in ("mat", "vec"):
                a, b = getattr(u, region)
                if b > a:
                    sa, sb = L.shard_range(u, region)
                    comm.reduce_scatter_mean(gs[sa:sb], g[a:b].contiguous())
        want = (full * (sum(range(1, world + 1)) / world))[torch.from_numpy(L.full_to_shard_index(rank))]
        ok_rs = torch.allclose(gs, want, atol=1e-6)
        t = torch.tensor([float(rank + 1)]); comm.all_reduce_sum(t)
        m = torch.tensor([float(rank)]); comm.all_reduce_max(m)
        ret[rank] = (ok_gather, ok_rs, t.item(), m.item())
    finally:
        dist.destroy_process_group()


def _runtime_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dinov3_jax.engine.params import ModuleStore, backbone_spec
        from dinov3_jax.fsdp.runtime import Comm, FsdpRuntime
        st = ModuleStore("backbone", backbone_spec(CFG), CFG, "cpu", world=world, rank=rank)
        L = st.layout
        torch.manual_seed(0)
        full = torch.randn(L.n)
        idx = torch.from_numpy(L.full_to_shard_index(rank))
        for teacher, scale in ((False, 1.0), (True, -2.0)):
            (st.t_master if teacher else st.master).copy_(full[idx] * scale)
            (st.t_bf16_shard if teacher else st.bf16_shard).copy_((full[idx] * scale)[:L.n_mat_shard].to(torch.bfloat16))
        rt = FsdpRuntime(Comm(), {"backbone": st}, "cpu")
        rt.prefetch([("backbone", u, t) for t in (True, False) for u in L.units])
        for t in (True, False):
            for u in L.units:
                rt.acquire("backbone", u.name, t)
        ok = True
        for teacher, scale in ((False, 1.0), (True, -2.0)):
            ok &= torch.equal(st.t_vecs if teacher else st.vecs, full[L.n_mat:] * scale)
            ok &= torch.equal(st.t_bf16 if teacher else st.bf16, (full[:L.n_mat] * scale).to(torch.bfloat16))
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


def test_gloo_world2_runtime_prefetch_fills_the_compute_buffers():
    """FsdpRuntime.prefetch / acquire: per-unit matrix gathers + one vector all-gather and a permutation per module
    reproduce the single-GPU buffers for student and teacher."""
    world = 2
    ret = mp.Manager().dict()
    mp.spawn(_runtime_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert all(ret[r] for r in range(world))


def test_gloo_world2_gather_and_reduce_scatter():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    for r in range(world):
        ok_gather, ok_rs, s, m = ret[r]
        assert ok_gather and ok_rs and s == 3.0 and m == 1.0


@pytest.mark.parametrize("world", [2, 4, 8])
def test_push_reduce_scatter_addresses_cover_every_gradient_once(world, monkeypatch):
    """The push reduce-scatter (fsdp/runtime.py: scatter_spec for the GEMM epilogue + _push_ranges for the rest) must add
    every element of a unit's gradient exactly once into the shard slice that full_to_shard_index assigns to it.
    The D3_EP_SCATTER / d3_scatter_add_peers address rule (owner = g // shard, slot = g % shard) is emulated in numpy."""
    from dinov3_jax import ops
    from dinov3_jax.fsdp.runtime import FsdpRuntime
    spec = backbone_spec(CFG)
    L, offsets, padded = build_layout("backbone", spec, world)
    grad = torch.arange(1, L.n + 1, dtype=torch.float32)            # element i carries value i+1
    shards = [np.zeros(L.n_shard, dtype=np.float64) for _ in range(world)]
    base = [r * 10**9 for r in range(world)]                         # fake, disjoint "peer pointers" (byte addresses)

    def emulate(peers, off, shard, values):
        for i, v in enumerate(values):
            g = off + i
            r, slot = g // shard, g % shard
            byte = peers[r] + 4 * slot
            owner = next(k for k in range(world) if base[k] <= byte < base[k] + 10**9)
            shards[owner][(byte - base[owner]) // 4] += v

    class Store:
        pass
    st = Store()
    st.layout, st.grad = L, grad
    rt = FsdpRuntime.__new__(FsdpRuntime)
    rt.world, rt.push, rt.stores, rt._peer_ptrs = world, True, {"backbone": st}, {"backbone": base}
    monkeypatch.setattr(ops, "scatter_add_peers",
                        lambda src, peers, off, shard, alpha: emulate(peers, off, shard, (src.double() * alpha).tolist()))
    for u in L.units:
        fused = tuple(t for t in u.tensors if t.endswith(("mlp/Dense_1/kernel", "mlp/Dense_0/kernel", "attn/qkv/kernel")))
        for t in fused:                                              # what the GEMM epilogue would do for this tensor
            peers, off, shard = rt.scatter_spec("backbone", u.name, t)
            n = int(np.prod(dict((nm, sh) for nm, sh, _ in spec)[t]))
            emulate(peers, off, shard, grad[offsets[t]: offsets[t] + n].double().tolist())
        rt._push_ranges("backbone", u, fused)
    scale = 1.0 / world
    for r in range(world):
        idx = L.full_to_shard_index(r)
        want = grad.double().numpy()[idx]
        pad = np.ones(L.n, dtype=bool)
        for nm, sh, _ in spec:
            pad[offsets[nm]: offsets[nm] + int(np.prod(sh))] = False
        got = shards[r]
        fused_mask = np.zeros(L.n, dtype=bool)
        for nm, sh, _ in spec:
            if nm.endswith(("mlp/Dense_1/kernel", "mlp/Dense_0/kernel", "attn/qkv/kernel")):
                fused_mask[offsets[nm]: offsets[nm] + int(np.prod(sh))] = True
        # fused tensors were emulated unscaled, the pushed ranges carry 1/world; alignment padding of fused tensors is
        # never pushed (its gradient is identically zero)
        expect = np.where(fused_mask[idx], want, want * scale)
        expect = np.where(pad[idx] & _fused_padding(L, offsets, padded, spec)[idx], 0.0, expect)
        assert np.allclose(got, expect), r


def _fused_padding(L, offsets, padded, spec):
    m = np.zeros(L.n, dtype=bool)
    for nm, sh, _ in spec:
        if nm.endswith(("mlp/Dense_1/kernel", "mlp/Dense_0/kernel", "attn/qkv/kernel")):
            m[offsets[nm] + int(np.prod(sh)): offsets[nm] + padded[nm]] = True
    return m


def test_ac_compile_parallelize_policy(monkeypatch):
    """fsdp/ac_compile_parallelize.py:20-44: >= 2-D leaves are split on their largest divisible axis whatever their
    size, 1-D leaves never; the slices of all ranks tile the leaf."""
    from dinov3_jax.fsdp import ac_compile_parallelize as acp
    from dinov3_jax.fsdp.utils import Partitioned
    tree = {"k": torch.arange(6 * 8, dtype=torch.float32).reshape(6, 8), "bias": torch.arange(4096 * 4, dtype=torch.float32),
            "odd": torch.zeros(3, 5), "blk": {"cube": torch.arange(4 * 6 * 2, dtype=torch.float32).reshape(4, 6, 2)}}
    parts = []
    for r in range(2):
        monkeypatch.setattr(acp, "_axis_index", lambda name="dp", r=r: r)
        monkeypatch.setattr(acp, "_axis_size", lambda name="dp": 2)
        parts.append(acp.ac_compile_parallelize(tree, None, None))
    for p in parts:
        assert isinstance(p["k"], Partitioned) and p["k"].axis == 1            # 8 is the largest axis
        assert isinstance(p["blk"]["cube"], Partitioned) and p["blk"]["cube"].axis == 1
        assert not isinstance(p["bias"], Partitioned) and not isinstance(p["odd"], Partitioned)
    assert torch.equal(torch.cat([p["k"].value for p in parts], dim=1), tree["k"])
    assert torch.equal(torch.cat([p["blk"]["cube"].value for p in parts], dim=1), tree["blk"]["cube"])
