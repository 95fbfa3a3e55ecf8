"""Distributed top-k KoLeo and the DINO local-loss weight schedule without a GPU: the float64 oracle
(tests/koleo_oracle.py) on hand-computed cases, `linear_warmup_cosine_decay` at its boundaries, the mapping of the
7B recipes' `dino` blocks and its refusals, the host-side argument checks of d3_koleo_topk_rows, what ptxas makes of
csrc/koleo.cu, and the rank-order exchange of the gradient slabs over a gloo group."""
import ctypes as C
import math
import os
import re
import socket
import subprocess

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import koleo_oracle as oracle
from dinov3_jax.configs import DinoV3SetupArgs, setup_config
from dinov3_jax.engine.config import EngineConfig, config_from_reference_cfg


# ------------------------------------------------------------------------------------------------ oracle by hand
def test_duplicate_rows_tie_to_the_lower_index():
    x = torch.tensor([[1.0, 0.0], [0.0, 1.0], [0.0, 1.0], [-1.0, 0.0]], dtype=torch.float64)
    nbr = oracle.neighbours(x, 0, 4, 0, 4, 2)
    assert nbr[0].tolist() == [1, 2]          # dots 0, 0, -1: the tie 1 / 2 goes to 1
    assert nbr[1].tolist() == [2, 0]          # its duplicate first, then the tie 0 / 3 goes to 0
    assert nbr[2].tolist() == [1, 0]
    assert nbr[3].tolist() == [1, 2]
    assert oracle.neighbours(x, 0, 4, 0, 4, 1)[:, 0].tolist() == [1, 2, 1, 1]


def test_topk_one_on_one_rank_is_the_plain_koleo():
    from oracle.losses import koleo_loss
    torch.manual_seed(0)
    x = torch.randn(12, 16, dtype=torch.float64)
    nbr = oracle.neighbours(x, 0, 12, 0, 12, 1)
    assert abs(oracle.rank_loss(x, 0, 12, 1, nbr).item() - koleo_loss(x).item()) < 1e-12


def test_orthogonal_rows_with_two_neighbours():
    x = torch.eye(4, dtype=torch.float64) * 3.0
    nbr = oracle.neighbours(x, 0, 4, 0, 4, 2)
    assert nbr.tolist() == [[1, 2], [0, 2], [0, 1], [0, 1]]     # every dot is 0: the lowest other indices
    want = -math.log(math.sqrt(2) * 3 / (3 + 1e-8) + 2e-8)
    assert abs(oracle.rank_loss(x, 0, 4, 2, nbr).item() - want) < 1e-12


def test_a_rank_searches_only_its_own_group():
    world, B, G = 4, 2, 4
    assert [oracle.group_of(r, world, B, G) for r in range(world)] == [(0, 4), (0, 4), (4, 4), (4, 4)]
    assert oracle.group_of(3, world, B, None) == (0, 8)
    x = torch.zeros(8, 3, dtype=torch.float64)
    x[:, 2] = 1.0
    x[4, 0] = 0.01                           # row 4's nearest overall is row 0 (identical direction) ...
    x[0, 0] = 0.01
    x[5, 1] = 0.5
    x[6, 1] = 1.0
    x[7, 0] = -1.0
    assert oracle.neighbours(x, 4, 2, 0, 8, 1)[0, 0] == 0
    assert oracle.neighbours(x, 4, 2, 4, 4, 1)[0, 0] == 5     # ... but its group is rows 4..7
    losses, grad, lists = oracle.loss_and_grad(x + 0.001 * torch.arange(24.0).reshape(8, 3).double(), world, B, G, 2)
    for r in range(world):
        g0, gn = oracle.group_of(r, world, B, G)
        assert ((lists[r] >= g0) & (lists[r] < g0 + gn)).all()
    assert losses.shape == (world,) and grad.shape == (8, 3)


# ------------------------------------------------------------------------------------------------ schedule
def test_linear_warmup_cosine_decay_boundaries():
    from dinov3_jax.train.cosine_lr_scheduler import linear_warmup_cosine_decay
    s = linear_warmup_cosine_decay(start=0.0, peak=1.0, end=0.25, warmup_iterations=4, total_iterations=12,
                                   cosine_iterations=5).schedule
    assert len(s) == 12
    assert s[:4].tolist() == [0.0, 0.25, 0.5, 0.75]                 # endpoint=False: the peak is not reached
    assert s[4] == 1.0 and s[8] == 0.25                             # the cosine starts at the peak, ends at end
    assert abs(s[6] - (0.25 + 0.75 * 0.5)) < 1e-15                  # its midpoint
    assert s[9:].tolist() == [0.25] * 3                             # then end
    d = linear_warmup_cosine_decay(1.0, 1.0, 0.5, 2, 6).schedule    # cosine defaults to total - warmup
    assert d[:3].tolist() == [1.0, 1.0, 1.0] and d[-1] == 0.5 and len(d) == 6
    assert linear_warmup_cosine_decay(0.5, 0.5, 0.5, 0, 7, 0).schedule.tolist() == [0.5] * 7
    with pytest.raises(ValueError):
        linear_warmup_cosine_decay(0.0, 1.0, 0.0, 5, 8, 4)


# ------------------------------------------------------------------------------------------------ 7B recipes
# The `dino` blocks (and the gram schedules) of DINOv3's three 7B training recipes, as shipped.
RECIPES = {
    "dinov3_vit7b16_pretrain": ("""
dino: {loss_weight: 1.0, global_ignore_diagonal: true, head_n_prototypes: 262144, head_bottleneck_dim: 512,
  head_norm_last_layer: false, head_nlayers: 3, head_hidden_dim: 8192, koleo_loss_weight: 0.1,
  koleo_loss_distributed: false, koleo_topk: 1, koleo_distributed_replicas: 0,
  koleo_distributed_loss_group_size: null, force_weight_norm: false}
train: {batch_size_per_gpu: 16, OFFICIAL_EPOCH_LENGTH: 1000}
optim: {epochs: 1000}
"""),
    "dinov3_vit7b16_gram_anchor": ("""
dino: {loss_weight: 1.0, global_ignore_diagonal: true, head_n_prototypes: 262144, head_bottleneck_dim: 512,
  head_norm_last_layer: false, head_nlayers: 3, head_hidden_dim: 8192, koleo_loss_weight: 0.1,
  koleo_loss_distributed: false, koleo_topk: 1, koleo_distributed_replicas: 0,
  koleo_distributed_loss_group_size: null, koleo_distributed_loss_group_data: true, force_weight_norm: false,
  reweight_dino_local_loss: true,
  local_loss_weight_schedule: {start: 1, peak: 1, end: 0.5, warmup_epochs: 1000, cosine_epochs: 1}}
gram: {use_loss: true, ema_teacher: true,
  loss_weight_schedule: {start: 0, peak: 0, end: 2.0, warmup_epochs: 1000, cosine_epochs: 1}}
train: {batch_size_per_gpu: 16, OFFICIAL_EPOCH_LENGTH: 1000}
optim: {epochs: 1200}
"""),
    "dinov3_vit7b16_high_res_adapt": ("""
dino: {loss_weight: 1.0, global_ignore_diagonal: true, head_n_prototypes: 262144, head_bottleneck_dim: 512,
  head_norm_last_layer: false, head_nlayers: 3, head_hidden_dim: 8192, koleo_loss_weight: 0.1,
  koleo_loss_distributed: true, koleo_topk: 1, koleo_distributed_replicas: 0,
  koleo_distributed_loss_group_size: 16, force_weight_norm: false, reweight_dino_local_loss: true,
  local_loss_weight_schedule: {start: 0.5, peak: 0.5, end: 0.5, warmup_epochs: 0, cosine_epochs: 0},
  koleo_distributed_loss_group_data: true}
gram: {use_loss: true, ema_teacher: true,
  loss_weight_schedule: {start: 1.5, peak: 1.5, end: 1.5, warmup_epochs: 0, cosine_epochs: 0}}
train: {batch_size_per_gpu: 8, OFFICIAL_EPOCH_LENGTH: 1000}
optim: {epochs: 30}
"""),
}


def _cfg(tmp_path, text, *opts):
    p = tmp_path / "recipe.yaml"
    p.write_text(text)
    return setup_config(DinoV3SetupArgs(config_file=str(p), opts=list(opts)))


@pytest.mark.parametrize("name", sorted(RECIPES))
def test_the_7b_recipes_dino_blocks_map(tmp_path, name):
    from dinov3_jax.train import SSLMetaArch
    cfg = _cfg(tmp_path, RECIPES[name])
    e = config_from_reference_cfg(cfg)
    m = SSLMetaArch(cfg)
    if name == "dinov3_vit7b16_high_res_adapt":
        assert (e.koleo_distributed, e.koleo_topk, e.koleo_group_size) == (True, 1, 16)
        assert m.dino_local_loss_schedule.schedule.tolist() == [0.5] * 30000
        assert m.gram_loss_schedule.schedule.tolist() == [1.5] * 30000
    else:
        assert (e.koleo_distributed, e.koleo_topk, e.koleo_group_size) == (False, 1, None)
    if name == "dinov3_vit7b16_gram_anchor":
        s = m.dino_local_loss_schedule.schedule
        assert len(s) == 1_200_000 and s[0] == 1.0 and s[999_999] == 1.0 and s[1_000_000] == 1.0
        assert s[1_000_999] == 0.5 and s[-1] == 0.5 and 0.5 < s[1_000_500] < 1.0
        g = m.gram_loss_schedule.schedule
        assert g[999_999] == 0.0 and g[1_000_999] == 2.0 and g[-1] == 2.0
    if name == "dinov3_vit7b16_pretrain":
        assert m.dino_local_loss_schedule is None and m.gram_loss_schedule is None
        assert e == config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=[
            "dino.head_n_prototypes=262144", "dino.head_bottleneck_dim=512", "dino.head_hidden_dim=8192",
            "train.batch_size_per_gpu=16"])))


def test_the_defaults_select_the_plain_koleo():
    e = config_from_reference_cfg(setup_config(DinoV3SetupArgs()))
    assert (e.koleo_distributed, e.koleo_topk, e.koleo_group_size) == (False, 1, None)
    assert (EngineConfig().koleo_distributed, EngineConfig().koleo_topk, EngineConfig().koleo_group_size) == \
        (False, 1, None)


def test_refusals(tmp_path):
    on = ["dino.koleo_loss_distributed=true", "train.batch_size_per_gpu=8"]
    ok = config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=on + ["dino.koleo_distributed_loss_group_size=32",
                                                                             "dino.koleo_topk=16"])))
    assert (ok.koleo_group_size, ok.koleo_topk) == (32, 16)
    bad = [(["dino.koleo_distributed_loss_group_size=12"], ValueError, "multiple of"),
           (["dino.koleo_distributed_loss_group_data=false"], NotImplementedError, "group_data"),
           (["dino.koleo_distributed_loss_group_size=8", "dino.koleo_topk=8"], ValueError, "koleo_topk 8"),
           (["dino.koleo_topk=17"], ValueError, "koleo_topk 17"),
           (["dino.koleo_topk=0"], ValueError, "koleo_topk 0"),
           (["dino.koleo_distributed_replicas=2"], ValueError, "replicas")]
    for extra, exc, msg in bad:
        with pytest.raises(exc, match=msg):
            config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=on + extra)))
    with pytest.raises(ValueError, match="koleo_loss_distributed"):
        config_from_reference_cfg(setup_config(DinoV3SetupArgs(opts=["dino.koleo_topk=2"])))
    from dinov3_jax.engine.koleo import ranks_per_group
    assert ranks_per_group(8, 8, None, 1) == 8 and ranks_per_group(8, 8, 16, 4) == 2 and ranks_per_group(1, 4, None, 3) == 1
    for args, msg in (((8, 8, 24, 1), "divide"), ((4, 8, 12, 1), "multiple"), ((1, 4, None, 4), "koleo_topk 4"),
                      ((2, 4, 4, 4), "koleo_topk 4")):
        with pytest.raises(ValueError, match=msg):
            ranks_per_group(*args)


# ------------------------------------------------------------------------------------------------ host-side checks
def test_kernel_arguments_are_checked_on_the_host():
    """Every check comes before any CUDA call, so it answers without a device."""
    from dinov3_jax import _native
    lib = _native.lib()
    fake = C.c_void_p(256)
    f = lambda *a: lib.d3_koleo_topk_rows(*a)
    # x, N, D, g0, gn, row0, B, topk, eps, w_metric, w_grad, scratch, scratch_floats, metric, dx, stream
    good = [fake, 8, 16, 0, 8, 0, 4, 2, 1e-8, 1.0, 1.0, fake, 8 * 16 + 8 + 2 * 4 * 2, fake, fake, None]
    cases = [({2: 6}, b"multiple of 4"), ({2: 8192}, b"multiple of 4"), ({1: 1}, b"N >= 2"),
             ({3: 2, 4: 7}, b"group"), ({4: 1}, b"group"), ({5: 6}, b"local rows"), ({6: 0}, b"local rows"),
             ({3: 4, 4: 4, 5: 0}, b"local rows"), ({7: 0}, b"topk"), ({7: 17}, b"topk"), ({4: 4, 7: 4}, b"topk"),
             ({0: None}, b"null"), ({14: None}, b"null"), ({0: C.c_void_p(260)}, b"16-byte"),
             ({12: 8 * 16 + 8 + 2 * 4 * 2 - 1}, b"scratch")]
    for change, msg in cases:
        a = list(good)
        for k, v in change.items():
            a[k] = v
        assert f(*a) == -1 and msg in lib.d3_last_error(), (change, lib.d3_last_error())


# ------------------------------------------------------------------------------------------------ ptxas
def test_koleo_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert "koleo.cu" in b.SOURCES
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", "koleo.cu"), "-o",
                                       str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    seen = set()
    for name, stack, st, ld in props:
        if "koleo_topk" in name:
            seen.add(name)
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # norm, scan, loss, backward, metric
    assert len(seen) == 5, sorted(seen)


# ------------------------------------------------------------------------------------------------ exchange (gloo)
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _exchange_worker(rank, world, port, G, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dinov3_jax.engine.koleo import DistributedKoLeo
        from dinov3_jax.fsdp.runtime import Comm
        B, D, ng = 2, 4, 2
        k = DistributedKoLeo(Comm(), B, D, ng, 1, G, "cpu")
        R = k.R
        # rank r's contribution to gathered row b of group member m, crop c: a value naming all four
        for c in range(ng):
            for m in range(R):
                for b in range(B):
                    k.dxg[c, m * B + b] = 1000 * rank + 100 * c + 10 * m + b
        got = [k.exchange(c).clone() for c in range(ng)]
        g0 = (rank // R) * R
        ok = True
        for c in range(ng):
            for r in range(R):                  # slab r comes from group member r (global rank g0 + r), in rank order
                want = torch.tensor([1000 * (g0 + r) + 100 * c + 10 * (rank - g0) + b for b in range(B)],
                                    dtype=torch.float32)[:, None].expand(B, D)
                ok &= torch.equal(got[c][r], want)
        ret[rank] = (R, bool(ok))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,G", [(2, None), (4, 4)])
def test_gloo_exchange_returns_every_slab_to_its_owner_in_rank_order(world, G):
    """DistributedKoLeo.exchange over gloo: rank q receives, in rank order, the dx rows of q from every member of its
    loss group (world 4, G = 2 images per rank x 2 ranks: two groups built with new_group)."""
    ret = mp.Manager().dict()
    mp.spawn(_exchange_worker, args=(world, _free_port(), G, ret), nprocs=world, join=True)
    R = world if G is None else G // 2
    assert all(ret[r] == (R, True) for r in range(world)), dict(ret)
