"""-m gpu: d3_koleo_topk_rows against the float64 statement of the distributed top-k KoLeo (tests/koleo_oracle.py).

Ranks are simulated on one GPU: the kernel runs once per rank on the same gathered matrix, into one dx (the sum over
ranks in rank order, what the exchange of engine/koleo.py adds up), and Sigma_r L_r with its gradient comes from
float64 autograd.  Neighbour lists are compared exactly on the rows whose k-th and (k+1)-th dots are separated by
more than fp32 can blur (1e-5); the loss (1e-5 relative) and the gradient (1e-4 of its largest entry) are compared on
the kernel's own lists.  Then the engine: koleo_distributed with topk 1 against the default engine, topk 4 against
the oracle, the local DINO weight, the default engine against the bits of the commit before these options
(tests/golden/koleo_default_step.npz), and two ranks on two GPUs (skipped with fewer).  Also on the GPU: exact ties
go to the lower index, a NaN class token keeps every neighbour index inside the group, and KoLeoLossDistributed with
topk > 1 and loss groups.
"""
import dataclasses
import os
import socket

import numpy as np
import pytest
import torch

import koleo_oracle as oracle

pytestmark = pytest.mark.gpu

EPS = 1e-8
DS = (384, 1024, 1536, 4096)


def _run(x, world, B, G, k, w_metric=1.0, w_grad=1.0):
    """(per-rank metrics, dx summed over ranks in rank order, per-rank neighbour lists) from the kernel."""
    from dinov3_jax import ops
    N, D = x.shape
    scratch = ops.koleo_topk_scratch(N, D, B, k, x.device)
    dx = torch.zeros_like(x)
    mets, lists = [], []
    for r in range(world):
        g0, gn = oracle.group_of(r, world, B, G)
        met = torch.zeros(1, device=x.device)
        ops.koleo_topk(x, (g0, gn), r * B, B, k, scratch, met, dx, w_metric, w_grad, EPS)
        mets.append(met)
        lists.append(scratch[N * D + N:N * D + N + B * k].view(torch.int32).view(B, k).cpu().numpy().astype(np.int64))
    torch.cuda.synchronize()
    return torch.cat(mets).cpu(), dx, lists


def _check(x, world, B, G, k):
    mets, dx, lists = _run(x, world, B, G, k)
    xc = x.cpu().double()
    losses, grad, _ = oracle.loss_and_grad(xc, world, B, G, k, EPS, nbrs=lists)
    for r in range(world):
        g0, gn = oracle.group_of(r, world, B, G)
        want = oracle.neighbours(xc, r * B, B, g0, gn, k, EPS)
        sep = oracle.margins(xc, r * B, B, g0, gn, k, EPS) > 1e-5
        assert sep.mean() > 0.5, "inputs not separated enough to check the lists"
        assert (np.sort(lists[r][sep], 1) == np.sort(want[sep], 1)).all(), r
        assert ((lists[r] >= g0) & (lists[r] < g0 + gn) & (lists[r] != (r * B + np.arange(B))[:, None])).all()
    assert torch.allclose(mets.double(), losses, rtol=1e-5, atol=0), (mets, losses)
    err = (dx.cpu().double() - grad).abs().max().item()
    assert err <= 1e-4 * grad.abs().max().item(), err


CASES = [(w, B, k, G) for w in (1, 2, 4, 8) for B in (2, 8, 64) for k in (1, 2, 4, 16) for G in (None, "2B")
         if (G is None or 2 <= w) and k <= (w * B if G is None else 2 * B) - 1]


@pytest.mark.parametrize("world,B,k,G", CASES)
def test_simulated_ranks_match_float64_autograd(world, B, k, G):
    G = 2 * B if G == "2B" else G
    i = CASES.index((world, B, k, None if G is None else "2B"))
    D = DS[i % len(DS)]                                       # every D over the cases, every case one D
    torch.manual_seed(i)
    x = torch.randn(world * B, D, device="cuda") * (1.0 + torch.rand(world * B, 1, device="cuda"))
    _check(x, world, B, G, k)


def test_every_width_at_one_case():
    for j, D in enumerate(DS):
        torch.manual_seed(100 + j)
        _check(torch.randn(4 * 8, D, device="cuda"), 4, 8, 16, 4)


def test_a_65536_row_group():
    N, D, B, k = 65536, 384, 64, 4
    torch.manual_seed(7)
    x = torch.randn(N, D, device="cuda")
    from dinov3_jax import ops
    row0 = 40000
    met, dx = torch.zeros(1, device="cuda"), torch.zeros_like(x)
    scratch = ops.koleo_topk_scratch(N, D, B, k, "cuda")
    ops.koleo_topk(x, (0, N), row0, B, k, scratch, met, dx, 1.0, 1.0, EPS)
    lists = scratch[N * D + N:N * D + N + B * k].view(torch.int32).view(B, k).cpu().numpy().astype(np.int64)
    xc = x.cpu().double()
    want = oracle.neighbours(xc, row0, B, 0, N, k, EPS)
    sep = oracle.margins(xc, row0, B, 0, N, k, EPS) > 1e-5
    assert sep.mean() > 0.5 and (np.sort(lists[sep], 1) == np.sort(want[sep], 1)).all()
    xd = xc.clone().requires_grad_(True)
    L = oracle.rank_loss(xd, row0, B, k, lists, EPS)
    L.backward()
    assert abs(met.item() - L.item()) <= 1e-5 * abs(L.item())
    err = (dx.cpu().double() - xd.grad).abs().max().item()
    assert err <= 1e-4 * xd.grad.abs().max().item()


def test_reruns_are_byte_identical():
    torch.manual_seed(3)
    x = torch.randn(8 * 64, 1024, device="cuda")
    a = _run(x, 8, 64, None, 16)
    b = _run(x, 8, 64, None, 16)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all((p == q).all() for p, q in zip(a[2], b[2]))


def test_topk_one_on_one_rank_agrees_with_the_plain_kernel():
    from dinov3_jax import ops
    torch.manual_seed(5)
    B, D = 64, 1024
    x = torch.randn(B, D, device="cuda")
    mets, dx, _ = _run(x, 1, B, None, 1, w_metric=0.5, w_grad=0.1)
    met0, dx0 = torch.zeros(1, device="cuda"), torch.zeros_like(x)
    e = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device="cuda")
    ops.koleo_fwd_bwd(x, e(B, D), e(B), e(B, dt=torch.int32), e(B), met0, dx0, 0.5, 0.1)
    assert abs(mets.item() - met0.item()) <= 1e-6 * abs(met0.item())
    assert (dx - dx0).abs().max().item() <= 1e-6 * dx0.abs().max().item()


def test_kernel_arguments_are_checked_before_launch():
    from dinov3_jax import _native, ops
    x = torch.randn(8, 16, device="cuda")
    s = ops.koleo_topk_scratch(8, 16, 4, 2, "cuda")
    met, dx = torch.zeros(1, device="cuda"), torch.zeros_like(x)
    with pytest.raises(_native.NativeError, match="topk"):
        ops.koleo_topk(x, (0, 2), 0, 1, 2, s, met, dx, 1.0, 1.0)
    with pytest.raises(_native.NativeError, match="scratch"):
        ops.koleo_topk(x, (0, 8), 0, 4, 2, s[:-1], met, dx, 1.0, 1.0)
    assert met.item() == 0.0 and dx.abs().sum().item() == 0.0


def test_duplicate_rows_tie_to_the_lower_index_on_the_gpu():
    torch.manual_seed(11)
    D = 384
    b = torch.randn(D)
    x = torch.randn(12, D)
    x[1] = x[2] = x[3] = b                       # three identical rows: their dots with any row are the same bits
    x[0] = b + 0.01 * torch.randn(D)             # its three nearest are rows 1, 2 and 3, in a three-way tie
    mets, dx, lists = _run(x.cuda(), 3, 4, None, 3)
    xc = x.double()
    for r in range(3):
        assert (lists[r] == oracle.neighbours(xc, r * 4, 4, 0, 12, 3)).all(), r
    assert lists[0][0].tolist() == [1, 2, 3] and lists[0][1][:2].tolist() == [2, 3] and lists[0][2][:2].tolist() == [1, 3]


def test_a_nan_row_gives_a_nan_loss_and_neighbours_inside_the_group():
    """A non-finite class token (a diverging run) makes its dots NaN; they rank below every number, so every index
    stays inside the group: the loss of the rank that owns the row is NaN, the other rank's is finite."""
    torch.manual_seed(12)
    world, B, k = 2, 8, 4
    x = torch.randn(world * B, 384, device="cuda")
    x[3, 7] = float("nan")
    x[5, 0] = float("inf")                       # xn = inf * 0 = NaN as well
    mets, dx, lists = _run(x, world, B, None, k)
    for r in range(world):
        assert ((lists[r] >= 0) & (lists[r] < world * B) & (lists[r] != (r * B + torch.arange(B).numpy())[:, None])).all()
        assert not ({3, 5} & set(lists[r][[i for i in range(B) if r * B + i not in (3, 5)]].reshape(-1).tolist()))
    assert torch.isnan(mets[0]) and torch.isfinite(mets[1])
    assert torch.isfinite(dx[B:]).all()


def test_koleo_loss_distributed_class_with_topk_and_groups():
    from dinov3_jax.loss import KoLeoLoss, KoLeoLossDistributed
    torch.manual_seed(13)
    x = torch.randn(16, 384)
    for k in (2, 5):
        got = KoLeoLossDistributed(topk=k)(x.cuda()).item()
        want = oracle.loss_and_grad(x.double(), 1, 16, None, k, EPS)[0].item()
        assert abs(got - want) <= 1e-5 * abs(want), k
    # topk 1 with the whole batch as the group is the plain KoLeo
    assert abs(KoLeoLossDistributed(topk=1, loss_group_size=16)(x.cuda()).item() - KoLeoLoss()(x.cuda()).item()) < 1e-5
    for kw in (dict(topk=1, loss_group_size=12), dict(topk=16)):
        with pytest.raises(ValueError):
            KoLeoLossDistributed(**kw)(x.cuda())
    with pytest.raises(ValueError):
        KoLeoLossDistributed(topk=17)


def test_default_engine_computes_the_bits_of_the_commit_before_it():
    """tests/golden/koleo_default_step.npz holds the metrics and the sha256 of every gradient and updated parameter of
    one default step, written by the library before distributed KoLeo and the local-loss weight went in."""
    import importlib.util
    here = os.path.dirname(os.path.abspath(__file__))
    spec = importlib.util.spec_from_file_location("make_koleo_default_golden",
                                                  os.path.join(here, "golden", "make_koleo_default_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    g = np.load(os.path.join(here, "golden", "koleo_default_step.npz"))
    mnames, mvals, names, digests = gen.step_digest()
    assert mnames == g["metric_names"].tolist() and mvals == g["metrics"].tolist()
    assert names == g["tensor_names"].tolist()
    bad = [n for n, d, w in zip(names, digests, g["sha256"].tolist()) if d != w]
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ the engine
HYPER = dict(lr=0.0, wd=0.0, last_layer_lr=0.0, momentum=1.0, teacher_temp=0.05)


def _engine(B, seed=0, comm=None, device="cuda", **kw):
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg = tiny_cfg()
    batch = synthetic_batch(cfg, B, seed)
    ecfg = dataclasses.replace(from_oracle_cfg(cfg), **kw)
    eng = Engine(ecfg, B, device=device, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1), comm=comm)
    eng.params.load_reference_tree(init_params(cfg, 0, perturb=0.05))
    return eng, batch


def _step(eng, batch, **kw):
    eng.train_step(batch, **HYPER, **kw)
    torch.cuda.synchronize()
    return eng.read_metrics(), {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}


def test_engine_topk_one_reproduces_the_default_engine():
    m0, g0 = _step(*_engine(8))
    m1, g1 = _step(*_engine(8, koleo_distributed=True))
    for k in ("koleo_loss", "total_loss", "dino_local_crops_loss", "ibot_loss"):
        assert abs(m1[k] - m0[k]) <= 1e-5 * abs(m0[k]), k
    num = sum(((g1[k] - g) ** 2).sum() for k, g in g0.items())
    den = sum((g ** 2).sum() for g in g0.values())
    assert float(torch.sqrt(num / den)) < 1e-4


def test_engine_topk_four_equals_the_oracle():
    B, k = 8, 4
    eng, batch = _engine(B, koleo_distributed=True, koleo_topk=k, dino_loss_weight=0.0, ibot_loss_weight=0.0)
    m, _ = _step(eng, batch)
    want, L = 0.0, []
    for c in range(2):
        x = eng.cls_f32[c * B:(c + 1) * B].cpu().double()
        losses, grad, _ = oracle.loss_and_grad(x, 1, B, None, k, EPS)
        want += losses.item() / 2
        # with the DINO and iBOT weights at 0 the class-token gradient is the KoLeo term alone
        got = eng.h_s_dino.dA0[c * B:(c + 1) * B].cpu().double()
        assert (got - 0.1 * grad).abs().max().item() <= 1e-4 * 0.1 * grad.abs().max().item()
    assert abs(m["koleo_loss"] - want) <= 1e-5 * abs(want)


def test_local_dino_weight_scales_only_the_local_term():
    w_grads, mets = {}, {}
    B = 8
    for w in (0.0, 0.5, 1.0):
        eng, batch = _engine(B, koleo_loss_weight=0.0, ibot_loss_weight=0.0)
        base = eng.ce_dino[3].clone()
        mets[w], w_grads[w] = _step(eng, batch, dino_local_loss_weight=w)
        ng = eng.cfg.n_global * B                  # global rows first, then the local crops' rows
        assert torch.equal(eng.ce_dino[3][:ng], base[:ng])
        assert torch.equal(eng.ce_dino[3][ng:], base[ng:] * w) and (base[ng:] > 0).all()
    for w, m in mets.items():
        assert m["dino_local_loss_weight"] == w
        assert m["dino_local_crops_loss"] == mets[1.0]["dino_local_crops_loss"]     # the metric is the raw term
    l_scale = 16 / 18
    assert abs((mets[1.0]["total_loss"] - mets[0.5]["total_loss"])
               - 0.5 * l_scale * mets[1.0]["dino_local_crops_loss"]) < 1e-5
    # g(w) = g_global + w g_local: the local part at 0.5 is half the local part at 1
    num = sum(((w_grads[0.5][k] - w_grads[0.0][k]) - 0.5 * (w_grads[1.0][k] - w_grads[0.0][k])).pow(2).sum()
              for k in w_grads[0.0])
    den = sum((0.5 * (w_grads[1.0][k] - w_grads[0.0][k])).pow(2).sum() for k in w_grads[0.0])
    # the local crops' token rows scale by a power of two exactly; only the fp32 sums over rows round differently
    assert float(den) > 0 and float(torch.sqrt(num / den)) < 1e-4


def test_default_engine_reports_weight_one_and_keeps_its_tables():
    eng, batch = _engine(4)
    wg = eng.ce_dino[3].clone()
    m, _ = _step(eng, batch)
    assert m["dino_local_loss_weight"] == 1.0 and torch.equal(eng.ce_dino[3], wg)
    eng.set_dino_local_loss_weight(0.25)
    eng.set_dino_local_loss_weight(1.0)
    assert torch.equal(eng.ce_dino[3], wg)


# ------------------------------------------------------------------------------------------------ two GPUs
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _two_rank_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from dinov3_jax import _native
        from dinov3_jax.fsdp.runtime import Comm
        _native.init(rank)
        B, k = 4, 3
        eng, batch = _engine(B, seed=rank, comm=Comm(), device=f"cuda:{rank}", koleo_distributed=True, koleo_topk=k,
                             dino_loss_weight=0.0, ibot_loss_weight=0.0)
        m, _ = _step(eng, batch)
        ret[rank] = (m["koleo_loss"], eng.cls_f32[:2 * B].cpu(), eng.h_s_dino.dA0[:2 * B].cpu())
    finally:
        dist.destroy_process_group()


def test_two_ranks_on_two_gpus_equal_the_single_process_oracle():
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    world, B, k = 2, 4, 3
    ret = mp.Manager().dict()
    mp.spawn(_two_rank_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    want = 0.0
    for c in range(2):
        x = torch.cat([ret[r][1][c * B:(c + 1) * B] for r in range(world)]).double()
        losses, grad, _ = oracle.loss_and_grad(x, world, B, None, k, EPS)
        want += losses.mean().item() / 2                     # mean over crops, then over ranks
        for r in range(world):
            got = ret[r][2][c * B:(c + 1) * B].double()
            assert (got - 0.1 * grad[r * B:(r + 1) * B]).abs().max().item() <= 1e-4 * 0.1 * grad.abs().max().item()
    assert abs(ret[0][0] - want) <= 1e-5 * abs(want) and ret[0][0] == ret[1][0]
