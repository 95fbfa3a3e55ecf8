"""-m gpu: DINO and iBOT heads of different sizes through the engine.

  * the loss terms against the reference's SSLMetaArch.__call__ run with two head geometries (heads_vectors.npz);
  * a tiny step against the fp32 oracle, with Sinkhorn and with softmax centering;
  * bit-reproducibility, and explicit ibot_* sizes equal to the DINO head's give the bits of unset ones;
  * the DINOv3 recipe heads (262 144 / 98 304 prototypes, hidden 8192 / 4096, bottleneck 512 / 384) at ViT-L width;
  * checkpoint round trip, do_train, and the 2-GPU FSDP step (skipped on one GPU).

Tolerances are those of test_engine_gpu.py: loss terms 1e-3 relative (5e-3 against the peaky golden fixture),
gradients 3e-2 norm-wise globally and 6e-2 per tensor.
"""
import dataclasses
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

HYPER = dict(lr=1e-3, wd=0.04, last_layer_lr=5e-4, momentum=0.99, teacher_temp=0.05)
IBOT = (136, 96, 48)          # (K, hidden, bottleneck) of the iBOT head next to the DINO head of _tiny()


def _tiny():
    from oracle import tiny_cfg
    return tiny_cfg(n_prototypes=264, head_hidden=136, head_bottleneck=40, layerscale=0.5)


def _with_ibot(ecfg, ibot=IBOT):
    return dataclasses.replace(ecfg, ibot_n_prototypes=ibot[0], ibot_head_hidden=ibot[1], ibot_head_bottleneck=ibot[2])


def _params(cfg, seed, ibot=IBOT):
    """Oracle parameters with the DINO head at cfg's sizes and the iBOT head at `ibot`."""
    from oracle.model import init_params
    P = init_params(cfg, seed, perturb=0.05)
    Pi = init_params(dataclasses.replace(cfg, n_prototypes=ibot[0], head_hidden=ibot[1], head_bottleneck=ibot[2]),
                     seed + 100, perturb=0.05)
    P.update({k: v for k, v in Pi.items() if "_ibot_head/" in k})
    return P


def _grad_check(grads_e, grads, grad_tol=3e-2, tensor_tol=6e-2):
    num = sum(((grads_e[k].reshape(g.shape) - g) ** 2).sum() for k, g in grads.items())
    den = sum((g ** 2).sum() for g in grads.values())
    assert float(torch.sqrt(num / den)) < grad_tol
    gmax = max(float(g.norm()) for g in grads.values())
    for k, g in grads.items():
        if float(g.norm()) < 1e-3 * gmax:
            continue
        e = float((grads_e[k].reshape(g.shape) - g).norm() / g.norm())
        assert e < tensor_tol, (k, e)


@pytest.mark.parametrize("case", ["a", "c"])
def test_engine_loss_against_reference_meta_arch_golden_with_distinct_heads(case):
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from test_head_dims_cpu import heads_case, heads_golden
    G = heads_golden()
    cfg, ibot, P, batch, temp = heads_case(G, case, dtype=torch.float32)
    B = batch["global_batch_size"]
    batch["collated_global_crops"] = batch["collated_global_crops"].to(torch.bfloat16)
    batch["collated_local_crops"] = batch["collated_local_crops"].to(torch.bfloat16)
    eng = Engine(_with_ibot(from_oracle_cfg(cfg), ibot), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    eng.params.load_reference_tree(P)
    eng.set_batch(batch)
    eng.forward_backward(temp)
    torch.cuda.synchronize()
    met = eng.read_metrics()
    tol = 5e-3
    want = float(G[f"ssl_{case}_loss"])
    assert abs(met["total_loss"] - want) < tol * abs(want), (met["total_loss"], want)
    for k in ("dino_local_crops_loss", "dino_global_crops_loss", "ibot_loss"):
        w = float(G[f"ssl_{case}_metric/{k}"])
        assert abs(met[k] - w) < tol * abs(w), (k, met[k], w)
    w = float(G[f"ssl_{case}_metric/koleo_loss"])
    assert abs(met["koleo_loss"] - w) < 2e-2 * max(abs(w), 0.05)


def test_tiny_step_with_distinct_heads_matches_oracle():
    """DINO head K = 264 / hidden 136 / bottleneck 40, iBOT head 136 / 96 / 48: the joint Sinkhorn buffers hold the
    two heads at offsets 0 and 264."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle.batch import synthetic_batch
    from oracle.step import init_opt_state, train_step
    cfg, B = _tiny(), 4
    P = _params(cfg, 0)
    batch = synthetic_batch(cfg, B, 0)
    eng = Engine(_with_ibot(from_oracle_cfg(cfg)), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    assert eng.sk_ibot.off == 264 and eng.sk_mx2.numel() == 264 + 136
    eng.params.load_reference_tree(P)
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    grads_e = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
    eng.optimizer_step(HYPER["lr"], HYPER["wd"], HYPER["last_layer_lr"], HYPER["momentum"])
    torch.cuda.synchronize()
    met = eng.read_metrics()
    _, _, loss, m, grads = train_step(P, init_opt_state(P), batch, cfg, **HYPER)
    assert abs(met["total_loss"] - loss.item()) <= 1e-3 * abs(loss.item())
    for k in ("dino_local_crops_loss", "dino_global_crops_loss", "ibot_loss"):
        assert abs(met[k] - float(m[k])) <= 1e-3 * abs(float(m[k])), k
    _grad_check(grads_e, grads)
    for k in ("student_backbone_grad_norm", "student_dino_head_grad_norm", "student_ibot_head_grad_norm"):
        assert abs(met[k] - float(m[k])) < 2e-2 * float(m[k]), k


def test_softmax_centering_with_distinct_heads_matches_oracle():
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle.batch import synthetic_batch
    from oracle.step import ssl_forward
    cfg, B = _tiny(), 3
    P = _params(cfg, 1)
    batch = synthetic_batch(cfg, B, 2)
    eng = Engine(_with_ibot(from_oracle_cfg(cfg)), B, max_masked=int(batch["mask_indices_list"].shape[0]), centering="softmax")
    eng.params.load_reference_tree(P)
    cd, ci = torch.randn(264) * 0.01, torch.randn(IBOT[0]) * 0.01
    eng.center_dino.copy_(cd); eng.center_ibot.copy_(ci)
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    met = eng.read_metrics()
    centers = {"dino": cd.clone().reshape(1, -1), "ibot": ci.clone().reshape(1, -1), "momentum": 0.9}
    student = {k: v.clone().requires_grad_(True) for k, v in P.items() if k.startswith("student_")}
    full = dict(P); full.update(student)
    loss, m = ssl_forward(full, batch, HYPER["teacher_temp"], cfg, centers=centers)
    assert abs(met["total_loss"] - loss.item()) < 1e-3 * abs(loss.item())
    for k in ("dino_local_crops_loss", "dino_global_crops_loss", "ibot_loss"):
        assert abs(met[k] - float(m[k])) <= 1e-3 * abs(float(m[k])), k
    assert torch.allclose(eng.center_dino.cpu(), centers["dino"].reshape(-1), atol=1e-5)
    assert torch.allclose(eng.center_ibot.cpu(), centers["ibot"].reshape(-1), atol=1e-5)
    keys = list(student)
    gl = torch.autograd.grad(loss, [student[k] for k in keys], allow_unused=True)
    grads = {k: (g if g is not None else torch.zeros_like(student[k])) for k, g in zip(keys, gl)}
    _grad_check({k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}, grads)


def _steps(cfg, params, batch, B, n, centering="sinkhorn_knopp"):
    from dinov3_jax.engine import Engine
    eng = Engine(cfg, B, max_masked=int(batch["mask_indices_list"].shape[0]), centering=centering)
    eng.params.load_reference_tree(params)
    for _ in range(n):
        eng.train_step(batch, **HYPER)
    torch.cuda.synchronize()
    out = (eng.read_metrics(), {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()},
           {k: v.cpu() for k, v in eng.params.export_reference_tree("param").items()})
    del eng
    return out


def _assert_same_bits(r0, r1):
    (m0, g0, p0), (m1, g1, p1) = r0, r1
    assert m0 == m1
    assert g0.keys() == g1.keys() and p0.keys() == p1.keys()
    assert all(torch.equal(g0[k], g1[k]) for k in g0), [k for k in g0 if not torch.equal(g0[k], g1[k])][:5]
    assert all(torch.equal(p0[k], p1[k]) for k in p0), [k for k in p0 if not torch.equal(p0[k], p1[k])][:5]


@pytest.mark.parametrize("centering", ["sinkhorn_knopp", "softmax"])
def test_distinct_heads_steps_are_bit_reproducible(centering):
    from dinov3_jax.engine import config_for
    from dinov3_jax.engine.synth import reference_like_params, synthetic_batch
    cfg = dataclasses.replace(config_for("vit_small", n_prototypes=4096, ibot_n_prototypes=2048, ibot_head_hidden=1024,
                                         ibot_head_bottleneck=128), depth=2)
    params = reference_like_params(cfg, 0)
    assert tuple(params["student_ibot_head/last_layer/kernel"].shape) == (128, 2048)
    batch = synthetic_batch(cfg, 4, seed=3)
    _assert_same_bits(_steps(cfg, params, batch, 4, 2, centering), _steps(cfg, params, batch, 4, 2, centering))


def test_explicit_equal_ibot_sizes_give_the_bits_of_unset_ones():
    from dinov3_jax.engine import config_for
    from dinov3_jax.engine.synth import reference_like_params, synthetic_batch
    cfg = dataclasses.replace(config_for("vit_small", n_prototypes=4096), depth=2)
    same = dataclasses.replace(cfg, ibot_n_prototypes=4096, ibot_head_hidden=2048, ibot_head_bottleneck=256)
    assert cfg.head_dims("ibot_head") == same.head_dims("ibot_head")
    params = reference_like_params(cfg, 0)
    batch = synthetic_batch(cfg, 4, seed=3)
    _assert_same_bits(_steps(cfg, params, batch, 4, 2), _steps(same, params, batch, 4, 2))


# ------------------------------------------------------------------------------------------------ DINOv3 recipe heads
def _recipe_cfg():
    from dinov3_jax.engine import config_for
    return dataclasses.replace(config_for("vit_large", n_prototypes=262144, head_hidden=8192, head_bottleneck=512,
                                          ibot_n_prototypes=98304, ibot_head_hidden=4096, ibot_head_bottleneck=384),
                               depth=2)


@pytest.mark.parametrize("R,K", [(128, 262144), (640, 262144), (1024, 98304)])
def test_sinkhorn_and_cross_entropy_at_recipe_prototype_counts(R, K):
    """Sinkhorn-Knopp + cross-entropy at the DINOv3 heads' prototype counts against the float64 oracle (as
    test_real_shapes_gpu.py does at 65 536); R = 128 / 640 are the teacher / student DINO rows of B = 64."""
    from dinov3_jax import ops
    from oracle.losses import ibot_loss_masked, sinkhorn_knopp
    temp = 0.04
    g = torch.Generator(device="cuda").manual_seed(K + R)
    L = torch.randn(R, K, device="cuda", generator=g) * 0.05
    mx = torch.full((K,), float("-inf"), device="cuda"); ops.colmax(L, mx)
    btot = torch.tensor([float(R)], device="cuda")
    a, s, av = None, torch.zeros(K, device="cuda"), torch.empty(R, device="cuda")
    for _ in range(3):
        s.zero_(); ops.sinkhorn_colsum(L, mx, temp, a, s); ops.sinkhorn_rowsum(L, mx, temp, s, btot, av); a = av
    S = torch.randn(R, K, device="cuda", generator=g) * 0.5
    t0 = torch.arange(R, dtype=torch.int32, device="cuda"); t1 = torch.full((R,), -1, dtype=torch.int32, device="cuda")
    nrows = 128.0
    wm = torch.full((R,), 1.0 / nrows, device="cuda"); wg = torch.full((R,), 1.0 / nrows, device="cuda")
    slot = torch.full((R,), 3, dtype=torch.int32, device="cuda")
    metric = torch.zeros(4, device="cuda"); dS = torch.empty(R, K, device="cuda", dtype=torch.bfloat16)
    ops.ce_fwd_bwd(S, 0.1, L, mx, temp, s, a, btot, t0, t1, wm, wg, slot, metric, dS)
    torch.cuda.synchronize()
    assert torch.isfinite(metric).all() and torch.isfinite(dS.float()).all()
    Qr = sinkhorn_knopp(L.cpu().double(), temp, float(R))
    Sr = S.cpu().double().requires_grad_(True)
    loss = ibot_loss_masked(Sr, Qr, 0.1, n_mask_rows=int(nrows))
    loss.backward()
    assert abs(metric[3].item() - loss.item()) < 1e-4 * abs(loss.item()), (metric[3].item(), loss.item())
    e = float((dS.cpu().double() - Sr.grad).norm() / Sr.grad.norm())
    assert e < 6e-3, e


def test_recipe_heads_train_step_at_vit_large_width():
    """One step with the DINOv3 heads at ViT-L width (2 blocks, B = 2): prototype GEMMs with N = 262 144 at K = 512 and
    N = 98 304 at K = 384, hidden GEMMs of 8192^2 / 4096^2 and their split-K weight gradients, the L2 norm at C = 512
    / 384, Sinkhorn and cross-entropy at both prototype counts.  At init the student's distribution is close to uniform,
    so each cross-entropy row is ~ln K: dino_local_crops_loss ~ ln 262 144, and ibot_loss ~ (M / 2B) ln 98 304 (the
    iBOT sum over the M masked rows is divided by the 2B masks, DESIGN.md section 2)."""
    from dinov3_jax.engine import Engine
    from dinov3_jax.engine.synth import init_reference_like, synthetic_batch
    cfg, B = _recipe_cfg(), 2
    batch = synthetic_batch(cfg, B, seed=1)
    M = int(batch["mask_indices_list"].shape[0])
    assert M > 0
    eng = Engine(cfg, B, max_masked=M)
    init_reference_like(eng, seed=0)
    assert eng.h_s_dino.logits.shape == (cfg.n_global * B + cfg.n_local * B, 262144)
    assert eng.h_s_ibot.logits.shape == (M, 98304) and eng.h_s_ibot.U3.shape == (M, 384)
    eng.train_step(batch, **HYPER)
    torch.cuda.synchronize()
    m = eng.read_metrics()
    assert all(math.isfinite(v) for v in m.values()), m
    assert abs(m["dino_local_crops_loss"] - math.log(262144)) < 0.1, m["dino_local_crops_loss"]
    want = M / (2 * B) * math.log(98304)
    assert abs(m["ibot_loss"] - want) < 0.01 * want, (m["ibot_loss"], want)
    assert m["student_dino_head_grad_norm"] > 0 and m["student_ibot_head_grad_norm"] > 0


# ------------------------------------------------------------------------------------------------ state and loops
def test_checkpoint_round_trip_with_distinct_heads_resumes_identically(tmp_path):
    from dinov3_jax.checkpointer import engine_state, load_checkpoint, load_engine_state, save_checkpoint
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle.batch import synthetic_batch
    cfg, B = _tiny(), 2
    ecfg = _with_ibot(from_oracle_cfg(cfg))
    batch = synthetic_batch(cfg, B, 0)
    mm = max(int(batch["mask_indices_list"].shape[0]), 1)
    a = Engine(ecfg, B, max_masked=mm)
    a.params.load_reference_tree(_params(cfg, 0))
    a.train_step(batch, **HYPER)
    params, opt = engine_state(a)
    save_checkpoint(tmp_path / "1", iteration=1, params=params, optimizer_state=opt)
    ck = load_checkpoint(tmp_path / "1", abstract_model_params=params, abstract_optimizer_state=opt)
    b = Engine(ecfg, B, max_masked=mm)
    load_engine_state(b, ck["model_params"], ck["optimizer_state"])
    assert b.step_count == a.step_count == 1
    for what in ("param", "m", "v"):
        ta, tb = a.params.export_reference_tree(what), b.params.export_reference_tree(what)
        assert tuple(ta["student_ibot_head/last_layer/kernel"].shape) == (IBOT[2], IBOT[0])
        assert all(torch.equal(ta[k], tb[k]) for k in ta), what
    for e in (a, b):
        e.train_step(batch, **HYPER)
    la, lb = a.read_metrics()["total_loss"], b.read_metrics()["total_loss"]
    assert abs(la - lb) <= 1e-5 * abs(la)
    pa, pb = a.params.export_reference_tree("param"), b.params.export_reference_tree("param")
    assert max(float((pa[k] - pb[k]).abs().max()) for k in pa) < 1e-5


def test_do_train_runs_three_iterations_with_distinct_heads():
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train.train import do_train
    cfg = setup_config(DinoV3SetupArgs(opts=["student.arch=vit_small", "train.batch_size_per_gpu=2",
                                             "dino.head_n_prototypes=1024", "ibot.head_n_prototypes=512",
                                             "dino.head_hidden_dim=256", "ibot.head_hidden_dim=128",
                                             "dino.head_bottleneck_dim=64", "ibot.head_bottleneck_dim=32"]))
    arch = SSLMetaArch(cfg)
    assert arch.engine_config.head_dims("ibot_head") == (128, 32, 512)
    m = do_train(cfg, arch, max_iters=3, print_freq=1)
    assert abs(m["dino_local_crops_loss"] - math.log(1024)) < 0.05 and m["total_loss"] == m["total_loss"]


def test_two_gpu_fsdp_step_with_distinct_heads_equals_multi_rank_oracle():
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29547", os.path.join(root, "tools", "check_fsdp.py"),
                        "--distinct-heads"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "FSDP CHECK OK" in r.stdout, r.stdout[-2000:]
