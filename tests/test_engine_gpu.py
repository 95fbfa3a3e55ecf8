"""-m gpu: the full step (teacher + student forward, losses, hand-written backward, clip + AdamW + EMA) through the
C ABI against the CPU oracle on the same seeded inputs.

Tolerances (stated per BASELINE.json north_star: 1e-3 rel for the fp32-level quantities; the engine computes in bf16
with fp32 accumulation, so tensors that pass through bf16 GEMM operands are compared norm-wise at the bf16 level):
  loss and loss terms      : 1e-3 relative vs the fp32 oracle (measured ~1e-6)
  gradients (norm-wise)    : 3e-2 vs the fp32 oracle, per tensor 6e-2 (measured ~1.2e-2 global: bf16 operand rounding)
  optimizer / EMA          : 1e-5 given identical gradients (kernel test) — here: update direction sanity only
  token / mask indexing    : bit-exact (test_kernels_gpu.py)
"""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

HYPER = dict(lr=1e-3, wd=0.04, last_layer_lr=5e-4, momentum=0.99, teacher_temp=0.05)


def run_pair(cfg, B, perturb=0.05, seed=0):
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    from oracle.step import init_opt_state, train_step
    P = init_params(cfg, seed, perturb=perturb)
    batch = synthetic_batch(cfg, B, seed)
    eng = Engine(from_oracle_cfg(cfg), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    eng.params.load_reference_tree(P)
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    grads_e = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
    eng.optimizer_step(HYPER["lr"], HYPER["wd"], HYPER["last_layer_lr"], HYPER["momentum"])
    torch.cuda.synchronize()
    met = eng.read_metrics()
    newp_e = {k: v.cpu() for k, v in eng.params.export_reference_tree("param").items()}
    newp, st, loss, m, grads = train_step(P, init_opt_state(P), batch, cfg, **HYPER)
    return dict(P=P, met=met, grads_e=grads_e, newp_e=newp_e, newp=newp, loss=loss, m=m, grads=grads, eng=eng)


def check(r, loss_tol=1e-3, grad_tol=3e-2, tensor_tol=6e-2):
    assert abs(r["met"]["total_loss"] - r["loss"].item()) <= loss_tol * abs(r["loss"].item())
    for k in ("dino_local_crops_loss", "dino_global_crops_loss", "ibot_loss"):
        assert abs(r["met"][k] - float(r["m"][k])) <= loss_tol * abs(float(r["m"][k])), k
    assert abs(r["met"]["koleo_loss"] - float(r["m"]["koleo_loss"])) <= 2e-2 * max(abs(float(r["m"]["koleo_loss"])), 0.05)
    num = sum(((r["grads_e"][k].reshape(g.shape) - g) ** 2).sum() for k, g in r["grads"].items())
    den = sum((g ** 2).sum() for g in r["grads"].values())
    assert float(torch.sqrt(num / den)) < grad_tol
    gmax = max(float(g.norm()) for g in r["grads"].values())
    for k, g in r["grads"].items():
        if float(g.norm()) < 1e-3 * gmax:
            continue       # tensors whose gradient is at the bf16 noise floor of the step
        e = float((r["grads_e"][k].reshape(g.shape) - g).norm() / g.norm())
        assert e < tensor_tol, (k, e)
    for k in ("student_backbone_grad_norm", "student_dino_head_grad_norm", "student_ibot_head_grad_norm"):
        assert abs(r["met"][k] - float(r["m"][k])) < 2e-2 * float(r["m"][k]), k


def test_tiny_step_matches_oracle():
    from oracle import tiny_cfg
    check(run_pair(tiny_cfg(), 4))


def test_tiny_step_layerscale_one():
    from oracle import tiny_cfg
    check(run_pair(tiny_cfg(layerscale=1.0), 4))


def test_tiny_step_single_gelu_and_other_seed():
    from oracle import tiny_cfg
    check(run_pair(tiny_cfg(mlp_second_act=False, layerscale=0.5), 2, seed=3))


def test_ragged_shapes_three_heads_odd_batch():
    from oracle import tiny_cfg
    cfg = tiny_cfg(embed_dim=192, heads=3, depth=1, n_prototypes=264, head_hidden=136, head_bottleneck=40, global_size=80, local_size=48)
    check(run_pair(cfg, 3, seed=1))


def test_patch14_configuration():
    """ViT-g/14-style geometry: patch 14 (im2col rows of 588 elements, padded to 592 for TMA), 4x4 / 2x2 patch grids."""
    from oracle import tiny_cfg
    check(run_pair(tiny_cfg(patch=14, global_size=56, local_size=28, layerscale=0.3), 2, seed=2))


def test_updates_move_parameters_like_the_oracle():
    """AdamW step 1 is lr*sign(g): compare the sign pattern where the gradient is well above the noise floor, and the
    teacher EMA identity teacher' = m*teacher + (1-m)*student' exactly (fp32)."""
    from oracle import tiny_cfg
    r = run_pair(tiny_cfg(layerscale=1.0), 4)
    agree, total = 0, 0
    for k, g in r["grads"].items():
        big = g.abs() > 0.2 * g.abs().max()
        d_e = (r["newp_e"][k].reshape(g.shape) - r["P"][k])[big]
        d_o = (r["newp"][k] - r["P"][k])[big]
        agree += int((torch.sign(d_e) == torch.sign(d_o)).sum()); total += int(big.sum())
    assert agree / total > 0.995
    for k in r["grads"]:
        tk = "teacher_" + k[len("student_"):]
        want = r["P"][tk] * HYPER["momentum"] + r["newp_e"][k].reshape(r["P"][tk].shape) * (1 - HYPER["momentum"])
        assert torch.allclose(r["newp_e"][tk].reshape(want.shape), want, atol=1e-6, rtol=1e-5), k


def test_second_step_runs_and_launch_counter():
    from dinov3_jax import _native
    from oracle import tiny_cfg
    r = run_pair(tiny_cfg(), 2)
    eng = r["eng"]
    _native.reset_launch_count()
    eng.train_step(None, **HYPER)
    torch.cuda.synchronize()
    assert _native.launch_count() > 50
    m = eng.read_metrics()
    assert all(v == v for v in m.values())      # no NaN


def test_batch_from_reference_collate_contract():
    """set_batch accepts exactly the reference's collate dict (keys / dtypes / layouts of data/collate.py:72-93)."""
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import init_reference_like, synthetic_batch
    cfg = dataclasses.replace(config_for("vit_small"), depth=1, n_prototypes=256, head_hidden=128, head_bottleneck=64)
    batch = synthetic_batch(cfg, 2, seed=5)
    assert batch["collated_global_crops"].shape == (4, 224, 224, 3) and batch["collated_masks"].dtype == torch.bool
    eng = Engine(cfg, 2, max_masked=int(batch["mask_indices_list"].shape[0]))
    init_reference_like(eng)
    eng.train_step(batch, **HYPER)
    m = eng.read_metrics()
    assert abs(m["dino_local_crops_loss"] - 5.545) < 0.01      # log(256) at init


def test_softmax_centering_path_matches_oracle():
    """Optional teacher normalisation of the north_star list: center EMA + softmax((x-c)/temp) instead of Sinkhorn."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    from oracle.step import ssl_forward
    cfg = tiny_cfg(layerscale=0.5)
    B = 3
    P = init_params(cfg, 0, perturb=0.05)
    batch = synthetic_batch(cfg, B, 2)
    eng = Engine(from_oracle_cfg(cfg), B, max_masked=int(batch["mask_indices_list"].shape[0]), centering="softmax")
    eng.params.load_reference_tree(P)
    K = cfg.n_prototypes
    c0 = torch.randn(K) * 0.01
    eng.center_dino.copy_(c0); eng.center_ibot.copy_(-c0)
    eng.set_batch(batch)
    eng.forward_backward(0.05)
    met = eng.read_metrics()
    centers = {"dino": c0.clone().reshape(1, K), "ibot": (-c0).reshape(1, K), "momentum": 0.9}
    student = {k: v.clone().requires_grad_(True) for k, v in P.items() if k.startswith("student_")}
    full = dict(P); full.update(student)
    loss, m = ssl_forward(full, batch, 0.05, cfg, centers=centers)
    assert abs(met["total_loss"] - loss.item()) < 1e-3 * abs(loss.item())
    assert torch.allclose(eng.center_dino.cpu(), centers["dino"].reshape(-1), atol=1e-5)
    assert torch.allclose(eng.center_ibot.cpu(), centers["ibot"].reshape(-1), atol=1e-5)
    keys = list(student)
    gl = torch.autograd.grad(loss, [student[k] for k in keys], allow_unused=True)
    ge = eng.params.export_reference_tree("grad")
    num = sum(((ge[k].cpu().reshape(g.shape) - g) ** 2).sum() for k, g in zip(keys, gl) if g is not None)
    den = sum((g ** 2).sum() for g in gl if g is not None)
    assert float(torch.sqrt(num / den)) < 3e-2


@pytest.mark.parametrize("case", ["a", "b", "c"])
def test_engine_loss_against_reference_meta_arch_golden(case):
    """Engine forward vs numbers produced by the reference's own SSLMetaArch.__call__ (tests/golden/make_golden.py);
    the oracle is not involved.  Loss terms 1e-3 rel would be the fp32 bar; these fixtures use large-amplitude head
    weights (peaky softmax), so the bf16-operand tolerance 5e-3 is stated here."""
    from conftest import reference_vectors
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from test_golden_reference import ssl_case
    G = reference_vectors()
    cfg, P, batch, temp = ssl_case(case, dtype=torch.float32)
    B = batch["global_batch_size"]
    batch["collated_global_crops"] = batch["collated_global_crops"].to(torch.bfloat16)
    batch["collated_local_crops"] = batch["collated_local_crops"].to(torch.bfloat16)
    eng = Engine(from_oracle_cfg(cfg), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
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


def test_checkpoint_round_trip_resumes_identically(tmp_path):
    """engine -> reference-named pytree -> disk -> fresh engine: parameters, Adam moments and the step counter survive,
    and the next step from the restored engine equals the next step of the original (checkpointer adapter, §8f.4)."""
    from dinov3_jax.checkpointer import engine_state, load_checkpoint, load_engine_state, save_checkpoint
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg = tiny_cfg(layerscale=0.5)
    B = 2
    batch = synthetic_batch(cfg, B, 0)
    mm = max(int(batch["mask_indices_list"].shape[0]), 1)
    a = Engine(from_oracle_cfg(cfg), B, max_masked=mm)
    a.params.load_reference_tree(init_params(cfg, 0, perturb=0.05))
    a.train_step(batch, **HYPER)
    params, opt = engine_state(a)
    save_checkpoint(tmp_path / "1", iteration=1, params=params, optimizer_state=opt)
    ck = load_checkpoint(tmp_path / "1", abstract_model_params=params, abstract_optimizer_state=opt)
    b = Engine(from_oracle_cfg(cfg), B, max_masked=mm)
    load_engine_state(b, ck["model_params"], ck["optimizer_state"])
    assert b.step_count == a.step_count == 1
    for what in ("param", "m", "v"):
        ta, tb = a.params.export_reference_tree(what), b.params.export_reference_tree(what)
        assert all(torch.equal(ta[k], tb[k]) for k in ta), what
    for e in (a, b):
        e.train_step(batch, **HYPER)
    la, lb = a.read_metrics()["total_loss"], b.read_metrics()["total_loss"]
    assert abs(la - lb) <= 1e-5 * abs(la)
    pa, pb = a.params.export_reference_tree("param"), b.params.export_reference_tree("param")
    worst = max(float((pa[k] - pb[k]).abs().max()) for k in pa)
    assert worst < 1e-5            # fp32 atomics in the gradient reductions are the only source of run-to-run difference


def test_step_with_storage_tokens_and_layernormbf16():
    """SURVEY §8f.1: 4 register tokens (N = 1 + 4 + P, RoPE prefix 5, storage-token gradients) and eps 1e-5."""
    from oracle import tiny_cfg
    r = run_pair(tiny_cfg(n_storage=4, ln_eps=1e-5, layerscale=0.5), 3, seed=2)
    check(r)
    g = r["grads"]["student_backbone/storage_tokens"]
    e = float((r["grads_e"]["student_backbone/storage_tokens"].reshape(g.shape) - g).norm() / g.norm())
    assert e < 6e-2


def _loader_fixture():
    import os
    import numpy as np
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "loader_batch.npz"))
    b = {k: torch.from_numpy(z[k]) for k in z.files}
    for k in ("collated_global_crops", "collated_local_crops"):
        b[k] = b[k].view(torch.bfloat16)
    return b


def test_loader_batch_from_reference_augmentation_through_engine_matches_oracle():
    """Loader -> engine end to end: a batch made by the reference's own DataAugmentationDINO (fixture, see
    tests/golden/make_loader_fixture.py) and this repo's collate goes through `Engine.train_step` unchanged, and the
    loss equals the oracle's on the same batch."""
    from oracle import cfg_for
    from oracle.model import init_params
    from oracle.step import init_opt_state, train_step
    from dinov3_jax.engine import Engine, from_oracle_cfg
    cfg = dataclasses.replace(cfg_for("vit_small", global_size=64, local_size=32, n_prototypes=512, head_hidden=256,
                                      head_bottleneck=64, layerscale=0.1), depth=2)
    batch = _loader_fixture()
    B = batch["collated_local_crops"].shape[0] // cfg.n_local
    P = init_params(cfg, 0, perturb=0.05)
    eng = Engine(from_oracle_cfg(cfg), B, max_masked=int(batch["mask_indices_list"].shape[0]))
    eng.params.load_reference_tree(P)
    eng.train_step(batch, **HYPER)
    met = eng.read_metrics()
    _, _, loss, m, _ = train_step(P, init_opt_state(P), batch, cfg, **HYPER)
    assert abs(met["total_loss"] - loss.item()) < 1e-3 * abs(loss.item()), (met["total_loss"], loss.item())


def test_reference_call_contract_train_step_then_update_ema():
    """`train_step(params, batch, optimizer_state, teacher_temp, iteration, root_rngs)` -> (params, optimizer_state,
    loss, metrics) followed by `model.update_ema()(ema_params, params, mom)` (train/train.py:491-565,666;
    ssl_meta_arch.py:644-660) gives exactly the state of the fused engine step."""
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.engine.synth import init_reference_like
    from dinov3_jax.train.ssl_meta_arch import SSLMetaArch
    from dinov3_jax.train.train import build_optimizer, build_schedulers, make_state, train_step
    opts = ["train.batch_size_per_gpu=2", "student.arch=vit_small", "crops.global_crops_size=64", "crops.local_crops_size=32",
            "dino.head_n_prototypes=512", "ibot.head_n_prototypes=512", "dino.head_hidden_dim=256", "ibot.head_hidden_dim=256",
            "dino.head_bottleneck_dim=64", "ibot.head_bottleneck_dim=64", "optim.epochs=2", "train.OFFICIAL_EPOCH_LENGTH=10",
            "optim.warmup_epochs=1", "teacher.warmup_teacher_temp_epochs=1", "optim.freeze_last_layer_epochs=0"]
    batch = _loader_fixture()
    M = int(batch["mask_indices_list"].shape[0])
    out = []
    for mode in ("reference_calls", "fused"):
        config = setup_config(DinoV3SetupArgs(opts=opts))
        model = SSLMetaArch(config)
        eng = model.build_engine(max_masked=M)
        init_reference_like(eng, seed=3)
        lr_s, wd_s, mom_s, temp_s, last_s = build_schedulers(config)
        it = 4
        if mode == "reference_calls":
            optimizer = build_optimizer(config, model.get_params_groups(), lr_s, wd_s, last_s)
            params, ema_params, opt_state = make_state(eng, optimizer)
            assert set(params.keys()) == {"student_backbone", "student_dino_head", "student_ibot_head", "teacher_backbone",
                                          "teacher_dino_head", "teacher_ibot_head"}
            t_before = ema_params["teacher_backbone"]["norm/scale"].clone()
            params, opt_state, loss, metrics = train_step(params, batch, opt_state, temp_s[it], it, None)
            assert torch.equal(ema_params["teacher_backbone"]["norm/scale"], t_before)       # teacher untouched by train_step
            for k in ("dino_local_crops_loss", "dino_global_crops_loss", "koleo_loss", "ibot_loss",
                      "student_backbone_grad_norm", "student_dino_head_grad_norm", "student_ibot_head_grad_norm"):
                assert k in metrics
            ema_params = model.update_ema()(ema_params, params, mom_s[it])
        else:
            eng.train_step(batch, teacher_temp=float(temp_s[it]), lr=float(lr_s[it]), wd=float(wd_s[it]),
                           last_layer_lr=float(last_s[it]), momentum=float(mom_s[it]))
            loss = eng.read_metrics()["total_loss"]
        out.append((loss, eng.params.export_reference_tree("param")))
    (la, pa), (lb, pb) = out
    assert abs(la - lb) <= 1e-5 * abs(lb)
    for k in pa:
        assert torch.allclose(pa[k], pb[k], atol=2e-6, rtol=1e-5), k


def test_step_with_swiglu_ffn():
    """SURVEY §8f.1: SwiGLU FFN (layers/ffn_layers.py:52-76, hidden 2/3 * 4D rounded up to swiglu_align) on the GPU path:
    w1 | w2 projections, fused silu-gate kernel, w3 + LayerScale, and the hand-written backward."""
    from oracle import tiny_cfg
    r = run_pair(tiny_cfg(ffn_layer="swiglu", swiglu_align=64, layerscale=0.5), 3, seed=4)
    check(r)
    for name in ("mlp/w1/kernel", "mlp/w2/kernel", "mlp/w3/kernel", "mlp/w1/bias", "mlp/w2/bias", "mlp/w3/bias"):
        k = f"student_backbone/blocks_0/{name}"
        g = r["grads"][k]
        e = float((r["grads_e"][k].reshape(g.shape) - g).norm() / g.norm())
        assert e < 6e-2, (name, e)


def test_step_with_mask_k_bias():
    """SURVEY §8f.1: student.mask_k_bias (upstream LinearKMaskedBias): the k third of the qkv bias does not reach the
    forward and gets no gradient; the parameter stays where it was (zero)."""
    from oracle import tiny_cfg
    r = run_pair(tiny_cfg(mask_k_bias=True, layerscale=0.5), 3, seed=5)
    check(r)
    D = 128
    for i in range(2):
        k = f"student_backbone/blocks_{i}/attn/qkv/bias"
        assert float(r["grads_e"][k].reshape(-1)[D:2 * D].abs().max()) == 0.0
        assert float(r["newp_e"][k].reshape(-1)[D:2 * D].abs().max()) == 0.0
        gq = r["grads"][k].reshape(-1)
        assert float(gq[D:2 * D].abs().max()) == 0.0                      # the oracle agrees: masked bias, zero gradient


def test_activation_remat_equals_stashing():
    """train.checkpointing (ssl_default_config.yaml:88): recomputing each student block in the backward gives the same
    loss and the same gradients as keeping its activations.  The recomputing path takes the LayerScale / GELU backward
    of the MLP branch from the stand-alone kernel instead of the tail fused into the LayerNorm backward; both compute du
    with the same arithmetic, so every gradient is bit-identical except the two column sums that kernel forms in
    another order (ls2/gamma and the fc2 bias), which agree to 1e-5."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg = tiny_cfg(layerscale=0.5, depth=3)
    B = 3
    P = init_params(cfg, 0, perturb=0.05)
    batch = synthetic_batch(cfg, B, 1)
    out = []
    for remat in (False, True):
        eng = Engine(from_oracle_cfg(cfg), B, max_masked=int(batch["mask_indices_list"].shape[0]), remat=remat)
        assert eng.student.per_block == (not remat)
        eng.params.load_reference_tree(P)
        eng.set_batch(batch)
        eng.forward_backward(HYPER["teacher_temp"])
        g = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
        eng.optimizer_step(HYPER["lr"], HYPER["wd"], HYPER["last_layer_lr"], HYPER["momentum"])
        out.append((eng.read_metrics()["total_loss"], g))
    (la, ga), (lb, gb) = out
    assert la == lb
    assert ga.keys() == gb.keys()
    for k in ga:
        if k.endswith("/ls2/gamma") or k.endswith("/mlp/Dense_1/bias"):
            assert float((ga[k] - gb[k]).norm() / ga[k].norm()) < 1e-5, k
        else:
            assert torch.equal(ga[k], gb[k]), k


# --------------------------------------------------------------------------------------------------- Gram anchoring (8f.2)
def _gram_pair(mode, only_gram):
    """Engine step with the Gram term vs oracle.step.ssl_forward(gram=...) under autograd."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    from oracle.step import ssl_forward
    kw = dict(dino_loss_weight=0.0, ibot_loss_weight=0.0, koleo_loss_weight=0.0) if only_gram else {}
    cfg = tiny_cfg(layerscale=0.5, **kw)
    B, W = 3, 25.0
    P = init_params(cfg, 6, perturb=0.05)
    batch = synthetic_batch(cfg, B, 6)
    remove_neg = mode == "frozen_remove_neg"
    used = mode[len("ema_"):] if mode in ("ema_masked", "ema_unmasked") else "all"
    img_level = mode == "ema_img_level"
    ema = mode.startswith("ema")
    gram = dict(weight=W, ema_teacher=ema, normalized=mode != "ema_img_level", img_level=img_level, remove_neg=remove_neg,
                remove_only_teacher_neg=img_level, tokens_used=used)
    ecfg = dataclasses.replace(from_oracle_cfg(cfg), gram_use_loss=True, gram_loss_weight=W, gram_ema_teacher=ema,
                               gram_remove_neg=remove_neg, gram_it_load_ema_teacher=0, gram_tokens_used=used,
                               gram_img_level=img_level, gram_remove_only_teacher_neg=img_level,
                               gram_normalized=mode != "ema_img_level")
    eng = Engine(ecfg, B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    eng.params.load_reference_tree(P)
    full = dict(P)
    if mode == "snapshot":               # gram teacher := EMA teacher, taken inside the step by the schedule
        for k, v in P.items():
            if k.startswith("teacher_backbone/"):
                full["gram_backbone/" + k[len("teacher_backbone/"):]] = v
    elif not ema:                        # a different frozen network, loaded from a checkpoint tree
        P2 = init_params(cfg, 7, perturb=0.05)
        tree = {k[len("teacher_backbone/"):]: v for k, v in P2.items() if k.startswith("teacher_backbone/")}
        eng.gram_teacher_load(tree)
        full.update({"gram_backbone/" + k: v for k, v in tree.items()})
    student = {k: v.detach().clone().requires_grad_(True) for k, v in P.items() if k.startswith("student_")}
    full.update(student)
    loss, m = ssl_forward(full, batch, HYPER["teacher_temp"], cfg, gram=gram)
    keys = list(student)
    gl = torch.autograd.grad(loss, [student[k] for k in keys], allow_unused=True)
    grads = {k: (g if g is not None else torch.zeros_like(student[k])) for k, g in zip(keys, gl)}
    eng.train_step(batch, iteration=0, **HYPER) if mode == "snapshot" else (eng.set_batch(batch), eng.forward_backward(HYPER["teacher_temp"]))
    met = eng.read_metrics()
    grads_e = None
    if mode != "snapshot":
        grads_e = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
    return met, float(loss), m, grads, grads_e


def test_checkpoint_keeps_the_frozen_gram_teacher(tmp_path):
    """The frozen gram teacher (taken from the EMA teacher at gram.it_load_ema_teacher) is part of the saved state: a
    restored engine has the Gram term active with the same frozen weights, and its next step matches the original's."""
    from dinov3_jax.checkpointer import engine_state, load_checkpoint, load_engine_state, save_checkpoint
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg = tiny_cfg(layerscale=0.5)
    B = 2
    batch = synthetic_batch(cfg, B, 0)
    mm = max(int(batch["mask_indices_list"].shape[0]), 1)
    ecfg = dataclasses.replace(from_oracle_cfg(cfg), gram_use_loss=True, gram_loss_weight=10.0, gram_it_load_ema_teacher=0,
                               gram_update_frequency=1000)
    a = Engine(ecfg, B, max_masked=mm)
    a.params.load_reference_tree(init_params(cfg, 0, perturb=0.05))
    a.train_step(batch, iteration=0, **HYPER)             # snapshot of the EMA teacher taken inside this step
    assert a.gram_active and "gram_loss" in a.read_metrics()
    params, opt = engine_state(a)
    assert "gram_backbone" in params
    save_checkpoint(tmp_path / "0", iteration=0, params=params, optimizer_state=opt)
    b = Engine(ecfg, B, max_masked=mm)
    ck = load_checkpoint(tmp_path / "0", abstract_model_params=engine_state(b)[0], strict_loading=False)
    load_engine_state(b, ck["model_params"], ck["optimizer_state"])
    assert b.gram_active
    ga, gb = a.gram_net.mods["backbone"], b.gram_net.mods["backbone"]
    assert torch.equal(ga.bf16, gb.bf16) and torch.equal(ga.vecs, gb.vecs)
    assert ga.bf16.float().abs().sum() > 0            # a snapshot was taken, not the zero-initialised store
    for e in (a, b):
        e.train_step(batch, iteration=1, **HYPER)
    ma, mb = a.read_metrics(), b.read_metrics()
    assert abs(ma["gram_loss"] - mb["gram_loss"]) <= 1e-5 * abs(ma["gram_loss"])
    assert abs(ma["total_loss"] - mb["total_loss"]) <= 1e-5 * abs(ma["total_loss"])


def test_gram_teacher_at_its_own_resolution():
    """crops.gram_teacher_crops_size != global_crops_size: the frozen gram teacher runs on `collated_gram_teacher_crops`
    (data/collate.py:33-38,81-82) through a third token stream and its patch tokens are resized (bicubic) to the student's
    grid before the Gram matrices; loss and gradients against the oracle (F.interpolate)."""
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    from oracle.step import ssl_forward
    cfg = tiny_cfg(layerscale=0.5)
    B, W, GS = 2, 25.0, 96                       # student global crops 64^2 (4x4 patches), gram teacher 96^2 (6x6)
    P = init_params(cfg, 8, perturb=0.05)
    batch = synthetic_batch(cfg, B, 8)
    g = torch.Generator().manual_seed(3)
    batch["collated_gram_teacher_crops"] = torch.randn(cfg.n_global * B, GS, GS, 3, generator=g).to(torch.bfloat16)
    for aa in (False, True):
        ecfg = dataclasses.replace(from_oracle_cfg(cfg), gram_use_loss=True, gram_loss_weight=W, gram_it_load_ema_teacher=0,
                                   gram_teacher_size=GS, gram_resize_antialias=aa)
        eng = Engine(ecfg, B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
        eng.params.load_reference_tree(P)
        P2 = init_params(cfg, 9, perturb=0.05)
        tree = {k[len("teacher_backbone/"):]: v for k, v in P2.items() if k.startswith("teacher_backbone/")}
        eng.gram_teacher_load(tree)
        full = dict(P)
        full.update({"gram_backbone/" + k: v for k, v in tree.items()})
        student = {k: v.detach().clone().requires_grad_(True) for k, v in P.items() if k.startswith("student_")}
        full.update(student)
        loss, m = ssl_forward(full, batch, HYPER["teacher_temp"], cfg,
                              gram=dict(weight=W, ema_teacher=False, remove_neg=False, remove_only_teacher_neg=False,
                                        resize_antialias=aa))
        keys = list(student)
        gl = torch.autograd.grad(loss, [student[k] for k in keys], allow_unused=True)
        eng.set_batch(batch)
        eng.forward_backward(HYPER["teacher_temp"])
        met = eng.read_metrics()
        assert abs(met["gram_loss"] - float(m["gram_loss"])) < 2e-2 * float(m["gram_loss"]), (aa, met["gram_loss"], float(m["gram_loss"]))
        assert abs(met["total_loss"] - float(loss.detach())) < 2e-3 * abs(float(loss.detach()))
        ge = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
        num = sum(((ge[k].reshape(g_.shape) - g_) ** 2).sum() for k, g_ in zip(keys, gl) if g_ is not None)
        den = sum((g_ ** 2).sum() for g_ in gl if g_ is not None)
        assert float(torch.sqrt(num / den)) < 3e-2


@pytest.mark.parametrize("mode", ["ema", "frozen", "frozen_remove_neg", "snapshot", "ema_masked", "ema_unmasked", "ema_img_level"])
def test_step_with_gram_anchoring(mode):
    """SURVEY 8f.2 on the GPU path: Gram-anchoring term (loss/gram_loss.py:13-50 at batch level; train/ssl_meta_arch.py:
    527-541) with the EMA teacher, a frozen gram teacher loaded from a tree, negative removal, the scheduled snapshot of
    the EMA teacher (gram.it_load_ema_teacher), gram.tokens_used masked / unmasked (ragged row counts), and per-image Gram
    matrices (gram.img_level, un-normalised features, teacher-only negative removal)."""
    met, loss, m, grads, grads_e = _gram_pair(mode, only_gram=False)
    assert abs(met["gram_loss"] - float(m["gram_loss"])) < 2e-2 * float(m["gram_loss"]), (met["gram_loss"], float(m["gram_loss"]))
    assert met["gram_loss_weight"] == 25.0
    assert abs(met["total_loss"] - loss) < 2e-3 * abs(loss)
    if grads_e is not None:
        num = sum(((grads_e[k].reshape(g.shape) - g) ** 2).sum() for k, g in grads.items())
        den = sum((g ** 2).sum() for g in grads.values())
        assert float(torch.sqrt(num / den)) < 3e-2


def test_gram_term_gradient_alone():
    """Only the Gram term carries weight: every backbone gradient is the Gram backward (similarity GEMMs, d3_gram_diff,
    G Xs GEMM, row-normalisation backward, scatter into the final-norm gradient) and nothing else."""
    met, loss, m, grads, grads_e = _gram_pair("frozen", only_gram=True)
    assert abs(met["total_loss"] - loss) < 2e-2 * abs(loss)
    bb = {k: g for k, g in grads.items() if k.startswith("student_backbone/") and float(g.norm()) > 0}
    num = sum(((grads_e[k].reshape(g.shape) - g) ** 2).sum() for k, g in bb.items())
    den = sum((g ** 2).sum() for g in bb.values())
    assert float(den) > 0 and float(torch.sqrt(num / den)) < 4e-2
    for k, g in grads.items():
        if not k.startswith("student_backbone/"):
            assert float(grads_e[k].abs().max()) == 0.0, k        # no gradient reaches the heads


def test_training_steps_are_bit_reproducible():
    """Two engines with the same parameters and batch run three training steps each: every gradient, parameter and
    metric is the same bit for bit (the step's reductions add their partial sums in a fixed order)."""
    _assert_steps_bit_reproducible("sinkhorn_knopp")


def test_training_steps_with_softmax_centering_are_bit_reproducible():
    """The same with the optional softmax centering, whose column sums are slab reductions too."""
    _assert_steps_bit_reproducible("softmax")


def _assert_steps_bit_reproducible(centering):
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import reference_like_params, synthetic_batch
    cfg = dataclasses.replace(config_for("vit_small", n_prototypes=4096), depth=2)
    params = reference_like_params(cfg, 0)
    B = 4
    batch = synthetic_batch(cfg, B, seed=3)
    runs = []
    for _ in range(2):
        eng = Engine(cfg, B, max_masked=int(batch["mask_indices_list"].shape[0]), centering=centering)
        eng.params.load_reference_tree(params)
        for _ in range(3):
            eng.train_step(batch, **HYPER)
        torch.cuda.synchronize()
        runs.append((eng.read_metrics(), {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()},
                     {k: v.cpu() for k, v in eng.params.export_reference_tree("param").items()}))
        del eng
    (m0, g0, p0), (m1, g1, p1) = runs
    assert m0 == m1
    assert all(torch.equal(g0[k], g1[k]) for k in g0), [k for k in g0 if not torch.equal(g0[k], g1[k])][:5]
    assert all(torch.equal(p0[k], p1[k]) for k in p0), [k for k in p0 if not torch.equal(p0[k], p1[k])][:5]
