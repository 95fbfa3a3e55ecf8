"""-m gpu: distillation from a frozen teacher of another architecture through the engine.

  (a) the loss terms against the reference's SSLMetaArch.__call__ with distillation.enabled (distill_vectors.npz);
  (b) a step against the fp32 distillation oracle (tests/distill_helpers.py) for a ViT-B teacher (head_dim 64) and a
      4096-wide, 32-head, one-block swiglu64 teacher without a qkv bias, both teaching a small ViT-S student;
  (c) the frozen teacher stays bit-identical over three steps and teacher_* follows the EMA of the student;
  (d) the mask_token gets no gradient (the student's global crops carry no mask tokens);
  (e) two runs compute the same bits;
  (f) a teacher loaded from a save_checkpoint directory gives the teacher logits of that run's own teacher pass;
  (g) a saved and reloaded distillation run resumes bit-identically;
  (h) the fixed-flag GEMM for the qkv projection without a bias equals the run-time-flag epilogue bit for bit.

Tolerances are those of test_engine_gpu.py: loss terms 1e-3 relative (5e-3 against the peaky golden fixture),
gradients 3e-2 norm-wise globally and 6e-2 per tensor.
"""
import dataclasses

import pytest
import torch

from distill_helpers import distill_params, distill_train_step, frozen_tree

pytestmark = pytest.mark.gpu

HYPER = dict(lr=1e-3, wd=0.04, last_layer_lr=5e-4, momentum=0.99, teacher_temp=0.05)
S_IBOT = (136, 96, 48)


def _student():
    from oracle.arch import ModelCfg
    return ModelCfg(embed_dim=384, depth=2, heads=6, global_size=64, local_size=32, n_local=4, n_prototypes=264,
                    head_hidden=136, head_bottleneck=40, layerscale=0.5)


def _teacher(kind):
    from oracle.arch import ModelCfg
    if kind == "vit_base":
        return ModelCfg(embed_dim=768, depth=2, heads=12, global_size=64, local_size=32, n_local=4, n_prototypes=264,
                        head_hidden=200, head_bottleneck=56, n_storage=4, ln_eps=1e-5), (136, 120, 64), True
    return ModelCfg(embed_dim=4096, depth=1, heads=32, ffn_ratio=3.0, ffn_layer="swiglu", swiglu_align=64,
                    global_size=64, local_size=32, n_local=4, n_prototypes=264, head_hidden=256, head_bottleneck=64,
                    n_storage=4, ln_eps=1e-5), (136, 192, 72), False


def _ecfg(cfg, ibot, qkv_bias=True):
    from dinov3_jax.engine import from_oracle_cfg
    return dataclasses.replace(from_oracle_cfg(cfg), ibot_n_prototypes=ibot[0], ibot_head_hidden=ibot[1],
                               ibot_head_bottleneck=ibot[2], qkv_bias=qkv_bias)


def _engine(cfg, tcfg, t_ibot, qkv_bias, P, B, max_masked):
    from dinov3_jax.engine import Engine
    eng = Engine(_ecfg(cfg, S_IBOT), B, max_masked=max(max_masked, 1), distill=_ecfg(tcfg, t_ibot, qkv_bias))
    eng.params.load_reference_tree({k: v.float() for k, v in P.items() if not k.startswith("distill_")})
    eng.distill_teacher_load({m: {k: v.float() for k, v in t.items()} for m, t in frozen_tree(P).items()})
    return eng


def _setup(kind="vit_base", B=4, seed=0, formula=False):
    from oracle.batch import synthetic_batch
    cfg = _student()
    tcfg, t_ibot, qkv_bias = _teacher(kind)
    P = distill_params(cfg, S_IBOT, tcfg, t_ibot, seed, qkv_bias, formula=formula, dtype=torch.float32)
    batch = synthetic_batch(cfg, B, seed)
    return cfg, tcfg, t_ibot, qkv_bias, P, batch


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


def _bits(eng):
    return {k: v.cpu() for k, v in eng.params.export_reference_tree("param").items()}


def _frozen_bits(eng):
    return [t.clone() for s in eng.t_net.mods.values() for t in (s.bf16, s.vecs)]


@pytest.mark.parametrize("case", ["a", "b"])
def test_engine_loss_against_reference_meta_arch_golden_with_distillation(case):
    from dinov3_jax.engine import Engine
    from distill_helpers import STUDENT_IBOT, TEACHER_IBOT
    from test_distill_cpu import distill_case, distill_golden
    G = distill_golden()
    cfg, tcfg, P, batch, temp = distill_case(G, case, dtype=torch.float32)
    B = batch["global_batch_size"]
    batch["collated_global_crops"] = batch["collated_global_crops"].to(torch.bfloat16)
    batch["collated_local_crops"] = batch["collated_local_crops"].to(torch.bfloat16)
    eng = Engine(_ecfg(cfg, STUDENT_IBOT), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1),
                 distill=_ecfg(tcfg, TEACHER_IBOT, qkv_bias=False))
    eng.params.load_reference_tree({k: v for k, v in P.items() if not k.startswith("distill_")})
    eng.distill_teacher_load(frozen_tree(P))
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


@pytest.mark.parametrize("kind", ["vit_base", "hd128_swiglu64_noqkvbias"])
def test_distillation_step_matches_oracle(kind):
    from oracle.step import init_opt_state
    cfg, tcfg, t_ibot, qkv_bias, P, batch = _setup(kind)
    B = batch["global_batch_size"]
    eng = _engine(cfg, tcfg, t_ibot, qkv_bias, P, B, int(batch["mask_indices_list"].shape[0]))
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    torch.cuda.synchronize()
    met = eng.read_metrics()
    grads_e = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
    _, _, loss, m, grads = distill_train_step(P, init_opt_state(P), batch, cfg, tcfg, **HYPER)
    assert abs(met["total_loss"] - loss.item()) <= 1e-3 * abs(loss.item())
    for k in ("dino_local_crops_loss", "dino_global_crops_loss", "ibot_loss"):
        assert abs(met[k] - float(m[k])) <= 1e-3 * abs(float(m[k])), k
    _grad_check(grads_e, grads)
    # (d) no mask tokens in the student's global crops: the mask token gets no gradient at all
    assert bool((grads_e["student_backbone/mask_token"] == 0).all())


def test_frozen_teacher_stays_and_ema_follows_the_student():
    cfg, tcfg, t_ibot, qkv_bias, P, batch = _setup("vit_base", seed=1)
    eng = _engine(cfg, tcfg, t_ibot, qkv_bias, P, batch["global_batch_size"], int(batch["mask_indices_list"].shape[0]))
    frozen0 = _frozen_bits(eng)
    prev = _bits(eng)
    mom = HYPER["momentum"]
    for _ in range(3):
        eng.train_step(batch, **HYPER)
        torch.cuda.synchronize()
        cur = _bits(eng)
        for k in cur:
            if k.startswith("teacher_"):
                s = cur["student_" + k[len("teacher_"):]]
                want = prev[k] * mom + s * (1 - mom)
                assert torch.allclose(cur[k], want, rtol=1e-6, atol=1e-7), k
        prev = cur
    for a, b in zip(frozen0, _frozen_bits(eng)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def test_distillation_is_bit_reproducible():
    runs = []
    for _ in range(2):
        cfg, tcfg, t_ibot, qkv_bias, P, batch = _setup("hd128_swiglu64_noqkvbias", seed=2)
        eng = _engine(cfg, tcfg, t_ibot, qkv_bias, P, batch["global_batch_size"], int(batch["mask_indices_list"].shape[0]))
        for _ in range(2):
            eng.train_step(batch, **HYPER)
        runs.append((_bits(eng), eng.read_metrics()["total_loss"]))
        del eng
    (a, la), (b, lb) = runs
    assert la == lb
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_teacher_from_a_checkpoint_gives_that_runs_teacher_logits(tmp_path):
    """A plain run of the teacher architecture is saved; a distilling engine loads its teacher_* subtrees the way
    SSLMetaArch does, and its teacher pass gives the saved run's own teacher logits bit for bit."""
    import types
    from dinov3_jax.checkpointer import engine_state, save_checkpoint
    from dinov3_jax.engine import Engine
    from dinov3_jax.train.ssl_meta_arch import SSLMetaArch
    cfg, tcfg, t_ibot, qkv_bias, P, batch = _setup("vit_base", seed=3)
    B, M = batch["global_batch_size"], int(batch["mask_indices_list"].shape[0])
    plain = Engine(_ecfg(tcfg, t_ibot), B, max_masked=M)
    Pt = distill_params(tcfg, t_ibot, tcfg, t_ibot, 5, True, formula=False, dtype=torch.float32)
    plain.params.load_reference_tree({k: v for k, v in Pt.items() if not k.startswith("distill_")})
    plain.train_step(batch, **HYPER)                       # the saved teacher_* is an EMA, not the initial copy
    params, opt = engine_state(plain)
    save_checkpoint(tmp_path / "teacher_run", iteration=0, params=params, optimizer_state=opt)
    plain.set_batch(batch)
    plain.forward_backward(HYPER["teacher_temp"])
    want = (plain.h_t_dino.logits.clone(), plain.h_t_ibot.logits[:M].clone())
    eng = Engine(_ecfg(cfg, S_IBOT), B, max_masked=M, distill=_ecfg(tcfg, t_ibot))
    eng.params.load_reference_tree({k: v for k, v in P.items() if not k.startswith("distill_")})
    SSLMetaArch.load_distillation_teacher(types.SimpleNamespace(engine=eng, PARAM_MODULES=SSLMetaArch.PARAM_MODULES),
                                          str(tmp_path / "teacher_run"))
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    torch.cuda.synchronize()
    assert torch.equal(eng.h_t_dino.logits.view(torch.int32), want[0].view(torch.int32))
    assert torch.equal(eng.h_t_ibot.logits[:M].view(torch.int32), want[1].view(torch.int32))


def test_distillation_run_resumes_bit_identically(tmp_path):
    from dinov3_jax.checkpointer import engine_state, load_checkpoint, load_engine_state, save_checkpoint
    cfg, tcfg, t_ibot, qkv_bias, P, batch = _setup("hd128_swiglu64_noqkvbias", seed=4)
    B, M = batch["global_batch_size"], int(batch["mask_indices_list"].shape[0])
    a = _engine(cfg, tcfg, t_ibot, qkv_bias, P, B, M)
    a.train_step(batch, **HYPER)
    params, opt = engine_state(a)
    save_checkpoint(tmp_path / "0", iteration=0, params=params, optimizer_state=opt)
    b = _engine(cfg, tcfg, t_ibot, qkv_bias, P, B, M)           # a fresh build loads the frozen teacher again
    ck = load_checkpoint(tmp_path / "0")
    load_engine_state(b, ck["model_params"], ck["optimizer_state"])
    assert b.step_count == a.step_count == 1
    for e in (a, b):
        e.train_step(batch, **HYPER)
    ta, tb = _bits(a), _bits(b)
    for k in ta:
        assert torch.equal(ta[k], tb[k]), k
    assert a.read_metrics()["total_loss"] == b.read_metrics()["total_loss"]


@pytest.mark.parametrize("m,k,n,bn", [(8352, 4096, 12288, 0), (8352, 4096, 12288, 64), (333, 320, 200, 128),
                                      (130, 72, 136, 64), (1000, 4096, 12296, 0)])
def test_plain_forward_gemm_matches_runtime_epilogue(m, k, n, bn):
    """(0, 1, no flags): the qkv projection of a teacher without a qkv bias (vit_7b: K = 4096, N = 12 288 at B = 16,
    8352 teacher tokens), and ragged M / N / K."""
    from gemm_epilogue_helpers import BF16_TOL, fixed_and_runtime, inputs, reference, rel
    torch.manual_seed(m + n)
    x = inputs((0, 1), (), m, k, n, k ** -0.5)
    out, _ = fixed_and_runtime(x, bn)
    assert rel(out, reference(x, 1.0)[1]) < BF16_TOL


def test_do_train_distills_from_a_saved_run_and_resumes(tmp_path):
    """A ViT-B run saved by do_train teaches a ViT-S student through the YAML keys; the resumed student run loads the
    frozen teacher again (it is not in the student's checkpoint)."""
    import math
    import yaml
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train.train import do_train
    heads = {"dino": {"head_n_prototypes": 1024, "head_hidden_dim": 256, "head_bottleneck_dim": 64},
             "ibot": {"head_n_prototypes": 512, "head_hidden_dim": 128, "head_bottleneck_dim": 32}}
    t_yaml = {"student": {"arch": "vit_base", "n_storage_tokens": 4, "norm_layer": "layernormbf16"},
              "dino": dict(heads["dino"], head_hidden_dim=384), "ibot": dict(heads["ibot"], head_bottleneck_dim=48),
              "train": {"batch_size_per_gpu": 2, "output_dir": str(tmp_path / "teacher")},
              "checkpointing": {"period": 1, "max_to_keep": 1}}
    (tmp_path / "teacher.yaml").write_text(yaml.safe_dump(t_yaml))
    t_cfg = setup_config(DinoV3SetupArgs(config_file=str(tmp_path / "teacher.yaml")))
    do_train(t_cfg, SSLMetaArch(t_cfg), max_iters=2, print_freq=1)
    opts = ["student.arch=vit_small", "train.batch_size_per_gpu=2", f"train.output_dir={tmp_path / 'student'}",
            "checkpointing.period=1", "distillation.enabled=true", f"distillation.full_cfg_path={tmp_path / 'teacher.yaml'}",
            f"distillation.checkpoint_path={tmp_path / 'teacher' / 'ckpt' / '1'}"]
    opts += [f"{h}.{k}={v}" for h, kv in heads.items() for k, v in kv.items()]
    cfg = setup_config(DinoV3SetupArgs(opts=opts))
    arch = SSLMetaArch(cfg)
    assert arch.distill_config.embed_dim == 768 and arch.distill_config.head_dims("dino_head") == (384, 64, 1024)
    m = do_train(cfg, arch, max_iters=2, print_freq=1)
    assert math.isfinite(m["total_loss"])
    frozen = [t.clone() for s in arch.engine.t_net.mods.values() for t in (s.bf16, s.vecs)]
    arch2 = SSLMetaArch(cfg)
    m2 = do_train(cfg, arch2, resume=True, max_iters=3, print_freq=1)
    assert arch2.engine.step_count == 3 and math.isfinite(m2["total_loss"])
    for a, b in zip(frozen, [t for s in arch2.engine.t_net.mods.values() for t in (s.bf16, s.vecs)]):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
