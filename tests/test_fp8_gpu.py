"""-m gpu: the FP8 GEMM and quantizers against the FP8 arithmetic of tests/fp8_oracle.py.

  (1) d3_quant_rows_e4m3 / d3_quant_cols_e4m3_t give the oracle quantizer's bits and scales;
  (2) d3_gemm_e4m3 against the float64 product of the dequantised operands, for every epilogue the blocks use, on
      ragged M / N (fp32 outputs within 1e-3 of the largest magnitude, bf16 outputs at bf16 tolerance);
  (3) K = 4096 with all-positive operands: promoting the tensor core's sums into fp32 keeps every element within 5e-4 relative;
  (4) two calls give the same bits, and K % 16 != 0 or misaligned operands are refused;
  (5) one Engine(fp8=True) step against the FP8 oracle (with the engine's bf16 storage points, Emu(True)), at the loss
      tolerances of test_engine_gpu.check, and nearer to it than to the bf16 oracle (the step did not run bf16);
  (6) remat gives the bits of stashing (but for the MLP LayerScale tail, whose two kernels differ in bf16 as well);
  (7) two FP8 steps give the same bits;
  (8) Gram-anchoring and distillation steps with FP8 are finite and match the FP8 oracle's losses within the loss
      tolerances of their bf16 tests.
The gradients are compared at a looser bound than bf16's 3e-2: e4m3 rounding is a step function, and the engine's and
the oracle's operands, equal to bf16 rounding, land on different sides of a rounding boundary for a few per cent of the
elements; each such element moves by a whole e4m3 step (2^-4 relative).  Measured global relative L2: 0.066 (mlp),
0.106 (swiglu64), where the FP8 oracle itself is 0.13 / 0.31 away from the bf16 oracle.
"""
import dataclasses

import pytest
import torch

from fp8_oracle import dequant, fp8_oracle, quant_rows as oracle_quant_rows

pytestmark = pytest.mark.gpu

bf16, f32, u8 = torch.bfloat16, torch.float32, torch.uint8
HYPER = dict(lr=1e-3, wd=0.04, last_layer_lr=5e-4, momentum=0.99, teacher_temp=0.05)


def _wide_range(R, C, seed):
    """bf16 rows whose maxima span the bf16 range (subnormal to 2^120), with zero rows and exact zeros mixed in."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, C, generator=g, dtype=torch.float64)
    e = torch.randint(-130, 120, (R, 1), generator=g).double()
    x = x * torch.pow(2.0, e)
    x[::7] = 0.0
    x[:, ::5] = 0.0
    return x.to(bf16)


@pytest.mark.parametrize("R,C,pad", [(37, 200, 0), (64, 256, 0), (129, 1024, 8), (5, 72, 24)])
def test_quant_rows_matches_oracle_bits(R, C, pad):
    from dinov3_jax import ops
    big = _wide_range(R, C + pad, R + C).cuda()
    x = big[:, pad:]                                   # a strided view (row stride C + pad)
    q = torch.full((R, C + 16), 0x55, dtype=u8, device="cuda")
    s = torch.empty(R, dtype=f32, device="cuda")
    ops.quant_rows(x, q, s)
    qo, so = oracle_quant_rows(x.cpu())
    assert torch.equal(s.cpu(), so)
    assert torch.equal(q[:, :C].cpu(), qo)
    assert bool((q[:, C:] == 0x55).all())               # nothing written past C


@pytest.mark.parametrize("R,C", [(200, 72), (1024, 3072), (96, 130)])
def test_quant_cols_t_matches_oracle_bits(R, C):
    from dinov3_jax import ops
    W = _wide_range(R, C, 3 * R + C).cuda()
    ld = (R + 15) // 16 * 16
    qt = torch.empty(C, ld, dtype=u8, device="cuda")
    s = torch.empty(C, dtype=f32, device="cuda")
    ops.quant_cols_t(W, qt, s)
    qo, so = oracle_quant_rows(W.cpu().T)
    assert torch.equal(s.cpu(), so)
    assert torch.equal(qt[:, :R].cpu(), qo)


def test_quantizer_non_finite_inputs_stay_non_finite():
    from dinov3_jax import ops
    x = torch.tensor([[float("inf"), 3.0, float("nan"), -float("inf")] + [1.0] * 12], dtype=bf16, device="cuda")
    q = torch.empty(1, 16, dtype=u8, device="cuda")
    s = torch.empty(1, dtype=f32, device="cuda")
    ops.quant_rows(x, q, s)
    qo, so = oracle_quant_rows(x.cpu())
    assert torch.equal(q.cpu(), qo) and torch.equal(s.cpu(), so)


def _operands(M, N, K, seed, positive=False):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g)
    b = torch.randn(N, K, generator=g) * 0.05
    if positive:
        a, b = a.abs() + 0.01, b.abs() + 0.001
    qa, sa = oracle_quant_rows(a)
    qb, sb = oracle_quant_rows(b)
    ref = dequant(qa, sa) @ dequant(qb, sb).T
    _operands.abs_sum = dequant(qa, sa).abs() @ dequant(qb, sb).abs().T     # sum_k |a_k b_k| of every output
    return [t.cuda() for t in (qa, sa, qb, sb)], ref


def _gelu(u):
    return torch.nn.functional.gelu(u, approximate="tanh")


def _gelu_grad(u):
    t = torch.tanh(0.7978845608028654 * (u + 0.044715 * u ** 3))
    return 0.5 * (1 + t) + 0.5 * u * (1 - t * t) * 0.7978845608028654 * (1 + 3 * 0.044715 * u * u)


EPILOGUES = {
    "plain": dict(), "bias": dict(bias=True), "bias_gelu": dict(bias=True, gelu=True),
    "bias_gelu_pre": dict(bias=True, gelu=True, pre=True),
    "proj": dict(bias=True, gamma=True, resid=True, f32=True),
    "proj_pre": dict(bias=True, pre=True, gamma=True, resid=True, f32=True),
    "fc2_gelu": dict(bias=True, gelu=True, gamma=True, resid=True, f32=True),
    "fc2_gelu_pre": dict(bias=True, gelu=True, pre=True, gamma=True, resid=True, f32=True),
    "dgelu": dict(dgelu=True), "dgrad_f32": dict(f32=True), "dgrad_accum": dict(f32=True, accum=True),
}


@pytest.mark.parametrize("M,N,K", [(300, 192, 256), (128, 64, 1024), (77, 130, 144)])
@pytest.mark.parametrize("name", list(EPILOGUES))
def test_gemm_e4m3_epilogues_against_float64(name, M, N, K):
    from dinov3_jax import ops
    f = EPILOGUES[name]
    (qa, sa, qb, sb), acc = _operands(M, N, K, M + N + K)
    g = torch.Generator().manual_seed(7)
    bias = torch.randn(N, generator=g) * 0.1
    gamma = torch.rand(N, generator=g) + 0.5
    resid = torch.randn(M, N, generator=g)
    u = torch.randn(M, N, generator=g).to(bf16)
    old = torch.randn(M, N, generator=g)
    v = acc.clone()
    if f.get("bias"):
        v = v + bias.double()
    pre = v.clone()
    if f.get("gelu"):
        v = _gelu(v)
    if f.get("dgelu"):
        v = v * _gelu_grad(u.double())
    if f.get("gamma"):
        v = v * gamma.double()
    if f.get("resid"):
        v = v + resid.double()
    if f.get("accum"):
        v = v + old.double()
    out = (old.clone() if f.get("accum") else torch.zeros(M, N)).to(f32 if f.get("f32") else bf16).cuda()
    store_pre = torch.empty(M, N, dtype=bf16, device="cuda") if f.get("pre") else None
    ops.gemm_e4m3(qa, sa, qb, sb, out, bias=bias.cuda() if f.get("bias") else None, gelu=bool(f.get("gelu")),
                  store_pre=store_pre, dgelu_of=u.cuda() if f.get("dgelu") else None,
                  gamma=gamma.cuda() if f.get("gamma") else None, resid=resid.cuda() if f.get("resid") else None,
                  accum=bool(f.get("accum")))
    # elementwise: |out - ref| <= rtol |ref| + 5e-4 sum_k |a_k b_k| (times gamma, and 1.2 for GELU / GELU'): the
    # tensor core's FP8 sums err relative to the magnitude of their terms, which an output that cancels does not show;
    # 5e-4 is the bound of the all-positive K = 4096 test below, where the two coincide
    rtol = 1e-3 if f.get("f32") else 1e-2
    atol = 5e-4 * _operands.abs_sum * (gamma.double() if f.get("gamma") else 1.0)
    if f.get("gelu") or f.get("dgelu"):
        atol = atol * 1.2
    _close(out, v, rtol, atol, name)
    if store_pre is not None:
        _close(store_pre, pre, 1e-2, 5e-4 * _operands.abs_sum, name + "/pre")


def _close(got, ref, rtol, atol, what):
    d = (got.cpu().double() - ref).abs()
    bound = rtol * ref.abs() + atol
    bad = d > bound
    assert not bool(bad.any()), (what, int(bad.sum()), float((d / bound).max()))


def test_gemm_e4m3_runtime_epilogue_on_odd_n():
    """N odd runs the run-time-flag epilogue; it agrees with the fixed-flag instance on the columns they share."""
    from dinov3_jax import ops
    (qa, sa, qb, sb), acc = _operands(200, 132, 512, 3)
    out = torch.empty(200, 132, dtype=f32, device="cuda")
    ops.gemm_e4m3(qa, sa, qb, sb, out)
    assert float((out.cpu().double() - acc).abs().max() / acc.abs().max()) < 1e-3
    odd = torch.empty(200, 131, dtype=f32, device="cuda")
    ops.gemm_e4m3(qa, sa, qb[:131], sb[:131], odd)
    assert torch.equal(out[:, :131], odd)


def test_gemm_e4m3_promotion_at_k4096():
    from dinov3_jax import ops
    (qa, sa, qb, sb), acc = _operands(256, 256, 4096, 11, positive=True)
    out = torch.empty(256, 256, dtype=f32, device="cuda")
    ops.gemm_e4m3(qa, sa, qb, sb, out)
    rel = float(((out.cpu().double() - acc).abs() / acc.abs()).max())
    assert rel <= 5e-4, rel


def test_gemm_e4m3_is_deterministic_and_checks_arguments():
    from dinov3_jax import ops
    from dinov3_jax._native import NativeError
    (qa, sa, qb, sb), _ = _operands(1000, 1024, 1024, 5)
    o1 = torch.empty(1000, 1024, dtype=f32, device="cuda")
    o2 = torch.empty_like(o1)
    ops.gemm_e4m3(qa, sa, qb, sb, o1)
    ops.gemm_e4m3(qa, sa, qb, sb, o2)
    assert torch.equal(o1, o2)
    with pytest.raises(NativeError, match="multiple of 16"):
        ops.gemm_e4m3(qa[:, :1000], sa, qb[:, :1000], sb, o1)
    with pytest.raises(NativeError, match="aligned"):
        ops.gemm_e4m3(qa[:, 8:1016], sa, qb[:, 8:1016], sb, o1)


# ---------------------------------------------------------------------------------------------------------- the step
def _cfg(kind):
    from oracle import tiny_cfg
    if kind == "mlp_hd64":
        return tiny_cfg()
    return tiny_cfg(embed_dim=256, heads=2, ffn_layer="swiglu", swiglu_align=64, n_storage=4, mask_k_bias=True,
                    ln_eps=1e-5, layerscale=0.5)


def _step(cfg, B, batch, P, fp8=True, **kw):
    from dinov3_jax.engine import Engine, from_oracle_cfg
    eng = Engine(from_oracle_cfg(cfg), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1), fp8=fp8, **kw)
    eng.params.load_reference_tree(P)
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    torch.cuda.synchronize()
    return eng, {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}


def _rel(ge, go):
    num = sum(((ge[k].reshape(g.shape) - g) ** 2).sum() for k, g in go.items())
    return float(torch.sqrt(num / sum((g ** 2).sum() for g in go.values())))


@pytest.mark.parametrize("kind", ["mlp_hd64", "swiglu64_storage_maskk_hd128"])
def test_fp8_step_matches_the_fp8_oracle(kind):
    from oracle.batch import synthetic_batch
    from oracle.model import Emu, init_params
    from oracle.step import init_opt_state, train_step
    cfg, B = _cfg(kind), 4
    P = init_params(cfg, 0, perturb=0.05)
    batch = synthetic_batch(cfg, B, 0)
    eng, grads_e = _step(cfg, B, batch, P)
    met = eng.read_metrics()
    with fp8_oracle():
        _, _, loss, m, grads8 = train_step(P, init_opt_state(P), batch, cfg, emu=Emu(True), **HYPER)
    _, _, _, _, grads16 = train_step(P, init_opt_state(P), batch, cfg, emu=Emu(True), **HYPER)
    assert abs(met["total_loss"] - loss.item()) <= 1e-3 * abs(loss.item())
    for k in ("dino_local_crops_loss", "dino_global_crops_loss", "ibot_loss"):
        assert abs(met[k] - float(m[k])) <= 1e-3 * abs(float(m[k])), k
    # KoLeo (log of each cls token's nearest-neighbour distance over B = 4) moves with single e4m3 rounding flips:
    # measured 2.1e-2 (mlp), against bf16's 2e-2 bound
    assert abs(met["koleo_loss"] - float(m["koleo_loss"])) <= 5e-2 * max(abs(float(m["koleo_loss"])), 0.05)
    d8, d16 = _rel(grads_e, grads8), _rel(grads_e, grads16)
    assert d8 < 0.15, d8
    assert d8 < 0.6 * d16, (d8, d16)     # measured 0.50 (mlp) and 0.32 (swiglu64) of the distance to bf16


def test_fp8_remat_and_repeat_give_the_same_bits():
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    cfg, B = _cfg("swiglu64_storage_maskk_hd128"), 3
    P = init_params(cfg, 1, perturb=0.05)
    batch = synthetic_batch(cfg, B, 1)
    (e0, g0), (e1, g1), (e2, g2) = _step(cfg, B, batch, P), _step(cfg, B, batch, P), _step(cfg, B, batch, P, remat=True)
    assert all(torch.equal(g1[k], g0[k]) for k in g0)
    assert e1.read_metrics() == e0.read_metrics()
    # remat recomputes the block through the same FP8 path; only the MLP branch's LayerScale tail (ls_act_bwd instead of
    # the LayerNorm backward's fused tail) sums in another order, in bf16 as well
    tail = ("/ls2/gamma", "/mlp/w3/bias", "/mlp/Dense_1/bias")
    assert all(torch.equal(g2[k], g0[k]) for k in g0 if not k.endswith(tail))
    assert e2.read_metrics()["total_loss"] == e0.read_metrics()["total_loss"]


def test_fp8_gram_step_matches_the_fp8_oracle():
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import Emu, init_params
    from oracle.step import ssl_forward
    cfg, B, W = tiny_cfg(layerscale=0.5), 3, 25.0
    P = init_params(cfg, 6, perturb=0.05)
    batch = synthetic_batch(cfg, B, 6)
    ecfg = dataclasses.replace(from_oracle_cfg(cfg), gram_use_loss=True, gram_loss_weight=W, gram_ema_teacher=False,
                               gram_it_load_ema_teacher=0)
    eng = Engine(ecfg, B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1), fp8=True)
    eng.params.load_reference_tree(P)
    tree = {k[len("teacher_backbone/"):]: v for k, v in init_params(cfg, 7, perturb=0.05).items()
            if k.startswith("teacher_backbone/")}
    eng.gram_teacher_load(tree)
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    met = eng.read_metrics()
    full = dict(P)
    full.update({"gram_backbone/" + k: v for k, v in tree.items()})
    gram = dict(weight=W, ema_teacher=False, normalized=True, img_level=False, remove_neg=False,
                remove_only_teacher_neg=False, tokens_used="all")
    with fp8_oracle(), torch.no_grad():
        loss, m = ssl_forward(full, batch, HYPER["teacher_temp"], cfg, emu=Emu(True), gram=gram)
    assert all(torch.isfinite(torch.tensor(v)) for v in met.values())
    assert abs(met["gram_loss"] - float(m["gram_loss"])) < 2e-2 * float(m["gram_loss"])
    assert abs(met["total_loss"] - float(loss)) < 2e-3 * abs(float(loss))


def test_fp8_distillation_step_matches_the_fp8_oracle():
    from dinov3_jax.engine import Engine
    from distill_helpers import distill_train_step, frozen_tree
    from oracle.step import init_opt_state
    from test_distill_gpu import S_IBOT, _ecfg, _setup
    cfg, tcfg, t_ibot, qkv_bias, P, batch = _setup("vit_base")
    B = batch["global_batch_size"]
    eng = Engine(_ecfg(cfg, S_IBOT), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1),
                 distill=_ecfg(tcfg, t_ibot, qkv_bias), fp8=True)
    eng.params.load_reference_tree({k: v.float() for k, v in P.items() if not k.startswith("distill_")})
    eng.distill_teacher_load({m: {k: v.float() for k, v in t.items()} for m, t in frozen_tree(P).items()})
    assert eng.t_net.fp8 and eng.student_net.fp8
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    met = eng.read_metrics()
    with fp8_oracle():
        _, _, loss, m, _ = distill_train_step(P, init_opt_state(P), batch, cfg, tcfg, **HYPER)
    assert all(torch.isfinite(torch.tensor(v)) for v in met.values())
    assert abs(met["total_loss"] - loss.item()) <= 1e-3 * abs(loss.item())
    for k in ("dino_local_crops_loss", "dino_global_crops_loss", "ibot_loss"):
        assert abs(met[k] - float(m[k])) <= 1e-3 * abs(float(m[k])), k

