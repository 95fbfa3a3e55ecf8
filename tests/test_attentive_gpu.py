"""GPU: the attentive probe.  Forward and backward against the unfolded float64 probe (tests/attentive_oracle.py) on
bf16-exact tokens across widths, frame counts, patch counts and batch sizes, with query scales that make the softmax
sharp; byte-identical parameters after 20 steps on a rerun; a probe that learns a task carried by frame 0 only; and
`do_attentive_eval` end to end on a small random-weight backbone (the JSON, byte-identical reruns, any worker count).

Bounds.  The pooling and the query path run in fp32, so the pooled output a = Wv ybar + bv (taken in float64 from the
kernel's ybar) is within 1e-3 relative L2 of the oracle's: the fp32 online softmax over up to 4 096 tokens, at scores
up to ~50, keeps ~1e-5.  The loss passes through bf16 GEMM operands (ybar, a, LN2's output, the MLP activations, z):
each rounding is <= 2^-9 relative, and a batch-mean cross-entropy of random logits moves by < 1e-3 of itself.  A
single clip's loss is not averaged: at D = 1536 it measured 1.4e-3 off, so the single-clip case runs at D = 384.  Gradients
take a few more bf16 roundings (the classifier, MLP and attention output gradients) and the softmax backward's
cancellation p (dp - c): 1e-2 relative L2 per parameter.  The matrices the GEMMs read are set to bf16-exact values
so that only the roundings above remain."""
import json

import numpy as np
import pytest
import torch

import attentive_oracle as oracle

pytestmark = pytest.mark.gpu
f64 = torch.float64
GEMM_MATS = ("Wv", "Wo", "W1", "W2", "Wc")

# (D, H, T, P, B, classes, query scale): every D, T, P and B at least once; scales 8 and 20 make the softmax sharp
CASES = [(384, 6, 1, 196, 1, 10, 1.0), (384, 6, 16, 196, 3, 400, 8.0), (1024, 16, 16, 196, 16, 400, 1.0),
         (1024, 16, 1, 256, 3, 10, 20.0), (1536, 24, 16, 256, 3, 10, 8.0), (1536, 24, 1, 196, 16, 400, 20.0),
         (1024, 16, 16, 256, 16, 10, 20.0), (384, 6, 16, 256, 16, 10, 20.0)]


def _probe(D, H, T, C, B, params, **kw):
    from dinov3_jax import ops
    from dinov3_jax.eval.attentive import AttentiveProbe
    probe = AttentiveProbe(D, H, T, C, B, 100, device="cuda", **kw)
    for name, v in params.items():
        t = probe.params[name]
        src = v.float()
        if name in GEMM_MATS:
            src = src.bfloat16().float()
        if name in ("Wc", "bc"):
            t.zero_()
            t[:C].copy_(src.cuda())
        else:
            t.copy_(src.cuda())
    ops.cast_f32_bf16(probe.p[:probe.n_mats], probe.p_bf16)
    return probe


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


@pytest.mark.parametrize("D,H,T,P,B,C,qs", CASES)
def test_forward_and_backward_match_the_unfolded_probe(native, D, H, T, P, B, C, qs):
    params = oracle.make_params(D, H, T, C, seed=D + T + P + B, query_scale=qs, dtype=torch.float32)
    probe = _probe(D, H, T, C, B, params)
    exact = {k: (v.bfloat16() if k in GEMM_MATS else v).double() for k, v in params.items()}
    g = torch.Generator().manual_seed(B * 31 + P)
    x = (torch.randn(B, T * P, D, generator=g) * 2).bfloat16()
    labels = torch.randint(0, C, (B,), generator=g)
    loss = probe.gradients(x.cuda(), labels).item()
    ref = oracle.unfolded({k: v.cuda() for k, v in exact.items()}, x.double().cuda(), T, H, labels.cuda())
    dh = D // H
    Wv = exact["Wv"].cuda()
    a = torch.cat([probe.ybar[:B, h].double() @ Wv[h * dh:(h + 1) * dh].T for h in range(H)], 1) + exact["bv"].cuda()
    assert _rel(a, ref["a"]) <= 1e-3
    assert abs(loss - ref["loss"].item()) <= 1e-3 * abs(ref["loss"].item())
    for name in oracle.NAMES:
        got = probe.grads[name][:C] if name in ("Wc", "bc") else probe.grads[name]
        assert _rel(got, ref["grads"][name]) <= 1e-2, (name, _rel(got, ref["grads"][name]))


def test_twenty_steps_are_byte_identical(native):
    D, H, T, P, B, C = 384, 6, 4, 49, 8, 7

    def run():
        from dinov3_jax.eval.attentive import AttentiveProbe
        probe = AttentiveProbe(D, H, T, C, B, 20, lr=1e-3, warmup_iterations=3, seed=3, device="cuda")
        g = torch.Generator().manual_seed(0)
        for it in range(20):
            x = (torch.randn(B, T * P, D, generator=g) * 2).bfloat16().cuda()
            probe.step(x, torch.randint(0, C, (B,), generator=g), it)
        return probe.p.cpu().numpy().tobytes()

    assert run() == run()


def test_probe_learns_a_label_carried_by_frame_0(native):
    """Every frame carries a class direction; only frame 0's is the label's, the others are random classes.  Without
    the temporal embedding the pooling could not tell frame 0 apart."""
    from dinov3_jax.eval.attentive import AttentiveProbe
    D, H, T, P, B, C, steps = 384, 6, 4, 16, 32, 4, 400
    g = torch.Generator().manual_seed(0)
    dirs = torch.randn(C, D, generator=g)

    def batch(n):
        y = torch.randint(0, C, (n,), generator=g)
        other = torch.randint(0, C, (n, T), generator=g)
        other[:, 0] = y
        x = torch.randn(n, T, P, D, generator=g) + 1.5 * dirs[other][:, :, None, :]
        return x.reshape(n, T * P, D).bfloat16().cuda(), y

    probe = AttentiveProbe(D, H, T, C, B, steps, lr=3e-3, warmup_iterations=20, seed=0, device="cuda")
    for it in range(steps):
        x, y = batch(B)
        probe.step(x, y, it)
    hits = 0
    for _ in range(8):
        x, y = batch(B)
        hits += int((probe.forward(x)[:, :C].argmax(1).cpu() == y).sum())
    assert hits / (8 * B) >= 0.9, hits


def _npz(path, n, seed):
    rng = np.random.default_rng(seed)
    labels = np.arange(n) % 3
    base = np.array([[200, 40, 40], [40, 200, 40], [40, 40, 200]], np.int16)
    videos = base[labels][:, None, None, None, :] + rng.integers(-60, 60, (n, 10, 40, 56, 3))
    np.savez(path, videos=np.clip(videos, 0, 255).astype(np.uint8), labels=labels)


def test_do_attentive_eval_end_to_end(native, tmp_path):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.models import DinoVisionTransformer
    from dinov3_jax.train.train import do_attentive_eval
    from features_helpers import tree
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    flat = init_backbone(ModelCfg(embed_dim=384, depth=2, heads=6, layerscale=0.5), torch.Generator().manual_seed(0))
    model = DinoVisionTransformer(tree(flat), embed_dim=384, n_blocks=2, num_heads=6)
    _npz(tmp_path / "train.npz", 12, 0)
    _npz(tmp_path / "val.npz", 5, 1)
    opts = [f"train.output_dir={tmp_path / 'out'}",
            f"evaluation.attentive.train_dataset_path={tmp_path / 'train.npz'}",
            f"evaluation.attentive.val_dataset_path={tmp_path / 'val.npz'}", "evaluation.attentive.crop_size=32",
            "evaluation.attentive.batch_size=4", "evaluation.attentive.num_frames=4",
            "evaluation.attentive.frame_step=2", "evaluation.attentive.epochs=2", "evaluation.attentive.num_workers=0"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    config.evaluation.attentive.learning_rates = [1e-3, 1e-2]
    res = do_attentive_eval(config, model, "manual_0")
    path = tmp_path / "out" / "eval" / "manual_0" / "results_attentive.json"
    first = path.read_bytes()
    written = json.loads(first)
    for key in ("probes", "best_probe", "top1", "top5", "mean_per_class", "train_videos", "val_videos", "train_clips",
                "val_clips", "protocol", "config"):
        assert key in written, key
    assert set(written["probes"]) == {"probe_lr_0_00100", "probe_lr_0_01000"} and res["top1"] == written["top1"]
    counts = tuple(written[k] for k in ("train_videos", "val_videos", "train_clips", "val_clips"))
    assert counts == (12, 5, 24, 30)
    do_attentive_eval(config, model, "manual_0")
    assert path.read_bytes() == first
    config.evaluation.attentive.num_workers = 2
    do_attentive_eval(config, model, "manual_0")
    got = json.loads(path.read_bytes())
    got["config"].pop("num_workers"), written["config"].pop("num_workers")
    assert got == written
