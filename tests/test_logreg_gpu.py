"""GPU: the logistic-regression evaluation.  The objective and gradient of a batched evaluation against float64 (across
problem counts, class paddings, row chunks and feature widths, and bit-identical on a rerun); the L-BFGS sweep
against scipy's optimum for every strength of the grid, batched and alone; and the evaluation end to end on a small
random-weight backbone (the JSON, byte-identical reruns, val top-1 against scipy at the chosen strength)."""
import json
import math

import numpy as np
import pytest
import torch

import logreg_oracle as oracle

pytestmark = pytest.mark.gpu
f64 = torch.float64

# (G problems, classes, N rows, K features, chunk rows): every G, class count, N and K at least once, chunk crossings
CASES = [(1, 2, 1, 384, 8192), (3, 10, 7, 1024, 8192), (45, 101, 1000, 384, 256), (3, 1000, 1000, 2048, 8192),
         (1, 101, 40000, 1024, 8192), (45, 10, 40000, 2048, 8192), (3, 2, 40000, 384, 8192),
         (45, 1000, 7, 1024, 8192), (1, 1000, 40000, 384, 8192), (45, 2, 1000, 2048, 512)]


@pytest.mark.parametrize("G,C,N,K,chunk", CASES)
def test_objective_and_gradient_match_float64(native, G, C, N, K, chunk):
    from dinov3_jax.eval.logreg import LogRegSweep
    g = torch.Generator().manual_seed(G * 7 + C + N + K)
    X = torch.randn(N, K, generator=g)
    y = torch.randint(0, C, (N,), generator=g)
    cs = [float(v) for v in np.logspace(-3, 3, G)] if G > 1 else [1.0]
    sw = LogRegSweep(C, cs, chunk_rows=chunk, device="cuda")
    sw._prepare(X, y)
    Cp = sw.Cp
    theta = torch.zeros(G, sw.P)
    W = torch.randn(G, C, K, generator=g) * (2.0 / math.sqrt(K))
    b = torch.randn(G, C, generator=g)
    theta[:, :Cp * K].view(G, Cp, K)[:, :C] = W
    theta[:, Cp * K:Cp * K + C] = b
    theta = theta.cuda()
    out = sw._evaluate(theta, list(range(G)))
    grad = sw.grad_out.clone()
    out2 = sw._evaluate(theta, list(range(G)))
    assert np.array_equal(out, out2) and torch.equal(grad, sw.grad_out), "two evaluations differ"
    Xd, yd = X.cuda().double(), y.cuda()
    for p in range(G):
        F, gW, gb = oracle.objective(W[p].cuda().double(), b[p].cuda().double(), Xd, yd, cs[p])
        assert abs(out[p, 0] - F) <= 1e-5 * abs(F), (p, out[p, 0], F)
        got = grad[p, :Cp * K].view(Cp, K)
        assert (got[C:] == 0).all() and (grad[p, Cp * K + C:] == 0).all()
        want = torch.cat([gW.reshape(-1), gb])
        have = torch.cat([got[:C].reshape(-1), grad[p, Cp * K:Cp * K + C]]).double()
        rel = ((have - want).norm() / want.norm()).item()
        assert rel <= 1e-5, (p, cs[p], rel)
        assert out[p, 2] == pytest.approx(have.abs().max().item(), rel=1e-6)


def test_split_operands_beyond_65535_rows(native):
    """hi + lo parts of every row, in both operand layouts, at a row count above one grid dimension's limit."""
    from dinov3_jax import ops
    N, K, chunk = 70000, 24, 8192
    X = torch.randn(N, K, generator=torch.Generator().manual_seed(0)).cuda()
    rows = -(-N // chunk) * chunk
    xa = torch.empty(rows, 3 * K, dtype=torch.bfloat16, device="cuda")
    xg = torch.empty(3 * rows, K, dtype=torch.bfloat16, device="cuda")
    ops.logreg_split_x(X, chunk, xa, xg)
    h = X.to(torch.bfloat16)
    lo = (X - h.float()).to(torch.bfloat16)
    assert torch.equal(xa[:N], torch.cat([h, h, lo], 1)) and (xa[N:] == 0).all()
    g = xg.view(-1, 3, chunk, K)
    hp = torch.zeros(rows, K, dtype=torch.bfloat16, device="cuda")
    lp = hp.clone()
    hp[:N], lp[:N] = h, lo
    hp, lp = hp.view(-1, chunk, K), lp.view(-1, chunk, K)
    assert torch.equal(g[:, 0], hp) and torch.equal(g[:, 1], lp) and torch.equal(g[:, 2], hp)


# ------------------------------------------------------------------------------------------------ solver vs scipy
@pytest.fixture(scope="module")
def fixture_fits():
    X, y = oracle.clustered(2500, 256, 10, seed=5)
    Xtr, ytr, Xva = X[:2000], y[:2000], X[2000:]
    fits = {c: oracle.scipy_fit(Xtr, ytr, 10, c, device="cuda") for c in oracle.default_grid()}
    return Xtr, ytr, Xva, fits


def _check(sw, g, c, Xtr, ytr, Xva, fit, preds):
    """The failed bounds of problem g (an empty list when it meets them all)."""
    Ws, bs, Fs = fit
    W, b = sw.W[g].double(), sw.b[g].double()
    F = oracle.objective(W, b, Xtr.cuda(), ytr.cuda(), c)[0]
    info, bad = sw.info[g], []
    if abs(F - Fs) > 1e-6 * abs(Fs):
        bad.append(("objective", c, F, Fs, info))
    if c <= 1e2:
        rel = (torch.cat([W.reshape(-1), b]) - torch.cat([Ws.reshape(-1), bs])).norm() / torch.cat(
            [Ws.reshape(-1), bs]).norm()
        if rel.item() > 1e-3:
            bad.append(("parameters", c, rel.item(), info))
    z = Xva.cuda().double() @ Ws.T + bs
    top2 = z.topk(2, 1).values
    margin = top2[:, 0] - top2[:, 1]
    differ = preds.long() != z.argmax(1)
    if (differ & (margin >= 1e-4)).any():
        bad.append(("predictions", c, int(differ.sum()), info))
    return bad


def test_sweep_matches_scipy_for_every_strength(native, fixture_fits):
    from dinov3_jax.eval.logreg import LogRegSweep
    Xtr, ytr, Xva, fits = fixture_fits
    grid = oracle.default_grid()
    sw = LogRegSweep(10, grid, device="cuda").fit(Xtr, ytr)
    preds = sw.predict(Xva, k=1)[:, :, 0]
    bad = [b for g, c in enumerate(grid) for b in _check(sw, g, c, Xtr, ytr, Xva, fits[c], preds[:, g])]
    assert not bad, bad
    assert {i["stop"] for i in sw.info} <= {"gtol", "ftol", "max_iter", "line_search"}


@pytest.mark.parametrize("index", [0, 22, 36, 44])
def test_one_strength_alone_meets_the_same_bounds(native, fixture_fits, index):
    from dinov3_jax.eval.logreg import LogRegSweep
    Xtr, ytr, Xva, fits = fixture_fits
    c = oracle.default_grid()[index]
    sw = LogRegSweep(10, [c], device="cuda").fit(Xtr, ytr)
    bad = _check(sw, 0, c, Xtr, ytr, Xva, fits[c], sw.predict(Xva, k=1)[:, 0, 0])
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ end to end
def _npz(path, n, seed):
    rng = np.random.default_rng(seed)
    labels = np.arange(n) % 3
    base = np.array([[200, 40, 40], [40, 200, 40], [40, 40, 200]], np.int16)
    images = base[labels][:, None, None, :] + rng.integers(-60, 60, (n, 80, 80, 3))
    np.savez(path, images=np.clip(images, 0, 255).astype(np.uint8), labels=labels)


def test_do_logreg_eval_end_to_end(native, tmp_path):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.eval import make_eval_dataset
    from dinov3_jax.eval.logreg import extract_logreg_features
    from dinov3_jax.models import DinoVisionTransformer
    from dinov3_jax.train.train import do_logreg_eval
    from features_helpers import tree
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    flat = init_backbone(ModelCfg(embed_dim=384, depth=2, heads=6, layerscale=0.5), torch.Generator().manual_seed(0))
    model = DinoVisionTransformer(tree(flat), embed_dim=384, n_blocks=2, num_heads=6)
    _npz(tmp_path / "train.npz", 90, 0)
    _npz(tmp_path / "val.npz", 31, 1)
    grid = [1e-4, 1e-2, 1.0, 1e2, 1e4]
    opts = [f"train.output_dir={tmp_path / 'out'}", f"evaluation.logreg.train_dataset_path={tmp_path / 'train.npz'}",
            f"evaluation.logreg.val_dataset_path={tmp_path / 'val.npz'}", "evaluation.logreg.resize_size=72",
            "evaluation.logreg.crop_size=64", "evaluation.logreg.batch_size=16", "evaluation.logreg.num_workers=0"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    config.evaluation.logreg.C_values = grid
    res = do_logreg_eval(config, model, "manual_0")
    path = tmp_path / "out" / "eval" / "manual_0" / "results_logreg.json"
    first = path.read_bytes()
    written = json.loads(first)
    for key in ("sweep", "best_C", "refit", "top1", "top5", "mean_per_class", "protocol", "config", "n_holdout"):
        assert key in written, key
    assert written["best_C"] in grid and len(written["sweep"]) == 5 and res["top1"] == written["top1"]
    for row in written["sweep"]:
        assert set(row) == {"C", "holdout_top1", "iterations", "evaluations", "stop"}
    assert written["n_holdout"] == 9 and written["n_fit"] == 81 and written["n_val"] == 31
    do_logreg_eval(config, model, "manual_0")
    assert path.read_bytes() == first
    kw = dict(batch_size=16, num_workers=0, resize_size=72, crop_size=64)
    tr_f, tr_y = extract_logreg_features(model, make_eval_dataset(str(tmp_path / "train.npz")), **kw)
    va_f, va_y = extract_logreg_features(model, make_eval_dataset(str(tmp_path / "val.npz")), **kw)
    Ws, bs, _ = oracle.scipy_fit(tr_f.cpu(), tr_y.cpu(), 3, written["best_C"], device="cuda")
    top1 = 100.0 * ((va_f.double() @ Ws.T + bs).argmax(1) == va_y).double().mean().item()
    assert abs(top1 - written["top1"]) <= 100.0 / 31 + 1e-9, (top1, written["top1"])
