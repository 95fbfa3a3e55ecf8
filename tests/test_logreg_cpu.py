"""Logistic-regression evaluation without a GPU: the float64 oracle (tests/logreg_oracle.py) against finite
differences and scipy, the grid and the stratified split, the line search on a known function, the
`evaluation.logreg` block, the --eval logreg flags, the host-side argument checks and what ptxas makes of
csrc/logreg.cu."""
import ctypes as C
import json
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import logreg_oracle as oracle


# ------------------------------------------------------------------------------------------------ oracle
def test_oracle_gradient_matches_central_differences():
    g = torch.Generator().manual_seed(0)
    X = torch.randn(23, 6, generator=g, dtype=torch.float64)
    y = torch.randint(0, 4, (23,), generator=g)
    W = torch.randn(4, 6, generator=g, dtype=torch.float64)
    b = torch.randn(4, generator=g, dtype=torch.float64)
    for c in (1e-2, 1.0, 1e3):
        _, gW, gb = oracle.objective(W, b, X, y, c)
        h = 1e-6
        for i, j in ((0, 0), (3, 5), (2, 1)):
            Wp, Wm = W.clone(), W.clone()
            Wp[i, j] += h; Wm[i, j] -= h
            fd = (oracle.objective(Wp, b, X, y, c)[0] - oracle.objective(Wm, b, X, y, c)[0]) / (2 * h)
            assert abs(fd - gW[i, j].item()) < 1e-8, (c, i, j)
        for i in range(4):
            bp, bm = b.clone(), b.clone()
            bp[i] += h; bm[i] -= h
            fd = (oracle.objective(W, bp, X, y, c)[0] - oracle.objective(W, bm, X, y, c)[0]) / (2 * h)
            assert abs(fd - gb[i].item()) < 1e-8, (c, i)


def test_scipy_optima_are_stationary_over_the_grid():
    X, y = oracle.clustered(300, 16, 4, seed=1)
    for c in oracle.default_grid():
        W, b, _ = oracle.scipy_fit(X, y, 4, c)
        _, gW, gb = oracle.objective(W, b, X, y, c)
        assert max(gW.abs().max().item(), gb.abs().max().item()) < 1e-8, c


def test_default_grid():
    from dinov3_jax.eval.logreg import default_C_values
    grid = default_C_values()
    assert len(grid) == 45 and grid == oracle.default_grid()
    assert grid[0] == pytest.approx(1e-6, rel=1e-12) and grid[-1] == pytest.approx(1e5, rel=1e-12)
    assert all(b / a == pytest.approx(10 ** (11 / 44), rel=1e-12) for a, b in zip(grid, grid[1:]))


def test_stratified_split_is_seeded_covers_every_class_and_is_disjoint():
    from dinov3_jax.eval.logreg import stratified_holdout
    rng = np.random.default_rng(3)
    y = np.concatenate([np.full(n, c) for c, n in enumerate([1, 2, 3, 9, 10, 11, 25, 104])])
    y = y[rng.permutation(y.size)]
    fit, hold = stratified_holdout(y, 0.1, seed=7)
    fit2, hold2 = stratified_holdout(y, 0.1, seed=7)
    assert np.array_equal(fit, fit2) and np.array_equal(hold, hold2)
    assert not np.array_equal(hold, stratified_holdout(y, 0.1, seed=8)[1])
    assert np.intersect1d(fit, hold).size == 0 and np.union1d(fit, hold).size == y.size
    counts = {c: int((y[hold] == c).sum()) for c in range(8)}
    assert counts == {0: 0, 1: 1, 2: 1, 3: 1, 4: 1, 5: 1, 6: 2, 7: 10}
    ofit, ohold = oracle.holdout(y, 0.1, 7)
    assert np.array_equal(fit, ofit) and np.array_equal(hold, ohold)


def test_strong_wolfe_search_on_a_quadratic():
    """f(t) = (t - 3)^2 along d = 1 from 0: the search ends at a point meeting both Wolfe conditions."""
    from dinov3_jax.eval.logreg import C1, C2, _strong_wolfe
    for t0 in (1e-3, 1.0, 50.0):
        f = lambda t: (t - 3.0) ** 2
        df = lambda t: 2.0 * (t - 3.0)
        gen = _strong_wolfe(f(0.0), df(0.0), t0)
        t = next(gen)
        try:
            while True:
                t = gen.send((f(t), df(t)))
        except StopIteration as e:
            ok, evals, exact = e.value
        assert ok and exact and evals <= 20, t0
        assert f(t) <= f(0.0) + C1 * t * df(0.0) and abs(df(t)) <= -C2 * df(0.0), (t0, t)


# ------------------------------------------------------------------------------------------------ config, flags
def test_defaults_carry_the_logreg_block():
    from dinov3_jax.configs import get_default_config
    assert get_default_config().evaluation.logreg == {
        "train_dataset_path": "", "val_dataset_path": "", "C_values": None, "holdout_fraction": 0.1,
        "max_iter": 1000, "tol": 1e-6, "history": 10, "avgpool": False, "batch_size": 256, "resize_size": 256,
        "crop_size": 224, "num_workers": 8, "seed": 0}


def test_do_logreg_eval_without_datasets_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_logreg_eval
    assert do_logreg_eval(get_default_config(), None, "training_9") == {}
    out = capsys.readouterr().out
    assert out.count("\n") == 1 and "nothing evaluated" in out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_names_logreg_after_the_linear_probe(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match=r"--eval linear\), logistic regression \(--eval logreg\), .*"
                                                  r"and instance retrieval \(--eval retrieval\)$"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_logreg_reaches_do_logreg_eval_and_nothing_else(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_logreg_eval", lambda config, model, header: calls.append((str(model), header))
                        or {"ok": 4})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval", "do_video_eval",
                 "do_correspondence_eval", "do_discovery_eval", "do_retrieval_eval", "do_train"):
        monkeypatch.setattr(train, name, lambda *a, _n=name, **k: pytest.fail(f"--eval-only --eval logreg ran {_n}"))
    ck = tmp_path / "ckpt" / "5"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 5, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "logreg", "--output-dir", str(tmp_path)]) == {"ok": 4}
    assert calls == [(str(ck), "manual_6")]


# ------------------------------------------------------------------------------------------------ host-side checks
def test_kernel_arguments_are_checked_on_the_host():
    from dinov3_jax import _native
    lib = _native.lib()
    fake = C.c_void_p(256)
    assert lib.d3_logreg_split_x(fake, 12, 4, 12, 64, fake, fake, None) == -1
    assert b"multiple of 8" in lib.d3_last_error()
    assert lib.d3_logreg_split_x(fake, 16, 4, 16, 100, fake, fake, None) == -1
    assert b"chunk" in lib.d3_last_error()
    assert lib.d3_logreg_weights(fake, 8 * 16 + 9, fake, 1, 8, 16, fake, fake, None) == -1
    assert b"P = Cp K + Cp" in lib.d3_last_error()
    assert lib.d3_logreg_xent(fake, 16, fake, fake, 3, 2, 2, 5, 8, 1.0, fake, fake, 16, None) == -1
    assert b"n <= rows" in lib.d3_last_error()
    assert lib.d3_logreg_xent(fake, 8, fake, fake, 2, 2, 2, 5, 8, 1.0, fake, fake, 16, None) == -1
    assert b"ld and ld_r" in lib.d3_last_error()
    for m in (0, 65):
        assert lib.d3_logreg_direction(*[fake] * 8, 1, 100, m, fake, fake, None) == -1
        assert b"1 <= m <= 64" in lib.d3_last_error()
        assert lib.d3_logreg_accept(*[fake] * 8, 1, 100, m, fake, None) == -1
        assert b"1 <= m <= 64" in lib.d3_last_error()


# ------------------------------------------------------------------------------------------------ ptxas
def test_logreg_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert "logreg.cu" in b.SOURCES
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", "logreg.cu"), "-o",
                                       str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    seen = set()
    for name, stack, st, ld in props:
        if "lr_" in name:
            seen.add(name)
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # split, weights, xent, rows sum, finish, combine, trial, dot, axpy, scale, accept
    assert len(seen) == 11, sorted(seen)
