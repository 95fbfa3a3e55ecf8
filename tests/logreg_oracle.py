"""Float64 statement of the logistic-regression evaluation (dinov3_jax/eval/logreg.py): the scaled objective
F_c = (1/N) sum_i CE(W x_i + b, y_i) + ||W||^2 / (2 c N) and its gradient, the default grid, the stratified split, and
scipy's L-BFGS-B for the optimum."""
import math

import numpy as np
import torch

f64 = torch.float64


def default_grid():
    return [float(v) for v in np.logspace(-6.0, 5.0, 45)]


def objective(W, b, X, y, c):
    """(F_c, dF/dW, dF/db) in float64; W [C, K], b [C], X [N, K], y [N] (any device)."""
    W, b, X = (torch.as_tensor(t).to(f64) for t in (W, b, X))
    y = torch.as_tensor(y).long().to(X.device)
    N = X.shape[0]
    z = X @ W.T + b
    lse = torch.logsumexp(z, 1)
    F = (lse - z.gather(1, y[:, None])[:, 0]).sum() / N + (W * W).sum() / (2.0 * c * N)
    R = torch.softmax(z, 1)
    R[torch.arange(N, device=X.device), y] -= 1.0
    R /= N
    return F.item(), R.T @ X + W / (c * N), R.sum(0)


def holdout(labels, fraction=0.1, seed=0):
    """(fit, held-out) sorted index arrays: per class floor(fraction n_c), at least 1 where n_c >= 2 and at most
    n_c - 1, from a seeded permutation of the class's indices, classes in increasing order."""
    y = np.asarray(labels).astype(np.int64)
    rng = np.random.default_rng(seed)
    hold = []
    for c in sorted(set(y.tolist())):
        idx = np.nonzero(y == c)[0]
        n = len(idx)
        k = 0 if n < 2 else min(n - 1, max(1, math.floor(fraction * n)))
        hold += rng.permutation(idx)[:k].tolist()
    hold = sorted(hold)
    return np.array(sorted(set(range(len(y))) - set(hold)), np.int64), np.array(hold, np.int64)


def newton_polish(W, b, X, y, c, steps=3):
    """Newton steps on F_c with the exact Hessian, plus the projector on 'every bias + t' (the bias is unpenalised, so
    the Hessian is singular along it, and the gradient has no component there).  An L-BFGS line search compares
    objective values and stalls where F changes by float64 rounding; Newton steps do not.  Runs on X's device."""
    X = torch.as_tensor(X).to(f64)
    dev = X.device
    W, b = W.to(dev).clone(), b.to(dev).clone()
    y = torch.as_tensor(y).long().to(dev)
    N, K = X.shape
    C = W.shape[0]
    Xa = torch.cat([X, torch.ones(N, 1, dtype=f64, device=dev)], 1)
    for _ in range(steps):
        _, gW, gb = objective(W, b, X, y, c)
        p = torch.softmax(X @ W.T + b, 1)
        H = torch.empty(C, K + 1, C, K + 1, dtype=f64, device=dev)
        for a in range(C):
            w = p[:, a:a + 1] * (torch.eye(C, dtype=f64, device=dev)[a] - p)          # [N, C]
            H[a] = (Xa.T @ (w[:, :, None] * Xa[:, None, :]).reshape(N, -1)).reshape(K + 1, C, K + 1) / N
        H = H.reshape(C * (K + 1), C * (K + 1))
        reg = torch.zeros(C, K + 1, dtype=f64, device=dev)
        reg[:, :K] = 1.0 / (c * N)
        H += torch.diag(reg.reshape(-1))
        g = torch.cat([gW, gb[:, None]], 1).reshape(-1)
        u = torch.zeros(C, K + 1, dtype=f64, device=dev)
        u[:, K] = 1.0 / math.sqrt(C)
        u = u.reshape(-1)
        step = torch.linalg.solve(H + torch.outer(u, u), -g).reshape(C, K + 1)
        W += step[:, :K]
        b += step[:, K]
    return W, b


def scipy_fit(X, y, num_classes, c, maxiter=20000, device="cpu"):
    """(W [C, K], b [C], F) at the optimum of F_c by scipy's L-BFGS-B from zero, then `newton_polish`; the float64
    objective runs on `device`."""
    from scipy.optimize import minimize
    X = torch.as_tensor(X).to(device=device, dtype=f64)
    y = torch.as_tensor(y).long().to(device)
    C, K = num_classes, X.shape[1]

    def fun(v):
        t = torch.from_numpy(v).to(device)
        F, gW, gb = objective(t[:C * K].view(C, K), t[C * K:], X, y, c)
        return F, torch.cat([gW.reshape(-1), gb]).cpu().numpy()

    r = minimize(fun, np.zeros(C * K + C), jac=True, method="L-BFGS-B", tol=1e-12,
                 options={"maxiter": maxiter, "maxfun": 2 * maxiter, "maxcor": 20, "gtol": 1e-12})
    v = torch.from_numpy(r.x).to(device)
    W, b = newton_polish(v[:C * K].view(C, K), v[C * K:], X, y, c)
    return W, b, objective(W, b, X, y, c)[0]


def clustered(n, dim, classes, seed, separation=1.5):
    """Seeded overlapping Gaussian clusters (unit noise per feature, centres about `separation` noise deviations
    apart): features float32 [n, dim], labels int64 [n], every class present."""
    g = torch.Generator().manual_seed(seed)
    centres = torch.randn(classes, dim, generator=g, dtype=f64) * (separation / math.sqrt(2.0 * dim))
    y = torch.arange(n) % classes
    y = y[torch.randperm(n, generator=g)]
    X = centres[y] + torch.randn(n, dim, generator=g, dtype=f64)
    return X.float(), y
