"""Logistic-regression evaluation of a frozen backbone: multinomial logistic regression on fixed features with a sweep
over the regularisation strength, this project's protocol modelled on DINOv2's `log_regression` evaluation.

Features are the teacher's last-block class token of the eval transform (the k-NN transform: Resize 256, CenterCrop
224), fp32 and not normalised; with `avgpool` the class token is followed by the last block's patch mean.  For each
strength c the objective is sklearn's multinomial `c * sum_i CE(W x_i + b, y_i) + ||W||^2 / 2` (bias unpenalised),
minimised in the scaled form F_c = (1/N) sum_i CE + ||W||^2 / (2 c N), which has the same minimiser.  A stratified,
seeded share of train is held out; every c is fitted on the rest, the c with the best held-out top-1 (ties to the
smaller c) is refitted from zero on the whole train set and scored on val (top-1, top-5, mean per-class accuracy).

The solver is L-BFGS (history 10, from W = 0, b = 0) with a strong-Wolfe line search, run for every c of the grid at
once: one evaluation of F and grad F for all problems still searching is one logits GEMM over the rows, one fused
cross-entropy kernel, one gradient GEMM and one regulariser kernel (csrc/logreg.cu), and a problem that has stopped
leaves the batch.  The GEMMs split the fp32 operands into bf16 hi + lo parts ([Xh | Xh | Xl] . [Wh | Wl | Wh]^T), which
keeps the objective and gradient at fp32 quality.  The line-search control runs on the host, on one G-sized vector
per evaluation; everything per element runs on the GPU.  Every reduction has a fixed order: two runs give the same
bits.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .. import ops
from .knn import RGB_MEAN, RGB_STD, _device, _pack

bf16, f32, i32 = torch.bfloat16, torch.float32, torch.int32
CHUNK_ROWS = 8192          # rows per logits / gradient GEMM: fixed by the configuration, so the sums' order is too
MAX_CHAIN_KBLOCKS = 64     # longest tensor-core accumulation chain (64-wide k-blocks) kept in one GEMM slice
C1, C2 = 1e-4, 0.9         # strong-Wolfe constants
MAX_LS_EVALS = 20
CURVATURE_EPS = 1e-10      # a pair with s.y <= eps ||s|| ||y|| is not stored
FTOL = 1e-12               # stop when F falls by less than FTOL |F| over an iteration
APPROX_EPS = 1e-6          # approximate Wolfe: F may exceed F(0) by APPROX_EPS |F(0)| (its float32 resolution)


def _splits(kdim: int) -> int:
    """GEMM slices for a contraction of kdim: no accumulation chain longer than MAX_CHAIN_KBLOCKS k-blocks (the tensor
    core's fp32 accumulation drifts over longer ones; the slices are added in fp32, in order)."""
    return -(-(-(-kdim // 64)) // MAX_CHAIN_KBLOCKS)


def default_C_values() -> list:
    """The default grid: 45 strengths 10^linspace(-6, 5, 45)."""
    return [float(v) for v in 10.0 ** np.linspace(-6.0, 5.0, 45)]


def stratified_holdout(labels, fraction: float = 0.1, seed: int = 0):
    """(fit indices, held-out indices), both sorted int64 numpy arrays.  Per class of n_c images, floor(fraction n_c)
    are held out, at least 1 where n_c >= 2 and at most n_c - 1, drawn by a seeded permutation of the class's indices
    (classes in increasing order from one numpy generator)."""
    y = np.asarray(labels).reshape(-1).astype(np.int64)
    rng = np.random.default_rng(int(seed))
    hold = []
    for c in np.unique(y):
        idx = np.flatnonzero(y == c)
        k = int(math.floor(float(fraction) * idx.size))
        if idx.size >= 2:
            k = min(max(k, 1), idx.size - 1)
        else:
            k = 0
        if k:
            hold.append(rng.permutation(idx)[:k])
    hold = np.sort(np.concatenate(hold)) if hold else np.zeros(0, np.int64)
    mask = np.ones(y.size, bool)
    mask[hold] = False
    return np.flatnonzero(mask).astype(np.int64), hold.astype(np.int64)


def _cubic_min(x1, f1, g1, x2, f2, g2, lo, hi):
    """Minimiser of the cubic through (x1, f1, f'(x1) = g1) and (x2, f2, g2), clipped to [lo, hi]; the midpoint when
    the cubic has none or an input is not finite."""
    vals = (x1, f1, g1, x2, f2, g2)
    if all(math.isfinite(v) for v in vals) and x1 != x2:
        d1 = g1 + g2 - 3.0 * (f1 - f2) / (x1 - x2)
        sq = d1 * d1 - g1 * g2
        if sq >= 0.0:
            d2 = math.copysign(math.sqrt(sq), x2 - x1)
            den = g2 - g1 + 2.0 * d2
            if den != 0.0:
                t = x2 - (x2 - x1) * (g2 + d2 - d1) / den
                if math.isfinite(t):
                    return min(max(t, lo), hi)
    return 0.5 * (lo + hi)


def _strong_wolfe(f0: float, g0: float, t: float):
    """Line search along a descent direction (g0 = grad . d < 0) as a generator: it yields a step, receives (F, grad .
    d) there, and returns (accepted, evaluations, exact).  Bracketing with cubic extrapolation, then zoom with
    safeguarded cubic interpolation (Nocedal & Wright, algorithms 3.5 and 3.6); at most MAX_LS_EVALS evaluations.

    A step is accepted when it meets the strong Wolfe conditions (exact = True) or, where the sufficient-decrease test
    fails, the approximate Wolfe conditions of Hager & Zhang (exact = False): C2 g0 <= g <= (2 C1 - 1) g0 and F <= F(0)
    + APPROX_EPS |F(0)|.  Near the optimum the change of F along a step falls below the resolution of a float32
    objective while the gradient still resolves it; along a convex line the gradient test implies the decrease.
    When it accepts, the last evaluated step is the accepted one."""
    evals = 0
    tp, fp, gp = 0.0, f0, g0

    def approx(f, g):
        return C2 * g0 <= g <= (2.0 * C1 - 1.0) * g0 and f <= f0 + APPROX_EPS * abs(f0)

    lo = hi = None
    while True:
        f, g = yield t
        evals += 1
        finite = math.isfinite(f) and math.isfinite(g)
        if finite and f > f0 + C1 * t * g0 and approx(f, g):
            return True, evals, False
        if not finite or f > f0 + C1 * t * g0 or (evals > 1 and f >= fp):
            lo, hi = (tp, fp, gp), (t, f, g)
            break
        if abs(g) <= -C2 * g0:
            return True, evals, True
        if g >= 0.0:
            lo, hi = (t, f, g), (tp, fp, gp)
            break
        if evals >= MAX_LS_EVALS:
            return False, evals, True
        tn = _cubic_min(tp, fp, gp, t, f, g, t + 0.01 * (t - tp), 10.0 * t)
        tp, fp, gp, t = t, f, g, tn
    while evals < MAX_LS_EVALS:
        a, b = min(lo[0], hi[0]), max(lo[0], hi[0])
        if not b > a:
            break
        t = _cubic_min(*lo, *hi, a, b)
        if min(t - a, b - t) < 0.1 * (b - a):
            t = 0.5 * (a + b)
        f, g = yield t
        evals += 1
        finite = math.isfinite(f) and math.isfinite(g)
        if not finite or f > f0 + C1 * t * g0 or f >= lo[1]:
            if finite and approx(f, g):
                return True, evals, False
            hi = (t, f, g)
        else:
            if abs(g) <= -C2 * g0:
                return True, evals, True
            if g * (hi[0] - lo[0]) >= 0.0:
                hi = lo
            lo = (t, f, g)
    return False, evals, True


class LogRegSweep:
    """Multinomial logistic regression for every strength of `C_values` at once, on device features.

    `fit(features, labels)` solves every problem (see the module docstring) and leaves W [G, num_classes, K], b [G,
    num_classes] and per-problem `info` ({"C", "iterations", "evaluations", "stop"}, stop one of "gtol", "ftol",
    "max_iter", "line_search").  `predict(features)` returns each problem's 5 best classes per row.  chunk_rows: rows
    per GEMM (a multiple of 64); it fixes the order of every sum, so results do not depend on free memory."""

    def __init__(self, num_classes: int, C_values=None, *, max_iter: int = 1000, tol: float = 1e-6, history: int = 10,
                 chunk_rows: int = CHUNK_ROWS, device=None):
        self.device = _device(device)
        self.num_classes = int(num_classes)
        if not 2 <= self.num_classes <= 32768:
            raise ValueError("num_classes must be in [2, 32768]")
        self.C_values = [float(c) for c in (default_C_values() if C_values is None else C_values)]
        if not self.C_values or min(self.C_values) <= 0.0:
            raise ValueError("C_values must be a non-empty list of positive strengths")
        self.max_iter, self.tol, self.history = int(max_iter), float(tol), int(history)
        if not 1 <= self.history <= 64:
            raise ValueError("history must be in [1, 64]")
        self.chunk = int(chunk_rows)
        if self.chunk < 64 or self.chunk % 64:
            raise ValueError("chunk_rows must be a positive multiple of 64")
        self.G, self.Cp = len(self.C_values), -(-self.num_classes // 8) * 8
        self.info, self.theta, self.K = None, None, None

    # ------------------------------------------------------------------------------------------------ evaluation
    def _evaluate(self, src, slots, d=None):
        """F, grad F of the problems in `slots` at src [G, P] into self.grad_out; returns float64 [Ga, 4] on the
        host: (F, grad . d, max |grad|, ||grad||^2)."""
        Ga, Cp, K, chunk = len(slots), self.Cp, self.K, self.chunk
        act = torch.tensor(slots, dtype=i32).to(self.device)
        GC = Ga * Cp
        wcat, bias = self.wcat[:GC], self.bias[:GC]
        ops.logreg_weights(src, act, Cp, K, wcat, bias)
        self.loss.zero_()
        gw = self.gw.view(-1)[:GC * K].view(GC, K)
        gw.zero_()
        self.gb.zero_()
        logits = self.logits.view(-1)[:chunk * GC].view(chunk, GC)
        r = self.r.view(-1)[:3 * chunk * GC].view(3 * chunk, GC)
        for c0 in range(0, self.rows, chunk):
            if self.sk_logits > 1:
                logits.zero_()
            ops.gemm(self.xa[c0:c0 + chunk], wcat, logits, accum=self.sk_logits > 1, split_k=self.sk_logits)
            ops.logreg_xent(logits, bias, self.labels[c0:], min(chunk, self.N - c0), Ga, self.num_classes, Cp,
                            1.0 / self.N, self.loss, r)
            ops.gemm(r, self.xg[3 * c0:3 * c0 + 3 * chunk], gw, a_mn=True, b_mn=True, accum=True,
                     split_k=self.sk_grad)
            ops.colsum_bf16(r[:chunk], self.gb[:GC])
            ops.colsum_bf16(r[2 * chunk:], self.gb[:GC])
        ops.logreg_finish(src, gw, self.gb, self.loss, self.icn, d, act, Cp, K, self.grad_out, self.out)
        return self.out[:Ga].cpu().numpy()

    def _prepare(self, features, labels):
        """The split operands, the labels and the evaluation buffers for features fp32 [N, K], labels [N]."""
        dev = self.device
        X = torch.as_tensor(features).to(device=dev, dtype=f32).contiguous()
        if X.dim() != 2 or X.shape[0] < 1 or X.shape[1] % 8:
            raise ValueError(f"features must be [N >= 1, K] with K a multiple of 8, got {tuple(X.shape)}")
        y = torch.as_tensor(labels).reshape(-1)
        if y.numel() != X.shape[0]:
            raise ValueError(f"{X.shape[0]} features but {y.numel()} labels")
        if int(y.min()) < 0 or int(y.max()) >= self.num_classes:
            raise ValueError(f"labels must lie in [0, {self.num_classes})")
        N, K = int(X.shape[0]), int(X.shape[1])
        G, Cp, chunk = self.G, self.Cp, self.chunk
        self.N, self.K, self.P = N, K, Cp * K + Cp
        self.rows = -(-N // chunk) * chunk
        self.sk_logits, self.sk_grad = _splits(3 * K), _splits(3 * chunk)
        self.xa = torch.empty(self.rows, 3 * K, dtype=bf16, device=dev)
        self.xg = torch.empty(3 * self.rows, K, dtype=bf16, device=dev)
        ops.logreg_split_x(X, chunk, self.xa, self.xg)
        self.labels = y.to(device=dev, dtype=i32).contiguous()
        self.wcat = torch.empty(G * Cp, 3 * K, dtype=bf16, device=dev)
        self.bias = torch.empty(G * Cp, dtype=f32, device=dev)
        self.logits = torch.empty(chunk, G * Cp, dtype=f32, device=dev)
        self.r = torch.empty(3 * chunk, G * Cp, dtype=bf16, device=dev)
        self.gw = torch.empty(G * Cp, K, dtype=f32, device=dev)
        self.gb = torch.empty(G * Cp, dtype=f32, device=dev)
        self.loss = torch.empty(G, dtype=torch.float64, device=dev)
        self.out = torch.empty(G, 4, dtype=torch.float64, device=dev)
        self.icn = torch.tensor([1.0 / (c * N) for c in self.C_values], dtype=f32).to(dev)
        self.grad_out = torch.zeros(G, self.P, dtype=f32, device=dev)

    def fit(self, features, labels):
        """Solve every problem on features fp32 [N, K] (K % 8 == 0) and labels [N] in [0, num_classes)."""
        self._prepare(features, labels)
        dev, G, m, P = self.device, self.G, self.history, self.P
        acc = torch.empty(G, 3, dtype=torch.float64, device=dev)
        theta, d, theta_t, grad_t = (torch.zeros(G, P, dtype=f32, device=dev) for _ in range(4))
        grad = self.grad_out
        S, Y = (torch.zeros(G, m, P, dtype=f32, device=dev) for _ in range(2))
        rho_h, gamma_h = np.zeros((G, m), np.float32), np.ones(G, np.float32)
        count_h, newest_h = np.zeros(G, np.int32), np.full(G, m - 1, np.int32)
        rho, gamma = torch.zeros(G, m, dtype=f32, device=dev), torch.ones(G, dtype=f32, device=dev)
        count, newest = torch.zeros(G, dtype=i32, device=dev), torch.zeros(G, dtype=i32, device=dev)
        alpha, slot = torch.zeros(G, dtype=f32, device=dev), torch.zeros(G, dtype=i32, device=dev)
        gd = torch.empty(G, dtype=torch.float64, device=dev)

        def upload():
            rho.copy_(torch.from_numpy(rho_h)); gamma.copy_(torch.from_numpy(gamma_h))
            count.copy_(torch.from_numpy(count_h)); newest.copy_(torch.from_numpy(newest_h))

        res = self._evaluate(theta, list(range(G)))
        f = res[:, 0].copy()
        gmax, gn2 = res[:, 2].copy(), res[:, 3].copy()
        gtol = self.tol * np.maximum(1.0, gmax)
        iters, evals = np.zeros(G, np.int64), np.ones(G, np.int64)
        stop = [None] * G
        for g in range(G):
            if not math.isfinite(f[g]):
                stop[g] = "line_search"
            elif gmax[g] <= gtol[g]:
                stop[g] = "gtol"
            elif self.max_iter <= 0:
                stop[g] = "max_iter"
        self.grad_out = grad_t
        while True:
            run = [g for g in range(G) if stop[g] is None]
            if not run:
                break
            upload()
            act = torch.tensor(run, dtype=i32).to(dev)
            ops.logreg_direction(grad, S, Y, rho, gamma, count, newest, act, d, gd)
            gdh = gd[:len(run)].cpu().numpy()
            reset = [g for g, v in zip(run, gdh) if not v < 0.0 and count_h[g] > 0]
            if reset:                                   # not a descent direction: drop the history, go downhill
                count_h[reset] = 0
                upload()
                ops.logreg_direction(grad, S, Y, rho, gamma, count, newest, act, d, gd)
                gdh = gd[:len(run)].cpu().numpy()
            searches, pending = {}, []
            for g, g0 in zip(run, gdh):
                if not g0 < 0.0:
                    stop[g] = "gtol"
                    continue
                t0 = 1.0 if count_h[g] > 0 else min(1.0, 1.0 / math.sqrt(gn2[g]))
                gen = _strong_wolfe(float(f[g]), float(g0), t0)
                searches[g] = (gen, next(gen))
                pending.append(g)
            last, exact = {}, {}
            ok = []
            while pending:
                al = np.zeros(G, np.float32)
                for g in pending:
                    al[g] = searches[g][1]
                alpha.copy_(torch.from_numpy(al))
                pact = torch.tensor(pending, dtype=i32).to(dev)
                ops.logreg_trial(theta, d, alpha, pact, theta_t)
                res = self._evaluate(theta_t, pending, d)
                nxt = []
                for g, row in zip(pending, res):
                    evals[g] += 1
                    last[g] = row
                    gen = searches[g][0]
                    try:
                        searches[g] = (gen, gen.send((float(row[0]), float(row[1]))))
                        nxt.append(g)
                    except StopIteration as e:
                        if e.value[0]:
                            ok.append(g)
                            exact[g] = e.value[2]
                        else:
                            stop[g] = "line_search"
                pending = nxt
            if not ok:
                continue
            ok.sort()
            slot.copy_(torch.from_numpy(((newest_h + 1) % m).astype(np.int32)))
            ops.logreg_accept(theta, grad, theta_t, grad_t, S, Y, slot, torch.tensor(ok, dtype=i32).to(dev), acc)
            acch = acc[:len(ok)].cpu().numpy()
            for g, (sy, yy, ss) in zip(ok, acch):
                f_old = f[g]
                f[g], gmax[g], gn2[g] = last[g][0], last[g][2], last[g][3]
                iters[g] += 1
                if sy > CURVATURE_EPS * math.sqrt(ss * yy):
                    newest_h[g] = (newest_h[g] + 1) % m
                    count_h[g] = min(count_h[g] + 1, m)
                    rho_h[g, newest_h[g]] = 1.0 / sy
                    gamma_h[g] = sy / yy
                elif count_h[g] == m:                   # the skipped pair overwrote the oldest one
                    count_h[g] = m - 1
                if gmax[g] <= gtol[g]:
                    stop[g] = "gtol"
                elif exact[g] and f_old - f[g] < FTOL * abs(f[g]):
                    stop[g] = "ftol"            # (after an approximate-Wolfe step the change of F is below resolution)
                elif iters[g] >= self.max_iter:
                    stop[g] = "max_iter"
        self.theta = theta
        self.objective = [float(v) for v in f]
        self.info = [{"C": c, "iterations": int(iters[g]), "evaluations": int(evals[g]), "stop": stop[g],
                      "objective": float(f[g])} for g, c in enumerate(self.C_values)]
        for name in ("xa", "xg", "logits", "r", "gw", "wcat", "grad_out"):
            setattr(self, name, None)
        return self

    @property
    def W(self) -> torch.Tensor:
        """fp32 [G, num_classes, K] on the device."""
        return self.theta[:, :self.Cp * self.K].view(self.G, self.Cp, self.K)[:, :self.num_classes]

    @property
    def b(self) -> torch.Tensor:
        """fp32 [G, num_classes] on the device."""
        return self.theta[:, self.Cp * self.K:][:, :self.num_classes]

    # ------------------------------------------------------------------------------------------------ prediction
    def predict(self, features, k: int = 5) -> torch.Tensor:
        """int32 [Nq, G, k]: each problem's k best classes per row (logit desc, ties to the lower class), the logits
        from the same split GEMM as the fit."""
        if self.theta is None:
            raise RuntimeError("predict before fit")
        dev, G, Cp, K, chunk = self.device, self.G, self.Cp, self.K, self.chunk
        X = torch.as_tensor(features).to(device=dev, dtype=f32).contiguous()
        if X.dim() != 2 or X.shape[1] != K:
            raise ValueError(f"features must be [Nq, {K}], got {tuple(X.shape)}")
        Nq = int(X.shape[0])
        k = int(k)
        preds = torch.empty(Nq, G * k, dtype=i32, device=dev)
        if Nq == 0:
            return preds.view(0, G, k)
        rows = -(-Nq // chunk) * chunk
        xa = torch.empty(rows, 3 * K, dtype=bf16, device=dev)
        ops.logreg_split_x(X, chunk, xa)
        act = torch.arange(G, dtype=i32).to(dev)
        wcat = torch.empty(G * Cp, 3 * K, dtype=bf16, device=dev)
        bias = torch.empty(G * Cp, dtype=f32, device=dev)
        ops.logreg_weights(self.theta, act, Cp, K, wcat, bias)
        sk = _splits(3 * K)
        logits = torch.empty(chunk, G * Cp, dtype=f32, device=dev)
        top_s = torch.empty(chunk, G * k, dtype=f32, device=dev)
        for r0 in range(0, Nq, chunk):
            n = min(chunk, Nq - r0)
            logits.copy_(bias.view(1, -1).expand(chunk, -1))
            ops.gemm(xa[r0:r0 + chunk], wcat, logits, accum=True, split_k=sk)
            for g in range(G):
                ops.topk_merge(logits[:n, g * Cp:(g + 1) * Cp], top_s[:n, k * g:k * g + k],
                               preds[r0:r0 + n, k * g:k * g + k], offset=0, valid=self.num_classes, fresh=True)
        return preds.view(Nq, G, k)


def accuracies(preds: torch.Tensor, labels, num_classes: int) -> dict:
    """{"top1", "top5", "mean_per_class"} in percent from int32 [N, 5] predictions; the per-class mean is over the
    classes present in `labels`."""
    y = torch.as_tensor(labels).reshape(-1).to(device=preds.device, dtype=torch.int64)
    hit1 = (preds[:, 0].long() == y)
    hit5 = (preds.long() == y[:, None]).any(1)
    per_n = torch.bincount(y, minlength=num_classes).cpu().numpy()
    per_hit = torch.bincount(y[hit1], minlength=num_classes).cpu().numpy()
    present = per_n > 0
    n = max(int(y.numel()), 1)
    return {"top1": 100.0 * int(hit1.sum()) / n, "top5": 100.0 * int(hit5.sum()) / n,
            "mean_per_class": float(100.0 * np.mean(per_hit[present] / per_n[present])) if present.any() else 0.0}


def extract_logreg_features(model, dataset, *, avgpool: bool = False, batch_size: int = 256, num_workers: int = 8,
                            resize_size: int = 256, crop_size: int = 224, rgb_mean=RGB_MEAN, rgb_std=RGB_STD,
                            device=None):
    """(fp32 features [N, D or 2 D], labels int64 [N]) on the GPU, not normalised: the last block's class token of
    the eval transform, followed with `avgpool` by the last block's patch mean."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    loader = torch.utils.data.DataLoader(dataset, batch_size=int(batch_size), shuffle=False, drop_last=False,
                                         num_workers=int(num_workers), collate_fn=_pack,
                                         pin_memory=dev.type == "cuda", persistent_workers=False)
    feats, labels, n0 = None, torch.empty(len(dataset), dtype=torch.int64, device=dev), 0
    for flat, desc, y in loader:
        n = desc.shape[0]
        sizes = [(int(h), int(w)) for h, w in desc[:, 1:].tolist()]
        x = torch.empty(n, crop_size, crop_size, 3, dtype=bf16, device=dev)
        ops.eval_resize_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True), x, resize=resize_size,
                             max_taps=ops.eval_max_taps(sizes, resize_size), mean=rgb_mean, std=rgb_std)
        patches, cls = model.get_intermediate_layers(x, n=1, return_class_token=True)[-1]
        D = cls.shape[1]
        if feats is None:
            feats = torch.empty(len(dataset), 2 * D if avgpool else D, dtype=f32, device=dev)
        feats[n0:n0 + n, :D].copy_(cls)
        if avgpool:
            mean = ops.pool_tokens(patches.contiguous(), torch.empty(n, 1, D, dtype=f32, device=dev),
                                   copy_tokens=False)
            feats[n0:n0 + n, D:].copy_(mean.view(n, D))
        labels[n0:n0 + n] = y.to(dev)
        n0 += n
    if feats is None:
        raise ValueError("empty dataset")
    return feats, labels


def eval_log_regression(model, train_dataset, val_dataset, *, C_values=None, holdout_fraction: float = 0.1,
                        max_iter: int = 1000, tol: float = 1e-6, history: int = 10, avgpool: bool = False,
                        batch_size: int = 256, resize_size: int = 256, crop_size: int = 224, num_workers: int = 8,
                        seed: int = 0, rgb_mean=RGB_MEAN, rgb_std=RGB_STD, num_classes: int | None = None,
                        chunk_rows: int = CHUNK_ROWS, **_ignored) -> dict:
    """The logistic-regression evaluation of `model` (a DinoVisionTransformer): {"sweep": [{"C", "holdout_top1",
    "iterations", "evaluations", "stop"}, ...], "best_C", "refit": {"iterations", "evaluations", "stop"}, "top1",
    "top5", "mean_per_class" (val, percent), "n_fit", "n_holdout", "n_val", "num_classes", "feature_dim"}.  The extra
    keys of an `evaluation.logreg` config block (dataset paths) are accepted and ignored."""
    kw = dict(avgpool=bool(avgpool), batch_size=batch_size, num_workers=num_workers, resize_size=int(resize_size),
              crop_size=int(crop_size), rgb_mean=rgb_mean, rgb_std=rgb_std)
    train_f, train_y = extract_logreg_features(model, train_dataset, **kw)
    val_f, val_y = extract_logreg_features(model, val_dataset, **kw)
    if num_classes is None:
        num_classes = int(max(int(train_y.max()), int(val_y.max()))) + 1
    grid = default_C_values() if C_values is None else [float(c) for c in C_values]
    solver = dict(max_iter=max_iter, tol=tol, history=history, chunk_rows=chunk_rows, device=train_f.device)
    fit_i, hold_i = stratified_holdout(train_y.cpu().numpy(), holdout_fraction, seed)
    if hold_i.size == 0:
        raise ValueError("the held-out split is empty: the train set needs a class with at least 2 images")
    fit_t, hold_t = (torch.from_numpy(v).to(train_f.device) for v in (fit_i, hold_i))
    sweep = LogRegSweep(num_classes, grid, **solver).fit(train_f[fit_t], train_y[fit_t])
    hold_pred = sweep.predict(train_f[hold_t], k=1)
    hold_hits = (hold_pred[:, :, 0].long() == train_y[hold_t][:, None]).sum(0).cpu().numpy()
    hold_top1 = [100.0 * int(h) / hold_i.size for h in hold_hits]
    best = min(range(len(grid)), key=lambda g: (-int(hold_hits[g]), grid[g]))
    keys = ("iterations", "evaluations", "stop")
    rows = [{"C": grid[g], "holdout_top1": hold_top1[g], **{k: info[k] for k in keys}}
            for g, info in enumerate(sweep.info)]
    del sweep
    refit = LogRegSweep(num_classes, [grid[best]], **solver).fit(train_f, train_y)
    metrics = accuracies(refit.predict(val_f, k=5)[:, 0], val_y, num_classes)
    return {"sweep": rows, "best_C": grid[best], "refit": {k: refit.info[0][k] for k in keys}, **metrics,
            "n_fit": int(fit_i.size), "n_holdout": int(hold_i.size), "n_val": int(val_y.numel()),
            "num_classes": int(num_classes), "feature_dim": int(train_f.shape[1])}
