"""GPU: the logistic-regression evaluation (eval/logreg.py) at a Food-101 shape: N = 75 750 train rows, 101 classes,
D = 1024 (the class token) or 2048 (with avgpool), the default 45-strength grid, on seeded synthetic clustered
features (the cost depends on the shapes and on how many iterations each strength takes, not on images).

Reports, per D:
- one batched evaluation of F and grad F for all 45 problems: its time, the part spent in the GEMMs (CUDA events
  around each d3_gemm_bf16 call) and the rest, and the GEMMs' TFLOP/s over their own time;
- the whole sweep (45 strengths at once, on 90 % of the rows) and the refit at one strength on all rows, wall clock
  ending in a device synchronise, with each strength's iterations;
- a torch float32 baseline: torch.optim.LBFGS(history 10, line_search_fn="strong_wolfe") on the same objective, one
  strength at a time, for the strengths given by --baseline-c (the full grid one at a time takes too long to run here).
The card, its power limit and maximum SM clock are printed with the numbers.

python tools/bench_logreg.py [--dims 1024 2048] [--baseline-c 1e-4 1 1e4]
"""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import torch

from dinov3_jax import _native, ops
from dinov3_jax.eval.logreg import LogRegSweep, default_C_values, stratified_holdout
from gpu_timing import card, cuda_ms

N, CLASSES = 75750, 101


def features(D, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn(CLASSES, D, generator=g, device="cuda") * (1.5 / math.sqrt(2.0 * D))
    y = torch.arange(N, device="cuda") % CLASSES
    return centres[y] + torch.randn(N, D, generator=g, device="cuda"), y


def torch_lbfgs(X, y, c, max_iter=1000, tol=1e-6):
    """Seconds and iterations of torch's float32 L-BFGS on F_c = mean CE + ||W||^2 / (2 c N) from zero."""
    W = torch.zeros(CLASSES, X.shape[1], device="cuda", requires_grad=True)
    b = torch.zeros(CLASSES, device="cuda", requires_grad=True)
    opt = torch.optim.LBFGS([W, b], lr=1, max_iter=max_iter, history_size=10, tolerance_grad=tol,
                            tolerance_change=1e-12, line_search_fn="strong_wolfe")
    n = X.shape[0]

    def closure():
        opt.zero_grad()
        loss = torch.nn.functional.cross_entropy(X @ W.T + b, y) + (W * W).sum() / (2.0 * c * n)
        loss.backward()
        return loss

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    opt.step(closure)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, opt.state[opt._params[0]]["n_iter"]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--dims", type=int, nargs="+", default=[1024, 2048])
    p.add_argument("--baseline-c", type=float, nargs="*", default=[1e-4, 1.0, 1e4])
    p.add_argument("--iters", type=int, default=10)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_logreg needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    _native.init(0)
    out = {"card": card(), "N": N, "classes": CLASSES, "grid": len(default_C_values())}
    for D in a.dims:
        X, y = features(D)
        grid = default_C_values()
        sw = LogRegSweep(CLASSES, grid, device="cuda")
        sw._prepare(X, y)
        theta = torch.zeros(sw.G, sw.P, device="cuda")
        slots = list(range(sw.G))
        ms = cuda_ms(lambda: sw._evaluate(theta, slots), a.iters, 2)
        ops.PROFILE = []
        sw._evaluate(theta, slots)
        torch.cuda.synchronize()
        gemm_ms = sum(e0.elapsed_time(e1) for _, _, e0, e1, _ in ops.PROFILE)
        gemm_flop = sum(f for _, f, _, _, _ in ops.PROFILE)
        ops.PROFILE = None
        del sw, theta
        torch.cuda.empty_cache()
        fit_i, _ = stratified_holdout(y.cpu().numpy(), 0.1, 0)
        fit_t = torch.from_numpy(fit_i).cuda()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sweep = LogRegSweep(CLASSES, grid, device="cuda").fit(X[fit_t], y[fit_t])
        torch.cuda.synchronize()
        t_sweep = time.perf_counter() - t0
        info = sweep.info
        del sweep
        t0 = time.perf_counter()
        refit = LogRegSweep(CLASSES, [1.0], device="cuda").fit(X, y)
        torch.cuda.synchronize()
        t_refit = time.perf_counter() - t0
        base = {}
        for c in a.baseline_c:
            sec, it = torch_lbfgs(X, y, c)
            base[f"{c:g}"] = {"seconds": round(sec, 3), "iterations": int(it)}
        out[f"D={D}"] = {
            "evaluation_ms": round(ms, 3), "evaluation_gemm_ms": round(gemm_ms, 3),
            "evaluation_other_ms": round(ms - gemm_ms, 3), "gemm_tflops": round(gemm_flop / gemm_ms / 1e9, 1),
            "sweep_seconds": round(t_sweep, 2), "refit_seconds_at_c=1": round(t_refit, 2),
            "refit_iterations": refit.info[0]["iterations"],
            "sweep_iterations": [i["iterations"] for i in info], "sweep_stops": [i["stop"] for i in info],
            "torch_lbfgs_fp32_one_c": base}
        del X, y, refit
        torch.cuda.empty_cache()
        print(json.dumps({k: out[k] for k in ("card", f"D={D}")}), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
