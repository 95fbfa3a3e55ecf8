"""Float64 statement of the linear depth probe's arithmetic (dinov3_jax/eval/depth.py) in torch, on any device: the
"linear" bin head's cell depth, bilinear upsampling with align_corners=False as explicit interpolation matrices, the
scale-invariant log loss with its gradient to the bin logits written out by hand (not by autograd), and the per-image
metrics of the clamped prediction."""
import torch

EPS, LAMBDA, FLOOR = 1e-3, 0.15, 0.1
f64 = torch.float64


def interp_matrix(n_out: int, n_in: int, device=None) -> torch.Tensor:
    """A [n_out, n_in] with upsampled = A @ x along one axis: torch's source index s = max((o + 0.5) * n_in / n_out
    - 0.5, 0), cells i0 = floor(s), i1 = min(i0 + 1, n_in - 1), weights (1 - (s - i0), s - i0)."""
    A = torch.zeros(n_out, n_in, dtype=f64)
    for o in range(n_out):
        s = max((o + 0.5) * n_in / n_out - 0.5, 0.0)
        i0 = int(s)
        i1 = min(i0 + 1, n_in - 1)
        A[o, i0] += 1.0 - (s - i0)
        A[o, i1] += s - i0
    return A.to(device)


def centres(n_bins: int, lo: float, hi: float, device=None) -> torch.Tensor:
    return torch.linspace(lo, hi, n_bins, dtype=f64, device=device)


def cell_depth(z: torch.Tensor, lo: float, hi: float):
    """(d, S) per cell of bin logits z [..., n_bins]: q = relu(z) + 0.1, S = sum q, d = sum q c / S."""
    z = z.to(f64)
    q = torch.relu(z) + FLOOR
    S = q.sum(-1)
    return (q * centres(z.shape[-1], lo, hi, z.device)).sum(-1) / S, S


def upsample(d: torch.Tensor, Hl: int, Wl: int) -> torch.Tensor:
    """[B, h, w] -> [B, Hl, Wl]"""
    _, h, w = d.shape
    return torch.einsum("yi,bij,xj->byx", interp_matrix(Hl, h, d.device), d, interp_matrix(Wl, w, d.device))


def valid_mask(gt: torch.Tensor, lo: float, hi: float) -> torch.Tensor:
    return (gt > lo) & (gt <= hi)


def si_loss(z: torch.Tensor, gt: torch.Tensor, lo: float, hi: float):
    """(L, dL/dz [B, h, w, n_bins], valid count, envelope [B, h, w]) for bin logits z [B, h, w, n_bins] and ground
    truth gt [B, Hl, Wl].  The envelope is the adjoint of sum over pixels of ((|g - mean| + 1e-5) / (N - 1)
    + 0.15 |mean| / N) / L / (d_hat + 1e-3): the magnitudes each cell's dL/dd adds up, plus a 1e-5 slack on g for the
    fp32 rounding of the logs and of d."""
    B, h, w, nb = z.shape
    _, Hl, Wl = gt.shape
    z, gt = z.to(f64), gt.to(f64)
    d, S = cell_depth(z, lo, hi)
    Ay, Ax = interp_matrix(Hl, h, z.device), interp_matrix(Wl, w, z.device)
    dh = torch.einsum("yi,bij,xj->byx", Ay, d, Ax)
    valid = valid_mask(gt, lo, hi)
    n = int(valid.sum())
    if n < 2:
        return 0.0, torch.zeros_like(z), n, torch.zeros_like(d)
    g = torch.where(valid, torch.log(dh + EPS) - torch.log(torch.where(valid, gt, 1.0) + EPS), 0.0)
    mu = g.sum() / n
    var = (torch.where(valid, g - mu, 0.0) ** 2).sum() / (n - 1)
    L = torch.sqrt(var + LAMBDA * mu * mu)
    dg = torch.where(valid, ((g - mu) / (n - 1) + LAMBDA * mu / n) / L, 0.0)
    dd = torch.einsum("yi,byx,xj->bij", Ay, dg / (dh + EPS), Ax)
    mag = torch.where(valid, (((g - mu).abs() + 1e-5) / (n - 1) + LAMBDA * mu.abs() / n) / L, 0.0)
    env = torch.einsum("yi,byx,xj->bij", Ay, mag / (dh + EPS), Ax)
    c = centres(nb, lo, hi, z.device)
    dz = (z > 0).to(f64) * (c - d[..., None]) / S[..., None] * dd[..., None]
    return float(L), dz, n, env


METRIC_NAMES = ("abs_rel", "sq_rel", "rmse", "rmse_log", "log10", "a1", "a2", "a3")


def metric_sums(z: torch.Tensor, gt: torch.Tensor, lo: float, hi: float, crop=None):
    """(float64 [B, 9] per-image sums (count, |e| / t, e^2 / t, e^2, (ln p - ln t)^2, |log10 p - log10 t|, a1..a3
    hits), int [B, 3] per-image pixels whose max(p / t, t / p) lies within 1e-5 relative of 1.25^k) for the prediction
    p = upsampled cell depth clamped to [lo, hi], over the valid pixels inside crop = (top, bottom, left, right)."""
    B, h, w, _ = z.shape
    _, Hl, Wl = gt.shape
    d, _ = cell_depth(z, lo, hi)
    p = upsample(d, Hl, Wl).clamp(lo, hi)
    t = gt.to(f64)
    m = valid_mask(t, lo, hi)
    if crop is not None:
        keep = torch.zeros_like(m)
        keep[:, crop[0]:crop[1], crop[2]:crop[3]] = True
        m &= keep
    t = torch.where(m, t, 1.0)
    e = p - t
    r = torch.maximum(p / t, t / p)
    cols = [torch.ones_like(p), e.abs() / t, e * e / t, e * e, (torch.log(p) - torch.log(t)) ** 2,
            (torch.log10(p) - torch.log10(t)).abs()] + [(r < 1.25 ** k).to(f64) for k in (1, 2, 3)]
    sums = torch.stack([(c * m).sum((1, 2)) for c in cols], 1)
    near = torch.stack([(((r / 1.25 ** k) - 1).abs() < 1e-5) & m for k in (1, 2, 3)], 1).sum((2, 3))
    return sums, near


def metrics(sums) -> dict:
    """Each metric averaged over the images with a valid pixel, from metric_sums' per-image sums."""
    s = torch.as_tensor(sums, dtype=f64)
    s = s[s[:, 0] > 0]
    n = s[:, 0]
    per = [s[:, 1] / n, s[:, 2] / n, (s[:, 3] / n).sqrt(), (s[:, 4] / n).sqrt(), s[:, 5] / n, s[:, 6] / n,
           s[:, 7] / n, s[:, 8] / n]
    return {k: float(v.mean()) for k, v in zip(METRIC_NAMES, per)}
