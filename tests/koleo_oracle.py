"""Float64 statement of the distributed top-k KoLeo (dino.koleo_loss_distributed; parity unpinned, engine/koleo.py).

x [N, D] holds every rank's B rows in rank order.  Rank r's loss group is the R = G / B consecutive ranks that contain
it (G = None: all N rows).  For each of its rows i the neighbours are the k largest dots xn_i . xn_j over the group's
other rows, ties to the lower index, and L_r = -mean_{i, s} log(||xn_i - xn_nbr(i, s)|| + eps + eps).
"""
import numpy as np
import torch

EPS = 1e-8


def normalize(x, eps=EPS):
    return x / (x.norm(dim=-1, keepdim=True) + eps)


def group_of(rank, world, B, G):
    """(g0, gn): the row range of rank's loss group."""
    R = world if G is None else G // B
    assert (G is None or G % B == 0) and world % R == 0
    return (rank // R) * R * B, R * B


def neighbours(x, row0, B, g0, gn, k, eps=EPS):
    """[B, k] gathered indices: the k largest dots over rows [g0, g0 + gn) but the row itself, ties to the lower j."""
    xn = normalize(torch.as_tensor(x, dtype=torch.float64), eps).numpy()
    out = np.zeros((B, k), dtype=np.int64)
    cols = np.arange(g0, g0 + gn)
    for b in range(B):
        i = row0 + b
        keep = cols[cols != i]
        d = xn[keep] @ xn[i]
        order = np.lexsort((keep, -d))                  # dot descending, then index ascending
        out[b] = keep[order[:k]]
    return out


def margins(x, row0, B, g0, gn, k, eps=EPS):
    """[B]: the gap between the k-th and the (k+1)-th dot of each row (inf when there is no (k+1)-th)."""
    xn = normalize(torch.as_tensor(x, dtype=torch.float64), eps).numpy()
    cols = np.arange(g0, g0 + gn)
    out = np.full(B, np.inf)
    for b in range(B):
        i = row0 + b
        d = np.sort(xn[cols[cols != i]] @ xn[i])[::-1]
        if d.size > k:
            out[b] = d[k - 1] - d[k]
    return out


def rank_loss(x, row0, B, k, nbr, eps=EPS):
    """L_r (a float64 torch scalar, differentiable in x) for the given neighbour lists [B, k]."""
    xn = normalize(x, eps)
    xi = xn[row0:row0 + B].repeat_interleave(k, dim=0)
    xj = xn[torch.as_tensor(np.asarray(nbr).reshape(-1))]
    d = (xi - xj).norm(dim=-1) + eps
    return -torch.log(d + eps).mean()


def loss_and_grad(x, world, B, G, k, eps=EPS, nbrs=None):
    """[world] losses L_r, the gradient of sum_r L_r w.r.t. x (float64) and each rank's neighbour lists."""
    xd = torch.as_tensor(x, dtype=torch.float64).clone().requires_grad_(True)
    losses, lists = [], []
    for r in range(world):
        g0, gn = group_of(r, world, B, G)
        nbr = neighbours(xd.detach(), r * B, B, g0, gn, k, eps) if nbrs is None else nbrs[r]
        lists.append(nbr)
        losses.append(rank_loss(xd, r * B, B, k, nbr, eps))
    torch.stack(losses).sum().backward()
    return torch.stack(losses).detach(), xd.grad, lists
