"""The object discovery protocol (dinov3_jax/eval/discovery.py) stated in float64 on the CPU: the dense graph, the
generalized eigenproblem solved by scipy.linalg.eigh, the bipartition with TokenCut's sign flip, scipy.ndimage.label's
4-connected components, and the IoU / CorLoc score."""
import numpy as np
import scipy.linalg
import scipy.ndimage


def graph(feats, tau=0.2, eps=1e-5):
    """(A [N, N], d [N]) of the patch features feats [N, D]: A_ij = 1 if <f_i, f_j> > tau else eps, d = A 1."""
    f = np.asarray(feats, np.float64)
    A = np.where(f @ f.T > tau, 1.0, eps)
    return A, A.sum(1)


def fiedler(A, d):
    """(x [N], lambda_2, lambda_3): the generalized eigenvector of (D - A) x = lambda D x at the second-smallest
    eigenvalue (scipy normalises x^T D x = 1), and the next eigenvalue for the gap."""
    vals, vecs = scipy.linalg.eigh(np.diag(d) - A, np.diag(d), subset_by_index=[1, min(2, len(d) - 1)])
    return vecs[:, 0], float(vals[0]), float(vals[-1]) if len(vals) > 1 else float("inf")


def bipartition(x):
    """(fg bool [N], seed): x_i > mean(x), complemented when the seed argmax |x_i| (lowest index on ties) is not in it."""
    x = np.asarray(x, np.float64)
    fg = x > x.mean()
    seed = int(np.argmax(np.abs(x)))
    return (fg if fg[seed] else ~fg), seed


def component_box(fg, seed, grid, patch, size):
    """The pixel box [x0 p, y0 p, (x1 + 1) p, (y1 + 1) p], clipped to size (H, W), of the 4-connected component of the
    h x w mask fg that holds the seed."""
    h, w = grid
    labels, _ = scipy.ndimage.label(np.asarray(fg).reshape(h, w))
    ys, xs = np.nonzero(labels == labels.reshape(-1)[seed])
    H, W = size
    return [min(xs.min() * patch, W), min(ys.min() * patch, H), min((xs.max() + 1) * patch, W),
            min((ys.max() + 1) * patch, H)]


def iou(box, gts):
    """float64 [B]: IoU of box with each ground-truth row [B, 4] on continuous areas, no + 1."""
    b = np.asarray(box, np.float64)
    out = []
    for g in np.asarray(gts, np.float64).reshape(-1, 4):
        iw = max(0.0, min(b[2], g[2]) - max(b[0], g[0]))
        ih = max(0.0, min(b[3], g[3]) - max(b[1], g[1]))
        inter = iw * ih
        union = (b[2] - b[0]) * (b[3] - b[1]) + (g[2] - g[0]) * (g[3] - g[1]) - inter
        out.append(inter / union if union > 0 else 0.0)
    return np.array(out)


def discover(feats, grid, patch, size, tau=0.2, eps=1e-5):
    """The whole per-image protocol: {"x", "lambda2", "gap", "fg", "seed", "box"} from the features [h w, D]."""
    A, d = graph(feats, tau, eps)
    x, lam2, lam3 = fiedler(A, d)
    fg, seed = bipartition(x)
    return {"x": x, "lambda2": lam2, "gap": lam3 - lam2, "fg": fg, "seed": seed,
            "box": component_box(fg, seed, grid, patch, size)}
