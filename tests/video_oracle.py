"""The video object segmentation protocol of dinov3_jax/eval/video.py in float64 numpy: label propagation through the
windowed top-k affinities, the upsampled, normalised argmax label map, and the DAVIS 2017 J and F counts.  The GPU
kernels (csrc/video.cu) are checked against it; it is itself pinned to a torch restatement of DINO's
label_propagation and to hand-computed J / F cases (tests/test_video_cpu.py)."""
import math

import numpy as np
from scipy import ndimage


def window_candidates(q, h, w, radius, n_ctx):
    """(context frame, source row) of every candidate of target patch q, in candidate order: frame, row, column."""
    qy, qx = divmod(q, w)
    ys = range(max(qy - radius, 0), min(qy + radius, h - 1) + 1)
    xs = range(max(qx - radius, 0), min(qx + radius, w - 1) + 1)
    return [(c, y * w + x) for c in range(n_ctx) for y in ys for x in xs]


def propagate(target, ctx_feats, ctx_labels, h, w, radius, topk, temperature):
    """(soft labels float64 [P, C], kth [P], next [P]) of one target frame: target [P, D] and each context frame's
    features [P, D] as float64, labels [P, C].  kth / next are each row's k-th and (k+1)-th largest similarity
    (-inf where there is none), for telling a near tie at the threshold."""
    target = np.asarray(target, dtype=np.float64)
    sims = [target @ np.asarray(f, dtype=np.float64).T for f in ctx_feats]
    return propagate_sims(sims, ctx_labels, h, w, radius, topk, temperature)


def propagate_sims(sims, ctx_labels, h, w, radius, topk, temperature):
    """`propagate` from the similarities [P, P] of the target rows to each context frame's rows."""
    sims = [np.asarray(x, dtype=np.float64) for x in sims]
    labs = [np.asarray(l, dtype=np.float64) for l in ctx_labels]
    P, C = sims[0].shape[0], labs[0].shape[1]
    out = np.zeros((P, C))
    kth, nxt = np.full(P, -np.inf), np.full(P, -np.inf)
    for q in range(P):
        cand = window_candidates(q, h, w, radius, len(sims))
        x = np.array([sims[c][q, s] for c, s in cand])
        a = np.exp(x / temperature)
        order = np.sort(x)[::-1]
        thr = np.sort(a)[::-1][topk - 1] if len(a) >= topk else 0.0
        if len(order) >= topk:
            kth[q] = order[topk - 1]
        if len(order) > topk:
            nxt[q] = order[topk]
        keep = a >= thr
        wgt = a[keep] / a[keep].sum()
        rows = np.stack([labs[c][s] for (c, s), k in zip(cand, keep) if k])
        out[q] = wgt @ rows
    return out, kth, nxt


def nearest_exact_index(out_size, in_size):
    """torch's nearest-exact source index, in fp32 as torch computes it."""
    scale = np.float32(in_size) / np.float32(out_size)
    d = np.arange(out_size, dtype=np.float32)
    return np.minimum(np.floor((d + np.float32(0.5)) * scale).astype(np.int64), in_size - 1)


def upsample(soft, patch):
    """float64 [C, h p, w p]: torch bilinear (align_corners=False) of soft [h, w, C] by the factor `patch`."""
    soft = np.asarray(soft, dtype=np.float64)
    h, w, C = soft.shape

    def axis(n):
        s = np.maximum((np.arange(n * patch) + 0.5) / patch - 0.5, 0.0)
        i0 = np.floor(s).astype(np.int64)
        return i0, np.minimum(i0 + 1, n - 1), s - i0

    y0, y1, ly = axis(h)
    x0, x1, lx = axis(w)
    t = soft.transpose(2, 0, 1)
    top = t[:, y0][:, :, x0] * (1 - lx) + t[:, y0][:, :, x1] * lx
    bot = t[:, y1][:, :, x0] * (1 - lx) + t[:, y1][:, :, x1] * lx
    return top * (1 - ly)[:, None] + bot * ly[:, None]


def label_map(soft, patch, out_h, out_w):
    """(labels uint8 [out_h, out_w], margin float64 [out_h, out_w]): the argmax of the upsampled soft map with each
    channel of maximum > 0 min-max normalised over the frame, taken at the nearest-exact pixel; margin is the gap
    between the two largest normalised channel values there."""
    up = upsample(soft, patch)
    for c in range(up.shape[0]):
        mx, mn = up[c].max(), up[c].min()
        if mx > 0:
            up[c] = (up[c] - mn) / (mx - mn) if mx > mn else 0.0
    sel = up[:, nearest_exact_index(out_h, up.shape[1])][:, :, nearest_exact_index(out_w, up.shape[2])]
    labels = sel.argmax(0).astype(np.uint8)
    srt = np.sort(sel, axis=0)
    margin = srt[-1] - srt[-2] if sel.shape[0] > 1 else np.full(labels.shape, np.inf)
    return labels, margin


def boundary(mask):
    """DAVIS' seg2bmap at the mask's own size: a pixel differing from its right, lower or lower-right neighbour; the
    last row compares with the right one, the last column with the lower one, the bottom-right pixel is 0."""
    m = np.asarray(mask, dtype=bool)
    e, s, se = np.zeros_like(m), np.zeros_like(m), np.zeros_like(m)
    e[:, :-1] = m[:, 1:]
    s[:-1, :] = m[1:, :]
    se[:-1, :-1] = m[1:, 1:]
    b = (m ^ e) | (m ^ s) | (m ^ se)
    b[-1, :] = m[-1, :] ^ e[-1, :]
    b[:, -1] = m[:, -1] ^ s[:, -1]
    b[-1, -1] = False
    return b


def disk(r):
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    return x * x + y * y <= r * r


def radius(height, width):
    return int(math.ceil(0.008 * math.hypot(height, width)))


def jf_counts(pred, gt, num_objects, r):
    """int64 [K, 6] for one frame: intersection, union (outside void), pred and gt boundary pixels, pred and gt
    boundary pixels within the disk of radius r of the other's boundary."""
    pred, gt = np.asarray(pred), np.asarray(gt)
    void = gt == 255
    out = np.zeros((num_objects, 6), dtype=np.int64)
    for k in range(1, num_objects + 1):
        pm, gm = (pred == k) & ~void, gt == k
        bp, bg = boundary(pm), boundary(gm)
        dp = ndimage.binary_dilation(bp, structure=disk(r)) if bp.any() else np.zeros_like(bp)
        dg = ndimage.binary_dilation(bg, structure=disk(r)) if bg.any() else np.zeros_like(bg)
        out[k - 1] = [(pm & gm).sum(), (pm | gm).sum(), bp.sum(), bg.sum(), (bp & dg).sum(), (bg & dp).sum()]
    return out


def j_and_f(pred, gt, num_objects):
    """(J [K], F [K]) of one frame, straight from the DAVIS definitions."""
    r = radius(*np.asarray(gt).shape)
    J, F = [], []
    for inter, union, nbp, nbg, mp, mg in jf_counts(pred, gt, num_objects, r):
        J.append(1.0 if union == 0 else inter / union)
        if nbp == 0 and nbg == 0:
            p = rc = 1.0
        elif nbp == 0:
            p, rc = 1.0, 0.0
        elif nbg == 0:
            p, rc = 0.0, 1.0
        else:
            p, rc = mp / nbp, mg / nbg
        F.append(0.0 if p + rc == 0 else 2 * p * rc / (p + rc))
    return np.array(J), np.array(F)
