"""Float64 statement of the linear segmentation probe's per-pixel arithmetic (dinov3_jax/eval/segmentation.py):
bilinear upsampling with align_corners=False as explicit interpolation matrices, the mean cross-entropy over the
pixels not labelled 255 with its gradient to the patch logits, the argmax confusion matrix, and mIoU / mAcc / aAcc."""
import numpy as np

IGNORE = 255


def interp_matrix(n_out: int, n_in: int) -> np.ndarray:
    """A [n_out, n_in] with upsampled = A @ x along one axis: torch's source index s = max((o + 0.5) * n_in / n_out
    - 0.5, 0), cells i0 = floor(s), i1 = min(i0 + 1, n_in - 1), weights (1 - (s - i0), s - i0)."""
    A = np.zeros((n_out, n_in))
    for o in range(n_out):
        s = max((o + 0.5) * n_in / n_out - 0.5, 0.0)
        i0 = int(np.floor(s))
        i1 = min(i0 + 1, n_in - 1)
        lam = s - i0
        A[o, i0] += 1.0 - lam
        A[o, i1] += lam
    return A


def upsample(logits: np.ndarray, Hl: int, Wl: int) -> np.ndarray:
    """[B, h, w, C] -> [B, Hl, Wl, C]"""
    _, h, w, _ = logits.shape
    return np.einsum("yi,bijc,xj->byxc", interp_matrix(Hl, h), logits, interp_matrix(Wl, w), optimize=True)


def xent(logits: np.ndarray, labels: np.ndarray):
    """(loss, d loss / d logits [B, h, w, C], valid pixel count): the mean over the pixels with label < C of the
    cross-entropy of the upsampled logits (loss and gradient 0 when no pixel is valid)."""
    B, h, w, C = logits.shape
    _, Hl, Wl = labels.shape
    z = upsample(logits.astype(np.float64), Hl, Wl)
    m = z.max(-1, keepdims=True)
    lse = (m + np.log(np.exp(z - m).sum(-1, keepdims=True)))[..., 0]
    valid = labels < C
    n = int(valid.sum())
    if n == 0:
        return 0.0, np.zeros_like(logits, dtype=np.float64), 0
    y = np.where(valid, labels, 0).astype(np.int64)
    zy = np.take_along_axis(z, y[..., None], -1)[..., 0]
    loss = float(((lse - zy) * valid).sum() / n)
    g = np.exp(z - lse[..., None])
    np.put_along_axis(g, y[..., None], np.take_along_axis(g, y[..., None], -1) - 1.0, -1)
    g *= valid[..., None] / n
    grad = np.einsum("yi,byxc,xj->bijc", interp_matrix(Hl, h), g, interp_matrix(Wl, w), optimize=True)
    return loss, grad, n


def grad_envelope(logits: np.ndarray, labels: np.ndarray) -> np.ndarray:
    """sum over pixels of w * |softmax - onehot| / count per patch logit: the size of the terms each gradient element
    adds, which bounds the rounding of any order of summation."""
    B, h, w, C = logits.shape
    _, Hl, Wl = labels.shape
    z = upsample(logits.astype(np.float64), Hl, Wl)
    p = np.exp(z - z.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    valid = labels < C
    n = max(int(valid.sum()), 1)
    y = np.where(valid, labels, 0).astype(np.int64)
    np.put_along_axis(p, y[..., None], np.abs(np.take_along_axis(p, y[..., None], -1) - 1.0), -1)
    p *= valid[..., None] / n
    return np.einsum("yi,byxc,xj->bijc", interp_matrix(Hl, h), p, interp_matrix(Wl, w), optimize=True)


def confusion(logits: np.ndarray, labels: np.ndarray, C: int):
    """(int64 [C, C] counts of (label, argmax) over the pixels with label < C, ties to the lower class; the per-pixel
    gap between the two best upsampled logits)."""
    _, Hl, Wl = labels.shape
    z = upsample(logits.astype(np.float64), Hl, Wl)
    pred = z.argmax(-1)
    top2 = np.sort(z, -1)[..., -2:]
    gap = top2[..., 1] - top2[..., 0]
    valid = labels < C
    conf = np.bincount(labels[valid].astype(np.int64) * C + pred[valid], minlength=C * C).reshape(C, C)
    return conf, gap


def metrics(conf: np.ndarray) -> dict:
    """mIoU over the classes with a non-empty union, mAcc over the classes present in the labels, aAcc; percent."""
    conf = np.asarray(conf, dtype=np.float64)
    tp, gt, pred = np.diag(conf), conf.sum(1), conf.sum(0)
    union = gt + pred - tp
    ious = [tp[c] / union[c] for c in range(len(tp)) if union[c] > 0]
    accs = [tp[c] / gt[c] for c in range(len(tp)) if gt[c] > 0]
    return {"mIoU": 100.0 * sum(ious) / len(ious), "mAcc": 100.0 * sum(accs) / len(accs),
            "aAcc": 100.0 * tp.sum() / gt.sum()}
