"""The keypoint correspondence protocol (dinov3_jax/eval/correspondence.py) stated in float64 on the CPU: the target map
is materialised at full resolution with torch's F.interpolate, and every cosine is computed and compared there."""
import numpy as np
import torch
import torch.nn.functional as Fn


def upsample(feat, out_hw):
    """float64 [H, W, D]: torch's bilinear F.interpolate (align_corners=False) of the patch map feat [h, w, D]."""
    f = torch.as_tensor(np.asarray(feat), dtype=torch.float64).permute(2, 0, 1)[None]
    return Fn.interpolate(f, size=tuple(out_hw), mode="bilinear", align_corners=False)[0].permute(1, 2, 0)


def descriptor(feat, out_hw, x, y):
    """float64 [D]: U(y, x) of the upsampled map (not normalised)."""
    return upsample(feat, out_hw)[y, x].numpy()


def cosines(q, feat, out_hw, chunk=64):
    """float64 [K, H * W]: the cosine of every descriptor row of q [K, D] with every pixel of the upsampled map, 0 where
    either norm is 0."""
    U = upsample(feat, out_hw).reshape(-1, np.asarray(feat).shape[-1])
    un = torch.linalg.vector_norm(U, dim=1)
    q = torch.as_tensor(np.asarray(q), dtype=torch.float64).reshape(-1, U.shape[1])
    out = []
    for k0 in range(0, len(q), chunk):
        qc = q[k0:k0 + chunk]
        den = torch.linalg.vector_norm(qc, dim=1)[:, None] * un[None]
        num = qc @ U.T
        out.append(torch.where(den > 0, num / torch.where(den > 0, den, 1.0), 0.0))
    return torch.cat(out).numpy() if out else np.zeros((0, U.shape[0]))


TIE = 1e-12      # float64 rounding of equal values (the bands of pixels that read one row of cells, say)


def match(q, feat, out_hw):
    """(x, y) int [K, 2] of the best pixel per descriptor, the lowest index y W + x among the maxima (cosines within
    TIE of the largest), and the cosine matrix [K, H * W]."""
    cos = cosines(q, feat, out_hw)
    idx = np.argmax(cos >= cos.max(1, keepdims=True) - TIE, axis=1)      # the first True
    W = int(out_hw[1])
    return np.stack([idx % W, idx // W], axis=1), cos


def keypoint_pixel(u, size, S):
    """The resized pixel of keypoint coordinate u in an image of `size` pixels: clamp(floor((u + 0.5) S / size), 0,
    S - 1)."""
    return np.clip(np.floor((np.asarray(u, dtype=np.float64) + 0.5) * S / size), 0, S - 1).astype(np.int64)


def back_map(p, size, S):
    """The original-image coordinate of resized pixel p: (p + 0.5) size / S - 0.5."""
    return (np.asarray(p, dtype=np.float64) + 0.5) * size / S - 0.5


def pck(pairs, alphas):
    """Per-point and per-image PCK from pairs = [(pred [n, 2], trg [n, 2], bbox (x1, y1, x2, y2), category)]: a keypoint
    is correct at alpha when its distance is <= alpha * max(x2 - x1, y2 - y1).  Returns {"PCK@a", "PCK-image@a",
    "categories": {c: {...}}}; pairs without keypoints count in neither mean."""
    def score(sel):
        out = {}
        for a in alphas:
            hits, per_img = [], []
            for pred, trg, box, _ in sel:
                if len(trg) == 0:
                    continue
                d = np.sqrt(((np.asarray(pred, np.float64) - np.asarray(trg, np.float64)) ** 2).sum(1))
                ok = d <= a * max(box[2] - box[0], box[3] - box[1])
                hits += ok.tolist()
                per_img.append(ok.mean())
            out[f"PCK@{a:g}"] = float(np.mean(hits))
            out[f"PCK-image@{a:g}"] = float(np.mean(per_img))
        return out
    res = score(pairs)
    res["categories"] = {c: score([p for p in pairs if p[3] == c]) for c in sorted({p[3] for p in pairs})}
    return res
