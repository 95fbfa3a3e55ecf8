"""Semantic keypoint correspondence: the nearest neighbour of each source keypoint's descriptor among the pixels of the
bilinearly upsampled target features, scored by PCK.  This is the project's protocol, modelled on the SPair-71k
semantic correspondence evaluation that Probe3D and DINOv3 report; defaults image_size = 512, alphas = (0.01, 0.05,
0.1).

Pairs.  An SPair-71k root: every PairAnnotation/<split>/*.json (default split "test") in sorted file-name order, of
which the fields src_imname, trg_imname, category, src_kps, trg_kps and trg_bndbox are read; the images are
JPEGImages/<category>/<imname>.  Or an .npz holding images (uint8 [N, H, W, 3]), pairs (int [M, 2]: source and target
index), src_kps / trg_kps (float [M, Kmax, 2], x then y), n_kps (int [M]), trg_bbox (float [M, 4]: x1 y1 x2 y2) and
categories (str [M]).

Images.  Every image is resized to image_size x image_size (S, a multiple of the patch size): torch's bilinear
interpolation (align_corners=False, antialias=False) of the image in [0, 1], then the crop mean / std
(d3_video_resize).

Features.  The teacher's last-block normalised patch tokens (`get_intermediate_layers(x, n=1)`), each row
L2-normalised in fp32 and rounded to bf16 (d3_knn_normalize).  The pairs are taken category by category, and each image
of a category is extracted once however many pairs it appears in.

Keypoints.  A keypoint (u, v) is in pixel-index coordinates of its W x H image.  Its resized pixel is
x = clamp(floor((u + 0.5) S / W), 0, S - 1), and y the same with v and H.  A predicted pixel (x*, y*) maps back to
((x* + 0.5) W_t / S - 0.5, (y* + 0.5) H_t / S - 0.5) in the W_t x H_t target; at S = W this is the identity.

Upsampling.  U(y, x) is torch's bilinear F.interpolate(align_corners=False) of the [h, w, D] patch map to S x S:
source position max((y + 0.5) h / S - 0.5, 0), and at the last row and column the two corners are the same cell.

Match.  The source descriptor is q = U_s(y_k, x_k), L2-normalised and rounded to bf16 (d3_corr_descriptors).  The
prediction is the target pixel with the largest <q, U_t(y, x)> / (||q|| ||U_t(y, x)||) over all S^2 pixels, the lowest
y S + x on ties; no window, soft-argmax, flip or refinement.  The cosine is exact at every pixel without a
full-resolution map: the numerator is the 4-tap blend of the patch similarities <q, f> (d3_gemm_bf16, one GEMM per
target image over every keypoint that has it as target) and ||U_t||^2 is the corner weights' quadratic form in the
per-patch Gram (d3_corr_gram); d3_corr_argmax evaluates both at every pixel and keeps the best.

Score.  A keypoint is correct at alpha when its distance to the target keypoint is <= alpha max(x2 - x1, y2 - y1) of
the target box.  Per alpha: the per-point PCK over all keypoints pooled ("PCK@alpha"), the per-image PCK, the mean
over pairs of each pair's fraction correct ("PCK-image@alpha"; a pair without keypoints is left out of it), and both
per category.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops
from .knn import RGB_MEAN, RGB_STD, _device

bf16, f32 = torch.bfloat16, torch.float32


def keypoint_pixels(kps, width: int, height: int, S: int) -> np.ndarray:
    """int64 [n, 2] resized pixels (x, y) of keypoints kps [n, 2] (u, v) in a width x height image:
    clamp(floor((u + 0.5) S / width), 0, S - 1), and the same for v."""
    k = np.asarray(kps, dtype=np.float64).reshape(-1, 2)
    size = np.array([width, height], dtype=np.float64)
    return np.clip(np.floor((k + 0.5) * S / size), 0, S - 1).astype(np.int64)


def back_map(xy, width: int, height: int, S: int) -> np.ndarray:
    """float64 [n, 2] coordinates in a width x height image of resized pixels xy [n, 2]: (x + 0.5) width / S - 0.5."""
    p = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
    return (p + 0.5) * np.array([width, height], dtype=np.float64) / S - 0.5


def pck_scores(pairs, alphas) -> dict:
    """{"PCK@a", "PCK-image@a"} for each alpha over pairs = [(pred [n, 2], trg [n, 2], bbox (x1, y1, x2, y2))]: per point
    over all keypoints pooled, per image as the mean over the pairs that have keypoints of each pair's fraction."""
    out = {}
    dist = [np.sqrt(((np.asarray(p, np.float64) - np.asarray(t, np.float64)) ** 2).sum(1)) for p, t, _ in pairs]
    size = [max(b[2] - b[0], b[3] - b[1]) for _, _, b in pairs]
    for a in alphas:
        ok = [d <= a * s for d, s in zip(dist, size)]
        pooled = np.concatenate(ok) if ok else np.zeros(0, bool)
        per_img = [o.mean() for o in ok if len(o)]
        out[f"PCK@{a:g}"] = float(pooled.mean()) if len(pooled) else float("nan")
        out[f"PCK-image@{a:g}"] = float(np.mean(per_img)) if per_img else float("nan")
    return out


def image_features(model, images, S: int, batch_size: int, rgb_mean, rgb_std, device) -> torch.Tensor:
    """bf16 [n * h * w, D] L2-normalised last-block patch tokens of the uint8 HWC images (any sizes) resized to S x S,
    `batch_size` images per forward."""
    p, D = int(model.patch_size), int(model.embed_dim)
    P = (S // p) ** 2
    feats = torch.empty(len(images) * P, D, dtype=bf16, device=device)
    for b0 in range(0, len(images), batch_size):
        chunk = [np.ascontiguousarray(im, dtype=np.uint8) for im in images[b0:b0 + batch_size]]
        offs = np.cumsum([0] + [im.size for im in chunk])
        flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in chunk])).to(device)
        desc = torch.tensor([[int(o), im.shape[0], im.shape[1]] for o, im in zip(offs, chunk)], dtype=torch.int64,
                            device=device)
        n = len(chunk)
        x = ops.video_resize(flat, desc, torch.empty(n, S, S, 3, dtype=bf16, device=device), mean=rgb_mean, std=rgb_std)
        patches = model.get_intermediate_layers(x, n=1)[0]
        ops.knn_normalize(patches.reshape(n * P, D).contiguous(), y_bf16=feats[b0 * P:(b0 + n) * P])
    return feats


def match_keypoints(feats: torch.Tensor, grid, S: int, kp, targets) -> tuple:
    """(xy int32 [K, 2], cosine fp32 [K]) on the device: the best target pixel of each keypoint.  feats bf16
    [n_maps * h * w, D] holds the patch maps; kp int [K, 3] = (source map, x, y) at S x S; targets int [K] the target
    map of each keypoint, ascending, so that the keypoints of one target are contiguous: one GEMM and one argmax per
    target map."""
    h, w = grid
    P, D, dev = h * w, feats.shape[1], feats.device
    n_maps = feats.shape[0] // P
    kp = np.asarray(kp, dtype=np.int32).reshape(-1, 3)
    targets = np.asarray(targets, dtype=np.int64).reshape(-1)
    K = len(kp)
    assert len(targets) == K and (np.diff(targets) >= 0).all()
    q = torch.empty(K, D, dtype=bf16, device=dev)
    qnorm = torch.empty(K, dtype=f32, device=dev)
    xy = torch.empty(K, 2, dtype=torch.int32, device=dev)
    cosine = torch.empty(K, dtype=f32, device=dev)
    if K == 0:
        return xy, cosine
    ops.corr_descriptors(feats, n_maps, grid, (S, S), kp, q, qnorm)
    used = np.unique(targets)
    gram = torch.empty(n_maps * P, 5, dtype=f32, device=dev)
    ops.corr_gram(feats, n_maps, grid, gram)
    starts = np.searchsorted(targets, used, side="left")
    ends = np.searchsorted(targets, used, side="right")
    ld = -(-P // 8) * 8                                          # 16-byte aligned fp32 similarity rows
    sim = torch.empty(int((ends - starts).max()), ld, dtype=f32, device=dev)
    for t, a, b in zip(used.tolist(), starts.tolist(), ends.tolist()):
        s = ops.gemm(q[a:b], feats[t * P:(t + 1) * P], sim[:b - a, :P])
        ops.corr_argmax(s, gram[t * P:(t + 1) * P], qnorm[a:b], grid, (S, S), xy[a:b], cosine[a:b])
    return xy, cosine


def eval_correspondence(model, dataset, *, image_size: int = 512, alphas=(0.01, 0.05, 0.1), batch_size: int = 16,
                        num_workers: int = 4, device=None, rgb_mean=RGB_MEAN, rgb_std=RGB_STD, **_ignored) -> dict:
    """PCK of nearest-neighbour keypoint transfer through `model`'s patch features over the pairs of `dataset` (as
    SPairDataset: `pairs`, `load_image`).  Returns {"PCK@a", "PCK-image@a" for each alpha, "categories": {name:
    {"PCK@a", "PCK-image@a", "n_pairs", "n_keypoints"}}, "n_pairs", "n_keypoints", "protocol"}.  The extra keys of
    an `evaluation.correspondence` block (dataset_path, split) are accepted and ignored."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    S, p = int(image_size), int(model.patch_size)
    alphas = [float(a) for a in alphas]
    if S < p or S % p:
        raise ValueError(f"image_size {S} must be a positive multiple of the patch size {p}")
    if not alphas or min(alphas) <= 0:
        raise ValueError(f"alphas must be positive, got {alphas}")
    protocol = {"image_size": S, "alphas": alphas}
    grid = (S // p, S // p)
    pairs = list(dataset.pairs)
    if not pairs:
        raise ValueError("the dataset holds no pair")
    by_cat = {}
    for i, pr in enumerate(pairs):
        by_cat.setdefault(pr["category"], []).append(i)
    scored, per_cat = [], {}
    for cat in sorted(by_cat):
        idx = by_cat[cat]
        ims = sorted({pairs[i]["src"] for i in idx} | {pairs[i]["trg"] for i in idx})
        local = {g: j for j, g in enumerate(ims)}
        loader = torch.utils.data.DataLoader(_Images(dataset, ims), batch_size=None, shuffle=False,
                                             num_workers=int(num_workers), collate_fn=_identity,
                                             persistent_workers=False)
        images = list(loader)
        sizes = [(im.shape[1], im.shape[0]) for im in images]           # (W, H)
        with torch.no_grad():
            feats = image_features(model, images, S, int(batch_size), rgb_mean, rgb_std, dev)
        del images
        order = sorted(idx, key=lambda i: (local[pairs[i]["trg"]], i))  # keypoints of one target contiguous
        kp, tg, spans = [], [], {}
        for i in order:
            pr = pairs[i]
            s, t = local[pr["src"]], local[pr["trg"]]
            px = keypoint_pixels(pr["src_kps"], *sizes[s], S)
            spans[i] = (len(kp), len(kp) + len(px))
            kp += [(s, int(x), int(y)) for x, y in px]
            tg += [t] * len(px)
        xy, _ = match_keypoints(feats, grid, S, kp, tg)
        xy = xy.cpu().numpy()
        del feats
        cat_pairs = []
        for i in idx:
            pr = pairs[i]
            a, b = spans[i]
            pred = back_map(xy[a:b], *sizes[local[pr["trg"]]], S)
            cat_pairs.append((pred, np.asarray(pr["trg_kps"], np.float64).reshape(-1, 2), list(pr["trg_bbox"])))
        per_cat[cat] = {**pck_scores(cat_pairs, alphas), "n_pairs": len(idx),
                        "n_keypoints": int(sum(len(t) for _, t, _ in cat_pairs))}
        scored += cat_pairs
    return {**pck_scores(scored, alphas), "categories": per_cat, "n_pairs": len(scored),
            "n_keypoints": int(sum(len(t) for _, t, _ in scored)), "protocol": protocol}


class _Images:
    """The images `indices` of a correspondence dataset, decoded in DataLoader workers."""

    def __init__(self, dataset, indices):
        self.dataset, self.indices = dataset, list(indices)

    def __len__(self):
        return len(self.indices)

    def __getitem__(self, i):
        return self.dataset.load_image(self.indices[i])


def _identity(item):
    return item
