"""Unsupervised object discovery: TokenCut's normalized cut on the patch-affinity graph of each image, scored by CorLoc.
This is the project's protocol, modelled on TokenCut and on LOST's PASCAL VOC evaluation; defaults tau = 0.2,
eps = 1e-5.

Images.  A PASCAL VOC root (VOC2007 or VOC2012): the ids of ImageSets/Main/<split>.txt (default "trainval"), the
images JPEGImages/<id>.jpg and the boxes of Annotations/<id>.xml.  Or an .npz holding images (uint8 [N, Hmax, Wmax, 3]),
sizes (int [N, 2]: H, W; image i is images[i, :H, :W]), boxes (float [N, Bmax, 4]: x1 y1 x2 y2) and n_boxes (int [N]).
Images are not resized (TokenCut and LOST run at native resolution).  Each image is normalised with the crop mean and
std (d3_video_resize at its own size, an identity resampling) and zero-padded at the right and bottom to the next
multiple of the patch size p, the zeros written after the normalisation; its grid is h = ceil(H / p) by
w = ceil(W / p).  Images are grouped by grid, in the dataset's order within a grid, and extracted `batch_size` at a time.

Features.  The teacher's last-block normalised patch tokens (`get_intermediate_layers(x, n=1)`), each row L2-normalised
in fp32 and rounded to bf16 (d3_knn_normalize).  TokenCut used the last attention layer's keys; this protocol uses the
output tokens, as the video and correspondence evaluations do.

Graph.  s = F F^T (d3_gemm_bf16, fp32 out).  A_ij = 1 if s_ij > tau, else eps, the diagonal included; d_i = sum_j A_ij
(d3_od_graph, from the integer count of entries above tau).

Eigenvector.  The generalized eigenvector x of (D - A) x = lambda D x with the second-smallest lambda.  Equivalently
the eigenvector y of M = D^-1/2 A D^-1/2 with the second-largest eigenvalue theta, x = D^-1/2 y, lambda_2 = 1 - theta;
M's top eigenpair is (1, D^1/2 1) in closed form, simple because every A_ij > 0.  d3_od_fiedler finds it by deflated
Lanczos with full reorthogonalisation, stopping when the residual bound falls to 1e-6 or after 256 steps; an image that
reaches 256 steps first still gets a box and is counted in n_unconverged.

Bipartition.  The foreground candidates are the patches with x_i > mean(x); the seed is argmax |x_i|, the lowest index
on ties; if the seed is not a candidate the complement is taken (TokenCut's sign flip: the result does not depend on the
eigenvector's sign or scale).

Box.  The 4-connected component of the foreground that holds the seed (scipy.ndimage.label's default structure); its
grid bounding box [x0, y0, x1, y1] gives the pixel box [x0 p, y0 p, (x1 + 1) p, (y1 + 1) p], clipped to the W x H image
(d3_od_box).

Score.  Ground truth is every object/bndbox of the VOC XML, VOC's 1-based inclusive corners becoming
[xmin - 1, ymin - 1, xmax, ymax]; remove_difficult (default false) drops the objects marked difficult.  An image left
with no ground-truth box is not scored.  IoU is computed on areas of continuous coordinates, without a + 1.  CorLoc is
the fraction of scored images whose box reaches IoU >= 0.5 with at least one ground-truth box.  Also reported: n_images
(the scored images) and n_unconverged; with save_boxes, each image's box and best IoU.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops
from .knn import RGB_MEAN, RGB_STD, _device

bf16, f32 = torch.bfloat16, torch.float32


def grid_of(size, patch: int) -> tuple:
    """(h, w) = (ceil(H / patch), ceil(W / patch)) of an image of size (H, W)."""
    return -(-int(size[0]) // patch), -(-int(size[1]) // patch)


def box_iou(box, gts) -> np.ndarray:
    """float64 [B]: the IoU of box (x1, y1, x2, y2) with each row of gts [B, 4], on continuous areas (no + 1)."""
    b = np.asarray(box, np.float64).reshape(4)
    g = np.asarray(gts, np.float64).reshape(-1, 4)
    iw = np.clip(np.minimum(b[2], g[:, 2]) - np.maximum(b[0], g[:, 0]), 0, None)
    ih = np.clip(np.minimum(b[3], g[:, 3]) - np.maximum(b[1], g[:, 1]), 0, None)
    inter = iw * ih
    union = (b[2] - b[0]) * (b[3] - b[1]) + (g[:, 2] - g[:, 0]) * (g[:, 3] - g[:, 1]) - inter
    return np.where(union > 0, inter / np.where(union > 0, union, 1.0), 0.0)


def corloc(boxes, gts) -> float:
    """The fraction of images whose box (boxes[i]) has IoU >= 0.5 with some row of gts[i]."""
    hits = [bool(len(g)) and box_iou(b, g).max() >= 0.5 for b, g in zip(boxes, gts)]
    return float(np.mean(hits)) if hits else float("nan")


def image_features(model, images, rgb_mean, rgb_std, device) -> torch.Tensor:
    """bf16 [n, h * w, D]: the L2-normalised last-block patch tokens of uint8 HWC images that share one grid (h, w):
    each image normalised at its own size and zero-padded to h p x w p."""
    p, D = int(model.patch_size), int(model.embed_dim)
    h, w = grid_of(images[0].shape[:2], p)
    n = len(images)
    x = torch.zeros(n, h * p, w * p, 3, dtype=bf16, device=device)
    for b, im in enumerate(images):
        im = np.ascontiguousarray(im, dtype=np.uint8)
        H, W = im.shape[:2]
        assert grid_of((H, W), p) == (h, w), "the images of one batch must share a grid"
        desc = torch.tensor([[0, H, W]], dtype=torch.int64, device=device)
        one = torch.empty(1, H, W, 3, dtype=bf16, device=device)
        ops.video_resize(torch.from_numpy(im.reshape(-1)).to(device), desc, one, mean=rgb_mean, std=rgb_std)
        x[b, :H, :W] = one[0]
    patches = model.get_intermediate_layers(x, n=1)[0]
    feats = torch.empty(n, h * w, D, dtype=bf16, device=device)
    ops.knn_normalize(patches.reshape(n * h * w, D).contiguous(), y_bf16=feats.view(n * h * w, D))
    return feats


def normalized_cut(feats: torch.Tensor, tau: float = 0.2, eps: float = 1e-5, k_max: int = 256) -> dict:
    """The graph and eigenvector of each image of feats bf16 [n, P, D] (unit rows) on the device: {"sim" fp32 [n, P, P]
    view, "bits", "degree", "x" fp32 [n, P], "lambda2", "iters", "converged"}."""
    n, P, D = feats.shape
    dev = feats.device
    ld = -(-P // 8) * 8                                          # 16-byte aligned fp32 similarity rows
    sim = torch.empty(n, P, ld, dtype=f32, device=dev)[:, :, :P]
    for m in range(n):
        ops.gemm(feats[m], feats[m], sim[m])
    bits = torch.empty(n, P, -(-P // 32), dtype=torch.int32, device=dev)
    degree = torch.empty(n, P, dtype=f32, device=dev)
    ops.od_graph(sim, tau, eps, bits, degree)
    x = torch.empty(n, P, dtype=f32, device=dev)
    lam = torch.empty(n, dtype=f32, device=dev)
    iters = torch.empty(n, dtype=torch.int32, device=dev)
    conv = torch.empty(n, dtype=torch.int32, device=dev)
    ops.od_fiedler(bits, degree, eps, x, lam, iters, conv, k_max=k_max)
    return {"sim": sim, "bits": bits, "degree": degree, "x": x, "lambda2": lam, "iters": iters, "converged": conv}


def boxes_of(x: torch.Tensor, grid, patch: int, sizes, gts) -> dict:
    """d3_od_box on the device for eigenvectors x fp32 [n, h * w]: {"fg" uint8 [n, h * w], "box" int32 [n, 4],
    "iou" fp32 [n], "hit" int32 [n]}; sizes [(H, W)] and gts [float [B_i, 4]] per image."""
    n, dev = x.shape[0], x.device
    b_max = max([len(g) for g in gts] + [1])
    gt = np.zeros((n, b_max, 4), np.float32)
    for i, g in enumerate(gts):
        gt[i, :len(g)] = np.asarray(g, np.float32).reshape(-1, 4)
    out = {"fg": torch.empty(n, x.shape[1], dtype=torch.uint8, device=dev),
           "box": torch.empty(n, 4, dtype=torch.int32, device=dev), "iou": torch.empty(n, dtype=f32, device=dev),
           "hit": torch.empty(n, dtype=torch.int32, device=dev)}
    ops.od_box(x, grid, patch, sizes, [len(g) for g in gts], torch.from_numpy(gt).to(dev), out["fg"], out["box"],
               out["iou"], out["hit"])
    return out


def eval_object_discovery(model, dataset, *, tau: float = 0.2, eps: float = 1e-5, batch_size: int = 16,
                          num_workers: int = 4, save_boxes: bool = False, device=None, rgb_mean=RGB_MEAN,
                          rgb_std=RGB_STD, **_ignored) -> dict:
    """CorLoc of TokenCut boxes through `model`'s patch features over `dataset` (as VOCDiscoveryDataset: `names`,
    `sizes`, `boxes`, `load_image`).  Returns {"CorLoc", "n_images", "n_unconverged", "protocol"} and, with
    save_boxes, "boxes": {name: {"box": [x0, y0, x1, y1], "iou"}}.  The extra keys of an `evaluation.discovery` block
    (dataset_path, split, remove_difficult) are accepted and ignored."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    p = int(model.patch_size)
    tau, eps = float(tau), float(eps)
    if not 0.0 < eps < 1.0:
        raise ValueError(f"eps must lie in (0, 1), got {eps}")
    scored = [i for i in range(len(dataset)) if len(dataset.boxes[i])]
    if not scored:
        raise ValueError("the dataset holds no image with a ground-truth box")
    order = sorted(scored, key=lambda i: (grid_of(dataset.sizes[i], p), i))
    loader = torch.utils.data.DataLoader(_Images(dataset, order), batch_size=None, shuffle=False,
                                         num_workers=int(num_workers), collate_fn=_identity, persistent_workers=False)
    per_image, chunk = {}, []

    def run(chunk):
        idx = [i for i, _ in chunk]
        grid = grid_of(dataset.sizes[idx[0]], p)
        with torch.no_grad():
            feats = image_features(model, [im for _, im in chunk], rgb_mean, rgb_std, dev)
        cut = normalized_cut(feats, tau, eps)
        out = boxes_of(cut["x"], grid, p, [dataset.sizes[i] for i in idx], [dataset.boxes[i] for i in idx])
        box, iou, hit = out["box"].cpu().numpy(), out["iou"].cpu().numpy(), out["hit"].cpu().numpy()
        conv = cut["converged"].cpu().numpy()
        for k, i in enumerate(idx):
            per_image[i] = (box[k].tolist(), float(iou[k]), bool(hit[k]), bool(conv[k]))

    for i, im in zip(order, loader):
        if im.shape[:2] != tuple(dataset.sizes[i]):
            raise ValueError(f"image {dataset.names[i]}: decoded size {im.shape[:2]} differs from the annotated "
                             f"{tuple(dataset.sizes[i])}")
        if chunk and (len(chunk) == int(batch_size) or grid_of(dataset.sizes[chunk[0][0]], p) != grid_of(im.shape, p)):
            run(chunk)
            chunk = []
        chunk.append((i, im))
    run(chunk)
    res = {"CorLoc": float(np.mean([per_image[i][2] for i in scored])), "n_images": len(scored),
           "n_unconverged": int(sum(not per_image[i][3] for i in scored)),
           "protocol": {"tau": tau, "eps": eps, "patch_size": p}}
    if save_boxes:
        res["boxes"] = {str(dataset.names[i]): {"box": per_image[i][0], "iou": per_image[i][1]} for i in scored}
    return res


class _Images:
    """The images `indices` of a discovery dataset, decoded in DataLoader workers."""

    def __init__(self, dataset, indices):
        self.dataset, self.indices = dataset, list(indices)

    def __len__(self):
        return len(self.indices)

    def __getitem__(self, i):
        return self.dataset.load_image(self.indices[i])


def _identity(item):
    return item
