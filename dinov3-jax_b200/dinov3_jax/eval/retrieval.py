"""Instance retrieval on revisited Oxford / Paris: a multi-scale class-token descriptor per image, cosine ranking, and
the revisited mAP and mP@k of the Easy, Medium and Hard protocols.  This is the project's protocol, modelled on the
revisited benchmark (Radenovic et al., 2018) run the way DINO's eval_image_retrieval.py runs it.

Data.  A revisited root holds gnd_<dataset>.pkl (dataset roxford5k or rparis6k) with `imlist` (database names),
`qimlist` (query names) and `gnd`, one dict per query with `bbx` (x1, y1, x2, y2) and the database indices `easy`,
`hard` and `junk` (lists or ndarrays); the images are jpg/<name>.jpg.  The pickle is read by a restricted unpickler that
builds only builtin containers, numbers, strings and numpy arrays, and refuses any other global before it is called.
Or an .npz holding db_images (uint8 [N, Hmax, Wmax, 3]) with db_sizes (int [N, 2]: H, W), q_images and q_sizes likewise,
q_bbx (float [Q, 4]) and easy / hard / junk as CSR pairs (easy_ptr int [Q + 1], easy_idx int, ...).

Query crop.  A query image is cut to [floor x1, floor y1, ceil x2, ceil y2], clipped to the image.  Database images are
not cropped.

Sizes.  For an image (or query crop) of H x W, r = min(1, image_size / max(H, W)) (an image is never enlarged, as with a
thumbnail; image_size 512 by default).  At each scale s of `scales` (default 1, 2^-1/2, 1/2) each side becomes
max(p, p * floor(side * r * s / p + 0.5)), computed in float64 on the host: every input is a whole number of patches,
with no padding tokens and no dropped border pixels.

Resize.  Each (image, scale) is resized from uint8 straight to its size with torch's antialiased bicubic filter
(F.interpolate(mode="bicubic", antialias=True, align_corners=False) on float values; the source window is the crop),
normalised with the crop mean and std and stored as bf16 (d3_ret_resize).  This replaces DINO's PIL Lanczos thumbnail
and its second, bilinear rescale.  The inputs are grouped by size; within a group they keep the dataset's order (then
the scale order) and are extracted `batch_size` at a time.

Descriptor.  The teacher's last-block class token after the final norm (`model(x)`), in fp32, at each scale; the
descriptor is the L2-normalised sum over the scales in the listed order (DINO's multi_scale; d3_ret_scale_sum, then
d3_knn_normalize), rounded to bf16 for the similarity GEMM.

Ranking.  s = Q DB^T (d3_gemm_bf16, fp32 out).  Database images are ordered by descending s, ties to the lower database
index first (d3_ret_rank_ap: exact integer ranks, no full sort).

Ground truth per protocol:  Easy: ok = easy, junk = junk + hard.  Medium: ok = easy + hard, junk = junk.  Hard:
ok = hard, junk = junk + easy.  An index in both ok and junk counts as ok.

Scores.  r_0 < r_1 < ... are the 0-based ranks of the ok images, each reduced by the number of junk images ranked above
it.  AP = sum_j ((r_j = 0 ? 1 : j / r_j) + (j + 1) / (r_j + 1)) / (2 n_ok), the revisited trapezoid, summed in fp64 in
ascending rank order.  mP@k for k in 1, 5, 10: with 1-based junk-free ranks, kq = min(max rank, k) and
P = |{rank <= kq}| / kq.  A query without ok images is left out of that protocol's means; n_empty counts them.  mAP and
mP@k are reported in percent, for Easy, Medium and Hard; with save_ranks, also each query's AP per protocol and its
top-100 database indices (d3_topk_merge).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .. import ops
from .knn import RGB_MEAN, RGB_STD, _device

bf16, f32 = torch.bfloat16, torch.float32
PROTOCOLS = ("easy", "medium", "hard")
KS = (1, 5, 10)
SCALES = (1.0, 2.0 ** -0.5, 0.5)


def scaled_size(size, image_size: int, scale: float, patch: int) -> tuple:
    """(h, w) in pixels of an H x W image at one scale: r = min(1, image_size / max(H, W)), each side
    max(p, p * floor(side * r * scale / p + 0.5)), in float64."""
    H, W = int(size[0]), int(size[1])
    r = min(1.0, float(image_size) / max(H, W))
    return tuple(max(patch, patch * math.floor(side * r * float(scale) / patch + 0.5)) for side in (H, W))


def query_box(bbx, size) -> tuple:
    """(x0, y0, x1, y1): the query box (x1, y1, x2, y2) widened to whole pixels, [floor x1, floor y1, ceil x2, ceil y2],
    and clipped to the H x W image."""
    H, W = int(size[0]), int(size[1])
    x1, y1, x2, y2 = (float(v) for v in bbx)
    box = (max(0, math.floor(x1)), max(0, math.floor(y1)), min(W, math.ceil(x2)), min(H, math.ceil(y2)))
    if box[2] <= box[0] or box[3] <= box[1]:
        raise ValueError(f"query box {[x1, y1, x2, y2]} leaves nothing of its {H} x {W} image")
    return box


def plan_inputs(sizes, boxes, image_size: int, scales, patch: int) -> list:
    """[(out (h, w), image i, scale index s, crop box)] of every (image, scale), ordered by size, then image, then
    scale.  boxes: a crop box per image (x0, y0, x1, y1), or None for whole images."""
    items = []
    for i, (H, W) in enumerate(sizes):
        box = (0, 0, int(W), int(H)) if boxes is None else tuple(boxes[i])
        crop = (box[3] - box[1], box[2] - box[0])
        for s, sc in enumerate(scales):
            items.append((scaled_size(crop, image_size, sc, patch), i, s, box))
    return sorted(items, key=lambda t: (t[0], t[1], t[2]))


def batches(items, batch_size: int):
    """The planned inputs cut into batches of one size, at most batch_size each."""
    out, cur = [], []
    for it in items:
        if cur and (len(cur) == int(batch_size) or cur[0][0] != it[0]):
            out.append(cur)
            cur = []
        cur.append(it)
    if cur:
        out.append(cur)
    return out


def resize_batch(images, batch, rgb_mean, rgb_std, device) -> torch.Tensor:
    """bf16 [n, h, w, 3]: each planned input of one batch (d3_ret_resize); images[k] the uint8 HWC image of batch[k]."""
    imgs = [np.ascontiguousarray(im, dtype=np.uint8) for im in images]
    offs = np.concatenate([[0], np.cumsum([im.size for im in imgs])[:-1]]).astype(np.int64)
    desc = [[int(o), im.shape[0], im.shape[1], *it[3]] for o, im, it in zip(offs, imgs, batch)]
    flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).to(device)
    h, w = batch[0][0]
    x = torch.empty(len(batch), h, w, 3, dtype=bf16, device=device)
    return ops.ret_resize(flat, desc, x, mean=rgb_mean, std=rgb_std)


def extract_descriptors(model, sizes, boxes, load, *, image_size: int = 512, scales=SCALES, batch_size: int = 16,
                        num_workers: int = 4, rgb_mean=RGB_MEAN, rgb_std=RGB_STD, device=None) -> dict:
    """{"desc": bf16 [n, D] unit descriptors, "cls": fp32 [S, n, D] the class tokens per scale} of the n images of
    `sizes` (cropped to `boxes`, or whole when None), `load(i)` giving image i as uint8 HWC."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    p, D, S, n = int(model.patch_size), int(model.embed_dim), len(scales), len(sizes)
    plan = batches(plan_inputs(sizes, boxes, image_size, scales, p), batch_size)
    loader = torch.utils.data.DataLoader(_Inputs(load, plan), batch_size=None, shuffle=False,
                                         num_workers=int(num_workers), collate_fn=_identity, persistent_workers=False)
    cls = torch.empty(S, n, D, dtype=f32, device=dev)
    for batch, images in zip(plan, loader):
        with torch.no_grad():
            tok = model(resize_batch(images, batch, rgb_mean, rgb_std, dev))
        ii = torch.tensor([it[1] for it in batch], device=dev)
        ss = torch.tensor([it[2] for it in batch], device=dev)
        cls[ss, ii] = tok
    total = torch.empty(n, D, dtype=f32, device=dev)
    ops.ret_scale_sum(cls, total)
    desc = torch.empty(n, D, dtype=bf16, device=dev)
    ops.knn_normalize(total, y_bf16=desc)
    return {"desc": desc, "cls": cls}


def csr(lists) -> tuple:
    """(ptr int64 [Q + 1], idx int64) of per-query index lists."""
    lens = [len(l) for l in lists]
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = np.concatenate([np.asarray(l, np.int64).reshape(-1) for l in lists]) if lists else np.zeros(0, np.int64)
    return ptr, idx.astype(np.int64)


def rank_queries(qdesc: torch.Tensor, dbdesc: torch.Tensor, easy, hard, junk, top: int = 0) -> dict:
    """The revisited scores of bf16 query descriptors [Q, D] against the database [N, D] (d3_gemm_bf16, then
    d3_ret_rank_ap): {"sim" fp32 [Q, N] view, "ranks" int32, "ap" fp64 [Q, 3], "pk" fp64 [Q, 3, 3], "n_ok" int32
    [Q, 3]} and, with top > 0, "top" int32 [Q, min(top, N)] the most similar database indices (d3_topk_merge)."""
    Q, N, dev = qdesc.shape[0], dbdesc.shape[0], qdesc.device
    sim = torch.empty(Q, -(-N // 8) * 8, dtype=f32, device=dev)[:, :N]       # 16-byte aligned fp32 rows
    ops.gemm(qdesc, dbdesc, sim)
    lists = [csr(l) for l in (easy, hard, junk)]
    out = {"sim": sim, "ranks": torch.empty(sum(len(l[1]) for l in lists), dtype=torch.int32, device=dev),
           "ap": torch.empty(Q, 3, dtype=torch.float64, device=dev),
           "pk": torch.empty(Q, 3, 3, dtype=torch.float64, device=dev),
           "n_ok": torch.empty(Q, 3, dtype=torch.int32, device=dev)}
    ops.ret_rank_ap(sim, N, *lists, out["ranks"], out["ap"], out["pk"], out["n_ok"])
    if top > 0:
        k = min(int(top), N)
        ts = torch.empty(Q, k, dtype=f32, device=dev)
        out["top"] = torch.empty(Q, k, dtype=torch.int32, device=dev)
        ops.topk_merge(sim, ts, out["top"], offset=0, valid=N, fresh=True)
    return out


def summarize(ap, pk, n_ok) -> dict:
    """{"mAP", "mP@k", "n_empty"} in percent over the queries with ok images, per protocol, from per-query fp64
    ap [Q, 3], pk [Q, 3, 3] and n_ok [Q, 3] (numpy); the means are taken in query order."""
    res = {"mAP": {}, "mP@k": {}, "n_empty": {}}
    for p, name in enumerate(PROTOCOLS):
        keep = n_ok[:, p] > 0
        res["n_empty"][name] = int((~keep).sum())
        res["mAP"][name] = 100.0 * float(np.mean(ap[keep, p])) if keep.any() else float("nan")
        res["mP@k"][name] = {str(k): (100.0 * float(np.mean(pk[keep, p, t])) if keep.any() else float("nan"))
                             for t, k in enumerate(KS)}
    return res


def eval_instance_retrieval(model, dataset, *, image_size: int = 512, scales=SCALES, batch_size: int = 16,
                            num_workers: int = 4, save_ranks: bool = False, device=None, rgb_mean=RGB_MEAN,
                            rgb_std=RGB_STD, **_ignored) -> dict:
    """Revisited mAP and mP@k (percent) of `model`'s multi-scale class-token descriptors over `dataset` (as
    RevisitedDataset).  Returns {"mAP": {protocol: float}, "mP@k": {protocol: {"1", "5", "10"}}, "n_empty":
    {protocol: int}, "n_queries", "n_database", "protocol"} and, with save_ranks, "ranks": {query name: {"ap":
    {protocol: float or None}, "top": [the 100 most similar database indices]}}.  The extra keys of an
    `evaluation.retrieval` block (dataset_path, dataset) are accepted and ignored."""
    scales = [float(s) for s in scales]
    if not scales or not all(s > 0 for s in scales):
        raise ValueError(f"scales must be positive, got {scales}")
    if int(image_size) < 1:
        raise ValueError(f"image_size must be positive, got {image_size}")
    kw = dict(image_size=int(image_size), scales=scales, batch_size=batch_size, num_workers=num_workers,
              rgb_mean=rgb_mean, rgb_std=rgb_std, device=device)
    qboxes = [query_box(b, s) for b, s in zip(dataset.q_bbx, dataset.q_sizes)]
    db = extract_descriptors(model, dataset.db_sizes, None, dataset.load_db, **kw)
    qs = extract_descriptors(model, dataset.q_sizes, qboxes, dataset.load_query, **kw)
    out = rank_queries(qs["desc"], db["desc"], dataset.easy, dataset.hard, dataset.junk, top=100 if save_ranks else 0)
    ap, pk, n_ok = out["ap"].cpu().numpy(), out["pk"].cpu().numpy(), out["n_ok"].cpu().numpy()
    res = summarize(ap, pk, n_ok)
    res.update({"n_queries": len(dataset.q_sizes), "n_database": len(dataset.db_sizes),
                "protocol": {"dataset": dataset.name, "image_size": int(image_size), "scales": scales,
                             "patch_size": int(model.patch_size), "descriptor": "class token, multi-scale sum"}})
    if save_ranks:
        top = out["top"].cpu().numpy()
        res["ranks"] = {str(dataset.q_names[q]): {"ap": {name: (float(ap[q, p]) if n_ok[q, p] else None)
                                                         for p, name in enumerate(PROTOCOLS)},
                                                  "top": top[q].tolist()} for q in range(len(dataset.q_sizes))}
    return res


class _Inputs:
    """The images of each planned batch, decoded in DataLoader workers."""

    def __init__(self, load, plan):
        self.load, self.plan = load, plan

    def __len__(self):
        return len(self.plan)

    def __getitem__(self, b):
        return [self.load(i) for _, i, _, _ in self.plan[b]]


def _identity(item):
    return item
