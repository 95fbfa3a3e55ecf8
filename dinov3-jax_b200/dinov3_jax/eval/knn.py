"""k-NN classification of a frozen backbone's class token: the protocol of DINO, DINOv2 and DINOv3.

Features are the backbone's `x_norm_clstoken`, L2-normalised.  The bank is the train split, the queries the val split.
Each query keeps its max(nb_knn) most similar bank rows (dot product; ties to the lower bank index); for each k the
weights are softmax(sims[:k] / T), a class scores the weights of its neighbours among the first k, and the 5 best
classes (ties to the lower class index) give top-1 and top-5 accuracy.

Every step runs on the GPU through the library: the eval transform (d3_eval_resize_crop), the normalisation
(d3_knn_normalize), the similarities (d3_gemm_bf16, fp32 out, one query tile against one bank chunk at a time), the
running top-k (d3_topk_merge) and the vote (d3_knn_vote).  The neighbour lists do not depend on the chunk or tile sizes.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops

bf16, f32 = torch.bfloat16, torch.float32
ROW_ALIGN = 256                 # bank rows are padded with zeros to this multiple (whole GEMM tiles per chunk)
RGB_MEAN, RGB_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _device(device):
    if device is not None:
        return torch.device(device)
    if not torch.cuda.is_available():
        raise RuntimeError("k-NN evaluation runs on the GPU: no CUDA device")
    return torch.device("cuda", torch.cuda.current_device())


def _normalized_bf16(x: torch.Tensor, rows: int, dev) -> torch.Tensor:
    """L2-normalised bf16 copy of x [R, D] in a zeroed [rows >= R, D] buffer."""
    x = torch.as_tensor(x).to(device=dev, dtype=f32).contiguous()
    out = torch.zeros(rows, x.shape[1], dtype=bf16, device=dev)
    ops.knn_normalize(x, y_bf16=out)
    return out


class KnnClassifier:
    """A bank of L2-normalised bf16 train features and their labels, searched chunk by chunk.

    train_features [N, D] (any float dtype, CPU or GPU; D % 8 == 0), train_labels [N] in [0, num_classes).
    chunk: bank rows per similarity GEMM (rounded up to a multiple of 256); query_tile: queries per GEMM.  The fp32
    similarity buffer is query_tile x chunk (1 GiB at the defaults)."""

    def __init__(self, train_features, train_labels, num_classes: int, *, chunk: int = 65536, query_tile: int = 4096,
                 device=None):
        dev = _device(device)
        feats = torch.as_tensor(train_features)
        if feats.dim() != 2 or feats.shape[0] < 1:
            raise ValueError(f"train_features must be [N, D] with N >= 1, got {tuple(feats.shape)}")
        self.N, self.D = int(feats.shape[0]), int(feats.shape[1])
        if self.D % 8:
            raise ValueError(f"feature dimension {self.D} must be a multiple of 8 (bf16 GEMM rows of 16 bytes)")
        labels = torch.as_tensor(train_labels).reshape(-1)
        if labels.numel() != self.N:
            raise ValueError(f"{self.N} features but {labels.numel()} labels")
        self.num_classes = int(num_classes)
        if not 1 <= self.num_classes <= 32768:
            raise ValueError("num_classes must be in [1, 32768]")
        if int(labels.min()) < 0 or int(labels.max()) >= self.num_classes:
            raise ValueError(f"labels must lie in [0, {self.num_classes})")
        self.device = dev
        self.chunk = max(ROW_ALIGN, -(-int(chunk) // ROW_ALIGN) * ROW_ALIGN)
        self.query_tile = max(1, int(query_tile))
        self.bank = _normalized_bf16(feats, -(-self.N // ROW_ALIGN) * ROW_ALIGN, dev)
        self.labels = labels.to(device=dev, dtype=torch.int32).contiguous()

    def _search(self, queries, k: int):
        """(sims fp32 [Q, k], idx int32 [Q, k]) of the k most similar bank rows, sorted."""
        if not 1 <= k <= min(1024, self.N):
            raise ValueError(f"k = {k} must be in [1, min(1024, bank size {self.N})]")
        q = torch.as_tensor(queries)
        if q.dim() != 2 or q.shape[1] != self.D:
            raise ValueError(f"queries must be [Q, {self.D}], got {tuple(q.shape)}")
        Q = int(q.shape[0])
        qn = _normalized_bf16(q, Q, self.device)
        top_sim = torch.empty(Q, k, dtype=f32, device=self.device)
        top_idx = torch.empty(Q, k, dtype=torch.int32, device=self.device)
        tq = min(self.query_tile, Q)
        sims = torch.empty(tq, self.chunk, dtype=f32, device=self.device)
        rows = self.bank.shape[0]
        for q0 in range(0, Q, tq):
            nq = min(tq, Q - q0)
            for c0 in range(0, rows, self.chunk):
                cols = min(self.chunk, rows - c0)
                s = sims[:nq, :cols]
                ops.gemm(qn[q0:q0 + nq], self.bank[c0:c0 + cols], s)
                ops.topk_merge(s, top_sim[q0:q0 + nq], top_idx[q0:q0 + nq], offset=c0, valid=min(cols, self.N - c0),
                               fresh=c0 == 0)
        return top_sim, top_idx

    def search(self, queries, k: int):
        """(sims fp32 [Q, k], idx int64 [Q, k]): each query's k most similar bank rows, similarity descending, ties to the
        lower bank index."""
        s, i = self._search(queries, int(k))
        return s, i.long()

    def predict(self, queries, nb_knn=(10, 20, 100, 200), temperature: float = 0.07) -> torch.Tensor:
        """int32 [Q, len(nb_knn), 5]: the 5 best classes of the weighted vote of each k in nb_knn."""
        nb_knn = [int(k) for k in nb_knn]
        s, i = self._search(queries, max(nb_knn))
        preds = torch.empty(s.shape[0], len(nb_knn), 5, dtype=torch.int32, device=self.device)
        return ops.knn_vote(s, i, self.labels, nb_knn, float(temperature), self.num_classes, preds)

    def evaluate(self, queries, labels, nb_knn=(10, 20, 100, 200), temperature: float = 0.07) -> dict:
        """{k: {"top1": %, "top5": %}} over the queries (micro accuracy)."""
        nb_knn = [int(k) for k in nb_knn]
        preds = self.predict(queries, nb_knn, temperature)
        y = torch.as_tensor(labels).reshape(-1, 1).to(device=self.device, dtype=torch.int32)
        hit = preds == y[:, None, :]                                  # [Q, n_k, 5]
        top1 = hit[:, :, 0].double().mean(0) * 100.0
        top5 = hit.any(-1).double().mean(0) * 100.0
        return {k: {"top1": float(top1[j]), "top5": float(top5[j])} for j, k in enumerate(nb_knn)}


def _pack(batch):
    """DataLoader collate: images of any size -> (flat uint8, desc int64 [n, 3] = (offset, H, W), labels int64)."""
    imgs = [np.ascontiguousarray(im, dtype=np.uint8) for im, _ in batch]
    for im in imgs:
        if im.ndim != 3 or im.shape[2] != 3:
            raise ValueError(f"expected HWC RGB uint8 images, got shape {im.shape}")
    sizes = np.array([im.size for im in imgs], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    desc = np.stack([offs, [im.shape[0] for im in imgs], [im.shape[1] for im in imgs]], 1).astype(np.int64)
    flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs]))
    return flat, torch.from_numpy(desc), torch.tensor([int(t) for _, t in batch], dtype=torch.int64)


def extract_features(model, dataset, *, batch_size: int = 256, num_workers: int = 8, resize_size: int = 256,
                     crop_size: int = 224, rgb_mean=RGB_MEAN, rgb_std=RGB_STD, device=None):
    """(normalised fp32 features [N, D], labels int64 [N]) on the GPU: every image goes through the eval transform
    (d3_eval_resize_crop) and `model(x)` (the class token of a DinoVisionTransformer), batch by batch, the last batch
    possibly partial."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    loader = torch.utils.data.DataLoader(dataset, batch_size=int(batch_size), shuffle=False, drop_last=False,
                                         num_workers=int(num_workers), collate_fn=_pack,
                                         pin_memory=dev.type == "cuda", persistent_workers=False)
    feats, labels, n0 = None, torch.empty(len(dataset), dtype=torch.int64, device=dev), 0
    for flat, desc, y in loader:
        n = desc.shape[0]
        sizes = [(int(h), int(w)) for h, w in desc[:, 1:].tolist()]
        x = torch.empty(n, crop_size, crop_size, 3, dtype=bf16, device=dev)
        ops.eval_resize_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True), x, resize=resize_size,
                             max_taps=ops.eval_max_taps(sizes, resize_size), mean=rgb_mean, std=rgb_std)
        cls = model(x)
        if feats is None:
            feats = torch.empty(len(dataset), cls.shape[1], dtype=f32, device=dev)
        ops.knn_normalize(cls, y_f32=feats[n0:n0 + n])
        labels[n0:n0 + n] = y.to(dev)
        n0 += n
    if feats is None:
        raise ValueError("empty dataset")
    return feats, labels


def eval_knn(model, train_dataset, val_dataset, *, nb_knn=(10, 20, 100, 200), temperature: float = 0.07,
             batch_size: int = 256, resize_size: int = 256, crop_size: int = 224, num_workers: int = 8,
             rgb_mean=RGB_MEAN, rgb_std=RGB_STD, num_classes: int | None = None, chunk: int = 65536,
             query_tile: int = 4096, **_ignored) -> dict:
    """k-NN top-1 / top-5 accuracy (percent) of `model`'s class token, per k: {k: {"top1", "top5"}}.  The extra keys
    of an `evaluation.knn` config block (dataset paths) are accepted and ignored."""
    kw = dict(batch_size=batch_size, num_workers=num_workers, resize_size=resize_size, crop_size=crop_size,
              rgb_mean=rgb_mean, rgb_std=rgb_std)
    train_f, train_y = extract_features(model, train_dataset, **kw)
    val_f, val_y = extract_features(model, val_dataset, **kw)
    if num_classes is None:
        num_classes = int(max(int(train_y.max()), int(val_y.max()))) + 1
    nb_knn = [int(k) for k in nb_knn]
    if max(nb_knn) > train_f.shape[0]:
        raise ValueError(f"nb_knn up to {max(nb_knn)} needs at least that many train images, got {train_f.shape[0]}")
    clf = KnnClassifier(train_f, train_y, num_classes, chunk=chunk, query_tile=query_tile, device=train_f.device)
    return clf.evaluate(val_f, val_y, nb_knn, temperature)
