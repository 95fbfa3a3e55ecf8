"""Linear-probe evaluation of a frozen backbone: the linear protocol of DINOv2's eval/linear.py, which DINOv3 keeps.

Features per image are `get_intermediate_layers(x, n=max(n_last_blocks_list), return_class_token=True)` (final norm
applied), written once per batch as one bf16 row [cls_{L-n_max} | ... | cls_{L-1} | mean(patches_{L-1})]
(d3_pool_tokens for the mean, d3_linear_inputs for the row).  One classifier per (n, avgpool, lr) of the grid reads
the column window [(n_max - n) * D, (n_max + avgpool) * D) of that row.  All classifiers train at once: the logits are
one d3_gemm_bf16 per window (fp32 out, bias epilogue, the window's classifiers stacked along N), the loss the sum of
their batch-mean cross-entropies (d3_linear_xent_fwd_bwd, dZ in bf16), the weight gradients dZ^T . X (d3_gemm_bf16),
the bias gradients d3_colsum_bf16 and the update torch's SGD(momentum=0.9) with lr * batch_size / 256 per classifier
on a cosine schedule (d3_sgd_momentum, fp32 master weights, bf16 copies for the next forward).

The train transform is RandomResizedCrop(crop, scale=(0.08, 1), ratio=(3/4, 4/3), bicubic, antialias) +
RandomHorizontalFlip(0.5) + normalisation, on the GPU (d3_train_resized_crop, torchvision's uint8-tensor arithmetic);
val images take the eval transform of the k-NN evaluation.  Every random draw is made in the main process, in batch
order, from generators seeded by `seed`: the sample order (`seed`), then per image its crop box and its flip
(`seed + 1`).  DataLoader workers only decode, so the result does not depend on `num_workers`.
"""
from __future__ import annotations

import math

import torch

from .. import ops
from .knn import RGB_MEAN, RGB_STD, _device, _pack

bf16, f32 = torch.bfloat16, torch.float32
K_ALIGN = 64            # the weight-gradient GEMMs contract over the batch: it is padded with zero rows to whole k-blocks
LEARNING_RATES = (1e-5, 2e-5, 5e-5, 1e-4, 2e-4, 5e-4, 1e-3, 2e-3, 5e-3, 1e-2, 2e-2, 5e-2, 0.1)
N_LAST_BLOCKS_LIST = (1, 4)
AVGPOOLS = (False, True)
SCALE, RATIO = (0.08, 1.0), (3.0 / 4.0, 4.0 / 3.0)
MOMENTUM = 0.9


def classifier_name(n: int, avgpool: bool, lr: float) -> str:
    return f"classifier_{n}_blocks_avgpool_{avgpool}_lr_{lr:.5f}".replace(".", "_")


def classifier_grid(n_last_blocks_list=N_LAST_BLOCKS_LIST, avgpools=AVGPOOLS, learning_rates=LEARNING_RATES):
    """[(n, avgpool, lr)] in grid order: n outermost, lr innermost."""
    return [(int(n), bool(a), float(lr)) for n in n_last_blocks_list for a in avgpools for lr in learning_rates]


def cosine_lr(lr0: float, t: int, total: int) -> float:
    """CosineAnnealingLR(T_max=total, eta_min=0) at iteration t (0-based)."""
    return lr0 * (1.0 + math.cos(math.pi * t / total)) / 2.0


def sample_crop_box(gen: torch.Generator, height: int, width: int, scale=SCALE, ratio=RATIO):
    """(top, left, h, w): torchvision's RandomResizedCrop.get_params with its draws, in its order, taken from `gen`
    instead of the global generator (10 attempts, then the centre-crop fallback)."""
    area = height * width
    log_ratio = torch.log(torch.tensor(ratio))
    for _ in range(10):
        target_area = area * torch.empty(1).uniform_(scale[0], scale[1], generator=gen).item()
        aspect_ratio = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1], generator=gen)).item()
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < w <= width and 0 < h <= height:
            i = torch.randint(0, height - h + 1, size=(1,), generator=gen).item()
            j = torch.randint(0, width - w + 1, size=(1,), generator=gen).item()
            return i, j, h, w
    in_ratio = float(width) / float(height)
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w, h = width, height
    return (height - h) // 2, (width - w) // 2, h, w


def sample_train_boxes(gen: torch.Generator, sizes) -> torch.Tensor:
    """int32 [n, 5] = (top, left, h, w, flip) for images of (H, W) `sizes`: per image its crop box, then its flip
    (torch.rand(1) < 0.5, RandomHorizontalFlip's draw), in image order."""
    rows = []
    for H, W in sizes:
        box = sample_crop_box(gen, int(H), int(W))
        rows.append(box + (int(torch.rand(1, generator=gen).item() < 0.5),))
    return torch.tensor(rows, dtype=torch.int32).reshape(-1, 5)


class InfiniteBatchSampler:
    """`iterations` batches of `batch_size` indices from successive seeded permutations of range(n)."""

    def __init__(self, n: int, batch_size: int, iterations: int, seed: int):
        if n < 1:
            raise ValueError("empty train dataset")
        self.n, self.batch_size, self.iterations, self.seed = int(n), int(batch_size), int(iterations), int(seed)

    def __len__(self):
        return self.iterations

    def __iter__(self):
        g = torch.Generator().manual_seed(self.seed)
        pending = []
        for _ in range(self.iterations):
            while len(pending) < self.batch_size:
                pending += torch.randperm(self.n, generator=g).tolist()
            yield pending[:self.batch_size]
            pending = pending[self.batch_size:]


def write_linear_inputs(model, images: torch.Tensor, n_max: int, out: torch.Tensor) -> torch.Tensor:
    """out[:B, :(n_max + 1) * D] = [cls of the last n_max blocks, in block order | mean of the last block's patch
    tokens] (bf16) for the NHWC images [B, S, S, 3]."""
    layers = model.get_intermediate_layers(images, n=n_max, return_class_token=True)
    patches = layers[-1][0]
    B, _, D = patches.shape
    mean = ops.pool_tokens(patches, torch.empty(B, 1, D, dtype=f32, device=patches.device), copy_tokens=False)
    return ops.linear_inputs([cls for _, cls in layers] + [mean.view(B, D)], out)


class LinearClassifiers:
    """The grid of linear classifiers Linear(D * (n + avgpool), num_classes), trained together on the input rows of
    `write_linear_inputs` (width (n_max + 1) * D, bf16).

    Weights start as N(0, 0.01) drawn in grid order from a CPU generator seeded with `seed`, biases as 0.  The classes
    are padded to Cp = a multiple of 8 rows per classifier; the padding rows stay zero.  `iterations` is the length of
    the cosine schedule."""

    def __init__(self, embed_dim: int, num_classes: int, batch_size: int, iterations: int, *,
                 n_last_blocks_list=N_LAST_BLOCKS_LIST, avgpools=AVGPOOLS, learning_rates=LEARNING_RATES, seed: int = 0,
                 device=None):
        dev = _device(device)
        D, C, B = int(embed_dim), int(num_classes), int(batch_size)
        if D < 8 or D % 8:
            raise ValueError(f"embed_dim {D} must be a positive multiple of 8 (bf16 GEMM rows of 16 bytes)")
        if not 2 <= C <= 32768:
            raise ValueError("num_classes must be in [2, 32768]")
        if B < 1 or int(iterations) < 1:
            raise ValueError("batch_size and iterations must be positive")
        self.grid = classifier_grid(n_last_blocks_list, avgpools, learning_rates)
        if not self.grid:
            raise ValueError("empty classifier grid")
        self.names = [classifier_name(*g) for g in self.grid]
        self.D, self.num_classes, self.batch_size, self.iterations = D, C, B, int(iterations)
        self.n_max = max(n for n, _, _ in self.grid)
        if min(n for n, _, _ in self.grid) < 1:
            raise ValueError("n_last_blocks_list entries must be >= 1")
        self.width = (self.n_max + 1) * D
        self.G, self.Cp = len(self.grid), -(-C // 8) * 8
        self.device = dev
        # classifiers reading the same input window, consecutive in grid order: (first, count, column, width)
        self.groups = []
        for g, (n, a, _) in enumerate(self.grid):
            col, w = (self.n_max - n) * D, (n + int(a)) * D
            last = self.groups[-1] if self.groups else None
            if last and last[2] == col and last[3] == w:
                self.groups[-1] = (last[0], last[1] + 1, col, w)
            else:
                self.groups.append((g, 1, col, w))
        gen = torch.Generator().manual_seed(int(seed))
        Cp = self.Cp
        self.W, self.W_bf16, self.mW, self.gW = [], [], [], []
        for _, cnt, _, w in self.groups:
            host = torch.zeros(cnt * Cp, w)
            for k in range(cnt):
                host[k * Cp:k * Cp + C] = torch.empty(C, w).normal_(0.0, 0.01, generator=gen)
            W = host.to(dev)
            Wb = torch.empty(W.shape, dtype=bf16, device=dev)
            ops.cast_f32_bf16(W, Wb)
            self.W.append(W)
            self.W_bf16.append(Wb)
            self.mW.append(torch.zeros_like(W))
            self.gW.append(torch.zeros_like(W))
        self.bias, self.m_bias, self.g_bias = (torch.zeros(self.G * Cp, dtype=f32, device=dev) for _ in range(3))
        self.lr = torch.tensor([lr * B / 256.0 for _, _, lr in self.grid], dtype=f32, device=dev)
        self.Bp = -(-B // K_ALIGN) * K_ALIGN
        self.x = torch.zeros(self.Bp, self.width, dtype=bf16, device=dev)      # rows >= batch_size stay zero
        self.dz = torch.zeros(self.Bp, self.G * Cp, dtype=bf16, device=dev)
        self.logits = torch.empty(B, self.G * Cp, dtype=f32, device=dev)
        self.loss = torch.zeros(self.G, dtype=f32, device=dev)
        self.labels = torch.empty(B, dtype=torch.int32, device=dev)
        self.steps = 0

    def _logits(self, x: torch.Tensor, out: torch.Tensor):
        Cp = self.Cp
        for (g0, cnt, col, w), Wb in zip(self.groups, self.W_bf16):
            ops.gemm(x[:, col:col + w], Wb, out[:, g0 * Cp:(g0 + cnt) * Cp], bias=self.bias[g0 * Cp:(g0 + cnt) * Cp])
        return out

    def step(self, inputs: torch.Tensor, labels, it: int) -> torch.Tensor:
        """One SGD step of every classifier on a batch of input rows (bf16 [batch_size, width]; `self.x` itself is
        taken as is) at schedule iteration `it`.  Returns the device fp32 [G] batch-mean losses (no host sync)."""
        B, Cp = self.batch_size, self.Cp
        if inputs.data_ptr() != self.x.data_ptr():
            if inputs.dtype != bf16 or tuple(inputs.shape) != (B, self.width):
                raise ValueError(f"inputs must be bf16 [{B}, {self.width}], got {inputs.dtype} {tuple(inputs.shape)}")
            self.x[:B].copy_(inputs)
        y = torch.as_tensor(labels).reshape(-1)
        if y.numel() != B:
            raise ValueError(f"{y.numel()} labels for a batch of {B}")
        self.labels.copy_(y)
        self._logits(self.x[:B], self.logits)
        ops.linear_xent_fwd_bwd(self.logits, self.labels, self.num_classes, Cp, self.loss, self.dz)
        for (g0, cnt, col, w), gW in zip(self.groups, self.gW):
            ops.gemm(self.dz[:, g0 * Cp:(g0 + cnt) * Cp], self.x[:, col:col + w], gW, a_mn=True, b_mn=True)
        self.g_bias.zero_()
        ops.colsum_bf16(self.dz[:B], self.g_bias)
        scale = cosine_lr(1.0, int(it), self.iterations)
        first = self.steps == 0
        for (g0, cnt, _, _), W, gW, mW, Wb in zip(self.groups, self.W, self.gW, self.mW, self.W_bf16):
            ops.sgd_momentum(W, gW, mW, Wb, self.lr[g0:g0 + cnt], Cp, lr_scale=scale, momentum=MOMENTUM, first=first)
        ops.sgd_momentum(self.bias, self.g_bias, self.m_bias, None, self.lr, Cp, lr_scale=scale, momentum=MOMENTUM,
                         first=first)
        self.steps += 1
        return self.loss

    def predict(self, inputs: torch.Tensor, chunk: int = 1024) -> torch.Tensor:
        """int32 [N, G, 5]: each classifier's 5 best classes per input row (logit desc, ties to the lower class; -1
        where there are fewer than 5 classes), through d3_topk_merge on every classifier's logit slice."""
        x = torch.as_tensor(inputs).to(device=self.device, dtype=bf16)
        if x.dim() != 2 or x.shape[1] != self.width:
            raise ValueError(f"inputs must be [N, {self.width}], got {tuple(x.shape)}")
        x = x.contiguous()
        N, G, Cp = x.shape[0], self.G, self.Cp
        preds = torch.empty(N, G * 5, dtype=torch.int32, device=self.device)
        t = min(int(chunk), max(N, 1))
        logits = torch.empty(t, G * Cp, dtype=f32, device=self.device)
        top_s = torch.empty(t, G * 5, dtype=f32, device=self.device)
        for r0 in range(0, N, t):
            n = min(t, N - r0)
            self._logits(x[r0:r0 + n], logits[:n])
            for g in range(G):
                ops.topk_merge(logits[:n, g * Cp:(g + 1) * Cp], top_s[:n, 5 * g:5 * g + 5],
                               preds[r0:r0 + n, 5 * g:5 * g + 5], offset=0, valid=self.num_classes, fresh=True)
        return preds.view(N, G, 5)

    def hits(self, inputs: torch.Tensor, labels) -> torch.Tensor:
        """int64 [G, 2] device counts of top-1 and top-5 hits over the rows."""
        preds = self.predict(inputs)
        y = torch.as_tensor(labels).reshape(-1, 1, 1).to(device=self.device, dtype=torch.int32)
        hit = preds == y
        return torch.stack([hit[:, :, 0].sum(0), hit.any(-1).sum(0)], 1)

    def evaluate(self, inputs: torch.Tensor, labels) -> dict:
        """{name: {"top1": %, "top5": %}} over the rows (micro accuracy)."""
        return _accuracies(self.names, self.hits(inputs, labels), int(torch.as_tensor(labels).numel()))

    def state_dict(self) -> dict:
        """{name: {"weight": fp32 [num_classes, D * (n + avgpool)], "bias": fp32 [num_classes]}} on the host."""
        out, C, Cp = {}, self.num_classes, self.Cp
        for (g0, cnt, _, _), W in zip(self.groups, self.W):
            for k in range(cnt):
                g = g0 + k
                out[self.names[g]] = {"weight": W[k * Cp:k * Cp + C].cpu().clone(),
                                      "bias": self.bias[g * Cp:g * Cp + C].cpu().clone()}
        return out


def _accuracies(names, hits: torch.Tensor, total: int) -> dict:
    h = hits.double().cpu() * (100.0 / max(total, 1))
    return {name: {"top1": float(h[g, 0]), "top5": float(h[g, 1])} for g, name in enumerate(names)}


def _num_classes(*datasets) -> int:
    targets = [t for ds in datasets for t in getattr(ds, "targets", [])]
    if not targets:
        raise ValueError("num_classes is needed for datasets without `targets`")
    return int(max(targets)) + 1


def eval_linear(model, train_dataset, val_dataset, *, epochs: int = 10, epoch_length: int = 1250, batch_size: int = 128,
                learning_rates=LEARNING_RATES, n_last_blocks_list=N_LAST_BLOCKS_LIST, avgpools=AVGPOOLS,
                crop_size: int = 224, resize_size: int = 256, num_workers: int = 8, seed: int = 0, rgb_mean=RGB_MEAN,
                rgb_std=RGB_STD, num_classes: int | None = None, device=None, **_ignored) -> dict:
    """Linear-probe top-1 / top-5 accuracy (percent) of `model` (a DinoVisionTransformer): {name: {"top1", "top5"}} per
    classifier and "best_classifier": {"name", "top1", "top5"} (the best val top-1, ties to the first in grid order).
    The extra keys of an `evaluation.linear` config block (dataset paths) are accepted and ignored."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    if num_classes is None:
        num_classes = _num_classes(train_dataset, val_dataset)
    iterations = int(epochs) * int(epoch_length)
    B, S = int(batch_size), int(crop_size)
    clf = LinearClassifiers(model.embed_dim, num_classes, B, iterations, n_last_blocks_list=n_last_blocks_list,
                            avgpools=avgpools, learning_rates=learning_rates, seed=seed, device=dev)
    pin = dev.type == "cuda"
    sampler = InfiniteBatchSampler(len(train_dataset), B, iterations, seed)
    loader = torch.utils.data.DataLoader(train_dataset, batch_sampler=sampler, num_workers=int(num_workers),
                                         collate_fn=_pack, pin_memory=pin, persistent_workers=False)
    aug = torch.Generator().manual_seed(int(seed) + 1)
    images = torch.empty(B, S, S, 3, dtype=bf16, device=dev)
    for it, (flat, desc, y) in enumerate(loader):
        boxes = sample_train_boxes(aug, desc[:, 1:].tolist())
        ops.train_resized_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True), boxes.to(dev), images,
                               max_taps=ops.train_max_taps(boxes.tolist(), S), mean=rgb_mean, std=rgb_std)
        write_linear_inputs(model, images, clf.n_max, clf.x)
        clf.step(clf.x, y, it)
    val_loader = torch.utils.data.DataLoader(val_dataset, batch_size=B, shuffle=False, drop_last=False,
                                             num_workers=int(num_workers), collate_fn=_pack, pin_memory=pin,
                                             persistent_workers=False)
    hits, total = torch.zeros(clf.G, 2, dtype=torch.int64, device=dev), 0
    feats = torch.empty(B, clf.width, dtype=bf16, device=dev)
    for flat, desc, y in val_loader:
        n = desc.shape[0]
        ops.eval_resize_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True), images[:n],
                             resize=int(resize_size), max_taps=ops.eval_max_taps(desc[:, 1:].tolist(), int(resize_size)),
                             mean=rgb_mean, std=rgb_std)
        write_linear_inputs(model, images[:n], clf.n_max, feats)
        hits += clf.hits(feats[:n], y)
        total += n
    if total == 0:
        raise ValueError("empty val dataset")
    results = _accuracies(clf.names, hits, total)
    best = clf.names[0]
    for name in clf.names[1:]:
        if results[name]["top1"] > results[best]["top1"]:
            best = name
    results["best_classifier"] = {"name": best, **results[best]}
    return results
