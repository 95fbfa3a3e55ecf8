"""Linear semantic-segmentation probe of a frozen backbone: the number DINOv3 leads with for its dense features (ADE20K
mIoU), with this project's own statement of the protocol.

Features are the patch tokens of the last `n_last_blocks` blocks with the final norm applied
(`get_intermediate_layers(x, n=n)`), concatenated along channels into one bf16 row per patch, [B * h * w, n * D]
(d3_linear_inputs, the same bits as `out_dtype=bf16`).  The head is BatchNorm without affine parameters (the 1 x 1
convolution absorbs them) followed by a 1 x 1 convolution, i.e. a GEMM of [B * h * w, n * D] by [n * D, Cp] plus a bias:

- BatchNorm uses the batch statistics over the B * h * w rows in training and updates running statistics with
  momentum 0.1 (d3_seg_bn_stats, fixed-order column sums through slab_combine); evaluation uses the running statistics.
  x_hat is written in bf16 once (d3_seg_bn_apply).
- The logits are d3_gemm_bf16 (fp32 out, bias epilogue), the loss the mean over the batch's valid pixels of the
  cross-entropy of the logits upsampled bilinearly (align_corners=False) to the label crop, label 255 ignored
  (d3_seg_xent_fwd_bwd, which never materialises full-resolution logits or their gradient).  The backbone is frozen,
  so the only gradients are dW = dZ^T . x_hat (d3_gemm_bf16) and db = colsum(dZ) (d3_colsum_bf16).
- The update is AdamW (torch's defaults: betas (0.9, 0.999), eps 1e-8, decoupled weight decay on the weights and the
  bias) through d3_adamw_ema with one segment, no clipping, and the EMA operands left unchanged (momentum 1).  The
  learning rate is `seg_lr`: a linear warm-up over `warmup_iterations`, times a polynomial (power 1) decay to 0 over
  `iterations`.

The train transform runs on the GPU (d3_seg_crop): per image the host draws a scale in [0.5, 2.0] applied to the size
whose shorter side is `crop_size`, a `crop_size`^2 box in the resized image and a horizontal flip (p = 0.5).  The image
takes the eval transform's antialiased bicubic arithmetic and the labels nearest-neighbour sampling from the same box;
where the box leaves the resized image the pixels are 0 and the labels 255.  Every draw is made in the main process,
in batch order: the sample order from `seed`, the crop parameters from `seed + 1`, so the result does not depend on
`num_workers`.  No photometric distortion and no `cat_max_ratio`.

Evaluation: each val image is resized (the same arithmetic) so that its shorter side is `crop_size` and its longer side
a multiple of the patch size, and goes through the backbone whole (no sliding window).  d3_seg_predict_confusion
upsamples the logits bilinearly to the original label size, takes the argmax (ties to the lower class) and counts the
pixels labelled < num_classes into an int64 confusion matrix, from which `seg_metrics` gives mIoU (over the classes
with a non-empty union), mAcc and aAcc.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops
from ..engine.params import SEG_DTYPE
from .knn import RGB_MEAN, RGB_STD, _device
from .linear import K_ALIGN, InfiniteBatchSampler

bf16, f32 = torch.bfloat16, torch.float32
IGNORE_LABEL = 255
SCALE_RANGE = (0.5, 2.0)
BN_EPS, BN_MOMENTUM = 1e-5, 0.1
ROWS_PER_COPY = 65535           # d3_linear_inputs runs one grid row per feature row


def seg_lr(lr0: float, t: int, total: int, warmup: int) -> float:
    """The learning rate at iteration t (0-based): lr0 * min(1, (t + 1) / warmup) * (1 - t / total)."""
    warm = min(1.0, (t + 1) / warmup) if warmup > 0 else 1.0
    return lr0 * warm * max(0.0, 1.0 - t / total)


def sample_seg_box(gen: torch.Generator, height: int, width: int, crop: int):
    """(rh, rw, top, left, flip) for one H x W image: the resized size (a scale drawn in [0.5, 2.0] times the size whose
    shorter side is `crop`, rounded half up), then the top and left of a crop x crop box inside it (0 along an axis
    shorter than the crop), then the flip; drawn from `gen` in that order."""
    s = torch.empty(1).uniform_(SCALE_RANGE[0], SCALE_RANGE[1], generator=gen).item()
    r = crop * s / min(height, width)
    rh, rw = max(1, int(height * r + 0.5)), max(1, int(width * r + 0.5))
    top = int(torch.randint(0, max(rh - crop, 0) + 1, (1,), generator=gen).item())
    left = int(torch.randint(0, max(rw - crop, 0) + 1, (1,), generator=gen).item())
    flip = int(torch.rand(1, generator=gen).item() < 0.5)
    return rh, rw, top, left, flip


def sample_seg_boxes(gen: torch.Generator, sizes, crop: int) -> torch.Tensor:
    """int32 [n, 6] = (rh, rw, top, left, flip, 0) for images of (H, W) `sizes`, in image order."""
    rows = [sample_seg_box(gen, int(H), int(W), int(crop)) + (0,) for H, W in sizes]
    return torch.tensor(rows, dtype=torch.int32).reshape(-1, 6)


def eval_size(height: int, width: int, crop: int, patch: int):
    """(rh, rw) of the evaluation resize: the shorter side becomes `crop`, the longer side long * crop / short rounded
    to the nearest multiple of `patch` (at least one patch)."""
    short, long = min(height, width), max(height, width)
    new_long = max(patch, int(long * crop / short / patch + 0.5) * patch)
    return (crop, new_long) if height <= width else (new_long, crop)


def _pack_seg(batch):
    """DataLoader collate: (image, label map) pairs of any size -> (flat uint8 images, flat uint8 labels, desc int64
    [n, 3] = (image byte offset, H, W)); image n's labels start at desc[n, 0] / 3."""
    imgs = [np.ascontiguousarray(im, dtype=np.uint8) for im, _ in batch]
    labs = [np.ascontiguousarray(lb, dtype=np.uint8) for _, lb in batch]
    for im, lb in zip(imgs, labs):
        if im.ndim != 3 or im.shape[2] != 3 or lb.shape != im.shape[:2]:
            raise ValueError(f"expected an HWC RGB uint8 image and an HW label map, got {im.shape} and {lb.shape}")
    offs = np.concatenate([[0], np.cumsum([im.size for im in imgs])[:-1]])
    desc = np.stack([offs, [im.shape[0] for im in imgs], [im.shape[1] for im in imgs]], 1).astype(np.int64)
    flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs]))
    return flat, torch.from_numpy(np.concatenate([lb.reshape(-1) for lb in labs])), torch.from_numpy(desc)


def write_seg_features(model, images: torch.Tensor, n: int, out: torch.Tensor) -> torch.Tensor:
    """out[:B * h * w, :n * D] = bf16 [patches of block L - n | ... | patches of block L - 1] (final norm applied), one
    row per patch in (image, row, column) order, for the NHWC images [B, H, W, 3]."""
    layers = model.get_intermediate_layers(images, n=int(n))
    B, P, D = layers[0].shape
    M = B * P
    srcs = [t.reshape(M, D) for t in layers]
    for r0 in range(0, M, ROWS_PER_COPY):
        r1 = min(M, r0 + ROWS_PER_COPY)
        ops.linear_inputs([s[r0:r1] for s in srcs], out[r0:r1])
    return out


class SegLinearHead:
    """BatchNorm (no affine) + 1 x 1 convolution from `in_dim` channels to `num_classes`, trained on `rows` feature
    rows per step (B * h * w of a train batch).

    The weight W [Cp, in_dim] starts as N(0, 0.01) from a CPU generator seeded with `seed` and the bias as 0; the
    classes are padded to Cp = a multiple of 8 rows, which stay zero.  Running statistics start at (0, 1)."""

    def __init__(self, in_dim: int, num_classes: int, rows: int, iterations: int, *, lr: float = 1e-3,
                 weight_decay: float = 1e-3, warmup_iterations: int = 1500, seed: int = 0, device=None):
        dev = _device(device)
        K, C = int(in_dim), int(num_classes)
        if K < 8 or K % 8:
            raise ValueError(f"in_dim {K} must be a positive multiple of 8 (bf16 GEMM rows of 16 bytes)")
        if not 2 <= C <= 256:
            raise ValueError("num_classes must be in [2, 256]")
        if int(rows) < 1 or int(iterations) < 1:
            raise ValueError("rows and iterations must be positive")
        self.K, self.num_classes, self.rows, self.iterations = K, C, int(rows), int(iterations)
        self.lr, self.weight_decay, self.warmup = float(lr), float(weight_decay), int(warmup_iterations)
        self.Cp = Cp = -(-C // 8) * 8
        self.device = dev
        n = Cp * K + Cp
        host = torch.zeros(n)
        host[:C * K] = torch.empty(C, K).normal_(0.0, 0.01, generator=torch.Generator().manual_seed(int(seed))).reshape(-1)
        # flat [W | bias] buffers for d3_adamw_ema: parameters, gradients, moments
        self.p = host.to(dev)
        self.g, self.m, self.v = (torch.zeros(n, dtype=f32, device=dev) for _ in range(3))
        self.W, self.bias = self.p[:Cp * K].view(Cp, K), self.p[Cp * K:]
        self.gW, self.g_bias = self.g[:Cp * K].view(Cp, K), self.g[Cp * K:]
        self.W_bf16 = torch.empty(Cp, K, dtype=bf16, device=dev)
        ops.cast_f32_bf16(self.p[:Cp * K], self.W_bf16)
        # the kernel's EMA operands: at momentum 1 they keep their values, nothing reads them
        self._ema, self._ema_bf16 = torch.zeros(n, dtype=f32, device=dev), torch.zeros(Cp * K, dtype=bf16, device=dev)
        segs = np.zeros(1, dtype=SEG_DTYPE)
        segs[0] = (0, 1.0, 1.0, 0, 0)
        self.segs = torch.from_numpy(segs.view(np.uint8).copy()).to(dev)
        self.running_mean = torch.zeros(K, dtype=f32, device=dev)
        self.running_var = torch.ones(K, dtype=f32, device=dev)
        self.mean, self.var = torch.empty(K, dtype=f32, device=dev), torch.empty(K, dtype=f32, device=dev)
        Mp = -(-self.rows // K_ALIGN) * K_ALIGN            # the weight-gradient GEMM contracts over the rows
        self.xh = torch.zeros(Mp, K, dtype=bf16, device=dev)
        self.dz = torch.zeros(Mp, Cp, dtype=bf16, device=dev)
        self.logits_buf = torch.empty(self.rows, Cp, dtype=f32, device=dev)
        self.loss = torch.zeros(1, dtype=f32, device=dev)
        self.count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.steps = 0

    def step(self, x: torch.Tensor, labels: torch.Tensor, hw, it: int) -> torch.Tensor:
        """One AdamW step on the feature rows x (bf16 [rows, in_dim], B * h * w patches in (image, row, column) order)
        against the label crops (uint8 [B, Hl, Wl] on the device) at schedule iteration `it`.  Returns the device fp32
        [1] loss (no host sync)."""
        M, K, Cp = self.rows, self.K, self.Cp
        if x.dtype != bf16 or tuple(x.shape) != (M, K):
            raise ValueError(f"x must be bf16 [{M}, {K}], got {x.dtype} {tuple(x.shape)}")
        B = labels.shape[0]
        if B * int(hw[0]) * int(hw[1]) != M:
            raise ValueError(f"{B} label maps of {tuple(hw)} patches do not make {M} rows")
        ops.seg_bn_stats(x, self.mean, self.var, self.running_mean, self.running_var, BN_MOMENTUM)
        ops.seg_bn_apply(x, self.mean, self.var, self.xh, BN_EPS)
        ops.gemm(self.xh[:M], self.W_bf16, self.logits_buf, bias=self.bias)
        ops.seg_xent_fwd_bwd(self.logits_buf, labels, hw, self.num_classes, self.loss, self.count, dz_bf16=self.dz,
                             Cp=Cp)
        ops.gemm(self.dz, self.xh, self.gW, a_mn=True, b_mn=True)
        self.g_bias.zero_()
        ops.colsum_bf16(self.dz[:M], self.g_bias)
        self.steps += 1
        lr = seg_lr(self.lr, int(it), self.iterations, self.warmup)
        ops.adamw_ema(self.p, self.g, self.m, self.v, self._ema, self.W_bf16, self._ema_bf16, Cp * K, self.segs, 1, None,
                      0.0, lr, lr, self.weight_decay, self.steps, 1.0)
        return self.loss

    def logits(self, x: torch.Tensor) -> torch.Tensor:
        """fp32 [N, Cp] logits of bf16 feature rows [N, in_dim] with the running statistics (columns >= num_classes
        are the zero padding classes)."""
        N_ = x.shape[0]
        xh = torch.empty(N_, self.K, dtype=bf16, device=self.device)
        ops.seg_bn_apply(x, self.running_mean, self.running_var, xh, BN_EPS)
        out = torch.empty(N_, self.Cp, dtype=f32, device=self.device)
        return ops.gemm(xh, self.W_bf16, out, bias=self.bias)

    def state_dict(self) -> dict:
        """{"weight": fp32 [num_classes, in_dim], "bias": [num_classes], "running_mean", "running_var": [in_dim]} on
        the host."""
        C = self.num_classes
        return {"weight": self.W[:C].cpu().clone(), "bias": self.bias[:C].cpu().clone(),
                "running_mean": self.running_mean.cpu().clone(), "running_var": self.running_var.cpu().clone()}


def seg_metrics(conf) -> dict:
    """{"mIoU", "mAcc", "aAcc", "per_class_iou"} in percent from an int [C, C] confusion matrix (rows: label, columns:
    prediction).  mIoU averages the classes with a non-empty union, mAcc the classes present in the labels;
    per_class_iou is None for a class with an empty union."""
    conf = np.asarray(conf, dtype=np.int64)
    tp = np.diag(conf).astype(np.float64)
    gt, pred = conf.sum(1).astype(np.float64), conf.sum(0).astype(np.float64)
    union = gt + pred - tp
    if gt.sum() == 0:
        raise ValueError("no val pixel has a label below num_classes")
    iou = np.divide(tp, union, out=np.zeros_like(tp), where=union > 0)
    acc = np.divide(tp, gt, out=np.zeros_like(tp), where=gt > 0)
    return {"mIoU": float(100.0 * iou[union > 0].mean()), "mAcc": float(100.0 * acc[gt > 0].mean()),
            "aAcc": float(100.0 * tp.sum() / gt.sum()),
            "per_class_iou": [float(100.0 * v) if u > 0 else None for v, u in zip(iou, union)]}


def eval_segmentation(model, train_dataset, val_dataset, *, num_classes: int = 150, n_last_blocks: int = 1,
                      batch_size: int = 16, crop_size: int = 512, iterations: int = 40000, lr: float = 1e-3,
                      weight_decay: float = 1e-3, warmup_iterations: int = 1500, num_workers: int = 8, seed: int = 0,
                      rgb_mean=RGB_MEAN, rgb_std=RGB_STD, device=None, **_ignored) -> dict:
    """Train the linear segmentation head on `train_dataset` for `iterations` steps of `batch_size` crops, then score
    `val_dataset`: {"mIoU", "mAcc", "aAcc", "per_class_iou"} in percent (see `seg_metrics`).  Datasets yield (uint8
    HWC RGB, uint8 HW class ids, 255 = ignore).  The extra keys of an `evaluation.segmentation` block (dataset paths)
    are accepted and ignored."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    p, S, B, n = int(model.patch_size), int(crop_size), int(batch_size), int(n_last_blocks)
    if S % p:
        raise ValueError(f"crop_size {S} must be a multiple of the patch size {p}")
    h = w = S // p
    K = n * int(model.embed_dim)
    head = SegLinearHead(K, num_classes, B * h * w, iterations, lr=lr, weight_decay=weight_decay,
                         warmup_iterations=warmup_iterations, seed=seed, device=dev)
    pin = dev.type == "cuda"
    loader = torch.utils.data.DataLoader(train_dataset, batch_sampler=InfiniteBatchSampler(len(train_dataset), B,
                                                                                           iterations, seed),
                                         num_workers=int(num_workers), collate_fn=_pack_seg, pin_memory=pin,
                                         persistent_workers=False)
    aug = torch.Generator().manual_seed(int(seed) + 1)
    images = torch.empty(B, S, S, 3, dtype=bf16, device=dev)
    labels = torch.empty(B, S, S, dtype=torch.uint8, device=dev)
    x = torch.empty(B * h * w, K, dtype=bf16, device=dev)
    for it, (flat, lab, desc) in enumerate(loader):
        sizes = desc[:, 1:].tolist()
        boxes = sample_seg_boxes(aug, sizes, S)
        ops.seg_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True), boxes.to(dev), images,
                     max_taps=ops.seg_max_taps(sizes, boxes[:, :2].tolist()), labels=lab.to(dev, non_blocking=True),
                     label_out=labels, mean=rgb_mean, std=rgb_std)
        write_seg_features(model, images, n, x)
        head.step(x, labels, (h, w), it)
    val_loader = torch.utils.data.DataLoader(val_dataset, batch_size=1, shuffle=False, num_workers=int(num_workers),
                                             collate_fn=_pack_seg, pin_memory=pin, persistent_workers=False)
    C = head.num_classes
    conf = torch.zeros(C, C, dtype=torch.int64, device=dev)
    for flat, lab, desc in val_loader:
        H, W = (int(v) for v in desc[0, 1:])
        rh, rw = eval_size(H, W, S, p)
        img = torch.empty(1, rh, rw, 3, dtype=bf16, device=dev)
        ops.seg_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True),
                     torch.tensor([[rh, rw, 0, 0, 0, 0]], dtype=torch.int32, device=dev), img,
                     max_taps=ops.seg_max_taps([(H, W)], [(rh, rw)]), mean=rgb_mean, std=rgb_std)
        feats = torch.empty((rh // p) * (rw // p), K, dtype=bf16, device=dev)
        write_seg_features(model, img, n, feats)
        ops.seg_predict_confusion(head.logits(feats), lab.to(dev, non_blocking=True).view(1, H, W), (rh // p, rw // p),
                                  C, conf)
    return seg_metrics(conf.cpu().numpy())
