"""Linear monocular-depth probe of a frozen backbone: DINOv3's second dense linear probe (NYUv2 depth), with this
project's own statement of the protocol, modelled on DINOv2 / DINOv3's linear depth head.

Features are the patch tokens of the last `n_last_blocks` blocks with the final norm applied
(`get_intermediate_layers(x, n=n)`); with `use_cls_token` each block's class token is appended to every patch row of
its image.  A row is bf16 [patch_1 .. patch_n | cls_1 .. cls_n], [B * h * w, n * D * (1 + use_cls_token)], the same
bits as torch.cat of the fp32 outputs rounded to bf16.  The head is the segmentation probe's BatchNorm without affine
parameters (d3_seg_bn_stats / d3_seg_bn_apply) and a 1 x 1 convolution to `n_bins` logits z (d3_gemm_bf16, fp32 out,
bias epilogue), then "linear" bin normalisation: q_k = relu(z_k) + 0.1, depth d = sum_k q_k c_k / sum_k q_k with
c = linspace(min_depth, max_depth, n_bins).

- The loss is the scale-invariant log loss of the cell depth upsampled bilinearly (align_corners=False) to the depth
  crop, over its valid pixels (min_depth < gt <= max_depth): g = log(d_hat + 1e-3) - log(gt + 1e-3),
  L = sqrt(var(g) + 0.15 mean(g)^2) with the unbiased variance, 0 with fewer than 2 valid pixels
  (d3_depth_head_fwd_bwd, which never materialises a full-resolution depth or gradient).  No gradient-matching term.
- The update is AdamW through d3_adamw_ema with one segment, no clipping and EMA momentum 1, on the segmentation
  probe's schedule (`seg_lr`: linear warm-up, then a power-1 decay to 0).

The train transform runs on the GPU (d3_depth_crop): per image the host draws a `crop_size` = [h_c, w_c] box at
scale 1 and a horizontal flip (p = 0.5).  The image takes d3_seg_crop's arithmetic and the depth plane nearest
sampling from the same box; where the box leaves the image the image is 0 and the depth 0 (invalid).  Every draw is
made in the main process, in batch order: the sample order from `seed`, the boxes from `seed + 1`, so the result does
not depend on `num_workers`.  No rotation and no colour augmentation.

Evaluation: each val image is resized so that its shorter side is h_c and its longer side a multiple of the patch
size (`eval_size`; a 480 x 640 NYU frame at h_c = 416 becomes 416 x 560) and goes through the backbone whole.
d3_depth_predict_metrics upsamples the cell depth to the original ground-truth size, clamps it to
[min_depth, max_depth] and sums the per-image metrics over the valid pixels, inside the Eigen crop with
`eval_crop="eigen"`; `depth_metrics` averages each metric over the images.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops
from ..engine.params import SEG_DTYPE
from .knn import RGB_MEAN, RGB_STD, _device
from .linear import K_ALIGN, InfiniteBatchSampler
from .segmentation import BN_EPS, BN_MOMENTUM, ROWS_PER_COPY, eval_size, seg_lr

bf16, f32 = torch.bfloat16, torch.float32
EIGEN_CROP = (45, 471, 41, 601)          # rows [45, 471), columns [41, 601) of a 480 x 640 map
EIGEN_SIZE = (480, 640)
METRICS = ("abs_rel", "sq_rel", "rmse", "rmse_log", "log10", "a1", "a2", "a3")


def sample_depth_boxes(gen: torch.Generator, sizes, crop) -> torch.Tensor:
    """int32 [n, 6] = (H, W, top, left, flip, 0) for images of (H, W) `sizes`, in image order: per image the top and
    left of an h_c x w_c box (0 along an axis shorter than the box), then the flip, drawn from `gen` in that order."""
    hc, wc = int(crop[0]), int(crop[1])
    rows = []
    for H, W in sizes:
        H, W = int(H), int(W)
        top = int(torch.randint(0, max(H - hc, 0) + 1, (1,), generator=gen).item())
        left = int(torch.randint(0, max(W - wc, 0) + 1, (1,), generator=gen).item())
        flip = int(torch.rand(1, generator=gen).item() < 0.5)
        rows.append((H, W, top, left, flip, 0))
    return torch.tensor(rows, dtype=torch.int32).reshape(-1, 6)


def _pack_depth(batch):
    """DataLoader collate: (image, depth map) pairs of any size -> (flat uint8 images, flat fp32 depths, desc int64
    [n, 3] = (image byte offset, H, W)); image n's depths start at element desc[n, 0] / 3."""
    imgs = [np.ascontiguousarray(im, dtype=np.uint8) for im, _ in batch]
    deps = [np.ascontiguousarray(d, dtype=np.float32) for _, d in batch]
    for im, d in zip(imgs, deps):
        if im.ndim != 3 or im.shape[2] != 3 or d.shape != im.shape[:2]:
            raise ValueError(f"expected an HWC RGB uint8 image and an HW depth map, got {im.shape} and {d.shape}")
    offs = np.concatenate([[0], np.cumsum([im.size for im in imgs])[:-1]])
    desc = np.stack([offs, [im.shape[0] for im in imgs], [im.shape[1] for im in imgs]], 1).astype(np.int64)
    flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs]))
    return flat, torch.from_numpy(np.concatenate([d.reshape(-1) for d in deps])), torch.from_numpy(desc)


def write_depth_features(model, images: torch.Tensor, n: int, use_cls_token: bool, out: torch.Tensor) -> torch.Tensor:
    """out[:B * h * w, :n * D * (1 + use_cls_token)] = bf16 [patches of block L - n | ... | patches of block L - 1 |
    cls of block L - n | ... | cls of block L - 1] (final norm applied), one row per patch in (image, row, column)
    order, for the NHWC images [B, H, W, 3]; an image's class tokens repeat on each of its patch rows."""
    layers = model.get_intermediate_layers(images, n=int(n), return_class_token=True)
    B, P, D = layers[0][0].shape
    M, nD = B * P, int(n) * D
    srcs = [p.reshape(M, D) for p, _ in layers]
    for r0 in range(0, M, ROWS_PER_COPY):
        r1 = min(M, r0 + ROWS_PER_COPY)
        ops.linear_inputs([s[r0:r1] for s in srcs], out[r0:r1])
    if use_cls_token:
        cls = torch.cat([c for _, c in layers], 1)
        out[:M, nD:2 * nD].view(B, P, nD).copy_(cls[:, None, :].expand(B, P, nD))
    return out


class DepthLinearHead:
    """BatchNorm (no affine) + 1 x 1 convolution from `in_dim` channels to `n_bins` depth-bin logits, trained on `rows`
    feature rows per step (B * h * w of a train batch).

    The weight W [Cp, in_dim] starts as N(0, 0.01) from a CPU generator seeded with `seed` and the bias as 0; the bins
    are padded to Cp = a multiple of K_ALIGN rows, which stay zero.  Running statistics start at (0, 1)."""

    def __init__(self, in_dim: int, rows: int, iterations: int, *, n_bins: int = 256, min_depth: float = 0.001,
                 max_depth: float = 10.0, lr: float = 1e-3, weight_decay: float = 1e-3, warmup_iterations: int = 1500,
                 seed: int = 0, device=None):
        dev = _device(device)
        K, C = int(in_dim), int(n_bins)
        if K < 8 or K % 8:
            raise ValueError(f"in_dim {K} must be a positive multiple of 8 (bf16 GEMM rows of 16 bytes)")
        if C < 2:
            raise ValueError("n_bins must be at least 2")
        if not 0.0 <= float(min_depth) < float(max_depth):
            raise ValueError(f"need 0 <= min_depth < max_depth, got {min_depth}, {max_depth}")
        if int(rows) < 1 or int(iterations) < 1:
            raise ValueError("rows and iterations must be positive")
        self.K, self.n_bins, self.rows, self.iterations = K, C, int(rows), int(iterations)
        self.min_depth, self.max_depth = float(min_depth), float(max_depth)
        self.lr, self.weight_decay, self.warmup = float(lr), float(weight_decay), int(warmup_iterations)
        self.Cp = Cp = -(-C // K_ALIGN) * K_ALIGN
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

    def step(self, x: torch.Tensor, depths: torch.Tensor, hw, it: int) -> torch.Tensor:
        """One AdamW step on the feature rows x (bf16 [rows, in_dim], B * h * w patches in (image, row, column) order)
        against the depth crops (fp32 [B, Hc, Wc] on the device, metres) at schedule iteration `it`.  Returns the
        device fp32 [1] loss (no host sync)."""
        M, K, Cp = self.rows, self.K, self.Cp
        if x.dtype != bf16 or tuple(x.shape) != (M, K):
            raise ValueError(f"x must be bf16 [{M}, {K}], got {x.dtype} {tuple(x.shape)}")
        B = depths.shape[0]
        if B * int(hw[0]) * int(hw[1]) != M:
            raise ValueError(f"{B} depth maps of {tuple(hw)} patches do not make {M} rows")
        ops.seg_bn_stats(x, self.mean, self.var, self.running_mean, self.running_var, BN_MOMENTUM)
        ops.seg_bn_apply(x, self.mean, self.var, self.xh, BN_EPS)
        ops.gemm(self.xh[:M], self.W_bf16, self.logits_buf, bias=self.bias)
        ops.depth_head_fwd_bwd(self.logits_buf, depths, hw, self.n_bins, self.min_depth, self.max_depth, self.loss,
                               self.count, dz_bf16=self.dz, Cp=Cp)
        ops.gemm(self.dz, self.xh, self.gW, a_mn=True, b_mn=True)
        self.g_bias.zero_()
        ops.colsum_bf16(self.dz[:M], self.g_bias)
        self.steps += 1
        lr = seg_lr(self.lr, int(it), self.iterations, self.warmup)
        ops.adamw_ema(self.p, self.g, self.m, self.v, self._ema, self.W_bf16, self._ema_bf16, Cp * K, self.segs, 1, None,
                      0.0, lr, lr, self.weight_decay, self.steps, 1.0)
        return self.loss

    def logits(self, x: torch.Tensor) -> torch.Tensor:
        """fp32 [N, Cp] bin logits of bf16 feature rows [N, in_dim] with the running statistics (columns >= n_bins are
        the zero padding bins)."""
        N_ = x.shape[0]
        xh = torch.empty(N_, self.K, dtype=bf16, device=self.device)
        ops.seg_bn_apply(x, self.running_mean, self.running_var, xh, BN_EPS)
        out = torch.empty(N_, self.Cp, dtype=f32, device=self.device)
        return ops.gemm(xh, self.W_bf16, out, bias=self.bias)

    def state_dict(self) -> dict:
        """{"weight": fp32 [n_bins, in_dim], "bias": [n_bins], "running_mean", "running_var": [in_dim]} on the host."""
        C = self.n_bins
        return {"weight": self.W[:C].cpu().clone(), "bias": self.bias[:C].cpu().clone(),
                "running_mean": self.running_mean.cpu().clone(), "running_var": self.running_var.cpu().clone()}


def depth_metrics(sums) -> dict:
    """{"abs_rel", "sq_rel", "rmse", "rmse_log", "log10", "a1", "a2", "a3"}, each the mean over the images with a valid
    pixel of the per-image value, from the [n_images, 9] per-image sums of d3_depth_predict_metrics (count, |e| / t,
    e^2 / t, e^2, (ln p - ln t)^2, |log10 p - log10 t|, the a1..a3 hits)."""
    s = np.asarray(sums, dtype=np.float64).reshape(-1, 9)
    s = s[s[:, 0] > 0]
    if not len(s):
        raise ValueError("no val pixel has a valid depth")
    n = s[:, 0]
    per = {"abs_rel": s[:, 1] / n, "sq_rel": s[:, 2] / n, "rmse": np.sqrt(s[:, 3] / n),
           "rmse_log": np.sqrt(s[:, 4] / n), "log10": s[:, 5] / n, "a1": s[:, 6] / n, "a2": s[:, 7] / n,
           "a3": s[:, 8] / n}
    return {k: float(per[k].mean()) for k in METRICS}


def eigen_crop(height: int, width: int, eval_crop: str):
    """(top, bottom, left, right) of the pixels scored: the Eigen crop of a 480 x 640 map, or the whole map."""
    if eval_crop == "none":
        return 0, int(height), 0, int(width)
    if eval_crop != "eigen":
        raise ValueError(f"eval_crop must be 'eigen' or 'none', got {eval_crop!r}")
    if (int(height), int(width)) != EIGEN_SIZE:
        raise ValueError(f"eval_crop 'eigen' is defined for 480 x 640 depth maps, got {height} x {width}")
    return EIGEN_CROP


def eval_depth(model, train_dataset, val_dataset, *, n_last_blocks: int = 1, use_cls_token: bool = True,
               n_bins: int = 256, min_depth: float = 0.001, max_depth: float = 10.0, batch_size: int = 16,
               crop_size=(416, 544), iterations: int = 38400, lr: float = 1e-3, weight_decay: float = 1e-3,
               warmup_iterations: int = 1500, eval_crop: str = "eigen", num_workers: int = 8, seed: int = 0,
               rgb_mean=RGB_MEAN, rgb_std=RGB_STD, device=None, **_ignored) -> dict:
    """Train the linear depth head on `train_dataset` for `iterations` steps of `batch_size` crops, then score
    `val_dataset` (see `depth_metrics`).  Datasets yield (uint8 HWC RGB, fp32 HW depth in metres).  The extra keys of an
    `evaluation.depth` block (dataset paths, depth_scale) are accepted and ignored."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    p, B, n = int(model.patch_size), int(batch_size), int(n_last_blocks)
    hc, wc = (int(v) for v in crop_size)
    if hc % p or wc % p or hc < p or wc < p:
        raise ValueError(f"crop_size {[hc, wc]} must be positive multiples of the patch size {p}")
    eigen_crop(*EIGEN_SIZE, eval_crop)                 # reject an unknown eval_crop before training
    h, w = hc // p, wc // p
    K = n * int(model.embed_dim) * (2 if use_cls_token else 1)
    head = DepthLinearHead(K, B * h * w, iterations, n_bins=n_bins, min_depth=min_depth, max_depth=max_depth, lr=lr,
                           weight_decay=weight_decay, warmup_iterations=warmup_iterations, seed=seed, device=dev)
    pin = dev.type == "cuda"
    loader = torch.utils.data.DataLoader(train_dataset, batch_sampler=InfiniteBatchSampler(len(train_dataset), B,
                                                                                           iterations, seed),
                                         num_workers=int(num_workers), collate_fn=_pack_depth, pin_memory=pin,
                                         persistent_workers=False)
    aug = torch.Generator().manual_seed(int(seed) + 1)
    images = torch.empty(B, hc, wc, 3, dtype=bf16, device=dev)
    depths = torch.empty(B, hc, wc, dtype=f32, device=dev)
    x = torch.empty(B * h * w, K, dtype=bf16, device=dev)
    for it, (flat, dep, desc) in enumerate(loader):
        sizes = desc[:, 1:].tolist()
        boxes = sample_depth_boxes(aug, sizes, (hc, wc))
        ops.depth_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True), boxes.to(dev), images,
                       max_taps=ops.seg_max_taps(sizes, sizes), depths=dep.to(dev, non_blocking=True),
                       depth_out=depths, mean=rgb_mean, std=rgb_std)
        write_depth_features(model, images, n, use_cls_token, x)
        head.step(x, depths, (h, w), it)
    val_loader = torch.utils.data.DataLoader(val_dataset, batch_size=1, shuffle=False, num_workers=int(num_workers),
                                             collate_fn=_pack_depth, pin_memory=pin, persistent_workers=False)
    sums = torch.zeros(len(val_dataset), 9, dtype=torch.float64, device=dev)
    for i, (flat, dep, desc) in enumerate(val_loader):
        H, W = (int(v) for v in desc[0, 1:])
        rh, rw = eval_size(H, W, hc, p)
        img = torch.empty(1, rh, rw, 3, dtype=bf16, device=dev)
        ops.depth_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True),
                       torch.tensor([[rh, rw, 0, 0, 0, 0]], dtype=torch.int32, device=dev), img,
                       max_taps=ops.seg_max_taps([(H, W)], [(rh, rw)]), mean=rgb_mean, std=rgb_std)
        feats = torch.empty((rh // p) * (rw // p), K, dtype=bf16, device=dev)
        write_depth_features(model, img, n, use_cls_token, feats)
        ops.depth_predict_metrics(head.logits(feats), dep.to(dev, non_blocking=True).view(1, H, W),
                                  (rh // p, rw // p), head.n_bins, head.min_depth, head.max_depth, sums[i:i + 1],
                                  crop=eigen_crop(H, W, eval_crop))
    return depth_metrics(sums.cpu().numpy())
