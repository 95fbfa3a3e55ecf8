"""Semi-supervised video object segmentation by label propagation: the temporal-consistency check of dense features that
needs no training, modelled on DINO's eval_video_segmentation.py and scored with the DAVIS 2017 J and F statistics.
This is the project's restatement of the protocol; defaults n_last_frames = 7, size_mask_neighborhood = 12, topk = 5,
temperature = 0.1, short_side = 480.

Frames.  Each frame is resized so that its short side is `short_side` and its long side is
floor(short_side * long / short / 64) * 64 (854 x 480 -> 832 x 480): torch's bilinear interpolation
(align_corners=False, antialias=False) of the frame in [0, 1], then the ImageNet mean / std (d3_video_resize).  The
features are the teacher's last-block normalised patch tokens (`get_intermediate_layers(x, n=1)`, class and storage
tokens dropped), each row L2-normalised in fp32 and rounded to bf16 (d3_knn_normalize).  A sequence's features are
all extracted first, in batches; the propagation does not change them.

First frame.  Its annotation is read at patch resolution by nearest-exact (PIL's NEAREST), void (255) as 0, and becomes
a one-hot map over C = K + 1 channels, K the largest object id of frame 0.

Propagating to frame t.  The context is frame 0 (its one-hot map) and the soft maps of the last `n_last_frames`
propagated frames, oldest first, kept at patch resolution and not normalised.  The similarities of frame t's rows to the
context rows are d3_gemm_bf16 products with fp32 results.  For each target patch q, every context patch within
`size_mask_neighborhood` rows and columns of q, in every context frame, is a candidate with weight
a = exp(<f_q, f_s> / temperature); the candidates whose a is at least the k-th largest are kept (ties at the threshold
all kept; all of them when there are fewer than k), their weights normalised to sum 1, and q's soft label is the
weighted sum of their label rows (d3_video_propagate).  The label map at the annotation size: the soft map upsampled by
the patch size (bilinear, align_corners=False), each channel min-max normalised over the upsampled frame unless its
maximum is <= 0, the argmax over channels (lowest index on ties), resized by nearest-exact (d3_video_label_map).

Scores (d3_video_jf_counts, then the host).  For each object k = 1..K and each frame but the first and the last: J, the
IoU of the masks outside void (1 for an empty union), and F, the boundary F-measure: boundaries (a pixel that differs
from its right, lower or lower-right neighbour) of the masks with void cleared, matched within a disk of radius
ceil(0.008 * sqrt(H^2 + W^2)); no boundary in either mask gives P = R = 1, in the GT only P = 1, R = 0, in the
prediction only P = 0, R = 1.  Each object gets Mean, Recall (fraction > 0.5) and Decay (mean of the first of four
overlapping bins minus that of the last) for J and for F; the global scores are means over all objects of all
sequences and J&F-Mean = (J-Mean + F-Mean) / 2.
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch

from .. import ops
from .knn import RGB_MEAN, RGB_STD, _device

bf16, f32 = torch.bfloat16, torch.float32
MAX_CHANNELS = 32                     # background and up to 31 objects: d3_video_propagate's lane per channel
STAT_NAMES = ("Mean", "Recall", "Decay")


def video_size(height: int, width: int, short_side: int, patch: int):
    """(rh, rw) of the frame resize: the short side becomes `short_side`, the long side
    floor(short_side * long / short / 64) * 64; both must be multiples of the patch size."""
    short, long = min(height, width), max(height, width)
    new_long = int((short_side * long / short) // 64 * 64)
    if new_long < 64 or short_side % patch or new_long % patch:
        raise ValueError(f"a {height} x {width} frame at short side {short_side} becomes {short_side} x {new_long}, "
                         f"which is not a positive multiple of the patch size {patch}")
    return (short_side, new_long) if height <= width else (new_long, short_side)


def nearest_exact_index(out_size: int, in_size: int) -> np.ndarray:
    """Source index of each of out_size outputs under torch's nearest-exact (PIL's NEAREST), in fp32 like torch:
    min(floor((d + 0.5) * in / out), in - 1)."""
    scale = np.float32(in_size) / np.float32(out_size)
    d = np.arange(out_size, dtype=np.float32)
    return np.minimum(np.floor((d + np.float32(0.5)) * scale).astype(np.int64), in_size - 1)


def first_frame_labels(mask: np.ndarray, h: int, w: int, channels: int) -> np.ndarray:
    """fp32 [h * w, channels] one-hot rows of the annotation `mask` (uint8 [H, W]) read at h x w by nearest-exact,
    void (255) as background."""
    H, W = mask.shape
    small = mask[nearest_exact_index(h, H)][:, nearest_exact_index(w, W)].astype(np.int64)
    small[small == 255] = 0
    return np.eye(channels, dtype=np.float32)[small.reshape(-1)]


def boundary_radius(height: int, width: int) -> int:
    """The disk radius of the boundary match, ceil(0.008 * the image diagonal): 8 at 480 x 854."""
    return int(math.ceil(0.008 * math.hypot(height, width)))


def decay_bins(n: int):
    """The frame ranges of the four Decay bins over n scored frames: ids = round(linspace(1, n, 5) + 1e-10) - 1 and
    bin i = [ids[i], ids[i + 1]], neighbouring bins sharing one frame."""
    ids = (np.round(np.linspace(1, n, 5) + 1e-10) - 1).astype(np.int64)
    return [(int(ids[i]), int(ids[i + 1]) + 1) for i in range(4)]


def statistics(values) -> dict:
    """{"Mean", "Recall", "Decay"} of one object's per-frame J or F values (the DAVIS statistics)."""
    v = np.asarray(values, dtype=np.float64)
    bins = [v[a:b] for a, b in decay_bins(len(v))]
    return {"Mean": float(np.nanmean(v)), "Recall": float(np.nanmean(v > 0.5)),
            "Decay": float(np.nanmean(bins[0]) - np.nanmean(bins[3]))}


def jf_from_counts(counts) -> tuple:
    """(J, F) float64 [frames, objects] from d3_video_jf_counts' [frames, objects, 6] integer counts."""
    c = np.asarray(counts, dtype=np.int64)
    inter, union, nbp, nbg, mp, mg = (c[..., i].astype(np.float64) for i in range(6))
    with np.errstate(divide="ignore", invalid="ignore"):
        J = np.where(union == 0, 1.0, inter / union)
        P = np.where(nbp == 0, 1.0, np.where(nbg == 0, 0.0, mp / nbp))
        R = np.where(nbg == 0, 1.0, np.where(nbp == 0, 0.0, mg / nbg))
        F = np.where(P + R == 0, 0.0, 2 * P * R / (P + R))
    return J, F


def default_palette() -> list:
    """The PASCAL VOC / DAVIS colour map (768 ints), for sequences that come without a palette."""
    pal = []
    for i in range(256):
        r = g = b = 0
        c = i
        for j in range(8):
            r |= (c & 1) << (7 - j)
            g |= ((c >> 1) & 1) << (7 - j)
            b |= ((c >> 2) & 1) << (7 - j)
            c >>= 3
        pal += [r, g, b]
    return pal


def save_palette_masks(directory, masks: np.ndarray, palette) -> None:
    """masks uint8 [N, H, W] -> directory/%05d.png palette PNGs."""
    from PIL import Image
    os.makedirs(directory, exist_ok=True)
    for i, m in enumerate(masks):
        im = Image.fromarray(np.ascontiguousarray(m), mode="P")
        im.putpalette(palette)
        im.save(os.path.join(directory, f"{i:05d}.png"))


def sequence_features(model, frames: torch.Tensor, hw, batch_size: int, rgb_mean, rgb_std) -> torch.Tensor:
    """bf16 [N * h * w, D] L2-normalised last-block patch tokens of the uint8 frames [N, H, W, 3] (on the device)
    resized to hw = (rh, rw), `batch_size` frames per forward."""
    N, H, W, _ = frames.shape
    rh, rw = hw
    p, D = int(model.patch_size), int(model.embed_dim)
    P = (rh // p) * (rw // p)
    flat = frames.reshape(-1)
    feats = torch.empty(N * P, D, dtype=bf16, device=frames.device)
    for b0 in range(0, N, batch_size):
        b1 = min(N, b0 + batch_size)
        desc = torch.tensor([[i * H * W * 3, H, W] for i in range(b0, b1)], dtype=torch.int64, device=frames.device)
        x = ops.video_resize(flat, desc, torch.empty(b1 - b0, rh, rw, 3, dtype=bf16, device=frames.device),
                             mean=rgb_mean, std=rgb_std)
        patches = model.get_intermediate_layers(x, n=1)[0]
        ops.knn_normalize(patches.reshape((b1 - b0) * P, D).contiguous(), y_bf16=feats[b0 * P:b1 * P])
    return feats


def propagate_sequence(feats: torch.Tensor, first: np.ndarray, grid, n_frames: int, out_hw, *, patch: int,
                       n_last_frames: int, size_mask_neighborhood: int, topk: int, temperature: float):
    """(soft labels fp32 [N, h * w, C], label maps uint8 [N, H, W]) on the device of the features bf16 [N * h * w, D]:
    frame 0 carries `first` (the annotation, void as background), frames 1.. the propagated maps."""
    dev = feats.device
    h, w = grid
    P = h * w
    H, W = out_hw
    mask0 = first.copy()
    mask0[mask0 == 255] = 0
    C = int(mask0.max()) + 1
    labels = torch.zeros(n_frames, P, C, dtype=f32, device=dev)
    labels[0].copy_(torch.from_numpy(first_frame_labels(first, h, w, C)))
    pred = torch.empty(n_frames, H, W, dtype=torch.uint8, device=dev)
    pred[0].copy_(torch.from_numpy(mask0))
    ld = -(-P // 8) * 8                                   # 16-byte aligned fp32 similarity rows
    sim0 = torch.empty(P, ld, dtype=f32, device=dev)[:, :P]
    simr_buf = torch.empty(P, -(-max(n_last_frames, 1) * P // 8) * 8, dtype=f32, device=dev)
    for t in range(1, n_frames):
        tgt = feats[t * P:(t + 1) * P]
        ops.gemm(tgt, feats[:P], sim0)
        r0 = max(1, t - n_last_frames)
        simr = labr = None
        if t > r0:
            simr = ops.gemm(tgt, feats[r0 * P:t * P], simr_buf[:, :(t - r0) * P])
            labr = labels[r0:t].view((t - r0) * P, C)
        ops.video_propagate(sim0, simr, labels[0], labr, grid, size_mask_neighborhood, topk, temperature, labels[t])
        ops.video_label_map(labels[t], grid, patch, pred[t])
    return labels, pred


def eval_video_segmentation(model, dataset, *, n_last_frames: int = 7, size_mask_neighborhood: int = 12,
                            topk: int = 5, temperature: float = 0.1, short_side: int = 480, batch_size: int = 16,
                            num_workers: int = 4, save_masks: bool = False, output_dir=None, rgb_mean=RGB_MEAN,
                            rgb_std=RGB_STD, device=None, return_masks: bool = False, **_ignored) -> dict:
    """J and F of label propagation through `model`'s patch features over the sequences of `dataset` (items
    {"name", "frames", "masks", "palette"}, as DavisDataset).  Returns {"J&F-Mean", "J-Mean", "J-Recall", "J-Decay",
    "F-Mean", "F-Recall", "F-Decay", "sequences": {name: {"J-Mean", "F-Mean", "objects": {id: {"J-Mean", ...}}}},
    "protocol"}; with return_masks also "masks": {name: uint8 [N, H, W]}.  save_masks writes the predicted masks to
    output_dir/Annotations/480p/<name>/%05d.png with frame 0's palette.  The extra keys of an `evaluation.video` block
    (dataset_path) are accepted and ignored."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    protocol = {"n_last_frames": int(n_last_frames), "size_mask_neighborhood": int(size_mask_neighborhood),
                "topk": int(topk), "temperature": float(temperature), "short_side": int(short_side)}
    if protocol["n_last_frames"] < 0 or protocol["size_mask_neighborhood"] < 0 or not 1 <= protocol["topk"] <= 32:
        raise ValueError(f"need n_last_frames >= 0, size_mask_neighborhood >= 0 and 1 <= topk <= 32, got {protocol}")
    if save_masks and not output_dir:
        raise ValueError("save_masks needs output_dir")
    p = int(model.patch_size)
    loader = torch.utils.data.DataLoader(dataset, batch_size=None, shuffle=False, num_workers=int(num_workers),
                                         collate_fn=_identity, persistent_workers=False)
    per_seq, objects, masks_out = {}, [], {}
    for seq in loader:
        name, masks = seq["name"], np.asarray(seq["masks"], dtype=np.uint8)
        N, H, W = masks.shape
        if N < 3:
            raise ValueError(f"sequence {name}: {N} frames; J and F score frames 1 .. N - 2, so at least 3 are needed")
        K = int(np.where(masks[0] == 255, 0, masks[0]).max())
        if not 1 <= K < MAX_CHANNELS:
            raise ValueError(f"sequence {name}: frame 0 holds {K} objects; 1 to {MAX_CHANNELS - 1} are supported")
        rh, rw = video_size(H, W, protocol["short_side"], p)
        frames = torch.from_numpy(np.ascontiguousarray(seq["frames"], dtype=np.uint8)).to(dev)
        feats = sequence_features(model, frames, (rh, rw), int(batch_size), rgb_mean, rgb_std)
        del frames
        _, pred = propagate_sequence(feats, masks[0], (rh // p, rw // p), N, (H, W), patch=p,
                                     n_last_frames=protocol["n_last_frames"],
                                     size_mask_neighborhood=protocol["size_mask_neighborhood"], topk=protocol["topk"],
                                     temperature=protocol["temperature"])
        gt = torch.from_numpy(np.ascontiguousarray(masks)).to(dev)
        counts = torch.empty(N - 2, K, 6, dtype=torch.int64, device=dev)
        ops.video_jf_counts(pred[1:N - 1], gt[1:N - 1], K, boundary_radius(H, W), counts)
        J, F = jf_from_counts(counts.cpu().numpy())
        objs = {}
        for k in range(K):
            sj, sf = statistics(J[:, k]), statistics(F[:, k])
            objs[str(k + 1)] = {**{f"J-{s}": sj[s] for s in STAT_NAMES}, **{f"F-{s}": sf[s] for s in STAT_NAMES}}
            objects.append(objs[str(k + 1)])
        per_seq[name] = {"J-Mean": float(np.mean([o["J-Mean"] for o in objs.values()])),
                         "F-Mean": float(np.mean([o["F-Mean"] for o in objs.values()])), "objects": objs}
        if save_masks or return_masks:
            host = pred.cpu().numpy()
            if save_masks:
                save_palette_masks(os.path.join(str(output_dir), "Annotations", "480p", name), host,
                                   seq["palette"] or default_palette())
            if return_masks:
                masks_out[name] = host
    if not objects:
        raise ValueError("the dataset holds no sequence")
    res = {k: float(np.mean([o[k] for o in objects])) for k in
           [f"{m}-{s}" for m in ("J", "F") for s in STAT_NAMES]}
    res = {"J&F-Mean": (res["J-Mean"] + res["F-Mean"]) / 2, **res, "sequences": per_seq, "protocol": protocol}
    if return_masks:
        res["masks"] = masks_out
    return res


def _identity(item):
    return item
