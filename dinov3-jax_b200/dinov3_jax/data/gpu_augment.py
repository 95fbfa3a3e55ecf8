"""On-GPU DINO multi-crop augmentation and batch assembly (SURVEY §8f.3): the step before the training hot path.

`GpuDataAugmentationDINO` has the constructor of the reference's `DataAugmentationDINO`
(dinov3_jax/data/augmentations.py:23-56) but works on a whole BATCH of decoded uint8 images that already sit in HBM
([B, H, W, 3]) and returns the collated crop tensors of `collate_data_and_cast` (data/collate.py:72-93: crop-major NHWC
in `param_dtype`) directly — no per-sample PIL objects, no host loop over pixels.  Only the random PARAMETERS are drawn
on the host (a few dozen scalars per image, numpy), following torchvision's sampling rules:

  RandomResizedCrop.get_params   10 attempts of area ~ U(scale) * H * W, log-ratio ~ U(log 3/4, log 4/3), integer box,
                                 centre-crop fallback; interpolation bicubic with antialias (what PIL does when it shrinks)
  RandomHorizontalFlip           p = 0.5 (0 when horizontal_flips is false)
  ColorJitter(0.4, 0.4, 0.2, 0.1) applied with p = 0.8, ops in a random order; RandomGrayscale p = 0.2
  GaussianBlur(kernel 9, sigma ~ U(0.1, 2))  — the reference wraps it as RandomApply(p = 1 - p_arg)
                                 (data/transforms.py:30-33), so the blur probabilities AS CODED are 0.0 / 0.9 / 0.5 for
                                 global crop 1 / global crop 2 / local crops; that is what is followed here
  RandomSolarize(threshold 128)  p = 0.2, second global crop only
  ToTensor + Normalize(mean, std)

The other options of the reference constructor follow data/augmentations.py:70-230:

  gram_teacher_crops_size        the global "base" crops are taken at max(global, gram) and resized (bicubic,
                                 antialias) to both sizes; with gram_teacher_no_distortions the global crop is resized
                                 before its distortions and the gram crop is the undistorted base, otherwise both are
                                 resized from the distorted base.  Batch key `collated_gram_teacher_crops`, crop-major.
  local_crops_subset_of_global_crops
                                 local crop c is a local x local window of base crop 1 (c < n/2) or 2, at offsets
                                 randint(0, (global - local) // patch) * patch, after the local jitter and blur of the
                                 WHOLE base; it inherits the base's flip
  share_color_jitter             one ColorJitter + RandomGrayscale per source image, before any crop; no per-crop jitter
  teacher_no_color_jitter        only fills `global_crops_teacher`, which the collate never reads: no effect on the batch

A batch is either a dense [B, H, W, 3] uint8 tensor or a `RaggedImages`: B images of their own sizes packed into one
buffer, as a real dataset decodes them.  Each image's crop boxes are drawn from its own size, and the first crop reads
it in place (csrc/augment.cu: a dense batch is a ragged batch of equal sizes); everything after that first crop works
on dense crops.

The kernels (csrc/augment.cu) are deterministic functions of those parameters and are tested against torchvision's
float implementations.  `GpuBatchPipeline` adds the iBOT block masks (host `MaskingGenerator`, as in the reference's
collate) and yields the batch dict `Engine.set_batch` consumes.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from .. import _native as N
from .collate import collate_masks
from .masking import MaskingGenerator

CROP_DTYPE = np.dtype([("img", "<i4"), ("x0", "<i4"), ("y0", "<i4"), ("w", "<i4"), ("h", "<i4"), ("flip", "<i4"),
                       ("order", "<i4", (4,)), ("fb", "<f4"), ("fc", "<f4"), ("fs", "<f4"), ("fh", "<f4"),
                       ("gray", "<i4"), ("solarize", "<i4")])
assert CROP_DTYPE.itemsize == 64
IMAGE_DTYPE = np.dtype([("off", "<i8"), ("h", "<i4"), ("w", "<i4")])      # one row of a ragged batch's image table
assert IMAGE_DTYPE.itemsize == 16

IMAGENET_DEFAULT_MEAN = (0.485, 0.456, 0.406)
IMAGENET_DEFAULT_STD = (0.229, 0.224, 0.225)


def _resized_crop_params(rng, H, W, scale, ratio=(3.0 / 4.0, 4.0 / 3.0)):
    """torchvision RandomResizedCrop.get_params -> (y0, x0, h, w)."""
    area = H * W
    log_ratio = (math.log(ratio[0]), math.log(ratio[1]))
    for _ in range(10):
        target = area * rng.uniform(scale[0], scale[1])
        ar = math.exp(rng.uniform(log_ratio[0], log_ratio[1]))
        w = int(round(math.sqrt(target * ar)))
        h = int(round(math.sqrt(target / ar)))
        if 0 < w <= W and 0 < h <= H:
            return int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w
    in_ratio = W / H
    if in_ratio < ratio[0]:
        w, h = W, int(round(W / ratio[0]))
    elif in_ratio > ratio[1]:
        h, w = H, int(round(H * ratio[1]))
    else:
        w, h = W, H
    return (H - h) // 2, (W - w) // 2, h, w


class RaggedImages:
    """B images of their own sizes: `data` is one 1-D buffer holding each image's HWC pixels in turn (uint8, or fp32 in
    [0, 1]), `sizes` their (H, W).  `table` is the image table the kernels read, with each image's first pixel."""

    def __init__(self, data: torch.Tensor, sizes):
        self.data = data
        self.sizes = np.asarray(sizes, dtype=np.int64).reshape(-1, 2)
        assert (self.sizes > 0).all(), "every image needs at least one pixel"
        pix = self.sizes[:, 0] * self.sizes[:, 1]
        self.table = np.zeros(len(self.sizes), dtype=IMAGE_DTYPE)
        self.table["off"][1:] = np.cumsum(pix)[:-1]
        self.table["h"], self.table["w"] = self.sizes[:, 0], self.sizes[:, 1]
        self.n_pix = int(pix.sum())
        assert data.dim() == 1 and data.numel() == 3 * self.n_pix, (tuple(data.shape), self.n_pix)
        self._d_table = None

    @classmethod
    def from_images(cls, images, device=None) -> "RaggedImages":
        """Pack a list of [H, W, 3] tensors or arrays (one dtype) into one buffer on `device`."""
        ts = [torch.as_tensor(im) for im in images]
        data = torch.cat([t.reshape(-1) for t in ts])
        return cls(data if device is None else data.to(device), [t.shape[:2] for t in ts])

    def __len__(self):
        return len(self.sizes)

    def with_data(self, data: torch.Tensor) -> "RaggedImages":
        """The same images' layout over another buffer (the fp32 jittered copy of share_color_jitter)."""
        out = RaggedImages(data, self.sizes)
        out._d_table = self._d_table if data.device == self.device else None
        return out

    @property
    def device(self):
        return self.data.device

    def image(self, i: int) -> torch.Tensor:
        """Image i as an [H, W, 3] view of the buffer."""
        o, (h, w) = int(self.table["off"][i]), self.sizes[i]
        return self.data[3 * o:3 * (o + h * w)].view(int(h), int(w), 3)

    def d_table(self) -> torch.Tensor:
        if self._d_table is None:
            self._d_table = torch.from_numpy(self.table.view(np.uint8).reshape(-1).copy()).to(self.device, non_blocking=True)
        return self._d_table


class GpuDataAugmentationDINO:
    def __init__(self, global_crops_scale, local_crops_scale, local_crops_number, global_crops_size=224,
                 local_crops_size=96, gram_teacher_crops_size=None, gram_teacher_no_distortions=False,
                 teacher_no_color_jitter=False, local_crops_subset_of_global_crops=False, patch_size=16,
                 share_color_jitter=False, horizontal_flips=True, mean=IMAGENET_DEFAULT_MEAN, std=IMAGENET_DEFAULT_STD,
                 seed: int = 0, out_dtype=torch.bfloat16):
        assert out_dtype == torch.bfloat16, "the kernels emit bf16 (compute_precision.param_dtype: bf16)"
        if isinstance(gram_teacher_crops_size, (list, tuple)):
            raise NotImplementedError("a list of gram_teacher_crops_size values (multi-resolution crops): build one "
                                      "augmentation per resolution")
        self.global_scale, self.local_scale = tuple(global_crops_scale), tuple(local_crops_scale)
        self.n_local, self.gs, self.ls = int(local_crops_number), int(global_crops_size), int(local_crops_size)
        if local_crops_subset_of_global_crops:
            if self.n_local % 2:
                raise ValueError(f"local_crops_subset_of_global_crops needs an even local_crops_number, got {self.n_local} "
                                 "(half of the local crops come from each global crop)")
            if (self.gs - self.ls) // patch_size < 1:
                raise ValueError(f"local_crops_subset_of_global_crops: (global_crops_size - local_crops_size) // patch_size "
                                 f"= ({self.gs} - {self.ls}) // {patch_size} leaves no offset to draw")
        self.gram = None if gram_teacher_crops_size is None else int(gram_teacher_crops_size)
        self.gram_no_distortions = bool(gram_teacher_no_distortions)
        self.subset, self.patch = bool(local_crops_subset_of_global_crops), int(patch_size)
        self.share_color_jitter = bool(share_color_jitter)
        self.base_size = max(self.gs, self.gram or 0)    # augmentations.py:73: global and gram crops come from one base
        self.flip_p = 0.5 if horizontal_flips else 0.0
        self.mean = (C.c_float * 3)(*[float(v) for v in mean])
        self.std = (C.c_float * 3)(*[float(v) for v in std])
        self.rng = np.random.default_rng(seed)
        self._scratch = {}

    # ---- host: random parameters ----------------------------------------------------------------------------------
    def _color(self, rec, i):
        """RandomApply([ColorJitter], p=0.8) + RandomGrayscale(p=0.2) into record i."""
        rng = self.rng
        if rng.random() < 0.8:
            rec["order"][i] = rng.permutation(4)
            rec["fb"][i], rec["fc"][i] = rng.uniform(0.6, 1.4), rng.uniform(0.6, 1.4)
            rec["fs"][i], rec["fh"][i] = rng.uniform(0.8, 1.2), rng.uniform(-0.1, 0.1)
        else:
            rec["order"][i] = -1
        rec["gray"][i] = int(rng.random() < 0.2)

    def sample(self, B: int, H, W):
        """Crop records (crop-major: crop index outer, image inner, like the collate's stacking) and blur sigmas for the
        2 global and n_local local crop sets.  The global records' boxes are the base crops at `base_size`.  With
        local_crops_subset_of_global_crops a local record is a window: img = its base crop's row in the global records,
        (y0, x0) = (rx, ry), w = h = local size, no flip of its own.  H and W are the images' sizes: one int for the
        whole batch, or one per image; each image's boxes are drawn from its own size, with the same draws either way."""
        rng = self.rng
        Hs, Ws = (np.broadcast_to(np.asarray(v, dtype=np.int64), (B,)) for v in (H, W))
        g = np.zeros(2 * B, dtype=CROP_DTYPE)
        l = np.zeros(self.n_local * B, dtype=CROP_DTYPE)
        gb = np.zeros(2 * B, dtype=np.float32)
        lb = np.zeros(self.n_local * B, dtype=np.float32)

        def fill(rec, i, img, scale, blur_apply_p, solarize_p, sig):
            y0, x0, h, w = _resized_crop_params(rng, int(Hs[img]), int(Ws[img]), scale)
            rec["img"][i], rec["x0"][i], rec["y0"][i], rec["w"][i], rec["h"][i] = img, x0, y0, w, h
            rec["flip"][i] = int(rng.random() < self.flip_p)
            if self.share_color_jitter:
                rec["order"][i] = -1                            # the source image was jittered instead
            else:
                self._color(rec, i)
            sig[i] = rng.uniform(0.1, 2.0) if rng.random() < blur_apply_p else 0.0
            rec["solarize"][i] = int(rng.random() < solarize_p)

        def fill_window(i, base):
            l["img"][i], l["w"][i], l["h"][i] = base, self.ls, self.ls
            if self.share_color_jitter:
                l["order"][i] = -1
            else:
                self._color(l, i)
            lb[i] = rng.uniform(0.1, 2.0) if rng.random() < 0.5 else 0.0
            l["y0"][i], l["x0"][i] = rng.integers(0, (self.gs - self.ls) // self.patch, 2) * self.patch   # rx (row), ry

        for b in range(B):
            # reference GaussianBlur(p=...) applies the blur with probability 1 - p (data/transforms.py:30-33)
            fill(g, 0 * B + b, b, self.global_scale, 1.0 - 1.0, 0.0, gb)          # global_transfo1: GaussianBlur(p=1.0)
            fill(g, 1 * B + b, b, self.global_scale, 1.0 - 0.1, 0.2, gb)          # global_transfo2: GaussianBlur(p=0.1), Solarize(0.2)
            for c in range(self.n_local):
                if self.subset:                                 # crops 0 .. n/2-1 from base 1, the rest from base 2
                    fill_window(c * B + b, (0 if c < self.n_local // 2 else 1) * B + b)
                else:
                    fill(l, c * B + b, b, self.local_scale, 1.0 - 0.5, 0.0, lb)   # local_transfo: GaussianBlur(p=0.5)
        return (g, gb), (l, lb)

    def sample_source_jitter(self, B: int) -> np.ndarray:
        """share_color_jitter: one ColorJitter + RandomGrayscale record per source image (img = b)."""
        s = np.zeros(B, dtype=CROP_DTYPE)
        s["img"] = np.arange(B)
        for b in range(B):
            self._color(s, b)
        return s

    # ---- device: kernels ----------------------------------------------------------------------------------------------
    def _buf(self, key, shape, dtype, device):
        t = self._scratch.get(key)
        if t is None or t.shape != tuple(shape) or t.device != device:
            t = torch.empty(shape, dtype=dtype, device=device)
            self._scratch[key] = t
        return t

    @staticmethod
    def _dev(records: np.ndarray, dev):
        return torch.from_numpy(records.view(np.uint8).reshape(-1).copy()).to(dev, non_blocking=True)

    def _crop(self, src, crops: np.ndarray, d_crops, S: int, key, clamp: bool = True) -> torch.Tensor:
        """[n, S, S, 3] fp32 resized crops of src (uint8 images, or fp32 [0,1] images; dense or RaggedImages) by the
        host records `crops`, whose device copy is d_crops."""
        lib = N.init()
        n = crops.shape[0]
        x = self._buf((key, S), (n, S, S, 3), torch.float32, src.device)
        if isinstance(src, RaggedImages):
            hw = src.sizes[crops["img"]]
            assert ((crops["img"] >= 0) & (crops["img"] < len(src))).all()
            assert ((crops["x0"] >= 0) & (crops["y0"] >= 0) & (crops["w"] > 0) & (crops["h"] > 0)
                    & (crops["x0"] + crops["w"] <= hw[:, 1]) & (crops["y0"] + crops["h"] <= hw[:, 0])).all(), \
                "a crop box reaches outside its image"
            h_crops = crops.ctypes.data_as(C.c_void_p)
            if src.data.dtype == torch.uint8:
                N.check(lib.d3_aug_resized_crop_ragged(N.ptr(src.data), N.ptr(src.d_table()), len(src), N.ptr(d_crops),
                                                       h_crops, n, N.ptr(x), S, N.stream_ptr()), "d3_aug_resized_crop_ragged")
            else:
                N.check(lib.d3_aug_resized_crop_ragged_f32(N.ptr(src.data), N.ptr(src.d_table()), len(src), N.ptr(d_crops),
                                                           h_crops, n, N.ptr(x), S, int(clamp), N.stream_ptr()),
                        "d3_aug_resized_crop_ragged_f32")
            return x
        B, H, W, _ = src.shape
        if src.dtype == torch.uint8:
            N.check(lib.d3_aug_resized_crop(N.ptr(src), B, H, W, N.ptr(d_crops), n, N.ptr(x), S, N.stream_ptr()),
                    "d3_aug_resized_crop")
        else:
            N.check(lib.d3_aug_resized_crop_f32(N.ptr(src), B, H, W, N.ptr(d_crops), n, N.ptr(x), S, int(clamp),
                                                N.stream_ptr()), "d3_aug_resized_crop_f32")
        return x

    def _resize(self, x: torch.Tensor, S: int, key, clamp: bool) -> torch.Tensor:
        """Resize(S, bicubic) of every [M, M] image of x; the identity when M == S."""
        n, M = x.shape[0], x.shape[1]
        if M == S:
            return x
        whole = self._whole(n, M)
        return self._crop(x, whole, self._dev(whole, x.device), S, key, clamp)

    @staticmethod
    def _whole(n: int, M: int) -> np.ndarray:
        """Records of the whole [M, M] image i with no flip, jitter, grayscale or solarize."""
        r = np.zeros(n, dtype=CROP_DTYPE)
        r["img"], r["w"], r["h"], r["order"] = np.arange(n), M, M, -1
        return r

    def _finish(self, x: torch.Tensor, d_crops) -> torch.Tensor:
        n, S = x.shape[0], x.shape[1]
        out = torch.empty(n, S, S, 3, dtype=torch.bfloat16, device=x.device)
        N.check(N.init().d3_aug_finish(N.ptr(x), N.ptr(out), N.ptr(d_crops), n, S, self.mean, self.std, N.stream_ptr()),
                "d3_aug_finish")
        return out

    def _distort(self, x: torch.Tensor, d_crops, sigmas: np.ndarray, finish: bool = True) -> torch.Tensor:
        """ColorJitter + RandomGrayscale (in place on x), GaussianBlur, then Solarize + Normalize -> bf16 when `finish`;
        otherwise the blurred fp32 crops."""
        lib = N.init()
        n, S = x.shape[0], x.shape[1]
        dev = x.device
        d_sig = torch.from_numpy(sigmas.astype(np.float32)).to(dev, non_blocking=True)
        t1 = self._buf(("t1", S), (n, S, S, 3), torch.float32, dev)
        t2 = self._buf(("t2", S), (n, S, S, 3), torch.float32, dev)
        gsum = torch.zeros(n, dtype=torch.float32, device=dev)
        s = N.stream_ptr()
        N.check(lib.d3_aug_color(N.ptr(x), N.ptr(d_crops), n, S, N.ptr(gsum), s), "d3_aug_color")
        N.check(lib.d3_aug_blur(N.ptr(x), N.ptr(t1), N.ptr(t2), N.ptr(d_sig), n, S, s), "d3_aug_blur")
        return self._finish(t2, d_crops) if finish else t2

    def apply(self, images_u8, crops: np.ndarray, sigmas: np.ndarray, S: int) -> torch.Tensor:
        """images_u8 [B,H,W,3] uint8 on the GPU, or a RaggedImages (or the fp32 jittered sources of
        share_color_jitter); returns [n_crops, S, S, 3] bf16 (normalised)."""
        data = images_u8.data if isinstance(images_u8, RaggedImages) else images_u8
        assert data.dtype in (torch.uint8, torch.float32) and data.is_cuda and data.is_contiguous()
        assert isinstance(images_u8, RaggedImages) or images_u8.shape[-1] == 3
        d_crops = self._dev(crops, data.device)
        return self._distort(self._crop(images_u8, crops, d_crops, S, "x"), d_crops, sigmas)

    def jitter_sources(self, images_u8, recs: np.ndarray):
        """share_color_jitter: fp32 copy of the sources, each jittered with its record: [B,H,W,3] for a dense batch, a
        RaggedImages with the same layout for a ragged one (contrast takes each image's own mean gray)."""
        dev = images_u8.device
        d_recs = self._dev(recs, dev)
        if isinstance(images_u8, RaggedImages):
            B = len(images_u8)
            n = 3 * images_u8.n_pix                             # one buffer that grows to the largest batch seen
            if self._scratch.get("src_ragged") is None or self._scratch["src_ragged"].numel() < n:
                self._scratch["src_ragged"] = torch.empty(n, dtype=torch.float32, device=dev)
            x = self._scratch["src_ragged"][:n]
            gsum = torch.zeros(B, dtype=torch.float32, device=dev)
            N.check(N.init().d3_aug_color_images_ragged(N.ptr(images_u8.data), images_u8.n_pix, N.ptr(images_u8.d_table()),
                                                        B, N.ptr(d_recs), recs.ctypes.data_as(C.c_void_p), N.ptr(x),
                                                        N.ptr(gsum), N.stream_ptr()), "d3_aug_color_images_ragged")
            return images_u8.with_data(x)
        B, H, W, _ = images_u8.shape
        x = self._buf(("src", H, W), (B, H, W, 3), torch.float32, dev)
        gsum = torch.zeros(B, dtype=torch.float32, device=dev)
        N.check(N.init().d3_aug_color_images(N.ptr(images_u8), B, H, W, N.ptr(d_recs), N.ptr(x), N.ptr(gsum),
                                             N.stream_ptr()), "d3_aug_color_images")
        return x

    def local_windows(self, base: torch.Tensor, crops: np.ndarray, sigmas: np.ndarray) -> torch.Tensor:
        """local_crops_subset_of_global_crops: [n_crops, L, L, 3] bf16 windows of the fp32 base crops [n_base, M, M, 3],
        each cut after its own jitter and blur of the whole base."""
        n_base, M = base.shape[0], base.shape[1]
        n, L = crops.shape[0], self.ls
        assert (crops["img"] < n_base).all() and (crops["x0"] + L <= M).all() and (crops["y0"] + L <= M).all()
        dev = base.device
        d_crops = self._dev(crops, dev)
        d_sig = torch.from_numpy(sigmas.astype(np.float32)).to(dev, non_blocking=True)
        win = self._buf(("win", L), (n, L + 8, L + 8, 3), torch.float32, dev)
        tmp = self._buf(("wtmp", L), (n, L + 8, L, 3), torch.float32, dev)
        y = self._buf(("wy", L), (n, L, L, 3), torch.float32, dev)
        gsum = torch.zeros(n, dtype=torch.float32, device=dev)
        N.check(N.init().d3_aug_local_windows(N.ptr(base), n_base, M, N.ptr(d_crops), N.ptr(d_sig), n, L, N.ptr(win),
                                              N.ptr(tmp), N.ptr(y), N.ptr(gsum), N.stream_ptr()), "d3_aug_local_windows")
        return self._finish(y, d_crops)

    def __call__(self, images_u8) -> dict:
        """images_u8: a dense [B, H, W, 3] uint8 tensor on the GPU, or a RaggedImages of uint8 images there."""
        if isinstance(images_u8, RaggedImages):
            B, H, W = len(images_u8), images_u8.sizes[:, 0], images_u8.sizes[:, 1]
        else:
            B, H, W, _ = images_u8.shape
        src = images_u8
        if self.share_color_jitter:
            src = self.jitter_sources(images_u8, self.sample_source_jitter(B))
        (g, gb), (l, lb) = self.sample(B, H, W)
        if self.gram is None and not self.subset:
            return {"collated_global_crops": self.apply(src, g, gb, self.gs),
                    "collated_local_crops": self.apply(src, l, lb, self.ls)}
        # base crops at max(global, gram); what reads the undistorted base runs before the jitter works in place on it
        dev = images_u8.device
        d_g = self._dev(g, dev)
        base = self._crop(src, g, d_g, self.base_size, "base")
        out = {"collated_local_crops": self.local_windows(base, l, lb) if self.subset else self.apply(src, l, lb, self.ls)}
        if self.gram is None:
            out["collated_global_crops"] = self._distort(base, d_g, gb)
        elif self.gram_no_distortions:                        # augmentations.py:98-101, :200-201
            d_whole = self._dev(self._whole(2 * B, self.base_size), dev)
            out["collated_gram_teacher_crops"] = self._finish(self._resize(base, self.gram, "gram", True), d_whole)
            out["collated_global_crops"] = self._distort(self._resize(base, self.gs, "x", True), d_g, gb)
        else:                                                 # :105-108, :202-204: resize the distorted, normalised base
            y = self._distort(base, d_g, gb, finish=False)
            N.check(N.init().d3_aug_solarize(N.ptr(y), N.ptr(d_g), 2 * B, self.base_size, N.stream_ptr()), "d3_aug_solarize")
            d_whole = self._dev(self._whole(2 * B, self.base_size), dev)
            out["collated_global_crops"] = self._finish(self._resize(y, self.gs, "x", False), d_whole)
            out["collated_gram_teacher_crops"] = self._finish(self._resize(y, self.gram, "gram", False), d_whole)
        return out


class GpuBatchPipeline:
    """uint8 image batch on the GPU (dense or ragged) -> the batch dict of data/collate.py:72-93 (crops from the kernels above, iBOT block
    masks from the reference's host generator as in its collate).  `config` is the reference-shaped config."""

    def __init__(self, config, seed: int = 0):
        c = config.crops
        self.aug = GpuDataAugmentationDINO(c.global_crops_scale, c.local_crops_scale, c.local_crops_number,
                                           global_crops_size=c.global_crops_size, local_crops_size=c.local_crops_size,
                                           gram_teacher_crops_size=c.get("gram_teacher_crops_size", None),
                                           gram_teacher_no_distortions=c.get("gram_teacher_no_distortions", False),
                                           local_crops_subset_of_global_crops=c.get("localcrops_subset_of_globalcrops", False),
                                           share_color_jitter=c.get("share_color_jitter", False),
                                           horizontal_flips=c.get("horizontal_flips", True),
                                           mean=c.get("rgb_mean", IMAGENET_DEFAULT_MEAN), std=c.get("rgb_std", IMAGENET_DEFAULT_STD),
                                           patch_size=config.student.patch_size, seed=seed)
        grid = c.global_crops_size // config.student.patch_size
        self.n_tokens = grid * grid
        self.mask_generator = MaskingGenerator(input_size=(grid, grid),
                                               max_num_patches=0.5 * c.global_crops_size // config.student.patch_size
                                               * c.global_crops_size // config.student.patch_size)
        self.mask_ratio = tuple(config.ibot.mask_ratio_min_max)
        self.mask_probability = config.ibot.mask_sample_probability
        self.circular = bool(config.ibot.get("mask_random_circular_shift", False))

    def __call__(self, images_u8) -> dict:
        """images_u8: a dense [B, H, W, 3] uint8 tensor on the GPU, or a RaggedImages of uint8 images there."""
        out = self.aug(images_u8)
        n_global = out["collated_global_crops"].shape[0]
        out.update(collate_masks(n_global, self.n_tokens, self.mask_ratio, self.mask_probability, self.mask_generator,
                                 self.circular))
        out["global_batch_size"] = len(images_u8)
        return out
