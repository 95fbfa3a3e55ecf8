"""Pretraining on real images: `train.dataset_path=gpu:<dataset>` reads image files, decodes them on the host and crops
and augments them on the GPU, each image at its own size.

Dataset strings (after the `gpu:` prefix):

  ImageNet:split=TRAIN|VAL:root=R[:extra=...]   R/train/<wnid>/*.JPEG, or R/val/<wnid>/* for VAL; `extra` is accepted
                                                 and ignored, so the reference's ImageNet string works after the prefix
  ImageFolder:root=R                             every image file under R, recursively (labels are not needed: SSL
                                                 ignores them)

Files are listed sorted by directory, then by file name.  DataLoader workers (`train.num_workers`) decode each file
with `PIL.Image.open(path).convert("RGB")` (no EXIF transpose) and pack the B images of a batch into one uint8 buffer
plus their sizes; workers never touch CUDA.  The main process copies that buffer to the GPU on a copy stream (the copy
of batch i + 1 runs under step i), draws the augmentation parameters from each image's own size, runs the ragged
augmentation kernels (data/gpu_augment.py) and adds the iBOT masks.

The image indices of iteration i (`SeededBatchSampler`) and every crop, flip, jitter, blur and solarize parameter of
iteration i are functions of (train.seed, rank, world, i) alone: they do not depend on num_workers or on what this
process ran before, so a resumed run sees the crops the uninterrupted run saw.  The iBOT masks come from the host
`random` / `numpy.random` streams like the reference's collate, and are not resume-exact."""
from __future__ import annotations

import os

import numpy as np
import torch

IMG_EXTENSIONS = (".jpg", ".jpeg", ".png", ".ppm", ".bmp", ".pgm", ".tif", ".tiff", ".webp")
PREFIX = "gpu:"


def list_images(root) -> list:
    """Every file under root (recursively, following links) with an image extension: sorted by directory, then by
    file name."""
    out = []
    for d, _, files in sorted(os.walk(str(root), followlinks=True)):
        out += [os.path.join(d, f) for f in sorted(files) if f.lower().endswith(IMG_EXTENSIONS)]
    return out


def decode_rgb(path) -> np.ndarray:
    """PIL.Image.open(path).convert("RGB") as uint8 [H, W, 3] (torchvision's pil_loader; no EXIF transpose).  A file
    that cannot be decoded raises an error that names it."""
    from PIL import Image
    try:
        with Image.open(path) as im:
            return np.asarray(im.convert("RGB"), dtype=np.uint8)
    except Exception as e:
        raise OSError(f"cannot decode image {path}: {e}") from e


def _imagenet_files(root: str, split: str) -> list:
    d = os.path.join(root, split.lower())
    if not os.path.isdir(d):
        raise FileNotFoundError(f"ImageNet root {root}: no {split.lower()}/ directory")
    out = []
    for wnid in sorted(e.name for e in os.scandir(d) if e.is_dir()):
        names = sorted(e.name for e in os.scandir(os.path.join(d, wnid)) if e.is_file() and not e.name.startswith("."))
        out += [os.path.join(d, wnid, f) for f in names if split == "VAL" or f.endswith(".JPEG")]
    return out


_KEYS = {"ImageNet": ("split", "root", "extra"), "ImageFolder": ("root",)}


def parse_dataset_path(path: str) -> tuple:
    """`gpu:<name>:key=value:...` -> (name, {key: value}).  Unknown names or keys raise ValueError."""
    if not path.startswith(PREFIX):
        raise ValueError(f"{path!r}: not a {PREFIX} dataset string")
    name, *fields = path[len(PREFIX):].split(":")
    if name not in _KEYS:
        raise ValueError(f"{path!r}: unknown dataset {name!r} (known: {', '.join(_KEYS)})")
    kw = {}
    for f in fields:
        k, sep, v = f.partition("=")
        if not sep or k not in _KEYS[name]:
            raise ValueError(f"{path!r}: unknown key {f!r} for {name} (keys: {', '.join(_KEYS[name])})")
        kw[k] = v
    if "root" not in kw:
        raise ValueError(f"{path!r}: {name} needs root=<directory>")
    if name == "ImageNet" and kw.get("split") not in ("TRAIN", "VAL"):
        raise ValueError(f"{path!r}: ImageNet needs split=TRAIN or split=VAL")
    return name, kw


def dataset_files(path: str) -> list:
    """The sorted image files a `gpu:` dataset string names.  A missing root, or one without images, raises
    FileNotFoundError naming it."""
    name, kw = parse_dataset_path(path)
    root = kw["root"]
    if not os.path.isdir(root):
        raise FileNotFoundError(f"dataset root {root} does not exist")
    files = _imagenet_files(root, kw["split"]) if name == "ImageNet" else list_images(root)
    if not files:
        raise FileNotFoundError(f"dataset root {root} holds no images")
    return files


class ImageFiles(torch.utils.data.Dataset):
    """Item i: (i, the decoded uint8 [H, W, 3] image of files[i])."""

    def __init__(self, files):
        self.files = list(files)

    def __len__(self):
        return len(self.files)

    def __getitem__(self, i):
        return i, decode_rgb(self.files[i])


def pack_images(samples) -> dict:
    """Worker-side collate: B (index, [H, W, 3] uint8) samples -> one packed uint8 buffer of their HWC pixels, their
    sizes [B, 2] and their indices [B]."""
    pixels = torch.from_numpy(np.concatenate([np.ascontiguousarray(im).reshape(-1) for _, im in samples]))
    return {"indices": torch.tensor([i for i, _ in samples], dtype=torch.int64),
            "sizes": torch.tensor([im.shape[:2] for _, im in samples], dtype=torch.int64).reshape(-1, 2),
            "pixels": pixels}


def _shutdown(it) -> None:
    stop = getattr(it, "_shutdown_workers", None)            # joins the worker processes now, not at garbage collection
    if stop is not None:
        stop()


class GpuImageLoader:
    """The `gpu:` training loader: iterating it yields the batch dicts `Engine.set_batch` consumes, from
    `start_iter` on.  `close()` (or the end of a `with` block) shuts the DataLoader workers down."""

    def __init__(self, config, start_iter: int = 0, rank: int = 0, world: int = 1, device=None):
        from .gpu_augment import GpuBatchPipeline
        from .synthetic import SeededBatchSampler
        self.files = dataset_files(str(config.train.dataset_path))
        self.B = int(config.train.batch_size_per_gpu)
        self.seed, self.rank, self.world, self.start_iter = int(config.train.seed), int(rank), int(world), int(start_iter)
        self.num_workers = int(config.train.get("num_workers", 0))
        if len(self.files) // self.world < self.B:
            raise ValueError(f"{config.train.dataset_path}: {len(self.files)} images give rank {self.rank} of "
                             f"{self.world} fewer than one batch of {self.B}")
        self.sampler = SeededBatchSampler(len(self.files), self.B, seed=self.seed, rank=self.rank, world=self.world,
                                          advance=self.start_iter * self.B)
        self.pipe = GpuBatchPipeline(config, seed=self.seed)
        self.device = device
        self._gens = []

    def rng(self, iteration: int) -> np.random.Generator:
        """The augmentation parameters' generator of `iteration`: a function of (seed, rank, world, iteration) only."""
        return np.random.default_rng([self.seed, self.rank, self.world, int(iteration)])

    def draw(self, iteration: int, sizes):
        """The crop records and blur sigmas of `iteration` for images of `sizes` [B, 2] (what the augmentation draws)."""
        aug = self.pipe.aug
        aug.rng = self.rng(iteration)
        sizes = np.asarray(sizes).reshape(-1, 2)
        src = aug.sample_source_jitter(len(sizes)) if aug.share_color_jitter else None
        return src, aug.sample(len(sizes), sizes[:, 0], sizes[:, 1])

    def host_batches(self):
        """The packed host batches from `start_iter` on (pinned when CUDA is available); closing the generator shuts
        the workers down."""
        dl = torch.utils.data.DataLoader(ImageFiles(self.files), batch_sampler=self.sampler, num_workers=self.num_workers,
                                         collate_fn=pack_images, pin_memory=torch.cuda.is_available())
        it = iter(dl)
        try:
            yield from it
        finally:
            _shutdown(it)

    def __iter__(self):
        from .gpu_augment import RaggedImages
        dev = torch.device(self.device if self.device is not None else
                           f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}")
        copy_stream = torch.cuda.Stream(device=dev)

        def upload(host):
            with torch.cuda.stream(copy_stream):
                pixels = host["pixels"].to(dev, non_blocking=True)
            return host, pixels, copy_stream.record_event()

        def batches():
            hosts = self.host_batches()
            self._gens.append(hosts)
            try:
                nxt = upload(next(hosts))
                for it in range(self.start_iter, 1 << 62):
                    host, pixels, ready = nxt
                    stream = torch.cuda.current_stream(dev)
                    stream.wait_event(ready)
                    pixels.record_stream(stream)
                    self.pipe.aug.rng = self.rng(it)
                    batch = self.pipe(RaggedImages(pixels, host["sizes"].numpy()))
                    nxt = upload(next(hosts))          # batch it + 1's copy overlaps step it
                    yield batch
            finally:
                hosts.close()

        gen = batches()
        self._gens.append(gen)
        return gen

    def close(self) -> None:
        """Shut down every iterator's workers (idempotent)."""
        for g in self._gens:
            g.close()
        self._gens = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
