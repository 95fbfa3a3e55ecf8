"""Labelled image datasets for evaluation.  Each item is (uint8 HWC RGB numpy array, int label); images keep their own
sizes, the eval transform runs on the GPU (`ops.eval_resize_crop`).  Decoding is host plumbing in DataLoader workers."""
from __future__ import annotations

import os

import numpy as np

IMG_EXTENSIONS = (".jpg", ".jpeg", ".png", ".ppm", ".bmp", ".pgm", ".tif", ".tiff", ".webp")


class ImageFolder:
    """root/<class>/**/<image>: classes are the sorted subdirectory names (label = position), files are sorted, like
    torchvision.datasets.ImageFolder.  Images are decoded with PIL and converted to RGB."""

    def __init__(self, root):
        self.root = str(root)
        self.classes = sorted(e.name for e in os.scandir(self.root) if e.is_dir())
        if not self.classes:
            raise FileNotFoundError(f"no class directories under {self.root}")
        self.class_to_idx = {c: i for i, c in enumerate(self.classes)}
        self.samples = []
        for c in self.classes:
            for d, _, files in sorted(os.walk(os.path.join(self.root, c), followlinks=True)):
                self.samples += [(os.path.join(d, f), self.class_to_idx[c]) for f in sorted(files)
                                 if f.lower().endswith(IMG_EXTENSIONS)]
        self.targets = [t for _, t in self.samples]

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        from PIL import Image
        path, target = self.samples[i]
        with Image.open(path) as im:
            return np.asarray(im.convert("RGB"), dtype=np.uint8), target


class NpzDataset:
    """An .npz file with `images` (uint8 [N, H, W, 3]) and `labels` (integers [N])."""

    def __init__(self, path):
        with np.load(path, allow_pickle=False) as z:
            self.images = np.asarray(z["images"])
            self.targets = [int(v) for v in np.asarray(z["labels"]).reshape(-1)]
        if self.images.dtype != np.uint8 or self.images.ndim != 4 or self.images.shape[-1] != 3:
            raise ValueError(f"{path}: images must be uint8 [N, H, W, 3], got {self.images.dtype} {self.images.shape}")
        if len(self.targets) != len(self.images):
            raise ValueError(f"{path}: {len(self.images)} images but {len(self.targets)} labels")
        self.classes = sorted(set(self.targets))

    def __len__(self):
        return len(self.targets)

    def __getitem__(self, i):
        return self.images[i], self.targets[i]


def make_eval_dataset(path):
    """An .npz file -> NpzDataset, a directory -> ImageFolder."""
    path = str(path)
    return NpzDataset(path) if path.endswith(".npz") else ImageFolder(path)
