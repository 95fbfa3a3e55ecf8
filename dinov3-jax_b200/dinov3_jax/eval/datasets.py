"""Labelled image datasets for evaluation.  Each item is (uint8 HWC RGB numpy array, int label), for segmentation
(uint8 HWC RGB, uint8 HW label map), or for depth (uint8 HWC RGB, fp32 HW depth in metres); a video dataset yields
whole sequences (`DavisDataset`), a correspondence dataset keypoint pairs over its images (`SPairDataset`), a
discovery dataset images with their object boxes (`VOCDiscoveryDataset`), a retrieval dataset database and query
images with per-query ground-truth lists (`RevisitedDataset`), a video classification dataset the frames of labelled
videos (`VideoClassListDataset`).  Images
keep their own sizes, the transforms run on the GPU (`ops.eval_resize_crop`, `ops.seg_crop`, `ops.depth_crop`,
`ops.video_resize`).  Decoding is host plumbing in DataLoader workers."""
from __future__ import annotations

import os
import pickle

import numpy as np

from ..data.image_loader import IMG_EXTENSIONS, decode_rgb, list_images


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
            self.samples += [(p, self.class_to_idx[c]) for p in list_images(os.path.join(self.root, c))]
        self.targets = [t for _, t in self.samples]

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        path, target = self.samples[i]
        return decode_rgb(path), target


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


IGNORE_LABEL = 255


def reduce_zero_label(label: np.ndarray) -> np.ndarray:
    """ADE20K's label convention: 0 (other) becomes 255 (ignored) and every other value v becomes v - 1 (255 stays)."""
    label = np.asarray(label, dtype=np.uint8)
    return np.where((label == 0) | (label == IGNORE_LABEL), IGNORE_LABEL, label.astype(np.int16) - 1).astype(np.uint8)


class ADE20KSegmentation:
    """ADE20K SceneParsing (150 classes) in the layout of the reference's data/datasets/ade20k.py: the file names of
    `split` ("train" or "val") come from root/ADE20K_object150_<split>.txt, sorted; image `name` is root/images/<name>
    and its label map root/annotations/<name without extension>.png.  Items are (uint8 HWC RGB, uint8 HW class ids,
    255 = ignore) after `reduce_zero_label`."""

    def __init__(self, root, split: str = "train"):
        if split not in ("train", "val"):
            raise ValueError(f"split must be 'train' or 'val', got {split!r}")
        self.root, self.split = str(root), split
        with open(os.path.join(self.root, f"ADE20K_object150_{split}.txt")) as f:
            names = sorted(line.strip() for line in f.read().strip().split("\n") if line.strip())
        self.images = [os.path.join(self.root, "images", n) for n in names]
        self.labels = [os.path.join(self.root, "annotations", os.path.splitext(n)[0] + ".png") for n in names]

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        from PIL import Image
        with Image.open(self.images[i]) as im:
            img = np.asarray(im.convert("RGB"), dtype=np.uint8)
        with Image.open(self.labels[i]) as lb:
            label = reduce_zero_label(np.asarray(lb))
        if label.shape != img.shape[:2]:
            raise ValueError(f"{self.labels[i]}: label {label.shape} does not match image {img.shape[:2]}")
        return img, label


class SegNpzDataset:
    """An .npz file with `images` (uint8 [N, H, W, 3]) and `labels` (uint8 [N, H, W], class ids, 255 = ignore)."""

    def __init__(self, path):
        with np.load(path, allow_pickle=False) as z:
            self.images = np.asarray(z["images"])
            self.labels = np.asarray(z["labels"])
        if self.images.dtype != np.uint8 or self.images.ndim != 4 or self.images.shape[-1] != 3:
            raise ValueError(f"{path}: images must be uint8 [N, H, W, 3], got {self.images.dtype} {self.images.shape}")
        if self.labels.dtype != np.uint8 or self.labels.shape != self.images.shape[:3]:
            raise ValueError(f"{path}: labels must be uint8 {list(self.images.shape[:3])}, got {self.labels.dtype} "
                             f"{list(self.labels.shape)}")

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return self.images[i], self.labels[i]


def make_seg_dataset(path, split: str = "train"):
    """An .npz file -> SegNpzDataset, a directory -> ADE20KSegmentation(path, split)."""
    path = str(path)
    return SegNpzDataset(path) if path.endswith(".npz") else ADE20KSegmentation(path, split)


class DepthNpzDataset:
    """An .npz file with `images` (uint8 [N, H, W, 3]) and `depths` (float32 [N, H, W], metres; values outside
    (min_depth, max_depth] are not scored)."""

    def __init__(self, path):
        with np.load(path, allow_pickle=False) as z:
            self.images = np.asarray(z["images"])
            self.depths = np.asarray(z["depths"])
        if self.images.dtype != np.uint8 or self.images.ndim != 4 or self.images.shape[-1] != 3:
            raise ValueError(f"{path}: images must be uint8 [N, H, W, 3], got {self.images.dtype} {self.images.shape}")
        if self.depths.dtype != np.float32 or self.depths.shape != self.images.shape[:3]:
            raise ValueError(f"{path}: depths must be float32 {list(self.images.shape[:3])}, got {self.depths.dtype} "
                             f"{list(self.depths.shape)}")

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return self.images[i], self.depths[i]


class DepthListDataset:
    """root/<split>.txt lists one `rgb_path depth_path` pair per line, relative to root (the NYU Depth v2 layout);
    pairs are sorted by rgb path.  The depth is a 16-bit PNG holding metres * depth_scale (default 1000: millimetres);
    0 means no measurement."""

    def __init__(self, root, split: str = "train", depth_scale: float = 1000.0):
        if split not in ("train", "val"):
            raise ValueError(f"split must be 'train' or 'val', got {split!r}")
        if not float(depth_scale) > 0:
            raise ValueError(f"depth_scale must be positive, got {depth_scale}")
        self.root, self.split, self.depth_scale = str(root), split, float(depth_scale)
        pairs = []
        with open(os.path.join(self.root, f"{split}.txt")) as f:
            for n, line in enumerate(f, 1):
                if not line.strip():
                    continue
                parts = line.split()
                if len(parts) != 2:
                    raise ValueError(f"{split}.txt line {n}: expected 'rgb_path depth_path', got {line.strip()!r}")
                pairs.append(tuple(os.path.join(self.root, p) for p in parts))
        pairs.sort()
        for paths in pairs:
            for q in paths:
                if not os.path.isfile(q):
                    raise FileNotFoundError(f"{split}.txt names {q}, which does not exist")
        self.images, self.depth_files = [a for a, _ in pairs], [b for _, b in pairs]

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        from PIL import Image
        with Image.open(self.images[i]) as im:
            img = np.asarray(im.convert("RGB"), dtype=np.uint8)
        with Image.open(self.depth_files[i]) as dp:
            raw = np.asarray(dp)
        if raw.dtype not in (np.uint16, np.int32) or raw.ndim != 2:
            raise ValueError(f"{self.depth_files[i]}: expected a 16-bit single-channel PNG, got {raw.dtype} {raw.shape}")
        if raw.shape != img.shape[:2]:
            raise ValueError(f"{self.depth_files[i]}: depth {raw.shape} does not match image {img.shape[:2]}")
        return img, (raw.astype(np.float64) / self.depth_scale).astype(np.float32)


def make_depth_dataset(path, split: str = "train", depth_scale: float = 1000.0):
    """An .npz file -> DepthNpzDataset, a directory -> DepthListDataset(path, split, depth_scale)."""
    path = str(path)
    return DepthNpzDataset(path) if path.endswith(".npz") else DepthListDataset(path, split, depth_scale)


class DavisDataset:
    """The DAVIS 2017 semi-supervised layout: root/ImageSets/2017/<split>.txt lists the sequences;
    root/JPEGImages/480p/<seq>/*.jpg are the frames and root/Annotations/480p/<seq>/*.png the palette annotations, one
    per frame, both sorted by name.  Item i is {"name", "frames" uint8 [N, H, W, 3], "masks" uint8 [N, H, W] (object ids,
    255 void), "palette" (frame 0's, a list of 768 ints)}."""

    def __init__(self, root, split: str = "val"):
        self.root, self.split = str(root), split
        lst = os.path.join(self.root, "ImageSets", "2017", f"{split}.txt")
        if not os.path.isfile(lst):
            raise FileNotFoundError(f"{lst} does not exist")
        with open(lst) as f:
            self.sequences = [line.strip() for line in f if line.strip()]
        self.frames, self.annotations = [], []
        for seq in self.sequences:
            fd = os.path.join(self.root, "JPEGImages", "480p", seq)
            ad = os.path.join(self.root, "Annotations", "480p", seq)
            for d in (fd, ad):
                if not os.path.isdir(d):
                    raise FileNotFoundError(f"{split}.txt names sequence {seq}, but {d} does not exist")
            frames = sorted(os.path.join(fd, e) for e in os.listdir(fd) if e.lower().endswith(".jpg"))
            annots = sorted(os.path.join(ad, e) for e in os.listdir(ad) if e.lower().endswith(".png"))
            if not frames or len(frames) != len(annots):
                raise ValueError(f"{fd} holds {len(frames)} frames but {ad} holds {len(annots)} annotations")
            self.frames.append(frames)
            self.annotations.append(annots)

    def __len__(self):
        return len(self.sequences)

    def __getitem__(self, i):
        from PIL import Image
        frames, masks, palette = [], [], None
        for fp, ap in zip(self.frames[i], self.annotations[i]):
            with Image.open(fp) as im:
                frames.append(np.asarray(im.convert("RGB"), dtype=np.uint8))
            with Image.open(ap) as an:
                if an.mode != "P":
                    raise ValueError(f"{ap}: expected a palette PNG, got mode {an.mode}")
                if palette is None:
                    palette = an.getpalette()
                masks.append(np.asarray(an, dtype=np.uint8))
            if masks[-1].shape != frames[-1].shape[:2] or frames[-1].shape != frames[0].shape:
                raise ValueError(f"{ap}: annotation {masks[-1].shape} does not match frame {frames[-1].shape[:2]} "
                                 f"(frame 0 {frames[0].shape[:2]})")
        return {"name": self.sequences[i], "frames": np.stack(frames), "masks": np.stack(masks), "palette": palette}


class VideoNpzDataset:
    """An .npz file with `frames` (uint8 [N, H, W, 3]), `masks` (uint8 [N, H, W], object ids, 255 void) and
    `sequence_starts` (int, the first frame of each sequence, ascending from 0).  Sequence i is named "%05d" % i and
    has no palette."""

    def __init__(self, path):
        with np.load(path, allow_pickle=False) as z:
            self.frames, self.masks = np.asarray(z["frames"]), np.asarray(z["masks"])
            starts = np.asarray(z["sequence_starts"])
        if self.frames.dtype != np.uint8 or self.frames.ndim != 4 or self.frames.shape[-1] != 3:
            raise ValueError(f"{path}: frames must be uint8 [N, H, W, 3], got {self.frames.dtype} {self.frames.shape}")
        if self.masks.dtype != np.uint8 or self.masks.shape != self.frames.shape[:3]:
            raise ValueError(f"{path}: masks must be uint8 {list(self.frames.shape[:3])}, got {self.masks.dtype} "
                             f"{list(self.masks.shape)}")
        n = len(self.frames)
        if (starts.ndim != 1 or not len(starts) or starts[0] != 0 or (np.diff(starts) <= 0).any()
                or starts[-1] >= n):
            raise ValueError(f"{path}: sequence_starts must ascend from 0 and stay below {n}, got {starts.tolist()}")
        self.bounds = list(zip(starts.tolist(), starts[1:].tolist() + [n]))

    def __len__(self):
        return len(self.bounds)

    def __getitem__(self, i):
        a, b = self.bounds[i]
        return {"name": f"{i:05d}", "frames": self.frames[a:b], "masks": self.masks[a:b], "palette": None}


def make_video_dataset(path, split: str = "val"):
    """An .npz file -> VideoNpzDataset, a directory -> DavisDataset(path, split)."""
    path = str(path)
    return VideoNpzDataset(path) if path.endswith(".npz") else DavisDataset(path, split)


def _field(path, source, name):
    if name not in source:
        raise ValueError(f"{path}: field {name!r} is missing")
    return source[name]


class SPairDataset:
    """The SPair-71k layout: every root/PairAnnotation/<split>/*.json, in sorted file-name order, is one pair, read for
    src_imname, trg_imname, category, src_kps, trg_kps ([n, 2] x then y) and trg_bndbox (x1 y1 x2 y2); the images are
    root/JPEGImages/<category>/<imname>.  `pairs[i]` is {"src", "trg" (image indices), "category", "src_kps",
    "trg_kps" (float64 [n, 2]), "trg_bbox" (4 floats)}; `load_image(j)` decodes image j to uint8 HWC RGB.  Errors name
    the file and the field."""

    def __init__(self, root, split: str = "test"):
        import json
        self.root, self.split = str(root), split
        d = os.path.join(self.root, "PairAnnotation", split)
        if not os.path.isdir(d):
            raise FileNotFoundError(f"{d} does not exist")
        files = sorted(e for e in os.listdir(d) if e.endswith(".json"))
        if not files:
            raise FileNotFoundError(f"{d} holds no pair annotation (*.json)")
        self.images, index, self.pairs = [], {}, []
        for name in files:
            path = os.path.join(d, name)
            with open(path) as f:
                a = json.load(f)
            cat = str(_field(path, a, "category"))
            ims = []
            for key in ("src_imname", "trg_imname"):
                im = os.path.join(self.root, "JPEGImages", cat, str(_field(path, a, key)))
                if im not in index:
                    if not os.path.isfile(im):
                        raise FileNotFoundError(f"{path}: {key} names {im}, which does not exist")
                    index[im] = len(self.images)
                    self.images.append(im)
                ims.append(index[im])
            kps = []
            for key in ("src_kps", "trg_kps"):
                k = np.asarray(_field(path, a, key), dtype=np.float64)
                if k.size == 0:
                    k = k.reshape(0, 2)
                if k.ndim != 2 or k.shape[1] != 2:
                    raise ValueError(f"{path}: field {key!r} must be a list of [x, y], got shape {list(k.shape)}")
                kps.append(k)
            if len(kps[0]) != len(kps[1]):
                raise ValueError(f"{path}: field 'trg_kps' has {len(kps[1])} points, 'src_kps' {len(kps[0])}")
            box = np.asarray(_field(path, a, "trg_bndbox"), dtype=np.float64).reshape(-1)
            if box.shape != (4,):
                raise ValueError(f"{path}: field 'trg_bndbox' must be x1 y1 x2 y2, got {box.tolist()}")
            self.pairs.append({"src": ims[0], "trg": ims[1], "category": cat, "src_kps": kps[0], "trg_kps": kps[1],
                               "trg_bbox": box.tolist()})

    def __len__(self):
        return len(self.pairs)

    def __getitem__(self, i):
        return self.pairs[i]

    def load_image(self, j):
        from PIL import Image
        with Image.open(self.images[j]) as im:
            return np.asarray(im.convert("RGB"), dtype=np.uint8)


class CorrespondenceNpzDataset:
    """An .npz file with images (uint8 [N, H, W, 3]), pairs (int [M, 2]: source and target index), src_kps / trg_kps
    (float [M, Kmax, 2], x then y, the first n_kps[m] rows of pair m used), n_kps (int [M]), trg_bbox (float [M, 4]:
    x1 y1 x2 y2) and categories (str [M]); the same `pairs` and `load_image` as SPairDataset."""

    def __init__(self, path):
        path = str(path)
        with np.load(path, allow_pickle=False) as z:
            f = {k: np.asarray(_field(path, z, k)) for k in ("images", "pairs", "src_kps", "trg_kps", "n_kps",
                                                              "trg_bbox", "categories")}
        self.images = f["images"]
        if self.images.dtype != np.uint8 or self.images.ndim != 4 or self.images.shape[-1] != 3:
            raise ValueError(f"{path}: field 'images' must be uint8 [N, H, W, 3], got {self.images.dtype} "
                             f"{list(self.images.shape)}")
        pairs = f["pairs"]
        M = len(pairs)
        if pairs.ndim != 2 or pairs.shape[1] != 2 or pairs.dtype.kind not in "iu":
            raise ValueError(f"{path}: field 'pairs' must be int [M, 2], got {pairs.dtype} {list(pairs.shape)}")
        if M and (pairs.min() < 0 or pairs.max() >= len(self.images)):
            raise ValueError(f"{path}: field 'pairs' indexes outside the {len(self.images)} images")
        for k in ("src_kps", "trg_kps"):
            if f[k].ndim != 3 or f[k].shape[0] != M or f[k].shape[2] != 2:
                raise ValueError(f"{path}: field {k!r} must be float [{M}, Kmax, 2], got {list(f[k].shape)}")
        n = f["n_kps"].reshape(-1)
        if n.shape != (M,) or n.dtype.kind not in "iu" or (M and (n.min() < 0 or n.max() > f["src_kps"].shape[1]
                                                               or n.max() > f["trg_kps"].shape[1])):
            raise ValueError(f"{path}: field 'n_kps' must be int [{M}] within [0, Kmax], got {n.dtype} {n.tolist()}")
        if f["trg_bbox"].shape != (M, 4):
            raise ValueError(f"{path}: field 'trg_bbox' must be float [{M}, 4], got {list(f['trg_bbox'].shape)}")
        if f["categories"].shape != (M,) or f["categories"].dtype.kind not in "US":
            raise ValueError(f"{path}: field 'categories' must be str [{M}], got {f['categories'].dtype} "
                             f"{list(f['categories'].shape)}")
        self.pairs = [{"src": int(pairs[m, 0]), "trg": int(pairs[m, 1]), "category": str(f["categories"][m]),
                       "src_kps": f["src_kps"][m, :n[m]].astype(np.float64),
                       "trg_kps": f["trg_kps"][m, :n[m]].astype(np.float64),
                       "trg_bbox": f["trg_bbox"][m].astype(np.float64).tolist()} for m in range(M)]

    def __len__(self):
        return len(self.pairs)

    def __getitem__(self, i):
        return self.pairs[i]

    def load_image(self, j):
        return self.images[j]


def make_correspondence_dataset(path, split: str = "test"):
    """An .npz file -> CorrespondenceNpzDataset, a directory -> SPairDataset(path, split)."""
    path = str(path)
    return CorrespondenceNpzDataset(path) if path.endswith(".npz") else SPairDataset(path, split)


class VOCDiscoveryDataset:
    """A PASCAL VOC root (VOC2007 or VOC2012): the ids of root/ImageSets/Main/<split>.txt, the images
    root/JPEGImages/<id>.jpg and the annotations root/Annotations/<id>.xml (size/height, size/width and every
    object/bndbox).  VOC's 1-based inclusive corners become [xmin - 1, ymin - 1, xmax, ymax]; remove_difficult drops
    the objects whose `difficult` is 1.  `names`, `sizes` [(H, W)] and `boxes` [float64 [B, 4]] are read up front;
    `load_image(i)` decodes image i to uint8 HWC RGB.  Errors name the file and the field."""

    def __init__(self, root, split: str = "trainval", remove_difficult: bool = False):
        import xml.etree.ElementTree as ET
        self.root, self.split = str(root), split
        lst = os.path.join(self.root, "ImageSets", "Main", f"{split}.txt")
        if not os.path.isfile(lst):
            raise FileNotFoundError(f"{lst} does not exist")
        with open(lst) as f:
            self.names = [line.split()[0] for line in f if line.strip()]
        self.sizes, self.boxes = [], []
        for name in self.names:
            path = os.path.join(self.root, "Annotations", f"{name}.xml")
            if not os.path.isfile(path):
                raise FileNotFoundError(f"{split}.txt names {name}, but {path} does not exist")
            try:
                tree = ET.parse(path).getroot()
            except ET.ParseError as e:
                raise ValueError(f"{path}: not valid XML ({e})") from None
            self.sizes.append((int(_xml_number(path, tree, "size/height")), int(_xml_number(path, tree, "size/width"))))
            boxes = []
            for obj in tree.findall("object"):
                if remove_difficult and obj.find("difficult") is not None and _xml_number(path, obj, "difficult"):
                    continue
                if obj.find("bndbox") is None:
                    raise ValueError(f"{path}: field 'object/bndbox' is missing")
                x1, y1, x2, y2 = (_xml_number(path, obj, f"bndbox/{k}") for k in ("xmin", "ymin", "xmax", "ymax"))
                boxes.append([x1 - 1.0, y1 - 1.0, x2, y2])
            self.boxes.append(np.asarray(boxes, np.float64).reshape(-1, 4))
        self.images = [os.path.join(self.root, "JPEGImages", f"{name}.jpg") for name in self.names]

    def __len__(self):
        return len(self.names)

    def load_image(self, i):
        from PIL import Image
        with Image.open(self.images[i]) as im:
            return np.asarray(im.convert("RGB"), dtype=np.uint8)


def _xml_number(path, node, field) -> float:
    e = node.find(field)
    if e is None or e.text is None or not e.text.strip():
        raise ValueError(f"{path}: field {field!r} is missing")
    try:
        return float(e.text)
    except ValueError:
        raise ValueError(f"{path}: field {field!r} is not a number: {e.text.strip()!r}") from None


class DiscoveryNpzDataset:
    """An .npz file with images (uint8 [N, Hmax, Wmax, 3]), sizes (int [N, 2]: H, W; image i is images[i, :H, :W]),
    boxes (float [N, Bmax, 4]: x1 y1 x2 y2, 0-based continuous corners) and n_boxes (int [N], the first n_boxes[i] rows
    used); the same `names`, `sizes`, `boxes` and `load_image` as VOCDiscoveryDataset, image i named "%05d" % i."""

    def __init__(self, path):
        path = str(path)
        with np.load(path, allow_pickle=False) as z:
            f = {k: np.asarray(_field(path, z, k)) for k in ("images", "sizes", "boxes", "n_boxes")}
        im = f["images"]
        if im.dtype != np.uint8 or im.ndim != 4 or im.shape[-1] != 3:
            raise ValueError(f"{path}: field 'images' must be uint8 [N, H, W, 3], got {im.dtype} {list(im.shape)}")
        n = len(im)
        sz = f["sizes"]
        if (sz.shape != (n, 2) or sz.dtype.kind not in "iu"
                or (n and (sz.min() < 1 or sz[:, 0].max() > im.shape[1] or sz[:, 1].max() > im.shape[2]))):
            raise ValueError(f"{path}: field 'sizes' must be int [{n}, 2] within [1, {im.shape[1]}] x "
                             f"[1, {im.shape[2]}], got {sz.dtype} {list(sz.shape)}")
        bx = f["boxes"]
        if bx.ndim != 3 or bx.shape[0] != n or bx.shape[2] != 4 or bx.dtype.kind != "f":
            raise ValueError(f"{path}: field 'boxes' must be float [{n}, Bmax, 4], got {bx.dtype} {list(bx.shape)}")
        nb = f["n_boxes"].reshape(-1)
        if nb.shape != (n,) or nb.dtype.kind not in "iu" or (n and (nb.min() < 0 or nb.max() > bx.shape[1])):
            raise ValueError(f"{path}: field 'n_boxes' must be int [{n}] within [0, {bx.shape[1]}], got {nb.dtype} "
                             f"{nb.tolist()}")
        self.images = im
        self.names = [f"{i:05d}" for i in range(n)]
        self.sizes = [(int(h), int(w)) for h, w in sz]
        self.boxes = [bx[i, :nb[i]].astype(np.float64) for i in range(n)]

    def __len__(self):
        return len(self.images)

    def load_image(self, i):
        H, W = self.sizes[i]
        return self.images[i, :H, :W]


def make_discovery_dataset(path, split: str = "trainval", remove_difficult: bool = False):
    """An .npz file -> DiscoveryNpzDataset, a directory -> VOCDiscoveryDataset(path, split, remove_difficult)."""
    path = str(path)
    return DiscoveryNpzDataset(path) if path.endswith(".npz") else VOCDiscoveryDataset(path, split, remove_difficult)


def make_eval_dataset(path):
    """An .npz file -> NpzDataset, a directory -> ImageFolder."""
    path = str(path)
    return NpzDataset(path) if path.endswith(".npz") else ImageFolder(path)


RETRIEVAL_DATASETS = ("roxford5k", "rparis6k")


class _GndUnpickler(pickle.Unpickler):
    """Builds builtin containers, numbers, strings and numpy arrays only: any other global is refused before it is
    called, so a ground-truth pickle cannot run code."""

    ALLOWED = {("builtins", n) for n in ("set", "frozenset", "list", "dict", "tuple", "int", "float", "complex", "bool",
                                         "str", "bytes", "bytearray")} | {("_codecs", "encode")} | {
        (m, n) for m in ("numpy.core.multiarray", "numpy._core.multiarray") for n in ("_reconstruct", "scalar")} | {
        ("numpy", "ndarray"), ("numpy", "dtype")}

    def __init__(self, f, path):
        super().__init__(f)
        self.path = path

    def find_class(self, module, name):
        if ("builtins" if module == "__builtin__" else module, name) not in self.ALLOWED:     # protocol 2 spelling
            raise pickle.UnpicklingError(f"{self.path}: refuses the global {module}.{name} (only builtin containers, "
                                         "numbers, strings and numpy arrays may be loaded)")
        return super().find_class(module, name)


def _gnd_indices(path, q, field, value, n) -> np.ndarray:
    a = np.asarray(value)
    if a.size and (a.dtype.kind not in "iu" or a.min() < 0 or a.max() >= n):
        raise ValueError(f"{path}: field 'gnd[{q}].{field}' must hold database indices in [0, {n})")
    return a.astype(np.int64).reshape(-1)


class RevisitedDataset:
    """A revisited Oxford / Paris root: root/gnd_<dataset>.pkl (imlist, qimlist, gnd: per query bbx, easy, hard, junk,
    as lists or ndarrays) and the images root/jpg/<name>.jpg.  `db_names`, `q_names`, `db_sizes` and `q_sizes` [(H, W)]
    (read from the JPEG headers), `q_bbx` float64 [Q, 4] (x1, y1, x2, y2), `easy`, `hard` and `junk` (int64 arrays per
    query) are read up front; `load_db(i)` / `load_query(i)` decode an image to uint8 HWC RGB.  The pickle is loaded by
    a restricted unpickler.  Errors name the file and the field."""

    def __init__(self, root, dataset: str = "roxford5k"):
        from PIL import Image
        if dataset not in RETRIEVAL_DATASETS:
            raise ValueError(f"dataset must be one of {RETRIEVAL_DATASETS}, got {dataset!r}")
        self.root, self.name = str(root), dataset
        path = os.path.join(self.root, f"gnd_{dataset}.pkl")
        if not os.path.isfile(path):
            raise FileNotFoundError(f"{path} does not exist")
        with open(path, "rb") as f:
            cfg = _GndUnpickler(f, path).load()
        if not isinstance(cfg, dict):
            raise ValueError(f"{path}: expected a dict with imlist, qimlist and gnd")
        for k in ("imlist", "qimlist", "gnd"):
            if k not in cfg:
                raise ValueError(f"{path}: field {k!r} is missing")
        self.db_names, self.q_names = [str(v) for v in cfg["imlist"]], [str(v) for v in cfg["qimlist"]]
        gnd, n = list(cfg["gnd"]), len(self.db_names)
        if len(gnd) != len(self.q_names):
            raise ValueError(f"{path}: field 'gnd' has {len(gnd)} entries for {len(self.q_names)} queries")
        self.q_bbx, self.easy, self.hard, self.junk = [], [], [], []
        for q, g in enumerate(gnd):
            for k in ("bbx", "easy", "hard", "junk"):
                if not isinstance(g, dict) or k not in g:
                    raise ValueError(f"{path}: field 'gnd[{q}].{k}' is missing")
            bbx = np.asarray(g["bbx"], np.float64).reshape(-1)
            if bbx.shape != (4,) or not np.isfinite(bbx).all():
                raise ValueError(f"{path}: field 'gnd[{q}].bbx' must be 4 finite numbers (x1, y1, x2, y2)")
            self.q_bbx.append(bbx)
            for k, lst in (("easy", self.easy), ("hard", self.hard), ("junk", self.junk)):
                lst.append(_gnd_indices(path, q, k, g[k], n))
        self.q_bbx = np.asarray(self.q_bbx, np.float64).reshape(-1, 4)
        self.db_images = [os.path.join(self.root, "jpg", f"{v}.jpg") for v in self.db_names]
        self.q_images = [os.path.join(self.root, "jpg", f"{v}.jpg") for v in self.q_names]
        self.db_sizes, self.q_sizes = [], []
        for files, sizes in ((self.db_images, self.db_sizes), (self.q_images, self.q_sizes)):
            for p in files:
                if not os.path.isfile(p):
                    raise FileNotFoundError(f"{path} names {os.path.basename(p)[:-4]}, but {p} does not exist")
                with Image.open(p) as im:
                    sizes.append((im.height, im.width))

    @staticmethod
    def _load(path):
        from PIL import Image
        with Image.open(path) as im:
            return np.asarray(im.convert("RGB"), dtype=np.uint8)

    def load_db(self, i):
        return self._load(self.db_images[i])

    def load_query(self, i):
        return self._load(self.q_images[i])


class RetrievalNpzDataset:
    """An .npz file with db_images (uint8 [N, Hmax, Wmax, 3]) and db_sizes (int [N, 2]: H, W), q_images and q_sizes
    likewise, q_bbx (float [Q, 4]: x1 y1 x2 y2) and the easy, hard and junk lists as CSR pairs (easy_ptr int [Q + 1]
    from 0, easy_idx int database indices, and likewise hard_* and junk_*); the same fields and loaders as
    RevisitedDataset, images named "%05d" % i.  Errors name the file and the field."""

    def __init__(self, path, dataset: str = "roxford5k"):
        path = str(path)
        keys = ["db_images", "db_sizes", "q_images", "q_sizes", "q_bbx"] + [f"{k}_{s}" for k in ("easy", "hard", "junk")
                                                                           for s in ("ptr", "idx")]
        with np.load(path, allow_pickle=False) as z:
            f = {k: np.asarray(_field(path, z, k)) for k in keys}
        self.name = str(dataset)
        for pre in ("db", "q"):
            im, sz = f[f"{pre}_images"], f[f"{pre}_sizes"]
            if im.dtype != np.uint8 or im.ndim != 4 or im.shape[-1] != 3:
                raise ValueError(f"{path}: field '{pre}_images' must be uint8 [n, H, W, 3], got {im.dtype} "
                                 f"{list(im.shape)}")
            n = len(im)
            if (sz.shape != (n, 2) or sz.dtype.kind not in "iu"
                    or (n and (sz.min() < 1 or sz[:, 0].max() > im.shape[1] or sz[:, 1].max() > im.shape[2]))):
                raise ValueError(f"{path}: field '{pre}_sizes' must be int [{n}, 2] within [1, {im.shape[1]}] x "
                                 f"[1, {im.shape[2]}], got {sz.dtype} {list(sz.shape)}")
        N, Q = len(f["db_images"]), len(f["q_images"])
        bbx = f["q_bbx"]
        if bbx.shape != (Q, 4) or bbx.dtype.kind not in "fiu" or not np.isfinite(bbx).all():
            raise ValueError(f"{path}: field 'q_bbx' must be finite [{Q}, 4], got {bbx.dtype} {list(bbx.shape)}")
        lists = {}
        for k in ("easy", "hard", "junk"):
            ptr, idx = f[f"{k}_ptr"].reshape(-1), f[f"{k}_idx"].reshape(-1)
            if (ptr.shape != (Q + 1,) or ptr.dtype.kind not in "iu" or ptr[0] != 0 or (np.diff(ptr) < 0).any()
                    or ptr[-1] != len(idx)):
                raise ValueError(f"{path}: field '{k}_ptr' must be int [{Q + 1}], from 0, non-decreasing, up to "
                                 f"len({k}_idx) = {len(idx)}")
            if idx.size and (idx.dtype.kind not in "iu" or idx.min() < 0 or idx.max() >= N):
                raise ValueError(f"{path}: field '{k}_idx' must hold database indices in [0, {N})")
            lists[k] = [idx[ptr[q]:ptr[q + 1]].astype(np.int64) for q in range(Q)]
        self.easy, self.hard, self.junk = lists["easy"], lists["hard"], lists["junk"]
        self.db, self.q = f["db_images"], f["q_images"]
        self.db_sizes = [(int(h), int(w)) for h, w in f["db_sizes"]]
        self.q_sizes = [(int(h), int(w)) for h, w in f["q_sizes"]]
        self.q_bbx = bbx.astype(np.float64)
        self.db_names, self.q_names = [f"{i:05d}" for i in range(N)], [f"{i:05d}" for i in range(Q)]

    def load_db(self, i):
        H, W = self.db_sizes[i]
        return self.db[i, :H, :W]

    def load_query(self, i):
        H, W = self.q_sizes[i]
        return self.q[i, :H, :W]


def make_retrieval_dataset(path, dataset: str = "roxford5k"):
    """An .npz file -> RetrievalNpzDataset, a directory -> RevisitedDataset(path, dataset)."""
    path = str(path)
    return RetrievalNpzDataset(path, dataset) if path.endswith(".npz") else RevisitedDataset(path, dataset)


class VideoClassListDataset:
    """A list file of `path label` lines, one per video, paths relative to the list's directory.  A path is a video
    file, decoded with OpenCV (cv2, imported when a video is read), or a directory of frame images sorted by name.
    `frame_count(i)` is the container's frame count (a directory's image count); `load_frames(i, indices)` decodes only
    up to the last index asked for and clamps the indices to the frames actually decoded.  A video that cannot be
    opened or has no frame is an error naming its path."""

    def __init__(self, path):
        self.path = str(path)
        root = os.path.dirname(os.path.abspath(self.path))
        self.samples = []
        with open(self.path) as f:
            for k, line in enumerate(f, 1):
                if not line.strip():
                    continue
                parts = line.rsplit(None, 1)
                if len(parts) != 2 or not parts[1].lstrip("-").isdigit():
                    raise ValueError(f"{self.path}:{k}: expected `path label`, got {line.strip()!r}")
                self.samples.append((os.path.join(root, parts[0].strip()), int(parts[1])))
        if not self.samples:
            raise ValueError(f"{self.path}: no videos listed")
        self.targets = [t for _, t in self.samples]

    def __len__(self):
        return len(self.samples)

    def _frame_files(self, d):
        files = sorted(f for f in os.listdir(d) if f.lower().endswith(IMG_EXTENSIONS))
        if not files:
            raise ValueError(f"{d}: no frame images")
        return [os.path.join(d, f) for f in files]

    def frame_count(self, i) -> int:
        path = self.samples[i][0]
        if os.path.isdir(path):
            return len(self._frame_files(path))
        import cv2
        cap = cv2.VideoCapture(path)
        try:
            if not cap.isOpened():
                raise ValueError(f"{path}: cannot open the video")
            return max(int(cap.get(cv2.CAP_PROP_FRAME_COUNT)), 1)
        finally:
            cap.release()

    def load_frames(self, i, indices) -> np.ndarray:
        """uint8 [len(indices), H, W, 3] RGB frames."""
        path = self.samples[i][0]
        need = max(int(j) for j in indices)
        if os.path.isdir(path):
            from PIL import Image
            files = self._frame_files(path)
            frames = {}
            for j in sorted(set(min(int(j), len(files) - 1) for j in indices)):
                with Image.open(files[j]) as im:
                    frames[j] = np.asarray(im.convert("RGB"), dtype=np.uint8)
            return np.stack([frames[min(int(j), len(files) - 1)] for j in indices])
        import cv2
        cap = cv2.VideoCapture(path)
        try:
            if not cap.isOpened():
                raise ValueError(f"{path}: cannot open the video")
            decoded = []
            while len(decoded) <= need:
                ok, frame = cap.read()
                if not ok:
                    break
                decoded.append(frame)
        finally:
            cap.release()
        if not decoded:
            raise ValueError(f"{path}: no frame could be decoded")
        return np.stack([cv2.cvtColor(decoded[min(int(j), len(decoded) - 1)], cv2.COLOR_BGR2RGB) for j in indices])


class VideoClassNpzDataset:
    """An .npz file with `videos` (uint8 [N, F, H, W, 3]) and `labels` (integers [N])."""

    def __init__(self, path):
        with np.load(path, allow_pickle=False) as z:
            self.videos = np.asarray(z["videos"])
            self.targets = [int(v) for v in np.asarray(z["labels"]).reshape(-1)]
        if self.videos.dtype != np.uint8 or self.videos.ndim != 5 or self.videos.shape[-1] != 3:
            raise ValueError(f"{path}: videos must be uint8 [N, F, H, W, 3], got {self.videos.dtype} "
                             f"{self.videos.shape}")
        if len(self.targets) != len(self.videos):
            raise ValueError(f"{path}: {len(self.videos)} videos but {len(self.targets)} labels")

    def __len__(self):
        return len(self.targets)

    def frame_count(self, i) -> int:
        return int(self.videos.shape[1])

    def load_frames(self, i, indices) -> np.ndarray:
        last = self.videos.shape[1] - 1
        return self.videos[i][[min(int(j), last) for j in indices]]


def make_video_class_dataset(path):
    """A `.npz` path -> VideoClassNpzDataset; any other path -> VideoClassListDataset (a list file)."""
    return VideoClassNpzDataset(path) if str(path).endswith(".npz") else VideoClassListDataset(path)
