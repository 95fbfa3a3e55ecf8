"""CPU: the `gpu:` training datasets (data/image_loader.py) — dataset strings, listing, decode, the per-image parameter
draws, the host batches the DataLoader workers pack — and the argument checks of the ragged augmentation entry points."""
import ctypes
import multiprocessing
import os

import numpy as np
import pytest
import torch
from PIL import Image


def _write_images(root, n, seed=0, lo=20, hi=90):
    """n seeded images of random sizes under root/<a|b>/[sub/], JPEG and PNG."""
    rng = np.random.default_rng(seed)
    paths = []
    for i in range(n):
        d = root / ("a" if i % 2 else "b") / ("sub" if i % 3 == 0 else "")
        d.mkdir(parents=True, exist_ok=True)
        h, w = (int(v) for v in rng.integers(lo, hi, 2))
        img = Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        p = d / (f"img{i:03d}.png" if i % 4 == 0 else f"img{i:03d}.jpg")
        img.save(p)
        paths.append(str(p))
    return paths


def _cfg(path, B=4, workers=0, seed=3, extra=()):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    opts = [f"train.dataset_path={path}", f"train.batch_size_per_gpu={B}", f"train.num_workers={workers}",
            f"train.seed={seed}", "student.arch=vit_small", "crops.global_crops_size=64", "crops.local_crops_size=32"]
    return setup_config(DinoV3SetupArgs(opts=opts + list(extra)))


# ---- dataset strings and listing -------------------------------------------------------------------------------------

def test_dataset_strings_accept_known_keys_and_reject_others(tmp_path):
    from dinov3_jax.data.image_loader import parse_dataset_path
    assert parse_dataset_path(f"gpu:ImageFolder:root={tmp_path}") == ("ImageFolder", {"root": str(tmp_path)})
    name, kw = parse_dataset_path("gpu:ImageNet:split=TRAIN:root=/data/in1k:extra=/data/extra")
    assert name == "ImageNet" and kw == {"split": "TRAIN", "root": "/data/in1k", "extra": "/data/extra"}
    assert parse_dataset_path("gpu:ImageNet:split=VAL:root=/r")[1]["split"] == "VAL"
    for bad in ("gpu:ImageFolder:root=/r:split=TRAIN", "gpu:ImageFolder:root=/r:bogus", "gpu:ImageNet:split=TEST:root=/r",
                "gpu:ImageNet:root=/r", "gpu:ImageFolder", "gpu:ImageNet22k:root=/r", "ImageFolder:root=/r"):
        with pytest.raises(ValueError):
            parse_dataset_path(bad)


def test_missing_or_empty_root_names_the_root(tmp_path):
    from dinov3_jax.data.image_loader import dataset_files
    missing = tmp_path / "nope"
    with pytest.raises(FileNotFoundError, match=str(missing)):
        dataset_files(f"gpu:ImageFolder:root={missing}")
    empty = tmp_path / "empty"
    (empty / "sub").mkdir(parents=True)
    (empty / "sub" / "readme.txt").write_text("no images here")
    with pytest.raises(FileNotFoundError, match=str(empty)):
        dataset_files(f"gpu:ImageFolder:root={empty}")
    with pytest.raises(FileNotFoundError, match=str(empty)):
        dataset_files(f"gpu:ImageNet:split=TRAIN:root={empty}")


def test_image_folder_listing_is_recursive_and_sorted(tmp_path):
    from dinov3_jax.data.image_loader import dataset_files
    paths = _write_images(tmp_path, 10)
    (tmp_path / "a" / "notes.txt").write_text("skip me")
    Image.fromarray(np.zeros((4, 4, 3), np.uint8)).save(tmp_path / "b" / "UPPER.PNG")   # extensions match any case
    files = dataset_files(f"gpu:ImageFolder:root={tmp_path}")
    expect = sorted(paths + [str(tmp_path / "b" / "UPPER.PNG")], key=lambda p: (os.path.dirname(p), os.path.basename(p)))
    assert files == expect


def test_imagenet_listing_follows_the_train_and_val_layouts(tmp_path):
    from dinov3_jax.data.image_loader import dataset_files
    for split, names in (("train", ["n02_b.JPEG", "n02_a.JPEG", "n02_c.png"]), ("val", ["v2.JPEG", "v1.JPEG", "v3.png"])):
        for wnid in ("n02", "n01"):
            (tmp_path / split / wnid).mkdir(parents=True)
            for f in names:
                Image.fromarray(np.zeros((4, 4, 3), np.uint8)).save(tmp_path / split / wnid / f, format="PNG")
    tr = dataset_files(f"gpu:ImageNet:split=TRAIN:root={tmp_path}:extra=ignored")
    assert [os.path.relpath(p, tmp_path) for p in tr] == [f"train/{w}/{f}" for w in ("n01", "n02")
                                                          for f in ("n02_a.JPEG", "n02_b.JPEG")]
    va = dataset_files(f"gpu:ImageNet:split=VAL:root={tmp_path}")
    assert [os.path.relpath(p, tmp_path) for p in va] == [f"val/{w}/{f}" for w in ("n01", "n02")
                                                          for f in ("v1.JPEG", "v2.JPEG", "v3.png")]


# ---- decode ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode,ext", [("L", "png"), ("RGBA", "png"), ("P", "png"), ("CMYK", "jpg"), ("RGB", "jpg")])
def test_decode_gives_rgb_uint8_like_pil_convert(tmp_path, mode, ext):
    from dinov3_jax.data.image_loader import decode_rgb
    rng = np.random.default_rng(1)
    src = Image.fromarray(rng.integers(0, 256, (13, 21, 3), dtype=np.uint8)).convert(mode)
    p = tmp_path / f"x.{ext}"
    src.save(p)
    got = decode_rgb(p)
    with Image.open(p) as im:
        assert im.mode == mode
        ref = np.asarray(im.convert("RGB"))
    assert got.dtype == np.uint8 and got.shape == (13, 21, 3) and np.array_equal(got, ref)


def test_undecodable_file_raises_naming_it(tmp_path):
    from dinov3_jax.data.image_loader import ImageFiles
    bad = tmp_path / "broken.jpg"
    bad.write_bytes(b"\xff\xd8 this is not a jpeg")
    with pytest.raises(OSError, match="broken.jpg"):
        ImageFiles([str(bad)])[0]


# ---- parameter draws ---------------------------------------------------------------------------------------------------

def test_ragged_draws_keep_every_box_inside_its_own_image():
    from dinov3_jax.data.gpu_augment import GpuDataAugmentationDINO
    sizes = np.array([[17, 300], [300, 17], [480, 640], [40, 50], [2000, 1500], [96, 96]] * 4)
    for opts in ({}, {"gram_teacher_crops_size": 96}):
        aug = GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), 8, global_crops_size=64, local_crops_size=32, seed=4,
                                      **opts)
        (g, _), (l, _) = aug.sample(len(sizes), sizes[:, 0], sizes[:, 1])
        for rec in (g, l):
            H, W = sizes[rec["img"], 0], sizes[rec["img"], 1]
            assert (rec["x0"] >= 0).all() and (rec["y0"] >= 0).all() and (rec["w"] > 0).all() and (rec["h"] > 0).all()
            assert (rec["x0"] + rec["w"] <= W).all() and (rec["y0"] + rec["h"] <= H).all()
        assert (g["w"][:len(sizes)][sizes[:, 1] == 17] <= 17).all()


def test_equal_sizes_draw_the_dense_records():
    from dinov3_jax.data.gpu_augment import GpuDataAugmentationDINO
    for opts in ({}, {"share_color_jitter": True}, {"local_crops_subset_of_global_crops": True},
                 {"gram_teacher_crops_size": 96}):
        mk = lambda: GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), 8, global_crops_size=64, local_crops_size=32,
                                             seed=11, **opts)
        a, b = mk(), mk()
        B = 6
        for _ in range(3):
            (g0, gb0), (l0, lb0) = a.sample(B, 120, 90)
            (g1, gb1), (l1, lb1) = b.sample(B, np.full(B, 120), np.full(B, 90))
            assert g0.tobytes() == g1.tobytes() and l0.tobytes() == l1.tobytes()
            assert np.array_equal(gb0, gb1) and np.array_equal(lb0, lb1)
        assert a.rng.random() == b.rng.random()                     # both consumed the stream identically


def test_draws_of_an_iteration_do_not_depend_on_what_ran_before(tmp_path):
    from dinov3_jax.data.image_loader import GpuImageLoader
    _write_images(tmp_path, 12)
    sizes = np.array([[30, 40], [55, 21], [80, 80], [25, 70]])
    for extra in ((), ("crops.share_color_jitter=true",)):
        cfg = _cfg(f"gpu:ImageFolder:root={tmp_path}", extra=extra)
        first = GpuImageLoader(cfg).draw(5, sizes)
        ld = GpuImageLoader(cfg)
        for it in range(5):
            ld.draw(it, sizes)
        sixth = ld.draw(5, sizes)
        flat = lambda d: [np.asarray(x).tobytes() for x in (d[0] if d[0] is not None else np.zeros(0),
                                                             *d[1][0], *d[1][1])]
        assert flat(first) == flat(sixth)
        assert flat(first) != flat(ld.draw(6, sizes))
        other_rank = GpuImageLoader(cfg, rank=1, world=2).draw(5, sizes)
        assert flat(first) != flat(other_rank)


# ---- host batches ------------------------------------------------------------------------------------------------------

def _host(cfg, n, **kw):
    from dinov3_jax.data.image_loader import GpuImageLoader
    ld = GpuImageLoader(cfg, **kw)
    gen = ld.host_batches()
    try:
        return [next(gen) for _ in range(n)]
    finally:
        gen.close()


def test_host_batches_do_not_depend_on_worker_count_and_pack_the_decoded_images(tmp_path):
    from dinov3_jax.data.image_loader import dataset_files, decode_rgb
    _write_images(tmp_path, 23)
    path = f"gpu:ImageFolder:root={tmp_path}"
    files = dataset_files(path)
    b0 = _host(_cfg(path, workers=0), 8)                               # 8 batches of 4 cross an epoch of 23 images
    b2 = _host(_cfg(path, workers=2), 8)
    assert not multiprocessing.active_children()
    for x, y in zip(b0, b2):
        assert torch.equal(x["indices"], y["indices"]) and torch.equal(x["sizes"], y["sizes"])
        assert torch.equal(x["pixels"], y["pixels"])
    x = b0[3]
    imgs = [decode_rgb(files[i]) for i in x["indices"].tolist()]
    assert x["sizes"].tolist() == [list(im.shape[:2]) for im in imgs]
    assert x["pixels"].dtype == torch.uint8 and np.array_equal(x["pixels"].numpy(),
                                                               np.concatenate([im.reshape(-1) for im in imgs]))
    resumed = _host(_cfg(path, workers=2), 3, start_iter=5)             # the sampler resumes at start_iter * B
    assert [r["indices"].tolist() for r in resumed] == [r["indices"].tolist() for r in b0[5:8]]
    assert not multiprocessing.active_children()


def test_ranks_of_a_world_of_two_see_disjoint_images(tmp_path):
    _write_images(tmp_path, 24)
    cfg = _cfg(f"gpu:ImageFolder:root={tmp_path}", workers=2)
    r0 = sum((b["indices"].tolist() for b in _host(cfg, 3, rank=0, world=2)), [])
    r1 = sum((b["indices"].tolist() for b in _host(cfg, 3, rank=1, world=2)), [])
    assert len(r0) == len(r1) == 12 and not set(r0) & set(r1)
    assert not multiprocessing.active_children()


def test_a_dataset_smaller_than_one_batch_per_rank_is_refused(tmp_path):
    from dinov3_jax.data.image_loader import GpuImageLoader
    _write_images(tmp_path, 5)
    with pytest.raises(ValueError, match="fewer than one batch"):
        GpuImageLoader(_cfg(f"gpu:ImageFolder:root={tmp_path}", B=4), rank=0, world=2)


def test_loader_builder_routes_the_gpu_prefix_only(tmp_path):
    from dinov3_jax.data.image_loader import GpuImageLoader
    from dinov3_jax.train.train import build_data_loader_from_cfg
    _write_images(tmp_path, 8)
    ld = build_data_loader_from_cfg(_cfg(f"gpu:ImageFolder:root={tmp_path}"), model=None, start_iter=2)
    assert isinstance(ld, GpuImageLoader) and ld.sampler.advance == 8 and ld.start_iter == 2
    with pytest.raises(FileNotFoundError):
        build_data_loader_from_cfg(_cfg(f"gpu:ImageFolder:root={tmp_path / 'missing'}"), model=None)


# ---- C ABI -------------------------------------------------------------------------------------------------------------

def test_ragged_entry_points_refuse_bad_arguments_without_a_gpu():
    from dinov3_jax import _native
    from dinov3_jax.data.gpu_augment import CROP_DTYPE
    lib = _native.lib()
    rec = np.zeros(3, dtype=CROP_DTYPE)
    rec["img"] = [0, 1, 2]
    h = rec.ctypes.data_as(ctypes.c_void_p)
    fake = ctypes.c_void_p(0x1000)                                      # never dereferenced: refused before CUDA
    for name, args in (
            ("d3_aug_resized_crop_ragged", lambda s, t, n, c, hc, o: (s, t, n, c, hc, 3, o, 32, None)),
            ("d3_aug_resized_crop_ragged_f32", lambda s, t, n, c, hc, o: (s, t, n, c, hc, 3, o, 32, 1, None))):
        fn = getattr(lib, name)
        assert fn(*args(None, fake, 3, fake, h, fake)) == -1 and b"null" in lib.d3_last_error()
        assert fn(*args(fake, fake, 3, fake, None, fake)) == -1 and b"null" in lib.d3_last_error()
        assert fn(*args(fake, fake, 0, fake, h, fake)) == -1 and b"n_img" in lib.d3_last_error()
        assert fn(*args(fake, fake, 2, fake, h, fake)) == -1 and b"crop 2 reads image 2" in lib.d3_last_error()
    rec["img"][1] = -1
    assert lib.d3_aug_resized_crop_ragged(fake, fake, 3, fake, h, 3, fake, 32, None) == -1
    rc = lib.d3_aug_color_images_ragged(fake, 100, fake, 3, fake, None, fake, fake, None)
    assert rc == -1 and b"null" in lib.d3_last_error()
    rc = lib.d3_aug_color_images_ragged(fake, 100, fake, 0, fake, h, fake, fake, None)
    assert rc == -1 and b"n_img" in lib.d3_last_error()
    rc = lib.d3_aug_color_images_ragged(fake, 100, fake, 3, fake, h, fake, fake, None)
    assert rc == -1 and b"reads image -1" in lib.d3_last_error()
    rc = lib.d3_aug_color_images_ragged(fake, 100, fake, 3, fake, h, fake, None, None)
    assert rc == -1


def test_ragged_entry_points_are_declared_and_bound():
    import re
    from conftest import ROOT
    from dinov3_jax import _native
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dinov3_b200.h")).read(), flags=re.S)
    for name, nargs in (("d3_aug_resized_crop_ragged", 9), ("d3_aug_resized_crop_ragged_f32", 10),
                        ("d3_aug_color_images_ragged", 9)):
        decl = re.search(name + r"\s*\(([^)]*)\)", src).group(1)
        assert decl.count(",") + 1 == nargs == len(_native.SIGNATURES[name]), name
    assert _native.lib().d3_abi_version() == 7
