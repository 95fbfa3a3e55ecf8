"""-m gpu: ragged image batches through the on-GPU augmentation (csrc/augment.cu, data/gpu_augment.py) and the `gpu:`
training loader (data/image_loader.py) through do_train."""
import multiprocessing

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# (H, W): thin strips, a VGA frame, squares smaller than the 64-pixel crop (the kernel upsamples), odd sizes
SIZES = [(17, 300), (300, 17), (480, 640), (20, 30), (45, 45), (130, 97), (64, 64), (251, 333), (8, 120)]


def _images(sizes, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in sizes]


def _records(sizes, n_per, rng, flips=True):
    """Random boxes inside each image (some the whole image), half of them flipped."""
    from dinov3_jax.data.gpu_augment import CROP_DTYPE
    rec = np.zeros(len(sizes) * n_per, dtype=CROP_DTYPE)
    rec["order"] = -1
    for i in range(len(rec)):
        b = i % len(sizes)
        H, W = sizes[b]
        h, w = (H, W) if i < len(sizes) else (int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1)))
        rec["img"][i], rec["h"][i], rec["w"][i] = b, h, w
        rec["y0"][i], rec["x0"][i] = rng.integers(0, H - h + 1), rng.integers(0, W - w + 1)
        rec["flip"][i] = int(flips and rng.random() < 0.5)
    return rec


def _aug(**kw):
    from dinov3_jax.data.gpu_augment import GpuDataAugmentationDINO
    return GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), 4, global_crops_size=64, local_crops_size=32, seed=7, **kw)


def _dense_crop(aug, img, rec, S, clamp=True):
    """The dense kernel on one image alone, with the record pointed at image 0."""
    r = rec.copy()
    r["img"] = 0
    return aug._crop(img[None].contiguous(), r, aug._dev(r, img.device), S, ("dense", S), clamp).clone()


def test_ragged_crops_equal_the_dense_kernel_on_each_image_alone(native):
    from dinov3_jax.data.gpu_augment import RaggedImages
    imgs = [t.cuda() for t in _images(SIZES)]
    rng = np.random.default_rng(0)
    rec = _records(SIZES, 4, rng)
    aug = _aug()
    for src, clamps in ((RaggedImages.from_images(imgs), (True,)),
                        (RaggedImages.from_images([t.float() / 255 for t in imgs]), (True, False))):
        for S, clamp in ((64, c) for c in clamps):
            got = aug._crop(src, rec, aug._dev(rec, src.device), S, "ragged", clamp).clone()
            for i in range(len(rec)):
                ref = _dense_crop(aug, src.image(int(rec["img"][i])), rec[i:i + 1], S, clamp)[0]
                assert torch.equal(got[i], ref), (S, clamp, i, rec[i])
    with pytest.raises(AssertionError, match="outside its image"):
        bad = rec[:1].copy()
        bad["w"] = SIZES[0][1] + 1
        aug._crop(RaggedImages.from_images(imgs), bad, aug._dev(bad, "cuda"), 64, "ragged")


def test_ragged_crops_match_torchvision_resized_crop(native):
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms.v2 import functional as F
    from dinov3_jax.data.gpu_augment import RaggedImages
    imgs = _images(SIZES, seed=1)
    rec = _records(SIZES, 3, np.random.default_rng(1))
    aug = _aug()
    src = RaggedImages.from_images(imgs, "cuda")
    for S in (64, 32):
        got = aug._crop(src, rec, aug._dev(rec, src.device), S, "ragged").cpu()
        for i in range(len(rec)):
            x = imgs[rec["img"][i]].permute(2, 0, 1).float() / 255
            ref = F.resized_crop(x, int(rec["y0"][i]), int(rec["x0"][i]), int(rec["h"][i]), int(rec["w"][i]), [S, S],
                                 interpolation=InterpolationMode.BICUBIC, antialias=True).clamp(0, 1).permute(1, 2, 0)
            if rec["flip"][i]:
                ref = ref.flip(1)
            err = float((got[i] - ref).abs().max())
            assert err < 2e-3, (S, i, err)


def _close(a, b):
    """Equal bits, up to the float atomic sum of contrast's mean gray (csrc/augment.cu, as on the dense path): its order
    can change from run to run and move the last bits of that mean, so of the fp32 pixels contrast blends, and by at
    most one bf16 step a small share of the bf16 crops."""
    if torch.equal(a, b):
        return True
    d = (a.float() - b.float()).abs()
    if a.dtype == torch.float32:
        ok = float(d.max()) < 4e-6
    else:
        ok = float((d > 0).float().mean()) < 1e-2 and bool((d <= 2 ** -7 * b.float().abs().clamp(min=1.0)).all())
    if not ok:
        print(f"differ: {float((d > 0).float().mean()):.2e} of elements, max {float(d.max()):.2e}")
    return ok


@pytest.mark.parametrize("opts", [{}, {"gram_teacher_crops_size": 96, "gram_teacher_no_distortions": True},
                                  {"gram_teacher_crops_size": 96}, {"local_crops_subset_of_global_crops": True},
                                  {"share_color_jitter": True}],
                         ids=["default", "gram_no_distortions", "gram", "subset_locals", "share_color_jitter"])
def test_equal_size_ragged_batch_gives_the_dense_pipeline(native, opts):
    from dinov3_jax.data.gpu_augment import RaggedImages
    imgs = [t.cuda() for t in _images([(120, 90)] * 6, seed=2)]
    dense, ragged = _aug(**opts), _aug(**opts)
    for _ in range(2):
        a = dense(torch.stack(imgs))
        b = ragged(RaggedImages.from_images(imgs))
        assert a.keys() == b.keys()
        for k in a:
            assert a[k].shape == b[k].shape and _close(b[k], a[k]), k


def test_shared_jitter_on_mixed_sizes_equals_each_image_alone(native):
    from dinov3_jax.data.gpu_augment import RaggedImages
    imgs = [t.cuda() for t in _images(SIZES, seed=3)]
    aug = _aug(share_color_jitter=True)
    aug.rng = np.random.default_rng(5)
    recs = aug.sample_source_jitter(len(imgs))
    (g, gb), _ = aug.sample(len(imgs), [h for h, _ in SIZES], [w for _, w in SIZES])
    src = aug.jitter_sources(RaggedImages.from_images(imgs), recs)
    jittered = [src.image(b).clone() for b in range(len(imgs))]
    out = aug.apply(src, g, gb, 64)
    for b, img in enumerate(imgs):
        one = recs[b:b + 1].copy()
        one["img"] = 0
        alone = aug.jitter_sources(img[None].contiguous(), one)
        assert _close(jittered[b], alone[0]), b
        for i in np.flatnonzero(g["img"] == b):
            r = g[i:i + 1].copy()
            r["img"] = 0
            assert _close(out[i], aug.apply(alone.contiguous(), r, gb[i:i + 1], 64)[0]), (b, i)


def _write_folder(root, n=48, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    for i in range(n):
        d = root / f"c{i % 3}"
        d.mkdir(parents=True, exist_ok=True)
        h, w = (int(v) for v in rng.integers(40, 300, 2))
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(d / f"{i:03d}.{'png' if i % 3 else 'jpg'}")


def test_do_train_on_an_image_folder_resumes_with_the_same_crops(tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train import train
    _write_folder(tmp_path / "imgs")
    seen = {}

    real = train.build_data_loader_from_cfg

    def recording(config, model, start_iter=0):
        loader = real(config, model, start_iter)

        def gen():
            it = iter(loader)
            try:
                for k in range(start_iter, 1 << 30):
                    b = next(it)
                    seen.setdefault(str(config.train.output_dir), {})[k] = {
                        key: b[key].clone() for key in ("collated_global_crops", "collated_local_crops")}
                    yield b
            finally:
                loader.close()
        return gen()
    monkeypatch.setattr(train, "build_data_loader_from_cfg", recording)

    def cfg(out):
        opts = [f"train.dataset_path=gpu:ImageFolder:root={tmp_path / 'imgs'}", "train.batch_size_per_gpu=4",
                "train.num_workers=2", "student.arch=vit_small", "crops.global_crops_size=64", "crops.local_crops_size=32",
                "dino.head_n_prototypes=512", "ibot.head_n_prototypes=512", "dino.head_hidden_dim=256",
                "ibot.head_hidden_dim=256", "dino.head_bottleneck_dim=64", "ibot.head_bottleneck_dim=64",
                "optim.epochs=1", "train.OFFICIAL_EPOCH_LENGTH=8", "optim.warmup_epochs=0",
                "teacher.warmup_teacher_temp_epochs=0", "optim.freeze_last_layer_epochs=0", f"train.output_dir={out}",
                "checkpointing.period=2", "checkpointing.max_to_keep=1"]
        return setup_config(DinoV3SetupArgs(opts=opts))

    c = cfg(tmp_path / "full")
    m = train.do_train(c, SSLMetaArch(c), max_iters=3, print_freq=1)
    assert m["total_loss"] == m["total_loss"] and 0 < m["total_loss"] < 1e4
    assert not multiprocessing.active_children()
    c = cfg(tmp_path / "split")
    train.do_train(c, SSLMetaArch(c), max_iters=2, print_freq=1)          # stops after iteration 1 (checkpoint 1)
    assert not multiprocessing.active_children()
    m = train.do_train(c, SSLMetaArch(c), resume=True, max_iters=3, print_freq=1)
    assert m["total_loss"] == m["total_loss"]
    assert not multiprocessing.active_children()
    full, split = seen[str(tmp_path / "full")], seen[str(tmp_path / "split")]
    for k in ("collated_global_crops", "collated_local_crops"):
        for it in (0, 1, 2):                                               # 2: the first iteration after the resume
            assert _close(split[it][k], full[it][k]), (k, it)
        assert not _close(full[1][k], full[2][k])


def test_loader_workers_end_when_do_train_raises(tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.engine.core import Engine
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train.train import do_train
    _write_folder(tmp_path / "imgs", n=16)
    opts = [f"train.dataset_path=gpu:ImageFolder:root={tmp_path / 'imgs'}", "train.batch_size_per_gpu=4",
            "train.num_workers=2", "student.arch=vit_small", "crops.global_crops_size=64", "crops.local_crops_size=32",
            "dino.head_n_prototypes=512", "ibot.head_n_prototypes=512", "dino.head_hidden_dim=256",
            "ibot.head_hidden_dim=256", "dino.head_bottleneck_dim=64", "ibot.head_bottleneck_dim=64",
            f"train.output_dir={tmp_path}"]
    c = setup_config(DinoV3SetupArgs(opts=opts))

    def boom(self, *a, **k):
        raise RuntimeError("step failed")
    monkeypatch.setattr(Engine, "train_step", boom)
    with pytest.raises(RuntimeError, match="step failed"):
        do_train(c, SSLMetaArch(c), max_iters=2, print_freq=1)
    assert not multiprocessing.active_children()
