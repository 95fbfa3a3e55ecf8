"""CPU: the random parameters of the on-GPU augmentation for the DataAugmentationDINO options beyond the defaults, and
that the default options still draw exactly what they drew before those options existed."""
import hashlib

import numpy as np
import pytest

from dinov3_jax.data.gpu_augment import GpuDataAugmentationDINO

# sha256 of the default-option records below, as drawn before gram / subset / shared-jitter support was added
DEFAULT_RECORDS_SHA256 = "94cde5fe4b68e4c050a698c567c20e420263ed056a77c6e8f55310c4d335a52b"


def _aug(**kw):
    kw.setdefault("global_crops_size", 64)
    kw.setdefault("local_crops_size", 32)
    return GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), kw.pop("n_local", 4), seed=kw.pop("seed", 0), **kw)


def test_default_records_are_unchanged():
    h = hashlib.sha256()
    for seed, (gs, ls, n, flips) in enumerate([(224, 96, 8, True), (64, 32, 4, True), (256, 112, 6, False)]):
        a = GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), n, global_crops_size=gs, local_crops_size=ls,
                                    horizontal_flips=flips, seed=seed)
        for B, H, W in [(4, 224, 224), (3, 150, 333)]:
            (g, gb), (l, lb) = a.sample(B, H, W)
            for arr in (g, gb, l, lb):
                h.update(arr.tobytes())
    assert h.hexdigest() == DEFAULT_RECORDS_SHA256


def test_teacher_no_color_jitter_draws_nothing_and_changes_nothing():
    a, b = _aug(seed=5), _aug(seed=5, teacher_no_color_jitter=True)
    for _ in range(2):
        (ga, gba), (la, lba) = a.sample(3, 100, 120)
        (gb_, gbb), (lb_, lbb) = b.sample(3, 100, 120)
        assert ga.tobytes() == gb_.tobytes() and la.tobytes() == lb_.tobytes()
        assert np.array_equal(gba, gbb) and np.array_equal(lba, lbb)


@pytest.mark.parametrize("gs,ls,patch,n", [(64, 32, 16, 4), (224, 96, 16, 8), (256, 112, 16, 6), (98, 42, 14, 2)])
def test_subset_windows(gs, ls, patch, n):
    """local_crops_subset_of_global_crops: window offsets are multiples of the patch in [0, (gs - ls) // patch) * patch,
    half of the windows come from each global crop of the same image, and a window has no flip or resized crop."""
    a = _aug(global_crops_size=gs, local_crops_size=ls, n_local=n, patch_size=patch,
             local_crops_subset_of_global_crops=True, seed=3)
    B = 5
    _, (l, lb) = a.sample(B, 200, 240)
    assert l.shape == (n * B,)
    top = ((gs - ls) // patch - 1) * patch
    for key in ("x0", "y0"):
        assert (l[key] % patch == 0).all() and (l[key] >= 0).all() and (l[key] <= top).all()
    assert (l["w"] == ls).all() and (l["h"] == ls).all() and (l["flip"] == 0).all() and (l["solarize"] == 0).all()
    for c in range(n):
        rows = l["img"][c * B:(c + 1) * B]
        assert (rows == (0 if c < n // 2 else B) + np.arange(B)).all()
    assert ((lb == 0) | ((lb >= 0.1) & (lb <= 2.0))).all()
    # many draws reach both ends of the offset range
    _, (l2, _) = a.sample(200, 200, 240)
    assert l2["x0"].min() == 0 and l2["x0"].max() == top and l2["y0"].max() == top


def test_shared_jitter_records():
    """share_color_jitter: the crops carry no jitter or grayscale of their own; one record per source image does."""
    a = _aug(share_color_jitter=True, seed=4)
    src = a.sample_source_jitter(64)
    assert (src["img"] == np.arange(64)).all()
    jit = src["order"][:, 0] >= 0
    assert 0.6 < jit.mean() < 0.95 and 0 < src["gray"].mean() < 0.4
    assert all(sorted(o) == [0, 1, 2, 3] for o in src["order"][jit])
    assert (src["order"][~jit] == -1).all()
    (g, gb), (l, lb) = a.sample(8, 120, 90)
    for r in (g, l):
        assert (r["order"] == -1).all() and (r["gray"] == 0).all()
        assert (r["fb"] == 0).all() and (r["fh"] == 0).all()
    assert (gb[:8] == 0).all() and (gb[8:] > 0).any()        # the blur is still drawn per crop


def test_gram_records_are_base_crops():
    """With a gram size the global records are the base crops at max(global, gram) (same draws: RandomResizedCrop's
    parameters do not depend on the output size)."""
    a, b = _aug(seed=9), _aug(seed=9, gram_teacher_crops_size=96, gram_teacher_no_distortions=True)
    assert b.base_size == 96 and _aug(gram_teacher_crops_size=48).base_size == 64
    (ga, _), (la, _) = a.sample(4, 150, 150)
    (gb_, _), (lb_, _) = b.sample(4, 150, 150)
    assert ga.tobytes() == gb_.tobytes() and la.tobytes() == lb_.tobytes()


def test_rejections():
    with pytest.raises(ValueError, match="even"):
        _aug(n_local=3, local_crops_subset_of_global_crops=True)
    with pytest.raises(ValueError, match="no offset"):
        _aug(global_crops_size=64, local_crops_size=56, patch_size=16, local_crops_subset_of_global_crops=True)
    with pytest.raises(ValueError, match="no offset"):
        _aug(global_crops_size=96, local_crops_size=96, local_crops_subset_of_global_crops=True)
    with pytest.raises(NotImplementedError):
        _aug(gram_teacher_crops_size=[256, 512])
    # the same sizes without the subset option are fine
    _aug(n_local=3)
    _aug(global_crops_size=64, local_crops_size=56)


def test_pipeline_passes_the_crop_options():
    """GpuBatchPipeline reads the YAML spellings of the crop options (crops.localcrops_subset_of_globalcrops, ...)."""
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.data.gpu_augment import GpuBatchPipeline
    opts = ["crops.global_crops_size=64", "crops.local_crops_size=32", "crops.gram_teacher_crops_size=96",
            "crops.gram_teacher_no_distortions=true", "crops.localcrops_subset_of_globalcrops=true",
            "crops.share_color_jitter=true", "crops.local_crops_number=4", "student.patch_size=16"]
    aug = GpuBatchPipeline(setup_config(DinoV3SetupArgs(opts=opts))).aug
    assert aug.gram == 96 and aug.gram_no_distortions and aug.subset and aug.share_color_jitter and aug.patch == 16
    assert aug.base_size == 96
    default = GpuBatchPipeline(setup_config(DinoV3SetupArgs(opts=opts[:2]))).aug
    assert default.gram is None and not default.subset and not default.share_color_jitter
