"""CPU: the host data path either side of the hot path — the package overlay that lets the reference's loaders /
augmentations (which "stay") resolve next to this package, the reference-shaped loader builder, the resumable sampler,
and the committed loader fixture (produced by the reference's own DataAugmentationDINO, tests/golden/make_loader_fixture.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT


def _stub_reference(root):
    """A stand-in reference checkout: the two data modules the overlay leaves to the reference (augmentations,
    transforms), each recording where it was imported from."""
    data = root / "dinov3_jax" / "data"
    data.mkdir(parents=True)
    for name in ("augmentations", "transforms"):
        (data / f"{name}.py").write_text("ORIGIN = 'reference'\n")
    return str(root)


def test_overlay_resolves_reference_data_modules_but_hot_path_stays_here(tmp_path):
    ref = _stub_reference(tmp_path / "reference")
    code = ("import sys; sys.path.insert(0, %r); sys.path.append(%r)\n"
            "import dinov3_jax.data.augmentations as a, dinov3_jax.data.transforms as t\n"
            "import dinov3_jax.data.masking as m, dinov3_jax.data.collate as c, dinov3_jax.train.train as tr, dinov3_jax.loss as l\n"
            "print(a.__file__); print(t.__file__); print(m.__file__); print(c.__file__); print(tr.__file__); print(l.__file__)\n"
            % (os.path.join(ROOT, "dinov3-jax_b200"), ref))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    files = out.stdout.strip().splitlines()
    assert files[0].startswith(ref) and files[1].startswith(ref)                    # stay in the reference
    assert all(f.startswith(ROOT) for f in files[2:]), files                        # hot path + jax-free data pieces


def test_missing_reference_loader_raises_a_helpful_import_error():
    import importlib.util
    import dinov3_jax.data as d
    if importlib.util.find_spec("dinov3_jax.data.loaders") is not None:
        pytest.skip("a reference checkout is on sys.path")
    with pytest.raises(ImportError, match="reference"):
        d.make_data_loader  # noqa: B018


def test_fixture_has_the_collate_contract():
    b = np.load(os.path.join(GOLDEN, "loader_batch.npz"))
    assert b["collated_global_crops"].shape == (4, 64, 64, 3) and b["collated_local_crops"].shape == (16, 32, 32, 3)
    assert b["collated_masks"].dtype == np.bool_ and b["collated_masks"].shape == (4, 16)
    idx = b["mask_indices_list"]
    assert np.array_equal(idx, np.flatnonzero(b["collated_masks"].reshape(-1)))          # bit-exact index contract
    assert int(b["n_masked_patches"][0]) == idx.shape[0]
    g = torch.from_numpy(b["collated_global_crops"]).view(torch.bfloat16).float()
    assert torch.isfinite(g).all() and 0.3 < float(g.std()) < 3.0                         # ImageNet-normalised pixels


def test_seeded_batch_sampler_resumes_where_it_stopped():
    from dinov3_jax.data.synthetic import SeededBatchSampler
    a = iter(SeededBatchSampler(103, 4, seed=5, rank=1, world=2))
    first = [next(a) for _ in range(40)]                 # crosses several epochs (51 samples / rank -> 12 batches each)
    b = iter(SeededBatchSampler(103, 4, seed=5, rank=1, world=2, advance=17 * 4))
    assert [next(b) for _ in range(23)] == first[17:]
    other = iter(SeededBatchSampler(103, 4, seed=5, rank=0, world=2))
    assert not set(sum(first[:12], [])) & set(sum([next(other) for _ in range(12)], []))   # ranks see disjoint samples


def test_args_parser_keeps_the_reference_flags():
    from dinov3_jax.train.train import get_args_parser
    a = get_args_parser().parse_args(["--config-file", "x.yaml", "--no-resume", "--output-dir", "out", "7",
                                      "--opts", "a.b=1", "c=2"])
    assert a.seed == 7 and a.config_file == "x.yaml" and a.no_resume and a.opts == ["a.b=1", "c=2"]
    assert get_args_parser().parse_args([]).seed == 12                      # train/train.py:66 default


def test_gpu_augment_parameter_sampling_follows_torchvision_rules():
    """Host side of the on-GPU augmentation: crop boxes inside the image with area / aspect ratio in the configured
    ranges, crop-major record order, the reference's blur probabilities as coded (0.0 / 0.9 / 0.5), solarize only on the
    second global crop, and the 64-byte record layout the kernels read."""
    from dinov3_jax.data.gpu_augment import CROP_DTYPE, GpuDataAugmentationDINO
    assert CROP_DTYPE.itemsize == 64 and CROP_DTYPE.fields["order"][1] == 24 and CROP_DTYPE.fields["fb"][1] == 40
    aug = GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), 8, seed=1)
    B, H, W = 64, 300, 400
    (g, gb), (l, lb) = aug.sample(B, H, W)
    assert g.shape == (2 * B,) and l.shape == (8 * B,)
    assert (g["img"] == np.tile(np.arange(B), 2)).all() and (l["img"] == np.tile(np.arange(B), 8)).all()
    for rec, scale in ((g, (0.32, 1.0)), (l, (0.05, 0.32))):
        assert (rec["x0"] >= 0).all() and (rec["y0"] >= 0).all() and (rec["x0"] + rec["w"] <= W).all() and (rec["y0"] + rec["h"] <= H).all()
        area = rec["w"] * rec["h"] / (H * W)
        assert area.min() > scale[0] * 0.9 and area.max() < scale[1] * 1.1
        ratio = rec["w"] / rec["h"]
        assert ratio.min() > 0.74 and ratio.max() < 1.35
    assert (gb[:B] == 0).all()                               # GaussianBlur(p=1.0) -> RandomApply(p=0.0): never applied
    assert 0.75 < (gb[B:] > 0).mean() <= 1.0                 # GaussianBlur(p=0.1) -> applied with probability 0.9
    assert 0.35 < (lb > 0).mean() < 0.65
    assert g["solarize"][:B].sum() == 0 and 0 < g["solarize"][B:].sum() < B and l["solarize"].sum() == 0
    jit = g["order"][:, 0] >= 0
    assert 0.6 < jit.mean() < 0.95 and all(sorted(o) == [0, 1, 2, 3] for o in g["order"][jit])


def test_multi_resolution_builder_accepts_one_triple_and_rejects_lists():
    """train/train.py:718-769: one (global, local, gram) size triple builds the ordinary loader with seed + 1; resolution
    lists raise (the engine is laid out for one triple)."""
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train.train import build_multi_resolution_data_loader_from_cfg

    class Model:
        pass
    cfg = setup_config(DinoV3SetupArgs(opts=["train.dataset_path=synthetic", "student.arch=vit_small", "train.batch_size_per_gpu=1"]))
    from dinov3_jax.engine import config_from_reference_cfg
    m = Model(); m.engine_config = config_from_reference_cfg(cfg)
    loader = build_multi_resolution_data_loader_from_cfg(cfg, m, 0)
    b = next(iter(loader))
    assert tuple(b["collated_global_crops"].shape) == (2, 224, 224, 3) and tuple(b["collated_local_crops"].shape) == (8, 96, 96, 3)
    cfg.crops.global_crops_size, cfg.crops.local_crops_size = [224, 448], [96, 112]
    cfg.crops.gram_teacher_crops_size, cfg.crops.global_local_crop_pairs_ratios = [None, None], [1.0, 1.0]
    with pytest.raises(NotImplementedError):
        build_multi_resolution_data_loader_from_cfg(cfg, m, 0)
