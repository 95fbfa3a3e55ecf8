"""Linear depth probe without a GPU: the list and .npz dataset layouts, the `evaluation.depth` block, the --eval depth
flags, the host draws, the Eigen crop, the float64 oracle (tests/depth_oracle.py) on a hand-computed case and against
torch autograd, the metric averaging, and what ptxas makes of csrc/depth.cu."""
import json
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import depth_oracle


# ------------------------------------------------------------------------------------------------ datasets
def _list_tree(root, pairs_train, pairs_val, rng, scale=1000):
    from PIL import Image
    (root / "rgb").mkdir(parents=True)
    (root / "depth").mkdir()
    raw = {}
    for split, names in (("train", pairs_train), ("val", pairs_val)):
        lines = []
        for i, n in enumerate(names):
            H, W = 12 + i, 16 + 2 * i
            Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(root / "rgb" / f"{n}.jpg")
            mm = rng.integers(0, 12000, (H, W)).astype(np.uint16)
            mm[0, :3] = (0, 1000, 65535)
            Image.fromarray(mm).save(root / "depth" / f"{n}.png")
            raw[n] = mm
            lines.append(f"rgb/{n}.jpg depth/{n}.png")
        (root / f"{split}.txt").write_text("\n".join(lines) + "\n")
    return raw


def test_depth_list_layout_sorted_pairs_and_depth_scale(tmp_path):
    from dinov3_jax.eval import DepthListDataset, make_depth_dataset
    rng = np.random.default_rng(0)
    raw = _list_tree(tmp_path, ["b", "a", "c"], ["z", "y"], rng)
    ds = DepthListDataset(tmp_path, "train")
    assert len(ds) == 3 and [os.path.basename(p) for p in ds.images] == ["a.jpg", "b.jpg", "c.jpg"]
    assert [os.path.basename(p) for p in ds.depth_files] == ["a.png", "b.png", "c.png"]
    img, dep = ds[1]
    assert img.dtype == np.uint8 and img.shape[2] == 3 and dep.dtype == np.float32 and dep.shape == img.shape[:2]
    assert np.array_equal(dep, (raw["b"].astype(np.float64) / 1000).astype(np.float32))
    assert dep[0, :3].tolist() == [0.0, 1.0, pytest.approx(65.535)]
    val = make_depth_dataset(str(tmp_path), "val", depth_scale=256)
    assert isinstance(val, DepthListDataset) and os.path.basename(val.images[0]) == "y.jpg"
    assert np.array_equal(val[0][1], (raw["y"].astype(np.float64) / 256).astype(np.float32))
    with pytest.raises(ValueError):
        DepthListDataset(tmp_path, "test")


def test_depth_list_errors_missing_file_bad_line_and_size_mismatch(tmp_path):
    from PIL import Image
    from dinov3_jax.eval import DepthListDataset
    rng = np.random.default_rng(1)
    _list_tree(tmp_path, ["a", "b"], ["c"], rng)
    (tmp_path / "val.txt").write_text("rgb/c.jpg depth/missing.png\n")
    with pytest.raises(FileNotFoundError, match="missing.png"):
        DepthListDataset(tmp_path, "val")
    (tmp_path / "val.txt").write_text("rgb/c.jpg\n")
    with pytest.raises(ValueError, match="line 1"):
        DepthListDataset(tmp_path, "val")
    Image.fromarray(np.zeros((5, 7), np.uint16)).save(tmp_path / "depth" / "b.png")
    ds = DepthListDataset(tmp_path, "train")
    with pytest.raises(ValueError, match="does not match"):
        ds[1]


def test_depth_npz_dataset_and_its_errors(tmp_path):
    from dinov3_jax.eval import DepthNpzDataset, make_depth_dataset
    imgs = np.zeros((3, 8, 12, 3), np.uint8)
    deps = np.linspace(0.5, 9.0, 3 * 8 * 12, dtype=np.float32).reshape(3, 8, 12)
    np.savez(tmp_path / "ok.npz", images=imgs, depths=deps)
    ds = make_depth_dataset(str(tmp_path / "ok.npz"))
    assert isinstance(ds, DepthNpzDataset) and len(ds) == 3
    im, d = ds[2]
    assert im.shape == (8, 12, 3) and d.dtype == np.float32 and np.array_equal(d, deps[2])
    for name, kw, msg in (("a", dict(images=imgs.astype(np.float32), depths=deps), "images must be uint8"),
                          ("b", dict(images=imgs, depths=deps.astype(np.float64)), "depths must be float32"),
                          ("c", dict(images=imgs, depths=deps[:, :4]), "depths must be float32")):
        np.savez(tmp_path / f"{name}.npz", **kw)
        with pytest.raises(ValueError, match=msg):
            DepthNpzDataset(tmp_path / f"{name}.npz")


# ------------------------------------------------------------------------------------------------ config, flags
def test_defaults_carry_the_depth_block():
    from dinov3_jax.configs import get_default_config
    depth = get_default_config().evaluation.depth
    assert depth == {"train_dataset_path": "", "val_dataset_path": "", "n_last_blocks": 1, "use_cls_token": True,
                     "n_bins": 256, "min_depth": 0.001, "max_depth": 10.0, "batch_size": 16, "crop_size": [416, 544],
                     "iterations": 38400, "lr": 1e-3, "weight_decay": 1e-3, "warmup_iterations": 1500,
                     "eval_crop": "eigen", "depth_scale": 1000, "num_workers": 8, "seed": 0}


def test_do_depth_eval_without_datasets_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_depth_eval
    assert do_depth_eval(get_default_config(), None, "training_9") == {}
    assert "nothing evaluated" in capsys.readouterr().out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_still_raises_naming_knn(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match="knn"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_depth_reaches_do_depth_eval_and_nothing_else(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_depth_eval",
                        lambda config, model, header: calls.append((str(model), header)) or {"ok": 4})
    monkeypatch.setattr(train, "do_test", lambda *a, **k: pytest.fail("--eval depth must not run k-NN"))
    monkeypatch.setattr(train, "do_linear_eval", lambda *a, **k: pytest.fail("--eval depth must not run the linear probe"))
    monkeypatch.setattr(train, "do_seg_eval", lambda *a, **k: pytest.fail("--eval depth must not run segmentation"))
    monkeypatch.setattr(train, "do_train", lambda *a, **k: pytest.fail("--eval-only must not train"))
    ck = tmp_path / "ckpt" / "6"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 6, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "depth", "--output-dir", str(tmp_path)]) == {"ok": 4}
    assert calls == [(str(ck), "manual_7")]


# ------------------------------------------------------------------------------------------------ host draws
def test_host_draws_depend_on_seed_only_not_on_num_workers(tmp_path):
    from dinov3_jax.eval.datasets import DepthNpzDataset
    from dinov3_jax.eval.depth import _pack_depth, sample_depth_boxes
    from dinov3_jax.eval.linear import InfiniteBatchSampler
    rng = np.random.default_rng(0)
    np.savez(tmp_path / "d.npz", images=rng.integers(0, 256, (7, 40, 50, 3), dtype=np.uint8),
             depths=rng.uniform(0.1, 9, (7, 40, 50)).astype(np.float32))
    ds = DepthNpzDataset(tmp_path / "d.npz")

    def draws(workers, seed):
        loader = torch.utils.data.DataLoader(ds, batch_sampler=InfiniteBatchSampler(len(ds), 3, 5, seed),
                                             num_workers=workers, collate_fn=_pack_depth)
        aug = torch.Generator().manual_seed(seed + 1)
        out = []
        for flat, dep, desc in loader:
            out.append((flat.sum().item(), dep.sum().item(), desc.tolist(),
                        sample_depth_boxes(aug, desc[:, 1:].tolist(), (32, 48)).tolist()))
        return out

    a = draws(0, 4)
    assert a == draws(2, 4) and a != draws(0, 5)
    boxes = [b for _, _, _, bx in a for b in bx]
    assert any(b[4] for b in boxes) and not all(b[4] for b in boxes)
    assert all(b[:2] == [40, 50] and 0 <= b[2] <= 8 and 0 <= b[3] <= 2 and b[5] == 0 for b in boxes)
    # replayed by hand from the generator: top, left, flip per image, in image order
    g1, g2 = torch.Generator().manual_seed(9), torch.Generator().manual_seed(9)
    want = []
    for H, W in ((480, 640), (300, 500)):
        top = torch.randint(0, max(H - 416, 0) + 1, (1,), generator=g2).item()
        left = torch.randint(0, max(W - 544, 0) + 1, (1,), generator=g2).item()
        want.append([H, W, top, left, int(torch.rand(1, generator=g2).item() < 0.5), 0])
    assert sample_depth_boxes(g1, [(480, 640), (300, 500)], (416, 544)).tolist() == want
    assert want[1][2:4] == [0, 0]


def test_eval_resize_of_an_nyu_frame():
    from dinov3_jax.eval.segmentation import eval_size
    assert eval_size(480, 640, 416, 16) == (416, 560)


def test_eigen_crop_mask():
    from dinov3_jax.eval.depth import eigen_crop
    assert eigen_crop(480, 640, "eigen") == (45, 471, 41, 601)
    assert eigen_crop(375, 1242, "none") == (0, 375, 0, 1242)
    with pytest.raises(ValueError, match="480 x 640"):
        eigen_crop(481, 640, "eigen")
    with pytest.raises(ValueError, match="eval_crop"):
        eigen_crop(480, 640, "garg")
    # every pixel valid: the crop keeps 426 x 560 of them, exactly rows 45..470 and columns 41..600
    z = torch.zeros(1, 30, 40, 8)
    gt = torch.full((1, 480, 640), 2.0)
    sums, _ = depth_oracle.metric_sums(z, gt, 0.001, 10.0, crop=(45, 471, 41, 601))
    assert sums[0, 0].item() == 426 * 560
    gt[0, 45, 41] = gt[0, 470, 600] = 50.0          # out of range inside the crop: left out
    gt[0, 44, :] = gt[0, :, 601] = 3.0              # outside the crop: changes nothing
    s2, _ = depth_oracle.metric_sums(z, gt, 0.001, 10.0, crop=(45, 471, 41, 601))
    assert s2[0, 0].item() == 426 * 560 - 2 and torch.allclose(s2[0, 1:], sums[0, 1:] * (426 * 560 - 2) / (426 * 560))


# ------------------------------------------------------------------------------------------------ float64 oracle
def test_oracle_hand_computed_2x2_to_4x4():
    # 3 bins at 1, 2, 3 m; cell logits -> q = relu(z) + 0.1 -> d
    lo, hi = 1.0, 3.0
    z = torch.tensor([[[[0.0, 0.0, 0.0], [0.9, -1.0, 0.0]], [[0.0, 0.0, 0.3], [-1.0, -1.0, 1.4]]]])
    d_want = [[0.6 / 0.3, 1.5 / 1.2], [1.5 / 0.6, 4.8 / 1.7]]      # 2, 1.25, 2.5, 2.8235...
    d, S = depth_oracle.cell_depth(z, lo, hi)
    assert torch.allclose(d[0], torch.tensor(d_want, dtype=torch.float64), rtol=1e-6)
    assert torch.allclose(S[0], torch.tensor([[0.3, 1.2], [0.6, 1.7]], dtype=torch.float64), rtol=1e-6)
    a = [1.0, 0.75, 0.25, 0.0]                    # weight of cell 0 along an axis of 2 -> 4
    up = [[sum(wy * wx * d_want[i][j] for i, wy in enumerate((a[y], 1 - a[y])) for j, wx in enumerate((a[x], 1 - a[x])))
           for x in range(4)] for y in range(4)]
    assert torch.allclose(depth_oracle.upsample(d, 4, 4)[0], torch.tensor(up, dtype=torch.float64), rtol=1e-6)
    gt = [[2.0, 1.3, 0.0, 2.9], [1.1, 2.2, 2.6, 2.4], [3.5, 1.9, 2.7, 1.6], [2.5, 2.5, 2.8, 1.0]]
    valid = [(y, x) for y in range(4) for x in range(4) if lo < gt[y][x] <= hi]
    assert len(valid) == 13                       # 0.0, 3.5 and 1.0 (not > min_depth) are left out
    g = [math.log(up[y][x] + 1e-3) - math.log(gt[y][x] + 1e-3) for y, x in valid]
    mu = sum(g) / len(g)
    var = sum((v - mu) ** 2 for v in g) / (len(g) - 1)
    L_want = math.sqrt(var + 0.15 * mu * mu)
    L, dz, n, _ = depth_oracle.si_loss(z.float(), torch.tensor([gt]), lo, hi)
    assert n == 13 and L == pytest.approx(L_want, rel=1e-6)
    # dL/dz of bin 2 of cell (1, 1): 1[z > 0] (c - d) / S * sum over pixels of w dL/dd_hat
    dd = sum((1 - a[y]) * (1 - a[x]) * ((gi - mu) / 12 + 0.15 * mu / 13) / L_want / (up[y][x] + 1e-3)
             for (y, x), gi in zip(valid, g))
    assert dz[0, 1, 1, 2].item() == pytest.approx((3.0 - 4.8 / 1.7) / 1.7 * dd, rel=1e-5)
    assert dz[0, 1, 1, 0].item() == 0.0 and dz[0, 0, 0].abs().sum().item() == 0.0     # z <= 0: no gradient
    # metrics: p clamped to [1, 3] (no clamping needed here), per image over the valid pixels
    sums, _ = depth_oracle.metric_sums(z.float(), torch.tensor([gt]), lo, hi)
    p = [up[y][x] for y, x in valid]
    t = [gt[y][x] for y, x in valid]
    ratio = [max(pi / ti, ti / pi) for pi, ti in zip(p, t)]
    want = [13, sum(abs(pi - ti) / ti for pi, ti in zip(p, t)), sum((pi - ti) ** 2 / ti for pi, ti in zip(p, t)),
            sum((pi - ti) ** 2 for pi, ti in zip(p, t)), sum((math.log(pi) - math.log(ti)) ** 2 for pi, ti in zip(p, t)),
            sum(abs(math.log10(pi) - math.log10(ti)) for pi, ti in zip(p, t))] + \
           [sum(r < 1.25 ** k for r in ratio) for k in (1, 2, 3)]
    assert sums[0].tolist() == pytest.approx(want, rel=1e-6)
    assert want[6] < want[7] < want[8] < 13       # each threshold changes the count here
    m = depth_oracle.metrics(sums)
    assert m["rmse"] == pytest.approx(math.sqrt(want[3] / 13)) and m["a1"] == pytest.approx(want[6] / 13)


def _autograd_reference(z, gt, lo, hi):
    import torch.nn.functional as Fn
    z = z.double().clone().requires_grad_(True)
    q = torch.relu(z) + 0.1
    d = (q * torch.linspace(lo, hi, z.shape[-1], dtype=torch.float64)).sum(-1) / q.sum(-1)
    dh = Fn.interpolate(d[:, None], size=gt.shape[1:], mode="bilinear", align_corners=False)[:, 0]
    valid = (gt > lo) & (gt <= hi)
    g = torch.log(dh[valid] + 1e-3) - torch.log(gt[valid].double() + 1e-3)
    L = torch.sqrt(torch.var(g) + 0.15 * g.mean() ** 2)
    L.backward()
    return L.item(), z.grad


@pytest.mark.parametrize("shape", [(1, 3, 5, 7, 11, 16), (2, 3, 5, 7, 11, 9), (2, 6, 4, 3, 5, 5)])
def test_oracle_gradient_matches_torch_autograd_float64(shape):
    B, h, w, Hl, Wl, nb = shape
    g = torch.Generator().manual_seed(nb)
    z = torch.randn(B, h, w, nb, generator=g, dtype=torch.float64) * 2 - 0.5
    gt = torch.rand(B, Hl, Wl, generator=g, dtype=torch.float64) * 9 + 0.5
    gt[torch.rand(B, Hl, Wl, generator=g) < 0.15] = 0.0
    gt[torch.rand(B, Hl, Wl, generator=g) < 0.1] = 12.0
    lo, hi = 0.001, 10.0
    L_ref, grad = _autograd_reference(z, gt, lo, hi)
    L, dz, n, env = depth_oracle.si_loss(z, gt, lo, hi)
    assert n == int(((gt > lo) & (gt <= hi)).sum()) and n < B * Hl * Wl
    assert L == pytest.approx(L_ref, rel=1e-12)
    assert torch.allclose(dz, grad, rtol=1e-9, atol=1e-14)
    assert (env >= 0).all()


def test_oracle_fewer_than_two_valid_pixels_gives_zero():
    z = torch.randn(1, 2, 2, 4)
    gt = torch.zeros(1, 4, 4)
    assert depth_oracle.si_loss(z, gt, 0.001, 10.0)[:3:2] == (0.0, 0)
    gt[0, 1, 1] = 3.0
    L, dz, n, _ = depth_oracle.si_loss(z, gt, 0.001, 10.0)
    assert (L, n) == (0.0, 1) and (dz == 0).all()


def test_depth_metrics_average_per_image_and_skip_empty_images():
    from dinov3_jax.eval.depth import depth_metrics
    rng = np.random.default_rng(0)
    s = np.abs(rng.normal(size=(4, 9))) * 10
    s[:, 0] = [100, 0, 50, 7]
    s[:, 6:] = np.minimum(s[:, 6:], s[:, :1])
    got = depth_metrics(s)
    want = depth_oracle.metrics(torch.from_numpy(s))
    assert sorted(got) == sorted(depth_oracle.METRIC_NAMES)
    for k in got:
        assert got[k] == pytest.approx(want[k], rel=1e-12)
    assert got["rmse"] == pytest.approx(np.mean([np.sqrt(s[i, 3] / s[i, 0]) for i in (0, 2, 3)]))
    with pytest.raises(ValueError):
        depth_metrics(np.zeros((2, 9)))


# ------------------------------------------------------------------------------------------------ ptxas
def test_depth_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert "depth.cu" in b.SOURCES
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", "depth.cu"), "-o",
                                       str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    seen = set()
    for name, stack, st, ld in props:
        if "depth_" in name:
            seen.add(name)
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # cell depth, moments, loss, gradient tiles, dZ, metric tiles, per-image metrics, depth-plane crop
    assert len(seen) == 8, sorted(seen)
