"""Linear segmentation probe without a GPU: the ADE20K dataset layout and the .npz form, the `evaluation.segmentation`
block, the --eval seg flags, the host draws, the schedule, the metrics, the float64 oracle (tests/seg_oracle.py) on
hand-computed cases and against torch's own float64 interpolate + cross-entropy, and what ptxas makes of the kernels."""
import json
import os
import re
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import torch

import seg_oracle


# ------------------------------------------------------------------------------------------------ datasets
def _ade_tree(root, names_train, names_val, rng):
    from PIL import Image
    (root / "images").mkdir(parents=True)
    (root / "annotations").mkdir()
    for split, names in (("train", names_train), ("val", names_val)):
        (root / f"ADE20K_object150_{split}.txt").write_text("\n".join(names) + "\n")
        for i, n in enumerate(names):
            H, W = 10 + i, 14 + 2 * i
            Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(root / "images" / n)
            lab = rng.integers(0, 151, (H, W)).astype(np.uint8)
            lab[0, :3] = (0, 1, 150)
            Image.fromarray(lab).save(root / "annotations" / (os.path.splitext(n)[0] + ".png"))


def test_ade20k_layout_split_files_sorted_order_and_zero_label_reduction(tmp_path):
    from PIL import Image
    from dinov3_jax.eval import ADE20KSegmentation, make_seg_dataset
    rng = np.random.default_rng(0)
    _ade_tree(tmp_path, ["b_2.jpg", "a_1.png", "c_3.jpg"], ["z.png", "y.png"], rng)
    ds = ADE20KSegmentation(tmp_path, "train")
    assert len(ds) == 3 and [os.path.basename(p) for p in ds.images] == ["a_1.png", "b_2.jpg", "c_3.jpg"]
    assert [os.path.basename(p) for p in ds.labels] == ["a_1.png", "b_2.png", "c_3.png"]
    img, lab = ds[1]
    assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3 and lab.dtype == np.uint8
    assert lab.shape == img.shape[:2]
    raw = np.asarray(Image.open(tmp_path / "annotations" / "b_2.png"))
    assert (lab[raw == 0] == 255).all() and (lab[raw > 0] == raw[raw > 0] - 1).all()
    assert lab[0, :3].tolist() == [255, 0, 149] and lab[lab != 255].max() <= 149
    val = make_seg_dataset(str(tmp_path), "val")
    assert isinstance(val, ADE20KSegmentation) and len(val) == 2 and os.path.basename(val.images[0]) == "y.png"
    with pytest.raises(ValueError):
        ADE20KSegmentation(tmp_path, "test")


def test_reduce_zero_label_keeps_255():
    from dinov3_jax.eval.datasets import reduce_zero_label
    assert reduce_zero_label(np.array([0, 1, 2, 150, 255], dtype=np.uint8)).tolist() == [255, 0, 1, 149, 255]


def test_seg_npz_dataset_and_its_errors(tmp_path):
    from dinov3_jax.eval import SegNpzDataset, make_seg_dataset
    imgs = np.zeros((3, 8, 12, 3), np.uint8)
    labs = np.full((3, 8, 12), 255, np.uint8)
    labs[1, :4] = 2
    np.savez(tmp_path / "ok.npz", images=imgs, labels=labs)
    ds = make_seg_dataset(str(tmp_path / "ok.npz"))
    assert isinstance(ds, SegNpzDataset) and len(ds) == 3
    im, lb = ds[1]
    assert im.shape == (8, 12, 3) and lb.dtype == np.uint8 and (lb[:4] == 2).all() and (lb[4:] == 255).all()
    for name, kw, msg in (("a", dict(images=imgs.astype(np.float32), labels=labs), "images must be uint8"),
                          ("b", dict(images=imgs[..., :2], labels=labs), "images must be uint8"),
                          ("c", dict(images=imgs, labels=labs.astype(np.int32)), "labels must be uint8"),
                          ("d", dict(images=imgs, labels=labs[:, :4]), "labels must be uint8")):
        np.savez(tmp_path / f"{name}.npz", **kw)
        with pytest.raises(ValueError, match=msg):
            SegNpzDataset(tmp_path / f"{name}.npz")


# ------------------------------------------------------------------------------------------------ config, flags
def test_defaults_carry_the_segmentation_block():
    from dinov3_jax.configs import get_default_config
    seg = get_default_config().evaluation.segmentation
    assert seg == {"train_dataset_path": "", "val_dataset_path": "", "num_classes": 150, "n_last_blocks": 1,
                   "batch_size": 16, "crop_size": 512, "iterations": 40000, "lr": 1e-3, "weight_decay": 1e-3,
                   "warmup_iterations": 1500, "num_workers": 8, "seed": 0}


def test_do_seg_eval_without_datasets_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_seg_eval
    assert do_seg_eval(get_default_config(), None, "training_9") == {}
    assert "nothing evaluated" in capsys.readouterr().out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_still_raises_naming_knn(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match="knn"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_seg_reaches_do_seg_eval_and_never_do_train(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_seg_eval", lambda config, model, header: calls.append((str(model), header)) or {"ok": 3})
    monkeypatch.setattr(train, "do_test", lambda *a, **k: pytest.fail("--eval seg must not run k-NN"))
    monkeypatch.setattr(train, "do_linear_eval", lambda *a, **k: pytest.fail("--eval seg must not run the linear probe"))
    monkeypatch.setattr(train, "do_train", lambda *a, **k: pytest.fail("--eval-only must not train"))
    ck = tmp_path / "ckpt" / "11"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 11, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "seg", "--output-dir", str(tmp_path)]) == {"ok": 3}
    assert calls == [(str(ck), "manual_12")]


# ------------------------------------------------------------------------------------------------ host draws
def _npz_seg(path, n, seed):
    rng = np.random.default_rng(seed)
    sizes = [(int(rng.integers(20, 60)), int(rng.integers(20, 60))) for _ in range(n)]
    H, W = max(s[0] for s in sizes), max(s[1] for s in sizes)
    np.savez(path, images=rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8),
             labels=rng.integers(0, 4, (n, H, W), dtype=np.uint8))


def test_host_draws_depend_on_seed_only_not_on_num_workers(tmp_path):
    from dinov3_jax.eval.datasets import SegNpzDataset
    from dinov3_jax.eval.linear import InfiniteBatchSampler
    from dinov3_jax.eval.segmentation import _pack_seg, sample_seg_boxes
    _npz_seg(tmp_path / "d.npz", 7, 0)
    ds = SegNpzDataset(tmp_path / "d.npz")

    def draws(workers, seed):
        loader = torch.utils.data.DataLoader(ds, batch_sampler=InfiniteBatchSampler(len(ds), 3, 5, seed),
                                             num_workers=workers, collate_fn=_pack_seg)
        aug = torch.Generator().manual_seed(seed + 1)
        out = []
        for flat, lab, desc in loader:
            out.append((flat.sum().item(), lab.sum().item(), desc.tolist(),
                        sample_seg_boxes(aug, desc[:, 1:].tolist(), 32).tolist()))
        return out

    a = draws(0, 4)
    assert a == draws(2, 4) and a != draws(0, 5)
    boxes = [b for _, _, _, bx in a for b in bx]
    assert any(b[4] for b in boxes) and not all(b[4] for b in boxes)


def test_seg_box_draws_scale_range_and_crop_placement():
    from dinov3_jax.eval.segmentation import sample_seg_box
    g = torch.Generator().manual_seed(0)
    for H, W in [(375, 500), (512, 683), (100, 40), (40, 100)]:
        for _ in range(50):
            rh, rw, top, left, flip = sample_seg_box(g, H, W, 64)
            s = min(rh, rw) / 64
            assert 0.5 - 0.05 <= s <= 2.0 + 0.05, (H, W, rh, rw)
            assert abs(rh / H - rw / W) <= 1.0 / min(H, W) + 1.0 / 64
            assert 0 <= top <= max(rh - 64, 0) and 0 <= left <= max(rw - 64, 0) and flip in (0, 1)
    # replayed by hand from the generator: scale, top, left, flip
    g1, g2 = torch.Generator().manual_seed(9), torch.Generator().manual_seed(9)
    s = torch.empty(1).uniform_(0.5, 2.0, generator=g2).item()
    rh, rw = int(300 * 64 * s / 300 + 0.5), int(500 * 64 * s / 300 + 0.5)
    top = torch.randint(0, max(rh - 64, 0) + 1, (1,), generator=g2).item()
    left = torch.randint(0, max(rw - 64, 0) + 1, (1,), generator=g2).item()
    flip = int(torch.rand(1, generator=g2).item() < 0.5)
    assert sample_seg_box(g1, 300, 500, 64) == (rh, rw, top, left, flip)


def test_eval_size_short_side_crop_long_side_patch_multiple():
    from dinov3_jax.eval.segmentation import eval_size
    assert eval_size(512, 683, 512, 16) == (512, 688)        # 683 -> 42.7 patches -> 43
    assert eval_size(683, 512, 512, 16) == (688, 512)
    assert eval_size(375, 500, 512, 16) == (512, 688)        # 682.7 -> 42.67 -> 43 patches
    assert eval_size(300, 300, 512, 16) == (512, 512)
    assert eval_size(100, 4000, 32, 16) == (32, 1280)


def test_schedule_warmup_then_linear_decay_to_zero():
    from dinov3_jax.eval.segmentation import seg_lr
    T, Wu = 100, 10
    lrs = [seg_lr(1e-3, t, T, Wu) for t in range(T)]
    assert lrs[0] == pytest.approx(1e-3 * 0.1 * 1.0) and lrs[9] == pytest.approx(1e-3 * 0.91)
    assert all(a < b for a, b in zip(lrs[:9], lrs[1:10]))
    assert all(a > b for a, b in zip(lrs[9:], lrs[10:])) and lrs[-1] == pytest.approx(1e-5)
    assert seg_lr(1e-3, T, T, Wu) == 0.0


def test_seg_metrics_against_oracle_and_by_hand():
    from dinov3_jax.eval.segmentation import seg_metrics
    conf = np.array([[5, 1, 0], [2, 3, 0], [0, 0, 0]])
    r = seg_metrics(conf)
    # class 0: 5 / (6 + 7 - 5) = 5/8; class 1: 3 / (5 + 4 - 3) = 1/2; class 2: empty union, left out
    assert r["mIoU"] == pytest.approx(100 * (5 / 8 + 1 / 2) / 2) and r["per_class_iou"][2] is None
    assert r["mAcc"] == pytest.approx(100 * (5 / 6 + 3 / 5) / 2) and r["aAcc"] == pytest.approx(100 * 8 / 11)
    rng = np.random.default_rng(0)
    big = rng.integers(0, 50, (7, 7))
    big[3] = 0
    big[:, 3] = 0
    want = seg_oracle.metrics(big)
    got = seg_metrics(big)
    for k in ("mIoU", "mAcc", "aAcc"):
        assert got[k] == pytest.approx(want[k], rel=1e-12)


# ------------------------------------------------------------------------------------------------ float64 oracle
def _frac_matrix(A):
    return [[Fraction(v).limit_denominator(1000) for v in row] for row in A]


def test_interp_matrix_hand_computed_2_to_4_3_to_7_5_to_11():
    F = Fraction
    assert _frac_matrix(seg_oracle.interp_matrix(4, 2)) == [[1, 0], [F(3, 4), F(1, 4)], [F(1, 4), F(3, 4)], [0, 1]]
    assert _frac_matrix(seg_oracle.interp_matrix(7, 3)) == [
        [1, 0, 0], [F(6, 7), F(1, 7), 0], [F(3, 7), F(4, 7), 0], [0, 1, 0], [0, F(4, 7), F(3, 7)],
        [0, F(1, 7), F(6, 7)], [0, 0, 1]]
    A = _frac_matrix(seg_oracle.interp_matrix(11, 5))
    want = [[1, 0, 0, 0, 0], [F(9, 11), F(2, 11), 0, 0, 0], [F(4, 11), F(7, 11), 0, 0, 0],
            [0, F(10, 11), F(1, 11), 0, 0], [0, F(5, 11), F(6, 11), 0, 0], [0, 0, 1, 0, 0],
            [0, 0, F(6, 11), F(5, 11), 0], [0, 0, F(1, 11), F(10, 11), 0], [0, 0, 0, F(7, 11), F(4, 11)],
            [0, 0, 0, F(2, 11), F(9, 11)], [0, 0, 0, 0, 1]]
    assert A == want


def test_xent_and_confusion_hand_computed_2x2_to_4x4():
    # two classes; class 1 has logit 4 at cell (0, 0) only, class 0 is 0 everywhere: the upsampled class-1 logit at
    # (y, x) is 4 * a[y] * a[x] with a = (1, 3/4, 1/4, 0)
    L = np.zeros((1, 2, 2, 2))
    L[0, 0, 0, 1] = 4.0
    lab = np.zeros((1, 4, 4), np.uint8)
    lab[0, 0, 0] = 1
    lab[0, 3, :] = 255
    a = [1.0, 0.75, 0.25, 0.0]
    total, n = 0.0, 0
    for y in range(3):
        for x in range(4):
            z1 = 4 * a[y] * a[x]
            total += np.log1p(np.exp(z1)) - (z1 if lab[0, y, x] == 1 else 0.0)
            n += 1
    loss, grad, count = seg_oracle.xent(L, lab)
    assert count == 12 and loss == pytest.approx(total / n, rel=1e-14)
    # the gradient of a cell is the adjoint: sum over pixels of its weight times (p - onehot) / n
    g00 = 0.0
    for y in range(3):
        for x in range(4):
            z1 = 4 * a[y] * a[x]
            p1 = 1 / (1 + np.exp(-z1))
            g00 += a[y] * a[x] * (p1 - (1.0 if lab[0, y, x] == 1 else 0.0)) / n
    assert grad[0, 0, 0, 1] == pytest.approx(g00, rel=1e-13) and grad[0, 0, 0, 0] == pytest.approx(-g00, rel=1e-13)
    conf, gap = seg_oracle.confusion(L, lab, 2)
    # argmax is 1 where z1 > 0, i.e. y, x in {0, 1, 2}: label 1 only at (0, 0), label 0 at the 8 others of those and
    # at (y, 3) for the 3 rows; row 3 is ignored
    assert conf.tolist() == [[3, 8], [0, 1]]


def test_oracle_matches_torch_float64_interpolate_cross_entropy_3x5_to_7x11():
    import torch.nn.functional as Fn
    g = torch.Generator().manual_seed(0)
    for B, h, w, Hl, Wl, C in ((2, 3, 5, 7, 11, 4), (1, 2, 2, 4, 4, 3), (2, 6, 4, 3, 5, 5)):
        L = torch.randn(B, h, w, C, generator=g, dtype=torch.float64) * 3
        lab = torch.randint(0, C, (B, Hl, Wl), generator=g)
        lab[0, 0] = 255
        Lt = L.clone().requires_grad_(True)
        up = Fn.interpolate(Lt.permute(0, 3, 1, 2), size=(Hl, Wl), mode="bilinear", align_corners=False)
        ref = Fn.cross_entropy(up, lab, ignore_index=255)
        ref.backward()
        loss, grad, n = seg_oracle.xent(L.numpy(), lab.numpy().astype(np.uint8))
        assert n == int((lab != 255).sum())
        assert loss == pytest.approx(ref.item(), rel=1e-12)
        assert np.allclose(grad, Lt.grad.numpy(), rtol=1e-10, atol=1e-14)
        assert np.allclose(seg_oracle.upsample(L.numpy(), Hl, Wl), up.detach().permute(0, 2, 3, 1).numpy(), atol=1e-12)
        conf, _ = seg_oracle.confusion(L.numpy(), lab.numpy().astype(np.uint8), C)
        pred = up.argmax(1)
        keep = lab != 255
        want = torch.bincount(lab[keep] * C + pred[keep], minlength=C * C).reshape(C, C)
        assert conf.tolist() == want.tolist()


# ------------------------------------------------------------------------------------------------ ptxas
def test_new_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    seen = set()
    for src in ("seg.cu", "knn.cu"):
        cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", src), "-o", str(tmp_path / "x.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                           r"(\d+) bytes spill loads", r.stderr)
        for name, stack, st, ld in props:
            if "seg_" in name:
                seen.add(name)
                assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # 8 class-chunk instances of each per-pixel kernel, 5 other seg.cu kernels, 2 crop instances
    assert len(seen) == 8 + 8 + 5 + 2, sorted(seen)
