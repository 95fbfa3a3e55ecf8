"""Video object segmentation without a GPU: the float64 oracle (tests/video_oracle.py) against a torch restatement of
DINO's label_propagation and hand-computed J / F cases, the Decay bins, the frame resize rule, the DAVIS and .npz
layouts, the `evaluation.video` block, the --eval video flags, and what ptxas makes of csrc/video.cu."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import video_oracle


# ------------------------------------------------------------------------------------------------ propagation
def _dino_label_propagation(target, ctx_feats, ctx_labels, h, w, radius, topk, temperature):
    """DINO's label_propagation, restated literally in torch float64: a dense affinity with the neighbourhood mask
    applied, topk over all sources, aff[aff < kth] = 0, column normalisation and segs @ aff."""
    n = len(ctx_feats)
    feat_tar = torch.as_tensor(target, dtype=torch.float64)                         # [P, D]
    feat_src = torch.stack([torch.as_tensor(f, dtype=torch.float64) for f in ctx_feats]).transpose(1, 2)
    aff = torch.exp(torch.bmm(feat_tar[None].expand(n, -1, -1), feat_src) / temperature)     # [n, P_tar, P_src]
    mask = torch.zeros(h, w, h, w, dtype=torch.float64)
    for i in range(h):
        for j in range(w):
            for p in range(2 * radius + 1):
                for q in range(2 * radius + 1):
                    if 0 <= i - radius + p < h and 0 <= j - radius + q < w:
                        mask[i, j, i - radius + p, j - radius + q] = 1
    aff = aff * mask.reshape(h * w, h * w)[None]
    aff = aff.transpose(2, 1).reshape(-1, h * w)                                     # [n * P_src, P_tar]
    tk_val, _ = torch.topk(aff, dim=0, k=topk)
    tk_val_min, _ = torch.min(tk_val, dim=0)
    aff[aff < tk_val_min] = 0
    aff = aff / torch.sum(aff, keepdim=True, axis=0)
    segs = torch.cat([torch.as_tensor(l, dtype=torch.float64) for l in ctx_labels]).T   # [C, n * P_src]
    return (segs @ aff).T.numpy()


def _features(rng, n, P, D):
    f = rng.normal(size=(n, P, D))
    return f / np.linalg.norm(f, axis=-1, keepdims=True)


@pytest.mark.parametrize("case", [(5, 7, 2, 3, 5, 4, "window smaller than the grid"),
                                  (4, 3, 5, 2, 3, 3, "window covering the grid"),
                                  (6, 5, 1, 4, 1, 5, "k = 1"),
                                  (3, 4, 9, 3, 32, 2, "k above the candidate count")], ids=lambda c: c[-1])
def test_oracle_propagate_equals_dino_label_propagation(case):
    h, w, radius, n_ctx, k, C, _ = case
    rng = np.random.default_rng(h * w + k)
    P = h * w
    f = _features(rng, n_ctx + 1, P, 16)
    labs = [rng.random((P, C)) for _ in range(n_ctx)]
    got, kth, _ = video_oracle.propagate(f[0], list(f[1:]), labs, h, w, radius, k, 0.1)
    want = _dino_label_propagation(f[0], list(f[1:]), labs, h, w, radius, k, 0.1)
    assert np.allclose(got, want, rtol=1e-12, atol=1e-14)
    if radius >= max(h, w):
        assert np.isfinite(kth).all() == (n_ctx * P >= k)


def test_oracle_propagate_keeps_every_tie_at_the_threshold():
    # two context frames with identical features: every score appears twice, so the k-th largest always ties
    h, w, k = 4, 5, 3
    rng = np.random.default_rng(3)
    f = _features(rng, 2, h * w, 8)
    labs = [np.eye(3)[rng.integers(0, 3, h * w)], np.eye(3)[rng.integers(0, 3, h * w)]]
    got, kth, nxt = video_oracle.propagate(f[0], [f[1], f[1]], labs, h, w, 1, k, 0.1)
    want = _dino_label_propagation(f[0], [f[1], f[1]], labs, h, w, 1, k, 0.1)
    assert np.allclose(got, want, rtol=1e-12, atol=1e-14)
    # k = 3 of pairs: the 3rd and 4th largest are one pair, so four candidates are kept, not three
    assert np.array_equal(kth, nxt)
    q = 7
    cand = video_oracle.window_candidates(q, h, w, 1, 2)
    x = np.array([f[0][q] @ f[1][s] for _, s in cand])
    keep = x >= np.sort(x)[::-1][k - 1]
    assert keep.sum() == 4
    a = np.exp(x[keep] / 0.1)
    rows = np.stack([labs[c][s] for (c, s), kp in zip(cand, keep) if kp])
    assert np.allclose(got[q], (a / a.sum()) @ rows)


# ------------------------------------------------------------------------------------------------ J and F
def _square(H, W, y, x, n, k=1):
    m = np.zeros((H, W), np.uint8)
    m[y:y + n, x:x + n] = k
    return m


def test_j_and_f_of_a_square_shifted_by_one_pixel():
    gt, pred = _square(40, 50, 10, 10, 8), _square(40, 50, 10, 11, 8)
    J, F = video_oracle.j_and_f(pred, gt, 1)
    assert J[0] == pytest.approx(56 / 72)                    # 8 x 7 shared of 8 x 9
    # the shift is one pixel, within the radius ceil(0.008 * 64.03) = 1, so every boundary pixel matches
    c = video_oracle.jf_counts(pred, gt, 1, 1)[0]
    assert c[2] == c[3] == c[4] == c[5] > 0 and F[0] == 1.0
    assert video_oracle.radius(40, 50) == 1
    # a two-pixel shift at radius 1: only part of the boundaries match, and by hand
    pred2 = _square(40, 50, 10, 12, 8)
    b_gt, b_pr = video_oracle.boundary(gt == 1), video_oracle.boundary(pred2 == 1)
    near = lambda b: np.array([[b[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2][np.array(
        [[dy * dy + dx * dx <= 1 for dx in range(max(x - 1, 0) - x, min(x + 2, 50) - x)]
         for dy in range(max(y - 1, 0) - y, min(y + 2, 40) - y)])].any() for x in range(50)] for y in range(40)])
    P_ = (b_pr & near(b_gt)).sum() / b_pr.sum()
    R_ = (b_gt & near(b_pr)).sum() / b_gt.sum()
    assert 0 < P_ < 1 and 0 < R_ < 1
    assert video_oracle.j_and_f(pred2, gt, 1)[1][0] == pytest.approx(2 * P_ * R_ / (P_ + R_))


def test_boundary_of_a_square_by_hand():
    b = video_oracle.boundary(_square(6, 7, 2, 2, 2) == 1)
    want = np.zeros((6, 7), bool)
    want[1, 1:4] = True                 # the row above, from the upper-left diagonal neighbour on
    want[2:4, 1] = True                 # the column to the left
    want[2, 3] = want[3, 2] = want[3, 3] = True      # the square's pixels next to a 0 on the right, below or diagonally
    assert np.array_equal(b, want), b.astype(int)
    # the last row compares only with the right neighbour, the last column only with the lower one, the corner is 0
    m = np.zeros((3, 3), bool)
    m[2, 1] = m[1, 2] = True
    b = video_oracle.boundary(m)
    assert b[2].tolist() == [True, True, False] and b[:, 2].tolist() == [True, True, False]


def test_j_and_f_of_empty_masks():
    gt, empty = _square(30, 30, 5, 5, 6), np.zeros((30, 30), np.uint8)
    J, F = video_oracle.j_and_f(empty, gt, 1)            # empty prediction: P = 1, R = 0
    assert (J[0], F[0]) == (0.0, 0.0)
    J, F = video_oracle.j_and_f(gt, empty, 1)            # empty GT: P = 0, R = 1
    assert (J[0], F[0]) == (0.0, 0.0)
    J, F = video_oracle.j_and_f(empty, empty, 1)         # both empty: J = 1, P = R = 1
    assert (J[0], F[0]) == (1.0, 1.0)
    from dinov3_jax.eval.video import jf_from_counts
    c = np.stack([video_oracle.jf_counts(a, b, 1, 1) for a, b in ((empty, gt), (gt, empty), (empty, empty))])
    J, F = jf_from_counts(c)
    assert J[:, 0].tolist() == [0.0, 0.0, 1.0] and F[:, 0].tolist() == [0.0, 0.0, 1.0]


def test_void_pixels_are_left_out_of_j_and_f():
    gt = _square(30, 30, 5, 5, 6)
    pred = _square(30, 30, 5, 5, 6)
    pred[5:11, 11:14] = 1                                 # 18 extra predicted pixels ...
    gt_void = gt.copy()
    gt_void[5:11, 11:14] = 255                            # ... all void
    J, F = video_oracle.j_and_f(pred, gt_void, 1)
    assert J[0] == 1.0 and F[0] == 1.0
    J2, _ = video_oracle.j_and_f(pred, gt, 1)
    assert J2[0] == pytest.approx(36 / 54)


def test_disk_radius_at_480p():
    from dinov3_jax.eval.video import boundary_radius
    assert boundary_radius(480, 854) == video_oracle.radius(480, 854) == 8
    assert video_oracle.disk(8).sum() == sum(2 * int(np.floor(np.sqrt(64 - y * y))) + 1 for y in range(-8, 9))


def test_jf_counts_agree_with_the_package_formula_on_random_masks():
    from dinov3_jax.eval.video import jf_from_counts
    rng = np.random.default_rng(0)
    gt = rng.integers(0, 3, (20, 30)).astype(np.uint8)
    gt[rng.random((20, 30)) < 0.1] = 255
    pred = rng.integers(0, 3, (20, 30)).astype(np.uint8)
    J, F = jf_from_counts(video_oracle.jf_counts(pred, gt, 2, video_oracle.radius(20, 30))[None])
    J2, F2 = video_oracle.j_and_f(pred, gt, 2)
    assert np.allclose(J[0], J2) and np.allclose(F[0], F2)


# ------------------------------------------------------------------------------------------------ statistics
def test_decay_bins_share_one_frame():
    from dinov3_jax.eval.video import decay_bins, statistics
    assert decay_bins(3) == [(0, 2), (1, 2), (1, 3), (2, 3)]
    assert decay_bins(4) == [(0, 2), (1, 3), (2, 3), (2, 4)]
    assert decay_bins(10) == [(0, 3), (2, 6), (5, 8), (7, 10)]
    v = np.array([0.9, 0.8, 0.4, 0.3, 0.7, 0.6, 0.2, 0.1, 0.5, 0.0])
    s = statistics(v)
    assert s["Mean"] == pytest.approx(v.mean()) and s["Recall"] == pytest.approx(0.4)     # 0.5 itself is not > 0.5
    assert s["Decay"] == pytest.approx(v[0:3].mean() - v[7:10].mean())
    assert statistics([1.0, 0.5, 0.25])["Decay"] == pytest.approx(0.75 - 0.25)


# ------------------------------------------------------------------------------------------------ resize and labels
def test_frame_resize_rule():
    from dinov3_jax.eval.video import video_size
    assert video_size(480, 854, 480, 16) == (480, 832)         # landscape
    assert video_size(854, 480, 480, 16) == (832, 480)         # portrait
    assert video_size(480, 640, 480, 16) == (480, 640)         # already a multiple of 64
    assert video_size(480, 480, 480, 8) == (480, 448)         # the long side rounds down even when equal
    with pytest.raises(ValueError, match="patch size"):
        video_size(480, 854, 480, 14)


def test_first_frame_labels_read_by_nearest_exact():
    from PIL import Image
    from dinov3_jax.eval.video import first_frame_labels
    rng = np.random.default_rng(1)
    m = rng.integers(0, 4, (37, 53)).astype(np.uint8)
    m[rng.random(m.shape) < 0.1] = 255
    oh = first_frame_labels(m, 5, 7, 4)
    small = np.asarray(Image.fromarray(m).resize((7, 5), Image.NEAREST)).astype(np.int64)
    small[small == 255] = 0
    assert np.array_equal(oh.argmax(1).reshape(5, 7), small) and (oh.sum(1) == 1).all()
    t = torch.nn.functional.interpolate(torch.from_numpy(m)[None, None].float(), size=(5, 7), mode="nearest-exact")
    t = t[0, 0].long()
    t[t == 255] = 0
    assert np.array_equal(t.numpy(), small)


# ------------------------------------------------------------------------------------------------ datasets
def _davis_tree(root, seqs, rng, sizes=None):
    from PIL import Image
    from dinov3_jax.eval.video import default_palette
    (root / "ImageSets" / "2017").mkdir(parents=True)
    (root / "ImageSets" / "2017" / "val.txt").write_text("\n".join(seqs) + "\n")
    out = {}
    for i, s in enumerate(seqs):
        H, W = (sizes or {}).get(s, (12 + i, 20))
        fd, ad = root / "JPEGImages" / "480p" / s, root / "Annotations" / "480p" / s
        fd.mkdir(parents=True)
        ad.mkdir(parents=True)
        masks = []
        for t in range(3 + i):
            Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(fd / f"{t:05d}.jpg")
            m = rng.integers(0, 3, (H, W)).astype(np.uint8)
            m[0, 0] = 255
            im = Image.fromarray(m, mode="P")
            im.putpalette(default_palette())
            im.save(ad / f"{t:05d}.png")
            masks.append(m)
        out[s] = np.stack(masks)
    return out


def test_davis_layout(tmp_path):
    from dinov3_jax.eval import DavisDataset, make_video_dataset
    from dinov3_jax.eval.video import default_palette
    masks = _davis_tree(tmp_path, ["bear", "car"], np.random.default_rng(0))
    ds = make_video_dataset(str(tmp_path))
    assert isinstance(ds, DavisDataset) and len(ds) == 2 and ds.sequences == ["bear", "car"]
    item = ds[1]
    assert item["name"] == "car" and item["frames"].shape == (4, 13, 20, 3) and item["frames"].dtype == np.uint8
    assert np.array_equal(item["masks"], masks["car"]) and item["palette"][:768] == default_palette()


def test_davis_errors_name_the_path(tmp_path):
    from PIL import Image
    from dinov3_jax.eval import DavisDataset
    with pytest.raises(FileNotFoundError, match="val.txt"):
        DavisDataset(tmp_path)
    _davis_tree(tmp_path, ["a", "b"], np.random.default_rng(1))
    (tmp_path / "ImageSets" / "2017" / "val.txt").write_text("a\nmissing\n")
    with pytest.raises(FileNotFoundError, match="missing"):
        DavisDataset(tmp_path)
    (tmp_path / "ImageSets" / "2017" / "val.txt").write_text("a\nb\n")
    os.remove(tmp_path / "Annotations" / "480p" / "b" / "00001.png")
    with pytest.raises(ValueError, match=str(tmp_path / "Annotations" / "480p" / "b")):
        DavisDataset(tmp_path)
    Image.fromarray(np.zeros((5, 5), np.uint8), mode="P").save(tmp_path / "Annotations" / "480p" / "b" / "00001.png")
    ds = DavisDataset(tmp_path)
    with pytest.raises(ValueError, match="00001.png.*does not match"):
        ds[1]


def test_video_npz_dataset_and_its_errors(tmp_path):
    from dinov3_jax.eval import VideoNpzDataset, make_video_dataset
    frames = np.arange(7 * 6 * 8 * 3, dtype=np.uint8).reshape(7, 6, 8, 3)
    masks = (np.arange(7 * 6 * 8) % 3).astype(np.uint8).reshape(7, 6, 8)
    np.savez(tmp_path / "v.npz", frames=frames, masks=masks, sequence_starts=np.array([0, 3]))
    ds = make_video_dataset(str(tmp_path / "v.npz"))
    assert isinstance(ds, VideoNpzDataset) and len(ds) == 2
    s = ds[1]
    assert s["name"] == "00001" and np.array_equal(s["frames"], frames[3:]) and np.array_equal(s["masks"], masks[3:])
    for name, kw, msg in (("a", dict(frames=frames.astype(np.float32), masks=masks), "frames must be uint8"),
                          ("b", dict(frames=frames, masks=masks[:, :5]), "masks must be uint8"),
                          ("c", dict(frames=frames, masks=masks.astype(np.int32)), "masks must be uint8")):
        np.savez(tmp_path / f"{name}.npz", sequence_starts=np.array([0]), **kw)
        with pytest.raises(ValueError, match=msg):
            VideoNpzDataset(tmp_path / f"{name}.npz")
    for starts in ([1], [0, 0], [0, 7]):
        np.savez(tmp_path / "d.npz", frames=frames, masks=masks, sequence_starts=np.array(starts))
        with pytest.raises(ValueError, match="sequence_starts"):
            VideoNpzDataset(tmp_path / "d.npz")


# ------------------------------------------------------------------------------------------------ config, flags
def test_defaults_carry_the_video_block():
    from dinov3_jax.configs import get_default_config
    assert get_default_config().evaluation.video == {
        "dataset_path": "", "n_last_frames": 7, "size_mask_neighborhood": 12, "topk": 5, "temperature": 0.1,
        "short_side": 480, "batch_size": 16, "num_workers": 4, "save_masks": False}


def test_do_video_eval_without_dataset_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_video_eval
    assert do_video_eval(get_default_config(), None, "training_9") == {}
    assert "nothing evaluated" in capsys.readouterr().out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_still_raises_naming_knn_and_video(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match="knn.*--eval video"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_video_reaches_do_video_eval_and_nothing_else(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_video_eval",
                        lambda config, model, header: calls.append((str(model), header)) or {"ok": 5})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval", "do_train"):
        monkeypatch.setattr(train, name, lambda *a, _n=name, **k: pytest.fail(f"--eval-only --eval video ran {_n}"))
    ck = tmp_path / "ckpt" / "8"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 8, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "video", "--output-dir", str(tmp_path)]) == {"ok": 5}
    assert calls == [(str(ck), "manual_9")]


# ------------------------------------------------------------------------------------------------ ptxas
def test_video_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert "video.cu" in b.SOURCES
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", "video.cu"), "-o",
                                       str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    seen = set()
    for name, stack, st, ld in props:
        if "video_" in name:
            seen.add(name)
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # resize, propagation, min / max, min / max merge, label map, J and F counts
    assert len(seen) == 6, sorted(seen)
