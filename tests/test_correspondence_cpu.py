"""Keypoint correspondence without a GPU: the float64 oracle (tests/correspondence_oracle.py) on a hand-computed case,
the closed form the argmax kernel evaluates (per-patch Gram and the 4-tap blend of the patch similarities) against the
materialised cosine, the keypoint mapping, the PCK averaging, the SPair-71k and .npz layouts, the
`evaluation.correspondence` block, the --eval correspondence flags, and what ptxas makes of csrc/correspondence.cu."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import correspondence_oracle as oracle


# ------------------------------------------------------------------------------------------------ oracle by hand
def test_oracle_on_a_2x2_map_at_4x4_by_hand():
    # corners e0, e1 (top) and e2, e0 + e2 (bottom) in 3 dimensions, S = 4: source positions max((d + 0.5) / 2 - 0.5, 0)
    # = 0, 0.25, 0.75, 1 (the last clamped to the last cell), so rows / columns 0 and 3 are pure cells
    f = np.array([[[1, 0, 0], [0, 1, 0]], [[0, 0, 1], [1, 0, 1]]], dtype=np.float64)
    U = oracle.upsample(f, (4, 4)).numpy()
    assert np.allclose(U[0, 0], f[0, 0]) and np.allclose(U[3, 3], f[1, 1]) and np.allclose(U[0, 3], f[0, 1])
    assert np.allclose(U[0, 1], 0.75 * f[0, 0] + 0.25 * f[0, 1])
    assert np.allclose(U[2, 1], 0.25 * (0.75 * f[0, 0] + 0.25 * f[0, 1]) + 0.75 * (0.75 * f[1, 0] + 0.25 * f[1, 1]))
    # q = e1: cosine 1 exactly on the 2 x 2 block of pixels that read only cell (0, 1), the lowest index wins
    xy, cos = oracle.match(np.array([[0.0, 1.0, 0.0]]), f, (4, 4))
    assert xy.tolist() == [[3, 0]] and cos[0, 3] == 1.0 and cos[0].max() == 1.0
    assert (cos[0].reshape(4, 4) == 1.0).sum() == 1
    # q = e0: ties at cosine 1 on pixel (0, 0) only; q = e0 + e2: the pure corner (3, 3)
    assert oracle.match(np.array([[1.0, 0, 0]]), f, (4, 4))[0].tolist() == [[0, 0]]
    assert oracle.match(np.array([[1.0, 0, 1]]), f, (4, 4))[0].tolist() == [[3, 3]]
    # an exact tie: a constant map gives every pixel the same cosine, pixel 0 wins
    c = np.ones((2, 2, 3))
    xy, cos = oracle.match(np.array([[1.0, 2.0, 0.5]]), c, (4, 4))
    assert xy.tolist() == [[0, 0]] and np.ptp(cos) == 0
    # a zero descriptor: cosine 0 everywhere, pixel 0
    assert oracle.match(np.zeros((1, 3)), f, (4, 4))[0].tolist() == [[0, 0]]


# ------------------------------------------------------------------------------------------------ closed form
def _src(d, n, S):
    return max((d + 0.5) * n / S - 0.5, 0.0)


def closed_form_cosines(q, feat, out_hw):
    """float64 [K, H * W]: the argmax kernel's algebra: the per-patch Gram (norm; right, lower, lower-right, lower-left
    dots), the corner pairs read from it with coinciding corners at the last row / column substituted (and their
    weights folded into one), and <q, U> = sum_a w_a <q, f_a>."""
    h, w, D = feat.shape
    H, W = out_hw
    s = np.asarray(q, np.float64) @ feat.reshape(-1, D).T                    # [K, h w]
    gram = np.zeros((h * w, 5))
    for i in range(h):
        for j in range(w):
            f = feat[i, j]
            gram[i * w + j] = [f @ f, f @ feat[i, j + 1] if j + 1 < w else 0.0,
                               f @ feat[i + 1, j] if i + 1 < h else 0.0,
                               f @ feat[i + 1, j + 1] if i + 1 < h and j + 1 < w else 0.0,
                               f @ feat[i + 1, j - 1] if i + 1 < h and j > 0 else 0.0]
    qn = np.linalg.norm(q, axis=1)
    out = np.zeros((len(s), H * W))
    for y in range(H):
        fy = _src(y, h, H)
        ty = int(fy)
        y1 = min(ty + 1, h - 1)
        ly = fy - ty if y1 != ty else 0.0                                    # coinciding rows folded into one
        for x in range(W):
            fx = _src(x, w, W)
            tx = int(fx)
            x1 = min(tx + 1, w - 1)
            lx = fx - tx if x1 != tx else 0.0
            A, B, C, Dd = ty * w + tx, ty * w + x1, y1 * w + tx, y1 * w + x1
            col1, row1 = x1 == tx, y1 == ty
            AA, BB, CC, DD = gram[A, 0], gram[B, 0], gram[C, 0], gram[Dd, 0]
            AB = AA if col1 else gram[A, 1]
            AC = AA if row1 else gram[A, 2]
            AD = AB if row1 else (AC if col1 else gram[A, 3])
            BD = BB if row1 else gram[B, 2]
            CD = CC if col1 else gram[C, 1]
            BC = AC if col1 else (AB if row1 else gram[B, 4])
            wA, wB, wC, wD = (1 - ly) * (1 - lx), (1 - ly) * lx, ly * (1 - lx), ly * lx
            n2 = (wA * wA * AA + wB * wB * BB + wC * wC * CC + wD * wD * DD
                  + 2 * (wA * (wB * AB + wC * AC + wD * AD) + wB * (wC * BC + wD * BD) + wC * wD * CD))
            num = wA * s[:, A] + wB * s[:, B] + wC * s[:, C] + wD * s[:, Dd]
            out[:, y * W + x] = num / (qn * np.sqrt(max(n2, 0.0)))
    return out


@pytest.mark.parametrize("case", [(3, 5, 24, 40), (4, 1, 32, 8), (1, 6, 5, 48), (5, 9, 80, 144), (2, 2, 7, 9),
                                  (7, 7, 112, 112)], ids=lambda c: f"{c[0]}x{c[1]}_to_{c[2]}x{c[3]}")
def test_closed_form_equals_the_materialised_cosine(case):
    h, w, H, W = case
    rng = np.random.default_rng(h * 10 + w)
    feat = rng.normal(size=(h, w, 8))
    q = rng.normal(size=(3, 8))
    want = oracle.cosines(q, feat, (H, W))
    got = closed_form_cosines(q, feat, (H, W))
    assert np.abs(got - want).max() < 1e-12


# ------------------------------------------------------------------------------------------------ keypoints
def test_keypoint_mapping_identity_clamping_and_back():
    from dinov3_jax.eval.correspondence import back_map, keypoint_pixels
    u = np.array([[0, 0], [5, 7], [511, 511], [100.4, 200.6]])
    assert np.array_equal(keypoint_pixels(u, 512, 512, 512), np.floor(u + 0.5).astype(np.int64))
    assert np.array_equal(back_map(keypoint_pixels(u[:3], 512, 512, 512), 512, 512, 512), u[:3])
    # clamping at both edges: beyond the image on either side lands on the first / last pixel
    out = keypoint_pixels(np.array([[-3.0, -0.9], [700.0, 399.6], [639.4, 0.0]]), 640, 400, 512)
    assert out.tolist() == [[0, 0], [511, 511], [511, 0]]
    # downscaling: u = 10 in 640 wide at S = 512 -> floor(10.5 * 0.8) = 8; y = 20 in 400 -> floor(20.5 * 1.28) = 26
    assert keypoint_pixels(np.array([[10.0, 20.0]]), 640, 400, 512).tolist() == [[8, 26]]
    assert np.array_equal(keypoint_pixels(np.array([[10.0, 20.0]]), 640, 400, 512),
                          np.stack([oracle.keypoint_pixel(10.0, 640, 512), oracle.keypoint_pixel(20.0, 400, 512)])[None])
    # the back-mapping: pixel centres, (x + 0.5) W / S - 0.5
    assert np.allclose(back_map(np.array([[8, 26]]), 640, 400, 512), [[10.125, 20.203125]])
    assert np.allclose(back_map(np.array([[8, 26]]), 640, 400, 512),
                       [[oracle.back_map(8, 640, 512), oracle.back_map(26, 400, 512)]])


# ------------------------------------------------------------------------------------------------ PCK
def test_pck_threshold_averaging_and_categories():
    from dinov3_jax.eval.correspondence import pck_scores
    box = [0.0, 0.0, 100.0, 40.0]                        # max side 100: alpha 0.1 -> 10 pixels
    trg = np.array([[50.0, 20.0], [10.0, 10.0], [0.0, 0.0]])
    pred = trg + np.array([[6.0, 8.0], [10.0, 0.0], [10.0, 0.5]])        # distances 10 (exactly), 10, 10.01
    s = pck_scores([(pred, trg, box)], [0.1])
    assert s["PCK@0.1"] == pytest.approx(2 / 3) and s["PCK-image@0.1"] == pytest.approx(2 / 3)
    # unequal keypoint counts: pair A 1 of 1 correct, pair B 1 of 4 -> per point 2 / 5, per image (1 + 1 / 4) / 2
    a = (np.array([[0.0, 0.0]]), np.array([[0.0, 0.0]]), box)
    tb = np.zeros((4, 2))
    b = (tb + np.array([[0.0, 0.0], [50.0, 0.0], [50.0, 0.0], [50.0, 0.0]]), tb, box)
    s = pck_scores([a, b], [0.01, 0.1])
    assert s["PCK@0.1"] == pytest.approx(2 / 5) and s["PCK-image@0.1"] == pytest.approx(0.625)
    assert s["PCK@0.01"] == pytest.approx(2 / 5)
    # the oracle's statement agrees, and splits by category
    o = oracle.pck([a + ("cat",), b + ("dog",)], [0.1])
    assert o["PCK@0.1"] == pytest.approx(2 / 5) and o["PCK-image@0.1"] == pytest.approx(0.625)
    assert o["categories"]["cat"]["PCK@0.1"] == 1.0 and o["categories"]["dog"]["PCK@0.1"] == 0.25


# ------------------------------------------------------------------------------------------------ datasets
def _spair_tree(root, rng, pairs):
    """root/JPEGImages/<cat>/<name>.jpg and root/PairAnnotation/test/<id>.json for pairs [(id, cat, src, trg, n)]."""
    from PIL import Image
    sizes = {}
    for pid, cat, src, trg, n in pairs:
        for im in (src, trg):
            d = root / "JPEGImages" / cat
            d.mkdir(parents=True, exist_ok=True)
            if (cat, im) not in sizes:
                sizes[(cat, im)] = (20 + len(sizes), 30)
                Image.fromarray(rng.integers(0, 256, sizes[(cat, im)] + (3,), dtype=np.uint8)).save(d / im)
        a = {"src_imname": src, "trg_imname": trg, "category": cat, "src_kps": rng.random((n, 2)).tolist(),
             "trg_kps": rng.random((n, 2)).tolist(), "trg_bndbox": [1, 2, 11, 22], "src_imsize": [30, 20, 3]}
        d = root / "PairAnnotation" / "test"
        d.mkdir(parents=True, exist_ok=True)
        (d / f"{pid}.json").write_text(json.dumps(a))
    return sizes


def test_spair_layout(tmp_path):
    from dinov3_jax.eval import SPairDataset, make_correspondence_dataset
    rng = np.random.default_rng(0)
    _spair_tree(tmp_path, rng, [("0002-a-b:cat", "cat", "a.jpg", "b.jpg", 3), ("0001-b-c:cat", "cat", "b.jpg", "c.jpg", 2),
                                ("0003-a-a:dog", "dog", "a.jpg", "a.jpg", 1)])
    ds = make_correspondence_dataset(str(tmp_path))
    assert isinstance(ds, SPairDataset) and len(ds) == 3
    # sorted file names: 0001 first; images indexed in first-seen order, (category, name) distinct
    assert [p["category"] for p in ds.pairs] == ["cat", "cat", "dog"]
    assert ds.images == [str(tmp_path / "JPEGImages" / c / n) for c, n in
                         (("cat", "b.jpg"), ("cat", "c.jpg"), ("cat", "a.jpg"), ("dog", "a.jpg"))]
    assert (ds[0]["src"], ds[0]["trg"], ds[1]["src"], ds[1]["trg"], ds[2]["src"], ds[2]["trg"]) == (0, 1, 2, 0, 3, 3)
    assert ds[1]["src_kps"].shape == (3, 2) and ds[1]["trg_bbox"] == [1.0, 2.0, 11.0, 22.0]
    im = ds.load_image(1)
    assert im.dtype == np.uint8 and im.shape[2] == 3


def test_spair_errors_name_the_file_and_field(tmp_path):
    from dinov3_jax.eval import SPairDataset
    with pytest.raises(FileNotFoundError, match="PairAnnotation"):
        SPairDataset(tmp_path)
    rng = np.random.default_rng(1)
    _spair_tree(tmp_path, rng, [("p1", "cat", "a.jpg", "b.jpg", 2)])
    path = tmp_path / "PairAnnotation" / "test" / "p1.json"
    good = json.loads(path.read_text())
    for edit, exc, msg in ((lambda a: a.pop("trg_bndbox"), ValueError, "p1.json: field 'trg_bndbox' is missing"),
                           (lambda a: a.pop("category"), ValueError, "p1.json: field 'category'"),
                           (lambda a: a.update(trg_kps=a["trg_kps"][:1]), ValueError, "p1.json: field 'trg_kps'"),
                           (lambda a: a.update(src_kps=[[1, 2, 3]]), ValueError, "p1.json: field 'src_kps'"),
                           (lambda a: a.update(trg_bndbox=[1, 2]), ValueError, "p1.json: field 'trg_bndbox'"),
                           (lambda a: a.update(trg_imname="zz.jpg"), FileNotFoundError, "p1.json: trg_imname.*zz.jpg")):
        a = dict(good)
        edit(a)
        path.write_text(json.dumps(a))
        with pytest.raises(exc, match=msg):
            SPairDataset(tmp_path)


def _npz(path, **over):
    rng = np.random.default_rng(2)
    f = dict(images=rng.integers(0, 256, (3, 10, 12, 3), dtype=np.uint8), pairs=np.array([[0, 1], [2, 2]]),
             src_kps=rng.random((2, 4, 2)) * 10, trg_kps=rng.random((2, 4, 2)) * 10, n_kps=np.array([4, 2]),
             trg_bbox=np.array([[0, 0, 12, 10], [1, 1, 5, 5]], dtype=np.float64), categories=np.array(["x", "y"]))
    f.update(over)
    np.savez(path, **{k: v for k, v in f.items() if v is not None})
    return f


def test_correspondence_npz_and_its_errors(tmp_path):
    from dinov3_jax.eval import CorrespondenceNpzDataset, make_correspondence_dataset
    f = _npz(tmp_path / "c.npz")
    ds = make_correspondence_dataset(str(tmp_path / "c.npz"))
    assert isinstance(ds, CorrespondenceNpzDataset) and len(ds) == 2
    assert ds[1]["src"] == ds[1]["trg"] == 2 and ds[1]["category"] == "y"
    assert np.array_equal(ds[1]["trg_kps"], f["trg_kps"][1, :2]) and ds[0]["src_kps"].shape == (4, 2)
    assert np.array_equal(ds.load_image(2), f["images"][2])
    for name, over, msg in (("a", dict(categories=None), "field 'categories' is missing"),
                            ("b", dict(images=np.zeros((3, 10, 12), np.uint8)), "field 'images'"),
                            ("c", dict(pairs=np.array([[0, 3], [2, 2]])), "field 'pairs'"),
                            ("d", dict(n_kps=np.array([5, 2])), "field 'n_kps'"),
                            ("e", dict(trg_bbox=np.zeros((2, 3))), "field 'trg_bbox'"),
                            ("f", dict(src_kps=np.zeros((2, 4, 3))), "field 'src_kps'"),
                            ("g", dict(categories=np.array([1, 2])), "field 'categories'")):
        _npz(tmp_path / f"{name}.npz", **over)
        with pytest.raises(ValueError, match=re.escape(str(tmp_path / f"{name}.npz")) + ".*" + msg):
            CorrespondenceNpzDataset(tmp_path / f"{name}.npz")


# ------------------------------------------------------------------------------------------------ config, flags
def test_defaults_carry_the_correspondence_block():
    from dinov3_jax.configs import get_default_config
    assert get_default_config().evaluation.correspondence == {
        "dataset_path": "", "split": "test", "image_size": 512, "alphas": [0.01, 0.05, 0.1], "batch_size": 16,
        "num_workers": 4}


def test_do_correspondence_eval_without_dataset_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_correspondence_eval
    assert do_correspondence_eval(get_default_config(), None, "training_9") == {}
    assert "nothing evaluated" in capsys.readouterr().out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_raises_naming_knn_video_and_correspondence(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match="knn.*--eval video.*--eval correspondence"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_correspondence_reaches_do_correspondence_eval_and_nothing_else(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_correspondence_eval",
                        lambda config, model, header: calls.append((str(model), header)) or {"ok": 6})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval", "do_video_eval", "do_train"):
        monkeypatch.setattr(train, name,
                            lambda *a, _n=name, **k: pytest.fail(f"--eval-only --eval correspondence ran {_n}"))
    ck = tmp_path / "ckpt" / "8"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 8, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "correspondence", "--output-dir", str(tmp_path)]) == {"ok": 6}
    assert calls == [(str(ck), "manual_9")]


# ------------------------------------------------------------------------------------------------ ptxas
def test_correspondence_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert "correspondence.cu" in b.SOURCES
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", "correspondence.cu"), "-o",
                                       str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    seen = set()
    for name, stack, st, ld in props:
        if "corr_" in name:
            seen.add(name)
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # descriptors, Gram, argmax tiles, argmax merge
    assert len(seen) == 4, sorted(seen)
