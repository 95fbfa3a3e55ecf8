"""Object discovery without a GPU: the float64 oracle (tests/discovery_oracle.py) on a hand-built case, the closed-form
top eigenpair and the D^-1/2 equivalence the kernel relies on, the VOC and .npz layouts, IoU and CorLoc, the
`evaluation.discovery` block, the --eval discovery flags, and what ptxas makes of csrc/discovery.cu."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.linalg
import torch

import discovery_oracle as oracle


def _two_groups(h, w, rows, cols, D=8):
    """Unit features of an h x w grid: e0 on the object cells (rows x cols), e1 elsewhere."""
    f = np.zeros((h, w, D))
    f[..., 1] = 1.0
    f[rows[0]:rows[1], cols[0]:cols[1]] = 0.0
    f[rows[0]:rows[1], cols[0]:cols[1], 0] = 1.0
    return f.reshape(h * w, D)


# ------------------------------------------------------------------------------------------------ oracle by hand
def test_oracle_finds_a_2x2_object_on_a_4x5_grid():
    feats = _two_groups(4, 5, (1, 3), (2, 4))
    A, d = oracle.graph(feats)
    assert A[7, 13] == 1.0 and A[0, 7] == 1e-5 and A[0, 0] == 1.0        # the diagonal is in the graph
    assert d[7] == pytest.approx(4 + 16e-5) and d[0] == pytest.approx(16 + 4e-5)
    res = oracle.discover(feats, (4, 5), 16, (64, 80))
    assert res["box"] == [32, 16, 64, 48]
    assert sorted(np.nonzero(res["fg"])[0].tolist()) == [7, 8, 12, 13]
    # either sign of the eigenvector gives the same bipartition: one of the two goes through the flip
    fg_pos, s_pos = oracle.bipartition(res["x"])
    fg_neg, s_neg = oracle.bipartition(-res["x"])
    assert np.array_equal(fg_pos, fg_neg) and s_pos == s_neg and s_pos in (7, 8, 12, 13)
    # clipping to a 60 x 70 image whose last row and column of patches are partial
    big = _two_groups(4, 5, (2, 4), (3, 5))
    assert oracle.discover(big, (4, 5), 16, (60, 70))["box"] == [48, 32, 70, 60]


def test_bipartition_seed_ties_and_the_flip():
    # |x| ties between index 1 and 3: the lowest index is the seed; 3.0 > mean, so no flip
    x = np.array([0.0, 3.0, -1.0, -3.0, 1.0])
    fg, seed = oracle.bipartition(x)
    assert seed == 1 and fg.tolist() == [False, True, False, False, True]
    # the seed (-3 at index 1) below the mean: the complement is taken
    fg, seed = oracle.bipartition(np.array([1.0, -3.0, 0.5, 3.0, 0.0]))
    assert seed == 1 and fg.tolist() == [False, True, False, False, True]
    # two blobs of one mask: only the seed's component makes the box
    fg = np.zeros((3, 6), bool)
    fg[0, 0:2] = fg[2, 4:6] = True
    fg[1, 1] = True                                                        # 4-connected to the first blob
    assert oracle.component_box(fg.reshape(-1), 17, (3, 6), 10, (30, 60)) == [40, 20, 60, 30]
    assert oracle.component_box(fg.reshape(-1), 0, (3, 6), 10, (30, 60)) == [0, 0, 20, 20]
    diag = np.zeros((2, 2), bool)
    diag[0, 0] = diag[1, 1] = True                                         # diagonal cells are not 4-connected
    assert oracle.component_box(diag.reshape(-1), 0, (2, 2), 8, (16, 16)) == [0, 0, 8, 8]


# ------------------------------------------------------------------------------------------------ eigenproblem
@pytest.mark.parametrize("grid", [(1, 9), (7, 1), (5, 7), (12, 10)], ids=lambda g: f"{g[0]}x{g[1]}")
def test_top_eigenpair_and_the_normalized_form(grid):
    h, w = grid
    N = h * w
    rng = np.random.default_rng(N)
    f = rng.normal(size=(N, 16)) + 2.0 * (np.arange(N) % 3 == 0)[:, None] * rng.normal(size=16)
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    A, d = oracle.graph(f)
    Dm = np.diag(d ** -0.5)
    M = Dm @ A @ Dm
    u = np.sqrt(d) / np.linalg.norm(np.sqrt(d))
    assert np.abs(M @ u - u).max() < 1e-10                                 # (1, D^1/2 1) in closed form
    theta, Y = np.linalg.eigh(M)
    assert theta[-1] == pytest.approx(1.0, abs=1e-10) and theta[-2] < 1.0 - 1e-10   # simple
    x, lam2, _ = oracle.fiedler(A, d)
    assert abs((1.0 - theta[-2]) - lam2) < 1e-10
    y = Y[:, -2]
    xs = Dm @ y                                                            # x = D^-1/2 y, y^T y = 1 <=> x^T D x = 1
    assert abs(abs(xs @ (d * x)) - 1.0) < 1e-10
    assert np.abs((np.diag(d) - A) @ x - lam2 * d * x).max() < 1e-10
    vals = scipy.linalg.eigh(np.diag(d) - A, np.diag(d), eigvals_only=True)
    assert vals[0] == pytest.approx(0.0, abs=1e-10)


# ------------------------------------------------------------------------------------------------ score
def test_iou_and_corloc_on_hand_made_boxes():
    from dinov3_jax.eval.discovery import box_iou, corloc
    gts = np.array([[0.0, 0.0, 10.0, 10.0], [20.0, 20.0, 30.0, 40.0]])
    # half overlap with the first: 50 / (100 + 100 - 50); none with the second
    assert box_iou([5, 0, 15, 10], gts).tolist() == pytest.approx([1 / 3, 0.0])
    assert oracle.iou([5, 0, 15, 10], gts).tolist() == pytest.approx([1 / 3, 0.0])
    assert box_iou([20, 20, 30, 40], gts)[1] == 1.0
    # exactly 0.5: [0, 0, 10, 10] against [0, 0, 10, 20] -> 100 / 200, a hit
    assert box_iou([0, 0, 10, 10], [[0, 0, 10, 20]])[0] == 0.5
    boxes = [[0, 0, 10, 10], [5, 0, 15, 10], [20, 20, 30, 40]]
    assert corloc(boxes, [[[0, 0, 10, 20]], gts, gts]) == pytest.approx(2 / 3)
    assert corloc([[0, 0, 4, 4]], [[[0, 0, 4, 4]]]) == 1.0


# ------------------------------------------------------------------------------------------------ datasets
def _voc_tree(root, objects, split="trainval"):
    """root/ImageSets/Main/<split>.txt, root/Annotations/<id>.xml and root/JPEGImages/<id>.jpg for objects =
    {id: (H, W, [(xmin, ymin, xmax, ymax, difficult)])}."""
    from PIL import Image
    for d in ("ImageSets/Main", "Annotations", "JPEGImages"):
        (root / d).mkdir(parents=True, exist_ok=True)
    (root / "ImageSets" / "Main" / f"{split}.txt").write_text("".join(f"{k}\n" for k in objects))
    for k, (H, W, objs) in objects.items():
        Image.fromarray(np.zeros((H, W, 3), np.uint8)).save(root / "JPEGImages" / f"{k}.jpg")
        body = "".join(f"<object><name>cat</name><difficult>{df}</difficult><bndbox><xmin>{a}</xmin><ymin>{b}</ymin>"
                       f"<xmax>{c}</xmax><ymax>{e}</ymax></bndbox></object>" for a, b, c, e, df in objs)
        (root / "Annotations" / f"{k}.xml").write_text(
            f"<annotation><size><width>{W}</width><height>{H}</height><depth>3</depth></size>{body}</annotation>")


def test_voc_layout_corners_and_difficult(tmp_path):
    from dinov3_jax.eval import VOCDiscoveryDataset, make_discovery_dataset
    _voc_tree(tmp_path, {"000005": (40, 50, [(1, 1, 10, 20, 0), (5, 6, 50, 40, 1)]), "000007": (30, 20, [])})
    ds = make_discovery_dataset(str(tmp_path))
    assert isinstance(ds, VOCDiscoveryDataset) and len(ds) == 2 and ds.names == ["000005", "000007"]
    assert ds.sizes == [(40, 50), (30, 20)]
    # 1-based inclusive -> [xmin - 1, ymin - 1, xmax, ymax]: the full image is [0, 0, W, H]
    assert ds.boxes[0].tolist() == [[0.0, 0.0, 10.0, 20.0], [4.0, 5.0, 50.0, 40.0]]
    assert ds.boxes[1].shape == (0, 4)
    assert make_discovery_dataset(str(tmp_path), remove_difficult=True).boxes[0].tolist() == [[0.0, 0.0, 10.0, 20.0]]
    im = ds.load_image(1)
    assert im.dtype == np.uint8 and im.shape == (30, 20, 3)


def test_voc_errors_name_the_file_and_field(tmp_path):
    from dinov3_jax.eval import VOCDiscoveryDataset
    with pytest.raises(FileNotFoundError, match="ImageSets"):
        VOCDiscoveryDataset(tmp_path)
    _voc_tree(tmp_path, {"a": (10, 10, [(1, 1, 5, 5, 0)])})
    path = tmp_path / "Annotations" / "a.xml"
    good = path.read_text()
    for text, msg in ((good.replace("<height>10</height>", ""), "a.xml: field 'size/height' is missing"),
                      (good.replace("<xmax>5</xmax>", "<xmax>five</xmax>"), "a.xml: field 'bndbox/xmax' is not a number"),
                      (good.replace("<ymin>1</ymin>", ""), "a.xml: field 'bndbox/ymin' is missing"),
                      (good.replace("<bndbox>", "<box>").replace("</bndbox>", "</box>"), "a.xml: field 'object/bndbox'"),
                      ("<annotation>", "a.xml: not valid XML")):
        path.write_text(text)
        with pytest.raises(ValueError, match=msg):
            VOCDiscoveryDataset(tmp_path)
    path.unlink()
    with pytest.raises(FileNotFoundError, match="names a, but .*a.xml does not exist"):
        VOCDiscoveryDataset(tmp_path)


def _npz(path, **over):
    rng = np.random.default_rng(2)
    f = dict(images=rng.integers(0, 256, (3, 20, 24, 3), dtype=np.uint8), sizes=np.array([[20, 24], [17, 9], [20, 1]]),
             boxes=np.array([[[0, 0, 5, 5], [1, 1, 4, 4]], [[2, 2, 9, 17], [0, 0, 0, 0]], [[0, 0, 1, 1], [0, 0, 0, 0]]],
                            dtype=np.float32), n_boxes=np.array([2, 1, 0]))
    f.update(over)
    np.savez(path, **{k: v for k, v in f.items() if v is not None})
    return f


def test_discovery_npz_and_its_errors(tmp_path):
    from dinov3_jax.eval import DiscoveryNpzDataset, make_discovery_dataset
    f = _npz(tmp_path / "d.npz")
    ds = make_discovery_dataset(str(tmp_path / "d.npz"))
    assert isinstance(ds, DiscoveryNpzDataset) and len(ds) == 3 and ds.names == ["00000", "00001", "00002"]
    assert ds.sizes == [(20, 24), (17, 9), (20, 1)]
    assert ds.boxes[1].tolist() == [[2.0, 2.0, 9.0, 17.0]] and ds.boxes[2].shape == (0, 4)
    assert np.array_equal(ds.load_image(1), f["images"][1, :17, :9])
    for name, over, msg in (("a", dict(n_boxes=None), "field 'n_boxes' is missing"),
                            ("b", dict(images=np.zeros((3, 20, 24), np.uint8)), "field 'images'"),
                            ("c", dict(sizes=np.array([[20, 24], [21, 9], [20, 1]])), "field 'sizes'"),
                            ("d", dict(sizes=np.array([[20, 24], [17, 0], [20, 1]])), "field 'sizes'"),
                            ("e", dict(boxes=np.zeros((3, 2, 3), np.float32)), "field 'boxes'"),
                            ("f", dict(n_boxes=np.array([3, 1, 0])), "field 'n_boxes'"),
                            ("g", dict(n_boxes=np.array([1, -1, 0])), "field 'n_boxes'")):
        _npz(tmp_path / f"{name}.npz", **over)
        with pytest.raises(ValueError, match=re.escape(str(tmp_path / f"{name}.npz")) + ".*" + msg):
            DiscoveryNpzDataset(tmp_path / f"{name}.npz")


def test_grid_of_rounds_up():
    from dinov3_jax.eval.discovery import grid_of
    assert grid_of((375, 500), 16) == (24, 32) and grid_of((384, 512), 16) == (24, 32) and grid_of((1, 17), 16) == (1, 2)


# ------------------------------------------------------------------------------------------------ config, flags
def test_defaults_carry_the_discovery_block():
    from dinov3_jax.configs import get_default_config
    assert get_default_config().evaluation.discovery == {
        "dataset_path": "", "split": "trainval", "tau": 0.2, "eps": 1e-5, "remove_difficult": False, "batch_size": 16,
        "num_workers": 4, "save_boxes": False}


def test_do_discovery_eval_without_dataset_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_discovery_eval
    assert do_discovery_eval(get_default_config(), None, "training_9") == {}
    assert "nothing evaluated" in capsys.readouterr().out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_raises_naming_every_mode_with_discovery_last(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match="knn.*--eval video.*--eval correspondence.*--eval discovery"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_discovery_reaches_do_discovery_eval_and_nothing_else(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_discovery_eval", lambda config, model, header: calls.append((str(model), header))
                        or {"ok": 7})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval", "do_video_eval",
                 "do_correspondence_eval", "do_train"):
        monkeypatch.setattr(train, name, lambda *a, _n=name, **k: pytest.fail(f"--eval-only --eval discovery ran {_n}"))
    ck = tmp_path / "ckpt" / "8"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 8, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "discovery", "--output-dir", str(tmp_path)]) == {"ok": 7}
    assert calls == [(str(ck), "manual_9")]


# ------------------------------------------------------------------------------------------------ ptxas
def test_discovery_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert "discovery.cu" in b.SOURCES
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", "discovery.cu"), "-o",
                                       str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    seen = set()
    for name, stack, st, ld in props:
        if "od_" in name:
            seen.add(name)
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # graph, fiedler, box
    assert len(seen) == 3, sorted(seen)
