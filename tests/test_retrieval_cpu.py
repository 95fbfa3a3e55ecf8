"""Instance retrieval without a GPU: the float64 oracle (tests/retrieval_oracle.py) on hand-computed cases, the size and
crop-box rules, the revisited root (with its restricted unpickler) and the .npz layout, the `evaluation.retrieval`
block, the --eval retrieval flags, the host-side argument checks of the kernels, and what ptxas makes of
csrc/retrieval.cu."""
import ctypes as C
import json
import os
import pickle
import re
import subprocess

import numpy as np
import pytest
import torch

import retrieval_oracle as oracle


def _sim(order, N):
    """A similarity row that ranks the indices of `order` first, in that order, and the rest after, by index."""
    s = np.zeros(N)
    for r, i in enumerate(order):
        s[i] = 1.0 - 0.01 * r
    rest = [i for i in range(N) if i not in order]
    for r, i in enumerate(rest):
        s[i] = -0.001 * r
    return s


# ------------------------------------------------------------------------------------------------ oracle by hand
def test_perfect_ranking_gives_ap_one():
    s = _sim([4, 2, 7], 10)
    sc = oracle.query_scores(s, [4, 2], [7], [])
    assert sc["easy"][0] == 1.0 and sc["medium"][0] == 1.0
    assert sc["easy"][1] == [1.0, 1.0, 1.0]                      # 2 positives: kq = 2 for k = 5, 10
    # Hard: 7 is ok and the easy images 4, 2 above it are junk, so it is first
    assert sc["hard"][0] == 1.0 and sc["hard"][2] == 1


def test_positive_behind_junk_takes_its_junk_free_rank():
    # ranks: 0 junk, 1 ok, 2 other, 3 ok -> junk-free ranks 0 and 2
    s = _sim([0, 1, 2, 3], 6)
    ap, pk, n = oracle.query_scores(s, [1, 3], [], [0])["easy"]
    assert n == 2
    assert ap == pytest.approx(((1.0 + 1.0) + (1 / 2 + 2 / 3)) / 4, abs=1e-15)
    assert oracle.junk_free_ranks(oracle.ranks(s), {1, 3}, {0}).tolist() == [0, 2]
    # P@1 = 1; P@5 and P@10: 1-based ranks 1, 3, kq = 3 -> 2 / 3
    assert pk == pytest.approx([1.0, 2 / 3, 2 / 3], abs=1e-15)


def test_ties_go_to_the_lower_index():
    s = np.array([0.5, 0.5, 0.5, 0.5, 0.9])
    assert oracle.order(s).tolist() == [4, 0, 1, 2, 3]
    assert oracle.ranks(s).tolist() == [1, 2, 3, 4, 0]
    ap = oracle.query_scores(s, [3], [], [])["easy"][0]
    assert ap == pytest.approx((0.0 / 4 + 1 / 5) / 2)         # j = 0 at rank 4: (0 / 4 + 1 / 5) / 2


def test_query_without_positives_is_excluded_and_counted():
    sims = np.stack([_sim([0, 1], 5), _sim([2], 5)])
    res, per = oracle.evaluate(sims, [[0], [2]], [[1], []], [[], []])
    assert np.isnan(per[1]["hard"][0]) and per[1]["hard"][2] == 0
    assert res["n_empty"] == {"easy": 0, "medium": 0, "hard": 1}
    assert res["mAP"]["hard"] == pytest.approx(100.0 * per[0]["hard"][0])
    # query 0, Hard: 1 is ok at rank 1, the easy 0 above it is junk -> junk-free rank 0
    assert per[0]["hard"][0] == 1.0


def test_protocol_sets_and_the_overlap_rule():
    easy, hard, junk = [1, 2], [3, 2], [4, 1]
    assert oracle.ok_junk(easy, hard, junk, "easy") == ({1, 2}, {3, 4})      # 2 and 1 are ok, not junk
    assert oracle.ok_junk(easy, hard, junk, "medium") == ({1, 2, 3}, {4})
    assert oracle.ok_junk(easy, hard, junk, "hard") == ({2, 3}, {1, 4})
    s = _sim([1, 4, 3, 2, 0], 5)
    sc = oracle.query_scores(s, easy, hard, junk)
    # Easy: ok 1 (rank 0), 2 (rank 3, junk 4 and 3 above it -> 1)
    assert sc["easy"][0] == pytest.approx(((1 + 1) + (1 / 1 + 2 / 2)) / 4)
    # Medium: ok 1 (0), 3 (2 - 1 = 1), 2 (3 - 1 = 2): a perfect list
    assert sc["medium"][0] == 1.0
    # Hard: junk 1, 4 above 3 (rank 2 -> 0) and 2 (rank 3 -> 1): perfect
    assert sc["hard"][0] == 1.0


def test_precision_at_k_with_fewer_than_k_positives():
    r = np.array([0, 3])                                         # 1-based ranks 1 and 4
    assert oracle.precision_at(r, 1) == 1.0
    assert oracle.precision_at(r, 5) == pytest.approx(2 / 4)     # kq = min(4, 5)
    assert oracle.precision_at(r, 10) == pytest.approx(2 / 4)
    r = np.array([1, 2, 6, 20])                                  # 1-based 2, 3, 7, 21
    assert oracle.precision_at(r, 1) == 0.0 and oracle.precision_at(r, 5) == pytest.approx(2 / 5)
    assert oracle.precision_at(r, 10) == pytest.approx(3 / 10)


# ------------------------------------------------------------------------------------------------ sizes, crops
def test_size_rule():
    from dinov3_jax.eval.retrieval import SCALES, scaled_size
    # an Oxford image: r = 1/2
    assert [scaled_size((768, 1024), 512, s, 16) for s in SCALES] == [(384, 512), (272, 368), (192, 256)]
    assert [scaled_size((1024, 768), 512, s, 16) for s in SCALES] == [(512, 384), (368, 272), (256, 192)]
    # never enlarged (r = 1), rounded to the nearest multiple of p, at least p
    assert scaled_size((300, 200), 512, 1.0, 16) == (304, 208)
    assert scaled_size((10, 20), 512, 0.5, 16) == (16, 16)
    assert scaled_size((600, 24), 512, 1.0, 14) == (518, 14)       # 24 * 512 / 600 = 20.48 -> 14
    assert SCALES[1] == 0.7071067811865476


def test_crop_box_rule_and_the_plan():
    from dinov3_jax.eval.retrieval import batches, plan_inputs, query_box
    assert query_box((10.4, 20.6, 100.2, 50.0), (40, 90)) == (10, 20, 90, 40)
    assert query_box((0, 0, 5, 5), (40, 90)) == (0, 0, 5, 5)
    assert query_box((-3.5, -1.0, 2.1, 7.9), (40, 90)) == (0, 0, 3, 8)
    with pytest.raises(ValueError, match="leaves nothing"):
        query_box((95.0, 1.0, 99.0, 5.0), (40, 90))
    plan = plan_inputs([(64, 48), (48, 64), (64, 48)], None, 64, (1.0, 0.5), 16)
    # at scale 1/2 every image is 32 x 32 (24 / 16 + 0.5 rounds down to 2)
    assert [(p[0], p[1], p[2]) for p in plan] == [((32, 32), 0, 1), ((32, 32), 1, 1), ((32, 32), 2, 1),
                                                  ((48, 64), 1, 0), ((64, 48), 0, 0), ((64, 48), 2, 0)]
    assert plan[0][3] == (0, 0, 48, 64)
    assert [[(p[1], p[2]) for p in b] for b in batches(plan, 2)] == [
        [(0, 1), (1, 1)], [(2, 1)], [(1, 0)], [(0, 0), (2, 0)]]
    cropped = plan_inputs([(64, 48)], [(8, 4, 40, 36)], 512, (1.0,), 16)
    assert cropped == [((32, 32), 0, 0, (8, 4, 40, 36))]


# ------------------------------------------------------------------------------------------------ datasets
def _revisited_root(root, dataset="roxford5k", as_arrays=False, protocol=pickle.DEFAULT_PROTOCOL):
    from PIL import Image
    (root / "jpg").mkdir(parents=True, exist_ok=True)
    db = {"all_souls_1": (30, 40), "radcliffe_2": (50, 20), "christ_3": (24, 24)}
    qs = {"all_souls_q": (60, 80), "radcliffe_q": (40, 30)}
    for name, (H, W) in {**db, **qs}.items():
        Image.fromarray(np.full((H, W, 3), 100, np.uint8)).save(root / "jpg" / f"{name}.jpg")
    wrap = (lambda v, dt=np.int64: np.asarray(v, dt)) if as_arrays else (lambda v, dt=None: list(v))
    gnd = [{"bbx": wrap([1.5, 2.0, 60.2, 40.7], np.float64), "easy": wrap([0]), "hard": wrap([2]), "junk": wrap([])},
           {"bbx": wrap([0.0, 0.0, 30.0, 40.0], np.float64), "easy": wrap([1, 2]), "hard": wrap([]),
            "junk": wrap([0])}]
    cfg = {"imlist": list(db), "qimlist": list(qs), "gnd": gnd}
    (root / f"gnd_{dataset}.pkl").write_bytes(pickle.dumps(cfg, protocol=protocol))
    return db, qs


@pytest.mark.parametrize("as_arrays,protocol", [(False, 4), (True, 4), (True, 2)],
                         ids=["lists", "ndarrays", "ndarrays-protocol2"])
def test_revisited_root_loads(tmp_path, as_arrays, protocol):
    from dinov3_jax.eval import RevisitedDataset, make_retrieval_dataset
    db, qs = _revisited_root(tmp_path, as_arrays=as_arrays, protocol=protocol)
    ds = make_retrieval_dataset(str(tmp_path), "roxford5k")
    assert isinstance(ds, RevisitedDataset) and ds.name == "roxford5k"
    assert ds.db_names == list(db) and ds.q_names == list(qs)
    assert ds.db_sizes == list(db.values()) and ds.q_sizes == list(qs.values())
    assert ds.q_bbx.tolist() == [[1.5, 2.0, 60.2, 40.7], [0.0, 0.0, 30.0, 40.0]]
    assert [e.tolist() for e in ds.easy] == [[0], [1, 2]] and [e.tolist() for e in ds.hard] == [[2], []]
    assert [e.tolist() for e in ds.junk] == [[], [0]]
    assert ds.load_db(1).shape == (50, 20, 3) and ds.load_query(0).dtype == np.uint8
    with pytest.raises(FileNotFoundError, match="gnd_rparis6k.pkl"):
        RevisitedDataset(tmp_path, "rparis6k")
    with pytest.raises(ValueError, match="dataset must be one of"):
        RevisitedDataset(tmp_path, "oxford5k")


class _Exploit:
    def __init__(self, marker):
        self.marker = marker

    def __reduce__(self):
        return (os.system, (f"touch {self.marker}",))


def test_revisited_pickle_naming_os_system_is_refused_unexecuted(tmp_path):
    from dinov3_jax.eval import RevisitedDataset
    _revisited_root(tmp_path)
    marker = tmp_path / "executed"
    cfg = {"imlist": ["all_souls_1"], "qimlist": [], "gnd": [], "x": _Exploit(marker)}
    path = tmp_path / "gnd_roxford5k.pkl"
    path.write_bytes(pickle.dumps(cfg))
    with pytest.raises(pickle.UnpicklingError, match=re.escape(str(path)) + ".*(posix|os)\\.system"):
        RevisitedDataset(tmp_path)
    assert not marker.exists()


def test_revisited_errors_name_the_file_and_field(tmp_path):
    from dinov3_jax.eval import RevisitedDataset
    _revisited_root(tmp_path)
    path = tmp_path / "gnd_roxford5k.pkl"
    good = pickle.loads(path.read_bytes())
    for change, msg in ((lambda c: c["gnd"][1].update(easy=[3]), r"'gnd\[1\].easy' must hold database indices"),
                        (lambda c: c["gnd"][0].pop("junk"), r"'gnd\[0\].junk' is missing"),
                        (lambda c: c["gnd"][0].update(bbx=[1, 2, 3]), r"'gnd\[0\].bbx' must be 4 finite"),
                        (lambda c: c.pop("qimlist"), "field 'qimlist' is missing"),
                        (lambda c: c["gnd"].pop(), "'gnd' has 1 entries for 2 queries")):
        cfg = pickle.loads(pickle.dumps(good))
        change(cfg)
        path.write_bytes(pickle.dumps(cfg))
        with pytest.raises(ValueError, match=re.escape(str(path)) + ".*" + msg):
            RevisitedDataset(tmp_path)
    path.write_bytes(pickle.dumps(good))
    (tmp_path / "jpg" / "christ_3.jpg").unlink()
    with pytest.raises(FileNotFoundError, match="names christ_3"):
        RevisitedDataset(tmp_path)


def _npz(path, **over):
    rng = np.random.default_rng(4)
    f = dict(db_images=rng.integers(0, 256, (3, 20, 24, 3), dtype=np.uint8), db_sizes=np.array([[20, 24], [17, 9],
                                                                                                  [20, 1]]),
             q_images=rng.integers(0, 256, (2, 16, 16, 3), dtype=np.uint8), q_sizes=np.array([[16, 16], [10, 12]]),
             q_bbx=np.array([[0.0, 0.0, 8.0, 8.0], [1.5, 2.5, 11.0, 9.2]]),
             easy_ptr=np.array([0, 1, 3]), easy_idx=np.array([2, 0, 1]), hard_ptr=np.array([0, 0, 1]),
             hard_idx=np.array([2]), junk_ptr=np.array([0, 2, 2]), junk_idx=np.array([0, 1]))
    f.update(over)
    np.savez(path, **{k: v for k, v in f.items() if v is not None})
    return f


def test_retrieval_npz_and_its_errors(tmp_path):
    from dinov3_jax.eval import RetrievalNpzDataset, make_retrieval_dataset
    f = _npz(tmp_path / "r.npz")
    ds = make_retrieval_dataset(str(tmp_path / "r.npz"), "rparis6k")
    assert isinstance(ds, RetrievalNpzDataset) and ds.name == "rparis6k"
    assert ds.db_names == ["00000", "00001", "00002"] and ds.q_names == ["00000", "00001"]
    assert ds.db_sizes == [(20, 24), (17, 9), (20, 1)] and ds.q_sizes == [(16, 16), (10, 12)]
    assert [e.tolist() for e in ds.easy] == [[2], [0, 1]] and [e.tolist() for e in ds.hard] == [[], [2]]
    assert [e.tolist() for e in ds.junk] == [[0, 1], []]
    assert np.array_equal(ds.load_db(1), f["db_images"][1, :17, :9])
    assert np.array_equal(ds.load_query(1), f["q_images"][1, :10, :12])
    for name, over, msg in (("a", dict(junk_idx=None), "field 'junk_idx' is missing"),
                            ("b", dict(db_images=np.zeros((3, 20, 24), np.uint8)), "field 'db_images'"),
                            ("c", dict(q_sizes=np.array([[16, 17], [10, 12]])), "field 'q_sizes'"),
                            ("d", dict(q_bbx=np.zeros((2, 3))), "field 'q_bbx'"),
                            ("e", dict(easy_ptr=np.array([0, 2, 1])), "field 'easy_ptr'"),
                            ("f", dict(hard_ptr=np.array([1, 1, 1])), "field 'hard_ptr'"),
                            ("g", dict(junk_ptr=np.array([0, 1])), "field 'junk_ptr'"),
                            ("h", dict(easy_idx=np.array([2, 0, 3])), "field 'easy_idx'"),
                            ("i", dict(hard_idx=np.array([-1])), "field 'hard_idx'")):
        _npz(tmp_path / f"{name}.npz", **over)
        with pytest.raises(ValueError, match=re.escape(str(tmp_path / f"{name}.npz")) + ".*" + msg):
            RetrievalNpzDataset(tmp_path / f"{name}.npz")


# ------------------------------------------------------------------------------------------------ config, flags
def test_defaults_carry_the_retrieval_block():
    from dinov3_jax.configs import get_default_config
    assert get_default_config().evaluation.retrieval == {
        "dataset_path": "", "dataset": "roxford5k", "image_size": 512, "scales": [1.0, 0.7071067811865476, 0.5],
        "batch_size": 16, "num_workers": 4, "save_ranks": False}


def test_do_retrieval_eval_without_dataset_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_retrieval_eval
    assert do_retrieval_eval(get_default_config(), None, "training_9") == {}
    assert "nothing evaluated" in capsys.readouterr().out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_raises_naming_every_mode_with_retrieval_last(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match=r"knn.*--eval video.*--eval correspondence.*--eval discovery\), "
                                                  r"and instance retrieval \(--eval retrieval\)$"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_retrieval_reaches_do_retrieval_eval_and_nothing_else(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_retrieval_eval", lambda config, model, header: calls.append((str(model), header))
                        or {"ok": 3})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval", "do_video_eval",
                 "do_correspondence_eval", "do_discovery_eval", "do_train"):
        monkeypatch.setattr(train, name, lambda *a, _n=name, **k: pytest.fail(f"--eval-only --eval retrieval ran {_n}"))
    ck = tmp_path / "ckpt" / "8"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 8, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "retrieval", "--output-dir", str(tmp_path)]) == {"ok": 3}
    assert calls == [(str(ck), "manual_9")]


# ------------------------------------------------------------------------------------------------ host-side checks
def test_kernel_arguments_are_checked_on_the_host():
    """The list and crop checks come before any CUDA call, so they answer without a device."""
    from dinov3_jax import _native
    lib = _native.lib()
    fake = C.c_void_p(256)
    ints = lambda *v: (C.c_int * max(len(v), 1))(*v)
    out = [fake] * 4
    ok_ptr, no_idx = ints(0, 0), ints()
    for easy, msg in (((ints(0, 1), ints(5)), b"outside [0, N)"), ((ints(0, 1), ints(-1)), b"outside [0, N)"),
                      ((ints(1, 1), ints(0)), b"start at 0"), ((ints(0, 8193), ints(*([0] * 8193))), b"8192")):
        rc = lib.d3_ret_rank_ap(fake, 8, 1, 5, easy[0], easy[1], ok_ptr, no_idx, ok_ptr, no_idx, *out, None)
        assert rc == -1 and msg in lib.d3_last_error(), lib.d3_last_error()
    rc = lib.d3_ret_rank_ap(fake, 4, 1, 5, ok_ptr, no_idx, ok_ptr, no_idx, ok_ptr, no_idx, *out, None)
    assert rc == -1 and b"lds >= N" in lib.d3_last_error()
    ms = (C.c_float * 3)(0.5, 0.5, 0.5)
    desc = lambda *v: (C.c_longlong * 7)(*v)
    for d, msg in ((desc(0, 10, 10, 0, 0, 11, 10), b"crop box"), (desc(0, 10, 10, 4, 0, 4, 10), b"crop box"),
                   (desc(1, 10, 10, 0, 0, 10, 10), b"outside the source buffer")):
        rc = lib.d3_ret_resize(fake, 300, d, 1, 16, 16, ms, ms, fake, None)
        assert rc == -1 and msg in lib.d3_last_error(), lib.d3_last_error()


# ------------------------------------------------------------------------------------------------ ptxas
def test_retrieval_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert "retrieval.cu" in b.SOURCES
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", "retrieval.cu"), "-o",
                                       str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    seen = set()
    for name, stack, st, ld in props:
        if "ret_" in name:
            seen.add(name)
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # resize, scale sum, sort, count, ap
    assert len(seen) == 5, sorted(seen)
