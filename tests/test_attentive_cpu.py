"""Attentive-probe video classification without a GPU: the fold of csrc/attentive.cu restated in float64 against the
unfolded probe (tests/attentive_oracle.py), clip and view sampling, the three dataset layouts, the train clips'
independence from the worker count, the `evaluation.attentive` block, the --eval attentive flags, the host-side
argument checks and what ptxas makes of csrc/attentive.cu."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import attentive_oracle as oracle


# ------------------------------------------------------------------------------------------------ the fold
@pytest.mark.parametrize("D,H,T,P,B,query_scale", [(16, 2, 3, 5, 2, 1.0), (24, 3, 1, 7, 3, 8.0), (32, 4, 4, 9, 1, 20.0),
                                                    (48, 6, 2, 4, 5, 3.0)])
def test_fold_matches_the_unfolded_probe(D, H, T, P, B, query_scale):
    """The folded forward (keys folded into the query, values out of the sum) and the token pass's backward as the
    kernels compute it, against autograd through the keys and values of every token: float64 rounding only."""
    p = oracle.make_params(D, H, T, 11, seed=D + T, query_scale=query_scale)
    g = torch.Generator().manual_seed(B)
    x = torch.randn(B, T * P, D, generator=g, dtype=torch.float64) * 3
    labels = torch.randint(0, 11, (B,), generator=g)
    u, f = oracle.unfolded(p, x, T, H, labels), oracle.folded(p, x, T, H, labels)
    assert torch.allclose(f["a"], u["a"], rtol=0, atol=1e-10 * u["a"].abs().max().item())
    assert abs(f["loss"].item() - u["loss"].item()) <= 1e-10 * abs(u["loss"].item())
    for name in oracle.NAMES:
        ref = u["grads"][name]
        assert (f["grads"][name] - ref).abs().max().item() <= 1e-10 * max(ref.abs().max().item(), 1e-30), name


# ------------------------------------------------------------------------------------------------ clips and views
def test_clip_indices_clamp_to_the_last_frame():
    from dinov3_jax.eval.attentive import clip_indices, clip_span
    assert clip_span(16, 4) == 61
    assert clip_indices(100, 3, 4, 4) == [3, 7, 11, 15]
    assert clip_indices(10, 2, 4, 3) == [2, 5, 8, 9]
    assert clip_indices(1, 0, 3, 4) == [0, 0, 0]


def test_val_starts_and_view_boxes():
    from dinov3_jax.eval.attentive import val_clip_starts, view_boxes
    assert val_clip_starts(100, 16, 4, 2) == [0, 39]
    assert val_clip_starts(100, 16, 4, 3) == [0, 20, 39]
    assert val_clip_starts(100, 16, 4, 1) == [19]
    assert val_clip_starts(30, 16, 4, 2) == [0, 0]                  # shorter than a clip: every start is 0
    assert view_boxes(240, 320, 3) == [(0, 0, 240, 240), (0, 40, 240, 240), (0, 80, 240, 240)]
    assert view_boxes(320, 240, 3) == [(0, 0, 240, 240), (40, 0, 240, 240), (80, 0, 240, 240)]
    assert view_boxes(240, 320, 1) == [(0, 40, 240, 240)]
    assert view_boxes(64, 64, 3) == [(0, 0, 64, 64)] * 3


def test_train_draws_depend_on_seed_iteration_and_slot_only():
    from dinov3_jax.eval.attentive import sample_train_box, sample_train_clip
    draw = lambda seed, it, slot, n: (lambda r: (tuple(r[0]), sample_train_box(r[1], 120, 160)))(
        sample_train_clip(seed, it, slot, n, 16, 4))
    a = draw(0, 5, 3, 200)
    assert a == draw(0, 5, 3, 200)
    assert len({draw(0, 5, s, 200) for s in range(8)}) == 8
    assert draw(1, 5, 3, 200) != a and draw(0, 6, 3, 200) != a
    for it in range(50):
        idx, (top, left, h, w, flip) = draw(0, it, 0, 200)
        assert 0 <= idx[0] <= 200 - 61 and idx == tuple(range(idx[0], idx[0] + 61, 4))
        assert 0 <= top and top + h <= 120 and 0 <= left and left + w <= 160 and flip in (0, 1)
        assert 0.3 * 120 * 160 * 0.99 <= h * w <= 120 * 160
    idx, _ = draw(0, 0, 0, 20)                                       # shorter than a clip: clamped from start 0
    assert idx == (0, 4, 8, 12, 16) + (19,) * 11


def test_probe_lr_schedule():
    from dinov3_jax.eval.attentive import probe_lr
    assert probe_lr(1.0, 0, 100, 10) == pytest.approx(0.1)
    assert probe_lr(1.0, 9, 100, 10) == pytest.approx(1.0)
    assert probe_lr(1.0, 10, 100, 10) == pytest.approx(1.0)
    assert probe_lr(1.0, 55, 100, 10) == pytest.approx(0.5)
    assert probe_lr(1.0, 99, 100, 0) == pytest.approx(0.5 * (1 + np.cos(np.pi * 99 / 100)))


# ------------------------------------------------------------------------------------------------ datasets
def _video(n, F, H, W, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (n, F, H, W, 3), dtype=np.uint8)


def test_npz_layout_and_its_errors(tmp_path):
    from dinov3_jax.eval import make_video_class_dataset
    v = _video(3, 5, 8, 12, 0)
    np.savez(tmp_path / "v.npz", videos=v, labels=np.array([2, 0, 1]))
    ds = make_video_class_dataset(str(tmp_path / "v.npz"))
    assert len(ds) == 3 and ds.targets == [2, 0, 1] and ds.frame_count(1) == 5
    assert np.array_equal(ds.load_frames(1, [0, 4, 9]), v[1][[0, 4, 4]])
    np.savez(tmp_path / "bad.npz", videos=v[..., 0], labels=np.array([2, 0, 1]))
    with pytest.raises(ValueError, match="bad.npz"):
        make_video_class_dataset(str(tmp_path / "bad.npz"))


def test_list_of_frame_directories(tmp_path):
    from PIL import Image
    from dinov3_jax.eval import make_video_class_dataset
    v = _video(2, 4, 6, 10, 1)
    for i in range(2):
        d = tmp_path / "frames" / f"clip{i}"
        d.mkdir(parents=True)
        for t in range(4):
            Image.fromarray(v[i, t]).save(d / f"{t:05d}.png")
    (tmp_path / "list.txt").write_text("frames/clip0 3\n\nframes/clip1 1\n")
    ds = make_video_class_dataset(str(tmp_path / "list.txt"))
    assert len(ds) == 2 and ds.targets == [3, 1] and ds.frame_count(0) == 4
    assert np.array_equal(ds.load_frames(1, [3, 1, 7]), v[1][[3, 1, 3]])
    (tmp_path / "bad.txt").write_text("frames/clip0\n")
    with pytest.raises(ValueError, match="bad.txt:1"):
        make_video_class_dataset(str(tmp_path / "bad.txt"))


def test_list_of_video_files(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from dinov3_jax.eval import make_video_class_dataset
    H, W, F = 32, 48, 7
    frames = [np.full((H, W, 3), (30 * t, 255 - 30 * t, 100), np.uint8) for t in range(F)]
    writer = cv2.VideoWriter(str(tmp_path / "a.avi"), cv2.VideoWriter_fourcc(*"MJPG"), 10, (W, H))
    for f in frames:
        writer.write(cv2.cvtColor(f, cv2.COLOR_RGB2BGR))
    writer.release()
    (tmp_path / "list.txt").write_text("a.avi 4\nmissing.avi 0\n")
    ds = make_video_class_dataset(str(tmp_path / "list.txt"))
    assert ds.frame_count(0) == F
    got = ds.load_frames(0, [0, 6, 20])
    assert got.shape == (3, H, W, 3) and got.dtype == np.uint8
    for k, t in enumerate([0, 6, 6]):                                # MJPG is lossy: the colour of the frame
        assert np.abs(got[k].astype(int).mean((0, 1)) - frames[t][0, 0]).max() < 8, (k, t)
    with pytest.raises(ValueError, match="missing.avi"):
        ds.frame_count(1)
    with pytest.raises(ValueError, match="missing.avi"):
        ds.load_frames(1, [0])


def test_train_clips_do_not_depend_on_the_worker_count(tmp_path):
    from dinov3_jax.eval import make_video_class_dataset
    from dinov3_jax.eval.attentive import _ClipBatches, _collate_train, _TrainClips
    v = _video(7, 9, 20, 28, 2)
    np.savez(tmp_path / "v.npz", videos=v, labels=np.arange(7) % 3)
    ds = make_video_class_dataset(str(tmp_path / "v.npz"))

    def batches(workers):
        loader = torch.utils.data.DataLoader(_TrainClips(ds, 4, 2, seed=5), batch_sampler=_ClipBatches(7, 3, 6, 5),
                                             num_workers=workers, collate_fn=_collate_train)
        return list(loader)

    a, b = batches(0), batches(2)
    assert len(a) == 6
    for x, y in zip(a, b):
        for s, t in zip(x, y):
            assert torch.equal(s, t)
    assert a[0][2].shape == (3,) and all(0 <= int(y) < 3 for y in a[0][2])
    assert a[0][3].shape == (12, 5) and torch.equal(a[0][3][0], a[0][3][3])   # one box per clip, on all its frames


# ------------------------------------------------------------------------------------------------ config, flags
def test_defaults_carry_the_attentive_block():
    from dinov3_jax.configs import get_default_config
    assert get_default_config().evaluation.attentive == {
        "train_dataset_path": "", "val_dataset_path": "", "learning_rates": [1e-4, 3e-4, 1e-3], "epochs": 20,
        "warmup_epochs": 0, "weight_decay": 0.01, "batch_size": 16, "num_frames": 16, "frame_step": 4,
        "num_segments": 2, "num_views": 3, "crop_size": 224, "num_workers": 8, "seed": 0}


def test_do_attentive_eval_without_datasets_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_attentive_eval
    assert do_attentive_eval(get_default_config(), None, "training_9") == {}
    out = capsys.readouterr().out
    assert out.count("\n") == 1 and "nothing evaluated" in out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_names_attentive_after_logreg(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match=r"logistic regression \(--eval logreg\), attentive-probe video "
                                                  r"classification \(--eval attentive\), the linear segmentation.*"
                                                  r"and instance retrieval \(--eval retrieval\)$"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_attentive_reaches_do_attentive_eval_and_nothing_else(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_attentive_eval", lambda config, model, header: calls.append((str(model), header))
                        or {"ok": 5})
    for name in ("do_test", "do_linear_eval", "do_logreg_eval", "do_seg_eval", "do_depth_eval", "do_video_eval",
                 "do_correspondence_eval", "do_discovery_eval", "do_retrieval_eval", "do_train"):
        monkeypatch.setattr(train, name, lambda *a, _n=name, **k: pytest.fail(f"--eval-only --eval attentive ran {_n}"))
    ck = tmp_path / "ckpt" / "8"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 8, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "attentive", "--output-dir", str(tmp_path)]) == {"ok": 5}
    assert calls == [(str(ck), "manual_9")]


def test_probe_refuses_a_backbone_wider_than_1536():
    from dinov3_jax.eval.attentive import AttentiveProbe
    with pytest.raises(NotImplementedError, match="4096 is wider than 1536"):
        AttentiveProbe(4096, 32, 16, 400, 16, 10)
    with pytest.raises(ValueError, match="heads"):
        AttentiveProbe(384, 5, 16, 400, 16, 10)


# ------------------------------------------------------------------------------------------------ host-side checks
def test_kernel_arguments_are_checked_on_the_host():
    from dinov3_jax import _native
    lib = _native.lib()
    fake = C.c_void_p(256)
    for fn in (lambda *a: lib.d3_atp_pool_fwd(fake, fake, fake, fake, fake, *a, fake, fake, None),
               lambda *a: lib.d3_atp_pool_bwd(*[fake] * 8, *a, fake, fake, fake, fake, None)):
        for B, T, P, D, H in ((2, 16, 196, 2048, 16), (2, 16, 196, 1020, 6), (2, 16, 196, 384, 5),
                              (0, 16, 196, 384, 6), (2, 0, 196, 384, 6), (2, 16, 0, 384, 6)):
            assert fn(B, T, P, D, H) == -1
            assert b"D a multiple of 8 in [8, 1536] divisible by H" in lib.d3_last_error()
    assert lib.d3_atp_pool_fwd(C.c_void_p(264), fake, fake, fake, fake, 2, 16, 196, 384, 6, fake, fake, None) == -1
    assert b"16-byte aligned" in lib.d3_last_error()
    assert lib.d3_atp_query_fwd(fake, fake, fake, fake, 384, 5, fake, fake, None) == -1
    assert b"dividing D" in lib.d3_last_error()
    assert lib.d3_atp_query_bwd(*[fake] * 5, 384, 7, *[fake] * 4, None) == -1
    assert b"dividing D" in lib.d3_last_error()
    assert lib.d3_atp_gelu_erf_bwd(fake, 8, fake, 16, 4, 16, fake, 16, None) == -1
    assert b"ld_out >= cols" in lib.d3_last_error()


# ------------------------------------------------------------------------------------------------ ptxas
def test_attentive_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert "attentive.cu" in b.SOURCES
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", "attentive.cu"), "-o",
                                       str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    seen = set()
    for name, stack, st, ld in props:
        if "atp_" in name:
            seen.add(name)
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    # forward and backward pass for 1..6 columns per thread, merge, q, kt, dq, dq0, GELU'
    assert len(seen) == 18, sorted(seen)
