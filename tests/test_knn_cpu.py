"""k-NN evaluation without a GPU: the configuration block, the no-dataset path of do_test, the --eval / --eval-only
flags, the evaluation datasets, and the float64 statement of the protocol (tests/knn_oracle.py) on hand-computed
cases."""
import json

import numpy as np
import pytest
import torch

import knn_oracle


def test_defaults_carry_the_evaluation_block():
    from dinov3_jax.configs import get_default_config
    ev = get_default_config().evaluation
    assert ev.eval_period_iterations == 12500
    assert ev.knn == {"train_dataset_path": "", "val_dataset_path": "", "nb_knn": [10, 20, 100, 200], "temperature": 0.07,
                      "batch_size": 256, "resize_size": 256, "crop_size": 224, "num_workers": 8}


def test_do_test_without_datasets_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_test
    assert do_test(get_default_config(), None, "training_9") == {}
    assert "nothing evaluated" in capsys.readouterr().out
    assert not torch.cuda.is_initialized()


def test_reference_config_files_key_is_accepted(tmp_path):
    import yaml
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    (tmp_path / "c.yaml").write_text(yaml.safe_dump({"evaluation": {"eval_period_iterations": 5, "low_freq_every": 5,
                                                                   "config_files": {"high_freq": "x.yaml"}}}))
    cfg = setup_config(DinoV3SetupArgs(config_file=str(tmp_path / "c.yaml")))
    assert cfg.evaluation.eval_period_iterations == 5 and cfg.evaluation.knn.nb_knn == [10, 20, 100, 200]


def test_eval_type_other_than_knn_raises(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match="knn"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_without_weights_or_checkpoint_raises(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(FileNotFoundError, match="--eval-pretrained-weights"):
        main(["--eval-only", "--output-dir", str(tmp_path)])


@pytest.mark.parametrize("source", ["weights", "latest"])
def test_eval_only_reaches_do_test_and_never_do_train(tmp_path, monkeypatch, source):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_test", lambda config, model, header: calls.append((str(model), header)) or {"ok": 1})
    monkeypatch.setattr(train, "do_train", lambda *a, **k: pytest.fail("--eval-only must not train"))
    ck = tmp_path / "ckpt" / "41"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 41, "leaves": {}, "scalars": {}}))
    args = ["--eval-only", "--eval", "knn", "--output-dir", str(tmp_path)]
    if source == "weights":
        args += ["--eval-pretrained-weights", str(ck)]
    assert train.main(args) == {"ok": 1}
    assert calls == [(str(ck), "manual_42")]


def test_image_folder_labels_are_sorted_class_directories(tmp_path):
    from PIL import Image
    from dinov3_jax.eval import ImageFolder
    for cls, n in (("zebra", 2), ("ant", 1), ("moth", 3)):
        (tmp_path / cls).mkdir()
        for i in range(n):
            Image.fromarray(np.full((5 + i, 7, 3), 40 * i, np.uint8)).save(tmp_path / cls / f"{n - i}.png")
    (tmp_path / "moth" / "notes.txt").write_text("not an image")
    ds = ImageFolder(tmp_path)
    assert ds.classes == ["ant", "moth", "zebra"]
    assert ds.targets == [0, 1, 1, 1, 2, 2]
    assert [p.split("/")[-1] for p, _ in ds.samples] == ["1.png", "1.png", "2.png", "3.png", "1.png", "2.png"]
    img, y = ds[1]
    assert img.dtype == np.uint8 and img.shape == (7, 7, 3) and y == 1          # moth/1.png is i = 2: 7 rows


def test_npz_dataset(tmp_path):
    from dinov3_jax.eval import NpzDataset, make_eval_dataset
    imgs = np.arange(4 * 6 * 5 * 3, dtype=np.uint8).reshape(4, 6, 5, 3)
    np.savez(tmp_path / "d.npz", images=imgs, labels=np.array([3, 0, 3, 1]))
    ds = make_eval_dataset(tmp_path / "d.npz")
    assert isinstance(ds, NpzDataset) and len(ds) == 4 and ds.targets == [3, 0, 3, 1]
    img, y = ds[2]
    assert y == 3 and np.array_equal(img, imgs[2])
    np.savez(tmp_path / "bad.npz", images=imgs.astype(np.float32), labels=np.zeros(4))
    with pytest.raises(ValueError, match="uint8"):
        NpzDataset(tmp_path / "bad.npz")


def test_eval_max_taps_covers_every_window():
    from dinov3_jax import ops
    assert ops.eval_max_taps([(256, 256)], 256) == 5                 # identity / upscale: support 2
    assert ops.eval_max_taps([(375, 500)], 256) == 2 * 3 + 1          # 375 / 256 = 1.46: support 2.93
    assert ops.eval_max_taps([(64, 4000), (375, 500)], 256) == 7      # upscaled short side, long side 4000 / 16000


# --------------------------------------------------------------------------------------- the protocol, by hand
def test_oracle_ties_go_to_the_lower_bank_index():
    bank = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 0.0], [0.6, 0.8], [1.0, 0.0]])
    sims, idx, _ = knn_oracle.topk(np.array([[1.0, 0.0]]), bank, 4)
    assert idx.tolist() == [[0, 2, 4, 3]] and sims.tolist() == [[1.0, 1.0, 1.0, 0.6]]


def test_oracle_softmax_weighting():
    # two neighbours of class 1 at 0.5 and 0.4 against one of class 0 at 0.6: with T = 0.1 the weights are
    # e^6, e^5, e^4 over their sum, so class 0 (0.665) wins over class 1 (0.245 + 0.090 = 0.335) ...
    sims, idx, labels = np.array([[0.6, 0.5, 0.4]]), np.array([[0, 1, 2]]), np.array([0, 1, 1])
    assert knn_oracle.vote(sims, idx, labels, [3], 0.1, 2)[0, 0, :2].tolist() == [0, 1]
    # ... while at T = 1 the weights are nearly flat (0.367, 0.332, 0.301) and class 1 wins with 0.633
    assert knn_oracle.vote(sims, idx, labels, [3], 1.0, 2)[0, 0, :2].tolist() == [1, 0]
    # k = 1 looks at the first neighbour only
    assert knn_oracle.vote(sims, idx, labels, [1], 1.0, 2)[0, 0, 0] == 0


def test_oracle_top5_ties_go_to_the_lower_class_index():
    # equal sims: every neighbour weighs 1/4; classes 7 and 2 get 1/4 each, 5 gets 1/2; the classes without votes
    # (score 0) fill the top 5 from index 0 upwards
    sims, idx, labels = np.full((1, 4), 0.3), np.array([[0, 1, 2, 3]]), np.array([7, 5, 2, 5])
    assert knn_oracle.vote(sims, idx, labels, [4], 0.07, 9)[0, 0].tolist() == [5, 2, 7, 0, 1]


def test_oracle_accuracy_micro_percent():
    preds = np.array([[[1, 2, 3, 4, 5]], [[0, 1, 2, 3, 4]], [[9, 8, 7, 6, 5]], [[2, 0, 1, 3, 4]]])
    assert knn_oracle.accuracy(preds, [1, 1, 0, 2], [20]) == {20: {"top1": 50.0, "top5": 75.0}}
