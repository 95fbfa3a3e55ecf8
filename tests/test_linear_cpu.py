"""Linear-probe evaluation without a GPU: the `evaluation.linear` configuration block, the --eval / --eval-only flags,
the no-dataset path of do_linear_eval, the train-crop sampler against torchvision's RandomResizedCrop.get_params, the
cosine schedule against CosineAnnealingLR, the classifier grid and names, and what ptxas makes of the new kernels."""
import json
import os
import re
import subprocess

import pytest
import torch


def test_defaults_carry_the_linear_block():
    from dinov3_jax.configs import get_default_config
    lin = get_default_config().evaluation.linear
    assert lin == {"train_dataset_path": "", "val_dataset_path": "", "epochs": 10, "epoch_length": 1250,
                   "batch_size": 128,
                   "learning_rates": [1e-5, 2e-5, 5e-5, 1e-4, 2e-4, 5e-4, 1e-3, 2e-3, 5e-3, 1e-2, 2e-2, 5e-2, 0.1],
                   "n_last_blocks_list": [1, 4], "avgpools": [False, True], "crop_size": 224, "resize_size": 256,
                   "num_workers": 8, "seed": 0}


def test_do_linear_eval_without_datasets_returns_empty_and_touches_no_gpu(capsys):
    from dinov3_jax.configs import get_default_config
    from dinov3_jax.train.train import do_linear_eval
    assert do_linear_eval(get_default_config(), None, "training_9") == {}
    assert "nothing evaluated" in capsys.readouterr().out
    assert not torch.cuda.is_initialized()


def test_eval_type_other_than_knn_or_linear_raises(tmp_path):
    from dinov3_jax.train.train import main
    with pytest.raises(NotImplementedError, match="knn"):
        main(["--eval=other", "--output-dir", str(tmp_path)])


def test_eval_only_linear_reaches_do_linear_eval_and_never_do_train(tmp_path, monkeypatch):
    from dinov3_jax.train import train
    calls = []
    monkeypatch.setattr(train, "do_linear_eval", lambda config, model, header: calls.append((str(model), header)) or {"ok": 2})
    monkeypatch.setattr(train, "do_test", lambda *a, **k: pytest.fail("--eval linear must not run k-NN"))
    monkeypatch.setattr(train, "do_train", lambda *a, **k: pytest.fail("--eval-only must not train"))
    ck = tmp_path / "ckpt" / "7"
    ck.mkdir(parents=True)
    (ck / "manifest.json").write_text(json.dumps({"iteration": 7, "leaves": {}, "scalars": {}}))
    assert train.main(["--eval-only", "--eval", "linear", "--output-dir", str(tmp_path)]) == {"ok": 2}
    assert calls == [(str(ck), "manual_8")]


def _draws(sampler, sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return [sampler(g, H, W) for H, W in sizes]


SIZES = [(375, 500), (500, 375), (224, 224), (1000, 257), (64, 4000), (1000, 10), (10, 1000), (7, 7), (301, 333)]


def test_crop_sampler_makes_torchvision_get_params_draws():
    from torchvision.transforms import RandomResizedCrop
    from dinov3_jax.eval.linear import sample_crop_box
    for seed in range(5):
        torch.manual_seed(seed)
        want = [RandomResizedCrop.get_params(torch.empty(3, H, W), (0.08, 1.0), (3 / 4, 4 / 3)) for H, W in SIZES * 3]
        got = _draws(sample_crop_box, SIZES * 3, seed)
        assert got == [tuple(w) for w in want], seed
    # narrower than the smallest ratio: no attempt fits, the fallback keeps the width and takes h = round(w / (3/4))
    assert sample_crop_box(torch.Generator().manual_seed(0), 1000, 10) == (493, 0, 13, 10)
    # wider than the largest ratio: the height is kept
    assert sample_crop_box(torch.Generator().manual_seed(0), 10, 1000) == (0, 493, 10, 13)


def test_train_boxes_interleave_crop_and_flip_draws_like_torchvision():
    from torchvision.transforms import RandomHorizontalFlip, RandomResizedCrop
    from dinov3_jax.eval.linear import sample_train_boxes
    torch.manual_seed(3)
    want = []
    for H, W in SIZES:
        i, j, h, w = RandomResizedCrop.get_params(torch.empty(3, H, W), (0.08, 1.0), (3 / 4, 4 / 3))
        flipped = RandomHorizontalFlip(0.5)(torch.arange(2).view(1, 1, 2))[0, 0, 0].item() == 1
        want.append([i, j, h, w, int(flipped)])
    got = sample_train_boxes(torch.Generator().manual_seed(3), SIZES)
    assert got.dtype == torch.int32 and got.tolist() == want
    assert 0 < sum(r[4] for r in want) < len(want)


def test_cosine_schedule_equals_cosine_annealing_lr():
    from dinov3_jax.eval.linear import cosine_lr
    T = 37
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([{"params": [p], "lr": 0.05}], momentum=0.9, weight_decay=0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T, eta_min=0)
    for t in range(T):
        assert cosine_lr(0.05, t, T) == pytest.approx(opt.param_groups[0]["lr"], rel=1e-12, abs=1e-18), t
        opt.step()
        sched.step()


def test_classifier_grid_and_names():
    from dinov3_jax.eval.linear import LEARNING_RATES, classifier_grid, classifier_name
    grid = classifier_grid()
    assert len(grid) == 52 and grid[0] == (1, False, 1e-5) and grid[13] == (1, True, 1e-5) and grid[26] == (4, False, 1e-5)
    assert [lr for _, _, lr in grid[:13]] == list(LEARNING_RATES)
    names = [classifier_name(*g) for g in grid]
    assert names[0] == "classifier_1_blocks_avgpool_False_lr_0_00001"
    assert names[12] == "classifier_1_blocks_avgpool_False_lr_0_10000"
    assert names[-1] == "classifier_4_blocks_avgpool_True_lr_0_10000"
    assert names[20] == "classifier_1_blocks_avgpool_True_lr_0_00200"
    assert len(set(names)) == 52


def test_infinite_sampler_is_seeded_and_crosses_epochs():
    from dinov3_jax.eval.linear import InfiniteBatchSampler
    s = InfiniteBatchSampler(10, 4, 6, seed=5)
    a, b = list(s), list(s)
    assert a == b and len(a) == 6 and all(len(x) == 4 for x in a)
    g = torch.Generator().manual_seed(5)
    flat = torch.randperm(10, generator=g).tolist() + torch.randperm(10, generator=g).tolist() + \
        torch.randperm(10, generator=g).tolist()
    assert sum(a, []) == flat[:24]
    assert list(InfiniteBatchSampler(10, 4, 6, seed=6)) != a


def test_train_max_taps_covers_every_box():
    from dinov3_jax import ops
    assert ops.train_max_taps([(0, 0, 100, 224, 0)], 224) == 5          # upscale / identity: support 2
    assert ops.train_max_taps([(0, 0, 500, 300, 1)], 224) == 2 * 5 + 1   # 500 / 224 = 2.23: support 4.46
    assert ops.train_max_taps([(0, 0, 20, 30, 0), (0, 0, 224, 4000, 0)], 224) == 2 * 36 + 1


def test_new_kernels_have_no_stack_or_spills(tmp_path):
    import importlib.util
    from conftest import ROOT
    pkg = os.path.join(ROOT, "dinov3-jax_b200")
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(pkg, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    seen = set()
    for src in ("knn.cu", "linear.cu", "optim.cu"):
        cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(pkg, "csrc", src), "-o", str(tmp_path / "x.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                           r"(\d+) bytes spill loads", r.stderr)
        for name, stack, st, ld in props:
            if any(k in name for k in ("eval_resize_crop_kernel", "linear_inputs_kernel", "linear_xent_kernel",
                                       "sgd_momentum_kernel")):
                seen.add(name)
                assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)
    assert len(seen) == 5, seen
