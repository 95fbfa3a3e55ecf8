"""-m gpu: linear-probe evaluation (csrc/linear.cu, d3_train_resized_crop in csrc/knn.cu, d3_sgd_momentum in
csrc/optim.cu, dinov3_jax/eval/linear.py).  The train crop against torchvision's uint8 resized_crop + hflip, the
cross-entropy against float64, SGD against torch.optim.SGD, LinearClassifiers against a torch restatement with the same
roundings and against the plain fp32 DINOv2 module, and the evaluation end to end through --eval-only and do_train."""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


# ------------------------------------------------------------------------------------------------ train crop
def _image(H, W, rng):
    yy, xx = np.mgrid[0:H, 0:W]
    base = 127 + 100 * np.sin(xx[..., None] / 7.0 + np.arange(3)) * np.cos(yy[..., None] / 11.0)
    return np.clip(base + rng.normal(0, 40, (H, W, 3)), 0, 255).astype(np.uint8)


def _torchvision_resized_crop(img, box, S):
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms.v2 import functional as TF
    i, j, h, w, flip = box
    t = TF.resized_crop(torch.from_numpy(img).permute(2, 0, 1), i, j, h, w, [S, S],
                        interpolation=InterpolationMode.BICUBIC, antialias=True)
    if flip:
        t = TF.hflip(t)
    return t.permute(1, 2, 0).numpy()


def test_train_resized_crop_equals_torchvision(native):
    from dinov3_jax import ops
    from dinov3_jax.eval.knn import _pack
    from dinov3_jax.eval.linear import sample_crop_box
    rng = np.random.default_rng(0)
    sizes = [(375, 500), (500, 375), (224, 224), (1000, 257), (64, 4000), (1000, 10), (301, 333), (90, 120)]
    imgs = [_image(H, W, rng) for H, W in sizes]
    S = 224
    boxes = [(10, 20, 300, 400, 0),        # downscale
             (100, 50, 60, 90, 1),         # upscale, flipped
             (0, 0, 224, 224, 1),          # identity, flipped
             (3, 1, 997, 256, 0),          # whole width, tall
             sample_crop_box(torch.Generator().manual_seed(1), 64, 4000) + (1,),
             sample_crop_box(torch.Generator().manual_seed(0), 1000, 10) + (0,),        # the fallback box
             (150, 100, 151, 233, 1),      # the bottom-right corner
             (0, 0, 90, 120, 0)]           # the whole image, upscaled
    assert boxes[5][:4] == (493, 0, 13, 10)
    flat, desc, _ = _pack([(im, 0) for im in imgs])
    bx = torch.tensor(boxes, dtype=torch.int32)
    taps = ops.train_max_taps(boxes, S)
    u8 = torch.empty(len(imgs), S, S, 3, dtype=torch.uint8, device="cuda")
    ops.train_resized_crop(flat.cuda(), desc.cuda(), bx.cuda(), u8, max_taps=taps)
    x = torch.empty(len(imgs), S, S, 3, dtype=bf16, device="cuda")
    ops.train_resized_crop(flat.cuda(), desc.cuda(), bx.cuda(), x, max_taps=taps, mean=MEAN, std=STD)
    mean, std = torch.tensor(MEAN, device="cuda"), torch.tensor(STD, device="cuda")
    for b, (im, box) in enumerate(zip(imgs, boxes)):
        want = _torchvision_resized_crop(im, box, S)
        got = u8[b].cpu().numpy()
        assert np.array_equal(got, want), (sizes[b], box, np.abs(got.astype(int) - want.astype(int)).max(),
                                           (got != want).sum())
        norm = (torch.from_numpy(want).cuda().float() / 255 - mean) / std
        assert ((x[b].float() - norm).abs() <= norm.abs() * 2.0 ** -8 + 1e-6).all(), sizes[b]
    # a second launch gives the same bits
    again = torch.empty_like(u8)
    ops.train_resized_crop(flat.cuda(), desc.cuda(), bx.cuda(), again, max_taps=taps)
    assert torch.equal(again, u8)


# ------------------------------------------------------------------------------------------------ cross-entropy
@pytest.mark.parametrize("C", [2, 10, 1000, 21841])
@pytest.mark.parametrize("B", [1, 37, 128])
@pytest.mark.parametrize("G", [1, 13])
def test_linear_xent_against_float64(native, B, C, G):
    from dinov3_jax import ops
    Cp = -(-C // 8) * 8
    g = torch.Generator().manual_seed(B * 100003 + C * 7 + G)
    z = torch.full((B, G * Cp), float("nan"))                       # the padding columns must never be read
    for k in range(G):
        z[:, k * Cp:k * Cp + C] = (torch.rand(B, C, generator=g) * 2 - 1) * 100.0
    y = torch.randint(0, C, (B,), generator=g, dtype=torch.int32)
    y[0] = 0
    y[-1] = C - 1
    loss = torch.empty(G, device="cuda")
    Bp = B + 5
    dz = torch.full((Bp, G * Cp), 7.0, dtype=bf16, device="cuda")
    ops.linear_xent_fwd_bwd(z.cuda(), y.cuda(), C, Cp, loss, dz)
    for k in range(G):
        zk = z[:, k * Cp:k * Cp + C].double()
        lse = torch.logsumexp(zk, 1)
        want_loss = (lse - zk[torch.arange(B), y.long()]).mean()
        assert loss[k].item() == pytest.approx(want_loss.item(), rel=1e-5, abs=1e-4), k
        p = torch.softmax(zk, 1)
        p[torch.arange(B), y.long()] -= 1.0
        want = p / B
        got = dz[:B, k * Cp:k * Cp + C].double().cpu()
        # bf16 rounding, plus a few fp32 ulps of 1 where the label's probability is close to 1
        assert ((got - want).abs() <= want.abs() * 2.0 ** -8 + 2.5e-7 / B).all(), k
        assert (dz[:B, k * Cp + C:(k + 1) * Cp] == 0).all()
    assert (dz[B:] == 7.0).all()                                      # rows past the batch are not written
    again = torch.empty(G, device="cuda")
    ops.linear_xent_fwd_bwd(z.cuda(), y.cuda(), C, Cp, again, dz)
    assert torch.equal(again, loss)


# ------------------------------------------------------------------------------------------------ SGD
def test_sgd_momentum_matches_torch_sgd(native):
    from dinov3_jax import ops
    G, Cp, K = 3, 16, 24
    lrs = [0.5, 0.05, 0.003]
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(G * Cp, K, generator=g)
    grads = [torch.randn(G * Cp, K, generator=g) for _ in range(3)]
    ref = [torch.nn.Parameter(p0[k * Cp:(k + 1) * Cp].clone().cuda()) for k in range(G)]
    opt = torch.optim.SGD([{"params": [ref[k]], "lr": lrs[k]} for k in range(G)], momentum=0.9, weight_decay=0)
    p, m = p0.cuda().contiguous(), torch.zeros(G * Cp, K, device="cuda")
    pb = torch.empty(G * Cp, K, dtype=bf16, device="cuda")
    lr = torch.tensor(lrs, device="cuda")
    for step in range(3):
        for k in range(G):
            ref[k].grad = grads[step][k * Cp:(k + 1) * Cp].cuda()
        opt.step()
        ops.sgd_momentum(p, grads[step].cuda(), m, pb, lr, Cp, lr_scale=1.0, momentum=0.9, first=step == 0)
        want = torch.cat([r.detach() for r in ref])
        assert ((p - want).abs() <= 1e-6 * want.abs().max()).all(), step
        assert torch.equal(pb, p.to(bf16))
    # the bias form (one column) and a learning-rate scale
    b, mb, gb = torch.zeros(G * Cp, device="cuda"), torch.zeros(G * Cp, device="cuda"), torch.ones(G * Cp, device="cuda")
    ops.sgd_momentum(b, gb, mb, None, lr, Cp, lr_scale=0.5, first=True)
    assert torch.allclose(b, -0.5 * lr.repeat_interleave(Cp), rtol=1e-6)


# ------------------------------------------------------------------------------------------------ classifiers
D, NCLS, B, STEPS = 384, 10, 128, 50


def _cluster_data(seed, n, spread=1.0):
    g = torch.Generator().manual_seed(seed)
    centers = 0.1 * torch.randn(NCLS, 5 * D, generator=g)
    y = torch.randint(0, NCLS, (n,), generator=g)
    x = centers[y] + spread * torch.randn(n, 5 * D, generator=g)
    return x, y


def _batches(n, seed):
    g = torch.Generator().manual_seed(seed)
    order = torch.cat([torch.randperm(n, generator=g) for _ in range(-(-STEPS * B // n))])
    return [order[t * B:(t + 1) * B] for t in range(STEPS)]


def _restated_step(Ws, bs, bufs, x, y, lrs, t, same_rounding):
    """One step of the torch restatement: fp32 logits from (bf16 inputs and weights, same_rounding) or fp32 ones, the
    summed batch-mean cross-entropies, SGD(momentum=0.9) with the cosine schedule."""
    from dinov3_jax.eval.linear import classifier_grid, cosine_lr
    scale = cosine_lr(1.0, t, STEPS)
    for k, (n, a, _) in enumerate(classifier_grid()):
        xw = x[:, (4 - n) * D:(4 + int(a)) * D]
        W = Ws[k].to(bf16).float() if same_rounding else Ws[k]
        logits = xw @ W.T + bs[k]
        pr = torch.softmax(logits.double(), 1).float()
        pr[torch.arange(B), y] -= 1.0
        dz = pr / B
        if same_rounding:
            dz = dz.to(bf16).float()
        gW, gb = dz.T @ xw, dz.sum(0)
        for j, (p, gr) in enumerate(((Ws[k], gW), (bs[k], gb))):
            buf = bufs.get((k, j))
            bufs[(k, j)] = gr.clone() if buf is None else buf * 0.9 + gr
            p -= (lrs[k] * scale) * bufs[(k, j)]


def test_linear_classifiers_against_torch_restatements(native):
    from dinov3_jax.eval.linear import LinearClassifiers, classifier_grid
    torch.backends.cuda.matmul.allow_tf32 = False
    xtr, ytr = _cluster_data(0, 3000)
    xva, yva = _cluster_data(0, 8000 + 3000)
    xva, yva = xva[3000:], yva[3000:]
    xtr_b = xtr.to(bf16)
    clf = LinearClassifiers(D, NCLS, B, STEPS, seed=3, device="cuda")
    init = clf.state_dict()
    grid = classifier_grid()
    lrs = [lr * B / 256 for _, _, lr in grid]
    runs = {}
    for same in (True, False):
        Ws = [init[name]["weight"].clone().cuda() for name in clf.names]
        bs = [init[name]["bias"].clone().cuda() for name in clf.names]
        runs[same] = (Ws, bs, {})
    for t, idx in enumerate(_batches(3000, 1)):
        clf.step(xtr_b[idx].cuda(), ytr[idx], t)
        for same in (True, False):
            x = (xtr_b[idx] if same else xtr[idx]).float().cuda()
            _restated_step(*runs[same], x, ytr[idx].cuda(), lrs, t, same)
    got = clf.state_dict()
    Ws, bs, _ = runs[True]
    for k, name in enumerate(clf.names):
        mine = torch.cat([got[name]["weight"], got[name]["bias"][:, None]], 1)
        ref = torch.cat([Ws[k], bs[k][:, None]], 1).cpu()
        err = ((mine - ref).norm() / ref.norm()).item()
        # the bias alone is small and carries every bf16 rounding of dZ that the two GEMM orders resolve differently
        b_err = ((got[name]["bias"] - bs[k].cpu()).norm() / max(bs[k].norm().item(), 1e-12)).item()
        assert err < 1e-3 and b_err < 5e-3, (name, err, b_err)
    # the plain fp32 module: val top-1 within 1 point per classifier, and the same best classifier
    res = clf.evaluate(xva.to(bf16), yva)
    Ws, bs, _ = runs[False]
    xv = xva.cuda()
    ref = {}
    for k, (n, a, _) in enumerate(grid):
        logits = xv[:, (4 - n) * D:(4 + int(a)) * D] @ Ws[k].T + bs[k]
        ref[clf.names[k]] = 100.0 * (logits.argmax(1).cpu() == yva).double().mean().item()
    top1 = [res[name]["top1"] for name in clf.names]
    # fp32: 10 % (the smallest lrs) .. 95.8 % (4 blocks + avgpool, lr 0.05), the runner-up 0.3 points below
    assert max(top1) > 80.0 and min(top1) < max(top1) - 5.0, top1
    for name in clf.names:
        assert abs(res[name]["top1"] - ref[name]) <= 1.0, (name, res[name], ref[name])
    best = max(clf.names, key=lambda nm: (res[nm]["top1"], -clf.names.index(nm)))
    best_ref = max(clf.names, key=lambda nm: (ref[nm], -clf.names.index(nm)))
    assert best == best_ref, (best, res[best], best_ref, ref[best_ref])


def test_linear_classifiers_are_bit_reproducible(native):
    from dinov3_jax.eval.linear import LinearClassifiers
    xtr, ytr = _cluster_data(2, 600)
    states = []
    for _ in range(2):
        clf = LinearClassifiers(D, NCLS, B, 5, n_last_blocks_list=[1, 4], seed=7, device="cuda")
        for t, idx in enumerate(_batches(600, 3)[:5]):
            clf.step(xtr[idx].to(bf16).cuda(), ytr[idx], t)
        states.append(clf.state_dict())
    for name in states[0]:
        assert torch.equal(states[0][name]["weight"], states[1][name]["weight"])
        assert torch.equal(states[0][name]["bias"], states[1][name]["bias"])


# ------------------------------------------------------------------------------------------------ end to end
def _tiny_vit_checkpoint(path, depth=4):
    from dinov3_jax.checkpointer import save_checkpoint, tree_from_flat
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=384, depth=depth, heads=6, layerscale=0.5)
    flat = init_backbone(cfg, torch.Generator().manual_seed(0))
    save_checkpoint(path, iteration=4, params={"teacher_backbone": tree_from_flat(flat)})
    return flat


def _color_folder(root, n_per_class, seed):
    from PIL import Image
    rng = np.random.default_rng(seed)
    for c, rgb in enumerate(((200, 40, 40), (40, 60, 210))):
        (root / f"class{c}").mkdir(parents=True)
        for i in range(n_per_class):
            H, W = int(rng.integers(60, 120)), int(rng.integers(60, 120))
            img = np.clip(np.array(rgb) + rng.normal(0, 30, (H, W, 3)), 0, 255).astype(np.uint8)
            Image.fromarray(img).save(root / f"class{c}" / f"{i:03d}.png")


def _opts(tmp_path, workers=2):
    return ["student.arch=vit_small", f"evaluation.linear.train_dataset_path={tmp_path / 'train'}",
            f"evaluation.linear.val_dataset_path={tmp_path / 'val'}", "evaluation.linear.epochs=2",
            "evaluation.linear.epoch_length=10", "evaluation.linear.batch_size=8", "evaluation.linear.resize_size=72",
            "evaluation.linear.crop_size=64", f"evaluation.linear.num_workers={workers}"]


def test_write_linear_inputs_layout(native, tmp_path):
    from dinov3_jax import ops
    from dinov3_jax.eval.linear import write_linear_inputs
    from dinov3_jax.models import DinoVisionTransformer
    from features_helpers import tree
    flat = _tiny_vit_checkpoint(tmp_path / "w")
    model = DinoVisionTransformer(tree(flat), embed_dim=384, n_blocks=4, num_heads=6)
    x = torch.randn(3, 64, 64, 3, generator=torch.Generator().manual_seed(0)).cuda()
    out = torch.zeros(3, 5 * 384 + 8, dtype=bf16, device="cuda")
    write_linear_inputs(model, x, 4, out)
    layers = model.get_intermediate_layers(x, n=4, return_class_token=True)
    mean = ops.pool_tokens(layers[-1][0], torch.empty(3, 1, 384, device="cuda"), copy_tokens=False).view(3, 384)
    want = torch.cat([c for _, c in layers] + [mean], 1).to(bf16)
    assert torch.equal(out[:, :5 * 384], want) and (out[:, 5 * 384:] == 0).all()
    assert (mean - layers[-1][0].mean(1)).abs().max().item() < 1e-5


def test_eval_only_linear_writes_results_linear_json(native, tmp_path):
    from dinov3_jax.eval.linear import classifier_grid, classifier_name
    from dinov3_jax.train.train import main
    _tiny_vit_checkpoint(tmp_path / "weights")
    _color_folder(tmp_path / "train", 12, 0)
    _color_folder(tmp_path / "val", 8, 1)
    outs = []
    for run, workers in (("a", 2), ("b", 0)):
        res = main(["--eval-only", "--eval", "linear", "--eval-pretrained-weights", str(tmp_path / "weights"),
                    "--output-dir", str(tmp_path / run), "--opts"] + _opts(tmp_path, workers))
        outs.append((tmp_path / run / "eval" / "manual_5" / "results_linear.json").read_text())
        written = json.loads(outs[-1])
        names = [classifier_name(*g) for g in classifier_grid()]
        assert sorted(written) == sorted(names + ["best_classifier"]) and written == res
        best = written["best_classifier"]
        assert best["top1"] > 90.0 and best["top1"] == max(written[n]["top1"] for n in names), best
        assert best["name"] == next(n for n in names if written[n]["top1"] == best["top1"])
    assert outs[0] == outs[1]                  # same seed, other worker count: the same file


def test_do_train_calls_do_linear_eval_at_the_eval_period(native, tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch, train
    calls = []
    monkeypatch.setattr(train, "do_linear_eval", lambda config, model, header: calls.append(header) or {})
    monkeypatch.setattr(train, "do_test", lambda *a: pytest.fail("no k-NN datasets are configured"))
    opts = _opts(tmp_path) + ["train.batch_size_per_gpu=2", f"train.output_dir={tmp_path}", "checkpointing.period=100",
                              "evaluation.eval_period_iterations=2", "dino.head_n_prototypes=1024",
                              "ibot.head_n_prototypes=1024"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    train.do_train(config, SSLMetaArch(config), max_iters=4, print_freq=1)
    assert calls == ["training_1", "training_3"]
