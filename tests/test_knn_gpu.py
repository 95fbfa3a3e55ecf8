"""-m gpu: k-NN evaluation (csrc/knn.cu, dinov3_jax/eval).  d3_topk_merge and d3_knn_vote against the float64
statement of the protocol (tests/knn_oracle.py) on the same bf16-rounded features, d3_eval_resize_crop against
torchvision's uint8 Resize + CenterCrop, KnnClassifier.evaluate against a torch fp32 restatement of the upstream
k-NN code, and the evaluation end to end through --eval-only, extract_features and do_train."""
import json

import numpy as np
import pytest
import torch

import knn_oracle

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16


def _unit(n, d, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, d, generator=g)


def _clf(bank, labels=None, C=1, **kw):
    from dinov3_jax.eval import KnnClassifier
    labels = torch.zeros(bank.shape[0], dtype=torch.int64) if labels is None else labels
    return KnnClassifier(bank, labels, C, device="cuda", **kw)


def _bf16_queries(q):
    from dinov3_jax import ops
    out = torch.zeros(q.shape[0], q.shape[1], dtype=bf16, device="cuda")
    ops.knn_normalize(q.to("cuda", f32).contiguous(), y_bf16=out)
    return out.double().cpu().numpy()


def _check_against_float64(sims, idx, ref_s, ref_i, all_s):
    """sims within 1e-5; an index may differ from float64's only where float64 has another candidate within 1e-5."""
    sims, idx = sims.cpu().numpy(), idx.cpu().numpy()
    assert np.abs(sims - ref_s).max() < 1e-5
    got = np.take_along_axis(all_s, idx, 1)                        # float64 sims of the returned rows
    assert np.abs(got - sims).max() < 1e-5
    k = idx.shape[1]
    nxt = np.sort(all_s, 1)[:, ::-1][:, : k + 1]                   # float64's (k+1) best values
    for q, j in zip(*np.nonzero(idx != ref_i)):
        near = (j > 0 and nxt[q, j - 1] - nxt[q, j] < 1e-5) or nxt[q, j] - nxt[q, j + 1] < 1e-5
        assert near, (q, j, idx[q, j], ref_i[q, j])
    assert (idx != ref_i).mean() < 0.01


@pytest.mark.parametrize("N", [3000, 100003])
def test_topk_merge_against_float64(native, N):
    D, Q = 64, 160
    bank, queries = _unit(N, D, N), _unit(Q, D, N + 1)
    chunks = (1024, 65536) if N == 3000 else (4096, 33000)
    clfs = [_clf(bank, chunk=c, query_tile=t) for c, t in zip(chunks, (Q, 37))]
    bank64 = clfs[0].bank[:N].double().cpu().numpy()
    q64 = _bf16_queries(queries)
    for k in (1, 10, 200, 1024):
        ref_s, ref_i, all_s = knn_oracle.topk(q64, bank64, k)
        outs = [c.search(queries, k) for c in clfs]
        _check_against_float64(*outs[0], ref_s, ref_i, all_s)
        for s, i in outs[1:]:                                       # other chunk size and query tiling: same bits
            assert torch.equal(s, outs[0][0]) and torch.equal(i, outs[0][1]), k
        again = clfs[0].search(queries, k)
        assert torch.equal(again[0], outs[0][0]) and torch.equal(again[1], outs[0][1]), k
        assert outs[0][1].dtype == torch.int64 and outs[0][0].dtype == f32


def test_topk_merge_duplicated_rows_lower_index_first(native):
    N, D = 9000, 32
    bank = _unit(N, D, 5)
    for dup in (17, 4000, 8999):
        bank[dup] = bank[5]
    clf = _clf(bank, chunk=512)
    s, i = clf.search(bank[5:6], 6)
    assert i[0, :4].tolist() == [5, 17, 4000, 8999]
    assert torch.equal(s[0, :4], s[0, :1].expand(4))
    # all rows equal: the k lowest indices, whatever the chunking
    same = bank[:1].expand(2500, D).contiguous()
    for chunk in (256, 4096):
        s, i = _clf(same, chunk=chunk).search(same[:3], 300)
        assert i.tolist() == [list(range(300))] * 3


def test_topk_merge_argument_errors(native):
    from dinov3_jax import _native, ops
    s = torch.zeros(4, 64, device="cuda")
    ts, ti = torch.empty(4, 1025, device="cuda"), torch.empty(4, 1025, dtype=torch.int32, device="cuda")
    with pytest.raises(_native.NativeError, match="1024"):
        ops.topk_merge(s, ts, ti, offset=0)
    with pytest.raises(ValueError):
        _clf(_unit(10, 16, 0)).search(_unit(2, 16, 1), 11)


@pytest.mark.parametrize("C", [1000, 21841])
def test_knn_vote_against_float64(native, C):
    from dinov3_jax import ops
    Q, K, N = 300, 200, 50000
    g = torch.Generator().manual_seed(C)
    sims = torch.sort(torch.rand(Q, K, generator=g) * 0.6 + 0.2, 1, descending=True).values
    idx = torch.randint(0, N, (Q, K), generator=g, dtype=torch.int32)
    # few classes per query so that the scores collect several neighbours
    labels = torch.randint(0, C, (N,), generator=g, dtype=torch.int32)
    labels[torch.randint(0, N, (N // 2,), generator=g)] = torch.randint(0, 7, (N // 2,), generator=g, dtype=torch.int32)
    nb = [10, 20, 100, 200]
    preds = torch.empty(Q, len(nb), 5, dtype=torch.int32, device="cuda")
    ops.knn_vote(sims.cuda(), idx.cuda(), labels.cuda(), nb, 0.07, C, preds)
    want = knn_oracle.vote(sims.numpy(), idx.numpy(), labels.numpy(), nb, 0.07, C)
    assert np.array_equal(preds.cpu().numpy(), want)
    again = torch.empty_like(preds)
    ops.knn_vote(sims.cuda(), idx.cuda(), labels.cuda(), nb, 0.07, C, again)
    assert torch.equal(again, preds)


# ------------------------------------------------------------------------------------------------ eval transform
SIZES = [(375, 500), (500, 375), (224, 224), (1000, 257), (64, 4000), (301, 333)]     # (H, W)


def _torchvision_crop(img, resize, crop):
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms.v2 import functional as TF
    t = torch.from_numpy(img).permute(2, 0, 1)
    r = TF.resize(t, [resize], interpolation=InterpolationMode.BICUBIC, antialias=True)
    return TF.center_crop(r, [crop]).permute(1, 2, 0).numpy()


def test_eval_resize_crop_against_torchvision(native):
    from dinov3_jax import ops
    from dinov3_jax.eval.knn import _pack
    rng = np.random.default_rng(0)
    imgs = []
    for H, W in SIZES:          # smooth structure plus noise: overshooting edges and flat areas
        yy, xx = np.mgrid[0:H, 0:W]
        base = 127 + 100 * np.sin(xx[..., None] / 7.0 + np.arange(3)) * np.cos(yy[..., None] / 11.0)
        imgs.append(np.clip(base + rng.normal(0, 40, (H, W, 3)), 0, 255).astype(np.uint8))
    flat, desc, _ = _pack([(im, 0) for im in imgs])
    taps = ops.eval_max_taps(SIZES, 256)
    u8 = torch.empty(len(imgs), 224, 224, 3, dtype=torch.uint8, device="cuda")
    ops.eval_resize_crop(flat.cuda(), desc.cuda(), u8, resize=256, max_taps=taps)
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    x = torch.empty(len(imgs), 224, 224, 3, dtype=bf16, device="cuda")
    ops.eval_resize_crop(flat.cuda(), desc.cuda(), x, resize=256, max_taps=taps, mean=mean, std=std)
    for b, im in enumerate(imgs):
        want = _torchvision_crop(im, 256, 224).astype(np.int32)
        got = u8[b].cpu().numpy().astype(np.int32)
        assert np.abs(got - want).max() <= 1, (SIZES[b], np.abs(got - want).max())
        norm = ((u8[b].float() / 255 - torch.tensor(mean, device="cuda")) / torch.tensor(std, device="cuda")).to(bf16)
        assert (x[b].float() - norm.float()).abs().max().item() <= 0.02, SIZES[b]
    # a smaller crop of a whole batch of one image size, and the identity (224 -> 224)
    same = _pack([(imgs[0], 0)] * 3)
    out = torch.empty(3, 160, 160, 3, dtype=torch.uint8, device="cuda")
    ops.eval_resize_crop(same[0].cuda(), same[1].cuda(), out, resize=192, max_taps=ops.eval_max_taps([SIZES[0]], 192))
    assert np.abs(out[2].cpu().numpy().astype(int) - _torchvision_crop(imgs[0], 192, 160).astype(int)).max() <= 1
    ident = _pack([(imgs[2], 0)])
    out = torch.empty(1, 224, 224, 3, dtype=torch.uint8, device="cuda")
    ops.eval_resize_crop(ident[0].cuda(), ident[1].cuda(), out, resize=224, max_taps=5)
    assert np.array_equal(out[0].cpu().numpy(), imgs[2])


# ------------------------------------------------------------------------------------------------ classifier
def _clusters(C, N, Q, D, spread, seed):
    g = torch.Generator().manual_seed(seed)
    centers = torch.nn.functional.normalize(torch.randn(C, D, generator=g), dim=1)
    ytr, yva = torch.randint(0, C, (N,), generator=g), torch.randint(0, C, (Q,), generator=g)
    xtr = centers[ytr] + spread * torch.randn(N, D, generator=g) / D ** 0.5
    xva = centers[yva] + spread * torch.randn(Q, D, generator=g) / D ** 0.5
    return xtr, ytr, xva, yva


def _upstream_knn(xtr, ytr, xva, yva, C, nb_knn, T):
    """torch fp32 restatement of the upstream k-NN module: mm, topk, softmax of the max-k sims, one-hot weighted sums."""
    tr, va = torch.nn.functional.normalize(xtr.cuda(), dim=1), torch.nn.functional.normalize(xva.cuda(), dim=1)
    sims, idx = (va @ tr.T).topk(max(nb_knn), dim=1)
    w = torch.softmax(sims / T, 1)
    votes = torch.nn.functional.one_hot(ytr.cuda()[idx], C) * w[..., None]
    out = {}
    for k in nb_knn:
        top5 = votes[:, :k].sum(1).topk(5, dim=1).indices
        y = yva.cuda()[:, None]
        out[k] = {"top1": 100.0 * (top5[:, 0:1] == y).double().mean().item(),
                  "top5": 100.0 * (top5 == y).any(1).double().mean().item()}
    return out


def test_knn_classifier_evaluate_against_upstream_fp32(native):
    C, N, Q, D, nb = 100, 20000, 2000, 768, [10, 20, 100, 200]
    # fp32 top-1 95.8 % at k = 10 .. 99.95 % at k = 200.  (In a noisier regime, 56 .. 95 %, the bf16 bank moves
    # a few borderline queries: 0.1 - 0.2 pp, DESIGN.md section 9.)
    xtr, ytr, xva, yva = _clusters(C, N, Q, D, 4.0, 0)
    got = _clf(xtr, ytr, C, chunk=8192, query_tile=1024).evaluate(xva, yva, nb, 0.07)
    want = _upstream_knn(xtr, ytr, xva, yva, C, nb, 0.07)
    assert 50.0 < got[10]["top1"] < 99.0                            # a regime where the neighbours matter
    for k in nb:
        for m in ("top1", "top5"):
            assert abs(got[k][m] - want[k][m]) <= 0.1 + 1e-9, (k, m, got[k], want[k])
    xtr, ytr, xva, yva = _clusters(C, N, Q, D, 0.3, 1)
    sep = _clf(xtr, ytr, C).evaluate(xva, yva, nb, 0.07)
    assert all(v["top1"] == 100.0 and v["top5"] == 100.0 for v in sep.values()), sep


# ------------------------------------------------------------------------------------------------ end to end
def _tiny_vit_checkpoint(path, iteration=4):
    from dinov3_jax.checkpointer import save_checkpoint, tree_from_flat
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=384, depth=2, heads=6, layerscale=0.5)
    flat = init_backbone(cfg, torch.Generator().manual_seed(0))
    save_checkpoint(path, iteration=iteration, params={"teacher_backbone": tree_from_flat(flat)})
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


def _opts(tmp_path):
    return ["student.arch=vit_small", f"evaluation.knn.train_dataset_path={tmp_path / 'train'}",
            f"evaluation.knn.val_dataset_path={tmp_path / 'val'}", "evaluation.knn.nb_knn=[1,5,10]",
            "evaluation.knn.resize_size=72", "evaluation.knn.crop_size=64", "evaluation.knn.batch_size=7",
            "evaluation.knn.num_workers=2"]


def test_eval_only_writes_results_knn_json(native, tmp_path):
    from dinov3_jax.train.train import main
    _tiny_vit_checkpoint(tmp_path / "weights")
    _color_folder(tmp_path / "train", 12, 0)
    _color_folder(tmp_path / "val", 8, 1)
    res = main(["--eval-only", "--eval-pretrained-weights", str(tmp_path / "weights"), "--output-dir",
                str(tmp_path / "out"), "--opts"] + _opts(tmp_path))
    written = json.loads((tmp_path / "out" / "eval" / "manual_5" / "results_knn.json").read_text())
    assert sorted(written) == ["1", "10", "5"] and set(res) == {1, 5, 10}
    for k, v in written.items():
        assert v["top1"] > 90.0 and v["top5"] == 100.0, (k, v)


def test_extract_features_matches_the_model_bitwise(native, tmp_path):
    from dinov3_jax import ops
    from dinov3_jax.eval import ImageFolder, extract_features
    from dinov3_jax.eval.knn import _pack
    from dinov3_jax.models import DinoVisionTransformer
    from features_helpers import tree
    flat = _tiny_vit_checkpoint(tmp_path / "weights")
    model = DinoVisionTransformer(tree(flat), embed_dim=384, n_blocks=2, num_heads=6)
    _color_folder(tmp_path / "imgs", 5, 2)
    ds = ImageFolder(tmp_path / "imgs")
    feats, labels = extract_features(model, ds, batch_size=4, num_workers=0, resize_size=72, crop_size=64)
    assert feats.shape == (10, 384) and labels.tolist() == [0] * 5 + [1] * 5
    flat_u8, desc, _ = _pack([ds[i] for i in range(len(ds))])
    x = torch.empty(len(ds), 64, 64, 3, dtype=bf16, device="cuda")
    ops.eval_resize_crop(flat_u8.cuda(), desc.cuda(), x, resize=72, max_taps=ops.eval_max_taps(desc[:, 1:].tolist(), 72),
                         mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
    want = torch.empty(len(ds), 384, device="cuda")
    for b0 in (0, 4, 8):                                            # the batches extract_features ran, the last partial
        ops.knn_normalize(model(x[b0:b0 + 4]), y_f32=want[b0:b0 + 4])
    assert torch.equal(feats, want)
    ref = torch.nn.functional.normalize(model(x[:4]), dim=1)
    assert (feats[:4] - ref).abs().max().item() < 1e-6


def test_do_train_calls_do_test_at_the_eval_period(native, tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch, train
    calls = []
    monkeypatch.setattr(train, "do_test", lambda config, model, header: calls.append(header) or {})
    opts = _opts(tmp_path) + ["train.batch_size_per_gpu=2", f"train.output_dir={tmp_path}", "checkpointing.period=100",
                              "evaluation.eval_period_iterations=2", "dino.head_n_prototypes=1024",
                              "ibot.head_n_prototypes=1024"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    train.do_train(config, SSLMetaArch(config), max_iters=2, print_freq=1)
    assert calls == ["training_1"]
