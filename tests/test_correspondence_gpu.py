"""-m gpu: keypoint correspondence (csrc/correspondence.cu, dinov3_jax/eval/correspondence.py).  The descriptors and the
Gram against float64; the argmax against the float64 statement in tests/correspondence_oracle.py, which materialises
the upsampled target (pinned on the CPU to hand-computed cases and to the kernel's closed form); exact ties; a torch
fp32 restatement; an image matched against itself through a tiny ViT; bit-reproducibility; and the evaluation end to end
through --eval-only and do_train."""
import json

import numpy as np
import pytest
import torch

import correspondence_oracle as oracle

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16


def _unit_bf16(rows, D, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.nn.functional.normalize(torch.randn(rows, D, generator=g), dim=1).to(bf16).cuda()


def _smooth_maps(n, h, w, D, seed):
    """bf16 unit rows of n [h, w, D] maps that vary smoothly over the grid (neighbouring patches correlate, as real
    features do), so the upsampled cosine has a structured maximum rather than noise."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(n, D, 4, 4, generator=g)
    up = torch.nn.functional.interpolate(base, size=(h, w), mode="bilinear", align_corners=False)
    x = up.permute(0, 2, 3, 1) + 0.3 * torch.randn(n, h, w, D, generator=g)
    return torch.nn.functional.normalize(x.reshape(-1, D), dim=1).to(bf16).cuda()


def _descriptors(feats, n_maps, hw, out_hw, kp):
    from dinov3_jax import ops
    K, D = len(kp), feats.shape[1]
    q = torch.empty(K, D, dtype=bf16, device="cuda")
    qn = torch.empty(K, device="cuda")
    ops.corr_descriptors(feats, n_maps, hw, out_hw, kp, q, qn)
    return q, qn


def _match(q, qn, target, hw, out_hw):
    """The kernel path for one target map: Gram, GEMM, argmax."""
    from dinov3_jax import ops
    h, w = hw
    P, K = h * w, q.shape[0]
    gram = ops.corr_gram(target, 1, hw, torch.empty(P, 5, device="cuda"))
    sim = ops.gemm(q, target, torch.empty(K, -(-P // 8) * 8, device="cuda")[:, :P])
    xy = torch.empty(K, 2, dtype=torch.int32, device="cuda")
    cos = torch.empty(K, device="cuda")
    ops.corr_argmax(sim, gram, qn, hw, out_hw, xy, cos)
    return xy, cos


# ------------------------------------------------------------------------------------------------ descriptors, Gram
@pytest.mark.parametrize("case", [(2, 2, 32, 32, 64), (7, 7, 112, 112, 1024), (5, 9, 80, 144, 64),
                                  (32, 32, 512, 512, 64)], ids=lambda c: f"{c[0]}x{c[1]}_to_{c[2]}x{c[3]}_D{c[4]}")
def test_descriptors_against_float64(native, case):
    h, w, H, W, D = case
    n_maps = 3
    feats = _smooth_maps(n_maps, h, w, D, seed=h * w)
    rng = np.random.default_rng(D)
    sy, sx = H // h, W // w
    # interior pixels, both pixels of every kind of cell border, the first / last rows and columns and the corners
    special = [(0, 0), (W - 1, H - 1), (W - 1, 0), (0, H - 1), (sx // 2 - 1, sy // 2), (sx // 2, sy // 2 - 1),
               (W - 1, H // 2), (W // 2, H - 1), (W - sx // 2, H - sy // 2), (W - sx // 2 - 1, H - sy // 2 - 1)]
    pts = special + [(int(rng.integers(0, W)), int(rng.integers(0, H))) for _ in range(40)]
    kp = np.array([(i % n_maps, x, y) for i, (x, y) in enumerate(pts)], dtype=np.int32)
    q, qn = _descriptors(feats, n_maps, (h, w), (H, W), kp)
    fh = feats.double().cpu().numpy().reshape(n_maps, h, w, D)
    U = [oracle.upsample(fh[m], (H, W)).numpy() for m in range(n_maps)]
    want = np.stack([U[m][y, x] for m, x, y in kp])
    want /= np.linalg.norm(want, axis=1, keepdims=True)
    got = q.double().cpu().numpy()
    err = np.abs(got - want)
    # bf16 rounding of the fp32 value: half an ulp, 2^-9 relative; the fp32 blend and norm are far below it
    assert (err <= 2.0 ** -8 * np.abs(want) + 1e-6).all(), err.max()
    assert np.allclose(qn.double().cpu().numpy(), np.linalg.norm(got, axis=1), rtol=1e-6)
    again, qn2 = _descriptors(feats, n_maps, (h, w), (H, W), kp)
    assert torch.equal(again, q) and torch.equal(qn2, qn)


def test_gram_against_float64(native):
    from dinov3_jax import ops
    n, h, w, D = 2, 5, 9, 1024
    feats = _unit_bf16(n * h * w, D, seed=3)
    gram = torch.full((n * h * w, 5), float("nan"), device="cuda")
    ops.corr_gram(feats, n, (h, w), gram)
    f = feats.double().cpu().numpy().reshape(n, h, w, D)
    want = np.zeros((n, h, w, 5))
    for m in range(n):
        for i in range(h):
            for j in range(w):
                a = f[m, i, j]
                want[m, i, j] = [a @ a, a @ f[m, i, j + 1] if j + 1 < w else 0, a @ f[m, i + 1, j] if i + 1 < h else 0,
                                 a @ f[m, i + 1, j + 1] if i + 1 < h and j + 1 < w else 0,
                                 a @ f[m, i + 1, j - 1] if i + 1 < h and j > 0 else 0]
    assert np.allclose(gram.double().cpu().numpy().reshape(n, h, w, 5), want, rtol=0, atol=2e-6)


def test_arguments_are_checked_before_any_launch(native):
    from dinov3_jax import _native, ops
    feats = _unit_bf16(2 * 4, 64, seed=1)
    q = torch.empty(1, 64, dtype=bf16, device="cuda")
    qn = torch.empty(1, device="cuda")
    for kp in ([(0, 32, 0)], [(0, 0, -1)], [(2, 0, 0)]):
        with pytest.raises(_native.NativeError, match="keypoint"):
            ops.corr_descriptors(feats, 2, (2, 2), (32, 32), kp, q, qn)
    with pytest.raises(_native.NativeError, match="multiple of 8"):
        ops.corr_gram(feats[:, :60], 2, (2, 2), torch.empty(8, 5, device="cuda"))
    with pytest.raises(_native.NativeError, match="aligned"):
        ops.corr_gram(feats.view(-1)[4:4 + 7 * 64].view(7, 64), 1, (2, 2), torch.empty(4, 5, device="cuda"))


# ------------------------------------------------------------------------------------------------ argmax
ARGMAX_CASES = [(2, 2, 32, 32, 64, 1), (2, 2, 32, 32, 1024, 257), (7, 7, 112, 112, 1024, 37),
                (5, 9, 80, 144, 64, 300), (32, 32, 512, 512, 64, 300)]


@pytest.mark.parametrize("case", ARGMAX_CASES, ids=lambda c: f"{c[0]}x{c[1]}_to_{c[2]}x{c[3]}_D{c[4]}_K{c[5]}")
def test_argmax_against_float64(native, case):
    h, w, H, W, D, K = case
    maps = _smooth_maps(2, h, w, D, seed=K + D)               # map 0 the source, map 1 the target
    rng = np.random.default_rng(K)
    kp = np.stack([np.zeros(K), rng.integers(0, W, K), rng.integers(0, H, K)], 1).astype(np.int32)
    q, qn = _descriptors(maps, 2, (h, w), (H, W), kp)
    target = maps[h * w:]
    xy, cos = _match(q, qn, target, (h, w), (H, W))
    got_xy, got_cos = xy.cpu().numpy(), cos.double().cpu().numpy()
    want_xy, C = oracle.match(q.double().cpu().numpy(), target.double().cpu().numpy().reshape(h, w, D), (H, W))
    best = C.max(1)
    at_pick = C[np.arange(K), got_xy[:, 1] * W + got_xy[:, 0]]
    same = (got_xy == want_xy).all(1)
    print(f"argmax {case}: {int((~same).sum())} of {K} picks differ, worst cosine gap {np.abs(got_cos - best).max():.2e}")
    assert np.abs(got_cos - best).max() <= 1e-5                 # the kernel's cosine at its pick is the maximum
    assert (best - at_pick <= 1e-5).all()                       # every differing pick is a near-tie
    assert same.mean() >= 0.99
    xy2, cos2 = _match(q, qn, target, (h, w), (H, W))
    assert torch.equal(xy2, xy) and torch.equal(cos2, cos)


def test_exact_ties_go_to_the_lowest_index(native):
    from dinov3_jax import ops
    h, w, H, W, D = 6, 9, 96, 144, 64
    # a constant map: dyadic values make every product and sum exact, so every pixel's cosine is the same bits
    f = torch.zeros(D)
    f[:4] = 0.5
    q = torch.zeros(2, D, dtype=bf16, device="cuda")
    q[0, 0] = 1
    q[1, :4] = 0.5
    qn = torch.tensor([1.0, 1.0], device="cuda")
    xy, cos = _match(q, qn, f.to(bf16).cuda().repeat(h * w, 1), (h, w), (H, W))
    assert xy.tolist() == [[0, 0], [0, 0]] and cos.tolist() == [0.5, 1.0]
    # a periodic map (period 2 x 3 cells): each pixel's cosine is a function of its place in the period, so the
    # maximum repeats; its features (four entries of +-1/2) keep every product and sum of the kernel exact, so equal
    # cosines are equal bits wherever they sit, the clamped last rows and columns included
    g = torch.Generator().manual_seed(4)
    cell = torch.zeros(2 * 3, D)
    for c in range(6):
        cell[c, torch.randperm(D, generator=g)[:4]] = torch.randint(0, 2, (4,), generator=g).float() - 0.5
    per = cell.reshape(2, 3, D).repeat(h // 2, w // 3, 1).reshape(h * w, D).to(bf16).cuda()
    qs = (torch.randint(-2, 3, (32, D), generator=g).float() / 4).to(bf16).cuda()
    qn = torch.linalg.vector_norm(qs.float(), dim=1).contiguous()
    xy, cos = _match(qs, qn, per, (h, w), (H, W))
    want, C = oracle.match(qs.double().cpu().numpy(), per.double().cpu().numpy().reshape(h, w, D), (H, W))
    top = C.max(1, keepdims=True)
    tied = C >= top - oracle.TIE
    n_max = tied.sum(1)
    gap = top[:, 0] - np.where(tied, -np.inf, C).max(1)
    assert (n_max >= 2).all(), n_max                            # every maximum is an exact tie
    clear = gap > 1e-6                                          # and, for most, clear of the runner-up
    assert clear.mean() >= 0.5, gap
    assert np.array_equal(xy.cpu().numpy()[clear], want[clear])     # the lowest index wins, as in float64
    assert np.abs(cos.double().cpu().numpy() - top[:, 0]).max() <= 1e-6


def test_torch_fp32_restatement_agrees(native):
    import torch.nn.functional as Fn
    h, w, S, D, K = 8, 8, 128, 384, 500
    maps = _smooth_maps(2, h, w, D, seed=11)
    g = torch.Generator().manual_seed(2)
    kp = torch.stack([torch.zeros(K, dtype=torch.int64), torch.randint(0, S, (K,), generator=g),
                      torch.randint(0, S, (K,), generator=g)], 1).numpy()
    q, qn = _descriptors(maps, 2, (h, w), (S, S), kp)
    target = maps[h * w:]
    xy, _ = _match(q, qn, target, (h, w), (S, S))
    U = Fn.interpolate(target.float().reshape(1, h, w, D).permute(0, 3, 1, 2), size=(S, S), mode="bilinear",
                       align_corners=False)[0].reshape(D, -1)
    cos = (q.float() @ U) / (torch.linalg.vector_norm(q.float(), dim=1)[:, None] * torch.linalg.vector_norm(U, dim=0))
    idx = cos.argmax(1)
    want = torch.stack([idx % S, idx // S], 1).to(torch.int32)
    agree = (xy == want).all(1).float().mean().item()
    print(f"torch fp32 restatement: {agree:.4f} of {K} picks identical")
    assert agree >= 0.99


# ------------------------------------------------------------------------------------------------ end to end
def _tiny_vit_checkpoint(path, depth=4):
    from dinov3_jax.checkpointer import save_checkpoint, tree_from_flat
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=384, depth=depth, heads=6, layerscale=0.5)
    flat = init_backbone(cfg, torch.Generator().manual_seed(0))
    save_checkpoint(path, iteration=4, params={"teacher_backbone": tree_from_flat(flat)})


def _images(rng, sizes):
    """Random smooth colour fields with noise, one per (H, W)."""
    out = []
    for H, W in sizes:
        base = rng.random((4, 5, 3)) * 255
        yy, xx = np.arange(H) * 4 // H, np.arange(W) * 5 // W
        im = base[yy][:, xx] + rng.normal(0, 30, (H, W, 3))
        out.append(np.clip(im, 0, 255).astype(np.uint8))
    return out


def _pairs_npz(path, seed=0):
    """Five images of one size (an .npz holds one), three categories, pairs that share images and unequal keypoint
    counts."""
    rng = np.random.default_rng(seed)
    H, W = 96, 128
    images = np.stack(_images(rng, [(H, W)] * 5))
    pairs = np.array([[0, 1], [2, 1], [1, 0], [3, 4], [4, 4], [0, 3]])
    n = np.array([5, 3, 7, 1, 4, 6])
    kmax = int(n.max())
    kps = lambda: np.stack([rng.random((kmax, 2)) * [W - 1, H - 1] for _ in pairs])
    np.savez(path, images=images, pairs=pairs, src_kps=kps(), trg_kps=kps(), n_kps=n,
             trg_bbox=np.tile([[4.0, 6.0, 100.0, 80.0]], (len(pairs), 1)),
             categories=np.array(["cat", "cat", "cat", "dog", "dog", "bird"]))


def test_an_image_matched_to_itself_scores_one(native, tmp_path):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.eval import CorrespondenceNpzDataset, eval_correspondence
    from dinov3_jax.train.train import eval_backbone
    _tiny_vit_checkpoint(tmp_path / "weights")
    rng = np.random.default_rng(5)
    H, W, M = 128, 128, 3
    images = np.stack(_images(rng, [(H, W)] * M))
    kps = rng.random((M, 12, 2)) * (W - 1)
    np.savez(tmp_path / "self.npz", images=images, pairs=np.stack([np.arange(M)] * 2, 1), src_kps=kps, trg_kps=kps,
             n_kps=np.full(M, 12), trg_bbox=np.tile([[0.0, 0.0, W, H]], (M, 1)), categories=np.array(["a"] * M))
    model = eval_backbone(setup_config(DinoV3SetupArgs(opts=["student.arch=vit_small"])), str(tmp_path / "weights"))
    res = eval_correspondence(model, CorrespondenceNpzDataset(tmp_path / "self.npz"), image_size=128, num_workers=0)
    print("self-match:", {k: v for k, v in res.items() if k.startswith("PCK")})
    assert res["PCK@0.1"] == 1.0 and res["PCK-image@0.1"] == 1.0
    assert res["n_pairs"] == M and res["n_keypoints"] == 12 * M


def _opts(tmp_path):
    return ["student.arch=vit_small", f"evaluation.correspondence.dataset_path={tmp_path / 'c.npz'}",
            "evaluation.correspondence.image_size=128", "evaluation.correspondence.batch_size=2",
            "evaluation.correspondence.num_workers=0"]


def test_eval_only_correspondence_writes_the_same_results_twice(native, tmp_path):
    from dinov3_jax.train.train import main
    _tiny_vit_checkpoint(tmp_path / "weights")
    _pairs_npz(tmp_path / "c.npz")
    outs = []
    for run in ("a", "b"):
        res = main(["--eval-only", "--eval", "correspondence", "--eval-pretrained-weights", str(tmp_path / "weights"),
                    "--output-dir", str(tmp_path / run), "--opts"] + _opts(tmp_path))
        outs.append((tmp_path / run / "eval" / "manual_5" / "results_correspondence.json").read_text())
        written = json.loads(outs[-1])
        assert written == res
        scores = [f"PCK{kind}@{a}" for a in ("0.01", "0.05", "0.1") for kind in ("", "-image")]
        assert sorted(written) == sorted(scores + ["categories", "n_pairs", "n_keypoints", "protocol", "config"])
        assert all(0.0 <= written[k] <= 1.0 for k in scores)
        assert written["n_pairs"] == 6 and written["n_keypoints"] == 26
        assert sorted(written["categories"]) == ["bird", "cat", "dog"]
        assert written["categories"]["cat"]["n_pairs"] == 3 and written["categories"]["cat"]["n_keypoints"] == 15
        assert sorted(written["categories"]["dog"]) == sorted(scores + ["n_pairs", "n_keypoints"])
        assert written["protocol"] == {"image_size": 128, "alphas": [0.01, 0.05, 0.1]}
        assert written["config"]["dataset_path"] == str(tmp_path / "c.npz")
    assert outs[0] == outs[1]
    print("correspondence end to end:", {k: v for k, v in json.loads(outs[0]).items() if k.startswith("PCK")})


def test_do_train_calls_do_correspondence_eval_at_the_eval_period(native, tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch, train
    calls = []
    monkeypatch.setattr(train, "do_correspondence_eval", lambda config, model, header: calls.append(header) or {})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval", "do_video_eval"):
        monkeypatch.setattr(train, name, lambda *a, _n=name: pytest.fail(f"{_n}: no dataset is configured"))
    opts = _opts(tmp_path) + ["train.batch_size_per_gpu=2", f"train.output_dir={tmp_path}", "checkpointing.period=100",
                              "evaluation.eval_period_iterations=2", "dino.head_n_prototypes=1024",
                              "ibot.head_n_prototypes=1024"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    train.do_train(config, SSLMetaArch(config), max_iters=4, print_freq=1)
    assert calls == ["training_1", "training_3"]
