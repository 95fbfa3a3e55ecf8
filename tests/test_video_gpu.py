"""-m gpu: video object segmentation by label propagation (csrc/video.cu, dinov3_jax/eval/video.py).  The frame resize
against torch's bilinear; the propagation, the label map and the J / F counts against the float64 statement in
tests/video_oracle.py (pinned on the CPU to DINO's label_propagation and to hand-computed J / F); a sequence of
identical frames; bit-reproducibility; and the evaluation end to end through --eval-only, save_masks and do_train."""
import json

import numpy as np
import pytest
import torch

import video_oracle

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


# ------------------------------------------------------------------------------------------------ resize
@pytest.mark.parametrize("sizes", [[(480, 854), (480, 832)], [(37, 53), (64, 128)], [(854, 480), (832, 480)],
                                   [(100, 60), (48, 40)]], ids=str)
def test_video_resize_against_torch_bilinear(native, sizes):
    import torch.nn.functional as Fn
    from dinov3_jax import ops
    (H, W), (rh, rw) = sizes
    rng = np.random.default_rng(H + W)
    frames = torch.from_numpy(rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)).cuda()
    desc = torch.tensor([[i * H * W * 3, H, W] for i in range(3)], dtype=torch.int64, device="cuda")
    out = ops.video_resize(frames.reshape(-1), desc, torch.empty(3, rh, rw, 3, dtype=bf16, device="cuda"),
                           mean=MEAN, std=STD)
    x = frames.permute(0, 3, 1, 2).float() / 255.0
    want = Fn.interpolate(x, size=(rh, rw), mode="bilinear", align_corners=False, antialias=False)
    want = ((want - torch.tensor(MEAN, device="cuda")[:, None, None]) / torch.tensor(STD, device="cuda")[:, None, None])
    want = want.permute(0, 2, 3, 1)
    err = (out.float() - want).abs()
    # bf16 rounding of the fp32 value: half an ulp, 2^-9 relative; fp32 differences of the arithmetic are far below
    assert (err <= 2.0 ** -8 * want.abs() + 1e-6).all(), err.max().item()
    assert (out == want.to(bf16)).float().mean().item() > 0.99


# ------------------------------------------------------------------------------------------------ propagation
def _unit_bf16(n, P, D, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n * P, D, generator=g)
    return torch.nn.functional.normalize(x, dim=1).to(bf16).cuda()


PROP_CASES = [(7, 9, 1, 1, 1, 2), (13, 11, 4, 12, 5, 9), (5, 7, 8, 20, 32, 32), (30, 52, 8, 12, 5, 9),
              (9, 5, 3, 12, 32, 2), (11, 13, 6, 1, 5, 32), (2, 3, 2, 0, 5, 2), (30, 52, 1, 12, 5, 2)]


@pytest.mark.parametrize("case", PROP_CASES, ids=lambda c: f"{c[0]}x{c[1]}_ctx{c[2]}_r{c[3]}_k{c[4]}_C{c[5]}")
def test_propagate_against_float64(native, case):
    from dinov3_jax import ops
    h, w, n_ctx, r, k, C = case
    P, D = h * w, 64
    feats = _unit_bf16(n_ctx + 1, P, D, seed=P + k + C)          # frame 0, the n_ctx - 1 recent frames, the target
    g = torch.Generator().manual_seed(C)
    lab0 = torch.eye(C)[torch.randint(0, C, (P,), generator=g)]
    labr = torch.rand((n_ctx - 1) * P, C, generator=g)
    tgt = feats[n_ctx * P:]
    ld = -(-P // 8) * 8
    sim0 = ops.gemm(tgt, feats[:P], torch.empty(P, ld, device="cuda")[:, :P])
    simr = None
    if n_ctx > 1:
        buf = torch.empty(P, -(-(n_ctx - 1) * P // 8) * 8, device="cuda")
        simr = ops.gemm(tgt, feats[P:n_ctx * P], buf[:, :(n_ctx - 1) * P])
    out = torch.full((P, C), float("nan"), device="cuda")
    ops.video_propagate(sim0, simr, lab0.cuda(), labr.cuda() if n_ctx > 1 else None, (h, w), r, k, 0.1, out)
    fh = feats.double().cpu().numpy()
    ctx = [fh[:P]] + [fh[c * P:(c + 1) * P] for c in range(1, n_ctx)]
    labs = [lab0.numpy()] + [labr[(c - 1) * P:c * P].numpy() for c in range(1, n_ctx)]
    want, kth, nxt = video_oracle.propagate(fh[n_ctx * P:], ctx, labs, h, w, r, k, 0.1)
    got = out.double().cpu().numpy()
    with np.errstate(invalid="ignore"):
        near = np.isfinite(nxt) & (kth - nxt < 1e-4)
    far = ~near
    err = np.abs(got - want) / (np.abs(want) + 1e-6)
    print(f"propagate {case}: worst rel error {err[far].max() if far.any() else 0:.2e} on {far.sum()} rows, "
          f"{near.sum()} near ties")
    assert np.allclose(got[far], want[far], rtol=1e-5, atol=1e-7)
    if near.any():
        # the tie rule on the kernel's own fp32 similarities: every candidate at the threshold is kept
        sims = [sim0.double().cpu().numpy()] + [simr[:, (c - 1) * P:c * P].double().cpu().numpy()
                                                for c in range(1, n_ctx)]
        tie, _, _ = video_oracle.propagate_sims(sims, labs, h, w, r, k, 0.1)
        assert np.allclose(got[near], tie[near], rtol=1e-5, atol=1e-7)
    again = torch.empty_like(out)
    ops.video_propagate(sim0, simr, lab0.cuda(), labr.cuda() if n_ctx > 1 else None, (h, w), r, k, 0.1, again)
    assert torch.equal(again, out)


def test_propagate_keeps_exact_ties(native):
    # three context frames with the same features: every similarity appears three times, so ties sit at every k
    from dinov3_jax import ops
    h, w, C, k = 6, 7, 4, 5
    P = h * w
    f = _unit_bf16(2, P, 32, seed=5)
    g = torch.Generator().manual_seed(1)
    lab0 = torch.eye(C)[torch.randint(0, C, (P,), generator=g)]
    labr = torch.rand(2 * P, C, generator=g)
    ctx = torch.cat([f[:P], f[:P], f[:P]])
    tgt = f[P:]
    sim0 = ops.gemm(tgt, ctx[:P], torch.empty(P, 48, device="cuda")[:, :P])
    simr = ops.gemm(tgt, ctx[P:], torch.empty(P, 88, device="cuda")[:, :2 * P])
    assert torch.equal(simr[:, :P], sim0) and torch.equal(simr[:, P:], sim0)
    out = torch.empty(P, C, device="cuda")
    ops.video_propagate(sim0, simr, lab0.cuda(), labr.cuda(), (h, w), 2, k, 0.1, out)
    s = sim0.double().cpu().numpy()
    labs = [lab0.numpy(), labr[:P].numpy(), labr[P:].numpy()]
    want, kth, nxt = video_oracle.propagate_sims([s, s, s], labs, h, w, 2, k, 0.1)
    assert np.allclose(out.double().cpu().numpy(), want, rtol=1e-5, atol=1e-7)
    # k = 5 of triples: the 5th largest is the second copy of the 2nd-largest score, whose third copy is kept too
    assert (kth == nxt).all()


# ------------------------------------------------------------------------------------------------ label map
LABEL_CASES = [(30, 52, 16, 480, 854, 9), (7, 9, 8, 61, 77, 3), (30, 52, 16, 480, 832, 32), (5, 4, 14, 70, 56, 2),
               (11, 6, 16, 200, 101, 5)]


@pytest.mark.parametrize("case", LABEL_CASES, ids=lambda c: f"{c[0]}x{c[1]}_p{c[2]}_to_{c[3]}x{c[4]}_C{c[5]}")
def test_label_map_against_float64(native, case):
    from dinov3_jax import ops
    h, w, p, H, W, C = case
    g = torch.Generator().manual_seed(h * w + C)
    soft = torch.rand(h * w, C, generator=g) ** 3
    soft[:, 1] = 0.0                                     # a channel never predicted: max <= 0, left as it is
    if C > 3:
        soft[:, 2] = -torch.rand(h * w, generator=g)     # a negative channel: also left as it is
    out = torch.full((H, W), 99, dtype=torch.uint8, device="cuda")
    ops.video_label_map(soft.cuda(), (h, w), p, out)
    want, margin = video_oracle.label_map(soft.double().numpy().reshape(h, w, C), p, H, W)
    got = out.cpu().numpy()
    ok = (got == want) | (margin < 1e-6)
    print(f"label map {case}: {int((got != want).sum())} pixels differ, {int((margin < 1e-6).sum())} near ties")
    assert ok.all(), np.argwhere(~ok)[:5]
    again = torch.empty_like(out)
    ops.video_label_map(soft.cuda(), (h, w), p, again)
    assert torch.equal(again, out)


# ------------------------------------------------------------------------------------------------ J and F counts
def _blobs(H, W, K, seed, void=0.0):
    """Label maps made of nearest-upsampled random cells (so boundaries are long and shared), with random void."""
    rng = np.random.default_rng(seed)
    cells = rng.integers(0, K + 1, (max(H // 23, 2), max(W // 31, 2)))
    m = np.ascontiguousarray(cells[np.arange(H) * cells.shape[0] // H][:, np.arange(W) * cells.shape[1] // W],
                             dtype=np.uint8)
    flip = rng.random((H, W)) < 0.01
    m[flip] = rng.integers(0, K + 1, int(flip.sum()))
    m[rng.random((H, W)) < void] = 255
    return m


@pytest.mark.parametrize("case", [(480, 854, 3, None), (37, 53, 2, None), (100, 7, 4, None), (61, 45, 3, 5),
                                  (1, 40, 2, None)], ids=str)
def test_jf_counts_equal_float64_integers(native, case):
    from dinov3_jax import ops
    H, W, K, r = case
    r = video_oracle.radius(H, W) if r is None else r
    F = 3
    gt = np.stack([_blobs(H, W, K, 10 * i, void=0.02) for i in range(F)])
    assert gt.flags.c_contiguous
    pred = np.stack([_blobs(H, W, K, 10 * i + 1) for i in range(F - 1)] + [np.where(gt[-1] == 255, 0, gt[-1])])
    counts = torch.full((F, K, 6), -1, dtype=torch.int64, device="cuda")
    ops.video_jf_counts(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(), K, r, counts)
    want = np.stack([video_oracle.jf_counts(pred[i], gt[i], K, r) for i in range(F)])
    assert np.array_equal(counts.cpu().numpy(), want), (counts.cpu().numpy() - want)
    assert (want[..., 2:] > 0).any()


# ------------------------------------------------------------------------------------------------ sequences
def _stripes(h, w, p, widths):
    """uint8 [h p, w p] vertical bands of labels 0, 1, 2, ... cycling, `widths` patches wide, and their patch map."""
    cols = np.concatenate([np.full(wd, i % 3, np.uint8) for i, wd in enumerate(widths)])[:w]
    small = np.tile(cols, (h, 1))
    return np.repeat(np.repeat(small, p, 0), p, 1), small


def test_identical_frames_reproduce_frame_0(native):
    from dinov3_jax import ops
    from dinov3_jax.eval.video import propagate_sequence
    h, w, p, N = 6, 10, 16, 9
    mask, small = _stripes(h, w, p, [3, 2, 3, 2])
    f = _unit_bf16(1, h * w, 64, seed=2)
    feats = f.repeat(N, 1)
    labels, pred = propagate_sequence(feats, mask, (h, w), N, mask.shape, patch=p, n_last_frames=7,
                                      size_mask_neighborhood=12, topk=5, temperature=0.1)
    for t in range(1, N):
        assert np.array_equal(labels[t].argmax(1).view(h, w).cpu().numpy(), small), t
    gt = torch.from_numpy(np.stack([mask] * N)).cuda()
    counts = torch.empty(N - 2, 2, 6, dtype=torch.int64, device="cuda")
    ops.video_jf_counts(pred[1:N - 1], gt[1:N - 1], 2, video_oracle.radius(*mask.shape), counts)
    from dinov3_jax.eval.video import jf_from_counts
    J, F = jf_from_counts(counts.cpu().numpy())
    assert (J == 1.0).all() and (F == 1.0).all()


def test_a_whole_sequence_gives_the_same_bits_twice(native):
    from dinov3_jax.eval.video import propagate_sequence
    h, w, p, N = 12, 20, 16, 14
    mask = _blobs(200, 333, 3, seed=4, void=0.02)             # the annotation size, not the resized frame's
    feats = _unit_bf16(N, h * w, 128, seed=7)
    runs = [propagate_sequence(feats, mask, (h, w), N, (200, 333), patch=p, n_last_frames=7,
                               size_mask_neighborhood=12, topk=5, temperature=0.1) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


# ------------------------------------------------------------------------------------------------ end to end
def _tiny_vit_checkpoint(path, depth=4):
    from dinov3_jax.checkpointer import save_checkpoint, tree_from_flat
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=384, depth=depth, heads=6, layerscale=0.5)
    flat = init_backbone(cfg, torch.Generator().manual_seed(0))
    save_checkpoint(path, iteration=4, params={"teacher_backbone": tree_from_flat(flat)})


def _moving_squares_npz(path, lengths, H=120, W=200, seed=0):
    """Sequences of noisy backgrounds with two coloured squares moving a few pixels per frame; masks 1 and 2 are the
    squares, a thin void band around the first."""
    rng = np.random.default_rng(seed)
    frames, masks = [], []
    for n in lengths:
        bg = rng.integers(0, 256, 3)
        cols = rng.integers(0, 256, (2, 3))
        pos = rng.integers(4, 80, (2, 2))
        vel = rng.integers(-2, 3, (2, 2))
        for t in range(n):
            im = np.clip(bg + rng.normal(0, 20, (H, W, 3)), 0, 255)
            m = np.zeros((H, W), np.uint8)
            for o in range(2):
                y, x = np.clip(pos[o] + vel[o] * t, 0, [H - 24, W - 24])
                im[y:y + 24, x:x + 24] = cols[o]
                if o == 0:
                    m[max(y - 1, 0):y + 25, max(x - 1, 0):x + 25] = 255
                m[y:y + 24, x:x + 24] = o + 1
            frames.append(im.astype(np.uint8))
            masks.append(m)
    np.savez(path, frames=np.stack(frames), masks=np.stack(masks),
             sequence_starts=np.concatenate([[0], np.cumsum(lengths)[:-1]]))


def _opts(tmp_path, save=False):
    return ["student.arch=vit_small", f"evaluation.video.dataset_path={tmp_path / 'v.npz'}",
            "evaluation.video.short_side=128", "evaluation.video.batch_size=4", "evaluation.video.num_workers=0",
            f"evaluation.video.save_masks={save}"]


STATS = ["J&F-Mean", "J-Mean", "J-Recall", "J-Decay", "F-Mean", "F-Recall", "F-Decay"]


def test_eval_only_video_writes_results_video_json(native, tmp_path):
    from dinov3_jax.train.train import main
    _tiny_vit_checkpoint(tmp_path / "weights")
    _moving_squares_npz(tmp_path / "v.npz", [6, 5])
    outs = []
    for run in ("a", "b"):
        res = main(["--eval-only", "--eval", "video", "--eval-pretrained-weights", str(tmp_path / "weights"),
                    "--output-dir", str(tmp_path / run), "--opts"] + _opts(tmp_path))
        outs.append((tmp_path / run / "eval" / "manual_5" / "results_video.json").read_text())
        written = json.loads(outs[-1])
        assert written == res
        assert sorted(written) == sorted(STATS + ["sequences", "protocol", "config"])
        assert all(0.0 <= written[k] <= 1.0 for k in STATS if "Decay" not in k)
        assert sorted(written["sequences"]) == ["00000", "00001"]
        assert sorted(written["sequences"]["00000"]["objects"]) == ["1", "2"]
        assert written["protocol"] == {"n_last_frames": 7, "size_mask_neighborhood": 12, "topk": 5,
                                       "temperature": 0.1, "short_side": 128}
        assert written["config"]["dataset_path"] == str(tmp_path / "v.npz")
        assert written["J&F-Mean"] == pytest.approx((written["J-Mean"] + written["F-Mean"]) / 2)
    assert outs[0] == outs[1]
    print("video end to end:", {k: round(json.loads(outs[0])[k], 4) for k in STATS})


def test_save_masks_writes_palette_pngs_of_the_returned_labels(native, tmp_path):
    from PIL import Image
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.eval import make_video_dataset
    from dinov3_jax.eval.video import default_palette, eval_video_segmentation
    from dinov3_jax.train.train import eval_backbone
    _tiny_vit_checkpoint(tmp_path / "weights")
    _moving_squares_npz(tmp_path / "v.npz", [4, 3], seed=1)
    model = eval_backbone(setup_config(DinoV3SetupArgs(opts=["student.arch=vit_small"])), str(tmp_path / "weights"))
    res = eval_video_segmentation(model, make_video_dataset(tmp_path / "v.npz"), short_side=128, num_workers=0,
                                  save_masks=True, output_dir=tmp_path / "out", return_masks=True)
    ds = make_video_dataset(tmp_path / "v.npz")
    for i, name in enumerate(["00000", "00001"]):
        labels = res["masks"][name]
        assert labels.shape == ds[i]["masks"].shape and labels.max() <= 2
        assert np.array_equal(labels[0], np.where(ds[i]["masks"][0] == 255, 0, ds[i]["masks"][0]))
        for t in range(len(labels)):
            with Image.open(tmp_path / "out" / "Annotations" / "480p" / name / f"{t:05d}.png") as im:
                assert im.mode == "P" and im.getpalette()[:768] == default_palette()
                assert np.array_equal(np.asarray(im), labels[t])


def test_do_train_calls_do_video_eval_at_the_eval_period(native, tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch, train
    calls = []
    monkeypatch.setattr(train, "do_video_eval", lambda config, model, header: calls.append(header) or {})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval"):
        monkeypatch.setattr(train, name, lambda *a, _n=name: pytest.fail(f"{_n}: no dataset is configured"))
    opts = _opts(tmp_path) + ["train.batch_size_per_gpu=2", f"train.output_dir={tmp_path}", "checkpointing.period=100",
                              "evaluation.eval_period_iterations=2", "dino.head_n_prototypes=1024",
                              "ibot.head_n_prototypes=1024"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    train.do_train(config, SSLMetaArch(config), max_iters=4, print_freq=1)
    assert calls == ["training_1", "training_3"]
