"""-m gpu: unsupervised object discovery (csrc/discovery.cu, dinov3_jax/eval/discovery.py).  The graph against the float64
threshold; the eigenpair against scipy.linalg.eigh on the same graph, on odd and non-square grids; the bipartition and
box against tests/discovery_oracle.py on synthetic objects; the argument checks; bit-reproducibility; and the
evaluation end to end through --eval-only and do_train."""
import json

import numpy as np
import pytest
import torch

import discovery_oracle as oracle

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16
TAU, EPS = 0.2, 1e-5


def _clustered(n, h, w, D, seed):
    """bf16 unit features [n, h w, D] of clustered scenes: a background class, an object rectangle and a smaller second
    blob, each a random centre plus noise, so the normalized cut has a clear object."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        centres = torch.randn(3, D, generator=g)
        lab = torch.zeros(h, w, dtype=torch.long)
        y0, x0 = int(torch.randint(0, max(1, h // 2), (1,), generator=g)), int(torch.randint(0, max(1, w // 2), (1,), generator=g))
        lab[y0:y0 + max(1, h // 3), x0:x0 + max(1, w // 3)] = 1
        lab[h - max(1, h // 6):, w - max(1, w // 6):] = 2
        f = centres[lab.reshape(-1)] + 0.8 * torch.randn(h * w, D, generator=g)
        out.append(torch.nn.functional.normalize(f, dim=1))
    return torch.stack(out).to(bf16).cuda()


def _cut(feats, k_max=256):
    from dinov3_jax.eval.discovery import normalized_cut
    return normalized_cut(feats, TAU, EPS, k_max)


def _dense(bits, P):
    """bool [n, P, P] from the bit matrix."""
    b = bits.cpu().numpy().view(np.uint32)
    n, _, words = b.shape
    out = (b[..., None] >> np.arange(32, dtype=np.uint32)) & 1
    return out.reshape(n, P, words * 32)[:, :, :P].astype(bool)


# ------------------------------------------------------------------------------------------------ graph
@pytest.mark.parametrize("grid", [(1, 45), (7, 13), (32, 24)], ids=lambda g: f"{g[0]}x{g[1]}")
def test_graph_against_float64(native, grid):
    h, w = grid
    P, n = h * w, 3
    feats = _clustered(n, h, w, 256, seed=P)
    cut = _cut(feats)
    got = _dense(cut["bits"], P)
    f = feats.double().cpu().numpy()
    S = f @ f.transpose(0, 2, 1)
    want = S > TAU
    near = np.abs(S - TAU) < 1e-5
    print(f"graph {grid}: {int(near.sum())} of {S.size} pairs within 1e-5 of tau")
    assert near.mean() < 1e-3
    assert np.array_equal(got[~near], want[~near])
    c = got.sum(2)
    deg = cut["degree"].double().cpu().numpy()
    assert np.allclose(deg, c + (P - c) * EPS, rtol=1e-6, atol=0)
    A = np.where(want, 1.0, EPS)
    rows = ~near.any(2)
    assert np.allclose(deg[rows], A.sum(2)[rows], rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------ eigenpair
@pytest.mark.parametrize("grid", [(1, 40), (40, 1), (7, 13), (32, 24), (32, 32), (64, 64)],
                         ids=lambda g: f"{g[0]}x{g[1]}")
def test_eigenpair_against_scipy(native, grid):
    h, w = grid
    P = h * w
    n = 1 if P > 2000 else 3
    feats = _clustered(n, h, w, 128, seed=P + 1)
    cut = _cut(feats)
    A_bits = _dense(cut["bits"], P)
    x = cut["x"].double().cpu().numpy()
    lam = cut["lambda2"].double().cpu().numpy()
    iters = cut["iters"].cpu().numpy()
    assert cut["converged"].cpu().numpy().all(), iters
    checked = 0
    for m in range(n):
        A = np.where(A_bits[m], 1.0, EPS)
        d = A.sum(1)
        xr, l2, l3 = oracle.fiedler(A, d)
        cos = abs(x[m] @ (d * xr)) / np.sqrt((x[m] @ (d * x[m])) * (xr @ (d * xr)))
        print(f"eigenpair {grid}[{m}]: {iters[m]} steps, lambda2 {lam[m]:.6f} (scipy {l2:.6f}), gap {l3 - l2:.2e}, "
              f"1 - |cos_D| {1 - cos:.1e}")
        assert abs(x[m] @ (d * x[m]) - 1.0) < 1e-3                     # x^T D x = 1
        if l3 - l2 >= 1e-3:
            checked += 1
            assert abs(lam[m] - l2) <= 1e-5
            assert cos >= 1 - 1e-4
    assert checked >= 1


def test_unconverged_image_still_gets_a_box(native):
    from dinov3_jax.eval.discovery import boxes_of
    h, w = 32, 24
    feats = _clustered(2, h, w, 128, seed=5)
    cut = _cut(feats, k_max=2)
    assert cut["iters"].tolist() == [2, 2] and cut["converged"].tolist() == [0, 0]
    out = boxes_of(cut["x"], (h, w), 16, [(h * 16, w * 16)] * 2, [np.array([[0.0, 0.0, 10.0, 10.0]])] * 2)
    box = out["box"].cpu().numpy()
    assert ((box[:, 2] > box[:, 0]) & (box[:, 3] > box[:, 1])).all()


# ------------------------------------------------------------------------------------------------ bipartition, box
def _shapes():
    """(name, grid, size (H, W), x [h w] with the object positive)."""
    rng = np.random.default_rng(0)
    out = []
    h, w = 9, 11
    rect = np.full((h, w), -0.3)
    rect[2:5, 3:9] = 1.0
    out.append(("rectangle", (h, w), (144, 176), rect))
    L = np.full((h, w), -0.3)
    L[1:8, 2:4] = 0.9
    L[6:8, 2:9] = 0.9
    out.append(("L", (h, w), (144, 176), L))
    blobs = np.full((h, w), -0.2)
    blobs[1:3, 1:3] = 1.0                                            # the seed's blob (largest |x|)
    blobs[5:8, 6:10] = 0.8                                           # a second foreground blob, not connected
    out.append(("two blobs", (h, w), (144, 176), blobs))
    border = np.full((7, 13), -0.25)
    border[4:, 9:] = 1.0                                             # touches the padded bottom-right patches
    out.append(("border", (7, 13), (100, 200), border))
    line = np.full((1, 30), -0.1)
    line[0, 12:20] = 0.7
    out.append(("1 x w", (1, 30), (10, 470), line))
    col = np.full((25, 1), -0.1)
    col[3:9, 0] = 0.6
    out.append(("h x 1", (25, 1), (390, 5), col))
    for name, grid, size, x in list(out):
        out.append((name + " negated", grid, size, -x))              # the sign flip
    return [(name, grid, size, x + 1e-3 * rng.standard_normal(x.shape)) for name, grid, size, x in out]


@pytest.mark.parametrize("case", _shapes(), ids=lambda c: c[0])
def test_box_on_synthetic_objects(native, case):
    from dinov3_jax.eval.discovery import boxes_of
    name, grid, size, x = case
    xt = torch.tensor(x.reshape(1, -1), dtype=f32, device="cuda")
    gts = [np.array([[0.0, 0.0, 32.0, 48.0], [40.0, 30.0, 120.0, 90.0]])]
    out = boxes_of(xt, grid, 16, [size], gts)
    x64 = xt.double().cpu().numpy()[0]
    fg, seed = oracle.bipartition(x64)
    want = oracle.component_box(fg, seed, grid, 16, size)
    assert np.array_equal(out["fg"].cpu().numpy()[0].astype(bool), fg)
    assert out["box"].cpu().numpy()[0].tolist() == want
    best = oracle.iou(want, gts[0]).max()
    assert out["iou"].item() == pytest.approx(best, abs=1e-6) and out["hit"].item() == int(best >= 0.5)


@pytest.mark.parametrize("grid", [(7, 13), (32, 24)], ids=lambda g: f"{g[0]}x{g[1]}")
def test_bipartition_and_box_match_the_oracle_end_to_end(native, grid):
    from dinov3_jax.eval.discovery import boxes_of
    h, w = grid
    n = 4
    feats = _clustered(n, h, w, 128, seed=h * w + 7)
    cut = _cut(feats)
    sizes = [(h * 16 - 5, w * 16 - 3)] * n
    out = boxes_of(cut["x"], grid, 16, sizes, [np.zeros((0, 4))] * n)
    f = feats.double().cpu().numpy()
    A_bits = _dense(cut["bits"], h * w)
    for m in range(n):
        A = np.where(A_bits[m], 1.0, EPS)
        xr, _, _ = oracle.fiedler(A, A.sum(1))
        fg, seed = oracle.bipartition(xr)
        margin = 1e-3 * np.abs(xr).max()
        clear = np.abs(xr - xr.mean()) > margin
        got = out["fg"].cpu().numpy()[m].astype(bool)
        assert np.array_equal(got[clear], fg[clear]), int((got != fg)[clear].sum())
        assert out["box"].cpu().numpy()[m].tolist() == oracle.component_box(fg, seed, grid, 16, sizes[m])
        assert out["iou"][m].item() == 0.0 and out["hit"][m].item() == 0
    assert f.shape == (n, h * w, 128)


# ------------------------------------------------------------------------------------------------ arguments
def test_arguments_are_checked_before_any_launch(native):
    from dinov3_jax import _native, ops
    from dinov3_jax.eval.discovery import boxes_of
    big = 4097
    sim = torch.empty(1, big, big + 3, device="cuda")[:, :, :big]
    before = _native.launch_count()
    with pytest.raises(_native.NativeError, match="4096"):
        ops.od_graph(sim, TAU, EPS, torch.empty(1, big, -(-big // 32), dtype=torch.int32, device="cuda"),
                     torch.empty(1, big, device="cuda"))
    P = 12
    buf = torch.empty(1 * P * 16 + 1, device="cuda")
    off = buf[1:].view(1, P, 16)[:, :, :P]                           # rows 16-byte misaligned
    bits = torch.empty(1, P, 1, dtype=torch.int32, device="cuda")
    deg = torch.empty(1, P, device="cuda")
    with pytest.raises(_native.NativeError, match="aligned"):
        ops.od_graph(off, TAU, EPS, bits, deg)
    x = torch.empty(1, P, device="cuda")
    small = [torch.empty(1, dtype=dt, device="cuda") for dt in (f32, torch.int32, torch.int32)]
    with pytest.raises(_native.NativeError, match="k_max"):
        ops.od_fiedler(bits, deg, EPS, x, *small, k_max=0)
    with pytest.raises(_native.NativeError, match="k_max"):
        ops.od_fiedler(bits, deg, EPS, x, *small, k_max=257)
    xs = torch.zeros(1, P, device="cuda")
    with pytest.raises(_native.NativeError, match="count"):
        ops.od_box(xs, (3, 4), 16, [(48, 64)], [3], torch.zeros(1, 2, 4, device="cuda"),
                   torch.empty(1, P, dtype=torch.uint8, device="cuda"), torch.empty(1, 4, dtype=torch.int32, device="cuda"),
                   torch.empty(1, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda"))
    with pytest.raises(_native.NativeError, match="grid"):
        boxes_of(xs, (3, 4), 16, [(49, 64)], [np.zeros((1, 4))])
    assert _native.launch_count() == before


# ------------------------------------------------------------------------------------------------ reproducibility
def test_two_runs_give_the_same_bytes(native):
    from dinov3_jax.eval.discovery import boxes_of
    h, w = 32, 24
    feats = _clustered(4, h, w, 256, seed=9)
    runs = []
    for _ in range(2):
        cut = _cut(feats)
        out = boxes_of(cut["x"], (h, w), 16, [(h * 16, w * 16)] * 4, [np.array([[0.0, 0.0, 99.0, 99.0]])] * 4)
        runs.append([cut["x"].cpu(), cut["lambda2"].cpu(), cut["iters"].cpu(), out["box"].cpu(), out["iou"].cpu()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ end to end
def _tiny_vit_checkpoint(path, depth=4):
    from dinov3_jax.checkpointer import save_checkpoint, tree_from_flat
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=384, depth=depth, heads=6, layerscale=0.5)
    flat = init_backbone(cfg, torch.Generator().manual_seed(0))
    save_checkpoint(path, iteration=4, params={"teacher_backbone": tree_from_flat(flat)})


def _scenes_npz(path, seed=0):
    """Five images of two sizes (grids 4 x 5 and 6 x 4 at patch 16) in one padded array: a textured background with one
    bright rectangle, its box the ground truth."""
    rng = np.random.default_rng(seed)
    sizes = [(64, 80), (96, 60), (64, 80), (90, 64), (61, 77)]
    Hm, Wm = max(s[0] for s in sizes), max(s[1] for s in sizes)
    images = np.zeros((len(sizes), Hm, Wm, 3), np.uint8)
    boxes = np.zeros((len(sizes), 2, 4), np.float32)
    for i, (H, W) in enumerate(sizes):
        im = rng.normal(90, 25, (H, W, 3))
        y0, x0 = int(rng.integers(0, H // 2)), int(rng.integers(0, W // 2))
        y1, x1 = y0 + H // 3, x0 + W // 3
        im[y0:y1, x0:x1] = rng.random(3) * 120 + 130
        images[i, :H, :W] = np.clip(im, 0, 255).astype(np.uint8)
        boxes[i, 0] = [x0, y0, x1, y1]
    np.savez(path, images=images, sizes=np.array(sizes), boxes=boxes, n_boxes=np.array([1, 1, 1, 1, 0]))
    return images, sizes, boxes


def _opts(tmp_path):
    return ["student.arch=vit_small", f"evaluation.discovery.dataset_path={tmp_path / 'd.npz'}",
            "evaluation.discovery.batch_size=2", "evaluation.discovery.num_workers=0",
            "evaluation.discovery.save_boxes=true"]


def test_eval_only_discovery_writes_the_same_results_twice_and_the_oracle_boxes(native, tmp_path):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.eval.discovery import image_features
    from dinov3_jax.train.train import eval_backbone, main
    _tiny_vit_checkpoint(tmp_path / "weights")
    images, sizes, boxes = _scenes_npz(tmp_path / "d.npz")
    outs = []
    for run in ("a", "b"):
        res = main(["--eval-only", "--eval", "discovery", "--eval-pretrained-weights", str(tmp_path / "weights"),
                    "--output-dir", str(tmp_path / run), "--opts"] + _opts(tmp_path))
        outs.append((tmp_path / run / "eval" / "manual_5" / "results_discovery.json").read_text())
        written = json.loads(outs[-1])
        assert written == res
        assert sorted(written) == ["CorLoc", "boxes", "config", "n_images", "n_unconverged", "protocol"]
        assert written["n_images"] == 4 and written["n_unconverged"] == 0          # image 4 has no box: not scored
        assert sorted(written["boxes"]) == ["00000", "00001", "00002", "00003"]
        assert written["protocol"] == {"tau": 0.2, "eps": 1e-5, "patch_size": 16}
        assert written["config"]["dataset_path"] == str(tmp_path / "d.npz")
    assert outs[0] == outs[1]
    written = json.loads(outs[0])
    print("discovery end to end:", written)
    # the oracle's boxes from the same extracted features
    model = eval_backbone(setup_config(DinoV3SetupArgs(opts=["student.arch=vit_small"])), str(tmp_path / "weights"))
    hits = []
    for i in range(4):
        H, W = sizes[i]
        with torch.no_grad():
            f = image_features(model, [images[i, :H, :W]], (0.485, 0.456, 0.406), (0.229, 0.224, 0.225), "cuda")
        grid = (-(-H // 16), -(-W // 16))
        want = oracle.discover(f[0].double().cpu().numpy(), grid, 16, (H, W))
        got = written["boxes"][f"{i:05d}"]
        print(f"image {i}: box {got['box']} (oracle {want['box']}), gap {want['gap']:.2e}")
        assert got["box"] == want["box"]
        best = oracle.iou(want["box"], boxes[i, :1]).max()
        assert got["iou"] == pytest.approx(best, abs=1e-6)
        hits.append(best >= 0.5)
    assert written["CorLoc"] == pytest.approx(np.mean(hits))


def test_do_train_calls_do_discovery_eval_at_the_eval_period(native, tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch, train
    calls = []
    monkeypatch.setattr(train, "do_discovery_eval", lambda config, model, header: calls.append(header) or {})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval", "do_video_eval", "do_correspondence_eval"):
        monkeypatch.setattr(train, name, lambda *a, _n=name: pytest.fail(f"{_n}: no dataset is configured"))
    opts = _opts(tmp_path) + ["train.batch_size_per_gpu=2", f"train.output_dir={tmp_path}", "checkpointing.period=100",
                              "evaluation.eval_period_iterations=2", "dino.head_n_prototypes=1024",
                              "ibot.head_n_prototypes=1024"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    train.do_train(config, SSLMetaArch(config), max_iters=4, print_freq=1)
    assert calls == ["training_1", "training_3"]
