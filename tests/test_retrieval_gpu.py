"""-m gpu: instance retrieval (csrc/retrieval.cu, dinov3_jax/eval/retrieval.py).  The crop-and-resize against torch's
float64 antialiased bicubic; the exact ranks, AP and P@k against tests/retrieval_oracle.py on heavily tied similarities
from N = 1 to 2^20; the argument checks; and the evaluation end to end through --eval-only (its descriptors against
DinoVisionTransformer on the same inputs, its scores against the oracle, two byte-identical runs) and do_train."""
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import retrieval_oracle as oracle

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
# the kernel takes mean and std as fp32: the references use the same values
MEAN32 = [float(np.float32(v)) for v in MEAN]
STD32 = [float(np.float32(v)) for v in STD]


def _reference(img, box, out_hw):
    """float64 [h, w, 3]: torch's antialiased bicubic of the crop box of a uint8 HWC image, then normalised."""
    x0, y0, x1, y1 = box
    crop = torch.from_numpy(np.ascontiguousarray(img[y0:y1, x0:x1])).double().permute(2, 0, 1)[None]
    r = F.interpolate(crop, size=out_hw, mode="bicubic", antialias=True, align_corners=False)[0].permute(1, 2, 0)
    return (r / 255.0 - torch.tensor(MEAN32, dtype=torch.float64)) / torch.tensor(STD32, dtype=torch.float64)


def _bf16_ulp(x):
    a = np.abs(x)
    return np.where(a > 0, np.exp2(np.floor(np.log2(np.where(a > 0, a, 1.0))) - 7), 2.0 ** -133)


# ------------------------------------------------------------------------------------------------ resize
def test_resize_within_one_bf16_ulp_of_torch_float64(native):
    from dinov3_jax import ops
    rng = np.random.default_rng(0)
    # (image H, W, crop box, output h, w): 2x and 4x downscales, odd ratios, a small crop enlarged, a 1-pixel-wide
    # crop, and a large downscale
    cases = [((96, 128), (0, 0, 128, 96), (48, 64)), ((96, 128), (0, 0, 128, 96), (32, 32)),
             ((77, 131), (5, 9, 120, 70), (48, 80)), ((60, 50), (10, 20, 23, 31), (32, 48)),
             ((40, 40), (7, 0, 8, 40), (16, 16)), ((700, 300), (0, 0, 300, 700), (64, 32)),
             ((33, 65), (0, 0, 65, 33), (80, 48))]
    for (H, W), box, (h, w) in cases:
        imgs = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(2)]
        imgs[1] = np.clip(imgs[1].astype(np.int64) // 64 * 80, 0, 255).astype(np.uint8)    # hard edges
        flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).cuda()
        desc = [[k * H * W * 3, H, W, *box] for k in range(2)]
        out = torch.empty(2, h, w, 3, dtype=bf16, device="cuda")
        ops.ret_resize(flat, desc, out, mean=MEAN, std=STD)
        got = out.double().cpu().numpy()
        for k in range(2):
            ref = _reference(imgs[k], box, (h, w)).numpy()
            err = np.abs(got[k] - ref)
            ratio = (err / _bf16_ulp(ref)).max()
            print(f"resize {H}x{W} box {box} -> {h}x{w}: max error {err.max():.2e}, {ratio:.3f} bf16 ulp")
            assert (err <= _bf16_ulp(ref)).all()


def test_resize_identity_is_plain_normalisation(native):
    from dinov3_jax import ops
    rng = np.random.default_rng(1)
    H, W = 48, 80
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    out = torch.empty(1, H, W, 3, dtype=bf16, device="cuda")
    ops.ret_resize(torch.from_numpy(img.reshape(-1)).cuda(), [[0, H, W, 0, 0, W, H]], out, mean=MEAN, std=STD)
    want = ((torch.from_numpy(img).double() / 255.0 - torch.tensor(MEAN32, dtype=torch.float64))
            / torch.tensor(STD32, dtype=torch.float64)).to(bf16)
    assert torch.equal(out[0].cpu(), want)


# ------------------------------------------------------------------------------------------------ rank / AP
def _lists(rng, Q, N, sizes=(6, 4, 5)):
    """Overlapping easy / hard / junk lists per query (duplicates within and across lists; some lists empty)."""
    out = {"easy": [], "hard": [], "junk": []}
    for q in range(Q):
        for name, n in zip(("easy", "hard", "junk"), sizes):
            k = 0 if (q + len(name)) % 5 == 0 else int(rng.integers(1, n + 1))
            out[name].append(rng.integers(0, N, k))
        if N > 1 and len(out["easy"][q]) and q % 2:
            out["junk"][q] = np.concatenate([out["junk"][q], out["easy"][q][:1]])     # easy and junk overlap
            out["hard"][q] = np.concatenate([out["hard"][q], out["easy"][q][-1:]])    # easy and hard overlap
    return out


def _check_rank_ap(sim, lists):
    from dinov3_jax import ops
    from dinov3_jax.eval.retrieval import csr
    Q, N = sim.shape
    ld = -(-N // 4) * 4
    s = torch.zeros(Q, ld, dtype=f32, device="cuda")
    s[:, :N] = torch.from_numpy(sim)
    cs = [csr(lists[k]) for k in ("easy", "hard", "junk")]
    total = sum(len(c[1]) for c in cs)
    ranks = torch.empty(total, dtype=torch.int32, device="cuda")
    ap = torch.empty(Q, 3, dtype=torch.float64, device="cuda")
    pk = torch.empty(Q, 3, 3, dtype=torch.float64, device="cuda")
    n_ok = torch.empty(Q, 3, dtype=torch.int32, device="cuda")
    ops.ret_rank_ap(s[:, :N], N, *cs, ranks, ap, pk, n_ok)
    ranks, ap, pk, n_ok = ranks.cpu().numpy(), ap.cpu().numpy(), pk.cpu().numpy(), n_ok.cpu().numpy()
    # integer ranks, exactly
    off = 0
    for k, (ptr, idx) in zip(("easy", "hard", "junk"), cs):
        for q in range(Q):
            want = oracle.ranks(sim[q])[idx[ptr[q]:ptr[q + 1]]]
            assert np.array_equal(ranks[off + ptr[q]:off + ptr[q + 1]], want), (k, q)
        off += len(idx)
    # AP and P@k within 1e-12, NaN where there is no ok image
    for q in range(Q):
        sc = oracle.query_scores(sim[q], lists["easy"][q], lists["hard"][q], lists["junk"][q])
        for p, name in enumerate(oracle.PROTOCOLS):
            a, pks, n = sc[name]
            assert n_ok[q, p] == n
            if n == 0:
                assert np.isnan(ap[q, p]) and np.isnan(pk[q, p]).all()
            else:
                assert abs(ap[q, p] - a) <= 1e-12 and np.abs(pk[q, p] - pks).max() <= 1e-12
    return ap, pk, n_ok


@pytest.mark.parametrize("N", [1, 31, 4993, 1 << 20])
def test_rank_ap_against_the_oracle_on_tied_similarities(native, N):
    rng = np.random.default_rng(N)
    Q = 7 if N < (1 << 20) else 3
    levels = np.array([-0.25, -0.0, 0.0, 0.125, 0.5, 0.75], np.float32)      # a few values: most columns tie
    sim = levels[rng.integers(0, len(levels), (Q, N))]
    lists = _lists(rng, Q, N)
    if N >= 4993:                                                             # long lists, over every chunk
        big = rng.integers(0, N, 3000)
        lists["easy"][0] = big[:1500]
        lists["hard"][0] = big[1000:2500]
        lists["junk"][0] = rng.integers(0, N, 2000)
    ap, _, n_ok = _check_rank_ap(sim, lists)
    print(f"rank/AP N={N}: n_ok {n_ok.tolist()}, AP {np.round(ap, 4).tolist()}")


def test_rank_ap_is_the_same_bits_twice(native):
    rng = np.random.default_rng(3)
    sim = rng.normal(size=(5, 3000)).astype(np.float32).round(2)
    lists = _lists(rng, 5, 3000)
    a = _check_rank_ap(sim, lists)
    b = _check_rank_ap(sim, lists)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def test_arguments_are_refused_before_any_launch(native):
    from dinov3_jax import _native, ops
    sim = torch.zeros(2, 16, device="cuda")
    out = (torch.empty(1, dtype=torch.int32, device="cuda"), torch.empty(2, 3, dtype=torch.float64, device="cuda"),
           torch.empty(2, 3, 3, dtype=torch.float64, device="cuda"), torch.empty(2, 3, dtype=torch.int32, device="cuda"))
    empty = ([0, 0, 0], [])
    before = _native.launch_count()
    for easy, msg in ((([0, 1, 1], [16]), "outside"), (([0, 1, 0], [3]), "decrease"), (([1, 1, 1], [3]), "start at 0")):
        with pytest.raises(_native.NativeError, match=msg):
            ops.ret_rank_ap(sim, 16, easy, empty, empty, *out)
    with pytest.raises(_native.NativeError, match="8192"):
        ops.ret_rank_ap(sim, 16, ([0, 8193, 8193], [1] * 8193), empty, empty,
                        torch.empty(8193, dtype=torch.int32, device="cuda"), *out[1:])
    x = torch.empty(1, 16, 16, 3, dtype=bf16, device="cuda")
    src = torch.zeros(20 * 20 * 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(_native.NativeError, match="crop box"):
        ops.ret_resize(src, [[0, 20, 20, 0, 0, 21, 20]], x, mean=MEAN, std=STD)
    with pytest.raises(_native.NativeError, match="source buffer"):
        ops.ret_resize(src, [[3, 20, 20, 0, 0, 20, 20]], x, mean=MEAN, std=STD)
    assert _native.launch_count() == before


# ------------------------------------------------------------------------------------------------ end to end
def _tiny_vit_checkpoint(path, depth=4):
    from dinov3_jax.checkpointer import save_checkpoint, tree_from_flat
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=384, depth=depth, heads=6, layerscale=0.5)
    flat = init_backbone(cfg, torch.Generator().manual_seed(0))
    save_checkpoint(path, iteration=4, params={"teacher_backbone": tree_from_flat(flat)})


def _revisited_root(root, seed=0):
    """A synthetic revisited root: 12 database images of three sizes (three 'landmarks', each a coloured pattern on
    noise) and 4 queries cropped from images of the same landmarks; ground truth by landmark."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    (root / "jpg").mkdir(parents=True)
    sizes = [(96, 128), (128, 96), (80, 80)]
    colours = rng.integers(40, 220, (3, 3))
    db, land = [], []
    for i in range(12):
        H, W = sizes[i % 3]
        L = i % 4 % 3
        im = rng.normal(120, 30, (H, W, 3))
        y0, x0 = int(rng.integers(0, H // 3)), int(rng.integers(0, W // 3))
        im[y0:y0 + H // 2, x0:x0 + W // 2] = colours[L]
        Image.fromarray(np.clip(im, 0, 255).astype(np.uint8)).save(root / "jpg" / f"db_{i}.jpg", quality=95)
        db.append(f"db_{i}")
        land.append(L)
    qs, gnd = [], []
    for q in range(4):
        L = q % 3
        im = rng.normal(120, 30, (112, 112, 3))
        im[20:80, 30:90] = colours[L]
        Image.fromarray(np.clip(im, 0, 255).astype(np.uint8)).save(root / "jpg" / f"q_{q}.jpg", quality=95)
        qs.append(f"q_{q}")
        same = [i for i in range(12) if land[i] == L]
        gnd.append({"bbx": np.array([15.5, 10.2, 95.0, 90.7]), "easy": same[:2], "hard": np.array(same[2:], np.int64),
                    "junk": [(same[0] + 1) % 12] if q != 3 else []})
    gnd[3]["easy"], gnd[3]["hard"] = [], []                                 # a query with no positives
    import pickle
    (root / "gnd_roxford5k.pkl").write_bytes(pickle.dumps({"imlist": db, "qimlist": qs, "gnd": gnd}))


def _opts(tmp_path):
    return ["student.arch=vit_small", f"evaluation.retrieval.dataset_path={tmp_path / 'root'}",
            "evaluation.retrieval.image_size=96", "evaluation.retrieval.batch_size=3",
            "evaluation.retrieval.num_workers=0", "evaluation.retrieval.save_ranks=true"]


def test_eval_only_retrieval_end_to_end(native, tmp_path):
    from dinov3_jax import ops
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.eval import make_retrieval_dataset
    from dinov3_jax.eval.retrieval import (SCALES, batches, extract_descriptors, plan_inputs, query_box,
                                           rank_queries, resize_batch)
    from dinov3_jax.train.train import eval_backbone, main
    _tiny_vit_checkpoint(tmp_path / "weights")
    _revisited_root(tmp_path / "root")
    outs = []
    for run in ("a", "b"):
        res = main(["--eval-only", "--eval", "retrieval", "--eval-pretrained-weights", str(tmp_path / "weights"),
                    "--output-dir", str(tmp_path / run), "--opts"] + _opts(tmp_path))
        outs.append((tmp_path / run / "eval" / "manual_5" / "results_retrieval.json").read_text())
        written = json.loads(outs[-1])
        assert written == res
        assert sorted(written) == ["config", "mAP", "mP@k", "n_database", "n_empty", "n_queries", "protocol", "ranks"]
        assert written["n_queries"] == 4 and written["n_database"] == 12
        assert written["n_empty"] == {"easy": 1, "medium": 1, "hard": 1}
        assert written["protocol"]["scales"] == [1.0, 0.7071067811865476, 0.5]
        assert written["config"]["dataset_path"] == str(tmp_path / "root")
        assert written["ranks"]["q_3"]["ap"] == {"easy": None, "medium": None, "hard": None}
        assert all(len(v["top"]) == 12 for v in written["ranks"].values())
    assert outs[0] == outs[1]
    written = json.loads(outs[0])
    print("retrieval end to end:", {k: written[k] for k in ("mAP", "mP@k", "n_empty")})

    # the descriptors: DinoVisionTransformer's class token on the same resized inputs, bit for bit
    model = eval_backbone(setup_config(DinoV3SetupArgs(opts=["student.arch=vit_small"])), str(tmp_path / "weights"))
    ds = make_retrieval_dataset(str(tmp_path / "root"), "roxford5k")
    kw = dict(image_size=96, scales=list(SCALES), batch_size=3, num_workers=0)
    boxes = [query_box(b, s) for b, s in zip(ds.q_bbx, ds.q_sizes)]
    got = {"db": extract_descriptors(model, ds.db_sizes, None, ds.load_db, **kw),
           "q": extract_descriptors(model, ds.q_sizes, boxes, ds.load_query, **kw)}
    for key, sizes, bx, load in (("db", ds.db_sizes, None, ds.load_db), ("q", ds.q_sizes, boxes, ds.load_query)):
        cls = torch.empty_like(got[key]["cls"])
        for batch in batches(plan_inputs(sizes, bx, 96, list(SCALES), 16), 3):
            x = resize_batch([load(i) for _, i, _, _ in batch], batch, MEAN, STD, "cuda")
            with torch.no_grad():
                tok = model.forward_features(x)["x_norm_clstoken"]
            for k, (_, i, s, _) in enumerate(batch):
                cls[s, i] = tok[k]
        assert torch.equal(cls, got[key]["cls"])
        total = (cls[0] + cls[1]) + cls[2]                                 # the scale order
        same = torch.empty_like(got[key]["desc"])
        ops.knn_normalize(total, y_bf16=same)
        assert torch.equal(same, got[key]["desc"])
        want = total.double() / total.double().norm(dim=1, keepdim=True)
        assert (got[key]["desc"].double() - want).abs().max().item() <= 2.0 ** -8
    # the scores: the oracle on the same similarities
    out = rank_queries(got["q"]["desc"], got["db"]["desc"], ds.easy, ds.hard, ds.junk, top=100)
    res, _ = oracle.evaluate(out["sim"].double().cpu().numpy(), ds.easy, ds.hard, ds.junk)
    assert res["n_empty"] == written["n_empty"]
    for p in oracle.PROTOCOLS:
        assert abs(res["mAP"][p] - written["mAP"][p]) <= 1e-10
        for k in ("1", "5", "10"):
            assert abs(res["mP@k"][p][k] - written["mP@k"][p][k]) <= 1e-10
    for q in range(4):
        assert out["top"][q].tolist() == written["ranks"][ds.q_names[q]]["top"]
        assert out["top"][q].tolist() == oracle.order(out["sim"][q].double().cpu().numpy()).tolist()


def test_do_train_calls_do_retrieval_eval_at_the_eval_period(native, tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch, train
    calls = []
    monkeypatch.setattr(train, "do_retrieval_eval", lambda config, model, header: calls.append(header) or {})
    for name in ("do_test", "do_linear_eval", "do_seg_eval", "do_depth_eval", "do_video_eval", "do_correspondence_eval",
                 "do_discovery_eval"):
        monkeypatch.setattr(train, name, lambda *a, _n=name: pytest.fail(f"{_n}: no dataset is configured"))
    opts = _opts(tmp_path) + ["train.batch_size_per_gpu=2", f"train.output_dir={tmp_path}", "checkpointing.period=100",
                              "evaluation.eval_period_iterations=2", "dino.head_n_prototypes=1024",
                              "ibot.head_n_prototypes=1024"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    train.do_train(config, SSLMetaArch(config), max_iters=4, print_freq=1)
    assert calls == ["training_1", "training_3"]
