"""-m gpu: the linear depth probe (csrc/depth.cu, dinov3_jax/eval/depth.py).  The loss and its gradient, and the
per-image metrics, against the float64 statement in tests/depth_oracle.py (pinned to torch autograd on the CPU); the
crops against d3_seg_crop and torch's 'nearest'; the head's steps against a torch fp32 restatement; and the
evaluation end to end through --eval-only and do_train."""
import json

import numpy as np
import pytest
import torch

import depth_oracle

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
LO, HI = 0.001, 10.0


# ------------------------------------------------------------------------------------------------ loss and gradient
def _case(B, h, w, Hl, Wl, nb, seed, shift=0.0, invalid=0.25, all_invalid=False):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, h, w, nb, generator=g) * 2.0 + shift
    gt = torch.rand(B, Hl, Wl, generator=g) * 8.0 + 0.3
    bad = torch.rand(B, Hl, Wl, generator=g) < invalid
    gt[bad] = torch.where(torch.rand(B, Hl, Wl, generator=g) < 0.5, 0.0, 12.0)[bad]   # missing, or beyond max_depth
    if all_invalid:
        gt.zero_()
    return z, gt


HEAD_CASES = [(2, 26, 34, 416, 544, 256, 0.0, False), (1, 30, 40, 480, 640, 256, 0.0, False),
              (3, 7, 9, 50, 61, 64, 0.0, False), (2, 13, 11, 40, 70, 100, -2.0, False),
              (1, 8, 6, 5, 4, 32, 0.0, False), (16, 26, 34, 416, 544, 256, 0.0, False),
              (2, 5, 6, 80, 96, 16, 0.0, True)]


@pytest.mark.parametrize("case", HEAD_CASES,
                         ids=lambda c: f"B{c[0]}_{c[1]}x{c[2]}_to_{c[3]}x{c[4]}_bins{c[5]}_shift{c[6]}_none{int(c[7])}")
def test_depth_head_against_float64(native, case):
    from dinov3_jax import ops
    B, h, w, Hl, Wl, nb, shift, none = case
    z, gt = _case(B, h, w, Hl, Wl, nb, seed=B * 13 + nb, shift=shift, all_invalid=none)
    Cp = -(-nb // 64) * 64
    L = torch.full((B * h * w, Cp + 8), float("nan"))                # columns >= n_bins are never read
    L[:, :nb] = z.reshape(-1, nb)
    L, G = L.cuda(), gt.cuda()
    loss, count = torch.empty(1, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
    dz = torch.full((B * h * w + 3, Cp), 7.0, device="cuda")
    dzb = torch.full((B * h * w + 3, Cp), 7.0, dtype=bf16, device="cuda")
    ops.depth_head_fwd_bwd(L, G, (h, w), nb, LO, HI, loss, count, dz_f32=dz, dz_bf16=dzb, Cp=Cp)
    want_loss, want_dz, n, env = depth_oracle.si_loss(z.cuda(), G, LO, HI)
    assert count.item() == n
    got = dz[:B * h * w, :nb].double().view(B, h, w, nb)
    if none:
        assert n == 0 and loss.item() == 0.0 and (got == 0).all()
    else:
        assert loss.item() == pytest.approx(want_loss, rel=1e-5)
        d, S = depth_oracle.cell_depth(z.cuda(), LO, HI)
        c = depth_oracle.centres(nb, LO, HI, "cuda")
        # dZ = 1[z > 0] (c - d) / S * dL/dd.  dL/dd is a fixed-order fp32 sum of terms w dL/dd_hat, each within a few
        # fp32 ulps plus the rounding of g (covered by the oracle's 1e-5 slack) of its float64 value: its error is far
        # below 2^-12 of the envelope `env` of those terms.  d carries about 1e-6 d of fp32 rounding, which (c - d)
        # sees as an absolute error: a slack of 0.1 (max - min) at 2^-12 covers it by more than ten times.
        bound = 2.0 ** -12 * ((c - d[..., None]).abs() + 0.1 * (HI - LO)) / S[..., None] * env[..., None]
        ratio = ((got - want_dz).abs() / (bound + 1e-30)).max().item()
        nz = (z <= 0).double().mean().item()
        print(f"depth head {case}: loss rel {abs(loss.item() - want_loss) / want_loss:.1e}, worst err / bound "
              f"{ratio:.3f}, {100 * nz:.0f}% of z <= 0")
        assert ratio <= 1.0
        assert (got[z.cuda() <= 0] == 0).all()
    assert (dz[:B * h * w, nb:] == 0).all() and (dz[B * h * w:] == 7.0).all()
    # the bf16 copy is the fp32 gradient rounded to nearest: within 2^-9 of it, i.e. of the bound above plus 2^-9
    assert torch.equal(dzb[:B * h * w], dz[:B * h * w].to(bf16))
    loss2, dz2 = torch.empty(1, device="cuda"), torch.empty_like(dz)
    ops.depth_head_fwd_bwd(L, G, (h, w), nb, LO, HI, loss2, count, dz_f32=dz2, Cp=Cp)
    assert torch.equal(loss2, loss) and torch.equal(dz2[:B * h * w], dz[:B * h * w])


def test_depth_head_single_valid_pixel_gives_zero(native):
    from dinov3_jax import ops
    z, gt = _case(1, 4, 4, 16, 16, 32, seed=1, all_invalid=True)
    gt[0, 3, 5] = 2.0
    loss, count = torch.empty(1, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
    dz = torch.full((16, 64), 7.0, device="cuda")
    ops.depth_head_fwd_bwd(z.reshape(16, 32).cuda(), gt.cuda(), (4, 4), 32, LO, HI, loss, count, dz_f32=dz, Cp=64)
    assert count.item() == 1 and loss.item() == 0.0 and (dz == 0).all()


# ------------------------------------------------------------------------------------------------ metrics
@pytest.mark.parametrize("case", [(1, 26, 35, 480, 640, 256, True), (1, 26, 35, 480, 640, 256, False),
                                  (3, 30, 40, 480, 640, 64, True), (2, 9, 7, 45, 61, 32, False)])
def test_depth_predict_metrics_against_float64(native, case):
    from dinov3_jax import ops
    B, h, w, Hl, Wl, nb, eigen = case
    z, gt = _case(B, h, w, Hl, Wl, nb, seed=31 + nb + B)
    z[0, :2] = -3.0                                  # all bins at the floor: depth (min + max) / 2
    z[-1, -1, :, nb // 2:] = 40.0                    # deep cells, some clamped to max_depth
    crop = (45, 471, 41, 601) if eigen else None
    sums = torch.full((B, 9), 7.0, dtype=torch.float64, device="cuda")
    ops.depth_predict_metrics(z.reshape(-1, nb).cuda(), gt.cuda(), (h, w), nb, LO, HI, sums, crop=crop)
    want, near = depth_oracle.metric_sums(z.cuda(), gt.cuda(), LO, HI, crop=crop)
    assert torch.equal(sums[:, 0], want[:, 0])
    # fp32 per-pixel terms summed in fixed order in a tile, fp64 across tiles
    assert torch.allclose(sums[:, 1:6], want[:, 1:6], rtol=1e-5, atol=0)
    # a pixel whose ratio lies within fp32 rounding of 1.25^k may count on either side
    diff = (sums[:, 6:] - want[:, 6:]).abs()
    print(f"depth metrics {case}: hit counts differ by {diff.max().item():.0f}, near ties {near.max().item()}")
    assert (diff <= near).all(), (diff, near)
    again = torch.empty_like(sums)
    ops.depth_predict_metrics(z.reshape(-1, nb).cuda(), gt.cuda(), (h, w), nb, LO, HI, again, crop=crop)
    assert torch.equal(again, sums)


# ------------------------------------------------------------------------------------------------ crops
def test_depth_crop_image_is_seg_crop_and_depth_is_torch_nearest(native):
    import torch.nn.functional as Fn
    from dinov3_jax import ops
    from dinov3_jax.eval.depth import _pack_depth, sample_depth_boxes
    rng = np.random.default_rng(0)
    hc, wc = 48, 64
    sizes = [(60, 80), (48, 64), (40, 100), (70, 50), (33, 47)]
    imgs = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in sizes]
    deps = [rng.uniform(0.1, 9.0, (H, W)).astype(np.float32) for H, W in sizes]
    boxes = sample_depth_boxes(torch.Generator().manual_seed(3), sizes, (hc, wc)).tolist()
    boxes += [[90, 120, 20, 30, 1, 0], [30, 40, 0, 0, 0, 0], [48, 64, 0, 0, 1, 0], [35, 52, 0, 3, 1, 0],
              [66, 94, 18, 30, 0, 0]]                # resized boxes, some leaving the image
    imgs, deps, sizes = imgs * 2, deps * 2, sizes * 2
    flat, dflat, desc = _pack_depth(list(zip(imgs, deps)))
    bx = torch.tensor(boxes, dtype=torch.int32).cuda()
    taps = ops.seg_max_taps(sizes, [b[:2] for b in boxes])
    n = len(imgs)
    for dt in (torch.uint8, bf16):
        kw = {} if dt == torch.uint8 else dict(mean=MEAN, std=STD)
        x = torch.empty(n, hc, wc, 3, dtype=dt, device="cuda")
        ref = torch.empty_like(x)
        d = torch.full((n, hc, wc), 7.0, device="cuda")
        ops.depth_crop(flat.cuda(), desc.cuda(), bx, x, max_taps=taps, depths=dflat.cuda(), depth_out=d, **kw)
        ops.seg_crop(flat.cuda(), desc.cuda(), bx, ref, max_taps=taps, **kw)
        assert torch.equal(x, ref)
    assert any(b[0] - b[2] < hc or b[1] - b[3] < wc for b in boxes)
    for i, (dep, box) in enumerate(zip(deps, boxes)):
        rh, rw, top, left, flip = box[:5]
        up = Fn.interpolate(torch.from_numpy(dep).cuda()[None, None], size=(rh, rw), mode="nearest")[0, 0]
        vh, vw = min(hc, rh - top), min(wc, rw - left)
        win = up[top:top + vh, left:left + vw]
        want = torch.zeros(hc, wc, device="cuda")
        want[:vh, :vw] = win.flip(1) if flip else win
        assert torch.equal(d[i], want), (sizes[i], box)


# ------------------------------------------------------------------------------------------------ head steps
def test_head_steps_against_torch_fp32_restatement(native):
    import torch.nn.functional as Fn
    from dinov3_jax.eval.depth import DepthLinearHead
    from dinov3_jax.eval.segmentation import seg_lr
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    B, h, w, K, NB, S, STEPS, T = 4, 8, 8, 256, 64, 128, 6, 20
    g = torch.Generator().manual_seed(0)
    proj = torch.randn(K, generator=g) / K ** 0.5
    head = DepthLinearHead(K, B * h * w, T, n_bins=NB, min_depth=LO, max_depth=HI, lr=1e-2, weight_decay=1e-2,
                           warmup_iterations=3, seed=1, device="cuda")
    init = head.state_dict()
    bn = torch.nn.BatchNorm1d(K, affine=False, momentum=0.1).cuda()
    lin = torch.nn.Linear(K, NB).cuda()
    with torch.no_grad():
        lin.weight.copy_(init["weight"])
        lin.bias.zero_()
    opt = torch.optim.AdamW(lin.parameters(), lr=1e-2, weight_decay=1e-2)
    c = torch.linspace(LO, HI, NB, device="cuda")
    for t in range(STEPS):
        feats = (torch.randn(B, h, w, K, generator=g) * 2.0 + 0.5).to(bf16)
        cell = 1.0 + 6.0 * torch.sigmoid(feats.float() @ proj)            # depth a smooth function of the features
        gt = Fn.interpolate(cell[:, None], size=(S, S), mode="bilinear", align_corners=False)[:, 0]
        gt[:, :10] = 0.0                                                 # missing depth
        head.step(feats.view(-1, K).cuda(), gt.cuda(), (h, w), t)
        for grp in opt.param_groups:
            grp["lr"] = seg_lr(1e-2, t, T, 3)
        bn.train()
        z = lin(bn(feats.float().cuda().view(-1, K)))
        q = torch.relu(z) + 0.1
        d = ((q * c).sum(-1) / q.sum(-1)).view(B, 1, h, w)
        dh = Fn.interpolate(d, size=(S, S), mode="bilinear", align_corners=False)[:, 0]
        G = gt.cuda()
        valid = (G > LO) & (G <= HI)
        gl = torch.log(dh[valid] + 1e-3) - torch.log(G[valid] + 1e-3)
        loss = torch.sqrt(torch.var(gl) + 0.15 * gl.mean() ** 2)
        opt.zero_grad()
        loss.backward()
        if t == 0:
            # one gradient from the same weights, bf16 x_hat, W and dZ against fp32.  The logits differ by about 2^-9
            # of their spread, so the few whose relu gate sits that close to 0 (about 0.1 %) flip it and carry their
            # whole dZ term: about sqrt(1e-3) = 3 % relative in L2 (on an H100: 3.6 % for W, 2.9 % for the bias)
            gw, gb = head.gW[:NB].cpu(), head.g_bias[:NB].cpu()
            rw, rb = lin.weight.grad.cpu(), lin.bias.grad.cpu()
            gerr = ((gw - rw).norm() / rw.norm()).item(), ((gb - rb).norm() / rb.norm()).item()
            print(f"depth head first gradient: weight rel L2 {gerr[0]:.2e}, bias {gerr[1]:.2e}")
            assert max(gerr) < 6e-2, gerr
        opt.step()
        assert head.loss.item() == pytest.approx(loss.item(), rel=2e-2), t
    got = head.state_dict()
    W_ref = lin.weight.detach().cpu()
    err = ((got["weight"] - W_ref).norm() / W_ref.norm()).item()
    moved = ((W_ref - init["weight"]).norm() / W_ref.norm()).item()
    print(f"depth head steps: weight error {err:.3e}, moved {moved:.3f}")
    # bf16 x_hat, W and dZ against fp32 throughout.  AdamW's first steps are lr * sign(gradient) per element, so an
    # element whose gradient is no larger than that rounding takes a full step either way, and after 6 steps the
    # weights stay within 15 % of the distance they moved (on an H100: 12.5 %); the bias starts at 0, so the distance
    # it moved is its norm
    assert err < 0.15 * moved and moved > 0.2, (err, moved)
    b_err = ((got["bias"] - lin.bias.detach().cpu()).norm() / lin.bias.detach().norm()).item()
    print(f"depth head steps: bias error {b_err:.3e} of its norm")
    assert b_err < 0.15, b_err
    assert torch.allclose(got["running_mean"], bn.running_mean.cpu(), rtol=1e-3, atol=1e-3)
    assert torch.allclose(got["running_var"], bn.running_var.cpu(), rtol=1e-3, atol=1e-3)


# ------------------------------------------------------------------------------------------------ features
def test_feature_rows_are_torch_cat_of_patches_and_class_tokens(native, tmp_path):
    from dinov3_jax.eval.depth import write_depth_features
    from dinov3_jax.train.train import eval_backbone
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    _tiny_vit_checkpoint(tmp_path / "weights")
    model = eval_backbone(setup_config(DinoV3SetupArgs(opts=["student.arch=vit_small"])), str(tmp_path / "weights"))
    x = torch.randn(2, 32, 48, 3, generator=torch.Generator().manual_seed(0)).to(bf16).cuda()
    layers = model.get_intermediate_layers(x, n=2, return_class_token=True)
    B, P, D = layers[0][0].shape
    want = torch.cat([p for p, _ in layers] + [c[:, None].expand(B, P, D) for _, c in layers], -1)
    out = torch.zeros(B * P + 5, 4 * D + 8, dtype=bf16, device="cuda")
    write_depth_features(model, x, 2, True, out)
    assert torch.equal(out[:B * P, :4 * D], want.reshape(B * P, 4 * D).to(bf16))
    assert (out[B * P:] == 0).all() and (out[:, 4 * D:] == 0).all()
    out2 = torch.zeros(B * P, 2 * D, dtype=bf16, device="cuda")
    write_depth_features(model, x, 2, False, out2)
    assert torch.equal(out2, want[..., :2 * D].reshape(B * P, 2 * D).to(bf16))


# ------------------------------------------------------------------------------------------------ end to end
def _tiny_vit_checkpoint(path, depth=4):
    from dinov3_jax.checkpointer import save_checkpoint, tree_from_flat
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=384, depth=depth, heads=6, layerscale=0.5)
    flat = init_backbone(cfg, torch.Generator().manual_seed(0))
    save_checkpoint(path, iteration=4, params={"teacher_backbone": tree_from_flat(flat)})


def _colour_depth(rgb):
    """depth in metres, a smooth function of the colour: 0.5 + 6 (0.7 r + 0.3 b) / 255"""
    rgb = np.asarray(rgb, dtype=np.float64)
    return 0.5 + 6.0 * (0.7 * rgb[..., 0] + 0.3 * rgb[..., 2]) / 255.0


def _colour_npz(path, n, seed):
    """Images of 96 x 128 made of 32 x 32 blocks of random flat colours with noise; the depth of a pixel is
    `_colour_depth` of its block's colour, missing (0) in a few blocks."""
    rng = np.random.default_rng(seed)
    H, W = 96, 128
    imgs, deps = np.zeros((n, H, W, 3), np.uint8), np.zeros((n, H, W), np.float32)
    for i in range(n):
        for by in range(H // 32):
            for bx in range(W // 32):
                col = rng.integers(0, 256, 3)
                sl = (i, slice(32 * by, 32 * by + 32), slice(32 * bx, 32 * bx + 32))
                imgs[sl] = np.clip(col + rng.normal(0, 12, (32, 32, 3)), 0, 255).astype(np.uint8)
                deps[sl] = _colour_depth(col) if rng.random() > 0.1 else 0.0
    np.savez(path, images=imgs, depths=deps)


def _opts(tmp_path, workers=2, iterations=300):
    return ["student.arch=vit_small", f"evaluation.depth.train_dataset_path={tmp_path / 'train.npz'}",
            f"evaluation.depth.val_dataset_path={tmp_path / 'val.npz'}", "evaluation.depth.batch_size=4",
            "evaluation.depth.crop_size=[64,96]", f"evaluation.depth.iterations={iterations}",
            "evaluation.depth.lr=0.01", "evaluation.depth.warmup_iterations=10", "evaluation.depth.eval_crop=none",
            f"evaluation.depth.num_workers={workers}"]


def test_eval_only_depth_writes_results_depth_json(native, tmp_path):
    from dinov3_jax.train.train import main
    _tiny_vit_checkpoint(tmp_path / "weights")
    _colour_npz(tmp_path / "train.npz", 32, 0)
    _colour_npz(tmp_path / "val.npz", 8, 1)
    metrics = ["a1", "a2", "a3", "abs_rel", "log10", "rmse", "rmse_log", "sq_rel"]
    outs = []
    for run, workers in (("a", 2), ("b", 0)):
        res = main(["--eval-only", "--eval", "depth", "--eval-pretrained-weights", str(tmp_path / "weights"),
                    "--output-dir", str(tmp_path / run), "--opts"] + _opts(tmp_path, workers))
        outs.append((tmp_path / run / "eval" / "manual_5" / "results_depth.json").read_text())
        written = json.loads(outs[-1])
        assert written == res and sorted(written) == sorted(metrics + ["config"])
        assert all(np.isfinite(written[k]) for k in metrics)
        assert written["config"]["crop_size"] == [64, 96] and written["config"]["n_bins"] == 256
    # same seed, other worker count: the same file but for the echoed num_workers
    a, b = json.loads(outs[0]), json.loads(outs[1])
    assert a["config"].pop("num_workers") == 2 and b["config"].pop("num_workers") == 0 and a == b
    # the baseline: the train set's mean valid depth everywhere, scored the same way (per-image rmse, averaged)
    with np.load(tmp_path / "train.npz") as z:
        dtr = z["depths"]
    mean_depth = dtr[(dtr > LO) & (dtr <= HI)].astype(np.float64).mean()
    with np.load(tmp_path / "val.npz") as z:
        dv = z["depths"].astype(np.float64)
    base = np.mean([np.sqrt(((mean_depth - d[(d > LO) & (d <= HI)]) ** 2).mean()) for d in dv])
    print("depth end to end:", {k: round(written[k], 4) for k in metrics}, f"mean-depth rmse {base:.4f}")
    assert written["rmse"] < base, (written["rmse"], base)


def test_do_train_calls_do_depth_eval_at_the_eval_period(native, tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch, train
    calls = []
    monkeypatch.setattr(train, "do_depth_eval", lambda config, model, header: calls.append(header) or {})
    monkeypatch.setattr(train, "do_test", lambda *a: pytest.fail("no k-NN datasets are configured"))
    monkeypatch.setattr(train, "do_linear_eval", lambda *a: pytest.fail("no linear-probe datasets are configured"))
    monkeypatch.setattr(train, "do_seg_eval", lambda *a: pytest.fail("no segmentation datasets are configured"))
    opts = _opts(tmp_path) + ["train.batch_size_per_gpu=2", f"train.output_dir={tmp_path}", "checkpointing.period=100",
                              "evaluation.eval_period_iterations=2", "dino.head_n_prototypes=1024",
                              "ibot.head_n_prototypes=1024"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    train.do_train(config, SSLMetaArch(config), max_iters=4, print_freq=1)
    assert calls == ["training_1", "training_3"]
