"""-m gpu: the linear segmentation probe (csrc/seg.cu, d3_seg_crop in csrc/knn.cu, dinov3_jax/eval/segmentation.py).
The per-pixel cross-entropy and the confusion matrix against float64 torch on the GPU (F.interpolate + cross_entropy +
autograd, the statement tests/seg_oracle.py is pinned to on the CPU), the crops against torchvision's resize, the
BatchNorm statistics against float64, one head step against a torch fp32 restatement, and the evaluation end to end
through --eval-only and do_train."""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
f32, bf16 = torch.float32, torch.bfloat16
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


# ------------------------------------------------------------------------------------------------ cross-entropy
def _xent_case(B, h, w, Hl, Wl, C, seed, all_ignored=()):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, h, w, C, generator=g) * 4.0
    labels = torch.randint(0, C, (B, Hl, Wl), generator=g).to(torch.uint8)
    labels[torch.rand(B, Hl, Wl, generator=g) < 0.1] = 255
    for b in all_ignored:
        labels[b] = 255
    return logits, labels


def _float64_reference(logits, labels):
    """(loss, d loss / d logits [B, h, w, C], envelope [B, h, w, C]) in float64 on the GPU: F.interpolate(bilinear,
    align_corners=False) + F.cross_entropy(ignore_index=255) and autograd; the envelope is the adjoint of
    |softmax - onehot| / n over the valid pixels (the magnitudes each gradient element sums)."""
    import torch.nn.functional as Fn
    B, Hl, Wl = labels.shape
    L = logits.double().cuda().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    y = labels.long().cuda()
    up = Fn.interpolate(L, size=(Hl, Wl), mode="bilinear", align_corners=False)
    loss = Fn.cross_entropy(up, y, ignore_index=255)
    grad, = torch.autograd.grad(loss, L)
    with torch.no_grad():
        valid = y != 255
        p = torch.softmax(up.detach(), 1)
        onehot = torch.zeros_like(p).scatter_(1, torch.where(valid, y, 0)[:, None], 1.0)
        mag = (p - onehot).abs() * valid[:, None] / valid.sum()
        del p, onehot
    env, = torch.autograd.grad(up, L, grad_outputs=mag)
    return loss.item(), grad.permute(0, 2, 3, 1), env.permute(0, 2, 3, 1)


XENT_CASES = [(1, 32, 32, 512, 512, 150, ()), (16, 32, 32, 512, 512, 19, ()), (16, 32, 32, 512, 512, 150, (3,)),
              (1, 37, 50, 592, 800, 150, ()), (2, 37, 50, 592, 800, 19, (1,)), (1, 64, 48, 40, 70, 21, ()),
              (1, 32, 32, 512, 512, 150, (0,))]


@pytest.mark.parametrize("case", XENT_CASES, ids=lambda c: f"B{c[0]}_{c[1]}x{c[2]}_to_{c[3]}x{c[4]}_C{c[5]}_ign{len(c[6])}")
def test_seg_xent_against_float64(native, case):
    from dinov3_jax import ops
    B, h, w, Hl, Wl, C, ign = case
    logits, labels = _xent_case(B, h, w, Hl, Wl, C, seed=B * 7 + C, all_ignored=ign)
    Cp = -(-C // 8) * 8
    L = torch.full((B * h * w, Cp), float("nan"))                   # the padding columns are never read
    L[:, :C] = logits.reshape(-1, C)
    L, lab = L.cuda(), labels.cuda()
    loss, count = torch.empty(1, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
    dz = torch.full((B * h * w + 3, Cp), 7.0, device="cuda")
    dzb = torch.full((B * h * w + 3, Cp), 7.0, dtype=bf16, device="cuda")
    ops.seg_xent_fwd_bwd(L, lab, (h, w), C, loss, count, dz_f32=dz, dz_bf16=dzb, Cp=Cp)
    n = int((labels != 255).sum())
    assert count.item() == n
    if n == 0:
        assert loss.item() == 0.0 and (dz[:B * h * w] == 0).all()
    else:
        want_loss, want_grad, env = _float64_reference(logits, labels)
        assert loss.item() == pytest.approx(want_loss, rel=1e-5)
        got = dz[:B * h * w, :C].double().view(B, h, w, C)
        ratio = ((got - want_grad).abs() / (2.0 ** -12 * env + 1e-12)).max().item()
        print(f"seg xent {case[:6]}: loss rel {abs(loss.item() - want_loss) / want_loss:.1e}, worst err / bound {ratio:.3f}")
        # every gradient element is a fixed-order fp32 sum of terms w * (p - onehot) / n: its error stays within
        # 2^-12 (32 fp32 ulps) of the sum of their magnitudes (on an H100: worst ratio 0.001-0.004 for the upsampling
        # cases, 0.22 for the 64 x 48 -> 40 x 70 downsampling one; loss within 1.2e-7 relative)
        assert ratio <= 1.0
    assert (dz[:B * h * w, C:] == 0).all() and (dz[B * h * w:] == 7.0).all()
    assert torch.equal(dzb[:B * h * w], dz[:B * h * w].to(bf16))
    # two calls: the same bits
    loss2, dz2 = torch.empty(1, device="cuda"), torch.empty_like(dz)
    ops.seg_xent_fwd_bwd(L, lab, (h, w), C, loss2, count, dz_f32=dz2, Cp=Cp)
    assert torch.equal(loss2, loss) and torch.equal(dz2[:B * h * w], dz[:B * h * w])


# ------------------------------------------------------------------------------------------------ confusion
@pytest.mark.parametrize("case", [(1, 37, 50, 592, 800, 150), (4, 32, 32, 512, 512, 19), (2, 20, 30, 17, 45, 7)])
def test_seg_predict_confusion_against_float64(native, case):
    from dinov3_jax import ops
    B, h, w, Hl, Wl, C = case
    logits, labels = _xent_case(B, h, w, Hl, Wl, C, seed=11 + C)
    conf = torch.zeros(C, C, dtype=torch.int64, device="cuda")
    ops.seg_predict_confusion(logits.reshape(-1, C).cuda(), labels.cuda(), (h, w), C, conf)
    import torch.nn.functional as Fn
    up = Fn.interpolate(logits.double().cuda().permute(0, 3, 1, 2), size=(Hl, Wl), mode="bilinear", align_corners=False)
    top2 = up.topk(2, dim=1).values
    pred, gap = up.argmax(1), top2[:, 0] - top2[:, 1]
    y = labels.long().cuda()
    valid = y < C
    want = torch.bincount(y[valid] * C + pred[valid], minlength=C * C).view(C, C)
    # pixels whose two best float64 logits are within fp32 rounding of each other may go either way
    near = int(((gap < 1e-5 * (1.0 + logits.abs().max().item())) & valid).sum())
    diff = (conf - want).abs().sum().item()
    print(f"seg confusion {case}: {diff} counts differ, {near} near-tie pixels of {int(valid.sum())}")
    # on an H100: no count differed; 91 of 425 978 and 123 of 943 223 pixels were near ties
    assert diff <= 2 * near, (diff, near)
    assert near <= 1e-3 * valid.sum().item(), near
    assert conf.sum().item() == valid.sum().item()
    again = torch.zeros_like(conf)
    ops.seg_predict_confusion(logits.reshape(-1, C).cuda(), labels.cuda(), (h, w), C, again)
    assert torch.equal(again, conf)


# ------------------------------------------------------------------------------------------------ crops
def _image(H, W, rng):
    yy, xx = np.mgrid[0:H, 0:W]
    base = 127 + 100 * np.sin(xx[..., None] / 7.0 + np.arange(3)) * np.cos(yy[..., None] / 11.0)
    return np.clip(base + rng.normal(0, 40, (H, W, 3)), 0, 255).astype(np.uint8)


def _restated_crop(img, lab, box, S):
    """torchvision's uint8 bicubic antialiased resize to (rh, rw), the window at (top, left), the flip within the part
    inside the resized image, padding 0 / 255 at the bottom / right; labels by torch's 'nearest' in fp32."""
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms.v2 import functional as TF
    rh, rw, top, left, flip = box[:5]
    H, W = lab.shape
    r = TF.resize(torch.from_numpy(img).permute(2, 0, 1), [rh, rw], interpolation=InterpolationMode.BICUBIC,
                  antialias=True).permute(1, 2, 0).numpy()
    vh, vw = min(S, rh - top), min(S, rw - left)
    out = np.zeros((S, S, 3), np.uint8)
    lo = np.full((S, S), 255, np.uint8)
    win = r[top:top + vh, left:left + vw]
    ys = np.minimum(np.floor(np.arange(top, top + vh, dtype=np.float32) * np.float32(H / rh)).astype(int), H - 1)
    xs = np.minimum(np.floor(np.arange(left, left + vw, dtype=np.float32) * np.float32(W / rw)).astype(int), W - 1)
    lw = lab[ys][:, xs]
    if flip:
        win, lw = win[:, ::-1], lw[:, ::-1]
    out[:vh, :vw], lo[:vh, :vw] = win, lw
    return out, lo


def test_seg_crop_against_torchvision_and_nearest_labels(native):
    from dinov3_jax import ops
    from dinov3_jax.eval.segmentation import _pack_seg, sample_seg_boxes
    rng = np.random.default_rng(0)
    S = 64
    sizes = [(75, 100), (100, 75), (64, 64), (40, 200), (130, 90), (33, 47)]
    imgs = [_image(H, W, rng) for H, W in sizes]
    labs = [rng.integers(0, 150, (H, W)).astype(np.uint8) for H, W in sizes]
    boxes = sample_seg_boxes(torch.Generator().manual_seed(3), sizes, S).tolist()
    boxes += [[32, 40, 0, 0, 1, 0],          # smaller than the crop both ways, flipped
              [128, 90, 64, 30, 0, 0],       # a box that leaves the image on the right
              [64, 64, 0, 0, 0, 0], [200, 150, 136, 86, 1, 0], [50, 70, 0, 6, 1, 0], [64, 91, 0, 27, 0, 0]]
    imgs, labs, sizes = imgs * 2, labs * 2, sizes * 2
    flat, lab_flat, desc = _pack_seg(list(zip(imgs, labs)))
    bx = torch.tensor(boxes, dtype=torch.int32).cuda()
    taps = ops.seg_max_taps(sizes, [b[:2] for b in boxes])
    u8 = torch.empty(len(imgs), S, S, 3, dtype=torch.uint8, device="cuda")
    lo = torch.empty(len(imgs), S, S, dtype=torch.uint8, device="cuda")
    ops.seg_crop(flat.cuda(), desc.cuda(), bx, u8, max_taps=taps, labels=lab_flat.cuda(), label_out=lo)
    x = torch.empty(len(imgs), S, S, 3, dtype=bf16, device="cuda")
    ops.seg_crop(flat.cuda(), desc.cuda(), bx, x, max_taps=taps, mean=MEAN, std=STD)
    mean, std = torch.tensor(MEAN, device="cuda"), torch.tensor(STD, device="cuda")
    assert any(b[0] < S or b[1] - b[3] < S for b in boxes)
    for b, (im, lb, box) in enumerate(zip(imgs, labs, boxes)):
        want, want_lab = _restated_crop(im, lb, box, S)
        got = u8[b].cpu().numpy()
        assert np.array_equal(got, want), (sizes[b], box, (got != want).sum())
        assert np.array_equal(lo[b].cpu().numpy(), want_lab), (sizes[b], box)
        norm = (torch.from_numpy(want).cuda().float() / 255 - mean) / std
        vh, vw = min(S, box[0] - box[2]), min(S, box[1] - box[3])
        inside = torch.zeros(S, S, 1, dtype=torch.bool, device="cuda")
        inside[:vh, :vw] = True
        norm = torch.where(inside, norm, torch.zeros_like(norm))
        assert ((x[b].float() - norm).abs() <= norm.abs() * 2.0 ** -8 + 1e-6).all(), (sizes[b], box)


# ------------------------------------------------------------------------------------------------ BatchNorm
def test_bn_stats_and_normalised_rows_against_float64(native):
    from dinov3_jax import ops
    g = torch.Generator().manual_seed(0)
    M, N = 3000, 384
    x = (torch.randn(M, N, generator=g) * torch.rand(N, generator=g) * 3 + torch.randn(N, generator=g) * 40).to(bf16)
    xd = x.double()
    mean, var = torch.empty(N, device="cuda"), torch.empty(N, device="cuda")
    rm, rv = torch.full((N,), 0.5, device="cuda"), torch.full((N,), 2.0, device="cuda")
    ops.seg_bn_stats(x.cuda(), mean, var, rm, rv, momentum=0.1)
    m64, v64 = xd.mean(0), xd.var(0, unbiased=False)
    assert ((mean.double().cpu() - m64).abs() <= 1e-6 * (m64.abs() + v64.sqrt())).all()
    assert ((var.double().cpu() - v64).abs() <= 1e-5 * v64 + 1e-9).all()
    assert torch.allclose(rm.double().cpu(), 0.9 * 0.5 + 0.1 * m64, rtol=1e-5, atol=1e-5)
    assert torch.allclose(rv.double().cpu(), 0.9 * 2.0 + 0.1 * xd.var(0, unbiased=True), rtol=1e-5, atol=1e-6)
    out = torch.zeros(M + 2, N + 8, dtype=bf16, device="cuda")
    ops.seg_bn_apply(x.cuda(), mean, var, out, eps=1e-5)
    ref = (xd - m64) / (v64 + 1e-5).sqrt()
    got = out[:M, :N].double().cpu()
    assert ((got - ref).abs() <= 2.0 ** -8 * ref.abs() + 1e-4).all()
    assert (out[M:] == 0).all() and (out[:, N:] == 0).all()
    again = torch.empty(N, device="cuda")
    ops.seg_bn_stats(x.cuda(), again, torch.empty(N, device="cuda"))
    assert torch.equal(again, mean)


# ------------------------------------------------------------------------------------------------ head step
def test_head_steps_against_torch_fp32_restatement(native):
    import torch.nn.functional as Fn
    from dinov3_jax.eval.segmentation import SegLinearHead, seg_lr
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    B, h, w, K, C, S, STEPS = 4, 8, 8, 256, 19, 128, 6
    g = torch.Generator().manual_seed(0)
    centers = torch.randn(C, K, generator=g)
    head = SegLinearHead(K, C, B * h * w, 20, lr=1e-2, weight_decay=1e-2, warmup_iterations=3, seed=1, device="cuda")
    init = head.state_dict()
    bn = torch.nn.BatchNorm2d(K, affine=False, momentum=0.1).cuda()
    conv = torch.nn.Conv2d(K, C, 1).cuda()
    with torch.no_grad():
        conv.weight.copy_(init["weight"].view(C, K, 1, 1))
        conv.bias.zero_()
    opt = torch.optim.AdamW(conv.parameters(), lr=1e-2, weight_decay=1e-2)
    for t in range(STEPS):
        cls = torch.randint(0, C, (B, h, w), generator=g)
        feats = (centers[cls] + 2.0 * torch.randn(B, h, w, K, generator=g)).to(bf16)
        labels = torch.nn.functional.interpolate(cls[:, None].float(), size=(S, S), mode="nearest")[:, 0].to(torch.uint8)
        labels[:, :10] = 255
        head.step(feats.view(-1, K).cuda(), labels.cuda(), (h, w), t)
        for grp in opt.param_groups:
            grp["lr"] = seg_lr(1e-2, t, 20, 3)
        bn.train()
        z = conv(bn(feats.float().cuda().permute(0, 3, 1, 2)))
        up = Fn.interpolate(z, size=(S, S), mode="bilinear", align_corners=False)
        loss = Fn.cross_entropy(up, labels.long().cuda(), ignore_index=255)
        opt.zero_grad()
        loss.backward()
        opt.step()
        assert head.loss.item() == pytest.approx(loss.item(), rel=2e-2), t
    got = head.state_dict()
    W_ref = conv.weight.detach().view(C, K).cpu()
    err = ((got["weight"] - W_ref).norm() / W_ref.norm()).item()
    moved = ((W_ref - init["weight"]).norm() / W_ref.norm()).item()
    # bf16 x_hat, W and dZ against fp32 throughout: a few percent of the distance the weights moved
    assert err < 0.05 * moved and moved > 0.5, (err, moved)
    assert ((got["bias"] - conv.bias.detach().cpu()).norm() / conv.bias.detach().norm()).item() < 0.05
    assert torch.allclose(got["running_mean"], bn.running_mean.cpu(), rtol=1e-3, atol=1e-3)
    assert torch.allclose(got["running_var"], bn.running_var.cpu(), rtol=1e-3, atol=1e-3)


# ------------------------------------------------------------------------------------------------ end to end
def _tiny_vit_checkpoint(path, depth=4):
    from dinov3_jax.checkpointer import save_checkpoint, tree_from_flat
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=384, depth=depth, heads=6, layerscale=0.5)
    flat = init_backbone(cfg, torch.Generator().manual_seed(0))
    save_checkpoint(path, iteration=4, params={"teacher_backbone": tree_from_flat(flat)})


COLORS = ((200, 40, 40), (40, 60, 210), (30, 190, 60), (230, 230, 40))


def _region_npz(path, n, seed):
    """Images of 96 x 128 whose 32 x 32 blocks (aligned to the patch grid) are flat colours, one per class, with
    noise; a few blocks are labelled 255."""
    rng = np.random.default_rng(seed)
    H, W = 96, 128
    imgs, labs = np.zeros((n, H, W, 3), np.uint8), np.zeros((n, H, W), np.uint8)
    for i in range(n):
        for by in range(H // 32):
            for bx in range(W // 32):
                c = int(rng.integers(0, len(COLORS)))
                sl = (i, slice(32 * by, 32 * by + 32), slice(32 * bx, 32 * bx + 32))
                imgs[sl] = np.clip(np.array(COLORS[c]) + rng.normal(0, 20, (32, 32, 3)), 0, 255).astype(np.uint8)
                labs[sl] = c if rng.random() > 0.1 else 255
    np.savez(path, images=imgs, labels=labs)


def _opts(tmp_path, workers=2):
    return ["student.arch=vit_small", f"evaluation.segmentation.train_dataset_path={tmp_path / 'train.npz'}",
            f"evaluation.segmentation.val_dataset_path={tmp_path / 'val.npz'}", "evaluation.segmentation.num_classes=4",
            "evaluation.segmentation.batch_size=4", "evaluation.segmentation.crop_size=64",
            "evaluation.segmentation.iterations=60", "evaluation.segmentation.lr=0.01",
            "evaluation.segmentation.warmup_iterations=5", f"evaluation.segmentation.num_workers={workers}"]


def test_eval_only_seg_writes_results_segmentation_json(native, tmp_path):
    from dinov3_jax.train.train import main
    _tiny_vit_checkpoint(tmp_path / "weights")
    _region_npz(tmp_path / "train.npz", 24, 0)
    _region_npz(tmp_path / "val.npz", 8, 1)
    outs = []
    for run, workers in (("a", 2), ("b", 0)):
        res = main(["--eval-only", "--eval", "seg", "--eval-pretrained-weights", str(tmp_path / "weights"),
                    "--output-dir", str(tmp_path / run), "--opts"] + _opts(tmp_path, workers))
        outs.append((tmp_path / run / "eval" / "manual_5" / "results_segmentation.json").read_text())
        written = json.loads(outs[-1])
        assert written == res and sorted(written) == ["aAcc", "mAcc", "mIoU", "per_class_iou"]
        assert len(written["per_class_iou"]) == 4
        print("segmentation end to end:", {k: written[k] for k in ("mIoU", "mAcc", "aAcc")})
        # chance is 25 % accuracy and about 14 % mIoU over four equally likely classes; a first run on an H100 gave
        # mIoU 81.6, mAcc 89.8, aAcc 89.9
        assert written["mIoU"] > 60.0, written
    assert outs[0] == outs[1]                  # same seed, other worker count: the same file


def test_do_train_calls_do_seg_eval_at_the_eval_period(native, tmp_path, monkeypatch):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch, train
    calls = []
    monkeypatch.setattr(train, "do_seg_eval", lambda config, model, header: calls.append(header) or {})
    monkeypatch.setattr(train, "do_test", lambda *a: pytest.fail("no k-NN datasets are configured"))
    monkeypatch.setattr(train, "do_linear_eval", lambda *a: pytest.fail("no linear-probe datasets are configured"))
    opts = _opts(tmp_path) + ["train.batch_size_per_gpu=2", f"train.output_dir={tmp_path}", "checkpointing.period=100",
                              "evaluation.eval_period_iterations=2", "dino.head_n_prototypes=1024",
                              "ibot.head_n_prototypes=1024"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    train.do_train(config, SSLMetaArch(config), max_iters=4, print_freq=1)
    assert calls == ["training_1", "training_3"]
