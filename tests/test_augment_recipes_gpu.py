"""-m gpu: the DataAugmentationDINO options beyond the defaults on the GPU (gram-teacher crops, local crops cut from the
global crops, shared colour jitter): each new kernel against torch / torchvision's float ops with the same parameters,
both gram modes end to end against the reference's transform order (data/augmentations.py:70-230), and the batch ->
engine hand-off of the gram crops."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

pytestmark = pytest.mark.gpu

MEAN, STD = torch.tensor([0.485, 0.456, 0.406]), torch.tensor([0.229, 0.224, 0.225])


def _records(n):
    from dinov3_jax.data.gpu_augment import CROP_DTYPE
    r = np.zeros(n, dtype=CROP_DTYPE)
    r["order"] = -1
    return r


def _dev(rec):
    return torch.from_numpy(rec.view(np.uint8).reshape(-1).copy()).cuda()


def _random_jitter(rec, rng, orders):
    for i, o in enumerate(orders):
        rec["order"][i] = o
        rec["fb"][i], rec["fc"][i], rec["fs"][i], rec["fh"][i] = (rng.uniform(0.6, 1.4), rng.uniform(0.6, 1.4),
                                                                  rng.uniform(0.8, 1.2), rng.uniform(-0.1, 0.1))
        rec["gray"][i] = i % 3 == 0


def _resize(chw, S, clamp):
    """torchvision Resize(S, bicubic) of a CHW float image (antialiased bicubic; a PIL image is clamped)."""
    if chw.shape[-1] == S and chw.shape[-2] == S:
        return chw
    y = Fn.interpolate(chw[None], size=(S, S), mode="bicubic", antialias=True, align_corners=False)[0]
    return y.clamp(0, 1) if clamp else y


def _jitter(chw, rec, i):
    """RandomApply(ColorJitter) in the drawn order + RandomGrayscale, torchvision float ops."""
    from torchvision.transforms.v2 import functional as F
    if rec["order"][i][0] >= 0:
        for op in rec["order"][i]:
            chw = (F.adjust_brightness(chw, float(rec["fb"][i])) if op == 0 else
                   F.adjust_contrast(chw, float(rec["fc"][i])) if op == 1 else
                   F.adjust_saturation(chw, float(rec["fs"][i])) if op == 2 else F.adjust_hue(chw, float(rec["fh"][i])))
    if rec["gray"][i]:
        chw = F.rgb_to_grayscale(chw, num_output_channels=3)
    return chw


def _blur(chw, sigma):
    from torchvision.transforms.v2 import functional as F
    return chw if sigma <= 0 else F.gaussian_blur(chw, kernel_size=[9, 9], sigma=[float(sigma)] * 2)


def _solarize(chw, on):
    return torch.where(chw >= 128 / 255, 1 - chw, chw) if on else chw


def _normalize(chw):
    return (chw - MEAN[:, None, None]) / STD[:, None, None]


def _base(img_u8, rec, i, M):
    """RandomResizedCrop(M, bicubic) + flip of record i, as a CHW float image."""
    x0, y0, w, h = (int(rec[k][i]) for k in ("x0", "y0", "w", "h"))
    crop = img_u8[y0:y0 + h, x0:x0 + w].permute(2, 0, 1).float() / 255.0
    out = _resize(crop, M, True) if (w, h) != (M, M) else crop
    return out.flip(-1) if rec["flip"][i] else out


def _close_bf16(got, ref_chw, what):
    """bf16 output [S,S,3] against an fp32 CHW reference rounded to bf16: at most one bf16 ulp of the normalised range
    where the fp32 arithmetic rounds differently, and rarely."""
    ref = ref_chw.permute(1, 2, 0).to(torch.bfloat16).float()
    err = (got.float().cpu() - ref).abs()
    assert float(err.max()) < 3e-2 and float(err.mean()) < 1e-3, (what, float(err.max()), float(err.mean()))


@pytest.mark.parametrize("clamp", [1, 0])
def test_float_source_resized_crop_and_resize(clamp):
    """d3_aug_resized_crop_f32: crops of a float source, and Resize of a whole base (full box) down and up, with the
    clamp of a PIL image (1) or without it, as after Normalize (0)."""
    from dinov3_jax import _native as N
    lib = N.init()
    g = torch.Generator().manual_seed(4)
    imgs = torch.rand(3, 150, 210, 3, generator=g) if clamp else torch.randn(3, 150, 210, 3, generator=g)
    boxes = [(0, 10, 20, 120, 100, 0), (1, 0, 0, 210, 150, 1), (2, 50, 40, 30, 24, 0), (1, 100, 30, 97, 119, 1)]
    rec = _records(len(boxes))
    for i, (img, x0, y0, w, h, flip) in enumerate(boxes):
        rec["img"][i], rec["x0"][i], rec["y0"][i], rec["w"][i], rec["h"][i], rec["flip"][i] = img, x0, y0, w, h, flip
    d_rec, src = _dev(rec), imgs.cuda()          # held: a temporary's memory could be reused before the kernel runs
    for S in (64, 32):
        out = torch.empty(len(boxes), S, S, 3, device="cuda")
        N.check(lib.d3_aug_resized_crop_f32(N.ptr(src), 3, 150, 210, N.ptr(d_rec), len(boxes), N.ptr(out), S,
                                            clamp, N.stream_ptr()), "crop_f32")
        for i, (img, x0, y0, w, h, flip) in enumerate(boxes):
            ref = _resize(imgs[img, y0:y0 + h, x0:x0 + w].permute(2, 0, 1), S, clamp).permute(1, 2, 0)
            ref = ref.flip(1) if flip else ref
            assert float((out[i].cpu() - ref).abs().max()) < 2e-3, (S, i)
    # base -> global / gram: the whole [M, M] base, down- and up-sampled
    for M, S in ((96, 64), (64, 96), (112, 48)):
        base = torch.rand(2, M, M, 3, generator=g) if clamp else torch.randn(2, M, M, 3, generator=g)
        whole = _records(2)
        whole["img"], whole["w"], whole["h"] = [0, 1], M, M
        out = torch.empty(2, S, S, 3, device="cuda")
        d_base, d_whole = base.cuda(), _dev(whole)
        N.check(lib.d3_aug_resized_crop_f32(N.ptr(d_base), 2, M, M, N.ptr(d_whole), 2, N.ptr(out), S, clamp,
                                            N.stream_ptr()), "resize_f32")
        for i in range(2):
            ref = _resize(base[i].permute(2, 0, 1), S, clamp).permute(1, 2, 0)
            assert float((out[i].cpu() - ref).abs().max()) < 2e-3, (M, S, i)


def test_whole_image_jitter_on_non_square_sources():
    """d3_aug_color_images (share_color_jitter): ColorJitter in the drawn order + RandomGrayscale of whole H x W uint8
    images into an fp32 copy, against torchvision on the float image."""
    import itertools
    from dinov3_jax import _native as N
    lib = N.init()
    orders = list(itertools.permutations(range(4)))[::4] + [(-1, -1, -1, -1)]
    n, H, W = len(orders), 37, 53
    g = torch.Generator().manual_seed(5)
    imgs = torch.randint(0, 256, (n, H, W, 3), generator=g, dtype=torch.uint8)
    rec = _records(n)
    rec["img"] = np.arange(n)
    _random_jitter(rec, np.random.default_rng(1), orders)
    x = torch.empty(n, H, W, 3, device="cuda")
    gsum = torch.zeros(n, device="cuda")
    src, d_rec = imgs.cuda(), _dev(rec)
    N.check(lib.d3_aug_color_images(N.ptr(src), n, H, W, N.ptr(d_rec), N.ptr(x), N.ptr(gsum), N.stream_ptr()),
            "color_images")
    for i in range(n):
        ref = _jitter(imgs[i].permute(2, 0, 1).float() / 255.0, rec, i).permute(1, 2, 0)
        assert float((x[i].cpu() - ref).abs().max()) < 2e-5, (i, orders[i])


def test_local_windows_match_transform_then_slice():
    """d3_aug_local_windows (local_crops_subset_of_global_crops): each window equals jitter + grayscale + blur of the
    WHOLE base followed by the slice, at offsets 0 and the largest one (the blur's halo reflects at the base border)."""
    from dinov3_jax.data.gpu_augment import GpuDataAugmentationDINO
    M, L = 80, 32
    aug = GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), 2, global_crops_size=M, local_crops_size=L,
                                  local_crops_subset_of_global_crops=True, patch_size=16)
    g = torch.Generator().manual_seed(6)
    base = torch.rand(2, M, M, 3, generator=g)
    offs = [(0, 0), (M - L, M - L), (0, M - L), (M - L, 16), (16, 0), (32, 48)]
    orders = [(1, 0, 2, 3), (3, 2, 1, 0), (0, 1, 2, 3), (-1, -1, -1, -1), (2, 3, 0, 1), (1, 3, 2, 0)]
    sig = np.array([2.0, 1.3, 0.0, 0.7, 0.4, 1.9], dtype=np.float32)
    rec = _records(len(offs))
    _random_jitter(rec, np.random.default_rng(2), orders)
    for i, (ry, rx) in enumerate(offs):
        rec["img"][i], rec["y0"][i], rec["x0"][i], rec["w"][i], rec["h"][i] = i % 2, ry, rx, L, L
    got = aug.local_windows(base.cuda(), rec, sig)
    for i, (ry, rx) in enumerate(offs):
        whole = _blur(_jitter(base[i % 2].permute(2, 0, 1), rec, i), sig[i])
        _close_bf16(got[i], _normalize(whole[:, ry:ry + L, rx:rx + L]), ("window", i))


def _aug_pair(**kw):
    """Two augmenters with the same seed: one draws the records the test replays, the other runs the kernels."""
    from dinov3_jax.data.gpu_augment import GpuDataAugmentationDINO
    make = lambda: GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), 4, global_crops_size=64, local_crops_size=32,
                                           patch_size=16, seed=11, **kw)
    return make(), make()


def _images(B, H=120, W=150, seed=7):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)


@pytest.mark.parametrize("gram", [96, 48])
@pytest.mark.parametrize("no_distortions", [True, False])
def test_gram_crops_end_to_end(gram, no_distortions):
    """Global and gram crops against a torchvision composition of the reference's order: base at max(global, gram);
    no distortions: Resize(global) before jitter / blur / solarize, gram = Normalize(Resize(gram)(base)); otherwise the
    distortions and Normalize run on the base and both crops are Resize of the normalised tensor."""
    probe, aug = _aug_pair(gram_teacher_crops_size=gram, gram_teacher_no_distortions=no_distortions)
    B = 3
    imgs = _images(B)
    (g, gb), _ = probe.sample(B, imgs.shape[1], imgs.shape[2])
    out = aug(imgs.cuda())
    M = max(64, gram)
    assert out["collated_global_crops"].shape == (2 * B, 64, 64, 3)
    assert out["collated_gram_teacher_crops"].shape == (2 * B, gram, gram, 3)
    assert out["collated_gram_teacher_crops"].dtype == torch.bfloat16
    for i in range(2 * B):
        base = _base(imgs[int(g["img"][i])], g, i, M)
        if no_distortions:
            glob = _normalize(_solarize(_blur(_jitter(_resize(base, 64, True), g, i), gb[i]), g["solarize"][i]))
            gr = _normalize(_resize(base, gram, True))
        else:
            y = _normalize(_solarize(_blur(_jitter(base, g, i), gb[i]), g["solarize"][i]))
            glob, gr = _resize(y, 64, False), _resize(y, gram, False)
        _close_bf16(out["collated_global_crops"][i], glob, ("global", i))
        _close_bf16(out["collated_gram_teacher_crops"][i], gr, ("gram", i))


def test_shared_jitter_and_subset_locals_end_to_end():
    """share_color_jitter + local_crops_subset_of_global_crops through __call__: every crop comes from the jittered
    source, and local crop c of image b is the window of base 1 (c < n/2) or 2 after its blur."""
    probe, aug = _aug_pair(share_color_jitter=True, local_crops_subset_of_global_crops=True)
    B = 2
    imgs = _images(B, 100, 90)
    src_rec = probe.sample_source_jitter(B)
    (g, gb), (l, lb) = probe.sample(B, 100, 90)
    out = aug(imgs.cuda())
    src = [_jitter(imgs[b].permute(2, 0, 1).float() / 255.0, src_rec, b) for b in range(B)]
    bases = []
    for i in range(2 * B):
        x0, y0, w, h = (int(g[k][i]) for k in ("x0", "y0", "w", "h"))
        base = _resize(src[int(g["img"][i])][:, y0:y0 + h, x0:x0 + w], 64, True)
        bases.append(base.flip(-1) if g["flip"][i] else base)
        _close_bf16(out["collated_global_crops"][i], _normalize(_solarize(_blur(bases[i], gb[i]), g["solarize"][i])),
                    ("global", i))
    assert out["collated_local_crops"].shape == (4 * B, 32, 32, 3)
    for i in range(4 * B):
        c, b = divmod(i, B)
        assert int(l["img"][i]) == (0 if c < 2 else B) + b
        ry, rx = int(l["y0"][i]), int(l["x0"][i])
        whole = _blur(bases[int(l["img"][i])], lb[i])
        _close_bf16(out["collated_local_crops"][i], _normalize(whole[:, ry:ry + 32, rx:rx + 32]), ("local", i))


def _gram_opts():
    return ["train.batch_size_per_gpu=4", "student.arch=vit_small", "crops.global_crops_size=64", "crops.local_crops_size=32",
            "crops.gram_teacher_crops_size=96", "crops.gram_teacher_no_distortions=true", "gram.use_loss=true",
            "gram.it_load_ema_teacher=0", "dino.head_n_prototypes=512", "ibot.head_n_prototypes=512",
            "dino.head_hidden_dim=256", "ibot.head_hidden_dim=256", "dino.head_bottleneck_dim=64",
            "ibot.head_bottleneck_dim=64"]


def test_gpu_batch_pipeline_feeds_the_gram_teacher():
    """GpuBatchPipeline with crops.gram_teacher_crops_size != global: `collated_gram_teacher_crops` [2B, 96, 96, 3] bf16,
    image b's crops at rows b and B + b, each the undistorted base of the matching global record; then a train step
    with a frozen gram teacher (snapshot of the EMA teacher at iteration 0) gives a finite, non-zero gram loss."""
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.data.gpu_augment import GpuBatchPipeline
    from dinov3_jax.engine.synth import init_reference_like
    from dinov3_jax.train.ssl_meta_arch import SSLMetaArch
    config = setup_config(DinoV3SetupArgs(opts=_gram_opts()))
    pipe = GpuBatchPipeline(config, seed=3)
    B = 4
    imgs = _images(B, 224, 224, seed=8)
    probe = copy.copy(pipe.aug)
    probe.rng = copy.deepcopy(pipe.aug.rng)
    (g, _), _ = probe.sample(B, 224, 224)
    batch = pipe(imgs.cuda())
    gc = batch["collated_gram_teacher_crops"]
    assert gc.shape == (2 * B, 96, 96, 3) and gc.dtype == torch.bfloat16
    assert batch["collated_global_crops"].shape == (2 * B, 64, 64, 3)
    for b in range(B):
        for i in (b, B + b):
            assert int(g["img"][i]) == b
            _close_bf16(gc[i], _normalize(_base(imgs[b], g, i, 96)), ("gram", i))
    model = SSLMetaArch(config)
    eng = model.build_engine(max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    init_reference_like(eng, seed=0)
    eng.train_step(batch, teacher_temp=0.05, lr=1e-3, wd=0.04, last_layer_lr=5e-4, momentum=0.99)
    m = eng.read_metrics()
    assert np.isfinite(m["gram_loss"]) and m["gram_loss"] > 0, m
    assert np.isfinite(m["total_loss"])


def test_do_train_feeds_gram_crops_from_the_gpu_pipeline(tmp_path):
    """train.dataset_path=synthetic:gpu with a gram teacher at 96^2: the on-GPU augmentation feeds the gram stream."""
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train.train import do_train
    opts = [o for o in _gram_opts() if not o.startswith("train.batch_size")] + [
        "train.dataset_path=synthetic:gpu", "train.batch_size_per_gpu=2", "optim.epochs=1", "train.OFFICIAL_EPOCH_LENGTH=4",
        "optim.warmup_epochs=0", "teacher.warmup_teacher_temp_epochs=0", "optim.freeze_last_layer_epochs=0",
        f"train.output_dir={tmp_path}", "checkpointing.period=100"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    m = do_train(config, SSLMetaArch(config), resume=False, max_iters=3, print_freq=1)
    assert m["total_loss"] == m["total_loss"] and m["total_loss"] > 0
    assert np.isfinite(m["gram_loss"]) and m["gram_loss"] > 0
