"""GPU: the `gpu:` image loader (data/image_loader.py) on seeded JPEGs this script writes to its output directory.

  (a) host decode + pack throughput (images/s) of the DataLoader workers, for several num_workers, with the core count;
  (b) ragged augmentation ms/batch at B = 64 and the ViT-L crop sizes (2 x 224^2 + 8 x 96^2), for an ImageNet-like
      size mix and for a high-resolution set, beside the dense 224^2 batch of `synthetic:gpu`;
  (c) ViT-L/16 B = 64 training-loop ms/step fed by `gpu:ImageFolder` and by `synthetic:gpu`, alternated round by round
      on one engine.

Prints the card and its power limit with the numbers.  Usage: python tools/bench_loader.py [--out DIR]"""
import argparse
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dinov3-jax_b200"))
import numpy as np
import torch

from gpu_timing import card, cuda_ms_each


def write_set(root, n, kind, seed):
    """n seeded JPEGs.  imagenet: short side ~ U(300, 500), aspect in [3/4, 4/3], plus a few extreme aspects and a few
    images under 100 px; hires: long and short sides in [1500, 4000].  Smooth noise, so that the JPEGs have ImageNet-like
    file sizes rather than incompressible ones."""
    from PIL import Image
    os.makedirs(root, exist_ok=True)
    rng = np.random.default_rng(seed)
    for i in range(n):
        p = os.path.join(root, f"{i:05d}.jpg")
        if os.path.exists(p):
            continue
        if kind == "imagenet":
            if i % 50 == 7:
                h, w = (int(v) for v in rng.integers(40, 100, 2))                     # tiny
            elif i % 50 == 13:
                s = int(rng.integers(150, 300))
                h, w = (s, 4 * s) if rng.random() < 0.5 else (4 * s, s)              # extreme aspect
            else:
                s, a = rng.uniform(300, 500), rng.uniform(3 / 4, 4 / 3)
                h, w = (int(s), int(s * a)) if a >= 1 else (int(s / a), int(s))
        else:
            h, w = (int(v) for v in rng.integers(1500, 4001, 2))
        small = rng.integers(0, 256, (max(h // 8, 2), max(w // 8, 2), 3), dtype=np.uint8)
        Image.fromarray(small).resize((w, h), Image.BILINEAR).save(p, quality=90)
    return root


def host_throughput(files, B, workers, n_batches=30, warmup=5):
    from dinov3_jax.data.image_loader import ImageFiles, pack_images
    from dinov3_jax.data.synthetic import SeededBatchSampler
    dl = torch.utils.data.DataLoader(ImageFiles(files), batch_sampler=SeededBatchSampler(len(files), B, seed=0),
                                     num_workers=workers, collate_fn=pack_images, pin_memory=True)
    it = iter(dl)
    try:
        for _ in range(warmup):
            next(it)
        t0 = time.perf_counter()
        for _ in range(n_batches):
            next(it)
        return n_batches * B / (time.perf_counter() - t0)
    finally:
        getattr(it, "_shutdown_workers", lambda: None)()


def ragged_batch(files, B):
    from dinov3_jax.data.gpu_augment import RaggedImages
    from dinov3_jax.data.image_loader import decode_rgb
    return RaggedImages.from_images([torch.from_numpy(decode_rgb(f).copy()) for f in files[:B]], "cuda")


def train_config(path, out, B, workers):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    return setup_config(DinoV3SetupArgs(opts=[f"train.dataset_path={path}", f"train.batch_size_per_gpu={B}",
                                              f"train.num_workers={workers}", "student.arch=vit_large",
                                              f"train.output_dir={out}"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_loader"),
                    help="where the seeded JPEGs are written (and reused by a later run)")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--n-images", type=int, default=1024)
    ap.add_argument("--workers", default="1,2,4,8,16")
    ap.add_argument("--train-workers", type=int, default=0, help="num_workers of (c); 0: the largest of --workers "
                    "that the host's cores allow")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_loader measures on the GPU"
    from dinov3_jax.data.gpu_augment import GpuDataAugmentationDINO
    from dinov3_jax.data.image_loader import list_images
    B, cores = args.batch, os.cpu_count()
    print(card(), f"host cores: {cores}", flush=True)
    imnet = sorted(list_images(write_set(os.path.join(args.out, "imagenet_like"), args.n_images, "imagenet", 0)))
    hires = sorted(list_images(write_set(os.path.join(args.out, "hires"), B, "hires", 1)))
    from PIL import Image
    for name, fs in (("imagenet-like", imnet), ("high-resolution", hires)):
        s = np.array([Image.open(f).size for f in fs])
        print(f"set {name}: {len(fs)} JPEGs, W {s[:, 0].min()}-{s[:, 0].max()}, H {s[:, 1].min()}-{s[:, 1].max()}, "
              f"mean {s.prod(1).mean() / 1e6:.2f} MPix, {sum(os.path.getsize(f) for f in fs) / len(fs) / 1e3:.0f} kB/file",
              flush=True)

    # (a) host decode + pack
    workers = [w for w in (int(v) for v in args.workers.split(",")) if w <= max(cores, 1)]
    for w in workers:
        r = host_throughput(imnet, B, w)
        print(f"(a) decode+pack imagenet-like, num_workers={w:2d}: {r:8.0f} images/s", flush=True)

    # (b) augmentation
    aug = GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), 8, global_crops_size=224, local_crops_size=96, seed=0)
    dense = torch.randint(0, 256, (B, 224, 224, 3), device="cuda", dtype=torch.uint8)
    for name, batch in (("dense 224x224 (synthetic:gpu)", dense), ("ragged imagenet-like", ragged_batch(imnet, B)),
                        ("ragged high-resolution", ragged_batch(hires, B))):
        ts = sorted(cuda_ms_each(lambda: aug(batch), 20, 3))
        print(f"(b) augmentation B={B} {name:32s} {ts[len(ts) // 2]:8.2f} ms/batch (median of 20, min {ts[0]:.2f})",
              flush=True)
        del batch

    # (c) training loop on one ViT-L engine, alternating the two loaders
    from dinov3_jax.engine.synth import init_reference_like
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train.train import build_data_loader_from_cfg, build_schedulers
    tw = args.train_workers or max(w for w in workers)
    cfg_f = train_config(f"gpu:ImageFolder:root={os.path.join(args.out, 'imagenet_like')}", args.out, B, tw)
    cfg_s = train_config("synthetic:gpu", args.out, B, tw)
    model = SSLMetaArch(cfg_f)
    engine = model.build_engine(device="cuda:0")
    init_reference_like(engine, seed=0)
    lr_s, wd_s, mom_s, temp_s, last_s = build_schedulers(cfg_f)
    loaders = {"gpu:ImageFolder": build_data_loader_from_cfg(cfg_f, model), "synthetic:gpu": build_data_loader_from_cfg(cfg_s, model)}
    its = {k: iter(v) for k, v in loaders.items()}
    ms = {k: [] for k in loaders}
    try:
        def run(name, n):
            for _ in range(n):
                engine.train_step(next(its[name]), teacher_temp=float(temp_s[0]), lr=float(lr_s[0]), wd=float(wd_s[0]),
                                  last_layer_lr=float(last_s[0]), momentum=float(mom_s[0]))
            torch.cuda.synchronize()
        for name in loaders:                                   # warm-up: workers started, kernels loaded
            run(name, 3)
        for _ in range(args.rounds):
            for name in loaders:
                t0 = time.perf_counter()
                run(name, args.steps)
                ms[name].append((time.perf_counter() - t0) * 1e3 / args.steps)
        m = engine.read_metrics()
        assert m["total_loss"] == m["total_loss"], "NaN loss"
    finally:
        for v in its.values():
            getattr(v, "close", lambda: None)()
        loaders["gpu:ImageFolder"].close()
    for name, v in ms.items():
        print(f"(c) ViT-L/16 B={B} train step, {name:16s} (num_workers={tw}): "
              f"{' '.join(f'{x:.1f}' for x in v)} ms/step over {args.rounds} alternated rounds of {args.steps} "
              f"(median {np.median(v):.1f}, spread {min(v):.1f}-{max(v):.1f})", flush=True)


if __name__ == "__main__":
    main()
