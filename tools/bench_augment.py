"""GPU: milliseconds per batch of the on-GPU DINO augmentation (data/gpu_augment.py: host parameter draws + kernels, CUDA
events around each call), for the default options at the ViT-L sizes, each further DataAugmentationDINO option at those
sizes, and the 7B gram-anchoring recipe's sizes (dinov3_vit7b16_gram_anchor.yaml).  Prints the card and its power limit
with the numbers."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dinov3-jax_b200"))
import torch

from dinov3_jax.data.gpu_augment import GpuDataAugmentationDINO
from gpu_timing import card, cuda_ms_each

VITL = dict(global_crops_size=224, local_crops_size=96)
CASES = [   # name, images per batch, source H x W, options
    ("default (2 x 224^2 + 8 x 96^2)", 64, (224, 224), {}),
    ("gram 256, no distortions", 64, (224, 224), dict(gram_teacher_crops_size=256, gram_teacher_no_distortions=True)),
    ("gram 256, with distortions", 64, (224, 224), dict(gram_teacher_crops_size=256)),
    ("local crops subset of global crops", 64, (224, 224), dict(local_crops_subset_of_global_crops=True)),
    ("share colour jitter", 64, (224, 224), dict(share_color_jitter=True)),
    ("teacher_no_color_jitter", 64, (224, 224), dict(teacher_no_color_jitter=True)),
    ("7B gram recipe (2 x 256^2 + 8 x 112^2, gram 512^2, no distortions, no flips)", 16, (512, 512),
     dict(global_crops_size=256, local_crops_size=112, gram_teacher_crops_size=512, gram_teacher_no_distortions=True,
          horizontal_flips=False)),
]


def main(iters: int = 20, warmup: int = 3):
    assert torch.cuda.is_available(), "bench_augment measures on the GPU"
    print(card())
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, B, (H, W), opts in CASES:
        kw = dict(VITL)
        kw.update(opts)
        aug = GpuDataAugmentationDINO((0.32, 1.0), (0.05, 0.32), 8, seed=0, **kw)
        imgs = torch.randint(0, 256, (B, H, W, 3), generator=g, device="cuda", dtype=torch.uint8)
        ts = sorted(cuda_ms_each(lambda: aug(imgs), iters, warmup))
        print(f"  B={B:3d} src {H}x{W}  {name:78s} {ts[len(ts) // 2]:8.2f} ms/batch (median of {iters}, "
              f"min {ts[0]:.2f})")


if __name__ == "__main__":
    main()
