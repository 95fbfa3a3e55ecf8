"""Generates tests/golden/loader_batch.npz: ONE batch produced by the reference's own host data path
(`dinov3_jax/data/augmentations.py::DataAugmentationDINO` executed from a reference checkout through the package overlay,
on the noise images of the reference's decoder, data/datasets/decoders.py:31-34) and collated by this repo's
`collate_data_and_cast` (pinned bit-exactly against the reference function in test_golden_reference.py).
Usage:  DINOV3_JAX_REFERENCE=<checkout of Dhia-naouali/dinov3-jax> python tests/golden/make_loader_fixture.py
"""
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200"))
REF_ROOT = os.path.abspath(os.environ.get("DINOV3_JAX_REFERENCE", "dinov3-jax-reference"))
sys.path.append(REF_ROOT)          # AFTER the package: only what the overlay does not define resolves there

from dinov3_jax.configs import DinoV3SetupArgs, setup_config  # noqa: E402
from dinov3_jax.train.ssl_meta_arch import SSLMetaArch  # noqa: E402
from dinov3_jax.train.train import build_data_loader_from_cfg  # noqa: E402

OPTS = ["train.dataset_path=synthetic:noise", "train.batch_size_per_gpu=2", "student.arch=vit_small",
        "crops.global_crops_size=64", "crops.local_crops_size=32", "dino.head_n_prototypes=512",
        "ibot.head_n_prototypes=512", "dino.head_hidden_dim=256", "ibot.head_hidden_dim=256",
        "dino.head_bottleneck_dim=64", "ibot.head_bottleneck_dim=64", "train.seed=7"]


def make():
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    config = setup_config(DinoV3SetupArgs(opts=OPTS))
    model = SSLMetaArch(config)
    import dinov3_jax.data.augmentations as aug
    assert aug.__file__.startswith(REF_ROOT + os.sep), aug.__file__
    loader = build_data_loader_from_cfg(config, model, start_iter=0)
    return next(iter(loader))


if __name__ == "__main__":
    b = make()
    out = {}
    for k, v in b.items():
        if torch.is_tensor(v):
            out[k] = v.view(torch.int16).numpy() if v.dtype == torch.bfloat16 else v.numpy()
        else:
            out[k] = np.asarray(v)
    p = os.path.join(os.path.dirname(os.path.abspath(__file__)), "loader_batch.npz")
    np.savez_compressed(p, **out)
    print({k: (v.shape, v.dtype) for k, v in out.items()}, os.path.getsize(p))
