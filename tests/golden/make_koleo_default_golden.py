"""Writes koleo_default_step.npz: the metrics and the sha256 of every gradient and updated parameter of one default
training step (KoLeo per rank, no local-loss weight) of the tiny oracle configuration on one H100.

The committed file was written by the library of the commit before the distributed KoLeo and the local-loss weight
went in, so tests/test_koleo_gpu.py pins that a default engine computes the same bits as before them.

    python tests/golden/make_koleo_default_golden.py --tree <repository root to import from> --out <file.npz>
"""
import argparse
import hashlib
import os
import sys

import numpy as np

HYPER = dict(lr=1e-3, wd=0.04, last_layer_lr=5e-4, momentum=0.99, teacher_temp=0.05)
METRICS = ("dino_local_crops_loss", "dino_local_loss_weight", "dino_global_crops_loss", "koleo_loss", "ibot_loss",
           "total_loss")


def step_digest():
    """(metric names, values, tensor names, sha256 hex digests) of one default step, B = 8."""
    import torch
    from dinov3_jax import _native
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    _native.init(0)
    cfg = tiny_cfg()
    B = 8
    batch = synthetic_batch(cfg, B, 0)
    eng = Engine(from_oracle_cfg(cfg), B, max_masked=max(int(batch["mask_indices_list"].shape[0]), 1))
    eng.params.load_reference_tree(init_params(cfg, 0, perturb=0.05))
    eng.set_batch(batch)
    eng.forward_backward(HYPER["teacher_temp"])
    grads = {f"grad/{k}": v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
    eng.optimizer_step(HYPER["lr"], HYPER["wd"], HYPER["last_layer_lr"], HYPER["momentum"])
    torch.cuda.synchronize()
    met = eng.read_metrics()
    params = {f"param/{k}": v.cpu() for k, v in eng.params.export_reference_tree("param").items()}
    tensors = {**grads, **params}
    names = sorted(tensors)
    digests = [hashlib.sha256(tensors[n].contiguous().numpy().tobytes()).hexdigest() for n in names]
    return list(METRICS), [float(met[m]) for m in METRICS], names, digests


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--tree", required=True)
    p.add_argument("--out", required=True)
    a = p.parse_args()
    tree = os.path.abspath(a.tree)
    sys.path[:0] = [os.path.join(tree, "dinov3-jax_b200"), tree]
    mnames, mvals, names, digests = step_digest()
    np.savez(a.out, metric_names=np.array(mnames), metrics=np.array(mvals, dtype=np.float64),
             tensor_names=np.array(names), sha256=np.array(digests))
    print(f"wrote {a.out}: {len(names)} tensors, total_loss {mvals[-1]!r}")


if __name__ == "__main__":
    main()
