"""CUDA-native DINOv3 SSL training hot path behind the reference's module names (Dhia-naouali/dinov3-jax).

This package provides `dinov3_jax.{train, fsdp, layers, loss, models, checkpointer, configs, distributed}` and the
jax-free pieces of `dinov3_jax.data` (collate, masking).  It is an OVERLAY: put it first on PYTHONPATH and, if the
parts of the reference that stay (data loaders / augmentations / datasets, eval, hub, logging ...) are needed, put a
reference checkout AFTER it — sub-modules this package does not define then resolve from that checkout
(`pkgutil.extend_path`), while everything on the training hot path resolves here.  Nothing is imported from the
reference unless the user puts it on the path.
"""
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)
