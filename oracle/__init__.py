"""CPU oracle for the DINOv3 SSL training hot path — TEST INFRASTRUCTURE ONLY.

This package is a plain-PyTorch (fp32 / fp64, CPU) restatement of the arithmetic of the reference
Dhia-naouali/dinov3-jax @ 27e64762 for the path BASELINE.json names: student/teacher ViT forward, DINO / iBOT /
KoLeo heads and losses, gradient, per-submodule clip, AdamW and teacher EMA.  Every function cites the reference
file:line it follows (paths relative to the reference checkout, `dinov3_jax/...`).

Who may import it: only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` / `--impl reference`
legs, and there only as the checker (or the timed CPU baseline) — never from the product path under
`dinov3-jax_b200/`.  The product path has no CPU fallback and fails loudly without the CUDA library.

PARITY STATUS: the reference ships no golden vectors, known-answer tests or numeric asserts (SURVEY.md §4, §8c) and
its third-party stack (jax 0.7.1 / flax 0.11.2 / optax 0.2.5) is not installable in the build container, so the
reference cannot be executed end to end here.  The oracle is pinned as far as that allows:
  * `data/masking.py`, `data/collate.py` (mask part), `train/cosine_lr_scheduler.py` are pure numpy/torch and ARE
    imported from a reference checkout by `tests/golden/make_golden.py`; the oracle's restatement is bit-exact against them;
  * the loss / RoPE / param-group files and the whole model side — `models/vision_transformer.py`
    (DinoVisionTransformer on multi-crop input with iBOT masks) with every layer under it (patch_embed, block,
    attention, ffn_layers, layer_scale, rope) and `layers/dino_head.py` — are executed *unmodified* under a small
    numpy-backed shim of the jax / flax API (`oracle/jaxshim`: mini flax.linen Module tree + parameter naming,
    semantics of the third-party ops restated per SURVEY.md Appendix F); outputs are committed as fixtures under
    `tests/golden/` and the oracle matches them to 1e-11 in float64;
  * `train/ssl_meta_arch.py` SSLMetaArch.setup + __call__ (the forward of the training step: teacher / student passes,
    heads, iBOT gathers, Sinkhorns, loss weights, metrics) runs unmodified under the same shim on the reference's
    default YAML; `oracle.step.ssl_forward` matches its loss and metrics to 1e-9 (the oracle's gradients are torch
    autograd of that function);
  * `build_schedulers` and the gradient-clipping block of `train_step` (train/train.py:124-182,516-541) are exec'ed from
    their source text; the schedules are reproduced bit-exactly, the clipping to 1e-12;
  * the ViT forward is cross-checked against an independent implementation of upstream DINOv3 (Hugging Face
    transformers' DINOv3ViTModel) to 2e-6 — RoPE, attention, LayerScale, token order, register tokens, mask token;
  * analytic micro-cases (uniform Sinkhorn, LN of constant rows, orthogonal KoLeo pairs ...) in `tests/`, and the AdamW
    rule against torch.optim.AdamW.
What is therefore *not* pinned: the third-party op semantics themselves (flax gelu/LayerNorm/attention defaults,
optax adamw), the optax.multi_transform wiring / update application of train/train.py (imports optax), and the call path
of the Gram-anchoring term (train/ssl_meta_arch.py:337-347 does not execute in the reference; loss/gram_loss.py itself is
pinned through tests/golden) — "parity unpinned" for those, stated here and in DESIGN.md.
"""
from .arch import ARCHS, ModelCfg, tiny_cfg, cfg_for  # noqa: F401
