"""GPU: keypoint correspondence (dinov3_jax/eval/correspondence.py) at the SPair-71k evaluation shape: ViT-L/16 (random
weights), 500 x 375 images resized to S = 512 (32 x 32 patches, D = 1 024), 10 keypoints per pair.

Timed apart, with CUDA events after a warm-up:
  1. feature extraction per image, in batches of 16: d3_video_resize, get_intermediate_layers(n=1), d3_knn_normalize;
  2. the match per pair: d3_corr_descriptors, d3_corr_gram of the target, the similarity GEMM (10 x 1 024 x 1 024) and
     d3_corr_argmax over the 512 x 512 pixels, together and each alone;
  3. the torch statement of the same match: F.interpolate of the target map to 512 x 512 (fp32), channel normalisation,
     the cosine with the descriptors and the argmax, on the same GPU.
Then the fraction of identical predictions of 2 and 3 over every pair of the 16 extracted images (240 pairs), and
the largest cosine gap (torch's) between the two picks where they differ.

Prints the card, its power limit and maximum SM clock with the numbers.   python tools/bench_correspondence.py [--iters N]
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import numpy as np
import torch
import torch.nn.functional as Fn

from bench_features import CONFIGS, PATCH, R, random_tree
from dinov3_jax import ops
from dinov3_jax.eval.correspondence import image_features
from dinov3_jax.models import DinoVisionTransformer
from gpu_timing import card, cuda_ms

bf16, f32 = torch.bfloat16, torch.float32
H, W, S, B, KP = 375, 500, 512, 16, 10
h = w = S // PATCH
P = h * w
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def vit_l():
    _, D, L, Hh, ffn, ratio, mkb, norm_layer = CONFIGS["vitl"]
    g = torch.Generator(device="cuda").manual_seed(0)
    return DinoVisionTransformer(random_tree(D, L, ffn, ratio, g), patch_size=PATCH, embed_dim=D, n_blocks=L,
                                 num_heads=Hh, ffn_ratio=ratio, ffn_layer=ffn, mask_k_bias=mkb, n_storage_tokens=R,
                                 norm_layer=norm_layer)


def images(rng):
    """Smooth random colour fields with noise, so that the features have structure to match."""
    out = []
    for _ in range(B):
        base = rng.random((6, 8, 3)) * 255
        im = base[np.arange(H) * 6 // H][:, np.arange(W) * 8 // W] + rng.normal(0, 25, (H, W, 3))
        out.append(np.clip(im, 0, 255).astype(np.uint8))
    return out


class Pair:
    """The buffers of one pair's match: source map 0, target map 1 of `feats`."""

    def __init__(self, feats, src, trg, kp_xy):
        D = feats.shape[1]
        self.feats, self.trg = feats, trg
        self.kp = [(src, int(x), int(y)) for x, y in kp_xy]
        self.q = torch.empty(KP, D, dtype=bf16, device="cuda")
        self.qn = torch.empty(KP, device="cuda")
        self.gram = torch.empty(P, 5, device="cuda")
        self.sim = torch.empty(KP, P, device="cuda")
        self.xy = torch.empty(KP, 2, dtype=torch.int32, device="cuda")
        self.cos = torch.empty(KP, device="cuda")
        self.n_maps = feats.shape[0] // P

    def descriptors(self):
        ops.corr_descriptors(self.feats, self.n_maps, (h, w), (S, S), self.kp, self.q, self.qn)

    def gram_(self):
        ops.corr_gram(self.feats[self.trg * P:(self.trg + 1) * P], 1, (h, w), self.gram)

    def gemm(self):
        ops.gemm(self.q, self.feats[self.trg * P:(self.trg + 1) * P], self.sim)

    def argmax(self):
        ops.corr_argmax(self.sim, self.gram, self.qn, (h, w), (S, S), self.xy, self.cos)

    def match(self):
        self.descriptors(); self.gram_(); self.gemm(); self.argmax()

    def torch_match(self):
        """F.interpolate of the target map to S x S in fp32, normalised over channels, cosine with the normalised
        descriptors, argmax: the statement the kernels replace."""
        t = self.feats[self.trg * P:(self.trg + 1) * P].float().reshape(1, h, w, -1).permute(0, 3, 1, 2)
        U = Fn.interpolate(t, size=(S, S), mode="bilinear", align_corners=False)[0].reshape(t.shape[1], -1)
        U = U / torch.linalg.vector_norm(U, dim=0, keepdim=True)
        qf = self.q.float()
        cos = (qf / torch.linalg.vector_norm(qf, dim=1, keepdim=True)) @ U
        idx = cos.argmax(1)
        return torch.stack([idx % S, idx // S], 1).to(torch.int32), cos


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    from dinov3_jax import _native
    _native.init(0)
    print(card())
    rng = np.random.default_rng(0)
    ims = images(rng)
    model = vit_l()
    with torch.no_grad():
        extract = lambda: image_features(model, ims, S, B, MEAN, STD, "cuda")
        ms = cuda_ms(extract, max(args.iters // 4, 3), 2)
        feats = extract()
    print(f"features (resize {W}x{H} -> {S}x{S}, ViT-L/16 get_intermediate_layers n=1, L2 normalise) batch {B}: "
          f"{ms:.2f} ms, {ms / B:.2f} ms per image")

    pair = Pair(feats, 0, 1, rng.integers(0, S, (KP, 2)))
    t = {name: cuda_ms(fn, args.iters, 3) for name, fn in
         (("pair", pair.match), ("descriptors", pair.descriptors), ("gram", pair.gram_), ("gemm", pair.gemm),
          ("argmax", pair.argmax), ("torch", pair.torch_match))}
    print(f"match per pair ({KP} keypoints, {h}x{w} patches -> {S}x{S} pixels, D {feats.shape[1]}): {t['pair']:.3f} ms; "
          f"d3_corr_descriptors {t['descriptors'] * 1e3:.1f} us, d3_corr_gram {t['gram'] * 1e3:.1f} us, GEMM "
          f"{t['gemm'] * 1e3:.1f} us, d3_corr_argmax {t['argmax'] * 1e3:.1f} us")
    print(f"torch statement per pair (F.interpolate to {S}x{S} fp32, normalise, cosine, argmax): {t['torch']:.3f} ms "
          f"({t['torch'] / t['pair']:.0f}x the kernels)")

    same = total = 0
    gap = 0.0
    for s in range(B):
        for d in range(B):
            if s == d:
                continue
            pr = Pair(feats, s, d, rng.integers(0, S, (KP, 2)))
            pr.match()
            xy, cos = pr.torch_match()
            eq = (pr.xy == xy).all(1)
            same += int(eq.sum())
            total += KP
            if not eq.all():                    # torch's cosine at its own pick minus at the kernels' pick
                at = cos.gather(1, (pr.xy[:, 1] * S + pr.xy[:, 0]).long()[:, None])[:, 0]
                gap = max(gap, float((cos.max(1).values - at)[~eq].max()))
    print(f"identical predictions, kernels vs torch fp32: {same} of {total} ({same / total:.4f}); where they differ, "
          f"torch's cosine at its pick exceeds its cosine at the kernels' pick by at most {gap:.2e}")
    print(card())


if __name__ == "__main__":
    main()
