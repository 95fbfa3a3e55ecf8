"""GPU: unsupervised object discovery (dinov3_jax/eval/discovery.py) at PASCAL VOC shapes: ViT-L/16 (random weights),
batches of B = 16 images of 375 x 500 (a 24 x 32 grid, N = 768) and of 500 x 500 (32 x 32, N = 1 024), each a textured
background with one bright rectangle.

Timed apart, with CUDA events after a warm-up, per image:
  1. feature extraction in batches of 16: normalisation and padding, get_intermediate_layers(n=1), d3_knn_normalize;
  2. the similarity GEMMs (d3_gemm_bf16, fp32 out) and d3_od_graph;
  3. d3_od_fiedler, with its mean Lanczos step count and the unconverged images;
  4. d3_od_box.
Random weights make every patch similar to every other: at tau = 0.2 the graph is complete and the cut trivial (the
density is printed).  So the timed graphs use tau = the batch's median similarity, which puts half the pairs above it
and gives Lanczos real work; the protocol's tau is 0.2.
Baselines on the same graphs: torch.linalg.eigh (cuSOLVER) of M = D^-1/2 A D^-1/2 on the GPU, batched, in float32 and
in float64; scipy.linalg.eigh(D - A, D, subset_by_index=[1, 1]) on the host.  Then how often the kernels' box equals
the box of each cuSOLVER eigenvector (through the same d3_od_box).

Prints the card, its power limit and maximum SM clock with the numbers.   python tools/bench_discovery.py [--iters N]
"""
import argparse
import os
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import numpy as np
import scipy.linalg
import torch

from bench_features import CONFIGS, PATCH, R, random_tree
from dinov3_jax import ops
from dinov3_jax.eval.discovery import boxes_of, image_features, normalized_cut
from dinov3_jax.models import DinoVisionTransformer
from gpu_timing import card, cuda_ms

bf16, f32 = torch.bfloat16, torch.float32
B, TAU, EPS = 16, 0.2, 1e-5
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
SIZES = [(375, 500), (500, 500)]


def vit_l():
    _, D, L, Hh, ffn, ratio, mkb, norm_layer = CONFIGS["vitl"]
    g = torch.Generator(device="cuda").manual_seed(0)
    return DinoVisionTransformer(random_tree(D, L, ffn, ratio, g), patch_size=PATCH, embed_dim=D, n_blocks=L,
                                 num_heads=Hh, ffn_ratio=ratio, ffn_layer=ffn, mask_k_bias=mkb, n_storage_tokens=R,
                                 norm_layer=norm_layer)


def scenes(rng, H, W):
    out = []
    for _ in range(B):
        im = rng.normal(90, 30, (H, W, 3))
        y0, x0 = int(rng.integers(0, H // 2)), int(rng.integers(0, W // 2))
        im[y0:y0 + H // 3, x0:x0 + W // 3] = rng.random(3) * 120 + 130
        out.append(np.clip(im, 0, 255).astype(np.uint8))
    return out


def dense_graph(bits, P):
    """fp64 A [n, P, P] on the device from the bit matrix."""
    shifts = torch.arange(32, device=bits.device, dtype=torch.int64)
    b = (bits.to(torch.int64)[..., None] >> shifts) & 1
    on = b.reshape(bits.shape[0], P, -1)[:, :, :P].bool()
    return torch.where(on, 1.0, EPS).double()


def _density(bits, P):
    return float(sum(bin(v & 0xffffffff).count("1") for v in bits.cpu().reshape(-1).tolist())) / (bits.shape[0] * P * P)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    from dinov3_jax import _native
    _native.init(0)
    print(card())
    rng = np.random.default_rng(0)
    model = vit_l()
    for H, W in SIZES:
        h, w = -(-H // PATCH), -(-W // PATCH)
        P = h * w
        ims = scenes(rng, H, W)
        with torch.no_grad():
            extract = lambda: image_features(model, ims, MEAN, STD, "cuda")
            t_feat = cuda_ms(extract, max(args.iters // 2, 2), 1)
            feats = extract()
        n, D = feats.shape[0], feats.shape[2]
        cut = normalized_cut(feats, TAU, EPS)
        dense = _density(cut["bits"], P)
        tau = float(cut["sim"].float().quantile(0.5) if P * P * n <= 2 ** 24 else
                    cut["sim"].reshape(-1)[::7].float().quantile(0.5))
        cut = normalized_cut(feats, tau, EPS)
        sim = cut["sim"]
        bits, degree = cut["bits"], cut["degree"]
        x, lam, iters, conv = cut["x"], cut["lambda2"], cut["iters"], cut["converged"]

        def graph():
            for m in range(n):
                ops.gemm(feats[m], feats[m], sim[m])
            ops.od_graph(sim, tau, EPS, bits, degree)

        sizes, gts = [(H, W)] * n, [np.array([[0.0, 0.0, W / 3, H / 3]])] * n
        t_graph = cuda_ms(graph, args.iters, 2)
        t_fied = cuda_ms(lambda: ops.od_fiedler(bits, degree, EPS, x, lam, iters, conv), args.iters, 2)
        t_box = cuda_ms(lambda: boxes_of(x, (h, w), PATCH, sizes, gts), args.iters, 2)
        it = iters.cpu().numpy()
        print(f"{H}x{W}: graph density at tau {TAU}: {dense:.4f}; timed at the median similarity tau {tau:.4f} "
              f"(density {_density(bits, P):.4f})")
        print(f"{H}x{W} (grid {h}x{w}, N {P}, D {D}), B {n}, per image: features {t_feat / n:.3f} ms; GEMM + "
              f"d3_od_graph {t_graph / n * 1e3:.1f} us; d3_od_fiedler {t_fied / n * 1e3:.1f} us ({t_fied:.3f} ms per "
              f"batch, one CTA per image; Lanczos steps mean {it.mean():.1f}, min {it.min()}, max {it.max()}, "
              f"{int((conv == 0).sum())} unconverged); d3_od_box {t_box / n * 1e3:.1f} us (with the host-side "
              f"ground-truth upload)")

        A = dense_graph(bits, P)
        d = A.sum(2)
        ds = d.rsqrt()
        M64 = ds[:, :, None] * A * ds[:, None, :]
        M32 = M64.float()
        t64 = cuda_ms(lambda: torch.linalg.eigh(M64), 2, 1)
        t32 = cuda_ms(lambda: torch.linalg.eigh(M32), 2, 1)
        An, dn = A.cpu().numpy(), d.cpu().numpy()
        k = min(n, 4)
        t0 = time.perf_counter()
        for m in range(k):
            scipy.linalg.eigh(np.diag(dn[m]) - An[m], np.diag(dn[m]), subset_by_index=[1, 1])
        t_host = (time.perf_counter() - t0) / k * 1e3
        print(f"  baselines per image: torch.linalg.eigh (cuSOLVER) of M float32 {t32 / n:.3f} ms, float64 "
              f"{t64 / n:.3f} ms ({n} batched); scipy.linalg.eigh(D - A, D, subset_by_index=[1, 1]) on the host "
              f"{t_host:.1f} ms (mean of {k})")
        ours = boxes_of(x, (h, w), PATCH, sizes, gts)["box"].cpu()
        for name, M in (("float32", M32), ("float64", M64)):
            _, Y = torch.linalg.eigh(M)
            xr = (Y[:, :, -2] * ds.to(Y.dtype)).float().contiguous()
            theirs = boxes_of(xr, (h, w), PATCH, sizes, gts)["box"].cpu()
            same = int((ours == theirs).all(1).sum())
            lam_err = float((lam.double() - (1 - torch.linalg.eigvalsh(M64)[:, -2])).abs().max())
            print(f"  same box as cuSOLVER {name}: {same} of {n}; max |lambda2 - cuSOLVER float64| {lam_err:.1e}")
    print(card())


if __name__ == "__main__":
    main()
