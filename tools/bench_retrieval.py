"""GPU: instance retrieval (dinov3_jax/eval/retrieval.py) at revisited Oxford shapes: ViT-L/16 (random weights), a
synthetic Oxford-shaped set of 4 993 database images of 1024 x 768 and 768 x 1024 and 70 queries, image_size 512 and
scales 1, 2^-1/2, 1/2 (grids 24 x 32, 17 x 23 and 12 x 16 and their transposes).

Timed apart, with CUDA events after a warm-up:
  1. d3_ret_resize of one batch of 16 uint8 images (1024 x 768) to each scale's size, alone and with the packing and
     host-to-device copy of the images;
  2. the extraction of one batch of 16 at each scale (packing, upload, resize, ViT-L forward, class token);
  3. at N = 4 993 database descriptors (random unit bf16 vectors, D = 1 024) and 70 queries: the similarity GEMM
     (d3_gemm_bf16, fp32 out), then d3_ret_rank_ap with Oxford-like lists (per query 5-60 easy, 5-120 hard and 5-80
     junk images), whole (with its host-side list checks and upload) and its three kernels alone (torch.profiler);
  4. the same at N = 2^20 database descriptors.
The whole-set extraction time is then computed from the per-batch times (not timed as one run).

Prints the card, its power limit and maximum SM clock with the numbers.   python tools/bench_retrieval.py [--iters N]
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import numpy as np
import torch

from bench_discovery import vit_l
from bench_features import PATCH
from dinov3_jax import ops
from dinov3_jax.eval.retrieval import SCALES, csr, rank_queries, resize_batch, scaled_size
from gpu_timing import card, cuda_ms

bf16, f32 = torch.bfloat16, torch.float32
B, Q, N_OXFORD, D = 16, 70, 4993, 1024
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def oxford_lists(rng, n_db):
    sizes = {"easy": (5, 60), "hard": (5, 120), "junk": (5, 80)}
    return [[rng.choice(n_db, int(rng.integers(*sizes[k])), replace=False) for _ in range(Q)]
            for k in ("easy", "hard", "junk")]


def ranking(rng, n_db, iters):
    """ms of the similarity GEMM and of d3_ret_rank_ap for Q queries against n_db random unit descriptors."""
    q = torch.nn.functional.normalize(torch.randn(Q, D, device="cuda"), dim=1).to(bf16)
    db = torch.nn.functional.normalize(torch.randn(n_db, D, device="cuda"), dim=1).to(bf16)
    easy, hard, junk = oxford_lists(rng, n_db)
    out = rank_queries(q, db, easy, hard, junk)
    sim = out["sim"]
    lists = [csr(l) for l in (easy, hard, junk)]
    t_gemm = cuda_ms(lambda: ops.gemm(q, db, sim), iters, 2)
    t_rank = cuda_ms(lambda: ops.ret_rank_ap(sim, n_db, *lists, out["ranks"], out["ap"], out["pk"], out["n_ok"]),
                     iters, 2)
    n_listed = sum(len(l[1]) for l in lists)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            ops.ret_rank_ap(sim, n_db, *lists, out["ranks"], out["ap"], out["pk"], out["n_ok"])
        torch.cuda.synchronize()
    kernels = {e.key: getattr(e, "device_time_total", 0.0) / 1e3 / iters for e in prof.key_averages()
               if "ret_" in e.key}
    return t_gemm, t_rank, n_listed, kernels


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
    ims = [rng.integers(0, 256, (768, 1024, 3), dtype=np.uint8) for _ in range(B)]
    total_ms = 0.0
    for s, sc in enumerate(SCALES):
        out_hw = scaled_size((768, 1024), 512, sc, PATCH)
        batch = [(out_hw, i, s, (0, 0, 1024, 768)) for i in range(B)]
        t_upload = cuda_ms(lambda: resize_batch(ims, batch, MEAN, STD, "cuda"), args.iters, 2)
        flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in ims])).cuda()
        desc = [[i * ims[0].size, 768, 1024, 0, 0, 1024, 768] for i in range(B)]
        x = torch.empty(B, *out_hw, 3, dtype=bf16, device="cuda")
        t_resize = cuda_ms(lambda: ops.ret_resize(flat, desc, x, mean=MEAN, std=STD), args.iters, 2)

        def extract():
            with torch.no_grad():
                return model(resize_batch(ims, batch, MEAN, STD, "cuda"))

        t_extract = cuda_ms(extract, max(args.iters // 2, 2), 1)
        total_ms += t_extract / B * N_OXFORD
        print(f"scale {sc:.4f}: {out_hw[0]} x {out_hw[1]} ({out_hw[0] // PATCH * out_hw[1] // PATCH} patches), batch of "
              f"{B}: d3_ret_resize {t_resize:.3f} ms, {t_upload:.3f} ms with the packing and upload of the images; "
              f"extraction {t_extract:.2f} ms "
              f"({t_extract / B:.3f} ms per image)")
    print(f"extraction of {N_OXFORD} database images at the three scales, from the per-batch times: "
          f"{total_ms / 1e3:.1f} s (JPEG decoding not included)")
    for n_db in (N_OXFORD, 1 << 20):
        t_gemm, t_rank, n_listed, kernels = ranking(rng, n_db, args.iters)
        print(f"N = {n_db}, Q = {Q}, {n_listed} listed entries: similarity GEMM {t_gemm:.3f} ms; d3_ret_rank_ap "
              f"{t_rank:.3f} ms (with the list checks and upload); its kernels alone: "
              + ", ".join(f"{k.split('(')[0]} {v:.3f} ms" for k, v in kernels.items()))
    print(card())


if __name__ == "__main__":
    main()
