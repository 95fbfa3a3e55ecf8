"""GPU: the k-NN evaluation at the ImageNet-1k shape (dinov3_jax/eval/knn.py).

  * search and vote: Q = 50 000 queries against N = 1 281 167 bank rows, D = 1024, k = 200, C = 1 000, on seeded
    clustered unit features.  The similarity GEMM (d3_gemm_bf16) and the top-k merge (d3_topk_merge) are timed apart with
    CUDA events around every call (after a warm-up pass), the vote (d3_knn_vote) on its own.  A torch baseline runs
    torch.mm (bf16, cuBLAS) and torch.topk on the same chunks; its neighbour lists (torch.topk over the library's fp32
    similarities, merged chunk by chunk) are compared with the library's: the fraction of identical lists and the
    difference in top-1 accuracy of the upstream vote;
  * the eval transform (d3_eval_resize_crop): images/s for 500 x 375 sources -> 224^2 crops, batches of 256;
  * ViT-L/16 class-token extraction (DinoVisionTransformer, random weights), batches of 256 at 224^2.

Prints the card and its power limit with the numbers.   python tools/bench_knn.py [--queries Q] [--bank N]
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import torch

from dinov3_jax import ops
from dinov3_jax.eval import KnnClassifier
from gpu_timing import card, cuda_ms

bf16, f32 = torch.bfloat16, torch.float32


def clustered(n, centers, g, spread=4.0):
    y = torch.randint(0, centers.shape[0], (n,), device="cuda", generator=g)
    x = torch.empty(n, centers.shape[1], device="cuda")
    for i in range(0, n, 1 << 17):
        j = min(n, i + (1 << 17))
        x[i:j] = centers[y[i:j]] + spread * torch.randn(j - i, centers.shape[1], device="cuda", generator=g) / centers.shape[1] ** 0.5
    return x, y


def bench_search(Q, N, D, k, C, chunk, tile):
    g = torch.Generator(device="cuda").manual_seed(0)
    centers = torch.nn.functional.normalize(torch.randn(C, D, device="cuda", generator=g), dim=1)
    xtr, ytr = clustered(N, centers, g)
    xva, yva = clustered(Q, centers, g)
    clf = KnnClassifier(xtr, ytr, C, chunk=chunk, query_tile=tile, device="cuda")
    del xtr
    qn = torch.zeros(Q, D, dtype=bf16, device="cuda")
    ops.knn_normalize(xva, y_bf16=qn)
    top_s, top_i = torch.empty(Q, k, device="cuda"), torch.empty(Q, k, dtype=torch.int32, device="cuda")
    sims = torch.empty(tile, clf.chunk, device="cuda")
    rows = clf.bank.shape[0]
    pairs = [(q0, min(tile, Q - q0), c0, min(clf.chunk, rows - c0)) for q0 in range(0, Q, tile) for c0 in range(0, rows, clf.chunk)]

    def run(record):
        for q0, nq, c0, cols in pairs:
            s = sims[:nq, :cols]
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)] if record is not None else None
            ev and ev[0].record()
            ops.gemm(qn[q0:q0 + nq], clf.bank[c0:c0 + cols], s)
            ev and ev[1].record()
            ops.topk_merge(s, top_s[q0:q0 + nq], top_i[q0:q0 + nq], offset=c0, valid=min(cols, clf.N - c0), fresh=c0 == 0)
            ev and ev[2].record()
            if record is not None:
                record.append(ev)
    run(None)                                                       # warm-up
    rec = []
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    run(rec)
    t1.record()
    torch.cuda.synchronize()
    total = t0.elapsed_time(t1)
    gemm_ms = sum(e[0].elapsed_time(e[1]) for e in rec)
    topk_ms = sum(e[1].elapsed_time(e[2]) for e in rec)
    nb = [10, 20, 100, 200]
    preds = torch.empty(Q, len(nb), 5, dtype=torch.int32, device="cuda")
    vote_ms = cuda_ms(lambda: ops.knn_vote(top_s, top_i, clf.labels, nb, 0.07, C, preds), 3, 2)
    acc = {k_: 100.0 * (preds[:, j, 0] == yva).float().mean().item() for j, k_ in enumerate(nb)}
    flops = 2.0 * Q * rows * D
    sim_bytes = 2 * 4.0 * Q * rows
    print(f"search Q={Q} N={N} D={D} k={k} (bank chunk {clf.chunk}, query tile {tile}, {len(pairs)} GEMM + merge pairs)")
    print(f"  total {total:9.1f} ms   GEMM {gemm_ms:9.1f} ms ({flops / gemm_ms / 1e9:6.1f} TFLOP/s)   top-k merge "
          f"{topk_ms:9.1f} ms ({sim_bytes / 2 / topk_ms / 1e6:6.1f} GB/s of fp32 similarities read)")
    print(f"  vote (k in {nb}, C={C}) {vote_ms:.2f} ms;  top-1 % {acc}")

    # torch baseline on the same chunks: cuBLAS bf16 mm for time; topk over the library's fp32 similarities for lists
    mm_out = torch.empty(tile, clf.chunk, dtype=bf16, device="cuda")
    bs, bi = torch.empty(Q, k, device="cuda"), torch.empty(Q, k, dtype=torch.int64, device="cuda")

    def baseline(record):
        for q0, nq, c0, cols in pairs:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            torch.mm(qn[q0:q0 + nq], clf.bank[c0:c0 + cols].t(), out=mm_out[:nq, :cols])
            ev[1].record()
            s = sims[:nq, :cols]
            ops.gemm(qn[q0:q0 + nq], clf.bank[c0:c0 + cols], s)
            e_mid = torch.cuda.Event(enable_timing=True)
            e_mid.record()
            valid = min(cols, clf.N - c0)
            cs, ci = torch.topk(s[:, :valid], min(k, valid), dim=1)
            ci += c0
            if c0 == 0:
                bs[q0:q0 + nq], bi[q0:q0 + nq] = cs, ci
            else:
                ms, mi = torch.topk(torch.cat([bs[q0:q0 + nq], cs], 1), k, dim=1)
                bs[q0:q0 + nq], bi[q0:q0 + nq] = ms, torch.gather(torch.cat([bi[q0:q0 + nq], ci], 1), 1, mi)
            ev[2].record()
            record.append((ev[0], ev[1], e_mid, ev[2]))
    baseline([])
    rec = []
    baseline(rec)
    torch.cuda.synchronize()
    mm_ms = sum(e[0].elapsed_time(e[1]) for e in rec)
    tk_ms = sum(e[2].elapsed_time(e[3]) for e in rec)
    same = (bi == top_i.long()).all(1).float().mean().item()
    w = torch.softmax(bs / 0.07, 1)
    lab = clf.labels.long()[bi]
    b_acc = {}
    for k_ in nb:
        scores = torch.zeros(Q, C, device="cuda").scatter_add_(1, lab[:, :k_], w[:, :k_])
        b_acc[k_] = 100.0 * (scores.argmax(1) == yva).float().mean().item()
    print(f"  torch baseline: torch.mm {mm_ms:9.1f} ms, torch.topk merge {tk_ms:9.1f} ms;  identical neighbour lists "
          f"{100 * same:.3f} %;  top-1 % {b_acc} (difference {max(abs(acc[k_] - b_acc[k_]) for k_ in nb):.3f} pp)")


def bench_transform(batch=256, iters=10):
    from dinov3_jax.eval.knn import _pack
    g = torch.Generator().manual_seed(0)
    imgs = [torch.randint(0, 256, (375, 500, 3), generator=g, dtype=torch.uint8).numpy() for _ in range(batch)]
    flat, desc, _ = _pack([(im, 0) for im in imgs])
    flat, desc = flat.cuda(), desc.cuda()
    out = torch.empty(batch, 224, 224, 3, dtype=bf16, device="cuda")
    taps = ops.eval_max_taps([(375, 500)], 256)
    ms = cuda_ms(lambda: ops.eval_resize_crop(flat, desc, out, resize=256, max_taps=taps, mean=(0.485, 0.456, 0.406),
                                              std=(0.229, 0.224, 0.225)), iters, 2)
    print(f"eval transform 500x375 -> 256 -> 224^2: {ms:.3f} ms per batch of {batch}, {batch / ms * 1e3:,.0f} images/s")


def bench_extract(batch=256, iters=5):
    from dinov3_jax.checkpointer import tree_from_flat
    from dinov3_jax.models import DinoVisionTransformer
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=1024, depth=24, heads=16)
    model = DinoVisionTransformer(tree_from_flat(init_backbone(cfg, torch.Generator().manual_seed(0))), embed_dim=1024,
                                  n_blocks=24, num_heads=16)
    x = torch.randn(batch, 224, 224, 3, device="cuda").to(bf16)
    ms = cuda_ms(lambda: model(x), iters, 2)
    print(f"ViT-L/16 class tokens at 224^2: {ms:.1f} ms per batch of {batch}, {batch / ms * 1e3:,.0f} images/s "
          f"(1 331 167 images: {1331167 / batch * ms / 1e3 / 60:.1f} min)")


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--queries", type=int, default=50000)
    p.add_argument("--bank", type=int, default=1281167)
    p.add_argument("--dim", type=int, default=1024)
    p.add_argument("--k", type=int, default=200)
    p.add_argument("--classes", type=int, default=1000)
    p.add_argument("--chunk", type=int, default=65536)
    p.add_argument("--tile", type=int, default=4096)
    a = p.parse_args()
    assert torch.cuda.is_available(), "bench_knn measures on the GPU"
    from dinov3_jax import _native
    _native.init(0)
    print(card())
    bench_transform()
    bench_extract()
    bench_search(a.queries, a.bank, a.dim, a.k, a.classes, a.chunk, a.tile)


if __name__ == "__main__":
    main()
