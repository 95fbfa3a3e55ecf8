"""GPU: time the HBM-bound backward kernels at the ViT-L student-stream shape (T=44160, D=1024) and print achieved GB/s
against their algorithmic bytes (DESIGN.md §4)."""
import sys, os
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dinov3-jax_b200"))
import torch
from dinov3_jax import ops

T, D = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (44160, 1024)
dev = "cuda"
bf = torch.bfloat16
x = torch.randn(T, D, device=dev); dyb = torch.randn(T, D, device=dev).to(bf); add = torch.randn(T, D, device=dev)
mean, rstd = torch.zeros(T, device=dev), torch.ones(T, device=dev)
sc = torch.ones(D, device=dev); gam = torch.ones(D, device=dev)
dx = torch.empty(T, D, device=dev); ds, db = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
u = torch.randn(T, D, device=dev).to(bf); du = torch.empty(T, D, device=dev, dtype=bf)
dg, dbl = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
O = torch.randn(T, D, device=dev).to(bf)
big = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(name, fn, nbytes, it=20):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(it):
        big.zero_()                      # flush L2
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    ms = ts[len(ts) // 2]
    print(f"  {name:58s} {ms * 1e3:8.1f} us   {nbytes / ms / 1e6:8.1f} GB/s")


TD = T * D
print(f"T={T} D={D}")
timeit("layernorm_bwd_ls plain", lambda: ops.layernorm_bwd_ls(dyb, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db), TD * (2 + 4 + 4 + 4))
timeit("layernorm_bwd_ls linear tail", lambda: ops.layernorm_bwd_ls(dyb, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db, ls_gamma=gam, ls_du=du, ls_dbias=dbl), TD * (2 + 4 + 4 + 4 + 2))
timeit("layernorm_bwd_ls gelu tail", lambda: ops.layernorm_bwd_ls(dyb, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db, ls_gamma=gam, ls_u=u, ls_gelu=True, ls_du=du, ls_dgamma=dg, ls_dbias=dbl), TD * (2 + 4 + 4 + 4 + 2 + 2))
timeit("ls_act_bwd gelu", lambda: ops.ls_act_bwd(add, u, gam, du, dg, dbl, True), TD * (4 + 2 + 2))
timeit("ls_act_bwd linear", lambda: ops.ls_act_bwd(add, u, gam, du, dg, dbl, False), TD * (4 + 2 + 2))
y = torch.empty(T, D, device=dev, dtype=bf)
timeit("layernorm_fwd bf16 out", lambda: ops.layernorm_fwd(x, sc, sc, y, mean, rstd), TD * (4 + 2))
cs = torch.zeros(3 * D, device=dev); q = torch.randn(T, 3 * D, device=dev).to(bf)
timeit("colsum_bf16 [T,3D]", lambda: ops.colsum_bf16(q, cs), TD * 3 * 2)
h = torch.randn(T, 4 * D, device=dev).to(bf); cs4 = torch.zeros(4 * D, device=dev)
timeit("colsum_bf16 [T,4D]", lambda: ops.colsum_bf16(h, cs4), TD * 4 * 2)

# ---- head / loss kernels at the iBOT shape (M = 3771 masked tokens, K = 65536 prototypes)
if len(sys.argv) <= 2:
    M, K = 3771, 65536
    Lt = torch.randn(M, K, device=dev) * 0.3; S = torch.randn(M, K, device=dev)
    mx = torch.full((K,), float("-inf"), device=dev); sv = torch.zeros(K, device=dev); a = torch.ones(M, device=dev)
    btot = torch.full((1,), float(M), device=dev)
    MK = M * K
    print(f"M={M} K={K}")
    timeit("colmax", lambda: ops.colmax(Lt, mx), MK * 4)
    timeit("sinkhorn_colsum", lambda: ops.sinkhorn_colsum(Lt, mx, 0.05, a, sv), MK * 4)
    sv.fill_(1.0)
    timeit("sinkhorn_rowsum", lambda: ops.sinkhorn_rowsum(Lt, mx, 0.05, sv, btot, a), MK * 4)
    t0 = torch.arange(M, device=dev, dtype=torch.int32); t1 = torch.full((M,), -1, device=dev, dtype=torch.int32)
    wm = torch.ones(M, device=dev); wg = torch.ones(M, device=dev); slot = torch.zeros(M, device=dev, dtype=torch.int32)
    metric = torch.zeros(8, device=dev); dS = torch.empty(M, K, device=dev, dtype=bf)
    timeit("ce_fwd_bwd (iBOT: 1 teacher row per student row)", lambda: ops.ce_fwd_bwd(S, 0.1, Lt, mx, 0.05, sv, a, btot, t0, t1, wm, wg, slot, metric, dS), MK * (4 + 4 + 2))
    dOo = torch.randn(T, D, device=dev).to(bf); dl = torch.empty(T // 197, 16, 197, device=dev)
