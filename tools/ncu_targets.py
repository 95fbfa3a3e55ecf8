"""One launch of each HBM-bound / attention kernel at the ViT-L student-stream shape, for
`ncu --set full --clock-control none -k regex:d3 -o profile_out/r01_ncu_hbm python tools/ncu_targets.py`."""
import os, sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dinov3-jax_b200"))
import torch
from dinov3_jax import ops

dev, bf = "cuda", torch.bfloat16
T, D, H = 44160, 1024, 16
x = torch.randn(T, D, device=dev); dyb = torch.randn(T, D, device=dev).to(bf); add = torch.randn(T, D, device=dev)
mean, rstd = torch.zeros(T, device=dev), torch.ones(T, device=dev)
sc = torch.ones(D, device=dev); gam = torch.ones(D, device=dev)
dx = torch.empty(T, D, device=dev); ds, db = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
u = torch.randn(T, D, device=dev).to(bf); du = torch.empty(T, D, device=dev, dtype=bf)
dg, dbl = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
y = torch.empty(T, D, device=dev, dtype=bf)
torch.cuda.synchronize()
ops.layernorm_fwd(x, sc, sc, y, mean, rstd)
ops.layernorm_bwd_ls(dyb, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db, ls_gamma=gam, ls_du=du, ls_dbias=dbl)
ops.layernorm_bwd_ls(dyb, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db, ls_gamma=gam, ls_u=u, ls_gelu=True, ls_du=du, ls_dgamma=dg, ls_dbias=dbl)
q = torch.randn(T, 3 * D, device=dev).to(bf); cs = torch.zeros(3 * D, device=dev)
ops.colsum_bf16(q, cs)
M, K = 3771, 65536
Lt = torch.randn(M, K, device=dev) * 0.3; S = torch.randn(M, K, device=dev)
mx = torch.full((K,), float("-inf"), device=dev); sv = torch.zeros(K, device=dev); a = torch.ones(M, device=dev)
btot = torch.full((1,), float(M), device=dev)
ops.colmax(Lt, mx)
ops.sinkhorn_colsum(Lt, mx, 0.05, a, sv)
ops.sinkhorn_rowsum(Lt, mx, 0.05, sv, btot, a)
t0 = torch.arange(M, device=dev, dtype=torch.int32); t1 = torch.full((M,), -1, device=dev, dtype=torch.int32)
wm = torch.ones(M, device=dev); wg = torch.ones(M, device=dev); slot = torch.zeros(M, device=dev, dtype=torch.int32)
metric = torch.zeros(8, device=dev); dS = torch.empty(M, K, device=dev, dtype=bf)
ops.ce_fwd_bwd(S, 0.1, Lt, mx, 0.05, sv, a, btot, t0, t1, wm, wg, slot, metric, dS)
# attention at the global-crop shape: 128 crops x 16 heads x 197 tokens
n, N = 128, 197
qkv = torch.randn(n * N, 3 * D, device=dev).to(bf); o = torch.empty(n * N, D, device=dev, dtype=bf)
lse = torch.empty(n, H, N, device=dev); delta = torch.empty(n, H, N, device=dev)
ops.attn_fwd(qkv, o, lse, n, N, D, H)
do = torch.randn(n * N, D, device=dev).to(bf); dqkv = torch.empty(n * N, 3 * D, device=dev, dtype=bf)
ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H)
torch.cuda.synchronize()
print("done")
