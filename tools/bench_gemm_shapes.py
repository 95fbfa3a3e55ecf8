"""GPU microbench: every GEMM call shape of one ViT-L/16 B=64 training step, with its real epilogue, timed in isolation."""
import os, statistics, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200"))
import torch
from dinov3_jax import ops

from gpu_timing import card, cuda_ms

dev = "cuda"
bf, f32 = torch.bfloat16, torch.float32
D, Hd = 1024, 4096
Tt, Ts = 25216, 44160


def cases():
    """(name, FLOP, fn(tile_n)) of the 13 GEMM shapes of one student block, forward and backward."""
    T = Ts
    X = torch.randn(T, D, device=dev).to(bf); H = torch.randn(T, Hd, device=dev).to(bf)
    Wqkv = torch.randn(D, 3 * D, device=dev).to(bf); Wp = torch.randn(D, D, device=dev).to(bf)
    W1 = torch.randn(D, Hd, device=dev).to(bf); W2 = torch.randn(Hd, D, device=dev).to(bf)
    b3, b1, bd = torch.randn(3 * D, device=dev), torch.randn(Hd, device=dev), torch.randn(D, device=dev)
    gam = torch.randn(D, device=dev)
    QKV = torch.empty(T, 3 * D, device=dev, dtype=bf); Xf = torch.randn(T, D, device=dev); Xo = torch.empty(T, D, device=dev)
    P = torch.empty(T, D, device=dev, dtype=bf); U1 = torch.empty(T, Hd, device=dev, dtype=bf); Hh = torch.empty(T, Hd, device=dev, dtype=bf)
    dU2 = torch.randn(T, D, device=dev).to(bf); dU1 = torch.empty(T, Hd, device=dev, dtype=bf); dQKV = torch.randn(T, 3 * D, device=dev).to(bf)
    dZ = torch.empty(T, D, device=dev, dtype=bf)
    gW2 = torch.empty(Hd, D, device=dev); gW1 = torch.empty(D, Hd, device=dev); gWqkv = torch.empty(D, 3 * D, device=dev); gWp = torch.empty(D, D, device=dev)
    return [
        ("fwd qkv   [T,D]x[D,3D] +bias",            2 * T * D * 3 * D, lambda tn: ops.gemm(X, Wqkv, QKV, b_mn=True, bias=b3, tile_n=tn)),
        ("fwd proj  +bias,pre,gamma,resid(f32)",     2 * T * D * D,     lambda tn: ops.gemm(X, Wp, Xo, b_mn=True, bias=bd, store_pre=P, gamma=gam, resid=Xf, tile_n=tn)),
        ("fwd fc1   +bias,pre,gelu",                 2 * T * D * Hd,    lambda tn: ops.gemm(X, W1, Hh, b_mn=True, bias=b1, gelu=True, store_pre=U1, tile_n=tn)),
        ("fwd fc1   +bias,gelu (teacher)",           2 * T * D * Hd,    lambda tn: ops.gemm(X, W1, Hh, b_mn=True, bias=b1, gelu=True, tile_n=tn)),
        ("fwd fc2   +bias,pre,gelu,gamma,resid",     2 * T * D * Hd,    lambda tn: ops.gemm(H, W2, Xo, b_mn=True, bias=bd, gelu=True, store_pre=P, gamma=gam, resid=Xf, tile_n=tn)),
        ("dgrad fc2 [T,D]x[D,4D] *gelu'(u1)",        2 * T * D * Hd,    lambda tn: ops.gemm(dU2, W2, dU1, dgelu_of=U1, tile_n=tn)),
        ("dgrad fc1 [T,4D]x[4D,D]",                  2 * T * D * Hd,    lambda tn: ops.gemm(H, W1, dZ, tile_n=tn)),
        ("dgrad proj[T,D]x[D,D]",                    2 * T * D * D,     lambda tn: ops.gemm(dU2, Wp, dZ, tile_n=tn)),
        ("dgrad qkv [T,3D]x[3D,D]",                  2 * T * D * 3 * D, lambda tn: ops.gemm(dQKV, Wqkv, dZ, tile_n=tn)),
        ("wgrad fc2 [4D,T]x[T,D] f32",               2 * T * D * Hd,    lambda tn: ops.gemm(H, dU2, gW2, a_mn=True, b_mn=True, accum=True, tile_n=tn)),
        ("wgrad fc1 [D,T]x[T,4D] f32",               2 * T * D * Hd,    lambda tn: ops.gemm(X, H, gW1, a_mn=True, b_mn=True, accum=True, tile_n=tn)),
        ("wgrad qkv [D,T]x[T,3D] f32",               2 * T * D * 3 * D, lambda tn: ops.gemm(X, dQKV, gWqkv, a_mn=True, b_mn=True, accum=True, tile_n=tn)),
        ("wgrad proj[D,T]x[T,D] f32",                2 * T * D * D,     lambda tn: ops.gemm(X, dU2, gWp, a_mn=True, b_mn=True, accum=True, tile_n=tn)),
    ]


def run(widths, batches, only=None):
    """Every shape at every tile width (0 = the automatic choice), the widths alternated shape by shape within each of
    `batches` batches; prints the median time per shape and width, and each median's min-max over the batches."""
    cs = [c for c in cases() if not only or only in c[0]]
    ms = {(c[0], w): [] for c in cs for w in widths}
    for _ in range(batches):
        for name, _, fn in cs:
            for w in widths:
                ms[(name, w)].append(cuda_ms(lambda: fn(w), 8, 3))
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(f"  {'shape':44s}" + "".join(f" {'auto' if w == 0 else w:>21}" for w in widths))
    tot = {w: [0.0, 0] for w in widths}
    for name, fl, _ in cs:
        row = f"  {name:44s}"
        for w in widths:
            v = ms[(name, w)]
            row += f" {med[(name, w)]:6.3f} ms {fl / med[(name, w)] / 1e9:5.0f} TF/s"
            tot[w][0] += med[(name, w)]; tot[w][1] += fl
        print(row + "   spread " + " ".join(f"{(max(ms[(name, w)]) - min(ms[(name, w)])) / med[(name, w)] * 100:.1f}%"
                                            for w in widths), flush=True)
    print(f"  {'sum of medians':44s}" + "".join(f" {tot[w][0]:6.3f} ms {tot[w][1] / tot[w][0] / 1e9:5.0f} TF/s" for w in widths))


if __name__ == "__main__":
    # bench_gemm_shapes.py [batches] [width ...] [--only SUBSTRING]; widths default to auto, 128, 256
    args = sys.argv[1:]
    only = None
    if "--only" in args:
        i = args.index("--only"); only = args[i + 1]; del args[i:i + 2]
    batches = int(args[0]) if args else 5
    widths = [int(a) for a in args[1:]] or [0, 128, 256]
    print(card())
    print(f"== student stream T={Ts}, {batches} batches, widths {widths} (0 = automatic)")
    run(widths, batches, only)
