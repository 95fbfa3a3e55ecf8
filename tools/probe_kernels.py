"""GPU probe of every non-GEMM kernel against PyTorch fp32 on the same device (one group per subprocess)."""
import math, os, subprocess, sys, time
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def report(name, a, b, tol):
    r = rel(a, b); mx = (a.float() - b.float()).abs().max().item()
    nan = int(torch.isnan(a.float()).sum())
    print(f"  {name}: rel={r:.3e} maxabs={mx:.3e} nan={nan} {'ok' if (r < tol and nan == 0) else 'BAD'}", flush=True)


def attn_ref(qkv, n, N, D, H):
    q, k, v = qkv.float().reshape(n, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * 0.125
    p = torch.softmax(s, -1)
    o = (p @ v).permute(0, 2, 1, 3).reshape(n * N, D)
    return o, torch.logsumexp(s, -1)


def g_attn_fwd():
    for (n, N, H) in [(3, 197, 2), (5, 37, 2), (2, 128, 1), (2, 257, 1), (4, 50, 3), (128, 197, 16)]:
        D = 64 * H
        qkv = (torch.randn(n * N, 3 * D, device="cuda") * 1.0).to(torch.bfloat16)
        o = torch.full((n * N, D), float("nan"), device="cuda", dtype=torch.bfloat16)
        lse = torch.zeros(n, H, N, device="cuda")
        ops.attn_fwd(qkv, o, lse, n, N, D, H); torch.cuda.synchronize()
        ro, rl = attn_ref(qkv, n, N, D, H)
        report(f"attn_fwd n={n} N={N} H={H} o", o, ro, 1e-2)
        report(f"attn_fwd n={n} N={N} H={H} lse", lse, rl, 1e-4)
    n, N, H = 128, 197, 16; D = 1024
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16); o = torch.empty(n * N, D, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(n, H, N, device="cuda")
    for _ in range(3): ops.attn_fwd(qkv, o, lse, n, N, D, H)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(10): ops.attn_fwd(qkv, o, lse, n, N, D, H)
    e.record(); torch.cuda.synchronize()
    ms = s.elapsed_time(e) / 10
    print(f"  perf attn_fwd n=128 N=197 H=16: {ms:.3f} ms  {4*N*N*D*n/ms/1e9:.1f} TFLOP/s")


def g_attn_bwd():
    for (n, N, H) in [(2, 128, 1), (3, 197, 2), (5, 37, 2), (4, 50, 3), (2, 256, 1)]:
        D = 64 * H
        qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
        do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
        x = qkv.float().requires_grad_(True)
        ro, _ = attn_ref(x, n, N, D, H)
        ro.backward(do.float())
        o = torch.empty(n * N, D, device="cuda", dtype=torch.bfloat16); lse = torch.zeros(n, H, N, device="cuda")
        ops.attn_fwd(qkv, o, lse, n, N, D, H)
        dqkv = torch.full((n * N, 3 * D), float("nan"), device="cuda", dtype=torch.bfloat16)
        delta = torch.zeros(n, H, N, device="cuda")
        ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H); torch.cuda.synchronize()
        g = x.grad
        report(f"attn_bwd n={n} N={N} H={H} dq", dqkv[:, :D], g[:, :D], 2e-2)
        report(f"attn_bwd n={n} N={N} H={H} dk", dqkv[:, D:2*D], g[:, D:2*D], 2e-2)
        report(f"attn_bwd n={n} N={N} H={H} dv", dqkv[:, 2*D:], g[:, 2*D:], 2e-2)
    n, N, H = 128, 197, 16; D = 1024
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16); o = torch.empty(n * N, D, device="cuda", dtype=torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16); dqkv = torch.empty_like(qkv)
    lse = torch.zeros(n, H, N, device="cuda"); delta = torch.zeros(n, H, N, device="cuda")
    ops.attn_fwd(qkv, o, lse, n, N, D, H)
    for _ in range(2): ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(5): ops.attn_bwd(qkv, o, do, lse, delta, dqkv, n, N, D, H)
    e.record(); torch.cuda.synchronize()
    print(f"  perf attn_bwd n=128 N=197 H=16: {s.elapsed_time(e)/5:.3f} ms")


def g_elementwise():
    from oracle.model import rope_sincos, rope_apply, layer_norm
    dev = "cuda"
    # im2col
    n, Hh, p = 3, 64, 16
    img = torch.randn(n, Hh, Hh, 3, device=dev).to(torch.bfloat16)
    out = torch.empty(n * (Hh // p) ** 2, p * p * 3, device=dev, dtype=torch.bfloat16)
    ops.im2col(img, out, p)
    ref = img.reshape(n, Hh // p, p, Hh // p, p, 3).permute(0, 1, 3, 2, 4, 5).reshape(out.shape)
    print("  im2col exact:", bool((out == ref).all()))
    # tokens
    P, D = 16, 128
    tok = torch.randn(n * P, D, device=dev); cls = torch.randn(D, device=dev); mt = torch.randn(D, device=dev)
    masks = (torch.rand(n, P, device=dev) < 0.3)
    X = torch.empty(n, P + 1, D, device=dev)
    ops.assemble_tokens(tok, cls, mt, masks.to(torch.uint8), X, n, P, D)
    refX = torch.cat([cls.expand(n, 1, D), torch.where(masks[..., None], mt, tok.reshape(n, P, D))], 1)
    print("  assemble_tokens exact:", bool((X == refX).all()))
    dX = torch.randn(n, P + 1, D, device=dev); dTok = torch.empty(n * P, D, device=dev, dtype=torch.bfloat16)
    dcls = torch.zeros(D, device=dev); dm = torch.zeros(D, device=dev)
    ops.assemble_tokens_bwd(dX, masks.to(torch.uint8), dTok, dcls, dm, n, P, D)
    report("assemble_bwd dTok", dTok, torch.where(masks[..., None], torch.zeros_like(dX[:, 1:]), dX[:, 1:]).reshape(n * P, D), 4e-3)
    report("assemble_bwd dcls", dcls, dX[:, 0].sum(0), 1e-5)
    report("assemble_bwd dmask", dm, (dX[:, 1:] * masks[..., None]).sum((0, 1)), 1e-5)
    # layernorm
    for (T, D) in [(1000, 384), (4433, 1024)]:
        x = torch.randn(T, D, device=dev) * 2 + 0.5; sc = torch.randn(D, device=dev); bi = torch.randn(D, device=dev)
        y = torch.empty(T, D, device=dev, dtype=torch.bfloat16); yf = torch.empty(T, D, device=dev)
        mean = torch.empty(T, device=dev); rstd = torch.empty(T, device=dev)
        ops.layernorm_fwd(x, sc, bi, y, mean, rstd); ops.layernorm_fwd(x, sc, bi, yf, mean, rstd)
        xr = x.clone().requires_grad_(True); scr = sc.clone().requires_grad_(True); bir = bi.clone().requires_grad_(True)
        ref = layer_norm(xr, scr, bir, 1e-6)
        report(f"ln_fwd bf16 T={T} D={D}", y, ref, 4e-3); report(f"ln_fwd f32 T={T} D={D}", yf, ref, 1e-5)
        dy = torch.randn(T, D, device=dev); ref.backward(dy)
        add = torch.randn(T, D, device=dev)
        dx = torch.empty(T, D, device=dev); ds = torch.zeros(D, device=dev); db = torch.zeros(D, device=dev)
        ops.layernorm_bwd_ls(dy, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db)
        report("ln_bwd dx(f32 dy)", dx, xr.grad + add, 1e-4); report("ln_bwd dscale", ds, scr.grad, 1e-4); report("ln_bwd dbias", db, bir.grad, 1e-4)
        dyb = dy.to(torch.bfloat16); dx2 = torch.empty(T, D, device=dev)
        ops.layernorm_bwd_ls(dyb, x, mean, rstd, sc, dx2)
        xr.grad = None; layer_norm(xr, sc, bi, 1e-6).backward(dyb.float())
        report("ln_bwd dx(bf16 dy)", dx2, xr.grad, 1e-4)
    # rope
    n, Hp, H = 3, 6, 2; N = Hp * Hp + 1; D = 64 * H
    sin, cos = rope_sincos(Hp, Hp, 64, 100.0, torch.float32); sin, cos = sin.to(dev), cos.to(dev)
    qkv = torch.randn(n * N, 3 * D, device=dev).to(torch.bfloat16)
    ref = qkv.float().reshape(n, N, 3, H, 64).clone()
    for w in (0, 1):
        ref[:, 1:, w] = rope_apply(ref[:, 1:, w].transpose(1, 2), sin, cos).transpose(1, 2)
    q2 = qkv.clone(); ops.rope(q2, sin.contiguous(), cos.contiguous(), N, 1, D, 64)
    report("rope fwd", q2, ref.reshape(n * N, 3 * D), 4e-3)
    # inverse: <rope(x), g> == <x, rope_inv(g)>
    g = torch.randn(n * N, 3 * D, device=dev).to(torch.bfloat16); gi = g.clone()
    ops.rope(gi, sin.contiguous(), cos.contiguous(), N, 1, D, 64, inverse=True)
    lhs = (ref.reshape(n * N, 3 * D) * g.float()).sum().item(); rhs = (qkv.float() * gi.float()).sum().item()
    print(f"  rope adjoint: {lhs:.4f} vs {rhs:.4f} {'ok' if abs(lhs-rhs) < 2e-2*abs(lhs)+0.5 else 'BAD'}")
    # gather / scatter / token rows
    P = 16; nn_ = 4; D = 128
    src = torch.randn(nn_ * (P + 1), D, device=dev)
    midx = torch.tensor([0, 3, 17, 18, 40, 63], device=dev, dtype=torch.int64)
    rows = torch.empty(6, dtype=torch.int32, device=dev); ops.token_rows(midx, rows, 6, P, 0)
    want = (midx // P * (P + 1) + 1 + midx % P).int()
    print("  token_rows exact:", bool((rows == want).all()))
    crow = torch.empty(nn_, dtype=torch.int32, device=dev); ops.token_rows(None, crow, nn_, P, 1)
    print("  cls rows exact:", bool((crow == torch.arange(nn_, device=dev).int() * (P + 1)).all()))
    gb = torch.empty(6, D, device=dev, dtype=torch.bfloat16); gf = torch.empty(6, D, device=dev)
    ops.gather_rows(src, rows, 6, D, gb, gf)
    print("  gather exact:", bool((gf == src[want.long()]).all()), bool((gb == src[want.long()].to(torch.bfloat16)).all()))
    dst = torch.zeros_like(src); ops.scatter_add_rows(gf, rows, dst, 6, D)
    ref = torch.zeros_like(src); ref[want.long()] += gf
    print("  scatter exact:", bool((dst == ref).all()))
    # l2norm
    R, Cc = 300, 256
    u = torch.randn(R, Cc, device=dev); y = torch.empty(R, Cc, device=dev, dtype=torch.bfloat16); nr = torch.empty(R, device=dev)
    ops.l2norm_fwd(u, y, nr)
    ur = u.clone().requires_grad_(True); yr = ur / (ur.norm(dim=-1, keepdim=True) + 1e-12)
    report("l2norm fwd", y, yr, 4e-3)
    g = torch.randn(R, Cc, device=dev).to(torch.bfloat16); yr.backward(g.float())
    du = torch.empty(R, Cc, device=dev, dtype=torch.bfloat16); ops.l2norm_bwd(g, u, nr, du)
    report("l2norm bwd", du, ur.grad, 6e-3)
    # ls_act_bwd
    T, D = 777, 384
    dX = torch.randn(T, D, device=dev); ub = torch.randn(T, D, device=dev).to(torch.bfloat16); gam = torch.randn(D, device=dev)
    for use_gelu in (True, False):
        uu = ub.float().requires_grad_(True); gg = gam.clone().requires_grad_(True)
        act = torch.nn.functional.gelu(uu, approximate="tanh") if use_gelu else uu
        (gg * act * dX).sum().backward()
        du = torch.empty(T, D, device=dev, dtype=torch.bfloat16); dg = torch.zeros(D, device=dev); db = torch.zeros(D, device=dev)
        ops.ls_act_bwd(dX, ub, gam, du, dg, db, use_gelu)
        report(f"ls_act_bwd gelu={use_gelu} du", du, uu.grad, 5e-3); report("  dgamma", dg, gg.grad, 1e-4); report("  dbias", db, du.float().sum(0), 1e-4)
    xb = torch.randn(1001, 1152, device=dev).to(torch.bfloat16); cs = torch.zeros(1152, device=dev)
    ops.colsum_bf16(xb, cs); report("colsum_bf16", cs, xb.float().sum(0), 1e-5)
    xb = torch.randn(50, 7 * 2, device=dev).to(torch.bfloat16); cs = torch.zeros(14, device=dev)
    ops.colsum_bf16(xb, cs); report("colsum_bf16 small", cs, xb.float().sum(0), 1e-5)
    src = torch.randn(100003 * 4, device=dev); dstb = torch.empty(100003 * 4, device=dev, dtype=torch.bfloat16)
    ops.cast_f32_bf16(src, dstb); print("  cast exact:", bool((dstb == src.to(torch.bfloat16)).all()))


def g_losses():
    from oracle.losses import sinkhorn_knopp, dino_loss, ibot_loss_masked, koleo_loss
    dev = "cuda"
    R, K, temp = 24, 4096, 0.05
    L = torch.randn(R, K, device=dev) * 0.3
    mx = torch.full((K,), float("-inf"), device=dev); ops.colmax(L, mx)
    print("  colmax exact:", bool(torch.equal(mx, L.max(0).values)))
    btot = torch.tensor([float(R)], device=dev)
    a = None; s = torch.zeros(K, device=dev); av = torch.empty(R, device=dev)
    for it in range(3):
        s.zero_(); ops.sinkhorn_colsum(L, mx, temp, a, s); ops.sinkhorn_rowsum(L, mx, temp, s, btot, av); a = av
    Q = torch.empty(R, K, device=dev); ops.sinkhorn_probs(L, mx, temp, s, a, btot, Q)
    Qr = sinkhorn_knopp(L.double(), temp, R).float()
    report("sinkhorn probs", Q, Qr, 1e-4)
    # CE: dino-like pairing, S rows 10*B, teacher 2*B
    B = R // 2
    S = (torch.randn(10 * B, K, device=dev) * 0.5)
    Sr = S.double().requires_grad_(True)
    sg, sl = Sr[: 2 * B].reshape(2, B, K), Sr[2 * B:].reshape(8, B, K)
    Tq = Qr.double().reshape(2, B, K)
    Ll = dino_loss(sl, Tq, 0.1, False); Lg = dino_loss(sg, Tq, 0.1, True)
    wl, wgl = 16 / 18, 2 / 18
    (wl * Ll + wgl * Lg).backward()
    t0 = torch.empty(10 * B, dtype=torch.int32); t1 = torch.empty(10 * B, dtype=torch.int32)
    wm = torch.empty(10 * B); wg = torch.empty(10 * B); slot = torch.empty(10 * B, dtype=torch.int32)
    for i in range(10 * B):
        sidx, b = divmod(i, B)
        if sidx < 2:
            t0[i] = (1 - sidx) * B + b; t1[i] = -1; wm[i] = 1.0 / (B * 2); wg[i] = wgl / (B * 2); slot[i] = 1
        else:
            t0[i] = b; t1[i] = B + b; wm[i] = 1.0 / (B * 16); wg[i] = wl / (B * 16); slot[i] = 0
    metric = torch.zeros(4, device=dev); dS = torch.empty(10 * B, K, device=dev, dtype=torch.bfloat16)
    ops.ce_fwd_bwd(S, 0.1, L, mx, temp, s, a, btot, t0.to(dev), t1.to(dev), wm.to(dev), wg.to(dev), slot.to(dev), metric, dS)
    print(f"  ce metric local {metric[0].item():.6f} vs {Ll.item():.6f}; global {metric[1].item():.6f} vs {Lg.item():.6f}")
    report("ce dS", dS, Sr.grad, 6e-3)
    # koleo
    Bk, D = 64, 384
    x = torch.randn(Bk, D, device=dev)
    xr = x.double().requires_grad_(True); lk = koleo_loss(xr); (0.1 * lk).backward()
    xn = torch.empty(Bk, D, device=dev); nr = torch.empty(Bk, device=dev); nn = torch.empty(Bk, dtype=torch.int32, device=dev)
    cf = torch.empty(Bk, device=dev); met = torch.zeros(1, device=dev); dx = torch.zeros(Bk, D, device=dev)
    ops.koleo_fwd_bwd(x, xn, nr, nn, cf, met, dx, 1.0, 0.1)
    print(f"  koleo loss {met.item():.6f} vs {lk.item():.6f}")
    report("koleo dx", dx, xr.grad, 1e-4)


def g_optim():
    import numpy as np
    dev = "cuda"
    n = 4096 * 3 + 64
    p = torch.randn(n, device=dev); g = torch.randn(n, device=dev) * 0.01; m = torch.randn(n, device=dev) * 0.001
    v = torch.rand(n, device=dev) * 1e-4; t = torch.randn(n, device=dev)
    ss = torch.zeros(1, device=dev); ops.sumsq(g, ss); report("sumsq", ss, (g.double() ** 2).sum().float().reshape(1), 1e-5)
    segs_np = np.zeros(3, dtype=[("start", "<i8"), ("lr", "<f4"), ("wd", "<f4"), ("last", "<i4"), ("pad", "<i4")])
    segs_np["start"] = [0, 4096, 8192 + 64]; segs_np["lr"] = [1.0, 0.5, 0.2]; segs_np["wd"] = [1.0, 0.0, 1.0]; segs_np["last"] = [0, 0, 1]
    segs = torch.from_numpy(segs_np.view(np.uint8)).to(dev)
    lr, llr, wd, mom, step, maxn = 1e-3, 5e-4, 0.04, 0.99, 3, 0.5
    P0, M0, V0, T0 = p.double(), m.double(), v.double(), t.double()
    scale = min(1.0, maxn / (math.sqrt(ss.item()) + 1e-6)); G = g.double() * scale
    idx = torch.arange(n, device=dev)
    lrm = torch.where(idx < 4096, 1.0, torch.where(idx < 8256, 0.5, 0.2)).double()
    wdm = torch.where(idx < 4096, 1.0, torch.where(idx < 8256, 0.0, 1.0)).double()
    base = torch.where(idx < 8256, lr, llr).double()
    M1 = 0.9 * M0 + 0.1 * G; V1 = 0.999 * V0 + 0.001 * G * G
    upd = (M1 / (1 - 0.9 ** step)) / ((V1 / (1 - 0.999 ** step)).sqrt() + 1e-8) + wd * wdm * P0
    P1 = P0 - base * lrm * upd; T1 = T0 * mom + P1 * (1 - mom)
    pb = torch.zeros(8192, device=dev, dtype=torch.bfloat16); tb = torch.zeros(8192, device=dev, dtype=torch.bfloat16)
    ops.adamw_ema(p, g, m, v, t, pb, tb, 8192, segs, 3, ss, maxn, lr, llr, wd, step, mom)
    report("adamw p", p, P1, 1e-6); report("adamw m", m, M1, 1e-6); report("adamw v", v, V1, 1e-6); report("ema teacher", t, T1, 1e-6)
    print("  bf16 copies exact:", bool((pb == p[:8192].to(torch.bfloat16)).all()), bool((tb == t[:8192].to(torch.bfloat16)).all()))


GROUPS = {"attn_fwd": g_attn_fwd, "attn_bwd": g_attn_bwd, "elementwise": g_elementwise, "losses": g_losses, "optim": g_optim}

if __name__ == "__main__":
    if len(sys.argv) == 2 and sys.argv[1] in GROUPS:
        import torch
        from dinov3_jax import ops
        torch.manual_seed(0)
        GROUPS[sys.argv[1]]()
        sys.exit(0)
    names = sys.argv[1:] or list(GROUPS)
    for g in names:
        print(f"== {g}", flush=True)
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, __file__, g], timeout=180)
            print(f"== exit {r.returncode} in {time.time()-t0:.1f}s", flush=True)
        except subprocess.TimeoutExpired:
            print("== TIMEOUT (hang)", flush=True)
