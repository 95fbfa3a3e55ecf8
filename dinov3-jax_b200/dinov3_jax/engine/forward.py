"""The one ViT forward: kernel launches that read weights through a `Net` and write a `Stream` / `HeadBufs`.  The
engine's student, EMA, distillation and gram teachers, the feature model and the layer wrappers all run these pieces."""
from __future__ import annotations

import math

import torch

from .. import ops
from .config import EngineConfig

f32, bf16, u8 = torch.float32, torch.bfloat16, torch.uint8


def rope_tables(Hp: int, Wp: int, head_dim: int, base: float, device):
    """sin / cos [Hp*Wp, head_dim] fp32 — layers/rope_position_encoding.py:36-40,64-73,117-123 (normalize 'separate').
    Host-side table construction (a few KB, once per crop size); the rotation itself is d3_rope."""
    dt = torch.float64
    periods = base ** (2.0 * torch.arange(head_dim // 4, dtype=dt) / (head_dim // 2))
    ch = torch.arange(0.5, Hp, dtype=dt) / Hp
    cw = torch.arange(0.5, Wp, dtype=dt) / Wp
    coords = torch.stack(torch.meshgrid(ch, cw, indexing="ij"), dim=-1).reshape(-1, 2)
    coords = 2.0 * coords - 1.0
    ang = 2 * math.pi * coords[:, :, None] / periods[None, None, :]
    ang = ang.reshape(ang.shape[0], -1)
    ang = torch.cat([ang, ang], dim=-1)
    # the reference computes the tables in fp32 (SURVEY A8); fp64 -> fp32 rounding differs by < 1 ulp
    return (torch.sin(ang).to(f32).to(device).contiguous(), torch.cos(ang).to(f32).to(device).contiguous())


class CropSet:
    """`n_crops` crops of an Hp x Wp patch grid inside a token stream; `rope`: (sin, cos) instead of the grid's own."""

    def __init__(self, cfg: EngineConfig, n_crops: int, Hp: int, Wp: int, row0: int, device, rope=None):
        self.n = n_crops
        self.Hp, self.Wp = Hp, Wp
        self.P = Hp * Wp
        self.N = self.P + cfg.prefix
        self.T = n_crops * self.N
        self.row0 = row0
        self.sin, self.cos = rope if rope is not None else rope_tables(Hp, Wp, cfg.head_dim, cfg.rope_base, device)
        kdim = cfg.patch * cfg.patch * 3
        kpad = (kdim + 7) // 8 * 8             # TMA needs 16-byte row strides (patch 14: 588 -> 592, padding zeroed)
        self.patches = torch.empty(n_crops * self.P, kpad, dtype=bf16, device=device)[:, :kdim]


class Stream:
    """Activation buffers of one network pass over a list of crop sets (teacher: global only; student: global+local)."""

    def __init__(self, cfg: EngineConfig, sets, device, stash: bool, remat: bool = False, fp8: bool = False):
        D, Hd, L = cfg.embed_dim, cfg.ffn_width, cfg.depth
        swiglu = cfg.ffn_layer == "swiglu"
        self.sets = sets
        T = self.T = sum(s.T for s in sets)
        self.stash = stash                    # keep what the backward needs
        self.per_block = stash and not remat  # ... for every block (False: one scratch set, blocks are recomputed)
        nb = L if self.per_block else 1
        e = lambda *shape, dt=bf16: torch.empty(*shape, dtype=dt, device=device)
        self.X = [e(T, D, dt=f32) for _ in range(L + 1)] if stash else [e(T, D, dt=f32), e(T, D, dt=f32)]
        self.Xmid = [e(T, D, dt=f32) for _ in range(nb)]
        self.Y = [e(T, D) for _ in range(nb)]
        self.QKV = [e(T, 3 * D) for _ in range(nb)]
        self.O = [e(T, D) for _ in range(nb)]
        self.Z = [e(T, D) for _ in range(nb)]
        self.Hh = [e(T, Hd) for _ in range(nb)]
        self.Xn = e(T, D, dt=f32) if stash else self.X[(L + 1) % 2]   # no stash: the buffer block L-1 read from
        self.Pa = None
        self.X12 = e(T, 2 * Hd) if (swiglu and not stash) else None       # teacher pass: [x1 | x2] scratch
        self.LSE = [[e(s.n, cfg.heads, s.N, dt=f32) for s in sets] for _ in range(nb)]
        if stash:
            self.U1 = [e(T, 2 * Hd if swiglu else Hd) for _ in range(nb)]   # mlp: u1; swiglu: [x1 | x2]
            self.U2 = [e(T, D) for _ in range(nb)]
            # FP8: the attention projection before LayerScale 1, whose gradient the backward takes from it
            self.Pa = [e(T, D) for _ in range(nb)] if fp8 else None
            self.stats = [[e(T, dt=f32) for _ in range(4)] for _ in range(nb)]   # mean1, rstd1, mean2, rstd2
            self.fstats = [e(T, dt=f32), e(T, dt=f32)]

    def x_in(self, i):
        return self.X[i] if self.stash else self.X[i % 2]

    def x_out(self, i):
        return self.X[i + 1] if self.stash else self.X[(i + 1) % 2]

    def b(self, lst, i):
        return lst[i] if self.per_block else lst[0]


class HeadBufs:
    def __init__(self, cfg: EngineConfig, module: str, R: int, device, stash: bool):
        D = cfg.embed_dim
        Hh, Bn, K = cfg.head_dims(module)
        e = lambda *shape, dt=bf16: torch.empty(*shape, dtype=dt, device=device)
        self.A0 = e(R, D)
        self.H1, self.H2 = e(R, Hh), e(R, Hh)
        self.U3 = e(R, Bn, dt=f32)
        self.nrm = e(R, dt=f32)
        self.Yn = e(R, Bn)
        self.logits = e(R, K, dt=f32)
        if stash:
            self.Ua, self.Ub = e(R, Hh), e(R, Hh)
            self.dS = e(R, K)
            self.dYn, self.dU3 = e(R, Bn), e(R, Bn)
            self.dUb, self.dUa = e(R, Hh), e(R, Hh)
            self.dA0 = e(R, D, dt=f32)


class Net:
    """What one forward pass reads: a model's configuration and its weights.  `mods` maps "backbone" / "dino_head" /
    "ibot_head" to stores with w(name, teacher) / vec(name, teacher); `teacher` selects the EMA copy of a ParamStore.
    `fsdp` gathers a unit before it is read; None when the weights are resident (a FrozenStore).
    `fp8`: the block linears run in e4m3 (`linear`, `dgrad`) on scratch that belongs to this Net, so passes on other
    streams do not share it."""

    def __init__(self, cfg: EngineConfig, mods: dict, teacher: bool, fsdp=None, fp8: bool = False):
        self.cfg, self.mods, self.teacher, self.fsdp = cfg, mods, teacher, fsdp
        self.fp8 = bool(fp8)
        self._scratch = {}

    def acquire(self, module: str, unit: str):
        if self.fsdp is not None:
            self.fsdp.acquire(module, unit, self.teacher)

    def scratch(self, key: str, shape, dtype, device):
        """A [shape] view of this Net's buffer `key`, grown when a call needs more (stream order keeps reuse safe)."""
        n = math.prod(shape)
        b = self._scratch.get(key)
        if b is None or b.numel() < n:
            b = self._scratch[key] = torch.empty(n, dtype=dtype, device=device)
        return b[:n].view(*shape)


def _e4m3_rows(net: Net, which: str, x):
    """x (bf16 [R, C] view) quantized per row into net's scratch `which`: (e4m3 [R, C], fp32 scales [R])."""
    R, C = x.shape
    return ops.quant_rows(x, net.scratch("q" + which, (R, C), u8, x.device), net.scratch("s" + which, (R,), f32, x.device))


def linear(net: Net, x, W, out, **ep):
    """out = epilogue(x W) of a block linear (W [in, out]): the bf16 GEMM, or with net.fp8 x per token row and W per
    output column in e4m3 (W^T, K-major) on d3_gemm_e4m3.  `ep`: the epilogue arguments of ops.gemm."""
    if not net.fp8:
        return ops.gemm(x, W, out, b_mn=True, **ep)
    qx, sx = _e4m3_rows(net, "a", x)
    K, Nn = W.shape
    qw, sw = ops.quant_cols_t(W, net.scratch("qb", (Nn, K), u8, W.device), net.scratch("sb", (Nn,), f32, W.device))
    return ops.gemm_e4m3(qx, sx, qw, sw, out, **ep)


def dgrad(net: Net, dy, W, out, **ep):
    """out = epilogue(dy W^T), the input gradient of a block linear: bf16, or with net.fp8 the bf16 dy and W both per
    row in e4m3 (both K-major as they are stored, no transpose)."""
    if not net.fp8:
        return ops.gemm(dy, W, out, **ep)
    qd, sd = _e4m3_rows(net, "a", dy)
    qw, sw = _e4m3_rows(net, "b", W)
    return ops.gemm_e4m3(qd, sd, qw, sw, out, **ep)


def embed(net: Net, st: Stream, images, masks_list):
    """X0 = [cls | storage | patch embeddings (mask_token where masked)] of each crop set's bf16 NHWC images."""
    cfg, bb, teacher = net.cfg, net.mods["backbone"], net.teacher
    net.acquire("backbone", "embed")
    X0 = st.x_in(0)
    Wpe = bb.w("patch_embed/proj/kernel", teacher)
    for cs, img, masks in zip(st.sets, images, masks_list):
        tok = st.b(st.Xmid, 0)[cs.row0: cs.row0 + cs.n * cs.P]      # scratch until block 0 writes it
        ops.im2col(img, cs.patches, cfg.patch)
        ops.gemm(cs.patches, Wpe, tok, b_mn=True, bias=bb.vec("patch_embed/proj/bias", teacher))
        ops.assemble_tokens(tok, bb.vec("cls_token", teacher), bb.vec("mask_token", teacher), masks,
                            X0[cs.row0: cs.row0 + cs.T], cs.n, cs.P, cfg.embed_dim,
                            storage=bb.vec("storage_tokens", teacher) if cfg.n_storage else None)


def block_fwd(net: Net, st: Stream, i: int):
    """Block i (layers/block.py:195-201): st.x_in(i) -> st.x_out(i), stashing what the backward reads when st.stash."""
    cfg, bb, teacher = net.cfg, net.mods["backbone"], net.teacher
    D, H = cfg.embed_dim, cfg.heads
    net.acquire("backbone", f"blocks_{i}")
    p = f"blocks_{i}/"
    v = lambda n: bb.vec(p + n, teacher)
    lin = lambda x, n, out, **ep: linear(net, x, bb.w(p + n, teacher), out, **ep)
    X, Xmid, Xo = st.x_in(i), st.b(st.Xmid, i), st.x_out(i)
    Y, QKV, O, Z, Hh = st.b(st.Y, i), st.b(st.QKV, i), st.b(st.O, i), st.b(st.Z, i), st.b(st.Hh, i)
    stats = st.b(st.stats, i) if st.stash else [None] * 4
    ops.layernorm_fwd(X, v("norm1/scale"), v("norm1/bias"), Y, stats[0], stats[1], cfg.ln_eps)
    lin(Y, "attn/qkv/kernel", QKV, bias=v("attn/qkv/bias") if cfg.qkv_bias else None)
    lses = st.b(st.LSE, i)
    for cs, lse in zip(st.sets, lses):
        q = QKV[cs.row0: cs.row0 + cs.T]
        ops.rope(q, cs.sin, cs.cos, cs.N, cfg.prefix, D, cfg.head_dim)
        ops.attn_fwd(q, O[cs.row0: cs.row0 + cs.T], lse if st.stash else None, cs.n, cs.N, D, H)
    lin(O, "attn/proj/kernel", Xmid, bias=v("attn/proj/bias"), gamma=v("ls1/gamma"), resid=X,
        store_pre=st.b(st.Pa, i) if st.Pa is not None else None)
    ops.layernorm_fwd(Xmid, v("norm2/scale"), v("norm2/bias"), Z, stats[2], stats[3], cfg.ln_eps)
    if cfg.ffn_layer == "swiglu":
        # SwiGLUFFN (layers/ffn_layers.py:71-76): h = silu(z W1 + b1) * (z W2 + b2); x_out = x_mid + g2 * (h W3 + b3)
        Hs = cfg.swiglu_hidden
        X12 = st.b(st.U1, i) if st.stash else st.X12
        lin(Z, "mlp/w1/kernel", X12[:, :Hs], bias=v("mlp/w1/bias"))
        lin(Z, "mlp/w2/kernel", X12[:, Hs:], bias=v("mlp/w2/bias"))
        ops.swiglu_fwd(X12, Hh)
        lin(Hh, "mlp/w3/kernel", Xo, bias=v("mlp/w3/bias"), store_pre=st.b(st.U2, i) if st.stash else None,
            gamma=v("ls2/gamma"), resid=Xmid)
        return
    lin(Z, "mlp/Dense_0/kernel", Hh, bias=v("mlp/Dense_0/bias"), gelu=True, store_pre=st.b(st.U1, i) if st.stash else None)
    lin(Hh, "mlp/Dense_1/kernel", Xo, bias=v("mlp/Dense_1/bias"), gelu=cfg.mlp_second_act,
        store_pre=st.b(st.U2, i) if st.stash else None, gamma=v("ls2/gamma"), resid=Xmid)


def backbone_fwd(net: Net, st: Stream, images, masks_list):
    """embed, every block, then the final LayerNorm of every token into st.Xn."""
    cfg, bb, teacher = net.cfg, net.mods["backbone"], net.teacher
    embed(net, st, images, masks_list)
    for i in range(cfg.depth):
        block_fwd(net, st, i)
    XL = st.x_in(cfg.depth)
    net.acquire("backbone", "norm")
    fs = st.fstats if st.stash else [None, None]
    ops.layernorm_fwd(XL, bb.vec("norm/scale", teacher), bb.vec("norm/bias", teacher), st.Xn, fs[0], fs[1], cfg.ln_eps)


def head_fwd(net: Net, hb: HeadBufs, module: str, R: int, stash: bool):
    """DINOHead (layers/dino_head.py:65-85) on the first R rows of hb.A0 -> hb.Yn (bottleneck) and hb.logits."""
    hd, teacher = net.mods[module], net.teacher
    w = lambda n: hd.w(n, teacher)
    v = lambda n: hd.vec(n, teacher)
    r = lambda t: t[:R]
    net.acquire(module, "head")
    if R == 0:
        return
    ops.gemm(r(hb.A0), w("mlp/layers_0/kernel"), r(hb.H1), b_mn=True, bias=v("mlp/layers_0/bias"), gelu=True,
             store_pre=r(hb.Ua) if stash else None)
    ops.gemm(r(hb.H1), w("mlp/layers_2/kernel"), r(hb.H2), b_mn=True, bias=v("mlp/layers_2/bias"), gelu=True,
             store_pre=r(hb.Ub) if stash else None)
    ops.gemm(r(hb.H2), w("mlp/layers_4/kernel"), r(hb.U3), b_mn=True, bias=v("mlp/layers_4/bias"))
    ops.l2norm_fwd(r(hb.U3), r(hb.Yn), r(hb.nrm), 1e-12)
    ops.gemm(r(hb.Yn), w("last_layer/kernel"), r(hb.logits), b_mn=True)
