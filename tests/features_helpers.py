"""CPU restatement (fp32 / fp64) of upstream DINOv3's `get_intermediate_layers` (models/vision_transformer.py:262-313,
read as intended: the reference's own method cannot run, DESIGN.md §2), built from the oracle's layers, and the
parameter-tree helpers the feature tests share."""
import torch

from oracle.arch import ModelCfg
from oracle.model import Emu, block_forward, layer_norm, patch_embed, rope_sincos


def prepare_tokens(P: dict, x, cfg: ModelCfg):
    """models/vision_transformer.py:173-203 without masks: [B, H, W, 3] -> [B, 1 + R + P, D] and the RoPE (sin, cos)."""
    t, (Hp, Wp) = patch_embed(P, x, cfg, Emu(False))
    parts = [(P["cls_token"] + 0 * P["mask_token"]).expand(t.shape[0], -1, -1)]
    if cfg.n_storage:
        parts.append(P["storage_tokens"].to(t.dtype).expand(t.shape[0], -1, -1))
    t = torch.cat(parts + [t], dim=1)
    return t, rope_sincos(Hp, Wp, cfg.head_dim, cfg.rope_base, t.dtype)


def final_norm(P: dict, t, cfg: ModelCfg, untie_cls_and_patch_norms: bool = False):
    """models/vision_transformer.py:223-236 (deterministic branch): `norm` over every token, or `cls_norm` over the
    1 + R prefix tokens and `norm` over the patches.  Returns (cls [B, D], storage [B, R, D], patches [B, P, D])."""
    R = cfg.n_storage
    xn = layer_norm(t, P["norm/scale"], P["norm/bias"], cfg.ln_eps)
    pre = layer_norm(t[:, :1 + R], P["cls_norm/scale"], P["cls_norm/bias"], cfg.ln_eps) if untie_cls_and_patch_norms \
        else xn[:, :1 + R]
    return pre[:, 0], pre[:, 1:], xn[:, 1 + R:]


def intermediate_layers(P: dict, x, n, cfg: ModelCfg, norm: bool = True, untie_cls_and_patch_norms: bool = False):
    """x [B, H, W, 3]; n = the last n blocks (int) or a list of block indices.  Returns, in block order, one dict per
    selected block with "cls" [B, D], "storage" [B, R, D] and "patches" [B, P, D] (norm=False: the raw block output)."""
    t, (s, c) = prepare_tokens(P, x, cfg)
    take = range(cfg.depth - n, cfg.depth) if isinstance(n, int) else list(n)
    R, outs = cfg.n_storage, []
    for i in range(cfg.depth):
        t = block_forward(P, f"blocks_{i}/", t, s, c, cfg, Emu(False))
        if i in take:
            parts = final_norm(P, t, cfg, untie_cls_and_patch_norms) if norm else (t[:, 0], t[:, 1:1 + R], t[:, 1 + R:])
            outs.append(dict(zip(("cls", "storage", "patches"), parts)))
    assert len(outs) == len(take), f"only {len(outs)} / {len(take)} blocks found"
    return outs


def tree(flat: dict, device=None) -> dict:
    """flat "a/b/c" -> nested dict (optionally moved to `device`)."""
    out = {}
    for k, v in flat.items():
        cur = out
        parts = k.split("/")
        for p in parts[:-1]:
            cur = cur.setdefault(p, {})
        cur[parts[-1]] = v if device is None else v.to(device)
    return out


def add_norm(bp: dict, name: str, D: int, key: int, dtype=torch.float64) -> dict:
    """bp plus a non-trivial LayerNorm `name` (scale near 1, small bias) from oracle.model.hash_uniform."""
    from oracle.model import hash_uniform
    u = torch.from_numpy(hash_uniform(2 * D, key)).to(dtype)
    return {**bp, f"{name}/scale": 1.0 + 0.2 * u[:D], f"{name}/bias": 0.1 * u[D:]}
