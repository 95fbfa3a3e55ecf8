"""GPU: dense-feature extraction, DinoVisionTransformer.get_intermediate_layers(x, n=4, reshape=True, norm=True), on
random weights for three backbones at 224^2 (B=64), 512^2 (B=16) and 1024^2 (B=4).  Prints images/s, peak memory, the
d3_layernorm_tokens_out time and GB/s (its algorithmic bytes: X read once, the outputs written once) against the
H100 SXM's 3.35 TB/s, and, when transformers is importable, the same call through Hugging Face's DINOv3ViTModel in bf16
with SDPA (the last four hidden states, its final norm, reshaped) as a baseline.  Timed calls alternate between the two
after a warm-up of every shape.

    python tools/bench_features.py [--iters 5] [--configs vitl,vithp,vit7b] [--sizes 224,512,1024]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dinov3-jax_b200"))
import torch

from dinov3_jax import _native, ops
from dinov3_jax.models import DinoVisionTransformer
from gpu_timing import card, cuda_ms, cuda_ms_each

f32, bf16 = torch.float32, torch.bfloat16
HBM_BYTES_PER_S = 3.35e12                 # H100 SXM data sheet
CONFIGS = {   # name: (embed_dim, blocks, heads, ffn_layer, ffn_ratio, mask_k_bias, norm_layer)
    "vitl": ("ViT-L/16 mlp mask_k_bias", 1024, 24, 16, "mlp", 4.0, True, "layernormbf16"),
    "vithp": ("ViT-H+/16 swiglu", 1280, 32, 20, "swiglu", 6.0, False, "layernormbf16"),
    "vit7b": ("vit_7b width, 4 blocks, swiglu64", 4096, 4, 32, "swiglu64", 3.0, True, "layernormbf16"),
}
SIZES = {224: 64, 512: 16, 1024: 4}
R, PATCH = 4, 16


def random_tree(D, L, ffn, ratio, g):
    rnd = lambda *s, std=0.02: (torch.randn(*s, device="cuda", generator=g) * std)
    ones = lambda k: 1 + rnd(k, std=0.05)
    hidden = int(D * ratio)
    t = {"patch_embed": {"proj": {"kernel": rnd(PATCH, PATCH, 3, D), "bias": rnd(D)}}, "cls_token": rnd(1, 1, D),
         "mask_token": rnd(1, D), "storage_tokens": rnd(1, R, D), "norm": {"scale": ones(D), "bias": rnd(D)}}
    for i in range(L):
        b = {"norm1": {"scale": ones(D), "bias": rnd(D)}, "norm2": {"scale": ones(D), "bias": rnd(D)},
             "attn": {"qkv": {"kernel": rnd(D, 3 * D), "bias": rnd(3 * D)}, "proj": {"kernel": rnd(D, D), "bias": rnd(D)}},
             "ls1": {"gamma": ones(D)}, "ls2": {"gamma": ones(D)}}
        if ffn == "mlp":
            b["mlp"] = {"Dense_0": {"kernel": rnd(D, hidden), "bias": rnd(hidden)},
                        "Dense_1": {"kernel": rnd(hidden, D), "bias": rnd(D)}}
        else:
            align = {"swiglu": 8, "swiglu64": 64}[ffn]
            d = int(hidden * 2 / 3)
            Hs = d + (-d % align)
            b["mlp"] = {"w1": {"kernel": rnd(D, Hs), "bias": rnd(Hs)}, "w2": {"kernel": rnd(D, Hs), "bias": rnd(Hs)},
                        "w3": {"kernel": rnd(Hs, D), "bias": rnd(D)}}
        t[f"blocks_{i}"] = b
    return t


def hf_model(D, L, H, ffn, ratio, mask_k_bias, size):
    try:
        from transformers.models.dinov3_vit import DINOv3ViTConfig, DINOv3ViTModel
    except ImportError:
        return None
    swiglu = ffn != "mlp"
    hidden = int(D * ratio)
    if swiglu:
        d = int(hidden * 2 / 3)
        hidden = d + (-d % {"swiglu": 8, "swiglu64": 64}[ffn])
    cfg = DINOv3ViTConfig(patch_size=PATCH, hidden_size=D, intermediate_size=hidden, num_hidden_layers=L, num_attention_heads=H,
                          hidden_act="silu" if swiglu else "gelu", layer_norm_eps=1e-5, image_size=size, key_bias=not mask_k_bias,
                          num_register_tokens=R, use_gated_mlp=swiglu, attn_implementation="sdpa")
    return DINOv3ViTModel(cfg).to(device="cuda", dtype=bf16).eval()


def hf_features(model, x_nchw, n=4):
    out = model(pixel_values=x_nchw, output_hidden_states=True)
    B, _, H, W = x_nchw.shape
    feats = []
    for h in out.hidden_states[-n:]:
        p = model.norm(h)[:, 1 + R:]
        feats.append(p.reshape(B, H // PATCH, W // PATCH, -1).permute(0, 3, 1, 2).contiguous())
    return feats


def kernel_time(B, N, D, Hp, Wp, out_dtype, channels_first, iters=20):
    """Median d3_layernorm_tokens_out time over `iters` launches, L2 flushed before each; returns (ms, bytes)."""
    X = torch.randn(B, N, D, device="cuda")
    sc, bi = torch.ones(D, device="cuda"), torch.zeros(D, device="cuda")
    cls, st = torch.empty(B, D, dtype=out_dtype, device="cuda"), torch.empty(B, R, D, dtype=out_dtype, device="cuda")
    pt = torch.empty(*((B, D, Hp, Wp) if channels_first else (B, Hp * Wp, D)), dtype=out_dtype, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    call = lambda: ops.layernorm_tokens_out(X, cls, st, pt, Hp, Wp, norm=(sc, bi), eps=1e-5, channels_first=channels_first)
    ts = sorted(cuda_ms_each(call, iters, 1, before=flush.zero_))
    nbytes = B * N * D * (4 + out_dtype.itemsize) + 4 * D * 4
    return ts[len(ts) // 2], nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--sizes", default=",".join(map(str, SIZES)))
    ap.add_argument("--no-hf", action="store_true")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _native.init(0)
    print(f"card: {card()}")
    g = torch.Generator(device="cuda").manual_seed(0)
    for key in args.configs.split(","):
        name, D, L, H, ffn, ratio, mkb, norm_layer = CONFIGS[key]
        model = DinoVisionTransformer(random_tree(D, L, ffn, ratio, g), patch_size=PATCH, embed_dim=D, n_blocks=L, num_heads=H,
                                      ffn_ratio=ratio, ffn_layer=ffn, mask_k_bias=mkb, n_storage_tokens=R, norm_layer=norm_layer)
        print(f"\n{name}: D={D} blocks={L} heads={H} ffn={ffn} ratio={ratio} R={R}")
        for size in map(int, args.sizes.split(",")):
            B = SIZES[size]
            Hp = size // PATCH
            x = torch.randn(B, size, size, 3, device="cuda").to(bf16)
            ours = lambda: model.get_intermediate_layers(x, n=4, reshape=True, norm=True)
            hf = None if args.no_hf else hf_model(D, L, H, ffn, ratio, mkb, size)
            x_nchw = x.permute(0, 3, 1, 2).contiguous()
            theirs = (lambda: hf_features(hf, x_nchw)) if hf is not None else None
            with torch.no_grad():
                for fn in (ours, theirs):           # warm-up of every shape
                    if fn is not None:
                        fn(); fn(); torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                ours(); torch.cuda.synchronize()
                peak_ours = torch.cuda.max_memory_allocated() - base
                peak_hf = None
                if theirs is not None:
                    torch.cuda.reset_peak_memory_stats()
                    theirs(); torch.cuda.synchronize()
                    peak_hf = torch.cuda.max_memory_allocated() - base
                t_ours, t_hf = [], []
                for _ in range(args.iters):         # alternate the two, one call each; both were warmed up above
                    t_ours.append(cuda_ms(ours, 1, 0))
                    if theirs is not None:
                        t_hf.append(cuda_ms(theirs, 1, 0))
            med = lambda ts: sorted(ts)[len(ts) // 2]
            line = (f"  {size:4d}^2 B={B:2d}: ours {med(t_ours):8.2f} ms  {B / med(t_ours) * 1e3:8.1f} img/s  "
                    f"peak +{peak_ours / 2**20:7.0f} MiB over the weights")
            if theirs is not None:
                line += (f" | HF bf16 sdpa {med(t_hf):8.2f} ms  {B / med(t_hf) * 1e3:8.1f} img/s  "
                         f"peak +{peak_hf / 2**20:7.0f} MiB")
            print(line)
            N = 1 + R + Hp * Hp
            for dt in (f32, bf16):
                for cf in (True, False):
                    ms, nb = kernel_time(B, N, D, Hp, Hp, dt, cf)
                    print(f"      d3_layernorm_tokens_out {'fp32' if dt == f32 else 'bf16'} "
                          f"{'channels-first' if cf else 'channels-last '}: {ms * 1e3:7.1f} us  {nb / ms / 1e6:7.0f} GB/s  "
                          f"{nb / ms / 1e-3 / HBM_BYTES_PER_S * 100:5.1f}% of 3.35 TB/s")
            del hf, theirs
            torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()
    print(f"\ncard: {card()}")


if __name__ == "__main__":
    main()
