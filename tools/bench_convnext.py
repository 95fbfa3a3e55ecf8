"""ConvNeXt forward throughput: this project's ConvNeXt.forward_features against Hugging Face's DINOv3ConvNextModel on the
same GPU, in fp32 and under bf16 autocast, with the outputs compared; and the bandwidth of d3_dwconv7_layernorm at
every stage shape.  Weights are random (upstream_state_dict, the tests' generator); timing is CUDA events around K
forward passes after W warm-up passes.  One JSON line per measurement on stdout; --out FILE also writes them all
as one JSON list.

    python tools/bench_convnext.py [--sizes tiny,small,base,large] [--res 224,512] [--batch 16] [--steps 10]
                                   [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "dinov3-jax_b200"), ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from gpu_timing import card, cuda_ms  # noqa: E402

HBM_TBS = 3.35     # H100 SXM HBM3 peak


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _hf_state_dict(sd):
    from test_convnext_cpu import _hf_state_dict
    return _hf_state_dict(sd)


def bench_model(size, res, B, steps, warmup):
    from transformers import DINOv3ConvNextConfig, DINOv3ConvNextModel
    from convnext_helpers import upstream_state_dict
    from dinov3_jax.checkpointer import convert_convnext_torch_hub_state_dict
    from dinov3_jax.models import ConvNeXt, convnext_sizes
    arch = convnext_sizes[size]
    sd = upstream_state_dict(arch["depths"], arch["dims"], seed=0, dtype=torch.float32)
    ours = ConvNeXt(convert_convnext_torch_hub_state_dict(sd), **arch)
    hf = DINOv3ConvNextModel(DINOv3ConvNextConfig(depths=arch["depths"], hidden_sizes=arch["dims"], layer_norm_eps=1e-6,
                                                  hidden_act="gelu")).cuda().eval()
    hf.load_state_dict(_hf_state_dict(sd), strict=True)
    x = torch.randn(B, res, res, 3, generator=torch.Generator().manual_seed(res)).cuda()
    xc = x.permute(0, 3, 1, 2).contiguous()
    with torch.no_grad():
        ff = ours.forward_features(x)
        ref = hf(pixel_values=xc).last_hidden_state
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ref_bf = hf(pixel_values=xc).last_hidden_state
        mine = torch.cat([ff["x_norm_clstoken"][:, None], ff["x_norm_patchtokens"]], dim=1)
        t_ours = cuda_ms(lambda: ours.forward_features(x), steps, warmup)
        t_fp32 = cuda_ms(lambda: hf(pixel_values=xc), steps, warmup)

        def hf_bf16():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                hf(pixel_values=xc)
        t_bf16 = cuda_ms(hf_bf16, steps, warmup)
    del hf
    torch.cuda.empty_cache()
    return {"kind": "model", "size": size, "res": res, "batch": B, "ours_ms": round(t_ours, 3),
            "hf_fp32_ms": round(t_fp32, 3), "hf_bf16_autocast_ms": round(t_bf16, 3),
            "ours_img_per_s": round(B / t_ours * 1e3, 1), "speedup_vs_fp32": round(t_fp32 / t_ours, 2),
            "speedup_vs_bf16": round(t_bf16 / t_ours, 2), "rel_err_vs_hf_fp32": _rel(mine, ref),
            "rel_err_hf_bf16_vs_hf_fp32": _rel(ref_bf.float(), ref)}


def bench_dwconv(C, H, W, n, steps, warmup):
    from dinov3_jax import ops
    X = torch.randn(n, H, W, C, device="cuda")
    w, wb = torch.randn(49, C, device="cuda") / 7, torch.randn(C, device="cuda")
    sc, bi = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    Y = torch.empty(n * H * W, C, dtype=torch.bfloat16, device="cuda")
    t = cuda_ms(lambda: ops.dwconv7_layernorm(X, w, wb, sc, bi, Y), steps, warmup)
    nbytes = X.numel() * 4 + Y.numel() * 2
    tbs = nbytes / (t * 1e-3) / 1e12
    return {"kind": "dwconv7_layernorm", "n": n, "H": H, "W": W, "C": C, "us": round(t * 1e3, 2),
            "TB_s": round(tbs, 3), "pct_of_3.35TB_s": round(100 * tbs / HBM_TBS, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="tiny,small,base,large")
    ap.add_argument("--res", default="224,512")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write every result as one JSON list to this file")
    a = ap.parse_args()
    from dinov3_jax import _native
    _native.init(0)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    rows = [dict(kind="device", **card())]
    print(json.dumps(rows[0]), flush=True)
    from dinov3_jax.models import convnext_sizes
    for res in [int(r) for r in a.res.split(",")]:
        for size in a.sizes.split(","):
            rows.append(bench_model(size, res, a.batch, a.steps, a.warmup))
            print(json.dumps(rows[-1]), flush=True)
    # every (channels, stage) a released size has: the map is res / 4 / 2^stage on a side
    shapes = sorted({(C, i) for s in convnext_sizes.values() for i, C in enumerate(s["dims"])})
    for res in [int(r) for r in a.res.split(",")]:
        for C, stage in shapes:
            hw = res // (4 << stage)
            rows.append(bench_dwconv(C, hw, hw, a.batch, 4 * a.steps, a.warmup))
            print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
