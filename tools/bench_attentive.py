"""GPU: the attentive probe (eval/attentive.py) at the ViT-L/16 video shape: 16 clips x 16 frames at 224^2 (P = 196
tokens per frame, N = 3 136 per clip, D = 1024, H = 16), 400 classes, on seeded synthetic bf16 tokens.

Reports:
- the backbone's features per iteration: a random-weight ViT-L/16 (24 blocks) through get_intermediate_layers(n=1,
  bf16) on the 256 frames of one batch;
- each pooling kernel (d3_atp_pool_fwd, d3_atp_pool_bwd) and the GB/s it reaches over the token bytes it must read
  (B * T * P * D * 2 bytes, once per pass);
- the whole probe step (forward, backward, AdamW);
- a torch restatement of the unfolded probe on the same tokens and parameters: nn.Linear keys and values over every
  token, scaled_dot_product_attention, bf16 autocast, autograd and torch.optim.AdamW (fused=False); its step time
  and the relative L2 difference of every parameter gradient of the two sides.
The card, its power limit and maximum SM clock are printed with the numbers.

python tools/bench_attentive.py [--iters 20] [--no-backbone]
"""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT, os.path.join(ROOT, "tests")]
import torch
import torch.nn.functional as F

from dinov3_jax import _native, ops
from dinov3_jax.eval.attentive import AttentiveProbe
from gpu_timing import card, cuda_ms

B, T, P, D, H, C = 16, 16, 196, 1024, 16, 400


class TorchProbe(torch.nn.Module):
    """The probe as written: keys and values of every token, SDPA, the MLP block and the classifier."""

    def __init__(self, params):
        super().__init__()
        self.p = torch.nn.ParameterDict({k: torch.nn.Parameter(v.detach().clone()) for k, v in params.items()})

    def forward(self, x):
        p, (n, N, _) = self.p, x.shape
        dh = D // H
        u = x.float() + p["e"].repeat_interleave(N // T, 0)[None]
        y = F.layer_norm(u, (D,), p["g1"], p["b1"], 1e-6)
        q = F.linear(p["q0"], p["Wq"], p["bq"]).view(1, H, 1, dh).expand(n, H, 1, dh)
        k = F.linear(y, p["Wk"]).view(n, N, H, dh).transpose(1, 2)
        v = F.linear(y, p["Wv"], p["bv"]).view(n, N, H, dh).transpose(1, 2)
        a = F.scaled_dot_product_attention(q, k, v).reshape(n, D)
        z = p["q0"] + F.linear(a, p["Wo"], p["bo"])
        z = z + F.linear(F.gelu(F.linear(F.layer_norm(z, (D,), p["g2"], p["b2"], 1e-6), p["W1"], p["bf1"])),
                         p["W2"], p["bf2"])
        return F.linear(z, p["Wc"], p["bc"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--no-backbone", action="store_true")
    args = ap.parse_args()
    _native.init()
    out = {"card": card(), "shape": {"clips": B, "frames": T, "tokens_per_frame": P, "D": D, "heads": H, "classes": C}}
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn(B, T * P, D, generator=g, device="cuda") * 2).bfloat16()
    y = torch.randint(0, C, (B,), generator=g, device="cuda")
    token_bytes = x.numel() * 2
    if not args.no_backbone:
        from dinov3_jax.models import DinoVisionTransformer
        from features_helpers import tree
        from oracle.arch import ModelCfg
        from oracle.model import init_backbone
        flat = init_backbone(ModelCfg(embed_dim=D, depth=24, heads=H), torch.Generator().manual_seed(0))
        model = DinoVisionTransformer(tree(flat), embed_dim=D, n_blocks=24, num_heads=H)
        images = torch.randn(B * T, 224, 224, 3, generator=g, device="cuda").bfloat16()
        ms = cuda_ms(lambda: model.get_intermediate_layers(images, n=1, out_dtype=torch.bfloat16), 3, 2)
        out["backbone_ms_per_iteration"] = round(ms, 2)
        del model
    probe = AttentiveProbe(D, H, T, C, B, 1000, lr=1e-3, seed=0, device="cuda")
    probe.gradients(x, y)
    Pm = probe.params
    fwd = lambda: ops.atp_pool_fwd(x, T, Pm["e"], Pm["g1"], Pm["b1"], probe.kt, probe.ybar, probe.lse)
    bwd = lambda: ops.atp_pool_bwd(x, T, Pm["e"], Pm["g1"], Pm["b1"], probe.kt, probe.lse, probe.ybar, probe.dybar,
                                   probe.dkt, probe.grads["g1"], probe.grads["b1"], probe.grads["e"])
    for name, fn in (("pool_fwd", fwd), ("pool_bwd", bwd)):
        ms = cuda_ms(fn, args.iters, 3)
        out[name] = {"ms": round(ms, 4), "GB_per_s_over_token_bytes": round(token_bytes / ms / 1e6, 1)}
    out["token_bytes"] = token_bytes
    # the gradients of both sides at the same parameters, before any step
    ref = TorchProbe({k: v.clone() for k, v in Pm.items() if k not in ("Wc", "bc")} |
                     {"Wc": Pm["Wc"][:C].clone(), "bc": Pm["bc"][:C].clone()}).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = F.cross_entropy(ref(x).float(), y)
    loss.backward()
    probe.gradients(x, y)
    diff = {}
    for k, prm in ref.p.items():
        mine = probe.grads[k][:C] if k in ("Wc", "bc") else probe.grads[k]
        diff[k] = float((mine.double() - prm.grad.double()).norm() / prm.grad.double().norm())
    out["grad_rel_l2_vs_torch"] = {k: f"{v:.2e}" for k, v in diff.items()}
    out["probe_step_ms"] = round(cuda_ms(lambda: probe.step(x, y, 0), args.iters, 3), 3)
    opt = torch.optim.AdamW(ref.parameters(), lr=1e-3, weight_decay=0.01, fused=False)

    def torch_step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            l = F.cross_entropy(ref(x).float(), y)
        l.backward()
        opt.step()

    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out["torch_unfolded_step_ms"] = round(cuda_ms(torch_step, args.iters, 3), 3)
    out["torch_unfolded_step_peak_extra_GB"] = round((torch.cuda.max_memory_allocated() - base) / 1e9, 2)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    probe.step(x, y, 0)
    torch.cuda.synchronize()
    out["probe_step_peak_extra_GB"] = round((torch.cuda.max_memory_allocated() - base) / 1e9, 3)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
