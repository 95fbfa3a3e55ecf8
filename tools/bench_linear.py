"""GPU: one linear-probe iteration at the ImageNet-1k shape (dinov3_jax/eval/linear.py): ViT-L/16, B = 128, the
default grid of 52 classifiers (n in {1, 4} x avgpool in {False, True} x 13 learning rates), 1 000 classes.

Timed apart, with CUDA events after a warm-up:
  * the train crop (d3_train_resized_crop, bf16 out) of 128 packed 500 x 375 images with seeded RandomResizedCrop
    boxes and flips;
  * the ViT-L feature forward (get_intermediate_layers of the last 4 blocks, random weights) and the input rows
    (d3_pool_tokens + d3_linear_inputs);
  * the head work of LinearClassifiers.step: the logit GEMMs, the cross-entropy, the weight-gradient GEMMs, the bias
    column sums and SGD.
The baseline is a torch restatement of the DINOv2 module on the same input rows (as fp32): 52 nn.Linear heads, the
sum of F.cross_entropy, torch.optim.SGD(momentum=0.9, foreach=True) with one lr per head and CosineAnnealingLR.  Both
sides start from the same weights and take the same batches; the relative L2 difference of their weights is printed
per classifier group, against the 1e-3 of the GPU test's same-rounding restatement.

Prints the card and its power limit with the numbers.   python tools/bench_linear.py [--iters N]
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [os.path.join(ROOT, "dinov3-jax_b200"), ROOT]
import torch

from dinov3_jax import ops
from dinov3_jax.eval.linear import LinearClassifiers, sample_train_boxes, write_linear_inputs
from gpu_timing import card, cuda_ms

bf16, f32 = torch.bfloat16, torch.float32
B, C, D, S = 128, 1000, 1024, 224


def bench_crop(iters):
    from dinov3_jax.eval.knn import _pack
    g = torch.Generator().manual_seed(0)
    imgs = [torch.randint(0, 256, (375, 500, 3), generator=g, dtype=torch.uint8).numpy() for _ in range(B)]
    flat, desc, _ = _pack([(im, 0) for im in imgs])
    boxes = sample_train_boxes(torch.Generator().manual_seed(1), [(375, 500)] * B)
    taps = ops.train_max_taps(boxes.tolist(), S)
    flat, desc, bx = flat.cuda(), desc.cuda(), boxes.cuda()
    out = torch.empty(B, S, S, 3, dtype=bf16, device="cuda")
    ms = cuda_ms(lambda: ops.train_resized_crop(flat, desc, bx, out, max_taps=taps, mean=(0.485, 0.456, 0.406),
                                                std=(0.229, 0.224, 0.225)), iters, 2)
    print(f"train crop 500x375 -> RandomResizedCrop 224^2 + flip: {ms:.3f} ms per batch of {B}, "
          f"{B / ms * 1e3:,.0f} images/s")
    return out


def bench_features(images, out, iters):
    from dinov3_jax.checkpointer import tree_from_flat
    from dinov3_jax.models import DinoVisionTransformer
    from oracle.arch import ModelCfg
    from oracle.model import init_backbone
    cfg = ModelCfg(embed_dim=D, depth=24, heads=16)
    model = DinoVisionTransformer(tree_from_flat(init_backbone(cfg, torch.Generator().manual_seed(0))), embed_dim=D,
                                  n_blocks=24, num_heads=16)
    ms = cuda_ms(lambda: write_linear_inputs(model, images, 4, out), iters, 2)
    print(f"ViT-L/16 features (last 4 blocks' class tokens + patch mean) at 224^2: {ms:.1f} ms per batch of {B}, "
          f"{B / ms * 1e3:,.0f} images/s")
    return ms


def head_flops(clf):
    return sum(2 * 2 * B * cnt * clf.Cp * w for _, cnt, _, w in clf.groups)


def bench_heads(iters):
    total = 10 * 1250
    clf = LinearClassifiers(D, C, B, total, seed=0, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(2)
    xs = [torch.randn(B, clf.width, device="cuda", generator=g).to(bf16) for _ in range(4)]
    ys = [torch.randint(0, C, (B,), device="cuda", generator=g) for _ in range(4)]
    init = clf.state_dict()
    # torch restatement of the DINOv2 module (fp32), same initial weights
    heads = []
    for (n, a, _), name in zip(clf.grid, clf.names):
        lin = torch.nn.Linear((n + int(a)) * D, C, device="cuda")
        with torch.no_grad():
            lin.weight.copy_(init[name]["weight"])
            lin.bias.zero_()
        heads.append(lin)
    opt = torch.optim.SGD([{"params": h.parameters(), "lr": lr * B / 256} for h, (_, _, lr) in zip(heads, clf.grid)],
                          momentum=0.9, weight_decay=0, foreach=True)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, total, eta_min=0)

    def torch_step(t):
        x, y = xs[t % 4].float(), ys[t % 4]
        loss = sum(torch.nn.functional.cross_entropy(h(x[:, (4 - n) * D:(4 + int(a)) * D]), y)
                   for h, (n, a, _) in zip(heads, clf.grid))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        sched.step()

    steps = [0]

    def ours():
        clf.step(xs[steps[0] % 4], ys[steps[0] % 4], steps[0])
        steps[0] += 1

    tq = [0]

    def theirs():
        torch_step(tq[0])
        tq[0] += 1

    # the same 6 steps on both sides, then the weights compared
    for _ in range(6):
        ours()
        theirs()
    torch.cuda.synchronize()
    got = clf.state_dict()
    worst = {}
    for h, (n, a, _), name in zip(heads, clf.grid, clf.names):
        rel = ((got[name]["weight"] - h.weight.detach().cpu()).norm() / h.weight.detach().cpu().norm()).item()
        key = f"n={n} avgpool={a}"
        worst[key] = max(worst.get(key, 0.0), rel)
    print("weights after 6 steps, max relative L2 difference to the torch fp32 module per window: " +
          ", ".join(f"{k}: {v:.2e}" for k, v in worst.items()) +
          f" ({'within' if max(worst.values()) <= 1e-3 else 'ABOVE'} 1e-3)")
    ms = cuda_ms(ours, iters, 2)
    ms_t = cuda_ms(theirs, iters, 2)
    fl = head_flops(clf)
    print(f"head work (52 classifiers, {C} classes, B = {B}): {ms:.2f} ms per step "
          f"({fl / 1e9:.1f} GFLOP of GEMMs, {fl / ms / 1e9:.0f} TFLOP/s over the whole step); torch baseline "
          f"{ms_t:.2f} ms ({ms_t / ms:.2f}x)")
    return ms


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=20)
    a = p.parse_args()
    assert torch.cuda.is_available(), "bench_linear measures on the GPU"
    from dinov3_jax import _native
    _native.init(0)
    torch.backends.cuda.matmul.allow_tf32 = False
    print(card())
    images = bench_crop(a.iters)
    out = torch.empty(B, 5 * D, dtype=bf16, device="cuda")
    ms_f = bench_features(images, out, max(3, a.iters // 4))
    ms_h = bench_heads(a.iters)
    print(f"one probe iteration without decoding: features {ms_f:.1f} ms + heads {ms_h:.2f} ms "
          f"(heads {100 * ms_h / (ms_f + ms_h):.1f} % of it)")


if __name__ == "__main__":
    main()
