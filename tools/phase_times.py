"""GPU: time the phases of one ViT-L/16 B=64 step with CUDA events (teacher fwd, student fwd, heads+losses, backward, optimizer)."""
import os, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200"))
import torch
from dinov3_jax.engine import Engine, config_for
from dinov3_jax.engine.synth import synthetic_batch, init_reference_like
from dinov3_jax import ops

arch = sys.argv[1] if len(sys.argv) > 1 else "vit_large"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 64
cfg = config_for(arch)
batch = synthetic_batch(cfg, B, 0)
eng = Engine(cfg, B, max_masked=int(batch["mask_indices_list"].shape[0]))
init_reference_like(eng)
eng.set_batch(batch)
hyper = dict(teacher_temp=0.04, lr=1e-4, wd=0.04, last_layer_lr=0.0, momentum=0.996)
for _ in range(3): eng.train_step(None, **hyper)
marks = []
def mark(name):
    e = torch.cuda.Event(enable_timing=True); e.record(); marks.append((name, e))
import dinov3_jax.engine.core as core      # the forward pieces are module functions the engine calls by name
owner = {"backbone_fwd": core, "head_fwd": core, "sinkhorn": core, "_head_bwd": eng, "_block_bwd": eng, "optimizer_step": eng}
orig = {k: getattr(o, k) for k, o in owner.items()}
def wrap(name, label_fn):
    f = orig[name]
    def g(*a, **k):
        r = f(*a, **k); mark(label_fn(*a, **k)); return r
    setattr(owner[name], name, g)
wrap("backbone_fwd", lambda net, *a: f"backbone fwd {'teacher' if net.teacher else 'student'}")
wrap("head_fwd", lambda net, *a, **k: f"heads fwd {'teacher' if net.teacher else 'student'}")
wrap("sinkhorn", lambda *a, **k: "sinkhorn")
wrap("_head_bwd", lambda *a, **k: "heads bwd (+CE, before)")
wrap("_block_bwd", lambda i, *a: "blocks bwd")
wrap("optimizer_step", lambda *a, **k: "optimizer (sumsq+adamw+ema)")
mark("start")
eng.train_step(None, **hyper)
mark("end")
torch.cuda.synchronize()
agg = {}
for (n0, e0), (n1, e1) in zip(marks, marks[1:]):
    agg[n1] = agg.get(n1, 0.0) + e0.elapsed_time(e1)
tot = marks[0][1].elapsed_time(marks[-1][1])
print(f"{arch} B={B}: step {tot:.2f} ms")
for k, v in agg.items():
    print(f"  {k:34s} {v:8.2f} ms  {100*v/tot:5.1f}%")
