"""GPU: where does the multi-GPU step lose time against the single-GPU step?  (VERDICT r01 item 5: the scaling timeline.)

Run once as `python tools/scaling_breakdown.py` (1 GPU) and once under torchrun (N ranks) ON THE SAME BOX; rank 0 prints
  * the step time (CUDA events, steady state),
  * the step's phases (events at the phase boundaries of the real, two-stream step),
  * a single-stream instrumented step: every tensor-core GEMM launch timed, grouped by (kind, shape, scatter epilogue),
  * the time the compute stream spends WAITING for parameter gathers (acquire) — measured as the difference between the
    phase with and without the gathers queued (N > 1 only; acquire waits are timed through events recorded before /
    after each wait).
"""
import os, sys, time
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200"))
import torch

rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1)); lr_ = int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(lr_)
comm = None
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr_))
    from dinov3_jax.fsdp.runtime import Comm
    comm = Comm(dist.group.WORLD)
from dinov3_jax import _native, ops
from dinov3_jax.engine import Engine, config_for
from dinov3_jax.engine.synth import synthetic_batch, init_reference_like

_native.init(lr_)
arch = sys.argv[1] if len(sys.argv) > 1 else "vit_large"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 64
cfg = config_for(arch)
batch = synthetic_batch(cfg, B, seed=rank)
eng = Engine(cfg, B, device=f"cuda:{lr_}", max_masked=int(batch["mask_indices_list"].shape[0]), comm=comm)
init_reference_like(eng, seed=0)
eng.set_batch(batch)
hyper = dict(teacher_temp=0.04, lr=1e-4, wd=0.04, last_layer_lr=0.0, momentum=0.996)


def barrier():
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()


for _ in range(4):
    eng.train_step(None, **hyper)
barrier()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(6):
    eng.train_step(None, **hyper)
e1.record()
barrier()
step_ms = e0.elapsed_time(e1) / 6

# ---- phases of the real step
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
wrap("_head_bwd", lambda *a, **k: "heads bwd (+CE, KoLeo before)")
wrap("_block_bwd", lambda i, *a: "blocks bwd")
wrap("optimizer_step", lambda *a, **k: "grad fence + sumsq + adamw/ema")
# ---- exposed waits: events on the compute stream right before / after every acquire() (parameter gathers) and
# finish_grads() (push fence / reduce-scatter completion)
waits = []
if world > 1:
    _acq, _fin = eng.fsdp.acquire, eng.fsdp.finish_grads
    def acquire_timed(module, unit_name, teacher):
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); _acq(module, unit_name, teacher); b.record()
        waits.append((f"{'T' if teacher else 'S'}:{module}/{unit_name}", a, b))
    def finish_timed():
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); _fin(); b.record()
        waits.append(("finish_grads", a, b))
    eng.fsdp.acquire, eng.fsdp.finish_grads = acquire_timed, finish_timed
phase_runs = []
wait_runs = []
for rep in range(3):
    waits.clear()
    marks.clear()
    barrier()
    mark("start")
    eng.train_step(None, **hyper)
    mark("end")
    torch.cuda.synchronize()
    agg = {}
    for (n0, a), (n1, b) in zip(marks, marks[1:]):
        agg[n1] = agg.get(n1, 0.0) + a.elapsed_time(b)
    agg["TOTAL"] = marks[0][1].elapsed_time(marks[-1][1])
    phase_runs.append(agg)
    wait_runs.append([(n, x.elapsed_time(y)) for n, x, y in waits])
for k, o in owner.items():
    setattr(o, k, orig[k])
if world > 1:
    eng.fsdp.acquire, eng.fsdp.finish_grads = _acq, _fin
phases = {k: sorted(r[k] for r in phase_runs)[1] for k in phase_runs[0]}     # median of 3

# ---- single-stream instrumented step: GEMM launches grouped
overlap, eng.wgrad_overlap = eng.wgrad_overlap, False
scat_seen = []
orig_gemm_check = None
ops.PROFILE = []
# tag scatter launches: wrap ops.gemm to remember whether `scatter` was passed
_g = ops.gemm
def gemm_tagged(*a, **k):
    n0 = len(ops.PROFILE)
    r = _g(*a, **k)
    if len(ops.PROFILE) > n0:
        scat_seen.append(k.get("scatter") is not None)
    return r
ops.gemm = gemm_tagged
if hasattr(core, "ops"):
    core.ops.gemm = gemm_tagged
barrier()
s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
s0.record()
eng.train_step(None, **hyper)
s1.record()
torch.cuda.synchronize()
prof, ops.PROFILE = ops.PROFILE, None
ops.gemm = _g
eng.wgrad_overlap = overlap
single_ms = s0.elapsed_time(s1)
groups = {}
for p, sc in zip(prof, scat_seen + [False] * (len(prof) - len(scat_seen))):
    M, N, K, amn, bmn = p[4]
    kind = "wgrad" if (amn and bmn) else ("fwd" if bmn else "dgrad")
    key = (kind, M, N, K, "scatter" if sc else "")
    g = groups.setdefault(key, [0, 0.0, 0.0])
    g[0] += 1; g[1] += p[2].elapsed_time(p[3]); g[2] += p[1]
if rank == 0:
    print(f"== {arch} B={B}/GPU world={world} push={getattr(eng.fsdp, 'push', None) if world > 1 else None}")
    print(f"step {step_ms:.2f} ms   (single-stream instrumented step {single_ms:.2f} ms)")
    for k, v in phases.items():
        print(f"  phase {k:34s} {v:8.2f} ms")
    if wait_runs and wait_runs[-1]:
        wr = wait_runs[-1]
        print(f"  exposed waits on the compute stream (last run): gathers teacher {sum(v for n, v in wr if n.startswith('T:')):.2f} ms, "
              f"student {sum(v for n, v in wr if n.startswith('S:')):.2f} ms, finish_grads {sum(v for n, v in wr if n == 'finish_grads'):.2f} ms")
        print("   largest: " + ", ".join(f"{n} {v:.3f}" for n, v in sorted(wr, key=lambda t: -t[1])[:8]))
        print("   first 6: " + ", ".join(f"{n} {v:.3f}" for n, v in wr[:6]))
    tot = sum(g[1] for g in groups.values())
    print(f"  GEMM launches {len(prof)}, {tot:.2f} ms, {sum(g[2] for g in groups.values()) / tot / 1e9:.0f} TF/s")
    for key, g in sorted(groups.items(), key=lambda kv: -kv[1][1]):
        print(f"    {key[0]:6s} M={key[1]:6d} N={key[2]:6d} K={key[3]:6d} {key[4]:8s} n={g[0]:4d} {g[1]:8.2f} ms {g[2] / g[1] / 1e9:7.0f} TF/s")
if world > 1:
    torch.distributed.destroy_process_group()
