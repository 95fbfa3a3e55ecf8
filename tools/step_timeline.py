"""GPU: kernel timeline of steady-state training steps (CUPTI through torch.profiler; there is no nsys in the image).

  python tools/step_timeline.py [arch] [B]                       (1 GPU)
  torchrun --nproc-per-node N tools/step_timeline.py [arch] [B]  (N ranks; rank 0 writes)

Writes profile_out/timeline_w<world>.json: every GPU activity (kernels, memcpys, memsets) of 2 steps with stream, start,
duration; and prints a summary: busy time per stream, idle gaps on the compute stream, time per kernel name.
`tools/timeline_diff.py a.json b.json` compares two of them (1 GPU vs N GPUs: where the extra milliseconds go).
"""
import json, os, sys
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
from dinov3_jax import _native
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
for _ in range(4):
    eng.train_step(None, **hyper)
torch.cuda.synchronize()
if world > 1:
    torch.distributed.barrier()
from torch.profiler import profile, ProfilerActivity
NSTEP = 3
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(NSTEP):
        eng.train_step(None, **hyper)
    torch.cuda.synchronize()
tmp = f"/tmp/trace_{rank}.json"
prof.export_chrome_trace(tmp)
if rank == 0:
    ev = json.load(open(tmp))["traceEvents"]
    acts = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    acts.sort(key=lambda e: e["ts"])
    rows = [{"name": e["name"][:96], "cat": e["cat"], "stream": e.get("args", {}).get("stream"), "ts": e["ts"], "dur": e["dur"]}
            for e in acts]
    # steps are delimited by the AdamW kernels of the backbone (the largest adamw launch ends a step)
    ends = [i for i, r in enumerate(rows) if "adamw_ema" in r["name"]]
    os.makedirs(os.path.join(ROOT, "profile_out"), exist_ok=True)
    out = os.path.join(ROOT, "profile_out", f"timeline_w{world}.json")
    json.dump({"world": world, "arch": arch, "B": B, "nstep": NSTEP, "rows": rows}, open(out, "w"))
    t0, t1 = rows[0]["ts"], max(r["ts"] + r["dur"] for r in rows)
    print(f"== {arch} B={B} world={world}: {len(rows)} GPU activities over {(t1 - t0) / 1e3:.2f} ms = {(t1 - t0) / 1e3 / NSTEP:.2f} ms/step (under CUPTI)")
    streams = {}
    for r in rows:
        streams.setdefault(r["stream"], []).append(r)
    main = max(streams, key=lambda s: sum(r["dur"] for r in streams[s]))
    for s_, rs in sorted(streams.items(), key=lambda kv: -sum(r["dur"] for r in kv[1])):
        print(f"  stream {s_}: {len(rs):5d} activities, busy {sum(r['dur'] for r in rs) / 1e3 / NSTEP:8.2f} ms/step{'   <- compute stream' if s_ == main else ''}")
    rs = streams[main]
    gaps = [(b["ts"] - (a["ts"] + a["dur"]), a["name"], b["name"]) for a, b in zip(rs, rs[1:])]
    idle = sum(g for g, _, _ in gaps if g > 0)
    print(f"  compute stream idle: {idle / 1e3 / NSTEP:.2f} ms/step in {len(gaps)} gaps; gaps > 20 us: {sum(1 for g, _, _ in gaps if g > 20)} totalling {sum(g for g, _, _ in gaps if g > 20) / 1e3 / NSTEP:.2f} ms/step")
    big = sorted(gaps, key=lambda g: -g[0])[:10]
    for g, a, b in big:
        print(f"     gap {g:8.1f} us  after {a[:50]}  before {b[:50]}")
    byname = {}
    for r in rows:
        k = r["name"].split("(")[0][:70]
        d = byname.setdefault(k, [0, 0.0]); d[0] += 1; d[1] += r["dur"]
    for k, (n, d) in sorted(byname.items(), key=lambda kv: -kv[1][1])[:28]:
        print(f"    {d / 1e3 / NSTEP:8.2f} ms/step  n={n / NSTEP:7.1f}  {k}")
if world > 1:
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()
