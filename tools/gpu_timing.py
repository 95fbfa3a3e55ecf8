"""The card query and the CUDA-event timing loops of the benchmark scripts in tools/: every number they print is timed
here and printed beside the card it was measured on."""
import subprocess

import torch


def card() -> dict:
    """Name, power limit and maximum SM clock of the device torch is using.  nvidia-smi does not follow
    CUDA_VISIBLE_DEVICES, so it is asked for the device by UUID, not by index.  A field that cannot be read is
    "not read"; this never raises, and it only queries."""
    out = dict.fromkeys(("gpu", "power_limit", "sm_clock_max"), "not read")
    try:
        props = torch.cuda.get_device_properties(torch.cuda.current_device())
        out["gpu"] = props.name
        q = subprocess.run(["nvidia-smi", "-i", f"GPU-{props.uuid}", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        fields = [f.strip() for f in q.stdout.split(",")]
        if q.returncode == 0 and len(fields) == 2:
            out.update((k, v) for k, v in zip(("power_limit", "sm_clock_max"), fields) if v and not v.startswith("["))
    except Exception:
        pass
    return out


def cuda_ms(fn, iters, warmup):
    """Milliseconds per call of fn: `warmup` untimed calls, then one CUDA event pair around `iters` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def cuda_ms_each(fn, iters, warmup, before=None):
    """Milliseconds of each of `iters` calls of fn, each between its own CUDA event pair, after `warmup` untimed calls.
    `before` (an L2 flush, say) runs untimed ahead of every timed call."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if before is not None:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts
