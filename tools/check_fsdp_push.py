"""torchrun --nproc-per-node N tools/check_fsdp_push.py : the NVLink push reduce-scatter (GEMM-epilogue scatter +
d3_scatter_add_peers) at ViT-L block dimensions (D=1024, 16 heads, hidden 4096, N=197/37), small depth / batch / K so a
step takes milliseconds: compares the pushed gradient shards with the NCCL reduce-scatter of the same step
(oracle-free: same engine, same batch, D3_FSDP_PUSH toggled through the runtime)."""
import os, sys, dataclasses
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist


def main():
    rank, world, lr_ = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr_)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr_))
    from dinov3_jax import _native
    from dinov3_jax.engine import Engine, config_for
    from dinov3_jax.engine.synth import reference_like_params, synthetic_batch
    from dinov3_jax.fsdp.runtime import Comm
    _native.init(lr_)
    depth = int(os.environ.get("CHK_DEPTH", "2")); B = int(os.environ.get("CHK_B", "4"))
    cfg = dataclasses.replace(config_for("vit_large", n_prototypes=8192, layerscale=0.1), depth=depth)
    params = reference_like_params(cfg, 0)
    batch = synthetic_batch(cfg, B, seed=10 + rank)
    M = torch.tensor([batch["mask_indices_list"].shape[0]], device="cuda")
    dist.all_reduce(M, op=dist.ReduceOp.MAX)
    grads = {}
    modes = os.environ.get("CHK_MODES", "nccl,push").split(",")
    for mi, mode in enumerate(modes):
        os.environ["D3_FSDP_PUSH"] = "1" if mode == "push" else "0"
        eng = Engine(cfg, B, device=f"cuda:{lr_}", max_masked=int(M.item()), comm=Comm())
        assert eng.fsdp.push == (mode == "push"), (mode, eng.fsdp.push)
        eng.params.load_reference_tree(params)
        eng.set_batch(batch)
        for _ in range(int(os.environ.get("CHK_STEPS", "2"))):
            eng.forward_backward(0.05)
            eng.fsdp.finish_grads()
            torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.synchronize()
        grads[mi] = {k: v.float().cpu() for k, v in eng.params.export_reference_tree("grad").items()}
        loss = eng.read_metrics()["total_loss"]
        if rank == 0:
            print(f"[{mode}] world={world} loss {loss:.6f}", flush=True)
        del eng
        torch.cuda.empty_cache()
        dist.barrier()
    if rank == 0:
        num = sum(float(((grads[1][k] - grads[0][k]) ** 2).sum()) for k in grads[0])
        den = sum(float((grads[0][k] ** 2).sum()) for k in grads[0])
        rel = (num / den) ** 0.5
        worst = sorted(((float((grads[1][k] - grads[0][k]).norm() / (grads[0][k].norm() + 1e-30)), k) for k in grads[0]), reverse=True)[:12]
        for e, k in worst:
            print(f"   {e:.3e}  {k}  |g|={float(grads[0][k].norm()):.3e}", flush=True)
        print(f"{modes[1]} vs {modes[0]} gradient shards: rel {rel:.3e} -> {'PUSH CHECK OK' if rel < 1e-3 else 'PUSH CHECK FAILED'}", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
