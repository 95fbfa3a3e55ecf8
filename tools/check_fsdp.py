"""torchrun --nproc-per-node N tools/check_fsdp.py : N-GPU FSDP step (rank-local images, sharded state, NCCL all-gather
/ reduce-scatter) against the multi-rank oracle on the same batches: loss, averaged gradients (re-assembled from the
shards) and one optimizer step."""
import os, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "dinov3-jax_b200")); sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist


def main():
    rank, world, lr_ = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr_)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr_))
    from dinov3_jax import _native
    from dinov3_jax.engine import Engine, from_oracle_cfg
    from dinov3_jax.fsdp.runtime import Comm
    from oracle import tiny_cfg
    from oracle.batch import synthetic_batch
    from oracle.model import init_params
    from oracle.step import grads_multi, clip_by_module, param_multipliers, adamw_update
    _native.init(lr_)
    cfg = tiny_cfg(layerscale=0.5)
    B = 2
    P = init_params(cfg, 0, perturb=0.05)
    ecfg = from_oracle_cfg(cfg)
    if "--distinct-heads" in sys.argv:      # an iBOT head with its own sizes (the oracle reads them from the parameters)
        import dataclasses
        K, Hh, Bn = 136, 96, 48
        Pi = init_params(dataclasses.replace(cfg, n_prototypes=K, head_hidden=Hh, head_bottleneck=Bn), 1, perturb=0.05)
        P.update({k: v for k, v in Pi.items() if "_ibot_head/" in k})
        ecfg = dataclasses.replace(ecfg, ibot_n_prototypes=K, ibot_head_hidden=Hh, ibot_head_bottleneck=Bn)
    batches = [synthetic_batch(cfg, B, seed=r) for r in range(world)]
    hyper = dict(lr=1e-3, wd=0.04, last_layer_lr=5e-4, momentum=0.99, teacher_temp=0.05)
    eng = Engine(ecfg, B, device=f"cuda:{lr_}", max_masked=max(int(b["mask_indices_list"].shape[0]) for b in batches), comm=Comm())
    eng.params.load_reference_tree(P)
    if rank == 0:
        print("gradient reduce-scatter path:", "push over NVLink peer memory (GEMM epilogue + d3_scatter_add_peers)" if eng.fsdp.push else "NCCL reduce_scatter", flush=True)
    eng.set_batch(batches[rank])
    eng.forward_backward(hyper["teacher_temp"])
    eng.fsdp.finish_grads()
    grads_e = {k: v.cpu() for k, v in eng.params.export_reference_tree("grad").items()}
    eng.optimizer_step(hyper["lr"], hyper["wd"], hyper["last_layer_lr"], hyper["momentum"])
    torch.cuda.synchronize()
    met = eng.read_metrics()
    newp_e = {k: v.cpu() for k, v in eng.params.export_reference_tree("param").items()}
    # second step exercises the gather of updated shards
    eng.train_step(None, **hyper)
    torch.cuda.synchronize()
    met2 = eng.read_metrics()
    if rank == 0:
        loss, mets, grads = grads_multi(P, batches, hyper["teacher_temp"], cfg)
        print(f"world={world}: loss oracle={loss.item():.6f} engine={met['total_loss']:.6f} rel={abs(loss.item()-met['total_loss'])/abs(loss.item()):.2e}")
        num = sum(((grads_e[k].reshape(g.shape) - g) ** 2).sum() for k, g in grads.items()); den = sum((g ** 2).sum() for g in grads.values())
        grel = float(torch.sqrt(num / den))
        worst = max(((float((grads_e[k].reshape(g.shape) - g).norm() / (g.norm() + 1e-30)), k) for k, g in grads.items() if g.norm() > 1e-3))
        print(f"  averaged grads: global rel={grel:.3e} worst={worst[1]} {worst[0]:.3e}")
        # optimizer on the engine's own gradients (isolates the sharded AdamW/EMA from bf16 gradient noise)
        clipped, norms = clip_by_module({k: grads_e[k].reshape(P[k].shape) for k in grads}, cfg.clip_grad)
        mults = param_multipliers(list(grads), cfg.depth)
        err = 0.0
        for k in grads:
            lm, wm, last = mults[k]
            p1, _, _ = adamw_update(P[k], clipped[k], torch.zeros_like(P[k]), torch.zeros_like(P[k]), 1, lm * (hyper["last_layer_lr"] if last else hyper["lr"]), wm * hyper["wd"])
            err = max(err, float((newp_e[k].reshape(p1.shape) - p1).abs().max() / (hyper["lr"])))
            tk = "teacher_" + k[len("student_"):]
            t1 = P[tk] * hyper["momentum"] + p1 * (1 - hyper["momentum"])
            err = max(err, float((newp_e[tk].reshape(t1.shape) - t1).abs().max() / hyper["lr"]))
        for k, v in norms.items():
            print(f"  {k}: oracle-of-engine-grads={float(v):.6f} engine={met[k]:.6f}")
        print(f"  sharded AdamW/EMA max |dp| error / lr = {err:.3e}")
        ok = abs(loss.item() - met["total_loss"]) < 1e-3 * abs(loss.item()) and grel < 3e-2 and err < 2e-2 and met2["total_loss"] == met2["total_loss"]
        print(f"  step-2 loss {met2['total_loss']:.6f}  ->  {'FSDP CHECK OK' if ok else 'FSDP CHECK FAILED'}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
