"""-m gpu: the reference-named layer / loss objects (dinov3_jax.layers, dinov3_jax.loss) against the oracle."""
import pytest
import torch

pytestmark = pytest.mark.gpu
BF = 8e-3


def rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-30)).item()


def nest(flat: dict) -> dict:
    out = {}
    for k, v in flat.items():
        cur = out
        parts = k.split("/")
        for p in parts[:-1]:
            cur = cur.setdefault(p, {})
        cur[parts[-1]] = v.cuda()
    return out


@pytest.fixture(scope="module")
def setup(native):
    from oracle import tiny_cfg
    from oracle.model import init_params, sub
    cfg = tiny_cfg(layerscale=0.7)
    P = init_params(cfg, 0, perturb=0.05)
    return cfg, P, sub


def test_block_and_attention_and_mlp(setup):
    from dinov3_jax.layers import Mlp, RopePositionEmbedding, SelfAttention, SelfAttentionBlock
    from oracle.model import Emu, block_forward, rope_sincos
    cfg, P, sub = setup
    bp = sub(P, "student_backbone")
    blk = nest(sub(bp, "blocks_0"))
    n, Hp = 3, 4
    N, D = Hp * Hp + 1, cfg.embed_dim
    x = torch.randn(n, N, D)
    sin, cos = rope_sincos(Hp, Hp, 64, 100.0, torch.float32)
    want = block_forward(bp, "blocks_0/", x, sin, cos, cfg, Emu(False))
    rope = RopePositionEmbedding(embed_dim=D, num_heads=cfg.heads)(H=Hp, W=Hp)
    got = SelfAttentionBlock(blk, dim=D, num_heads=cfg.heads)(x.cuda(), rope=rope)
    assert rel(got, want) < BF
    # Mlp alone: gelu(gelu(x W1 + b1) W2 + b2)
    from oracle.model import gelu
    xm = torch.randn(50, D)
    wm = gelu(gelu(xm @ bp["blocks_0/mlp/Dense_0/kernel"] + bp["blocks_0/mlp/Dense_0/bias"]) @ bp["blocks_0/mlp/Dense_1/kernel"] + bp["blocks_0/mlp/Dense_1/bias"])
    assert rel(Mlp(blk["mlp"])(xm.cuda()), wm) < BF
    # SelfAttention alone
    from oracle.model import attention
    qkv = x @ bp["blocks_0/attn/qkv/kernel"] + bp["blocks_0/attn/qkv/bias"]
    wa = attention(qkv, cfg.heads, sin, cos, Emu(False)) @ bp["blocks_0/attn/proj/kernel"] + bp["blocks_0/attn/proj/bias"]
    assert rel(SelfAttention(blk["attn"], dim=D, num_heads=cfg.heads, qkv_bias=True)(x.cuda(), rope=rope), wa) < BF


def test_patch_embed_and_head(setup):
    from dinov3_jax.layers import DINOHead, PatchEmbed
    from oracle.model import Emu, head_forward, patch_embed
    cfg, P, sub = setup
    bp = sub(P, "student_backbone")
    img = torch.randn(2, 64, 64, 3).to(torch.bfloat16)
    want, _ = patch_embed(bp, img.float(), cfg, Emu(False))
    got = PatchEmbed(nest(sub(bp, "patch_embed")), patch_size=16, embed_dim=cfg.embed_dim)(img.cuda())
    assert got.shape == (2, 4, 4, cfg.embed_dim) and rel(got.reshape(2, 16, -1), want) < BF   # conv kernel is rounded to bf16 for the tensor cores
    with pytest.raises(AssertionError):
        PatchEmbed(nest(sub(bp, "patch_embed")), patch_size=16, embed_dim=cfg.embed_dim)(torch.zeros(1, 60, 64, 3, device="cuda", dtype=torch.bfloat16))
    hp = sub(P, "student_dino_head")
    x = torch.randn(37, cfg.embed_dim)
    head = DINOHead(nest(hp), in_dim=cfg.embed_dim, out_dim=cfg.n_prototypes, hidden_dim=cfg.head_hidden, bottleneck_dim=cfg.head_bottleneck)
    assert rel(head(x.cuda()), head_forward(hp, x)) < BF


def test_loss_objects_match_oracle(setup):
    from dinov3_jax.loss import DINOLoss, KoLeoLoss, iBOTPatchLoss
    from oracle.losses import dino_loss, ibot_loss_masked, koleo_loss, sinkhorn_knopp
    K, B = 512, 6
    torch.manual_seed(1)
    t_logits = torch.randn(2 * B, K) * 0.3
    dl = DINOLoss(K)
    Q = dl.sinkhorn_knopp_teacher(t_logits.cuda(), teacher_temp=0.05)
    Qr = sinkhorn_knopp(t_logits.double(), 0.05, 2 * B).float()
    assert rel(Q, Qr) < 1e-4
    sl, sg = torch.randn(8, B, K), torch.randn(2, B, K)
    tp = Qr.reshape(2, B, K)
    assert abs(dl(sl.cuda(), tp.cuda()).item() - dino_loss(sl, tp, 0.1, False).item()) < 1e-4 * 8
    assert abs(dl(sg.cuda(), tp.cuda(), ignore_diagonal=True).item() - dino_loss(sg, tp, 0.1, True).item()) < 1e-4 * 8
    M = 19
    il = iBOTPatchLoss(K)
    pl = torch.randn(M, K) * 0.3
    Qp = il.sinkhorn_knopp_teacher(pl.cuda(), teacher_temp=0.05, n_masked_patches_tensor=torch.tensor([M]))
    Qpr = sinkhorn_knopp(pl.double(), 0.05, float(M)).float()
    assert rel(Qp, Qpr) < 1e-4
    sp = torch.randn(M, K)
    masks = torch.zeros(2 * B, 16, dtype=torch.bool)
    got = il.forward_masked(sp.cuda(), Qpr.cuda(), student_masks_flat=masks, n_masked_patches=M, masks_weight=torch.ones(M))
    assert abs(got.item() - ibot_loss_masked(sp, Qpr, 0.1, 2 * B).item()) < 1e-3
    x = torch.randn(32, 128)
    assert abs(KoLeoLoss()(x.cuda()).item() - koleo_loss(x).item()) < 1e-5


def test_unsupported_options_raise():
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch
    with pytest.raises(NotImplementedError):
        SSLMetaArch(setup_config(DinoV3SetupArgs(opts=["train.centering=centering"])))
    with pytest.raises(NotImplementedError):
        SSLMetaArch(setup_config(DinoV3SetupArgs(opts=["student.norm_layer=rmsnorm"])))


def test_do_train_runs_three_iterations():
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train.train import do_train
    cfg = setup_config(DinoV3SetupArgs(opts=["student.arch=vit_small", "train.batch_size_per_gpu=2", "dino.head_n_prototypes=1024",
                                             "ibot.head_n_prototypes=1024", "dino.head_hidden_dim=256", "ibot.head_hidden_dim=256"]))
    m = do_train(cfg, SSLMetaArch(cfg), max_iters=3, print_freq=1)
    assert abs(m["dino_local_crops_loss"] - 6.93) < 0.05 and m["total_loss"] == m["total_loss"]


def test_do_train_checkpoints_and_resumes(tmp_path):
    from dinov3_jax.checkpointer import find_all_checkpoints
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train.train import do_train
    opts = ["student.arch=vit_small", "train.batch_size_per_gpu=2", "dino.head_n_prototypes=1024", "ibot.head_n_prototypes=1024",
            "dino.head_hidden_dim=256", "ibot.head_hidden_dim=256", "checkpointing.period=2", "checkpointing.max_to_keep=1"]
    cfg = setup_config(DinoV3SetupArgs(opts=opts, output_dir=str(tmp_path)))
    do_train(cfg, SSLMetaArch(cfg), max_iters=4, print_freq=1)
    assert [p.name for p in find_all_checkpoints(tmp_path / "ckpt")] == ["3"]          # period 2, keep last 1
    m = do_train(cfg, SSLMetaArch(cfg), resume=True, max_iters=5, print_freq=1)        # runs iteration 4 only
    assert m["total_loss"] == m["total_loss"]


def test_vit_and_head_against_reference_golden(native):
    """CUDA forward (dinov3_jax.models.DinoVisionTransformer, dinov3_jax.layers.DINOHead) against vectors produced by
    executing the reference's own module code (tests/golden/make_golden.py) — no oracle in between.  bf16-operand /
    fp32-accumulate tolerance, norm-wise."""
    from conftest import reference_vectors
    from dinov3_jax.layers import DINOHead
    from dinov3_jax.models import DinoVisionTransformer
    G = reference_vectors()
    tree = lambda prefix: nest({k[len(prefix):]: torch.from_numpy(G[k]) for k in G if k.startswith(prefix)})
    model = DinoVisionTransformer(tree("vit_param/"), img_size=64, patch_size=16, embed_dim=128, n_blocks=2, num_heads=2,
                                  layerscale_init=0.5)
    og, ol = model([torch.from_numpy(G["vit_global"]), torch.from_numpy(G["vit_local"])],
                   masks=[torch.from_numpy(G["vit_masks"]), None], is_training=True)
    for o, tag in ((og, "g"), (ol, "l")):
        assert rel(o["x_norm_clstoken"], torch.from_numpy(G[f"vit_{tag}_cls"])) < 2e-2
        assert rel(o["x_norm_patchtokens"], torch.from_numpy(G[f"vit_{tag}_patch"])) < 2e-2
    assert rel(model(torch.from_numpy(G["vit_global"])), torch.from_numpy(G["vit_g_cls"])) > 1e-2      # masks matter
    head = DINOHead(tree("head_param/"), in_dim=128, out_dim=48, hidden_dim=64, bottleneck_dim=32)
    x = torch.from_numpy(G["head_x"]).cuda()
    assert rel(head(x), torch.from_numpy(G["head_logits"])) < 2e-2
    assert rel(head(x, no_last_layer=True), torch.from_numpy(G["head_bottleneck"])) < 2e-2


def test_do_train_with_the_gpu_data_pipeline(tmp_path):
    """train.dataset_path=synthetic:gpu: images in HBM -> on-GPU augmentation + masks -> engine, through do_train."""
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    from dinov3_jax.train import SSLMetaArch
    from dinov3_jax.train.train import do_train
    opts = ["train.dataset_path=synthetic:gpu", "train.batch_size_per_gpu=2", "student.arch=vit_small", "crops.global_crops_size=64",
            "crops.local_crops_size=32", "dino.head_n_prototypes=512", "ibot.head_n_prototypes=512", "dino.head_hidden_dim=256",
            "ibot.head_hidden_dim=256", "dino.head_bottleneck_dim=64", "ibot.head_bottleneck_dim=64", "optim.epochs=1",
            "train.OFFICIAL_EPOCH_LENGTH=4", "optim.warmup_epochs=0", "teacher.warmup_teacher_temp_epochs=0",
            "optim.freeze_last_layer_epochs=0", f"train.output_dir={tmp_path}", "checkpointing.period=100"]
    config = setup_config(DinoV3SetupArgs(opts=opts))
    m = do_train(config, SSLMetaArch(config), resume=False, max_iters=3, print_freq=1)
    assert m["total_loss"] == m["total_loss"] and m["total_loss"] > 0
