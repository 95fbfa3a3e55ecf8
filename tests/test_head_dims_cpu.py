"""DINO and iBOT heads of different sizes, host side: the YAML keys, the per-head parameter specs and FSDP shard
layouts, and the oracle against the reference's SSLMetaArch.__call__ run with two head geometries
(tests/golden/make_heads_golden.py)."""
import dataclasses
import os

import numpy as np
import pytest
import torch

from dinov3_jax.engine.config import EngineConfig, config_for, config_from_reference_cfg
from dinov3_jax.engine.params import ParamStore, head_spec

# dino.head_* / ibot.head_* of the DINOv3 recipes (dinov3_vit7b16_pretrain, dinov3_vitl16_lvd1689m_distilled, ...)
DINOV3_HEADS = ["dino.head_n_prototypes=262144", "dino.head_hidden_dim=8192", "dino.head_bottleneck_dim=512",
                "ibot.head_n_prototypes=98304", "ibot.head_hidden_dim=4096", "ibot.head_bottleneck_dim=384"]
TINY = EngineConfig(embed_dim=128, depth=2, heads=2, n_prototypes=264, head_hidden=136, head_bottleneck=40,
                    ibot_n_prototypes=136, ibot_head_hidden=96, ibot_head_bottleneck=48)


def _setup(opts):
    from dinov3_jax.configs import DinoV3SetupArgs, setup_config
    return setup_config(DinoV3SetupArgs(opts=["student.arch=vit_large"] + opts))


def test_dinov3_head_keys_map_onto_the_ibot_fields():
    cfg = config_from_reference_cfg(_setup(DINOV3_HEADS))
    assert (cfg.n_prototypes, cfg.head_hidden, cfg.head_bottleneck) == (262144, 8192, 512)
    assert (cfg.ibot_n_prototypes, cfg.ibot_head_hidden, cfg.ibot_head_bottleneck) == (98304, 4096, 384)
    assert cfg.head_dims("dino_head") == (8192, 512, 262144)
    assert cfg.head_dims("ibot_head") == (4096, 384, 98304)


def test_only_the_differing_ibot_keys_are_set():
    cfg = config_from_reference_cfg(_setup(["ibot.head_n_prototypes=32768"]))
    assert (cfg.ibot_n_prototypes, cfg.ibot_head_hidden, cfg.ibot_head_bottleneck) == (32768, None, None)
    assert cfg.head_dims("ibot_head") == (2048, 256, 32768)


@pytest.mark.parametrize("heads", [[], ["dino.head_n_prototypes=4096", "ibot.head_n_prototypes=4096",
                                        "dino.head_hidden_dim=1024", "ibot.head_hidden_dim=1024"]])
def test_equal_head_keys_give_the_configuration_of_one_shared_size(heads):
    cfg = config_from_reference_cfg(_setup(heads))
    assert cfg.ibot_n_prototypes is None and cfg.ibot_head_hidden is None and cfg.ibot_head_bottleneck is None
    assert cfg == dataclasses.replace(cfg, ibot_n_prototypes=None, ibot_head_hidden=None, ibot_head_bottleneck=None)
    assert cfg.head_dims("ibot_head") == cfg.head_dims("dino_head")


def test_ibot_sizes_follow_the_dino_head_unless_set():
    cfg = config_for("vit_small", n_prototypes=4096)
    assert cfg.head_dims("ibot_head") == (2048, 256, 4096)       # not the 65 536 of a concrete default
    with pytest.raises(ValueError):
        cfg.head_dims("backbone")


def test_default_parameter_specs_are_unchanged():
    cfg = EngineConfig()
    D, Hh, Bn, K = 384, 2048, 256, 65536
    want = [("mlp/layers_0/kernel", (D, Hh), "mat"), ("mlp/layers_0/bias", (Hh,), "vec"),
            ("mlp/layers_2/kernel", (Hh, Hh), "mat"), ("mlp/layers_2/bias", (Hh,), "vec"),
            ("mlp/layers_4/kernel", (Hh, Bn), "mat"), ("mlp/layers_4/bias", (Bn,), "vec"),
            ("last_layer/kernel", (Bn, K), "mat")]
    assert head_spec(cfg) == head_spec(cfg, "dino_head") == head_spec(cfg, "ibot_head") == want


def test_per_head_specs_and_parameter_groups():
    from dinov3_jax.train.ssl_meta_arch import SSLMetaArch
    d = dict((n, s) for n, s, _ in head_spec(TINY, "dino_head"))
    i = dict((n, s) for n, s, _ in head_spec(TINY, "ibot_head"))
    assert d["mlp/layers_0/kernel"] == (128, 136) and d["last_layer/kernel"] == (40, 264)
    assert i["mlp/layers_0/kernel"] == (128, 96) and i["mlp/layers_2/kernel"] == (96, 96)
    assert i["mlp/layers_4/kernel"] == (96, 48) and i["last_layer/kernel"] == (48, 136)
    arch = SSLMetaArch(_setup(DINOV3_HEADS))
    groups = arch.get_params_groups()
    assert "student_ibot_head/last_layer/kernel" in groups and groups["student_ibot_head/last_layer/kernel"][2] is True
    assert len([k for k in groups if k.startswith("student_ibot_head/")]) == 7


@pytest.mark.parametrize("world", [1, 2, 4])
def test_fsdp_shards_partition_each_head_unit(world):
    """Every element of each head's flat buffer is owned by exactly one rank, the head is one FSDP unit, and the
    optimiser segments cover each tensor once (the layout follows the spec; nothing is special-cased per head)."""
    for rank in range(world):
        ps = ParamStore(TINY, "cpu", world=world, rank=rank)
        for module in ("dino_head", "ibot_head"):
            st = ps.mods[module]
            assert [u.name for u in st.layout.units] == ["head"]
            assert st.shapes == {n: s for n, s, _ in head_spec(TINY, module)}
    seen = {m: None for m in ("dino_head", "ibot_head")}
    for rank in range(world):
        ps = ParamStore(TINY, "cpu", world=world, rank=rank)
        for m in seen:
            L = ps.mods[m].layout
            if seen[m] is None:
                seen[m] = np.zeros(L.n, dtype=np.int32)
            seen[m][L.full_to_shard_index(rank)] += 1
    for m, s in seen.items():
        assert (s == 1).all(), m
    n_d = ParamStore(TINY, "cpu").mods["dino_head"].n
    n_i = ParamStore(TINY, "cpu").mods["ibot_head"].n
    assert n_d != n_i


def test_checkpoint_tree_follows_the_specs():
    """The reference-named tree the checkpointer saves has each head's own shapes."""
    ps = ParamStore(TINY, "cpu")
    tree = ps.export_reference_tree("param")
    assert tuple(tree["student_dino_head/last_layer/kernel"].shape) == (40, 264)
    assert tuple(tree["teacher_ibot_head/last_layer/kernel"].shape) == (48, 136)
    assert tuple(tree["student_ibot_head/mlp/layers_2/kernel"].shape) == (96, 96)


# ------------------------------------------------------------------------------------------------ golden
def heads_golden():
    from conftest import GOLDEN
    with np.load(os.path.join(GOLDEN, "heads_vectors.npz")) as z:
        return {k: z[k] for k in z.files}


def heads_case(G, case, dtype=torch.float64):
    """The closed-form inputs of a heads_vectors.npz case: (oracle ModelCfg with the DINO sizes, iBOT sizes,
    parameters, batch, teacher temperature)."""
    from oracle.arch import ModelCfg
    from oracle.model import formula_images, formula_params
    B, n_local, seed, n_storage, norm_bf16 = (int(v) for v in G[f"ssl_{case}_spec"])
    Kd, Hd, Bd = (int(v) for v in G["dino_dims"])
    ibot = tuple(int(v) for v in G["ibot_dims"])
    cfg = ModelCfg(embed_dim=128, depth=2, heads=2, global_size=64, local_size=32, n_local=n_local, n_prototypes=Kd,
                   head_hidden=Hd, head_bottleneck=Bd, n_storage=n_storage, ln_eps=1e-5 if norm_bf16 else 1e-6)
    # tests/golden/make_heads_golden.py: heads_params
    P = formula_params(cfg, seed, dtype)
    Pi = formula_params(dataclasses.replace(cfg, n_prototypes=ibot[0], head_hidden=ibot[1], head_bottleneck=ibot[2]),
                        seed, dtype)
    P.update({k: v for k, v in Pi.items() if k.split("/", 1)[0].endswith("_ibot_head")})
    masks = torch.from_numpy(G[f"ssl_{case}_masks"])
    idx = torch.from_numpy(G[f"ssl_{case}_mask_indices"])
    batch = {"collated_global_crops": formula_images((2 * B, 64, 64, 3), 100 + seed, dtype),
             "collated_local_crops": formula_images((n_local * B, 32, 32, 3), 200 + seed, dtype),
             "collated_masks": masks, "mask_indices_list": idx,
             "n_masked_patches": torch.tensor([idx.shape[0]]), "upperbound": int(idx.shape[0]), "global_batch_size": B}
    return cfg, ibot, P, batch, float(G[f"ssl_{case}_teacher_temp"])


@pytest.mark.parametrize("case", ["a", "c"])
def test_oracle_matches_reference_meta_arch_with_distinct_heads(case):
    from oracle.step import ssl_forward
    G = heads_golden()
    cfg, ibot, P, batch, temp = heads_case(G, case)
    assert tuple(P["student_ibot_head/last_layer/kernel"].shape) == (ibot[2], ibot[0])
    loss, metrics = ssl_forward(P, batch, temp, cfg, dtype=torch.float64)
    want = float(G[f"ssl_{case}_loss"])
    assert abs(float(loss) - want) < 1e-9 * abs(want)
    keys = [k.split("/", 1)[1] for k in G if k.startswith(f"ssl_{case}_metric/")]
    assert set(keys) == {"local_batch_size", "dino_local_crops_loss", "dino_local_loss_weight", "dino_global_crops_loss",
                         "koleo_loss", "ibot_loss"}
    for k in keys:
        w = float(G[f"ssl_{case}_metric/{k}"])
        assert abs(float(metrics[k]) - w) < 1e-9 * max(abs(w), 1.0), k
