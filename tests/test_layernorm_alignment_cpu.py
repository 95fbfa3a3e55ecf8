"""The LayerNorm entry points reject operands that their 16-byte loads (and the backward's bulk row copies) cannot
read, before any CUDA call.  The addresses are never dereferenced; on a GPU machine the test is skipped so that it
never launches anything."""
import pytest

BASE = 1 << 40          # fake device addresses, 16-byte aligned, 1 GB apart


def _lib():
    import torch
    from dinov3_jax import _native
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    return _native.lib()


@pytest.mark.parametrize("bad", ["dy", "scale", "ls_gamma"])
def test_layernorm_bwd_rejects_operands_at_8_mod_16(bad):
    lib = _lib()
    T, D = 64, 1536      # a width without a ring instance: ln_bwd_ls_kernel, whose float4 loads need 16 bytes
    p = {k: BASE + i * (1 << 30) for i, k in enumerate(
        ("dy", "x", "mean", "rstd", "scale", "dx", "dscale", "dbias", "ls_gamma", "ls_du", "ls_dbias"))}
    p[bad] += 8
    rc = lib.d3_layernorm_bwd_ls(p["dy"], 1, p["x"], p["mean"], p["rstd"], p["scale"], None, p["dx"], p["dscale"],
                                 p["dbias"], T, D, p["ls_gamma"], None, 0, p["ls_du"], None, p["ls_dbias"], None)
    assert rc == -1
    assert b"misaligned" in lib.d3_last_error()


def test_layernorm_fwd_rejects_x_at_8_mod_16():
    lib = _lib()
    x, sc, bi, y = (BASE + i * (1 << 30) for i in range(4))
    rc = lib.d3_layernorm_fwd(x + 8, sc, bi, y, 0, None, None, 64, 1536, 1e-6, None)
    assert rc == -1
    assert b"16-byte aligned" in lib.d3_last_error()
