"""Attention shape limits are checked before any CUDA call, so they are reported without a GPU."""
import pytest


@pytest.mark.parametrize("N", [32769, 100000])
def test_attention_rejects_crops_above_the_token_bound(N):
    from dinov3_jax import _native
    lib = _native.lib()
    assert lib.d3_attn_fwd(None, None, None, 1, N, 64, 1, None) == -1
    assert b"32768" in lib.d3_last_error()
    assert lib.d3_attn_bwd(None, None, None, None, None, None, 1, N, 64, 1, None, None, 0, None) == -1
    assert b"32768" in lib.d3_last_error()


def test_attention_rejects_more_than_2_31_token_rows():
    from dinov3_jax import _native
    lib = _native.lib()
    assert lib.d3_attn_fwd(None, None, None, 65536, 32768, 64, 1, None) == -1
    assert b"2^31" in lib.d3_last_error()
