"""The C-ABI library loads without a GPU and exports every symbol include/dinov3_b200.h declares."""
import ctypes
import os
import re

from conftest import ROOT


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "dinov3_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(d3_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported():
    from dinov3_jax import _native
    lib = _native.lib()
    names = declared_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/dinov3_b200.h but not exported"


def test_python_signature_table_matches_header():
    from dinov3_jax import _native
    declared = set(declared_symbols())
    bound = set(_native.SIGNATURES) | set(_native.NO_ARG_SYMBOLS)
    assert declared == bound, (declared - bound, bound - declared)


def test_abi_version_7_and_error_string():
    """Version 7: the scatter-mode and SM-limit setters are gone (the peer push has one form, the persistent grids use
    every SM).  Version 6: the plain KoLeo is d3_koleo_fwd_bwd_rows over all rows.  Version 5: the attention debug trace
    (d3_debug_attn_trace) is gone.  Version 4: the plain LayerNorm backward and the atomic-free Sinkhorn sums have no
    entry points of their own."""
    from dinov3_jax import _native
    lib = _native.lib()
    assert lib.d3_abi_version() == 7
    assert isinstance(lib.d3_last_error(), bytes)


def test_argument_errors_are_reported_without_gpu():
    """Validation happens before any CUDA call: null pointers -> D3_ERR_ARG (-1) and a message."""
    from dinov3_jax import _native
    lib = _native.lib()
    ep = _native.GemmEpilogue()
    rc = lib.d3_gemm_bf16(None, 8, 0, None, 8, 0, 128, 128, 64, ctypes.byref(ep), 0, 0, None)
    assert rc == -1 and b"null" in lib.d3_last_error()
    rc = lib.d3_im2col(None, None, 768, 1, 30, 30, 16, None)
    assert rc == -1


def test_no_cpu_fallback():
    """Without a GPU the product path must raise, not silently compute on the CPU."""
    import pytest
    import torch
    from dinov3_jax import _native
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_native.NativeError):
        _native.init()
