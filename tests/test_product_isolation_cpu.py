"""CPU: the product package must not reach into the test infrastructure (oracle/, tests/) or the reference checkout, and
must not carry a CPU fallback for the CUDA path."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "dinov3-jax_b200", "dinov3_jax")


def _sources():
    for d, _, files in os.walk(PKG):
        for f in files:
            if f.endswith(".py"):
                p = os.path.join(d, f)
                yield p, open(p).read()


def test_product_never_imports_oracle_tests_or_reference():
    bad = []
    for p, src in _sources():
        for pat in (r"^\s*(from|import)\s+oracle\b", r"^\s*(from|import)\s+tests\b", r"DINOV3_JAX_REFERENCE", r"jaxshim"):
            if re.search(pat, src, flags=re.M):
                bad.append((os.path.relpath(p, ROOT), pat))
    assert not bad, bad


def test_no_cpu_fallback_in_the_native_loader():
    src = open(os.path.join(PKG, "_native.py")).read()
    assert "NativeError" in src and "raise" in src
    ops = open(os.path.join(PKG, "ops.py")).read()
    assert "except ImportError" not in ops and "torch.matmul" not in ops and ".cpu()" not in ops


def test_bench_and_entry_do_not_read_the_reference_checkout():
    for name in ("bench.py", "__graft_entry__.py"):
        assert "DINOV3_JAX_REFERENCE" not in open(os.path.join(ROOT, name)).read(), name
