"""What ptxas makes of csrc/attention.cu for sm_90a, checked without a GPU: every kernel compiles with no stack frame and
no spills, and no wgmma chain is serialized (ptxas C7520: a wgmma waits on a warpgroup arrive the compiler inserted in a
divergent path, which once cost attn_bwd_fused_kernel a tenth of its instructions)."""
import importlib.util
import os
import re
import subprocess

from conftest import ROOT

PKG = os.path.join(ROOT, "dinov3-jax_b200")
KERNELS = {"attn_fwd_kernel", "attn_fwd_stream_kernel", "attn_bwd_fused_kernel", "attn_bwd_dkdv_kernel",
           "attn_bwd_dq_kernel", "attn_delta_kernel", "attn_fwd_hd128_kernel", "attn_bwd_dkdv_hd128_kernel",
           "attn_bwd_dq_hd128_kernel"}


def _build_module():
    spec = importlib.util.spec_from_file_location("d3_build", os.path.join(PKG, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _unmangled(name):
    """d3::attn_fwd_kernel from _ZN2d315attn_fwd_kernelE...: the length-prefixed identifier after the namespace."""
    m = re.match(r"_ZN2d3(\d+)", name)
    return name[m.end():m.end() + int(m.group(1))] if m else name


def test_attention_kernels_have_no_stack_spills_or_serialized_wgmma(tmp_path):
    b = _build_module()
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(PKG, "csrc", "attention.cu"),
                                       "-o", str(tmp_path / "attention.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    names = {_unmangled(m) for m, *_ in props}
    assert KERNELS <= names, KERNELS - names
    bad = [(m, stack, st, ld) for m, stack, st, ld in props if (stack, st, ld) != ("0", "0", "0")]
    assert not bad, bad
    serialized = [line for line in log.splitlines() if "C7520" in line]
    assert not serialized, serialized
