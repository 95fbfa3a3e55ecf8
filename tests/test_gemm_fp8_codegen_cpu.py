"""What ptxas makes of the FP8 GEMM instances (gemm_tc.cu, E4M3 = true) and the e4m3 quantizers (fp8.cu) for sm_90a,
checked without a GPU: no stack frame, no spills, and no serialized wgmma (C7510 / C7514 / C7520).  Two m64n64 chains
plus their promotion temporary must fit the 168 registers a thread of the 384-thread GEMM CTA is compiled for."""
import os
import re
import subprocess

from conftest import ROOT
from test_attention_codegen_cpu import _build_module, _unmangled

PKG = os.path.join(ROOT, "dinov3-jax_b200")
E4M3_INSTANCES = 12        # 11 fixed epilogue flag sets and the run-time-flag one (dispatch_e4m3)
QUANT_KERNELS = {"quant_rows_kernel", "colmax_kernel", "quant_cols_t_kernel"}


def _ptxas(src, tmp_path):
    b = _build_module()
    cmd = [b.find_nvcc()] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(PKG, "csrc", src), "-o", str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    props = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    return log, props


def test_e4m3_gemm_instances_have_no_stack_spills_or_serialized_wgmma(tmp_path):
    log, props = _ptxas("gemm_tc.cu", tmp_path)
    e4m3 = [p for p in props if _unmangled(p[0]) == "gemm_kernel" and "Lb1EEEv" in p[0]]
    assert len(e4m3) == E4M3_INSTANCES, [p[0] for p in e4m3]
    bad = [(m, stack, st, ld) for m, stack, st, ld in e4m3 if (stack, st, ld) != ("0", "0", "0")]
    assert not bad, bad
    serialized = [line for line in log.splitlines() if re.search(r"C75(10|14|20)", line)]
    assert not serialized, serialized


def test_e4m3_quantizers_have_no_stack_or_spills(tmp_path):
    log, props = _ptxas("fp8.cu", tmp_path)
    assert QUANT_KERNELS <= {_unmangled(m) for m, *_ in props}
    bad = [(m, stack, st, ld) for m, stack, st, ld in props if (stack, st, ld) != ("0", "0", "0")]
    assert not bad, bad
