"""Build libdinov3_b200.so in-tree with nvcc for sm_90a (no torch extension machinery: a plain C-ABI library)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
OUT = ROOT / "libdinov3_b200.so"
SOURCES = ["api.cu", "gemm_tc.cu", "attention.cu", "elementwise.cu", "losses.cu", "optim.cu", "augment.cu", "convnext.cu", "fp8.cu", "knn.cu", "linear.cu", "seg.cu", "depth.cu", "video.cu", "correspondence.cu", "discovery.cu", "retrieval.cu", "koleo.cu", "logreg.cu", "attentive.cu"]
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def find_nvcc() -> str:
    """$NVCC, then nvcc on PATH, then the toolkit under $CUDA_HOME (default /usr/local/cuda)."""
    if os.environ.get("NVCC"):
        return os.environ["NVCC"]
    found = shutil.which("nvcc")
    if found:
        return found
    cand = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda")) / "bin" / "nvcc"
    if cand.exists():
        return str(cand)
    raise RuntimeError("nvcc not found: set NVCC or CUDA_HOME, or put the CUDA toolkit's bin/ on PATH")


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    nvcc = find_nvcc()
    objdir = ROOT / "build"
    objdir.mkdir(exist_ok=True)
    # objects built with other flags (another GPU architecture) are never reused
    stamp = objdir / "flags.txt"
    if not stamp.exists() or stamp.read_text() != " ".join(FLAGS):
        force = True
    headers = list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + [ROOT.parent / "include" / "dinov3_b200.h"]
    jobs = []
    for src in SOURCES:
        obj = objdir / (src + ".o")
        if force or _stale(obj, [CSRC / src] + headers):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc] + FLAGS + ["-c", str(CSRC / src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose and r.stderr:
            print(r.stderr)
        return src

    if jobs:
        with ThreadPoolExecutor(max_workers=min(6, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    objs = [str(objdir / (s + ".o")) for s in SOURCES]
    if jobs or not OUT.exists():
        r = subprocess.run([nvcc, "-shared", "-o", str(OUT)] + objs + ["-lcudart"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(" ".join(FLAGS))
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
