"""In-tree build of the sm_90a CUDA library (``sonar_b200/lib/libsonar_b200.so``).

nvcc cross-compiles without a GPU.  The explicit ``-gencode arch=compute_90a,code=sm_90a``
form is required: a bare ``-arch=sm_90a`` also emits a ``compute_90`` PTX pass in which
``wgmma.*`` does not assemble.
"""

from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIB_DIR = ROOT / "lib"
LIB_PATH = LIB_DIR / "libsonar_b200.so"
SOURCES = ["encoder.cu", "gemm_wgmma.cu", "gemm_skinny.cu", "attention_tc.cu", "elementwise.cu", "xsim.cu", "decoder.cu", "beam.cu", "fbank.cu", "conformer.cu", "attention_relpos_tc.cu", "latent_attention.cu", "lstm.cu", "blaser.cu"]
HEADERS = ["common.cuh", "attention_wgmma.cuh", "sonar_b200_internal.h", "../../include/sonar_b200.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC or add /usr/local/cuda/bin to PATH)")


def _digest() -> str:
    h = hashlib.sha256()
    for name in SOURCES + HEADERS:
        p = (CSRC / name).resolve()
        if p.exists():
            h.update(name.encode())
            h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA source for sm_90a into one shared library (incremental:
    skipped when sources + flags hash matches the stamp next to the library)."""
    LIB_DIR.mkdir(exist_ok=True)
    stamp = LIB_DIR / "build.stamp"
    digest = _digest()
    if not force and LIB_PATH.exists() and stamp.exists() and stamp.read_text().strip() == digest:
        return LIB_PATH
    nvcc = _nvcc()
    objs = []
    log_lines = []
    for name in SOURCES:
        src = CSRC / name
        if not src.exists():
            continue
        obj = LIB_DIR / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log_lines.append("$ " + " ".join(cmd))
        log_lines.append(r.stdout)
        log_lines.append(r.stderr)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"nvcc failed on {name}")
        objs.append(str(obj))
    cmd = [nvcc, "-shared", "-o", str(LIB_PATH), *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log_lines += ["$ " + " ".join(cmd), r.stdout, r.stderr]
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc link failed")
    (LIB_DIR / "build.log").write_text("\n".join(log_lines))
    stamp.write_text(digest)
    if verbose:
        print("\n".join(log_lines))
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
