"""Build libdmpnn_sm90.so in-tree with nvcc for sm_90a (H100); build() writes it under chemprop_b200/lib/."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "lib" / "libdmpnn_sm90.so"
SOURCES = ["api_misc.cu", "dataset.cu", "layout.cu", "linear.cu", "segment.cu", "step_fused.cu", "step_fused_fwd.cu", "step_fused_bwd.cu", "step_fused_far_fwd.cu", "step_fused_far_bwd.cu", "step_fused_atom_fwd.cu", "step_fused_atom_bwd.cu", "linear_tc.cu", "wgrad_tc.cu", "gemm_x3.cu", "head.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xptxas=-v", "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def collate_ext_path() -> Path:
    import sysconfig

    return PKG / "lib" / ("_collate_ext" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))


def build_collate_ext(force: bool = False) -> Path | None:
    """The host-side collate as a CPython extension (gcc; no CUDA).  Optional: BatchMolGraph falls back to the ctypes
    path without it, so a missing compiler / header only costs collate speed."""
    import sysconfig

    src, out = CSRC / "collate_ext.c", collate_ext_path()
    if not src.exists():
        return None
    if not force and out.exists() and out.stat().st_mtime > src.stat().st_mtime:
        return out
    try:
        import numpy as np

        cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
        inc = sysconfig.get_paths()["include"]
        if not cc or not os.path.exists(os.path.join(inc, "Python.h")):
            return None
        out.parent.mkdir(parents=True, exist_ok=True)
        cmd = [cc, "-O2", "-fPIC", "-shared", "-I", inc, "-I", np.get_include(), str(src), "-o", str(out)]
        subprocess.run(cmd, check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        return out
    except Exception as e:  # noqa: BLE001
        sys.stderr.write(f"[collate_ext] not built: {e}\n")
        return None


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = [CSRC / s for s in SOURCES] + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "dmpnn.h"]
    return any(d.exists() and d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = True) -> Path:
    build_collate_ext(force)
    if not force and not needs_build():
        return LIB
    LIB.parent.mkdir(parents=True, exist_ok=True)
    objs = []
    nvcc = _nvcc()
    bdir = PKG / "lib" / "obj"
    bdir.mkdir(parents=True, exist_ok=True)
    procs = []
    for s in SOURCES:
        src = CSRC / s
        if not src.exists():
            continue
        obj = bdir / (s + ".o")
        objs.append(obj)
        if not force and obj.exists() and obj.stat().st_mtime > max(
            [src.stat().st_mtime] + [h.stat().st_mtime for h in CSRC.glob("*.cuh")]
            + [(PKG.parent / "include" / "dmpnn.h").stat().st_mtime]
        ):
            continue
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {s}")
        if verbose:
            for line in out.splitlines():
                if "error" in line or "warning" in line.lower() or "spill" in line and "0 bytes spill" not in line:
                    print(f"[{s}] {line}")
    cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
