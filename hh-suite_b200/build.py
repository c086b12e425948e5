"""Build the product library in-tree: hh-suite_b200/libhhg.so (sm_90a only, no other arch)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "hhg_api.cu")
import glob  # noqa: E402

# every source the library is built from: a stale .so after editing any kernel header is a parity trap
DEPS = sorted(glob.glob(os.path.join(HERE, "csrc", "*.cu*")) + glob.glob(os.path.join(HERE, "csrc", "*.h")) +
              glob.glob(os.path.join(os.path.dirname(HERE), "include", "*.h")))
OUT = os.path.join(HERE, "libhhg.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-fmad=false",            # belt and braces: the kernels use explicit _rn intrinsics anyway
         "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off",   # host-side flog2/fpow2 must not be fused either
         "-diag-suppress", "177", "-shared"]


def stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build_variant(tag: str, defines: list[str]) -> str:
    """Developer helper: compile a kernel variant (-D switches) to hh-suite_b200/variants/libhhg_<tag>.so."""
    vdir = os.path.join(HERE, "variants")
    os.makedirs(vdir, exist_ok=True)
    out = os.path.join(vdir, f"libhhg_{tag}.so")
    subprocess.check_call([NVCC] + FLAGS + [f"-D{d}" for d in defines] + ["-o", out, SRC])
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    if force or stale():
        if not os.path.exists(NVCC):
            if os.path.exists(OUT):
                return OUT          # GPU box without a toolchain: use the shipped library
            raise RuntimeError("nvcc not found and libhhg.so missing")
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT, SRC]
        subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
