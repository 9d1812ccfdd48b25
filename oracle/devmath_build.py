"""Builds the device-math probe oracle/devmath/devmath.cu -> oracle/_build/libdevmath_sm90.so (test infrastructure).

Compiled with exactly the library's nvcc flags (pna_b200._lib.NVCC_FLAGS), so that its powf / expf are the ones the
add-on kernels inline; it includes none of the library's headers.  Cross-compiles without a GPU.
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "devmath", "devmath.cu")
LIB = os.path.join(HERE, "_build", "libdevmath_sm90.so")


def build(out: str = LIB, force: bool = False) -> str:
    from pna_b200 import _lib
    if not force and os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(SRC), os.path.getmtime(_lib.__file__)):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    cmd = ["nvcc"] + list(_lib.NVCC_FLAGS) + ["-shared", SRC, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    return out
