"""Host-side checks of the tensor-core linear's backward (pna_linear_bwd_data / pna_linear_bwd_weight): argument validation
before any launch, the workspace query, and the SASS of its kernels (no atomics: the result is a fixed function of the
inputs).  No compute call is made here."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from pna_b200 import _lib

DUMMY = 256                                  # 16-byte aligned, never dereferenced: validation fails first


def ws_bytes(n_rows, n_in, n_out, n_scalers):
    nb = C.c_size_t(0)
    assert _lib.lib().pna_linear_bwd_workspace_bytes(n_rows, n_in, n_out, n_scalers, C.byref(nb)) == 0
    return nb.value


def test_backward_entry_points_validate_without_gpu():
    L = _lib.lib()
    data, weight = L.pna_linear_bwd_data, L.pna_linear_bwd_weight
    # data(grad_y, ld, row_scale, S, weight, grad_a, ld, n_rows, n_in, n_out, ws, ws_bytes, stream)
    assert data(None, 0, None, 1, None, None, 0, 0, 64, 128, None, 0, None) == 0                 # no rows: nothing to do
    assert data(None, 0, None, 1, None, None, 0, 5, 60, 128, None, 0, None) == -2                # n_in % 32
    assert data(None, 0, None, 3, None, None, 0, 5, 100, 128, None, 0, None) == -2               # 100 / 3 is not a K width
    assert data(None, 0, None, 1, None, None, 0, 5, 64, 100, None, 0, None) == -2                # n_out not 64/128/256
    assert data(None, 0, None, 1, None, None, 0, 5, 64, 128, None, 0, None) == -1                # null pointers
    assert data(None, 0, None, 9, None, None, 0, 0, 288, 64, None, 0, None) == -1                # more scalers than exist
    assert data(DUMMY, 128, None, 3, DUMMY, DUMMY, 96, 5, 288, 128, DUMMY, 1 << 30, None) == -1  # row_scale missing
    assert b"pna_linear_bwd_data" in L.pna_last_error()
    assert data(DUMMY, 128, None, 1, DUMMY, DUMMY, 64, 5, 64, 128, DUMMY, 16, None) == -5        # workspace too small
    assert b"pna_linear_bwd_data" in L.pna_last_error() and b"workspace" in L.pna_last_error()
    # weight(grad_y, ld, a, lda, row_scale, S, grad_weight, n_rows, n_in, n_out, ws, ws_bytes, stream)
    assert weight(None, 0, None, 0, None, 3, None, 0, 96, 64, None, 0, None) == 0
    assert weight(None, 0, None, 0, None, 1, None, 5, 48, 64, None, 0, None) == -2
    assert weight(None, 0, None, 0, None, 1, None, 5, 64, 32, None, 0, None) == -2
    assert weight(None, 0, None, 0, None, 1, None, 5, 64, 64, None, 0, None) == -1
    assert weight(None, 0, None, 0, None, 6, None, 5, 192, 64, None, 0, None) == -1
    assert weight(DUMMY, 64, DUMMY, 32, None, 2, DUMMY, 5, 64, 64, DUMMY, 1 << 30, None) == -1
    assert b"pna_linear_bwd_weight" in L.pna_last_error()
    n = 169_343
    assert weight(DUMMY, 128, DUMMY, 512, DUMMY, 3, DUMMY, n, 1536, 128, DUMMY, ws_bytes(n, 1536, 128, 3) - 4, None) == -5
    assert b"pna_linear_bwd_weight" in L.pna_last_error() and b"workspace" in L.pna_last_error()
    assert weight(DUMMY, 128, DUMMY, 512, DUMMY, 3, DUMMY, n, 1536, 128, None, 1 << 40, None) == -5
    # misaligned operands are refused, not read
    assert data(DUMMY + 4, 128, None, 1, DUMMY, DUMMY, 64, 5, 64, 128, DUMMY, 1 << 30, None) == -2
    assert weight(DUMMY, 130, DUMMY, 64, None, 1, DUMMY, 5, 64, 128, DUMMY, 1 << 30, None) == -2


def test_workspace_query():
    L = _lib.lib()
    nb = C.c_size_t(0)
    assert L.pna_linear_bwd_workspace_bytes(10, 64, 64, 1, None) == -1
    assert L.pna_linear_bwd_workspace_bytes(10, 60, 64, 1, C.byref(nb)) == -2
    assert L.pna_linear_bwd_workspace_bytes(10, 64, 96, 1, C.byref(nb)) == -2
    assert L.pna_linear_bwd_workspace_bytes(-1, 64, 64, 1, C.byref(nb)) == -1
    # at least the data gradient's hi / lo weight images, zero rows or not
    assert ws_bytes(0, 1536, 128, 1) >= 2 * 1536 * 128 * 4
    assert ws_bytes(1, 96 * 5, 256, 5) >= 2 * 96 * 5 * 256 * 4
    sizes = [ws_bytes(n, 1536, 128, 3) for n in (1, 1000, 10_000, 169_343, 1_000_003)]
    assert sizes == sorted(sizes) and sizes[-1] > sizes[0]                     # grows with n_rows (the weight partials)
    assert ws_bytes(169_343, 1536, 128, 3) < 64 << 20
    assert ws_bytes(169_343, 1536, 128, 1) == ws_bytes(169_343, 1536, 128, 3)


def test_backward_kernels_have_no_atomics():
    """cuobjdump of the built library: the kernels of pna_linear_bwd_data / _weight contain no ATOM / RED instruction."""
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump, cu++filt and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        kernels[m.group(1)] = m.group(2)
    names = subprocess.run(["cu++filt"], input="\n".join(kernels), capture_output=True, text=True, check=True).stdout.split("\n")
    demangled = dict(zip(kernels, names))
    bwd = [k for k, n in demangled.items()
           if any(s in n for s in ("k_linear_bwd_weight", "k_sum_splits", "k_split_weight_t", "k_linear_3xtf32"))]
    # k_linear_3xtf32: O = 64 / 128 / 256 forward instances, and the folding instances of the data gradient's 64 / 128 slabs
    assert len(bwd) == 3 + 1 + 1 + 3 + 2, [demangled[k] for k in bwd]
    for k in bwd:
        assert not re.findall(r"\b(?:ATOM|ATOMG|ATOMS|RED|REDG)\b", kernels[k]), demangled[k]
