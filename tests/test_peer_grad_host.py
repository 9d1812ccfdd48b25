"""Host-side checks of the peer plane's backward: the SASS of its kernel instances, and the Python entry point's binding."""
import os
import re
import shutil
import subprocess

import pytest

from pna_b200 import _lib


def test_peer_slot_instances_have_no_atomics():
    """cuobjdump of the built library: the instances pna_aggregate_bwd_peer_slots launches (k_peer_bwd_rows,
    k_peer_bwd_hub_stats and k_peer_bwd_hub_scatter: the per-slot bodies with PEER = true) contain no ATOM / RED
    instruction."""
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if "k_peer_bwd_" in m.group(1):
            kernels[m.group(1)] = re.findall(r"\b(?:ATOM|ATOMG|ATOMS|RED|REDG)\b", m.group(2))
    # 4 (element type, vector width) pairs x 6 lane-group widths x 3 kernels
    assert len(kernels) == 4 * 6 * 3
    assert {re.search(r"k_peer_bwd_[a-z_]+", k).group(0) for k in kernels} == \
        {"k_peer_bwd_rows", "k_peer_bwd_hub_stats", "k_peer_bwd_hub_scatter"}
    for k, found in kernels.items():
        assert not found, f"{k}: {found[:4]}"


def test_binding_matches_the_header():
    header = open(os.path.join(_lib.REPO_ROOT, "include", "pna_b200.h")).read()
    assert re.search(r"^int pna_aggregate_bwd_peer_slots\(", header, re.M)
    assert "pna_aggregate_bwd_peer_slots" in _lib.EXPORTED_SYMBOLS
    L = _lib.lib()
    assert L.pna_aggregate_bwd_peer_slots.argtypes == L.pna_aggregate_bwd_slots.argtypes
    assert L.pna_aggregate_bwd_peer_slots(None, None, 0, 0, 4, None, 4, None, 0, None) == -1     # null descriptor
    d = _lib.AggStruct(n_rows=4, n_feat=8, n_towers=1, n_aggr=1, n_scalers=1, split_threshold=16, chunk_edges=8,
                       gathered=256, rowptr=256, col=256)               # never dereferenced: refused first
    import ctypes as C
    gs = C.c_void_p(256)
    assert L.pna_aggregate_bwd_peer_slots(C.byref(d), gs, 8, 0, 8, gs, 8, None, 0, None) == -1     # no peer table
    assert b"peer_gathered" in L.pna_last_error()
