"""Slot weights (pna_aggregate_fwd_weighted / _bwd_weighted / _bwd_slots_weighted) without a GPU: the binding of the new entry
points, the refusals (status codes, returned before anything is enqueued), and the SASS of the new kernels."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from pna_b200 import _lib

UNSUPPORTED = -2
FAKE = 0x1000            # never dereferenced: every call below returns before it reads a buffer
ENTRY_POINTS = ("pna_aggregate_fwd_weighted", "pna_aggregate_bwd_weighted", "pna_aggregate_bwd_slots_weighted")


HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pna_b200.h")
_CTYPE = {"const pna_agg_t*": C.POINTER(_lib.AggStruct), "pna_stream_t": C.c_void_p, "int64_t": C.c_int64, "int32_t": C.c_int32}


def _header_params(name):
    """parameter types of `name`'s prototype in the header, pointers other than the descriptor as void*"""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", src)
    assert m, name
    types = []
    for p in m.group(1).split(","):
        t = " ".join(p.split()[:-1]).replace(" *", "*")
        types.append(_CTYPE.get(t, C.c_void_p if t.endswith("*") else None))
    return types


def test_entry_points_are_bound_as_the_header_declares_them():
    """Each weighted entry point is the unweighted call with (slot_weight, scaler_degree_f) after the descriptor; the ctypes
    binding has the header's parameter list, and the descriptor keeps its layout."""
    L = _lib.lib()
    for n in ENTRY_POINTS:
        assert n in _lib.EXPORTED_SYMBOLS
        assert list(getattr(L, n).argtypes) == _header_params(n), n
    for n, base in zip(ENTRY_POINTS, ("pna_aggregate_fwd", "pna_aggregate_bwd", "pna_aggregate_bwd_slots")):
        assert _header_params(n) == _header_params(base)[:1] + [C.c_void_p, C.c_void_p] + _header_params(base)[1:], n
    assert _lib.AggStruct._fields_[-1][0] == "degree_col"          # the weights are arguments, not descriptor fields
    assert _lib.query(_lib.QUERY_SIZEOF_AGG) == C.sizeof(_lib.AggStruct)
    assert _lib.query(_lib.QUERY_ABI_VERSION) == 8


def _desc(aggrs, **kw):
    na, ac = _lib.pack_codes(aggrs, _lib.ALL_AGGR_CODES, "aggregator")
    d = _lib.AggStruct(gathered=FAKE, ld_gathered=8, rowptr=FAKE, col=FAKE, out=FAKE, ld_out=64, n_rows=4, n_feat=8, n_towers=1,
                       n_aggr=na, aggr_codes=ac, n_scalers=1, scaler_codes=0, avg_log=1.0, avg_lin=1.0, split_threshold=64,
                       chunk_edges=32)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _calls(L, d, sw, sdf):
    """(forward, atomic backward, per-slot backward) status codes of the weighted entry points on descriptor d"""
    return (L.pna_aggregate_fwd_weighted(C.byref(d), sw, sdf, None),
            L.pna_aggregate_bwd_weighted(C.byref(d), sw, sdf, FAKE, 64, FAKE, 8, None, 0, None),
            L.pna_aggregate_bwd_slots_weighted(C.byref(d), sw, sdf, FAKE, 64, 0, 8, FAKE, 8, None, 0, None))


@pytest.mark.parametrize("aggr", ["moment3", "moment4", "moment5", "softmax", "softmin", "normalised_mean"])
@pytest.mark.parametrize("which", ["slot_weight", "scaler_degree_f"])
def test_aggregators_without_a_weighted_form_are_refused(aggr, which):
    L = _lib.lib()
    sw, sdf = (FAKE, None) if which == "slot_weight" else (None, FAKE)
    assert _calls(L, _desc(["mean", aggr]), sw, sdf) == (UNSUPPORTED,) * 3
    assert b"slot_weight" in L.pna_last_error()


def test_row_ids_and_the_peer_plane_are_refused():
    L = _lib.lib()
    aggrs = ["mean", "max", "min", "std"]
    for kw in (dict(row_ids=FAKE, n_row_ids=2), dict(peer_gathered=FAKE, peer_shift=8)):
        assert _calls(L, _desc(aggrs, **kw), FAKE, FAKE) == (UNSUPPORTED,) * 3
    assert L.pna_aggregate_fwd_weighted(C.byref(_desc(aggrs, ld_out=7)), FAKE, None, None) == -1    # a row is 4 * 8 wide
    assert L.pna_aggregate_fwd_weighted(C.byref(_desc(aggrs, n_rows=0)), FAKE, None, None) == 0     # nothing to do
    assert L.pna_aggregate_bwd_slots_weighted(C.byref(_desc(aggrs)), FAKE, None, FAKE, 64, 0, 8, None, 8, None, 0, None) == -1
    # NULL weights and degree: exactly the unweighted call (which needs no weighted form of the list)
    d = _desc(["mean", "moment3"], n_rows=0)
    assert L.pna_aggregate_fwd_weighted(C.byref(d), None, None, None) == 0


def test_slots_and_split_row_instances_have_no_atomics():
    """The deterministic backward's instances (SLOTS), every split-row kernel and the forward have no ATOM / RED; the atomic
    instances of the per-slot kernels do."""
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump, cu++filt and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if "k_aw_" in m.group(1):
            kernels[m.group(1)] = re.findall(r"\b(?:ATOM|ATOMG|RED|REDG)\b", m.group(2))
    names = subprocess.run(["cu++filt"], input="\n".join(kernels), capture_output=True, text=True, check=True).stdout.split("\n")
    demangled = dict(zip(kernels, names))
    atomic = [k for k, n in demangled.items() if "(bool)0>" in n]
    rest = [k for k in kernels if k not in atomic]
    # forward: rows, chunk, hub_final x 2 types; backward: chunk_stats, hub_coef x 2 types, hub_bias, rows / chunk_grad SLOTS x 2
    assert len(rest) == 6 + 4 + 1 + 4 and len(atomic) == 4
    for k in rest:
        assert not kernels[k], f"{demangled[k]}: {kernels[k][:4]}"
    assert all(kernels[k] for k in atomic)
