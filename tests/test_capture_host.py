"""CUDA-graph capture rules, checked without a GPU: the guard, the cache bypass and the pinning of pna_b200.capture
under a simulated capture (torch.cuda.is_current_stream_capturing patched), and the new C status code."""
import gc
import os
import re
import weakref

import pytest
import torch

import pna_b200
from pna_b200 import _lib, capture, csr as csr_mod, dense, dist, readout
from pna_b200.csr import CSRGraph

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def capturing(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)


@pytest.fixture
def no_library(monkeypatch):
    """Fails the test if anything reaches the C library (i.e. would enqueue work)."""
    def refuse():
        raise AssertionError("the C library was called")
    monkeypatch.setattr(_lib, "lib", refuse)


def _toy_csr(n=4, e=3) -> CSRGraph:
    i = torch.zeros(n + 1, dtype=torch.int32)
    return CSRGraph(n_nodes=n, n_edges=e, rowptr=i, col=torch.zeros(e, dtype=torch.int32), perm=torch.zeros(e, dtype=torch.int32),
                    split_threshold=64, chunk_edges=64, hub_info=torch.zeros(0, 4, dtype=torch.int32),
                    chunk_items=torch.zeros(0, 2, dtype=torch.int32), n_hubs=0, n_chunks=0, max_degree=1)


def test_header_defines_capturing_status_and_lib_matches():
    src = open(os.path.join(ROOT, "include", "pna_b200.h")).read()
    m = re.search(r"PNA_ERR_CAPTURING\s*=\s*(-?\d+)", src)
    assert m and int(m.group(1)) == _lib.PNA_ERR_CAPTURING == -6
    assert re.search(r"#define PNA_ABI_VERSION 8\b", src) and _lib.ABI_VERSION == 8
    assert issubclass(pna_b200.CaptureError, RuntimeError) and pna_b200.CaptureError is capture.CaptureError


def test_not_capturing_without_cuda_context():
    assert capture.capturing() is False or torch.cuda.is_initialized()
    capture.guard("anything")                 # outside a capture: no error


class _Graph:
    batch_num_nodes = [2, 3]
    ndata = {}


@pytest.mark.parametrize("call", [
    lambda: csr_mod.build_csr(torch.zeros(3, dtype=torch.long), torch.zeros(3, dtype=torch.long), 4),
    lambda: _toy_csr().masked_view(torch.ones(4, dtype=torch.uint8)),
    lambda: _toy_csr().transposed(4),
    lambda: _toy_csr().slot_transposed(4),
    lambda: dense.DenseGraphs(torch.ones(2, 3, 3)),
    lambda: readout.segment_reduce(torch.zeros(5, 4), torch.tensor([0, 0, 1, 1, 1])),
    lambda: readout.global_mean_pool(torch.zeros(5, 4), torch.tensor([0, 0, 1, 1, 1])),
    lambda: readout._graph_batch(_Graph(), torch.device("cpu")),
    lambda: dist.PullAggregator.check(object.__new__(dist.PullAggregator)),
    lambda: dist.PullAggregator.exchange(object.__new__(dist.PullAggregator)),
    lambda: dist.PeerAggregator.barrier(object.__new__(dist.PeerAggregator)),
    lambda: dist.PeerAggregator.pna_aggregate(object.__new__(dist.PeerAggregator), torch.zeros(2, 4), ["sum"], ["identity"], {}),
    lambda: dist.HaloAggregator.aggregate(object.__new__(dist.HaloAggregator), ["sum"], ["identity"], {}),
], ids=["build_csr", "masked_view", "transposed", "slot_transposed", "DenseGraphs", "segment_reduce_no_size",
        "global_mean_pool_no_size", "graph_batch_first_use", "pull_check", "pull_exchange", "peer_barrier", "peer_aggregate",
        "halo_aggregate"])
def test_guard_raises_before_any_work(call, capturing, no_library):
    with pytest.raises(capture.CaptureError, match="CUDA graph capture"):
        call()


def test_guard_names_the_missing_state(capturing):
    with pytest.raises(capture.CaptureError, match="run one eager step on this graph first"):
        csr_mod.csr_from_edge_index(torch.zeros(2, 3, dtype=torch.long), 4)
    with pytest.raises(capture.CaptureError, match="slot-transposed CSR"):
        _toy_csr().slot_transposed(4)


def test_guard_is_silent_outside_a_capture():
    # the same calls fail on the CPU as they always have, not with CaptureError
    with pytest.raises(ValueError, match="CUDA"):
        csr_mod.build_csr(torch.zeros(3, dtype=torch.long), torch.zeros(3, dtype=torch.long), 4)
    g = _Graph()
    batch, n = readout._graph_batch(g, torch.device("cpu"))
    assert n == 2 and batch.tolist() == [0, 0, 1, 1, 1]


def test_built_state_is_used_inside_a_capture(capturing):
    c = _toy_csr()
    t = _toy_csr(4, 3)
    c._partials[("S", 4)] = t
    assert c.slot_transposed(4) is t
    g = _Graph()
    g._pna_b200_batch = torch.tensor([0, 0, 1, 1, 1])
    assert readout._graph_batch(g, torch.device("cpu"))[1] == 2


def test_sized_readout_does_not_raise(capturing, monkeypatch):
    batch = torch.tensor([0, 0, 1, 1, 1])
    fake = _toy_csr(2, 5)
    readout._CACHE[(batch.data_ptr(), csr_mod.tensor_version(batch), 5, 2, str(batch.device))] = (batch, fake)
    seen = []
    monkeypatch.setattr(readout, "pna_aggregate", lambda x, c, *a, **k: seen.append(c) or torch.zeros(2, x.size(1)))
    try:
        assert readout.global_add_pool(torch.zeros(5, 4), batch, size=2).shape == (2, 4)
        assert seen == [fake]
    finally:
        readout._CACHE.clear()


def test_readout_size_none_unchanged_outside_capture(monkeypatch):
    seen = []
    monkeypatch.setattr(readout, "batch_csr", lambda b, n: seen.append(n) or None)
    monkeypatch.setattr(readout, "pna_aggregate", lambda *a, **k: None)
    readout.segment_reduce(torch.zeros(5, 4), torch.tensor([0, 0, 1, 1, 2]))
    assert seen == [3]


# ---- cache bypass ------------------------------------------------------------------------------------------------
def _pyg(edge_dim=None, pre_layers=1):
    torch.manual_seed(0)
    return pna_b200.PNAConv(16, 16, ["mean", "max"], ["identity", "amplification"], torch.tensor([0, 3, 5, 2]), towers=2,
                            edge_dim=edge_dim, pre_layers=pre_layers)


def _dgl(edge_features=False, pretrans_layers=1):
    torch.manual_seed(0)
    return pna_b200.PNALayer(16, 16, ["mean", "max"], ["identity", "amplification"], {"log": 1.0, "lin": 2.0}, dropout=0.0,
                             graph_norm=False, batch_norm=False, towers=2, edge_features=edge_features, edge_dim=4,
                             pretrans_layers=pretrans_layers)


PACKS = {
    "pyg_prepared": (_pyg, lambda m: m._prepared(16), "_prep"),
    "pyg_message_weights": (lambda: _pyg(edge_dim=4, pre_layers=2), lambda m: m._message_weights(), "_msg_pack"),
    "pyg_tensor_core_pack": (_pyg, lambda m: m._tensor_core_pack(16), "_tc"),
    "dgl_affine_terms": (_dgl, lambda m: m._affine_terms(torch.ones(3, 16), 8), "_uv_pack"),
    "dgl_message_weights": (lambda: _dgl(True, 2), lambda m: m._message_weights(), "_msg_pack"),
}


def _leaves(v):
    if isinstance(v, dict):
        return [t for t in v.values() if isinstance(t, torch.Tensor)]
    return [t for t in v if isinstance(t, torch.Tensor)]


@pytest.mark.parametrize("name", sorted(PACKS))
def test_weight_packs_bypass_the_cache_while_capturing(name, monkeypatch):
    make, call, attr = PACKS[name]
    m = make()
    with torch.no_grad():
        first = call(m)
        cached = getattr(m, attr)
        again = call(m)
        # eager: hit as before (the same tensors come back for the packs that return the cache entry)
        if name != "dgl_affine_terms":
            assert all(a is b for a, b in zip(_leaves(first), _leaves(again)))
        assert getattr(m, attr) is cached
        monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
        inside = call(m)
        assert getattr(m, attr) is cached                       # not written
        if name != "dgl_affine_terms":
            assert not any(a is b for a, b in zip(_leaves(first), _leaves(inside)))     # not read: packed again
        for a, b in zip(_leaves(first), _leaves(inside)):
            assert torch.equal(a, b)


def test_dgl_affine_pack_is_rebuilt_while_capturing(monkeypatch):
    m = _dgl()
    with torch.no_grad():
        m._affine_terms(torch.ones(3, 16), 8)
        key, (w_uv, _) = m._uv_pack
        built = []
        real = torch.block_diag
        monkeypatch.setattr(torch, "block_diag", lambda *a: built.append(1) or real(*a))
        m._affine_terms(torch.ones(3, 16), 8)
        assert built == []                                     # eager: cache hit
        monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
        m._affine_terms(torch.ones(3, 16), 8)
        assert built and m._uv_pack[1][0] is w_uv


# ---- pinning -----------------------------------------------------------------------------------------------------
class _Fake:
    def __init__(self, *a, **k):
        pass


def test_pinning_keeps_csr_cache_entries_alive(monkeypatch):
    monkeypatch.setattr(csr_mod, "build_csr", lambda *a, **k: _Fake())
    csr_mod.clear_csr_cache()
    ei0 = torch.zeros(2, 3, dtype=torch.long)
    ref = weakref.ref(csr_mod.csr_from_edge_index(ei0, 4))
    with capture.pinned() as keep:
        monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
        assert csr_mod.csr_from_edge_index(ei0, 4) is ref()          # a hit inside the capture is recorded
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    others = [torch.zeros(2, 4 + k, dtype=torch.long) for k in range(csr_mod._CACHE_SIZE + 4)]
    for ei in others:
        csr_mod.csr_from_edge_index(ei, 4)
    assert all(v[0] is not ei0 for v in csr_mod._CACHE.values())     # evicted
    gc.collect()
    assert ref() is not None and ref() in keep.objects
    del keep
    gc.collect()
    assert ref() is None
    csr_mod.clear_csr_cache()


def test_pinning_keeps_dense_graphs_alive(monkeypatch):
    monkeypatch.setattr(dense, "DenseGraphs", _Fake)
    dense._CACHE.clear()
    adj0 = torch.ones(2, 3, 3)
    ref = weakref.ref(dense.dense_graphs(adj0, False))
    with capture.pinned() as keep:
        monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
        assert dense.dense_graphs(adj0, False) is ref()
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    adjs = [torch.ones(2, 3, 3) for _ in range(12)]
    for a in adjs:
        dense.dense_graphs(a, False)
    assert all(v[0] is not adj0 for v in dense._CACHE.values())
    gc.collect()
    assert ref() is not None
    del keep
    gc.collect()
    assert ref() is None
    dense._CACHE.clear()


def test_pinning_keeps_readout_csrs_alive(monkeypatch):
    monkeypatch.setattr(readout, "build_csr", lambda *a, **k: _Fake())
    readout._CACHE.clear()
    b0 = torch.tensor([0, 0, 1])
    ref = weakref.ref(readout.batch_csr(b0, 2))
    with capture.pinned() as keep:
        monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
        assert readout.batch_csr(b0, 2) is ref()
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    bs = [torch.tensor([0, 0, 1]) for _ in range(12)]
    for b in bs:
        readout.batch_csr(b, 2)
    gc.collect()
    assert ref() is not None
    del keep
    gc.collect()
    assert ref() is None
    readout._CACHE.clear()


def test_nothing_is_pinned_outside_a_capture_or_handle(monkeypatch):
    with capture.pinned() as keep:
        capture.pin(_Fake())                  # not capturing
    assert keep.objects == []
    monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    capture.pin(_Fake())                      # capturing, but no handle: nothing to record into
    assert capture._ACTIVE == []


def test_dense_column_mask_is_made_once_per_layer(capturing):
    lay = dense.PNALayer(4, 4, ["mean", "max"], ["identity"], {"log": 1.0}, towers=1)
    with pytest.raises(capture.CaptureError):
        lay._columns(12, ["_skip", "max"], torch.device("cpu"))


def test_dense_column_mask_cached_outside_capture():
    lay = dense.PNALayer(4, 4, ["mean", "max"], ["identity"], {"log": 1.0}, towers=1)
    m = lay._columns(12, ["_skip", "max"], torch.device("cpu"))
    assert m.tolist() == [False] * 4 + [False] * 4 + [True] * 4
    assert lay._columns(12, ["_skip", "max"], torch.device("cpu")) is m
