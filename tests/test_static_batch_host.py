"""StaticBatch without a GPU: the masked batch norm against nn.BatchNorm1d on the real rows, the capacity checks of copy_,
build() under a simulated capture (padded entry points only, nothing read back), and the header's new entry points."""
import contextlib
import os
import re
import types

import pytest
import torch

from pna_b200 import _lib, capture
from pna_b200.static_batch import StaticBatch, _PaddedBuild, masked_batch_norm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- masked batch norm ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("momentum", [0.1, None], ids=["momentum", "cumulative"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "plain"])
def test_masked_batch_norm_matches_batchnorm1d_on_the_real_rows(momentum, affine):
    torch.manual_seed(0)
    F, cap = 6, 40
    ref = torch.nn.BatchNorm1d(F, momentum=momentum, affine=affine).double()
    bn = torch.nn.BatchNorm1d(F, momentum=momentum, affine=affine).double()
    if affine:
        with torch.no_grad():
            ref.weight.uniform_(0.5, 1.5)
            ref.bias.uniform_(-0.5, 0.5)
        bn.load_state_dict(ref.state_dict())
    for step, n in enumerate([31, 17, 40, 5]):
        for mode in (True, False):
            ref.train(mode)
            bn.train(mode)
            x = torch.randn(n, F, dtype=torch.double) * 3 + 1
            xp = torch.cat([x, torch.randn(cap - n, F, dtype=torch.double) * 100]).requires_grad_(True)
            xr = x.clone().requires_grad_(True)
            mask = torch.arange(cap) < n
            g = torch.randn(cap, F, dtype=torch.double)
            y = masked_batch_norm(bn, xp, mask)
            want = ref(xr)
            torch.testing.assert_close(y[:n], want)
            assert torch.equal(y[n:], torch.zeros_like(y[n:]))
            (y * g).sum().backward()
            (want * g[:n]).sum().backward()
            torch.testing.assert_close(xp.grad[:n], xr.grad)
            assert torch.equal(xp.grad[n:], torch.zeros_like(xp.grad[n:]))
            if affine:
                torch.testing.assert_close(bn.weight.grad, ref.weight.grad)
                torch.testing.assert_close(bn.bias.grad, ref.bias.grad)
                bn.zero_grad()
                ref.zero_grad()
            torch.testing.assert_close(bn.running_mean, ref.running_mean)
            torch.testing.assert_close(bn.running_var, ref.running_var)
            assert int(bn.num_batches_tracked) == int(ref.num_batches_tracked) == step + 1


# ---- copy_: capacities checked on the host, before any work ----------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("the C library was called")
    monkeypatch.setattr(_lib, "lib", refuse)


def _host_batch(N=10, E=12, G=3):
    sb = object.__new__(StaticBatch)
    sb.max_nodes, sb.max_edges, sb.max_graphs = N, E, G
    sb._inputs = {}
    sb.src = sb.dst = sb.batch = None          # any copy would fail on these
    return sb


@pytest.mark.parametrize("what,kw", [
    ("max_nodes", dict(batch_num_nodes=[5, 6])),
    ("max_edges", dict(src=torch.zeros(13, dtype=torch.long), dst=torch.zeros(13, dtype=torch.long), batch_num_nodes=[3])),
    ("max_graphs", dict(batch_num_nodes=[1, 1, 1, 1])),
    ("max_nodes", dict(edge_index=torch.zeros(2, 4, dtype=torch.long), batch=torch.zeros(11, dtype=torch.long), num_graphs=1)),
])
def test_copy_refuses_an_exceeded_capacity_before_any_work(what, kw, no_library):
    kw.setdefault("src", torch.zeros(4, dtype=torch.long))
    kw.setdefault("dst", torch.zeros(4, dtype=torch.long))
    if "edge_index" in kw:
        kw.pop("src"), kw.pop("dst")
    with pytest.raises(ValueError, match=what):
        _host_batch().copy_(**kw)


def test_copy_refuses_features_of_the_wrong_row_count(no_library):
    with pytest.raises(ValueError, match="ndata"):
        _host_batch().copy_(src=torch.zeros(4, dtype=torch.long), dst=torch.zeros(4, dtype=torch.long), batch_num_nodes=[4],
                            ndata={"x": torch.zeros(5, 2)})


def test_copy_is_refused_inside_a_capture(monkeypatch, no_library):
    monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(capture.CaptureError):
        _host_batch().copy_(src=torch.zeros(1, dtype=torch.long), dst=torch.zeros(1, dtype=torch.long), batch_num_nodes=[2])


# ---- build(): capture-legal --------------------------------------------------------------------------------------------
class _FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*a):
            self.calls.append(name)
            if name == "pna_csr_padded_workspace_bytes":
                a[2]._obj.value = 1024
            return 0
        return call


def test_build_under_a_capture_calls_only_the_padded_entry_points(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    monkeypatch.setattr(_lib, "query", lambda what: 64)
    N, E, G = 8, 12, 3
    sb = object.__new__(StaticBatch)
    sb.max_nodes, sb.max_edges, sb.max_graphs, sb.device = N, E, G, torch.device("cpu")
    src, dst, batch = torch.zeros(E, dtype=torch.long), torch.full((E,), -1), torch.full((N,), -1)
    status = torch.zeros(3, 4, dtype=torch.int32)
    sb._transpose_dst = torch.full((E,), -1)
    sb._rows = _PaddedBuild(N, E, N, src, dst, status[0])
    sb._slots = _PaddedBuild(N, E, E, torch.arange(E), sb._transpose_dst, status[1])
    sb._readout = _PaddedBuild(G, N, N, torch.arange(N), batch, status[2])
    sb.csr = sb._rows.csr
    sb.csr._dst = torch.zeros(E, dtype=torch.long)
    assert sb.csr.padded and sb.csr.split_threshold > E
    fake.calls.clear()

    def refuse(*a, **k):
        raise AssertionError("a host read inside build()")
    monkeypatch.setattr(torch.Tensor, "item", refuse)
    monkeypatch.setattr(torch.Tensor, "cpu", refuse)
    monkeypatch.setattr(torch.Tensor, "tolist", refuse)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(torch.cuda, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    sb.build()
    assert fake.calls == ["pna_csr_build_padded", "pna_csr_slot_rows", "pna_csr_build_padded", "pna_csr_build_padded"]


def test_padded_csr_refuses_what_it_cannot_serve():
    from pna_b200.csr import CSRGraph
    c = CSRGraph(n_nodes=2, n_edges=3, rowptr=torch.zeros(3, dtype=torch.int32), col=torch.zeros(3, dtype=torch.int32),
                 perm=torch.zeros(3, dtype=torch.int32), split_threshold=4, chunk_edges=1,
                 hub_info=torch.zeros(0, 4, dtype=torch.int32), chunk_items=torch.zeros(0, 2, dtype=torch.int32), n_hubs=0,
                 n_chunks=0, max_degree=0, padded=True)
    with pytest.raises(ValueError, match="transposed"):
        c.transposed(2)
    with pytest.raises(ValueError, match="dst_of_slot"):
        c.dst_of_slot


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_header_declares_the_padded_entry_points_and_the_abi_is_still_8():
    src = open(os.path.join(ROOT, "include", "pna_b200.h")).read()
    assert re.search(r"#define PNA_ABI_VERSION 8\b", src) and _lib.ABI_VERSION == 8
    assert re.search(r"int pna_csr_build_padded\(const int64_t\* src, const int64_t\* dst, pna_csr_t\* csr, int32_t\* status,", src)
    assert re.search(r"int pna_csr_slot_rows\(const int32_t\* rowptr, const int32_t\* col, int64_t n_rows, int64_t n_slots,", src)
    assert re.search(r"int pna_csr_padded_workspace_bytes\(int64_t n_nodes, int64_t n_edges, size_t\* bytes\);", src)
    L = _lib.lib()
    assert L.pna_query(_lib.QUERY_ABI_VERSION) == 8
    assert {"pna_csr_build_padded", "pna_csr_slot_rows", "pna_csr_padded_workspace_bytes"} <= set(_lib.EXPORTED_SYMBOLS)


def test_padded_build_refuses_bad_arguments_before_any_work():
    import ctypes as C
    L = _lib.lib()
    st = _lib.CsrStruct(n_nodes=4, n_edges=10, split_threshold=10, chunk_edges=1)
    status = C.c_int32(0)
    assert L.pna_csr_build_padded(None, None, C.byref(st), C.byref(status), None, 0, None) == _lib.PNA_OK - 1   # split <= E
    assert b"split_threshold" in L.pna_last_error()
    assert L.pna_csr_build_padded(None, None, C.byref(st), None, None, 0, None) == -1                          # no status word
    assert L.pna_csr_slot_rows(None, None, 4, 0, None, None, None) == 0                                         # nothing to do
    assert L.pna_csr_slot_rows(None, None, 4, 3, None, None, None) == -1
    nb = C.c_size_t(0)
    assert L.pna_csr_padded_workspace_bytes(-1, 0, C.byref(nb)) == -1
