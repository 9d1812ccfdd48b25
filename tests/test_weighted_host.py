"""Host-side plumbing of softmax / softmin / normalised_mean / identity: codes, the layers that take them and those that
do not, the backward mode they select, the inputs normalised_mean refuses, and the SASS of their deterministic instances."""
import contextlib
import types

import pytest
import torch

from pna_b200 import _lib, aggregate as agg

REGISTRY = ["mean", "sum", "max", "min", "identity", "std", "var", "normalised_mean", "softmax", "softmin", "moment3", "moment4",
            "moment5"]          # models/pytorch/pna/aggregators.py:149-152


def test_codes_pack_into_nibbles():
    assert [_lib.ALL_AGGR_CODES[m] for m in _lib.WEIGHTED] == [9, 10, 11]
    assert all(m not in _lib.AGGR_CODES for m in _lib.WEIGHTED)       # the table every flavour accepts is unchanged
    assert _lib.AGGR_CODES == {"sum": 0, "mean": 1, "min": 2, "max": 3, "var": 4, "std": 5, "_skip": 15}
    n, codes = _lib.pack_codes(["mean", "softmax", "max", "softmin", "normalised_mean", "std"], _lib.ALL_AGGR_CODES, "aggregator")
    assert n == 6 and codes == 1 | 9 << 4 | 3 << 8 | 10 << 12 | 11 << 16 | 5 << 20


def test_dense_layer_constructs_with_every_registry_name():
    from pna_b200 import dense
    avg = {"log": 1.5, "lin": 3.0}
    for a in REGISTRY:
        lay = dense.PNALayer(8, 8, ["mean", a], ["identity", "amplification"], avg, towers=2)
        assert lay.towers[0].posttrans.fully_connected[0].linear.in_features == (2 * 2 + 1) * 4
    for a in ("softmax", "softmin", "normalised_mean", "identity"):
        dense.PNALayer(8, 8, ["mean", a], ["identity"], avg, self_loop=True)
    for a in _lib.WEIGHTED:
        assert a in dense._SELF_FIRST


def test_dense_identity_columns_and_scale_factors():
    """identity's block: X_ii per tower in every scaler's slot, scaled like the kernel epilogue (1 where D == 0)."""
    from pna_b200 import dense
    avg = {"log": 1.5, "lin": 3.0}
    lay = dense.PNALayer(4, 4, ["mean", "identity"], ["identity", "attenuation", "linear"], avg, towers=2)
    g = types.SimpleNamespace(scaler_degree=torch.tensor([0, 2, 5], dtype=torch.int32))
    x = torch.arange(12, dtype=torch.float32).view(3, 4) + 1
    blk = lay._identity_block(x, g).view(3, 2, 1 + 3 * 2, 2)
    mask = lay._columns(blk[0].numel(), ["_skip", "identity"], "cpu").view(2, 7, 2)
    assert mask[:, [2, 4, 6]].all() and not mask[:, [0, 1, 3, 5]].any()
    D = torch.tensor([0.0, 2.0, 5.0])
    att = torch.where(D > 0, 1.5 / torch.log(D + 1), torch.ones_like(D))
    for t in range(2):
        xt = x[:, 2 * t:2 * t + 2]
        torch.testing.assert_close(blk[:, t, 2], xt)
        torch.testing.assert_close(blk[:, t, 4], xt * att[:, None])
        torch.testing.assert_close(blk[:, t, 6], xt * (D / 3.0)[:, None])


@pytest.mark.parametrize("m", ["softmax", "softmin", "normalised_mean", "identity"])
def test_pyg_and_dgl_layers_refuse_the_new_names(m):
    from pna_b200 import dgl_layers, pyg
    deg = torch.tensor([0, 3, 5, 2])
    with pytest.raises(KeyError):
        pyg.PNAConvSimple(8, 8, ["mean", m], ["identity"], deg)
    with pytest.raises(KeyError):
        pyg.PNAConv(8, 8, ["mean", m], ["identity"], deg)
    with pytest.raises(KeyError):
        dgl_layers.PNASimpleLayer(8, 8, f"mean {m}", "identity", {"log": 1.0, "lin": 1.0}, 0.0, False, False)


class _RecordingLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append(name)
            return 0
        return call


@pytest.mark.parametrize("aggrs,want", [(["mean", "softmax"], "pna_aggregate_bwd"), (["softmin"], "pna_aggregate_bwd"),
                                        (["normalised_mean", "max"], "pna_aggregate_bwd"),
                                        (["mean", "std"], "pna_aggregate_bwd_coef")])
def test_coef_mode_takes_the_atomic_path(monkeypatch, aggrs, want):
    monkeypatch.setenv("PNA_B200_BWD", "coef")
    rec = _RecordingLib()
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    monkeypatch.setattr(_lib, "query", lambda what: 16384)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(agg, "aggregate_forward", lambda *a, **k: torch.zeros(4, 16))
    n, f = 4, 8
    csr = types.SimpleNamespace(n_nodes=n, n_edges=6, sources_unique=False, n_hubs=0, n_chunks=0, split_threshold=64,
                                chunk_edges=32, rowptr=torch.zeros(n + 1, dtype=torch.int32), col=torch.zeros(6, dtype=torch.int32),
                                hub_info=None, chunk_items=None, transposed=lambda n_src: None)
    x = torch.zeros(n, f)
    go = torch.zeros(n, len(aggrs) * f)
    agg.aggregate_backward(go, x, csr, aggrs, ["identity"], {"log": 1.0})
    assert rec.calls[0] == want


def test_normalised_mean_refuses_rows_that_are_not_the_csrs():
    csr = types.SimpleNamespace(n_nodes=5, n_edges=7)
    avg = {"log": 1.0, "lin": 1.0}
    for kw, rows in ((dict(), 6), (dict(messages_in_csr_order=True), 7)):
        for fn in (agg.aggregate_forward, agg.pna_aggregate):
            with pytest.raises(ValueError, match="normalised_mean"):
                fn(torch.zeros(rows, 4), csr, ["mean", "normalised_mean"], ["identity"], avg, **kw)
    with pytest.raises(ValueError, match="normalised_mean"):
        agg.aggregate_forward(torch.zeros(5, 4), csr, ["normalised_mean"], ["identity"], avg,
                              peer=(torch.zeros(2, dtype=torch.int64), 8))
    # the other names pass this check (and stop at the next one: no CUDA tensor here)
    with pytest.raises(ValueError, match="CUDA"):
        agg.aggregate_forward(torch.zeros(6, 4), csr, ["softmax"], ["identity"], avg)


def test_deterministic_weighted_instances_have_no_atomics():
    """cuobjdump of the built library: the weighted kernels pna_aggregate_bwd_slots launches contain no ATOM / RED; the
    atomic instances of the row and chunk kernels still do (they add into grad_gathered[col[slot]])."""
    import os
    import re
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump, cu++filt and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if "k_wsum_" in m.group(1):
            kernels[m.group(1)] = re.findall(r"\b(?:ATOM|ATOMG|RED|REDG)\b", m.group(2))
    names = subprocess.run(["cu++filt"], input="\n".join(kernels), capture_output=True, text=True, check=True).stdout.split("\n")
    demangled = dict(zip(kernels, names))
    atomic = [k for k, n in demangled.items() if ("k_wsum_bwd_rows" in n or "k_wsum_bwd_chunk_grad" in n) and "(bool)0>" in n]
    others = [k for k in demangled if k not in atomic]
    assert len(atomic) == 4 and len(others) == 9 + 11      # 9 forward, 15 backward instances in all
    for k in others:
        assert not kernels[k], f"{demangled[k]}: {kernels[k][:4]}"
    assert all(kernels[k] for k in atomic)
