"""Host-side plumbing of the moment aggregators: codes, the layers that take them and those that do not, the backward mode
they select, and the SASS of their deterministic instances."""
import contextlib
import types

import pytest
import torch

from pna_b200 import _lib, aggregate as agg


def test_codes_pack_into_nibbles():
    assert [_lib.ALL_AGGR_CODES[m] for m in _lib.MOMENTS] == [6, 7, 8]
    assert all(m not in _lib.AGGR_CODES for m in _lib.MOMENTS)        # the table every flavour accepts is unchanged
    n, codes = _lib.pack_codes(["mean", "moment3", "max", "moment4", "moment5", "std"], _lib.ALL_AGGR_CODES, "aggregator")
    assert n == 6 and codes == 1 | 6 << 4 | 3 << 8 | 7 << 12 | 8 << 16 | 5 << 20


def test_dense_layer_accepts_moments_and_refuses_them_with_self_loop():
    from pna_b200 import dense
    avg = {"log": 1.5, "lin": 3.0}
    lay = dense.PNALayer(8, 8, ["mean", "moment3", "moment5"], ["identity"], avg, towers=2)
    assert lay.towers[0].posttrans.fully_connected[0].linear.in_features == (3 + 1) * 4
    for m in _lib.MOMENTS:
        assert m in dense._SELF_FIRST
        with pytest.raises(NotImplementedError, match="self_loop"):
            dense.PNALayer(8, 8, ["mean", m], ["identity"], avg, self_loop=True)
    dense.PNALayer(8, 8, ["mean", "std"], ["identity"], avg, self_loop=True)    # unchanged without moments


@pytest.mark.parametrize("m", ["moment3", "moment4", "moment5"])
def test_pyg_and_dgl_layers_still_refuse_moments(m):
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


@pytest.mark.parametrize("aggrs,want", [(["mean", "moment4"], "pna_aggregate_bwd"), (["mean", "std"], "pna_aggregate_bwd_coef")])
def test_coef_mode_takes_the_atomic_path_for_moments(monkeypatch, aggrs, want):
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


def test_deterministic_moment_instances_have_no_atomics():
    """cuobjdump of the built library: the moment kernels pna_aggregate_bwd_slots launches contain no ATOM / RED; the atomic
    instance of the row kernel still does (it adds into grad_gathered[col[slot]])."""
    import os
    import re
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump, cu++filt and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if "k_mom_" in m.group(1):
            kernels[m.group(1)] = re.findall(r"\b(?:ATOM|ATOMG|RED|REDG)\b", m.group(2))
    names = subprocess.run(["cu++filt"], input="\n".join(kernels), capture_output=True, text=True, check=True).stdout.split("\n")
    demangled = dict(zip(kernels, names))
    atomic = [k for k, n in demangled.items() if ("k_mom_bwd_rows" in n or "k_mom_bwd_chunk_grad" in n) and "(bool)0>" in n]
    # every other moment kernel: the forward, the shared split-row passes and the per-slot (deterministic) instances
    others = [k for k in demangled if k not in atomic]
    assert len(atomic) == 4 and len(others) == 9 + 12      # 9 forward, 16 backward instances in all
    for k in others:
        assert not kernels[k], f"{demangled[k]}: {kernels[k][:4]}"
    assert all(kernels[k] for k in atomic)
