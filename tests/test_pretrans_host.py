"""Host-side plumbing of the dense layer with pretrans_layers >= 2: reference state_dicts load, the width limit is named,
normalised_mean takes messages in CSR order with degree_col, the binding matches the header, and the SASS of the edge-MLP
kernels has no atomics."""
import os
import re
import shutil
import subprocess
import types

import pytest
import torch

from pna_b200 import _lib, aggregate as agg, dense

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "dense_pretrans.pt")


def test_reference_state_dicts_load_strictly():
    g = torch.load(GOLDEN)
    assert {c["ctor"]["pretrans_layers"] for c in g["cases"].values()} == {2, 3}
    for name, c in g["cases"].items():
        lay = dense.PNALayer(aggregators=c["aggregators"], scalers=g["scalers"], avg_d=c["avg_d"], **c["ctor"])
        lay.load_state_dict(c["state_dict"], strict=True)
        L = c["ctor"]["pretrans_layers"]
        assert len(lay.towers[0].pretrans.fully_connected) == L and not lay.towers[0].pretrans.is_single_affine(), name


def test_tower_width_above_the_kernel_limit_is_refused():
    avg = {"log": 1.5, "lin": 3.0}
    dense.PNALayer(128, 128, ["mean"], ["identity"], avg, towers=2, pretrans_layers=2)          # F_t = 64
    with pytest.raises(NotImplementedError, match="64"):
        dense.PNALayer(130, 130, ["mean"], ["identity"], avg, towers=2, pretrans_layers=2)
    with pytest.raises(NotImplementedError, match="64"):
        dense.PNALayer(72, 72, ["mean"], ["identity"], avg, towers=2, pretrans_layers=3, divide_input=False)
    dense.PNALayer(130, 130, ["mean"], ["identity"], avg, towers=2, pretrans_layers=1)          # the affine path: no limit
    # moments with self_loop keep their refusal whatever pretrans_layers is
    with pytest.raises(NotImplementedError, match="moment"):
        dense.PNALayer(8, 8, ["mean", "moment3"], ["identity"], avg, self_loop=True, pretrans_layers=2)


def test_normalised_mean_takes_messages_in_csr_order_with_degree_col():
    csr = types.SimpleNamespace(n_nodes=5, n_edges=7)
    avg = {"log": 1.0, "lin": 1.0}
    dcol = torch.zeros(7, dtype=torch.int32)
    # without degree_col: the refusal of the parent library; with it, the call passes this check (and stops at the next:
    # no CUDA tensor here)
    with pytest.raises(ValueError, match="normalised_mean"):
        agg.aggregate_forward(torch.zeros(7, 4), csr, ["normalised_mean"], ["identity"], avg, messages_in_csr_order=True)
    with pytest.raises(ValueError, match="CUDA"):
        agg.aggregate_forward(torch.zeros(7, 4), csr, ["normalised_mean"], ["identity"], avg, messages_in_csr_order=True,
                              degree_col=dcol)
    with pytest.raises(ValueError, match="normalised_mean"):       # a peer table stays refused
        agg.aggregate_forward(torch.zeros(5, 4), csr, ["normalised_mean"], ["identity"], avg, degree_col=dcol,
                              peer=(torch.zeros(2, dtype=torch.int64), 8))


def test_binding_matches_the_header():
    names = [f[0] for f in _lib.AggStruct._fields_]
    assert names[-1] == "degree_col" and names[-2] == "work_counter"      # appended: the ABI stays version 8
    assert _lib.ABI_VERSION == 8
    hdr = open(os.path.join(os.path.dirname(HERE), "include", "pna_b200.h")).read()
    assert re.search(r"#define PNA_EDGE_MLP_MAX_WIDTH (\d+)", hdr).group(1) == str(_lib.EDGE_MLP_MAX_WIDTH)
    assert {"pna_edge_mlp_fwd", "pna_edge_mlp_bwd"} <= set(_lib.EXPORTED_SYMBOLS)


def test_edge_mlp_kernels_have_no_atomics():
    """cuobjdump of the built library: every instance of k_edge_mlp_fwd / k_edge_mlp_bwd (5 width buckets x exact or not)
    contains no ATOM / RED."""
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if "k_edge_mlp_" in m.group(1):
            kernels[m.group(1)] = re.findall(r"\b(?:ATOM|ATOMG|RED|REDG)\b", m.group(2))
    assert len(kernels) == 20
    for k, atoms in kernels.items():
        assert not atoms, k
