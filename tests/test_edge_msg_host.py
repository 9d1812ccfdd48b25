"""Host-side plumbing of the edge-message path of the DGL PNALayer and the PyG PNAConv: the reference state_dicts of the
fixtures load strictly, the binding matches the header, the layers pick the kernel for exactly the inputs it takes, and the
SASS of the edge-message kernels has no atomics."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from pna_b200 import _lib, dgl_layers, edge_mlp, pyg

HERE = os.path.dirname(os.path.abspath(__file__))
DGL_FIXTURES = ("dgl_edge_msgs", "dgl_edge_msgs_zinc", "dgl_edge_msgs_wide75")


def _load(name):
    return torch.load(os.path.join(HERE, "golden", name + ".pt"), weights_only=False)


def test_reference_state_dicts_load_strictly():
    layers = set()
    for fixture in DGL_FIXTURES:
        for name, c in _load(fixture)["cases"].items():
            lay = dgl_layers.PNALayer(aggregators=c["aggregators"], scalers=c["scalers"], avg_d=c["avg_d"], **c["ctor"])
            lay.load_state_dict(c["state_dict"], strict=True)
            assert all(tw.pretrans.is_linear_relu() for tw in lay.towers), name
            assert set(c["params64"]) == set(c["ref_err"]) == {k for k, _ in lay.named_parameters()}, name
            layers.add(c["ctor"]["pretrans_layers"])
    assert layers == {1, 2, 3}
    g = _load("pyg_edge_msgs")
    for name, c in g["cases"].items():
        conv = pyg.PNAConv(aggregators=c["aggregators"], scalers=c["scalers"], deg=c["deg"], **c["ctor"])
        conv.load_state_dict(c["state_dict"], strict=True)
    # every graph has an in-degree-0 node and a row above the split threshold
    for name in DGL_FIXTURES + ("pyg_edge_msgs",):
        indeg = torch.bincount(_load(name)["edge_index"][1])
        assert int(indeg.min()) == 0 and int(indeg.max()) >= 256


def test_binding_matches_the_header():
    assert _lib.ABI_VERSION == 8
    hdr = open(os.path.join(os.path.dirname(HERE), "include", "pna_b200.h")).read()
    assert {"pna_edge_msg_fwd", "pna_edge_msg_bwd"} <= set(_lib.EXPORTED_SYMBOLS)
    for name, n_args in (("pna_edge_msg_fwd", 17), ("pna_edge_msg_bwd", 10)):
        decl = re.search(rf"int {name}\((.*?)\);", hdr, re.S).group(1)
        assert len(decl.split(",")) == n_args, name


def test_kernel_selection_follows_the_inputs():
    """float32 CUDA inputs take the kernel; other dtypes, L >= 2 above the 64-wide register limit, and training steps on
    small graphs do not."""
    avg = {"log": 1.5, "lin": 3.0}
    big = edge_mlp.FUSED_TRAINING_MIN_EDGES
    lay = dgl_layers.PNALayer(20, 20, "mean", "identity", avg, 0.0, False, False, towers=5, pretrans_layers=2,
                              edge_features=True, edge_dim=4)
    h32 = torch.zeros(3, 20)
    e32 = torch.zeros(3, 4)
    assert not lay._fused_messages_ok(h32, e32, 0)                       # a CPU tensor
    fake = type("T", (), {"is_cuda": True, "dtype": torch.float32})
    fake16 = type("T", (), {"is_cuda": True, "dtype": torch.bfloat16})
    assert lay._fused_messages_ok(fake, fake, big) and not lay._fused_messages_ok(fake16, fake16, big)
    assert not lay._fused_messages_ok(fake, None, big)                     # edge features announced but not given
    wide = dgl_layers.PNALayer(66, 66, "mean", "identity", avg, 0.0, False, False, towers=1, pretrans_layers=2)
    assert not wide._fused_messages_ok(fake, None, big)
    wide1 = dgl_layers.PNALayer(75, 75, "mean", "identity", avg, 0.0, False, False, towers=5, pretrans_layers=1,
                                divide_input=False, edge_features=True, edge_dim=4)
    assert wide1._fused_messages_ok(fake, fake, big)                       # one layer: any width
    wide1.towers[0].pretrans.fully_connected[0].dropout = torch.nn.Dropout(0.1)
    assert not wide1._fused_messages_ok(fake, fake, big)                   # not a Linear/ReLU stack
    deg = torch.tensor([0, 4, 2])
    conv = pyg.PNAConv(16, 16, ["mean"], ["identity"], deg, edge_dim=4, towers=2, pre_layers=2)
    assert conv._fused_messages_ok(fake, fake, big) and not conv._fused_messages_ok(fake16, fake16, big)
    assert not pyg.PNAConv(65, 65, ["mean"], ["identity"], deg, pre_layers=2)._fused_messages_ok(fake, None, big)
    assert pyg.PNAConv(65, 65, ["mean"], ["identity"], deg, edge_dim=3)._fused_messages_ok(fake, fake, big)
    # with autograd, only from FUSED_TRAINING_MIN_EDGES edges on; without, any size
    assert not conv._fused_messages_ok(fake, fake, big - 1) and conv._fused_messages_ok(fake, fake, big)
    assert not lay._fused_messages_ok(fake, fake, big - 1) and lay._fused_messages_ok(fake, fake, big)
    with torch.no_grad():
        assert conv._fused_messages_ok(fake, fake, 1) and lay._fused_messages_ok(fake, fake, 1)


def test_edge_msg_kernels_have_no_atomics():
    """cuobjdump of the built library: every instance of k_edge_msg_fwd / k_edge_msg_fwd_affine / k_edge_msg_bwd contains no
    ATOM / RED."""
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if "k_edge_msg_" in m.group(1):
            kernels[m.group(1)] = re.findall(r"\b(?:ATOM|ATOMG|RED|REDG)\b", m.group(2))
    assert len(kernels) == 21          # fwd and bwd: 5 width buckets x exact or not; the one-layer forward
    for k, atoms in kernels.items():
        assert not atoms, k
