"""Mixed precision on the host: the layers' kernel selection under bf16, fp16 and no autocast (the one autocast helper,
aggregate.boundary_dtype, is monkeypatched: torch.autocast("cuda") switches itself off without a GPU), the fp32-only
wrappers' TypeError before any launch, the binding of the bf16 entry points against the header, and their SASS."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from pna_b200 import _lib, aggregate, dense, dgl_layers, edge_mlp, linear, pyg, readout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = {"pna_edge_msg_fwd_bf16": "pna_edge_msg_fwd", "pna_edge_msg_bwd_bf16": "pna_edge_msg_bwd",
       "pna_linear_towers_scaled_fwd_bf16": "pna_linear_towers_scaled_fwd"}
MODES = {"bf16": torch.bfloat16, "fp16": torch.float32, "off": None}     # autocast dtype -> boundary_dtype()


@pytest.fixture(params=list(MODES))
def mode(request, monkeypatch):
    monkeypatch.setattr(aggregate, "boundary_dtype", lambda: MODES[request.param])
    return request.param


class _Fake:
    """What the path decisions read of a tensor: device, dtype, row count (no GPU here)."""
    is_cuda = True

    def __init__(self, dtype=torch.float32, n=100):
        self.dtype, self._n = dtype, n

    def size(self, i):
        return self._n


def _conv(**k):
    kw = dict(towers=4, divide_input=True)
    kw.update(k)
    return pyg.PNAConv(128, 128, ["mean", "min", "max", "std"], ["identity", "amplification", "attenuation"],
                       torch.tensor([0, 3, 5, 2]), **kw)


def _dgl(**k):
    return dgl_layers.PNALayer(70, 70, "mean max min std", "identity amplification attenuation", {"log": 1.5, "lin": 3.0}, 0.0,
                               True, True, towers=5, **k)


def test_boundary_dtype_reads_cuda_autocast():
    assert aggregate.boundary_dtype() is None             # no autocast region (and none can be entered without CUDA)
    h = torch.zeros(2, dtype=torch.float16)
    assert aggregate.at_boundary(h) is h and aggregate.at_boundary(None) is None


def test_at_boundary_upcasts_fp16_only(mode):
    h, b, f = (torch.zeros(2, 3, dtype=d) for d in (torch.float16, torch.bfloat16, torch.float32))
    assert aggregate.at_boundary(h).dtype == (torch.float16 if mode == "off" else torch.float32)
    assert aggregate.at_boundary(b) is b and aggregate.at_boundary(f) is f


def test_message_kernel_selection(mode):
    """Inside autocast the fused messages are taken whatever the input's dtype (the GEMMs make the operands); outside,
    as before, float32 inputs only.  bf16 weights (an explicit bf16 model) never."""
    big = edge_mlp.FUSED_TRAINING_MIN_EDGES
    amp = mode != "off"
    for x in (_Fake(torch.float32), _Fake(torch.bfloat16), _Fake(torch.float16)):
        want = amp or x.dtype == torch.float32
        conv = _conv(edge_dim=16, pre_layers=2)
        assert conv._fused_messages_ok(x, x, big) == want, (mode, x.dtype)
        assert not conv._fused_messages_ok(x, x, big - 1)                    # small training steps: torch path, unchanged
        assert not conv.bfloat16()._fused_messages_ok(x, x, big)
        lay = _dgl(pretrans_layers=2, edge_features=True, edge_dim=4)
        assert lay._fused_messages_ok(x, x, big) == want, (mode, x.dtype)
        assert not lay._fused_messages_ok(x, None, big)                      # edge features announced but not given
        assert not lay.bfloat16()._fused_messages_ok(x, x, big)


def test_compact_tower_selection(mode):
    """The compact tower path: under either autocast for any input dtype (the aggregate is bf16 or fp32), outside autocast
    for float32 only; fp32 weights always; the shape and size rules unchanged."""
    n = linear.TOWERS_COMPACT_MIN_ROWS
    amp = mode != "off"
    for dt in (torch.float32, torch.bfloat16):
        want = amp or dt == torch.float32
        assert _conv()._compact(_Fake(dt, n), 32) == want
        assert _dgl()._compact(_Fake(dt, n), 16) == want
        assert not _conv()._compact(_Fake(dt, n - 1), 32) and not _dgl()._compact(_Fake(dt, n - 1), 16)
        assert not _conv().bfloat16()._compact(_Fake(dt, n), 32) and not _dgl().bfloat16()._compact(_Fake(dt, n), 16)
    with torch.no_grad():
        assert not _conv()._compact(_Fake(n=n), 32)
    # the PNAConvSimple / PNASimpleLayer compact path keeps its float32-only answer
    assert not linear.compact_path_ok(_Fake(torch.bfloat16), 128, 128, 3)
    assert linear.compact_path_ok(_Fake(torch.float32), 128, 128, 3)


def test_dense_edge_mlp_takes_the_bf16_message_entry(monkeypatch):
    """bf16 A / Bm with fp32 weights go to edge_messages without edge term at pitch F_t; bf16 weights do not (an explicit
    bf16 model keeps the fp32-only edge-MLP check)."""
    seen = []
    monkeypatch.setattr(edge_mlp, "edge_messages", lambda *a, **k: seen.append((a, k)) or "msgs")
    A = torch.zeros(4, 6, dtype=torch.bfloat16)
    W, bW = torch.zeros(1, 2, 3, 3), torch.zeros(1, 2, 3)
    assert edge_mlp.edge_mlp(A, A, torch.zeros(6), W, bW, None, 2) == "msgs"
    assert seen and seen[0][1] == {} and len(seen[0][0]) == 7
    with pytest.raises(TypeError):
        edge_mlp.edge_mlp(A, A, torch.zeros(6, dtype=torch.bfloat16), W.bfloat16(), bW.bfloat16(),
                          type("G", (), {"n_nodes": 4})(), 2)


def test_readout_and_dense_call_the_boundary(monkeypatch):
    """The readout hands its input through at_boundary (fp16 under autocast: fp32), the dense edge-MLP path its A / Bm."""
    calls = []
    monkeypatch.setattr(readout, "pna_aggregate", lambda x, *a, **k: calls.append(x.dtype) or x)
    monkeypatch.setattr(readout, "batch_csr", lambda b, n: None)
    monkeypatch.setattr(aggregate, "boundary_dtype", lambda: torch.float32)
    readout.segment_reduce(torch.zeros(3, 2, dtype=torch.float16), torch.zeros(3, dtype=torch.long), 1)
    monkeypatch.setattr(aggregate, "boundary_dtype", lambda: None)
    readout.segment_reduce(torch.zeros(3, 2, dtype=torch.float16), torch.zeros(3, dtype=torch.long), 1)
    assert calls == [torch.float32, torch.float16]
    assert dense.at_boundary is aggregate.at_boundary


def _no_launch(monkeypatch):
    def boom():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", boom)


def test_fp32_wrappers_raise_type_error_before_any_launch(monkeypatch):
    _no_launch(monkeypatch)
    bf = lambda *s: torch.zeros(*s, dtype=torch.bfloat16)
    f32 = lambda *s: torch.zeros(*s)
    calls = [
        lambda: linear.linear_tf32x3(bf(4, 32), f32(64, 32), None),
        lambda: linear.linear_tf32x3(f32(4, 32), bf(64, 32), f32(64)),
        lambda: linear.linear_tf32x3(f32(4, 32), f32(64, 32), bf(64)),
        lambda: linear.linear_scaled_tf32x3(bf(4, 32), f32(4, 3), f32(64, 96), None),
        lambda: linear.linear_scaled_tf32x3(f32(4, 32), bf(4, 3), f32(64, 96), None),
        lambda: linear.linear_bwd_tf32x3(bf(4, 64), f32(4, 32), None, f32(64, 32)),
        lambda: linear.linear_bwd_tf32x3(f32(4, 64), bf(4, 32), None, f32(64, 32)),
        lambda: linear.linear_bwd_tf32x3(f32(4, 64), f32(4, 32), None, bf(64, 32)),
        # the towers forward takes a bf16 aggregate, but no other bf16 operand, and no fp16 aggregate
        lambda: linear.linear_towers_scaled_tf32x3(f32(4, 2 * 5 * 4).half(), f32(4, 3), f32(2, 8, 4 + 3 * 16), None),
        lambda: linear.linear_towers_scaled_tf32x3(bf(4, 2 * 5 * 4), bf(4, 3), f32(2, 8, 4 + 3 * 16), None),
        lambda: linear.linear_towers_scaled_tf32x3(bf(4, 2 * 5 * 4), f32(4, 3), bf(2, 8, 4 + 3 * 16), None),
        lambda: linear.linear_towers_scaled_tf32x3(bf(4, 2 * 5 * 4), f32(4, 3), f32(2, 8, 4 + 3 * 16), bf(2, 8)),
        lambda: linear.linear_towers_bwd_data(bf(4, 16), f32(4, 3), f32(2, 8, 4 + 3 * 16), (4, 40)),
        lambda: linear.linear_towers_bwd_data(f32(4, 16), f32(4, 3), bf(2, 8, 4 + 3 * 16), (4, 40)),
    ]
    for i, call in enumerate(calls):
        with pytest.raises(TypeError):
            call()


def _prototype(name):
    src = open(os.path.join(ROOT, "include", "pna_b200.h")).read()
    m = re.search(r"^int\s+" + name + r"\s*\(([^)]*)\);", src, flags=re.M)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", list(NEW))
def test_bf16_entry_points_match_the_header(name):
    """Exported, declared with the fp32 call's argument count (2-byte operands as void pointers), bound with its ctypes."""
    params, fp32 = _prototype(name), _prototype(NEW[name])
    assert name in _lib.EXPORTED_SYMBOLS and len(params) == len(fp32)
    for p, q in zip(params, fp32):
        assert p.split()[-1] == q.split()[-1] and ("*" in p) == ("*" in q), (p, q)
    L = _lib.lib()
    fn = getattr(L, name)
    assert fn.restype == C.c_int and fn.argtypes == getattr(L, NEW[name]).argtypes
    assert _lib.ABI_VERSION == 8 == L.pna_query(_lib.QUERY_ABI_VERSION)
    assert _lib.EDGE_MLP_MAX_WIDTH == 64


def test_bf16_entry_points_refuse_what_the_fp32_ones_refuse():
    L = _lib.lib()
    fwd, bwd, twr = L.pna_edge_msg_fwd_bf16, L.pna_edge_msg_bwd_bf16, L.pna_linear_towers_scaled_fwd_bf16
    assert fwd(None, None, 4, 10, None, None, None, None, None, None, 0, 2, 8, 8, None, None, None) == -1     # n_layers 0
    assert fwd(None, None, 4, 10, None, None, None, None, None, None, 2, 2, 65, 65, None, None, None) == -2   # width 65
    assert fwd(None, None, 4, 10, None, None, None, None, None, None, 1, 2, 8, 7, None, None, None) == -1     # pitch < width
    assert fwd(None, None, 4, 10, None, None, None, None, None, None, 1, 2, 8, 8, None, None, None) == -1     # null pointers
    assert fwd(None, None, 4, 0, None, None, None, None, None, None, 1, 2, 8, 8, None, None, None) == 0       # nothing to do
    assert bwd(None, 8, None, None, 10, 1, 2, 8, None, None) == -1
    assert bwd(None, 8, None, None, 10, 2, 2, 65, None, None) == -2
    assert twr(None, 0, None, 3, None, None, None, 0, 0, 5, 16, 4, 14, None) == 0
    assert twr(None, 0, None, 3, None, None, None, 0, 10, 9, 16, 4, 8, None) == -2
    assert twr(None, 400, None, 3, None, None, None, 16, 10, 2, 16, 4, 8, None) == -1


def test_no_atomics_in_the_bf16_instances():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if "k_bf16_msg_" in m.group(1) or "k_towers_bf16_3xtf32" in m.group(1):
            kernels[m.group(1)] = m.group(2)
    msg = [k for k in kernels if "k_bf16_msg_" in k]
    assert len(msg) == 21 and len(kernels) == 22     # fwd, bwd: 5 width buckets x exact or not; one-layer fwd; the towers fwd
    for k, body in kernels.items():
        ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]+)", body)
        assert ops and not any(op.split(".")[0] in ("ATOM", "ATOMS", "ATOMG", "RED", "REDG", "REDUX") for op in ops), k
    assert any(op.startswith("HGMMA") for op in re.findall(r"\b(HGMMA\S*)", kernels[[k for k in kernels if "towers" in k][0]]))
