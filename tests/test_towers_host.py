"""CPU-side checks of the tower post linear (pna_linear_towers_scaled_fwd / pna_linear_towers_bwd_data): the ctypes binding
against the header, no atomics in the built kernels, the layers' path decisions per constructor and dtype, and the numpy
restatement (tests/towers_paths_ref.py) against float64 and its exact-tier budget."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import towers_paths_ref as R
from pna_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("pna_linear_towers_scaled_fwd", "pna_linear_towers_bwd_data")
_CTYPE = {"int64_t": C.c_int64, "int32_t": C.c_int32}


def _prototype(name):
    src = open(os.path.join(ROOT, "include", "pna_b200.h")).read()
    m = re.search(r"^int\s+" + name + r"\s*\(([^)]*)\);", src, flags=re.M)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", NEW)
def test_binding_matches_the_header(name):
    params = _prototype(name)
    assert name in _lib.EXPORTED_SYMBOLS
    L = _lib.lib()
    fn = getattr(L, name)
    assert fn.restype == C.c_int and len(fn.argtypes) == len(params)
    for p, t in zip(params, fn.argtypes):
        want = C.c_void_p if "*" in p or p.startswith("pna_stream_t") else _CTYPE[p.split()[0]]
        assert t == want, (p, t)
    assert _lib.ABI_VERSION == 8 == L.pna_query(_lib.QUERY_ABI_VERSION)


def test_bad_shapes_return_status_codes():
    L = _lib.lib()
    fwd, bwd = L.pna_linear_towers_scaled_fwd, L.pna_linear_towers_bwd_data
    # (n_rows, T, F, A, O): zero rows launch nothing; T = 9, O = 65, T * O > 256, F % 4 != 0 are unsupported
    assert fwd(None, 0, None, 3, None, None, None, 0, 0, 5, 16, 4, 14, None) == 0
    assert bwd(None, 0, None, 3, None, None, 0, 0, 5, 16, 4, 14, None) == 0
    for t, f, o in ((9, 16, 8), (1, 16, 65), (8, 16, 33), (2, 18, 8)):
        assert fwd(None, 0, None, 3, None, None, None, 0, 10, t, f, 4, o, None) == -2
        assert bwd(None, 0, None, 3, None, None, 0, 10, t, f, 4, o, None) == -2
    assert fwd(None, 0, None, 6, None, None, None, 0, 10, 2, 16, 4, 8, None) == -1       # S = 6
    assert fwd(None, 400, None, 3, None, None, None, 16, 10, 2, 16, 4, 8, None) == -1    # null pointers


def test_no_atomics_in_the_tower_kernels():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    bodies = re.split(r"\n\s*Function : ", sass)
    found = [b for b in bodies if b.split("\n", 1)[0].strip().startswith("_ZN3pna15k_towers_3xtf32")]
    assert len(found) == 2                                          # forward and data gradient
    for b in found:
        ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]+)", b)
        assert ops and not any(op.split(".")[0] in ("ATOM", "ATOMS", "ATOMG", "RED", "REDG", "REDUX") for op in ops)
        assert any(op.startswith("HGMMA") for op in ops)            # the tensor cores do the products


class _FakeCuda:
    """What the path decision reads of x: device, dtype, row count (no GPU here)."""
    is_cuda = True

    def __init__(self, dtype=torch.float32, n=100):
        self.dtype, self._n = dtype, n

    def size(self, i):
        return self._n


def _pyg(**k):
    import pna_b200
    deg = torch.tensor([0, 3, 5, 2])
    kw = dict(towers=4, divide_input=True)
    kw.update(k)
    args = (kw.pop("fin", 128), kw.pop("fout", 128), ["mean", "min", "max", "std"], kw.pop("scalers", ["identity", "amplification", "attenuation"]), deg)
    return pna_b200.PNAConv(*args, **kw)


def _dgl(**k):
    import pna_b200
    kw = dict(towers=5, divide_input=True)
    kw.update(k)
    return pna_b200.PNALayer(kw.pop("fin", 70), kw.pop("fout", 70), "mean max min std",
                             kw.pop("scalers", "identity amplification attenuation"), {"log": 1.5, "lin": 3.0}, 0.0, True, True, **kw)


def test_path_decisions_per_constructor_and_dtype(monkeypatch):
    from pna_b200 import linear, padding as pad
    x = _FakeCuda(n=linear.TOWERS_COMPACT_MIN_ROWS)
    fp = lambda f: pad.padded_width(f, torch.float32)
    assert _pyg()._compact(x, fp(32))                                   # T 4, O_t 32, Fp 32
    assert _pyg(edge_dim=16)._compact(x, fp(32))
    assert _pyg(pre_layers=2, post_layers=2)._compact(x, fp(32))
    assert _pyg(fin=75, fout=75, towers=5)._compact(x, fp(15))          # O_t = 15, Fp = 16
    assert _pyg(fin=64, fout=64, towers=1)._compact(x, fp(64))          # one tower, O_t = 64
    assert not _pyg(fin=65, fout=65, towers=1, divide_input=False)._compact(x, fp(65))   # O_t = 65 > 64
    assert not _pyg(fin=72, fout=72, towers=9)._compact(x, fp(8))       # 9 towers
    assert not _pyg(scalers=["identity"])._compact(x, fp(32))           # S == 1
    assert not _pyg()._compact(_FakeCuda(torch.bfloat16), fp(32))
    assert not _pyg()._compact(_FakeCuda(n=0), fp(32))
    assert not _pyg().double()._compact(x, fp(32))
    d = _dgl()
    assert d._compact(x, fp(14))                                        # ZINC: T 5, O_t 14, Fp 16
    assert _dgl(divide_input=False, fin=16, fout=70)._compact(x, fp(16))
    assert not _dgl(scalers="identity")._compact(x, fp(14))
    assert not _dgl()._compact(_FakeCuda(torch.bfloat16), fp(14))
    assert not _dgl(towers=1, fin=70, fout=70)._compact(x, fp(70))      # O_t = 70 > 64
    assert not _pyg()._compact(_FakeCuda(n=linear.TOWERS_COMPACT_MIN_ROWS - 1), fp(32))     # small graphs
    assert not d._compact(_FakeCuda(n=linear.TOWERS_COMPACT_MIN_ROWS - 1), fp(14))
    with torch.no_grad():                                                # inference keeps the materialised path
        assert not _pyg()._compact(x, fp(32)) and not d._compact(x, fp(14))
    for var in ("PNA_B200_COMPACT_POST", "PNA_B200_TENSOR_LINEAR"):
        monkeypatch.setenv(var, "0")
        assert not _pyg()._compact(x, fp(32)) and not d._compact(x, fp(14))
        monkeypatch.delenv(var)


@pytest.mark.parametrize("case", R.CASES[:6])
def test_restatement_is_within_its_bars_of_float64(case):
    n, t_n, fp, o, n_aggr, s_n = case
    a, c, w, b, gy = R.case_data(case, grid=False)
    y, bar = R.fwd_restate(a, c, w, b, fp, n_aggr, bars=True)
    per, af = (1 + n_aggr) * fp, n_aggr * fp
    want = np.zeros_like(y, dtype=np.float64)
    ga_want = np.zeros((n, t_n * per))
    for t in range(t_n):
        a_t = a[:, t * per:(t + 1) * per]
        x = np.concatenate([a_t[:, :fp]] + [a_t[:, fp:] * c[:, s:s + 1] for s in range(s_n)], axis=1).astype(np.float64)
        want[:, t * o:(t + 1) * o] = x @ w[t].astype(np.float64).T + b[t]
        g_t = gy[:, t * o:(t + 1) * o]
        w64 = w[t].astype(np.float64)
        ga_want[:, t * per:t * per + fp] = g_t.astype(np.float64) @ w64[:, :fp]
        ga_want[:, t * per + fp:(t + 1) * per] = sum((g_t * c[:, s:s + 1]).astype(np.float64) @ w64[:, fp + s * af:fp + (s + 1) * af]
                                                     for s in range(s_n))                  # fl(c_s gy), as the kernel forms it
    assert (np.abs(y - want) <= bar).all()
    g, gbar = R.bwd_restate(gy, c, w, fp, n_aggr, bars=True)
    assert (np.abs(g - ga_want) <= gbar).all()


@pytest.mark.parametrize("case", R.CASES)
def test_grid_data_stays_in_the_exact_tier(case):
    n, t_n, fp, o, n_aggr, s_n = case
    a, c, w, b, gy = R.case_data(case, grid=True)
    assert R.budget("fwd", a, c, w, fp, n_aggr) <= 2 ** 12
    assert R.budget("bwd", gy, c, w, fp, n_aggr) <= 2 ** 12
