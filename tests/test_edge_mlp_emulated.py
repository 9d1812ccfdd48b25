"""The edge-MLP kernels (csrc/pna_edge_mlp.cu) executed on the HOST, thread by thread (tests/emu), through the real C entry
points pna_edge_mlp_fwd / pna_edge_mlp_bwd:
  * bit for bit equal to the scalar C restatement of their rounding order (tests/edge_mlp_oracle.c);
  * within (F_t + 2) * L * 2^-24 * c_L of a float64 evaluation, c_L = |A[i]| + |Bm[j]| + |b1| carried through |W_k|, |b_k|;
  * the pre-activation gradients G_k within the same kind of bar of float64 autograd;
  * bad descriptors rejected.
PNA_EMU_ASAN=1 (tests/emu/build_emu.py) bounds-checks every access of the emulated kernels."""
import ctypes as C
import importlib.util
import os
import shutil
import subprocess

import pytest
import torch

pytestmark = pytest.mark.skipif(shutil.which("g++") is None or shutil.which("gcc") is None, reason="needs g++ and gcc")

HERE = os.path.dirname(os.path.abspath(__file__))
PNA_OK, PNA_ERR_BAD_ARG, PNA_ERR_UNSUPPORTED = 0, -1, -2
P = C.c_void_p


def _build_emu():
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    return be.build("pna_edge_mlp.cu")


def _build_oracle():
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    src = os.path.join(HERE, "edge_mlp_oracle.c")
    lib = os.path.join(be.BUILD, "libedge_mlp_oracle.so")
    os.makedirs(be.BUILD, exist_ok=True)
    if not os.path.exists(lib) or os.path.getmtime(lib) < os.path.getmtime(src):
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", lib, src], check=True)
    return lib


@pytest.fixture(scope="module")
def emu():
    try:
        L = C.CDLL(_build_emu())
    except Exception as exc:            # no CUDA headers on this machine
        pytest.skip(f"emulation library did not build: {exc}")
    L.emu_last_error.restype = C.c_char_p
    L.pna_edge_mlp_fwd.argtypes = [P, P, C.c_int64, C.c_int64, P, P, P, P, P, C.c_int32, C.c_int32, C.c_int32, P, P, P]
    L.pna_edge_mlp_bwd.argtypes = [P, P, P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, P, P]
    return L


@pytest.fixture(scope="module")
def oracle():
    L = C.CDLL(_build_oracle())
    L.edge_mlp_fwd_ref.argtypes = [P, P, C.c_int64, C.c_int64, P, P, P, P, P, C.c_int, C.c_int, C.c_int, P, P]
    L.edge_mlp_bwd_ref.argtypes = [P, P, P, C.c_int64, C.c_int, C.c_int, C.c_int, P]
    return L


def _p(t):
    return None if t is None else t.data_ptr()


class Case:
    """A destination-sorted CSR with empty rows and more than one CTA of slots, random first-layer halves and weights."""

    def __init__(self, F, L, T, n=40, seed=0):
        g = torch.Generator().manual_seed(seed * 1000 + F * 31 + L * 7 + T)
        deg = torch.randint(0, 12, (n,), generator=g)
        deg[::7] = 0
        self.n, self.F, self.L, self.T = n, F, L, T
        self.rowptr = torch.cat([torch.zeros(1, dtype=torch.int64), deg.cumsum(0)]).to(torch.int32)
        self.E = int(self.rowptr[-1])
        self.col = torch.randint(0, n, (self.E,), generator=g, dtype=torch.int32)
        self.dst = torch.repeat_interleave(torch.arange(n), deg)
        TF = T * F
        self.A = torch.randn(n, TF, generator=g)
        self.Bm = torch.randn(n, TF, generator=g)
        self.b1 = 0.3 * torch.randn(TF, generator=g)
        self.W = torch.randn(L - 1, T, F, F, generator=g) / max(F, 1) ** 0.5
        self.bW = 0.3 * torch.randn(L - 1, T, F, generator=g)
        self.dM = torch.randn(self.E, TF, generator=g)

    def fwd(self, lib, fn="pna_edge_mlp_fwd"):
        TF = self.T * self.F
        M = torch.full((self.E, TF), float("nan"))
        act = torch.full((self.L - 1, self.E, TF), float("nan"))
        args = (_p(self.rowptr), _p(self.col), self.n, self.E, _p(self.A), _p(self.Bm), _p(self.b1), _p(self.W), _p(self.bW),
                self.L, self.T, self.F, _p(M), _p(act))
        if fn == "pna_edge_mlp_fwd":
            assert lib.pna_edge_mlp_fwd(*args, None) == PNA_OK, lib.emu_last_error()
        else:
            lib.edge_mlp_fwd_ref(*args)
        return M, act

    def bwd(self, lib, act, fn="pna_edge_mlp_bwd"):
        G = torch.full((self.L - 1, self.E, self.T * self.F), float("nan"))
        args = (_p(self.dM), _p(act), _p(self.W), self.E, self.L, self.T, self.F, _p(G))
        if fn == "pna_edge_mlp_bwd":
            assert lib.pna_edge_mlp_bwd(*args, None) == PNA_OK, lib.emu_last_error()
        else:
            lib.edge_mlp_bwd_ref(*args)
        return G

    def float64(self):
        """Float64 messages, activations and (autograd) pre-activation gradients of the same MLP."""
        E, T, F = self.E, self.T, self.F
        pre = [(self.A.double()[self.dst] + self.Bm.double()[self.col.long()] + self.b1.double()).requires_grad_(True)]
        z = torch.relu(pre[0])
        for k in range(2, self.L + 1):
            u = torch.einsum("toc,etc->eto", self.W[k - 2].double(), z.view(E, T, F)).reshape(E, T * F) + \
                self.bW[k - 2].double().reshape(-1)
            u.retain_grad()
            pre.append(u)
            z = u if k == self.L else torch.relu(u)
        (z * self.dM.double()).sum().backward()
        return z.detach(), [p.grad for p in pre[:-1]], [p.detach() for p in pre[:-1]]

    def bars(self):
        """(F_t + 2) * L * 2^-24 * c_L per message element; the same carried backwards for G_k, from |dM|."""
        E, T, F = self.E, self.T, self.F
        c = self.A.double().abs()[self.dst] + self.Bm.double().abs()[self.col.long()] + self.b1.double().abs()
        for k in range(2, self.L + 1):
            c = torch.einsum("toc,etc->eto", self.W[k - 2].double().abs(), c.view(E, T, F)).reshape(E, T * F) + \
                self.bW[k - 2].double().abs().reshape(-1)
        g = self.dM.double().abs()
        gb = []
        for k in range(self.L, 1, -1):
            g = torch.einsum("toc,eto->etc", self.W[k - 2].double().abs(), g.view(E, T, F)).reshape(E, T * F)
            gb.insert(0, g)
        u = 2.0 ** -24 * (F + 2) * self.L
        return u * c, [u * x for x in gb]


SHAPES = [(F, L, T) for F in (1, 3, 4, 16, 64) for L in (2, 3, 4) for T in (1, 2, 3, 4)]


@pytest.mark.parametrize("F,L,T", SHAPES)
def test_forward_and_backward_match_the_c_oracle_bit_for_bit(emu, oracle, F, L, T):
    c = Case(F, L, T)
    assert c.E > 128 and (c.rowptr[1:] == c.rowptr[:-1]).any()
    M, act = c.fwd(emu)
    M0, act0 = c.fwd(oracle, "ref")
    assert torch.equal(M.view(torch.int32), M0.view(torch.int32))
    assert torch.equal(act.view(torch.int32), act0.view(torch.int32))
    G = c.bwd(emu, act)
    G0 = c.bwd(oracle, act0, "ref")
    assert torch.equal(G.view(torch.int32), G0.view(torch.int32))


@pytest.mark.parametrize("F,L,T", SHAPES)
def test_within_the_bar_of_float64(emu, F, L, T):
    c = Case(F, L, T, seed=1)
    M, act = c.fwd(emu)
    M64, G64, pre64 = c.float64()
    barM, barG = c.bars()
    err = (M.double() - M64).abs()
    assert (err <= barM).all(), float((err / barM).max())
    G = c.bwd(emu, act)
    # a ReLU mask that fp32 and float64 set differently (a pre-activation within rounding of 0) changes the gradient of that
    # (slot, tower) by design; such rows are left out (and must be rare)
    E = c.E
    flip = torch.zeros(E, T, dtype=torch.bool)
    for k in range(L - 1):
        flip |= ((act[k] > 0) != (pre64[k] > 0)).view(E, T, F).any(2)
    assert flip.float().mean() < 0.02
    keep = (~flip).repeat_interleave(F, 1)
    for k in range(L - 1):
        err = (G[k].double() - G64[k]).abs()
        assert ((err <= barG[k]) | ~keep).all(), (k, float((err / barG[k].clamp_min(1e-300))[keep].max()))


def test_no_stored_activations_gives_the_same_messages(emu):
    c = Case(16, 3, 2, seed=2)
    M, _ = c.fwd(emu)
    M2 = torch.empty_like(M)
    assert emu.pna_edge_mlp_fwd(_p(c.rowptr), _p(c.col), c.n, c.E, _p(c.A), _p(c.Bm), _p(c.b1), _p(c.W), _p(c.bW), c.L, c.T,
                                c.F, _p(M2), None, None) == PNA_OK
    assert torch.equal(M, M2)


def test_bad_descriptors_are_rejected(emu):
    c = Case(8, 3, 2, seed=3)
    M = torch.empty(c.E, 16)
    G = torch.empty(2, c.E, 16)
    act = torch.zeros(2, c.E, 16)

    def fwd(L=3, T=2, F=8, E=None, **null):
        ptrs = dict(rowptr=c.rowptr, col=c.col, a=c.A, b=c.Bm, b1=c.b1, W=c.W, bW=c.bW, M=M)
        for k in null:
            ptrs[k] = None
        return emu.pna_edge_mlp_fwd(_p(ptrs["rowptr"]), _p(ptrs["col"]), c.n, c.E if E is None else E, _p(ptrs["a"]),
                                    _p(ptrs["b"]), _p(ptrs["b1"]), _p(ptrs["W"]), _p(ptrs["bW"]), L, T, F, _p(ptrs["M"]),
                                    None, None)

    def bwd(L=3, T=2, F=8, **null):
        ptrs = dict(dM=c.dM, act=act, W=c.W, G=G)
        for k in null:
            ptrs[k] = None
        return emu.pna_edge_mlp_bwd(_p(ptrs["dM"]), _p(ptrs["act"]), _p(ptrs["W"]), c.E, L, T, F, _p(ptrs["G"]), None)

    for fn in (fwd, bwd):
        assert fn(L=1) == PNA_ERR_BAD_ARG and b"n_layers" in emu.emu_last_error()
        assert fn(L=0) == PNA_ERR_BAD_ARG
        assert fn(F=65) == PNA_ERR_UNSUPPORTED and b"width" in emu.emu_last_error()
        assert fn(F=0) == PNA_ERR_BAD_ARG
        assert fn(T=0) == PNA_ERR_BAD_ARG
    assert fwd(E=-1) == PNA_ERR_BAD_ARG
    for k in ("rowptr", "col", "a", "b", "b1", "W", "bW", "M"):
        assert fwd(**{k: 1}) == PNA_ERR_BAD_ARG, k
    for k in ("dM", "act", "W", "G"):
        assert bwd(**{k: 1}) == PNA_ERR_BAD_ARG, k
    assert fwd(E=0, rowptr=1, col=1, a=1) == PNA_OK        # nothing to do: no pointer is read
