"""The edge-message kernels (csrc/pna_edge_mlp.cu: k_edge_msg_fwd, k_edge_msg_fwd_affine, k_edge_msg_bwd) executed on the
HOST, thread by thread (tests/emu), through the real C entry points pna_edge_msg_fwd / pna_edge_msg_bwd:
  * bit for bit equal to the scalar C restatement of their rounding order (tests/edge_msg_oracle.c), over L = 1..4, tower
    widths up to 64 (up to 130 at L = 1), 1 to 5 towers, pitch = width and padded, with and without the edge term;
  * without an edge term and at pitch = width, bit for bit equal to pna_edge_mlp_fwd / pna_edge_mlp_bwd;
  * pad columns exactly 0;
  * within (F_t + 3) * L * 2^-24 * c_L of a float64 evaluation, c_1 = |A[i]| + |Bm[j]| + |b1| + |C[s]| carried through
    |W_k|, |b_k|; the pre-activation gradients within the same kind of bar of float64 autograd;
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
P_ = C.c_void_p


def _build_emu_module():
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    return be


def _build_oracle():
    be = _build_emu_module()
    src = os.path.join(HERE, "edge_msg_oracle.c")
    lib = os.path.join(be.BUILD, "libedge_msg_oracle.so")
    os.makedirs(be.BUILD, exist_ok=True)
    if not os.path.exists(lib) or os.path.getmtime(lib) < os.path.getmtime(src):
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", lib, src], check=True)
    return lib


@pytest.fixture(scope="module")
def emu():
    try:
        L = C.CDLL(_build_emu_module().build("pna_edge_mlp.cu"))
    except Exception as exc:            # no CUDA headers on this machine
        pytest.skip(f"emulation library did not build: {exc}")
    L.emu_last_error.restype = C.c_char_p
    L.pna_edge_msg_fwd.argtypes = [P_, P_, C.c_int64, C.c_int64, P_, P_, P_, P_, P_, P_, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_int32, P_, P_, P_]
    L.pna_edge_msg_bwd.argtypes = [P_, C.c_int32, P_, P_, C.c_int64, C.c_int32, C.c_int32, C.c_int32, P_, P_]
    L.pna_edge_mlp_fwd.argtypes = [P_, P_, C.c_int64, C.c_int64, P_, P_, P_, P_, P_, C.c_int32, C.c_int32, C.c_int32, P_, P_, P_]
    L.pna_edge_mlp_bwd.argtypes = [P_, P_, P_, C.c_int64, C.c_int32, C.c_int32, C.c_int32, P_, P_]
    return L


@pytest.fixture(scope="module")
def oracle():
    L = C.CDLL(_build_oracle())
    L.edge_msg_fwd_ref.argtypes = [P_, P_, C.c_int64, C.c_int64, P_, P_, P_, P_, P_, P_, C.c_int, C.c_int, C.c_int, C.c_int,
                                   P_, P_]
    L.edge_msg_bwd_ref.argtypes = [P_, C.c_int, P_, P_, C.c_int64, C.c_int, C.c_int, C.c_int, P_]
    return L


def _p(t):
    return None if t is None else t.data_ptr()


def _padded(F):
    """A pitch above F: the aggregation's 16-byte width, or F + 3 where F already is a multiple of 4."""
    return (F + 3) // 4 * 4 if F % 4 else F + 3


class Case:
    """A destination-sorted CSR with empty rows and more than one CTA of slots, random first-layer halves, edge term
    and weights."""

    def __init__(self, F, L, T, P=None, term=True, n=48, seed=0):
        g = torch.Generator().manual_seed(seed * 1000 + F * 31 + L * 7 + T)
        deg = torch.randint(0, 12, (n,), generator=g)
        deg[::7] = 0
        self.n, self.F, self.L, self.T, self.P = n, F, L, T, F if P is None else P
        self.rowptr = torch.cat([torch.zeros(1, dtype=torch.int64), deg.cumsum(0)]).to(torch.int32)
        self.E = int(self.rowptr[-1])
        self.col = torch.randint(0, n, (self.E,), generator=g, dtype=torch.int32)
        self.dst = torch.repeat_interleave(torch.arange(n), deg)
        TF = T * F
        self.A = torch.randn(n, TF, generator=g)
        self.Bm = torch.randn(n, TF, generator=g)
        self.b1 = 0.3 * torch.randn(TF, generator=g)
        self.C = torch.randn(self.E, TF, generator=g) if term else None
        self.W = torch.randn(L - 1, T, F, F, generator=g) / max(F, 1) ** 0.5
        self.bW = 0.3 * torch.randn(L - 1, T, F, generator=g)
        self.dM = torch.randn(self.E, T * self.P, generator=g)

    def fwd(self, lib, ref=False):
        M = torch.full((self.E, self.T * self.P), float("nan"))
        act = torch.full((max(self.L - 1, 0), self.E, self.T * self.F), float("nan"))
        args = (_p(self.rowptr), _p(self.col), self.n, self.E, _p(self.A), _p(self.Bm), _p(self.b1), _p(self.C),
                _p(self.W), _p(self.bW), self.L, self.T, self.F, self.P, _p(M), _p(act) if self.L > 1 else None)
        if ref:
            lib.edge_msg_fwd_ref(*args)
        else:
            assert lib.pna_edge_msg_fwd(*args, None) == PNA_OK, lib.emu_last_error()
        return M, act

    def bwd(self, lib, act, ref=False):
        G = torch.full((self.L - 1, self.E, self.T * self.F), float("nan"))
        args = (_p(self.dM), self.P, _p(act), _p(self.W), self.E, self.L, self.T, self.F, _p(G))
        if ref:
            lib.edge_msg_bwd_ref(*args)
        else:
            assert lib.pna_edge_msg_bwd(*args, None) == PNA_OK, lib.emu_last_error()
        return G

    def unpadded(self, M):
        return M.view(self.E, self.T, self.P)[:, :, :self.F].reshape(self.E, self.T * self.F)

    def float64(self):
        """Float64 messages [E, T*F], and (autograd) pre-activation gradients of layers 1 .. L-1 and pre-activations."""
        E, T, F = self.E, self.T, self.F
        u1 = self.A.double()[self.dst] + self.Bm.double()[self.col.long()] + self.b1.double()
        if self.C is not None:
            u1 = u1 + self.C.double()
        pre = [u1.requires_grad_(True)]
        z = u1 if self.L == 1 else torch.relu(u1)
        for k in range(2, self.L + 1):
            u = torch.einsum("toc,etc->eto", self.W[k - 2].double(), z.view(E, T, F)).reshape(E, T * F) + \
                self.bW[k - 2].double().reshape(-1)
            u.retain_grad()
            pre.append(u)
            z = u if k == self.L else torch.relu(u)
        (z * self.unpadded(self.dM).double()).sum().backward()
        return z.detach(), [p.grad for p in pre[:-1]], [p.detach() for p in pre[:-1]]

    def bars(self):
        """(F_t + 3) * L * 2^-24 * c_L per message element; the same carried backwards for G_k, from |dM|."""
        E, T, F = self.E, self.T, self.F
        c = self.A.double().abs()[self.dst] + self.Bm.double().abs()[self.col.long()] + self.b1.double().abs()
        if self.C is not None:
            c = c + self.C.double().abs()
        for k in range(2, self.L + 1):
            c = torch.einsum("toc,etc->eto", self.W[k - 2].double().abs(), c.view(E, T, F)).reshape(E, T * F) + \
                self.bW[k - 2].double().abs().reshape(-1)
        g = self.unpadded(self.dM).double().abs()
        gb = []
        for k in range(self.L, 1, -1):
            g = torch.einsum("toc,eto->etc", self.W[k - 2].double().abs(), g.view(E, T, F)).reshape(E, T * F)
            gb.insert(0, g)
        u = 2.0 ** -24 * (F + 3) * self.L
        return u * c, [u * x for x in gb]


def _bits(t):
    return t.view(torch.int32)


SHAPES = ([(1, F, T) for F in (1, 5, 14, 16, 20, 64, 75, 130) for T in (1, 2, 5)] +
          [(L, F, T) for L in (2, 3, 4) for F in (1, 5, 14, 16, 20, 64) for T in (1, 2, 5)])


@pytest.mark.parametrize("term", [True, False])
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("L,F,T", SHAPES)
def test_forward_and_backward_match_the_c_oracle_bit_for_bit(emu, oracle, L, F, T, padded, term):
    c = Case(F, L, T, P=_padded(F) if padded else F, term=term)
    assert c.E > 128 and (c.rowptr[1:] == c.rowptr[:-1]).any()
    M, act = c.fwd(emu)
    M0, act0 = c.fwd(oracle, ref=True)
    assert torch.equal(_bits(M), _bits(M0))
    pads = M.view(c.E, T, c.P)[:, :, F:]
    assert torch.equal(_bits(pads), torch.zeros_like(_bits(pads)))          # exact +0.0, every pad column
    if L == 1:
        assert emu.pna_edge_msg_bwd(_p(c.dM), c.P, None, None, c.E, 1, T, F, None, None) == PNA_ERR_BAD_ARG
        return
    assert torch.equal(_bits(act), _bits(act0))
    G = c.bwd(emu, act)
    G0 = c.bwd(oracle, act0, ref=True)
    assert torch.equal(_bits(G), _bits(G0))


@pytest.mark.parametrize("L,F,T", [s for s in SHAPES if s[0] >= 2])
def test_without_edge_term_at_pitch_width_the_bits_of_the_edge_mlp(emu, L, F, T):
    c = Case(F, L, T, term=False, seed=4)
    M, act = c.fwd(emu)
    M1 = torch.full_like(M, float("nan"))
    act1 = torch.full_like(act, float("nan"))
    assert emu.pna_edge_mlp_fwd(_p(c.rowptr), _p(c.col), c.n, c.E, _p(c.A), _p(c.Bm), _p(c.b1), _p(c.W), _p(c.bW), L, T, F,
                                _p(M1), _p(act1), None) == PNA_OK
    assert torch.equal(_bits(M), _bits(M1)) and torch.equal(_bits(act), _bits(act1))
    G = c.bwd(emu, act)
    G1 = torch.full_like(G, float("nan"))
    assert emu.pna_edge_mlp_bwd(_p(c.dM), _p(act), _p(c.W), c.E, L, T, F, _p(G1), None) == PNA_OK
    assert torch.equal(_bits(G), _bits(G1))


@pytest.mark.parametrize("L,F,T", [(1, 14, 5), (1, 75, 1), (1, 130, 2), (2, 14, 5), (2, 64, 1), (3, 5, 2), (3, 16, 5),
                                   (4, 20, 2)])
def test_within_the_bar_of_float64(emu, L, F, T):
    c = Case(F, L, T, P=_padded(F), seed=1)
    M, act = c.fwd(emu)
    M64, G64, pre64 = c.float64()
    barM, barG = c.bars()
    err = (c.unpadded(M).double() - M64).abs()
    assert (err <= barM).all(), float((err / barM).max())
    if L == 1:
        return
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


def test_bad_descriptors_are_rejected(emu):
    c = Case(8, 3, 2, P=12, seed=3)
    M = torch.empty(c.E, 2 * 12)
    G = torch.empty(2, c.E, 16)
    act = torch.zeros(2, c.E, 16)

    def fwd(L=3, T=2, F=8, P=12, E=None, **null):
        ptrs = dict(rowptr=c.rowptr, col=c.col, a=c.A, b=c.Bm, b1=c.b1, C=c.C, W=c.W, bW=c.bW, M=M)
        for k in null:
            ptrs[k] = None
        return emu.pna_edge_msg_fwd(_p(ptrs["rowptr"]), _p(ptrs["col"]), c.n, c.E if E is None else E, _p(ptrs["a"]),
                                    _p(ptrs["b"]), _p(ptrs["b1"]), _p(ptrs["C"]), _p(ptrs["W"]), _p(ptrs["bW"]), L, T, F, P,
                                    _p(ptrs["M"]), None, None)

    def bwd(L=3, T=2, F=8, P=12, **null):
        ptrs = dict(dM=c.dM, act=act, W=c.W, G=G)
        for k in null:
            ptrs[k] = None
        return emu.pna_edge_msg_bwd(_p(ptrs["dM"]), P, _p(ptrs["act"]), _p(ptrs["W"]), c.E, L, T, F, _p(ptrs["G"]), None)

    assert fwd(L=0) == PNA_ERR_BAD_ARG and b"n_layers" in emu.emu_last_error()
    assert bwd(L=1) == PNA_ERR_BAD_ARG and b"n_layers" in emu.emu_last_error()
    for fn in (fwd, bwd):
        assert fn(L=0) == PNA_ERR_BAD_ARG
        assert fn(F=65, P=65) == PNA_ERR_UNSUPPORTED and b"width" in emu.emu_last_error()
        assert fn(P=7) == PNA_ERR_BAD_ARG and b"msg_pitch" in emu.emu_last_error()
        assert fn(F=0) == PNA_ERR_BAD_ARG
        assert fn(T=0) == PNA_ERR_BAD_ARG
    assert fwd(E=-1) == PNA_ERR_BAD_ARG
    for k in ("rowptr", "col", "a", "b", "b1", "W", "bW", "M"):
        assert fwd(**{k: 1}) == PNA_ERR_BAD_ARG, k
    for k in ("dM", "act", "W", "G"):
        assert bwd(**{k: 1}) == PNA_ERR_BAD_ARG, k
    # one layer: any width, and the hidden weights, biases and activations are not required
    assert fwd(L=1, F=8, P=8, W=1, bW=1) == PNA_OK
    assert fwd(L=1, F=10, P=12, T=1, W=1, bW=1, C=1) == PNA_OK
    assert fwd(E=0, rowptr=1, col=1, a=1) == PNA_OK        # nothing to do: no pointer is read
