"""The bf16-storage edge-message kernels (csrc/pna_edge_mlp.cu: k_bf16_msg_fwd, k_bf16_msg_fwd_affine, k_bf16_msg_bwd) executed
on the HOST, thread by thread (tests/emu), through pna_edge_msg_fwd_bf16 / pna_edge_msg_bwd_bf16, against the fp32 entry
points of the same emulated library on the widened operands, bit for bit:
  * messages and stored activations:  bf16 call == RN_bf16(fp32 call on A.float(), Bm.float(), C.float());
  * pre-activation gradients:         bf16 call on (dM, z_bf16) == fp32 call on (dM.float(), z_bf16.float());
  * pad columns exactly +0;
over L = 1..4, tower widths 4 to 64 (also 75 and 130 at L = 1), pitch = width and padded, with and without the edge term."""
import ctypes as C
import importlib.util
import os
import shutil

import pytest
import torch

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

HERE = os.path.dirname(os.path.abspath(__file__))
P_ = C.c_void_p


@pytest.fixture(scope="module")
def emu():
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    try:
        L = C.CDLL(be.build("pna_edge_mlp.cu"))
    except Exception as exc:            # no CUDA headers on this machine
        pytest.skip(f"emulation library did not build: {exc}")
    L.emu_last_error.restype = C.c_char_p
    fwd = [P_, P_, C.c_int64, C.c_int64, P_, P_, P_, P_, P_, P_, C.c_int32, C.c_int32, C.c_int32, C.c_int32, P_, P_, P_]
    bwd = [P_, C.c_int32, P_, P_, C.c_int64, C.c_int32, C.c_int32, C.c_int32, P_, P_]
    L.pna_edge_msg_fwd.argtypes = L.pna_edge_msg_fwd_bf16.argtypes = fwd
    L.pna_edge_msg_bwd.argtypes = L.pna_edge_msg_bwd_bf16.argtypes = bwd
    return L


def _p(t):
    return None if t is None else t.data_ptr()


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _padded(F):
    """A pitch above F: the bf16 aggregation's 16-byte width, or F + 3 where F already is a multiple of 8."""
    return (F + 7) // 8 * 8 if F % 8 else F + 3


class Case:
    """A destination-sorted CSR with empty rows and more than one CTA of slots; bf16 A / Bm / C / dM, fp32 b1 and weights."""

    def __init__(self, F, L, T, P, term, n=48, seed=0):
        g = torch.Generator().manual_seed(seed * 1000 + F * 31 + L * 7 + T)
        deg = torch.randint(0, 12, (n,), generator=g)
        deg[::7] = 0
        self.n, self.F, self.L, self.T, self.P = n, F, L, T, P
        self.rowptr = torch.cat([torch.zeros(1, dtype=torch.int64), deg.cumsum(0)]).to(torch.int32)
        self.E = int(self.rowptr[-1])
        self.col = torch.randint(0, n, (self.E,), generator=g, dtype=torch.int32)
        TF = T * F
        self.A = torch.randn(n, TF, generator=g).bfloat16()
        self.Bm = torch.randn(n, TF, generator=g).bfloat16()
        self.b1 = 0.3 * torch.randn(TF, generator=g)
        self.C = torch.randn(self.E, TF, generator=g).bfloat16() if term else None
        self.W = torch.randn(L - 1, T, F, F, generator=g) / max(F, 1) ** 0.5
        self.bW = 0.3 * torch.randn(L - 1, T, F, generator=g)
        self.dM = torch.randn(self.E, T * P, generator=g).bfloat16()

    def fwd(self, lib, dt):
        up = (lambda t: t) if dt == torch.bfloat16 else (lambda t: None if t is None else t.float())
        M = torch.full((self.E, self.T * self.P), float("nan"), dtype=dt)
        act = torch.full((max(self.L - 1, 0), self.E, self.T * self.F), float("nan"), dtype=dt)
        entry = lib.pna_edge_msg_fwd_bf16 if dt == torch.bfloat16 else lib.pna_edge_msg_fwd
        A, Bm, Cs = up(self.A), up(self.Bm), up(self.C)
        rc = entry(_p(self.rowptr), _p(self.col), self.n, self.E, _p(A), _p(Bm), _p(self.b1), _p(Cs), _p(self.W), _p(self.bW),
                   self.L, self.T, self.F, self.P, _p(M), _p(act) if self.L > 1 else None, None)
        assert rc == 0, lib.emu_last_error()
        return M, act

    def bwd(self, lib, dM, act):
        G = torch.full((self.L - 1, self.E, self.T * self.F), float("nan"))
        entry = lib.pna_edge_msg_bwd_bf16 if act.dtype == torch.bfloat16 else lib.pna_edge_msg_bwd
        assert entry(_p(dM), self.P, _p(act), _p(self.W), self.E, self.L, self.T, self.F, _p(G), None) == 0, lib.emu_last_error()
        return G


SHAPES = ([(1, F, T) for F in (4, 5, 14, 16, 20, 64, 75, 130) for T in (1, 3)] +
          [(L, F, T) for L in (2, 3, 4) for F in (4, 5, 14, 16, 20, 64) for T in (1, 3)])


@pytest.mark.parametrize("term", [True, False])
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("L,F,T", SHAPES)
def test_bf16_storage_is_the_fp32_kernel_rounded_once(emu, L, F, T, padded, term):
    c = Case(F, L, T, _padded(F) if padded else F, term)
    assert c.E > 128 and (c.rowptr[1:] == c.rowptr[:-1]).any()
    M16, act16 = c.fwd(emu, torch.bfloat16)
    M32, act32 = c.fwd(emu, torch.float32)
    assert torch.equal(_bits(M16), _bits(M32.bfloat16()))
    pads = M16.view(c.E, T, c.P)[:, :, F:]
    assert torch.equal(_bits(pads), torch.zeros_like(_bits(pads)))          # exact +0, every pad column
    if L == 1:
        assert emu.pna_edge_msg_bwd_bf16(_p(c.dM), c.P, None, None, c.E, 1, T, F, None, None) == -1
        return
    assert torch.equal(_bits(act16), _bits(act32.bfloat16()))
    G16 = c.bwd(emu, c.dM, act16)
    G32 = c.bwd(emu, c.dM.float(), act16.float())
    assert torch.equal(_bits(G16), _bits(G32))
    assert (G16 == 0).any() and (G16 != 0).any()                            # the ReLU mask is exercised


def test_dense_layer_entry_is_the_edge_mlp_arithmetic(emu):
    """No edge term at pitch = width: the bf16 entry rounds what pna_edge_mlp_fwd computes (the dense layer under bf16
    autocast)."""
    c = Case(16, 3, 2, 16, term=False, seed=5)
    M16, act16 = c.fwd(emu, torch.bfloat16)
    emu.pna_edge_mlp_fwd.argtypes = [P_, P_, C.c_int64, C.c_int64, P_, P_, P_, P_, P_, C.c_int32, C.c_int32, C.c_int32, P_, P_, P_]
    M = torch.full((c.E, 32), float("nan"))
    act = torch.full((2, c.E, 32), float("nan"))
    A, Bm = c.A.float(), c.Bm.float()
    assert emu.pna_edge_mlp_fwd(_p(c.rowptr), _p(c.col), c.n, c.E, _p(A), _p(Bm), _p(c.b1), _p(c.W),
                                _p(c.bW), 3, 2, 16, _p(M), _p(act), None) == 0
    assert torch.equal(_bits(M16), _bits(M.bfloat16())) and torch.equal(_bits(act16), _bits(act.bfloat16()))
