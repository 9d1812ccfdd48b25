"""Set2Set / S2SReadout without a GPU: the float64 restatement of the kernels' algebra (tests/set2set_ref.py) against the
reference's own autograd (tests/golden/s2s_readout.pt, made by tools/gen_golden_set2set.py), parameter names and seeded
initialisation against the reference's, the C entry points' refusals (status codes, returned before anything touches a
device) and the saved-buffer size."""
import ctypes as C
import os
import sys

import pytest
import torch

import pna_b200
from pna_b200 import _lib, set2set as S

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import set2set_ref as R  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "s2s_readout.pt")
BAD_ARG, UNSUPPORTED = -1, -2
FAKE = 0x1000            # never dereferenced: every call below returns before it reads a buffer


def cases():
    return torch.load(GOLDEN)


def _module(case):
    torch.manual_seed(case["seed"])
    return pna_b200.S2SReadout(**case["ctor"]) if case["kind"] == "s2s" else pna_b200.Set2Set(**case["ctor"])


@pytest.mark.parametrize("name", sorted(torch.load(GOLDEN)))
def test_restatement_matches_the_reference_autograd(name):
    """Forward and the hand-written BPTT in float64 against the reference's fp32 autograd: within fp32 rounding."""
    case = cases()[name]
    out, grads = R.readout(case)
    assert set(case["grads"]) <= set(grads)
    scale = case["out"].abs().max().item()
    assert (out - case["out"].double()).abs().max().item() <= 1e-5 * scale
    for k, want in case["grads"].items():
        err = (grads[k] - want.double()).abs().max().item()
        assert err <= 2e-5 * want.abs().max().item() + 1e-12, (k, err)


@pytest.mark.parametrize("B,N,D,steps", [(3, 5, 4, None), (2, 1, 3, 4), (2, 6, 5, 1), (4, 3, 2, 7)])
def test_restatement_matches_float64_autograd(B, N, D, steps):
    """The BPTT, gate gradients and weight GEMMs against torch autograd of the reference loop, both in float64."""
    g = torch.Generator().manual_seed(B * 100 + N * 10 + D)
    torch.manual_seed(B + N + D)
    lstm = torch.nn.LSTM(2 * D, D, batch_first=True).double()
    x = torch.randn(B, N, D, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(B, 2 * D, generator=g, dtype=torch.float64)
    out = R.torch_loop(x, steps, lstm)
    params = [getattr(lstm, p) for p in R.PARAMS]
    want = torch.autograd.grad((out * w).sum(), [x] + params)
    mine, recs = R.forward(x.detach(), steps, *[p.detach() for p in params])
    got = R.backward(x.detach(), params[0].detach(), params[1].detach(), recs, w)
    assert torch.allclose(mine, out.detach(), rtol=0, atol=1e-12)
    for k, v in zip(("x",) + R.PARAMS, want):
        assert torch.allclose(got[k], v, rtol=0, atol=1e-11), k
    assert got["gates"].shape == (steps or N, B, 4 * D)


@pytest.mark.parametrize("name", sorted(torch.load(GOLDEN)))
def test_state_dict_and_seeded_init_match_the_reference(name):
    """Built after the reference's seed, the parameters are bit for bit the reference's; every key loads strictly."""
    case = cases()[name]
    mod = _module(case)
    sd = case["state_dict"]
    assert list(mod.state_dict()) == list(sd)
    for k, p in mod.named_parameters():
        assert torch.equal(p.detach(), sd[k]), k
    mod.load_state_dict(sd)
    assert isinstance(mod.set2set.lstm if case["kind"] == "s2s" else mod.lstm, torch.nn.LSTM)


def test_constructor_and_forward_refusals():
    with pytest.raises(ValueError):
        pna_b200.Set2Set(4, nhid=4)                                 # nhid <= nin, as the reference
    with pytest.raises(NotImplementedError):
        pna_b200.Set2Set(4, num_layers=2)
    s = pna_b200.Set2Set(4, nhid=10, activation="relu")             # accepted at construction, as the reference
    with pytest.raises(ValueError, match="nhid == 2"):
        s(torch.zeros(2, 3, 4))
    with pytest.raises(ValueError, match="CUDA"):
        pna_b200.Set2Set(4)(torch.zeros(2, 3, 4))                    # no CPU path
    with pytest.raises(ValueError):
        pna_b200.Set2Set(4)(torch.zeros(2, 3, 5))


def test_entry_points_return_status_codes_without_a_device():
    L = _lib.lib()
    for n in ("pna_set2set_saved_floats", "pna_set2set_fwd", "pna_set2set_bwd"):
        assert n in _lib.EXPORTED_SYMBOLS
    fwd = lambda x, B, N, D, T, out=FAKE: L.pna_set2set_fwd(x, B, N, D, T, FAKE, FAKE, FAKE, FAKE, out, None, None)  # noqa: E731
    bwd = lambda x, B, N, D, T, gg=FAKE: L.pna_set2set_bwd(x, B, N, D, T, FAKE, FAKE, FAKE, FAKE, None, gg, None)  # noqa: E731
    assert fwd(None, 4, 8, 16, 8) == BAD_ARG
    assert b"pna_set2set_fwd" in L.pna_last_error()
    assert fwd(FAKE, 4, 8, 16, 8, out=None) == BAD_ARG
    assert bwd(FAKE, 4, 8, 16, 8, gg=None) == BAD_ARG
    for B, N, D, T in ((0, 8, 16, 8), (4, 0, 16, 8), (4, 8, 0, 8), (4, 8, 16, 0), (-1, 8, 16, 8)):
        assert fwd(FAKE, B, N, D, T) == BAD_ARG
        assert bwd(FAKE, B, N, D, T) == BAD_ARG
    assert fwd(FAKE, 4, 8, 129, 8) == UNSUPPORTED                  # D > 128
    assert fwd(FAKE, 4, 129, 128, 8) == UNSUPPORTED                # N * D > 16384
    assert b"16384" in L.pna_last_error()
    assert bwd(FAKE, 4, 16385, 1, 8) == UNSUPPORTED
    assert fwd(FAKE, 1 << 31, 8, 16, 8) == UNSUPPORTED             # more graphs than a grid holds


def test_saved_floats():
    for B, N, D, T in ((128, 32, 16, 32), (3, 100, 66, 200), (1, 1, 1, 1), (300, 128, 128, 256)):
        assert S.saved_floats(B, N, D, T) == T * B * (7 * D + N)
    L = _lib.lib()
    n = C.c_int64(-5)
    assert L.pna_set2set_saved_floats(4, 8, 16, 8, None) == BAD_ARG
    assert L.pna_set2set_saved_floats(0, 8, 16, 8, C.byref(n)) == BAD_ARG and n.value == -5
    assert L.pna_set2set_saved_floats(4, 8, 256, 8, C.byref(n)) == UNSUPPORTED
    assert L.pna_set2set_saved_floats((1 << 31) - 1, 128, 128, (1 << 31) - 1, C.byref(n)) == UNSUPPORTED   # overflows int64


def test_header_documents_the_saved_layout():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pna_b200.h")).read()
    assert "q*_t (2D) | c_t (D) | i_t f_t g_t o_t" in src and "7D + n_nodes" in src
