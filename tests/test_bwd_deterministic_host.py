"""Host-side choices of the deterministic backward: which mode torch's switch selects, and the feature slabs that bound its
per-slot scratch."""
import pytest
import torch

from pna_b200 import _lib, aggregate as agg


@pytest.fixture
def restore_flag():
    yield
    torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("env", [None, "atomic", "coef"])
def test_torch_switch_selects_the_deterministic_backward_over_the_environment(monkeypatch, restore_flag, env):
    if env is None:
        monkeypatch.delenv("PNA_B200_BWD", raising=False)
    else:
        monkeypatch.setenv("PNA_B200_BWD", env)
    assert agg.backward_mode() == (env or "atomic")
    torch.use_deterministic_algorithms(True)
    assert agg.backward_mode() == "deterministic"
    torch.use_deterministic_algorithms(True, warn_only=True)
    assert agg.backward_mode() == "deterministic"
    torch.use_deterministic_algorithms(False)
    assert agg.backward_mode() == (env or "atomic")


def test_slab_width_is_the_full_row_unless_the_scratch_or_the_forward_bounds_it(monkeypatch):
    max_f = _lib.query(_lib.QUERY_MAX_FEATURES)
    assert agg.DETERMINISTIC_SCRATCH_BYTES == 1 << 30
    assert agg.deterministic_slab_width(1_000_000, 256, 4) == 256                # 1 GB: fits
    assert agg.deterministic_slab_width(0, 300, 4) == 300
    w = agg.deterministic_slab_width(10_000_000, 256, 4)                        # 10 GB: slabs of <= 1 GiB
    assert w % 4 == 0 and 10_000_000 * w * 4 <= 1 << 30 and 10_000_000 * (w + 4) * 4 > 1 << 30
    assert agg.deterministic_slab_width(10_000_000, 256, 8) % 8 == 0
    assert agg.deterministic_slab_width(100, max_f + 100, 4) == max_f           # the forward kernel's limit
    monkeypatch.setattr(agg, "DETERMINISTIC_SCRATCH_BYTES", 1000 * 4 * 10)
    assert agg.deterministic_slab_width(1000, 64, 4) == 8
    assert agg.deterministic_slab_width(1000, 64, 8) == 8
    assert agg.deterministic_slab_width(10**9, 64, 4) == 4                      # never below one aligned chunk


def test_deterministic_kernel_instances_have_no_atomics():
    """cuobjdump of the built library: the kernels pna_aggregate_bwd_slots launches (the per-slot instances of k_bwd_*, and
    k_bwd_hub_bias) contain no ATOM / RED instruction; the atomic instances still do."""
    import os
    import re
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump, cu++filt and the built library")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if "k_bwd_" in m.group(1):
            kernels[m.group(1)] = re.findall(r"\b(?:ATOM|ATOMG|RED|REDG)\b", m.group(2))
    names = subprocess.run(["cu++filt"], input="\n".join(kernels), capture_output=True, text=True, check=True).stdout.split("\n")
    demangled = dict(zip(kernels, names))
    slots = [k for k, n in demangled.items() if "(bool)1>" in n or "k_bwd_hub_bias" in n]
    atomic = [k for k, n in demangled.items() if "(bool)0>" in n and ("k_bwd_rows" in n or "k_bwd_hub_scatter" in n)]
    # 4 (element type, vector width) pairs x 6 lane-group widths x 4 kernels, and k_bwd_hub_bias per vector width x 6
    assert len(slots) == 4 * 6 * 4 + 3 * 6
    for k in slots:
        assert not kernels[k], f"{demangled[k]}: {kernels[k][:4]}"
    assert atomic and all(kernels[k] for k in atomic)
