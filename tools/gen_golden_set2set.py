"""Generate tests/golden/s2s_readout.pt by RUNNING THE REFERENCE'S OWN ``models/layers.py`` (``Set2Set``, ``S2SReadout``) on
the CPU: inputs, constructor arguments, seeds, state_dicts, outputs and the reference autograd's gradients of
sum(out * w) with respect to x and every parameter.

    PYTHONPATH=. python tools/gen_golden_set2set.py      (needs the reference checkout; PNA_REFERENCE overrides its location)

``models/layers.py`` imports only torch, so no shim is needed.  The fixture stays well under 1 MB: at D = 66 the LSTM alone
has 70 k parameters, so the eval-mode case there stores the gradients of x and of the MLP, and the train-mode case those of
every parameter.  TEST INFRASTRUCTURE ONLY.
"""
import os
import sys

import torch

REF = os.environ.get("PNA_REFERENCE", "/root/reference")
sys.path.insert(0, REF)
from models.layers import S2SReadout, Set2Set  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "s2s_readout.pt")


def run(mod, x, train, keep_lstm_grads=True):
    mod.train(train)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        shape = mod(x).shape
    w = torch.randn(shape, generator=g)
    xg = x.clone().requires_grad_(True)
    mod.zero_grad()
    out = mod(xg)
    (out * w).sum().backward()
    grads = {"x": xg.grad.clone()}
    grads.update({k: p.grad.clone() for k, p in mod.named_parameters() if keep_lstm_grads or ".lstm." not in "." + k})
    return dict(out=out.detach(), w=w, grads=grads, train=train)


def s2s_cases(name, seed, B, N, D, hidden, cases):
    torch.manual_seed(seed)
    mod = S2SReadout(D, hidden, 3, fc_layers=3, final_activation="LeakyReLU")
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(B, N, D, generator=g)
    mod.train()
    with torch.no_grad():                                     # running statistics that differ from their initial values
        for _ in range(3):
            mod(torch.randn(B, N, D, generator=g))
    sd = {k: v.clone() for k, v in mod.state_dict().items()}
    common = dict(kind="s2s", seed=seed, ctor=dict(in_size=D, hidden_size=hidden, out_size=3, fc_layers=3,
                                                   final_activation="LeakyReLU"), x=x, steps=None, state_dict=sd,
                  final_activation="LeakyReLU")
    train = run(mod, x, True)
    mod.load_state_dict(sd)                                   # the eval case sees the same running statistics
    evl = run(mod, x, False, keep_lstm_grads=D <= 16)
    cases[f"{name}_train"] = {**common, **train}
    cases[f"{name}_eval"] = {**common, **evl}


def set2set_case(name, seed, B, N, D, steps, cases):
    torch.manual_seed(seed)
    mod = Set2Set(D, steps=steps)
    x = torch.randn(B, N, D, generator=torch.Generator().manual_seed(seed + 1))
    cases[name] = dict(kind="set2set", seed=seed, ctor=dict(nin=D, steps=steps), x=x, steps=steps,
                       state_dict={k: v.clone() for k, v in mod.state_dict().items()}, **run(mod, x, True))


def main():
    cases = {}
    s2s_cases("s2s16", 101, 6, 9, 16, 16, cases)
    s2s_cases("s2s66", 102, 4, 7, 66, 16, cases)
    set2set_case("set2set_steps1", 103, 3, 5, 8, 1, cases)
    set2set_case("set2set_steps2n", 104, 3, 5, 8, 10, cases)
    set2set_case("set2set_n1", 105, 4, 1, 8, None, cases)
    s2s_cases("s2s16_n1", 106, 5, 1, 16, 16, cases)
    torch.save(cases, OUT)
    print(f"{OUT}: {os.path.getsize(OUT) / 1024:.0f} KiB, {len(cases)} cases")


if __name__ == "__main__":
    main()
