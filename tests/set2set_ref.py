"""Float64 restatement of the Set2Set kernels (pna_b200/csrc/pna_set2set.cu) and the fp32 yardsticks they are judged by.

``forward`` / ``backward`` are the algebra the kernels implement, step for step: the LSTM cell in gate order i, f, g, o,
the max-subtracted softmax, the hand-written back-propagation through time with its pre-activation gate gradients, and
the three weight-gradient GEMMs over the ``T * B`` gate rows (``pna_b200/set2set.py``).  ``torch_loop`` is the reference's
loop in torch ops around an ``nn.LSTM`` (what the reference's ``Set2Set.forward`` runs), used in fp32 on the CPU as the
yardstick of fp32 rounding.  ``mlp`` is the MLP of ``S2SReadout`` in torch ops, for the readout's end-to-end checks.
TEST INFRASTRUCTURE ONLY."""
import torch

PARAMS = ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0")


def forward(x, steps, w_ih, w_hh, b_ih, b_hh):
    """q* after T = steps or N steps, and per step the record the kernel saves: (q*_t, c_t, i, f, g, o, alpha_t)."""
    B, N, D = x.shape
    qs, c = x.new_zeros(B, 2 * D), x.new_zeros(B, D)
    recs = []
    for _ in range(steps or N):
        G = qs @ w_ih.t() + qs[:, :D] @ w_hh.t() + b_ih + b_hh
        i, f = torch.sigmoid(G[:, :D]), torch.sigmoid(G[:, D:2 * D])
        g, o = torch.tanh(G[:, 2 * D:3 * D]), torch.sigmoid(G[:, 3 * D:])
        c = f * c + i * g
        q = o * torch.tanh(c)
        e = torch.einsum("bnd,bd->bn", x, q)
        a = torch.softmax(e, 1)
        qs = torch.cat([q, torch.einsum("bn,bnd->bd", a, x)], 1)
        recs.append((qs, c, i, f, g, o, a))
    return qs, recs


def backward(x, w_ih, w_hh, recs, grad_out):
    """Gradients of x and of the four LSTM parameters from grad_out [B, 2D], and the gate gradients [T, B, 4D]."""
    B, N, D = x.shape
    T = len(recs)
    dqs, dc, dx = grad_out.clone(), x.new_zeros(B, D), torch.zeros_like(x)
    dG = x.new_zeros(T, B, 4 * D)
    for t in reversed(range(T)):
        qs, c, i, f, g, o, a = recs[t]
        q, dr = qs[:, :D], dqs[:, D:]
        da = torch.einsum("bnd,bd->bn", x, dr)                      # attention: r = sum_i alpha_i x_i, e_i = x_i . q
        de = a * (da - (a * da).sum(1, keepdim=True))
        dx += a[..., None] * dr[:, None, :] + de[..., None] * q[:, None, :]
        dq = dqs[:, :D] + torch.einsum("bn,bnd->bd", de, x)
        cp = recs[t - 1][1] if t > 0 else torch.zeros_like(c)       # cell: q = o tanh(c), c = f c_prev + i g
        tc = torch.tanh(c)
        dc = dc + dq * o * (1 - tc * tc)
        dG[t] = torch.cat([dc * g * i * (1 - i), dc * cp * f * (1 - f), dc * i * (1 - g * g), dq * tc * o * (1 - o)], 1)
        dc = dc * f
        dqs = dG[t] @ w_ih                                          # recurrence: the input q*_{t-1} and the hidden q_{t-1}
        dqs[:, :D] += dG[t] @ w_hh
    G = dG.reshape(T * B, 4 * D)
    Qp = torch.stack([r[0] for r in recs[:-1]]).reshape((T - 1) * B, 2 * D) if T > 1 else x.new_zeros(0, 2 * D)
    db = G.sum(0)
    return {"x": dx, "weight_ih_l0": G[B:].t() @ Qp, "weight_hh_l0": G[B:].t() @ Qp[:, :D], "bias_ih_l0": db,
            "bias_hh_l0": db.clone(), "gates": dG}


def torch_loop(x, steps, lstm):
    """The reference's Set2Set loop in torch ops around the nn.LSTM `lstm` (any device, any dtype)."""
    B, N, D = x.shape
    hc = (x.new_zeros(1, B, D), x.new_zeros(1, B, D))
    qs = x.new_zeros(B, 1, 2 * D)
    for _ in range(steps or N):
        q, hc = lstm(qs, hc)
        a = torch.softmax(torch.matmul(x, q.transpose(1, 2)), dim=1)
        qs = torch.cat([q, (a * x).sum(1, keepdim=True)], -1)
    return qs.squeeze(1)


def mlp(h, sd, train, final_activation, prefix="mlp."):
    """S2SReadout's MLP from a state_dict: Linear -> activation -> batch norm (batch statistics in train mode, running ones
    in eval) on every layer but the last, whose activation is `final_activation` and which has no norm."""
    n = 0
    while f"{prefix}fully_connected.{n}.linear.weight" in sd:
        n += 1
    for k in range(n):
        p = f"{prefix}fully_connected.{k}."
        h = h @ sd[p + "linear.weight"].to(h.dtype).t() + sd[p + "linear.bias"].to(h.dtype)
        if k < n - 1:
            h = torch.relu(h)
            if train:
                mean, var = h.mean(0), h.var(0, unbiased=False)
            else:
                mean, var = sd[p + "b_norm.running_mean"].to(h.dtype), sd[p + "b_norm.running_var"].to(h.dtype)
            h = (h - mean) / torch.sqrt(var + 1e-5) * sd[p + "b_norm.weight"].to(h.dtype) + sd[p + "b_norm.bias"].to(h.dtype)
        elif final_activation.lower() == "leakyrelu":
            h = torch.nn.functional.leaky_relu(h, 0.01)
        elif final_activation.lower() == "relu":
            h = torch.relu(h)
    return h


def readout(case, dtype=torch.float64):
    """A golden case restated: its output and the gradients of sum(out * w) w.r.t. x and every parameter, in `dtype`."""
    sd = {k: v.to(dtype) if v.is_floating_point() else v for k, v in case["state_dict"].items()}
    pre = "set2set.lstm." if case["kind"] == "s2s" else "lstm."
    x = case["x"].to(dtype)
    w = [sd[pre + p] for p in PARAMS]
    qs, recs = forward(x, case["steps"], *w)
    grads = {}
    if case["kind"] == "s2s":
        h = qs.clone().requires_grad_(True)
        mlp_params = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k.startswith("mlp.") and "running" not in k
                      and "num_batches" not in k}
        out = mlp(h, {**sd, **mlp_params}, case["train"], case["final_activation"])
        go, *gp = torch.autograd.grad((out * case["w"].to(dtype)).sum(), [h] + list(mlp_params.values()))
        grads.update(dict(zip(mlp_params, gp)))
    else:
        out, go = qs, case["w"].to(dtype)
    g = backward(x, w[0], w[1], recs, go)
    grads["x"] = g["x"]
    grads.update({pre + p: g[p] for p in PARAMS})
    return out.detach(), grads
