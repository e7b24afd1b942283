"""tests/adam_ref.py against torch on the CPU: its chain rule equals autograd through exp, sigmoid and q / |q|, its update is
torch.optim.Adam's bit for bit over 20 steps, and SceneAdam's densify bookkeeping (adam_state_after_densify) gathers, zeroes
and re-derives the right rows."""
import math

import numpy as np
import torch

import adam_ref
from adam_ref import GROUPS

LR = [1.6e-4, 5e-3, 5e-2, 1e-3, 2.5e-3, 1.25e-4]


def _params(n=37, seed=0):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn((n, 60), generator=g, dtype=torch.float64)
    p[:, 4:7] = p[:, 4:7] * 0.5 - 3.0
    p[:, 8:12] += torch.tensor([2.0, 0, 0, 0], dtype=torch.float64)
    return p, g


def test_chain_rule_equals_autograd():
    p, g = _params()
    gv = torch.randn((p.shape[0], 60), generator=g, dtype=torch.float64)
    x = p.clone().requires_grad_()
    (adam_ref.activate(x) * gv).sum().backward()
    got = adam_ref.chain(p, gv)
    want = x.grad.clone()
    assert want[:, 3].abs().max() == 0 and got[:, 3].abs().max() == 0
    for name, cols in GROUPS.items():
        err = float((got[:, cols] - want[:, cols]).abs().max() / want[:, cols].abs().max())
        assert err <= 1e-12, (name, err)


def test_update_equals_torch_adam_bitwise():
    p, g = _params()
    betas, eps = (0.9, 0.999), 1e-15
    groups = {name: p[:, cols].clone().contiguous().requires_grad_() for name, cols in GROUPS.items()}
    opt = torch.optim.Adam([{"params": [t], "lr": LR[k]} for k, t in enumerate(groups.values())], betas=betas, eps=eps,
                           foreach=False)
    P, M, V = p.clone(), torch.zeros_like(p), torch.zeros_like(p)
    for t in range(1, 21):
        grad = torch.randn((p.shape[0], 60), generator=g, dtype=torch.float64)
        for name, cols in GROUPS.items():
            groups[name].grad = grad[:, cols].contiguous()
        opt.step()
        P, M, V = adam_ref.adam_update(P, M, V, grad, LR, betas[0], betas[1], eps, 1 - betas[0] ** t, (1 - betas[1] ** t) ** 0.5)
        for name, cols in GROUPS.items():
            st = opt.state[groups[name]]
            assert torch.equal(P[:, cols], groups[name].detach()), (t, name)
            assert torch.equal(M[:, cols], st["exp_avg"]) and torch.equal(V[:, cols], st["exp_avg_sq"]), (t, name)
    assert torch.equal(P[:, 3], p[:, 3]) and not M[:, 3].any()


def test_update_leaves_other_rows():
    p, g = _params()
    grad = torch.randn(p.shape, generator=g, dtype=torch.float64)
    rows = torch.arange(p.shape[0]) % 3 == 0
    P, M, V = adam_ref.adam_update(p, torch.zeros_like(p), torch.zeros_like(p), grad, LR, 0.9, 0.999, 1e-15, 0.1, 0.001 ** 0.5, rows)
    assert torch.equal(P[~rows], p[~rows]) and not M[~rows].any() and not V[~rows].any()
    assert (P[rows][:, 0:3] != p[rows][:, 0:3]).all()


def test_densify_bookkeeping(gs):
    """A hand-built table of 4 rows: row 1 is cloned, row 2 split into two children, row 3 pruned."""
    vertices = torch.zeros((4, 60))
    vertices[:, 4:7] = torch.tensor([[0.01, 0.01, 0.01], [0.02, 0.01, 0.01], [0.5, 0.2, 0.1], [0.03, 0.02, 0.02]])
    vertices[:, 7] = torch.tensor([0.5, 0.6, 0.7, 0.8])
    vertices[:, 8] = 1.0
    vertices[:, 0] = torch.arange(4.0)
    params = gs.raw_parameters(vertices)
    m = torch.arange(4.0)[:, None].expand(4, 60) + 1.0
    v = m * 10.0
    # densify_and_prune's output for clone = {1}, split = {2}, prune = {3}: kept 0, 1; clone of 1; two children of 2
    source = torch.tensor([0, 1, 1, 2, 2])
    new = vertices[source].clone()
    new[3:, 4:7] = vertices[2, 4:7] / 1.6
    new[3, 0:3] += torch.tensor([0.1, -0.2, 0.3])
    new[4, 0:3] -= torch.tensor([0.05, 0.0, 0.1])
    P, M, V = gs.adam_state_after_densify(params, m, v, vertices, new, source)
    assert torch.equal(P[:3], params[source[:3]]) and torch.equal(M[:3], m[source[:3]]) and torch.equal(V[:3], v[source[:3]])
    assert not M[3:].any() and not V[3:].any()
    assert torch.equal(P[3:, 0:3], new[3:, 0:3])
    assert torch.equal(P[3:, 4:7], torch.log(vertices[2, 4:7] / 1.6).expand(2, 3))
    assert torch.equal(P[3:, 7:], params[2, 7:].expand(2, 53))
    assert np.allclose(P[3:, 4:7].numpy(), np.log(vertices[2, 4:7].numpy() / 1.6))
    # s / 1.6 != s, the test a child is recognised by, from the smallest normal scale to the largest finite one
    for s in [math.ldexp(1.0, -126), 1e-3, 1.0, 3.0e38]:
        t = torch.tensor(s, dtype=torch.float32)
        assert bool(t > 0) and bool(t / 1.6 != t)
