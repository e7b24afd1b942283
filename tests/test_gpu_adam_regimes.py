"""gsb_adam_step element by element against the float64 reference (tests/adam_ref.py, itself torch.optim.Adam) across the
settings and values training meets: beta1 in {0, 0.3, 0.5, 0.9, 0.99} (both branches of the moment's lerp, and its boundary
1 - beta1 = 0.5), beta2 in {0, 0.99, 0.999}, eps in {1e-15, 1e-8}, steps 1, 2, 1000 and 30 000 (where the bias corrections
round to 1.0f), a group with lr = 0, raw parameters across a trained scene's range (log scale -12..3, logits to +-20,
quaternion norms 0.05..20, SH +-5), gradients of 1e-12..1e2 with exact-zero rows, and the real gradients of the scale and
edge scenes' frames, dense and selective; the scene a step leaves equals an upload of its records.

The step is checked in two halves, each per element with a bound derived from fp32 rounding (u = 2^-24, a factor of about 2
to spare).  A float64 comparison of the whole step is ill-conditioned: Adam divides the moment by the root of the second
moment, so at step 1 the update is lr sign(g) whatever |g|, and a chained gradient that fp32 rounds to 0 (d logit at
logit 20, where o (1 - o) is below ulp(1)) or that changes sign moves a parameter by a whole lr.  So
- the chain rule: with beta1 = beta2 = 0 the first moment after the step is exactly the kernel's chained fp32 gradient g32,
  which is compared with adam_ref.chain;
- Adam: the step with the settings under test is compared with adam_ref.adam_update fed g32."""
import numpy as np
import pytest

import adam_ref
import edge_scene
import scale_scene
from adam_ref import GROUPS
from test_gpu_adam import LR, _assert_coherent, _frame_grad, _start

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
N_ROWS = 4096
BETA1 = [0.0, 0.3, 0.5, 0.9, 0.99]
BETA2 = [0.0, 0.99, 0.999]
EPS = [1e-15, 1e-8]
STEPS = [1, 2, 1000, 30000]


def _torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def twin(gs):
    """A second context for the chain-rule captures, so they leave the stepped context's scene and frame alone."""
    c = gs.Context(0)
    yield c
    c.close()


def synthetic_state(seed=0):
    """(params, exp_avg, exp_avg_sq, grad_vertices) float32 numpy, N_ROWS rows across a trained scene's range; every 16th
    row has an exactly zero gradient.  The moments are as Adam leaves them, |m| <= sqrt(v), so a step moves a parameter
    by about lr at most and the log scales stay where expf is finite."""
    rng = np.random.default_rng(seed)
    n = N_ROWS
    p = np.zeros((n, 60))
    p[:, 0:3] = rng.uniform(-10, 10, (n, 3))
    p[:, 3] = 1.0
    p[:, 4:7] = rng.uniform(-12, 3, (n, 3))
    p[:, 7] = rng.choice([13.8, -13.8, 20.0, -20.0, 0.0], n) + np.where(rng.random(n) < 0.5, 0.0, rng.uniform(-2, 2, n))
    q = rng.standard_normal((n, 4))
    p[:, 8:12] = q / np.linalg.norm(q, axis=1, keepdims=True) * np.exp(rng.uniform(np.log(0.05), np.log(20), (n, 1)))
    p[:, 12:60] = rng.uniform(-5, 5, (n, 48))

    def magnitudes(shape):
        return rng.choice([-1, 1], shape) * 10.0 ** rng.uniform(-12, 2, shape)

    g = magnitudes((n, 60))
    g[::16] = 0.0
    m = magnitudes((n, 60)) * 1e-2
    v = m * m * 10.0 ** rng.uniform(0, 2, (n, 60))  # |m| <= sqrt(v), as Adam's moments keep it
    g[:, 3] = m[:, 3] = v[:, 3] = 0.0
    return tuple(np.ascontiguousarray(a, np.float32) for a in (p, m, v, g))


def chain32(gs, ctx, params, grad):
    """The kernel's chained fp32 gradient of `grad` at `params` (CUDA tensors): exp_avg after a beta1 = beta2 = 0 step."""
    torch = _torch()
    n = params.shape[0]
    ctx.upload(adam_ref.activate(params.cpu()).float().numpy())
    p, m, s = params.clone(), torch.zeros_like(params), torch.zeros_like(params)
    ctx.adam_step(p, m, s, grad, torch.empty_like(params), gs.adam_config([0.0] * 6, betas=(0.0, 0.0), step=1))
    torch.cuda.synchronize()
    assert m.shape[0] == n
    return m.double().cpu()


def check_chain(params, grad, g32):
    """g32 against adam_ref.chain per element: position and SH exact; d log s within 2^-21 relative (expf's 2 ulp and a
    product); d logit within |do| 2^-22 + 2^-21 relative (o (1 - o) in fp32 is good to ~ulp(1) absolute near saturation);
    dq within 2^-19 (|dq^_i| + sum_j |dq^_j|) / |q| + 2^-21 relative (the projection cancels)."""
    p, g = params.double().cpu(), grad.double().cpu()
    ref = adam_ref.chain(p, g)
    err = (g32 - ref).abs()
    for name in ("position", "sh_dc", "sh_rest"):
        assert bool((err[:, GROUPS[name]] == 0).all()), name
    assert bool((g32[:, 3] == 0).all())
    s = GROUPS["scale"]
    assert bool((err[:, s] <= 2.0 ** -21 * ref[:, s].abs()).all()), float((err[:, s] / ref[:, s].abs()).nan_to_num().max())
    o = GROUPS["opacity"]
    assert bool((err[:, o] <= 2.0 ** -22 * g[:, o].abs() + 2.0 ** -21 * ref[:, o].abs()).all())
    r = GROUPS["rotation"]
    norm = p[:, r].norm(dim=1, keepdim=True)
    bound = 2.0 ** -19 * (g[:, r].abs() + g[:, r].abs().sum(1, keepdim=True)) / norm + 2.0 ** -21 * ref[:, r].abs()
    assert bool((err[:, r] <= bound).all()), float((err[:, r] / bound).max())


def check_adam(cfg, before, after, g32, rows):
    """The stepped (params, exp_avg, exp_avg_sq) against adam_ref.adam_update fed g32, per element, on `rows` (bool);
    every other row and column 3 bit-identical to `before`.  Bounds: |dm| <= 4u (|m| + |g| + |m_old|) (g - m and the lerp
    rounded, w1 = 1 - beta1 rounded); |dv| <= 4u v + 2^-148 (three roundings of non-negative terms, the last also where v
    is subnormal, as it is for d logit ~ 1e-21 at logit 20); |dx| <= 2u |x| + (lr / bc1)
    (bound_m + 16u |m|) / denom (the moment's error, and denom, the quotient and the step size each a few u)."""
    torch = _torch()
    p0, m0, v0 = (t.double().cpu() for t in before)
    P, M, V = (t.double().cpu() for t in after)
    lr = list(cfg.lr)
    Pr, Mr, Vr = adam_ref.adam_update(p0, m0, v0, g32, lr, cfg.beta1, cfg.beta2, cfg.eps, cfg.bias_correction1,
                                      cfg.bias_correction2_sqrt, rows)
    worst = {}
    for k, (name, cols) in enumerate(GROUPS.items()):
        sel = (rows, cols)
        bm = 4 * U * (Mr[sel].abs() + g32[sel].abs() + m0[sel].abs())
        assert bool(((M[sel] - Mr[sel]).abs() <= bm).all()), ("exp_avg", name)
        assert bool(((V[sel] - Vr[sel]).abs() <= 4 * U * Vr[sel] + 2.0 ** -148).all()), ("exp_avg_sq", name)
        denom = Vr[sel].sqrt() / cfg.bias_correction2_sqrt + cfg.eps
        bx = 2 * U * Pr[sel].abs() + lr[k] / cfg.bias_correction1 * (bm + 16 * U * Mr[sel].abs()) / denom
        ex = (P[sel] - Pr[sel]).abs()
        assert bool((ex <= bx).all()), ("params", name, float((ex / bx).nan_to_num().max()))
        worst[name] = float((ex / bx).nan_to_num().max())
        if lr[k] == 0:
            assert bool((P[sel] == p0[sel]).all()), ("lr = 0 moved", name)
    for a, b in zip(after, before):
        a, b = a.cpu(), b.cpu()
        assert torch.equal(a[~rows].view(torch.int32), b[~rows].view(torch.int32))
        assert torch.equal(a[:, 3].view(torch.int32), b[:, 3].view(torch.int32))
    return worst


def check_vertices(params, vertices, rows):
    """The records written: activate(params) of the kernel's own parameters, per element: position and SH exact, scale
    within 2^-21 relative (expf), opacity 2^-21 relative (1 / (1 + expf(-x))), q / |q| 2^-21 relative, each also within
    2^-126 absolute (below the smallest normal float expf underflows, and 1 / (1 + expf(-x)) is 0 once expf(-x)
    overflows); a scale past the largest float is +inf.  With beta2 = 0, v = g^2 and m / sqrt(v) is unbounded, so a log
    scale can leave expf's range."""
    P, Vx = params.double().cpu()[rows], vertices.double().cpu()[rows]
    ref = adam_ref.activate(P)
    err = (Vx - ref).abs()
    for name in ("position", "sh_dc", "sh_rest"):
        assert bool((err[:, GROUPS[name]] == 0).all()), name
    assert bool((Vx[:, 3] == 1).all())
    big = ref[:, GROUPS["scale"]] > np.finfo(np.float32).max
    assert bool((Vx[:, GROUPS["scale"]][big] == np.inf).all())
    err[:, GROUPS["scale"]][big] = 0.0
    for name in ("scale", "opacity", "rotation"):
        c = GROUPS[name]
        assert bool((err[:, c] <= 2.0 ** -21 * ref[:, c].abs() + 2.0 ** -126).all()), name


def step_and_check(gs, ctx, twin, state, gv, cfg, rows):
    torch = _torch()
    p, m, s = (t.clone() for t in state)
    g32 = chain32(gs, twin, p, gv)
    check_chain(p, gv, g32)
    out = torch.empty_like(p)
    ctx.adam_step(p, m, s, gv, out, cfg)
    torch.cuda.synchronize()
    worst = check_adam(cfg, state, (p, m, s), g32, rows)
    check_vertices(p, out, rows)
    return (p, m, s, out), worst


@pytest.mark.parametrize("step", STEPS)
@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("beta2", BETA2)
@pytest.mark.parametrize("beta1", BETA1)
def test_settings_across_the_parameter_range(gs, twin, beta1, beta2, eps, step):
    torch = _torch()
    p, m, v, g = (torch.from_numpy(a).cuda() for a in synthetic_state())
    ctx = gs.Context(0)
    try:
        ctx.upload(adam_ref.activate(p.cpu()).float().numpy())
        cfg = gs.adam_config(LR, betas=(beta1, beta2), eps=eps, step=step)
        rows = torch.ones(N_ROWS, dtype=torch.bool)
        (p1, _, _, out), worst = step_and_check(gs, ctx, twin, (p, m, v), g, cfg, rows)
        torch.cuda.synchronize()
        fresh = gs.Context(0)
        try:  # the scene words equal an upload of the records
            fresh.upload(out.cpu().numpy())
            assert np.array_equal(ctx.download(gs.BUF_COV3D).view(np.uint32), fresh.download(gs.BUF_COV3D).view(np.uint32))
        finally:
            fresh.close()
    finally:
        ctx.close()
    if step == 30000:
        assert cfg.bias_correction1 == 1.0 and (beta2 == 0.0 or cfg.bias_correction2_sqrt == 1.0)
    print(f"beta1 {beta1} beta2 {beta2} eps {eps} step {step}: params error / bound per group {worst}")


def test_lr_zero_group_stays_bit_identical(gs, twin):
    torch = _torch()
    p, m, v, g = (torch.from_numpy(a).cuda() for a in synthetic_state(seed=1))
    ctx = gs.Context(0)
    try:
        ctx.upload(adam_ref.activate(p.cpu()).float().numpy())
        for k, name in enumerate(GROUPS):
            lr = list(LR)
            lr[k] = 0.0
            cfg = gs.adam_config(lr, step=2)
            (p1, m1, _, _), _ = step_and_check(gs, ctx, twin, (p, m, v), g, cfg, torch.ones(N_ROWS, dtype=torch.bool))
            c = GROUPS[name]
            assert torch.equal(p1[:, c].view(torch.int32), p[:, c].view(torch.int32)), name
            assert not torch.equal(m1[:, c], m[:, c])  # the moments still move
            others = [GROUPS[o] for o in GROUPS if o != name]
            assert all(not torch.equal(p1[:, o], p[:, o]) for o in others)
    finally:
        ctx.close()


def test_zero_gradient_rows_still_move(gs, twin):
    """Dense mode, torch's semantics: a row whose gradient is exactly 0 decays its moments and moves by the decayed
    moment wherever the reference's move exceeds 2^-21 of the parameter."""
    torch = _torch()
    p, m, v, g = (torch.from_numpy(a).cuda() for a in synthetic_state(seed=2))
    ctx = gs.Context(0)
    try:
        ctx.upload(adam_ref.activate(p.cpu()).float().numpy())
        cfg = gs.adam_config(LR, step=5)
        (p1, m1, v1, _), _ = step_and_check(gs, ctx, twin, (p, m, v), g, cfg, torch.ones(N_ROWS, dtype=torch.bool))
        zero = (g == 0).all(1)
        assert int(zero.sum()) == N_ROWS // 16
        cols = torch.cat([torch.arange(0, 3), torch.arange(4, 60)])
        z = zero.cpu()
        pr, _, _ = adam_ref.adam_update(p.cpu(), m.cpu(), v.cpu(), torch.zeros(N_ROWS, 60), list(cfg.lr), cfg.beta1, cfg.beta2,
                                        cfg.eps, cfg.bias_correction1, cfg.bias_correction2_sqrt, z)
        p0, p1, m0, m1, v0, v1 = (t.cpu()[z][:, cols] for t in (p, p1, m, m1, v, v1))
        moves = (pr[z][:, cols] - p0.double()).abs() > 2.0 ** -21 * p0.double().abs()
        assert float(moves.double().mean()) > 0.5
        assert bool((p1[moves] != p0[moves]).all())
        assert bool((m1.abs() < m0.abs()).all()) and bool((v1 < v0).all())
    finally:
        ctx.close()


REAL = [(scale_scene, "axis"), (scale_scene, "rotated_odd"), (edge_scene, "axis"), (edge_scene, "rotated_odd")]


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
@pytest.mark.parametrize("case", REAL, ids=[f"{m.__name__}-{c}" for m, c in REAL])
def test_real_frame_gradients(gs, twin, case, selective):
    """The gradient of a frame of the scale scene (huge, tiny and needle Gaussians) or the edge scene (duplicates,
    saturated colours, frame-sized Gaussians), at beta1 0.9 and 0.3 (both lerp branches); the stepped scene renders what
    an upload of its records renders at the scene's cameras."""
    torch = _torch()
    mod, cam = case
    vtx = mod.vertices()
    vtx = vtx[0] if isinstance(vtx, tuple) else vtx
    u = mod.camera(cam)
    ctx = gs.Context(0)
    try:
        v = torch.from_numpy(np.ascontiguousarray(vtx)).cuda()
        state = _start(gs, vtx, seed=3)
        for beta1, step in ((0.9, 3), (0.3, 1000)):
            ctx.upload(v)
            gv, surv = _frame_grad(ctx, v, u)
            assert 100 < int(surv.sum()) < v.shape[0]
            rows = surv.cpu() if selective else torch.ones(v.shape[0], dtype=torch.bool)
            cfg = gs.adam_config(LR, betas=(beta1, 0.999), step=step, selective=selective)
            (p1, _, _, out), worst = step_and_check(gs, ctx, twin, state, gv, cfg, rows)
            print(f"{mod.__name__} {cam} beta1 {beta1}: params error / bound per group {worst}")
        if not selective:
            v = out
        else:  # the rows the frame did not keep hold their uploaded records
            v = v.clone()
            v[surv] = out[surv]
        _assert_coherent(gs, ctx, v, [mod.camera(c) for c in mod.CAMERAS if c in ("axis", "rotated_odd")])
    finally:
        ctx.close()
