"""gsb_mcmc_noise / gsb_mcmc_relocate / SceneAdam's 3DGS-MCMC loop (DESIGN.md section 16): the noise against the numpy
Philox restatement and the float64 Box-Muller, gated rows untouched, reproducible words, a KS test of 3e6 normals; the
relocation against the float64 reference word by word, copies, zero moments, untouched rows and every precondition; the
resident scene after either entry renders what an upload of its records renders; and the training loop under a budget.
Scenes: c1's records (10 000), an odd-sized set (10 007) and the full-size garden stand-in (5.8 M)."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

import mcmc_ref
import scenes
from backward_util import expect, grad_image, render
from test_gpu_adam import SIX, _assert_coherent

pytestmark = pytest.mark.gpu

NOISE, RELOCATE = "gsb_mcmc_noise", "gsb_mcmc_relocate"
SEED, STEP, SCALE = 0x5EED_0000_1234_ABCD, 7, 80.0


def _torch():
    import torch

    return torch


@pytest.fixture
def mctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _records(name):
    if name == "c1":
        return scenes.c1()[1]
    if name == "odd":
        return scenes.c1(n=10_007, seed=9)[1]
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench
    import gs_b200

    return bench.make_scene(gs_b200, bench.WORKLOADS["garden-standin"])


def _garden_camera(gs):
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    return bench.cameras(gs, bench.WORKLOADS["garden-standin"])[0]


def _state(gs, vtx, seed=0):
    """(vertices, params, exp_avg, exp_avg_sq) float32 CUDA tensors: the records, their raw parameters and seeded moments."""
    torch = _torch()
    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    return v, gs.raw_parameters(v), torch.randn(v.shape, generator=g, device="cuda"), torch.rand(v.shape, generator=g, device="cuda")


def _bits(t):
    return t.contiguous().view(_torch().int32)


# ---------------------------------------------------------------- noise
@pytest.mark.parametrize("scene", ["c1", "odd", "garden"])
def test_noise_matches_reference(gs, mctx, scene):
    torch = _torch()
    v, p, _, _ = _state(gs, _records(scene))
    v[::97, 7] = 0.95  # gated rows (o >= 0.9: the gate is exactly 0)
    v[1::5, 7] = 0.02  # rows the gate lets move (0.18)
    mctx.upload(v)
    cov = mctx.download(gs.BUF_COV3D)
    v0, p0 = v.clone(), p.clone()
    mctx.mcmc_noise(p, v, SCALE, SEED, STEP)
    torch.cuda.synchronize()
    opacity = v0[:, 7].cpu().numpy()
    want, bound, _ = mcmc_ref.noise_reference(p0.cpu().numpy(), cov, opacity, SCALE, SEED, STEP)
    got = p[:, 0:3].double().cpu().numpy()
    err = np.abs(got - want)
    print(f"{scene}: n {v.shape[0]}, worst |p - p_ref| / bound {float((err / np.maximum(bound, 1e-300)).max()):.3f}")
    assert bool((err <= bound).all())
    gated = v0[:, 7] >= 0.9
    assert int(gated.sum()) > 0
    assert torch.equal(_bits(p[gated]), _bits(p0[gated])) and torch.equal(_bits(v[gated]), _bits(v0[gated]))
    low = v0[:, 7] == 0.02
    assert float((p[low, 0:3] != p0[low, 0:3]).any(1).float().mean()) > 0.99
    # params and records hold the same positions (the scene's: test_scene_after_entry_equals_upload_and_frames); nothing
    # else changes, Sigma included
    assert torch.equal(_bits(p[:, 0:3]), _bits(v[:, 0:3]))
    assert torch.equal(_bits(p[:, 3:]), _bits(p0[:, 3:])) and torch.equal(_bits(v[:, 3:]), _bits(v0[:, 3:]))
    assert np.array_equal(mctx.download(gs.BUF_COV3D).view(np.uint32), cov.view(np.uint32))
    if scene == "garden":  # the resident positions render as an upload of the records does
        _assert_coherent(gs, mctx, v, [_garden_camera(gs)])


def _identity_scene(gs, ctx, n):
    """n records at the origin with scale 1, identity rotation and opacity 0.005: Sigma = I and the gate is 1/2 exactly, so
    with scale 2 the noise moves each row by exactly (eps0, eps1, eps2)."""
    torch = _torch()
    v = torch.zeros((n, 60), dtype=torch.float32, device="cuda")
    v[:, 3] = 1.0
    v[:, 4:7] = 1.0
    v[:, 7] = 0.005
    v[:, 8] = 1.0
    ctx.upload(v)
    return v


def _eps(ctx, v, seed, step, stream=None):
    torch = _torch()
    p = torch.zeros_like(v)
    ctx.mcmc_noise(p, v, 2.0, seed, step, stream=stream)
    torch.cuda.synchronize()
    return p[:, 0:3].clone()


def test_noise_normals_words_and_statistics(gs, mctx):
    """On the Sigma = I scene the positions are the normals themselves: within 1e-6 (1 + |eps|) of the float64 Box-Muller
    of the restated Philox words (a word that differs in any of the bits (float)x keeps moves eps far past that), identical
    over calls, a side stream and a fresh context, different for another step or seed; 3e6 normals pass a KS test against
    N(0, 1) and their correlations across components, rows and steps are below 5e-3."""
    torch = _torch()
    from scipy.stats import kstest

    n = 1_000_000
    v = _identity_scene(gs, mctx, n)
    eps = _eps(mctx, v, SEED, STEP)
    want = mcmc_ref.box_muller(mcmc_ref.uniforms(mcmc_ref.noise_words(np.arange(n), SEED, STEP)))
    e = eps.double().cpu().numpy()
    err = np.abs(e - want) / (1 + np.abs(want))
    print(f"eps vs float64 Box-Muller: worst {float(err.max()):.2e} (1 + |eps|)")
    assert float(err.max()) <= 1e-6
    assert torch.equal(_bits(_eps(mctx, v, SEED, STEP)), _bits(eps))
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        on_side = _eps(mctx, v, SEED, STEP, stream=side)
    assert torch.equal(_bits(on_side), _bits(eps))
    fresh = gs.Context(0)
    try:
        vf = _identity_scene(gs, fresh, n)
        assert torch.equal(_bits(_eps(fresh, vf, SEED, STEP)), _bits(eps))
    finally:
        fresh.close()
    nxt = _eps(mctx, v, SEED, STEP + 1).double().cpu().numpy()
    other = _eps(mctx, v, SEED + 1, STEP).double().cpu().numpy()
    assert float(np.mean(nxt == e)) < 1e-4 and float(np.mean(other == e)) < 1e-4
    ks = kstest(e.reshape(-1), "norm")
    corr = {"01": np.corrcoef(e[:, 0], e[:, 1])[0, 1], "02": np.corrcoef(e[:, 0], e[:, 2])[0, 1],
            "12": np.corrcoef(e[:, 1], e[:, 2])[0, 1], "rows": np.corrcoef(e[:-1].reshape(-1), e[1:].reshape(-1))[0, 1],
            "steps": np.corrcoef(e.reshape(-1), nxt.reshape(-1))[0, 1], "seeds": np.corrcoef(e.reshape(-1), other.reshape(-1))[0, 1]}
    print(f"KS D {ks.statistic:.2e} p {ks.pvalue:.3f}; mean {e.mean():.2e} var {e.var():.5f}; correlations {corr}")
    assert ks.pvalue > 1e-3
    assert all(abs(c) < 5e-3 for c in corr.values()), corr


# ---------------------------------------------------------------- relocation
def _expected_sources(v0, counts, min_opacity):
    """Record values (opacity, 3 scales) of every source row, from the fp64 rule (tests/mcmc_ref.py) per source."""
    rows = sorted(counts)
    out = np.empty((len(rows), 4))
    vv = v0[rows].double().cpu().numpy()
    mo = float(np.float32(min_opacity))
    for i, s in enumerate(rows):
        x, coeff = mcmc_ref.relocation_coeff(vv[i, 7], counts[s] + 1)
        out[i, 0] = min(max(x, mo), 1.0 - 2.0 ** -23)
        out[i, 1:] = vv[i, 4:7] * coeff
    return rows, out


def _one_rounding(got, want):
    """|got - want| <= one fp32 spacing at want (got is fp32, want the fp64 value it rounds)."""
    w32 = np.abs(want).astype(np.float32)
    return np.abs(got.astype(np.float64) - want) <= np.spacing(w32).astype(np.float64)


def _check_relocation(gs, ctx, before, after, cov0, dst, src, min_opacity, sample=None):
    torch = _torch()
    p0, m0, s0, v0 = before
    p, m, s, v = after
    counts = {}
    for j in src.tolist():
        counts[j] = counts.get(j, 0) + 1
    if sample is not None:  # the full-size scene: the rule on a sample of the sources, everything else on all rows
        keys = sorted(counts)
        pick = np.random.default_rng(0).choice(len(keys), min(sample, len(keys)), replace=False)
        counts_checked = {keys[i]: counts[keys[i]] for i in pick}
    else:
        counts_checked = counts
    rows, want = _expected_sources(v0, counts_checked, min_opacity)
    got = v[rows][:, 4:8].double().cpu().numpy()
    assert bool(_one_rounding(got[:, 3], want[:, 0]).all())
    assert bool(_one_rounding(got[:, 0:3], want[:, 1:]).all())
    # raw parameters: within one rounding of fp64 log / logit of the fp32 record values the entry wrote
    rec = v[rows][:, 4:8].double().cpu().numpy()
    want_p = np.concatenate([np.log(rec[:, 0:3]), np.log(rec[:, 3:4] / (1 - rec[:, 3:4]))], 1)
    assert bool(_one_rounding(p[rows][:, 4:8].double().cpu().numpy(), want_p).all())
    srcs = torch.tensor(sorted(counts), dtype=torch.int64, device="cuda")
    # every other column of a source is untouched
    for a, b in ((p, p0), (v, v0)):
        assert torch.equal(_bits(a[srcs][:, :4]), _bits(b[srcs][:, :4])) and torch.equal(_bits(a[srcs][:, 8:]), _bits(b[srcs][:, 8:]))
    # copies and zero moments
    d, sr = dst.long(), src.long()
    for a in (p, v):
        assert torch.equal(_bits(a[d]), _bits(a[sr]))
    touched = torch.zeros(v.shape[0], dtype=torch.bool, device="cuda")
    touched[d] = True
    touched[srcs] = True
    for a in (m, s):
        assert bool((a[touched] == 0).all()) and not bool(torch.signbit(a[touched]).any())
    rest = ~touched
    for a, b in zip(after, before):
        assert torch.equal(_bits(a[rest]), _bits(b[rest]))
    cov1 = ctx.download(gs.BUF_COV3D).reshape(-1, 6)
    rest_np = rest.cpu().numpy()
    assert np.array_equal(cov1[rest_np].view(np.uint32), cov0[rest_np].view(np.uint32))
    assert np.array_equal(cov1[d.cpu().numpy()].view(np.uint32), cov1[sr.cpu().numpy()].view(np.uint32))
    return len(counts)


def _dead_and_sources(gs, v, frac, generator, heavy=None):
    """dst = a `frac` of the rows made dead (opacity 0.004), src = live rows drawn by opacity; `heavy` (row, times) forces a
    source to appear that many times."""
    torch = _torch()
    n = v.shape[0]
    dead = torch.zeros(n, dtype=torch.bool)
    dead[torch.randperm(n, generator=generator)[: int(frac * n)]] = True
    dead = dead.cuda()
    v[dead, 7] = 0.004
    w = torch.where(dead, torch.zeros_like(v[:, 7]), v[:, 7])
    dst = torch.nonzero(dead)[:, 0].to(torch.int32)
    src = gs.mcmc_sample(w, dst.shape[0], generator).to(torch.int32)
    if heavy is not None:
        row, times = heavy
        src[:times] = int(torch.nonzero(~dead)[row, 0])
    return dst, src


@pytest.mark.parametrize("scene", ["c1", "odd", "garden"])
def test_relocate_matches_reference(gs, mctx, scene):
    torch = _torch()
    v, p, m, s = _state(gs, _records(scene))
    v[::53, 7] = 1.0  # x = 1 is clamped to 1 - 2^-23
    g = torch.Generator().manual_seed(1)
    dst, src = _dead_and_sources(gs, v, 0.05, g, heavy=(3, 60))  # one source with r = 61 > 51
    mctx.upload(v)
    cov0 = mctx.download(gs.BUF_COV3D).reshape(-1, 6)
    before = [t.clone() for t in (p, m, s, v)]
    mctx.mcmc_relocate(p, m, s, v, dst, src, 0.005)
    torch.cuda.synchronize()
    sources = _check_relocation(gs, mctx, before, (p, m, s, v), cov0, dst, src, 0.005, sample=4000 if scene == "garden" else None)
    if scene == "c1":  # the whole float64 reference (tests/mcmc_ref.py) as well
        ref = mcmc_ref.relocate_reference(*before, dst.cpu(), src.cpu(), 0.005)
        for got, want in zip((p, m, s, v), ref):
            assert bool(_one_rounding(got.double().cpu().numpy(), want.numpy()).all())
    print(f"{scene}: {dst.shape[0]} rows relocated onto {sources} sources")
    _assert_coherent(gs, mctx, v, SIX if scene != "garden" else [_garden_camera(gs)])


def test_relocate_preconditions_and_errors(gs, mctx):
    torch = _torch()
    v, p, m, s = _state(gs, scenes.c1()[1])
    n = v.shape[0]
    i32 = dict(dtype=torch.int32, device="cuda")
    dst, src = torch.tensor([5, 6, 7], **i32), torch.tensor([1, 1, 2], **i32)

    def raw(c, d=dst, sr=src, k=None, mo=0.005, arrays=None, shift=0):
        a = arrays or (p, m, s, v)
        ptrs = [None if t is None else t.data_ptr() + shift for t in a]
        kk = (3 if d is None else d.shape[0]) if k is None else k
        return lambda: c._ck(gs.lib.gsb_mcmc_relocate(c.h, *ptrs, None if d is None else d.data_ptr(),
                                                      None if sr is None else sr.data_ptr(), kk, mo, None))

    assert gs.lib.gsb_mcmc_relocate(None, p.data_ptr(), m.data_ptr(), s.data_ptr(), v.data_ptr(), dst.data_ptr(), src.data_ptr(),
                                    3, 0.005, None) == gs.ERR_INVALID
    expect(gs, mctx, gs.ERR_NO_SCENE, raw(mctx), RELOCATE)
    mctx.upload(v)
    before = [t.clone() for t in (p, m, s, v)]
    cov0 = mctx.download(gs.BUF_COV3D)
    host_side = [raw(mctx, arrays=(p, None, s, v)), raw(mctx, shift=4), raw(mctx, d=None), raw(mctx, k=n), raw(mctx, mo=1.0),
                 raw(mctx, mo=-0.1), raw(mctx, mo=float("nan"))]
    device_side = [  # index >= n in src and in dst, a repeated destination, a destination that is also a source
        raw(mctx, sr=torch.tensor([1, n, 2], **i32)), raw(mctx, d=torch.tensor([5, 6, n + 3], **i32)),
        raw(mctx, d=torch.tensor([5, 6, 5], **i32)), raw(mctx, d=torch.tensor([5, 1, 7], **i32)),
        raw(mctx, sr=torch.tensor([1, 7, 2], **i32)), raw(mctx, sr=torch.tensor([1, 2, -1], **i32))]
    for fn in host_side + device_side:
        expect(gs, mctx, gs.ERR_INVALID, fn, RELOCATE)
        torch.cuda.synchronize()
        for a, b in zip((p, m, s, v), before):
            assert torch.equal(_bits(a), _bits(b))
        assert np.array_equal(mctx.download(gs.BUF_COV3D).view(np.uint32), cov0.view(np.uint32))
    raw(mctx, d=None, sr=None, k=0)()  # k = 0: nothing to do, NULL index arrays allowed
    mctx.mcmc_relocate(p, m, s, v, dst[:0], src[:0])
    for a, b in zip((p, m, s, v), before):
        assert torch.equal(_bits(a), _bits(b))
    with pytest.raises(ValueError):
        mctx.mcmc_relocate(p, m, s, v, dst.long(), src)
    with pytest.raises(ValueError):
        mctx.mcmc_relocate(p, m, s, v, dst, src[:2])
    with pytest.raises(ValueError):
        mctx.mcmc_relocate(p[:-1], m, s, v, dst, src)
    raw(mctx)()  # a valid call
    _fp16_and_sharded(gs, mctx, v, raw, RELOCATE)


def _fp16_and_sharded(gs, ctx, v, raw, entry):
    ctx.set_sh_storage(True)
    ctx.upload(v)
    expect(gs, ctx, gs.ERR_INVALID, raw(ctx), entry)
    ctx.set_sh_storage(False)
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, raw(c0), entry)
    finally:
        grp.close()


def test_noise_errors(gs, mctx):
    v, p, _, _ = _state(gs, scenes.c1()[1])

    def raw(c, params=p, scale=1.0, shift=0):
        return lambda: c._ck(gs.lib.gsb_mcmc_noise(c.h, None if params is None else params.data_ptr() + shift, v.data_ptr(),
                                                   scale, 1, 2, None))

    assert gs.lib.gsb_mcmc_noise(None, p.data_ptr(), v.data_ptr(), 1.0, 1, 2, None) == gs.ERR_INVALID
    expect(gs, mctx, gs.ERR_NO_SCENE, raw(mctx), NOISE)
    mctx.upload(v)
    for fn in (raw(mctx, params=None), raw(mctx, shift=4), raw(mctx, scale=-1.0), raw(mctx, scale=float("nan")),
               raw(mctx, scale=float("inf"))):
        expect(gs, mctx, gs.ERR_INVALID, fn, NOISE)
    with pytest.raises(ValueError):
        mctx.mcmc_noise(p.double(), v, 1.0, 1, 2)
    raw(mctx)()
    _fp16_and_sharded(gs, mctx, v, raw, NOISE)


# ---------------------------------------------------------------- the scene after either entry
def _entries(gs, ctx, p, m, s, v, which):
    torch = _torch()
    if which == "noise":
        ctx.mcmc_noise(p, v, SCALE, SEED, STEP)
    else:
        dst, src = _dead_and_sources(gs, v.clone(), 0.05, torch.Generator().manual_seed(2))
        ctx.mcmc_relocate(p, m, s, v, dst, src)


@pytest.mark.parametrize("which", ["noise", "relocate"])
def test_scene_after_entry_equals_upload_and_frames(gs, mctx, which):
    """The resident scene renders what an upload of `vertices` renders (6 cameras x levels 0/1/2 x EXACT/FAST); a backward
    pass is refused until the next frame; the next frame replays the captured graph and equals a frame without graphs."""
    torch = _torch()
    v, p, m, s = _state(gs, scenes.c1()[1])
    u = scenes.camera("c1")
    mctx.upload(v)
    mctx.set_timers(False)
    render(mctx, u)
    gi = torch.from_numpy(grad_image(u)).cuda()
    gv = torch.empty_like(v)
    _entries(gs, mctx, p, m, s, v, which)
    torch.cuda.synchronize()
    expect(gs, mctx, gs.ERR_INVALID, lambda: mctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr()), "gsb_render_backward")
    render(mctx, u)
    mctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr())  # a frame later: fine
    _entries(gs, mctx, p, m, s, v, which)
    with_graph = mctx.render(u)
    mctx.set_graph(False)
    without = mctx.render(u)
    mctx.set_graph(True)
    assert np.array_equal(with_graph.view(np.uint32), without.view(np.uint32))
    mctx.set_timers(True)
    _assert_coherent(gs, mctx, v, SIX)


# ---------------------------------------------------------------- training under a budget
POSES = [([0, 0, 5], [1, 0, 0, 0]), ([0.6, 0.1, 5.2], scenes.quat_axis_angle([0, 1, 0], 6)),
         ([-0.5, -0.3, 4.8], scenes.quat_axis_angle([1, 0, 0], -5))]
MCMC_LR = [1.6e-4, 5e-3, 5e-2, 1e-3, 1e-2, 5e-4]


def _train(gs, ctx, steps=600):
    """From every 8th Gaussian of c1 (scales x 1.5), cap_max = 2 x the start: the MCMC loop with relocate(cap_max,
    growth=0.25) every 50 steps from step 50.  Returns (optimizer, sizes after every step, rows below the floor after each
    relocate, losses before and after)."""
    torch = _torch()
    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    views = [gs.uniforms_from_camera(pp, q, 45.0, 0.1, 1000.0, 320, 240) for pp, q in POSES]
    with torch.no_grad():
        targets = [gs.render_torch(ctx, full, uu).clone() for uu in views]
    start = full[::8].clone()
    start[:, 4:7] *= 1.5
    cap = 2 * start.shape[0]
    opt = gs.SceneAdam(ctx, start, MCMC_LR, selective=False, seed=123)
    gen = torch.Generator().manual_seed(7)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")

    def loss():
        ms = [gs.image_metrics(ctx, opt.render(uu), t) for uu, t in zip(views, targets)]
        return sum(0.8 * mm["l1"] + 0.2 * (1 - mm["ssim"]) for mm in ms) / len(ms)

    loss0, sizes, below = loss(), [], []
    for it in range(1, steps + 1):
        k = it % 3
        ctx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g, opacity_reg=0.01, scale_reg=0.01)
        opt.inject_noise()
        if it % 50 == 0:
            opt.relocate(cap, growth=0.25, generator=gen)
            below.append(int((opt.vertices[:, 7] < 0.005).sum()))
        sizes.append(opt.vertices.shape[0])
    return opt, cap, sizes, below, loss0, loss()


def test_mcmc_training_under_a_budget(gs, mctx):
    torch = _torch()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        opt, cap, sizes, below, loss0, loss1 = _train(gs, mctx)
        words = [_bits(t).cpu() for t in (opt.params, opt.exp_avg, opt.exp_avg_sq, opt.vertices)]
        twin = gs.Context(0)
        try:
            opt2, *_ = _train(gs, twin)
            words2 = [_bits(t).cpu() for t in (opt2.params, opt2.exp_avg, opt2.exp_avg_sq, opt2.vertices)]
        finally:
            twin.close()
    finally:
        torch.use_deterministic_algorithms(prev)
    print(f"MCMC: n {sizes[0]} -> {sizes[-1]} (cap {cap}), loss {loss0:.5f} -> {loss1:.5f}, rows below the floor after "
          f"each relocate {below}")
    assert max(sizes) <= cap and sizes[-1] == cap
    assert all(b == 0 for b in below)
    assert loss1 < loss0
    for a, b in zip(words, words2):
        assert torch.equal(a, b)


def test_regularisers_off_keep_the_step(gs, mctx):
    """step(g) and step(g, opacity_reg=0, scale_reg=0) give the same words; non-zero values add exactly lambda / n and
    lambda / (3 n) to the gradient."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    g = torch.from_numpy(grad_image(u)).cuda()
    out = []
    for kw in ({}, {"opacity_reg": 0.0, "scale_reg": 0.0}, {"opacity_reg": 0.01, "scale_reg": 0.02}):
        ctx = gs.Context(0)
        try:
            torch.use_deterministic_algorithms(True)
            opt = gs.SceneAdam(ctx, torch.from_numpy(vtx).cuda(), MCMC_LR, selective=False)
            opt.render(u)
            opt.step(g, **kw)
            torch.cuda.synchronize()
            out.append((opt.grad.clone(), opt.params.clone()))
        finally:
            torch.use_deterministic_algorithms(False)
            ctx.close()
    assert torch.equal(_bits(out[0][0]), _bits(out[1][0])) and torch.equal(_bits(out[0][1]), _bits(out[1][1]))
    n = vtx.shape[0]
    want = out[0][0].clone()
    want[:, 7] += 0.01 / n
    want[:, 4:7] += 0.02 / (3 * n)
    assert torch.equal(_bits(out[2][0]), _bits(want))
