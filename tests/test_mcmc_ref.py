"""CPU side of 3DGS-MCMC (tests/mcmc_ref.py, DESIGN.md section 16): the numpy Philox4x32-10 reproduces Random123's known
answers; the entry's fp64 relocation rule equals the paper's double sum evaluated at 100 digits and preserves the line
integral of opacity; mcmc_sample never picks a zero-weight row, reproduces its draws and follows the weights; and
relocate_reference gives the expected values on a hand-built table."""
import math

import numpy as np
import pytest
import torch

import mcmc_ref


@pytest.mark.parametrize("key, ctr, want", [
    ((0x00000000, 0x00000000), (0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff), (0xffffffff,) * 4, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0xa4093822, 0x299f31d0), (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
], ids=["zeros", "ones", "pi"])
def test_philox_known_answers(key, ctr, want):
    got = mcmc_ref.philox4x32_10(np.array([ctr], np.uint32), np.array(key, np.uint32))[0]
    assert [int(w) for w in got] == list(want)


def test_noise_words_layout():
    """Counter (row, lo32(step), hi32(step), 0) and key (lo32(seed), hi32(seed)), as the entry states them."""
    seed, step = 0x0123456789ABCDEF, 0xFEDCBA9876543210
    got = mcmc_ref.noise_words(np.array([5]), seed, step)[0]
    want = mcmc_ref.philox4x32_10(np.array([[5, 0x76543210, 0xFEDCBA98, 0]], np.uint32), np.array([0x89ABCDEF, 0x01234567], np.uint32))[0]
    assert np.array_equal(got, want)
    u = mcmc_ref.uniforms(np.array([0, 0xFFFFFFFF], np.uint32))
    assert u[0] > 0 and u[1] == 1.0  # (0, 1]: the logs are finite


ALPHAS = [0.005, 0.05, 0.5, 0.99, 1.0 - 2.0 ** -23]


def test_single_sum_equals_the_papers_double_sum():
    """The hockey-stick reduction in fp64 against the double sum at 100 digits, r = 2 ... 120.  Two cancellations set the
    fp64 rule's accuracy: the alternating sum's, whose condition number sum |term| / |denom| reaches ~10^4 at alpha near
    1 (its terms grow like (-log(1 - alpha))^j / j!), and 1 - (1 - alpha)^(1/r)'s, whose rounding is 2^-53 / x relative.
    At the same x (the fp64 x taken exactly) the single sum is within 1e-12 or 8 cond 2^-53 relative of the double sum;
    the whole rule is within that plus 2^-52 / x of an all-decimal evaluation."""
    worst_sum = worst_rule = 0.0
    for alpha in ALPHAS:
        for r in range(2, 121):
            x, coeff, cond = mcmc_ref.relocation_coeff(alpha, r, with_cond=True)
            at_x = float(mcmc_ref.paper_coeff_decimal(alpha, r, x=x))
            exact = float(mcmc_ref.paper_coeff_decimal(alpha, r))
            e_sum, e_rule = abs(coeff - at_x) / at_x, abs(coeff - exact) / exact
            worst_sum, worst_rule = max(worst_sum, e_sum), max(worst_rule, e_rule)
            tol = max(1e-12, 8 * cond * 2.0 ** -53)
            assert e_sum <= tol, (alpha, r, coeff, at_x, cond)
            assert e_rule <= tol + 2.0 ** -52 / x, (alpha, r, coeff, exact, cond)
    print(f"fp64 single sum vs 100-digit double sum: worst relative error {worst_sum:.2e} at the same x, "
          f"{worst_rule:.2e} for the whole rule")


@pytest.mark.parametrize("alpha", ALPHAS)
@pytest.mark.parametrize("r", [2, 3, 7, 51, 52, 120])
def test_relocation_preserves_the_line_integral(alpha, r):
    """r copies of opacity x and scale c = coeff composite, along a line through the centre, to what the source did:
    int_0^inf 1 - (1 - x exp(-u^2 / c^2))^r du == alpha sqrt(pi) / 2 (the source at scale 1)."""
    from scipy.integrate import quad

    x, c = mcmc_ref.relocation_coeff(alpha, r)

    def f(u):
        return -math.expm1(r * math.log1p(-x * math.exp(-(u / c) ** 2)))

    got, _ = quad(f, 0.0, math.inf, epsabs=1e-14, epsrel=1e-13, limit=200)
    assert abs(got - alpha * math.sqrt(math.pi) / 2) <= 1e-10, (got, alpha * math.sqrt(math.pi) / 2)


def test_mcmc_sample_skips_zero_weights_and_reproduces(gs):
    w = torch.tensor([0.0, 0.3, 0.0, 0.0, 1e-30, 0.7, 0.0, 2.0, 0.0, 0.0])
    a = gs.mcmc_sample(w, 200_000, torch.Generator().manual_seed(3))
    b = gs.mcmc_sample(w, 200_000, torch.Generator().manual_seed(3))
    c = gs.mcmc_sample(w, 200_000, torch.Generator().manual_seed(4))
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert a.dtype == torch.int64 and int(a.min()) >= 0 and int(a.max()) <= 7
    assert not bool((w[a] == 0).any())
    # a total the draws round up to: trailing zero rows are still never chosen
    one = gs.mcmc_sample(torch.tensor([1.0, 0.0, 0.0]), 1000, torch.Generator().manual_seed(0))
    assert bool((one == 0).all())
    with pytest.raises(ValueError):
        gs.mcmc_sample(torch.zeros(4), 3)
    with pytest.raises(ValueError):
        gs.mcmc_sample(torch.tensor([1.0, -0.5]), 3)


def test_mcmc_sample_chi_square(gs):
    from scipy.stats import chisquare

    w = torch.tensor([5.0, 1.0, 0.0, 3.0, 0.5, 0.5, 10.0, 2.0, 0.0, 8.0])
    k = 400_000
    idx = gs.mcmc_sample(w, k, torch.Generator().manual_seed(11))
    counts = torch.bincount(idx, minlength=w.numel()).double()
    live = w > 0
    expected = w.double() / w.double().sum() * k
    assert float(counts[~live].sum()) == 0.0
    stat, p = chisquare(counts[live].numpy(), expected[live].numpy())
    print(f"chi-square {stat:.2f}, p {p:.3f}")
    assert p > 1e-3


def _table():
    """n = 80 rows: row 0 (alpha 0.6) sampled twice (r = 3); row 1 (alpha 0.006) once, its x clamped to min_opacity;
    row 2 (alpha 0.9) 59 times (r = 60 > 51); row 3 (alpha 1.0) once, its x clamped to 1 - 2^-23.  dst: rows 10 ... 72."""
    g = torch.Generator().manual_seed(5)
    v = torch.rand((80, 60), generator=g) + 0.1
    v[:, 3] = 1.0
    v[:4, 7] = torch.tensor([0.6, 0.006, 0.9, 1.0])
    p = torch.randn((80, 60), generator=g)
    m = torch.randn((80, 60), generator=g)
    s = torch.rand((80, 60), generator=g)
    src = [0, 0, 1] + [2] * 59 + [3]
    dst = list(range(10, 10 + len(src)))
    return p, m, s, v, dst, src


def test_relocate_reference_on_a_hand_built_table():
    p, m, s, v, dst, src = _table()
    P, A, M, R = mcmc_ref.relocate_reference(p, m, s, v, dst, src, 0.005)
    V = v.double()
    # r = 3 at alpha 0.6: the closed form 3x - 3x^2/sqrt(2) + x^3/sqrt(3)
    x = 1 - (1 - float(np.float32(0.6))) ** (1 / 3)
    coeff = float(np.float32(0.6)) / (3 * x - 3 * x * x / math.sqrt(2) + x ** 3 / math.sqrt(3))
    assert abs(float(R[0, 7]) - x) <= 1e-15
    assert torch.allclose(R[0, 4:7], V[0, 4:7] * coeff, rtol=1e-14, atol=0)
    # r = 2 at alpha 0.006: x = 1 - sqrt(0.994) < 0.005 is clamped, the scale keeps the unclamped rule
    x1 = 1 - math.sqrt(1 - float(np.float32(0.006)))
    assert x1 < 0.005 and float(R[1, 7]) == float(np.float32(0.005))
    c1 = float(np.float32(0.006)) / (2 * x1 - x1 * x1 / math.sqrt(2))
    assert torch.allclose(R[1, 4:7], V[1, 4:7] * c1, rtol=1e-14, atol=0)
    # r = 60, past the paper's 51-entry binomial table
    want = float(mcmc_ref.paper_coeff_decimal(float(np.float32(0.9)), 60))
    assert torch.allclose(R[2, 4:7], V[2, 4:7] * want, rtol=1e-12, atol=0)
    # alpha 1: x = 1 is clamped to 1 - 2^-23
    assert float(R[3, 7]) == 1.0 - 2.0 ** -23
    # raw parameters of the sources from the fp32 record values; moments zero on sources and destinations
    for r in range(4):
        o = float(np.float32(float(R[r, 7])))
        assert float(P[r, 7]) == math.log(o / (1 - o))
        assert torch.equal(P[r, 4:7], torch.from_numpy(R[r, 4:7].numpy().astype(np.float32)).double().log())
        assert torch.equal(P[r, :4], p[r, :4].double()) and torch.equal(P[r, 8:], p[r, 8:].double())
        assert torch.equal(R[r, :4], V[r, :4]) and torch.equal(R[r, 8:], V[r, 8:])
    for d, s_ in zip(dst, src):
        assert torch.equal(P[d], P[s_]) and torch.equal(R[d], R[s_])
    touched = sorted(set(dst) | set(src))
    assert bool((A[touched] == 0).all()) and bool((M[touched] == 0).all())
    rest = [i for i in range(80) if i not in touched]
    for got, was in ((P, p), (A, m), (M, s), (R, v)):
        assert torch.equal(got[rest], was[rest].double())
