"""References of gsb_mcmc_noise and gsb_mcmc_relocate (include/gs_b200.h, DESIGN.md section 16).

philox4x32_10        Random123's philox4x32_10 restated in numpy uint32 arithmetic, vectorised over counters
uniforms             ((float)x + 0.5f) * 2^-32 in float32, as the kernel forms them (two exact-or-rounded IEEE ops)
box_muller           the three normals of the kernel, in float64 from those float32 uniforms
noise_reference      the positions after the noise, in float64, with a bound on the fp32 kernel's distance from them
relocation_coeff     the fp64 rule of the entry (x, the single alternating sum, coeff), in numpy
paper_coeff_decimal  the paper's double sum over i and k, in `decimal` at 100 digits (independent of the single sum)
relocate_reference   every array after a relocation, in float64 torch, before the entry's rounding to fp32
"""
from decimal import Decimal, getcontext
from math import comb

import numpy as np

M0, M1 = np.uint32(0xD2511F53), np.uint32(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)


def _mulhilo(a, b):
    p = a.astype(np.uint64) * np.uint64(b)
    return (p >> np.uint64(32)).astype(np.uint32), (p & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def philox4x32_10(counter, key):
    """counter: (..., 4) uint32, key: (2,) or (..., 2) uint32 -> (..., 4) uint32."""
    c = [np.asarray(counter, np.uint32)[..., i].copy() for i in range(4)]
    key = np.asarray(key, np.uint32)
    k0, k1 = key[..., 0].copy(), key[..., 1].copy()
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0 = k0 + W0
                k1 = k1 + W1
            hi0, lo0 = _mulhilo(c[0], M0)
            hi1, lo1 = _mulhilo(c[2], M1)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, -1)


def noise_words(rows, seed, step):
    """The Philox words of the noise for row indices `rows`: counter (i, lo32(step), hi32(step), 0), key (lo32, hi32)(seed)."""
    rows = np.asarray(rows, np.uint64)
    ctr = np.zeros(rows.shape + (4,), np.uint32)
    ctr[..., 0] = rows.astype(np.uint32)
    ctr[..., 1] = np.uint32(step & 0xFFFFFFFF)
    ctr[..., 2] = np.uint32(step >> 32)
    return philox4x32_10(ctr, np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint32))


def uniforms(words):
    """((float)x + 0.5f) * 2^-32 in float32, in (0, 1]."""
    return (words.astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -32)


def box_muller(u):
    """(..., 4) float32 uniforms -> (..., 3) float64 normals: eps0, eps1 from u0, u1 and eps2 from u2, u3."""
    u = u.astype(np.float64)
    rho0 = np.sqrt(-2.0 * np.log(u[..., 0]))
    rho2 = np.sqrt(-2.0 * np.log(u[..., 2]))
    return np.stack([rho0 * np.cos(2 * np.pi * u[..., 1]), rho0 * np.sin(2 * np.pi * u[..., 1]),
                     rho2 * np.cos(2 * np.pi * u[..., 3])], -1)


def sigma_rows(cov):
    """(n, 6) float32 Sigma words (S00, S01, S02, S11, S12, S22) -> (n, 3, 3) float64."""
    c = cov.astype(np.float64)
    return np.stack([np.stack([c[:, 0], c[:, 1], c[:, 2]], -1), np.stack([c[:, 1], c[:, 3], c[:, 4]], -1),
                     np.stack([c[:, 2], c[:, 4], c[:, 5]], -1)], -2)


def gate(opacity):
    """1 / (1 + exp(100 (o - 0.005f))) in float64 of the float32 opacity and the float32 constant."""
    z = 100.0 * (opacity.astype(np.float64) - float(np.float32(0.005)))
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(z))


def noise_reference(params, cov, opacity, scale, seed, step):
    """(p', bound): float64 positions after the noise and, per component, a bound on the fp32 kernel's distance from them.
    params (n, 60) float32, cov (n, 6) float32 Sigma words, opacity (n,) float32 (the scene's words).

    The bound sums: the last rounding of p' (2^-24 |p'|); eps within 1e-6 (1 + |eps|) (cospif / sinpif / logf / sqrtf);
    the gate's fp32 argument z = 100 (o - 0.005f), whose two roundings move exp by up to 2 |z| 2^-24 relative, plus
    expf, the add, the divide and the two products of e (16 roundings); and the three products and two sums of Sigma e
    (8 roundings of sum |S_rk e_k|)."""
    n = params.shape[0]
    eps = box_muller(uniforms(noise_words(np.arange(n), seed, step)))
    S = sigma_rows(cov)
    gs = gate(opacity) * float(np.float32(scale))
    e = eps * gs[:, None]
    d = np.einsum("nrk,nk->nr", S, e)
    p = params[:, 0:3].astype(np.float64) + d
    u = 2.0 ** -24
    g_rel = (2.0 * np.abs(100.0 * (opacity.astype(np.float64) - 0.005)) + 16.0) * u
    per_k = (np.abs(eps) * (g_rel[:, None] + 8 * u) + 1.01e-6 * (1.0 + np.abs(eps))) * np.abs(gs)[:, None]
    bound = u * np.abs(p) + np.einsum("nrk,nk->nr", np.abs(S), per_k)
    return p, bound, eps


def relocation_coeff(alpha, r, with_cond=False):
    """The entry's fp64 rule for one source: (x, coeff), and with_cond the alternating sum's condition number
    sum |term| / |denom| as a third value."""
    x = 1.0 - (1.0 - float(alpha)) ** (1.0 / r)
    denom, t, total = 0.0, 1.0, 0.0
    for j in range(1, r + 1):
        t = t * (r - j + 1) / j * x
        term = t / np.sqrt(float(j))
        denom = denom + term if j % 2 else denom - term
        total += term
    return (x, float(alpha) / denom, total / abs(denom)) if with_cond else (x, float(alpha) / denom)


def paper_coeff_decimal(alpha, r, digits=100, x=None):
    """coeff = alpha / sum_{i=1..r} sum_{k=0..i-1} C(i-1, k) (-1)^k x^(k+1) / sqrt(k+1), x = 1 - (1 - alpha)^(1/r), in
    decimal arithmetic at `digits` digits (alpha taken exactly from its float64 value; x, when given, likewise)."""
    getcontext().prec = digits
    a = Decimal(float(alpha))
    x = 1 - (1 - a) ** (Decimal(1) / Decimal(r)) if x is None else Decimal(float(x))
    powers = [x ** (k + 1) for k in range(r)]
    roots = [Decimal(k + 1).sqrt() for k in range(r)]
    denom = Decimal(0)
    for i in range(1, r + 1):
        for k in range(i):
            term = comb(i - 1, k) * powers[k] / roots[k]
            denom += -term if k % 2 else term
    return a / denom


def relocate_reference(params, exp_avg, exp_avg_sq, vertices, dst, src, min_opacity):
    """Every array after gsb_mcmc_relocate(dst, src), in float64 torch from float32 inputs: (params, exp_avg, exp_avg_sq,
    vertices), each (n, 60).  A source's record values are the fp64 rule before their rounding to fp32; its params' logit
    and log scale are taken, as the entry does, from the fp32 roundings of those record values."""
    import torch

    P, A, M, V0 = (t.detach().cpu().double().clone() for t in (params, exp_avg, exp_avg_sq, vertices))
    R = V0.clone()  # the records after the call
    dst = [int(i) for i in dst]
    src = [int(i) for i in src]
    counts = {}
    for s in src:
        counts[s] = counts.get(s, 0) + 1
    hi = 1.0 - 2.0 ** -23
    min_opacity = float(np.float32(min_opacity))  # the entry's argument is a float
    for s, c in counts.items():
        alpha = float(V0[s, 7])
        x, coeff = relocation_coeff(alpha, c + 1)
        o = min(max(x, float(min_opacity)), hi)
        R[s, 7] = o
        R[s, 4:7] = V0[s, 4:7] * coeff
        o32 = float(np.float32(o))
        s32 = torch.from_numpy(R[s, 4:7].numpy().astype(np.float32)).double()
        P[s, 4:7] = torch.log(s32)
        P[s, 7] = np.log(o32 / (1.0 - o32))
        A[s] = 0.0
        M[s] = 0.0
    for d, s in zip(dst, src):
        P[d] = P[s]
        R[d] = R[s]
        A[d] = 0.0
        M[d] = 0.0
    return P, A, M, R
