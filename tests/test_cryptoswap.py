"""Two-coin cryptoswap (Curve v2, twocrypto-ng) pools, kind 8: the invariant, its concavity over the accepted (A, gamma)
domain, the per-pool optimal trade, its Hessian coefficient, the per-thread solver, the pool-parallel kernel and every
solve path.

CPU: the invariant against 50-digit decimal; the concavity of D(t, 1) in decimal at the corners and midpoints of the
accepted domain; the longdouble reference (tests/xp_cryptoswap.py) against a brute-force maximisation along the curve in
mpmath (no marginal-rate formula); the no-trade band; the product limit A -> 0; hc by finite differences; near-peg pools;
cfmm_small::cryptoswap_pair and the per-thread solver compiled for the host; rejections; the contract conversion.
GPU (H100): cfmm_arb_eval in its four instances on 1M pools near and far from the peg, the Hessian kernels, every solve
path certified, in-place updates (one store and rank stores), unit covariance and the C ABI's return codes.

Error bounds.  As for StableSwap (tests/test_stableswap.py): a trading pool's post-trade balance solves
log s(t) = log q*, which fp64 evaluates with an absolute error of a few u (here through the inner solve for the curve
point as well), so the flows carry an error of ~c u X_a / |phi'| = c u gamma hc / nu_a; they are compared with
    |dflow| <= 1e-12 gross + 8 u max(R) / gamma + COND u gamma hc / nu_a.
"""
import ctypes as C
import os
import subprocess
import types
from decimal import Decimal, getcontext

import mpmath as mp
import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib, instances as I
from cfmm_routing_code_b200.pools import (HostPools, KIND_CRYPTOSWAP_HOST, CRYPTO_A_RANGE, CRYPTO_GAMMA_RANGE,
                                          check_pool_update, cryptoswap_invariant)
import small_host
import xp_cryptoswap as XK

U = 2.0 ** -53
COND = 256.0
HERE = os.path.dirname(os.path.abspath(__file__))
FEES = [1.0, 0.9995, 0.997, 0.99]


# ------------------------------------------------------------------------------------------------------ helpers
def _dec_f(y0, y1, A, G, D):
    K0 = 4 * y0 * y1 / (D * D)
    K = A * K0 * G * G / ((G + 1 - K0) ** 2)
    return K * D * (y0 + y1) + y0 * y1 - K * D * D - D * D / 4


def _dec_D(y0, y1, A, G, iters=190):
    """the invariant by bisection on [2 sqrt(y0 y1), y0 + y1] in decimal (f > 0 below the root)"""
    y0, y1, A, G = Decimal(y0), Decimal(y1), Decimal(A), Decimal(G)
    lo, hi = 2 * (y0 * y1).sqrt(), y0 + y1
    for _ in range(iters):
        mid = (lo + hi) / 2
        lo, hi = (mid, hi) if _dec_f(y0, y1, A, G, mid) > 0 else (lo, mid)
    return (lo + hi) / 2


_HOST = None


def _host():
    """tests/host_harness/cryptoswap_host.cpp: cfmm_small::cryptoswap_pair and the cryptoswap solver instance, host build"""
    global _HOST
    if _HOST is None:
        src = os.path.join(HERE, "host_harness", "cryptoswap_host.cpp")
        hdr = os.path.join(HERE, "..", "cfmm_routing_code_b200", "csrc", "cfmm_small.cuh")
        lib = os.path.join(HERE, "_build", "libcryptoswap_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src],
                           check=True)
        _HOST = C.CDLL(lib)
    return _HOST


def host_pairs(R, c, A, G, g, nu):
    m = len(g)
    arr = [np.ascontiguousarray(x, np.float64) for x in (R, c, A, G, g, nu)]
    D, L, hc = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m)
    p_ = lambda x: x.ctypes.data_as(C.c_void_p)
    _host().cryptoswap_host_pairs(C.c_longlong(m), *[p_(x) for x in arr], p_(D), p_(L), p_(hc))
    return D, L, hc


def marginal(R, p, A, G, Dv):
    """token-0 price (in token 1) at which the pool is on its band edge with gamma = 1: (p0 / p1) s(R)"""
    ua = p[0] * R[0] / Dv
    f, _, _ = XK._phi(np.log(np.array([ua], XK.LD)), XK.LD(A), XK.LD(G), XK.LD(0))
    return float(p[0] / p[1] * np.exp(f[0]))


def random_pools(m, seed, far=0.5):
    """m pools over the accepted domain, some near their peg (balance ratios within 1e-9 .. 1e-2 of the scale), the rest
    far from it (up to 1e4x); prices near and away from the marginal rate"""
    rng = np.random.default_rng(seed)
    A = np.exp(rng.uniform(np.log(CRYPTO_A_RANGE[0]), np.log(CRYPTO_A_RANGE[1]), m))
    G = np.exp(rng.uniform(np.log(CRYPTO_GAMMA_RANGE[0]), np.log(CRYPTO_GAMMA_RANGE[1]), m))
    p = np.exp(rng.normal(0, 1, (m, 2)))
    V = np.exp(rng.normal(8, 2, m))
    isfar = rng.random(m) < far
    k = np.where(isfar, np.exp(rng.uniform(-9, 9, m)),
                 1 + rng.choice([-1, 1], m) * np.exp(rng.uniform(np.log(1e-9), np.log(1e-2), m)))
    R = np.stack([V * k / p[:, 0], V / p[:, 1]], 1)
    g = np.array(FEES)[rng.integers(0, 4, m)]
    Dv = cryptoswap_invariant(R, p, A, G)
    # the pool's own price, from the reference's marginal rate: prices within +-3 band widths, and some far outside
    base = np.array([marginal(R[i], p[i], A[i], G[i], Dv[i]) for i in range(m)]) if m <= 5000 else p[:, 0] / p[:, 1]
    dev = np.where(rng.random(m) < 0.7, rng.normal(0, 0.01, m), rng.normal(0, 1, m))
    nu = np.stack([base * np.exp(dev), np.ones(m)], 1) * np.exp(rng.normal(0, 1, m))[:, None]
    return R, p, A, G, Dv, g, nu


def flow_bound(Dx, Lx, hx, g, nu, R, eps=U, rel=1e-12):
    gross = (np.abs(Dx) + np.abs(Lx)).sum(1).astype(float)
    a = np.where(Dx[:, 0] > 0, 0, 1)
    nua = np.asarray(nu, float)[np.arange(len(g)), a]
    g = np.asarray(g, float)
    return rel * gross + 8 * eps * np.asarray(R, float).reshape(-1, 2).max(1) / g + \
        COND * eps * g * np.abs(hx.astype(float)) / nua


def crypto_hp(R, p, A, G, g, toks=None, n=None):
    m = len(g)
    toks = np.tile([0, 1], (m, 1)) if toks is None else toks
    n = int(toks.max()) + 1 if n is None else n
    return HostPools(n, np.arange(0, 2 * m + 1, 2, dtype=np.int64), np.ascontiguousarray(toks, np.int32).ravel(),
                     np.ascontiguousarray(R, np.float64).ravel(), np.ascontiguousarray(p, np.float64).ravel(),
                     np.asarray(g, np.float64), np.full(m, KIND_CRYPTOSWAP_HOST, np.uint8), np.asarray(A, np.float64),
                     cgam=np.asarray(G, np.float64))


def _check_against_xp(D, L, hc, R, p, A, G, Dv, g, nu):
    c = XK.LD(p) / XK.LD(Dv)[:, None]
    Dx, Lx, hx = XK.cryptoswap_response(R, c, A, G, g, nu)
    bound = flow_bound(Dx, Lx, hx, g, nu, R)
    err = np.maximum(np.abs(D - Dx.astype(float)).max(1), np.abs(L - Lx.astype(float)).max(1))
    assert np.all(err <= bound), float((err / bound).max())
    tr = (hx > 0) & (hc > 0)
    mism = (hc > 0) != (hx > 0)
    gross_x = (np.abs(Dx) + np.abs(Lx)).sum(1).astype(float)
    assert np.all(gross_x[mism] <= bound[mism]), int(mism.sum())
    rel = np.abs(hc[tr] - hx[tr].astype(float)) / hx[tr].astype(float)
    return Dx, Lx, hx, float(rel.max()) if tr.any() else 0.0


# ====================================================================================================== CPU
def test_invariant_matches_decimal():
    getcontext().prec = 50
    worst = 0.0
    rng = np.random.default_rng(0)
    for A in (CRYPTO_A_RANGE[0], 0.5, 10.0, 400.0, CRYPTO_A_RANGE[1]):
        for G in (CRYPTO_GAMMA_RANGE[0], 1.45e-4, 2e-2, CRYPTO_GAMMA_RANGE[1]):
            for t in (1e-5, 0.01, 1 - 1e-9, 1.0, 1 + 1e-6, 3.0, 1e5):
                s = float(np.exp(rng.normal(0, 20)))
                y = np.array([t * s, s])
                d = float(cryptoswap_invariant(y[None], np.ones((1, 2)), [A], [G])[0])
                ref = _dec_D(y[0], y[1], A, G)
                worst = max(worst, float(abs(Decimal(d) - ref) / ref))
    assert worst <= 2e-15, worst


def test_invariant_is_concave_over_the_accepted_domain():
    """D(t, 1) concave in t (so the pool's trading set is convex) at the corners and midpoints of the accepted (A, gamma)
    domain, over t in [1e-5, 1e5] on a 0.25-decade grid and densely near t = 1: second differences in 50-digit decimal"""
    getcontext().prec = 50
    la, lg = np.log(CRYPTO_A_RANGE), np.log(CRYPTO_GAMMA_RANGE)
    As = np.exp([la[0], la.mean(), la[1]])
    Gs = np.exp([lg[0], lg.mean(), lg[1]])
    ts = list(10.0 ** np.arange(-5, 5.01, 0.25)) + [1 + s * d for d in (1e-9, 1e-7, 1e-5, 1e-3, 1e-2, 0.1, 0.3)
                                                   for s in (-1, 1)]
    for A in As:
        for G in Gs:
            for t in ts:
                h = Decimal(t) * Decimal(10) ** -6 if abs(t - 1) > 1e-3 else Decimal(10) ** -12
                T = Decimal(t)
                d2 = _dec_D(T + h, 1, A, G, 175) + _dec_D(T - h, 1, A, G, 175) - 2 * _dec_D(T, 1, A, G, 175)
                assert d2 < 0, (A, G, t, d2)


def _mp_brute(R, c, A, G, g, nu, a):
    """max over X_a >= R_a of nu_b (R_b - X_b) - nu_a (X_a - R_a) / gamma along the curve (mpmath, 30 digits, golden
    section in log X_a; u_b by bisection on the invariant): (Delta_a, Lambda_b), no marginal-rate formula used"""
    mp.mp.dps = 30
    b = 1 - a
    Ra, Rb, ca, cb = (mp.mpf(float(v)) for v in (R[a], R[b], c[a], c[b]))
    A_, G_, g_, na, nb = (mp.mpf(float(v)) for v in (A, G, g, nu[a], nu[b]))

    def ub_of(ua):
        lo, hi = max(1 - ua, mp.mpf(0)), 1 / (4 * ua)
        for _ in range(110):
            mid = (lo + hi) / 2
            K0 = 4 * ua * mid
            K = A_ * K0 * G_ ** 2 / (G_ + 1 - K0) ** 2
            lo, hi = (lo, mid) if K * (ua + mid - 1) + ua * mid - mp.mpf(1) / 4 > 0 else (mid, hi)
        return (lo + hi) / 2

    prof = lambda z: nb * (Rb - ub_of(ca * Ra * mp.e ** z) / cb) - na * Ra * (mp.e ** z - 1) / g_
    lo, hi = mp.mpf(0), mp.mpf(14)
    r = (mp.sqrt(5) - 1) / 2
    x1, x2 = hi - r * (hi - lo), lo + r * (hi - lo)
    f1, f2 = prof(x1), prof(x2)
    for _ in range(110):
        if f1 < f2:
            lo, x1, f1 = x1, x2, f2; x2 = lo + r * (hi - lo); f2 = prof(x2)
        else:
            hi, x2, f2 = x2, x1, f1; x1 = hi - r * (hi - lo); f1 = prof(x1)
    z = (lo + hi) / 2
    if not prof(z) > 0:
        return 0.0, 0.0
    xa = Ra * mp.e ** z
    return float((xa - Ra) / g_), float(Rb - ub_of(ca * xa) / cb)


def test_xp_and_host_match_brute_force_along_the_curve():
    R, p, A, G, Dv, g, nu = random_pools(14, seed=1)
    c = p / Dv[:, None]
    Dx, Lx, _ = XK.cryptoswap_response(R, XK.LD(p) / XK.LD(Dv)[:, None], A, G, g, nu)
    Dh, Lh, _ = host_pairs(R, c, A, G, g, nu)
    for i in range(len(g)):
        for a in (0, 1):
            d, l = _mp_brute(R[i], c[i], A[i], G[i], g[i], nu[i], a)
            sc = max(abs(d), abs(l), 1e-300)
            for DD, LL in ((Dx.astype(float), Lx.astype(float)), (Dh, Lh)):
                # the golden section finds the maximiser to ~1e-15 relative (the objective is flat there)
                assert abs(DD[i, a] - d) <= 1e-9 * sc + 1e-12 * R[i].max() and \
                    abs(LL[i, 1 - a] - l) <= 1e-9 * sc + 1e-12 * R[i].max(), (i, a, DD[i], LL[i], d, l)


def test_no_trade_band_is_exact():
    R, p, A, G, Dv, g, _ = random_pools(300, seed=2)
    g = np.full(len(g), 0.997)
    base = np.array([marginal(R[i], p[i], A[i], G[i], Dv[i]) for i in range(len(g))])
    for f in (0.9971, 1.0, 1 / 0.9971):
        nu = np.stack([base * f, np.ones(len(g))], 1)
        D, L, hc = host_pairs(R, p / Dv[:, None], A, G, g, nu)
        assert np.all(D == 0) and np.all(L == 0) and np.all(hc == 0)


def test_small_A_is_the_product_pool_on_scaled_reserves():
    """A -> 0: K -> 0 and the curve is y0 y1 = D^2 / 4, the constant product on y = p x"""
    rng = np.random.default_rng(3)
    m = 300
    G = np.exp(rng.uniform(np.log(CRYPTO_GAMMA_RANGE[0]), np.log(CRYPTO_GAMMA_RANGE[1]), m))
    p = np.exp(rng.normal(0, 1, (m, 2)))
    R = np.exp(rng.normal(5, 1, (m, 2))) / p                          # scaled balances within ~10x of each other
    g = np.array(FEES)[rng.integers(0, 4, m)]
    nu = np.stack([p[:, 0] / p[:, 1] * np.exp(rng.normal(0, 1, m)), np.ones(m)], 1)
    A = np.full(m, 1e-10)                             # (below the accepted domain: the harness takes any A)
    Dv = cryptoswap_invariant(R, p, A, G)
    D, L, _ = host_pairs(R, p / Dv[:, None], A, G, g, nu)
    y = R * p
    mu = nu / p
    for a in (0, 1):
        b = 1 - a
        t = np.sqrt(np.maximum(g * mu[:, b] * y[:, b] / (mu[:, a] * y[:, a]), 1.0))
        Dp = R[:, a] * (t - 1) / g
        Lp = R[:, b] * (1 - 1 / t)
        sc = np.abs(Dp) + np.abs(Lp) + 1e-300
        assert np.all(np.abs(D[:, a] - Dp) <= 1e-7 * sc) and np.all(np.abs(L[:, b] - Lp) <= 1e-7 * sc)


def test_hc_matches_finite_differences():
    """hc = nu_0 d(Lambda_0 - Delta_0) / d log nu_0 (the scaled Hessian's pair coefficient), central differences in fp64
    (step 1e-6: rounding ~1e-10 of the flows, truncation ~1e-12)"""
    R, p, A, G, Dv, g, nu = random_pools(400, seed=4)
    c = p / Dv[:, None]
    _, _, hc = host_pairs(R, c, A, G, g, nu)
    h = 1e-6
    up, dn = nu.copy(), nu.copy()
    up[:, 0] *= np.exp(h); dn[:, 0] *= np.exp(-h)
    Du, Lu, _ = host_pairs(R, c, A, G, g, up)
    Dd, Ld, _ = host_pairs(R, c, A, G, g, dn)
    fd = nu[:, 0] * ((Lu[:, 0] - Du[:, 0]) - (Ld[:, 0] - Dd[:, 0])) / (2 * h)
    D0, L0, _ = host_pairs(R, c, A, G, g, nu)
    a = np.where(D0[:, 0] > 0, 0, 1)
    Xa = R[np.arange(len(g)), a] + g * D0[np.arange(len(g)), a]
    # the band edge itself is not differentiable: keep pools whose trade is well inside on both sides
    ok = (hc > 0) & (np.abs(fd - hc) <= 1e-4 * hc + 1e-5 * nu[:, 0] * Xa)
    trading = (hc > 0).sum()
    assert trading > 100 and ok.sum() >= trading - 3, (int(trading), int(ok.sum()))


def test_near_peg_pools_match_xp():
    """balance ratios within 1e-9 .. 1e-3 of the price scale and gamma down to the accepted minimum: the cancellation-free
    forms of 1 - K0 and s - 1 keep the fp64 kernel within the flow bound of the longdouble reference"""
    rng = np.random.default_rng(5)
    m = 2000
    A = np.exp(rng.uniform(np.log(1.0), np.log(CRYPTO_A_RANGE[1]), m))
    G = np.exp(rng.uniform(np.log(CRYPTO_GAMMA_RANGE[0]), np.log(1e-3), m))
    p = np.exp(rng.normal(0, 1, (m, 2)))
    k = 1 + rng.choice([-1, 1], m) * np.exp(rng.uniform(np.log(1e-9), np.log(1e-3), m))
    R = np.stack([1e4 * k / p[:, 0], 1e4 / p[:, 1]], 1)
    Dv = cryptoswap_invariant(R, p, A, G)
    g = np.array([1.0, 0.9999, 0.9995])[rng.integers(0, 3, m)]
    nu = np.stack([p[:, 0] / p[:, 1] * np.exp(rng.normal(0, 1e-4, m)), np.ones(m)], 1)
    D, L, hc = host_pairs(R, p / Dv[:, None], A, G, g, nu)
    *_, hrel = _check_against_xp(D, L, hc, R, p, A, G, Dv, g, nu)
    assert (hc > 0).sum() > m // 3 and hrel <= 1e-6, ((hc > 0).sum(), hrel)


def test_host_pair_matches_xp_reference():
    R, p, A, G, Dv, g, nu = random_pools(4000, seed=6)
    D, L, hc = host_pairs(R, p / Dv[:, None], A, G, g, nu)
    *_, hrel = _check_against_xp(D, L, hc, R, p, A, G, Dv, g, nu)
    assert (hc > 0).sum() > 1000 and hrel <= 1e-6, hrel


def _small_crypto_problem(rng):
    """3-6 tokens: a product chain plus cryptoswap pools between tokens 0..2, near or far from their peg"""
    n = int(rng.integers(3, 7))
    prices = np.exp(rng.normal(0, 1, n))
    li, res, fees, kinds, w = [], [], [], [], []
    for i in range(n - 1):
        liq = np.exp(rng.normal(4, 1))
        li.append([i, i + 1]); res.append(list(liq / prices[[i, i + 1]] * np.exp(0.05 * rng.standard_normal(2))))
        fees.append(0.997); kinds.append("product"); w.append(None)
    for _ in range(int(rng.integers(2, 5))):
        a, b = (int(x) for x in rng.choice(3, 2, replace=False))
        sh = float(np.exp(rng.choice([0.0, 0.0, 0.5, -1.0]) + 0.002 * rng.standard_normal()))
        V = np.exp(rng.normal(5, 1))
        li.append([a, b]); res.append([V / prices[a] * np.exp(0.02 * rng.standard_normal()), V / (prices[b] * sh)])
        fees.append(float(rng.choice([0.9995, 0.997]))); kinds.append("cryptoswap")
        w.append((float(rng.choice([2.5, 10.0, 400.0])), float(rng.choice([1.45e-4, 2e-3, 2e-2])),
                  float(prices[a]), float(prices[b] * sh)))
    d = dict(n_tokens=n, local_indices=li, reserves=res, fees=fees, kinds=kinds, weights=w)
    return HostPools.from_lists(n, li, res, fees, kinds, w), d, prices


def _utilities(rng, n, prices):
    U_ = XK.Utility
    us = [U_.arbitrage(prices * np.exp(0.01 * rng.standard_normal(n)))]
    us.append(U_.swap(n, 0, 1, float(np.exp(rng.normal(1, 1)) / prices[0])))
    basket = np.zeros(n); basket[1] = float(np.exp(rng.normal(0, 1)) / prices[1])
    basket[2] = float(np.exp(rng.normal(0, 1)) / prices[2])
    us.append(U_.liquidate(n, 0, basket))
    return us


def _csr_args(hp):
    """the cfmm_csr_pools arrays: kind 8's w = p / D, logrw = (A, G) per pool; log(R / w) elsewhere"""
    slot_kind = np.repeat(hp.kind, np.diff(hp.pool_ptr))
    logrw = np.log(np.maximum(hp.reserves, 1e-300) / np.where(slot_kind == 0, hp.weights, 1.0))
    w = np.asarray(hp.weights, np.float64).copy()
    cs = np.nonzero(hp.kind == KIND_CRYPTOSWAP_HOST)[0]
    f = hp.pool_ptr[cs]
    w[f] = hp.weights[f] / hp.inv[cs]; w[f + 1] = hp.weights[f + 1] / hp.inv[cs]
    logrw[f] = hp.amp[cs]; logrw[f + 1] = hp.cgam[cs]
    return [np.ascontiguousarray(x, t) for x, t in ((hp.pool_ptr, np.int64), (hp.tok_idx, np.int32),
                                                    (hp.reserves, np.float64), (w, np.float64),
                                                    (logrw, np.float64), (hp.gamma, np.float64), (hp.kind, np.uint8))]


def _host_solve(hp, specs, tol=1e-9, crypto=True):
    """the per-thread solver built for the host: its cryptoswap instance, or (crypto=False) the plain one"""
    n, B, nnz = hp.n_tokens, len(specs), len(hp.tok_idx)
    c = np.stack([u.c for u in specs]).astype(float); a = np.stack([u.a for u in specs]).astype(float)
    fl = np.ascontiguousarray(np.stack([np.asarray(u.eq, np.uint8) | (np.asarray(u.pinned, np.uint8) << 1)
                                        for u in specs]), np.uint8)
    nu = np.ascontiguousarray(np.stack([np.where(u.c > 0, u.c, np.median(u.c[u.c > 0]) if (u.c > 0).any() else 1.0)
                                        for u in specs]))
    keep = _csr_args(hp)
    psi = np.zeros((B, n)); st = np.zeros((B, 8)); d = np.zeros((B, nnz)); l = np.zeros((B, nnz))
    p_ = lambda x: x.ctypes.data_as(C.c_void_p)
    if crypto:
        fn = _host().cryptoswap_host_solve
        fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 7 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
        fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), tol)
    else:
        small_host.load().small_host_solve(n, hp.m, *[p_(k) for k in keep], B, None, p_(c), p_(a), p_(fl), p_(nu),
                                           p_(psi), p_(st), p_(d), p_(l), nnz, tol, 1)
    return dict(nu=nu, psi=psi, stats=st, delta=d, lam=l)


def _as_result(hp, out, p):
    ptr = hp.pool_ptr
    return types.SimpleNamespace(value=out["stats"][p][0], dual_value=out["stats"][p][1], psi=out["psi"][p],
                                 nu=out["nu"][p], deltas=[out["delta"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                 lambdas=[out["lam"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])


def test_existing_solver_instances_reject_cryptoswap_pools():
    """the plain instance (and, through the same kind check, the StableSwap, StableSwap-n and concentrated ones, whose
    accepted kinds stop at 4 and 6) refuse kind 8: status 3, NaN results"""
    rng = np.random.default_rng(100)
    hp, _, prices = _small_crypto_problem(rng)
    out = _host_solve(hp, _utilities(rng, hp.n_tokens, prices), crypto=False)
    assert np.all(out["stats"][:, 7] == 3) and np.all(np.isnan(out["stats"][:, 0]))
    import test_stableswap as TS
    out = TS._host_solve(hp, _utilities(rng, hp.n_tokens, prices), stable=True)
    assert np.all(out["stats"][:, 7] == 3)


def test_host_solver_matches_oracle_step_for_step():
    """same algorithm: same value and prices, and every problem certifies; iteration counts may differ where a line
    search barely accepts a step (the oracle evaluates the pools in numpy, the solver in C++)"""
    same = total = 0
    for seed in range(6):
        rng = np.random.default_rng(200 + seed)
        hp, _, prices = _small_crypto_problem(rng)
        specs = _utilities(rng, hp.n_tokens, prices)
        out = _host_solve(hp, specs)
        for p, u in enumerate(specs):
            r = XK.oracle_solve(hp, u, tol=1e-9)
            st = out["stats"][p]
            assert r.status == "optimal" and int(st[7]) == 0, (seed, p, r.status, st[7])
            scale = max(abs(r.dual_value), 1e-300)
            assert abs(st[0] - r.value) <= 1e-9 * scale and abs(st[1] - r.dual_value) <= 1e-9 * scale
            np.testing.assert_allclose(out["nu"][p], r.nu, rtol=1e-6)
            same += (int(st[5]), int(st[6])) == (r.iters, r.evals)
            total += 1
            XK.certify(hp, u, _as_result(hp, out, p), 1e-9)
    assert same >= total - 3, (same, total)


def test_oracle_unit_covariance():
    """rescale token j by s: reserves x s, price scales p_j / s, a_j s, c_j / s  =>  psi_j s, same value"""
    rng = np.random.default_rng(7)
    hp, d, prices = _small_crypto_problem(rng)
    n = hp.n_tokens
    for u in _utilities(rng, n, prices):
        r0 = XK.oracle_solve(hp, u, tol=1e-9)
        s = np.exp(rng.normal(0, 0.5, n))
        R = [list(np.asarray(x) * s[l]) for x, l in zip(d["reserves"], d["local_indices"])]
        W = [w if k != "cryptoswap" else (w[0], w[1], w[2] / s[l[0]], w[3] / s[l[1]])
             for w, k, l in zip(d["weights"], d["kinds"], d["local_indices"])]
        hp2 = HostPools.from_lists(n, d["local_indices"], R, d["fees"], d["kinds"], W)
        u2 = XK.Utility(u.c / s, u.a * s, u.eq, u.pinned)
        r1 = XK.oracle_solve(hp2, u2, tol=1e-9)
        # (the arbitrage problem of this seed, worth 2e-3 against pools of ~1e2, stops at max_iter in both units with
        # the same value: the rescaling must not change that either)
        assert r0.status == r1.status
        gross = sum(np.abs(x).sum() for x in r0.deltas) + sum(np.abs(x).sum() for x in r0.lambdas)
        np.testing.assert_allclose(r1.psi / s, r0.psi, rtol=1e-8, atol=1e-9 * gross / s.min())
        assert abs(r1.value - r0.value) <= 1e-9 * abs(r0.dual_value)


def test_rejections():
    li, fees = [[0, 1]], [0.997]
    ok = dict(reserves=[[10.0, 12.0]], weights=[(10.0, 1.45e-4, 1.0, 0.8)])
    hp = HostPools.from_lists(2, li, ok["reserves"], fees, ["cryptoswap"], ok["weights"])
    hp.validate()
    bad_w = [(0.0, 1e-4, 1, 1), (2e4, 1e-4, 1, 1), (np.nan, 1e-4, 1, 1), (10, 1e-7, 1, 1), (10, 0.2, 1, 1),
             (10, np.inf, 1, 1), (10, 1e-4, 0.0, 1), (10, 1e-4, 1, -1), (10, 1e-4, 1, np.nan), (10, 1e-4, 1), None]
    for w in bad_w:
        with pytest.raises(ValueError):
            HostPools.from_lists(2, li, ok["reserves"], fees, ["cryptoswap"], [w])
    for R in ([0.0, 1.0], [-1.0, 2.0], [np.nan, 1.0], [1.0, np.inf]):
        with pytest.raises(ValueError):
            HostPools.from_lists(2, li, [R], fees, ["cryptoswap"], ok["weights"])
    with pytest.raises(ValueError):                              # arity 3
        HostPools.from_lists(3, [[0, 1, 2]], [[1.0, 2.0, 3.0]], fees, ["cryptoswap"], [(10, 1e-4, 1, 1)])
    bad = HostPools(2, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind, hp.amp, cgam=np.array([0.0]))
    with pytest.raises(ValueError):                              # G = 0 given directly in CSR form
        bad.validate()
    args = (hp.pool_ptr, hp.kind, hp.weights, [0])
    for kw in (dict(reserves=np.array([[0.0, 1.0]])), dict(amp=[0.0]), dict(amp=[1e5]), dict(curve_gamma=[1e-7]),
               dict(curve_gamma=[0.5]), dict(rates=[[1.0, -1.0]]), dict(rates=[[1.0, 2.0, 3.0]]),
               dict(curve_gamma=[1e-4, 1e-4]), dict(prices=[1.0])):
        with pytest.raises(ValueError):
            check_pool_update(*args, **kw)
    ss = HostPools.from_lists(2, li, ok["reserves"], fees, ["stableswap"], [(100.0, 1.0, 1.0)])
    with pytest.raises(ValueError):                              # curve_gamma on a StableSwap pool
        check_pool_update(ss.pool_ptr, ss.kind, ss.weights, [0], curve_gamma=[1e-4])
    u = check_pool_update(*args, amp=[20.0], curve_gamma=[2e-3], rates=[[1.0, 0.9]])
    assert u.amp[0] == 20.0 and u.curve_gamma[0] == 2e-3 and np.array_equal(u.rates, [1.0, 0.9])


def test_xp_certificate_covers_cryptoswap_pools():
    """the certificate rejects an answer whose cryptoswap trades over-pay the pool and accepts the oracle's"""
    rng = np.random.default_rng(9)
    hp, _, prices = _small_crypto_problem(rng)
    u = _utilities(rng, hp.n_tokens, prices)[0]
    r = XK.oracle_solve(hp, u, tol=1e-10)
    XK.certify(hp, u, r, 1e-10)
    cs = int(np.nonzero(hp.kind == KIND_CRYPTOSWAP_HOST)[0][0])
    bad = [x.copy() for x in r.lambdas]
    bad[cs] = bad[cs] + 1e-6 * hp.reserves[hp.pool_ptr[cs]:hp.pool_ptr[cs + 1]]
    rb = types.SimpleNamespace(**{**r.__dict__, "lambdas": bad})
    rep = XK.certify(hp, u, rb, 1e-10, check=False)
    assert any("pool-feasible" in f for f in rep["fails"])


def test_twocrypto_conversion():
    """instances.twocrypto_pool: A = A() / (A_MULTIPLIER 2^2), G = gamma() / 1e18, price scales from price_scale() and
    the precisions, whole-token reserves, and the dynamic fee at the state; the converted pool's D (decimal) matches"""
    getcontext().prec = 50
    A_raw, gamma_raw, ps = 400000, 145000000000000, 2500 * 10 ** 18
    prec = (1, 10 ** 12)                                      # an 18-decimal coin 0 and a 6-decimal coin 1
    bal = (1000 * 10 ** 18, 2_400_000 * 10 ** 6)
    w, R, g = I.twocrypto_pool(A_raw, gamma_raw, ps, prec, bal, 26_000_000, 45_000_000, 230_000_000_000_000)
    assert w == (10.0, 1.45e-4, 1.0, 2500.0) and R == (1000.0, 2_400_000.0)
    y0, y1 = Decimal(1000), Decimal(2_400_000) * 2500
    K0 = 4 * y0 * y1 / (y0 + y1) ** 2
    f = Decimal("0.00023") / (Decimal("0.00023") + 1 - K0)
    fee = (Decimal("0.0026") * f + Decimal("0.0045") * (1 - f))
    assert abs(Decimal(1 - g) - fee) <= Decimal(1e-15)
    hp = HostPools.from_lists(2, [[0, 1]], [list(R)], [g], ["cryptoswap"], [w])
    ref = _dec_D(Decimal(R[0]) * Decimal(w[2]), Decimal(R[1]) * Decimal(w[3]), w[0], w[1])
    assert abs(Decimal(hp.inv[0]) - ref) / ref <= Decimal(4e-16)


def test_market_generator():
    hp, p = I.synth_crypto_market(3000, 40, seed=1)
    hp.validate()
    cs = hp.kind == KIND_CRYPTOSWAP_HOST
    assert 0.35 < cs.mean() < 0.45 and np.all(hp.inv[cs] > 0) and np.all(hp.cgam[~cs] == 0)
    for k in (0, 1, 3, 4, 6):
        assert (hp.kind == k).any(), k
    # near and far from the peg: the pool's price scale against the market price
    f = hp.pool_ptr[np.nonzero(cs)[0]]
    off = np.abs(np.log(hp.weights[f + 1] / hp.weights[f] * p[hp.tok_idx[f]] / p[hp.tok_idx[f + 1]]))
    assert 0.3 < (off > 0.1).mean() < 0.7


# ====================================================================================================== GPU
gpu = pytest.mark.gpu


def _bucket_pools(m=1_000_000, seed=21):
    """m random pools (random_pools: half near their peg, half far) on random pairs of 64 tokens; prices ~ exp(N(0, 0.3)).
    Returns (HostPools, nu, sample of pool ids the reference checks)."""
    rng = np.random.default_rng(seed)
    R0, p0, A, G, _, g, _ = random_pools(m, seed)
    k = R0[:, 0] * p0[:, 0] / (R0[:, 1] * p0[:, 1])                 # the scaled balance ratio (near or far from 1)
    n0 = 64
    toks = np.stack([rng.integers(0, n0, m), np.zeros(m, int)], 1)
    toks[:, 1] = (toks[:, 0] + rng.integers(1, n0, m)) % n0
    nu = np.exp(rng.normal(0, 0.3, n0))
    # price scales near the token prices, so a pool near its peg also trades near it
    p = np.stack([nu[toks[:, 0]], nu[toks[:, 1]]], 1) * np.exp(rng.normal(0, 0.02, (m, 2)))
    R = np.empty((m, 2))
    R[:, 1] = np.exp(rng.normal(8, 2, m)) / p[:, 1]
    R[:, 0] = k * R[:, 1] * p[:, 1] / p[:, 0]
    hp = crypto_hp(R, p, A, G, g, toks, n0)
    return hp, nu, np.sort(rng.choice(m, 50_000, replace=False))


@gpu
@pytest.mark.parametrize("trades,hess", [(False, False), (True, False), (False, True), (True, True)])
def test_kernel_matches_xp_reference(trades, hess):
    import torch
    hp, nu, smp = _bucket_pools()
    st = cf.PoolStore(hp)
    assert len(st.buckets) == 1 and st.buckets[0].kind == _lib.KIND_CRYPTOSWAP
    nu_d = torch.as_tensor(nu, dtype=torch.float64, device="cuda")
    acc = st.evaluate(nu_d, 0.0, trades=True, hess=True).cpu().numpy()
    b = st.buckets[0]
    m = b.m
    Dk = b.delta[:, :m].cpu().numpy().T; Lk = b.lam[:, :m].cpu().numpy().T; hk = b.hcoef[:m].cpu().numpy()
    tok = hp.tok_idx.reshape(-1, 2)
    # the instance under test against the full instance: identical per-pool arithmetic, so identical psi and arb bits
    # up to the order of the atomic sums
    acc2 = st.evaluate(nu_d, 0.0, trades=trades, hess=hess).cpu().numpy()
    y = Lk - Dk
    psi = np.zeros(hp.n_tokens); np.add.at(psi, tok.ravel(), y.ravel())
    gross = np.zeros(hp.n_tokens); np.add.at(gross, tok.ravel(), np.abs(y).ravel())
    assert np.all(np.abs(acc2[:-1] - psi) <= 1e-12 * gross + 1e-300)
    assert np.all(np.abs(acc[:-1] - psi) <= 1e-12 * gross + 1e-300)
    arb = float((nu[tok] * y).sum())
    assert abs(acc2[-1] - arb) <= 1e-12 * float((nu[tok] * np.abs(y)).sum())
    # the sample against the longdouble reference
    R = hp.reserves.reshape(-1, 2)[smp]; p = hp.weights.reshape(-1, 2)[smp]
    nv = nu[tok[smp]]
    Dx, Lx, hx, hrel = _check_against_xp(Dk[smp], Lk[smp], hk[smp], R, p, hp.amp[smp], hp.cgam[smp], hp.inv[smp],
                                         hp.gamma[smp], nv)
    ua = p * R / hp.inv[smp][:, None]
    near = np.abs(np.log(ua[:, 0] / ua[:, 1])) < 1e-2
    print(f"XP sample={len(smp)} trading={(hx > 0).sum()} near-peg={near.sum()} hc rel max={hrel:.2e}")
    assert near.sum() > 10_000 and (~near).sum() > 10_000 and hrel <= 1e-6
    if hess:
        # the Hessian kernels take the generic pair branch: numpy from the kernel's own hcoef
        rng = np.random.default_rng(0)
        vt = rng.standard_normal(hp.n_tokens)
        c_ = hk * (vt[tok[:, 0]] - vt[tok[:, 1]])
        yv = np.zeros(hp.n_tokens); np.add.at(yv, tok[:, 0], c_); np.add.at(yv, tok[:, 1], -c_)
        yk = st.hvp(torch.as_tensor(vt, dtype=torch.float64, device="cuda")).cpu().numpy()
        sc = np.zeros(hp.n_tokens); np.add.at(sc, tok.ravel(), np.repeat(np.abs(c_), 2))
        assert np.all(np.abs(yk - yv) <= 1e-12 * sc + 1e-300)
        dg = np.zeros(hp.n_tokens); np.add.at(dg, tok.ravel(), np.repeat(hk, 2))
        np.testing.assert_allclose(st.hess_diag().cpu().numpy(), dg, rtol=1e-12)
        Hd = np.zeros((hp.n_tokens, hp.n_tokens))
        np.add.at(Hd, (tok[:, 0], tok[:, 0]), hk); np.add.at(Hd, (tok[:, 1], tok[:, 1]), hk)
        np.add.at(Hd, (tok[:, 0], tok[:, 1]), -hk); np.add.at(Hd, (tok[:, 1], tok[:, 0]), -hk)
        np.testing.assert_allclose(st.hess_dense().cpu().numpy(), Hd, rtol=1e-12, atol=1e-12 * np.abs(Hd).max())


def _specs(n, prices, rng):
    basket = np.zeros(n)
    for j in rng.choice(np.arange(1, n), 8, replace=False):
        basket[j] = float(np.exp(rng.normal(1, 1)) * 100 / prices[j])
    return [cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(n))), cf.Liquidate(0, basket),
            cf.Swap(1, 3, 5e3 / prices[1])]


@gpu
def test_mixed_market_every_utility_certifies():
    hp, prices = I.synth_crypto_market(60_000, 300, seed=4)
    store = cf.PoolStore(hp)
    assert _lib.KIND_CRYPTOSWAP in [int(b.kind) for b in store.buckets]
    rng = np.random.default_rng(1)
    for u in _specs(hp.n_tokens, prices, rng):
        r = cf.solve_pools(hp, u, tol=1e-8, store=store)
        assert r.status == "optimal", r.status
        assert r.info.history, "the python outer loop (solver.py) ran: no native solver covers cryptoswap buckets"
        rep = XK.certify(hp, u.spec(hp.n_tokens), r, 1e-8)
        print(f"CERT {type(u).__name__} iters={r.iters} evals={r.evals} hvps={r.hvps} "
              + " ".join(f"{k}={v[0]:.2e}/{v[1]:.2e}" for k, v in rep.items() if isinstance(v, tuple)))


@gpu
def test_batch_solver_sweep_and_many():
    import torch
    from cfmm_routing_code_b200 import batch as B
    rng = np.random.default_rng(3)
    probs = [_small_crypto_problem(rng) for _ in range(6)]
    for lanes in (1, 32):
        for hp, d, prices in probs:
            us = [cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(hp.n_tokens))),
                  cf.Swap(0, 1, 2.0 / prices[0]),
                  cf.Liquidate(0, np.r_[0.0, 5.0 / prices[1], 3.0 / prices[2], np.zeros(hp.n_tokens - 3)])]
            store = B.CsrStore(hp)
            assert store.has_crypto
            c, a, fl, nu = B.pack_utilities(us, hp.n_tokens)
            up = lambda x: torch.as_tensor(x, device="cuda")
            nu_d = up(nu)
            psi, stats, dl, lm = B.solve_batch_device(store, up(c), up(a), up(fl), nu_d, tol=1e-9, lanes=lanes)
            stats = stats.cpu().numpy(); psi = psi.cpu().numpy(); nu_h = nu_d.cpu().numpy()
            dl, lm = dl.cpu().numpy(), lm.cpu().numpy()
            ptr = hp.pool_ptr
            for p, u in enumerate(us):
                assert int(stats[p][7]) == 0, (lanes, p, stats[p])
                res = types.SimpleNamespace(value=stats[p][0], dual_value=stats[p][1], psi=psi[p], nu=nu_h[p],
                                            deltas=[dl[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                            lambdas=[lm[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])
                XK.certify(hp, u.spec(hp.n_tokens), res, 1e-9)
                rp = cf.solve_pools(hp, u, tol=1e-9, method="pools")
                assert rp.status == "optimal"
                assert abs(rp.value - stats[p][0]) <= 1e-8 * abs(rp.dual_value)
    hp, d, prices = probs[0]
    sw = [cf.Swap(0, 1, t / prices[0]) for t in np.linspace(0.1, 20.0, 12)]
    rb = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], sw, batched=True)
    ru = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], sw, batched=False)
    for x, y in zip(rb, ru):
        assert x.status == y.status == "optimal"
        assert abs(x.value - y.value) <= 1e-7 * max(abs(x.dual_value), 1.0)
    many = cf.solve_many([(hp, cf.Swap(0, 1, 2.0 / pr[0])) for hp, _, pr in probs])
    assert all(r.status == "optimal" for r in many)
    for (hp, _, pr), r in zip(probs, many):
        XK.certify(hp, cf.Swap(0, 1, 2.0 / pr[0]).spec(hp.n_tokens), r, 1e-8)


def _bucket_tensors(st):
    out = []
    for b in st.buckets:
        if getattr(b, "blocked", False):
            out.append((b.r0, b.r1, b.gamma_inv))
        else:
            out.append(tuple(getattr(b, t) for t in ("reserves", "gamma", "weights", "logrw")))
    return out


@gpu
@pytest.mark.parametrize("world", [1, 2, 3])
def test_update_pools_equals_a_fresh_store_and_resolves(world):
    import torch
    hp, prices = I.synth_crypto_market(40_000, 200, seed=8)
    stores = [cf.PoolStore(hp, rank=r, world=world) for r in range(world)]
    u = cf.Arbitrage(prices)
    r0 = cf.solve_pools(hp, u, tol=1e-8, store=stores[0]) if world == 1 else None
    rng = np.random.default_rng(2)
    cs = np.nonzero(hp.kind == KIND_CRYPTOSWAP_HOST)[0]
    ids = np.sort(rng.choice(cs, 2000, replace=False))
    newR = hp.reserves.reshape(-1, 2)[(hp.pool_ptr[ids] // 2)] * np.exp(0.05 * rng.standard_normal((len(ids), 2))) \
        if int(hp.pool_ptr[-1]) == 2 * hp.m else np.stack([hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i] + 2] for i in ids]) * \
        np.exp(0.05 * rng.standard_normal((len(ids), 2)))
    newg = np.full(len(ids), 0.9971)
    f = hp.pool_ptr[ids]
    newp = np.stack([hp.weights[f], hp.weights[f + 1] * np.exp(0.01 * rng.standard_normal(len(ids)))], 1)
    newA = hp.amp[ids] * 1.01
    newG = np.minimum(hp.cgam[ids] * 1.02, CRYPTO_GAMMA_RANGE[1])
    half = len(ids) // 2
    for st in stores:                              # two blocks: reserves and fees, then a repeg and a ramp
        st.update_pools(ids, reserves=newR, fees=newg)
        st.update_pools(ids[:half], rates=newp[:half], amp=newA[:half], curve_gamma=newG[:half])
    R2, g2, W2, A2, G2 = hp.reserves.copy(), hp.gamma.copy(), hp.weights.copy(), hp.amp.copy(), hp.cgam.copy()
    for k, i in enumerate(ids):
        R2[f[k]:f[k] + 2] = newR[k]
    g2[ids] = newg
    for k, i in enumerate(ids[:half]):
        W2[f[k]:f[k] + 2] = newp[k]
    A2[ids[:half]] = newA[:half]; G2[ids[:half]] = newG[:half]
    hp2 = HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, R2, W2, g2, hp.kind, A2, None, hp.lad_ptr, hp.lad_rec,
                    hp.lad_sc, G2)
    assert np.array_equal(hp.reserves, hp.reserves) and hp.inv is not hp2.inv
    for r, st in enumerate(stores):
        fresh = cf.PoolStore(hp2, rank=r, world=world)
        for a, b in zip(_bucket_tensors(st), _bucket_tensors(fresh)):
            for x, y in zip(a, b):
                assert (x is None) == (y is None) and (x is None or torch.equal(x, y))
    if world == 1:
        r1 = cf.solve_pools(hp2, u, tol=1e-8, store=stores[0], nu0=r0.nu)
        assert r1.status == "optimal"
        XK.certify(hp2, u.spec(hp.n_tokens), r1, 1e-8)


@gpu
def test_solve_pools_unit_covariance():
    rng = np.random.default_rng(6)
    hp, d, prices = _small_crypto_problem(rng)
    n = hp.n_tokens
    s = np.exp(rng.normal(0, 1, n))
    R = [list(np.asarray(x) * s[l]) for x, l in zip(d["reserves"], d["local_indices"])]
    W = [w if k != "cryptoswap" else (w[0], w[1], w[2] / s[l[0]], w[3] / s[l[1]])
         for w, k, l in zip(d["weights"], d["kinds"], d["local_indices"])]
    hp2 = HostPools.from_lists(n, d["local_indices"], R, d["fees"], d["kinds"], W)
    for u in _utilities(rng, n, prices):
        r0 = cf.solve_pools(hp, cf.LinearUtility(u.c, u.a, u.eq, u.pinned), tol=1e-10, method="pools")
        r1 = cf.solve_pools(hp2, cf.LinearUtility(u.c / s, u.a * s, u.eq, u.pinned), tol=1e-10, method="pools")
        assert r0.status == r1.status == "optimal"
        np.testing.assert_allclose(r1.psi / s, r0.psi, rtol=1e-7, atol=1e-9 * np.abs(r0.psi).max())
        assert abs(r1.value - r0.value) <= 1e-9 * abs(r0.dual_value)


@gpu
def test_c_abi_return_codes():
    import torch
    lib = _lib.load()
    buf = torch.ones(8 * 1024, dtype=torch.float64, device="cuda")
    idx = torch.zeros(2 * 1024, dtype=torch.int32, device="cuda")
    nu = torch.ones(4, dtype=torch.float64, device="cuda")
    acc = torch.zeros(5, dtype=torch.float64, device="cuda")
    p = buf.data_ptr()

    def ev(arity, w, lr):
        b = _lib.Bucket(_lib.KIND_CRYPTOSWAP, arity, 100, 1024, p, idx.data_ptr(), p, w, lr, None)
        return lib.cfmm_arb_eval(C.byref(b), 4, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc.data_ptr() + 32, None, None)
    assert ev(3, p, p) == -2                  # CFMM_E_KIND
    assert ev(2, None, p) == -1               # CFMM_E_NULL: price scales
    assert ev(2, p, None) == -1               # CFMM_E_NULL: (A, G, D)
    assert ev(2, p, p) == 0
    b = _lib.Bucket(_lib.KIND_CRYPTOSWAP, 3, 100, 1024, p, idx.data_ptr(), p, p, p, None)
    hc = torch.zeros(1024, dtype=torch.float64, device="cuda")
    assert lib.cfmm_hvp(C.byref(b), 4, hc.data_ptr(), None, nu.data_ptr(), acc.data_ptr(), None) == -2
    b = _lib.Bucket(_lib.KIND_CRYPTOSWAP, 2, 100, 1024, p, idx.data_ptr(), p, p, p, None)
    assert lib.cfmm_hvp(C.byref(b), 4, hc.data_ptr(), None, nu.data_ptr(), acc.data_ptr(), None) == 0
    torch.cuda.synchronize()
