"""Three-coin cryptoswap (Curve v2, tricrypto-ng) pools, device kind 9: the invariant, its concavity over the accepted
(A, gamma) domain, the per-pool optimal trade and its Hessian edge weights, the per-thread solver, the pool-parallel
kernels and the solve paths.

CPU: the invariant against 50-digit decimal bisection, including far corners; the Hessian of D on the plane sum(v) = 0
in 50-digit decimal at the corners and midpoints of the accepted domain; cfmm_small::cryptoswap3 compiled for the host:
its post-trade point on the curve (decimal), its optimality against a brute-force maximisation over the two-dimensional
curve (mpmath), the exact no-trade band, one idle coin, the A -> 0 geometric-mean limit, a dust-sized balance, the edge
weights against finite differences (PSD, Hs 1 = 0), the host build and near-peg pools against the longdouble reference
tests/xp_tricrypto.py; the tricrypto solver instance certified by that reference's certificate; rejections, status 3
from the other instances, the contract conversion and unit covariance.
GPU (H100): cfmm_arb_eval's four instances on 1M pools against the host build and a sample against the reference, the
HVP, diagonal and dense Hessian against a torch assembly from the edge weights, certified solves through solve_pools,
solve_batch, solve_sweep and solve_many, in-place updates (one store and rank stores) and the C ABI's return codes.
"""
import ctypes as C
import functools
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
                                          check_pool_update, tricrypto_invariant)
import small_host
import xp_tricrypto as XT

HERE = os.path.dirname(os.path.abspath(__file__))
FEES = [1.0, 0.9995, 0.997, 0.99]
EDGES = [(0, 1), (0, 2), (1, 2)]
gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------ helpers
def _dec_F(y, A, G, D):
    S, P = y[0] + y[1] + y[2], y[0] * y[1] * y[2]
    K0 = 27 * P / (D * D * D)
    K = A * K0 * G * G / ((G + 1 - K0) ** 2)
    return K * D * D * S + P - K * D * D * D - (D / 3) ** 3


def _dec_D(y, A, G, iters=190):
    """the invariant by bisection on [3 P^(1/3), S] in decimal (F > 0 below the root)"""
    y = [v if isinstance(v, Decimal) else Decimal(float(v)) for v in y]
    A, G = Decimal(float(A)), Decimal(float(G))
    lo = 3 * (y[0] * y[1] * y[2]) ** (Decimal(1) / 3)
    hi = y[0] + y[1] + y[2]
    for _ in range(iters):
        mid = (lo + hi) / 2
        lo, hi = (mid, hi) if _dec_F(y, A, G, mid) > 0 else (lo, mid)
    return (lo + hi) / 2


_HOST = None


def _host():
    """tests/host_harness/tricrypto_host.cpp: cfmm_small::cryptoswap3 and the tricrypto solver instance, host build"""
    global _HOST
    if _HOST is None:
        src = os.path.join(HERE, "host_harness", "tricrypto_host.cpp")
        hdr = os.path.join(HERE, "..", "cfmm_routing_code_b200", "csrc", "cfmm_small.cuh")
        lib = os.path.join(HERE, "_build", "libtricrypto_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src],
                           check=True)
        _HOST = C.CDLL(lib)
    return _HOST


def host_pools(R, c, A, G, g, nu):
    m = len(g)
    arr = [np.ascontiguousarray(x, np.float64) for x in (R, c, A, G, g, nu)]
    D, L, w = np.zeros((m, 3)), np.zeros((m, 3)), np.zeros((m, 3))
    mask = np.zeros(m, np.uint32)
    p_ = lambda x: x.ctypes.data_as(C.c_void_p)
    _host().tricrypto_host_pools(C.c_longlong(m), *[p_(x) for x in arr], p_(D), p_(L), p_(w), p_(mask))
    return D, L, w, mask


def edges_to_hs(w):
    """(m, 3) edge weights -> (m, 3, 3) blocks sum_{a<b} w_ab (e_a - e_b)(e_a - e_b)'"""
    H = np.zeros((len(w), 3, 3))
    for q, (a, b) in enumerate(EDGES):
        H[:, a, a] += w[:, q]; H[:, b, b] += w[:, q]
        H[:, a, b] -= w[:, q]; H[:, b, a] -= w[:, q]
    return H


def random_pools(m, seed, far=0.5):
    """m pools over the accepted domain, some near their peg (balances within 1e-9 .. 1e-2 of the scale), the rest far
    from it (up to ~1e4x per coin); prices near the pool's scale and some far from it"""
    rng = np.random.default_rng(seed)
    A = np.exp(rng.uniform(np.log(CRYPTO_A_RANGE[0]), np.log(CRYPTO_A_RANGE[1]), m))
    G = np.exp(rng.uniform(np.log(CRYPTO_GAMMA_RANGE[0]), np.log(CRYPTO_GAMMA_RANGE[1]), m))
    p = np.exp(rng.normal(0, 1, (m, 3)))
    V = np.exp(rng.normal(8, 2, m))
    isfar = rng.random(m) < far
    k = np.where(isfar[:, None], np.exp(rng.uniform(-4.5, 4.5, (m, 3))),
                 1 + rng.choice([-1, 1], (m, 3)) * np.exp(rng.uniform(np.log(1e-9), np.log(1e-2), (m, 3))))
    R = V[:, None] * k / p
    g = np.array(FEES)[rng.integers(0, 4, m)]
    Dv = tricrypto_invariant(R, p, A, G)
    dev = np.where(rng.random((m, 3)) < 0.7, rng.normal(0, 0.01, (m, 3)), rng.normal(0, 0.5, (m, 3)))
    nu = p * np.exp(dev) * np.exp(rng.normal(0, 1, m))[:, None]
    return R, p, A, G, Dv, g, nu


def tri_hp(R, p, A, G, g, toks=None, n=None):
    m = len(g)
    toks = np.tile([0, 1, 2], (m, 1)) if toks is None else toks
    n = int(toks.max()) + 1 if n is None else n
    return HostPools(n, np.arange(0, 3 * m + 1, 3, dtype=np.int64), np.ascontiguousarray(toks, np.int32).ravel(),
                     np.ascontiguousarray(R, np.float64).ravel(), np.ascontiguousarray(p, np.float64).ravel(),
                     np.asarray(g, np.float64), np.full(m, KIND_CRYPTOSWAP_HOST, np.uint8), np.asarray(A, np.float64),
                     cgam=np.asarray(G, np.float64))


def _value(nu, D, L):
    return (nu * (L - D)).sum(-1)


U = 2.0 ** -53
COND = 256.0


def flow_bound(Hs, g, nu, R, rel=1e-12):
    """per pool and coin: rel gross + 8 u max(R) / gamma + COND u sum_b |Hs_jb| / nu_j.  A trading pool's answer solves
    its conditions in log prices with an absolute error of a few u (the inner and outer roots), which moves flow j by
    ~ sum_b |Hs_jb| / nu_j per unit of that error; as for the two-coin bound of tests/test_cryptoswap.py"""
    return (rel * np.abs(Hs).sum((1, 2))[:, None] / nu + 8 * U * R.max(1)[:, None] / g[:, None] +
            COND * U * np.abs(Hs).sum(2) / nu)


def _check_against_xp(D, L, w, mask, R, p, A, G, Dv, g, nu):
    """the first len(R) pools of (D, L, w, mask) against xp_tricrypto: flows within flow_bound (gross flows included),
    the same traded set except where the reference's flows are within the bound of 0; returns the worst relative
    edge-weight difference against the reference's finite differences on 200 of them"""
    n = len(R)
    D, L, w, mask = D[:n], L[:n], w[:n], mask[:n]
    c = XT.LD(p) / XT.LD(Dv)[:, None]
    Dx, Lx, mx = XT.tricrypto_response(R, c, A, G, g, nu)
    Hs = edges_to_hs(w)
    gross = (np.abs(Dx) + np.abs(Lx)).sum(1).astype(float)[:, None]
    bound = flow_bound(Hs, g, nu, R) + 1e-12 * gross
    err = np.maximum(np.abs(D - Dx.astype(float)), np.abs(L - Lx.astype(float)))
    assert np.all(err <= bound), float((err / bound).max())
    mism = mask != mx
    assert np.all(gross[mism, 0] <= 3 * bound[mism].max(1)), int(mism.sum())
    k = min(n, 200)
    wx, mx2, same = XT.edges_fd(R[:k], c[:k], A[:k], G[:k], g[:k], nu[:k])
    ok = same & (mx2 != 0) & (mx2 == mask[:k])
    sw = np.abs(wx.astype(float)).max(1) + 1e-300
    rel = (np.abs(w[:k] - wx.astype(float)).max(1) / sw)[ok]
    return float(rel.max()) if ok.any() else 0.0


def test_host_matches_xp_reference():
    """cfmm_small::cryptoswap3 (host build) against the longdouble reference over the accepted domain, near and far
    from the peg: flows within the flow bound, edge weights within 1e-6 of the reference's finite differences"""
    R, p, A, G, Dv, g, nu = random_pools(1200, seed=6)
    D, L, w, mask = host_pools(R, p / Dv[:, None], A, G, g, nu)
    assert (mask != 0).sum() > 600
    assert _check_against_xp(D, L, w, mask, R, p, A, G, Dv, g, nu) <= 1e-6


# ====================================================================================================== CPU
def test_invariant_matches_decimal():
    getcontext().prec = 50
    worst = 0.0
    rng = np.random.default_rng(0)
    for A in (CRYPTO_A_RANGE[0], 0.27, 6.3, 100.0, CRYPTO_A_RANGE[1]):
        for G in (CRYPTO_GAMMA_RANGE[0], 1.45e-4, 2e-2, CRYPTO_GAMMA_RANGE[1]):
            for t in ((1, 1, 1), (1 + 1e-9, 1, 1 - 1e-9), (1.01, 0.99, 1), (3, 1, 0.5), (1e5, 1, 1e-5), (1e-5, 1e5, 1)):
                s = float(np.exp(rng.normal(0, 20)))
                y = np.array(t, float) * s
                d = float(tricrypto_invariant(y[None], np.ones((1, 3)), [A], [G])[0])
                ref = _dec_D(y, A, G)
                worst = max(worst, float(abs(Decimal(d) - ref) / ref))
    assert worst <= 4e-15, worst


def _dec_hess_plane(t, A, G):
    """the Hessian of D(y) at y = t restricted to sum(v) = 0 (basis (1, -1, 0), (1, 1, -2) / sqrt 3), central second
    differences in decimal with a relative step of 1e-12"""
    y = [Decimal(float(v)) for v in t]
    h = min(y) * Decimal(10) ** -12
    b1 = [Decimal(1), Decimal(-1), Decimal(0)]
    b2 = [Decimal(1) / Decimal(3).sqrt(), Decimal(1) / Decimal(3).sqrt(), -2 / Decimal(3).sqrt()]
    D = lambda v: _dec_D([y[j] + v[j] for j in range(3)], A, G, 160)
    sc = lambda a, v: [a * x for x in v]
    ad = lambda u, v: [x + z for x, z in zip(u, v)]
    d0 = D([0, 0, 0])
    h11 = (D(sc(h, b1)) + D(sc(-h, b1)) - 2 * d0) / (h * h)
    h22 = (D(sc(h, b2)) + D(sc(-h, b2)) - 2 * d0) / (h * h)
    h12 = (D(sc(h, ad(b1, b2))) + D(sc(-h, ad(b1, b2))) - D(sc(h, b1)) - D(sc(-h, b1)) - D(sc(h, b2)) -
           D(sc(-h, b2)) + 2 * d0) / (2 * h * h)
    return h11, h12, h22


def test_invariant_is_concave_over_the_accepted_domain():
    """D(y) concave on the plane sum(v) = 0 (the trading set is convex) at the corners and midpoints of the accepted
    (A, gamma) domain, from 1e-9 off the peg out to 1e5:1 in each direction: both eigenvalues of the 2 x 2 plane Hessian
    negative (trace < 0 and determinant > 0), in 50-digit decimal"""
    getcontext().prec = 50
    la, lg = np.log(CRYPTO_A_RANGE), np.log(CRYPTO_GAMMA_RANGE)
    As = np.exp([la[0], la.mean(), la[1]])
    Gs = np.exp([lg[0], lg.mean(), lg[1]])
    pts = [(1 + 1e-9, 1, 1), (1, 1 + 1e-6, 1 - 1e-6), (1.01, 1, 0.99), (2, 1, 1), (1, 0.5, 1), (10, 1, 0.1),
           (1e3, 1, 1), (1, 1, 1e-3), (1e5, 1, 1e-5), (1e-5, 1e5, 1), (1, 1e-5, 1e5)]
    for A in As:
        for G in Gs:
            for t in pts:
                h11, h12, h22 = _dec_hess_plane(t, A, G)
                assert h11 + h22 < 0 and h11 * h22 - h12 * h12 > 0, (A, G, t, h11, h12, h22)


def _dec_D_of(X, p, A, G):
    return _dec_D([Decimal(float(x)) * Decimal(float(q)) for x, q in zip(X, p)], A, G, 170)


def test_trade_stays_on_the_curve_in_decimal():
    """the post-trade balances R + gamma Delta - Lambda keep D (to a few ulp of the flows), in decimal"""
    getcontext().prec = 50
    R, p, A, G, Dv, g, nu = random_pools(40, seed=1)
    D, L, w, mask = host_pools(R, p / Dv[:, None], A, G, g, nu)
    assert (mask == 7).sum() > 10
    for i in np.nonzero(mask)[0]:
        X = R[i] + g[i] * D[i] - L[i]
        d0 = _dec_D_of(R[i], p[i], A[i], G[i])
        d1 = _dec_D_of(X, p[i], A[i], G[i])
        assert abs(d1 - d0) / d0 <= Decimal(4e-14), (i, float((d1 - d0) / d0))


def _mp_brute(R, p, A, G, g, nu):
    """the best value over the curve D(X) = D(R): X_0, X_1 free (log coordinates, a coarse grid then Nelder-Mead style
    pattern search), X_2 by bisection on the invariant in mpmath (30 digits); no stationarity formula used"""
    mp.mp.dps = 30
    Rm = [mp.mpf(float(v)) for v in R]
    pm = [mp.mpf(float(v)) for v in p]
    A_, G_, g_ = mp.mpf(float(A)), mp.mpf(float(G)), mp.mpf(float(g))
    nm = [mp.mpf(float(v)) for v in nu]

    def F(y, D):
        S, P = y[0] + y[1] + y[2], y[0] * y[1] * y[2]
        K0 = 27 * P / D ** 3
        K = A_ * K0 * G_ ** 2 / (G_ + 1 - K0) ** 2
        return K * D * D * S + P - K * D ** 3 - (D / 3) ** 3

    y0 = [r * q for r, q in zip(Rm, pm)]
    lo, hi = 3 * (y0[0] * y0[1] * y0[2]) ** (mp.mpf(1) / 3), y0[0] + y0[1] + y0[2]
    for _ in range(110):
        mid = (lo + hi) / 2
        lo, hi = (mid, hi) if F(y0, mid) > 0 else (lo, mid)
    D0 = (lo + hi) / 2

    def val(z0, z1):
        x0, x1 = Rm[0] * mp.e ** z0, Rm[1] * mp.e ** z1
        a, b = mp.mpf(-60), mp.mpf(60)                   # log X_2 / R_2; D grows with X_2
        for _ in range(100):
            c = (a + b) / 2
            y = [x0 * pm[0], x1 * pm[1], Rm[2] * mp.e ** c * pm[2]]
            # D(y) >= D0 iff F(y, D0) >= 0 (F > 0 below the root)
            a, b = (a, c) if F(y, D0) >= 0 else (c, b)
        X = [x0, x1, Rm[2] * mp.e ** b]
        return sum((nm[j] * (Rm[j] - X[j]) if X[j] < Rm[j] else -nm[j] * (X[j] - Rm[j]) / g_) for j in range(3))

    best, bz = val(0, 0), (mp.mpf(0), mp.mpf(0))
    step = mp.mpf(1)
    while step > mp.mpf(1e-9):
        moved = False
        for d0, d1 in ((1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (-1, -1), (1, -1), (-1, 1)):
            z = (bz[0] + d0 * step, bz[1] + d1 * step)
            v = val(*z)
            if v > best:
                best, bz, moved = v, z, True
                break
        if not moved:
            step /= 2
    return float(best)


def test_host_matches_brute_force_over_the_curve():
    R, p, A, G, Dv, g, nu = random_pools(8, seed=11)
    D, L, _, mask = host_pools(R, p / Dv[:, None], A, G, g, nu)
    v = _value(nu, D, L)
    for i in range(len(g)):
        b = _mp_brute(R[i], p[i], A[i], G[i], g[i], nu[i])
        sc = float((nu[i] * R[i]).sum())
        # the host value is the optimum: the search cannot beat it, and it finds it to its step's accuracy
        assert b <= v[i] + 1e-12 * sc and b >= v[i] - 1e-9 * sc, (i, b, v[i])


def test_no_trade_band_is_exact_and_one_coin_idle():
    R, p, A, G, Dv, g, _ = random_pools(400, seed=2)
    c = p / Dv[:, None]
    # at the pool's own marginal prices (nu = dPhi/du at u0, pi = nu / c) any fee < 1 leaves it idle: exactly 0
    u0 = c * R
    m0 = 1 - 27 * u0.prod(1)
    K = A * G * G * (1 - m0) / (G + m0) ** 2
    Q = (G + 3 * m0 - 2 * m0 * m0) / (27 * (G + m0))
    nu = c * (K[:, None] + Q[:, None] / u0)
    gg = np.full(len(g), 0.997)
    D, L, w, mask = host_pools(R, c, A, G, gg, nu * np.exp(np.array([4e-4, -4e-4, 0.0])))
    assert np.all(D == 0) and np.all(L == 0) and np.all(w == 0) and np.all(mask == 0)
    # coin 1's price between the others: it may stay idle while 0 and 2 trade
    nu2 = nu * np.array([1.02, 1.0, 0.98])
    D, L, w, mask = host_pools(R, c, A, G, gg, nu2)
    idle = mask != 7
    assert idle.sum() > 50, int(idle.sum())
    for j in range(3):
        off = (mask >> j & 1) == 0
        assert np.all(D[off, j] == 0) and np.all(L[off, j] == 0)
    for q, (a, b) in enumerate(EDGES):
        off = ((mask >> a & 1) == 0) | ((mask >> b & 1) == 0)
        assert np.all(w[off, q] == 0)


def test_small_A_is_the_geometric_mean_pool_on_scaled_balances():
    """A -> 0: K -> 0 and the curve is y0 y1 y2 = (D/3)^3, the equal-weight geometric mean on y = p x: its trade at
    prices mu = nu / p is u_j = clamp(u0_j, t gamma / mu_j, t / mu_j) with prod u = prod u0, t by bisection"""
    rng = np.random.default_rng(3)
    m = 200
    G = np.exp(rng.uniform(np.log(CRYPTO_GAMMA_RANGE[0]), np.log(CRYPTO_GAMMA_RANGE[1]), m))
    p = np.exp(rng.normal(0, 1, (m, 3)))
    R = np.exp(rng.normal(5, 1, (m, 3))) / p
    g = np.array(FEES)[rng.integers(0, 4, m)]
    nu = p * np.exp(rng.normal(0, 0.5, (m, 3)))
    A = np.full(m, 1e-12)                                  # (below the accepted domain: the harness takes any A)
    Dv = tricrypto_invariant(R, p, A, G)
    D, L, _, _ = host_pools(R, p / Dv[:, None], A, G, g, nu)
    y0, mu = R * p, nu / p
    lt_lo, lt_hi = np.full(m, -80.0), np.full(m, 80.0)
    for _ in range(200):
        lt = 0.5 * (lt_lo + lt_hi)
        y = np.clip(y0, np.exp(lt)[:, None] * g[:, None] / mu, np.exp(lt)[:, None] / mu)
        big = np.log(y).sum(1) > np.log(y0).sum(1)
        lt_hi = np.where(big, lt, lt_hi); lt_lo = np.where(big, lt_lo, lt)
    y = np.clip(y0, np.exp(lt)[:, None] * g[:, None] / mu, np.exp(lt)[:, None] / mu)
    X = y / p
    Dg, Lg = np.maximum(X - R, 0) / g[:, None], np.maximum(R - X, 0)
    sc = (np.abs(Dg) + np.abs(Lg)).sum(1)[:, None] + 1e-300
    assert np.all(np.abs(D - Dg) <= 1e-7 * sc) and np.all(np.abs(L - Lg) <= 1e-7 * sc)


def test_dust_balance():
    """one balance 1e-12 of the others (far corner): flows finite, the pool buys the dust coin back, and the curve holds
    to 1e-9 (the fp64 invariant and the 1e12 balance ratio limit it there)"""
    getcontext().prec = 50
    R = np.array([[1e6, 1e6, 1e-6], [1e-6, 2e6, 1e6]])
    p = np.ones((2, 3)); A = np.array([6.3, 0.27]); G = np.array([1e-4, 2e-2]); g = np.array([0.997, 0.9995])
    Dv = tricrypto_invariant(R, p, A, G)
    nu = np.ones((2, 3))
    D, L, w, mask = host_pools(R, p / Dv[:, None], A, G, g, nu)
    assert np.all(np.isfinite(D)) and np.all(np.isfinite(L)) and np.all(np.isfinite(w)) and np.all(mask != 0)
    for i in range(2):
        X = R[i] + g[i] * D[i] - L[i]
        assert _dec_D_of(X, p[i], A[i], G[i]) >= _dec_D_of(R[i], p[i], A[i], G[i]) * (1 - Decimal(1e-9))
        assert _value(nu[i], D[i], L[i]) > 0


def test_edge_weights_match_finite_differences():
    """Hs_ab = nu_a d(Lambda_a - Delta_a) / d log nu_b from the edge weights, against central differences in fp64
    (step 1e-6); Hs is PSD and Hs 1 = 0 to rounding"""
    R, p, A, G, Dv, g, nu = random_pools(600, seed=4)
    c = p / Dv[:, None]
    D0, L0, w, mask = host_pools(R, c, A, G, g, nu)
    Hs = edges_to_hs(w)
    h = 1e-6
    ok = np.ones(len(g), bool)
    for j in range(3):
        up, dn = nu.copy(), nu.copy()
        up[:, j] *= np.exp(h); dn[:, j] *= np.exp(-h)
        Du, Lu, _, mu_ = host_pools(R, c, A, G, g, up)
        Dd, Ld, _, md = host_pools(R, c, A, G, g, dn)
        fd = nu * ((Lu - Du) - (Ld - Dd)) / (2 * h)
        sc = np.abs(Hs).max((1, 2)) + 1e-300
        same = (mu_ == mask) & (md == mask)                      # the traded set does not change within the step
        ok &= ~same | (np.abs(fd - Hs[:, :, j]).max(1) <= 1e-6 * sc)
    trading = mask != 0
    assert trading.sum() > 300 and (ok & trading).sum() >= trading.sum() - 3, (int(trading.sum()), int(ok.sum()))
    ev = np.linalg.eigvalsh(Hs)
    big = np.abs(ev).max(1) + 1e-300
    assert np.all(ev[:, 0] >= -1e-12 * big)
    assert np.all(np.abs(Hs.sum(2)).max(1) <= 1e-12 * big)


def test_near_peg_pools_keep_their_digits():
    """balances within 1e-9 .. 1e-3 of the price scale and gamma down to the accepted minimum: the cancellation-free
    forms keep the fp64 flows within the flow bound of the longdouble reference, the same pool in another coin order
    gives the same flows, and the post-trade point holds D"""
    rng = np.random.default_rng(5)
    m = 2000
    A = np.exp(rng.uniform(np.log(1.0), np.log(CRYPTO_A_RANGE[1]), m))
    G = np.exp(rng.uniform(np.log(CRYPTO_GAMMA_RANGE[0]), np.log(1e-3), m))
    p = np.exp(rng.normal(0, 1, (m, 3)))
    k = 1 + rng.choice([-1, 1], (m, 3)) * np.exp(rng.uniform(np.log(1e-9), np.log(1e-3), (m, 3)))
    R = 1e4 * k / p
    Dv = tricrypto_invariant(R, p, A, G)
    g = np.array([1.0, 0.9999, 0.9995])[rng.integers(0, 3, m)]
    nu = p * np.exp(rng.normal(0, 1e-4, (m, 3)))
    D, L, w, mask = host_pools(R, p / Dv[:, None], A, G, g, nu)
    assert (mask != 0).sum() > m // 3
    perm = [2, 0, 1]
    _check_against_xp(D, L, w, mask, R[:400], p[:400], A[:400], G[:400], Dv[:400], g[:400], nu[:400])
    D2, L2, _, _ = host_pools(R[:, perm], p[:, perm] / Dv[:, None], A, G, g, nu[:, perm])
    gross = (np.abs(D) + np.abs(L)).sum(1)[:, None] + 1e-300
    assert np.all(np.abs(D2 - D[:, perm]) <= 1e-8 * gross) and np.all(np.abs(L2 - L[:, perm]) <= 1e-8 * gross)
    X = R + g[:, None] * D - L
    Dn = tricrypto_invariant(X, p, A, G)
    assert np.all(np.abs(Dn / Dv - 1) <= 1e-13)


# ------------------------------------------------------------------------------------------------ solver instance
def _small_tri_problem(rng):
    """4-6 tokens: a product chain plus a tricrypto pool on tokens 0..2 and one on 1..3"""
    n = int(rng.integers(4, 7))
    prices = np.exp(rng.normal(0, 1, n))
    li, R, f, k, w = [], [], [], [], []
    for j in range(n - 1):
        V = float(np.exp(rng.normal(7, 1)))
        li.append([j, j + 1]); R.append([V / prices[j], V / prices[j + 1]]); f.append(0.997); k.append("product"); w.append(None)
    for toks in ([0, 1, 2], [1, 2, 3]):
        sc = prices[toks] * np.exp(rng.normal(0, 0.05, 3))
        V = float(np.exp(rng.normal(8, 1)))
        li.append(toks); R.append(list(V / sc * np.exp(rng.normal(0, 0.02, 3))))
        f.append(float(rng.choice([0.9995, 0.997]))); k.append("cryptoswap")
        w.append((float(np.exp(rng.uniform(np.log(0.1), np.log(100)))), float(np.exp(rng.uniform(np.log(1e-5), np.log(2e-2)))),
                  *map(float, sc)))
    d = dict(local_indices=li, reserves=R, fees=f, kinds=k, weights=w)
    hp = HostPools.from_lists(n, li, R, f, k, w)
    return hp, d, prices


def _utilities(rng, n, prices):
    basket = np.zeros(n); basket[1] = 5.0 / prices[1]; basket[2] = 3.0 / prices[2]
    return [cf.Arbitrage(prices * np.exp(0.02 * rng.standard_normal(n))), cf.Liquidate(0, basket),
            cf.Swap(1, 0, 2.0 / prices[1])]


def _host_specs(rng, n, prices):
    """the utilities as c, a, eq, pinned vectors (the per-thread solver's host build takes them)"""
    import xp_cryptoswap as XK
    U_ = XK.Utility
    basket = np.zeros(n); basket[1] = 5.0 / prices[1]; basket[2] = 3.0 / prices[2]
    return [U_.arbitrage(prices * np.exp(0.02 * rng.standard_normal(n))), U_.swap(n, 1, 0, 2.0 / prices[1]),
            U_.liquidate(n, 0, basket)]


def _csr_args(hp):
    """the cfmm_csr_pools arrays: cryptoswap w = p / D, logrw = (A, G); three-coin pools kind 9"""
    slot_kind = np.repeat(hp.kind, np.diff(hp.pool_ptr))
    logrw = np.log(np.maximum(hp.reserves, 1e-300) / np.where(slot_kind == 0, hp.weights, 1.0))
    w = np.asarray(hp.weights, np.float64).copy()
    kind = np.array(hp.kind, np.uint8)
    cs = np.nonzero(hp.kind == KIND_CRYPTOSWAP_HOST)[0]
    for i in cs:
        f, e = hp.pool_ptr[i], hp.pool_ptr[i + 1]
        w[f:e] = hp.weights[f:e] / hp.inv[i]
        logrw[f] = hp.amp[i]; logrw[f + 1] = hp.cgam[i]
        if e - f == 3:
            kind[i] = 9
    return [np.ascontiguousarray(x, t) for x, t in ((hp.pool_ptr, np.int64), (hp.tok_idx, np.int32),
                                                    (hp.reserves, np.float64), (w, np.float64),
                                                    (logrw, np.float64), (hp.gamma, np.float64), (kind, np.uint8))]


def _host_solve(hp, specs, tol=1e-9, tri=True):
    n, B, nnz = hp.n_tokens, len(specs), len(hp.tok_idx)
    c = np.stack([u.c for u in specs]).astype(float); a = np.stack([u.a for u in specs]).astype(float)
    fl = np.ascontiguousarray(np.stack([np.asarray(u.eq, np.uint8) | (np.asarray(u.pinned, np.uint8) << 1)
                                        for u in specs]), np.uint8)
    nu = np.ascontiguousarray(np.stack([np.where(u.c > 0, u.c, np.median(u.c[u.c > 0]) if (u.c > 0).any() else 1.0)
                                        for u in specs]))
    keep = _csr_args(hp)
    psi = np.zeros((B, n)); st = np.zeros((B, 8)); d = np.zeros((B, nnz)); l = np.zeros((B, nnz))
    p_ = lambda x: x.ctypes.data_as(C.c_void_p)
    if tri:
        fn = _host().tricrypto_host_solve
        fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 7 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
        fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), tol)
    else:
        small_host.load().small_host_solve(n, hp.m, *[p_(k) for k in keep], B, None, p_(c), p_(a), p_(fl), p_(nu),
                                           p_(psi), p_(st), p_(d), p_(l), nnz, tol, 1)
    return dict(nu=nu, psi=psi, stats=st, delta=d, lam=l)


def _pool_feasible(hp, deltas, lambdas, rel=1e-10):
    """every three-coin pool's post-trade D at least its D before, to rel"""
    for i in np.nonzero((hp.kind == KIND_CRYPTOSWAP_HOST) & (np.diff(hp.pool_ptr) == 3))[0]:
        f = hp.pool_ptr[i]
        X = hp.reserves[f:f + 3] + hp.gamma[i] * np.asarray(deltas[i]) - np.asarray(lambdas[i])
        assert np.all(X > 0)
        Dn = tricrypto_invariant(X[None], hp.weights[f:f + 3][None], [hp.amp[i]], [hp.cgam[i]])[0]
        assert Dn >= hp.inv[i] * (1 - rel), (i, Dn / hp.inv[i] - 1)


def test_existing_solver_instances_reject_tricrypto_pools():
    """the plain instance (and, through the same kind check, every instance before this one) refuses kind 9: status 3"""
    rng = np.random.default_rng(100)
    hp, _, prices = _small_tri_problem(rng)
    out = _host_solve(hp, _host_specs(rng, hp.n_tokens, prices), tri=False)
    assert np.all(out["stats"][:, 7] == 3) and np.all(np.isnan(out["stats"][:, 0]))
    import test_cryptoswap as TC
    keep = _csr_args(hp)
    assert int((keep[6] == 9).sum()) == 2
    # the cryptoswap instance's host build, on the same CSR arrays (kind 9 in the kind bytes)
    n, B = hp.n_tokens, 1
    u = _host_specs(rng, n, prices)[0]
    c = np.ascontiguousarray(u.c[None], float); a = np.ascontiguousarray(u.a[None], float)
    fl = np.zeros((1, n), np.uint8); nu = np.ascontiguousarray(u.c[None], float)
    psi = np.zeros((1, n)); st = np.zeros((1, 8)); d = np.zeros((1, len(hp.tok_idx))); l = np.zeros_like(d)
    p_ = lambda x: x.ctypes.data_as(C.c_void_p)
    fn = TC._host().cryptoswap_host_solve
    fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 7 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
    fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), 1e-9)
    assert st[0, 7] == 3


def test_host_solver_solves_and_is_feasible():
    """the tricrypto instance reaches its tolerance on every utility, its trades keep every pool's invariant, and the
    dual value bounds the primal value"""
    for seed in range(5):
        rng = np.random.default_rng(200 + seed)
        hp, _, prices = _small_tri_problem(rng)
        specs = _host_specs(rng, hp.n_tokens, prices)
        out = _host_solve(hp, specs)
        ptr = hp.pool_ptr
        for p in range(len(specs)):
            st = out["stats"][p]
            assert int(st[7]) == 0, (seed, p, st)
            assert st[1] >= st[0] - 1e-7 * max(abs(st[1]), 1.0)
            assert st[2] <= 1e-6 * max(abs(st[1]), 1.0), st
            _pool_feasible(hp, [out["delta"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                           [out["lam"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])


def test_xp_certificate_covers_tricrypto_pools():
    """the longdouble certificate accepts the host-built tricrypto solver's answers and rejects one whose three-coin
    trades over-pay a pool"""
    for seed in range(3):
        rng = np.random.default_rng(300 + seed)
        hp, _, prices = _small_tri_problem(rng)
        specs = _host_specs(rng, hp.n_tokens, prices)
        out = _host_solve(hp, specs, tol=1e-10)
        for p, u in enumerate(specs):
            r = _as_result(hp, out, p)
            XT.certify(hp, u, r, 1e-9)
    tri = int(np.nonzero(np.diff(hp.pool_ptr) == 3)[0][0])
    bad = [x.copy() for x in r.lambdas]
    bad[tri] = bad[tri] + 1e-6 * hp.reserves[hp.pool_ptr[tri]:hp.pool_ptr[tri + 1]]
    rb = types.SimpleNamespace(**{**r.__dict__, "lambdas": bad})
    rep_ = XT.certify(hp, specs[-1], rb, 1e-9, check=False)
    assert any("pool-feasible" in f for f in rep_["fails"])


def _as_result(hp, out, p):
    ptr = hp.pool_ptr
    return types.SimpleNamespace(value=out["stats"][p][0], dual_value=out["stats"][p][1], psi=out["psi"][p],
                                 nu=out["nu"][p], deltas=[out["delta"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                 lambdas=[out["lam"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])


def test_rejections():
    li = [[0, 1, 2]]
    R = [[1.0, 2.0, 3.0]]
    ok = (10.0, 1e-3, 1.0, 1.0, 1.0)
    HostPools.from_lists(3, li, R, [0.997], ["cryptoswap"], [ok])
    for bad in [(10.0, 1e-3, 1.0, 1.0), (0.0, 1e-3, 1.0, 1.0, 1.0), (1e5, 1e-3, 1.0, 1.0, 1.0),
                (10.0, 0.5, 1.0, 1.0, 1.0), (10.0, 1e-3, -1.0, 1.0, 1.0), (10.0, 1e-3, 1.0, np.inf, 1.0)]:
        with pytest.raises(ValueError):
            HostPools.from_lists(3, li, R, [0.997], ["cryptoswap"], [bad])
    with pytest.raises(ValueError):
        HostPools.from_lists(3, li, [[1.0, 0.0, 3.0]], [0.997], ["cryptoswap"], [ok])
    with pytest.raises(ValueError):                                    # four coins
        HostPools.from_lists(4, [[0, 1, 2, 3]], [[1.0] * 4], [0.997], ["cryptoswap"], [(10.0, 1e-3, 1, 1, 1, 1)])
    hp = HostPools.from_lists(3, li, R, [0.997], ["cryptoswap"], [ok])
    with pytest.raises(ValueError):
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], amp=[0.0])
    with pytest.raises(ValueError):
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], rates=[[1.0, -1.0, 1.0]])
    with pytest.raises(ValueError):
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], reserves=[[1.0, 2.0]])
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], rates=[[1.0, 2.0, 3.0]], curve_gamma=[2e-3])
    assert u.rates.shape == (3,) and u.curve_gamma[0] == 2e-3


def test_tricrypto_conversion():
    """a USDT/WBTC/WETH-like state: A() = 1707629, gamma() = 11809167828997, price scales 1e18-fixed"""
    w, x, g = I.tricrypto_pool(1707629, 11809167828997, (65000 * 10 ** 18, 3400 * 10 ** 18), (10 ** 12, 10 ** 10, 1),
                               (30_000_000 * 10 ** 6, 460 * 10 ** 8, 8800 * 10 ** 18), 3_000_000, 30_000_000,
                               500_000_000_000_000)
    assert w[0] == pytest.approx(1707629 / 270000) and w[1] == pytest.approx(1.1809167828997e-5)
    assert w[2:] == (1.0, 65000.0, 3400.0)
    assert x == pytest.approx((3e7, 460.0, 8800.0))
    assert 1 - 0.003 <= g <= 1 - 0.0003
    hp = HostPools.from_lists(3, [[0, 1, 2]], [list(x)], [g], ["cryptoswap"], [w])
    hp.validate()
    assert np.isfinite(hp.inv[0]) and hp.inv[0] > 0


def test_market_generator_keeps_the_two_coin_market():
    hp, p = I.synth_tricrypto_market(3000, 40, seed=3)
    hp.validate()
    ar = np.diff(hp.pool_ptr)
    tri = (hp.kind == KIND_CRYPTOSWAP_HOST) & (ar == 3)
    assert tri.sum() == 900 and ((hp.kind == KIND_CRYPTOSWAP_HOST) & (ar == 2)).sum() > 0
    a, pa = I.synth_crypto_market(100, 12, seed=5)
    b, pb = I.synth_crypto_market(100, 12, seed=5)
    assert np.array_equal(a.reserves, b.reserves) and np.array_equal(pa, pb)


def test_oracle_unit_covariance_of_the_pool():
    """scaling token j's unit by s_j (reserves * s, price scales / s, prices / s) leaves the trades' values unchanged"""
    R, p, A, G, Dv, g, nu = random_pools(300, seed=9)
    s = np.exp(np.random.default_rng(1).normal(0, 2, (300, 3)))
    D, L, _, mask = host_pools(R, p / Dv[:, None], A, G, g, nu)
    Dv2 = tricrypto_invariant(R * s, p / s, A, G)
    D2, L2, _, mask2 = host_pools(R * s, (p / s) / Dv2[:, None], A, G, g, nu / s)
    gross = (np.abs(D) + np.abs(L)).sum(1)[:, None] + 1e-300
    same = mask == mask2
    assert same.sum() >= 295
    assert np.all(np.abs(D2[same] / s[same] - D[same]) <= 1e-8 * gross[same])
    assert np.all(np.abs(L2[same] / s[same] - L[same]) <= 1e-8 * gross[same])


# ====================================================================================================== GPU
@functools.lru_cache(maxsize=1)
def _bucket_pools(m=1_000_000, seed=21):
    """m random_pools on random triples of 64 tokens, their prices and the host build's answer (shared by the four
    instances)"""
    rng = np.random.default_rng(seed)
    R0, p0, A, G, _, g, _ = random_pools(m, seed)
    n0 = 64
    toks = np.stack([rng.choice(n0, 3, replace=False) for _ in range(1000)])[rng.integers(0, 1000, m)]
    nu = np.exp(rng.normal(0, 0.3, n0))
    k = R0 * p0 / (R0 * p0).sum(1, keepdims=True)                       # scaled balance shares, near or far from 1/3
    p = nu[toks] * np.exp(rng.normal(0, 0.02, (m, 3)))
    R = k * np.exp(rng.normal(8, 2, m))[:, None] / p
    hp = tri_hp(R, p, A, G, g, toks, n0)
    return hp, nu, host_pools(R, p / hp.inv[:, None], A, G, g, nu[toks])


@gpu
@pytest.mark.parametrize("trades,hess", [(False, False), (True, False), (False, True), (True, True)])
def test_kernel_matches_host_build(trades, hess):
    import torch
    hp, nu, (Dh, Lh, wh, mh) = _bucket_pools()
    st = cf.PoolStore(hp)
    assert len(st.buckets) == 1 and st.buckets[0].kind == _lib.KIND_CRYPTOSWAP_3
    nu_d = torch.as_tensor(nu, dtype=torch.float64, device="cuda")
    acc = st.evaluate(nu_d, 0.0, trades=True, hess=True).cpu().numpy()
    b = st.buckets[0]
    m = b.m
    Dk = b.delta[:, :m].cpu().numpy().T; Lk = b.lam[:, :m].cpu().numpy().T
    wk = b.hcoef[:, :m].cpu().numpy().T; mk = b.hmask[:m].cpu().numpy().astype(np.uint32)
    tok = hp.tok_idx.reshape(-1, 3)
    R = hp.reserves.reshape(-1, 3); p = hp.weights.reshape(-1, 3)
    gross = (np.abs(Dh) + np.abs(Lh)).sum(1) + 1e-300
    # the same per-pool code compiled twice (device and host libm differ in the last bits of exp, log and expm1, and
    # fma contraction differs): flows within 1e-9 of the gross flow on all but a few ill-conditioned pools, 1e-6 on all
    ef = np.maximum(np.abs(Dk - Dh).max(1), np.abs(Lk - Lh).max(1)) / gross
    sw = np.abs(wh).max(1) + 1e-300
    same = mk == mh
    ew = np.abs(wk - wh)[same].max(1) / sw[same]
    print(f"KERNEL vs host: flows rel max {ef.max():.2e} (>1e-9: {(ef > 1e-9).sum()}), mask mismatches "
          f"{(~same).sum()}, edge weights rel max {ew.max():.2e} (>1e-7: {(ew > 1e-7).sum()})")
    assert (ef > 1e-9).sum() <= 1e-4 * m and ef.max() <= 1e-6
    assert (~same).sum() <= 1e-4 * m and (ew > 1e-7).sum() <= 1e-4 * m
    acc2 = st.evaluate(nu_d, 0.0, trades=trades, hess=hess).cpu().numpy()
    y = Lk - Dk
    psi = np.zeros(hp.n_tokens); np.add.at(psi, tok.ravel(), y.ravel())
    gs = np.zeros(hp.n_tokens); np.add.at(gs, tok.ravel(), np.abs(y).ravel())
    assert np.all(np.abs(acc2[:-1] - psi) <= 1e-12 * gs + 1e-300)
    assert np.all(np.abs(acc[:-1] - psi) <= 1e-12 * gs + 1e-300)
    arb = float((nu[tok] * y).sum())
    assert abs(acc2[-1] - arb) <= 1e-12 * float((nu[tok] * np.abs(y)).sum())
    near = np.abs(np.log(R * p / hp.inv[:, None] * 3)).max(1) < 1e-2
    print(f"KERNEL pools={m} trading={(mk != 0).sum()} near-peg={near.sum()}")
    assert near.sum() > 100_000 and (mk != 0).sum() > 100_000
    if trades and hess:
        # a sample, near and far from the peg, against the longdouble reference
        smp = np.sort(np.random.default_rng(7).choice(m, 3000, replace=False))
        hrel = _check_against_xp(Dk[smp], Lk[smp], wk[smp], mk[smp], R[smp], p[smp], hp.amp[smp], hp.cgam[smp],
                                 hp.inv[smp], hp.gamma[smp], nu[tok[smp]])
        print(f"XP sample={len(smp)} near-peg={near[smp].sum()} edge weights rel max={hrel:.2e}")
        assert near[smp].sum() > 300 and hrel <= 1e-6
    if hess:
        rng = np.random.default_rng(0)
        vt = rng.standard_normal(hp.n_tokens)
        Hs = torch.as_tensor(edges_to_hs(wk * (mk != 0)[:, None]), device="cuda")
        T = torch.as_tensor(tok, device="cuda", dtype=torch.int64)
        vv = torch.as_tensor(vt, device="cuda")[T]
        yv = torch.zeros(hp.n_tokens, dtype=torch.float64, device="cuda").index_add_(0, T.reshape(-1),
                                                                                    (Hs @ vv[:, :, None]).reshape(-1))
        yk = st.hvp(torch.as_tensor(vt, dtype=torch.float64, device="cuda"))
        sc = torch.zeros(hp.n_tokens, dtype=torch.float64, device="cuda").index_add_(
            0, T.reshape(-1), (Hs.abs() @ vv.abs()[:, :, None]).reshape(-1))
        assert bool(((yk - yv).abs() <= 1e-12 * sc + 1e-300).all())
        dg = torch.zeros(hp.n_tokens, dtype=torch.float64, device="cuda").index_add_(
            0, T.reshape(-1), torch.diagonal(Hs, dim1=1, dim2=2).reshape(-1))
        torch.testing.assert_close(st.hess_diag(), dg, rtol=1e-12, atol=1e-12 * float(dg.abs().max()))
        Hd = torch.zeros(hp.n_tokens * hp.n_tokens, dtype=torch.float64, device="cuda")
        flat = (T[:, :, None] * hp.n_tokens + T[:, None, :]).reshape(-1)
        Hd.index_add_(0, flat, Hs.reshape(-1))
        torch.testing.assert_close(st.hess_dense(), Hd.reshape(hp.n_tokens, hp.n_tokens), rtol=1e-12,
                                   atol=1e-12 * float(Hd.abs().max()))


def _specs(n, prices, rng):
    basket = np.zeros(n)
    for j in rng.choice(np.arange(1, n), 8, replace=False):
        basket[j] = float(np.exp(rng.normal(1, 1)) * 100 / prices[j])
    return [cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(n))), cf.Liquidate(0, basket),
            cf.Swap(1, 3, 5e3 / prices[1])]


@gpu
def test_mixed_market_every_utility_solves():
    hp, prices = I.synth_tricrypto_market(12_000, 300, seed=4)
    store = cf.PoolStore(hp)
    assert _lib.KIND_CRYPTOSWAP_3 in [int(b.kind) for b in store.buckets]
    rng = np.random.default_rng(1)
    for u in _specs(hp.n_tokens, prices, rng):
        r = cf.solve_pools(hp, u, tol=1e-8, store=store)
        assert r.status == "optimal", r.status
        rep_ = XT.certify(hp, u.spec(hp.n_tokens), r, 1e-8)
        print(f"CERT {type(u).__name__} iters={r.iters} evals={r.evals} hvps={r.hvps} "
              + " ".join(f"{k}={v[0]:.2e}/{v[1]:.2e}" for k, v in rep_.items() if isinstance(v, tuple)))


@gpu
def test_batch_solver_sweep_and_many():
    import torch
    from cfmm_routing_code_b200 import batch as B
    rng = np.random.default_rng(3)
    probs = [_small_tri_problem(rng) for _ in range(6)]
    for lanes in (1, 32):
        for hp, d, prices in probs:
            us = _utilities(rng, hp.n_tokens, prices)
            store = B.CsrStore(hp)
            assert store.has_crypto3
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
                XT.certify(hp, u.spec(hp.n_tokens), res, 1e-9)
                rp = cf.solve_pools(hp, u, tol=1e-9, method="pools")
                assert rp.status == "optimal"
                XT.certify(hp, u.spec(hp.n_tokens), rp, 1e-9)
                assert abs(rp.value - stats[p][0]) <= 1e-7 * max(abs(rp.dual_value), 1.0)
    hp, d, prices = probs[0]
    sw = [cf.Swap(1, 0, t / prices[1]) for t in np.linspace(0.1, 20.0, 12)]
    rb = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], sw, batched=True)
    ru = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], sw, batched=False)
    for x, y, u in zip(rb, ru, sw):
        assert x.status == y.status == "optimal"
        assert abs(x.value - y.value) <= 1e-7 * max(abs(x.dual_value), 1.0)
        XT.certify(hp, u.spec(hp.n_tokens), x, 1e-8)
    many = cf.solve_many([(hp, cf.Swap(1, 0, 2.0 / pr[1])) for hp, _, pr in probs])
    assert all(r.status == "optimal" for r in many)
    for (hp, _, pr), r in zip(probs, many):
        XT.certify(hp, cf.Swap(1, 0, 2.0 / pr[1]).spec(hp.n_tokens), r, 1e-8)


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
    hp, prices = I.synth_tricrypto_market(12_000, 200, seed=8)
    stores = [cf.PoolStore(hp, rank=r, world=world) for r in range(world)]
    u = cf.Arbitrage(prices)
    r0 = cf.solve_pools(hp, u, tol=1e-8, store=stores[0]) if world == 1 else None
    rng = np.random.default_rng(2)
    tri = np.nonzero((hp.kind == KIND_CRYPTOSWAP_HOST) & (np.diff(hp.pool_ptr) == 3))[0]
    ids = np.sort(rng.choice(tri, 1200, replace=False))
    f = hp.pool_ptr[ids]
    sl = f[:, None] + np.arange(3)
    newR = hp.reserves[sl] * np.exp(0.05 * rng.standard_normal((len(ids), 3)))
    newg = np.full(len(ids), 0.9971)
    newp = hp.weights[sl] * np.exp(0.01 * rng.standard_normal((len(ids), 3)))
    newA = hp.amp[ids] * 1.01
    newG = np.minimum(hp.cgam[ids] * 1.02, CRYPTO_GAMMA_RANGE[1])
    half = len(ids) // 2
    for st in stores:
        st.update_pools(ids, reserves=newR, fees=newg)
        st.update_pools(ids[:half], rates=newp[:half], amp=newA[:half], curve_gamma=newG[:half])
    R2, g2, W2, A2, G2 = hp.reserves.copy(), hp.gamma.copy(), hp.weights.copy(), hp.amp.copy(), hp.cgam.copy()
    R2[sl] = newR
    g2[ids] = newg
    W2[sl[:half]] = newp[:half]
    A2[ids[:half]] = newA[:half]; G2[ids[:half]] = newG[:half]
    hp2 = HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, R2, W2, g2, hp.kind, A2, None, hp.lad_ptr, hp.lad_rec,
                    hp.lad_sc, G2)
    for r, st in enumerate(stores):
        fresh = cf.PoolStore(hp2, rank=r, world=world)
        for a, b in zip(_bucket_tensors(st), _bucket_tensors(fresh)):
            for x, y in zip(a, b):
                assert (x is None) == (y is None) and (x is None or torch.equal(x, y))
    if world == 1:
        r1 = cf.solve_pools(hp2, u, tol=1e-8, store=stores[0], nu0=r0.nu)
        assert r1.status == "optimal"
        XT.certify(hp2, u.spec(hp.n_tokens), r1, 1e-8)


@gpu
def test_c_abi_return_codes():
    import torch
    lib = _lib.load()
    buf = torch.ones(8 * 1024, dtype=torch.float64, device="cuda")
    idx = torch.zeros(3 * 1024, dtype=torch.int32, device="cuda")
    nu = torch.ones(4, dtype=torch.float64, device="cuda")
    acc = torch.zeros(5, dtype=torch.float64, device="cuda")
    p = buf.data_ptr()

    def ev(arity, w, lr):
        b = _lib.Bucket(_lib.KIND_CRYPTOSWAP_3, arity, 100, 1024, p, idx.data_ptr(), p, w, lr, None)
        return lib.cfmm_arb_eval(C.byref(b), 4, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc.data_ptr() + 32, None, None)
    assert ev(2, p, p) == -2                  # CFMM_E_KIND
    assert ev(4, p, p) == -2
    assert ev(3, None, p) == -1               # CFMM_E_NULL: price scales
    assert ev(3, p, None) == -1               # CFMM_E_NULL: (A, G, D)
    assert ev(3, p, p) == 0
    b = _lib.Bucket(_lib.KIND_CRYPTOSWAP_3, 3, 100, 1024, p, idx.data_ptr(), p, p, p, None)
    hc = torch.zeros(3 * 1024, dtype=torch.float64, device="cuda")
    mk = torch.zeros(1024, dtype=torch.int32, device="cuda")
    assert lib.cfmm_hvp(C.byref(b), 4, hc.data_ptr(), None, nu.data_ptr(), acc.data_ptr(), None) == -1
    assert lib.cfmm_hess_diag(C.byref(b), 4, hc.data_ptr(), None, acc.data_ptr(), None) == -1
    assert lib.cfmm_hvp(C.byref(b), 4, hc.data_ptr(), mk.data_ptr(), nu.data_ptr(), acc.data_ptr(), None) == 0
    H = torch.zeros(16, dtype=torch.float64, device="cuda")
    assert lib.cfmm_hess_dense(C.byref(b), 4, hc.data_ptr(), mk.data_ptr(), H.data_ptr(), None) == 0
    torch.cuda.synchronize()
