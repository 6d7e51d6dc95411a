"""Two-coin StableSwap (Curve) pools, kind 4: the invariant, the per-pool optimal trade, its Hessian coefficient, the
per-thread solver, the pool-parallel kernel and every solve path.

CPU: the invariant against 40-digit decimal; the fp64 oracle and the longdouble reference (tests/xp_stableswap.py)
against a brute-force maximisation along the curve in decimal; the product / constant-sum limits; hc by finite
differences; cfmm_small::stableswap_pair and the per-thread solver compiled for the host; unit covariance; rejections.
GPU (H100): cfmm_arb_eval and the Hessian kernels on a 200k-pool bucket, every solve path certified, in-place updates,
covariance through solve_pools, and the C ABI's return codes.

Error bounds.  A trading pool's post-trade balance solves log s(t) = log q*, t = log u_a; fp64 evaluates log s with an
absolute error of a few u, so t carries an error of ~c u / |phi'| (phi' = dlog s/dt < 0) -- the problem's own
conditioning: a relative change u of a price moves the exact answer as much.  The flows move by X_a dt, and since
hc = nu_a X_a / (gamma |phi'|),  X_a / |phi'| = gamma hc / nu_a.  So fp64 flows are compared with
    |dflow| <= 1e-12 gross + COND u gamma hc / nu_a          (COND = 64: >= 4x the observed constant),
and hc itself, relative, with 1e-10 + COND u / |phi'| (its log derivative along t is O(1) times 1/|phi'|).
"""
import ctypes as C
import os
import subprocess
from decimal import Decimal, getcontext

import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib, instances as I
from cfmm_routing_code_b200.pools import (HostPools, KIND_STABLESWAP_HOST, check_pool_update, stableswap_invariant)
import small_host
import xp_reference as X
import xp_stableswap as XS

U = 2.0 ** -53
COND = 64.0
AS = [1e-6, 1.0, 100.0, 2000.0, 1e6]
GAMMAS = [1.0, 0.9997, 0.99, 0.5]
HERE = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------------------------ helpers
def _dec_get_D(y0, y1, A):
    """Curve's get_D in 50-digit decimal, iterated to 1e-45"""
    y0, y1, A = Decimal(y0), Decimal(y1), Decimal(A)
    S, D, ann = y0 + y1, y0 + y1, 4 * A
    for _ in range(2000):
        dp = D * D / (2 * y0) * D / (2 * y1)
        Dn = (ann * S + 2 * dp) * D / ((ann - 1) * D + 3 * dp)
        if abs(Dn - D) <= D * Decimal(10) ** -45:
            return Dn
        D = Dn
    raise AssertionError("decimal get_D did not converge")


def _dec_get_xb(Xa, Ra, Rb, ra, rb, A, Dv):
    """token-b balance on the curve 4A(y0+y1) + D = 4AD + D^3/(4 y0 y1) at token-a balance Xa (decimal)"""
    ya = Decimal(ra) * Xa
    b = ya + Dv / (4 * A) - Dv
    c = Dv ** 3 / (16 * A * ya)
    yb = 2 * c / (b + (b * b + 4 * c).sqrt()) if b > 0 else ((b * b + 4 * c).sqrt() - b) / 2
    return yb / Decimal(rb)


def _brute(R, r, A, Dv, g, nu, a):
    """max over Xa >= R_a of nu_b (R_b - X_b(Xa)) - nu_a (Xa - R_a)/gamma by bisection on the sign of a symmetric
    difference quotient of that objective (decimal, 80 digits): (Delta_a, Lambda_b), no marginal-rate formula used"""
    getcontext().prec = 80
    b = 1 - a
    Ra, Rb = Decimal(R[a]), Decimal(R[b])
    A_, D_, g_, na, nb = Decimal(A), Decimal(Dv), Decimal(g), Decimal(nu[a]), Decimal(nu[b])
    h = lambda x: nb * (Rb - _dec_get_xb(x, Ra, Rb, r[a], r[b], A_, D_)) - na * (x - Ra) / g_
    rising = lambda x: h(x * (1 + Decimal(10) ** -50)) > h(x * (1 - Decimal(10) ** -50))
    if not rising(Ra):
        return Decimal(0), Decimal(0)
    lo, hi = Ra, Ra * 2
    while rising(hi):
        lo, hi = hi, hi * 2
    for _ in range(240):
        mid = (lo + hi) / 2
        lo, hi = (mid, hi) if rising(mid) else (lo, mid)
    x = (lo + hi) / 2
    return (x - Ra) / g_, Rb - _dec_get_xb(x, Ra, Rb, r[a], r[b], A_, D_)


def _marginal(R, r, A, Dv):
    """s0 = F_0 / F_1 at the reserves (longdouble): -dX_1/dX_0 = (r0 / r1) s0"""
    u = X.ld(np.asarray(R) * np.asarray(r)) / X.ld(Dv)
    G = 1 / (4 * u[0] * u[1])
    return (4 * X.ld(A) + G / u[0]) / (4 * X.ld(A) + G / u[1])


_HOST = None


def _host():
    """tests/host_harness/stableswap_host.cpp: cfmm_small::stableswap_pair compiled for the host"""
    global _HOST
    if _HOST is None:
        src = os.path.join(HERE, "host_harness", "stableswap_host.cpp")
        hdr = os.path.join(HERE, "..", "cfmm_routing_code_b200", "csrc", "cfmm_small.cuh")
        lib = os.path.join(HERE, "_build", "libstableswap_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src],
                           check=True)
        _HOST = C.CDLL(lib)
    return _HOST


def host_pairs(R, r, A, Dv, g, nu):
    m = len(g)
    arr = [np.ascontiguousarray(x, np.float64) for x in (R, r, A, Dv, g, nu)]
    D, L, hc = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m)
    p_ = lambda x: x.ctypes.data_as(C.c_void_p)
    _host().stableswap_host_pairs(C.c_longlong(m), *[p_(x) for x in arr], p_(D), p_(L), p_(hc))
    return D, L, hc


def random_pools(m, seed, A_range=(1e-6, 1e6), imb=3.0):
    """m random pools (R, r (m, 2), A, D, gamma (m,)) and prices nu (m, 2) near and away from the pools' marginal rates"""
    rng = np.random.default_rng(seed)
    A = np.exp(rng.uniform(np.log(A_range[0]), np.log(A_range[1]), m))
    r = np.exp(rng.normal(0, 0.5, (m, 2)))
    V = np.exp(rng.normal(8, 2, m))
    k = np.exp(imb * rng.standard_normal(m))
    R = np.stack([V * k / r[:, 0], V / k / r[:, 1]], 1)
    g = np.array(GAMMAS)[rng.integers(0, 4, m)]
    D = stableswap_invariant(R, r, A)
    s0 = np.array([float(_marginal(R[i], r[i], A[i], D[i])) for i in range(m)]) if m <= 2000 else None
    base = r[:, 0] / r[:, 1] * (s0 if s0 is not None else 1.0)
    nu = np.stack([base * np.exp(rng.normal(0, 0.05, m)), np.ones(m)], 1) * np.exp(rng.normal(0, 1, m))[:, None]
    return R, r, A, D, g, nu


def edge_pools():
    """every A of AS x every fee x imbalances 1e-6 .. 1e6 x prices inside, at the edges of and far outside the no-trade
    band [gamma, 1/gamma] (r0 s0 / r1) of token-0 prices"""
    R, r, A, Dv, g, nu = [], [], [], [], [], []
    for a in AS:
        for gm in GAMMAS:
            for imb in (1e-6, 1e-2, 1.0, 1e2, 1e6):
                RR = np.array([1e3 * np.sqrt(imb), 1e3 / np.sqrt(imb)]); rr = np.array([1.0, 1.0])
                d = float(stableswap_invariant(RR[None], rr[None], [a])[0])
                p0 = float(rr[0] / rr[1] * _marginal(RR, rr, a, d))
                for f in (gm * (1 - 1e-6), gm * (1 + 1e-6), 1 / gm * (1 - 1e-6), 1 / gm * (1 + 1e-6), 1e-3, 0.3, 3.0, 1e3,
                          np.sqrt(gm)):
                    R.append(RR); r.append(rr); A.append(a); Dv.append(d); g.append(gm); nu.append([p0 * f, 1.0])
    return tuple(np.array(x, float) for x in (R, r, A, Dv, g, nu))


def flow_bound(Dx, Lx, hx, g, nu, R, eps=U, rel=1e-12):
    """per pool: rel gross + 8 eps max(R) / gamma + COND eps gamma hc / nu_a (see the module docstring; the middle term:
    Delta_a = (X_a - R_a) / gamma and Lambda_b = R_b - X_b are differences of balances, exact to a rounding of R)"""
    gross = (np.abs(Dx) + np.abs(Lx)).sum(1).astype(float)
    a = np.where(Dx[:, 0] > 0, 0, 1)
    nua = np.asarray(nu, float)[np.arange(len(g)), a]
    g = np.asarray(g, float)
    return rel * gross + 8 * eps * np.asarray(R, float).reshape(-1, 2).max(1) / g + \
        COND * eps * g * np.abs(hx.astype(float)) / nua


def _stable_hp(R, r, A, g, toks=None, n=None):
    m = len(g)
    toks = np.tile([0, 1], (m, 1)) if toks is None else toks
    n = int(toks.max()) + 1 if n is None else n
    return HostPools(n, np.arange(0, 2 * m + 1, 2, dtype=np.int64), np.ascontiguousarray(toks, np.int32).ravel(),
                     np.ascontiguousarray(R, np.float64).ravel(), np.ascontiguousarray(r, np.float64).ravel(),
                     np.asarray(g, np.float64), np.full(m, KIND_STABLESWAP_HOST, np.uint8), np.asarray(A, np.float64))


# ====================================================================================================== CPU
def test_invariant_matches_decimal_get_D():
    getcontext().prec = 50
    worst = 0.0
    for A in AS:
        for imb, size in [(x, 7e2) for x in (1e-6, 1e-4, 1e-2, 1.0, 1e2, 1e4, 1e6)] + [(3.0, 1e-200), (3.0, 1e200)]:
            for rr in ((1.0, 1.0), (1.3, 0.7)):
                R = np.array([[size * imb, size]])
                d = stableswap_invariant(R, np.array([rr]), [A])[0]
                ref = _dec_get_D(R[0, 0] * rr[0], R[0, 1] * rr[1], A)
                worst = max(worst, float(abs(Decimal(d) - ref) / ref))
    assert worst <= 1e-15, worst


def test_oracle_and_xp_match_brute_force_along_the_curve():
    R, r, A, Dv, g, nu = edge_pools()
    rng = np.random.default_rng(7)
    pick = rng.choice(len(g), 240, replace=False)
    Dx, Lx, hx = XS.stableswap_response(R, r, A, Dv, g, nu)
    worst = {"xp": 0.0, "oracle": 0.0}
    for i in pick:
        a = 0 if Dx[i, 0] > 0 else 1
        bd, bl = _brute(R[i], r[i], A[i], Dv[i], g[i], nu[i], a)
        Do, Lo, ho = XS.arb_stableswap_scalar(R[i], r[i], A[i], Dv[i], g[i], nu[i])
        inside = Dx[i].max() == 0
        if inside:                                               # inside the no-trade band: exactly no trade
            # (the brute force may find a trade of the size of D's own rounding: D is fp64, the search is not)
            assert bd <= 8 * U * max(R[i]) and np.all(Do == 0) and np.all(Lo == 0) and ho == 0, i
            continue
        gross = float(bd + bl)
        cond = float(g[i] * hx[i] / nu[i, a])
        dec = lambda x: Decimal(np.format_float_scientific(np.longdouble(x), unique=True))
        res = 8 * max(R[i]) / g[i]
        # both are held to the fp64 flow bound (the reference's own error is far below it, so this checks the math)
        for tag, D_, L_, tol in (("xp", Dx[i], Lx[i], 1e-12 * gross + (res + COND * cond) * U),
                                 ("oracle", Do, Lo, 1e-12 * gross + (res + COND * cond) * U)):
            e = max(abs(dec(D_[a]) - bd), abs(dec(L_[1 - a]) - bl))
            assert float(e) <= tol, (tag, i, A[i], g[i], float(e), tol)
            worst[tag] = max(worst[tag], float(e) / tol)
    print("brute force: worst error / bound", worst)


def test_no_trade_band_is_exact():
    R, r, A, Dv, g, nu = edge_pools()
    s0 = np.array([float(_marginal(R[i], r[i], A[i], Dv[i])) for i in range(len(g))])
    p0 = r[:, 0] / r[:, 1] * s0
    ratio = nu[:, 0] / (nu[:, 1] * p0)
    inside = (ratio >= g * (1 + 1e-9)) & (ratio <= (1 / g) * (1 - 1e-9))
    outside = (ratio < g * (1 - 1e-9)) | (ratio > (1 / g) * (1 + 1e-9))
    assert inside.sum() >= 100 and outside.sum() >= 300
    for fn in (lambda: XS.stableswap_response(R, r, A, Dv, g, nu), lambda: host_pairs(R, r, A, Dv, g, nu)):
        D, L, h = fn()
        assert np.all(D[inside] == 0) and np.all(L[inside] == 0) and np.all(h[inside] == 0)
        assert np.all((D[outside] > 0).any(1) & (h[outside] > 0))     # just outside the band: a (tiny) trade


def test_small_A_is_the_product_pool_on_scaled_reserves():
    # (the invariant's 4A (y0 + y1) term is relatively 4A y / D: balances within ~10x of each other and trades of a few
    # percent keep it near 1e-8, far below the 1e-6 asserted)
    R, r, _, _, g, nu = random_pools(500, seed=3, imb=0.5)
    A = np.full(len(g), 1e-9)
    Dv = stableswap_invariant(R, r, A)
    D, L, _ = host_pairs(R, r, A, Dv, g, nu)
    y, mu = R * r, nu / r
    for a, b in ((0, 1), (1, 0)):
        go = g * mu[:, b] * y[:, b] > mu[:, a] * y[:, a]
        t = np.sqrt(np.where(go, g * mu[:, b] * y[:, b] / (mu[:, a] * y[:, a]), 1.0))
        Dp = np.where(go, y[:, a] * (t - 1) / g / r[:, a], 0.0)
        Lp = np.where(go, y[:, b] * (1 - 1 / t) / r[:, b], 0.0)
        np.testing.assert_allclose(D[:, a], Dp, rtol=1e-6, atol=1e-12 * R.max())
        np.testing.assert_allclose(L[:, b], Lp, rtol=1e-6, atol=1e-12 * R.max())


def test_large_A_approaches_the_constant_sum_rule():
    """a balanced pool with rates (1.1, 1): the realised price Lambda_1 / Delta_0 of a trade approaches gamma r0 / r1 as
    A grows, and the trade direction follows the constant-sum rule gamma mu_b > mu_a on the scaled prices"""
    R, r, g = np.array([[1e6 / 1.1, 1e6]]), np.array([[1.1, 1.0]]), np.array([0.9996])
    nu = np.array([[1.1 * 1.002, 1.0]])                         # token 0 slightly rich: sell token 1 for it? no: buy 1
    gaps = []
    for A in (1.0, 1e2, 1e4, 1e6):
        Dv = stableswap_invariant(R, r, [A])
        D, L, _ = host_pairs(R, r, [A], Dv, g, nu)
        mu = nu[0] / r[0]
        a = 0 if g[0] * mu[1] > mu[0] else 1                    # constant-sum rule on scaled prices
        assert D[0, a] > 0 and D[0, 1 - a] == 0, A
        price = L[0, 1 - a] / D[0, a]                            # units of b per unit of a tendered
        lim = g[0] * r[0, a] / r[0, 1 - a]
        gaps.append(abs(price - lim) / lim)
    assert all(x > y for x, y in zip(gaps, gaps[1:])) and gaps[-1] <= 1e-3, gaps


def test_hc_matches_finite_differences():
    R, r, A, Dv, g, nu = random_pools(400, seed=11, A_range=(1e-3, 1e5), imb=1.0)
    _, _, hc = host_pairs(R, r, A, Dv, g, nu)
    h = 1e-7                                                     # longdouble: rounding ~1e-19 / h, truncation ~h^2
    ys = []
    for sgn in (1, -1):
        n2 = nu.astype(np.longdouble).copy(); n2[:, 0] *= np.exp(np.longdouble(sgn * h))
        D, L, _ = XS.stableswap_response(R, r, A, Dv, g, n2)
        ys.append(L[:, 0] - D[:, 0])
    fd = (nu[:, 0] * (ys[0] - ys[1]) / (2 * h)).astype(float)
    trade = hc > 0
    assert trade.sum() >= 200
    # central difference: O(h^2) truncation; pools whose step crosses the band edge are excluded (y_0 has a kink there)
    _, _, hp_ = XS.stableswap_response(R, r, A, Dv, g, nu * np.exp([[h, 0]]))
    _, _, hm_ = XS.stableswap_response(R, r, A, Dv, g, nu * np.exp([[-h, 0]]))
    smooth = trade & (hp_ > 0) & (hm_ > 0)
    np.testing.assert_allclose(hc[smooth], fd[smooth], rtol=1e-5)
    assert np.all(hc[~trade] == 0) and np.all(np.abs(fd[(hp_ == 0) & (hm_ == 0)]) == 0)


def test_host_pair_matches_xp_reference():
    hp, nu = _bucket_pools()                        # the GPU test's 200k pools: they once caught a Newton crawl
    tok = hp.tok_idx.reshape(-1, 2)
    sets = [random_pools(3000, seed=s) for s in (1, 2)] + [edge_pools()] + \
        [(hp.reserves.reshape(-1, 2), hp.weights.reshape(-1, 2), hp.amp, hp.inv, hp.gamma, nu[tok])]
    worst = 0.0
    for R, r, A, Dv, g, nu in sets:
        D, L, hc = host_pairs(R, r, A, Dv, g, nu)
        Dx, Lx, hx = XS.stableswap_response(R, r, A, Dv, g, nu)
        bound = flow_bound(Dx, Lx, hx, g, nu, R)
        err = np.maximum(np.abs(D - Dx.astype(float)).max(1), np.abs(L - Lx.astype(float)).max(1))
        assert np.all(err <= bound), float((err / np.maximum(bound, 1e-300)).max())
        worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
        # hc jumps at the band edge: pools within rounding of it may trade (tinily, inside the flow bound) in one and
        # not the other; everywhere else both trade or neither does
        tr = (hx > 0) & (hc > 0)
        a = np.where(Dx[:, 0] > 0, 0, 1)
        Xa = (R[np.arange(len(g)), a] + g * Dx[np.arange(len(g)), a]).astype(float)
        inv_dphi = (g * hx.astype(float) / (nu[np.arange(len(g)), a] * Xa))      # 1 / |phi'|
        rel = np.abs(hc - hx.astype(float)) / np.where(tr, hx.astype(float), 1.0)
        assert np.all(rel[tr] <= 1e-10 + COND * U * inv_dphi[tr] * (1 + inv_dphi[tr])), float(rel[tr].max())
    print("host pair: worst flow error / bound", worst)


def _small_stable_problem(rng):
    """3-6 tokens: a product chain over all tokens plus StableSwap pools between tokens 0..2 (value ~1 each)"""
    n = int(rng.integers(3, 7))
    prices = np.exp(rng.normal(0, 1, n)); prices[:3] = [1.0, 1.001, 0.999]
    li, res, fees, kinds, w = [], [], [], [], []
    for i in range(n - 1):
        liq = np.exp(rng.normal(4, 1))
        li.append([i, i + 1]); res.append(list(liq / prices[[i, i + 1]] * np.exp(0.05 * rng.standard_normal(2))))
        fees.append(0.997); kinds.append("product"); w.append(None)
    for _ in range(int(rng.integers(2, 6))):
        a, b = rng.choice(3, 2, replace=False)
        V = np.exp(rng.normal(5, 1)); k = np.exp(0.3 * rng.standard_normal())
        li.append([int(a), int(b)]); res.append([V * k / prices[a], V / k / prices[b]])
        fees.append(float(rng.choice([0.9996, 0.9999]))); kinds.append("stableswap")
        w.append((float(rng.choice([10.0, 100.0, 2000.0])), 1.0, 1.0))
    d = dict(n_tokens=n, local_indices=li, reserves=res, fees=fees, kinds=kinds, weights=w)
    return HostPools.from_lists(n, li, res, fees, kinds, w), d, prices


def _utilities(rng, n, prices):
    U_ = XS.Utility
    us = [U_.arbitrage(prices * np.exp(0.01 * rng.standard_normal(n)))]
    us.append(U_.swap(n, 0, 1, float(np.exp(rng.normal(3, 1)))))
    basket = np.zeros(n); basket[1] = float(np.exp(rng.normal(2, 1))); basket[2] = float(np.exp(rng.normal(1, 1)))
    us.append(U_.liquidate(n, 0, basket))
    return us


def _csr_args(hp):
    """the cfmm_csr_pools arrays of a HostPools: kind 4's logrw = (A, D) per pool, log(R / w) elsewhere"""
    slot_kind = np.repeat(hp.kind, np.diff(hp.pool_ptr))
    logrw = np.log(np.maximum(hp.reserves, 1e-300) / np.where(slot_kind == 0, hp.weights, 1.0))
    ss = np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0]
    logrw[hp.pool_ptr[ss]] = hp.amp[ss]; logrw[hp.pool_ptr[ss] + 1] = hp.inv[ss]
    return [np.ascontiguousarray(x, t) for x, t in ((hp.pool_ptr, np.int64), (hp.tok_idx, np.int32),
                                                    (hp.reserves, np.float64), (hp.weights, np.float64),
                                                    (logrw, np.float64), (hp.gamma, np.float64), (hp.kind, np.uint8))]


def _host_solve(hp, specs, tol=1e-9, stable=True):
    """the per-thread solver built for the host: its StableSwap instance (tests/host_harness/stableswap_host.cpp) or,
    stable=False, the plain one through tests/small_host.py's harness"""
    n, B, nnz = hp.n_tokens, len(specs), len(hp.tok_idx)
    c = np.stack([u.c for u in specs]).astype(float); a = np.stack([u.a for u in specs]).astype(float)
    fl = np.ascontiguousarray(np.stack([np.asarray(u.eq, np.uint8) | (np.asarray(u.pinned, np.uint8) << 1)
                                        for u in specs]), np.uint8)
    nu = np.ascontiguousarray(np.stack([np.where(u.c > 0, u.c, np.median(u.c[u.c > 0]) if (u.c > 0).any() else 1.0)
                                        for u in specs]))
    keep = _csr_args(hp)
    psi = np.zeros((B, n)); st = np.zeros((B, 8)); d = np.zeros((B, nnz)); l = np.zeros((B, nnz))
    p_ = lambda x: x.ctypes.data_as(C.c_void_p)
    if stable:
        fn = _host().stableswap_host_solve
        fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 7 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
        fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), tol)
    else:
        small_host.load().small_host_solve(n, hp.m, *[p_(k) for k in keep], B, None, p_(c), p_(a), p_(fl), p_(nu),
                                           p_(psi), p_(st), p_(d), p_(l), nnz, tol, 1)
    return dict(nu=nu, psi=psi, stats=st, delta=d, lam=l)


def test_plain_solver_instance_rejects_stableswap_pools():
    """the solver instance without StableSwap support (k_batch_solve, kept at its register budget) refuses them:
    status 3, NaN results, like any pool the closed forms do not cover"""
    rng = np.random.default_rng(100)
    hp, _, prices = _small_stable_problem(rng)
    out = _host_solve(hp, _utilities(rng, hp.n_tokens, prices), stable=False)
    assert np.all(out["stats"][:, 7] == 3) and np.all(np.isnan(out["stats"][:, 0]))


def test_host_solver_matches_oracle_step_for_step():
    """same algorithm: same values and prices, and the same iteration and evaluation counts on 21 of these 24 problems.
    The oracle evaluates the pools with numpy, the solver in C++; their last bits differ, and in three problems a line
    search that barely accepts (or rejects) a step takes another path: seed 3, problem 2 (Liquidate, 5 tokens, 7 pools)
    ends after 18 iterations / 23 evaluations against the oracle's 15 / 20; seed 4, problem 0 (Arbitrage, 5 tokens,
    9 pools) after 16 / 81 against 16 / 84; seed 7, problem 0 (Arbitrage, 3 tokens) after 18 / 67 against 18 / 68.  All
    end optimal at the same value.  The mismatches are listed exactly, so any other one fails."""
    expected_paths_differ = {(3, 2), (4, 0), (7, 0)}
    differ = set()
    for seed in range(8):
        rng = np.random.default_rng(100 + seed)
        hp, _, prices = _small_stable_problem(rng)
        specs = _utilities(rng, hp.n_tokens, prices)
        out = _host_solve(hp, specs)
        for p, u in enumerate(specs):
            r = XS.oracle_solve(hp, u, tol=1e-9)
            st = out["stats"][p]
            assert r.status == "optimal" and int(st[7]) == 0, (seed, p, r.status, st[7])
            scale = max(abs(r.dual_value), 1e-300)
            assert abs(st[0] - r.value) <= 1e-9 * scale and abs(st[1] - r.dual_value) <= 1e-9 * scale
            np.testing.assert_allclose(out["nu"][p], r.nu, rtol=1e-7)
            if (int(st[5]), int(st[6])) != (r.iters, r.evals):
                differ.add((seed, p))
            XS.certify(hp, u, _as_result(hp, out, p), 1e-9)
    assert differ <= expected_paths_differ, differ


def _as_result(hp, out, p):
    import types
    ptr = hp.pool_ptr
    return types.SimpleNamespace(value=out["stats"][p][0], dual_value=out["stats"][p][1], psi=out["psi"][p],
                                 nu=out["nu"][p], deltas=[out["delta"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                 lambdas=[out["lam"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])


def test_oracle_unit_covariance():
    """rescale token j by s: reserves x s, r_j / s, a_j s, c_j / s  =>  nu_j / s, psi_j s, same value"""
    rng = np.random.default_rng(5)
    hp, d, prices = _small_stable_problem(rng)
    n = hp.n_tokens
    for u in _utilities(rng, n, prices):
        r0 = XS.oracle_solve(hp, u, tol=1e-10)
        s = np.exp(rng.normal(0, 1, n))          # (the price floor is 1e-12 max|c|: keep rescaled prices well above it)
        R = [list(np.asarray(x) * s[l]) for x, l in zip(d["reserves"], d["local_indices"])]
        W = [w if k != "stableswap" else (w[0], w[1] / s[l[0]], w[2] / s[l[1]])
             for w, k, l in zip(d["weights"], d["kinds"], d["local_indices"])]
        hp2 = HostPools.from_lists(n, d["local_indices"], R, d["fees"], d["kinds"], W)
        u2 = XS.Utility(u.c / s, u.a * s, u.eq, u.pinned)
        r1 = XS.oracle_solve(hp2, u2, tol=1e-10)
        assert r0.status == r1.status == "optimal"
        # (prices are not compared: inside a pool's no-trade band the optimal dual prices are not unique)
        gross = sum(np.abs(x).sum() for x in r0.deltas) + sum(np.abs(x).sum() for x in r0.lambdas)
        np.testing.assert_allclose(r1.psi / s, r0.psi, rtol=1e-10, atol=1e-10 * gross / s.min())
        assert abs(r1.value - r0.value) <= 1e-10 * abs(r0.dual_value)


def test_rejections():
    li, fees = [[0, 1]], [0.9996]
    ok = dict(reserves=[[10.0, 12.0]], weights=[(100.0, 1.0, 1.0)])
    HostPools.from_lists(2, li, ok["reserves"], fees, ["stableswap"], ok["weights"]).validate()
    bad_w = [(0.0, 1, 1), (-5.0, 1, 1), (np.nan, 1, 1), (np.inf, 1, 1), (2e7, 1, 1), (100, 0.0, 1), (100, -1, 1),
             (100, np.nan, 1), (100, 1, np.inf), (100, 1), None]
    for w in bad_w:
        with pytest.raises(ValueError):
            HostPools.from_lists(2, li, ok["reserves"], fees, ["stableswap"], [w])
    for R in ([0.0, 1.0], [-1.0, 2.0], [np.nan, 1.0], [1.0, np.inf]):
        with pytest.raises(ValueError):
            HostPools.from_lists(2, li, [R], fees, ["stableswap"], ok["weights"])
    with pytest.raises(ValueError):                              # arity 3
        HostPools.from_lists(3, [[0, 1, 2]], [[1.0, 2.0, 3.0]], fees, ["stableswap"], [(100.0, 1, 1)])
    hp = HostPools.from_lists(2, li, ok["reserves"], fees, ["stableswap"], ok["weights"])
    bad = HostPools(2, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind, np.array([0.0]))
    with pytest.raises(ValueError):                              # A = 0 given directly in CSR form
        bad.validate()
    for R in ([[0.0, 1.0]], [[-1.0, 1.0]], [[np.nan, 1.0]], [[1.0, np.inf]]):
        with pytest.raises(ValueError):
            check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], np.array(R))
    with pytest.raises(ValueError):                              # a vector of the wrong arity
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], [[1.0, 2.0, 3.0]])
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], np.array([[3.0, 4.0]]))
    assert np.array_equal(u.reserves, [3.0, 4.0])


def test_xp_certificate_covers_stableswap_pools():
    """the certificate rejects an answer whose StableSwap trades over-pay the pool (infeasible) and accepts the oracle's"""
    rng = np.random.default_rng(9)
    hp, _, prices = _small_stable_problem(rng)
    u = _utilities(rng, hp.n_tokens, prices)[0]
    r = XS.oracle_solve(hp, u, tol=1e-10)
    XS.certify(hp, u, r, 1e-10)
    ss = int(np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0][0])
    bad = [x.copy() for x in r.lambdas]
    bad[ss] = bad[ss] + 1e-6 * hp.reserves[hp.pool_ptr[ss]:hp.pool_ptr[ss + 1]]
    import types
    rb = types.SimpleNamespace(**{**r.__dict__, "lambdas": bad})
    rep = XS.certify(hp, u, rb, 1e-10, check=False)
    assert any("pool-feasible" in f for f in rep["fails"])


def test_market_generator():
    s = I.synth_stable_market(3000, 40, seed=1)
    s.pop("prices")
    hp = HostPools(**s)
    hp.validate()
    ss = hp.kind == KIND_STABLESWAP_HOST
    assert 0.25 < ss.mean() < 0.35 and np.all(hp.inv[ss] > 0) and np.all(hp.amp[~ss] == 0)


# ====================================================================================================== GPU
gpu = pytest.mark.gpu


def _bucket_pools(m=200_000, seed=21):
    """random pools over 64 tokens (random pairs, prices nu ~ exp(N(0, 0.3))) plus the CPU edge set, each edge pool on a
    token pair of its own priced as edge_pools() intends (inside, at the edges of and far outside its no-trade band).
    Returns (HostPools, nu)."""
    R, r, A, Dv, g, _ = random_pools(m, seed, A_range=(1e-6, 1e6), imb=2.0)
    ER, Er, EA, _, Eg, Enu = edge_pools()
    rng = np.random.default_rng(seed)
    n0, ne = 64, len(Eg)
    toks = np.stack([rng.integers(0, n0, m), np.zeros(m, int)], 1)
    toks[:, 1] = (toks[:, 0] + rng.integers(1, n0, m)) % n0
    et = n0 + np.arange(2 * ne).reshape(ne, 2)
    nu = np.concatenate([np.exp(rng.normal(0, 0.3, n0)), Enu.ravel()])
    hp = _stable_hp(np.concatenate([R, ER]), np.concatenate([r, Er]), np.concatenate([A, EA]), np.concatenate([g, Eg]),
                    np.concatenate([toks, et]), n0 + 2 * ne)
    return hp, nu


@gpu
@pytest.mark.parametrize("trades,hess", [(False, False), (True, False), (False, True), (True, True)])
def test_kernel_matches_xp_reference(trades, hess):
    import torch
    hp, nu = _bucket_pools()
    st = cf.PoolStore(hp)
    assert len(st.buckets) == 1 and st.buckets[0].kind == _lib.KIND_STABLESWAP
    nu_d = torch.as_tensor(nu, dtype=torch.float64, device="cuda")
    acc = st.evaluate(nu_d, 0.0, trades=trades, hess=hess).cpu().numpy()
    psi, arbv = acc[:-1], acc[-1]
    ref = XS.response(hp, nu)
    tok = hp.tok_idx.reshape(-1, 2)
    Dx, Lx, hx = ref["delta"].reshape(-1, 2), ref["lam"].reshape(-1, 2), ref["h"]
    bound = flow_bound(Dx, Lx, hx, hp.gamma, nu[tok], hp.reserves)
    # psi: every token sums k_j flows, each within `bound` of the exact one, in any order: 4 k_j u gross_j more
    psi_x, gross, k = X.flows(hp, ref["delta"], ref["lam"])
    b_tok = np.zeros(hp.n_tokens)
    np.add.at(b_tok, tok.ravel(), np.repeat(bound, 2))
    err_psi = np.abs(psi - psi_x.astype(float))
    lim_psi = b_tok + 4 * U * np.maximum(k.astype(float), 1) * gross.astype(float)
    assert np.all(err_psi <= lim_psi), float((err_psi / lim_psi).max())
    # arb: sum_i nu'(L - D): the flow errors weighted by prices, plus 4 m u of the price-weighted gross
    lim_arb = float((nu[tok].max(1) * 2 * bound).sum() + 4 * hp.m * U * (nu * gross.astype(float)).sum())
    assert abs(arbv - float(ref["arb"].sum())) <= lim_arb
    b = st.buckets[0]
    m = b.m
    if trades:
        Dk = b.delta[:, :m].cpu().numpy().T; Lk = b.lam[:, :m].cpu().numpy().T
        err = np.maximum(np.abs(Dk - Dx.astype(float)).max(1), np.abs(Lk - Lx.astype(float)).max(1))
        assert np.all(err <= bound), float((err / bound).max())
    if hess:
        hk = b.hcoef[:m].cpu().numpy()
        # hc jumps from 0 at the band edge: a pool exactly on it (the edge set's gamma = 1, price = marginal rate) may
        # trade by a rounding in one precision and not in the other; its exact trade is then within the flow bound of 0
        mism = (hk > 0) != (hx > 0)
        gross_x = (np.abs(Dx) + np.abs(Lx)).sum(1).astype(float)
        assert np.all(gross_x[mism] <= bound[mism]) and mism.sum() <= 40, int(mism.sum())
        tr = (hx > 0) & (hk > 0)
        a = np.where(Dx[:, 0] > 0, 0, 1)
        Xa = (hp.reserves.reshape(-1, 2)[np.arange(m), a] + hp.gamma * Dx[np.arange(m), a]).astype(float)
        inv_dphi = hp.gamma * hx.astype(float) / (nu[tok][np.arange(m), a] * Xa)
        rel = np.abs(hk - hx.astype(float)) / np.where(tr, hx.astype(float), 1.0)
        assert np.all(rel[tr] <= 1e-10 + COND * U * inv_dphi[tr] * (1 + inv_dphi[tr])), float(rel[tr].max())
        assert np.all(hk[~tr & ~mism] == 0)
        # the Hessian kernels take the generic pair branch: numpy from the kernel's own hcoef
        rng = np.random.default_rng(0)
        vt = rng.standard_normal(hp.n_tokens)
        c_ = hk * (vt[tok[:, 0]] - vt[tok[:, 1]])
        y = np.zeros(hp.n_tokens); np.add.at(y, tok[:, 0], c_); np.add.at(y, tok[:, 1], -c_)
        yk = st.hvp(torch.as_tensor(vt, dtype=torch.float64, device="cuda")).cpu().numpy()
        sc = np.zeros(hp.n_tokens); np.add.at(sc, tok.ravel(), np.repeat(np.abs(c_), 2))
        assert np.all(np.abs(yk - y) <= 8 * U * np.maximum(k.astype(float), 1) * sc + 1e-300)
        dg = np.zeros(hp.n_tokens); np.add.at(dg, tok.ravel(), np.repeat(hk, 2))
        np.testing.assert_allclose(st.hess_diag().cpu().numpy(), dg, rtol=1e-12)
        Hd = np.zeros((hp.n_tokens, hp.n_tokens))
        np.add.at(Hd, (tok[:, 0], tok[:, 0]), hk); np.add.at(Hd, (tok[:, 1], tok[:, 1]), hk)
        np.add.at(Hd, (tok[:, 0], tok[:, 1]), -hk); np.add.at(Hd, (tok[:, 1], tok[:, 0]), -hk)
        np.testing.assert_allclose(st.hess_dense().cpu().numpy(), Hd, rtol=1e-12, atol=1e-12 * np.abs(Hd).max())


def _mixed_market(m=120_000, n=400, seed=4):
    s = I.synth_stable_market(m, n, seed)
    prices = s.pop("prices")
    return HostPools(**s), prices


def _specs(n, prices, rng):
    basket = np.zeros(n)
    for j in rng.choice(np.arange(1, n), 8, replace=False):
        basket[j] = float(np.exp(rng.normal(1, 1)) * 100 / prices[j])
    return [cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(n))), cf.Liquidate(0, basket),
            cf.Swap(1, 3, 5e3 / prices[1])]


@gpu
def test_mixed_market_every_utility_certifies():
    hp, prices = _mixed_market()
    store = cf.PoolStore(hp)
    kinds = sorted(int(b.kind) for b in store.buckets)
    assert _lib.KIND_STABLESWAP in kinds and len(store.buckets) >= 3
    rng = np.random.default_rng(1)
    for u in _specs(hp.n_tokens, prices, rng):
        r = cf.solve_pools(hp, u, tol=1e-8, store=store)
        assert r.status == "optimal", r.status
        assert r.info.history, "the python outer loop (solver.py) ran: no native solver covers StableSwap buckets"
        rep = XS.certify(hp, u.spec(hp.n_tokens), r, 1e-8)
        print(f"CERT {type(u).__name__} iters={r.iters} evals={r.evals} hvps={r.hvps} "
              + " ".join(f"{k}={v[0]:.2e}/{v[1]:.2e}" for k, v in rep.items() if isinstance(v, tuple)))


@gpu
def test_batch_solver_and_sweep():
    from cfmm_routing_code_b200 import batch as B
    rng = np.random.default_rng(3)
    probs = [_small_stable_problem(rng) for _ in range(6)]
    for lanes in (1, 32):
        for hp, d, prices in probs:
            us = [cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(hp.n_tokens))),
                  cf.Swap(0, 1, 20.0), cf.Liquidate(0, np.r_[0.0, 5.0, 3.0, np.zeros(hp.n_tokens - 3)])]
            store = B.CsrStore(hp)
            c, a, fl, nu = B.pack_utilities(us, hp.n_tokens)
            import torch
            up = lambda x: torch.as_tensor(x, device="cuda")
            nu_d = up(nu)
            psi, stats, dl, lm = B.solve_batch_device(store, up(c), up(a), up(fl), nu_d, tol=1e-9, lanes=lanes)
            stats = stats.cpu().numpy(); psi = psi.cpu().numpy(); nu_h = nu_d.cpu().numpy()
            dl, lm = dl.cpu().numpy(), lm.cpu().numpy()
            ptr = hp.pool_ptr
            import types
            for p, u in enumerate(us):
                assert int(stats[p][7]) == 0, (lanes, p, stats[p])
                res = types.SimpleNamespace(value=stats[p][0], dual_value=stats[p][1], psi=psi[p], nu=nu_h[p],
                                            deltas=[dl[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                            lambdas=[lm[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])
                XS.certify(hp, u.spec(hp.n_tokens), res, 1e-9)
                rp = cf.solve_pools(hp, u, tol=1e-9, method="pools")
                assert rp.status == "optimal"
                assert abs(rp.value - stats[p][0]) <= 1e-8 * abs(rp.dual_value)
    hp, d, prices = probs[0]
    sw = [cf.Swap(0, 1, t) for t in np.linspace(1.0, 400.0, 12)]
    rb = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], sw, batched=True)
    ru = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], sw, batched=False)
    for x, y in zip(rb, ru):
        assert x.status == y.status == "optimal"
        assert abs(x.value - y.value) <= 1e-7 * max(abs(x.dual_value), 1.0)
    many = cf.solve_many([(hp, cf.Swap(0, 1, 20.0)) for hp, _, _ in probs])
    assert all(r.status == "optimal" for r in many)


@gpu
def test_update_pools_equals_a_fresh_store_and_resolves():
    import torch
    hp, prices = _mixed_market(m=100_000, n=300, seed=8)
    store = cf.PoolStore(hp)
    u = cf.Arbitrage(prices)
    r0 = cf.solve_pools(hp, u, tol=1e-8, store=store)
    rng = np.random.default_rng(2)
    ids = np.sort(rng.choice(hp.m, 5000, replace=False))
    ar = np.diff(hp.pool_ptr)[ids]
    newR = [hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] * np.exp(0.05 * rng.standard_normal(k)) for i, k in zip(ids, ar)]
    newg = np.where(hp.kind[ids] == KIND_STABLESWAP_HOST, 0.9998, 0.997)
    store.update_pools(ids, reserves=newR, fees=newg)
    R2 = hp.reserves.copy(); g2 = hp.gamma.copy()
    for i, x in zip(ids, newR):
        R2[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] = x
    g2[ids] = newg
    hp2 = HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, R2, hp.weights, g2, hp.kind, hp.amp)
    fresh = cf.PoolStore(hp2)
    assert (hp2.kind[ids] == KIND_STABLESWAP_HOST).sum() > 500
    for a, b in zip(store.buckets, fresh.buckets):
        assert a.kind == b.kind
        if getattr(a, "blocked", False):
            for t in ("r0", "r1", "gamma_inv"):
                assert torch.equal(getattr(a, t), getattr(b, t))
            continue
        for t in ("reserves", "gamma", "weights", "logrw"):
            x, y = getattr(a, t), getattr(b, t)
            assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), (a.kind, t)
    r1 = cf.solve_pools(hp2, u, tol=1e-8, store=store, nu0=r0.nu)
    assert r1.status == "optimal"
    XS.certify(hp2, u.spec(hp.n_tokens), r1, 1e-8)


@gpu
def test_solve_pools_unit_covariance():
    rng = np.random.default_rng(6)
    hp, d, prices = _small_stable_problem(rng)
    n = hp.n_tokens
    s = np.exp(rng.normal(0, 1, n))
    R = [list(np.asarray(x) * s[l]) for x, l in zip(d["reserves"], d["local_indices"])]
    W = [w if k != "stableswap" else (w[0], w[1] / s[l[0]], w[2] / s[l[1]])
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
        b = _lib.Bucket(_lib.KIND_STABLESWAP, arity, 100, 1024, p, idx.data_ptr(), p, w, lr, None)
        return lib.cfmm_arb_eval(C.byref(b), 4, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc.data_ptr() + 32, None, None)
    assert ev(3, p, p) == -2                  # CFMM_E_KIND
    assert ev(2, None, p) == -1               # CFMM_E_NULL: rates
    assert ev(2, p, None) == -1               # CFMM_E_NULL: (A, D)
    assert ev(2, p, p) == 0
    torch.cuda.synchronize()
