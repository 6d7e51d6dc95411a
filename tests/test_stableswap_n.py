"""n-coin StableSwap (Curve) pools: kind 4 with 2..8 coins on the host, kind 5 (CFMM_KIND_STABLESWAP_N) on the device.

CPU: the n-coin invariant against 50-digit decimal; the amplification convention against the contracts' integer get_D;
cfmm_small::stableswap_n compiled for the host against the longdouble reference (tests/xp_stableswap_n.py), the KKT
conditions in decimal, the two-coin pair function, the A -> 0 geometric-mean limit and the no-trade band; the Hessian
by finite differences; the per-thread solver's n-coin instance against the oracle; validation.
GPU (H100): k_eval_stable_n against the reference for arity 3..8 in all four (trades, hess) instances and against
k_eval_stable at arity 2; HVP / diagonal / dense consistency; every solve path on mixed markets, certified; in-place
updates; bucket assignment.

Error bounds.  The flows of a trading pool are x_j = R_j exp(z_j) with z_j = l - bA_j (or l - bB_j), differences of
logarithms of size |l| ~ log(1 / q) <= 20 (q = Q / a), each carrying a few u of absolute error; the root of h moves l
by the problem's own conditioning.  Flows are compared with flow_tol: 1e-10 of the pool's gross trade plus
64 u (1 + |l|) R_j, plus (where a second method or precision is compared) the conditioning term 64 u sum_i |Hs_ji| / nu_j
and arg_tol, the rounding of the expm1 denominators (derived in its docstring).
"""
import ctypes as C
import os
import subprocess
import types
from decimal import Decimal, getcontext

import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib, instances as I
from cfmm_routing_code_b200.pools import (HostPools, KIND_STABLESWAP_HOST, check_pool_update, stableswap_invariant,
                                          stableswap_invariant_any, stableswap_invariant_n)
import xp_reference as X
import xp_stableswap as XS
import xp_stableswap_n as XN

U = 2.0 ** -53
HERE = os.path.dirname(os.path.abspath(__file__))
ANN_MAX = 4e7


# ------------------------------------------------------------------------------------------------------ helpers
def _dec_get_D(y, ann):
    """get_D with the whitepaper coefficient ann = A n^n in 50-digit decimal, from D = S, iterated to 1e-45"""
    getcontext().prec = 50
    y = [Decimal(float(v)) for v in y]
    n = len(y)
    S, D, ann = sum(y), sum(y), Decimal(float(ann))
    for _ in range(20000):
        dp = D
        for v in y:
            dp = dp * D / (n * v)
        Dn = (ann * S + n * dp) * D / ((ann - 1) * D + (n + 1) * dp)
        if abs(Dn - D) <= D * Decimal(10) ** -45:
            return Dn
        D = Dn
    raise AssertionError("decimal get_D did not converge")


_HOST = None


def _host():
    """tests/host_harness/stableswap_n_host.cpp: cfmm_small::stableswap_n compiled for the host"""
    global _HOST
    if _HOST is None:
        src = os.path.join(HERE, "host_harness", "stableswap_n_host.cpp")
        hdr = os.path.join(HERE, "..", "cfmm_routing_code_b200", "csrc", "cfmm_small.cuh")
        lib = os.path.join(HERE, "_build", "libstableswap_n_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src],
                           check=True)
        _HOST = C.CDLL(lib)
    return _HOST


p_ = lambda x: x.ctypes.data_as(C.c_void_p)


def host_pools(R, r, A, Dv, g, nu):
    m, k = R.shape
    arr = [np.ascontiguousarray(x, np.float64) for x in (R, r, A, Dv, g, nu)]
    D, L, h = np.zeros((m, k)), np.zeros((m, k)), np.zeros((m, k))
    mask = np.zeros(m, np.uint32)
    _host().stablen_host_pools(C.c_longlong(m), C.c_int(k), *[p_(x) for x in arr], p_(D), p_(L), p_(h), p_(mask))
    return D, L, h, mask


def host_hvp(h, z):
    m, k = h.shape
    y = np.zeros((m, k))
    _host().stablen_host_hvp(C.c_longlong(m), C.c_int(k), p_(np.ascontiguousarray(h)), p_(np.ascontiguousarray(z)),
                             p_(y))
    return y


def random_pools(m, n, seed, peg=True, ann_range=(1e-3, ANN_MAX), at_max=True):
    """m pools of n coins: R, r (m, n), A, D, gamma (m,), and prices nu (m, n) near the peg (value ~1 per scaled unit,
    mispriced by ~0.1 %) or far from it (mispriced by ~30 %); balances value-imbalanced by ~e^N(0, 0.5) (near) or
    ~e^N(0, 3) (far)"""
    rng = np.random.default_rng(seed)
    ann = np.exp(rng.uniform(np.log(ann_range[0]), np.log(ann_range[1]), m))
    if peg and at_max:
        ann[: m // 4] = ANN_MAX                                          # the largest allowed coefficient
    A = ann / float(n ** n)
    r = np.exp(rng.normal(0, 0.3, (m, n)))
    V = np.exp(rng.normal(8, 2, m))
    R = V[:, None] * np.exp((0.5 if peg else 3.0) * rng.standard_normal((m, n))) / r
    g = np.array([1.0, 0.9999, 0.9996, 0.99])[rng.integers(0, 4, m)]
    Dv = stableswap_invariant_any(R, r, A)
    nu = r * np.exp((1e-3 if peg else 0.3) * rng.standard_normal((m, n))) * np.exp(rng.normal(0, 1, m))[:, None]
    return R, r, A, Dv, g, nu


def flow_tol(D, L, R, l, Hs=None, nu=None):
    """1e-10 gross + 64 u (1 + |l|) R_j, plus, given the pool's scaled Hessian Hs and prices nu, the conditioning term
    64 u sum_i |Hs_ji| / nu_j: a relative rounding u of the prices moves the exact flow of coin j by that much"""
    gross = (np.abs(D) + np.abs(L)).sum(1, keepdims=True)
    tol = 1e-10 * gross + 64 * U * (1 + np.abs(l))[:, None] * R
    if Hs is not None:
        tol = tol + 64 * U * np.abs(Hs).sum(2) / nu
    return tol


def arg_tol(R, r, A, Dv, g, nu, D, L):
    """Per slot, the rounding of stableswap_n's denominators: a traded coin's post-trade scaled balance is u_j = q / e_j,
    e_j = expm1(arg_j), where arg_j (dB_j + tau, or dB_j + log gamma + tau for a coin that shrinks) is a sum of terms of
    sizes up to log(pi_max / pi_min), |log gamma| and tau <= T = log1p(q / min u), but can itself be as small as q / u_j
    near the peg.  The terms and their two additions round by u each, and tau, the root of a Newton iteration in
    log tau, is known to u tau (2 + |log tau|): arg_j carries up to 8 u Lam, Lam = log(pi_max / pi_min) + |log gamma|
    + T (2 + |log T|), and log u_j moves by that times dlog e / darg = 1 + u_j / q.  So the flow of coin j carries
    8 u Lam (1 + u_j / q) x'_j, x' = R + gamma D - L (0 on untraded slots).
    This is the error of the representation (tau is referenced to pi_min / gamma, so the arguments of the other side's
    coins are differences), not of the problem's conditioning."""
    n = R.shape[1]
    xp = R + g[:, None] * D - L
    u = r * xp / Dv[:, None]
    q = 1.0 / (A * n ** n * n ** n * np.prod(u, 1))
    pi = nu / r
    T_ = np.log1p(q / u.min(1))
    lam = np.log(pi.max(1) / pi.min(1)) + np.abs(np.log(g)) + T_ * (2 + np.abs(np.log(T_)))
    traded = (D != 0) | (L != 0)
    return np.where(traded, 8 * U * lam[:, None] * (1 + u / q[:, None]) * xp, 0.0)


def _lq(R, r, A, Dv):
    """l0 = log(Q0 / a) per pool (the scale of the log terms)"""
    n = R.shape[1]
    u0 = r * R / Dv[:, None]
    return -(n * np.log(n) + np.log(u0).sum(1)) - np.log(A * n ** n)


def _stable_hp(R, r, A, g, toks=None, n=None):
    m, k = R.shape
    toks = np.tile(np.arange(k), (m, 1)) if toks is None else toks
    n = int(toks.max()) + 1 if n is None else n
    return HostPools(n, np.arange(0, k * m + 1, k, dtype=np.int64), np.ascontiguousarray(toks, np.int32).ravel(),
                     np.ascontiguousarray(R, np.float64).ravel(), np.ascontiguousarray(r, np.float64).ravel(),
                     np.asarray(g, np.float64), np.full(m, KIND_STABLESWAP_HOST, np.uint8), np.asarray(A, np.float64))


# ====================================================================================================== CPU
def test_invariant_matches_decimal_get_D():
    rng = np.random.default_rng(0)
    worst = 0.0
    for n in range(3, 9):
        ys, ann = [], []
        for e in (0.0, -3.0, -20.0, -100.0, -200.0):                     # one coin at 10^e of the sum, the rest mixed
            for a in (1e-3, 1.0, 100.0, 1e4, ANN_MAX):
                y = np.exp(rng.normal(0, 1, n)); y /= y.sum(); y[0] = 10.0 ** e if e else y[0]
                ys.append(y); ann.append(a)
        ys = np.array(ys); ann = np.array(ann)
        r = np.exp(rng.normal(0, 1, ys.shape))
        R = ys / r * np.exp(rng.normal(0, 5, len(ys)))[:, None]          # a variety of rates and scales
        D = stableswap_invariant_n(R, r, ann / n ** n)
        for i in range(len(ys)):
            d = _dec_get_D(R[i] * r[i], ann[i])
            rel = abs(Decimal(float(D[i])) - d) / d
            worst = max(worst, float(rel))
            assert rel <= Decimal(4e-15), (n, i, float(rel))
    print("worst relative error of D:", worst)
    # two coins: the same bits as the two-coin function, also through HostPools
    R, r, A, _, g, _ = random_pools(500, 2, 1)
    assert np.array_equal(stableswap_invariant_any(R, r, A), stableswap_invariant(R, r, A))
    assert np.array_equal(_stable_hp(R, r, A, g).inv, stableswap_invariant(R, r, A))


def _contract_get_D(xp, A_contract):
    """the published StableSwap contract iteration (integers, Ann = A() * N): D_P = D * prod(D / (x_j N))"""
    N = len(xp)
    S = sum(xp)
    D, Ann = S, A_contract * N
    for _ in range(255):
        D_P = D
        for x in xp:
            D_P = D_P * D // (x * N)
        Dprev = D
        D = (Ann * S + D_P * N) * D // ((Ann - 1) * D + (N + 1) * D_P)
        if abs(D - Dprev) <= 1:
            return D
    raise AssertionError("contract get_D did not converge")


def test_amplification_convention_matches_the_contracts():
    """A contract's A() is A n^(n-1) in the whitepaper convention these functions take: get_D of the contracts equals
    stableswap_invariant(..., A() / n^(n-1)) to integer rounding"""
    rng = np.random.default_rng(1)
    for n in (2, 3, 4):
        for A_c in (10, 100, 2000, 100000):
            for _ in range(5):
                xp = [int(v) for v in (np.exp(rng.normal(0, 0.7, n)) * 1e24)]
                Dc = _contract_get_D(xp, A_c)
                D = float(stableswap_invariant_any(np.array([xp], float), np.ones((1, n)), [A_c / n ** (n - 1)])[0])
                assert abs(D - Dc) <= 1e-14 * Dc + n, (n, A_c, D, Dc)
                if n > 2:          # taking A() as the whitepaper A models a pool n^(n-1) times more amplified
                    Dw = float(stableswap_invariant_any(np.array([xp], float), np.ones((1, n)), [float(A_c)])[0])
                    assert abs(Dw - Dc) > 1e-9 * Dc


@pytest.mark.parametrize("n", [3, 4, 6, 8])
@pytest.mark.parametrize("peg", [True, False])
def test_host_matches_xp_reference(n, peg):
    R, r, A, Dv, g, nu = random_pools(400, n, 10 * n + peg, peg=peg)
    D, L, h, mask = host_pools(R, r, A, Dv, g, nu)
    Dx, Lx, hx, _ = XN.stablen_response(R, r, A, Dv, g, nu)
    tol = flow_tol(Dx.astype(float), Lx.astype(float), R, _lq(R, r, A, Dv)) + \
        arg_tol(R, r, A, Dv, g, nu, Dx.astype(float), Lx.astype(float))
    err = np.maximum(np.abs(D - Dx.astype(float)), np.abs(L - Lx.astype(float)))
    assert np.all(err <= tol), float((err / tol).max())
    tr = (hx != 0).any(1)
    assert tr.sum() >= 300 and np.array_equal(mask != 0, tr)
    rel = np.abs(h - hx.astype(float)) / np.maximum(np.abs(hx.astype(float)), 1e-300)
    assert np.all(rel[hx != 0] <= 1e-6), float(rel[hx != 0].max())
    # feasibility of the fp64 trades, in longdouble
    # the post-trade balance x' = R + gamma D - L of a coin drained far below R carries a relative rounding of u R / x'
    xp = R + g[:, None] * D - L
    feas = XN.stablen_feasibility(R, r, A, Dv, g, D, L).astype(float)
    assert np.all(feas <= 1e-13 + 8 * U * (R / xp).max(1)), float((feas / (1e-13 + 8 * U * (R / xp).max(1))).max())
    print(f"n={n} peg={peg}: worst flow error / bound {float((err / tol).max()):.3g}")


def _dec_kkt(R, r, A, Dv, g, nu, D, L):
    """in 50-digit decimal: (relative drop of D(R') below D, spread of p_j / dG_j over the traded coordinates, worst
    band violation of the untraded ones), with mu = the traded coordinates' mean p_j / dG_j"""
    getcontext().prec = 50
    n = len(R)
    Dd = lambda v: Decimal(float(v))
    y = [Dd(r[j]) * (Dd(R[j]) + Dd(g) * Dd(D[j]) - Dd(L[j])) for j in range(n)]
    ann = Dd(A) * n ** n
    Dn = _dec_get_D(y, ann)
    drop = (Dd(Dv) - Dn) / Dd(Dv)
    u = [v / Dd(Dv) for v in y]
    Q = Decimal(1)
    for v in u:
        Q = Q / (n * v)
    dG = [ann + Q / v for v in u]
    pi = [Dd(nu[j]) / Dd(r[j]) for j in range(n)]
    tr = [j for j in range(n) if D[j] > 0 or L[j] > 0]
    p = [pi[j] / Dd(g) if D[j] > 0 else pi[j] for j in range(n)]
    mus = [p[j] / dG[j] for j in tr]
    mu = sum(mus) / len(mus)
    spread = max(abs(m_ - mu) / mu for m_ in mus)
    band = Decimal(0)
    for j in range(n):
        if j not in tr:     # pi_j <= mu dG_j <= pi_j / gamma
            band = max(band, (pi[j] - mu * dG[j]) / pi[j], (mu * dG[j] - pi[j] / Dd(g)) / pi[j])
    return float(drop), float(spread), float(band)


def test_kkt_conditions_in_decimal():
    """the returned trades are feasible (D(R') >= D(R)), equalise p_j / dG_j over the traded coordinates and leave
    the others inside their band -- checked in decimal, with no formula of the method"""
    for n, peg, seed in ((3, True, 1), (3, False, 2), (4, True, 3), (5, False, 4), (8, True, 5)):
        R, r, A, Dv, g, nu = random_pools(12, n, seed, peg=peg)
        D, L, h, mask = host_pools(R, r, A, Dv, g, nu)
        for i in np.nonzero(mask)[0]:
            drop, spread, band = _dec_kkt(R[i], r[i], A[i], Dv[i], g[i], nu[i], D[i], L[i])
            assert drop <= 1e-14 and spread <= 1e-7 and band <= 1e-7, (n, i, drop, spread, band)


def test_two_coins_match_the_pair_function():
    R, r, A, Dv, g, nu = random_pools(2000, 2, 7, peg=True)
    R2, r2, A2, Dv2, g2, nu2 = random_pools(2000, 2, 8, peg=False)
    R, r, A, Dv, g, nu = (np.concatenate([a, b]) for a, b in zip((R, r, A, Dv, g, nu), (R2, r2, A2, Dv2, g2, nu2)))
    D, L, h, mask = host_pools(R, r, A, Dv, g, nu)
    m = len(g)
    Dp, Lp, hc = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m)
    _host().stablen_host_pairs(C.c_longlong(m), *[p_(np.ascontiguousarray(x, np.float64)) for x in (R, r, A, Dv, g, nu)],
                               p_(Dp), p_(Lp), p_(hc))
    tol = flow_tol(Dp, Lp, R, _lq(R, r, A, Dv)) + arg_tol(R, r, A, Dv, g, nu, Dp, Lp)
    assert np.all(np.maximum(np.abs(D - Dp), np.abs(L - Lp)) <= tol)
    Hs = XN.hess_block(h)
    both = (hc > 0) & (mask == 3)
    assert both.sum() > 2000
    rel = np.abs(Hs[both, 0, 0] - hc[both]) / hc[both]
    assert rel.max() <= 1e-6, float(rel.max())
    # a pool one function trades and the other does not sits on the band's edge: its trade is within the tolerance of 0
    edge = (hc > 0) != (mask == 3)
    assert np.all((np.abs(Dp) + np.abs(Lp))[edge] <= tol[edge])


def test_small_A_is_the_geometric_mean_pool():
    """A -> 0: the pool becomes prod(y) >= prod(y0), the equal-weight geometric mean of the scaled balances; the trades
    differ by O(A n^n)"""
    for n in (3, 5):
        R, r, _, _, g, nu = random_pools(300, n, 20 + n, peg=False)
        for ann in (1e-6, 1e-8):
            A = np.full(len(g), ann / n ** n)
            Dv = stableswap_invariant_n(R, r, A)
            D, L, _, _ = host_pools(R, r, A, Dv, g, nu)
            Dg, Lg, _ = X._geomean(X.ld(R), X.ld(np.full_like(R, 1.0 / n)), X.ld(g), X.ld(nu))
            gross = (np.abs(Dg) + np.abs(Lg)).astype(float).sum(1, keepdims=True) + R.max(1, keepdims=True)
            err = np.maximum(np.abs(D - Dg.astype(float)), np.abs(L - Lg.astype(float)))
            assert np.all(err <= 50 * ann * gross + 1e-12 * gross), (n, ann, float((err / gross).max()))


def test_no_trade_band_is_exact():
    """prices inside the band (pi_j proportional to dG_j(u0) times a factor within [1, 1/gamma]): exactly zero"""
    rng = np.random.default_rng(3)
    for n in (3, 4, 8):
        R, r, A, Dv, g, _ = random_pools(500, n, 30 + n)
        g = np.where(g == 1.0, 0.999, g)
        u0 = r * R / Dv[:, None]
        a = A * n ** n
        Q0 = 1.0 / (n ** n * np.prod(u0, 1))
        dG = a[:, None] + Q0[:, None] / u0
        f = np.exp(rng.uniform(0.05, 0.95, (len(g), n)) * -np.log(g)[:, None])   # in (1, 1/gamma), off the edges
        nu = r * dG * f * np.exp(rng.normal(0, 1, len(g)))[:, None]
        D, L, h, mask = host_pools(R, r, A, Dv, g, nu)
        assert np.all(D == 0) and np.all(L == 0) and np.all(h == 0) and np.all(mask == 0)


def test_hessian_matches_finite_differences():
    """Hs_ij = nu_i dpsi_i / dlog nu_j by central differences of the longdouble flows (whose method shares nothing with
    the closed form of Hs); Hs 1 = 0; Hs is PSD; the host's O(k) product equals the dense block of the host's h"""
    rng = np.random.default_rng(4)
    LD = np.longdouble
    for n in (2, 3, 4, 6):
        for peg in (True, False):
            R, r, A, Dv, g, nu = random_pools(200, n, 40 + n + peg, peg=peg, ann_range=(1e-2, 1e4), at_max=False)
            _, _, hx, Hs = XN.stablen_response(R, r, A, Dv, g, nu)
            eps = LD(1e-7)
            ok = (hx != 0).any(1)
            fd = np.zeros_like(Hs)
            for j in range(n):
                up, dn = nu.astype(LD), nu.astype(LD)
                up[:, j] *= np.exp(eps); dn[:, j] *= np.exp(-eps)
                Du, Lu, hu, _ = XN.stablen_response(R, r, A, Dv, g, up)
                Dd, Ld, hd, _ = XN.stablen_response(R, r, A, Dv, g, dn)
                ok &= ((hu != 0) == (hx != 0)).all(1) & ((hd != 0) == (hx != 0)).all(1)    # the same traded set
                fd[:, :, j] = nu * ((Lu - Du) - (Ld - Dd)) / (2 * eps)
            sc = np.abs(Hs).max((1, 2))
            err = np.abs(fd - Hs).max((1, 2))
            assert ok.sum() > 150
            assert np.all(err[ok] <= 1e-6 * sc[ok]), (n, peg, float((err[ok] / sc[ok]).max()))
            assert np.all(np.abs(Hs.sum(2)) <= 1e-15 * sc[:, None] + 1e-300)
            assert np.all(np.linalg.eigvalsh(Hs.astype(float)) >= -1e-12 * sc[:, None].astype(float))
            _, _, h, _ = host_pools(R, r, A, Dv, g, nu)
            z = rng.standard_normal((len(g), n))
            Hh = XN.hess_block(h)
            sh = (h * h).max(1)[:, None]                                 # both forms round at the size of h^2
            assert np.all(np.abs(host_hvp(h, z) - np.einsum("mij,mj->mi", Hh, z)) <= 1e-13 * sh * np.abs(z).sum(1)[:, None])


# ------------------------------------------------------------------------------------------- the per-thread solver
def _small_problem(rng):
    """4-6 tokens: a product chain over all tokens plus StableSwap pools of 2, 3 and 4 coins among tokens 0..3"""
    n = int(rng.integers(4, 7))
    prices = np.exp(rng.normal(0, 1, n)); prices[:4] = [1.0, 1.001, 0.999, 1.0005]
    li, res, fees, kinds, w = [], [], [], [], []
    for i in range(n - 1):
        liq = np.exp(rng.normal(4, 1))
        li.append([i, i + 1]); res.append(list(liq / prices[[i, i + 1]] * np.exp(0.05 * rng.standard_normal(2))))
        fees.append(0.997); kinds.append("product"); w.append(None)
    for k in (3, 4, 2, int(rng.integers(2, 5))):
        t = [int(x) for x in rng.choice(4, k, replace=False)]
        V = np.exp(rng.normal(5, 1)); imb = np.exp(0.3 * rng.standard_normal(k))
        li.append(t); res.append(list(V * imb / prices[t]))
        fees.append(float(rng.choice([0.9996, 0.9999]))); kinds.append("stableswap")
        w.append((float(rng.choice([10.0, 100.0, 2000.0])) / k ** (k - 1),) + (1.0,) * k)
    d = dict(n_tokens=n, local_indices=li, reserves=res, fees=fees, kinds=kinds, weights=w)
    return HostPools.from_lists(n, li, res, fees, kinds, w), d, prices


def _utilities(rng, n, prices):
    U_ = XN.Utility
    us = [U_.arbitrage(prices * np.exp(0.01 * rng.standard_normal(n)))]
    us.append(U_.swap(n, 0, 1, float(np.exp(rng.normal(3, 1)))))
    basket = np.zeros(n); basket[1] = float(np.exp(rng.normal(2, 1))); basket[2] = float(np.exp(rng.normal(1, 1)))
    us.append(U_.liquidate(n, 0, basket))
    return us


def _csr_args(hp):
    """the cfmm_csr_pools arrays of a HostPools: kind 4's logrw = (A, D) at a pool's first two slots"""
    slot_kind = np.repeat(hp.kind, np.diff(hp.pool_ptr))
    logrw = np.log(np.maximum(hp.reserves, 1e-300) / np.where(slot_kind == 0, hp.weights, 1.0))
    ss = np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0]
    logrw[hp.pool_ptr[ss]] = hp.amp[ss]; logrw[hp.pool_ptr[ss] + 1] = hp.inv[ss]
    return [np.ascontiguousarray(x, t) for x, t in ((hp.pool_ptr, np.int64), (hp.tok_idx, np.int32),
                                                    (hp.reserves, np.float64), (hp.weights, np.float64),
                                                    (logrw, np.float64), (hp.gamma, np.float64), (hp.kind, np.uint8))]


def _host_solve(hp, specs, tol=1e-9, entry="stablen_host_solve"):
    n, B, nnz = hp.n_tokens, len(specs), len(hp.tok_idx)
    c = np.stack([u.c for u in specs]).astype(float); a = np.stack([u.a for u in specs]).astype(float)
    fl = np.ascontiguousarray(np.stack([np.asarray(u.eq, np.uint8) | (np.asarray(u.pinned, np.uint8) << 1)
                                        for u in specs]), np.uint8)
    nu = np.ascontiguousarray(np.stack([np.where(u.c > 0, u.c, np.median(u.c[u.c > 0]) if (u.c > 0).any() else 1.0)
                                        for u in specs]))
    keep = _csr_args(hp)
    psi = np.zeros((B, n)); st = np.zeros((B, 8)); d = np.zeros((B, nnz)); l = np.zeros((B, nnz))
    if entry == "stablen_host_solve":
        fn = _host().stablen_host_solve
    else:                                   # the two-coin instance, from test_stableswap.py's harness
        import test_stableswap as TS
        fn = TS._host().stableswap_host_solve
    fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 7 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
    fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), tol)
    return dict(nu=nu, psi=psi, stats=st, delta=d, lam=l)


def _as_result(hp, out, p):
    ptr = hp.pool_ptr
    return types.SimpleNamespace(value=out["stats"][p][0], dual_value=out["stats"][p][1], psi=out["psi"][p],
                                 nu=out["nu"][p], deltas=[out["delta"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                 lambdas=[out["lam"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])


def test_two_coin_instance_rejects_n_coin_pools():
    rng = np.random.default_rng(200)
    hp, _, prices = _small_problem(rng)
    out = _host_solve(hp, _utilities(rng, hp.n_tokens, prices), entry="two-coin")
    assert np.all(out["stats"][:, 7] == 3) and np.all(np.isnan(out["stats"][:, 0]))


def test_host_solver_matches_oracle_step_for_step():
    """same algorithm: same values and prices on all 24 problems, certified; the same iteration and evaluation counts
    wherever the line searches take the same path.  The oracle evaluates the pools with numpy, the solver in C++: in a
    step that the Armijo test barely accepts (or rejects) their last bits can send the two down different paths, so
    those counts are compared over the set and the number of problems whose path differs is bounded."""
    differ = []
    for seed in range(8):
        rng = np.random.default_rng(200 + seed)
        hp, _, prices = _small_problem(rng)
        assert set(np.diff(hp.pool_ptr)[hp.kind == KIND_STABLESWAP_HOST]) >= {3, 4}
        specs = _utilities(rng, hp.n_tokens, prices)
        out = _host_solve(hp, specs)
        for p, u in enumerate(specs):
            r = XN.oracle_solve(hp, u, tol=1e-9)
            st = out["stats"][p]
            assert r.status == "optimal" and int(st[7]) == 0, (seed, p, r.status, st[7])
            scale = max(abs(r.dual_value), 1e-300)
            assert abs(st[0] - r.value) <= 1e-9 * scale and abs(st[1] - r.dual_value) <= 1e-9 * scale
            np.testing.assert_allclose(out["nu"][p], r.nu, rtol=1e-7)
            if (int(st[5]), int(st[6])) != (r.iters, r.evals):
                differ.append((seed, p, (int(st[5]), int(st[6])), (r.iters, r.evals)))
            XN.certify(hp, u, _as_result(hp, out, p), 1e-9)
    print("paths that differ:", differ)
    assert len(differ) <= 4, differ


def test_validation():
    li3, fees = [[0, 1, 2]], [0.9996]
    R3 = [[10.0, 12.0, 9.0]]
    for k in range(2, 9):
        hp = HostPools.from_lists(k, [list(range(k))], [[5.0] * k], fees, ["stableswap"], [(1.0,) + (1.0,) * k])
        hp.validate()
        assert hp.inv[0] == pytest.approx(5.0 * k)
    with pytest.raises(ValueError):                               # 9 coins
        HostPools.from_lists(9, [list(range(9))], [[5.0] * 9], fees, ["stableswap"], [(1e-3,) + (1.0,) * 9])
    with pytest.raises(ValueError):                               # the weights of a two-coin pool on three coins
        HostPools.from_lists(3, li3, R3, fees, ["stableswap"], [(100.0, 1, 1)])
    for w in [(0.0, 1, 1, 1), (-1.0, 1, 1, 1), (np.nan, 1, 1, 1), (ANN_MAX / 27 * 1.001, 1, 1, 1), (100, 0, 1, 1),
              (100, 1, np.inf, 1), (100, 1, 1, 1, 1), None]:
        with pytest.raises(ValueError):
            HostPools.from_lists(3, li3, R3, fees, ["stableswap"], [w])
    HostPools.from_lists(3, li3, R3, fees, ["stableswap"], [(ANN_MAX / 27, 1, 1, 1)]).validate()
    for R in ([0.0, 1.0, 1.0], [1.0, -1.0, 2.0], [1.0, np.nan, 1.0]):
        with pytest.raises(ValueError):
            HostPools.from_lists(3, li3, [R], fees, ["stableswap"], [(100.0, 1, 1, 1)])
    hp = HostPools.from_lists(3, li3, R3, fees, ["stableswap"], [(100.0, 1, 1, 1)])
    bad = HostPools(3, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind, np.array([2e6]))
    with pytest.raises(ValueError):                               # A n^n = 5.4e7 given directly in CSR form
        bad.validate()
    for R in ([[0.0, 1.0, 1.0]], [[1.0, np.inf, 1.0]]):
        with pytest.raises(ValueError):
            check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], np.array(R))
    with pytest.raises(ValueError):
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], [[1.0, 2.0]])
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], np.array([[3.0, 4.0, 5.0]]))
    assert np.array_equal(u.reserves, [3.0, 4.0, 5.0])


def test_market_generator():
    s = I.synth_stable_n_market(3000, 40, seed=1)
    s.pop("prices")
    hp = HostPools(**s)
    hp.validate()
    ss = hp.kind == KIND_STABLESWAP_HOST
    ar = np.diff(hp.pool_ptr)
    assert set(ar[ss].tolist()) == {2, 3, 4} and np.all(hp.inv[ss] > 0)


# ====================================================================================================== GPU
gpu = pytest.mark.gpu


def _bucket(n, m, seed):
    """m pools of n coins over 48 tokens (half near the peg at up to the largest coefficient, half far from it)"""
    R1, r1, A1, _, g1, nu1 = random_pools(m // 2, n, seed, peg=True)
    R2, r2, A2, _, g2, nu2 = random_pools(m - m // 2, n, seed + 1, peg=False)
    R, r, A, g = (np.concatenate(x) for x in ((R1, R2), (r1, r2), (A1, A2), (g1, g2)))
    rng = np.random.default_rng(seed)
    n_tok = 48
    toks = np.argsort(rng.random((m, n_tok)), 1)[:, :n]
    nu_t = np.exp(rng.normal(0, 0.3, n_tok))
    # rates carry the per-pool price pattern of random_pools against the token prices
    nu_p = np.concatenate([nu1, nu2])
    r = r * nu_t[toks] / nu_p
    hp = _stable_hp(R, r, A, g, toks, n_tok)
    return hp, nu_t


_REF = {}


def _bucket_and_ref(n, m=25_000):
    """the bucket of _bucket and its longdouble reference, computed once per arity for the four kernel instances"""
    if n not in _REF:
        hp, nu = _bucket(n, m, 50 + n)
        _REF[n] = (hp, nu, XN.response(hp, nu))
    return _REF[n]


@gpu
@pytest.mark.parametrize("trades,hess", [(False, False), (True, False), (False, True), (True, True)])
def test_kernel_matches_xp_reference(trades, hess):
    """k_eval_stable_n<K> for K = 3..8 on 25k pools each (half near the peg, a quarter of those at the largest allowed
    coefficient, half far off it) against the longdouble reference: psi, arb, trades and the per-slot h"""
    import torch
    for n in range(3, 9):
        hp, nu, ref = _bucket_and_ref(n)
        st = cf.PoolStore(hp)
        assert len(st.buckets) == 1 and st.buckets[0].kind == _lib.KIND_STABLESWAP_N and st.buckets[0].arity == n
        acc = st.evaluate(torch.as_tensor(nu, dtype=torch.float64, device="cuda"), 0.0, trades=trades,
                          hess=hess).cpu().numpy()
        tok = hp.tok_idx.reshape(-1, n)
        Dx, Lx = ref["delta"].reshape(-1, n).astype(float), ref["lam"].reshape(-1, n).astype(float)
        R = hp.reserves.reshape(-1, n)
        r = hp.weights.reshape(-1, n)
        tol = flow_tol(Dx, Lx, R, _lq(R, r, hp.amp, hp.inv), ref["hslot"][n][2].astype(float), nu[tok]) + \
            arg_tol(R, r, hp.amp, hp.inv, hp.gamma, nu[tok], Dx, Lx)
        psi_x, gross, k = X.flows(hp, ref["delta"], ref["lam"])
        b_tok = np.zeros(hp.n_tokens); np.add.at(b_tok, tok.ravel(), tol.ravel())
        lim = b_tok + 4 * U * np.maximum(k.astype(float), 1) * gross.astype(float)
        assert np.all(np.abs(acc[:-1] - psi_x.astype(float)) <= lim)
        lim_arb = float((nu[tok] * tol).sum() + 4 * hp.m * U * (nu * gross.astype(float)).sum())
        assert abs(acc[-1] - float(ref["arb"].sum())) <= lim_arb
        b = st.buckets[0]
        m = b.m
        if trades:
            Dk, Lk = b.delta[:, :m].cpu().numpy().T, b.lam[:, :m].cpu().numpy().T
            assert np.all(np.maximum(np.abs(Dk - Dx), np.abs(Lk - Lx)) <= tol)
        if hess:
            hk = b.hcoef[:, :m].cpu().numpy().T
            mk = b.hmask[:m].cpu().numpy().astype(np.uint32)
            _, hx, _ = ref["hslot"][n]
            hx = hx.astype(float)
            tr = (hk != 0) & (hx != 0)
            # a slot on the edge of its band may trade in one precision and not in the other: within tol of 0 there
            edge = (hk != 0) != (hx != 0)
            assert np.all((np.abs(Dx) + np.abs(Lx))[edge] <= tol[edge]) and edge.any(1).sum() <= 0.002 * m
            rel = np.abs(hk - hx) / np.where(tr, np.abs(hx), 1.0)
            assert np.all(rel[tr] <= 1e-6), float(rel[tr].max())
            bits = (mk[:, None] >> np.arange(n)) & 1
            assert np.array_equal(bits == 1, hk != 0)
        print(f"n={n}: psi error / bound {float((np.abs(acc[:-1] - psi_x.astype(float)) / lim).max()):.3g}")


@gpu
def test_kernel_two_coins_matches_the_two_coin_kernel():
    """the same 200k two-coin pools through kind 5 (arity 2) and kind 4: flows within flow_tol, with hc's conditioning
    term and arg_tol's rounding of the n-coin denominators, and Hs_00 within 1e-6 relative of hc"""
    import torch
    hp, nu = _bucket(2, 200_000, 5)
    st4 = cf.PoolStore(hp)
    assert st4.buckets[0].kind == _lib.KIND_STABLESWAP
    st5 = cf.PoolStore(hp)
    b = cf.pools.DeviceBucket(hp, cf.pools.BucketSpec(hp, _lib.KIND_STABLESWAP_N, 2, None), st5.device)
    st5.buckets = [b]
    nu_d = torch.as_tensor(nu, dtype=torch.float64, device="cuda")
    a4 = st4.evaluate(nu_d, 0.0, trades=True, hess=True).cpu().numpy()
    a5 = st5.evaluate(nu_d, 0.0, trades=True, hess=True).cpu().numpy()
    m = hp.m
    R = hp.reserves.reshape(-1, 2)
    D4, L4 = st4.buckets[0].delta[:, :m].cpu().numpy().T, st4.buckets[0].lam[:, :m].cpu().numpy().T
    D5, L5 = b.delta[:, :m].cpu().numpy().T, b.lam[:, :m].cpu().numpy().T
    hc = st4.buckets[0].hcoef[:m].cpu().numpy()
    H2 = hc[:, None, None] * np.array([[1.0, -1.0], [-1.0, 1.0]])
    r2, nu2 = hp.weights.reshape(-1, 2), nu[hp.tok_idx.reshape(-1, 2)]
    tol = flow_tol(D4, L4, R, _lq(R, r2, hp.amp, hp.inv), H2, nu2) + arg_tol(R, r2, hp.amp, hp.inv, hp.gamma, nu2, D4, L4)
    # a pool on the edge of its band may trade by one method and not by the other: its trade is within tol of 0
    edge = (hc > 0) != (b.hmask[:m].cpu().numpy() != 0)
    err = np.maximum(np.abs(D4 - D5), np.abs(L4 - L5))
    assert np.all(err[~edge] <= tol[~edge]) and np.all((np.abs(D4) + np.abs(L4))[edge] <= tol[edge] + 1e-12)
    Hs = XN.hess_block(b.hcoef[:, :m].cpu().numpy().T)
    both = (hc > 0) & (Hs[:, 0, 0] > 0)
    assert np.all(np.abs(Hs[both, 0, 0] - hc[both]) <= 1e-6 * hc[both])
    assert abs(a4[-1] - a5[-1]) <= 1e-9 * np.abs(a4[-1]) + 1e-9


@gpu
def test_hessian_kernels_agree():
    """HVP = the dense matrix times v, and the diagonal = the dense diagonal, per arity and over a mixed store"""
    import torch
    rng = np.random.default_rng(0)
    s = I.synth_stable_n_market(60_000, 200, seed=3, arities=(2, 3, 4, 6, 8))
    prices = s.pop("prices")
    hp = HostPools(**s)
    st = cf.PoolStore(hp)
    kinds = {(int(b.kind), int(b.arity)) for b in st.buckets}
    assert {(_lib.KIND_STABLESWAP, 2), (_lib.KIND_STABLESWAP_N, 3), (_lib.KIND_STABLESWAP_N, 8)} <= kinds
    nu = torch.as_tensor(prices * np.exp(0.01 * rng.standard_normal(hp.n_tokens)), dtype=torch.float64, device="cuda")
    st.evaluate(nu, 0.0, trades=False, hess=True)
    H = st.hess_dense().cpu().numpy()
    v = rng.standard_normal(hp.n_tokens)
    y = st.hvp(torch.as_tensor(v, dtype=torch.float64, device="cuda")).cpu().numpy()
    sc = np.abs(H).max()
    np.testing.assert_allclose(y, H @ v, rtol=0, atol=1e-11 * sc * np.abs(v).sum())
    np.testing.assert_allclose(st.hess_diag().cpu().numpy(), np.diag(H), rtol=1e-9, atol=1e-12 * sc)
    np.testing.assert_allclose(H, H.T, rtol=0, atol=1e-12 * sc)
    assert np.abs(H.sum(1)).max() <= 1e-9 * sc                   # every pool block has Hs 1 = 0


def _mixed(m, n, seed, arities=(2, 3, 4)):
    s = I.synth_stable_n_market(m, n, seed, arities=arities)
    prices = s.pop("prices")
    return HostPools(**s), prices


def _specs(n, prices, rng):
    basket = np.zeros(n)
    for j in rng.choice(np.arange(1, n), 6, replace=False):
        basket[j] = float(np.exp(rng.normal(1, 1)) * 100 / prices[j])
    return [cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(n))), cf.Liquidate(0, basket),
            cf.Swap(1, 3, 5e3 / prices[1])]


@gpu
@pytest.mark.parametrize("linear_solver", ["dense", "cg"])
def test_mixed_market_certifies_through_solver_py(linear_solver):
    hp, prices = _mixed(60_000, 300, 4)
    store = cf.PoolStore(hp)
    assert _lib.KIND_STABLESWAP_N in {int(b.kind) for b in store.buckets}
    rng = np.random.default_rng(1)
    for u in _specs(hp.n_tokens, prices, rng):
        r = cf.solve_pools(hp, u, tol=1e-8, store=store, linear_solver=linear_solver)
        assert r.status == "optimal", r.status
        assert r.info.history
        rep = XN.certify(hp, u.spec(hp.n_tokens), r, 1e-8)
        print(f"CERT {linear_solver} {type(u).__name__} iters={r.iters} evals={r.evals} hvps={r.hvps} "
              + " ".join(f"{k}={v[0]:.2e}/{v[1]:.2e}" for k, v in rep.items() if isinstance(v, tuple)))


@gpu
def test_per_thread_solver_and_every_entry():
    """small problems with 2-, 3- and 4-coin pools through the per-thread solver (both lane counts), solve_pools,
    solve, solve_sweep and solve_many, certified; and a 3pool-like pool given as (A, 1, 1, 1)"""
    import torch
    from cfmm_routing_code_b200 import batch as B
    rng = np.random.default_rng(3)
    probs = [_small_problem(rng) for _ in range(5)]
    for lanes in (1, 32):
        for hp, d, prices in probs:
            us = [cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(hp.n_tokens))),
                  cf.Swap(0, 1, 20.0), cf.Liquidate(0, np.r_[0.0, 5.0, 3.0, np.zeros(hp.n_tokens - 3)])]
            store = B.CsrStore(hp)
            assert store.has_stableswap_n
            c, a, fl, nu = B.pack_utilities(us, hp.n_tokens)
            up = lambda x: torch.as_tensor(x, device="cuda")
            nu_d = up(nu)
            psi, stats, dl, lm = B.solve_batch_device(store, up(c), up(a), up(fl), nu_d, tol=1e-9, lanes=lanes)
            stats, psi, nu_h = stats.cpu().numpy(), psi.cpu().numpy(), nu_d.cpu().numpy()
            dl, lm = dl.cpu().numpy(), lm.cpu().numpy()
            ptr = hp.pool_ptr
            for p, u in enumerate(us):
                assert int(stats[p][7]) == 0, (lanes, p, stats[p])
                res = types.SimpleNamespace(value=stats[p][0], dual_value=stats[p][1], psi=psi[p], nu=nu_h[p],
                                            deltas=[dl[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                            lambdas=[lm[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])
                XN.certify(hp, u.spec(hp.n_tokens), res, 1e-9)
                if lanes == 1:
                    rp = cf.solve_pools(hp, u, tol=1e-9, method="pools")
                    assert rp.status == "optimal" and rp.info.history
                    XN.certify(hp, u.spec(hp.n_tokens), rp, 1e-9)
                    assert abs(rp.value - stats[p][0]) <= 1e-8 * abs(rp.dual_value)
    hp, d, prices = probs[0]
    sw = [cf.Swap(0, 1, t) for t in np.linspace(1.0, 400.0, 8)]
    rb = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], sw, batched=True)
    ru = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], sw, batched=False)
    for x, y in zip(rb, ru):
        assert x.status == y.status == "optimal"
        assert abs(x.value - y.value) <= 1e-7 * max(abs(x.dual_value), 1.0)
    many = cf.solve_many([(hp, cf.Swap(0, 1, 20.0)) for hp, _, _ in probs])
    assert all(r.status == "optimal" for r in many)
    # 3pool: DAI / USDC / USDT in one pool (A() = 2000 -> whitepaper A = 2000 / 9), traded against product pools
    li = [[0, 1, 2], [0, 1], [1, 2], [0, 2]]
    R = [[1.0e6, 0.9e6, 1.1e6], [1e6, 1.01e6], [1e6, 0.99e6], [2e6, 2e6]]
    kinds, w = ["stableswap", "product", "product", "product"], [(2000.0 / 9, 1.0, 1.0, 1.0), None, None, None]
    fees = [0.9999, 0.997, 0.997, 0.997]
    hp3 = HostPools.from_lists(3, li, R, fees, kinds, w)
    for u in (cf.Swap(0, 2, 1e4), cf.Swap(2, 1, 3e4), cf.Liquidate(0, np.array([0.0, 2e4, 1e4]))):
        for method in ("thread", "pools"):
            r = cf.solve(li, R, fees, kinds, w, utility=u, method=method)
            assert r.status == "optimal", (method, type(u).__name__, r.status)
            XN.certify(hp3, u.spec(3), r, 1e-8)
            assert np.abs(r.deltas[0]).sum() + np.abs(r.lambdas[0]).sum() > 0


@gpu
def test_update_pools_equals_a_fresh_store_and_resolves():
    import torch
    hp, prices = _mixed(60_000, 200, 8, arities=(2, 3, 4, 5, 6, 7, 8))
    store = cf.PoolStore(hp)
    u = cf.Arbitrage(prices)
    r0 = cf.solve_pools(hp, u, tol=1e-8, store=store)
    rng = np.random.default_rng(2)
    ids = np.sort(rng.choice(hp.m, 4000, replace=False))
    ar = np.diff(hp.pool_ptr)[ids]
    newR = [hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] * np.exp(0.05 * rng.standard_normal(k))
            for i, k in zip(ids, ar)]
    newg = np.where(hp.kind[ids] == KIND_STABLESWAP_HOST, 0.9998, 0.997)
    store.update_pools(ids, reserves=newR, fees=newg)
    R2 = hp.reserves.copy(); g2 = hp.gamma.copy()
    for i, x in zip(ids, newR):
        R2[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] = x
    g2[ids] = newg
    hp2 = HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, R2, hp.weights, g2, hp.kind, hp.amp)
    fresh = cf.PoolStore(hp2)
    for k in range(3, 9):                          # every coin count's D recomputed in place (n = 8: 8-wide sums)
        assert ((hp2.kind[ids] == KIND_STABLESWAP_HOST) & (ar == k)).sum() > 50, k
    for a, b in zip(store.buckets, fresh.buckets):
        assert (a.kind, a.arity) == (b.kind, b.arity)
        if getattr(a, "blocked", False):
            for t in ("r0", "r1", "gamma_inv"):
                assert torch.equal(getattr(a, t), getattr(b, t))
            continue
        for t in ("reserves", "gamma", "weights", "logrw"):
            x, y = getattr(a, t), getattr(b, t)
            assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), (a.kind, t)
    r1 = cf.solve_pools(hp2, u, tol=1e-8, store=store, nu0=r0.nu)
    assert r1.status == "optimal"
    XN.certify(hp2, u.spec(hp.n_tokens), r1, 1e-8)


@gpu
def test_buckets_and_c_abi():
    """two-coin pools stay in a kind-4 bucket; kind 5 takes arity 2..8 and refuses the rest; kind 4 still refuses 3"""
    import torch
    hp, _ = _mixed(20_000, 100, 9)
    st = cf.PoolStore(hp)
    ka = sorted((int(b.kind), int(b.arity)) for b in st.buckets if b.kind in (_lib.KIND_STABLESWAP, _lib.KIND_STABLESWAP_N))
    assert ka == [(_lib.KIND_STABLESWAP, 2), (_lib.KIND_STABLESWAP_N, 3), (_lib.KIND_STABLESWAP_N, 4)]
    lib = _lib.load()
    buf = torch.ones(8 * 1024, dtype=torch.float64, device="cuda")
    idx = torch.zeros(8 * 1024, dtype=torch.int32, device="cuda")
    nu = torch.ones(4, dtype=torch.float64, device="cuda")
    acc = torch.zeros(5, dtype=torch.float64, device="cuda")
    p = buf.data_ptr()

    def ev(kind, arity, w, lr):
        b = _lib.Bucket(kind, arity, 100, 1024, p, idx.data_ptr(), p, w, lr, None)
        return lib.cfmm_arb_eval(C.byref(b), 4, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc.data_ptr() + 32, None, None)
    assert ev(_lib.KIND_STABLESWAP, 3, p, p) == -2
    for k in (1, 9):
        assert ev(_lib.KIND_STABLESWAP_N, k, p, p) == -2
    assert ev(_lib.KIND_STABLESWAP_N, 3, None, p) == -1 and ev(_lib.KIND_STABLESWAP_N, 3, p, None) == -1
    for k in range(2, 9):
        assert ev(_lib.KIND_STABLESWAP_N, k, p, p) == 0
    torch.cuda.synchronize()
