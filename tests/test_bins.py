"""Price-bin pools: Liquidity Book bins, order books and limit orders as one pool kind (host kind 10, CFMM_KIND_BINS).

CPU: the records and the validation rules; cfmm_small::bins_pair compiled for the host against the longdouble reference
(tests/xp_bins.py: every bin walked on its own, no records, no search) at eps = 0 and eps > 0, its hc against central
differences; the per-thread solver's bins instance (host build) against scipy's HiGHS on bins-only LPs, certified by
xp_bins; bin_fills; instances.lb_bins and order_book against decimal.
GPU (H100): k_eval_bins in all four (trades, hess) instances against the reference, the Hessian kernels; the reference
scripts' constant-sum pool written as a one-bin pool on every solve path; bins markets against linprog, against their
bins_split form and against constant-sum pools; mixed markets of every kind, certified; a 100k-pool market; units;
rank stores; fee updates; C ABI codes.

Error bounds.  Both sides read the same f64 prices and holdings.  The records hold each cumulative sum rounded once
from extended precision, and a flow is one record plus at most one product of a slope and a partial width, then divided
or multiplied by gamma: a few ulp of the pool's capacity in that token (sum x and S_bid for token 0, sum y and
sum p x / gamma for token 1).  The tests allow 1e-12 of that capacity, masking pools whose price ratio is within 1e-12
(relative) of a segment's slope, where the exact answer flips between two breakpoints.
"""
import ctypes as C
import dataclasses
import os
import subprocess
import types
from decimal import Decimal, getcontext

import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib, instances as I
from cfmm_routing_code_b200.pools import (BINS_K_MAX, HostPools, KIND_BINS_HOST, bin_fills, bin_records,
                                          check_pool_update)
import xp_bins as XB
import xp_reference as X

HERE = os.path.dirname(os.path.abspath(__file__))
p_ = lambda x: x.ctypes.data_as(C.c_void_p)
_HOST = None


def _host():
    """tests/host_harness/bins_host.cpp: cfmm_small::bins_pair and the solver's bins instance, host build"""
    global _HOST
    if _HOST is None:
        src = os.path.join(HERE, "host_harness", "bins_host.cpp")
        hdr = os.path.join(HERE, "..", "cfmm_routing_code_b200", "csrc", "cfmm_small.cuh")
        lib = os.path.join(HERE, "_build", "libbins_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src],
                           check=True)
        _HOST = C.CDLL(lib)
    return _HOST


def random_bins(rng, K, mode=None):
    """(prices, x, y) of K bins: geometric prices anywhere in 1e-6 .. 1e6, holdings log-normal; mode 'ask' / 'bid'
    (one-sided), 'both' (an active bin holding both tokens) or 'gap' (a spread between the sides)"""
    mode = mode or rng.choice(["ask", "bid", "both", "gap"])
    step = np.exp(rng.uniform(np.log(1e-4), np.log(0.05)))
    lo = rng.uniform(np.log(1e-6), np.log(1e6) - K * step)
    p = np.exp(lo + step * np.arange(K))
    p = np.maximum.accumulate(p)
    v = np.exp(rng.uniform(-3, 6, K))
    act = int(rng.integers(0, K))
    x = np.where(np.arange(K) > act, v / p, 0.0)
    y = np.where(np.arange(K) < act, v, 0.0)
    if mode == "ask":
        x, y = v / p, np.zeros(K)
    elif mode == "bid":
        x, y = np.zeros(K), v
    elif mode == "both":
        x[act], y[act] = 0.4 * v[act] / p[act], 0.6 * v[act]
    if not (x.any() or y.any()):                  # one bin and a gap: the bin holds token 0
        x[act] = v[act] / p[act]
    return p, x, y


def _pool_args(pools):
    """records, P [m][4] (first, nb, z, p_ref) of a list of (prices, x, y)"""
    recs, P, first = [], [], 0
    for p, x, y in pools:
        r, z, pref, _ = bin_records(p, x, y)
        recs.append(r); P.append((first, len(r), z, pref)); first += len(r)
    return np.ascontiguousarray(np.concatenate(recs)), np.ascontiguousarray(np.asarray(P, np.float64))


def host_pairs(pools, g, n0, n1, eps, tbar):
    rec, P = _pool_args(pools)
    m = len(pools)
    D, L, hc, t = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m), np.zeros(m)
    f = _host().bins_host_pools
    f.argtypes = [C.c_longlong] + [C.c_void_p] * 6 + [C.c_double] + [C.c_void_p] * 4
    f(m, p_(rec), p_(P), p_(np.ascontiguousarray(tbar, float)), p_(np.ascontiguousarray(g, float)),
      p_(np.ascontiguousarray(n0, float)), p_(np.ascontiguousarray(n1, float)), eps, p_(D), p_(L), p_(hc), p_(t))
    return D, L, hc, t


def _scales(p, x, y, g):
    """capacity scales of the two tokens: (sum x + S_bid, sum y + sum p x / gamma)"""
    return x.sum() + (y / (g * p)).sum(), y.sum() + (p * x).sum() / g


def _near_slope(p, x, y, g, r, tol=1e-12):
    s = np.concatenate([p[x > 0] / g, g * p[y > 0]])
    return bool(np.any(np.abs(r - s) <= tol * s))


def _case_pools(rng, n, Ks=(1, 2, 5, 40)):
    out = []
    for q in range(n):
        K = int(Ks[q % len(Ks)])
        p, x, y = random_bins(rng, K)
        g = 1.0 if q % 3 == 0 else float(rng.choice([0.9999, 0.997, 0.99]))
        out.append((p, x, y, g))
    return out


def _prices_for(rng, p, x, y, g, tie, near=0.0):
    """(n0, n1): a random price ratio across the pool's range, exactly one bin's price (tie; n1 = 1, so r is that price:
    with gamma = 1, r on a slope), or within a relative `near` of one bin's price"""
    if tie:
        return float(p[int(rng.integers(0, len(p)))]), 1.0
    n1 = float(np.exp(rng.uniform(-3, 3)))
    if near:
        return float(p[int(rng.integers(0, len(p)))] * np.exp(near * rng.standard_normal())) * n1, n1
    return float(np.exp(rng.uniform(np.log(p[0]) - 0.05, np.log(p[-1]) + 0.05))) * n1, n1


def test_bins_pair_exact_against_reference():
    rng = np.random.default_rng(1)
    cases = _case_pools(rng, 400)
    n0 = np.zeros(len(cases)); n1 = np.zeros(len(cases)); ties = np.zeros(len(cases), bool)
    for q, (p, x, y, g) in enumerate(cases):
        ties[q] = g == 1.0 and q % 2 == 0
        n0[q], n1[q] = _prices_for(rng, p, x, y, g, ties[q])
    D, L, hc, t = host_pairs([c[:3] for c in cases], [c[3] for c in cases], n0, n1, 0.0, np.zeros(len(cases)))
    assert np.all(hc == 0)
    checked = 0
    for q, (p, x, y, g) in enumerate(cases):
        if not ties[q] and _near_slope(p, x, y, g, n0[q] / n1[q]):
            continue
        Dx, Lx = XB.exact(p, x, y, g, n0[q], n1[q])
        s0, s1 = _scales(p, x, y, g)
        assert abs(float(Dx[0]) - D[q, 0]) <= 1e-12 * s0 and abs(float(Lx[0]) - L[q, 0]) <= 1e-12 * s0, q
        assert abs(float(Dx[1]) - D[q, 1]) <= 1e-12 * s1 and abs(float(Lx[1]) - L[q, 1]) <= 1e-12 * s1, q
        checked += 1
    assert checked >= 350 and ties.sum() >= 50


def test_bins_pair_smoothed_against_reference_and_hc_by_differences():
    rng = np.random.default_rng(2)
    cases = _case_pools(rng, 200)
    m = len(cases)
    n0 = np.zeros(m); n1 = np.zeros(m); tbar = np.zeros(m)
    for q, (p, x, y, g) in enumerate(cases):
        n0[q], n1[q] = _prices_for(rng, p, x, y, g, False, near=[0.0, 1e-3, 1e-5][q % 3])
        lo, hi = -(y / (g * p)).sum(), x.sum()
        tbar[q] = 0.0 if q % 4 == 0 else rng.uniform(lo, hi)
    for eps in (0.1, 1e-3):
        D, L, hc, t = host_pairs([c[:3] for c in cases], [c[3] for c in cases], n0, n1, eps, tbar)
        for q, (p, x, y, g) in enumerate(cases):
            _, z, pref, _ = bin_records(p, x, y)
            tx, cx = XB.smoothed(p, x, y, g, n0[q], n1[q], eps, tbar[q], pref)
            s0, s1 = _scales(p, x, y, g)
            assert abs(float(tx) - t[q]) <= 1e-12 * s0, (eps, q, float(tx), t[q])
            assert abs(float(tx) - (L[q, 0] - D[q, 0])) <= 1e-12 * s0
            assert abs(float(-cx) - (L[q, 1] - D[q, 1])) <= 1e-12 * s1 * max(1.0, 1.0 / eps), (eps, q)
        # hc: nu0 dt / dlog nu0 by central differences, away from breakpoints
        d = 1e-7
        _, _, hp_, tp = host_pairs([c[:3] for c in cases], [c[3] for c in cases], n0 * np.exp(d), n1, eps, tbar)
        _, _, hm_, tm = host_pairs([c[:3] for c in cases], [c[3] for c in cases], n0 * np.exp(-d), n1, eps, tbar)
        inside = (hc > 0) & (hp_ > 0) & (hm_ > 0)
        fd = n0 * (tp - tm) / (2 * d)
        assert inside.sum() >= 10
        np.testing.assert_allclose(hc[inside], fd[inside], rtol=1e-5)
        assert np.all(hc[(hp_ == 0) & (hm_ == 0)] == 0)


def test_bins_pair_large_pool():
    """K = 2^16 bins and K = 1, both sides, many price ratios"""
    rng = np.random.default_rng(3)
    for K in (1 << 16, 1):
        p, x, y = random_bins(rng, K, "both")
        for g in (1.0, 0.997):
            n1 = np.ones(64)
            n0 = np.exp(rng.uniform(np.log(p[0]) - 0.01, np.log(p[-1]) + 0.01, 64))
            D, L, _, _ = host_pairs([(p, x, y)] * 64, np.full(64, g), n0, n1, 0.0, np.zeros(64))
            s0, s1 = _scales(p, x, y, g)
            for q in range(64):
                if _near_slope(p, x, y, g, n0[q]):
                    continue
                Dx, Lx = XB.exact(p, x, y, g, n0[q], 1.0)
                assert np.all(np.abs(np.asarray(Dx, float) - D[q]) <= 1e-12 * np.array([s0, s1]))
                assert np.all(np.abs(np.asarray(Lx, float) - L[q]) <= 1e-12 * np.array([s0, s1]))


def test_records_layout():
    p, x, y = np.array([1.0, 2.0, 3.0, 4.0]), np.array([0.0, 0.0, 1.0, 2.0]), np.array([5.0, 6.0, 3.0, 0.0])
    rec, z, pref, sums = bin_records(p, x, y)
    assert z == 3 and pref == 3.0 and sums == (3.0, 14.0)
    # bids outward from t = 0: 3 / 3, 6 / 2, 5 / 1 of token 0; asks: 1, then 2 more
    np.testing.assert_allclose(rec[:, 0], [-(1.0 + 3.0 + 5.0), -(1.0 + 3.0), -1.0, 0.0, 1.0, 3.0])
    np.testing.assert_allclose(rec[:, 1], [-14.0, -9.0, -3.0, 0.0, 3.0, 11.0])
    np.testing.assert_array_equal(rec[:, 2], [1.0, 2.0, 3.0, 3.0, 4.0, 0.0])
    np.testing.assert_array_equal(rec[:, 3], [0, 1, 2, 2, 3, -1])


def test_validation():
    ok = lambda w, R=None, li=(0, 1): HostPools.from_lists(2, [list(li)], [R], [0.997], ["bins"], [w])
    ok(([1.0, 2.0], [0.0, 1.0], [1.0, 0.0])).validate()
    ok(([2.0], [1.0], [1.0])).validate()
    bad = [(([2.0, 1.0], [0, 1.0], [1.0, 0]), None, (0, 1)),          # decreasing prices
           (([1.0, 1.0], [0, 1.0], [1.0, 0]), None, (0, 1)),          # repeated price
           (([0.0, 1.0], [0, 1.0], [1.0, 0]), None, (0, 1)),          # price 0
           (([1.0, np.inf], [0, 1.0], [1.0, 0]), None, (0, 1)),
           (([1.0, 2.0], [1.0, 0.0], [0.0, 1.0]), None, (0, 1)),      # crossed
           (([1.0, 2.0], [-1.0, 1.0], [0.0, 0.0]), None, (0, 1)),     # negative
           (([1.0, 2.0], [np.nan, 1.0], [0.0, 0.0]), None, (0, 1)),
           (([1.0, 2.0], [0.0, 0.0], [0.0, 0.0]), None, (0, 1)),      # all zero
           (([1.0, 2.0], [0.0, 1.0]), None, (0, 1)),                  # not a triple
           (([1.0, 2.0], [0.0, 1.0], [1.0]), None, (0, 1)),           # lengths
           (([1.0], [1.0], [0.0]), [1.0, 0.0], (0, 1)),                # reserves given
           (([1.0], [1.0], [0.0]), None, (0, 0)),                      # one token
           (([1.0], [1.0], [0.0]), None, (0, 1, 2))]                   # three tokens
    for w, R, li in bad:
        with pytest.raises(ValueError):
            ok(w, R, li)
    with pytest.raises(ValueError):
        ok((np.arange(1, BINS_K_MAX + 2, dtype=float), np.ones(BINS_K_MAX + 1), np.zeros(BINS_K_MAX + 1)))
    hp = ok(([1.0, 2.0], [0.0, 1.0], [1.0, 0.0]))
    for broken in (dict(bin_zp=np.array([[0.0, 1.0]])), dict(bin_zp=np.array([[1.0, -1.0]])),
                   dict(bin_rec=hp.bin_rec[::-1].copy())):
        with pytest.raises(ValueError):
            dataclasses.replace(hp, **broken).validate()
    with pytest.raises(ValueError):
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], reserves=[[1.0, 1.0]])
    check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], fees=[0.99])


def test_bin_fills_sum_to_flows_and_are_feasible():
    rng = np.random.default_rng(4)
    for q in range(60):
        p, x, y = random_bins(rng, int(rng.choice([1, 3, 30])))
        g = float(rng.choice([1.0, 0.997]))
        hp = HostPools.from_lists(2, [[0, 1]], [None], [g], ["bins"], [(p, x, y)])
        n0 = float(np.exp(rng.uniform(np.log(p[0]) - 0.02, np.log(p[-1]) + 0.02)))
        if _near_slope(p, x, y, g, n0):
            continue
        D, L = (np.asarray(v, float) for v in XB.exact(p, x, y, g, n0, 1.0))
        t = L[0] - D[0]
        bins, f0, f1 = bin_fills(hp, 0, t)
        s0, s1 = _scales(p, x, y, g)
        assert abs(f0.sum() - t) <= 1e-12 * s0 and abs(f1.sum() - (L[1] - D[1])) <= 1e-12 * s1
        for k, a, b in zip(bins, f0, f1):                         # each bin's own constant-sum set, at its price
            if a > 0:
                assert a <= x[k] + 1e-12 * s0 and -b * g >= p[k] * a - 1e-12 * s1
            else:
                assert b <= y[k] + 1e-12 * s1 and b <= g * p[k] * -a + 1e-12 * s1
        assert len(set(bins.tolist())) == len(bins)
    with pytest.raises(ValueError):
        bin_fills(HostPools.from_lists(2, [[0, 1]], [[1.0, 1.0]], [1.0], ["product"]), 0, 0.1)


def test_lb_bins_and_order_book_against_decimal():
    getcontext().prec = 50
    ids = [8388600, 8388607, 8388608, 8388609, 8388650]
    rx = [0, 0, 3 * 10 ** 17, 10 ** 18, 5 * 10 ** 18]
    ry = [7 * 10 ** 6, 2 * 10 ** 6, 10 ** 6, 0, 0]
    p, x, y = I.lb_bins(8388608, 25, ids, rx, ry, 18, 6)
    for k, i in enumerate(ids):
        ref = (Decimal(1) + Decimal(25) / Decimal(10000)) ** (i - 2 ** 23) * Decimal(10) ** 12
        assert p[k] == float(ref)
        assert x[k] == float(Decimal(rx[k]) / Decimal(10) ** 18) and y[k] == float(Decimal(ry[k]) / Decimal(10) ** 6)
    HostPools.from_lists(2, [[0, 1]], [None], [0.998], ["bins"], [(p, x, y)]).validate()
    with pytest.raises(ValueError):
        I.lb_bins(8388608, 25, ids, [1] + rx[1:], ry, 18, 6)      # X below the active bin
    with pytest.raises(ValueError):
        I.lb_bins(8388608, 25, ids, rx, ry[:4] + [1], 18, 6)      # Y above it
    p, x, y = I.order_book([(1.9, 2.0), (2.0, 1.0), (1.9, 0.5)], [(2.1, 3.0), (2.2, 0.25)])
    np.testing.assert_array_equal(p, [1.9, 2.0, 2.1, 2.2])
    np.testing.assert_array_equal(x, [0, 0, 3.0, 0.25])
    assert y[0] == 1.9 * 2.0 + 1.9 * 0.5 and y[1] == 2.0 and y[2] == y[3] == 0
    with pytest.raises(ValueError):
        I.order_book([(2.2, 1.0)], [(2.1, 1.0)])
    p, x, y = I.order_book([(2.0, 1.0)], [(2.0, 1.0)])            # a bid and an ask at one price share a bin
    assert len(p) == 1 and x[0] == 1.0 and y[0] == 2.0


# ---------------------------------------------------------------------------------------------------------------------
# the per-thread solver's bins instance (host build) against HiGHS on LPs

def _csr_args(hp):
    """the cfmm_csr_pools arrays and the records, as CsrStore writes them (no concentrated pools here)"""
    w = hp.weights.copy()
    slot_kind = np.repeat(hp.kind, np.diff(hp.pool_ptr))
    logrw = np.log(np.maximum(hp.reserves, 1e-300) / np.where(slot_kind == 0, hp.weights, 1.0))
    bn = np.nonzero(hp.kind == KIND_BINS_HOST)[0]
    f = hp.pool_ptr[bn]
    w[f], w[f + 1] = hp.bin_zp[bn, 0], hp.bin_zp[bn, 1]
    logrw[f], logrw[f + 1] = hp.bin_ptr[bn], hp.bin_ptr[bn + 1] - hp.bin_ptr[bn]
    rec = np.ascontiguousarray(hp.bin_rec if len(hp.bin_rec) else np.zeros((1, 4)))
    return [np.ascontiguousarray(x, t) for x, t in ((hp.pool_ptr, np.int64), (hp.tok_idx, np.int32),
                                                    (hp.reserves, np.float64), (w, np.float64), (logrw, np.float64),
                                                    (hp.gamma, np.float64), (hp.kind, np.uint8))] + [rec]


def _host_solve(hp, specs, tol=1e-9):
    n, B, nnz = hp.n_tokens, len(specs), len(hp.tok_idx)
    c = np.stack([u.c for u in specs]).astype(float); a = np.stack([u.a for u in specs]).astype(float)
    fl = np.ascontiguousarray(np.stack([np.asarray(u.eq, np.uint8) | (np.asarray(u.pinned, np.uint8) << 1)
                                        for u in specs]), np.uint8)
    nu = np.ascontiguousarray(np.stack([np.where(u.c > 0, u.c, np.median(u.c[u.c > 0]) if (u.c > 0).any() else 1.0)
                                        for u in specs]))
    keep = _csr_args(hp)
    psi = np.zeros((B, n)); st = np.zeros((B, 8)); d = np.zeros((B, nnz)); l = np.zeros((B, nnz))
    fn = _host().bins_host_solve
    fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 8 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
    fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), tol)
    return dict(nu=nu, psi=psi, stats=st, delta=d, lam=l)


def _result(hp, out, p):
    ptr = hp.pool_ptr
    return types.SimpleNamespace(value=out["stats"][p][0], dual_value=out["stats"][p][1], psi=out["psi"][p],
                                 nu=out["nu"][p], deltas=[out["delta"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                 lambdas=[out["lam"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])


def lp_value(pools, n, spec):
    """max c'psi over the bins' constant-sum sets (each bin its own variables) and the token box of spec, by HiGHS.
    pools: [(i, j, prices, x, y, gamma)] (sum pools as one bin at price 1)"""
    from scipy.optimize import linprog
    cols, A = [], []                 # per bin and direction: one variable u >= 0 (token tendered before the fee)
    ub = []
    for (i, j, p, x, y, g) in pools:
        for k in range(len(p)):
            if x[k] > 0:             # tender token j, receive token i: u of j buys g u / p of i, up to x
                col = np.zeros(n); col[j] -= 1.0; col[i] += g / p[k]; A.append(col); ub.append(x[k] * p[k] / g)
            if y[k] > 0:             # tender token i, receive token j: u of i buys g p u of j, up to y
                col = np.zeros(n); col[i] -= 1.0; col[j] += g * p[k]; A.append(col); ub.append(y[k] / (g * p[k]))
    M = np.array(A).T                # psi = M u
    c, a = np.asarray(spec.c, float), np.asarray(spec.a, float)
    eq, pin = np.asarray(spec.eq, bool), np.asarray(spec.pinned, bool)
    ineq = ~eq & ~pin
    res = linprog(-(c @ M), A_ub=-M[ineq], b_ub=a[ineq], A_eq=M[eq] if eq.any() else None,
                  b_eq=-a[eq] if eq.any() else None, bounds=[(0, u) for u in ub], method="highs")
    assert res.status == 0, res.message
    return -res.fun


def bins_lp_market(rng, n=4, m=6, with_sum=True, cycles=False):
    """a connected market of bins pools (and constant-sum pools) on n tokens: (local_indices, kinds, weights, fees, lp
    pools, prices).  Without cycles every pool bids below and asks above the tokens' price ratio and constant-sum pools
    join tokens 2 and 3 of equal price: the market for Swap, Liquidate and the linear utility (with arbitrage cycles a
    linear market's optimum can leave a token worthless, a price no positive-price dual method reaches).  With cycles
    every pool's mid is 10 % off: the market for Arbitrage, which is worth 0 without them."""
    prices = np.exp(rng.standard_normal(n))
    prices[3] = prices[2]
    li, kinds, w, R, fees, lp = [], [], [], [], [], []
    for q in range(m):
        i, j = (q % n, (q + 1) % n) if q < n else tuple(rng.choice(n, 2, replace=False))
        g = float(rng.choice([1.0, 0.997]))
        if with_sum and q % 3 == 2:
            Rs = np.exp(rng.uniform(0, 3, 2))
            li.append([2, 3]); kinds.append("sum"); w.append(None); R.append(list(Rs)); fees.append(g)
            lp.append((2, 3, np.array([1.0]), Rs[:1], Rs[1:], g))
            continue
        mid = prices[i] / prices[j] * (np.exp(0.1 * rng.standard_normal()) if cycles else 1.0)
        K = int(rng.integers(1, 6))
        side = np.arange(K) - K // 2
        p = mid * np.exp(0.01 * (side + 0.5) + 0.002 * rng.uniform(0, 1, K) * np.sign(side + 0.5))
        v = np.exp(rng.uniform(0, 3, K))
        x = np.where(side >= 0, v / p, 0.0); y = np.where(side < 0, v, 0.0)
        li.append([i, j]); kinds.append("bins"); w.append((p, x, y)); R.append(None); fees.append(g)
        lp.append((i, j, p, x, y, g))
    return li, kinds, w, R, fees, lp, prices


def _lp_cases(rng, seed_sum=True, m=6):
    """[(HostPools, lp pools, utility)]: Arbitrage on a market with cycles, Swap, Liquidate and a linear utility on one
    without"""
    out = []
    for cycles in (True, False):
        li, kinds, w, R, fees, lp, prices = bins_lp_market(rng, m=m, with_sum=seed_sum, cycles=cycles)
        hp = HostPools.from_lists(4, li, R, fees, kinds, w)
        us = [cf.Arbitrage(prices * np.exp(0.02 * rng.standard_normal(4)))] if cycles else \
            [cf.Swap(0, 2, 1.0), cf.Liquidate(0, np.r_[0.0, 0.5, 0.3, 0.2]),
             cf.LinearUtility(np.r_[prices[0], 0.0, 0.0, 0.0], np.r_[0.0, 0.2, 0.3, 0.0], np.zeros(4, bool),
                              np.zeros(4, bool))]
        out += [(hp, lp, u) for u in us]
    return out


def test_host_solver_bins_against_linprog():
    for seed in range(6):
        rng = np.random.default_rng(500 + seed)
        for p, (hp, lp, u) in enumerate(_lp_cases(rng, seed % 2 == 0)):
            out = _host_solve(hp, [u.spec(4)])
            assert int(out["stats"][0][7]) == 0, (seed, p, out["stats"][0])
            v = lp_value(lp, 4, u.spec(4))
            assert abs(out["stats"][0][0] - v) <= 1e-7 * abs(v), (seed, p, out["stats"][0][0], v)
            XB.certify(hp, u.spec(4), _result(hp, out, 0), 1e-8)


def test_xp_bins_dual_matches_linprog():
    """the reference's exact response is the pools' conjugate: at the solver's prices its dual bound is the LP value"""
    rng = np.random.default_rng(7)
    for p, (hp, lp, u) in enumerate(_lp_cases(rng, False)):
        sp = u.spec(4)
        nu = _host_solve(hp, [sp], tol=1e-10)["nu"][0]
        D = float(((X.ld(nu) - X.ld(sp.c)) * X.ld(sp.a)).sum() + XB._XPB.arb(hp, nu))
        v = lp_value(lp, 4, sp)
        assert abs(D - v) <= 1e-8 * abs(v), (p, D, v)


# ---------------------------------------------------------------------------------------------------------------------
# GPU

def _store(hp):
    return cf.PoolStore(hp, device="cuda:0")


def _gpu_pools(rng, m):
    """m random bins pools on tokens 0 .. 63 (HostPools) and their (prices, x, y, gamma)"""
    K = rng.choice([1, 2, 8, 64], m, p=[0.3, 0.3, 0.3, 0.1])
    cases = [random_bins(rng, int(k)) + (float(rng.choice([1.0, 0.9995, 0.997])),) for k in K]
    n_tok = 64
    a = rng.integers(0, n_tok, m); b = (a + rng.integers(1, n_tok, m)) % n_tok
    hp = HostPools.from_lists(n_tok, np.stack([a, b], 1).tolist(), [None] * m, [c[3] for c in cases], ["bins"] * m,
                              [c[:3] for c in cases])
    return hp, cases, a, b


@pytest.mark.gpu
def test_eval_kernel_against_reference():
    """k_eval_bins (plain, trades, hess; eps = 0 and > 0) on 10^5 pools, every pool against xp_bins (exact and
    smoothed) and against the host build; HVP, diagonal and dense against the pair decomposition of hcoef"""
    import torch
    rng = np.random.default_rng(11)
    m = 100_000
    hp, cases, a, b = _gpu_pools(rng, m)
    st = _store(hp)
    bk = st.buckets[0]
    assert bk.kind == _lib.KIND_BINS
    # token prices: each pool's mid somewhere across its range (a per-pool ratio needs per-pool tokens: use the
    # reference on the pools' own ratio, whatever it is)
    nu = np.exp(rng.uniform(-2, 2, 64))
    r = nu[a] / nu[b]
    # rescale the pools' prices so that r falls inside each pool's range (1 % off its middle, so that one-bin pools
    # are not priced exactly at r): rebuild the pools around r
    off = np.exp(0.01 * rng.standard_normal(m))
    cases = [(c[0] * r[q] * off[q] / np.sqrt(c[0][0] * c[0][-1]),) + c[1:] for q, c in enumerate(cases)]
    hp = HostPools.from_lists(64, np.stack([a, b], 1).tolist(), [None] * m, [c[3] for c in cases], ["bins"] * m,
                              [c[:3] for c in cases])
    st = _store(hp)
    bk = st.buckets[0]
    nut = torch.as_tensor(nu, dtype=torch.float64, device="cuda:0")
    sel = bk.sel
    tbar = np.where(rng.random(m) < 0.5, 0.0, rng.uniform(-1, 1, m) * np.array([c[1].sum() for c in cases]))
    for eps in (0.0, 0.05):
        bk.theta_bar.zero_()
        bk.theta_bar[0, :m] = torch.as_tensor(tbar[sel], dtype=torch.float64, device="cuda:0")
        Dh, Lh, hch, _ = host_pairs([c[:3] for c in cases], [c[3] for c in cases], nu[a], nu[b], eps,
                                    tbar if eps > 0 else np.zeros(m))
        accs = []
        for trades, hess in ((False, False), (True, False), (False, True), (True, True)):
            acc = st.evaluate(nut, eps, trades=trades, hess=hess).cpu().numpy().copy()
            accs.append(acc)
            if trades:
                D = bk.delta[:, :m].cpu().numpy().T; L = bk.lam[:, :m].cpu().numpy().T
                # the device contracts products into FMAs, the host build need not: equal to a few ulp of the flows
                np.testing.assert_allclose(D, Dh[sel], rtol=1e-13, atol=1e-15 * np.abs(Dh).max())
                np.testing.assert_allclose(L, Lh[sel], rtol=1e-13, atol=1e-15 * np.abs(Lh).max())
            if hess:
                np.testing.assert_allclose(bk.hcoef[:m].cpu().numpy(), hch[sel], rtol=1e-13, atol=1e-15 * hch.max())
        for acc in accs[1:]:
            np.testing.assert_allclose(acc, accs[0], rtol=1e-12, atol=1e-9 * np.abs(accs[0]).max())
        psi = np.zeros(64)
        np.add.at(psi, a, Lh[:, 0] - Dh[:, 0]); np.add.at(psi, b, Lh[:, 1] - Dh[:, 1])
        np.testing.assert_allclose(accs[0][:64], psi, rtol=1e-9, atol=1e-9 * np.abs(psi).max())
        # the device's trades (the last trades evaluation) against the reference, every pool, grouped by bin count
        Dd, Ld = np.zeros((m, 2)), np.zeros((m, 2))
        Dd[sel], Ld[sel] = D, L
        Ks = np.array([len(c[0]) for c in cases])
        checked = 0
        for K in np.unique(Ks).tolist():
            ix = np.nonzero(Ks == K)[0]
            P, Xb, Yb = (np.stack([cases[q][k] for q in ix]) for k in range(3))
            g = np.array([cases[q][3] for q in ix])
            s0 = Xb.sum(1) + (Yb / (g[:, None] * P)).sum(1)
            s1 = Yb.sum(1) + (P * Xb).sum(1) / g
            if eps == 0.0:
                Dx, Lx = (np.asarray(v, float) for v in XB.exact_many(P, Xb, Yb, g, nu[a[ix]], nu[b[ix]]))
                slope = np.concatenate([np.where(Xb > 0, P / g[:, None], np.nan), np.where(Yb > 0, g[:, None] * P, np.nan)], 1)
                ok = ~np.any(np.abs(r[ix][:, None] - slope) <= 1e-12 * slope, 1)        # not within 1e-12 of a slope
                sc = np.stack([s0, s1], 1)
                assert np.all(np.abs(Dx - Dd[ix])[ok] <= 1e-12 * sc[ok]), K
                assert np.all(np.abs(Lx - Ld[ix])[ok] <= 1e-12 * sc[ok]), K
                checked += int(ok.sum())
            else:
                tx, cx = (np.asarray(v, float) for v in XB.smoothed_many(P, Xb, Yb, g, nu[a[ix]], nu[b[ix]], eps,
                                                                          tbar[ix], hp.bin_zp[ix, 1]))
                assert np.all(np.abs(tx - (Ld[ix, 0] - Dd[ix, 0])) <= 1e-12 * s0), K
                assert np.all(np.abs(-cx - (Ld[ix, 1] - Dd[ix, 1])) <= 1e-12 * s1 / eps), K
                checked += len(ix)
        assert checked >= 0.95 * m
        if eps > 0.0:                             # Hessian kernels against the pair decomposition
            st.evaluate(nut, eps, trades=False, hess=True)
            h = np.zeros(m); h[:] = bk.hcoef[:m].cpu().numpy()
            ta, tb = a[sel], b[sel]
            H = np.zeros((64, 64))
            np.add.at(H, (ta, ta), h); np.add.at(H, (tb, tb), h); np.add.at(H, (ta, tb), -h); np.add.at(H, (tb, ta), -h)
            v = rng.standard_normal(64)
            np.testing.assert_allclose(st.hvp(torch.as_tensor(v, dtype=torch.float64, device="cuda:0")).cpu().numpy(),
                                       H @ v, rtol=1e-9, atol=1e-9 * np.abs(H @ v).max())
            np.testing.assert_allclose(st.hess_diag().cpu().numpy(), np.diag(H), rtol=1e-9)
            np.testing.assert_allclose(st.hess_dense().cpu().numpy(), H, rtol=1e-9, atol=1e-9 * np.abs(H).max())
            assert (h > 0).sum() > 1000


def _as_bins(d):
    """a reference instance with its constant-sum pool written as one bin at price 1 with the same reserves and fee"""
    kinds, R, w = list(d["kinds"]), list(d["reserves"]), list(d["weights"]) if d.get("weights") else [None] * len(d["kinds"])
    for i, k in enumerate(kinds):
        if k == "sum":
            kinds[i] = "bins"; w[i] = ([1.0], [float(R[i][0])], [float(R[i][1])]); R[i] = None
    return {**d, "kinds": kinds, "reserves": R, "weights": w}


def _paths():
    return [dict(method="thread"), dict(method="pools", native=False), dict(method="pools", native="hostloop")]


@pytest.mark.gpu
def test_reference_scripts_with_the_sum_pool_as_one_bin():
    import json
    with open(os.path.join(HERE, "golden", "reference_run.json")) as f:
        ref = json.load(f)
    for kw in _paths():
        d = _as_bins(I.arbitrage_instance()); g = ref["arbitrage"]
        hp = HostPools.from_lists(d["n_tokens"], d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"])
        r = cf.solve_pools(hp, cf.Arbitrage(d["market_value"]), tol=1e-9, **kw)
        assert r.status == "optimal" and abs(r.value - g["value"]) <= 1e-8 * abs(g["value"]), (kw, r.value)
        np.testing.assert_allclose(r.psi, g["psi"], atol=1e-6 * np.abs(g["psi"]).max())
        for i in range(5):
            np.testing.assert_allclose(r.deltas[i], g["deltas"][i], atol=5e-5)
            np.testing.assert_allclose(r.lambdas[i], g["lambdas"][i], atol=5e-5)
        d = _as_bins(I.liquidation_instance()); g = ref["liquidation"]
        hp = HostPools.from_lists(d["n_tokens"], d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"])
        r = cf.solve_pools(hp, cf.Liquidate(d["target"], d["current_assets"]), tol=1e-9, **kw)
        assert r.status == "optimal" and abs(r.psi[4] - g["value"]) <= 1e-8 * g["value"], (kw, r.psi)
        np.testing.assert_allclose(r.psi, g["psi"], atol=1e-6 * np.abs(g["psi"]).max())
        d = _as_bins(I.two_asset_instance()); g = ref["two_asset"]
        hp = HostPools.from_lists(d["n_tokens"], d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"])
        for j, t in enumerate(d["amounts"]):
            r = cf.solve_pools(hp, cf.Swap(d["tok_in"], d["tok_out"], t), tol=1e-9, **kw)
            assert r.status == "optimal" and abs(r.value - g["u_t"][j]) <= 1e-6 * max(1.0, g["u_t"][j]), (kw, j)
            for k in range(5):
                np.testing.assert_allclose(r.lambdas[k] - r.deltas[k], g["flows"][j][k], atol=5e-5)


@pytest.mark.gpu
def test_lp_oracle_on_every_path():
    for seed in range(6):
        rng = np.random.default_rng(700 + seed)
        for hp, lp, u in _lp_cases(rng, True, m=8):
            v = lp_value(lp, 4, u.spec(4))
            for kw in _paths():
                r = cf.solve_pools(hp, u, tol=1e-9, **kw)
                assert r.status == "optimal", (seed, kw, r.status)
                assert abs(r.value - v) <= 1e-7 * max(abs(v), 1e-9), (seed, kw, r.value, v)
                XB.certify(hp, u.spec(4), r, 1e-8)


@pytest.mark.gpu
def test_split_and_constant_sum_equivalences():
    rng = np.random.default_rng(21)
    for seed in range(3):
        hp, prices = I.synth_bins_market(300, 12, 40 + seed, K=(1, 32))
        sp, _ = I.bins_split(hp)
        u = cf.Arbitrage(prices)
        for kw in _paths()[1:]:
            a = cf.solve_pools(hp, u, tol=1e-9, **kw)
            b = cf.solve_pools(sp, u, tol=1e-9, **kw)
            assert a.status == b.status == "optimal", (kw, a.status, b.status)
            XB.certify(hp, u.spec(12), a, 1e-8)
            XB.certify(sp, u.spec(12), b, 1e-8)
            assert abs(a.value - b.value) <= 1e-7 * abs(a.value)
            np.testing.assert_allclose(a.psi, b.psi, atol=1e-6 * np.abs(a.psi).max())
    # one bin at price p is a constant-sum pool after token 1 is rescaled by p.  The two sides hold similar depth (y / p
    # near x): the bin's smoothing is one ramp over both sides (sigma = S / eps), a constant-sum pool's one per side,
    # so with one side much deeper the bin's ramp is the steeper one on the shallow side and can reach its fp64 floor
    # short of a 1e-9 certificate where the constant-sum pool does not (DESIGN §4)
    for q in range(8):
        p = float(np.exp(rng.uniform(-5, 5)))
        v = float(np.exp(rng.uniform(0, 2)))
        x, y = v * np.exp(0.3 * rng.standard_normal()), v * p * np.exp(0.3 * rng.standard_normal())
        g = float(rng.choice([1.0, 0.9995, 0.997]))
        pr = np.array([1.0, 1.0 / p, 0.7])                          # token 1 in the bin's units is worth 1/p
        li = [[0, 1], [0, 2], [1, 2]]                                # token 1 of the sum market = p of the bins one
        hb = HostPools.from_lists(3, li, [None, [5.0, 2.1], [4.0 * p, 2.0]], [g, 0.997, 0.997],
                                  ["bins", "product", "product"], [([p], [x], [y]), None, None])
        hs = HostPools.from_lists(3, li, [[x, y / p], [5.0, 2.1], [4.0, 2.0]], [g, 0.997, 0.997],
                                  ["sum", "product", "product"])
        ub = cf.Arbitrage(pr * np.exp(0.05 * rng.standard_normal(3)))
        us = cf.Arbitrage(ub.c * np.array([1.0, p, 1.0]))
        a = cf.solve_pools(hb, ub, tol=1e-9, method="pools", native=False)
        b = cf.solve_pools(hs, us, tol=1e-9, method="pools", native=False)
        assert a.status == b.status == "optimal", (q, a.status, b.status)
        assert abs(a.value - b.value) <= 4e-9 * abs(a.value), (q, a.value, b.value)
        np.testing.assert_allclose(a.psi * np.array([1.0, 1.0 / p, 1.0]), b.psi, atol=1e-7 * np.abs(b.psi).max())


def _mixed_market(seed):
    """a small market of bins pools beside every other kind: synth_tricrypto_market's mix (constant product, weighted,
    constant sum, ranges, ladders, StableSwap of 2..4 coins, two- and three-coin cryptoswap) and synth_bins_market's
    Liquidity-Book-like pools, order books and limit orders, on 6 tokens"""
    ht, prices = I.synth_tricrypto_market(60, 6, 900 + seed, frac_tri=0.1)
    hb, _ = I.synth_bins_market(10, 6, 900 + seed, K=(1, 16), frac_lb=0.4, frac_book=0.3, frac_order=0.3)
    return _merge(ht, hb), prices


def _disjoint(hps):
    """markets on disjoint token sets as one HostPools (market k's tokens after market k-1's)"""
    cat = lambda name, dt: np.concatenate([np.asarray(getattr(h, name), dt).reshape(len(getattr(h, name)), -1)
                                           if name in ("lad_rec", "bin_rec", "lad_sc", "bin_zp")
                                           else np.asarray(getattr(h, name), dt) for h in hps])
    ptrs, lptrs, bptrs, toks = [np.zeros(1, np.int64)], [np.zeros(1, np.int64)], [np.zeros(1, np.int64)], []
    t0 = 0
    for h in hps:
        ptrs.append(np.asarray(h.pool_ptr[1:], np.int64) + ptrs[-1][-1])
        lptrs.append(np.asarray(h.lad_ptr[1:], np.int64) + lptrs[-1][-1])
        bptrs.append(np.asarray(h.bin_ptr[1:], np.int64) + bptrs[-1][-1])
        toks.append(np.asarray(h.tok_idx, np.int64) + t0)
        t0 += h.n_tokens
    return HostPools(t0, np.concatenate(ptrs), np.concatenate(toks).astype(np.int32), cat("reserves", np.float64),
                     cat("weights", np.float64), cat("gamma", np.float64), cat("kind", np.uint8), cat("amp", np.float64),
                     cat("inv", np.float64), np.concatenate(lptrs), cat("lad_rec", np.float64), cat("lad_sc", np.float64),
                     cat("cgam", np.float64), np.concatenate(bptrs), cat("bin_rec", np.float64), cat("bin_zp", np.float64))


def _certify_many(markets, specs, results, tol):
    """xp_bins.certify of many solved markets at once, as one problem on their disjoint token sets (one pass of the
    extended-precision references over all their pools), then every market's own exact duality gap: its dual bound
    D = sum (nu^ - c) a + sum_i arb_i(nu^) against P = c'psi of its trades, with xp_reference's check 4 and bounds on
    each market's tokens: -eps - V <= (D - P) / |D| <= 2 tol + eps"""
    from cfmm_routing_code_b200.solver import DualSpec
    big = _disjoint(markets)
    spec = DualSpec(*(np.concatenate([getattr(s, f) for s in specs]) for f in ("c", "a", "eq", "pinned")))
    res = types.SimpleNamespace(value=sum(r.value for r in results), dual_value=sum(r.dual_value for r in results),
                                psi=np.concatenate([r.psi for r in results]), nu=np.concatenate([r.nu for r in results]),
                                deltas=[d for r in results for d in r.deltas],
                                lambdas=[l for r in results for l in r.lambdas])
    c, a = X.ld(spec.c), X.ld(spec.a)
    ineq = ~spec.eq & ~spec.pinned
    nuh = np.where(spec.pinned, c, np.where(ineq, np.maximum(X.ld(res.nu), c), X.ld(res.nu)))   # certify's nu^
    out = XB._XPB.response(big, nuh)
    arb = out["arb"]
    orig = XB._XPB.response                      # the certificate's dual bound reads the same response: evaluate once
    XB._XPB.response = lambda h, v: out if h is big and np.array_equal(X.ld(v), nuh) else orig(h, v)
    try:
        XB.certify(big, spec, res, tol)
    finally:
        XB._XPB.response = orig
    d, l = XB._XPB._trades(res, big)
    psi_xp, gross, _ = XB._XPB.flows(big, d, l)
    s = X.ld(res.psi) + a
    viol = np.where(spec.pinned, X.ld(0), np.where(spec.eq, np.abs(s), np.maximum(-s, 0)))
    t0 = p0 = 0
    for k, h in enumerate(markets):
        tk, pk = slice(t0, t0 + h.n_tokens), slice(p0, p0 + h.m)
        D = ((nuh[tk] - c[tk]) * a[tk]).sum() + arb[pk].sum()
        P = (c[tk] * psi_xp[tk]).sum()
        aD = max(abs(D), X.LD(1e-300))
        eps = X.LD(X.ROUND_REL) * (nuh[tk] * gross[tk]).sum() / aD
        V = (np.abs(nuh[tk] - c[tk]) * viol[tk]).sum() / aD
        assert -eps - V <= (D - P) / aD <= 2 * tol + eps, (k, float(D), float(P), float(eps), float(V))
        t0 += h.n_tokens; p0 += h.m


@pytest.mark.gpu
def test_mixed_markets_certified():
    """bins beside every other kind (two- and three-coin cryptoswap included): 200 small markets on the per-thread path
    (cfmm_batch_solve_bins, one launch), 24 on each pool path (solver.py and the native host loop), every one optimal
    and certified by xp_bins"""
    rng = np.random.default_rng(31)
    probs = []
    for seed in range(200):
        hp, prices = _mixed_market(seed)
        probs.append((hp, cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(6)))))
    kinds = np.unique(np.concatenate([hp.kind for hp, _ in probs]))
    assert set(kinds.tolist()) >= {0, 1, 3, 4, 6, 8, 10}
    assert any(np.any(np.diff(hp.pool_ptr)[hp.kind == 8] == 3) for hp, _ in probs)
    rs = cf.solve_many(probs, tol=1e-8)
    assert [r.status for r in rs] == ["optimal"] * len(probs)
    _certify_many([hp for hp, _ in probs], [u.spec(6) for _, u in probs], rs, 1e-8)
    for kw in _paths()[1:]:
        rs = [cf.solve_pools(hp, u, tol=1e-8, **kw) for hp, u in probs[:24]]
        assert [r.status for r in rs] == ["optimal"] * 24, kw
        _certify_many([hp for hp, _ in probs[:24]], [u.spec(6) for _, u in probs[:24]], rs, 1e-8)


def _merge(h1, h2):
    """two HostPools on the same tokens as one (h2's bins records after h1's)"""
    from cfmm_routing_code_b200.batch import pack_problems
    hp, *_ = pack_problems([(h1, cf.Arbitrage(np.ones(h1.n_tokens))), (h2, cf.Arbitrage(np.ones(h2.n_tokens)))])
    return hp


@pytest.mark.gpu
def test_large_market_two_loops_and_split():
    hp, prices = I.synth_bins_market(100_000, 1000, 5)
    u = cf.Arbitrage(prices)
    a = cf.solve_pools(hp, u, tol=1e-6, method="pools", native=False)
    b = cf.solve_pools(hp, u, tol=1e-6, method="pools", native="hostloop")
    assert a.status == b.status == "optimal", (a.status, b.status)
    assert abs(a.value - b.value) <= 1e-9 * abs(a.value), (a.value, b.value)
    XB.certify(hp, u.spec(1000), a, 1e-6)
    sp, _ = I.bins_split(hp)
    c = cf.solve_pools(sp, u, tol=1e-6, method="pools", native=False)
    assert c.status == "optimal" and abs(a.value - c.value) <= 1e-6 * abs(a.value), (a.value, c.value)


@pytest.mark.gpu
def test_unit_invariance():
    rng = np.random.default_rng(41)
    hp, prices = I.synth_bins_market(400, 10, 77, K=(1, 32))
    u = cf.Arbitrage(prices)
    base = cf.solve_pools(hp, u, tol=1e-9, method="pools", native=False)
    assert base.status == "optimal"
    for s in (1e3, 1e-3):
        k = np.ones(10); k[rng.choice(10, 4, replace=False)] = s       # new unit = s old units
        sc = _rescale(hp, k)
        r = cf.solve_pools(sc, cf.Arbitrage(prices * k), tol=1e-9, method="pools", native=False)
        assert r.status == "optimal"
        assert abs(r.value - base.value) <= 1e-7 * abs(base.value)
        np.testing.assert_allclose(r.psi * k, base.psi, atol=1e-6 * np.abs(base.psi).max())


def _rescale(hp, k):
    """hp in new token units (amounts of token j divided by k_j): bins prices scale by k_0 / k_1"""
    ptr = hp.pool_ptr
    li, R, fees, kinds, w = [], [], [], [], []
    for i in range(hp.m):
        t = hp.tok_idx[ptr[i]:ptr[i + 1]]
        li.append(t.tolist()); fees.append(float(hp.gamma[i]))
        if hp.kind[i] == KIND_BINS_HOST:
            p, x, y = (np.asarray(v, float) for v in XB.bins_of(hp, i))
            pr = np.unique(p)
            xs = np.array([x[p == q].sum() for q in pr]); ys = np.array([y[p == q].sum() for q in pr])
            kinds.append("bins"); R.append(None); w.append((pr * k[t[0]] / k[t[1]], xs / k[t[0]], ys / k[t[1]]))
        else:
            kinds.append("product"); R.append((hp.reserves[ptr[i]:ptr[i + 1]] / k[t]).tolist()); w.append(None)
    return HostPools.from_lists(hp.n_tokens, li, R, fees, kinds, w)


@pytest.mark.gpu
def test_rank_stores_sum_to_the_single_store():
    import torch
    hp, prices = I.synth_bins_market(20_000, 200, 9)
    nu = torch.as_tensor(prices * np.exp(0.01 * np.random.default_rng(0).standard_normal(200)), dtype=torch.float64,
                         device="cuda:0")
    one = cf.PoolStore(hp, device="cuda:0").evaluate(nu, 0.0).cpu().numpy()
    for world in (2, 4):
        tot = sum(cf.PoolStore(hp, device="cuda:0", rank=r, world=world).evaluate(nu, 0.0).cpu().numpy()
                  for r in range(world))
        np.testing.assert_allclose(tot, one, rtol=1e-10, atol=1e-10 * np.abs(one).max())


@pytest.mark.gpu
def test_fee_updates_and_rejected_reserves():
    import torch
    hp, prices = I.synth_bins_market(5000, 50, 13)
    st = cf.PoolStore(hp, device="cuda:0")
    ids = np.nonzero(hp.kind == KIND_BINS_HOST)[0][:100]
    fees = np.full(len(ids), 0.995)
    st.update_pools(ids, fees=fees)
    hp2 = HostPools(**{**hp.__dict__})
    hp2.gamma = hp.gamma.copy(); hp2.gamma[ids] = fees
    fresh = cf.PoolStore(hp2, device="cuda:0")
    for b1, b2 in zip(st.buckets, fresh.buckets):
        if getattr(b1, "blocked", False):
            continue
        for name in ("reserves", "tok_idx", "gamma", "weights", "logrw", "theta_bar"):
            t1, t2 = getattr(b1, name, None), getattr(b2, name, None)
            assert (t1 is None) == (t2 is None)
            if t1 is not None:
                assert torch.equal(t1, t2), name
    plain = [b for b in st.buckets if not getattr(b, "blocked", False)]
    before = [(b.reserves.clone(), b.gamma.clone()) for b in plain]
    with pytest.raises(ValueError):
        st.update_pools([int(ids[0]), 0], reserves=[[1.0, 1.0], [1.0, 1.0]])
    assert all(torch.equal(r, b.reserves) and torch.equal(g, b.gamma) for (r, g), b in zip(before, plain))
    prod = np.nonzero(hp.kind != KIND_BINS_HOST)[0][:3]
    st.update_pools(prod, reserves=np.ones((3, 2)))                  # other pools of the store still update


@pytest.mark.gpu
def test_abi_codes():
    import torch
    lib = _lib.load()
    hp, prices = I.synth_bins_market(100, 10, 17, frac_lb=1.0, frac_book=0.0, frac_order=0.0)
    st = cf.PoolStore(hp, device="cuda:0")
    b = st.buckets[0]
    nu = torch.ones(10, dtype=torch.float64, device="cuda:0")
    acc = torch.zeros(11, dtype=torch.float64, device="cuda:0")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ev = lambda bk: lib.cfmm_arb_eval(C.byref(bk), 10, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc[10:].data_ptr(),
                                      None, s)
    assert ev(b.c_bucket) == 0
    E_NULL, E_KIND = -1, -2                                            # CFMM_E_NULL, CFMM_E_KIND
    for change, code in ((dict(arity=3), E_KIND), (dict(weights=None), E_NULL), (dict(theta_bar=None), E_NULL),
                         (dict(logrw=None), E_NULL), (dict(kind=7), E_KIND)):
        bk = _lib.Bucket(b.c_bucket.kind, b.c_bucket.arity, b.c_bucket.n_pools, b.c_bucket.stride, b.c_bucket.reserves,
                         b.c_bucket.tok_idx, b.c_bucket.gamma, b.c_bucket.weights, b.c_bucket.logrw,
                         b.c_bucket.theta_bar)
        for k, v in change.items():
            setattr(bk, k, v)
        assert ev(bk) == code, change
    move = torch.zeros(1, dtype=torch.float64, device="cuda:0")
    out = b.out_struct(True, True)
    assert lib.cfmm_bins_update_multipliers(C.byref(b.c_bucket), out.delta, None, b.theta_bar.data_ptr(),
                                            move.data_ptr(), s) == E_NULL
    sb = b.c_bucket
    bk = _lib.Bucket(1, 2, sb.n_pools, sb.stride, sb.reserves, sb.tok_idx, sb.gamma, sb.weights, sb.logrw, sb.theta_bar)
    assert lib.cfmm_bins_update_multipliers(C.byref(bk), out.delta, out.lambda_, b.theta_bar.data_ptr(),
                                            move.data_ptr(), s) == E_KIND               # a constant-sum bucket
    assert lib.cfmm_sum_update_multipliers(C.byref(b.c_bucket), out.lambda_, b.theta_bar.data_ptr(), move.data_ptr(),
                                           s) == E_KIND                                 # and the other way round
    assert lib.cfmm_bins_update_multipliers(C.byref(b.c_bucket), out.delta, out.lambda_, b.theta_bar.data_ptr(),
                                            move.data_ptr(), s) == 0
    torch.cuda.synchronize()
