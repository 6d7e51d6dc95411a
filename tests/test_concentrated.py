"""Concentrated-liquidity pools: a whole Uniswap-v3 tick ladder as one pool (host kind 6, CFMM_KIND_CONCENTRATED).

CPU: the records, the derived state and reserves, and instances.v3_ladder against 50-digit decimal; cfmm_small::ladder_pair
compiled for the host against the longdouble reference (tests/xp_concentrated.py: the sum of the intervals' exact
bounded-product trades, no tables, no search) and, at T = 1, against bounded_pair; hc against finite differences; the
per-thread solver's concentrated instance on a market and on the same market as ranges; validation; packing.
GPU (H100): k_eval_ladder in all four (trades, hess) instances against the reference and against the range-decomposed
bucket; the Hessian kernels; every solve path on markets that mix ladders with every other kind, certified and compared
with the decomposed market; in-place price updates; rank stores; C ABI codes.

Error bounds (ladder_tol).  Inputs are the same f64 b, L, s for the product and the reference, so two sources remain.
(1) Rounding of the arithmetic: every flow is a sum of at most three terms (partial interval at each end, one table
difference), each a product or difference of values no larger than the token amounts involved, held = reserve + |flow|;
the table entries are within (u/2 + T eps_ld) of the exact sums of b and L (ladder_records).  That is <= (16 u + 4 T
eps_ld) (reserve + |D| + |L|) with room for the final division by gamma.  (2) The target sqrt price s_f = sqrt(nu0 /
(gamma nu1)) (or its mirror) is rounded by <= 1.5 u s_f (a product, a quotient, a square root), and a flow moves with it
at rate L(s_f) (token 1) and L(s_f) / s_f^2 (token 0), over gamma for a tender: <= 1.5 u Lmax s_f (token 1) and
1.5 u Lmax / s_f (token 0), over gamma, with Lmax the pool's largest liquidity (a bound on L(s_f) on either side of a
bound); ladder_tol takes 8 u, for a margin of more than 4 over what this term alone can reach.  The tests assert the
observed error is at most a quarter of the bound, and print the ratio.
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
from cfmm_routing_code_b200.pools import (HostPools, KIND_CONCENTRATED_HOST, LADDER_T_MAX, check_pool_update,
                                          ladder_records, ladder_state)
import xp_concentrated as XC
import xp_reference as X

U = 2.0 ** -53
EPS_LD = float(np.finfo(np.longdouble).eps)
HERE = os.path.dirname(os.path.abspath(__file__))
p_ = lambda x: x.ctypes.data_as(C.c_void_p)
_HOST = None


def _host():
    """tests/host_harness/ladder_host.cpp: cfmm_small::ladder_pair and the solver's concentrated instance, host build"""
    global _HOST
    if _HOST is None:
        src = os.path.join(HERE, "host_harness", "ladder_host.cpp")
        hdr = os.path.join(HERE, "..", "cfmm_routing_code_b200", "csrc", "cfmm_small.cuh")
        lib = os.path.join(HERE, "_build", "libladder_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src],
                           check=True)
        _HOST = C.CDLL(lib)
    return _HOST


def _ladder_args(hp):
    sel = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    lp = hp.lad_ptr
    P = np.ascontiguousarray(np.stack([hp.lad_sc[sel, 0], hp.lad_sc[sel, 1], lp[sel], lp[sel + 1] - lp[sel] - 1], 1))
    tok = hp.tok_idx[hp.pool_ptr[sel][:, None] + np.arange(2)]
    return sel, P, tok


def host_pools(hp, nu):
    """ladder_pair (host build) on every ladder pool of hp at token prices nu: sel, D, L (n, 2), hc (n,)"""
    sel, P, tok = _ladder_args(hp)
    m = len(sel)
    n0, n1 = np.ascontiguousarray(nu[tok[:, 0]]), np.ascontiguousarray(nu[tok[:, 1]])
    g = np.ascontiguousarray(hp.gamma[sel])
    D, L, hc = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m)
    _host().ladder_host_pools(C.c_longlong(m), p_(np.ascontiguousarray(hp.lad_rec)), p_(P), p_(g), p_(n0), p_(n1),
                              p_(D), p_(L), p_(hc))
    return sel, D, L, hc


def ladder_tol(hp, sel, nu, D, L):
    """per-slot bound (n, 2) on |flow - exact| of the ladder pools sel (module docstring)"""
    R = hp.reserves[hp.pool_ptr[sel][:, None] + np.arange(2)]
    lp = hp.lad_ptr
    T = (lp[sel + 1] - lp[sel] - 1).astype(float)
    Lmax = np.maximum.reduceat(hp.lad_rec[:, 1], lp[:-1][sel]) if len(sel) else np.zeros(0)
    tok = hp.tok_idx[hp.pool_ptr[sel][:, None] + np.arange(2)]
    g = hp.gamma[sel]
    n0, n1 = nu[tok[:, 0]], nu[tok[:, 1]]
    sf = np.where(np.abs(D[:, 0]) + np.abs(L[:, 1]) > 0, np.sqrt(n0 / (g * n1)), np.sqrt(g * n0 / n1))
    rnd = (16 * U + 4 * T * EPS_LD)[:, None] * (R + np.abs(D) + np.abs(L)) / g[:, None]
    cond = 8 * U * Lmax[:, None] * np.stack([1 / sf, sf], 1) / g[:, None]
    return rnd + cond


def random_ladders(m, T, seed, full_range=False):
    """m ladders of T intervals (bounds as prices, liquidity with ~15 % empty intervals) and a current price each"""
    rng = np.random.default_rng(seed)
    if full_range:
        lo, hi = 1.0001 ** -887272, 1.0001 ** 887272
        inner = np.sort(np.exp(rng.uniform(-20, 20, (m, T - 1))), 1) if T > 1 else np.zeros((m, 0))
        bounds = np.concatenate([np.full((m, 1), lo), inner, np.full((m, 1), hi)], 1)
    else:
        w = np.exp(rng.uniform(np.log(1e-4), np.log(0.05), (m, T)))
        bounds = np.exp(rng.normal(0, 2, (m, 1)) + np.concatenate([np.zeros((m, 1)), np.cumsum(w, 1)], 1))
    liq = np.exp(rng.normal(6, 2, (m, T))) * (rng.random((m, T)) > 0.15)
    liq[np.arange(m), rng.integers(0, T, m)] = np.exp(rng.normal(6, 2, m))
    u = rng.uniform(-0.1, 1.1, m)
    price = np.exp(np.log(bounds[:, 0]) + u * (np.log(bounds[:, -1]) - np.log(bounds[:, 0])))
    on = rng.random(m) < 0.1                                              # a tenth exactly on a bound
    price[on] = bounds[on, rng.integers(0, T + 1, on.sum())]
    return bounds, liq, price


def ladder_hp(bounds, liq, price, gam):
    m = len(price)
    li = [[0, 1]] * m
    return HostPools.from_lists(2, li, [None] * m, gam, ["concentrated"] * m,
                                [(price[i], bounds[i], liq[i]) for i in range(m)])


def _targets(hp, rng):
    """per-pool target sqrt prices for the cases of the issue: in the no-trade band, inside the current interval, across
    one / several / all bounds, past both ends, exactly on a bound.  Returns sqrt-price targets (m,)."""
    sel = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    lp = hp.lad_ptr
    out = np.empty(len(sel))
    for n_, i in enumerate(sel.tolist()):
        b = hp.lad_rec[lp[i]:lp[i + 1], 0]
        s, c = hp.lad_sc[i]
        c = int(c)
        T = len(b) - 1
        case = rng.integers(0, 8)
        if case == 0:
            out[n_] = s                                                    # the no-trade band (with gamma < 1)
        elif case == 1:
            out[n_] = b[c] + rng.uniform(0, 1) * (b[c + 1] - b[c])
        elif case == 2:
            out[n_] = b[min(c + 1, T)] + rng.uniform(0, 1) * (b[min(c + 2, T)] - b[min(c + 1, T)])
        elif case == 3:
            k = int(rng.integers(0, T + 1)); out[n_] = b[k] * (1 + rng.uniform(-1e-3, 1e-3))
        elif case == 4:
            out[n_] = b[0] * rng.uniform(0.1, 1.0)                          # past the bottom (all intervals)
        elif case == 5:
            out[n_] = b[-1] * rng.uniform(1.0, 10.0)                        # past the top
        elif case == 6:
            out[n_] = b[int(rng.integers(0, T + 1))]                        # exactly on a bound
        else:
            out[n_] = s * np.exp(rng.normal(0, 0.01))
    return out


def _eval_one_by_one(hp, targets, g):
    """ladder pools each with its own token pair (tokens 2i, 2i+1): a copy of hp with distinct tokens, and token prices
    that put each pool's falling / rising target at `targets` (nu1 = 1, nu0 = target^2 gamma or target^2 / gamma)"""
    m = hp.m
    tok = np.arange(2 * m, dtype=np.int32)
    hq = HostPools(2 * m, hp.pool_ptr, tok, hp.reserves, hp.weights, hp.gamma, hp.kind, None, None, hp.lad_ptr,
                   hp.lad_rec, hp.lad_sc)
    s = hp.lad_sc[:, 0]
    t2 = targets * targets
    nu = np.ones(2 * m)
    nu[0::2] = np.where(targets < s, t2 * g, t2 / g)
    return hq, nu


# ====================================================================================================== CPU
def test_records_state_and_reserves_match_decimal():
    """records {b, L, Y, X}, (s, c) and the reserves against 50-digit decimal: full-range bounds (ticks +-887272), empty
    intervals, a price on a bound, prices outside the ladder"""
    getcontext().prec = 50
    worst = 0.0
    for seed, (T, fr) in enumerate([(1, False), (5, True), (17, False), (300, True), (64, False)]):
        bounds, liq, price = random_ladders(40, T, 10 + seed, full_range=fr)
        price[0] = bounds[0, 0] * 0.5; price[1] = bounds[1, -1] * 2.0; price[2] = bounds[2, T // 2 if T > 1 else 1]
        hp = ladder_hp(bounds, liq, price, np.full(40, 0.997))
        hp.validate()
        for i in range(40):
            rec = hp.lad_rec[hp.lad_ptr[i]:hp.lad_ptr[i + 1]]
            # b_k: one correctly rounded sqrt of the f64 price.  Y, X, x, y: against the exact sums of the STORED b_k and L
            # (the records are what the kernel reads; a rounded b_k moves b_{k+1} - b_k by its own ulp, which is input)
            for k in range(T + 1):
                bd = Decimal(float(bounds[i, k])).sqrt()
                assert abs(Decimal(rec[k, 0]) - bd) <= Decimal(U) * bd, (i, k)
            b = [Decimal(float(x)) for x in rec[:, 0]]
            L = [Decimal(float(x)) for x in liq[i]] + [Decimal(0)]
            Y = [sum((L[j] * (b[j + 1] - b[j]) for j in range(k)), Decimal(0)) for k in range(T + 1)]
            Xs = [sum((L[j] * (1 / b[j] - 1 / b[j + 1]) for j in range(k, T)), Decimal(0)) for k in range(T + 1)]
            for k in range(T + 1):
                for col, ref in ((2, Y[k]), (3, Xs[k])):
                    # extended-precision sums rounded once: u/2 + T eps_ld, bounded by 4 u + 4 T eps_ld
                    bound = (4 * U + 4 * T * EPS_LD) * float(ref)
                    err = abs(float(Decimal(rec[k, col]) - ref))
                    worst = max(worst, err / bound if bound > 0 else (0.0 if err == 0 else np.inf))
                    assert err <= bound, (i, k, col, err, bound)
            sp = Decimal(float(price[i])).sqrt()
            s = Decimal(float(hp.lad_sc[i, 0]))                           # sqrt(price) rounded once, or clamped to an end
            assert s in (b[0], b[T]) or abs(s - sp) <= Decimal(U) * sp
            c = max(k for k in range(T) if b[k] <= s)
            assert hp.lad_sc[i, 1] == c, (i, hp.lad_sc[i], c)
            y = Y[c] + L[c] * (s - b[c]); x = Xs[c + 1] + L[c] * (1 / s - 1 / b[c + 1])
            for got, ref in ((hp.reserves[2 * i], x), (hp.reserves[2 * i + 1], y)):
                # table entry (as above) plus one partial interval formed in extended precision, rounded once
                bound = (8 * U + 4 * T * EPS_LD) * float(ref) + 1e-300
                err = abs(float(Decimal(got) - ref))
                worst = max(worst, err / bound)
                assert err <= bound, (i, err, bound)
    print(f"records / reserves: worst observed / bound {worst:.3g}")
    assert worst <= 0.25


def test_v3_ladder_matches_decimal():
    getcontext().prec = 50
    ticks = [-887272, -100000, -5, 0, 7, 60000, 887272]
    net = [10 ** 18, 5 * 10 ** 17, 0, -2 * 10 ** 17, 3 * 10 ** 15, -3 * 10 ** 15, -13 * 10 ** 17]
    for d0, d1 in ((18, 6), (6, 18), (8, 8), (0, 3)):
        sqx = 79228162514264337593543950336 * 3 // 7
        price, bounds, liq = I.v3_ladder(sqx, ticks[::-1], net[::-1], d0, d1)
        dd = Decimal(10) ** (d0 - d1)
        assert abs(Decimal(price) / (Decimal(sqx) ** 2 / Decimal(2) ** 192 * dd) - 1) <= Decimal(U)
        for t, b in zip(ticks, bounds):
            assert abs(Decimal(b) / (Decimal("1.0001") ** t * dd) - 1) <= Decimal(U)
        run, sc = 0, (Decimal(10) ** (-(d0 + d1))).sqrt()
        for x, l in zip(net, liq):
            run += x
            assert abs(Decimal(l) - run * sc) <= Decimal(U) * run * sc
        assert len(liq) == len(bounds) - 1 and liq[2] == liq[1]
        hp = HostPools.from_lists(2, [[0, 1]], [None], [0.997], ["concentrated"], [(price, bounds, liq)])
        hp.validate()
    with pytest.raises(ValueError):
        I.v3_ladder(sqx, [0, 10], [-5, 5], 18, 18)                           # negative running liquidity


@pytest.mark.parametrize("T", [1, 2, 9, 64, 512, 4096])
def test_ladder_pair_matches_reference(T):
    """T intervals, gammas {1, 0.9997, 0.99, 0.5}; targets in the no-trade band, inside the current interval, across one,
    several and all bounds, past both ends and exactly on bounds"""
    rng = np.random.default_rng(T)
    m = 400 if T <= 512 else 60
    bounds, liq, price = random_ladders(m, T, 100 + T)
    g = np.array([1.0, 0.9997, 0.99, 0.5])[rng.integers(0, 4, m)]
    hp = ladder_hp(bounds, liq, price, g)
    hq, nu = _eval_one_by_one(hp, _targets(hp, rng), g)
    sel, D, L, hc = host_pools(hq, nu)
    _, Dx, Lx, hx = XC.ladder_response(hq, nu)
    Dx, Lx = Dx.astype(float), Lx.astype(float)
    tol = ladder_tol(hq, sel, nu, Dx, Lx)
    err = np.maximum(np.abs(D - Dx), np.abs(L - Lx))
    r = (err / tol).max()
    print(f"T={T}: flows observed / bound {r:.3g}; trading {float(np.mean(np.abs(D).sum(1) > 0)):.2f}")
    assert r <= 0.25
    assert np.all((D >= 0) & (L >= 0)) and np.all(D[:, 0] * D[:, 1] == 0) and np.all(L[:, 0] * L[:, 1] == 0)
    # hc: equal to the reference's except where the target sits within its rounding of a bound (there either side's L)
    # or of s (the edge of the no-trade band: a zero trade in one precision, an infinitesimal one in the other)
    hs = 0.5 * np.sqrt(nu[0::2] * nu[1::2] / g)
    near = np.zeros(m, bool)
    for i in range(m):
        b = np.r_[hp.lad_rec[hp.lad_ptr[i]:hp.lad_ptr[i + 1], 0], hp.lad_sc[i, 0]]     # (and s: the band's edge)
        for t in (np.sqrt(nu[2 * i] / (g[i] * nu[2 * i + 1])), np.sqrt(g[i] * nu[2 * i] / nu[2 * i + 1])):
            near[i] |= bool(np.any(np.abs(b - t) <= 8 * U * b))
    hx = hx.astype(float)
    ok = np.abs(hc - hx) <= 1e-13 * np.maximum(hx, hc)
    assert np.all(ok | near), np.nonzero(~(ok | near))[0][:5]
    Lall = [hp.lad_rec[hp.lad_ptr[i]:hp.lad_ptr[i + 1], 1] for i in range(m)]
    for i in np.nonzero(~ok)[0]:
        assert np.any(np.abs(hc[i] - Lall[i] * hs[i]) <= 1e-13 * hc[i]) or hc[i] == 0


def test_one_interval_matches_bounded_pair():
    """T = 1: ladder_pair equals bounded_pair on the same position (v3_position arithmetic) to a few ulp of the virtual
    reserves, plus the target's rounding"""
    rng = np.random.default_rng(7)
    m = 3000
    bounds, liq, price = random_ladders(m, 1, 7)
    liq = np.maximum(liq, 1.0)
    g = np.array([1.0, 0.9997, 0.99, 0.5])[rng.integers(0, 4, m)]
    hp = ladder_hp(bounds, liq, price, g)
    hq, nu = _eval_one_by_one(hp, _targets(hp, rng), g)
    sel, D, L, hc = host_pools(hq, nu)
    rg, owner = I.ladder_ranges(hq)
    assert rg.m == m and np.array_equal(owner, np.arange(m))
    R, o = rg.reserves.reshape(-1, 2), rg.weights.reshape(-1, 2)
    Db, Lb, hb = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m)
    n0, n1 = np.ascontiguousarray(nu[0::2]), np.ascontiguousarray(nu[1::2])
    _host().ladder_host_bounded(C.c_longlong(m), p_(np.ascontiguousarray(R)), p_(np.ascontiguousarray(o)),
                                p_(np.ascontiguousarray(g)), p_(n0), p_(n1), p_(Db), p_(Lb), p_(hb))
    V = R + o
    tol = 16 * U * (V + np.abs(D) + np.abs(L)) / g[:, None] + ladder_tol(hq, sel, nu, D, L)
    r = (np.maximum(np.abs(D - Db), np.abs(L - Lb)) / tol).max()
    print(f"T=1 vs bounded_pair: observed / bound {r:.3g}")
    assert r <= 0.25
    both = (hc > 0) & (hb > 0)
    assert np.all(np.abs(hc[both] - hb[both]) <= 1e-12 * hb[both])


def test_hc_matches_finite_differences():
    """hc = nu0 dpsi_0 / dlog nu0 (the scaled Hessian's coefficient), by central differences in log-price, away from
    bounds (where psi has a kink in its derivative)"""
    rng = np.random.default_rng(11)
    bounds, liq, price = random_ladders(300, 32, 11)
    g = np.array([1.0, 0.9997, 0.99])[rng.integers(0, 3, 300)]
    hp = ladder_hp(bounds, liq, price, g)
    hq, nu = _eval_one_by_one(hp, _targets(hp, rng), g)
    _, D, L, hc = host_pools(hq, nu)
    h = 1e-6
    up, dn = nu.copy(), nu.copy()
    up[0::2] *= np.exp(h); dn[0::2] *= np.exp(-h)
    _, Du, Lu, _ = host_pools(hq, up)
    _, Dd, Ld, _ = host_pools(hq, dn)
    fd = ((Lu[:, 0] - Du[:, 0]) - (Ld[:, 0] - Dd[:, 0])) / (2 * h) * nu[0::2]
    # the one-sided derivatives agree (no bound or end within the step) where both steps see the same interval
    # (hc itself moves by a relative h / 2 with nu0 inside an interval)
    same = np.abs(hc - XC.ladder_response(hq, up)[3].astype(float)) <= 1e-5 * (hc + 1e-300)
    same &= np.abs(hc - XC.ladder_response(hq, dn)[3].astype(float)) <= 1e-5 * (hc + 1e-300)
    same &= hc > 0
    assert same.sum() > 100
    np.testing.assert_allclose(fd[same], hc[same], rtol=1e-5)


def _small_market(rng, T=(2, 40), empty=0.2):
    """5 tokens: two ladders, product pools over all tokens, a two- and a three-coin StableSwap pool, a constant-sum pair"""
    n = 5
    prices = np.array([1.0, 1.001, 2.5, 0.4, 7.0])
    li, res, fees, kinds, w = [], [], [], [], []
    for i in range(n - 1):
        li.append([i, i + 1]); res.append(list(np.exp(rng.normal(4, 0.5)) / prices[[i, i + 1]]))
        fees.append(0.997); kinds.append("product"); w.append(None)
    li.append([0, 1]); res.append([300.0, 310.0]); fees.append(0.9996); kinds.append("stableswap"); w.append((100.0, 1, 1))
    li.append([0, 1, 2]); res.append([200.0, 190.0, 80.0]); fees.append(0.9996); kinds.append("stableswap")
    w.append((50.0, 1.0, 1.0, 2.5))
    li.append([2, 3]); res.append([5.0, 6.0]); fees.append(0.999); kinds.append("sum"); w.append(None)
    for a, b in ((0, 2), (3, 4)):
        t = int(rng.integers(T[0], T[1] + 1))
        p = prices[a] / prices[b] * np.exp(rng.normal(0, 0.03))
        bounds = p * np.exp(np.linspace(-0.2, 0.2, t + 1) + rng.normal(0, 0.001))
        liq = np.exp(rng.normal(5, 1, t)) * (rng.random(t) >= empty); liq[t // 2] = 100.0
        li.append([a, b]); res.append(None); fees.append(0.997); kinds.append("concentrated")
        w.append((p, bounds, liq))
    hp = HostPools.from_lists(n, li, res, fees, kinds, w)
    return hp, dict(local_indices=li, reserves=res, fees=fees, kinds=kinds, weights=w), prices


def _csr_args(hp):
    """the cfmm_csr_pools arrays and the records, as CsrStore writes them"""
    slot_kind = np.repeat(hp.kind, np.diff(hp.pool_ptr))
    w = hp.weights.copy()
    logrw = np.log(np.maximum(hp.reserves, 1e-300) / np.where(slot_kind == 0, hp.weights, 1.0))
    ss = np.nonzero(hp.kind == 4)[0]
    logrw[hp.pool_ptr[ss]] = hp.amp[ss]; logrw[hp.pool_ptr[ss] + 1] = hp.inv[ss]
    cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    f = hp.pool_ptr[cl]
    w[f], w[f + 1] = hp.lad_sc[cl, 0], hp.lad_sc[cl, 1]
    logrw[f], logrw[f + 1] = hp.lad_ptr[cl], hp.lad_ptr[cl + 1] - hp.lad_ptr[cl] - 1
    rec = np.ascontiguousarray(hp.lad_rec if len(hp.lad_rec) else np.zeros((1, 4)))
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
    fn = _host().ladder_host_solve
    fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 8 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
    fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), tol)
    return dict(nu=nu, psi=psi, stats=st, delta=d, lam=l)


def _result(hp, out, p):
    ptr = hp.pool_ptr
    return types.SimpleNamespace(value=out["stats"][p][0], dual_value=out["stats"][p][1], psi=out["psi"][p],
                                 nu=out["nu"][p], deltas=[out["delta"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                 lambdas=[out["lam"][p][ptr[i]:ptr[i + 1]] for i in range(hp.m)])


def _utils(n, prices, rng):
    return [cf.Arbitrage(prices * np.exp(0.02 * rng.standard_normal(n))), cf.Swap(0, 4, 30.0),
            cf.Liquidate(0, np.r_[0.0, 5.0, 3.0, 2.0, 1.0])]


def _sum_ranges(hp, rg, owner, trades):
    """per pool of the ladder market: the sum of its ranges' trades (trades: Result.deltas / lambdas of the range form,
    one vector per pool, or one CSR array for stores of more than 100k pools)"""
    flat = np.concatenate([np.asarray(x, float).ravel() for x in trades])
    sel = np.nonzero(hp.kind[owner] == KIND_CONCENTRATED_HOST)[0]
    out = np.zeros((hp.m, 2))
    np.add.at(out, owner[sel], flat[rg.pool_ptr[sel][:, None] + np.arange(2)])
    return out


def test_host_solver_ladders_and_ranges_agree():
    """the concentrated instance solves the market and the same market as ranges to the same value and psi, certified"""
    for seed in range(4):
        rng = np.random.default_rng(300 + seed)
        hp, _, prices = _small_market(rng)
        rg, owner = I.ladder_ranges(hp)
        us = [u.spec(hp.n_tokens) for u in _utils(hp.n_tokens, prices, rng)]
        a = _host_solve(hp, us)
        b = _host_solve(rg, us)
        for p, u in enumerate(us):
            assert int(a["stats"][p][7]) == 0 and int(b["stats"][p][7]) == 0, (seed, p, a["stats"][p], b["stats"][p])
            sc = abs(a["stats"][p][1])
            assert abs(a["stats"][p][0] - b["stats"][p][0]) <= 1e-8 * sc
            np.testing.assert_allclose(a["psi"][p], b["psi"][p], rtol=1e-6, atol=1e-7 * np.abs(b["psi"][p]).max())
            XC.certify(hp, u, _result(hp, a, p), 1e-9)


def test_validation():
    b, L = [1.0, 1.1, 1.3], [5.0, 0.0]
    ok = lambda **kw: HostPools.from_lists(2, [kw.get("li", [0, 1])], [kw.get("R", None)], [0.997], ["concentrated"],
                                           [kw.get("w", (1.05, b, L))])
    ok().validate()
    bad = [dict(li=[0, 1, 1]), dict(li=[0, 0]), dict(R=[1.0, 1.0]), dict(w=(1.05, [1.0, 1.0, 1.3], L)),
           dict(w=(1.05, [1.0, 1.3, 1.1], L)), dict(w=(1.05, [0.0, 1.1, 1.3], L)), dict(w=(1.05, [1.0, np.inf, 1.3], L)),
           dict(w=(1.05, b, [-1.0, 2.0])), dict(w=(1.05, b, [np.nan, 2.0])), dict(w=(1.05, b, [0.0, 0.0])),
           dict(w=(0.0, b, L)), dict(w=(-1.0, b, L)), dict(w=(np.nan, b, L)), dict(w=(np.inf, b, L)),
           dict(w=(1.05, b, [1.0])), dict(w=(1.05, [1.0], [])), dict(w=(1.05, b))]
    for kw in bad:
        with pytest.raises(ValueError):
            ok(**kw)
    big = np.exp(np.linspace(0, 1, LADDER_T_MAX + 2))
    with pytest.raises(ValueError):                                      # more intervals than the cap
        ok(w=(1.5, big, np.ones(LADDER_T_MAX + 1)))
    hp = ok()
    for field, val in (("lad_sc", np.array([[2.0, 0.0]])), ("lad_sc", np.array([[1.05, 0.0]]))):
        h2 = HostPools(2, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind, None, None, hp.lad_ptr,
                       hp.lad_rec, val)
        with pytest.raises(ValueError):
            h2.validate()
    r2 = hp.lad_rec.copy(); r2[-1, 1] = 1.0
    with pytest.raises(ValueError):
        HostPools(2, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind, None, None, hp.lad_ptr, r2,
                  hp.lad_sc).validate()
    with pytest.raises(ValueError):                                      # reserves= on a concentrated pool
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], np.array([[1.0, 1.0]]))
    with pytest.raises(ValueError):
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], prices=[-1.0])
    hq = HostPools.from_lists(2, [[0, 1]], [[1.0, 1.0]], [0.997], ["product"], [None])
    with pytest.raises(ValueError):                                      # prices= on another kind
        check_pool_update(hq.pool_ptr, hq.kind, hq.weights, [0], prices=[1.0])
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], fees=[0.99], prices=[1.2])
    assert u.prices[0] == 1.2 and u.gamma[0] == 0.99


def test_state_is_elementwise_and_clamped():
    bounds, liq, price = random_ladders(50, 8, 3)
    hp = ladder_hp(bounds, liq, price, np.full(50, 0.997))
    ids = np.array([3, 17, 40])
    s, c, x, y = ladder_state(hp.lad_ptr, hp.lad_rec, ids, price[ids])
    assert np.array_equal(s, hp.lad_sc[ids, 0]) and np.array_equal(c, hp.lad_sc[ids, 1])
    assert np.array_equal(x, hp.reserves[2 * ids]) and np.array_equal(y, hp.reserves[2 * ids + 1])
    s, c, x, y = ladder_state(hp.lad_ptr, hp.lad_rec, [0, 0], [bounds[0, 0] * 0.01, bounds[0, -1] * 100])
    b = hp.lad_rec[hp.lad_ptr[0]:hp.lad_ptr[1]]
    assert s[0] == b[0, 0] and c[0] == 0 and y[0] == 0 and s[1] == b[-1, 0] and c[1] == 7 and x[1] == 0


def test_pack_problems_shifts_record_offsets():
    from cfmm_routing_code_b200 import batch as B
    rng = np.random.default_rng(5)
    probs = [(_small_market(rng)[0], cf.Swap(0, 4, 10.0)) for _ in range(3)]
    merged = B.pack_problems(probs)[0]
    merged.validate()
    k = 0
    for hp, _ in probs:
        for i in np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]:
            j = k + i
            a = merged.lad_rec[merged.lad_ptr[j]:merged.lad_ptr[j + 1]]
            assert np.array_equal(a, hp.lad_rec[hp.lad_ptr[i]:hp.lad_ptr[i + 1]])
            assert np.array_equal(merged.lad_sc[j], hp.lad_sc[i])
        k += hp.m


def test_market_generator_and_ranges():
    hp, prices = I.synth_concentrated_market(4000, 40, seed=2, T=(1, 128))
    hp.validate()
    assert {0, 1, 3, 4, 6} <= set(np.unique(hp.kind).tolist())
    rg, owner = I.ladder_ranges(hp)
    rg.validate()
    nu = prices * np.exp(0.02 * np.random.default_rng(0).standard_normal(hp.n_tokens))
    a, b = XC.response(hp, nu), XC.response(rg, nu)
    assert abs(float(a["arb"].sum() - b["arb"].sum())) <= 1e-12 * float(np.abs(a["arb"]).sum())


# ====================================================================================================== GPU
gpu = pytest.mark.gpu
_REF = {}


def _big_bucket():
    """>= 100k ladder pools with 1..512 intervals over 64 tokens, the reference and the range form (computed once)"""
    if "big" not in _REF:
        hp, prices = I.synth_concentrated_market(100_000, 64, seed=21, T=(1, 512), frac_ladder=1.0)
        nu = prices * np.exp(0.03 * np.random.default_rng(1).standard_normal(64))
        rg, owner = I.ladder_ranges(hp)
        _REF["big"] = (hp, nu, XC.response(hp, nu), rg, owner)
    return _REF["big"]


@gpu
@pytest.mark.parametrize("trades,hess", [(False, False), (True, False), (False, True), (True, True)])
def test_kernel_matches_reference_and_ranges(trades, hess):
    import torch
    hp, nu, ref, rg, owner = _big_bucket()
    assert (hp.kind == KIND_CONCENTRATED_HOST).sum() >= 100_000
    st = cf.PoolStore(hp)
    assert [int(b.kind) for b in st.buckets] == [_lib.KIND_CONCENTRATED]
    nud = torch.as_tensor(nu, dtype=torch.float64, device="cuda")
    acc = st.evaluate(nud, 0.0, trades=trades, hess=hess).cpu().numpy()
    sel = np.arange(hp.m)
    Dx, Lx = ref["delta"].reshape(-1, 2).astype(float), ref["lam"].reshape(-1, 2).astype(float)
    tol = ladder_tol(hp, sel, nu, Dx, Lx)
    psi_x, gross, k = X.flows(hp, ref["delta"], ref["lam"])
    b_tok = np.zeros(hp.n_tokens); np.add.at(b_tok, hp.tok_idx, tol.ravel())
    lim = b_tok + 4 * U * np.maximum(k.astype(float), 1) * gross.astype(float)
    r_psi = (np.abs(acc[:-1] - psi_x.astype(float)) / lim).max()
    lim_arb = float((nu[hp.tok_idx].reshape(-1, 2) * tol).sum() + 4 * hp.m * U * (nu * gross.astype(float)).sum())
    assert abs(acc[-1] - float(ref["arb"].sum())) <= lim_arb
    b = st.buckets[0]
    if trades:
        Dk, Lk = b.delta[:, :hp.m].cpu().numpy().T, b.lam[:, :hp.m].cpu().numpy().T
        r_tr = (np.maximum(np.abs(Dk - Dx), np.abs(Lk - Lx)) / tol).max()
        assert r_tr <= 0.25, r_tr
        d, l = st.gather_trades()
        assert np.array_equal(d.reshape(-1, 2), Dk) and np.array_equal(l.reshape(-1, 2), Lk)
        print(f"trades observed / bound {r_tr:.3g}")
    # the range-decomposed bucket (kind 3): psi, arb and hcoef to summation-order tolerance
    sr = cf.PoolStore(rg)
    assert [int(x.kind) for x in sr.buckets] == [_lib.KIND_BOUNDED]
    acc_r = sr.evaluate(nud, 0.0, trades=False, hess=hess).cpu().numpy()
    assert np.all(np.abs(acc[:-1] - acc_r[:-1]) <= 2 * lim)
    assert abs(acc[-1] - acc_r[-1]) <= 2 * lim_arb
    if hess:
        hk = b.hcoef[:hp.m].cpu().numpy()
        hr = np.zeros(hp.m); np.add.at(hr, owner, sr.buckets[0].hcoef[:rg.m].cpu().numpy())
        hx = ref["h"].astype(float)
        edge = np.abs(hk - hx) > 1e-12 * np.maximum(hk, hx)
        assert edge.mean() <= 1e-3, edge.mean()                           # targets within rounding of a bound
        assert np.all(np.abs(hk - hr)[~edge] <= 1e-12 * np.maximum(hk, hr)[~edge] + 1e-300)
    print(f"psi observed / bound {r_psi:.3g}")
    assert r_psi <= 0.25


def _mixed(m, n, seed, T=(1, 64)):
    hp, prices = I.synth_concentrated_market(m, n, seed, T=T)
    return hp, prices


@gpu
def test_hessian_kernels_match_the_decomposition():
    import torch
    hp, prices = _mixed(60_000, 200, 4)
    rg, _ = I.ladder_ranges(hp)
    st, sr = cf.PoolStore(hp), cf.PoolStore(rg)
    nu = torch.as_tensor(prices * np.exp(0.01 * np.random.default_rng(0).standard_normal(200)), dtype=torch.float64,
                         device="cuda")
    st.evaluate(nu, 0.0, hess=True); sr.evaluate(nu, 0.0, hess=True)
    H, Hr = st.hess_dense().cpu().numpy(), sr.hess_dense().cpu().numpy()
    sc = np.abs(Hr).max()
    np.testing.assert_allclose(H, Hr, rtol=0, atol=1e-9 * sc)
    v = np.random.default_rng(1).standard_normal(200)
    vt = torch.as_tensor(v, dtype=torch.float64, device="cuda")
    np.testing.assert_allclose(st.hvp(vt).cpu().numpy(), H @ v, rtol=0, atol=1e-11 * sc * np.abs(v).sum())
    np.testing.assert_allclose(st.hess_diag().cpu().numpy(), np.diag(Hr), rtol=1e-9, atol=1e-12 * sc)


def _check_answer(hp, rg, owner, u, r, rr, tol):
    """certificate; value, nu, psi vs the decomposed market's solve; each ladder's trade vs the sum of its ranges'"""
    XC.certify(hp, u.spec(hp.n_tokens), r, tol)
    sc = max(abs(r.dual_value), 1e-300)
    assert abs(r.value - rr.value) <= 20 * tol * sc, (r.value, rr.value)
    # nu is unique only up to the fee bands of the pools that do not trade at the optimum: within 1 - gamma
    np.testing.assert_allclose(r.nu, rr.nu, rtol=1.0 - float(hp.gamma.min()))
    gross = np.abs(np.asarray(r.psi)).max()
    np.testing.assert_allclose(r.psi, rr.psi, rtol=0, atol=1e-5 * gross + 1e-9)
    if len(r.deltas) == hp.m:
        cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
        d = _sum_ranges(hp, rg, owner, rr.deltas)
        l = _sum_ranges(hp, rg, owner, rr.lambdas)
        D = np.stack([r.deltas[i] for i in cl]); L = np.stack([r.lambdas[i] for i in cl])
        scl = np.abs(D).sum(1) + np.abs(L).sum(1) + hp.reserves[hp.pool_ptr[cl][:, None] + np.arange(2)].sum(1)
        # two solves to tol: their prices differ by the conditioning of the dual; the ladders' trades follow
        assert np.all(np.maximum(np.abs(D - d[cl]), np.abs(L - l[cl])).max(1) <= 1e-4 * scl + 1e-9)


@gpu
@pytest.mark.parametrize("linear_solver", ["dense", "cg"])
def test_solver_py_paths(linear_solver):
    hp, prices = _mixed(60_000, 120, 5)
    rg, owner = I.ladder_ranges(hp)
    store = cf.PoolStore(hp)
    assert _lib.KIND_CONCENTRATED in {int(b.kind) for b in store.buckets}
    assert {_lib.KIND_STABLESWAP, _lib.KIND_STABLESWAP_N, _lib.KIND_BOUNDED, _lib.KIND_SUM} <= {int(b.kind) for b in store.buckets}
    rng = np.random.default_rng(1)
    for u in (cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(hp.n_tokens))), cf.Swap(3, 9, 500.0 / prices[3])):
        r = cf.solve_pools(hp, u, tol=1e-8, store=store, linear_solver=linear_solver, want_trades=True)
        assert r.status == "optimal" and r.info.history                  # solver.py ran (the native solvers keep none)
        rr = cf.solve_pools(rg, u, tol=1e-8, linear_solver=linear_solver)
        assert rr.status == "optimal"
        # hp.m <= 100k: one trade pair per pool
        _check_answer(hp, rg, owner, u, r, rr, 1e-8)


@gpu
def test_thread_sweep_batch_and_many():
    from cfmm_routing_code_b200 import batch as B
    rng = np.random.default_rng(9)
    probs = [_small_market(rng) for _ in range(3)]
    for hp, d, prices in probs:
        rg, owner = I.ladder_ranges(hp)
        assert B.CsrStore(hp).has_ladder and not B.CsrStore(rg).has_ladder
        for u in _utils(hp.n_tokens, prices, rng):
            r = cf.solve_pools(hp, u, tol=1e-9, method="thread")
            assert r.status == "optimal" and r.info is None                # the per-thread solver ran
            rr = cf.solve_pools(rg, u, tol=1e-9, method="thread")
            _check_answer(hp, rg, owner, u, r, rr, 1e-9)
            # solver.py's stopping rule bounds the exact gap of a smoothed constant-sum solve by its tol only loosely:
            # solved one decade tighter, the answer must certify at 1e-9 like the others
            rp = cf.solve(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], utility=u,
                          method="pools", tol=1e-10)
            assert rp.status == "optimal" and rp.info.history
            _check_answer(hp, rg, owner, u, rp, rr, 1e-9)
        sw = [cf.Swap(0, 4, t) for t in np.linspace(1.0, 60.0, 32)]
        for us in (sw[:1], sw):                                            # 1 and 32 problems: a warp / a thread each
            res = cf.solve_sweep(d["local_indices"], d["reserves"], d["fees"], d["kinds"], d["weights"], us,
                                 batched=True)
            resr = B.solve_batch(rg, us, tol=1e-8)
            for u, x, y in zip(us, res, resr):
                assert x.status == "optimal" and x.info is None
                _check_answer(hp, rg, owner, u, x, y, 1e-8)
            res2 = B.solve_batch(hp, us, tol=1e-8)
            for x, y in zip(res2, res):
                assert abs(x.value - y.value) <= 1e-12 * abs(y.dual_value)
        for lanes in (1, 32):
            store = B.CsrStore(hp)
            import torch
            c, a, fl, nu = B.pack_utilities(sw, hp.n_tokens)
            up = lambda x: torch.as_tensor(x, device="cuda")
            psi, stats, dl, lm = B.solve_batch_device(store, up(c), up(a), up(fl), up(nu), tol=1e-9, lanes=lanes)
            assert np.all(stats.cpu().numpy()[:, 7] == 0)
    many = cf.solve_many([(hp, cf.Swap(0, 4, 20.0)) for hp, _, _ in probs])
    for (hp, _, _), r in zip(probs, many):
        assert r.status == "optimal"
        rg, owner = I.ladder_ranges(hp)
        rr = cf.solve_pools(rg, cf.Swap(0, 4, 20.0), tol=1e-8, method="thread")
        _check_answer(hp, rg, owner, cf.Swap(0, 4, 20.0), r, rr, 1e-8)


@gpu
def test_two_150_interval_pools_run_on_the_per_thread_path():
    rng = np.random.default_rng(4)
    hp, d, prices = _small_market(rng, T=(150, 150), empty=0.0)
    assert np.all(np.diff(hp.lad_ptr)[hp.kind == KIND_CONCENTRATED_HOST] == 151)
    rg, owner = I.ladder_ranges(hp)
    assert rg.m > cf.api.SMALL_POOLS >= hp.m
    u = cf.Swap(0, 4, 25.0)
    r = cf.solve_pools(hp, u, tol=1e-9)
    assert r.status == "optimal" and r.info is None and r.hvps == 0        # method 'auto' picked the per-thread solver
    rr = cf.solve_pools(rg, u, tol=1e-9)
    assert rr.info is not None                                             # the ranges fall off it
    _check_answer(hp, rg, owner, u, r, rr, 1e-9)


@gpu
def test_update_prices_and_fees_equals_a_fresh_store():
    import torch
    rng = np.random.default_rng(2)
    hp, prices = _mixed(40_000, 100, 6)
    store = cf.PoolStore(hp)
    u = cf.Arbitrage(prices)
    r0 = cf.solve_pools(hp, u, tol=1e-8, store=store)
    cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    ids = np.sort(rng.choice(cl, 3000, replace=False))
    newp = hp.lad_sc[ids, 0] ** 2 * np.exp(0.03 * rng.standard_normal(len(ids)))
    newp[:5] = [1e-30, 1e30, hp.lad_rec[hp.lad_ptr[ids[2]], 0] ** 2, newp[3], newp[4]]
    newg = np.full(len(ids), 0.9991)
    plain = [b for b in store.buckets if not getattr(b, "blocked", False)]
    before = [(b.reserves.clone(), b.gamma.clone()) for b in plain]
    with pytest.raises(ValueError):                                       # reserves= on a concentrated pool: nothing written
        store.update_pools(ids[:2], reserves=np.ones((2, 2)))
    for b, (R, g) in zip(plain, before):
        assert torch.equal(b.reserves, R) and torch.equal(b.gamma, g)
    store.update_pools(ids, fees=newg, prices=newp)
    s, c, x, y = ladder_state(hp.lad_ptr, hp.lad_rec, ids, newp)
    sc2 = hp.lad_sc.copy(); sc2[ids, 0], sc2[ids, 1] = s, c
    R2 = hp.reserves.copy(); R2[hp.pool_ptr[ids]], R2[hp.pool_ptr[ids] + 1] = x, y
    g2 = hp.gamma.copy(); g2[ids] = newg
    hp2 = HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, R2, hp.weights, g2, hp.kind, hp.amp, None, hp.lad_ptr,
                    hp.lad_rec, sc2)
    hp2.validate()
    fresh = cf.PoolStore(hp2)
    for a, b in zip(store.buckets, fresh.buckets):
        assert (a.kind, a.arity) == (b.kind, b.arity)
        if getattr(a, "blocked", False):
            continue
        for t in ("reserves", "gamma", "weights", "logrw"):
            xa, xb = getattr(a, t), getattr(b, t)
            assert (xa is None) == (xb is None) and (xa is None or torch.equal(xa, xb)), (a.kind, t)
    r1 = cf.solve_pools(hp2, u, tol=1e-8, store=store, nu0=r0.nu)
    assert r1.status == "optimal"
    XC.certify(hp2, u.spec(hp.n_tokens), r1, 1e-8)


@gpu
def test_rank_stores_sum_to_the_single_store():
    import torch
    hp, prices = _mixed(30_000, 80, 7)
    nu = torch.as_tensor(prices, dtype=torch.float64, device="cuda")
    one = cf.PoolStore(hp).evaluate(nu, 0.0).cpu().numpy().copy()
    for world in (2, 3):
        tot = np.zeros_like(one)
        nrec = 0
        for r in range(world):
            st = cf.PoolStore(hp, rank=r, world=world)
            tot += st.evaluate(nu, 0.0, reduce=False).cpu().numpy()
            nrec += sum(int(b.weights.numel()) // 4 for b in st.buckets if b.kind == _lib.KIND_CONCENTRATED)
        assert nrec == len(hp.lad_rec)                                    # every rank uploads only its pools' records
        np.testing.assert_allclose(tot, one, rtol=1e-12, atol=1e-12 * np.abs(one).max())


@gpu
def test_c_abi_codes():
    import torch
    lib = _lib.load()
    buf = torch.ones(8 * 1024, dtype=torch.float64, device="cuda")
    idx = torch.zeros(8 * 1024, dtype=torch.int32, device="cuda")
    nu = torch.ones(4, dtype=torch.float64, device="cuda")
    acc = torch.zeros(5, dtype=torch.float64, device="cuda")
    p = buf.data_ptr()

    def ev(arity, w, lr):
        b = _lib.Bucket(_lib.KIND_CONCENTRATED, arity, 100, 1024, p, idx.data_ptr(), p, w, lr, None)
        return lib.cfmm_arb_eval(C.byref(b), 4, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc.data_ptr() + 32, None, None)
    assert ev(3, p, p) == -2 and ev(1, p, p) == -2
    assert ev(2, None, p) == -1 and ev(2, p, None) == -1
    from cfmm_routing_code_b200 import batch as B
    hp, _, _ = _small_market(np.random.default_rng(0))
    store = B.CsrStore(hp)
    work = store.work(1)
    f = torch.zeros(8, dtype=torch.float64, device="cuda")
    bt = _lib.Batch(1, None, f.data_ptr(), f.data_ptr(), f.data_ptr(), f.data_ptr(), f.data_ptr(), f.data_ptr(), None,
                    None, 0)
    prm = _lib.BatchParams(1e-8, 0.1, 1e-4, 0.5, 1e-12, 60, 100)
    assert lib.cfmm_batch_solve_concentrated(C.byref(store.c_pools), None, C.byref(bt), C.byref(prm), work.data_ptr(),
                                             None) == -1
    torch.cuda.synchronize()
