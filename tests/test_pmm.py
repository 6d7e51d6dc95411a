"""DODO proactive-market-maker (PMM) pools as one pool kind (host kind 12, CFMM_KIND_PMM).

CPU: cfmm_small::pmm_pair compiled for the host against the mpmath reference (tests/xp_pmm.py: the curve's two pieces
as points, flows as differences of points at 60 digits) on random pools with k log-uniform over [PMM_K_MIN, 1], pi over
16 decades, states on both pieces (from a hair to far off the meeting point) and at it, prices on both sides of the
pool's, within 1e-12 of it, in the no-trade band, and across pi (two-leg trades); hc against the reference's central
differences; post-trade feasibility; the mirror pool; homogeneity and token-1 units; the k = 1 product limit and the k
-> 0 constant-sum limit; the target rule against mpmath; the validation rules; pmm_pool against decimal; the host-built
per-thread solver, certified and against a scipy primal solve.
GPU (H100): k_eval_pair<PMM> in all four (trades, hess) instances under both scatter strategies on 10^6 pools against
the host build, and through the launch-strategy harness of tests/test_launch_strategies.py; the Hessian kernels;
certified solves on solver.py, the host loop and native=True, mixed with every other kind, and on the per-thread
paths; stores sharded over 1-3 ranks; reserve, fee and pmm= updates equal to a fresh store; the C ABI codes.

Error bound.  Both sides read the same f64 parameters, targets and reserves.  The kernel computes each flow from one
subtraction of the short coordinate (or the cancellation-free T z / (w (w + 1))) times a sum of positive terms, so its
error is a few ulp of the flow, plus the error of the price p* = nu0 / (gamma nu1) (a few ulp, amplified by the flow's
sensitivity p* |d flow / d p*|), plus a few ulp of the reserve where the end point is rounded next to it.  The tests
allow 64 u (R_j + |flow_j| + p* |d flow_j / d p*|), u = 2^-53, per flow, as for the other closed-form kinds.
"""
import ctypes as C
import os
import subprocess

import mpmath as mp
import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib
from cfmm_routing_code_b200.pools import HostPools, KIND_ECLP_HOST, KIND_PMM_HOST, PMM_K_MIN, pmm_targets
import xp_pmm as XM

HERE = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -53
p_ = lambda x: x.ctypes.data_as(C.c_void_p)
_HOST = None


def _host():
    """tests/host_harness/pmm_host.cpp: cfmm_small::pmm_pair, host build"""
    global _HOST
    if _HOST is None:
        src = os.path.join(HERE, "host_harness", "pmm_host.cpp")
        hdr = os.path.join(HERE, "..", "cfmm_routing_code_b200", "csrc", "cfmm_small.cuh")
        lib = os.path.join(HERE, "_build", "libpmm_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src],
                           check=True)
        _HOST = C.CDLL(lib)
    return _HOST


def host_pairs(R, P, g, n0, n1):
    """pmm_pair of every pool: R [m, 2] = (B, Q), P [m, 4] = (pi, k, B0, Q0); returns D, L [m, 2], hc [m]"""
    m = len(g)
    D, L, hc = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m)
    f = _host().pmm_host_pools
    f.argtypes = [C.c_longlong] + [C.c_void_p] * 8
    c = lambda a: np.ascontiguousarray(a, np.float64)
    f(m, p_(c(R)), p_(c(P)), p_(c(g)), p_(c(n0)), p_(c(n1)), p_(D), p_(L), p_(hc))
    return D, L, hc


def pool_price(R, P):
    """the pools' marginal price (f64; the decisions below keep a margin from it)"""
    B, Q = R[:, 0], R[:, 1]
    pi, k, B0, Q0 = P.T
    return np.where(B < B0, pi * (1 - k + k * (B0 / B) ** 2), np.where(Q < Q0, pi / (1 - k + k * (Q0 / Q) ** 2), pi))


def random_pools(rng, m):
    """(R, P): pi over 16 decades, k log-uniform over [PMM_K_MIN, 1], targets of different value, a third of the pools
    at the meeting point and a third on each piece, from 1e-9 to 0.999 of the short target off it; P after the target
    rule"""
    pi = 10.0 ** rng.uniform(-8, 8, m)
    k = np.exp(rng.uniform(np.log(PMM_K_MIN), 0.0, m))
    B0 = 10.0 ** rng.uniform(-3, 6, m)
    Q0 = pi * B0 * 10.0 ** rng.uniform(-3, 3, m)
    side = rng.integers(0, 3, m)
    f = 1.0 - 10.0 ** rng.uniform(-9, np.log10(0.999), m)          # short reserve over its target
    B = np.where(side == 1, B0 * f, B0)
    Q = np.where(side == 2, Q0 * f, Q0)
    Q = np.where(side == 1, Q0 + pi * (B0 - B) * (1 + k * (B0 - B) / B), Q)
    B = np.where(side == 2, B0 + (Q0 - Q) * (1 + k * (Q0 - Q) / Q) / pi, B)
    R = np.stack([B, Q], axis=1)
    P = pmm_targets(R, np.stack([pi, k, np.where(side == 1, np.maximum(B0, np.nextafter(B, np.inf)), B0),
                                 np.where(side == 2, np.maximum(Q0, np.nextafter(Q, np.inf)), Q0)], axis=1))
    return R, P


def random_prices(rng, R, P, g):
    """the mid price nu0 / nu1 of each pool: far either side, within 1e-12 .. 1e-3 of the pool's price, in the no-trade
    band, across pi (a trade in two legs) and within 1e-12 .. 1e-3 of pi"""
    m = len(g)
    Pp, pi = pool_price(R, P), P[:, 0]
    mode = rng.integers(0, 5, m)
    far = Pp * 10.0 ** rng.uniform(-4, 4, m)
    near = Pp * (1 + np.where(rng.random(m) < 0.5, -1, 1) * 10.0 ** rng.uniform(-12, -3, m))
    band = Pp * g ** rng.uniform(-0.99, 0.99, m)
    across = pi * np.where(Pp >= pi, 10.0 ** -rng.uniform(0, 2, m), 10.0 ** rng.uniform(0, 2, m))
    at_pi = pi * (1 + np.where(rng.random(m) < 0.5, -1, 1) * 10.0 ** rng.uniform(-12, -3, m))
    ps = np.choose(mode, [far, near, band, across, at_pi])
    n1 = 10.0 ** rng.uniform(-2, 2, m)
    return ps * n1, n1


def case_set(seed, m):
    rng = np.random.default_rng(seed)
    R, P = random_pools(rng, m)
    g = np.where(rng.random(m) < 0.3, 1.0, 1.0 - 10.0 ** rng.uniform(-4, -1.5, m))
    n0, n1 = random_prices(rng, R, P, g)
    return R, P, g, n0, n1


def reference(P, R, g, n0, n1, D, L):
    """xp_pmm.reference_rows over all pools, on every core"""
    from concurrent.futures import ProcessPoolExecutor
    import multiprocessing as mpr
    n = max(1, min(os.cpu_count() or 1, 32))
    parts = np.array_split(np.arange(len(g)), 4 * n)
    chunks = [(P[k], R[k], g[k], n0[k], n1[k], D[k], L[k]) for k in parts if len(k)]
    if n == 1 or len(g) < 2000:
        return np.concatenate([XM.reference_rows(c) for c in chunks])
    with ProcessPoolExecutor(n, mp_context=mpr.get_context("spawn")) as ex:    # workers import xp_pmm only
        return np.concatenate(list(ex.map(XM.reference_rows, chunks)))


def check_against_reference(P, R, g, n0, n1, D, L, hc):
    """every flow within 64 u (R_j + |flow_j| + p* |d flow_j / d p*|) of the reference; hc within 1e-7 of the
    reference's central difference; the post-trade state on or above the curve within 64 u of the pool's value at the
    trade's price; returns the worst normalised flow error"""
    ref = reference(P, R, g, n0, n1, D, L)
    dy = np.abs(ref[:, 4:6])
    worst = 0.0
    for j in range(2):
        for kern, want in ((D[:, j], ref[:, j]), (L[:, j], ref[:, 2 + j])):
            tol = 64 * U * (R[:, j] + np.abs(want) + dy[:, j])
            err = np.abs(kern - want)
            bad = np.nonzero(err > tol)[0]
            assert len(bad) == 0, [(i, P[i], R[i], g[i], n0[i], n1[i], kern[i], want[i]) for i in bad[:3]]
            worst = max(worst, float(np.max(np.where(tol > 0, err / np.where(tol > 0, tol, 1), 0.0), initial=0.0)))
    # post-trade: b', q' > 0 and on or above the curve, in token 1 at the larger of the pool's and the trade's price
    ps = np.maximum(ref[:, 7], np.maximum(n0 / (g * n1), g * n0 / n1))
    scale = 64 * U * (R[:, 1] + ps * R[:, 0] + np.abs(D[:, 1]) + np.abs(L[:, 1]) + dy[:, 1]
                      + ps * (np.abs(D[:, 0]) + np.abs(L[:, 0]) + dy[:, 0]))
    assert np.all(ref[:, 9] > 0) and np.all(ref[:, 10] > 0)
    bad = np.nonzero(ref[:, 8] < -scale)[0]
    assert len(bad) == 0, [(i, P[i], R[i], ref[i, 8], scale[i]) for i in bad[:3]]
    # hc jumps where p* crosses a kink of the pool's dual (its price, and pi, where the curvature of the two pieces
    # differs): within a few ulp of one the kernel's rounded p* and the reference's exact one may lie on either side
    kink = np.zeros(len(g), bool)
    for p in (n0 / (g * n1), g * n0 / n1):
        for kp in (ref[:, 7], P[:, 0]):
            kink |= np.abs(p - kp) <= 8 * U * kp
    hr = ref[:, 6]
    bad = np.nonzero(~kink & (np.abs(hc - hr) > 1e-7 * np.abs(hr)))[0]
    assert len(bad) == 0, [(i, P[i], R[i], g[i], n0[i], n1[i], hc[i], hr[i]) for i in bad[:3]]
    return worst


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
N_PAIR = int(os.environ.get("PMM_TEST_POOLS", "100000"))


def test_pmm_pair_against_reference():
    """10^5 random pools (PMM_TEST_POOLS to change it), every flow, hc and the post-trade state against the 60-digit
    reference"""
    R, P, g, n0, n1 = case_set(1, N_PAIR)
    D, L, hc = host_pairs(R, P, g, n0, n1)
    assert np.all(np.isfinite(D)) and np.all(np.isfinite(L)) and np.all(np.isfinite(hc))
    assert np.all(D >= 0) and np.all(L >= 0) and np.all(hc >= 0)
    # every kind of trade occurs: both directions, two legs (across pi) both ways, and none
    t0, t1 = D[:, 0] > 0, D[:, 1] > 0
    pp = pool_price(R, P)
    ps = np.where(t0, n0 / (g * n1), g * n0 / n1)
    assert t0.sum() > N_PAIR // 5 and t1.sum() > N_PAIR // 5 and (~t0 & ~t1).sum() > N_PAIR // 20
    assert (t0 & (pp > P[:, 0]) & (ps < P[:, 0])).sum() > N_PAIR // 50
    assert (t1 & (pp < P[:, 0]) & (ps > P[:, 0])).sum() > N_PAIR // 50
    check_against_reference(P, R, g, n0, n1, D, L, hc)


def test_no_trade_band_is_exact():
    R, P, g, _, _ = case_set(2, 3000)
    R, P, g = R[g < 1], P[g < 1], g[g < 1]                              # at gamma = 1 the band is the one price P
    rng = np.random.default_rng(3)
    n1 = 10.0 ** rng.uniform(-2, 2, len(g))
    n0 = pool_price(R, P) * g ** rng.uniform(-0.999, 0.999, len(g)) * n1
    D, L, hc = host_pairs(R, P, g, n0, n1)
    assert np.all(D == 0) and np.all(L == 0) and np.all(hc == 0)


def test_mirror_pool_trades_the_mirror_image():
    """(b <-> q, B0 <-> Q0, pi -> 1/pi) at swapped prices: the mirror trade; 1/pi is rounded, which moves the flows by
    a few ulp times their sensitivity"""
    R, P, g, n0, n1 = case_set(5, 4000)
    pi, k, B0, Q0 = P.T
    Pm = np.stack([1 / pi, k, Q0, B0], axis=1)
    Rm = R[:, ::-1].copy()
    D, L, hc = host_pairs(R, P, g, n0, n1)
    Dm, Lm, hcm = host_pairs(Rm, Pm, g, n1, n0)
    pp = pool_price(R, P)
    ok = np.ones(len(g), bool)                                          # away from the band's edges and from pi
    for p in (n0 / (g * n1), g * n0 / n1):
        ok &= (np.abs(np.log(p / pp)) > 1e-9) & (np.abs(np.log(p / pi)) > 1e-9)
    ps = np.where(D[:, 0] > 0, n0 / (g * n1), g * n0 / n1)
    # p* |d flow_0 / d p*| = hc / nu0 (hc = nu0 p* |d flow_0 / d p*| for the gross flow), and token 1 moves p* times that
    s0 = hc / n0
    for j, sens in ((0, s0), (1, s0 * ps)):
        sc = R[:, j] + np.abs(D[:, j]) + np.abs(L[:, j]) + sens
        assert np.all((np.abs(Dm[:, 1 - j] - D[:, j]) <= 64 * U * sc)[ok])
        assert np.all((np.abs(Lm[:, 1 - j] - L[:, j]) <= 64 * U * sc)[ok])
    # hc is the coefficient of [[1, -1], [-1, 1]]: the same for the mirror, to its own sensitivity to p* / pi
    rel = 64 * U * (1 + ps / (P[:, 1] * np.minimum(ps, pi) + np.abs(ps - pi)))
    assert np.all((np.abs(hcm - hc) <= rel * np.abs(hc))[ok])


def test_homogeneity_and_token_units():
    R, P, g, n0, n1 = case_set(6, 4000)
    D, L, hc = host_pairs(R, P, g, n0, n1)
    for s in (2.0 ** 20, 2.0 ** -24):                    # reserves and targets scaled exactly: bit for bit
        P2 = P.copy(); P2[:, 2:] *= s
        assert np.array_equal(pmm_targets(R * s, P2), P2)
        D2, L2, hc2 = host_pairs(R * s, P2, g, n0, n1)
        assert np.array_equal(D2, D * s) and np.array_equal(L2, L * s) and np.array_equal(hc2, hc * s)
        # token 1 counted in units 1/s: pi, Q, Q0 times s, nu1 over s; token-1 flows times s, the rest unchanged
        P3 = P.copy(); P3[:, 0] *= s; P3[:, 3] *= s
        R3 = R.copy(); R3[:, 1] *= s
        assert np.array_equal(pmm_targets(R3, P3), P3)
        D3, L3, hc3 = host_pairs(R3, P3, g, n0, n1 / s)
        assert np.array_equal(D3[:, 0], D[:, 0]) and np.array_equal(L3[:, 0], L[:, 0])
        assert np.array_equal(D3[:, 1], D[:, 1] * s) and np.array_equal(L3[:, 1], L[:, 1] * s)
        assert np.array_equal(hc3, hc)
    P4 = P.copy(); P4[:, 2:] *= 1e-7                     # an inexact scale: to rounding
    D4, L4, _ = host_pairs(R * 1e-7, P4, g, n0, n1)
    scl = (R.sum(1) + D.sum(1) + L.sum(1))[:, None] * 1e-7
    assert np.all(np.abs(D4 - D * 1e-7) <= 1e-6 * scl) and np.all(np.abs(L4 - L * 1e-7) <= 1e-6 * scl)


def test_k_one_is_the_product_pool():
    """k = 1 with Q0 = pi B0: both pieces are the hyperbola b q = pi B0^2, the constant-product pool"""
    rng = np.random.default_rng(8)
    m = 3000
    B = 10.0 ** rng.uniform(-2, 4, m)
    Q = 10.0 ** rng.uniform(-2, 4, m)
    pi = Q / B * 10.0 ** rng.uniform(-1, 1, m)                         # B0 = sqrt(BQ / pi), Q0 = pi B0
    B0 = np.sqrt(B * Q / pi)
    P = np.stack([pi, np.ones(m), B0, pi * B0], axis=1)
    g = np.where(rng.random(m) < 0.3, 1.0, 0.997)
    n1 = np.ones(m)
    n0 = Q / B * 10.0 ** rng.uniform(-2, 2, m)
    D, L, hc = host_pairs(np.stack([B, Q], 1), P, g, n0, n1)
    # constant product at price p* (the pool's curve b q = B Q): b* = sqrt(B Q / p*)
    lo, hi = n0 / (g * n1), g * n0 / n1
    t0, t1 = lo < Q / B, hi > Q / B
    ps = np.where(t0, lo, hi)
    bs, qs = np.sqrt(B * Q / ps), np.sqrt(B * Q * ps)
    # B0 and Q0 only reproduce the hyperbola through (B, Q) to rounding: compare at 1e-10 of the pool's depth
    for got, want, s in ((D[:, 0], np.where(t0, (bs - B) / g, 0.0), B + Q / ps), (L[:, 0], np.where(t1, B - bs, 0.0), B),
                         (D[:, 1], np.where(t1, (qs - Q) / g, 0.0), Q + B * ps), (L[:, 1], np.where(t0, Q - qs, 0.0), Q)):
        assert np.all(np.abs(got - want) <= 1e-10 * (s + np.abs(want))), np.max(np.abs(got - want) / (s + np.abs(want)))


def test_small_k_converges_to_the_sum_pool_at_sqrt_k():
    """pi = 1, k -> 0: the pool (B, Q) becomes the constant-sum pool at price 1 with the same reserves (eps = 0: all of
    one reserve at a price past the band), the error falling as sqrt(k)"""
    rng = np.random.default_rng(9)
    m = 400
    B = 10.0 ** rng.uniform(0, 3, m)
    Q = B * 10.0 ** rng.uniform(-1, 1, m)       # the O(k (Q / B)) terms stay below the sqrt(k) term's 1 %
    g = np.full(m, 0.997)
    n1 = np.ones(m)
    n0 = np.where(rng.random(m) < 0.5, 0.9, 1.1)                      # past the band on either side of pi = 1
    side = rng.integers(0, 2, m)                                       # at the meeting point, or base short
    err = {}
    for k in (1e-6, 1e-8):                     # the math, so also below PMM_K_MIN
        W = pmm_targets(np.stack([B, Q], 1), np.stack([np.ones(m), np.full(m, k), np.where(side == 1, 2 * B, B),
                                                       np.where(side == 1, Q / 2, Q)], axis=1))
        D, L, _ = host_pairs(np.stack([B, Q], 1), W, g, n0, n1)
        t0 = n0 < g * n1                                               # the sum pool pays out all of Q (or all of B)
        sD0, sL1 = np.where(t0, Q / g, 0.0), np.where(t0, Q, 0.0)
        sL0, sD1 = np.where(~t0, B, 0.0), np.where(~t0, B / g, 0.0)
        e = np.abs(np.stack([D[:, 0] - sD0, L[:, 1] - sL1, L[:, 0] - sL0, D[:, 1] - sD1])) / (B + Q)
        err[k] = e.max(0)
    ratio = err[1e-6] / err[1e-8]
    assert np.all(err[1e-6] < 0.01) and np.all((ratio > 9) & (ratio < 11)), (ratio.min(), ratio.max())


def test_targets_against_mpmath():
    rng = np.random.default_rng(10)
    m = 600
    pi = 10.0 ** rng.uniform(-6, 6, m); k = np.exp(rng.uniform(np.log(PMM_K_MIN), 0, m))
    B0 = 10.0 ** rng.uniform(-3, 6, m); Q0 = pi * B0 * 10.0 ** rng.uniform(-2, 2, m)
    side = rng.integers(0, 3, m)
    f = 10.0 ** rng.uniform(-12, 1, m)
    B = np.where(side == 1, B0 / (1 + f), B0 * (1 + f))                # given targets off the reserves either way
    Q = np.where(side == 2, Q0 / (1 + f), Q0 * (1 + f))
    R, G = np.stack([B, Q], 1), np.stack([pi, k, B0, Q0], 1)
    W = pmm_targets(R, G)
    assert np.array_equal(pmm_targets(R, W), W)                        # idempotent
    for i in range(m):
        # the reserves on or above the curve of the rounded targets (pmm_targets steps a target down until they are)
        assert XM.excess(*W[i], B[i], Q[i]) >= 0, (i, G[i], R[i], W[i])
        b0, q0 = XM.targets(B[i], Q[i], *G[i])
        assert abs(W[i, 2] - float(b0)) <= 4 * U * float(b0), (i, G[i], R[i], W[i], float(b0))
        assert abs(W[i, 3] - float(q0)) <= 4 * U * float(q0), (i, G[i], R[i], W[i], float(q0))
    assert np.array_equal(W[side == 0, 2:], R[side == 0])              # neither short: the reserves
    with pytest.raises(ValueError):
        pmm_targets([[1.0, 1.0]], [[1.0, 0.5, 2.0, 2.0]])              # both short


def test_validation():
    good = (100.0, 0.1, 20.0, 1500.0)

    def mk(w=good, r=(10.0, 2000.0), toks=(0, 1)):
        return HostPools.from_lists(2, [toks], [r], [0.997], ["pmm"], [w])
    hp = mk()
    assert hp.kind[0] == KIND_PMM_HOST and hp.pmm.shape == (1, 4) and hp.pmm[0, 3] == 1500.0 and hp.pmm[0, 2] > 10.0
    hp.validate()
    for w in ((0.0, 0.1, 20.0, 1500.0), (-1.0, 0.1, 20.0, 1500.0), (100.0, 1.5, 20.0, 1500.0),
              (100.0, PMM_K_MIN / 2, 20.0, 1500.0), (100.0, 0.1, 0.0, 1500.0), (100.0, 0.1, 20.0, -1.0),
              (float("nan"), 0.1, 20.0, 1500.0), (100.0, 0.1, float("inf"), 1500.0), good[:3]):
        with pytest.raises(ValueError):
            mk(w=w)
    with pytest.raises(ValueError, match="k = 0"):
        mk(w=(100.0, 0.0, 20.0, 1500.0))
    with pytest.raises(ValueError, match="both"):
        mk(w=(100.0, 0.1, 20.0, 2500.0))
    for r in ((0.0, 1.0), (-1.0, 1.0), (float("inf"), 1.0), (1.0,)):
        with pytest.raises(ValueError):
            mk(r=r)
    with pytest.raises(ValueError):
        mk(toks=(0, 0))
    # validate: a target that is not the rule's
    hp = mk()
    hp.pmm[0, 2] *= 1 + 1e-15
    with pytest.raises(ValueError):
        hp.validate()
    hp = mk()
    hp.pmm = np.zeros((1, 3))
    with pytest.raises(ValueError):
        hp.validate()


def test_pmm_pool_against_decimal():
    """instances.pmm_pool against a decimal restatement: reserves and targets over 10^decimals, pi = i / 1e18 times
    10^(base - quote decimals), k = K / 1e18, gamma = 1 - (lp + mt) / 1e18, the short target by the rule at 50 digits"""
    from decimal import Decimal, getcontext
    from cfmm_routing_code_b200 import instances as I
    getcontext().prec = 50
    res, tgt, dec = (1_234_567_890_123_456_789_012, 3_456_789_012_345), (2_000_000_000_000_000_000_000,
                                                                         3_000_000_000_000), (18, 6)
    i_raw, K_raw, lp, mt = 1_650_000_000, 250_000_000_000_000_000, 3_000_000_000_000_000, 1_000_000_000_000_000
    pi = Decimal(i_raw) / Decimal(10) ** 18 * Decimal(10) ** 12
    k = Decimal(K_raw) / Decimal(10) ** 18
    for rs in (0, 1, 2):                                 # ONE, ABOVE_ONE (base short), BELOW_ONE (quote short)
        res_, tgt_ = (res, tgt) if rs < 2 else ((res[0], 3_000_000_000_000), (10 ** 21, 4_000_000_000_000))
        Bd, Qd = Decimal(res_[0]) / Decimal(10) ** 18, Decimal(res_[1]) / Decimal(10) ** 6
        B0d, Q0d = Decimal(tgt_[0]) / Decimal(10) ** 18, Decimal(tgt_[1]) / Decimal(10) ** 6
        r, w, gam = I.pmm_pool(res_, tgt_, rs, i_raw, K_raw, lp, mt, dec)
        assert r == [float(Bd), float(Qd)]
        assert w[0] == float(pi) and w[1] == float(k) and gam == float(1 - Decimal(lp + mt) / Decimal(10) ** 18)
        if rs == 0:
            want = (Bd, Qd)
        elif rs == 1:
            d = Qd - Q0d
            want = (Bd + 2 * d / (pi * (1 + (1 + 4 * k * d / (pi * Bd)).sqrt())), Q0d)
        else:
            d = Bd - B0d
            want = (B0d, Qd + 2 * pi * d / (1 + (1 + 4 * k * pi * d / Qd).sqrt()))
        for got, x in zip(w[2:], want):
            assert abs(Decimal(got) - x) <= 8 * Decimal(U) * x, (rs, got, x)
        hp = HostPools.from_lists(2, [[0, 1]], [r], [gam], ["pmm"], [w])
        assert tuple(hp.pmm[0]) == w                     # from_lists leaves the converted targets as they are
    with pytest.raises(ValueError):                      # a DVM: quote target 0
        I.pmm_pool(res, (0, 0), 1, i_raw, K_raw, lp, mt, dec)
    with pytest.raises(ValueError):
        I.pmm_pool(res, tgt, 3, i_raw, K_raw, lp, mt, dec)


def test_update_checks():
    from cfmm_routing_code_b200.pools import check_pool_update
    hp = HostPools.from_lists(3, [[0, 1], [1, 2]], [[10.0, 2000.0], [2.0, 3.0]], [0.997, 0.997], ["pmm", "product"],
                              [(100.0, 0.1, 20.0, 1500.0), None])
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], reserves=[[12.0, 1900.0]], fees=[0.99],
                          pmm=[(100.0, 0.2, 20.0, 1500.0)])
    assert u.reserves.tolist() == [12.0, 1900.0] and u.pmm.tolist() == [[100.0, 0.2, 20.0, 1500.0]]
    for bad in ([[0.0, 1.0]], [[-1.0, 1.0]], [[np.inf, 1.0]]):
        with pytest.raises(ValueError):
            check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], reserves=bad)
    for bad in ([(100.0, 0.0, 20.0, 1500.0)], [(100.0, 2.0, 20.0, 1500.0)], [(0.0, 0.1, 20.0, 1500.0)],
                [(100.0, 0.1, 20.0)], [(100.0, 0.1, np.nan, 1500.0)]):
        with pytest.raises(ValueError):
            check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], pmm=bad)
    with pytest.raises(ValueError):                      # both sides short
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], reserves=[[10.0, 1000.0]],
                          pmm=[(100.0, 0.1, 20.0, 1500.0)])
    with pytest.raises(ValueError):                      # pmm= on another kind
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [1], pmm=[(1.0, 0.1, 2.0, 3.0)])
    with pytest.raises(ValueError):
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], prices=[1.0])


def _csr_args(hp):
    """the cfmm_csr_pools arrays and the records, as batch.CsrStore writes them (no concentrated, bins or E-CLP pools)"""
    w = hp.weights.copy()
    slot_kind = np.repeat(hp.kind, np.diff(hp.pool_ptr))
    logrw = np.log(np.maximum(hp.reserves, 1e-300) / np.where(slot_kind == 0, hp.weights, 1.0))
    pm = np.nonzero(hp.kind == KIND_PMM_HOST)[0]
    logrw[hp.pool_ptr[pm]] = np.arange(len(pm))
    rec = np.ascontiguousarray(hp.pmm[pm].reshape(-1) if len(pm) else np.zeros(4))
    return [np.ascontiguousarray(x, t) for x, t in ((hp.pool_ptr, np.int64), (hp.tok_idx, np.int32),
                                                    (hp.reserves, np.float64), (w, np.float64), (logrw, np.float64),
                                                    (hp.gamma, np.float64), (hp.kind, np.uint8))] + [rec]


def _host_solve(hp, specs, tol=1e-9):
    import types
    n, B, nnz = hp.n_tokens, len(specs), len(hp.tok_idx)
    c = np.stack([u.c for u in specs]).astype(float); a = np.stack([u.a for u in specs]).astype(float)
    fl = np.ascontiguousarray(np.stack([np.asarray(u.eq, np.uint8) | (np.asarray(u.pinned, np.uint8) << 1)
                                        for u in specs]), np.uint8)
    nu = np.ascontiguousarray(np.stack([np.where(u.c > 0, u.c, np.median(u.c[u.c > 0]) if (u.c > 0).any() else 1.0)
                                        for u in specs]))
    keep = _csr_args(hp)
    psi = np.zeros((B, n)); st = np.zeros((B, 8)); d = np.zeros((B, nnz)); l = np.zeros((B, nnz))
    fn = _host().pmm_host_solve
    fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 8 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
    fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), tol)
    ptr = hp.pool_ptr
    return [types.SimpleNamespace(value=st[p][0], dual_value=st[p][1], psi=psi[p], nu=nu[p], status=int(st[p][7]),
                                  deltas=[d[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                  lambdas=[l[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)]) for p in range(B)]


def _pmm_near(rng, p):
    """(reserves, weights) of a PMM pool whose guide price sits around the market price p (token 1 per token 0), at
    its meeting point or on either piece, k log-uniform over [PMM_K_MIN, 1]"""
    pi = p * np.exp(rng.normal(0, 0.02))
    k = float(np.exp(rng.uniform(np.log(PMM_K_MIN), 0.0)))
    B0 = 10.0 * rng.uniform(1, 2)
    Q0 = pi * B0 * rng.uniform(0.5, 2)
    side = int(rng.integers(0, 3))
    B, Q = B0, Q0
    if side == 1:
        B = B0 * rng.uniform(0.5, 0.99)
        Q = Q0 + pi * (B0 - B) * (1 + k * (B0 - B) / B)
    elif side == 2:
        Q = Q0 * rng.uniform(0.5, 0.99)
        B = B0 + (Q0 - Q) * (1 + k * (Q0 - Q) / Q) / pi
    return [float(B), float(Q)], (float(pi), k, float(B0), float(Q0))


def _reference_with_pmms(seed):
    """the reference's arbitrage.py instance with three PMM pools added between its tokens"""
    from cfmm_routing_code_b200 import instances as I
    d = I.arbitrage_instance()
    rng = np.random.default_rng(seed)
    mv = np.asarray(d["market_value"], float)
    n = len(mv)
    li, res, fees, kinds, wts = (list(d[k]) for k in ("local_indices", "reserves", "fees", "kinds", "weights"))
    for _ in range(3):
        i, j = (int(t) for t in rng.choice(n, 2, replace=False))
        r, w = _pmm_near(rng, mv[i] / mv[j])
        li.append([i, j]); res.append(r); fees.append(0.997); kinds.append("pmm"); wts.append(w)
    return HostPools.from_lists(n, li, res, fees, kinds, wts), mv


def test_host_solver_on_reference_instance_with_pmms_certified():
    """the per-thread solver's PMM instance (host build) on the reference's arbitrage.py instance with PMM pools added,
    for the three utilities; every answer certified by xp_pmm.certify"""
    from cfmm_routing_code_b200.api import Arbitrage, Liquidate, Swap
    for seed in range(4):
        hp, mv = _reference_with_pmms(seed)
        n = hp.n_tokens
        utils = [Arbitrage(mv), Liquidate(0, np.r_[0.0, np.full(n - 1, 2.0)]), Swap(1, 0, 1.0)]
        specs = [u.spec(n) for u in utils]
        for spec, r in zip(specs, _host_solve(hp, specs)):
            assert r.status == 0, (seed, r.status)
            XM.certify(hp, spec, r, 1e-9)


def _curve_np(P, b):
    """the curve's quote balance at base balance b > 0 (numpy; the quote piece by the stable root of its quadratic)"""
    pi, k, B0, Q0 = P
    d = B0 - b
    c = (b - B0) * pi
    s = Q0 + c
    e = 2 * c * Q0 / (s + np.sqrt(np.maximum(s * s - 4 * (1 - k) * c * Q0, 0.0)))
    return np.where(b <= B0, Q0 + pi * d * (1 + k * d / np.maximum(b, 1e-300)), Q0 - e)


def _primal(hp, c, x0):
    """max c'psi s.t. psi >= 0 over PMM pools only, every pool's post-trade state on or above its curve and > 0: scipy
    SLSQP on (D, L) >= 0, fp64"""
    from scipy.optimize import minimize
    m, n = hp.m, hp.n_tokens
    tok = hp.tok_idx.reshape(m, 2)
    R = hp.reserves.reshape(m, 2)
    g = hp.gamma

    def split(z):
        return z[:2 * m].reshape(m, 2), z[2 * m:].reshape(m, 2)

    def psi(z):
        D, L = split(z)
        return np.bincount(tok.ravel(), (L - D).ravel(), n)

    cons = [{"type": "ineq", "fun": psi}]
    for i in range(m):
        def above(z, i=i):
            D, L = split(z)
            b, q = R[i] + g[i] * D[i] - L[i]
            return (q - _curve_np(hp.pmm[i], max(b, 1e-12 * R[i, 0]))) / hp.pmm[i, 3]
        cons.append({"type": "ineq", "fun": above})
        cons.append({"type": "ineq", "fun": lambda z, i=i: R[i] + g[i] * split(z)[0][i] - split(z)[1][i]})
    scale = np.abs(c).max()
    res = minimize(lambda z: -(c @ psi(z)) / scale, x0, method="SLSQP", bounds=[(0, None)] * (4 * m),
                   constraints=cons, options={"ftol": 1e-15, "maxiter": 2000})
    return -res.fun * scale


def test_host_solver_against_scipy_primal():
    """PMM-only arbitrage markets: the per-thread solver's value against an independent scipy primal solve"""
    from cfmm_routing_code_b200.api import Arbitrage
    rng = np.random.default_rng(17)
    for trial in range(6):
        n = 3
        price = np.exp(rng.normal(0, 0.2, n))
        li, res, fees, wts = [], [], [], []
        for _ in range(4):
            i, j = (int(t) for t in rng.choice(n, 2, replace=False))
            r, w = _pmm_near(rng, price[i] / price[j] * np.exp(rng.normal(0, 0.05)))
            w = (w[0], float(10.0 ** rng.uniform(-2, 0)), w[2], w[3])          # k away from 0: a well-scaled primal
            li.append([i, j]); res.append(r); fees.append(0.997); wts.append(w)
        hp = HostPools.from_lists(n, li, res, fees, ["pmm"] * 4, wts)
        spec = Arbitrage(price).spec(n)
        r = _host_solve(hp, [spec], tol=1e-10)[0]
        assert r.status == 0
        XM.certify(hp, spec, r, 1e-10)
        x0 = np.concatenate([np.concatenate(r.deltas), np.concatenate(r.lambdas)]) * 0.5
        v = _primal(hp, np.asarray(spec.c, float), x0)
        assert abs(v - r.value) <= 1e-7 * max(abs(r.value), np.abs(price).max() * 1e-3), (trial, v, r.value)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _pmm_hostpools(seed, m, n_tokens):
    """m random PMM pools on random token pairs (as case_set) and token prices nu: each pool's token 1 counted in the
    units that put nu0 / nu1 where case_set's prices put it, so that the mix of trades (far, near, none, across pi) is
    case_set's; returns (hp, a, b, P, R, g, nu)"""
    R, P, g, n0, n1 = case_set(seed, m)
    rng = np.random.default_rng(seed + 100)
    a = rng.integers(0, n_tokens, m)
    b = (a + 1 + rng.integers(0, n_tokens - 1, m)) % n_tokens
    nu = np.exp(rng.normal(0, 1, n_tokens))
    c = nu[a] / nu[b] / (n0 / n1)
    R = R.copy(); P = P.copy()
    R[:, 1] *= c; P[:, 0] *= c; P[:, 3] *= c
    P = pmm_targets(R, P)
    hp = HostPools(n_tokens, np.arange(0, 2 * m + 1, 2, dtype=np.int64), np.stack([a, b], 1).reshape(-1).astype(np.int32),
                   R.reshape(-1).copy(), np.zeros(2 * m), g, np.full(m, KIND_PMM_HOST, np.uint8), pmm=P)
    return hp, a, b, P, R, g, nu


@pytest.fixture
def scatter_auto():
    lib = _lib.load()
    yield lib
    lib.cfmm_set_scatter_mode(0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_eval_kernel_against_host_build(scatter_auto, mode):
    """10^6 pools, all four (trades, hess) cells, global (1) and shared (2) scatter; every pool against the host build
    of pmm_pair (itself checked against the 60-digit reference above); psi and arb against sums of the flows; the
    Hessian kernels against the pool decomposition of hcoef"""
    import torch
    lib = scatter_auto
    n, m = (2000 if mode == 2 else 40000), 1_000_000
    hp, a, b, P, R, g, nu = _pmm_hostpools(11, m, n)
    hp.validate()
    store = cf.PoolStore(hp, device="cuda:0")
    assert [bk.kind for bk in store.buckets] == [_lib.KIND_PMM]
    rng = np.random.default_rng(12)
    nu_t = torch.as_tensor(nu, dtype=torch.float64, device="cuda:0")
    lib.cfmm_set_scatter_mode(mode)
    D, L, hc = host_pairs(R, P, g, nu[a], nu[b])
    assert (D[:, 0] > 0).sum() > m // 10 and (D[:, 1] > 0).sum() > m // 10
    bk = store.buckets[0]
    for trades in (False, True):
        for hess in (False, True):
            acc = store.evaluate(nu_t, trades=trades, hess=hess).cpu().numpy()
            y0, y1 = L[:, 0] - D[:, 0], L[:, 1] - D[:, 1]
            psi = np.bincount(a, y0, n) + np.bincount(b, y1, n)
            gross = np.bincount(a, np.abs(y0), n) + np.bincount(b, np.abs(y1), n)
            assert np.all(np.abs(acc[:n] - psi) <= 1e-12 * gross + 64 * U * (
                np.bincount(a, R[:, 0], n) + np.bincount(b, R[:, 1], n)))
            arb = nu[a] * y0 + nu[b] * y1
            assert abs(acc[n] - arb.sum()) <= 1e-12 * np.abs(arb).sum()
            # the device contracts products and sums into fma where the host build does not: a few ulp apart
            if trades:
                Dk = bk.delta[:, :m].cpu().numpy().T
                Lk = bk.lam[:, :m].cpu().numpy().T
                for kern, host in ((Dk, D), (Lk, L)):
                    assert np.all(np.abs(kern - host) <= 64 * U * (np.abs(host) + R))
                assert np.array_equal(Dk == 0, D == 0) and np.array_equal(Lk == 0, L == 0)
            if hess:
                hk = bk.hcoef[:m].cpu().numpy()
                assert np.all(np.abs(hk - hc) <= 64 * U * np.abs(hc)) and np.array_equal(hk == 0, hc == 0)
    # Hessian kernels against hcoef: Hs = sum_i hc_i (e_a - e_b)(e_a - e_b)'
    store.evaluate(nu_t, hess=True)
    v = rng.normal(size=n)
    y = store.hvp(torch.as_tensor(v / nu, device="cuda:0")).cpu().numpy()
    w = hc * (v[a] / nu[a] - v[b] / nu[b])
    want = np.bincount(a, w, n) - np.bincount(b, w, n)
    assert np.allclose(y, want, rtol=1e-10, atol=1e-12 * np.abs(hc).sum() / n)
    dg = store.hess_diag().cpu().numpy()
    assert np.allclose(dg, np.bincount(a, hc, n) + np.bincount(b, hc, n), rtol=1e-12, atol=0)


@pytest.mark.gpu
def test_launch_strategy_cells_and_anchor():
    """the launch-strategy harness of tests/test_launch_strategies.py on a 100k-pool PMM bucket: every (trades, hess)
    cell under global and shared scatter (per-pool outputs equal across strategies, psi / arb against exact sums,
    hvp / diag / dense against hcoef), then a 500-pool sample of the flows against xp_pmm"""
    import test_launch_strategies as TL
    lib = _lib.load()

    def set_mode(mode):
        _lib.check(lib.cfmm_set_scatter_mode(mode), "cfmm_set_scatter_mode")
    hp, a, b, P, R, g, nu = _pmm_hostpools(13, 100_000, 64)
    try:
        inst = TL.Inst(hp, nu)
        assert inst.kind == _lib.KIND_PMM
        for mode in (TL.GLOBAL, TL.SHARED):
            for trades, hess in TL.FLAGS:
                TL.check_cell(inst, mode, trades, hess, set_mode, anchor=False)
        set_mode(TL.GLOBAL)
        acc, out = inst.eval(True, True)
    finally:
        set_mode(TL.AUTO)
    smp = np.sort(np.random.default_rng(3).choice(inst.m, 500, replace=False))
    sel = inst.sel[smp]
    D, L, h = out["D"][:, smp].T, out["L"][:, smp].T, out["h"][smp]
    check_against_reference(P[sel], R[sel], g[sel], nu[a[sel]], nu[b[sel]], D, L, h)


@pytest.mark.gpu
def test_k_one_matches_the_product_kernel():
    """k = 1 with Q0 = pi B0 is the constant-product pool: k_eval_pair<PMM> on such pools against the same pools as kind
    'product' through the product kernel (plain layout), flows and psi"""
    import torch
    rng = np.random.default_rng(8)
    m, n = 20000, 64
    a = rng.integers(0, n, m)
    b = (a + rng.integers(1, n, m)) % n
    B, Q = 10.0 ** rng.uniform(-2, 4, m), 10.0 ** rng.uniform(-2, 4, m)
    pi = Q / B * 10.0 ** rng.uniform(-1, 1, m)
    B0 = np.sqrt(B * Q / pi)
    R = np.stack([B, Q], axis=1)
    P = pmm_targets(R, np.stack([pi, np.ones(m), B0, pi * B0], axis=1))
    g = np.where(rng.random(m) < 0.3, 1.0, 0.997)
    toks = np.stack([a, b], 1).astype(np.int32)
    hp = HostPools(n, np.arange(0, 2 * m + 1, 2, dtype=np.int64), toks.reshape(-1), R.reshape(-1).copy(),
                   np.zeros(2 * m), g, np.full(m, KIND_PMM_HOST, np.uint8), pmm=P)
    hq = HostPools.from_pairs(n, toks, R, g)
    nu = torch.as_tensor(np.exp(rng.normal(0, 1, n)), device="cuda:0")
    out = []
    for h in (hp, hq):
        st = cf.PoolStore(h, device="cuda:0", layout="plain")
        acc = st.evaluate(nu, trades=True).cpu().numpy()
        out.append((acc,) + st.gather_trades())
    (ap, dp, lp), (aq, dq, lq) = out
    # B0 and Q0 reproduce the hyperbola through (B, Q) to rounding: 1e-10 of each slot's reserve and flow
    sc = R.reshape(-1)
    assert np.all(np.abs(dp - dq) <= 1e-10 * (sc + dq)) and np.all(np.abs(lp - lq) <= 1e-10 * (sc + lq))
    gross = np.bincount(toks.reshape(-1), sc + dq + lq, n)
    assert np.all(np.abs(ap[:n] - aq[:n]) <= 1e-10 * gross)


@pytest.mark.gpu
def test_dense_hessian_small(scatter_auto):
    import torch
    hp, a, b, P, R, g, nu = _pmm_hostpools(21, 5000, 40)
    store = cf.PoolStore(hp, device="cuda:0")
    store.evaluate(torch.as_tensor(nu, device="cuda:0"), hess=True)
    H = store.hess_dense().cpu().numpy()
    _, _, hc = host_pairs(R, P, g, nu[a], nu[b])
    want = np.zeros((40, 40))
    np.add.at(want, (a, a), hc); np.add.at(want, (b, b), hc); np.add.at(want, (a, b), -hc); np.add.at(want, (b, a), -hc)
    assert np.allclose(H[:40, :40] if H.ndim == 2 else H.reshape(40, 40), want, rtol=1e-12, atol=1e-12 * np.abs(hc).max())


def _mixed_market(seed, n=6):
    """PMM pools beside E-CLP, product, weighted, sum, bounded, StableSwap, concentrated, cryptoswap and bins pools (the
    E-CLP tests' market); returns (n, local_indices, reserves, fees, kinds, weights, market prices)"""
    import test_eclp as TE
    n, li, res, fees, kinds, wts, price = TE._mixed_market(seed, n)
    rng = np.random.default_rng(seed + 1000)
    for _ in range(4):
        i, j = (int(t) for t in rng.choice(n, 2, replace=False))
        r, w = _pmm_near(rng, price[i] / price[j])
        li.append([i, j]); res.append(r); fees.append(0.997); kinds.append("pmm"); wts.append(w)
    return n, li, res, fees, kinds, wts, price


def _pmm_market(seed, n=6, m=12):
    """m PMM pools around the market prices of n tokens, every token on a pool"""
    rng = np.random.default_rng(seed)
    price = np.exp(rng.normal(0, 0.3, n))
    li, res, fees, kinds, wts = [], [], [], [], []
    for q in range(m):
        i, j = (q % n, (q + 1 + int(rng.integers(0, n - 1))) % n)
        r, w = _pmm_near(rng, price[i] / price[j])
        li.append([i, j]); res.append(r); fees.append(0.997); kinds.append("pmm"); wts.append(w)
    return n, li, res, fees, kinds, wts, price


@pytest.mark.gpu
@pytest.mark.parametrize("native", [False, "hostloop", True])
@pytest.mark.parametrize("seed", range(4))
def test_mixed_markets_certified(seed, native):
    """solver.py, the host loop and native=True (which falls back to solver.py: the store is not one blocked bucket) on
    markets of PMM pools beside every other kind, for the three utilities; every answer optimal and certified by
    xp_pmm.certify"""
    n, li, res, fees, kinds, wts, price = _mixed_market(seed)
    hp = HostPools.from_lists(n, li, res, fees, kinds, wts)
    for util in (cf.Arbitrage(price), cf.Liquidate(0, np.r_[0.0, 1.0, 0.5, 0.0, 0.0, 0.0]), cf.Swap(1, 2, 0.5)):
        r = cf.solve_pools(hp, util, device="cuda:0", tol=1e-9, native=native, method="pools")
        assert r.status == "optimal", (seed, native, util, r.status)
        XM.certify(hp, util.spec(n), r, 1e-9)


@pytest.mark.gpu
def test_synth_market_certified():
    """instances.synth_pmm_market (k over [PMM_K_MIN, 1], pools on both pieces and at the meeting point) solved on
    solver.py and the host loop, certified"""
    from cfmm_routing_code_b200 import instances as I
    hp, p = I.synth_pmm_market(400, 12, seed=3)
    hp.validate()
    assert (hp.kind == KIND_PMM_HOST).sum() == 120 and (hp.kind == KIND_ECLP_HOST).any()
    for native in (False, "hostloop"):
        r = cf.solve_pools(hp, cf.Arbitrage(p), device="cuda:0", tol=1e-9, native=native, method="pools")
        assert r.status == "optimal", native
        XM.certify(hp, cf.Arbitrage(p).spec(hp.n_tokens), r, 1e-9)


@pytest.mark.gpu
def test_per_thread_paths_certified():
    """the per-thread solver (cfmm_batch_solve_pmm): solve_batch on the reference instance with PMM pools for the three
    utilities, solve_many over mixed markets, solve_sweep over a Swap ladder; every answer optimal and certified"""
    from cfmm_routing_code_b200.api import Arbitrage, Liquidate, Swap
    hp, mv = _reference_with_pmms(0)
    n = hp.n_tokens
    utils = [Arbitrage(mv), Liquidate(0, np.r_[0.0, np.full(n - 1, 2.0)]), Swap(1, 0, 1.0)]
    rs = cf.solve_batch(hp, utils, tol=1e-9, device="cuda:0")
    for u, r in zip(utils, rs):
        assert r.status == "optimal"
        XM.certify(hp, u.spec(n), r, 1e-9)
    # against the host build of the same instance: the same iteration, to rounding
    hr = _host_solve(hp, [u.spec(n) for u in utils])
    for r, h in zip(rs, hr):
        assert abs(r.value - h.value) <= 1e-9 * max(1.0, abs(h.value))
    probs = []
    for seed in range(30):
        m = _mixed_market(100 + seed)
        probs.append((HostPools.from_lists(m[0], *m[1:6]), cf.Arbitrage(m[6])))
    rs = cf.solve_many(probs, tol=1e-9, device="cuda:0")
    for (h, u), r in zip(probs, rs):
        assert r.status == "optimal"
        XM.certify(h, u.spec(h.n_tokens), r, 1e-9)
    n6, li, res, fees, kinds, wts, price = _mixed_market(7)
    utils = [cf.Swap(1, 2, t) for t in np.linspace(0.1, 3.0, 12)]
    rs = cf.solve_sweep(li, res, fees, kinds, wts, utils, n_tokens=n6, tol=1e-9, device="cuda:0")
    hp6 = HostPools.from_lists(n6, li, res, fees, kinds, wts)
    for u, r in zip(utils, rs):
        assert r.status == "optimal"
        XM.certify(hp6, u.spec(n6), r, 1e-9)
    r = cf.solve(li, res, fees, kinds, wts, utility=cf.Arbitrage(price), device="cuda:0", method="thread", tol=1e-9)
    assert r.status == "optimal"
    XM.certify(hp6, cf.Arbitrage(price).spec(n6), r, 1e-9)


@pytest.mark.gpu
def test_older_per_thread_entries_give_pmm_problems_status_3():
    import torch
    from cfmm_routing_code_b200 import batch as BT
    hp, mv = _reference_with_pmms(1)
    store = BT.CsrStore(hp, device="cuda:0")
    assert store.has_pmm
    n = hp.n_tokens
    spec = cf.Arbitrage(mv).spec(n)
    lib = store.lib
    for name in ("cfmm_batch_solve", "cfmm_batch_solve_stableswap", "cfmm_batch_solve_stableswap_n",
                 "cfmm_batch_solve_concentrated", "cfmm_batch_solve_cryptoswap", "cfmm_batch_solve_tricrypto",
                 "cfmm_batch_solve_bins", "cfmm_batch_solve_eclp"):
        f64 = dict(dtype=torch.float64, device="cuda:0")
        c = torch.as_tensor(np.asarray(spec.c, float)[None], **f64); a = torch.as_tensor(np.asarray(spec.a, float)[None], **f64)
        fl = torch.as_tensor((np.asarray(spec.eq, np.uint8) | (np.asarray(spec.pinned, np.uint8) << 1))[None],
                             device="cuda:0")
        nu = c.clone(); psi = torch.empty(1, n, **f64); stats = torch.empty(1, 8, **f64)
        batch = _lib.Batch(1, None, c.data_ptr(), a.data_ptr(), fl.data_ptr(), nu.data_ptr(), psi.data_ptr(),
                           stats.data_ptr(), None, None, store.nnz)
        prm = _lib.BatchParams(1e-9, 0.1, 1e-4, 0.5, 1e-12, 60, 100)
        _lib.check(lib.cfmm_set_batch_lanes(1))
        work = store.work(1)
        args = [C.byref(store.c_pools)]
        if name not in ("cfmm_batch_solve", "cfmm_batch_solve_stableswap", "cfmm_batch_solve_stableswap_n"):
            args.append(store.records.data_ptr())
        rc = getattr(lib, name)(*args, C.byref(batch), C.byref(prm), work.data_ptr(), None)
        assert rc == 0, name
        torch.cuda.synchronize()
        assert int(stats[0, 7].item()) == 3, name
    assert lib.cfmm_batch_solve_pmm(C.byref(store.c_pools), None, None, None, None, None) == -1


@pytest.mark.gpu
def test_rank_stores_sum_to_the_single_store():
    import torch
    hp, a, b, P, R, g, nu = _pmm_hostpools(31, 30001, 300)
    nu = torch.as_tensor(nu, device="cuda:0")
    one = cf.PoolStore(hp, device="cuda:0").evaluate(nu).cpu().numpy()
    for world in (2, 3):
        tot = sum(cf.PoolStore(hp, device="cuda:0", rank=k, world=world).evaluate(nu).cpu().numpy() for k in range(world))
        assert np.allclose(tot, one, rtol=1e-12, atol=1e-12 * np.abs(one).max())


def _same_buckets(store, fresh):
    import torch
    for b1, b2 in zip(store.buckets, fresh.buckets):
        if getattr(b1, "blocked", False):                 # the constant-product pools: not updated here
            continue
        for name in ("reserves", "gamma", "weights", "logrw", "tok_idx"):
            t1, t2 = getattr(b1, name), getattr(b2, name)
            assert (t1 is None) == (t2 is None) and (t1 is None or torch.equal(t1, t2)), (b1.kind, name)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3])
def test_updates_equal_a_fresh_store(world):
    """update_pools blocks of reserves= (swaps, one across pi), fees= and pmm= (new rows, with and without reserves=) on
    every rank of a 1-, 2- or 3-rank store (the mixed market on one rank, a market of PMM pools on several): each equal
    bit for bit to a fresh store of the updated literals; the caller's HostPools untouched; the warm re-solve of the
    single store certified on solver.py and the host loop"""
    n, li, res, fees, kinds, wts, price = _mixed_market(3) if world == 1 else _pmm_market(3)
    hp = HostPools.from_lists(n, li, res, fees, kinds, wts)
    keep = hp.pmm.copy(), hp.reserves.copy(), hp.gamma.copy()
    stores = [cf.PoolStore(hp, device="cuda:0", rank=k, world=world) for k in range(world)]
    ids = np.nonzero(np.asarray(hp.kind) == KIND_PMM_HOST)[0]
    rng = np.random.default_rng(5)
    res2, fees2, wts2 = list(res), list(fees), list(wts)
    # block 1: swaps along each curve (the first crosses pi), new fees
    newR = []
    for q, i in enumerate(ids[:3]):
        pi, k, B0, Q0 = hp.pmm[i]
        pool = XM.Pool(pi, k, B0, Q0)
        ps = pi * (0.5 if q == 0 else rng.uniform(0.98, 1.02))
        with mp.workdps(XM.DPS):
            b, qq = pool.end(mp.mpf(ps))
        newR.append([float(b), float(qq) * (1 + 1e-9)])                # a hair above the curve (fees kept in the pool)
    newg = [0.999, 0.995, 1.0]
    for s in stores:
        s.update_pools(ids[:3], reserves=newR, fees=newg)
    for q, i in enumerate(ids[:3]):
        res2[i], fees2[i], wts2[i] = newR[q], newg[q], tuple(hp.pmm[i])
    hp2 = HostPools.from_lists(n, li, res2, fees2, kinds, wts2)
    for k, s in enumerate(stores):
        _same_buckets(s, cf.PoolStore(hp2, device="cuda:0", rank=k, world=world))
    # block 2: new rows (a DPP reset: new pi, k and targets) with new reserves for one pool, rows alone for another
    rows = [(hp2.pmm[ids[0], 0] * 1.01, 0.3, hp2.reserves[hp2.pool_ptr[ids[0]]] * 1.2, 1.0),
            (hp2.pmm[ids[1], 0], 0.05, 1e-3, 1e-3)]
    rows[0] = (rows[0][0], rows[0][1], rows[0][2], hp2.reserves[hp2.pool_ptr[ids[0]] + 1] * 0.8)
    R0 = [res2[ids[0]][0] * 1.1, res2[ids[0]][1]]
    for s in stores:
        s.update_pools(ids[:1], reserves=[R0], pmm=rows[:1])
        s.update_pools(ids[1:2], pmm=rows[1:2])
    res2[ids[0]], wts2[ids[0]], wts2[ids[1]] = R0, rows[0], rows[1]
    hp3 = HostPools.from_lists(n, li, res2, fees2, kinds, wts2)
    for k, s in enumerate(stores):
        _same_buckets(s, cf.PoolStore(hp3, device="cuda:0", rank=k, world=world))
    assert np.array_equal(hp.pmm, keep[0]) and np.array_equal(hp.reserves, keep[1]) and np.array_equal(hp.gamma, keep[2])
    if world == 1:
        for native in (False, "hostloop"):
            r = cf.solve_pools(hp3, cf.Arbitrage(price), store=stores[0], device="cuda:0", tol=1e-9, native=native,
                               method="pools")
            assert r.status == "optimal", native
            XM.certify(hp3, cf.Arbitrage(price).spec(n), r, 1e-9)


@pytest.mark.gpu
def test_invalid_entry_changes_nothing():
    """an invalid entry in a 1000-pool block (a bad k, or reserves both below their targets) raises and writes
    nothing"""
    import torch
    hp, a, b, P, R, g, _ = _pmm_hostpools(41, 1000, 50)
    st = cf.PoolStore(hp, device="cuda:0")
    bk = st.buckets[0]
    before = bk.weights.clone(), bk.reserves.clone(), bk.gamma.clone()
    rows = P.copy()
    rows[:, 1] = 0.5
    rows[777, 1] = 0.0
    with pytest.raises(ValueError):
        st.update_pools(np.arange(1000), pmm=rows, fees=np.full(1000, 0.99))
    bad = R * 1.1
    sh = int(np.nonzero((R[:, 0] < P[:, 2]))[0][0])                # a base-short pool: push its quote below Q0 too
    bad[sh, 1] = P[sh, 3] * 0.5
    with pytest.raises(ValueError):
        st.update_pools(np.arange(1000), reserves=bad, fees=np.full(1000, 0.99))
    assert torch.equal(before[0], bk.weights) and torch.equal(before[1], bk.reserves) and torch.equal(before[2], bk.gamma)


@pytest.mark.gpu
def test_abi_codes():
    import ctypes
    import torch
    lib = _lib.load()
    hp, *_ = _pmm_hostpools(51, 100, 10)
    store = cf.PoolStore(hp, device="cuda:0")
    bk = store.buckets[0]
    nu = torch.ones(10, dtype=torch.float64, device="cuda:0")
    acc = torch.zeros(11, dtype=torch.float64, device="cuda:0")
    c = _lib.Bucket.from_buffer_copy(bk.c_bucket)
    assert c.kind == 12 == _lib.KIND_PMM
    assert lib.cfmm_arb_eval(ctypes.byref(c), 10, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc[10:].data_ptr(),
                             None, None) == 0
    c.arity = 3
    assert lib.cfmm_arb_eval(ctypes.byref(c), 10, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc[10:].data_ptr(),
                             None, None) == -2
    c.arity = 2
    c.weights = None
    assert lib.cfmm_arb_eval(ctypes.byref(c), 10, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc[10:].data_ptr(),
                             None, None) == -1
