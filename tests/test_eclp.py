"""Elliptic concentrated-liquidity pools (Gyroscope E-CLP) as one pool kind (host kind 11, CFMM_KIND_ECLP).

CPU: cfmm_small::eclp_pair compiled for the host against the mpmath reference (tests/xp_eclp.py: the pool in its circle
frame, flows as differences of boundary points at 60 digits) on random pools over lam in [1, 1e8], phi across
(0, pi/2), ranges 1e-4 to 1e4 wide, prices deep inside, far outside and within 1e-12 of the pool's, both caps and the
no-trade band; hc against the reference's central differences; post-trade feasibility; the mirror pool; homogeneity;
eclp_state against mpmath; the validation rules and the (c, s) normalisation.
GPU (H100): k_eval_pair<ECLP> in all four (trades, hess) instances under both scatter strategies against the host build;
the Hessian kernels against hcoef; certified solves on solver.py and the host loop, mixed with every other kind; the
store sharded over loopback ranks; reserve and fee updates; the C ABI codes.

Error bound.  Both sides read the same f64 prices, state and balances.  The kernel computes each flow from one
cancellation-free quotient, so its error is a few ulp of the flow, plus the error of the price p* = nu0 / (gamma nu1)
(a few ulp, amplified by the flow's sensitivity p* |d flow / d p*|), plus a few ulp of the reserve where the flow is the
reserve itself (a cap).  The tests allow 64 u (R_j + |flow_j| + p* |d flow_j / d p*|), u = 2^-53, per flow.
"""
import ctypes as C
import math
import os
import subprocess

import mpmath as mp
import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib
from cfmm_routing_code_b200.pools import HostPools, KIND_ECLP_HOST, _check_eclp, _eclp_xy, eclp_state
import xp_eclp as XE

HERE = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -53
p_ = lambda x: x.ctypes.data_as(C.c_void_p)
_HOST = None


def _host():
    """tests/host_harness/eclp_host.cpp: cfmm_small::eclp_pair, host build"""
    global _HOST
    if _HOST is None:
        src = os.path.join(HERE, "host_harness", "eclp_host.cpp")
        hdr = os.path.join(HERE, "..", "cfmm_routing_code_b200", "csrc", "cfmm_small.cuh")
        lib = os.path.join(HERE, "_build", "libeclp_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src],
                           check=True)
        _HOST = C.CDLL(lib)
    return _HOST


def host_pairs(R, P7, g, n0, n1):
    """eclp_pair of every pool: R [m, 2], P7 [m, 7] = (alpha, beta, c, s, lam, r, p); returns D, L [m, 2], hc [m]"""
    m = len(g)
    D, L, hc = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m)
    f = _host().eclp_host_pools
    f.argtypes = [C.c_longlong] + [C.c_void_p] * 8
    c = lambda a: np.ascontiguousarray(a, np.float64)
    f(m, p_(c(R)), p_(c(P7)), p_(c(g)), p_(c(n0)), p_(c(n1)), p_(D), p_(L), p_(hc))
    return D, L, hc


def random_params(rng, m):
    """(alpha, beta, c, s, lam) [m, 5]: lam log-uniform in [1, 1e8], phi across (0, pi/2), ranges 1e-4 to 1e4 wide
    (beta / alpha - 1), placed around the peg s / c, or off it by up to e^3"""
    lam = 10.0 ** rng.uniform(0, 8, m)
    lam[rng.random(m) < 0.05] = 1.0
    lam[rng.random(m) < 0.05] = 1e8
    phi = rng.uniform(0.005, np.pi / 2 - 0.005, m)
    c, s = np.cos(phi), np.sin(phi)
    w = 10.0 ** rng.uniform(-4, 4, m)
    peg = s / c
    centre = peg * np.exp(np.where(rng.random(m) < 0.5, 0.0, rng.uniform(-3, 3, m)))
    alpha = centre / np.sqrt(1 + w) * np.exp(rng.uniform(-0.5, 0.5, m) * np.log1p(w))
    beta = alpha * (1 + w)
    return np.stack([alpha, beta, c, s, lam], axis=1)


def random_state(rng, P, r_lo=-3, r_hi=6):
    """balances [m, 2] at a price in the range (log-uniform), at either end (one side empty), with r log-uniform"""
    m = len(P)
    a, b = P[:, 0], P[:, 1]
    p = np.exp(rng.uniform(np.log(a), np.log(b)))
    u = rng.random(m)
    p = np.where(u < 0.05, a, np.where(u < 0.1, b, p))
    r = 10.0 ** rng.uniform(r_lo, r_hi, m)
    X, Y = _eclp_xy(a, b, P[:, 2], P[:, 3], P[:, 4] ** 2, p)
    R = np.stack([r * X, r * Y], axis=1)
    R[u < 0.05, 1] = 0.0
    R[(u >= 0.05) & (u < 0.1), 0] = 0.0
    return R


def random_prices(rng, P, st, g):
    """(n0, n1) with p* deep inside the range, far outside it, within 1e-12 .. 1e-3 of the pool's price, or in the
    no-trade band"""
    m = len(P)
    a, b, p = P[:, 0], P[:, 1], st[:, 1]
    mode = rng.integers(0, 5, m)
    inside = np.exp(rng.uniform(np.log(a), np.log(b)))
    outside = np.where(rng.random(m) < 0.5, a / 10.0 ** rng.uniform(0, 3, m), b * 10.0 ** rng.uniform(0, 3, m))
    near = p * (1 + np.where(rng.random(m) < 0.5, -1, 1) * 10.0 ** rng.uniform(-12, -3, m))
    band = p * g ** rng.uniform(-0.99, 0.99, m)
    ps = np.choose(mode, [inside, outside, near, band, inside])
    n1 = 10.0 ** rng.uniform(-2, 2, m)
    return ps * n1, n1                                   # the mid price nu0 / nu1; the kernel applies the fee


def case_set(seed, m):
    rng = np.random.default_rng(seed)
    P = random_params(rng, m)
    R = random_state(rng, P)
    st = eclp_state(R, P)
    g = np.where(rng.random(m) < 0.3, 1.0, 1.0 - 10.0 ** rng.uniform(-4, -1.5, m))
    n0, n1 = random_prices(rng, P, st, g)
    return P, R, st, g, n0, n1


def reference(P, R, st, g, n0, n1, D, L):
    """xp_eclp.reference_rows over all pools, on every core"""
    from concurrent.futures import ProcessPoolExecutor
    import multiprocessing as mpr
    n = max(1, min(os.cpu_count() or 1, 32))
    parts = np.array_split(np.arange(len(g)), 4 * n)
    chunks = [(P[k], R[k], st[k], g[k], n0[k], n1[k], D[k], L[k]) for k in parts if len(k)]
    if n == 1 or len(g) < 2000:
        return np.concatenate([XE.reference_rows(c) for c in chunks])
    with ProcessPoolExecutor(n, mp_context=mpr.get_context("spawn")) as ex:    # workers import xp_eclp only
        return np.concatenate(list(ex.map(XE.reference_rows, chunks)))


def check_against_reference(P, R, st, g, n0, n1, D, L, hc):
    """every flow within 64 u (R_j + |flow_j| + p* |d flow_j / d p*|) of the reference, hc within 1e-7, post-trade
    state feasible to the same tolerance; returns the worst normalised flow error"""
    ref = reference(P, R, st, g, n0, n1, D, L)
    dy = np.abs(ref[:, 4:6])
    worst = 0.0
    for j in range(2):
        for kern, want in ((D[:, j], ref[:, j]), (L[:, j], ref[:, 2 + j])):
            tol = 64 * U * (R[:, j] + np.abs(want) + dy[:, j])
            err = np.abs(kern - want)
            bad = np.nonzero(err > tol)[0]
            assert len(bad) == 0, [(i, P[i], R[i], st[i], g[i], n0[i], n1[i], kern[i], want[i]) for i in bad[:3]]
            worst = max(worst, float(np.max(np.where(tol > 0, err / np.where(tol > 0, tol, 1), 0.0), initial=0.0)))
    # post-trade balances of the kernel's trade: >= 0 and inside the ellipse, to the same tolerance
    scale = 64 * U * (R.sum(1) + np.abs(D).sum(1) + np.abs(L).sum(1) + dy.sum(1))
    assert np.all(ref[:, 8] >= -scale) and np.all(ref[:, 9] >= -scale)
    assert np.all(ref[:, 7] <= scale * np.maximum(1.0, P[:, 4]))
    # hc jumps where p* crosses a kink of the pool's dual (its price p, alpha, beta): within a few ulp of one the
    # kernel's rounded p* and the reference's exact one may lie on different sides, so hc is not compared there
    ps0, ps1 = n0 / (g * n1), g * n0 / n1
    kink = np.zeros(len(g), bool)
    for ps in (ps0, ps1):
        for k in (st[:, 1], P[:, 0], P[:, 1]):
            kink |= np.abs(ps - k) <= 8 * U * k
    hr = ref[:, 6]
    bad = np.nonzero(~kink & (np.abs(hc - hr) > 1e-7 * np.abs(hr)))[0]
    assert len(bad) == 0, [(i, hc[i], hr[i]) for i in bad[:3]]
    return worst


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
N_PAIR = int(os.environ.get("ECLP_TEST_POOLS", "100000"))


def test_eclp_pair_against_reference():
    """10^5 random pools (ECLP_TEST_POOLS to change it), every flow and hc against the 60-digit reference"""
    P, R, st, g, n0, n1 = case_set(1, N_PAIR)
    P7 = np.concatenate([P, st], axis=1)
    D, L, hc = host_pairs(R, P7, g, n0, n1)
    check_against_reference(P, R, st, g, n0, n1, D, L, hc)
    # the cases are there: both tenders, both caps, no trade
    ps0, ps1 = n0 / (g * n1), g * n0 / n1
    t0, t1 = ps0 < st[:, 1], ps1 > st[:, 1]
    for case in (t0 & (ps0 <= P[:, 0]), t1 & (ps1 >= P[:, 1]), t0 & (ps0 > P[:, 0]), t1 & (ps1 < P[:, 1]), ~t0 & ~t1):
        assert case.sum() > N_PAIR // 100


def test_no_trade_band_is_exact():
    P, R, st, g, _, _ = case_set(2, 2000)
    P, R, st, g = P[g < 1], R[g < 1], st[g < 1], g[g < 1]              # at gamma = 1 the band is the one price p
    rng = np.random.default_rng(3)
    n1 = 10.0 ** rng.uniform(-2, 2, len(g))
    n0 = st[:, 1] * g ** rng.uniform(-0.999, 0.999, len(g)) * n1
    D, L, hc = host_pairs(R, np.concatenate([P, st], axis=1), g, n0, n1)
    assert np.all(D == 0) and np.all(L == 0) and np.all(hc == 0)


def test_caps_pay_out_the_whole_reserve():
    P, R, st, g, _, _ = case_set(4, 2000)
    n1 = np.ones(len(g))
    D, L, hc = host_pairs(R, np.concatenate([P, st], axis=1), g, P[:, 0] * g * 1e-3, n1)     # p* far below alpha
    assert np.array_equal(L[:, 1], R[:, 1]) and np.all(L[:, 0] == 0) and np.all(hc == 0)
    D, L, hc = host_pairs(R, np.concatenate([P, st], axis=1), g, P[:, 1] / g * 1e3, n1)      # p* far above beta
    assert np.array_equal(L[:, 0], R[:, 0]) and np.all(L[:, 1] == 0) and np.all(hc == 0)


def test_mirror_pool_trades_the_mirror_image():
    P, R, st, g, n0, n1 = case_set(5, 3000)
    a, b, c, s, lam = P.T
    Pm = np.stack([1 / b, 1 / a, s, c, lam], axis=1)
    Rm = R[:, ::-1].copy()
    stm = eclp_state(Rm, Pm)
    # the mirror's range is rounded (1/beta, 1/alpha): on a narrow range that moves r and the flows by a few ulp times
    # (beta + alpha) / (beta - alpha)
    rt = 1e-12 + 64 * U * (a + b) / (b - a)
    assert np.all(np.abs(stm[:, 1] * st[:, 1] - 1.0) <= rt)
    assert np.all(np.abs(stm[:, 0] / st[:, 0] - 1.0) <= rt)
    D, L, hc = host_pairs(R, np.concatenate([P, st], axis=1), g, n0, n1)
    Dm, Lm, hcm = host_pairs(Rm, np.concatenate([Pm, stm], axis=1), g, n1, n0)
    scale = R.sum(1) + np.abs(D).sum(1) + np.abs(L).sum(1)
    band = np.abs(np.log(n0 / (n1 * st[:, 1]))) - np.abs(np.log(g))
    ok = np.abs(band) > 1e-9                            # not on the edge of the no-trade band
    ok &= rt < 1e-6
    assert np.all(np.abs(Dm[:, ::-1] - D)[ok] <= 1e3 * (rt * scale)[ok, None])
    assert np.all(np.abs(Lm[:, ::-1] - L)[ok] <= 1e3 * (rt * scale)[ok, None])
    # hc is the coefficient of [[1, -1], [-1, 1]]: the same for the mirror
    assert np.all(np.abs(hcm - hc)[ok] <= 1e3 * (rt * np.abs(hc))[ok])


def test_homogeneity():
    P, R, st, g, n0, n1 = case_set(6, 3000)
    D, L, hc = host_pairs(R, np.concatenate([P, st], axis=1), g, n0, n1)
    for k in (2.0 ** 20, 2.0 ** -24):                  # exact scalings: bit for bit
        st2 = eclp_state(R * k, P)
        assert np.array_equal(st2[:, 0], st[:, 0] * k) and np.array_equal(st2[:, 1], st[:, 1])
        D2, L2, hc2 = host_pairs(R * k, np.concatenate([P, st2], axis=1), g, n0, n1)
        assert np.array_equal(D2, D * k) and np.array_equal(L2, L * k) and np.array_equal(hc2, hc * k)
    st2 = eclp_state(R * 1e-7, P)
    assert np.all(np.abs(st2[:, 0] / (st[:, 0] * 1e-7) - 1) <= 1e-12)


def test_state_against_mpmath():
    rng = np.random.default_rng(7)
    P = random_params(rng, 400)
    R = random_state(rng, P)
    st = eclp_state(R, P)
    for i in range(len(P)):
        r, p = XE.state(*P[i], R[i, 0], R[i, 1])
        assert abs(st[i, 1] - float(p)) <= 8 * U * float(p), (i, P[i], R[i], st[i], float(p))
        # r is x / X(p) (or y / Y(p)): the error of p and of the quotient add, and reach about 9 ulp here
        assert abs(st[i, 0] - float(r)) <= 16 * U * float(r), (i, P[i], R[i], st[i], float(r))
    # the identities: x(beta) = 0, y(alpha) = 0, and the balances' price is p
    with mp.workdps(XE.DPS):
        for i in range(20):
            pool = XE.Pool(*P[i])
            assert abs(pool.point(1, pool.beta)[0]) < mp.mpf(10) ** -40
            assert abs(pool.point(1, pool.alpha)[1]) < mp.mpf(10) ** -40
            pm = (pool.alpha + pool.beta) / 2
            e = pm * mp.mpf(10) ** -20
            t1, t2 = pool.point(1, pm - e), pool.point(1, pm + e)
            assert abs(-(t2[1] - t1[1]) / (t2[0] - t1[0]) / pm - 1) < mp.mpf(10) ** -15


def test_validation():
    good = (0.9, 1.1, math.cos(0.7), math.sin(0.7), 100.0)

    def mk(w=good, r=(1.0, 1.0), toks=(0, 1)):
        return HostPools.from_lists(2, [toks], [r], [0.997], ["eclp"], [w])
    hp = mk()
    assert hp.kind[0] == KIND_ECLP_HOST and hp.eclp.shape == (1, 7)
    hp.validate()
    for w in ((1.1, 0.9) + good[2:], (0.0,) + good[1:], good[:2] + (-0.1, 1.0, 100.0), good[:2] + (0.8, 0.8, 100.0),
              good[:4] + (0.5,), good[:4] + (2e8,), good[:4] + (float("nan"),), good[:4]):
        with pytest.raises(ValueError):
            mk(w=w)
    for r in ((0.0, 0.0), (-1.0, 1.0), (float("inf"), 1.0), (1.0,)):
        with pytest.raises(ValueError):
            mk(r=r)
    with pytest.raises(ValueError):
        mk(toks=(0, 0))
    # c, s normalised by hypot
    w = (0.9, 1.1, math.cos(0.7) * (1 + 4e-13), math.sin(0.7) * (1 + 4e-13), 100.0)
    hp = mk(w=w)
    assert abs(math.hypot(hp.eclp[0, 2], hp.eclp[0, 3]) - 1) <= 2 * U


def test_eclp_pool_against_decimal():
    from decimal import Decimal, getcontext
    from cfmm_routing_code_b200 import instances as I
    getcontext().prec = 50
    bal, dec = [123456789012345678901234, 987654321098], [18, 6]
    prm = [998_000_000_000_000_000, 1_002_000_000_000_000_000, 707_106_781_186_547_524, 707_106_781_186_547_524,
           2_000_000_000_000_000_000_000]
    rates = [1_050_000_000_000_000_000, 1]
    res, w = I.eclp_pool(bal, dec, prm, rates)
    want_r = [Decimal(bal[0]) / Decimal(10) ** 18 * Decimal(rates[0]) / Decimal(10) ** 18,
              Decimal(bal[1]) / Decimal(10) ** 6]
    assert res == [float(x) for x in want_r]
    assert w == tuple(float(Decimal(v) / Decimal(10) ** 18) for v in prm)
    hp = HostPools.from_lists(2, [[0, 1]], [res], [0.9995], ["eclp"], [w])
    assert w[0] <= hp.eclp[0, 6] <= w[1]
    # a known pool: its price at the balances lies in the range, and its peg is s / c
    assert abs(w[3] / w[2] - 1.0) < 1e-15


def test_update_checks():
    from cfmm_routing_code_b200.pools import check_pool_update
    hp = HostPools.from_lists(3, [[0, 1], [1, 2]], [[1.0, 1.0], [2.0, 3.0]], [0.997, 0.997], ["eclp", "product"],
                              [(0.9, 1.1, math.cos(0.78), math.sin(0.78), 50.0), None])
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], reserves=[[0.0, 2.0]], fees=[0.99])
    assert u.reserves.tolist() == [0.0, 2.0]
    for bad in ([[0.0, 0.0]], [[-1.0, 1.0]], [[np.inf, 1.0]]):
        with pytest.raises(ValueError):
            check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], reserves=bad)
    with pytest.raises(ValueError):                      # E-CLP parameters are structure
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, [0], prices=[1.0])


def _csr_args(hp):
    """the cfmm_csr_pools arrays and the records, as batch.CsrStore writes them (no concentrated or bins pools here)"""
    w = hp.weights.copy()
    slot_kind = np.repeat(hp.kind, np.diff(hp.pool_ptr))
    logrw = np.log(np.maximum(hp.reserves, 1e-300) / np.where(slot_kind == 0, hp.weights, 1.0))
    ec = np.nonzero(hp.kind == KIND_ECLP_HOST)[0]
    rec = np.zeros((len(ec), 8))
    E = hp.eclp[ec]
    rec[:, 0:3], rec[:, 3:5], rec[:, 5:7] = E[:, 2:5], E[:, 0:2], E[:, 5:7]
    logrw[hp.pool_ptr[ec]] = 2 * np.arange(len(ec))
    rec = np.ascontiguousarray(rec.reshape(-1) if len(ec) else np.zeros(8))
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
    fn = _host().eclp_host_solve
    fn.argtypes = [C.c_int, C.c_longlong] + [C.c_void_p] * 8 + [C.c_int] + [C.c_void_p] * 8 + [C.c_double]
    fn(n, hp.m, *[p_(k) for k in keep], B, p_(c), p_(a), p_(fl), p_(nu), p_(psi), p_(st), p_(d), p_(l), tol)
    ptr = hp.pool_ptr
    return [types.SimpleNamespace(value=st[p][0], dual_value=st[p][1], psi=psi[p], nu=nu[p], status=int(st[p][7]),
                                  deltas=[d[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)],
                                  lambdas=[l[p][ptr[i]:ptr[i + 1]] for i in range(hp.m)]) for p in range(B)]


def _eclp_near(rng, p, lam_hi=3):
    """weights of an E-CLP whose peg and range sit around the market price p (token 1 per token 0)"""
    phi = np.arctan(p * np.exp(rng.normal(0, 0.05)))
    h = math.hypot(math.cos(phi), math.sin(phi))
    return (p * rng.uniform(0.7, 0.95), p * rng.uniform(1.05, 1.4), math.cos(phi) / h, math.sin(phi) / h,
            10.0 ** rng.uniform(0, lam_hi))


def _reference_with_eclps(seed):
    """the reference's arbitrage.py instance with three E-CLPs added between its tokens"""
    from cfmm_routing_code_b200 import instances as I
    d = I.arbitrage_instance()
    rng = np.random.default_rng(seed)
    mv = np.asarray(d["market_value"], float)
    n = len(mv)
    li, res, fees, kinds, wts = (list(d[k]) for k in ("local_indices", "reserves", "fees", "kinds", "weights"))
    for _ in range(3):
        i, j = (int(t) for t in rng.choice(n, 2, replace=False))
        p = mv[i] / mv[j] * np.exp(rng.normal(0, 0.05))     # token j per token i at (about) the market's prices
        li.append([i, j]); res.append([rng.uniform(5, 50), p * rng.uniform(5, 50)]); fees.append(0.997)
        kinds.append("eclp"); wts.append(_eclp_near(rng, p))
    return HostPools.from_lists(n, li, res, fees, kinds, wts), mv


def test_host_solver_on_reference_instance_with_eclps_certified():
    """the per-thread solver's E-CLP instance (host build) on the reference's arbitrage.py instance with E-CLPs added,
    for the three utilities; every answer certified by xp_eclp.certify"""
    from cfmm_routing_code_b200.api import Arbitrage, Liquidate, Swap
    for seed in range(4):
        hp, mv = _reference_with_eclps(seed)
        n = hp.n_tokens
        utils = [Arbitrage(mv), Liquidate(0, np.r_[0.0, np.full(n - 1, 2.0)]), Swap(1, 0, 1.0)]
        specs = [u.spec(n) for u in utils]
        for spec, r in zip(specs, _host_solve(hp, specs)):
            assert r.status == 0, (seed, r.status)
            XE.certify(hp, spec, r, 1e-9)


def _soc_primal(hp, c, x0):
    """max c'psi s.t. psi >= 0 over E-CLP pools only, every pool's post-trade balances inside its ellipse and >= 0:
    scipy SLSQP on (D, L) >= 0, the ellipse as ||A (t' - r chi)||^2 <= r^2 (an SOC constraint), fp64"""
    from scipy.optimize import minimize
    m, n = hp.m, hp.n_tokens
    tok = hp.tok_idx.reshape(m, 2)
    R = hp.reserves.reshape(m, 2)
    g = hp.gamma
    A, chi = [], []
    for i in range(m):
        with mp.workdps(XE.DPS):
            P = XE.Pool(*hp.eclp[i, :5])
            A.append(np.array([[float(v) for v in row] for row in P.A])); chi.append(np.array([float(v) for v in P.chi]))
    r = hp.eclp[:, 5]

    def split(z):
        return z[:2 * m].reshape(m, 2), z[2 * m:].reshape(m, 2)

    def psi(z):
        D, L = split(z)
        return np.bincount(tok.ravel(), (L - D).ravel(), n)

    cons = [{"type": "ineq", "fun": psi}]
    for i in range(m):
        def ell(z, i=i):
            D, L = split(z)
            u = A[i] @ (R[i] + g[i] * D[i] - L[i] - r[i] * chi[i])
            return (r[i] ** 2 - u @ u) / r[i] ** 2
        cons.append({"type": "ineq", "fun": ell})
        cons.append({"type": "ineq", "fun": lambda z, i=i: R[i] + g[i] * split(z)[0][i] - split(z)[1][i]})
    scale = np.abs(c).max()
    res = minimize(lambda z: -(c @ psi(z)) / scale, x0, method="SLSQP", bounds=[(0, None)] * (4 * m),
                   constraints=cons, options={"ftol": 1e-15, "maxiter": 2000})
    return -res.fun * scale


def test_host_solver_against_scipy_soc_primal():
    """E-CLP-only arbitrage markets: the per-thread solver's value against an independent scipy SOC primal solve"""
    from cfmm_routing_code_b200.api import Arbitrage
    rng = np.random.default_rng(17)
    for trial in range(6):
        n = 3
        price = np.exp(rng.normal(0, 0.2, n))
        li, res, fees, wts = [], [], [], []
        for _ in range(4):
            i, j = (int(t) for t in rng.choice(n, 2, replace=False))
            p = price[i] / price[j] * np.exp(rng.normal(0, 0.05))
            li.append([i, j]); res.append([rng.uniform(5, 50), p * rng.uniform(5, 50)]); fees.append(0.997)
            wts.append(_eclp_near(rng, p, lam_hi=1))
        hp = HostPools.from_lists(n, li, res, fees, ["eclp"] * 4, wts)
        spec = Arbitrage(price).spec(n)
        r = _host_solve(hp, [spec], tol=1e-10)[0]
        assert r.status == 0
        XE.certify(hp, spec, r, 1e-10)
        x0 = np.concatenate([np.concatenate(r.deltas), np.concatenate(r.lambdas)]) * 0.5
        v = _soc_primal(hp, np.asarray(spec.c, float), x0)
        assert abs(v - r.value) <= 1e-7 * max(abs(r.value), np.abs(price).max() * 1e-3), (trial, v, r.value)


def ladder_of(P, st, T):
    """weights (price, bounds, liquidity) of the v3 ladder of T intervals that matches the E-CLP (P = (alpha, beta, c, s,
    lam), st = (r, p)) in token 1 at T + 1 geometric price bounds: interval k holds the pool's token 1 between b_k and
    b_k+1, L_k (sqrt(b_k+1) - sqrt(b_k)) = r (b_k+1 - b_k) C(b_k, b_k+1).  A test helper, not a product API."""
    from cfmm_routing_code_b200.pools import _eclp_BC
    a, b, c, s, lam = P
    bd = a * (b / a) ** (np.arange(T + 1) / T)
    bd[0], bd[-1] = a, b
    dy = st[0] * (bd[1:] - bd[:-1]) * _eclp_BC(np.full(T, c), np.full(T, s), lam * lam, bd[:-1], bd[1:])[1]
    return float(st[1]), bd, dy / (np.sqrt(bd[1:]) - np.sqrt(bd[:-1]))


def _ladder_pairs(hp, g, n0, n1):
    """cfmm_small::ladder_pair of every (concentrated) pool of hp, host build (tests/host_harness/ladder_host.cpp)"""
    src = os.path.join(HERE, "host_harness", "ladder_host.cpp")
    lib = os.path.join(HERE, "_build", "libladder_eclp_host.so")
    if not os.path.exists(lib) or os.path.getmtime(lib) < os.path.getmtime(src):
        os.makedirs(os.path.dirname(lib), exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-o", lib, src], check=True)
    f = C.CDLL(lib).ladder_host_pools
    f.argtypes = [C.c_longlong] + [C.c_void_p] * 8
    m = hp.m
    lp = np.asarray(hp.lad_ptr, np.int64)
    P = np.ascontiguousarray(np.stack([hp.lad_sc[:, 0], hp.lad_sc[:, 1], lp[:-1], lp[1:] - lp[:-1] - 1], 1), np.float64)
    D, L, hc = np.zeros((m, 2)), np.zeros((m, 2)), np.zeros(m)
    cc = lambda x: np.ascontiguousarray(x, np.float64)
    f(m, p_(cc(hp.lad_rec)), p_(P), p_(cc(g)), p_(cc(n0)), p_(cc(n1)), p_(D), p_(L), p_(hc))
    return D, L


def test_ladder_approximation_converges_at_order_2():
    """a v3 ladder matching the pool's token-1 amounts at T + 1 price bounds trades like the pool to O(1/T^2): the
    error falls by 16x (order 2) from T = 1024 to T = 4096"""
    rng = np.random.default_rng(23)
    m = 40
    P = random_params(rng, m)
    P[:, 4] = 10.0 ** rng.uniform(0, 1.5, m)               # the ladder's intervals must resolve the peg's width, ~1 / lam
    w = 10.0 ** rng.uniform(-1, 0.5, m)                    # ranges 10 % .. 3x wide
    P[:, 1] = P[:, 0] * (1 + w)
    P = _check_eclp(P, np.ones((m, 2)))
    pc = np.exp(rng.uniform(np.log(P[:, 0]), np.log(P[:, 1])))
    X, Y = _eclp_xy(P[:, 0], P[:, 1], P[:, 2], P[:, 3], P[:, 4] ** 2, pc)
    R = np.stack([100 * X, 100 * Y], 1)
    st = eclp_state(R, P)
    g = np.full(m, 0.997)
    ps = np.exp(rng.uniform(np.log(P[:, 0]), np.log(P[:, 1])))      # p* inside the range: no cap
    n1 = np.ones(m)
    n0 = ps * n1
    De, Le, _ = host_pairs(R, np.concatenate([P, st], 1), g, n0, n1)
    err = {}
    for T in (256, 1024, 4096):
        lads = [ladder_of(P[i], st[i], T) for i in range(m)]
        hp = HostPools.from_lists(2, [[0, 1]] * m, [None] * m, g, ["concentrated"] * m, lads)
        Dl, Ll = _ladder_pairs(hp, g, n0, n1)
        scale = R.sum(1) + np.abs(De).sum(1) + np.abs(Le).sum(1)
        err[T] = float(np.max((np.abs(Dl - De).sum(1) + np.abs(Ll - Le).sum(1)) / scale))
    order = math.log(err[1024] / err[4096], 4)
    assert 1.7 <= order <= 2.3, (err, order)
    assert err[4096] < err[1024] < err[256]


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _eclp_hostpools(seed, m, n_tokens):
    """m random E-CLPs on random token pairs (as case_set), with their nu"""
    P, R, st, g, n0, n1 = case_set(seed, m)
    P = _check_eclp(P, R)                                # (c, s) normalised by hypot, as from_lists stores them
    st = eclp_state(R, P)
    rng = np.random.default_rng(seed + 100)
    a = rng.integers(0, n_tokens, m)
    b = (a + 1 + rng.integers(0, n_tokens - 1, m)) % n_tokens
    hp = HostPools(n_tokens, np.arange(0, 2 * m + 1, 2, dtype=np.int64), np.stack([a, b], 1).reshape(-1).astype(np.int32),
                   R.reshape(-1).copy(), np.zeros(2 * m), g, np.full(m, KIND_ECLP_HOST, np.uint8),
                   eclp=np.concatenate([P, st], axis=1))
    return hp, a, b, P, R, st, g


@pytest.fixture
def scatter_auto():
    lib = _lib.load()
    yield lib
    lib.cfmm_set_scatter_mode(0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_eval_kernel_against_host_build(scatter_auto, mode):
    """10^6 pools, all four (trades, hess) cells, global (1) and shared (2) scatter; every pool against the host build
    of eclp_pair (itself checked against the 60-digit reference above); psi and arb against sums of the flows; the
    Hessian kernels against the pool decomposition of hcoef"""
    import torch
    lib = scatter_auto
    n, m = (2000 if mode == 2 else 40000), 1_000_000
    hp, a, b, P, R, st, g = _eclp_hostpools(11, m, n)
    hp.validate()
    store = cf.PoolStore(hp, device="cuda:0")
    assert [bk.kind for bk in store.buckets] == [_lib.KIND_ECLP]
    rng = np.random.default_rng(12)
    nu = np.exp(rng.normal(0, 1, n))
    # prices that exercise the range: each pool's p* spread over its range and beyond
    nu_t = torch.as_tensor(nu, dtype=torch.float64, device="cuda:0")
    lib.cfmm_set_scatter_mode(mode)
    D, L, hc = host_pairs(R, np.concatenate([P, st], 1), g, nu[a], nu[b])
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
def test_dense_hessian_small(scatter_auto):
    import torch
    hp, a, b, P, R, st, g = _eclp_hostpools(21, 5000, 40)
    store = cf.PoolStore(hp, device="cuda:0")
    nu = np.exp(np.random.default_rng(2).normal(0, 1, 40))
    store.evaluate(torch.as_tensor(nu, device="cuda:0"), hess=True)
    H = store.hess_dense().cpu().numpy()
    _, _, hc = host_pairs(R, np.concatenate([P, st], 1), g, nu[a], nu[b])
    want = np.zeros((40, 40))
    np.add.at(want, (a, a), hc); np.add.at(want, (b, b), hc); np.add.at(want, (a, b), -hc); np.add.at(want, (b, a), -hc)
    assert np.allclose(H[:40, :40] if H.ndim == 2 else H.reshape(40, 40), want, rtol=1e-12, atol=1e-12 * np.abs(hc).max())


def _mixed_market(seed, n=6, lam_hi=3.0):
    """E-CLPs beside product, weighted, sum, bounded, StableSwap, concentrated, cryptoswap and bins pools; returns
    (n, local_indices, reserves, fees, kinds, weights, market prices)"""
    rng = np.random.default_rng(seed)
    li, res, fees, kinds, wts = [], [], [], [], []
    price = np.exp(rng.normal(0, 0.3, n))
    def pair():
        i, j = rng.choice(n, 2, replace=False)
        return [int(i), int(j)], price[i] / price[j]       # token-1 per token-0 market price
    for _ in range(4):                                    # E-CLPs around the market price
        l, p = pair()
        phi = np.arctan(p * np.exp(rng.normal(0, 0.01)))
        h = math.hypot(math.cos(phi), math.sin(phi))
        w = (p * 0.9, p * 1.1, math.cos(phi) / h, math.sin(phi) / h, 10.0 ** rng.uniform(0, lam_hi))
        li.append(l); res.append([float(10 * rng.uniform(1, 2)), float(10 * p * rng.uniform(1, 2))]); fees.append(0.997)
        kinds.append("eclp"); wts.append(w)
    for kind in ("product", "geomean", "sum", "bounded_product", "stableswap", "concentrated", "cryptoswap", "bins"):
        l, p = pair()
        if kind == "geomean":
            l = [int(t) for t in rng.choice(n, 3, replace=False)]
            li.append(l); res.append([10.0 / price[t] for t in l]); wts.append([1, 2, 3])
        elif kind == "concentrated":
            li.append(l); res.append(None); wts.append((p, [p * 0.8, p, p * 1.25], [20.0, 30.0]))
        elif kind == "bins":
            li.append(l); res.append(None); wts.append(([p * 0.99, p * 1.01], [0.0, 3.0], [3.0 * p, 0.0]))
        else:
            li.append(l); res.append([10.0, 10.0 * p])
            wts.append(None if kind in ("product", "sum") else (1.0, 2.0) if kind == "bounded_product"
                       else (50.0, 1.0, 1.0 / p) if kind == "stableswap" else (4.0, 1e-3, 1.0, 1.0 / p))
        fees.append(0.997); kinds.append(kind)
    reach, grew = {0}, True                              # every token reachable from token 0 (else a product pool to it)
    while grew:
        grew = False
        for l in li:
            if reach & set(l) and not set(l) <= reach:
                reach |= set(l); grew = True
    for t in sorted(set(range(n)) - reach):
        li.append([0, t]); res.append([10.0, 10.0 * price[0] / price[t]]); fees.append(0.997); kinds.append("product")
        wts.append(None)
    return n, li, res, fees, kinds, wts, price


@pytest.mark.gpu
@pytest.mark.parametrize("native", [False, "hostloop", True])
@pytest.mark.parametrize("seed", range(6))
def test_mixed_markets_certified(seed, native):
    """solver.py, the host loop and native=True (which falls back to solver.py: the store is not one blocked bucket) on
    markets of E-CLPs beside every other kind, for the three utilities; every answer optimal and certified by
    xp_eclp.certify"""
    n, li, res, fees, kinds, wts, price = _mixed_market(seed)
    hp = HostPools.from_lists(n, li, res, fees, kinds, wts)
    for util in (cf.Arbitrage(price), cf.Liquidate(0, np.r_[0.0, 1.0, 0.5, 0.0, 0.0, 0.0]), cf.Swap(1, 2, 0.5)):
        r = cf.solve_pools(hp, util, device="cuda:0", tol=1e-9, native=native, method="pools")
        assert r.status == "optimal", (seed, native, util, r.status)
        XE.certify(hp, util.spec(n), r, 1e-9)


@pytest.mark.gpu
def test_whole_market_ladder_approximation():
    """the market with every E-CLP replaced by its ladder_of at T intervals: the solve's value approaches the E-CLP
    market's at order about 2 in T"""
    n, li, res, fees, kinds, wts, price = _mixed_market(2, lam_hi=1.5)
    hp = HostPools.from_lists(n, li, res, fees, kinds, wts)
    u = cf.Arbitrage(price)
    r = cf.solve_pools(hp, u, device="cuda:0", tol=1e-12, method="pools")
    assert r.status == "optimal"
    err = {}
    for T in (256, 1024):
        k2, r2, w2 = list(kinds), list(res), list(wts)
        for i in np.nonzero(hp.kind == KIND_ECLP_HOST)[0].tolist():
            k2[i], r2[i], w2[i] = "concentrated", None, ladder_of(hp.eclp[i, :5], hp.eclp[i, 5:], T)
        h2 = HostPools.from_lists(n, li, r2, fees, k2, w2)
        rl = cf.solve_pools(h2, u, device="cuda:0", tol=1e-12, method="pools")
        assert rl.status == "optimal"
        err[T] = abs(rl.value - r.value) / abs(r.value)
    assert err[1024] <= err[256] / 8, err


@pytest.mark.gpu
def test_per_thread_paths_certified():
    """the per-thread solver (cfmm_batch_solve_eclp): solve_batch on the reference instance with E-CLPs for the three
    utilities, solve_many over mixed markets, solve_sweep over a Swap ladder; every answer optimal and certified"""
    from cfmm_routing_code_b200.api import Arbitrage, Liquidate, Swap
    hp, mv = _reference_with_eclps(0)
    n = hp.n_tokens
    utils = [Arbitrage(mv), Liquidate(0, np.r_[0.0, np.full(n - 1, 2.0)]), Swap(1, 0, 1.0)]
    rs = cf.solve_batch(hp, utils, tol=1e-9, device="cuda:0")
    for u, r in zip(utils, rs):
        assert r.status == "optimal"
        XE.certify(hp, u.spec(n), r, 1e-9)
    # against the host build of the same instance: the same iteration, to rounding
    hr = _host_solve(hp, [u.spec(n) for u in utils])
    for r, h in zip(rs, hr):
        assert abs(r.value - h.value) <= 1e-9 * max(1.0, abs(h.value))
    probs = []
    for seed in range(40):
        m = _mixed_market(100 + seed)
        probs.append((HostPools.from_lists(m[0], *m[1:6]), cf.Arbitrage(m[6])))
    rs = cf.solve_many(probs, tol=1e-9, device="cuda:0")
    for (h, u), r in zip(probs, rs):
        assert r.status == "optimal"
        XE.certify(h, u.spec(h.n_tokens), r, 1e-9)
    n6, li, res, fees, kinds, wts, price = _mixed_market(7)
    utils = [cf.Swap(1, 2, t) for t in np.linspace(0.1, 3.0, 12)]
    rs = cf.solve_sweep(li, res, fees, kinds, wts, utils, n_tokens=n6, tol=1e-9, device="cuda:0")
    hp6 = HostPools.from_lists(n6, li, res, fees, kinds, wts)
    for u, r in zip(utils, rs):
        assert r.status == "optimal"
        XE.certify(hp6, u.spec(n6), r, 1e-9)
    r = cf.solve(li, res, fees, kinds, wts, utility=cf.Arbitrage(price), device="cuda:0", method="thread", tol=1e-9)
    assert r.status == "optimal"
    XE.certify(hp6, cf.Arbitrage(price).spec(n6), r, 1e-9)


@pytest.mark.gpu
def test_older_per_thread_entries_give_eclp_problems_status_3():
    import torch
    from cfmm_routing_code_b200 import batch as BT
    hp, mv = _reference_with_eclps(1)
    store = BT.CsrStore(hp, device="cuda:0")
    n = hp.n_tokens
    spec = cf.Arbitrage(mv).spec(n)
    lib = store.lib
    for name in ("cfmm_batch_solve", "cfmm_batch_solve_stableswap", "cfmm_batch_solve_stableswap_n",
                 "cfmm_batch_solve_concentrated", "cfmm_batch_solve_cryptoswap", "cfmm_batch_solve_tricrypto",
                 "cfmm_batch_solve_bins"):
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
    assert lib.cfmm_batch_solve_eclp(C.byref(store.c_pools), None, None, None, None, None) == -1


@pytest.mark.gpu
def test_rank_stores_sum_to_the_single_store():
    import torch
    hp, a, b, P, R, st, g = _eclp_hostpools(31, 30001, 300)
    nu = torch.as_tensor(np.exp(np.random.default_rng(3).normal(0, 1, 300)), device="cuda:0")
    one = cf.PoolStore(hp, device="cuda:0").evaluate(nu).cpu().numpy()
    for world in (2, 3):
        tot = sum(cf.PoolStore(hp, device="cuda:0", rank=k, world=world).evaluate(nu).cpu().numpy() for k in range(world))
        assert np.allclose(tot, one, rtol=1e-12, atol=1e-12 * np.abs(one).max())


@pytest.mark.gpu
def test_updates_equal_a_fresh_store():
    import torch
    n, li, res, fees, kinds, wts, price = _mixed_market(3)
    hp = HostPools.from_lists(n, li, res, fees, kinds, wts)
    store = cf.PoolStore(hp, device="cuda:0")
    ids = np.nonzero(np.asarray(hp.kind) == KIND_ECLP_HOST)[0][:3]
    rng = np.random.default_rng(5)
    newR = [[res[i][0] * rng.uniform(0.5, 1.5), res[i][1] * rng.uniform(0.5, 1.5)] for i in ids]
    newR[0][0] = 0.0                                      # one pool emptied of token 0
    newg = [0.999, 0.995, 1.0]
    store.update_pools(ids, reserves=newR, fees=newg)
    res2, fees2 = list(res), list(fees)
    for k, i in enumerate(ids):
        res2[i], fees2[i] = newR[k], newg[k]
    fresh = cf.PoolStore(HostPools.from_lists(n, li, res2, fees2, kinds, wts), device="cuda:0")
    for b1, b2 in zip(store.buckets, fresh.buckets):
        if getattr(b1, "blocked", False):                 # the constant-product pools: not updated here
            continue
        for name in ("reserves", "gamma", "weights", "logrw", "tok_idx"):
            t1, t2 = getattr(b1, name), getattr(b2, name)
            assert (t1 is None) == (t2 is None) and (t1 is None or torch.equal(t1, t2)), (b1.kind, name)
    r = cf.solve_pools(HostPools.from_lists(n, li, res2, fees2, kinds, wts), cf.Arbitrage(price), store=store,
                       device="cuda:0", tol=1e-9)
    assert r.status == "optimal"
    # an invalid entry (negative reserve) in a 1000-pool block changes nothing
    hp2, *_ = _eclp_hostpools(41, 1000, 50)
    st2 = cf.PoolStore(hp2, device="cuda:0")
    before = st2.buckets[0].weights.clone(), st2.buckets[0].reserves.clone()
    bad = hp2.reserves.reshape(-1, 2) * 1.1
    bad[777, 1] = -1.0
    with pytest.raises(ValueError):
        st2.update_pools(np.arange(1000), reserves=bad, fees=np.full(1000, 0.99))
    assert torch.equal(before[0], st2.buckets[0].weights) and torch.equal(before[1], st2.buckets[0].reserves)


@pytest.mark.gpu
def test_abi_codes():
    import ctypes
    import torch
    lib = _lib.load()
    hp, *_ = _eclp_hostpools(51, 100, 10)
    store = cf.PoolStore(hp, device="cuda:0")
    bk = store.buckets[0]
    nu = torch.ones(10, dtype=torch.float64, device="cuda:0")
    acc = torch.zeros(11, dtype=torch.float64, device="cuda:0")
    c = _lib.Bucket.from_buffer_copy(bk.c_bucket)
    assert lib.cfmm_arb_eval(ctypes.byref(c), 10, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc[10:].data_ptr(),
                             None, None) == 0
    c.arity = 3
    assert lib.cfmm_arb_eval(ctypes.byref(c), 10, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc[10:].data_ptr(),
                             None, None) == -2
    c.arity = 2
    c.weights = None
    assert lib.cfmm_arb_eval(ctypes.byref(c), 10, nu.data_ptr(), None, 0.0, acc.data_ptr(), acc[10:].data_ptr(),
                             None, None) == -1
