"""The extended-precision reference (tests/xp_reference.py) against 40-digit arithmetic and the fp64 oracle, and its
certificate against good and deliberately broken answers.  CPU only."""
import decimal
import types
from decimal import Decimal

import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import instances as I
from cfmm_routing_code_b200.solver import solve_dual
from cpu_evaluator import OracleEvaluator
from oracle import cfmm_oracle as O
import helpers as H
import xp_reference as X


# ---- 40-digit scalar restatements of the four kinds -----------------------------------------------------------------
def _dec(x):
    return Decimal(float(x))                    # exact: every input is an fp64 number


def _dec_product(R, V, g, nu, cap_at=None):
    """constant product on V (= R, or R + o for a bounded pool whose payout is capped at R)"""
    D = [Decimal(0)] * 2; L = [Decimal(0)] * 2
    p = [nu[0] * V[0], nu[1] * V[1]]
    for a, b in ((0, 1), (1, 0)):
        if g * p[b] > p[a]:
            t = (g * p[b] / p[a]).sqrt()
            L[b] = V[b] * (1 - 1 / t); D[a] = V[a] * (t - 1) / g
            if cap_at is not None and L[b] > R[b]:
                L[b] = R[b]; D[a] = V[a] * R[b] / (g * cap_at[b])
    return D, L


def _dec_sum(R, g, nu):
    D = [Decimal(0)] * 2; L = [Decimal(0)] * 2
    for a, b in ((0, 1), (1, 0)):
        if g * nu[b] > nu[a]:
            L[b] = R[b]; D[a] = R[b] / g
    return D, L


def _dec_geomean(R, w, g, nu):
    k = len(R)
    tB = [(R[j] * nu[j] / w[j]).ln() for j in range(k)]
    lg = g.ln()
    tA = [t - lg for t in tB]
    if max(tB) <= min(tA):
        return [Decimal(0)] * k, [Decimal(0)] * k

    def h(s):
        return sum(w[j] * (max(s - tA[j], Decimal(0)) + min(s - tB[j], Decimal(0))) for j in range(k))
    bps = sorted(tA + tB)
    s = None
    for lo, hi in zip(bps[:-1], bps[1:]):
        hl, hr = h(lo), h(hi)
        if hl <= 0 <= hr:
            s = lo if hr == hl else lo - hl * (hi - lo) / (hr - hl)
            break
    assert s is not None
    D = [R[j] * ((max(s - tA[j], Decimal(0))).exp() - 1) / g for j in range(k)]
    L = [-R[j] * ((min(s - tB[j], Decimal(0))).exp() - 1) for j in range(k)]
    return D, L


def _decimal_response(hp, nu):
    ptr = hp.pool_ptr
    D = [None] * len(hp.reserves); L = [None] * len(hp.reserves)
    with decimal.localcontext() as ctx:
        ctx.prec = 40
        for i in range(hp.m):
            sl = slice(ptr[i], ptr[i + 1])
            R = [_dec(x) for x in hp.reserves[sl]]
            w = [_dec(x) for x in hp.weights[sl]]
            n_ = [_dec(nu[t]) for t in hp.tok_idx[sl]]
            g = _dec(hp.gamma[i])
            if hp.kind[i] == X.KIND_SUM:
                d, l = _dec_sum(R, g, n_)
            elif hp.kind[i] == X.KIND_BOUNDED:
                d, l = _dec_product(R, [R[0] + w[0], R[1] + w[1]], g, n_, cap_at=w)
            elif len(R) == 2 and hp.weights[sl][0] == hp.weights[sl][1] == 0.5:
                d, l = _dec_product(R, R, g, n_)
            else:
                d, l = _dec_geomean(R, w, g, n_)
            for j, s in enumerate(range(ptr[i], ptr[i + 1])):
                D[s], L[s] = d[j], l[j]
    return D, L


def _edge_pools(rng):
    """pools of every kind at the edges where a closed form goes wrong: prices 1e-12 off the no-trade cone on either
    side, fee 1.0, arity 2..9 and 32, bounded pools in range, at the payout cap and out of range"""
    n = 48
    nu = np.exp(rng.normal(0, 1, n))
    # the last four tokens sit on the constant-sum switch gamma nu_b = nu_a: a tie, and 1e-12 to either side of it
    nu[-4:] = [1.0, 1.0, (1 + 1e-12) / 0.997, (1 - 1e-12) / 0.997]
    li, res, fees, kinds, wts = [], [], [], [], []

    def add(toks, R, g, kd, w=None):
        li.append([int(t) for t in toks]); res.append([float(x) for x in R]); fees.append(float(g))
        kinds.append(kd); wts.append(w)
    for i in range(120):                                       # constant product
        a, b = rng.choice(n, 2, replace=False)
        g = [0.997, 1.0, 0.9, 0.9995][i % 4]
        R0 = float(np.exp(rng.normal(6, 2)))
        q = nu[a] * R0 / (g * nu[b])                           # R1 that puts gamma p1 exactly on p0
        R1 = q * [1 + 1e-12, 1 - 1e-12, np.exp(rng.normal(0, 0.3)), np.exp(rng.normal(0, 3))][(i // 4) % 4]
        add((a, b), (R0, R1), g, "product")
    for k in list(range(2, 10)) + [32]:                        # weighted, every arity
        for i in range(12):
            toks = rng.choice(n, k, replace=False)
            w = rng.dirichlet(np.ones(k))
            R = np.exp(rng.normal(6, 1)) * w / nu[toks] * np.exp([0.0, 1e-9, 0.05, 1.0][i % 4] * rng.standard_normal(k))
            add(toks, R, [0.997, 1.0, 0.99][i % 3], "geomean", list(w))
    for i in range(60):                                        # constant sum, near and on the LP's switch
        a, b = rng.choice(n, 2, replace=False)
        g = [0.997, 1.0, 0.9995][i % 3]
        if i % 4 == 3:
            a, b, g = n - 4, [n - 3, n - 2, n - 1][(i // 4) % 3], [1.0, 0.997, 0.997][(i // 4) % 3]
        R = np.exp(rng.normal(5, 1, 2))
        add((a, b), R, g, "sum")
    for i in range(90):                                        # bounded product: in range / at the cap / out of range
        a, b = rng.choice(n, 2, replace=False)
        p = nu[a] / nu[b]
        where = [1.0, 0.9, 3.0, 0.2, 1.3, 0.75][i % 6]         # where the position's price sits against the market's
        lo, hi = p * where * np.exp(-0.1), p * where * np.exp(0.1)
        R, o = I.v3_position(np.exp(rng.normal(5, 1)), lo, hi, p * where * np.exp(0.05 * rng.standard_normal()))
        if i % 12 == 11:
            R, o = I.v3_position(np.exp(rng.normal(5, 1)), lo, hi, hi * 2)      # out of range: token 1 only
        add((a, b), R, [0.997, 1.0, 0.99][i % 3], "bounded_product", list(o))
    hp = cf.HostPools.from_lists(n, li, res, fees, kinds, wts)
    return hp, nu


def test_reference_agrees_with_40_digit_arithmetic_on_every_kind():
    rng = np.random.default_rng(7)
    hp, nu = _edge_pools(rng)
    r = X.response(hp, nu)
    Dd, Ld = _decimal_response(hp, nu)
    ar = np.diff(hp.pool_ptr)
    pool = np.repeat(np.arange(hp.m), ar)
    virt = hp.reserves + np.where(np.repeat(hp.kind, ar) == X.KIND_BOUNDED, hp.weights, 0.0)
    with decimal.localcontext() as ctx:
        ctx.prec = 40
        err = np.array([float(abs(Decimal(str(r["delta"][s])) - Dd[s]) + abs(Decimal(str(r["lam"][s])) - Ld[s]))
                        for s in range(len(Dd))])
        size = np.array([float(max(abs(Dd[s]), abs(Ld[s]))) for s in range(len(Dd))])
    scale = np.maximum.reduceat(np.maximum(virt, size), hp.pool_ptr[:-1])[pool]     # the pool's reserves (or trade)
    rel = err / scale
    # longdouble carries 64 bits (u = 5.4e-20); the geomean root goes through logs of magnitude <~ 20 and arity <= 32
    # breakpoint sums: a few hundred u at most, i.e. ~1e-17 of the reserves
    assert rel.max() <= 1e-17, (rel.max(), int(pool[rel.argmax()]))
    # every kind trades somewhere in the set, and the cap / out-of-range branches of the bounded pools are taken
    traded = np.add.reduceat(np.abs(r["lam"]) > 0, hp.pool_ptr[:-1]) > 0
    for kd in (X.KIND_GEOMEAN, X.KIND_SUM, X.KIND_BOUNDED):
        assert traded[hp.kind == kd].any() and (~traded[hp.kind == kd]).any()
    bnd = np.repeat(hp.kind == X.KIND_BOUNDED, ar)
    assert np.any(bnd & (r["lam"] == hp.reserves) & (hp.reserves > 0)) and np.any(bnd & (hp.reserves == 0))


@pytest.mark.parametrize("case", ["mixed", "v3"])
def test_reference_agrees_with_the_fp64_oracle(case):
    if case == "mixed":
        hp, s = H.mixed_host_pools(6000, 120, seed=21)
        nus = [H.random_prices(s["prices"], k, 0.03) for k in range(3)]
    else:
        hp = H.host_pools(I.v3_instance())
        nus = [np.array(x) for x in ([1.31, 1.02, 0.47], [1.0, 1.0, 0.5], [3.0, 1.0, 0.2], [0.3, 1.0, 2.0])]
    bk = O.Buckets(H.oracle_pools(hp))
    for nu in nus:
        ref = O.evaluate(bk, nu, 0.0, want_trades=True)
        r = X.response(hp, nu)
        Rmax = np.repeat(np.maximum.reduceat(hp.reserves + hp.weights * (np.repeat(hp.kind, np.diff(hp.pool_ptr)) == 3),
                                             hp.pool_ptr[:-1]), np.diff(hp.pool_ptr))
        # the oracle is fp64: its closed forms err by ~1e-15 of the reserves, its logs by a little more
        assert np.max(np.abs(r["delta"] - ref["delta"]) / Rmax) <= 1e-12
        assert np.max(np.abs(r["lam"] - ref["lam"]) / Rmax) <= 1e-12
        psi, gross, k = X.flows(hp, r["delta"], r["lam"])
        assert np.max(np.abs(psi - ref["psi"]) / (gross + 1e-300)) <= 1e-11
        assert abs(r["arb"].sum() - ref["arb"]) <= 1e-11 * float((X.ld(nu) * gross).sum())


# ---- the certificate -------------------------------------------------------------------------------------------------
def _spec(u):
    return cf.DualSpec(u.c, u.a, u.eq, u.pinned)


def _mixed_problems():
    """(HostPools, oracle utility) pairs: small problems of every kind with every utility, and a 1500-pool mixed market"""
    rng = np.random.default_rng(31)
    out = []
    for _ in range(4):
        hp, d, prices = H.random_small_problem(rng)
        out += [(hp, u) for u in H.random_utilities(rng, hp.n_tokens, prices)]
    hp, s = H.mixed_host_pools(1500, 40, seed=3)
    basket = I.synth_basket(40, s["prices"], seed=3, n_assets=6)
    out += [(hp, O.Utility.arbitrage(s["prices"])), (hp, O.Utility.liquidate(40, 0, basket)),
            (hp, O.Utility.swap(40, 3, 5, float(np.exp(6.0) / s["prices"][3])))]
    return out


def test_certificate_accepts_oracle_solutions_of_every_utility():
    for hp, u in _mixed_problems():
        ro = O.solve(H.oracle_pools(hp), u, tol=1e-9)
        assert ro.status == "optimal"
        X.certify(hp, u, ro, 1e-9)


def test_certificate_accepts_the_cpu_twin_of_the_solver():
    """solver.solve_dual over the oracle-backed evaluator: the product's outer loop, certified from its own answer"""
    for hp, u in _mixed_problems()[-3:] + _mixed_problems()[:3]:
        ev = OracleEvaluator(hp)
        info = solve_dual(ev, _spec(u), tol=1e-9)
        assert info.status == "optimal"
        d, l = ev.gather_trades()
        r = types.SimpleNamespace(value=info.primal_value, dual_value=info.dual_value, psi=info.psi.numpy(),
                                  nu=info.nu.numpy(), deltas=[d], lambdas=[l])
        X.certify(hp, _spec(u), r, 1e-9)


def _solved(u_kind):
    hp, s = H.mixed_host_pools(1500, 40, seed=3)
    u = {"arb": O.Utility.arbitrage(s["prices"]),
         "liq": O.Utility.liquidate(40, 0, I.synth_basket(40, s["prices"], seed=3, n_assets=6))}[u_kind]
    ro = O.solve(H.oracle_pools(hp), u, tol=1e-9)
    assert ro.status == "optimal"
    X.certify(hp, u, ro, 1e-9)
    d, l = np.concatenate(ro.deltas), np.concatenate(ro.lambdas)
    return hp, u, ro, d, l


def _as_result(ro, **kw):
    f = dict(value=ro.value, dual_value=ro.dual_value, psi=ro.psi.copy(), nu=ro.nu.copy(),
             deltas=[np.concatenate(ro.deltas)], lambdas=[np.concatenate(ro.lambdas)])
    f.update(kw)
    return types.SimpleNamespace(**f)


def test_certificate_rejects_each_broken_answer():
    hp, u, ro, d, l = _solved("arb")
    pool = np.repeat(np.arange(hp.m), np.diff(hp.pool_ptr))
    gm = np.repeat(hp.kind == X.KIND_GEOMEAN, np.diff(hp.pool_ptr))
    # (1) one trading pool's trades zeroed: psi no longer is the sum of the trades
    i = int(pool[np.argmax(l)])
    d1, l1 = d.copy(), l.copy()
    sl = slice(hp.pool_ptr[i], hp.pool_ptr[i + 1])
    d1[sl] = 0.0; l1[sl] = 0.0
    with pytest.raises(AssertionError, match="psi does not match the trades"):
        X.certify(hp, u, _as_result(ro, deltas=[d1], lambdas=[l1]), 1e-9)
    # (2) one Lambda of a weighted pool that trades >= 1e-3 of its reserve, times 1 + 1e-9: the pool's invariant drops by
    # w (1e-9 L / x) >= 5e-12 > FEAS_TOL for the pool picked (L / x >= 1e-2 asserted)
    frac = np.where(gm, l / (hp.reserves - l), 0.0)                  # L / x_post of the slot paying out
    s_ = int(np.argmax(frac))
    assert l[s_] >= 1e-3 * hp.reserves[s_] and frac[s_] >= 1e-2
    l2 = l.copy(); l2[s_] *= 1 + 1e-9
    with pytest.raises(AssertionError, match="not pool-feasible"):
        X.certify(hp, u, _as_result(ro, lambdas=[l2]), 1e-9)
    # (3) value off by 1e-9 relative
    with pytest.raises(AssertionError, match="reported value disagrees"):
        X.certify(hp, u, _as_result(ro, value=ro.value * (1 + 1e-9)), 1e-9)
    # (5) nu_j < c_j on an Arbitrage token (a token at its bound nu = c, moved 1e-9 below it)
    j = int(np.argmin(ro.nu / u.c))
    nu5 = ro.nu.copy(); nu5[j] = u.c[j] * (1 - 1e-9)
    with pytest.raises(AssertionError, match="nu < c on an inequality token"):
        X.certify(hp, u, _as_result(ro, nu=nu5), 1e-9)
    # (6) every trade halved, psi and value recomputed from the halved trades: pool-feasible (each pool's feasible set is
    # convex and holds both R and the optimal post-trade point), psi = psi*/2 >= 0 meets the Arbitrage constraints, the
    # scalars agree -- only the dual bound can tell that half the value is left on the table
    psi6, _, _ = X.flows(hp, d / 2, l / 2)
    res6 = _as_result(ro, deltas=[d / 2], lambdas=[l / 2], psi=psi6.astype(float),
                      value=float((X.ld(u.c) * psi6).sum()))
    fails = X.certify(hp, u, res6, 1e-9, check=False)["fails"]
    assert len(fails) == 1 and fails[0].startswith("dual bound does not close the gap"), fails       # check 4 alone
    with pytest.raises(AssertionError, match="dual bound does not close the gap"):
        X.certify(hp, u, res6, 1e-9)
    # (7) every Lambda times 1 + 1e-9, psi and value recomputed: the pools pay out more than their invariants allow, and
    # the claimed value beats the dual bound -- which pool-feasible trades never can (D - P >= -V, certify's check 4)
    l7 = l * (1 + 1e-9)
    psi7, _, _ = X.flows(hp, d, l7)
    res7 = _as_result(ro, lambdas=[l7], psi=psi7.astype(float), value=float((X.ld(u.c) * psi7).sum()))
    with pytest.raises(AssertionError, match="primal value exceeds the dual bound"):
        X.certify(hp, u, res7, 1e-9)
    hp, u, ro, d, l = _solved("liq")
    # (8) the liquidation's trades taken at a price vector moved 1e-3 on one token: pool-feasible and self-consistent,
    # but the basket is no longer sold exactly and the value falls short of the dual bound
    nu8 = ro.nu.copy(); nu8[5] *= 1 + 1e-3
    r8 = X.response(hp, nu8)
    psi8, _, _ = X.flows(hp, r8["delta"], r8["lam"])
    res8 = _as_result(ro, deltas=[r8["delta"].astype(float)], lambdas=[r8["lam"].astype(float)],
                      psi=psi8.astype(float), value=float((X.ld(u.c) * psi8).sum()))
    with pytest.raises(AssertionError, match="dual bound does not close the gap"):
        X.certify(hp, u, res8, 1e-9)
    # (4) a pinned nu != c (the liquidation target)
    nu4 = ro.nu.copy(); nu4[0] *= 1 + 1e-12
    with pytest.raises(AssertionError, match="nu differs from c on a pinned token"):
        X.certify(hp, u, _as_result(ro, nu=nu4), 1e-9)
