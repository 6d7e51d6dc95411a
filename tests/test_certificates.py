"""Every solve path's returned answer -- trades, psi, nu, value -- certified in extended precision (xp_reference.certify),
from a few tokens to 65 536, and the evaluation kernel's variants against the extended-precision reference.  H100."""
import numpy as np
import pytest
import torch

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib, batch as B, instances as I, pools as PL
import helpers as H
import xp_reference as X

pytestmark = pytest.mark.gpu

F64 = dict(dtype=torch.float64, device="cuda")


def clustered_market(m, n, seed, cluster=256, hub_frac=0.05):
    """A routing graph of the kind real markets have: tokens in clusters of `cluster` consecutive ids; ~95% of the pools
    pair two tokens of one cluster, the rest pair the first tokens ("hubs") of two random clusters, so any two tokens are
    about 6 hops apart.  The token-keyed sort of the blocked layout keeps every tile of such a market far below its
    per-tile token cap at any size (uniformly random pairs stop fitting somewhere above ~8k tokens).  Reserves, fees and
    prices are drawn as in instances.synth_const_product."""
    assert n % cluster == 0
    rng = np.random.default_rng(seed)
    p = np.exp(rng.standard_normal(n))
    nc = n // cluster
    home = rng.integers(0, nc, m) * cluster
    a = home + rng.integers(0, cluster, m)
    b = home + (a - home + 1 + rng.integers(0, cluster - 1, m)) % cluster
    hub = rng.random(m) < hub_frac
    ca = rng.integers(0, nc, m)
    cb = (ca + 1 + rng.integers(0, nc - 1, m)) % nc
    a, b = np.where(hub, ca * cluster, a), np.where(hub, cb * cluster, b)
    liq = np.exp(8.0 + 1.5 * rng.standard_normal(m))
    R = np.stack([liq / p[a], liq / p[b]], 1) * np.exp(0.02 * rng.standard_normal((m, 2)))
    gamma = np.array([0.997, 0.999, 0.9995])[rng.integers(0, 3, m)]
    hp = cf.HostPools.from_pairs(n, np.stack([a, b], 1), R, gamma)
    return hp, dict(prices=p)


def _market(n):
    """(HostPools, prices) at token count n: uniformly random pairs while the blocked layout holds them, clustered above"""
    if n >= 16_384:
        return clustered_market({16_384: 300_000, 65_536: 600_000}[n], n, seed=n % 97)
    m = 20_000 if n < 4000 else 200_000 if n < 8000 else 400_000
    hp, s = H.cp_host_pools(m, n, seed=3)
    return hp, s


def _native_store(hp):
    st = cf.PoolStore(hp)
    assert len(st.buckets) == 1 and st.buckets[0].blocked            # one blocked bucket: the native solvers apply
    return st


def _report(tag, r, rep):
    """one line per certificate, for the record: each measured quantity with its bound"""
    q = " ".join(f"{k}={v[0]:.2e}/{v[1]:.2e}" for k, v in rep.items() if isinstance(v, tuple))
    print(f"CERT {tag} status={r.status} iters={r.iters} evals={r.evals} hvps={r.hvps} {q}")


def _utility(name, hp, prices):
    """(utility, nu0): an Arbitrage at the market prices, a Liquidate of a min(16, n-1)-token basket into token 0, a Swap
    of token 0 for token 1"""
    n = hp.n_tokens
    if name == "arbitrage":
        return cf.Arbitrage(prices), None
    if name == "liquidate":
        return cf.Liquidate(0, I.synth_basket(n, prices, seed=2, n_assets=min(16, n - 1))), prices / prices[0]
    return cf.Swap(0, 1, 0.5 * float(np.exp(8.0)) / prices[0]), prices / prices[1]


# ---- G1: the token-count regimes of the native solvers -----------------------------------------------------------------
@pytest.mark.parametrize("util_name", ["arbitrage", "liquidate", "swap"])
@pytest.mark.parametrize("n", [15, 17, 33, 4095, 4097, 8193, 16_384, 65_536])
def test_native_solvers_certify_at_every_token_count_regime(n, util_name):
    """The persistent solver cuts its vector algebra into nsl = min(256, ceil(n/16)) slices, one warp per slice, one token
    per lane: n = 15 is one slice; 4097 gives ragged slices of 16-17 tokens; 8193 slices of 32-33, the loops' second lane
    turn; 65 536 slices of 256, eight turns.  Both native solvers (persistent kernel, C++ host loop) must return a
    certified answer, and the same prices.  (The 65 536-token swap is where an unbounded truncated-CG step stalled the
    persistent solver and solver.py's CG loop: every trial of the line search sat on the +-20 log-price clamp.)"""
    hp, s = _market(n)
    st = _native_store(hp)
    tol = 1e-8
    util, nu0 = _utility(util_name, hp, s["prices"])
    spec = util.spec(n)
    rs = {}
    for impl in ("hostloop", "persist"):
        r = cf.solve_pools(hp, util, nu0=nu0, tol=tol, store=st, native=impl, method="pools")
        assert r.info.history == [], impl                                # a native loop, not solver.py
        assert r.status == "optimal", (n, util_name, impl, r.status, r.iters)
        _report(f"G1 n={n} {util_name} {impl}", r, X.certify(hp, spec, r, tol))
        rs[impl] = r
    np.testing.assert_allclose(rs["persist"].nu, rs["hostloop"].nu, rtol=1e-6)


# ---- G2: the python loop at the linear_solver switch ------------------------------------------------------------------
@pytest.mark.parametrize("case", ["dense-256", "cg-257", "cg-clustered-16384"])
def test_python_loop_certifies_on_both_sides_of_the_linear_solver_switch(case):
    """solver.py picks the dense Cholesky up to 256 tokens (constant product) and CG above"""
    if case == "cg-clustered-16384":
        hp, s = clustered_market(300_000, 16_384, seed=5)
    else:
        n = int(case.split("-")[1])
        hp, s = H.cp_host_pools(20_000, n, seed=n)
    util = cf.Arbitrage(s["prices"])
    r = cf.solve_pools(hp, util, tol=1e-8, native=False, method="pools")
    assert len(r.info.history) > 0 and r.status == "optimal"               # the python loop
    assert (r.hvps == 0) == case.startswith("dense")                       # Cholesky takes no Hessian-vector product
    _report(f"G2 {case}", r, X.certify(hp, util.spec(hp.n_tokens), r, 1e-8))


# ---- G3: the full-size configurations, trades included ----------------------------------------------------------------
def test_full_size_configs_return_certified_trades():
    """BASELINE.json configs[4] (1M constant-product pools, 4096 tokens; the persistent solver) and configs[2] / [3] (100k
    mixed pools, 1000 tokens; the python loop with smoothed constant-sum trades, pool-feasible by construction)"""
    hp, s = H.cp_host_pools(1_000_000, 4096, seed=3)
    st = _native_store(hp)
    util = cf.Arbitrage(s["prices"])
    r = cf.solve_pools(hp, util, tol=1e-6, store=st)
    assert r.info.history == [] and r.status == "optimal" and len(r.deltas) == 1          # flat trades past 100k pools
    _report("G3 cfg4", r, X.certify(hp, util.spec(4096), r, 1e-6))
    del st
    for seed, name in ((1, "cfg2"), (2, "cfg3")):
        hp, s = H.mixed_host_pools(100_000, 1000, seed=seed)
        if seed == 1:
            util, nu0 = cf.Arbitrage(s["prices"]), None
        else:
            util, nu0 = cf.Liquidate(0, I.synth_basket(1000, s["prices"], seed=2)), s["prices"] / s["prices"][0]
        r = cf.solve_pools(hp, util, nu0=nu0, tol=1e-6)
        assert len(r.info.history) > 0 and r.status == "optimal"
        _report(f"G3 {name}", r, X.certify(hp, util.spec(1000), r, 1e-6))


# ---- G4: the batch solver, a problem per thread and per warp ----------------------------------------------------------
class _Spec:
    def __init__(self, u):
        self.u = u

    def spec(self, n):
        return cf.DualSpec(self.u.c, self.u.a, self.u.eq, self.u.pinned)


def _small_cases():
    rng = np.random.default_rng(41)
    out = []
    for _ in range(6):
        hp, d, prices = H.random_small_problem(rng)
        out += [(hp, _Spec(u)) for u in H.random_utilities(rng, hp.n_tokens, prices)]
    d = I.arbitrage_instance(); out.append((H.host_pools(d), cf.Arbitrage(d["market_value"])))
    d = I.liquidation_instance(); out.append((H.host_pools(d), cf.Liquidate(d["target"], d["current_assets"])))
    d = I.two_asset_instance()
    out += [(H.host_pools(d), cf.Swap(d["tok_in"], d["tok_out"], d["amounts"][j])) for j in (1, 24, 49)]
    return out


@pytest.mark.parametrize("lanes", [1, 32])
def test_batch_solver_certifies_per_thread_and_per_warp(lanes, monkeypatch):
    lib = _lib.load()
    seen = []
    real = lib.cfmm_set_batch_lanes

    def spy(k):
        seen.append(int(k))
        return real(k)
    monkeypatch.setattr(lib, "cfmm_set_batch_lanes", spy)
    monkeypatch.setattr(B, "LANES_SMALL_BATCH", lanes)                 # a one-problem batch runs at this many lanes
    try:
        for k, (hp, util) in enumerate(_small_cases()):
            seen.clear()
            r = cf.solve_pools(hp, util, tol=1e-9, method="thread")
            assert seen == [lanes] and r.info is None                    # the batch kernel, at `lanes` lanes per problem
            assert r.status == "optimal", k
            _report(f"G4 lanes={lanes} #{k}", r, X.certify(hp, util.spec(hp.n_tokens), r, 1e-9))
    finally:
        real(1)


# ---- G5: after an in-place update -------------------------------------------------------------------------------------
def _with(hp, ids, R=None, g=None):
    """a copy of hp with the reserves (CSR rows, one vector per pool) and fees of pools `ids` replaced"""
    res, gam = hp.reserves.copy(), hp.gamma.copy()
    if R is not None:
        u = PL.check_pool_update(hp.pool_ptr, hp.kind, hp.weights, ids, reserves=R)
        res[u.slots] = u.reserves
    if g is not None:
        gam[np.asarray(ids)] = g
    out = cf.HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, res, hp.weights, gam, hp.kind)
    if getattr(hp, "_uniform_product", False):
        out._uniform_product = True
    return out


def test_warm_solve_after_an_in_place_update_certifies_against_the_new_market():
    hp, s = H.cp_host_pools(600_000, 4096, seed=11)
    st = _native_store(hp)
    util = cf.Arbitrage(s["prices"])
    before = cf.solve_pools(hp, util, tol=1e-8, store=st, want_trades=False)
    assert before.status == "optimal"
    rng = np.random.default_rng(12)
    ids = rng.choice(hp.m, hp.m // 100, replace=False)
    R = hp.reserves.reshape(-1, 2)[ids] * np.exp(0.01 * rng.standard_normal((len(ids), 2)))
    g = rng.choice([0.997, 0.998, 0.999, 0.9995], len(ids))
    st.update_pools(ids, reserves=R, fees=g)
    r = cf.solve_pools(hp, util, tol=1e-8, store=st, nu0=before.nu)
    assert r.info.history == [] and r.status == "optimal"
    hp1 = _with(hp, ids, R, g)
    _report("G5 update", r, X.certify(hp1, util.spec(4096), r, 1e-8))
    with pytest.raises(AssertionError, match="not pool-feasible|psi does not match"):
        X.certify(hp, util.spec(4096), r, 1e-8)                          # the trades are the new market's, not the old


# ---- G6: every (trades, hess) instance of the blocked evaluation kernel -----------------------------------------------
@pytest.mark.parametrize("case", ["uniform-4096", "clustered-32768"])
def test_every_blocked_evaluation_instance_matches_the_xp_reference(case):
    """The solver loops call k_blocked with (trades, hess) = (0, 1) and (0, 0), the one-off read-back with (1, 0), the
    oracle parity tests with (1, 1).  psi, arb and hcoef of each against the extended-precision reference.

    Bounds (u = 2^-53).  A flow f = R x takes ~12 roundings of O(1) quantities at prices near the pools' own (p0, p1, their
    product, rsqrt, a, b, 1 - b, the fee factor, R), so |f - f_exact| <= 16 u (R + |f|); summing k_j flows adds k_j u
    gross_j.  Hence |psi_j - psi_xp_j| <= 16 u (Rsum_j + k_j gross_j).  arb sums the nu-weighted flows along a tree: each thread
    chains 4 fma per tile (its 2 pools x 2 flows) over its CTA's tiles, the CTA reduces its threads in < 32 levels, and
    one atomicAdd per CTA with a non-zero sum -- at most one per tile -- chains the CTAs.  Every flow passes at most
    4 T + 32 + T roundings (T = tiles), so |arb - arb_xp| <= 16 u nu'(Rsum + gross) + (5 T + 32) u nu'gross.  hcoef = sqrt(p0 p1 / gamma)/2 takes ~6 roundings:
    16 u of itself; a pool within 1e-12 of its no-trade cone may fall on either side and is left out."""
    if case == "uniform-4096":
        hp, s = H.cp_host_pools(200_000, 4096, seed=19)
    else:
        hp, s = clustered_market(400_000, 32_768, seed=23)
    st = _native_store(hp)
    n, b = hp.n_tokens, st.buckets[0]
    nu = H.random_prices(s["prices"], 7, 0.01)
    ref = X.response(hp, nu)
    psi_x, gross, k = X.flows(hp, ref["delta"], ref["lam"])
    Rsum, = X.token_sums(hp, X.ld(hp.reserves))
    u = X.U64
    b_psi = 16 * u * (Rsum + k * gross)
    nuL = X.ld(nu)
    T = int(b.c_blocked.n_tiles)
    b_arb = 16 * u * (nuL * (Rsum + gross)).sum() + (5 * T + 32) * u * (nuL * gross).sum()
    arb_x = ref["arb"].sum()
    order = b.order.cpu().numpy().astype(np.int64)
    R2 = hp.reserves.reshape(-1, 2)
    p0, p1 = nu[hp.tok_idx[0::2]] * R2[:, 0], nu[hp.tok_idx[1::2]] * R2[:, 1]
    edge = np.minimum(np.abs(np.log(hp.gamma * p1 / p0)), np.abs(np.log(hp.gamma * p0 / p1))) < 1e-12
    worst = {}
    for trades in (False, True):
        for hess in (False, True):
            acc = st.evaluate(torch.as_tensor(nu, **F64), 0.0, trades=trades, hess=hess).cpu().numpy()
            e = np.abs(X.ld(acc[:n]) - psi_x)
            assert np.all(e <= b_psi), (trades, hess, int(np.argmax(e - b_psi)))
            ea = abs(X.ld(acc[n]) - arb_x)
            assert ea <= b_arb, (trades, hess, float(ea), float(b_arb))
            worst[trades, hess] = (float((e / b_psi).max()), float(ea / b_arb))
            if hess:
                h = np.zeros(hp.m); h[order] = b.hcoef[:b.m].cpu().numpy()
                hx = ref["h"]
                ok = ~edge
                assert np.array_equal(h[ok] != 0, hx[ok] != 0), (trades, hess)
                eh = np.abs(X.ld(h[ok]) - hx[ok])
                assert np.all(eh <= 16 * u * hx[ok]), (trades, hess)
                worst[trades, hess] += (float((eh / np.maximum(16 * u * hx[ok], 1e-300)).max()),)
            if trades:
                d, l = st.gather_trades()
                Rrep = np.repeat(np.maximum(R2[:, 0], R2[:, 1]), 2)
                for x, xr in ((d, ref["delta"]), (l, ref["lam"])):
                    assert np.all(np.abs(X.ld(x) - xr) <= 16 * u * (X.ld(Rrep) + np.abs(xr)))
    print(f"CERT G6 {case} edge_pools={int(edge.sum())} worst(psi, arb[, h]) / bound: {worst}")
