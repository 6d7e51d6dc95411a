"""The C++ market loop (cfmm_market_solve, csrc/cfmm_solver.cu): solve_pools(native="hostloop") on stores of every pool
kind, against solver.py and the extended-precision certificates; its dense Cholesky; its C ABI checks."""
import ctypes as C

import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib, instances as I
from cfmm_routing_code_b200.pools import HostPools
import helpers as H
import xp_concentrated as XC
import xp_cryptoswap as XCS
import xp_reference as X
import xp_stableswap as XS
import xp_stableswap_n as XN
import xp_tricrypto as XT

gpu = pytest.mark.gpu


def _torch():
    import torch
    return torch


# ---- the dense factorisation ---------------------------------------------------------------------------------------
def _chol(A):
    """cfmm_dense_cholesky on a symmetric numpy matrix: (L, info)"""
    torch = _torch()
    lib = _lib.load()
    a = torch.as_tensor(np.ascontiguousarray(A), dtype=torch.float64, device="cuda").clone()
    info = torch.full((1,), -1.0, dtype=torch.float64, device="cuda")
    _lib.check(lib.cfmm_dense_cholesky(len(A), a.data_ptr(), info.data_ptr(),
                                       C.c_void_p(torch.cuda.current_stream().cuda_stream)), "cfmm_dense_cholesky")
    torch.cuda.synchronize()
    return np.tril(a.cpu().numpy()), float(info.item())


def _laplacian_plus_shift(n, rng, shift):
    """the solver's kind of matrix: a weighted graph Laplacian (Hs 1 = 0 for every pool) over n tokens with pool weights
    spread over 12 decades, plus a tiny diagonal shift (the damping ladder's first rung)"""
    m = 4 * n
    i, j = rng.integers(0, n, m), rng.integers(0, n, m)
    keep = i != j
    i, j = i[keep], j[keep]
    w = 10.0 ** rng.uniform(-6, 6, len(i))
    L = np.zeros((n, n))
    np.add.at(L, (i, j), -w); np.add.at(L, (j, i), -w)
    np.add.at(L, (i, i), w); np.add.at(L, (j, j), w)
    k = np.arange(n - 1)                      # a chain keeps the graph connected
    L[k, k + 1] -= 1.0; L[k + 1, k] -= 1.0; L[k, k] += 1.0; L[k + 1, k + 1] += 1.0
    return L + shift * np.mean(np.diag(L)) * np.eye(n)


@gpu
@pytest.mark.parametrize("n", [1, 63, 64, 65, 256, 1000, 4096])
def test_cholesky_matches_numpy_on_spd_and_laplacian_matrices(n):
    rng = np.random.default_rng(n)
    B = rng.standard_normal((n, n))
    A = B @ B.T / n + np.eye(n)
    L, info = _chol(A)
    assert info == 0.0
    Ln = np.linalg.cholesky(A)
    assert np.abs(L - Ln).max() <= 1e-12 * np.abs(Ln).max()
    A = _laplacian_plus_shift(n, rng, 1e-8) if n > 1 else np.array([[3e-7]])
    L, info = _chol(A)
    assert info == 0.0
    Ln = np.linalg.cholesky(A)
    # an ill-conditioned matrix: backward error of the factorisation, and the factor against LAPACK's
    assert np.abs(L @ L.T - A).max() <= 1e-13 * np.abs(A).max()
    assert np.abs(L - Ln).max() <= 1e-9 * np.abs(Ln).max()


@gpu
@pytest.mark.parametrize("n", [1, 65, 1000])
def test_cholesky_reports_indefinite_and_nan_matrices(n):
    rng = np.random.default_rng(7)
    B = rng.standard_normal((n, n))
    A = B @ B.T / n + np.eye(n)
    bad = A.copy(); k = n // 2
    bad[k, k] = -1.0 - np.abs(bad[k]).sum()        # indefinite: fails at pivot k + 1 at the latest
    _, info = _chol(bad)
    assert 1 <= info <= k + 1
    for (i, j) in ((n - 1, 0), (k, k)):
        nan = A.copy(); nan[i, j] = np.nan; nan[j, i] = np.nan
        _, info = _chol(nan)
        assert info >= 1, (i, j)
    _, info = _chol(-np.eye(n))
    assert info == 1.0


# ---- every pool kind, every utility --------------------------------------------------------------------------------
def _utilities(n, prices, rng):
    """an Arbitrage near the market prices, a Liquidate of an up-to-8-token basket into token 0, a Swap into token 0"""
    basket = np.zeros(n)
    for j in rng.choice(np.arange(1, n), min(8, n - 1), replace=False):
        basket[j] = float(np.exp(rng.normal(1, 1)) * 100 / prices[j])
    return [cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(n))), cf.Liquidate(0, basket),
            cf.Swap(1, 0, 5.0 / prices[1])]


def _from_dict(s):
    s = dict(s)
    prices = s.pop("prices")
    return HostPools(**s), prices


def _markets():
    """(name, HostPools, prices, xp module) at test sizes"""
    out = []
    for name in ("arbitrage", "liquidation", "two_asset"):
        d = getattr(I, name + "_instance")()
        hp = H.host_pools(d)
        out.append((name, hp, np.ones(hp.n_tokens), X))
    d = I.v3_instance()
    out.append(("v3", H.host_pools(d), np.asarray(d["market_value"], float), X))
    hp, s = H.mixed_host_pools(8000, 150, seed=1)
    out.append(("mixed", hp, s["prices"], X))
    out.append(("stable",) + _from_dict(I.synth_stable_market(6000, 60, seed=1)) + (XS,))
    out.append(("stable_n",) + _from_dict(I.synth_stable_n_market(6000, 60, seed=1)) + (XN,))
    out.append(("concentrated",) + I.synth_concentrated_market(4000, 40, seed=2) + (XC,))
    out.append(("crypto",) + I.synth_crypto_market(6000, 80, seed=3) + (XCS,))
    out.append(("tricrypto",) + I.synth_tricrypto_market(6000, 80, seed=3) + (XT,))
    return out


def _same_value(r, rp, tol=1e-8):
    assert abs(r.value - rp.value) <= tol * max(abs(rp.dual_value), abs(rp.value), 1e-300), (r.value, rp.value)


@gpu
@pytest.mark.parametrize("case", ["arbitrage", "liquidation", "two_asset", "v3", "mixed", "stable", "stable_n",
                                  "concentrated", "crypto", "tricrypto"])
def test_every_pool_kind_and_utility_certifies_through_the_market_loop(case):
    name, hp, prices, xp = next(m for m in _markets() if m[0] == case)
    store = cf.PoolStore(hp)
    rng = np.random.default_rng(5)
    tol = 1e-8
    for u in _utilities(hp.n_tokens, prices, rng):
        r = cf.solve_pools(hp, u, tol=tol, store=store, native="hostloop", method="pools")
        rp = cf.solve_pools(hp, u, tol=tol, store=store, native=False, method="pools")
        assert r.info.history == [] and len(rp.info.history) > 0, case     # the C++ loop, then solver.py
        assert rp.status == "optimal", (case, type(u).__name__, rp.status)
        assert r.status == "optimal", (case, type(u).__name__, r.status, r.iters)
        rep = xp.certify(hp, u.spec(hp.n_tokens), r, tol)
        _same_value(r, rp)
        print(f"CERT {case} {type(u).__name__} iters={r.iters}/{rp.iters} evals={r.evals}/{rp.evals} "
              f"gap={rep['gap'][0]:.2e}")


# ---- both linear solvers on both sides of the switch ---------------------------------------------------------------
@gpu
def test_dense_and_cg_on_both_sides_of_the_switch():
    # constant product + weighted, no constant-sum pools: dense at 256 tokens, CG at 257
    for n, kw in ((256, {}), (257, {}), (257, dict(linear_solver="dense")), (256, dict(linear_solver="cg"))):
        s = I.synth_mixed(6000, n, seed=3, frac_product=0.7, frac_weighted=0.3)
        hp = cf.HostPools(n, s["pool_ptr"], s["tok_idx"], s["reserves"], s["weights"], s["gamma"], s["kind"])
        assert not np.any(hp.kind == 1)
        u = cf.Arbitrage(s["prices"])
        store = cf.PoolStore(hp)
        r = cf.solve_pools(hp, u, tol=1e-8, store=store, native="hostloop", **kw)
        assert r.status == "optimal" and r.info.history == []
        X.certify(hp, u.spec(n), r, 1e-8)
        dense = kw.get("linear_solver", "dense" if n <= 256 else "cg") == "dense"
        assert (r.hvps == 0) == dense, (n, kw, r.hvps)              # CG runs on Hessian-vector products
        _same_value(r, cf.solve_pools(hp, u, tol=1e-8, store=store, native=False, **kw))
    # constant-sum pools at 1000 tokens: auto is dense
    hp, s = H.mixed_host_pools(20_000, 1000, seed=4)
    assert np.any(hp.kind == 1)
    u = cf.Arbitrage(s["prices"])
    store = cf.PoolStore(hp)
    r = cf.solve_pools(hp, u, tol=1e-8, store=store, native="hostloop")
    assert r.status == "optimal" and r.hvps == 0
    X.certify(hp, u.spec(1000), r, 1e-8)
    _same_value(r, cf.solve_pools(hp, u, tol=1e-8, store=store, native=False))
    # forced CG on a constant-sum market: may run out of iterations, never 'optimal' without the certificate
    r = cf.solve_pools(hp, u, tol=1e-8, store=store, native="hostloop", linear_solver="cg", max_iter=30, max_outer=8)
    assert r.info.history == []
    if r.status == "optimal":
        X.certify(hp, u.spec(1000), r, 1e-8)
        assert abs(r.gap) <= 1e-8


@gpu
def test_full_size_mixed_configs_certify():
    """BASELINE configs[2] and [3]: 100k mixed pools over 1000 tokens"""
    hp, s = H.mixed_host_pools(100_000, 1000, seed=1)
    u = cf.Arbitrage(s["prices"])
    r = cf.solve_pools(hp, u, tol=1e-6, native="hostloop")
    assert r.status == "optimal" and r.info.history == []
    X.certify(hp, u.spec(1000), r, 1e-6)
    hp, s = H.mixed_host_pools(100_000, 1000, seed=2)
    u = cf.Liquidate(0, I.synth_basket(1000, s["prices"], seed=2))
    r = cf.solve_pools(hp, u, nu0=s["prices"] / s["prices"][0], tol=1e-6, native="hostloop")
    assert r.status == "optimal" and r.info.history == []
    X.certify(hp, u.spec(1000), r, 1e-6)


@gpu
def test_blocked_bucket_beside_plain_buckets():
    """constant-product pools whose blocked build leaves a residual plain bucket, plus weighted pools: the blocked
    bucket is evaluated by cfmm_blocked_eval inside the loop, the rest by cfmm_arb_eval"""
    n = 16_384                    # uniformly random pairs over this many tokens overflow some tiles' token lists
    s = I.synth_mixed(300_000, n, seed=9, frac_product=0.9, frac_weighted=0.1)
    hp = cf.HostPools(n, s["pool_ptr"], s["tok_idx"], s["reserves"], s["weights"], s["gamma"], s["kind"])
    store = cf.PoolStore(hp)
    assert getattr(store.buckets[0], "blocked", False)
    kinds = [int(b.kind) for b in store.buckets[1:]]
    assert _lib.KIND_GEOMEAN in kinds
    assert len(store.buckets[0].residual) > 0 and _lib.KIND_PRODUCT in kinds
    lib = store.lib
    for u in _utilities(n, s["prices"], np.random.default_rng(2))[:2]:
        lib.cfmm_reset_launch_count()
        r = cf.solve_pools(hp, u, tol=1e-8, store=store, native="hostloop")
        assert r.status == "optimal" and r.info.history == []
        assert lib.cfmm_launch_count() > 0
        X.certify(hp, u.spec(n), r, 1e-8)
        _same_value(r, cf.solve_pools(hp, u, tol=1e-8, store=store, native=False))


@gpu
def test_warm_solve_after_update_pools_certifies_against_a_fresh_store():
    """a new block on a mixed market (StableSwap, weighted, constant-sum, constant-product pools): reserves and fees
    in place, then a warm market-loop solve from the previous prices"""
    from cfmm_routing_code_b200.pools import KIND_STABLESWAP_HOST
    hp, prices = _from_dict(I.synth_stable_market(6000, 60, seed=2))
    store = cf.PoolStore(hp)
    u = cf.Arbitrage(prices)
    r0 = cf.solve_pools(hp, u, tol=1e-8, store=store, native="hostloop")
    assert r0.status == "optimal"
    rng = np.random.default_rng(2)
    ids = np.sort(rng.choice(hp.m, 600, replace=False))
    ar = np.diff(hp.pool_ptr)[ids]
    newR = [hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] * np.exp(0.05 * rng.standard_normal(k)) for i, k in zip(ids, ar)]
    newg = np.where(hp.kind[ids] == KIND_STABLESWAP_HOST, 0.9998, 0.997)
    store.update_pools(ids, reserves=newR, fees=newg)
    R2 = hp.reserves.copy(); g2 = hp.gamma.copy()
    for i, x in zip(ids, newR):
        R2[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] = x
    g2[ids] = newg
    hp2 = HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, R2, hp.weights, g2, hp.kind, hp.amp)
    r1 = cf.solve_pools(hp2, u, nu0=r0.nu, tol=1e-8, store=store, native="hostloop")
    assert r1.status == "optimal" and r1.info.history == []
    XS.certify(hp2, u.spec(hp.n_tokens), r1, 1e-8)
    rf = cf.solve_pools(hp2, u, tol=1e-8, store=cf.PoolStore(hp2), native="hostloop")
    _same_value(r1, rf)


@gpu
def test_infeasible_problem_is_flagged_by_the_market_loop():
    class Need:                                   # psi_1 == +100 with 10 in the only pool; objective: psi_0
        def spec(self, n):
            return cf.DualSpec(np.array([1.0, 0.0]), np.array([0.0, -100.0]), np.array([False, True]),
                               np.array([True, False]))
    hp = cf.HostPools.from_lists(2, [[0, 1]], [[10.0, 10.0]], [0.997], ["product"], [None])
    store = cf.PoolStore(hp, layout="plain")
    r = cf.solve_pools(hp, Need(), store=store, method="pools", native="hostloop", max_iter=60)
    assert r.info.history == [] and r.status == "infeasible"

    class Fine(Need):
        def spec(self, n):
            return cf.DualSpec(np.array([1.0, 0.0]), np.array([0.0, -5.0]), np.array([False, True]),
                               np.array([True, False]))
    r = cf.solve_pools(hp, Fine(), store=store, method="pools", native="hostloop")
    assert r.status == "optimal" and abs(r.psi[1] - 5.0) <= 1e-6 and r.info.history == []


# ---- the C ABI -----------------------------------------------------------------------------------------------------
def _abi_args(store, spec, nu0):
    torch = _torch()
    f64 = dict(dtype=torch.float64, device="cuda")
    n = store.n_tokens
    t = dict(c=torch.as_tensor(spec.c, **f64), a=torch.as_tensor(spec.a, **f64),
             eq=torch.as_tensor(np.asarray(spec.eq, np.uint8), device="cuda"),
             pinned=torch.as_tensor(np.asarray(spec.pinned, np.uint8), device="cuda"),
             nu=torch.as_tensor(nu0, **f64).clone(), psi=torch.empty(n, **f64))
    return t


@gpu
def test_c_abi_solves_a_mixed_store_like_solve_pools():
    torch = _torch()
    hp, s = H.mixed_host_pools(8000, 150, seed=1)
    store = cf.PoolStore(hp)
    lib = store.lib
    u = cf.Arbitrage(s["prices"])
    spec = u.spec(150)
    ref = cf.solve_pools(hp, u, tol=1e-8, store=store, native="hostloop")
    buckets, outs, nb, blk, blk_out = store.market_structs()
    blk_p = C.byref(blk) if blk is not None else None
    nbytes = lib.cfmm_market_solve_work_bytes(buckets, nb, blk_p, 150, 0)
    assert nbytes > 0
    work = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    t = _abi_args(store, spec, cf.solver.default_nu0(spec))
    prm = _lib.MarketParams(1e-8, 1e-12 * float(np.abs(spec.c).max()), 0.1, 1e-4, 0.5, 100, 200, 60, 0)
    res = _lib.SolveResult()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = lambda **o: [o.get(k, v) for k, v in dict(
        b=buckets, o=outs, nb=nb, blk=blk_p, bo=C.byref(blk_out) if blk_out is not None else None, n=150,
        c=t["c"].data_ptr(), a=t["a"].data_ptr(), eq=t["eq"].data_ptr(), pinned=t["pinned"].data_ptr(),
        nu=t["nu"].data_ptr(), psi=t["psi"].data_ptr(), work=work.data_ptr(), prm=C.byref(prm), res=C.byref(res),
        st=st).items()]
    assert lib.cfmm_market_solve(*args()) == 0
    assert res.status == 0
    # the same loop on the same store; the pool kernels accumulate with atomics, so runs agree to rounding only
    np.testing.assert_allclose(t["nu"].cpu().numpy(), ref.nu, rtol=1e-12)
    np.testing.assert_allclose(t["psi"].cpu().numpy(), ref.psi, rtol=0, atol=1e-9 * np.abs(ref.psi).max())
    assert abs(res.primal_value - ref.value) <= 1e-12 * abs(ref.dual_value)
    assert res.iters == ref.iters
    # the documented codes, and nothing launched
    lib.cfmm_reset_launch_count()
    assert lib.cfmm_market_solve(*args(c=None)) == -1
    assert lib.cfmm_market_solve(*args(work=None)) == -1
    assert lib.cfmm_market_solve(*args(o=None)) == -1
    assert lib.cfmm_market_solve(*args(n=0)) == -3
    assert lib.cfmm_market_solve(*args(nb=-1)) == -3
    assert lib.cfmm_market_solve(*args(nb=0, blk=None)) == -3                     # no pools at all
    prm.linear_solver = 1
    assert lib.cfmm_market_solve(*args(n=5000)) == -3                             # forced dense beyond 4096
    prm.linear_solver = 0
    ks = [k for k in range(nb) if buckets[k].kind == _lib.KIND_SUM]
    assert ks
    bad = (_lib.EvalOut * nb)(*[outs[k] for k in range(nb)])
    bad[ks[0]].lambda_ = None
    assert lib.cfmm_market_solve(*args(o=bad)) == -1
    bad[ks[0]].lambda_ = outs[ks[0]].lambda_
    bad[0].hcoef = None
    assert lib.cfmm_market_solve(*args(o=bad)) == -1
    assert lib.cfmm_launch_count() == 0
