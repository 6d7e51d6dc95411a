"""In-place updates of reserves and fees on a resident PoolStore (PoolStore.update_pools, cfmm_blocked_update): a changed
market is re-solved without a rebuild.  The host checks run on the CPU; on the GPU, an updated store must equal, bit for
bit, a store built from the updated data -- blocked slabs, tables and fee records, plain buckets, shards -- evaluate like it
right away, and solve like it."""
import numpy as np
import pytest
import torch

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib
from cfmm_routing_code_b200 import pools as PL
import helpers as H

P = 1024


def _ptr(ar):
    return np.concatenate([[0], np.cumsum(ar)]).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_host_checks_reject_bad_ids_lengths_and_values():
    ptr = _ptr([2, 3, 2, 2])                          # a pair, a 3-token weighted pool, two pairs
    kind = np.zeros(4, np.uint8)
    w = np.full(ptr[-1], 0.5)
    ok = dict(reserves=[[1.0, 2.0], [1.0, 1.0, 1.0]], fees=[0.997, 0.999])
    PL.check_pool_update(ptr, kind, w, [0, 1], **ok)
    for ids, kw in (([0, 0], ok),                                                       # repeated id
                    ([0, 4], ok), ([-1, 1], ok),                                        # out of range
                    ([0, 1], dict(reserves=[[1.0, 2.0], [1.0, 1.0]])),                  # wrong arity
                    ([0, 2], dict(reserves=np.ones((2, 3)))),                           # wrong arity, (n, k) array
                    ([0, 1], dict(fees=[0.997, 1.5])), ([0, 1], dict(fees=[0.0, 0.9])),  # fee outside (0, 1]
                    ([0, 1], dict(fees=[np.nan, 0.9])),
                    ([0, 1], dict(reserves=[[1.0, 0.0], [1.0, 1.0, 1.0]])),             # non-positive reserve
                    ([0, 1], dict(reserves=[[1.0, -2.0], [1.0, 1.0, 1.0]])),
                    ([0, 1], dict(reserves=[[1.0, np.inf], [1.0, 1.0, 1.0]])),
                    ([0, 1], dict(reserves=[[1.0, 2.0], [1.0, np.nan, 1.0]])),
                    ([0, 1], dict(fees=[0.99])),                                        # one fee per pool
                    ([0, 1], {})):                                                      # nothing to update
        with pytest.raises(ValueError):
            PL.check_pool_update(ptr, kind, w, ids, **kw)


def test_host_checks_apply_the_bounded_product_rules_with_the_stores_offsets():
    ptr = _ptr([2, 2])
    kind = np.array([PL.KIND_BOUNDED_HOST, 0], np.uint8)
    w = np.array([0.0, 3.0, 0.5, 0.5])                # pool 0: offsets (0, 3)
    u = PL.check_pool_update(ptr, kind, w, [0], reserves=[[2.0, 0.0]])                  # zero real reserve, virtual 3
    assert u.reserves.tolist() == [2.0, 0.0]
    for R in ([[2.0, -1.0]], [[0.0, 1.0]]):           # negative real reserve; zero virtual reserve (offset 0)
        with pytest.raises(ValueError):
            PL.check_pool_update(ptr, kind, w, [0], reserves=R)
    with pytest.raises(ValueError):                   # pool 1 is a plain pair: zero is not allowed
        PL.check_pool_update(ptr, kind, w, [1], reserves=[[2.0, 0.0]])


def test_host_checks_flatten_reserves_into_csr_slot_order():
    ptr = _ptr([2, 3, 2, 4])
    kind = np.zeros(4, np.uint8)
    w = np.full(ptr[-1], 0.25)
    u = PL.check_pool_update(ptr, kind, w, [3, 0, 1], reserves=[[7, 8, 9, 10], [1, 2], np.array([3.0, 4, 5])],
                             fees=[0.9, 0.99, 0.999])
    assert u.ids.tolist() == [3, 0, 1] and u.ptr.tolist() == [0, 4, 6, 9]
    assert u.slots.tolist() == [7, 8, 9, 10, 0, 1, 2, 3, 4]
    assert u.reserves.tolist() == [7, 8, 9, 10, 1, 2, 3, 4, 5] and u.gamma.tolist() == [0.9, 0.99, 0.999]
    u2 = PL.check_pool_update(ptr, kind, w, [2, 0], reserves=np.array([[5.0, 6.0], [1.0, 2.0]]))
    assert u2.slots.tolist() == [5, 6, 0, 1] and u2.reserves.tolist() == [5, 6, 1, 2] and u2.gamma is None


# ---------------------------------------------------------------------------------------------------------------- GPU
F64 = dict(dtype=torch.float64, device="cuda")


def _bits(x):
    x = x.detach().contiguous().cpu()
    return x.view(torch.int64) if x.dtype == torch.float64 else x.to(torch.int64)


def resident(store):
    """every resident array of every bucket (theta_bar excluded: the solver resets it), as CPU bit patterns; token lists
    and row tables up to each tile's ntok / nrow (the native builder leaves the rest unwritten)"""
    out = {}
    for k, b in enumerate(store.buckets):
        if getattr(b, "blocked", False):
            t = b.tables
            d = t["desc"].cpu().to(torch.int64)
            for name, x in (("r0", b.r0), ("r1", b.r1), ("gamma_inv", b.gamma_inv), ("order", b.order), ("pw", t["pw"]),
                            ("desc", t["desc"]), ("fee", t["fee"])):
                out[k, name] = _bits(x)
            for name, col in (("tok", 0), ("rows", 1)):
                x = _bits(t[name])
                out[k, name] = torch.where(torch.arange(x.shape[1])[None, :] < d[:, col:col + 1], x, 0)
        else:
            for name in ("reserves", "tok_idx", "gamma", "weights", "logrw"):
                x = getattr(b, name)
                if x is not None:
                    out[k, name] = _bits(x)
    return out


def assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


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


def _cp_update(seed=11):
    """600k constant-product pools over 4096 tokens whose tile U streams its slab (20 distinct fees), and an update of 1%
    of the pools: reserves moved by ~1%; fees: a fourth tier on ~2000 pools over many tiles, 14 new distinct fees in tile
    V (3 tiers + 14 = 17: the tile loses its code), tile U's 20 odd fees back to a tier (coded again)"""
    m, n = 600_000, 4096
    hp0, s = H.cp_host_pools(m, n, seed=seed)
    order = cf.PoolStore(hp0).buckets[0].order.cpu().numpy().astype(np.int64)     # the layout depends on tokens only
    U, V = 17, 301
    odd = order[U * P:U * P + 20]
    s["gamma"] = s["gamma"].copy()
    s["gamma"][odd] = 0.99 + 1e-4 * np.arange(20)
    hp = cf.HostPools.from_pairs(n, s["idx"], s["reserves"], s["gamma"])
    rng = np.random.default_rng(seed + 1)
    ids = np.unique(np.concatenate([rng.choice(m, m // 100, replace=False), odd, order[V * P:V * P + 14]]))
    rng.shuffle(ids)
    R = hp.reserves.reshape(-1, 2)[ids] * np.exp(0.01 * rng.standard_normal((len(ids), 2)))
    g = hp.gamma[ids].copy()
    g[rng.random(len(ids)) < 1 / 3] = 0.998                                           # fourth tier
    tierv = np.isin(ids, order[V * P:V * P + 14])
    g[tierv] = 0.98 + 1e-4 * np.arange(14)
    g[np.isin(ids, odd)] = 0.997
    return hp, s, ids, R, g, order, (U, V)


@pytest.mark.gpu
def test_updated_blocked_store_equals_a_fresh_build_bit_for_bit():
    hp, s, ids, R, g, order, (U, V) = _cp_update()
    st = cf.PoolStore(hp)
    b = st.buckets[0]
    assert len(st.buckets) == 1 and b.blocked and b.tables["tok_per_tile"] is None          # the native layout
    nfee0 = b.tables["fee"][:, 0].cpu()
    assert int(nfee0[U]) == 0 and int(nfee0[V]) > 0
    # tiles whose 1/gamma slab changes: their fee records are rebuilt
    pos = np.empty(len(order), np.int64)
    pos[order] = np.arange(len(order))
    changed = (1.0 / g).view(np.int64) != (1.0 / hp.gamma[ids]).view(np.int64)
    touched = len(np.unique(pos[ids[changed]] // P))
    assert touched > 100
    host = (hp.reserves.copy(), hp.gamma.copy())
    rebuilt = st.update_pools(ids, reserves=R, fees=g)
    assert rebuilt == touched
    hp1 = _with(hp, ids, R, g)
    fresh = cf.PoolStore(hp1)
    assert_same(resident(st), resident(fresh))
    nfee = b.tables["fee"][:, 0].cpu()
    assert 0 < int(nfee[U]) <= 16 and int(nfee[V]) == 0 and int((nfee == 0).sum()) == 1  # back to coded / uncoded
    assert np.array_equal(hp.reserves, host[0]) and np.array_equal(hp.gamma, host[1])      # the caller's data is untouched


@pytest.mark.gpu
def test_evaluation_right_after_an_update_sees_the_new_tiles():
    hp, s, ids, R, g, order, _ = _cp_update(seed=12)
    st = cf.PoolStore(hp)
    n = hp.n_tokens
    nu = torch.as_tensor(H.random_prices(s["prices"], 3, spread=0.02), **F64)
    st.evaluate(nu, trades=True, hess=True)                     # tiles of the old data were streamed just before
    st.update_pools(ids, reserves=R, fees=g)
    a1 = st.evaluate(nu, trades=True, hess=True).clone()        # programmatic dependent launch at its default (on)
    fresh = cf.PoolStore(_with(hp, ids, R, g))
    a0 = fresh.evaluate(nu, trades=True, hess=True).clone()
    b1, b0 = st.buckets[0], fresh.buckets[0]
    for x1, x0 in ((b1.delta, b0.delta), (b1.lam, b0.lam), (b1.hcoef, b0.hcoef)):
        assert torch.equal(_bits(x1), _bits(x0))
    scale = float(a0[:n].abs().max())
    assert float((a1[:n] - a0[:n]).abs().max()) <= 1e-15 * scale                           # atomic order only
    assert abs(float(a1[n] - a0[n])) <= 1e-14 * abs(float(a0[n]))


def _mixed_with_residual():
    """H.mixed_host_pools(30_000, 400) plus 1024 constant-product pools on disjoint pairs of 2048 further tokens: the
    blocked bucket is built by the torch builder (mixed kinds), and tiles that would touch too many tokens leave their
    pools in a plain residual bucket"""
    hp0, s = H.mixed_host_pools(30_000, 400, seed=7)
    rng = np.random.default_rng(8)
    nf = 1024
    fr = 400 + np.arange(2 * nf, dtype=np.int32)
    ptr = np.concatenate([hp0.pool_ptr, hp0.pool_ptr[-1] + 2 * np.arange(1, nf + 1)])
    hp = cf.HostPools(400 + 2 * nf, ptr, np.concatenate([hp0.tok_idx, fr]),
                      np.concatenate([hp0.reserves, np.exp(rng.normal(8, 1, 2 * nf))]),
                      np.concatenate([hp0.weights, np.full(2 * nf, 0.5)]),
                      np.concatenate([hp0.gamma, np.full(nf, 0.997)]), np.concatenate([hp0.kind, np.zeros(nf, np.uint8)]))
    prices = np.concatenate([s["prices"], np.exp(rng.normal(0, 1, 2 * nf))])
    return hp, prices


def _random_update(hp, rng, frac):
    """new reserves (one vector per pool, moved ~1%) and fees (a few tiers) of a random fraction of the pools"""
    ids = rng.choice(hp.m, max(1, int(frac * hp.m)), replace=False)
    R = [hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] * np.exp(0.01 * rng.standard_normal(hp.pool_ptr[i + 1] - hp.pool_ptr[i]))
         for i in ids]
    g = rng.choice([0.997, 0.998, 0.999, 0.9995], len(ids))
    return ids, R, g


def _kinds(store):
    return {("blocked" if getattr(b, "blocked", False) else b.kind) for b in store.buckets}


@pytest.mark.gpu
def test_a_rejected_update_leaves_every_bucket_unchanged():
    hp, _ = _mixed_with_residual()
    st = cf.PoolStore(hp)
    before = resident(st)
    rng = np.random.default_rng(1)
    ids, R, g = _random_update(hp, rng, 1000 / hp.m)
    k = 517
    for what in ("negative", "nan", "fee"):
        RR, gg = [r.copy() for r in R], g.copy()
        if what == "negative":
            RR[k][0] = -1.0
        elif what == "nan":
            RR[k][1] = np.nan
        else:
            gg[k] = 1.0 + 1e-12
        with pytest.raises(ValueError):
            st.update_pools(ids, reserves=RR, fees=gg)
        assert_same(resident(st), before)
    # the device check of the blocked bucket, past the host checks: one bad entry, nothing written
    b = next(b for b in st.buckets if getattr(b, "blocked", False))
    pos = np.arange(0, b.m, 7)
    Rb = np.exp(rng.normal(5, 1, (2, len(pos))))
    Rb[1, 40] = -Rb[1, 40]
    with pytest.raises(ValueError):
        b.write_update(st.lib, pos, Rb, np.full(len(pos), 0.99), st._stream())
    with pytest.raises(ValueError):                             # position past the bucket's pools
        b.write_update(st.lib, np.array([0, b.m]), None, np.array([0.99, 0.99]), st._stream())
    assert_same(resident(st), before)


@pytest.mark.gpu
def test_mixed_stores_of_every_bucket_kind_update_like_fresh_builds():
    hp, prices = _mixed_with_residual()
    cases = [(hp, cf.Arbitrage(prices))]
    rng = np.random.default_rng(5)
    while True:                                                  # a small problem with bounded_product pools
        hs, d, ps = H.random_small_problem(rng)
        if np.any(hs.kind == PL.KIND_BOUNDED_HOST) and np.any(hs.kind == PL.KIND_SUM_HOST):
            break
    cases.append((hs, cf.Arbitrage(ps)))
    for hp, util in cases:
        st = cf.PoolStore(hp)
        blocked = [b for b in st.buckets if getattr(b, "blocked", False)]
        assert blocked and blocked[0].tables["tok_per_tile"] is not None                    # the torch builder
        ids, R, g = _random_update(hp, rng, 0.2 if hp.m > 100 else 1.0)
        if hp.m > 100:
            assert len(blocked[0].residual) > 0 and {_lib.KIND_SUM, _lib.KIND_GEOMEAN, _lib.KIND_PRODUCT} <= _kinds(st)
            ids = np.concatenate([ids, [i for i in range(hp.m - 1024, hp.m) if i not in set(ids.tolist())][:50]])
            R += [hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i] + 2] * 1.01 for i in ids[len(R):]]
            g = np.concatenate([g, np.full(len(ids) - len(g), 0.9995)])
        owner = st._pool_map()[0][ids]
        assert len(np.unique(owner)) == len(st.buckets)                                     # every bucket gets pools
        st.update_pools(ids, reserves=R, fees=g)
        hp1 = _with(hp, ids, R, g)
        fresh = cf.PoolStore(hp1)
        assert_same(resident(st), resident(fresh))
        r1 = cf.solve_pools(hp, util, store=st, want_trades=False)
        r0 = cf.solve_pools(hp1, util, store=fresh, want_trades=False)
        assert r1.status == r0.status == "optimal"
        assert abs(r1.value - r0.value) <= 1e-9 * abs(r0.value)


@pytest.mark.gpu
def test_persistent_solve_on_an_updated_store_matches_a_fresh_store_and_the_oracle():
    from oracle import c_oracle as CO
    hp, s, ids, R, g, order, _ = _cp_update(seed=13)
    util = cf.Arbitrage(s["prices"])
    st = cf.PoolStore(hp)
    before = cf.solve_pools(hp, util, tol=1e-8, store=st, want_trades=False)
    assert before.status == "optimal"
    st.update_pools(ids, reserves=R, fees=g)
    hp1 = _with(hp, ids, R, g)
    fresh = cf.PoolStore(hp1)
    ru = cf.solve_pools(hp, util, tol=1e-8, store=st, want_trades=False)
    rf = cf.solve_pools(hp1, util, tol=1e-8, store=fresh, want_trades=False)
    assert ru.info.history == [] and ru.status == rf.status == "optimal"                   # the persistent kernel
    assert (ru.iters, ru.evals, ru.hvps) == (rf.iters, rf.evals, rf.hvps)
    np.testing.assert_allclose(ru.nu, rf.nu, rtol=1e-9)
    nu_o, psi_o, ro = CO.solve_pairs(s["idx"], hp1.reserves.reshape(-1, 2), hp1.gamma, hp.n_tokens, s["prices"], tol=1e-8)
    assert int(ro.status) == 0
    assert abs(ru.value - ro.primal_value) <= 1e-7 * abs(ro.primal_value)
    warm = cf.solve_pools(hp, util, tol=1e-8, store=st, nu0=before.nu, want_trades=False)
    assert warm.status == "optimal"
    assert abs(warm.value - ru.value) <= 1e-7 * abs(ru.value)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_every_shard_takes_its_own_pools_from_the_full_update(world):
    hp, s = H.cp_host_pools(29_000, 1000, seed=4)
    rng = np.random.default_rng(world)
    ids = rng.choice(hp.m, 3000, replace=False)
    R = hp.reserves.reshape(-1, 2)[ids] * np.exp(0.01 * rng.standard_normal((len(ids), 2)))
    g = rng.choice([0.997, 0.998, 0.999, 0.9995], len(ids))
    hp1 = _with(hp, ids, R, g)
    for r in range(world):
        st = cf.PoolStore(hp, rank=r, world=world)
        assert len(st.buckets) == 1 and st.buckets[0].blocked
        lo, hi = (hp.m * r) // world, (hp.m * (r + 1)) // world
        other = (ids < lo) | (ids >= hi)
        before = resident(st)
        st.update_pools(ids[other], reserves=R[other], fees=g[other])                       # nothing of this rank's
        assert_same(resident(st), before)
        st.update_pools(ids, reserves=R, fees=g)
        assert_same(resident(st), resident(cf.PoolStore(hp1, rank=r, world=world)))
