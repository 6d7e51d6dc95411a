"""In-place structural updates of a resident PoolStore: new tick ladders of concentrated pools (mints and burns, T may
change) and new amplifications A and rates of StableSwap pools (PoolStore.update_pools(ladders=, amp=, rates=)).

CPU: check_pool_update rejects every bad entry; the store's host records (LadderSlab, new_ladders) follow a seeded
sequence of mints, burns and price moves bit for bit against HostPools.from_lists, through compactions; D after new A
and rates against from_lists.
GPU (H100): cfmm_ladder_splice against a torch gather; blocks that mix every kind of update leave every bucket tensor
equal to a fresh store of the updated literals (one store and the rank stores of two and three ranks), and the warm
re-solve certified; an invalid entry in a large update changes nothing; C ABI codes.
"""
import ctypes as C

import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib
from cfmm_routing_code_b200.pools import (ANN_MAX, HostPools, KIND_CONCENTRATED_HOST, KIND_STABLESWAP_HOST, LADDER_T_MAX,
                                          LadderSlab, check_pool_update, new_ladders, stableswap_invariant_any)
import xp_concentrated as XC

gpu = pytest.mark.gpu
bits = lambda a: np.ascontiguousarray(a, np.float64).view(np.int64)


def _ladder(rng, p, T, width=0.004):
    """a ladder of T intervals around price p (the price itself may lie past either end)"""
    lo = np.log(p) - width * T * rng.uniform(-0.1, 1.1)
    bounds = np.exp(lo + width * np.arange(T + 1))
    liq = np.exp(rng.normal(6.0, 1.0, T)) * (rng.random(T) >= 0.2)
    liq[rng.integers(0, T)] = 400.0
    return (float(p), bounds, liq)


def _market(rng, n_tokens=12, n_cp=40, n_lad=30, n_ss=(6, 5, 4), n_sum=6, T=(1, 40)):
    """literals of a mixed market: constant product, ladders, 2- to 4-coin StableSwap (with rates), constant sum"""
    prices = np.exp(rng.normal(0, 0.5, n_tokens))
    li, res, fees, kinds, w = [], [], [], [], []
    def pair():
        a = int(rng.integers(0, n_tokens)); b = int((a + rng.integers(1, n_tokens)) % n_tokens)
        return a, b
    for _ in range(n_cp):
        a, b = pair()
        li.append([a, b]); res.append(list(np.exp(rng.normal(5, 0.5)) / prices[[a, b]] * np.exp(rng.normal(0, 0.02, 2))))
        fees.append(0.997); kinds.append("product"); w.append(None)
    for _ in range(n_lad):
        a, b = pair()
        t = int(rng.integers(T[0], T[1] + 1))
        li.append([a, b]); res.append(None); fees.append(0.997); kinds.append("concentrated")
        w.append(_ladder(rng, prices[a] / prices[b] * np.exp(rng.normal(0, 0.02)), t))
    for k, cnt in zip((2, 3, 4), n_ss):
        for _ in range(cnt):
            tk = [int(x) for x in rng.choice(n_tokens, k, replace=False)]
            r = np.exp(rng.normal(0, 0.05, k)) / prices[tk] * prices[tk[0]]
            li.append(tk); res.append(list(np.exp(rng.normal(6, 0.3)) / (r * prices[tk]) * prices[tk[0]]))
            fees.append(0.9996); kinds.append("stableswap"); w.append((float(rng.uniform(20, 200)),) + tuple(r))
    for _ in range(n_sum):
        a, b = pair()
        li.append([a, b]); res.append(list(np.exp(rng.normal(4, 0.3)) / prices[[a, b]])); fees.append(0.999)
        kinds.append("sum"); w.append(None)
    return dict(n=n_tokens, li=li, res=res, fees=fees, kinds=kinds, w=w), prices


def _hp(d):
    return HostPools.from_lists(d["n"], d["li"], d["res"], d["fees"], d["kinds"], d["w"])


# -- host checks ------------------------------------------------------------------------------------------------------
def _bad_updates(d, hp):
    cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    ss = np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0]
    ar = np.diff(hp.pool_ptr)
    s3 = ss[ar[ss] == 3][0]
    s2 = ss[ar[ss] == 2][0]
    good = d["w"][cl[0]]
    p, b, L = good
    cp = 0
    return [
        ("ladders on a product pool", [cp], dict(ladders=[good])),
        ("ladders with prices", [cl[0]], dict(ladders=[good], prices=[1.0])),
        ("unsorted bounds", [cl[0]], dict(ladders=[(p, b[::-1], L)])),
        ("equal bounds", [cl[0]], dict(ladders=[(p, np.r_[b[0], b[0], b[2:]], L)] if len(b) > 2 else [(p, [1.0, 1.0], [1.0])])),
        ("all-zero liquidity", [cl[0]], dict(ladders=[(p, b, np.zeros_like(L))])),
        ("negative liquidity", [cl[0]], dict(ladders=[(p, b, np.r_[-1.0, L[1:]])])),
        ("too many intervals", [cl[0]], dict(ladders=[(1.0, np.linspace(1.0, 2.0, LADDER_T_MAX + 2),
                                                         np.ones(LADDER_T_MAX + 1))])),
        ("nan price", [cl[0]], dict(ladders=[(np.nan, b, L)])),
        ("inf bound", [cl[0]], dict(ladders=[(p, np.r_[b[:-1], np.inf], L)])),
        ("nan liquidity", [cl[0]], dict(ladders=[(p, b, np.r_[np.nan, L[1:]])])),
        ("not a triple", [cl[0]], dict(ladders=[(p, b)])),
        ("one ladder for two pools", cl[:2].tolist(), dict(ladders=[good])),
        ("amp on a ladder", [cl[0]], dict(amp=[10.0])),
        ("rates on a product pool", [cp], dict(rates=[[1.0, 1.0]])),
        ("wrong rate count", [s3], dict(rates=[[1.0, 1.0]])),
        ("A n^n over the limit", [s3], dict(amp=[ANN_MAX / 27 * 1.01])),
        ("A <= 0", [s2], dict(amp=[0.0])),
        ("zero rate", [s3], dict(rates=[[1.0, 0.0, 1.0]])),
        ("negative rate", [s2], dict(rates=[[1.0, -2.0]])),
        ("nan rate", [s3], dict(rates=[[1.0, np.nan, 1.0]])),
        ("nan A", [s2], dict(amp=[np.nan])),
        ("repeated id", [cl[0], cl[0]], dict(ladders=[good, good])),
        ("id out of range", [hp.m], dict(amp=[10.0])),
        ("negative id", [-1], dict(amp=[10.0])),
    ]


def test_check_rejects_bad_structural_updates():
    d, _ = _market(np.random.default_rng(0))
    hp = _hp(d)
    for what, ids, kw in _bad_updates(d, hp):
        with pytest.raises(ValueError):
            check_pool_update(hp.pool_ptr, hp.kind, hp.weights, ids, **kw)
            pytest.fail(what)
    cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    ss = np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0]
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, cl[:3], ladders=[d["w"][i] for i in cl[:3]], fees=[0.99] * 3)
    assert len(u.ladders) == 3 and u.gamma is not None
    ar = np.diff(hp.pool_ptr)[ss]
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, ss, amp=np.full(len(ss), 50.0),
                          rates=[np.ones(k) for k in ar])
    assert len(u.rates) == ar.sum()


# -- host state -------------------------------------------------------------------------------------------------------
def _host_pool_state(hp, i):
    r = hp.lad_rec[hp.lad_ptr[i]:hp.lad_ptr[i + 1]]
    return r, hp.lad_sc[i], hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i] + 2]


def test_ladder_slab_follows_mints_and_burns_bit_for_bit():
    rng = np.random.default_rng(5)
    d, prices = _market(rng, n_cp=4, n_lad=8, n_ss=(2, 1, 1), n_sum=1, T=(1, 12))
    hp = _hp(d)
    cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    slab = LadderSlab(hp.lad_ptr, hp.lad_rec)
    sc = {i: hp.lad_sc[i] for i in cl}
    res = {i: hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i] + 2] for i in cl}
    compactions = 0
    # T of pool cl[0] goes 1 -> 4096 -> 1; the others grow, shrink or keep T, with prices past either end
    path0 = [1, 4096, 4096, 1, 2, 1]
    for step in range(24):
        k = int(rng.integers(1, len(cl) + 1))
        ids = np.sort(rng.choice(cl, k, replace=False))
        if step < len(path0) and cl[0] not in ids:
            ids = np.sort(np.r_[ids, cl[0]])
        if step % 4 == 3:                                       # a price move only
            p = np.array([d["w"][i][0] for i in ids]) * np.exp(rng.normal(0, 0.3, len(ids)))
            p[0] = 1e-30 if step % 8 == 3 else 1e30
            s, c, x, y = slab.state(ids, p)
            for j, i in enumerate(ids.tolist()):
                d["w"][i] = (float(p[j]), d["w"][i][1], d["w"][i][2])
                sc[i], res[i] = np.array([s[j], c[j]]), np.array([x[j], y[j]])
        else:
            lads = []
            for i in ids.tolist():
                T0 = len(d["w"][i][2])
                if i == cl[0] and step < len(path0):
                    T = path0[step]
                else:
                    T = int(np.clip(T0 + rng.integers(-3, 4), 1, 40))
                lads.append(_ladder(rng, d["w"][i][0] * np.exp(rng.normal(0, 0.5)), T))
            u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, ids, ladders=lads)
            rec, cnt, s, c, x, y = new_ladders(u.ladders)
            before = len(slab.base)
            slab.replace(ids, rec, cnt)
            compactions += int(before > 0 and len(slab.base) == 0) + int(before == 0 and slab.dead == 0)
            for j, i in enumerate(ids.tolist()):
                d["w"][i] = lads[j]
                sc[i], res[i] = np.array([s[j], c[j]]), np.array([x[j], y[j]])
        assert slab.dead <= slab.live
        ref = _hp(d)
        for i in cl.tolist():
            r, sc_ref, res_ref = _host_pool_state(ref, i)
            assert np.array_equal(bits(slab.records(i)), bits(r)), (step, i)
            assert np.array_equal(bits(sc[i]), bits(sc_ref)) and np.array_equal(bits(res[i]), bits(res_ref)), (step, i)
        # a price-only update after the step reads the slab's records: the same bits as the fresh HostPools
        p = np.array([d["w"][i][0] for i in cl]) * np.exp(rng.normal(0, 0.1, len(cl)))
        s, c, x, y = slab.state(cl, p)
        ref2 = _hp(dict(d, w=[(float(p[list(cl).index(i)]),) + tuple(w[1:]) if i in cl else w
                              for i, w in enumerate(d["w"])]))
        assert np.array_equal(bits(np.stack([s, c], 1)), bits(ref2.lad_sc[cl]))
    assert len(slab.records(cl[0])) == len(d["w"][cl[0]][2]) + 1
    assert compactions >= 2


def test_invariant_after_new_amp_and_rates():
    rng = np.random.default_rng(8)
    d, _ = _market(rng)
    hp = _hp(d)
    ss = np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0]
    ids = np.sort(rng.choice(ss, 9, replace=False))
    ar = np.diff(hp.pool_ptr)[ids]
    A = rng.uniform(5, 400, len(ids))
    rates = [np.exp(rng.normal(0, 0.1, k)) for k in ar]
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, ids, amp=A, rates=rates)
    for i, j in enumerate(ids.tolist()):
        d["w"][j] = (float(A[i]),) + tuple(rates[i])
    ref = _hp(d)
    for k in np.unique(ar).tolist():
        e = np.nonzero(ar == k)[0]
        rs = u.ptr[e][:, None] + np.arange(k)
        R = hp.reserves[u.slots[rs]]
        D = stableswap_invariant_any(R, u.rates[rs], u.amp[e])           # as PoolStore.update_pools forms it
        assert np.array_equal(bits(D), bits(ref.inv[ids[e]]))


# -- GPU --------------------------------------------------------------------------------------------------------------
def _splice(lib, bucket, pos, cnt, rec, state, out, work=None):
    import torch
    dev = "cuda"
    pos_t = torch.as_tensor(np.asarray(pos, np.int64), device=dev)
    cnt_t = torch.as_tensor(np.asarray(cnt, np.int64), device=dev)
    rec_t = torch.as_tensor(np.ascontiguousarray(rec, np.float64), device=dev)
    st_t = torch.as_tensor(np.ascontiguousarray(state, np.float64), device=dev)
    nb = lib.cfmm_ladder_splice_work_bytes(bucket.n_pools, len(pos))
    w = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
    status = (C.c_int64 * 2)()
    rc = lib.cfmm_ladder_splice(C.byref(bucket), len(pos), pos_t.data_ptr(), cnt_t.data_ptr(), rec_t.data_ptr(),
                                len(rec), st_t.data_ptr(), out.data_ptr(), out.numel() // 4, status, w.data_ptr(), nb, None)
    return rc, status[0], status[1]


def _splice_bucket(rng, counts, stride=None):
    """a concentrated bucket of pools with the given record counts (records: random payload), on the device"""
    import torch
    m = len(counts)
    stride = stride or max(1024, -(-m // 1024) * 1024)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]])
    rec = torch.as_tensor(rng.standard_normal((int(np.sum(counts)), 4)), device="cuda").reshape(-1)
    logrw = torch.zeros((4, stride), dtype=torch.float64, device="cuda")
    logrw[2, :m] = torch.as_tensor(first.astype(float)); logrw[3, :m] = torch.as_tensor(np.asarray(counts, float) - 1)
    logrw[0, :m] = torch.as_tensor(rng.standard_normal(m)); logrw[1, :m] = 7.0
    R = torch.as_tensor(rng.standard_normal((2, stride)), device="cuda")
    tok = torch.zeros((2, stride), dtype=torch.int32, device="cuda")
    g = torch.ones(stride, dtype=torch.float64, device="cuda")
    b = _lib.Bucket(_lib.KIND_CONCENTRATED, 2, m, stride, R.data_ptr(), tok.data_ptr(), g.data_ptr(), rec.data_ptr(),
                    logrw.data_ptr(), None)
    return b, dict(rec=rec, logrw=logrw, R=R, keep=(tok, g))


def _gather_reference(t, counts, pos, cnt, newrec):
    """the spliced records by a torch repeat_interleave gather over [old records | new records]"""
    import torch
    old = t["rec"].view(-1, 4)
    allrec = torch.cat([old, torch.as_tensor(newrec, device="cuda").view(-1, 4)])
    c = torch.as_tensor(np.asarray(counts, np.int64), device="cuda").clone()
    src = torch.as_tensor(np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64), device="cuda")
    if len(pos):
        p = torch.as_tensor(np.asarray(pos, np.int64), device="cuda")
        c[p] = torch.as_tensor(np.asarray(cnt, np.int64), device="cuda")
        src[p] = old.shape[0] + torch.as_tensor(np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64), device="cuda")
    first = torch.cumsum(c, 0) - c
    idx = torch.repeat_interleave(src - first, c) + torch.arange(int(c.sum()), device="cuda")
    return allrec[idx], first, c


@gpu
def test_splice_kernel_matches_a_gather():
    import torch
    lib = _lib.load()
    rng = np.random.default_rng(11)
    cases = []
    counts = rng.integers(2, 70, 5000)
    cases.append((counts, np.sort(rng.choice(5000, 700, replace=False)), None))            # counts change
    cases.append((counts, np.sort(rng.choice(5000, 300, replace=False)), "same"))          # no count changes
    cases.append((counts, np.zeros(0, np.int64), None))                                    # nothing changes
    big = rng.integers(2, 5, 3000); big[1234] = 2 ** 20 + 1                                # one pool of 2^20 intervals
    cases.append((big, np.array([3, 1234, 2999]), None))
    cases.append((big, np.array([1234]), "small"))                                         # 2^20 -> 1 interval
    for counts, pos, how in cases:
        b, t = _splice_bucket(rng, counts)
        cnt = (counts[pos] if how == "same" else np.full(len(pos), 2) if how == "small"
               else rng.integers(2, 90, len(pos)))
        newrec = rng.standard_normal((int(cnt.sum()), 4))
        state = rng.standard_normal((len(pos), 4))
        ref, first, c = _gather_reference(t, counts, pos, cnt, newrec)
        out = torch.full((4 * (ref.shape[0] + 17),), np.nan, dtype=torch.float64, device="cuda")
        lr0, R0 = t["logrw"].clone(), t["R"].clone()
        rc, bad, total = _splice(lib, b, pos, cnt, newrec, state, out)
        assert rc == 0 and bad == 0 and total == ref.shape[0]
        assert torch.equal(out[:4 * total].view(-1, 4), ref)
        assert torch.isnan(out[4 * total:]).all()                                          # nothing past the total
        m = len(counts)
        assert torch.equal(t["logrw"][2, :m], first.double()) and torch.equal(t["logrw"][3, :m], (c - 1).double())
        keep = np.setdiff1d(np.arange(m), pos)
        kp = torch.as_tensor(keep, device="cuda")
        assert torch.equal(t["logrw"][:2, kp], lr0[:2, kp]) and torch.equal(t["R"][:, kp], R0[:, kp])
        assert torch.equal(t["logrw"][:, m:], lr0[:, m:]) and torch.equal(t["R"][:, m:], R0[:, m:])
        if len(pos):
            pp = torch.as_tensor(pos, device="cuda")
            st = torch.as_tensor(state, device="cuda")
            assert torch.equal(t["logrw"][0, pp], st[:, 0]) and torch.equal(t["logrw"][1, pp], st[:, 1])
            assert torch.equal(t["R"][0, pp], st[:, 2]) and torch.equal(t["R"][1, pp], st[:, 3])


@gpu
def test_splice_c_abi_codes_and_rejections():
    import torch
    lib = _lib.load()
    rng = np.random.default_rng(12)
    counts = rng.integers(2, 9, 100)
    b, t = _splice_bucket(rng, counts)
    out = torch.zeros(4 * 2000, dtype=torch.float64, device="cuda")
    rec = rng.standard_normal((3, 4)); st = np.zeros((1, 4))
    status = (C.c_int64 * 2)()
    work = torch.empty(lib.cfmm_ladder_splice_work_bytes(100, 1), dtype=torch.uint8, device="cuda")
    nb = work.numel()
    pos = torch.as_tensor([5], device="cuda"); cnt = torch.as_tensor([3], device="cuda")
    recd, std = torch.as_tensor(rec, device="cuda"), torch.as_tensor(st, device="cuda")

    def call(bk, p=pos, n=cnt, r=recd, s=std, o=out, w=work, wb=nb, sh=status, n_chg=1, n_records=3):
        return lib.cfmm_ladder_splice(C.byref(bk) if bk is not None else None, n_chg,
                                      p.data_ptr() if p is not None else None, n.data_ptr() if n is not None else None,
                                      r.data_ptr() if r is not None else None, n_records,
                                      s.data_ptr() if s is not None else None, o.data_ptr() if o is not None else None,
                                      2000, sh, w.data_ptr() if w is not None else None, wb, None)
    assert call(None) == -1
    assert call(b, p=None) == -1 and call(b, n=None) == -1 and call(b, r=None) == -1 and call(b, s=None) == -1
    assert call(b, o=None) == -1 and call(b, w=None) == -1
    for kind, arity in ((_lib.KIND_BOUNDED, 2), (_lib.KIND_STABLESWAP_N, 3), (_lib.KIND_CONCENTRATED, 3)):
        bk = _lib.Bucket(kind, arity, b.n_pools, b.stride, b.reserves, b.tok_idx, b.gamma, b.weights, b.logrw, None)
        assert call(bk) == -2
    nw = _lib.Bucket(*[getattr(b, f) for f, _ in _lib.Bucket._fields_]); nw.weights = None
    assert call(nw) == -1
    assert call(b, n_chg=101) == -3 and call(b, n_chg=-1) == -3 and call(b, wb=nb - 1) == -3
    assert lib.cfmm_ladder_splice_work_bytes(10, 11) == -3
    # entries the device rejects: nothing is written, status[0] counts them
    lr0, R0 = t["logrw"].clone(), t["R"].clone()
    out.fill_(-5.0)
    for p_, n_, nrec in (([100], [3], 3), ([5], [1], 1), ([5], [3], 4), ([5], [2 ** 20 + 2], 2 ** 20 + 2)):
        r_ = torch.zeros((max(nrec, 1), 4), dtype=torch.float64, device="cuda")
        rc = call(b, p=torch.as_tensor(p_, device="cuda"), n=torch.as_tensor(n_, device="cuda"), r=r_, n_records=nrec)
        assert rc == 0 and status[0] > 0, (p_, n_)
    w2 = torch.empty(lib.cfmm_ladder_splice_work_bytes(100, 2), dtype=torch.uint8, device="cuda")
    rc = call(b, p=torch.as_tensor([7, 5], device="cuda"), n=torch.as_tensor([2, 2], device="cuda"),
              r=torch.zeros((4, 4), dtype=torch.float64, device="cuda"), s=torch.zeros((2, 4), dtype=torch.float64,
                                                                                      device="cuda"),
              w=w2, wb=w2.numel(), n_chg=2, n_records=4)
    assert rc == 0 and status[0] > 0                                                       # positions out of order
    small = torch.zeros(4 * 10, dtype=torch.float64, device="cuda")
    rc = lib.cfmm_ladder_splice(C.byref(b), 0, None, None, None, 0, None, small.data_ptr(), 10, status, work.data_ptr(),
                                nb, None)
    assert rc == 0 and status[0] > 0                                                       # the output is too small
    assert torch.equal(t["logrw"], lr0) and torch.equal(t["R"], R0) and bool((out == -5.0).all())
    assert bool((small == 0).all())
    torch.cuda.synchronize()


def _bucket_tensors(store):
    out = []
    for b in store.buckets:
        if getattr(b, "blocked", False):
            out.append(("blocked",) + tuple(getattr(b, n).clone() for n in ("r0", "r1", "gamma_inv")))
            continue
        out.append((int(b.kind), int(b.arity)) + tuple(None if getattr(b, n) is None else getattr(b, n).clone()
                                                       for n in ("reserves", "gamma", "weights", "logrw")))
    return out


def _assert_equal_tensors(xa, xb, what):
    import torch
    assert len(xa) == len(xb), what
    for a, b in zip(xa, xb):
        assert a[:2] == b[:2] if a[0] != "blocked" else a[0] == b[0], what
        for x, y in zip(a[2:] if a[0] != "blocked" else a[1:], b[2:] if b[0] != "blocked" else b[1:]):
            assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), (what, a[:2])


def _block(rng, d, hp, prices, big=False):
    """one block of mixed updates of the literals d (returned as update_pools calls; d is updated in place)"""
    cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    ss = np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0]
    cp = np.nonzero(np.array([k == "product" for k in d["kinds"]]))[0]
    calls = []
    ids = np.sort(rng.choice(cl, len(cl) // 3, replace=False))            # mints and burns, T changes for some
    lads, g = [], []
    for i in ids.tolist():
        T0 = len(d["w"][i][2])
        T = T0 if rng.random() < 0.4 else int(np.clip(T0 + rng.integers(-5, 6), 1, 60))
        lads.append(_ladder(rng, d["w"][i][0] * np.exp(rng.normal(0, 0.01)), T))
    g = np.where(rng.random(len(ids)) < 0.3, 0.9995, 0.997)
    calls.append(dict(pool_ids=ids, ladders=lads, fees=g))
    rest = np.setdiff1d(cl, ids)                                         # other ladders move price
    pm = np.sort(rng.choice(rest, len(rest) // 2, replace=False))
    newp = np.array([d["w"][i][0] for i in pm]) * np.exp(rng.normal(0, 0.01, len(pm)))
    calls.append(dict(pool_ids=pm, prices=newp))
    sr = np.sort(rng.choice(ss, len(ss) // 2, replace=False))           # new rates; a few a ramp step of A with reserves
    ar = np.diff(hp.pool_ptr)[sr]
    rates = [np.asarray(d["w"][i][1:]) * np.exp(rng.normal(0, 0.002, k)) for i, k in zip(sr.tolist(), ar)]
    calls.append(dict(pool_ids=sr, rates=rates))
    sa = np.setdiff1d(ss, sr)[:3]
    A = np.array([d["w"][i][0] for i in sa]) * 1.01
    R = [np.asarray(d["res"][i]) * np.exp(rng.normal(0, 0.01, len(d["res"][i]))) for i in sa]
    calls.append(dict(pool_ids=sa, amp=A, reserves=R))
    sb = np.setdiff1d(ss, np.r_[sr, sa])[:3]                             # later reserves= on pools with new A and rates
    if len(sb):
        R2 = [np.asarray(d["res"][i]) * np.exp(rng.normal(0, 0.01, len(d["res"][i]))) for i in sb]
        calls.append(dict(pool_ids=sb, reserves=R2, fees=np.full(len(sb), 0.9993)))
    pc = cp[:10]                                                         # constant product pools, reserves and fees
    calls.append(dict(pool_ids=pc, reserves=np.array([d["res"][i] for i in pc]) * 1.003, fees=np.full(len(pc), 0.996)))
    # the literals after the block
    for c in calls:
        for k, i in enumerate(np.asarray(c["pool_ids"]).tolist()):
            w = d["w"][i]
            if "ladders" in c:
                d["w"][i] = c["ladders"][k]
            if "prices" in c:
                d["w"][i] = (float(c["prices"][k]), w[1], w[2])
            if "rates" in c:
                d["w"][i] = (d["w"][i][0],) + tuple(c["rates"][k])
            if "amp" in c:
                d["w"][i] = (float(c["amp"][k]),) + tuple(d["w"][i][1:])
            if "reserves" in c:
                d["res"][i] = list(np.asarray(c["reserves"][k], float))
            if "fees" in c:
                d["fees"][i] = float(c["fees"][k])
    return calls


@gpu
@pytest.mark.parametrize("world", [1, 2, 3])
def test_blocks_of_structural_updates_equal_a_fresh_store(world):
    rng = np.random.default_rng(20 + world)
    d, prices = _market(rng, n_tokens=16, n_cp=1500, n_lad=240, n_ss=(30, 24, 18), n_sum=30, T=(1, 50))
    hp = _hp(d)
    stores = [cf.PoolStore(hp, rank=r, world=world) for r in range(world)]
    u = cf.Arbitrage(prices)
    prev = cf.solve_pools(hp, u, tol=1e-8, store=stores[0]) if world == 1 else None
    for blk in range(4):
        calls = _block(rng, d, hp, prices)
        for c in calls:
            for st in stores:
                st.update_pools(**c)
        hp2 = _hp(d)
        for r, st in enumerate(stores):
            _assert_equal_tensors(_bucket_tensors(st), _bucket_tensors(cf.PoolStore(hp2, rank=r, world=world)),
                                  (world, blk, r))
        if world == 1:
            res = cf.solve_pools(hp2, u, tol=1e-8, store=stores[0], nu0=prev.nu)
            assert res.status == "optimal"
            XC.certify(hp2, u.spec(hp.n_tokens), res, 1e-8)
            cold = cf.solve_pools(hp2, u, tol=1e-8, store=cf.PoolStore(hp2))
            assert abs(res.value - cold.value) <= 20 * 1e-8 * max(abs(cold.dual_value), 1e-300), (res.value, cold.value)
            prev = res
    # the caller's HostPools was not modified
    ref = _hp(_market(np.random.default_rng(20 + world), n_tokens=16, n_cp=1500, n_lad=240, n_ss=(30, 24, 18),
                      n_sum=30, T=(1, 50))[0])
    for f in ("reserves", "weights", "gamma", "amp", "inv", "lad_ptr", "lad_rec", "lad_sc"):
        assert np.array_equal(bits(getattr(hp, f)), bits(getattr(ref, f))), f


@gpu
def test_an_invalid_entry_changes_nothing():
    rng = np.random.default_rng(31)
    d, prices = _market(rng, n_tokens=16, n_cp=1500, n_lad=400, n_ss=(40, 30, 20), n_sum=30, T=(1, 50))
    hp = _hp(d)
    store = cf.PoolStore(hp)
    u = cf.Arbitrage(prices)
    for c in _block(rng, d, hp, prices):                                 # a structural update first: own host state
        store.update_pools(**c)
    hp2 = _hp(d)
    r0 = cf.solve_pools(hp2, u, tol=1e-8, store=store)
    cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    ss = np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0]
    ar = np.diff(hp.pool_ptr)[ss]
    before = _bucket_tensors(store)
    slab = store._ladders()
    host = (slab.first.copy(), slab.T.copy(), slab.n_own, slab.live, slab.dead, store._weights_host.copy(),
            store._amp_host.copy())
    lads = [_ladder(rng, d["w"][i][0], int(rng.integers(1, 80))) for i in cl]
    bad_lads = list(lads); bad_lads[-1] = (lads[-1][0], lads[-1][1], -lads[-1][2])
    rates = [np.ones(k) * 1.01 for k in ar]
    bad_rates = list(rates); bad_rates[-1] = np.r_[rates[-1][:-1], 0.0]
    for kw in (dict(pool_ids=cl, ladders=bad_lads, fees=np.full(len(cl), 0.99)),
               dict(pool_ids=ss, rates=bad_rates, amp=np.full(len(ss), 30.0)),
               dict(pool_ids=ss, amp=np.r_[np.full(len(ss) - 1, 30.0), ANN_MAX]),
               dict(pool_ids=np.r_[cl, 0], ladders=lads + [lads[0]])):
        with pytest.raises(ValueError):
            store.update_pools(**kw)
        _assert_equal_tensors(_bucket_tensors(store), before, str(kw.keys()))
        assert np.array_equal(slab.first, host[0]) and np.array_equal(slab.T, host[1])
        assert (slab.n_own, slab.live, slab.dead) == host[2:5]
        assert np.array_equal(store._weights_host, host[5]) and np.array_equal(store._amp_host, host[6])
    r1 = cf.solve_pools(hp2, u, tol=1e-8, store=store)
    assert r1.value == r0.value and np.array_equal(r1.nu, r0.nu)
