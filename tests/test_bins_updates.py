"""In-place updates of price-bin pools on a resident PoolStore: a pool's whole new (prices, x, y) after a Liquidity Book
swap, a deposit or withdrawal, a changed order book or a filled limit order (PoolStore.update_pools(bins=); K may
change).

CPU: check_pool_update(bins=) rejects every bad entry; the store's host records (a LadderSlab over bin_rec, new_bins)
follow a seeded sequence of replacements bit for bit against HostPools built with the replaced pools' bin_records,
through compactions.
GPU (H100): cfmm_bins_splice against a torch gather, its C ABI codes and rejections; blocks of bins=, fees=, ladders=,
prices= and reserves= updates leave every bucket tensor equal to a fresh store (one store and the rank stores of two and
three ranks) and the warm re-solve certified on both loops; PoolStore.bin_fills after updates; an invalid entry in a
large update changes nothing.
"""
import ctypes as C

import numpy as np
import pytest

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib, instances as I
from cfmm_routing_code_b200.pools import (BINS_K_MAX, HostPools, KIND_BINS_HOST, KIND_CONCENTRATED_HOST, LadderSlab,
                                          bin_fills, bin_records, check_pool_update, new_bins)
import xp_bins as XB

gpu = pytest.mark.gpu
bits = lambda a: np.ascontiguousarray(a, np.float64).view(np.int64)
EVENTS = ("swap", "deposit", "withdraw", "book", "fill")


def _triple(hp, i):
    """(prices, x, y) of bins pool i read back from its records (the active bin's two segments merged)"""
    p, x, y = (np.asarray(v, np.float64) for v in XB.bins_of(hp, i))
    pr, inv = np.unique(p, return_inverse=True)
    return pr, np.bincount(inv, x, len(pr)), np.bincount(inv, y, len(pr))


def _with_bins(hp, new):
    """hp with the bins pools of `new` (pool -> bin_records) replaced: records, (z, p_ref) and reserves"""
    bn = np.nonzero(hp.kind == KIND_BINS_HOST)[0]
    bp = np.asarray(hp.bin_ptr, np.int64)
    recs, zp, R = [], np.array(hp.bin_zp, np.float64), np.array(hp.reserves, np.float64)
    for i in bn.tolist():
        if i in new:
            r, z, pref, sums = new[i]
            recs.append(r); zp[i] = (z, pref); R[hp.pool_ptr[i]:hp.pool_ptr[i] + 2] = sums
        else:
            recs.append(hp.bin_rec[bp[i]:bp[i + 1]])
    cnt = np.zeros(hp.m, np.int64); cnt[bn] = [len(r) for r in recs]
    ptr = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    return HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, R, hp.weights, hp.gamma, hp.kind, hp.amp, hp.inv, hp.lad_ptr,
                     hp.lad_rec, hp.lad_sc, hp.cgam, ptr, np.concatenate(recs), zp)


def _ladder(rng, p, T, width=0.004):
    lo = np.log(p) - width * T * rng.uniform(-0.1, 1.1)
    bounds = np.exp(lo + width * np.arange(T + 1))
    liq = np.exp(rng.normal(6.0, 1.0, T)) * (rng.random(T) >= 0.2)
    liq[rng.integers(0, T)] = 400.0
    return (float(p), bounds, liq)


def _market(rng, n_tokens=16, n_cp=600, n_lad=80, n_bins=200, K=(1, 16)):
    """literals of a market of constant-product pools, ladders and bins pools (Liquidity Book bins, order books, limit
    orders: the shapes of instances.synth_bins_market)"""
    hb, prices = I.synth_bins_market(n_cp + n_bins, n_tokens, int(rng.integers(1 << 30)), K=K,
                                     frac_lb=0.6 * n_bins / (n_cp + n_bins), frac_book=0.2 * n_bins / (n_cp + n_bins),
                                     frac_order=0.2 * n_bins / (n_cp + n_bins))
    li, res, fees, kinds, w = [], [], [], [], []
    for i in range(hb.m):
        t = hb.tok_idx[hb.pool_ptr[i]:hb.pool_ptr[i] + 2].tolist()
        li.append(t); fees.append(float(hb.gamma[i]))
        if hb.kind[i] == KIND_BINS_HOST:
            res.append(None); kinds.append("bins"); w.append(_triple(hb, i))
        else:
            res.append(hb.reserves[hb.pool_ptr[i]:hb.pool_ptr[i] + 2].tolist()); kinds.append("product"); w.append(None)
    for _ in range(n_lad):
        a = int(rng.integers(0, n_tokens)); b = int((a + rng.integers(1, n_tokens)) % n_tokens)
        li.append([a, b]); res.append(None); fees.append(0.997); kinds.append("concentrated")
        w.append(_ladder(rng, prices[a] / prices[b] * np.exp(rng.normal(0, 0.02)), int(rng.integers(1, 30))))
    return dict(n=n_tokens, li=li, res=res, fees=fees, kinds=kinds, w=w), prices


def _hp(d):
    return HostPools.from_lists(d["n"], d["li"], d["res"], d["fees"], d["kinds"], d["w"])


# -- host checks ------------------------------------------------------------------------------------------------------
def test_check_rejects_bad_bins_updates():
    d, _ = _market(np.random.default_rng(0), n_cp=20, n_lad=5, n_bins=20)
    hp = _hp(d)
    bn = np.nonzero(hp.kind == KIND_BINS_HOST)[0]
    cl = np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0]
    good = I.order_book([(0.9, 1.0), (0.8, 2.0)], [(1.1, 1.0)])
    p, x, y = good
    bad = [
        ("bins on a product pool", [0], dict(bins=[good])),
        ("bins on a ladder", [cl[0]], dict(bins=[good])),
        ("one triple for two pools", bn[:2].tolist(), dict(bins=[good])),
        ("three triples for two pools", bn[:2].tolist(), dict(bins=[good] * 3)),
        ("not a triple", [bn[0]], dict(bins=[(p, x)])),
        ("None", [bn[0]], dict(bins=[None])),
        ("lengths differ", [bn[0]], dict(bins=[(p, x[:2], y)])),
        ("no bins", [bn[0]], dict(bins=[([], [], [])])),
        ("unsorted prices", [bn[0]], dict(bins=[(p[::-1], x, y)])),
        ("repeated price", [bn[0]], dict(bins=[(np.r_[p[0], p[0], p[2]], x, y)])),
        ("zero price", [bn[0]], dict(bins=[(np.r_[0.0, p[1:]], x, y)])),
        ("negative holding", [bn[0]], dict(bins=[(p, x, np.r_[-1.0, y[1:]])])),
        ("nan holding", [bn[0]], dict(bins=[(p, np.r_[np.nan, x[1:]], y)])),
        ("inf holding", [bn[0]], dict(bins=[(p, x, np.r_[np.inf, y[1:]])])),
        ("all-zero holdings", [bn[0]], dict(bins=[(p, 0 * x, 0 * y)])),
        ("crossed book", [bn[0]], dict(bins=[([1.0, 2.0], [1.0, 0.0], [0.0, 1.0])])),
        ("records out of fp64 range", [bn[0]], dict(bins=[([1e300, 1e301], [1e300, 1e300], [0.0, 0.0])])),
        ("too many bins", [bn[0]], dict(bins=[(np.arange(1.0, BINS_K_MAX + 2), np.ones(BINS_K_MAX + 1),
                                               np.zeros(BINS_K_MAX + 1))])),
        ("repeated id", [bn[0], bn[0]], dict(bins=[good, good])),
        ("reserves on a bins pool", [bn[0]], dict(reserves=[[1.0, 1.0]])),
        ("bins with a bad fee", [bn[0]], dict(bins=[good], fees=[1.5])),
    ]
    for what, ids, kw in bad:
        with pytest.raises(ValueError):
            check_pool_update(hp.pool_ptr, hp.kind, hp.weights, ids, **kw)
            pytest.fail(what)
    with pytest.raises(ValueError, match=r"bins\[1\]"):                     # the message names the entry
        check_pool_update(hp.pool_ptr, hp.kind, hp.weights, bn[:2], bins=[good, ([1.0, 2.0], [1.0, 0.0], [0.0, 1.0])])
    u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, bn[:3], bins=[good] * 3, fees=[0.99] * 3)
    assert len(u.bins) == 3 and u.gamma is not None
    rec, cnt, state = new_bins([good])
    r, z, pref, sums = bin_records(*good)
    assert np.array_equal(bits(rec), bits(r)) and cnt.tolist() == [len(r)]
    assert np.array_equal(bits(state), bits(np.array([[z, pref, sums[0], sums[1]]])))


# -- host state -------------------------------------------------------------------------------------------------------
def test_bin_slab_follows_replacements_bit_for_bit():
    rng = np.random.default_rng(5)
    hp, _ = I.synth_bins_market(600, 20, 3, K=(1, 32))
    bn = np.nonzero(hp.kind == KIND_BINS_HOST)[0]
    lit = {i: _triple(hp, i) for i in bn.tolist()}
    new = {}                                                  # pool -> bin_records of its current triple
    state = {}                                                # pool -> (z, p_ref, sum x, sum y) from new_bins
    slab = LadderSlab(hp.bin_ptr, hp.bin_rec)
    big, side = int(bn[0]), int(bn[1])
    # pool `big` goes K = 1 -> 2^16 -> 1; pool `side` is a one-sided book that becomes two-sided and back
    path_big = {0: 1, 3: 1 << 16, 4: 1 << 16, 6: 1}
    books = [I.order_book([], [(1.0 + 0.01 * j, 1.0) for j in range(5)]),
             I.order_book([(0.99 - 0.01 * j, 2.0) for j in range(4)], [(1.0 + 0.01 * j, 1.0) for j in range(5)]),
             I.order_book([(0.99 - 0.01 * j, 2.0) for j in range(4)], [])]
    compactions, n_steps = 0, 220
    for step in range(n_steps):
        ids = np.sort(rng.choice(bn, int(rng.integers(1, 40)), replace=False))
        ids = np.union1d(ids, [big, side]) if step < 12 else ids
        tr = []
        for i in ids.tolist():
            if i == big and step in path_big:
                K = path_big[step]
                t = (1.0 + 1e-4 * np.arange(K), np.where(np.arange(K) >= K // 2, 1.0, 0.0),
                     np.where(np.arange(K) < K // 2, 1.0, 0.0) if K > 1 else np.zeros(1))
            elif i == side and step < 12:
                t = books[[0, 1, 2, 1, 0][step % 5]]
            else:
                t = I.bins_event(rng, lit[i], rng.choice(EVENTS), k_max=48)
            tr.append(t)
        u = check_pool_update(hp.pool_ptr, hp.kind, hp.weights, ids, bins=tr)
        rec, cnt, st = new_bins([(np.asarray(t[0], float), np.asarray(t[1], float), np.asarray(t[2], float))
                                 for t in tr])
        before = len(slab.base)
        slab.replace(ids, rec, cnt)
        compactions += int(before > 0 and len(slab.base) == 0) + int(before == 0 and slab.dead == 0)
        for k, i in enumerate(ids.tolist()):
            lit[i] = tr[k]; new[i] = u.bins[k]; state[i] = st[k]
        assert slab.dead <= slab.live
        ref = _with_bins(hp, new)
        # every pool's records, gathered from the slab, against the fresh HostPools' bin_rec, in one comparison
        cnt_all = slab.T[bn] + 1
        start = np.concatenate([[0], np.cumsum(cnt_all)[:-1]])
        idx = np.repeat(slab.first[bn] - start, cnt_all) + np.arange(int(cnt_all.sum()))
        got = np.stack([slab.col(idx, k) for k in range(4)], 1)
        assert np.array_equal(bits(got), bits(ref.bin_rec)), step
        ch = np.asarray(sorted(state), np.int64)
        want = np.c_[ref.bin_zp[ch], ref.reserves[ref.pool_ptr[ch]], ref.reserves[ref.pool_ptr[ch] + 1]]
        assert np.array_equal(bits(np.stack([state[i] for i in ch.tolist()])), bits(want)), step
    ref.validate()
    assert slab.T[big] + 1 == len(bin_records(*lit[big])[0])
    assert compactions >= 1


# -- GPU --------------------------------------------------------------------------------------------------------------
def _bins_bucket(rng, counts, stride=None):
    """a bins bucket of pools with the given record counts (records: random payload), on the device, stride > m"""
    import torch
    m = len(counts)
    stride = stride or max(1024, -(-m // 1024) * 1024 + 1024)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]])
    rec = torch.as_tensor(rng.standard_normal((int(np.sum(counts)), 4)), device="cuda").reshape(-1)
    logrw = torch.as_tensor(rng.standard_normal((4, stride)), device="cuda")
    logrw[0, :m] = torch.as_tensor(first.astype(float)); logrw[1, :m] = torch.as_tensor(np.asarray(counts, float))
    R = torch.as_tensor(rng.standard_normal((2, stride)), device="cuda")
    tok = torch.zeros((2, stride), dtype=torch.int32, device="cuda")
    g = torch.ones(stride, dtype=torch.float64, device="cuda")
    tb = torch.as_tensor(rng.standard_normal((2, stride)), device="cuda")
    b = _lib.Bucket(_lib.KIND_BINS, 2, m, stride, R.data_ptr(), tok.data_ptr(), g.data_ptr(), rec.data_ptr(),
                    logrw.data_ptr(), tb.data_ptr())
    return b, dict(rec=rec, logrw=logrw, R=R, tb=tb, keep=(tok, g))


def _splice(lib, bucket, pos, cnt, rec, state, out, entry="cfmm_bins_splice"):
    import torch
    pos_t = torch.as_tensor(np.asarray(pos, np.int64), device="cuda")
    cnt_t = torch.as_tensor(np.asarray(cnt, np.int64), device="cuda")
    rec_t = torch.as_tensor(np.ascontiguousarray(rec, np.float64).reshape(-1, 4), device="cuda")
    st_t = torch.as_tensor(np.ascontiguousarray(state, np.float64).reshape(-1, 4), device="cuda")
    nb = lib.cfmm_ladder_splice_work_bytes(bucket.n_pools, len(pos))
    w = torch.empty(max(nb, 1), dtype=torch.uint8, device="cuda")
    status = (C.c_int64 * 2)()
    rc = getattr(lib, entry)(C.byref(bucket), len(pos), pos_t.data_ptr(), cnt_t.data_ptr(), rec_t.data_ptr(),
                             len(rec_t), st_t.data_ptr(), out.data_ptr(), out.numel() // 4, status, w.data_ptr(), nb,
                             None)
    return rc, status[0], status[1]


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
def test_bins_splice_kernel_matches_a_gather():
    import torch
    lib = _lib.load()
    rng = np.random.default_rng(11)
    counts = rng.integers(2, 40, 3000)
    big = rng.integers(2, 6, 2000); big[777] = 2 ** 20 + 2                           # one pool of 2^20 bins
    cases = [(counts, np.zeros(0, np.int64), None),                                   # n_chg = 0
             (counts, np.array([1234]), None),                                        # one pool
             (counts, np.arange(3000), None),                                         # every pool
             (counts, np.sort(rng.choice(3000, 500, replace=False)), None),
             (big, np.array([5, 777, 1999]), None),                                   # 2^20 + 2 -> a few
             (big, np.array([777]), 2 ** 20 + 1),                                     # -> 2^20 + 1 records
             (rng.integers(2, 6, 1000), np.array([0, 500, 999]), 2 ** 20 + 2)]        # a few -> 2^20 + 2
    for counts, pos, n_new in cases:
        b, t = _bins_bucket(rng, counts)
        cnt = np.full(len(pos), n_new) if n_new else rng.integers(2, 60, len(pos))
        if n_new and len(pos) > 1:
            cnt[1:] = rng.integers(2, 60, len(pos) - 1)
        newrec = rng.standard_normal((int(cnt.sum()), 4))
        state = rng.standard_normal((len(pos), 4))
        ref, first, c = _gather_reference(t, counts, pos, cnt, newrec)
        out = torch.full((4 * (ref.shape[0] + 17),), np.nan, dtype=torch.float64, device="cuda")
        lr0, R0, tb0 = t["logrw"].clone(), t["R"].clone(), t["tb"].clone()
        rc, bad, total = _splice(lib, b, pos, cnt, newrec, state, out)
        assert rc == 0 and bad == 0 and total == ref.shape[0]
        assert torch.equal(out[:4 * total].view(-1, 4), ref)
        assert torch.isnan(out[4 * total:]).all()
        m = len(counts)
        assert torch.equal(t["logrw"][0, :m], first.double()) and torch.equal(t["logrw"][1, :m], c.double())
        keep = torch.as_tensor(np.setdiff1d(np.arange(m), pos), device="cuda")
        assert torch.equal(t["logrw"][2:, keep], lr0[2:, keep]) and torch.equal(t["R"][:, keep], R0[:, keep])
        assert torch.equal(t["logrw"][:, m:], lr0[:, m:]) and torch.equal(t["R"][:, m:], R0[:, m:])
        assert torch.equal(t["tb"], tb0)                                                # theta_bar is not touched
        if len(pos):
            pp = torch.as_tensor(pos, device="cuda")
            st = torch.as_tensor(state, device="cuda")
            assert torch.equal(t["logrw"][2, pp], st[:, 0]) and torch.equal(t["logrw"][3, pp], st[:, 1])
            assert torch.equal(t["R"][0, pp], st[:, 2]) and torch.equal(t["R"][1, pp], st[:, 3])


@gpu
def test_bins_splice_c_abi_codes_and_rejections():
    import torch
    lib = _lib.load()
    rng = np.random.default_rng(12)
    counts = rng.integers(2, 9, 100)
    b, t = _bins_bucket(rng, counts)
    out = torch.zeros(4 * 2000, dtype=torch.float64, device="cuda")
    status = (C.c_int64 * 2)()
    work = torch.empty(lib.cfmm_ladder_splice_work_bytes(100, 1), dtype=torch.uint8, device="cuda")
    nb = work.numel()
    pos = torch.as_tensor([5], device="cuda"); cnt = torch.as_tensor([3], device="cuda")
    recd = torch.as_tensor(rng.standard_normal((3, 4)), device="cuda")
    std = torch.zeros((1, 4), dtype=torch.float64, device="cuda")

    def call(bk, p=pos, n=cnt, r=recd, s=std, o=out, w=work, wb=nb, n_chg=1, n_records=3, entry="cfmm_bins_splice",
             o_ptr=None):
        return getattr(lib, entry)(C.byref(bk) if bk is not None else None, n_chg,
                                   p.data_ptr() if p is not None else None, n.data_ptr() if n is not None else None,
                                   r.data_ptr() if r is not None else None, n_records,
                                   s.data_ptr() if s is not None else None,
                                   o_ptr if o_ptr is not None else o.data_ptr() if o is not None else None,
                                   2000, status, w.data_ptr() if w is not None else None, wb, None)
    # CFMM_E_NULL
    assert call(None) == -1
    assert call(b, p=None) == -1 and call(b, n=None) == -1 and call(b, r=None) == -1 and call(b, s=None) == -1
    assert call(b, o=None) == -1 and call(b, w=None) == -1
    nw = _lib.Bucket(*[getattr(b, f) for f, _ in _lib.Bucket._fields_]); nw.weights = None
    assert call(nw) == -1
    # CFMM_E_KIND: a concentrated, product or three-coin bucket; cfmm_ladder_splice on a bins bucket
    for kind, arity in ((_lib.KIND_CONCENTRATED, 2), (_lib.KIND_PRODUCT, 2), (_lib.KIND_BINS, 3)):
        bk = _lib.Bucket(kind, arity, b.n_pools, b.stride, b.reserves, b.tok_idx, b.gamma, b.weights, b.logrw,
                         b.theta_bar)
        assert call(bk) == -2
    assert call(b, entry="cfmm_ladder_splice") == -2
    # CFMM_E_SIZE: sizes, short work, misaligned buffers, output == weights
    assert call(b, n_chg=101) == -3 and call(b, n_chg=-1) == -3 and call(b, wb=nb - 1) == -3
    assert call(b, o_ptr=out.data_ptr() + 8) == -3
    assert call(b, r=recd.view(-1)[1:]) == -3
    assert call(b, o_ptr=b.weights) == -3
    mis = _lib.Bucket(*[getattr(b, f) for f, _ in _lib.Bucket._fields_]); mis.weights = b.weights + 8
    assert call(mis) == -3
    # entries the device rejects: nothing is written anywhere, status[0] counts them
    lr0, R0, rec0, tb0 = t["logrw"].clone(), t["R"].clone(), t["rec"].clone(), t["tb"].clone()
    out.fill_(-5.0)
    for p_, n_, nrec in (([100], [3], 3), ([5], [1], 1), ([5], [2 ** 20 + 3], 2 ** 20 + 3), ([5], [3], 4),
                         ([5], [3], 2)):
        r_ = torch.zeros((max(nrec, 1), 4), dtype=torch.float64, device="cuda")
        rc = call(b, p=torch.as_tensor(p_, device="cuda"), n=torch.as_tensor(n_, device="cuda"), r=r_, n_records=nrec)
        assert rc == 0 and status[0] > 0, (p_, n_, nrec)
    w2 = torch.empty(lib.cfmm_ladder_splice_work_bytes(100, 2), dtype=torch.uint8, device="cuda")
    for pp in ([7, 5], [5, 5]):                                                     # unsorted, repeated positions
        rc = call(b, p=torch.as_tensor(pp, device="cuda"), n=torch.as_tensor([2, 2], device="cuda"),
                  r=torch.zeros((4, 4), dtype=torch.float64, device="cuda"),
                  s=torch.zeros((2, 4), dtype=torch.float64, device="cuda"), w=w2, wb=w2.numel(), n_chg=2, n_records=4)
        assert rc == 0 and status[0] > 0, pp
    small = torch.zeros(4 * 10, dtype=torch.float64, device="cuda")
    rc = lib.cfmm_bins_splice(C.byref(b), 0, None, None, None, 0, None, small.data_ptr(), 10, status, work.data_ptr(),
                              nb, None)
    assert rc == 0 and status[0] > 0                                                # the capacity is too small
    torch.cuda.synchronize()
    assert torch.equal(t["logrw"], lr0) and torch.equal(t["R"], R0) and torch.equal(t["rec"], rec0)
    assert torch.equal(t["tb"], tb0) and bool((out == -5.0).all()) and bool((small == 0).all())


_NAMES = ("reserves", "tok_idx", "gamma", "weights", "logrw", "theta_bar")


def _bucket_tensors(store):
    out = []
    for b in store.buckets:
        if getattr(b, "blocked", False):
            out.append(("blocked",) + tuple(getattr(b, n).clone() for n in ("r0", "r1", "gamma_inv")))
            continue
        out.append((int(b.kind), int(b.arity)) + tuple(None if getattr(b, n) is None else getattr(b, n).clone()
                                                       for n in _NAMES))
    return out


def _assert_equal_tensors(xa, xb, what):
    import torch
    assert len(xa) == len(xb), what
    for a, b in zip(xa, xb):
        assert a[0] == b[0] and (a[0] == "blocked" or a[:2] == b[:2]), what
        for x, y in zip(a[1:] if a[0] == "blocked" else a[2:], b[1:] if b[0] == "blocked" else b[2:]):
            assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), (what, a[:2])


def _block(rng, d, k_bins=None):
    """one block of mixed updates of the literals d (returned as update_pools calls; d is updated in place): bins= and
    fees= of bins pools, ladders= and prices= of concentrated pools, reserves= and fees= of product pools"""
    kinds = np.asarray(d["kinds"])
    bn, cl, cp = (np.nonzero(kinds == k)[0] for k in ("bins", "concentrated", "product"))
    calls = []
    ids = np.sort(rng.choice(bn, k_bins or len(bn) // 3, replace=False))
    tr = [I.bins_event(rng, d["w"][i], rng.choice(EVENTS), k_max=32) for i in ids.tolist()]
    calls.append(dict(pool_ids=ids, bins=tr, fees=np.where(rng.random(len(ids)) < 0.3, 0.998, 0.9995)))
    fb = np.sort(rng.choice(np.setdiff1d(bn, ids), 5, replace=False))                 # a fee change alone
    calls.append(dict(pool_ids=fb, fees=np.full(len(fb), 0.9997)))
    li = np.sort(rng.choice(cl, len(cl) // 4, replace=False))
    calls.append(dict(pool_ids=li, ladders=[_ladder(rng, d["w"][i][0] * np.exp(rng.normal(0, 0.01)),
                                                    int(rng.integers(1, 30))) for i in li.tolist()]))
    pm = np.sort(rng.choice(np.setdiff1d(cl, li), len(cl) // 4, replace=False))
    calls.append(dict(pool_ids=pm, prices=np.array([d["w"][i][0] for i in pm.tolist()]) *
                      np.exp(rng.normal(0, 0.01, len(pm)))))
    pc = np.sort(rng.choice(cp, 20, replace=False))
    calls.append(dict(pool_ids=pc, reserves=np.array([d["res"][i] for i in pc.tolist()]) *
                      np.exp(rng.normal(0, 0.003, (len(pc), 2))), fees=np.full(len(pc), 0.996)))
    for c in calls:
        for k, i in enumerate(np.asarray(c["pool_ids"]).tolist()):
            if "bins" in c:
                d["w"][i] = c["bins"][k]
            if "ladders" in c:
                d["w"][i] = c["ladders"][k]
            if "prices" in c:
                d["w"][i] = (float(c["prices"][k]),) + tuple(d["w"][i][1:])
            if "reserves" in c:
                d["res"][i] = list(np.asarray(c["reserves"][k], float))
            if "fees" in c:
                d["fees"][i] = float(c["fees"][k])
    return calls


def _snapshot(d):
    return dict(d, res=list(d["res"]), fees=list(d["fees"]), w=list(d["w"]))


@gpu
@pytest.mark.parametrize("world", [1, 2, 3])
def test_blocks_of_bins_updates_equal_a_fresh_store(world):
    import torch
    rng = np.random.default_rng(40 + world)
    d, prices = _market(rng)
    d0 = _snapshot(d)
    hp = _hp(d)
    hp_bits = {f: bits(getattr(hp, f)).copy() for f in ("reserves", "gamma", "bin_rec", "bin_zp", "lad_rec")}
    stores = [cf.PoolStore(hp, rank=r, world=world) for r in range(world)]
    u = cf.Arbitrage(prices)
    tol = 1e-6
    prev = {}
    if world == 1:
        prev = {p: cf.solve_pools(hp, u, tol=tol, store=stores[0], native=p, want_trades=False)
                for p in (False, "hostloop")}
    for blk in range(3):
        tb = [[None if getattr(b, "theta_bar", None) is None else b.theta_bar.clone() for b in st.buckets]
              for st in stores]
        calls = _block(rng, d)
        for c in calls:
            for st in stores:
                st.update_pools(**c)
        hp2 = _hp(d)
        bins_ids = calls[0]["pool_ids"]
        for r, st in enumerate(stores):
            fresh = cf.PoolStore(hp2, rank=r, world=world)
            # the replaced pools' multipliers restart at 0, the others keep theirs; after a reset every tensor of
            # every bucket equals the fresh store's
            bi, loc = st._pool_map()
            for k, b in enumerate(st.buckets):
                if b.kind == _lib.KIND_BINS:
                    mine = torch.as_tensor(loc[bins_ids[bi[bins_ids] == k]], device="cuda")
                    others = torch.ones(b.stride, dtype=torch.bool, device="cuda"); others[mine] = False
                    assert bool((b.theta_bar[:, mine] == 0).all())
                    assert torch.equal(b.theta_bar[:, others], tb[r][k][:, others])
            st.reset_multipliers()
            _assert_equal_tensors(_bucket_tensors(st), _bucket_tensors(fresh), (world, blk, r))
        if world == 1:
            spec = u.spec(d["n"])
            cold = cf.solve_pools(hp2, u, tol=tol, store=cf.PoolStore(hp2), native=False, want_trades=False)
            assert cold.status == "optimal"
            for path in (False, "hostloop"):
                res = cf.solve_pools(hp2, u, tol=tol, store=stores[0], nu0=prev[path].nu, native=path)
                assert res.status == "optimal", (blk, path, res.status)
                XB.certify(hp2, spec, res, tol)
                assert abs(res.value - cold.value) <= 20 * tol * max(abs(cold.dual_value), 1e-300), \
                    (path, res.value, cold.value)
                prev[path] = res
    # the caller's HostPools was not modified
    for f, v in hp_bits.items():
        assert np.array_equal(bits(getattr(hp, f)), v), f
    assert np.array_equal(bits(_hp(d0).bin_rec), hp_bits["bin_rec"])


@gpu
def test_store_bin_fills_after_updates():
    rng = np.random.default_rng(50)
    d, _ = _market(rng, n_cp=100, n_lad=10, n_bins=80)
    hp = _hp(d)
    st = cf.PoolStore(hp)
    for _ in range(3):
        for c in _block(rng, d):
            st.update_pools(**c)
    hp2 = _hp(d)
    bn = np.nonzero(hp2.kind == KIND_BINS_HOST)[0]
    for i in bn.tolist():
        S = hp2.reserves[hp2.pool_ptr[i]:hp2.pool_ptr[i] + 2]
        for t in (0.0, 0.3 * S[0], 2.0 * S[0] + 1.0, -0.5 * S[1] / d["w"][i][0][0], -1e9):
            a, b = st.bin_fills(i, t), bin_fills(hp2, i, t)
            for x, y in zip(a, b):
                assert np.array_equal(bits(x) if x.dtype == np.float64 else x, bits(y) if y.dtype == np.float64 else y)
    with pytest.raises(ValueError):
        st.bin_fills(0, 1.0)                                                        # a product pool
    with pytest.raises(ValueError):
        st.bin_fills(hp.m, 1.0)
    two = [cf.PoolStore(hp2, rank=r, world=2) for r in range(2)]
    i = int(bn[two[0]._pool_map()[0][bn] < 0][0])
    two[1].bin_fills(i, 1.0)
    with pytest.raises(ValueError):
        two[0].bin_fills(i, 1.0)                                                    # held by the other rank


@gpu
def test_an_invalid_bins_entry_changes_nothing():
    rng = np.random.default_rng(61)
    d, prices = _market(rng, n_cp=1500, n_lad=40, n_bins=1500, K=(1, 8))
    hp = _hp(d)
    store = cf.PoolStore(hp)
    for c in _block(rng, d):                                                        # the store has its own slab first
        store.update_pools(**c)
    bn = np.nonzero(hp.kind == KIND_BINS_HOST)[0]
    ids = np.sort(rng.choice(bn, 1000, replace=False))
    tr = [I.bins_event(rng, d["w"][i], rng.choice(EVENTS), k_max=32) for i in ids.tolist()]
    bad = list(tr); bad[500] = ([1.0, 2.0], [1.0, 0.0], [0.0, 1.0])                  # crossed
    before = _bucket_tensors(store)
    bk = next(b for b in store.buckets if b.kind == _lib.KIND_BINS)
    ptr = (bk.c_bucket.weights, bk.weights.data_ptr())
    slab = store._bins()
    host = (slab.first.copy(), slab.T.copy(), slab.n_own, slab.live, slab.dead, slab.own[:slab.n_own].copy())
    with pytest.raises(ValueError, match=r"bins\[500\]"):
        store.update_pools(ids, bins=bad, fees=np.full(len(ids), 0.99))
    _assert_equal_tensors(_bucket_tensors(store), before, "crossed")
    assert (bk.c_bucket.weights, bk.weights.data_ptr()) == ptr
    assert np.array_equal(slab.first, host[0]) and np.array_equal(slab.T, host[1])
    assert (slab.n_own, slab.live, slab.dead) == host[2:5] and np.array_equal(slab.own[:slab.n_own], host[5])
    store.update_pools(ids, bins=tr)                                                # the next valid block succeeds
    for k, i in enumerate(ids.tolist()):
        d["w"][i] = tr[k]
    store.reset_multipliers()
    _assert_equal_tensors(_bucket_tensors(store), _bucket_tensors(cf.PoolStore(_hp(d))), "after")
