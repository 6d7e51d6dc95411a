"""Times blocks of replaced price-bin pools applied in place on the resident store (update_pools(bins=)), against a
rebuild of the market.

Market: instances.synth_bins_market(--pools, --tokens, seed 1, K=(1, 256)): every bins pool is re-declared once as its
(prices, x, y) literals, which both paths then follow.  Per block (three blocks per k, the first one a warm-up), k bins
pools get one seeded event each (instances.bins_event): a Liquidity Book swap that empties the active bin and moves it
one to three bins, a deposit or withdrawal that changes K, an order-book change (levels taken through the mid and
reposted, a new level past the far end, sizes moved) or a partial fill of a limit order.
  update path:   PoolStore.update_pools(ids, bins=) (host clock around the synchronous call);
  splice alone:  cfmm_bins_splice on the store's bins bucket with k pools' own records (CUDA-event median of 20);
  rebuild path:  HostPools.from_lists of every literal + PoolStore (host clock, synchronised).
Then, on a K = (1, 16) market of the same size, one block per k followed by a warm re-solve from the previous prices on
the updated store, against a cold solve on a rebuilt store, both at tol 1e-6 on solver.py's loop, with their status.
The card's name and power limit are printed with the numbers.
    python scripts/time_bins_update.py [--pools 100000] [--tokens 1000] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cfmm_routing_code_b200 as cf                                   # noqa: E402
from cfmm_routing_code_b200 import _lib, instances as I               # noqa: E402
from cfmm_routing_code_b200.pools import HostPools, KIND_BINS_HOST    # noqa: E402
from time_stableswap_n import _events, card                          # noqa: E402

KS = (100, 1000, 10_000)
EVENTS = ("swap", "deposit", "withdraw", "book", "fill")


def literals(hp):
    """every pool of hp as from_lists literals; bins pools' (prices, x, y) read back from their records (the active
    bin's two segments merged)"""
    li, res, fees, kinds, w = [], [], [], [], []
    bp, rec = np.asarray(hp.bin_ptr, np.int64), np.asarray(hp.bin_rec, np.float64).reshape(-1, 4)
    for i in range(hp.m):
        li.append(hp.tok_idx[hp.pool_ptr[i]:hp.pool_ptr[i] + 2].tolist()); fees.append(float(hp.gamma[i]))
        if hp.kind[i] != KIND_BINS_HOST:
            res.append(hp.reserves[hp.pool_ptr[i]:hp.pool_ptr[i] + 2].tolist()); kinds.append("product"); w.append(None)
            continue
        r, z = rec[bp[i]:bp[i + 1]], int(hp.bin_zp[i, 0])
        seg = np.arange(len(r) - 1)
        pr, inv = np.unique(r[seg, 2], return_inverse=True)
        x = np.bincount(inv, np.where(seg >= z, r[seg + 1, 0] - r[seg, 0], 0.0), len(pr))
        y = np.bincount(inv, np.where(seg < z, r[seg + 1, 1] - r[seg, 1], 0.0), len(pr))
        res.append(None); kinds.append("bins"); w.append((pr, x, y))
    return dict(n=hp.n_tokens, li=li, res=res, fees=fees, kinds=kinds, w=w)


def from_literals(d):
    return HostPools.from_lists(d["n"], d["li"], d["res"], d["fees"], d["kinds"], d["w"])


def block(rng, d, bn, k):
    ids = np.sort(rng.choice(bn, k, replace=False))
    return ids, [I.bins_event(rng, d["w"][i], rng.choice(EVENTS)) for i in ids.tolist()]


def apply(d, ids, tr):
    for i, t in zip(ids.tolist(), tr):
        d["w"][i] = t


def time_splice(store, k, rng):
    """CUDA-event median of cfmm_bins_splice on the store's bins bucket: k pools with their own records and state (the
    bucket's tensors keep their values; the output buffer is never swapped in)"""
    b = next(x for x in store.buckets if x.kind == _lib.KIND_BINS)
    lr = b.logrw[:, :b.m].cpu().numpy()
    pos = np.sort(rng.choice(b.m, k, replace=False))
    first, cnt = lr[0, pos].astype(np.int64), lr[1, pos].astype(np.int64)
    src = np.concatenate([first[j] + np.arange(cnt[j]) for j in range(k)])
    rec = b.weights.view(-1, 4)[torch.as_tensor(src, device="cuda")].contiguous()
    state = torch.as_tensor(np.stack([lr[2, pos], lr[3, pos], b.reserves[0, pos].cpu().numpy(),
                                      b.reserves[1, pos].cpu().numpy()], 1), device="cuda")
    pos_t = torch.as_tensor(pos, device="cuda"); cnt_t = torch.as_tensor(cnt, device="cuda")
    out = torch.empty(4 * b.n_rec, dtype=torch.float64, device="cuda")
    nb = int(store.lib.cfmm_ladder_splice_work_bytes(b.m, k))
    work = torch.empty(nb, dtype=torch.uint8, device="cuda")
    status = (C.c_int64 * 2)()
    bk = _lib.Bucket(*[getattr(b.c_bucket, f) for f, _ in _lib.Bucket._fields_])
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run():
        _lib.check(store.lib.cfmm_bins_splice(C.byref(bk), k, pos_t.data_ptr(), cnt_t.data_ptr(), rec.data_ptr(),
                                              len(rec), state.data_ptr(), out.data_ptr(), b.n_rec, status,
                                              work.data_ptr(), nb, st), "cfmm_bins_splice")
        assert status[0] == 0 and status[1] == b.n_rec
    us = _events(run, 20, 3)
    assert torch.equal(out, b.weights)                         # the same records, spliced into the same places
    return us, b.n_rec


def bins_equal(a, b):
    x = next(t for t in a.buckets if t.kind == _lib.KIND_BINS)
    y = next(t for t in b.buckets if t.kind == _lib.KIND_BINS)
    return all(torch.equal(getattr(x, n), getattr(y, n)) for n in ("reserves", "gamma", "weights", "logrw"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=100_000)
    ap.add_argument("--tokens", type=int, default=1000)
    ap.add_argument("--json", default=None, help="also write the records here")
    args = ap.parse_args()
    gpu = card()
    print("card:", gpu, flush=True)
    out = dict(gpu=gpu, pools=args.pools, tokens=args.tokens)
    hp0, prices = I.synth_bins_market(args.pools, args.tokens, seed=1, K=(1, 256))
    d = literals(hp0)
    hp = from_literals(d)
    bn = np.nonzero(hp.kind == KIND_BINS_HOST)[0]
    store = cf.PoolStore(hp)
    torch.cuda.synchronize()
    print(f"K = (1, 256): {hp.m} pools, {len(bn)} bins pools, {len(hp.bin_rec)} records", flush=True)
    rng = np.random.default_rng(0)
    recs = []
    for k in KS:
        for rep in range(3):
            ids, tr = block(rng, d, bn, k)
            dK = sum(len(t[0]) != len(d["w"][i][0]) for i, t in zip(ids.tolist(), tr))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            store.update_pools(ids, bins=tr)
            torch.cuda.synchronize()
            t_upd = time.perf_counter() - t0
            apply(d, ids, tr)
            t0 = time.perf_counter()
            h2 = from_literals(d)
            t_host = time.perf_counter() - t0
            t0 = time.perf_counter()
            st2 = cf.PoolStore(h2)
            torch.cuda.synchronize()
            t_build = time.perf_counter() - t0
            same = bins_equal(store, st2)
            del st2
            r = dict(k=k, K_changed=int(dK), update_ms=1e3 * t_upd, hostpools_ms=1e3 * t_host,
                     build_ms=1e3 * t_build, equal=bool(same), timed=rep > 0)
            recs.append(r)
            print(f"k {k:6d} (K changed {dK:5d}): update {r['update_ms']:8.2f} ms | HostPools {r['hostpools_ms']:8.1f} ms "
                  f"+ store {r['build_ms']:7.1f} ms | bins bucket equal to the rebuilt one: {same}", flush=True)
    summary = {}
    print(f"\nmedians of the timed blocks per k ({gpu}); {args.pools} pools, {args.tokens} tokens, K = (1, 256)")
    print(f"{'k':>6s} {'update':>10s} {'splice':>10s} | {'HostPools':>10s} {'store':>9s} {'rebuild':>10s}")
    for k in KS:
        rs = [x for x in recs if x["k"] == k and x["timed"]]
        med = lambda key: float(np.median([x[key] for x in rs]))
        us, total = time_splice(store, k, rng)
        summary[k] = dict(update_ms=med("update_ms"), splice_us=us, records=total, hostpools_ms=med("hostpools_ms"),
                          build_ms=med("build_ms"), rebuild_ms=med("hostpools_ms") + med("build_ms"))
        print(f"{k:6d} {med('update_ms'):8.2f}ms {us:8.1f}us | {med('hostpools_ms'):8.1f}ms {med('build_ms'):7.1f}ms "
              f"{summary[k]['rebuild_ms']:8.1f}ms")
    out.update(blocks=recs, summary=summary)
    del store
    torch.cuda.empty_cache()

    # warm re-solve after an update against a cold solve of the rebuilt store, K = (1, 16)
    hp1, prices = I.synth_bins_market(args.pools, args.tokens, seed=2, K=(1, 16))
    d = literals(hp1)
    hp = from_literals(d)
    bn = np.nonzero(hp.kind == KIND_BINS_HOST)[0]
    util = cf.Arbitrage(prices)
    tol = 1e-6
    store = cf.PoolStore(hp)
    prev = cf.solve_pools(hp, util, tol=tol, store=store, native=False, want_trades=False)
    print(f"\nK = (1, 16): {hp.m} pools, {len(hp.bin_rec)} records; first solve {prev.status} in "
          f"{1e3 * prev.wall_s:.0f} ms", flush=True)
    solves = []
    for k in KS:
        ids, tr = block(rng, d, bn, k)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        store.update_pools(ids, bins=tr)
        torch.cuda.synchronize()
        t_upd = time.perf_counter() - t0
        t0 = time.perf_counter()
        r = cf.solve_pools(hp, util, tol=tol, store=store, nu0=prev.nu, native=False, want_trades=False)
        torch.cuda.synchronize()
        t_warm = time.perf_counter() - t0
        prev = r
        apply(d, ids, tr)
        t0 = time.perf_counter()
        h2 = from_literals(d)
        st2 = cf.PoolStore(h2)
        torch.cuda.synchronize()
        t_reb = time.perf_counter() - t0
        t0 = time.perf_counter()
        c = cf.solve_pools(h2, util, tol=tol, store=st2, native=False, want_trades=False)
        torch.cuda.synchronize()
        t_cold = time.perf_counter() - t0
        del st2
        s = dict(k=k, update_ms=1e3 * t_upd, warm_ms=1e3 * t_warm, warm=(r.status, r.iters, r.evals, r.hvps),
                 rebuild_ms=1e3 * t_reb, cold_ms=1e3 * t_cold, cold=(c.status, c.iters, c.evals, c.hvps),
                 rel_value_diff=abs(r.value - c.value) / abs(c.value))
        solves.append(s)
        print(f"k {k:6d}: update {s['update_ms']:7.1f} ms + warm solve {s['warm_ms']:7.0f} ms {s['warm']} | rebuild "
              f"{s['rebuild_ms']:7.0f} ms + cold solve {s['cold_ms']:7.0f} ms {s['cold']} | values differ "
              f"{s['rel_value_diff']:.1e}", flush=True)
    out.update(solves=solves)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
