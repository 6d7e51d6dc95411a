"""Times a block of mints, burns, price moves and StableSwap rate / A changes re-solved on the resident store, against a
rebuild.

The market is instances.synth_concentrated_market at --pools pools (half of them ladders of T in (1, 64)) over --tokens
tokens; every ladder is re-declared once as literals (price, bounds = b^2, liquidity), which both paths then follow.
Per block (six blocks per k, the first one a warm-up):
  - k ladders get a mint or a burn: liquidity added to or removed from a run of intervals; a third of them initialise a
    tick inside the run (T + 1) and a third clear one (T - 1);
  - 10 000 other ladders move price;
  - 1 % of the StableSwap pools get new rates (the rate-bearing coins' oracles), five a ramp step of A (x 1.0005).
  update path:  PoolStore.update_pools (ladders=, prices=, rates=, amp=; synchronous) + solve_pools(..., store=, nu0=
                previous nu), warm;
  rebuild path: HostPools of the updated literals (ladder_records of every ladder, grouped by T; D of every StableSwap
                pool) + PoolStore + solve_pools from the default prices, cold;
both at tol 1e-6 without trades, alternated in the same run; medians over the five timed blocks of each k.  Then
cfmm_ladder_splice alone on the store's concentrated bucket (CUDA-event medians): k pools with new records of the same
count, and k pools whose count changes.  The card's name and power limit are printed with the numbers.
    python scripts/time_ladder_update.py [--pools 100000] [--tokens 1000] [--json out.json]
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
from cfmm_routing_code_b200.pools import (HostPools, KIND_CONCENTRATED_HOST, KIND_STABLESWAP_HOST,  # noqa: E402
                                          ladder_records, ladder_state)
from time_stableswap_n import _events, card                          # noqa: E402

KS = (100, 1000, 10_000)


def literals(hp):
    """every ladder of hp as (price, bounds, liquidity) literals"""
    lp, rec = hp.lad_ptr, hp.lad_rec
    out = {}
    for i in np.nonzero(hp.kind == KIND_CONCENTRATED_HOST)[0].tolist():
        r = rec[lp[i]:lp[i + 1]]
        out[i] = (float(hp.lad_sc[i, 0]) ** 2, r[:, 0] ** 2, r[:-1, 1].copy())
    return out


def rebuild(base, lad):
    """HostPools of the current literals: base's other pools (reserves, weights, amp as updated) and the ladders lad"""
    ids = np.asarray(sorted(lad), np.int64)
    T = np.asarray([len(lad[i][2]) for i in ids.tolist()], np.int64)
    recs = [None] * len(ids)
    for t in np.unique(T).tolist():
        sel = np.nonzero(T == t)[0]
        B = np.stack([lad[ids[j]][1] for j in sel.tolist()]); L = np.stack([lad[ids[j]][2] for j in sel.tolist()])
        for j, r in zip(sel.tolist(), ladder_records(B, L)):
            recs[j] = r
    lad_ptr = np.zeros(base.m + 1, np.int64)
    cnt = np.zeros(base.m, np.int64); cnt[ids] = T + 1
    lad_ptr[1:] = np.cumsum(cnt)
    rec = np.concatenate(recs)
    s, c, x, y = ladder_state(lad_ptr, rec, ids, [lad[i][0] for i in ids.tolist()])
    sc = np.zeros((base.m, 2)); sc[ids, 0], sc[ids, 1] = s, c
    R = base.reserves.copy(); R[base.pool_ptr[ids]], R[base.pool_ptr[ids] + 1] = x, y
    return HostPools(base.n_tokens, base.pool_ptr, base.tok_idx, R, base.weights, base.gamma, base.kind, base.amp, None,
                     lad_ptr, rec, sc)


def mint_or_burn(rng, lit):
    """a mint or burn on a run of intervals; a third initialise a tick inside it (T + 1), a third clear one (T - 1)"""
    p, b, L = lit
    b, L = b.copy(), L.copy()
    T = len(L)
    what = rng.integers(0, 3)
    if what == 1 and T < 64:                                  # a new tick splits interval j
        j = int(rng.integers(0, T))
        b = np.insert(b, j + 1, np.sqrt(b[j] * b[j + 1])); L = np.insert(L, j + 1, L[j])
    elif what == 2 and T > 1:                                 # an interior tick is cleared: intervals j, j + 1 merge
        j = int(rng.integers(0, T - 1))
        b = np.delete(b, j + 1); L = np.delete(L, j + 1)
    T = len(L)
    lo = int(rng.integers(0, T)); hi = int(rng.integers(lo, T)) + 1
    L[lo:hi] = np.maximum(L[lo:hi] + np.exp(6.0 + rng.standard_normal()) * rng.choice([-0.5, 1.0]), 0.0)
    if not np.any(L > 0):
        L[lo] = np.exp(6.0)
    return (p, b, L)


def time_splice(store, k, rng, change):
    """CUDA-event median of cfmm_ladder_splice on the store's concentrated bucket: k pools, the same record counts or
    changed ones (payload: the pools' own records, so the ladders stay valid)"""
    b = next(x for x in store.buckets if x.kind == _lib.KIND_CONCENTRATED)
    lr = b.logrw[:, :b.m].cpu().numpy()
    pos = np.sort(rng.choice(b.m, k, replace=False))
    first, T = lr[2, pos].astype(np.int64), lr[3, pos].astype(np.int64)
    cnt = T + 1
    if change:
        cnt = np.where(T > 1, T, T + 2)                       # one record fewer (T > 1) or one more
    src = np.concatenate([first[j] + np.minimum(np.arange(cnt[j]), T[j]) for j in range(k)])
    rec = b.weights.view(-1, 4)[torch.as_tensor(src, device="cuda")].contiguous()
    state = torch.as_tensor(np.stack([lr[0, pos], np.minimum(lr[1, pos], cnt - 2), b.reserves[0, pos].cpu().numpy(),
                                      b.reserves[1, pos].cpu().numpy()], 1), device="cuda")
    pos_t = torch.as_tensor(pos, device="cuda"); cnt_t = torch.as_tensor(cnt, device="cuda")
    total = b.n_rec + int(cnt.sum() - (T + 1).sum())
    out = torch.empty(4 * total, dtype=torch.float64, device="cuda")
    nb = int(store.lib.cfmm_ladder_splice_work_bytes(b.m, k))
    work = torch.empty(nb, dtype=torch.uint8, device="cuda")
    status = (C.c_int64 * 2)()
    bk = _lib.Bucket(*[getattr(b.c_bucket, f) for f, _ in _lib.Bucket._fields_])
    # the splice writes logrw and reserves in place; with the same counts it writes what is there (the output buffer is
    # never swapped in), changed counts are undone after every call (inside the timed interval: ~2.4 MB of copies)
    lr_save, R_save = b.logrw.clone(), b.reserves.clone()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run():
        _lib.check(store.lib.cfmm_ladder_splice(C.byref(bk), k, pos_t.data_ptr(), cnt_t.data_ptr(), rec.data_ptr(),
                                                len(rec), state.data_ptr(), out.data_ptr(), total, status,
                                                work.data_ptr(), nb, st), "cfmm_ladder_splice")
        assert status[0] == 0 and status[1] == total
        if change:
            b.logrw.copy_(lr_save); b.reserves.copy_(R_save)
    us = _events(run, 20, 3)
    b.logrw.copy_(lr_save); b.reserves.copy_(R_save)
    return us, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=100_000)
    ap.add_argument("--tokens", type=int, default=1000)
    ap.add_argument("--json", default=None, help="also write the per-block records here")
    args = ap.parse_args()
    gpu = card()
    print("card:", gpu, flush=True)
    hp0, prices = I.synth_concentrated_market(args.pools, args.tokens, seed=1, T=(1, 64))
    lad = literals(hp0)
    hp = rebuild(hp0, lad)                                    # the literals' HostPools: both paths start here
    cur = HostPools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, hp.reserves.copy(), hp.weights.copy(), hp.gamma.copy(),
                    hp.kind, hp.amp.copy())                   # the rebuild path's other pools (reserves, rates, A)
    cl = np.asarray(sorted(lad), np.int64)
    ss = np.nonzero(hp.kind == KIND_STABLESWAP_HOST)[0]
    ar = np.diff(hp.pool_ptr)
    util = cf.Arbitrage(prices)
    tol = 1e-6
    store = cf.PoolStore(hp)
    prev = cf.solve_pools(hp, util, tol=tol, store=store, want_trades=False)
    print(f"{hp.m} pools: {len(cl)} ladders ({len(hp.lad_rec)} records), {len(ss)} StableSwap; first solve "
          f"{prev.status} in {1e3 * prev.wall_s:.1f} ms", flush=True)
    rng = np.random.default_rng(0)
    recs, blk = [], 0
    for k in KS:
        for rep in range(6):
            ids = np.sort(rng.choice(cl, k, replace=False))
            new = [mint_or_burn(rng, lad[i]) for i in ids.tolist()]
            mv = np.sort(rng.choice(np.setdiff1d(cl, ids), 10_000, replace=False))
            newp = np.array([lad[i][0] for i in mv.tolist()]) * np.exp(0.002 * rng.standard_normal(len(mv)))
            sr = np.sort(rng.choice(ss, max(1, len(ss) // 100), replace=False))
            rates = [cur.weights[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] * np.exp(1e-4 * rng.standard_normal(ar[i]))
                     for i in sr.tolist()]
            sa = np.sort(rng.choice(np.setdiff1d(ss, sr), 5, replace=False))
            A = cur.amp[sa] * 1.0005
            dT = sum(len(n[2]) != len(lad[i][2]) for n, i in zip(new, ids.tolist()))
            # update path
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            store.update_pools(ids, ladders=new)
            store.update_pools(mv, prices=newp)
            store.update_pools(sr, rates=rates)
            store.update_pools(sa, amp=A)
            t_upd = time.perf_counter() - t0
            t0 = time.perf_counter()
            r = cf.solve_pools(hp, util, tol=tol, store=store, nu0=prev.nu, want_trades=False)
            torch.cuda.synchronize()
            t_warm = time.perf_counter() - t0
            prev = r
            # rebuild path, same data
            for i, n in zip(ids.tolist(), new):
                lad[i] = n
            for i, p in zip(mv.tolist(), newp.tolist()):
                lad[i] = (p, lad[i][1], lad[i][2])
            for i, w in zip(sr.tolist(), rates):
                cur.weights[hp.pool_ptr[i]:hp.pool_ptr[i + 1]] = w
            cur.amp[sa] = A
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            h2 = rebuild(cur, lad)
            t_host = time.perf_counter() - t0
            t0 = time.perf_counter()
            st2 = cf.PoolStore(h2)
            torch.cuda.synchronize()
            t_build = time.perf_counter() - t0
            t0 = time.perf_counter()
            rc = cf.solve_pools(h2, util, tol=tol, store=st2, want_trades=False)
            torch.cuda.synchronize()
            t_cold = time.perf_counter() - t0
            del st2
            rec = dict(block=blk, k=k, T_changed=int(dT), update_ms=1e3 * t_upd, warm_ms=1e3 * t_warm,
                       warm=(r.status, r.iters, r.evals, r.hvps), hostpools_ms=1e3 * t_host, build_ms=1e3 * t_build,
                       cold_ms=1e3 * t_cold, cold=(rc.status, rc.iters, rc.evals, rc.hvps),
                       rel_value_diff=abs(r.value - rc.value) / abs(rc.value), timed=rep > 0)
            recs.append(rec)
            print(f"block {blk:2d} k {k:6d} (T changed {dT:5d}): update {rec['update_ms']:8.2f} ms + warm solve "
                  f"{rec['warm_ms']:7.2f} ms {rec['warm']} | HostPools {rec['hostpools_ms']:8.2f} ms + store "
                  f"{rec['build_ms']:7.2f} ms + cold solve {rec['cold_ms']:7.2f} ms {rec['cold']} | values differ "
                  f"{rec['rel_value_diff']:.1e}", flush=True)
            blk += 1
    print(f"\nmedians of the 5 timed blocks per k ({gpu}); {args.pools} pools, {args.tokens} tokens, tol {tol:g}, "
          "no trades")
    print(f"{'k':>6s} {'update':>9s} {'warm solve':>11s} {'update path':>12s} | {'HostPools':>10s} {'store':>8s} "
          f"{'cold solve':>11s} {'rebuild path':>13s}")
    summary = {}
    for k in KS:
        rs = [x for x in recs if x["k"] == k and x["timed"]]
        med = lambda key: float(np.median([x[key] for x in rs]))
        upd = float(np.median([x["update_ms"] + x["warm_ms"] for x in rs]))
        reb = float(np.median([x["hostpools_ms"] + x["build_ms"] + x["cold_ms"] for x in rs]))
        summary[k] = dict(update_ms=med("update_ms"), warm_ms=med("warm_ms"), update_path_ms=upd,
                          hostpools_ms=med("hostpools_ms"), build_ms=med("build_ms"), cold_ms=med("cold_ms"),
                          rebuild_path_ms=reb)
        print(f"{k:6d} {med('update_ms'):7.2f}ms {med('warm_ms'):9.2f}ms {upd:10.2f}ms | {med('hostpools_ms'):8.2f}ms "
              f"{med('build_ms'):6.2f}ms {med('cold_ms'):9.2f}ms {reb:11.2f}ms")
    print("\ncfmm_ladder_splice alone (CUDA events, median of 20):")
    sp = {}
    for k in KS:
        for change in (False, True):
            us, total = time_splice(store, k, rng, change)
            sp[f"k{k}_{'T_changes' if change else 'same_T'}"] = us
            print(f"  k {k:6d} {'T changes' if change else 'same T   '}: {us:8.1f} us  ({total} records, "
                  f"{32 * total / 1e6:.1f} MB copied)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(gpu=gpu, blocks=recs, summary=summary, splice_us=sp), f, indent=1)


if __name__ == "__main__":
    main()
