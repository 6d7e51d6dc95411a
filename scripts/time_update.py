"""Times a changed market re-solved on the resident store against a rebuild.

The bench instance (1M constant-product pools, 4096 tokens, pinned host arrays, Arbitrage utility) goes through blocks.
Each block moves the reserves of k random pools by ~1% (k = 100, 10 000, 100 000; ten blocks per k, the first one a
warm-up); every tenth block also moves fees, and two of those push one tile past 16 distinct fees and back.  Per block:
  update path:  PoolStore.update_pools (synchronous) + solve_pools(..., store=, nu0=previous nu), warm;
  rebuild path: PoolStore(updated host data) + solve_pools(..., store=) from the default prices, cold;
both at tol 1e-6 without trades, alternated in the same run.  Medians over the nine timed blocks of each k.
    python scripts/time_update.py [--json out.json]
"""
import argparse, json, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import instances as I

P = 1024


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=20).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None, help="also write the per-block records here")
    args = ap.parse_args()
    m, n = 1_000_000, 4096
    s = I.synth_const_product(m, n, seed=3)
    hp = cf.HostPools.from_pairs(n, s["idx"], s["reserves"], s["gamma"]).pin_memory()
    cur = cf.HostPools.from_pairs(n, s["idx"], s["reserves"].copy(), s["gamma"].copy()).pin_memory()   # rebuild path's data
    util = cf.Arbitrage(s["prices"])
    tol = 1e-6
    name, limit = gpu_info()
    print(f"GPU: {name}, power limit {limit}", flush=True)
    store = cf.PoolStore(hp)
    prev = cf.solve_pools(hp, util, tol=tol, store=store, want_trades=False)
    order = store.buckets[0].order.cpu().numpy().astype(np.int64)
    odd = order[100 * P:100 * P + 14]                             # 14 pools of tile 100: 3 tiers + 14 = 17 distinct fees
    rng = np.random.default_rng(0)
    recs, blk = [], 0
    for k in (100, 10_000, 100_000):
        for rep in range(10):
            ids = rng.choice(m, k, replace=False)
            R = cur.reserves.reshape(-1, 2)[ids] * np.exp(0.01 * rng.standard_normal((k, 2)))
            g = None
            if blk % 10 == 5:                                     # fees move too
                g = cur.gamma[ids].copy()
                g[rng.random(k) < 0.1] = 0.998
                if blk in (15, 25):                               # tile 100 past 16 distinct fees (15), back (25)
                    keep = ~np.isin(ids, odd)
                    ids = np.concatenate([ids[keep], odd])
                    R = cur.reserves.reshape(-1, 2)[ids] * np.exp(0.01 * rng.standard_normal((len(ids), 2)))
                    g = np.concatenate([g[keep], 0.98 + 1e-4 * np.arange(14) if blk == 15 else np.full(14, 0.997)])
            # update path
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rebuilt = store.update_pools(ids, reserves=R, fees=g)
            t_upd = time.perf_counter() - t0
            t0 = time.perf_counter()
            r = cf.solve_pools(hp, util, tol=tol, store=store, nu0=prev.nu, want_trades=False)
            torch.cuda.synchronize()
            t_warm = time.perf_counter() - t0
            prev = r
            # rebuild path, same data
            cur.reserves.reshape(-1, 2)[ids] = R
            if g is not None:
                cur.gamma[ids] = g
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st2 = cf.PoolStore(cur)
            torch.cuda.synchronize()
            t_build = time.perf_counter() - t0
            t0 = time.perf_counter()
            rc = cf.solve_pools(cur, util, tol=tol, store=st2, want_trades=False)
            torch.cuda.synchronize()
            t_cold = time.perf_counter() - t0
            del st2
            rec = dict(block=blk, k=k, fees=g is not None, fee_records_rebuilt=rebuilt, update_ms=1e3 * t_upd,
                       warm_ms=1e3 * t_warm, warm_solver_ms=1e3 * r.wall_s, warm=(r.status, r.iters, r.evals, r.hvps),
                       build_ms=1e3 * t_build, cold_ms=1e3 * t_cold, cold_solver_ms=1e3 * rc.wall_s,
                       cold=(rc.status, rc.iters, rc.evals, rc.hvps), rel_value_diff=abs(r.value - rc.value) / abs(rc.value),
                       timed=rep > 0)
            recs.append(rec)
            print(f"block {blk:2d} k {k:6d} fees {'y' if g is not None else 'n'} (records {rebuilt:3d}): update "
                  f"{rec['update_ms']:7.3f} ms + warm solve {rec['warm_ms']:6.3f} ms {rec['warm']} | build "
                  f"{rec['build_ms']:6.3f} ms + cold solve {rec['cold_ms']:6.3f} ms {rec['cold']} | values differ "
                  f"{rec['rel_value_diff']:.1e}", flush=True)
            blk += 1
    print(f"\nmedians of the 9 timed blocks per k ({name}, power limit {limit}); tol {tol:g}, no trades")
    print(f"{'k':>7s} {'update':>9s} {'warm solve':>11s} {'(solver)':>9s} {'it/ev/hv':>9s} {'update path':>12s} | "
          f"{'build':>8s} {'cold solve':>11s} {'(solver)':>9s} {'it/ev/hv':>9s} {'rebuild path':>13s}")
    for k in (100, 10_000, 100_000):
        rs = [x for x in recs if x["k"] == k and x["timed"]]
        med = lambda key: float(np.median([x[key] for x in rs]))
        medi = lambda key, i: int(np.median([x[key][i] for x in rs]))
        upd_path = float(np.median([x["update_ms"] + x["warm_ms"] for x in rs]))
        reb_path = float(np.median([x["build_ms"] + x["cold_ms"] for x in rs]))
        print(f"{k:7d} {med('update_ms'):7.3f}ms {med('warm_ms'):9.3f}ms {med('warm_solver_ms'):7.3f}ms "
              f"{medi('warm', 1):3d}/{medi('warm', 2):2d}/{medi('warm', 3):2d} {upd_path:10.3f}ms | {med('build_ms'):6.3f}ms "
              f"{med('cold_ms'):9.3f}ms {med('cold_solver_ms'):7.3f}ms {medi('cold', 1):3d}/{medi('cold', 2):2d}/"
              f"{medi('cold', 3):2d} {reb_path:11.3f}ms")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(gpu=name, power_limit=limit, blocks=recs), f, indent=1)


if __name__ == "__main__":
    main()
