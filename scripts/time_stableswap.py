"""Time the StableSwap evaluation kernel and a mixed-market solve.

1. cfmm_arb_eval on 1M StableSwap pools near their peg (the representative case) and far off it, against 1M product
   pools in a plain bucket, with and without trades / Hessian coefficients: CUDA-event medians over --reps launches
   after --warmup.
2. solve_pools on the mixed market of tests/test_stableswap.py (instances.synth_stable_market: product, weighted and
   StableSwap pools) under Arbitrage, Liquidate and Swap at tol 1e-8: wall time, iterations, evaluations.

    python scripts/time_stableswap.py [--pools 1000000] [--tokens 2000] [--reps 50] [--warmup 10]
Prints one line per measurement and a JSON summary line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cfmm_routing_code_b200 as cf                                   # noqa: E402
from cfmm_routing_code_b200 import instances as I, pools as PL     # noqa: E402


def _events(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts))


def stores(m, n, seed=0):
    """1M-pool plain buckets on one random pair graph: StableSwap pools near their peg (tokens worth 1 +- 0.2 %, balances
    within ~2x of value-balanced, A in {50, 200, 2000}, rates 1: the representative case; there the curve is flat and
    each trading pool's Newton solve works hardest), the same StableSwap pools with reserves of tokens whose prices
    differ by factors of ~e (far off peg: large trades on the curved part), and constant-product pools with those
    reserves."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, n, m); b = (a + rng.integers(1, n, m)) % n
    g = np.array([0.9996, 0.9999, 0.997])[rng.integers(0, 3, m)]
    A = np.array([50.0, 200.0, 2000.0])[rng.integers(0, 3, m)]
    ptr = np.arange(0, 2 * m + 1, 2, dtype=np.int64)
    tok = np.stack([a, b], 1).astype(np.int32).ravel()
    V = np.exp(8 + 1.5 * rng.standard_normal(m))
    p_peg = np.exp(0.002 * rng.uniform(-1, 1, n))
    k = np.exp(0.35 * rng.standard_normal(m))
    R_peg = np.stack([V * k / p_peg[a], V / k / p_peg[b]], 1)
    p_far = np.exp(rng.standard_normal(n))
    R_far = np.stack([V / p_far[a], V / p_far[b]], 1) * np.exp(0.02 * rng.standard_normal((m, 2)))
    ss = lambda R: PL.HostPools(n, ptr, tok, R.ravel(), np.ones(2 * m), g, np.full(m, PL.KIND_STABLESWAP_HOST, np.uint8), A)
    cp = PL.HostPools(n, ptr, tok, R_far.ravel(), np.full(2 * m, 0.5), g, np.zeros(m, np.uint8))
    return [("stableswap_peg", PL.PoolStore(ss(R_peg), layout="plain"), p_peg),
            ("stableswap_offpeg", PL.PoolStore(ss(R_far), layout="plain"), p_far),
            ("product_plain", PL.PoolStore(cp, layout="plain"), p_far)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=1_000_000)
    ap.add_argument("--tokens", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--mixed-pools", type=int, default=120_000)
    args = ap.parse_args()
    out = {"gpu": torch.cuda.get_device_name(0)}
    rng = np.random.default_rng(1)
    for name, st, p in stores(args.pools, args.tokens):
        nu = torch.as_tensor(p * np.exp(0.01 * rng.standard_normal(args.tokens)), dtype=torch.float64, device="cuda")
        for trades, hess in ((False, False), (True, True)):
            us = _events(lambda: st.evaluate(nu, 0.0, trades=trades, hess=hess), args.reps, args.warmup)
            key = f"{name}_eval{'_trades_hess' if trades else ''}_us"
            out[key] = us
            print(f"{key}: {us:.1f} us  ({args.pools} pools, {args.tokens} tokens)")
        del st
        torch.cuda.empty_cache()
    s = I.synth_stable_market(args.mixed_pools, 400, seed=4)
    prices = s.pop("prices")
    hp = PL.HostPools(**s)
    store = cf.PoolStore(hp)
    rng = np.random.default_rng(1)
    basket = np.zeros(hp.n_tokens)
    for j in rng.choice(np.arange(1, hp.n_tokens), 8, replace=False):
        basket[j] = float(np.exp(rng.normal(1, 1)) * 100 / prices[j])
    utils = {"arbitrage": cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(hp.n_tokens))),
             "liquidate": cf.Liquidate(0, basket), "swap": cf.Swap(1, 3, 5e3 / prices[1])}
    for name, u in utils.items():
        cf.solve_pools(hp, u, tol=1e-8, store=store, want_trades=False)          # warm-up (first launches, allocations)
        ws = []
        for _ in range(3):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            r = cf.solve_pools(hp, u, tol=1e-8, store=store, want_trades=False)
            torch.cuda.synchronize(); ws.append(time.perf_counter() - t0)
        out[f"mixed_{name}_ms"] = 1e3 * float(np.median(ws))
        print(f"mixed {name}: {1e3 * np.median(ws):.2f} ms  status={r.status} iters={r.iters} evals={r.evals} "
              f"hvps={r.hvps}  ({hp.m} pools: {int((hp.kind == 4).sum())} StableSwap)")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
