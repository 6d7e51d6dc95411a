"""Time the n-coin StableSwap evaluation kernel (k_eval_stable_n), its Hessian-vector product and mixed-market solves.

1. cfmm_arb_eval on --pools 3-coin and 4-coin StableSwap pools (kind 5), near their peg (tokens worth 1 +- 0.2 %,
   balances within ~2x of value-balanced: the representative case) and far off it (token prices differing by factors
   of ~e), next to the same number of 2-coin pools (kind 4, k_eval_stable) on the same token graph, with and without
   trades / Hessian coefficients: CUDA-event medians over --reps launches after --warmup.
2. One cfmm_hvp on each n-coin bucket, after an evaluation with hess=True (CUDA-event median).
3. solve_pools on instances.synth_stable_n_market (product pools plus 2-, 3- and 4-coin StableSwap pools) under
   Arbitrage, Liquidate and Swap at tol 1e-8, with solver.py's dense and CG linear solvers: wall-clock medians of 3
   after a warm-up, iterations and evaluations.
The card's name and power limit are read in the same run and printed with the numbers.

    python scripts/time_stableswap_n.py [--pools 1000000] [--tokens 2000] [--reps 30] [--warmup 5]
Prints one line per measurement and a JSON summary line.
"""
import argparse
import json
import os
import subprocess
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                   # the name from torch at least
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({type(e).__name__})"
    return q


def stores(m, n, k, peg, seed=0):
    """a plain bucket of m StableSwap pools of k coins on one random token graph, and the token prices"""
    rng = np.random.default_rng(seed)
    toks = np.stack([rng.choice(n, k, replace=False) for _ in range(min(m, 4096))])
    toks = toks[rng.integers(0, len(toks), m)] if m > len(toks) else toks
    toks = (toks + rng.integers(0, n, m)[:, None]) % n                  # spread over the graph, still distinct per pool
    g = np.array([0.9996, 0.9999, 0.99995])[rng.integers(0, 3, m)]
    A = np.array([100.0, 1000.0, 2e4])[rng.integers(0, 3, m)] / float(k ** k)
    V = np.exp(8 + 1.5 * rng.standard_normal(m))
    if peg:
        p = np.exp(0.002 * rng.uniform(-1, 1, n))
        R = V[:, None] * np.exp(0.35 * rng.standard_normal((m, k))) / p[toks]
    else:
        p = np.exp(rng.standard_normal(n))
        R = V[:, None] / p[toks] * np.exp(0.02 * rng.standard_normal((m, k)))
        p = p * np.exp(0.3 * rng.standard_normal(n))                    # far from the pools' balance
    hp = PL.HostPools(n, np.arange(0, k * m + 1, k, dtype=np.int64), toks.astype(np.int32).ravel(), R.ravel(),
                      np.ones(k * m), g, np.full(m, PL.KIND_STABLESWAP_HOST, np.uint8), A)
    return PL.PoolStore(hp, layout="plain"), p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=1_000_000)
    ap.add_argument("--tokens", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--mixed-pools", type=int, default=120_000)
    args = ap.parse_args()
    out = {"gpu": card()}
    print("card:", out["gpu"])
    rng = np.random.default_rng(1)
    for peg in (True, False):
        for k in (2, 3, 4):
            st, p = stores(args.pools, args.tokens, k, peg)
            nu = torch.as_tensor(p * np.exp(0.001 * rng.standard_normal(args.tokens)), dtype=torch.float64, device="cuda")
            name = f"k{k}_{'peg' if peg else 'offpeg'}"
            for trades, hess in ((False, False), (True, True)):
                us = _events(lambda: st.evaluate(nu, 0.0, trades=trades, hess=hess), args.reps, args.warmup)
                key = f"{name}_eval{'_trades_hess' if trades else ''}_us"
                out[key] = us
                print(f"{key}: {us:.1f} us  ({args.pools} pools of {k} coins, bucket kind {st.buckets[0].kind})")
            if k > 2:
                st.evaluate(nu, 0.0, trades=False, hess=True)
                v = torch.randn(args.tokens, dtype=torch.float64, device="cuda")
                us = _events(lambda: st.hvp(v), args.reps, args.warmup)
                out[f"{name}_hvp_us"] = us
                print(f"{name}_hvp: {us:.1f} us")
            del st
            torch.cuda.empty_cache()
    s = I.synth_stable_n_market(args.mixed_pools, 400, seed=4)
    prices = s.pop("prices")
    hp = PL.HostPools(**s)
    store = cf.PoolStore(hp)
    rng = np.random.default_rng(1)
    basket = np.zeros(hp.n_tokens)
    for j in rng.choice(np.arange(1, hp.n_tokens), 6, replace=False):
        basket[j] = float(np.exp(rng.normal(1, 1)) * 100 / prices[j])
    utils = {"arbitrage": cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(hp.n_tokens))),
             "liquidate": cf.Liquidate(0, basket), "swap": cf.Swap(1, 3, 5e3 / prices[1])}
    ar = np.diff(hp.pool_ptr)[hp.kind == PL.KIND_STABLESWAP_HOST]
    for ls in ("dense", "cg"):
        for name, u in utils.items():
            cf.solve_pools(hp, u, tol=1e-8, store=store, want_trades=False, linear_solver=ls)     # warm-up
            ws = []
            for _ in range(3):
                torch.cuda.synchronize(); t0 = time.perf_counter()
                r = cf.solve_pools(hp, u, tol=1e-8, store=store, want_trades=False, linear_solver=ls)
                torch.cuda.synchronize(); ws.append(time.perf_counter() - t0)
            out[f"mixed_{ls}_{name}_ms"] = 1e3 * float(np.median(ws))
            print(f"mixed {ls} {name}: {1e3 * np.median(ws):.2f} ms  status={r.status} iters={r.iters} evals={r.evals} "
                  f"hvps={r.hvps}  ({hp.m} pools; StableSwap of 2/3/4 coins: "
                  f"{(ar == 2).sum()}/{(ar == 3).sum()}/{(ar == 4).sum()})")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
