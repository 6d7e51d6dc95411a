"""Time the three-coin cryptoswap evaluation kernel, one HVP and a mixed-market solve.

1. cfmm_arb_eval on 1M three-coin cryptoswap pools (kind 9) near their peg (balances within 3 % of the price scales)
   and far from it (each coin 2x .. 30x off), next to 1M two-coin cryptoswap pools (kind 8) whose two balances are off
   by the same factors, plain and with trades and Hessian coefficients: CUDA-event medians over --reps launches after
   --warmup.
2. One HVP (cfmm_hvp) on each 1M-pool bucket.
3. solve_pools on instances.synth_tricrypto_market (three-coin pools beside every other kind) under Arbitrage,
   Liquidate and Swap at tol 1e-6: wall time, iterations, evaluations.

    python scripts/time_tricrypto.py [--pools 1000000] [--tokens 2000] [--reps 50] [--warmup 10]
Prints one line per measurement and a JSON summary line (with the card's name, power limit and SM clock).
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


def stores(m, n, seed=0):
    """1M-pool plain buckets on one random token graph: three-coin cryptoswap pools (A in {0.1, 1, 6.3, 50}, curve gamma
    in {1.45e-4, 2e-3, 2e-2}) with scaled balances near their peg and far from it, and two-coin cryptoswap pools with the
    same parameters whose first two coins carry the same balance offsets"""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, n, m); b = (a + rng.integers(1, n, m)) % n; c = (b + rng.integers(1, n - 1, m)) % n
    c = np.where(c == a, (c + 1) % n, c)
    g = np.array([0.9995, 0.9974, 0.9955])[rng.integers(0, 3, m)]
    A = np.array([0.1, 1.0, 6.3, 50.0])[rng.integers(0, 4, m)]
    G = np.array([1.45e-4, 2e-3, 2e-2])[rng.integers(0, 3, m)]
    p = np.exp(rng.standard_normal(n))
    V = np.exp(8 + 1.5 * rng.standard_normal(m))
    out = []
    for name, k in (("peg", np.exp(rng.uniform(-0.03, 0.03, (m, 3)))),
                    ("far", np.exp(rng.choice([-1, 1], (m, 3)) * rng.uniform(np.log(2), np.log(30), (m, 3))))):
        tok3 = np.stack([a, b, c], 1)
        R3 = V[:, None] * k / p[tok3]
        t3 = PL.HostPools(n, np.arange(0, 3 * m + 1, 3, dtype=np.int64), tok3.astype(np.int32).ravel(), R3.ravel(),
                          p[tok3].ravel(), g, np.full(m, PL.KIND_CRYPTOSWAP_HOST, np.uint8), A, cgam=G)
        out.append((f"tricrypto_{name}", PL.PoolStore(t3, layout="plain"), p))
        del t3
        tok2 = tok3[:, :2]
        t2 = PL.HostPools(n, np.arange(0, 2 * m + 1, 2, dtype=np.int64), tok2.astype(np.int32).ravel(),
                          R3[:, :2].ravel(), p[tok2].ravel(), g, np.full(m, PL.KIND_CRYPTOSWAP_HOST, np.uint8), A, cgam=G)
        out.append((f"cryptoswap_{name}", PL.PoolStore(t2, layout="plain"), p))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=1_000_000)
    ap.add_argument("--tokens", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--mixed-pools", type=int, default=120_000)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi}
    print(f"GPU: {smi}")
    rng = np.random.default_rng(1)
    for name, st, p in stores(args.pools, args.tokens):
        nu = torch.as_tensor(p * np.exp(0.01 * rng.standard_normal(args.tokens)), dtype=torch.float64, device="cuda")
        for trades, hess in ((False, False), (True, True)):
            us = _events(lambda: st.evaluate(nu, 0.0, trades=trades, hess=hess), args.reps, args.warmup)
            key = f"{name}_eval{'_trades_hess' if trades else ''}_us"
            out[key] = us
            print(f"{key}: {us:.1f} us  ({args.pools} pools, {args.tokens} tokens)")
        vt = torch.randn(args.tokens, dtype=torch.float64, device="cuda")
        us = _events(lambda: st.hvp(vt), args.reps, args.warmup)
        out[f"{name}_hvp_us"] = us
        print(f"{name}_hvp_us: {us:.1f} us")
        del st
        torch.cuda.empty_cache()
    hp, prices = I.synth_tricrypto_market(args.mixed_pools, 400, seed=4)
    store = cf.PoolStore(hp)
    n3 = int(((hp.kind == PL.KIND_CRYPTOSWAP_HOST) & (np.diff(hp.pool_ptr) == 3)).sum())
    rng = np.random.default_rng(1)
    basket = np.zeros(hp.n_tokens)
    for j in rng.choice(np.arange(1, hp.n_tokens), 8, replace=False):
        basket[j] = float(np.exp(rng.normal(1, 1)) * 100 / prices[j])
    utils = {"arbitrage": cf.Arbitrage(prices * np.exp(0.01 * rng.standard_normal(hp.n_tokens))),
             "liquidate": cf.Liquidate(0, basket), "swap": cf.Swap(1, 3, 5e3 / prices[1])}
    for name, u in utils.items():
        cf.solve_pools(hp, u, tol=1e-6, store=store, want_trades=False)          # warm-up (first launches, allocations)
        ws = []
        for _ in range(3):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            r = cf.solve_pools(hp, u, tol=1e-6, store=store, want_trades=False)
            torch.cuda.synchronize(); ws.append(time.perf_counter() - t0)
        out[f"mixed_{name}_ms"] = 1e3 * float(np.median(ws))
        print(f"mixed {name}: {1e3 * np.median(ws):.2f} ms  status={r.status} iters={r.iters} evals={r.evals} "
              f"hvps={r.hvps}  ({hp.m} pools: {n3} three-coin cryptoswap)")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
