"""Time concentrated-liquidity pools (k_eval_ladder) against the same market written as ranges (k_eval_pair, kind 3).

The same seeded market (instances.synth_concentrated_market with every pool a ladder: --pools ladders of T intervals,
~10 % of them empty) is built twice: as ladder pools (kind 6) and as its non-empty intervals, one bounded_product pool
each (instances.ladder_ranges), for T in --T.  For each form:
1. cfmm_arb_eval, plain and with trades and Hessian coefficients: CUDA-event medians over --reps launches after --warmup;
2. one cfmm_hvp after an evaluation with hess=True (CUDA-event median);
3. solve_pools (Arbitrage at prices 1 % off the market's) to tol 1e-6 through solver.py: wall-clock median of 3 after a
   warm-up, with iterations, evaluations and Hessian-vector products.
The card's name and power limit are read in the same run and printed with the numbers.

    python scripts/time_concentrated.py [--pools 100000] [--tokens 1000] [--T 1,16,256] [--reps 30] [--warmup 5]
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
from cfmm_routing_code_b200 import instances as I                    # noqa: E402
from time_stableswap_n import _events, card                          # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=100_000)
    ap.add_argument("--tokens", type=int, default=1000)
    ap.add_argument("--T", default="1,16,256")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    out = {"gpu": card()}
    print("card:", out["gpu"])
    for T in [int(t) for t in args.T.split(",")]:
        hp, prices = I.synth_concentrated_market(args.pools, args.tokens, seed=T, T=T, frac_ladder=1.0)
        rg, _ = I.ladder_ranges(hp)
        rng = np.random.default_rng(T)
        nu_h = prices * np.exp(0.01 * rng.standard_normal(args.tokens))
        nu = torch.as_tensor(nu_h, dtype=torch.float64, device="cuda")
        u = cf.Arbitrage(nu_h)
        for form, h in (("ladder", hp), ("ranges", rg)):
            st = cf.PoolStore(h)
            kinds = sorted({int(b.kind) for b in st.buckets})
            name = f"T{T}_{form}"
            for trades, hess in ((False, False), (True, True)):
                us = _events(lambda: st.evaluate(nu, 0.0, trades=trades, hess=hess), args.reps, args.warmup)
                key = f"{name}_eval{'_trades_hess' if trades else ''}_us"
                out[key] = us
                print(f"{key}: {us:.1f} us  ({h.m} pools, bucket kinds {kinds})")
            st.evaluate(nu, 0.0, trades=False, hess=True)
            v = torch.randn(args.tokens, dtype=torch.float64, device="cuda")
            us = _events(lambda: st.hvp(v), args.reps, args.warmup)
            out[f"{name}_hvp_us"] = us
            print(f"{name}_hvp: {us:.1f} us")
            cf.solve_pools(h, u, tol=1e-6, store=st, want_trades=False)             # warm-up
            ws = []
            for _ in range(3):
                torch.cuda.synchronize(); t0 = time.perf_counter()
                r = cf.solve_pools(h, u, tol=1e-6, store=st, want_trades=False)
                torch.cuda.synchronize(); ws.append(time.perf_counter() - t0)
            out[f"{name}_solve_ms"] = 1e3 * float(np.median(ws))
            out[f"{name}_solve_counts"] = [r.iters, r.evals, r.hvps, r.status]
            print(f"{name}_solve: {1e3 * np.median(ws):.2f} ms  status={r.status} iters={r.iters} evals={r.evals} "
                  f"hvps={r.hvps}")
            del st
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
