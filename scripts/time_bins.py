"""Time price-bin pools (k_eval_bins) against the same market written as one-bin pools (instances.bins_split).

The same seeded market (instances.synth_bins_market with every pool a bins pool: 60 % Liquidity-Book-like pools and
30 % order books of K bins, 10 % single limit orders) is built twice: as bins pools and as one one-bin pool per bin, for
K in --K.  For each form:
1. cfmm_arb_eval, plain and with trades and Hessian coefficients (eps = 1e-3, the smoothed form the solvers evaluate):
   CUDA-event medians over --reps launches after --warmup;
2. one cfmm_hvp after an evaluation with hess=True (CUDA-event median);
3. solve_pools (Arbitrage at prices 1 % off the market's) to tol 1e-6 through solver.py and through the native host
   loop (native="hostloop"): wall-clock median of 3 after a warm-up, with iterations, evaluations and Hessian-vector
   products.
The card's name and power limit are read in the same run and printed with the numbers.

    python scripts/time_bins.py [--pools 100000] [--tokens 1000] [--K 1,16,256] [--reps 30] [--warmup 5] [--json PATH]
Prints one line per measurement and a JSON summary line (also written to PATH with --json).
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
    ap.add_argument("--K", default="1,16,256")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    out = {"gpu": card()}
    print("card:", out["gpu"])
    for K in [int(k) for k in args.K.split(",")]:
        hp, prices = I.synth_bins_market(args.pools, args.tokens, seed=K, K=K, frac_lb=0.6, frac_book=0.3,
                                         frac_order=0.1)
        sp, _ = I.bins_split(hp)
        rng = np.random.default_rng(K)
        nu_h = prices * np.exp(0.01 * rng.standard_normal(args.tokens))
        nu = torch.as_tensor(nu_h, dtype=torch.float64, device="cuda")
        u = cf.Arbitrage(nu_h)
        for form, h in (("bins", hp), ("split", sp)):
            st = cf.PoolStore(h)
            name = f"K{K}_{form}"
            out[f"{name}_pools"], out[f"{name}_records"] = h.m, int(len(h.bin_rec))
            for trades, hess in ((False, False), (True, True)):
                us = _events(lambda: st.evaluate(nu, 1e-3, trades=trades, hess=hess), args.reps, args.warmup)
                key = f"{name}_eval{'_trades_hess' if trades else ''}_us"
                out[key] = us
                print(f"{key}: {us:.1f} us  ({h.m} pools, {len(h.bin_rec)} records)")
            st.evaluate(nu, 1e-3, trades=False, hess=True)
            v = torch.randn(args.tokens, dtype=torch.float64, device="cuda")
            us = _events(lambda: st.hvp(v), args.reps, args.warmup)
            out[f"{name}_hvp_us"] = us
            print(f"{name}_hvp: {us:.1f} us")
            for loop, native in (("solver_py", False), ("hostloop", "hostloop")):
                cf.solve_pools(h, u, tol=1e-6, store=st, want_trades=False, native=native)      # warm-up
                ws = []
                for _ in range(3):
                    torch.cuda.synchronize(); t0 = time.perf_counter()
                    r = cf.solve_pools(h, u, tol=1e-6, store=st, want_trades=False, native=native)
                    torch.cuda.synchronize(); ws.append(time.perf_counter() - t0)
                out[f"{name}_{loop}_solve_ms"] = 1e3 * float(np.median(ws))
                out[f"{name}_{loop}_solve_counts"] = [r.iters, r.evals, r.hvps, r.status, r.value]
                print(f"{name}_{loop}_solve: {1e3 * np.median(ws):.2f} ms  status={r.status} iters={r.iters} "
                      f"evals={r.evals} hvps={r.hvps} value={r.value:.12g}")
            del st
            torch.cuda.empty_cache()
    print(json.dumps(out))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
