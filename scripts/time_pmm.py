"""Time DODO proactive-market-maker pools (PMM, k_eval_pair<CFMM_KIND_PMM>).

1. cfmm_arb_eval on --pools PMM pools, plain and with trades and Hessian coefficients, beside the same number of
   bounded-product pools on the same token pairs at the same prices, the two forms alternated launch by launch (CUDA-event
   medians over --reps after --warmup);
2. one cfmm_hvp after an evaluation with hess=True, both forms;
3. solve_pools of instances.synth_pmm_market(--market, --tokens) to tol 1e-6 through solver.py and the native host loop
   (native="hostloop"), for Arbitrage, Liquidate and Swap: wall-clock median of 3 after a warm-up, with the counts;
4. --quotes per-thread quotes (solve_batch, one Swap each) on the reference's arbitrage.py instance with three PMM pools.
The card's name and power limit are read in the same run and printed with the numbers.

    python scripts/time_pmm.py [--pools 1000000] [--market 100000] [--tokens 1000] [--quotes 4096] [--json PATH]
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
from cfmm_routing_code_b200.pools import HostPools, KIND_BOUNDED_HOST, KIND_PMM_HOST, PMM_K_MIN, pmm_targets  # noqa: E402
from time_eclp import _alternated                                    # noqa: E402
from time_stableswap_n import card                                   # noqa: E402


def pair_markets(m, n, seed):
    """m PMM pools and m bounded products (one v3 range each) on the same random token pairs, both around the market
    price: the PMM pools at their meeting point or a little off it on either piece, k log-uniform over [PMM_K_MIN, 1]"""
    rng = np.random.default_rng(seed)
    p = np.exp(rng.normal(0, 1, n))
    a = rng.integers(0, n, m)
    b = (a + rng.integers(1, n, m)) % n
    mid = p[a] / p[b]
    k = np.exp(rng.uniform(np.log(PMM_K_MIN), 0.0, m))
    Q0 = 1e4 / p[b]
    B0 = Q0 / mid
    side = rng.integers(0, 3, m)
    off = np.exp(np.abs(0.01 * rng.standard_normal(m)))
    B = np.where(side == 1, B0 * np.sqrt(k / (off - 1 + k)), B0)
    Q = np.where(side == 2, Q0 * np.sqrt(k / (off - 1 + k)), Q0)
    Q = np.where(side == 1, Q0 + mid * (B0 - B) * (1 + k * (B0 - B) / B), Q)
    B = np.where(side == 2, B0 + (Q0 - Q) * (1 + k * (Q0 - Q) / Q) / mid, B)
    R = np.stack([B, Q], axis=1)
    W = pmm_targets(R, np.stack([mid, k, np.where(side == 1, np.maximum(B0, np.nextafter(B, np.inf)), B0),
                                 np.where(side == 2, np.maximum(Q0, np.nextafter(Q, np.inf)), Q0)], axis=1))
    ptr = np.arange(0, 2 * m + 1, 2, dtype=np.int64)
    tok = np.stack([a, b], 1).reshape(-1).astype(np.int32)
    g = np.full(m, 0.997)
    pm = HostPools(n, ptr, tok, R.reshape(-1).copy(), np.zeros(2 * m), g, np.full(m, KIND_PMM_HOST, np.uint8), pmm=W)
    # the bounded product of the range [0.8, 1.25] x mid at about the same price and depth
    pc = mid
    Lq = np.sqrt(B * Q) + 1.0
    sp, sa, sb = np.sqrt(pc), np.sqrt(0.8 * mid), np.sqrt(1.25 * mid)
    Rb = np.stack([Lq * (1 / sp - 1 / sb), Lq * (sp - sa)], axis=1)
    off_b = np.stack([Lq / sb, Lq * sa], axis=1)
    bp = HostPools(n, ptr, tok, Rb.reshape(-1).copy(), off_b.reshape(-1).copy(), g,
                   np.full(m, KIND_BOUNDED_HOST, np.uint8))
    return pm, bp, p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=1_000_000)
    ap.add_argument("--market", type=int, default=100_000)
    ap.add_argument("--tokens", type=int, default=1000)
    ap.add_argument("--quotes", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    out = {"gpu": card()}
    print("card:", out["gpu"])
    pm, bp, p = pair_markets(args.pools, args.tokens, 1)
    sp, sb = cf.PoolStore(pm), cf.PoolStore(bp)
    nu = torch.as_tensor(p * np.exp(0.02 * np.random.default_rng(2).standard_normal(args.tokens)), device="cuda")
    out["eval_bytes_per_pool"] = {"pmm": sp.algorithmic_bytes_per_eval() // args.pools,
                                  "bounded": sb.algorithmic_bytes_per_eval() // args.pools}
    for trades, hess in ((False, False), (True, True)):
        tp, tb = _alternated(lambda: sp.evaluate(nu, trades=trades, hess=hess),
                             lambda: sb.evaluate(nu, trades=trades, hess=hess), args.reps, args.warmup)
        key = "eval_trades_hess" if trades else "eval"
        out[f"{key}_us"] = {"pmm": tp, "bounded": tb, "ratio": tp / tb}
        print(f"{key}: pmm {tp:.1f} us, bounded product {tb:.1f} us, ratio {tp / tb:.2f} ({args.pools} pools)")
    sp.evaluate(nu, hess=True); sb.evaluate(nu, hess=True)
    v = torch.randn(args.tokens, dtype=torch.float64, device="cuda")
    tp, tb = _alternated(lambda: sp.hvp(v), lambda: sb.hvp(v), args.reps, args.warmup)
    out["hvp_us"] = {"pmm": tp, "bounded": tb}
    print(f"hvp: pmm {tp:.1f} us, bounded product {tb:.1f} us")
    del sp, sb
    torch.cuda.empty_cache()

    hp, prices = I.synth_pmm_market(args.market, args.tokens, 3)
    st = cf.PoolStore(hp)
    n = args.tokens
    assets = np.zeros(n); assets[1:6] = 1e3 / prices[1:6]
    utils = {"arbitrage": cf.Arbitrage(prices * np.exp(0.01 * np.random.default_rng(4).standard_normal(n))),
             "liquidate": cf.Liquidate(0, assets), "swap": cf.Swap(1, 0, 10.0 / prices[1])}
    for uname, u in utils.items():
        for loop, native in (("solver_py", False), ("hostloop", "hostloop")):
            cf.solve_pools(hp, u, tol=1e-6, store=st, want_trades=False, native=native)
            ws = []
            for _ in range(3):
                torch.cuda.synchronize(); t0 = time.perf_counter()
                r = cf.solve_pools(hp, u, tol=1e-6, store=st, want_trades=False, native=native)
                torch.cuda.synchronize(); ws.append(time.perf_counter() - t0)
            out[f"solve_{uname}_{loop}_ms"] = 1e3 * float(np.median(ws))
            out[f"solve_{uname}_{loop}_counts"] = [r.iters, r.evals, r.hvps, r.status, r.value]
            print(f"solve {uname} {loop}: {1e3 * np.median(ws):.1f} ms status={r.status} iters={r.iters} "
                  f"evals={r.evals} hvps={r.hvps} value={r.value:.12g}")
    del st
    torch.cuda.empty_cache()

    d = I.arbitrage_instance()
    mv = np.asarray(d["market_value"], float)
    li, res, fees, kinds, wts = (list(d[k]) for k in ("local_indices", "reserves", "fees", "kinds", "weights"))
    for (i, j), kk in zip(((0, 1), (1, 2), (0, 2)), (1e-3, 0.1, 1.0)):
        q = mv[i] / mv[j]
        li.append([i, j]); res.append([20.0, 20.0 * q]); fees.append(0.997); kinds.append("pmm")
        wts.append((q, kk, 20.0, 20.0 * q))
    hq = HostPools.from_lists(len(mv), li, res, fees, kinds, wts)
    qs = [cf.Swap(1, 0, t) for t in np.linspace(0.01, 5.0, args.quotes)]
    cf.solve_batch(hq, qs[:64], tol=1e-8)
    ws = []
    for _ in range(3):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        rs = cf.solve_batch(hq, qs, tol=1e-8)
        torch.cuda.synchronize(); ws.append(time.perf_counter() - t0)
    out["quotes_ms"] = 1e3 * float(np.median(ws))
    out["quotes_optimal"] = sum(r.status == "optimal" for r in rs)
    print(f"{args.quotes} per-thread quotes: {1e3 * np.median(ws):.1f} ms, {out['quotes_optimal']} optimal")
    print(json.dumps(out))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
