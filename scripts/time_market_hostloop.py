"""Time solve_pools(native="hostloop") -- the C++ market loop, cfmm_market_solve -- against solver.py (native=False) on
mixed markets, alternated in one run, and the loop's dense Cholesky against torch.linalg.cholesky_ex.

    python scripts/time_market_hostloop.py [--reps 3] [--json results.json]

Markets: BASELINE configs[2] and [3] (synth_mixed(100_000, 1000, seed=1|2)), synth_concentrated_market(100_000, 1000),
synth_crypto_market(120_000, 400) and synth_tricrypto_market(120_000, 400), each under Arbitrage, Liquidate and Swap, to
1e-6.  Reports wall-clock medians, iterations, evaluations, HVPs and the max |difference| of value and nu, with the GPU's
name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cfmm_routing_code_b200 as cf                     # noqa: E402
from cfmm_routing_code_b200 import _lib, instances as I  # noqa: E402
from cfmm_routing_code_b200.pools import HostPools      # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def markets():
    s = I.synth_mixed(100_000, 1000, seed=1)
    yield "cfg2", HostPools(1000, s["pool_ptr"], s["tok_idx"], s["reserves"], s["weights"], s["gamma"], s["kind"]), s["prices"]
    s = I.synth_mixed(100_000, 1000, seed=2)
    yield "cfg3", HostPools(1000, s["pool_ptr"], s["tok_idx"], s["reserves"], s["weights"], s["gamma"], s["kind"]), s["prices"]
    yield ("concentrated",) + I.synth_concentrated_market(100_000, 1000, seed=1)
    yield ("crypto",) + I.synth_crypto_market(120_000, 400, seed=1)
    yield ("tricrypto",) + I.synth_tricrypto_market(120_000, 400, seed=1)


def utilities(n, prices):
    return [("arbitrage", cf.Arbitrage(prices), None),
            ("liquidate", cf.Liquidate(0, I.synth_basket(n, prices, seed=2)), prices / prices[0]),
            ("swap", cf.Swap(1, 0, 5e3 / prices[1]), prices / prices[0])]


def time_cholesky(n, reps=10):
    lib = _lib.load()
    rng = np.random.default_rng(n)
    B = torch.as_tensor(rng.standard_normal((n, n)), dtype=torch.float64, device="cuda")
    A = B @ B.T / n + torch.eye(n, dtype=torch.float64, device="cuda")
    work = torch.empty_like(A)
    info = torch.zeros(1, dtype=torch.float64, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = {}
    for name in ("native", "torch") * 2:                 # warm-up, then the timed pass
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(reps):
            work.copy_(A)
            e0.record()
            if name == "native":
                _lib.check(lib.cfmm_dense_cholesky(n, work.data_ptr(), info.data_ptr(), st), "cfmm_dense_cholesky")
            else:
                torch.linalg.cholesky_ex(work)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        out[name] = float(np.median(ts))
    assert float(info.item()) == 0.0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    rows = []
    info = gpu_info()
    print("GPU:", info, flush=True)
    for name, hp, prices in markets():
        store = cf.PoolStore(hp)
        for uname, u, nu0 in utilities(hp.n_tokens, prices):
            t = {"hostloop": [], "python": []}
            res = {}
            for rep in range(args.reps + 1):                   # the first round warms both paths up
                for impl, native in (("hostloop", "hostloop"), ("python", False)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    r = cf.solve_pools(hp, u, nu0=nu0, tol=1e-6, store=store, native=native, want_trades=False)
                    torch.cuda.synchronize()
                    if rep:
                        t[impl].append(time.perf_counter() - t0)
                    res[impl] = r
            a, b = res["hostloop"], res["python"]
            row = dict(market=name, utility=uname, m=hp.m, n=hp.n_tokens,
                       hostloop_ms=1e3 * float(np.median(t["hostloop"])), python_ms=1e3 * float(np.median(t["python"])),
                       status=(a.status, b.status), iters=(a.iters, b.iters), evals=(a.evals, b.evals),
                       hvps=(a.hvps, b.hvps), d_value_rel=abs(a.value - b.value) / max(abs(b.dual_value), 1e-300),
                       d_nu_rel=float(np.max(np.abs(a.nu - b.nu) / np.abs(b.nu))))
            rows.append(row)
            print(json.dumps(row), flush=True)
    chol = {n: time_cholesky(n) for n in (256, 1000, 4096)}
    for n, v in chol.items():
        print(f"cholesky n={n}: native {v['native']:.3f} ms, torch.linalg.cholesky_ex {v['torch']:.3f} ms", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(gpu=info, solves=rows, cholesky_ms=chol), f, indent=1)


if __name__ == "__main__":
    main()
