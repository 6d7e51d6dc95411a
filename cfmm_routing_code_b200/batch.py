"""Batches of small routing problems: every ``prob.solve()`` of the batch in ONE kernel launch.

The reference solves its problems one at a time and, for the sweep of two-asset.py:40-100, rebuilds the cvxpy problem
for each of the 50 trade sizes.  Here the pools (the literals of two-asset.py:5-31) are uploaded once as CSR arrays and
``cfmm_batch_solve`` (csrc/cfmm_small.cu) runs one complete dual solve per GPU thread.  Nothing here has a CPU path.
"""
from __future__ import annotations

import ctypes as C
import time
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .pools import HostPools, KIND_BINS_HOST, KIND_CONCENTRATED_HOST, KIND_CRYPTOSWAP_HOST, KIND_ECLP_HOST, \
    KIND_GEOMEAN_HOST, KIND_PMM_HOST, KIND_STABLESWAP_HOST
from .solver import default_nu0

NTOK_MAX = 64      # cfmm_small::NTOK_MAX
ARITY_MAX = 8      # cfmm_small::KMAX


def batch_applicable(hp: HostPools) -> bool:
    """Whether the per-thread solver covers this pool set (token count and arities of the reference's instances do)."""
    if hp.n_tokens > NTOK_MAX or hp.m == 0:
        return False
    return int(np.diff(hp.pool_ptr).max()) <= ARITY_MAX


class CsrStore:
    """The CSR pool arrays in HBM (what `local_indices`, `reserves`, `fees` of arbitrage.py:6-28 become)."""

    def __init__(self, hp: HostPools, device="cuda"):
        if not torch.cuda.is_available():
            raise _lib.CfmmError("cfmm_routing_code_b200 needs a CUDA device (there is no CPU fallback)")
        hp.validate()
        if not batch_applicable(hp):
            raise ValueError(f"the batched solver takes at most {NTOK_MAX} tokens and arity <= {ARITY_MAX}")
        self.lib = _lib.load()
        self.hp, self.device = hp, torch.device(device)
        self.n_tokens, self.m, self.nnz = hp.n_tokens, hp.m, int(len(hp.tok_idx))
        dev = self.device
        per_slot_kind = np.repeat(np.asarray(hp.kind), np.diff(hp.pool_ptr))
        w = np.where(per_slot_kind == KIND_GEOMEAN_HOST, hp.weights, 1.0)      # log(R/w) is a weighted-pool quantity
        self.pool_ptr = torch.as_tensor(np.ascontiguousarray(hp.pool_ptr, np.int64), device=dev)
        self.tok = torch.as_tensor(np.ascontiguousarray(hp.tok_idx, np.int32), device=dev)
        self.R = torch.as_tensor(np.ascontiguousarray(hp.reserves, np.float64), device=dev)
        self.w = torch.as_tensor(np.ascontiguousarray(hp.weights, np.float64), device=dev)
        self.logrw = torch.log(torch.clamp(self.R, min=1e-300) / torch.as_tensor(w, device=dev))
        ss = np.nonzero(np.asarray(hp.kind) == KIND_STABLESWAP_HOST)[0]
        self.has_stableswap = bool(len(ss))         # -> cfmm_batch_solve_stableswap (its own kernel instance)
        # pools of more than two coins -> cfmm_batch_solve_stableswap_n (a third instance, which takes every arity)
        self.has_stableswap_n = bool(len(ss)) and bool(np.any(np.diff(np.asarray(hp.pool_ptr))[ss] > 2))
        if len(ss):                                  # StableSwap pools: A at the first slot, the invariant D at the second
            first = torch.as_tensor(np.asarray(hp.pool_ptr)[ss], device=dev)
            self.logrw[first] = torch.as_tensor(np.asarray(hp.amp, np.float64)[ss], device=dev)
            self.logrw[first + 1] = torch.as_tensor(np.asarray(hp.inv, np.float64)[ss], device=dev)
        cl = np.nonzero(np.asarray(hp.kind) == KIND_CONCENTRATED_HOST)[0]
        self.has_ladder = bool(len(cl))              # -> cfmm_batch_solve_concentrated (a fourth instance)
        self.records = None
        if len(cl):                                  # concentrated pools: (s, c) in the w slots, (first record, T) in logrw
            first = torch.as_tensor(np.asarray(hp.pool_ptr)[cl], device=dev)
            lp = np.asarray(hp.lad_ptr, np.int64)
            sc = np.asarray(hp.lad_sc, np.float64)[cl]
            self.w[first] = torch.as_tensor(sc[:, 0], device=dev)
            self.w[first + 1] = torch.as_tensor(sc[:, 1], device=dev)
            self.logrw[first] = torch.as_tensor(lp[cl].astype(np.float64), device=dev)
            self.logrw[first + 1] = torch.as_tensor((lp[cl + 1] - lp[cl] - 1).astype(np.float64), device=dev)
            self.records = torch.as_tensor(np.ascontiguousarray(hp.lad_rec, np.float64).reshape(-1), device=dev)
        bn = np.nonzero(np.asarray(hp.kind) == KIND_BINS_HOST)[0]
        self.has_bins = bool(len(bn))                # -> cfmm_batch_solve_bins (a seventh instance)
        if len(bn):                                  # bins pools: (z, p_ref) in the w slots, (first record, nb) in logrw;
            first = torch.as_tensor(np.asarray(hp.pool_ptr)[bn], device=dev)   # their records after the ladders'
            bp = np.asarray(hp.bin_ptr, np.int64)
            n_lad = len(np.asarray(hp.lad_rec).reshape(-1, 4))
            zp = np.asarray(hp.bin_zp, np.float64)[bn]
            self.w[first] = torch.as_tensor(zp[:, 0], device=dev)
            self.w[first + 1] = torch.as_tensor(zp[:, 1], device=dev)
            self.logrw[first] = torch.as_tensor((bp[bn] + n_lad).astype(np.float64), device=dev)
            self.logrw[first + 1] = torch.as_tensor((bp[bn + 1] - bp[bn]).astype(np.float64), device=dev)
            self.records = torch.as_tensor(np.concatenate([np.asarray(hp.lad_rec, np.float64).reshape(-1),
                                                           np.asarray(hp.bin_rec, np.float64).reshape(-1)]), device=dev)
        ec = np.nonzero(np.asarray(hp.kind) == KIND_ECLP_HOST)[0]
        self.has_eclp = bool(len(ec))                # -> cfmm_batch_solve_eclp (an eighth instance)
        if len(ec):                                  # E-CLP pools: one record {c, s, lam, alpha, beta, r, p, 0} each after
            lad = np.asarray(hp.lad_rec, np.float64).reshape(-1)      # the ladders' and bins' records, its index (units
            bns = np.asarray(hp.bin_rec, np.float64).reshape(-1)      # of 4 f64) in the pool's first logrw slot
            E = np.asarray(hp.eclp, np.float64)[ec]
            rec = np.zeros((len(ec), 8))
            rec[:, 0:3], rec[:, 3:5], rec[:, 5:7] = E[:, 2:5], E[:, 0:2], E[:, 5:7]
            first = torch.as_tensor(np.asarray(hp.pool_ptr)[ec], device=dev)
            at = (len(lad) + len(bns)) // 4 + 2 * np.arange(len(ec))
            self.logrw[first] = torch.as_tensor(at.astype(np.float64), device=dev)
            self.records = torch.as_tensor(np.concatenate([lad, bns, rec.reshape(-1)]), device=dev)
        pm = np.nonzero(np.asarray(hp.kind) == KIND_PMM_HOST)[0]
        self.has_pmm = bool(len(pm))                 # -> cfmm_batch_solve_pmm (a ninth instance)
        if len(pm):                                  # PMM pools: one record {pi, k, B0, Q0} each after every record
            prev = torch.zeros(0, dtype=torch.float64, device=dev) if self.records is None else self.records   # above,
            first = torch.as_tensor(np.asarray(hp.pool_ptr)[pm], device=dev)    # its index in the first logrw slot
            self.logrw[first] = torch.as_tensor((prev.numel() // 4 + np.arange(len(pm))).astype(np.float64), device=dev)
            self.records = torch.cat([prev, torch.as_tensor(np.asarray(hp.pmm, np.float64)[pm].reshape(-1), device=dev)])
        cs = np.nonzero(np.asarray(hp.kind) == KIND_CRYPTOSWAP_HOST)[0]
        ptr = np.asarray(hp.pool_ptr, np.int64)
        c3 = cs[ptr[cs + 1] - ptr[cs] == 3]
        self.has_crypto = bool(len(cs))              # -> cfmm_batch_solve_cryptoswap (a fifth instance)
        self.has_crypto3 = bool(len(c3))             # -> cfmm_batch_solve_tricrypto (a sixth instance)
        if len(cs):                                  # cryptoswap pools: p_j / D in the w slots, (A, G) in logrw
            first = ptr[cs]
            Dv = np.asarray(hp.inv, np.float64)[cs]
            W = np.asarray(hp.weights, np.float64)
            fd = torch.as_tensor(first, device=dev)
            self.w[fd] = torch.as_tensor(W[first] / Dv, device=dev)
            self.w[fd + 1] = torch.as_tensor(W[first + 1] / Dv, device=dev)
            if len(c3):                              # the third coin of the three-coin pools
                self.w[torch.as_tensor(ptr[c3] + 2, device=dev)] = torch.as_tensor(W[ptr[c3] + 2] / np.asarray(hp.inv)[c3],
                                                                                   device=dev)
            self.logrw[fd] = torch.as_tensor(np.asarray(hp.amp, np.float64)[cs], device=dev)
            self.logrw[fd + 1] = torch.as_tensor(np.asarray(hp.cgam, np.float64)[cs], device=dev)
        self.gamma = torch.as_tensor(np.ascontiguousarray(hp.gamma, np.float64), device=dev)
        kind = np.array(hp.kind, np.uint8)
        kind[c3] = _lib.KIND_CRYPTOSWAP_3            # three-coin cryptoswap pools are kind 9 in the C ABI
        self.kind = torch.as_tensor(kind, device=dev)
        self.c_pools = _lib.CsrPools(self.n_tokens, self.m, self.nnz, self.pool_ptr.data_ptr(), self.tok.data_ptr(),
                                     self.R.data_ptr(), self.w.data_ptr(), self.logrw.data_ptr(),
                                     self.gamma.data_ptr(), self.kind.data_ptr())
        self._work = None

    def work(self, n_problems: int, nnz_max: int = 0) -> torch.Tensor:
        nbytes = self.lib.cfmm_batch_solve_work_bytes(C.byref(self.c_pools), n_problems, nnz_max)
        if nbytes < 0:
            _lib.check(int(nbytes), "cfmm_batch_solve_work_bytes")
        if self._work is None or self._work.numel() < nbytes:
            self._work = torch.empty(max(int(nbytes), 8), dtype=torch.uint8, device=self.device)
        return self._work


SMALL_BATCH = 512            # up to this many problems a warp per problem beats a thread per problem
LANES_SMALL_BATCH = 32


@torch.no_grad()
def solve_batch_device(store: CsrStore, c: torch.Tensor, a: torch.Tensor, flags: torch.Tensor, nu: torch.Tensor,
                       tol: float = 1e-8, want_trades: bool = True, pool_range: Optional[torch.Tensor] = None,
                       max_outer: int = 60, max_inner: int = 100, nnz_max: int = 0, lanes: Optional[int] = None):
    """Device-resident form: c, a [B, n] f64, flags [B, n] u8, nu [B, n] f64 (start prices, overwritten with the
    solution).  Returns (psi [B, n], stats [B, 8], delta, lambda [B, nnz] or None).  Asynchronous on the current stream.
    pool_range [B, 2] int64 (device): problem p uses pools [lo, hi) -- disjoint problems packed into one CSR array; then
    delta / lambda are [1, nnz] and nnz_max (slots of the largest problem) sizes the workspace."""
    B, n = c.shape
    if n != store.n_tokens:
        raise ValueError("utilities must have one entry per token")
    dev = store.device
    f64 = dict(dtype=torch.float64, device=dev)
    psi = torch.empty(B, n, **f64)
    stats = torch.empty(B, 8, **f64)
    shared = pool_range is None
    delta = lam = None
    if want_trades:
        delta = torch.zeros(B if shared else 1, store.nnz, **f64)
        lam = torch.zeros(B if shared else 1, store.nnz, **f64)
    if lanes is None:
        # a problem per warp for small batches (latency: a sweep of 50 problems spreads over more lanes), a problem
        # per thread for large ones (throughput: thousands of problems fill the GPU either way)
        lanes = LANES_SMALL_BATCH if B <= SMALL_BATCH else 1
    _lib.check(store.lib.cfmm_set_batch_lanes(int(lanes)), "cfmm_set_batch_lanes")
    work = store.work(B, nnz_max)
    batch = _lib.Batch(B, None if shared else pool_range.data_ptr(), c.data_ptr(), a.data_ptr(), flags.data_ptr(),
                       nu.data_ptr(), psi.data_ptr(), stats.data_ptr(),
                       delta.data_ptr() if want_trades else None, lam.data_ptr() if want_trades else None,
                       store.nnz if shared else 0)
    prm = _lib.BatchParams(float(tol), 0.1, 1e-4, 0.5, 1e-12, int(max_outer), int(max_inner))
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    if store.has_pmm:
        _lib.check(store.lib.cfmm_batch_solve_pmm(C.byref(store.c_pools), store.records.data_ptr(), C.byref(batch),
                                                  C.byref(prm), work.data_ptr(), st), "cfmm_batch_solve_pmm")
        return psi, stats, delta, lam
    if store.has_eclp:
        _lib.check(store.lib.cfmm_batch_solve_eclp(C.byref(store.c_pools), store.records.data_ptr(), C.byref(batch),
                                                   C.byref(prm), work.data_ptr(), st), "cfmm_batch_solve_eclp")
        return psi, stats, delta, lam
    if store.has_bins:
        _lib.check(store.lib.cfmm_batch_solve_bins(C.byref(store.c_pools), store.records.data_ptr(), C.byref(batch),
                                                   C.byref(prm), work.data_ptr(), st), "cfmm_batch_solve_bins")
        return psi, stats, delta, lam
    if store.has_crypto3:
        _lib.check(store.lib.cfmm_batch_solve_tricrypto(C.byref(store.c_pools),
                                                        store.records.data_ptr() if store.records is not None else None,
                                                        C.byref(batch), C.byref(prm), work.data_ptr(), st),
                   "cfmm_batch_solve_tricrypto")
        return psi, stats, delta, lam
    if store.has_crypto:
        _lib.check(store.lib.cfmm_batch_solve_cryptoswap(C.byref(store.c_pools),
                                                         store.records.data_ptr() if store.records is not None else None,
                                                         C.byref(batch), C.byref(prm), work.data_ptr(), st),
                   "cfmm_batch_solve_cryptoswap")
        return psi, stats, delta, lam
    if store.has_ladder:
        _lib.check(store.lib.cfmm_batch_solve_concentrated(C.byref(store.c_pools), store.records.data_ptr(),
                                                           C.byref(batch), C.byref(prm), work.data_ptr(), st),
                   "cfmm_batch_solve_concentrated")
        return psi, stats, delta, lam
    entry = (store.lib.cfmm_batch_solve_stableswap_n if store.has_stableswap_n else
             store.lib.cfmm_batch_solve_stableswap if store.has_stableswap else store.lib.cfmm_batch_solve)
    _lib.check(entry(C.byref(store.c_pools), C.byref(batch), C.byref(prm), work.data_ptr(), st), "cfmm_batch_solve")
    return psi, stats, delta, lam


def pack_utilities(utilities: Sequence, n: int, nu0=None):
    """Host-side [B, n] arrays of the utilities' linear+box form (api.Arbitrage / Liquidate / Swap .spec())."""
    B = len(utilities)
    c = np.empty((B, n)); a = np.empty((B, n)); fl = np.empty((B, n), np.uint8); nu = np.empty((B, n))
    for p, u in enumerate(utilities):
        sp = u.spec(n)
        c[p] = sp.c; a[p] = sp.a
        fl[p] = np.asarray(sp.eq, np.uint8) | (np.asarray(sp.pinned, np.uint8) << 1)
        nu[p] = default_nu0(sp) if nu0 is None else np.asarray(nu0[p] if np.ndim(nu0) == 2 else nu0, float)
    return c, a, fl, nu


def solve_batch(hp: HostPools, utilities: Sequence, nu0=None, tol: float = 1e-8, device="cuda",
                want_trades: bool = True, store: Optional[CsrStore] = None, max_inner: int = 100):
    """All problems (same pools, one utility each) in one launch.  Returns a list of api.Result."""
    from .api import Result, infeasible_suspected
    t0 = time.perf_counter()
    from .api import _check_structurally_feasible
    for u in utilities:
        _check_structurally_feasible(hp, u.spec(hp.n_tokens))
    store = store or CsrStore(hp, device=device)
    n, dev = hp.n_tokens, store.device
    c, a, fl, nu = pack_utilities(utilities, n, nu0)
    up = lambda x: torch.as_tensor(x, device=dev)
    nu_d = up(nu)
    psi, stats, delta, lam = solve_batch_device(store, up(c), up(a), up(fl), nu_d, tol=tol, want_trades=want_trades,
                                                max_inner=max_inner)
    stats_h = stats.cpu().numpy()              # the one synchronisation of the call
    psi_h, nu_h = psi.cpu().numpy(), nu_d.cpu().numpy()
    if want_trades:
        d_h, l_h = delta.cpu().numpy(), lam.cpu().numpy()
    wall = time.perf_counter() - t0
    ptr = hp.pool_ptr
    names = {0: "optimal", 1: "max_iter", 2: "stalled", 3: "rejected"}
    out: List = []
    for p in range(len(utilities)):
        s = stats_h[p]
        deltas = [d_h[p, ptr[i]:ptr[i + 1]] for i in range(hp.m)] if want_trades else []
        lambdas = [l_h[p, ptr[i]:ptr[i + 1]] for i in range(hp.m)] if want_trades else []
        status = names[int(s[7])]
        if status in ("max_iter", "stalled") and infeasible_suspected(utilities[p].spec(hp.n_tokens), nu_h[p], psi_h[p], status):
            status = "infeasible"
        out.append(Result(value=float(s[0]), psi=psi_h[p], deltas=deltas, lambdas=lambdas, nu=nu_h[p],
                          dual_value=float(s[1]), gap=float(s[2]), primal_infeas=float(s[3]), iters=int(s[5]),
                          evals=int(s[6]), hvps=0, status=status, wall_s=wall, info=None))
    return out


def pack_problems(problems: Sequence):
    """Concatenate independent small problems [(HostPools, utility), ...] into one CSR array + per-problem pool ranges.
    Token indices stay local to each problem; problems with fewer tokens than the widest are padded with tokens no pool
    touches, pinned at price 1 (objective-only, zero coefficient)."""
    n = max(hp.n_tokens for hp, _ in problems)
    B = len(problems)
    ptr = [np.zeros(1, np.int64)]
    lptr = [np.zeros(1, np.int64)]               # concentrated records: their per-pool offsets shift like pool_ptr
    bptr = [np.zeros(1, np.int64)]               # bins records likewise
    ranges = np.empty((B, 2), np.int64)
    c = np.zeros((B, n)); a = np.zeros((B, n)); fl = np.full((B, n), 2, np.uint8); nu = np.ones((B, n))
    m0, off0, nnz_max = 0, 0, 0
    for p, (hp, u) in enumerate(problems):
        hp.validate()
        ptr.append(np.asarray(hp.pool_ptr[1:], np.int64) + off0)
        lptr.append(np.asarray(hp.lad_ptr[1:], np.int64) + lptr[-1][-1])
        bptr.append(np.asarray(hp.bin_ptr[1:], np.int64) + bptr[-1][-1])
        ranges[p] = (m0, m0 + hp.m)
        m0 += hp.m
        off0 += int(hp.pool_ptr[-1])
        nnz_max = max(nnz_max, int(hp.pool_ptr[-1]))
        sp = u.spec(hp.n_tokens)
        k = hp.n_tokens
        c[p, :k] = sp.c; a[p, :k] = sp.a
        fl[p, :k] = np.asarray(sp.eq, np.uint8) | (np.asarray(sp.pinned, np.uint8) << 1)
        nu[p, :k] = default_nu0(sp)
        c[p, k:] = 1.0
    cat = lambda name, dt: np.concatenate([np.asarray(getattr(hp, name), dt) for hp, _ in problems])
    merged = HostPools(n, np.concatenate(ptr), cat("tok_idx", np.int32), cat("reserves", np.float64),
                       cat("weights", np.float64), cat("gamma", np.float64), cat("kind", np.uint8),
                       cat("amp", np.float64), cat("inv", np.float64), np.concatenate(lptr),
                       np.concatenate([np.asarray(hp.lad_rec, np.float64).reshape(-1, 4) for hp, _ in problems]),
                       np.concatenate([np.asarray(hp.lad_sc, np.float64).reshape(-1, 2) for hp, _ in problems]),
                       cat("cgam", np.float64), np.concatenate(bptr),
                       np.concatenate([np.asarray(hp.bin_rec, np.float64).reshape(-1, 4) for hp, _ in problems]),
                       np.concatenate([np.asarray(hp.bin_zp, np.float64).reshape(-1, 2) for hp, _ in problems]),
                       np.concatenate([np.asarray(hp.eclp, np.float64).reshape(-1, 7) for hp, _ in problems]),
                       np.concatenate([np.asarray(hp.pmm, np.float64).reshape(-1, 4) for hp, _ in problems]))
    return merged, ranges, c, a, fl, nu, nnz_max


def solve_many(problems: Sequence, tol: float = 1e-8, device="cuda", want_trades: bool = True):
    """Independent small problems -- each its own pools and utility, e.g. one per market or per block -- in ONE launch.
    problems: [(HostPools, utility), ...].  Returns a list of api.Result, in order."""
    from .api import Result
    t0 = time.perf_counter()
    if len(problems) == 0:
        return []
    merged, ranges, c, a, fl, nu, nnz_max = pack_problems(problems)
    store = CsrStore(merged, device=device)
    dev = store.device
    up = lambda x: torch.as_tensor(x, device=dev)
    nu_d = up(nu)
    psi, stats, delta, lam = solve_batch_device(store, up(c), up(a), up(fl), nu_d, tol=tol, want_trades=want_trades,
                                                pool_range=up(ranges), nnz_max=nnz_max)
    stats_h, psi_h, nu_h = stats.cpu().numpy(), psi.cpu().numpy(), nu_d.cpu().numpy()
    if want_trades:
        d_h, l_h = delta.cpu().numpy()[0], lam.cpu().numpy()[0]
    wall = time.perf_counter() - t0
    names = {0: "optimal", 1: "max_iter", 2: "stalled", 3: "rejected"}
    out: List = []
    ptr = merged.pool_ptr
    for p, (hp, _) in enumerate(problems):
        s, k = stats_h[p], hp.n_tokens
        lo, hi = ranges[p]
        deltas = [d_h[ptr[i]:ptr[i + 1]] for i in range(lo, hi)] if want_trades else []
        lambdas = [l_h[ptr[i]:ptr[i + 1]] for i in range(lo, hi)] if want_trades else []
        out.append(Result(value=float(s[0]), psi=psi_h[p, :k], deltas=deltas, lambdas=lambdas, nu=nu_h[p, :k],
                          dual_value=float(s[1]), gap=float(s[2]), primal_infeas=float(s[3]), iters=int(s[5]),
                          evals=int(s[6]), hvps=0, status=names[int(s[7])], wall_s=wall, info=None))
    return out
