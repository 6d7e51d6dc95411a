"""Drop-in boundary for the reference's cvxpy call site.

The reference has no library API: a script builds literals (arbitrage.py:5-36), wires cvxpy objects
(arbitrage.py:50-78) and calls ``prob.solve()`` (arbitrage.py:82), then reads ``prob.value`` /
``psi.value`` / ``deltas[i].value`` / ``lambdas[i].value`` (arbitrage.py:84, liquidation.py:87,
two-asset.py:94-100).  ``solve()`` takes the same literals and returns those same quantities.
"""
from __future__ import annotations

import dataclasses
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .pools import HostPools, PoolStore
from .solver import Comm, DualSpec, SolveInfo, solve_dual


# ----------------------------------------------------------------------------------------------
# utilities  U(psi)
# ----------------------------------------------------------------------------------------------
class Arbitrage:
    """maximise market_value @ psi  s.t. psi >= 0          (arbitrage.py:57, :77)"""

    def __init__(self, market_value):
        self.c = np.asarray(market_value, float)
        if np.any(self.c <= 0):
            raise ValueError("market_value must be positive")

    def spec(self, n):
        if len(self.c) != n:
            raise ValueError("market_value needs one entry per token")
        return DualSpec(self.c, np.zeros(n), np.zeros(n, bool), np.zeros(n, bool))


class Liquidate:
    """maximise psi[target]  s.t. psi[j] + current_assets[j] == 0 for j != target   (liquidation.py:57, :77-80)"""

    def __init__(self, target, current_assets):
        self.target = int(target)
        self.assets = np.asarray(current_assets, float)

    def spec(self, n):
        if len(self.assets) != n:
            raise ValueError("current_assets needs one entry per token")
        c = np.zeros(n); c[self.target] = 1.0
        a = self.assets.copy(); a[self.target] = 0.0
        eq = np.ones(n, bool); eq[self.target] = False
        pinned = np.zeros(n, bool); pinned[self.target] = True
        return DualSpec(c, a, eq, pinned)


class Swap:
    """maximise psi[tok_out]  s.t. psi + t e_in >= 0        (two-asset.py:41-45, :66, :86)"""

    def __init__(self, tok_in, tok_out, t):
        self.tok_in, self.tok_out, self.t = int(tok_in), int(tok_out), float(t)

    def spec(self, n):
        c = np.zeros(n); c[self.tok_out] = 1.0
        a = np.zeros(n); a[self.tok_in] = self.t
        return DualSpec(c, a, np.zeros(n, bool), np.zeros(n, bool))


class LinearUtility:
    """maximise c @ psi  s.t.  psi_j + a_j >= 0 | psi_j + a_j == 0 (eq) | psi_j unconstrained (pinned): the linear + box form
    the three utilities above reduce to, for any mix of them (what cvxpy_compat recognises in a model's objective and
    token constraints)"""

    def __init__(self, c, a, eq, pinned):
        self.c, self.a = np.asarray(c, float), np.asarray(a, float)
        self.eq, self.pinned = np.asarray(eq, bool), np.asarray(pinned, bool)
        if np.any(self.c < 0) or np.any(self.pinned & (self.c <= 0)) or np.any(self.eq & self.pinned):
            raise ValueError("LinearUtility: c >= 0, unconstrained tokens need c > 0, eq and pinned exclude each other")

    def spec(self, n):
        if not (len(self.c) == len(self.a) == len(self.eq) == len(self.pinned) == n):
            raise ValueError("LinearUtility needs one entry per token")
        return DualSpec(self.c, self.a, self.eq, self.pinned)


# ----------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Result:
    value: float                  # prob.value                      arbitrage.py:84
    psi: np.ndarray               # psi.value                       liquidation.py:87
    deltas: List[np.ndarray]      # deltas[i].value                 two-asset.py:97
    lambdas: List[np.ndarray]     # lambdas[i].value                two-asset.py:97
    nu: np.ndarray                # optimal dual prices (new)
    dual_value: float
    gap: float
    primal_infeas: float
    iters: int
    evals: int
    hvps: int
    status: str                   # 'optimal' | 'max_iter' | 'stalled' | 'infeasible' (suspected)   (cf. prob.status)
    wall_s: float
    info: Optional[SolveInfo] = None


def solve(local_indices, reserves, fees, kinds, weights=None, utility=None, n_tokens: Optional[int] = None,
          nu0=None, tol: float = 1e-8, max_iter: int = 100, device="cuda", verbose: bool = False,
          **solver_kw) -> Result:
    """Solve the routing problem the reference scripts pose.  `kinds[i]` in {'geomean','product','sum'}
    names the cvxpy atom on pool i (arbitrage.py:63-74); `weights[i]` is the geo_mean ``p=`` vector.  Two more kinds:
    'bounded_product' (weights[i] = virtual-reserve offsets) and 'stableswap' (weights[i] = (A, r_0, ..., r_{n-1}), a
    Curve pool of 2..8 coins with the whitepaper A = A() / n^(n-1); see HostPools.from_lists).  And 'concentrated':
    weights[i] = (price, bounds, liquidity), a whole Uniswap-v3 tick ladder as one pool, with reserves[i] = None (see
    HostPools.from_lists and instances.v3_ladder).  And 'cryptoswap': weights[i] = (A, gamma, p_0, p_1), a two-coin Curve v2
    (twocrypto-ng) pool with the whitepaper A, the curve's gamma and the price scales (see HostPools.from_lists and
    instances.twocrypto_pool).  And 'eclp': reserves[i] = (x, y), weights[i] = (alpha, beta, c, s, lam), a Gyroscope
    elliptic concentrated-liquidity pool (see HostPools.from_lists and instances.eclp_pool).  And 'pmm': reserves[i] =
    (B, Q), weights[i] = (pi, k, B0, Q0), a DODO proactive market maker with its guide price, slippage factor and
    targets (see HostPools.from_lists and instances.pmm_pool).  Problems with StableSwap, concentrated, cryptoswap, E-CLP
    or PMM pools run solver.py, the native host loop or the per-thread solver, never the native blocked and persistent
    solvers."""
    if utility is None:
        raise ValueError("utility is required: Arbitrage(c) | Liquidate(target, assets) | Swap(i, o, t)")
    if n_tokens is None:
        n_tokens = 1 + max(int(t) for l in local_indices for t in l)
    hp = HostPools.from_lists(n_tokens, local_indices, reserves, fees, kinds, weights)
    return solve_pools(hp, utility, nu0=nu0, tol=tol, max_iter=max_iter, device=device, verbose=verbose,
                       **solver_kw)


def _check_structurally_feasible(hp: HostPools, spec) -> None:
    """A token that must change hands (psi_j + a_j == 0 with a_j != 0, or psi_j + a_j >= 0 with a_j < 0) but sits in no
    pool makes the program infeasible (cvxpy would set prob.status = 'infeasible'; the scripts never look at it).  The
    dual method would only see that token's price drift to its floor, so it is rejected up front."""
    a = np.asarray(spec.a, float)
    need = ((np.asarray(spec.eq, bool) & (a != 0)) | (~np.asarray(spec.eq, bool) & ~np.asarray(spec.pinned, bool) & (a < 0)))
    if need.any():
        present = np.zeros(hp.n_tokens, bool)
        present[np.asarray(hp.tok_idx)] = True
        bad = np.nonzero(need & ~present)[0]
        if len(bad):
            raise ValueError(f"infeasible problem: token(s) {bad.tolist()} must be traded (non-zero endowment / demand) "
                             "but appear in no pool")


def infeasible_suspected(spec, nu, psi, status: str) -> bool:
    """cvxpy would set prob.status = 'infeasible' (arbitrage.py:82 never looks) when no trade meets the constraints on
    psi.  The dual method cannot prove that, but it shows an unmistakable pattern: the solve ends uncertified AND the price
    of a token whose constraint is still badly violated has run away -- to the floor (a token that must be sold but
    nobody can take: liquidation.py:77-80 with an unroutable basket entry) or to the sky (a token that must be received
    in a quantity the pools cannot deliver).  Returns True for that pattern only."""
    if status == "optimal":
        return False
    nu = np.asarray(nu, float); psi = np.asarray(psi, float)
    a = np.asarray(spec.a, float); eq = np.asarray(spec.eq, bool); pinned = np.asarray(spec.pinned, bool)
    s = psi + a
    viol = np.where(pinned, 0.0, np.where(eq, np.abs(s), np.maximum(-s, 0.0)))
    scale = max(float(np.abs(a).max(initial=0.0)), float(np.abs(np.where(pinned, 0.0, psi)).max(initial=0.0)), 1e-300)
    bad = viol > 1e-3 * scale
    if not bad.any() or not np.all(np.isfinite(nu)):
        return bool(bad.any())
    ok = ~bad & (nu > 0)
    ref = float(np.median(nu[ok])) if ok.any() else float(np.max(np.abs(np.asarray(spec.c, float)), initial=1.0))
    return bool(np.any(bad & ((nu <= 1e-8 * ref) | (nu >= 1e8 * ref))))


SMALL_POOLS = 256        # up to here one GPU thread walks all pools of a problem faster than a launch per evaluation


def _small_applicable(hp: HostPools, comm: Comm, verbose, solver_kw) -> bool:
    from . import batch as _batch
    return (comm.dist is None and not verbose and not solver_kw and hp.m <= SMALL_POOLS
            and _batch.batch_applicable(hp))


def _native_applicable(store: PoolStore, comm: Comm, solver_kw) -> bool:
    """one blocked constant-product bucket (per rank); pool-sharded runs need the NVLink peer context"""
    return ((comm.dist is None or getattr(store, "reduces_internally", False))
            and len(store.buckets) == 1 and getattr(store.buckets[0], "blocked", False)
            and solver_kw.get("linear_solver", "auto") in ("auto", "cg") and not solver_kw.get("verbose"))


def _enable_peer(store: PoolStore, comm: Comm) -> None:
    """world > 1: switch the store to the in-kernel NVLink all-reduce when symmetric memory is available (collective:
    every rank reaches the same decision because availability is a property of the node)"""
    if comm.dist is None or getattr(store, "reduces_internally", False) or store.device.type != "cuda":
        return
    if comm.dist.get_backend() != "nccl" or store.n_tokens + 1 > 64 * 256:
        return
    try:
        store.enable_peer_allreduce()
    except Exception as e:                      # no symmetric memory / no peer access: NCCL keeps doing the all-reduce
        import warnings
        warnings.warn(f"peer all-reduce unavailable ({type(e).__name__}: {e}); using torch.distributed all_reduce")


def _solve_native(store: PoolStore, spec, nu0, tol, max_iter, cg_max=200, impl="persist") -> SolveInfo:
    """The whole outer loop in one C call: impl 'persist' = ONE persistent cooperative kernel (csrc/cfmm_persist.cu: the
    host launches once and reads one result struct), 'hostloop' = C++ host loop over per-pass launches
    (csrc/cfmm_solver.cu).  Same method, same stopping rule, same results up to summation order."""
    import ctypes as C
    import time
    from .solver import default_nu0
    t0 = time.perf_counter()
    b = store.buckets[0]
    n, dev = store.n_tokens, store.device
    f64 = dict(dtype=torch.float64, device=dev)
    c = torch.as_tensor(np.asarray(spec.c, float), **f64)
    a = torch.as_tensor(np.asarray(spec.a, float), **f64)
    eq = torch.as_tensor(np.asarray(spec.eq, np.uint8), device=dev)
    pinned = torch.as_tensor(np.asarray(spec.pinned, np.uint8), device=dev)
    nu = torch.as_tensor(default_nu0(spec) if nu0 is None else np.asarray(nu0, float), **f64).clone()
    psi = torch.empty(n, **f64)
    if impl not in ("persist", "hostloop"):
        raise ValueError("native must be True / 'persist' / 'hostloop' / False")
    work_bytes = store.lib.cfmm_persist_solve_work_bytes if impl == "persist" else store.lib.cfmm_blocked_solve_work_bytes
    entry = store.lib.cfmm_persist_solve if impl == "persist" else store.lib.cfmm_blocked_solve_peer
    nbytes = work_bytes(C.byref(b.c_blocked), n)
    if nbytes <= 0:
        raise _lib.CfmmError("solve work_bytes failed")
    if getattr(store, "_solve_work", None) is None or store._solve_work.numel() < nbytes:
        store._solve_work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    scale = max(float(np.abs(spec.c).max()), 1.0)
    prm = _lib.SolveParams(float(tol), 1e-12 * scale, int(max_iter), int(cg_max))
    res = _lib.SolveResult()
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    peer = getattr(store, "_peer", None) if getattr(store, "reduces_internally", False) else None
    pc = peer.c_struct() if peer is not None else None
    rc = entry(C.byref(b.c_blocked), n, c.data_ptr(), a.data_ptr(), eq.data_ptr(), pinned.data_ptr(), nu.data_ptr(),
               psi.data_ptr(), store._solve_work.data_ptr(), C.byref(prm), C.byref(res),
               C.byref(pc) if pc is not None else None, st)
    if pc is not None:
        peer.absorb(pc)                 # the reductions of this solve advanced the shared sequence numbers
    _lib.check(rc, "cfmm_persist_solve" if impl == "persist" else "cfmm_blocked_solve")
    store.evals += res.evals
    store.hvps += res.hvps
    status = {0: "optimal", 1: "max_iter", 2: "stalled"}[res.status]
    return SolveInfo(nu=nu, psi=psi, dual_value=res.dual_value, primal_value=res.primal_value, gap=res.gap,
                     primal_infeas=res.primal_infeas, err=res.err, iters=res.iters, outer=1, evals=res.evals,
                     hvps=res.hvps, status=status, wall_s=time.perf_counter() - t0, history=[])


MARKET_KW = ("linear_solver", "cg_max", "eps", "eps_min", "eps_shrink", "max_outer")


def _market_applicable(store: PoolStore, native, verbose, solver_kw) -> bool:
    """native="hostloop" on a single-GPU store of any pool kinds, with solver.py keywords the C++ loop takes"""
    return native == "hostloop" and store.world == 1 and not verbose and all(k in MARKET_KW for k in solver_kw)


def _solve_market(store: PoolStore, spec, nu0, tol, max_iter, linear_solver="auto", cg_max=200, eps=0.1,
                  eps_min=1e-4, eps_shrink=0.5, max_outer=60) -> SolveInfo:
    """The whole of solver.py's loop in one C call (cfmm_market_solve, csrc/cfmm_solver.cu): every pool kind, the dense or
    PCG Newton systems and the method of multipliers, with the final read-back's trades left in the store's buckets."""
    import ctypes as C
    import time
    from .solver import default_nu0
    t0 = time.perf_counter()
    ls = {"auto": 0, "dense": 1, "cg": 2}.get(linear_solver)
    if ls is None:
        raise ValueError("linear_solver must be 'auto', 'dense' or 'cg'")
    n, dev = store.n_tokens, store.device
    f64 = dict(dtype=torch.float64, device=dev)
    c = torch.as_tensor(np.asarray(spec.c, float), **f64)
    a = torch.as_tensor(np.asarray(spec.a, float), **f64)
    eq = torch.as_tensor(np.asarray(spec.eq, np.uint8), device=dev)
    pinned = torch.as_tensor(np.asarray(spec.pinned, np.uint8), device=dev)
    nu = torch.as_tensor(default_nu0(spec) if nu0 is None else np.asarray(nu0, float), **f64).clone()
    psi = torch.empty(n, **f64)
    buckets, outs, nb, blk, blk_out = store.market_structs()
    blk_p = C.byref(blk) if blk is not None else None
    nbytes = store.lib.cfmm_market_solve_work_bytes(buckets, nb, blk_p, n, ls)
    _lib.check(min(int(nbytes), 0), "cfmm_market_solve_work_bytes")
    if getattr(store, "_market_work", None) is None or store._market_work.numel() < nbytes:
        store._market_work = None
        store._market_work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    scale = max(float(np.abs(spec.c).max()), 1.0)
    prm = _lib.MarketParams(float(tol), 1e-12 * scale, float(eps), float(eps_min), float(eps_shrink), int(max_iter),
                            int(cg_max), int(max_outer), ls)
    res = _lib.SolveResult()
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    rc = store.lib.cfmm_market_solve(buckets, outs, nb, blk_p, C.byref(blk_out) if blk_out is not None else None, n,
                                     c.data_ptr(), a.data_ptr(), eq.data_ptr(), pinned.data_ptr(), nu.data_ptr(),
                                     psi.data_ptr(), store._market_work.data_ptr(), C.byref(prm), C.byref(res), st)
    _lib.check(rc, "cfmm_market_solve")
    store.evals += res.evals
    store.hvps += res.hvps
    status = {0: "optimal", 1: "max_iter", 2: "stalled"}[res.status]
    return SolveInfo(nu=nu, psi=psi, dual_value=res.dual_value, primal_value=res.primal_value, gap=res.gap,
                     primal_infeas=res.primal_infeas, err=res.err, iters=res.iters, outer=1, evals=res.evals,
                     hvps=res.hvps, status=status, wall_s=time.perf_counter() - t0, history=[])


def solve_pools(hp: HostPools, utility, nu0=None, tol: float = 1e-8, max_iter: int = 100, device="cuda",
                verbose: bool = False, store: Optional[PoolStore] = None, want_trades: bool = True,
                native=True, method: str = "auto", **solver_kw) -> Result:
    """Same as solve() on CSR host arrays.  Under torch.distributed (world_size > 1) every rank passes the
    full problem and keeps its contiguous shard; psi/value are global, deltas/lambdas are this rank's.
    method: 'pools' = pool-parallel kernels under the outer loop (any size); 'thread' = the whole solve in one GPU
    thread (<= 64 tokens, arity <= 8); 'auto' picks 'thread' up to SMALL_POOLS pools.
    native (constant-product problems): True / 'persist' = the persistent solver kernel, 'hostloop' = the C++ host loop
    over per-pass launches, False = the python loop (solver.py).  native='hostloop' on any other single-GPU store (every
    pool kind, mixed) runs the C++ market loop (cfmm_market_solve), which takes the solver_kw linear_solver, cg_max, eps,
    eps_min, eps_shrink and max_outer; other keywords, or verbose, keep solver.py."""
    comm = Comm()
    if method not in ("auto", "pools", "thread"):
        raise ValueError("method must be 'auto', 'pools' or 'thread'")
    _check_structurally_feasible(hp, utility.spec(hp.n_tokens))
    if method == "thread" or (method == "auto" and store is None and _small_applicable(hp, comm, verbose, solver_kw)):
        # problems of the reference's own size (5 pools): the whole solve in one launch of the per-thread solver
        # (csrc/cfmm_small.cu) instead of one launch per dual evaluation -- 10x less latency, same certificate
        from . import batch as _batch
        return _batch.solve_batch(hp, [utility], nu0=None if nu0 is None else np.asarray(nu0, float)[None, :],
                                  tol=tol, device=device, want_trades=want_trades, max_inner=max_iter)[0]
    if store is None:
        rank = comm.dist.get_rank() if comm.dist is not None else 0
        world = comm.dist.get_world_size() if comm.dist is not None else 1
        store = PoolStore(hp, device=device, rank=rank, world=world)
    if store.world > 1:
        _enable_peer(store, comm)
    else:
        comm = Comm(enabled=False)          # an unsharded store under an initialised process group: nothing to reduce
    spec = utility.spec(hp.n_tokens)
    if native and not verbose and _native_applicable(store, comm, solver_kw):
        info = _solve_native(store, spec, nu0, tol, max_iter, solver_kw.get("cg_max", 200),
                             impl="persist" if native is True else native)
        if want_trades:          # one more pass of the eval kernel to emit Delta / Lambda at the solution
            store.evaluate(info.nu, 0.0, trades=True, hess=False)
    elif _market_applicable(store, native, verbose, solver_kw):
        # any other single-GPU store: the C++ market loop; its final read-back already left the trades in the buckets
        info = _solve_market(store, spec, nu0, tol, max_iter, **solver_kw)
    else:
        info = solve_dual(store, spec, nu0=nu0, tol=tol, max_inner=max_iter, comm=comm, verbose=verbose,
                          final_trades=want_trades, **solver_kw)
    deltas: List[np.ndarray] = []
    lambdas: List[np.ndarray] = []
    if want_trades:
        d, l = store.gather_trades()
        ptr = hp.pool_ptr
        deltas = [d[ptr[i]:ptr[i + 1]] for i in range(hp.m)] if hp.m <= 100_000 else [d]
        lambdas = [l[ptr[i]:ptr[i + 1]] for i in range(hp.m)] if hp.m <= 100_000 else [l]
    psi_h, nu_h = info.psi.cpu().numpy(), info.nu.cpu().numpy()
    status = "infeasible" if infeasible_suspected(spec, nu_h, psi_h, info.status) else info.status
    return Result(value=info.primal_value, psi=psi_h, deltas=deltas, lambdas=lambdas,
                  nu=nu_h, dual_value=info.dual_value, gap=info.gap,
                  primal_infeas=info.primal_infeas, iters=info.iters, evals=info.evals, hvps=info.hvps,
                  status=status, wall_s=info.wall_s, info=info)


def solve_sweep(local_indices, reserves, fees, kinds, weights, utilities, n_tokens: Optional[int] = None,
                tol: float = 1e-8, device="cuda", batched: Optional[bool] = None, **solver_kw) -> List[Result]:
    """The loop of two-asset.py:40-100 as one call: the same pools under a sequence of utilities (there: Swap(0, 2, t)
    for t in linspace(0, 50)), where the reference rebuilds the whole cvxpy problem per t (two-asset.py:47-91).
    batched (default whenever the pools fit: <= 64 tokens, arity <= 8): ALL utilities are solved by one kernel launch,
    one problem per thread (`batch.solve_batch`).  Otherwise the pool buckets are uploaded once and the solves run in
    turn, each warm-started from the previous prices."""
    from . import batch as _batch
    if n_tokens is None:
        n_tokens = 1 + max(int(t) for l in local_indices for t in l)
    hp = HostPools.from_lists(n_tokens, local_indices, reserves, fees, kinds, weights)
    if batched is None:
        batched = _batch.batch_applicable(hp) and not solver_kw
    if batched:
        return _batch.solve_batch(hp, list(utilities), tol=tol, device=device)
    store = PoolStore(hp, device=device)
    out: List[Result] = []
    nu = None
    for u in utilities:
        r = solve_pools(hp, u, nu0=nu, tol=tol, store=store, **solver_kw)
        nu = r.nu if r.status == "optimal" else None
        out.append(r)
    return out
