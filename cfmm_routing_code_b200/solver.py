"""Outer dual solver: what replaces `prob.solve()` (arbitrage.py:81-82 / liquidation.py:84-85 /
two-asset.py:90-91) once the per-pool subproblems are evaluated by the CUDA kernels.

    minimise   g(nu) = sum_j (nu_j - c_j) a_j + sum_i arb_i(A_i' nu)
    over       nu_j >= c_j (inequality tokens) | nu_j > 0 free (equality tokens) | nu_j = c_j (objective-only)

grad g = a + psi(nu) and the Hessian is sum_i A_i H_i A_i', so one dual evaluation is one pass of the
pool kernels plus (multi-GPU) ONE all-reduce of the (n_tokens+1)-vector [psi | arb].

Method: projected (active-set) Newton in log-price coordinates; the Newton system is solved either by
Jacobi-preconditioned truncated CG on kernel Hessian-vector products (large n, matrix free) or by a
dense Cholesky (small n).  Constant-sum pools make g piecewise linear; they are handled by the method of
multipliers on their fills (theta_bar), which keeps every inner problem smooth and converges to the exact
kink solution (both reference instances sit on such a kink).

The vector algebra is torch on whatever device the evaluator lives on; the evaluator protocol is
    n_tokens, has_sum, evaluate(nu, eps, trades, hess) -> acc[n+1], hvp(vt), hess_diag(), hess_dense(),
    update_multipliers() -> move[1], reset_multipliers()
`PoolStore` (CUDA) is the only evaluator this package ships.
"""
from __future__ import annotations

import dataclasses
import time
from typing import Optional

import numpy as np
import torch


DT_MAX = 3.0      # largest log-price change of one Newton step (dense or CG)
LM_SHIFTS = (1e-14, 1e-8, 1e-6, 1e-4, 1e-2, 1.0)     # damping ladder of the dense Newton system, times the mean diagonal


@dataclasses.dataclass
class DualSpec:
    """Utility in 'linear + box' form (see api.Arbitrage / Liquidate / Swap)."""
    c: np.ndarray        # objective coefficients on psi
    a: np.ndarray        # endowment: constraint is psi_j + a_j >= 0 | == 0
    eq: np.ndarray       # bool: psi_j + a_j == 0
    pinned: np.ndarray   # bool: psi_j unconstrained, nu_j = c_j


@dataclasses.dataclass
class SolveInfo:
    nu: torch.Tensor
    psi: torch.Tensor
    dual_value: float
    primal_value: float
    gap: float
    primal_infeas: float
    err: float
    iters: int
    outer: int
    evals: int
    hvps: int
    status: str
    wall_s: float
    history: list


class Comm:
    """Sum all-reduce over torch.distributed when world_size > 1, else a no-op."""

    def __init__(self, enabled: bool = True):
        import torch.distributed as dist
        self.dist = dist if (enabled and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1) else None
        self.calls = 0

    def allreduce(self, t: torch.Tensor) -> torch.Tensor:
        if self.dist is not None:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM)
            self.calls += 1
        return t

    def allreduce_max(self, t: torch.Tensor) -> torch.Tensor:
        if self.dist is not None:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return t


def default_nu0(spec: DualSpec) -> np.ndarray:
    c = np.asarray(spec.c, float)
    pos = c[c > 0]
    scale = float(np.median(pos)) if len(pos) else 1.0
    return np.where(c > 0, c, scale)


def solve_dual(ev, spec: DualSpec, nu0=None, tol: float = 1e-8, eps: float = 0.1, eps_min: float = 1e-4,
               eps_shrink: float = 0.5, max_outer: int = 60, max_inner: int = 100, linear_solver: str = "auto", cg_max: int = 200, comm: Optional[Comm] = None,
               verbose: bool = False, final_trades: bool = True, lookahead: Optional[int] = None) -> SolveInfo:
    t_start = time.perf_counter()
    comm = comm or Comm()
    n = ev.n_tokens
    dev = ev.device
    f64 = dict(dtype=torch.float64, device=dev)
    c = torch.as_tensor(np.asarray(spec.c, float), **f64)
    a = torch.as_tensor(np.asarray(spec.a, float), **f64)
    eq = torch.as_tensor(np.asarray(spec.eq, bool), device=dev)
    fixed = torch.as_tensor(np.asarray(spec.pinned, bool), device=dev)
    scale = max(float(np.abs(spec.c).max()), 1.0)
    floor = 1e-12 * scale
    lb = torch.where(eq, torch.full_like(c, floor), torch.clamp(c, min=floor))
    nu = torch.as_tensor(default_nu0(spec) if nu0 is None else np.asarray(nu0, float), **f64).clone()
    nu = torch.maximum(nu, lb)
    nu = torch.where(fixed, c, nu)
    has_sum = bool(ev.has_sum)
    eps_t = float(eps) if has_sum else 0.0
    if has_sum:
        ev.reset_multipliers()
    if linear_solver == "auto":
        linear_solver = "dense" if (n <= 256 or (has_sum and n <= 4096)) else "cg"
    if lookahead is None:
        # every look-ahead round is one more factorisation: worth it where evaluations dominate (tiny n, or a CPU
        # evaluator in the tests), not where a 1000 x 1000 Cholesky costs more than a pool pass (measured on cfg3)
        lookahead = 3 if (n <= 64 or dev.type == "cpu") else 0
    evals0, hvps0 = ev.evals, ev.hvps
    a_inf = float(np.abs(np.asarray(spec.a, float)).max())
    notfixed = (~fixed).to(torch.float64)
    history = []
    internal = bool(getattr(ev, "reduces_internally", False))     # PoolStore.enable_peer_allreduce(): no NCCL needed

    def G(nu_, hess=True, trades=False):
        acc = ev.evaluate(nu_, eps_t, trades=trades, hess=hess)
        if not internal:
            acc = comm.allreduce(acc)
        psi = acc[:n].clone()
        g = torch.dot(nu_ - c, a) + acc[n]
        return psi, g

    def kkt(nu_, psi_, g_, err_prev):
        """free set + KKT residual = max of
          * value-weighted: sum_free |nu_j (a_j+psi_j)| / |g|  (bounds the relative gap and the value of the infeasibility)
          * per token:      max_free |a_j+psi_j| / max(|a|_inf, max over the CONSTRAINED tokens |psi_j|)  -- the reference
            enforces psi_j + a_j == 0 / complementarity token by token (liquidation.py:77-80, arbitrage.py:77), so a
            cheap token must not hide a large residual behind its small price, nor behind the (unconstrained,
            objective-only) output of the target token."""
        grad_ = a + psi_
        # active-set width: a token counts as 'at its bound' within a relative 1e-3 * (KKT residual).  (Round 1 used the
        # residual itself: on the 1M-pool instance that froze ~1000 tokens just above their bounds for a dozen iterations --
        # 26 Newton steps / 136 pool passes; with the narrow band the same solve takes 9 steps / 49 passes.)
        thr = min(1e-2, max(1e-3 * (err_prev if np.isfinite(err_prev) else 1e-2), 1e-14))
        near = (nu_ <= lb * (1.0 + thr)) & ~eq
        fr_ = (~(fixed | (near & (grad_ > 0)))).to(torch.float64)
        pg_ = nu_ * grad_ * fr_
        st = torch.stack([pg_.abs().sum(), g_.abs(), torch.dot(nu_, grad_.abs()), (grad_ * fr_).abs().max(),
                          (psi_ * notfixed).abs().max()]).tolist()
        feas = st[3] / max(a_inf, st[4], 1e-300)
        return max(st[0] / max(st[1], 1e-3 * st[2], 1e-300), feas), grad_, fr_, pg_

    iters = 0
    status = "max_iter"
    err = float("inf")
    outer_done = 0
    move = 1.0
    failed_before = False
    for outer in range(max_outer):
        outer_done = outer + 1
        psi, g = G(nu)
        inner_status = "max_iter"
        # early outer passes need not be solved tightly: the multipliers are still moving
        inner_tol = max(tol, min(1e-3, 1e-2 * move)) if has_sum else tol
        err, grad, fr, pg = kkt(nu, psi, g, err)
        for _ in range(max_inner):
            iters += 1
            history.append((time.perf_counter() - t_start, ev.evals - evals0, err))
            if verbose:
                print(f"outer {outer} it {iters} g={float(g):.15g} err={err:.3e} free={int(fr.sum())}")
            if err <= inner_tol:
                inner_status = "optimal"
                break
            rhs = -pg
            # ---- Newton direction in log-price coordinates: Hs dt = -(nu*grad) on the free set
            pgfull = nu * grad
            Hs = comm.allreduce(ev.hess_dense()) if linear_solver == "dense" else None
            diag = None if linear_solver == "dense" else (ev.hess_diag() if internal else comm.allreduce(ev.hess_diag()))

            def newton_dir(fr_, x0=None):
                if linear_solver == "dense":
                    H0 = Hs * fr_[:, None] * fr_[None, :]
                    dbar = max(float(torch.diagonal(H0).sum()) / max(int(fr_.sum()), 1), 1e-300)
                    rhs_ = (-pgfull * fr_)[:, None]
                    d_ = None
                    # (near-)singular free-set systems (every pool tying some free prices to the rest saturated) give an
                    # enormous step along the null directions: climb the damping ladder (Levenberg-Marquardt shift
                    # mu * mean diagonal) until the step is a sane price change
                    for r_ in range(rung0, len(LM_SHIFTS)):
                        rung_used[0] = max(rung_used[0], r_)
                        Hm = H0 + torch.diag((1.0 - fr_) + (LM_SHIFTS[r_] * dbar) * fr_)
                        L, info = torch.linalg.cholesky_ex(Hm)
                        if int(info) != 0:
                            continue
                        d_ = torch.cholesky_solve(rhs_, L)[:, 0]
                        if float(d_.abs().max()) <= DT_MAX:
                            break
                    if d_ is None:
                        d_ = torch.linalg.lstsq(H0 + torch.diag((1.0 - fr_) + dbar * fr_), rhs_).solution[:, 0]
                    return d_ * fr_
                return _pcg(ev, comm, -pgfull * fr_, fr_, diag, eta=min(0.1, err ** 0.5), max_it=cg_max, x0=x0)

            fr0 = fr
            rung0, rung_used = 0, [0]
            while True:          # a failed search along a barely damped (null-space dominated) direction is retried with
                fr = fr0         # the next rung of the damping ladder before the iteration is declared stalled
                rung_used[0] = rung0
                dt = newton_dir(fr)
                # ---- look-ahead on the active set: a token held at its bound (grad > 0) whose PREDICTED gradient after
                # this step, nu*grad + Hs dt, is negative would be released at the next iteration anyway; release it now
                # and re-solve (warm started).  Costs Hessian-vector products only, saves whole Newton iterations
                # (the all-at-bound start of the arbitrage utility otherwise frees tokens layer by layer).
                bound_act = (fr == 0) & ~fixed
                for _la in range(lookahead if linear_solver == "dense" else 0):   # with CG the extra HVPs eat the gain
                    if not bool(bound_act.any()):
                        break
                    Hd = (Hs @ dt) if linear_solver == "dense" else _reduce_hvp(ev, comm, dt)
                    newly = bound_act & ((pgfull + Hd) < 0)
                    if not bool(newly.any()):
                        break
                    fr2 = fr + newly.to(fr.dtype)
                    dt2 = newton_dir(fr2, x0=dt)
                    bad = newly & (dt2 <= 0)                 # would be pushed below its bound after all: keep it active
                    if bool(bad.any()):
                        fr2 = fr2 - bad.to(fr.dtype)
                        dt2 = dt2 * fr2
                    fr, dt = fr2, dt2
                    bound_act = (fr == 0) & ~fixed
                pg = pgfull * fr
                slope = torch.dot(pg, dt)     # = grad . (nu*dt)
                if not bool(torch.isfinite(slope)) or float(slope) >= 0.0:
                    dt = -pg / pg.abs().max().clamp(min=1e-300)
                # (near-)singular system, e.g. every pool tying the free prices to a bound is saturated: keep the
                # direction, bound the step to a price factor of e^3 and let the line search find the kink.  A truncated-CG
                # step can be as long (a swap over 65 536 tokens gave one of ~1e14): unbounded, every trial of the search
                # sits on the +-20 clamp below -- the same point -- until the 50 halvings run out
                big = float(dt.abs().max())
                if big > DT_MAX:
                    dt = dt * (DT_MAX / big)
                # ---- projected Armijo backtracking along nu * exp(alpha dt)
                alpha = 1.0
                g0 = float(g)
                ok = False
                for _ls in range(50):
                    nu_t = torch.maximum(nu * torch.exp(torch.clamp(alpha * dt, -20.0, 20.0)), lb)
                    nu_t = torch.where(fixed, c, nu_t)
                    psi_t, g_t = G(nu_t)
                    lin = float(torch.dot(grad, nu_t - nu))
                    if _ls == 0:
                        lin1 = lin             # predicted decrease of the FULL step
                    gt = float(g_t)
                    if gt <= g0 + 1e-4 * lin:
                        ok = True
                        break
                    if abs(gt - g0) <= 1e-13 * abs(g0) or abs(lin1) <= 1e-9 * abs(g0):
                        # the (full) step is below what g resolves in fp64 (g is a sum of cancelling flows: the Armijo
                        # decrease 1e-4 |lin| would be under 1e-13 |g|): judge it by the KKT residual instead
                        if kkt(nu_t, psi_t, g_t, err)[0] < 0.99 * err:
                            ok = True
                            break
                        if alpha < 1e-3:
                            break
                    alpha *= 0.5
                if ok or linear_solver != "dense" or rung_used[0] >= len(LM_SHIFTS) - 1:
                    break
                rung0 = rung_used[0] + 1
            if not ok:
                inner_status = "stalled"
                break
            nu, psi, g = nu_t, psi_t, g_t
            err, grad, fr, pg = kkt(nu, psi, g, err)
        if not has_sum:
            status = inner_status
            break
        # method of multipliers.  The smoothed trades are pool-feasible, so (exact dual - primal) at this nu
        # is a true optimality certificate; stop on it rather than on the multiplier step, whose floor is
        # (fp64 resolution of the price ratio) / eps.
        psi_s, _ = G(nu, hess=False, trades=True)
        acc0 = ev.evaluate(nu, 0.0, trades=False, hess=False)
        acc0 = acc0 if internal else comm.allreduce(acc0)
        dual_now = float(torch.dot(nu - c, a) + acc0[n])
        gap_now = (dual_now - float(torch.dot(c, psi_s))) / max(abs(dual_now), 1e-300)
        if verbose:
            print(f"outer {outer}: eps {eps_t:.1e} last move {move:.3e} gap {gap_now:.3e}")
        if inner_status == "optimal" and err <= tol and abs(gap_now) <= tol:
            status = "optimal"      # the only certified exit: KKT residual AND exact duality gap within tol
            break           # multipliers stay as they are: the read-back below reproduces psi_s
        # not certified (loose inner tolerance, or multipliers / ramp still moving): falling out of the loop is 'max_iter'
        status = inner_status if inner_status != "optimal" else "max_iter"
        if inner_status != "optimal" and failed_before and eps_t <= float(eps_min):
            break           # ramp at its narrowest, two failed passes: residual is at the fp64 floor (ratio / eps)
        failed_before = inner_status != "optimal"
        move = float(comm.allreduce_max(ev.update_multipliers().clone()))
        eps_t = max(float(eps_min), eps_t * float(eps_shrink))
    # ---- final read-back + certificate: primal from the (smoothed, pool-feasible) trades, dual exact
    psi_f, _ = G(nu, hess=False, trades=final_trades)
    if has_sum:
        acc0 = ev.evaluate(nu, 0.0, trades=False, hess=False)
        acc0 = acc0 if internal else comm.allreduce(acc0)
        arb_exact = float(acc0[n])
    else:
        arb_exact = float(torch.dot(nu, psi_f))     # arb = nu'psi for the exact evaluation
    dual = float(torch.dot(nu - c, a)) + arb_exact
    primal = float(torch.dot(c, psi_f))
    s = psi_f + a
    viol = torch.where(fixed, torch.zeros_like(s), torch.where(eq, s.abs(), torch.clamp(-s, min=0.0)))
    # value-weighted infeasibility relative to the dual value (scale-free)
    infeas = float(torch.dot(nu, viol)) / max(abs(dual), 1e-300)
    gap = (dual - primal) / max(abs(dual), 1e-300)
    return SolveInfo(nu=nu, psi=psi_f, dual_value=dual, primal_value=primal, gap=gap, primal_infeas=infeas,
                     err=err, iters=iters, outer=outer_done, evals=ev.evals - evals0, hvps=ev.hvps - hvps0,
                     status=status, wall_s=time.perf_counter() - t_start, history=history)


def _reduce_hvp(ev, comm, vt):
    y = ev.hvp(vt)
    return (y if getattr(ev, "reduces_internally", False) else comm.allreduce(y)).clone()


def _pcg(ev, comm, rhs, fr, diag, eta, max_it, x0=None):
    """Truncated Jacobi-PCG for Hs x = rhs restricted to the free coordinates (fr = 0/1 mask)."""
    minv = fr / torch.clamp(diag, min=1e-300)
    if x0 is None:
        x = torch.zeros_like(rhs)
        r = rhs * fr
    else:
        x = x0 * fr
        r = (rhs - _reduce_hvp(ev, comm, x)) * fr
    z = minv * r
    p = z.clone()
    rz = torch.dot(r, z)
    r0 = float(torch.sqrt(torch.dot(z, r)))
    if r0 == 0.0:
        return x
    for k in range(max_it):
        Hp = ev.hvp(p)
        Hp = (Hp if getattr(ev, "reduces_internally", False) else comm.allreduce(Hp)) * fr
        pHp = torch.dot(p, Hp)
        vals = torch.stack([pHp, rz, torch.dot(p, p * torch.clamp(diag, min=1e-300))]).tolist()
        if vals[0] <= 1e-14 * vals[2]:          # (near-)zero curvature: homogeneity direction
            if k == 0:
                x = p.clone()
            break
        alpha = vals[1] / vals[0]
        x = x + alpha * p
        r = r - alpha * Hp
        z = minv * r
        rz_new = torch.dot(r, z)
        rn = float(rz_new)
        if rn <= 0.0 or rn ** 0.5 <= eta * r0:
            break
        p = z + (rn / vals[1]) * p
        rz = rz_new
    return x
