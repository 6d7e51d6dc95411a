"""n-coin StableSwap (Curve) pools for the test references (test helper, not a test module).

Kind 4 of the host CSR convention with 2..8 coins: rates r in ``weights``, the whitepaper amplification A in
``HostPools.amp`` and the invariant D of the reserves in ``HostPools.inv``.  With y = r x, a = A n^n and u = y / D the
pool keeps
    G(u) = a sum(u) + 1 - a - Q(u) >= 0,      Q(u) = 1 / (n^n prod(u)),
which at n = 2 is the two-coin constraint of tests/xp_stableswap.py.

* ``stablen_response`` -- the exact optimal trades of such pools at prices nu, and the pool's block of the scaled
  Hessian, in any numpy float type (longdouble for the extended-precision reference, float64 for the oracle).  It
  restates the method of cfmm_small::stableswap_n: prices pi = nu / r, log price ratios dB_j = log(pi_j / pi_min), and
  the unknown tau = log(pi_min / (gamma a mu)) > 0 for the constraint's multiplier mu.  At fixed tau the stationary
  point is u_j = u0_j exp(z_j), z_j = max(l - bA_j, 0) + min(l - bB_j, 0) with l = log(Q / a),
  bA_j = log(u0_j expm1(dB_j + tau)), bB_j = log(u0_j expm1(dB_j + log gamma + tau)) (-inf when that expm1 <= 0), and
  l solves the piecewise-linear, strictly increasing F(l) = (l - l0) + sum_j z_j(l) = 0, exactly from its breakpoints.
  The outer equation h(tau) = sum_j u0_j expm1(z_j) - q0 expm1(l - l0) = G / a = 0 falls in tau and is solved by
  bracketing and bisection-safeguarded Newton in log tau, to the type's precision.
* ``stablen_feasibility`` -- per pool, the relative drop of the invariant of the post-trade balances (<= 0 feasible).
* ``response`` / ``pool_feasibility`` / ``certify`` / ``oracle_solve`` -- tests/xp_stableswap.py's functions with
  the pools of more than two coins added, through private copies of xp_reference.py and the oracle, as that module does
  for two coins.

What is independent of what.  ``stablen_response`` at two precisions is one method; the independent checks, in
tests/test_stableswap_n.py, are the KKT conditions in 50-digit decimal, finite differences of the trades, the two-coin
pair function, the A -> 0 geometric-mean limit and the no-trade band.
"""
from __future__ import annotations

import os
import types

import numpy as np

import xp_reference as XP
import xp_stableswap as XS

KIND_STABLESWAP = 4
HERE = os.path.dirname(os.path.abspath(__file__))
LD = np.longdouble


def _inner(tau, dB, lg, lu0, l0):
    """l(tau) and the per-coin z, bA, bB, eA, eB at tau (arrays over pools)"""
    eA = np.expm1(dB + tau[:, None])
    eB = np.expm1(dB + lg[:, None] + tau[:, None])
    with np.errstate(divide="ignore", invalid="ignore"):
        bA = lu0 + np.log(eA)
        bB = np.where(eB > 0, lu0 + np.log(np.where(eB > 0, eB, 1)), -np.inf)
    T = np.concatenate([bA, bB], 1)                                     # (m, 2n) breakpoints, -inf ones never chosen
    with np.errstate(invalid="ignore"):                                 # (-inf) - (-inf): a breakpoint that is never chosen
        F = (T - l0[:, None]) + (np.maximum(T[:, :, None] - bA[:, None, :], 0)
                                 + np.minimum(T[:, :, None] - bB[:, None, :], 0)).sum(2)
    ok = np.isfinite(T) & (F <= 0)
    Tl = np.where(ok, T, -np.inf)
    iL = Tl.argmax(1)
    sL = np.take_along_axis(T, iL[:, None], 1)[:, 0]
    FL = np.take_along_axis(F, iL[:, None], 1)[:, 0]
    any_ok = ok.any(1)
    # no breakpoint with F <= 0: the root lies left of the smallest one, where only the finite bB still bind
    Tf = np.where(np.isfinite(T), T, np.inf)
    iM = Tf.argmin(1)
    sM = np.take_along_axis(T, iM[:, None], 1)[:, 0]
    FM = np.take_along_axis(F, iM[:, None], 1)[:, 0]
    slope_r = 1 + (sL[:, None] >= bA).sum(1) + (sL[:, None] < bB).sum(1)
    slope_l = 1 + np.isfinite(bB).sum(1)
    l = np.where(any_ok, sL - FL / slope_r.astype(T.dtype), sM - FM / slope_l.astype(T.dtype))
    z = np.maximum(l[:, None] - bA, 0) + np.minimum(l[:, None] - bB, 0)
    return l, z, eA, eB


def _h(tau, dB, lg, lu0, l0, u0, q0):
    l, z, eA, eB = _inner(tau, dB, lg, lu0, l0)
    h = (u0 * np.expm1(z)).sum(1) - q0 * np.expm1(l - l0)
    u = u0 * np.exp(z)
    q = q0 * np.exp(l - l0)
    tr = z != 0
    e = np.where(z > 0, eA, eB)
    with np.errstate(divide="ignore", invalid="ignore"):
        kap = np.where(tr, 1 + 1 / np.where(tr, e, 1), 0)
    k = tr.sum(1)
    lt = kap.sum(1) / (1 + k)
    dh = (np.where(tr, u * (lt[:, None] - kap), 0)).sum(1) - q * lt        # dh / dtau (< 0)
    return h, dh * tau, l, z, u, q                                      # (and dh / dlog tau)


def stablen_response(R, r, A, Dv, g, nu, dtype=LD):
    """R, r, nu: (m, n); A, Dv, g: (m,).  Returns D, L, h (m, n) (h_j of the Hessian formula, 0 off the traded set) and
    Hs (m, n, n), the pool's scaled Hessian nu_i nu_j dpsi_i / dnu_j, in `dtype`."""
    R, r, nu = (np.asarray(x).astype(dtype) for x in (R, r, nu))
    m, n = R.shape
    A, Dv, g = (np.asarray(x).astype(dtype).reshape(-1) for x in (A, Dv, g))
    D = np.zeros((m, n), dtype); L = np.zeros((m, n), dtype); hj = np.zeros((m, n), dtype)
    Hs = np.zeros((m, n, n), dtype)
    a = A * dtype(n ** n)
    u0 = r * R / Dv[:, None]
    lu0 = np.log(u0)
    l0 = -(dtype(n) * np.log(dtype(n)) + lu0.sum(1)) - np.log(a)
    q0 = np.exp(l0)
    pi = nu / r
    pmin = pi.min(1)
    dB = np.log(pi / pmin[:, None])
    lg = np.log(g)
    c = dB - np.log1p(q0[:, None] / u0)
    go = lg + c.max(1) > c.min(1)
    if not go.any():
        return D, L, hj, Hs
    s = np.nonzero(go)[0]
    dB, lg, lu0, l0, u0, q0 = dB[s], lg[s], lu0[s], l0[s], u0[s], q0[s]
    args = (dB, lg, lu0, l0, u0, q0)
    tiny = np.finfo(dtype).eps
    sg = np.log(-c[s].min(1))                                           # log tau at which the last grower stops (q = q0)
    f, _, *_ = _h(np.exp(sg), *args)
    lo = np.where(f > 0, sg, -np.inf); hi = np.where(f > 0, np.inf, sg)
    step = 1.0
    need = ~np.isfinite(lo) | ~np.isfinite(hi)
    while need.any() and step <= 512:                                   # bracket: h(lo) > 0 >= h(hi)
        up = need & np.isinf(hi)
        tr_ = np.clip(np.where(up, lo + step, hi - step), -700, np.log(600.0))
        fv, _, *_ = _h(np.exp(np.where(need, tr_, sg)), *args)
        lo = np.where(need & (fv > 0), tr_, lo); hi = np.where(need & ~(fv > 0), tr_, hi)
        need = ~np.isfinite(lo) | ~np.isfinite(hi)
        step *= 2
    t = np.where(np.isfinite(lo), lo, hi)
    dx_old = hi - lo; dx = dx_old.copy()
    act = np.ones(len(s), bool)
    for _ in range(400):
        if not act.any():
            break
        f, df, *_ = _h(np.exp(t), *args)
        lo = np.where(act & (f > 0), t, lo)
        hi = np.where(act & ~(f > 0), t, hi)
        with np.errstate(invalid="ignore", divide="ignore"):
            tn = t - f / df
        bis = ~((tn > lo) & (tn < hi)) | (np.abs(2 * f) > np.abs(dx_old * df))
        stp = np.where(bis, (hi - lo) / 2, tn - t)
        done = (f == 0) | (hi - lo <= 4 * tiny * (1 + np.abs(t)))
        upd = act & ~done
        dx_old = np.where(upd, dx, dx_old); dx = np.where(upd, stp, dx)
        t = np.where(upd, np.where(bis, lo + stp, tn), t)
        act &= ~(done | (np.abs(stp) <= tiny * (1 + np.abs(t))))
    tau = np.exp(t)
    _, _, l, z, u, q = _h(tau, *args)
    Rs, gs, pis = R[s], g[s], pi[s]
    D[s] = np.where(z > 0, Rs * np.expm1(z) / gs[:, None], 0)
    L[s] = np.where(z < 0, -Rs * np.expm1(z), 0)
    tr = z != 0
    p = np.where(z > 0, pis / gs[:, None], pis)
    cc = Dv[s] * gs * np.exp(tau) / (pmin[s] * q)
    h = np.where(tr, np.sqrt(cc)[:, None] * p * u, 0)
    hj[s] = h
    Hs[s] = hess_block(h)
    return D, L, hj, Hs


def hess_block(h):
    """Hs (m, n, n) from the per-slot h (m, n), 0 off the traded set: C - (C1)(C1)' / (1'C1), C = diag(h^2) - h h'/(1+k)"""
    k = (h != 0).sum(1).astype(h.dtype)
    C = np.einsum("mi,ij->mij", h * h, np.eye(h.shape[1], dtype=h.dtype)) - h[:, :, None] * h[:, None, :] / (1 + k)[:, None, None]
    C1 = C.sum(2)
    s1 = C1.sum(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = C - C1[:, :, None] * C1[:, None, :] / np.where(s1 > 0, s1, 1)[:, None, None]
    return np.where((s1 > 0)[:, None, None], out, 0)


def stablen_feasibility(R, r, A, Dv, g, D, L):
    """Per pool: the relative drop of the invariant, (D - D(y')) / D to first order, of the post-trade scaled balances
    y' = r (R + gamma D - L) (<= 0 is feasible), and -min(D, L) / R for the sign of the trades.  With
    f(D) = a sum(y') + D - a D - D^(n+1) / (n^n prod y'), df/dD = 1 - a - (n+1) D^n / (n^n prod y') < 0 at the root,
    D(y') - D = -f / (df/dD) + O(f^2)."""
    R, r, D, L = (XP.ld(x) for x in (R, r, D, L))
    n = R.shape[1]
    A, Dv, g = (XP.ld(x).reshape(-1) for x in (A, Dv, g))
    a = A * LD(n ** n)
    y = r * (R + g[:, None] * D - L)
    with np.errstate(invalid="ignore", divide="ignore"):
        w = Dv[:, None] / (LD(n) * y)
        P = np.prod(w, 1)                                               # D^n / (n^n prod y)
        f = a * y.sum(1) + Dv - a * Dv - Dv * P
        dfdD = 1 - a - (n + 1) * P
        v = (f / dfdD) / Dv
    v = np.where((y > 0).all(1) & np.isfinite(v), v, LD(np.inf))
    return np.maximum(v, (-np.minimum(D, L) / R).max(1))


def _groups(hp):
    """(n, pool ids, (m, n) offsets) of the StableSwap pools of more than two coins"""
    ss = np.nonzero(np.asarray(hp.kind) == KIND_STABLESWAP)[0]
    ptr = np.asarray(hp.pool_ptr, np.int64)
    ar = ptr[ss + 1] - ptr[ss]
    return [(int(k), ss[ar == k], ptr[ss[ar == k]][:, None] + np.arange(k)) for k in np.unique(ar[ar > 2]).tolist()]


# ---------------------------------------------------------------------------------------------- extended precision
def _two_coin_only(hp):
    """hp with its StableSwap pools of more than two coins marked as a kind no reference evaluates (they are added
    separately), so the two-coin reference's fixed arity-2 gathers never see them"""
    kind = np.asarray(hp.kind).copy()
    for _, sel, _ in _groups(hp):
        kind[sel] = 255
    return types.SimpleNamespace(**{**hp.__dict__, "kind": kind})


def response(hp, nu):
    """xp_stableswap.response with the pools of more than two coins (longdouble); h of those pools is per slot"""
    out = XS.response(_two_coin_only(hp), nu)
    out["hslot"] = {}
    for k, sel, off in _groups(hp):
        nv = XP.ld(nu)[np.asarray(hp.tok_idx, np.int64)[off]]
        D, L, h, Hs = stablen_response(np.asarray(hp.reserves)[off], np.asarray(hp.weights)[off], hp.amp[sel],
                                       hp.inv[sel], hp.gamma[sel], nv)
        out["delta"][off.ravel()] = D.ravel(); out["lam"][off.ravel()] = L.ravel()
        out["arb"][sel] = (nv * (L - D)).sum(1)
        out["hslot"][k] = (sel, h, Hs)
    return out


def pool_feasibility(hp, delta, lam):
    worst = XS.pool_feasibility(_two_coin_only(hp), delta, lam)
    for _, sel, off in _groups(hp):
        d, l = XP.ld(delta), XP.ld(lam)
        v = stablen_feasibility(np.asarray(hp.reserves)[off], np.asarray(hp.weights)[off], hp.amp[sel], hp.inv[sel],
                                hp.gamma[sel], d[off], l[off])
        worst = max(worst, v.max())
    return worst


_XPN = XS._module_copy(os.path.join(HERE, "xp_reference.py"), "_xp_reference_stableswap_n")
_XPN.response = response
_XPN.pool_feasibility = pool_feasibility


def certify(hp, spec, result, tol, check=True):
    """xp_reference.certify (same five checks, same bounds) with StableSwap pools of 2..8 coins covered"""
    return _XPN.certify(hp, spec, result, tol, check)


# ---------------------------------------------------------------------------------------------- fp64 oracle
_O = XS._module_copy(os.path.join(HERE, "..", "oracle", "cfmm_oracle.py"), "_cfmm_oracle_stableswap_n")
_evaluate2 = XS._evaluate


def _evaluate(bk, nu, eps=0.0, want_trades=False, want_hess=False):
    """xp_stableswap's oracle evaluate (the oracle plus two-coin StableSwap groups) plus the groups of more coins"""
    big = [g for g in bk.groups if g["kind"] == KIND_STABLESWAP and g["k"] > 2]
    rest = types.SimpleNamespace(pools=bk.pools, groups=[g for g in bk.groups if not (g["kind"] == KIND_STABLESWAP
                                                                                    and g["k"] > 2)])
    out = _evaluate2(rest, nu, eps, want_trades, want_hess)
    nu = np.asarray(nu, float)
    for g in big:
        idx = g["idx"]
        D, L, _, Hb = stablen_response(g["R"], g["w"], bk.pools.amp[g["sel"]], bk.pools.inv[g["sel"]], g["gamma"],
                                       nu[idx], dtype=np.float64)
        y = L - D
        np.add.at(out["psi"], idx.ravel(), y.ravel())
        out["arb"] += float(np.sum(nu[idx] * y))
        if want_trades:
            out["delta"][g["off"].ravel()] = D.ravel(); out["lam"][g["off"].ravel()] = L.ravel()
        if want_hess:
            k = idx.shape[1]
            np.add.at(out["hess_scaled"], (np.repeat(idx, k, 1).ravel(), np.tile(idx, (1, k)).ravel()), Hb.ravel())
    return out


_O.evaluate = _evaluate
Utility = _O.Utility


def oracle_solve(hp, util, **kw):
    p = _O.Pools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind)
    p.amp, p.inv = np.asarray(hp.amp, float), np.asarray(hp.inv, float)
    return _O.solve(p, util, **kw)
