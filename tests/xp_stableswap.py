"""StableSwap (two-coin Curve) pools for the test references (test helper, not a test module).

Kind 4 of the host CSR convention: rates (r0, r1) in ``weights``, the amplification A in ``HostPools.amp`` and the
invariant D of the reserves in ``HostPools.inv``.  With y_j = r_j x_j the pool constraint is
    4A (y0' + y1') + D >= 4A D + D^3 / (4 y0' y1')      (y' = the post-trade scaled balances, D = D(R)).

* ``stableswap_response`` -- the exact optimal trades of such pools at prices nu, in any numpy float type (longdouble
  for the extended-precision reference, float64 for the oracle).  In units of D (u = y / D) the marginal rate along the
  curve is s = F_a / F_b with F_a = 4A + G / u_a, F_b = 4A + G / u_b, G = 1 / (4 u_a u_b); tendering a pays iff
  gamma mu_b s(R) > mu_a (mu_j = nu_j / r_j), and then the post-trade u_a solves log s = log(mu_a / (gamma mu_b)), a
  monotone equation in t = log u_a, solved here by bracketing and bisection-safeguarded Newton to the type's precision.
  hc = nu_0 dy_0/dlog nu_0 = -nu_a X_a / (gamma dlog s/dt).
* ``response`` / ``pool_feasibility`` / ``certify`` -- tests/xp_reference.py's functions with kind 4 added: the same
  certificate (its bounds and their derivations are unchanged), evaluated on a private copy of that module whose
  ``response`` and ``pool_feasibility`` also cover StableSwap pools.
* ``oracle_solve`` -- oracle/cfmm_oracle.py's ``solve`` (the same algorithm as the per-thread solver) on problems with
  StableSwap pools: a private copy of the oracle module whose ``evaluate`` adds the kind-4 groups in fp64.

What is independent of what.  ``stableswap_response`` is one function at two precisions and restates the same method
as cfmm_small::stableswap_pair, so the fp64 oracle and the longdouble reference do not check that method against each
other.  The independent checks, in tests/test_stableswap.py, are: Curve's get_D in 50-digit decimal; a brute-force
maximisation of each pool's profit along the curve in 80-digit decimal (no marginal-rate formula); hc against finite
differences of the trades; and the product (A -> 0) and constant-sum (A -> inf) limits.  The private module copies
rely on certify and solve looking ``response``, ``pool_feasibility`` and ``evaluate`` up as module globals; the test
that the certificate rejects an infeasible StableSwap trade fails if that ever stops being so.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np

import xp_reference as XP

KIND_STABLESWAP = 4
HERE = os.path.dirname(os.path.abspath(__file__))
LD = np.longdouble


def get_y(ua, A):
    """u_b on the curve at u_a (units of D): the positive root of u^2 + b u - c, b = u_a + 1/(4A) - 1, c = 1/(16 A u_a)"""
    one = np.ones_like(ua)
    b = (ua - one) + one / (4 * A)
    c = one / (16 * A * ua)
    sq = np.sqrt(b * b + 4 * c)
    with np.errstate(invalid="ignore", divide="ignore"):
        pos = 2 * c / (b + sq)
    return np.where(b > 0, pos, (sq - b) / 2)


def _phi(t, A, logq):
    ua = np.exp(t)
    ub = get_y(ua, A)
    G = 1 / (4 * ua * ub)
    Fa, Fb = 4 * A + G / ua, 4 * A + G / ub
    kap = -(Fa / Fb) * (ua / ub)
    d = (G / ua) * (-2 - kap) / Fa - (G / ub) * (-1 - 2 * kap) / Fb
    dl = G * (ub - ua) / (ua * ub * Fb)                         # s = 1 + dl: log1p near 1, the plain ratio far from it
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(np.abs(dl) < 0.5, np.log1p(dl), np.log(Fa / Fb)) - logq, d


def stableswap_response(R, r, A, Dv, g, nu, dtype=LD):
    """R, r, nu: (m, 2); A, Dv, g: (m,).  Returns D, L (m, 2) and hc (m,) in `dtype`."""
    R, r, nu = (np.asarray(x).astype(dtype).reshape(-1, 2) for x in (R, r, nu))
    A, Dv, g = (np.asarray(x).astype(dtype).reshape(-1) for x in (A, Dv, g))
    m = len(g)
    D = np.zeros((m, 2), dtype); L = np.zeros((m, 2), dtype); hc = np.zeros(m, dtype)
    u = r * R / Dv[:, None]
    mu = nu / r
    G0 = 1 / (4 * u[:, 0] * u[:, 1])
    tiny = np.finfo(dtype).eps
    for a, b in ((0, 1), (1, 0)):
        Fa, Fb = 4 * A + G0 / u[:, a], 4 * A + G0 / u[:, b]
        dl = G0 * (u[:, b] - u[:, a]) / (u[:, a] * u[:, b] * Fb)
        s0 = np.where(np.abs(dl) < 0.5, 1 + dl, Fa / Fb)
        go = g * mu[:, b] * s0 > mu[:, a]
        if not go.any():
            continue
        sel = np.nonzero(go)[0]
        Ag, logq = A[sel], np.log(mu[sel, a] / (g[sel] * mu[sel, b]))
        lo = np.log(u[sel, a]); hi = lo.copy()
        need = np.ones(len(sel), bool)
        step = 1.0
        while need.any() and step <= 512:                       # upper bracket: phi(hi) <= 0
            hi = np.where(need, lo + step, hi)
            f, _ = _phi(hi, Ag, logq)
            grow = need & (f > 0)
            lo = np.where(grow, hi, lo)
            need = grow
            step *= 2
        # Newton, with a bisection step whenever it would leave the bracket or not halve the step before last
        t = lo.copy()
        dx_old = hi - lo; dx = dx_old.copy()
        act = np.ones(len(sel), bool)
        for _ in range(400):
            if not act.any():
                break
            f, df = _phi(t, Ag, logq)
            lo = np.where(act & (f > 0), t, lo)
            hi = np.where(act & ~(f > 0), t, hi)
            with np.errstate(invalid="ignore", divide="ignore"):
                tn = t - f / df
            bis = ~((tn > lo) & (tn < hi)) | (np.abs(2 * f) > np.abs(dx_old * df))
            step = np.where(bis, (hi - lo) / 2, tn - t)
            done = (f == 0) | (hi - lo <= 4 * tiny * (1 + np.abs(t)))
            upd = act & ~done
            dx_old = np.where(upd, dx, dx_old); dx = np.where(upd, step, dx)
            t = np.where(upd, np.where(bis, lo + step, tn), t)
            act &= ~(done | (np.abs(step) <= tiny * (1 + np.abs(t))))
        ua = np.exp(t)
        ub = get_y(ua, Ag)
        Xa = np.maximum(ua * Dv[sel] / r[sel, a], R[sel, a])
        Xb = ub * Dv[sel] / r[sel, b]
        D[sel, a] = (Xa - R[sel, a]) / g[sel]
        L[sel, b] = np.maximum(R[sel, b] - Xb, 0)
        _, df = _phi(t, Ag, logq)
        hc[sel] += np.where(df < 0, -nu[sel, a] * Xa / (g[sel] * df), 0)
    return D, L, hc


def _stable_sel(hp):
    sel = np.nonzero(np.asarray(hp.kind) == KIND_STABLESWAP)[0]
    return sel, np.asarray(hp.pool_ptr, np.int64)[sel][:, None] + np.arange(2)[None, :]


# ---------------------------------------------------------------------------------------------- extended precision
def response(hp, nu):
    """xp_reference.response with StableSwap pools (longdouble)"""
    out = XP.response(hp, nu)
    sel, off = _stable_sel(hp)
    if len(sel):
        nv = XP.ld(nu)[np.asarray(hp.tok_idx, np.int64)[off]]
        D, L, hc = stableswap_response(np.asarray(hp.reserves)[off], np.asarray(hp.weights)[off], hp.amp[sel],
                                       hp.inv[sel], hp.gamma[sel], nv)
        out["delta"][off.ravel()] = D.ravel(); out["lam"][off.ravel()] = L.ravel()
        out["arb"][sel] = (nv * (L - D)).sum(1); out["h"][sel] = hc
    return out


def stableswap_feasibility(R, r, A, Dv, g, D, L):
    """Per pool: the relative drop of the invariant, (D - D(y')) / D to first order, of the post-trade scaled balances
    y' = r (R + gamma D - L) (<= 0 is feasible), and -min(D, L) / R for the sign of the trades.  With
    f(y', D) = 4A (y0' + y1') + D - 4A D - D^3 / (4 y0' y1'), which falls in D at the root (df/dD = 1 - 4A - 3 D^2/(4 y0'
    y1') < 0 there), D(y') - D = -f / (df/dD) + O(f^2)."""
    R, r, D, L = (XP.ld(x).reshape(-1, 2) for x in (R, r, D, L))
    A, Dv, g = (XP.ld(x).reshape(-1) for x in (A, Dv, g))
    y = r * (R + g[:, None] * D - L)
    P = y[:, 0] * y[:, 1]
    with np.errstate(invalid="ignore", divide="ignore"):
        f = 4 * A * (y[:, 0] + y[:, 1]) + Dv - 4 * A * Dv - Dv ** 3 / (4 * P)
        dfdD = 1 - 4 * A - 3 * Dv ** 2 / (4 * P)
        v = (f / dfdD) / Dv                                     # = -(D(y') - D) / D: > 0 means the invariant dropped
    v = np.where((y > 0).all(1) & np.isfinite(v), v, LD(np.inf))
    return np.maximum(v, (-np.minimum(D, L) / R).max(1))


def pool_feasibility(hp, delta, lam):
    """xp_reference.pool_feasibility with StableSwap pools"""
    worst = XP.pool_feasibility(hp, delta, lam)
    sel, off = _stable_sel(hp)
    if len(sel):
        d, l = XP.ld(delta), XP.ld(lam)
        v = stableswap_feasibility(np.asarray(hp.reserves)[off], np.asarray(hp.weights)[off], hp.amp[sel], hp.inv[sel],
                                   hp.gamma[sel], d[off], l[off])
        worst = max(worst, v.max())
    return worst


def _module_copy(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod                                     # (dataclasses look their module up while decorating)
    spec.loader.exec_module(mod)
    return mod


_XPS = _module_copy(os.path.join(HERE, "xp_reference.py"), "_xp_reference_stableswap")
_XPS.response = response
_XPS.pool_feasibility = pool_feasibility


def arb(hp, nu):
    return response(hp, nu)["arb"].sum()


def certify(hp, spec, result, tol, check=True):
    """xp_reference.certify (same five checks, same bounds) with StableSwap pools covered"""
    return _XPS.certify(hp, spec, result, tol, check)


# ---------------------------------------------------------------------------------------------- fp64 oracle
_O = _module_copy(os.path.join(HERE, "..", "oracle", "cfmm_oracle.py"), "_cfmm_oracle_stableswap")
_evaluate0 = _O.evaluate


def _evaluate(bk, nu, eps=0.0, want_trades=False, want_hess=False):
    """cfmm_oracle.evaluate plus the StableSwap groups (the kind-4 groups come last, as in the oracle's group order)"""
    stable = [g for g in bk.groups if g["kind"] == KIND_STABLESWAP]
    rest = types.SimpleNamespace(pools=bk.pools, groups=[g for g in bk.groups if g["kind"] != KIND_STABLESWAP])
    out = _evaluate0(rest, nu, eps, want_trades, want_hess)
    nu = np.asarray(nu, float)
    for g in stable:
        idx = g["idx"]
        D, L, hc = stableswap_response(g["R"], g["w"], bk.pools.amp[g["sel"]], bk.pools.inv[g["sel"]], g["gamma"],
                                       nu[idx], dtype=np.float64)
        y = L - D
        np.add.at(out["psi"], idx.ravel(), y.ravel())
        out["arb"] += float(np.sum(nu[idx] * y))
        if want_trades:
            out["delta"][g["off"].ravel()] = D.ravel(); out["lam"][g["off"].ravel()] = L.ravel()
        if want_hess:
            Hs = out["hess_scaled"]
            i0, i1 = idx[:, 0], idx[:, 1]
            np.add.at(Hs, (i0, i0), hc); np.add.at(Hs, (i1, i1), hc)
            np.add.at(Hs, (i0, i1), -hc); np.add.at(Hs, (i1, i0), -hc)
    return out


_O.evaluate = _evaluate
Utility = _O.Utility


def oracle_pools(hp):
    """the oracle's Pools of a HostPools, carrying the StableSwap constants (amp, inv) along"""
    p = _O.Pools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind)
    p.amp, p.inv = np.asarray(hp.amp, float), np.asarray(hp.inv, float)
    return p


def oracle_solve(hp, util, **kw):
    return _O.solve(oracle_pools(hp), util, **kw)


def arb_stableswap_scalar(R, r, A, Dv, gamma, nu):
    """one pool's optimal trade (fp64): D, L (2,) and hc"""
    D, L, hc = stableswap_response(np.reshape(R, (1, 2)), np.reshape(r, (1, 2)), [A], [Dv], [gamma],
                                   np.reshape(nu, (1, 2)), dtype=np.float64)
    return D[0], L[0], float(hc[0])
