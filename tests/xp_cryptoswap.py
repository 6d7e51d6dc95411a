"""Two-coin cryptoswap (Curve v2, twocrypto-ng) pools for the test references (test helper, not a test module).

Kind 7 of the host CSR convention: price scales (p0, p1) in ``weights``, the whitepaper A in ``HostPools.amp``, the
curve gamma G in ``HostPools.cgam`` and the invariant D of the reserves in ``HostPools.inv``.  With y = p x,
K0 = 4 y0 y1 / D^2 and K = A K0 G^2 / (G + 1 - K0)^2 the pool keeps D(y') >= D(R), D(y) the root of
K D (y0 + y1) + y0 y1 = K D^2 + (D/2)^2 in [2 sqrt(y0 y1), y0 + y1].

* ``cryptoswap_response`` -- the optimal trades of such pools at prices nu, in any numpy float type (longdouble for the
  extended-precision reference, float64 for the oracle): the method of cfmm_small::cryptoswap_pair (the curve point
  from the root m = 1 - K0 of h(m) = A G^2 (1 - m)(e^2 - m) - u_a m (G + m)^2, e = 2 u_a - 1; the marginal rate
  s = F_a / F_b; a safeguarded Newton iteration on log s = log(mu_a / (gamma mu_b)) in t = log u_a), vectorised, run to
  the type's precision.  hc = -nu_a X_a / (gamma dlog s/dt).
* ``response`` / ``pool_feasibility`` / ``certify`` -- xp_concentrated's (every other kind) with kind 8 added, on a
  private copy of tests/xp_reference.py, as xp_stableswap builds its own.  The feasibility of a trade is the relative
  drop (D - D(y')) / D of the invariant, D(y') found by bisection in the dtype, with no marginal-rate formula.
* ``oracle_solve`` -- oracle/cfmm_oracle.py's ``solve`` on problems with cryptoswap pools (and every kind
  xp_stableswap_n's oracle takes): a private copy whose ``evaluate`` adds the kind-8 groups in fp64.

What is independent of what.  ``cryptoswap_response`` restates the kernel's method at two precisions, so the fp64
oracle and the longdouble reference do not check that method against each other.  The independent checks, in
tests/test_cryptoswap.py, are: the invariant in 50-digit decimal; a brute-force maximisation of each pool's profit
along the curve in mpmath (no marginal-rate formula); hc against finite differences of the trades; the product limit
A -> 0; and the certificate's feasibility check above.
"""
from __future__ import annotations

import os
import types

import numpy as np

import xp_reference as XP
import xp_stableswap as XS
import xp_stableswap_n as XN
import xp_concentrated as XC

KIND_CRYPTOSWAP = 8
HERE = os.path.dirname(os.path.abspath(__file__))
LD = np.longdouble


def curve_point(ua, A, G):
    """(u_b, dl, m, K, K', K'') on the curve D = 1 at u_a, elementwise; dl = u_a + u_b - 1, m = 1 - K0"""
    one = np.ones_like(ua)
    ag2 = A * G * G
    e = 2 * ua - one
    e2 = e * e
    hi = np.minimum(e2 * A / (A + ua), np.minimum(e2, one))
    gh = G + hi
    Kh = ag2 * (one - hi) / (gh * gh)
    lo = np.minimum(e2 * Kh / (Kh + ua), hi)
    m = (lo + hi) / 2
    tiny = np.finfo(ua.dtype).eps
    act = hi > 0
    m = np.where(act, m, hi)
    for _ in range(200):
        if not act.any():
            break
        g = G + m
        f = ag2 * (one - m) * (e2 - m) - ua * m * g * g
        lo = np.where(act & (f > 0), m, lo)
        hi = np.where(act & ~(f > 0), m, hi)
        df = -ag2 * ((one - m) + (e2 - m)) - ua * g * (G + 3 * m)
        with np.errstate(invalid="ignore", divide="ignore"):
            mn = m - f / df
        mn = np.where((mn > lo) & (mn < hi), mn, (lo + hi) / 2)
        done = (f == 0) | ~(hi - lo > 2 * tiny * m) | (np.abs(mn - m) <= tiny * m)
        m = np.where(act & ~((f == 0) | ~(hi - lo > 2 * tiny * m)), mn, m)
        act &= ~done
    g = G + m
    g2 = g * g
    K = ag2 * (one - m) / g2
    K1 = ag2 * (G + 2 - m) / (g2 * g)
    K2 = ag2 * (4 * G + 6 - 2 * m) / (g2 * g2)
    with np.errstate(invalid="ignore", divide="ignore"):
        dl = np.where(m > e2 / 2, m / (4 * K), (e2 - m) / (4 * ua))
        ub = np.where(ua <= 1, (one - ua) + dl, (one - m) / (4 * ua))
    return ub, dl, m, K, K1, K2


def _phi(t, A, G, logq):
    """log s - logq at u_a = exp(t), its derivative in t, and u_b"""
    ua = np.exp(t)
    ub, dl, m, K, K1, K2 = curve_point(ua, A, G)
    d = dl - (2 * ua - 1)
    cc = 1 + 4 * dl * K1
    Fa, Fb = K + ub * cc, K + ua * cc
    sm1 = cc * d / Fb
    s = 1 + sm1
    w = d - sm1 * ua
    Q = 8 * K1 * (-sm1 * w - s * dl) + 16 * K2 * dl * w * w - 2 * s
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.where(np.abs(sm1) < 0.5, np.log1p(sm1), np.log(Fa / Fb)) - logq
    return f, ua * Q / Fa, ub


def cryptoswap_response(R, c, A, G, g, nu, dtype=LD):
    """R, c, nu: (m, 2) with c = p / D; A, G, g: (m,).  Returns D, L (m, 2) and hc (m,) in `dtype`."""
    R, c, nu = (np.asarray(x).astype(dtype).reshape(-1, 2) for x in (R, c, nu))
    A, G, g = (np.asarray(x).astype(dtype).reshape(-1) for x in (A, G, g))
    m = len(g)
    D = np.zeros((m, 2), dtype); L = np.zeros((m, 2), dtype); hc = np.zeros(m, dtype)
    mu = nu / c
    tiny = np.finfo(dtype).eps
    for a, b in ((0, 1), (1, 0)):
        logq = np.log(mu[:, a] / (g * mu[:, b]))
        t0 = np.log(c[:, a] * R[:, a])
        f0, _, _ = _phi(t0, A, G, logq)
        sel = np.nonzero(f0 > 0)[0]
        if not len(sel):
            continue
        As, Gs, lq = A[sel], G[sel], logq[sel]
        lo = t0[sel]; hi = lo.copy()
        need = np.ones(len(sel), bool)
        step = 1.0
        while need.any() and step <= 512:
            hi = np.where(need, lo + step, hi)
            f, _, _ = _phi(hi, As, Gs, lq)
            grow = need & (f > 0)
            lo = np.where(grow, hi, lo)
            need = grow
            step *= 2
        t = lo.copy()
        dx_old = hi - lo; dx = dx_old.copy()
        act = np.ones(len(sel), bool)
        for _ in range(400):
            if not act.any():
                break
            f, df, _ = _phi(t, As, Gs, lq)
            lo = np.where(act & (f > 0), t, lo)
            hi = np.where(act & ~(f > 0), t, hi)
            with np.errstate(invalid="ignore", divide="ignore"):
                tn = t - f / df
            bis = ~((tn > lo) & (tn < hi)) | (np.abs(2 * f) > np.abs(dx_old * df))
            st = np.where(bis, (hi - lo) / 2, tn - t)
            done = (f == 0) | (hi - lo <= 4 * tiny * (1 + np.abs(t)))
            upd = act & ~done
            dx_old = np.where(upd, dx, dx_old); dx = np.where(upd, st, dx)
            t = np.where(upd, np.where(bis, lo + st, tn), t)
            act &= ~(done | (np.abs(st) <= tiny * (1 + np.abs(t))))
        _, df, ub = _phi(t, As, Gs, lq)
        Xa = np.maximum(np.exp(t) / c[sel, a], R[sel, a])
        Xb = ub / c[sel, b]
        D[sel, a] = (Xa - R[sel, a]) / g[sel]
        L[sel, b] = np.maximum(R[sel, b] - Xb, 0)
        hc[sel] += np.where(df < 0, -nu[sel, a] * Xa / (g[sel] * df), 0)
    return D, L, hc


def invariant(y, A, G, dtype=LD):
    """D of scaled balances y (m, 2) by bisection on the invariant in `dtype` (no derivative, no special forms)"""
    y = np.asarray(y).astype(dtype).reshape(-1, 2)
    A, G = (np.asarray(x).astype(dtype).reshape(-1) for x in (A, G))
    lo, hi = 2 * np.sqrt(y[:, 0] * y[:, 1]), y[:, 0] + y[:, 1]
    for _ in range(80):
        d = (lo + hi) / 2
        K0 = 4 * y[:, 0] * y[:, 1] / (d * d)
        K = A * K0 * G * G / (G + 1 - K0) ** 2
        f = K * d * (y[:, 0] + y[:, 1]) + y[:, 0] * y[:, 1] - K * d * d - d * d / 4
        lo = np.where(f > 0, d, lo)
        hi = np.where(f > 0, hi, d)
    return (lo + hi) / 2


def _crypto_sel(hp):
    sel = np.nonzero(np.asarray(hp.kind) == KIND_CRYPTOSWAP)[0]
    return sel, np.asarray(hp.pool_ptr, np.int64)[sel][:, None] + np.arange(2)[None, :]


def _scaled(hp, sel, off):
    """c = p / D of the pools sel, in longdouble"""
    return XP.ld(np.asarray(hp.weights)[off]) / XP.ld(np.asarray(hp.inv)[sel])[:, None]


def _others(hp):
    kind = np.asarray(hp.kind).copy()
    kind[kind == KIND_CRYPTOSWAP] = 255
    return types.SimpleNamespace(**{**hp.__dict__, "kind": kind, "m": len(hp.gamma)})


# ---------------------------------------------------------------------------------------------- extended precision
def response(hp, nu):
    """xp_concentrated.response (every other kind) with the cryptoswap pools (longdouble)"""
    out = XC.response(_others(hp), nu)
    sel, off = _crypto_sel(hp)
    if len(sel):
        nv = XP.ld(nu)[np.asarray(hp.tok_idx, np.int64)[off]]
        D, L, hc = cryptoswap_response(np.asarray(hp.reserves)[off], _scaled(hp, sel, off), hp.amp[sel],
                                       np.asarray(hp.cgam)[sel], hp.gamma[sel], nv)
        out["delta"][off.ravel()] = D.ravel(); out["lam"][off.ravel()] = L.ravel()
        out["arb"][sel] = (nv * (L - D)).sum(1); out["h"][sel] = hc
    return out


def cryptoswap_feasibility(R, p, A, G, Dv, g, D, L):
    """Per pool: (D - D(y')) / D for the post-trade scaled balances y' = p (R + gamma D - L) (<= 0 is feasible), and
    -min(D, L) / R for the sign of the trades"""
    R, p, D, L = (XP.ld(x).reshape(-1, 2) for x in (R, p, D, L))
    A, G, Dv, g = (XP.ld(x).reshape(-1) for x in (A, G, Dv, g))
    y = p * (R + g[:, None] * D - L)
    ok = (y > 0).all(1)
    Dn = invariant(np.where(ok[:, None], y, 1), A, G)
    v = np.where(ok, (Dv - Dn) / Dv, LD(np.inf))
    return np.maximum(v, (-np.minimum(D, L) / R).max(1))


def pool_feasibility(hp, delta, lam):
    worst = XC.pool_feasibility(_others(hp), delta, lam)
    sel, off = _crypto_sel(hp)
    if len(sel):
        d, l = XP.ld(delta), XP.ld(lam)
        v = cryptoswap_feasibility(np.asarray(hp.reserves)[off], np.asarray(hp.weights)[off], hp.amp[sel],
                                   np.asarray(hp.cgam)[sel], hp.inv[sel], hp.gamma[sel], d[off], l[off])
        worst = max(worst, v.max())
    return worst


_XPK = XS._module_copy(os.path.join(HERE, "xp_reference.py"), "_xp_reference_cryptoswap")
_XPK.response = response
_XPK.pool_feasibility = pool_feasibility


def certify(hp, spec, result, tol, check=True):
    """xp_reference.certify (same five checks, same bounds) with cryptoswap pools and every other kind covered"""
    return _XPK.certify(hp, spec, result, tol, check)


# ---------------------------------------------------------------------------------------------- fp64 oracle
_O = XS._module_copy(os.path.join(HERE, "..", "oracle", "cfmm_oracle.py"), "_cfmm_oracle_cryptoswap")
_evaluate_n = XN._evaluate


def _evaluate(bk, nu, eps=0.0, want_trades=False, want_hess=False):
    """xp_stableswap_n's oracle evaluate plus the cryptoswap groups"""
    cs = [g for g in bk.groups if g["kind"] == KIND_CRYPTOSWAP]
    rest = types.SimpleNamespace(pools=bk.pools, groups=[g for g in bk.groups if g["kind"] != KIND_CRYPTOSWAP])
    out = _evaluate_n(rest, nu, eps, want_trades, want_hess)
    nu = np.asarray(nu, float)
    for g in cs:
        idx, sel = g["idx"], g["sel"]
        c = np.asarray(g["w"], float) / bk.pools.inv[sel][:, None]
        D, L, hc = cryptoswap_response(g["R"], c, bk.pools.amp[sel], bk.pools.cgam[sel], g["gamma"], nu[idx],
                                       dtype=np.float64)
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


def oracle_solve(hp, util, **kw):
    p = _O.Pools(hp.n_tokens, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind)
    p.amp, p.inv, p.cgam = np.asarray(hp.amp, float), np.asarray(hp.inv, float), np.asarray(hp.cgam, float)
    return _O.solve(p, util, **kw)
