"""Three-coin cryptoswap (Curve v2, tricrypto-ng) pools for the test references (test helper, not a test module).

Host kind 8 with three tokens (device kind 9): price scales (p0, p1, p2) in ``weights``, the whitepaper A in
``HostPools.amp``, the curve gamma G in ``HostPools.cgam`` and the invariant D of the reserves in ``HostPools.inv``.
With y = p x, K0 = 27 y0 y1 y2 / D^3 and K = A K0 G^2 / (G + 1 - K0)^2 the pool keeps D(y') >= D(R), D(y) the root of
K D^2 S + P = K D^3 + (D/3)^3 in [3 P^(1/3), S].

* ``invariant`` -- D by plain bisection on that cubic in the dtype (no derivative, no special forms).
* ``tricrypto_response`` -- the optimal trades at prices nu in any numpy float type (longdouble for the
  extended-precision reference): the KKT characterisation of cfmm_small::cryptoswap3 (at fixed m = 1 - K0 the
  traded balances are u_j = clamp(u0_j, Q / (pi_j / (gamma mu) - K), Q / (pi_j / mu - K)); the price level from
  P = (1 - m) / 27, m from S - 1 = m / (27 K)), but every root found by fixed-count bisection, vectorised, to the
  type's precision, with no Newton step and no derivative.  The no-trade band as the kernel states it.
* ``edges_fd`` -- the scaled Hessian's edge weights by central differences of the response in the dtype, with no
  Hessian formula: Hs_ab = nu_a d(Lambda_a - Delta_a) / d log nu_b.
* ``response`` / ``pool_feasibility`` / ``certify`` -- xp_cryptoswap's (every other kind, two-coin cryptoswap included)
  with the three-coin pools added.  The feasibility of a trade is the relative drop (D - D(y')) / D of the invariant,
  D(y') by ``invariant``.

What is independent of what.  ``tricrypto_response`` restates the kernel's KKT conditions, so it checks the kernel's
root finding, its cancellation-free forms and its precision, not the conditions themselves.  Those are checked in
tests/test_tricrypto.py by a brute-force maximisation over the curve in mpmath, the invariant and the post-trade point in
decimal, the geometric-mean limit A -> 0, and here by the certificate, whose feasibility check and dual bound use
``invariant`` and the response only.
"""
from __future__ import annotations

import os
import types

import numpy as np

import xp_reference as XP
import xp_stableswap as XS
import xp_cryptoswap as XK

KIND_CRYPTOSWAP = 8
HERE = os.path.dirname(os.path.abspath(__file__))
LD = np.longdouble


def invariant(y, A, G, dtype=LD, iters=90):
    """D of scaled balances y (m, 3) by bisection on [3 P^(1/3), S] in `dtype` (F > 0 below the root)"""
    y = np.asarray(y).astype(dtype).reshape(-1, 3)
    A, G = (np.asarray(x).astype(dtype).reshape(-1) for x in (A, G))
    S, P = y.sum(1), y[:, 0] * y[:, 1] * y[:, 2]
    lo, hi = 3 * np.cbrt(P), S.copy()
    for _ in range(iters):
        d = (lo + hi) / 2
        K0 = 27 * P / (d * d * d)
        K = A * K0 * G * G / (G + 1 - K0) ** 2
        f = K * d * d * S + P - K * d * d * d - (d / 3) ** 3
        lo = np.where(f > 0, d, lo)
        hi = np.where(f > 0, hi, d)
    return (lo + hi) / 2


def tricrypto_response(R, c, A, G, g, nu, dtype=LD, iters=76):
    """Optimal trades (Delta, Lambda) (m, 3) of three-coin pools with c = p / D at prices nu (m, 3), and the traded
    slots as a bit mask (m,).  Nested fixed-count bisection: x = logit(m) in [-700, 700] outside, s = log tau in
    [-700, 6.39] inside, each root bracketed by the sign of a monotone function."""
    R, c, nu = (np.asarray(x).astype(dtype).reshape(-1, 3) for x in (R, c, nu))
    A, G, g = (np.asarray(x).astype(dtype).reshape(-1) for x in (A, G, g))
    m_ = len(g)
    u0 = c * R
    lu0 = np.log(u0)
    e0 = 3 * u0 - 1
    sl0 = np.log1p(e0).sum(1)
    pi = nu / c
    pmin = pi.min(1)
    dB = np.log(pi / pmin[:, None])
    lg = np.log(g)
    ag2 = A * G * G
    m0 = np.maximum(-np.expm1(sl0), 0)
    om0 = np.exp(sl0)
    Kc = ag2 * om0 / (G + m0) ** 2
    Qc = (G + 3 * m0 - 2 * m0 * m0) / (27 * (G + m0))
    cj = dB - np.log(Kc[:, None] + Qc[:, None] / u0)
    trade = lg + cj.max(1) > cj.min(1)

    def z_of(s, l):
        tau = np.exp(s)[:, None]
        eA = np.expm1(dB + tau)
        eB = np.expm1(dB + lg[:, None] + tau)
        zA = l[:, None] - (lu0 + np.log(eA))
        with np.errstate(invalid="ignore", divide="ignore"):
            zB = np.where(eB > 0, l[:, None] - (lu0 + np.log(np.where(eB > 0, eB, 1))), np.inf)
        return np.maximum(zA, 0) + np.minimum(zB, 0)

    def inner(x):
        m = 1 / (1 + np.exp(-x))
        om = 1 / (1 + np.exp(x))
        gm = G + m
        K = ag2 * om / (gm * gm)
        qn = G + 3 * m - 2 * m * m
        l = np.log(qn * gm / (27 * ag2 * om))
        with np.errstate(divide="ignore"):
            tgt = np.log1p(-m) - sl0                     # -inf at x = 700 in float64: E1 > 0 there, s goes to its top
        lo, hi = np.full(m_, dtype(-700)), np.full(m_, dtype(6.39))
        for _ in range(iters):
            s = (lo + hi) / 2
            f = z_of(s, l).sum(1) - tgt
            lo = np.where(f > 0, s, lo)
            hi = np.where(f > 0, hi, s)
        s = (lo + hi) / 2
        z = z_of(s, l)
        r = (e0 + 3 * u0 * np.expm1(z)).sum(1) - m / (9 * K)
        return r, z

    lo, hi = np.full(m_, dtype(-700)), np.full(m_, dtype(700))
    for _ in range(iters):
        x = (lo + hi) / 2
        r, _ = inner(x)
        lo = np.where(r > 0, x, lo)
        hi = np.where(r > 0, hi, x)
    _, z = inner((lo + hi) / 2)
    z = np.where(trade[:, None], z, 0)
    ex = np.expm1(z)
    D = np.where(z > 0, R * ex / g[:, None], 0)
    L = np.where(z < 0, -R * ex, 0)
    mask = ((z != 0) * np.array([1, 2, 4])).sum(1).astype(np.uint32)
    return D, L, mask


def edges_fd(R, c, A, G, g, nu, dtype=LD, h=1e-8):
    """(w01, w02, w12) = -Hs_ab by central differences of tricrypto_response in log nu (step h), and a flag per pool
    that the traded set stays the same over every step (the band edges are not differentiable)"""
    nu = np.asarray(nu).astype(dtype).reshape(-1, 3)
    _, _, mask = tricrypto_response(R, c, A, G, g, nu, dtype)
    Hs = np.zeros((len(nu), 3, 3), dtype)
    same = np.ones(len(nu), bool)
    for b in range(3):
        f = []
        for sgn in (1, -1):
            nb = nu.copy()
            nb[:, b] *= np.exp(dtype(sgn * h))
            D, L, mk = tricrypto_response(R, c, A, G, g, nb, dtype)
            same &= mk == mask
            f.append(L - D)
        Hs[:, :, b] = nu * (f[0] - f[1]) / (2 * h)
    w = np.stack([-Hs[:, 0, 1], -Hs[:, 0, 2], -Hs[:, 1, 2]], 1)
    return w, mask, same


def _tri_sel(hp):
    ptr = np.asarray(hp.pool_ptr, np.int64)
    sel = np.nonzero((np.asarray(hp.kind) == KIND_CRYPTOSWAP) & (np.diff(ptr) == 3))[0]
    return sel, ptr[sel][:, None] + np.arange(3)[None, :]


def _others(hp):
    """hp with its three-coin pools marked as a kind no other reference evaluates"""
    sel, _ = _tri_sel(hp)
    kind = np.asarray(hp.kind).copy()
    kind[sel] = 255
    return types.SimpleNamespace(**{**hp.__dict__, "kind": kind, "m": len(hp.gamma)})


def response(hp, nu):
    """xp_cryptoswap.response (every other kind) with the three-coin pools (longdouble); their h is 0 (unused by the
    certificate)"""
    out = XK.response(_others(hp), nu)
    sel, off = _tri_sel(hp)
    if len(sel):
        nv = XP.ld(nu)[np.asarray(hp.tok_idx, np.int64)[off]]
        c = XP.ld(np.asarray(hp.weights)[off]) / XP.ld(np.asarray(hp.inv)[sel])[:, None]
        D, L, _ = tricrypto_response(np.asarray(hp.reserves)[off], c, hp.amp[sel], np.asarray(hp.cgam)[sel],
                                     hp.gamma[sel], nv)
        out["delta"][off.ravel()] = D.ravel(); out["lam"][off.ravel()] = L.ravel()
        out["arb"][sel] = (nv * (L - D)).sum(1); out["h"][sel] = 0
    return out


def tricrypto_feasibility(R, p, A, G, Dv, g, D, L):
    """Per pool: (D - D(y')) / D for y' = p (R + gamma D - L) (<= 0 is feasible), and -min(D, L) / R"""
    R, p, D, L = (XP.ld(x).reshape(-1, 3) for x in (R, p, D, L))
    A, G, Dv, g = (XP.ld(x).reshape(-1) for x in (A, G, Dv, g))
    y = p * (R + g[:, None] * D - L)
    ok = (y > 0).all(1)
    Dn = invariant(np.where(ok[:, None], y, 1), A, G)
    v = np.where(ok, (Dv - Dn) / Dv, LD(np.inf))
    return np.maximum(v, (-np.minimum(D, L) / R).max(1))


def pool_feasibility(hp, delta, lam):
    worst = XK.pool_feasibility(_others(hp), delta, lam)
    sel, off = _tri_sel(hp)
    if len(sel):
        d, l = XP.ld(delta), XP.ld(lam)
        v = tricrypto_feasibility(np.asarray(hp.reserves)[off], np.asarray(hp.weights)[off], hp.amp[sel],
                                  np.asarray(hp.cgam)[sel], hp.inv[sel], hp.gamma[sel], d[off], l[off])
        worst = max(worst, v.max())
    return worst


_XPT = XS._module_copy(os.path.join(HERE, "xp_reference.py"), "_xp_reference_tricrypto")
_XPT.response = response
_XPT.pool_feasibility = pool_feasibility


def certify(hp, spec, result, tol, check=True):
    """xp_reference.certify (same five checks, same bounds) with three-coin pools and every other kind covered"""
    return _XPT.certify(hp, spec, result, tol, check)
