"""Extended-precision reference for elliptic concentrated-liquidity pools (Gyroscope E-CLP), in mpmath.

Independent of the package (it reads only the data of a HostPools): the pool is stated in its circle frame.
A = [[c/lam, -s/lam], [s, c]] maps the pool's balances t to u = A (t - r chi), and the pool keeps ||u|| <= r.  At price p (token 1 per token 0) the boundary point
is where the ellipse's inward normal A' u points along (p, 1), so u(p) = -r A^-T (p, 1) / ||A^-T (p, 1)|| and
t(p) = r chi + A^-1 u(p); chi is fixed by x(beta) = 0 and y(alpha) = 0.  Flows are differences of such points,
computed at 50+ digits, and the optimal trade at prices nu ends where the marginal price meets nu0 / (gamma nu1)
(tender 0) or gamma nu0 / nu1 (tender 1), clamped to the range.  The state (r, p) of balances (x, y) is found by
bisection on the ratio x / y.  Nothing here shares a formula with cfmm_small::eclp_pair.
"""
from __future__ import annotations

import mpmath as mp

DPS = 60


class Pool:
    """One E-CLP in the circle frame, all values mpf."""

    def __init__(self, alpha, beta, c, s, lam):
        self.alpha, self.beta = mp.mpf(alpha), mp.mpf(beta)
        self.c, self.s, self.lam = mp.mpf(c), mp.mpf(s), mp.mpf(lam)
        c, s, lam = self.c, self.s, self.lam
        self.A = ((c / lam, -s / lam), (s, c))
        # A^-1 (det A = (c^2 + s^2) / lam), written out for the 2x2
        det = (c * c + s * s) / lam
        self.Ai = ((c / det, s / lam / det), (-s / det, c / lam / det))
        self.chi = (-self._w(self.beta)[0], -self._w(self.alpha)[1])

    def _w(self, p):
        """A^-1 u(p) / r: the boundary point relative to r chi, per unit r"""
        A = self.A
        # v = A^-T (p, 1): solve A' v = (p, 1)
        a, b, cc, d = A[0][0], A[1][0], A[0][1], A[1][1]           # A' = [[a, b], [cc, d]]
        det = a * d - b * cc
        v0, v1 = (d * p - b) / det, (a - cc * p) / det
        nv = mp.sqrt(v0 * v0 + v1 * v1)
        u0, u1 = -v0 / nv, -v1 / nv
        Ai = self.Ai
        return (Ai[0][0] * u0 + Ai[0][1] * u1, Ai[1][0] * u0 + Ai[1][1] * u1)

    def point(self, r, p):
        w = self._w(mp.mpf(p))
        return (r * (self.chi[0] + w[0]), r * (self.chi[1] + w[1]))

    def inside(self, r, t):
        """||A (t - r chi)|| / r - 1 (<= 0: feasible)"""
        d0, d1 = t[0] - r * self.chi[0], t[1] - r * self.chi[1]
        A = self.A
        u0, u1 = A[0][0] * d0 + A[0][1] * d1, A[1][0] * d0 + A[1][1] * d1
        return mp.sqrt(u0 * u0 + u1 * u1) / r - 1

    def state(self, x, y):
        """(r, p) of balances (x, y): p by bisection on x / y = X(p) / Y(p), then r"""
        x, y = mp.mpf(x), mp.mpf(y)
        if x == 0:
            p = self.beta
        elif y == 0:
            p = self.alpha
        else:
            lo, hi = self.alpha, self.beta
            for _ in range(4 * DPS):
                mid = (lo + hi) / 2
                X, Y = self.point(1, mid)
                if x * Y < y * X:
                    lo = mid
                else:
                    hi = mid
            p = (lo + hi) / 2
        X, Y = self.point(1, p)
        r = y / Y if X == 0 else x / X if Y == 0 or X * y <= Y * x else y / Y
        return r, p

    def flows(self, r, p, gam, pstar0, pstar1):
        """(D0, D1, L0, L1) of the optimal trade of the state (r, p); pstar0 = nu0 / (gam nu1), pstar1 = gam nu0 / nu1"""
        r, p, gam = mp.mpf(r), mp.mpf(p), mp.mpf(gam)
        t = self.point(r, p)
        if pstar0 < p:
            q = max(pstar0, self.alpha)
            tq = self.point(r, q)
            return (tq[0] - t[0]) / gam, mp.mpf(0), mp.mpf(0), t[1] - tq[1]
        if pstar1 > p:
            q = min(pstar1, self.beta)
            tq = self.point(r, q)
            return mp.mpf(0), (tq[1] - t[1]) / gam, t[0] - tq[0], mp.mpf(0)
        return (mp.mpf(0),) * 4


def response(alpha, beta, c, s, lam, r, p, gam, n0, n1, rel=mp.mpf("1e-25")):
    """The trade at prices (n0, n1), the central differences of the net flows in log nu0 (which give hc and the flows'
    sensitivity to the prices), and the post-trade feasibility.  Returns dict of mpf."""
    with mp.workdps(DPS):
        P = Pool(alpha, beta, c, s, lam)
        r, p, gam, n0, n1 = (mp.mpf(v) for v in (r, p, gam, n0, n1))

        def at(f):
            return P.flows(r, p, gam, n0 * f / (gam * n1), gam * n0 * f / n1)
        D0, D1, L0, L1 = at(1)
        hp, hm = at(1 + rel), at(1 - rel)
        # net flows y_j = L_j - D_j; d y / d log nu0
        dy0 = ((hp[2] - hp[0]) - (hm[2] - hm[0])) / (2 * rel)
        dy1 = ((hp[3] - hp[1]) - (hm[3] - hm[1])) / (2 * rel)
        t = P.point(r, p)
        after = (t[0] + gam * D0 - L0, t[1] + gam * D1 - L1)
        return {"D": (D0, D1), "L": (L0, L1), "dy0": dy0, "dy1": dy1, "hc": n0 * dy0,
                "feas": P.inside(r, after), "after": after, "t": t}


def reference_rows(args):
    """the reference's (D0, D1, L0, L1, dy0, dy1, hc, excess * r, after0, after1) of each pool of a chunk (P [k, 5], R,
    st [k, 2], g, n0, n1 [k], D, L [k, 2]), with the feasibility of the given trades D, L on the reference's curve"""
    import numpy as np
    P, R, st, g, n0, n1, D, L = args
    out = np.zeros((len(g), 10))
    for i in range(len(g)):
        ref = response(*P[i], st[i, 0], st[i, 1], g[i], n0[i], n1[i])
        excess, after = certify_terms(*P[i], st[i, 0], R[i, 0], R[i, 1], g[i], D[i], L[i])
        out[i] = [float(v) for v in (*ref["D"], *ref["L"], ref["dy0"], ref["dy1"], ref["hc"], excess * st[i, 0], *after)]
    return out


def state(alpha, beta, c, s, lam, x, y):
    with mp.workdps(DPS):
        return Pool(alpha, beta, c, s, lam).state(x, y)


def certify_terms(alpha, beta, c, s, lam, r, x, y, gam, D, L):
    """E-CLP terms for xp_reference-style certificates: the scaled excess of the post-trade state over the pool's
    ellipse (<= 0 feasible) and whether the post-trade balances stay >= 0."""
    with mp.workdps(DPS):
        P = Pool(alpha, beta, c, s, lam)
        after = (mp.mpf(x) + mp.mpf(gam) * mp.mpf(D[0]) - mp.mpf(L[0]),
                 mp.mpf(y) + mp.mpf(gam) * mp.mpf(D[1]) - mp.mpf(L[1]))
        return P.inside(mp.mpf(r), after), after


# ----------------------------------------------------------------------------------------------------------------------
# certificates of whole markets: xp_bins (every other kind) with the E-CLP pools added
# ----------------------------------------------------------------------------------------------------------------------
KIND_ECLP = 11
_STATE = {}


def _pool_state(hp, i):
    """(Pool, r, p, x, y) of E-CLP pool i: the reference's own state of the pool's balances (hp.eclp supplies only the
    parameters)"""
    import numpy as np
    ptr = np.asarray(hp.pool_ptr, np.int64)
    x, y = float(hp.reserves[ptr[i]]), float(hp.reserves[ptr[i] + 1])
    prm = tuple(float(v) for v in np.asarray(hp.eclp)[i, :5])
    key = prm + (x, y)
    if key not in _STATE:
        with mp.workdps(DPS):
            P = Pool(*prm)
            _STATE[key] = (P,) + P.state(x, y) + (x, y)
    return _STATE[key]


def _others(hp):
    import types
    import numpy as np
    kind = np.asarray(hp.kind).copy()
    kind[kind == KIND_ECLP] = 255
    return types.SimpleNamespace(**{**hp.__dict__, "kind": kind, "m": len(kind)})


def market_response(hp, nu):
    """xp_bins.response (every other kind) with the E-CLP pools' exact trades (h = 0: not used by the certificate)"""
    import numpy as np
    import xp_bins as XB
    import xp_reference as XP
    out = XB.response(_others(hp), nu)
    nu = XP.ld(nu)
    ptr, tok = np.asarray(hp.pool_ptr, np.int64), np.asarray(hp.tok_idx, np.int64)
    for i in np.nonzero(np.asarray(hp.kind) == KIND_ECLP)[0].tolist():
        o = ptr[i]
        n0, n1 = nu[tok[o]], nu[tok[o + 1]]
        P, r, p, x, y = _pool_state(hp, i)
        g = float(hp.gamma[i])
        with mp.workdps(DPS):
            m0, m1, gm = mp.mpf(float(n0)), mp.mpf(float(n1)), mp.mpf(g)
            D0, D1, L0, L1 = P.flows(r, p, gm, m0 / (gm * m1), gm * m0 / m1)
        D = XP.ld([float(D0), float(D1)]); L = XP.ld([float(L0), float(L1)])
        out["delta"][o:o + 2] = D; out["lam"][o:o + 2] = L
        out["arb"][i] = n0 * (L[0] - D[0]) + n1 * (L[1] - D[1]); out["h"][i] = 0
    return out


def eclp_feasibility(hp, i, D, L):
    """the post-trade balances' distance outside the pool's ellipse, ||A (t' - r chi)|| - r, over the pool's token scale
    x + y + r (<= 0 feasible); -t'_j and -min(D, L) over the same scale"""
    P, r, p, x, y = _pool_state(hp, i)
    g = float(hp.gamma[i])
    with mp.workdps(DPS):
        after = (mp.mpf(x) + mp.mpf(g) * mp.mpf(float(D[0])) - mp.mpf(float(L[0])),
                 mp.mpf(y) + mp.mpf(g) * mp.mpf(float(D[1])) - mp.mpf(float(L[1])))
        sc = mp.mpf(x) + mp.mpf(y) + r
        v = max(P.inside(r, after) * r / sc, -after[0] / sc, -after[1] / sc,
                -min(float(D[0]), float(D[1]), float(L[0]), float(L[1])) / sc)
    import xp_reference as XP
    return XP.LD(float(v))


def pool_feasibility(hp, delta, lam):
    import numpy as np
    import xp_bins as XB
    import xp_reference as XP
    worst = XB.pool_feasibility(_others(hp), delta, lam)
    ptr = np.asarray(hp.pool_ptr, np.int64)
    for i in np.nonzero(np.asarray(hp.kind) == KIND_ECLP)[0].tolist():
        o = ptr[i]
        worst = max(worst, eclp_feasibility(hp, i, XP.ld(delta)[o:o + 2], XP.ld(lam)[o:o + 2]))
    return worst


_XPE = None


def certify(hp, spec, result, tol, check=True):
    """xp_reference.certify (same five checks, same bounds) with E-CLP pools and every other kind covered"""
    global _XPE
    if _XPE is None:
        import os
        import xp_stableswap as XS
        _XPE = XS._module_copy(os.path.join(os.path.dirname(os.path.abspath(__file__)), "xp_reference.py"),
                               "_xp_reference_eclp")
        _XPE.response = market_response
        _XPE.pool_feasibility = pool_feasibility
    return _XPE.certify(hp, spec, result, tol, check)
