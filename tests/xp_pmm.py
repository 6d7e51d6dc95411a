"""Extended-precision reference for DODO proactive-market-maker (PMM) pools, in mpmath.

Independent of the package (it reads only the data of a HostPools).  The pool's curve is stated by its two pieces as
points: base short, (b, Q0 + pi (B0 - b)(1 + k (B0 - b) / b)) for b <= B0; quote short, (B0 + (Q0 - q)(1 + k (Q0 - q)
/ q) / pi, q) for q <= Q0.  The pool's state is the point of its short coordinate (B if B < B0, Q if Q < Q0, else the
meeting point).  The marginal price pi (1 - k + k B0^2 / b^2) (or pi / (1 - k + k Q0^2 / q^2)) is inverted for the
end point, b* = B0 sqrt(k pi / (p* - pi + k pi)) or q* = Q0 sqrt(k p* / (pi - p* + k p*)), and every flow is a
difference of two such points at 60 digits.  The vertical excess q - curve(b) of a point measures feasibility: for b >
B0, curve(b) is the root of the quote piece's quadratic.  Nothing here shares a formula with cfmm_small::pmm_pair.
"""
from __future__ import annotations

import mpmath as mp

DPS = 60


class Pool:
    """One PMM pool, all values mpf."""

    def __init__(self, pi, k, B0, Q0):
        self.pi, self.k, self.B0, self.Q0 = (mp.mpf(v) for v in (pi, k, B0, Q0))

    def base_point(self, b):
        d = self.B0 - b
        return b, self.Q0 + self.pi * d * (1 + self.k * d / b)

    def quote_point(self, q):
        e = self.Q0 - q
        return self.B0 + e * (1 + self.k * e / q) / self.pi, q

    def curve(self, b):
        """the quote balance of the curve at base balance b > 0"""
        if b <= self.B0:
            return self.base_point(b)[1]
        c = (b - self.B0) * self.pi                    # (1 - k) e^2 - (Q0 + c) e + c Q0 = 0, the root e < Q0
        s = self.Q0 + c
        e = 2 * c * self.Q0 / (s + mp.sqrt(s * s - 4 * (1 - self.k) * c * self.Q0))
        return self.Q0 - e

    def start(self, B, Q):
        """(point, marginal price) of the state"""
        if B < self.B0:
            return self.base_point(B), self.pi * (1 - self.k + self.k * self.B0 ** 2 / B ** 2)
        if Q < self.Q0:
            return self.quote_point(Q), self.pi / (1 - self.k + self.k * self.Q0 ** 2 / Q ** 2)
        return (self.B0, self.Q0), self.pi

    def end(self, ps):
        if ps >= self.pi:
            return self.base_point(self.B0 * mp.sqrt(self.k * self.pi / (ps - self.pi + self.k * self.pi)))
        return self.quote_point(self.Q0 * mp.sqrt(self.k * ps / (self.pi - ps + self.k * ps)))

    def flows(self, B, Q, gam, lo, hi):
        """(D0, D1, L0, L1) of the optimal trade: tender 0 if lo < P (the price falls to lo), tender 1 if hi > P"""
        s, P = self.start(B, Q)
        if lo < P:
            e = self.end(lo)
            return (e[0] - s[0]) / gam, mp.mpf(0), mp.mpf(0), s[1] - e[1]
        if hi > P:
            e = self.end(hi)
            return mp.mpf(0), (e[1] - s[1]) / gam, s[0] - e[0], mp.mpf(0)
        return (mp.mpf(0),) * 4


def response(pi, k, B0, Q0, B, Q, gam, n0, n1, rel=mp.mpf("1e-25")):
    """The trade at prices (n0, n1), the central differences of the net flows in log nu0 (which give hc and the flows'
    sensitivity to the prices) and the pool's price.  Returns dict of mpf."""
    with mp.workdps(DPS):
        P = Pool(pi, k, B0, Q0)
        B, Q, gam, n0, n1 = (mp.mpf(v) for v in (B, Q, gam, n0, n1))

        def at(f):
            return P.flows(B, Q, gam, n0 * f / (gam * n1), gam * n0 * f / n1)
        D0, D1, L0, L1 = at(1)
        hp, hm = at(1 + rel), at(1 - rel)
        dy0 = ((hp[2] - hp[0]) - (hm[2] - hm[0])) / (2 * rel)
        dy1 = ((hp[3] - hp[1]) - (hm[3] - hm[1])) / (2 * rel)
        return {"D": (D0, D1), "L": (L0, L1), "dy0": dy0, "dy1": dy1, "hc": n0 * dy0, "price": P.start(B, Q)[1]}


def excess(pi, k, B0, Q0, b, q):
    """the vertical excess q - curve(b) of the point (b, q) (>= 0: on or above the curve; -inf for b <= 0)"""
    with mp.workdps(DPS):
        b, q = mp.mpf(b), mp.mpf(q)
        if b <= 0:
            return -mp.inf
        return q - Pool(pi, k, B0, Q0).curve(b)


def after_trade(B, Q, gam, D, L):
    """the pool's balances after the trade (D, L), exact"""
    with mp.workdps(DPS):
        g = mp.mpf(gam)
        return (mp.mpf(B) + g * mp.mpf(float(D[0])) - mp.mpf(float(L[0])),
                mp.mpf(Q) + g * mp.mpf(float(D[1])) - mp.mpf(float(L[1])))


def reference_rows(args):
    """the reference's (D0, D1, L0, L1, dy0, dy1, hc, price, excess after, b after, q after) of each pool of a chunk
    (P [k, 4] = (pi, k, B0, Q0), R [k, 2], g, n0, n1 [k]), with the given trades D, L [k, 2] for the post-trade terms"""
    import numpy as np
    P, R, g, n0, n1, D, L = args
    out = np.zeros((len(g), 11))
    for i in range(len(g)):
        ref = response(*P[i], R[i, 0], R[i, 1], g[i], n0[i], n1[i])
        with mp.workdps(DPS):
            b, q = after_trade(R[i, 0], R[i, 1], g[i], D[i], L[i])
            ex = excess(*P[i], b, q)
        out[i] = [float(v) for v in (*ref["D"], *ref["L"], ref["dy0"], ref["dy1"], ref["hc"], ref["price"], ex, b, q)]
    return out


def targets(B, Q, pi, k, B0, Q0):
    """the adjusted-target rule at 60 digits: (B0, Q0) with the short side's target re-derived so that (B, Q) lies on
    the curve, from the root of pi k d^2 / b + pi d - (Q - Q0) = 0 (or its mirror)"""
    with mp.workdps(DPS):
        B, Q, pi, k, B0, Q0 = (mp.mpf(v) for v in (B, Q, pi, k, B0, Q0))
        if B < B0 and Q >= Q0:
            a, bb, c = pi * k / B, pi, -(Q - Q0)
            return B + (-bb + mp.sqrt(bb * bb - 4 * a * c)) / (2 * a), Q0
        if Q < Q0 and B >= B0:
            a, bb, c = k / (pi * Q), 1 / pi, -(B - B0)
            return B0, Q + (-bb + mp.sqrt(bb * bb - 4 * a * c)) / (2 * a)
        if B >= B0 and Q >= Q0:
            return B, Q
        raise ValueError("both sides short")


# ----------------------------------------------------------------------------------------------------------------------
# certificates of whole markets: xp_eclp (every other kind) with the PMM pools added
# ----------------------------------------------------------------------------------------------------------------------
KIND_PMM = 12


def _pool(hp, i):
    import numpy as np
    ptr = np.asarray(hp.pool_ptr, np.int64)
    B, Q = float(hp.reserves[ptr[i]]), float(hp.reserves[ptr[i] + 1])
    return tuple(float(v) for v in np.asarray(hp.pmm)[i]), B, Q


def _others(hp):
    import types
    import numpy as np
    kind = np.asarray(hp.kind).copy()
    kind[kind == KIND_PMM] = 255
    return types.SimpleNamespace(**{**hp.__dict__, "kind": kind, "m": len(kind)})


def market_response(hp, nu):
    """xp_eclp.market_response (every other kind) with the PMM pools' exact trades (h = 0: not used by the certificate)"""
    import numpy as np
    import xp_eclp as XE
    import xp_reference as XP
    out = XE.market_response(_others(hp), nu)
    nu = XP.ld(nu)
    ptr, tok = np.asarray(hp.pool_ptr, np.int64), np.asarray(hp.tok_idx, np.int64)
    for i in np.nonzero(np.asarray(hp.kind) == KIND_PMM)[0].tolist():
        o = ptr[i]
        n0, n1 = nu[tok[o]], nu[tok[o + 1]]
        prm, B, Q = _pool(hp, i)
        g = float(hp.gamma[i])
        with mp.workdps(DPS):
            m0, m1, gm = mp.mpf(float(n0)), mp.mpf(float(n1)), mp.mpf(g)
            D0, D1, L0, L1 = Pool(*prm).flows(mp.mpf(B), mp.mpf(Q), gm, m0 / (gm * m1), gm * m0 / m1)
        D = XP.ld([float(D0), float(D1)]); L = XP.ld([float(L0), float(L1)])
        out["delta"][o:o + 2] = D; out["lam"][o:o + 2] = L
        out["arb"][i] = n0 * (L[0] - D[0]) + n1 * (L[1] - D[1]); out["h"][i] = 0
    return out


def pmm_feasibility(hp, i, D, L):
    """the post-trade balances' distance below the curve, -(q' - curve(b')), over the pool's value Q + P' B in token 1
    at the larger of its pre- and post-trade prices (<= 0 feasible); -b', -q' and -min(D, L) over the same scale"""
    prm, B, Q = _pool(hp, i)
    g = float(hp.gamma[i])
    with mp.workdps(DPS):
        b, q = after_trade(B, Q, g, D, L)
        pool = Pool(*prm)
        p0 = pool.start(mp.mpf(B), mp.mpf(Q))[1]
        p1 = pool.pi if b <= 0 or q <= 0 else (
            pool.pi * (1 - pool.k + pool.k * pool.B0 ** 2 / b ** 2) if b < pool.B0 else
            pool.pi / (1 - pool.k + pool.k * pool.Q0 ** 2 / q ** 2) if q < pool.Q0 else pool.pi)
        sc = mp.mpf(Q) + max(p0, p1) * mp.mpf(B)
        v = max(-excess(*prm, b, q) / sc if b > 0 else mp.mpf(1), -b / sc, -q / sc,
                -min(float(D[0]), float(D[1]), float(L[0]), float(L[1])) / sc)
    import xp_reference as XP
    return XP.LD(float(v))


def pool_feasibility(hp, delta, lam):
    import numpy as np
    import xp_eclp as XE
    import xp_reference as XP
    worst = XE.pool_feasibility(_others(hp), delta, lam)
    ptr = np.asarray(hp.pool_ptr, np.int64)
    for i in np.nonzero(np.asarray(hp.kind) == KIND_PMM)[0].tolist():
        o = ptr[i]
        worst = max(worst, pmm_feasibility(hp, i, XP.ld(delta)[o:o + 2], XP.ld(lam)[o:o + 2]))
    return worst


_XPM = None


def certify(hp, spec, result, tol, check=True):
    """xp_reference.certify (same five checks, same bounds) with PMM pools and every other kind covered"""
    global _XPM
    if _XPM is None:
        import os
        import xp_stableswap as XS
        _XPM = XS._module_copy(os.path.join(os.path.dirname(os.path.abspath(__file__)), "xp_reference.py"),
                               "_xp_reference_pmm")
        _XPM.response = market_response
        _XPM.pool_feasibility = pool_feasibility
    return _XPM.certify(hp, spec, result, tol, check)
