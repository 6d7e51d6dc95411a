"""Price-bin pools (kind 10: Liquidity Book bins, order books, limit orders) for the test references (test helper, not a
test module).

Extended precision, independent of the package (it imports neither the package nor ``oracle/``).  A bins pool trades
exactly like its bins as separate one-bin constant-sum pools with the same fee, so its exact (eps = 0) trade at prices
nu is the sum over its bins k of each bin's own fill, walked bin by bin in longdouble: the ask part (x_k > 0) fills iff
gamma nu0 > p_k nu1 (the pool pays x_k of token 0 for p_k x_k / gamma of token 1), the bid part (y_k > 0) fills iff
nu0 < gamma p_k nu1 (it takes y_k / (gamma p_k) of token 0 and pays y_k of token 1).  No records and no search: that is
what the product's bins_pair does, and what this checks.  The bins are given as (prices, x, y) per pool (bins_of reads
them back from a HostPools' records, which hold them exactly up to one rounding of each sum).

smoothed solves the eps > 0 response the same way: r t - C(t) - p_ref (t - tbar)^2 / (2 sigma) is concave, so its
maximum is the best of each segment's clipped stationary point, every segment tried.  pool_feasibility measures how far
a trade is outside the Minkowski sum of the bins' sets: the token 1 the pool gains must cover the least the bins need
for the token 0 they pay out (C0, the fee-free cost, walked bin by bin).  certify is xp_reference.certify (same five
checks and bounds) with these added to xp_tricrypto's response and feasibility, which cover every other kind.
"""
from __future__ import annotations

import os
import types

import numpy as np

import xp_reference as XP
import xp_stableswap as XS
import xp_tricrypto as XT

LD = XP.LD
KIND_BINS = 10
HERE = os.path.dirname(os.path.abspath(__file__))


def bins_of(hp, i):
    """(prices, x, y) of bins pool i as longdouble, the bins with holdings only, from its records: ask segments carry
    x = dT, bid segments y = -dC"""
    bp = np.asarray(hp.bin_ptr, np.int64)
    rec = np.asarray(hp.bin_rec, np.float64).reshape(-1, 4)[bp[i]:bp[i + 1]]
    z = int(hp.bin_zp[i, 0])
    T, Cc, q = XP.ld(rec[:, 0]), XP.ld(rec[:, 1]), XP.ld(rec[:, 2])
    seg = np.arange(len(rec) - 1)
    p = q[seg]
    x = np.where(seg >= z, T[1:] - T[:-1], 0)
    y = np.where(seg < z, Cc[1:] - Cc[:-1], 0)
    return p, x.astype(LD), y.astype(LD)


def exact(p, x, y, g, n0, n1):
    """(D (2,), L (2,)) of one bins pool at prices (n0, n1), bin by bin"""
    p, x, y = XP.ld(p), XP.ld(x), XP.ld(y)
    g, n0, n1 = LD(g), LD(n0), LD(n1)
    ask = (x > 0) & (g * n0 > p * n1)
    bid = (y > 0) & (n0 < g * p * n1)
    D = np.array([(y[bid] / (g * p[bid])).sum(), (p[ask] * x[ask] / g).sum()], dtype=LD)
    L = np.array([x[ask].sum(), y[bid].sum()], dtype=LD)
    return D, L


def segments(p, x, y, g):
    """the net-flow form at fee g: segments (lo, hi, slope, C at lo) in ascending t, longdouble, from the bins"""
    p, x, y, g = XP.ld(p), XP.ld(x), XP.ld(y), LD(g)
    bid = np.nonzero(y > 0)[0][::-1]
    ask = np.nonzero(x > 0)[0]
    out = []
    t = c = LD(0)
    for k in bid:                                        # outward from t = 0, descending price
        w = y[k] / (g * p[k])
        out.append((t - w, t, g * p[k], c - y[k]))
        t, c = t - w, c - y[k]
    out = out[::-1]
    t = c = LD(0)
    for k in ask:
        out.append((t, t + x[k], p[k] / g, c))
        t, c = t + x[k], c + p[k] * x[k] / g
    return out


def smoothed(p, x, y, g, n0, n1, eps, tbar, pref):
    """(t, C(t) + smoothing) of one bins pool, eps > 0: the best clipped stationary point over every segment"""
    segs = segments(p, x, y, g)
    r = LD(n0) / LD(n1)
    S = segs[-1][1] - segs[0][0]
    a = S / (LD(eps) * LD(pref))
    tbar = LD(tbar)
    best = None
    for lo, hi, s, c0 in segs:
        t = min(max(tbar + a * (r - s), lo), hi)
        C = c0 + s * (t - lo)
        f = r * t - C - (t - tbar) ** 2 / (2 * a)
        if best is None or f > best[0]:
            best = (f, t, C + (t - tbar) ** 2 / (2 * a))
    return best[1], best[2]


def exact_many(p, x, y, g, n0, n1):
    """exact for many pools of K bins each at once: p, x, y (m, K) (padding bins hold nothing), g, n0, n1 (m,).
    Returns D, L (m, 2), longdouble, the same bin-by-bin sums"""
    p, x, y = XP.ld(p), XP.ld(x), XP.ld(y)
    g, n0, n1 = (XP.ld(v)[:, None] for v in (g, n0, n1))
    ask = (x > 0) & (g * n0 > p * n1)
    bid = (y > 0) & (n0 < g * p * n1)
    D = np.stack([np.where(bid, y / (g * p), 0).sum(1), np.where(ask, p * x / g, 0).sum(1)], 1)
    L = np.stack([np.where(ask, x, 0).sum(1), np.where(bid, y, 0).sum(1)], 1)
    return D, L


def smoothed_many(p, x, y, g, n0, n1, eps, tbar, pref):
    """smoothed for many pools of K bins each at once (shapes as exact_many; tbar, pref (m,)): every bid and ask
    segment of every pool tried, padding bins giving empty segments at the ends.  Returns t, C(t) + smoothing (m,)"""
    p, x, y = XP.ld(p), XP.ld(x), XP.ld(y)
    g, n0, n1, tbar, pref = (XP.ld(v)[:, None] for v in (g, n0, n1, tbar, pref))
    pr, yr = p[:, ::-1], y[:, ::-1]                      # bids outward from t = 0: descending price
    w = yr / (g * pr)
    blo, bc = -np.cumsum(w, 1), -np.cumsum(yr, 1)
    ahi, ac = np.cumsum(x, 1), np.cumsum(p * x, 1) / g
    lo = np.concatenate([blo, ahi - x], 1)
    hi = np.concatenate([blo + w, ahi], 1)
    s = np.concatenate([g * pr, p / g], 1)
    c0 = np.concatenate([bc, ac - p * x / g], 1)
    r = n0 / n1
    a = (w.sum(1) + x.sum(1))[:, None] / (LD(eps) * pref)
    t = np.minimum(np.maximum(tbar + a * (r - s), lo), hi)
    C = c0 + s * (t - lo)
    sm = (t - tbar) ** 2 / (2 * a)
    k = np.argmax(r * t - C - sm, 1)
    rows = np.arange(len(k))
    return t[rows, k], (C + sm)[rows, k]


def cost0(p, x, y, u):
    """(c, excess): the fee-free least token 1 c the bins need to pay out u of token 0 (u < 0: minus the most they pay
    for -u) up to their depth, and the part of |u| past it (0 inside)"""
    p, x, y, u = XP.ld(p), XP.ld(x), XP.ld(y), LD(u)
    c = LD(0)
    if u >= 0:
        for k in np.nonzero(x > 0)[0]:
            f = min(x[k], u)
            c += p[k] * f
            u -= f
            if u <= 0:
                return c, LD(0)
        return c, max(u, LD(0))
    u = -u
    for k in np.nonzero(y > 0)[0][::-1]:
        f = min(y[k] / p[k], u)
        c -= p[k] * f
        u -= f
        if u <= 0:
            return c, LD(0)
    return c, max(u, LD(0))


def _others(hp):
    """hp with its bins pools marked as a kind no other reference evaluates"""
    kind = np.asarray(hp.kind).copy()
    kind[kind == KIND_BINS] = 255
    return types.SimpleNamespace(**{**hp.__dict__, "kind": kind, "m": len(kind)})


def response(hp, nu):
    """xp_tricrypto.response (every other kind) with the bins pools (exact, h = 0)"""
    out = XT.response(_others(hp), nu)
    nu = XP.ld(nu)
    sel = np.nonzero(np.asarray(hp.kind) == KIND_BINS)[0]
    ptr = np.asarray(hp.pool_ptr, np.int64)
    tok = np.asarray(hp.tok_idx, np.int64)
    for i in sel.tolist():
        o = ptr[i]
        n0, n1 = nu[tok[o]], nu[tok[o + 1]]
        D, L = exact(*bins_of(hp, i), np.asarray(hp.gamma, float)[i], n0, n1)
        out["delta"][o:o + 2] = D; out["lam"][o:o + 2] = L
        out["arb"][i] = n0 * (L[0] - D[0]) + n1 * (L[1] - D[1]); out["h"][i] = 0
    return out


def bins_feasibility(hp, i, D, L):
    """(C0(u) - e1) / scale with u = L0 - gamma D0, e1 = gamma D1 - L1 (<= 0 is feasible), the token 0 past the bins'
    depth over that depth, and -min(D, L) / scale; scale = sum(y) + sum(p x), the pool's value in token 1"""
    p, x, y = bins_of(hp, i)
    g = LD(np.asarray(hp.gamma, float)[i])
    D, L = XP.ld(D), XP.ld(L)
    sc = max((y.sum() + (p * x).sum()), LD(1e-300))
    u, e1 = L[0] - g * D[0], g * D[1] - L[1]
    c, past = cost0(p, x, y, u)
    depth = max(x.sum() if u >= 0 else (y / p).sum(), LD(1e-300))
    return max((c - e1) / sc, past / depth, (-np.minimum(D, L) / sc).max())


def pool_feasibility(hp, delta, lam):
    worst = XT.pool_feasibility(_others(hp), delta, lam)
    ptr = np.asarray(hp.pool_ptr, np.int64)
    for i in np.nonzero(np.asarray(hp.kind) == KIND_BINS)[0].tolist():
        o = ptr[i]
        worst = max(worst, bins_feasibility(hp, i, XP.ld(delta)[o:o + 2], XP.ld(lam)[o:o + 2]))
    return worst


_XPB = XS._module_copy(os.path.join(HERE, "xp_reference.py"), "_xp_reference_bins")
_XPB.response = response
_XPB.pool_feasibility = pool_feasibility


def certify(hp, spec, result, tol, check=True):
    """xp_reference.certify (same five checks, same bounds) with bins pools and every other kind covered"""
    return _XPB.certify(hp, spec, result, tol, check)
