"""Concentrated-liquidity pools (kind 6, a whole Uniswap-v3 tick ladder) for the test references (test helper, not a test
module).

Extended precision, independent of the package (it imports neither the package nor ``oracle/``): a ladder pool's exact
trade at prices nu is the SUM over its non-empty intervals k of the exact bounded-product trade of the position
v3_position(L_k, p_k, p_{k+1}, p) -- reserves (L_k (1/s_k - 1/b_{k+1}), L_k (s_k - b_k)), offsets (L_k / b_{k+1},
L_k b_k), s_k = s clamped to [b_k, b_{k+1}] -- evaluated by xp_reference's longdouble bounded-product closed form.  No
cumulative tables and no search: that is what the product's ladder_pair does, and what this checks.  Pool data is read
from the HostPools fields (lad_ptr, lad_rec: {b, L, Y, X} per bound, of which only b and L are used here, lad_sc: s).

pool_feasibility walks the intervals: a ladder trade is feasible iff its post-trade holdings (X', Y') lie on or above the
ladder's curve, Y' >= Y(s') at the sqrt price s' with X(s') = X' (X falls in s'), both sums formed here in longdouble from
b and L.  certify is xp_reference.certify (same five checks and bounds) on a private copy of that module whose response
and pool_feasibility add the ladder pools to those of xp_stableswap_n (every other kind).
"""
from __future__ import annotations

import os

import numpy as np

import xp_reference as XP
import xp_stableswap as XS
import xp_stableswap_n as XN

LD = XP.LD
KIND_CONCENTRATED = 6
HERE = os.path.dirname(os.path.abspath(__file__))


def intervals(hp):
    """every non-empty interval of every ladder pool: (pool, L, b_k, b_{k+1}) with b, L as longdouble"""
    lp = np.asarray(hp.lad_ptr, np.int64)
    rec = np.asarray(hp.lad_rec, np.float64).reshape(-1, 4)
    nrec = np.diff(lp)
    owner = np.repeat(np.arange(len(nrec)), nrec)
    last = np.zeros(len(rec), bool)
    last[lp[1:][nrec > 0] - 1] = True
    iv = np.nonzero(~last & (rec[:, 1] > 0))[0]
    return owner[iv], XP.ld(rec[iv, 1]), XP.ld(rec[iv, 0]), XP.ld(rec[iv + 1, 0])


def _per_pool(owner, m, *vals):
    """sums over each pool's intervals, longdouble (owner is sorted)"""
    starts = np.flatnonzero(np.r_[True, owner[1:] != owner[:-1]]) if len(owner) else np.zeros(0, np.int64)
    out = []
    for v in vals:
        full = np.zeros((m,) + v.shape[1:], LD)
        if len(owner):
            full[owner[starts]] = np.add.reduceat(v, starts, axis=0)
        out.append(full)
    return out


def ladder_response(hp, nu):
    """(sel, D, L (len(sel), 2), h (len(sel),)) of the ladder pools at prices nu: sums of the intervals' exact trades"""
    nu = XP.ld(nu)
    kind = np.asarray(hp.kind)
    sel = np.nonzero(kind == KIND_CONCENTRATED)[0]
    o, L, b, b1 = intervals(hp)
    s = np.minimum(np.maximum(XP.ld(np.asarray(hp.lad_sc, float)[o, 0]), b), b1)
    R = np.stack([L * (1 / s - 1 / b1), L * (s - b)], 1)
    off = np.stack([L / b1, L * b], 1)
    ptr = np.asarray(hp.pool_ptr, np.int64)
    tok = np.asarray(hp.tok_idx, np.int64)
    nv = nu[np.stack([tok[ptr[o]], tok[ptr[o] + 1]], 1)]
    D, Lm, h = XP._bounded(R, off, XP.ld(np.asarray(hp.gamma, float)[o]), nv)
    Dp, Lp, hp_ = _per_pool(o, hp.m, D, Lm, h)
    return sel, Dp[sel], Lp[sel], hp_[sel]


def _others(hp):
    """hp with its ladder pools marked as a kind no other reference evaluates"""
    import types
    kind = np.asarray(hp.kind).copy()
    kind[kind == KIND_CONCENTRATED] = 255
    return types.SimpleNamespace(**{**hp.__dict__, "kind": kind})


def response(hp, nu):
    """xp_stableswap_n.response (every other kind) with the ladder pools (longdouble); h of a ladder pool is its pair
    coefficient"""
    out = XN.response(_others(hp), nu)
    sel, D, L, h = ladder_response(hp, nu)
    if len(sel):
        ptr = np.asarray(hp.pool_ptr, np.int64)
        off = ptr[sel][:, None] + np.arange(2)
        nv = XP.ld(nu)[np.asarray(hp.tok_idx, np.int64)[off]]
        out["delta"][off.ravel()] = D.ravel(); out["lam"][off.ravel()] = L.ravel()
        out["arb"][sel] = (nv * (L - D)).sum(1); out["h"][sel] = h
    return out


def ladder_curve(hp, sel):
    """per ladder pool (of sel) the sums that define its curve, from b and L: (b (n, T+1) padded with +inf, L, Ycum, Xcum)
    as lists (one array per pool)"""
    lp = np.asarray(hp.lad_ptr, np.int64)
    rec = np.asarray(hp.lad_rec, np.float64).reshape(-1, 4)
    out = []
    for i in sel.tolist():
        b, L = XP.ld(rec[lp[i]:lp[i + 1], 0]), XP.ld(rec[lp[i]:lp[i + 1] - 1, 1])
        Y = np.concatenate([[LD(0)], np.cumsum(L * (b[1:] - b[:-1]))])
        X = np.concatenate([np.cumsum((L * (1 / b[:-1] - 1 / b[1:]))[::-1])[::-1], [LD(0)]])
        out.append((b, L, Y, X))
    return out


def ladder_feasibility(hp, sel, D, L):
    """per ladder pool: (Y(s') - Y') / Y_T with X(s') = X' (<= 0 is feasible), -X' / X_0 if X' < 0, and -min(D, L) over
    the pool's scale, for the trades D, L (n, 2) of the pools sel"""
    D, L = XP.ld(D).reshape(-1, 2), XP.ld(L).reshape(-1, 2)
    g = XP.ld(np.asarray(hp.gamma, float)[sel])
    s = XP.ld(np.asarray(hp.lad_sc, float)[sel, 0])
    v = np.zeros(len(sel), LD)
    for n_, (b, Lq, Y, X) in enumerate(ladder_curve(hp, sel)):
        c = min(max(int(np.searchsorted(b, s[n_], side="right")) - 1, 0), len(Lq) - 1)
        x = X[c + 1] + Lq[c] * (1 / s[n_] - 1 / b[c + 1])
        y = Y[c] + Lq[c] * (s[n_] - b[c])
        Xp = x + g[n_] * D[n_, 0] - L[n_, 0]
        Yp = y + g[n_] * D[n_, 1] - L[n_, 1]
        sx, sy = X[0], Y[-1]
        if Xp < 0:
            w = -Xp / sx
        elif Xp >= X[0]:
            w = -Yp / sy                                    # s' = b_0, Y(b_0) = 0
        else:
            # X' in [X_{j+1}, X_j): s' inside interval j (a non-empty one: X is constant over empty intervals)
            j = int(np.searchsorted(-X, -Xp, side="right")) - 1
            j = min(max(j, 0), len(Lq) - 1)
            sp = 1 / ((Xp - X[j + 1]) / Lq[j] + 1 / b[j + 1]) if Lq[j] > 0 else b[j + 1]
            w = (Y[j] + Lq[j] * (sp - b[j]) - Yp) / sy
        sc = np.array([sx, sy], dtype=LD)
        w = max(w, (-np.minimum(D[n_], L[n_]) / sc).max())
        v[n_] = w
    return v


def pool_feasibility(hp, delta, lam):
    worst = XN.pool_feasibility(_others(hp), delta, lam)
    sel = np.nonzero(np.asarray(hp.kind) == KIND_CONCENTRATED)[0]
    if len(sel):
        off = np.asarray(hp.pool_ptr, np.int64)[sel][:, None] + np.arange(2)
        worst = max(worst, ladder_feasibility(hp, sel, XP.ld(delta)[off], XP.ld(lam)[off]).max())
    return worst


_XPC = XS._module_copy(os.path.join(HERE, "xp_reference.py"), "_xp_reference_concentrated")
_XPC.response = response
_XPC.pool_feasibility = pool_feasibility


def certify(hp, spec, result, tol, check=True):
    """xp_reference.certify (same five checks, same bounds) with ladder pools and every other kind covered"""
    return _XPC.certify(hp, spec, result, tol, check)
