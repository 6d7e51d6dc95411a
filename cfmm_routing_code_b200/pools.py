"""Device-resident pool storage and the per-evaluation kernel calls.

Replaces the reference's dense local->global matrices A_i (arbitrage.py:42-48) with index rows, and
its python lists ``reserves`` / ``fees`` (arbitrage.py:14-28) with slot-major SoA buckets in HBM,
one bucket per (kind, arity).  All compute goes through libcfmm_b200.so; nothing here has a CPU path.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import functools
from collections.abc import Mapping
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib

KIND_GEOMEAN_HOST = 0   # host CSR convention: 0 = (weighted) geometric mean, 1 = constant sum
KIND_SUM_HOST = 1
KIND_BOUNDED_HOST = 3   # constant product on virtual reserves (reserves + offsets), real reserves >= 0; offsets ride in `weights`
KIND_STABLESWAP_HOST = 4  # StableSwap (Curve), 2..8 coins; rates ride in `weights`, the amplification in HostPools.amp
ANN_MAX = 4e7           # largest StableSwap coefficient A n^n accepted, any coin count (A <= 1e7 for two coins)
STABLE_ARITY_MAX = 8    # most coins of a StableSwap pool
KIND_CONCENTRATED_HOST = 6  # concentrated liquidity: a whole Uniswap-v3 tick ladder; records in HostPools.lad_rec
KIND_CRYPTOSWAP_HOST = 8  # Curve cryptoswap, 2 or 3 coins; price scales ride in `weights`, A in HostPools.amp, gamma in .cgam
KIND_BINS_HOST = 10     # price bins (Liquidity Book, order books, limit orders); records in HostPools.bin_rec
CRYPTO_A_RANGE = (1e-6, 1e4)       # accepted whitepaper A of cryptoswap pools (the concavity of D is checked over it)
CRYPTO_GAMMA_RANGE = (1e-6, 0.1)   # accepted curve gamma of cryptoswap pools (tests/test_cryptoswap.py checks the corners)
LADDER_T_MAX = 1 << 20  # most intervals of one concentrated pool (cfmm_small::LADDER_T_MAX)
BINS_K_MAX = 1 << 20    # most bins of one price-bin pool (cfmm_small::BINS_K_MAX)


def ladder_records(bounds, liquidity) -> np.ndarray:
    """Records of concentrated pools with T intervals each: bounds (m, T + 1) prices (token 1 per token 0), strictly
    increasing, and liquidity (m, T) >= 0.  Returns (m, T + 1, 4) f64 {b_k, L_k, Y_k, X_k}: the sqrt bound
    b_k = sqrt(bounds_k), the liquidity of [b_k, b_{k+1}) (L_T = 0), the token 1 held below b_k,
    Y_k = sum_{j<k} L_j (b_{j+1} - b_j), and the token 0 held above it, X_k = sum_{j>=k} L_j (1/b_j - 1/b_{j+1}).  The sums
    run in extended precision (numpy longdouble) over the f64 b and L and are rounded once, so each entry is within about
    an ulp of the exact sum of the stored b and L (for T up to a few thousand on x86-64)."""
    b = np.sqrt(np.asarray(bounds, np.float64).reshape(len(bounds), -1))
    Lq = np.asarray(liquidity, np.float64).reshape(len(b), -1)
    m, T1 = b.shape
    bl, Ll = b.astype(np.longdouble), Lq.astype(np.longdouble)
    Y = np.zeros((m, T1), np.longdouble); X = np.zeros((m, T1), np.longdouble)
    Y[:, 1:] = np.cumsum(Ll * (bl[:, 1:] - bl[:, :-1]), 1)
    X[:, :-1] = np.cumsum((Ll * ((bl[:, 1:] - bl[:, :-1]) / (bl[:, :-1] * bl[:, 1:])))[:, ::-1], 1)[:, ::-1]
    out = np.zeros((m, T1, 4))
    out[:, :, 0] = b
    out[:, :-1, 1] = Lq
    out[:, :, 2] = Y.astype(np.float64)
    out[:, :, 3] = X.astype(np.float64)
    return out


def ladder_state(lad_ptr, lad_rec, pool_ids, prices):
    """The per-pool state of concentrated pools at new prices: (s, c, x, y), each (n,) f64.  s = sqrt(price) clamped to
    [b_0, b_T] (the trading set is the same for every price beyond an end); c = the interval holding s (the largest c <= T - 1
    with b_c <= s); the real reserves y = Y_c + L_c (s - b_c) and x = X_{c+1} + L_c (b_{c+1} - s) / (s b_{c+1}), evaluated
    in extended precision and rounded once.  Elementwise: a pool's result does not depend on the other pools of the call,
    so PoolStore.update_pools writes the same bits as a fresh HostPools."""
    ids = np.asarray(pool_ids, np.int64).reshape(-1)
    ptr = np.asarray(lad_ptr, np.int64)
    rec = np.asarray(lad_rec, np.float64).reshape(-1, 4)
    first = ptr[ids]
    return _ladder_state(lambda i, k: rec[i, k], first, ptr[ids + 1] - first - 1, prices)


def _ladder_state(col, first, T, prices):
    """ladder_state on pools given by their first record and T, with col(i, k) = column k of records i"""
    with np.errstate(invalid="ignore"):
        s = np.minimum(np.maximum(np.sqrt(np.asarray(prices, np.float64).reshape(-1)), col(first, 0)), col(first + T, 0))
    lo, hi = np.zeros(len(first), np.int64), T - 1                   # the largest c in [lo, hi] with b_c <= s
    for _ in range(24):
        act = lo < hi
        if not act.any():
            break
        mid = (lo + hi + 1) // 2
        up = act & (col(first + mid, 0) <= s)
        lo = np.where(up, mid, lo)
        hi = np.where(act & ~up, mid - 1, hi)
    c = lo
    bc, Lc, Yc = (col(first + c, k).astype(np.longdouble) for k in (0, 1, 2))
    bc1, Xc1 = (col(first + c + 1, k).astype(np.longdouble) for k in (0, 3))
    sl = s.astype(np.longdouble)
    y = (Yc + Lc * (sl - bc)).astype(np.float64)
    x = (Xc1 + Lc * ((bc1 - sl) / (sl * bc1))).astype(np.float64)
    return s, c.astype(np.float64), x, y


def _check_ladder(price, bounds, liquidity, where=""):
    """The value rules of one concentrated pool given as (price, bounds, liquidity)"""
    p, b, L = np.asarray(price, float), np.asarray(bounds, float).reshape(-1), np.asarray(liquidity, float).reshape(-1)
    if p.size != 1 or not bool(np.isfinite(p) & (p > 0)):
        raise ValueError(f"{where}concentrated price must be finite and > 0")
    if len(b) < 2 or len(L) != len(b) - 1:
        raise ValueError(f"{where}concentrated pools need T + 1 >= 2 bounds and T liquidities")
    if len(L) > LADDER_T_MAX:
        raise ValueError(f"{where}concentrated pools take at most {LADDER_T_MAX} intervals")
    if not bool(np.all(np.isfinite(b) & (b > 0))) or not bool(np.all(b[1:] > b[:-1])):
        raise ValueError(f"{where}concentrated bounds must be finite, > 0 and strictly increasing")
    if not bool(np.all(np.isfinite(L) & (L >= 0))) or not bool(np.any(L > 0)):
        raise ValueError(f"{where}concentrated liquidity must be finite, >= 0 and not all zero")


def new_ladders(ladders):
    """Records and state of concentrated pools given as (price, bounds, liquidity) triples (already checked), each as
    HostPools.from_lists makes them: ladder_records of the pool alone (pools of equal T share one call; its rows do not
    interact) and ladder_state at its price.  Returns (records (sum(T + 1), 4) pool after pool, counts T + 1 (n,) int64,
    s, c, x, y (n,) f64)."""
    n = len(ladders)
    T = np.asarray([len(np.asarray(l[2]).reshape(-1)) for l in ladders], np.int64)
    recs = [None] * n
    for t in np.unique(T).tolist():
        sel = np.nonzero(T == t)[0].tolist()
        B = np.stack([np.asarray(ladders[k][1], np.float64).reshape(-1) for k in sel])
        L = np.stack([np.asarray(ladders[k][2], np.float64).reshape(-1) for k in sel])
        for k, r in zip(sel, ladder_records(B, L)):
            recs[k] = r
    cnt = T + 1
    rec = np.concatenate(recs) if n else np.zeros((0, 4))
    ptr = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    s, c, x, y = ladder_state(ptr, rec, np.arange(n), [float(l[0]) for l in ladders])
    return rec, cnt, s, c, x, y


class LadderSlab:
    """The host records of a store's concentrated pools (or of its price-bin pools), replaceable pool by pool
    (PoolStore.update_pools(ladders=), (bins=)).  Pool i's T[i] + 1 records start at first[i] of the concatenation
    [base | own] (T[i] = -1: no records; a bins pool's T is nb - 1): `base` is a HostPools' lad_rec (bin_rec), borrowed
    and never written, `own` an append-only slab of the record runs that replaced others.  A
    replacement appends its records and leaves the ones it supersedes dead; once the dead records outnumber the live
    ones, the live ones are compacted into a new slab in pool order and the base is let go.  So one replacement costs
    O(its records) plus O(m) integer work, amortised, not a copy of every record."""

    def __init__(self, lad_ptr, lad_rec):
        ptr = np.asarray(lad_ptr, np.int64)
        self.base = np.asarray(lad_rec, np.float64).reshape(-1, 4)
        self.first = ptr[:-1].copy()
        self.T = np.diff(ptr) - 1
        self.own = np.zeros((0, 4))
        self.n_own = 0
        self.live, self.dead = int(ptr[-1]), 0

    def col(self, i, k):
        """column k of records i (indices into [base | own])"""
        nb = len(self.base)
        if self.n_own == 0:
            return self.base[i, k]
        if nb == 0:
            return self.own[i, k]
        inb = i < nb
        return np.where(inb, self.base[np.where(inb, i, 0), k], self.own[np.where(inb, 0, i - nb), k])

    def records(self, pool: int) -> np.ndarray:
        """(T + 1, 4) records of one pool"""
        i = self.first[pool] + np.arange(self.T[pool] + 1)
        return np.stack([self.col(i, k) for k in range(4)], 1)

    def state(self, ids, prices):
        """ladder_state of pools ids at new prices, from these records"""
        ids = np.asarray(ids, np.int64)
        return _ladder_state(self.col, self.first[ids], self.T[ids], prices)

    def replace(self, ids, rec, cnt):
        """pools ids (distinct, concentrated) take new records rec, cnt[k] of them for ids[k], pool after pool"""
        ids = np.asarray(ids, np.int64)
        old = int((self.T[ids] + 1).sum())
        need = len(rec)
        if self.n_own + need > len(self.own):                         # grow geometrically: appends stay amortised O(1)
            grown = np.empty((max(2 * len(self.own), self.n_own + need), 4))
            grown[:self.n_own] = self.own[:self.n_own]
            self.own = grown
        self.own[self.n_own:self.n_own + need] = rec
        self.first[ids] = len(self.base) + self.n_own + np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
        self.T[ids] = np.asarray(cnt, np.int64) - 1
        self.n_own += need
        self.live += need - old
        self.dead += old
        if self.dead > self.live:
            self._compact()

    def _compact(self):
        lad = np.nonzero(self.T >= 0)[0]
        cnt = self.T[lad] + 1
        start = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
        i = np.repeat(self.first[lad] - start, cnt) + np.arange(int(cnt.sum()), dtype=np.int64)
        self.own = np.stack([self.col(i, k) for k in range(4)], 1)
        self.base = np.zeros((0, 4))
        self.n_own = len(self.own)
        self.first[lad] = start
        self.live, self.dead = self.n_own, 0


def stableswap_invariant(reserves, rates, amp) -> np.ndarray:
    """Invariant D of two-coin StableSwap pools: the root of 4A (y0 + y1) + D = 4A D + D^3 / (4 y0 y1) with the scaled
    balances y = rates * reserves.  reserves, rates: (m, 2); amp: (m,), the whitepaper amplification A (a contract's
    A() / n^(n-1) = A() / 2; earlier versions of this docstring called it Curve's A(), which it is not).  Curve's get_D Newton
    iteration in fp64 on the balances in units of y0 + y1 (the invariant is homogeneous of degree 1), from D = y0 + y1
    down to the root (monotone: the cubic is convex there); a pool stops once a step
    moves D by at most 2 ulp.  Elementwise: a pool's D does not depend on the other pools of the call, so a subset
    (PoolStore.update_pools) gives the same bits as the whole."""
    y = np.asarray(reserves, np.float64).reshape(-1, 2) * np.asarray(rates, np.float64).reshape(-1, 2)
    A = np.asarray(amp, np.float64).reshape(-1)
    scale = y[:, 0] + y[:, 1]
    with np.errstate(all="ignore"):
        y0, y1 = y[:, 0] / scale, y[:, 1] / scale                         # units of y0 + y1: nothing over- or underflows
        S = y0 + y1
        out = S.copy()
        act = np.arange(len(S))
        for _ in range(255):
            if len(act) == 0:
                break
            d, ann = out[act], 4.0 * A[act]
            dp = d * d / (2.0 * y0[act]) * d / (2.0 * y1[act])               # D^3 / (4 y0 y1)
            dn = (ann * S[act] + 2.0 * dp) * d / ((ann - 1.0) * d + 3.0 * dp)
            out[act] = dn
            act = act[~(np.abs(dn - d) <= 4.5e-16 * dn)]
    return out * scale


def stableswap_invariant_n(reserves, rates, amp) -> np.ndarray:
    """Invariant D of n-coin StableSwap pools (n = 2..8, one n per call): the root of
        A n^n sum(y) + D = A n^n D + D^(n+1) / (n^n prod(y)),     y = rates * reserves,
    with A the whitepaper amplification (a contract's A() / n^(n-1)).  reserves, rates: (m, n); amp: (m,).  Curve's get_D
    generalised: the Newton step D <- (Ann S + n D_P) D / ((Ann - 1) D + (n + 1) D_P), D_P = D^(n+1) / (n^n prod y),
    Ann = A n^n, in fp64 on the balances in units of S = sum(y).  It starts from the upper bound
    D0 = min(S, ((Ann + 1) S n^n prod y)^(1/(n+1))) (D_P <= Ann S + D <= (Ann + 1) S at the root), so an imbalanced
    pool does not crawl down from S; Newton on this convex function then falls monotonically to the root.  A pool stops
    once a step moves D by at most 2 ulp.  Elementwise, like stableswap_invariant.  Two-coin pools should go through
    stableswap_invariant, whose arithmetic HostPools has always used (stableswap_invariant_any dispatches)."""
    R = np.asarray(reserves, np.float64)
    n = R.shape[-1]
    y = R.reshape(-1, n) * np.asarray(rates, np.float64).reshape(-1, n)
    ann = np.asarray(amp, np.float64).reshape(-1) * float(n ** n)
    # every sum over the coins runs column by column in index order: numpy's row reductions take a different order
    # for C- and F-ordered inputs (at n = 8), and HostPools and PoolStore.update_pools must get the same bits
    colsum = lambda x: functools.reduce(lambda acc, j: acc + x[:, j], range(1, n), x[:, 0].copy())
    scale = colsum(y)
    with np.errstate(all="ignore"):
        y = y / scale[:, None]                                            # units of S: nothing over- or underflows
        S = colsum(y)
        lg = (np.log(ann + 1.0) + np.log(S) + n * np.log(n) + colsum(np.log(y))) / (n + 1)
        out = np.minimum(S, np.exp(lg) * (1.0 + 1e-12))
        act = np.arange(len(S))
        for _ in range(255):
            if len(act) == 0:
                break
            d, a_, ya = out[act], ann[act], y[act]
            dp = d.copy()
            for j in range(n):
                dp = dp * d / (n * ya[:, j])
            dn = (a_ * S[act] + n * dp) * d / ((a_ - 1.0) * d + (n + 1) * dp)
            out[act] = dn
            act = act[~(np.abs(dn - d) <= 4.5e-16 * dn)]
    return out * scale


def stableswap_invariant_any(reserves, rates, amp) -> np.ndarray:
    """D of StableSwap pools of one coin count: stableswap_invariant for two coins, stableswap_invariant_n for more"""
    n = np.asarray(reserves).shape[-1]
    return (stableswap_invariant if n == 2 else stableswap_invariant_n)(reserves, rates, amp)


def cryptoswap_invariant(reserves, scales, amp, cgam) -> np.ndarray:
    """Invariant D of two-coin cryptoswap pools: with y = scales * reserves, K0 = 4 y0 y1 / D^2 and
    K = A K0 G^2 / (G + 1 - K0)^2 the root D in [2 sqrt(y0 y1), y0 + y1] of
        f(D) = K D (y0 + y1) + y0 y1 - K D^2 - (D/2)^2.
    reserves, scales: (m, 2); amp: (m,), the whitepaper A; cgam: (m,), the curve gamma G.  Newton's method on f in D (what
    Curve's newton_D runs, here in fp64 and in units of y0 + y1, so nothing over- or underflows), from the upper bound
    D = y0 + y1, kept inside the bracket by a bisection step whenever Newton would leave it; where |y0 - y1| < D, 1 - K0
    is formed as ((y0 - y1)^2 - (S - D)(S + D)) / D^2, without cancellation near the peg.  A pool stops once a step moves D by at most
    2 ulp.  Elementwise, each pool's arithmetic in a fixed order: a subset (PoolStore.update_pools) gives the same bits as
    the whole."""
    y = np.asarray(reserves, np.float64).reshape(-1, 2) * np.asarray(scales, np.float64).reshape(-1, 2)
    A = np.asarray(amp, np.float64).reshape(-1)
    G = np.asarray(cgam, np.float64).reshape(-1)
    scale = y[:, 0] + y[:, 1]
    with np.errstate(all="ignore"):
        y0, y1 = y[:, 0] / scale, y[:, 1] / scale
        S, P, dy2 = y0 + y1, y0 * y1, (y0 - y1) * (y0 - y1)
        lo, hi = 2.0 * np.sqrt(P), S.copy()
        out = S.copy()
        act = np.arange(len(S))
        for _ in range(255):
            if len(act) == 0:
                break
            d, a, g, s_, p_ = out[act], A[act], G[act], S[act], P[act]
            # 1 - K0, from whichever form cancels less: (y0 - y1)^2 and S^2 - D^2 are each below D^2 where |y0 - y1| < D
            near = dy2[act] < d * d
            K0 = np.where(near, 0.0, 4.0 * p_ / (d * d))
            m = np.where(near, (dy2[act] - (s_ - d) * (s_ + d)) / (d * d), 1.0 - K0)
            K0 = np.where(near, 1.0 - m, K0)
            gm = g + m
            K = a * K0 * g * g / (gm * gm)
            f = K * d * (s_ - d) - 0.25 * m * d * d                        # y0 y1 - D^2 / 4 = -(1 - K0) D^2 / 4
            # df/dD: dK/dD = K'(K0) dK0/dD, dK0/dD = -2 K0 / D, K'(K0) = A G^2 (G + 2 - m) / (G + m)^3
            dK = -2.0 * K0 / d * a * g * g * (g + 2.0 - m) / (gm * gm * gm)
            fp = dK * d * (s_ - d) + K * (s_ - 2.0 * d) - 0.5 * d
            lo[act] = np.where(f > 0, d, lo[act])
            hi[act] = np.where(f > 0, hi[act], d)
            dn = d - f / fp
            dn = np.where(f == 0, d, np.where((dn > lo[act]) & (dn < hi[act]), dn, 0.5 * (lo[act] + hi[act])))
            out[act] = dn
            act = act[~((np.abs(dn - d) <= 4.5e-16 * dn) | (f == 0))]
    return out * scale


def tricrypto_invariant(reserves, scales, amp, cgam) -> np.ndarray:
    """Invariant D of three-coin cryptoswap pools (tricrypto-ng): with y = scales * reserves, S = sum y, P = prod y,
    K0 = 27 P / D^3 and K = A K0 G^2 / (G + 1 - K0)^2 the root D in [3 P^(1/3), S] of
        K D^2 S + P = K D^3 + (D/3)^3,   i.e.   F(D) = K (S - D) - (1 - K0) D / 27 = 0.
    reserves, scales: (m, 3); amp: (m,), the whitepaper A; cgam: (m,), the curve gamma G.  Newton's method on F in D, in
    fp64 and in units of S (homogeneous: nothing over- or underflows), from the upper bound D = S, kept inside the
    bracket by a bisection step whenever Newton would leave it.  Where every |e_j| < 1, e_j = 3 y_j / D - 1, 1 - K0 is
    formed as -(e_0 + e_1 + e_2 + e_0 e_1 + e_0 e_2 + e_1 e_2 + e_0 e_1 e_2) with e_0 + e_1 + e_2 = 3 (S - D) / D: no
    cancellation near the peg; elsewhere as 1 - 27 P / D^3.  A pool stops once a step moves D by at most 2 ulp.  Elementwise, each pool's arithmetic in a fixed
    order: a subset (PoolStore.update_pools) gives the same bits as the whole."""
    y = np.asarray(reserves, np.float64).reshape(-1, 3) * np.asarray(scales, np.float64).reshape(-1, 3)
    A = np.asarray(amp, np.float64).reshape(-1)
    G = np.asarray(cgam, np.float64).reshape(-1)
    scale = y.sum(1)
    with np.errstate(all="ignore"):
        u = y / scale[:, None]
        S = u.sum(1)
        lo, hi = 3.0 * np.cbrt(u[:, 0] * u[:, 1] * u[:, 2]), S.copy()
        out = S.copy()
        act = np.arange(len(S))
        for _ in range(255):
            if len(act) == 0:
                break
            d, a, g, s_ = out[act], A[act], G[act], S[act]
            e = (3.0 * u[act] - d[:, None]) / d[:, None]
            # near the peg (every |e_j| < 1) from the e_j; far from it 27 P / D^3 directly (the e_j terms cancel there)
            near = np.abs(e).max(1) < 1.0
            K0 = np.where(near, 0.0, 27.0 * (u[act, 0] / d) * (u[act, 1] / d) * (u[act, 2] / d))
            m = np.where(near, -(3.0 * (s_ - d) / d + (e[:, 0] * e[:, 1] + e[:, 0] * e[:, 2] + e[:, 1] * e[:, 2])
                                 + e[:, 0] * e[:, 1] * e[:, 2]), 1.0 - K0)
            K0 = np.where(near, 1.0 - m, K0)
            gm = g + m
            K = a * K0 * g * g / (gm * gm)
            K1 = a * g * g * (g + 1.0 + K0) / (gm * gm * gm)              # dK/dK0
            f = K * (s_ - d) - m * d / 27.0
            # dF/dD: dK0/dD = -3 K0 / D, dm/dD = 3 K0 / D
            fp = -3.0 * K0 * K1 * (s_ - d) / d - K - (m + 3.0 * K0) / 27.0
            lo[act] = np.where(f > 0, d, lo[act])
            hi[act] = np.where(f > 0, hi[act], d)
            dn = d - f / fp
            dn = np.where(f == 0, d, np.where((dn > lo[act]) & (dn < hi[act]), dn, 0.5 * (lo[act] + hi[act])))
            out[act] = dn
            act = act[~((np.abs(dn - d) <= 4.5e-16 * dn) | (f == 0))]
    return out * scale


def cryptoswap_invariant_any(reserves, scales, amp, cgam) -> np.ndarray:
    """cryptoswap_invariant or tricrypto_invariant by the pools' coin count (the last axis of reserves: 2 or 3)"""
    n = np.asarray(reserves).shape[-1]
    return (cryptoswap_invariant if n == 2 else tricrypto_invariant)(reserves, scales, amp, cgam)


def _crypto_groups(kind, pool_ptr):
    """(n, pool ids, (m, n) CSR offsets) of the cryptoswap pools, one entry per coin count"""
    cs = np.nonzero(np.asarray(kind) == KIND_CRYPTOSWAP_HOST)[0]
    if len(cs) == 0:
        return []
    ptr = np.asarray(pool_ptr, np.int64)
    ar = ptr[cs + 1] - ptr[cs]
    return [(int(k), cs[ar == k], ptr[cs[ar == k]][:, None] + np.arange(k)) for k in np.unique(ar).tolist()]


def _stable_groups(kind, pool_ptr):
    """(n, pool ids, (m, n) CSR offsets) of the StableSwap pools, one entry per coin count"""
    ss = np.nonzero(np.asarray(kind) == KIND_STABLESWAP_HOST)[0]
    if len(ss) == 0:
        return []
    ptr = np.asarray(pool_ptr, np.int64)
    ar = ptr[ss + 1] - ptr[ss]
    return [(int(k), ss[ar == k], ptr[ss[ar == k]][:, None] + np.arange(k)) for k in np.unique(ar).tolist()]


def _check_bins(prices, x, y, where=""):
    """The value rules of one price-bin pool given as (prices, x, y)"""
    p, x, y = (np.asarray(v, np.float64).reshape(-1) for v in (prices, x, y))
    if not (len(p) == len(x) == len(y)) or not 1 <= len(p) <= BINS_K_MAX:
        raise ValueError(f"{where}bins need 1..{BINS_K_MAX} bins with one price, x and y each")
    if not (np.all(np.isfinite(p) & (p > 0)) and np.all(np.diff(p) > 0)):
        raise ValueError(f"{where}bin prices must be finite, > 0 and strictly increasing")
    if not (np.all(np.isfinite(x) & (x >= 0)) and np.all(np.isfinite(y) & (y >= 0))) or not (x.any() or y.any()):
        raise ValueError(f"{where}bin holdings must be finite, >= 0 and not all zero")
    if x.any() and y.any() and p[y > 0].max() > p[x > 0].min():
        raise ValueError(f"{where}bins are crossed: a bin holding token 1 prices above a bin holding token 0")
    return p, x, y


def bin_records(prices, x, y):
    """Records of one price-bin pool (include/cfmm_b200.h, CFMM_KIND_BINS) from its checked (prices, x, y): (records
    (nb, 4) {T, C, q, bin}, z, p_ref, (sum x, sum y)).  Both sides are summed outward from t = 0 in extended precision and
    rounded once per record."""
    p, x, y = (np.asarray(v, np.float64) for v in (prices, x, y))
    ld = np.longdouble
    bid = np.nonzero(y > 0)[0][::-1]                 # descending price: outward from t = 0
    ask = np.nonzero(x > 0)[0]                       # ascending price
    z, nb = len(bid), len(bid) + len(ask) + 1
    rec = np.zeros((nb, 4))
    rec[z + 1:, 0] = np.cumsum(x[ask].astype(ld)).astype(np.float64)
    rec[z + 1:, 1] = np.cumsum(p[ask].astype(ld) * x[ask].astype(ld)).astype(np.float64)
    rec[z:nb - 1, 2], rec[z:nb - 1, 3] = p[ask], ask
    rec[:z, 0] = (-np.cumsum(y[bid].astype(ld) / p[bid].astype(ld))).astype(np.float64)[::-1]
    rec[:z, 1] = (-np.cumsum(y[bid].astype(ld))).astype(np.float64)[::-1]
    rec[:z, 2], rec[:z, 3] = p[bid][::-1], bid[::-1]
    rec[nb - 1, 3] = -1.0
    pref = float(p[ask[0]] if len(ask) else p[bid[0]])
    sums = (float(np.sum(x.astype(ld))), float(np.sum(y.astype(ld))))
    if not np.all(np.isfinite(rec)):
        raise ValueError("bin records must be finite (token amounts out of fp64 range?)")
    return rec, z, pref, sums


def new_bins(triples):
    """Records and state of price-bin pools given as (prices, x, y) triples (already checked), each as
    HostPools.from_lists makes them: bin_records of the pool alone.  Returns (records (sum nb, 4) pool after pool,
    counts nb (n,) int64, state (n, 4) f64 = (z, p_ref, sum x, sum y)), the arguments of cfmm_bins_splice."""
    return _pack_bins([bin_records(*t) for t in triples])


def _pack_bins(recs):
    """new_bins from the pools' bin_records results"""
    cnt = np.asarray([len(r[0]) for r in recs], np.int64)
    rec = np.concatenate([r[0] for r in recs]) if recs else np.zeros((0, 4))
    state = np.asarray([(r[1], r[2], r[3][0], r[3][1]) for r in recs], np.float64).reshape(-1, 4)
    return rec, cnt, state


def bin_fills(hp: "HostPools", i: int, t: float):
    """How a net trade t of price-bin pool i (t > 0: the pool pays out t of token 0; t < 0: it takes in -t; the net-flow
    form of CFMM_KIND_BINS) splits over its bins, best price first, at the bin prices and the pool's fee: (bins, flow0,
    flow1), each bin's caller-order index and the token 0 and token 1 it pays to the trader (negative: it receives them,
    tender before the fee).  The flows sum to (t, -C(t)) of the exact (eps = 0) evaluation; a t past the pool's depth is
    filled up to its depth."""
    if int(np.asarray(hp.kind)[i]) != KIND_BINS_HOST:
        raise ValueError(f"pool {i} is not a bins pool")
    rec = np.asarray(hp.bin_rec, np.float64).reshape(-1, 4)[int(hp.bin_ptr[i]):int(hp.bin_ptr[i + 1])]
    return _bin_fills(rec, int(hp.bin_zp[i, 0]), float(hp.gamma[i]), t)


def _bin_fills(rec, z, g, t):
    """bin_fills of one pool given by its records (nb, 4), the index z of its t = 0 record and its fee g"""
    bins, f0, f1 = [], [], []
    if t > 0:
        for j in range(z, len(rec) - 1):
            w = rec[j + 1, 0] - rec[j, 0]
            f = min(w, t - rec[j, 0]) if rec[j + 1, 0] > t else w
            bins.append(int(rec[j, 3])); f0.append(f); f1.append(-rec[j, 2] * f / g)
            if rec[j + 1, 0] >= t:
                break
    elif t < 0:
        for j in range(z - 1, -1, -1):
            w = (rec[j + 1, 0] - rec[j, 0]) / g               # token 0 tendered (before the fee) to empty the bin
            f = min(w, rec[j + 1, 0] / g - t)
            bins.append(int(rec[j, 3])); f0.append(-f); f1.append(g * rec[j, 2] * f)
            if rec[j, 0] / g <= t:
                break
    return np.asarray(bins, np.int64), np.asarray(f0), np.asarray(f1)


@dataclasses.dataclass
class HostPools:
    """CSR problem data on the host (numpy)."""
    n_tokens: int
    pool_ptr: np.ndarray   # int64 [m+1]
    tok_idx: np.ndarray    # int32 [nnz]
    reserves: np.ndarray   # f64 [nnz]
    weights: np.ndarray    # f64 [nnz]  normalised per pool; ignored for constant-sum; rates of StableSwap pools
    gamma: np.ndarray      # f64 [m]
    kind: np.ndarray       # uint8 [m]
    amp: Optional[np.ndarray] = None   # f64 [m]  StableSwap amplification A, 0 on other kinds (None: all zero)
    inv: Optional[np.ndarray] = None   # f64 [m]  StableSwap invariant D of the reserves, 0 on other kinds (None: computed)
    # concentrated pools (kind 6): pool i's T + 1 records are lad_rec[lad_ptr[i]:lad_ptr[i+1]] (none on other kinds),
    # {b_k, L_k, Y_k, X_k} as ladder_records; lad_sc[i] = (s, c), the current sqrt price and its interval (ladder_state).
    # Their reserves are the real (x, y) at s; their weights are 0.  None: no concentrated pools.
    lad_ptr: Optional[np.ndarray] = None   # int64 [m+1]
    lad_rec: Optional[np.ndarray] = None   # f64 [n_records, 4]
    lad_sc: Optional[np.ndarray] = None    # f64 [m, 2]
    # cryptoswap pools (kind 8): the curve gamma G (the whitepaper A is in amp, the invariant D in inv, the price scales in
    # weights); 0 on other kinds.  None: all zero.
    cgam: Optional[np.ndarray] = None      # f64 [m]
    # price-bin pools (kind 10): pool i's nb records are bin_rec[bin_ptr[i]:bin_ptr[i+1]] (none on other kinds), as
    # bin_records; bin_zp[i] = (z, p_ref).  Their reserves are (sum x, sum y); their weights are 0.  None: no bins pools.
    bin_ptr: Optional[np.ndarray] = None   # int64 [m+1]
    bin_rec: Optional[np.ndarray] = None   # f64 [n_records, 4]
    bin_zp: Optional[np.ndarray] = None    # f64 [m, 2]

    def __post_init__(self):
        m = len(self.gamma)
        if self.bin_ptr is None:
            self.bin_ptr = np.zeros(m + 1, np.int64)
        if self.bin_rec is None:
            self.bin_rec = np.zeros((0, 4))
        if self.bin_zp is None:
            self.bin_zp = np.zeros((m, 2))
        if self.lad_ptr is None:
            self.lad_ptr = np.zeros(m + 1, np.int64)
        if self.lad_rec is None:
            self.lad_rec = np.zeros((0, 4))
        if self.lad_sc is None:
            self.lad_sc = np.zeros((m, 2))
        if self.amp is None:
            self.amp = np.zeros(m)
        if self.cgam is None:
            self.cgam = np.zeros(m)
        if self.inv is None:
            self.inv = np.zeros(m)
            for _, ss, off in _stable_groups(self.kind, self.pool_ptr):
                self.inv[ss] = stableswap_invariant_any(self.reserves[off], self.weights[off], self.amp[ss])
            for k, cs, off in _crypto_groups(self.kind, self.pool_ptr):
                if k in (2, 3):
                    self.inv[cs] = cryptoswap_invariant_any(self.reserves[off], self.weights[off], self.amp[cs],
                                                            self.cgam[cs])

    @property
    def m(self) -> int:
        return int(len(self.gamma))

    @staticmethod
    def from_lists(n_tokens, local_indices, reserves, fees, kinds, weights=None) -> "HostPools":
        """From the reference's literals: local_indices / reserves / fees (arbitrage.py:6-28) plus
        which cvxpy atom constrains each pool (arbitrage.py:63-74): 'geomean' (with weights[i] = the
        ``p=`` vector), 'product' (cp.geo_mean on 2 tokens) or 'sum'.  Beyond the reference: 'bounded_product' (weights[i]
        = the two virtual-reserve offsets) and 'stableswap' (2..8 coins, weights[i] = (A, r_0, ..., r_{n-1}): the
        whitepaper amplification A, which is a contract's A() / n^(n-1), and Curve's rate multipliers; (A, 1, 1, 1) for a
        plain 3pool-like pool).  Earlier versions of this docstring called A Curve's A(); the math has always taken the
        whitepaper A.  And 'concentrated' (a whole Uniswap-v3 tick ladder as one pool): weights[i] = (price, bounds,
        liquidity) with the current price and the T + 1 price bounds in token 1 per token 0 (the caller's token units;
        instances.v3_ladder converts on-chain state), T >= 1 liquidities >= 0 (not all 0), at most LADDER_T_MAX; reserves[i]
        must be None: the real reserves are derived (ladder_state).  And 'cryptoswap' (a two-coin Curve v2 pool, twocrypto-ng):
        weights[i] = (A, G, p_0, p_1) with A the whitepaper amplification (K -> A K0 as G -> inf, StableSwap's A), G the
        curve's gamma (not the fee) and p_j the price scale times the precision of coin j (only p_0 / p_1 matters);
        A in CRYPTO_A_RANGE, G in CRYPTO_GAMMA_RANGE.  instances.twocrypto_pool converts a contract's state.  Three
        tokens (tricrypto-ng): weights[i] = (A, G, p_0, p_1, p_2), the same A and G rules, invariant tricrypto_invariant;
        instances.tricrypto_pool converts a contract's state.  And 'bins' (price bins: Liquidity Book bins, an order book,
        limit orders): weights[i] = (prices, x, y) with the K bins' prices in token 1 per token 0 (the caller's units),
        strictly increasing, and their holdings x of token 0 and y of token 1, finite, >= 0, not all 0, uncrossed (every
        bin with y > 0 prices at or below every bin with x > 0), 1 <= K <= BINS_K_MAX; reserves[i] must be None (they are
        (sum x, sum y)).  instances.lb_bins and instances.order_book build the triple."""
        m = len(local_indices)
        if not (len(reserves) == len(fees) == len(kinds) == m):
            raise ValueError("local_indices, reserves, fees, kinds must have one entry per pool")
        ptr = [0]; idx: List[int] = []; res: List[float] = []; wts: List[float] = []; kd: List[int] = []
        amp = np.zeros(m)
        cgam = np.zeros(m)
        lad = {}                                         # concentrated pool -> its records and price
        bins = {}                                        # bins pool -> bin_records
        for i, l in enumerate(local_indices):
            k = len(l)
            if kinds[i] == "bins":
                if k != 2 or len(set(int(t) for t in l)) != 2:
                    raise ValueError(f"pool {i}: bins pools need 2 distinct tokens")
                if reserves[i] is not None:
                    raise ValueError(f"pool {i}: a bins pool's reserves[i] must be None (they are derived)")
                if weights is None or weights[i] is None or len(weights[i]) != 3:
                    raise ValueError(f"pool {i}: bins needs weights[i] = (prices, x, y)")
                bins[i] = bin_records(*_check_bins(*weights[i], where=f"pool {i}: "))
                ptr.append(ptr[-1] + 2); idx += [int(t) for t in l]; res += list(bins[i][3]); wts += [0.0, 0.0]
                kd.append(KIND_BINS_HOST)
                continue
            if kinds[i] == "concentrated":
                if k != 2 or len(set(int(t) for t in l)) != 2:
                    raise ValueError(f"pool {i}: concentrated pools need 2 distinct tokens")
                if reserves[i] is not None:
                    raise ValueError(f"pool {i}: a concentrated pool's reserves[i] must be None (they are derived)")
                if weights is None or weights[i] is None or len(weights[i]) != 3:
                    raise ValueError(f"pool {i}: concentrated needs weights[i] = (price, bounds, liquidity)")
                price, bounds, liq = weights[i]
                _check_ladder(price, bounds, liq, f"pool {i}: ")
                lad[i] = (float(price), ladder_records(np.asarray(bounds, float)[None, :], np.asarray(liq, float)[None, :])[0])
                ptr.append(ptr[-1] + 2); idx += [int(t) for t in l]; res += [0.0, 0.0]; wts += [0.0, 0.0]
                kd.append(KIND_CONCENTRATED_HOST)
                continue
            if reserves[i] is None or len(reserves[i]) != k:
                raise ValueError(f"pool {i}: {0 if reserves[i] is None else len(reserves[i])} reserves for {k} tokens")
            if len(set(int(t) for t in l)) != k:
                raise ValueError(f"pool {i}: repeated token in local_indices")
            ptr.append(ptr[-1] + k)
            idx += [int(t) for t in l]
            res += [float(x) for x in reserves[i]]
            if kinds[i] == "sum":
                if k != 2:
                    raise ValueError("constant-sum pools must have 2 tokens (as arbitrage.py:11)")
                kd.append(KIND_SUM_HOST); wts += [0.0] * k
            elif kinds[i] == "bounded_product":
                # not a reference atom: one Uniswap-v3 tick range; weights[i] = the two virtual-reserve offsets
                o = None if (weights is None or weights[i] is None) else np.asarray(weights[i], float)
                if k != 2 or o is None or len(o) != 2 or np.any(o < 0) or not np.all(np.isfinite(o)):
                    raise ValueError(f"pool {i}: bounded_product needs 2 tokens and 2 non-negative offsets in weights[i]")
                kd.append(KIND_BOUNDED_HOST); wts += list(o)
            elif kinds[i] == "stableswap":
                p = None if (weights is None or weights[i] is None) else np.asarray(weights[i], float).reshape(-1)
                if not 2 <= k <= STABLE_ARITY_MAX or p is None or len(p) != k + 1:
                    raise ValueError(f"pool {i}: stableswap needs 2..{STABLE_ARITY_MAX} tokens and weights[i] = "
                                     "(A, r_0, ..., r_{n-1})")
                _check_stableswap(p[0], p[1:], reserves[i], f"pool {i}: ")
                kd.append(KIND_STABLESWAP_HOST); wts += [float(x) for x in p[1:]]; amp[i] = p[0]
            elif kinds[i] == "cryptoswap":
                p = None if (weights is None or weights[i] is None) else np.asarray(weights[i], float).reshape(-1)
                if k not in (2, 3) or p is None or len(p) != k + 2:
                    raise ValueError(f"pool {i}: cryptoswap needs 2 or 3 tokens and weights[i] = (A, gamma, p_0, ..., "
                                     "p_{n-1})")
                _check_cryptoswap(p[0], p[1], p[2:], reserves[i], f"pool {i}: ")
                kd.append(KIND_CRYPTOSWAP_HOST); wts += [float(x) for x in p[2:]]; amp[i] = p[0]; cgam[i] = p[1]
            elif kinds[i] in ("geomean", "product"):
                w = np.ones(k) if (weights is None or weights[i] is None) else np.asarray(weights[i], float)
                if len(w) != k or np.any(w <= 0):
                    raise ValueError(f"pool {i}: bad weights")
                kd.append(KIND_GEOMEAN_HOST); wts += list(w / w.sum())
            else:
                raise ValueError(f"pool {i}: unknown kind {kinds[i]!r}")
        res = np.asarray(res, np.float64)
        lad_ptr = np.zeros(m + 1, np.int64); lad_sc = np.zeros((m, 2)); recs = []
        if lad:
            cnt = np.zeros(m, np.int64)
            for i, (_, r) in lad.items():
                cnt[i] = len(r)
            lad_ptr[1:] = np.cumsum(cnt)
            recs = [lad[i][1] for i in sorted(lad)]
            ids = np.asarray(sorted(lad), np.int64)
            rec = np.concatenate(recs)
            sv, cv, x, y = ladder_state(lad_ptr, rec, ids, [lad[i][0] for i in ids.tolist()])
            lad_sc[ids, 0], lad_sc[ids, 1] = sv, cv
            first = np.asarray(ptr, np.int64)[ids]
            res[first], res[first + 1] = x, y
        bin_ptr = np.zeros(m + 1, np.int64); bin_zp = np.zeros((m, 2)); brec = None
        if bins:
            cnt = np.zeros(m, np.int64)
            for i, b in bins.items():
                cnt[i] = len(b[0]); bin_zp[i] = (b[1], b[2])
            bin_ptr[1:] = np.cumsum(cnt)
            brec = np.concatenate([bins[i][0] for i in sorted(bins)])
        return HostPools(int(n_tokens), np.asarray(ptr, np.int64), np.asarray(idx, np.int32),
                         res, np.asarray(wts, np.float64),
                         np.asarray(fees, np.float64), np.asarray(kd, np.uint8), amp, None, lad_ptr,
                         np.concatenate(recs) if recs else None, lad_sc, cgam, bin_ptr, brec, bin_zp)

    @staticmethod
    def from_pairs(n_tokens, idx, reserves, gamma) -> "HostPools":
        """m constant-product pools given as (m,2) arrays."""
        m = len(gamma)
        hp = HostPools(int(n_tokens), np.arange(0, 2 * m + 1, 2, dtype=np.int64),
                       np.ascontiguousarray(idx, np.int32).reshape(-1),
                       np.ascontiguousarray(reserves, np.float64).reshape(-1),
                       np.full(2 * m, 0.5), np.ascontiguousarray(gamma, np.float64), np.zeros(m, np.uint8))
        hp._uniform_product = True          # known structure: split_buckets / validation take the device-side path
        return hp

    def pin_memory(self) -> "HostPools":
        """Move the arrays into page-locked host memory (in place) so PoolStore uploads run at full PCIe speed."""
        keep = []
        for name in ("tok_idx", "reserves", "weights", "gamma", "kind", "pool_ptr"):
            t = torch.from_numpy(np.ascontiguousarray(getattr(self, name))).pin_memory()
            keep.append(t)
            setattr(self, name, t.numpy())
        self._pinned = keep                  # the numpy views borrow these tensors' storage
        return self

    def validate(self):
        slot_kind = np.repeat(np.asarray(self.kind), np.diff(self.pool_ptr)) if \
            np.any((self.kind == KIND_BOUNDED_HOST) | (self.kind == KIND_CONCENTRATED_HOST) | (self.kind == KIND_BINS_HOST)) \
            else None
        virt = self.reserves if slot_kind is None else self.reserves + np.where(slot_kind == KIND_BOUNDED_HOST, self.weights, 0.0)
        lo_ok = np.all(self.reserves > 0) if slot_kind is None else np.all(self.reserves >= 0) and \
            np.all((virt > 0) | (slot_kind == KIND_CONCENTRATED_HOST) | (slot_kind == KIND_BINS_HOST))
        if not lo_ok or not np.all(np.isfinite(self.reserves)):
            raise ValueError("reserves must be positive and finite (bounded_product: >= 0 with positive virtual reserves; "
                             "concentrated, bins: >= 0)")
        self._validate_ladders()
        self._validate_bins()
        if np.any(self.gamma <= 0) or np.any(self.gamma > 1):
            raise ValueError("fees (gamma) must lie in (0, 1]")
        if self.tok_idx.min(initial=0) < 0 or self.tok_idx.max(initial=0) >= self.n_tokens:
            raise ValueError("token index out of range")
        for k, ss, off in _stable_groups(self.kind, self.pool_ptr):
            if not 2 <= k <= STABLE_ARITY_MAX:
                raise ValueError(f"stableswap pools must have 2..{STABLE_ARITY_MAX} tokens")
            _check_stableswap(self.amp[ss], self.weights[off], self.reserves[off])
            D = np.asarray(self.inv, float)[ss]
            if not bool(np.all(np.isfinite(D) & (D > 0))):
                raise ValueError("stableswap invariant D must be finite and > 0 (scaled balances out of fp64 range?)")
        for k, cs, off in _crypto_groups(self.kind, self.pool_ptr):
            if k not in (2, 3):
                raise ValueError("cryptoswap pools must have 2 or 3 tokens")
            _check_cryptoswap(self.amp[cs], np.asarray(self.cgam, float)[cs], self.weights[off], self.reserves[off])
            D = np.asarray(self.inv, float)[cs]
            if not bool(np.all(np.isfinite(D) & (D > 0))):
                raise ValueError("cryptoswap invariant D must be finite and > 0 (scaled balances out of fp64 range?)")


    def _validate_bins(self):
        """The rules of price-bin pools on the CSR form: arity 2; 2 .. BINS_K_MAX + 2 records, none on other kinds; T
        strictly increasing and finite, record z = (0, 0), C finite, segment prices finite and > 0, p_ref finite, > 0."""
        kind, m = np.asarray(self.kind), self.m
        ptr = np.asarray(self.bin_ptr, np.int64)
        rec = np.asarray(self.bin_rec, np.float64).reshape(-1, 4)
        if len(ptr) != m + 1 or ptr[0] != 0 or np.any(np.diff(ptr) < 0) or ptr[-1] != len(rec):
            raise ValueError("bin_ptr must be a CSR pointer of m + 1 entries over bin_rec")
        bn = kind == KIND_BINS_HOST
        cnt = np.diff(ptr)
        if np.any(cnt[~bn] != 0) or np.any((cnt[bn] < 2) | (cnt[bn] > BINS_K_MAX + 2)):
            raise ValueError(f"bins pools need 1..{BINS_K_MAX} bins (2 .. {BINS_K_MAX + 2} records); other kinds none")
        if not bn.any():
            return
        ids = np.nonzero(bn)[0]
        if np.any(np.diff(self.pool_ptr)[ids] != 2):
            raise ValueError("bins pools must have 2 tokens")
        owner = np.repeat(np.arange(m), cnt)
        last = np.zeros(len(rec), bool); last[ptr[ids + 1] - 1] = True
        inc = np.ones(len(rec), bool); inc[1:] = (rec[1:, 0] > rec[:-1, 0]) | (owner[1:] != owner[:-1])
        if not (np.all(np.isfinite(rec)) and np.all(inc) and np.all((rec[~last, 2] > 0))):
            raise ValueError("bin records must be finite, T strictly increasing, segment prices > 0")
        z, pref = np.asarray(self.bin_zp, float)[ids, 0], np.asarray(self.bin_zp, float)[ids, 1]
        ok = (z == np.floor(z)) & (z >= 0) & (z < cnt[ids]) & np.isfinite(pref) & (pref > 0)
        zi = ptr[ids] + np.where(ok, z, 0).astype(np.int64)
        if not bool(np.all(ok & (rec[zi, 0] == 0) & (rec[zi, 1] == 0))):
            raise ValueError("bins (z, p_ref): record z must be the t = 0 breakpoint and p_ref finite and > 0")

    def _validate_ladders(self):
        """The rules of concentrated pools on the CSR form: arity 2; T + 1 records, 1 <= T <= LADDER_T_MAX, none on other
        kinds; bounds finite, > 0, strictly increasing; liquidity finite, >= 0, not all 0, L_T = 0; Y, X finite; (s, c) a
        state of ladder_state."""
        kind, m = np.asarray(self.kind), self.m
        ptr = np.asarray(self.lad_ptr, np.int64)
        rec = np.asarray(self.lad_rec, np.float64).reshape(-1, 4)
        if len(ptr) != m + 1 or ptr[0] != 0 or np.any(np.diff(ptr) < 0) or ptr[-1] != len(rec):
            raise ValueError("lad_ptr must be a CSR pointer of m + 1 entries over lad_rec")
        cl = kind == KIND_CONCENTRATED_HOST
        cnt = np.diff(ptr)
        if np.any(cnt[~cl] != 0) or np.any((cnt[cl] < 2) | (cnt[cl] > LADDER_T_MAX + 1)):
            raise ValueError(f"concentrated pools need 1..{LADDER_T_MAX} intervals (T + 1 records); other kinds none")
        if not cl.any():
            return
        ids = np.nonzero(cl)[0]
        if np.any(np.diff(self.pool_ptr)[ids] != 2):
            raise ValueError("concentrated pools must have 2 tokens")
        owner = np.repeat(np.arange(m), cnt)
        last = np.zeros(len(rec), bool); last[ptr[ids + 1] - 1] = True
        b, L = rec[:, 0], rec[:, 1]
        inc = np.ones(len(rec), bool); inc[1:] = (b[1:] > b[:-1]) | (owner[1:] != owner[:-1])
        if not (np.all(np.isfinite(b) & (b > 0)) and np.all(inc)):
            raise ValueError("concentrated bounds must be finite, > 0 and strictly increasing")
        if not (np.all(np.isfinite(L) & (L >= 0)) and np.all(L[last] == 0)):
            raise ValueError("concentrated liquidity must be finite and >= 0 (0 at the last bound)")
        if not np.all(np.bincount(owner, weights=(L > 0).astype(float), minlength=m)[ids] > 0):
            raise ValueError("concentrated liquidity must not be all zero")
        if not np.all(np.isfinite(rec[:, 2:])):
            raise ValueError("concentrated records must be finite (token amounts out of fp64 range?)")
        s, c = np.asarray(self.lad_sc, float)[ids, 0], np.asarray(self.lad_sc, float)[ids, 1]
        T = cnt[ids] - 1
        ok = np.isfinite(s) & (s >= rec[ptr[ids], 0]) & (s <= rec[ptr[ids] + T, 0]) & (c == np.floor(c)) & (c >= 0) & (c < T)
        ci = np.where(ok, c, 0).astype(np.int64)
        ok &= (rec[ptr[ids] + ci, 0] <= s) & ((rec[ptr[ids] + ci + 1, 0] > s) | (ci == T - 1))
        if not bool(np.all(ok)):
            raise ValueError("concentrated (s, c): s must lie in [b_0, b_T] and c be its interval")


def _check_cryptoswap(A, G, scales, reserves, where=""):
    """The value rules of cryptoswap pools: A in CRYPTO_A_RANGE, G in CRYPTO_GAMMA_RANGE (the domain over which the
    concavity of D is checked), price scales and reserves finite and > 0."""
    A, G, p, R = (np.asarray(x, float) for x in (A, G, scales, reserves))
    if not bool(np.all((A >= CRYPTO_A_RANGE[0]) & (A <= CRYPTO_A_RANGE[1]))):
        raise ValueError(f"{where}cryptoswap amplification A must lie in [{CRYPTO_A_RANGE[0]:g}, {CRYPTO_A_RANGE[1]:g}]")
    if not bool(np.all((G >= CRYPTO_GAMMA_RANGE[0]) & (G <= CRYPTO_GAMMA_RANGE[1]))):
        raise ValueError(f"{where}cryptoswap curve gamma must lie in [{CRYPTO_GAMMA_RANGE[0]:g}, {CRYPTO_GAMMA_RANGE[1]:g}]")
    if not bool(np.all(np.isfinite(p) & (p > 0))):
        raise ValueError(f"{where}cryptoswap price scales must be finite and > 0")
    if not bool(np.all(np.isfinite(R) & (R > 0))):
        raise ValueError(f"{where}cryptoswap reserves must be finite and > 0")


def _check_stableswap(A, rates, reserves, where=""):
    """The value rules of StableSwap pools of n coins (the last axis of rates): A finite, A > 0 and A n^n <= ANN_MAX
    (A <= 1e7 at n = 2), rates finite and > 0, reserves finite and > 0."""
    A, r, R = np.asarray(A, float), np.asarray(rates, float), np.asarray(reserves, float)
    n = r.shape[-1]
    if not bool(np.all((A > 0) & (A * float(n ** n) <= ANN_MAX))):
        raise ValueError(f"{where}stableswap amplification A must be finite, > 0 and A n^n <= {ANN_MAX:g} "
                         f"(A <= {ANN_MAX / n ** n:g} for {n} coins)")
    if not bool(np.all(np.isfinite(r) & (r > 0))):
        raise ValueError(f"{where}stableswap rates must be finite and > 0")
    if not bool(np.all(np.isfinite(R) & (R > 0))):
        raise ValueError(f"{where}stableswap reserves must be finite and > 0")


@dataclasses.dataclass
class PoolUpdate:
    """A checked update of some pools' reserves and fees (check_pool_update)."""
    ids: np.ndarray                  # int64 [n] global pool indices
    ptr: np.ndarray                  # int64 [n+1] pool k's slots are slots[ptr[k]:ptr[k+1]]
    slots: np.ndarray                # int64 [nnz] CSR offsets of the updated pools' slots, pool by pool, in slot order
    reserves: Optional[np.ndarray]   # f64 [nnz] new reserves at `slots`, or None
    gamma: Optional[np.ndarray]      # f64 [n] new fees, or None
    prices: Optional[np.ndarray] = None   # f64 [n] new prices of concentrated pools, or None
    ladders: Optional[list] = None        # [n] new (price, bounds f64, liquidity f64) of concentrated pools, or None
    amp: Optional[np.ndarray] = None      # f64 [n] new amplifications A of StableSwap pools, or None
    rates: Optional[np.ndarray] = None    # f64 [nnz] new rates (price scales) of StableSwap (cryptoswap) pools at `slots`
    curve_gamma: Optional[np.ndarray] = None   # f64 [n] new curve gammas of cryptoswap pools, or None
    bins: Optional[list] = None           # [n] bin_records of the new (prices, x, y) of price-bin pools, or None


def _pool_rows(vals, n, ar, what):
    """per-pool vectors of the pools' arities (a list, or an (n, k) array when all have arity k), flattened in order"""
    if isinstance(vals, np.ndarray) and vals.ndim == 2:
        if len(vals) != n or (n and bool(np.any(ar != vals.shape[1]))):
            raise ValueError(f"{what}: one row per pool, of the pool's arity")
        return np.ascontiguousarray(vals, np.float64).reshape(-1)
    if len(vals) != n:
        raise ValueError(f"{what}: one vector per pool")
    rows = [np.asarray(r, np.float64).reshape(-1) for r in vals]
    if any(len(r) != a for r, a in zip(rows, ar.tolist())):
        raise ValueError(f"{what}: a vector's length differs from its pool's arity")
    return np.concatenate(rows) if rows else np.zeros(0)


def check_pool_update(pool_ptr: np.ndarray, kind: np.ndarray, weights: np.ndarray, pool_ids, reserves=None,
                      fees=None, prices=None, ladders=None, amp=None, rates=None, curve_gamma=None,
                      bins=None) -> PoolUpdate:
    """Host checks of PoolStore.update_pools, on the problem's CSR arrays (pool_ptr, kind, weights as in HostPools).
    pool_ids: global pool indices, distinct and in range; reserves[k]: the new reserve vector of pool pool_ids[k] with the
    pool's arity (a row of the reference's `reserves` literal; an (n, k) array when all pools have arity k); fees[k]: its
    new gamma.  The values must pass the rules of HostPools.validate (bounded_product pools with their own offsets).
    prices[k]: the new price (token 1 per token 0) of pool pool_ids[k], which must then be concentrated; a concentrated pool
    takes no reserves (they are derived from its price).  ladders[k]: the new (price, bounds, liquidity) of concentrated
    pool pool_ids[k], the triple of HostPools.from_lists' weights[i] (T may differ from the pool's old T; the rules of
    from_lists); not together with prices=.  amp[k]: the new whitepaper A of StableSwap pool pool_ids[k], rates[k]: its new
    rate vector (the pool's arity; an (n, k) array as for reserves), under the rules of from_lists.  For cryptoswap pools
    amp[k] is the new whitepaper A, rates[k] the new price scales (p_0, p_1[, p_2]), curve_gamma[k] the new curve gamma (cryptoswap
    pools only); amp= and rates= may not mix StableSwap and cryptoswap pools in one call.  bins[k]: the new
    (prices, x, y) of price-bin pool pool_ids[k], the triple of HostPools.from_lists' weights[i] (K may differ from the
    pool's old K; the rules of from_lists, and records finite as bin_records checks); a bins pool takes no reserves=.
    Raises ValueError; returns the update with the reserves and rates flattened into the pools' CSR slot order and the
    new bins as their bin_records."""
    m = len(pool_ptr) - 1
    ids = np.asarray(pool_ids)
    if ids.ndim != 1 or (ids.size and not np.issubdtype(ids.dtype, np.integer)):
        raise ValueError("pool_ids must be a 1-d sequence of integer pool indices")
    ids = ids.astype(np.int64)
    n = len(ids)
    if all(x is None for x in (reserves, fees, prices, ladders, amp, rates, curve_gamma, bins)):
        raise ValueError("nothing to update: give reserves, fees, prices, ladders, amp, rates, curve_gamma, bins or "
                         "several")
    if n and (ids.min() < 0 or ids.max() >= m):
        raise ValueError(f"pool id out of range [0, {m})")
    if reserves is not None and bool(np.any(np.asarray(kind)[ids] == KIND_BINS_HOST)):
        raise ValueError("bins pools take no reserves= (their reserves are derived from the bins, which are structure)")
    conc = np.asarray(kind)[ids] == KIND_CONCENTRATED_HOST
    if reserves is not None and conc.any():
        raise ValueError("concentrated pools take prices=, not reserves= (their reserves are derived from the price)")
    pr = None
    if prices is not None:
        pr = np.ascontiguousarray(prices, np.float64).reshape(-1)
        if len(pr) != n:
            raise ValueError("prices: one per pool")
        if not bool(np.all(conc)):
            raise ValueError("prices= applies to concentrated pools only")
        if not bool(np.all(np.isfinite(pr) & (pr > 0))):
            raise ValueError("concentrated prices must be finite and > 0")
    srt = np.sort(ids)                                   # (np.unique hashes: 20x slower at 100k ids)
    if bool(np.any(srt[1:] == srt[:-1])):
        raise ValueError("repeated pool id")
    if int(pool_ptr[-1]) == 2 * m:       # every pool of a store has >= 2 tokens, so these are all pairs: no gathers
        ar = np.full(n, 2, np.int64)
        first = 2 * np.arange(n + 1, dtype=np.int64)
        slots = (2 * ids[:, None] + np.arange(2)).reshape(-1)
    else:
        ar = (pool_ptr[ids + 1] - pool_ptr[ids]).astype(np.int64)
        first = np.concatenate([[0], np.cumsum(ar)])
        slots = np.repeat(pool_ptr[ids] - first[:-1], ar) + np.arange(first[-1], dtype=np.int64)
    R = None
    if reserves is not None:
        R = _pool_rows(reserves, n, ar, "reserves")
        bounded = np.repeat(np.asarray(kind)[ids] == KIND_BOUNDED_HOST, ar)
        if bounded.any():
            virt = R + np.where(bounded, weights[slots], 0.0)
            ok = np.where(bounded, R >= 0, True) & (virt > 0)
        else:
            ok = R > 0
        if not (bool(np.all(ok)) and bool(np.all(np.isfinite(R)))):
            raise ValueError("reserves must be positive and finite (bounded_product: >= 0 with positive virtual reserves)")
    g = None
    if fees is not None:
        g = np.ascontiguousarray(fees, np.float64).reshape(-1)
        if len(g) != n:
            raise ValueError("fees: one per pool")
        if not bool(np.all((g > 0) & (g <= 1))):
            raise ValueError("fees (gamma) must lie in (0, 1]")
    lad = None
    if ladders is not None:
        if prices is not None:
            raise ValueError("ladders= and prices= cannot be combined (a ladder carries its price)")
        if len(ladders) != n:
            raise ValueError("ladders: one (price, bounds, liquidity) per pool")
        if not bool(np.all(conc)):
            raise ValueError("ladders= applies to concentrated pools only")
        lad = []
        for k, t in enumerate(ladders):
            if t is None or len(t) != 3:
                raise ValueError(f"ladders[{k}]: concentrated needs (price, bounds, liquidity)")
            _check_ladder(t[0], t[1], t[2], f"ladders[{k}]: ")
            lad.append((float(np.asarray(t[0], np.float64).reshape(-1)[0]), np.asarray(t[1], np.float64).reshape(-1),
                        np.asarray(t[2], np.float64).reshape(-1)))
    brec = None
    if bins is not None:
        if len(bins) != n:
            raise ValueError("bins: one (prices, x, y) per pool")
        if not bool(np.all(np.asarray(kind)[ids] == KIND_BINS_HOST)):
            raise ValueError("bins= applies to bins pools only")
        brec = []
        for k, t in enumerate(bins):
            if t is None or len(t) != 3:
                raise ValueError(f"bins[{k}]: bins needs (prices, x, y)")
            checked = _check_bins(*t, where=f"bins[{k}]: ")
            try:
                brec.append(bin_records(*checked))
            except ValueError as e:
                raise ValueError(f"bins[{k}]: {e}") from None
    A = W = CG = None
    crypto = np.asarray(kind)[ids] == KIND_CRYPTOSWAP_HOST
    if curve_gamma is not None:
        if not bool(np.all(crypto)):
            raise ValueError("curve_gamma= applies to cryptoswap pools only")
        CG = np.ascontiguousarray(curve_gamma, np.float64).reshape(-1)
        if len(CG) != n:
            raise ValueError("curve_gamma: one per pool")
    if n and (amp is not None or rates is not None or curve_gamma is not None) and bool(np.all(crypto)):
        if amp is not None:
            A = np.ascontiguousarray(amp, np.float64).reshape(-1)
            if len(A) != n:
                raise ValueError("amp: one per pool")
        if rates is not None:
            W = _pool_rows(rates, n, ar, "rates")
        _check_cryptoswap(np.full(n, CRYPTO_A_RANGE[0]) if A is None else A,
                          np.full(n, CRYPTO_GAMMA_RANGE[0]) if CG is None else CG,
                          np.ones(n) if W is None else W, np.ones(n))
    elif amp is not None or rates is not None:
        if not bool(np.all(np.asarray(kind)[ids] == KIND_STABLESWAP_HOST)):
            raise ValueError("amp= and rates= apply to StableSwap or cryptoswap pools only (not both in one call)")
        if amp is not None:
            A = np.ascontiguousarray(amp, np.float64).reshape(-1)
            if len(A) != n:
                raise ValueError("amp: one per pool")
        if rates is not None:
            W = _pool_rows(rates, n, ar, "rates")
        for k in np.unique(ar).tolist():         # the rules of from_lists per coin count (ones stand in for what is kept)
            sel = np.nonzero(ar == k)[0]
            _check_stableswap(np.ones(len(sel)) if A is None else A[sel],
                              np.ones((len(sel), k)) if W is None else W[first[sel][:, None] + np.arange(k)],
                              np.ones((len(sel), k)))
    return PoolUpdate(ids, first, slots, R, g, pr, lad, A, W, CG, brec)


class BucketSpec:
    """Which pools of a HostPools form one bucket.  `sel` = global pool indices (None = all pools, in order,
    the fast path for constant-product-only problems: no host-side gathers at all)."""

    def __init__(self, hp: HostPools, kind: int, arity: int, sel: Optional[np.ndarray], lo: int = 0,
                 hi: Optional[int] = None):
        self.hp, self.kind, self.arity, self._sel = hp, kind, arity, sel
        # sel is None: the contiguous block [lo, hi) of the pool list in its own order (a rank's shard, or everything)
        self.lo, self.hi = int(lo), int(hp.m if hi is None else hi)
        self._contiguous = sel is None
        self.m = (self.hi - self.lo) if sel is None else int(len(sel))
        self._off = None

    @property
    def identity(self) -> bool:
        """pools [lo, hi) in order: the raw host arrays are uploaded as they are and reordered on the GPU"""
        return self._contiguous

    @property
    def sel(self) -> np.ndarray:
        if self._sel is None:
            self._sel = np.arange(self.lo, self.hi, dtype=np.int64)
        return self._sel

    @property
    def off(self) -> np.ndarray:
        """(arity, m) CSR offsets of every slot of every pool of the bucket"""
        if self._off is None:
            self._off = self.hp.pool_ptr[self.sel][None, :] + np.arange(self.arity)[:, None]
        return self._off

    def subset(self, local_idx: np.ndarray) -> "BucketSpec":
        return BucketSpec(self.hp, self.kind, self.arity, self.sel[local_idx])


def split_buckets(hp: HostPools, rank: int = 0, world: int = 1) -> List["BucketSpec"]:
    """Group pools by (kind, arity); with world>1 keep this rank's contiguous block of each group."""
    m = hp.m
    if m == 0:
        return []
    if getattr(hp, "_uniform_product", False):
        lo, hi = (m * rank) // world, (m * (rank + 1)) // world
        return [BucketSpec(hp, _lib.KIND_PRODUCT, 2, None, lo, hi)]
    uniform_pairs = int(hp.pool_ptr[-1]) == 2 * m and (hp.pool_ptr[1] - hp.pool_ptr[0]) == 2 and \
        bool(np.all(np.diff(hp.pool_ptr[::max(1, m // 64)]) == 2 * max(1, m // 64))) and \
        bool(np.array_equal(hp.pool_ptr[:3], np.arange(0, 2 * min(m, 2) + 1, 2)[:3]))
    if uniform_pairs:
        uniform_pairs = bool(np.all(np.diff(hp.pool_ptr) == 2))
    if uniform_pairs and not hp.kind.any() and bool(np.all(hp.weights == 0.5)):
        lo, hi = (m * rank) // world, (m * (rank + 1)) // world
        return [BucketSpec(hp, _lib.KIND_PRODUCT, 2, None, lo, hi)]
    ar = np.diff(hp.pool_ptr)
    first = hp.pool_ptr[:-1]
    is_cp = (hp.kind == KIND_GEOMEAN_HOST) & (ar == 2)
    is_cp &= (hp.weights[first] == 0.5) & (hp.weights[np.minimum(first + 1, len(hp.weights) - 1)] == 0.5)
    keys = []
    if is_cp.any():
        keys.append((_lib.KIND_PRODUCT, 2, np.nonzero(is_cp)[0]))
    cs = hp.kind == KIND_SUM_HOST
    if cs.any():
        if np.any(ar[cs] != 2):
            raise ValueError("constant-sum pools must have 2 tokens")
        keys.append((_lib.KIND_SUM, 2, np.nonzero(cs)[0]))
    bp = hp.kind == KIND_BOUNDED_HOST
    if bp.any():
        if np.any(ar[bp] != 2):
            raise ValueError("bounded_product pools must have 2 tokens")
        keys.append((_lib.KIND_BOUNDED, 2, np.nonzero(bp)[0]))
    ss = hp.kind == KIND_STABLESWAP_HOST
    if ss.any():
        if np.any((ar[ss] < 2) | (ar[ss] > STABLE_ARITY_MAX)):
            raise ValueError(f"stableswap pools must have 2..{STABLE_ARITY_MAX} tokens")
        if np.any(ss & (ar == 2)):                  # two coins: the kind-4 bucket (k_eval_stable)
            keys.append((_lib.KIND_STABLESWAP, 2, np.nonzero(ss & (ar == 2))[0]))
        for k in np.unique(ar[ss & (ar > 2)]).tolist():  # more: one kind-5 bucket per coin count (k_eval_stable_n<K>)
            keys.append((_lib.KIND_STABLESWAP_N, int(k), np.nonzero(ss & (ar == k))[0]))
    cl = hp.kind == KIND_CONCENTRATED_HOST
    if cl.any():
        if np.any(ar[cl] != 2):
            raise ValueError("concentrated pools must have 2 tokens")
        keys.append((_lib.KIND_CONCENTRATED, 2, np.nonzero(cl)[0]))
    bn = hp.kind == KIND_BINS_HOST
    if bn.any():
        if np.any(ar[bn] != 2):
            raise ValueError("bins pools must have 2 tokens")
        keys.append((_lib.KIND_BINS, 2, np.nonzero(bn)[0]))
    cs = hp.kind == KIND_CRYPTOSWAP_HOST
    if cs.any():
        if np.any((ar[cs] != 2) & (ar[cs] != 3)):
            raise ValueError("cryptoswap pools must have 2 or 3 tokens")
        if np.any(cs & (ar == 2)):                  # two coins: the kind-8 bucket (k_eval_crypto)
            keys.append((_lib.KIND_CRYPTOSWAP, 2, np.nonzero(cs & (ar == 2))[0]))
        if np.any(cs & (ar == 3)):                  # three: the kind-9 bucket (k_eval_crypto3)
            keys.append((_lib.KIND_CRYPTOSWAP_3, 3, np.nonzero(cs & (ar == 3))[0]))
    gm = (hp.kind == KIND_GEOMEAN_HOST) & ~is_cp
    for k in np.unique(ar[gm]).tolist():
        if k < 2 or k > 32:
            raise ValueError(f"weighted pools support 2..32 tokens, got {k}")
        keys.append((_lib.KIND_GEOMEAN, int(k), np.nonzero(gm & (ar == k))[0]))
    out = []
    for kind, k, sel in keys:
        if world > 1:
            lo = (len(sel) * rank) // world
            hi = (len(sel) * (rank + 1)) // world
            sel = sel[lo:hi]
        out.append(BucketSpec(hp, kind, k, sel))
    return out


TILE = 1024     # pools per TMA tile of the PLAIN buckets (csrc/cfmm_kernels.cu kTile): slot stride is padded to a multiple of it


def _padded(arr2d: np.ndarray, stride: int, fill) -> np.ndarray:
    k, m = arr2d.shape
    out = np.full((k, stride), fill, dtype=arr2d.dtype)
    out[:, :m] = arr2d
    return out


class DeviceBucket:
    def __init__(self, hp: HostPools, spec, device):
        self.kind = spec.kind; self.arity = spec.arity
        self.spec = spec
        self.m = spec.m
        self.stride = max(TILE, -(-self.m // TILE) * TILE)
        f64 = dict(dtype=torch.float64, device=device)
        self.weights = self.logrw = self.theta_bar = None
        if spec.identity and self.arity == 2 and int(hp.pool_ptr[-1]) == 2 * hp.m:   # uniform pairs in order: transpose on the GPU
            m, lo, hi = self.m, spec.lo, spec.hi
            self.reserves = torch.ones((2, self.stride), **f64)
            self.reserves[:, :m] = torch.from_numpy(hp.reserves[2 * lo:2 * hi]).to(device).view(m, 2).t()
            self.tok_idx = torch.zeros((2, self.stride), dtype=torch.int32, device=device)
            self.tok_idx[:, :m] = torch.from_numpy(hp.tok_idx[2 * lo:2 * hi]).to(device).view(m, 2).t()
            self.gamma = torch.ones(self.stride, **f64)
            self.gamma[:m] = torch.from_numpy(hp.gamma[lo:hi]).to(device)
            R = W = None
        else:
            R = hp.reserves[spec.off]
            self.reserves = torch.as_tensor(_padded(R, self.stride, 1.0), **f64)
            self.tok_idx = torch.as_tensor(_padded(hp.tok_idx[spec.off].astype(np.int32), self.stride, 0),
                                           dtype=torch.int32, device=device)
            self.gamma = torch.as_tensor(_padded(hp.gamma[spec.sel][None, :], self.stride, 1.0)[0], **f64)
        if self.kind == _lib.KIND_GEOMEAN:
            W = hp.weights[spec.off]
            self.weights = torch.as_tensor(_padded(W, self.stride, 1.0), **f64)
            self.logrw = torch.as_tensor(_padded(np.log(R / W), self.stride, 0.0), **f64)
        if self.kind == _lib.KIND_BOUNDED:                 # the virtual-reserve offsets ride in the weights slot
            self.weights = torch.as_tensor(_padded(hp.weights[spec.off], self.stride, 1.0), **f64)
        if self.kind in (_lib.KIND_STABLESWAP, _lib.KIND_STABLESWAP_N):   # rates in the weights slot, (A, D) in two logrw rows
            self.weights = torch.as_tensor(_padded(hp.weights[spec.off], self.stride, 1.0), **f64)
            AD = np.stack([hp.amp[spec.sel], hp.inv[spec.sel]])
            self.logrw = torch.as_tensor(_padded(AD, self.stride, 1.0), **f64)
        if self.kind in (_lib.KIND_CRYPTOSWAP, _lib.KIND_CRYPTOSWAP_3):   # price scales in weights, (A, G, D) in logrw
            self.weights = torch.as_tensor(_padded(hp.weights[spec.off], self.stride, 1.0), **f64)
            AGD = np.stack([hp.amp[spec.sel], np.asarray(hp.cgam, np.float64)[spec.sel], hp.inv[spec.sel]])
            self.logrw = torch.as_tensor(_padded(AGD, self.stride, 1.0), **f64)
        if self.kind == _lib.KIND_CONCENTRATED:            # this bucket's records in the weights slot, (s, c, first, T) in logrw
            sel = spec.sel
            first = np.asarray(hp.lad_ptr, np.int64)[sel]
            cnt = np.asarray(hp.lad_ptr, np.int64)[sel + 1] - first
            loc = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
            gather = np.repeat(first - loc, cnt) + np.arange(int(cnt.sum()), dtype=np.int64)
            self.weights = torch.as_tensor(np.ascontiguousarray(np.asarray(hp.lad_rec, np.float64)[gather]).reshape(-1), **f64)
            self.n_rec = int(cnt.sum())
            self._rec_buf, self._rec_spare = self.weights, None      # splice_records writes the spare and swaps
            sc = np.asarray(hp.lad_sc, np.float64)[sel]
            P = np.stack([sc[:, 0], sc[:, 1], loc.astype(np.float64), (cnt - 1).astype(np.float64)])
            self.logrw = torch.as_tensor(_padded(P, self.stride, 0.0), **f64)
        if self.kind == _lib.KIND_BINS:                    # records in the weights slot, (first, nb, z, p_ref) in logrw
            sel = spec.sel
            first = np.asarray(hp.bin_ptr, np.int64)[sel]
            cnt = np.asarray(hp.bin_ptr, np.int64)[sel + 1] - first
            loc = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
            gather = np.repeat(first - loc, cnt) + np.arange(int(cnt.sum()), dtype=np.int64)
            self.weights = torch.as_tensor(np.ascontiguousarray(np.asarray(hp.bin_rec, np.float64)[gather]).reshape(-1), **f64)
            self.n_rec = int(cnt.sum())
            self._rec_buf, self._rec_spare = self.weights, None      # as for concentrated buckets
            zp = np.asarray(hp.bin_zp, np.float64)[sel]
            P = np.stack([loc.astype(np.float64), cnt.astype(np.float64), zp[:, 0], zp[:, 1]])
            self.logrw = torch.as_tensor(_padded(P, self.stride, 0.0), **f64)
        if self.kind in (_lib.KIND_SUM, _lib.KIND_BINS):
            self.theta_bar = torch.zeros((2, self.stride), **f64)
        self.delta = self.lam = self.hcoef = self.hmask = None
        self._device = device
        self.c_bucket = _lib.Bucket(
            self.kind, self.arity, self.m, self.stride, self.reserves.data_ptr(), self.tok_idx.data_ptr(),
            self.gamma.data_ptr(),
            self.weights.data_ptr() if self.weights is not None else None,
            self.logrw.data_ptr() if self.logrw is not None else None,
            self.theta_bar.data_ptr() if self.theta_bar is not None else None)

    @property
    def sel(self) -> np.ndarray:
        return self.spec.sel

    @property
    def off(self) -> np.ndarray:
        return self.spec.off

    def write_update(self, loc: np.ndarray, R: Optional[np.ndarray], gamma: Optional[np.ndarray],
                     W: Optional[np.ndarray] = None, amp: Optional[np.ndarray] = None, sc: Optional[np.ndarray] = None,
                     rates: Optional[np.ndarray] = None, AD: Optional[np.ndarray] = None,
                     cgam: Optional[np.ndarray] = None):
        """New reserves R (arity, n) and / or fees (n,) of the bucket-local pools `loc` (values already checked).
        Weighted pools also get logrw = log(R / W) with their weights W (arity, n), the expression of __init__;
        StableSwap pools get the invariant D of the new reserves from their rates W and amplification amp (n,), or, when
        their A or rates change, the new rates (arity, n) in the weights rows and AD = (A, D) (2, n) in logrw rows 0-1;
        cryptoswap pools likewise, with their curve gammas cgam (n,), and AD = (A, G, D) (3, n) in logrw rows 0-2;
        concentrated pools get their new (s, c) from sc (2, n), with R their derived reserves (ladder_state)."""
        f64 = dict(dtype=torch.float64, device=self._device)
        li = torch.as_tensor(loc, dtype=torch.int64, device=self._device)
        if sc is not None:
            self.logrw[:2, li] = torch.as_tensor(sc, **f64)
        if R is not None:
            self.reserves[:, li] = torch.as_tensor(R, **f64)
            if self.kind in (_lib.KIND_STABLESWAP, _lib.KIND_STABLESWAP_N):
                if AD is None:
                    self.logrw[1, li] = torch.as_tensor(stableswap_invariant_any(R.T, W.T, amp), **f64)
            elif self.kind in (_lib.KIND_CRYPTOSWAP, _lib.KIND_CRYPTOSWAP_3):
                if AD is None:
                    self.logrw[2, li] = torch.as_tensor(cryptoswap_invariant_any(R.T, W.T, amp, cgam), **f64)
            elif self.kind == _lib.KIND_GEOMEAN:
                self.logrw[:, li] = torch.as_tensor(np.log(R / W), **f64)
        if rates is not None:
            self.weights[:, li] = torch.as_tensor(rates, **f64)
        if AD is not None:
            self.logrw[:len(AD), li] = torch.as_tensor(AD, **f64)
        if gamma is not None:
            self.gamma[li] = torch.as_tensor(gamma, **f64)

    def splice_records(self, lib, loc: np.ndarray, rec: np.ndarray, cnt: np.ndarray, state: np.ndarray, n_total: int,
                       stream):
        """New records of the pools at the bucket-local positions `loc` (ascending): rec (sum(cnt), 4), pool after pool.
        Concentrated buckets (cfmm_ladder_splice): cnt[k] = T + 1 of pool loc[k], state (n, 4) = (s, c, x, y).  Price-bin
        buckets (cfmm_bins_splice): cnt[k] = nb, state = (z, p_ref, sum x, sum y), and the changed pools' theta_bar is
        zeroed (a fresh pool's multiplier).  The entry point writes every pool's records into the spare buffer in bucket
        order (n_total of them), then the two buffers swap, so c_bucket.weights moves (a CUDA graph captured over this
        bucket must be captured again).  Synchronous."""
        name = "cfmm_bins_splice" if self.kind == _lib.KIND_BINS else "cfmm_ladder_splice"
        dev = self._device
        if self._rec_spare is None or self._rec_spare.numel() < 4 * n_total:
            self._rec_spare = None
            self._rec_spare = torch.empty(4 * (n_total + n_total // 8), dtype=torch.float64, device=dev)
        f64 = dict(dtype=torch.float64, device=dev)
        pos = torch.as_tensor(np.asarray(loc, np.int64), device=dev)
        nrec = torch.as_tensor(np.asarray(cnt, np.int64), device=dev)
        recd = torch.as_tensor(np.ascontiguousarray(rec, np.float64), **f64)
        std = torch.as_tensor(np.ascontiguousarray(state, np.float64), **f64)
        nb = int(lib.cfmm_ladder_splice_work_bytes(self.m, len(loc)))
        if nb < 0:
            _lib.check(nb, "cfmm_ladder_splice_work_bytes")
        work = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
        status = (C.c_int64 * 2)()
        _lib.check(getattr(lib, name)(C.byref(self.c_bucket), len(loc), pos.data_ptr(), nrec.data_ptr(),
                                      recd.data_ptr(), len(rec), std.data_ptr(), self._rec_spare.data_ptr(),
                                      self._rec_spare.numel() // 4, status, work.data_ptr(), nb, stream), name)
        if status[0] != 0 or status[1] != n_total:
            raise _lib.CfmmError(f"{name} rejected the update ({status[0]} invalid entries, {status[1]} records "
                                 f"for {n_total} expected)")
        if self.theta_bar is not None and len(loc):
            self.theta_bar[:, pos] = 0.0
        self._rec_buf, self._rec_spare = self._rec_spare, self._rec_buf
        self.weights = self._rec_buf[:4 * n_total]
        self.n_rec = n_total
        self.c_bucket.weights = self.weights.data_ptr()

    def bytes_resident(self) -> int:
        n = 0
        for t in (self.reserves, self.tok_idx, self.gamma, self.weights, self.logrw, self.theta_bar):
            if t is not None:
                n += t.numel() * t.element_size()
        return n

    def out_struct(self, trades: bool, hess: bool):
        f64 = dict(dtype=torch.float64, device=self._device)
        if trades and self.delta is None:
            self.delta = torch.zeros((self.arity, self.stride), **f64)
            self.lam = torch.zeros((self.arity, self.stride), **f64)
        if hess and self.hcoef is None:
            # n-coin StableSwap: one coefficient h_j per slot ([arity][stride]); every other kind: one per pool
            self.hcoef = torch.zeros((self.arity, self.stride)
                                     if self.kind in (_lib.KIND_STABLESWAP_N, _lib.KIND_CRYPTOSWAP_3) else self.stride,
                                     **f64)
            self.hmask = torch.zeros(self.stride, dtype=torch.int32, device=self._device)
        return _lib.EvalOut(self.delta.data_ptr() if trades else None, self.lam.data_ptr() if trades else None,
                            self.hcoef.data_ptr() if hess else None, self.hmask.data_ptr() if hess else None)


def blocked_layout_info(lib):
    v = [C.c_int32() for _ in range(4)]
    _lib.check(lib.cfmm_blocked_layout_info(*[C.byref(x) for x in v]), "cfmm_blocked_layout_info")
    return tuple(int(x.value) for x in v)      # pools_per_tile, rows_stride, tok_stride, row_cap


def blocked_fee_words(lib) -> int:
    """32-bit words per tile of the fee record (include/cfmm_b200.h)"""
    return int(lib.cfmm_blocked_fee_words())


_FEE_MAX, _FEE_TAB, _FEE_CODE = 16, 4, 36          # distinct values of a coded tile; words of the table and of the codes


def fee_records(gamma_inv: torch.Tensor, P: int) -> torch.Tensor:
    """Fee records (include/cfmm_b200.h) of a blocked layout from its 1/gamma slab (n_tiles * P f64, padding included):
    per tile the header (nfee, 0, 0, 0), its distinct bit patterns in ascending order and a 4-bit index per pool into
    them.  A tile with more than 16 distinct values gets an all-zero record: it streams its slab.
    Returns (n_tiles, 36 + P // 8) int32."""
    dev = gamma_inv.device
    i64 = dict(dtype=torch.int64, device=dev)
    bits = gamma_inv.contiguous().view(torch.int64).view(-1, P)          # positive doubles order like their bit patterns
    T = bits.shape[0]
    s, _ = torch.sort(bits, dim=1)
    new = torch.ones_like(s, dtype=torch.bool)
    new[:, 1:] = s[:, 1:] != s[:, :-1]
    rank = torch.cumsum(new.to(torch.int64), 1) - 1                     # index of every sorted entry among the distinct
    nfee = rank[:, -1] + 1
    coded = (nfee <= _FEE_MAX)[:, None]
    table = torch.zeros((T, _FEE_MAX + 1), **i64)
    table.scatter_(1, rank.clamp(max=_FEE_MAX), s)                      # column 16 only collects tiles that are not coded
    table = torch.where(coded, table[:, :_FEE_MAX], 0)
    code = torch.where(coded, rank.gather(1, torch.searchsorted(s, bits)), 0)
    words = (code.view(T, P // 8, 8) << (4 * torch.arange(8, **i64))).sum(2)
    head = torch.zeros((T, _FEE_TAB), **i64)
    head[:, 0] = torch.where(coded[:, 0], nfee, 0)
    rec = torch.cat([head, table.view(torch.int32).to(torch.int64), words], 1)      # table: low word of each f64 first
    assert rec.shape[1] == _FEE_CODE + P // 8
    return torch.where(rec >= 2 ** 31, rec - 2 ** 32, rec).to(torch.int32).contiguous()


def unpack_pool_words(pw: torch.Tensor, P: int):
    """Pool words of a blocked layout (``lid0 | lid1 << 10 | p1 << 20``, see csrc/cfmm_blocked.cuh) in the two-word form,
    int32 each: local ids ``lid0 | lid1 << 16`` and flow-array positions ``pos0 | pos1 << 16``, where pos0 = l (the pool's
    index in its tile) and pos1 = P + p1."""
    w = pw.to(torch.int64) & 0xffffffff
    l = torch.arange(w.numel(), device=w.device) % P
    lid = (w & 0x3ff) | (((w >> 10) & 0x3ff) << 16)
    pos = l | ((P + (w >> 20)) << 16)
    return lid.to(torch.int32), pos.to(torch.int32)


class BlockedTables(Mapping):
    """The tables of a blocked layout, read-only and dict-like.  Stores the pool words ``pw``; ``lid`` and ``pos`` (the
    two-word form of unpack_pool_words) are computed on access."""
    _DERIVED = ("lid", "pos")

    def __init__(self, P: int, **tables):
        self._P = P
        self._t = tables

    def __getitem__(self, k):
        if k in self._DERIVED:
            return unpack_pool_words(self._t["pw"], self._P)[self._DERIVED.index(k)]
        return self._t[k]

    def __iter__(self):
        return iter(list(self._t) + list(self._DERIVED))

    def __len__(self):
        return len(self._t) + len(self._DERIVED)


def _tile_layout(a: torch.Tensor, b: torch.Tensor, n_tokens: int, P: int, row_cap: int) -> dict:
    """Tables of the pools with tokens (a, b), in blocked order, cut into tiles of P (csrc/cfmm_blocked.cuh): local ids
    numbered in token order, slot-1 positions, token lists, rows; and (ntok, nrow) per tile, to be checked against the
    table strides before anything is written at those strides."""
    dev = a.device
    i64 = dict(dtype=torch.int64, device=dev)
    mm = a.numel()
    ntiles = -(-mm // P)
    q = torch.arange(mm, **i64)
    tile = q // P
    # distinct tokens of every tile -> local ids and token list
    ck, perm = torch.sort(torch.cat([tile, tile]) * n_tokens + torch.cat([a, b]), stable=True)
    uniq, inv = torch.unique_consecutive(ck, return_inverse=True)
    u_tile = uniq // n_tokens
    ntok = torch.bincount(u_tile, minlength=ntiles)
    ltok_u = torch.arange(uniq.numel(), **i64) - (torch.cumsum(ntok, 0) - ntok)[u_tile]
    he_ltok = torch.empty(2 * mm, **i64)
    he_ltok[perm] = ltok_u[inv]
    lid0, lid1 = he_ltok[:mm], he_ltok[mm:]
    # slot 1: rank among the tile's slot-1 half-edges stably sorted by token (every tile but the last holds P pools)
    s1 = torch.argsort(tile * n_tokens + b, stable=True)
    p1 = torch.empty(mm, **i64)
    p1[s1] = q - tile[s1] * P
    # the flow array of every tile: slot 0 at g[l], slot 1 at g[P + p1]; F = local token of each flow, -1 where none
    F = torch.full((ntiles, 2 * P), -1, **i64)
    F[tile, q - tile * P] = lid0
    F[tile, P + p1] = lid1
    F = F.view(-1)
    c = torch.arange(F.numel(), **i64)
    real = F >= 0
    # runs of equal tokens inside each half, cut into rows of <= row_cap flows
    head = real & ((c % P == 0) | (F != torch.roll(F, 1)))
    start = torch.cummax(torch.where(head, c, -1), 0).values
    run = torch.cumsum(head.to(torch.int64), 0) - 1
    run_len = torch.bincount(run[real])
    o = c - start
    rh = real & (o % row_cap == 0)
    rc = c[rh]
    row_len = torch.clamp(run_len[run[rh]] - o[rh], max=row_cap)
    row_tile, row_start = rc // (2 * P), rc % (2 * P)
    # longest rows first inside each tile (the 32 rows a warp sums have nearly equal trip counts), ties in flow order
    srt = torch.argsort((row_tile * 64 + (63 - row_len)) * (2 * P) + row_start)
    row_tile, row_start, row_len, row_ltok = row_tile[srt], row_start[srt], row_len[srt], F[rc][srt]
    nrow = torch.bincount(row_tile, minlength=ntiles)
    return dict(ntiles=ntiles, ntok=ntok, nrow=nrow, uniq=uniq, u_tile=u_tile, ltok_u=ltok_u, lid0=lid0, lid1=lid1, p1=p1,
                row_tile=row_tile, row_start=row_start, row_len=row_len, row_ltok=row_ltok)


def build_blocked_pairs(idx: torch.Tensor, n_tokens: int, P: int, rows_stride: int, tok_stride: int, row_cap: int):
    """Layout builder for cfmm_blocked_pairs (see csrc/cfmm_blocked.cuh).  idx: (2, m) int64 token ids on the
    device.  Pools are sorted by (token block of slot 0, token block of slot 1, slot-0 token) and cut into tiles of P;
    each tile gets its distinct-token list, one pool word per pool (10-bit local ids, slot-1 flow position), and a table
    of rows (token, <= row_cap consecutive flows).
    Returns (order, residual, tables): `order` = bucket-local pool index at each blocked position, `residual` =
    pools left out because their tile would touch more than tok_stride tokens or need more than rows_stride rows (they
    go to a plain bucket), `tables` = BlockedTables."""
    dev = idx.device
    m = idx.shape[1]
    i64 = dict(dtype=torch.int64, device=dev)
    nb = max(1, int(round((m / P) ** 0.5)))
    a, b = idx[0], idx[1]
    # primary: (token block of slot 0, token block of slot 1); secondary: slot-0 token, so that the lanes of a warp
    # read the same nu_local entry (shared-memory broadcast) and a token's slot-0 flows are neighbours in the flow array
    key = ((a * nb // n_tokens) * nb + (b * nb // n_tokens)) * n_tokens + a
    order = torch.argsort(key, stable=True)
    residual = []
    for _pass in range(4):
        mm = order.numel()
        if mm == 0:
            break
        L = _tile_layout(a[order], b[order], n_tokens, P, row_cap)
        bad = (L["ntok"] > tok_stride) | (L["nrow"] > rows_stride)
        if not bool(bad.any()):
            break
        if _pass == 3:                       # give up blocking: everything left goes to the plain bucket
            residual.append(order); order = order[:0]; mm = 0
            break
        keep = ~bad[torch.arange(mm, **i64) // P]
        residual.append(order[~keep])
        order = order[keep]
    residual = torch.cat(residual) if residual else order[:0]
    if order.numel() == 0:
        return order, residual, None
    ntiles, ntok, nrow = L["ntiles"], L["ntok"], L["nrow"]
    M = ntiles * P
    # pool words; padding pool l of the last tile writes its zero flows to g[l] and g[P + l], past the real ones
    pw = (torch.arange(M, **i64) % P) << 20
    pw[:mm] = L["lid0"] | (L["lid1"] << 10) | (L["p1"] << 20)
    tok = torch.zeros((ntiles, tok_stride), dtype=torch.int32, device=dev)
    tok[L["u_tile"], L["ltok_u"]] = (L["uniq"] - L["u_tile"] * n_tokens).to(torch.int32)
    row_tile = L["row_tile"]
    n_rows = row_tile.numel()
    r_local = torch.arange(n_rows, **i64) - (torch.cumsum(nrow, 0) - nrow)[row_tile]
    rows = torch.zeros((ntiles, rows_stride), dtype=torch.int32, device=dev)
    word = L["row_start"] | (L["row_len"] << 16) | (L["row_ltok"] << 22)          # start:16 | len:6 | ltok:10 (may set bit 31)
    rows[row_tile, r_local] = torch.where(word >= 2 ** 31, word - 2 ** 32, word).to(torch.int32)
    desc = torch.stack([ntok, nrow, torch.zeros_like(ntok), torch.zeros_like(ntok)], 1).to(torch.int32).contiguous()
    tables = BlockedTables(P, n_tiles=ntiles, M=M, pw=pw.to(torch.int32), tok=tok, rows=rows, desc=desc,
                           rows_per_pool=n_rows / mm, tok_per_tile=float(ntok.double().mean()))
    return order, residual, tables


class BlockedBucket:
    """Constant-product pools in the token-blocked layout (HBM-bound kind; no per-pool atomics)."""
    kind = _lib.KIND_PRODUCT
    arity = 2
    blocked = True

    def __init__(self, hp: HostPools, spec, device, lib):
        self.spec = spec
        P, rows_stride, tok_stride, row_cap = blocked_layout_info(lib)
        f64 = dict(dtype=torch.float64, device=device)
        self.theta_bar = None
        self.delta = self.lam = self.hcoef = self.hmask = None
        self._device = device
        self._sel = self._off = None
        if spec.identity and int(hp.pool_ptr[-1]) == 2 * hp.m and self._build_native(hp, spec, device, lib, P, rows_stride, tok_stride):
            return                              # the whole layout was built by three launches of csrc/cfmm_layout.cu
        if spec.identity:                       # raw arrays go up as they are; all reordering happens on the GPU
            lo, hi = spec.lo, spec.hi            # a rank's shard uploads only its own slice of the (pinned) host arrays
            R = torch.from_numpy(hp.reserves[2 * lo:2 * hi]).to(device, non_blocking=True).view(-1, 2)
            idx = torch.from_numpy(hp.tok_idx[2 * lo:2 * hi]).to(device, non_blocking=True).view(-1, 2).to(torch.int64)
            gam = torch.from_numpy(hp.gamma[lo:hi]).to(device, non_blocking=True)
            if getattr(hp, "_validate_on_device", False):          # same checks as HostPools.validate(), on the GPU
                chk = torch.stack([R.min(), gam.min(), 1.0 - gam.max(), idx.min().double(),
                                   float(hp.n_tokens - 1) - idx.max().double(),
                                   torch.isfinite(R).all().double() - 0.5]).cpu()
                if bool((chk[:2] <= 0).any()) or bool((chk[2:] < 0).any()):
                    raise ValueError("invalid pool data (reserves > 0, fees in (0, 1], token ids in range, finite)")
        else:
            R = torch.as_tensor(np.ascontiguousarray(hp.reserves[spec.off].T), **f64)
            idx = torch.as_tensor(np.ascontiguousarray(hp.tok_idx[spec.off].T).astype(np.int64), device=device)
            gam = torch.as_tensor(np.ascontiguousarray(hp.gamma[spec.sel]), **f64)
        order, residual, t = build_blocked_pairs(idx.t(), hp.n_tokens, P, rows_stride, tok_stride, row_cap)
        self.order = order                               # blocked position -> bucket-local pool index (device)
        self.residual = residual.cpu().numpy() if residual.numel() else np.zeros(0, np.int64)
        self.m = int(order.numel())
        if self.m == 0:
            self.tables = None
            return
        self.stride = t["M"]

        def slab(vals, fill):
            out = torch.full((t["M"],), fill, **f64)
            out[:self.m] = vals
            return out
        self.r0 = slab(R[order, 0], 1.0)
        self.r1 = slab(R[order, 1], 1.0)
        self.gamma_inv = slab(1.0 / gam[order], 1.0)
        fee = fee_records(self.gamma_inv, P)
        if fee.shape[1] != blocked_fee_words(lib):
            raise _lib.CfmmError("fee record layout differs from the library's")
        self.tables = t = BlockedTables(P, **t._t, fee=fee)
        self.c_blocked = _lib.BlockedPairs(self.m, t["n_tiles"], P, 0, self.r0.data_ptr(), self.r1.data_ptr(),
                                           self.gamma_inv.data_ptr(), t["pw"].data_ptr(), fee.data_ptr(),
                                           t["rows"].data_ptr(), t["tok"].data_ptr(), t["desc"].data_ptr())

    def _build_native(self, hp, spec, device, lib, P, rows_stride, tok_stride) -> bool:
        """cfmm_blocked_build (csrc/cfmm_layout.cu): upload the pools' own arrays (this rank's slice) and build the blocked
        layout on the device in three launches.  False = not applicable (keys would not fit 32 bits, or some tile would
        touch more tokens than a tile may): the caller takes the general torch builder."""
        lo, hi = spec.lo, spec.hi
        m = hi - lo
        if m <= 0:
            return False
        nb = max(1, int(round((m / P) ** 0.5)))
        if nb * nb * hp.n_tokens >= 2 ** 32 or m >= 2 ** 31:
            return False
        T = -(-m // P)
        M = T * P
        f64 = dict(dtype=torch.float64, device=device)
        i32 = dict(dtype=torch.int32, device=device)
        idx = torch.from_numpy(np.ascontiguousarray(hp.tok_idx[2 * lo:2 * hi], np.int32)).to(device, non_blocking=True)
        R = torch.from_numpy(hp.reserves[2 * lo:2 * hi]).to(device, non_blocking=True)
        gam = torch.from_numpy(hp.gamma[lo:hi]).to(device, non_blocking=True)
        slabs = torch.empty((3, M), **f64)
        pw = torch.empty(M, **i32)
        rows = torch.empty((T, rows_stride), **i32)
        # the fee records share one allocation with the token lists: as a tensor of its own (~0.6 MB at 1M pools) they
        # land in the caching allocator's small-block pool and shift the store's small vectors (psi, Hessian product),
        # which made L2-hot Hessian products 23% slower on an H100
        tok_fee = torch.empty(T * (tok_stride + blocked_fee_words(lib)), **i32)
        tok, fee = tok_fee[:T * tok_stride].view(T, tok_stride), tok_fee[T * tok_stride:].view(T, -1)
        desc = torch.empty((T, 4), **i32)
        order = torch.empty(m, **i32)
        status = torch.empty(4, **i32)
        nbytes = int(lib.cfmm_blocked_build_work_bytes(m))
        if nbytes <= 0:
            return False
        work = torch.empty(nbytes, dtype=torch.uint8, device=device)
        cb = _lib.BlockedPairs(m, T, P, 0, slabs[0].data_ptr(), slabs[1].data_ptr(), slabs[2].data_ptr(), pw.data_ptr(),
                               fee.data_ptr(), rows.data_ptr(), tok.data_ptr(), desc.data_ptr())
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        rc = lib.cfmm_blocked_build(m, hp.n_tokens, idx.data_ptr(), R.data_ptr(), gam.data_ptr(), C.byref(cb), order.data_ptr(),
                                    status.data_ptr(), work.data_ptr(), nbytes, st)
        if rc == -3:                              # CFMM_E_SIZE: outside the native builder's key range
            return False
        _lib.check(rc, "cfmm_blocked_build")
        st_h = status.cpu()                       # the one synchronisation of the build
        if int(st_h[1]) != 0:
            raise ValueError("invalid pool data (reserves > 0 and finite, fees in (0, 1], two distinct token ids in range)")
        if int(st_h[0]) != 0:                     # a tile touches more tokens / needs more rows than it may: general builder
                                                  # + plain residual bucket
            return False
        self.order = order
        self.residual = np.zeros(0, np.int64)
        self.m = m
        self.stride = M
        self.r0, self.r1, self.gamma_inv = slabs[0], slabs[1], slabs[2]
        self._keep = (idx, R, gam, work)          # the build is asynchronous: its inputs live as long as the bucket
        self.tables = BlockedTables(P, n_tiles=T, M=M, pw=pw, tok=tok, rows=rows, desc=desc, fee=fee,
                                    rows_per_pool=int(st_h[2]) / m, tok_per_tile=None)
        self.c_blocked = cb
        return True

    # host-side index maps are only needed for read-back / dense assembly: built on first use
    @property
    def sel(self) -> np.ndarray:
        if self._sel is None:
            self._sel = self.spec.sel[self.order.cpu().numpy().astype(np.int64)]
        return self._sel

    @property
    def off(self) -> np.ndarray:
        if self._off is None:
            self._off = self.spec.hp.pool_ptr[self.sel][None, :] + np.arange(2)[:, None]
        return self._off

    def write_update(self, lib, pos: np.ndarray, R: Optional[np.ndarray], gamma: Optional[np.ndarray], stream) -> int:
        """cfmm_blocked_update: new reserves R (2, n) and / or fees (n,) of the pools at blocked positions `pos`.  Checks
        every entry on the device and writes nothing if one is invalid (ValueError).  Synchronous.  Returns the number
        of fee records rebuilt."""
        dev = self._device
        at = torch.as_tensor(np.asarray(pos, np.uint32).view(np.int32), device=dev)
        Rd = None if R is None else torch.as_tensor(np.ascontiguousarray(R.T), dtype=torch.float64, device=dev)
        gd = None if gamma is None else torch.as_tensor(gamma, dtype=torch.float64, device=dev)
        if getattr(self, "_upd_work", None) is None:
            nbytes = int(lib.cfmm_blocked_update_work_bytes(C.byref(self.c_blocked)))
            if nbytes < 0:
                _lib.check(nbytes, "cfmm_blocked_update_work_bytes")
            self._upd_work = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        status = (C.c_int32 * 2)()
        _lib.check(lib.cfmm_blocked_update(C.byref(self.c_blocked), len(pos), at.data_ptr(),
                                           Rd.data_ptr() if Rd is not None else None,
                                           gd.data_ptr() if gd is not None else None, status,
                                           self._upd_work.data_ptr(), self._upd_work.numel(), stream),
                   "cfmm_blocked_update")
        if status[0] != 0:
            raise ValueError(f"{status[0]} invalid pool update(s) (reserves > 0 and finite, fees in (0, 1]); "
                             "nothing was written")
        return int(status[1])

    def bytes_resident(self) -> int:
        if self.tables is None:
            return 0
        ts = [self.r0, self.r1, self.gamma_inv] + [self.tables[k] for k in ("pw", "tok", "rows", "desc", "fee")]
        return sum(x.numel() * x.element_size() for x in ts)

    def out_struct(self, trades: bool, hess: bool):
        f64 = dict(dtype=torch.float64, device=self._device)
        if trades and self.delta is None:
            self.delta = torch.zeros((2, self.stride), **f64)
            self.lam = torch.zeros((2, self.stride), **f64)
        if hess and self.hcoef is None:
            self.hcoef = torch.zeros(self.stride, **f64)
        return _lib.EvalOut(self.delta.data_ptr() if trades else None, self.lam.data_ptr() if trades else None,
                            self.hcoef.data_ptr() if hess else None, None)


class PeerContext:
    """Symmetric-memory buffers + sequence counters of the NVLink all-reduce kernel (csrc/cfmm_allreduce.cu), one per
    (process, token count): allocation and rendezvous cost milliseconds, so they are paid once, not per
    PoolStore / per solve.  All ranks must issue the same sequence of reductions (they do: every rank runs the same
    outer loop on bit-identical reduced vectors)."""

    def __init__(self, n_tokens: int, device, group):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        n = int(n_tokens)
        if n + 1 > 64 * 256:
            raise _lib.CfmmError("peer all-reduce supports n_tokens < 16384; use NCCL (Comm) beyond that")
        f64 = dict(dtype=torch.float64, device=device)
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.n_tokens = n
        w = self.world
        # receive areas: [3 slots][world sources][n cells of {value, sequence flag}] (zero = "nothing received yet")
        self.sym_acc = symm.empty((3 * w * (n + 1) * 2,), **f64); self.sym_acc.zero_()
        self.sym_y = symm.empty((3 * w * (n + 2) * 2,), **f64); self.sym_y.zero_()      # n-vectors (+2: the persistent solver appends p'Hp, p'Dp)
        self.hdl_acc = symm.rendezvous(self.sym_acc, group)
        self.hdl_y = symm.rendezvous(self.sym_y, group)
        self.red_acc = torch.zeros(n + 1, **f64)
        self.red_y = torch.zeros(n, **f64)
        self.seq = [0, 0]                   # last sequence number used on channel 0 ([psi | arb]) / 1 (n-vectors)
        torch.cuda.synchronize(device)
        dist.barrier(group)

    def next_seq(self, chan: int) -> int:
        self.seq[chan] += 1
        return self.seq[chan]

    def c_struct(self):
        """cfmm_peer_ctx for the native solvers (they advance the sequence numbers; read them back with absorb())"""
        return _lib.PeerCtx(int(self.hdl_acc.buffer_ptrs_dev), int(self.hdl_y.buffer_ptrs_dev), self.rank, self.world,
                            self.seq[0], self.seq[1])

    def absorb(self, c):
        self.seq = [int(c.seq_acc), int(c.seq_vec)]


_PEER_CONTEXTS: Dict[tuple, "PeerContext"] = {}


def peer_context(n_tokens: int, device, group=None) -> "PeerContext":
    """the process-wide PeerContext for this token count (created on first use; collective)"""
    import torch.distributed as dist
    group = group or dist.group.WORLD
    key = (int(n_tokens), id(group), str(torch.device(device)))
    if key not in _PEER_CONTEXTS:
        _PEER_CONTEXTS[key] = PeerContext(n_tokens, torch.device(device), group)
    return _PEER_CONTEXTS[key]


class PoolStore:
    """All pools of one problem (or one rank's shard of them), resident on one GPU."""

    def __init__(self, hp: HostPools, device="cuda", rank: int = 0, world: int = 1, validate: bool = True,
                 layout: str = "blocked"):
        if layout not in ("blocked", "plain"):
            raise ValueError("layout must be 'blocked' or 'plain'")
        if validate:
            if getattr(hp, "_uniform_product", False) and layout == "blocked":
                hp._validate_on_device = True           # checked after the upload, by reductions on the GPU
            else:
                hp.validate()
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.CfmmError("PoolStore needs a CUDA device: there is no CPU path in this package")
        if not torch.cuda.is_available():
            raise _lib.CfmmError("no CUDA device visible: the routing kernels have no CPU fallback")
        self.n_tokens = int(hp.n_tokens)
        self.m_total = hp.m
        self.pool_ptr = hp.pool_ptr
        self._tok_idx_host = hp.tok_idx
        # borrowed from hp and never written: update_pools(amp=, rates=) copies weights and amp first, and ladders live in
        # a LadderSlab over hp's records (made at the first update that needs them)
        self._kind_host, self._weights_host = hp.kind, hp.weights      # structure: kinds, weights / bounded offsets / rates
        self._amp_host = hp.amp                                          # StableSwap / cryptoswap amplification
        self._cgam_host = hp.cgam                                        # cryptoswap curve gamma
        self._own_stable = False                                         # weights / amp are this store's copies
        self._lad_host = (hp.lad_ptr, hp.lad_rec)                        # concentrated records
        self._lad = None                                                 # LadderSlab
        self._bins_host = (hp.bin_ptr, hp.bin_rec)                       # price-bin records
        self._bin = None                                                 # LadderSlab of the price-bin records
        self._where = None                                               # pool -> (bucket, position): update_pools
        self.rank, self.world = rank, world
        self.buckets = []
        for s in split_buckets(hp, rank, world):
            if s.kind == _lib.KIND_PRODUCT and layout == "blocked" and s.m > 0:
                bb = BlockedBucket(hp, s, self.device, self.lib)
                if bb.m > 0:
                    self.buckets.append(bb)
                if len(bb.residual):
                    self.buckets.append(DeviceBucket(hp, s.subset(bb.residual), self.device))
            else:
                self.buckets.append(DeviceBucket(hp, s, self.device))
        # the blocked bucket (at most one per store) goes first: its launch clears the ping-pong partner buffer
        self.buckets.sort(key=lambda b: 0 if getattr(b, "blocked", False) else 1)
        self._blocked_first = bool(self.buckets) and getattr(self.buckets[0], "blocked", False)
        assert sum(1 for b in self.buckets if getattr(b, "blocked", False)) <= 1
        self.m_local = sum(b.m for b in self.buckets)
        self.has_sum = bool(np.any((hp.kind == KIND_SUM_HOST) | (hp.kind == KIND_BINS_HOST)))
        self.has_geomean = any(b.kind == _lib.KIND_GEOMEAN for b in self.buckets)
        f64 = dict(dtype=torch.float64, device=self.device)
        # [psi | arb] (the one all-reduced buffer) and y are ping-ponged: a blocked launch clears the buffer of the
        # NEXT call, so steady-state evaluations need no memset node
        self._acc2 = torch.zeros((2, self.n_tokens + 1), **f64)
        self._y2 = torch.zeros((2, self.n_tokens), **f64)
        self._acc_i = 0
        self._y_i = 0
        self._move = torch.zeros(1, **f64)
        self.evals = 0
        self.hvps = 0

    # -- multi-GPU: peer-memory all-reduce -----------------------------------------------------------
    def enable_peer_allreduce(self, group=None):
        """Pool-sharded stores (world > 1): finish every evaluate()/hvp()/hess_diag() with the NVLink all-reduce kernel
        cfmm_allreduce_ll (PDL-chained behind the pool kernels: every rank pushes {value, seq} cells into the peers'
        receive areas, one NVLink one-way trip) instead of returning a partial for NCCL.  The buffers live in torch
        symmetric memory and are created ONCE per process and token count (peer_context()); every store of the
        process shares them.  Collective: every rank must call it, in the same order."""
        self._peer = peer_context(self.n_tokens, self.device, group)
        self.reduces_internally = True

    def _peer_reduce(self, chan, local, n, st):
        """all-reduce `local` (n doubles, this rank's partial) over the peer context; chan 0 = [psi | arb], 1 = n-vectors"""
        p = self._peer
        seq = p.next_seq(chan)
        hdl, out = (p.hdl_acc, p.red_acc) if chan == 0 else (p.hdl_y, p.red_y)
        _lib.check(self.lib.cfmm_allreduce_ll(local.data_ptr(), int(hdl.buffer_ptrs_dev), p.rank, p.world, n,
                                              (seq % 3) * p.world * n, n, out.data_ptr(), seq, st), "cfmm_allreduce_ll")
        return out

    # -- helpers -------------------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def bytes_resident(self) -> int:
        return sum(b.bytes_resident() for b in self.buckets)

    def algorithmic_bytes_per_eval(self) -> int:
        """SURVEY.md section 8(d): 32 B per 2-token pool, 28k+12 per weighted pool, 20k+24 per StableSwap pool (reserves,
        token ids, rates, gamma, A, D), 80 B per concentrated pool (token ids, gamma, (s, c, first record, T), and the b_c,
        L_c, b_{c+1} and end bound the kernel reads for a trade inside the current interval; one that crosses bounds
        reads O(log) records more), + nu, psi, arb."""
        n = 0
        for b in self.buckets:
            n += b.m * (28 * b.arity + 12 if b.kind == _lib.KIND_GEOMEAN else 48 if b.kind == _lib.KIND_BOUNDED
                        else 80 if b.kind == _lib.KIND_CONCENTRATED
                        else 64 if b.kind == _lib.KIND_STABLESWAP
                        else 72 if b.kind == _lib.KIND_CRYPTOSWAP
                        else 148 if b.kind == _lib.KIND_CRYPTOSWAP_3
                        else 20 * b.arity + 24 if b.kind == _lib.KIND_STABLESWAP_N else 32)
        return n + 16 * self.n_tokens + 8

    # -- the hot path --------------------------------------------------------------------------
    def evaluate(self, nu: torch.Tensor, eps: float = 0.0, trades: bool = False, hess: bool = False, reduce: bool = True):
        """psi(nu) (n_tokens) and arb(nu) (1) for this rank's pools, as views into one (n+1) buffer (all-reduced over
        the peer context when enable_peer_allreduce() was called, unless reduce=False: this rank's partial)."""
        st = self._stream()
        acc = self._acc2[self._acc_i]
        nxt = self._acc2[self._acc_i ^ 1]
        self._acc_i ^= 1
        if not self._blocked_first:       # otherwise the previous blocked launch already cleared `acc`
            _lib.check(self.lib.cfmm_zero(acc.data_ptr(), acc.numel() * 8, st), "cfmm_zero")
        lognu = torch.log(nu) if self.has_geomean else None
        for b in self.buckets:
            out = b.out_struct(trades, hess) if (trades or hess) else None
            if getattr(b, "blocked", False):
                rc = self.lib.cfmm_blocked_eval(C.byref(b.c_blocked), self.n_tokens, nu.data_ptr(), acc.data_ptr(),
                                                acc.data_ptr() + 8 * self.n_tokens,
                                                C.byref(out) if out is not None else None,
                                                nxt.data_ptr(), nxt.numel(), st)
                _lib.check(rc, "cfmm_blocked_eval")
                continue
            rc = self.lib.cfmm_arb_eval(C.byref(b.c_bucket), self.n_tokens, nu.data_ptr(),
                                        lognu.data_ptr() if lognu is not None else None, float(eps),
                                        acc.data_ptr(), acc.data_ptr() + 8 * self.n_tokens,
                                        C.byref(out) if out is not None else None, st)
            _lib.check(rc, "cfmm_arb_eval")
        self.evals += 1
        if reduce and getattr(self, "reduces_internally", False):
            return self._peer_reduce(0, acc, self.n_tokens + 1, st)
        return acc

    def hvp(self, vt: torch.Tensor) -> torch.Tensor:
        st = self._stream()
        y = self._y2[self._y_i]
        ynxt = self._y2[self._y_i ^ 1]
        self._y_i ^= 1
        if not self._blocked_first:
            _lib.check(self.lib.cfmm_zero(y.data_ptr(), y.numel() * 8, st), "cfmm_zero")
        for b in self.buckets:
            if getattr(b, "blocked", False):
                _lib.check(self.lib.cfmm_blocked_hvp(C.byref(b.c_blocked), self.n_tokens, b.hcoef.data_ptr(),
                                                     vt.data_ptr(), y.data_ptr(), ynxt.data_ptr(), st),
                           "cfmm_blocked_hvp")
                continue
            rc = self.lib.cfmm_hvp(C.byref(b.c_bucket), self.n_tokens, b.hcoef.data_ptr(),
                                   b.hmask.data_ptr(), vt.data_ptr(), y.data_ptr(), st)
            _lib.check(rc, "cfmm_hvp")
        self.hvps += 1
        if getattr(self, "reduces_internally", False):
            return self._peer_reduce(1, y, self.n_tokens, st)
        return y

    def hess_diag(self) -> torch.Tensor:
        st = self._stream()
        d = torch.zeros(self.n_tokens, dtype=torch.float64, device=self.device)
        for b in self.buckets:
            if getattr(b, "blocked", False):
                _lib.check(self.lib.cfmm_blocked_diag(C.byref(b.c_blocked), self.n_tokens, b.hcoef.data_ptr(),
                                                      d.data_ptr(), st), "cfmm_blocked_diag")
                continue
            _lib.check(self.lib.cfmm_hess_diag(C.byref(b.c_bucket), self.n_tokens, b.hcoef.data_ptr(),
                                               b.hmask.data_ptr(), d.data_ptr(), st), "cfmm_hess_diag")
        if getattr(self, "reduces_internally", False):
            return self._peer_reduce(1, d, self.n_tokens, st).clone()
        return d

    def hess_dense(self) -> torch.Tensor:
        st = self._stream()
        H = torch.zeros((self.n_tokens, self.n_tokens), dtype=torch.float64, device=self.device)
        for b in self.buckets:
            if getattr(b, "blocked", False):
                _lib.check(self.lib.cfmm_blocked_dense(C.byref(b.c_blocked), self.n_tokens, b.hcoef.data_ptr(), H.data_ptr(), st),
                           "cfmm_blocked_dense")
                continue
            _lib.check(self.lib.cfmm_hess_dense(C.byref(b.c_bucket), self.n_tokens, b.hcoef.data_ptr(),
                                                b.hmask.data_ptr(), H.data_ptr(), st), "cfmm_hess_dense")
        return H

    def update_multipliers(self) -> torch.Tensor:
        """theta_bar <- fills of the last trades=True evaluation; returns max relative change (device)."""
        st = self._stream()
        self._move.zero_()
        for b in self.buckets:
            if b.kind == _lib.KIND_SUM:
                _lib.check(self.lib.cfmm_sum_update_multipliers(C.byref(b.c_bucket), b.lam.data_ptr(),
                                                                b.theta_bar.data_ptr(), self._move.data_ptr(), st),
                           "cfmm_sum_update_multipliers")
            elif b.kind == _lib.KIND_BINS:
                _lib.check(self.lib.cfmm_bins_update_multipliers(C.byref(b.c_bucket), b.delta.data_ptr(), b.lam.data_ptr(),
                                                                 b.theta_bar.data_ptr(), self._move.data_ptr(), st),
                           "cfmm_bins_update_multipliers")
        return self._move

    def reset_multipliers(self):
        for b in self.buckets:
            if b.theta_bar is not None:
                b.theta_bar.zero_()

    def market_structs(self):
        """The arguments of cfmm_market_solve that describe this store's pools: (plain cfmm_bucket array, their
        cfmm_eval_out array (trades, hcoef, hmask), n_plain, the blocked bucket's cfmm_blocked_pairs or None, its
        cfmm_eval_out (trades) or None).  The arrays point at this store's buffers; gather_trades() reads the trades of
        the solve's final read-back."""
        plain = [b for b in self.buckets if not getattr(b, "blocked", False)]
        blk = [b for b in self.buckets if getattr(b, "blocked", False)]
        buckets = (_lib.Bucket * max(len(plain), 1))(*[b.c_bucket for b in plain])
        outs = (_lib.EvalOut * max(len(plain), 1))(*[b.out_struct(True, True) for b in plain])
        if not blk:
            return buckets, outs, len(plain), None, None
        return buckets, outs, len(plain), blk[0].c_blocked, blk[0].out_struct(True, False)

    # -- a changed market: new reserves / fees in place ------------------------------------------------
    def _pool_map(self):
        """(bucket index or -1, position in that bucket) of every global pool id, built once per store"""
        if self._where is None:
            bi = np.full(self.m_total, -1, np.int32)
            loc = np.zeros(self.m_total, np.int64)
            for k, b in enumerate(self.buckets):
                s = b.sel                # blocked bucket: the pool at every blocked position (the inverse of its order)
                bi[s] = k
                loc[s] = np.arange(len(s))
            self._where = (bi, loc)
        return self._where

    def _ladders(self) -> LadderSlab:
        if self._lad is None:
            self._lad = LadderSlab(*self._lad_host)
        return self._lad

    def _bins(self) -> LadderSlab:
        if self._bin is None:
            self._bin = LadderSlab(*self._bins_host)
        return self._bin

    def bin_fills(self, i: int, t: float):
        """pools.bin_fills of price-bin pool i as this store holds it now: its current bins (after update_pools(bins=);
        the caller's HostPools still describes the old ones) and its current fee, read from the device.  ValueError if
        pool i is not a bins pool or is held by another rank."""
        i = int(i)
        if not 0 <= i < self.m_total or int(np.asarray(self._kind_host)[i]) != KIND_BINS_HOST:
            raise ValueError(f"pool {i} is not a bins pool")
        bi, loc = self._pool_map()
        if bi[i] < 0:
            raise ValueError(f"pool {i} is held by another rank")
        b, j = self.buckets[bi[i]], int(loc[i])
        z, g = float(b.logrw[2, j]), float(b.gamma[j])
        return _bin_fills(self._bins().records(i), int(z), g, t)

    def update_pools(self, pool_ids, reserves=None, fees=None, prices=None, ladders=None, amp=None, rates=None,
                     curve_gamma=None, bins=None):
        """Set new reserves, fees, prices, ladders, bins, A and / or rates of some pools in place: the store then
        equals, bit for bit, a PoolStore built from a HostPools of the updated literals, without re-uploading the pools or
        rebuilding the blocked layout (which depends on the token ids only).  pool_ids: global pool indices (the order of
        the problem's local_indices); reserves[k]: the new reserve vector of pool pool_ids[k], with the pool's arity (an
        (n, 2) array for pairs); fees[k]: its new gamma in (0, 1].  At least one keyword.  Kinds, tokens, coin counts,
        weighted pools' weights and bounded_product offsets cannot change (they are structure: build a new store).
        A StableSwap pool's invariant D is recomputed from its new reserves, as HostPools does.  amp[k] / rates[k] (StableSwap
        pools only): its new whitepaper A / rate vector (a ramp of A, a moved rate oracle); D is then recomputed with
        stableswap_invariant_any from the pool's reserves after the call (the new ones if reserves= is given, else its
        current ones, read back from the device), and later reserves= updates use the new A and rates.
        Cryptoswap pools take reserves= and fees= (D recomputed with cryptoswap_invariant), rates= (new price scales: a
        repeg of price_scale), amp= and curve_gamma= (a step of ramp_A_gamma); D is then recomputed as for StableSwap.
        Concentrated pools take prices= (prices[k]: the new price of pool pool_ids[k], token 1 per token 0) instead of
        reserves=, which raises for them: their (s, c) and real reserves are recomputed with ladder_state, the function
        HostPools uses.  ladders[k] = (price, bounds, liquidity) (concentrated pools only, not with prices=): the pool's
        whole new ladder, the triple of HostPools.from_lists (instances.v3_ladder of its on-chain state after a Mint or
        Burn); T may change (1 .. LADDER_T_MAX).  Its records are made by ladder_records, as from_lists does, and
        cfmm_ladder_splice rewrites the bucket's records into a second device buffer, which the bucket then uses: a
        ladders= update moves the bucket's records pointer, so a CUDA graph captured over this store must be captured
        again.  The device keeps two record buffers of the concentrated bucket from the first ladders= update on.
        bins[k] = (prices, x, y) (price-bin pools only; with fees= for the same pools if wanted): the pool's whole new
        state, the triple of HostPools.from_lists (instances.lb_bins or instances.order_book of its state after a swap, a
        deposit or withdrawal, a changed book or a filled order); K may change (1 .. BINS_K_MAX), its tokens and which one
        is token 0 may not.  Its records are made by bin_records, as from_lists does, and cfmm_bins_splice rewrites the
        bucket's records like cfmm_ladder_splice: a bins= update also moves the bucket's records pointer, so a CUDA graph
        captured over this store must be captured again.  The replaced pools' multipliers (theta_bar) restart at 0, a
        fresh pool's.  A bins pool takes no reserves= (its reserves are derived from its bins).  store.bin_fills(i, t)
        splits a trade over the pool's current bins.

        All or nothing: bad ids (out of range, repeated), lengths or values (the rules of HostPools.from_lists and
        validate) raise ValueError before anything is written on the device or in the store's host state, and so does an
        entry the device check of the blocked bucket rejects.  Pools held by other ranks of a sharded store are skipped:
        give every rank the same full update.  The caller's HostPools is not modified: the store reads no host reserve or
        fee after construction, and keeps its own copies of the rates, amplifications (copied whole at the first amp= /
        rates= update), ladder and bin records (a LadderSlab each: appends, not copies of every record).  Synchronous.
        Returns the number of blocked tiles whose fee record was rebuilt.

        A new block of the same market is then re-solved warm from the previous prices:
            store.update_pools(ids, reserves=new_R, fees=new_gamma)
            res = solve_pools(hp, utility, store=store, nu0=res.nu)"""
        u = check_pool_update(self.pool_ptr, self._kind_host, self._weights_host, pool_ids, reserves, fees, prices,
                              ladders, amp, rates, curve_gamma, bins)
        bi, loc = self._pool_map()
        owner = bi[u.ids]
        plan = []
        for k, b in enumerate(self.buckets):
            e = np.nonzero(owner == k)[0]
            if len(e) == 0:
                continue
            if u.ladders is not None or u.bins is not None:   # concentrated / bins pools only (checked): in bucket order
                e = e[np.argsort(loc[u.ids[e]], kind="stable")]
            rs = u.ptr[e][None, :] + np.arange(b.arity)[:, None]          # (arity, n) indices into the update's slots
            ids = u.ids[e]
            R = None if u.reserves is None else u.reserves[rs]
            g = None if u.gamma is None else u.gamma[e]
            sc = lad = rt = AD = None
            if u.prices is not None:                 # concentrated pools only (checked): state and reserves at the price
                s, c, x, y = (self._lad.state(ids, u.prices[e]) if self._lad is not None else
                              ladder_state(self._lad_host[0], self._lad_host[1], ids, u.prices[e]))
                sc, R = np.stack([s, c]), np.stack([x, y])
            if u.ladders is not None:                # new records and state, as HostPools.from_lists makes them
                rec, cnt, s, c, x, y = new_ladders([u.ladders[j] for j in e.tolist()])
                n_total = b.n_rec + int(cnt.sum()) - int((self._ladders().T[ids] + 1).sum())
                lad = (rec, cnt, np.stack([s, c, x, y], 1), n_total)
            if u.bins is not None:                   # new records and (z, p_ref, sum x, sum y), as from_lists makes them
                rec, cnt, state = _pack_bins([u.bins[j] for j in e.tolist()])
                n_total = b.n_rec + int(cnt.sum()) - int((self._bins().T[ids] + 1).sum())
                lad = (rec, cnt, state, n_total)
            if u.amp is not None or u.rates is not None or u.curve_gamma is not None:
                # StableSwap or cryptoswap pools only (checked): D of the reserves after the call
                A = u.amp[e] if u.amp is not None else self._amp_host[ids]
                rt = u.rates[rs] if u.rates is not None else self._weights_host[u.slots[rs]]
                Rd = R if R is not None else b.reserves[:, torch.as_tensor(loc[ids], device=self.device)].cpu().numpy()
                if b.kind in (_lib.KIND_CRYPTOSWAP, _lib.KIND_CRYPTOSWAP_3):
                    G = u.curve_gamma[e] if u.curve_gamma is not None else self._cgam_host[ids]
                    D = cryptoswap_invariant_any(Rd.T, rt.T, A, G)
                    AD = np.stack([A, G, D])
                else:
                    D = stableswap_invariant_any(Rd.T, rt.T, A)
                    AD = np.stack([A, D])
                if not bool(np.all(np.isfinite(D) & (D > 0))):
                    raise ValueError("invariant D must be finite and > 0 (scaled balances out of fp64 range?)")
            plan.append((b, loc[ids], R, g, rs, ids, sc, lad, rt, AD))
        # the blocked bucket first: it checks its entries on the device and writes nothing if one is invalid
        rebuilt = 0
        for b, l, R, g, *_ in plan:
            if getattr(b, "blocked", False):
                rebuilt += b.write_update(self.lib, l, R, g, self._stream())
        for b, l, R, g, rs, ids, sc, lad, rt, AD in plan:
            if getattr(b, "blocked", False):
                continue
            if lad is not None:
                b.splice_records(self.lib, l, lad[0], lad[1], lad[2], lad[3], self._stream())
            W = self._weights_host[u.slots[rs]] if (R is not None and b.logrw is not None and AD is None) else None
            crypto = b.kind in (_lib.KIND_CRYPTOSWAP, _lib.KIND_CRYPTOSWAP_3)
            amp_ = self._amp_host[ids] if b.kind in (_lib.KIND_STABLESWAP, _lib.KIND_STABLESWAP_N) or crypto else None
            cg_ = self._cgam_host[ids] if crypto else None
            b.write_update(l, R, g, W, amp_, sc, None if u.rates is None else rt, AD, cg_)
        # the store's host state, once the device holds the update
        for b, l, R, g, rs, ids, sc, lad, rt, AD in plan:
            if lad is not None:
                (self._bins() if b.kind == _lib.KIND_BINS else self._ladders()).replace(ids, lad[0], lad[1])
            if AD is not None:
                if not self._own_stable:
                    self._weights_host, self._amp_host = self._weights_host.copy(), self._amp_host.copy()
                    self._cgam_host = self._cgam_host.copy()
                    self._own_stable = True
                self._amp_host[ids] = AD[0]
                if b.kind in (_lib.KIND_CRYPTOSWAP, _lib.KIND_CRYPTOSWAP_3):
                    self._cgam_host[ids] = AD[1]
                self._weights_host[u.slots[rs]] = rt
        torch.cuda.synchronize(self.device)
        return rebuilt

    def gather_trades(self):
        """Delta, Lambda of the last trades=True evaluation, CSR order of the ORIGINAL pools (host).
        Entries of pools living on other ranks are left at zero."""
        nnz = int(self.pool_ptr[-1])
        delta = np.zeros(nnz); lam = np.zeros(nnz)
        for b in self.buckets:
            if b.m == 0:
                continue
            delta[b.off.ravel()] = b.delta[:, :b.m].cpu().numpy().ravel()
            lam[b.off.ravel()] = b.lam[:, :b.m].cpu().numpy().ravel()
        return delta, lam
