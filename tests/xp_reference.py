"""Extended-precision reference of the per-pool optimal trades, and an oracle-free certificate of a returned answer
(test helper, not a test module).

Everything here is numpy ``longdouble``, vectorised, and imports neither the package's kernels nor ``oracle/``: each
kind's closed form is re-stated from the reference's constraints (arbitrage.py:60-74).  Pool data is read from the
CSR fields of a ``HostPools`` (``n_tokens``, ``pool_ptr``, ``tok_idx``, ``reserves``, ``weights``, ``gamma``,
``kind``); utilities from the four fields of their linear + box form (``c``, ``a``, ``eq``, ``pinned``).

response(hp, nu) gives the exact (eps = 0) optimal trades of every pool at prices nu:
    max  nu'(L - D)   s.t.  phi(R + gamma D - L) >= phi(R),  D, L >= 0
  * constant product    phi = sqrt(x0 x1)                  t = sqrt(gamma p_b / p_a), p = nu R
  * bounded product     phi = sqrt((x0+o0)(x1+o1)), x >= 0  the constant-product trade on V = R + o, payout capped at R
  * constant sum        phi = x0 + x1, x >= 0               an LP: fill the whole order when gamma nu_b > nu_a
  * weighted geomean    phi = prod x^w                      x_j = clip(R_j, gamma M w_j / nu_j, M w_j / nu_j), with
                        s = log M the root of h(s) = sum_j w_j [max(s - tA_j, 0) + min(s - tB_j, 0)],
                        tB_j = log(R_j nu_j / w_j), tA_j = tB_j - log gamma (h is piecewise linear and nondecreasing)
"""
from __future__ import annotations

import numpy as np

LD = np.longdouble
# x86-64: 80-bit extended (eps 2^-63); aarch64: binary128.  fp64 would make the reference as wrong as what it checks.
assert np.finfo(LD).eps <= 2.0 ** -63, "xp_reference needs an extended-precision numpy longdouble"

KIND_GEOMEAN, KIND_SUM, KIND_BOUNDED = 0, 1, 3          # host CSR kind codes
U64 = 2.0 ** -53                                         # unit roundoff of fp64


def ld(x):
    return np.asarray(x).astype(LD)


def _groups(hp):
    """(kind tag, pool ids, (m_g, k) slot offsets) per kind and arity; constant-product = geomean, arity 2, w = (1/2, 1/2)"""
    ptr = np.asarray(hp.pool_ptr, np.int64)
    ar = np.diff(ptr)
    kind = np.asarray(hp.kind)
    w = np.asarray(hp.weights, float)
    out = []
    for k in np.unique(ar):
        for kd in (KIND_GEOMEAN, KIND_SUM, KIND_BOUNDED):
            sel = np.nonzero((ar == k) & (kind == kd))[0]
            if len(sel) == 0:
                continue
            off = ptr[sel][:, None] + np.arange(k)[None, :]
            if kd == KIND_GEOMEAN and k == 2:
                cp = np.all(w[off] == 0.5, axis=1)
                for tag, s in (("product", cp), ("geomean", ~cp)):
                    if s.any():
                        out.append((tag, sel[s], off[s]))
            else:
                out.append(({KIND_GEOMEAN: "geomean", KIND_SUM: "sum", KIND_BOUNDED: "bounded"}[kd], sel, off))
    return out


def _product(R, g, nu):
    p = nu * R
    D = np.zeros_like(R); L = np.zeros_like(R); h = np.zeros(len(g), LD)
    for a, b in ((0, 1), (1, 0)):
        go = g * p[:, b] > p[:, a]
        t = np.sqrt(np.where(go, g * p[:, b] / p[:, a], LD(1)))
        D[:, a] = np.where(go, R[:, a] * (t - 1) / g, 0)
        L[:, b] = np.where(go, R[:, b] * (1 - 1 / t), 0)
        h = np.where(go, np.sqrt(p[:, 0] * p[:, 1] / g) / 2, h)
    return D, L, h


def _bounded(R, o, g, nu):
    V = R + o
    p = nu * V
    D = np.zeros_like(R); L = np.zeros_like(R); h = np.zeros(len(g), LD)
    for a, b in ((0, 1), (1, 0)):
        go = g * p[:, b] > p[:, a]
        t = np.sqrt(np.where(go, g * p[:, b] / p[:, a], LD(1)))
        Lb = V[:, b] * (1 - 1 / t)
        cap = go & (Lb > R[:, b])
        # at the cap the pool pays out all of R_b: (V_a + gamma D_a) o_b = V_a V_b  =>  D_a = V_a R_b / (gamma o_b)
        with np.errstate(divide="ignore", invalid="ignore"):
            Dcap = V[:, a] * R[:, b] / (g * o[:, b])
        L[:, b] = np.where(go, np.where(cap, R[:, b], Lb), 0)
        D[:, a] = np.where(go, np.where(cap, Dcap, V[:, a] * (t - 1) / g), 0)
        h = np.where(go & ~cap, np.sqrt(p[:, 0] * p[:, 1] / g) / 2, h)
    return D, L, h


def _sum(R, g, nu):
    D = np.zeros_like(R); L = np.zeros_like(R)
    for a, b in ((0, 1), (1, 0)):
        go = g * nu[:, b] > nu[:, a]             # one unit of a buys gamma of b: take the whole order, up to R_b
        L[:, b] = np.where(go, R[:, b], 0)
        D[:, a] = np.where(go, R[:, b] / g, 0)
    return D, L, np.zeros(len(g), LD)


def _geomean(R, w, g, nu):
    tB = np.log(R * nu / w)
    tA = tB - np.log(g)[:, None]
    trade = tB.max(1) > tA.min(1)
    T = np.concatenate([tA, tB], 1)                                                   # every breakpoint of h
    hT = (w[:, None, :] * (np.maximum(T[:, :, None] - tA[:, None, :], 0)
                           + np.minimum(T[:, :, None] - tB[:, None, :], 0))).sum(2)
    p = np.where(hT <= 0, T, LD(-np.inf)).argmax(1)                                   # last breakpoint with h <= 0
    rows = np.arange(len(p))
    sL, hL = T[rows, p], hT[rows, p]
    W = (w * ((sL[:, None] >= tA) | (sL[:, None] < tB))).sum(1)                       # slope of h right of sL
    s = np.where(hL < 0, sL - hL / np.where(W > 0, W, LD(1)), sL)
    zA = np.where(trade[:, None], np.maximum(s[:, None] - tA, 0), 0)
    zB = np.where(trade[:, None], np.minimum(s[:, None] - tB, 0), 0)
    D = R * np.expm1(zA) / g[:, None]
    L = -R * np.expm1(zB)
    return D, L, np.where(trade, np.exp(s), 0)


def response(hp, nu):
    """Exact optimal trades at prices nu (longdouble): dict(delta, lam [nnz, CSR slot order], arb [m] = nu'(L - D) per
    pool, h [m]).  h: the coefficient of [[1,-1],[-1,1]] in the scaled Hessian for 2-token kinds (sqrt(p0 p1/gamma)/2 on
    trading constant-product and uncapped bounded pools; 0 for the exact constant-sum LP), M = exp(s) for weighted
    pools of other shapes."""
    nu = ld(nu)
    R_all, w_all, g_all = ld(hp.reserves), ld(hp.weights), ld(hp.gamma)
    tok = np.asarray(hp.tok_idx, np.int64)
    nnz, m = len(R_all), len(g_all)
    delta = np.zeros(nnz, LD); lam = np.zeros(nnz, LD); arb = np.zeros(m, LD); h = np.zeros(m, LD)
    for tag, sel, off in _groups(hp):
        R, g, nv = R_all[off], g_all[sel], nu[tok[off]]
        if tag == "product":
            D, L, hh = _product(R, g, nv)
        elif tag == "bounded":
            D, L, hh = _bounded(R, w_all[off], g, nv)
        elif tag == "sum":
            D, L, hh = _sum(R, g, nv)
        else:
            D, L, hh = _geomean(R, w_all[off], g, nv)
        delta[off.ravel()] = D.ravel(); lam[off.ravel()] = L.ravel()
        arb[sel] = (nv * (L - D)).sum(1); h[sel] = hh
    return dict(delta=delta, lam=lam, arb=arb, h=h)


def token_sums(hp, *vals):
    """Per-token sums of per-slot longdouble arrays, in longdouble (np.add.at / bincount would go through float64):
    slots sorted by token, np.add.reduceat over each token's run."""
    tok = np.asarray(hp.tok_idx, np.int64)
    order = np.argsort(tok, kind="stable")
    t = tok[order]
    starts = np.flatnonzero(np.r_[True, t[1:] != t[:-1]]) if len(t) else np.zeros(0, np.int64)
    out = []
    for v in vals:
        full = np.zeros(hp.n_tokens, LD)
        if len(t):
            full[t[starts]] = np.add.reduceat(ld(v)[order], starts)
        out.append(full)
    return out


def flows(hp, delta, lam):
    """psi = sum_i A_i (L_i - D_i), gross_j = sum |flows| at token j, and k_j = the number of non-zero flows at j"""
    d, l = ld(delta), ld(lam)
    psi, gross, k = token_sums(hp, l - d, l + d, ((d != 0) | (l != 0)).astype(LD))
    return psi, gross, k


def arb(hp, nu):
    """sum_i arb_i(nu), in longdouble"""
    return response(hp, nu)["arb"].sum()


# ----------------------------------------------------------------------------------------------------------------------
# the certificate
# ----------------------------------------------------------------------------------------------------------------------
FEAS_TOL = 1e-12         # pool feasibility, in log / relative form: fp64 trades on the curve miss it by a few u times the
                         # relative size of the trade (|log change| <~ 8 u (1 + D/R + L/R)); 1e-12 is >= 100x that for any
                         # trade under 100x its reserve, and far below what a wrong trade moves (>= 1e-9 relative)
PSI_SAFETY = 4.0         # psi vs its trades: summing k_j flows in any order errs by <= (k_j - 1) u gross_j; a flow the
                         # kernel rounded differently from the trade it returned adds <= ~2 u |flow| more.  4 k_j u gross_j
                         # covers both with a factor of 2 to spare
ROUND_REL = 1e-12        # dual / primal values: they are sums of fp64 flows, each with relative error <= ~10 u, weighted
                         # by prices: |error| <= ~1e-15 nu'gross.  1e-12 nu'gross leaves 1000x for the reduction order


def _trades(result, hp):
    d = np.concatenate([np.asarray(x, float).ravel() for x in result.deltas]) if len(result.deltas) else np.zeros(0)
    l = np.concatenate([np.asarray(x, float).ravel() for x in result.lambdas]) if len(result.lambdas) else np.zeros(0)
    nnz = int(np.asarray(hp.pool_ptr)[-1])
    assert len(d) == len(l) == nnz, f"trades: {len(d)} / {len(l)} entries for {nnz} pool slots"
    return d, l


def pool_feasibility(hp, delta, lam):
    """Worst violation of each kind's constraint by the trades (<= 0 is feasible):
      product / geomean: -(sum_j w_j log1p((gamma D_j - L_j) / R_j))        (the invariant may not drop)
      bounded product:   -(sum_j log1p((gamma D_j - L_j) / V_j)) / 2,  and -x_j / V_j  (real reserves stay >= 0)
      constant sum:      -(sum_j (gamma D_j - L_j)) / sum_j R_j,  and (L_j - R_j) / sum_j R_j
    plus -min(D, L) / (the pool's reserve scale) for the sign of the trades.  Every kind is measured against a scale that
    stays positive when one real reserve is 0 (V_j for bounded pools, sum_j R_j for constant-sum ones).  Returns the max
    over pools (longdouble)."""
    d, l = ld(delta), ld(lam)
    R_all, w_all, g_all = ld(hp.reserves), ld(hp.weights), ld(hp.gamma)
    worst = LD(-np.inf)
    for tag, sel, off in _groups(hp):
        D, L, R, g = d[off], l[off], R_all[off], g_all[sel][:, None]
        ch = g * D - L
        if tag == "sum":
            sc = R.sum(1, keepdims=True)
            v = np.maximum(-ch.sum(1) / sc[:, 0], ((L - R) / sc).max(1))
        else:
            V = R + w_all[off] if tag == "bounded" else R
            with np.errstate(invalid="ignore", divide="ignore"):
                lg = np.log1p(ch / V)                               # a post-trade reserve <= 0: nan / -inf, infeasible
            lg = np.where(np.isnan(lg), LD(-np.inf), lg)
            v = -(lg.sum(1) / 2 if tag == "bounded" else (w_all[off] * lg).sum(1))
            if tag == "bounded":
                v = np.maximum(v, (-(R + ch) / V).max(1))
            sc = V                                                   # a bounded pool's real reserve may be 0
        v = np.maximum(v, (-np.minimum(D, L) / sc).max(1))
        worst = max(worst, v.max())
    return worst


def certify(hp, spec, result, tol, check=True):
    """Oracle-free certificate of a returned answer (result.deltas / lambdas / psi / nu / value / dual_value), computed in
    longdouble.  Raises AssertionError naming every check that fails; returns the measured quantities otherwise.

    1. pool-feasible trades: D, L >= 0 and no pool's invariant drops by more than FEAS_TOL (pool_feasibility).
    2. psi matches the trades: |psi_j - sum A(L - D)_j| <= PSI_SAFETY k_j u gross_j.
    3. token constraints: viol_j = |psi_j + a_j| (eq), max(-(psi_j + a_j), 0) (inequality), 0 (pinned), each
       <= tol S + 1e-12 gross_j with S = max(|a|_inf, max over constrained tokens |psi_j|): the per-token term of the
       stopping rule, which status 'optimal' promises.
    4. the dual bound closes the gap.  nu^ = result.nu projected on the dual-feasible set (= c on pinned tokens, >= c on
       inequality tokens, free on eq tokens); D = sum (nu^ - c) a + sum_i arb_i(nu^) and P = c'psi_xp (psi_xp = the
       trades' own sum).  For any pool-feasible trades with net flow psi,
           D - P = sum_j (nu^_j - c_j)(psi_j + a_j) + [sum_i arb_i(nu^) - nu^'psi],
       and the bracket is >= 0 because arb_i is the best any feasible trade of pool i earns at prices nu^.  The first sum
       is >= 0 when psi is feasible (each term: (>= 0)(>= 0), or a zero factor); psi may miss its constraints by viol_j
       (check 3), so D - P >= -V with V = sum_j |nu^_j - c_j| viol_j.  (V = 0 for a feasible psi: then D >= OPT >= P.)
       Above, the stopping rule bounds the value-weighted residual sum |nu_j (a_j + psi_j)| by tol |g|, which bounds the
       first sum, and the exact trades at nu make the bracket vanish (the smoothed constant-sum trades leave it at the
       certified exact gap, <= tol |D|); so D - P <= 2 tol |D| allows for both.  Asserted:
           -eps - V/|D| <= (D - P)/|D| <= 2 tol + eps,   eps = ROUND_REL (nu^'gross) / |D|.
    5. the reported scalars: |value - P| and |dual_value - D| <= eps |D|; nu finite and > 0, nu == c on pinned tokens,
       nu >= c (1 - 1e-15) on inequality tokens."""
    c, a = ld(spec.c), ld(spec.a)
    eq, pinned = np.asarray(spec.eq, bool), np.asarray(spec.pinned, bool)
    ineq = ~eq & ~pinned
    fails = []
    rep = {}                     # each measured quantity next to its bound, for the record
    d, l = _trades(result, hp)
    # 1
    feas = pool_feasibility(hp, d, l)
    rep["pool_feasibility"] = (float(feas), FEAS_TOL)
    if not feas <= FEAS_TOL:
        fails.append(f"trades are not pool-feasible: worst invariant drop {float(feas):.3e} > {FEAS_TOL:.0e}")
    # 2
    psi_xp, gross, k = flows(hp, d, l)
    psi = ld(result.psi)
    dpsi = np.abs(psi - psi_xp)
    bound2 = LD(PSI_SAFETY * U64) * np.maximum(k, 1) * gross
    r2 = np.where(dpsi > 0, dpsi / np.where(bound2 > 0, bound2, LD(1e-300)), 0)
    rep["psi_vs_trades"] = (float(r2.max(initial=0)), 1.0)
    if not np.all(dpsi <= bound2):
        j = int(np.argmax(dpsi - bound2))
        fails.append(f"psi does not match the trades: token {j}: |psi - sum| = {float(dpsi[j]):.3e} > "
                     f"{float(bound2[j]):.3e} (k = {int(k[j])}, gross = {float(gross[j]):.3e})")
    # 3
    s = psi + a
    viol = np.where(pinned, LD(0), np.where(eq, np.abs(s), np.maximum(-s, 0)))
    S = max(np.abs(a).max(initial=LD(0)), np.abs(np.where(pinned, LD(0), psi)).max(initial=LD(0)))
    bound3 = LD(tol) * S + LD(1e-12) * gross
    rep["token_constraints"] = (float((viol / max(S, LD(1e-300))).max(initial=0)), tol)
    if not np.all(viol <= bound3):
        j = int(np.argmax(viol - bound3))
        fails.append(f"token constraint violated: token {j}: {float(viol[j]):.3e} > {float(bound3[j]):.3e} (tol S)")
    # 4
    nu_r = ld(result.nu)
    nuh = np.where(pinned, c, np.where(ineq, np.maximum(nu_r, c), nu_r))
    D = ((nuh - c) * a).sum() + arb(hp, nuh)
    P = (c * psi_xp).sum()
    aD = max(abs(D), LD(1e-300))
    eps = LD(ROUND_REL) * (nuh * gross).sum() / aD
    V = (np.abs(nuh - c) * viol).sum() / aD
    gap = (D - P) / aD
    rep["gap"] = (float(gap), 2 * tol + float(eps)); rep["gap_lower"] = (float(-gap), float(eps + V))
    rep["D"], rep["P"] = float(D), float(P)
    if not gap <= LD(2 * tol) + eps:
        fails.append(f"dual bound does not close the gap: (D - P)/|D| = {float(gap):.3e} > {float(2 * tol + eps):.3e}")
    if not -eps - V <= gap:                     # only trades that are not pool-feasible get here (see above)
        fails.append(f"primal value exceeds the dual bound: (D - P)/|D| = {float(gap):.3e} < {float(-eps - V):.3e}")
    # 5
    dv = abs(ld(result.value) - P) / aD
    dd = abs(ld(result.dual_value) - D) / aD
    rep["value"] = (float(dv), float(eps)); rep["dual_value"] = (float(dd), float(eps))
    if not dv <= eps:
        fails.append(f"reported value disagrees with c'psi of the trades: {float(dv):.3e} > {float(eps):.3e} of |D|")
    if not dd <= eps:
        fails.append(f"reported dual_value disagrees with the dual bound: {float(dd):.3e} > {float(eps):.3e} of |D|")
    nu64 = np.asarray(result.nu, float)
    if not (np.all(np.isfinite(nu64)) and np.all(nu64 > 0)):
        fails.append("nu is not finite and positive")
    if not np.array_equal(nu64[pinned], np.asarray(spec.c, float)[pinned]):
        fails.append("nu differs from c on a pinned token")
    if not np.all(nu64[ineq] >= np.asarray(spec.c, float)[ineq] * (1 - 1e-15)):
        fails.append("nu < c on an inequality token (the dual box nu >= c)")
    if check and fails:
        raise AssertionError("certificate failed:\n  " + "\n  ".join(fails))
    rep["fails"] = fails
    return rep
