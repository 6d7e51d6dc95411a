"""Problem instances: the reference's three scripts as data, and the BASELINE.json synthetic configs.

Reference literals (problem DATA, not code):
  arbitrage_instance()   <- arbitrage.py:5-36    (4 tokens, 5 pools, market_value)
  liquidation_instance() <- liquidation.py:5-36  (5 tokens, 5 pools, current_assets)
  two_asset_instance()   <- two-asset.py:7-34    (3 tokens, 5 pools, amounts = linspace(0, 50))
Synthetic generators follow SURVEY.md section 8(d) (cfg 2-5), seeded numpy default_rng.
"""
from __future__ import annotations

import numpy as np


def _five_pools(first_pool, weights0, pair_a, pair_b, pair_c):
    # all three scripts share one shape: a weighted pool over every token, three
    # constant-product pairs and one constant-sum pair (the last two on the same pair)
    return dict(
        local_indices=[list(first_pool), list(pair_a), list(pair_b), list(pair_c), list(pair_c)],
        kinds=["geomean", "product", "product", "product", "sum"],
        weights=[list(weights0), None, None, None, None],
    )


def arbitrage_instance():
    d = _five_pools(range(4), (4, 3, 2, 1), (0, 1), (1, 2), (2, 3))
    d.update(
        n_tokens=4,
        reserves=[[4, 4, 4, 4], [10, 1], [1, 5], [40, 50], [10, 10]],
        fees=[0.998, 0.997, 0.997, 0.997, 0.999],
        market_value=[1.5, 10, 2, 3],
    )
    return d


def liquidation_instance():
    d = _five_pools(range(5), (5, 4, 3, 2, 1), (0, 1), (2, 3), (3, 4))
    d.update(
        n_tokens=5,
        reserves=[[4, 4, 4, 4, 4], [10, 1], [1, 5], [40, 50], [10, 10]],
        fees=[0.998, 0.997, 0.997, 0.997, 0.999],
        current_assets=[2, 1, 3, 5, 10],
        target=4,
    )
    return d


def two_asset_instance():
    d = _five_pools(range(3), (3, 2, 1), (0, 1), (1, 2), (0, 2))
    d.update(
        n_tokens=3,
        reserves=[[3, 0.2, 1], [10, 1], [1, 10], [20, 50], [10, 10]],
        fees=[0.98, 0.99, 0.96, 0.97, 0.99],
        amounts=np.linspace(0, 50),
        tok_in=0,
        tok_out=2,
    )
    return d


# ------------------------------------------------------------------------------------------
# synthetic configs (BASELINE.json configs[1..4]; SURVEY.md section 8d)
# ------------------------------------------------------------------------------------------
_FEES = np.array([0.997, 0.999, 0.9995])


def synth_const_product(m, n_tokens, seed, mispricing=0.02):
    """cfg 2 (m=10_000, n=256, seed 0) and cfg 5 (m=1_000_000, n=4096, seed 3)."""
    rng = np.random.default_rng(seed)
    p = np.exp(rng.standard_normal(n_tokens))
    a = rng.integers(0, n_tokens, m)
    b = (a + 1 + rng.integers(0, n_tokens - 1, m)) % n_tokens          # b != a
    liq = np.exp(8.0 + 1.5 * rng.standard_normal(m))
    Ra = liq / p[a] * np.exp(mispricing * rng.standard_normal(m))
    Rb = liq / p[b] * np.exp(mispricing * rng.standard_normal(m))
    gamma = _FEES[rng.integers(0, 3, m)]
    return dict(
        n_tokens=n_tokens, prices=p,
        idx=np.stack([a, b], 1).astype(np.int32), reserves=np.stack([Ra, Rb], 1), gamma=gamma,
    )


def synth_mixed(m, n_tokens, seed, frac_product=0.6, frac_weighted=0.3, mispricing=0.02):
    """cfg 3 / cfg 4 pool population: const-product, weighted (arity 2..8), const-sum pairs
    on tokens whose prices are within 1 %.  Returned in list form (CSR is built by the
    caller) plus the price vector."""
    rng = np.random.default_rng(seed)
    p = np.exp(rng.standard_normal(n_tokens))
    # make near-pegged token pairs exist: every 10th token copies its neighbour's price +-0.5 %
    peg = np.arange(1, n_tokens, 10)
    p[peg] = p[peg - 1] * np.exp(0.005 * rng.standard_normal(len(peg)))
    n_cp = int(round(frac_product * m)); n_w = int(round(frac_weighted * m)); n_cs = m - n_cp - n_w
    ptr = [0]; idx = []; res = []; wts = []; gam = []; kind = []
    cp = synth_const_product(n_cp, n_tokens, seed + 1000, mispricing)
    # rebuild const-product reserves against THIS price vector
    a, b = cp["idx"][:, 0], cp["idx"][:, 1]
    liq = np.exp(8.0 + 1.5 * rng.standard_normal(n_cp))
    Ra = liq / p[a] * np.exp(mispricing * rng.standard_normal(n_cp))
    Rb = liq / p[b] * np.exp(mispricing * rng.standard_normal(n_cp))
    out_idx = [np.stack([a, b], 1)]; out_R = [np.stack([Ra, Rb], 1)]
    out_w = [np.full((n_cp, 2), 0.5)]; out_g = [cp["gamma"]]; out_k = [np.zeros(n_cp, np.uint8)]
    out_ar = [np.full(n_cp, 2)]
    # weighted pools
    ar = rng.integers(2, 9, n_w)
    for k in range(2, 9):
        sel = np.nonzero(ar == k)[0]
        if len(sel) == 0:
            continue
        mk = len(sel)
        toks = np.argsort(rng.random((mk, n_tokens)), axis=1)[:, :k] if n_tokens <= 4096 and mk * n_tokens <= 5e7 \
            else np.stack([rng.choice(n_tokens, k, replace=False) for _ in range(mk)])
        w = rng.dirichlet(np.ones(k), mk)
        w = np.maximum(w, 0.02); w /= w.sum(1, keepdims=True)
        L = np.exp(8.0 + 1.5 * rng.standard_normal(mk))
        R = L[:, None] * w / p[toks] * np.exp(mispricing * rng.standard_normal((mk, k)))
        out_idx.append(toks); out_R.append(R); out_w.append(w)
        out_g.append(_FEES[rng.integers(0, 3, mk)]); out_k.append(np.zeros(mk, np.uint8))
        out_ar.append(np.full(mk, k))
    # const-sum pairs on pegged tokens
    pa = peg[rng.integers(0, len(peg), n_cs)]
    pb = pa - 1
    Rcs = np.exp(6.0 + rng.standard_normal((n_cs, 2)))
    out_idx.append(np.stack([pa, pb], 1)); out_R.append(Rcs); out_w.append(np.zeros((n_cs, 2)))
    out_g.append(_FEES[rng.integers(0, 3, n_cs)]); out_k.append(np.ones(n_cs, np.uint8))
    out_ar.append(np.full(n_cs, 2))
    arity = np.concatenate(out_ar)
    pool_ptr = np.concatenate([[0], np.cumsum(arity)]).astype(np.int64)
    return dict(
        n_tokens=n_tokens, prices=p, pool_ptr=pool_ptr,
        tok_idx=np.concatenate([x.ravel() for x in out_idx]).astype(np.int32),
        reserves=np.concatenate([x.ravel() for x in out_R]),
        weights=np.concatenate([x.ravel() for x in out_w]),
        gamma=np.concatenate(out_g), kind=np.concatenate(out_k),
    )


def synth_stable_market(m, n_tokens, seed, frac_stable=0.3, frac_weighted=0.1, n_stable=8, mispricing=0.02):
    """A market with a stablecoin cluster: tokens 0..n_stable-1 trade near 1 (within +-0.2 %), the last three of them
    are rate-bearing (worth 1.02 / 1.05 / 1.1 of the others: wrapped or yield-bearing stablecoins).  StableSwap pools
    (A in {50 .. 2000}, Curve's usual range; rates = the tokens' values) join pairs of the cluster, beside constant-
    product pools over all tokens (the cluster included) and weighted pools of arity 2..4.  Balances are imbalanced by
    up to ~2x and mispriced by `mispricing`.  Returns CSR arrays (HostPools(**out) minus `prices`) plus the prices."""
    rng = np.random.default_rng(seed)
    n_stable = min(n_stable, n_tokens)
    p = np.exp(rng.standard_normal(n_tokens))
    rate = np.ones(n_tokens)
    rate[max(0, n_stable - 3):n_stable] = [1.02, 1.05, 1.1][-min(3, n_stable):]
    p[:n_stable] = rate[:n_stable] * np.exp(0.002 * rng.uniform(-1, 1, n_stable))
    n_ss = int(round(frac_stable * m)) if n_stable >= 2 else 0
    n_w = int(round(frac_weighted * m)); n_cp = m - n_ss - n_w
    # constant product over all tokens
    a = rng.integers(0, n_tokens, n_cp); b = (a + rng.integers(1, n_tokens, n_cp)) % n_tokens
    liq = np.exp(8.0 + 1.5 * rng.standard_normal(n_cp))
    out_idx = [np.stack([a, b], 1)]
    out_R = [np.stack([liq / p[a], liq / p[b]], 1) * np.exp(mispricing * rng.standard_normal((n_cp, 2)))]
    out_w = [np.full((n_cp, 2), 0.5)]; out_g = [_FEES[rng.integers(0, 3, n_cp)]]; out_k = [np.zeros(n_cp, np.uint8)]
    out_ar = [np.full(n_cp, 2)]; out_amp = [np.zeros(n_cp)]
    # weighted pools
    for k in (2, 3, 4):
        mk = n_w // 3 + (1 if k - 2 < n_w % 3 else 0)
        if mk == 0 or k > n_tokens:
            continue
        toks = np.stack([rng.choice(n_tokens, k, replace=False) for _ in range(mk)])
        w = rng.dirichlet(np.ones(k), mk); w = np.maximum(w, 0.05); w /= w.sum(1, keepdims=True)
        L = np.exp(8.0 + 1.5 * rng.standard_normal(mk))
        out_idx.append(toks); out_R.append(L[:, None] * w / p[toks] * np.exp(mispricing * rng.standard_normal((mk, k))))
        out_w.append(w); out_g.append(_FEES[rng.integers(0, 3, mk)]); out_k.append(np.zeros(mk, np.uint8))
        out_ar.append(np.full(mk, k)); out_amp.append(np.zeros(mk))
    # StableSwap pools inside the cluster: value-balanced up to a factor ~2, rates = the tokens' values
    if n_ss:
        sa = rng.integers(0, n_stable, n_ss); sb = (sa + rng.integers(1, n_stable, n_ss)) % n_stable
        V = np.exp(9.0 + 1.5 * rng.standard_normal(n_ss))
        imb = np.exp(0.35 * rng.standard_normal(n_ss))
        R = np.stack([V * imb / p[sa], V / imb / p[sb]], 1) * np.exp(mispricing * rng.standard_normal((n_ss, 2)))
        out_idx.append(np.stack([sa, sb], 1)); out_R.append(R); out_w.append(np.stack([rate[sa], rate[sb]], 1))
        out_g.append(np.array([0.9996, 0.9999, 0.99995])[rng.integers(0, 3, n_ss)])
        out_k.append(np.full(n_ss, 4, np.uint8)); out_ar.append(np.full(n_ss, 2))
        out_amp.append(np.array([50.0, 100.0, 200.0, 1000.0, 2000.0])[rng.integers(0, 5, n_ss)])
    arity = np.concatenate(out_ar)
    return dict(
        n_tokens=n_tokens, prices=p,
        pool_ptr=np.concatenate([[0], np.cumsum(arity)]).astype(np.int64),
        tok_idx=np.concatenate([x.ravel() for x in out_idx]).astype(np.int32),
        reserves=np.concatenate([x.ravel() for x in out_R]),
        weights=np.concatenate([x.ravel() for x in out_w]),
        gamma=np.concatenate(out_g), kind=np.concatenate(out_k), amp=np.concatenate(out_amp),
    )


def synth_stable_n_market(m, n_tokens, seed, frac_stable=0.3, n_stable=8, mispricing=0.02, arities=(2, 3, 4)):
    """A market with StableSwap clusters of several coin counts: tokens 0..n_stable-1 trade near 1 (within +-0.2 %),
    the last two of them rate-bearing (worth 1.02 / 1.05 of the others).  StableSwap pools of each arity in `arities`
    (in equal shares, tokens drawn from the cluster without repetition; whitepaper A with A n^n in 100 .. 2e4, the
    coefficients of Curve's usual A() = 50 .. 5000 at n = 2..4; rates = the tokens' values) sit beside constant-product
    pools over all tokens, the cluster included.  Balances are value-imbalanced by up to ~2x and mispriced by
    `mispricing`.  Returns CSR arrays (HostPools(**out) minus `prices`) plus the prices."""
    rng = np.random.default_rng(seed)
    n_stable = min(n_stable, n_tokens)
    arities = [k for k in arities if k <= n_stable]
    p = np.exp(rng.standard_normal(n_tokens))
    rate = np.ones(n_tokens)
    rate[max(0, n_stable - 2):n_stable] = [1.02, 1.05][-min(2, n_stable):]
    p[:n_stable] = rate[:n_stable] * np.exp(0.002 * rng.uniform(-1, 1, n_stable))
    n_ss = int(round(frac_stable * m)) if arities else 0
    n_cp = m - n_ss
    a = rng.integers(0, n_tokens, n_cp); b = (a + rng.integers(1, n_tokens, n_cp)) % n_tokens
    liq = np.exp(8.0 + 1.5 * rng.standard_normal(n_cp))
    out_idx = [np.stack([a, b], 1)]
    out_R = [np.stack([liq / p[a], liq / p[b]], 1) * np.exp(mispricing * rng.standard_normal((n_cp, 2)))]
    out_w = [np.full((n_cp, 2), 0.5)]; out_g = [_FEES[rng.integers(0, 3, n_cp)]]; out_k = [np.zeros(n_cp, np.uint8)]
    out_ar = [np.full(n_cp, 2)]; out_amp = [np.zeros(n_cp)]
    for x, k in enumerate(arities):
        mk = n_ss // len(arities) + (1 if x < n_ss % len(arities) else 0)
        if mk == 0:
            continue
        toks = np.argsort(rng.random((mk, n_stable)), 1)[:, :k]
        V = np.exp(9.0 + 1.5 * rng.standard_normal(mk))
        imb = np.exp(0.35 * rng.standard_normal((mk, k)))
        out_idx.append(toks)
        out_R.append(V[:, None] * imb / p[toks] * np.exp(mispricing * rng.standard_normal((mk, k))))
        out_w.append(rate[toks]); out_g.append(np.array([0.9996, 0.9999, 0.99995])[rng.integers(0, 3, mk)])
        out_k.append(np.full(mk, 4, np.uint8)); out_ar.append(np.full(mk, k))
        out_amp.append(np.array([100.0, 1000.0, 2e4])[rng.integers(0, 3, mk)] / float(k ** k))
    arity = np.concatenate(out_ar)
    return dict(
        n_tokens=n_tokens, prices=p,
        pool_ptr=np.concatenate([[0], np.cumsum(arity)]).astype(np.int64),
        tok_idx=np.concatenate([x.ravel() for x in out_idx]).astype(np.int32),
        reserves=np.concatenate([x.ravel() for x in out_R]),
        weights=np.concatenate([x.ravel() for x in out_w]),
        gamma=np.concatenate(out_g), kind=np.concatenate(out_k), amp=np.concatenate(out_amp),
    )


def synth_basket(n_tokens, prices, seed, n_assets=16, scale=1e-3, liq_mean=np.exp(8.0)):
    """cfg 4 basket: a_j = exp(N(0,1)) * Lbar / p_j * 1e-3 on 16 random tokens, target token 0."""
    rng = np.random.default_rng(seed)
    toks = rng.choice(np.arange(1, n_tokens), n_assets, replace=False)
    a = np.zeros(n_tokens)
    a[toks] = np.exp(rng.standard_normal(n_assets)) * liq_mean / prices[toks] * scale
    return a


# ------------------------------------------------------------------------------------------
# bounded-liquidity constant product (a Uniswap-v3 tick range) -- not in the reference: the first
# "more trading functions" extension behind the per-pool interface (SURVEY section 8f-4)
# ------------------------------------------------------------------------------------------
def v3_position(liquidity, p_lo, p_hi, p):
    """Real reserves and virtual-reserve offsets of a concentrated-liquidity position: liquidity L on the price range
    [p_lo, p_hi] (token-1 per token-0) at current price p.  Returns (reserves [x, y], offsets [o_x, o_y]) such that
    (x + o_x)(y + o_y) = L^2 is the position's curve and x, y >= 0 what it can actually pay out."""
    p = float(np.clip(p, p_lo, p_hi))
    sp, sa, sb = np.sqrt(p), np.sqrt(p_lo), np.sqrt(p_hi)
    return [liquidity * (1 / sp - 1 / sb), liquidity * (sp - sa)], [liquidity / sb, liquidity * sa]


def v3_instance():
    """3 tokens; two tick ranges of a v3 pool on (0, 1) (adjacent ranges: the upper one holds token 0 only), one
    in-range position on (0, 2), a constant-product pair (1, 2) and a weighted 3-token pool."""
    r_a, o_a = v3_position(100.0, 0.8, 1.25, 1.0)
    r_b, o_b = v3_position(80.0, 1.25, 1.6, 1.0)        # out of range: all in token 0
    r_c, o_c = v3_position(50.0, 1.9, 2.2, 2.0)
    return dict(
        n_tokens=3,
        local_indices=[[0, 1], [0, 1], [0, 2], [1, 2], [0, 1, 2]],
        reserves=[r_a, r_b, r_c, [30.0, 20.0], [10.0, 12.0, 8.0]],
        fees=[0.997, 0.997, 0.9995, 0.997, 0.99],
        kinds=["bounded_product", "bounded_product", "bounded_product", "product", "geomean"],
        weights=[o_a, o_b, o_c, None, [2, 1, 1]],
        market_value=[1.3, 1.0, 0.45],
    )


# ------------------------------------------------------------------------------------------
# concentrated liquidity: a whole Uniswap-v3 tick ladder as one pool (kind "concentrated")
# ------------------------------------------------------------------------------------------
def v3_ladder(sqrt_price_x96, ticks, liquidity_net, decimals0, decimals1):
    """On-chain state of a Uniswap-v3 pool -> the (price, bounds, liquidity) of HostPools.from_lists' 'concentrated' kind,
    in human token units (token 1 per token 0).  sqrt_price_x96: slot0's sqrtPriceX96; ticks: the initialised ticks
    (any order); liquidity_net: each tick's liquidityNet (ints, as the contract stores them); decimals0/1: the tokens'
    decimals.  price = (sqrt_price_x96 / 2^96)^2 10^(d0 - d1), bounds_k = 1.0001^tick_k 10^(d0 - d1) over the sorted
    ticks, and the liquidity of [tick_k, tick_{k+1}) = the running sum of liquidity_net up to tick k, times
    10^(-(d0 + d1) / 2).  Computed in 40-digit decimal and rounded once to f64."""
    from decimal import Decimal, localcontext
    order = np.argsort(np.asarray([int(t) for t in ticks], np.int64), kind="stable")
    tk = [int(ticks[i]) for i in order]
    net = [int(liquidity_net[i]) for i in order]
    if len(tk) < 2 or len(set(tk)) != len(tk):
        raise ValueError("v3_ladder needs at least two distinct initialised ticks")
    with localcontext() as ctx:
        ctx.prec = 40
        dd = Decimal(10) ** (int(decimals0) - int(decimals1))
        price = float(Decimal(int(sqrt_price_x96)) ** 2 / Decimal(2) ** 192 * dd)
        bounds = [float(Decimal("1.0001") ** t * dd) for t in tk]
        lscale = (Decimal(10) ** (-(int(decimals0) + int(decimals1)))).sqrt()
        run, liq = 0, []
        for x in net[:-1]:
            run += x
            if run < 0:
                raise ValueError("liquidity_net sums to a negative liquidity")
            liq.append(float(Decimal(run) * lscale))
    return price, bounds, liq


def ladder_ranges(hp):
    """The same market with every concentrated pool written as its non-empty intervals, one bounded_product pool each:
    the arithmetic of v3_position on the records' sqrt bounds (reserves L (1/s_k - 1/b_{k+1}), L (s_k - b_k) and offsets
    L / b_{k+1}, L b_k with s_k = s clamped to [b_k, b_{k+1}]).  In exact arithmetic the two forms trade the same: the
    ladder's trading set is the Minkowski sum of its intervals'.  Returns (HostPools, owner): owner[j] = the pool of hp
    that pool j of the result comes from (other kinds are copied, in order)."""
    from .pools import HostPools, KIND_BOUNDED_HOST, KIND_CONCENTRATED_HOST
    ptr = np.asarray(hp.pool_ptr, np.int64)
    lp = np.asarray(hp.lad_ptr, np.int64)
    rec = np.asarray(hp.lad_rec, np.float64).reshape(-1, 4)
    kind = np.asarray(hp.kind)
    cl = kind == KIND_CONCENTRATED_HOST
    # one entry per interval of every concentrated pool (the last record of each pool closes its ladder)
    nrec = np.diff(lp)
    owner_r = np.repeat(np.arange(hp.m), nrec)
    last = np.zeros(len(rec), bool); last[lp[1:][nrec > 0] - 1] = True
    iv = np.nonzero(~last & (rec[:, 1] > 0))[0]                      # non-empty intervals
    o_iv = owner_r[iv]
    L, b, b1 = rec[iv, 1], rec[iv, 0], rec[iv + 1, 0]
    sk = np.minimum(np.maximum(np.asarray(hp.lad_sc, float)[o_iv, 0], b), b1)
    Rr = np.stack([L * (1 / sk - 1 / b1), L * (sk - b)], 1)
    Or = np.stack([L / b1, L * b], 1)
    # pools of the result: every non-concentrated pool once, every concentrated pool as its intervals, in pool order
    keep = np.nonzero(~cl)[0]
    owner = np.concatenate([keep, o_iv])
    order = np.argsort(owner, kind="stable")
    owner = owner[order]
    ar = np.where(cl, 2, np.diff(ptr))[owner]
    new_ptr = np.concatenate([[0], np.cumsum(ar)]).astype(np.int64)
    src_k = np.concatenate([keep, np.full(len(iv), -1)])[order]      # pool copied as it is, or -1: an interval
    src_i = np.concatenate([np.full(len(keep), -1), np.arange(len(iv))])[order]
    n = int(new_ptr[-1])
    tok = np.zeros(n, np.int32); R = np.zeros(n); w = np.zeros(n)
    kd = kind[owner].copy()
    cp = src_k >= 0
    within = np.arange(int(ar[cp].sum())) - np.repeat(np.cumsum(ar[cp]) - ar[cp], ar[cp])     # slot index in its pool
    slots_new = np.repeat(new_ptr[:-1][cp], ar[cp]) + within
    slots_old = np.repeat(ptr[src_k[cp]], ar[cp]) + within
    tok[slots_new] = hp.tok_idx[slots_old]; R[slots_new] = hp.reserves[slots_old]; w[slots_new] = hp.weights[slots_old]
    rng_ = ~cp
    first = new_ptr[:-1][rng_]
    ii = src_i[rng_]
    tok[first] = hp.tok_idx[ptr[o_iv[ii]]]; tok[first + 1] = hp.tok_idx[ptr[o_iv[ii]] + 1]
    R[first], R[first + 1] = Rr[ii, 0], Rr[ii, 1]
    w[first], w[first + 1] = Or[ii, 0], Or[ii, 1]
    kd[rng_] = KIND_BOUNDED_HOST
    out = HostPools(hp.n_tokens, new_ptr, tok, R, w, np.asarray(hp.gamma, float)[owner], kd,
                    np.asarray(hp.amp, float)[owner], np.asarray(hp.inv, float)[owner])
    return out, owner


def synth_concentrated_market(m, n_tokens, seed, T=(1, 64), frac_ladder=0.5, empty=0.1, mispricing=0.02):
    """A market of concentrated pools (a tick ladder each) beside every other kind: m pools, a frac_ladder share of them
    ladders on random token pairs with T intervals (an int, or a (lo, hi) range drawn log-uniformly) of geometric width
    0.2 % .. 2 %, each empty with probability `empty`, the current price mispriced by `mispricing` and placed anywhere in
    the ladder, a few pools past either end; the rest is synth_stable_n_market's mix (constant product, two- to four-coin
    StableSwap) plus 5 % constant-sum pairs and 5 % bounded_product ranges.  Returns (HostPools, prices)."""
    from .pools import (HostPools, KIND_BOUNDED_HOST, KIND_CONCENTRATED_HOST, KIND_SUM_HOST, ladder_records,
                        ladder_state)
    rng = np.random.default_rng(seed)
    n_lad = int(round(frac_ladder * m))
    n_sum = n_bnd = (m - n_lad) // 10
    base = synth_stable_n_market(m - n_lad - n_sum - n_bnd, n_tokens, seed, mispricing=mispricing)
    p = base.pop("prices")
    ptr = [np.asarray(base["pool_ptr"], np.int64)]
    tok, R, w = [base["tok_idx"]], [base["reserves"]], [base["weights"]]
    g, kd, amp = [base["gamma"]], [base["kind"]], [base["amp"]]
    def pairs(k):
        a = rng.integers(0, n_tokens, k)
        return a, (a + rng.integers(1, n_tokens, k)) % n_tokens
    a, b = pairs(n_sum)                                                  # constant-sum pairs
    tok.append(np.stack([a, b], 1).ravel()); R.append(np.exp(6.0 + rng.standard_normal(2 * n_sum)))
    w.append(np.zeros(2 * n_sum)); g.append(_FEES[rng.integers(0, 3, n_sum)]); kd.append(np.full(n_sum, KIND_SUM_HOST))
    amp.append(np.zeros(n_sum))
    a, b = pairs(n_bnd)                                                  # single ranges
    Lb = np.exp(6.0 + rng.standard_normal(n_bnd))
    pr = p[a] / p[b] * np.exp(mispricing * rng.standard_normal(n_bnd))
    sp, sa, sb = np.sqrt(pr), np.sqrt(pr * 0.9), np.sqrt(pr * 1.1)
    tok.append(np.stack([a, b], 1).ravel()); R.append(np.stack([Lb * (1 / sp - 1 / sb), Lb * (sp - sa)], 1).ravel())
    w.append(np.stack([Lb / sb, Lb * sa], 1).ravel()); g.append(_FEES[rng.integers(0, 3, n_bnd)])
    kd.append(np.full(n_bnd, KIND_BOUNDED_HOST)); amp.append(np.zeros(n_bnd))
    # ladders
    if np.ndim(T) == 0:
        Ts = np.full(n_lad, int(T))
    else:
        Ts = np.exp(rng.uniform(np.log(T[0]), np.log(T[1] + 1), n_lad)).astype(np.int64).clip(T[0], T[1])
    a, b = pairs(n_lad)
    price = p[a] / p[b] * np.exp(mispricing * rng.standard_normal(n_lad))
    m0 = sum(len(x) for x in g)
    recs = [None] * n_lad
    for t in np.unique(Ts).tolist():
        sel = np.nonzero(Ts == t)[0]
        wd = np.exp(rng.uniform(np.log(0.002), np.log(0.02), len(sel)))
        lo = np.log(price[sel]) - wd * t * rng.uniform(-0.05, 1.05, len(sel))        # some prices past either end
        bounds = np.exp(lo[:, None] + wd[:, None] * np.arange(t + 1))
        liq = np.exp(7.0 + rng.standard_normal((len(sel), t))) * (rng.random((len(sel), t)) >= empty)
        liq[np.arange(len(sel)), rng.integers(0, t, len(sel))] = np.exp(7.0)            # never all empty
        for x, r in zip(sel.tolist(), ladder_records(bounds, liq)):
            recs[x] = r
    tok.append(np.stack([a, b], 1).ravel()); w.append(np.zeros(2 * n_lad))
    g.append(np.array([0.9995, 0.997, 0.99])[rng.integers(0, 3, n_lad)])
    kd.append(np.full(n_lad, KIND_CONCENTRATED_HOST)); amp.append(np.zeros(n_lad))
    M = m0 + n_lad
    ar = np.concatenate([np.diff(ptr[0]), np.full(n_sum + n_bnd + n_lad, 2)])
    lad_ptr = np.zeros(M + 1, np.int64)
    lad_ptr[m0 + 1:] = np.cumsum(Ts + 1)
    rec = np.concatenate(recs) if n_lad else np.zeros((0, 4))
    ids = np.arange(m0, M)
    s, c, x, y = ladder_state(lad_ptr, rec, ids, price)
    R.append(np.stack([x, y], 1).ravel())
    sc = np.zeros((M, 2)); sc[ids, 0], sc[ids, 1] = s, c
    hp = HostPools(n_tokens, np.concatenate([[0], np.cumsum(ar)]).astype(np.int64),
                   np.concatenate(tok).astype(np.int32), np.concatenate(R), np.concatenate(w), np.concatenate(g),
                   np.concatenate(kd).astype(np.uint8), np.concatenate(amp), None, lad_ptr, rec, sc)
    return hp, p


TWOCRYPTO_A_MULTIPLIER = 10000      # twocrypto-ng stores A() = A * N^N * A_MULTIPLIER (N = 2), gamma() as 1e18 fixed point


def twocrypto_pool(A_raw, gamma_raw, price_scale, precisions, balances, mid_fee, out_fee, fee_gamma):
    """A two-coin Curve v2 (twocrypto-ng) pool's on-chain state as this package's 'cryptoswap' pool.
    A_raw = A(), gamma_raw = gamma() (1e18 fixed point), price_scale = price_scale() (coin 1 in coin 0, 1e18 fixed point),
    precisions = the contract's (10^(18 - decimals_0), 10^(18 - decimals_1)), balances = balances(0), balances(1) (raw
    integers), mid_fee / out_fee (1e10 fixed point) and fee_gamma (1e18).  Returns (weights, reserves, gamma): weights =
    (A, G, p_0, p_1) for HostPools.from_lists, reserves in whole tokens (balance * precision / 1e18) and the fee gamma
    = 1 - fee at the current state, fee = mid_fee f + out_fee (1 - f), f = fee_gamma / (fee_gamma + 1 - K0),
    K0 = 4 y0 y1 / (y0 + y1)^2 with y = p * reserves.  The contract charges that fee on the output and moves it with the
    trade, so this gamma is the pool's fee for small trades only (as for StableSwap pools, instances give the caller's
    conversion).  A = A_raw / (A_MULTIPLIER * 2^2) and G = gamma_raw / 1e18: the convention of the contract's comments
    (A_MULTIPLIER = 10000, A() scaled by N^N); it has not been checked against the contract's integer newton_D (see
    INTEGRATION.md)."""
    A = float(A_raw) / (TWOCRYPTO_A_MULTIPLIER * 4)
    G = float(gamma_raw) / 1e18
    x = np.array([float(balances[0]) * float(precisions[0]), float(balances[1]) * float(precisions[1])]) / 1e18
    p = np.array([1.0, float(price_scale) / 1e18])
    y = p * x
    K0 = 4.0 * y[0] * y[1] / (y[0] + y[1]) ** 2
    fg = float(fee_gamma) / 1e18
    f = fg / (fg + 1.0 - K0)
    fee = (float(mid_fee) * f + float(out_fee) * (1.0 - f)) / 1e10
    return (A, G, float(p[0]), float(p[1])), (float(x[0]), float(x[1])), 1.0 - fee


def synth_crypto_market(m, n_tokens, seed, frac_crypto=0.4, far=0.5, mispricing=0.02, T=(1, 16)):
    """A market of two-coin cryptoswap pools beside every other kind: a frac_crypto share of m pools are cryptoswap pools
    on random token pairs (A in {2.5 .. 400}, curve gamma in {1e-5 .. 2e-2}, fees 0.05 .. 0.45 %), value-balanced within a
    few percent; the price scale of a `far` share of them sits 20 % .. 4x away from the market price (the pool holds
    balances far from its peg), the others within 0.5 % of it.  The rest is synth_concentrated_market's mix (constant
    product, two- to four-coin StableSwap, constant sum, bounded_product ranges, tick ladders of T intervals).
    Returns (HostPools, prices)."""
    from .pools import HostPools, KIND_CRYPTOSWAP_HOST
    rng = np.random.default_rng(seed + 7919)
    n_cs = int(round(frac_crypto * m))
    base, p = synth_concentrated_market(m - n_cs, n_tokens, seed, T=T, mispricing=mispricing)
    a = rng.integers(0, n_tokens, n_cs)
    b = (a + rng.integers(1, n_tokens, n_cs)) % n_tokens
    off = rng.random(n_cs) < far
    sh = np.where(off, np.exp(rng.choice([-1.0, 1.0], n_cs) * rng.uniform(np.log(1.2), np.log(4.0), n_cs)),
                  np.exp(rng.uniform(-0.005, 0.005, n_cs)))
    scales = np.stack([p[a], p[b] * sh], 1)                      # the pool's internal price of b in a is off by sh
    V = np.exp(9.0 + 1.5 * rng.standard_normal(n_cs))
    R = V[:, None] / scales * np.exp(mispricing * rng.standard_normal((n_cs, 2)))
    A = np.array([2.5, 10.0, 40.0, 400.0])[rng.integers(0, 4, n_cs)]
    G = np.array([1e-5, 1.45e-4, 2e-3, 2e-2])[rng.integers(0, 4, n_cs)]
    gam = np.array([0.9995, 0.9974, 0.9955])[rng.integers(0, 3, n_cs)]
    m0 = base.m
    cg = np.concatenate([np.asarray(base.cgam, float), G])
    hp = HostPools(n_tokens, np.concatenate([base.pool_ptr, base.pool_ptr[-1] + 2 * np.arange(1, n_cs + 1)]).astype(np.int64),
                   np.concatenate([base.tok_idx, np.stack([a, b], 1).ravel()]).astype(np.int32),
                   np.concatenate([base.reserves, R.ravel()]), np.concatenate([base.weights, scales.ravel()]),
                   np.concatenate([base.gamma, gam]),
                   np.concatenate([base.kind, np.full(n_cs, KIND_CRYPTOSWAP_HOST, np.uint8)]).astype(np.uint8),
                   np.concatenate([base.amp, A]), None,
                   np.concatenate([base.lad_ptr, np.full(n_cs, base.lad_ptr[-1], np.int64)]), base.lad_rec,
                   np.concatenate([base.lad_sc, np.zeros((n_cs, 2))]), cg)
    assert hp.m == m0 + n_cs
    return hp, p


TRICRYPTO_A_MULTIPLIER = 10000      # tricrypto-ng stores A() = A * N^N * A_MULTIPLIER (N = 3), gamma() as 1e18 fixed point


def tricrypto_pool(A_raw, gamma_raw, price_scale, precisions, balances, mid_fee, out_fee, fee_gamma):
    """A three-coin Curve v2 (tricrypto-ng) pool's on-chain state as this package's three-token 'cryptoswap' pool.
    A_raw = A(), gamma_raw = gamma() (1e18 fixed point), price_scale = (price_scale(0), price_scale(1)) (coins 1 and 2 in
    coin 0, 1e18 fixed point), precisions = the contract's 10^(18 - decimals_j), balances = balances(0..2) (raw integers),
    mid_fee / out_fee (1e10 fixed point) and fee_gamma (1e18).  Returns (weights, reserves, gamma): weights =
    (A, G, p_0, p_1, p_2) for HostPools.from_lists, reserves in whole tokens (balance * precision / 1e18) and the fee
    gamma = 1 - fee at the current state, fee = mid_fee f + out_fee (1 - f), f = fee_gamma / (fee_gamma + 1 - K0),
    K0 = 27 y0 y1 y2 / (y0 + y1 + y2)^3 with y = p * reserves (the contract's fee is charged on the output and moves with
    the trade, so this gamma is the pool's fee for small trades only, as for twocrypto_pool).  A = A_raw /
    (A_MULTIPLIER * 3^3) and G = gamma_raw / 1e18: the convention of the contract's comments; it has not been checked
    against the contract's integer newton_D (see INTEGRATION.md)."""
    A = float(A_raw) / (TRICRYPTO_A_MULTIPLIER * 27)
    G = float(gamma_raw) / 1e18
    x = np.array([float(balances[j]) * float(precisions[j]) for j in range(3)]) / 1e18
    p = np.array([1.0, float(price_scale[0]) / 1e18, float(price_scale[1]) / 1e18])
    y = p * x
    K0 = 27.0 * y[0] * y[1] * y[2] / y.sum() ** 3
    fg = float(fee_gamma) / 1e18
    f = fg / (fg + 1.0 - K0)
    fee = (float(mid_fee) * f + float(out_fee) * (1.0 - f)) / 1e10
    return (A, G, float(p[0]), float(p[1]), float(p[2])), tuple(float(v) for v in x), 1.0 - fee


def synth_tricrypto_market(m, n_tokens, seed, frac_tri=0.3, far=0.5, mispricing=0.02, T=(1, 16)):
    """A market of three-coin cryptoswap pools beside every other kind: a frac_tri share of m pools are tricrypto pools
    on random token triples (A in {0.1 .. 50}, curve gamma in {1e-5 .. 2e-2}, fees 0.05 .. 0.45 %), value-balanced within
    a few percent; the price scales of a `far` share of them sit 20 % .. 4x away from the market prices, the others within
    0.5 %.  The rest is synth_crypto_market's mix (two-coin cryptoswap, constant product, StableSwap, constant sum,
    ranges and ladders).  n_tokens >= 3.  Returns (HostPools, prices)."""
    from .pools import HostPools, KIND_CRYPTOSWAP_HOST
    rng = np.random.default_rng(seed + 104729)
    n_t = int(round(frac_tri * m))
    base, p = synth_crypto_market(m - n_t, n_tokens, seed, mispricing=mispricing, T=T)
    tri = np.stack([rng.choice(n_tokens, 3, replace=False) for _ in range(n_t)]) if n_t else np.zeros((0, 3), int)
    off = rng.random(n_t) < far
    sh = np.where(off[:, None], np.exp(rng.choice([-1.0, 1.0], (n_t, 3)) * rng.uniform(np.log(1.2), np.log(4.0), (n_t, 3))),
                  np.exp(rng.uniform(-0.005, 0.005, (n_t, 3))))
    sh[:, 0] = 1.0
    scales = p[tri] * sh                                         # the pool's internal prices are off by sh
    V = np.exp(9.0 + 1.5 * rng.standard_normal(n_t))
    R = V[:, None] / scales * np.exp(mispricing * rng.standard_normal((n_t, 3)))
    A = np.array([0.1, 1.0, 6.3, 50.0])[rng.integers(0, 4, n_t)]
    G = np.array([1e-5, 1.45e-4, 2e-3, 2e-2])[rng.integers(0, 4, n_t)]
    gam = np.array([0.9995, 0.9974, 0.9955])[rng.integers(0, 3, n_t)]
    hp = HostPools(n_tokens, np.concatenate([base.pool_ptr, base.pool_ptr[-1] + 3 * np.arange(1, n_t + 1)]).astype(np.int64),
                   np.concatenate([base.tok_idx, tri.ravel()]).astype(np.int32),
                   np.concatenate([base.reserves, R.ravel()]), np.concatenate([base.weights, scales.ravel()]),
                   np.concatenate([base.gamma, gam]),
                   np.concatenate([base.kind, np.full(n_t, KIND_CRYPTOSWAP_HOST, np.uint8)]).astype(np.uint8),
                   np.concatenate([base.amp, A]), None,
                   np.concatenate([base.lad_ptr, np.full(n_t, base.lad_ptr[-1], np.int64)]), base.lad_rec,
                   np.concatenate([base.lad_sc, np.zeros((n_t, 2))]), np.concatenate([np.asarray(base.cgam, float), G]))
    return hp, p


LB_ID_OFFSET = 1 << 23      # Liquidity Book's bin id of price 1 (raw units)


def lb_bins(active_id, bin_step, ids, reserves_x, reserves_y, decimals_x, decimals_y):
    """A Liquidity Book (LFJ / Trader Joe v2.x) pair's bins as the (prices, x, y) of HostPools.from_lists' 'bins' kind:
    bin id k trades at (1 + bin_step / 1e4)^(k - 2^23) raw Y per raw X, so at (1 + bin_step / 1e4)^(k - 2^23) *
    10^(decimals_x - decimals_y) token Y per token X, computed in 40-digit decimal and rounded once; holdings are the raw
    reserves over 10^decimals.  Token X is the pool's token 0.  Bins above active_id must hold no Y and bins below it no
    X (ValueError otherwise); the rules of from_lists apply to the result.  The fee is the caller's (LB's variable and
    composition fees are not modelled)."""
    import decimal
    ids = np.asarray(ids, np.int64).reshape(-1)
    rx, ry = np.asarray(reserves_x, object).reshape(-1), np.asarray(reserves_y, object).reshape(-1)
    if not (len(ids) == len(rx) == len(ry)) or len(ids) == 0:
        raise ValueError("lb_bins: one reserve of each token per bin id")
    if not 1 <= int(bin_step) <= 10000:
        raise ValueError("lb_bins: bin_step must be 1 .. 10000 basis points")
    o = np.argsort(ids, kind="stable")
    ids, rx, ry = ids[o], rx[o], ry[o]
    if np.any(np.diff(ids) <= 0):
        raise ValueError("lb_bins: bin ids must be distinct")
    if any(int(v) < 0 for v in rx) or any(int(v) < 0 for v in ry):
        raise ValueError("lb_bins: reserves must be >= 0")
    if any(int(rx[k]) > 0 for k in np.nonzero(ids < active_id)[0]) or \
            any(int(ry[k]) > 0 for k in np.nonzero(ids > active_id)[0]):
        raise ValueError("lb_bins: bins below the active one hold only Y, bins above it only X")
    with decimal.localcontext() as ctx:
        ctx.prec = 40
        D = decimal.Decimal
        base = D(1) + D(int(bin_step)) / D(10000)
        scale = D(10) ** (int(decimals_x) - int(decimals_y))
        prices = np.array([float(base ** (int(k) - LB_ID_OFFSET) * scale) for k in ids.tolist()])
        x = np.array([float(D(int(v)) / D(10) ** int(decimals_x)) for v in rx])
        y = np.array([float(D(int(v)) / D(10) ** int(decimals_y)) for v in ry])
    return prices, x, y


def order_book(bids, asks):
    """An order book (or a batch of limit orders) as the (prices, x, y) of HostPools.from_lists' 'bins' kind: bids and
    asks are (price, size) levels, price in token 1 per token 0, size in token 0.  An ask is a bin holding x = size at
    its price; a bid one holding y = price * size; equal prices merge (a bid and an ask at the same price share a bin).
    A crossed book (a bid above an ask) raises ValueError."""
    lv = {}
    for side, levels in ((1, bids), (0, asks)):
        for pr, sz in levels:
            pr, sz = float(pr), float(sz)
            if not (np.isfinite(pr) and pr > 0 and np.isfinite(sz) and sz >= 0):
                raise ValueError("order_book: prices must be finite and > 0, sizes finite and >= 0")
            e = lv.setdefault(pr, [0.0, 0.0])
            e[side] += pr * sz if side else sz
    if not lv:
        raise ValueError("order_book: no levels")
    prices = np.array(sorted(lv))
    x = np.array([lv[p][0] for p in prices]); y = np.array([lv[p][1] for p in prices])
    if x.any() and y.any() and prices[y > 0].max() > prices[x > 0].min():
        raise ValueError("order_book: the book is crossed (a bid above an ask)")
    return prices, x, y


def bins_split(hp):
    """The same market with every bins pool written as its bins, one one-bin 'bins' pool each (the active bin keeps both
    holdings) at the pool's fee, holdings read back from the records (x = the width of an ask segment, y = minus the
    rise of C over a bid segment).  In exact arithmetic the two forms trade the same: a bins pool's trading set is the
    Minkowski sum of its bins'.  The other pools keep their order and come first, the one-bin pools follow in pool and
    price order.  Returns (HostPools, owner): owner[j] = the pool of hp that pool j of the result comes from."""
    from .pools import HostPools, KIND_BINS_HOST
    kind = np.asarray(hp.kind)
    ptr = np.asarray(hp.pool_ptr, np.int64)
    bn = kind == KIND_BINS_HOST
    keep = np.nonzero(~bn)[0]
    ar = np.diff(ptr)
    slots = np.repeat(ptr[keep], ar[keep]) + (np.arange(int(ar[keep].sum())) - np.repeat(
        np.concatenate([[0], np.cumsum(ar[keep])[:-1]]), ar[keep])) if len(keep) else np.zeros(0, np.int64)
    bp = np.asarray(hp.bin_ptr, np.int64)
    rec = np.asarray(hp.bin_rec, np.float64).reshape(-1, 4)
    cnt = np.diff(bp)
    owner_r = np.repeat(np.arange(hp.m), cnt)
    last = np.zeros(len(rec), bool); last[bp[1:][cnt > 0] - 1] = True
    seg = np.nonzero(~last)[0]                                       # every segment of every bins pool
    o = owner_r[seg]
    ask = (seg - bp[o]) >= np.asarray(hp.bin_zp, float)[o, 0]
    x = np.where(ask, rec[seg + 1, 0] - rec[seg, 0], 0.0)
    y = np.where(ask, 0.0, rec[seg + 1, 1] - rec[seg, 1])
    new = np.ones(len(seg), bool)                                    # the active bin's two segments become one pool
    new[1:] = (o[1:] != o[:-1]) | (rec[seg[1:], 3] != rec[seg[:-1], 3])
    gid = np.cumsum(new) - 1
    ng = int(gid[-1]) + 1 if len(seg) else 0
    xg, yg = np.bincount(gid, x, ng), np.bincount(gid, y, ng)
    first = seg[new]
    og, pg, bg = o[new], rec[first, 2], rec[first, 3]
    hy, hx = yg > 0, xg > 0
    nrec = 2 + (hx & hy)
    st = np.concatenate([[0], np.cumsum(nrec)[:-1]]).astype(np.int64)
    zg = hy.astype(np.int64)
    out_rec = np.zeros((int(nrec.sum()), 4))
    out_rec[st[hy]] = np.stack([-yg[hy] / pg[hy], -yg[hy], pg[hy], bg[hy]], 1)
    out_rec[st + zg, 2] = np.where(hx, pg, 0.0)
    out_rec[st + zg, 3] = np.where(hx, bg, -1.0)
    out_rec[st[hx] + zg[hx] + 1] = np.stack([xg[hx], pg[hx] * xg[hx], np.zeros(hx.sum()), np.full(hx.sum(), -1.0)], 1)
    M = len(keep) + ng
    new_ar = np.concatenate([ar[keep], np.full(ng, 2)])
    lad_ptr = np.concatenate([np.asarray(hp.lad_ptr, np.int64)[keep], np.full(ng + 1, np.asarray(hp.lad_ptr)[-1])])
    bin_ptr = np.zeros(M + 1, np.int64); bin_ptr[len(keep) + 1:] = np.cumsum(nrec)
    bin_zp = np.zeros((M, 2)); bin_zp[len(keep):, 0], bin_zp[len(keep):, 1] = zg, pg
    tok = np.asarray(hp.tok_idx)
    out = HostPools(hp.n_tokens, np.concatenate([[0], np.cumsum(new_ar)]).astype(np.int64),
                    np.concatenate([tok[slots], np.stack([tok[ptr[og]], tok[ptr[og] + 1]], 1).ravel()]).astype(np.int32),
                    np.concatenate([np.asarray(hp.reserves)[slots], np.stack([xg, yg], 1).ravel()]),
                    np.concatenate([np.asarray(hp.weights)[slots], np.zeros(2 * ng)]),
                    np.concatenate([np.asarray(hp.gamma)[keep], np.asarray(hp.gamma)[og]]),
                    np.concatenate([kind[keep], np.full(ng, KIND_BINS_HOST)]).astype(np.uint8),
                    np.concatenate([np.asarray(hp.amp)[keep], np.zeros(ng)]),
                    np.concatenate([np.asarray(hp.inv)[keep], np.zeros(ng)]),
                    lad_ptr, hp.lad_rec, np.concatenate([np.asarray(hp.lad_sc).reshape(-1, 2)[keep], np.zeros((ng, 2))]),
                    np.concatenate([np.asarray(hp.cgam)[keep], np.zeros(ng)]), bin_ptr, out_rec, bin_zp)
    return out, np.concatenate([keep, og]).astype(np.int64)


def synth_bins_market(m, n_tokens, seed, K=(1, 256), frac_lb=0.3, frac_book=0.1, frac_order=0.1, mispricing=0.02):
    """A market of price-bin pools beside constant-product pools: m pools, a frac_lb share Liquidity-Book-like pools on
    bin steps of 1 .. 100 bp with K bins (an int, or a (lo, hi) range drawn log-uniformly) around an active bin that
    holds both tokens, their liquidity shaped like a bell around it (spot) or flat (a wide range); a frac_book share
    order books (a spread of 2 .. 20 bp around the mid, K levels split between the sides, sizes log-normal); a
    frac_order share single limit orders (one bin holding one token, at up to 1 % through the price, fee 1); the rest
    constant product.  The mid of every bins pool is mispriced by `mispricing`.  Returns (HostPools, prices)."""
    from .pools import HostPools, KIND_BINS_HOST, KIND_GEOMEAN_HOST, bin_records
    rng = np.random.default_rng(seed)
    n_lb, n_book, n_ord = (int(round(f * m)) for f in (frac_lb, frac_book, frac_order))
    n_bins = n_lb + n_book + n_ord
    base = synth_const_product(m - n_bins, n_tokens, seed, mispricing=mispricing)
    p = base["prices"]
    a = rng.integers(0, n_tokens, n_bins)
    b = (a + rng.integers(1, n_tokens, n_bins)) % n_tokens
    mid = p[a] / p[b] * np.exp(mispricing * rng.standard_normal(n_bins))
    if np.ndim(K) == 0:
        Ks = np.full(n_bins, int(K))
    else:
        Ks = np.exp(rng.uniform(np.log(K[0]), np.log(K[1] + 1), n_bins)).astype(np.int64).clip(K[0], K[1])
    value = np.exp(8.0 + 1.5 * rng.standard_normal(n_bins)) / p[b]      # pool depth in token 1
    recs, zp, R, g = [], [], [], []
    for q in range(n_bins):
        k = int(Ks[q])
        if q < n_lb:                                   # Liquidity Book: bins around the active one
            step = float(rng.choice([1, 2, 5, 10, 15, 20, 25, 50, 100])) * 1e-4
            act = int(rng.integers(0, k))
            off = np.arange(k) - act
            prices = mid[q] * (1 + step) ** off
            shape = np.exp(-0.5 * (off / max(k / 6, 1.0)) ** 2) if rng.random() < 0.7 else np.ones(k)
            v = value[q] * shape / shape.sum()
            x = np.where(off > 0, v / prices, 0.0); y = np.where(off < 0, v, 0.0)
            share = rng.uniform(0.05, 0.95)
            x[act], y[act] = share * v[act] / prices[act], (1 - share) * v[act]
            fee = float(rng.choice([0.9999, 0.9995, 0.998]))
        elif q < n_lb + n_book:                        # order book: k levels split between bids and asks
            spread = rng.uniform(2e-4, 2e-3)
            nb = int(rng.integers(0, k + 1)) if k > 1 else int(rng.integers(0, 2))
            na = k - nb
            tick = rng.uniform(1e-4, 1e-3)
            bp_ = mid[q] * (1 - spread / 2) * (1 - tick) ** np.arange(nb)
            ap_ = mid[q] * (1 + spread / 2) * (1 + tick) ** np.arange(na)
            sz = value[q] / mid[q] * np.exp(rng.standard_normal(k)) / k
            prices = np.concatenate([bp_[::-1], ap_])
            x = np.concatenate([np.zeros(nb), sz[nb:]]); y = np.concatenate([bp_[::-1] * sz[:nb][::-1], np.zeros(na)])
            fee = 1.0
        else:                                          # one limit order, at up to 1 % through the mid
            sell = rng.random() < 0.5
            prices = np.array([mid[q] * (1 + (rng.uniform(-0.01, 0.01)))])
            sz = value[q] / mid[q] * np.exp(rng.standard_normal()) * 0.1
            x = np.array([sz if sell else 0.0]); y = np.array([0.0 if sell else prices[0] * sz])
            fee = 1.0
        r, z, pref, sums = bin_records(prices, x, y)
        recs.append(r); zp.append((z, pref)); R += list(sums); g.append(fee)
    m0 = m - n_bins
    M = m
    bin_ptr = np.zeros(M + 1, np.int64)
    bin_ptr[m0 + 1:] = np.cumsum([len(r) for r in recs])
    bin_zp = np.zeros((M, 2)); bin_zp[m0:] = np.asarray(zp).reshape(-1, 2)
    hp = HostPools(n_tokens, np.arange(0, 2 * M + 1, 2, dtype=np.int64),
                   np.concatenate([base["idx"].ravel(), np.stack([a, b], 1).ravel()]).astype(np.int32),
                   np.concatenate([base["reserves"].ravel(), R]),
                   np.concatenate([np.full(2 * m0, 0.5), np.zeros(2 * n_bins)]),
                   np.concatenate([base["gamma"], g]),
                   np.concatenate([np.full(m0, KIND_GEOMEAN_HOST), np.full(n_bins, KIND_BINS_HOST)]).astype(np.uint8),
                   None, None, None, None, None, None, bin_ptr, np.concatenate(recs) if recs else None, bin_zp)
    return hp, p


def bins_event(rng, triple, what=None, k_max=256):
    """One block's change of a price-bin pool given as its (prices, x, y), as the new triple (the rules of
    HostPools.from_lists hold for it): what = 'swap' (a Liquidity Book swap empties the active bin and moves it one to
    three bins: the top bids turn into asks at their prices, or the bottom asks into bids), 'deposit' (one to four bins
    added past an end, K grows up to k_max), 'withdraw' (one to four bins at an end removed, K shrinks, at least one
    bin with holdings stays), 'book' (order-book levels change: the mid moves through one to four ask or bid levels, which
    are taken and reposted on the other side at the same prices, a new level appears past the far end, and every size
    moves by a few percent) or 'fill' (a partial fill of the one-bin limit order: a share of its holding turns into the
    other token at its price; another pool gets a swap); None: one drawn at random."""
    p, x, y = (np.asarray(v, np.float64).reshape(-1).copy() for v in triple)
    what = what or rng.choice(["swap", "deposit", "withdraw", "book", "fill"])
    K = len(p)
    if what == "fill" and K == 1:
        f = rng.uniform(0.1, 0.9)
        if x[0] > 0:
            x[0], y[0] = x[0] * (1 - f), y[0] + p[0] * x[0] * f
        else:
            y[0], x[0] = y[0] * (1 - f), x[0] + y[0] / p[0] * f
        return p, x, y
    if what in ("swap", "fill", "book"):
        s = int(rng.integers(1, 4 if what != "book" else 5))
        down = (rng.random() < 0.5 and y.any()) or not x.any()
        if down:                                       # token 0 sold into the pool: the top bids become asks
            j = np.nonzero(y > 0)[0][::-1][:s]
            x[j] += y[j] / p[j]; y[j] = 0.0
        else:                                          # token 0 bought from the pool: the bottom asks become bids
            j = np.nonzero(x > 0)[0][:s]
            y[j] += x[j] * p[j]; x[j] = 0.0
        if what != "book":
            return p, x, y
        x *= np.exp(0.05 * rng.standard_normal(K)); y *= np.exp(0.05 * rng.standard_normal(K))
        what = "deposit"                               # and a new level past the far end
    step = float(np.exp(np.mean(np.log(p[1:] / p[:-1])))) if K > 1 else 1.001
    if what == "deposit" and K < k_max:
        n = int(min(rng.integers(1, 5), k_max - K))
        v = float(np.sum(x * p + y)) / max(K, 1)
        if rng.random() < 0.5:                         # new asks above
            q = p[-1] * step ** np.arange(1, n + 1)
            return np.r_[p, q], np.r_[x, v / q], np.r_[y, np.zeros(n)]
        q = p[0] * step ** -np.arange(n, 0, -1)         # new bids below
        return np.r_[q, p], np.r_[np.zeros(n), x], np.r_[np.full(n, v), y]
    if K > 1:                                          # withdraw (or a deposit past k_max): bins at one end go
        n = int(min(rng.integers(1, 5), K - 1))
        keep = slice(n, K) if rng.random() < 0.5 else slice(0, K - n)
        if (x[keep] > 0).any() or (y[keep] > 0).any():
            return p[keep], x[keep], y[keep]
    return p, x, y
