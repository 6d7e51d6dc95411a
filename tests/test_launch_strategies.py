"""Every plain-bucket evaluation and Hessian-product kernel under every launch strategy cfmm_arb_eval / cfmm_hvp can
pick, forced through cfmm_set_scatter_mode.  GPU (H100) only.

The launchers sum the per-pool results into psi / arb / y in one of three ways: a privatised n_tokens histogram in
shared memory flushed once per CTA (mode 2), red.add.f64 straight to global memory (mode 1), or, for constant-product
and constant-sum buckets, the TMA-staged kernel (mode 3).  In auto mode (0) the choice follows the instance's shape, so
a kernel test of one shape only ever runs one of them.  Here each instance runs under each strategy, and each cell
checks:

(a) per pool, delta / lambda / hcoef / hmask of the shared-scatter instance equal the global-scatter instance's bit for
    bit: both call the same per-pool device function, only the scatter differs.  The TMA kernel is a different body
    around the same product_pool / sum_order: the compiler may contract its products into FMAs differently, so it may
    differ from the LDG kernel by rounding, at most 2 ulp per entry.
(b) psi and arb equal the exactly rounded sums (math.fsum) of the kernel's own per-pool flows, plus the values the
    buffers held before the launch (every kernel adds), within 2 k_j u gross_j per token: k_j contributions summed in
    any order err by at most (k_j - 1) u gross_j.  Runs without trades are checked against the flows of the run with
    them.
(c) hvp, hess_diag and hess_dense against the pool decomposition of the kernel's own hcoef / hmask, summed in long
    double: the pair branch, xp_stableswap_n.hess_block for n-coin StableSwap, the three edge weights of three-coin
    cryptoswap and the weighted branch of geometric-mean pools.  Each pool's contribution carries a few u of its own
    terms' magnitude on top of the summation bound.
(d) on a fixed sample of at most 500 pools per cell, the flows against the kind's extended-precision reference within
    that kind's existing bound (the flow_bound / flow_tol / ladder_tol / _check_against_xp helpers of its test module;
    1e-12 of the pool's reserve scale for the closed-form kinds, as tests/test_gpu_parity.py).  With (a) this extends
    the full-instance reference checks of those modules to the strategy their shapes do not pick.

Then the shapes where scatter kernels go wrong: buckets of 0, 1, 255, 256 and 257 pools, 2 .. 12289 tokens (12288 is
a 96 KB histogram, the largest the shared instance takes; at 12289 mode 2 takes global scatter), every pool on token 0
and some on token n - 1, grids whose CTAs loop, TMA tiles, and buckets the TMA kernel must not take.
"""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib, instances as I
from cfmm_routing_code_b200.pools import HostPools, KIND_BOUNDED_HOST, KIND_GEOMEAN_HOST, KIND_SUM_HOST
import xp_concentrated as XC
import xp_bins as XB
import xp_reference as X
import xp_stableswap as XS
import xp_stableswap_n as XN
import test_bins as TB
import test_concentrated as TCL
import test_cryptoswap as TC
import test_stableswap as TS
import test_stableswap_n as TN
import test_tricrypto as TT

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
AUTO, GLOBAL, SHARED, TMA = 0, 1, 2, 3
CFMM_E_KIND = -2
FLAGS = [(False, False), (True, False), (False, True), (True, True)]
F64 = dict(dtype=torch.float64, device="cuda")
SAMPLE = 500
MASKED = (_lib.KIND_STABLESWAP_N, _lib.KIND_CRYPTOSWAP_3, _lib.KIND_GEOMEAN)     # kinds whose kernels write hmask


@pytest.fixture
def scatter_mode():
    """a setter for the process-wide launch strategy; always back to auto afterwards, so that no later test runs an
    instance other than the one its shape picks"""
    lib = _lib.load()
    assert lib.cfmm_set_scatter_mode(4) == CFMM_E_KIND
    assert lib.cfmm_set_scatter_mode(-1) == CFMM_E_KIND

    def set_mode(mode):
        _lib.check(lib.cfmm_set_scatter_mode(mode), "cfmm_set_scatter_mode")
    try:
        yield set_mode
    finally:
        lib.cfmm_set_scatter_mode(AUTO)


# ====================================================================================================== instances
def _rows(x, k):
    return np.asarray(x).reshape(-1, k)


def _csr(n, toks, R, W, g, kind, **kw):
    m, k = toks.shape
    return HostPools(int(n), np.arange(0, k * m + 1, k, dtype=np.int64), np.ascontiguousarray(toks, np.int32).ravel(),
                     np.ascontiguousarray(R, np.float64).ravel(), np.ascontiguousarray(W, np.float64).ravel(),
                     np.ascontiguousarray(g, np.float64), np.full(m, kind, np.uint8), **kw)


def _pairs(m, n, rng):
    a = rng.integers(0, n, m)
    return np.stack([a, (a + rng.integers(1, n, m)) % n], 1)


def _product(m=50_000, seed=1):
    s = I.synth_const_product(m, 64, seed=seed)
    hp = HostPools.from_pairs(64, s["idx"], s["reserves"], s["gamma"])
    return hp, s["prices"] * np.exp(0.01 * np.random.default_rng(seed).standard_normal(64))


def _sum(m=50_000, seed=2):
    """constant-sum pairs with prices on both sides of the fill switch gamma nu_b = nu_a"""
    rng = np.random.default_rng(seed)
    toks = _pairs(m, 64, rng)
    nu = np.exp(rng.normal(0, 0.01, 64))
    R = np.exp(rng.normal(6, 2, (m, 2)))
    g = np.array([1.0, 0.9995, 0.997, 0.99])[rng.integers(0, 4, m)]
    return _csr(64, toks, R, np.full((m, 2), 0.5), g, KIND_SUM_HOST), nu


def _bounded(m=50_000, seed=3):
    """constant product on virtual reserves R + o: uncapped trades, trades capped at R, and o = 0"""
    rng = np.random.default_rng(seed)
    toks = _pairs(m, 64, rng)
    nu = np.exp(rng.normal(0, 0.3, 64))
    V = np.exp(rng.normal(8, 2, m))
    R = V[:, None] / nu[toks] * np.exp(rng.normal(0, 0.05, (m, 2)))
    o = R * np.exp(rng.normal(1, 2, (m, 2))) * (rng.random((m, 2)) < 0.9)
    g = np.array([1.0, 0.997, 0.99])[rng.integers(0, 3, m)]
    return _csr(64, toks, R, o, g, KIND_BOUNDED_HOST), nu


def _geomean(k, m=40_000, seed=4):
    """weighted pools of k coins on 64 tokens, reserves in balance with the prices up to ~2 %: inside the no-trade band,
    at its edges and outside it, some slots trading and others idle"""
    rng = np.random.default_rng(seed + k)
    toks = np.argsort(rng.random((m, 64)), 1)[:, :k]
    nu = np.exp(rng.normal(0, 0.5, 64))
    w = rng.dirichlet(np.ones(k), m)
    R = np.exp(rng.normal(8, 2, m))[:, None] * w / nu[toks] * np.exp(rng.normal(0, 0.02, (m, k)))
    g = np.array([1.0, 0.997, 0.99, 0.9])[rng.integers(0, 4, m)]
    return _csr(64, toks, R, w, g, KIND_GEOMEAN_HOST), nu


def _crypto(m=50_000, seed=21):
    hp, nu, _ = TC._bucket_pools(m, seed)
    return hp, nu


def _tricrypto(m=30_000, seed=21):
    """tests/test_tricrypto.py's bucket of random_pools on random triples of 64 tokens, at 30k pools"""
    rng = np.random.default_rng(seed)
    R0, p0, A, G, _, g, _ = TT.random_pools(m, seed)
    toks = np.stack([rng.choice(64, 3, replace=False) for _ in range(1000)])[rng.integers(0, 1000, m)]
    nu = np.exp(rng.normal(0, 0.3, 64))
    k = R0 * p0 / (R0 * p0).sum(1, keepdims=True)
    p = nu[toks] * np.exp(rng.normal(0, 0.02, (m, 3)))
    R = k * np.exp(rng.normal(8, 2, m))[:, None] / p
    return TT.tri_hp(R, p, A, G, g, toks, 64), nu


def _concentrated(m=20_000, seed=21):
    hp, prices = I.synth_concentrated_market(m, 64, seed=seed, T=(1, 64), frac_ladder=1.0)
    return hp, prices * np.exp(0.03 * np.random.default_rng(1).standard_normal(64))


def _bins_cases(rng, m, n, toks):
    """m random_bins pools (1, 2, 8 or 64 bins) on the token pairs toks, rebuilt around their token price ratio (1 %
    off each pool's middle) so that most trade, as tests/test_bins.py's kernel test"""
    nu = np.exp(rng.uniform(-2, 2, n))
    K = rng.choice([1, 2, 8, 64], m, p=[0.3, 0.3, 0.3, 0.1])
    r = nu[toks[:, 0]] / nu[toks[:, 1]]
    off = np.exp(0.01 * rng.standard_normal(m))
    cases = []
    for q in range(m):
        p, x, y = TB.random_bins(rng, int(K[q]))
        cases.append((p * r[q] * off[q] / np.sqrt(p[0] * p[-1]), x, y, float(rng.choice([1.0, 0.9995, 0.997]))))
    hp = HostPools.from_lists(n, toks.tolist(), [None] * m, [c[3] for c in cases], ["bins"] * m,
                              [c[:3] for c in cases])
    return hp, nu


def _bins(m=20_000, seed=11):
    rng = np.random.default_rng(seed)
    return _bins_cases(rng, m, 64, _pairs(m, 64, rng))


# ------------------------------------------------------------------------------------------ extended-precision anchors
def _nu_rows(inst, sel):
    return inst.nu[_rows(inst.hp.tok_idx, inst.A)[sel]]


def _anchor_closed_form(inst, sel, D, L):
    """product, constant-sum, bounded and geometric-mean pools against xp_reference's closed forms: within 1e-12 of the
    pool's reserve scale (of its trade, where that is larger), as the oracle comparisons of tests/test_gpu_parity.py"""
    hp, k = inst.hp, inst.A
    R, W, g, nv = _rows(hp.reserves, k)[sel], _rows(hp.weights, k)[sel], hp.gamma[sel], _nu_rows(inst, sel)
    ok = np.ones(len(sel), bool)
    scale = R.max(1)
    if inst.kind == _lib.KIND_PRODUCT:
        Dx, Lx, _ = X._product(X.ld(R), X.ld(g), X.ld(nv))
    elif inst.kind == _lib.KIND_BOUNDED:
        Dx, Lx, _ = X._bounded(X.ld(R), X.ld(W), X.ld(g), X.ld(nv))
        scale = (R + W).max(1)
    elif inst.kind == _lib.KIND_GEOMEAN:
        Dx, Lx, _ = X._geomean(X.ld(R), X.ld(W), X.ld(g), X.ld(nv))
    elif inst.eps == 0.0:
        Dx, Lx, _ = X._sum(X.ld(R), X.ld(g), X.ld(nv))
        # a price within 1e-12 of the fill switch fills by a rounding in one precision and not in the other
        ok = np.all(np.abs(g[:, None] * nv[:, ::-1] / nv - 1) > 1e-12, 1)
    else:
        Dx, Lx = _sum_smoothed(R, g, nv, inst.eps, inst.theta.T[inst.pos[sel]])
        scale = scale * (1 + 1 / inst.eps)
    Dx, Lx = Dx.astype(float), Lx.astype(float)
    gross = (np.abs(Dx) + np.abs(Lx)).sum(1)
    bound = 1e-12 * np.maximum(scale, gross)[:, None]
    err = np.maximum(np.abs(D - Dx), np.abs(L - Lx))
    assert np.all(err[ok] <= bound[ok]), float((err / bound)[ok].max())


def _sum_smoothed(R, g, nv, eps, thbar):
    """the proximal fill of both orders of constant-sum pools in long double: order A tenders token 0 for up to R_1
    (multiplier theta_bar row 1), order B tenders token 1 for up to R_0 (row 0); th = clip(thbar + sigma z, 0, R_b),
    sigma = R_b / eps, z = gamma nu_b / nu_a - 1, paying (r th - psi) / gamma"""
    R, g, nv, thbar = X.ld(R), X.ld(g), X.ld(nv), X.ld(thbar)
    D = np.zeros_like(R); L = np.zeros_like(R)
    for a, b, tcol in ((0, 1, 1), (1, 0, 0)):
        r = g * nv[:, b] / nv[:, a]
        z = r - 1
        sigma = R[:, b] / X.LD(eps)
        th = np.minimum(np.maximum(thbar[:, tcol] + sigma * z, 0), R[:, b])
        d = th - thbar[:, tcol]
        psi = th * z - d * d / (2 * sigma)
        L[:, b] = th
        D[:, a] = (r * th - psi) / g
    return D, L


def _anchor_stable(inst, sel, D, L):
    hp = inst.hp
    R, r, nv = _rows(hp.reserves, 2)[sel], _rows(hp.weights, 2)[sel], _nu_rows(inst, sel)
    Dx, Lx, hx = XS.stableswap_response(R, r, hp.amp[sel], hp.inv[sel], hp.gamma[sel], nv)
    bound = TS.flow_bound(Dx, Lx, hx, hp.gamma[sel], nv, R)
    err = np.maximum(np.abs(D - Dx.astype(float)).max(1), np.abs(L - Lx.astype(float)).max(1))
    assert np.all(err <= bound), float((err / bound).max())


def _anchor_stable_n(inst, sel, D, L):
    hp, k = inst.hp, inst.A
    R, r, nv = _rows(hp.reserves, k)[sel], _rows(hp.weights, k)[sel], _nu_rows(inst, sel)
    A, Dv, g = hp.amp[sel], hp.inv[sel], hp.gamma[sel]
    Dx, Lx, _, Hs = XN.stablen_response(R, r, A, Dv, g, nv)
    Dx, Lx = Dx.astype(float), Lx.astype(float)
    tol = TN.flow_tol(Dx, Lx, R, TN._lq(R, r, A, Dv), Hs.astype(float), nv) + TN.arg_tol(R, r, A, Dv, g, nv, Dx, Lx)
    err = np.maximum(np.abs(D - Dx), np.abs(L - Lx))
    assert np.all(err <= tol), float((err / tol).max())


def _anchor_crypto(inst, sel, D, L, h):
    hp = inst.hp
    TC._check_against_xp(D, L, h, _rows(hp.reserves, 2)[sel], _rows(hp.weights, 2)[sel], hp.amp[sel], hp.cgam[sel],
                         hp.inv[sel], hp.gamma[sel], _nu_rows(inst, sel))


def _anchor_tricrypto(inst, sel, D, L, h, mk):
    hp = inst.hp
    TT._check_against_xp(D, L, h, mk, _rows(hp.reserves, 3)[sel], _rows(hp.weights, 3)[sel], hp.amp[sel], hp.cgam[sel],
                         hp.inv[sel], hp.gamma[sel], _nu_rows(inst, sel))


def _anchor_concentrated(inst, sel, D, L):
    ref = inst.memo("xp", lambda: XC.response(inst.hp, inst.nu))
    Dx, Lx = _rows(ref["delta"], 2)[sel].astype(float), _rows(ref["lam"], 2)[sel].astype(float)
    tol = TCL.ladder_tol(inst.hp, sel, inst.nu, Dx, Lx)
    err = np.maximum(np.abs(D - Dx), np.abs(L - Lx))
    assert np.all(err <= tol), float((err / tol).max())


def _anchor_bins(inst, sel, D, L):
    """xp_bins bin by bin (eps = 0: within 1e-12 of each token's capacity, pools priced within 1e-12 of a segment's slope
    masked) or its smoothed form (eps > 0: the net flows), as tests/test_bins.py's kernel test"""
    hp, nv = inst.hp, _nu_rows(inst, sel)
    checked = 0
    for q, i in enumerate(sel.tolist()):
        p, x, y = (np.asarray(v, float) for v in XB.bins_of(hp, i))
        g = float(hp.gamma[i])
        s0, s1 = TB._scales(p, x, y, g)
        if inst.eps == 0.0:
            if TB._near_slope(p, x, y, g, nv[q, 0] / nv[q, 1]):
                continue
            Dx, Lx = (np.asarray(v, float) for v in XB.exact(p, x, y, g, nv[q, 0], nv[q, 1]))
            sc = np.array([s0, s1])
            assert np.all(np.abs(D[q] - Dx) <= 1e-12 * sc) and np.all(np.abs(L[q] - Lx) <= 1e-12 * sc), i
        else:
            t, c = XB.smoothed(p, x, y, g, nv[q, 0], nv[q, 1], inst.eps, inst.theta[0, inst.pos[i]], hp.bin_zp[i, 1])
            assert abs(float(t) - (L[q, 0] - D[q, 0])) <= 1e-12 * s0, i
            assert abs(-float(c) - (L[q, 1] - D[q, 1])) <= 1e-12 * s1 / inst.eps, i
        checked += 1
    assert checked >= 0.9 * len(sel), checked


def _anchor(inst, sample, out):
    """(d): the per-pool flows of `out` (bucket order) on the bucket positions `sample` against the kind's reference"""
    sel = inst.sel[sample]
    D, L = out["D"][:, sample].T, out["L"][:, sample].T
    kd = inst.kind
    if kd in (_lib.KIND_PRODUCT, _lib.KIND_SUM, _lib.KIND_BOUNDED, _lib.KIND_GEOMEAN):
        _anchor_closed_form(inst, sel, D, L)
    elif kd == _lib.KIND_STABLESWAP:
        _anchor_stable(inst, sel, D, L)
    elif kd == _lib.KIND_STABLESWAP_N:
        _anchor_stable_n(inst, sel, D, L)
    elif kd == _lib.KIND_CRYPTOSWAP:
        _anchor_crypto(inst, sel, D, L, out["h"][sample])
    elif kd == _lib.KIND_CRYPTOSWAP_3:
        _anchor_tricrypto(inst, sel, D, L, out["h"][:, sample].T, out["mk"][sample].astype(np.uint32))
    elif kd == _lib.KIND_CONCENTRATED:
        _anchor_concentrated(inst, sel, D, L)
    else:
        _anchor_bins(inst, sel, D, L)


# ====================================================================================================== the harness
class Inst:
    """one single-bucket plain-layout store, its prices, and the C ABI calls on it with fresh output buffers"""

    def __init__(self, hp, nu, eps=0.0, theta_seed=None, force=None):
        self.hp, self.nu, self.eps = hp, np.asarray(nu, np.float64), float(eps)
        self.st = cf.PoolStore(hp, layout="plain")
        if force is not None:     # two-coin StableSwap pools as a kind-5 bucket (split_buckets makes them kind 4)
            self.st.buckets = [cf.pools.DeviceBucket(hp, cf.pools.BucketSpec(hp, force[0], force[1], None),
                                                     self.st.device)]
        assert len(self.st.buckets) == 1, [(int(b.kind), int(b.arity)) for b in self.st.buckets]
        self.b = self.st.buckets[0]
        self.kind, self.A, self.m, self.n = int(self.b.kind), int(self.b.arity), int(self.b.m), int(hp.n_tokens)
        self.tok = self.b.tok_idx[:, :self.m].cpu().numpy().astype(np.int64)
        self.sel = np.asarray(self.b.sel, np.int64) if self.m else np.zeros(0, np.int64)
        self.pos = np.empty(hp.m, np.int64); self.pos[self.sel] = np.arange(self.m)
        self.theta = None
        if theta_seed is not None:        # multipliers: constant-sum fills in [0, R_b], bins net flows within the depth
            rng = np.random.default_rng(theta_seed)
            if self.kind == _lib.KIND_SUM:
                R = self.b.reserves[:, :self.m].cpu().numpy()
                th = np.where(rng.random((2, self.m)) < 0.3, 0.0, rng.random((2, self.m)) * R[::-1])
            else:
                S = np.array([np.asarray(XB.bins_of(hp, i)[1], float).sum() for i in self.sel.tolist()])
                th = np.stack([np.where(rng.random(self.m) < 0.3, 0.0, rng.uniform(-1, 1, self.m) * S),
                               np.zeros(self.m)])
            self.theta = th
            self.b.theta_bar[:, :self.m] = torch.as_tensor(th, **F64)
        self.nu_d = torch.as_tensor(self.nu, **F64)
        self.lognu_d = torch.log(self.nu_d)
        rng = np.random.default_rng(99)
        self.base = np.concatenate([rng.uniform(-1, 1, self.n), [rng.uniform(-1, 1)]])   # what psi | arb held before
        self._memo = {}

    def memo(self, key, fn):
        if key not in self._memo:
            self._memo[key] = fn()
        return self._memo[key]

    def stream(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def eval(self, trades, hess, bucket=None):
        """cfmm_arb_eval into [psi | arb] = base; returns (acc, per-pool outputs (bucket order), unwritten sentinels
        checked)"""
        cb = bucket if bucket is not None else self.b.c_bucket
        m, A, ld = int(cb.n_pools), self.A, int(cb.stride)
        acc = torch.as_tensor(self.base, **F64).clone()
        bufs = {}
        if trades:
            bufs["D"] = torch.full((A, ld), np.nan, **F64)
            bufs["L"] = torch.full((A, ld), np.nan, **F64)
        if hess:
            bufs["h"] = torch.full((A, ld) if self.kind in (_lib.KIND_STABLESWAP_N, _lib.KIND_CRYPTOSWAP_3)
                                   else (ld,), np.nan, **F64)
            bufs["mk"] = torch.full((ld,), -1, dtype=torch.int32, device="cuda")
        ptr = lambda k: bufs[k].data_ptr() if k in bufs else None
        out = _lib.EvalOut(ptr("D"), ptr("L"), ptr("h"), ptr("mk"))
        rc = self.st.lib.cfmm_arb_eval(C.byref(cb), self.n,
                                       self.nu_d.data_ptr(), self.lognu_d.data_ptr(), self.eps, acc.data_ptr(),
                                       acc.data_ptr() + 8 * self.n, C.byref(out) if bufs else None, self.stream())
        _lib.check(rc, "cfmm_arb_eval")
        torch.cuda.synchronize()
        res = {k: v[..., :m].cpu().numpy() for k, v in bufs.items()}
        # every pool's slots were written
        for k in ("D", "L", "h"):
            if k in res:
                assert not np.isnan(res[k]).any(), f"{k}: {int(np.isnan(res[k]).sum())} slots not written"
        if hess and self.kind in MASKED:
            assert np.all(res["mk"] != -1), "hmask not written"
        return acc.cpu().numpy(), res

    def hess_calls(self, h, mk, vt, base_y, base_d, base_H):
        """cfmm_hvp / cfmm_hess_diag / cfmm_hess_dense (dense when base_H is given) from the given hcoef / hmask"""
        b, lib, st = self.b, self.st.lib, self.stream()
        hd = torch.as_tensor(np.ascontiguousarray(_pad(h, b.stride)), **F64)
        md = torch.as_tensor(np.ascontiguousarray(_pad(mk, b.stride)), dtype=torch.int32, device="cuda")
        y = torch.as_tensor(base_y, **F64).clone()
        d = torch.as_tensor(base_d, **F64).clone()
        vd = torch.as_tensor(vt, **F64)
        _lib.check(lib.cfmm_hvp(C.byref(b.c_bucket), self.n, hd.data_ptr(), md.data_ptr(), vd.data_ptr(), y.data_ptr(),
                                st), "cfmm_hvp")
        _lib.check(lib.cfmm_hess_diag(C.byref(b.c_bucket), self.n, hd.data_ptr(), md.data_ptr(), d.data_ptr(), st),
                   "cfmm_hess_diag")
        H = None
        if base_H is not None:
            Hd = torch.as_tensor(base_H, **F64).clone()
            _lib.check(lib.cfmm_hess_dense(C.byref(b.c_bucket), self.n, hd.data_ptr(), md.data_ptr(), Hd.data_ptr(), st),
                       "cfmm_hess_dense")
            H = Hd.cpu().numpy()
        torch.cuda.synchronize()
        return y.cpu().numpy(), d.cpu().numpy(), H


def _pad(x, stride):
    x = np.asarray(x)
    out = np.zeros(x.shape[:-1] + (stride,), x.dtype)
    out[..., :x.shape[-1]] = x
    return out


# ------------------------------------------------------------------------------------------------------- the checks
def _ulps(a, b):
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def check_same_pools(got, ref, mode, kind):
    """(a): the per-pool outputs of a (trades, hess) run under `mode` against those of the global-scatter run"""
    for k in ref:
        if k not in got or (k == "mk" and kind not in MASKED):
            continue
        a, b = got[k], ref[k]
        if mode == TMA and k != "mk":
            u = _ulps(a, b)
            assert np.all(u <= 2), (k, float(u.max()))
        else:
            diff = a.view(np.uint64 if a.dtype == np.float64 else np.uint32) != \
                b.view(np.uint64 if b.dtype == np.float64 else np.uint32)
            assert not diff.any(), (k, int(diff.sum()), "pools differ bitwise between global and shared scatter")


def _fsum_by_token(tok, vals, n, base):
    """per token, math.fsum of base_j and the values at j (exactly rounded), their gross and their count"""
    t = np.asarray(tok, np.int64).ravel(); v = np.asarray(vals, np.float64).ravel()
    nz = v != 0
    t, v = t[nz], v[nz]
    order = np.argsort(t, kind="stable")
    t, v = t[order], v[order]
    cut = np.searchsorted(t, np.arange(n + 1))
    exact = np.array([math.fsum([base[j]] + v[cut[j]:cut[j + 1]].tolist()) for j in range(n)])
    gross = np.abs(base[:n]) + np.bincount(t, np.abs(v), n)
    k = (base[:n] != 0) + np.bincount(t, minlength=n)
    return exact, gross, k


def check_sums(inst, acc, tok, y):
    """(b): psi = base + the flows y (arity, m) summed per token, arb = base + sum nu (L - D), each within 2 k u gross"""
    n = inst.n
    exact, gross, k = _fsum_by_token(tok, y, n, inst.base)
    lim = 2 * k * U * gross
    err = np.abs(acc[:n] - exact)
    assert np.all(err <= lim), (int(np.argmax(err - lim)), float(np.max(err / np.where(lim > 0, lim, 1e-300))))
    # nu_j y products: long double (64-bit significand) split into two doubles, summed exactly
    p = X.ld(inst.nu)[tok] * X.ld(y)
    hi = p.astype(np.float64)
    lo = (p - X.ld(hi)).astype(np.float64)
    arb = math.fsum([inst.base[n]] + hi.ravel().tolist() + lo.ravel().tolist())
    gross_a = abs(inst.base[n]) + float(np.abs(hi).sum())
    lim_a = 2 * (y.size + 1) * U * gross_a
    assert abs(acc[n] - arb) <= lim_a, (acc[n], arb, lim_a)


def _pool_parts(inst, h, mk, vt):
    """the pool decomposition of the Hessian from the kernel's hcoef / hmask, long double: per pool the slots' tokens
    (m, k), their hvp contributions and diagonal entries with rounding scales (m, k), and the dense entries with their
    scales (m, k, k).  Pools the kernels skip contribute 0."""
    kd, A, tok = inst.kind, inst.A, inst.tok.T
    z = X.ld(vt)[tok]
    if kd == _lib.KIND_STABLESWAP_N:
        hl = X.ld(h.T)
        kk = (hl != 0).sum(1).astype(X.LD)
        Ca = np.einsum("mi,ij->mij", hl * hl, np.eye(A, dtype=X.LD)) + np.abs(hl)[:, :, None] * np.abs(hl)[:, None, :] \
            / (1 + kk)[:, None, None]
        C1a = Ca.sum(2)
        Hc = XN.hess_block(hl)
        s1 = (np.einsum("mi,ij->mij", hl * hl, np.eye(A, dtype=X.LD)) - hl[:, :, None] * hl[:, None, :]
              / (1 + kk)[:, None, None]).sum((1, 2))
        S = Ca + C1a[:, :, None] * C1a[:, None, :] / np.where(s1 > 0, s1, 1)[:, None, None]
        on = (mk != 0)[:, None, None] & (s1 > 0)[:, None, None]
        Hs = np.where(on, Hc, 0); S = np.where(on, S, 0) * 8 * (A + 4)
        yv = (Hs @ z[:, :, None])[:, :, 0]
        ys = (S @ np.abs(z)[:, :, None])[:, :, 0]
        return tok, yv, ys, np.diagonal(Hs, 0, 1, 2), np.diagonal(S, 0, 1, 2), Hs, S
    if kd == _lib.KIND_CRYPTOSWAP_3:
        w = X.ld(h.T) * (mk != 0)[:, None]
        Hs = np.zeros((inst.m, 3, 3), X.LD)
        for q, (a, b) in enumerate(((0, 1), (0, 2), (1, 2))):
            Hs[:, a, a] += w[:, q]; Hs[:, b, b] += w[:, q]
            Hs[:, a, b] -= w[:, q]; Hs[:, b, a] -= w[:, q]
        S = np.abs(Hs) * 4
        return (tok, (Hs @ z[:, :, None])[:, :, 0], (S @ np.abs(z)[:, :, None])[:, :, 0], np.diagonal(Hs, 0, 1, 2),
                np.diagonal(S, 0, 1, 2), Hs, np.zeros_like(S))
    if kd == _lib.KIND_GEOMEAN:
        W = X.ld(_rows(inst.hp.weights, A)[inst.sel])
        act = (mk[:, None].astype(np.int64) >> np.arange(A)) & 1 == 1
        M = X.ld(h) * (mk != 0)
        wa = np.where(act, W, 0)
        Wa = wa.sum(1)
        Wa = np.where(Wa > 0, Wa, 1)
        Hs = M[:, None, None] * (np.einsum("mi,ij->mij", wa, np.eye(A, dtype=X.LD)) - wa[:, :, None] * wa[:, None, :]
                                 / Wa[:, None, None])
        S = M[:, None, None] * (np.einsum("mi,ij->mij", wa, np.eye(A, dtype=X.LD)) + wa[:, :, None] * wa[:, None, :]
                                / Wa[:, None, None]) * 2 * (A + 4)
        return (tok, (Hs @ z[:, :, None])[:, :, 0], (S @ np.abs(z)[:, :, None])[:, :, 0], np.diagonal(Hs, 0, 1, 2),
                np.diagonal(S, 0, 1, 2), Hs, S)
    hl = X.ld(h)                                        # the pair branch: h [[1, -1], [-1, 1]]
    c = hl * (z[:, 0] - z[:, 1])
    yv = np.stack([c, -c], 1)
    ys = 4 * np.abs(yv)
    dv = np.stack([hl, hl], 1)
    Hs = hl[:, None, None] * np.array([[1, -1], [-1, 1]], X.LD)
    return tok, yv, ys, dv, np.zeros_like(dv), Hs, np.zeros_like(Hs)


def _ld_scatter(n, idx, vals):
    out = np.zeros(n, X.LD)
    np.add.at(out, np.asarray(idx, np.int64).ravel(), np.asarray(vals, X.LD).ravel())
    return out


def _check_acc(got, base, idx, vals, scales, n):
    """got = base + the values scattered to idx, within their rounding scales plus 2 k u gross"""
    ref = X.ld(base) + _ld_scatter(n, idx, vals)
    gross = np.abs(base) + _ld_scatter(n, idx, np.abs(vals)).astype(float)
    k = (base != 0) + _ld_scatter(n, idx, (np.asarray(vals) != 0).astype(X.LD)).astype(float)
    lim = U * _ld_scatter(n, idx, scales).astype(float) + 2 * k * U * gross
    err = np.abs(got - ref.astype(float))
    assert np.all(err <= lim), float(np.max(err / np.where(lim > 0, lim, 1e-300)))


def check_hessians(inst, h, mk):
    """(c): hvp, hess_diag and (up to 2048 tokens) hess_dense from (h, mk), under the current mode, into buffers that
    already hold values, against the pool decomposition"""
    n = inst.n
    rng = np.random.default_rng(5)
    vt, by, bd = rng.standard_normal(n), rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    bH = rng.uniform(-1, 1, (n, n)) if n <= 2048 else None
    y, d, H = inst.hess_calls(h, mk, vt, by, bd, bH)
    tok, yv, ys, dv, ds, Hs, S = _pool_parts(inst, h, mk, vt)
    _check_acc(y, by, tok, yv, ys, n)
    _check_acc(d, bd, tok, dv, ds, n)
    if H is not None:
        flat = tok[:, :, None] * n + tok[:, None, :]
        _check_acc(H.ravel(), bH.ravel(), flat, Hs, S, n * n)


def full_run(inst, mode, set_mode):
    """the (trades, hess) = (True, True) run under `mode`, once per instance and mode"""
    def run():
        set_mode(mode)
        return inst.eval(True, True)
    return inst.memo(("full", mode), run)


def check_cell(inst, mode, trades, hess, set_mode, anchor=True):
    """one (instance, strategy, flags) cell: (a) - (d)"""
    acc_f, full = full_run(inst, mode, set_mode)
    if mode != GLOBAL:
        check_same_pools(full, full_run(inst, GLOBAL, set_mode)[1], mode, inst.kind)
    set_mode(mode)
    acc, out = (acc_f, full) if (trades and hess) else inst.eval(trades, hess)
    src = {**full, **out} if trades else full         # the flows of this run, the Hessian outputs of the full one
    check_sums(inst, acc, inst.tok, src["L"] - src["D"])
    if hess:
        check_hessians(inst, out["h"], out["mk"] if inst.kind in MASKED else np.zeros(inst.m, np.int32))
    if anchor and inst.m:
        smp = inst.memo("sample", lambda: np.sort(np.random.default_rng(3).choice(inst.m, min(SAMPLE, inst.m),
                                                                                   replace=False)))
        # once per distinct set of sampled outputs: (a) makes the strategies' sets one
        key = b"".join(np.ascontiguousarray(v[..., smp]).tobytes() for v in src.values())
        inst.memo(("anchor", key), lambda: _anchor(inst, smp, src))


# ====================================================================================================== the matrix
TARGETS = {
    "product": lambda: Inst(*_product()),
    "sum": lambda: Inst(*_sum()),
    "sum-eps": lambda: Inst(*_sum(), eps=0.05, theta_seed=1),
    "bounded": lambda: Inst(*_bounded()),
    "stableswap": lambda: Inst(*TS._bucket_pools(30_000)),
    "cryptoswap": lambda: Inst(*_crypto()),
    "concentrated": lambda: Inst(*_concentrated()),
    "bins": lambda: Inst(*_bins()),
    "bins-eps": lambda: Inst(*_bins(), eps=0.05, theta_seed=2),
    "cryptoswap3": lambda: Inst(*_tricrypto()),
    **{f"stableswap_n{k}": (lambda k=k: Inst(*TN._bucket(k, 20_000, 50 + k), force=(_lib.KIND_STABLESWAP_N, k)))
       for k in range(2, 9)},
    **{f"geomean{k}": (lambda k=k: Inst(*_geomean(k))) for k in (2, 3, 4, 5, 6, 7, 8, 13)},
}
KIND_OF = {"product": _lib.KIND_PRODUCT, "sum": _lib.KIND_SUM, "sum-eps": _lib.KIND_SUM, "bounded": _lib.KIND_BOUNDED,
           "stableswap": _lib.KIND_STABLESWAP, "cryptoswap": _lib.KIND_CRYPTOSWAP,
           "concentrated": _lib.KIND_CONCENTRATED, "bins": _lib.KIND_BINS, "bins-eps": _lib.KIND_BINS,
           "cryptoswap3": _lib.KIND_CRYPTOSWAP_3,
           **{f"stableswap_n{k}": _lib.KIND_STABLESWAP_N for k in range(2, 9)},
           **{f"geomean{k}": _lib.KIND_GEOMEAN for k in (2, 3, 4, 5, 6, 7, 8, 13)}}
STRATEGY = {"global": GLOBAL, "shared": SHARED, "tma": TMA}
CELLS = [pytest.param(t, s, tr, hs, id=f"{t}-{s}-{'T' if tr else 'F'}{'H' if hs else 'F'}")
         for t in TARGETS for s in (("global", "shared", "tma") if t in ("product", "sum", "sum-eps")
                                    else ("global", "shared"))
         for tr, hs in FLAGS]


@functools.lru_cache(maxsize=None)
def instance(target):
    inst = TARGETS[target]()
    assert inst.kind == KIND_OF[target], (target, inst.kind)
    return inst


def test_scatter_mode_switch_rejects_unknown_modes(scatter_mode):
    lib = _lib.load()
    for m in (AUTO, GLOBAL, SHARED, TMA):
        scatter_mode(m)
    assert lib.cfmm_set_scatter_mode(4) == CFMM_E_KIND
    assert lib.cfmm_set_scatter_mode(-7) == CFMM_E_KIND


@pytest.mark.parametrize("target,strategy,trades,hess", CELLS)
def test_instance_under_strategy(target, strategy, trades, hess, scatter_mode):
    inst = instance(target)
    if target.startswith("geomean"):
        assert inst.A == int(target[7:])
    check_cell(inst, STRATEGY[strategy], trades, hess, scatter_mode)


# ====================================================================================================== shapes
def _hot_tokens(m, n, k, rng):
    """(m, k) token ids: every pool on token 0, the others spread over 1 .. n - 1 with the last pool (and every
    (n - 1)-th) on token n - 1"""
    toks = np.zeros((m, k), np.int64)
    if k == 2:
        toks[:, 1] = 1 + np.arange(m) % (n - 1)
        toks[-1:, 1] = n - 1
        flip = np.arange(m) % 2 == 1                  # token 0 in slot 0 and in slot 1
        toks[flip] = toks[flip][:, ::-1]
        return toks
    for i in range(m):
        rest = rng.choice(np.arange(1, n - 1), k - 2, replace=False)
        toks[i] = np.concatenate([[0, n - 1], rest])[rng.permutation(k)]
    return toks


def _tile(hp, reps):
    """hp's pools repeated reps times on the same tokens"""
    m = hp.m
    bp = np.asarray(hp.bin_ptr, np.int64)
    kw = dict(amp=np.tile(hp.amp, reps), inv=np.tile(hp.inv, reps), cgam=np.tile(hp.cgam, reps))
    if bp[-1] > 0:
        cnt = np.tile(np.diff(bp), reps)
        kw.update(bin_ptr=np.concatenate([[0], np.cumsum(cnt)]), bin_rec=np.tile(hp.bin_rec, (reps, 1)),
                  bin_zp=np.tile(hp.bin_zp, (reps, 1)))
    k = int(hp.pool_ptr[1])
    return HostPools(hp.n_tokens, np.arange(0, k * m * reps + 1, k, dtype=np.int64), np.tile(hp.tok_idx, reps),
                     np.tile(hp.reserves, reps), np.tile(hp.weights, reps), np.tile(hp.gamma, reps),
                     np.tile(hp.kind, reps), **kw)


def _shape_instance(kind, m, n, seed=0):
    """m pools of `kind` ("product", "stableswap_n8", "bins") on n tokens, hot on token 0 and n - 1 (at most 1024
    distinct pools, repeated)"""
    rng = np.random.default_rng(seed + m + 7 * n)
    m0 = min(m, 1024)
    if kind == "product":
        toks = _hot_tokens(m0, n, 2, rng)
        nu = np.exp(rng.normal(0, 0.3, n))
        R = np.exp(rng.normal(8, 2, m0))[:, None] / nu[toks] * np.exp(rng.normal(0, 0.05, (m0, 2)))
        g = np.array([1.0, 0.997, 0.99])[rng.integers(0, 3, m0)]
        hp = _csr(n, toks, R, np.full((m0, 2), 0.5), g, KIND_GEOMEAN_HOST)
    elif kind == "stableswap_n8":
        R, r, A, _, g, nu_p = TN.random_pools(m0, 8, seed + 1, peg=m0 % 2 == 0)
        toks = _hot_tokens(m0, n, 8, rng)
        nu = np.exp(rng.normal(0, 0.3, n))
        hp = TN._stable_hp(R, r * nu[toks] / nu_p, A, g, toks, n)
    else:
        toks = _hot_tokens(m0, n, 2, rng)
        hp, nu = _bins_cases(rng, m0, n, toks)
    if m > m0:
        hp = _tile(hp, -(-m // m0))
        if hp.m > m:
            hp = _first(hp, m)
    return Inst(hp, nu)


def _first(hp, m):
    k = int(hp.pool_ptr[1])
    bp = np.asarray(hp.bin_ptr, np.int64)
    kw = dict(amp=hp.amp[:m], inv=hp.inv[:m], cgam=hp.cgam[:m])
    if bp[-1] > 0:
        kw.update(bin_ptr=bp[:m + 1], bin_rec=hp.bin_rec[:bp[m]], bin_zp=hp.bin_zp[:m])
    return HostPools(hp.n_tokens, hp.pool_ptr[:m + 1], hp.tok_idx[:k * m], hp.reserves[:k * m], hp.weights[:k * m],
                     hp.gamma[:m], hp.kind[:m], **kw)


SHAPE_KINDS = ("product", "stableswap_n8", "bins")
SHAPES = [pytest.param(kd, m, n, id=f"{kd}-m{m}-n{n}") for kd in SHAPE_KINDS for m in (1, 255, 256, 257)
          for n in (2, 3, 257, 12288, 12289) if not (kd == "stableswap_n8" and n < 8)]


@pytest.mark.parametrize("strategy", ["global", "shared"])
@pytest.mark.parametrize("kind,m,n", SHAPES)
def test_bucket_and_token_shapes(kind, m, n, strategy, scatter_mode):
    """both flag extremes at every bucket size around a CTA (255 .. 257) and token counts around the 96 KB histogram;
    shared runs bitwise equal to global ones"""
    inst = _shape_instance(kind, m, n)
    for trades, hess in ((True, True), (False, False)):
        check_cell(inst, STRATEGY[strategy], trades, hess, scatter_mode, anchor=kind == "product")


@pytest.mark.parametrize("strategy", ["global", "shared", "tma"])
def test_empty_bucket_leaves_the_buffers_untouched(strategy, scatter_mode):
    inst = _shape_instance("product", 1, 257)
    scatter_mode(STRATEGY[strategy])
    b = inst.b.c_bucket
    empty = _lib.Bucket(b.kind, b.arity, 0, b.stride, b.reserves, b.tok_idx, b.gamma, b.weights, b.logrw, b.theta_bar)
    acc, _ = inst.eval(True, True, bucket=empty)
    assert acc.tobytes() == inst.base.tobytes()
    y = torch.as_tensor(inst.base[:-1], **F64).clone()
    h = torch.ones(b.stride, **F64)
    _lib.check(inst.st.lib.cfmm_hvp(C.byref(empty), inst.n, h.data_ptr(), None, inst.nu_d.data_ptr(), y.data_ptr(),
                                    inst.stream()), "cfmm_hvp")
    torch.cuda.synchronize()
    assert y.cpu().numpy().tobytes() == inst.base[:-1].tobytes()


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("strategy", ["global", "shared"])
@pytest.mark.parametrize("kind", SHAPE_KINDS)
def test_grid_stride_loops(kind, strategy, scatter_mode):
    """more pools than the capped grid has threads: every CTA of the global instance (8 CTAs per SM; 4 for n-coin
    StableSwap) goes round its loop at least twice, and the shared one's (2 per SM) more often"""
    per_sm = 4 if kind == "stableswap_n8" else 8
    m = 2 * _num_sms() * per_sm * 256 + 123
    inst = _shape_instance(kind, m, 257)
    assert inst.m == m
    check_cell(inst, STRATEGY[strategy], True, True, scatter_mode, anchor=kind == "product")
    check_cell(inst, STRATEGY[strategy], False, False, scatter_mode, anchor=False)


@pytest.mark.parametrize("target", ["product", "sum-eps"])
@pytest.mark.parametrize("m", [517, 3000, "several"])
def test_tma_tiles(target, m, scatter_mode):
    """the TMA kernel on a partial tile, a bucket that is not a whole number of tiles, and enough tiles that each CTA
    (two per SM) takes several rounds of its three-stage ring; against the LDG kernel with global scatter"""
    if m == "several":
        m = 4 * 2 * _num_sms() * 1024 + 517
    rng = np.random.default_rng(m)
    if target == "product":
        toks = _hot_tokens(m, 64, 2, rng)
        nu = np.exp(rng.normal(0, 0.3, 64))
        R = np.exp(rng.normal(8, 2, m))[:, None] / nu[toks] * np.exp(rng.normal(0, 0.05, (m, 2)))
        hp = _csr(64, toks, R, np.full((m, 2), 0.5), np.full(m, 0.997), KIND_GEOMEAN_HOST)
        inst = Inst(hp, nu)
    else:
        hp, nu = _sum(m, seed=7)
        inst = Inst(hp, nu, eps=0.05, theta_seed=3)
    for trades, hess in FLAGS:
        check_cell(inst, TMA, trades, hess, scatter_mode, anchor=True)


def _realigned(inst, stride, offset):
    """inst's bucket re-laid at `stride` (any value >= m), each array starting `offset` elements into its allocation;
    returns (Bucket, the tensors keeping it alive)"""
    b, m = inst.b, inst.m
    keep = []

    def lay(t, dtype):
        rows = t[..., :m]
        flat = torch.zeros(offset + (rows.shape[0] if rows.dim() == 2 else 1) * stride, dtype=dtype, device="cuda")
        v = flat[offset:].view(-1, stride) if rows.dim() == 2 else flat[offset:]
        v[..., :m] = rows
        keep.append(flat)
        return v.data_ptr()
    th = lay(b.theta_bar, torch.float64) if b.theta_bar is not None else None
    return _lib.Bucket(b.kind, b.arity, m, stride, lay(b.reserves, torch.float64), lay(b.tok_idx, torch.int32),
                       lay(b.gamma, torch.float64), None, None, th), keep


@pytest.mark.parametrize("target", ["product", "sum-eps"])
@pytest.mark.parametrize("stride_pad,offset", [(5, 0), (0, 1), (3, 1)], ids=["stride", "misaligned", "both"])
def test_buckets_the_tma_kernel_must_not_take(target, stride_pad, offset, scatter_mode):
    """a stride that is not a whole number of tiles, or arrays not 16-byte aligned: auto and TMA mode take the LDG
    kernel, whose per-pool results equal the global-scatter run's bit for bit (the shapes keep auto on global)"""
    inst = Inst(*(_product(20_480) if target == "product" else _sum(20_480)),
                **({} if target == "product" else dict(eps=0.05, theta_seed=4)))
    stride = inst.m + stride_pad if stride_pad else inst.b.stride
    bucket, keep = _realigned(inst, stride, offset)
    _, ref = full_run(inst, GLOBAL, scatter_mode)
    for mode in (AUTO, TMA):
        scatter_mode(mode)
        acc, out = inst.eval(True, True, bucket=bucket)
        check_same_pools(out, ref, GLOBAL, inst.kind)
        check_sums(inst, acc, inst.tok, out["L"] - out["D"])
    del keep


@pytest.mark.parametrize("strategy", ["auto", "global", "shared", "tma"])
def test_several_buckets_add_into_one_psi(strategy, scatter_mode):
    """a plain store of every two-token kind, weighted and n-coin pools evaluated into one [psi | arb]: each bucket's
    kernel adds to what the previous ones left"""
    scatter_mode({"auto": AUTO, **STRATEGY}[strategy])
    hp, prices = I.synth_concentrated_market(30_000, 200, seed=5, T=(1, 16))
    st = cf.PoolStore(hp, layout="plain")
    assert len(st.buckets) >= 5, [int(b.kind) for b in st.buckets]
    nu = prices * np.exp(0.02 * np.random.default_rng(2).standard_normal(200))
    acc = st.evaluate(torch.as_tensor(nu, **F64), 0.0, trades=True).cpu().numpy()
    toks, ys = [], []
    for b in st.buckets:
        toks.append(b.tok_idx[:, :b.m].cpu().numpy().ravel())
        ys.append((b.lam[:, :b.m] - b.delta[:, :b.m]).cpu().numpy().ravel())
    tok, y = np.concatenate(toks), np.concatenate(ys)
    exact, gross, k = _fsum_by_token(tok, y, 200, np.zeros(201))
    assert np.all(np.abs(acc[:200] - exact) <= 2 * k * U * gross)
    p = X.ld(nu)[tok] * X.ld(y)
    assert abs(acc[200] - float(p.sum())) <= 2 * (y.size + 1) * U * float(np.abs(p).sum())
