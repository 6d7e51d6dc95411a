"""Fee records of the blocked layout (include/cfmm_b200.h): a tile with at most 16 distinct 1/gamma values carries them in
a per-tile table plus a 4-bit code per pool, and the evaluation reads the table instead of streaming the 1/gamma slab.
The torch builder (pools.fee_records) is checked on the CPU; the native builder (csrc/cfmm_layout.cu) against it, and the
evaluation and the persistent solve with records against the same stores without them, on the GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib
from cfmm_routing_code_b200 import instances as I
from cfmm_routing_code_b200 import pools as PL
import helpers as H

P = 1024
TIERS = np.array([0.997, 0.999, 0.9995])


def decode(rec, P):
    """(nfee, table bit patterns (n_tiles, 16) int64, codes (n_tiles, P)) of fee records (n_tiles, words) int32"""
    r = rec.to(torch.int64) & 0xffffffff
    nfee = r[:, 0]
    table = r[:, 4:36:2] | (r[:, 5:36:2] << 32)
    l = torch.arange(P)
    codes = (r[:, 36 + (l >> 3)] >> (4 * (l & 7))) & 15
    return nfee, table, codes


def slab(gi_real, P):
    """the 1/gamma slab of a blocked layout: real pools, then padding pools at 1.0 up to whole tiles"""
    m = len(gi_real)
    out = torch.ones(-(-m // P) * P, dtype=torch.float64)
    out[:m] = torch.as_tensor(gi_real, dtype=torch.float64)
    return out


def test_torch_fee_record_decodes_bit_for_bit_to_the_slab():
    rng = np.random.default_rng(0)
    gi = slab(1.0 / TIERS[rng.integers(0, 3, 5 * P)], P)
    rec = PL.fee_records(gi, P)
    assert rec.shape == (5, 36 + P // 8) and rec.dtype == torch.int32
    nfee, table, codes = decode(rec, P)
    bits = gi.view(torch.int64).view(-1, P)
    assert bool((nfee == 3).all())
    assert torch.equal(table.gather(1, codes), bits)                                    # table[code(l)] is the slab entry
    assert bool((table[:, :3][:, 1:] > table[:, :3][:, :-1]).all())                     # ascending bit patterns
    assert bool((table[:, 3:] == 0).all()) and bool((rec[:, 1:4] == 0).all())


def test_tile_with_17_distinct_fees_streams_its_slab():
    rng = np.random.default_rng(1)
    f16, f17 = 1.0 + np.arange(16) * 1e-3, 1.0 + np.arange(17) * 1e-3
    gi = torch.cat([slab(f16[rng.integers(0, 16, P)], P), slab(f17[rng.integers(0, 17, P)], P),
                    slab(np.r_[f17, f17[rng.integers(0, 17, P - 17)]], P)])
    rec = PL.fee_records(gi, P)
    nfee, table, codes = decode(rec, P)
    assert nfee.tolist() == [16, 0, 0]
    assert torch.equal(table[0].gather(0, codes[0]), gi[:P].view(torch.int64))
    assert bool((rec[1:] == 0).all())                                                   # the record is inert


def test_ragged_last_tile_includes_padding_in_its_table():
    rng = np.random.default_rng(2)
    m = 2 * P + 300
    gi = slab(1.0 / TIERS[rng.integers(0, 3, m)], P)
    nfee, table, codes = decode(PL.fee_records(gi, P), P)
    one = torch.tensor([1.0], dtype=torch.float64).view(torch.int64)
    assert nfee.tolist() == [3, 3, 4]                                                   # 1.0 (padding) joins the three tiers
    assert int(table[2, 0]) == int(one)                                                 # 1.0 is the smallest 1/gamma
    assert bool((codes[2, 300:] == 0).all()) and bool((codes[2, :300] > 0).all())
    assert torch.equal(table.gather(1, codes), gi.view(torch.int64).view(-1, P))


# ---------------------------------------------------------------------------------------------------------------- GPU
F64 = dict(dtype=torch.float64, device="cuda")


def _instance(m, n, seed, fees):
    """constant-product pools of synth_const_product with fees by blocked position: 'tiers' = the three tiers everywhere
    (every tile coded), 'uniform' = drawn from (0.99, 1] (no tile coded), 'mixed' = tiers on even tiles and uniform on
    odd ones, so every CTA that walks more than one tile meets both kinds"""
    s = I.synth_const_product(m, n, seed)
    if fees != "tiers":
        rng = np.random.default_rng(seed)
        uni = 1.0 - 0.01 * rng.random(m)                                               # (0.99, 1]
        if fees == "uniform":
            s["gamma"] = uni
        else:
            hp = cf.HostPools.from_pairs(n, s["idx"], s["reserves"], s["gamma"])
            order = cf.PoolStore(hp).buckets[0].order.cpu().numpy().astype(np.int64)   # the layout depends on tokens only
            odd = np.zeros(m, bool)
            odd[order] = (np.arange(m) // P) % 2 == 1
            s["gamma"] = np.where(odd, uni, s["gamma"])
    return cf.HostPools.from_pairs(n, s["idx"], s["reserves"], s["gamma"]), s


def _eval(lib, cb, n, nu, M, out):
    acc = torch.zeros(n + 1, **F64)
    outs = None
    if out:
        outs = (torch.zeros((2, M), **F64), torch.zeros((2, M), **F64), torch.zeros(M, **F64))
        eo = _lib.EvalOut(outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), None)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.cfmm_blocked_eval(C.byref(cb), n, nu.data_ptr(), acc.data_ptr(), acc.data_ptr() + 8 * n,
                                     C.byref(eo) if out else None, None, 0, st), "cfmm_blocked_eval")
    torch.cuda.synchronize()
    return acc, outs


@pytest.mark.gpu
def test_native_fee_records_match_the_torch_function():
    for m, n in ((5000, 300), (1025, 300), (200_000, 4096)):
        hp, s = H.cp_host_pools(m, n, seed=m % 13)
        b = cf.PoolStore(hp).buckets[0]
        assert b.blocked and b.tables["tok_per_tile"] is None                            # the native path built it
        assert torch.equal(b.tables["fee"].cpu(), PL.fee_records(b.gamma_inv.cpu(), P)), (m, n)
        assert bool((b.tables["fee"][:, 0] > 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("fees,coded", [("tiers", "all"), ("uniform", "none"), ("mixed", "some")])
def test_evaluation_with_fee_records_equals_the_slab_evaluation(fees, coded):
    m, n = 600_000, 4096                                       # 586 tiles: two or three per CTA
    hp, s = _instance(m, n, 21, fees)
    st = cf.PoolStore(hp)
    b = st.buckets[0]
    nfee = b.tables["fee"][:, 0].cpu()
    assert {"all": bool((nfee > 0).all()), "none": bool((nfee == 0).all()),
            "some": bool((nfee[0::2] > 0).all() and (nfee[1::2] == 0).all())}[coded]
    bare = _lib.BlockedPairs.from_buffer_copy(b.c_blocked)
    bare.fee = None                                            # every tile streams its slab
    nu = torch.as_tensor(s["prices"] * np.exp(0.02 * np.random.default_rng(3).standard_normal(n)), **F64)
    for out in (False, True):
        a1, o1 = _eval(st.lib, b.c_blocked, n, nu, b.stride, out)
        a0, o0 = _eval(st.lib, bare, n, nu, b.stride, out)
        scale = float(a0[:n].abs().max())
        assert float((a1[:n] - a0[:n]).abs().max()) <= 1e-15 * scale                  # atomic order only
        # arb: one red.add per CTA into a single sum, larger than any psi entry; a few ulps of it move with the CTA order
        assert abs(float(a1[n] - a0[n])) <= 1e-14 * abs(float(a0[n]))
        if out:
            for x1, x0 in zip(o1, o0):                                                  # delta, lambda, hcoef
                assert torch.equal(x1.view(torch.int64), x0.view(torch.int64))


@pytest.mark.gpu
def test_persistent_solve_with_fee_records_takes_the_slab_path_and_matches_the_oracle():
    from oracle import c_oracle as CO
    m, n = 600_000, 4096
    hp, s = _instance(m, n, 22, "mixed")
    st = cf.PoolStore(hp)
    util = cf.Arbitrage(s["prices"])
    rf = cf.solve_pools(hp, util, tol=1e-8, store=st, want_trades=False)
    b = st.buckets[0]
    keep = b.c_blocked.fee
    b.c_blocked.fee = None
    try:
        r0 = cf.solve_pools(hp, util, tol=1e-8, store=st, want_trades=False)
    finally:
        b.c_blocked.fee = keep
    assert rf.info.history == [] and rf.status == r0.status == "optimal"                 # the persistent kernel
    assert (rf.iters, rf.evals, rf.hvps) == (r0.iters, r0.evals, r0.hvps)
    np.testing.assert_allclose(rf.nu, r0.nu, rtol=1e-9)
    nu_o, psi_o, ro = CO.solve_pairs(s["idx"], s["reserves"], s["gamma"], n, s["prices"], tol=1e-8)
    assert int(ro.status) == 0
    assert abs(rf.value - ro.primal_value) <= 1e-7 * abs(ro.primal_value)
    np.testing.assert_allclose(rf.nu, nu_o, rtol=1e-4)
