"""The one-word-per-pool blocked layout (csrc/cfmm_blocked.cuh): pool words, the row-table bound, and agreement of the
native builder (csrc/cfmm_layout.cu) with the torch builder (pools.build_blocked_pairs)."""
import numpy as np
import pytest
import torch

import cfmm_routing_code_b200 as cf
from cfmm_routing_code_b200 import _lib
from cfmm_routing_code_b200 import instances as I
from cfmm_routing_code_b200 import pools as PL

import helpers as H


def test_pool_words_unpack_to_ids_and_flow_positions():
    P = 1024
    lid0 = torch.tensor([0, 1023, 5, 0])
    lid1 = torch.tensor([1023, 0, 7, 0])
    p1 = torch.tensor([3, 1023, 0, 1027 % P])
    pw = (lid0 | lid1 << 10 | p1 << 20).to(torch.int32)
    lid, pos = PL.unpack_pool_words(pw, P)
    assert torch.equal(lid.to(torch.int64), lid0 | lid1 << 16)
    assert torch.equal(pos.to(torch.int64) & 0xffff, torch.arange(4))                 # slot 0: the pool's own index
    assert torch.equal(pos.to(torch.int64) >> 16, P + p1)                               # slot 1: second half of the array


def test_torch_builder_stores_one_word_per_pool():
    lib = _lib.load()
    P, rs, ts, cap = PL.blocked_layout_info(lib)
    s = I.synth_const_product(5000, 300, 0)
    idx = torch.as_tensor(s["idx"].T.astype(np.int64).copy())
    order, res, t = PL.build_blocked_pairs(idx, 300, P, rs, ts, cap)
    assert t["pw"].dtype == torch.int32 and t["pw"].numel() == t["M"]
    assert set(t) >= {"pw", "lid", "pos", "rows", "tok", "desc"}
    w = t["pw"].to(torch.int64)
    assert int(w.max()) < 2 ** 30 and int(((w >> 20) & 0x3ff).max()) < P
    nq = len(order)
    pad = torch.arange(nq, t["M"]) % P
    assert torch.equal(w[nq:], pad << 20)                # padding pools: zero flows to g[l] and g[P + l], no row covers them


def test_tiles_needing_more_rows_than_the_table_go_to_the_residual():
    """a ring of 1024 pools over 1024 tokens: one tile of 1024 tokens (allowed), but every token is a run of length 1 in
    both halves of the flow array -> 2048 rows, more than the row table holds"""
    lib = _lib.load()
    P, rs, ts, cap = PL.blocked_layout_info(lib)
    n = 1024
    a = torch.arange(n, dtype=torch.int64)
    idx = torch.stack([a, (a + 1) % n])
    order, res, t = PL.build_blocked_pairs(idx, n, P, rs, ts, cap)
    assert len(order) == 0 and t is None and sorted(res.tolist()) == list(range(n))


@pytest.mark.gpu
def test_native_and_torch_builders_build_the_same_layout():
    lib = _lib.load()
    P, rs, ts, cap = PL.blocked_layout_info(lib)
    for m, n in ((5000, 300), (1025, 300), (200_000, 4096)):
        hp, _ = H.cp_host_pools(m, n, seed=m % 13)
        b = cf.PoolStore(hp).buckets[0]
        assert b.blocked and b.tables["tok_per_tile"] is None                          # the native path built it
        idx = torch.as_tensor(hp.tok_idx.reshape(-1, 2).T.astype(np.int64).copy(), device="cuda")
        order, res, t = PL.build_blocked_pairs(idx, n, P, rs, ts, cap)
        assert len(res) == 0 and torch.equal(b.order.to(torch.int64), order)
        assert torch.equal(b.tables["pw"], t["pw"]) and torch.equal(b.tables["desc"], t["desc"])
        d = t["desc"].cpu()
        for tile in range(t["n_tiles"]):
            ntok, nrow = int(d[tile, 0]), int(d[tile, 1])
            assert torch.equal(b.tables["rows"][tile, :nrow], t["rows"][tile, :nrow])
            assert torch.equal(b.tables["tok"][tile, :ntok], t["tok"][tile, :ntok])


@pytest.mark.gpu
def test_native_builder_hands_row_overflow_to_the_general_builder():
    """the ring above through PoolStore: the native builder reports the tile, the pools land in a plain bucket, and the
    evaluation still matches the oracle"""
    from oracle import cfmm_oracle as O
    n = 1024
    a = np.arange(n)
    rng = np.random.default_rng(5)
    hp = cf.HostPools.from_pairs(n, np.stack([a, (a + 1) % n], 1), rng.uniform(1.0, 2.0, (n, 2)), np.full(n, 0.997))
    st = cf.PoolStore(hp)
    assert sum(bk.m for bk in st.buckets) == n
    assert sum(bk.m for bk in st.buckets if getattr(bk, "blocked", False)) == 0
    nu = np.exp(0.1 * rng.standard_normal(n))
    acc = st.evaluate(torch.as_tensor(nu, dtype=torch.float64, device="cuda")).cpu().numpy()
    Po = O.Pools(n, hp.pool_ptr, hp.tok_idx, hp.reserves, hp.weights, hp.gamma, hp.kind)
    ev = O.evaluate(O.Buckets(Po), nu)
    assert np.max(np.abs(acc[:-1] - ev["psi"])) <= 1e-9 * np.abs(ev["psi"]).max()
