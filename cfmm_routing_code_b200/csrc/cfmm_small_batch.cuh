// cfmm_small_batch.cuh -- the per-thread batch solver's kernel body, shared by the translation units that instantiate it
// (cfmm_small.cu: the plain and StableSwap instances; cfmm_small_ladder.cu: the concentrated one; cfmm_small_crypto.cu:
// the cryptoswap one; cfmm_small_tricrypto.cu: the three-coin cryptoswap one; cfmm_small_bins.cu: the price-bin one).
// Each includer gets its own copy in an anonymous namespace; the lane setting and the argument checks live in
// cfmm_small.cu.
#pragma once
#include "cfmm_dev.cuh"
#include "cfmm_small.cuh"

namespace cfmm {
extern int g_batch_lanes;            // cfmm_set_batch_lanes: 1 | 32
// the checks every cfmm_batch_solve* entry makes before its launch: CFMM_OK, or the error code to return
int batch_solve_check(const cfmm_csr_pools* pools, const cfmm_batch* batch, const cfmm_batch_params* prm, void* work);
}  // namespace cfmm

namespace {

constexpr int kSmallThreads = 32;     // one warp per CTA: a sweep of 50 problems spreads over 2 SMs, 10^5 over all 132

// LANES = 1: one problem per thread (throughput: 10^5 .. 10^6 problems).  LANES = 32: one problem per warp, the pool
// loop of every evaluation split over the lanes (latency: a handful of problems, or problems with hundreds of pools);
// each lane keeps its own copy of the state at work[(p * LANES + lane)], so `stride` counts lanes, not problems.
// STABLE: also evaluate StableSwap pools (k_batch_solve_stable); without it such a pool makes its problem status 3.
// STABLE_N: StableSwap pools of 2..8 coins (k_batch_solve_stable_n).  LADDER: concentrated pools too, their records in
// `rec` (k_batch_solve_ladder).  CRYPTO: two-coin cryptoswap pools too (k_batch_solve_crypto).  CRYPTO3: three-coin
// cryptoswap pools too (k_batch_solve_tricrypto).  BINS: price-bin pools too (k_batch_solve_bins).  ECLP: E-CLP pools
// too (k_batch_solve_eclp).  PMM: DODO PMM pools too (k_batch_solve_pmm).
template <int LANES, bool STABLE, bool STABLE_N = false, bool LADDER = false, bool CRYPTO = false, bool CRYPTO3 = false,
          bool BINS = false, bool ECLP = false, bool PMM = false>
__device__ __forceinline__ void batch_solve_body(const cfmm_small::Pools& P, const cfmm_batch& B, const cfmm_small::Params& prm,
                                                 int n, long long n_pools, double* work, long long stride,
                                                 const double* rec = nullptr) {
    const long long gt = (long long)blockIdx.x * kSmallThreads + threadIdx.x;
    const long long p = LANES == 1 ? gt : gt / LANES;
    const int lane = LANES == 1 ? 0 : (int)(gt % LANES);
    if (p >= B.n_problems) return;
    cfmm_small::Problem Q;
    Q.n = n;
    Q.p0 = B.pool_range ? B.pool_range[2 * p] : 0;
    Q.p1 = B.pool_range ? B.pool_range[2 * p + 1] : n_pools;
    double* st = B.stats + 8 * p;
    if (Q.p0 < 0 || Q.p1 > n_pools || Q.p0 > Q.p1) {
        if (lane == 0) {
            for (int x = 0; x < 7; ++x) st[x] = NAN;
            st[7] = 3.0;
        }
        return;
    }
    Q.off0 = P.pool_ptr[Q.p0];
    Q.c = B.c + p * n;
    Q.a = B.a + p * n;
    Q.flags = B.flags + p * n;
    Q.delta = B.delta ? B.delta + p * B.trade_stride : nullptr;
    Q.lam = B.lambda ? B.lambda + p * B.trade_stride : nullptr;
    const cfmm_small::Stats r = cfmm_small::solve_one<LANES, STABLE, STABLE_N, LADDER, CRYPTO, CRYPTO3, BINS, ECLP, PMM>(
        P, Q, prm, B.nu + p * n, B.psi + p * n, work + (LANES == 1 ? p : p * LANES + lane), stride, lane, rec);
    if (lane == 0) {
        st[0] = r.value; st[1] = r.dual; st[2] = r.gap; st[3] = r.infeas; st[4] = r.err;
        st[5] = (double)r.iters; st[6] = (double)r.evals; st[7] = (double)r.status;
    }
}

inline long long padded(long long b) { return (b + kSmallThreads - 1) / kSmallThreads * kSmallThreads; }

}  // namespace
