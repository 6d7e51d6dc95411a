// cfmm_small_pmm.cu -- the per-thread batch solver's instance for pool sets with DODO PMM pools.
//
// The same solve as cfmm_small.cu (cfmm_small::solve_one, one problem per thread or per warp), in its own kernel
// instance: DODO PMM pools (cfmm_small::pmm_pair, kind 12, one 4-f64 record {pi, k, B0, Q0} each after the E-CLP pools'
// records in `rec`) beside every kind the E-CLP instance takes, so the other eight instances keep their registers.
// A translation unit of its own, so the build compiles it in parallel with the others.
#include "cfmm_small_batch.cuh"

using namespace cfmm;

namespace {

template <int LANES>
__global__ void __launch_bounds__(kSmallThreads)
k_batch_solve_pmm(cfmm_small::Pools P, cfmm_batch B, cfmm_small::Params prm, int n, long long n_pools,
                  double* work, long long stride, const double* __restrict__ rec) {
    batch_solve_body<LANES, true, true, true, true, true, true, true, true>(P, B, prm, n, n_pools, work, stride, rec);
}

}  // namespace

extern "C" int cfmm_batch_solve_pmm(const cfmm_csr_pools* pools, const double* records, const cfmm_batch* batch,
                                    const cfmm_batch_params* prm, void* work, void* stream) {
    if (!records) return CFMM_E_NULL;
    const int rc = batch_solve_check(pools, batch, prm, work);
    if (rc != CFMM_OK || batch->n_problems == 0) return rc;
    cfmm_small::Pools P{pools->pool_ptr, pools->tok_idx, pools->reserves, pools->weights, pools->logrw, pools->gamma,
                        pools->kind};
    cfmm_small::Params q{prm->tol, prm->eps0, prm->eps_min, prm->eps_shrink, prm->floor_rel, prm->max_outer, prm->max_inner};
    const long long stride = padded(batch->n_problems) * g_batch_lanes;      // state slots = CUDA threads
    const unsigned grid = (unsigned)(stride / kSmallThreads);
    cudaStream_t st = (cudaStream_t)stream;
    if (g_batch_lanes == 32)
        k_batch_solve_pmm<32><<<grid, kSmallThreads, 0, st>>>(P, *batch, q, pools->n_tokens, pools->n_pools,
                                                              (double*)work, stride, records);
    else
        k_batch_solve_pmm<1><<<grid, kSmallThreads, 0, st>>>(P, *batch, q, pools->n_tokens, pools->n_pools,
                                                             (double*)work, stride, records);
    return check_launch();
}
