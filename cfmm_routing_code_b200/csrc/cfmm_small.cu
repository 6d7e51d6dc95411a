// cfmm_small.cu -- batches of SMALL routing problems, one problem per thread, the whole solve in one launch.
//
// Replaces the python loop of two-asset.py:40-100 (50 cvxpy problems built and solved one after the other) and, more
// generally, N independent prob.solve() calls (arbitrage.py:81-82) on problems of the reference's own size (5 pools,
// 3-5 tokens) by ONE kernel: thread p runs cfmm_small::solve_one on problem p.  Parallelism is over problems; the pool
// data of a shared-pool sweep is read by all lanes at the same address (one broadcast transaction per warp), the
// per-problem state is element-interleaved so lane accesses coalesce.
#include "cfmm_small_batch.cuh"

using namespace cfmm;

namespace {

template <int LANES>
__global__ void __launch_bounds__(kSmallThreads)
k_batch_solve(cfmm_small::Pools P, cfmm_batch B, cfmm_small::Params prm, int n, long long n_pools, double* work,
              long long stride) {
    batch_solve_body<LANES, false>(P, B, prm, n, n_pools, work, stride);
}

// the same solve for pool sets that hold StableSwap pools: its own instance, so that the Newton loops of
// cfmm_small::stableswap_pair do not raise k_batch_solve's register count for problems without them
template <int LANES>
__global__ void __launch_bounds__(kSmallThreads)
k_batch_solve_stable(cfmm_small::Pools P, cfmm_batch B, cfmm_small::Params prm, int n, long long n_pools, double* work,
                     long long stride) {
    batch_solve_body<LANES, true>(P, B, prm, n, n_pools, work, stride);
}

// and for pool sets with StableSwap pools of more than two coins: a third instance, so that the n-coin evaluation
// (cfmm_small::stableswap_n) leaves the other two instances' registers as they are
template <int LANES>
__global__ void __launch_bounds__(kSmallThreads)
k_batch_solve_stable_n(cfmm_small::Pools P, cfmm_batch B, cfmm_small::Params prm, int n, long long n_pools, double* work,
                       long long stride) {
    batch_solve_body<LANES, true, true>(P, B, prm, n, n_pools, work, stride);
}

}  // namespace

int cfmm::g_batch_lanes = 1;

int cfmm::batch_solve_check(const cfmm_csr_pools* pools, const cfmm_batch* batch, const cfmm_batch_params* prm,
                            void* work) {
    if (!pools || !batch || !prm) return CFMM_E_NULL;
    if (batch->n_problems == 0) return CFMM_OK;
    if (!pools->pool_ptr || !pools->tok_idx || !pools->reserves || !pools->weights || !pools->logrw || !pools->gamma ||
        !pools->kind || !batch->c || !batch->a || !batch->flags || !batch->nu || !batch->psi || !batch->stats || !work)
        return CFMM_E_NULL;
    if ((batch->delta == nullptr) != (batch->lambda == nullptr)) return CFMM_E_NULL;
    if (batch->n_problems < 0 || pools->n_pools < 0 || pools->nnz < 0 || batch->trade_stride < 0) return CFMM_E_SIZE;
    if (pools->n_tokens < 1 || pools->n_tokens > cfmm_small::NTOK_MAX) return CFMM_E_KIND;
    return CFMM_OK;
}

extern "C" int64_t cfmm_batch_solve_work_bytes(const cfmm_csr_pools* pools, int32_t n_problems, int64_t nnz_max) {
    if (!pools) return CFMM_E_NULL;
    if (n_problems < 0 || pools->n_tokens < 1 || pools->n_tokens > cfmm_small::NTOK_MAX || pools->nnz < 0) return CFMM_E_SIZE;
    const int64_t cap = (nnz_max > 0 && nnz_max < pools->nnz) ? nnz_max : pools->nnz;    // slots of the largest problem
    return (int64_t)sizeof(double) * cfmm_small::work_doubles(pools->n_tokens, cap) * padded(n_problems) * g_batch_lanes;
}

extern "C" int cfmm_set_batch_lanes(int32_t lanes) {
    if (lanes != 1 && lanes != 32) return CFMM_E_KIND;
    g_batch_lanes = lanes;
    return CFMM_OK;
}

namespace {
int batch_solve(const cfmm_csr_pools* pools, const cfmm_batch* batch, const cfmm_batch_params* prm, void* work,
                void* stream, int stable) {
    const int rc = cfmm::batch_solve_check(pools, batch, prm, work);
    if (rc != CFMM_OK || batch->n_problems == 0) return rc;
    cfmm_small::Pools P{pools->pool_ptr, pools->tok_idx, pools->reserves, pools->weights, pools->logrw, pools->gamma,
                        pools->kind};
    cfmm_small::Params q{prm->tol, prm->eps0, prm->eps_min, prm->eps_shrink, prm->floor_rel, prm->max_outer, prm->max_inner};
    const long long stride = padded(batch->n_problems) * g_batch_lanes;      // state slots = CUDA threads
    const unsigned grid = (unsigned)(stride / kSmallThreads);
    cudaStream_t st = (cudaStream_t)stream;
    if (stable == 2) {
        if (g_batch_lanes == 32)
            k_batch_solve_stable_n<32><<<grid, kSmallThreads, 0, st>>>(P, *batch, q, pools->n_tokens, pools->n_pools,
                                                                       (double*)work, stride);
        else
            k_batch_solve_stable_n<1><<<grid, kSmallThreads, 0, st>>>(P, *batch, q, pools->n_tokens, pools->n_pools,
                                                                      (double*)work, stride);
    } else if (stable == 1) {
        if (g_batch_lanes == 32)
            k_batch_solve_stable<32><<<grid, kSmallThreads, 0, st>>>(P, *batch, q, pools->n_tokens, pools->n_pools,
                                                                     (double*)work, stride);
        else
            k_batch_solve_stable<1><<<grid, kSmallThreads, 0, st>>>(P, *batch, q, pools->n_tokens, pools->n_pools,
                                                                    (double*)work, stride);
    } else if (g_batch_lanes == 32) {
        k_batch_solve<32><<<grid, kSmallThreads, 0, st>>>(P, *batch, q, pools->n_tokens, pools->n_pools, (double*)work,
                                                          stride);
    } else {
        k_batch_solve<1><<<grid, kSmallThreads, 0, st>>>(P, *batch, q, pools->n_tokens, pools->n_pools, (double*)work,
                                                         stride);
    }
    return check_launch();
}
}  // namespace

extern "C" int cfmm_batch_solve(const cfmm_csr_pools* pools, const cfmm_batch* batch, const cfmm_batch_params* prm,
                                void* work, void* stream) {
    return batch_solve(pools, batch, prm, work, stream, 0);
}

extern "C" int cfmm_batch_solve_stableswap(const cfmm_csr_pools* pools, const cfmm_batch* batch,
                                           const cfmm_batch_params* prm, void* work, void* stream) {
    return batch_solve(pools, batch, prm, work, stream, 1);
}

extern "C" int cfmm_batch_solve_stableswap_n(const cfmm_csr_pools* pools, const cfmm_batch* batch,
                                             const cfmm_batch_params* prm, void* work, void* stream) {
    return batch_solve(pools, batch, prm, work, stream, 2);
}

