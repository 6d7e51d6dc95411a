// Test-only host build of cfmm_small::cryptoswap3 (csrc/cfmm_small.cuh), the per-pool three-coin cryptoswap math that
// k_eval_crypto3 and the per-thread solver run on the device, and of the solver's tricrypto instance.  Not part of the
// product.
#include <vector>
#include "../../cfmm_routing_code_b200/csrc/cfmm_small.cuh"

// R, c, nu: [m][3] (c = price scale / D); A, G, gamma: [m]; out D, L, w: [m][3] (w = edge weights w01, w02, w12),
// mask: [m]
extern "C" void tricrypto_host_pools(long long m, const double* R, const double* c, const double* A, const double* G,
                                     const double* gamma, const double* nu, double* D, double* L, double* w,
                                     unsigned* mask) {
    for (long long i = 0; i < m; ++i) {
        const double* r = R + 3 * i;
        const double* cc = c + 3 * i;
        const double* n = nu + 3 * i;
        mask[i] = cfmm_small::cryptoswap3(r[0], r[1], r[2], cc[0], cc[1], cc[2], A[i], G[i], gamma[i], n[0], n[1], n[2],
                                          D + 3 * i, L + 3 * i, w + 3 * i);
    }
}

// The per-thread solver's tricrypto instance (solve_one<1, true, true, true, true, true>, what k_batch_solve_tricrypto
// runs per thread) over the problems of a batch that share all pools; the arguments of cryptoswap_host.cpp.  No
// concentrated pools: the record pointer is null.
extern "C" int tricrypto_host_solve(int n_tokens, long long n_pools, const long long* pool_ptr, const int* tok,
                                    const double* R, const double* w, const double* logrw, const double* gamma,
                                    const unsigned char* kind, int n_problems, const double* c, const double* a,
                                    const unsigned char* flags, double* nu, double* psi, double* stats, double* delta,
                                    double* lam, double tol) {
    using namespace cfmm_small;
    Pools P{(const int64_t*)pool_ptr, tok, R, w, logrw, gamma, kind};
    Params prm{tol, 0.1, 1e-4, 0.5, 1e-12, 60, 100};
    const int64_t nnz = pool_ptr[n_pools];
    std::vector<double> work((size_t)work_doubles(n_tokens, nnz));
    for (int p = 0; p < n_problems; ++p) {
        Problem Q;
        Q.n = n_tokens;
        Q.p0 = 0; Q.p1 = n_pools; Q.off0 = 0;
        Q.c = c + (size_t)p * n_tokens; Q.a = a + (size_t)p * n_tokens; Q.flags = flags + (size_t)p * n_tokens;
        Q.delta = delta + (size_t)p * nnz; Q.lam = lam + (size_t)p * nnz;
        Stats r = solve_one<1, true, true, true, true, true>(P, Q, prm, nu + (size_t)p * n_tokens,
                                                             psi + (size_t)p * n_tokens, work.data(), 1);
        double* st = stats + 8 * p;
        st[0] = r.value; st[1] = r.dual; st[2] = r.gap; st[3] = r.infeas; st[4] = r.err;
        st[5] = r.iters; st[6] = r.evals; st[7] = r.status;
    }
    return 0;
}
