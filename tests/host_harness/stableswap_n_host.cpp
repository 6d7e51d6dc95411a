// Test-only host build of cfmm_small::stableswap_n (csrc/cfmm_small.cuh), the n-coin StableSwap math that
// k_eval_stable_n and the per-thread solver run on the device, of its O(k) Hessian product, and of the solver's n-coin
// instance.  Not part of the product.
#include <vector>
#include "../../cfmm_routing_code_b200/csrc/cfmm_small.cuh"

// R, r, nu, D, L, h: [m][k] row-major; A, Dv, gamma: [m]; mask: [m]
extern "C" void stablen_host_pools(long long m, int k, const double* R, const double* r, const double* A,
                                   const double* Dv, const double* gamma, const double* nu, double* D, double* L,
                                   double* h, unsigned* mask) {
    for (long long i = 0; i < m; ++i)
        mask[i] = cfmm_small::stableswap_n<cfmm_small::KMAX>(k, R + i * k, r + i * k, A[i], Dv[i], gamma[i], nu + i * k,
                                                             D + i * k, L + i * k, h + i * k);
}

// y = Hs z per pool from the per-slot h: h, z, y [m][k]
extern "C" void stablen_host_hvp(long long m, int k, const double* h, const double* z, double* y) {
    for (long long i = 0; i < m; ++i) cfmm_small::stablen_hvp<cfmm_small::KMAX>(k, h + i * k, z + i * k, y + i * k);
}

// the two-coin pair function on the same pools (k = 2), for the cross-check
extern "C" void stablen_host_pairs(long long m, const double* R, const double* r, const double* A, const double* Dv,
                                   const double* gamma, const double* nu, double* D, double* L, double* hc) {
    for (long long i = 0; i < m; ++i)
        cfmm_small::stableswap_pair(R[2 * i], R[2 * i + 1], r[2 * i], r[2 * i + 1], A[i], Dv[i], gamma[i], nu[2 * i],
                                    nu[2 * i + 1], D + 2 * i, L + 2 * i, hc[i]);
}

// The per-thread solver's n-coin instance (solve_one<1, true, true>, what k_batch_solve_stable_n runs per thread) over
// the problems of a batch that share all pools; the arguments of stableswap_host.cpp's stableswap_host_solve.
extern "C" int stablen_host_solve(int n_tokens, long long n_pools, const long long* pool_ptr, const int* tok,
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
        Stats r = solve_one<1, true, true>(P, Q, prm, nu + (size_t)p * n_tokens, psi + (size_t)p * n_tokens, work.data(), 1);
        double* st = stats + 8 * p;
        st[0] = r.value; st[1] = r.dual; st[2] = r.gap; st[3] = r.infeas; st[4] = r.err;
        st[5] = r.iters; st[6] = r.evals; st[7] = r.status;
    }
    return 0;
}
