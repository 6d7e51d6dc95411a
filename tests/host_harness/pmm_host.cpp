// Test-only host build of cfmm_small::pmm_pair (csrc/cfmm_small.cuh), the DODO PMM math that k_eval_pair and the
// per-thread solver run on the device, and of the solver's PMM instance.  Not part of the product.
#include <vector>
#include "../../cfmm_routing_code_b200/csrc/cfmm_small.cuh"

// R [m][2] = (B, Q); P [m][4] = (pi, k, B0, Q0); gamma, nu0, nu1 [m]; D, L [m][2]; hc [m]
extern "C" void pmm_host_pools(long long m, const double* R, const double* P, const double* gamma, const double* nu0,
                               const double* nu1, double* D, double* L, double* hc) {
    for (long long i = 0; i < m; ++i) {
        const double* q = P + 4 * i;
        cfmm_small::pmm_pair(R[2 * i], R[2 * i + 1], q[0], q[1], q[2], q[3], gamma[i], nu0[i], nu1[i], D + 2 * i,
                             L + 2 * i, hc[i]);
    }
}

// The per-thread solver's PMM instance (solve_one<1, true, true, true, true, true, true, true, true>, what
// k_batch_solve_pmm runs per thread) over problems that share all pools; the CSR arrays of cfmm_csr_pools plus the
// records.
extern "C" int pmm_host_solve(int n_tokens, long long n_pools, const long long* pool_ptr, const int* tok,
                              const double* R, const double* w, const double* logrw, const double* gamma,
                              const unsigned char* kind, const double* rec, int n_problems, const double* c,
                              const double* a, const unsigned char* flags, double* nu, double* psi, double* stats,
                              double* delta, double* lam, double tol) {
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
        Stats r = solve_one<1, true, true, true, true, true, true, true, true>(P, Q, prm, nu + (size_t)p * n_tokens,
                                                                                psi + (size_t)p * n_tokens, work.data(),
                                                                                1, 0, rec);
        double* st = stats + 8 * p;
        st[0] = r.value; st[1] = r.dual; st[2] = r.gap; st[3] = r.infeas; st[4] = r.err;
        st[5] = r.iters; st[6] = r.evals; st[7] = r.status;
    }
    return 0;
}
