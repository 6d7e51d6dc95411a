// cfmm_solver.cu -- native outer loop for problems made of one token-blocked constant-product bucket.
//
// Same algorithm as solver.py (projected Newton in log-price coordinates, Jacobi-PCG on kernel Hessian-vector
// products, Armijo backtracking along nu*exp(alpha dt)), with the n_token-sized vector algebra fused into a
// handful of single-CTA kernels and the host loop in C++: what replaces `prob.solve()` (arbitrage.py:81-82) when
// every pool is a Uniswap-v2 style constant-product pool (arbitrage.py:68-70).  The per-pool work is still done by
// cfmm_blocked_eval / cfmm_blocked_hvp / cfmm_blocked_diag; this file only removes the Python/torch launch overhead
// (~20 ms per solve at 1M pools) around them.
#include <math.h>
#include <string.h>

#include "cfmm_dev.cuh"

using namespace cfmm;

namespace {

constexpr int kVT = 1024;      // threads of the single-CTA vector kernels

// scalar slots (device array, mirrored to pinned host memory)
enum { S_ABS_PG = 0, S_G, S_NU_ABS_GRAD, S_ERR, S_RZ, S_R0, S_STOP, S_GT, S_LIN, S_SLOPE, S_PRIMAL, S_INFEAS, S_ARB, S_COUNT = 16 };

__device__ __forceinline__ double block_sum(double v, double* sh) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = (threadIdx.x < kVT / 32) ? sh[threadIdx.x] : 0.0;
    if (threadIdx.x < 32) {
        t = warp_sum(t);
        if (threadIdx.x == 0) sh[32] = t;
    }
    __syncthreads();
    return sh[32];
}

__device__ __forceinline__ double block_max(double v, double* sh) {
    v = warp_max(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = (threadIdx.x < kVT / 32) ? sh[threadIdx.x] : 0.0;
    if (threadIdx.x < 32) {
        t = warp_max(t);
        if (threadIdx.x == 0) sh[32] = t;
    }
    __syncthreads();
    return sh[32];
}

struct Vecs {
    int n;
    const double *c, *a, *lb;
    const unsigned char *eq, *fixed;
    double *grad, *fr, *pg, *dt, *x, *r, *z, *p, *minv, *diag;
    double* sc;
};

// KKT residual / free set at (nu, acc = [psi | arb]):  err = sum_free |nu (a+psi)| / max(|g|, 1e-3 nu'|grad|)
__global__ void __launch_bounds__(kVT) k_kkt(Vecs V, const double* nu, const double* acc, double thr) {
    __shared__ double sh[33];
    double s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, m0 = 0, m1 = 0;
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        const double g = V.a[j] + acc[j];
        const bool near = (nu[j] <= V.lb[j] * (1.0 + thr)) && !V.eq[j];
        const bool act = V.fixed[j] || (near && g > 0.0);
        const double f = act ? 0.0 : 1.0;
        const double pg = nu[j] * g * f;
        V.grad[j] = g; V.fr[j] = f; V.pg[j] = pg;
        s0 += fabs(pg);
        s1 += (nu[j] - V.c[j]) * V.a[j];
        s2 += nu[j] * fabs(g);
        s3 += V.c[j] * acc[j];
        const double sl = acc[j] + V.a[j];
        const double viol = V.fixed[j] ? 0.0 : (V.eq[j] ? fabs(sl) : fmax(-sl, 0.0));
        s4 += nu[j] * viol;
        m0 = fmax(m0, fabs(g) * f);                          // per-token residual on the free set
        m1 = fmax(m1, fmax(fabs(V.a[j]), V.fixed[j] ? 0.0 : fabs(acc[j])));   // its scale: max(|a|_inf, constrained |psi_j|)
    }
    s0 = block_sum(s0, sh); s1 = block_sum(s1, sh); s2 = block_sum(s2, sh); s3 = block_sum(s3, sh);
    s4 = block_sum(s4, sh);
    m0 = block_max(m0, sh); m1 = block_max(m1, sh);
    if (threadIdx.x == 0) {
        const double g = s1 + acc[V.n];
        V.sc[S_ABS_PG] = s0; V.sc[S_G] = g; V.sc[S_NU_ABS_GRAD] = s2; V.sc[S_ARB] = acc[V.n];
        // max of the value-weighted residual and the per-token one (liquidation.py:77-80 constrains psi token by token)
        V.sc[S_ERR] = fmax(s0 / fmax(fmax(fabs(g), 1e-3 * s2), 1e-300), m0 / fmax(m1, 1e-300));
        V.sc[S_PRIMAL] = s3; V.sc[S_INFEAS] = s4 / fmax(fabs(g), 1e-300);
    }
}

// trial point of the line search: g_t and grad . (nu_t - nu)
__global__ void __launch_bounds__(kVT) k_trial(Vecs V, const double* nu, const double* nut, const double* acct) {
    __shared__ double sh[33];
    double s1 = 0, s2 = 0;
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        s1 += (nut[j] - V.c[j]) * V.a[j];
        s2 += V.grad[j] * (nut[j] - nu[j]);
    }
    s1 = block_sum(s1, sh); s2 = block_sum(s2, sh);
    if (threadIdx.x == 0) { V.sc[S_GT] = s1 + acct[V.n]; V.sc[S_LIN] = s2; }
}

__global__ void __launch_bounds__(kVT) k_cg_init(Vecs V) {
    __shared__ double sh[33];
    double rz = 0;
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        const double mi = V.fr[j] / fmax(V.diag[j], 1e-300);
        const double r = -V.pg[j];
        const double z = mi * r;
        V.minv[j] = mi; V.x[j] = 0.0; V.r[j] = r; V.z[j] = z; V.p[j] = z;
        rz += r * z;
    }
    rz = block_sum(rz, sh);
    if (threadIdx.x == 0) { V.sc[S_RZ] = rz; V.sc[S_R0] = sqrt(fmax(rz, 0.0)); V.sc[S_STOP] = (rz <= 0.0) ? 1.0 : 0.0; }
}

// one PCG iteration after y = Hs p:  stop flags: 1 = converged, 2 = (near-)zero curvature
__global__ void __launch_bounds__(kVT) k_cg_step(Vecs V, const double* y, double eta, int first) {
    __shared__ double sh[33];
    if (V.sc[S_STOP] != 0.0) return;                // an earlier iteration of this batch already finished the solve
    double pHp = 0, pdp = 0;
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        const double hp = y[j] * V.fr[j];
        pHp += V.p[j] * hp;
        pdp += V.p[j] * V.p[j] * fmax(V.diag[j], 1e-300);
    }
    pHp = block_sum(pHp, sh); pdp = block_sum(pdp, sh);
    const double rz = V.sc[S_RZ];
    if (pHp <= 1e-14 * pdp) {                       // homogeneity direction: g is linear along nu
        if (first)
            for (int j = threadIdx.x; j < V.n; j += kVT) V.x[j] = V.p[j];
        if (threadIdx.x == 0) V.sc[S_STOP] = 2.0;
        return;
    }
    const double alpha = rz / pHp;
    double rzn = 0;
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        const double hp = y[j] * V.fr[j];
        V.x[j] += alpha * V.p[j];
        const double r = V.r[j] - alpha * hp;
        const double z = V.minv[j] * r;
        V.r[j] = r; V.z[j] = z;
        rzn += r * z;
    }
    rzn = block_sum(rzn, sh);
    const bool done = (rzn <= 0.0) || (sqrt(fmax(rzn, 0.0)) <= eta * V.sc[S_R0]);
    if (!done) {
        const double beta = rzn / rz;
        for (int j = threadIdx.x; j < V.n; j += kVT) V.p[j] = V.z[j] + beta * V.p[j];
    }
    __syncthreads();
    if (threadIdx.x == 0) { V.sc[S_RZ] = rzn; V.sc[S_STOP] = done ? 1.0 : 0.0; }
}

// dt <- x if it is a descent direction in value units (pg . dt < 0), else scaled steepest descent; then at most kDtMax
// in every coordinate (solver.py DT_MAX: a truncated-CG step can be ~1e14 long, and every trial of the search would sit
// on k_step's +-20 clamp)
__global__ void __launch_bounds__(kVT) k_direction(Vecs V) {
    __shared__ double sh[33];
    double s = 0, mx = 0, xm = 0;
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        s += V.pg[j] * V.x[j]; mx = fmax(mx, fabs(V.pg[j])); xm = fmax(xm, fabs(V.x[j]));
    }
    s = block_sum(s, sh); mx = block_max(mx, sh); xm = block_max(xm, sh);
    const bool ok = isfinite(s) && s < 0.0;
    const double sc = ok && xm > kDtMax ? kDtMax / xm : 1.0;       // steepest descent is at most 1 long already
    for (int j = threadIdx.x; j < V.n; j += kVT) V.dt[j] = ok ? V.x[j] * sc : -V.pg[j] / fmax(mx, 1e-300);
    if (threadIdx.x == 0) V.sc[S_SLOPE] = s;
}

__global__ void __launch_bounds__(kVT) k_step(Vecs V, const double* nu, double alpha, double* nut) {
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        const double e = fmin(fmax(alpha * V.dt[j], -20.0), 20.0);
        const double v = fmax(nu[j] * exp(e), V.lb[j]);
        nut[j] = V.fixed[j] ? V.c[j] : v;
    }
}

__global__ void __launch_bounds__(kVT) k_bounds(int n, const double* c, const unsigned char* eq, const unsigned char* fixed,
                                                double floor_, double* lb, double* nu) {
    for (int j = threadIdx.x; j < n; j += kVT) {
        const double l = eq[j] ? floor_ : fmax(c[j], floor_);
        lb[j] = l;
        nu[j] = fixed[j] ? c[j] : fmax(nu[j], l);
    }
}

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// slab stride of a blocked layout (= BlockedArgs::M in cfmm_blocked.cu)
inline size_t hcoef_stride(const cfmm_blocked_pairs* b) { return (size_t)b->n_tiles * (size_t)b->pools_per_tile; }

}  // namespace

extern "C" {

int64_t cfmm_blocked_solve_work_bytes(const cfmm_blocked_pairs* b, int32_t n_tokens) {
    if (!b || n_tokens <= 0) return CFMM_E_SIZE;
    const size_t n = (size_t)n_tokens;
    const size_t M = hcoef_stride(b);
    size_t bytes = 0;
    bytes += align_up(8 * M);                 // hcoef
    bytes += 2 * align_up(8 * (n + 1));       // [psi | arb] ping-pong
    bytes += 2 * align_up(8 * n);             // y ping-pong
    bytes += 13 * align_up(8 * n);            // nut, lb, grad, fr, pg, dt, x, r, z, p, minv, diag, spare (sharded: local diag)
    bytes += align_up(8 * S_COUNT);
    bytes += 2 * align_up(8 * (n + 1)) + align_up(8 * n);      // sharded solve: all-reduced [psi | arb] ping-pong, reduced y
    return (int64_t)bytes;
}

int cfmm_blocked_solve(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* c, const double* a,
                       const uint8_t* eq, const uint8_t* pinned, double* nu, double* psi_out, void* work,
                       const cfmm_solve_params* prm, cfmm_solve_result* res, void* stream) {
    return cfmm_blocked_solve_peer(b, n_tokens, c, a, eq, pinned, nu, psi_out, work, prm, res, nullptr, stream);
}

int cfmm_blocked_solve_peer(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* c, const double* a,
                            const uint8_t* eq, const uint8_t* pinned, double* nu, double* psi_out, void* work,
                            const cfmm_solve_params* prm, cfmm_solve_result* res, cfmm_peer_ctx* peer, void* stream) {
    if (!b || !c || !a || !eq || !pinned || !nu || !psi_out || !work || !prm || !res) return CFMM_E_NULL;
    if (n_tokens <= 0 || b->n_tiles <= 0) return CFMM_E_SIZE;
    if (peer && (!peer->recv_acc_dev || !peer->recv_vec_dev)) return CFMM_E_NULL;
    if (peer && (peer->world < 2 || peer->world > 16 || peer->rank < 0 || peer->rank >= peer->world)) return CFMM_E_SIZE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int n = n_tokens;
    const size_t M = hcoef_stride(b);
    // ---- carve the work buffer
    unsigned char* w = static_cast<unsigned char*>(work);
    auto take = [&](size_t bytes) { unsigned char* p = w; w += align_up(bytes); return p; };
    double* hcoef = reinterpret_cast<double*>(take(8 * M));
    double* acc[2] = {reinterpret_cast<double*>(take(8 * (n + 1))), reinterpret_cast<double*>(take(8 * (n + 1)))};
    double* yb[2] = {reinterpret_cast<double*>(take(8 * n)), reinterpret_cast<double*>(take(8 * n))};
    double* nut = reinterpret_cast<double*>(take(8 * n));
    double* lb = reinterpret_cast<double*>(take(8 * n));
    Vecs V;
    V.n = n; V.c = c; V.a = a; V.lb = lb; V.eq = eq; V.fixed = pinned;
    V.grad = reinterpret_cast<double*>(take(8 * n)); V.fr = reinterpret_cast<double*>(take(8 * n));
    V.pg = reinterpret_cast<double*>(take(8 * n)); V.dt = reinterpret_cast<double*>(take(8 * n));
    V.x = reinterpret_cast<double*>(take(8 * n)); V.r = reinterpret_cast<double*>(take(8 * n));
    V.z = reinterpret_cast<double*>(take(8 * n)); V.p = reinterpret_cast<double*>(take(8 * n));
    V.minv = reinterpret_cast<double*>(take(8 * n)); V.diag = reinterpret_cast<double*>(take(8 * n));
    double* diag_loc = reinterpret_cast<double*>(take(8 * n));      // sharded: this rank's partial diagonal
    V.sc = reinterpret_cast<double*>(take(8 * S_COUNT));
    double* red[2] = {reinterpret_cast<double*>(take(8 * (n + 1))), reinterpret_cast<double*>(take(8 * (n + 1)))};
    double* yred = reinterpret_cast<double*>(take(8 * n));
    // sharded: all-reduce `local` (len doubles) into `out` on channel 0 ([psi | arb]) or 1 (n-vectors)
    auto reduce = [&](int chan, const double* local, int len, double* out) -> int {
        uint64_t& seq = chan == 0 ? peer->seq_acc : peer->seq_vec;
        ++seq;
        return cfmm_allreduce_ll(local, chan == 0 ? peer->recv_acc_dev : peer->recv_vec_dev, peer->rank, peer->world, len,
                                 (int64_t)(seq % 3) * peer->world * len, len, out, seq, st);
    };

    static thread_local double* hsc = nullptr;          // pinned mirror of the scalar slots
    if (!hsc && cudaHostAlloc(&hsc, 8 * S_COUNT, cudaHostAllocDefault) != cudaSuccess) return CFMM_E_CUDA;
    auto fetch = [&]() {
        cudaMemcpyAsync(hsc, V.sc, 8 * S_COUNT, cudaMemcpyDeviceToHost, st);
        return cudaStreamSynchronize(st) == cudaSuccess;
    };
    int ai = 0, yi = 0, evals = 0, hvps = 0, rc = 0;
    cudaMemsetAsync(acc[0], 0, 8 * (n + 1), st);
    cudaMemsetAsync(yb[0], 0, 8 * n, st);
    cudaMemsetAsync(V.sc, 0, 8 * S_COUNT, st);
    k_bounds<<<1, kVT, 0, st>>>(n, c, eq, pinned, prm->nu_floor, lb, nu);
    cfmm_eval_out out;
    out.delta = nullptr; out.lambda = nullptr; out.hcoef = hcoef; out.hmask = nullptr;
    // evaluate at `x` into acc[ai]; returns the buffer used
    auto eval = [&](const double* x) -> double* {
        double* cur = acc[ai];
        double* nxt = acc[ai ^ 1];
        ai ^= 1;
        rc = cfmm_blocked_eval(b, n, x, cur, cur + n, &out, nxt, n + 1, st);
        ++evals;
        if (peer && !rc) {                       // every rank continues with the sum over the shards
            rc = reduce(0, cur, n + 1, red[ai]);
            return red[ai];
        }
        return cur;
    };
    double* cur_nu = nu;           // the caller's buffer and `nut` swap roles as steps are accepted
    double* oth_nu = nut;
    double* cur_acc = eval(cur_nu);
    if (rc) return rc;
    double err = INFINITY;
    int iters = 0, status = 1;     // 0 optimal, 1 max_iter, 2 stalled
    bool have_kkt = false;         // V.grad / fr / pg and the host scalars describe (cur_nu, cur_acc)
    constexpr int kCgBatch = 3;    // PCG iterations launched per host synchronisation
    for (; iters < prm->max_iter;) {
        ++iters;
        const double thr = fmin(1e-2, fmax(1e-3 * (isfinite(err) ? err : 1e-2), 1e-14));     // active-set width (see solver.py)
        if (!have_kkt) {
            k_kkt<<<1, kVT, 0, st>>>(V, cur_nu, cur_acc, thr);
            if (!fetch()) return CFMM_E_CUDA;
        }
        err = hsc[S_ERR];
        const double g0 = hsc[S_G];
        if (err <= prm->tol) { status = 0; break; }
        // ---- Newton direction: Jacobi-PCG on Hs dt = -(nu * grad) over the free set
        double* dg = peer ? diag_loc : V.diag;
        cudaMemsetAsync(dg, 0, 8 * n, st);
        rc = cfmm_blocked_diag(b, n, hcoef, dg, st);
        if (!rc && peer) rc = reduce(1, dg, n, V.diag);
        if (rc) return rc;
        k_cg_init<<<1, kVT, 0, st>>>(V);
        const double eta = fmin(0.1, sqrt(err));
        for (int k = 0; k < prm->cg_max;) {
            // a batch of iterations per synchronisation; k_cg_step turns into a no-op once the stop flag is set
            for (int bi = 0; bi < kCgBatch && k < prm->cg_max; ++bi, ++k) {
                double* y = yb[yi];
                double* ynx = yb[yi ^ 1];
                yi ^= 1;
                rc = cfmm_blocked_hvp(b, n, hcoef, V.p, y, ynx, st);
                if (!rc && peer) { rc = reduce(1, y, n, yred); y = yred; }
                if (rc) return rc;
                ++hvps;
                k_cg_step<<<1, kVT, 0, st>>>(V, y, eta, k == 0);
            }
            if (!fetch()) return CFMM_E_CUDA;
            if (hsc[S_STOP] != 0.0) break;
        }
        k_direction<<<1, kVT, 0, st>>>(V);
        // ---- projected Armijo backtracking along nu * exp(alpha dt); the KKT data of the trial point is computed
        // speculatively behind it, so an accepted step (the rule) costs one synchronisation
        double alpha = 1.0, lin1 = 0.0;
        bool ok = false;
        for (int ls = 0; ls < 50; ++ls) {
            k_step<<<1, kVT, 0, st>>>(V, cur_nu, alpha, oth_nu);
            double* acct = eval(oth_nu);
            if (rc) return rc;
            k_trial<<<1, kVT, 0, st>>>(V, cur_nu, oth_nu, acct);          // uses the OLD gradient: before k_kkt
            k_kkt<<<1, kVT, 0, st>>>(V, oth_nu, acct, thr);
            if (!fetch()) return CFMM_E_CUDA;
            const double gt = hsc[S_GT], lin = hsc[S_LIN];
            if (ls == 0) lin1 = lin;                 // predicted decrease of the FULL step
            if (gt <= g0 + 1e-4 * lin) { ok = true; cur_acc = acct; break; }
            if (fabs(gt - g0) <= 1e-13 * fabs(g0) || fabs(lin1) <= 1e-9 * fabs(g0)) {
                // the (full) step is below what g resolves in fp64 (a sum of cancelling flows): judge it by the KKT
                // residual instead (same rule as solver.py)
                if (hsc[S_ERR] < 0.99 * err) { ok = true; cur_acc = acct; break; }
                if (alpha < 1e-3) break;
            }
            // rejected: the gradient buffers now belong to the trial -- restore them at the current point
            cur_acc = eval(cur_nu);
            if (rc) return rc;
            k_kkt<<<1, kVT, 0, st>>>(V, cur_nu, cur_acc, thr);
            alpha *= 0.5;
        }
        if (!ok) { status = 2; break; }
        double* t = cur_nu; cur_nu = oth_nu; oth_nu = t;
        have_kkt = true;
    }
    if (status != 0) {
        // max_iter or stalled: make buffers and host scalars consistent with the accepted point
        cur_acc = eval(cur_nu);
        if (rc) return rc;
        k_kkt<<<1, kVT, 0, st>>>(V, cur_nu, cur_acc, 1e-14);
        if (!fetch()) return CFMM_E_CUDA;
        err = hsc[S_ERR];
    }
    if (cur_nu != nu) cudaMemcpyAsync(nu, cur_nu, 8 * n, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(psi_out, cur_acc, 8 * n, cudaMemcpyDeviceToDevice, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) { g_last_err = cudaGetLastError(); return CFMM_E_CUDA; }
    res->dual_value = hsc[S_G];
    res->primal_value = hsc[S_PRIMAL];
    res->gap = (hsc[S_G] - hsc[S_PRIMAL]) / fmax(fabs(hsc[S_G]), 1e-300);
    res->primal_infeas = hsc[S_INFEAS];
    res->err = err;
    res->iters = iters; res->evals = evals; res->hvps = hvps; res->status = status;
    return CFMM_OK;
}

}  // extern "C"
