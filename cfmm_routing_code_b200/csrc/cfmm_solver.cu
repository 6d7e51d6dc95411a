// cfmm_solver.cu -- native outer loop for a market of any pool kinds: plain buckets (cfmm_bucket, every CFMM_KIND_*)
// plus at most one token-blocked constant-product bucket.
//
// Same algorithm as solver.py (projected Newton in log-price coordinates, Jacobi-PCG on kernel Hessian-vector
// products or a dense Cholesky with a Levenberg-Marquardt ladder, the active-set look-ahead, Armijo backtracking along
// nu*exp(alpha dt), the method of multipliers on constant-sum fills), with the n_token-sized vector algebra fused into
// a handful of single-CTA kernels and the host loop in C++: what replaces `prob.solve()` (arbitrage.py:81-82).  The
// per-pool work is still done by cfmm_arb_eval / cfmm_blocked_eval and their Hessian kernels, issued in the order
// PoolStore issues them; this file only removes the Python/torch launch overhead around them.
// cfmm_blocked_solve(_peer) is the one-blocked-bucket case (Jacobi-PCG, no read-back pass).
#include <math.h>
#include <string.h>

#include "cfmm_dev.cuh"

using namespace cfmm;

namespace {

constexpr int kVT = 1024;      // threads of the single-CTA vector kernels

// scalar slots (device array, mirrored to pinned host memory)
enum { S_ABS_PG = 0, S_G, S_NU_ABS_GRAD, S_ERR, S_RZ, S_R0, S_STOP, S_GT, S_LIN, S_SLOPE, S_PRIMAL, S_INFEAS, S_ARB,
       S_INFO, S_DMAX, S_DBAR, S_CNT, S_MOVE,
       S_SUM_A = 20, S_SUM_B = 25,    // two k_sums blocks of 5: (nu-c)'a, c'psi, nu'psi, nu'viol, arb
       S_COUNT = 32 };
constexpr int kNB = 64;         // panel width of the blocked Cholesky
constexpr int kDenseMax = 4096; // largest dense Newton system (k_newton_solve keeps the right-hand side in shared memory)
constexpr double kLmShifts[6] = {1e-14, 1e-8, 1e-6, 1e-4, 1e-2, 1.0};   // solver.py LM_SHIFTS

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

// ---- market loop: vectors of the read-back and the multiplier passes, log(nu) of the weighted pools

// sc[base..base+4] = (nu-c)'a, c'psi, nu'psi, nu'viol, arb  of acc = [psi | arb]  (solver.py's final certificate)
__global__ void __launch_bounds__(kVT) k_sums(Vecs V, const double* nu, const double* acc, int base) {
    __shared__ double sh[33];
    double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        s0 += (nu[j] - V.c[j]) * V.a[j];
        s1 += V.c[j] * acc[j];
        s2 += nu[j] * acc[j];
        const double sl = acc[j] + V.a[j];
        s3 += nu[j] * (V.fixed[j] ? 0.0 : (V.eq[j] ? fabs(sl) : fmax(-sl, 0.0)));
    }
    s0 = block_sum(s0, sh); s1 = block_sum(s1, sh); s2 = block_sum(s2, sh); s3 = block_sum(s3, sh);
    if (threadIdx.x == 0) {
        V.sc[base] = s0; V.sc[base + 1] = s1; V.sc[base + 2] = s2; V.sc[base + 3] = s3; V.sc[base + 4] = acc[V.n];
    }
}

__global__ void __launch_bounds__(kVT) k_log(int n, const double* x, double* y) {
    for (int j = threadIdx.x; j < n; j += kVT) y[j] = log(x[j]);
}

// ---- dense Newton direction (solver.py newton_dir, linear_solver="dense")

// sc[S_DBAR] = mean free diagonal of H0 = Hs masked to the free set fr (at least 1e-300)
__global__ void __launch_bounds__(kVT) k_dense_dbar(int n, const double* Hs, const double* fr, double* sc) {
    __shared__ double sh[33];
    double s = 0, k = 0;
    for (int j = threadIdx.x; j < n; j += kVT) {
        s += Hs[(size_t)j * n + j] * fr[j] * fr[j];
        k += fr[j];
    }
    s = block_sum(s, sh); k = block_sum(k, sh);
    if (threadIdx.x == 0) sc[S_DBAR] = fmax(s / fmax(k, 1.0), 1e-300);
}

// W = H0 + diag((1 - fr) + shift * dbar * fr), H0 = Hs fr fr'.  Every rung starts again from the unmodified Hs.  W is
// read as column-major (element (i, j) at W[j n + i]); Hs is symmetric, so this is Hs's own row-major layout.
__global__ void k_dense_assemble(int n, const double* Hs, const double* fr, double shift, const double* sc, double* W) {
    const double sd = shift * sc[S_DBAR];
    const size_t nn = (size_t)n * n;
    for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < nn; q += (size_t)gridDim.x * blockDim.x) {
        const int j = (int)(q / n), i = (int)(q % n);
        double v = Hs[q] * fr[i] * fr[j];
        if (i == j) v += (1.0 - fr[i]) + sd * fr[i];
        W[q] = v;
    }
}

// Blocked right-looking Cholesky, A = L L', in place on the lower triangle of the column-major W; the upper triangle is
// not read.  Panel k0: k_chol_diag factors the kNB x kNB diagonal block, k_chol_panel solves the rows below it,
// k_chol_update subtracts L21 L21' from the trailing lower triangle (plain fp64 FMA).  A pivot that is not positive and
// finite stops the factorisation: *info = its 1-based index (LAPACK's / cholesky_ex's convention) and every later launch
// returns at once.  *info must be 0 on entry.
__global__ void __launch_bounds__(256) k_chol_diag(int n, int k0, double* W, double* info) {
    __shared__ double a[kNB][kNB + 1];           // a[col][row]
    if (*info != 0.0) return;
    const int kb = min(kNB, n - k0);
    for (int q = threadIdx.x; q < kb * kb; q += blockDim.x) {
        const int c = q / kb, r = q % kb;
        a[c][r] = W[(size_t)(k0 + c) * n + k0 + r];
    }
    __syncthreads();
    for (int j = 0; j < kb; ++j) {
        const double d = a[j][j];
        if (!(d > 0.0) || !isfinite(d)) {         // uniform: every thread read the same shared value
            if (threadIdx.x == 0) *info = (double)(k0 + j + 1);
            return;
        }
        const double s = sqrt(d);
        __syncthreads();
        for (int r = j + threadIdx.x; r < kb; r += blockDim.x) a[j][r] = (r == j) ? s : a[j][r] / s;
        __syncthreads();
        const int m = kb - j - 1;
        for (int q = threadIdx.x; q < m * m; q += blockDim.x) {
            const int c = j + 1 + q / m, r = j + 1 + q % m;
            if (r >= c) a[c][r] -= a[j][r] * a[j][c];
        }
        __syncthreads();
    }
    for (int q = threadIdx.x; q < kb * kb; q += blockDim.x) {
        const int c = q / kb, r = q % kb;
        if (r >= c) W[(size_t)(k0 + c) * n + k0 + r] = a[c][r];
    }
}

// rows k0 + kNB + 64 blockIdx.x + t of the panel: L21 = A21 L11^-T, one row per thread (a panel below exists only when
// the diagonal block is a full kNB wide)
__global__ void __launch_bounds__(64) k_chol_panel(int n, int k0, double* W, const double* info) {
    __shared__ double L[kNB][kNB];               // L[col][row] of the factored diagonal block
    if (*info != 0.0) return;
    for (int q = threadIdx.x; q < kNB * kNB; q += blockDim.x) {
        const int c = q / kNB, r = q % kNB;
        L[c][r] = W[(size_t)(k0 + c) * n + k0 + r];
    }
    __syncthreads();
    const int row = k0 + kNB + blockIdx.x * 64 + threadIdx.x;
    if (row >= n) return;
    double v[kNB];
#pragma unroll
    for (int j = 0; j < kNB; ++j) v[j] = W[(size_t)(k0 + j) * n + row];
#pragma unroll
    for (int j = 0; j < kNB; ++j) {
        double x = v[j];
#pragma unroll
        for (int p = 0; p < j; ++p) x -= v[p] * L[p][j];
        v[j] = x / L[j][j];
    }
#pragma unroll
    for (int j = 0; j < kNB; ++j) W[(size_t)(k0 + j) * n + row] = v[j];
}

// trailing update A22 -= L21 L21', one 64 x 64 tile of the lower triangle per CTA (grid T x T, the upper tiles return)
__global__ void __launch_bounds__(256) k_chol_update(int n, int k0, double* W, const double* info) {
    __shared__ double As[32][64], Bs[32][64];
    if (*info != 0.0 || blockIdx.x > blockIdx.y) return;
    const int base = k0 + kNB;
    const int i0 = base + blockIdx.y * 64, j0 = base + blockIdx.x * 64;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;      // rows i0 + tx + 16 a, columns j0 + ty + 16 b
    double acc[4][4] = {};
    for (int pc = 0; pc < kNB; pc += 32) {
        for (int q = threadIdx.x; q < 32 * 64; q += 256) {
            const int p = q >> 6, r = q & 63;
            const size_t col = (size_t)(k0 + pc + p) * n;
            As[p][r] = (i0 + r < n) ? W[col + i0 + r] : 0.0;
            Bs[p][r] = (j0 + r < n) ? W[col + j0 + r] : 0.0;
        }
        __syncthreads();
#pragma unroll 8
        for (int p = 0; p < 32; ++p) {
            double x[4], y[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) { x[t] = As[p][tx + 16 * t]; y[t] = Bs[p][ty + 16 * t]; }
#pragma unroll
            for (int s = 0; s < 4; ++s)
#pragma unroll
                for (int t = 0; t < 4; ++t) acc[s][t] = fma(x[s], y[t], acc[s][t]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int s = 0; s < 4; ++s)
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = i0 + tx + 16 * s, j = j0 + ty + 16 * t;
            if (i < n && j < n && i >= j) W[(size_t)j * n + i] -= acc[s][t];
        }
}

// copy the factor's strictly lower part to the upper triangle (W[j n + i] = L(j, i), i < j), so that the back
// substitution reads row j of L contiguously
__global__ void k_chol_mirror(int n, double* W, const double* info) {
    __shared__ double t[32][33];
    if (*info != 0.0 || blockIdx.x > blockIdx.y) return;
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;      // source tile: rows r0.., columns c0.. (r0 >= c0)
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int c = c0 + k, r = r0 + threadIdx.x;
        if (r < n && c < n) t[k][threadIdx.x] = W[(size_t)c * n + r];
    }
    __syncthreads();
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int r = r0 + k, c = c0 + threadIdx.x;            // destination (c, r) of source (r, c): W[r n + c]
        if (r < n && c < n && r > c) W[(size_t)r * n + c] = t[threadIdx.x][k];
    }
}

int chol_factor(int n, double* W, double* info, cudaStream_t st) {
    for (int k0 = 0; k0 < n; k0 += kNB) {
        k_chol_diag<<<1, 256, 0, st>>>(n, k0, W, info);
        const int rest = n - k0 - kNB;
        if (rest > 0) {
            const int T = (rest + 63) / 64;
            k_chol_panel<<<T, 64, 0, st>>>(n, k0, W, info);
            k_chol_update<<<dim3(T, T), 256, 0, st>>>(n, k0, W, info);
        }
    }
    const int T = (n + 31) / 32;
    k_chol_mirror<<<dim3(T, T), dim3(32, 8), 0, st>>>(n, W, info);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { g_last_err = e; return CFMM_E_CUDA; }
    return CFMM_OK;
}

// x = fr * (L L')^-1 (-(nu grad) fr) from the mirrored factor W, and sc[S_DMAX] = max |x|; x is left as it was when the
// factorisation failed (the ladder keeps the last factored direction).  One CTA: forward then back substitution, one
// column per step.
__global__ void __launch_bounds__(kVT) k_newton_solve(Vecs V, const double* nu, const double* fr, const double* W,
                                                      double* x) {
    __shared__ double y[kDenseMax];
    __shared__ double sh[33];
    if (V.sc[S_INFO] != 0.0) return;
    const int n = V.n;
    for (int j = threadIdx.x; j < n; j += kVT) y[j] = -(nu[j] * V.grad[j]) * fr[j];
    __syncthreads();
    for (int j = 0; j < n; ++j) {                              // L y = b
        const double yj = y[j] / W[(size_t)j * n + j];
        __syncthreads();
        if (threadIdx.x == 0) y[j] = yj;
        for (int i = j + 1 + threadIdx.x; i < n; i += kVT) y[i] -= W[(size_t)j * n + i] * yj;
        __syncthreads();
    }
    for (int j = n - 1; j >= 0; --j) {                         // L' x = y
        const double xj = y[j] / W[(size_t)j * n + j];
        __syncthreads();
        if (threadIdx.x == 0) y[j] = xj;
        for (int i = threadIdx.x; i < j; i += kVT) y[i] -= W[(size_t)j * n + i] * xj;
        __syncthreads();
    }
    double mx = 0, bad = 0;
    for (int j = threadIdx.x; j < n; j += kVT) {
        const double v = y[j] * fr[j];
        x[j] = v;
        mx = fmax(mx, fabs(v));
        bad += isfinite(v) ? 0.0 : 1.0;
    }
    mx = block_max(mx, sh); bad = block_sum(bad, sh);
    if (threadIdx.x == 0) V.sc[S_DMAX] = bad > 0.0 ? INFINITY : mx;      // as torch's max: a NaN is never <= kDtMax
}

// ---- active-set look-ahead (solver.py, dense only)

// y = Hs x, Hs row-major: one warp per row
__global__ void k_matvec(int n, const double* Hs, const double* x, double* y) {
    const int row = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (row >= n) return;
    double s = 0;
    for (int k = lane; k < n; k += 32) s += Hs[(size_t)row * n + k] * x[k];
    s = warp_sum(s);
    if (lane == 0) y[row] = s;
}

// newly = bound & (nu grad + Hd < 0) with bound = held at its bound, not pinned; fr2 = fr + newly; sc[S_CNT] = #newly
__global__ void __launch_bounds__(kVT) k_release(Vecs V, const double* nu, const double* hd, double* fr2, double* newly) {
    __shared__ double sh[33];
    double k = 0;
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        const bool nw = V.fr[j] == 0.0 && !V.fixed[j] && (nu[j] * V.grad[j] + hd[j]) < 0.0;
        newly[j] = nw ? 1.0 : 0.0;
        fr2[j] = V.fr[j] + (nw ? 1.0 : 0.0);
        k += nw ? 1.0 : 0.0;
    }
    k = block_sum(k, sh);
    if (threadIdx.x == 0) V.sc[S_CNT] = k;
}

// a released token the new direction x2 would push down stays active: fr = fr2 - bad, x = x2 fr, pg = nu grad fr
__global__ void __launch_bounds__(kVT) k_keep(Vecs V, const double* nu, const double* fr2, const double* newly,
                                              const double* x2) {
    for (int j = threadIdx.x; j < V.n; j += kVT) {
        const double f = fr2[j] - ((newly[j] != 0.0 && x2[j] <= 0.0) ? 1.0 : 0.0);
        V.fr[j] = f;
        V.x[j] = x2[j] * f;
        V.pg[j] = nu[j] * V.grad[j] * f;
    }
}

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// slab stride of a blocked layout (= BlockedArgs::M in cfmm_blocked.cu)
inline size_t hcoef_stride(const cfmm_blocked_pairs* b) { return (size_t)b->n_tiles * (size_t)b->pools_per_tile; }

// The pools of one solve: plain buckets (their per-pool results in outs) and at most one blocked constant-product
// bucket (its hcoef lives in the work buffer, its trades go to blk_out when given)
struct Market {
    const cfmm_bucket* b = nullptr;
    const cfmm_eval_out* outs = nullptr;
    int nb = 0;
    const cfmm_blocked_pairs* blk = nullptr;
    const cfmm_eval_out* blk_out = nullptr;
    bool has_sum = false, has_geo = false;
};

struct LoopCfg {
    double tol, nu_floor, eps0, eps_min, eps_shrink;
    int max_iter, cg_max, max_outer;
    bool dense;          // dense Cholesky Newton systems instead of Jacobi-PCG
    int lookahead;       // active-set look-ahead rounds (dense only)
    bool market;         // solver.py's final read-back pass and its err bookkeeping; false: cfmm_blocked_solve
};

// bytes of the work buffer: the blocked solve's layout is the prefix of the market loop's
size_t work_layout(size_t M, size_t n, bool market, bool dense) {
    size_t bytes = 0;
    bytes += align_up(8 * M);                 // hcoef of the blocked bucket
    bytes += 2 * align_up(8 * (n + 1));       // [psi | arb] ping-pong
    bytes += 2 * align_up(8 * n);             // y ping-pong
    bytes += 13 * align_up(8 * n);            // nut, lb, grad, fr, pg, dt, x, r, z, p, minv, diag, spare (sharded: local diag)
    bytes += align_up(8 * S_COUNT);
    bytes += 2 * align_up(8 * (n + 1)) + align_up(8 * n);      // sharded solve: all-reduced [psi | arb] ping-pong, reduced y
    if (market) {
        bytes += 5 * align_up(8 * n);         // log nu, look-ahead: fr2, x2, Hd, newly
        if (dense) bytes += 2 * align_up(8 * n * n);           // Hs, the factor
    }
    return bytes;
}

bool resolve_dense(int linear_solver, int n, bool has_sum) {     // solver.py linear_solver="auto"
    return linear_solver == 1 || (linear_solver == 0 && (n <= 256 || (has_sum && n <= kDenseMax)));
}

bool uses_hmask(int kind) {
    return kind == CFMM_KIND_GEOMEAN || kind == CFMM_KIND_STABLESWAP_N || kind == CFMM_KIND_CRYPTOSWAP_3;
}

enum { E_HESS, E_TRADES, E_BARE };     // what an evaluation writes besides [psi | arb] (PoolStore.evaluate's hess / trades)

int run_loop(const Market& mk, int n, const double* c, const double* a, const uint8_t* eq, const uint8_t* pinned,
             double* nu, double* psi_out, void* work, const LoopCfg& cfg, cfmm_solve_result* res, cfmm_peer_ctx* peer,
             cudaStream_t st) {
    const size_t M = mk.blk ? hcoef_stride(mk.blk) : 0;
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
    double *lognu = nullptr, *fr2 = nullptr, *x2 = nullptr, *hd = nullptr, *newly = nullptr, *Hs = nullptr, *W = nullptr;
    if (cfg.market) {
        lognu = reinterpret_cast<double*>(take(8 * n));
        fr2 = reinterpret_cast<double*>(take(8 * n)); x2 = reinterpret_cast<double*>(take(8 * n));
        hd = reinterpret_cast<double*>(take(8 * n)); newly = reinterpret_cast<double*>(take(8 * n));
        if (cfg.dense) {
            Hs = reinterpret_cast<double*>(take(8 * (size_t)n * n));
            W = reinterpret_cast<double*>(take(8 * (size_t)n * n));
        }
    }
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
    k_bounds<<<1, kVT, 0, st>>>(n, c, eq, pinned, cfg.nu_floor, lb, nu);
    if (mk.has_sum)                                     // solver.py: ev.reset_multipliers()
        for (int k = 0; k < mk.nb; ++k)
            if ((mk.b[k].kind == CFMM_KIND_SUM || mk.b[k].kind == CFMM_KIND_BINS) && mk.b[k].n_pools > 0)
                cudaMemsetAsync(const_cast<double*>(mk.b[k].theta_bar), 0, 8 * 2 * (size_t)mk.b[k].stride, st);
    // evaluate at `x` into acc[ai]; returns the buffer used.  The calls and their order are PoolStore.evaluate's.
    auto eval = [&](const double* x, double eps, int what) -> double* {
        double* cur = acc[ai];
        double* nxt = acc[ai ^ 1];
        ai ^= 1;
        if (mk.blk) {
            cfmm_eval_out bo;
            bo.delta = nullptr; bo.lambda = nullptr; bo.hcoef = nullptr; bo.hmask = nullptr;
            if (what == E_HESS) bo.hcoef = hcoef;
            if (what == E_TRADES && mk.blk_out) { bo.delta = mk.blk_out->delta; bo.lambda = mk.blk_out->lambda; }
            const bool any = what == E_HESS || (what == E_TRADES && mk.blk_out);
            rc = cfmm_blocked_eval(mk.blk, n, x, cur, cur + n, any ? &bo : nullptr, nxt, n + 1, st);
        } else {
            rc = cfmm_zero(cur, 8 * (int64_t)(n + 1), st);
        }
        if (!rc && mk.has_geo) k_log<<<1, kVT, 0, st>>>(n, x, lognu);
        for (int k = 0; !rc && k < mk.nb; ++k) {
            cfmm_eval_out po;
            po.delta = nullptr; po.lambda = nullptr; po.hcoef = nullptr; po.hmask = nullptr;
            if (what == E_HESS) { po.hcoef = mk.outs[k].hcoef; po.hmask = mk.outs[k].hmask; }
            if (what == E_TRADES) { po.delta = mk.outs[k].delta; po.lambda = mk.outs[k].lambda; }
            rc = cfmm_arb_eval(&mk.b[k], n, x, mk.has_geo ? lognu : nullptr, eps, cur, cur + n,
                               what == E_BARE ? nullptr : &po, st);
        }
        ++evals;
        if (peer && !rc) {                       // every rank continues with the sum over the shards
            rc = reduce(0, cur, n + 1, red[ai]);
            return red[ai];
        }
        return cur;
    };
    // y = Hs v (PoolStore.hvp)
    auto hvp = [&](const double* v) -> double* {
        double* y = yb[yi];
        double* ynx = yb[yi ^ 1];
        yi ^= 1;
        rc = mk.blk ? cfmm_blocked_hvp(mk.blk, n, hcoef, v, y, ynx, st) : cfmm_zero(y, 8 * (int64_t)n, st);
        for (int k = 0; !rc && k < mk.nb; ++k) rc = cfmm_hvp(&mk.b[k], n, mk.outs[k].hcoef, mk.outs[k].hmask, v, y, st);
        if (!rc && peer) { rc = reduce(1, y, n, yred); y = yred; }
        return y;
    };
    // the dense Newton direction on the free set fr_ into xo (solver.py newton_dir): the damping ladder from rung0
    int rung0 = 0, rung_used = 0;
    double* cur_nu = nu;           // the caller's buffer and `nut` swap roles as steps are accepted
    double* oth_nu = nut;
    auto newton_dense = [&](const double* fr_, double* xo) -> int {
        k_dense_dbar<<<1, kVT, 0, st>>>(n, Hs, fr_, V.sc);
        cudaMemsetAsync(xo, 0, 8 * n, st);       // no rung factors: x = 0, and k_direction takes steepest descent
        const int grid = (int)std::min<size_t>(((size_t)n * n + 255) / 256, 8192);
        for (int r = rung0; r < 6; ++r) {
            rung_used = std::max(rung_used, r);
            k_dense_assemble<<<grid, 256, 0, st>>>(n, Hs, fr_, kLmShifts[r], V.sc, W);
            cudaMemsetAsync(V.sc + S_INFO, 0, 8, st);
            const int e = chol_factor(n, W, V.sc + S_INFO, st);
            if (e) return e;
            k_newton_solve<<<1, kVT, 0, st>>>(V, cur_nu, fr_, W, xo);
            if (!fetch()) return CFMM_E_CUDA;
            if (hsc[S_INFO] != 0.0) continue;    // not positive definite: next rung
            if (hsc[S_DMAX] <= kDtMax) break;    // a sane price change
        }
        return CFMM_OK;
    };
    const double eps_init = mk.has_sum ? cfg.eps0 : 0.0;
    double eps_t = eps_init;
    double* cur_acc = nullptr;
    double err = INFINITY, move = 1.0;
    int iters = 0, status = 1;     // 0 optimal, 1 max_iter, 2 stalled
    bool failed_before = false;
    constexpr int kCgBatch = 3;    // PCG iterations launched per host synchronisation
    for (int outer = 0; outer < cfg.max_outer; ++outer) {
        cur_acc = eval(cur_nu, eps_t, E_HESS);
        if (rc) return rc;
        int inner_status = 1;
        // early outer passes need not be solved tightly: the multipliers are still moving
        const double inner_tol = mk.has_sum ? fmax(cfg.tol, fmin(1e-3, 1e-2 * move)) : cfg.tol;
        bool have_kkt = false;     // V.grad / fr / pg and the host scalars describe (cur_nu, cur_acc)
        for (int it = 0; it < cfg.max_iter; ++it) {
            ++iters;
            const double thr = fmin(1e-2, fmax(1e-3 * (isfinite(err) ? err : 1e-2), 1e-14));  // active-set width (see solver.py)
            if (!have_kkt) {
                k_kkt<<<1, kVT, 0, st>>>(V, cur_nu, cur_acc, thr);
                if (!fetch()) return CFMM_E_CUDA;
            }
            err = hsc[S_ERR];
            const double g0 = hsc[S_G];
            if (err <= inner_tol) { inner_status = 0; break; }
            // ---- Newton direction on Hs dt = -(nu * grad) over the free set: dense Cholesky or Jacobi-PCG
            if (cfg.dense) {
                cudaMemsetAsync(Hs, 0, 8 * (size_t)n * n, st);
                if (mk.blk) rc = cfmm_blocked_dense(mk.blk, n, hcoef, Hs, st);
                for (int k = 0; !rc && k < mk.nb; ++k)
                    rc = cfmm_hess_dense(&mk.b[k], n, mk.outs[k].hcoef, mk.outs[k].hmask, Hs, st);
                if (rc) return rc;
            } else {
                double* dg = peer ? diag_loc : V.diag;
                cudaMemsetAsync(dg, 0, 8 * n, st);
                if (mk.blk) rc = cfmm_blocked_diag(mk.blk, n, hcoef, dg, st);
                for (int k = 0; !rc && k < mk.nb; ++k)
                    rc = cfmm_hess_diag(&mk.b[k], n, mk.outs[k].hcoef, mk.outs[k].hmask, dg, st);
                if (!rc && peer) rc = reduce(1, dg, n, V.diag);
                if (rc) return rc;
            }
            rung0 = 0;
            bool ok = false;
            for (;;) {     // a failed search along a barely damped direction is retried from the next rung of the ladder
                rung_used = rung0;
                if (cfg.dense) {
                    if ((rc = newton_dense(V.fr, V.x))) return rc;
                    // look-ahead: a token held at its bound whose predicted gradient after this step, nu*grad + Hs dt,
                    // is negative is released now and the system solved again
                    for (int la = 0; la < cfg.lookahead; ++la) {
                        k_matvec<<<(n + 7) / 8, 256, 0, st>>>(n, Hs, V.x, hd);
                        k_release<<<1, kVT, 0, st>>>(V, cur_nu, hd, fr2, newly);
                        if (!fetch()) return CFMM_E_CUDA;
                        if (hsc[S_CNT] == 0.0) break;
                        if ((rc = newton_dense(fr2, x2))) return rc;
                        k_keep<<<1, kVT, 0, st>>>(V, cur_nu, fr2, newly, x2);
                    }
                } else {
                    k_cg_init<<<1, kVT, 0, st>>>(V);
                    const double eta = fmin(0.1, sqrt(err));
                    for (int k = 0; k < cfg.cg_max;) {
                        // a batch of iterations per synchronisation; k_cg_step turns into a no-op once the stop flag is set
                        for (int bi = 0; bi < kCgBatch && k < cfg.cg_max; ++bi, ++k) {
                            double* y = hvp(V.p);
                            if (rc) return rc;
                            ++hvps;
                            k_cg_step<<<1, kVT, 0, st>>>(V, y, eta, k == 0);
                        }
                        if (!fetch()) return CFMM_E_CUDA;
                        if (hsc[S_STOP] != 0.0) break;
                    }
                }
                k_direction<<<1, kVT, 0, st>>>(V);
                // ---- projected Armijo backtracking along nu * exp(alpha dt); the KKT data of the trial point is
                // computed speculatively behind it, so an accepted step (the rule) costs one synchronisation
                double alpha = 1.0, lin1 = 0.0;
                bool restored = true;      // V and cur_acc describe the current point, not the last trial
                for (int ls = 0; ls < 50; ++ls) {
                    k_step<<<1, kVT, 0, st>>>(V, cur_nu, alpha, oth_nu);
                    double* acct = eval(oth_nu, eps_t, E_HESS);
                    if (rc) return rc;
                    restored = false;
                    k_trial<<<1, kVT, 0, st>>>(V, cur_nu, oth_nu, acct);          // uses the OLD gradient: before k_kkt
                    k_kkt<<<1, kVT, 0, st>>>(V, oth_nu, acct, thr);
                    if (!fetch()) return CFMM_E_CUDA;
                    const double gt = hsc[S_GT], lin = hsc[S_LIN];
                    if (ls == 0) lin1 = lin;                 // predicted decrease of the FULL step
                    if (gt <= g0 + 1e-4 * lin) { ok = true; cur_acc = acct; break; }
                    if (fabs(gt - g0) <= 1e-13 * fabs(g0) || fabs(lin1) <= 1e-9 * fabs(g0)) {
                        // the (full) step is below what g resolves in fp64 (a sum of cancelling flows): judge it by the
                        // KKT residual instead (same rule as solver.py)
                        if (hsc[S_ERR] < 0.99 * err) { ok = true; cur_acc = acct; break; }
                        if (alpha < 1e-3) break;
                    }
                    // rejected: the gradient buffers now belong to the trial -- restore them at the current point
                    cur_acc = eval(cur_nu, eps_t, E_HESS);
                    if (rc) return rc;
                    k_kkt<<<1, kVT, 0, st>>>(V, cur_nu, cur_acc, thr);
                    restored = true;
                    alpha *= 0.5;
                }
                if (ok || !cfg.dense || rung_used >= 5) break;
                rung0 = rung_used + 1;
                if (!restored) {
                    cur_acc = eval(cur_nu, eps_t, E_HESS);
                    if (rc) return rc;
                    k_kkt<<<1, kVT, 0, st>>>(V, cur_nu, cur_acc, thr);
                }
            }
            if (!ok) { inner_status = 2; break; }
            double* t = cur_nu; cur_nu = oth_nu; oth_nu = t;
            have_kkt = true;
            if (cfg.market) err = hsc[S_ERR];    // solver.py: the accepted point's residual, also for the next band
        }
        if (!mk.has_sum) { status = inner_status; break; }
        // ---- method of multipliers.  The smoothed trades are pool-feasible, so (exact dual - primal) at this nu is a
        // true optimality certificate; stop on it rather than on the multiplier step
        double* ps = eval(cur_nu, eps_t, E_TRADES);
        if (rc) return rc;
        k_sums<<<1, kVT, 0, st>>>(V, cur_nu, ps, S_SUM_A);
        double* a0 = eval(cur_nu, 0.0, E_BARE);
        if (rc) return rc;
        k_sums<<<1, kVT, 0, st>>>(V, cur_nu, a0, S_SUM_B);
        if (!fetch()) return CFMM_E_CUDA;
        const double dual_now = hsc[S_SUM_B] + hsc[S_SUM_B + 4];
        const double gap_now = (dual_now - hsc[S_SUM_A + 1]) / fmax(fabs(dual_now), 1e-300);
        if (inner_status == 0 && err <= cfg.tol && fabs(gap_now) <= cfg.tol) { status = 0; break; }
        status = inner_status != 0 ? inner_status : 1;
        if (inner_status != 0 && failed_before && eps_t <= cfg.eps_min) break;   // ramp at its narrowest, two failed passes
        failed_before = inner_status != 0;
        cudaMemsetAsync(V.sc + S_MOVE, 0, 8, st);
        for (int k = 0; !rc && k < mk.nb; ++k)
            if (mk.b[k].kind == CFMM_KIND_SUM)
                rc = cfmm_sum_update_multipliers(&mk.b[k], mk.outs[k].lambda, const_cast<double*>(mk.b[k].theta_bar),
                                                 V.sc + S_MOVE, st);
            else if (mk.b[k].kind == CFMM_KIND_BINS)
                rc = cfmm_bins_update_multipliers(&mk.b[k], mk.outs[k].delta, mk.outs[k].lambda,
                                                  const_cast<double*>(mk.b[k].theta_bar), V.sc + S_MOVE, st);
        if (rc) return rc;
        if (!fetch()) return CFMM_E_CUDA;
        move = hsc[S_MOVE];
        eps_t = fmax(cfg.eps_min, eps_t * cfg.eps_shrink);
    }
    if (!cfg.market) {
        if (status != 0) {
            // max_iter or stalled: make buffers and host scalars consistent with the accepted point
            cur_acc = eval(cur_nu, 0.0, E_HESS);
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
    } else {
        // ---- final read-back + certificate (solver.py): psi and the trades at the last eps (the smoothed trades are
        // pool-feasible), the dual exact: from an eps = 0 evaluation with constant-sum pools, else nu'psi
        double* pf = eval(cur_nu, eps_t, E_TRADES);
        if (rc) return rc;
        cudaMemcpyAsync(psi_out, pf, 8 * n, cudaMemcpyDeviceToDevice, st);
        k_sums<<<1, kVT, 0, st>>>(V, cur_nu, pf, S_SUM_A);
        if (mk.has_sum) {
            double* a0 = eval(cur_nu, 0.0, E_BARE);
            if (rc) return rc;
            k_sums<<<1, kVT, 0, st>>>(V, cur_nu, a0, S_SUM_B);
        }
        if (cur_nu != nu) cudaMemcpyAsync(nu, cur_nu, 8 * n, cudaMemcpyDeviceToDevice, st);
        if (!fetch()) { g_last_err = cudaGetLastError(); return CFMM_E_CUDA; }
        const double arb = mk.has_sum ? hsc[S_SUM_B + 4] : hsc[S_SUM_A + 2];
        const double dual = hsc[S_SUM_A] + arb, primal = hsc[S_SUM_A + 1];
        res->dual_value = dual;
        res->primal_value = primal;
        res->gap = (dual - primal) / fmax(fabs(dual), 1e-300);
        res->primal_infeas = hsc[S_SUM_A + 3] / fmax(fabs(dual), 1e-300);
    }
    res->err = err;
    res->iters = iters; res->evals = evals; res->hvps = hvps; res->status = status;
    return CFMM_OK;
}

// the plain buckets' checks of cfmm_market_solve(_work_bytes); outs == NULL: sizes only
int check_market(const cfmm_bucket* buckets, const cfmm_eval_out* outs, int32_t n_buckets,
                 const cfmm_blocked_pairs* blocked, int32_t n_tokens, int32_t linear_solver, Market* mk, bool* dense) {
    if (n_buckets > 0 && !buckets) return CFMM_E_NULL;
    if (n_tokens <= 0 || n_buckets < 0 || linear_solver < 0 || linear_solver > 2) return CFMM_E_SIZE;
    int64_t pools = 0;
    if (blocked) {
        if (blocked->n_tiles <= 0 || blocked->n_pools < 0) return CFMM_E_SIZE;
        pools += blocked->n_pools;
    }
    for (int k = 0; k < n_buckets; ++k) {
        const cfmm_bucket& b = buckets[k];
        if (b.n_pools < 0) return CFMM_E_SIZE;
        if (b.kind == CFMM_KIND_GEOMEAN) mk->has_geo = true;
        if (b.n_pools == 0) continue;
        pools += b.n_pools;
        if (b.kind == CFMM_KIND_SUM || b.kind == CFMM_KIND_BINS) mk->has_sum = true;
        if (!outs) continue;
        if (!outs[k].hcoef || (uses_hmask(b.kind) && !outs[k].hmask)) return CFMM_E_NULL;
        if (b.kind == CFMM_KIND_SUM && (!outs[k].lambda || !b.theta_bar)) return CFMM_E_NULL;
        if (b.kind == CFMM_KIND_BINS && (!outs[k].delta || !outs[k].lambda || !b.theta_bar)) return CFMM_E_NULL;
    }
    if (pools == 0) return CFMM_E_SIZE;
    *dense = resolve_dense(linear_solver, n_tokens, mk->has_sum);
    if (*dense && n_tokens > kDenseMax) return CFMM_E_SIZE;
    return CFMM_OK;
}

}  // namespace

extern "C" {

int64_t cfmm_blocked_solve_work_bytes(const cfmm_blocked_pairs* b, int32_t n_tokens) {
    if (!b || n_tokens <= 0) return CFMM_E_SIZE;
    return (int64_t)work_layout(hcoef_stride(b), (size_t)n_tokens, false, false);
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
    Market mk;
    mk.blk = b;
    const LoopCfg cfg{prm->tol, prm->nu_floor, 0.0, 0.0, 0.0, prm->max_iter, prm->cg_max, 1, false, 0, false};
    return run_loop(mk, n_tokens, c, a, eq, pinned, nu, psi_out, work, cfg, res, peer, static_cast<cudaStream_t>(stream));
}

int64_t cfmm_market_solve_work_bytes(const cfmm_bucket* buckets, int32_t n_buckets, const cfmm_blocked_pairs* blocked,
                                     int32_t n_tokens, int32_t linear_solver) {
    Market mk;
    bool dense = false;
    const int e = check_market(buckets, nullptr, n_buckets, blocked, n_tokens, linear_solver, &mk, &dense);
    if (e) return e;
    return (int64_t)work_layout(blocked ? hcoef_stride(blocked) : 0, (size_t)n_tokens, true, dense);
}

int cfmm_market_solve(const cfmm_bucket* buckets, const cfmm_eval_out* outs, int32_t n_buckets,
                      const cfmm_blocked_pairs* blocked, const cfmm_eval_out* blocked_out, int32_t n_tokens,
                      const double* c, const double* a, const uint8_t* eq, const uint8_t* pinned, double* nu,
                      double* psi_out, void* work, const cfmm_market_params* prm, cfmm_solve_result* res, void* stream) {
    if (!c || !a || !eq || !pinned || !nu || !psi_out || !work || !prm || !res) return CFMM_E_NULL;
    if (n_buckets > 0 && !outs) return CFMM_E_NULL;
    Market mk;
    bool dense = false;
    const int e = check_market(buckets, outs, n_buckets, blocked, n_tokens, prm->linear_solver, &mk, &dense);
    if (e) return e;
    mk.b = buckets; mk.outs = outs; mk.nb = n_buckets; mk.blk = blocked; mk.blk_out = blocked_out;
    const LoopCfg cfg{prm->tol, prm->nu_floor, prm->eps0, prm->eps_min, prm->eps_shrink, prm->max_iter, prm->cg_max,
                      prm->max_outer, dense, (dense && n_tokens <= 64) ? 3 : 0, true};
    return run_loop(mk, n_tokens, c, a, eq, pinned, nu, psi_out, work, cfg, res, nullptr,
                    static_cast<cudaStream_t>(stream));
}

int cfmm_dense_cholesky(int32_t n, double* a, double* info, void* stream) {
    if (!a || !info) return CFMM_E_NULL;
    if (n <= 0 || n > kDenseMax) return CFMM_E_SIZE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaMemsetAsync(info, 0, 8, st);
    return chol_factor(n, a, info, st);
}

}  // extern "C"
