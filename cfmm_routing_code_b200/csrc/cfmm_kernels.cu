// cfmm_kernels.cu -- sm_90a kernels + C ABI for the per-pool optimal-arbitrage hot path.
//
// What the reference does with one cvxpy `prob.solve()` (arbitrage.py:81-82) is done here by
// dual decomposition: at fixed token prices nu every pool's subproblem
//     max nu'(L - D)  s.t.  phi_i(R + gamma D - L) >= phi_i(R),  D, L >= 0     (arbitrage.py:60-74)
// is independent and has a closed / finite form; the kernels evaluate all pools and reduce
//     psi = sum_i A_i (L_i - D_i)   (arbitrage.py:54)   and   arb = sum_i nu_i'(L_i - D_i).
// fp64 throughout, HBM-bound for the 2-token kinds (32 B/pool), no tensor cores (no contraction).
#include <math.h>

#include "cfmm_dev.cuh"
#include "cfmm_small.cuh"     // bounded_pair(), eclp_pair(), pmm_pair(), ladder_pair(), bins_pair(), ...: the per-pool math, shared with the per-thread solver

namespace cfmm {
std::atomic<long long> g_launches{0};
int g_scatter_mode = 0;
thread_local cudaError_t g_last_err = cudaSuccess;
static int g_num_sms = 0;
int num_sms() {
    if (g_num_sms == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            g_num_sms = n;
        else
            g_num_sms = 132;
    }
    return g_num_sms;
}
}  // namespace cfmm

using namespace cfmm;

namespace {

constexpr int kThreads = 256;

// ---------------------------------------------------------------------------------------------
// scatter targets: global red.add.f64, or a shared-memory privatised copy of the n_token vector
// ---------------------------------------------------------------------------------------------
struct GlobalScatter {
    double* out;
    __device__ __forceinline__ void init(double*, int) {}
    __device__ __forceinline__ void add(int tok, double v) { atomicAdd(out + tok, v); }
    __device__ __forceinline__ void flush(double*, int) {}
};

struct SharedScatter {
    double* out;
    double* hist;
    __device__ __forceinline__ void init(double* smem, int n) {
        hist = smem;
        for (int j = threadIdx.x; j < n; j += blockDim.x) hist[j] = 0.0;
        __syncthreads();
    }
    __device__ __forceinline__ void add(int tok, double v) { atomicAdd(hist + tok, v); }
    __device__ __forceinline__ void flush(double*, int n) {
        __syncthreads();
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            double v = hist[j];
            if (v != 0.0) atomicAdd(out + j, v);
        }
    }
};

__device__ __forceinline__ void block_accumulate(double v, double* target) {
    __shared__ double part[kThreads / 32];
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        double s = (threadIdx.x < kThreads / 32) ? part[threadIdx.x] : 0.0;
        s = warp_sum(s);
        if (threadIdx.x == 0 && s != 0.0) atomicAdd(target, s);
    }
}

// ---------------------------------------------------------------------------------------------
// per-pool closed forms
// ---------------------------------------------------------------------------------------------
// constant product, arbitrage.py:68-70.  Trade 0->1 iff gamma nu1 R1 > nu0 R0:
//   x0 = R0 t, x1 = R1 / t, t = sqrt(gamma nu1 R1 / (nu0 R0)); D0 = (x0-R0)/gamma, L1 = R1 - x1.
// hcoef = sqrt(nu0 R0 nu1 R1 / gamma) / 2  (Hs_i = hcoef [[1,-1],[-1,1]] in log-price coords).
__device__ __forceinline__ void product_pool(double R0, double R1, double g, double n0, double n1,
                                             double& y0, double& y1, double& h) {
    const double p0 = n0 * R0, p1 = n1 * R1;
    const bool fwd = g * p1 > p0;
    const bool bwd = g * p0 > p1;
    y0 = 0.0; y1 = 0.0; h = 0.0;
    if (fwd || bwd) {
        const double num = fwd ? p1 : p0, den = fwd ? p0 : p1;
        const double q = g * num / den;
        const double t = sqrt(q);
        const double Rin = fwd ? R0 : R1, Rout = fwd ? R1 : R0;
        const double din = Rin * (t - 1.0) / g;       // Delta on the tendered token
        const double lout = Rout * (1.0 - 1.0 / t);   // Lambda on the received token
        y0 = fwd ? -din : lout;
        y1 = fwd ? lout : -din;
        h = 0.5 * sqrt(p0 * p1 / g);
    }
}

// one constant-sum limit order (tender a, receive up to Rb of b), proximal-multiplier smoothing:
//   psi(z) = max_{0<=th<=Rb} th z - (th - thbar)^2 / (2 sigma), sigma = Rb/eps, z = gamma nu_b/nu_a - 1
// returns fill th = Lambda_b, pay = Delta_a = (r th - psi)/gamma, curvature term.  arbitrage.py:73-74.
__device__ __forceinline__ void sum_order(double Rb, double g, double na, double nb, double thbar, double eps,
                                          double& th, double& pay, double& h) {
    const double r = g * nb / na;
    const double z = r - 1.0;
    if (eps <= 0.0) {
        th = z > 0.0 ? Rb : 0.0;
        pay = th / g;       // (r th - th z)/gamma
        h = 0.0;
        return;
    }
    const double sigma = Rb / eps;
    th = fmin(fmax(thbar + sigma * z, 0.0), Rb);
    const double d = th - thbar;
    const double psi = th * z - d * d / (2.0 * sigma);
    pay = (r * th - psi) / g;
    h = (th > 0.0 && th < Rb) ? sigma * nb * r : 0.0;
}

template <int KIND, typename Scatter, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kThreads)
k_eval_pair(long long m, long long ld, int n_tokens, const double* __restrict__ R, const int* __restrict__ idx,
            const double* __restrict__ gamma, const double* __restrict__ thbar, double eps,
            const double* __restrict__ nu, double* psi, double* arb, double* delta, double* lambda,
            double* hcoef) {
    extern __shared__ double smem[];
    Scatter sc{psi};
    sc.init(smem, n_tokens);
    double acc = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double R0 = R[i], R1 = R[ld + i], g = gamma[i];
        const int i0 = idx[i], i1 = idx[ld + i];
        const double n0 = __ldg(nu + i0), n1 = __ldg(nu + i1);
        double y0, y1, h;
        if (KIND == CFMM_KIND_PRODUCT) {
            product_pool(R0, R1, g, n0, n1, y0, y1, h);
        } else if (KIND == CFMM_KIND_BOUNDED_PRODUCT) {
            // `thbar` carries the per-slot auxiliary array of the bucket: here the virtual-reserve offsets
            double D[2], L[2];
            cfmm_small::bounded_pair(R0, R1, thbar[i], thbar[ld + i], g, n0, n1, D, L, h);
            y0 = L[0] - D[0];
            y1 = L[1] - D[1];
            if (TRADES) {
                delta[i] = D[0]; delta[ld + i] = D[1];
                lambda[i] = L[0]; lambda[ld + i] = L[1];
            }
        } else if (KIND == CFMM_KIND_ECLP) {
            // `thbar` carries the bucket's weights [7][ld] = (alpha, beta, c, s, lam, r, p)
            double D[2], L[2];
            cfmm_small::eclp_pair(R0, R1, thbar[i], thbar[ld + i], thbar[2 * ld + i], thbar[3 * ld + i],
                                  thbar[4 * ld + i], thbar[5 * ld + i], thbar[6 * ld + i], g, n0, n1, D, L, h);
            y0 = L[0] - D[0];
            y1 = L[1] - D[1];
            if (TRADES) {
                delta[i] = D[0]; delta[ld + i] = D[1];
                lambda[i] = L[0]; lambda[ld + i] = L[1];
            }
        } else if (KIND == CFMM_KIND_PMM) {
            // `thbar` carries the bucket's weights [4][ld] = (pi, k, B0, Q0)
            double D[2], L[2];
            cfmm_small::pmm_pair(R0, R1, thbar[i], thbar[ld + i], thbar[2 * ld + i], thbar[3 * ld + i], g, n0, n1, D, L,
                                 h);
            y0 = L[0] - D[0];
            y1 = L[1] - D[1];
            if (TRADES) {
                delta[i] = D[0]; delta[ld + i] = D[1];
                lambda[i] = L[0]; lambda[ld + i] = L[1];
            }
        } else {
            // order A pays out token 1 (tender 0), order B pays out token 0 (tender 1)
            double thA, payA, hA, thB, payB, hB;
            sum_order(R1, g, n0, n1, thbar ? thbar[ld + i] : 0.0, eps, thA, payA, hA);
            sum_order(R0, g, n1, n0, thbar ? thbar[i] : 0.0, eps, thB, payB, hB);
            y0 = thB - payA;
            y1 = thA - payB;
            h = hA + hB;
            if (TRADES) {
                delta[i] = payA; delta[ld + i] = payB;
                lambda[i] = thB; lambda[ld + i] = thA;
            }
        }
        if (TRADES && KIND == CFMM_KIND_PRODUCT) {
            delta[i] = fmax(-y0, 0.0); delta[ld + i] = fmax(-y1, 0.0);
            lambda[i] = fmax(y0, 0.0); lambda[ld + i] = fmax(y1, 0.0);
        }
        if (HESS) hcoef[i] = h;
        if (y0 != 0.0) sc.add(i0, y0);
        if (y1 != 0.0) sc.add(i1, y1);
        acc += n0 * y0 + n1 * y1;
    }
    sc.flush(smem, n_tokens);
    block_accumulate(acc, arb);
}

// two-coin StableSwap: cfmm_small::stableswap_pair (a safeguarded Newton solve per trading pool, compute-bound rather
// than HBM-bound), one thread per pool.  rates [2][ld] (the bucket's weights), AD [2][ld] = (A, D) (the bucket's logrw).
template <typename Scatter, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kThreads)
k_eval_stable(long long m, long long ld, int n_tokens, const double* __restrict__ R, const int* __restrict__ idx,
              const double* __restrict__ gamma, const double* __restrict__ rates, const double* __restrict__ AD,
              const double* __restrict__ nu, double* psi, double* arb, double* delta, double* lambda, double* hcoef) {
    extern __shared__ double smem[];
    Scatter sc{psi};
    sc.init(smem, n_tokens);
    double acc = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const int i0 = idx[i], i1 = idx[ld + i];
        const double n0 = __ldg(nu + i0), n1 = __ldg(nu + i1);
        double D[2], L[2], h;
        cfmm_small::stableswap_pair(R[i], R[ld + i], rates[i], rates[ld + i], AD[i], AD[ld + i], gamma[i], n0, n1, D, L, h);
        const double y0 = L[0] - D[0], y1 = L[1] - D[1];
        if (TRADES) {
            delta[i] = D[0]; delta[ld + i] = D[1];
            lambda[i] = L[0]; lambda[ld + i] = L[1];
        }
        if (HESS) hcoef[i] = h;
        if (y0 != 0.0) sc.add(i0, y0);
        if (y1 != 0.0) sc.add(i1, y1);
        acc += n0 * y0 + n1 * y1;
    }
    sc.flush(smem, n_tokens);
    block_accumulate(acc, arb);
}

// two-coin cryptoswap (Curve v2): cfmm_small::cryptoswap_pair (a safeguarded Newton solve per trading pool around an
// inner one for the curve point, compute-bound), one thread per pool.  scales [2][ld] = the price scales p (the bucket's
// weights), AGD [3][ld] = (A, G, D) (the bucket's logrw); the kernel passes c = p / D.
template <typename Scatter, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kThreads)
k_eval_crypto(long long m, long long ld, int n_tokens, const double* __restrict__ R, const int* __restrict__ idx,
              const double* __restrict__ gamma, const double* __restrict__ scales, const double* __restrict__ AGD,
              const double* __restrict__ nu, double* psi, double* arb, double* delta, double* lambda, double* hcoef) {
    extern __shared__ double smem[];
    Scatter sc{psi};
    sc.init(smem, n_tokens);
    double acc = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const int i0 = idx[i], i1 = idx[ld + i];
        const double n0 = __ldg(nu + i0), n1 = __ldg(nu + i1);
        const double Dv = AGD[2 * ld + i];
        double D[2], L[2], h;
        cfmm_small::cryptoswap_pair(R[i], R[ld + i], scales[i] / Dv, scales[ld + i] / Dv, AGD[i], AGD[ld + i], gamma[i],
                                    n0, n1, D, L, h);
        const double y0 = L[0] - D[0], y1 = L[1] - D[1];
        if (TRADES) {
            delta[i] = D[0]; delta[ld + i] = D[1];
            lambda[i] = L[0]; lambda[ld + i] = L[1];
        }
        if (HESS) hcoef[i] = h;
        if (y0 != 0.0) sc.add(i0, y0);
        if (y1 != 0.0) sc.add(i1, y1);
        acc += n0 * y0 + n1 * y1;
    }
    sc.flush(smem, n_tokens);
    block_accumulate(acc, arb);
}

// concentrated liquidity (a whole tick ladder per pool): cfmm_small::ladder_pair, one thread per pool.  rec = the AoS
// records (the bucket's weights), P [4][ld] = (s, c, first record, T) (the bucket's logrw).  The reserves are not read:
// the flows come from the records.  A trade that stays in the current interval reads records c and c + 1; one that
// crosses k bounds O(log k) more.
template <typename Scatter, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kThreads)
k_eval_ladder(long long m, long long ld, int n_tokens, const int* __restrict__ idx, const double* __restrict__ gamma,
              const double* __restrict__ rec, const double* __restrict__ P, const double* __restrict__ nu, double* psi,
              double* arb, double* delta, double* lambda, double* hcoef) {
    extern __shared__ double smem[];
    Scatter sc{psi};
    sc.init(smem, n_tokens);
    double acc = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const int i0 = idx[i], i1 = idx[ld + i];
        const double n0 = __ldg(nu + i0), n1 = __ldg(nu + i1);
        double D[2], L[2], h;
        cfmm_small::ladder_pair(rec + 4 * (long long)P[2 * ld + i], (long long)P[3 * ld + i], (long long)P[ld + i], P[i],
                                gamma[i], n0, n1, D, L, h);
        const double y0 = L[0] - D[0], y1 = L[1] - D[1];
        if (TRADES) {
            delta[i] = D[0]; delta[ld + i] = D[1];
            lambda[i] = L[0]; lambda[ld + i] = L[1];
        }
        if (HESS) hcoef[i] = h;
        if (y0 != 0.0) sc.add(i0, y0);
        if (y1 != 0.0) sc.add(i1, y1);
        acc += n0 * y0 + n1 * y1;
    }
    sc.flush(smem, n_tokens);
    block_accumulate(acc, arb);
}

// price bins (Liquidity Book bins, order books, limit orders): cfmm_small::bins_pair, one thread per pool.  rec = the
// AoS records (the bucket's weights), P [4][ld] = (first record, nb, z, p_ref) (the bucket's logrw), tbar = theta_bar
// row 0 (read only when eps > 0).  The reserves are not read.  A trade that stays in the segment next to t = 0 reads
// O(1) records; one that crosses k breakpoints O(log k) more.
template <typename Scatter, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kThreads)
k_eval_bins(long long m, long long ld, int n_tokens, const int* __restrict__ idx, const double* __restrict__ gamma,
            const double* __restrict__ rec, const double* __restrict__ P, const double* __restrict__ tbar, double eps,
            const double* __restrict__ nu, double* psi, double* arb, double* delta, double* lambda, double* hcoef) {
    extern __shared__ double smem[];
    Scatter sc{psi};
    sc.init(smem, n_tokens);
    double acc = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const int i0 = idx[i], i1 = idx[ld + i];
        const double n0 = __ldg(nu + i0), n1 = __ldg(nu + i1);
        double D[2], L[2], h;
        cfmm_small::bins_pair(rec + 4 * (long long)P[i], (long long)P[ld + i], (long long)P[2 * ld + i], P[3 * ld + i],
                              eps > 0.0 ? tbar[i] : 0.0, gamma[i], n0, n1, eps, D, L, h);
        const double y0 = L[0] - D[0], y1 = L[1] - D[1];
        if (TRADES) {
            delta[i] = D[0]; delta[ld + i] = D[1];
            lambda[i] = L[0]; lambda[ld + i] = L[1];
        }
        if (HESS) hcoef[i] = h;
        if (y0 != 0.0) sc.add(i0, y0);
        if (y1 != 0.0) sc.add(i1, y1);
        acc += n0 * y0 + n1 * y1;
    }
    sc.flush(smem, n_tokens);
    block_accumulate(acc, arb);
}

// n-coin StableSwap, arity K (3..8; 2 for the cross-check against k_eval_stable): cfmm_small::stableswap_n (a
// breakpoint root per step of a safeguarded Newton iteration, compute-bound), one thread per pool.  rates [K][ld] (the
// bucket's weights), AD [2][ld] = (A, D) (the bucket's logrw).  hcoef [K][ld] = the per-slot h_j, hmask = traded slots.
template <int K, typename Scatter, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kThreads)
k_eval_stable_n(long long m, long long ld, int n_tokens, const double* __restrict__ R, const int* __restrict__ idx,
                const double* __restrict__ gamma, const double* __restrict__ rates, const double* __restrict__ AD,
                const double* __restrict__ nu, double* psi, double* arb, double* delta, double* lambda, double* hcoef,
                uint32_t* hmask) {
    extern __shared__ double smem[];
    Scatter sc{psi};
    sc.init(smem, n_tokens);
    double acc = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        double Rl[K], rl[K], nl[K], D[K], L[K], h[K];
        int id[K];
#pragma unroll
        for (int j = 0; j < K; ++j) {
            id[j] = idx[(long long)j * ld + i];
            Rl[j] = R[(long long)j * ld + i];
            rl[j] = rates[(long long)j * ld + i];
            nl[j] = __ldg(nu + id[j]);
        }
        const uint32_t mask = cfmm_small::stableswap_n<K>(K, Rl, rl, AD[i], AD[ld + i], gamma[i], nl, D, L, h);
#pragma unroll
        for (int j = 0; j < K; ++j) {
            if (TRADES) { delta[(long long)j * ld + i] = D[j]; lambda[(long long)j * ld + i] = L[j]; }
            if (HESS) hcoef[(long long)j * ld + i] = h[j];
            const double y = L[j] - D[j];
            if (y != 0.0) {
                sc.add(id[j], y);
                acc += nl[j] * y;
            }
        }
        if (HESS) hmask[i] = mask;
    }
    sc.flush(smem, n_tokens);
    block_accumulate(acc, arb);
}

// three-coin cryptoswap (tricrypto-ng): cfmm_small::cryptoswap3 (a safeguarded Newton solve in m = 1 - K0 around an
// inner one for the price level, compute-bound), one thread per pool.  scales [3][ld] = the price scales p (the bucket's
// weights), AGD [3][ld] = (A, G, D) (the bucket's logrw); the kernel passes c = p / D.  hcoef [3][ld] = the edge weights
// (w01, w02, w12) of the pool's scaled Hessian block, hmask = traded slots.
template <typename Scatter, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kThreads)
k_eval_crypto3(long long m, long long ld, int n_tokens, const double* __restrict__ R, const int* __restrict__ idx,
               const double* __restrict__ gamma, const double* __restrict__ scales, const double* __restrict__ AGD,
               const double* __restrict__ nu, double* psi, double* arb, double* delta, double* lambda, double* hcoef,
               uint32_t* hmask) {
    extern __shared__ double smem[];
    Scatter sc{psi};
    sc.init(smem, n_tokens);
    double acc = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const int i0 = idx[i], i1 = idx[ld + i], i2 = idx[2 * ld + i];
        const double n0 = __ldg(nu + i0), n1 = __ldg(nu + i1), n2 = __ldg(nu + i2);
        const double Dv = AGD[2 * ld + i];
        double D[3], L[3], w[3];
        const uint32_t mask = cfmm_small::cryptoswap3(R[i], R[ld + i], R[2 * ld + i], scales[i] / Dv, scales[ld + i] / Dv,
                                                      scales[2 * ld + i] / Dv, AGD[i], AGD[ld + i], gamma[i], n0, n1, n2,
                                                      D, L, w);
        const double y0 = L[0] - D[0], y1 = L[1] - D[1], y2 = L[2] - D[2];
        if (TRADES) {
            delta[i] = D[0]; delta[ld + i] = D[1]; delta[2 * ld + i] = D[2];
            lambda[i] = L[0]; lambda[ld + i] = L[1]; lambda[2 * ld + i] = L[2];
        }
        if (HESS) {
            hcoef[i] = w[0]; hcoef[ld + i] = w[1]; hcoef[2 * ld + i] = w[2];
            hmask[i] = mask;
        }
        if (y0 != 0.0) sc.add(i0, y0);
        if (y1 != 0.0) sc.add(i1, y1);
        if (y2 != 0.0) sc.add(i2, y2);
        acc += n0 * y0 + n1 * y1 + n2 * y2;
    }
    sc.flush(smem, n_tokens);
    block_accumulate(acc, arb);
}

// ---------------------------------------------------------------------------------------------
// TMA-staged variant of the 2-token kernel: persistent CTAs, each walking tiles of kTile pools.
// One elected thread issues five 1-D bulk copies per tile (cp.async.bulk -> UBLKCP: R0, R1, gamma,
// idx0, idx1 slabs, 32 B/pool) into a kStages-deep shared-memory ring; completion is signalled on
// an mbarrier per stage (expect_tx), so kStages-1 tiles (~64 KB per CTA) are always in flight from
// HBM regardless of occupancy.  A __syncthreads per tile hands the drained stage back to the
// producer.  nu is gathered through L1 (n_tokens * 8 B stays cache resident).
// ---------------------------------------------------------------------------------------------
constexpr int kTile = 1024;          // pools per tile: 32 KB per stage
constexpr int kStages = 3;
constexpr int kTmaThreads = 512;
constexpr int kPoolsPerThread = kTile / kTmaThreads;

struct __align__(128) PairStage {
    double R0[kTile];
    double R1[kTile];
    double g[kTile];
    int i0[kTile];
    int i1[kTile];
};
constexpr unsigned kStageBytes = sizeof(PairStage);
static_assert(kStageBytes == 32u * kTile, "32 B per pool");

__device__ __forceinline__ void issue_pair_tile(PairStage* st, uint64_t* bar, long long tile, long long ld,
                                                const double* R, const int* idx, const double* gamma) {
    const long long o = tile * kTile;
    mbar_expect_tx(bar, kStageBytes);
    bulk_g2s(st->R0, R + o, kTile * 8, bar);
    bulk_g2s(st->R1, R + ld + o, kTile * 8, bar);
    bulk_g2s(st->g, gamma + o, kTile * 8, bar);
    bulk_g2s(st->i0, idx + o, kTile * 4, bar);
    bulk_g2s(st->i1, idx + ld + o, kTile * 4, bar);
}

template <int KIND, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kTmaThreads, 2)
k_eval_pair_tma(long long m, long long ld, int n_tokens, const double* __restrict__ R, const int* __restrict__ idx,
                const double* __restrict__ gamma, const double* __restrict__ thbar, double eps,
                const double* __restrict__ nu, double* psi, double* arb, double* delta, double* lambda,
                double* hcoef) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    PairStage* stages = reinterpret_cast<PairStage*>(smem_raw);
    __shared__ uint64_t full[kStages];
    __shared__ double part[kTmaThreads / 32];
    const int tid = threadIdx.x;
    const long long ntiles = (m + kTile - 1) / kTile;
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(&full[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            const long long t = (long long)blockIdx.x + (long long)s * gridDim.x;
            if (t < ntiles) issue_pair_tile(&stages[s], &full[s], t, ld, R, idx, gamma);
        }
    }
    double acc = 0.0;
    int stage = 0;
    unsigned parity = 0;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        mbar_wait(&full[stage], parity);
        const PairStage& S = stages[stage];
#pragma unroll
        for (int u = 0; u < kPoolsPerThread; ++u) {
            const int l = tid + u * kTmaThreads;
            const long long i = tile * kTile + l;
            if (i < m) {
                const double R0 = S.R0[l], R1 = S.R1[l], g = S.g[l];
                const int i0 = S.i0[l], i1 = S.i1[l];
                const double n0 = __ldg(nu + i0), n1 = __ldg(nu + i1);
                double y0, y1, h;
                if (KIND == CFMM_KIND_PRODUCT) {
                    product_pool(R0, R1, g, n0, n1, y0, y1, h);
                    if (TRADES) {
                        delta[i] = fmax(-y0, 0.0); delta[ld + i] = fmax(-y1, 0.0);
                        lambda[i] = fmax(y0, 0.0); lambda[ld + i] = fmax(y1, 0.0);
                    }
                } else {
                    double thA, payA, hA, thB, payB, hB;
                    sum_order(R1, g, n0, n1, thbar ? thbar[ld + i] : 0.0, eps, thA, payA, hA);
                    sum_order(R0, g, n1, n0, thbar ? thbar[i] : 0.0, eps, thB, payB, hB);
                    y0 = thB - payA;
                    y1 = thA - payB;
                    h = hA + hB;
                    if (TRADES) {
                        delta[i] = payA; delta[ld + i] = payB;
                        lambda[i] = thB; lambda[ld + i] = thA;
                    }
                }
                if (HESS) hcoef[i] = h;
                if (y0 != 0.0) atomicAdd(psi + i0, y0);
                if (y1 != 0.0) atomicAdd(psi + i1, y1);
                acc += n0 * y0 + n1 * y1;
            }
        }
        __syncthreads();                      // every thread is done reading this stage
        if (tid == 0) {
            const long long nxt = tile + (long long)kStages * gridDim.x;
            if (nxt < ntiles) {
                fence_proxy_async();
                issue_pair_tile(&stages[stage], &full[stage], nxt, ld, R, idx, gamma);
            }
        }
        if (++stage == kStages) { stage = 0; parity ^= 1u; }
    }
    acc = warp_sum(acc);
    if ((tid & 31) == 0) part[tid >> 5] = acc;
    __syncthreads();
    if (tid < 32) {
        double s = (tid < kTmaThreads / 32) ? part[tid] : 0.0;
        s = warp_sum(s);
        if (tid == 0 && s != 0.0) atomicAdd(arb, s);
    }
}

// ---------------------------------------------------------------------------------------------
// weighted geometric mean, arity K (arbitrage.py:65).  One thread per pool.
//   tB_j = log(R_j/w_j) + log nu_j,  tA_j = tB_j - log gamma
//   h(s) = sum_j w_j [max(s - tA_j, 0) + min(s - tB_j, 0)]  is piecewise linear, nondecreasing;
//   no trade iff max tB <= min tA; else the root is exact from the breakpoint with the largest
//   h <= 0 and the slope to its right.  D_j = R_j expm1(max(s-tA_j,0))/gamma, L_j = -R_j expm1(min(s-tB_j,0)).
// ---------------------------------------------------------------------------------------------
template <int K, typename Scatter, bool TRADES, bool HESS>
__global__ void __launch_bounds__(kThreads)
k_eval_geomean(long long m, long long ld, int karity, int n_tokens, const double* __restrict__ R, const int* __restrict__ idx,
               const double* __restrict__ gamma, const double* __restrict__ W, const double* __restrict__ logrw,
               const double* __restrict__ nu, const double* __restrict__ lognu, double* psi, double* arb,
               double* delta, double* lambda, double* hcoef, uint32_t* hmask) {
    extern __shared__ double smem[];
    Scatter sc{psi};
    sc.init(smem, n_tokens);
    constexpr int KMAX = (K > 0) ? K : 32;
    const int k = (K > 0) ? K : karity;
    double acc = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double g = gamma[i];
        const double lg = log(g);
        double tB[KMAX], w[KMAX];
        int id[KMAX];
        double maxB = -INFINITY, minA = INFINITY;
#pragma unroll
        for (int j = 0; j < KMAX; ++j) {
            if (j < k) {
                id[j] = idx[(long long)j * ld + i];
                w[j] = W[(long long)j * ld + i];
                tB[j] = logrw[(long long)j * ld + i] + __ldg(lognu + id[j]);
                maxB = fmax(maxB, tB[j]);
                minA = fmin(minA, tB[j] - lg);
            }
        }
        const bool trade = maxB > minA;
        double s = 0.0;
        if (trade) {
            double sL = -INFINITY, hL = 0.0;
#pragma unroll 1
            for (int p = 0; p < 2 * k; ++p) {
                const double T = (p < k) ? tB[p] - lg : tB[p - k];
                double hh = 0.0;
#pragma unroll
                for (int j = 0; j < KMAX; ++j)
                    if (j < k) hh += w[j] * (fmax(T - (tB[j] - lg), 0.0) + fmin(T - tB[j], 0.0));
                if (hh <= 0.0 && T > sL) { sL = T; hL = hh; }
            }
            double Wr = 0.0;
#pragma unroll
            for (int j = 0; j < KMAX; ++j)
                if (j < k) Wr += ((sL >= tB[j] - lg) || (sL < tB[j])) ? w[j] : 0.0;
            s = (hL < 0.0) ? sL - hL / Wr : sL;
        }
        uint32_t mask = 0;
#pragma unroll
        for (int j = 0; j < KMAX; ++j) {
            if (j < k) {
                const double zA = trade ? fmax(s - (tB[j] - lg), 0.0) : 0.0;
                const double zB = trade ? fmin(s - tB[j], 0.0) : 0.0;
                const double z = (zA > 0.0) ? zA : zB;
                double y = 0.0;
                if (z != 0.0 || TRADES) {
                    const double Rj = R[(long long)j * ld + i];
                    const double e = expm1(z);
                    const double D = (zA > 0.0) ? Rj * e / g : 0.0;
                    const double L = (zB < 0.0) ? -Rj * e : 0.0;
                    y = L - D;
                    if (TRADES) { delta[(long long)j * ld + i] = D; lambda[(long long)j * ld + i] = L; }
                }
                if (z != 0.0) {
                    mask |= 1u << j;
                    sc.add(id[j], y);
                    acc += __ldg(nu + id[j]) * y;
                }
            }
        }
        if (HESS) { hcoef[i] = trade ? exp(s) : 0.0; hmask[i] = mask; }
    }
    sc.flush(smem, n_tokens);
    block_accumulate(acc, arb);
}

// ---------------------------------------------------------------------------------------------
// Hessian-vector product / diagonal / dense assembly, log-price coordinates
//   2-token kinds:  Hs_i = h [[1,-1],[-1,1]]
//   geomean:        Hs_i = M (diag(w_act) - w_act w_act'/W_act)
//   n-coin StableSwap: Hs_i = C - (C1)(C1)'/(1'C1), C = diag(h^2) - h h'/(1 + k)   (cfmm_small::stableswap_n)
// ---------------------------------------------------------------------------------------------
template <typename Scatter>
__global__ void __launch_bounds__(kThreads)
k_hvp_pair(long long m, long long ld, int n_tokens, const int* __restrict__ idx, const double* __restrict__ hcoef,
           const double* __restrict__ vt, double* y) {
    extern __shared__ double smem[];
    Scatter sc{y};
    sc.init(smem, n_tokens);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double h = hcoef[i];
        if (h != 0.0) {
            const int i0 = idx[i], i1 = idx[ld + i];
            const double c = h * (__ldg(vt + i0) - __ldg(vt + i1));
            sc.add(i0, c);
            sc.add(i1, -c);
        }
    }
    sc.flush(smem, n_tokens);
}

template <typename Scatter>
__global__ void __launch_bounds__(kThreads)
k_hvp_geomean(long long m, long long ld, int k, int n_tokens, const int* __restrict__ idx, const double* __restrict__ W,
              const double* __restrict__ hcoef, const uint32_t* __restrict__ hmask,
              const double* __restrict__ vt, double* y) {
    extern __shared__ double smem[];
    Scatter sc{y};
    sc.init(smem, n_tokens);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double M = hcoef[i];
        const uint32_t mask = hmask[i];
        if (M != 0.0 && mask) {
            double Wa = 0.0, wv = 0.0;
            for (int j = 0; j < k; ++j)
                if (mask >> j & 1u) {
                    const double wj = W[(long long)j * ld + i];
                    Wa += wj;
                    wv += wj * __ldg(vt + idx[(long long)j * ld + i]);
                }
            const double tbar = wv / Wa;
            for (int j = 0; j < k; ++j)
                if (mask >> j & 1u) {
                    const int t = idx[(long long)j * ld + i];
                    sc.add(t, M * W[(long long)j * ld + i] * (__ldg(vt + t) - tbar));
                }
        }
    }
    sc.flush(smem, n_tokens);
}

__global__ void __launch_bounds__(kThreads)
k_diag_pair(long long m, long long ld, const int* __restrict__ idx, const double* __restrict__ hcoef, double* diag) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double h = hcoef[i];
        if (h != 0.0) { atomicAdd(diag + idx[i], h); atomicAdd(diag + idx[ld + i], h); }
    }
}

__global__ void __launch_bounds__(kThreads)
k_diag_geomean(long long m, long long ld, int k, const int* __restrict__ idx, const double* __restrict__ W,
               const double* __restrict__ hcoef, const uint32_t* __restrict__ hmask, double* diag) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double M = hcoef[i];
        const uint32_t mask = hmask[i];
        if (M != 0.0 && mask) {
            double Wa = 0.0;
            for (int j = 0; j < k; ++j)
                if (mask >> j & 1u) Wa += W[(long long)j * ld + i];
            for (int j = 0; j < k; ++j)
                if (mask >> j & 1u) {
                    const double wj = W[(long long)j * ld + i];
                    atomicAdd(diag + idx[(long long)j * ld + i], M * wj * (1.0 - wj / Wa));
                }
        }
    }
}

__global__ void __launch_bounds__(kThreads)
k_dense_pair(long long m, long long ld, int n, const int* __restrict__ idx, const double* __restrict__ hcoef, double* H) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double h = hcoef[i];
        if (h != 0.0) {
            const long long a = idx[i], b = idx[ld + i];
            atomicAdd(H + a * n + a, h); atomicAdd(H + b * n + b, h);
            atomicAdd(H + a * n + b, -h); atomicAdd(H + b * n + a, -h);
        }
    }
}

__global__ void __launch_bounds__(kThreads)
k_dense_geomean(long long m, long long ld, int k, int n, const int* __restrict__ idx, const double* __restrict__ W,
                const double* __restrict__ hcoef, const uint32_t* __restrict__ hmask, double* H) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double M = hcoef[i];
        const uint32_t mask = hmask[i];
        if (M != 0.0 && mask) {
            double Wa = 0.0;
            for (int j = 0; j < k; ++j)
                if (mask >> j & 1u) Wa += W[(long long)j * ld + i];
            for (int j = 0; j < k; ++j) {
                if (!(mask >> j & 1u)) continue;
                const double wj = W[(long long)j * ld + i];
                const long long tj = idx[(long long)j * ld + i];
                for (int l = 0; l < k; ++l) {
                    if (!(mask >> l & 1u)) continue;
                    const double wl = W[(long long)l * ld + i];
                    const long long tl = idx[(long long)l * ld + i];
                    atomicAdd(H + tj * n + tl, M * ((j == l ? wj : 0.0) - wj * wl / Wa));
                }
            }
        }
    }
}

// n-coin StableSwap: Hs_TT = C - (C1)(C1)' / (1'C1), C = diag(h^2) - h h' / (1 + k), from the per-slot h (hcoef
// [arity][ld], 0 off the traded set T, k = |T|); O(arity) per pool (cfmm_small::stablen_hvp).
template <typename Scatter>
__global__ void __launch_bounds__(kThreads)
k_hvp_stable_n(long long m, long long ld, int k, int n_tokens, const int* __restrict__ idx,
               const double* __restrict__ hcoef, const uint32_t* __restrict__ hmask, const double* __restrict__ vt,
               double* y) {
    extern __shared__ double smem[];
    Scatter sc{y};
    sc.init(smem, n_tokens);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        if (!hmask[i]) continue;
        double h[cfmm_small::KMAX], z[cfmm_small::KMAX], out[cfmm_small::KMAX];
        int id[cfmm_small::KMAX];
#pragma unroll
        for (int j = 0; j < cfmm_small::KMAX; ++j) {
            if (j < k) {
                id[j] = idx[(long long)j * ld + i];
                h[j] = hcoef[(long long)j * ld + i];
                z[j] = __ldg(vt + id[j]);
            }
        }
        cfmm_small::stablen_hvp<cfmm_small::KMAX>(k, h, z, out);
#pragma unroll
        for (int j = 0; j < cfmm_small::KMAX; ++j)
            if (j < k && h[j] != 0.0) sc.add(id[j], out[j]);
    }
    sc.flush(smem, n_tokens);
}

// the (C1)_j and 1'C1 of pool i's block (cfmm_small::stablen_c1), h loaded from hcoef [arity][ld]
__device__ __forceinline__ double stable_n_c1(long long i, long long ld, int k, const double* __restrict__ hcoef,
                                              double* h, double* c1, double& inv) {
#pragma unroll
    for (int j = 0; j < cfmm_small::KMAX; ++j)
        if (j < k) h[j] = hcoef[(long long)j * ld + i];
    return cfmm_small::stablen_c1<cfmm_small::KMAX>(k, h, c1, inv);
}

// diagonal: C_jj - (C1)_j^2 / (1'C1), C_jj = h_j^2 k / (1 + k)
__global__ void __launch_bounds__(kThreads)
k_diag_stable_n(long long m, long long ld, int k, const int* __restrict__ idx, const double* __restrict__ hcoef,
                const uint32_t* __restrict__ hmask, double* diag) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        if (!hmask[i]) continue;
        double h[cfmm_small::KMAX], c1[cfmm_small::KMAX], inv;
        const double s1 = stable_n_c1(i, ld, k, hcoef, h, c1, inv);
        if (!(s1 > 0.0)) continue;
#pragma unroll
        for (int j = 0; j < cfmm_small::KMAX; ++j)
            if (j < k && h[j] != 0.0)
                atomicAdd(diag + idx[(long long)j * ld + i], h[j] * h[j] * (1.0 - inv) - c1[j] * c1[j] / s1);
    }
}

__global__ void __launch_bounds__(kThreads)
k_dense_stable_n(long long m, long long ld, int k, int n, const int* __restrict__ idx, const double* __restrict__ hcoef,
                 const uint32_t* __restrict__ hmask, double* H) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        if (!hmask[i]) continue;
        double h[cfmm_small::KMAX], c1[cfmm_small::KMAX], inv;
        const double s1 = stable_n_c1(i, ld, k, hcoef, h, c1, inv);
        if (!(s1 > 0.0)) continue;
#pragma unroll
        for (int x = 0; x < cfmm_small::KMAX; ++x) {
            if (x >= k || h[x] == 0.0) continue;
            const long long tx = idx[(long long)x * ld + i];
#pragma unroll
            for (int y = 0; y < cfmm_small::KMAX; ++y) {
                if (y >= k || h[y] == 0.0) continue;
                const long long ty = idx[(long long)y * ld + i];
                atomicAdd(H + tx * n + ty, (x == y ? h[x] * h[x] : 0.0) - h[x] * h[y] * inv - c1[x] * c1[y] / s1);
            }
        }
    }
}

// three-coin cryptoswap: Hs = sum_{a<b} w_ab (e_a - e_b)(e_a - e_b)' over the pool's three edges, the weights in hcoef
// [3][ld] = (w01, w02, w12) (cfmm_small::cryptoswap3); O(1) per pool.  Pools without a trade (hmask 0) are skipped.
template <typename Scatter>
__global__ void __launch_bounds__(kThreads)
k_hvp_crypto3(long long m, long long ld, int n_tokens, const int* __restrict__ idx, const double* __restrict__ hcoef,
              const uint32_t* __restrict__ hmask, const double* __restrict__ vt, double* y) {
    extern __shared__ double smem[];
    Scatter sc{y};
    sc.init(smem, n_tokens);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        if (!hmask[i]) continue;
        const int t0 = idx[i], t1 = idx[ld + i], t2 = idx[2 * ld + i];
        const double z0 = __ldg(vt + t0), z1 = __ldg(vt + t1), z2 = __ldg(vt + t2);
        const double e01 = hcoef[i] * (z0 - z1), e02 = hcoef[ld + i] * (z0 - z2), e12 = hcoef[2 * ld + i] * (z1 - z2);
        sc.add(t0, e01 + e02);
        sc.add(t1, e12 - e01);
        sc.add(t2, -e02 - e12);
    }
    sc.flush(smem, n_tokens);
}

__global__ void __launch_bounds__(kThreads)
k_diag_crypto3(long long m, long long ld, const int* __restrict__ idx, const double* __restrict__ hcoef,
               const uint32_t* __restrict__ hmask, double* diag) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        if (!hmask[i]) continue;
        const double w01 = hcoef[i], w02 = hcoef[ld + i], w12 = hcoef[2 * ld + i];
        atomicAdd(diag + idx[i], w01 + w02);
        atomicAdd(diag + idx[ld + i], w01 + w12);
        atomicAdd(diag + idx[2 * ld + i], w02 + w12);
    }
}

__global__ void __launch_bounds__(kThreads)
k_dense_crypto3(long long m, long long ld, int n, const int* __restrict__ idx, const double* __restrict__ hcoef,
                const uint32_t* __restrict__ hmask, double* H) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        if (!hmask[i]) continue;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const double w = hcoef[q * ld + i];
            if (w == 0.0) continue;
            const long long a = idx[(q == 2 ? 1 : 0) * ld + i], b = idx[(q == 0 ? 1 : 2) * ld + i];
            atomicAdd(H + a * n + a, w); atomicAdd(H + b * n + b, w);
            atomicAdd(H + a * n + b, -w); atomicAdd(H + b * n + a, -w);
        }
    }
}

__global__ void __launch_bounds__(kThreads)
k_sum_update(long long m, long long ld, const double* __restrict__ R, const double* __restrict__ lambda,
             double* thbar, double* move) {
    double mx = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < 2 * m; q += stride) {
        const long long i = (q < m) ? q : ld + (q - m);
        const double th = lambda[i];
        mx = fmax(mx, fabs(th - thbar[i]) / R[i]);
        thbar[i] = th;
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0 && mx > 0.0) {
        // non-negative doubles order like their bit patterns
        atomicMax(reinterpret_cast<unsigned long long*>(move), (unsigned long long)__double_as_longlong(mx));
    }
}

// price bins: tbar <- t = lambda_0 - delta_0 (row 0 of theta_bar; row 1 is not used), move = max |change| / S with S
// the width of the pool's net-flow domain at its fee
__global__ void __launch_bounds__(kThreads)
k_bins_update(long long m, long long ld, const double* __restrict__ rec, const double* __restrict__ P,
              const double* __restrict__ gamma, const double* __restrict__ delta, const double* __restrict__ lambda,
              double* thbar, double* move) {
    double mx = 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        const double* rp = rec + 4 * (long long)P[i];
        const double S = rp[4 * ((long long)P[ld + i] - 1)] - rp[0] / gamma[i];
        const double t = lambda[i] - delta[i];
        mx = fmax(mx, fabs(t - thbar[i]) / S);
        thbar[i] = t;
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0 && mx > 0.0)
        atomicMax(reinterpret_cast<unsigned long long*>(move), (unsigned long long)__double_as_longlong(mx));
}

// ---------------------------------------------------------------------------------------------
// launch helpers
// ---------------------------------------------------------------------------------------------
inline int grid_for(long long m, int blocks_per_sm) {
    long long need = (m + kThreads - 1) / kThreads;
    long long cap = (long long)num_sms() * blocks_per_sm;
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

inline bool use_shared(int n_tokens, long long m) {
    if (g_scatter_mode == 1 || g_scatter_mode == 3) return false;
    const bool fits = (size_t)n_tokens * sizeof(double) <= 96 * 1024;
    if (g_scatter_mode == 2) return fits;
    // auto: privatise only when each CTA makes many more contributions than it has bins to flush
    return fits && (2 * m / ((long long)num_sms() * 2) > 8LL * n_tokens);
}

template <typename K>
inline void allow_smem(K kernel, size_t bytes) {
    if (bytes > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

inline bool tma_ok(const cfmm_bucket* b) {
    auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    return (b->stride % kTile) == 0 && al(b->reserves) && al(b->tok_idx) && al(b->gamma);
}

template <int KIND, bool TRADES, bool HESS>
int launch_pair(const cfmm_bucket* b, int n_tokens, const double* nu, double eps, double* psi, double* arb,
                const cfmm_eval_out* out, cudaStream_t st) {
    const long long m = b->n_pools;
    double* delta = out ? out->delta : nullptr;
    double* lambda = out ? out->lambda : nullptr;
    double* hcoef = out ? out->hcoef : nullptr;
    // per-slot auxiliary array: fill multipliers of constant-sum orders | virtual-reserve offsets of bounded products |
    // the parameters and state of E-CLPs | the parameters and targets of PMMs.  None of the last three has a TMA-staged
    // kernel: the LDG path only.
    constexpr bool kWeights = KIND == CFMM_KIND_BOUNDED_PRODUCT || KIND == CFMM_KIND_ECLP || KIND == CFMM_KIND_PMM;
    const double* aux = kWeights ? b->weights : b->theta_bar;
    if (!kWeights && (g_scatter_mode == 0 || g_scatter_mode == 3) && tma_ok(b)) {
        auto kern = k_eval_pair_tma<kWeights ? CFMM_KIND_PRODUCT : KIND, TRADES, HESS>;
        const size_t sm = (size_t)kStages * kStageBytes;
        static bool attr_set = false;      // per instantiation
        if (!attr_set) {
            cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            attr_set = true;
        }
        const long long ntiles = (m + kTile - 1) / kTile;
        const long long cap = 2LL * num_sms();
        const int grid = (int)(ntiles < cap ? ntiles : cap);
        kern<<<grid, kTmaThreads, sm, st>>>(m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->theta_bar,
                                            eps, nu, psi, arb, delta, lambda, hcoef);
        return check_launch();
    }
    if (use_shared(n_tokens, m)) {
        const size_t sm = (size_t)n_tokens * sizeof(double);
        auto kern = k_eval_pair<KIND, SharedScatter, TRADES, HESS>;
        allow_smem(kern, sm);
        kern<<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, aux,
                                                    eps, nu, psi, arb, delta, lambda, hcoef);
    } else {
        k_eval_pair<KIND, GlobalScatter, TRADES, HESS><<<grid_for(m, 8), kThreads, 0, st>>>(
            m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, aux, eps, nu, psi, arb, delta, lambda, hcoef);
    }
    return check_launch();
}

// StableSwap buckets: the LDG path only (the kernel is compute-bound; there is no TMA-staged variant)
template <bool TRADES, bool HESS>
int launch_stable(const cfmm_bucket* b, int n_tokens, const double* nu, double* psi, double* arb,
                  const cfmm_eval_out* out, cudaStream_t st) {
    const long long m = b->n_pools;
    double* delta = out ? out->delta : nullptr;
    double* lambda = out ? out->lambda : nullptr;
    double* hcoef = out ? out->hcoef : nullptr;
    if (use_shared(n_tokens, m)) {
        const size_t sm = (size_t)n_tokens * sizeof(double);
        auto kern = k_eval_stable<SharedScatter, TRADES, HESS>;
        allow_smem(kern, sm);
        kern<<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights,
                                                    b->logrw, nu, psi, arb, delta, lambda, hcoef);
    } else {
        k_eval_stable<GlobalScatter, TRADES, HESS><<<grid_for(m, 8), kThreads, 0, st>>>(
            m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights, b->logrw, nu, psi, arb, delta, lambda,
            hcoef);
    }
    return check_launch();
}

// cryptoswap buckets: the LDG path only, as for StableSwap
template <bool TRADES, bool HESS>
int launch_crypto(const cfmm_bucket* b, int n_tokens, const double* nu, double* psi, double* arb,
                  const cfmm_eval_out* out, cudaStream_t st) {
    const long long m = b->n_pools;
    double* delta = out ? out->delta : nullptr;
    double* lambda = out ? out->lambda : nullptr;
    double* hcoef = out ? out->hcoef : nullptr;
    if (use_shared(n_tokens, m)) {
        const size_t sm = (size_t)n_tokens * sizeof(double);
        auto kern = k_eval_crypto<SharedScatter, TRADES, HESS>;
        allow_smem(kern, sm);
        kern<<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights,
                                                    b->logrw, nu, psi, arb, delta, lambda, hcoef);
    } else {
        k_eval_crypto<GlobalScatter, TRADES, HESS><<<grid_for(m, 8), kThreads, 0, st>>>(
            m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights, b->logrw, nu, psi, arb, delta, lambda,
            hcoef);
    }
    return check_launch();
}

// three-coin cryptoswap buckets: the LDG path only, as for two coins
template <bool TRADES, bool HESS>
int launch_crypto3(const cfmm_bucket* b, int n_tokens, const double* nu, double* psi, double* arb,
                   const cfmm_eval_out* out, cudaStream_t st) {
    const long long m = b->n_pools;
    double* delta = out ? out->delta : nullptr;
    double* lambda = out ? out->lambda : nullptr;
    double* hcoef = out ? out->hcoef : nullptr;
    uint32_t* hmask = out ? out->hmask : nullptr;
    if (use_shared(n_tokens, m * 3 / 2)) {
        const size_t sm = (size_t)n_tokens * sizeof(double);
        auto kern = k_eval_crypto3<SharedScatter, TRADES, HESS>;
        allow_smem(kern, sm);
        kern<<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights,
                                                    b->logrw, nu, psi, arb, delta, lambda, hcoef, hmask);
    } else {
        k_eval_crypto3<GlobalScatter, TRADES, HESS><<<grid_for(m, 8), kThreads, 0, st>>>(
            m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights, b->logrw, nu, psi, arb, delta, lambda,
            hcoef, hmask);
    }
    return check_launch();
}

int dispatch_crypto3(const cfmm_bucket* b, int n_tokens, const double* nu, double* psi, double* arb,
                     const cfmm_eval_out* out, cudaStream_t st) {
    const bool trades = out && out->delta && out->lambda;
    const bool hess = out && out->hcoef && out->hmask;
    if (trades && hess) return launch_crypto3<true, true>(b, n_tokens, nu, psi, arb, out, st);
    if (trades) return launch_crypto3<true, false>(b, n_tokens, nu, psi, arb, out, st);
    if (hess) return launch_crypto3<false, true>(b, n_tokens, nu, psi, arb, out, st);
    return launch_crypto3<false, false>(b, n_tokens, nu, psi, arb, out, st);
}

// n-coin StableSwap buckets: the LDG path only, as for two coins
template <int K, bool TRADES, bool HESS>
int launch_stable_n(const cfmm_bucket* b, int n_tokens, const double* nu, double* psi, double* arb,
                    const cfmm_eval_out* out, cudaStream_t st) {
    const long long m = b->n_pools;
    double* delta = out ? out->delta : nullptr;
    double* lambda = out ? out->lambda : nullptr;
    double* hcoef = out ? out->hcoef : nullptr;
    uint32_t* hmask = out ? out->hmask : nullptr;
    if (use_shared(n_tokens, m * K / 2)) {
        const size_t sm = (size_t)n_tokens * sizeof(double);
        auto kern = k_eval_stable_n<K, SharedScatter, TRADES, HESS>;
        allow_smem(kern, sm);
        kern<<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights,
                                                    b->logrw, nu, psi, arb, delta, lambda, hcoef, hmask);
    } else {
        k_eval_stable_n<K, GlobalScatter, TRADES, HESS><<<grid_for(m, 4), kThreads, 0, st>>>(
            m, b->stride, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights, b->logrw, nu, psi, arb, delta, lambda,
            hcoef, hmask);
    }
    return check_launch();
}

template <int K>
int dispatch_stable_n(const cfmm_bucket* b, int n_tokens, const double* nu, double* psi, double* arb,
                      const cfmm_eval_out* out, cudaStream_t st) {
    const bool trades = out && out->delta && out->lambda;
    const bool hess = out && out->hcoef && out->hmask;
    if (trades && hess) return launch_stable_n<K, true, true>(b, n_tokens, nu, psi, arb, out, st);
    if (trades) return launch_stable_n<K, true, false>(b, n_tokens, nu, psi, arb, out, st);
    if (hess) return launch_stable_n<K, false, true>(b, n_tokens, nu, psi, arb, out, st);
    return launch_stable_n<K, false, false>(b, n_tokens, nu, psi, arb, out, st);
}

// concentrated buckets: the LDG path only, like the StableSwap kinds (the records are read by a data-dependent search)
template <bool TRADES, bool HESS>
int launch_ladder(const cfmm_bucket* b, int n_tokens, const double* nu, double* psi, double* arb,
                  const cfmm_eval_out* out, cudaStream_t st) {
    const long long m = b->n_pools;
    double* delta = out ? out->delta : nullptr;
    double* lambda = out ? out->lambda : nullptr;
    double* hcoef = out ? out->hcoef : nullptr;
    if (use_shared(n_tokens, m)) {
        const size_t sm = (size_t)n_tokens * sizeof(double);
        auto kern = k_eval_ladder<SharedScatter, TRADES, HESS>;
        allow_smem(kern, sm);
        kern<<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->tok_idx, b->gamma, b->weights, b->logrw, nu,
                                                    psi, arb, delta, lambda, hcoef);
    } else {
        k_eval_ladder<GlobalScatter, TRADES, HESS><<<grid_for(m, 8), kThreads, 0, st>>>(
            m, b->stride, n_tokens, b->tok_idx, b->gamma, b->weights, b->logrw, nu, psi, arb, delta, lambda, hcoef);
    }
    return check_launch();
}

// price-bin buckets: the LDG path only, like the concentrated kind
template <bool TRADES, bool HESS>
int launch_bins(const cfmm_bucket* b, int n_tokens, const double* nu, double eps, double* psi, double* arb,
                const cfmm_eval_out* out, cudaStream_t st) {
    const long long m = b->n_pools;
    double* delta = out ? out->delta : nullptr;
    double* lambda = out ? out->lambda : nullptr;
    double* hcoef = out ? out->hcoef : nullptr;
    if (use_shared(n_tokens, m)) {
        const size_t sm = (size_t)n_tokens * sizeof(double);
        auto kern = k_eval_bins<SharedScatter, TRADES, HESS>;
        allow_smem(kern, sm);
        kern<<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->tok_idx, b->gamma, b->weights, b->logrw,
                                                    b->theta_bar, eps, nu, psi, arb, delta, lambda, hcoef);
    } else {
        k_eval_bins<GlobalScatter, TRADES, HESS><<<grid_for(m, 8), kThreads, 0, st>>>(
            m, b->stride, n_tokens, b->tok_idx, b->gamma, b->weights, b->logrw, b->theta_bar, eps, nu, psi, arb, delta,
            lambda, hcoef);
    }
    return check_launch();
}

template <int KIND, bool TRADES, bool HESS>
int launch_kind(const cfmm_bucket* b, int n_tokens, const double* nu, double eps, double* psi, double* arb,
                const cfmm_eval_out* out, cudaStream_t st) {
    if constexpr (KIND == CFMM_KIND_CONCENTRATED)
        return launch_ladder<TRADES, HESS>(b, n_tokens, nu, psi, arb, out, st);
    else if constexpr (KIND == CFMM_KIND_BINS)
        return launch_bins<TRADES, HESS>(b, n_tokens, nu, eps, psi, arb, out, st);
    else if constexpr (KIND == CFMM_KIND_STABLESWAP)
        return launch_stable<TRADES, HESS>(b, n_tokens, nu, psi, arb, out, st);
    else if constexpr (KIND == CFMM_KIND_CRYPTOSWAP)
        return launch_crypto<TRADES, HESS>(b, n_tokens, nu, psi, arb, out, st);
    else
        return launch_pair<KIND, TRADES, HESS>(b, n_tokens, nu, eps, psi, arb, out, st);
}

template <int KIND>
int dispatch_pair(const cfmm_bucket* b, int n_tokens, const double* nu, double eps, double* psi, double* arb,
                  const cfmm_eval_out* out, cudaStream_t st) {
    const bool trades = out && out->delta && out->lambda;
    const bool hess = out && out->hcoef;
    if (trades && hess) return launch_kind<KIND, true, true>(b, n_tokens, nu, eps, psi, arb, out, st);
    if (trades) return launch_kind<KIND, true, false>(b, n_tokens, nu, eps, psi, arb, out, st);
    if (hess) return launch_kind<KIND, false, true>(b, n_tokens, nu, eps, psi, arb, out, st);
    return launch_kind<KIND, false, false>(b, n_tokens, nu, eps, psi, arb, out, st);
}

template <int K, bool TRADES, bool HESS>
int launch_geomean(const cfmm_bucket* b, int n_tokens, const double* nu, const double* lognu, double* psi,
                   double* arb, const cfmm_eval_out* out, cudaStream_t st) {
    const long long m = b->n_pools;
    double* delta = out ? out->delta : nullptr;
    double* lambda = out ? out->lambda : nullptr;
    double* hcoef = out ? out->hcoef : nullptr;
    uint32_t* hmask = out ? out->hmask : nullptr;
    if (use_shared(n_tokens, m * b->arity / 2)) {
        const size_t sm = (size_t)n_tokens * sizeof(double);
        auto kern = k_eval_geomean<K, SharedScatter, TRADES, HESS>;
        allow_smem(kern, sm);
        kern<<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, b->arity, n_tokens, b->reserves, b->tok_idx, b->gamma,
                                                    b->weights, b->logrw, nu, lognu, psi, arb, delta, lambda,
                                                    hcoef, hmask);
    } else {
        k_eval_geomean<K, GlobalScatter, TRADES, HESS><<<grid_for(m, 4), kThreads, 0, st>>>(
            m, b->stride, b->arity, n_tokens, b->reserves, b->tok_idx, b->gamma, b->weights, b->logrw, nu, lognu, psi, arb,
            delta, lambda, hcoef, hmask);
    }
    return check_launch();
}

template <int K>
int dispatch_geomean_flags(const cfmm_bucket* b, int n_tokens, const double* nu, const double* lognu,
                           double* psi, double* arb, const cfmm_eval_out* out, cudaStream_t st) {
    const bool trades = out && out->delta && out->lambda;
    const bool hess = out && out->hcoef && out->hmask;
    if (trades && hess) return launch_geomean<K, true, true>(b, n_tokens, nu, lognu, psi, arb, out, st);
    if (trades) return launch_geomean<K, true, false>(b, n_tokens, nu, lognu, psi, arb, out, st);
    if (hess) return launch_geomean<K, false, true>(b, n_tokens, nu, lognu, psi, arb, out, st);
    return launch_geomean<K, false, false>(b, n_tokens, nu, lognu, psi, arb, out, st);
}

int validate(const cfmm_bucket* b, int n_tokens) {
    if (!b) return CFMM_E_NULL;
    if (b->n_pools < 0 || n_tokens <= 0 || b->stride < b->n_pools) return CFMM_E_SIZE;
    if (b->n_pools > 0 && (!b->reserves || !b->tok_idx || !b->gamma)) return CFMM_E_NULL;
    switch (b->kind) {
        case CFMM_KIND_PRODUCT:
        case CFMM_KIND_SUM:
            if (b->arity != 2) return CFMM_E_KIND;
            break;
        case CFMM_KIND_GEOMEAN:
            if (b->arity < 2 || b->arity > 32) return CFMM_E_KIND;
            if (b->n_pools > 0 && (!b->weights || !b->logrw)) return CFMM_E_NULL;
            break;
        case CFMM_KIND_BOUNDED_PRODUCT:
            if (b->arity != 2) return CFMM_E_KIND;
            if (b->n_pools > 0 && !b->weights) return CFMM_E_NULL;       // the offsets
            break;
        case CFMM_KIND_STABLESWAP:
            if (b->arity != 2) return CFMM_E_KIND;
            if (b->n_pools > 0 && (!b->weights || !b->logrw)) return CFMM_E_NULL;   // rates; (A, D)
            break;
        case CFMM_KIND_STABLESWAP_N:
            if (b->arity < 2 || b->arity > 8) return CFMM_E_KIND;
            if (b->n_pools > 0 && (!b->weights || !b->logrw)) return CFMM_E_NULL;   // rates; (A, D)
            break;
        case CFMM_KIND_CONCENTRATED:
            if (b->arity != 2) return CFMM_E_KIND;
            if (b->n_pools > 0 && (!b->weights || !b->logrw)) return CFMM_E_NULL;   // records; (s, c, first, T)
            break;
        case CFMM_KIND_CRYPTOSWAP:
            if (b->arity != 2) return CFMM_E_KIND;
            if (b->n_pools > 0 && (!b->weights || !b->logrw)) return CFMM_E_NULL;   // price scales; (A, G, D)
            break;
        case CFMM_KIND_CRYPTOSWAP_3:
            if (b->arity != 3) return CFMM_E_KIND;
            if (b->n_pools > 0 && (!b->weights || !b->logrw)) return CFMM_E_NULL;   // price scales; (A, G, D)
            break;
        case CFMM_KIND_BINS:
            if (b->arity != 2) return CFMM_E_KIND;
            if (b->n_pools > 0 && (!b->weights || !b->logrw || !b->theta_bar)) return CFMM_E_NULL;   // records; tbar
            break;
        case CFMM_KIND_ECLP:
            if (b->arity != 2) return CFMM_E_KIND;
            if (b->n_pools > 0 && !b->weights) return CFMM_E_NULL;       // (alpha, beta, c, s, lam, r, p)
            break;
        case CFMM_KIND_PMM:
            if (b->arity != 2) return CFMM_E_KIND;
            if (b->n_pools > 0 && !b->weights) return CFMM_E_NULL;       // (pi, k, B0, Q0)
            break;
        default:
            return CFMM_E_KIND;
    }
    return CFMM_OK;
}

}  // namespace

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int cfmm_arb_eval(const cfmm_bucket* b, int32_t n_tokens, const double* nu, const double* log_nu, double eps,
                  double* psi, double* arb, const cfmm_eval_out* out, void* stream) {
    int rc = validate(b, n_tokens);
    if (rc) return rc;
    if (!nu || !psi || !arb) return CFMM_E_NULL;
    if (b->n_pools == 0) return CFMM_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (b->kind) {
        case CFMM_KIND_PRODUCT:
            return dispatch_pair<CFMM_KIND_PRODUCT>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_SUM:
            return dispatch_pair<CFMM_KIND_SUM>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_BOUNDED_PRODUCT:
            return dispatch_pair<CFMM_KIND_BOUNDED_PRODUCT>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_STABLESWAP:
            return dispatch_pair<CFMM_KIND_STABLESWAP>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_CONCENTRATED:
            return dispatch_pair<CFMM_KIND_CONCENTRATED>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_CRYPTOSWAP:
            return dispatch_pair<CFMM_KIND_CRYPTOSWAP>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_BINS:
            return dispatch_pair<CFMM_KIND_BINS>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_ECLP:
            return dispatch_pair<CFMM_KIND_ECLP>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_PMM:
            return dispatch_pair<CFMM_KIND_PMM>(b, n_tokens, nu, eps, psi, arb, out, st);
        case CFMM_KIND_CRYPTOSWAP_3:
            return dispatch_crypto3(b, n_tokens, nu, psi, arb, out, st);
        case CFMM_KIND_STABLESWAP_N:
            switch (b->arity) {
                case 2: return dispatch_stable_n<2>(b, n_tokens, nu, psi, arb, out, st);
                case 3: return dispatch_stable_n<3>(b, n_tokens, nu, psi, arb, out, st);
                case 4: return dispatch_stable_n<4>(b, n_tokens, nu, psi, arb, out, st);
                case 5: return dispatch_stable_n<5>(b, n_tokens, nu, psi, arb, out, st);
                case 6: return dispatch_stable_n<6>(b, n_tokens, nu, psi, arb, out, st);
                case 7: return dispatch_stable_n<7>(b, n_tokens, nu, psi, arb, out, st);
                default: return dispatch_stable_n<8>(b, n_tokens, nu, psi, arb, out, st);
            }
        default:
            break;
    }
    if (!log_nu) return CFMM_E_NULL;
    switch (b->arity) {
        case 2: return dispatch_geomean_flags<2>(b, n_tokens, nu, log_nu, psi, arb, out, st);
        case 3: return dispatch_geomean_flags<3>(b, n_tokens, nu, log_nu, psi, arb, out, st);
        case 4: return dispatch_geomean_flags<4>(b, n_tokens, nu, log_nu, psi, arb, out, st);
        case 5: return dispatch_geomean_flags<5>(b, n_tokens, nu, log_nu, psi, arb, out, st);
        case 6: return dispatch_geomean_flags<6>(b, n_tokens, nu, log_nu, psi, arb, out, st);
        case 7: return dispatch_geomean_flags<7>(b, n_tokens, nu, log_nu, psi, arb, out, st);
        case 8: return dispatch_geomean_flags<8>(b, n_tokens, nu, log_nu, psi, arb, out, st);
        default: return dispatch_geomean_flags<0>(b, n_tokens, nu, log_nu, psi, arb, out, st);
    }
}

int cfmm_hvp(const cfmm_bucket* b, int32_t n_tokens, const double* hcoef, const uint32_t* hmask,
             const double* vt, double* y, void* stream) {
    int rc = validate(b, n_tokens);
    if (rc) return rc;
    if (!hcoef || !vt || !y) return CFMM_E_NULL;
    if (b->n_pools == 0) return CFMM_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long m = b->n_pools;
    const bool sh = use_shared(n_tokens, m * b->arity / 2);
    const size_t sm = sh ? (size_t)n_tokens * sizeof(double) : 0;
    if (b->kind == CFMM_KIND_STABLESWAP_N) {
        if (!hmask) return CFMM_E_NULL;
        if (sh) {
            allow_smem(k_hvp_stable_n<SharedScatter>, sm);
            k_hvp_stable_n<SharedScatter><<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, b->arity, n_tokens,
                                                                                b->tok_idx, hcoef, hmask, vt, y);
        } else {
            k_hvp_stable_n<GlobalScatter><<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, b->arity, n_tokens,
                                                                               b->tok_idx, hcoef, hmask, vt, y);
        }
    } else if (b->kind == CFMM_KIND_CRYPTOSWAP_3) {
        if (!hmask) return CFMM_E_NULL;
        if (sh) {
            allow_smem(k_hvp_crypto3<SharedScatter>, sm);
            k_hvp_crypto3<SharedScatter><<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->tok_idx, hcoef,
                                                                               hmask, vt, y);
        } else {
            k_hvp_crypto3<GlobalScatter><<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, n_tokens, b->tok_idx, hcoef,
                                                                              hmask, vt, y);
        }
    } else if (b->kind == CFMM_KIND_GEOMEAN) {
        if (!hmask) return CFMM_E_NULL;
        if (sh) {
            allow_smem(k_hvp_geomean<SharedScatter>, sm);
            k_hvp_geomean<SharedScatter><<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, b->arity, n_tokens, b->tok_idx,
                                                                               b->weights, hcoef, hmask, vt, y);
        } else {
            k_hvp_geomean<GlobalScatter><<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, b->arity, n_tokens, b->tok_idx,
                                                                              b->weights, hcoef, hmask, vt, y);
        }
    } else {
        if (sh) {
            allow_smem(k_hvp_pair<SharedScatter>, sm);
            k_hvp_pair<SharedScatter><<<grid_for(m, 2), kThreads, sm, st>>>(m, b->stride, n_tokens, b->tok_idx, hcoef, vt, y);
        } else {
            k_hvp_pair<GlobalScatter><<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, n_tokens, b->tok_idx, hcoef, vt, y);
        }
    }
    return check_launch();
}

int cfmm_hess_diag(const cfmm_bucket* b, int32_t n_tokens, const double* hcoef, const uint32_t* hmask,
                   double* diag, void* stream) {
    int rc = validate(b, n_tokens);
    if (rc) return rc;
    if (!hcoef || !diag) return CFMM_E_NULL;
    if (b->n_pools == 0) return CFMM_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long m = b->n_pools;
    if (b->kind == CFMM_KIND_STABLESWAP_N) {
        if (!hmask) return CFMM_E_NULL;
        k_diag_stable_n<<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, b->arity, b->tok_idx, hcoef, hmask, diag);
    } else if (b->kind == CFMM_KIND_CRYPTOSWAP_3) {
        if (!hmask) return CFMM_E_NULL;
        k_diag_crypto3<<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, b->tok_idx, hcoef, hmask, diag);
    } else if (b->kind == CFMM_KIND_GEOMEAN) {
        if (!hmask) return CFMM_E_NULL;
        k_diag_geomean<<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, b->arity, b->tok_idx, b->weights, hcoef, hmask, diag);
    } else {
        k_diag_pair<<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, b->tok_idx, hcoef, diag);
    }
    return check_launch();
}

int cfmm_hess_dense(const cfmm_bucket* b, int32_t n_tokens, const double* hcoef, const uint32_t* hmask,
                    double* H, void* stream) {
    int rc = validate(b, n_tokens);
    if (rc) return rc;
    if (!hcoef || !H) return CFMM_E_NULL;
    if (b->n_pools == 0) return CFMM_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long m = b->n_pools;
    if (b->kind == CFMM_KIND_STABLESWAP_N) {
        if (!hmask) return CFMM_E_NULL;
        k_dense_stable_n<<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, b->arity, n_tokens, b->tok_idx, hcoef, hmask,
                                                               H);
    } else if (b->kind == CFMM_KIND_CRYPTOSWAP_3) {
        if (!hmask) return CFMM_E_NULL;
        k_dense_crypto3<<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, n_tokens, b->tok_idx, hcoef, hmask, H);
    } else if (b->kind == CFMM_KIND_GEOMEAN) {
        if (!hmask) return CFMM_E_NULL;
        k_dense_geomean<<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, b->arity, n_tokens, b->tok_idx, b->weights, hcoef,
                                                              hmask, H);
    } else {
        k_dense_pair<<<grid_for(m, 8), kThreads, 0, st>>>(m, b->stride, n_tokens, b->tok_idx, hcoef, H);
    }
    return check_launch();
}

int cfmm_sum_update_multipliers(const cfmm_bucket* b, const double* lambda, double* theta_bar_out, double* move,
                                void* stream) {
    if (!b) return CFMM_E_NULL;
    if (b->kind != CFMM_KIND_SUM || b->arity != 2) return CFMM_E_KIND;
    if (b->n_pools < 0) return CFMM_E_SIZE;
    if (b->n_pools == 0) return CFMM_OK;
    if (!lambda || !theta_bar_out || !move || !b->reserves) return CFMM_E_NULL;
    k_sum_update<<<grid_for(2 * b->n_pools, 8), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        b->n_pools, b->stride, b->reserves, lambda, theta_bar_out, move);
    return check_launch();
}

int cfmm_bins_update_multipliers(const cfmm_bucket* b, const double* delta, const double* lambda, double* theta_bar_out,
                                 double* move, void* stream) {
    if (!b) return CFMM_E_NULL;
    if (b->kind != CFMM_KIND_BINS || b->arity != 2) return CFMM_E_KIND;
    if (b->n_pools < 0 || b->stride < b->n_pools) return CFMM_E_SIZE;
    if (b->n_pools == 0) return CFMM_OK;
    if (!delta || !lambda || !theta_bar_out || !move || !b->weights || !b->logrw || !b->gamma) return CFMM_E_NULL;
    k_bins_update<<<grid_for(b->n_pools, 8), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        b->n_pools, b->stride, b->weights, b->logrw, b->gamma, delta, lambda, theta_bar_out, move);
    return check_launch();
}

int cfmm_zero(void* ptr, int64_t bytes, void* stream) {
    if (!ptr) return CFMM_E_NULL;
    if (bytes < 0) return CFMM_E_SIZE;
    cudaError_t e = cudaMemsetAsync(ptr, 0, (size_t)bytes, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) { g_last_err = e; return CFMM_E_CUDA; }
    return CFMM_OK;
}

int cfmm_set_scatter_mode(int32_t mode) {
    if (mode < 0 || mode > 3) return CFMM_E_KIND;
    g_scatter_mode = mode;
    return CFMM_OK;
}

int64_t cfmm_launch_count(void) { return g_launches.load(); }
void cfmm_reset_launch_count(void) { g_launches.store(0); }
const char* cfmm_last_cuda_error(void) { return cudaGetErrorString(g_last_err); }
const char* cfmm_version(void) { return "cfmm_b200 0.1 (sm_90a)"; }

}  // extern "C"
