// cfmm_small.cuh -- the WHOLE dual solve of one small routing problem in one thread.
//
// The reference's three scripts are small problems (5 pools, 3-5 tokens), and two-asset.py solves 50 of them in a
// python loop, rebuilding the cvxpy problem each time (two-asset.py:40-100).  A batch of such problems is data
// parallel over PROBLEMS, not pools: one thread owns one problem and runs the complete method -- per-pool closed
// forms (arbitrage.py:60-74), psi (arbitrage.py:54), projected Newton in log-price coordinates with a dense Hessian,
// method of multipliers on the constant-sum fills -- without ever leaving the kernel.  Same algorithm, constants and
// control flow as oracle/cfmm_oracle.py::solve (which the tests check it against).
//
// All per-problem state lives in a caller-provided workspace, element-interleaved across problems (element e of
// problem p at work[e * stride + p]) so the 32 problems of a warp touch consecutive addresses.
//
// The file is plain C++ when compiled without nvcc: tests/ builds it for the host to check the control flow without a
// GPU.  The product only ever runs it through k_batch_solve (cfmm_small.cu).
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define CFMM_HD __host__ __device__
#define CFMM_UNROLL _Pragma("unroll")
#else
#define CFMM_HD
#define CFMM_UNROLL
#endif

namespace cfmm_small {

constexpr int KMAX = 8;              // largest weighted-pool arity (the reference uses 3..5; cfg3/4 use 2..8)
constexpr int NTOK_MAX = 64;         // dense n x n Newton systems per thread: keep n small
constexpr double TINY = 1e-300;
constexpr double DT_MAX = 3.0;       // largest log-price change of one Newton step

struct Pools {                       // CSR problem data (device pointers in the kernel)
    const int64_t* pool_ptr;         // [m+1]
    const int32_t* tok;              // [nnz]   token of every slot            arbitrage.py:6-12
    const double* R;                 // [nnz]   reserves                       arbitrage.py:14-20
    const double* w;                 // [nnz]   normalised weights | 0 on constant-sum pools | virtual offsets (kind 3) |
                                     //         rates (kind 4) | p_j / D (kinds 8, 9)
    const double* logrw;             // [nnz]   log(R/w) | kind 4: A at the pool's first slot, its invariant D at the second |
                                     //         kinds 8, 9: A, then the curve gamma G
    const double* gamma;             // [m]     fees                           arbitrage.py:22-28
    const uint8_t* kind;             // [m]     1 = constant sum; 3 = bounded-liquidity product; 4 = StableSwap (2 coins;
                                     //         2..KMAX in the STABLE_N instance); 8 = two-coin cryptoswap (CRYPTO instance);
                                     //         9 = three-coin cryptoswap (CRYPTO3 instance);
                                     //         0 or 2 = weighted geometric mean
                                     //         (constant product = equal weights)
};

struct Params {
    double tol, eps0, eps_min, eps_shrink, floor_rel;
    int max_outer, max_inner;
};

struct Vec {                         // strided view into the interleaved workspace
    double* p;
    int64_t s;
    CFMM_HD double& operator[](int64_t j) const { return p[j * s]; }
};

struct Problem {
    int n;                           // tokens
    int64_t p0, p1;                  // pool range
    int64_t off0;                    // pool_ptr[p0]
    const double* c;                 // [n] objective                         arbitrage.py:31-36 / liquidation.py:57
    const double* a;                 // [n] endowment                         liquidation.py:30-36 / two-asset.py:45
    const uint8_t* flags;            // [n] bit0: psi_j + a_j == 0, bit1: psi_j free (nu_j = c_j)
    Vec theta_bar, theta_new;        // [nnz of the problem] multipliers of the constant-sum limit orders
    double* delta;                   // nullable; indexed by CSR offset
    double* lam;
};

struct Stats { double value, dual, gap, infeas, err; int iters, evals, status; };

CFMM_HD inline bool is_eq(const Problem& Q, int j) { return Q.flags[j] & 1; }
CFMM_HD inline bool is_pinned(const Problem& Q, int j) { return Q.flags[j] & 2; }

// Constant product on virtual reserves V = R + o with the real reserves R >= 0 (one Uniswap-v3 tick range; not a
// reference atom).  The optimal trade is the constant-product one on V; when it would pay out more than R_b the payout
// is capped there and the tender follows from the curve, (V_a + gamma D_a)(V_b - R_b) = V_a V_b.  hc = coefficient of
// [[1,-1],[-1,1]] in the scaled Hessian (0 at the cap: the trade no longer depends on the prices).
// Shared by the per-thread solver below and the pool-parallel kernel k_eval_pair (cfmm_kernels.cu).
CFMM_HD inline void bounded_pair(double R0, double R1, double o0, double o1, double gam, double n0, double n1,
                                 double* D, double* L, double& hc) {
    const double R[2] = {R0, R1}, o[2] = {o0, o1};
    const double V[2] = {R0 + o0, R1 + o1};
    const double pv[2] = {n0 * V[0], n1 * V[1]};
    D[0] = D[1] = L[0] = L[1] = 0.0;
    hc = 0.0;
    for (int dir = 0; dir < 2; ++dir) {
        const int ta = dir, tb = 1 - dir;
        if (gam * pv[tb] > pv[ta]) {
            const double t = sqrt(gam * pv[tb] / pv[ta]);
            const double lout = V[tb] * (1.0 - 1.0 / t);
            if (lout > R[tb]) {                                        // payout capped by the real reserve
                L[tb] = R[tb];
                D[ta] = V[ta] * R[tb] / (o[tb] * gam);
            } else {
                L[tb] = lout;
                D[ta] = V[ta] * (t - 1.0) / gam;
                hc += 0.5 * sqrt(pv[0] * pv[1] / gam);
            }
        }
    }
}

// Elliptic concentrated-liquidity pool (Gyroscope E-CLP; not a reference atom).  Price range [alpha, beta] (token 1 per
// token 0), rotation (c, s) = (cos phi, sin phi), stretch lam >= 1; A = [[c/lam, -s/lam], [s, c]], M = (A'A)^-1 with
// M00 = s^2 + lam^2 c^2, M01 = -cs (lam^2 - 1), det M = lam^2.  The pool keeps ||A (t - r chi)|| <= r, t >= 0; its
// boundary is t(p) = r (chi - f(p)), p in [alpha, beta], f(p) = M (p, 1)' / h(p), h(p)^2 = (p, 1) M (p, 1)', and the
// marginal price at t(p) is p.  The pool's state is (r, p): the invariant and the price of its balances.
// Every flow is a difference t(q) - t(p) written as (p - q) times a positive quotient, never a difference of points:
//   f_x(p1) - f_x(p2) = (p1 - p2) B(p1, p2),  B = (Tx + D) / (h1 h2 (h1 + h2)),  D = lam^2,
//   f_y(p2) - f_y(p1) = (p1 - p2) C(p1, p2),  C = (Ty + D p1 p2) / (h1 h2 (h1 p2 + h2 p1)),
//   gx(p) = M00 p + M01 = lam^2 c (c p - s) + s (s p + c),  gy(p) = M01 p + M11 = c (s p + c) - lam^2 s (c p - s)
//   (c p - s by one fma: no lam^2 cancellation near the peg s / c),  h^2 = (gx^2 + D) / M00,
//   Tx = M00 h1 h2 - gx1 gx2 = D (gx1^2 + gx2^2 + D) / (M00 h1 h2 + gx1 gx2)  (the latter if gx1 gx2 > 0),
//   Ty = M11 h1 h2 - gy1 gy2 = D (gy1^2 p2^2 + gy2^2 p1^2 + D p1^2 p2^2) / (M11 h1 h2 + gy1 gy2)  (if gy1 gy2 > 0).
// C is B of the mirrored pool (tokens swapped, p -> 1/p, (c, s) -> (s, c)) at (1/p1, 1/p2), over p1 p2, written in p:
// rounding 1/p would cost up to p / |p - s/c| ulp of the flow near the peg when lam is large.
CFMM_HD inline double eclp_h(double c, double s, double D, double p) {
    const double g = D * c * fma(c, p, -s) + s * fma(s, p, c);
    return sqrt(fma(g, g, D) / fma(D * c, c, s * s));
}

CFMM_HD inline void eclp_BC(double c, double s, double D, double p1, double p2, double& B, double& C) {
    const double M00 = fma(D * c, c, s * s), M11 = fma(D * s, s, c * c);
    const double e1 = fma(c, p1, -s), e2 = fma(c, p2, -s), o1 = fma(s, p1, c), o2 = fma(s, p2, c);
    const double gx1 = D * c * e1 + s * o1, gx2 = D * c * e2 + s * o2;
    const double gy1 = c * o1 - D * s * e1, gy2 = c * o2 - D * s * e2;
    const double h1 = sqrt(fma(gx1, gx1, D) / M00), h2 = sqrt(fma(gx2, gx2, D) / M00);
    const double hh = h1 * h2;
    const double xx = gx1 * gx2, yy = gy1 * gy2, q12 = p1 * p2;
    const double Tx = xx > 0.0 ? D * (fma(gx1, gx1, fma(gx2, gx2, D)) / fma(M00, hh, xx)) : fma(M00, hh, -xx);
    const double Ty = yy > 0.0 ? D * (fma(gy1 * p2, gy1 * p2, fma(gy2 * p1, gy2 * p1, D * q12 * q12)) / fma(M11, hh, yy))
                               : fma(M11, hh, -yy);
    B = (Tx + D) / (hh * (h1 + h2));
    C = fma(D, q12, Ty) / (hh * fma(h1, p2, h2 * p1));
}

// The optimal trade at prices (n0, n1) of the pool (x, y) = the reserves at its state (r, p), fee gam.  Tender 0 iff
// p* = n0 / (gam n1) < p: the price falls to q = max(p*, alpha), D_0 = r (p - q) B(p, q) / gam, L_1 = r (p - q) C(p, q)
// (= y at q = alpha).  Tender 1 iff p* = gam n0 / n1 > p: the price rises to q = min(p*, beta), L_0 = r (q - p) B(p, q)
// (= x at q = beta), D_1 = r (q - p) C(p, q) / gam.  hc = r lam^2 n1 p*^2 / h(p*)^3, over gam when tendering 1, 0 at a
// cap or with no trade.
CFMM_HD inline void eclp_pair(double x, double y, double alpha, double beta, double c, double s, double lam, double r,
                              double p, double gam, double n0, double n1, double* Dl, double* Ll, double& hc) {
    Dl[0] = Dl[1] = Ll[0] = Ll[1] = 0.0;
    hc = 0.0;
    const double D = lam * lam;
    const double lo = n0 / (gam * n1), hi = gam * n0 / n1;
    const bool t0 = lo < p, t1 = hi > p;
    if (!t0 && !t1) return;
    const double ps = t0 ? lo : hi;
    const bool cap = t0 ? ps <= alpha : ps >= beta;
    const double q = cap ? (t0 ? alpha : beta) : ps;
    const double dq = t0 ? p - q : q - p;                                   // >= 0
    double B, C;
    eclp_BC(c, s, D, p, q, B, C);
    // token 0 and token 1 moved along the arc; at a cap the side paid out is the whole reserve, exactly
    const double fx = t1 && cap ? x : r * dq * B;
    const double fy = t0 && cap ? y : r * dq * C;
    if (t0) {
        Dl[0] = fx / gam;
        Ll[1] = fy;
    } else {
        Ll[0] = fx;
        Dl[1] = fy / gam;
    }
    if (!cap) {
        const double h = eclp_h(c, s, D, ps);
        hc = r * D * n1 * ps * ps / (h * h * h);
        if (t1) hc /= gam;
    }
}

// DODO proactive market maker (PMM; not a reference atom).  Guide price pi > 0 (token 1 per token 0), slippage factor
// 0 < k <= 1, targets (B0, Q0).  Two pieces meet at (B0, Q0) with slope -pi.  Base short (b <= B0): q - Q0 = pi d (1 +
// k d / b), d = B0 - b, marginal price pi (1 - k + k B0^2 / b^2) >= pi.  Quote short (q <= Q0): the mirror, b - B0 =
// (e / pi)(1 + k e / q), e = Q0 - q, price pi / (1 - k + k Q0^2 / q^2) <= pi.  The reserves (B, Q) lie on the curve
// through the adjusted-target rule (pools.pmm_targets): B < B0 (base short), Q < Q0 (quote short), or (B, Q) = (B0, Q0).
// The end point at price p* is closed form on its piece: w = sqrt(1 + z), b* = B0 / w with z = (p* - pi) / (k pi), or
// q* = Q0 / w with z = (pi - p*) / (k p*).  Along a piece the short token moves by |s2 - s1| and the other by the
// integral |s2 - s1| (1 - k + k T^2 / (s1 s2)), times pi (base piece) or over pi (quote piece), never a difference of
// two curve points; a leg from the target to s* moves T (1 - 1 / w) = T z / (w (w + 1)) (pmm_gap).
CFMM_HD inline double pmm_gap(double T, double z, double w) { return z < 3.0 ? T * (z / (w * (w + 1.0))) : T - T / w; }

// The optimal trade at prices (n0, n1) of the pool (B, Q), fee gam.  The pool's price P = pi (1 + k ((B0/B)^2 - 1))
// on the base piece, pi / (1 + k ((Q0/Q)^2 - 1)) on the quote piece, pi at equilibrium.  Tender 0 iff p* = n0 / (gam
// n1) < P: the price falls to p*.  Tender 1 iff p* = gam n0 / n1 > P: it rises to p*.  A trade that crosses pi runs
// in two legs that meet at (B0, Q0).  Never a cap: b*, q* > 0 at every finite price.  hc = n1 p*^2 b* / (2 (k pi + p* -
// pi)) for p* >= pi, n1 pi q* / (2 (k p* + pi - p*)) below, over gam when tendering 1, 0 with no trade.
CFMM_HD inline void pmm_pair(double B, double Q, double pi, double k, double B0, double Q0, double gam, double n0,
                             double n1, double* Dl, double* Ll, double& hc) {
    Dl[0] = Dl[1] = Ll[0] = Ll[1] = 0.0;
    hc = 0.0;
    const bool bs = B < B0, qs = !bs && Q < Q0;                             // base short | quote short | equilibrium
    const double rb = B0 / B, rq = Q0 / Q;
    const double P = bs ? pi * fma(k, fma(rb, rb, -1.0), 1.0) : qs ? pi / fma(k, fma(rq, rq, -1.0), 1.0) : pi;
    const double lo = n0 / (gam * n1), hi = gam * n0 / n1;
    const bool t0 = lo < P, t1 = hi > P;
    if (!t0 && !t1) return;
    const double ps = t0 ? lo : hi;
    const bool eb = ps >= pi;                                               // the trade ends on the base piece
    const double z = eb ? (ps - pi) / (k * pi) : (pi - ps) / (k * ps);
    const double w = sqrt(1.0 + z);
    const double T = eb ? B0 : Q0, se = T / w;                              // the end piece's target and end point
    double db = 0.0, dq = 0.0;                                              // token 0 and token 1 moved, >= 0
    double s = eb ? B : Q;                                                  // where the end piece's leg starts
    if (eb && qs) {                                                         // quote piece back to (B0, Q0) first
        dq = Q0 - Q;
        db = dq * fma(k, rq, 1.0 - k) / pi;
        s = B0;
    } else if (!eb && bs) {                                                 // base piece back to (B0, Q0) first
        db = B0 - B;
        dq = pi * (db * fma(k, rb, 1.0 - k));
        s = Q0;
    }
    const double d = s == T ? pmm_gap(T, z, w) : fmax(t0 == eb ? se - s : s - se, 0.0);
    const double o = d * fma(k, (T / s) * w, 1.0 - k);                      // T^2 / (s s*) = (T / s) w
    if (eb) { db += d; dq += pi * o; } else { dq += d; db += o / pi; }
    if (t0) {
        Dl[0] = db / gam;
        Ll[1] = dq;
    } else {
        Ll[0] = db;
        Dl[1] = dq / gam;
    }
    hc = eb ? n1 * ps * se * (ps / (2.0 * fma(k, pi, ps - pi))) : n1 * pi * se / (2.0 * fma(k, ps, pi - ps));
    if (t1) hc /= gam;
}

// Concentrated-liquidity pool (a whole Uniswap-v3 tick ladder): sqrt-price bounds b_0 < ... < b_T, liquidity L_k on
// [b_k, b_{k+1}), current sqrt price s in [b_0, b_T] inside interval c (b_c <= s, c <= T - 1).  One record per bound,
// rec[4k .. 4k+3] = {b_k, L_k, Y_k, X_k}: Y_k = sum_{j<k} L_j (b_{j+1} - b_j) (token 1 below b_k), X_k =
// sum_{j>=k} L_j (1/b_j - 1/b_{j+1}) (token 0 above b_k), L_T = 0.  The trading set is the Minkowski sum of the
// intervals' bounded-product sets, so at prices nu every interval moves to the same target sqrt price:
//   tender 0 (the price falls) iff s* = sqrt(nu0 / (gamma nu1)) < s: s_f = max(s*, b_0), L_1 = y - Y(s_f),
//     D_0 = (X(s_f) - x) / gamma;
//   tender 1 (the price rises) iff s* = sqrt(gamma nu0 / nu1) > s: s_f = min(s*, b_T), D_1 = (Y(s_f) - y) / gamma,
//     L_0 = x - X(s_f);
//   hc = L(s_f) sqrt(nu0 nu1 / gamma) / 2, L(s_f) = the liquidity of the interval j the trade ends in.  At an exact
//   bound s_f = b_j that is the interval above it, [b_j, b_{j+1}); past either end of the ladder (s* < b_0, s* >= b_T)
//   and in an empty interval it is 0.  At T = 1 this is bounded_pair.
// Precision: inside interval c the flows come from L_c and s - s_f (token 0: (s - s_f) / (s s_f), not a difference of
// reciprocals), never from table differences;
// across intervals they are the partial intervals at both ends plus the table difference over the whole intervals
// between them, so the absolute error stays a few ulp of the reserves.  j is found by searching outward from c: c
// first, then an exponential search toward s_f and a binary search, O(log |j - c|) record reads, fixed loop bounds.
// Shared by the per-thread solver and k_eval_ladder (cfmm_kernels.cu).
constexpr int64_t LADDER_T_MAX = int64_t(1) << 20;   // most intervals of one pool (pools.LADDER_T_MAX)
constexpr int LADDER_SEARCH = 22;                    // >= log2(LADDER_T_MAX) + 2: the search loops' fixed bound

// The largest j in [lo, hi) with b_j <= x, given b_lo <= x < b_hi (hi may be T + 1: b_{T+1} = +inf).
CFMM_HD inline int64_t ladder_bisect(const double* rec, int64_t lo, int64_t hi, double x) {
    for (int it = 0; it < LADDER_SEARCH; ++it) {
        if (hi - lo <= 1) break;
        const int64_t mid = lo + (hi - lo) / 2;
        if (rec[4 * mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

CFMM_HD inline void ladder_pair(const double* rec, int64_t T, int64_t c, double s, double gam, double n0, double n1,
                                double* D, double* L, double& hc) {
    D[0] = D[1] = L[0] = L[1] = 0.0;
    hc = 0.0;
    const double bc = rec[4 * c], Lc = rec[4 * c + 1], bc1 = rec[4 * (c + 1)];
    const double hs = 0.5 * sqrt(n0 * n1 / gam);
    const double sdn = sqrt(n0 / (gam * n1)), sup = sqrt(gam * n0 / n1);
    if (sdn < s) {                                                     // tender token 0: the price falls to s_f
        const double b0 = rec[0];
        const double sf = fmax(sdn, b0);
        int64_t j = c;
        if (sf < bc) {                                                 // below interval c: exponential, then binary search
            int64_t hi = c, lo = c;
            for (int it = 0, step = 1; it < LADDER_SEARCH; ++it, step *= 2) {
                lo = hi - step > 0 ? hi - step : 0;
                if (rec[4 * lo] <= sf) break;
                hi = lo;
            }
            j = ladder_bisect(rec, lo, hi, sf);
        }
        const double Lj = rec[4 * j + 1];
        if (j == c) {
            L[1] = Lc * (s - sf);
            D[0] = Lc * ((s - sf) / (s * sf)) / gam;
        } else {                                                       // partial c, whole intervals j+1 .. c-1, partial j
            const double bj1 = rec[4 * (j + 1)];
            L[1] = Lc * (s - bc) + (rec[4 * c + 2] - rec[4 * (j + 1) + 2]) + Lj * (bj1 - sf);
            D[0] = (Lc * ((s - bc) / (s * bc)) + (rec[4 * (j + 1) + 3] - rec[4 * c + 3]) + Lj * ((bj1 - sf) / (sf * bj1))) / gam;
        }
        if (sdn >= b0) hc = Lj * hs;
    } else if (sup > s) {                                              // tender token 1: the price rises to s_f
        const double bT = rec[4 * T];
        const double sf = fmin(sup, bT);
        int64_t j = c;
        if (sf >= bc1) {                                               // above interval c (j = T: past the top)
            int64_t lo = c + 1, hi = c + 1;
            for (int it = 0, step = 1; it < LADDER_SEARCH; ++it, step *= 2) {
                hi = lo + step < T + 1 ? lo + step : T + 1;
                if (hi > T || rec[4 * hi] > sf) break;
                lo = hi;
            }
            j = ladder_bisect(rec, lo, hi, sf);
        }
        const double Lj = rec[4 * j + 1];                              // L_T = 0
        if (j == c) {
            D[1] = Lc * (sf - s) / gam;
            L[0] = Lc * ((sf - s) / (s * sf));
        } else {                                                       // partial c, whole intervals c+1 .. j-1, partial j
            const double bj = rec[4 * j];
            D[1] = (Lc * (bc1 - s) + (rec[4 * j + 2] - rec[4 * (c + 1) + 2]) + Lj * (sf - bj)) / gam;
            L[0] = Lc * ((bc1 - s) / (s * bc1)) + (rec[4 * (c + 1) + 3] - rec[4 * j + 3]) + Lj * ((sf - bj) / (bj * sf));
        }
        hc = Lj * hs;
    }
}

// Price-bin pool (Liquidity Book bins, an order book, limit orders): bins k at prices p_k (token 1 per token 0) holding
// x_k of token 0 and y_k of token 1, uncrossed (every bin with y > 0 prices at or below every bin with x > 0); its
// trading set is the Minkowski sum of the bins' constant-sum sets.  In net-flow form the pool pays out t of token 0 for
// the least C(t) of token 1, C convex piecewise linear: slope p_k / gamma over x_k for t > 0 (asks, ascending), slope
// gamma p_k over y_k / (gamma p_k) for t < 0 (bids, descending).  One fee-free record per breakpoint j = 0 .. nb - 1,
// ascending in t, rec[4j .. 4j+3] = {T_j, C_j, q_j, bin}: record z is (0, 0); above it T is the cumulative x and C the
// cumulative p x of the asks, below it T is minus the cumulative y / p and C minus the cumulative y of the bids, both
// accumulated outward from t = 0; q_j = the price of the segment (j, j+1) and bin its bin (0 and -1 on the last record).
// The fee is applied here: breakpoint j is at (T_j / gamma, C_j) below z and (T_j, C_j / gamma) above it.
// Exact (eps <= 0): t* maximises r t - C(t), r = nu0 / nu1, a breakpoint; a segment fills only when strictly profitable
// (sum_order's rule).  Smoothed (eps > 0): t maximises r t - C(t) - (t - tbar)^2 / (2 a), a = sigma / p_ref, sigma =
// S / eps, S = the width of C's domain; the trader pays the smoothing term, so the trade stays pool-feasible.
// Flows (+t, -(C(t) + smoothing)); hc = a r nu0 inside a segment, 0 at a breakpoint or an end.  The end breakpoint is
// the largest j whose left end of the subgradient of t + a C'(t) is <= tbar + a r (exact: whose left segment fills),
// found by an exponential search outward from z and a bisection, O(log |j - z|) record reads, fixed loop bounds.
// Returns t.  Shared by the per-thread solver and k_eval_bins (cfmm_kernels.cu).
constexpr int64_t BINS_K_MAX = int64_t(1) << 20;     // most bins of one pool (pools.BINS_K_MAX): nb <= K + 2

CFMM_HD inline double bins_slope(const double* rec, int64_t j, int64_t z, double gam) {   // segment (j, j+1)
    return j < z ? gam * rec[4 * j + 2] : rec[4 * j + 2] / gam;
}

CFMM_HD inline double bins_pair(const double* rec, int64_t nb, int64_t z, double pref, double tbar, double gam,
                                double n0, double n1, double eps, double* D, double* L, double& hc) {
    D[0] = D[1] = L[0] = L[1] = 0.0;
    hc = 0.0;
    const double r = n0 / n1;
    const double tlo = rec[0] / gam, thi = rec[4 * (nb - 1)];
    const double a = eps > 0.0 ? (thi - tlo) / (eps * pref) : 0.0;
    auto tat = [&](int64_t j) { return j < z ? rec[4 * j] / gam : rec[4 * j]; };
    auto cat = [&](int64_t j) { return j > z ? rec[4 * j + 1] / gam : rec[4 * j + 1]; };
    // pred(j): breakpoint j is at or below the solution; true at j = 0, monotone (true ... false)
    auto pred = [&](int64_t j) {
        if (j <= 0) return true;
        if (eps > 0.0) return tat(j) - tbar <= a * (r - bins_slope(rec, j - 1, z, gam));
        return j <= z ? !(r < gam * rec[4 * (j - 1) + 2]) : gam * r > rec[4 * (j - 1) + 2];
    };
    int64_t lo, hi;                                                    // pred(lo), !pred(hi) (hi = nb: past the top)
    if (pred(z)) {
        lo = z; hi = nb;
        for (int it = 0, step = 1; it < LADDER_SEARCH; ++it, step *= 2) {
            const int64_t c = lo + step < nb ? lo + step : nb;
            if (c >= nb || !pred(c)) { hi = c; break; }
            lo = c;
        }
    } else {
        hi = z; lo = 0;
        for (int it = 0, step = 1; it < LADDER_SEARCH; ++it, step *= 2) {
            const int64_t c = hi - step > 0 ? hi - step : 0;
            if (pred(c)) { lo = c; break; }
            hi = c;
        }
    }
    for (int it = 0; it < LADDER_SEARCH; ++it) {
        if (hi - lo <= 1) break;
        const int64_t mid = lo + (hi - lo) / 2;
        if (pred(mid)) lo = mid; else hi = mid;
    }
    const int64_t j = lo;
    double t = tat(j), C = cat(j);
    if (eps > 0.0 && j < nb - 1) {
        const double s = bins_slope(rec, j, z, gam);
        const double w = tbar + a * (r - s);
        if (w > t) {                                                   // inside segment (j, j+1)
            t = fmin(w, tat(j + 1));
            C = j < z ? cat(j + 1) + s * (t - tat(j + 1)) : C + s * (t - tat(j));
            if (t < tat(j + 1)) hc = a * r * n0;
        }
    }
    const double sm = eps > 0.0 ? (t - tbar) * (t - tbar) / (2.0 * a) : 0.0;
    const double y1 = -(C + sm);
    L[0] = fmax(t, 0.0); D[0] = fmax(-t, 0.0);
    L[1] = fmax(y1, 0.0); D[1] = fmax(-y1, 0.0);
    return t;
}

// Two-coin StableSwap (Curve) pool: scaled balances y_j = r_j x_j on the invariant
//     4A (y0 + y1) + D = 4A D + D^3 / (4 y0 y1),        D = the invariant of the current reserves (precomputed),
// worked in units of D (u_j = y_j / D, so 4A (u0 + u1) + 1 = 4A + 1 / (4 u0 u1)) so nothing overflows.  Along the curve
// the marginal rate -du_b/du_a is s = F_a / F_b, F_a = 4A + G / u_a, F_b = 4A + G / u_b, G = 1 / (4 u_a u_b); in token
// units p = (r_a / r_b) s.  Tendering a pays iff gamma nu_b p(R) > nu_a; the optimal post-trade balance solves
// s(u_a) = q* = mu_a / (gamma mu_b) with the scaled prices mu_j = nu_j / r_j, found by a safeguarded Newton iteration on
// t = log u_a (s falls from +inf to 0 along the curve, so an upper bracket always exists).  u_b(u_a) is Curve's get_y:
// the positive root of u^2 + b u - c with b = u_a + 1/(4A) - 1, c = 1 / (16 A u_a), in the cancellation-free form.
// hc = nu_0 dy_0/dlog nu_0 = -nu_a X_a / (gamma dlog s/dt) at the solution (0 without a trade).
// Fixed iteration caps and a deterministic exit; shared by the per-thread solver and k_eval_stable (cfmm_kernels.cu).
CFMM_HD inline double stableswap_get_y(double ua, double A) {
    const double b = (ua - 1.0) + 0.25 / A, c = 0.0625 / (A * ua);
    const double sq = sqrt(b * b + 4.0 * c);
    return b > 0.0 ? 2.0 * c / (b + sq) : 0.5 * (sq - b);
}

// log s - logq at u_a = exp(t) on the curve, and its derivative in t
CFMM_HD inline double stableswap_phi(double t, double A, double logq, double* dphi) {
    const double ua = exp(t), ub = stableswap_get_y(ua, A);
    const double G = 0.25 / (ua * ub);
    const double Fa = 4.0 * A + G / ua, Fb = 4.0 * A + G / ub;
    const double kap = -(Fa / Fb) * (ua / ub);                          // dlog u_b / dlog u_a along the curve
    *dphi = (G / ua) * (-2.0 - kap) / Fa - (G / ub) * (-1.0 - 2.0 * kap) / Fb;
    // s = 1 + del, del = (F_a - F_b) / F_b without cancellation: log1p near s = 1, the plain ratio far from it
    const double del = G * (ub - ua) / (ua * ub * Fb);
    return (fabs(del) < 0.5 ? log1p(del) : log(Fa / Fb)) - logq;
}

// One direction of stableswap_pair: tender a, receive b.  Balances in units of D (ua, ub), scaled prices mu = nu / r.
// Writes the tender Delta_a and the payout Lambda_b and returns hc (all 0 without a trade).  Scalar arguments only: the
// two calls below take the directions with constant operands, so nothing is indexed by a loop variable (no stack).
CFMM_HD inline double stableswap_dir(double Ra, double Rb, double ra, double rb, double ua0, double ub0, double mua,
                                     double mub, double nua, double A, double Dinv, double gam, double& Da, double& Lb) {
    Da = Lb = 0.0;
    const double G0 = 0.25 / (ua0 * ub0);
    const double Fa = 4.0 * A + G0 / ua0, Fb = 4.0 * A + G0 / ub0;
    const double del = G0 * (ub0 - ua0) / (ua0 * ub0 * Fb);
    const double s0 = fabs(del) < 0.5 ? 1.0 + del : Fa / Fb;            // the marginal rate at R, as in stableswap_phi
    if (!(gam * mub * s0 > mua)) return 0.0;                            // no trade in this direction
    const double logq = log(mua / (gam * mub));
    double lo = log(ua0), hi = lo, dphi = 0.0;
    for (double step = 1.0; step <= 512.0; step *= 2.0) {               // upper bracket phi(hi) <= 0 (|t| < 700: exp finite)
        hi = lo + step;
        if (!(stableswap_phi(hi, A, logq, &dphi) > 0.0)) break;
        lo = hi;
    }
    // safeguarded Newton inside [lo, hi]: a bisection step whenever the Newton step would leave the bracket or would
    // not at least halve the step before last (a crawl where phi bends), so the bracket keeps shrinking
    double t = lo, dx_old = hi - lo, dx = dx_old;
    for (int it = 0; it < 100; ++it) {
        const double f = stableswap_phi(t, A, logq, &dphi);
        if (f > 0.0) lo = t; else hi = t;
        if (f == 0.0 || !(hi - lo > 4e-16 * (1.0 + fabs(t)))) break;
        const double tn = t - f / dphi;
        // phi is at the level of its own rounding (a few u of log s, u |log q*|): further steps would only chase that
        // noise (a flat curve, large A, |phi'| small); the last Newton step, inside the bracket, is as good as any
        if (fabs(f) <= 8e-16 * (1.0 + fabs(logq))) {
            if (tn > lo && tn < hi) t = tn;
            break;
        }
        if (!(tn > lo && tn < hi) || fabs(2.0 * f) > fabs(dx_old * dphi)) {
            dx_old = dx; dx = 0.5 * (hi - lo); t = lo + dx;
        } else {
            dx_old = dx; dx = tn - t; t = tn;
        }
        if (fabs(dx) <= 1e-15 * (1.0 + fabs(t))) break;
    }
    const double ua = exp(t), ub = stableswap_get_y(ua, A);
    const double Xa = fmax(ua * Dinv / ra, Ra), Xb = ub * Dinv / rb;
    Da = (Xa - Ra) / gam;
    Lb = fmax(Rb - Xb, 0.0);
    stableswap_phi(t, A, logq, &dphi);
    return dphi < 0.0 ? -nua * Xa / (gam * dphi) : 0.0;
}

CFMM_HD inline void stableswap_pair(double R0, double R1, double r0, double r1, double A, double Dinv, double gam,
                                    double n0, double n1, double* D, double* L, double& hc) {
    const double u0 = r0 * R0 / Dinv, u1 = r1 * R1 / Dinv, mu0 = n0 / r0, mu1 = n1 / r1;
    double d0, l1, d1, l0;
    hc = stableswap_dir(R0, R1, r0, r1, u0, u1, mu0, mu1, n0, A, Dinv, gam, d0, l1)
       + stableswap_dir(R1, R0, r1, r0, u1, u0, mu1, mu0, n1, A, Dinv, gam, d1, l0);
    D[0] = d0; D[1] = d1; L[0] = l0; L[1] = l1;
}

// Two-coin Curve cryptoswap (v2, twocrypto-ng) pool: scaled balances y_j = p_j x_j (p = price scale times precision),
// whitepaper amplification A and curve gamma G (not the fee gamma), the invariant of the current reserves D:
//     K0 = 4 y0 y1 / D^2,   K = A K0 G^2 / (G + 1 - K0)^2,   K D (y0 + y1) + y0 y1 = K D^2 + (D/2)^2.
// Worked in units of D (u = y / D, the caller passes c_j = p_j / D so u = c x): Phi(u) = K (u0 + u1 - 1) + u0 u1 - 1/4 = 0.
// Along the curve, with e = 2 u_a - 1, m = 1 - K0 and dl = u_a + u_b - 1 (dl >= 0), the invariant reads K dl = m / 4 and
// m = e^2 - 4 u_a dl, so m is the root in [0, min(e^2, 1)] of
//     h(m) = A G^2 (1 - m)(e^2 - m) - u_a m (G + m)^2,       strictly decreasing there (get_y: no closed form),
// bracketed by [e^2 K(hi) / (K(hi) + u_a), hi], hi = e^2 A / (A + u_a) (m = e^2 K / (K + u_a) with K falling in m).
// m, dl and u_b - u_a = dl - e are formed from e (exact: 2 u_a - 1 has no rounding where it is small), never as 1 - 4 u0 u1
// or u0 + u1 - 1, so near the peg they keep their digits against G (1e-5 .. 1e-4 in deployed pools).
// With K' = dK/dK0 = A G^2 (G + 2 - m) / (G + m)^3 and cc = 1 + 4 dl K', F_a = K + u_b cc, F_b = K + u_a cc, the marginal
// rate is s = F_a / F_b, s - 1 = cc (u_b - u_a) / F_b.  Tendering a pays iff gamma mu_b s(R) > mu_a with mu = nu / c; the
// optimal post-trade balance solves log s(u_a) = log(mu_a / (gamma mu_b)) by the stableswap_dir scheme in t = log u_a,
// with dlog s/dt = u_a (Phi_aa - 2 s Phi_ab + s^2 Phi_bb) / F_a, the curvature grouped so the large K' terms cancel
// analytically: 8 K' (-(s - 1)(d - (s - 1) u_a) - s dl) + 16 K'' dl (d - (s - 1) u_a)^2 - 2 s, d = u_b - u_a.
// hc = -nu_a X_a / (gamma dlog s/dt), as for StableSwap.  Fixed iteration caps, scalar arguments only (no stack);
// shared by the per-thread solver and k_eval_crypto (cfmm_kernels.cu).

// The curve point at u_a: u_b, dl, m and K, K', K''.  ag2 = A G^2.
CFMM_HD inline void crypto_point(double ua, double A, double G, double ag2, double& ub, double& dl, double& m, double& K,
                                 double& K1, double& K2) {
    const double e = 2.0 * ua - 1.0, e2 = e * e;
    const double mtop = fmin(e2, 1.0);
    double hi = fmin(e2 * A / (A + ua), mtop);
    const double gh = G + hi, Kh = ag2 * (1.0 - hi) / (gh * gh);
    double lo = fmin(e2 * Kh / (Kh + ua), hi);
    m = hi;
    if (hi > 0.0) {
        // safeguarded Newton on h inside [lo, hi] (h falls: h(lo) >= 0 >= h(hi)), from the upper end
        m = 0.5 * (lo + hi);
        for (int it = 0; it < 60; ++it) {
            const double g = G + m;
            const double f = ag2 * (1.0 - m) * (e2 - m) - ua * m * g * g;
            if (f > 0.0) lo = m; else hi = m;
            if (f == 0.0 || !(hi - lo > 2e-16 * m)) break;
            const double df = -ag2 * ((1.0 - m) + (e2 - m)) - ua * g * (G + 3.0 * m);
            double mn = m - f / df;
            if (!(mn > lo && mn < hi)) mn = 0.5 * (lo + hi);
            if (fabs(mn - m) <= 1e-16 * m) { m = mn; break; }
            m = mn;
        }
    }
    const double g = G + m, g2 = g * g;
    K = ag2 * (1.0 - m) / g2;
    K1 = ag2 * (G + 2.0 - m) / (g2 * g);
    K2 = ag2 * (4.0 * G + 6.0 - 2.0 * m) / (g2 * g2);
    // dl = m / (4K) where m is close to e^2 (e^2 - m cancels there), else (e^2 - m) / (4 u_a)
    dl = (m > 0.5 * e2) ? m / (4.0 * K) : (e2 - m) / (4.0 * ua);
    ub = ua <= 1.0 ? (1.0 - ua) + dl : (1.0 - m) / (4.0 * ua);
}

// log s - logq at u_a = exp(t) on the curve, and its derivative in t; ub out
CFMM_HD inline double crypto_phi(double t, double A, double G, double ag2, double logq, double* dphi, double& ub) {
    const double ua = exp(t);
    double dl, m, K, K1, K2;
    crypto_point(ua, A, G, ag2, ub, dl, m, K, K1, K2);
    const double d = dl - (2.0 * ua - 1.0);                             // u_b - u_a
    const double cc = 1.0 + 4.0 * dl * K1;
    const double Fa = K + ub * cc, Fb = K + ua * cc;
    const double sm1 = cc * d / Fb;                                      // s - 1
    const double s = 1.0 + sm1;
    const double w = d - sm1 * ua;                                       // u_b - s u_a
    const double Q = 8.0 * K1 * (-sm1 * w - s * dl) + 16.0 * K2 * dl * w * w - 2.0 * s;
    *dphi = ua * Q / Fa;
    return (fabs(sm1) < 0.5 ? log1p(sm1) : log(Fa / Fb)) - logq;
}

// One direction of cryptoswap_pair: tender a, receive b.  Balances in units of D (ua0 = ca Ra), scaled prices mu = nu / c.
// Writes the tender Delta_a and the payout Lambda_b and returns hc (all 0 without a trade).
CFMM_HD inline double crypto_dir(double Ra, double Rb, double ca, double cb, double mua, double mub, double nua, double A,
                                 double G, double gam, double& Da, double& Lb) {
    Da = Lb = 0.0;
    const double ag2 = A * G * G;
    const double logq = log(mua / (gam * mub));
    double dphi = 0.0, ub = 0.0;
    double lo = log(ca * Ra), hi = lo;
    if (!(crypto_phi(lo, A, G, ag2, logq, &dphi, ub) > 0.0)) return 0.0;   // no trade in this direction
    for (double step = 1.0; step <= 512.0; step *= 2.0) {               // upper bracket phi(hi) <= 0 (|t| < 700: exp finite)
        hi = lo + step;
        if (!(crypto_phi(hi, A, G, ag2, logq, &dphi, ub) > 0.0)) break;
        lo = hi;
    }
    // safeguarded Newton inside [lo, hi], as stableswap_dir
    double t = lo, dx_old = hi - lo, dx = dx_old;
    for (int it = 0; it < 100; ++it) {
        const double f = crypto_phi(t, A, G, ag2, logq, &dphi, ub);
        if (f > 0.0) lo = t; else hi = t;
        if (f == 0.0 || !(hi - lo > 4e-16 * (1.0 + fabs(t)))) break;
        const double tn = t - f / dphi;
        if (fabs(f) <= 8e-16 * (1.0 + fabs(logq))) {                   // phi at the level of its own rounding
            if (tn > lo && tn < hi) t = tn;
            break;
        }
        if (!(tn > lo && tn < hi) || fabs(2.0 * f) > fabs(dx_old * dphi)) {
            dx_old = dx; dx = 0.5 * (hi - lo); t = lo + dx;
        } else {
            dx_old = dx; dx = tn - t; t = tn;
        }
        if (fabs(dx) <= 1e-15 * (1.0 + fabs(t))) break;
    }
    crypto_phi(t, A, G, ag2, logq, &dphi, ub);
    const double Xa = fmax(exp(t) / ca, Ra), Xb = ub / cb;
    Da = (Xa - Ra) / gam;
    Lb = fmax(Rb - Xb, 0.0);
    return dphi < 0.0 ? -nua * Xa / (gam * dphi) : 0.0;
}

// c_j = p_j / D: the price scales over the invariant of the current reserves; A, G: the whitepaper amplification and gamma
CFMM_HD inline void cryptoswap_pair(double R0, double R1, double c0, double c1, double A, double G, double gam, double n0,
                                    double n1, double* D, double* L, double& hc) {
    const double mu0 = n0 / c0, mu1 = n1 / c1;
    double d0, l1, d1, l0;
    hc = crypto_dir(R0, R1, c0, c1, mu0, mu1, n0, A, G, gam, d0, l1)
       + crypto_dir(R1, R0, c1, c0, mu1, mu0, n1, A, G, gam, d1, l0);
    D[0] = d0; D[1] = d1; L[0] = l0; L[1] = l1;
}

// Three-coin Curve cryptoswap (tricrypto-ng) pool: y_j = p_j x_j, A, G as for two coins, the invariant D of the current
// reserves.  In units of D (u = y / D, the caller passes c_j = p_j / D): S = sum u, P = prod u, K0 = 27 P,
// K = A K0 G^2 / (G + 1 - K0)^2, and the pool keeps Phi(u) = K (S - 1) + P - 1/27 >= 0, with dPhi/du_j = K + Q / u_j,
// Q = P (1 + 27 (S - 1) K'), K' = dK/dK0.  That is the form a + Q / u_j of stableswap_n, so with pi_j = nu_j / c_j the
// stationary point at the multiplier mu is u_j = clamp(u0_j, Q / (pi_j / (gamma mu) - K), Q / (pi_j / mu - K)) and the
// pool is idle iff gamma max rho <= min rho, rho_j = pi_j / dPhi/du_j(u0) (flows and edge weights then exactly 0).
// K and Q are not constants: with m = 1 - K0 the curve gives P = (1 - m) / 27 and S - 1 = m / (27 K), so
//     K = A G^2 (1 - m) / (G + m)^2,   Q = (G + 3m - 2m^2) / (27 (G + m)),   l = log(Q / K),
// all functions of m.  At fixed m, with tau = log(pi_min / (gamma K mu)) and dB_j = log(pi_j / pi_min) as in
// stableswap_n, log u_j = log u0_j + z_j, z_j = max(l - bA_j, 0) + min(l - bB_j, 0), bA_j = log(u0_j expm1(dB_j + tau)),
// bB_j = log(u0_j expm1(dB_j + log gamma + tau)) (-inf if that expm1 <= 0): the denominators without cancellation.
// Two conditions close the system:
//   E1(tau; m) = sum_j z_j - log1p(-m) + sum_j log1p(e0_j) = 0   (P = (1 - m) / 27; e0_j = 3 u0_j - 1),
//        strictly falling in tau: one safeguarded Newton in log tau per m (crypto3_tau);
//   r(m) = sum_j e_j - m / (9 K) = 0   (S - 1 = m / (27 K); e_j = 3 u_j - 1 = e0_j + 3 u0_j expm1(z_j)),
//        r(0) >= 0 (AM-GM at P = 1/27) and r -> -inf as m -> 1; a root is a KKT point, so it is unique.  A safeguarded
//        Newton in x = log(m / (1 - m)) finds it, with m and 1 - m both formed from x (no 1 - m cancellation at
//        either end), dr/dm by the implicit derivative of E1: dtau/dm = (n_T l' + 1 / (1 - m)) / sum_T kap_j,
//        dz_j/dm = l' - kap_j dtau/dm, kap_j = 1 + 1 / expm1(.)_j.
// So 1 - K0 = m, S - 1 = sum e / 3 and the price-ratio denominators are never formed as differences near the peg.
// Hessian.  On the traded set T, p_T = mu g(u), g = dPhi/du, and Phi(u) = 0: with Z a basis of g-perp on T,
// du/dp = Z (Z'HZ)^-1 Z' / mu, H = d2Phi/du2 = a(w1' + 1w') + b ww' - Q diag(w^2), w = 1/u, a = 27 P K',
// b = Q + 729 P^2 (S - 1) K''; since Z'w = -(K/Q) Z'1, Z'HZ = c (Z'1)(Z'1)' - Q Z'diag(w^2)Z with
// c = (K/Q)(K - 2a + 729 P^2 (S - 1) K'' K / Q), and Z'1 = g_b - g_a = Q (u_a - u_b) / (u_a u_b) from e_a - e_b.
// The scaled block Hs_ij = -p_i p_j (du/dp)_ij is PSD with Hs 1 = 0 (Z'p = 0), so it is the three edge weights
// w_ij = -Hs_ij, (w01, w02, w12), 0 on an edge with an untraded end.  Writes D, L (flows) and w, returns the traded slots.
// Fixed iteration caps, 3-element register arrays under full unrolling; shared by the per-thread solver and
// k_eval_crypto3 (cfmm_kernels.cu).

// E1 at s = log tau and dE1/ds; z and kap (0 off the traded set) out
CFMM_HD inline double crypto3_e1(double s, const double* dB, double lg, const double* lu0, double l, double tgt,
                                 double* z, double* kap, double& de, double& sc) {
    const double tau = exp(s);
    double f = -tgt, sk = 0.0;
    sc = 1.0 + fabs(l) + fabs(tgt);
CFMM_UNROLL
    for (int j = 0; j < 3; ++j) {
        const double eA = expm1(dB[j] + tau), eB = expm1(dB[j] + lg + tau);
        const double bA = lu0[j] + log(eA);
        const double zA = l - bA;
        const double zB = eB > 0.0 ? l - (lu0[j] + log(eB)) : INFINITY;
        z[j] = fmax(zA, 0.0) + fmin(zB, 0.0);
        kap[j] = z[j] > 0.0 ? 1.0 + 1.0 / eA : (z[j] < 0.0 ? 1.0 + 1.0 / eB : 0.0);
        f += z[j];
        sk += kap[j];
        sc += fabs(bA) + fabs(z[j]);
    }
    de = -tau * sk;
    return f;
}

// the root of E1 in s = log tau, from s0 (bracketing, then a safeguarded Newton as stableswap_dir); z, kap out
CFMM_HD inline double crypto3_tau(double s0, const double* dB, double lg, const double* lu0, double l, double tgt,
                                  double* z, double* kap) {
    constexpr double SMIN = -700.0, SMAX = 6.39;                        // tau in (1e-304, 600): exp, expm1 finite
    double de = 0.0, sc = 0.0;
    double s = fmin(fmax(s0, SMIN), SMAX), lo = s, hi = s;
    if (crypto3_e1(s, dB, lg, lu0, l, tgt, z, kap, de, sc) > 0.0) {    // E1 falls in s
        for (double step = 0.5; step <= 1024.0 && lo < SMAX; step *= 2.0) {
            hi = fmin(lo + step, SMAX);
            if (!(crypto3_e1(hi, dB, lg, lu0, l, tgt, z, kap, de, sc) > 0.0)) break;
            lo = hi;
        }
    } else {
        for (double step = 0.5; step <= 1024.0 && hi > SMIN; step *= 2.0) {
            lo = fmax(hi - step, SMIN);
            if (crypto3_e1(lo, dB, lg, lu0, l, tgt, z, kap, de, sc) > 0.0) break;
            hi = lo;
        }
    }
    double t = 0.5 * (lo + hi), dx_old = hi - lo, dx = dx_old;
    for (int it = 0; it < 100; ++it) {
        const double f = crypto3_e1(t, dB, lg, lu0, l, tgt, z, kap, de, sc);
        if (f > 0.0) lo = t; else hi = t;
        if (f == 0.0 || !(hi - lo > 4e-16 * (1.0 + fabs(t)))) break;
        const double tn = t - f / de;
        if (fabs(f) <= 4.5e-16 * sc) {                                  // E1 at the level of its own rounding
            if (tn > lo && tn < hi) t = tn;
            break;
        }
        if (!(tn > lo && tn < hi) || fabs(2.0 * f) > fabs(dx_old * de)) {
            dx_old = dx; dx = 0.5 * (hi - lo); t = lo + dx;
        } else {
            dx_old = dx; dx = tn - t; t = tn;
        }
        if (fabs(dx) <= 1e-15 * (1.0 + fabs(t))) break;
    }
    crypto3_e1(t, dB, lg, lu0, l, tgt, z, kap, de, sc);
    return t;
}

// r at x = log(m / (1 - m)) and dr/dx; the inner root s (warm start in, root out), z, kap, m, 1 - m, K, Q out
CFMM_HD inline double crypto3_r(double x, double G, double ag2, const double* dB, double lg, const double* u0,
                                const double* lu0, const double* e0, double sl0, double& s, double* z, double* kap,
                                double& m, double& om, double& K, double& Q, double& dr, double& sc) {
    m = 1.0 / (1.0 + exp(-x));
    om = 1.0 / (1.0 + exp(x));
    const double g = G + m;
    K = ag2 * om / (g * g);
    const double K1 = ag2 * (G + 1.0 + om) / (g * g * g);               // dK/dK0 = -dK/dm
    const double qn = G + 3.0 * m - 2.0 * m * m;
    Q = qn / (27.0 * g);
    const double l = log(qn * g / (27.0 * ag2 * om));                   // log(Q / K)
    const double tgt = log1p(-m) - sl0;
    s = crypto3_tau(s, dB, lg, lu0, l, tgt, z, kap);
    // dl/dm = Q'/Q + K'/K, Q' = 2 (G - 2 G m - m^2) / (27 (G + m)^2)
    const double dl = 2.0 * (G - 2.0 * G * m - m * m) / (qn * g) + K1 / K;
    int nt = 0;
    double sk = 0.0;
CFMM_UNROLL
    for (int j = 0; j < 3; ++j) { nt += kap[j] != 0.0; sk += kap[j]; }
    const double dtau = nt ? (nt * dl + 1.0 / om) / sk : 0.0;
    double r = 0.0, d = 0.0;
    sc = 1.0;
CFMM_UNROLL
    for (int j = 0; j < 3; ++j) {
        const double ex = expm1(z[j]);
        const double e = e0[j] + 3.0 * u0[j] * ex;
        r += e;
        sc += fabs(e0[j]) + fabs(3.0 * u0[j] * ex);
        if (kap[j] != 0.0) d += 3.0 * u0[j] * (1.0 + ex) * (dl - kap[j] * dtau);
    }
    const double f = m * g * g / om;                                    // m / K = ag2 f
    r -= f / (9.0 * ag2);
    sc += f / (9.0 * ag2);
    d -= (g * (G + 3.0 * m) / om + f / om) / (9.0 * ag2);
    dr = d * m * om;
    return r;
}

// The 2 x 2 (or 1 x 1) block -Hs on the traded set from the answer; see the header comment.  ia, ib, ic: the traded
// slots (ic < 0: two traded).  Returns the edge weights in w[3] = (w01, w02, w12).
CFMM_HD inline void crypto3_edges(int ia, int ib, int ic, const double* u, const double* e, const double* p, double mu,
                                  double m, double om, double K, double Q, double K1, double K2, double* w) {
    w[0] = w[1] = w[2] = 0.0;
    const double Sm1 = m / (27.0 * K);
    const double a = om * K1;
    const double c = (K / Q) * (K - 2.0 * a + om * om * Sm1 * K2 * K / Q);
    if (ic < 0) {                                                       // Z = (g_b, -g_a): 1 x 1
        const double ga = K + Q / u[ia], gb = K + Q / u[ib];
        const double wa = 1.0 / u[ia], wb = 1.0 / u[ib];
        const double eta = Q * (e[ia] - e[ib]) / (3.0 * u[ia] * u[ib]);   // g_b - g_a
        const double B = c * eta * eta - Q * (gb * gb * wa * wa + ga * ga * wb * wb);
        if (B < 0.0) w[ia + ib - 1] = -p[ia] * p[ib] * ga * gb / (mu * B);   // edge (0,1) 0, (0,2) 1, (1,2) 2
        return;
    }
    // three traded: Z = [(g1, -g0, 0), (g2, 0, -g0)] in slot order
    const double g0 = K + Q / u[0], g1 = K + Q / u[1], g2 = K + Q / u[2];
    const double w0 = 1.0 / u[0], w1 = 1.0 / u[1], w2 = 1.0 / u[2];
    const double h1 = Q * (e[0] - e[1]) / (3.0 * u[0] * u[1]), h2 = Q * (e[0] - e[2]) / (3.0 * u[0] * u[2]);
    const double b11 = c * h1 * h1 - Q * (g1 * g1 * w0 * w0 + g0 * g0 * w1 * w1);
    const double b12 = c * h1 * h2 - Q * (g1 * g2 * w0 * w0);
    const double b22 = c * h2 * h2 - Q * (g2 * g2 * w0 * w0 + g0 * g0 * w2 * w2);
    const double det = b11 * b22 - b12 * b12;
    if (!(det > 0.0) || !(b11 < 0.0)) return;
    const double i11 = b22 / det, i12 = -b12 / det, i22 = b11 / det;
    const double N01 = -g0 * (g1 * i11 + g2 * i12), N02 = -g0 * (g1 * i12 + g2 * i22), N12 = g0 * g0 * i12;
    w[0] = p[0] * p[1] * N01 / mu;
    w[1] = p[0] * p[2] * N02 / mu;
    w[2] = p[1] * p[2] * N12 / mu;
}

// c_j = p_j / D; A, G: the whitepaper amplification and curve gamma.  Flows into D[3], L[3], edge weights into w[3];
// returns the traded slots as a bit mask.
CFMM_HD inline uint32_t cryptoswap3(double R0, double R1, double R2, double c0, double c1, double c2, double A,
                                    double G, double gam, double n0, double n1, double n2, double* D, double* L,
                                    double* w) {
    const double R[3] = {R0, R1, R2}, cc[3] = {c0, c1, c2}, nu[3] = {n0, n1, n2};
    double u0[3], lu0[3], e0[3], pi[3], dB[3], z[3], kap[3];
    double pmin = INFINITY, sl0 = 0.0;
CFMM_UNROLL
    for (int j = 0; j < 3; ++j) {
        D[j] = L[j] = w[j] = 0.0;
        u0[j] = cc[j] * R[j];
        lu0[j] = log(u0[j]);
        e0[j] = fma(3.0, u0[j], -1.0);
        sl0 += log1p(e0[j]);
        pi[j] = nu[j] / cc[j];
        pmin = fmin(pmin, pi[j]);
    }
    const double ag2 = A * G * G, lg = log(gam);
    // the current point: m0 = 1 - 27 P0, K0 and Q0 on the curve, then the band
    const double m0 = fmax(-expm1(sl0), 0.0), om0 = exp(sl0);
    const double gq = G + m0;
    const double Kc = ag2 * om0 / (gq * gq), Qc = (G + 3.0 * m0 - 2.0 * m0 * m0) / (27.0 * gq);
    double cmax = -INFINITY, cmin = INFINITY;
CFMM_UNROLL
    for (int j = 0; j < 3; ++j) {
        dB[j] = log(pi[j] / pmin);
        const double cj = dB[j] - log(Kc + Qc / u0[j]);
        cmax = fmax(cmax, cj);
        cmin = fmin(cmin, cj);
    }
    if (!(lg + cmax > cmin)) return 0u;                                 // the no-trade band: exactly nothing
    // outer: r(x) = 0 in x = logit(m), bracketed from the current m0
    constexpr double XMAX = 700.0;
    double s = 0.0, m = 0.0, om = 1.0, K = 0.0, Q = 0.0, dr = 0.0, sc = 0.0;
    const double x0 = fmin(fmax(log(fmax(m0, 1e-300)) - log(om0), -XMAX), XMAX);
    double lo = x0, hi = x0;
    if (crypto3_r(x0, G, ag2, dB, lg, u0, lu0, e0, sl0, s, z, kap, m, om, K, Q, dr, sc) > 0.0) {   // r falls in x
        for (double step = 1.0; step <= 1024.0 && lo < XMAX; step *= 2.0) {
            hi = fmin(lo + step, XMAX);
            if (!(crypto3_r(hi, G, ag2, dB, lg, u0, lu0, e0, sl0, s, z, kap, m, om, K, Q, dr, sc) > 0.0)) break;
            lo = hi;
        }
    } else {
        for (double step = 1.0; step <= 1024.0 && hi > -XMAX; step *= 2.0) {
            lo = fmax(hi - step, -XMAX);
            if (crypto3_r(lo, G, ag2, dB, lg, u0, lu0, e0, sl0, s, z, kap, m, om, K, Q, dr, sc) > 0.0) break;
            hi = lo;
        }
    }
    double t = 0.5 * (lo + hi), dx_old = hi - lo, dx = dx_old;
    for (int it = 0; it < 100; ++it) {
        const double f = crypto3_r(t, G, ag2, dB, lg, u0, lu0, e0, sl0, s, z, kap, m, om, K, Q, dr, sc);
        if (f > 0.0) lo = t; else hi = t;
        if (f == 0.0 || !(hi - lo > 4e-16 * (1.0 + fabs(t)))) break;
        const double tn = t - f / dr;
        if (fabs(f) <= 4.5e-16 * sc) {
            if (tn > lo && tn < hi) t = tn;
            break;
        }
        if (!(tn > lo && tn < hi) || fabs(2.0 * f) > fabs(dx_old * dr)) {
            dx_old = dx; dx = 0.5 * (hi - lo); t = lo + dx;
        } else {
            dx_old = dx; dx = tn - t; t = tn;
        }
        if (fabs(dx) <= 1e-15 * (1.0 + fabs(t))) break;
    }
    crypto3_r(t, G, ag2, dB, lg, u0, lu0, e0, sl0, s, z, kap, m, om, K, Q, dr, sc);
    // flows and the Hessian at the answer
    const double g = G + m;
    const double K1 = ag2 * (G + 1.0 + om) / (g * g * g), K2 = ag2 * (4.0 * G + 4.0 + 2.0 * om) / (g * g * g * g);
    const double mu = pmin * exp(-exp(s)) / (gam * K);
    double u[3], e[3], p[3];
    uint32_t mask = 0u;
    int ia = -1, ib = -1, ic = -1;
CFMM_UNROLL
    for (int j = 0; j < 3; ++j) {
        const double ex = expm1(z[j]);
        u[j] = u0[j] * exp(z[j]);
        e[j] = e0[j] + 3.0 * u0[j] * ex;
        p[j] = z[j] > 0.0 ? pi[j] / gam : pi[j];
        if (z[j] != 0.0) {
            if (z[j] > 0.0) D[j] = R[j] * ex / gam; else L[j] = -R[j] * ex;
            mask |= 1u << j;
            if (ia < 0) ia = j; else if (ib < 0) ib = j; else ic = j;
        }
    }
    if (ib >= 0) crypto3_edges(ia, ib, ic, u, e, p, mu, m, om, K, Q, K1, K2, w);
    return mask;
}

// n-coin StableSwap (Curve) pool, n = k = 2..KM coins.  Scaled balances y_j = r_j x_j, whitepaper amplification A,
// a = A n^n, and D = D(R) the invariant of the current reserves (precomputed).  In units of D (u_j = y_j / D) the pool
// keeps G(u) = a sum(u) + 1 - a - Q(u) >= 0, Q(u) = 1 / (n^n prod u); G is strictly concave on u > 0 and
// dG/du_j = a + Q / u_j.  With pi_j = nu_j / r_j a coordinate that grows pays p_j = pi_j / gamma per unit of u, one that
// shrinks earns p_j = pi_j, and the pool solves max -sum_j p_j(u_j - u0_j) s.t. G(u) >= 0.
//   No trade: rho_j = pi_j / dG/du_j(u0); the pool is idle iff gamma max rho <= min rho (in logs: c_j = log(pi_j /
//   pi_min) - log1p(Q0 / (a u0_j)), idle iff log gamma + max c <= min c).  Flows and h are then exactly 0.
//   Otherwise, for the multiplier mu of G and the value Q, the Lagrangian's stationary point is
//       u_j(mu, Q) = clamp(u0_j, Q / (pi_j / (gamma mu) - a), Q / (pi_j / mu - a))     (a denominator <= 0: +inf).
//   Near the peg with large a, pi_j / mu - a must not be formed as a difference: with dB_j = log(pi_j / pi_min) >= 0
//   and the unknown tau = log(pi_min / (gamma a mu)) > 0, the denominators are a expm1(dB_j + tau) and
//   a expm1(dB_j + log gamma + tau), without cancellation.  With l = log(Q / a), l0 = log(Q0 / a):
//       log u_j = log u0_j + z_j,   z_j = max(l - bA_j, 0) + min(l - bB_j, 0),
//       bA_j = log(u0_j expm1(dB_j + tau)),   bB_j = log(u0_j expm1(dB_j + log gamma + tau))  (-inf if that expm1 <= 0),
//   and Q = Q(u) reads F(l) = (l - l0) + sum_j z_j(l) = 0: piecewise linear with slope >= 1, so its root is exact from
//   the 2n breakpoints (as k_eval_geomean's).  h(tau) = sum_j u0_j expm1(z_j) - q0 expm1(l - l0) = G / a at that point
//   (formed from the changes, not from a sum(u) + 1 - a - Q) falls from +inf (tau -> 0) to -inf (tau -> inf); its root
//   is found by bracketing and a bisection-safeguarded Newton iteration in log tau (the stableswap_dir scheme), with
//   dh/dtau = sum_T u_j (l' - kap_j) - q l', kap_j = 1 + 1 / expm1(.)_j, l' = sum_T kap_j / (1 + k) over the traded set T.
//   Then x_j = R_j exp(z_j): D_j = R_j expm1(z_j) / gamma, L_j = -R_j expm1(z_j).
// Hessian.  Differentiating the KKT system p_j = mu dG/du_j (j in T), G = 0: with w = 1/u, -d2G_TT = Q (diag(w^2) + w w'),
// so by Sherman-Morrison its inverse is (diag(u^2) - u u' / (1 + k)) / Q, and eliminating dmu gives the scaled Hessian
// Hs_ij = nu_i nu_j dpsi_i/dnu_j on T x T:
//       v_j = p_j u_j,  c = D / (mu Q),  h_j = sqrt(c) v_j,  C = diag(h^2) - h h' / (1 + k),
//       Hs_TT = C - (C1)(C1)' / (1'C1),   zero outside T.
// It is PSD, Hs 1 = 0, and Hs z costs O(k): Cz = h^2 z - h (h.z) / (1 + k), C1 = h^2 - h sum(h) / (1 + k),
// 1'C1 = sum(h^2) - sum(h)^2 / (1 + k).  Here mu Q = pi_min e^-tau q / gamma (q = Q / a), so c = D gamma e^tau / (pi_min q).
// Arrays of KM entries with the first k used, every loop unrolled over KM: the kernel keeps them in registers.
// Writes D, L and h (0 on untraded slots) and returns the traded slots as a bit mask.  Fixed iteration caps and a
// deterministic exit; shared by the per-thread solver and k_eval_stable_n (cfmm_kernels.cu).

// h(tau) / a at tau = exp(sg), and dh/dsg; z [KM] and l out.  sc: the rounding scale of h (stopping rule)
template <int KM>
CFMM_HD inline double stablen_h(int k, double sg, const double* dB, double lg, const double* u0, const double* lu0,
                                double l0, double q0, double* z, double& l, double& dh, double& sc) {
    const double tau = exp(sg);
    double eA[KM], eB[KM], bA[KM], bB[KM];
CFMM_UNROLL
    for (int j = 0; j < KM; ++j) {
        if (j < k) {
            eA[j] = expm1(dB[j] + tau);
            eB[j] = expm1(dB[j] + lg + tau);
            bA[j] = lu0[j] + log(eA[j]);
            bB[j] = eB[j] > 0.0 ? lu0[j] + log(eB[j]) : -INFINITY;
        }
    }
    // the largest breakpoint with F <= 0 (sL, F there), and the smallest one (sM, F there)
    double sL = -INFINITY, FL = 0.0, sM = INFINITY, FM = 0.0;
CFMM_UNROLL
    for (int p = 0; p < 2 * KM; ++p) {
        if ((p < KM ? p : p - KM) < k) {
            const double T = p < KM ? bA[p] : bB[p - KM];
            if (fabs(T) < INFINITY) {
                double F = T - l0;
CFMM_UNROLL
                for (int j = 0; j < KM; ++j)
                    if (j < k) F += fmax(T - bA[j], 0.0) + fmin(T - bB[j], 0.0);
                if (F <= 0.0 && T > sL) { sL = T; FL = F; }
                if (T < sM) { sM = T; FM = F; }
            }
        }
    }
    double slope = 1.0;
    if (sL > -INFINITY) {
CFMM_UNROLL
        for (int j = 0; j < KM; ++j)
            if (j < k) slope += (sL >= bA[j] ? 1.0 : 0.0) + (sL < bB[j] ? 1.0 : 0.0);
        l = sL - FL / slope;
    } else {                                    // left of every breakpoint only the finite bB bind
CFMM_UNROLL
        for (int j = 0; j < KM; ++j)
            if (j < k) slope += bB[j] > -INFINITY ? 1.0 : 0.0;
        l = sM - FM / slope;
    }
    const double q = q0 * exp(l - l0);
    double h = -q0 * expm1(l - l0), skap = 0.0, su = 0.0, suk = 0.0;
    int kt = 0;
CFMM_UNROLL
    for (int j = 0; j < KM; ++j) {
        if (j < k) {
            z[j] = fmax(l - bA[j], 0.0) + fmin(l - bB[j], 0.0);
            h += u0[j] * expm1(z[j]);
            const double u = u0[j] * exp(z[j]);
            su += u;
            if (z[j] != 0.0) {
                const double kap = 1.0 + 1.0 / (z[j] > 0.0 ? eA[j] : eB[j]);
                ++kt; skap += kap; suk += u * kap;
            }
        }
    }
    double sut = 0.0;
CFMM_UNROLL
    for (int j = 0; j < KM; ++j)
        if (j < k && z[j] != 0.0) sut += u0[j] * exp(z[j]);
    const double lt = skap / (1.0 + kt);
    dh = tau * (sut * lt - suk - q * lt);
    sc = (su + q) * (1.0 + fabs(l));
    return h;
}

template <int KM>
CFMM_HD inline uint32_t stableswap_n(int k, const double* R, const double* r, double A, double Dv, double gam,
                                     const double* nu, double* D, double* L, double* hs) {
    double u0[KM], lu0[KM], pi[KM], dB[KM], z[KM];
    double nn = 1.0, slu = 0.0, pmin = INFINITY;
CFMM_UNROLL
    for (int j = 0; j < KM; ++j) {
        if (j < k) {
            nn *= (double)k;
            D[j] = L[j] = hs[j] = 0.0;
            u0[j] = r[j] * R[j] / Dv;
            lu0[j] = log(u0[j]);
            slu += lu0[j];
            pi[j] = nu[j] / r[j];
            pmin = fmin(pmin, pi[j]);
        }
    }
    const double a = A * nn;
    const double l0 = -((double)k * log((double)k) + slu) - log(a), q0 = exp(l0), lg = log(gam);
    double cmax = -INFINITY, cmin = INFINITY;
CFMM_UNROLL
    for (int j = 0; j < KM; ++j) {
        if (j < k) {
            dB[j] = log(pi[j] / pmin);
            const double c = dB[j] - log1p(q0 / u0[j]);
            cmax = fmax(cmax, c);
            cmin = fmin(cmin, c);
        }
    }
    if (!(lg + cmax > cmin)) return 0u;                                 // the no-trade band: exactly nothing
    constexpr double SMIN = -700.0, SMAX = 6.39;                        // log tau: tau in (1e-304, 600), exp finite
    double l = 0.0, dh = 0.0, sc = 0.0;
    // start where the last grower stops growing at Q = Q0, then bracket: h(lo) > 0 >= h(hi)
    const double sg = fmin(fmax(log(-cmin), SMIN), SMAX);
    double lo = sg, hi = sg;
    if (stablen_h<KM>(k, sg, dB, lg, u0, lu0, l0, q0, z, l, dh, sc) > 0.0) {
        for (double step = 1.0; step <= 512.0 && lo < SMAX; step *= 2.0) {
            hi = fmin(lo + step, SMAX);
            if (!(stablen_h<KM>(k, hi, dB, lg, u0, lu0, l0, q0, z, l, dh, sc) > 0.0)) break;
            lo = hi;
        }
    } else {
        for (double step = 1.0; step <= 512.0 && hi > SMIN; step *= 2.0) {
            lo = fmax(hi - step, SMIN);
            if (stablen_h<KM>(k, lo, dB, lg, u0, lu0, l0, q0, z, l, dh, sc) > 0.0) break;
            hi = lo;
        }
    }
    // safeguarded Newton inside [lo, hi] (h falls in log tau), as stableswap_dir
    double t = 0.5 * (lo + hi), dx_old = hi - lo, dx = dx_old;
    for (int it = 0; it < 100; ++it) {
        const double f = stablen_h<KM>(k, t, dB, lg, u0, lu0, l0, q0, z, l, dh, sc);
        if (f > 0.0) lo = t; else hi = t;
        if (f == 0.0 || !(hi - lo > 4e-16 * (1.0 + fabs(t)))) break;
        const double tn = t - f / dh;
        // h is at the level of its own rounding (the z_j carry absolute errors of a few u |l|): stop there
        if (fabs(f) <= 4.5e-16 * sc) {
            if (tn > lo && tn < hi) t = tn;
            break;
        }
        if (!(tn > lo && tn < hi) || fabs(2.0 * f) > fabs(dx_old * dh)) {
            dx_old = dx; dx = 0.5 * (hi - lo); t = lo + dx;
        } else {
            dx_old = dx; dx = tn - t; t = tn;
        }
        if (fabs(dx) <= 1e-15 * (1.0 + fabs(t))) break;
    }
    stablen_h<KM>(k, t, dB, lg, u0, lu0, l0, q0, z, l, dh, sc);
    const double q = q0 * exp(l - l0);
    const double sc_h = sqrt(Dv * gam * exp(exp(t)) / (pmin * q));
    uint32_t mask = 0u;
CFMM_UNROLL
    for (int j = 0; j < KM; ++j) {
        if (j < k && z[j] != 0.0) {
            const double e = expm1(z[j]);
            if (z[j] > 0.0) D[j] = R[j] * e / gam; else L[j] = -R[j] * e;
            hs[j] = sc_h * (z[j] > 0.0 ? pi[j] / gam : pi[j]) * u0[j] * exp(z[j]);
            mask |= 1u << j;
        }
    }
    return mask;
}

// The pieces of one n-coin StableSwap pool's block Hs = C - (C1)(C1)' / (1'C1), C = diag(h^2) - h h' / (1 + k), from its
// per-slot h (0 off the traded set T, k = |T|): c1 [KM] = C1 (0 off T), inv = 1 / (1 + k); returns 1'C1 (<= 0: fewer
// than two traded slots, the block is 0).  Shared by the per-thread solver's dense assembly, stablen_hvp and the diagonal
// and dense kernels of cfmm_kernels.cu.
template <int KM>
CFMM_HD inline double stablen_c1(int k, const double* h, double* c1, double& inv) {
    double sh = 0.0, sh2 = 0.0;
    int kt = 0;
CFMM_UNROLL
    for (int j = 0; j < KM; ++j)
        if (j < k && h[j] != 0.0) { ++kt; sh += h[j]; sh2 += h[j] * h[j]; }
    inv = 1.0 / (1.0 + kt);
CFMM_UNROLL
    for (int j = 0; j < KM; ++j)
        if (j < k) c1[j] = h[j] * h[j] - h[j] * sh * inv;
    return sh2 - sh * sh * inv;
}

// Hs z for one n-coin StableSwap pool from its per-slot h: (Hs z)_j, j < k, into y.  O(k): Cz = h^2 z - h (h.z) / (1 + k)
// and (C1)'z = 1'Cz.
template <int KM>
CFMM_HD inline void stablen_hvp(int k, const double* h, const double* zin, double* y) {
    double c1[KM], inv;
    const double s1 = stablen_c1<KM>(k, h, c1, inv);
    double shz = 0.0, c1z = 0.0;
CFMM_UNROLL
    for (int j = 0; j < KM; ++j)
        if (j < k) shz += h[j] * zin[j];
CFMM_UNROLL
    for (int j = 0; j < KM; ++j) {
        if (j < k) {
            y[j] = h[j] * h[j] * zin[j] - h[j] * shz * inv;                // (Cz)_j
            c1z += y[j];
        }
    }
    const double f = s1 > 0.0 ? c1z / s1 : 0.0;
CFMM_UNROLL
    for (int j = 0; j < KM; ++j)
        if (j < k) y[j] = s1 > 0.0 ? y[j] - c1[j] * f : 0.0;
}

#ifdef __CUDA_ARCH__
// sum over the LANES consecutive lanes that share a problem; x + y == y + x exactly, so every lane ends with the same bits
template <int LANES>
__device__ __forceinline__ double lanes_sum(double v) {
CFMM_UNROLL
    for (int o = LANES / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
#endif

// One dual evaluation of the problem: psi = sum_i A_i (L_i - D_i), returns arb = sum_i nu_i'(L_i - D_i).
// Hs (n x n, nullable) receives the scaled Hessian (true Hessian = diag(1/nu) Hs diag(1/nu)).
//
// LANES > 1 (device only): LANES threads of one warp own the SAME problem.  Every lane keeps a full private copy of the
// state and runs the identical instruction stream; only this pool loop is split (lane l takes pools l, l+LANES, ...)
// and the partial psi / arb / Hessian / fills are then summed over the lanes with an xor butterfly, which leaves
// bit-identical totals in every lane -- so the lanes never diverge and need no other communication.
// STABLE: the instance that also evaluates StableSwap pools (kind 4).  The plain instance keeps the register budget it
// had before that kind existed and rejects such pools (solve_one: status 3); cfmm_batch_solve_stableswap runs the other.
// STABLE_N (with STABLE): kind-4 pools of 2..KMAX coins, those of more than two through stableswap_n, whose k x k block
// of Hs is added to the dense system; cfmm_batch_solve_stableswap_n runs this third instance.  Without it a kind-4 pool
// of more than two coins makes its problem status 3.
// LADDER (with STABLE and STABLE_N): also concentrated pools (kind 6) through ladder_pair, their (s, c) in the pool's two
// w slots, (first record, T) in its two logrw slots and the records in `rec`; cfmm_batch_solve_concentrated runs this
// fourth instance.  The other instances give problems with such pools status 3.
// CRYPTO (with all three): also two-coin cryptoswap pools (kind 8) through cryptoswap_pair, c_j = p_j / D in the pool's
// two w slots and (A, G) in its two logrw slots; cfmm_batch_solve_cryptoswap runs this fifth instance.  The other
// instances give problems with such pools status 3.
// CRYPTO3 (with all four): also three-coin cryptoswap pools (kind 9) through cryptoswap3, c_j = p_j / D in the pool's
// three w slots and (A, G) in its first two logrw slots, the Hessian block added from the three edge weights;
// cfmm_batch_solve_tricrypto runs this sixth instance.  The other instances give problems with such pools status 3.
// BINS (with all five): also price-bin pools (kind 10) through bins_pair, (z, p_ref) in the pool's two w slots, (first
// record, nb) in its two logrw slots, the records in `rec` (shared with the concentrated pools') and the multiplier tbar in
// its first theta_bar slot; cfmm_batch_solve_bins runs this seventh instance.  The others give such problems status 3.
// ECLP (with all six): also E-CLP pools (kind 11) through eclp_pair, their record {c, s, lam, alpha, beta, r, p, 0} (two
// record slots) in `rec` after the ladders' and bins', its record index in the pool's first logrw slot;
// cfmm_batch_solve_eclp runs this eighth instance.  The others give such problems status 3.
// PMM (with all seven): also DODO PMM pools (kind 12) through pmm_pair, their record {pi, k, B0, Q0} (one record slot)
// in `rec` after the E-CLPs', its record index in the pool's first logrw slot; cfmm_batch_solve_pmm runs this ninth
// instance.  The others give such problems status 3.
template <int LANES, bool STABLE = false, bool STABLE_N = false, bool LADDER = false, bool CRYPTO = false,
          bool CRYPTO3 = false, bool BINS = false, bool ECLP = false, bool PMM = false>
CFMM_HD inline double evaluate(const Pools& P, const Problem& Q, const Vec& nu, const Vec& lognu, double eps,
                               const Vec& psi, const Vec* Hs, bool trades, bool store_fill, int lane,
                               const double* rec = nullptr) {
    const int n = Q.n;
    for (int j = 0; j < n; ++j) { lognu[j] = log(nu[j]); psi[j] = 0.0; }
    if (Hs) for (int e = 0; e < n * n; ++e) (*Hs)[e] = 0.0;
    if (LANES > 1 && store_fill) {
        const int64_t nnz = P.pool_ptr[Q.p1] - Q.off0;
        for (int64_t x = 0; x < nnz; ++x) Q.theta_new[x] = 0.0;
    }
    double arb = 0.0;
    for (int64_t i = Q.p0 + (LANES > 1 ? lane : 0); i < Q.p1; i += LANES) {
        const int64_t off = P.pool_ptr[i];
        const int k = (int)(P.pool_ptr[i + 1] - off);
        const double gam = P.gamma[i];
        double D[KMAX], L[KMAX];
        if (CRYPTO3 && P.kind[i] == 9) {                                  // c = p / D in w, (A, G) in logrw
            double w[3];
            const uint32_t mask = cryptoswap3(P.R[off], P.R[off + 1], P.R[off + 2], P.w[off], P.w[off + 1], P.w[off + 2],
                                              P.logrw[off], P.logrw[off + 1], gam, nu[P.tok[off]], nu[P.tok[off + 1]],
                                              nu[P.tok[off + 2]], D, L, w);
            if (Hs && mask) {                                              // Hs = sum_{a<b} w_ab (e_a - e_b)(e_a - e_b)'
                for (int q = 0; q < 3; ++q) {
                    if (w[q] == 0.0) continue;
                    const int ta = P.tok[off + (q == 2 ? 1 : 0)], tb = P.tok[off + (q == 0 ? 1 : 2)];
                    (*Hs)[ta * n + ta] += w[q]; (*Hs)[tb * n + tb] += w[q];
                    (*Hs)[ta * n + tb] -= w[q]; (*Hs)[tb * n + ta] -= w[q];
                }
            }
        } else if (CRYPTO && P.kind[i] == 8) {                            // c = p / D in w, (A, G) in logrw
            double hc = 0.0;
            cryptoswap_pair(P.R[off], P.R[off + 1], P.w[off], P.w[off + 1], P.logrw[off], P.logrw[off + 1], gam,
                            nu[P.tok[off]], nu[P.tok[off + 1]], D, L, hc);
            if (Hs && hc != 0.0) {
                const int t0 = P.tok[off], t1 = P.tok[off + 1];
                (*Hs)[t0 * n + t0] += hc; (*Hs)[t1 * n + t1] += hc;
                (*Hs)[t0 * n + t1] -= hc; (*Hs)[t1 * n + t0] -= hc;
            }
        } else if (BINS && P.kind[i] == 10) {                 // (z, p_ref) in w, (first record, nb) in logrw, tbar in theta_bar
            double hc = 0.0;
            const double t = bins_pair(rec + 4 * (int64_t)P.logrw[off], (int64_t)P.logrw[off + 1], (int64_t)P.w[off],
                                       P.w[off + 1], eps > 0.0 ? Q.theta_bar[off - Q.off0] : 0.0, gam, nu[P.tok[off]],
                                       nu[P.tok[off + 1]], eps, D, L, hc);
            if (store_fill) { Q.theta_new[off - Q.off0] = t; Q.theta_new[off - Q.off0 + 1] = 0.0; }
            if (Hs && hc != 0.0) {
                const int t0 = P.tok[off], t1 = P.tok[off + 1];
                (*Hs)[t0 * n + t0] += hc; (*Hs)[t1 * n + t1] += hc;
                (*Hs)[t0 * n + t1] -= hc; (*Hs)[t1 * n + t0] -= hc;
            }
        } else if (LADDER && P.kind[i] == 6) {                                   // (s, c) in w, (first record, T) in logrw
            double hc = 0.0;
            ladder_pair(rec + 4 * (int64_t)P.logrw[off], (int64_t)P.logrw[off + 1], (int64_t)P.w[off + 1], P.w[off], gam,
                        nu[P.tok[off]], nu[P.tok[off + 1]], D, L, hc);
            if (Hs && hc != 0.0) {
                const int t0 = P.tok[off], t1 = P.tok[off + 1];
                (*Hs)[t0 * n + t0] += hc; (*Hs)[t1 * n + t1] += hc;
                (*Hs)[t0 * n + t1] -= hc; (*Hs)[t1 * n + t0] -= hc;
            }
        } else if (STABLE_N && P.kind[i] == 4 && k > 2) {                       // rates in w, (A, D) in logrw's first two slots
            double Rl[KMAX], rl[KMAX], nl[KMAX], hl[KMAX];
            for (int j = 0; j < KMAX; ++j) {
                if (j < k) { Rl[j] = P.R[off + j]; rl[j] = P.w[off + j]; nl[j] = nu[P.tok[off + j]]; }
            }
            stableswap_n<KMAX>(k, Rl, rl, P.logrw[off], P.logrw[off + 1], gam, nl, D, L, hl);
            if (Hs) {                                                      // Hs_TT = C - (C1)(C1)' / (1'C1)
                double c1[KMAX], inv;
                const double s1 = stablen_c1<KMAX>(k, hl, c1, inv);
                if (s1 > 0.0) {
                    for (int x = 0; x < k; ++x) {
                        if (hl[x] == 0.0) continue;
                        const int tx = P.tok[off + x];
                        for (int y = 0; y < k; ++y) {
                            if (hl[y] == 0.0) continue;
                            (*Hs)[tx * n + P.tok[off + y]] += (x == y ? hl[x] * hl[x] : 0.0) - hl[x] * hl[y] * inv - c1[x] * c1[y] / s1;
                        }
                    }
                }
            }
        } else if (ECLP && P.kind[i] == 11) {                         // {c, s, lam, alpha, beta, r, p, 0} in rec
            double hc = 0.0;
            const double* e = rec + 4 * (int64_t)P.logrw[off];
            eclp_pair(P.R[off], P.R[off + 1], e[3], e[4], e[0], e[1], e[2], e[5], e[6], gam, nu[P.tok[off]],
                      nu[P.tok[off + 1]], D, L, hc);
            if (Hs && hc != 0.0) {
                const int t0 = P.tok[off], t1 = P.tok[off + 1];
                (*Hs)[t0 * n + t0] += hc; (*Hs)[t1 * n + t1] += hc;
                (*Hs)[t0 * n + t1] -= hc; (*Hs)[t1 * n + t0] -= hc;
            }
        } else if (PMM && P.kind[i] == 12) {                          // {pi, k, B0, Q0} in rec
            double hc = 0.0;
            const double* e = rec + 4 * (int64_t)P.logrw[off];
            pmm_pair(P.R[off], P.R[off + 1], e[0], e[1], e[2], e[3], gam, nu[P.tok[off]], nu[P.tok[off + 1]], D, L, hc);
            if (Hs && hc != 0.0) {
                const int t0 = P.tok[off], t1 = P.tok[off + 1];
                (*Hs)[t0 * n + t0] += hc; (*Hs)[t1 * n + t1] += hc;
                (*Hs)[t0 * n + t1] -= hc; (*Hs)[t1 * n + t0] -= hc;
            }
        } else if (P.kind[i] == 3 || (STABLE && P.kind[i] == 4)) {
            double hc = 0.0;
            if (!STABLE || P.kind[i] == 3)
                bounded_pair(P.R[off], P.R[off + 1], P.w[off], P.w[off + 1], gam, nu[P.tok[off]], nu[P.tok[off + 1]], D, L, hc);
            else                                                           // rates in w, (A, D) in logrw
                stableswap_pair(P.R[off], P.R[off + 1], P.w[off], P.w[off + 1], P.logrw[off], P.logrw[off + 1], gam,
                                nu[P.tok[off]], nu[P.tok[off + 1]], D, L, hc);
            if (Hs && hc != 0.0) {
                const int t0 = P.tok[off], t1 = P.tok[off + 1];
                (*Hs)[t0 * n + t0] += hc; (*Hs)[t1 * n + t1] += hc;
                (*Hs)[t0 * n + t1] -= hc; (*Hs)[t1 * n + t0] -= hc;
            }
        } else if (P.kind[i] != 1) {
            double wa[KMAX];
            double M = 0.0;
            if (k == 2 && P.w[off] == P.w[off + 1]) {                      // sqrt(x0 x1) >= sqrt(R0 R1), arbitrage.py:68-70
                const double R0 = P.R[off], R1 = P.R[off + 1];
                const double p0 = nu[P.tok[off]] * R0, p1 = nu[P.tok[off + 1]] * R1;
                const bool f = gam * p1 > p0, b = gam * p0 > p1;
                const double q = f ? gam * p1 / p0 : (b ? gam * p0 / p1 : 1.0);
                const double t = sqrt(q);
                D[0] = f ? R0 * (t - 1.0) / gam : 0.0;
                L[1] = f ? R1 * (1.0 - 1.0 / t) : 0.0;
                D[1] = b ? R1 * (t - 1.0) / gam : 0.0;
                L[0] = b ? R0 * (1.0 - 1.0 / t) : 0.0;
                M = (f || b) ? 2.0 * sqrt(p0 * p1 / gam) : 0.0;
                wa[0] = wa[1] = (f || b) ? 0.5 : 0.0;
            } else {                                                       // weighted geometric mean, arbitrage.py:65
                double tA[KMAX], tB[KMAX];
                const double lg = log(gam);
                double maxB = -INFINITY, minA = INFINITY;
                for (int j = 0; j < k; ++j) {
                    tB[j] = P.logrw[off + j] + lognu[P.tok[off + j]];
                    tA[j] = tB[j] - lg;
                    maxB = fmax(maxB, tB[j]);
                    minA = fmin(minA, tA[j]);
                }
                const bool trade = maxB > minA;
                double sL = -INFINITY, hL = 0.0;                            // largest breakpoint with h <= 0
                for (int cnd = 0; cnd < 2 * k; ++cnd) {
                    const double T = cnd < k ? tA[cnd] : tB[cnd - k];
                    double hT = 0.0;
                    for (int j = 0; j < k; ++j) hT += P.w[off + j] * (fmax(T - tA[j], 0.0) + fmin(T - tB[j], 0.0));
                    if (hT <= 0.0 && T > sL) { sL = T; hL = hT; }
                }
                double W = 0.0;
                for (int j = 0; j < k; ++j) if (sL >= tA[j] || sL < tB[j]) W += P.w[off + j];
                const double s = hL < 0.0 ? sL - hL / fmax(W, TINY) : sL;
                for (int j = 0; j < k; ++j) {
                    const double zA = trade ? fmax(s - tA[j], 0.0) : 0.0;
                    const double zB = trade ? fmin(s - tB[j], 0.0) : 0.0;
                    D[j] = P.R[off + j] * expm1(zA) / gam;
                    L[j] = -P.R[off + j] * expm1(zB);
                    wa[j] = (zA > 0.0 || zB < 0.0) ? P.w[off + j] : 0.0;
                }
                M = trade ? exp(s) : 0.0;
            }
            if (Hs && M > 0.0) {
                double Wa = 0.0;
                for (int j = 0; j < k; ++j) Wa += wa[j];
                Wa = fmax(Wa, TINY);
                for (int x = 0; x < k; ++x) {
                    const int tx = P.tok[off + x];
                    (*Hs)[tx * n + tx] += M * wa[x];
                    for (int y = 0; y < k; ++y) (*Hs)[tx * n + P.tok[off + y]] -= (M / Wa) * wa[x] * wa[y];
                }
            }
        } else {                                                           // constant sum with x >= 0, arbitrage.py:73-74
            double hc = 0.0;
            D[0] = D[1] = L[0] = L[1] = 0.0;
            for (int dir = 0; dir < 2; ++dir) {                            // limit order: tender ta, receive up to R_tb of tb
                const int ta = dir, tb = 1 - dir;
                const double na = nu[P.tok[off + ta]], nb = nu[P.tok[off + tb]];
                const double r = gam * nb / na, z = r - 1.0, Rb = P.R[off + tb];
                double th, ps, curv = 0.0;
                if (eps <= 0.0) {
                    th = z > 0.0 ? Rb : 0.0;
                    ps = th * z;
                } else {
                    const double sigma = Rb / eps, bar = Q.theta_bar[off - Q.off0 + tb];
                    th = fmin(fmax(bar + sigma * z, 0.0), Rb);
                    ps = th * z - (th - bar) * (th - bar) / (2.0 * sigma);
                    curv = (th > 0.0 && th < Rb) ? sigma : 0.0;
                }
                L[tb] = th;
                D[ta] = (r * th - ps) / gam;
                hc += curv * nb * r;
            }
            if (store_fill) { Q.theta_new[off - Q.off0] = L[0]; Q.theta_new[off - Q.off0 + 1] = L[1]; }
            if (Hs && hc != 0.0) {
                const int t0 = P.tok[off], t1 = P.tok[off + 1];
                (*Hs)[t0 * n + t0] += hc; (*Hs)[t1 * n + t1] += hc;
                (*Hs)[t0 * n + t1] -= hc; (*Hs)[t1 * n + t0] -= hc;
            }
        }
        for (int j = 0; j < k; ++j) {
            const double y = L[j] - D[j];
            const int t = P.tok[off + j];
            psi[t] += y;
            arb += nu[t] * y;
            if (trades && Q.delta) { Q.delta[off + j] = D[j]; Q.lam[off + j] = L[j]; }
        }
    }
#ifdef __CUDA_ARCH__
    if (LANES > 1) {
        arb = lanes_sum<LANES>(arb);
        for (int j = 0; j < n; ++j) psi[j] = lanes_sum<LANES>(psi[j]);
        if (Hs) for (int e = 0; e < n * n; ++e) (*Hs)[e] = lanes_sum<LANES>((*Hs)[e]);
        if (store_fill) {
            const int64_t nnz = P.pool_ptr[Q.p1] - Q.off0;
            for (int64_t x = 0; x < nnz; ++x) Q.theta_new[x] = lanes_sum<LANES>(Q.theta_new[x]);
        }
    }
#endif
    return arb;
}

CFMM_HD inline double dual_value(const Problem& Q, const Vec& nu, double arb) {
    double g = arb;
    for (int j = 0; j < Q.n; ++j) g += (nu[j] - Q.c[j]) * Q.a[j];
    return g;
}

// KKT residual of the box-constrained dual: err = sum_free |nu_j (a_j + psi_j)| / |g|; fills grad / pg / free mask.
CFMM_HD inline double kkt(const Problem& Q, const Vec& nu, const Vec& psi, const Vec& lb, double g, double err_prev,
                          const Vec& grad, const Vec& pg, uint64_t* free_mask) {
    const double ep = isfinite(err_prev) ? err_prev : 1e-2;
    const double thr = fmin(1e-2, fmax(1e-3 * ep, 1e-14));       // active-set width: 1e-3 x the KKT residual (see solver.py)
    double num = 0.0, wsum = 0.0, gmax = 0.0, scl = 0.0;
    uint64_t fm = 0;
    for (int j = 0; j < Q.n; ++j) {
        const double gr = Q.a[j] + psi[j];
        const bool near = nu[j] <= lb[j] * (1.0 + thr) && !is_eq(Q, j);
        const bool fr = !(is_pinned(Q, j) || (near && gr > 0.0));
        const double v = fr ? nu[j] * gr : 0.0;
        grad[j] = gr; pg[j] = v;
        if (fr) fm |= (uint64_t)1 << j;
        num += fabs(v);
        wsum += nu[j] * fabs(gr);
        if (fr) gmax = fmax(gmax, fabs(gr));
        scl = fmax(scl, fmax(fabs(Q.a[j]), is_pinned(Q, j) ? 0.0 : fabs(psi[j])));   // scale: constrained flows only
    }
    *free_mask = fm;
    // max of the value-weighted residual and the per-token one (the reference constrains psi token by token,
    // liquidation.py:77-80 / arbitrage.py:77: a cheap token must not hide a large residual behind its price)
    return fmax(num / fmax(fmax(fabs(g), 1e-3 * wsum), TINY), gmax / fmax(scl, TINY));
}

// Solve (Hs[free,free] + mu dbar I) x = -pg[free] (dbar = mean diagonal) by Gaussian elimination with partial pivoting;
// dt = 0 off the free set.  Returns 0 = descent direction, 1 = solved but not a descent direction, 2 = singular / not finite;
// *big = largest |x_j| (the caller climbs the damping ladder while it is not a sane log-price change).
CFMM_HD inline int newton_direction(int n, uint64_t free_mask, const Vec& Hs, const Vec& pg, const Vec& A,
                                     const Vec& dt, double mu, double* big) {
    int fidx[NTOK_MAX];
    int nf = 0;
    for (int j = 0; j < n; ++j) { dt[j] = 0.0; if (free_mask >> j & 1) fidx[nf++] = j; }
    *big = 0.0;
    if (nf == 0) return 1;
    double tr = 0.0;
    for (int x = 0; x < nf; ++x) tr += Hs[fidx[x] * n + fidx[x]];
    const double reg = mu * fmax(tr / nf, TINY);
    const int ld = nf + 1;                                                  // augmented [A | rhs], row-major in A
    for (int x = 0; x < nf; ++x) {
        for (int y = 0; y < nf; ++y) A[x * ld + y] = Hs[fidx[x] * n + fidx[y]] + (x == y ? reg : 0.0);
        A[x * ld + nf] = -pg[fidx[x]];
    }
    for (int col = 0; col < nf; ++col) {
        int piv = col;
        double best = fabs(A[col * ld + col]);
        for (int r = col + 1; r < nf; ++r) { const double v = fabs(A[r * ld + col]); if (v > best) { best = v; piv = r; } }
        if (!(best > 0.0) || !isfinite(best)) return 2;
        if (piv != col)
            for (int y = col; y <= nf; ++y) { const double t = A[col * ld + y]; A[col * ld + y] = A[piv * ld + y]; A[piv * ld + y] = t; }
        const double inv = 1.0 / A[col * ld + col];
        for (int r = col + 1; r < nf; ++r) {
            const double f = A[r * ld + col] * inv;
            if (f != 0.0) for (int y = col + 1; y <= nf; ++y) A[r * ld + y] -= f * A[col * ld + y];
        }
    }
    double slope = 0.0;
    bool finite = true;
    for (int x = nf - 1; x >= 0; --x) {
        double v = A[x * ld + nf];
        for (int y = x + 1; y < nf; ++y) v -= A[x * ld + y] * dt[fidx[y]];
        v /= A[x * ld + x];
        dt[fidx[x]] = v;
        finite = finite && isfinite(v);
        *big = fmax(*big, fabs(v));
    }
    for (int x = 0; x < nf; ++x) slope += pg[fidx[x]] * dt[fidx[x]];
    if (!finite) return 2;
    return slope < 0.0 ? 0 : 1;
}

// Workspace elements one problem needs (doubles): 12 n-vectors, 2 Hessians, the augmented system, 2 multiplier sets.
CFMM_HD inline int64_t work_doubles(int n, int64_t nnz) { return 12LL * n + 2LL * n * n + (int64_t)n * (n + 1) + 2 * nnz; }

// The solve.  nu_io [n]: start prices in, optimal prices out.  psi_out [n].  `work`/`stride`: interleaved workspace.
// rec: the concentrated and price-bin pools' records (LADDER and BINS instances only).
template <int LANES = 1, bool STABLE = false, bool STABLE_N = false, bool LADDER = false, bool CRYPTO = false,
          bool CRYPTO3 = false, bool BINS = false, bool ECLP = false, bool PMM = false>
CFMM_HD inline Stats solve_one(const Pools& P, Problem Q, const Params& prm, double* nu_io, double* psi_out,
                               double* work, int64_t stride, int lane = 0, const double* rec = nullptr) {
    const int n = Q.n;
    const int64_t nnz = P.pool_ptr[Q.p1] - Q.off0;
    int64_t e = 0;
    auto vec = [&](int64_t len) { Vec v{work + e * stride, stride}; e += len; return v; };
    Vec nuv[2] = {vec(n), vec(n)}, psiv[2] = {vec(n), vec(n)};
    Vec grad = vec(n), pg = vec(n), dt = vec(n), lb = vec(n), lognu = vec(n), grad_t = vec(n), pg_t = vec(n), spare = vec(n);
    Vec Hsv[2] = {vec(n * n), vec(n * n)};
    Vec A = vec((int64_t)n * (n + 1));
    Q.theta_bar = vec(nnz);
    Q.theta_new = vec(nnz);
    (void)spare;

    bool has_sum = false, bad = n < 1 || n > NTOK_MAX;
    for (int64_t i = Q.p0; i < Q.p1 && !bad; ++i) {                         // refuse what the closed forms do not cover
        const int64_t o = P.pool_ptr[i];
        const int k = (int)(P.pool_ptr[i + 1] - o);
        has_sum = has_sum || P.kind[i] == 1 || (BINS && P.kind[i] == 10);
        bad = (P.kind[i] > (STABLE ? 4 : 3) && !(LADDER && P.kind[i] == 6) && !(CRYPTO && P.kind[i] == 8) &&
               !(CRYPTO3 && P.kind[i] == 9) && !(BINS && P.kind[i] == 10) && !(ECLP && P.kind[i] == 11) &&
               !(PMM && P.kind[i] == 12)) || k < 2 ||
              k > KMAX || ((P.kind[i] == 1 || P.kind[i] == 3 || (STABLE && !STABLE_N && P.kind[i] == 4) ||
                (LADDER && P.kind[i] == 6) || (CRYPTO && P.kind[i] == 8) || (BINS && P.kind[i] == 10) ||
                (ECLP && P.kind[i] == 11) || (PMM && P.kind[i] == 12)) && k != 2) ||
              (CRYPTO3 && P.kind[i] == 9 && k != 3);
        for (int j = 0; j < k && !bad; ++j) bad = P.tok[o + j] < 0 || P.tok[o + j] >= n;
    }
    if (bad) {
        Stats st;
        st.value = st.dual = st.gap = st.infeas = st.err = NAN;
        st.iters = st.evals = 0; st.status = 3;                             // 3 = rejected input
        return st;
    }
    for (int64_t x = 0; x < nnz; ++x) { Q.theta_bar[x] = 0.0; Q.theta_new[x] = 0.0; }

    double scale = 1.0;
    for (int j = 0; j < n; ++j) scale = fmax(scale, fabs(Q.c[j]));
    const double floor_ = prm.floor_rel * scale;
    int cur = 0;
    for (int j = 0; j < n; ++j) {
        lb[j] = is_eq(Q, j) ? floor_ : fmax(Q.c[j], floor_);
        nuv[0][j] = is_pinned(Q, j) ? Q.c[j] : fmax(nu_io[j], lb[j]);
    }

    int evals = 0, iters = 0, status = 1;                                   // 0 optimal, 1 max_iter, 2 stalled
    double eps_t = has_sum ? prm.eps0 : 0.0;
    double err = INFINITY, move = 1.0, g = 0.0;
    bool failed_before = false;
    uint64_t free_mask = 0, fm_t = 0;

    for (int outer = 0; outer < prm.max_outer; ++outer) {
        g = dual_value(Q, nuv[cur], evaluate<LANES, STABLE, STABLE_N, LADDER, CRYPTO, CRYPTO3, BINS, ECLP, PMM>(P, Q, nuv[cur], lognu, eps_t, psiv[cur], &Hsv[cur], false, false, lane, rec));
        ++evals;
        int inner_status = 1;
        const double inner_tol = has_sum ? fmax(prm.tol, fmin(1e-3, 1e-2 * move)) : prm.tol;
        err = kkt(Q, nuv[cur], psiv[cur], lb, g, err, grad, pg, &free_mask);
        for (int it = 0; it < prm.max_inner; ++it) {
            ++iters;
#ifdef CFMM_SMALL_TRACE
            printf("outer=%d it=%d g=%.15g err=%.3e free=%d\n", outer, iters, g, err, __builtin_popcountll(free_mask));
#endif
            if (err <= inner_tol) { inner_status = 0; break; }
            // (near-)singular free-set systems (every pool tying some free prices to the rest saturated) give an enormous
            // step along the null directions: climb the damping ladder (Levenberg-Marquardt shift mu * mean diagonal)
            // until the step is a sane price change; the null directions then get a scaled gradient step
            const double mus[6] = {1e-14, 1e-8, 1e-6, 1e-4, 1e-2, 1.0};
            const int nxt = cur ^ 1;
            double alpha = 1.0, g_t = g;
            bool ok = false;
            for (int rung = 0;;) {
                int code = 2;
                for (;; ++rung) {                                        // climb until the step is a sane price change
                    double big = 0.0;
                    code = newton_direction(n, free_mask, Hsv[cur], pg, A, dt, mus[rung], &big);
                    if ((code != 2 && big <= DT_MAX) || rung == 5) break;
                }
                if (code != 0) {                                         // fall back to scaled steepest descent
                    double mx = 0.0;
                    for (int j = 0; j < n; ++j) mx = fmax(mx, fabs(pg[j]));
                    mx = fmax(mx, TINY);
                    for (int j = 0; j < n; ++j) dt[j] = -pg[j] / mx;
                }
                {                                                        // still too long after the largest shift:
                    double big = 0.0;                                    // keep the direction, bound the step
                    for (int j = 0; j < n; ++j) big = fmax(big, fabs(dt[j]));
                    if (big > DT_MAX) for (int j = 0; j < n; ++j) dt[j] *= DT_MAX / big;
                }
                alpha = 1.0;
                double lin1 = 0.0;                                       // predicted decrease of the FULL step
                for (int ls = 0; ls < 50; ++ls) {
                    double lin = 0.0;
                    for (int j = 0; j < n; ++j) {
                        const double st = fmin(fmax(alpha * dt[j], -20.0), 20.0);
                        const double v = is_pinned(Q, j) ? Q.c[j] : fmax(nuv[cur][j] * exp(st), lb[j]);
                        nuv[nxt][j] = v;
                        lin += grad[j] * (v - nuv[cur][j]);
                    }
                    g_t = dual_value(Q, nuv[nxt], evaluate<LANES, STABLE, STABLE_N, LADDER, CRYPTO, CRYPTO3, BINS, ECLP, PMM>(P, Q, nuv[nxt], lognu, eps_t, psiv[nxt], &Hsv[nxt], false, false, lane, rec));
                    ++evals;
                    if (ls == 0) lin1 = lin;
                    if (g_t <= g + 1e-4 * lin) { ok = true; break; }
                    if (fabs(g_t - g) <= 1e-13 * fabs(g) || fabs(lin1) <= 1e-9 * fabs(g)) {  // g cannot resolve this step
                        if (kkt(Q, nuv[nxt], psiv[nxt], lb, g_t, err, grad_t, pg_t, &fm_t) < 0.99 * err) { ok = true; break; }
                        if (alpha < 1e-3) break;
                    }
                    alpha *= 0.5;
                }
                // a failed search along a barely damped direction (null-space dominated: long step, no predicted gain):
                // damp harder and try again before giving up
                if (ok || rung == 5) break;
                ++rung;
            }
#ifdef CFMM_SMALL_TRACE
            { double mx = 0; int jm = 0; for (int j = 0; j < n; ++j) if (fabs(pg[j]) > mx) { mx = fabs(pg[j]); jm = j; }
              printf("   ok=%d alpha=%.3e g_t-g=%.3e maxpg=%.3e at %d dt=%.3e nu=%.17g lb=%.17g grad=%.3e mask=%llx\n", ok, alpha, g_t - g, mx, jm, dt[jm], nuv[cur][jm], lb[jm], grad[jm], (unsigned long long)free_mask); }
#endif
            if (!ok) { inner_status = 2; break; }
            cur = nxt; g = g_t;
            err = kkt(Q, nuv[cur], psiv[cur], lb, g, err, grad, pg, &free_mask);
        }
        if (!has_sum) { status = inner_status; break; }
        // exact duality gap at the current prices (trades from the smoothed problem, dual with eps = 0)
        evaluate<LANES, STABLE, STABLE_N, LADDER, CRYPTO, CRYPTO3, BINS, ECLP, PMM>(P, Q, nuv[cur], lognu, eps_t, psiv[cur ^ 1], nullptr, false, true, lane, rec);
        const double g_exact = dual_value(Q, nuv[cur], evaluate<LANES, STABLE, STABLE_N, LADDER, CRYPTO, CRYPTO3, BINS, ECLP, PMM>(P, Q, nuv[cur], lognu, 0.0, grad_t, nullptr, false, false, lane, rec));
        evals += 2;
        double primal = 0.0;
        for (int j = 0; j < n; ++j) primal += Q.c[j] * psiv[cur ^ 1][j];
        const double gap_now = (g_exact - primal) / fmax(fabs(g_exact), TINY);
        if (inner_status == 0 && err <= prm.tol && fabs(gap_now) <= prm.tol) { status = 0; break; }   // the only certified exit
        status = inner_status != 0 ? inner_status : 1;
        // the ramp cannot get narrower and the inner solve failed twice in a row: fp64 resolution of the price
        // ratio / eps bounds the reachable residual, more passes would not help
        if (inner_status != 0 && failed_before && eps_t <= prm.eps_min) break;
        failed_before = inner_status != 0;
        move = 0.0;
        for (int64_t i = Q.p0; i < Q.p1; ++i) {
            if (BINS && P.kind[i] == 10) {                               // tbar <- t; move relative to the domain width
                const int64_t o = P.pool_ptr[i] - Q.off0;
                const double* rp = rec + 4 * (int64_t)P.logrw[P.pool_ptr[i]];
                const double S = rp[4 * ((int64_t)P.logrw[P.pool_ptr[i] + 1] - 1)] - rp[0] / P.gamma[i];
                move = fmax(move, fabs(Q.theta_new[o] - Q.theta_bar[o]) / S);
                Q.theta_bar[o] = Q.theta_new[o];
                continue;
            }
            if (P.kind[i] != 1) continue;
            const int64_t o = P.pool_ptr[i] - Q.off0;
            for (int b = 0; b < 2; ++b) {
                move = fmax(move, fabs(Q.theta_new[o + b] - Q.theta_bar[o + b]) / P.R[P.pool_ptr[i] + b]);
                Q.theta_bar[o + b] = Q.theta_new[o + b];
            }
        }
        eps_t = fmax(prm.eps_min, eps_t * prm.eps_shrink);
    }

    // final read-out: trades and psi from the (smoothed) problem, dual value from the exact one
    const Vec& psi_f = psiv[cur ^ 1];
    evaluate<LANES, STABLE, STABLE_N, LADDER, CRYPTO, CRYPTO3, BINS, ECLP, PMM>(P, Q, nuv[cur], lognu, eps_t, psi_f, nullptr, true, false, lane, rec);
    const double dval = dual_value(Q, nuv[cur], evaluate<LANES, STABLE, STABLE_N, LADDER, CRYPTO, CRYPTO3, BINS, ECLP, PMM>(P, Q, nuv[cur], lognu, 0.0, grad_t, nullptr, false, false, lane, rec));
    evals += 2;
    double primal = 0.0, viol = 0.0;
    for (int j = 0; j < n; ++j) {
        const double s = psi_f[j] + Q.a[j];
        const double v = is_pinned(Q, j) ? 0.0 : (is_eq(Q, j) ? fabs(s) : fmax(-s, 0.0));
        viol += nuv[cur][j] * v;
        primal += Q.c[j] * psi_f[j];
        if (LANES == 1 || lane == 0) { nu_io[j] = nuv[cur][j]; psi_out[j] = psi_f[j]; }
    }
    Stats st;
    st.value = primal; st.dual = dval;
    st.gap = (dval - primal) / fmax(fabs(dval), TINY);
    st.infeas = viol / fmax(fabs(dval), TINY);
    st.err = err; st.iters = iters; st.evals = evals; st.status = status;
    return st;
}

}  // namespace cfmm_small
