/*
 * cfmm_b200.h -- C ABI of the H100-native (sm_90a) CFMM routing hot path (libcfmm_b200.so).
 *
 * The reference (angeris/cfmm-routing-code) has no FFI: its boundary is the cvxpy call site.
 * Each entry point below names the reference lines it replaces.  All pointers are DEVICE
 * pointers unless the name ends in _host; nothing is allocated inside the *_eval/_hvp calls;
 * every call is asynchronous on `stream` (a cudaStream_t passed as void*), capturable in a CUDA
 * graph, and returns 0 or a negative CFMM_E_* code.  No host threads, no CPU fallback.
 *
 * Pool storage ("bucket"): pools of one kind and one arity k, slot-major SoA, n_pools long, slot j of
 * pool i at [j*stride + i] (per-pool outputs delta/lambda use the same stride):
 *   reserves[k][n_pools]  f64   R_i            arbitrage.py:14-20  (reserves)
 *   tok_idx [k][n_pools]  i32   local_indices  arbitrage.py:6-12   (replaces dense A_i, :42-48)
 *   gamma   [n_pools]     f64   fees[i]        arbitrage.py:22-28
 *   weights [k][n_pools]  f64   normalised p/sum(p) of cp.geo_mean(x, p=...)   arbitrage.py:65
 *   logrw   [k][n_pools]  f64   log(R/w), precomputed once (weighted pools); StableSwap: (A, D) per pool ([2][n_pools])
 *   (StableSwap pools carry their rates in `weights`, bounded products their virtual-reserve offsets, concentrated
 *   pools their records; see CFMM_KIND_CONCENTRATED)
 *   theta_bar[2][n_pools] f64   constant-sum fills (multipliers of the kink), updated by the solver
 */
#ifndef CFMM_B200_H
#define CFMM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    CFMM_KIND_PRODUCT = 0, /* sqrt(x1 x2) >= sqrt(R1 R2)                 arbitrage.py:68-70 */
    CFMM_KIND_SUM = 1,     /* sum(x) >= sum(R), x >= 0                   arbitrage.py:73-74 */
    CFMM_KIND_GEOMEAN = 2, /* prod x^w >= prod R^w                       arbitrage.py:65    */
    CFMM_KIND_BOUNDED_PRODUCT = 3, /* sqrt((x1+o1)(x2+o2)) >= sqrt((R1+o1)(R2+o2)), x >= 0: constant product on virtual
                              reserves, one Uniswap-v3 tick range.  Not in the reference (a new atom for the cons list
                              of arbitrage.py:63-74); arity 2, the two offsets passed in `weights`                */
    CFMM_KIND_STABLESWAP = 4, /* two-coin StableSwap (Curve): 4A(y0+y1) + D >= 4AD + D^3/(4 y0 y1), y_j = r_j x_j, where
                              D = D(R) is the invariant of the current reserves.  Not in the reference; arity 2.
                              weights [2][stride] = the rates (r0, r1) > 0; logrw [2][stride] = per-pool constants:
                              slot 0 = A, slot 1 = D.  A is the whitepaper amplification (A n^n = 4A is the
                              coefficient), which is a contract's A() / n^(n-1) = A() / 2; earlier versions of this
                              header called it Curve's A(), which it is not.  Smooth (no kink): no theta_bar          */
    CFMM_KIND_STABLESWAP_N = 5, /* n-coin StableSwap (Curve), arity n = 2..8 (3pool: n = 3):
                              A n^n sum(y) + D >= A n^n D + D^(n+1) / (n^n prod y), y_j = r_j x_j, D = D(R); at n = 2
                              this is CFMM_KIND_STABLESWAP.  weights [n][stride] = the rates; logrw [2][stride]: slot 0 =
                              A (whitepaper, as kind 4), slot 1 = D.  cfmm_eval_out.hcoef is [n][stride]: the per-slot
                              h_j of the pool's scaled Hessian Hs = C - (C1)(C1)'/(1'C1), C = diag(h^2) - h h'/(1+k)
                              on its k traded slots (hmask), 0 on the others.  Arity 2 is accepted so both kinds can
                              run the same pools; the Python layer sends only n >= 3 here                             */
    CFMM_KIND_CONCENTRATED = 6 /* concentrated liquidity, a whole Uniswap-v3 tick ladder as one pool: sqrt-price bounds
                              b_0 < ... < b_T (price = token 1 per token 0), liquidity L_k >= 0 on [b_k, b_{k+1}), the
                              trading set the Minkowski sum of the intervals' bounded products.  Not in the reference;
                              arity 2.  weights = the records, AoS, 4 f64 per bound {b_k, L_k, Y_k, X_k} with
                              Y_k = sum_{j<k} L_j (b_{j+1} - b_j), X_k = sum_{j>=k} L_j (1/b_j - 1/b_{j+1}), L_T = 0;
                              a pool's T + 1 records are consecutive.  logrw [4][stride]: per pool slot 0 = the current
                              sqrt price s in [b_0, b_T], slot 1 = c (b_c <= s < b_{c+1}, c <= T - 1), slot 2 = the
                              index of its first record in `weights`, slot 3 = T (1 <= T <= 2^20); the integers are
                              exact in f64.  reserves [2][stride] = the real reserves (x, y) at s (not read by the
                              evaluation).  hcoef is per pool, as for every pair kind: the liquidity of the interval the
                              trade ends in (at an exact bound, the one above it; 0 past either end) times
                              sqrt(nu0 nu1 / gamma) / 2.  Smooth between bounds: no theta_bar                        */,
    CFMM_KIND_CRYPTOSWAP = 8  /* two-coin Curve cryptoswap (v2, twocrypto-ng): scaled balances y_j = p_j x_j (p = price
                              scale times precision), K0 = 4 y0 y1 / D^2, K = A K0 G^2 / (G + 1 - K0)^2, and the pool
                              keeps D(y) >= D(R) for the root D of K D (y0 + y1) + y0 y1 = K D^2 + (D/2)^2 with
                              2 sqrt(y0 y1) <= D <= y0 + y1.  Not in the reference; arity 2.  weights [2][stride] = the
                              price scales (p0, p1) > 0 (only their ratio matters); logrw [3][stride]: slot 0 = A (the
                              whitepaper amplification: K -> A K0 as G -> inf, StableSwap's A), slot 1 = G (the curve's
                              gamma, not the fee), slot 2 = D of the current reserves.  hcoef is per pool, as for every
                              pair kind.  Smooth: no theta_bar.  (7 is not a kind: cfmm_arb_eval returns CFMM_E_KIND
                              for it, as for any other unknown kind.)                                                 */,
    CFMM_KIND_CRYPTOSWAP_3 = 9 /* three-coin Curve cryptoswap (tricrypto-ng): y_j = p_j x_j, K0 = 27 y0 y1 y2 / D^3,
                              K = A K0 G^2 / (G + 1 - K0)^2, and the pool keeps D(y) >= D(R) for the root D of
                              K D^2 (y0 + y1 + y2) + y0 y1 y2 = K D^3 + (D/3)^3 with 3 (y0 y1 y2)^(1/3) <= D <=
                              y0 + y1 + y2.  Not in the reference; arity 3 (any other arity: CFMM_E_KIND).
                              weights [3][stride] = the price scales (p0, p1, p2) > 0; logrw [3][stride]: slot 0 = A,
                              slot 1 = G, slot 2 = D of the current reserves, as for kind 8.  hcoef is [3][stride]: the
                              edge weights (w01, w02, w12) of the pool's scaled Hessian block, Hs = sum_{a<b} w_ab
                              (e_a - e_b)(e_a - e_b)' (Hs 1 = 0; one weight may be negative, Hs is PSD), 0 on an edge
                              with an untraded end; hmask = the traded slots (required by the HVP, diagonal and dense
                              kernels).  Smooth: no theta_bar                                                        */,
    CFMM_KIND_BINS = 10       /* price bins (Liquidity Book bins, an order book, limit orders): bins k at prices p_k (token
                              1 per token 0) holding x_k >= 0 of token 0 and y_k >= 0 of token 1, uncrossed (every bin
                              with y > 0 prices at or below every bin with x > 0); bin k accepts (D, L) iff
                              p_k (x_k + gamma D_0 - L_0) + (y_k + gamma D_1 - L_1) >= p_k x_k + y_k and both new
                              holdings are >= 0, and the trading set is the Minkowski sum of the bins'.  Not in the
                              reference; arity 2.  In net-flow form the pool pays out t of token 0 for the least C(t) of
                              token 1, C convex piecewise linear on [-S_bid, S_ask] (asks: slope p_k / gamma over x_k;
                              bids: slope gamma p_k over y_k / (gamma p_k)).  weights = the records, AoS, 4 f64 per
                              breakpoint {T_j, C_j, q_j, bin}, ascending in T, fee-free: record z is (0, 0); above it T
                              is the cumulative x and C the cumulative p x of the asks, below it T is minus the
                              cumulative y / p and C minus the cumulative y of the bids, both accumulated outward from
                              t = 0; q_j = the price of segment (j, j+1) and bin its caller-order bin index (0 and -1 on
                              the last record).  The kernel applies the fee: T / gamma below z, C / gamma above it.  A
                              pool's nb records are consecutive.  logrw [4][stride]: slot 0 = the index of its first
                              record in `weights`, slot 1 = nb (2 .. 2^20 + 2), slot 2 = z (in the pool's records),
                              slot 3 = p_ref > 0 (a fixed price of the pool: the ask price at t = 0, else the bid
                              price).  reserves [2][stride] = (sum x, sum y) (not read by the evaluation).  eps = 0:
                              t maximises r t - C(t), r = nu0 / nu1, a segment filling only when strictly profitable.
                              eps > 0: t maximises r t - C(t) - p_ref (t - tbar)^2 / (2 sigma), sigma = S / eps, S =
                              S_bid + S_ask, with tbar = theta_bar row 0 (row 1 unused; required), and the trader
                              pays the smoothing term.  delta / lambda: the positive and negative parts of the flows
                              (t, -(C(t) + smoothing)).  hcoef per pool, as for every pair kind: (sigma / p_ref) r nu0
                              inside a segment, 0 at a breakpoint or an end.  cfmm_bins_update_multipliers advances
                              tbar.                                                                                    */,
    CFMM_KIND_ECLP = 11       /* elliptic concentrated liquidity (Gyroscope E-CLP): price range 0 < alpha < beta (token 1
                              per token 0), rotation c = cos(phi), s = sin(phi) >= 0, stretch 1 <= lam <= 1e8; with
                              A = [[c/lam, -s/lam], [s, c]] the pool keeps ||A (t - r chi)|| <= r and t >= 0, chi =
                              (f_x(beta), f_y(alpha)), f(p) = M (p, 1)' / sqrt((p, 1) M (p, 1)'), M = (A'A)^-1.  Its
                              balances lie on the arc t(p) = r (chi - f(p)), p in [alpha, beta], where the marginal
                              price is p.  Not in the reference; arity 2 (any other arity: CFMM_E_KIND).
                              weights [7][stride] = (alpha, beta, c, s, lam, r, p): the parameters, the invariant r and
                              the price p of the reserves (pools.eclp_state); reserves [2][stride] = (x, y), paid out
                              exactly at a cap.  logrw is not read.  hcoef is per pool, as for every pair kind:
                              r lam^2 nu1 p*^2 / h(p*)^3 (over gamma when tendering token 1), 0 at a cap.  Smooth: no
                              theta_bar.  The evaluation has no TMA-staged kernel.                                     */,
    CFMM_KIND_PMM = 12        /* DODO proactive market maker: guide price pi > 0 (token 1 per token 0), slippage factor
                              0 < k <= 1, targets B0, Q0 > 0.  Base short (b <= B0): q - Q0 = pi d (1 + k d / b), d =
                              B0 - b, marginal price pi (1 - k + k B0^2 / b^2); quote short (q <= Q0): the mirror (b <->
                              q, B0 <-> Q0, pi -> 1 / pi).  The pool keeps (b, q) on or above this convex curve; its
                              price runs over (0, inf), so it has no cap.  Not in the reference; arity 2 (any other
                              arity: CFMM_E_KIND).  weights [4][stride] = (pi, k, B0, Q0) with the reserves on the curve
                              (the adjusted-target rule, pools.pmm_targets: B < B0 and Q >= Q0, Q < Q0 and B >= B0,
                              or (B, Q) = (B0, Q0)); reserves [2][stride] = (B, Q).  logrw is not read.  hcoef per pool, as for every
                              pair kind: n1 p*^2 b* / (2 (k pi + p* - pi)) for p* >= pi, n1 pi q* / (2 (k p* + pi -
                              p*)) below, over gamma when tendering token 1.  Smooth: no theta_bar.  The evaluation has
                              no TMA-staged kernel.                                                                    */
};

enum {
    CFMM_OK = 0,
    CFMM_E_NULL = -1,      /* required pointer is NULL                                  */
    CFMM_E_KIND = -2,      /* unknown kind, or arity not supported for that kind         */
    CFMM_E_SIZE = -3,      /* negative / overflowing size                                */
    CFMM_E_CUDA = -4,      /* CUDA runtime error (see cfmm_last_cuda_error)              */
    CFMM_E_NODEVICE = -5,  /* no sm_90 device                                            */
    CFMM_E_STATE = -6      /* handle used in the wrong state                             */
};

typedef struct cfmm_bucket {
    int32_t kind;          /* CFMM_KIND_*                                                */
    int32_t arity;         /* tokens per pool: 2 for PRODUCT and SUM, 2..32 for GEOMEAN, 2..8 for STABLESWAP_N */
    int64_t n_pools;
    int64_t stride;        /* elements between consecutive slots (>= n_pools); the TMA-staged path needs
                              stride % 1024 == 0 and 16-byte aligned arrays, otherwise the LDG path runs */
    const double* reserves;
    const int32_t* tok_idx;
    const double* gamma;
    const double* weights;   /* GEOMEAN weights; BOUNDED_PRODUCT offsets; STABLESWAP(_N) rates; CONCENTRATED, BINS records;
                                ECLP (alpha, beta, c, s, lam, r, p); PMM (pi, k, B0, Q0) */
    const double* logrw;     /* GEOMEAN log(R/w); STABLESWAP(_N) (A, D); CONCENTRATED (s, c, first record, T);
                                BINS (first record, nb, z, p_ref) */
    const double* theta_bar; /* SUM and BINS only */
} cfmm_bucket;

/* Optional per-pool outputs of one evaluation (any pointer may be NULL). */
typedef struct cfmm_eval_out {
    double* delta;   /* [arity][n_pools]  = deltas[i].value    arbitrage.py:51, two-asset.py:97  */
    double* lambda;  /* [arity][n_pools]  = lambdas[i].value   arbitrage.py:52, two-asset.py:97  */
    double* hcoef;   /* [n_pools] curvature coefficient of arb_i in log-price coordinates        *
                      * (STABLESWAP_N: [arity][n_pools], one coefficient h_j per slot)          */
    uint32_t* hmask; /* [n_pools] GEOMEAN, STABLESWAP_N: bit j set iff token j is traded        */
} cfmm_eval_out;

/*
 * One dual evaluation over one bucket: for every pool solve the optimal-arbitrage subproblem at
 * prices nu (what `prob.solve()` does for all pools at once, arbitrage.py:81-82, restricted to
 * fixed nu), then ACCUMULATE
 *     psi[j]  += sum_i (A_i (Lambda_i - Delta_i))_j       (psi, arbitrage.py:54)
 *     arb[0]  += sum_i nu_i' (Lambda_i - Delta_i)          (the pool part of the dual value)
 * nu, log_nu: [n_tokens] (log_nu = log(nu), read by GEOMEAN buckets only).  eps: ramp width of the
 * constant-sum proximal smoothing (0 = exact bang-bang LP).  psi/arb must be zeroed by the caller
 * before the first bucket (cfmm_zero does it on the stream).
 */
int cfmm_arb_eval(const cfmm_bucket* bucket, int32_t n_tokens, const double* nu, const double* log_nu,
                  double eps, double* psi, double* arb, const cfmm_eval_out* out, void* stream);

/* y[j] += (Hs vt)_j where Hs = sum_i A_i Hs_i A_i' is the dual Hessian in log-price coordinates
 * (true Hessian = diag(1/nu) Hs diag(1/nu)), vt = v / nu.  Uses hcoef/hmask from cfmm_arb_eval. */
int cfmm_hvp(const cfmm_bucket* bucket, int32_t n_tokens, const double* hcoef, const uint32_t* hmask,
             const double* vt, double* y, void* stream);

/* diag[j] += (Hs)_jj  (Jacobi preconditioner). */
int cfmm_hess_diag(const cfmm_bucket* bucket, int32_t n_tokens, const double* hcoef, const uint32_t* hmask,
                   double* diag, void* stream);

/* H[j*n_tokens + k] += (Hs)_jk, dense row-major n_tokens x n_tokens (small n / direct solves). */
int cfmm_hess_dense(const cfmm_bucket* bucket, int32_t n_tokens, const double* hcoef, const uint32_t* hmask,
                    double* H, void* stream);

/*
 * Token-blocked storage for constant-product pools (the HBM-bound kind).  Built once per problem from
 * local_indices (arbitrage.py:6-12) by the layout builder (pools.py: build_blocked_pairs); pools are
 * reordered into tiles of `pools_per_tile` whose tokens fall into two narrow token blocks.  Per pool 24 B of
 * slabs + one 4 B pool word; per tile a token list, a row table, (ntok, nrow) and an optional fee record.  See
 * csrc/cfmm_blocked.cuh.  Strides of the per-tile tables come from cfmm_blocked_layout_info() and
 * cfmm_blocked_fee_words().
 * The evaluation writes the two flows of pool l of a tile to a per-tile array g[2P]: slot 0 to g[l], slot 1 to g[P + p1];
 * a row sums a contiguous run of g.
 *
 * Fee record of a tile (fee_words = 4 + 32 + P/8 32-bit words, a multiple of 4):
 *   [0]        nfee: 1..16 = the tile's gamma_inv slab takes nfee distinct values ("coded" tile);
 *              0 = more than 16 distinct values: the tile streams its gamma_inv slab and the rest of the record is zero
 *   [1..3]     0
 *   [4..35]    table: 16 f64, the tile's distinct gamma_inv bit patterns in ascending order (padding pools included),
 *              zero past nfee
 *   [36..]     codes: 4 bits per pool, pool l at bits 4 * (l & 7) of word 36 + (l >> 3)
 * On a coded tile table[code(l)] is bit for bit the gamma_inv slab entry of pool l, and the evaluation reads it instead
 * of the slab (7.5 B less HBM traffic per pool).  The gamma_inv slab is still required and must hold every tile's values.
 */
typedef struct cfmm_blocked_pairs {
    int64_t n_pools;          /* real pools (<= n_tiles * pools_per_tile; the rest is padding)          */
    int64_t n_tiles;
    int32_t pools_per_tile;   /* must equal the library's tile size                                      */
    int32_t reserved;
    const double* r0;         /* [n_tiles*P] reserves of slot 0, blocked order        arbitrage.py:14-20 */
    const double* r1;         /* [n_tiles*P] reserves of slot 1                                          */
    const double* gamma_inv;  /* [n_tiles*P] 1 / fees[i]                              arbitrage.py:22-28 */
    const uint32_t* pw;       /* [n_tiles*P] pool word: tile-local token ids lid0 | lid1 << 10 | p1 << 20, each < P;
                                 p1 = rank of the slot-1 half-edge among the tile's, stably sorted by token  */
    const uint32_t* fee;      /* [n_tiles][fee_words] fee records (above), or NULL: every tile streams its gamma_inv slab */
    const uint32_t* rows;     /* [n_tiles][rows_stride] start :16 | length 1..32 :6 | local token :10, longest first */
    const int32_t* tok;       /* [n_tiles][tok_stride] local token id -> global token id                 */
    const int32_t* desc;      /* [n_tiles][4] (ntok, nrow, 0, 0)                                          */
} cfmm_blocked_pairs;

int cfmm_blocked_layout_info(int32_t* pools_per_tile, int32_t* rows_stride, int32_t* tok_stride, int32_t* row_cap);
/* 32-bit words per tile of the fee record (its stride in cfmm_blocked_pairs.fee) */
int32_t cfmm_blocked_fee_words(void);
/* tuning knobs for experiments: 200/201 = programmatic dependent launch off/on; 300+c = row cap c (8..32) of layouts
 * built afterwards.  (The tile size is a compile-time constant of the library, 1024 pools: the fastest of 1024 / 960 /
 * 896 for the evaluation step on an H100.) */
int cfmm_set_blocked_config(int32_t cfg);

/*
 * Native layout builder (csrc/cfmm_layout.cu): the reference's literals -- local_indices as idx [m][2] int32, reserves
 * [m][2] f64, fees as gamma [m] f64 (arbitrage.py:6-28), contiguous on the device -- become the blocked layout in three
 * launches (pool keys + validation, radix sort, one CTA per tile).  `out`: a cfmm_blocked_pairs with n_pools = m,
 * n_tiles = ceil(m / P), pools_per_tile = P whose array members point at caller-allocated device buffers (strides from
 * cfmm_blocked_layout_info; slabs / pw of n_tiles * P entries); all of them are filled, and so are the fee records if
 * `fee` is not NULL.  order [m] uint32 (out):
 * the pool at every blocked position.  status [4] int32 (device, out): [0] tiles that touch more tokens, or need more
 * rows, than a tile may (then the layout is unusable: use a plain bucket), [1] != 0: invalid pools (reserves <= 0 or not finite, fees outside
 * (0, 1], token ids out of range or equal), [2] rows in total.  CFMM_E_SIZE if the sort keys would not fit 32 bits
 * (token_blocks^2 * n_tokens >= 2^32).  work: cfmm_blocked_build_work_bytes(m) bytes.  Asynchronous on `stream`.
 */
int64_t cfmm_blocked_build_work_bytes(int64_t n_pools);
int cfmm_blocked_build(int64_t n_pools, int32_t n_tokens, const int32_t* idx, const double* reserves, const double* gamma,
                       const cfmm_blocked_pairs* out, uint32_t* order, int32_t* status, void* work, int64_t work_bytes,
                       void* stream);

/*
 * In-place update of the reserves and fees of n_upd pools of a built blocked layout (a new block of the same market: the
 * layout depends on the token ids only, reserves and fees are payload).  at [n_upd] uint32: BLOCKED positions
 * (< b->n_pools; the builder's `order` maps position -> pool, the caller inverts it once).  reserves [n_upd][2] f64: new
 * R0, R1 in the pool's own slot order, or NULL; gamma [n_upd] f64: new fees, or NULL.  Positions must be distinct
 * (with repeats one of the values wins; the fee records stay consistent with the slab).
 * All or nothing: one launch checks every entry (position in range, reserves > 0 and finite, fee in (0, 1], the rules
 * of cfmm_blocked_build); only if none is invalid does a second launch write r0 / r1 and gamma_inv = 1.0 / gamma (the
 * builder's IEEE division), and a third rebuild the fee record of every tile whose gamma_inv slab changed (if b->fee is
 * not NULL).  The layout then equals, bit for bit, what cfmm_blocked_build makes of the updated data.
 * status_host [2] int32 (host, out): [0] invalid entries (nothing was written if > 0), [1] fee records rebuilt.
 * work: cfmm_blocked_update_work_bytes(b) bytes of device memory, cleared by every call (no initialisation needed).
 * SYNCHRONOUS on `stream`: the call returns after the stream has drained.  This is deliberate: the standalone blocked
 * kernels issue the bulk copies of their first tiles before they wait for the previous grid (programmatic dependent
 * launch), so an evaluation queued right behind the update kernels could stream the old r0 / r1 / fee record of its
 * first tiles.  Not capturable in a CUDA graph.
 * Plain buckets (cfmm_bucket) need no entry point: their slot-major arrays belong to the caller, who writes them
 * directly (for GEOMEAN pools keep logrw = log(reserves / weights) in step).
 */
int64_t cfmm_blocked_update_work_bytes(const cfmm_blocked_pairs* b);
int cfmm_blocked_update(const cfmm_blocked_pairs* b, int64_t n_upd, const uint32_t* at, const double* reserves,
                        const double* gamma, int32_t* status_host, void* work, int64_t work_bytes, void* stream);

/*
 * New tick ladders for n_chg pools of a CFMM_KIND_CONCENTRATED bucket (mints and burns; T may change), spliced into a
 * second record buffer.  pos [n_chg] int64: the changed BUCKET-LOCAL positions, strictly increasing, < b->n_pools;
 * n_rec [n_chg] int64: their new record counts T + 1 (2 .. 2^20 + 1); records [n_records][4] f64: their new records
 * (the AoS layout of CFMM_KIND_CONCENTRATED), pool after pool in `pos` order; state [n_chg][4] f64: their new
 * (s, c, x, y).  Every pool's records, old (from b->weights) or new, are copied into out_records [out_capacity][4] in
 * bucket order, each pool's first record being the exclusive scan of the record counts; logrw rows 2-3 (first record,
 * T) of every pool and rows 0-1 (s, c) and the reserves of the changed pools are written in place.  b->weights is only
 * read: the caller points the bucket at out_records afterwards (and keeps the old buffer for the next splice), so a
 * CUDA graph captured over the bucket must be captured again.  out_records must not overlap b->weights; b->weights,
 * records and out_records must be 16-byte aligned (CFMM_E_SIZE otherwise).  n_chg = 0 copies the records as they are.
 * All or nothing: if a position is out of range, repeated or out of order, a count out of range, the counts do not sum
 * to n_records or the new total exceeds out_capacity, nothing is written (bucket and out_records).
 * status_host [2] int64 (host, out): [0] invalid entries (nothing was written if > 0), [1] the bucket's new total of
 * records.  work: cfmm_ladder_splice_work_bytes(b->n_pools, n_chg) bytes of device memory (no initialisation needed).
 * CFMM_E_KIND unless kind CONCENTRATED, arity 2.  SYNCHRONOUS on `stream`, like cfmm_blocked_update.
 */
int64_t cfmm_ladder_splice_work_bytes(int64_t n_pools, int64_t n_chg);
int cfmm_ladder_splice(const cfmm_bucket* b, int64_t n_chg, const int64_t* pos, const int64_t* n_rec, const double* records,
                       int64_t n_records, const double* state, double* out_records, int64_t out_capacity,
                       int64_t* status_host, void* work, int64_t work_bytes, void* stream);

/*
 * New bins for n_chg pools of a CFMM_KIND_BINS bucket (a swap that empties the active bin, a deposit or withdrawal, a
 * changed book level, a filled limit order; K may change), spliced into a second record buffer.  The arguments and the
 * all-or-nothing contract of cfmm_ladder_splice, with: n_rec [n_chg] = the new record counts nb (2 .. 2^20 + 2);
 * records = their new records in the AoS layout of CFMM_KIND_BINS; state [n_chg][4] = their new (z, p_ref, sum x,
 * sum y).  logrw rows 0-1 (first record, nb) of every pool and rows 2-3 (z, p_ref) and the reserves (sum x, sum y) of the
 * changed pools are written in place; theta_bar is not touched (a caller that wants a replaced pool to start from a
 * fresh pool's multiplier zeroes its row-0 entry).  work: cfmm_ladder_splice_work_bytes(b->n_pools, n_chg) bytes (the
 * scans are the same).  CFMM_E_KIND unless kind BINS, arity 2.  SYNCHRONOUS on `stream`.
 */
int cfmm_bins_splice(const cfmm_bucket* b, int64_t n_chg, const int64_t* pos, const int64_t* n_rec, const double* records,
                     int64_t n_records, const double* state, double* out_records, int64_t out_capacity,
                     int64_t* status_host, void* work, int64_t work_bytes, void* stream);

/* Same contract as cfmm_arb_eval for a blocked constant-product bucket: psi/arb ACCUMULATE (one red.add per row
 * of <= 32 entries, ~0.35 per pool, instead of 2 per pool).  Per-pool outputs (delta/lambda [2][n_tiles*P], hcoef
 * [n_tiles*P]) are in BLOCKED order.  If zero_next != NULL the launch also clears zero_next[0..n_zero): callers that
 * ping-pong two [psi | arb] buffers never need a separate memset node between evaluations. */
int cfmm_blocked_eval(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* nu, double* psi, double* arb,
                      const cfmm_eval_out* out, double* zero_next, int64_t n_zero, void* stream);
/* y += Hs vt (optionally clearing zero_next[0..n_tokens) for the next call) and diag += diag(Hs), hcoef in blocked order. */
int cfmm_blocked_hvp(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* hcoef, const double* vt, double* y,
                     double* zero_next, void* stream);
int cfmm_blocked_diag(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* hcoef, double* diag, void* stream);
/* H[j*n_tokens + k] += (Hs)_jk of the blocked bucket, dense row-major (the direct Newton solves of small-n mixed problems) */
int cfmm_blocked_dense(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* hcoef, double* H, void* stream);

/*
 * Native outer loop (csrc/cfmm_solver.cu) for problems whose pools are ONE blocked constant-product bucket: the
 * whole of `prob.solve()` (arbitrage.py:81-82) in one call -- projected Newton-CG on the dual, all vectors on the
 * device, host loop in C++.  Utility in "linear + box" form: maximise c'psi s.t. psi_j + a_j >= 0 (eq[j]=0),
 * == 0 (eq[j]=1), unconstrained with nu_j = c_j (pinned[j]=1)  [arbitrage.py:57,77; liquidation.py:57,77-80;
 * two-asset.py:66,86].  c, a, eq, pinned, nu (in: start, out: solution), psi_out: device, n_tokens long.
 * work: device scratch of cfmm_blocked_solve_work_bytes() bytes.  res: host.  Synchronous on `stream`.
 */
typedef struct cfmm_solve_params {
    double tol;        /* stop when sum_free |nu_j (a_j + psi_j)| / |g| <= tol (bounds gap and infeasibility) */
    double nu_floor;   /* positivity floor for free prices                                                    */
    int32_t max_iter;  /* Newton iterations                                                                    */
    int32_t cg_max;    /* PCG iterations per Newton step                                                       */
} cfmm_solve_params;

typedef struct cfmm_solve_result {
    double dual_value, primal_value, gap, primal_infeas, err;
    int32_t iters, evals, hvps, status;   /* status: 0 optimal, 1 max_iter, 2 stalled */
} cfmm_solve_result;

int64_t cfmm_blocked_solve_work_bytes(const cfmm_blocked_pairs* b, int32_t n_tokens);
int cfmm_blocked_solve(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* c, const double* a,
                       const uint8_t* eq, const uint8_t* pinned, double* nu, double* psi_out, void* work,
                       const cfmm_solve_params* prm, cfmm_solve_result* res, void* stream);

/*
 * The same solve with the pools SHARDED over `world` GPUs (one process per GPU, SURVEY 8e): `b` holds this rank's
 * pools, every rank passes the same c / a / eq / pinned / nu and runs the same loop; each evaluation, Hessian-vector
 * product and Hessian diagonal is followed by the LL all-reduce (cfmm_allreduce_ll) of its (n_tokens+1)- or
 * n_tokens-vector over NVLink peer memory, so every rank sees bit-identical reduced vectors, takes identical decisions
 * and ends with identical nu / psi_out / res.  recv_acc_dev / recv_vec_dev: device arrays of `world` pointers to every
 * rank's receive areas ([3 slots][world][n_tokens+1] and [3 slots][world][n_tokens] cells of 16 B, zeroed once at
 * creation; torch symmetric memory: hdl.buffer_ptrs_dev).  seq_acc / seq_vec: last sequence numbers used on the two
 * channels (in), advanced by the reductions of this call (out) -- equal on all ranks.  peer == NULL: one GPU.
 */
typedef struct cfmm_peer_ctx {
    const void* recv_acc_dev;
    const void* recv_vec_dev;
    int32_t rank, world;
    uint64_t seq_acc, seq_vec;
} cfmm_peer_ctx;

int cfmm_blocked_solve_peer(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* c, const double* a,
                            const uint8_t* eq, const uint8_t* pinned, double* nu, double* psi_out, void* work,
                            const cfmm_solve_params* prm, cfmm_solve_result* res, cfmm_peer_ctx* peer, void* stream);

/*
 * Native outer loop (csrc/cfmm_solver.cu) for a market of ANY pool kinds on one GPU: the plain buckets
 * buckets[0..n_buckets) of every CFMM_KIND_* cfmm_arb_eval takes, plus at most one blocked constant-product bucket
 * (blocked, may be NULL).  The method of solver.py step for step: projected Newton on the dual, the Newton systems by
 * Jacobi-PCG on Hessian-vector products or by a dense fp64 Cholesky (Levenberg-Marquardt ladder, active-set
 * look-ahead up to n_tokens = 64), the method of multipliers on constant-sum fills (ramp eps0 -> eps_min by
 * eps_shrink per outer pass, at most max_outer passes), and the final read-back: psi and the trades at the last eps,
 * the dual value exact.  One difference: where no rung of the ladder factors, solver.py takes a least-squares step and
 * this loop the steepest-descent one.  cfmm_blocked_solve is this loop's one-blocked-bucket case.
 * outs[k]: bucket k's per-pool outputs, used as cfmm_arb_eval's `out`.  Every non-empty bucket needs hcoef, and hmask
 * for GEOMEAN, STABLESWAP_N and CRYPTOSWAP_3 (CFMM_E_NULL otherwise); delta / lambda receive the trades of the final
 * read-back (may be NULL, except lambda of a SUM bucket and both of a BINS bucket, whose theta_bar the loop resets and
 * advances: CFMM_E_NULL).
 * blocked_out: the blocked bucket's delta / lambda (blocked order), or NULL; its hcoef lives in `work`.
 * Utility, c / a / eq / pinned / nu / psi_out and res as for cfmm_blocked_solve; `work`:
 * cfmm_market_solve_work_bytes() bytes (same buckets, blocked, n_tokens and linear_solver).  Allocates no device memory;
 * SYNCHRONOUS on `stream`.  CFMM_E_SIZE: n_tokens <= 0, n_buckets < 0, no pools at all, linear_solver outside 0..2,
 * or a dense solve (forced, or chosen by auto) with n_tokens > 4096.  Nothing is launched when a check fails.
 */
typedef struct cfmm_market_params {   /* cfmm_solve_params is not changed (ABI) */
    double tol, nu_floor;
    double eps0, eps_min, eps_shrink;  /* constant-sum ramp continuation (solver.py: 0.1, 1e-4, 0.5)                   */
    int32_t max_iter;                  /* Newton iterations per outer pass                                            */
    int32_t cg_max;                    /* PCG iterations per Newton step                                              */
    int32_t max_outer;                 /* method-of-multipliers passes (60)                                           */
    int32_t linear_solver;             /* 0 auto (dense if n <= 256, or constant-sum pools and n <= 4096), 1 dense, 2 cg */
} cfmm_market_params;

int64_t cfmm_market_solve_work_bytes(const cfmm_bucket* buckets, int32_t n_buckets, const cfmm_blocked_pairs* blocked,
                                     int32_t n_tokens, int32_t linear_solver);
int cfmm_market_solve(const cfmm_bucket* buckets, const cfmm_eval_out* outs, int32_t n_buckets,
                      const cfmm_blocked_pairs* blocked, const cfmm_eval_out* blocked_out, int32_t n_tokens,
                      const double* c, const double* a, const uint8_t* eq, const uint8_t* pinned, double* nu,
                      double* psi_out, void* work, const cfmm_market_params* prm, cfmm_solve_result* res, void* stream);

/* The market loop's dense factorisation on its own: a (n x n, 1 <= n <= 4096, column-major; the lower triangle is
 * read) becomes L (A = L L') in place, with the strictly lower part also mirrored into the upper triangle.  *info
 * (device f64) = 0, or the 1-based index of the first pivot that is not positive and finite (then `a` is garbage).
 * Asynchronous on `stream`. */
int cfmm_dense_cholesky(int32_t n, double* a, double* info, void* stream);

/*
 * The same solve (one GPU or sharded, same arguments and results) as ONE persistent cooperative kernel
 * (csrc/cfmm_persist.cu): every CTA keeps its chunk of pool tiles for the whole solve and runs all evaluation /
 * Hessian-product / diagonal passes on it; every CTA also owns slices of the n_tokens-long vectors and updates them
 * between passes (two grid barriers per pass), and all CTAs run the same scalar state machine on the same reduced
 * sums, so they agree on the next pass without a broadcast; sharded runs all-reduce inside the slice update (LL pushes
 * over NVLink peer memory, every lane its own token).  The host launches once and reads one result struct -- no host
 * round trip per Newton iteration.  status 3 / CFMM_E_STATE: a peer or CTA never showed up within the spin limit (~3 s)
 * and the kernel gave up.  work: cfmm_persist_solve_work_bytes().
 */
int64_t cfmm_persist_solve_work_bytes(const cfmm_blocked_pairs* b, int32_t n_tokens);
int cfmm_set_persist_cooperative(int32_t on);   /* 1 (default) cooperative launch; 0 plain launch (single-GPU loopback tests) */
int cfmm_persist_last_profile(int64_t* out8);   /* development aid: CTA 0's cycle totals of the last persistent solve */
int cfmm_persist_solve(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* c, const double* a,
                       const uint8_t* eq, const uint8_t* pinned, double* nu, double* psi_out, void* work,
                       const cfmm_solve_params* prm, cfmm_solve_result* res, cfmm_peer_ctx* peer, void* stream);

/*
 * Batches of SMALL problems (the reference's own sizes: 5 pools, 3-5 tokens), one problem per thread, the whole
 * prob.solve() (arbitrage.py:81-82, liquidation.py:84-85, two-asset.py:90-91) of every problem in ONE launch.  Replaces
 * the python loop of two-asset.py:40-100 that builds and solves 50 cvxpy problems in turn.  All problems index the same
 * CSR pool arrays (the literals of arbitrage.py:5-28 flattened); problem p uses the pools [pool_range[2p],
 * pool_range[2p+1]) or, with pool_range == NULL, all of them (a sweep over utilities).  Limits: n_tokens <= 64, weighted
 * arity <= 8, constant-sum arity 2; a problem outside them gets status 3 and NaN results.
 */
typedef struct cfmm_csr_pools {
    int32_t n_tokens;
    int64_t n_pools, nnz;
    const int64_t* pool_ptr;   /* [n_pools+1]                                                        */
    const int32_t* tok_idx;    /* [nnz]  local_indices, arbitrage.py:6-12                             */
    const double* reserves;    /* [nnz]  arbitrage.py:14-20                                          */
    const double* weights;     /* [nnz]  normalised like cp.geo_mean(p=...), arbitrage.py:65; 0 on constant-sum pools;
                                         offsets of bounded products; rates of StableSwap pools; concentrated
                                         pools: the sqrt price s at the first slot, c at the second;
                                         cryptoswap pools (kinds 8, 9): p_j / D, the price scales over
                                         the invariant of the reserves (u = weights * reserves in units
                                         of D)                                                          */
    const double* logrw;       /* [nnz]  log(reserves / weights) (unused on constant-sum pools); StableSwap: A at the
                                         pool's first slot, D at its second; concentrated pools: the index of
                                         the first record at the first slot, T at the second; cryptoswap
                                         pools (kinds 8, 9): A at the first slot, the curve gamma G at
                                         the second                                                     */
    const double* gamma;       /* [n_pools] fees, arbitrage.py:22-28                                 */
    const uint8_t* kind;       /* [n_pools] CFMM_KIND_SUM | CFMM_KIND_BOUNDED_PRODUCT | CFMM_KIND_STABLESWAP |
                                            CFMM_KIND_CONCENTRATED | CFMM_KIND_CRYPTOSWAP |
                                            CFMM_KIND_CRYPTOSWAP_3 | CFMM_KIND_BINS | CFMM_KIND_ECLP |
                                            CFMM_KIND_PMM, else weighted geometric mean              */
} cfmm_csr_pools;

typedef struct cfmm_batch {
    int32_t n_problems;
    const int64_t* pool_range; /* nullable [n_problems][2]                                           */
    const double* c;           /* [n_problems][n_tokens] objective on psi (arbitrage.py:31-36,57)    */
    const double* a;           /* [n_problems][n_tokens] endowment (liquidation.py:30-36, two-asset.py:45) */
    const uint8_t* flags;      /* [n_problems][n_tokens] bit0: psi_j + a_j == 0; bit1: psi_j free    */
    double* nu;                /* [n_problems][n_tokens] in: start prices, out: optimal prices       */
    double* psi;               /* [n_problems][n_tokens] out: psi.value (liquidation.py:87)          */
    double* stats;             /* [n_problems][8] out: value (prob.value), dual, gap, infeasibility, kkt err, iters, evals, status */
    double* delta;             /* nullable; out: problem p's Delta at delta[p * trade_stride + csr offset] */
    double* lambda;            /* nullable together with delta                                       */
    int64_t trade_stride;      /* nnz for a shared-pool sweep, 0 for disjoint pool ranges            */
} cfmm_batch;

typedef struct cfmm_batch_params {
    double tol;                /* KKT residual and relative duality gap                              */
    double eps0, eps_min, eps_shrink; /* constant-sum ramp continuation (0.1, 1e-4, 0.5)               */
    double floor_rel;          /* lower bound of free prices relative to max |c| (1e-12)             */
    int32_t max_outer, max_inner;
} cfmm_batch_params;

/* nnz_max: CSR slots of the largest single problem (<= 0: every problem may use all pools->nnz slots) */
int64_t cfmm_batch_solve_work_bytes(const cfmm_csr_pools* pools, int32_t n_problems, int64_t nnz_max);
/* threads per problem: 1 (default; throughput of large batches) or 32 (one warp per problem, the pool loop of every
 * evaluation split over the lanes: latency of small batches / problems with many pools).  Set before sizing the work
 * buffer: it scales with the lane count. */
int cfmm_set_batch_lanes(int32_t lanes);
int cfmm_batch_solve(const cfmm_csr_pools* pools, const cfmm_batch* batch, const cfmm_batch_params* prm, void* work,
                     void* stream);
/* The same solve for pool sets that hold CFMM_KIND_STABLESWAP pools (cfmm_batch_solve gives their problems status 3).
 * A separate kernel instance: the per-pool Newton solve of those pools needs more registers than the other kinds, and
 * cfmm_batch_solve keeps the occupancy it has without them.  Same arguments, limits and workspace. */
int cfmm_batch_solve_stableswap(const cfmm_csr_pools* pools, const cfmm_batch* batch, const cfmm_batch_params* prm,
                                void* work, void* stream);
/* The same solve for pool sets that hold CFMM_KIND_STABLESWAP pools of more than two coins (kind 4 in the CSR arrays,
 * 2..8 coins; the two entry points above give their problems status 3).  A third kernel instance, so the other two keep
 * their registers.  Same arguments, limits and workspace. */
int cfmm_batch_solve_stableswap_n(const cfmm_csr_pools* pools, const cfmm_batch* batch, const cfmm_batch_params* prm,
                                  void* work, void* stream);
/* The same solve for pool sets that hold CFMM_KIND_CONCENTRATED pools, beside every kind cfmm_batch_solve_stableswap_n
 * takes (the three entry points above give their problems status 3).  records: the concentrated pools' records (the
 * AoS layout of CFMM_KIND_CONCENTRATED, device), indexed by the first-record slots of the CSR logrw; CFMM_E_NULL if
 * NULL.  A fourth kernel instance, so the others keep their registers.  Same limits and workspace. */
int cfmm_batch_solve_concentrated(const cfmm_csr_pools* pools, const double* records, const cfmm_batch* batch,
                                  const cfmm_batch_params* prm, void* work, void* stream);
/* The same solve for pool sets that hold CFMM_KIND_CRYPTOSWAP pools (two coins; the CSR layout above: p_j / D in the
 * weights, (A, G) in logrw), beside every kind cfmm_batch_solve_concentrated takes (the four entry points above give
 * their problems status 3).  records: as for cfmm_batch_solve_concentrated, and may be NULL when the pool set has no
 * concentrated pools.  A fifth kernel instance, so the others keep their registers.  Same limits and workspace. */
int cfmm_batch_solve_cryptoswap(const cfmm_csr_pools* pools, const double* records, const cfmm_batch* batch,
                                const cfmm_batch_params* prm, void* work, void* stream);
/* The same solve for pool sets that hold CFMM_KIND_CRYPTOSWAP_3 pools (three coins; p_j / D in the three weights slots,
 * (A, G) in the first two logrw slots), beside every kind cfmm_batch_solve_cryptoswap takes (the five entry points
 * above give their problems status 3).  records: as for cfmm_batch_solve_cryptoswap.  A sixth kernel instance, so the
 * others keep their registers.  Same limits and workspace. */
int cfmm_batch_solve_tricrypto(const cfmm_csr_pools* pools, const double* records, const cfmm_batch* batch,
                               const cfmm_batch_params* prm, void* work, void* stream);
/* The same solve for pool sets that hold CFMM_KIND_BINS pools, beside every kind cfmm_batch_solve_tricrypto takes (the
 * six entry points above give their problems status 3).  In the CSR arrays a bins pool carries z and p_ref in its two
 * weights slots, its first record and nb in its two logrw slots, and (sum x, sum y) in its reserves; records: the
 * concentrated and bins pools' records in one buffer (CFMM_E_NULL if NULL).  The multiplier tbar lives in the pool's
 * first theta_bar slot of the workspace.  A seventh kernel instance, so the others keep their registers.  Same limits
 * and workspace. */
int cfmm_batch_solve_bins(const cfmm_csr_pools* pools, const double* records, const cfmm_batch* batch,
                          const cfmm_batch_params* prm, void* work, void* stream);
/* The same solve for pool sets that hold CFMM_KIND_ECLP pools, beside every kind cfmm_batch_solve_bins takes (the seven
 * entry points above give their problems status 3).  In the CSR arrays an E-CLP pool carries (x, y) in its reserves and,
 * in its first logrw slot, the index r_i of its record in `records` (units of 4 f64, as the first-record slots of
 * concentrated and bins pools): records[4 r_i .. 4 r_i + 7] = {c, s, lam, alpha, beta, r, p, 0}, after the concentrated
 * and bins pools' records in the same buffer (CFMM_E_NULL if NULL).  An eighth kernel instance, so the others keep their
 * registers.  Same limits and workspace. */
int cfmm_batch_solve_eclp(const cfmm_csr_pools* pools, const double* records, const cfmm_batch* batch,
                          const cfmm_batch_params* prm, void* work, void* stream);
/* The same solve for pool sets that hold CFMM_KIND_PMM pools, beside every kind cfmm_batch_solve_eclp takes (the eight
 * entry points above give their problems status 3).  In the CSR arrays a PMM pool carries (B, Q) in its reserves and, in
 * its first logrw slot, the index r_i of its record in `records` (units of 4 f64): records[4 r_i .. 4 r_i + 3] = {pi, k,
 * B0, Q0}, after the E-CLP pools' records in the same buffer (CFMM_E_NULL if NULL).  A ninth kernel instance, so the
 * others keep their registers.  Same limits and workspace. */
int cfmm_batch_solve_pmm(const cfmm_csr_pools* pools, const double* records, const cfmm_batch* batch,
                         const cfmm_batch_params* prm, void* work, void* stream);

/*
 * All-reduce (sum) of n doubles over NVLink peer memory, the ONE collective of a pool-sharded dual evaluation (SURVEY
 * 8e), chained into the launch sequence (programmatic dependent launch) right behind the evaluation kernels.
 * Low-latency ("LL") protocol: every rank PUSHES its n doubles into a receive area of every
 * peer as 16-byte {value, seq} cells (flag travels with the data: one NVLink one-way trip, no hand-shake) and sums what
 * it received, in rank order.  peer_recv_dev: device array of `world` pointers to every rank's receive area
 * [3 slots][world sources][src_stride cells of 16 B]; slot_off_cells = (seq % 3) * world * src_stride.  seq >= 1,
 * strictly increasing, equal on all ranks.  The receive areas must start zeroed.
 */
int cfmm_allreduce_ll(const double* local, const void* peer_recv_dev, int32_t rank, int32_t world, int32_t n,
                      int64_t slot_off_cells, int64_t src_stride_cells, double* out, uint64_t seq, void* stream);

/* SUM buckets: theta_bar <- current fills (= lambda), returns max_i |change|/R in move[0] (device). */
int cfmm_sum_update_multipliers(const cfmm_bucket* bucket, const double* lambda, double* theta_bar_out,
                                double* move, void* stream);

/* BINS buckets: theta_bar row 0 (tbar) <- t = lambda_0 - delta_0, the net token-0 flows of the last trades evaluation
 * (delta, lambda [2][stride]); returns max_i |change| / S_i in move[0] (device; the caller zeroes it first), S_i the
 * width of pool i's net-flow domain at its fee.  CFMM_E_KIND unless kind BINS, arity 2. */
int cfmm_bins_update_multipliers(const cfmm_bucket* bucket, const double* delta, const double* lambda,
                                 double* theta_bar_out, double* move, void* stream);

/* cudaMemsetAsync(ptr, 0, bytes) on the stream -- lets a host language zero psi/arb without torch. */
int cfmm_zero(void* ptr, int64_t bytes, void* stream);

/* Tuning knob for experiments (0 = auto: TMA-staged kernel when the layout allows; 1 = LDG kernel +
 * global red.add; 2 = LDG kernel + shared-memory privatised histogram; 3 = TMA-staged kernel).  Not part of the reference-facing surface. */
int cfmm_set_scatter_mode(int32_t mode);

/* Introspection: number of kernel launches issued by this library since load / last reset. */
int64_t cfmm_launch_count(void);
void cfmm_reset_launch_count(void);
const char* cfmm_last_cuda_error(void);
const char* cfmm_version(void);

#ifdef __cplusplus
}
#endif
#endif /* CFMM_B200_H */
