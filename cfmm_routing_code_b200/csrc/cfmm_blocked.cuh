// cfmm_blocked.cuh -- device code shared by the token-blocked kernels (cfmm_blocked.cu: one launch per dual evaluation /
// Hessian product; cfmm_persist.cu: the whole outer loop in one persistent kernel).
//
// Why a blocked layout: psi = sum_i A_i (L_i - D_i) (arbitrage.py:54) is a scatter of 2 values per pool into n_tokens
// bins.  With red.global.add.f64 per value the L2 atomic units bound the kernel at ~8x the HBM time (measured, round 1).
// The sparsity pattern (local_indices, arbitrage.py:6-12) is static across dual iterations, so it is preprocessed once
// into tiles of P pools whose tokens fall in two narrow token blocks:
//   * a tile touches few distinct tokens: nu is gathered once per tile into shared memory (nu_local) and the pools
//     address it with 10-bit local ids;
//   * each pool thread writes its two net flows to a shared-memory array g[2P] (no atomics): slot 0 to g[l] (pool
//     order: the pools of a tile are sorted by slot-0 token, so a token's slot-0 flows are already neighbours), slot 1 to
//     g[P + p1], where p1 is the pool's rank among the tile's slot-1 half-edges stably sorted by token;
//   * "rows" = (token, <=32 consecutive entries of g) listed by a per-tile table are summed by one thread each, in a
//     fixed order (bit-reproducible), and only the row totals go to global memory: ~0.36 red.add per pool instead of 2.
// One 32-bit word per pool carries both local ids and p1 (lid0 | lid1 << 10 | p1 << 20).
// Fees come from a few tiers, so most tiles see at most 16 distinct 1/gamma values: such a tile carries them in a
// per-tile fee record (table of the distinct values + a 4-bit code per pool, 656 B at P = 1024) and the evaluation
// reads 1/gamma from the table instead of streaming the tile's 1/gamma slab.  Tiles with more distinct values stream
// the slab.
// HBM bytes per pool of the evaluation: 2 x 8 (R0, R1) + 4 (pool word) + ~3 (row/token tables) + 0.64 (fee record), plus
// 8 (1/gamma) on tiles that stream the slab.
// Pool slabs and the per-tile tables are staged through a shared-memory ring by 1-D bulk TMA copies
// (cp.async.bulk + mbarrier).
#pragma once
#include <math.h>

#include "cfmm_dev.cuh"

namespace cfmm {

#ifndef CFMM_TILE_P
#define CFMM_TILE_P 1024             // (build-time knobs for tile-size experiments: -DCFMM_TILE_P=... -DCFMM_CTAS_PER_SM=...)
#endif
#ifndef CFMM_CTAS_PER_SM
#define CFMM_CTAS_PER_SM 2
#endif
constexpr int kTileP = CFMM_TILE_P;  // pools per tile: 1M pools = 977 tiles over the H100's 264 resident CTAs -> 4 x 1024 on
                                     // the critical path (896: 1117 tiles -> 5 x 896); the evaluation step measured fastest
                                     // of 1024 / 960 / 896 on an H100
constexpr int kTileT = kTileP / 2;   // threads per CTA: two pools per thread
constexpr int kTileStages = 2;       // TMA ring depth
constexpr int kCtasPerSm = CFMM_CTAS_PER_SM;
static_assert(kTileP % 64 == 0 && kTileP <= 1024, "tile size: whole warps of two-pool threads, 10-bit fields of the pool word");

// pool word: local token id of slot 0 (10 bits) | of slot 1 (10 bits) << 10 | p1 (10 bits) << 20, where p1 = position of
// the slot-1 flow in the second half of the tile's flow array g (the slot-0 flow of pool l goes to g[l])
__device__ __forceinline__ int pw_lid0(uint32_t w) { return (int)(w & 0x3ffu); }
__device__ __forceinline__ int pw_lid1(uint32_t w) { return (int)((w >> 10) & 0x3ffu); }
__device__ __forceinline__ int pw_pos1(uint32_t w) { return (int)(w >> 20); }

template <int P>
struct BlockedCfg {
    // the layout builder guarantees <= P distinct tokens and <= kRowsMax rows per tile (tiles that would exceed
    // either go to the plain bucket)
    static constexpr int kTokMax = P;
    static constexpr int kRowCapMin = 8;                     // smallest row cap the tables are sized for
    static constexpr int kRowsMax = P + 2 * P / kRowCapMin + 8;
};

// fee record of a tile (include/cfmm_b200.h): header (nfee, 0, 0, 0) | table of kFeeMax f64 | codes, 4 bits per pool.
// nfee == 0: the tile has more than kFeeMax distinct 1/gamma values and streams its slab.
constexpr int kFeeMax = 16;
constexpr int kFeeTab = 4;                         // word of the table
constexpr int kFeeCode = kFeeTab + 2 * kFeeMax;    // word of the first code
template <int P>
__host__ __device__ constexpr int fee_words() { return kFeeCode + P / 8; }
static_assert(fee_words<kTileP>() % 4 == 0, "fee record: whole 16-byte units (one bulk copy)");
__device__ __forceinline__ unsigned fee_code(const uint32_t* codes, int l) { return (codes[l >> 3] >> (4 * (l & 7))) & 15u; }

// one ring stage: NF per-pool f64 slabs + pool words + row table + token list + fee record (NF == 3)
template <int P, int NF>
struct __align__(128) Stage {
    double a[NF][P];                              // a[2] (1/gamma) is not filled on a coded tile
    uint32_t pw[P];                               // lid0 | lid1 << 10 | p1 << 20
    uint32_t rows[BlockedCfg<P>::kRowsMax];       // start :16 | length (1..32) :6 | local token :10, longest first
    int32_t tok[BlockedCfg<P>::kTokMax];          // local token id -> global token id
    int4 desc;                                    // (ntok, nrow, 0, 0) of the tile in this stage
    uint32_t fee[fee_words<P>()];                 // fee record of the tile (evaluation with a fee record only)
};

struct BlockedArgs {
    long long n_tiles;
    long long M;                  // n_tiles * P (padded pool count = slab stride)
    const double* slab[3];        // NF slabs, each [M]
    const uint32_t* pw;           // [M] pool words
    const uint32_t* rows;         // [n_tiles][kRowsMax]
    const int32_t* tok;           // [n_tiles][kTokMax]
    const int4* desc;             // [n_tiles] (ntok, nrow, 0, 0)
    const uint32_t* fee;          // [n_tiles][fee_words] fee records, or null (every tile streams its 1/gamma slab)
    const double* vec;            // nu (eval) or vt (hvp); unused for diag
    const double* vec2;           // hvp inside the persistent solver: the direction is vec2 + beta * vec (PCG's p = z + beta p, formed on the fly)
    double beta;
    double* out;                  // psi / y / diag (+= via one red.add per row)
    double* zero_next;            // optional: buffer of n_zero doubles this launch clears for the NEXT call
    int n_zero;
    double* arb;                  // eval only
    double* delta;                // eval, optional: [2][M] blocked order
    double* lambda;
    double* hcoef;                // eval, optional: [M]
};

__device__ __forceinline__ unsigned round16(unsigned bytes) { return (bytes + 15u) & ~15u; }

// nfee of a tile's fee record (0 = no record or a tile that streams its 1/gamma slab); read by the producer thread
template <int P, int NF>
__device__ __forceinline__ unsigned tile_nfee(const BlockedArgs& A, long long tile) {
    return (NF == 3 && A.fee) ? __ldg(A.fee + tile * fee_words<P>()) : 0u;
}

// d = the tile's descriptor, nfee = tile_nfee of the tile.  The bytes the barrier expects and the copies issued follow
// from the same (nslab, rec): a mismatch would leave the barrier waiting forever.
template <int P, int NF>
__device__ __forceinline__ void issue_tile(Stage<P, NF>* st, uint64_t* bar, const BlockedArgs& A, long long tile,
                                           const int4 d, const unsigned nfee) {
    const bool rec = NF == 3 && A.fee != nullptr;                   // the fee record rides along
    const int nslab = rec && nfee != 0 ? NF - 1 : NF;               // coded tile: its 1/gamma slab (the last) stays behind
    const unsigned fee_b = rec ? 4u * fee_words<P>() : 0u;
    const unsigned rows_b = round16(4u * (unsigned)d.y);
    const unsigned tok_b = round16(4u * (unsigned)d.x);
    const long long off = tile * P;
    mbar_expect_tx(bar, (unsigned)(nslab * P * 8 + P * 4 + 16) + rows_b + tok_b + fee_b);
    bulk_g2s(&st->desc, A.desc + tile, 16, bar);
#pragma unroll
    for (int k = 0; k < NF; ++k)
        if (k < nslab) bulk_g2s(st->a[k], A.slab[k] + off, P * 8, bar);
    bulk_g2s(st->pw, A.pw + off, P * 4, bar);
    bulk_g2s(st->rows, A.rows + tile * BlockedCfg<P>::kRowsMax, rows_b, bar);
    bulk_g2s(st->tok, A.tok + tile * BlockedCfg<P>::kTokMax, tok_b, bar);
    if (rec) bulk_g2s(st->fee, A.fee + tile * fee_words<P>(), fee_b, bar);
}

// ---- per-pool operator: the two net flows (f0, f1) of a constant-product pool (arbitrage.py:68-70) ----------
// With gi = 1/gamma, p_j = nu_j R_j and v = rsqrt(p0 p1 gi):  a = p0 v, b = p1 v  (a b gi = 1).  The KKT solution is
//   b > 1 : tender token 0:  x0 = R0 b,       x1 = R1 a gi   =>  f0 = -R0 (b-1) gi,  f1 = R1 (1 - a gi)
//   a > 1 : tender token 1:  x1 = R1 a,       x0 = R0 b gi   =>  f1 = -R1 (a-1) gi,  f0 = R0 (1 - b gi)
//   else  : no-trade cone (then b gi >= 1 and a gi >= 1, so the "receive" expressions clamp to 0 by themselves).
// Written with selects only (no divergent branch on the direction).
// h = sqrt(p0 p1 / gamma)/2 = w v / 2 on trading pools (Hs_i = h [[1,-1],[-1,1]] in log-price coordinates).
// max(x, 0) on the bit pattern: a negative double has its sign bit set, so masking with ~(hi >> 31) zeroes it (3 integer
// instructions instead of the NaN-propagating fp64 max sequence)
__device__ __forceinline__ double clamp0(double x) {
    const int hi = __double2hiint(x);
    const int m = ~(hi >> 31);
    return __hiloint2double(hi & m, __double2loint(x) & m);
}

struct EvalOp {
    template <bool TRADES, bool HESS>
    __device__ __forceinline__ static void apply(const BlockedArgs& A, long long q, double R0, double R1, double gi,
                                                 double n0, double n1, double& f0, double& f1, double& acc) {
        const double p0 = n0 * R0, p1 = n1 * R1;
        const double w = p0 * p1 * gi;
        const double v = rsqrt(w);
        const double a = p0 * v, b = p1 * v;
        const double ob = 1.0 - b, oa = 1.0 - a;
        const double r0 = fma(-b, gi, 1.0), r1 = fma(-a, gi, 1.0);          // 1 - b gi, 1 - a gi  (received share)
        const double x0 = (ob < 0.0) ? ob * gi : clamp0(r0);
        const double x1 = (oa < 0.0) ? oa * gi : clamp0(r1);
        f0 = R0 * x0;
        f1 = R1 * x1;
        acc = fma(n0, f0, fma(n1, f1, acc));
        if (TRADES) {
            A.delta[q] = f0 < 0.0 ? -f0 : 0.0; A.delta[A.M + q] = f1 < 0.0 ? -f1 : 0.0;
            A.lambda[q] = f0 > 0.0 ? f0 : 0.0; A.lambda[A.M + q] = f1 > 0.0 ? f1 : 0.0;
        }
        if (HESS) A.hcoef[q] = (x0 != 0.0 || x1 != 0.0) ? 0.5 * w * v : 0.0;
    }
};

// row word: start (16 bits) | length (6 bits, 1..32) | local token (10 bits).  Rows of a tile are sorted by
// decreasing length by the builder, so the 32 rows of a warp have (nearly) equal trip counts.
__device__ __forceinline__ int row_start(uint32_t r) { return (int)(r & 0xffffu); }
__device__ __forceinline__ int row_len(uint32_t r) { return (int)((r >> 16) & 0x3fu); }
__device__ __forceinline__ int row_tok(uint32_t r) { return (int)(r >> 22); }

// gather of the price / direction vector: through the read-only path (ld.global.nc) in a kernel of its own; inside the
// persistent solver the vector is rewritten between passes of the same launch, so it is a plain (coherent) load there --
// the grid barrier between the writer and this pass (fence + atomic / ld.acquire) makes the new values visible
template <bool COHERENT>
__device__ __forceinline__ double load_vec(const double* p) { return COHERENT ? *p : __ldg(p); }
// MODE 1 inside the persistent solver (COHERENT): the gathered entry is vec2[t] + beta * vec[t]
template <int MODE, bool COHERENT>
__device__ __forceinline__ double gather_vec(const BlockedArgs& A, int t) {
    if (MODE == 1 && COHERENT) return fma(A.beta, A.vec[t], A.vec2[t]);
    return load_vec<COHERENT>(A.vec + t);
}

// Shared memory of one CTA of the TMA-staged pass: STAGES ring stages, nu_local [P], flows [2P]
template <int P, int STAGES>
constexpr size_t pass_smem_bytes(int nf) {
    return (size_t)STAGES * (nf == 3 ? sizeof(Stage<P, 3>) : sizeof(Stage<P, 1>)) + (size_t)(3 * P) * sizeof(double);
}

// One pass over this CTA's chunk of tiles [t_beg, t_end): MODE 0 evaluation (psi += flows, acc += nu'flows),
// 1 Hessian-vector product (y += Hs vt), 2 Hessian diagonal.  `full` = STAGES initialised mbarriers, `phase` = their
// current parities as a bit mask (carried across passes by the persistent kernel; 0 in a fresh launch).
// acc: eval: sum of nu'flows (= arb); persistent hvp: p'Hp, with acc2 = p'diag(H)p.
// PDL: the standalone kernels wait for the previous grid only after their first tiles are in flight.
template <int P, int THREADS, int STAGES, int MODE, bool TRADES, bool HESS, bool COHERENT, bool PDL>
__device__ __forceinline__ void blocked_pass(const BlockedArgs& A, unsigned char* smem_raw, uint64_t* full, unsigned& phase,
                                             long long t_beg, long long t_end, double& acc, double& acc2) {
    constexpr int NF = (MODE == 0) ? 3 : 1;
    using St = Stage<P, NF>;
    St* stages = reinterpret_cast<St*>(smem_raw);
    double* nul = reinterpret_cast<double*>(smem_raw + (size_t)STAGES * sizeof(St));      // [P]    nu_local
    double* g = nul + P;                                                                   // [2P] flows: slot 0 | slot 1
    const int tid = threadIdx.x;
    // Each CTA walks a CONTIGUOUS chunk of tiles.  Tiles are sorted by (token block of slot 0, of slot 1), so at any
    // moment the resident CTAs work on different token blocks and their red.adds hit different addresses (a
    // grid-strided walk would have all CTAs hammer the same ~130 tokens at once).
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            const long long t = t_beg + s;
            if (t < t_end) issue_tile<P, NF>(&stages[s], &full[s], A, t, __ldg(A.desc + t), tile_nfee<P, NF>(A, t));
        }
    }
    if (PDL) {
        // Programmatic dependent launch: everything above touches only this launch's own shared memory and the
        // constant pool tables, so it may run while the previous kernel on the stream is still draining.  From here
        // on we read vec / write out, zero_next -- wait for the previous grid, then let the next one start its ramp.
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }
    // clear the buffer the NEXT call accumulates into (nobody touches it during this launch)
    for (int j = blockIdx.x * THREADS + tid; j < A.n_zero; j += gridDim.x * THREADS) A.zero_next[j] = 0.0;
    int stage = 0;
    constexpr int NPRE = (P + THREADS - 1) / THREADS;       // nu_local values each thread prefetches
    // prologue: nu_local of this CTA's first tile
    if (t_beg < t_end) {
        mbar_wait(&full[0], phase & 1u);
        if (MODE != 2) {
            const int ntok = stages[0].desc.x;
            for (int t = tid; t < ntok; t += THREADS) nul[t] = gather_vec<MODE, COHERENT>(A, stages[0].tok[t]);
        }
    }
    __syncthreads();
    for (long long tile = t_beg; tile < t_end; ++tile) {
        St& S = stages[stage];                          // full (waited for when its nu_local was fetched)
        phase ^= 1u << stage;                           // the wait on this stage is behind us: its next fill has the other parity
        const int4 d = S.desc;                          // (ntok, nrow, 0, 0)
        // the producer thread fetches the descriptor of the tile it will issue at the end of this iteration
        const long long far = tile + STAGES;
        int4 dfar = make_int4(0, 0, 0, 0);
        unsigned nfar = 0;
        if (tid == 0 && far < t_end) { dfar = __ldg(A.desc + far); nfar = tile_nfee<P, NF>(A, far); }
        // ---- pool phase: per-pool flows, slot 0 to g[l], slot 1 to g[P + p1].  All loads and math of the thread's NPOOL
        // pools first, the shared-memory stores afterwards, so the independent chains overlap in the pipeline.
        // 1/gamma: from the tile's fee table on a coded tile (the same bits as its slab entry), else from the slab.
        {
            const bool coded = NF == 3 && A.fee != nullptr && S.fee[0] != 0u;        // uniform over the tile
            const double* ftab = reinterpret_cast<const double*>(S.fee + kFeeTab);
            constexpr int NPOOL = P / THREADS;
            double f0[NPOOL], f1[NPOOL];
            uint32_t ws[NPOOL];
#pragma unroll
            for (int u = 0; u < NPOOL; ++u) {
                const int l = tid + u * THREADS;
                const uint32_t w = S.pw[l];
                ws[u] = w;
                if (MODE == 0) {
                    const double gi = coded ? ftab[fee_code(S.fee + kFeeCode, l)] : S.a[NF > 2 ? 2 : 0][l];
                    EvalOp::apply<TRADES, HESS>(A, tile * P + l, S.a[0][l], S.a[NF > 1 ? 1 : 0][l], gi,
                                                nul[pw_lid0(w)], nul[pw_lid1(w)], f0[u], f1[u], acc);
                } else if (MODE == 1) {
                    const double pa = nul[pw_lid0(w)], pb = nul[pw_lid1(w)], h = S.a[0][l];
                    f0[u] = h * (pa - pb);
                    f1[u] = -f0[u];
                    if (COHERENT) {                    // the persistent solver's PCG: p'Hp and p'diag(H)p come with the pass
                        acc = fma(f0[u], pa - pb, acc);
                        acc2 = fma(h, fma(pa, pa, pb * pb), acc2);
                    }
                } else {
                    f0[u] = S.a[0][l];
                    f1[u] = f0[u];
                }
            }
#pragma unroll
            for (int u = 0; u < NPOOL; ++u) {
                g[tid + u * THREADS] = f0[u];
                g[P + pw_pos1(ws[u])] = f1[u];
            }
        }
        __syncthreads();                 // g complete; nu_local of this tile is dead from here on
        // ---- prefetch nu_local of the NEXT tile into registers: the L2 latency hides behind the row phase
        const long long nxt = tile + 1;
        const int nstage = (stage + 1 == STAGES) ? 0 : stage + 1;
        double pre[NPRE];
        int ntok_n = 0;
        if (nxt < t_end) {
            mbar_wait(&full[nstage], (phase >> nstage) & 1u);     // also makes the next iteration's stage reads safe
            if (MODE != 2) {
                ntok_n = stages[nstage].desc.x;
#pragma unroll
                for (int k = 0; k < NPRE; ++k) {
                    const int t = tid + k * THREADS;
                    pre[k] = (t < ntok_n) ? gather_vec<MODE, COHERENT>(A, stages[nstage].tok[t]) : 0.0;
                }
            }
        }
        // ---- row phase: one thread per row; a row is a CONTIGUOUS run of g (flows of one token in one half), rows
        // are sorted by length so a warp's 32 rows have (nearly) equal trip counts.
        // Fixed summation order; one red.add per row.
        for (int r = tid; r < d.y; r += THREADS) {
            const uint32_t rw = S.rows[r];
            const double* q = g + row_start(rw);
            const int len = row_len(rw);
            double s0 = 0.0, s1 = 0.0;
            int k = 0;
#pragma unroll 1
            for (; k + 4 <= len; k += 4) { s0 += q[k] + q[k + 2]; s1 += q[k + 1] + q[k + 3]; }
            if (k + 2 <= len) { s0 += q[k]; s1 += q[k + 1]; k += 2; }
            if (k < len) s0 += q[k];
            const double s = s0 + s1;
            if (s != 0.0) atomicAdd(A.out + S.tok[row_tok(rw)], s);
        }
        if (MODE != 2 && nxt < t_end) {
#pragma unroll
            for (int k = 0; k < NPRE; ++k) {
                const int t = tid + k * THREADS;
                if (t < ntok_n) nul[t] = pre[k];
            }
        }
        __syncthreads();                 // stage and g are free again; nu_local of the next tile is in place
        if (tid == 0 && far < t_end) {
            fence_proxy_async();
            issue_tile<P, NF>(&S, &full[stage], A, far, dfar, nfar);
        }
        stage = nstage;
    }
}

// sum of `acc` over the CTA, added to *target by one thread (part: THREADS / 32 doubles of shared memory)
template <int THREADS>
__device__ __forceinline__ void cta_accumulate(double acc, double* part, double* target) {
    const int tid = threadIdx.x;
    acc = warp_sum(acc);
    if ((tid & 31) == 0) part[tid >> 5] = acc;
    __syncthreads();
    if (tid < 32) {
        double s = (tid < THREADS / 32) ? part[tid] : 0.0;
        s = warp_sum(s);
        if (tid == 0 && s != 0.0) atomicAdd(target, s);
    }
}

// validated view of the caller's cfmm_blocked_pairs (cfmm_blocked.cu)
int fill_blocked_args(const cfmm_blocked_pairs* b, BlockedArgs& A);

}  // namespace cfmm
