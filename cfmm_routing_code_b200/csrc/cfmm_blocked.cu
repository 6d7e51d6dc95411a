// cfmm_blocked.cu -- token-blocked layout for 2-token pools: evaluation, Hessian-vector product and Hessian diagonal
// WITHOUT per-pool atomics, one launch per call.  The layout, the per-pool operator and the tile loop live in
// cfmm_blocked.cuh (shared with the persistent solver, cfmm_persist.cu).
#include <math.h>

#include "cfmm_blocked.cuh"

using namespace cfmm;

namespace {

// Evaluation (MODE 0): persistent CTAs (kCtasPerSm per SM), each walking a contiguous chunk of tiles through the
// TMA-staged pass of cfmm_blocked.cuh.
template <int P, int THREADS, int STAGES, int MODE /*0 eval, 1 hvp, 2 diag*/, bool TRADES, bool HESS>
__global__ void __launch_bounds__(THREADS, kCtasPerSm)
k_blocked(const BlockedArgs A) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t full[STAGES];
    __shared__ double part[THREADS / 32];
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    const long long t_beg = (A.n_tiles * (long long)blockIdx.x) / gridDim.x;
    const long long t_end = (A.n_tiles * (long long)(blockIdx.x + 1)) / gridDim.x;
    double acc = 0.0, acc2 = 0.0;
    unsigned phase = 0;
    blocked_pass<P, THREADS, STAGES, MODE, TRADES, HESS, false, true>(A, smem_raw, full, phase, t_beg, t_end, acc, acc2);
    if (MODE == 0) cta_accumulate<THREADS>(acc, part, A.arb);
}

// ---------------------------------------------------------------------------------------------------------------
// Variant "regs" (configuration 3): the per-pool slabs (R0, R1, 1/gamma, pool words) are read exactly once, so they
// go global -> registers directly (coalesced LDG, prefetched one tile ahead) instead of through shared memory.  Only
// the small per-tile tables (row table, token list, descriptor) ride a 4-deep TMA ring.  That frees ~80 KB of shared
// memory per CTA, which pays for double-buffered nu_local and flows, and those allow ONE barrier per tile: the row
// phase of tile k overlaps the pool phase of tile k+1 in other warps, and nu_local of tile k+1 is fetched from L2
// while tile k's pool phase computes.
// ---------------------------------------------------------------------------------------------------------------
template <int P>
struct __align__(128) TabStage {
    uint32_t rows[BlockedCfg<P>::kRowsMax];
    int32_t tok[BlockedCfg<P>::kTokMax];
    int4 desc;
};

template <int P>
__device__ __forceinline__ void issue_tables(TabStage<P>* st, uint64_t* bar, const BlockedArgs& A, long long tile,
                                             const int4 d) {
    const unsigned rows_b = round16(4u * (unsigned)d.y);
    const unsigned tok_b = round16(4u * (unsigned)d.x);
    mbar_expect_tx(bar, 16u + rows_b + tok_b);
    bulk_g2s(&st->desc, A.desc + tile, 16, bar);
    bulk_g2s(st->rows, A.rows + tile * BlockedCfg<P>::kRowsMax, rows_b, bar);
    bulk_g2s(st->tok, A.tok + tile * BlockedCfg<P>::kTokMax, tok_b, bar);
}

template <int NF>
struct PoolRegs {
    double a[NF];
    uint32_t pw;
};

template <int P, int THREADS, int NF, int NPOOL>
__device__ __forceinline__ void load_pools(PoolRegs<NF> (&r)[NPOOL], const BlockedArgs& A, long long tile, int tid) {
    const long long toff = tile * P;
#pragma unroll
    for (int u = 0; u < NPOOL; ++u) {
        const long long q = toff + tid + u * THREADS;
#pragma unroll
        for (int k = 0; k < NF; ++k) r[u].a[k] = __ldg(A.slab[k] + q);
        r[u].pw = __ldg(A.pw + q);
    }
}

// pull the slabs of `tile` from HBM into L2 ahead of the register loads (one thread, NF + 1 bulk prefetches)
template <int P, int NF>
__device__ __forceinline__ void prefetch_pools_l2(const BlockedArgs& A, long long tile) {
    constexpr int tp = P;
    const long long toff = tile * P;
#pragma unroll
    for (int k = 0; k < NF; ++k) bulk_prefetch_l2(A.slab[k] + toff, tp * 8);
    bulk_prefetch_l2(A.pw + toff, tp * 4);
}

template <int P, int THREADS, int STAGES, int MODE, bool TRADES, bool HESS>
__global__ void __launch_bounds__(THREADS, kCtasPerSm)
k_blocked_regs(const BlockedArgs A) {
    constexpr int NF = (MODE == 0) ? 3 : 1;
    constexpr int NPOOL = P / THREADS;
    constexpr int NPRE = (P + THREADS - 1) / THREADS;
    using St = TabStage<P>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    St* stages = reinterpret_cast<St*>(smem_raw);
    double* nul0 = reinterpret_cast<double*>(smem_raw + (size_t)STAGES * sizeof(St));      // [2][P]  nu_local
    double* g0 = nul0 + 2 * P;                                                              // [2][2P] flows
    __shared__ uint64_t full[STAGES];
    __shared__ double part[THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long t_beg = (A.n_tiles * (long long)blockIdx.x) / gridDim.x;
    const long long t_end = (A.n_tiles * (long long)(blockIdx.x + 1)) / gridDim.x;
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            const long long t = t_beg + s;
            if (t < t_end) issue_tables<P>(&stages[s], &full[s], A, t, __ldg(A.desc + t));
        }
        if (t_beg + 1 < t_end) prefetch_pools_l2<P, NF>(A, t_beg + 1);
        if (t_beg + 2 < t_end) prefetch_pools_l2<P, NF>(A, t_beg + 2);
    }
    PoolRegs<NF> cur[NPOOL], nxt[NPOOL];
    if (t_beg < t_end) load_pools<P, THREADS, NF, NPOOL>(cur, A, t_beg, tid);      // constant tables: before the PDL wait
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    for (int j = blockIdx.x * THREADS + tid; j < A.n_zero; j += gridDim.x * THREADS) A.zero_next[j] = 0.0;
    double acc = 0.0;
    if (t_beg < t_end) {
        mbar_wait(&full[0], 0);
        if (MODE != 2) {
            const int ntok = stages[0].desc.x;
            for (int t = tid; t < ntok; t += THREADS) nul0[t] = __ldg(A.vec + stages[0].tok[t]);
        }
    }
    __syncthreads();
    int stage = 0, pstage = 0, buf = 0;
    unsigned parity = 0;
    for (long long tile = t_beg; tile < t_end; ++tile) {
        St& S = stages[stage];
        const double* nul = nul0 + buf * P;
        double* g = g0 + buf * 2 * P;
        const long long nx = tile + 1;
        int nstage = stage + 1;
        unsigned nparity = parity;
        if (nstage == STAGES) { nstage = 0; nparity ^= 1u; }
        // 1. pool slabs of the next tile -> registers; nu_local of the next tile -> registers (both land while we compute)
        double pre[NPRE];
        int ntok_n = 0;
        if (tid == 0 && tile + 3 < t_end) prefetch_pools_l2<P, NF>(A, tile + 3);      // HBM -> L2, 3 tiles ahead
        if (nx < t_end) {
            load_pools<P, THREADS, NF, NPOOL>(nxt, A, nx, tid);
            mbar_wait(&full[nstage], nparity);
            if (MODE != 2) {
                ntok_n = stages[nstage].desc.x;
#pragma unroll
                for (int k = 0; k < NPRE; ++k) {
                    const int t = tid + k * THREADS;
                    pre[k] = (t < ntok_n) ? __ldg(A.vec + stages[nstage].tok[t]) : 0.0;
                }
            }
        }
        // 2. pool phase of this tile (registers + nu_local) -> flows
        {
            double f0[NPOOL], f1[NPOOL];
#pragma unroll
            for (int u = 0; u < NPOOL; ++u) {
                const uint32_t w = cur[u].pw;
                if (MODE == 0) {
                    EvalOp::apply<TRADES, HESS>(A, tile * P + tid + u * THREADS, cur[u].a[0], cur[u].a[NF > 1 ? 1 : 0],
                                                cur[u].a[NF > 2 ? 2 : 0], nul[pw_lid0(w)], nul[pw_lid1(w)], f0[u], f1[u],
                                                acc);
                } else if (MODE == 1) {
                    f0[u] = cur[u].a[0] * (nul[pw_lid0(w)] - nul[pw_lid1(w)]);
                    f1[u] = -f0[u];
                } else {
                    f0[u] = cur[u].a[0];
                    f1[u] = f0[u];
                }
            }
#pragma unroll
            for (int u = 0; u < NPOOL; ++u) {
                g[tid + u * THREADS] = f0[u];
                g[P + pw_pos1(cur[u].pw)] = f1[u];
            }
        }
        // 3. nu_local of the next tile into the other buffer (read last in the pool phase of tile-1: before barrier-1)
        if (MODE != 2 && nx < t_end) {
            double* nn = nul0 + (buf ^ 1) * P;
#pragma unroll
            for (int k = 0; k < NPRE; ++k) {
                const int t = tid + k * THREADS;
                if (t < ntok_n) nn[t] = pre[k];
            }
        }
        __syncthreads();      // flows of this tile and nu_local of the next are complete; everybody left tile-1's rows
        if (tid == 0 && tile > t_beg) {
            const long long far = tile - 1 + STAGES;
            if (far < t_end) {
                fence_proxy_async();
                issue_tables<P>(&stages[pstage], &full[pstage], A, far, __ldg(A.desc + far));
            }
        }
        // 4. row phase: overlaps the next tile's steps 1-3 in the warps that get there first
        const int nrow = S.desc.y;
        for (int r = tid; r < nrow; r += THREADS) {
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
#pragma unroll
        for (int u = 0; u < NPOOL; ++u) cur[u] = nxt[u];
        pstage = stage; stage = nstage; parity = nparity; buf ^= 1;
    }
    if (MODE == 0) {
        acc = warp_sum(acc);
        if (lane == 0) part[warp] = acc;
        __syncthreads();
        if (tid < 32) {
            double s = (tid < THREADS / 32) ? part[tid] : 0.0;
            s = warp_sum(s);
            if (tid == 0 && s != 0.0) atomicAdd(A.arb, s);
        }
    }
}

// dense assembly (small-n direct solves of mixed problems): H += sum_i A_i h_i [[1,-1],[-1,1]] A_i' straight from the blocked
// layout -- the pool's global tokens are its tile's token list at the local ids of its pool word
__global__ void __launch_bounds__(256)
k_blocked_dense(long long n_pools, int n, const uint32_t* __restrict__ pw, const int32_t* __restrict__ tok,
                const double* __restrict__ hcoef, double* H) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n_pools; q += (long long)gridDim.x * blockDim.x) {
        const double h = hcoef[q];
        if (h != 0.0) {
            const long long tile = q / kTileP;
            const uint32_t w = pw[q];
            const long long a = tok[tile * BlockedCfg<kTileP>::kTokMax + pw_lid0(w)];
            const long long b = tok[tile * BlockedCfg<kTileP>::kTokMax + pw_lid1(w)];
            atomicAdd(H + a * n + a, h); atomicAdd(H + b * n + b, h);
            atomicAdd(H + a * n + b, -h); atomicAdd(H + b * n + a, -h);
        }
    }
}

// ---- launch: evaluation through the TMA-staged pass; Hessian products / diagonal (1 slab, less data per tile) through
// the register-fed single-barrier variant -- each was the faster one for its mode when both were measured.  Both run
// kCtasPerSm CTAs of kTileT threads per SM.
int g_pdl = 1;
int g_row_cap = 32;

template <int MODE, bool TRADES, bool HESS>
int launch_tma(const BlockedArgs& A, cudaStream_t st) {
    constexpr int NF = (MODE == 0) ? 3 : 1;
    auto kern = k_blocked<kTileP, kTileT, kTileStages, MODE, TRADES, HESS>;
    const size_t sm = pass_smem_bytes<kTileP, kTileStages>(NF);
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
        attr = true;
    }
    const long long cap = (long long)kCtasPerSm * num_sms();
    const int grid = (int)(A.n_tiles < cap ? A.n_tiles : cap);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kTileT); cfg.dynamicSmemBytes = sm; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = g_pdl;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, A);
    return check_launch();
}

template <int MODE>
int launch_regs(const BlockedArgs& A, cudaStream_t st) {
    constexpr int P = kTileP, T = kTileT, S = 4;
    auto kern = k_blocked_regs<P, T, S, MODE, false, false>;
    const size_t sm = (size_t)S * sizeof(TabStage<P>) + (size_t)(2 * P + 4 * P) * sizeof(double);
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
        attr = true;
    }
    const long long cap = (long long)kCtasPerSm * num_sms();
    const int grid = (int)(A.n_tiles < cap ? A.n_tiles : cap);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(T); cfg.dynamicSmemBytes = sm; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = g_pdl;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, A);
    return check_launch();
}

}  // namespace

namespace cfmm {

int fill_blocked_args(const cfmm_blocked_pairs* b, BlockedArgs& A) {
    if (!b) return CFMM_E_NULL;
    if (b->pools_per_tile != kTileP) return CFMM_E_KIND;          // layout built for another library version
    if (b->n_tiles < 0 || b->n_pools < 0 || b->n_pools > b->n_tiles * (int64_t)kTileP) return CFMM_E_SIZE;
    if (b->n_tiles > 0 && (!b->pw || !b->rows || !b->tok || !b->desc)) return CFMM_E_NULL;
    A.n_tiles = b->n_tiles;
    A.M = b->n_tiles * (int64_t)kTileP;                            // slab stride (= where slot 1 of delta / lambda starts)
    A.pw = b->pw; A.rows = b->rows; A.tok = b->tok;
    A.desc = reinterpret_cast<const int4*>(b->desc);
    A.fee = b->fee;
    A.zero_next = nullptr; A.n_zero = 0;
    A.slab[0] = A.slab[1] = A.slab[2] = nullptr;
    A.vec = nullptr; A.vec2 = nullptr; A.beta = 0.0;
    A.out = nullptr; A.arb = nullptr; A.delta = A.lambda = A.hcoef = nullptr;
    return CFMM_OK;
}

}  // namespace cfmm

extern "C" {

int cfmm_blocked_layout_info(int32_t* pools_per_tile, int32_t* rows_stride, int32_t* tok_stride, int32_t* row_cap) {
    if (pools_per_tile) *pools_per_tile = kTileP;
    if (rows_stride) *rows_stride = BlockedCfg<kTileP>::kRowsMax;
    if (tok_stride) *tok_stride = BlockedCfg<kTileP>::kTokMax;
    if (row_cap) *row_cap = g_row_cap;
    return CFMM_OK;
}

int32_t cfmm_blocked_fee_words(void) { return fee_words<kTileP>(); }

int cfmm_set_blocked_config(int32_t cfg) {
    if (cfg >= 300) { const int c = cfg - 300; if (c < 8 || c > 32) return CFMM_E_KIND; g_row_cap = c; return CFMM_OK; }
    if (cfg == 200 || cfg == 201) { g_pdl = cfg - 200; return CFMM_OK; }      // programmatic dependent launch off / on
    return CFMM_E_KIND;
}

int cfmm_blocked_eval(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* nu, double* psi, double* arb,
                      const cfmm_eval_out* out, double* zero_next, int64_t n_zero, void* stream) {
    BlockedArgs A;
    int rc = fill_blocked_args(b, A);
    if (rc) return rc;
    if (n_tokens <= 0) return CFMM_E_SIZE;
    if (!nu || !psi || !arb) return CFMM_E_NULL;
    if (b->n_tiles == 0) return CFMM_OK;
    if (!b->r0 || !b->r1 || !b->gamma_inv) return CFMM_E_NULL;
    A.slab[0] = b->r0; A.slab[1] = b->r1; A.slab[2] = b->gamma_inv;
    A.vec = nu; A.out = psi; A.arb = arb;
    A.zero_next = zero_next; A.n_zero = zero_next ? (int)n_zero : 0;
    const bool trades = out && out->delta && out->lambda;
    const bool hess = out && out->hcoef;
    if (trades) { A.delta = out->delta; A.lambda = out->lambda; }
    if (hess) A.hcoef = out->hcoef;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (trades && hess) return launch_tma<0, true, true>(A, st);
    if (trades) return launch_tma<0, true, false>(A, st);
    if (hess) return launch_tma<0, false, true>(A, st);
    return launch_tma<0, false, false>(A, st);
}

int cfmm_blocked_hvp(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* hcoef, const double* vt, double* y,
                     double* zero_next, void* stream) {
    BlockedArgs A;
    int rc = fill_blocked_args(b, A);
    if (rc) return rc;
    if (n_tokens <= 0) return CFMM_E_SIZE;
    if (!hcoef || !vt || !y) return CFMM_E_NULL;
    if (b->n_tiles == 0) return CFMM_OK;
    A.slab[0] = hcoef; A.vec = vt; A.out = y;
    A.zero_next = zero_next; A.n_zero = zero_next ? n_tokens : 0;
    return launch_regs<1>(A, static_cast<cudaStream_t>(stream));
}

int cfmm_blocked_dense(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* hcoef, double* H, void* stream) {
    BlockedArgs A;
    int rc = fill_blocked_args(b, A);
    if (rc) return rc;
    if (n_tokens <= 0) return CFMM_E_SIZE;
    if (!hcoef || !H) return CFMM_E_NULL;
    if (b->n_tiles == 0) return CFMM_OK;
    // (pools of the padded tail carry hcoef = 0: the evaluation writes 0 for them)
    const long long total = b->n_tiles * (long long)kTileP;
    const long long need = (total + 255) / 256, cap = 8LL * num_sms();
    k_blocked_dense<<<(int)(need < cap ? need : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(total, n_tokens, b->pw, b->tok, hcoef, H);
    return check_launch();
}

int cfmm_blocked_diag(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* hcoef, double* diag, void* stream) {
    BlockedArgs A;
    int rc = fill_blocked_args(b, A);
    if (rc) return rc;
    if (n_tokens <= 0) return CFMM_E_SIZE;
    if (!hcoef || !diag) return CFMM_E_NULL;
    if (b->n_tiles == 0) return CFMM_OK;
    A.slab[0] = hcoef; A.out = diag;
    return launch_regs<2>(A, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
