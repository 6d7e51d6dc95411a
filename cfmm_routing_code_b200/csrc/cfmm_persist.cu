// cfmm_persist.cu -- the WHOLE outer loop of a constant-product routing problem in ONE persistent kernel.
//
// What replaces `prob.solve()` (arbitrage.py:81-82) for problems made of one token-blocked constant-product bucket
// (arbitrage.py:68-70): the same projected Newton / Jacobi-PCG / Armijo method as cfmm_solver.cu and solver.py, but the
// host never sees an intermediate scalar.  One cooperative launch of kCtasPerSm CTAs per SM:
//   * every CTA owns a fixed contiguous chunk of tiles and runs the pool passes (evaluation, Hessian-vector product,
//     Hessian diagonal: blocked_pass of cfmm_blocked.cuh) on it, for every pass of the solve;
//   * every CTA also owns slices of the n tokens and does the n_token-sized vector algebra (KKT residual, free set, PCG
//     recurrences, line search) for them -- one token per lane, no loop over n anywhere;
//   * two grid barriers per pass (after the pass; after the slice updates), then every CTA adds the slice partial sums
//     in slice order and runs the same scalar state machine: all CTAs agree on the next pass without any broadcast;
//   * pool-sharded over several GPUs (SURVEY 8e): the all-reduce of a pass's vector happens inside the slice update --
//     each lane pushes its token's partial to the peers (LL protocol of cfmm_allreduce.cu: 16-byte {value, seq} cells
//     over NVLink peer memory) and sums what they pushed in rank order, so every rank computes bit-identical scalars and
//     takes the same decisions.
// The host launches once and reads one result struct.  (A variant in which CTA 0 alone did the vector algebra and
// broadcast a command word was measured at 4.0 ms per 1M-pool solve against 2.7 ms for this one and removed.)
#include <math.h>
#include <string.h>

#include "cfmm_blocked.cuh"

using namespace cfmm;

namespace {

constexpr int PT = kTileT;                       // threads per CTA
constexpr unsigned long long kSpinLimit = 6000000000ull;     // ~3 s of SM clocks: a lost peer / launch must not hang the GPU


struct DevResult {                               // written by CTA 0, copied to the host after the kernel
    double dual_value, primal_value, gap, primal_infeas, err;
    int iters, evals, hvps, status;              // status 0 optimal, 1 max_iter, 2 stalled, 3 aborted (spin limit)
    unsigned long long seq_acc, seq_vec;
    long long prof[16];                          // CTA 0's clock64 totals: pass eval/hvp/diag, wait for the grid, vector algebra eval/hvp/diag, (unused)
};

struct PersistArgs {
    BlockedArgs B;                               // layout + slabs; vec / out / hcoef are set per pass on the device
    int n;
    const double *c, *a;
    const unsigned char *eq, *fixed;
    double* nu[2];                               // current / trial prices (nu[0] = the caller's buffer)
    double* acc[2];                              // [psi | arb] of nu[0] / nu[1]
    double *y, *diag, *hcoef;
    double *lb, *grad[2], *fr[2], *pg[2], *dt, *x, *r, *z, *p, *minv;
    unsigned* ctl;                               // 512 B, zeroed by the host: [0] grid-barrier counter | [32] abort flag (own 128-B lines)
    double tol, nu_floor;
    int max_iter, cg_max;
    LLCell* const* recv_acc;                     // pool-sharded: receive areas (device array of `world` pointers) or null
    LLCell* const* recv_vec;
    int rank, world;
    unsigned long long seq_acc, seq_vec;
    double* nu_out;                              // == nu[0]
    double* psi_out;
    DevResult* res;
};

__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

struct Kkt { double err, g, primal, infeas, lin; };

template <int MODE>
__device__ __forceinline__ void run_pass(const PersistArgs& S, const double* vec, double* out, unsigned char* smem_raw,
                                         uint64_t* full, unsigned& phase, long long t_beg, long long t_end, double* part,
                                         double beta) {
    BlockedArgs A = S.B;
    A.vec = vec; A.out = out; A.zero_next = nullptr; A.n_zero = 0;
    asm volatile("fence.proxy.async;" ::: "memory");         // hcoef: written through the generic proxy, read by TMA (async proxy)
    if (MODE == 0) { A.arb = out + S.n; A.hcoef = S.hcoef; }
    else A.slab[0] = S.hcoef;
    if (MODE == 1) { A.vec2 = S.z; A.beta = beta; }           // direction = z + beta p, formed by the gather
    double acc = 0.0, acc2 = 0.0;
    blocked_pass<kTileP, PT, kTileStages, MODE, false, MODE == 0, true, false>(A, smem_raw, full, phase, t_beg, t_end, acc, acc2);
    if (MODE == 0) {
        cta_accumulate<PT>(acc, part, A.arb);
        asm volatile("fence.proxy.async;" ::: "memory");     // hcoef written here (generic proxy) is read by TMA in later passes
    }
    if (MODE == 1) {                                         // p'Hp and p'diag(H)p ride behind the vector: y[n], y[n+1]
        cta_accumulate<PT>(acc, part, out + S.n);
        __syncthreads();
        cta_accumulate<PT>(acc2, part, out + S.n + 1);
    }
}

// =====================================================================================================================
// Distributed variant: NO boss.  The n tokens are cut into `nsl` slices (a function of n only, so the same on every rank
// of a sharded solve); slice s belongs to CTA s mod G and is worked by one warp, one token per lane -- every load of a
// slice phase is issued at once (one L2 round trip), nothing loops over n.  After a pass:
//     grid barrier A  ->  slice phase: [NVLink LL exchange of the slice] + element-wise update + slice partial sums
//     grid barrier B  ->  decide phase: every CTA adds the slice partials in slice order (same bits everywhere, on every
//                         rank) and runs the same scalar state machine, so all CTAs (and all ranks) agree on the next
//                         pass without a command broadcast.
// A sharded solve all-reduces inside the slice phase: each lane pushes ITS token to the peers and sums what they pushed
// (rank order) -- the exchange is spread over all CTAs instead of serialised in one.
// =====================================================================================================================
// Loads of data another CTA wrote before the last grid barrier: PLAIN loads.  The barrier is fence + bar.sync + atomic on
// the writer's side and ld.acquire.gpu + bar.sync on the reader's, which orders weak accesses across it (and the acquire
// refreshes this SM's L1); ld.global.cg would also be correct, but plain loads pipeline
// better.
__device__ __forceinline__ double ldw(const double* p) { return *p; }

constexpr int kSliceMax = 256;                   // slices (>= 1): min(256, ceil(n / 16))
constexpr int kQ = 10;                           // partial quantities per phase

enum { PH_KKT = 1, PH_DIAG = 2, PH_HVP = 3, PH_STEP = 4, PH_DONE = 5 };

struct DistArgs {
    PersistArgs P;
    double* accr[2];                             // all-reduced psi of nu[0] / nu[1] (what psi_out returns)
    double* y2[2];                               // Hs p ping-pong, [n + 2] each (+ p'Hp, p'diag(H)p)
    double* partial;                             // [2 parities][kQ][kSliceMax]
    int nsl;
};

struct DState {                                  // replicated in every CTA's shared memory; thread 0 updates it
    int phase, set, cur, iters, evals, hvps, status, cg_k, ls, yb, first_step, dir_ok, aborted, parity;
    double err, g0, rz, r0n, eta, alpha, lin1, beta, al, imx, thr, dsc;
    int flat;
    Kkt kc;
    unsigned long long seq_acc, seq_vec;
    unsigned bar;                                // grid barriers passed so far
    long long prof[16];
};

__device__ __forceinline__ void grid_barrier(unsigned* ctl, DState* ds) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned target = (++ds->bar) * gridDim.x;
        atomicAdd(ctl, 1u);
        const long long t0 = clock64();
        while (ld_acquire_gpu(ctl) < target) {
            if (ld_acquire_gpu(ctl + 32) != 0u) { ds->aborted = 1; break; }
            if ((unsigned long long)(clock64() - t0) > kSpinLimit) { ctl[32] = 1u; ds->aborted = 1; break; }
        }
    }
    __syncthreads();
}

// LL exchange of element j over the ranks (see cfmm_allreduce.cu): push this rank's partial into every peer's receive
// area, then sum what the peers pushed into ours, in rank order (same bits on every rank)
__device__ __forceinline__ void ll_push(double mine, LLCell* const* recv, long long slot, long long stride, int j, int rank,
                                        int world, unsigned long long seq) {
    for (int r = 0; r < world; ++r)
        if (r != rank) st_ll(recv[r] + slot + (long long)rank * stride + j, mine, seq);
}
// Sum over the ranks of element j, in rank order (same bits on every rank).  The peers' cells are polled FOUR AT A TIME:
// the loads of a round are independent, so a round costs one L2 round trip instead of one per peer (the one-after-the-
// other version cost ~19 us per phase at 8 ranks); cells that carry this step's sequence number are taken, the others
// are asked again.  Not inlined: seven call sites, and the four loads in flight must not add to the kernel's registers.
__device__ __noinline__ double ll_poll_sum(double mine, LLCell* const* recv, long long slot, long long stride, int j,
                                           int rank, int world, unsigned long long seq, unsigned* ctl) {
    const LLCell* base = recv[rank] + slot + j;
    const long long t0 = clock64();
    double s = 0.0;
    for (int r0 = 0; r0 < world; r0 += 4) {
        double v0 = 0.0, v1 = 0.0, v2 = 0.0, v3 = 0.0;
        unsigned pending = 0u;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (r0 + k < world && r0 + k != rank) pending |= 1u << k;
        unsigned spins = 0u;
        while (pending) {
            double t[4];
            unsigned long long f[4];
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (pending >> k & 1u) ld_ll(base + (long long)(r0 + k) * stride, t[k], f[k]);
            if ((pending & 1u) && f[0] == seq) { v0 = t[0]; pending &= ~1u; }
            if ((pending & 2u) && f[1] == seq) { v1 = t[1]; pending &= ~2u; }
            if ((pending & 4u) && f[2] == seq) { v2 = t[2]; pending &= ~4u; }
            if ((pending & 8u) && f[3] == seq) { v3 = t[3]; pending &= ~8u; }
            if (pending && (++spins & 63u) == 0u && (unsigned long long)(clock64() - t0) > kSpinLimit) { ctl[32] = 1u; break; }
        }
        if (r0 + 0 < world) s += (r0 + 0 == rank) ? mine : v0;
        if (r0 + 1 < world) s += (r0 + 1 == rank) ? mine : v1;
        if (r0 + 2 < world) s += (r0 + 2 == rank) ? mine : v2;
        if (r0 + 3 < world) s += (r0 + 3 == rank) ? mine : v3;
    }
    return s;
}

// MULTI = false is the single-GPU instantiation: no exchange code, no calls (the registers of the passes stay as they were)
template <bool MULTI>
__global__ void __launch_bounds__(PT, kCtasPerSm)
k_solve_dist(const __grid_constant__ DistArgs D) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t full[kTileStages];
    __shared__ double part[PT / 32];
    __shared__ double tot[kQ];
    __shared__ DState ds;
    const PersistArgs& S = D.P;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = S.n, nsl = D.nsl, G = gridDim.x;
    if (tid == 0) {
        for (int s = 0; s < kTileStages; ++s) mbar_init(&full[s], 1);
        mbar_fence_init();
        ds.phase = PH_KKT; ds.set = 0; ds.cur = 0; ds.iters = 0; ds.evals = 0; ds.hvps = 0; ds.status = 1; ds.cg_k = 0; ds.ls = 0;
        ds.yb = 0; ds.first_step = 1; ds.dir_ok = 0; ds.aborted = 0; ds.parity = 0; ds.flat = 0;
        ds.err = INFINITY; ds.g0 = 0.0; ds.rz = 0.0; ds.r0n = 0.0; ds.eta = 0.1; ds.alpha = 1.0; ds.lin1 = 0.0; ds.beta = 0.0;
        ds.al = 0.0; ds.imx = 0.0; ds.thr = 1e-5; ds.dsc = 1.0;
        ds.kc.err = INFINITY; ds.kc.g = 0.0; ds.kc.primal = 0.0; ds.kc.infeas = 0.0; ds.kc.lin = 0.0;
        ds.seq_acc = S.seq_acc; ds.seq_vec = S.seq_vec; ds.bar = 0;
        for (int k = 0; k < 16; ++k) ds.prof[k] = 0;
    }
    __syncthreads();
    const long long t_beg = (S.B.n_tiles * (long long)blockIdx.x) / G;
    const long long t_end = (S.B.n_tiles * (long long)(blockIdx.x + 1)) / G;
    unsigned phase_bits = 0;
    // ---- prologue: bounds, start point, cleared accumulator -- every slice by its owner
    for (int s0 = blockIdx.x + warp * G; s0 < nsl; s0 += (PT / 32) * G) {
        const int lo = (int)((long long)n * s0 / nsl), hi = (int)((long long)n * (s0 + 1) / nsl);
        for (int j = lo + lane; j < hi; j += 32) {
            const double l = S.eq[j] ? S.nu_floor : fmax(S.c[j], S.nu_floor);
            S.lb[j] = l;
            S.nu[0][j] = S.fixed[j] ? S.c[j] : fmax(S.nu[0][j], l);
            S.acc[0][j] = 0.0;
        }
        if (s0 == nsl - 1 && lane == 0) S.acc[0][n] = 0.0;
    }
    grid_barrier(S.ctl, &ds);
    for (;;) {
        const int phase = ds.phase, set = ds.set, cur = ds.cur;
        if (phase == PH_DONE || ds.aborted) break;
        const long long tp0 = clock64();
        // ---- the pass of this phase, on this CTA's tiles, then barrier A
        if (phase == PH_KKT) run_pass<0>(S, S.nu[set], S.acc[set], smem_raw, full, phase_bits, t_beg, t_end, part, 0.0);
        else if (phase == PH_HVP) run_pass<1>(S, S.p, D.y2[ds.yb], smem_raw, full, phase_bits, t_beg, t_end, part, ds.beta);
        else if (phase == PH_DIAG) run_pass<2>(S, nullptr, S.diag, smem_raw, full, phase_bits, t_beg, t_end, part, 0.0);
        const long long tp1 = clock64();
        if (phase != PH_STEP) grid_barrier(S.ctl, &ds);
        const long long tp2 = clock64();
        // ---- slice phase
        const int par = ds.parity;
        double* P0 = D.partial + (size_t)par * kQ * kSliceMax;
        constexpr bool multi = MULTI;
        unsigned long long seq = 0;
        if (phase == PH_KKT) seq = ds.seq_acc + 1; else if (phase == PH_DIAG || phase == PH_HVP) seq = ds.seq_vec + 1;
        const long long slot_acc = (long long)(seq % 3) * S.world * (n + 1), slot_vec = (long long)(seq % 3) * S.world * (n + 2);
        if (phase == PH_HVP) {                       // p'Hp and p'diag(H)p first: alpha feeds the element-wise update
            const double* yb = D.y2[ds.yb];
            if (multi) {
                // every push of this phase goes out before anybody polls: one NVLink trip covers the scalars and the slices
                for (int s0 = blockIdx.x + warp * G; s0 < nsl; s0 += (PT / 32) * G) {
                    const int lo = (int)((long long)n * s0 / nsl), hi = (int)((long long)n * (s0 + 1) / nsl);
                    for (int j = lo + lane; j < hi; j += 32) ll_push(ldw(yb + j), S.recv_vec, slot_vec, n + 2, j, S.rank, S.world, seq);
                    if (s0 == nsl - 1 && lane < 2) ll_push(ldw(yb + n + lane), S.recv_vec, slot_vec, n + 2, n + lane, S.rank, S.world, seq);
                }
            }
            if (tid == 0) {
                double pHp = ldw(yb + n), pdp = ldw(yb + n + 1);
                if (multi) {
                    pHp = ll_poll_sum(pHp, S.recv_vec, slot_vec, n + 2, n, S.rank, S.world, seq, S.ctl);
                    pdp = ll_poll_sum(pdp, S.recv_vec, slot_vec, n + 2, n + 1, S.rank, S.world, seq, S.ctl);
                }
                ds.flat = pHp <= 1e-14 * pdp;        // homogeneity direction: g is linear along nu
                ds.al = ds.flat ? 0.0 : ds.rz / pHp;
            }
            __syncthreads();
        }
        const double al = ds.al;
        const int flat = ds.flat;
        for (int s0 = blockIdx.x + warp * G; s0 < nsl; s0 += (PT / 32) * G) {
            const int lo = (int)((long long)n * s0 / nsl), hi = (int)((long long)n * (s0 + 1) / nsl);
            double q[kQ];
#pragma unroll
            for (int k = 0; k < kQ; ++k) q[k] = 0.0;
            for (int j = lo + lane; j < hi; j += 32) {
                if (phase == PH_KKT) {
                    double pj = ldw(S.acc[set] + j);
                    const double nj = ldw(S.nu[set] + j), aj = S.a[j], cj = S.c[j], lbj = ldw(S.lb + j);
                    const unsigned char ej = S.eq[j], fj = S.fixed[j];
                    const bool wl = set != cur;      // trial point: also grad_cur . (nu_trial - nu_cur)
                    const double np = wl ? ldw(S.nu[cur] + j) : 0.0, gp = wl ? ldw(S.grad[cur] + j) : 0.0;
                    if (multi) {
                        ll_push(pj, S.recv_acc, slot_acc, n + 1, j, S.rank, S.world, seq);
                        if (s0 == nsl - 1 && lane == 0) ll_push(ldw(S.acc[set] + n), S.recv_acc, slot_acc, n + 1, n, S.rank, S.world, seq);
                        pj = ll_poll_sum(pj, S.recv_acc, slot_acc, n + 1, j, S.rank, S.world, seq, S.ctl);
                    }
                    const double g = aj + pj;
                    const bool near = (nj <= lbj * (1.0 + ds.thr)) && !ej;
                    const bool act = fj || (near && g > 0.0);
                    const double f = act ? 0.0 : 1.0, v = nj * g * f;
                    S.grad[set][j] = g; S.fr[set][j] = f; S.pg[set][j] = v; D.accr[set][j] = pj;
                    S.diag[j] = 0.0;                 // the diagonal pass that may follow accumulates into it
                    q[0] += fabs(v); q[1] += (nj - cj) * aj; q[2] += nj * fabs(g); q[3] += cj * pj;
                    q[4] += nj * (fj ? 0.0 : (ej ? fabs(g) : fmax(-g, 0.0)));
                    q[5] += gp * (nj - np);
                    q[6] = fmax(q[6], fabs(g) * f);
                    q[7] = fmax(q[7], fmax(fabs(aj), fj ? 0.0 : fabs(pj)));
                } else if (phase == PH_DIAG) {
                    double d = ldw(S.diag + j);
                    const double f = ldw(S.fr[cur] + j), g = ldw(S.pg[cur] + j);
                    if (multi) {
                        ll_push(d, S.recv_vec, slot_vec, n + 2, j, S.rank, S.world, seq);
                        d = ll_poll_sum(d, S.recv_vec, slot_vec, n + 2, j, S.rank, S.world, seq, S.ctl);
                    }
                    const double mi = f / fmax(d, 1e-300), r = -g, z = mi * r;
                    S.minv[j] = mi; S.x[j] = 0.0; S.r[j] = r; S.z[j] = z; S.p[j] = z;
                    D.y2[0][j] = 0.0;
                    q[0] += r * z;
                    q[6] = fmax(q[6], fabs(g));
                } else if (phase == PH_HVP) {
                    double yv = ldw(D.y2[ds.yb] + j);
                    const double pp = ldw(S.p + j), zz = ldw(S.z + j), xx = ldw(S.x + j), rr = ldw(S.r + j),
                                 mm = ldw(S.minv + j), g = ldw(S.pg[cur] + j);
                    if (multi) yv = ll_poll_sum(yv, S.recv_vec, slot_vec, n + 2, j, S.rank, S.world, seq, S.ctl);   // pushed above
                    const double pj = fma(ds.beta, pp, zz);             // the direction the pass used
                    double xn = xx;
                    S.p[j] = pj;
                    if (flat) {
                        if (ds.cg_k == 0) { xn = pj; S.x[j] = xn; }
                    } else {
                        const double r = rr - al * yv, z = mm * r;
                        xn = fma(al, pj, xx);
                        S.x[j] = xn; S.r[j] = r; S.z[j] = z;
                        q[0] += r * z;
                    }
                    q[1] += g * xn;                  // pg . x: is x a descent direction (needed when PCG stops here)
                    q[6] = fmax(q[6], fabs(xn));     // max |x|: the step is bounded to kDtMax when PCG stops here
                    D.y2[ds.yb ^ 1][j] = 0.0;
                } else {                             // PH_STEP: direction (first step of a search) + trial point
                    const double g = ldw(S.pg[cur] + j), xx = ldw(S.x + j), v = ldw(S.nu[cur] + j), l = ldw(S.lb + j);
                    double d;
                    if (ds.first_step) { d = ds.dir_ok ? xx * ds.dsc : -g * ds.imx; S.dt[j] = d; }
                    else d = ldw(S.dt + j);
                    const double e = fmin(fmax(ds.alpha * d, -20.0), 20.0);
                    S.nu[cur ^ 1][j] = S.fixed[j] ? S.c[j] : fmax(v * exp(e), l);
                    S.acc[cur ^ 1][j] = 0.0;
                }
            }
            if (s0 == nsl - 1 && lane == 0) {        // the extras behind the vectors
                if (phase == PH_KKT) {
                    double arb = ldw(S.acc[set] + n);
                    if (multi) arb = ll_poll_sum(arb, S.recv_acc, slot_acc, n + 1, n, S.rank, S.world, seq, S.ctl);   // pushed with the slice
                    q[8] = arb;
                } else if (phase == PH_DIAG) { D.y2[0][n] = 0.0; D.y2[0][n + 1] = 0.0; }
                else if (phase == PH_HVP) { D.y2[ds.yb ^ 1][n] = 0.0; D.y2[ds.yb ^ 1][n + 1] = 0.0; }
                else S.acc[cur ^ 1][n] = 0.0;
            }
            if (phase != PH_STEP) {
#pragma unroll
                for (int k = 0; k < 6; ++k) q[k] = warp_sum(q[k]);
                q[6] = warp_max(q[6]); q[7] = warp_max(q[7]);
                if (lane == 0) {
#pragma unroll
                    for (int k = 0; k < 9; ++k) P0[k * kSliceMax + s0] = q[k];
                }
            }
        }
        const long long tp3 = clock64();
        grid_barrier(S.ctl, &ds);
        const long long tp4 = clock64();
        // ---- decide phase: slice partials -> totals (slice order: same bits in every CTA and on every rank)
        if (warp < 9 && phase != PH_STEP) {          // warp k totals quantity k: all loads of the phase in flight at once
            const int k = warp;
            const bool is_max = k == 6 || k == 7;
            double t = 0.0;
            for (int s = lane; s < nsl; s += 32) {
                const double v = ldw(P0 + k * kSliceMax + s);
                t = is_max ? fmax(t, v) : t + v;
            }
            t = is_max ? warp_max(t) : warp_sum(t);
            if (lane == 0) tot[k] = t;
        }
        __syncthreads();
        if (tid == 0) {
            ds.parity ^= 1;
            int next = PH_DONE;
            bool newton = false;
            if (ds.aborted) {
                next = PH_DONE;
            } else if (phase == PH_KKT) {
                ++ds.seq_acc; ++ds.evals;
                Kkt k;
                k.g = tot[1] + tot[8];
                k.err = fmax(tot[0] / fmax(fmax(fabs(k.g), 1e-3 * tot[2]), 1e-300), tot[6] / fmax(tot[7], 1e-300));
                k.primal = tot[3]; k.infeas = tot[4] / fmax(fabs(k.g), 1e-300); k.lin = tot[5];
                if (set == cur) {                    // the start point
                    ds.kc = k; ds.err = k.err; ds.g0 = k.g; newton = true;
                } else {                             // Armijo test along nu * exp(alpha dt)
                    if (ds.ls == 0) ds.lin1 = k.lin;
                    bool accept = k.g <= ds.g0 + 1e-4 * k.lin, stalled = false;
                    if (!accept && (fabs(k.g - ds.g0) <= 1e-13 * fabs(ds.g0) || fabs(ds.lin1) <= 1e-9 * fabs(ds.g0))) {
                        if (k.err < 0.99 * ds.err) accept = true;        // below what g resolves: judged by the KKT residual
                        else if (ds.alpha < 1e-3) stalled = true;
                    }
                    if (accept) { ds.cur = set; ds.kc = k; ds.err = k.err; ds.g0 = k.g; newton = true; }
                    else if (stalled || ++ds.ls >= 50) { ds.status = 2; next = PH_DONE; }
                    else { ds.alpha *= 0.5; ds.first_step = 0; next = PH_STEP; }
                }
                if (newton) {                        // same counting as cfmm_solver.cu: the final check is an iteration too
                    if (ds.iters >= S.max_iter) { ds.status = 1; next = PH_DONE; }
                    else {
                        ++ds.iters;
                        if (ds.err <= S.tol) { ds.status = 0; next = PH_DONE; }
                        else next = PH_DIAG;
                    }
                }
            } else if (phase == PH_DIAG) {
                ++ds.seq_vec;
                ds.rz = tot[0]; ds.r0n = sqrt(fmax(ds.rz, 0.0)); ds.eta = fmin(0.1, sqrt(ds.err));
                ds.imx = 1.0 / fmax(tot[6], 1e-300);
                ds.cg_k = 0; ds.beta = 0.0; ds.yb = 0;
                if (ds.rz <= 0.0) { ds.dir_ok = 0; ds.first_step = 1; ds.alpha = 1.0; ds.ls = 0; ds.lin1 = 0.0; next = PH_STEP; }
                else next = PH_HVP;
            } else if (phase == PH_HVP) {
                ++ds.seq_vec; ++ds.hvps;
                bool stop = flat != 0;
                if (!flat) {
                    const double rzn = tot[0];
                    stop = (rzn <= 0.0) || (sqrt(fmax(rzn, 0.0)) <= ds.eta * ds.r0n);
                    ds.beta = rzn / ds.rz;
                    ds.rz = rzn;
                }
                ++ds.cg_k; ds.yb ^= 1;
                if (!stop && ds.cg_k < S.cg_max) next = PH_HVP;
                else {
                    const double sdir = tot[1];
                    ds.dir_ok = (isfinite(sdir) && sdir < 0.0) ? 1 : 0;
                    // at most kDtMax per coordinate, as solver.py bounds it: a truncated-CG step can be ~1e14 long, and
                    // every trial of the search would then sit on the +-20 clamp of PH_STEP
                    ds.dsc = tot[6] > kDtMax ? kDtMax / tot[6] : 1.0;
                    ds.first_step = 1; ds.alpha = 1.0; ds.ls = 0; ds.lin1 = 0.0;
                    next = PH_STEP;
                }
            } else {                                 // PH_STEP -> evaluate the trial point
                ds.set = cur ^ 1;
                ds.thr = fmin(1e-2, fmax(1e-3 * (isfinite(ds.err) ? ds.err : 1e-2), 1e-14));     // active-set width (see solver.py)
                next = PH_KKT;
            }
            if (next == PH_DONE && ds.status == 1 && ds.err <= S.tol) ds.status = 0;
            ds.phase = next;
            if (blockIdx.x == 0) {
                ds.prof[phase == PH_KKT ? 0 : phase == PH_HVP ? 1 : phase == PH_DIAG ? 2 : 7] += tp1 - tp0;
                ds.prof[3] += tp2 - tp1; ds.prof[4] += tp3 - tp2; ds.prof[5] += tp4 - tp3; ds.prof[6] += clock64() - tp4;
            }
        }
        __syncthreads();
    }
    // ---- results: every slice owner copies its part; CTA 0 writes the scalars
    {
        const int cur = ds.cur;
        for (int s0 = blockIdx.x + warp * G; s0 < nsl; s0 += (PT / 32) * G) {
            const int lo = (int)((long long)n * s0 / nsl), hi = (int)((long long)n * (s0 + 1) / nsl);
            for (int j = lo + lane; j < hi; j += 32) {
                S.psi_out[j] = ldw(D.accr[cur] + j);
                if (cur != 0) S.nu_out[j] = ldw(S.nu[cur] + j);
            }
        }
        if (blockIdx.x == 0 && tid == 0) {
            DevResult R;
            R.dual_value = ds.kc.g; R.primal_value = ds.kc.primal;
            R.gap = (ds.kc.g - ds.kc.primal) / fmax(fabs(ds.kc.g), 1e-300);
            R.primal_infeas = ds.kc.infeas; R.err = ds.err;
            R.iters = ds.iters; R.evals = ds.evals; R.hvps = ds.hvps; R.status = ds.aborted ? 3 : ds.status;
            R.seq_acc = ds.seq_acc; R.seq_vec = ds.seq_vec;
            for (int k = 0; k < 16; ++k) R.prof[k] = ds.prof[k];
            *S.res = R;
        }
    }
}

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }
thread_local long long g_last_prof[16] = {0};
int g_persist_cooperative = 1;

}  // namespace

extern "C" {

int64_t cfmm_persist_solve_work_bytes(const cfmm_blocked_pairs* b, int32_t n_tokens) {
    if (!b || n_tokens <= 0) return CFMM_E_SIZE;
    const size_t n = (size_t)n_tokens;
    size_t bytes = align_up(8 * (size_t)b->n_tiles * (size_t)b->pools_per_tile);      // hcoef
    bytes += 2 * align_up(8 * (n + 1));       // [psi | arb] of the current / trial point
    bytes += 18 * align_up(8 * n) + align_up(8 * (n + 2));    // nu trial, diag, lb, grad x2, fr x2, pg x2, dt, x, r, z, p, minv (+3 spare); y (+ p'Hp, p'Dp)
    bytes += align_up(512) + align_up(sizeof(DevResult));
    bytes += 2 * align_up(8 * n) + 2 * align_up(8 * (n + 2)) + align_up(8 * (size_t)2 * kQ * kSliceMax);   // distributed variant
    return (int64_t)bytes;
}

int cfmm_persist_solve(const cfmm_blocked_pairs* b, int32_t n_tokens, const double* c, const double* a,
                       const uint8_t* eq, const uint8_t* pinned, double* nu, double* psi_out, void* work,
                       const cfmm_solve_params* prm, cfmm_solve_result* res, cfmm_peer_ctx* peer, void* stream) {
    if (!b || !c || !a || !eq || !pinned || !nu || !psi_out || !work || !prm || !res) return CFMM_E_NULL;
    if (n_tokens <= 0 || b->n_tiles <= 0) return CFMM_E_SIZE;
    if (!b->r0 || !b->r1 || !b->gamma_inv) return CFMM_E_NULL;
    if (peer && (!peer->recv_acc_dev || !peer->recv_vec_dev)) return CFMM_E_NULL;
    if (peer && (peer->world < 2 || peer->world > 16 || peer->rank < 0 || peer->rank >= peer->world)) return CFMM_E_SIZE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    PersistArgs S;
    memset(&S, 0, sizeof(S));
    int rc = fill_blocked_args(b, S.B);
    if (rc) return rc;
    S.B.slab[0] = b->r0; S.B.slab[1] = b->r1; S.B.slab[2] = b->gamma_inv;
    const int n = n_tokens;
    S.n = n; S.c = c; S.a = a; S.eq = eq; S.fixed = pinned;
    unsigned char* w = static_cast<unsigned char*>(work);
    auto take = [&](size_t bytes) { unsigned char* p = w; w += align_up(bytes); return p; };
    auto vec = [&]() { return reinterpret_cast<double*>(take(8 * (size_t)n)); };
    S.hcoef = reinterpret_cast<double*>(take(8 * (size_t)S.B.M));
    S.acc[0] = reinterpret_cast<double*>(take(8 * (size_t)(n + 1)));
    S.acc[1] = reinterpret_cast<double*>(take(8 * (size_t)(n + 1)));
    S.nu[0] = nu; S.nu[1] = vec();
    S.y = reinterpret_cast<double*>(take(8 * (size_t)(n + 2))); S.diag = vec(); S.lb = vec();
    S.grad[0] = vec(); S.grad[1] = vec(); S.fr[0] = vec(); S.fr[1] = vec(); S.pg[0] = vec(); S.pg[1] = vec();
    S.dt = vec(); S.x = vec(); S.r = vec(); S.z = vec(); S.p = vec(); S.minv = vec();
    vec(); vec(); vec();
    S.ctl = reinterpret_cast<unsigned*>(take(512));
    S.res = reinterpret_cast<DevResult*>(take(sizeof(DevResult)));
    S.tol = prm->tol; S.nu_floor = prm->nu_floor; S.max_iter = prm->max_iter; S.cg_max = prm->cg_max;
    S.nu_out = nu; S.psi_out = psi_out;
    if (peer) {
        S.recv_acc = static_cast<LLCell* const*>(const_cast<void*>(peer->recv_acc_dev));
        S.recv_vec = static_cast<LLCell* const*>(const_cast<void*>(peer->recv_vec_dev));
        S.rank = peer->rank; S.world = peer->world; S.seq_acc = peer->seq_acc; S.seq_vec = peer->seq_vec;
    } else {
        S.rank = 0; S.world = 1;
    }
    DistArgs D;
    D.accr[0] = vec(); D.accr[1] = vec();
    D.y2[0] = reinterpret_cast<double*>(take(8 * (size_t)(n + 2))); D.y2[1] = reinterpret_cast<double*>(take(8 * (size_t)(n + 2)));
    D.partial = reinterpret_cast<double*>(take(8 * (size_t)2 * kQ * kSliceMax));
    D.nsl = (n + 15) / 16 < kSliceMax ? ((n + 15) / 16 > 0 ? (n + 15) / 16 : 1) : kSliceMax;
    D.P = S;
    const size_t sm = pass_smem_bytes<kTileP, kTileStages>(3);
    const bool multi = S.world > 1;
    auto kern = multi ? k_solve_dist<true> : k_solve_dist<false>;
    static int occs[2] = {-1, -1};
    int& occ = occs[multi ? 1 : 0];
    if (occ < 0) {
        int o = -1;
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kern, PT, sm);
        if (e != cudaSuccess || o < 1) { g_last_err = e; return CFMM_E_CUDA; }
        occ = o;
    }
    const long long cap = (long long)occ * num_sms();
    const int grid = (int)(S.B.n_tiles < cap ? S.B.n_tiles : cap);
    cudaMemsetAsync(S.ctl, 0, 512, st);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(PT); cfg.dynamicSmemBytes = sm; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative;       // all CTAs co-resident (they wait for each other) or the launch fails
    at[0].val.cooperative = g_persist_cooperative;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, D);
    rc = check_launch();
    if (rc) return rc;
    static thread_local DevResult* hres = nullptr;          // pinned mirror of the result struct
    if (!hres && cudaHostAlloc(&hres, sizeof(DevResult), cudaHostAllocDefault) != cudaSuccess) return CFMM_E_CUDA;
    cudaMemcpyAsync(hres, S.res, sizeof(DevResult), cudaMemcpyDeviceToHost, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) { g_last_err = cudaGetLastError(); return CFMM_E_CUDA; }
    res->dual_value = hres->dual_value; res->primal_value = hres->primal_value; res->gap = hres->gap;
    res->primal_infeas = hres->primal_infeas; res->err = hres->err;
    res->iters = hres->iters; res->evals = hres->evals; res->hvps = hres->hvps; res->status = hres->status;
    if (peer) { peer->seq_acc = hres->seq_acc; peer->seq_vec = hres->seq_vec; }
    for (int k = 0; k < 16; ++k) g_last_prof[k] = hres->prof[k];
    return hres->status == 3 ? CFMM_E_STATE : CFMM_OK;
}

/* 1 (default): cooperative launch -- the driver guarantees that all CTAs of a solve are co-resident or fails the launch.
 * 0: plain launch (the grid is still sized to fit the device): for tests that run several "ranks" as concurrent solves on
 * ONE GPU (tests/test_loopback_ranks.py), where each small grid is resident anyway. */
int cfmm_set_persist_cooperative(int32_t on) {
    if (on != 0 && on != 1) return CFMM_E_KIND;
    g_persist_cooperative = on;
    return CFMM_OK;
}

/* CTA 0's clock64 totals of the last cfmm_persist_solve of this thread (SM cycles): [0..2] its own evaluation / Hessian-
 * product / diagonal passes, [3] grid barrier after the passes, [4] slice phases, [5] grid barrier after them, [6] decide
 * phases.  A development aid (where does the solve's time go), not a contract. */
int cfmm_persist_last_profile(int64_t* out8) {
    if (!out8) return CFMM_E_NULL;
    for (int k = 0; k < 16; ++k) out8[k] = g_last_prof[k];
    return CFMM_OK;
}

}  // extern "C"
