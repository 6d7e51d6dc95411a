// cfmm_layout.cu -- native builder of the token-blocked layout (cfmm_blocked_pairs) for constant-product pools.
//
// The reference describes a problem by local_indices / reserves / fees (arbitrage.py:6-28) and turns the indices into
// dense 0/1 matrices A_i (arbitrage.py:42-48).  Here the same literals, uploaded as they are, become the tiled layout the
// evaluation kernels stream (cfmm_blocked.cuh) in three launches:
//   1. k_pool_keys      one key per pool: (token block of slot 0, token block of slot 1, slot-0 token) -- pools whose two
//                       tokens fall into the same pair of narrow token blocks become neighbours; also validates the data
//   2. cub radix sort   of (key, pool id) pairs: the blocked order
//   3. k_build_tiles    ONE CTA PER TILE, everything in shared memory: sort the tile's 2P half-edges by token, number
//                       the distinct tokens (local ids, token list), rank the slot-1 half-edges in token order (their
//                       positions in the flow array), cut the runs of equal tokens in both halves of the flow array
//                       into rows of <= row_cap entries, order the rows longest first, gather the reserves /
//                       1/gamma slabs into blocked order, and code the tile's 1/gamma values (fee record).
// It replaces ~240 torch launches (sort / unique / bincount / repeat_interleave / index ...) and their host round trips.
#include <cub/cub.cuh>

#include "cfmm_blocked.cuh"

using namespace cfmm;

namespace {

constexpr int LT = kTileT;                 // threads per tile CTA
constexpr int LP = kTileP;                 // pools per tile
constexpr int LH = 2 * kTileP;             // half-edges per tile
constexpr int LI = 4;                      // items per thread of the block sorts (LT * LI == LH)
static_assert(LT * LI == LH, "block sort shape");
constexpr int LR = BlockedCfg<kTileP>::kRowsMax;
constexpr int LU = LP / LT;                // pools per thread in step 6
constexpr int LF = fee_words<kTileP>();    // words of a fee record

struct BuildArgs {
    long long m;
    int n_tokens, nb, row_cap, key_bits, tok_bits;
    const int32_t* idx;        // [m][2]
    const double* R;           // [m][2]
    const double* gamma;       // [m]
    const uint32_t* order;     // [m] sorted pool ids (blocked position -> pool)
    double *r0, *r1, *gi;      // [T * P]
    uint32_t* pw;              // [T * P]
    uint32_t* rows;            // [T][LR]
    int32_t* tok;              // [T][P]
    int4* desc;                // [T]
    uint32_t* fee;             // [T][LF] fee records, or null
    int32_t* status;           // [0] tiles touching more than P tokens or needing more than LR rows, [1] invalid pools,
                               // [2] total rows
};

struct MaxOp {
    __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; }
};

__global__ void __launch_bounds__(256)
k_pool_keys(long long m, int n_tokens, int nb, const int32_t* __restrict__ idx, const double* __restrict__ R,
            const double* __restrict__ gamma, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, int32_t* status) {
    int bad = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
        const int a = idx[2 * i], b = idx[2 * i + 1];
        const double R0 = R[2 * i], R1 = R[2 * i + 1], g = gamma[i];
        const bool ok = a >= 0 && a < n_tokens && b >= 0 && b < n_tokens && a != b && R0 > 0.0 && R1 > 0.0 && isfinite(R0) &&
                        isfinite(R1) && g > 0.0 && g <= 1.0;
        bad |= ok ? 0 : 1;
        const long long ba = ok ? ((long long)a * nb) / n_tokens : 0, bb = ok ? ((long long)b * nb) / n_tokens : 0;
        keys[i] = (uint32_t)((ba * nb + bb) * n_tokens + (ok ? a : 0));
        vals[i] = (uint32_t)i;
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicAdd(status + 1, 1);
}

using Sort = cub::BlockRadixSort<uint32_t, LT, LI, uint32_t>;
using Scan = cub::BlockScan<int, LT>;

struct FeeSmem {                           // shared memory of fee_record (a tile CTA of the builder or of the refresh)
    unsigned long long wmin[LT / 32];      // per-warp minima of a block min
    unsigned long long ftab[kFeeMax];      // the tile's distinct 1/gamma bit patterns, ascending
};

struct TileSmem {                          // dynamic shared memory of one tile CTA (> 48 KB with the cub scratch)
    union { typename Sort::TempStorage sort; typename Scan::TempStorage scan; } tmp;
    uint32_t sk[LH];                       // half-edges sorted by token: token id
    uint32_t sv[LH];                       //                              slot << 15 | pool-in-tile
    uint16_t gid[LH];                      // local token id of every sorted half-edge
    uint16_t ftok[LH];                     // local token of the flow at every position of the flow array (slot 0 | slot 1)
    uint16_t rlen[LH];                     // length of the run of equal tokens that starts at a position of the flow array
    uint16_t lidh[LP][2], p1h[LP];         // local ids and slot-1 position of every pool
    int ntok;
    FeeSmem fs;
};

// a tile the layout cannot hold: counted in status[0], its slabs and tables kept inert (never launched: the host falls back)
__device__ void inert_tile(const BuildArgs& B, long long tile) {
    const long long p0 = tile * LP;
    if (threadIdx.x == 0) { atomicAdd(B.status, 1); B.desc[tile] = make_int4(0, 0, 0, 0); }
    for (int l = threadIdx.x; l < LP; l += LT) {
        B.r0[p0 + l] = 1.0; B.r1[p0 + l] = 1.0; B.gi[p0 + l] = 1.0; B.pw[p0 + l] = 0u;
    }
    if (B.fee)
        for (int k = threadIdx.x; k < LF; k += LT) B.fee[tile * LF + k] = 0u;
}

// minimum over the tile CTA (every thread gets it)
__device__ unsigned long long block_min(unsigned long long x, FeeSmem& M) {
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long y = __shfl_xor_sync(0xffffffffu, x, o);
        x = y < x ? y : x;
    }
    if ((threadIdx.x & 31) == 0) M.wmin[threadIdx.x >> 5] = x;
    __syncthreads();
    x = M.wmin[0];
    for (int k = 1; k < LT / 32; ++k) x = M.wmin[k] < x ? M.wmin[k] : x;
    __syncthreads();
    return x;
}

// ---- 7. fee record `rec` (include/cfmm_b200.h) of a tile whose pool l = tid + u * LT has 1/gamma bit pattern gib[u],
// padding included: the distinct patterns in ascending order, one block min over the patterns above the last one per
// value (positive doubles order like their bit patterns), then a 4-bit index per pool.  More than kFeeMax values: all
// zero.  Shared by the builder (k_build_tiles) and the in-place update (k_refresh_fees).
__device__ void fee_record(uint32_t* rec, FeeSmem& M, const unsigned long long (&gib)[LU]) {
    const int tid = threadIdx.x;
    unsigned long long last = 0;
    int nfee = 0;
    bool over = false;
    for (;;) {
        unsigned long long c = ~0ull;                       // a NaN pattern: never a 1/gamma
#pragma unroll
        for (int u = 0; u < LU; ++u)
            if ((nfee == 0 || gib[u] > last) && gib[u] < c) c = gib[u];
        c = block_min(c, M);                                // (its barriers publish ftab[] written below)
        if (c == ~0ull) break;
        if (nfee == kFeeMax) { over = true; break; }
        if (tid == 0) M.ftab[nfee] = c;
        last = c;
        ++nfee;
    }
    if (over) nfee = 0;
    if (tid < kFeeTab) rec[tid] = tid == 0 ? (uint32_t)nfee : 0u;
    if (tid < 2 * kFeeMax) {
        const unsigned long long v = (tid >> 1) < nfee ? M.ftab[tid >> 1] : 0ull;
        rec[kFeeTab + tid] = (uint32_t)(tid & 1 ? v >> 32 : v);
    }
    // pool l sits at nibble l & 7 == tid & 7 of word l >> 3: the 8 lanes of one word OR their nibbles together
#pragma unroll
    for (int u = 0; u < LU; ++u) {
        unsigned code = 0;
        for (int e = 0; e < nfee; ++e) code = M.ftab[e] == gib[u] ? (unsigned)e : code;
        unsigned w = code << (4 * (tid & 7));
        w |= __shfl_xor_sync(0xffffffffu, w, 1);
        w |= __shfl_xor_sync(0xffffffffu, w, 2);
        w |= __shfl_xor_sync(0xffffffffu, w, 4);
        if ((tid & 7) == 0) rec[kFeeCode + ((tid + u * LT) >> 3)] = w;
    }
}

__global__ void __launch_bounds__(LT)
k_build_tiles(const BuildArgs B) {
    extern __shared__ __align__(16) unsigned char tile_smem_raw[];
    TileSmem& M = *reinterpret_cast<TileSmem*>(tile_smem_raw);
    auto& tmp = M.tmp;
    uint32_t* sk = M.sk; uint32_t* sv = M.sv; uint16_t* gid = M.gid; uint16_t* ftok = M.ftok; uint16_t* rlen = M.rlen;
    auto& lidh = M.lidh; uint16_t* p1h = M.p1h;
    int& s_ntok = M.ntok;
    const int tid = threadIdx.x;
    const long long tile = blockIdx.x;
    const long long p0 = tile * LP;
    const int np = (int)(B.m - p0 < LP ? B.m - p0 : LP);               // real pools in this tile
    const int nh = 2 * np;
    auto real = [&](int c) { return (c < LP ? c : c - LP) < np; };     // position c of the flow array holds a real flow
    // ---- 1. the tile's half-edges, slot-major (slot 0 of every pool, then slot 1), sorted by token (stable)
    uint32_t key[LI], val[LI];
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int h = tid * LI + u;                                     // blocked arrangement
        const int slot = h >= LP ? 1 : 0, l = h - slot * LP;
        if (l < np) {
            const uint32_t pool = B.order[p0 + l];
            key[u] = (uint32_t)B.idx[2 * (long long)pool + slot];
            val[u] = (uint32_t)(slot << 15 | l);
        } else {
            key[u] = 0xffffffffu; val[u] = 0u;                          // padding: sorts behind every token
        }
    }
    Sort(tmp.sort).Sort(key, val, 0, 32);
#pragma unroll
    for (int u = 0; u < LI; ++u) { sk[tid * LI + u] = key[u]; sv[tid * LI + u] = val[u]; }
    __syncthreads();
    // ---- 2. distinct tokens: heads -> local ids (exclusive scan), token list
    int head[LI], gpre[LI];
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int i = tid * LI + u;
        head[u] = (i < nh && (i == 0 || sk[i] != sk[i - 1])) ? 1 : 0;
    }
    int ntok;
    Scan(tmp.scan).ExclusiveSum(head, gpre, ntok);
    __syncthreads();
    if (ntok > LP) { inert_tile(B, tile); return; }                      // more tokens than a tile may touch: not blockable
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int i = tid * LI + u;
        if (i < nh) {
            const int g = gpre[u] + head[u] - 1;                         // local id of this half-edge's token
            gid[i] = (uint16_t)g;
            if (head[u]) B.tok[tile * LP + g] = (int32_t)sk[i];
        }
    }
    if (tid == 0) s_ntok = ntok;
    __syncthreads();
    // ---- 3. local ids of every pool; a slot-1 half-edge's rank among the slot-1 half-edges in token order (stable: pool
    // order within a token) is the position of its flow in the second half of the flow array, a slot-0 flow sits at its pool
    int s1[LI], p1[LI];
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int i = tid * LI + u;
        s1[u] = (i < nh && (sv[i] >> 15)) ? 1 : 0;
    }
    Scan(tmp.scan).ExclusiveSum(s1, p1);
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int i = tid * LI + u;
        if (i < nh) {
            const uint32_t v = sv[i];
            const int slot = v >> 15, l = v & 0x7fffu;
            lidh[l][slot] = gid[i];
            if (slot) { p1h[l] = (uint16_t)p1[u]; ftok[LP + p1[u]] = gid[i]; }
            else ftok[l] = gid[i];
        }
    }
    __syncthreads();
    // ---- 4. runs of equal tokens in each half of the flow array: slot 0 in pool order (the pools are sorted by slot-0
    // token within a key block), slot 1 in token order.  Every position learns where its run starts; run ends record
    // the run's length at the start
    int hs[LI], rs[LI];
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int c = tid * LI + u;
        hs[u] = (real(c) && (c == 0 || c == LP || ftok[c] != ftok[c - 1])) ? c : -1;
    }
    Scan(tmp.scan).InclusiveScan(hs, rs, MaxOp());
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int c = tid * LI + u;
        if (real(c) && (c + 1 == LP || c + 1 == LH || !real(c + 1) || ftok[c + 1] != ftok[c])) rlen[rs[u]] = (uint16_t)(c - rs[u] + 1);
    }
    __syncthreads();
    // ---- 5. rows: every run cut into rows of <= row_cap entries, sorted longest first (the 32 rows a warp sums then
    // have nearly equal trip counts; ties in flow-array order).  Key: (63 - length) << 11 | start
    const int cap = B.row_cap;
    uint32_t rkey[LI], rdum[LI];
    int nrow = 0;
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int c = tid * LI + u;
        const int o = c - rs[u];
        const bool rh = real(c) && o % cap == 0;
        rkey[u] = rh ? (uint32_t)(63 - min(cap, (int)rlen[rs[u]] - o)) << 11 | (uint32_t)c : 0xffffffffu;
        rdum[u] = 0u;
        nrow += __syncthreads_count(rh);
    }
    if (nrow > LR) { inert_tile(B, tile); return; }                      // more rows than the row table holds: not blockable
    Sort(tmp.sort).Sort(rkey, rdum, 0, 17);
#pragma unroll
    for (int u = 0; u < LI; ++u) {
        const int r = tid * LI + u;
        if (r < nrow) {
            const int c = (int)(rkey[u] & 0x7ffu);
            B.rows[tile * LR + r] = (uint32_t)c | (uint32_t)(63 - (int)(rkey[u] >> 11)) << 16 | (uint32_t)ftok[c] << 22;
        }
    }
    // ---- 6. pool words and slabs, blocked order; padding pool l writes zero flows to g[l] and g[P + l], past the real ones
    unsigned long long gib[LU];
#pragma unroll
    for (int u = 0; u < LU; ++u) {
        const int l = tid + u * LT;
        double gi = 1.0;
        if (l < np) {
            const uint32_t pool = B.order[p0 + l];
            B.pw[p0 + l] = (uint32_t)lidh[l][0] | (uint32_t)lidh[l][1] << 10 | (uint32_t)p1h[l] << 20;
            B.r0[p0 + l] = B.R[2 * (long long)pool]; B.r1[p0 + l] = B.R[2 * (long long)pool + 1];
            gi = 1.0 / B.gamma[pool];
        } else {
            B.pw[p0 + l] = (uint32_t)l << 20;
            B.r0[p0 + l] = 1.0; B.r1[p0 + l] = 1.0;
        }
        B.gi[p0 + l] = gi;
        gib[u] = (unsigned long long)__double_as_longlong(gi);
    }
    if (tid == 0) { B.desc[tile] = make_int4(s_ntok, nrow, 0, 0); atomicAdd(B.status + 2, nrow); }
    if (B.fee) fee_record(B.fee + tile * LF, M.fs, gib);
}

// ---- in-place update of a built layout (cfmm_blocked_update).  The layout depends on the token ids only; reserves and
// fees are payload: new values go to their blocked positions, and the fee record of every tile whose 1/gamma slab
// changed is rebuilt from the slab by fee_record, so the result is bit for bit what the builder makes of the new data.
// status[0]: invalid entries (the rules of k_pool_keys), status[1]: fee records rebuilt.
__global__ void __launch_bounds__(256)
k_update_check(long long n, long long n_pools, const uint32_t* __restrict__ at, const double* __restrict__ R,
               const double* __restrict__ gamma, int32_t* status) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        bool ok = at[i] < n_pools;
        if (R) {
            const double R0 = R[2 * i], R1 = R[2 * i + 1];
            ok = ok && R0 > 0.0 && R1 > 0.0 && isfinite(R0) && isfinite(R1);
        }
        if (gamma) {
            const double g = gamma[i];
            ok = ok && g > 0.0 && g <= 1.0;
        }
        if (!ok) atomicAdd(status, 1);
    }
}

// applies the update only if k_update_check found nothing wrong; flags the tile of every pool whose 1/gamma changed
__global__ void __launch_bounds__(256)
k_update_apply(long long n, const uint32_t* __restrict__ at, const double* __restrict__ R, const double* __restrict__ gamma,
               double* r0, double* r1, double* gi, uint32_t* flag, const int32_t* status) {
    if (*status != 0) return;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long p = at[i];
        if (R) { r0[p] = R[2 * i]; r1[p] = R[2 * i + 1]; }
        if (gamma) {
            const double g = 1.0 / gamma[i];                            // the builder's division
            if (__double_as_longlong(g) != __double_as_longlong(gi[p])) { gi[p] = g; flag[p / LP] = 1u; }
        }
    }
}

// one CTA per tile: a flagged tile rebuilds its fee record from its 1/gamma slab
__global__ void __launch_bounds__(LT)
k_refresh_fees(const double* __restrict__ gi, uint32_t* fee, const uint32_t* __restrict__ flag, int32_t* status) {
    __shared__ FeeSmem M;
    const long long tile = blockIdx.x;
    if (flag[tile] == 0u) return;
    unsigned long long gib[LU];
#pragma unroll
    for (int u = 0; u < LU; ++u) gib[u] = (unsigned long long)__double_as_longlong(gi[tile * LP + threadIdx.x + u * LT]);
    fee_record(fee + tile * LF, M, gib);
    if (threadIdx.x == 0) atomicAdd(status + 1, 1);
}

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

size_t sort_temp_bytes(long long m) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)m, 0, 32);
    return bytes;
}

}  // namespace

extern "C" {

int64_t cfmm_blocked_build_work_bytes(int64_t n_pools) {
    if (n_pools <= 0 || n_pools > 0x7fffffffLL) return CFMM_E_SIZE;
    return (int64_t)(4 * align_up(4 * (size_t)n_pools) + align_up(sort_temp_bytes(n_pools)));
}

/* Build the token-blocked layout of m constant-product pools on the device.  idx [m][2] int32, reserves [m][2] f64,
 * gamma [m] f64: the reference's local_indices / reserves / fees (arbitrage.py:6-28) as contiguous device arrays.
 * `out`: a cfmm_blocked_pairs whose array members point at caller-allocated device buffers of n_tiles = ceil(m / P)
 * tiles (strides from cfmm_blocked_layout_info / cfmm_blocked_fee_words); r0 / r1 / gamma_inv / pw / rows / tok / desc
 * are filled, and the fee records if out->fee is not NULL.
 * order [m] uint32 (device, out): pool at every blocked position.  status [4] int32 (device, zeroed by this call, out):
 * [0] tiles that touch more tokens, or need more rows, than a tile may (the caller must fall back to a plain bucket for
 * such problems),
 * [1] CTAs that saw invalid pools (reserves <= 0 or not finite, fees outside (0, 1], token ids out of range or equal),
 * [2] total rows.  Asynchronous on `stream`. */
int cfmm_blocked_build(int64_t n_pools, int32_t n_tokens, const int32_t* idx, const double* reserves, const double* gamma,
                       const cfmm_blocked_pairs* out, uint32_t* order, int32_t* status, void* work, int64_t work_bytes,
                       void* stream) {
    if (!idx || !reserves || !gamma || !out || !order || !status || !work) return CFMM_E_NULL;
    if (n_pools <= 0 || n_pools > 0x7fffffffLL || n_tokens <= 0) return CFMM_E_SIZE;
    if (work_bytes < cfmm_blocked_build_work_bytes(n_pools)) return CFMM_E_SIZE;
    const long long T = (n_pools + LP - 1) / LP;
    if (out->pools_per_tile != LP || out->n_tiles != T || out->n_pools != n_pools) return CFMM_E_SIZE;
    if (!out->r0 || !out->r1 || !out->gamma_inv || !out->pw || !out->rows || !out->tok || !out->desc) return CFMM_E_NULL;
    int row_cap = 32;
    cfmm_blocked_layout_info(nullptr, nullptr, nullptr, &row_cap);
    long long nb = (long long)llround(sqrt((double)n_pools / LP));
    if (nb < 1) nb = 1;
    if ((double)nb * nb * n_tokens >= 4294967296.0) return CFMM_E_SIZE;          // keys are 32-bit: the caller uses the general builder
    int key_bits = 1;
    while (key_bits < 32 && (1ull << key_bits) < (unsigned long long)(nb * nb) * (unsigned long long)n_tokens) ++key_bits;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned char* w = static_cast<unsigned char*>(work);
    auto take = [&](size_t bytes) { unsigned char* p = w; w += align_up(bytes); return p; };
    uint32_t* keys = reinterpret_cast<uint32_t*>(take(4 * (size_t)n_pools));
    uint32_t* vals = reinterpret_cast<uint32_t*>(take(4 * (size_t)n_pools));
    uint32_t* keys2 = reinterpret_cast<uint32_t*>(take(4 * (size_t)n_pools));
    take(4 * (size_t)n_pools);
    size_t temp_bytes = sort_temp_bytes(n_pools);
    void* temp = take(temp_bytes);
    cudaMemsetAsync(status, 0, 16, st);
    const int grid = (int)((n_pools + 255) / 256 < 4LL * num_sms() ? (n_pools + 255) / 256 : 4LL * num_sms());
    k_pool_keys<<<grid, 256, 0, st>>>(n_pools, n_tokens, (int)nb, idx, reserves, gamma, keys, vals, status);
    int rc = check_launch();
    if (rc) return rc;
    if (cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys, keys2, vals, order, (int)n_pools, 0, key_bits, st) != cudaSuccess) {
        g_last_err = cudaGetLastError();
        return CFMM_E_CUDA;
    }
    BuildArgs B;
    B.m = n_pools; B.n_tokens = n_tokens; B.nb = (int)nb; B.row_cap = row_cap; B.key_bits = key_bits; B.tok_bits = 32;
    B.idx = idx; B.R = reserves; B.gamma = gamma; B.order = order;
    B.r0 = const_cast<double*>(out->r0); B.r1 = const_cast<double*>(out->r1); B.gi = const_cast<double*>(out->gamma_inv);
    B.pw = const_cast<uint32_t*>(out->pw);
    B.rows = const_cast<uint32_t*>(out->rows); B.tok = const_cast<int32_t*>(out->tok);
    B.desc = reinterpret_cast<int4*>(const_cast<int32_t*>(out->desc));
    B.fee = const_cast<uint32_t*>(out->fee);
    B.status = status;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_build_tiles, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileSmem));
        attr = true;
    }
    k_build_tiles<<<(int)T, LT, sizeof(TileSmem), st>>>(B);
    return check_launch();
}

/* work of cfmm_blocked_update: the two status words, then one flag per tile */
int64_t cfmm_blocked_update_work_bytes(const cfmm_blocked_pairs* b) {
    if (!b) return CFMM_E_NULL;
    if (b->n_tiles < 0) return CFMM_E_SIZE;
    return (int64_t)(align_up(8) + align_up(4 * (size_t)b->n_tiles));
}

/* In-place update of the reserves and fees of n_upd pools of a built layout (include/cfmm_b200.h).  Check, apply (only
 * if the check found nothing), refresh the fee records of the tiles whose 1/gamma changed; then wait for the stream. */
int cfmm_blocked_update(const cfmm_blocked_pairs* b, int64_t n_upd, const uint32_t* at, const double* reserves,
                        const double* gamma, int32_t* status_host, void* work, int64_t work_bytes, void* stream) {
    if (!b || !status_host) return CFMM_E_NULL;
    if (n_upd < 0 || b->n_tiles < 0 || b->n_pools < 0 || b->n_pools > b->n_tiles * (int64_t)LP) return CFMM_E_SIZE;
    if (b->pools_per_tile != LP) return CFMM_E_KIND;
    status_host[0] = status_host[1] = 0;
    if (n_upd == 0) return CFMM_OK;
    if (!at || !work || !b->r0 || !b->r1 || !b->gamma_inv) return CFMM_E_NULL;
    if (work_bytes < cfmm_blocked_update_work_bytes(b)) return CFMM_E_SIZE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int32_t* status = static_cast<int32_t*>(work);
    uint32_t* flag = reinterpret_cast<uint32_t*>(static_cast<unsigned char*>(work) + align_up(8));
    // the whole work buffer is cleared here, so it needs no initialisation and may be shared between layouts
    if (cudaMemsetAsync(work, 0, (size_t)cfmm_blocked_update_work_bytes(b), st) != cudaSuccess) {
        g_last_err = cudaGetLastError();
        return CFMM_E_CUDA;
    }
    const int grid = (int)((n_upd + 255) / 256 < 4LL * num_sms() ? (n_upd + 255) / 256 : 4LL * num_sms());
    k_update_check<<<grid, 256, 0, st>>>(n_upd, b->n_pools, at, reserves, gamma, status);
    int rc = check_launch();
    if (rc) return rc;
    k_update_apply<<<grid, 256, 0, st>>>(n_upd, at, reserves, gamma, const_cast<double*>(b->r0), const_cast<double*>(b->r1),
                                         const_cast<double*>(b->gamma_inv), flag, status);
    rc = check_launch();
    if (rc) return rc;
    if (gamma && b->fee && b->n_tiles > 0) {
        k_refresh_fees<<<(int)b->n_tiles, LT, 0, st>>>(b->gamma_inv, const_cast<uint32_t*>(b->fee), flag, status);
        rc = check_launch();
        if (rc) return rc;
    }
    if (cudaMemcpyAsync(status_host, status, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) {
        g_last_err = cudaGetLastError();
        return CFMM_E_CUDA;
    }
    return CFMM_OK;
}

}  // extern "C"
