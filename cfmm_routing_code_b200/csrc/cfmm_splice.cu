// cfmm_splice.cu -- record splice of a bucket whose pools own runs of AoS records (4 f64 each, contiguous, in bucket
// order, in `weights`): new records for some of its pools.
//   cfmm_ladder_splice  concentrated buckets: a tick ladder of T intervals is T + 1 records; (first record, T) in logrw
//                       rows 2-3, the changed pools' (s, c) in rows 0-1.  A mint or burn that initialises or clears a tick
//                       changes T.
//   cfmm_bins_splice    price-bin buckets: nb records; (first record, nb) in logrw rows 0-1, the changed pools' (z, p_ref)
//                       in rows 2-3.  A swap that empties the active bin, a deposit, a withdrawal or a changed book level
//                       changes nb.
// Either way every later pool's records move, so the splice writes the whole record array anew into a second buffer:
//   1. k_splice_check   validate the changed entries (positions sorted, distinct, in range; counts in the kind's range)
//   2. cub scan         of the new pools' record counts: where each one's records start in the packed input
//   3. k_splice_counts  every pool's record count and source (old first record, or its offset in the packed input)
//   4. cub scan         of all counts: every pool's new first record, and the bucket's new total
//   5. k_splice_total   the packed input and the output buffer must match the scans (else nothing is written)
//   6. k_splice_copy    record-parallel copy into the output, 16-byte loads and stores
//   7. k_splice_state   the (first record, count) rows of every pool, the two state rows and the reserves of the changed
//                       ones
// Steps 6 and 7 write nothing if a check failed, so the bucket and the output are untouched by a rejected call.  The
// two entry points run the same kernels; which logrw rows hold what, and the count range, are plain arguments.
#include <cub/cub.cuh>

#include "cfmm_dev.cuh"

using namespace cfmm;

namespace {

// Where a kind keeps its per-pool splice state in logrw: rows `first` and `count` hold the first record and the record
// count minus `count_off`; rows `s0` and `s1` take state columns 0-1 of the changed pools.  Counts lie in 2 .. rec_max.
struct SpliceRows {
    int first, count, count_off, s0, s1;
    long long rec_max;
};
constexpr SpliceRows kLadderRows = {2, 3, 1, 0, 1, (1LL << 20) + 1};   // (first, T), (s, c); T <= 2^20 (LADDER_T_MAX)
constexpr SpliceRows kBinsRows = {0, 1, 0, 2, 3, (1LL << 20) + 2};     // (first, nb), (z, p_ref); K <= 2^20 (BINS_K_MAX)

__global__ void __launch_bounds__(256)
k_splice_check(long long n_chg, long long n_pools, long long rec_max, const int64_t* __restrict__ pos,
               const int64_t* __restrict__ n_rec, long long* __restrict__ newcnt, long long* status) {
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n_chg; k += (long long)gridDim.x * blockDim.x) {
        const long long p = pos[k], c = n_rec[k];
        const bool ok = p >= 0 && p < n_pools && (k == 0 || p > pos[k - 1]) && c >= 2 && c <= rec_max;
        newcnt[k] = ok ? c : 0;
        if (!ok) atomicAdd(reinterpret_cast<unsigned long long*>(status), 1ull);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) newcnt[n_chg] = 0;     // the scan's last entry is the total
}

// cnt[i] = the record count (logrw row `row_cnt` + cnt_off) and src[i] = the old first record (row `row_first`) of
// every pool; then k_splice_mark sets the changed pools' counts and their packed offsets, coded as -1 - offset
__global__ void __launch_bounds__(256)
k_splice_counts(long long n_pools, long long stride, int row_first, int row_cnt, int cnt_off,
                const double* __restrict__ logrw, long long* __restrict__ cnt, long long* __restrict__ src) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pools; i += (long long)gridDim.x * blockDim.x) {
        src[i] = (long long)logrw[row_first * stride + i];
        cnt[i] = (long long)logrw[row_cnt * stride + i] + cnt_off;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) cnt[n_pools] = 0;
}

__global__ void __launch_bounds__(256)
k_splice_mark(long long n_chg, long long n_pools, const int64_t* __restrict__ pos, const long long* __restrict__ newcnt,
              const long long* __restrict__ new_off, long long* cnt, long long* src) {
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n_chg; k += (long long)gridDim.x * blockDim.x) {
        const long long p = pos[k];
        if (p < 0 || p >= n_pools) continue;                         // rejected by k_splice_check: nothing is written
        cnt[p] = newcnt[k];
        src[p] = -1 - new_off[k];
    }
}

__global__ void k_splice_total(long long n_chg, long long n_pools, long long n_records, long long out_capacity,
                               const long long* __restrict__ new_off, const long long* __restrict__ first_new,
                               long long* status) {
    if (new_off[n_chg] != n_records || first_new[n_pools] > out_capacity) status[0] += 1;
    status[1] = first_new[n_pools];
}

// One thread per output record (two 16-byte loads and stores), so a pool of 2^20 intervals spreads over the whole
// grid.  A warp finds the pool of its first record by a binary search over the new first records; every pool holds at
// least two records, so the warp's 32 records lie in at most 17 pools, and each lane finds its own among the ends of
// the next 32 pools by a search over the lanes (shuffles).
__global__ void __launch_bounds__(256)
k_splice_copy(long long n_pools, const long long* __restrict__ first_new, const long long* __restrict__ src,
              const double2* __restrict__ old_rec, const double2* __restrict__ new_rec, double2* __restrict__ out,
              const long long* status) {
    if (status[0] != 0) return;
    const long long total = first_new[n_pools];
    const int lane = threadIdx.x & 31;
    const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w * 32 < total; w += n_warps) {
        const long long r0 = w * 32;
        long long lo = 0, hi = n_pools - 1;                           // the last pool whose first record is <= r0
        while (lo < hi) {
            const long long mid = (lo + hi + 1) >> 1;
            if (first_new[mid] <= r0) lo = mid; else hi = mid - 1;
        }
        const long long end = first_new[lo + 1 + lane < n_pools ? lo + 1 + lane : n_pools];   // end of pool lo + lane
        const long long r = r0 + lane;
        int j = 0;                                                    // pools lo .. lo + j - 1 end at or before r
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
            const long long e = __shfl_sync(0xffffffffu, end, j + step - 1);
            if (e <= r) j += step;
        }
        if (r < total) {
            const long long p = lo + j;
            const long long q = r - first_new[p];
            const long long s = src[p];
            const double2* from = s >= 0 ? old_rec + 2 * (s + q) : new_rec + 2 * (-1 - s + q);
            const double2 a = from[0], b = from[1];
            out[2 * r] = a;
            out[2 * r + 1] = b;
        }
    }
}

__global__ void __launch_bounds__(256)
k_splice_state(long long n_pools, long long n_chg, long long stride, int row_first, int row_cnt, int cnt_off, int row_s0,
               int row_s1, const long long* __restrict__ first_new, const int64_t* __restrict__ pos,
               const double* __restrict__ state, double* logrw, double* reserves, const long long* status) {
    if (status[0] != 0) return;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pools; i += (long long)gridDim.x * blockDim.x) {
        const long long f = first_new[i];
        logrw[row_first * stride + i] = (double)f;
        logrw[row_cnt * stride + i] = (double)(first_new[i + 1] - f - cnt_off);
    }
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n_chg; k += (long long)gridDim.x * blockDim.x) {
        const long long p = pos[k];
        logrw[row_s0 * stride + p] = state[4 * k];
        logrw[row_s1 * stride + p] = state[4 * k + 1];
        reserves[p] = state[4 * k + 2];
        reserves[stride + p] = state[4 * k + 3];
    }
}

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

size_t scan_temp_bytes(long long n) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const long long*)nullptr, (long long*)nullptr, (int)n);
    return bytes;
}

int grid_for(long long n) {
    const long long g = (n + 255) / 256;
    const long long cap = 8LL * num_sms();
    return (int)(g < 1 ? 1 : g < cap ? g : cap);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int splice(const SpliceRows& R, const cfmm_bucket* b, int64_t n_chg, const int64_t* pos, const int64_t* n_rec,
           const double* records, int64_t n_records, const double* state, double* out_records, int64_t out_capacity,
           int64_t* status_host, void* work, int64_t work_bytes, void* stream) {
    if (b->n_pools < 0 || b->stride < b->n_pools || n_chg < 0 || n_chg > b->n_pools || n_records < 0 || out_capacity < 0)
        return CFMM_E_SIZE;
    status_host[0] = status_host[1] = 0;
    if (b->n_pools == 0) return CFMM_OK;
    if (!b->weights || !b->logrw || !b->reserves || !out_records || !work) return CFMM_E_NULL;
    if (n_chg > 0 && (!pos || !n_rec || !records || !state)) return CFMM_E_NULL;
    const int64_t need = cfmm_ladder_splice_work_bytes(b->n_pools, n_chg);
    if (need < 0 || work_bytes < need) return CFMM_E_SIZE;
    if (!aligned16(b->weights) || !aligned16(out_records) || (records && !aligned16(records)) ||
        out_records == b->weights)
        return CFMM_E_SIZE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long m = b->n_pools, a = n_chg + 1;
    unsigned char* w = static_cast<unsigned char*>(work);
    auto take = [&](size_t bytes) { unsigned char* p = w; w += align_up(bytes); return p; };
    long long* status = reinterpret_cast<long long*>(take(16));
    long long* newcnt = reinterpret_cast<long long*>(take(8 * (size_t)a));
    long long* new_off = reinterpret_cast<long long*>(take(8 * (size_t)a));
    long long* cnt = reinterpret_cast<long long*>(take(8 * (size_t)(m + 1)));
    long long* src = reinterpret_cast<long long*>(take(8 * (size_t)(m + 1)));
    long long* first_new = reinterpret_cast<long long*>(take(8 * (size_t)(m + 1)));
    size_t t1 = scan_temp_bytes(a), t2 = scan_temp_bytes(m + 1);
    size_t temp_bytes = t1 > t2 ? t1 : t2;
    void* temp = take(temp_bytes);
    double* logrw = const_cast<double*>(b->logrw);
    double* reserves = const_cast<double*>(b->reserves);
    if (cudaMemsetAsync(status, 0, 16, st) != cudaSuccess) {
        g_last_err = cudaGetLastError();
        return CFMM_E_CUDA;
    }
    k_splice_check<<<grid_for(n_chg), 256, 0, st>>>(n_chg, m, R.rec_max, pos, n_rec, newcnt, status);
    int rc = check_launch();
    if (rc) return rc;
    if (cub::DeviceScan::ExclusiveSum(temp, temp_bytes, newcnt, new_off, (int)a, st) != cudaSuccess) {
        g_last_err = cudaGetLastError();
        return CFMM_E_CUDA;
    }
    k_splice_counts<<<grid_for(m), 256, 0, st>>>(m, b->stride, R.first, R.count, R.count_off, b->logrw, cnt, src);
    if ((rc = check_launch())) return rc;
    if (n_chg > 0) {
        k_splice_mark<<<grid_for(n_chg), 256, 0, st>>>(n_chg, m, pos, newcnt, new_off, cnt, src);
        if ((rc = check_launch())) return rc;
    }
    if (cub::DeviceScan::ExclusiveSum(temp, temp_bytes, cnt, first_new, (int)(m + 1), st) != cudaSuccess) {
        g_last_err = cudaGetLastError();
        return CFMM_E_CUDA;
    }
    k_splice_total<<<1, 1, 0, st>>>(n_chg, m, n_records, out_capacity, new_off, first_new, status);
    if ((rc = check_launch())) return rc;
    // the grid covers the output buffer's capacity; the kernel stops at the bucket's new total
    k_splice_copy<<<grid_for(out_capacity), 256, 0, st>>>(
        m, first_new, src, reinterpret_cast<const double2*>(b->weights), reinterpret_cast<const double2*>(records),
        reinterpret_cast<double2*>(out_records), status);
    if ((rc = check_launch())) return rc;
    k_splice_state<<<grid_for(m > n_chg ? m : n_chg), 256, 0, st>>>(m, n_chg, b->stride, R.first, R.count, R.count_off,
                                                                    R.s0, R.s1, first_new, pos, state, logrw, reserves,
                                                                    status);
    if ((rc = check_launch())) return rc;
    if (cudaMemcpyAsync(status_host, status, 16, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) {
        g_last_err = cudaGetLastError();
        return CFMM_E_CUDA;
    }
    return CFMM_OK;
}

}  // namespace

extern "C" {

/* work of cfmm_ladder_splice: status, the changed pools' counts and offsets, every pool's count, source and new first
 * record, and the scans' temporary storage */
int64_t cfmm_ladder_splice_work_bytes(int64_t n_pools, int64_t n_chg) {
    if (n_pools < 0 || n_chg < 0 || n_chg > n_pools || n_pools >= 0x7fffffffLL) return CFMM_E_SIZE;
    const size_t a = (size_t)n_chg + 1, m = (size_t)n_pools + 1;
    const size_t t1 = scan_temp_bytes((long long)a), t2 = scan_temp_bytes((long long)m);
    return (int64_t)(align_up(16) + 2 * align_up(8 * a) + 3 * align_up(8 * m) + align_up(t1 > t2 ? t1 : t2));
}

/* New records for n_chg pools of a concentrated bucket, spliced into out_records (include/cfmm_b200.h). */
int cfmm_ladder_splice(const cfmm_bucket* b, int64_t n_chg, const int64_t* pos, const int64_t* n_rec, const double* records,
                       int64_t n_records, const double* state, double* out_records, int64_t out_capacity,
                       int64_t* status_host, void* work, int64_t work_bytes, void* stream) {
    if (!b || !status_host) return CFMM_E_NULL;
    if (b->kind != CFMM_KIND_CONCENTRATED || b->arity != 2) return CFMM_E_KIND;
    return splice(kLadderRows, b, n_chg, pos, n_rec, records, n_records, state, out_records, out_capacity, status_host,
                  work, work_bytes, stream);
}

/* New records for n_chg pools of a price-bin bucket, spliced into out_records (include/cfmm_b200.h). */
int cfmm_bins_splice(const cfmm_bucket* b, int64_t n_chg, const int64_t* pos, const int64_t* n_rec, const double* records,
                     int64_t n_records, const double* state, double* out_records, int64_t out_capacity,
                     int64_t* status_host, void* work, int64_t work_bytes, void* stream) {
    if (!b || !status_host) return CFMM_E_NULL;
    if (b->kind != CFMM_KIND_BINS || b->arity != 2) return CFMM_E_KIND;
    return splice(kBinsRows, b, n_chg, pos, n_rec, records, n_records, state, out_records, out_capacity, status_host,
                  work, work_bytes, stream);
}

}  // extern "C"
