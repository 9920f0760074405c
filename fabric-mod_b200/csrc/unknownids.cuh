// fabgpu_block_unknown_identities: the distinct serialized identities a finished block looked up in the MSP table and did not find --
// the creators and endorsers the device could not decide (254), which the peer runs through its MSP before fabgpu_msp_identities_add.
// A miss is a signature job with tx != 0xffffffff whose resolved identity is -1 (resolve_job).  The steps below run on the slot's job
// records as the block left them, after the validator's kernels; all but the kernels are host+device, so the tests run them on the host.
//   uk_hash_job     one per job: sample_hash of a miss (0 otherwise)
//   uk_insert_job   one per job: a miss joins the open-addressing index, keyed by the job of its identity's representative; equal
//                   hashes are confirmed on the bytes, so distinct identities with one hash stay apart; atomicMin keeps each
//                   identity's first appearance (tx, k), creator (k = -1) before endorsers
//   uk_count_tx     one per transaction: the first appearances among its jobs
//   (scan)          exclusive offsets over the transactions
//   uk_emit_tx      one per transaction: (offset, length, tx) of each, in job order -- the order of first appearance
#pragma once
#include "blockdev.cuh"

namespace fabgpu { namespace bdev {

#define UK_EMPTY 0xffffffffu

struct UkArrays {
    const RawJob* raw; const int32_t* ident; const TxDev* txs;    // the block's job records, resolved identities and transactions
    uint32_t T, E_cap;                                            // transactions; endorsement-job capacity
    const uint32_t* n_end;                                        // endorsement jobs the walk handed out (may exceed E_cap)
    uint64_t* hash;                                               // [T + E_cap]
    uint32_t* index; uint32_t index_mask;                         // slots (power of two > 2 (T + E_cap)): representative job
    uint32_t* rep;                                                // [T + E_cap] per miss: its representative
    unsigned long long* first;                                    // [T + E_cap] per representative: smallest order of its identity
    uint32_t* cnt;                                                // [T + 1] first appearances per transaction, then offsets; [T] total
    uint32_t* out;                                                // 3 per listed identity: offset, length, first tx
};

BD_HD uint32_t uk_jobs(const UkArrays& a) { const uint32_t e = *a.n_end; return a.T + (e < a.E_cap ? e : a.E_cap); }
BD_HD bool uk_miss(const UkArrays& a, uint32_t j) { return a.raw[j].tx != 0xffffffffu && a.ident[j] < 0; }
BD_HD unsigned long long uk_order(const RawJob& r) { return ((unsigned long long)r.tx << 32) | (uint32_t)(r.k + 1); }

BD_HD uint32_t uk_cas(uint32_t* p, uint32_t cmp, uint32_t v)
{
#if defined(__CUDA_ARCH__)
    return atomicCAS(p, cmp, v);
#else
    const uint32_t o = *p; if (o == cmp) *p = v; return o;
#endif
}
BD_HD void uk_min(unsigned long long* p, unsigned long long v)
{
#if defined(__CUDA_ARCH__)
    atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}

BD_HD void uk_hash_job(const uint8_t* base, const UkArrays& a, uint32_t j)
{
    a.hash[j] = uk_miss(a, j) ? sample_hash(base + a.raw[j].ident.off, a.raw[j].ident.len) : 0;
    a.first[j] = ~0ull;
}

BD_HD void uk_insert_job(const uint8_t* base, const UkArrays& a, uint32_t j)
{
    if (a.hash[j] == 0) return;
    const Seg s = a.raw[j].ident;
    uint32_t r = j;
    for (uint32_t pos = (uint32_t)a.hash[j] & a.index_mask;; pos = (pos + 1) & a.index_mask) {
        const uint32_t o = uk_cas(&a.index[pos], UK_EMPTY, j);
        if (o == UK_EMPTY) break;
        if (a.hash[o] != a.hash[j]) continue;
        const Seg so = a.raw[o].ident;
        if (so.len == s.len && bytes_equal(base + so.off, base + s.off, s.len)) { r = o; break; }
    }
    a.rep[j] = r;
    uk_min(&a.first[r], uk_order(a.raw[j]));
}

// whether job j is the first appearance of its identity (after every uk_insert_job)
BD_HD bool uk_is_first(const UkArrays& a, uint32_t j) { return a.hash[j] != 0 && a.first[a.rep[j]] == uk_order(a.raw[j]); }

// job q of transaction t in first-appearance order: the creator job (t itself), then its endorsement jobs
BD_HD uint32_t uk_tx_job(const TxDev& tx, uint32_t t, uint32_t q) { return q == 0 ? t : tx.first_end_job + q - 1; }

BD_HD void uk_count_tx(const UkArrays& a, uint32_t t)
{
    const TxDev& tx = a.txs[t];
    uint32_t c = 0;
    for (uint32_t q = 0; q <= tx.n_end_jobs; q++) c += uk_is_first(a, uk_tx_job(tx, t, q));
    a.cnt[t] = c;
}

// after the scan: cnt[t] = the listed identities before transaction t
BD_HD void uk_emit_tx(const UkArrays& a, uint32_t t)
{
    const TxDev& tx = a.txs[t];
    uint32_t w = a.cnt[t];
    for (uint32_t q = 0; q <= tx.n_end_jobs; q++) {
        const uint32_t j = uk_tx_job(tx, t, q);
        if (!uk_is_first(a, j)) continue;
        a.out[3 * w] = a.raw[j].ident.off; a.out[3 * w + 1] = a.raw[j].ident.len; a.out[3 * w + 2] = t;
        w++;
    }
}

#if defined(__CUDACC__)
__global__ void __launch_bounds__(128) uk_hash_kernel(const uint8_t* __restrict__ block, UkArrays a)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < uk_jobs(a)) uk_hash_job(block, a, j);
}
__global__ void __launch_bounds__(128) uk_insert_kernel(const uint8_t* __restrict__ block, UkArrays a)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < uk_jobs(a)) uk_insert_job(block, a, j);
}
__global__ void __launch_bounds__(128) uk_count_kernel(UkArrays a)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.T) uk_count_tx(a, t);
}
// one CTA of 1024 threads: exclusive offsets over cnt[0, T), the total in cnt[T]
__global__ void __launch_bounds__(1024) uk_scan_kernel(UkArrays a)
{
    __shared__ uint32_t warp_sum[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, per = (a.T + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(a.T, tid * per), hi = min(a.T, lo + per);
    uint32_t c = 0;
    for (uint32_t t = lo; t < hi; t++) c += a.cnt[t];
    uint32_t x = c;
    for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t v = warp_sum[lane];
        for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += y; }
        warp_sum[lane] = v;
    }
    __syncthreads();
    uint32_t off = x - c + (warp ? warp_sum[warp - 1] : 0);
    for (uint32_t t = lo; t < hi; t++) { const uint32_t v = a.cnt[t]; a.cnt[t] = off; off += v; }
    if (tid == 0) a.cnt[a.T] = warp_sum[31];
}
__global__ void __launch_bounds__(128) uk_emit_kernel(UkArrays a)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.T) uk_emit_tx(a, t);
}
#endif

} }  // namespace fabgpu::bdev
