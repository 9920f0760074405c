// The block's deterministic update bytes (fabgpu_block_update_bytes): what deterministicBytesForPubAndHashUpdates
// (core/ledger/kvledger/txmgmt/txmgr/update_batch_bytes.go:29-105) returns for the batch fabgpu_block_updates hands back, the input of
// the block's commit hash.  proto.Marshal(Updates{kvwrites = 1}) of one KVWrite{namespace = 1, collection = 2, key = 3, isDelete = 4,
// value = 5, version_bytes = 6} per record (txmgr/updates.proto); proto3, so an empty string or bytes field and a false bool are left
// out.  Host+device code: the tests' host build runs the same steps one item at a time.
//
// Order: namespaces bytewise, namespace "" (the channel config, :39-44) skipped; within a namespace its public keys, then its
// collections by name, keys bytewise within each (sort.Strings, util.GetSortedKeys).  One merge sort of the records by (namespace,
// collection, key) gives that order, since a public record's collection is empty and sorts first: the rank merge of stateindex.cuh
// over UbItem, with the record index as the last key so that every item is distinct.  Namespace-"" records sort to the front and emit
// nothing.  namespace is set on the first KVWrite of each namespace (:50), collection on the first of each collection (:72).
// version_bytes is Height{block_num, tx}.ToBytes() (internal/version/version.go:50-54): EncodeOrderPreservingVarUint64 of both
// (common/ledger/util/util.go:32-52), a length byte then the big-endian bytes without leading zeros.
#pragma once
#include "updates.cuh"
#include "couchval.cuh"

namespace fabgpu { namespace bdev {

constexpr uint32_t UB_SHORT = 2048;     // a value up to this long is copied by its record's warp (ub_emit_kernel)
constexpr uint32_t UB_CHUNK = 16384;    // a longer one by one CTA per chunk of this many bytes (ub_long_kernel)

// One record of the batch as the sort sees it: byte ranges in the block, and its index in fabgpu_block_updates' records
struct UbItem { uint32_t ns_off, nl, coll_off, cl, key_off, kl, rec; };
struct UbRef { const uint8_t* ns; uint32_t nl; const uint8_t* coll; uint32_t cl; const uint8_t* key; uint32_t kl; uint32_t rec; };

BD_HD UbRef key_ref(const uint8_t* src, const UbItem& e)
{
    UbRef r; r.ns = src + e.ns_off; r.nl = e.nl; r.coll = src + e.coll_off; r.cl = e.cl; r.key = src + e.key_off; r.kl = e.kl; r.rec = e.rec;
    return r;
}
BD_HD int key_cmp(const UbRef& a, const UbRef& b)
{
    int c = bytes_cmp(a.ns, a.nl, b.ns, b.nl);
    if (!c) c = bytes_cmp(a.coll, a.cl, b.coll, b.cl);
    if (!c) c = bytes_cmp(a.key, a.kl, b.key, b.kl);
    return c ? c : a.rec == b.rec ? 0 : a.rec < b.rec ? -1 : 1;
}

struct UbArrays {
    const uint32_t* rec; uint32_t n;    // fabgpu_block_updates' records (UD_WORDS words each) and their count
    const uint8_t* blk;                 // the bytes the slot's block was submitted in
    UbItem* item;                       // per record; after the sort, per sorted position
    uint32_t* cidx;                     // per record: its index among the COMMITTED-value records, in record order
    const uint8_t* cval; const uint32_t* coff;   // the caller's committed values: value j is cval[coff[j] .. coff[j + 1])
    unsigned long long block_num;
    unsigned long long* off;            // n + 1, per sorted position: the framed KVWrite's length, then its offset (exclusive scan; [n] total)
    uint32_t* chunk;                    // n + 1, per sorted position: UB_CHUNK chunks of a long value, then the first one's index ([n] total)
    uint8_t* out;
    uint32_t* ctr;                      // [0] incomplete (an emitted name is not UTF-8), [1] COMMITTED-value records
};

// Where a KVWrite's pieces go: whether it names its namespace and collection, its value, its version bytes, its body length, and the
// offset of its value bytes from the start of the framed KVWrite
struct UbLayout {
    bool fns, fcoll, del; const uint8_t* val; uint32_t vl; uint8_t ver[18]; uint32_t verl; unsigned long long body, vat;
};

BD_HD uint32_t ub_vlen(unsigned long long v) { uint32_t n = 1; while (v >= 0x80) { v >>= 7; n++; } return n; }

// EncodeOrderPreservingVarUint64: 0 is the single byte 0x00, 256 is 02 01 00
BD_HD uint32_t ub_height_part(unsigned long long v, uint8_t* o)
{
    uint32_t size = 0;
    for (unsigned long long x = v; x; x >>= 8) size++;
    o[0] = (uint8_t)size;
    for (uint32_t k = 0; k < size; k++) o[1 + k] = (uint8_t)(v >> (8 * (size - 1 - k)));
    return 1 + size;
}

// Step 1, one thread per record: its sort item, and whether its value comes from the caller
BD_HD bool ub_item_rec(uint32_t i, UbArrays& a)
{
    const uint32_t* w = a.rec + (size_t)i * UD_WORDS;
    UbItem& e = a.item[i];
    e.ns_off = w[4]; e.nl = w[5]; e.coll_off = w[6]; e.cl = w[7]; e.key_off = w[8]; e.kl = w[9]; e.rec = i;
    return w[2] == UD_COMMITTED;
}

// Steps 2 (the sort passes, ri_sort_one) and 3 (cidx, an exclusive scan of ub_item_rec's answer) are in the kernels and the host build.

BD_HD void ub_layout(uint32_t p, const UbArrays& a, UbLayout& L)
{
    const UbItem& e = a.item[p];
    const uint32_t* w = a.rec + (size_t)e.rec * UD_WORDS;
    if (p == 0) L.fns = L.fcoll = true;
    else {
        const UbItem& q = a.item[p - 1];
        L.fns = bytes_cmp(a.blk + e.ns_off, e.nl, a.blk + q.ns_off, q.nl) != 0;
        L.fcoll = L.fns || bytes_cmp(a.blk + e.coll_off, e.cl, a.blk + q.coll_off, q.cl) != 0;
    }
    L.fcoll = L.fcoll && e.cl;
    L.del = w[1] == UD_DELETE;
    L.val = nullptr; L.vl = 0;
    if (w[2] == UD_BLOCK) { L.val = a.blk + w[10]; L.vl = w[11]; }
    else if (w[2] == UD_COMMITTED) { const uint32_t j = a.cidx[e.rec]; L.val = a.cval + a.coff[j]; L.vl = a.coff[j + 1] - a.coff[j]; }
    L.verl = ub_height_part(a.block_num, L.ver);
    L.verl += ub_height_part(w[0], L.ver + L.verl);
    unsigned long long b = 0;
    if (L.fns) b += 1 + ub_vlen(e.nl) + e.nl;
    if (L.fcoll) b += 1 + ub_vlen(e.cl) + e.cl;
    if (e.kl) b += 1 + ub_vlen(e.kl) + e.kl;
    if (L.del) b += 2;
    L.vat = 0;
    if (L.vl) { b += 1 + ub_vlen(L.vl); L.vat = b; b += L.vl; }
    b += 2 + L.verl;
    L.body = b;
    L.vat += 1 + ub_vlen(b);
}

// Step 4, one thread per sorted position: the framed KVWrite's length (0 for namespace ""), the chunks of a long value, and the UTF-8
// check of the names it emits (proto.Marshal fails on a proto3 string that is not valid UTF-8)
BD_HD void ub_size(uint32_t p, UbArrays& a)
{
    const UbItem& e = a.item[p];
    a.off[p] = 0; a.chunk[p] = 0;
    if (!e.nl) return;
    UbLayout L; ub_layout(p, a, L);
    if ((L.fns && !cv_utf8(a.blk + e.ns_off, e.nl)) || (L.fcoll && !cv_utf8(a.blk + e.coll_off, e.cl))) a.ctr[0] = 1;
    a.off[p] = 1 + ub_vlen(L.body) + L.body;
    if (L.vl > UB_SHORT) a.chunk[p] = (L.vl + UB_CHUNK - 1) / UB_CHUNK;
}

// Step 5 (off and chunk to exclusive scans) is in the kernels and the host build.

// A tag and a varint length at o + at (written by the lane that writes); returns the offset after them
BD_HD unsigned long long ub_tag(uint8_t* o, unsigned long long at, uint8_t tag, unsigned long long len, bool write)
{
    const uint32_t n = ub_vlen(len);
    if (write) {
        o[at] = tag;
        for (uint32_t k = 0; k < n; k++, len >>= 7) o[at + 1 + k] = (uint8_t)(k + 1 < n ? (len & 0x7f) | 0x80 : len);
    }
    return at + 1 + n;
}

BD_HD void ub_copy(uint8_t* d, const uint8_t* s, unsigned long long n, uint32_t lane, uint32_t lanes)
{
    for (unsigned long long j = lane; j < n; j += lanes) d[j] = s[j];
}

// Step 6, per sorted position, by `lanes` cooperating lanes: the framed KVWrite at its offset (a long value's bytes: step 7)
BD_HD void ub_emit(uint32_t p, const UbArrays& a, uint32_t lane, uint32_t lanes)
{
    const UbItem& e = a.item[p];
    if (!e.nl) return;
    UbLayout L; ub_layout(p, a, L);
    uint8_t* o = a.out + a.off[p];
    const bool w0 = lane == 0;
    unsigned long long at = ub_tag(o, 0, 0x0a, L.body, w0);
    if (L.fns) { at = ub_tag(o, at, 0x0a, e.nl, w0); ub_copy(o + at, a.blk + e.ns_off, e.nl, lane, lanes); at += e.nl; }
    if (L.fcoll) { at = ub_tag(o, at, 0x12, e.cl, w0); ub_copy(o + at, a.blk + e.coll_off, e.cl, lane, lanes); at += e.cl; }
    if (e.kl) { at = ub_tag(o, at, 0x1a, e.kl, w0); ub_copy(o + at, a.blk + e.key_off, e.kl, lane, lanes); at += e.kl; }
    if (L.del) { if (w0) { o[at] = 0x20; o[at + 1] = 1; } at += 2; }
    if (L.vl) { at = ub_tag(o, at, 0x2a, L.vl, w0); if (L.vl <= UB_SHORT) ub_copy(o + at, L.val, L.vl, lane, lanes); at += L.vl; }
    at = ub_tag(o, at, 0x32, L.verl, w0);
    if (w0) for (uint32_t k = 0; k < L.verl; k++) o[at + k] = L.ver[k];
}

// Step 7, per chunk of the long values, by `lanes` cooperating lanes: the position holding chunk c (the last one whose first chunk is
// not above c), and that chunk's bytes of its value
BD_HD void ub_long(uint32_t c, const UbArrays& a, uint32_t lane, uint32_t lanes)
{
    uint32_t lo = 0, hi = a.n;
    while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (a.chunk[mid] <= c) lo = mid + 1; else hi = mid; }
    const uint32_t p = lo - 1;
    UbLayout L; ub_layout(p, a, L);
    const unsigned long long from = (unsigned long long)(c - a.chunk[p]) * UB_CHUNK;
    const unsigned long long n = L.vl - from < UB_CHUNK ? L.vl - from : UB_CHUNK;
    ub_copy(a.out + a.off[p] + L.vat + from, L.val + from, n, lane, lanes);
}

#if defined(__CUDACC__)
// One CTA: exclusive block-wide scan of (x, y) over each thread's contiguous chunk; the thread's offsets and the totals
__device__ __forceinline__ void ub_block_scan(unsigned long long x, uint32_t y, unsigned long long& ox, uint32_t& oy, unsigned long long& tx_,
                                              uint32_t& ty)
{
    __shared__ unsigned long long sx[32]; __shared__ uint32_t sy[32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long vx = x; uint32_t vy = y;
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const unsigned long long a = __shfl_up_sync(0xffffffffu, vx, d); const uint32_t b = __shfl_up_sync(0xffffffffu, vy, d);
        if (lane >= d) { vx += a; vy += b; }
    }
    if (lane == 31) { sx[warp] = vx; sy[warp] = vy; }
    __syncthreads();
    if (warp == 0) {
        unsigned long long wx = lane < blockDim.x / 32 ? sx[lane] : 0; uint32_t wy = lane < blockDim.x / 32 ? sy[lane] : 0;
        for (uint32_t d = 1; d < 32; d <<= 1) {
            const unsigned long long a = __shfl_up_sync(0xffffffffu, wx, d); const uint32_t b = __shfl_up_sync(0xffffffffu, wy, d);
            if (lane >= d) { wx += a; wy += b; }
        }
        sx[lane] = wx; sy[lane] = wy;
    }
    __syncthreads();
    ox = vx - x + (warp ? sx[warp - 1] : 0); oy = vy - y + (warp ? sy[warp - 1] : 0);
    tx_ = sx[31]; ty = sy[31];
    __syncthreads();
}

__global__ void __launch_bounds__(256) ub_item_kernel(UbArrays a)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.n) a.cidx[i] = ub_item_rec(i, a) ? 1u : 0u;
}

__global__ void __launch_bounds__(256) ub_sort_kernel(const UbItem* __restrict__ in, UbItem* __restrict__ out, uint32_t n, uint32_t width,
                                                      const uint8_t* __restrict__ block)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ri_sort_one(in, i, n, width, block, out);
}

// One CTA of 1024: cidx from 0/1 to each record's index among the COMMITTED-value records; ctr[1] their count
__global__ void __launch_bounds__(1024) ub_cscan_kernel(UbArrays a)
{
    const uint32_t per = (a.n + blockDim.x - 1) / blockDim.x, lo = min(a.n, threadIdx.x * per), hi = min(a.n, lo + per);
    uint32_t c = 0;
    for (uint32_t i = lo; i < hi; i++) c += a.cidx[i];
    unsigned long long u0, u1; uint32_t off, tot;
    ub_block_scan(0, c, u0, off, u1, tot);
    for (uint32_t i = lo; i < hi; i++) { const uint32_t f = a.cidx[i]; a.cidx[i] = off; off += f; }
    if (threadIdx.x == 0) a.ctr[1] = tot;
}

__global__ void __launch_bounds__(256) ub_size_kernel(UbArrays a)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < a.n) ub_size(p, a);
}

// One CTA of 1024: off and chunk to exclusive scans, the totals at [n]
__global__ void __launch_bounds__(1024) ub_scan_kernel(UbArrays a)
{
    const uint32_t per = (a.n + blockDim.x - 1) / blockDim.x, lo = min(a.n, threadIdx.x * per), hi = min(a.n, lo + per);
    unsigned long long b = 0; uint32_t c = 0;
    for (uint32_t p = lo; p < hi; p++) { b += a.off[p]; c += a.chunk[p]; }
    unsigned long long ob, tb; uint32_t oc, tc;
    ub_block_scan(b, c, ob, oc, tb, tc);
    for (uint32_t p = lo; p < hi; p++) {
        const unsigned long long x = a.off[p]; const uint32_t y = a.chunk[p];
        a.off[p] = ob; a.chunk[p] = oc; ob += x; oc += y;
    }
    if (threadIdx.x == 0) { a.off[a.n] = tb; a.chunk[a.n] = tc; }
}

// One warp per sorted position
__global__ void __launch_bounds__(256) ub_emit_kernel(UbArrays a)
{
    const uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (p < a.n) ub_emit(p, a, threadIdx.x & 31, 32);
}

// One CTA per chunk of the long values
__global__ void __launch_bounds__(256) ub_long_kernel(UbArrays a)
{
    ub_long(blockIdx.x, a, threadIdx.x, blockDim.x);
}
#endif

} }  // namespace fabgpu::bdev
