// The ledger's private-data check of a block (fabgpu_validate_pvtdata): validateAndPreparePvtBatch's check path
// (core/ledger/kvledger/txmgmt/validation/batch_preparer.go:119-188) over the private data the caller holds, one marshalled
// rwset.TxPvtReadWriteSet per transaction.  Host+device code: the tests' host build runs the same steps one item at a time.
//
// For each entry the outcome is computed as if its transaction were VALID:
//   skip      containsPvtWrites (types.go:49-58) is false: no CollectionHashedReadWriteSet of the public read/write set carries a
//             pvt_rwset_hash (:136-138).  A present but empty hash is non-nil under golang/protobuf v1.3.3 (recalled, unverified): a
//             transaction whose only hashes are such is 254 when the entry holds a collection, OK when it holds none.
//   mismatch  validatePvtdata (:166-181): through the entry's namespaces and their collections in order, the first collection whose
//             SHA-256(rwset) differs from retrieveHash(namespace, collection) (types.go:62-78: the public namespaces in order, those of
//             another name skipped, the first collection of that name; no hash, or no such collection, never matches).  Every hash of the
//             entry is checked before any rwset is decoded (:146-152).
//   254       TxPvtRwSetFromProtoMsg (:153-156, rwset_proto_util.go:266-303) unmarshals every rwset as a KVRWSet: a level the project's
//             reader refuses, or a string field that is not valid UTF-8, at the first such collection.  Also an entry whose outer levels
//             do not parse, or whose transaction's read/write set the walk never reached (a non-endorser transaction included).
// The block's verdict comes from the entry with the smallest SeqInBlock whose outcome is mismatch or 254 and whose flag is VALID or 254
// (:133-135 skips every other flag): a mismatch when its flag is VALID, else 254.
//
// Wire layout (rwset.proto, as recalled: the file is not in the reference tree): TxPvtReadWriteSet{data_model = 1, ns_pvt_rwset = 2},
// NsPvtReadWriteSet{namespace = 1, collection_pvt_rwset = 2}, CollectionPvtReadWriteSet{collection_name = 1, rwset = 2}.
#pragma once
#include "couchval.cuh"

namespace fabgpu { namespace bdev {

// an entry's or record's outcome (fabgpu_validate_pvtdata's status codes)
enum : uint8_t { PV_OK = 0, PV_MISMATCH = 1, PV_SKIP = 2, PV_UNDET = 254 };
// what the scan leaves per entry: records to check, skipped, 254 as a whole, or only present-but-empty public hashes
enum : uint8_t { PE_CHECK = 0, PE_SKIP = 1, PE_UNDET = 2, PE_EMPTY_HASH = 3 };
// a record's check: bit 0 = its hash does not match, bit 1 = its rwset does not decode
enum : uint8_t { PR_MISMATCH = 1, PR_UNDECODABLE = 2 };
#define PV_REC_HINT 4u             // collection records per entry the arrays are first sized for

struct ShaJobP { uint32_t off[3]; uint32_t len[3]; };  // sha256.cuh's ShaJob

// One CollectionPvtReadWriteSet of an entry; segments are offsets into the private-data buffer
struct PvRec {
    Seg ns, coll, rw;
    uint32_t entry, ns_i, coll_i;
    uint8_t check;                 // PR_* bits, set by pv_check_rec
};

struct PvArrays {
    const uint8_t* pvt;            // the entries back to back
    const uint32_t* off;           // n_pvt + 1
    const uint32_t* seq;           // n_pvt: SeqInBlock of each entry
    uint32_t n_pvt;
    const uint8_t* flags;          // T final flags
    uint8_t* ent;                  // n_pvt: PE_*
    uint32_t* first; uint32_t* n_rec;   // n_pvt: records [first, first + n_rec) of the entry, in order
    PvRec* rec; uint32_t R_cap;
    ShaJobP* jobs;                 // R_cap: SHA-256 of each record's rwset
    const uint8_t* dig;            // R_cap x 32
    uint32_t* ctr;                 // [0]: records handed out (> R_cap: overflow)
    int32_t* status;               // 3 x n_pvt: code, namespace index, collection index
    unsigned long long* verdict;   // (seq << 32) | entry of the deciding entry, all ones = none
};

BD_HD bool pv_seg_eq(const uint8_t* a, Seg x, const uint8_t* b, Seg y)
{
    if (x.len != y.len) return false;
    for (uint32_t i = 0; i < x.len; i++) if (a[x.off + i] != b[y.off + i]) return false;
    return true;
}

// containsPvtWrites over a parsed TxReadWriteSet: PE_CHECK (some hash non-empty), PE_EMPTY_HASH (present hashes, all empty), PE_SKIP.
// NsReadWriteSet{collection_hashed_rwset = 3}, CollectionHashedReadWriteSet{pvt_rwset_hash = 3}: the last occurrence is the field.
BD_HD uint8_t pv_contains(const uint8_t* base, Seg results)
{
    bool present = false, nonempty = false;
    scan_msg(base, results, BD_F(2), BD_F(1), [&](uint32_t, Seg nsb) {
        scan_msg(base, nsb, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t f, Seg cb) {
            if (f != 3) return;
            bool has = false; Seg h; h.off = h.len = 0;
            scan_msg(base, cb, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t g, Seg c) { if (g == 3) { has = true; h = c; } });
            if (has) { present = true; if (h.len) nonempty = true; }
        });
    });
    return nonempty ? PE_CHECK : present ? PE_EMPTY_HASH : PE_SKIP;
}

// retrieveHash(ns, coll) == digest (types.go:62-78); ns and coll are segments of the private-data buffer
BD_HD bool pv_hash_matches(const uint8_t* blk, Seg results, const uint8_t* pvt, Seg ns, Seg coll, const uint8_t* digest)
{
    bool found = false, has = false; Seg hash; hash.off = hash.len = 0;
    scan_msg(blk, results, BD_F(2), BD_F(1), [&](uint32_t, Seg nsb) {
        if (found) return;
        Seg name; name.off = name.len = 0;
        scan_msg(blk, nsb, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t f, Seg b) { if (f == 1) name = b; });
        if (!pv_seg_eq(blk, name, pvt, ns)) return;
        scan_msg(blk, nsb, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t f, Seg cb) {
            if (found || f != 3) return;
            Seg cname, h; cname.off = cname.len = h.off = h.len = 0; bool hh = false;
            scan_msg(blk, cb, BD_F(1) | BD_F(2) | BD_F(3), 0, [&](uint32_t g, Seg c) { if (g == 1) cname = c; else if (g == 3) { h = c; hh = true; } });
            if (pv_seg_eq(blk, cname, pvt, coll)) { found = true; has = hh; hash = h; }
        });
    });
    if (!found || !has || hash.len != 32) return false;
    for (uint32_t i = 0; i < 32; i++) if (blk[hash.off + i] != digest[i]) return false;
    return true;
}

BD_HD bool pv_str(const uint8_t* base, Seg s) { return cv_utf8(base + s.off, s.len); }

// KVRead{key = 1, version = 2}, Version{block_num = 1, tx_num = 2}
BD_HD bool pv_read(const uint8_t* base, Seg r)
{
    bool ok = true;
    if (!scan_msg(base, r, BD_F(1) | BD_F(2), 0, [&](uint32_t h, Seg c) {
            if (h == 1) ok = ok && pv_str(base, c);
            else ok = ok && scan_msg(base, c, 0, BD_F(1) | BD_F(2), [](uint32_t, Seg) {}); })) return false;
    return ok;
}

// proto.Unmarshal of a KVRWSet{reads = 1, range_queries_info = 2, writes = 3, metadata_writes = 4} with every nested level:
// RangeQueryInfo{start_key = 1, end_key = 2, itr_exhausted = 3, raw_reads = 4, reads_merkle_hashes = 5}, QueryReads{kv_reads = 1},
// QueryReadsMerkleSummary{max_degree = 1, max_level = 2, max_level_hashes = 3}, KVWrite{key = 1, is_delete = 2, value = 3},
// KVMetadataWrite{key = 1, entries = 2}, KVMetadataEntry{name = 1, value = 2}.  false: a level does not parse, or a string is not UTF-8.
// on_write(field, body) is handed each KVWrite (field 3) and KVMetadataWrite (field 4) in wire order once its level has been read -- the
// private update batch (pvtupdates.cuh) walks the writes of rwsets the check found decodable; the check itself passes none.
struct PvNoWrites { BD_HD void operator()(uint32_t, Seg) const {} };
template <typename W = PvNoWrites>
BD_HD bool pv_decode(const uint8_t* base, Seg rw, W on_write = W())
{
    bool ok = true;
    auto none = [](uint32_t, Seg) {};
    if (!scan_msg(base, rw, BD_F(1) | BD_F(2) | BD_F(3) | BD_F(4), 0, [&](uint32_t g, Seg b) {
            if (!ok) return;
            if (g == 1) ok = pv_read(base, b);
            else if (g == 2)
                ok = scan_msg(base, b, BD_F(1) | BD_F(2) | BD_F(4) | BD_F(5), BD_F(3), [&](uint32_t h, Seg c) {
                    if (!ok) return;
                    if (h == 1 || h == 2) ok = pv_str(base, c);
                    else if (h == 4) ok = scan_msg(base, c, BD_F(1), 0, [&](uint32_t, Seg kv) { ok = ok && pv_read(base, kv); }) && ok;
                    else ok = scan_msg(base, c, BD_F(3), BD_F(1) | BD_F(2), none);
                }) && ok;
            else if (g == 3) {
                ok = scan_msg(base, b, BD_F(1) | BD_F(3), BD_F(2), [&](uint32_t h, Seg c) { if (h == 1) ok = ok && pv_str(base, c); }) && ok;
                if (ok) on_write(g, b);
            } else {
                ok = scan_msg(base, b, BD_F(1) | BD_F(2), 0, [&](uint32_t h, Seg c) {
                    if (h == 1) ok = ok && pv_str(base, c);
                    else ok = ok && scan_msg(base, c, BD_F(1) | BD_F(2), 0, [&](uint32_t q, Seg d) { if (q == 1) ok = ok && pv_str(base, d); });
                }) && ok;
                if (ok) on_write(g, b);
            }
        })) return false;
    return ok;
}

// The collections of one entry in order: on_coll(ns, coll, rwset, ns_i, coll_i).  A namespace's and a collection's fields are read in
// full before its collections are handed over (a later occurrence of a singular field wins).  false: an outer level does not parse, or
// a namespace or collection name is not UTF-8.
template <typename F>
BD_HD bool pv_entry_scan(const uint8_t* pvt, Seg entry, F on_coll)
{
    bool ok = true; uint32_t ns_i = 0;
    const bool top = scan_msg(pvt, entry, BD_F(2), BD_F(1), [&](uint32_t, Seg nsb) {
        if (!ok) return;
        Seg name; name.off = name.len = 0;
        if (!scan_msg(pvt, nsb, BD_F(1) | BD_F(2), 0, [&](uint32_t f, Seg b) { if (f == 1) { name = b; ok = ok && pv_str(pvt, b); } }) || !ok) { ok = false; return; }
        uint32_t coll_i = 0;
        scan_msg(pvt, nsb, BD_F(2), 0, [&](uint32_t, Seg cb) {
            if (!ok) return;
            Seg cname, rw; cname.off = cname.len = rw.off = rw.len = 0;
            if (!scan_msg(pvt, cb, BD_F(1) | BD_F(2), 0, [&](uint32_t g, Seg c) { if (g == 1) { cname = c; ok = ok && pv_str(pvt, c); } else rw = c; }) || !ok) {
                ok = false; return;
            }
            on_coll(name, cname, rw, ns_i, coll_i++);
        });
        ns_i++;
    });
    return top && ok;
}

// Stage 1, one thread per entry: the entry's collection records and SHA-256 jobs, and what the public read/write set says of it
BD_HD void pv_scan_entry(const uint8_t* blk, const TxDev* txs, uint32_t e, PvArrays& a)
{
    a.first[e] = 0; a.n_rec[e] = 0;
    const TxDev& tx = txs[a.seq[e]];
    Seg entry; entry.off = a.off[e]; entry.len = a.off[e + 1] - a.off[e];
    uint32_t n = 0;
    if (!mv_reached(tx) || !kl_scan_rwset<true>(blk, tx.results, [](Seg, Seg, Seg, uint32_t, Seg) { return true; }) ||
        !pv_entry_scan(a.pvt, entry, [&](Seg, Seg, Seg, uint32_t, uint32_t) { n++; })) {
        a.ent[e] = PE_UNDET;
        return;
    }
    a.ent[e] = pv_contains(blk, tx.results);
    if (a.ent[e] == PE_SKIP || n == 0) return;
    const uint32_t b = kl_atomic_add(a.ctr, n);
    if (b + n > a.R_cap || b + n < b) return;                        // overflow: the host grows the arrays and runs the scan again
    a.first[e] = b; a.n_rec[e] = n;
    uint32_t q = b;
    pv_entry_scan(a.pvt, entry, [&](Seg ns, Seg coll, Seg rw, uint32_t ns_i, uint32_t coll_i) {
        PvRec& r = a.rec[q];
        r.ns = ns; r.coll = coll; r.rw = rw; r.entry = e; r.ns_i = ns_i; r.coll_i = coll_i; r.check = 0;
        ShaJobP& j = a.jobs[q];
        j.off[0] = rw.off; j.len[0] = rw.len; j.off[1] = j.len[1] = j.off[2] = j.len[2] = 0;
        q++;
    });
}

// Stage 2, one thread per record (after the SHA-256 of its rwset): the public hash, then the decode
BD_HD void pv_check_rec(const uint8_t* blk, const TxDev* txs, uint32_t i, PvArrays& a)
{
    PvRec& r = a.rec[i];
    const TxDev& tx = txs[a.seq[r.entry]];
    uint8_t c = 0;
    if (!pv_hash_matches(blk, tx.results, a.pvt, r.ns, r.coll, a.dig + 32 * (size_t)i)) c |= PR_MISMATCH;
    if (!pv_decode(a.pvt, r.rw)) c |= PR_UNDECODABLE;
    r.check = c;
}

// Stage 3, one thread per entry: its outcome (the first mismatch in record order, else the first undecodable rwset) and its bid for the
// block's verdict
BD_HD void pv_verdict_entry(uint32_t e, PvArrays& a)
{
    int32_t code = PV_OK, ns = -1, coll = -1;
    const uint8_t st = a.ent[e];
    if (st == PE_UNDET) code = PV_UNDET;
    else if (st == PE_SKIP) code = PV_SKIP;
    else if (st == PE_EMPTY_HASH && a.n_rec[e]) code = PV_UNDET;
    else {
        for (uint32_t k = 0; k < a.n_rec[e] && code == PV_OK; k++) {
            const PvRec& r = a.rec[a.first[e] + k];
            if (r.check & PR_MISMATCH) { code = PV_MISMATCH; ns = (int32_t)r.ns_i; coll = (int32_t)r.coll_i; }
        }
        for (uint32_t k = 0; k < a.n_rec[e] && code == PV_OK; k++) {
            const PvRec& r = a.rec[a.first[e] + k];
            if (r.check & PR_UNDECODABLE) { code = PV_UNDET; ns = (int32_t)r.ns_i; coll = (int32_t)r.coll_i; }
        }
    }
    a.status[3 * e] = code; a.status[3 * e + 1] = ns; a.status[3 * e + 2] = coll;
    const uint8_t f = a.flags[a.seq[e]];
    if ((code == PV_MISMATCH || code == PV_UNDET) && (f == TXC_VALID || f == TXC_NOT_VALIDATED)) {
        const unsigned long long me = ((unsigned long long)a.seq[e] << 32) | e;
#if defined(__CUDA_ARCH__)
        atomicMin(a.verdict, me);
#else
        if (me < *a.verdict) *a.verdict = me;
#endif
    }
}

#if defined(__CUDACC__)
__global__ void __launch_bounds__(64)
pv_scan_kernel(const uint8_t* __restrict__ block, const TxDev* __restrict__ txs, PvArrays a)
{
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < a.n_pvt) pv_scan_entry(block, txs, e, a);
}

__global__ void __launch_bounds__(128)
pv_check_kernel(const uint8_t* __restrict__ block, const TxDev* __restrict__ txs, PvArrays a, uint32_t R)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < R) pv_check_rec(block, txs, i, a);
}

__global__ void __launch_bounds__(128)
pv_verdict_kernel(PvArrays a)
{
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < a.n_pvt) pv_verdict_entry(e, a);
}
#endif

} }  // namespace fabgpu::bdev
