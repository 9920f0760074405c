// The block's private update batch (fabgpu_block_pvt_updates): what validateAndPreparePvtBatch leaves in PvtUpdates for the transactions
// the MVCC stage left VALID (core/ledger/kvledger/txmgmt/validation/batch_preparer.go:119-160, 341-410).  Host+device code: the tests'
// host build runs the same steps one item at a time.
//
// Built from the check's collection records (pvtdata.cuh: PvRec, each rwset's segment already known) of the entries whose transaction is
// VALID and whose check passed, and from the hashed batch fabgpu_block_updates resolved (updates.cuh: UdKey per entry of the stage's
// block key table).
//   writes     addPvtRWSetToPvtUpdateBatch (:341-353): every KVWrite of the entry in wire order (pv_decode's walk), a Put of its value or a
//              Delete at (block, tx).  The batch is a map keyed on (ns, coll, key): here a hash table keyed on the key identity digest
//              (stateset.cuh), whose last writer -- the largest (tx, position among the entry's writes) -- is found with atomicMax, and
//              the first position of the key among that transaction's writes orders the records.  A Put of an absent value panics in
//              PutValAndMetadata (statedb.go:202-207): the batch is left to the peer.
//   renewals   incrementPvtdataVersionIfNeeded (:360-393) over the keys of every private KVMetadataWrite (:401-410), one per key: the hashed
//              record of (ns, coll, SHA-256(key)) is found with mv_find_key in the stage's key table.  No PUT there (nothing, a dropped
//              write, a DELETE -- bytes.Equal(hash, nil) never holds): nothing.  The key not in the private batch: a RENEW record, which
//              the peer resolves with GetPrivateData.  In the batch at another version: SHA-256 of its value (of nothing for a Delete)
//              against the hashed value hash from the block -- equal renews the record's version to the hashed record's, or, for a
//              Delete, is the reference's Put of a nil value (a panic: the batch is left to the peer); a value hash from the committed
//              state also leaves the batch to the peer.
#pragma once
#include "updates.cuh"
#include "pvtdata.cuh"

namespace fabgpu { namespace bdev {

enum : uint8_t { PK_PUT = 1, PK_DEL = 2, PK_META = 3 };              // item kinds
enum : uint32_t { PU_RENEW = 3 };                                   // record ops: UD_PUT, UD_DELETE, PU_RENEW (FABGPU_UPDATE_*)
constexpr uint32_t PU_WORDS = 11;
#define PU_W_HINT 4u               // private writes per entry the arrays are first sized for
#define PU_M_HINT 1u               // private metadata writes per entry

// One KVWrite or KVMetadataWrite of a VALID entry; segments are offsets into the private-data buffer
struct PuItem {
    uint32_t w[8];                 // the key identity digest of (ns, coll, key)
    Seg ns, coll, key, val;        // val: a write's value (the last field 3), when has_val
    uint32_t tx, pos;              // the transaction; the position among the entry's writes (metadata writes: among its metadata writes)
    uint32_t slot;                 // the key's entry of the table
    uint8_t kind, has_val, pad[2];
};

// One private key of the block.  tag: txid_mix of the digest (0 = empty), claimed by CAS; w written by the claimer.
struct PuKey {
    unsigned long long tag;
    unsigned long long last;       // ((tx << 32) | position) + 1 of the last write (0: only metadata writes)
    uint32_t w[8];
    uint32_t nfirst;               // UINT32_MAX - the key's first position among the last writer's writes
    uint32_t lrec;                 // the last write's item
    uint32_t nmeta;                // UINT32_MAX - the metadata write that stands for the key (its lowest item; 0: none)
    uint32_t hk;                   // the hashed key-table entry + 1 whose value hash the latest value is compared with (0: none)
    uint32_t renew;                // the version is renewed to the hashed record's
    uint32_t pad;
};

struct PuArrays {
    const uint8_t* pvt; const uint32_t* seq; uint32_t n_pvt, T;
    const uint8_t* flags;          // T: the stage's final flags
    const int32_t* status;         // the check's outcomes (3 per entry)
    const PvRec* rec; const uint32_t* first; const uint32_t* n_rec;   // the check's collection records
    uint32_t* wfirst; uint32_t* mfirst;   // per entry: its first write / metadata-write item
    uint32_t* tbase;               // per transaction: its write count, then (pu_base) its first write's position in transaction order
    PuItem* item; uint32_t W_cap;  // writes
    PuItem* meta; uint32_t M_cap;  // metadata writes
    ShaJobP* jobs; const uint8_t* dig;   // M_cap: SHA-256 of each metadata write's key, then of the latest value its key compares
    PuKey* key; uint32_t P_size; uint64_t seed;   // P_size: power of two >= 2 (W + M)
    // the hashed batch: the stage's block key table, fabgpu_block_updates' keys (ukey == nullptr: it has no record), segments and order
    MvccArrays stage; uint64_t stage_seed;
    const UdKey* ukey; const UdSeg* useg; const uint32_t* uokey; uint32_t n_h;
    const uint8_t* blk;            // the block (hashed value hashes)
    uint32_t* rmark;               // per hashed key-table entry: the private key entry + 1 of its RENEW record
    uint32_t* mark;                // per write position in transaction order: the key entry + 1 of the record placed there
    uint32_t* out_key;             // per record: its key entry (PUT / DELETE) or its hashed record's index (RENEW)
    uint32_t* out;                 // PU_WORDS words per record
    uint32_t* ctr;                 // [0] writes handed out (> W_cap: overflow), [1] metadata writes (> M_cap), [2] incomplete,
                                   // [3] PUT / DELETE records, [4] RENEW records
};

BD_HD void pu_incomplete(PuArrays& a) { a.ctr[2] = 1; }

BD_HD bool pu_eligible(uint32_t e, const PuArrays& a) { return a.flags[a.seq[e]] == TXC_VALID && a.status[3 * e] == PV_OK; }

// Every write and metadata write of entry e, in wire order: on(field, ns, coll, body) -- field 3 a KVWrite, 4 a KVMetadataWrite
template <typename F>
BD_HD void pu_walk(uint32_t e, const PuArrays& a, F on)
{
    for (uint32_t k = 0; k < a.n_rec[e]; k++) {
        const PvRec& r = a.rec[a.first[e] + k];
        pv_decode(a.pvt, r.rw, [&](uint32_t g, Seg body) { on(g, r.ns, r.coll, body); });
    }
}

// KVWrite{key = 1, is_delete = 2, value = 3} / KVMetadataWrite{key = 1, entries = 2} of a decodable rwset: the last occurrence of each
// field, as proto.Unmarshal keeps it; has: the value field is present (absent: a nil value; present but empty: []byte{})
BD_HD void pu_fields(const uint8_t* base, Seg body, bool md, PuItem& it, bool& del)
{
    it.key.off = it.key.len = it.val.off = it.val.len = 0; it.has_val = 0; del = false;
    Reader r; r.base = base; r.pos = body.off; r.end = body.off + body.len; r.ok = true;
    uint32_t f, wt; uint64_t x = 0; Seg b; b.off = b.len = 0;
    while (r.next(f, wt, x, b)) {
        if (f == 1 && wt == 2) it.key = b;
        else if (!md && f == 2 && wt == 0) del = x != 0;
        else if (!md && f == 3 && wt == 2) { it.val = b; it.has_val = 1; }
    }
}

// Step 1, one thread per entry: the items of a VALID entry whose check passed, in wire order, and its transaction's write count
BD_HD void pu_list_entry(uint32_t e, PuArrays& a)
{
    a.wfirst[e] = a.mfirst[e] = 0;
    if (!pu_eligible(e, a)) return;
    uint32_t nw = 0, nm = 0;
    pu_walk(e, a, [&](uint32_t g, Seg, Seg, Seg) { if (g == 3) nw++; else nm++; });
    const uint32_t t = a.seq[e];
    a.tbase[t] = nw;
    const uint32_t bw = nw ? kl_atomic_add(a.ctr, nw) : 0, bm = nm ? kl_atomic_add(a.ctr + 1, nm) : 0;
    if (bw + nw > a.W_cap || bw + nw < bw || bm + nm > a.M_cap || bm + nm < bm) return;   // overflow: the host grows and runs it again
    a.wfirst[e] = bw; a.mfirst[e] = bm;
    uint32_t qw = 0, qm = 0;
    pu_walk(e, a, [&](uint32_t g, Seg ns, Seg coll, Seg body) {
        const bool md = g == 4;
        PuItem& it = md ? a.meta[bm + qm] : a.item[bw + qw];
        bool del;
        pu_fields(a.pvt, body, md, it, del);
        it.ns = ns; it.coll = coll; it.tx = t; it.pos = md ? qm++ : qw++; it.slot = 0;
        it.kind = md ? PK_META : del ? PK_DEL : PK_PUT;
        if (it.kind == PK_PUT && !it.has_val) pu_incomplete(a);           // PutValAndMetadata of a nil value panics
        if (md) {
            ShaJobP& j = a.jobs[bm + it.pos];
            j.off[0] = it.key.off; j.len[0] = it.key.len; j.off[1] = j.len[1] = j.off[2] = j.len[2] = 0;
        }
    });
}

// Step 2 (after the SHA-256 of the metadata-written keys), the transactions' write positions: tbase[t] = writes of transactions below t
BD_HD void pu_base_host(PuArrays& a)
{
    uint32_t s = 0;
    for (uint32_t t = 0; t < a.T; t++) { const uint32_t c = a.tbase[t]; a.tbase[t] = s; s += c; }
}

BD_HD PuItem& pu_item(PuArrays& a, uint32_t i, uint32_t W) { return i < W ? a.item[i] : a.meta[i - W]; }

BD_HD unsigned long long pu_atomic_max64(unsigned long long* p, unsigned long long v)
{
#if defined(__CUDA_ARCH__)
    return atomicMax(p, v);
#else
    const unsigned long long o = *p; if (v > o) *p = v; return o;
#endif
}

// Step 3, one thread per item (W writes, then the metadata writes): its key's entry of the table, the key's last write, and the
// metadata write that stands for the key
BD_HD void pu_key_item(uint32_t i, uint32_t W, PuArrays& a)
{
    PuItem& it = pu_item(a, i, W);
    sv_key(a.pvt + it.ns.off, it.ns.len, a.pvt + it.coll.off, it.coll.len, a.pvt + it.key.off, it.key.len, it.w);
    unsigned long long tag = txid_mix(it.w, a.seed ^ 0x7f4a7c159e3779b9ull);
    if (tag == 0) tag = 1;
    uint32_t pos = (uint32_t)tag & (a.P_size - 1);
    for (uint32_t probe = 0; probe < a.P_size; probe++, pos = (pos + 1) & (a.P_size - 1)) {
#if defined(__CUDA_ARCH__)
        const unsigned long long old = atomicCAS(&a.key[pos].tag, 0ull, tag);
#else
        const unsigned long long old = a.key[pos].tag; if (old == 0) a.key[pos].tag = tag;
#endif
        if (old != 0 && old != tag) continue;
        PuKey& k = a.key[pos];
        if (old == 0) for (int j = 0; j < 8; j++) k.w[j] = it.w[j];        // compared with every item's digest in step 4
        it.slot = pos;
        if (i < W) pu_atomic_max64(&k.last, (((unsigned long long)it.tx << 32) | it.pos) + 1ull);
        else mv_atomic_max(&k.nmeta, UINT32_MAX - (i - W));
        return;
    }
    pu_incomplete(a);                                                // (the table holds 2 (W + M) entries: not reached)
}

// Step 4, one thread per item: two digests that share a tag share an entry (such a batch is left to the peer); the last write's item
// and the key's first position among the last writer's writes
BD_HD void pu_first_item(uint32_t i, uint32_t W, PuArrays& a)
{
    const PuItem& it = pu_item(a, i, W);
    PuKey& k = a.key[it.slot];
    if (!txid_equal(k.w, it.w)) { pu_incomplete(a); return; }
    if (i >= W || it.tx != (uint32_t)((k.last - 1) >> 32)) return;
    mv_atomic_max(&k.nfirst, UINT32_MAX - it.pos);
    if ((((unsigned long long)it.tx << 32) | it.pos) + 1ull == k.last) k.lrec = i;
}

// Step 5, one thread per metadata write (after the SHA-256 of its key): the renewal of its key, decided by the one standing for the key.
// Its job is turned into the SHA-256 of the latest value when the device compares it (of nothing otherwise).
BD_HD void pu_renew_meta(uint32_t m, PuArrays& a)
{
    const PuItem& it = a.meta[m];
    PuKey& k = a.key[it.slot];
    ShaJobP& j = a.jobs[m];
    j.off[0] = j.len[0] = 0;
    if (UINT32_MAX - k.nmeta != m || !a.ukey) return;
    uint32_t w[8];                                                   // hashUpdates.Get(ns, coll, SHA-256(key))
    sv_key(a.pvt + it.ns.off, it.ns.len, a.pvt + it.coll.off, it.coll.len, a.dig + 32 * (size_t)m, 32, w);
    const uint32_t hk = mv_find_key(a.stage, a.stage_seed, w);
    if (hk == UINT32_MAX) return;
    const UdKey& u = a.ukey[hk];
    if (u.op != UD_PUT) return;                                      // not in the hashed batch, or a DELETE there
    if (!k.last) { a.rmark[hk] = it.slot + 1; return; }              // the latest value is the committed one: the peer's GetPrivateData
    const PuItem& l = a.item[k.lrec];
    if (l.tx == u.L - 1) return;                                     // the versions are the same
    if (u.vsrc != UD_BLOCK) { pu_incomplete(a); return; }            // the hashed value hash is the committed one
    j.off[0] = l.val.off; j.len[0] = l.kind == PK_DEL ? 0 : l.val.len;
    k.hk = hk + 1;
}

// Step 6, one thread per key entry (after the SHA-256 of the compared values): the renewal's comparison, and the record's position
BD_HD void pu_mark_key(uint32_t p, PuArrays& a)
{
    PuKey& k = a.key[p];
    if (!k.tag || !k.last) return;
    if (k.hk) {
        const Seg h = a.useg[a.ukey[k.hk - 1].vrec].val;
        const uint8_t* d = a.dig + 32 * (size_t)(UINT32_MAX - k.nmeta);
        bool eq = h.len == 32;
        for (uint32_t i = 0; i < 32 && eq; i++) eq = a.blk[h.off + i] == d[i];
        if (eq) {
            if (a.item[k.lrec].kind == PK_DEL) pu_incomplete(a);     // Put of a nil value: the reference panics
            else k.renew = 1;
        }
    }
    const uint32_t tx = (uint32_t)((k.last - 1) >> 32);
    a.mark[a.tbase[tx] + (UINT32_MAX - k.nfirst)] = p + 1;
}

// Step 8, per output record: its words
BD_HD void pu_emit(uint32_t o, PuArrays& a)
{
    uint32_t* w = a.out + (size_t)o * PU_WORDS;
    if (o < a.ctr[3]) {
        const PuKey& k = a.key[a.out_key[o]];
        const PuItem& l = a.item[k.lrec];
        const bool put = l.kind == PK_PUT;
        w[0] = k.renew ? a.ukey[k.hk - 1].L - 1 : l.tx; w[1] = put ? UD_PUT : UD_DELETE;
        w[2] = l.ns.off; w[3] = l.ns.len; w[4] = l.coll.off; w[5] = l.coll.len; w[6] = l.key.off; w[7] = l.key.len;
        w[8] = put ? l.val.off : 0; w[9] = put ? l.val.len : 0; w[10] = UINT32_MAX;
        return;
    }
    const uint32_t h = a.out_key[o], hk = a.uokey[h];
    const PuKey& k = a.key[a.rmark[hk] - 1];
    const PuItem& m = a.meta[UINT32_MAX - k.nmeta];
    w[0] = a.ukey[hk].L - 1; w[1] = PU_RENEW;
    w[2] = m.ns.off; w[3] = m.ns.len; w[4] = m.coll.off; w[5] = m.coll.len; w[6] = m.key.off; w[7] = m.key.len;
    w[8] = w[9] = 0; w[10] = h;
}

#if defined(__CUDACC__)
__global__ void __launch_bounds__(64) pu_list_kernel(PuArrays a)
{
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < a.n_pvt) pu_list_entry(e, a);
}

// One CTA of 1024: tbase[t], the transaction-order position of each transaction's first write
__global__ void __launch_bounds__(1024) pu_base_kernel(PuArrays a)
{
    const uint32_t per = (a.T + blockDim.x - 1) / blockDim.x, lo = min(a.T, threadIdx.x * per), hi = min(a.T, lo + per);
    uint32_t c = 0;
    for (uint32_t t = lo; t < hi; t++) c += a.tbase[t];
    uint32_t off, unused, tot, tot2;
    ud_block_scan(c, 0, off, unused, tot, tot2);
    for (uint32_t t = lo; t < hi; t++) { const uint32_t v = a.tbase[t]; a.tbase[t] = off; off += v; }
}

__global__ void __launch_bounds__(256) pu_key_kernel(PuArrays a, uint32_t W, uint32_t N)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) pu_key_item(i, W, a);
}

__global__ void __launch_bounds__(256) pu_first_kernel(PuArrays a, uint32_t W, uint32_t N)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) pu_first_item(i, W, a);
}

__global__ void __launch_bounds__(128) pu_renew_kernel(PuArrays a, uint32_t M)
{
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m < M) pu_renew_meta(m, a);
}

__global__ void __launch_bounds__(256) pu_mark_kernel(PuArrays a)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < a.P_size) pu_mark_key(p, a);
}

// Step 7, one CTA of 1024: the PUT / DELETE records in position order, then the RENEW records in the hashed records' order; totals in
// ctr[3], ctr[4]
__global__ void __launch_bounds__(1024) pu_compact_kernel(PuArrays a, uint32_t W)
{
    uint32_t per = (W + blockDim.x - 1) / blockDim.x, lo = min(W, threadIdx.x * per), hi = min(W, lo + per);
    uint32_t c = 0;
    for (uint32_t q = lo; q < hi; q++) c += a.mark[q] != 0;
    uint32_t off, unused, n1, tot2;
    ud_block_scan(c, 0, off, unused, n1, tot2);
    for (uint32_t q = lo; q < hi; q++) if (a.mark[q]) a.out_key[off++] = a.mark[q] - 1;
    const uint32_t H = a.n_h;
    per = (H + blockDim.x - 1) / blockDim.x; lo = min(H, threadIdx.x * per); hi = min(H, lo + per);
    c = 0;
    for (uint32_t h = lo; h < hi; h++) c += a.rmark[a.uokey[h]] != 0;
    uint32_t n2;
    ud_block_scan(c, 0, off, unused, n2, tot2);
    off += n1;
    for (uint32_t h = lo; h < hi; h++) if (a.rmark[a.uokey[h]]) a.out_key[off++] = h;
    if (threadIdx.x == 0) { a.ctr[3] = n1; a.ctr[4] = n2; }
}

__global__ void __launch_bounds__(128) pu_emit_kernel(PuArrays a)
{
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o < a.ctr[3] + a.ctr[4]) pu_emit(o, a);
}
#endif

} }  // namespace fabgpu::bdev
