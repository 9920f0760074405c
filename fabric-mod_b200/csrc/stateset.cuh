// The world state's committed key versions on the device (fabgpu_state_versions) and the ledger's MVCC check over them
// (fabgpu_validate_mvcc): core/ledger/kvledger/txmgmt/validation/validator.go:82-281 (validateAndPrepareBatch, validateKVRead,
// validateKVReadHash), tx_ops.go:18-120 and types.go:81-111 (applyWriteSet), with LevelDB semantics.  Host+device code: the tests' host
// build runs the same stage one item at a time.
//
// Key identity: SHA-256 over u32le(len) || namespace || u32le(len) || collection || u32le(len) || key (the collection is empty for a
// public key; for a private key the key is its 32-byte hash).  The table is open addressing over 56-byte slots (digest, state, version)
// at a load of at most 1/2; the first probe is txid_mix of the digest with the context's seed, since key bytes are chosen by submitters.
// A removed key keeps its slot as SV_REMOVED (probes continue past it; an upsert of the same key takes it back).
//
// Range queries (RangeQueryInfo) are decided only while an ordered index of the public keys is installed (stateindex.cuh,
// fabgpu_state_versions_indexed); without one a VALID transaction with a range query is 254 (MV_RANGE).
#pragma once
#include "blockdev.cuh"
#if defined(__CUDACC__)
#include "sha256.cuh"
#endif

namespace fabgpu { namespace bdev {

enum : uint32_t { SV_EMPTY = 0, SV_CLAIMED = 1, SV_PRESENT = 2, SV_UNKNOWN = 3, SV_REMOVED = 4 };

struct StateSlot { uint32_t w[8]; uint32_t state; uint32_t pad; unsigned long long blk, txn; };

// count[0]: keys held (present or unknown), [1]: slots ever claimed (removed ones included), [2]: keys unknown
struct StateSetDev { StateSlot* slots; uint32_t mask; uint32_t broken; uint64_t seed; unsigned long long* count; };

// ---- SHA-256 of the key identity ------------------------------------------------------------------------------------------------
inline void sv_compress_host(uint32_t* h, uint32_t* w)
{
    static const uint32_t K[64] = {
        0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be,
        0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa,
        0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85,
        0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3,
        0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f,
        0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
    auto r = [](uint32_t x, int n) { return (x >> n) | (x << (32 - n)); };
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int i = 0; i < 64; i++) {
        if (i >= 16) {
            const uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
            w[i & 15] += (r(w15, 7) ^ r(w15, 18) ^ (w15 >> 3)) + w[(i + 9) & 15] + (r(w2, 17) ^ r(w2, 19) ^ (w2 >> 10));
        }
        const uint32_t t1 = hh + (r(e, 6) ^ r(e, 11) ^ r(e, 25)) + ((e & f) ^ (~e & g)) + K[i] + w[i & 15];
        const uint32_t t2 = (r(a, 2) ^ r(a, 13) ^ r(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

struct SvSha { uint32_t h[8]; uint32_t w[16]; uint32_t n; uint64_t total; };

BD_HD void sv_block(SvSha& s)
{
#if defined(__CUDA_ARCH__)
    sha256_compress(s.h, s.w);
#else
    sv_compress_host(s.h, s.w);
#endif
    s.n = 0;
    for (int k = 0; k < 16; k++) s.w[k] = 0;
}
BD_HD void sv_byte(SvSha& s, uint32_t b)
{
    s.w[s.n >> 2] |= (b & 0xffu) << (24 - 8 * (s.n & 3));
    s.total++;
    if (++s.n == 64) sv_block(s);
}
BD_HD void sv_part(SvSha& s, const uint8_t* p, uint32_t len)
{
    for (int k = 0; k < 4; k++) sv_byte(s, len >> (8 * k));
    for (uint32_t i = 0; i < len; i++) sv_byte(s, p[i]);
}

// The digest of (ns, coll, key) as 8 words (SHA-256's state words; the table only compares and mixes them)
BD_HD void sv_key(const uint8_t* ns, uint32_t ns_len, const uint8_t* coll, uint32_t coll_len, const uint8_t* key, uint32_t key_len, uint32_t out[8])
{
    SvSha s;
    const uint32_t iv[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    for (int k = 0; k < 8; k++) s.h[k] = iv[k];
    for (int k = 0; k < 16; k++) s.w[k] = 0;
    s.n = 0; s.total = 0;
    sv_part(s, ns, ns_len); sv_part(s, coll, coll_len); sv_part(s, key, key_len);
    const uint64_t bits = s.total * 8;
    sv_byte(s, 0x80);
    while (s.n != 56) sv_byte(s, 0);
    for (int k = 7; k >= 0; k--) sv_byte(s, (uint32_t)(bits >> (8 * k)));
    for (int k = 0; k < 8; k++) out[k] = s.h[k];
}

// ---- the committed table ---------------------------------------------------------------------------------------------------------
BD_HD uint32_t sv_state_acquire(const StateSlot* s)
{
#if defined(__CUDA_ARCH__)
    const uint32_t st = *reinterpret_cast<const volatile uint32_t*>(&s->state);
    __threadfence();
    return st;
#else
    return __atomic_load_n(&s->state, __ATOMIC_ACQUIRE);
#endif
}

BD_HD void sv_count(unsigned long long* c, int k, long long d)
{
    if (!d) return;
#if defined(__CUDA_ARCH__)
    atomicAdd(c + k, (unsigned long long)d);
#else
    c[k] += (unsigned long long)d;
#endif
}

// Sets the key's state (SV_PRESENT with its version, SV_UNKNOWN or SV_REMOVED).  Inserts running together carry different keys.
// Returns 1 when a slot was claimed, 0 when the key was held (or is removed and absent), -1 when no slot is free.
BD_HD int sv_upsert(const StateSetDev& t, const uint32_t w[8], uint32_t state, unsigned long long blk, unsigned long long txn)
{
    uint32_t pos = (uint32_t)txid_mix(w, t.seed) & t.mask;
    for (uint64_t n = 0; n <= (uint64_t)t.mask; n++, pos = (pos + 1) & t.mask) {
        StateSlot* s = t.slots + pos;
        uint32_t st = sv_state_acquire(s);
        if (st == SV_EMPTY) {
            if (state == SV_REMOVED) return 0;
#if defined(__CUDA_ARCH__)
            st = atomicCAS(&s->state, (uint32_t)SV_EMPTY, (uint32_t)SV_CLAIMED);
#else
            __atomic_compare_exchange_n(&s->state, &st, (uint32_t)SV_CLAIMED, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE);
#endif
            if (st == SV_EMPTY) {
                for (int k = 0; k < 8; k++) s->w[k] = w[k];
                s->blk = blk; s->txn = txn;
#if defined(__CUDA_ARCH__)
                __threadfence();
                atomicExch(&s->state, state);
#else
                __atomic_store_n(&s->state, state, __ATOMIC_RELEASE);
#endif
                sv_count(t.count, 0, 1); sv_count(t.count, 1, 1); sv_count(t.count, 2, state == SV_UNKNOWN);
                return 1;
            }
#if defined(__CUDA_ARCH__)
            if (st != SV_CLAIMED) __threadfence();
#endif
        }
        if (st == SV_CLAIMED) continue;
        if (txid_equal(s->w, w)) {
            const int held = st != SV_REMOVED, now = state != SV_REMOVED;
            sv_count(t.count, 0, now - held);
            sv_count(t.count, 2, (int)(state == SV_UNKNOWN) - (int)(st == SV_UNKNOWN));
            s->blk = blk; s->txn = txn; s->state = state;
            return 0;
        }
    }
    return -1;
}

// SV_PRESENT (with the version), SV_UNKNOWN, or SV_EMPTY for a key the table does not hold.  No upsert runs while this reads.
BD_HD uint32_t sv_lookup(const StateSetDev& t, const uint32_t w[8], unsigned long long& blk, unsigned long long& txn)
{
    uint32_t pos = (uint32_t)txid_mix(w, t.seed) & t.mask;
    for (uint64_t n = 0; n <= (uint64_t)t.mask; n++, pos = (pos + 1) & t.mask) {
        const StateSlot& s = t.slots[pos];
        const uint32_t st = s.state;
        if (st == SV_EMPTY) return SV_EMPTY;
        if (st != SV_CLAIMED && txid_equal(s.w, w)) {
            blk = s.blk; txn = s.txn;
            return st == SV_REMOVED ? SV_EMPTY : st;
        }
    }
    return SV_EMPTY;
}

} }  // namespace fabgpu::bdev

#include "stateindex.cuh"

namespace fabgpu { namespace bdev {

// ---- the MVCC stage over one block -----------------------------------------------------------------------------------------------
// record kinds: a read (public or hashed), a write, a deleting write, a metadata write with entries (metadataUpdate) and one without
// (metadataDelete); MvccRec::has_ver is a read's Version, a write's value (or value hash)
enum : uint8_t { MR_READ = 0, MR_PUT = 1, MR_DEL = 2, MR_META = 3, MR_MDEL = 4 };
// MvccRec::c -- reads: the committed comparison; writes: the key's committed existence
enum : uint8_t { MC_OK = 0, MC_FAIL = 1, MC_UNDET = 2, MC_ABSENT = 0, MC_EXISTS = 1 };
// per-transaction info bits
#define MV_RANGE 1u                // a RangeQueryInfo while no index is installed: phantom reads are not checked
#define MV_OPEN 2u                 // its write set cannot be enumerated (no ChaincodeAction.results, a non-endorser transaction, no parse)
#define MV_MARKED 4u               // touches a key that another transaction of the block writes first: the sequential walk decides it
// the walk's running state of a key in `updates` (validator.go:176-193)
enum : uint32_t { RS_NONE = 0, RS_PUT = 1, RS_DEL = 2, RS_UNDET = 3 };

struct MvccRec {
    uint32_t w[8];
    uint32_t tx, key;              // transaction; entry of the block's key table
    unsigned long long blk, txn;   // a read's version
    uint8_t kind, has_ver, c, pub; // pub: a key of a KVRWSet (not a hashed one)
    Seg ns, k;                     // the namespace and key bytes in the block
};

// One RangeQueryInfo of a VALID transaction (while an index is installed).  form: RF_NONE neither raw_reads nor reads_merkle_hashes
// (no reads), RF_RAW raw_reads (body: QueryReads), RF_MERKLE reads_merkle_hashes (body: QueryReadsMerkleSummary), RF_BAD a wire form
// not decided here.  lo, hi: the in-range slice of the block's sorted written public keys; endk: the end key's entry of the block's key
// table + 1 (0: the block does not write it).  c: the answer against the committed state alone; marked: an earlier transaction of the
// block writes a key of the range (or its end key, when served), so the walk decides it.  ib, id: the range's first positions in the
// index's base and delta, found once before the walk.
enum : uint8_t { RF_NONE = 0, RF_RAW = 1, RF_MERKLE = 2, RF_BAD = 3 };
struct MvccRange {
    uint32_t tx; Seg ns, start, end, body;
    uint32_t lo, hi, endk, degree, level;
    uint8_t exhausted, form, c, marked;
    unsigned long long ib, id;
};

// One entry per distinct key the block reads or writes.  tag: txid_mix of the digest (0 = empty), claimed by CAS; w written by the claimer.
struct MvccKey {
    unsigned long long tag;
    uint32_t w[8];
    uint32_t nfirst, nw, lastr;         // UINT32_MAX - earliest writer (0 none: the table starts zeroed), write records, latest reader + 1 (0 none)
    uint32_t wrec;                      // some write record (the only one when nw == 1)
    uint32_t rs, rs_tx, op_tx, op;      // the walk: running state, its writer, and the combined operation of transaction op_tx - 1
    uint32_t rng;                       // a later transaction's range covers the key after one of its writers: the walk tracks it
};

struct MvccArrays {
    MvccRec* rec; uint32_t R_cap;
    uint32_t* first_rec; uint32_t* n_rec; uint8_t* info;   // per transaction
    MvccKey* key; uint32_t K_size;                         // power of two >= 2 R
    uint32_t* ctr;                 // [0] records handed out (> R_cap: overflow), [1] alias, [2] first open transaction (UINT32_MAX none), [3] marked,
                                   // [4] range records handed out (> G_cap: overflow), [5] written public keys, [6] their bytes (an upper bound)
    uint32_t* mlist;               // the marked transactions in index order
    // range queries, while an index is installed (indexed = 1); without one these members are not read
    uint32_t indexed = 0; unsigned long long block = 0;
    MvccRange* rng = nullptr; uint32_t G_cap = 0; uint32_t* first_rng = nullptr; uint32_t* n_rng = nullptr;   // per transaction
    WrittenKey* wk = nullptr;                                                 // the block's written public keys, sorted (ctr[5] of them)
    MerkleState* mk = nullptr;                                                // per range record: its Merkle state (global scratch)
    StateIndexDev ix = {nullptr, nullptr, nullptr, 0, 0, 0};
};

BD_HD uint32_t mv_atomic_min(uint32_t* p, uint32_t v)
{
#if defined(__CUDA_ARCH__)
    return atomicMin(p, v);
#else
    const uint32_t o = *p; if (v < o) *p = v; return o;
#endif
}
BD_HD uint32_t mv_atomic_max(uint32_t* p, uint32_t v)
{
#if defined(__CUDA_ARCH__)
    return atomicMax(p, v);
#else
    const uint32_t o = *p; if (v > o) *p = v; return o;
#endif
}

// A Version{block_num = 1, tx_num = 2} message; repeated occurrences merge, as proto.Unmarshal merges them
BD_HD bool mv_version(const uint8_t* base, Seg v, unsigned long long& blk, unsigned long long& txn)
{
    Reader r; r.base = base; r.pos = v.off; r.end = v.off + v.len; r.ok = true;
    uint32_t f, wt; uint64_t x = 0; Seg b; b.off = b.len = 0;
    while (r.next(f, wt, x, b)) {
        if (f == 1 || f == 2) { if (wt != 0) return false; if (f == 1) blk = x; else txn = x; }
    }
    return r.ok;
}

// The transaction's write set can be enumerated: dispatch_plan reached ChaincodeAction.results of an endorser transaction
BD_HD bool mv_reached(const TxDev& tx)
{
    return tx.htype == 3 && tx.endorser_parse_ok && (tx.results.len > 0 || (tx.disp != TXC_BAD_HEADER_EXTENSION && tx.disp != TXC_BAD_RESPONSE_PAYLOAD));
}

// Every read, hashed read and write of a TxReadWriteSet, through kl_scan_rwset's parser with its reads enabled.
// on_rec(ns, coll, key, kind, has_ver, blk, txn, pub); on_range(ns, RangeQueryInfo).  false when a level does not parse.
template <typename F, typename G>
BD_HD bool mv_scan(const uint8_t* base, Seg results, F on_rec, G on_range)
{
    return kl_scan_rwset<true>(base, results, [&](Seg ns, Seg coll, Seg key, uint32_t g, Seg body) {
        // g: the field of the record in its set -- KVRWSet 1 read, 2 range query, 3 write, 4 metadata write;
        // HashedRWSet 11 hashed read, 12 hashed write, 13 hashed metadata write (kl_scan_rwset adds 10)
        if (g == 2) { on_range(ns, body); return true; }
        if (g == 1 || g == 11) {
            // KVRead{key = 1, version = 2}, KVReadHash{key_hash = 1, version = 2}: an absent version is nil, an empty one (0, 0)
            bool has = false; unsigned long long blk = 0, txn = 0; bool ok = true;
            if (!scan_msg(base, body, BD_F(1) | BD_F(2), 0, [&](uint32_t h, Seg v) { if (h == 2) { has = true; ok = ok && mv_version(base, v, blk, txn); } }) || !ok) return false;
            on_rec(ns, coll, key, (uint8_t)MR_READ, has, blk, txn, g < 10);
            return true;
        }
        // KVWrite{key = 1, is_delete = 2, value = 3}, KVWriteHash{key_hash = 1, is_delete = 2, value_hash = 3, is_purge = 4};
        // KVMetadataWrite{key = 1, entries = 2}, KVMetadataWriteHash{key_hash = 1, entries = 2}.  has: the value (a write without one
        // has a nil value) or any entry (none: Entries == nil, a metadataDelete, tx_ops.go:109-120)
        bool del = false, has = false;
        const bool md = g == 4 || g == 13;
        Reader r; r.base = base; r.pos = body.off; r.end = body.off + body.len; r.ok = true;
        uint32_t f, wt; uint64_t x = 0; Seg b; b.off = b.len = 0;
        while (r.next(f, wt, x, b)) {
            if (!md && f == 2 && wt == 0) del = x != 0;
            if (f == (md ? 2u : 3u)) has = true;
        }
        on_rec(ns, coll, key, (uint8_t)(md ? (has ? MR_META : MR_MDEL) : del ? MR_DEL : MR_PUT), has, 0ull, 0ull, g < 10);
        return true;
    });
}

// RangeQueryInfo{start_key = 1, end_key = 2, itr_exhausted = 3, oneof {raw_reads = 4, reads_merkle_hashes = 5}} (kv_rwset.proto, as
// recalled: the file is not in the reference tree); QueryReads{kv_reads = 1}; QueryReadsMerkleSummary{max_degree = 1, max_level = 2,
// max_level_hashes = 3}.  A scalar or string field given twice: the last wins, as proto.Unmarshal does.  RF_BAD: the message or its reads
// do not parse, both oneof fields are present, a oneof field is repeated, or max_degree / max_level does not fit 32 bits -- shapes whose
// decoding this stage does not restate.
BD_HD void mv_range_parse(const uint8_t* base, Seg info, MvccRange& g)
{
    g.start.off = g.start.len = g.end.off = g.end.len = g.body.off = g.body.len = 0;
    g.exhausted = 0; g.form = RF_NONE; g.degree = g.level = 0;
    Reader r; r.base = base; r.pos = info.off; r.end = info.off + info.len; r.ok = true;
    uint32_t f, wt, n4 = 0, n5 = 0; uint64_t x = 0; Seg b; b.off = b.len = 0;
    while (r.next(f, wt, x, b)) {
        if (f == 3) { if (wt != 0) { g.form = RF_BAD; return; } g.exhausted = x != 0; }
        else if (f == 1 || f == 2 || f == 4 || f == 5) {
            if (wt != 2) { g.form = RF_BAD; return; }
            if (f == 1) g.start = b; else if (f == 2) g.end = b; else { g.body = b; (f == 4 ? n4 : n5)++; }
        }
    }
    if (!r.ok || n4 + n5 > 1) { g.form = RF_BAD; return; }
    if (n4) {
        g.form = RF_RAW;
        bool ok = true;
        if (!scan_msg(base, g.body, BD_F(1), 0, [&](uint32_t, Seg kv) {
                unsigned long long blk = 0, txn = 0;
                if (!scan_msg(base, kv, BD_F(1) | BD_F(2), 0, [&](uint32_t h, Seg v) { if (h == 2) ok = ok && mv_version(base, v, blk, txn); })) ok = false;
            }) || !ok) g.form = RF_BAD;
    } else if (n5) {
        g.form = RF_MERKLE;
        Reader m; m.base = base; m.pos = g.body.off; m.end = g.body.off + g.body.len; m.ok = true;
        while (m.next(f, wt, x, b)) {
            if (f == 1 || f == 2) { if (wt != 0 || x > 0xffffffffull) { g.form = RF_BAD; return; } if (f == 1) g.degree = (uint32_t)x; else g.level = (uint32_t)x; }
            else if (f == 3 && wt != 2) { g.form = RF_BAD; return; }
        }
        if (!m.ok) g.form = RF_BAD;
    }
}

// Stage 1, one thread per transaction: the records of a transaction tv_flags leaves VALID or 254, with their key digests, and (index
// installed) the range records of a VALID one
BD_HD void mv_scan_tx(const uint8_t* base, const TxDev& tx, uint32_t t, uint8_t tv, MvccArrays& a)
{
    a.first_rec[t] = 0; a.n_rec[t] = 0; a.info[t] = 0;
    if (a.indexed) { a.first_rng[t] = 0; a.n_rng[t] = 0; }
    if (tv != TXC_VALID && tv != TXC_NOT_VALIDATED) return;
    uint32_t n = 0, n_range = 0;
    if (!mv_reached(tx) || !mv_scan(base, tx.results, [&](Seg, Seg, Seg, uint8_t, bool, unsigned long long, unsigned long long, bool) { n++; },
                                    [&](Seg, Seg) { n_range++; })) {
        a.info[t] = MV_OPEN;
        mv_atomic_min(a.ctr + 2, t);                                   // later VALID transactions may read its writes
        return;
    }
    const bool ranges = a.indexed && tv == TXC_VALID;
    a.info[t] = n_range && !a.indexed ? MV_RANGE : 0;
    if (ranges && n_range) {
        const uint32_t b = kl_atomic_add(a.ctr + 4, n_range);
        if (b + n_range <= a.G_cap && b + n_range >= b) {
            a.first_rng[t] = b; a.n_rng[t] = n_range;
            uint32_t q = b;
            mv_scan(base, tx.results, [&](Seg, Seg, Seg, uint8_t, bool, unsigned long long, unsigned long long, bool) {}, [&](Seg ns, Seg info) {
                MvccRange& g = a.rng[q++];
                g.tx = t; g.ns = ns; g.lo = g.hi = g.endk = 0; g.c = MC_OK; g.marked = 0; g.ib = g.id = 0;
                mv_range_parse(base, info, g);
            });
        }
    }
    if (n == 0) return;
    const uint32_t b = kl_atomic_add(a.ctr, n);
    if (b + n > a.R_cap || b + n < b) return;                        // overflow: the host grows the arrays and runs the stage again
    a.first_rec[t] = b; a.n_rec[t] = n;
    uint32_t q = b, bytes = 0;
    mv_scan(base, tx.results, [&](Seg ns, Seg coll, Seg key, uint8_t kind, bool has, unsigned long long blk, unsigned long long txn, bool pub) {
        MvccRec& r = a.rec[q++];
        sv_key(base + ns.off, ns.len, base + coll.off, coll.len, base + key.off, key.len, r.w);
        r.tx = t; r.key = 0; r.blk = blk; r.txn = txn; r.kind = kind; r.has_ver = has ? 1 : 0; r.c = 0; r.pub = pub ? 1 : 0;
        r.ns = ns; r.k = key;
        if (pub && kind != MR_READ) bytes += ns.len + key.len;
    }, [&](Seg, Seg) {});
    if (a.indexed && bytes) kl_atomic_add(a.ctr + 6, bytes);
}

// Stage 2, one thread per record: its entry in the block's key table, and the committed table's answer
BD_HD void mv_key_rec(uint32_t i, MvccArrays& a, const StateSetDev& set)
{
    MvccRec& r = a.rec[i];
    unsigned long long tag = txid_mix(r.w, set.seed ^ 0x9e3779b97f4a7c15ull);
    if (tag == 0) tag = 1;
    uint32_t pos = (uint32_t)tag & (a.K_size - 1);
    bool placed = false;
    for (uint32_t probe = 0; probe < a.K_size; probe++, pos = (pos + 1) & (a.K_size - 1)) {
#if defined(__CUDA_ARCH__)
        const unsigned long long old = atomicCAS(&a.key[pos].tag, 0ull, tag);
#else
        const unsigned long long old = a.key[pos].tag; if (old == 0) a.key[pos].tag = tag;
#endif
        if (old != 0 && old != tag) continue;
        MvccKey& e = a.key[pos];
        if (old == 0) for (int k = 0; k < 8; k++) e.w[k] = r.w[k];       // compared with every record's digest in stage 3
        if (r.kind == MR_READ) mv_atomic_max(&e.lastr, r.tx + 1);
        else {
            mv_atomic_max(&e.nfirst, UINT32_MAX - r.tx); kl_atomic_add(&e.nw, 1);
#if defined(__CUDA_ARCH__)
            atomicExch(&e.wrec, i);
#else
            e.wrec = i;
#endif
        }
        r.key = pos;
        placed = true;
        break;
    }
    if (!placed) a.ctr[1] = 1;
    unsigned long long blk = 0, txn = 0;
    const uint32_t st = set.broken ? SV_UNKNOWN : sv_lookup(set, r.w, blk, txn);
    if (r.kind == MR_READ)
        r.c = st == SV_UNKNOWN ? MC_UNDET : st == SV_EMPTY ? (r.has_ver ? MC_FAIL : MC_OK) : (r.has_ver && r.blk == blk && r.txn == txn ? MC_OK : MC_FAIL);
    else
        r.c = st == SV_UNKNOWN ? MC_UNDET : st == SV_EMPTY ? MC_ABSENT : MC_EXISTS;
}

// Stage 3, one thread per record: two digests that share a tag share an entry; such a block is not decided here
BD_HD void mv_check_rec(uint32_t i, MvccArrays& a)
{
    const MvccRec& r = a.rec[i];
    if (!txid_equal(a.key[r.key].w, r.w)) a.ctr[1] = 1;
}

BD_HD uint32_t mv_first(const MvccKey& e) { return UINT32_MAX - e.nfirst; }

// Some transaction's outcome depends on another's write of the key: two write records, or a read after the first write
BD_HD bool mv_contended(const MvccKey& e)
{
    return e.nw >= 2 || (e.nw >= 1 && e.lastr > mv_first(e) + 1) || (e.nw >= 1 && e.rng);
}

// ---- range queries (index installed) --------------------------------------------------------------------------------------------
// The entry of the block's key table holding digest w, or UINT32_MAX
BD_HD uint32_t mv_find_key(const MvccArrays& a, uint64_t seed, const uint32_t w[8])
{
    unsigned long long tag = txid_mix(w, seed ^ 0x9e3779b97f4a7c15ull);
    if (tag == 0) tag = 1;
    uint32_t pos = (uint32_t)tag & (a.K_size - 1);
    for (uint32_t probe = 0; probe < a.K_size; probe++, pos = (pos + 1) & (a.K_size - 1)) {
        const MvccKey& e = a.key[pos];
        if (e.tag == 0) return UINT32_MAX;
        if (e.tag == tag && txid_equal(e.w, w)) return pos;
    }
    return UINT32_MAX;
}

// One thread per entry of the block's key table: a public key some record writes joins the list the range records search (unsorted)
BD_HD void mv_written_key(uint32_t k, MvccArrays& a)
{
    const MvccKey& e = a.key[k];
    if (!e.tag || !e.nw) return;
    const MvccRec& r = a.rec[e.wrec];
    if (!r.pub) return;
    WrittenKey& o = a.wk[kl_atomic_add(a.ctr + 5, 1)];
    o.ns_off = r.ns.off; o.nl = r.ns.len; o.key_off = r.k.off; o.kl = r.k.len; o.k = k;
    for (int j = 0; j < 8; j++) o.w[j] = e.w[j];
}

// The combined iterator (combined_iterator.go) of one range over the committed state and -- in the walk -- `updates`, the running state
// of the block's keys that earlier VALID or 254 transactions wrote.  Candidates come in key order from the index (base and delta merged)
// and from the block's in-range written keys; where both hold a key the block's state wins.  A committed candidate the table does not
// hold is skipped (a dead index entry); a deleted key is skipped.  When itr_exhausted is false the end key is served once, after
// everything else: from the block's state, else from the table, not at all when absent or deleted.
struct RangeIt {
    const uint8_t* base; const MvccRange* g; const StateSetDev* set; const StateIndexDev* ix; const MvccArrays* a;
    bool use_block; uint64_t ib, id; uint32_t j; bool end_served;
};

BD_HD void rq_begin(RangeIt& it, const uint8_t* base, const MvccRange& g, const StateSetDev& set, const MvccArrays& a, bool use_block)
{
    it.base = base; it.g = &g; it.set = &set; it.ix = &a.ix; it.a = &a; it.use_block = use_block; it.end_served = false; it.j = g.lo;
    it.ib = g.ib; it.id = g.id;
}

BD_HD int rq_state(uint32_t rs, uint32_t rs_tx, unsigned long long block, unsigned long long& blk, unsigned long long& txn)
{
    if (rs == RS_PUT) { blk = block; txn = rs_tx; return 1; }
    return rs == RS_DEL ? 0 : 2;
}

// The next result: 1 (key bytes, version), 0 none left, 2 a candidate whose state is unknown (the answer is 254)
BD_HD int rq_next(RangeIt& it, const uint8_t*& key, uint32_t& kl, unsigned long long& blk, unsigned long long& txn)
{
    const MvccRange& g = *it.g; const StateIndexDev& x = *it.ix; const MvccArrays& a = *it.a;
    const KeyRef bound = key_ref(it.base + g.ns.off, g.ns.len, it.base + g.end.off, g.end.len);
    if (it.set->broken) return 2;
    for (;;) {
        const bool hb = it.ib < x.nb && ri_below_end(key_ref(x.heap, x.base[it.ib]), bound);
        const bool hd = it.id < x.nd && ri_below_end(key_ref(x.heap, x.delta[it.id]), bound);
        const IndexEntry* c = nullptr; bool from_base = false;
        if (hb && (!hd || key_cmp(key_ref(x.heap, x.base[it.ib]), key_ref(x.heap, x.delta[it.id])) < 0)) { c = x.base + it.ib; from_base = true; }
        else if (hd) c = x.delta + it.id;
        while (it.use_block && it.j < g.hi && a.key[a.wk[it.j].k].rs == RS_NONE) it.j++;
        const WrittenKey* u = it.use_block && it.j < g.hi ? a.wk + it.j : nullptr;
        if (!c && !u) break;
        const int cmp = !c ? 1 : !u ? -1 : key_cmp(key_ref(x.heap, *c), key_ref(it.base, *u));
        if (cmp <= 0) { if (from_base) it.ib++; else it.id++; }
        if (cmp >= 0) it.j++;
        if (cmp < 0) {
            const uint32_t st = sv_lookup(*it.set, c->w, blk, txn);
            if (st == SV_EMPTY) continue;
            if (st == SV_UNKNOWN) return 2;
            key = x.heap + c->off + c->nl; kl = c->kl;
            return 1;
        }
        const MvccKey& e = a.key[u->k];
        const int r = rq_state(e.rs, e.rs_tx, a.block, blk, txn);
        if (r == 0) continue;
        key = it.base + u->key_off; kl = u->kl;
        return r;
    }
    if (g.exhausted || it.end_served) return 0;
    it.end_served = true;
    key = it.base + g.end.off; kl = g.end.len;
    if (it.use_block && g.endk && a.key[g.endk - 1].rs != RS_NONE) {
        const MvccKey& e = a.key[g.endk - 1];
        return rq_state(e.rs, e.rs_tx, a.block, blk, txn);
    }
    uint32_t w[8];
    sv_key(it.base + g.ns.off, g.ns.len, nullptr, 0, it.base + g.end.off, g.end.len, w);
    const uint32_t st = sv_lookup(*it.set, w, blk, txn);
    return st == SV_PRESENT ? 1 : st == SV_UNKNOWN ? 2 : 0;
}

// validateRangeQuery (validator.go:216-237) over the iterator: MC_OK, MC_FAIL or MC_UNDET.  Results are drawn as the reference's
// validators draw them, so a candidate of unknown state past the point where the answer is settled is never reached.
// Raw reads (rangeQueryResultsValidator): the results must equal the recorded KVReads, key and version, with none left over.  A read
// without a Version that is reached with a result of its key is 254: convertToVersionHeight dereferences the nil Version and the
// reference panics (a read with a mismatching key returns false first).
// Merkle summary (rangeQueryHashValidator): the loop's early exits are restated after every result (mk_early) -- false, or 254 where the
// reference indexes MaxLevelHashes out of range and panics -- and at the end the summary Done() builds is compared with the recorded
// one.  The state lives in global scratch `m`, not on the thread's stack.
BD_HD uint8_t rq_eval(const uint8_t* base, const MvccRange& g, const StateSetDev& set, const MvccArrays& a, bool use_block, MerkleState* m)
{
    if (g.form == RF_BAD || (g.form == RF_MERKLE && g.degree < 2)) return MC_UNDET;   // newMerkleTree fails: the reference fails the commit
    RangeIt it;
    rq_begin(it, base, g, set, a, use_block);
    const uint8_t* key = nullptr; uint32_t kl = 0; unsigned long long blk = 0, txn = 0;
    if (g.form == RF_MERKLE) {
        mk_init(*m, base, g.body, g.degree, g.level);
        for (;;) {
            const int r = rq_next(it, key, kl, blk, txn);
            if (r == 2) return MC_UNDET;
            if (r == 0) break;
            mk_add(*m, key, kl, blk, txn);
            if (m->overflow) return MC_UNDET;
            const int e = mk_early(*m);
            if (e) return e == 1 ? MC_FAIL : MC_UNDET;
        }
        const int d = mk_done(*m, g.degree);
        return d < 0 ? MC_UNDET : d ? MC_OK : MC_FAIL;
    }
    int r = rq_next(it, key, kl, blk, txn);
    if (r == 2) return MC_UNDET;
    bool fail = false, panic = false;
    if (g.form == RF_RAW)
        scan_msg(base, g.body, BD_F(1), 0, [&](uint32_t, Seg kv) {
            if (fail || panic || r == 2) return;
            Seg rk; rk.off = rk.len = 0; unsigned long long rb = 0, rt = 0; bool hv = false;
            scan_msg(base, kv, BD_F(1) | BD_F(2), 0, [&](uint32_t h, Seg v) { if (h == 1) rk = v; else { hv = true; mv_version(base, v, rb, rt); } });
            if (r == 0 || bytes_cmp(key, kl, base + rk.off, rk.len) != 0) { fail = true; return; }
            if (!hv) { panic = true; return; }
            if (blk != rb || txn != rt) { fail = true; return; }
            r = rq_next(it, key, kl, blk, txn);
        });
    if (panic) return MC_UNDET;
    if (fail) return MC_FAIL;
    if (r == 2) return MC_UNDET;
    return r == 0 ? MC_OK : MC_FAIL;
}

// One thread per range record, before the walk: its slice of the block's sorted written public keys, whether an earlier transaction
// writes in it (those keys, and a written end key that will be served, count as contended from here on), and its answer against the
// committed state alone.
BD_HD void mv_range_rec(uint32_t q, const uint8_t* base, MvccArrays& a, const StateSetDev& set)
{
    MvccRange& g = a.rng[q];
    if (g.form == RF_BAD || (g.form == RF_MERKLE && g.degree < 2)) { g.c = MC_UNDET; return; }
    const uint32_t W = a.ctr[5];
    const KeyRef s = key_ref(base + g.ns.off, g.ns.len, base + g.start.off, g.start.len);
    const KeyRef bound = key_ref(base + g.ns.off, g.ns.len, base + g.end.off, g.end.len);
    g.lo = (uint32_t)ri_lower(a.wk, 0, W, base, s);
    uint32_t lo = g.lo, hi = W;                                       // the first key past the range: ri_below_end turns false once
    while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (ri_below_end(key_ref(base, a.wk[mid]), bound)) lo = mid + 1; else hi = mid; }
    g.hi = lo;
    bool marked = false;
    for (uint32_t j = g.lo; j < g.hi; j++) {
        MvccKey& e = a.key[a.wk[j].k];
        if (mv_first(e) < g.tx) { marked = true; e.rng = 1; }
    }
    if (!g.exhausted) {
        uint32_t w[8];
        sv_key(base + g.ns.off, g.ns.len, nullptr, 0, base + g.end.off, g.end.len, w);
        const uint32_t k = mv_find_key(a, set.seed, w);
        if (k != UINT32_MAX && a.key[k].nw) {
            g.endk = k + 1;
            if (mv_first(a.key[k]) < g.tx) { marked = true; a.key[k].rng = 1; }
        }
    }
    g.marked = marked ? 1 : 0;
    g.ib = ri_lower(a.ix.base, 0, a.ix.nb, a.ix.heap, s);
    g.id = ri_lower(a.ix.delta, 0, a.ix.nd, a.ix.heap, s);
    g.c = rq_eval(base, g, set, a, false, a.mk + q);
}

// In the walk: the answer of a marked range record against the running state; the committed answer stands when no key of the range (nor
// the end key) has entered `updates` yet
BD_HD uint8_t mv_range_walk(const uint8_t* base, uint32_t q, const StateSetDev& set, const MvccArrays& a)
{
    const MvccRange& g = a.rng[q];
    if (!g.marked) return g.c;                                     // (a form not decoded is never marked)
    bool moved = g.endk && a.key[g.endk - 1].rs != RS_NONE;
    for (uint32_t j = g.lo; j < g.hi && !moved; j++) moved = a.key[a.wk[j].k].rs != RS_NONE;
    return moved ? rq_eval(base, g, set, a, true, a.mk + q) : g.c;
}

// A write's keyOpsFlag: upsertVal 1, metadataUpdate 2, metadataDelete 4, keyDelete 8 (tx_ops.go:162-169).  prepareTxOps ADDS them per
// (transaction, key) in a uint8 (tx_ops.go:185-205), so a kind given twice carries into the next bit: two writes are 2, two deletes 16.
BD_HD uint32_t mv_weight(uint8_t kind) { return kind == MR_PUT ? 1u : kind == MR_META ? 2u : kind == MR_MDEL ? 4u : 8u; }

// What applyWriteSet does with a key of flag f (tx_ops.go:218-232, types.go:93-108): MR_DEL for isDelete, MR_PUT for isUpsertAndMetadataUpdate
// and isOnlyUpsert (the last write's value), MR_META for every other flag (the latest value re-put, or the key dropped when absent)
BD_HD uint8_t mv_class(uint32_t f)
{
    f &= 0xffu;
    if (f & 8u) return MR_DEL;
    if (((f & 1u) && (f & 6u)) || (f | 1u) == 1u) return MR_PUT;
    return MR_META;
}

// Stage 4, one thread per transaction: every flag other than VALID is copied; a VALID transaction that touches no key an earlier
// transaction of the block writes is decided on the committed table alone, the others are marked for the walk.
BD_HD void mv_mark_tx(uint32_t t, const uint8_t* tv, MvccArrays& a, uint8_t* flags)
{
    const uint8_t f = tv[t];
    flags[t] = f;
    if (f != TXC_VALID && f != TXC_NOT_VALIDATED) return;
    if (a.ctr[1] || a.ctr[0] > a.R_cap) { flags[t] = TXC_NOT_VALIDATED; return; }
    bool marked = false, fail = false, undet = false, nil_put = false;
    for (uint32_t q = a.first_rec[t]; q < a.first_rec[t] + a.n_rec[t]; q++) {
        const MvccRec& r = a.rec[q];
        const MvccKey& e = a.key[r.key];
        if (r.kind == MR_READ) {
            if (e.nw && mv_first(e) < t) marked = true;
            fail = fail || r.c == MC_FAIL; undet = undet || r.c == MC_UNDET;
        } else {
            marked = marked || mv_contended(e);
            nil_put = nil_put || (r.kind == MR_PUT && !r.has_ver);    // one write per key here: PutValAndMetadata of a nil value panics
        }
    }
    if (a.indexed)
        for (uint32_t q = a.first_rng[t]; q < a.first_rng[t] + a.n_rng[t]; q++) {
            const MvccRange& g = a.rng[q];
            marked = marked || g.marked;
            fail = fail || g.c == MC_FAIL; undet = undet || g.c == MC_UNDET;
        }
    if (marked) { a.info[t] |= MV_MARKED; return; }
    if (f != TXC_VALID) return;
    flags[t] = (a.info[t] & (MV_RANGE | MV_OPEN)) || t > a.ctr[2] || undet ? TXC_NOT_VALIDATED : fail ? 11 : nil_put ? TXC_NOT_VALIDATED : TXC_VALID;
}

// Stage 5, one thread, the marked transactions in index order: a VALID one is decided against the running state of the keys earlier
// transactions wrote, then the writes of every one left VALID or 254 enter that state.  Costs the transaction's own records.
// Indexed: the stage decides range records (base, set: the block and the table they read); the plain instantiation is the stage without
// an index, compiled without the range code
template <bool Indexed = false>
BD_HD void mv_walk_step(uint32_t t, const uint8_t* tv, MvccArrays& a, uint8_t* flags, const uint8_t* base = nullptr, const StateSetDev* set = nullptr)
{
    const uint32_t b = a.first_rec[t], end = b + a.n_rec[t];
    uint8_t f = tv[t];
    // the transaction's flag per key in the low byte (tx_ops.go:59-120,185-205), and in bit 8 whether its last write had no value (the
    // value an upsert leaves, tx_ops.go:185-189): in record order, which is each field's wire order as in the reference's slices
    for (uint32_t q = b; q < end; q++) {
        const MvccRec& r = a.rec[q];
        if (r.kind == MR_READ) continue;
        MvccKey& e = a.key[r.key];
        if (e.op_tx != t + 1) { e.op_tx = t + 1; e.op = 0; }
        const uint32_t nil = r.kind == MR_PUT ? (r.has_ver ? 0u : 0x100u) : e.op & 0x100u;
        e.op = ((e.op + mv_weight(r.kind)) & 0xffu) | nil;
    }
    if (f == TXC_VALID) {
        bool fail = false, undet = false, nil_put = false;
        for (uint32_t q = b; q < end; q++) {
            const MvccRec& r = a.rec[q];
            const MvccKey& e = a.key[r.key];
            if (r.kind == MR_READ) {
                const uint8_t c = e.nw && mv_first(e) < t ? (e.rs == RS_PUT || e.rs == RS_DEL ? MC_FAIL : e.rs == RS_UNDET ? MC_UNDET : r.c) : r.c;
                fail = fail || c == MC_FAIL; undet = undet || c == MC_UNDET;
            } else {
                // PutValAndMetadata panics on a nil value (statedb.go:202-205): an upsert whose last write has no value, or the latest
                // value of a key an earlier transaction of the block deleted -- or may have deleted (an undetermined writer)
                const uint8_t cls = mv_class(e.op);
                nil_put = nil_put || (cls == MR_PUT && (e.op & 0x100u)) || (cls == MR_META && (e.rs == RS_DEL || e.rs == RS_UNDET));
            }
        }
        if constexpr (Indexed)
            for (uint32_t q = a.first_rng[t]; q < a.first_rng[t] + a.n_rng[t]; q++) {
                const uint8_t c = mv_range_walk(base, q, *set, a);
                fail = fail || c == MC_FAIL; undet = undet || c == MC_UNDET;
            }
        f = (a.info[t] & (MV_RANGE | MV_OPEN)) || t > a.ctr[2] || undet ? TXC_NOT_VALIDATED : fail ? 11 : nil_put ? TXC_NOT_VALIDATED : TXC_VALID;
        flags[t] = f;
    }
    if (f != TXC_VALID && f != TXC_NOT_VALIDATED) return;
    for (uint32_t q = b; q < end; q++) {
        const MvccRec& r = a.rec[q];
        if (r.kind == MR_READ) continue;
        MvccKey& e = a.key[r.key];
        if (!mv_contended(e)) continue;
        if (f == TXC_NOT_VALIDATED) { e.rs = RS_UNDET; continue; }
        const uint8_t cls = mv_class(e.op);
        if (cls == MR_DEL) e.rs = RS_DEL;
        else if (cls == MR_PUT) { e.rs = RS_PUT; e.rs_tx = t; }
        else if (e.rs == RS_PUT) e.rs_tx = t;                         // metadata path: the latest value at this height (tx_ops.go:41-51)
        else if (e.rs == RS_NONE) {
            if (r.c == MC_EXISTS) { e.rs = RS_PUT; e.rs_tx = t; }
            else if (r.c == MC_UNDET) e.rs = RS_UNDET;                // absent: the operation is dropped
        }
    }
}

// Stage 6, one thread per entry of the block's key table: the key's final state enters the committed table at (block, tx)
BD_HD void mv_apply_key(uint32_t k, MvccArrays& a, const uint8_t* flags, const StateSetDev& set, unsigned long long block, int* full)
{
    const MvccKey& e = a.key[k];
    if (a.ctr[1] || a.ctr[0] > a.R_cap || !e.tag || !e.nw) return;
    uint32_t state = SV_EMPTY; unsigned long long txn = 0;
    if (mv_contended(e)) {
        if (e.rs == RS_PUT) { state = SV_PRESENT; txn = e.rs_tx; }
        else if (e.rs == RS_DEL) state = SV_REMOVED;
        else if (e.rs == RS_UNDET) state = SV_UNKNOWN;
    } else {
        const MvccRec& r = a.rec[e.wrec];
        const uint8_t f = flags[r.tx];
        if (f == TXC_NOT_VALIDATED) state = SV_UNKNOWN;
        else if (f == TXC_VALID) {
            txn = r.tx;
            if (r.kind == MR_PUT) state = SV_PRESENT;
            else if (r.kind == MR_DEL) state = SV_REMOVED;
            else state = r.c == MC_EXISTS ? SV_PRESENT : r.c == MC_UNDET ? SV_UNKNOWN : SV_EMPTY;
        }
    }
    if (state == SV_EMPTY) return;
    if (sv_upsert(set, e.w, state, state == SV_PRESENT ? block : 0ull, txn) < 0) *full = 1;
}

// ---- index maintenance (fabgpu_state_versions_update, and the stage after its apply) -----------------------------------------------
// One thread per candidate (sorted, keys distinct): flag[i] = 1 for a key the table now holds (present or unknown) that the index lacks,
// so a later range sees it -- and answers 254 for an unknown one
BD_HD void ix_flag(uint32_t i, const WrittenKey* c, const uint8_t* src, const StateIndexDev& x, const StateSetDev& set, uint32_t* flag)
{
    unsigned long long b = 0, t = 0;
    const uint32_t st = set.broken ? SV_EMPTY : sv_lookup(set, c[i].w, b, t);
    flag[i] = (st == SV_PRESENT || st == SV_UNKNOWN) && !ri_contains(x, key_ref(src, c[i])) ? 1u : 0u;
}

// A flagged candidate becomes entry `out` of the new run, its bytes at heap + at
BD_HD void ix_emit(const WrittenKey& c, const uint8_t* src, uint8_t* heap, unsigned long long at, IndexEntry& out)
{
    for (uint32_t k = 0; k < c.nl; k++) heap[at + k] = src[c.ns_off + k];
    for (uint32_t k = 0; k < c.kl; k++) heap[at + c.nl + k] = src[c.key_off + k];
    out.off = at; out.nl = c.nl; out.kl = c.kl;
    for (int k = 0; k < 8; k++) out.w[k] = c.w[k];
}

#if defined(__CUDACC__)
// fabgpu_state_versions / _update: one thread per entry of the call (keys distinct within the call)
__global__ void __launch_bounds__(256)
sv_insert_kernel(StateSetDev set, const StateSlot* __restrict__ rec, uint32_t n, int* __restrict__ full)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[8];
    for (int k = 0; k < 8; k++) w[k] = rec[i].w[k];
    if (sv_upsert(set, w, rec[i].state, rec[i].blk, rec[i].txn) < 0) *full = 1;
}

// Growth: one thread per slot of the old table re-inserts its key (removed keys are dropped)
__global__ void __launch_bounds__(256)
sv_rehash_kernel(StateSetDev set, const StateSlot* __restrict__ old, uint64_t n_old, int* __restrict__ full)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_old) return;
    const uint32_t st = old[i].state;
    if (st != SV_PRESENT && st != SV_UNKNOWN) return;
    uint32_t w[8];
    for (int k = 0; k < 8; k++) w[k] = old[i].w[k];
    if (sv_upsert(set, w, st, old[i].blk, old[i].txn) < 0) *full = 1;
}

__global__ void __launch_bounds__(64)
mv_scan_kernel(const uint8_t* __restrict__ block, const TxDev* __restrict__ txs, uint32_t T, const uint8_t* __restrict__ tv, MvccArrays a)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < T) mv_scan_tx(block, txs[t], t, tv[t], a);
}

__global__ void __launch_bounds__(256)
mv_key_kernel(MvccArrays a, StateSetDev set, uint32_t R)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < R) mv_key_rec(i, a, set);
}

__global__ void __launch_bounds__(256)
mv_check_kernel(MvccArrays a, uint32_t R)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < R) mv_check_rec(i, a);
}

__global__ void __launch_bounds__(128)
mv_mark_kernel(const uint8_t* __restrict__ tv, MvccArrays a, uint8_t* __restrict__ flags, uint32_t T)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < T) mv_mark_tx(t, tv, a, flags);
}

// Range queries: the block's written public keys (one thread per entry of the key table), their merge sort (one launch per pass, runs of
// `width`), then one thread per range record
__global__ void __launch_bounds__(256)
mv_written_kernel(MvccArrays a)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < a.K_size && !a.ctr[1] && a.ctr[0] <= a.R_cap) mv_written_key(k, a);
}

__global__ void __launch_bounds__(256)
mv_sort_kernel(const WrittenKey* __restrict__ in, WrittenKey* __restrict__ out, const uint32_t* __restrict__ ctr, uint32_t width, const uint8_t* __restrict__ block)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < ctr[5]) ri_sort_one(in, i, ctr[5], width, block, out);
}

__global__ void __launch_bounds__(128)
mv_range_kernel(const uint8_t* __restrict__ block, MvccArrays a, StateSetDev set, uint32_t G)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < G && !a.ctr[1] && a.ctr[0] <= a.R_cap) mv_range_rec(q, block, a, set);
}

// One CTA: the marked transactions are compacted by a block-wide scan (as in block_kl_resolve_kernel), then one thread walks them in
// index order.  mv_walk_kernel<false> is the stage without an index; <true> also decides the marked range records.
template <bool Indexed>
__global__ void __launch_bounds__(256)
mv_walk_kernel(const uint8_t* __restrict__ tv, MvccArrays a, uint8_t* __restrict__ flags, uint32_t T, const uint8_t* __restrict__ block, StateSetDev set)
{
    __shared__ uint32_t warp_sum[32];
    if (a.ctr[1] || a.ctr[0] > a.R_cap) return;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, per = (T + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(T, tid * per), hi = min(T, lo + per);
    uint32_t c = 0;
    for (uint32_t t = lo; t < hi; t++) c += (a.info[t] & MV_MARKED) != 0;
    uint32_t x = c;
    for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t v = lane < blockDim.x / 32 ? warp_sum[lane] : 0;
        for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += y; }
        warp_sum[lane] = v;
    }
    __syncthreads();
    uint32_t off = x - c + (warp ? warp_sum[warp - 1] : 0);
    for (uint32_t t = lo; t < hi; t++) if (a.info[t] & MV_MARKED) a.mlist[off++] = t;
    const uint32_t total = warp_sum[31];
    __syncthreads();
    if (tid != 0) return;
    a.ctr[3] = total;
    for (uint32_t k = 0; k < total; k++) mv_walk_step<Indexed>(a.mlist[k], tv, a, flags, block, &set);
}

__global__ void __launch_bounds__(256)
mv_apply_kernel(MvccArrays a, const uint8_t* __restrict__ flags, StateSetDev set, unsigned long long block, int* __restrict__ full)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < a.K_size) mv_apply_key(k, a, flags, set, block, full);
}

// Index maintenance over n sorted candidates (n_p: a device count instead): flags, then one CTA writes the flagged ones, in order, as the
// new run (icnt[2] entries) with their bytes appended to the heap (icnt[3]); the run merges with the delta; ix_fin_kernel settles the counts
__global__ void __launch_bounds__(256)
ix_flag_kernel(const WrittenKey* __restrict__ c, uint32_t n, const uint32_t* __restrict__ n_p, const uint8_t* __restrict__ src, StateIndexDev x,
               StateSetDev set, uint32_t* __restrict__ flag)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (n_p ? *n_p : n)) ix_flag(i, c, src, x, set, flag);
}

__global__ void __launch_bounds__(1024)
ix_compact_kernel(const WrittenKey* __restrict__ c, uint32_t n, const uint32_t* __restrict__ n_p, const uint8_t* __restrict__ src,
                  const uint32_t* __restrict__ flag, uint8_t* __restrict__ heap, IndexEntry* __restrict__ out, unsigned long long* __restrict__ icnt)
{
    __shared__ unsigned long long sn[32], sb[32];
    if (n_p) n = *n_p;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, per = (n + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(n, tid * per), hi = min(n, lo + per);
    unsigned long long cn = 0, cb = 0;
    for (uint32_t i = lo; i < hi; i++) if (flag[i]) { cn++; cb += c[i].nl + c[i].kl; }
    unsigned long long xn = cn, xb = cb;
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const unsigned long long yn = __shfl_up_sync(0xffffffffu, xn, d), yb = __shfl_up_sync(0xffffffffu, xb, d);
        if (lane >= d) { xn += yn; xb += yb; }
    }
    if (lane == 31) { sn[warp] = xn; sb[warp] = xb; }
    __syncthreads();
    if (warp == 0) {
        unsigned long long vn = lane < blockDim.x / 32 ? sn[lane] : 0, vb = lane < blockDim.x / 32 ? sb[lane] : 0;
        for (uint32_t d = 1; d < 32; d <<= 1) {
            const unsigned long long yn = __shfl_up_sync(0xffffffffu, vn, d), yb = __shfl_up_sync(0xffffffffu, vb, d);
            if (lane >= d) { vn += yn; vb += yb; }
        }
        sn[lane] = vn; sb[lane] = vb;
    }
    __syncthreads();
    const unsigned long long h0 = icnt[3];
    unsigned long long off = xn - cn + (warp ? sn[warp - 1] : 0), at = h0 + xb - cb + (warp ? sb[warp - 1] : 0);
    for (uint32_t i = lo; i < hi; i++)
        if (flag[i]) { ix_emit(c[i], src, heap, at, out[off]); off++; at += c[i].nl + c[i].kl; }
    __syncthreads();
    if (tid == 0) { icnt[2] = sn[31]; icnt[3] = h0 + sb[31]; }
}

// out = merge of the sorted runs A (*na entries) and B (*nb), keys disjoint; one thread per entry of either
__global__ void __launch_bounds__(256)
ix_merge_kernel(const IndexEntry* __restrict__ A, const unsigned long long* __restrict__ na, const IndexEntry* __restrict__ B,
                const unsigned long long* __restrict__ nb, const uint8_t* __restrict__ heap, IndexEntry* __restrict__ out)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, n_a = *na, n_b = *nb;
    if (i < n_a) ri_merge_one(A, i, B, n_b, heap, out, 0);
    else if (i < n_a + n_b) ri_merge_one(B, i - n_a, A, n_a, heap, out, 0);
}

// fold = 0: the new run joined the delta; 1: the delta joined the base
__global__ void ix_fin_kernel(unsigned long long* icnt, int fold)
{
    if (fold) { icnt[0] += icnt[1]; icnt[1] = 0; }
    else { icnt[1] += icnt[2]; icnt[2] = 0; }
}

// fabgpu_state_index_info: icnt[4] = entries the table holds (present or unknown)
__global__ void __launch_bounds__(256)
ix_live_kernel(StateIndexDev x, StateSetDev set, unsigned long long* __restrict__ icnt)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= x.nb + x.nd) return;
    const IndexEntry& e = i < x.nb ? x.base[i] : x.delta[i - x.nb];
    unsigned long long b = 0, t = 0;
    if (!set.broken && sv_lookup(set, e.w, b, t) != SV_EMPTY) atomicAdd(icnt + 4, 1ull);
}
#endif

} }  // namespace fabgpu::bdev
