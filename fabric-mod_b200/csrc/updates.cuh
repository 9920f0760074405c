// The block's public and hashed update batch (fabgpu_block_updates): what applyWriteSet leaves in publicUpdates and hashUpdates for the
// transactions the MVCC stage left VALID (core/ledger/kvledger/txmgmt/validation/types.go:81-111, tx_ops.go:18-232).  Host+device code: the
// tests' host build runs the same steps one item at a time.
//
// Built from what the stage left behind -- its records (MvccRec: transaction, key-table entry, kind, the committed existence `c` looked
// up before its apply), the per-transaction record ranges and the final flags -- never from the committed table, which the apply changed.
// Each (transaction, key) pair of a VALID write gets one entry of a hash table holding prepareTxOps' flag sum (mv_weight) and the pair's
// last upsert, last metadataUpdate and first write, in wire order (record indices of one transaction grow in wire order).  Every key then
// resolves from its last VALID writer L:
//   delete (flag & 8)                          DELETE
//   isUpsertAndMetadataUpdate                  PUT of L's last upsert, L's metadata bytes (nil without a metadataUpdate)
//   isOnlyUpsert                               PUT of L's last upsert, the metadata of the nearest earlier writer that sets it (below)
//   metadata path (every other flag)           PUT of the nearest earlier upsert's value (or the committed one), L's metadata bytes;
//                                              dropped when no earlier writer put the key and it is not committed (tx_ops.go:41-51)
// "Nearest earlier" is the largest VALID writer below L of the right class, found with atomicMax over the key's pairs -- no serial walk,
// O(records) in all.  A metadata-path writer sets the key's metadata only when it was not dropped, i.e. when an earlier writer of the
// block put or deleted the key, or the key is committed.  What the committed state supplies is left to the peer (COMMITTED sources); a
// resolution that depends on a key the table marks unknown makes the batch incomplete.
#pragma once
#include "stateset.cuh"

namespace fabgpu { namespace bdev {

// classes of a (transaction, key) flag sum: isDelete, isUpsertAndMetadataUpdate, isOnlyUpsert, the metadata path
enum : uint32_t { UC_DEL = 1, UC_PUTMD = 2, UC_UPSERT = 3, UC_META = 4 };
// record fields (FABGPU_UPDATE_* in fabgpu_ecdsa.h)
enum : uint32_t { UD_PUT = 1, UD_DELETE = 2 };
enum : uint32_t { UD_NONE = 0, UD_BLOCK = 1, UD_COMMITTED = 2 };                 // value source; metadata: nil, bytes, committed
constexpr uint32_t UD_WORDS = 14, UD_NONCANON = 0xffffffffu;

struct UdPair {
    unsigned long long tag;             // ((tx << 32) | key-table entry) + 1; 0 = empty
    uint32_t sum;                       // prepareTxOps' flag sum (mod 256 when read)
    uint32_t last_put, last_meta;       // record index + 1 of the last upsert / metadataUpdate (0 none)
    uint32_t nfirst;                    // UINT32_MAX - the pair's first write record
    uint32_t cls, pad;
};

struct UdKey {
    uint32_t L;                         // last VALID writer + 1 (0: no VALID write)
    uint32_t nfdup, nfm;                // UINT32_MAX - first writer of class delete / upsert (UC_DEL..UC_UPSERT), of the metadata path (0 none)
    uint32_t val_w, meta_w;             // nearest writer below L that sets the value / the metadata, + 1
    uint32_t pair_l;                    // L's pair
    uint32_t op, vsrc, vrec, msrc, mrec, nrec;   // the resolved record: value and metadata records, names (L's first write of the key)
};

// One needed record's byte ranges: names, and the value (an upsert) or the KVMetadataWrite body (a metadataUpdate); mlen: the metadata's
// Serialize length, UD_NONCANON when an entry is not canonical
struct UdSeg { Seg ns, coll, key, val; uint32_t mlen; };

struct UdArrays {
    const MvccRec* rec; const uint32_t* first_rec; const uint32_t* n_rec; const uint8_t* flags;   // the stage's (flags: final)
    uint32_t R, T, K;                   // records, transactions, key-table entries
    UdPair* pair; uint32_t P_size;      // power of two >= 2 R
    UdKey* key;                         // K entries
    uint32_t* base;                     // per transaction: its first record's position in transaction order
    uint32_t* mark;                     // per position: key-table entry + 1 of the record emitted there (0 none)
    uint8_t* need; uint8_t* txneed;     // per record / transaction: segments wanted
    UdSeg* seg;                         // per record
    uint32_t* out_key; uint32_t* out_moff;   // per output record
    uint32_t* out; uint8_t* meta;       // UD_WORDS words per record; metadata bytes
    uint32_t* ctr;                      // [0] incomplete, [1] records, [2] metadata bytes
};

BD_HD uint32_t ud_class(uint32_t f)
{
    f &= 0xffu;
    if (f & 8u) return UC_DEL;
    if ((f & 1u) && (f & 6u)) return UC_PUTMD;
    if ((f | 1u) == 1u) return UC_UPSERT;
    return UC_META;
}

BD_HD void ud_incomplete(UdArrays& a) { a.ctr[0] = 1; }

// the pair table's first probe (tags are transaction and table indices, not submitter-chosen bytes)
BD_HD uint64_t ud_mix(uint64_t h) { h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; return h ^ (h >> 33); }

BD_HD uint32_t ud_pair_find(const UdArrays& a, uint32_t tx, uint32_t k)
{
    const unsigned long long tag = (((unsigned long long)tx << 32) | k) + 1ull;
    uint32_t pos = (uint32_t)ud_mix(tag) & (a.P_size - 1);
    for (uint32_t probe = 0; probe < a.P_size; probe++, pos = (pos + 1) & (a.P_size - 1)) {
        if (a.pair[pos].tag == tag) return pos;
        if (a.pair[pos].tag == 0) return UINT32_MAX;
    }
    return UINT32_MAX;
}

// Step 1, one thread per record: a VALID write joins its (transaction, key) pair, and the key's last VALID writer
BD_HD void ud_pair_rec(uint32_t i, UdArrays& a)
{
    const MvccRec& r = a.rec[i];
    if (r.kind == MR_READ || a.flags[r.tx] != TXC_VALID) return;
    const unsigned long long tag = (((unsigned long long)r.tx << 32) | r.key) + 1ull;
    uint32_t pos = (uint32_t)ud_mix(tag) & (a.P_size - 1);
    for (uint32_t probe = 0; probe < a.P_size; probe++, pos = (pos + 1) & (a.P_size - 1)) {
#if defined(__CUDA_ARCH__)
        const unsigned long long old = atomicCAS(&a.pair[pos].tag, 0ull, tag);
#else
        const unsigned long long old = a.pair[pos].tag; if (old == 0) a.pair[pos].tag = tag;
#endif
        if (old != 0 && old != tag) continue;
        UdPair& p = a.pair[pos];
        kl_atomic_add(&p.sum, mv_weight(r.kind));
        if (r.kind == MR_PUT) mv_atomic_max(&p.last_put, i + 1);
        if (r.kind == MR_META) mv_atomic_max(&p.last_meta, i + 1);
        mv_atomic_max(&p.nfirst, UINT32_MAX - i);
        mv_atomic_max(&a.key[r.key].L, r.tx + 1);
        return;
    }
    ud_incomplete(a);                                              // (the table holds 2 R entries: not reached)
}

// Step 2, one thread per pair: its class; the key's first writers of each kind; L's pair
BD_HD void ud_class_pair(uint32_t p, UdArrays& a)
{
    UdPair& e = a.pair[p];
    if (!e.tag) return;
    const uint32_t tx = (uint32_t)((e.tag - 1) >> 32), k = (uint32_t)(e.tag - 1);
    e.cls = ud_class(e.sum);
    UdKey& u = a.key[k];
    mv_atomic_max(e.cls == UC_META ? &u.nfm : &u.nfdup, UINT32_MAX - tx);
    if (u.L == tx + 1) u.pair_l = p;
}

// Step 3, one thread per pair below its key's L: the nearest earlier writer that sets the value (an upsert, or a delete) and the one that
// sets the metadata (a delete, an upsert with metadata, or a metadata-path writer that was not dropped)
BD_HD void ud_walk_pair(uint32_t p, UdArrays& a)
{
    const UdPair& e = a.pair[p];
    if (!e.tag) return;
    const uint32_t tx = (uint32_t)((e.tag - 1) >> 32), k = (uint32_t)(e.tag - 1);
    UdKey& u = a.key[k];
    if (tx + 1 >= u.L) return;
    if (e.cls != UC_META) mv_atomic_max(&u.val_w, tx + 1);
    const bool put_before = u.nfdup && UINT32_MAX - u.nfdup < tx;
    const bool kept = e.cls == UC_DEL || e.cls == UC_PUTMD || (e.cls == UC_META && (put_before || a.rec[UINT32_MAX - e.nfirst].c == MC_EXISTS));
    if (kept) mv_atomic_max(&u.meta_w, tx + 1);
}

// Step 4 (before 5), the transactions' record positions in transaction order: base[t] = records of transactions below t
BD_HD void ud_base_host(UdArrays& a)
{
    uint32_t s = 0;
    for (uint32_t t = 0; t < a.T; t++) { a.base[t] = s; s += a.n_rec[t]; }
}

BD_HD void ud_want(UdArrays& a, uint32_t i) { a.need[i] = 1; a.txneed[a.rec[i].tx] = 1; }

// Step 5, one thread per key-table entry with a VALID write: the key's record (or none: a dropped metadata-only write)
BD_HD void ud_resolve_key(uint32_t k, UdArrays& a)
{
    UdKey& u = a.key[k];
    if (!u.L) return;
    const uint32_t L = u.L - 1;
    const UdPair& e = a.pair[u.pair_l];
    const uint8_t c = a.rec[UINT32_MAX - e.nfirst].c;             // the key's committed existence before the apply
    u.nrec = UINT32_MAX - e.nfirst;
    u.vsrc = UD_NONE; u.msrc = UD_NONE; u.op = 0;
    if (e.cls == UC_DEL) u.op = UD_DELETE;
    else if (e.cls == UC_PUTMD || e.cls == UC_UPSERT) {
        if (!e.last_put) { ud_incomplete(a); return; }            // a sum of 0 from metadata writes alone: a nil value
        u.op = UD_PUT; u.vsrc = UD_BLOCK; u.vrec = e.last_put - 1;
        if (e.cls == UC_PUTMD) {
            if (e.last_meta) { u.msrc = UD_BLOCK; u.mrec = e.last_meta - 1; }
        } else if (u.meta_w) {
            const uint32_t q = ud_pair_find(a, u.meta_w - 1, k);
            if (q == UINT32_MAX) { ud_incomplete(a); return; }
            if (a.pair[q].cls != UC_DEL && a.pair[q].last_meta) { u.msrc = UD_BLOCK; u.mrec = a.pair[q].last_meta - 1; }
        } else {
            // every earlier writer is an upsert or a dropped metadata-path writer: the committed metadata -- unless whether such a
            // writer was dropped is unknown
            if (c == MC_UNDET && u.nfm && UINT32_MAX - u.nfm < L) { ud_incomplete(a); return; }
            u.msrc = UD_COMMITTED;
        }
    } else {
        if (u.val_w) {
            const uint32_t q = ud_pair_find(a, u.val_w - 1, k);
            if (q == UINT32_MAX || a.pair[q].cls == UC_DEL || !a.pair[q].last_put) { ud_incomplete(a); return; }   // a deleted value: nil
            u.vsrc = UD_BLOCK; u.vrec = a.pair[q].last_put - 1;
        } else if (c == MC_EXISTS) u.vsrc = UD_COMMITTED;
        else if (c == MC_UNDET) { ud_incomplete(a); return; }
        else return;                                               // absent: the operation is dropped
        u.op = UD_PUT;
        if (e.last_meta) { u.msrc = UD_BLOCK; u.mrec = e.last_meta - 1; }
    }
    ud_want(a, u.nrec);
    if (u.vsrc == UD_BLOCK) ud_want(a, u.vrec);
    if (u.msrc == UD_BLOCK) ud_want(a, u.mrec);
    a.mark[a.base[L] + (u.nrec - a.first_rec[L])] = k + 1;
}

// A minimal varint at p (below end): its value and the byte after it; false when it is cut short, longer than needed, or over 32 bits
BD_HD bool ud_varint(const uint8_t* b, uint32_t& p, uint32_t end, uint32_t& v)
{
    v = 0;
    for (int shift = 0; shift < 35; shift += 7) {
        if (p >= end) return false;
        const uint8_t c = b[p++];
        if (shift == 28 && c > 0x0f) return false;
        v |= (uint32_t)(c & 0x7f) << shift;
        if (!(c & 0x80)) return c != 0 || shift == 0;
    }
    return false;
}

BD_HD uint32_t ud_varint_len(uint32_t v) { uint32_t n = 1; while (v >= 0x80) { v >>= 7; n++; } return n; }

// KVMetadataEntry{name = 1, value = 2} that golang/protobuf re-marshals to the same bytes: name then value, each at most once and
// non-empty when present, minimal tags and lengths, nothing else
BD_HD bool ud_entry_canonical(const uint8_t* b, Seg e)
{
    uint32_t p = e.off, end = e.off + e.len, n = 0;
    for (uint8_t tag = 0x0a; tag <= 0x12; tag += 8) {
        if (p < end && b[p] == tag) {
            p++;
            if (!ud_varint(b, p, end, n) || n == 0 || end - p < n) return false;
            p += n;
        }
    }
    return p == end;
}

// The Serialize length of a KVMetadataWrite body's entries (field 2, in wire order), UD_NONCANON when one is not canonical
BD_HD uint32_t ud_meta_len(const uint8_t* base, Seg body)
{
    Reader r; r.base = base; r.pos = body.off; r.end = body.off + body.len; r.ok = true;
    uint32_t f, wt, n = 0; uint64_t x = 0; Seg b; b.off = b.len = 0;
    while (r.next(f, wt, x, b))
        if (f == 2) {
            if (wt != 2 || !ud_entry_canonical(base, b)) return UD_NONCANON;
            n += 1 + ud_varint_len(b.len) + b.len;
        }
    return r.ok ? n : UD_NONCANON;
}

// Step 6, one thread per transaction holding a wanted record: one re-scan of its write set, as mv_scan enumerates records (every field
// but a range query), filling the wanted records' segments
BD_HD void ud_seg_tx(uint32_t t, const uint8_t* base, const TxDev& tx, UdArrays& a)
{
    if (!a.txneed[t]) return;
    uint32_t i = a.first_rec[t];
    kl_scan_rwset<true>(base, tx.results, [&](Seg ns, Seg coll, Seg key, uint32_t g, Seg body) {
        if (g == 2) return true;
        if (a.need[i]) {
            UdSeg& s = a.seg[i];
            s.ns = ns; s.coll = coll; s.key = key; s.val.off = s.val.len = 0; s.mlen = 0;
            if (a.rec[i].kind == MR_META) { s.val = body; s.mlen = ud_meta_len(base, body); }
            else if (a.rec[i].kind == MR_PUT) {                       // the value (value_hash): the last field 3, as proto.Unmarshal keeps
                Reader r; r.base = base; r.pos = body.off; r.end = body.off + body.len; r.ok = true;
                uint32_t f, wt; uint64_t x = 0; Seg b; b.off = b.len = 0;
                while (r.next(f, wt, x, b)) if (f == 3 && wt == 2) s.val = b;
            }
        }
        i++;
        return true;
    });
}

// Step 7, per position in transaction order: whether a record is emitted there, and its metadata bytes
BD_HD bool ud_at(uint32_t pos, UdArrays& a, uint32_t& k, uint32_t& bytes)
{
    bytes = 0;
    if (!a.mark[pos]) return false;
    k = a.mark[pos] - 1;
    const UdKey& u = a.key[k];
    if (u.msrc == UD_BLOCK) {
        bytes = a.seg[u.mrec].mlen;
        if (bytes == UD_NONCANON) { ud_incomplete(a); bytes = 0; }
    }
    return true;
}

// Step 8, per output record: its words and its metadata's Serialize bytes (0x12 varint(len) entry, in wire order)
BD_HD void ud_emit(uint32_t o, const uint8_t* base, UdArrays& a)
{
    const uint32_t k = a.out_key[o], moff = a.out_moff[o];
    const UdKey& u = a.key[k];
    const UdSeg& nm = a.seg[u.nrec];
    uint32_t* w = a.out + (size_t)o * UD_WORDS;
    w[0] = u.L - 1; w[1] = u.op; w[2] = u.vsrc; w[3] = u.msrc;
    w[4] = nm.ns.off; w[5] = nm.ns.len; w[6] = nm.coll.off; w[7] = nm.coll.len; w[8] = nm.key.off; w[9] = nm.key.len;
    w[10] = u.vsrc == UD_BLOCK ? a.seg[u.vrec].val.off : 0; w[11] = u.vsrc == UD_BLOCK ? a.seg[u.vrec].val.len : 0;
    w[12] = moff; w[13] = 0;
    if (u.msrc != UD_BLOCK) { w[12] = 0; return; }
    const Seg body = a.seg[u.mrec].val;
    Reader r; r.base = base; r.pos = body.off; r.end = body.off + body.len; r.ok = true;
    uint32_t f, wt, at = moff; uint64_t x = 0; Seg b; b.off = b.len = 0;
    while (r.next(f, wt, x, b))
        if (f == 2) {
            a.meta[at++] = 0x12;
            for (uint32_t v = b.len; ; v >>= 7) { if (v < 0x80) { a.meta[at++] = (uint8_t)v; break; } a.meta[at++] = (uint8_t)(v | 0x80); }
            for (uint32_t j = 0; j < b.len; j++) a.meta[at++] = base[b.off + j];
        }
    w[13] = at - moff;
}

#if defined(__CUDACC__)
__global__ void __launch_bounds__(256) ud_pair_kernel(UdArrays a)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.R) ud_pair_rec(i, a);
}

__global__ void __launch_bounds__(256) ud_class_kernel(UdArrays a)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < a.P_size) ud_class_pair(p, a);
}

__global__ void __launch_bounds__(256) ud_walk_kernel(UdArrays a)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < a.P_size) ud_walk_pair(p, a);
}

// One CTA: exclusive block-wide scan of (x, y) pairs over each thread's contiguous chunk; returns the thread's offsets, totals in tot
__device__ __forceinline__ void ud_block_scan(uint32_t x, uint32_t y, uint32_t& ox, uint32_t& oy, uint32_t& tx_, uint32_t& ty)
{
    __shared__ uint32_t sx[32], sy[32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t vx = x, vy = y;
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const uint32_t a = __shfl_up_sync(0xffffffffu, vx, d), b = __shfl_up_sync(0xffffffffu, vy, d);
        if (lane >= d) { vx += a; vy += b; }
    }
    if (lane == 31) { sx[warp] = vx; sy[warp] = vy; }
    __syncthreads();
    if (warp == 0) {
        uint32_t wx = lane < blockDim.x / 32 ? sx[lane] : 0, wy = lane < blockDim.x / 32 ? sy[lane] : 0;
        for (uint32_t d = 1; d < 32; d <<= 1) {
            const uint32_t a = __shfl_up_sync(0xffffffffu, wx, d), b = __shfl_up_sync(0xffffffffu, wy, d);
            if (lane >= d) { wx += a; wy += b; }
        }
        sx[lane] = wx; sy[lane] = wy;
    }
    __syncthreads();
    ox = vx - x + (warp ? sx[warp - 1] : 0); oy = vy - y + (warp ? sy[warp - 1] : 0);
    tx_ = sx[31]; ty = sy[31];
    __syncthreads();
}

// One CTA of 1024: base[t], the transaction-order position of each transaction's first record
__global__ void __launch_bounds__(1024) ud_base_kernel(UdArrays a)
{
    const uint32_t per = (a.T + blockDim.x - 1) / blockDim.x, lo = min(a.T, threadIdx.x * per), hi = min(a.T, lo + per);
    uint32_t c = 0;
    for (uint32_t t = lo; t < hi; t++) c += a.n_rec[t];
    uint32_t off, unused, tot, tot2;
    ud_block_scan(c, 0, off, unused, tot, tot2);
    for (uint32_t t = lo; t < hi; t++) { a.base[t] = off; off += a.n_rec[t]; }
}

__global__ void __launch_bounds__(256) ud_resolve_kernel(UdArrays a)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < a.K) ud_resolve_key(k, a);
}

__global__ void __launch_bounds__(64) ud_seg_kernel(const uint8_t* __restrict__ block, const TxDev* __restrict__ txs, UdArrays a)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.T) ud_seg_tx(t, block, txs[t], a);
}

// One CTA of 1024: the emitted records in position order, their metadata offsets, and the totals (ctr[1], ctr[2])
__global__ void __launch_bounds__(1024) ud_compact_kernel(UdArrays a)
{
    const uint32_t per = (a.R + blockDim.x - 1) / blockDim.x, lo = min(a.R, threadIdx.x * per), hi = min(a.R, lo + per);
    uint32_t cn = 0, cb = 0, k, b;
    for (uint32_t pos = lo; pos < hi; pos++) if (ud_at(pos, a, k, b)) { cn++; cb += b; }
    uint32_t on, ob, tn, tb;
    ud_block_scan(cn, cb, on, ob, tn, tb);
    for (uint32_t pos = lo; pos < hi; pos++)
        if (ud_at(pos, a, k, b)) { a.out_key[on] = k; a.out_moff[on] = ob; on++; ob += b; }
    if (threadIdx.x == 0) { a.ctr[1] = tn; a.ctr[2] = tb; }
}

__global__ void __launch_bounds__(128) ud_emit_kernel(const uint8_t* __restrict__ block, UdArrays a)
{
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o < a.ctr[1]) ud_emit(o, block, a);
}
#endif

} }  // namespace fabgpu::bdev
