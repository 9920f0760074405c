// The ordered index of the world state's public keys (fabgpu_state_versions_indexed) and the pieces of the range-query check that do not
// depend on the MVCC stage's arrays: bytewise key order, searches, the rank merges that sort and extend the index, and the Merkle summary
// of rwsetutil.RangeQueryResultsHelper (query_results_helper.go).  Host+device code: the tests' host build runs the same functions.
//
// The index holds the (namespace, key) bytes of public keys, sorted bytewise (namespace first), each with the key's digest; it only answers
// which keys of a range may exist.  Presence and version always come from sv_lookup on the version table, so a removed key may stay in
// the index as a dead entry (skipped: the table does not hold it) until the next install.  Two sorted arrays: a large base and a small
// delta of later insertions; lookups merge them (their keys are disjoint), and the delta is folded into the base when it passes 1/8 of it.
#pragma once
#include "blockdev.cuh"

namespace fabgpu { namespace bdev {

// heap bytes at `off`: the namespace, then the key
struct IndexEntry { unsigned long long off; uint32_t nl, kl; uint32_t w[8]; };
// A key the block (or an update call) may add: bytes at src + ns_off / key_off; k: its entry of the block's key table
struct WrittenKey { uint32_t ns_off, nl, key_off, kl, k; uint32_t w[8]; };
// counts of the index on the device: [0] base entries, [1] delta entries, [2] new entries of a maintenance step, [3] heap bytes used,
// [4] live entries (fabgpu_state_index_info)
struct StateIndexDev { const IndexEntry* base; const IndexEntry* delta; const uint8_t* heap; unsigned long long nb, nd; uint32_t on; };

struct KeyRef { const uint8_t* ns; uint32_t nl; const uint8_t* key; uint32_t kl; };

BD_HD KeyRef key_ref(const uint8_t* ns, uint32_t nl, const uint8_t* key, uint32_t kl)
{
    KeyRef r; r.ns = ns; r.nl = nl; r.key = key; r.kl = kl; return r;
}
BD_HD KeyRef key_ref(const uint8_t* heap, const IndexEntry& e) { return key_ref(heap + e.off, e.nl, heap + e.off + e.nl, e.kl); }
BD_HD KeyRef key_ref(const uint8_t* src, const WrittenKey& e) { return key_ref(src + e.ns_off, e.nl, src + e.key_off, e.kl); }

// bytewise comparison (strings.Compare): -1, 0, 1
BD_HD int bytes_cmp(const uint8_t* a, uint32_t al, const uint8_t* b, uint32_t bl)
{
    const uint32_t n = al < bl ? al : bl;
    for (uint32_t i = 0; i < n; i++) if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return al == bl ? 0 : al < bl ? -1 : 1;
}
BD_HD int key_cmp(const KeyRef& a, const KeyRef& b)
{
    const int c = bytes_cmp(a.ns, a.nl, b.ns, b.nl);
    return c ? c : bytes_cmp(a.key, a.kl, b.key, b.kl);
}

// The first position of arr[lo, hi) whose key is not below k (keys sorted).  R: the reference type key_ref(src, T) gives and key_cmp
// orders -- KeyRef here, the three-part UbRef of updatebytes.cuh
template <typename T, typename R>
BD_HD uint64_t ri_lower(const T* arr, uint64_t lo, uint64_t hi, const uint8_t* src, const R& k)
{
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (key_cmp(key_ref(src, arr[mid]), k) < 0) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// A key lies in [start, end) of its namespace; an empty end is the rest of the namespace (LevelDB's GetStateRangeScanIterator)
BD_HD bool ri_below_end(const KeyRef& k, const KeyRef& bound)
{
    if (bytes_cmp(k.ns, k.nl, bound.ns, bound.nl) != 0) return false;
    return bound.kl == 0 || bytes_cmp(k.key, k.kl, bound.key, bound.kl) < 0;
}

// The index holds the key (base or delta)
BD_HD bool ri_contains(const StateIndexDev& x, const KeyRef& k)
{
    uint64_t p = ri_lower(x.base, 0, x.nb, x.heap, k);
    if (p < x.nb && key_cmp(key_ref(x.heap, x.base[p]), k) == 0) return true;
    p = ri_lower(x.delta, 0, x.nd, x.heap, k);
    return p < x.nd && key_cmp(key_ref(x.heap, x.delta[p]), k) == 0;
}

// Rank merge, one element: element i of the sorted run `own` goes to position i + (elements of the sorted run `other` below it) of the
// merged output.  The runs' keys are disjoint, so every position is taken once.
template <typename T>
BD_HD void ri_merge_one(const T* own, uint64_t i, const T* other, uint64_t n_other, const uint8_t* src, T* out, uint64_t out_base)
{
    out[out_base + i + ri_lower(other, 0, n_other, src, key_ref(src, own[i]))] = own[i];
}

// One pass of the merge sort of n distinct keys (written keys; update_bytes' records): runs of `width` merge pairwise into runs of 2 width
template <typename T>
BD_HD void ri_sort_one(const T* in, uint32_t i, uint32_t n, uint32_t width, const uint8_t* src, T* out)
{
    const uint32_t r = i / width, pair = (r & ~1u) * width, partner = (r ^ 1u) * width;
    if (partner >= n) { out[i] = in[i]; return; }
    const uint32_t pe = partner + width < n ? partner + width : n;
    out[pair + (i - r * width) + (uint32_t)ri_lower(in, partner, pe, src, key_ref(src, in[i])) - partner] = in[i];
}

// ---- SHA-256 over a stream (rwsetutil's hashFunc) ----------------------------------------------------------------------------------
BD_HD void sv_init(SvSha& s)
{
    const uint32_t iv[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    for (int k = 0; k < 8; k++) s.h[k] = iv[k];
    for (int k = 0; k < 16; k++) s.w[k] = 0;
    s.n = 0; s.total = 0;
}
BD_HD void sv_bytes(SvSha& s, const uint8_t* p, uint32_t len) { for (uint32_t i = 0; i < len; i++) sv_byte(s, p[i]); }
BD_HD void sv_varint(SvSha& s, uint64_t v)
{
    while (v >= 0x80) { sv_byte(s, (uint32_t)(v & 0x7f) | 0x80u); v >>= 7; }
    sv_byte(s, (uint32_t)v);
}
BD_HD void sv_final(SvSha& s, uint32_t out[8])
{
    const uint64_t bits = s.total * 8;
    sv_byte(s, 0x80);
    while (s.n != 56) sv_byte(s, 0);
    for (int k = 7; k >= 0; k--) sv_byte(s, (uint32_t)(bits >> (8 * k)));
    for (int k = 0; k < 8; k++) out[k] = s.h[k];
}
BD_HD void sv_hash_bytes(SvSha& s, const uint32_t h[8]) { for (int k = 0; k < 32; k++) sv_byte(s, h[k >> 2] >> (24 - 8 * (k & 3))); }
BD_HD uint32_t varint_len(uint64_t v) { uint32_t n = 1; while (v >= 0x80) { v >>= 7; n++; } return n; }

// ---- rwsetutil.RangeQueryResultsHelper with hashing, streamed -------------------------------------------------------------------
// Each leaf is SHA-256 of proto.Marshal(QueryReads{kv_reads}) over max_degree + 1 results (the last, at Done, over fewer): deterministic
// proto3 -- KVRead{key = 1 (omitted when empty), version = 2 (always present: Version{block_num = 1, tx_num = 2}, zeros omitted)}.  A level
// holding more than max_degree hashes is replaced by one hash of their concatenation one level up (merkleTree.update); done() carries
// every lower level up (one hash as it is, more combined) and combines a top level above max_degree once more.
//
// Only the level the recorded summary names is compared, hash by hash as it is appended: a level is never changed except by appending
// until it is combined, and combining it raises the tree above it for good, so the summary can only equal the recorded one if every
// hash appended to that level since its last combination matched.
#define MK_LEVELS 20
struct MerkleState {
    SvSha leaf; uint64_t pending;                 // the leaf under construction and its results
    SvSha lv[MK_LEVELS]; uint32_t first[MK_LEVELS][8]; uint64_t cnt[MK_LEVELS];   // per level (index 0 = level 1): stream, first hash, count
    uint32_t max_level, degree;
    uint32_t rec_level; uint64_t rec_n, matched; bool overflow;   // the recorded summary's level and hash count; hashes matched there
    const uint8_t* base; Reader rec;                                  // the recorded max_level_hashes, in order
    long long last; uint32_t top[8]; Reader early;                    // rangeQueryHashValidator's lastMatchedIndex, the newest top hash,
                                                                      // the recorded hash it compares next
};

BD_HD bool mk_next_rec(MerkleState& m, Seg& h)
{
    uint32_t f, wt; uint64_t x = 0; Seg b; b.off = b.len = 0;
    while (m.rec.next(f, wt, x, b)) if (f == 3) { h = b; return true; }
    return false;
}

BD_HD void mk_append(MerkleState& m, uint32_t level, const uint32_t h[8])
{
    if (level > MK_LEVELS) { m.overflow = true; return; }
    const uint32_t i = level - 1;
    if (m.cnt[i] == 0) for (int k = 0; k < 8; k++) m.first[i][k] = h[k];
    sv_hash_bytes(m.lv[i], h);
    m.cnt[i]++;
    if (level > m.max_level) m.max_level = level;
    if (level == m.max_level) for (int k = 0; k < 8; k++) m.top[k] = h[k];
    if (level == m.rec_level) {
        Seg r; r.off = r.len = 0;
        bool eq = mk_next_rec(m, r) && r.len == 32;
        for (uint32_t k = 0; eq && k < 32; k++) eq = m.base[r.off + k] == (uint8_t)(h[k >> 2] >> (24 - 8 * (k & 3)));
        if (m.matched == m.cnt[i] - 1 && eq) m.matched++;
    }
}

// computeCombinedHash of a level's hashes; the level is emptied
BD_HD void mk_take(MerkleState& m, uint32_t level, uint32_t h[8])
{
    sv_final(m.lv[level - 1], h);
    sv_init(m.lv[level - 1]); m.cnt[level - 1] = 0;
}

// merkleTree.update: append, then replace each level holding more than max_degree hashes by their combination one level up
BD_HD void mk_push(MerkleState& m, uint32_t level, const uint32_t h[8])
{
    mk_append(m, level, h);
    while (!m.overflow && m.cnt[level - 1] > m.degree) {
        uint32_t c[8];
        mk_take(m, level, c);
        mk_append(m, ++level, c);
    }
}

// rec_body: the recorded QueryReadsMerkleSummary (already checked: max_degree >= 2, max_level below 2^32)
BD_HD void mk_init(MerkleState& m, const uint8_t* base, Seg rec_body, uint32_t degree, uint32_t rec_level)
{
    sv_init(m.leaf); m.pending = 0;
    for (int i = 0; i < MK_LEVELS; i++) { sv_init(m.lv[i]); m.cnt[i] = 0; }
    m.max_level = 1; m.degree = degree; m.rec_level = rec_level; m.rec_n = 0; m.matched = 0; m.overflow = false;
    m.base = base; m.rec.base = base; m.rec.pos = rec_body.off; m.rec.end = rec_body.off + rec_body.len; m.rec.ok = true;
    Reader r = m.rec; Seg h; h.off = h.len = 0; uint32_t f, wt; uint64_t x = 0;
    while (r.next(f, wt, x, h)) if (f == 3) m.rec_n++;
    m.last = -1; m.early = m.rec;
}

// rangeQueryHashValidator.validate's loop body after AddResult (rangequery_validator.go:110-141), over GetMerkleSummary's max level L and
// its n hashes: 0 go on, 1 return false, 2 the reference panics -- MaxLevelHashes[lastMatchedIndex] out of range, which happens when the
// max level rises after lastMatchedIndex passed 0 (the new level holds one hash).  At most one hash joins the top level per result, so
// lastMatchedIndex never lags by more than one: when it advances to n - 1 it names the newest top hash.
BD_HD int mk_early(MerkleState& m)
{
    const long long n = (long long)m.cnt[m.max_level - 1];
    if (m.max_level < m.rec_level || m.last == n - 1) return 0;
    if ((uint64_t)n > m.rec_n) return 1;
    if (++m.last >= n) return 2;
    Seg r; r.off = r.len = 0;
    uint32_t f, wt; uint64_t x = 0; Seg b; b.off = b.len = 0;
    while (m.early.next(f, wt, x, b)) if (f == 3) { r = b; break; }
    bool eq = r.len == 32;
    for (uint32_t k = 0; eq && k < 32; k++) eq = m.base[r.off + k] == (uint8_t)(m.top[k >> 2] >> (24 - 8 * (k & 3)));
    return eq ? 0 : 1;
}

BD_HD void mk_leaf(MerkleState& m)
{
    uint32_t h[8];
    sv_final(m.leaf, h);
    sv_init(m.leaf); m.pending = 0;
    mk_push(m, 1, h);
}

// RangeQueryResultsHelper.AddResult(NewKVRead(key, (blk, txn)))
BD_HD void mk_add(MerkleState& m, const uint8_t* key, uint32_t kl, unsigned long long blk, unsigned long long txn)
{
    const uint32_t vl = (blk ? 1 + varint_len(blk) : 0) + (txn ? 1 + varint_len(txn) : 0);
    const uint32_t rl = (kl ? 1 + varint_len(kl) + kl : 0) + 1 + varint_len(vl) + vl;
    sv_byte(m.leaf, 0x0a); sv_varint(m.leaf, rl);
    if (kl) { sv_byte(m.leaf, 0x0a); sv_varint(m.leaf, kl); sv_bytes(m.leaf, key, kl); }
    sv_byte(m.leaf, 0x12); sv_varint(m.leaf, vl);
    if (blk) { sv_byte(m.leaf, 0x08); sv_varint(m.leaf, blk); }
    if (txn) { sv_byte(m.leaf, 0x10); sv_varint(m.leaf, txn); }
    if (++m.pending > m.degree) mk_leaf(m);
}

// Done() and merkleSummariesEqual: 1 equal, 0 not (no summary -- max_degree or fewer results -- included), -1 beyond MK_LEVELS levels
BD_HD int mk_done(MerkleState& m, uint32_t rec_degree)
{
    if (m.max_level == 1 && m.cnt[0] == 0 && !m.overflow) return 0;      // no leaf was hashed: the tree is empty, Done() gives no summary
    if (m.pending) mk_leaf(m);
    for (uint32_t level = 1; level < m.max_level && !m.overflow; level++) {
        const uint32_t i = level - 1;
        if (m.cnt[i] == 0) continue;
        uint32_t h[8];
        if (m.cnt[i] == 1) { for (int k = 0; k < 8; k++) h[k] = m.first[i][k]; m.cnt[i] = 0; sv_init(m.lv[i]); }
        else mk_take(m, level, h);
        mk_append(m, level + 1, h);
    }
    if (!m.overflow && m.cnt[m.max_level - 1] > m.degree) {
        uint32_t h[8];
        const uint32_t top = m.max_level;
        mk_take(m, top, h);
        mk_append(m, top + 1, h);
    }
    if (m.overflow) return -1;
    return rec_degree == m.degree && m.rec_level == m.max_level && m.rec_n == m.cnt[m.max_level - 1] && m.matched == m.rec_n ? 1 : 0;
}

} }  // namespace fabgpu::bdev
