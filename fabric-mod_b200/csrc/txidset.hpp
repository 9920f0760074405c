// Host side of the committed tx-id set (fabgpu_committed_txids / _add): the argument checks, the canonical-form filter, the
// de-duplication within a call, and the table's sizing.  Shared by the library and the tests' host build.
#pragma once
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <random>
#include <vector>

#include "blockdev.cuh"

namespace fabgpu { namespace txid {

constexpr uint64_t MIN_SLOTS = 1024;

// A tx id can match only in its canonical form -- 64 characters of [0-9a-f], hex.EncodeToString(SHA-256(nonce || creator)) -- since a
// transaction reaches the ledger check only after protoutil.CheckTxID has passed.  Writes the 32 binary bytes and returns true for such
// an id; any other id (uppercase, another length, empty) can never match and is dropped.
inline bool canonical(const uint8_t* p, uint32_t len, uint8_t out[32])
{
    struct Table { int8_t v[256]; Table() { for (int c = 0; c < 256; c++) v[c] = c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : -1; } };
    static const Table t;
    if (len != 64) return false;
    int bad = 0;
    for (int i = 0; i < 32; i++) {
        const int hi = t.v[p[2 * i]], lo = t.v[p[2 * i + 1]];
        bad |= hi | lo;
        out[i] = (uint8_t)(hi << 4 | (lo & 15));
    }
    return bad >= 0;
}

// The records a call inserts: one per distinct canonical id, in the slot layout, with the state of the larger kind given for it
// (kind NULL = all 0).  Null or the refusal text (NULL arrays with n > 0, decreasing offsets, a kind other than 0 or 1).
inline const char* prepare(const uint8_t* blob, const uint32_t* off, const uint8_t* kind, size_t n, uint64_t seed, std::vector<bdev::TxidSlot>& out)
{
    out.clear();
    if (n && (!blob || !off)) return "committed tx-id arrays missing";
    for (size_t i = 0; i < n; i++) {
        if (off[i] > off[i + 1]) return "committed tx-id offsets decrease";
        if (kind && kind[i] > 1) return "committed tx-id kind is neither 0 (committed) nor 1 (unanswerable)";
    }
    out.reserve(n);
    for (size_t i = 0; i < n; i++) {
        uint8_t b[32];
        if (!canonical(blob + off[i], off[i + 1] - off[i], b)) continue;
        bdev::TxidSlot r;
        bdev::txid_words(b, r.w);
        r.state = bdev::TXID_COMMITTED + (kind ? kind[i] : 0);
        out.push_back(r);
    }
    // de-duplication through an open-addressing index under the table's seeded mix (a caller's ids cannot line up into one chain here
    // either); the first occurrence keeps its place and takes the larger state
    size_t cap = 16;
    while (cap < 2 * out.size()) cap <<= 1;
    std::vector<uint32_t> index(cap, UINT32_MAX);
    size_t m = 0;
    for (size_t i = 0; i < out.size(); i++)
        for (size_t h = bdev::txid_mix(out[i].w, seed) & (cap - 1);; h = (h + 1) & (cap - 1)) {
            if (index[h] == UINT32_MAX) { index[h] = (uint32_t)m; out[m++] = out[i]; break; }
            bdev::TxidSlot& o = out[index[h]];
            if (bdev::txid_equal(o.w, out[i].w)) { o.state = std::max(o.state, out[i].state); break; }
        }
    out.resize(m);
    return nullptr;
}

// A context's seed of the slot index (txid_mix): random, so that the probe chains of caller-chosen ids cannot be planned
inline uint64_t random_seed()
{
    std::random_device rd;
    return ((uint64_t)rd() << 32 ^ rd()) ^ (uint64_t)std::chrono::steady_clock::now().time_since_epoch().count();
}

// Slots for `ids` ids at a load of at most 1/2: the smallest power of two >= max(2 ids, MIN_SLOTS), doubled from `have` when given
inline uint64_t slots_for(uint64_t ids, uint64_t have = 0)
{
    uint64_t s = have ? have : MIN_SLOTS;
    while (s < 2 * ids) s <<= 1;
    return s;
}

} }  // namespace fabgpu::txid
