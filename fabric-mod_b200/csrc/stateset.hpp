// Host side of the world-state version table (fabgpu_state_versions / _update): the argument checks, the key digests of the entries a
// call gives, and the table's sizing.  Shared by the library and the tests' host build.
#pragma once
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "stateset.cuh"

namespace fabgpu { namespace stateset {

constexpr uint64_t MIN_SLOTS = 1024;

// The records a call upserts: entry i is (ns, coll, key) -> (ver[2i], ver[2i+1]); (UINT64_MAX, UINT64_MAX) removes the key.  Null or the
// refusal text (NULL arrays with n > 0, decreasing offsets, a key given twice).
inline const char* prepare(const uint8_t* ns_blob, const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                           const uint8_t* key_blob, const uint32_t* key_off, const uint64_t* ver, size_t n, uint64_t seed,
                           std::vector<bdev::StateSlot>& out)
{
    out.clear();
    if (n && (!ns_blob || !ns_off || !coll_off || !key_blob || !key_off || !ver)) return "state version arrays missing";
    for (size_t i = 0; i < n; i++)
        if (ns_off[i] > ns_off[i + 1] || coll_off[i] > coll_off[i + 1] || key_off[i] > key_off[i + 1]) return "state version offsets decrease";
    if (n && coll_off[n] > coll_off[0] && !coll_blob) return "state version arrays missing";
    out.resize(n);
    for (size_t i = 0; i < n; i++) {
        bdev::StateSlot& r = out[i];
        bdev::sv_key(ns_blob + ns_off[i], ns_off[i + 1] - ns_off[i], coll_blob ? coll_blob + coll_off[i] : nullptr, coll_off[i + 1] - coll_off[i],
                     key_blob + key_off[i], key_off[i + 1] - key_off[i], r.w);
        const bool removed = ver[2 * i] == UINT64_MAX && ver[2 * i + 1] == UINT64_MAX;
        r.state = removed ? bdev::SV_REMOVED : bdev::SV_PRESENT; r.pad = 0;
        r.blk = removed ? 0 : ver[2 * i]; r.txn = removed ? 0 : ver[2 * i + 1];
    }
    // a key given twice is refused: the inserts of one launch must carry different keys
    size_t cap = 16;
    while (cap < 2 * n) cap <<= 1;
    std::vector<uint32_t> index(cap, UINT32_MAX);
    for (size_t i = 0; i < n; i++)
        for (size_t h = bdev::txid_mix(out[i].w, seed) & (cap - 1);; h = (h + 1) & (cap - 1)) {
            if (index[h] == UINT32_MAX) { index[h] = (uint32_t)i; break; }
            if (bdev::txid_equal(out[index[h]].w, out[i].w)) return "state version key given twice in one call";
        }
    return nullptr;
}

// The public keys of a call that are not removals (collection empty, version not (UINT64_MAX, UINT64_MAX)), sorted by (namespace, key)
// bytewise: the index's install form and an update's insertions.  blob holds each key's namespace then key; recs: prepare's output.
inline void index_keys(const uint8_t* ns_blob, const uint32_t* ns_off, const uint32_t* coll_off, const uint8_t* key_blob, const uint32_t* key_off,
                       const uint64_t* ver, size_t n, const std::vector<bdev::StateSlot>& recs, std::vector<bdev::WrittenKey>& out,
                       std::vector<uint8_t>& blob)
{
    out.clear(); blob.clear();
    for (size_t i = 0; i < n; i++) {
        if (coll_off[i + 1] != coll_off[i] || (ver[2 * i] == UINT64_MAX && ver[2 * i + 1] == UINT64_MAX)) continue;
        bdev::WrittenKey c;
        c.nl = ns_off[i + 1] - ns_off[i]; c.kl = key_off[i + 1] - key_off[i]; c.k = 0;
        c.ns_off = (uint32_t)blob.size(); c.key_off = c.ns_off + c.nl;
        blob.insert(blob.end(), ns_blob + ns_off[i], ns_blob + ns_off[i + 1]);
        blob.insert(blob.end(), key_blob + key_off[i], key_blob + key_off[i + 1]);
        for (int k = 0; k < 8; k++) c.w[k] = recs[i].w[k];
        out.push_back(c);
    }
    const uint8_t* b = blob.data();
    std::sort(out.begin(), out.end(), [b](const bdev::WrittenKey& x, const bdev::WrittenKey& y) {
        return bdev::key_cmp(bdev::key_ref(b, x), bdev::key_ref(b, y)) < 0;
    });
}

// The delta is folded into the base when it holds more than this many entries
inline uint64_t index_fold_at(uint64_t base)
{
    const uint64_t f = std::min<uint64_t>(base / 8, 1u << 18);
    return std::max<uint64_t>(f, 4096);
}

// Slots for `keys` claimed slots at a load of at most 1/2: the smallest power of two >= max(2 keys, MIN_SLOTS), at least `have`
inline uint64_t slots_for(uint64_t keys, uint64_t have = 0)
{
    uint64_t s = have ? have : MIN_SLOTS;
    while (s < 2 * keys) s <<= 1;
    return s;
}

} }  // namespace fabgpu::stateset
