// Host mirror of the device MSP table's identity index (MspDev: id_blob / id_off and the hash slots ht_hash / ht_idx) for
// fabgpu_msp_configure and fabgpu_msp_identities_add: the argument checks of an add, the slots it changes, and growth.  Shared by the
// library and the tests' host build, which look identities up in it with the device's own msp_find.
#pragma once
#include <stdint.h>
#include <string.h>

#include <string>
#include <unordered_set>
#include <vector>

#include "blockdev.cuh"

namespace fabgpu { namespace msptab {

// Slots of an index holding n identities at a load below 1/4: the smallest power of two >= 4 n + 8, doubled from `have` when given
inline uint32_t slots_for(uint32_t n, uint32_t have = 8)
{
    uint32_t s = have < 8 ? 8 : have;
    while (s < 4 * n + 8) s <<= 1;
    return s;
}

struct Mirror {
    std::vector<uint8_t> blob;                 // the identities' serialized bytes, back to back
    std::vector<uint32_t> off{0};              // n + 1 offsets
    std::vector<uint64_t> ht_hash;             // slots; 0 = empty
    std::vector<int32_t> ht_idx;

    int32_t n() const { return (int32_t)off.size() - 1; }
    uint32_t size() const { return (uint32_t)ht_hash.size(); }

    // the view msp_find walks (only the index fields are set)
    bdev::MspDev view() const
    {
        bdev::MspDev m;
        memset(&m, 0, sizeof m);
        m.id_blob = blob.data(); m.id_off = off.data(); m.ht_hash = ht_hash.data(); m.ht_idx = ht_idx.data();
        m.ht_size = n() ? size() : 0; m.n_ids = n();
        return m;
    }
    int32_t find(const uint8_t* p, uint32_t len) const { return bdev::msp_find(view(), p, len); }

    // places identity i in the first free slot of its probe chain; returns the slot
    uint32_t place(int32_t i)
    {
        const uint64_t hv = bdev::sample_hash(blob.data() + off[i], off[i + 1] - off[i]);
        const uint32_t mask = size() - 1;
        uint32_t pos = (uint32_t)hv & mask;
        while (ht_hash[pos] != 0) pos = (pos + 1) & mask;
        ht_hash[pos] = hv; ht_idx[pos] = i;
        return pos;
    }
    void rebuild(uint32_t slots)
    {
        ht_hash.assign(slots, 0); ht_idx.assign(slots, -1);
        for (int32_t i = 0; i < n(); i++) place(i);
    }

    // fabgpu_msp_configure: the table holds exactly these identities
    void configure(const uint8_t* id_blob, const uint32_t* id_off, int n_ids)
    {
        // the bytes as the device holds them: everything up to the last offset, the offsets as given
        blob.assign(id_blob, id_blob + (n_ids ? id_off[n_ids] : 0));
        off.assign(id_off, id_off + (n_ids ? n_ids + 1 : 0));
        if (off.empty()) off.push_back(0);
        rebuild(slots_for((uint32_t)n_ids));
    }

    // The refusal text of an add, or null.  groups_on / bits_on: a group table / principal bits are installed; group and bits must be
    // given exactly when they are.
    const char* check_add(const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* mspid_blob, const uint32_t* mspid_off,
                          const uint8_t* keys_xy, const uint8_t* valid, const int32_t* group, const uint32_t* bits, int n_ids,
                          bool groups_on, bool bits_on) const
    {
        if (n_ids < 0) return "negative identity count";
        if (n_ids == 0) return (group && !groups_on) || (bits && !bits_on) ? "group or bits given for a table without them" : nullptr;
        if (!id_blob || !id_off || !mspid_blob || !mspid_off || !keys_xy || !valid) return "identity arrays missing";
        if (!group != !groups_on) return groups_on ? "a group table is installed: every admitted identity needs a group" : "no group table is installed: groups are not taken";
        if (!bits != !bits_on) return bits_on ? "principal bits are installed: every admitted identity needs its bits" : "no principal bits are installed: bits are not taken";
        std::unordered_set<std::string> seen;
        for (int i = 0; i < n_ids; i++) {
            if (id_off[i] > id_off[i + 1] || mspid_off[i] > mspid_off[i + 1]) return "identity offsets decrease";
            const uint32_t len = id_off[i + 1] - id_off[i];
            if (len == 0) return "empty identity";
            if (group && group[i] < 0) return "negative group";
            if (find(id_blob + id_off[i], len) >= 0) return "identity already in the table";
            if (!seen.emplace((const char*)id_blob + id_off[i], len).second) return "identity given twice";
        }
        if ((uint64_t)blob.size() + (id_off[n_ids] - id_off[0]) > 0xffffff00ull) return "identity bytes exceed 32-bit offsets";
        return nullptr;
    }

    // Appends checked identities.  Returns true when the index grew (it is then uploaded whole); else dirty holds the changed slots.
    bool add(const uint8_t* id_blob, const uint32_t* id_off, int n_ids, std::vector<uint32_t>& dirty)
    {
        dirty.clear();
        const int32_t n0 = n();
        blob.insert(blob.end(), id_blob + id_off[0], id_blob + id_off[n_ids]);
        for (int i = 0; i < n_ids; i++) off.push_back(off.back() + (id_off[i + 1] - id_off[i]));
        const uint32_t want = slots_for((uint32_t)n(), size());
        if (want != size()) { rebuild(want); return true; }
        for (int32_t i = n0; i < n(); i++) dirty.push_back(place(i));
        return false;
    }
};

} }  // namespace fabgpu::msptab
