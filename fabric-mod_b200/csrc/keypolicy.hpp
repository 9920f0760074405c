// Host side of fabgpu_key_policies / fabgpu_key_policies_update: the key policy table's host mirror, the argument checks, and the
// bookkeeping that lets the library upload only what a call changed.  The library and the tests' host build both use it.
#pragma once
#include <algorithm>
#include <cstring>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "blockdev.cuh"

namespace fabgpu { namespace bdev {

struct KeyPolicyTable {
    std::vector<KpSlot> slots;          // a power of two; empty: no table installed
    std::vector<uint8_t> blob;          // namespace || collection || key of the entries, back to back
    std::vector<int32_t> nodes;         // the table's policy nodes (4 ints each), appended after the `base` configured ones; child
                                        // indices count from the start of the whole array
    int32_t base = 0;                   // nodes given to fabgpu_msp_configure
    uint32_t live = 0, used = 0;        // entries; occupied slots (entries and removed entries)
    size_t blob_compact = 0, nodes_compact = 0;   // sizes right after the last rebuild: past twice that, the next update rebuilds
    // What the last successful call changed: everything (full), or the slots in `dirty`, the blob from blob_from and the nodes from
    // nodes_from on.
    bool full = false; std::vector<uint32_t> dirty; size_t blob_from = 0, nodes_from = 0;

    bool installed() const { return !slots.empty(); }
    int32_t n_nodes() const { return (int32_t)(nodes.size() / 4); }

    // replace = fabgpu_key_policies (the table becomes these entries; n = 0 with n_nodes = 0 removes it), else
    // fabgpu_key_policies_update (upserts; root -1 removes).  base: nodes configured by fabgpu_msp_configure.  Returns nullptr, or the
    // reason for refusing the call, with the table unchanged.
    const char* apply(bool replace, int32_t base_nodes, int32_t n_principals, const int32_t* nd, int n_nodes, const uint8_t* ns_blob,
                      const uint32_t* ns_off, const uint8_t* coll_blob, const uint32_t* coll_off, const uint8_t* key_blob,
                      const uint32_t* key_off, const int32_t* root, int n)
    {
        if (n < 0 || n_nodes < 0) return "negative count";
        if ((n && (!ns_blob || !ns_off || !coll_blob || !coll_off || !key_blob || !key_off || !root)) || (n_nodes && !nd))
            return "key policy arrays missing";
        if (!replace && !installed()) return "no key policy table installed";
        for (int i = 0; i < n; i++)
            if (ns_off[i] > ns_off[i + 1] || coll_off[i] > coll_off[i + 1] || key_off[i] > key_off[i + 1]) return "key policy offsets decrease";
        if (const char* err = check_nodes(nd, n_nodes, n_principals)) return err;
        std::unordered_set<std::string> seen;
        for (int i = 0; i < n; i++) {
            if (root[i] >= n_nodes || root[i] < KP_UNDECIDABLE) return "key policy root out of range";
            if (root[i] == -1 && replace) return "key policy removal (-1) in a replacing call";
            if (!seen.insert(triple(ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, i)).second)
                return "key policy given twice for one (namespace, collection, key)";
        }
        // accepted: from here on nothing fails
        dirty.clear(); full = false;
        if (replace) {
            slots.clear(); blob.clear(); nodes.clear(); live = used = 0; base = base_nodes; full = true;
            if (n == 0 && n_nodes == 0) return nullptr;
            uint32_t size = 16; while (size < 2u * (uint32_t)n + 16) size <<= 1;
            slots.assign(size, KpSlot{});
        }
        else if (2 * ((size_t)used + n) > slots.size()) rebuild((uint32_t)n);   // keep the table at most half full
        const int32_t first = base + this->n_nodes();                    // where this call's nodes go
        nodes_from = nodes.size(); blob_from = blob.size();
        for (int i = 0; i < n_nodes; i++) {
            const int32_t* x = nd + 4 * i;
            nodes.push_back(x[0]); nodes.push_back(x[1]); nodes.push_back(x[0] == 0 ? x[2] + first : 0); nodes.push_back(x[0] == 0 ? x[3] : 0);
        }
        for (int i = 0; i < n; i++) {
            const uint32_t nl = ns_off[i + 1] - ns_off[i], cl = coll_off[i + 1] - coll_off[i], kl = key_off[i + 1] - key_off[i];
            const int32_t r = root[i] >= 0 ? root[i] + first : root[i];
            upsert(ns_blob + ns_off[i], nl, coll_blob + coll_off[i], cl, key_blob + key_off[i], kl, r);
        }
        if (replace) { blob_compact = blob.size(); nodes_compact = nodes.size(); dirty.clear(); }
        else if (blob.size() > 2 * blob_compact + 65536 || nodes.size() > 2 * nodes_compact + 16384) rebuild(0);
        return nullptr;
    }

private:
    static std::string triple(const uint8_t* nb, const uint32_t* no, const uint8_t* cb, const uint32_t* co, const uint8_t* kb,
                              const uint32_t* ko, int i)
    {
        std::string s;
        for (auto p : {std::make_pair(nb + no[i], no[i + 1] - no[i]), std::make_pair(cb + co[i], co[i + 1] - co[i]), std::make_pair(kb + ko[i], ko[i + 1] - ko[i])}) {
            s.append(reinterpret_cast<const char*>(&p.second), 4);
            s.append(reinterpret_cast<const char*>(p.first), p.second);
        }
        return s;
    }

    // What eval_policy evaluates exactly, for a validation parameter (a SignaturePolicyEnvelope: NOutOf and SignedBy only): node types
    // 0 and 1, children inside this call's array, principals inside fabgpu_msp_configure's, no cycle, and no tree deeper than
    // BD_MAX_POLICY_DEPTH below any node.
    static const char* check_nodes(const int32_t* nd, int n_nodes, int32_t n_principals)
    {
        for (int i = 0; i < n_nodes; i++) {
            const int32_t* x = nd + 4 * i;
            if (x[0] != 0 && x[0] != 1) return "key policy node type is not NOutOf (0) or SignedBy (1)";
            if (x[0] == 0 && (x[2] < 0 || x[3] < 0 || (int64_t)x[2] + x[3] > n_nodes)) return "key policy node children out of range";
            if (x[0] == 1 && (x[1] < 0 || x[1] >= n_principals)) return "key policy SignedBy principal index out of range";
        }
        std::vector<int> height(n_nodes, -1);
        for (int i = 0; i < n_nodes; i++)
            if (node_height(nd, i, 0, height) < 0) return "key policy tree deeper than the device evaluates, or cyclic";
        return nullptr;
    }
    static int node_height(const int32_t* nd, int i, int path, std::vector<int>& height)
    {
        if (path > BD_MAX_POLICY_DEPTH) return -1;
        if (height[i] >= 0) return height[i];
        int h = 0;
        if (nd[4 * i] == 0)
            for (int c = nd[4 * i + 2]; c < nd[4 * i + 2] + nd[4 * i + 3]; c++) {
                const int hc = node_height(nd, c, path + 1, height);
                if (hc < 0 || hc + 1 > BD_MAX_POLICY_DEPTH) return -1;
                h = std::max(h, hc + 1);
            }
        return height[i] = h;
    }

    // the slot holding (ns, coll, key), removed or not, or the empty slot where it would go
    uint32_t find(uint64_t h, const uint8_t* ns, uint32_t nl, const uint8_t* coll, uint32_t cl, const uint8_t* key, uint32_t kl) const
    {
        const uint32_t mask = (uint32_t)slots.size() - 1;
        for (uint32_t pos = (uint32_t)h & mask;; pos = (pos + 1) & mask) {
            const KpSlot& s = slots[pos];
            if (s.hash == 0) return pos;
            if (s.hash == h && s.ns_len == nl && s.coll_len == cl && s.key_len == kl && memcmp(&blob[s.off], ns, nl) == 0 &&
                memcmp(&blob[s.off + nl], coll, cl) == 0 && memcmp(&blob[s.off + nl + cl], key, kl) == 0)
                return pos;
        }
    }

    void upsert(const uint8_t* ns, uint32_t nl, const uint8_t* coll, uint32_t cl, const uint8_t* key, uint32_t kl, int32_t r)
    {
        const uint64_t h = kl_key_hash(ns, nl, coll, cl, key, kl);
        const uint32_t pos = find(h, ns, nl, coll, cl, key, kl);
        KpSlot& s = slots[pos];
        if (s.hash != 0) {                                               // present (perhaps removed)
            const int32_t nr = r == -1 ? KP_REMOVED : r;
            if (s.root == nr) return;
            if (s.root == KP_REMOVED) live++;
            if (nr == KP_REMOVED) live--;
            s.root = nr;
        } else {
            if (r == -1) return;                                         // removing an absent key does nothing
            s.hash = h; s.off = (uint32_t)blob.size(); s.ns_len = nl; s.coll_len = cl; s.key_len = kl; s.root = r; s.pad = 0;
            blob.insert(blob.end(), ns, ns + nl); blob.insert(blob.end(), coll, coll + cl); blob.insert(blob.end(), key, key + kl);
            live++; used++;
        }
        dirty.push_back(pos);
    }

    // Rehash into a table that stays at most half full with `extra` more entries, dropping removed entries, and compact the blob and
    // the nodes to what live entries use (each distinct root's tree is copied once).
    void rebuild(uint32_t extra)
    {
        std::vector<KpSlot> old = std::move(slots);
        std::vector<uint8_t> old_blob = std::move(blob);
        std::vector<int32_t> old_nodes = std::move(nodes);
        uint32_t size = 16; while (size < 2u * (live + extra) + 16) size <<= 1;
        slots.assign(size, KpSlot{}); blob.clear(); nodes.clear(); live = used = 0;
        std::unordered_map<int32_t, int32_t> copied;                     // old root -> new root
        auto alloc = [&](int32_t k) { const int32_t at = base + n_nodes(); nodes.resize(nodes.size() + 4 * (size_t)k, 0); return at; };
        auto place = [&](auto& self, int32_t from, int32_t at) -> void {   // node `from` of the old array into slot `at` of the new one
            const int32_t* x = &old_nodes[4 * (size_t)(from - base)];
            const int32_t type = x[0], n = x[1], first = x[2], cnt = x[3];
            const int32_t block = type == 0 && cnt > 0 ? alloc(cnt) : 0;
            int32_t* y = &nodes[4 * (size_t)(at - base)];
            y[0] = type; y[1] = n; y[2] = type == 0 ? block : 0; y[3] = type == 0 ? cnt : 0;
            for (int32_t k = 0; type == 0 && k < cnt; k++) self(self, first + k, block + k);
        };
        for (const KpSlot& s : old) {
            if (s.hash == 0 || s.root == KP_REMOVED) continue;
            int32_t r = s.root;
            if (r >= 0) {
                auto it = copied.find(r);
                if (it != copied.end()) r = it->second;
                else { const int32_t at = alloc(1); place(place, r, at); copied[s.root] = at; r = at; }
            }
            upsert(&old_blob[s.off], s.ns_len, &old_blob[s.off + s.ns_len], s.coll_len, &old_blob[s.off + s.ns_len + s.coll_len], s.key_len, r);
        }
        blob_compact = blob.size(); nodes_compact = nodes.size();
        dirty.clear(); full = true;
    }
};

} }  // namespace fabgpu::bdev
