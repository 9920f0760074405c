// TEST HELPER (not product code): blockdev_host.cpp's host build of the device-side block logic, plus a decide stage with principal
// bits (fabgpu_msp_principal_bits) and a collection policy table (fabgpu_collection_policies).  Built as a library of its own; every
// other entry point is blockdev_host.cpp's.
#include "blockdev_host.cpp"

extern "C" {

// bd_decide with principal bits (ceil(n_principals / 32) words per identity, in the layout fabgpu_msp_principal_bits reads) and a
// collection table (n_coll entries as fabgpu_collection_policies takes them, laid out by the library's coll_table_fill).
// n_ids = 0: no bits (MSP-id member matching); n_coll = 0: no table.  Returns 0, or -1 when the table names one
// (namespace, collection) twice.
int bd_decide_coll(void* p, const uint8_t* sig_ok, const uint8_t* check_digests, const uint32_t* bits, int n_ids, int n_principals,
                   const uint8_t* coll_ns_blob, const uint32_t* coll_ns_off, const uint8_t* coll_blob, const uint32_t* coll_off,
                   const int32_t* coll_root, int n_coll, uint8_t* flags)
{
    H* h = (H*)p;
    std::vector<uint8_t> dig(32 * (size_t)(h->J_cap + 2 * h->T), 0);
    if (h->T) memcpy(dig.data() + 32 * (size_t)h->J_cap, check_digests, 64 * (size_t)h->T);
    const int W = (n_principals + 31) / 32;
    std::vector<uint32_t> words(bits, bits + (size_t)n_ids * W); words.push_back(0);
    PolicyDev pol; pol.nodes = h->nodes.data(); pol.n_nodes = (int32_t)h->nodes.size() / 4; pol.principal_code = h->principal_code.data(); pol.n_principals = (int32_t)h->principal_code.size();
    pol.ns_blob = h->ns_blob.data(); pol.ns_off = h->ns_off.data(); pol.ns_root = h->ns_root.data(); pol.n_ns = (int32_t)h->ns_root.size();
    pol.principal_bits = n_ids ? words.data() : nullptr; pol.bits_words = n_ids ? W : 0;
    uint32_t size = 8; while (size < (uint32_t)(2 * n_coll + 8)) size <<= 1;
    std::vector<uint64_t> ch(size, 0); std::vector<int32_t> ci(size, -1);
    if (n_coll) {
        if (!coll_table_fill(coll_ns_blob, coll_ns_off, coll_blob, coll_off, n_coll, size, ch.data(), ci.data())) return -1;
        pol.coll_ns_blob = coll_ns_blob; pol.coll_ns_off = coll_ns_off; pol.coll_name_blob = coll_blob; pol.coll_name_off = coll_off;
        pol.coll_root = coll_root; pol.coll_hash = ch.data(); pol.coll_idx = ci.data(); pol.coll_size = size;
    }
    const MspDev m = h->msp();
    std::vector<uint64_t> th(h->T, 0);
    for (uint32_t t = 0; t < h->T; t++)
        flags[t] = decide_tx(h->block.data(), h->txs[t], t, m, pol, [&](uint32_t j) { return sig_ok[j] != 0; }, h->jid.data(), dig.data(), h->J_cap, &th[t]);
    // duplicate pass as the shim does it
    std::multimap<uint64_t, uint32_t> seen;
    for (uint32_t t = 0; t < h->T; t++) {
        if (flags[t] != TXC_VALID) continue;
        const Seg id = h->txs[t].txid_ascii;
        bool dup = false;
        auto range = seen.equal_range(th[t]);
        for (auto it = range.first; it != range.second && !dup; ++it) {
            const Seg o = h->txs[it->second].txid_ascii;
            dup = o.len == id.len && memcmp(&h->block[o.off], &h->block[id.off], id.len) == 0;
        }
        if (dup) flags[t] = TXC_DUPLICATE_TXID; else seen.emplace(th[t], t);
    }
    return 0;
}

}  // extern "C"
