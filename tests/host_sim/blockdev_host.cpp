// TEST HELPER (not product code): runs the device-side block logic (fabric-mod_b200/csrc/blockdev.cuh: plan_tx, gate_signature,
// decide_tx -- the very functions the CUDA kernels call) on the host, one transaction at a time, so tests can compare it with
// the oracle on the CPU-only box.  Signature verdicts and SHA-256 digests are supplied by the test (oracle, hashlib).
// Built together with the library's blockval.cpp (split_block).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <vector>
#include "../../fabric-mod_b200/csrc/blockdev.cuh"
#include "../../fabric-mod_b200/csrc/blockval.hpp"

using namespace fabgpu::bdev;

struct H {
    std::vector<uint8_t> id_blob; std::vector<uint32_t> id_off; std::vector<int32_t> key_slot, msp_code, ht_idx, nodes, principal_code;
    std::vector<uint8_t> valid; std::vector<uint64_t> ht_hash; std::string channel;
    std::vector<int32_t> group, ns_root; std::vector<uint8_t> ns_blob; std::vector<uint32_t> ns_off;
    std::vector<uint8_t> block; std::vector<uint32_t> env_off;
    std::vector<TxDev> txs; std::vector<RawJob> raw; std::vector<ShaJobD> sha; std::vector<uint8_t> r, s, gate_ok; std::vector<int32_t> jks, jid;
    uint32_t T = 0, J_cap = 0, n_end = 0, stale = 0;
    MspDev msp() const {
        MspDev m; m.id_blob = id_blob.data(); m.id_off = id_off.data(); m.key_slot = key_slot.data(); m.valid = valid.data(); m.msp_code = msp_code.data();
        m.group = group.empty() ? nullptr : group.data();
        m.keys_xy = nullptr; m.ht_hash = ht_hash.data(); m.ht_idx = ht_idx.data(); m.ht_size = (uint32_t)ht_hash.size(); m.n_ids = (int32_t)valid.size(); return m;
    }
};

extern "C" {

void* bd_new(const uint8_t* id_blob, const uint32_t* id_off, const uint8_t* mspid_blob, const uint32_t* mspid_off, const uint8_t* valid, int n_ids,
             const int32_t* nodes, int n_nodes, const uint8_t* pr_blob, const uint32_t* pr_off, int n_pr, const char* channel)
{
    H* h = new H();
    h->id_blob.assign(id_blob, id_blob + id_off[n_ids]); h->id_off.assign(id_off, id_off + n_ids + 1);
    h->valid.assign(valid, valid + n_ids); h->key_slot.assign(n_ids, 0);
    std::map<std::string, int32_t> codes;
    auto code_of = [&](const std::string& s) { auto it = codes.find(s); if (it != codes.end()) return it->second; int32_t c = (int32_t)codes.size(); codes[s] = c; return c; };
    for (int i = 0; i < n_ids; i++) h->msp_code.push_back(code_of(std::string((const char*)mspid_blob + mspid_off[i], mspid_off[i + 1] - mspid_off[i])));
    for (int i = 0; i < n_pr; i++) h->principal_code.push_back(code_of(std::string((const char*)pr_blob + pr_off[i], pr_off[i + 1] - pr_off[i])));
    h->nodes.assign(nodes, nodes + 4 * n_nodes);
    uint32_t sz = 8; while (sz < (uint32_t)(4 * n_ids + 8)) sz <<= 1;
    h->ht_hash.assign(sz, 0); h->ht_idx.assign(sz, -1);
    for (int i = 0; i < n_ids; i++) {
        const uint64_t hv = sample_hash(id_blob + id_off[i], id_off[i + 1] - id_off[i]);
        uint32_t pos = (uint32_t)hv & (sz - 1);
        while (h->ht_hash[pos] != 0) pos = (pos + 1) & (sz - 1);
        h->ht_hash[pos] = hv; h->ht_idx[pos] = i;
    }
    h->channel = channel;
    return h;
}
void bd_free(void* p) { delete (H*)p; }
// de-duplication groups of the identities (Mspid + certificate) and the namespace -> policy root table
void bd_groups(void* p, const int32_t* group, int n_ids) { H* h = (H*)p; h->group.assign(group, group + n_ids); }
void bd_namespaces(void* p, const uint8_t* ns_blob, const uint32_t* ns_off, const int32_t* ns_root, int n_ns)
{
    H* h = (H*)p;
    h->ns_blob.assign(ns_blob, ns_blob + ns_off[n_ns]); h->ns_off.assign(ns_off, ns_off + n_ns + 1); h->ns_root.assign(ns_root, ns_root + n_ns);
    if (h->ns_blob.empty()) h->ns_blob.push_back(0);
}

// Plans every transaction; returns the number of endorsement jobs inside the arrays; J = T + n_end signature jobs, 2T check digests
// after J_cap.  ends_hint sizes the job arrays as the library does (J_cap = T (1 + ends_hint)).  poison = 1: the job arrays start
// filled with the byte 0xA5 instead of dead records, as device memory holds whatever the previous block left; every slot the later
// stages would read must then have been written by the walk.  bd_stale tells how many were not (those are not resolved here).
int bd_plan_ex(void* p, const uint8_t* blob, const uint32_t* env_off, int n_env, int ends_hint, int poison)
{
    H* h = (H*)p;
    h->block.assign(blob, blob + env_off[n_env]); h->env_off.assign(env_off, env_off + n_env + 1);
    h->T = (uint32_t)n_env; h->J_cap = h->T * (1 + (uint32_t)ends_hint); h->n_end = 0;
    h->txs.assign(h->T, TxDev()); h->sha.assign(h->J_cap + 2 * h->T, ShaJobD());
    { RawJob dead; dead.ident.off = dead.ident.len = dead.sig.off = dead.sig.len = 0; dead.tx = 0xffffffffu; dead.k = -1; h->raw.assign(h->J_cap, dead); }
    if (poison) {
        memset(h->raw.data(), 0xA5, sizeof(RawJob) * h->raw.size());
        memset(h->sha.data(), 0xA5, sizeof(ShaJobD) * h->sha.size());
    }
    h->r.assign(32 * (size_t)h->J_cap, 0); h->s.assign(32 * (size_t)h->J_cap, 0); h->gate_ok.assign(h->J_cap, 0); h->jks.assign(h->J_cap, -1); h->jid.assign(h->J_cap, -1);
    JobArrays ja; ja.sha = h->sha.data(); ja.r = h->r.data(); ja.s = h->s.data(); ja.key_slot = h->jks.data(); ja.identity = h->jid.data();
    ja.qx = nullptr; ja.qy = nullptr; ja.gate_ok = h->gate_ok.data(); ja.J_cap = h->J_cap; ja.T = h->T;
    const MspDev m = h->msp();
    for (uint32_t t = 0; t < h->T; t++) {
        Seg env; env.off = env_off[t]; env.len = env_off[t + 1] - env_off[t];
        walk_tx(h->block.data(), env, t, (const uint8_t*)h->channel.data(), (uint32_t)h->channel.size(), h->txs[t], h->raw.data(), ja,
                [&](uint32_t n) { uint32_t b = h->T + h->n_end; h->n_end += n; return b; });
    }
    // the device's later stages stop at min(J_cap, T + n_end): the walk may hand out more slots than there are
    const uint32_t J = std::min<uint64_t>(h->J_cap, (uint64_t)h->T + h->n_end);
    h->stale = 0;
    for (uint32_t j = 0; j < J; j++) {
        if (h->raw[j].tx == 0xA5A5A5A5u || h->sha[j].len[0] == 0xA5A5A5A5u) { h->stale++; continue; }
        resolve_job(h->block.data(), j, h->raw.data(), m, ja, h->txs.data());
    }
    return (int)(J - h->T);
}
int bd_plan(void* p, const uint8_t* blob, const uint32_t* env_off, int n_env) { return bd_plan_ex(p, blob, env_off, n_env, BD_ENDS_HINT, 0); }
int bd_stale(void* p) { return (int)((H*)p)->stale; }
// fabgpu_validate_block's split of a serialized common.Block: the envelopes' (offset, length) pairs, or -1 when the Block does not parse
int bd_split_block(const uint8_t* block, size_t len, uint32_t* out, int cap)
{
    std::vector<fabgpu::blockval::Seg> envs;
    if (!fabgpu::blockval::split_block(block, len, envs)) return -1;
    for (size_t i = 0; i < envs.size() && (int)i < cap; i++) { out[2 * i] = envs[i].off; out[2 * i + 1] = envs[i].len; }
    return (int)envs.size();
}
// job j (0 <= j < T + n_end): identity (-1 unused), gate_ok, r, s, message segments (6 uint32)
void bd_job(void* p, int j, int* identity, int* gate_ok, uint8_t* r, uint8_t* s, uint32_t* segs)
{
    H* h = (H*)p;
    *identity = h->jid[j]; *gate_ok = h->gate_ok[j];
    memcpy(r, &h->r[32 * (size_t)j], 32); memcpy(s, &h->s[32 * (size_t)j], 32);
    for (int k = 0; k < 3; k++) { segs[k] = h->sha[j].off[k]; segs[3 + k] = h->sha[j].len[k]; }
}
void bd_check(void* p, int t, uint32_t* segs)      // two check jobs of transaction t: 12 uint32
{
    H* h = (H*)p;
    for (int q = 0; q < 2; q++) for (int k = 0; k < 3; k++) { segs[6 * q + k] = h->sha[h->J_cap + 2 * t + q].off[k]; segs[6 * q + 3 + k] = h->sha[h->J_cap + 2 * t + q].len[k]; }
}
// sig_ok: T + n_end bytes; check_digests: 2T x 32 bytes (txid, proposal hash per transaction)
void bd_decide(void* p, const uint8_t* sig_ok, const uint8_t* check_digests, uint8_t* flags)
{
    H* h = (H*)p;
    std::vector<uint8_t> dig(32 * (size_t)(h->J_cap + 2 * h->T), 0);
    if (h->T) memcpy(dig.data() + 32 * (size_t)h->J_cap, check_digests, 64 * (size_t)h->T);
    PolicyDev pol; pol.nodes = h->nodes.data(); pol.n_nodes = (int32_t)h->nodes.size() / 4; pol.principal_code = h->principal_code.data(); pol.n_principals = (int32_t)h->principal_code.size();
    pol.ns_blob = h->ns_blob.data(); pol.ns_off = h->ns_off.data(); pol.ns_root = h->ns_root.data(); pol.n_ns = (int32_t)h->ns_root.size();
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
}
// the device DER gate alone
int bd_gate(const uint8_t* sig, uint32_t n, uint8_t* r, uint8_t* s) { return gate_signature(sig, n, r, s) ? 1 : 0; }
int bd_gate_status(const uint8_t* sig, uint32_t n, uint8_t* r, uint8_t* s) { return gate_signature_status(sig, n, r, s); }

}  // extern "C"
