// TEST HELPER (not product code): the world-state version table and the MVCC stage in the tests' host build -- the library's argument
// checks and key digests (stateset.hpp), the table's upsert, growth and lookup and the stage's six steps (stateset.cuh), run one item at
// a time in the order the library launches them.  The transactions' records come in as TxDev fields (results segment, header type).
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../fabric-mod_b200/csrc/stateset.hpp"

using namespace fabgpu::bdev;

struct HS {
    std::vector<StateSlot> table; unsigned long long count[3] = {0, 0, 0};
    uint64_t seed = 0, height = 0; bool installed = false, broken = false, open = false;
    StateSetDev dev()
    {
        StateSetDev d{table.data(), (uint32_t)(table.size() - 1), broken ? 1u : 0u, seed, count};
        return d;
    }
};

// Grows to hold `more` further claimed slots at a load of at most 1/2 (a rehash drops removed keys); false = over max_bytes
static bool hs_reserve(HS* s, uint64_t more, uint64_t min_slots, uint64_t max_bytes)
{
    if (!s->table.empty() && s->table.size() >= min_slots && s->count[1] + more <= s->table.size() / 2) return true;
    const uint64_t size = std::max(fabgpu::stateset::slots_for(s->count[0] + more, s->table.size()), min_slots);
    if (size * sizeof(StateSlot) > max_bytes) return false;
    std::vector<StateSlot> old(size);
    memset(old.data(), 0, size * sizeof(StateSlot));
    old.swap(s->table);
    s->count[0] = s->count[1] = s->count[2] = 0;
    const StateSetDev d = s->dev();
    for (const StateSlot& o : old)
        if (o.state == SV_PRESENT || o.state == SV_UNKNOWN) sv_upsert(d, o.w, o.state, o.blk, o.txn);
    return true;
}

extern "C" {

void* hs_new(unsigned long long seed) { HS* s = new HS(); s->seed = seed; return s; }
void hs_free(void* p) { delete (HS*)p; }

// replace = 1: fabgpu_state_versions (height, hint); 0: fabgpu_state_versions_update (height).  Null or the refusal / failure text;
// *failed = 1 when the call broke the table.
const char* hs_apply(void* p, int replace, const uint8_t* nb, const uint32_t* no, const uint8_t* cb, const uint32_t* co, const uint8_t* kb,
                     const uint32_t* ko, const uint64_t* ver, size_t n, unsigned long long height, size_t hint, unsigned long long max_bytes, int* failed)
{
    HS* s = (HS*)p;
    *failed = 0;
    std::vector<StateSlot> recs;
    if (const char* err = fabgpu::stateset::prepare(nb, no, cb, co, kb, ko, ver, n, s->seed, recs)) return err;
    const uint64_t cap = max_bytes ? max_bytes : ~0ull;
    uint64_t min_slots = 0;
    if (replace) {
        s->table.clear(); s->count[0] = s->count[1] = s->count[2] = 0; s->installed = s->broken = s->open = false; s->height = 0;
        if (n == 0 && hint == 0) return nullptr;
        s->installed = true; s->height = height;
        min_slots = fabgpu::stateset::slots_for(hint);
        if (min_slots * sizeof(StateSlot) > cap) min_slots = 0;
    } else {
        if (!s->installed) return "no state version table installed: call fabgpu_state_versions first";
        if (s->broken) return "the state version table is broken by a failed call: replace it with fabgpu_state_versions";
        if (height < s->height) return "state version height below the table's height";
    }
    if (!hs_reserve(s, recs.size(), min_slots, cap)) { s->broken = true; s->table.clear(); *failed = 1; return "state version table exceeds FABGPU_STATE_MAX_BYTES"; }
    const StateSetDev d = s->dev();
    for (const StateSlot& r : recs) sv_upsert(d, r.w, r.state, r.blk, r.txn);
    if (!replace && height > s->height) { s->height = height; s->open = false; }
    return nullptr;
}

void hs_info(void* p, unsigned long long out[4])
{
    HS* s = (HS*)p;
    const bool on = s->installed && !s->broken;
    out[0] = on ? s->count[0] : 0; out[1] = s->table.size(); out[2] = s->height; out[3] = on ? s->count[2] : 0;
}

// fabgpu_validate_mvcc over one block: results[2t], results[2t+1] = ChaincodeAction.results of transaction t, htype[t] its header type
// (3 = endorser, reached; anything else: not reached).  Null or the refusal text.
const char* hs_mvcc(void* p, const uint8_t* block, const uint32_t* results, const uint8_t* htype, unsigned long long block_num, const uint8_t* tv,
                    uint8_t* flags, size_t T, unsigned long long max_bytes, int* failed)
{
    HS* s = (HS*)p;
    *failed = 0;
    if (!s->installed) return "no state version table installed: call fabgpu_state_versions first";
    if (s->open) return "the previous block is open: fabgpu_state_versions_update(..., height = block_num + 1) first";
    if (block_num != s->height) return "block_num is not the table's height";
    if (T && (!tv || !flags)) return "flag arrays missing";
    if (s->broken) {
        for (size_t t = 0; t < T; t++) flags[t] = tv[t] == TXC_VALID ? TXC_NOT_VALIDATED : tv[t];
        return nullptr;
    }
    std::vector<TxDev> txs(T);
    for (size_t t = 0; t < T; t++) {
        memset(&txs[t], 0, sizeof(TxDev));
        txs[t].htype = htype[t]; txs[t].endorser_parse_ok = htype[t] == 3; txs[t].results.off = results[2 * t]; txs[t].results.len = results[2 * t + 1];
    }
    uint32_t R_cap = (uint32_t)(4 * T + 16);
    for (;;) {
        std::vector<MvccRec> rec(R_cap); std::vector<uint32_t> fr(T + 1), nr(T + 1), ml(T + 1); std::vector<uint8_t> info(T + 1);
        uint32_t ctr[4] = {0, 0, UINT32_MAX, 0};
        MvccArrays a; a.rec = rec.data(); a.R_cap = R_cap; a.first_rec = fr.data(); a.n_rec = nr.data(); a.info = info.data(); a.ctr = ctr; a.mlist = ml.data();
        for (uint32_t t = 0; t < T; t++) mv_scan_tx(block, txs[t], t, tv[t], a);
        if (ctr[0] > R_cap) { R_cap = ctr[0]; continue; }
        const uint32_t R = ctr[0];
        uint32_t K = 64; while (K < 2 * R) K <<= 1;
        std::vector<MvccKey> key(K);
        memset(key.data(), 0, K * sizeof(MvccKey));
        a.key = key.data(); a.K_size = K;
        const StateSetDev d0 = s->dev();
        for (uint32_t i = 0; i < R; i++) mv_key_rec(i, a, d0);
        for (uint32_t i = 0; i < R; i++) mv_check_rec(i, a);
        for (uint32_t t = 0; t < T; t++) mv_mark_tx(t, tv, a, flags);
        if (!ctr[1])
            for (uint32_t t = 0; t < T; t++) if (info[t] & MV_MARKED) mv_walk_step(t, tv, a, flags);
        if (!hs_reserve(s, R, 0, max_bytes ? max_bytes : ~0ull)) { s->broken = true; s->table.clear(); *failed = 1; return "state version table exceeds FABGPU_STATE_MAX_BYTES"; }
        const StateSetDev d = s->dev();
        int full = 0;
        for (uint32_t k = 0; k < K; k++) mv_apply_key(k, a, flags, d, block_num, &full);
        if (ctr[1] || ctr[2] != UINT32_MAX) s->open = true;
        else s->height = block_num + 1;
        return nullptr;
    }
}

// the state of one key (SV_*), its version in ver[2]
int hs_lookup(void* p, const uint8_t* ns, uint32_t nl, const uint8_t* coll, uint32_t cl, const uint8_t* key, uint32_t kl, unsigned long long ver[2])
{
    HS* s = (HS*)p;
    if (!s->installed || s->table.empty()) return -1;
    uint32_t w[8];
    sv_key(ns, nl, coll, cl, key, kl, w);
    return (int)sv_lookup(s->dev(), w, ver[0], ver[1]);
}

}  // extern "C"
