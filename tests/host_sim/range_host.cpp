// TEST HELPER (not product code): the MVCC stage with an ordered key index in the tests' host build -- mvcc_host.cpp's table and argument
// checks, plus the index (stateindex.cuh) and the range steps of the stage (stateset.cuh), run one item at a time in the order the
// library launches them: the written-key list and its merge-sort passes, the range records, the walk, the apply, then the index's
// flag / compact / merge maintenance and the fold.
#include "mvcc_host.cpp"

namespace {

struct RH {
    HS* hs = nullptr;
    bool indexed = false;
    std::vector<IndexEntry> base, delta; std::vector<uint8_t> heap;
    StateIndexDev dev() const
    {
        StateIndexDev d{base.data(), delta.data(), heap.data(), base.size(), delta.size(), indexed ? 1u : 0u};
        return d;
    }
};

// ix_flag -> ix_compact -> ix_merge over sorted candidates whose bytes are at src; then the fold when due
void rh_insert(RH* r, const std::vector<WrittenKey>& cand, const uint8_t* src)
{
    const uint32_t n = (uint32_t)cand.size();
    std::vector<uint32_t> flag(n + 1);
    const StateIndexDev x = r->dev();
    const StateSetDev set = r->hs->dev();
    for (uint32_t i = 0; i < n; i++) ix_flag(i, cand.data(), src, x, set, flag.data());
    uint64_t bytes = 0, m = 0;
    for (uint32_t i = 0; i < n; i++) if (flag[i]) { bytes += cand[i].nl + cand[i].kl; m++; }
    std::vector<IndexEntry> fresh(m + 1);
    unsigned long long at = r->heap.size();
    r->heap.resize(r->heap.size() + bytes);
    uint64_t j = 0;
    for (uint32_t i = 0; i < n; i++)
        if (flag[i]) { ix_emit(cand[i], src, r->heap.data(), at, fresh[j++]); at += cand[i].nl + cand[i].kl; }
    std::vector<IndexEntry> out(r->delta.size() + m + 1);
    for (uint64_t i = 0; i < r->delta.size(); i++) ri_merge_one(r->delta.data(), i, fresh.data(), m, r->heap.data(), out.data(), 0);
    for (uint64_t i = 0; i < m; i++) ri_merge_one(fresh.data(), i, r->delta.data(), r->delta.size(), r->heap.data(), out.data(), 0);
    out.resize(r->delta.size() + m);
    r->delta.swap(out);
    if (r->delta.size() > fabgpu::stateset::index_fold_at(r->base.size())) {
        std::vector<IndexEntry> nb(r->base.size() + r->delta.size() + 1);
        for (uint64_t i = 0; i < r->base.size(); i++) ri_merge_one(r->base.data(), i, r->delta.data(), r->delta.size(), r->heap.data(), nb.data(), 0);
        for (uint64_t i = 0; i < r->delta.size(); i++) ri_merge_one(r->delta.data(), i, r->base.data(), r->base.size(), r->heap.data(), nb.data(), 0);
        nb.resize(r->base.size() + r->delta.size());
        r->base.swap(nb); r->delta.clear();
    }
}

}  // namespace

extern "C" {

void* rh_new(unsigned long long seed) { RH* r = new RH(); r->hs = (HS*)hs_new(seed); return r; }
void rh_free(void* p) { RH* r = (RH*)p; hs_free(r->hs); delete r; }

// mode 0: fabgpu_state_versions_update; 1: fabgpu_state_versions; 2: fabgpu_state_versions_indexed
const char* rh_apply(void* p, int mode, const uint8_t* nb, const uint32_t* no, const uint8_t* cb, const uint32_t* co, const uint8_t* kb,
                     const uint32_t* ko, const uint64_t* ver, size_t n, unsigned long long height, size_t hint, unsigned long long max_bytes, int* failed)
{
    RH* r = (RH*)p;
    const char* err = hs_apply(r->hs, mode != 0, nb, no, cb, co, kb, ko, ver, n, height, hint, max_bytes, failed);
    if (*failed || mode != 0) { r->indexed = false; r->base.clear(); r->delta.clear(); r->heap.clear(); }
    if (err) return err;
    if (mode == 0 && !r->indexed) return nullptr;
    if (mode == 1 || (mode == 2 && !r->hs->installed)) return nullptr;
    std::vector<StateSlot> recs; std::vector<WrittenKey> keys; std::vector<uint8_t> blob;
    fabgpu::stateset::prepare(nb, no, cb, co, kb, ko, ver, n, r->hs->seed, recs);
    fabgpu::stateset::index_keys(nb, no, co, kb, ko, ver, n, recs, keys, blob);
    if (mode == 2) {
        r->indexed = true;
        r->heap = blob;
        r->base.resize(keys.size());
        for (size_t i = 0; i < keys.size(); i++) {
            r->base[i].off = keys[i].ns_off; r->base[i].nl = keys[i].nl; r->base[i].kl = keys[i].kl;
            for (int k = 0; k < 8; k++) r->base[i].w[k] = keys[i].w[k];
        }
        return nullptr;
    }
    rh_insert(r, keys, blob.data());
    return nullptr;
}

void rh_info(void* p, unsigned long long out[4]) { hs_info(((RH*)p)->hs, out); }

// fabgpu_state_index_info
void rh_index_info(void* p, unsigned long long out[3])
{
    RH* r = (RH*)p;
    out[0] = out[1] = out[2] = 0;
    if (!r->indexed) return;
    const StateSetDev set = r->hs->dev();
    for (const auto* v : {&r->base, &r->delta})
        for (const IndexEntry& e : *v) {
            unsigned long long b, t;
            out[0] += sv_lookup(set, e.w, b, t) != SV_EMPTY;
        }
    out[1] = r->base.size() + r->delta.size();
    out[2] = out[1] * sizeof(IndexEntry) + r->heap.size();
}

int rh_lookup(void* p, const uint8_t* ns, uint32_t nl, const uint8_t* coll, uint32_t cl, const uint8_t* key, uint32_t kl, unsigned long long ver[2])
{
    return hs_lookup(((RH*)p)->hs, ns, nl, coll, cl, key, kl, ver);
}

// fabgpu_validate_mvcc over one block, as hs_mvcc, with the range steps while an index is installed
const char* rh_mvcc(void* p, const uint8_t* block, const uint32_t* results, const uint8_t* htype, unsigned long long block_num, const uint8_t* tv,
                    uint8_t* flags, size_t T, unsigned long long max_bytes, int* failed)
{
    RH* r = (RH*)p;
    HS* s = r->hs;
    if (!r->indexed) return hs_mvcc(s, block, results, htype, block_num, tv, flags, T, max_bytes, failed);
    *failed = 0;
    if (s->open) return "the previous block is open: fabgpu_state_versions_update(..., height = block_num + 1) first";
    if (block_num != s->height) return "block_num is not the table's height";
    if (T && (!tv || !flags)) return "flag arrays missing";
    std::vector<TxDev> txs(T);
    for (size_t t = 0; t < T; t++) {
        memset(&txs[t], 0, sizeof(TxDev));
        txs[t].htype = htype[t]; txs[t].endorser_parse_ok = htype[t] == 3; txs[t].results.off = results[2 * t]; txs[t].results.len = results[2 * t + 1];
    }
    uint32_t R_cap = (uint32_t)(4 * T + 16), G_cap = (uint32_t)(T + 1);
    for (;;) {
        std::vector<MvccRec> rec(R_cap); std::vector<uint32_t> fr(T + 1), nr(T + 1), ml(T + 1), fg(T + 1), ng(T + 1); std::vector<uint8_t> info(T + 1);
        std::vector<MvccRange> rng(G_cap);
        uint32_t ctr[8] = {0, 0, UINT32_MAX, 0, 0, 0, 0, 0};
        MvccArrays a; a.rec = rec.data(); a.R_cap = R_cap; a.first_rec = fr.data(); a.n_rec = nr.data(); a.info = info.data(); a.ctr = ctr; a.mlist = ml.data();
        a.indexed = 1; a.block = block_num; a.rng = rng.data(); a.G_cap = G_cap; a.first_rng = fg.data(); a.n_rng = ng.data(); a.ix = r->dev();
        for (uint32_t t = 0; t < T; t++) mv_scan_tx(block, txs[t], t, tv[t], a);
        if (ctr[0] > R_cap || ctr[4] > G_cap) { R_cap = std::max(R_cap, ctr[0]); G_cap = std::max(G_cap, ctr[4]); continue; }
        const uint32_t R = ctr[0], G = ctr[4];
        uint32_t K = 64; while (K < 2 * R) K <<= 1;
        std::vector<MvccKey> key(K);
        memset(key.data(), 0, K * sizeof(MvccKey));
        a.key = key.data(); a.K_size = K;
        const StateSetDev d0 = s->dev();
        for (uint32_t i = 0; i < R; i++) mv_key_rec(i, a, d0);
        for (uint32_t i = 0; i < R; i++) mv_check_rec(i, a);
        std::vector<WrittenKey> wk(R + 1), wk2(R + 1);
        std::vector<MerkleState> mk(G + 1);
        a.mk = mk.data();
        a.wk = wk.data();
        if (!ctr[1]) for (uint32_t k = 0; k < K; k++) mv_written_key(k, a);
        for (uint32_t width = 1; width < R; width <<= 1) {
            for (uint32_t i = 0; i < ctr[5]; i++) ri_sort_one(wk.data(), i, ctr[5], width, block, wk2.data());
            wk.swap(wk2);
        }
        a.wk = wk.data();
        if (!ctr[1]) for (uint32_t q = 0; q < G; q++) mv_range_rec(q, block, a, d0);
        for (uint32_t t = 0; t < T; t++) mv_mark_tx(t, tv, a, flags);
        if (!ctr[1])
            for (uint32_t t = 0; t < T; t++) if (info[t] & MV_MARKED) mv_walk_step<true>(t, tv, a, flags, block, &d0);
        if (!hs_reserve(s, R, 0, max_bytes ? max_bytes : ~0ull)) {
            s->broken = true; s->table.clear(); *failed = 1; r->indexed = false; r->base.clear(); r->delta.clear(); r->heap.clear();
            return "state version table exceeds FABGPU_STATE_MAX_BYTES";
        }
        const StateSetDev d = s->dev();
        int full = 0;
        for (uint32_t k = 0; k < K; k++) mv_apply_key(k, a, flags, d, block_num, &full);
        wk.resize(ctr[5]);
        rh_insert(r, wk, block);
        if (ctr[1] || ctr[2] != UINT32_MAX) s->open = true;
        else s->height = block_num + 1;
        return nullptr;
    }
}

}  // extern "C"
