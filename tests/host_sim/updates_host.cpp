// TEST HELPER (not product code): the update batch (updates.cuh) in the tests' host build -- mvcc_host.cpp's table and stage, then the
// batch's steps one item at a time in the order fabgpu_block_updates launches them.  Built as a library of its own, or with
// UPDATES_MAIN as a program for AddressSanitizer / UndefinedBehaviorSanitizer runs over a corpus of mutated read/write sets.
#include "mvcc_host.cpp"
#include "../../fabric-mod_b200/csrc/updates.cuh"

extern "C" {

// hs_mvcc, then the batch: records (UD_WORDS words each, at most rec_cap) and metadata bytes (at most meta_cap); n_out = full counts,
// *complete as fabgpu_block_updates gives it.  Null or the refusal text.
const char* hs_updates(void* p, const uint8_t* block, const uint32_t* results, const uint8_t* htype, unsigned long long block_num, const uint8_t* tv,
                       uint8_t* flags, size_t T, uint32_t* out_rec, size_t rec_cap, uint8_t* out_meta, size_t meta_cap, size_t n_out[2], int* complete)
{
    HS* s = (HS*)p;
    n_out[0] = n_out[1] = 0; *complete = 0;
    if (!s->installed) return "no state version table installed: call fabgpu_state_versions first";
    if (s->open) return "the previous block is open: fabgpu_state_versions_update(..., height = block_num + 1) first";
    if (block_num != s->height) return "block_num is not the table's height";
    if (s->broken) {
        for (size_t t = 0; t < T; t++) flags[t] = tv[t] == TXC_VALID ? TXC_NOT_VALIDATED : tv[t];
        return nullptr;
    }
    std::vector<TxDev> txs(T + 1);
    for (size_t t = 0; t < T; t++) {
        memset(&txs[t], 0, sizeof(TxDev));
        txs[t].htype = htype[t]; txs[t].endorser_parse_ok = htype[t] == 3; txs[t].results.off = results[2 * t]; txs[t].results.len = results[2 * t + 1];
    }
    uint32_t R_cap = (uint32_t)(4 * T + 16);
    std::vector<MvccRec> rec; std::vector<uint32_t> fr(T + 1), nr(T + 1), ml(T + 1); std::vector<uint8_t> info(T + 1);
    uint32_t ctr[4];
    MvccArrays a;
    for (;;) {
        rec.assign(R_cap, MvccRec());
        ctr[0] = 0; ctr[1] = 0; ctr[2] = UINT32_MAX; ctr[3] = 0;
        a.rec = rec.data(); a.R_cap = R_cap; a.first_rec = fr.data(); a.n_rec = nr.data(); a.info = info.data(); a.ctr = ctr; a.mlist = ml.data();
        for (uint32_t t = 0; t < T; t++) mv_scan_tx(block, txs[t], t, tv[t], a);
        if (ctr[0] <= R_cap) break;
        R_cap = ctr[0];
    }
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
    if (!hs_reserve(s, R, 0, ~0ull)) { s->broken = true; s->table.clear(); return "state version table exceeds FABGPU_STATE_MAX_BYTES"; }
    const StateSetDev d = s->dev();
    int full = 0;
    for (uint32_t k = 0; k < K; k++) mv_apply_key(k, a, flags, d, block_num, &full);
    const bool open = ctr[1] || ctr[2] != UINT32_MAX;
    if (open) s->open = true;
    else s->height = block_num + 1;
    // the batch
    if (open || (T && memchr(flags, TXC_NOT_VALIDATED, T))) return nullptr;
    *complete = 1;
    if (R == 0) return nullptr;
    uint32_t P = 64; while (P < 2 * R) P <<= 1;
    std::vector<UdPair> pair(P); std::vector<UdKey> uk(K); std::vector<uint32_t> base(T + 1), mark(R), okey(R), omoff(R); std::vector<uint8_t> need(R), txneed(T + 1);
    std::vector<UdSeg> seg(R);
    memset(pair.data(), 0, P * sizeof(UdPair)); memset(uk.data(), 0, K * sizeof(UdKey)); memset(seg.data(), 0, R * sizeof(UdSeg));
    uint32_t uctr[3] = {0, 0, 0};
    UdArrays u;
    u.rec = rec.data(); u.first_rec = fr.data(); u.n_rec = nr.data(); u.flags = flags; u.R = R; u.T = (uint32_t)T; u.K = K;
    u.pair = pair.data(); u.P_size = P; u.key = uk.data(); u.base = base.data(); u.mark = mark.data(); u.need = need.data(); u.txneed = txneed.data();
    u.seg = seg.data(); u.out_key = okey.data(); u.out_moff = omoff.data(); u.out = nullptr; u.meta = nullptr; u.ctr = uctr;
    for (uint32_t i = 0; i < R; i++) ud_pair_rec(i, u);
    for (uint32_t q = 0; q < P; q++) ud_class_pair(q, u);
    for (uint32_t q = 0; q < P; q++) ud_walk_pair(q, u);
    ud_base_host(u);
    for (uint32_t k = 0; k < K; k++) ud_resolve_key(k, u);
    for (uint32_t t = 0; t < T; t++) ud_seg_tx(t, block, txs[t], u);
    uint32_t n = 0, mb = 0, k = 0, b = 0;
    for (uint32_t pos = 0; pos < R; pos++)
        if (ud_at(pos, u, k, b)) { okey[n] = k; omoff[n] = mb; n++; mb += b; }
    if (uctr[0]) { *complete = 0; return nullptr; }
    uctr[1] = n; uctr[2] = mb;
    std::vector<uint32_t> words((size_t)n * UD_WORDS + 1); std::vector<uint8_t> meta(mb + 1);
    u.out = words.data(); u.meta = meta.data();
    for (uint32_t o = 0; o < n; o++) ud_emit(o, block, u);
    n_out[0] = n; n_out[1] = mb;
    if (std::min<size_t>(n, rec_cap)) memcpy(out_rec, words.data(), std::min<size_t>(n, rec_cap) * UD_WORDS * 4);
    if (std::min<size_t>(mb, meta_cap)) memcpy(out_meta, meta.data(), std::min<size_t>(mb, meta_cap));
    return nullptr;
}

}  // extern "C"

#ifdef UPDATES_MAIN
// Corpus (little-endian u32): n_blocks, then per block T and per transaction (htype u8, tv u8, len, read/write set bytes); the table
// starts empty at height 1.  Prints one line per block: the flags and the batch's counts.
#include <stdio.h>
#include <string>

int main(int argc, char** argv)
{
    if (argc < 2) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    std::string g; char buf[65536]; size_t r;
    while ((r = fread(buf, 1, sizeof buf, f)) > 0) g.append(buf, r);
    fclose(f);
    size_t pos = 0;
    auto u32 = [&]() { uint32_t v = 0; if (pos + 4 <= g.size()) memcpy(&v, g.data() + pos, 4); pos += 4; return v; };
    void* s = hs_new(7);
    int failed = 0;
    uint32_t z[2] = {0, 0}; uint8_t zb[1] = {0}; uint64_t zv[2] = {0, 0};
    hs_apply(s, 1, zb, z, zb, z, zb, z, zv, 0, 1, 64, 0, &failed);
    const uint32_t nb = u32();
    unsigned long long height = 1;
    size_t complete_n = 0;
    for (uint32_t b = 0; b < nb && pos < g.size(); b++) {
        const uint32_t T = u32();
        std::vector<uint8_t> tv(T + 1), ht(T + 1), flags(T + 1); std::vector<uint32_t> res(2 * T + 2); std::string blob;
        for (uint32_t t = 0; t < T; t++) {
            const uint32_t h = u32(), len = u32();
            ht[t] = (uint8_t)(h & 0xff); tv[t] = (uint8_t)(h >> 8);
            res[2 * t] = (uint32_t)blob.size() + 8; res[2 * t + 1] = len;
            blob += std::string(8, '\0') + g.substr(std::min(pos, g.size()), len); pos += len;
        }
        blob += std::string(64, '\0');
        std::vector<uint8_t> bb(blob.begin(), blob.end());
        std::vector<uint32_t> rec(4096 * UD_WORDS); std::vector<uint8_t> meta(65536);
        size_t n_out[2]; int complete = 0;
        if (((HS*)s)->open) hs_apply(s, 0, zb, z, zb, z, zb, z, zv, 0, ++height, 0, 0, &failed);
        const char* err = hs_updates(s, bb.data(), res.data(), ht.data(), height, tv.data(), flags.data(), T, rec.data(), 4096, meta.data(), meta.size(), n_out, &complete);
        if (err) { printf("refused %s\n", err); continue; }
        if (!((HS*)s)->open) height++;
        complete_n += complete;
        printf("block %u complete %d records %zu bytes %zu\n", b, complete, n_out[0], n_out[1]);
    }
    printf("done %u blocks, %zu complete\n", nb, complete_n);
    hs_free(s);
    return 0;
}
#endif
