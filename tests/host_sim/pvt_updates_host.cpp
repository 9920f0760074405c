// TEST HELPER (not product code): the private update batch (pvtupdates.cuh) in the tests' host build -- mvcc_host.cpp's table and
// stage, the hashed batch's steps (updates.cuh), the private-data check's steps (pvtdata.cuh), then the private batch's steps one item
// at a time in the order fabgpu_block_pvt_updates launches them.  Built as a library, or with PU_MAIN as a program for AddressSanitizer /
// UndefinedBehaviorSanitizer runs over a corpus of mutated private data.
#include "updates_host.cpp"
#include "pvt_host.cpp"
#include "../../fabric-mod_b200/csrc/pvtupdates.cuh"

extern "C" {

// hs_mvcc, the hashed batch, the check with the stage's flags, and the private batch.  flags: T; hrec: the hashed records (UD_WORDS
// each, at most hcap; n_h their count); status / out as fabgpu_validate_pvtdata; rec: PU_WORDS each, at most rec_cap; n_out the full
// count; *complete as fabgpu_block_pvt_updates gives it.  Null or the refusal text.
const char* pu_host(void* p, const uint8_t* block, const uint32_t* results, const uint8_t* htype, unsigned long long block_num, const uint8_t* tv,
                    uint8_t* flags, size_t T, uint32_t* hrec, size_t hcap, size_t* n_h, const uint8_t* pvt, const uint32_t* off, const uint32_t* seq,
                    size_t n_pvt, int32_t* status, int32_t* out, uint32_t* rec, size_t rec_cap, size_t* n_out, int* complete)
{
    HS* s = (HS*)p;
    *n_h = 0; *n_out = 0; *complete = 0;
    if (!s->installed) return "no state version table installed: call fabgpu_state_versions first";
    if (s->open) return "the previous block is open: fabgpu_state_versions_update(..., height = block_num + 1) first";
    if (block_num != s->height) return "block_num is not the table's height";
    bool incomplete = false;
    std::vector<TxDev> txs(T + 1);
    for (size_t t = 0; t < T; t++) {
        memset(&txs[t], 0, sizeof(TxDev));
        txs[t].htype = htype[t]; txs[t].endorser_parse_ok = htype[t] == 3; txs[t].results.off = results[2 * t]; txs[t].results.len = results[2 * t + 1];
    }
    // the stage (hs_updates' steps, its arrays kept)
    std::vector<MvccRec> mrec; std::vector<uint32_t> fr(T + 1), nr(T + 1), ml(T + 1); std::vector<uint8_t> info(T + 1);
    uint32_t ctr[4] = {0, 0, UINT32_MAX, 0}, R = 0, K = 0;
    MvccArrays a;
    std::vector<MvccKey> key;
    if (s->broken) {
        for (size_t t = 0; t < T; t++) flags[t] = tv[t] == TXC_VALID ? TXC_NOT_VALIDATED : tv[t];
        incomplete = true;
    } else {
        uint32_t R_cap = (uint32_t)(4 * T + 16);
        for (;;) {
            mrec.assign(R_cap, MvccRec());
            ctr[0] = 0; ctr[1] = 0; ctr[2] = UINT32_MAX; ctr[3] = 0;
            a.rec = mrec.data(); a.R_cap = R_cap; a.first_rec = fr.data(); a.n_rec = nr.data(); a.info = info.data(); a.ctr = ctr; a.mlist = ml.data();
            for (uint32_t t = 0; t < T; t++) mv_scan_tx(block, txs[t], t, tv[t], a);
            if (ctr[0] <= R_cap) break;
            R_cap = ctr[0];
        }
        R = ctr[0];
        K = 64; while (K < 2 * R) K <<= 1;
        key.assign(K, MvccKey());
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
        incomplete = open || (T && memchr(flags, TXC_NOT_VALIDATED, T));
    }
    // the hashed batch
    uint32_t H = 0;
    std::vector<UdPair> pair; std::vector<UdKey> uk; std::vector<uint32_t> base(T + 1), mark, okey, omoff; std::vector<uint8_t> need, txneed(T + 1);
    std::vector<UdSeg> seg;
    if (!incomplete && R) {
        uint32_t P = 64; while (P < 2 * R) P <<= 1;
        pair.assign(P, UdPair()); uk.assign(K, UdKey()); mark.assign(R, 0); okey.assign(R, 0); omoff.assign(R, 0); need.assign(R, 0); seg.assign(R, UdSeg());
        memset(pair.data(), 0, P * sizeof(UdPair)); memset(uk.data(), 0, K * sizeof(UdKey)); memset(seg.data(), 0, R * sizeof(UdSeg));
        uint32_t uctr[3] = {0, 0, 0};
        UdArrays u;
        u.rec = mrec.data(); u.first_rec = fr.data(); u.n_rec = nr.data(); u.flags = flags; u.R = R; u.T = (uint32_t)T; u.K = K;
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
        if (uctr[0]) incomplete = true;
        else {
            uctr[1] = n; uctr[2] = mb;
            std::vector<uint32_t> words((size_t)n * UD_WORDS + 1); std::vector<uint8_t> meta(mb + 1);
            u.out = words.data(); u.meta = meta.data();
            for (uint32_t o = 0; o < n; o++) ud_emit(o, block, u);
            H = n; *n_h = n;
            if (std::min<size_t>(n, hcap)) memcpy(hrec, words.data(), std::min<size_t>(n, hcap) * UD_WORDS * 4);
        }
    }
    // the check, with the stage's flags (pv_host's steps, its arrays kept)
    out[0] = PV_OK; out[1] = out[2] = out[3] = -1;
    const uint32_t E = (uint32_t)n_pvt;
    std::vector<uint8_t> ent(E + 1);
    std::vector<uint32_t> first(E + 1), nrec(E + 1);
    uint32_t R_cap = 0, pctr[4];
    std::vector<PvRec> prec; std::vector<ShaJobP> jobs; std::vector<uint8_t> dig;
    unsigned long long verdict = ~0ull;
    PvArrays pa;
    pa.pvt = pvt; pa.off = off; pa.seq = seq; pa.n_pvt = E; pa.flags = flags; pa.ent = ent.data(); pa.first = first.data(); pa.n_rec = nrec.data();
    pa.ctr = pctr; pa.status = status; pa.verdict = &verdict;
    if (E) {
        for (;;) {
            prec.resize(R_cap + 1); jobs.resize(R_cap + 1); dig.resize(32 * (R_cap + 1));
            pa.rec = prec.data(); pa.R_cap = R_cap; pa.jobs = jobs.data(); pa.dig = dig.data();
            pctr[0] = 0;
            for (uint32_t e = 0; e < E; e++) pv_scan_entry(block, txs.data(), e, pa);
            if (pctr[0] <= R_cap) break;
            R_cap = pctr[0];
        }
        for (uint32_t i = 0; i < pctr[0]; i++) sha256(pvt + jobs[i].off[0], jobs[i].len[0], dig.data() + 32 * (size_t)i);
        for (uint32_t i = 0; i < pctr[0]; i++) pv_check_rec(block, txs.data(), i, pa);
        for (uint32_t e = 0; e < E; e++) pv_verdict_entry(e, pa);
        if (verdict != ~0ull) {
            const uint32_t e = (uint32_t)verdict, sq = (uint32_t)(verdict >> 32);
            const int32_t* es = status + 3 * (size_t)e;
            const bool mismatch = es[0] == PV_MISMATCH && flags[sq] == TXC_VALID;
            out[0] = mismatch ? PV_MISMATCH : PV_UNDET; out[1] = (int32_t)sq;
            out[2] = mismatch ? es[1] : -1; out[3] = mismatch ? es[2] : -1;
        }
    }
    if (incomplete || out[0] != PV_OK) return nullptr;
    if (E == 0) { *complete = 1; return nullptr; }
    // the private batch, with pvu_build's rerun on overflow (first sized for one write and no metadata write in all)
    uint32_t uctr2[5];
    std::vector<uint32_t> wfirst(E + 1), mfirst(E + 1), tbase(T + 1);
    std::vector<PuItem> item, meta; std::vector<ShaJobP> mjobs; std::vector<uint8_t> mdig;
    PuArrays b;
    b.pvt = pvt; b.seq = seq; b.n_pvt = E; b.T = (uint32_t)T; b.flags = flags; b.status = status; b.rec = prec.data(); b.first = first.data();
    b.n_rec = nrec.data(); b.wfirst = wfirst.data(); b.mfirst = mfirst.data(); b.tbase = tbase.data(); b.ctr = uctr2; b.seed = 0x1234;
    b.stage_seed = s->seed; b.stage.key = H ? key.data() : nullptr; b.stage.K_size = H ? K : 0;
    b.ukey = H ? uk.data() : nullptr; b.useg = H ? seg.data() : nullptr; b.uokey = H ? okey.data() : nullptr; b.n_h = H; b.blk = block;
    uint32_t W_cap = 1, M_cap = 0;
    for (;;) {
        item.assign(W_cap + 1, PuItem()); meta.assign(M_cap + 1, PuItem()); mjobs.assign(M_cap + 1, ShaJobP()); mdig.assign(32 * (M_cap + 1), 0);
        b.item = item.data(); b.W_cap = W_cap; b.meta = meta.data(); b.M_cap = M_cap; b.jobs = mjobs.data(); b.dig = mdig.data();
        std::fill(tbase.begin(), tbase.end(), 0u);
        for (int i = 0; i < 5; i++) uctr2[i] = 0;
        for (uint32_t e = 0; e < E; e++) pu_list_entry(e, b);
        if (uctr2[0] <= W_cap && uctr2[1] <= M_cap) break;
        W_cap = std::max(W_cap, uctr2[0]); M_cap = std::max(M_cap, uctr2[1]);
    }
    if (uctr2[2]) return nullptr;
    const uint32_t W = uctr2[0], M = uctr2[1];
    uint32_t P = 64; while (P < 2 * (W + M)) P <<= 1;
    std::vector<PuKey> pk(P); std::vector<uint32_t> pmark(W + 1, 0), rmark(K + 1, 0), pokey(W + H + 1);
    memset(pk.data(), 0, P * sizeof(PuKey));
    b.key = pk.data(); b.P_size = P; b.mark = pmark.data(); b.rmark = rmark.data(); b.out_key = pokey.data();
    for (uint32_t m = 0; m < M; m++) sha256(pvt + mjobs[m].off[0], mjobs[m].len[0], mdig.data() + 32 * (size_t)m);
    pu_base_host(b);
    for (uint32_t i = 0; i < W + M; i++) pu_key_item(i, W, b);
    for (uint32_t i = 0; i < W + M; i++) pu_first_item(i, W, b);
    for (uint32_t m = 0; m < M; m++) pu_renew_meta(m, b);
    for (uint32_t m = 0; m < M; m++) sha256(pvt + mjobs[m].off[0], mjobs[m].len[0], mdig.data() + 32 * (size_t)m);
    for (uint32_t q = 0; q < P; q++) pu_mark_key(q, b);
    uint32_t n1 = 0, n2 = 0;
    for (uint32_t q = 0; q < W; q++) if (pmark[q]) pokey[n1++] = pmark[q] - 1;
    for (uint32_t h = 0; h < H; h++) if (rmark[okey[h]]) pokey[n1 + n2++] = h;
    uctr2[3] = n1; uctr2[4] = n2;
    if (uctr2[2]) return nullptr;
    std::vector<uint32_t> words((size_t)(n1 + n2) * PU_WORDS + 1);
    b.out = words.data();
    for (uint32_t o = 0; o < n1 + n2; o++) pu_emit(o, b);
    *complete = 1; *n_out = n1 + n2;
    if (std::min<size_t>(n1 + n2, rec_cap)) memcpy(rec, words.data(), std::min<size_t>(n1 + n2, rec_cap) * PU_WORDS * 4);
    return nullptr;
}

}  // extern "C"

#ifdef PU_MAIN
// Corpus (little-endian u32): n_blocks; per block T, per transaction (htype | tv << 8) and a length-prefixed TxReadWriteSet, then n_pvt
// and per entry seq and a length-prefixed TxPvtReadWriteSet.  The table starts empty at height 1.  Every buffer is allocated at its
// exact length.  Prints one line per block: the verdict, whether the batch is complete and its record count.
int main(int argc, char** argv)
{
    if (argc < 2) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<uint8_t> all;
    uint8_t buf[65536]; size_t k;
    while ((k = fread(buf, 1, sizeof buf, f)) > 0) all.insert(all.end(), buf, buf + k);
    fclose(f);
    size_t p = 0;
    auto u32 = [&]() { uint32_t v = 0; if (p + 4 <= all.size()) memcpy(&v, all.data() + p, 4); p += 4; return v; };
    void* s = hs_new(7);
    int failed = 0;
    uint32_t z[2] = {0, 0}; uint8_t zb[1] = {0}; uint64_t zv[2] = {0, 0};
    hs_apply(s, 1, zb, z, zb, z, zb, z, zv, 0, 1, 64, 0, &failed);
    unsigned long long height = 1;
    const uint32_t nb = u32();
    for (uint32_t bi = 0; bi < nb && p < all.size(); bi++) {
        const uint32_t T = u32();
        std::vector<uint8_t> blob, htype(T + 1), tv(T + 1), flags(T + 1);
        std::vector<uint32_t> results(2 * T + 2);
        for (uint32_t t = 0; t < T; t++) {
            const uint32_t hf = u32(), len = u32();
            htype[t] = (uint8_t)hf; tv[t] = (uint8_t)(hf >> 8);
            results[2 * t] = (uint32_t)blob.size(); results[2 * t + 1] = len;
            blob.insert(blob.end(), all.begin() + p, all.begin() + p + len); p += len;
        }
        const uint32_t E = u32();
        std::vector<uint8_t> pb;
        std::vector<uint32_t> off(E + 1, 0), seq(E + 1);
        for (uint32_t e = 0; e < E; e++) {
            seq[e] = u32(); const uint32_t len = u32();
            pb.insert(pb.end(), all.begin() + p, all.begin() + p + len); p += len;
            off[e + 1] = (uint32_t)pb.size();
        }
        uint8_t* blk = new uint8_t[blob.size() ? blob.size() : 1];
        uint8_t* pv = new uint8_t[pb.size() ? pb.size() : 1];
        if (!blob.empty()) memcpy(blk, blob.data(), blob.size());
        if (!pb.empty()) memcpy(pv, pb.data(), pb.size());
        std::vector<int32_t> status(3 * (size_t)E + 3);
        std::vector<uint32_t> hrec(4096 * UD_WORDS), rec(4096 * PU_WORDS);
        int32_t out[4]; size_t n_h = 0, n_out = 0; int complete = 0;
        if (((HS*)s)->open) hs_apply(s, 0, zb, z, zb, z, zb, z, zv, 0, ++height, 0, 0, &failed);
        const char* err = pu_host(s, blk, results.data(), htype.data(), height, tv.data(), flags.data(), T, hrec.data(), 4096, &n_h, pv, off.data(),
                                  seq.data(), E, status.data(), out, rec.data(), 4096, &n_out, &complete);
        if (err) printf("refused %s\n", err);
        else {
            if (!((HS*)s)->open) height++;
            printf("%d %d %d %d complete %d records %zu\n", out[0], out[1], out[2], out[3], complete, n_out);
        }
        delete[] blk; delete[] pv;
    }
    hs_free(s);
    return 0;
}
#endif
