// TEST HELPER (not product code): the MVCC stage under CouchDB in the tests' host build -- range_host.cpp's stage and index, with the
// key refusals of fabgpu_state_versions* and the key and value pre-pass (couchval.cuh) run one item at a time in the order the library
// launches them: the write scan (counting first, then again once the arrays hold its writes), the per-write check, the per-transaction flag.
#include "range_host.cpp"
#include "../../fabric-mod_b200/csrc/couchval.cuh"

namespace {

struct CH { RH* rh = nullptr; bool couch = false; };

// cv_scan_tx -> cv_check_write -> the long values -> cv_flag_tx over the block, rewriting tv
void ch_prepass(const uint8_t* block, const uint32_t* results, const uint8_t* htype, uint8_t* tv, size_t T)
{
    std::vector<TxDev> txs(T);
    for (size_t t = 0; t < T; t++) {
        memset(&txs[t], 0, sizeof(TxDev));
        txs[t].htype = htype[t]; txs[t].endorser_parse_ok = htype[t] == 3; txs[t].results.off = results[2 * t]; txs[t].results.len = results[2 * t + 1];
    }
    uint32_t W_cap = 0;
    for (;;) {
        std::vector<CvWrite> w(W_cap + 1); std::vector<uint32_t> fw(T + 1), nw(T + 1), lng(W_cap + 1); std::vector<uint8_t> und(T + 1), code(W_cap + 1);
        uint32_t ctr[2] = {0, 0};
        CvArrays a; a.w = w.data(); a.W_cap = W_cap; a.first_w = fw.data(); a.n_w = nw.data(); a.undet = und.data(); a.code = code.data();
        a.lng = lng.data(); a.ctr = ctr;
        for (uint32_t t = 0; t < T; t++) cv_scan_tx(block, txs[t], t, tv[t], a);
        if (ctr[0] > W_cap) { W_cap = ctr[0]; continue; }
        for (uint32_t i = 0; i < ctr[0]; i++) cv_check_write(i, block, a);
        for (uint32_t k = 0; k < ctr[1]; k++) { const CvWrite& x = w[lng[k]]; code[lng[k]] = cv_code(cv_long_host(block + x.val.off, x.val.len)); }
        for (uint32_t t = 0; t < T; t++) cv_flag_tx(t, a, tv);
        return;
    }
}

}  // namespace

extern "C" {

void* ch_new(unsigned long long seed) { CH* c = new CH(); c->rh = (RH*)rh_new(seed); return c; }
void ch_free(void* p) { CH* c = (CH*)p; rh_free(c->rh); delete c; }
void* ch_range(void* p) { return ((CH*)p)->rh; }

// fabgpu_state_database
int ch_database(void* p, int kind)
{
    if (kind != 0 && kind != 1) return -3;
    ((CH*)p)->couch = kind == 1;
    return 0;
}

// rh_apply, with fabgpu_state_versions*'s refusal of versions for public keys CouchDB cannot hold (removals pass)
const char* ch_apply(void* p, int mode, const uint8_t* nb, const uint32_t* no, const uint8_t* cb, const uint32_t* co, const uint8_t* kb,
                     const uint32_t* ko, const uint64_t* ver, size_t n, unsigned long long height, size_t hint, unsigned long long max_bytes, int* failed)
{
    CH* c = (CH*)p;
    *failed = 0;
    std::vector<StateSlot> recs;
    if (const char* err = fabgpu::stateset::prepare(nb, no, cb, co, kb, ko, ver, n, c->rh->hs->seed, recs)) return err;
    if (c->couch)
        for (size_t i = 0; i < n; i++)
            if (co[i + 1] == co[i] && !(ver[2 * i] == UINT64_MAX && ver[2 * i + 1] == UINT64_MAX) && !cv_key_ok(kb + ko[i], ko[i + 1] - ko[i]))
                return "a public key CouchDB cannot hold";
    return rh_apply(c->rh, mode, nb, no, cb, co, kb, ko, ver, n, height, hint, max_bytes, failed);
}

// fabgpu_validate_mvcc: the pre-pass under CouchDB (on a table that can decide), then rh_mvcc over the rewritten flags
const char* ch_mvcc(void* p, const uint8_t* block, const uint32_t* results, const uint8_t* htype, unsigned long long block_num, const uint8_t* tv,
                    uint8_t* flags, size_t T, unsigned long long max_bytes, int* failed)
{
    CH* c = (CH*)p;
    std::vector<uint8_t> tv2(tv, tv + T);
    tv2.push_back(0);
    const HS* s = c->rh->hs;
    if (c->couch && s->installed && !s->broken && !s->open && block_num == s->height) ch_prepass(block, results, htype, tv2.data(), T);
    return rh_mvcc(c->rh, block, results, htype, block_num, tv2.data(), flags, T, max_bytes, failed);
}

// The verdict bits of each value (blob with n + 1 offsets); path as fabgpu_test_couch_values: 0 by length, 1 one thread, 2 one CTA
void ch_values(const uint8_t* blob, const uint32_t* off, size_t n, int path, uint32_t* out)
{
    for (size_t i = 0; i < n; i++) {
        const uint32_t len = off[i + 1] - off[i];
        out[i] = cv_test_long(path, len) ? cv_long_host(blob + off[i], len) : cv_short(blob + off[i], len);
    }
}

}  // extern "C"
